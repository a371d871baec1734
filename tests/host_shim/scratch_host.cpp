// Test infrastructure: csrc/amwg_summary_scratch.h (select_device and the per-device scratch pool of the summary entry points)
// compiled for the HOST against stub cudaMalloc / cudaFree / cudaSetDevice that count their calls, for
// tests/test_summary_scratch_host.py. The stub allocator hands out 256-byte-aligned host memory, as cudaMalloc does.
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <mutex>
#include <string>
#include <thread>

typedef int cudaError_t;
static const cudaError_t cudaSuccess = 0;
static const cudaError_t cudaErrorMemoryAllocation = 2;

static int g_mallocs = 0, g_frees = 0, g_set_devices = 0, g_last_device = -1;
static bool g_fail_next_malloc = false;

static cudaError_t cudaMalloc(void** p, size_t n) {
  ++g_mallocs;
  if (g_fail_next_malloc) { g_fail_next_malloc = false; return cudaErrorMemoryAllocation; }
  *p = std::aligned_alloc(256, (n + 255) / 256 * 256);
  return cudaSuccess;
}
static cudaError_t cudaFree(void* p) { ++g_frees; std::free(p); return cudaSuccess; }
static cudaError_t cudaSetDevice(int d) { ++g_set_devices; g_last_device = d; return cudaSuccess; }
static const char* cudaGetErrorString(cudaError_t e) { return e == cudaErrorMemoryAllocation ? "out of memory" : "stub error"; }

// as amwg_kernels.cu defines them ahead of the header
static std::string g_last_error;
static int fail(const std::string& msg) { g_last_error = msg; return -1; }
#define CUDA_TRY(expr)                                                                                 \
  do {                                                                                                 \
    cudaError_t _e = (expr);                                                                           \
    if (_e != cudaSuccess) return fail(std::string(#expr) + ": " + cudaGetErrorString(_e));           \
  } while (0)

#define private public          // the test reads a pool's size and tries its lock
#include "amwg_summary_scratch.h"
#undef private

using summary::Scratch;

extern "C" {

const char* hs_last_error() { return g_last_error.c_str(); }
void hs_fail_next_malloc() { g_fail_next_malloc = true; }

// counts[4] = { cudaMalloc, cudaFree, cudaSetDevice calls, the last device set }
void hs_counts(long long* counts) {
  counts[0] = g_mallocs; counts[1] = g_frees; counts[2] = g_set_devices; counts[3] = g_last_device;
}

int hs_select_device(int device) { return summary::select_device(device, "hs_select_device"); }

long long hs_pool_bytes(int device) { return (long long)Scratch::pools()[device].bytes; }

// One lease of the four parts sizes[0 .. 4) on `device`, released on return; ptrs[i] = the address of part i.
int hs_acquire(int device, const long long* sizes, unsigned long long* ptrs) {
  Scratch sc;
  if (sc.acquire(device, "hs_acquire", {(size_t)sizes[0], (size_t)sizes[1], (size_t)sizes[2], (size_t)sizes[3]})) return -1;
  for (int i = 0; i < 4; ++i) ptrs[i] = (unsigned long long)(uintptr_t)sc.part<char>(i);
  return 0;
}

// While a lease on `held` is alive, another thread tries the lock of `probe`'s pool: 1 when it got it, 0 when it did not, -1
// when the lease could not be taken.
int hs_try_lock_while_held(int held, int probe) {
  Scratch sc;
  if (sc.acquire(held, "hs_try_lock_while_held", {64})) return -1;
  int got = -1;
  std::thread t([&] {
    std::mutex& mu = Scratch::pools()[probe].mu;
    got = mu.try_lock() ? 1 : 0;
    if (got) mu.unlock();
  });
  t.join();
  return got;
}

}  // extern "C"
