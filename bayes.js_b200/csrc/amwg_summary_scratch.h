// Host side shared by the summary entry points (amwg_summary*.cuh): the device prologue and the device scratch. Host code only, so
// that tests/test_summary_scratch_host.py can compile it with g++ against stub CUDA calls. Included by amwg_kernels.cu after
// fail() and CUDA_TRY, ahead of the summary headers.
#pragma once

#include <cstddef>
#include <initializer_list>
#include <mutex>
#include <string>

namespace summary {

constexpr int kMaxDevices = 64;       // device indices with a scratch pool

// The prologue of every entry point that takes a device index: the index is checked before CUDA sees it, so an out-of-range one
// is refused in the entry's own words and never indexes the pools.
inline int select_device(int device, const char* who) {
  if (device < 0 || device >= kMaxDevices) return fail(std::string(who) + ": device index out of range");
  CUDA_TRY(cudaSetDevice(device));
  return 0;
}

// Device scratch that lives as long as the process: one pool per device, grown on demand (the old buffer freed, then a larger
// one allocated) and never shrunk, so a call allocates nothing once the pool is as large as its request. A lease holds the
// device's lock from acquire() until it is destroyed, that is until the entry point returns: its kernels and copies use the
// scratch until then, and another thread's call on the same device waits rather than reallocating the pool under them. An entry
// point holding a lease must not call another entry point (one lock per device: it would deadlock).
class Scratch {
 public:
  static constexpr int kMaxParts = 8;

  // Locks the pool of `device` (the caller's selected device) and lays out the parts of `bytes`, in the order given, each at a
  // 256-byte boundary. -1 with the error set when the pool cannot grow; the pool is then empty.
  int acquire(int device, const char* who, std::initializer_list<size_t> bytes) {
    if (device < 0 || device >= kMaxDevices) return fail(std::string(who) + ": device index out of range");
    if (bytes.size() > (size_t)kMaxParts) return fail(std::string(who) + ": too many scratch parts");
    size_t need = 0;
    int k = 0;
    for (size_t b : bytes) {
      off_[k++] = need;
      need += (b + 255) / 256 * 256;
    }
    Pool& pl = pools()[device];
    lock_ = std::unique_lock<std::mutex>(pl.mu);
    if (pl.bytes < need) {
      if (pl.p) cudaFree(pl.p);
      pl.p = nullptr;
      pl.bytes = 0;
      const cudaError_t e = cudaMalloc(&pl.p, need);
      if (e != cudaSuccess) {
        pl.p = nullptr;
        return fail(std::string(who) + ": allocating " + std::to_string(need) + " bytes of device scratch: " + cudaGetErrorString(e));
      }
      pl.bytes = need;
    }
    base_ = static_cast<char*>(pl.p);
    return 0;
  }

  template <class T>
  T* part(int i) const { return reinterpret_cast<T*>(base_ + off_[i]); }

 private:
  struct Pool {
    std::mutex mu;
    void* p = nullptr;
    size_t bytes = 0;
  };
  static Pool* pools() {
    static Pool pool[kMaxDevices];
    return pool;
  }

  std::unique_lock<std::mutex> lock_;
  char* base_ = nullptr;
  size_t off_[kMaxParts] = {};
};

}  // namespace summary
