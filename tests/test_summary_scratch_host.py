"""Host side of the summary entry points' shared prologue and scratch (csrc/amwg_summary_scratch.h), compiled with g++ against
stub cudaMalloc / cudaFree / cudaSetDevice (tests/host_shim/scratch_host.cpp): the parts of a lease are 256-byte aligned and
disjoint, the pool grows only for a larger request and never shrinks, a failed allocation empties the slot and names the caller,
an out-of-range device index is refused before any CUDA call, and a lease holds its device's lock and no other."""
import ctypes as C
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    out = tmp_path_factory.mktemp("scratch_host") / "libscratch_host.so"
    cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-pthread", "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"),
           os.path.join(ROOT, "tests", "host_shim", "scratch_host.cpp"), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(str(out))
    lib.hs_last_error.restype = C.c_char_p
    lib.hs_pool_bytes.restype = C.c_longlong
    return lib


def counts(H):
    c = (C.c_longlong * 4)()
    H.hs_counts(c)
    return {"malloc": c[0], "free": c[1], "set_device": c[2], "device": c[3]}


def acquire(H, device, sizes):
    s = (C.c_longlong * 4)(*sizes)
    p = (C.c_ulonglong * 4)()
    rc = H.hs_acquire(device, s, p)
    return rc, list(p)


def test_parts_are_aligned_disjoint_and_in_order(H):
    sizes = [1, 257, 0, 4096 + 8]
    rc, ptrs = acquire(H, 0, sizes)
    assert rc == 0
    assert all(p % 256 == 0 for p in ptrs)
    for i in range(3):                                           # in the order given, each starting past the previous one's end
        assert ptrs[i + 1] >= ptrs[i] + sizes[i]
    assert ptrs[1] - ptrs[0] == 256 and ptrs[2] - ptrs[1] == 512 and ptrs[3] == ptrs[2]
    assert H.hs_pool_bytes(0) == 256 + 512 + 0 + 4352           # the total the pool computed: every part rounded up to 256


def test_the_pool_grows_only_for_a_larger_request_and_never_shrinks(H):
    dev = 1
    before = counts(H)
    assert acquire(H, dev, [1000, 0, 0, 0])[0] == 0
    assert H.hs_pool_bytes(dev) == 1024
    c = counts(H)
    assert (c["malloc"], c["free"]) == (before["malloc"] + 1, before["free"])
    base = acquire(H, dev, [100, 100, 100, 100])[1][0]              # 1024 bytes: fits, nothing allocated
    assert acquire(H, dev, [8, 0, 0, 0])[1][0] == base              # smaller: fits, the pool keeps its size
    assert H.hs_pool_bytes(dev) == 1024 and counts(H)["malloc"] == c["malloc"] and counts(H)["free"] == c["free"]
    assert acquire(H, dev, [1025, 0, 0, 0])[0] == 0                 # larger: freed, then allocated at the new size
    assert H.hs_pool_bytes(dev) == 1280
    assert (counts(H)["malloc"], counts(H)["free"]) == (c["malloc"] + 1, c["free"] + 1)
    assert acquire(H, dev, [1, 0, 0, 0])[0] == 0
    assert H.hs_pool_bytes(dev) == 1280


def test_a_failed_allocation_empties_the_slot_and_names_the_caller(H):
    dev = 2
    assert acquire(H, dev, [512, 0, 0, 0])[0] == 0
    H.hs_fail_next_malloc()
    assert acquire(H, dev, [4096, 0, 0, 0])[0] != 0
    msg = H.hs_last_error()
    assert msg.startswith(b"hs_acquire: ") and b"out of memory" in msg, msg
    assert H.hs_pool_bytes(dev) == 0
    c = counts(H)
    assert acquire(H, dev, [8, 0, 0, 0])[0] == 0                    # the empty slot allocates again and frees nothing
    assert (counts(H)["malloc"], counts(H)["free"]) == (c["malloc"] + 1, c["free"])
    assert H.hs_pool_bytes(dev) == 256


@pytest.mark.parametrize("device", [-1, 64])
def test_an_out_of_range_device_is_refused_before_any_cuda_call(H, device):
    before = counts(H)
    assert H.hs_select_device(device) != 0
    assert H.hs_last_error() == b"hs_select_device: device index out of range"
    assert acquire(H, device, [8, 0, 0, 0])[0] != 0
    assert H.hs_last_error() == b"hs_acquire: device index out of range"
    assert counts(H) == before
    assert H.hs_select_device(63) == 0 and counts(H)["device"] == 63


def test_a_lease_holds_its_devices_lock_and_no_other(H):
    assert H.hs_try_lock_while_held(3, 3) == 0
    assert H.hs_try_lock_while_held(3, 4) == 1
    assert H.hs_try_lock_while_held(4, 3) == 1                      # device 3's lock was released when its lease ended
