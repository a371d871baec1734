"""Checkpoint images of tempered ladders without a GPU (csrc/amwg_checkpoint.h compiled with g++, DESIGN.md §2 "Checkpoints"): an
untempered image keeps its version-1 bytes; a tempered one adds K, beta, the round counter and every ladder's swap counts, round-trips,
is reassembled from several images at ladder boundaries, and is refused against a sampler with another ladder or none."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP = 0x1234ABCD5678EF01
D, P = 3, 2
TYPES, OFF, NCOMP = np.array([0, 0], np.int32), np.array([0, 1], np.int32), np.array([1, 2], np.int32)
BS = np.full(D, 50.0)
BETA = np.array([1.0, 0.5, 0.25, 0.125])


def _compile(tmp, name):
    out = tmp / ("lib" + name + ".so")
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "tests", "host_shim"),
           "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"), os.path.join(ROOT, "tests", "host_shim", name + ".cpp"), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(str(out))


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("temper_ckpt")
    lib = _compile(tmp, "checkpoint_temper_host")
    u64, vp = C.c_uint64, C.c_void_p
    lib.hs_image_size.restype, lib.hs_image_size.argtypes = u64, [u64] * 4
    lib.hs_write_image.restype = None
    lib.hs_write_image.argtypes = [C.c_uint32, C.c_uint32, u64, u64, u64, u64] + [vp] * 9 + [C.c_uint32, vp, u64, vp, vp]
    lib.hs_restore.restype = C.c_int
    lib.hs_restore.argtypes = [C.POINTER(vp), C.POINTER(C.c_int64), C.c_int, u64, u64, u64, C.c_int, C.c_int] + [vp] * 4 + \
        [C.c_uint32, vp, vp, vp, vp, vp, C.c_char_p, C.c_int64]
    old = _compile(tmp, "checkpoint_host")                     # the version-1 writer the untempered image must still equal
    old.hs_write_image.restype = None
    old.hs_write_image.argtypes = [C.c_uint32, C.c_uint32, u64, u64, u64, u64] + [vp] * 10
    old.hs_image_size.restype, old.hs_image_size.argtypes = u64, [u64] * 3
    lib.old = old
    return lib


def _p(a):
    return None if a is None else a.ctypes.data


def _arrays(first, n, seed=0):
    rng = np.random.default_rng(seed + first)
    g = np.arange(first, first + n)
    return {"state": rng.normal(size=(D, n)), "pls": rng.normal(size=(D, n)), "perm": np.array([0x10 if k % 2 else 0x01 for k in g], np.uint64),
            "rng_n": (g * 1000 + 7).astype(np.uint64), "acc": rng.integers(0, 9, (D, n)).astype(np.int32)}


def _write(H, first, n, K=0, rounds=0, beta=BETA, seed=0):
    a = _arrays(first, n, seed)
    acc = (np.arange(first // K, (first + n) // K)[:, None] * 100 + np.arange(K - 1)[None]).astype(np.uint64) if K else None
    out = np.zeros(H.hs_image_size(D, P, n, K), dtype=np.uint8)
    ad, it, bc = np.ones(D, np.uint64), np.full(D, 7.0), np.full(D, 3.0)
    b = np.ascontiguousarray(beta[:K]) if K else None
    H.hs_write_image(P, D, FP, 99, first, n, _p(ad), _p(it), _p(bc), _p(a["state"]), _p(a["pls"]), _p(a["perm"]), _p(a["rng_n"]), _p(a["acc"]),
                     None, K, _p(b), rounds, _p(acc), _p(out))
    return out, a, acc


def _restore(H, images, first, n, K=0, beta=BETA):
    ptrs = (C.c_void_p * len(images))(*[im.ctypes.data for im in images])
    sizes = (C.c_int64 * len(images))(*[im.size for im in images])
    st, rn, rounds = np.zeros((D, n)), np.zeros(n, np.uint64), C.c_uint64(0)
    acc = np.zeros((max(n // K, 1), max(K - 1, 1)), np.uint64) if K else np.zeros(1, np.uint64)
    err = C.create_string_buffer(512)
    b = np.ascontiguousarray(beta[:K]) if K else None
    rc = H.hs_restore(ptrs, sizes, len(images), FP, first, n, D, P, _p(TYPES), _p(OFF), _p(NCOMP), _p(BS), K, _p(b), _p(st), _p(rn),
                      C.addressof(rounds), _p(acc), err, len(err))
    return rc, err.value.decode(), st, rn, rounds.value, acc


def test_untempered_images_keep_their_version_one_bytes(H):
    for first, n in ((0, 5), (17, 12)):
        a = _arrays(first, n)
        new, _, _ = _write(H, first, n)
        old = np.zeros(H.old.hs_image_size(D, P, n), dtype=np.uint8)
        ad, it, bc = np.ones(D, np.uint64), np.full(D, 7.0), np.full(D, 3.0)
        H.old.hs_write_image(P, D, FP, 99, first, n, _p(ad), _p(it), _p(bc), _p(a["state"]), _p(a["pls"]), _p(a["perm"]), _p(a["rng_n"]),
                             _p(a["acc"]), None, _p(old))
        assert H.hs_image_size(D, P, n, 0) == H.old.hs_image_size(D, P, n) and np.array_equal(new, old)
        assert int.from_bytes(bytes(new[20:24]), "little") == 0


def test_tempered_image_round_trips(H):
    K, n = 4, 12
    img, a, acc = _write(H, 8, n, K, rounds=37)
    assert img.size == H.hs_image_size(D, P, n, 0) + 8 * K + 8 + 8 * (n // K) * (K - 1)
    assert int.from_bytes(bytes(img[20:24]), "little") == K
    rc, err, st, rn, rounds, got = _restore(H, [img], 8, n, K)
    assert rc == 0, err
    assert np.array_equal(st, a["state"]) and np.array_equal(rn, a["rng_n"]) and rounds == 37 and np.array_equal(got, acc)


def test_tempered_images_reassemble_at_ladder_boundaries(H):
    K = 4
    imgs = [_write(H, 0, 8, K, rounds=5), _write(H, 8, 12, K, rounds=5), _write(H, 20, 4, K, rounds=5)]
    allst = np.concatenate([x[1]["state"] for x in imgs], axis=1)
    allacc = np.concatenate([x[2] for x in imgs], axis=0)
    for first, n in ((4, 16), (0, 24), (12, 8), (20, 4)):
        rc, err, st, rn, rounds, acc = _restore(H, [x[0] for x in imgs[::-1]], first, n, K)
        assert rc == 0, err
        assert np.array_equal(st, allst[:, first:first + n]) and np.array_equal(acc, allacc[first // K:(first + n) // K]) and rounds == 5


def test_every_refused_ladder_case(H):
    K = 4
    t, _, _ = _write(H, 0, 8, K, rounds=3)
    u, _, _ = _write(H, 0, 8)
    cases = [
        ([t], 0, 8, 0, "restore: the image is of a tempered ladder (options.temperatures) and this sampler is not tempered"),
        ([u], 0, 8, K, "restore: this sampler is a tempered ladder (options.temperatures) and the image is not"),
        ([_write(H, 0, 8, K, 3, beta=np.array([1.0, 0.5, 0.25, 0.12]))[0]], 0, 8, K, "restore: the image was taken with other temperatures"),
        ([_write(H, 0, 6, 2, 3)[0]], 0, 6, 3, "restore: the image was taken with other temperatures"),
        ([t, _write(H, 8, 8, K, rounds=4)[0]], 0, 16, K, "restore: the images come from different runs, or from different points of one run"),
        ([t], 2, 4, K, "restore: the images split a ladder"),
    ]
    for images, first, n, k, msg in cases:
        rc, err = _restore(H, images, first, n, k)[:2]
        assert rc == -1 and err == msg, (err, msg)
    # a header whose ladder does not divide its chains, or a rung count outside 2..256, is a damaged image
    for k_bad in (1, 3, 257):
        bad = t.copy()
        bad[20:24] = np.frombuffer(np.uint32(k_bad).tobytes(), np.uint8)
        rc, err = _restore(H, [bad], 0, 8, K)[:2]
        assert rc == -1 and err == "restore: the image is truncated or its size does not match its header"
    bad = _write(H, 0, 8, K, 3)[0]
    bad[-20] ^= 1                                              # a bit of the accepts
    rc, err = _restore(H, [bad], 0, 8, K)[:2]
    assert rc == -1 and err == "restore: the image is damaged (checksum mismatch)"
