"""Checkpoints without a GPU: the image code of amwg_checkpoint_save / amwg_checkpoint_load (csrc/amwg_checkpoint.h compiled for the
host) against the restatement of the DESIGN.md layout (tests/ckpt_ref.py), every refusal of a restore with its message, the model
fingerprint through libamwg_b200.so, the argument handling of sampler.restore and the all-or-nothing decision of a distributed
restore over a world-2 gloo group."""
import ctypes as C
import os
import socket
import struct
import subprocess
import sys

import numpy as np
import pytest

import ckpt_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP = 0x1234_5678_9ABC_DEF0


@pytest.fixture(scope="module")
def H(tmp_path_factory):
    out = tmp_path_factory.mktemp("ckpt") / "libcheckpoint_host.so"
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "bayes.js_b200", "csrc"),
           os.path.join(ROOT, "tests", "host_shim", "checkpoint_host.cpp"), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(str(out))
    vp, u64 = C.c_void_p, C.c_uint64
    lib.hs_checksum.restype, lib.hs_checksum.argtypes = u64, [vp, u64]
    lib.hs_image_size.restype, lib.hs_image_size.argtypes = u64, [u64, u64, u64]
    lib.hs_write_image.restype = None
    lib.hs_write_image.argtypes = [C.c_uint32, C.c_uint32, u64, u64, u64, u64] + [vp] * 10
    lib.hs_restore.restype = C.c_int
    lib.hs_restore.argtypes = [C.POINTER(vp), C.POINTER(C.c_int64), C.c_int, u64, u64, u64, C.c_int, C.c_int] + [vp] * 14 + [C.c_char_p, C.c_int64]
    return lib


def _p(a):
    return None if a is None else a.ctypes.data


def host_write(H, P, D, seed, first, counters, arr):
    C_ = arr["rng_n"].shape[0]
    out = np.zeros(H.hs_image_size(D, P, C_), dtype=np.uint8)
    ad = np.asarray(counters[0], np.uint64); it = np.asarray(counters[1], np.float64); bc = np.asarray(counters[2], np.float64)
    c = {k: np.ascontiguousarray(v) for k, v in arr.items()}
    H.hs_write_image(P, D, FP, seed, first, C_, _p(ad), _p(it), _p(bc), _p(c["state"]), _p(c["pls"]), _p(c.get("perm")), _p(c["rng_n"]),
                     _p(c["acc"]), _p(c.get("perm_ext")), _p(out))
    return out.tobytes()


class Handle:
    """What a restore is checked against: a handle's model (fingerprint, parameter types, batch sizes) and chain range."""

    def __init__(self, D, P, first, n, types=None, batch_size=50.0, fingerprint=FP):
        self.D, self.P, self.first, self.n, self.fp = D, P, first, n, fingerprint
        self.types = np.asarray(types if types is not None else [0] * P, np.int32)
        per = [D // P + (1 if p < D % P else 0) for p in range(P)]
        self.n_comp = np.asarray(per, np.int32)
        self.off = np.concatenate([[0], np.cumsum(per)[:-1]]).astype(np.int32)
        self.bs = np.full(D, float(batch_size))


def host_restore(H, images, h):
    n = len(images)
    bufs = [np.frombuffer(b, dtype=np.uint8) for b in images]
    ptrs = (C.c_void_p * max(n, 1))(*[b.ctypes.data for b in bufs])
    sizes = (C.c_int64 * max(n, 1))(*[b.size for b in bufs])
    D, P, Cn = h.D, h.P, h.n
    out = {"state": np.full((D, Cn), np.nan), "pls": np.full((D, Cn), np.nan), "rng_n": np.zeros(Cn, np.uint64), "acc": np.full((D, Cn), -7, np.int32)}
    if P <= 16:
        out["perm"] = np.zeros(Cn, np.uint64)
    else:
        out["perm_ext"] = np.zeros((P, Cn), np.uint8)
    seed = C.c_uint64(0)
    ad, it, bc = np.zeros(D, np.uint64), np.zeros(D), np.zeros(D)
    err = C.create_string_buffer(512)
    rc = H.hs_restore(ptrs, sizes, n, h.fp, h.first, Cn, D, P, _p(h.types), _p(h.off), _p(h.n_comp), _p(h.bs), _p(out["state"]), _p(out["pls"]),
                      _p(out.get("perm")), _p(out["rng_n"]), _p(out["acc"]), _p(out.get("perm_ext")), C.addressof(seed), _p(ad), _p(it), _p(bc), err, len(err))
    if rc != 0:
        return err.value.decode()
    return out, seed.value, (ad, it, bc)


def _counters(D, it=7.0, bc=3.0):
    return ([1] * D, [it] * D, [bc] * D)


@pytest.mark.parametrize("D,P,Cn", [(3, 2, 5), (65, 3, 17), (40, 20, 9), (16, 16, 4), (300, 17, 3)])
def test_header_writes_the_restated_bytes_and_reads_them(H, D, P, Cn):
    rng = np.random.default_rng(D * 100 + P)
    arr = ckpt_ref.random_arrays(rng, D, P, Cn)
    counters = ([int(v) for v in rng.integers(0, 2, D)], rng.integers(0, 49, D).astype(float).tolist(), rng.integers(0, 9, D).astype(float).tolist())
    want = ckpt_ref.write(P, D, FP, 2**64 - 5, 2**33 + 1, counters, arr)
    got = host_write(H, P, D, 2**64 - 5, 2**33 + 1, counters, arr)
    assert got == want
    assert len(want) == ckpt_ref.header_bytes(D) + Cn * ckpt_ref.per_chain(D, P) + 8
    assert H.hs_checksum(want, len(want) - 8) == ckpt_ref.checksum(want[:-8]) == ckpt_ref.parse(want)["checksum"]
    q = ckpt_ref.parse(want)
    assert (q["version"], q["P"], q["D"], q["C"], q["seed"], q["first_chain"]) == (1, P, D, Cn, 2**64 - 5, 2**33 + 1)
    # the header reads what the restatement writes
    out, seed, (ad, it, bc) = host_restore(H, [want], Handle(D, P, 2**33 + 1, Cn))
    assert seed == 2**64 - 5 and ad.tolist() == counters[0] and it.tolist() == counters[1] and bc.tolist() == counters[2]
    for k, v in arr.items():
        assert np.array_equal(out[k], v), k


def test_image_sizes_of_the_baseline_configs(H):
    # config 2 (D=2), config 4 (D=65, P=3) and config 5 (D=8, P=1): the per-chain bytes of DESIGN.md §2
    assert ckpt_ref.per_chain(2, 2) == 56 and ckpt_ref.per_chain(65, 3) == 1316 and ckpt_ref.per_chain(8, 1) == 176
    for D, P, Cn in ((2, 2, 1 << 20), (65, 3, 1 << 16), (8, 1, 1 << 19), (300, 17, 10)):
        assert H.hs_image_size(D, P, Cn) == ckpt_ref.header_bytes(D) + Cn * ckpt_ref.per_chain(D, P) + 8


@pytest.mark.parametrize("P", [3, 20])
def test_assembly_from_any_images_into_any_range_is_numpy_slicing(H, P):
    rng = np.random.default_rng(P)
    D, total = 5 if P <= 16 else 24, 97
    arr = ckpt_ref.random_arrays(rng, D, P, total)
    counters = _counters(D)
    cases = [
        ([(0, 97)], (0, 97)), ([(0, 97)], (13, 40)), ([(0, 30), (30, 97)], (0, 97)), ([(30, 97), (0, 30)], (5, 91)),
        ([(0, 11), (11, 12), (12, 60), (60, 97)], (10, 61)), ([(60, 97), (12, 60), (0, 11), (11, 12)], (0, 97)),
        ([(0, 50), (50, 97)], (49, 2)), ([(0, 3), (3, 96)], (95, 1)), ([(40, 70)], (41, 28)),
    ]
    for shards, (first, n) in cases:
        imgs = [host_write(H, P, D, 99, a, counters, ckpt_ref.slice_chains(arr, a, b)) for a, b in shards]
        order = rng.permutation(len(imgs))
        out, seed, _ = host_restore(H, [imgs[k] for k in order], Handle(D, P, first, n))
        want = ckpt_ref.slice_chains(arr, first, first + n)
        assert seed == 99
        for k in want:
            assert np.array_equal(out[k], want[k]), (shards, first, n, k)


def _reseal(img: bytes) -> bytes:
    body = img[:-8]
    return body + struct.pack("<Q", ckpt_ref.checksum(body))


def _patch(img: bytes, off: int, data: bytes) -> bytes:
    return _reseal(img[:off] + data + img[off + len(data):])


def test_every_single_byte_flip_is_refused(H):
    rng = np.random.default_rng(5)
    D, P, Cn = 3, 2, 4
    img = host_write(H, P, D, 1, 0, _counters(D), ckpt_ref.random_arrays(rng, D, P, Cn))
    h = Handle(D, P, 0, Cn)
    assert isinstance(host_restore(H, [img], h), tuple)
    size_msg, sum_msg = "restore: the image is truncated or its size does not match its header", "restore: the image is damaged (checksum mismatch)"
    for i in range(len(img)):
        for bit in (0x01, 0x80):
            bad = bytearray(img)
            bad[i] ^= bit
            msg = host_restore(H, [bytes(bad)], h)
            if i < 8:
                assert msg == "restore: not a checkpoint image", (i, msg)
            elif i < 12:
                assert msg.startswith("restore: unsupported format version "), (i, msg)
            elif i < 24 or 48 <= i < 56:          # P, D, reserved, C: the size no longer matches, or (P <= 16 either way) the checksum
                assert msg in (size_msg, sum_msg), (i, msg)
            else:
                assert msg == sum_msg, (i, msg)


def test_every_refusal_has_its_message(H):
    rng = np.random.default_rng(6)
    D, P, Cn = 4, 3, 10
    arr = ckpt_ref.random_arrays(rng, D, P, Cn)
    img = host_write(H, P, D, 1, 0, _counters(D), arr)
    h = Handle(D, P, 0, Cn)
    hdr = ckpt_ref.header_bytes(D)
    perm_off = hdr + 16 * D * Cn
    a0, a1 = (host_write(H, P, D, 1, a, _counters(D), ckpt_ref.slice_chains(arr, a, b)) for a, b in ((0, 4), (4, 10)))
    cases = [
        ([b"not an image at all, clearly not" * 3], h, "restore: not a checkpoint image"),
        ([img[:40]], h, "restore: not a checkpoint image"),
        ([_patch(img, 8, struct.pack("<I", 2))], h, "restore: unsupported format version 2 (this library reads version 1)"),
        ([img[:-1]], h, "restore: the image is truncated or its size does not match its header"),
        ([img + b"\0"], h, "restore: the image is truncated or its size does not match its header"),
        ([img[:-8] + bytes(8)], h, "restore: the image is damaged (checksum mismatch)"),
        ([img], Handle(D, P, 0, Cn, fingerprint=FP + 1), "restore: the image was taken with a different model, data or options"),
        ([img], Handle(D + 1, P, 0, Cn), "restore: the image was taken with a different model, data or options"),
        ([a0, _patch(a1, 32, struct.pack("<Q", 2))], h, "restore: the images come from different runs, or from different points of one run"),
        ([a0, host_write(H, P, D, 1, 4, _counters(D, it=8.0), ckpt_ref.slice_chains(arr, 4, 10))], h,
         "restore: the images come from different runs, or from different points of one run"),
        ([a0], h, "restore: chains [4, 10) are not covered by the images"),
        ([a1], h, "restore: chains [0, 4) are not covered by the images"),
        ([host_write(H, P, D, 1, 0, _counters(D), ckpt_ref.slice_chains(arr, 0, 3)), a1], h, "restore: chains [3, 4) are not covered by the images"),
        ([a0, host_write(H, P, D, 1, 3, _counters(D), ckpt_ref.slice_chains(arr, 3, 10))], h, "restore: images overlap at chain 3"),
        ([img, a1], Handle(D, P, 2, 3), "restore: images overlap at chain 4"),
        ([_patch(img, perm_off + 8 * 6, struct.pack("<Q", 0x011))], h, "restore: chain 6 has an invalid substepper order"),      # 1, 1, 0
        ([_patch(img, perm_off + 8 * 2, struct.pack("<Q", 0x1021))], h, "restore: chain 2 has an invalid substepper order"),     # bits above 4P
        ([_patch(img, perm_off + 8 * 0, struct.pack("<Q", 0x312))], h, "restore: chain 0 has an invalid substepper order"),      # entry 3 >= P
        ([_patch(img, hdr + 16 * D * Cn + 16 * Cn + 4 * (2 * Cn + 5), struct.pack("<i", -1))], h, "restore: chain 5 has a negative acceptance count"),
        ([host_write(H, P, D, 1, 0, ([1] * D, [50.0] * D, [3.0] * D), arr)], h, "restore: invalid adaptation counters"),
        ([host_write(H, P, D, 1, 0, ([1] * D, [2.5] * D, [3.0] * D), arr)], h, "restore: invalid adaptation counters"),
        ([host_write(H, P, D, 1, 0, ([2] * D, [1.0] * D, [3.0] * D), arr)], h, "restore: invalid adaptation counters"),
        ([host_write(H, P, D, 1, 0, ([1] * D, [1.0] * D, [-1.0] * D), arr)], h, "restore: invalid adaptation counters"),
    ]
    for images, target, msg in cases:
        assert host_restore(H, images, target) == msg, msg
    # a subset of the chains: the invalid chain 6 is not taken, so the restore goes through
    bad = _patch(img, perm_off + 8 * 6, struct.pack("<Q", 0x011))
    assert isinstance(host_restore(H, [bad], Handle(D, P, 0, 6)), tuple)
    assert isinstance(host_restore(H, [bad], Handle(D, P, 7, 3)), tuple)


def test_binary_components_and_perm_ext_are_checked(H):
    rng = np.random.default_rng(7)
    D, P, Cn = 20, 18, 6                         # 18 named parameters: the order is one byte per parameter
    arr = ckpt_ref.random_arrays(rng, D, P, Cn)
    types = [0] * P
    types[4] = 2                                  # parameter 4 is binary (one component)
    h = Handle(D, P, 0, Cn, types=types)
    b = int(h.off[4])
    assert h.n_comp[4] == 1
    arr["state"][b] = rng.integers(0, 2, Cn)
    counters = ([1] * D, [7.0] * D, [3.0] * D)
    counters[0][b] = 0
    img = host_write(H, P, D, 1, 0, counters, arr)
    assert isinstance(host_restore(H, [img], h), tuple)
    hdr = ckpt_ref.header_bytes(D)
    st = arr["state"].copy()
    st[b, 3] = 0.5
    assert host_restore(H, [host_write(H, P, D, 1, 0, counters, dict(arr, state=st))], h) == "restore: chain 3 has a binary parameter other than 0 or 1"
    ad = list(counters[0])
    ad[b] = 1
    assert host_restore(H, [host_write(H, P, D, 1, 0, (ad, counters[1], counters[2]), arr)], h) == "restore: invalid adaptation counters"
    ext_off = hdr + 16 * D * Cn + 8 * Cn + 4 * D * Cn
    pe = arr["perm_ext"].copy()
    pe[7, 2] = pe[8, 2]                           # a repeated entry
    assert host_restore(H, [host_write(H, P, D, 1, 0, counters, dict(arr, perm_ext=pe))], h) == "restore: chain 2 has an invalid substepper order"
    assert host_restore(H, [_patch(img, ext_off + 0 * Cn + 5, bytes([18]))], h) == "restore: chain 5 has an invalid substepper order"


# ---- the model fingerprint, through libamwg_b200.so (no device) ------------------------------------------------------------------
def _norm(pkg, data, opts=None, params=None, sd=100):
    ld = pkg.ld

    def lp(state, d):
        l = 0
        l += ld.norm(state.mu, 0, sd)
        l += ld.unif(state.sigma, 0, 100)
        for i in range(len(d)):
            l += ld.norm(d[i], state.mu, state.sigma)
        return l
    params = params or {"mu": {"type": "real"}, "sigma": {"type": "real", "lower": 0}}
    return pkg.mcmc.AmwgSampler(params, lp, data, dict({"chains": 3, "_model_only": True}, **(opts or {}))).model_fingerprint()


def test_fingerprint_is_stable_and_sees_every_model_change_but_init(pkg):
    data = [183.0, 192, 182, 183, 177, 185, 188, 188, 182, 185] * 20
    base = _norm(pkg, data)
    assert base == _norm(pkg, list(data)) and 0 < base < 2**64                          # two lowerings of one model
    assert _norm(pkg, data, {"seed": 5, "chains": 7}) == base                           # chains and seed are not the model
    assert _norm(pkg, data, params={"mu": {"type": "real", "init": 180}, "sigma": {"type": "real", "lower": 0, "init": 4}}) == base   # init
    changed = [
        _norm(pkg, data[:-1] + [185.5]),                                                 # one data value
        _norm(pkg, data, {"batch_size": 40}),                                            # a stepper option
        _norm(pkg, data, {"params": {"sigma": {"prop_log_scale": 0.5}}}),
        _norm(pkg, data, {"faithful": True}),                                            # another lowering of the same log_post
        _norm(pkg, data, sd=99),                                                         # a constant
        _norm(pkg, data, params={"mu": {"type": "real", "upper": 1000}, "sigma": {"type": "real", "lower": 0}}),
    ]
    assert len(set(changed + [base])) == len(changed) + 1


def test_fingerprint_of_the_javascript_lowering_is_the_python_one(pkg):
    from js_host import JsHost, RecordingNative, make_model_struct
    rec = RecordingNative()
    h = JsHost(native=rec)
    h.it.set_global("amwg_trace", h.load("amwg_trace"))
    h.it.set_global("mcmc", h.load("mcmc"))
    h.it.set_global("ld", h.load("distributions"))
    data = [183.0, 192, 182, 183, 177, 185, 188, 188, 182, 185] * 20
    from oracle.minijs.minijs import to_js
    h.it.set_global("the_data", to_js(h.it, data))
    h.run("""var lp = function (state, data) { var log_post = 0; log_post += ld.norm(state.mu, 0, 100); log_post += ld.unif(state.sigma, 0, 100);
               for (var i = 0; i < data.length; i++) { log_post += ld.norm(data[i], state.mu, state.sigma); } return log_post; };
             new mcmc.AmwgSampler({mu: {type: "real"}, sigma: {type: "real", lower: 0}}, lp, the_data, {chains: 3});
             new mcmc.AmwgSampler({mu: {type: "real"}, sigma: {type: "real", lower: 0}}, lp, the_data, {chains: 3, faithful: true});""")
    L = pkg._ffi.lib()
    got = []
    for desc, _args in rec.created:
        m, _keep, _d = make_model_struct(pkg, desc)
        out = C.c_uint64(0)
        assert L.amwg_model_fingerprint(C.byref(m), C.byref(out)) == 0
        got.append(out.value)
    assert got == [_norm(pkg, data), _norm(pkg, data, {"faithful": True})]


# ---- sampler.restore: arguments and the distributed decision ---------------------------------------------------------------------
def test_restore_arguments(pkg):
    ri = pkg.mcmc.restore_images
    b = bytes(range(40))
    for arg in (b, bytearray(b), memoryview(b), [b], (bytearray(b), memoryview(b)), [memoryview(b)[::2]]):
        imgs = ri(arg)
        assert all(isinstance(a, np.ndarray) and a.dtype == np.uint8 for a in imgs)
    assert ri([memoryview(b)[::2]])[0].tobytes() == b[::2]
    assert ri(bytearray(b))[0].tobytes() == b and len(ri((b, b))) == 2
    for bad in ("image", 3, None, [], [b, "x"], {"a": b}, np.zeros(4, np.uint8)):
        with pytest.raises(pkg.mcmc.JsThrow) as e:
            ri(bad)
        assert str(e.value) == "restore expects a checkpoint image (bytes, bytearray or memoryview) or a list of them"


def test_restore_without_distribution_commits_once(pkg):
    calls = []

    def load(dry):
        calls.append(dry)
        return ""
    pkg.mcmc.restore_with(load)
    assert calls == [False]
    with pytest.raises(pkg.mcmc.JsThrow) as e:
        pkg.mcmc.restore_with(lambda dry: "restore: the image is damaged (checksum mismatch)")
    assert str(e.value) == "restore: the image is damaged (checksum mismatch)"


def _worker(rank, world, port, refusals, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    import __graft_entry__ as graft
    pkg = graft.load_package()
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        res = []
        for r in refusals:
            calls = []

            def load(dry, r=r, calls=calls):
                calls.append(dry)
                return r[rank] if dry else ""
            try:
                pkg.mcmc.restore_with(load, True, 0)
                res.append((None, calls))
            except pkg.mcmc.JsThrow as e:
                res.append((str(e), calls))
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def test_distributed_restore_is_all_or_nothing_over_gloo_world2():
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    gap = "restore: chains [4, 10) are not covered by the images"
    refusals = [("", ""), (gap, ""), ("", gap), (gap, "restore: the image is damaged (checksum mismatch)")]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, refusals, q)) for r in range(2)]
    [p.start() for p in procs]
    res = dict(q.get(timeout=120) for _ in procs)
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    other = "restore: refused on another rank; no rank was changed"
    assert res[0] == [(None, [True, False]), (gap, [True]), (other, [True]), (gap, [True])]
    assert res[1] == [(None, [True, False]), (other, [True]), (gap, [True]), ("restore: the image is damaged (checksum mismatch)", [True])]
