"""A restatement of the checkpoint image of DESIGN.md §2 "Checkpoints" in numpy and struct: the writer, the parser and the
assembly of a handle's chains from several images, independent of csrc/amwg_checkpoint.h, for tests/test_checkpoint_host.py."""
from __future__ import annotations

import struct

import numpy as np

MAGIC = b"AMWGCKPT"
VERSION = 1
BASIS, PRIME, MASK = 0xcbf29ce484222325, 0x100000001b3, (1 << 64) - 1


def mix(h: int, w: int) -> int:
    return ((h ^ w) * PRIME) & MASK


def mix_bytes(h: int, b: bytes) -> int:
    h = mix(h, len(b))
    pad = b + bytes(-len(b) % 8)
    for w in np.frombuffer(pad, dtype="<u8").tolist():
        h = mix(h, w)
    return h


def checksum(b: bytes) -> int:
    return mix_bytes(BASIS, b)


def per_chain(D: int, P: int) -> int:
    return 20 * D + 8 + (P if P > 16 else 8)


def header_bytes(D: int) -> int:
    return 56 + 24 * D


def write(P, D, fingerprint, seed, first_chain, counters, arrays) -> bytes:
    """counters: (is_adapting[D], iter_since[D], batch_count[D]); arrays: state, pls [D][C] f64, perm [C] u64 (P <= 16) or perm_ext
    [P][C] u8 (P > 16), rng_n [C] u64, acc [D][C] i32."""
    C = arrays["rng_n"].shape[0]
    out = [MAGIC, struct.pack("<IIII", VERSION, P, D, 0), struct.pack("<QQQQ", fingerprint, seed, first_chain, C)]
    ad, it, bc = counters
    for c in range(D):
        out.append(struct.pack("<Qdd", int(ad[c]), float(it[c]), float(bc[c])))
    out.append(np.asarray(arrays["state"], "<f8").reshape(D, C).tobytes())
    out.append(np.asarray(arrays["pls"], "<f8").reshape(D, C).tobytes())
    if P <= 16:
        out.append(np.asarray(arrays["perm"], "<u8").reshape(C).tobytes())
    out.append(np.asarray(arrays["rng_n"], "<u8").reshape(C).tobytes())
    out.append(np.asarray(arrays["acc"], "<i4").reshape(D, C).tobytes())
    if P > 16:
        out.append(np.asarray(arrays["perm_ext"], "u1").reshape(P, C).tobytes())
    body = b"".join(out)
    return body + struct.pack("<Q", checksum(body))


def parse(img: bytes) -> dict:
    """The fields of a well-formed image (no checks beyond the layout)."""
    version, P, D, _ = struct.unpack_from("<IIII", img, 8)
    fp, seed, first, C = struct.unpack_from("<QQQQ", img, 24)
    o = 56
    ad, it, bc = [], [], []
    for _c in range(D):
        a, i, b = struct.unpack_from("<Qdd", img, o)
        ad.append(a); it.append(i); bc.append(b)
        o += 24
    out = {"version": version, "P": P, "D": D, "fingerprint": fp, "seed": seed, "first_chain": first, "C": C, "counters": (ad, it, bc)}

    def take(name, dtype, rows, width):
        nonlocal o
        out[name] = np.frombuffer(img, dtype=dtype, count=rows * C, offset=o).reshape(rows, C) if rows > 1 or name in ("state", "pls", "acc", "perm_ext") \
            else np.frombuffer(img, dtype=dtype, count=C, offset=o)
        o += rows * C * width
    take("state", "<f8", D, 8)
    take("pls", "<f8", D, 8)
    if P <= 16:
        take("perm", "<u8", 1, 8)
    take("rng_n", "<u8", 1, 8)
    take("acc", "<i4", D, 4)
    if P > 16:
        take("perm_ext", "u1", P, 1)
    out["checksum"] = struct.unpack_from("<Q", img, o)[0]
    assert o + 8 == len(img)
    return out


def random_arrays(rng, D, P, C):
    """Arrays of a plausible run: valid substepper orders, non-negative counts."""
    a = {"state": rng.normal(size=(D, C)), "pls": rng.normal(size=(D, C)), "rng_n": rng.integers(0, 1 << 62, C, dtype=np.uint64),
         "acc": rng.integers(0, 50, (D, C)).astype(np.int32)}
    if P <= 16:
        perm = np.zeros(C, dtype=np.uint64)
        for c in range(C):
            for i, e in enumerate(rng.permutation(P)):
                perm[c] |= np.uint64(int(e) << (4 * i))
        a["perm"] = perm
    else:
        a["perm_ext"] = np.stack([rng.permutation(P) for _ in range(C)], axis=1).astype(np.uint8)
    return a


def slice_chains(arrays, a, b):
    """chains [a, b) of a set of arrays (chain axis last)"""
    return {k: v[..., a:b] for k, v in arrays.items()}
