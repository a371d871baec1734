"""The `amwg_native` calls of js/amwg_napi.cc for checkpoints, over the same C ABI with ctypes: `checkpoint` (amwg_checkpoint_size +
amwg_checkpoint_save) and `restore` (amwg_checkpoint_load), added to the device binding of tests/js_host.py so that js/mcmc.js's
`checkpoint()` and `restore()` drive the real libamwg_b200.so. The interpreter has no Buffer: an image is an opaque host object
that carries the Python bytes (`image_of` / `as_image` convert)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from js_host import DeviceNative
from oracle.minijs.minijs import JSArray, JSObject, JSThrow


def as_image(it, data: bytes) -> JSObject:
    o = it.new_object()
    o.image = bytes(data)
    return o


def image_of(o) -> bytes:
    return o.image


class CheckpointDeviceNative(DeviceNative):
    """DeviceNative plus the bindings `checkpoint(handle) -> image` and `restore(handle, [image, ...], dry_run) -> seed`."""

    def __call__(self, host):
        o = super().__call__(host)
        it = host.it
        L = self.pkg._ffi.lib()

        def checkpoint(this, a):
            n = C.c_int64(0)
            if L.amwg_checkpoint_size(self.handles[a[0]], C.byref(n)) != 0:
                self._fail()
            buf = np.empty(n.value, dtype=np.uint8)
            if L.amwg_checkpoint_save(self.handles[a[0]], buf.ctypes.data, n.value) != 0:
                self._fail()
            return as_image(it, buf.tobytes())

        def restore(this, a):
            items = a[1].items if isinstance(a[1], JSArray) else []
            if not all(hasattr(x, "image") for x in items):
                raise JSThrow("restore expects a Buffer or a list of Buffers")
            bufs = [np.frombuffer(x.image, dtype=np.uint8) for x in items]
            ptrs = (C.c_void_p * max(len(bufs), 1))(*[b.ctypes.data for b in bufs])
            sizes = (C.c_int64 * max(len(bufs), 1))(*[b.size for b in bufs])
            if L.amwg_checkpoint_load(self.handles[a[0]], ptrs, sizes, len(bufs), 1 if a[2] else 0) != 0:
                self._fail()
            return float(int.from_bytes(bufs[0][32:40].tobytes(), "little"))

        o.put("checkpoint", it.make_native("checkpoint", checkpoint))
        o.put("restore", it.make_native("restore", restore))
        return o
