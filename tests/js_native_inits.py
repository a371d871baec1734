"""The `amwg_native` calls of js/amwg_napi.cc for per-chain starting points, over the same C ABI with ctypes: `set_state`
(amwg_set_state) and `disperse_state` (amwg_disperse_state), added to the device binding of tests/js_host.py so that js/mcmc.js's
`set_state` and `options.init_radius` drive the real libamwg_b200.so."""
from __future__ import annotations

import ctypes as C

import numpy as np

from js_host import DeviceNative, _num_list
from oracle.minijs.minijs import JSThrow, undefined


class InitsDeviceNative(DeviceNative):
    """DeviceNative plus the bindings `set_state(handle, values[n_comp][chains])` and `disperse_state(handle, radius) -> failed chains`."""

    def __call__(self, host):
        o = super().__call__(host)
        it = host.it
        L = self.pkg._ffi.lib()

        def set_state(this, a):
            D, _nd, C_ = self.meta[a[0]]
            x = np.asarray(_num_list(a[1]), dtype=np.float64)
            if x.size != D * C_:
                raise JSThrow("amwg_native: set_state expects n_comp x chains numbers")
            if L.amwg_set_state(self.handles[a[0]], x.ctypes.data) != 0:
                self._fail()
            return undefined

        def disperse_state(this, a):
            failed = C.c_int64(0)
            if L.amwg_disperse_state(self.handles[a[0]], float(a[1]), C.byref(failed)) != 0 and failed.value == 0:
                self._fail()
            return float(failed.value)

        o.put("set_state", it.make_native("set_state", set_state))
        o.put("disperse_state", it.make_native("disperse_state", disperse_state))
        return o
