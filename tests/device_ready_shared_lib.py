"""ctypes loader for the shared ready-set test driver (tests/native/device_ready_shared.cu).  TEST INFRASTRUCTURE."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
NATIVE = os.path.join(HERE, "native")
LIB = os.path.join(NATIVE, "libdevice_ready_shared.so")
BASELINE, FENCE = 1, 2  # ds_serve flags


class DsDrain(C.Structure):  # struct ds_drain
    _fields_ = [("set", C.c_void_p), ("members", C.c_void_p), ("n", C.c_uint32), ("take_max", C.c_uint32),
                ("warp_base", C.c_uint32), ("mark_idle", C.c_uint32), ("rbuf", C.c_void_p), ("rcap", C.c_uint64),
                ("got", C.c_void_p), ("holder", C.c_void_p), ("taken", C.c_void_p), ("kept", C.c_void_p),
                ("idle", C.c_void_p), ("closed", C.c_void_p), ("keys", C.c_void_p), ("out", C.c_void_p),
                ("stop", C.c_void_p), ("max_iters", C.c_uint64)]


class DsServe(C.Structure):  # struct ds_serve
    _fields_ = [("sets", C.c_void_p), ("srv", C.c_void_p), ("cli", C.c_void_p), ("n", C.c_uint32), ("a", C.c_uint32),
                ("rounds", C.c_uint32), ("msg", C.c_uint32), ("servers", C.c_uint32), ("nsets", C.c_uint32),
                ("take_max", C.c_uint32), ("flags", C.c_uint32), ("sbuf", C.c_void_p), ("cbuf", C.c_void_p),
                ("state", C.c_void_p), ("keys", C.c_void_p), ("done", C.c_void_p), ("out", C.c_void_p),
                ("max_iters", C.c_uint64)]


assert C.sizeof(DsDrain) == 128 and C.sizeof(DsServe) == 112

_lib = None


def build():
    out = subprocess.run(["make", "-s", "-C", NATIVE, "-f", "device_ready_shared.mk"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("building the shared ready-set driver failed:\n" + out.stdout + out.stderr)
    return out.stderr  # ptxas -v report


def load():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        for name, args in (("ds_prepare", []), ("ds_wait", [C.c_int]),
                           ("ds_drain_launch", [C.c_void_p, C.c_uint32, C.c_int]),
                           ("ds_serve_launch", [C.c_void_p]),
                           ("ds_cost", [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]),
                           ("ds_zero", [C.c_void_p, C.c_uint64]), ("ds_copy", [C.c_void_p, C.c_void_p, C.c_uint64])):
            getattr(L, name).restype = C.c_int
            getattr(L, name).argtypes = args
        L.ds_error.restype = C.c_char_p
        _lib = L
    return _lib


class Device:
    """zeroed device memory by name (b200_mem_alloc_device), read back through the driver's stream"""

    def __init__(self, pkg):
        self.L, self.D, self.bufs = pkg.lib(), load(), {}

    def array(self, key, dtype, n):
        nbytes = max(1, n) * np.dtype(dtype).itemsize
        if key in self.bufs:
            self.L.b200_mem_free_device(self.bufs[key][0])
        p = self.L.b200_mem_alloc_device(nbytes)
        assert p
        assert self.D.ds_zero(p, nbytes) == 0, self.D.ds_error().decode()
        self.bufs[key] = (p, np.dtype(dtype), max(1, n))
        return p

    def read(self, key):
        p, dt, n = self.bufs[key]
        a = np.zeros(n, dt)
        assert self.D.ds_copy(a.ctypes.data, p, a.nbytes) == 0, self.D.ds_error().decode()
        return a

    def free(self):
        for p, _, _ in self.bufs.values():
            self.L.b200_mem_free_device(p)
        self.bufs = {}


def serve_totals(out, a, servers):
    """per-server rows of a ds_serve out array, and the time from the first server's start to the last one's end"""
    rows = out[2 * a:2 * a + 8 * servers].reshape(servers, 8)
    span_ns = int(rows[:, 7].max()) - int(rows[:, 6].min())
    return rows, span_ns
