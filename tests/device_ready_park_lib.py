"""ctypes loader for the parking ready-set test driver (tests/native/device_ready_park.cu).  TEST INFRASTRUCTURE."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
NATIVE = os.path.join(HERE, "native")
LIB = os.path.join(NATIVE, "libdevice_ready_park.so")


class DpServer(C.Structure):  # struct dp_server
    _fields_ = [("set", C.c_void_p), ("srv", C.c_void_p), ("n", C.c_uint32), ("msg", C.c_uint32),
                ("warps", C.c_uint32), ("idle_takes", C.c_uint32), ("sbuf", C.c_void_p), ("state", C.c_void_p),
                ("closed", C.c_void_p), ("out", C.c_void_p), ("max_iters", C.c_uint64), ("no_park", C.c_uint32),
                ("_pad", C.c_uint32)]


class DpClients(C.Structure):  # struct dp_clients
    _fields_ = [("cli", C.c_void_p), ("a", C.c_uint32), ("rounds", C.c_uint32), ("msg", C.c_uint32),
                ("conn_base", C.c_uint32), ("cbuf", C.c_void_p), ("out", C.c_void_p), ("max_iters", C.c_uint64)]


assert C.sizeof(DpServer) == 80 and C.sizeof(DpClients) == 48

_lib = None


def build():
    out = subprocess.run(["make", "-s", "-C", NATIVE, "-f", "device_ready_park.mk"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("building the parking ready-set driver failed:\n" + out.stdout + out.stderr)
    return out.stderr  # ptxas -v report


def load():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        for name, args in (("dp_prepare", []), ("dp_server_launch", [C.c_void_p]),
                           ("dp_server_wait", [C.POINTER(C.c_float)]), ("dp_clients_launch", [C.c_void_p]),
                           ("dp_clients_wait", []), ("dp_clients_running", []),
                           ("dp_zero", [C.c_void_p, C.c_uint64]), ("dp_copy", [C.c_void_p, C.c_void_p, C.c_uint64])):
            getattr(L, name).restype = C.c_int
            getattr(L, name).argtypes = args
        L.dp_error.restype = C.c_char_p
        _lib = L
    return _lib


def pattern(conn, rnd, msg):
    """the request bytes dp_client_kernel sends: word j = conn << 48 ^ round << 24 ^ j * golden"""
    j = np.arange(msg // 8, dtype=np.uint64)
    w = (np.uint64(conn) << np.uint64(48)) ^ (np.uint64(rnd) << np.uint64(24)) ^ (j * np.uint64(0x9E3779B97F4A7C15))
    return w.view(np.uint8)


class Server:
    """One parking echo server over the set `rs` and its n members (key = index): device buffers, and launches"""

    def __init__(self, pkg, rs, handles, msg, mem):
        self.L, self.D, self.mem, self.n, self.msg = pkg.lib(), load(), mem, len(handles), msg
        assert self.D.dp_prepare() == 0, self.D.dp_error().decode()
        self.setp = mem.blob("park-set", [rs.device()])
        self.hp = mem.blob("park-srv", handles)
        self.dev = []
        self.sbuf = self._dev(self.n * msg)
        self.state = self._dev(4 * (self.n + 1))
        self.closed = self._dev(4 * self.n)
        self.out = self._dev(64)
        self.runs, self.kernel_ms = 0, 0.0

    def _dev(self, nbytes):
        p = self.L.b200_mem_alloc_device(nbytes)
        assert p
        assert self.D.dp_zero(p, nbytes) == 0, self.D.dp_error().decode()
        self.dev.append(p)
        return p

    def launch(self, warps, idle_takes=64, no_park=False, max_iters=1 << 26):
        init = np.zeros(8, np.uint64)
        init[4] = np.uint64(0xFFFFFFFFFFFFFFFF)
        assert self.D.dp_copy(self.out, init.ctypes.data, 64) == 0
        s = DpServer(self.setp, self.hp, self.n, self.msg, warps, idle_takes, self.sbuf, self.state, self.closed,
                     self.out, max_iters, 1 if no_park else 0, 0)
        self._s = s
        assert self.D.dp_server_launch(C.byref(s)) == 0, self.D.dp_error().decode()

    def wait(self):
        ms = C.c_float(0)
        assert self.D.dp_server_wait(C.byref(ms)) == 0, self.D.dp_error().decode()
        o = np.zeros(8, np.uint64)
        assert self.D.dp_copy(o.ctypes.data, self.out, 64) == 0
        self.runs += 1
        self.kernel_ms += ms.value
        return dict(status=int(o[0]), replies=int(o[1]), taken=int(o[2]), busy_parks=int(o[3]), ms=ms.value)

    def closed_flags(self):
        o = np.zeros(self.n, np.uint32)
        assert self.D.dp_copy(o.ctypes.data, self.closed, o.nbytes) == 0
        return o

    def free(self):
        for p in self.dev:
            self.L.b200_mem_free_device(p)
        self.dev = []


class Clients:
    """a device client warps over the claimed client ends `handles`"""

    def __init__(self, pkg, handles, msg, mem, conn_base=0):
        self.L, self.D, self.a, self.msg = pkg.lib(), load(), len(handles), msg
        self.hp = mem.blob("park-cli%d" % conn_base, handles)
        self.cbuf = self.L.b200_mem_alloc_device(self.a * 2 * msg)
        self.outp, self.out = mem.array("park-cout%d" % conn_base, np.uint64, 2 * self.a)
        self.conn_base = conn_base

    def launch(self, rounds, max_iters=1 << 30):
        self.out[:] = 0
        self._c = DpClients(self.hp, self.a, rounds, self.msg, self.conn_base, self.cbuf, self.outp, max_iters)
        assert self.D.dp_clients_launch(C.byref(self._c)) == 0, self.D.dp_error().decode()

    def running(self):
        return self.D.dp_clients_running() == 1

    def wait(self, rounds):
        assert self.D.dp_clients_wait() == 0, self.D.dp_error().decode()
        rows = self.out.reshape(self.a, 2)
        assert (rows[:, 0] == 0).all(), ("mismatched replies", rows[:, 0])
        assert (rows[:, 1] == rounds).all(), ("rounds done", rows[:, 1])

    def free(self):
        self.L.b200_mem_free_device(self.cbuf)
