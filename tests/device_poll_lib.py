"""ctypes loader for the device poll / status / Disconnect test driver (tests/native/device_poll.cu).
TEST INFRASTRUCTURE."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
NATIVE = os.path.join(HERE, "native")
LIB = os.path.join(NATIVE, "libdevice_poll.so")

SEND, SEND_ALL, RECV, STATUS, WRITABLE, DISCONNECT, TORN, STREAM_SEND, STREAM_RECV, WAIT_EVENTS = range(1, 11)
OK, TIMEOUT = 0, 1
EV_READABLE, EV_WRITABLE = 0x1, 0x4
UNINITIALIZED, INITIALIZED, CONNECTED, HALF_CLOSED, DISCONNECTED, ERROR = range(6)


class DpOp(C.Structure):  # struct dp_op, tests/native/device_poll.cu
    _fields_ = [("kind", C.c_uint32), ("pair", C.c_uint32), ("slices", C.c_void_p), ("n", C.c_uint64),
                ("byte_idx", C.c_uint64), ("dst", C.c_void_p), ("cap", C.c_uint64), ("ret", C.c_uint64),
                ("calls", C.c_uint64), ("status", C.c_uint32), ("_pad", C.c_uint32)]


class DpServe(C.Structure):  # struct dp_serve, tests/native/device_poll.cu
    _fields_ = [("srv", C.c_void_p), ("cli", C.c_void_p), ("n", C.c_uint32), ("rounds", C.c_uint32),
                ("msg", C.c_uint32), ("mode", C.c_uint32), ("sbuf", C.c_void_p), ("cbuf", C.c_void_p),
                ("state", C.c_void_p), ("times", C.c_void_p), ("out", C.c_void_p), ("budget_ns", C.c_uint64),
                ("max_iters", C.c_uint64)]


assert C.sizeof(DpOp) == 72 and C.sizeof(DpServe) == 88

_lib = None


def build():
    out = subprocess.run(["make", "-s", "-C", NATIVE, "-f", "device_poll.mk"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("building the device poll driver failed:\n" + out.stdout + out.stderr)
    return out.stderr  # ptxas -v report


def load():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        L.dp_prepare.restype = C.c_int
        L.dp_launch.restype = C.c_int
        L.dp_launch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_uint64]
        L.dp_wait.restype = C.c_int
        L.dp_poll.restype = C.c_int
        L.dp_poll.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        L.dp_serve_launch.restype = C.c_int
        L.dp_serve_launch.argtypes = [C.c_void_p]
        L.dp_poll_time.restype = C.c_int
        L.dp_poll_time.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
        L.dp_error.restype = C.c_char_p
        _lib = L
    return _lib


class Pinned:
    """grow-only pinned (mapped) host buffers by name"""

    def __init__(self, L):
        self.L, self.bufs = L, {}

    def get(self, key, nbytes):
        p, n = self.bufs.get(key, (None, 0))
        if n < nbytes:
            if p:
                self.L.b200_mem_free_host(p)
            p = self.L.b200_mem_alloc_host(nbytes)
            assert p
            self.bufs[key] = (p, nbytes)
        return p

    def array(self, key, dtype, n):
        dt = np.dtype(dtype)
        p = self.get(key, max(1, n) * dt.itemsize)
        return p, np.ctypeslib.as_array((C.c_uint8 * (max(1, n) * dt.itemsize)).from_address(p)).view(dt)[:n]

    def free(self):
        for p, _ in self.bufs.values():
            self.L.b200_mem_free_host(p)
        self.bufs = {}


class Runner:
    """dp_kernel: lists of ops, one warp per list (lists run concurrently, the ops of a list in order); dp_poll: one
    b200_warp_poll.  Handles, ops and results live in pinned buffers."""

    def __init__(self, pkg):
        self.pkg, self.L, self.D = pkg, pkg.lib(), load()
        assert self.D.dp_prepare() == 0, self.D.dp_error()
        self.mem = Pinned(self.L)

    def handles(self, key, handles):
        hp = self.mem.get(key, 64 * max(1, len(handles)))
        for i, h in enumerate(handles):
            assert len(h) == 64
            C.memmove(hp + 64 * i, h, 64)
        return hp

    def launch(self, handles, lists, budget_s=30.0, max_iters=1 << 40):
        hp = self.handles("h", handles)
        nops = sum(len(x) for x in lists)
        opp = self.mem.get("ops", C.sizeof(DpOp) * max(1, nops))
        ops = (DpOp * max(1, nops)).from_address(opp)
        fp = self.mem.get("first", 4 * (len(lists) + 1))
        first = (C.c_uint32 * (len(lists) + 1)).from_address(fp)
        k = 0
        for w, lst in enumerate(lists):
            first[w] = k
            for d in lst:
                C.memset(C.addressof(ops[k]), 0, C.sizeof(DpOp))
                for key, v in d.items():
                    setattr(ops[k], key, v)
                k += 1
        first[len(lists)] = k
        assert self.D.dp_launch(hp, opp, fp, len(lists), int(budget_s * 1e9), max_iters) == 0, \
            self.D.dp_error().decode()
        self._pending = (ops, [len(x) for x in lists])

    def wait(self):
        assert self.D.dp_wait() == 0, self.D.dp_error().decode()
        ops, sizes = self._pending
        out, k = [], 0
        for n in sizes:
            out.append([dict(ret=ops[k + j].ret, calls=ops[k + j].calls, status=ops[k + j].status) for j in range(n)])
            k += n
        return out

    def run(self, handles, lists, budget_s=30.0, max_iters=1 << 40):
        self.launch(handles, lists, budget_s, max_iters)
        return self.wait()

    def one(self, h, **op):
        """one op on one handle; returns its `ret` (asserts it finished in time)"""
        r = self.run([h], [[dict(op, pair=0)]])[0][0]
        assert r["status"] == OK, r
        return r["ret"]

    def poll(self, handles, with_events=True, with_ready=True):
        """b200_warp_poll over `handles`: (count, events or None, ready or None)"""
        n = len(handles)
        hp = self.handles("ph", handles)
        ep, ev = self.mem.array("pe", np.uint32, n)
        rp, rd = self.mem.array("pr", np.uint32, n)
        cp, cnt = self.mem.array("pc", np.uint32, 1)
        ev[:] = 0xdead
        rd[:] = 0xdead
        cnt[:] = 0xdead
        assert self.D.dp_poll(hp, n, ep if with_events else None, rp if with_ready else None, cp) == 0, \
            self.D.dp_error().decode()
        c = int(cnt[0])
        return c, (ev.copy() if with_events else None), (rd[:c].copy() if with_ready else None)

    def close(self):
        self.mem.free()
