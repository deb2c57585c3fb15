"""ctypes loader for the device ready-set test driver (tests/native/device_ready.cu).  TEST INFRASTRUCTURE."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
NATIVE = os.path.join(HERE, "native")
LIB = os.path.join(NATIVE, "libdevice_ready.so")
WARP_SEND, BLOCK_SEND, WARP_DISC = 0, 1, 2


class DrDrain(C.Structure):  # struct dr_drain
    _fields_ = [("set", C.c_void_p), ("members", C.c_void_p), ("n", C.c_uint32), ("_pad0", C.c_uint32),
                ("rbuf", C.c_void_p), ("rcap", C.c_uint64), ("got", C.c_void_p), ("sbuf", C.c_void_p),
                ("scap", C.c_uint64), ("owe", C.c_void_p), ("sent", C.c_void_p), ("taken", C.c_void_p),
                ("kept", C.c_void_p), ("idle", C.c_void_p), ("closed", C.c_void_p), ("keys", C.c_void_p),
                ("out", C.c_void_p), ("stop", C.c_void_p), ("max_iters", C.c_uint64)]


class DrOp(C.Structure):  # struct dr_op
    _fields_ = [("h", C.c_void_p), ("slices", C.c_void_p), ("n", C.c_uint64), ("ret", C.c_uint64)]


class DrServe(C.Structure):  # struct dr_serve
    _fields_ = [("set", C.c_void_p), ("srv", C.c_void_p), ("cli", C.c_void_p), ("n", C.c_uint32), ("a", C.c_uint32),
                ("rounds", C.c_uint32), ("msg", C.c_uint32), ("sbuf", C.c_void_p), ("cbuf", C.c_void_p),
                ("state", C.c_void_p), ("out", C.c_void_p), ("max_iters", C.c_uint64)]


assert C.sizeof(DrDrain) == 144 and C.sizeof(DrOp) == 32 and C.sizeof(DrServe) == 80

_lib = None


def build():
    out = subprocess.run(["make", "-s", "-C", NATIVE, "-f", "device_ready.mk"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("building the device ready-set driver failed:\n" + out.stdout + out.stderr)
    return out.stderr  # ptxas -v report


def load():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        for name, args in (("dr_prepare", []), ("dr_wait", []), ("dr_drain_launch", [C.c_void_p]),
                           ("dr_ops", [C.c_int, C.c_void_p, C.c_int]),
                           ("dr_poll", [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]),
                           ("dr_serve_launch", [C.c_void_p]),
                           ("dr_cost", [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32,
                                        C.c_void_p])):
            getattr(L, name).restype = C.c_int
            getattr(L, name).argtypes = args
        L.dr_error.restype = C.c_char_p
        _lib = L
    return _lib


class Pinned:
    """pinned (mapped) host arrays by name, zeroed when made"""

    def __init__(self, L):
        self.L, self.bufs = L, {}

    def array(self, key, dtype, n):
        dt = np.dtype(dtype)
        nbytes = max(1, n) * dt.itemsize
        if key in self.bufs:
            self.L.b200_mem_free_host(self.bufs[key][0])
        p = self.L.b200_mem_alloc_host(nbytes)
        assert p
        a = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p)).view(dt)[:max(1, n)]
        a[:] = 0
        self.bufs[key] = (p, a)
        return p, a

    def blob(self, key, blobs):
        """consecutive 64-byte handles"""
        p, a = self.array(key, np.uint8, 64 * max(1, len(blobs)))
        for i, b in enumerate(blobs):
            assert len(b) == 64
            a[64 * i:64 * (i + 1)] = np.frombuffer(b, np.uint8)
        return p

    def free(self):
        for p, _ in self.bufs.values():
            self.L.b200_mem_free_host(p)
        self.bufs = {}


class Consumer:
    """The consumer side of one ready set over n members (key = index): received and owed bytes per member, and the
    per-launch counters of dr_drain_kernel."""

    def __init__(self, pkg, rs, handles, rcap, scap=8):
        self.pkg, self.D, self.mem = pkg, load(), Pinned(pkg.lib())
        assert self.D.dr_prepare() == 0, self.D.dr_error()
        self.n, self.rcap, self.scap = len(handles), rcap, scap
        m = self.mem
        self.setp = m.blob("set", [rs.device()])
        self.hp = m.blob("members", handles)
        self.rbuf_p, self.rbuf = m.array("rbuf", np.uint8, self.n * rcap)
        self.got_p, self.got = m.array("got", np.uint64, self.n)
        self.sbuf_p, self.sbuf = m.array("sbuf", np.uint8, self.n * scap)
        self.owe_p, self.owe = m.array("owe", np.uint64, self.n)
        self.sent_p, self.sent = m.array("sent", np.uint64, self.n)
        self.closed_p, self.closed = m.array("closed", np.uint32, self.n)
        self.keys_p, _ = m.array("keys", np.uint32, max(64, 2 * self.n))
        self.stop_p, self.stop = m.array("stop", np.uint32, 1)

    def set_handles(self, handles):
        self.hp = self.mem.blob("members", handles)

    def launch(self, with_stop=False, max_iters=1 << 22):
        m = self.mem
        self.taken_p, self.taken = m.array("taken", np.uint32, self.n)
        self.kept_p, self.kept = m.array("kept", np.uint32, self.n)
        self.idle_p, self.idle = m.array("idle", np.uint32, self.n)
        self.out_p, self.out = m.array("out", np.uint32, 4)
        self.stop[0] = 0
        d = DrDrain(self.setp, self.hp, self.n, 0, self.rbuf_p, self.rcap, self.got_p, self.sbuf_p, self.scap,
                    self.owe_p, self.sent_p, self.taken_p, self.kept_p, self.idle_p, self.closed_p, self.keys_p,
                    self.out_p, self.stop_p if with_stop else None, max_iters)
        self._d = d
        assert self.D.dr_drain_launch(C.byref(d)) == 0, self.D.dr_error().decode()

    def wait(self):
        assert self.D.dr_wait() == 0, self.D.dr_error().decode()
        return dict(status=int(self.out[0]), dups=int(self.out[1]), foreign=int(self.out[2]), takes=int(self.out[3]))

    def drain(self):
        self.launch()
        return self.wait()

    def ready(self):
        """READY members now (b200_warp_poll's READABLE, or a pending write with credit for one frame)"""
        ep, _ = self.mem.array("ev", np.uint32, self.n)
        rp, r = self.mem.array("rd", np.uint32, self.n)
        assert self.D.dr_poll(self.hp, self.n, ep, rp) == 0, self.D.dr_error().decode()
        return r.copy()

    def received(self, k):
        return self.rbuf[k * self.rcap:k * self.rcap + int(self.got[k])].copy()

    def close(self):
        self.mem.free()


def device_ops(pkg, kind, ops, mem):
    """ops: (handle bytes, pinned slice array pointer, nslices) -> per-op returns"""
    D = load()
    hp = mem.blob("oph", [h for h, _, _ in ops])
    opp, _ = mem.array("ops", np.uint8, C.sizeof(DrOp) * max(1, len(ops)))
    arr = (DrOp * max(1, len(ops))).from_address(opp)
    for i, (_, sl, n) in enumerate(ops):
        arr[i].h, arr[i].slices, arr[i].n, arr[i].ret = hp + 64 * i, sl, n, 0
    assert D.dr_ops(kind, opp, len(ops)) == 0, D.dr_error().decode()
    return [int(arr[i].ret) for i in range(len(ops))]
