"""ctypes loader for the device API test driver (tests/native/device_api.cu), and a trace adapter whose pairs are
driven from a user kernel through include/b200_device.cuh.  TEST INFRASTRUCTURE."""
import ctypes as C
import os
import subprocess

import numpy as np

from gpu_engine import GpuEngine

HERE = os.path.dirname(os.path.abspath(__file__))
NATIVE = os.path.join(HERE, "native")
LIB = os.path.join(NATIVE, "libdevice_api.so")

SEND, SEND_ALL, RECV, RECV_DRAIN, STREAM_SEND, STREAM_RECV, PING, PONG, READY = range(1, 10)
OK, TIMEOUT = 0, 1


class DaOp(C.Structure):  # struct da_op, tests/native/device_api.cu
    _fields_ = [("kind", C.c_uint32), ("pair", C.c_uint32), ("slices", C.c_void_p), ("n", C.c_uint64),
                ("byte_idx", C.c_uint64), ("dst", C.c_void_p), ("cap", C.c_uint64), ("times", C.c_void_p),
                ("ret", C.c_uint64), ("calls", C.c_uint64), ("status", C.c_uint32), ("_pad", C.c_uint32)]


assert C.sizeof(DaOp) == 80

_lib = None


def build():
    out = subprocess.run(["make", "-s", "-C", NATIVE, "-f", "device_api.mk"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("building the device API driver failed:\n" + out.stdout + out.stderr)
    return out.stderr  # ptxas -v report


def load():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        L.da_prepare.restype = C.c_int
        L.da_run.restype = C.c_int
        L.da_run.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_uint64]
        L.da_launch.restype = C.c_int
        L.da_launch.argtypes = L.da_run.argtypes
        L.da_wait.restype = C.c_int
        L.da_error.restype = C.c_char_p
        _lib = L
    return _lib


class Runner:
    """One launch = lists of ops, one warp per list (lists run concurrently, the ops of a list in order).  Handles,
    ops and list bounds live in grow-only pinned buffers."""

    def __init__(self, pkg):
        self.pkg, self.L, self.D = pkg, pkg.lib(), load()
        assert self.D.da_prepare() == 0, self.D.da_error()
        self.bufs = {}

    def _pinned(self, key, nbytes):
        p, n = self.bufs.get(key, (None, 0))
        if n < nbytes:
            if p:
                self.L.b200_mem_free_host(p)
            p = self.L.b200_mem_alloc_host(nbytes)
            assert p, self.pkg.last_error()
            self.bufs[key] = (p, nbytes)
        return p

    def run(self, handles, lists, budget_s=30.0, max_iters=1 << 40):
        """handles: 64-byte b200_dev_pair blobs; lists: lists of dicts of DaOp fields (`pair` indexes handles).
        Returns, per list, dicts with ret / calls / status of every op."""
        self.launch(handles, lists, budget_s, max_iters)
        return self.wait()

    def launch(self, handles, lists, budget_s=30.0, max_iters=1 << 40):
        """run() without waiting: the kernel is queued when this returns; wait() for the results"""
        hp = self._pinned("h", 64 * max(1, len(handles)))
        for i, h in enumerate(handles):
            assert len(h) == 64
            C.memmove(hp + 64 * i, h, 64)
        nops = sum(len(x) for x in lists)
        opp = self._pinned("ops", C.sizeof(DaOp) * max(1, nops))
        ops = (DaOp * max(1, nops)).from_address(opp)
        fp = self._pinned("first", 4 * (len(lists) + 1))
        first = (C.c_uint32 * (len(lists) + 1)).from_address(fp)
        k = 0
        for w, lst in enumerate(lists):
            first[w] = k
            for d in lst:
                C.memset(C.addressof(ops[k]), 0, C.sizeof(DaOp))
                for key, v in d.items():
                    setattr(ops[k], key, v)
                k += 1
        first[len(lists)] = k
        rc = self.D.da_launch(hp, opp, fp, len(lists), int(budget_s * 1e9), max_iters)
        assert rc == 0, self.D.da_error().decode()
        self._pending = (ops, [len(x) for x in lists])

    def wait(self):
        assert self.D.da_wait() == 0, self.D.da_error().decode()
        ops, sizes = self._pending
        out, k = [], 0
        for n in sizes:
            out.append([dict(ret=ops[k + j].ret, calls=ops[k + j].calls, status=ops[k + j].status) for j in range(n)])
            k += n
        return out


class DeviceEngine(GpuEngine):
    """trace.run_trace adapter.  The ends named in `drive` ("tx" and / or "rx") are claimed right after Connect and
    every op on them runs in a device warp: send / recv are one b200_warp_send / b200_warp_recv, send_all /
    recv_drain the rdma_flush / rdma_do_read loops inside the kernel.  The other end uses GpuEngine's host calls.
    Readiness answers, cursors and ring images come from the host queries (the mirrors the device calls publish).
    `config`: b200_config_set keys applied while the pairs are initialised (then set back to 0)."""
    kind = "device"

    def __init__(self, pkg, mem="device", misalign=0, drive=("tx", "rx"), config=None):
        super().__init__(pkg, mem, misalign)
        self.drive = drive
        self.config = dict(config or {})
        self.R = Runner(pkg)
        self.handles = {}

    def pair_pair(self, cap, max_sge=30):
        for k, v in self.config.items():
            self.pkg.config_set(k, v)
        try:
            tx, rx = super().pair_pair(cap, max_sge)
        finally:
            for k in self.config:
                self.pkg.config_set(k, 0)
        for name, p in (("tx", tx), ("rx", rx)):
            if name in self.drive:
                self.handles[p.h] = p.device_claim()
        return tx, rx

    def destroy(self, p):
        self.handles.pop(p.h, None)
        super().destroy(p)  # Disconnect releases the claim

    def _run1(self, p, **op):
        res = self.R.run([self.handles[p.h]], [[dict(op, pair=0)]])[0][0]
        assert res["status"] == OK, res
        return res

    def _slices(self, bufs):
        """the buffers back to back with odd gaps (consecutive slices at different alignments), misaligned by
        self.mis, in this engine's memory kind; the slice array in pinned memory"""
        offs, off = [], self.mis
        for b in bufs:
            offs.append(off)
            off += b.size + 3
        base = self._alloc(off)
        flat = np.zeros(off + 1, dtype=np.uint8)
        for b, o in zip(bufs, offs):
            flat[o:o + b.size] = b
        self._upload(base, flat[:off])
        sp = self.L.b200_mem_alloc_host(16 * max(1, len(bufs)))
        arr = (self.pkg.Slice * max(1, len(bufs))).from_address(sp)
        for i, (b, o) in enumerate(zip(bufs, offs)):
            arr[i].ptr, arr[i].len = base + o, b.size
        return base, sp

    def _send(self, p, bufs, byte_idx, kind):
        base, sp = self._slices(bufs)
        try:
            return self._run1(p, kind=kind, slices=sp, n=len(bufs), byte_idx=byte_idx)
        finally:
            self._free(base)
            self.L.b200_mem_free_host(sp)

    def _recv(self, p, cap, kind):
        base = self._alloc(cap + self.mis)
        try:
            r = self._run1(p, kind=kind, dst=base + self.mis, cap=cap)
            return self._download(base + self.mis, r["ret"]).copy(), r["calls"]
        finally:
            self._free(base)

    def send(self, p, bufs, byte_idx=0):
        if p.h not in self.handles:
            return super().send(p, bufs, byte_idx)
        return self._send(p, bufs, byte_idx, SEND)["ret"]

    def send_all(self, p, bufs, byte_idx=0):
        if p.h not in self.handles:
            return super().send_all(p, bufs, byte_idx)
        r = self._send(p, bufs, byte_idx, SEND_ALL)
        return r["ret"], r["calls"]

    def recv(self, p, cap):
        if p.h not in self.handles:
            return super().recv(p, cap)
        return self._recv(p, cap, RECV)[0]

    def recv_drain(self, p, cap):
        if p.h not in self.handles:
            return super().recv_drain(p, cap)
        return self._recv(p, cap, RECV_DRAIN)

    def device_ready(self, p):
        """(readable, has_message, has_pending_writes) as the device queries answer them"""
        r = self._run1(p, kind=READY)
        return r["ret"], r["calls"] & 1, r["calls"] >> 1
