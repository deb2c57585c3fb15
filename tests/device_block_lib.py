"""ctypes loader for the block-level device API test driver (tests/native/device_block.cu), and a trace adapter whose
pairs are driven from a user kernel's CTAs through include/b200_device_block.cuh.  TEST INFRASTRUCTURE."""
import ctypes as C
import os
import subprocess

from device_lib import DeviceEngine

HERE = os.path.dirname(os.path.abspath(__file__))
NATIVE = os.path.join(HERE, "native")
LIB = os.path.join(NATIVE, "libdevice_block.so")

SEND, RECV, STREAM_SEND, STREAM_RECV, WARP_SEND, WARP_RECV = range(1, 7)
OK, TIMEOUT = 0, 1
ONE_CALL, UNTIL_BLOCKED = 0x0, 0x1
THREADS, SMEM_BYTES = 288, 99072


class BdOp(C.Structure):  # struct bd_op, tests/native/device_block.cu
    _fields_ = [("kind", C.c_uint32), ("pair", C.c_uint32), ("slices", C.c_void_p), ("n", C.c_uint64),
                ("byte_idx", C.c_uint64), ("dst", C.c_void_p), ("cap", C.c_uint64), ("flags", C.c_int32),
                ("_pad0", C.c_uint32), ("ret", C.c_uint64), ("calls", C.c_uint64), ("status", C.c_uint32),
                ("_pad", C.c_uint32)]


assert C.sizeof(BdOp) == 80

_lib = None


def build():
    out = subprocess.run(["make", "-s", "-C", NATIVE, "-f", "device_block.mk"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("building the block device API driver failed:\n" + out.stdout + out.stderr)
    return out.stderr  # ptxas -v report


def load():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        L.bd_prepare.restype = C.c_int
        L.bd_max_resident.restype = C.c_int
        L.bd_launch.restype = C.c_int
        L.bd_launch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_uint64, C.c_void_p]
        L.bd_wait.restype = C.c_int
        L.bd_wait.argtypes = [C.c_void_p]
        L.bd_wrong_shape_run.restype = C.c_int
        L.bd_wrong_shape_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.bd_error.restype = C.c_char_p
        _lib = L
    return _lib


class Runner:
    """One launch = lists of ops, one CTA per list (lists run concurrently, the ops of a list in order).  Handles,
    ops and list bounds live in grow-only pinned buffers."""

    def __init__(self, pkg):
        self.pkg, self.L, self.D = pkg, pkg.lib(), load()
        assert self.D.bd_prepare() == 0, self.D.bd_error()
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

    def _fill(self, handles, lists):
        hp = self._pinned("h", 64 * max(1, len(handles)))
        for i, h in enumerate(handles):
            assert len(h) == 64
            C.memmove(hp + 64 * i, h, 64)
        nops = sum(len(x) for x in lists)
        opp = self._pinned("ops", C.sizeof(BdOp) * max(1, nops))
        ops = (BdOp * max(1, nops)).from_address(opp)
        fp = self._pinned("first", 4 * (len(lists) + 1))
        first = (C.c_uint32 * (len(lists) + 1)).from_address(fp)
        k = 0
        for w, lst in enumerate(lists):
            first[w] = k
            for d in lst:
                C.memset(C.addressof(ops[k]), 0, C.sizeof(BdOp))
                for key, v in d.items():
                    setattr(ops[k], key, v)
                k += 1
        first[len(lists)] = k
        return hp, opp, fp, ops

    def run(self, handles, lists, budget_s=30.0, max_iters=1 << 40, stream=None):
        """handles: 64-byte b200_dev_pair blobs; lists: lists of dicts of BdOp fields (`pair` indexes handles).
        Returns, per list, dicts with ret / calls / status of every op."""
        self.launch(handles, lists, budget_s, max_iters, stream)
        return self.wait()

    def launch(self, handles, lists, budget_s=30.0, max_iters=1 << 40, stream=None):
        """run() without waiting: the kernel is queued when this returns; wait() for the results"""
        self.prepare(handles, lists)
        self.fire(budget_s, max_iters, stream)

    def prepare(self, handles, lists):
        """write the handles and ops into the pinned buffers; fire() launches them (timing loops keep the Python work
        out of the timed window)"""
        hp, opp, fp, ops = self._fill(handles, lists)
        self._prepared = (hp, opp, fp, ops, [len(x) for x in lists])

    def fire(self, budget_s=30.0, max_iters=1 << 40, stream=None):
        hp, opp, fp, ops, sizes = self._prepared
        rc = self.D.bd_launch(hp, opp, fp, len(sizes), int(budget_s * 1e9), max_iters, stream)
        if rc != 0:
            raise RuntimeError("bd_launch: %s" % self.D.bd_error().decode())
        self._pending = (ops, sizes, stream)

    def wait(self):
        ops, sizes, stream = self._pending
        assert self.D.bd_wait(stream) == 0, self.D.bd_error().decode()
        out, k = [], 0
        for n in sizes:
            out.append([dict(ret=ops[k + j].ret, calls=ops[k + j].calls, status=ops[k + j].status) for j in range(n)])
            k += n
        return out

    def wrong_shape(self, handles, send, recv, threads):
        """a Send (dict of BdOp fields) and a Recv run by a CTA of `threads` threads: [(ret, calls)] * 2"""
        hp, opp, fp, ops = self._fill(handles, [[send, recv]])
        assert self.D.bd_wrong_shape_run(hp, opp, threads) == 0, self.D.bd_error().decode()
        return [(ops[i].ret, ops[i].calls) for i in range(2)]


class BlockEngine(DeviceEngine):
    """trace.run_trace adapter.  The ends named in `drive` are claimed right after Connect and every op on them runs
    in a device CTA: send / recv are one b200_block_send / b200_block_recv call (B200_BATCH_ONE_CALL), send_all /
    recv_drain one B200_BATCH_UNTIL_BLOCKED call each -- the mapping GpuEngine uses for batches.  The other end uses
    GpuEngine's host calls.  `warp_every`: every k-th op of a claimed end runs as a warp call from warp 0 of the
    same kind of CTA instead (send / recv only), so warp and block calls interleave on one pair."""
    kind = "block"

    def __init__(self, pkg, mem="device", misalign=0, drive=("tx", "rx"), config=None, warp_every=0):
        super().__init__(pkg, mem, misalign, drive, config)
        self.B = Runner(pkg)
        self.warp_every, self.nops = warp_every, 0

    def _run1(self, p, **op):
        self.nops += 1
        if self.warp_every and self.nops % self.warp_every == 0 and op.get("flags", 0) == ONE_CALL:
            op["kind"] = {SEND: WARP_SEND, RECV: WARP_RECV}[op["kind"]]
        res = self.B.run([self.handles[p.h]], [[dict(op, pair=0)]])[0][0]
        assert res["status"] == OK, res
        return res

    def send(self, p, bufs, byte_idx=0):
        if p.h not in self.handles:
            return super(DeviceEngine, self).send(p, bufs, byte_idx)
        return self._send(p, bufs, byte_idx, SEND)["ret"]

    def send_all(self, p, bufs, byte_idx=0):
        if p.h not in self.handles:
            return super(DeviceEngine, self).send_all(p, bufs, byte_idx)
        base, sp = self._slices(bufs)
        try:
            r = self._run1(p, kind=SEND, slices=sp, n=len(bufs), byte_idx=byte_idx, flags=UNTIL_BLOCKED)
        finally:
            self._free(base)
            self.L.b200_mem_free_host(sp)
        return r["ret"], r["calls"]

    def recv(self, p, cap):
        if p.h not in self.handles:
            return super(DeviceEngine, self).recv(p, cap)
        return self._recv(p, cap, RECV)[0]

    def recv_drain(self, p, cap):
        if p.h not in self.handles:
            return super(DeviceEngine, self).recv_drain(p, cap)
        base = self._alloc(cap + self.mis)
        try:
            r = self._run1(p, kind=RECV, dst=base + self.mis, cap=cap, flags=UNTIL_BLOCKED)
            return self._download(base + self.mis, r["ret"]).copy(), r["calls"]
        finally:
            self._free(base)
