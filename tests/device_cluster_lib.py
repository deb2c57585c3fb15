"""ctypes loader for the cluster-call test driver (tests/native/device_cluster.cu), and a trace adapter whose pairs are
driven from a user kernel's thread-block clusters through b200_cluster_send / b200_cluster_recv.  TEST INFRASTRUCTURE."""
import ctypes as C
import os
import subprocess

import device_block_lib as bl

HERE = os.path.dirname(os.path.abspath(__file__))
NATIVE = os.path.join(HERE, "native")
LIB = os.path.join(NATIVE, "libdevice_cluster.so")

SEND, RECV, STREAM_SEND, STREAM_RECV, WARP_SEND, WARP_RECV, BLOCK_SEND, BLOCK_RECV = range(1, 9)
OK, TIMEOUT = 0, 1
ONE_CALL, UNTIL_BLOCKED = 0x0, 0x1
THREADS, SMEM_BYTES = bl.THREADS, bl.SMEM_BYTES
CdOp = bl.BdOp  # struct cd_op has struct bd_op's layout

_lib = None


def build():
    out = subprocess.run(["make", "-s", "-C", NATIVE, "-f", "device_cluster.mk"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("building the cluster-call driver failed:\n" + out.stdout + out.stderr)
    return out.stderr  # ptxas -v report


def load():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB)
        L.cd_prepare.restype = C.c_int
        L.cd_max_clusters.restype = C.c_int
        L.cd_max_clusters.argtypes = [C.c_int]
        L.cd_launch.restype = C.c_int
        L.cd_launch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint64, C.c_uint64,
                                C.c_void_p]
        L.cd_wait.restype = C.c_int
        L.cd_wait.argtypes = [C.c_void_p]
        L.cd_wrong_shape_run.restype = C.c_int
        L.cd_wrong_shape_run.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 5
        L.cd_error.restype = C.c_char_p
        _lib = L
    return _lib


def max_clusters(k):
    """clusters of k CTAs the device can hold at once (0: it cannot place one)"""
    return load().cd_max_clusters(k)


class Runner(bl.Runner):
    """One launch = lists of ops, one cluster of `k` CTAs per list (lists run concurrently, the ops of a list in
    order).  The pinned buffers and run / launch / prepare / wait are those of the block driver's runner."""

    def __init__(self, pkg, k=2):
        self.pkg, self.L, self.D, self.k = pkg, pkg.lib(), load(), k
        assert self.D.cd_prepare() == 0, self.D.cd_error()
        self.bufs = {}

    def fire(self, budget_s=30.0, max_iters=1 << 40, stream=None):
        hp, opp, fp, ops, sizes = self._prepared
        rc = self.D.cd_launch(hp, opp, fp, len(sizes), self.k, int(budget_s * 1e9), max_iters, stream)
        if rc != 0:
            raise RuntimeError("cd_launch: %s" % self.D.cd_error().decode())
        self._pending = (ops, sizes, stream)

    def wait(self):
        ops, sizes, stream = self._pending
        assert self.D.cd_wait(stream) == 0, self.D.cd_error().decode()
        out, k = [], 0
        for n in sizes:
            out.append([dict(ret=ops[k + j].ret, calls=ops[k + j].calls, status=ops[k + j].status) for j in range(n)])
            k += n
        return out

    def wrong_shape(self, handles, send, recv, threads, grid=(1, 1), cluster=(1, 1)):
        """a Send (dict of CdOp fields) and a Recv run by a grid of CTAs of `threads` threads in clusters of
        cluster[0] x cluster[1]: [(ret, calls)] * 2 as CTA (0, 0) saw them"""
        hp, opp, fp, ops = self._fill(handles, [[send, recv]])
        assert self.D.cd_wrong_shape_run(hp, opp, threads, grid[0], grid[1], cluster[0], cluster[1]) == 0, \
            self.D.cd_error().decode()
        return [(ops[i].ret, ops[i].calls) for i in range(2)]


class ClusterEngine(bl.BlockEngine):
    """trace.run_trace adapter: BlockEngine's mapping, with every op of a claimed end run by a cluster of `k` CTAs
    (send / recv: one B200_BATCH_ONE_CALL cluster call; send_all / recv_drain: one B200_BATCH_UNTIL_BLOCKED call).
    `mix_every`: single calls of a claimed end cycle through cluster, block and warp calls -- every `mix_every`-th op
    is a block call from CTA rank 0, the one after it a warp call from its warp 0 -- so the three interleave on one
    pair."""
    kind = "cluster"

    def __init__(self, pkg, k, mem="device", misalign=0, drive=("tx", "rx"), config=None, mix_every=0):
        super().__init__(pkg, mem, misalign, drive, config)
        self.B = Runner(pkg, k)
        self.mix_every = mix_every

    def _run1(self, p, **op):
        self.nops += 1
        if self.mix_every and op.get("flags", 0) == ONE_CALL:
            m = self.nops % (self.mix_every + 1)
            if m == self.mix_every - 1:
                op["kind"] = {SEND: BLOCK_SEND, RECV: BLOCK_RECV}[op["kind"]]
            elif m == self.mix_every:
                op["kind"] = {SEND: WARP_SEND, RECV: WARP_RECV}[op["kind"]]
        res = self.B.run([self.handles[p.h]], [[dict(op, pair=0)]])[0][0]
        assert res["status"] == OK, res
        return res
