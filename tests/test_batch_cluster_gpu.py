"""GPU: batches launched with B200_BATCH_CLUSTER(k), k = 2, 4, 8 and 16 -- every op on a thread-block cluster of k CTAs
(k_cluster_send / k_cluster_recv).

Bar: what the same batch gives with field 0, bit for bit.  Checked against the golden records and the CPU models
(reference with max_sge 1 / 4 / 30 / 32, coalesced, stamped): every count and `calls`, partial_write, cursors and
readiness answers, the delivered bytes and the ring images with pads masked; against twin connections driven by
field-0 batches through the same ops; and on the five memory paths of test_batch_paths_gpu.py with canaries around
every slice and window.  Then batches beside the running service, the refusals, and a cluster Send batch over the
CUDA-IPC wire.  k = 16 is skipped where the device cannot place such a cluster."""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import pytest

import test_coalesce_gpu
import test_gpu_parity
import test_stamp_gpu
import trace
from gpu_engine import GpuEngine
from test_batch_paths_gpu import PATHS, Mem, _check_all, _model_send, _place_recvs, _place_sends, _recv_phase, \
    _send_phase
from test_submit_gpu import MODES, Conn, Service, _lens, _models

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "traces.json")))
_compare = test_gpu_parity._compare
KS = [2, 4, 8, 16]
MEMS = [("device", 0), ("device", 5), ("pinned", 9)]


def placeable(pkg, k):
    """an empty batch prepared with the flag: refused when the device cannot place one cluster of k CTAs"""
    L = pkg.lib()
    b = L.b200_batch_prepare_recv((pkg.RecvOp * 1)(), 0, pkg.cluster_flag(k))
    if not b:
        assert "cannot place" in pkg.last_error(), pkg.last_error()
        return False
    L.b200_batch_destroy(b)
    return True


@pytest.fixture
def k(gpu, request):
    if not placeable(gpu, request.param):
        pytest.skip("this device cannot place a cluster of %d CTAs of the batch kernels" % request.param)
    return request.param


def by_k(f):
    return pytest.mark.parametrize("k", KS, indirect=True)(f)


@pytest.fixture(scope="module")
def models(oracle):
    return _models(oracle)


class BatchEngine(GpuEngine):
    """trace.run_trace's engine with every op a one-op batch launched with B200_BATCH_CLUSTER(k): send / recv with
    B200_BATCH_ONE_CALL (one Send / Recv call), send_all / recv_drain with B200_BATCH_UNTIL_BLOCKED.  mem "pinned":
    the host-staged lanes."""

    def __init__(self, pkg, k, mem="device", misalign=0, config=None):
        super().__init__(pkg, mem, misalign)
        self.fl = pkg.cluster_flag(k)
        self.config = config or {}

    def pair_pair(self, cap, max_sge=30):
        for key, v in self.config.items():
            self.pkg.config_set(key, v)
        try:
            return super().pair_pair(cap, max_sge)
        finally:
            for key in self.config:
                self.pkg.config_set(key, 0)

    def _send(self, p, bufs, byte_idx, flags):
        offs, off = [], self.mis
        for b in bufs:
            offs.append(off)
            off += b.size + 3
        base = self._alloc(off)
        flat = np.zeros(off + 1, dtype=np.uint8)
        for b, o in zip(bufs, offs):
            flat[o:o + b.size] = b
        self._upload(base, flat[:off])
        sl = self.pkg.make_slices([(base + o, b.size) for b, o in zip(bufs, offs)])
        bt = self.pkg.Batch("send", [(p, sl, len(bufs), byte_idx)], flags | self.fl)
        try:
            bt.launch()
            return bt.results()[0], bt.calls()[0]
        finally:
            bt.destroy()
            self._free(base)

    def _recv(self, p, cap, flags):
        base = self._alloc(cap + self.mis)
        bt = self.pkg.Batch("recv", [(p, base + self.mis, cap)], flags | self.fl)
        try:
            bt.launch()
            n, calls = bt.results()[0], bt.calls()[0]
        finally:
            bt.destroy()
        out = self._download(base + self.mis, n).copy()
        self._free(base)
        return out, calls

    def send(self, p, bufs, byte_idx=0):
        return self._send(p, bufs, byte_idx, self.pkg.ONE_CALL)[0]

    def send_all(self, p, bufs, byte_idx=0):
        return self._send(p, bufs, byte_idx, self.pkg.UNTIL_BLOCKED)

    def recv(self, p, cap):
        return self._recv(p, cap, self.pkg.ONE_CALL)[0]

    def recv_drain(self, p, cap):
        return self._recv(p, cap, self.pkg.UNTIL_BLOCKED)


# ---- one-op batches against the golden records and the models

@by_k
def test_golden_traces(gpu, k):
    for i, name in enumerate(sorted(GOLDEN["traces"])):
        t = GOLDEN["traces"][name]
        mem, mis = MEMS[i % 3]
        recs = trace.run_trace(BatchEngine(gpu, k, mem, mis), t["cap"], [tuple(o) for o in t["ops"]],
                               GOLDEN["max_sge"])
        _compare(recs, t["records"], "golden %s k=%d [%s+%d]" % (name, k, mem, mis))


@by_k
@pytest.mark.parametrize("seed", range(2))
def test_random_traces_vs_oracle(gpu, oracle, k, seed):
    rng = np.random.default_rng(8100 + 10 * k + seed)
    cap = [1024, 65536][seed]
    ops = test_gpu_parity._random_ops(rng, cap, 60)
    mem, mis = MEMS[(seed + k) % 3]
    _compare(trace.run_trace(BatchEngine(gpu, k, mem, mis), cap, ops), trace.run_trace(oracle, cap, ops),
             "random seed %d cap %d k=%d [%s+%d]" % (seed, cap, k, mem, mis))


@by_k
@pytest.mark.parametrize("max_sge", [1, 4, 32])
def test_other_max_sge(gpu, oracle, k, max_sge):
    ops = [("send", [7] * 50, 1, 0), ("send_all", [9, 100] * 30, 2, 3), ("recv_drain", 1 << 16),
           ("send_all", [9, 100] * 30, 3, 0), ("recv_drain", 1 << 16), ("send", [5] * 40, 4, 2), ("recv", 3),
           ("send_all", [9, 20000] * 8, 5, 0), ("recv_drain", 1 << 18)]
    want = trace.run_trace(oracle, 1 << 18, ops, max_sge)
    got = trace.run_trace(BatchEngine(gpu, k, "device", 1), 1 << 18, ops, max_sge)
    _compare(got, want, "max_sge %d k=%d" % (max_sge, k))


@by_k
def test_coalesced_vs_model(gpu, models, k):
    rng = np.random.default_rng(8200 + k)
    cap = 65536
    ops = test_coalesce_gpu._random_ops(rng, cap, 50)
    got = trace.run_trace(BatchEngine(gpu, k, "device", 3, config={"B200_SEND_COALESCE": 1}), cap, ops)
    _compare(got, trace.run_trace(models["coal"], cap, ops), "coalesced k=%d" % k)


@by_k
@pytest.mark.parametrize("coalesced", [False, True])
def test_stamped_vs_model(gpu, k, coalesced):
    import stamp_lib
    rng = np.random.default_rng(8300 + 10 * k + coalesced)
    cap = 65536
    mem, mis = MEMS[(k + coalesced) % 3]
    eng = BatchEngine(gpu, k, mem, mis, config={"B200_RING_STAMPED": 1, "B200_SEND_COALESCE": int(coalesced)})
    test_stamp_gpu._replay(eng, stamp_lib.StampedOracle(coalesced=coalesced), cap,
                           test_stamp_gpu._random_ops(rng, cap, 60))


# ---- twin connections: field 0 on one, B200_BATCH_CLUSTER(k) on the other, through the same ops

def _twin_state(c, d):
    """both ends' state and readiness, and the receiver's ring image with pads masked (the bytes the reader never
    looks at)"""
    tx, rx, _, mrx = c.ends(d)
    st, sr = tx.state(), rx.state()
    img = rx.ring_image()
    if c.mode == "stamp":
        img[c.model.pads(mrx)] = 0
    else:
        img = trace.mask_pads(img, sr, c.cap)
    return st, sr, (rx.has_message(), rx.readable(), tx.has_pending_writes(), tx.writable()), img


@pytest.mark.parametrize("path", ["device", "staged", "zerocopy"])
@by_k
def test_twins_match_field_zero(gpu, models, k, path):
    """48 connections in every mode and ring size, twice: rounds of one send batch then one recv batch, the same ops
    on both sets, field 0 on one and k on the other.  Per op bytes and calls, both ends' state and readiness, the ring
    images, and every byte of both arenas are equal; the field-0 set also matches the models."""
    pkg = gpu
    rng = np.random.default_rng(8400 + 10 * k + PATHS.index(path))
    n = 24
    sets = [[Conn(pkg, models, MODES[i % 3], (1024, 4096, 16384, 65536)[(i // 3) % 4]) for i in range(n)]
            for _ in range(2)]
    mems = [Mem(pkg, path, 24 << 20) for _ in range(2)]
    fl = pkg.cluster_flag(k)
    try:
        for r in range(6):
            base = (pkg.ONE_CALL if r % 3 == 2 else pkg.UNTIL_BLOCKED) | mems[0].flags
            plan_s, plan_r = [], []
            for i in range(n):
                for d in (0, 1):
                    if rng.random() < 0.7:
                        lens, bidx = _lens(rng, sets[0][i].cap)
                        plan_s.append((i, d, trace.make_bufs(lens, int(rng.integers(0, 1 << 16))), bidx))
                    if rng.random() < 0.7:
                        plan_r.append((i, d, int(rng.integers(1, 2 * sets[0][i].cap))))
            seed = int(rng.integers(0, 1 << 30))
            got = []
            for conns, mem, f in zip(sets, mems, (base, base | fl)):
                prng = np.random.default_rng(seed)
                mem.reset()
                sends = [[conns[i], d, bufs, bidx] for i, d, bufs, bidx in plan_s]
                recvs = [[conns[i], d, cap, np.zeros(cap, np.uint8)] for i, d, cap in plan_r]
                sls = _place_sends(mem, sends, r % 2 == 1, prng)
                offs = _place_recvs(mem, recvs, prng)
                mem.upload()
                label = "%s k=%d round %d flags %#x" % (path, k, r, f)
                # both sets against the models as well: the models of the two sets advance identically
                _send_phase(pkg, conns, sends, sls, f, "batch", [mem], label)
                _recv_phase(pkg, conns, recvs, mem, offs, f, "batch", [mem], label)
                got.append(([_twin_state(c, d) for c in conns for d in (0, 1)], mem.read(0, mem.hi)))
            (s0, a0), (s1, a1) = got
            for j, (x, y) in enumerate(zip(s0, s1)):
                assert x[:3] == y[:3], "round %d conn %d dir %d: %s vs %s" % (r, j // 2, j % 2, x[:3], y[:3])
                assert np.array_equal(x[3], y[3]), "round %d conn %d dir %d: ring images differ" % (r, j // 2, j % 2)
            assert np.array_equal(a0, a1), "round %d: arenas differ" % r
    finally:
        for conns in sets:
            for c in conns:
                c.close()
        for m in mems:
            m.free()


# ---- the five memory paths with canaries, batches of 1, 3 and 64 ops

def _cluster_rounds(pkg, models, path, k, nops, seed, rounds=4):
    """rounds of one send batch and one recv batch of exactly `nops` ops each (ONE_CALL and UNTIL_BLOCKED in
    turn), the flag B200_BATCH_CLUSTER(k); on the staged paths the lanes permute the ops"""
    rng = np.random.default_rng(seed)
    nconn = (nops + 1) // 2
    conns = [Conn(pkg, models, MODES[i % 3], (1024, 4096, 16384, 65536)[(i // 3) % 4]) for i in range(nconn)]
    mem = Mem(pkg, path, 32 << 20)
    try:
        for r in range(rounds):
            flags = (pkg.ONE_CALL if r % 2 else pkg.UNTIL_BLOCKED) | mem.flags | pkg.cluster_flag(k)
            ends = [(c, d) for c in conns for d in (0, 1)]
            pick_s = [ends[i] for i in rng.permutation(len(ends))[:nops]]
            pick_r = [ends[i] for i in rng.permutation(len(ends))[:nops]]
            sends = []
            for c, d in pick_s:
                lens, bidx = _lens(rng, c.cap)
                sends.append([c, d, trace.make_bufs(lens, int(rng.integers(0, 1 << 16))), bidx])
            recvs = []
            for c, d in pick_r:
                cap = int(rng.integers(1, 2 * c.cap))
                recvs.append([c, d, cap, np.zeros(cap, np.uint8)])
            mem.reset()
            sls = _place_sends(mem, sends, r % 2 == 1, rng)
            offs = _place_recvs(mem, recvs, rng)
            mem.upload()
            label = "%s k=%d %d ops round %d" % (path, k, nops, r)
            _send_phase(pkg, conns, sends, sls, flags, "batch", [mem], label)
            _recv_phase(pkg, conns, recvs, mem, offs, flags, "batch", [mem], label)
    finally:
        for c in conns:
            c.close()
        mem.free()


@pytest.mark.parametrize("path", PATHS)
@by_k
def test_memory_paths_with_canaries(gpu, models, k, path):
    for j, nops in enumerate((1, 3, 64)):
        _cluster_rounds(gpu, models, path, k, nops, 8500 + 100 * k + 10 * PATHS.index(path) + j)


@pytest.mark.parametrize("path", ["device", "staged"])
@pytest.mark.parametrize("k", [4], indirect=True)
def test_pairs_send_recv_and_relaunch(gpu, models, k, path):
    """b200_pairs_send / recv take the flag, and a prepared cluster batch relaunched over several ring laps keeps
    matching the models"""
    pkg = gpu
    rng = np.random.default_rng(8600 + PATHS.index(path))
    conns = [Conn(pkg, models, MODES[i % 3], 16384) for i in range(6)]
    mem = Mem(pkg, path, 16 << 20)
    try:
        fl = pkg.UNTIL_BLOCKED | pkg.cluster_flag(k)
        sends = []
        for c in conns:
            for d in (0, 1):
                lens = [9, int(rng.integers(2000, 8000)), 9, int(rng.integers(1, 200))]
                sends.append([c, d, trace.make_bufs(lens, int(rng.integers(0, 1 << 16))), 3])
        recvs = [[c, d, 20000, np.zeros(20000, np.uint8)] for c in conns for d in (0, 1)]
        sls = _place_sends(mem, sends, False, rng)
        offs = _place_recvs(mem, recvs, rng)
        mem.upload()
        _send_phase(pkg, conns, sends, sls, fl, "pairs", [mem], "pairs_send k=%d" % k)
        _recv_phase(pkg, conns, recvs, mem, offs, fl, "pairs", [mem], "pairs_recv k=%d" % k)
        bs = pkg.Batch("send", [(c.ends(d)[0], sl, len(b), i) for (c, d, b, i), sl in zip(sends, sls)], fl)
        br = pkg.Batch("recv", [(c.ends(d)[1], mem.ptr(o), cap) for (c, d, cap, _), o in zip(recvs, offs)], fl)
        try:
            for lap in range(8):
                bs.launch()
                want = [_model_send(op, True) for op in sends]
                assert list(zip(bs.results(), bs.calls())) == want, "lap %d" % lap
                br.launch()
                res, calls = br.results(), br.calls()
                for i, op in enumerate(recvs):
                    c, d, cap = op[:3]
                    out, mc = c.model.recv_drain(c.ends(d)[3], cap)
                    assert (res[i], calls[i]) == (out.size, mc), "lap %d op %d" % (lap, i)
                    assert trace.sha(mem.read(offs[i], res[i])) == trace.sha(out), "lap %d op %d" % (lap, i)
                    mem.land(offs[i], cap, out, op[3])
                _check_all(conns, [mem], "lap %d" % lap)
        finally:
            bs.destroy()
            br.destroy()
    finally:
        for c in conns:
            c.close()
        mem.free()


# ---- beside the running service

def _pinned(L, n):
    p = L.b200_mem_alloc_host(n)
    assert p
    return p, np.ctypeslib.as_array((C.c_uint8 * n).from_address(p))


@pytest.mark.parametrize("batch_end", ["tx", "rx"])
@pytest.mark.parametrize("k", [2, 8], indirect=True)
def test_cluster_batch_beside_the_service(gpu, k, batch_end):
    """The service runs at its default size.  One end of a connection runs cluster batches (device memory) while the
    other end makes single calls through the owners and the pool at the same time: 240 chttp2-like slices through a
    16 KiB ring, lapped many times.  Every wait is bounded; the stream arrives whole, cursors and readiness agree."""
    pkg, L = gpu, gpu.lib()
    fl = pkg.cluster_flag(k)
    lens = [9, 1000, 9, 3000, 9, 500, 17, 2048] * 30
    total = sum(lens)
    rng = np.random.default_rng(8700 + k)
    src_np = rng.integers(0, 256, total, dtype=np.uint8)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(int)
    dev = L.b200_mem_alloc_device(total)
    assert L.b200_memcpy(dev, src_np.ctypes.data, total, 0, None) == 0
    assert L.b200_stream_sync(None) == 0
    hsrc, hsrc_np = _pinned(L, total)
    hsrc_np[:] = src_np
    hdst, hdst_np = _pinned(L, total)
    hdst_np[:] = 0
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 16384)
    tx, rx = pkg.connected_pair("cbs-tx-%s-%d" % (batch_end, k), "cbs-rx-%s-%d" % (batch_end, k))
    try:
        with Service(pkg, workers=0, arena=1 << 20):
            deadline = time.time() + 120
            idx = bidx = moved = got = 0
            if batch_end == "tx":
                while got < total and time.time() < deadline:
                    b = None
                    if idx < len(lens):
                        sl = pkg.make_slices([(dev + int(offs[j]), lens[j]) for j in range(idx, len(lens))])
                        b = pkg.Batch("send", [(tx, sl, len(lens) - idx, bidx)], pkg.UNTIL_BLOCKED | fl)
                        b.launch()
                    got += rx.recv_into(hdst + got, total - got)  # single calls beside the batch
                    if b is not None:
                        sent = b.results()[0]
                        b.destroy()
                        moved += sent
                        while sent > 0:
                            left = lens[idx] - bidx
                            if sent >= left:
                                sent, idx, bidx = sent - left, idx + 1, 0
                            else:
                                bidx, sent = bidx + sent, 0
                assert moved == total, "batch sender stalled at %d of %d" % (moved, total)
                assert got == total, "single-call receiver stalled at %d of %d" % (got, total)
                out = hdst_np
            else:
                dst_dev = L.b200_mem_alloc_device(total)
                while got < total and time.time() < deadline:
                    b = pkg.Batch("recv", [(rx, dst_dev + got, total - got)], pkg.UNTIL_BLOCKED | fl)
                    b.launch()
                    if idx < len(lens):  # single calls beside the batch
                        window = [(hsrc + int(offs[j]), lens[j]) for j in range(idx, min(idx + 4, len(lens)))]
                        sent = tx.send_raw(window, bidx)
                        moved += sent
                        while sent > 0:
                            left = lens[idx] - bidx
                            if sent >= left:
                                sent, idx, bidx = sent - left, idx + 1, 0
                            else:
                                bidx, sent = bidx + sent, 0
                    got += b.results()[0]
                    b.destroy()
                assert moved == total and got == total, "stalled: sent %d, received %d of %d" % (moved, got, total)
                out = np.zeros(total, np.uint8)
                assert L.b200_memcpy(out.ctypes.data, dst_dev, total, 1, None) == 0
                assert L.b200_stream_sync(None) == 0
                L.b200_mem_free_device(dst_dev)
            assert np.array_equal(out, src_np)
            st, sr = tx.state(), rx.state()
            assert sr["head"] == sr["moving_head"] == st["remote_tail"] and sr["remain"] == 0
            assert st["partial_write"] == 0
            assert not rx.has_message() and rx.readable() == 0 and not tx.has_pending_writes()
    finally:
        for p in (tx, rx):
            p.disconnect()
            p.putback()
        L.b200_mem_free_device(dev)
        L.b200_mem_free_host(hsrc)
        L.b200_mem_free_host(hdst)


# ---- refusals

def test_refusals_change_nothing(gpu):
    pkg, L = gpu, gpu.lib()
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 4096)
    a, b = pkg.connected_pair("bcref-a", "bcref-b")
    dev = L.b200_mem_alloc_device(4096)
    hbuf, hbuf_np = _pinned(L, 4096)
    msg = np.arange(100, dtype=np.uint8)
    assert b.send([msg]) == 100  # a frame waits in a's ring
    fl2 = pkg.cluster_flag(2)
    sl = pkg.make_slices([(dev, 100)])

    def snap():
        return a.state(), b.state(), a.ring_image().copy(), b.ring_image().copy()

    def same(x, y):
        return x[:2] == y[:2] and np.array_equal(x[2], y[2]) and np.array_equal(x[3], y[3])

    try:
        before = snap()
        # a device-claimed end: prepare refuses it with or without the field, and so does the launch of a batch
        # prepared before the claim
        prepared = pkg.Batch("recv", [(a, dev, 4096)], pkg.UNTIL_BLOCKED | fl2)
        a.device_claim()
        for f in (0, fl2, pkg.cluster_flag(8)):
            assert not L.b200_batch_prepare_recv((pkg.RecvOp * 1)(pkg.RecvOp(a.h, dev, 4096)), 1, f)
            assert "device-owned" in pkg.last_error() or "claim" in pkg.last_error(), pkg.last_error()
        assert L.b200_batch_launch(prepared.h, None) == -1
        prepared.destroy()
        a.device_release()
        assert same(snap(), before)
        # b200_pairs_submit and the post calls refuse the field, without and with the service
        sop = (pkg.SendOp * 1)(pkg.SendOp(b.h, sl, 1, 0))
        rop = (pkg.RecvOp * 1)(pkg.RecvOp(a.h, hbuf, 4096))
        acc, dlv = (C.c_uint64 * 1)(), (C.c_uint64 * 1)()
        for f in (fl2, pkg.cluster_flag(16) | pkg.UNTIL_BLOCKED):
            assert L.b200_pairs_submit(sop, 1, acc, rop, 1, dlv, f) == -1
            assert "B200_BATCH_CLUSTER" in pkg.last_error(), pkg.last_error()
        assert same(snap(), before)
        with Service(pkg, workers=4, arena=1 << 20):
            again = C.c_int(7)
            for f in (fl2, pkg.cluster_flag(4) | pkg.UNTIL_BLOCKED):
                assert L.b200_pairs_submit(sop, 1, acc, rop, 1, dlv, f) == -1
                assert "B200_BATCH_CLUSTER" in pkg.last_error()
                again.value = 7
                assert not L.b200_pair_post_send(b.h, sl, 1, 0, f, C.byref(again)) and again.value == 0
                assert "B200_BATCH_CLUSTER" in pkg.last_error()
                again.value = 7
                assert not L.b200_pair_post_recv(a.h, hbuf, 4096, f, C.byref(again)) and again.value == 0
                assert "B200_BATCH_CLUSTER" in pkg.last_error()
            assert same(snap(), before)
            # and the same calls with field 0 work: the frame is delivered through the service
            assert L.b200_pairs_submit(sop, 0, acc, rop, 1, dlv, 0) == 0 and dlv[0] == 100
            assert np.array_equal(hbuf_np[:100], msg)
        # bits above 7 are ignored, as before
        hbuf_np[:] = 0
        assert b.send([msg]) == 100
        bt = pkg.Batch("recv", [(a, hbuf, 4096)], pkg.UNTIL_BLOCKED | 0x100 | fl2)
        bt.launch()
        assert bt.results() == [100] and bt.calls() == [1]
        bt.destroy()
        assert np.array_equal(hbuf_np[:100], msg)
    finally:
        for p in (a, b):
            p.disconnect()
            p.putback()
        L.b200_mem_free_device(dev)
        L.b200_mem_free_host(hbuf)


# ---- the CUDA-IPC wire: a cluster Send batch in one process, a field-0 receiver in another (one GPU)

@pytest.mark.parametrize("k", [2, 8], indirect=True)
def test_cluster_send_batch_over_the_ipc_wire(k):
    """3 x 1 MiB chttp2-shaped messages through a 256 KiB ring: the cluster batch's frames land in the other process's
    ring and it needs the credit that comes back over the wire (system scope) to go on."""
    with tempfile.TemporaryDirectory() as d:
        procs = [subprocess.Popen([sys.executable, os.path.join(HERE, "batch_cluster_ipc_worker.py"), str(k), role,
                                   "0", d, "256", str(1 << 20), "3"], stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT, text=True)
                 for role in ("server", "client")]
        try:
            outs = [p.communicate(timeout=400)[0] for p in procs]
        finally:
            for p in procs:
                if p.poll() is None:
                    p.kill()
                    p.wait()
        assert all(p.returncode == 0 for p in procs), "\n".join(outs)
        cli, srv = [json.load(open(os.path.join(d, r + ".json"))) for r in ("client", "server")]
    assert cli["ok"] and not cli["pending"] and min(cli["calls"]) > 1
    assert srv["ok"] and srv["ring_empty"] and srv["half_closed"]
    assert cli["state"]["remote_tail"] == srv["state"]["head"] == srv["state"]["moving_head"]
