"""GPU: coalesced send framing (B200_SEND_COALESCE=1, DESIGN.md §2) on the CUDA path against the coalesced model
(tests/native/coalesce_oracle.c).  Same bit-exact bar as test_gpu_parity.py: every return value, `calls`, cursor,
readiness answer and the receiver's ring image with pads masked, through k_send (single calls, prepared batches),
the service's owner warps and pool, the endpoint, and the NVLink wire."""
import ctypes as C
import os
import subprocess
import sys
import tempfile
import json

import numpy as np
import pytest

import coalesce_lib
import endpoint_lib
import trace
from gpu_engine import GpuEngine

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
HERE = os.path.dirname(os.path.abspath(__file__))


class CoalescedGpuEngine(GpuEngine):
    """Pairs initialised in coalesced mode; the runtime's default is put back once they exist."""

    def pair_pair(self, cap, max_sge=30):
        self.pkg.config_set("B200_SEND_COALESCE", 1)
        try:
            return super().pair_pair(cap, max_sge)
        finally:
            self.pkg.config_set("B200_SEND_COALESCE", 0)


@pytest.fixture(scope="module")
def co():
    return coalesce_lib.CoalescedOracle()


def _compare(got, want, label):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, "%s: op %d (%s)\n got  %s\n want %s" % (label, i, w["op"], g, w)


def _random_ops(rng, cap, n_ops, max_slices=40, small=False):
    ops = []
    for _ in range(n_ops):
        k = rng.integers(0, 5)
        if k < 2:
            n = int(rng.integers(1, max_slices))
            style = rng.integers(0, 5)
            if style == 0:
                lens = [int(x) for x in rng.integers(1, 64, n)]
            elif style == 1:
                lens = [9 if i % 2 == 0 else int(rng.integers(1, min(16385, cap))) for i in range(n)]
            elif style == 2:
                lens = [int(x) for x in rng.integers(1, 2 * cap, max(1, n // 8))]
            elif style == 3:
                lens = [int(x) for x in rng.integers(0, 20, n)]           # zero-length slices included
            else:
                lens = [int(x) for x in rng.integers(1, 4, int(rng.integers(1, 1300)))]  # > 1024 slices
            if small:
                lens = [min(x, 1500) for x in lens[:5]]
            bidx = int(rng.integers(0, lens[0])) if lens[0] else 0
            ops.append(("send" if k == 0 or small else "send_all", lens, int(rng.integers(0, 1000)), bidx))
        elif k == 2:
            ops.append(("recv", int(rng.integers(1, cap))))
        else:
            ops.append(("recv_drain", int(rng.integers(1, 2 * cap))))
    return ops


@pytest.mark.parametrize("seed", range(10))
def test_random_traces_vs_coalesced_oracle(gpu, co, seed):
    rng = np.random.default_rng(9000 + seed)
    cap = [64, 1024, 2048, 4096, 65536][seed % 5]
    ops = _random_ops(rng, cap, 80)
    want = trace.run_trace(co, cap, ops)
    mem, mis = [("device", 0), ("device", 5), ("pinned", 9)][seed % 3]
    got = trace.run_trace(CoalescedGpuEngine(gpu, mem, mis), cap, ops)
    _compare(got, want, "coalesced random seed %d cap %d [%s+%d]" % (seed, cap, mem, mis))


def test_every_relative_alignment(gpu, co):
    """16 source alignments x 16 frame offsets of the first slice's bytes (byte_idx), partial reads after."""
    cap = 8192
    for mis in range(16):
        ops = []
        for b in range(16):
            ops += [("send_all", [9 + b, 1000 + mis, 37, 5, 9, 3], 50 + mis, b), ("recv", 3 + mis), ("recv_drain", 4000)]
        want = trace.run_trace(co, cap, ops)
        got = trace.run_trace(CoalescedGpuEngine(gpu, "device", mis), cap, ops)
        _compare(got, want, "coalesced alignment %d" % mis)


def test_single_calls_from_unregistered_memory(gpu, co):
    """b200_pair_send with plain host memory: the bounce staging of up to 1024 slices of one coalesced call."""
    cap = 65536
    ops = [("send", [9, 16384] * 40, 1, 0), ("recv_drain", 1 << 17), ("send", [1] * 1100, 2, 0), ("recv", 1 << 16),
           ("send", [7] * 1100, 3, 3), ("recv_drain", 1 << 17), ("send", [30000, 30000], 4, 100), ("recv_drain", 1 << 17)]
    _compare(trace.run_trace(CoalescedGpuEngine(gpu, "device", 0), cap, ops), trace.run_trace(co, cap, ops),
             "coalesced single calls")


def test_full_size_stream(gpu):
    """16 MiB rings, 4 MiB chttp2-shaped messages (514 slices), 4 connections in one batch, 9 messages each (the
    ring wraps twice): round trip is the identity, ONE frame per message (1 Send call, 1 Recv call) and an
    all-zero ring after the drain."""
    pkg, L = gpu, gpu.lib()
    pkg.config_set("GRPC_RDMA_RING_BUFFER_SIZE_KB", 16384)
    pkg.config_set("B200_SEND_COALESCE", 1)
    nconn = 4
    lens = pkg.chttp2_slice_lens(4 * 1024 * 1024)
    total = sum(lens)
    try:
        pairs = [pkg.connected_pair("cfs-tx%d" % c, "cfs-rx%d" % c) for c in range(nconn)]
    finally:
        pkg.config_set("B200_SEND_COALESCE", 0)
    src = L.b200_mem_alloc_device(nconn * total)
    dst = L.b200_mem_alloc_device(nconn * total)
    host = np.zeros((nconn, total), dtype=np.uint8)
    for c in range(nconn):
        i = np.arange(total, dtype=np.uint64)
        host[c] = ((i * np.uint64(2654435761) >> np.uint64(13)) + np.uint64(131 * c)) & np.uint64(255)
    assert L.b200_memcpy(src, host.ctypes.data, host.size, 0, None) == 0
    L.b200_stream_sync(None)
    sops, rops, keep = [], [], []
    for c in range(nconn):
        off, sl = 0, []
        for n in lens:
            sl.append((src + c * total + off, n))
            off += n
        arr = pkg.make_slices(sl)
        keep.append(arr)
        sops.append((pairs[c][0], arr, len(lens), 0))
        rops.append((pairs[c][1], dst + c * total, total))
    bs = pkg.Batch("send", sops, pkg.UNTIL_BLOCKED)
    br = pkg.Batch("recv", rops, pkg.UNTIL_BLOCKED)
    enc = 16 + (total + 7) // 8 * 8
    out = np.zeros_like(host)
    for it in range(9):
        bs.launch()
        br.launch()
        assert bs.results() == [total] * nconn and bs.calls() == [1] * nconn
        assert br.results() == [total] * nconn and br.calls() == [1] * nconn
        assert L.b200_memcpy(out.ctypes.data, dst, out.size, 1, None) == 0
        L.b200_stream_sync(None)
        assert np.array_equal(out, host), "iteration %d" % it
        for tx, rx in pairs:
            st, sr = tx.state(), rx.state()
            assert st["remote_tail"] == (enc * (it + 1)) % (16 << 20)
            assert sr["head"] == sr["moving_head"] == st["remote_tail"] and sr["remain"] == 0
            assert st["partial_write"] == 0 and not rx.has_message()
    for _, rx in pairs:
        assert not rx.ring_image().any(), "ring must read as all zero after a full drain"
    bs.destroy()
    br.destroy()
    L.b200_mem_free_device(src)
    L.b200_mem_free_device(dst)
    for tx, rx in pairs:
        tx.disconnect(); rx.disconnect(); tx.putback(); rx.putback()


def test_mixed_modes_in_one_batch(gpu, co, oracle):
    """A coalesced pair and a per-slice pair in the same batch launches: each matches its own model."""
    pkg = gpu
    cap = 16384
    lens = [9, 3000, 9, 17, 9, 2000, 9, 5000, 9, 700] * 3
    bufs = trace.make_bufs(lens, 31)
    flat = np.concatenate(bufs)
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", cap)
    pkg.config_set("GRPC_RDMA_MAX_SGE", 30)
    pkg.config_set("B200_SEND_COALESCE", 1)
    try:
        ctx, crx = pkg.connected_pair("mix-ctx", "mix-crx")
    finally:
        pkg.config_set("B200_SEND_COALESCE", 0)
    ptx, prx = pkg.connected_pair("mix-ptx", "mix-prx")
    L = pkg.lib()
    src = L.b200_mem_alloc_device(flat.size)
    assert L.b200_memcpy(src, flat.ctypes.data, flat.size, 0, None) == 0 and L.b200_stream_sync(None) == 0
    dst = [L.b200_mem_alloc_device(1 << 16) for _ in range(2)]
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    arr = pkg.make_slices([(src + int(o), n) for o, n in zip(offs, lens)])
    models = [(co, co.pair_pair(cap)), (oracle, oracle.pair_pair(cap))]
    idx = [(0, 0), (0, 0)]
    for rnd in range(6):
        ops = [(p, arr, len(lens), 0) for p in (ctx, ptx)]
        want = []
        for k, (eng, (mtx, mrx)) in enumerate(models):
            want.append(eng.send_all(mtx, bufs, 0))
        bs = pkg.Batch("send", ops, pkg.UNTIL_BLOCKED)
        bs.launch()
        got = list(zip(bs.results(), bs.calls()))
        bs.destroy()
        assert got == [tuple(w) for w in want], (rnd, got, want)
        br = pkg.Batch("recv", [(crx, dst[0], 1 << 16), (prx, dst[1], 1 << 16)], pkg.UNTIL_BLOCKED)
        br.launch()
        rgot = list(zip(br.results(), br.calls()))
        br.destroy()
        rwant = []
        for k, (eng, (mtx, mrx)) in enumerate(models):
            out, calls = eng.recv_drain(mrx, 1 << 16)
            rwant.append((out.size, calls))
            dev = np.zeros(max(out.size, 1), np.uint8)
            assert L.b200_memcpy(dev.ctypes.data, dst[k], out.size, 1, None) == 0 and L.b200_stream_sync(None) == 0
            assert np.array_equal(dev[:out.size], out)
        assert rgot == rwant, (rnd, rgot, rwant)
        for (eng, (mtx, mrx)), (tx, rx) in zip(models, [(ctx, crx), (ptx, prx)]):
            assert tx.state()["remote_tail"] == eng.state(mtx)["remote_tail"]
            assert rx.state()["head"] == eng.state(mrx)["head"]
            assert np.array_equal(trace.mask_pads(rx.ring_image(), rx.state(), cap),
                                  trace.mask_pads(eng.ring_image(mrx), eng.state(mrx), cap))
    for eng, (mtx, mrx) in models:
        eng.destroy(mtx), eng.destroy(mrx)
    for p in (ctx, crx, ptx, prx):
        p.disconnect(); p.putback()
    L.b200_mem_free_device(src)
    for d in dst:
        L.b200_mem_free_device(d)


# ---- endpoint (host slices -> coalesced k_send -> ring -> k_recv -> host slices)

@pytest.fixture(scope="module")
def drv(gpu):
    D, _ = endpoint_lib.load(gpu, need_oracle=False)
    return D


def _endpoint(gpu, ring):
    gpu.config_set("B200_RING_BUFFER_SIZE_BYTES", ring)
    gpu.config_set("GRPC_RDMA_MAX_SGE", 30)
    gpu.config_set("B200_SEND_COALESCE", 1)


def test_endpoint_conformance_and_echo(gpu, drv):
    try:
        _endpoint(gpu, 4 << 20)
        assert drv.drv_read_and_write(None, 10_000_000, 100_000, 8192, 0, 100, 0, None) == 0
        _endpoint(gpu, 65536)
        assert drv.drv_read_and_write(None, 20_000, 5_000, 1, 0, 100, 0, None) == 0
        assert drv.drv_read_and_write(None, 3_000_000, 3_000_000, 100_000, 0, 100, 0, None) == 0
        _endpoint(gpu, 1024)
        for i in (5, 9, 64, 513, 999):
            assert drv.drv_read_and_write(None, 40320, i, i, 0, 100, 0, None) == 0, i
        _endpoint(gpu, 4 << 20)
        nbytes = C.c_uint64(0)
        assert drv.drv_echo(None, 24, 4 * 1024 * 1024 - 1024, 777, 0, 1, 1, C.byref(nbytes)) == 0
        assert nbytes.value > 0
    finally:
        gpu.config_set("B200_SEND_COALESCE", 0)


# ---- the service: owner warps (small coalesced Send, eager push) and the pool

@pytest.fixture
def svc(gpu):
    L = gpu.lib()
    assert L.b200_service_start(4) == 0, gpu.last_error()
    yield gpu
    L.b200_service_stop()


@pytest.mark.parametrize("seed", range(4))
def test_traces_through_the_service(svc, co, seed):
    rng = np.random.default_rng(9500 + seed)
    cap = [1024, 4096, 65536, 1 << 20][seed]
    L = svc.lib()
    hits = L.b200_service_eager_hits()
    for small in (True, False):
        ops = _random_ops(rng, cap, 60, small=small)
        want = trace.run_trace(co, cap, ops)
        got = trace.run_trace(CoalescedGpuEngine(svc, "pinned", 3), cap, ops)
        _compare(got, want, "coalesced service seed %d cap %d small=%s" % (seed, cap, small))
    # unary-shaped calls: 5-byte prefix + message as separate slices, recv right after
    ops = []
    for k in range(20):
        ops += [("send", [9, 5, 100 + 37 * k], 40 + k, 0), ("recv", 1 << 16)]
    _compare(trace.run_trace(CoalescedGpuEngine(svc, "pinned", 3), cap, ops), trace.run_trace(co, cap, ops),
             "coalesced unary [service]")
    assert L.b200_service_eager_hits() > hits  # the owner pushed coalesced frames to the receiver's host slot


# ---- NVLink wire (two GPUs)

def test_stream_across_two_gpus_coalesced():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs on one machine")
    env = dict(os.environ, B200_SEND_COALESCE="1")
    with tempfile.TemporaryDirectory() as d:
        procs = [subprocess.Popen([sys.executable, os.path.join(HERE, "ipc_wire_worker.py"), role, str(dev), d,
                                   "4096", str(1 << 20), "6", "4"],
                                  stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
                 for role, dev in (("server", 1), ("client", 0))]
        outs = [p.communicate(timeout=500)[0] for p in procs]
        assert all(p.returncode == 0 for p in procs), "\n".join(outs)
        srv = json.load(open(os.path.join(d, "server.json")))
    assert srv["ok"] and srv["ring_empty"] and srv["half_closed"]
