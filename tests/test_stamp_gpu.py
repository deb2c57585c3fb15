"""GPU: stamped ring frames (B200_RING_STAMPED=1, DESIGN.md §2) on the CUDA path against the stamped model
(tests/native/stamp_oracle.c), bit for bit: return values, `calls`, cursors, readiness answers and the receiver's
ring image with the pad bytes of every frame image masked (retired frames stay in a stamped ring, so their pads
are part of the image)."""
import numpy as np
import pytest

import stamp_lib
import test_stamp_cpu
import trace
from gpu_engine import GpuEngine

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]


class StampedGpuEngine(GpuEngine):
    """Pairs initialised with B200_RING_STAMPED=1 (and B200_SEND_COALESCE when asked); defaults put back."""

    def __init__(self, pkg, mem="device", misalign=0, coalesced=False):
        super().__init__(pkg, mem, misalign)
        self.coalesced = coalesced

    def pair_pair(self, cap, max_sge=30):
        self.pkg.config_set("B200_RING_STAMPED", 1)
        self.pkg.config_set("B200_SEND_COALESCE", int(self.coalesced))
        try:
            tx, rx = super().pair_pair(cap, max_sge)
        finally:
            self.pkg.config_set("B200_RING_STAMPED", 0)
            self.pkg.config_set("B200_SEND_COALESCE", 0)
        assert tx.stamped() and rx.stamped()
        return tx, rx


def _stream(e, tx, rx, op):
    """the closed loop of trace.run_trace's "stream" op: (bytes, rounds, SHA-1, intact)"""
    _, lens, seed, rcap = op
    bufs = trace.make_bufs(lens, seed)
    idx = bidx = rounds = got = 0
    parts = []
    total = sum(int(x) for x in lens)
    while got < total and rounds < 10000:
        rounds += 1
        if idx < len(bufs):
            sent, _ = e.send_all(tx, bufs[idx:], bidx)
            while sent > 0:
                left = bufs[idx].size - bidx
                if sent >= left:
                    sent, idx, bidx = sent - left, idx + 1, 0
                else:
                    bidx, sent = bidx + sent, 0
        out, _ = e.recv_drain(rx, rcap)
        got += out.size
        parts.append(out)
    allb = np.concatenate(parts)
    return (int(allb.size), rounds, trace.sha(allb), bool(np.array_equal(allb, np.concatenate(bufs))))


def _replay(eng, model, cap, ops, images=True):
    """trace.run_trace on both, op by op, plus the masked ring image after every op."""
    gtx, grx = eng.pair_pair(cap)
    mtx, mrx = model.pair_pair(cap)
    try:
        for i, op in enumerate(ops):
            recs = []
            for e, tx, rx in ((eng, gtx, grx), (model, mtx, mrx)):
                rec = {}
                if op[0] in ("send", "send_all"):
                    bufs = trace.make_bufs(op[1], op[2])
                    rec["ret"] = e.send(tx, bufs, op[3]) if op[0] == "send" else e.send_all(tx, bufs, op[3])
                elif op[0] == "recv":
                    out = e.recv(rx, op[1])
                    rec["ret"], rec["sha"] = int(out.size), trace.sha(out)
                elif op[0] == "stream":
                    rec["ret"] = _stream(e, tx, rx, op)
                else:
                    out, calls = e.recv_drain(rx, op[1])
                    rec["ret"], rec["sha"] = (int(out.size), int(calls)), trace.sha(out)
                st_tx, st_rx = e.state(tx), e.state(rx)
                rec["tx"] = {k: st_tx[k] for k in ("remote_tail", "partial_write", "credit_remote_head")}
                rec["rx"] = {k: st_rx[k] for k in ("head", "moving_head", "remain", "internal_read_size")}
                rec["ready"] = (int(e.has_message(rx)), int(e.readable(rx)), int(e.has_pending_writes(tx)),
                                int(e.writable(tx)))
                recs.append(rec)
            g, w = recs
            for r in recs:
                r["ret"] = tuple(x if isinstance(x, (str, bool)) else int(x) for x in np.atleast_1d(r["ret"]).tolist())
            assert g == w, "op %d %s\n got  %s\n want %s" % (i, op[0], g, w)
            if images:
                pads = model.pads(mrx)
                gi, wi = eng.ring_image(grx), model.ring_image(mrx)
                gi[pads] = 0
                wi[pads] = 0
                bad = np.flatnonzero(gi != wi)
                assert bad.size == 0, "op %d %s: ring differs at %s" % (i, op[0], bad[:16])
    finally:
        eng.destroy(gtx)
        eng.destroy(grx)
        model.destroy(mtx)
        model.destroy(mrx)


@pytest.fixture(scope="module")
def so():
    return stamp_lib.StampedOracle()


@pytest.fixture(scope="module")
def soc():
    return stamp_lib.StampedOracle(coalesced=True)


def _golden():
    import json
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "traces.json")) as f:
        return json.load(f)["traces"]


@pytest.mark.parametrize("mem", [("device", 0), ("device", 5), ("pinned", 9)])
def test_golden_traces_vs_stamped_model(gpu, so, mem):
    for name, t in sorted(_golden().items()):
        _replay(StampedGpuEngine(gpu, *mem), so, t["cap"], [tuple(o) for o in t["ops"]],
                images=t["cap"] <= 1 << 17)


def _random_ops(rng, cap, n_ops):
    ops = []
    for _ in range(n_ops):
        k = rng.integers(0, 5)
        if k < 2:
            n = int(rng.integers(1, 40))
            style = rng.integers(0, 3)
            if style == 0:
                lens = [int(x) for x in rng.integers(1, 64, n)]
            elif style == 1:
                lens = [9 if i % 2 == 0 else int(rng.integers(1, min(16385, cap))) for i in range(n)]
            else:
                lens = [int(x) for x in rng.integers(1, 2 * cap, max(1, n // 8))]
            bidx = int(rng.integers(0, lens[0]))
            ops.append(("send" if k == 0 else "send_all", lens, int(rng.integers(0, 1000)), bidx))
        elif k == 2:
            ops.append(("recv", int(rng.integers(1, cap))))
        else:
            ops.append(("recv_drain", int(rng.integers(1, 2 * cap))))
    return ops


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("coalesced", [False, True])
def test_random_traces_vs_stamped_model(gpu, so, soc, seed, coalesced):
    rng = np.random.default_rng(7100 + seed)
    cap = [64, 1024, 4096, 65536][seed % 4]
    mem, mis = [("device", 0), ("device", 3), ("pinned", 11)][seed % 3]
    _replay(StampedGpuEngine(gpu, mem, mis, coalesced), soc if coalesced else so, cap, _random_ops(rng, cap, 120))


def test_every_relative_alignment(gpu, so):
    cap = 8192
    for mis in range(16):
        ops = []
        for b in range(16):
            ops += [("send_all", [9 + b, 1000 + mis, 37, 5, 9, 3], 50 + mis, b), ("recv", 3 + mis),
                    ("recv_drain", 4000)]
        _replay(StampedGpuEngine(gpu, "device", mis), so, cap, ops)


@pytest.mark.parametrize("coalesced", [False, True])
def test_full_size_laps(gpu, so, soc, coalesced):
    """16 MiB ring, 4 MiB chttp2 messages through closed loops for more than three laps (no images: cursors,
    returns and every delivered byte)."""
    lens = gpu.chttp2_slice_lens(4 << 20)
    ops = []
    for k in range(14):
        ops += [("send_all", lens, 500 + k, 0), ("recv_drain", [1 << 20, 5 << 20, 300000][k % 3]),
                ("recv_drain", 1 << 25)]
    _replay(StampedGpuEngine(gpu, "device", 0, coalesced), soc if coalesced else so, 16 << 20, ops, images=False)


def test_negotiation(gpu):
    pkg = gpu
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 4096)
    pkg.config_set("B200_RING_STAMPED", 1)
    try:
        a = pkg.Pair("neg-a")
    finally:
        pkg.config_set("B200_RING_STAMPED", 0)
    b = pkg.Pair("neg-b")
    assert a.connect(b.address()) and b.connect(a.address())
    assert not a.stamped() and not b.stamped()
    assert a.send([np.arange(100, dtype=np.uint8)]) == 100
    assert b.recv(1000).tolist() == list(range(100))
    assert not b.ring_image().any(), "a default connection clears what it reads"
    for p in (a, b):
        p.disconnect()
    pkg.config_set("B200_RING_STAMPED", 1)
    try:
        for p in (a, b):
            p.L.b200_pair_init(p.h)
    finally:
        pkg.config_set("B200_RING_STAMPED", 0)
    assert a.connect(b.address()) and b.connect(a.address())
    assert a.stamped() and b.stamped()
    assert a.send([np.arange(100, dtype=np.uint8)]) == 100
    assert b.recv(1000).tolist() == list(range(100))
    assert b.ring_image().any() and not b.has_message() and b.readable() == 0
    for p in (a, b):
        p.disconnect()
        p.putback()


@pytest.mark.parametrize("coalesced", [False, True])
def test_idle_ring_full_of_stale_frames(gpu, coalesced):
    """Message shapes whose ring bytes divide the ring: after every drain from the second lap on, the head sits on
    a complete frame of the last lap.  The poller scan reports nothing, readiness is 0 and Recv returns 0."""
    import ctypes as C
    pkg = gpu
    cap = 1 << 16
    eng = StampedGpuEngine(pkg, coalesced=coalesced)
    tx, rx = eng.pair_pair(cap)
    handles = (C.c_void_p * 1)(rx.h)
    ev = (C.c_uint32 * 1)()
    try:
        lens = test_stamp_cpu.STALE_SHAPES[coalesced]
        for k in range(100):
            bufs = trace.make_bufs(lens, k)
            n, _ = eng.send_all(tx, bufs, 0)
            out, _ = eng.recv_drain(rx, 1 << 20)
            assert out.size == n == sum(lens) and np.array_equal(out, np.concatenate(bufs))
            if k >= 32:
                assert test_stamp_cpu.stale_frame_at_head(rx.ring_image(), rx.state()["head"], cap) == "stamped", k
                assert pkg.lib().b200_poller_scan(handles, 1, ev) == 0 and ev[0] == 0, k
                assert not rx.has_message() and rx.readable() == 0 and rx.recv(1 << 16).size == 0, k
    finally:
        eng.destroy(tx)
        eng.destroy(rx)


def test_reference_format_payloads_are_not_frames(gpu):
    """As in test_stamp_cpu: last lap's payload holds a reference-format frame exactly where the head lands."""
    import ctypes as C
    pkg = gpu
    cap = 4096
    eng = StampedGpuEngine(pkg)
    tx, rx = eng.pair_pair(cap)
    try:
        body = np.zeros(2024, np.uint8)
        body[0:8] = np.frombuffer(np.uint64(8).tobytes(), np.uint8)
        body[16:24] = 0xFF
        for _ in range(2):
            assert eng.send(tx, [body], 0) == 2024 and eng.recv(rx, 1 << 20).size == 2024
        assert eng.send(tx, [np.full(8, 3, np.uint8)], 0) == 8
        assert eng.recv(rx, 1 << 20).tolist() == [3] * 8
        head = rx.state()["head"]
        assert head == 8 and test_stamp_cpu.stale_frame_at_head(rx.ring_image(), head, cap) == "reference"
        handles = (C.c_void_p * 1)(rx.h)
        ev = (C.c_uint32 * 1)()
        assert pkg.lib().b200_poller_scan(handles, 1, ev) == 0 and ev[0] == 0
        assert not rx.has_message() and rx.readable() == 0 and rx.recv(100).size == 0
    finally:
        eng.destroy(tx)
        eng.destroy(rx)


def test_stamped_and_default_pairs_in_one_batch(gpu, so, oracle):
    """A stamped pair and a reference-format pair in the same batch launches: each matches its own model."""
    pkg = gpu
    L = pkg.lib()
    cap = 16384
    lens = [9, 3000, 9, 17, 9, 2000, 9, 5000, 9, 700] * 3
    bufs = trace.make_bufs(lens, 31)
    flat = np.concatenate(bufs)
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", cap)
    pkg.config_set("GRPC_RDMA_MAX_SGE", 30)
    pkg.config_set("B200_RING_STAMPED", 1)
    try:
        stx, srx = pkg.connected_pair("smix-tx", "smix-rx")
    finally:
        pkg.config_set("B200_RING_STAMPED", 0)
    dtx, drx = pkg.connected_pair("dmix-tx", "dmix-rx")
    assert stx.stamped() and not dtx.stamped()
    src = L.b200_mem_alloc_device(flat.size)
    assert L.b200_memcpy(src, flat.ctypes.data, flat.size, 0, None) == 0 and L.b200_stream_sync(None) == 0
    dst = [L.b200_mem_alloc_device(1 << 16) for _ in range(2)]
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    arr = pkg.make_slices([(src + int(o), n) for o, n in zip(offs, lens)])
    models = [(so, so.pair_pair(cap)), (oracle, oracle.pair_pair(cap))]
    for rnd in range(8):
        bs = pkg.Batch("send", [(p, arr, len(lens), 0) for p in (stx, dtx)], pkg.UNTIL_BLOCKED)
        bs.launch()
        got = list(zip(bs.results(), bs.calls()))
        bs.destroy()
        assert got == [tuple(eng.send_all(mtx, bufs, 0)) for eng, (mtx, _) in models], rnd
        br = pkg.Batch("recv", [(srx, dst[0], 1 << 16), (drx, dst[1], 1 << 16)], pkg.UNTIL_BLOCKED)
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
        assert rgot == rwant, rnd
        for (eng, (mtx, mrx)), (tx, rx) in zip(models, [(stx, srx), (dtx, drx)]):
            assert tx.state()["remote_tail"] == eng.state(mtx)["remote_tail"]
            assert rx.state()["head"] == eng.state(mrx)["head"]
            assert (rx.has_message(), rx.readable()) == (eng.has_message(mrx), eng.readable(mrx))
        gi, wi = srx.ring_image(), so.ring_image(models[0][1][1])
        pads = so.pads(models[0][1][1])
        gi[pads] = 0
        wi[pads] = 0
        assert np.array_equal(gi, wi), rnd
        assert np.array_equal(trace.mask_pads(drx.ring_image(), drx.state(), cap),
                              trace.mask_pads(oracle.ring_image(models[1][1][1]), oracle.state(models[1][1][1]), cap))
    assert not drx.ring_image().any() and srx.ring_image().any()
    for eng, (mtx, mrx) in models:
        eng.destroy(mtx), eng.destroy(mrx)
    for p in (stx, srx, dtx, drx):
        p.disconnect(); p.putback()
    L.b200_mem_free_device(src)
    for d in dst:
        L.b200_mem_free_device(d)


# ---- the service: owner warps (small Send / Recv, eager push, owed Retire) and the pool

@pytest.fixture
def svc(gpu):
    L = gpu.lib()
    assert L.b200_service_start(4) == 0, gpu.last_error()
    yield gpu
    L.b200_service_stop()


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("coalesced", [False, True])
def test_traces_through_the_service(svc, so, soc, seed, coalesced):
    """Small ops run in the owner warps (stamped headers, write-through counters, eager push, owed Retire without
    the clear), large ones in the pool (send_body / recv_body); every op matches the stamped model."""
    rng = np.random.default_rng(9700 + seed)
    cap = [1024, 4096, 65536, 1 << 20][seed]
    L = svc.lib()
    model = soc if coalesced else so
    hits = L.b200_service_eager_hits()
    for small in (True, False):
        ops = _random_ops(rng, cap, 60)
        if small:
            ops = [(o[0], [min(x, 1500) for x in o[1][:5]], o[2], min(o[3], min(o[1][0], 1500) - 1))
                   if o[0] in ("send", "send_all") else o for o in ops]
            ops = [("send",) + o[1:] if o[0] == "send_all" else o for o in ops]
            ops = [("recv", o[1]) if o[0] == "recv_drain" else o for o in ops]
        _replay(StampedGpuEngine(svc, "pinned", 3, coalesced), model, cap, ops, images=cap <= 65536)
    ops = []
    for k in range(40):  # unary-shaped: 5-byte prefix + message, received right after (eager push, then Retire)
        ops += [("send", [9, 5, 100 + 37 * k], 40 + k, 0), ("recv", 1 << 16)]
    _replay(StampedGpuEngine(svc, "pinned", 3, coalesced), model, cap, ops, images=cap <= 65536)
    assert L.b200_service_eager_hits() > hits  # the owners pushed stamped frames to the receiver's host slot


# ---- endpoint (host slices -> stamped frames -> host slices), under the service and without it

@pytest.fixture(scope="module")
def drv(gpu):
    import endpoint_lib
    D, _ = endpoint_lib.load(gpu, need_oracle=False)
    return D


def _endpoint(gpu, ring):
    gpu.config_set("B200_RING_BUFFER_SIZE_BYTES", ring)
    gpu.config_set("GRPC_RDMA_MAX_SGE", 30)
    gpu.config_set("B200_RING_STAMPED", 1)


@pytest.mark.parametrize("service", [False, True])
def test_endpoint_conformance_and_echo(gpu, drv, service):
    import ctypes as C
    L = gpu.lib()
    if service:
        assert L.b200_service_start(8) == 0, gpu.last_error()
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
        launches = L.b200_launch_count()
        nbytes = C.c_uint64(0)
        assert drv.drv_echo(None, 24, 4 * 1024 * 1024 - 1024, 777, 0, 1, 1, C.byref(nbytes)) == 0
        assert nbytes.value > 0
        _endpoint(gpu, 1 << 20)
        assert drv.drv_echo(None, 24, 2_000_000, 4242, 200, 0, 1, None) == 0  # busy-poll only
        if service:
            assert L.b200_launch_count() == launches, "the service moves every byte: no kernel launches"
    finally:
        gpu.config_set("B200_RING_STAMPED", 0)
        if service:
            L.b200_service_stop()


# ---- NVLink wire (two GPUs)

def test_stream_across_two_gpus_stamped():
    import json
    import os
    import subprocess
    import sys
    import tempfile
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs on one machine")
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, B200_RING_STAMPED="1")
    with tempfile.TemporaryDirectory() as d:
        procs = [subprocess.Popen([sys.executable, os.path.join(here, "ipc_wire_worker.py"), role, str(dev), d,
                                   "4096", str(1 << 20), "12", "4"],
                                  stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
                 for role, dev in (("server", 1), ("client", 0))]
        outs = [p.communicate(timeout=500)[0] for p in procs]
        assert all(p.returncode == 0 for p in procs), "\n".join(outs)
        srv = json.load(open(os.path.join(d, "server.json")))
    # every message intact over > 3 laps; the ring keeps its retired frames (the connection ran stamped)
    assert srv["ok"] and srv["half_closed"] and not srv["ring_empty"]


def test_concurrent_send_and_recv_over_many_laps(gpu):
    """Send and Recv of one connection on two streams (B200_BATCH_CONCURRENT) over many laps of periodic frames:
    a receiver that neither cleared nor checked stamps would take last lap's frames."""
    import torch
    pkg = gpu
    L = pkg.lib()
    cap = 1 << 17  # retired-but-uncredited (< C/2) + one message in flight + the next one always fit
    eng = StampedGpuEngine(pkg)
    tx, rx = eng.pair_pair(cap)
    lens = [9, 2000] * 8
    total = sum(lens)
    rounds = 200  # > 20 laps
    msg = np.concatenate(trace.make_bufs(lens, 77))
    src = L.b200_mem_alloc_device(total)
    dst = L.b200_mem_alloc_device(total * rounds)
    assert L.b200_memcpy(src, msg.ctypes.data, total, 0, None) == 0 and L.b200_stream_sync(None) == 0
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    arr = pkg.make_slices([(src + int(o), n) for o, n in zip(offs, lens)])
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    flags = pkg.UNTIL_BLOCKED | 0x8  # B200_BATCH_CONCURRENT
    got = 0
    for r in range(rounds):
        bs = pkg.Batch("send", [(tx, arr, len(lens), 0)], flags)
        br = pkg.Batch("recv", [(rx, dst + got, total * rounds - got)], flags)
        bs.launch(s1.cuda_stream)
        br.launch(s2.cuda_stream)
        assert bs.results(s1.cuda_stream) == [total], r
        got += br.results(s2.cuda_stream)[0]
        bs.destroy()
        br.destroy()
    br = pkg.Batch("recv", [(rx, dst + got, total * rounds - got)], pkg.UNTIL_BLOCKED)
    br.launch()
    got += br.results()[0]
    br.destroy()
    assert got == total * rounds
    out = np.zeros(got, np.uint8)
    assert L.b200_memcpy(out.ctypes.data, dst, got, 1, None) == 0 and L.b200_stream_sync(None) == 0
    assert np.array_equal(out, np.tile(msg, rounds))
    assert not rx.has_message() and rx.recv(100).size == 0
    L.b200_mem_free_device(src)
    L.b200_mem_free_device(dst)
    eng.destroy(tx)
    eng.destroy(rx)
