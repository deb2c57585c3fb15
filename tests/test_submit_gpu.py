"""GPU: b200_pairs_submit with the service running -- the endpoint's data path (b200_endpoint.cc posts every ready
rdma_flush and rdma_do_read loop of a pass as one call) -- against the CPU models, pass by pass.

The bar is test_gpu_parity.py's, applied after every pass: each op's accepted / delivered count and the bytes
delivered, both pairs' cursors, the readiness answers and the receiver's ring image with pads masked.  `calls` is
not compared: a pass does not return it.  Slices come from plain numpy memory (staged in the pass's one pinned
bounce buffer), b200_mem_alloc_host, registered anonymous memory and device memory, mixed inside a pass;
destinations are pinned host or device memory.

Determinism: a pass never holds the Send and the Recv of one direction of a connection (those two run side by side
in the pool and either may win); the Send and the Recv of one pair may share a pass.  Where the endpoint does hold
both (its steady state) the tests check invariants instead of per-op values."""
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import coalesce_lib
import stamp_lib
import test_coalesce_gpu
import trace
from gpu_engine import GpuEngine
from submit_lib import SLICE_AREA, Arena, SubmitEngine, submit

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MODES = ("ref", "coal", "stamp")  # reference framing, B200_SEND_COALESCE=1, B200_RING_STAMPED=1
UB = 1  # B200_BATCH_UNTIL_BLOCKED
SRC_KINDS = Arena.KINDS + ("mixed",)
DST_KINDS = ("host", "registered", "device")


def _models(oracle):
    return {"ref": oracle, "coal": coalesce_lib.CoalescedOracle(), "stamp": stamp_lib.StampedOracle()}


@pytest.fixture(scope="module")
def models(oracle):
    return _models(oracle)


class Service:
    """b200_service_start(workers) with `owners` owner queues (None: the defaults; B200_SERVICE_OWNERS is read at
    every start) and an Arena allocated before the start and released after the stop."""

    def __init__(self, pkg, owners=None, workers=4, arena=64 << 20):
        self.pkg, self.L = pkg, pkg.lib()
        self.owners, self.workers, self.arena_bytes = owners, workers, arena

    def __enter__(self):
        self.arena = Arena(self.pkg, self.arena_bytes)
        old = os.environ.pop("B200_SERVICE_OWNERS", None)
        if self.owners is not None:
            os.environ["B200_SERVICE_OWNERS"] = str(self.owners)
        try:
            rc = self.L.b200_service_start(self.workers)
        finally:
            os.environ.pop("B200_SERVICE_OWNERS", None)
            if old is not None:
                os.environ["B200_SERVICE_OWNERS"] = old
        if rc != 0:
            self.arena.free()
            raise RuntimeError("b200_service_start: " + self.pkg.last_error())
        assert self.L.b200_service_running() == self.workers or (self.workers <= 0 and self.L.b200_service_running())
        return self

    def __exit__(self, *exc):
        self.L.b200_service_stop()
        assert self.L.b200_service_running() == 0
        self.arena.free()


@pytest.fixture
def svc(gpu, request):
    with Service(gpu, **getattr(request, "param", {})) as s:
        yield s


def _config(pkg, cap, mode):
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", cap)
    pkg.config_set("GRPC_RDMA_MAX_SGE", 30)
    pkg.config_set("B200_SEND_COALESCE", int(mode == "coal"))
    pkg.config_set("B200_RING_STAMPED", int(mode == "stamp"))


class Conn:
    """A bidirectional loopback connection (ends a, b) in one framing mode, and its twin in that mode's model."""
    count = 0

    def __init__(self, pkg, models, mode, cap):
        Conn.count += 1
        self.name = "sub%d-%s-%d" % (Conn.count, mode, cap)
        _config(pkg, cap, mode)
        try:
            self.a, self.b = pkg.connected_pair(self.name + "a", self.name + "b")
        finally:
            _config(pkg, cap, "ref")
        assert self.a.stamped() == self.b.stamped() == (mode == "stamp")
        self.mode, self.cap, self.model = mode, cap, models[mode]
        self.ma, self.mb = self.model.pair_pair(cap)

    def ends(self, d):
        """direction d = 0: a -> b, 1: b -> a.  (gpu tx, gpu rx, model tx, model rx)"""
        return (self.a, self.b, self.ma, self.mb) if d == 0 else (self.b, self.a, self.mb, self.ma)

    def close(self):
        for p in (self.a, self.b):
            p.disconnect()
            p.putback()
        self.model.destroy(self.ma)
        self.model.destroy(self.mb)


G = GpuEngine.__new__(GpuEngine)  # only its pair queries (state, has_message, ...) are used


def _view(e, tx, rx):
    st, sr = e.state(tx), e.state(rx)
    return {"tx": {k: st[k] for k in ("remote_tail", "partial_write", "credit_remote_head")},
            "rx": {k: sr[k] for k in ("head", "moving_head", "remain", "internal_read_size")},
            "ready": (int(e.has_message(rx)), int(e.readable(rx)), int(e.has_pending_writes(tx)), int(e.writable(tx)))}


def _views(c, model):
    e = c.model if model else G
    return [_view(e, *c.ends(d)[2 * model:2 * model + 2]) for d in (0, 1)]


def _check_image(c, d, label):
    _, rx, _, mrx = c.ends(d)
    gi, wi = rx.ring_image(), c.model.ring_image(mrx)
    if c.mode == "stamp":  # retired frames stay in a stamped ring: mask the pads of every frame image
        pads = c.model.pads(mrx)
        gi[pads] = 0
        wi[pads] = 0
    else:
        gi = trace.mask_pads(gi, rx.state(), c.cap)
        wi = trace.mask_pads(wi, c.model.state(mrx), c.cap)
    bad = np.flatnonzero(gi != wi)
    assert bad.size == 0, "%s: %s direction %d: ring differs at %s" % (label, c.name, d, bad[:16])


def _check_conn(c, label, images=True, dirs=(0, 1)):
    g, w = _views(c, False), _views(c, True)
    for d in dirs:
        assert g[d] == w[d], "%s: %s direction %d\n got  %s\n want %s" % (label, c.name, d, g[d], w[d])
        if images:
            _check_image(c, d, label)


def _advance(lens, idx, bidx, n):
    """the endpoint's outgoing slice index / byte_idx once `n` more bytes were accepted (rdma_bp_posix.cc:480-493)"""
    while n > 0:
        left = lens[idx] - bidx
        if n >= left:
            n, idx, bidx = n - left, idx + 1, 0
        else:
            bidx, n = bidx + n, 0
    return idx, bidx


# ---- passes of many ops: plan (random), run on the GPU, replay on the models

def _lens(rng, cap):
    n = int(rng.integers(1, 40))
    style = int(rng.integers(0, 4))
    if style == 0:
        lens = rng.integers(1, 64, n)
    elif style == 1:
        lens = [9 if i % 2 == 0 else rng.integers(1, min(16385, cap)) for i in range(n)]
    elif style == 2:
        lens = rng.integers(1, 2 * cap, max(1, n // 8))
    else:
        lens = rng.integers(0, 20, n)  # zero-length slices included
    lens = [int(x) for x in lens]
    return lens, int(rng.integers(0, lens[0])) if lens[0] else 0


def _plan(rng, conns, grow=0, dst_kinds=DST_KINDS):
    """One pass: per connection and direction nothing, a Send (rdma_flush loop) or a Recv (rdma_do_read loop) --
    never both of one direction.  grow > 0: every direction sends [9, 16384] * grow from plain memory."""
    plan = []
    for c in conns:
        for d in (0, 1):
            k = 1 if grow else int(rng.integers(0, 3))
            if k == 1:
                lens, bidx = ([9, 16384] * grow, 3) if grow else _lens(rng, c.cap)
                kind = "plain" if grow else SRC_KINDS[int(rng.integers(0, len(SRC_KINDS)))]
                kinds = [Arena.KINDS[int(x)] for x in rng.integers(0, 4, len(lens))] if kind == "mixed" else \
                    [kind] * len(lens)
                plan.append(("send", c, d, trace.make_bufs(lens, int(rng.integers(0, 1 << 16))), bidx, kinds))
            elif k == 2:
                plan.append(("recv", c, d, int(rng.integers(1, 2 * c.cap)), dst_kinds[int(rng.integers(0, len(dst_kinds)))]))
    return [plan[i] for i in rng.permutation(len(plan))]


def _unregistered(plan):
    """bytes of the pass that b200_pairs_submit stages in its bounce buffer (counted as it counts them)"""
    return sum((b.size + 15) // 16 * 16 for op in plan if op[0] == "send"
               for b, k in list(zip(op[3], op[5]))[:SLICE_AREA] if k == "plain")


def _desc(op):
    return "%s %s dir %d" % (op[0], op[1].name, op[2])


def _run_pass(pkg, conns, plan, arena):
    """post `plan` as one b200_pairs_submit pass: rc, error text, per op (count, SHA-1 of the bytes delivered), then
    every connection's view of both directions"""
    arena.reset()
    sends, recvs, where = [], [], []
    for i, op in enumerate(plan):
        tx, rx = op[1].ends(op[2])[:2]
        if op[0] == "send":
            sends.append((tx.h, arena.place(op[3], op[5], i), len(op[3]), op[4]))
            where.append(len(sends) - 1)
        else:
            dst = arena.alloc(op[4], op[3], i % 16)
            recvs.append((rx.h, dst, op[3]))
            where.append(len(recvs) - 1)
    rc, acc, dlv = submit(pkg, sends, recvs, UB)
    err = pkg.last_error() if rc else ""
    res = []
    for op, j in zip(plan, where):
        if op[0] == "send":
            res.append((int(acc[j]), None))
        else:
            res.append((int(dlv[j]), trace.sha(arena.get(op[4], recvs[j][1], dlv[j]))))
    return {"rc": rc, "err": err, "res": res, "views": [_views(c, False) for c in conns]}


def _model_pass(conns, plan):
    res = []
    for op in plan:
        c = op[1]
        _, _, mtx, mrx = c.ends(op[2])
        if op[0] == "send":
            res.append((int(c.model.send_all(mtx, op[3], op[4])[0]), None))
        else:
            out, _ = c.model.recv_drain(mrx, op[3])
            res.append((int(out.size), trace.sha(out)))
    return {"rc": 0, "err": "", "res": res, "views": [_views(c, True) for c in conns]}


def _compare_pass(conns, plan, got, want, label):
    assert got["rc"] == 0, "%s: rc %d (%s)" % (label, got["rc"], got["err"])
    for op, g, w in zip(plan, got["res"], want["res"]):
        assert g == w, "%s: %s\n got  %s\n want %s" % (label, _desc(op), g, w)
    for c, g, w in zip(conns, got["views"], want["views"]):
        for d in (0, 1):
            assert g[d] == w[d], "%s: %s direction %d\n got  %s\n want %s" % (label, c.name, d, g[d], w[d])


def _check_pass(pkg, conns, plan, arena, label, images=True):
    got = _run_pass(pkg, conns, plan, arena)
    _compare_pass(conns, plan, got, _model_pass(conns, plan), label)
    if images:
        for c in conns:
            for d in (0, 1):
                _check_image(c, d, label)


# ---- 1. single-connection replays: every op one pass (submit_lib.SubmitEngine)

GOLDEN = json.load(open(os.path.join(HERE, "golden", "traces.json")))


def _golden(eng, t, max_sge, label, ring_images=True):
    """a golden trace against its records, without `calls` (a pass does not return it)"""
    recs = trace.run_trace(eng, t["cap"], [tuple(o) for o in t["ops"]], max_sge, ring_images=ring_images)
    got, want = [[{k: v for k, v in r.items() if k != "calls"} for r in x] for x in (recs, t["records"])]
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, "%s: op %d (%s)\n got  %s\n want %s" % (label, i, w["op"], g, w)


@pytest.mark.parametrize("name", sorted(GOLDEN["traces"]))
def test_golden_traces_through_submit(svc, name):
    """Single calls as B200_BATCH_ONE_CALL ops, rdma_flush / rdma_do_read loops as B200_BATCH_UNTIL_BLOCKED ops,
    slices from every memory kind; everything runs in the resident kernels, nothing is launched."""
    L = svc.L
    launches = L.b200_launch_count()
    _golden(SubmitEngine(svc.pkg, svc.arena), GOLDEN["traces"][name], GOLDEN["max_sge"], "golden %s" % name)
    assert L.b200_launch_count() == launches


def test_golden_full_size_through_submit(svc):
    """The BASELINE-size fixture (16 MiB ring, 4 MiB chttp2-shaped messages, more than two laps) as submit passes."""
    with open(os.path.join(HERE, "golden", "traces_full.json")) as f:
        G = json.load(f)
    for name, t in G["traces"].items():
        _golden(SubmitEngine(svc.pkg, svc.arena), t, G["max_sge"], "golden full %s" % name, ring_images=False)


def _apply(e, tx, rx, op):
    if op[0] in ("send", "send_all"):
        bufs = trace.make_bufs(op[1], op[2])
        return int(e.send(tx, bufs, op[3]) if op[0] == "send" else e.send_all(tx, bufs, op[3])[0])
    out = e.recv(rx, op[1]) if op[0] == "recv" else e.recv_drain(rx, op[1])[0]
    return int(out.size), trace.sha(out)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("seed", range(3))
def test_random_traces_through_submit(svc, models, mode, seed):
    """test_coalesce_gpu's trace shapes (zero-length slices, > 1024 slices, slices larger than the ring), one op per
    pass, against the model of the connection's framing; an rdma_flush loop over more slices than one op takes is
    re-submitted from the returned position, as the endpoint does."""
    rng = np.random.default_rng(9900 + seed)
    cap = [1024, 4096, 65536][seed]
    ops = test_coalesce_gpu._random_ops(rng, cap, 60)
    pkg, L = svc.pkg, svc.L
    c = Conn(pkg, models, mode, cap)
    eng = SubmitEngine(pkg, svc.arena)
    launches = L.b200_launch_count()
    try:
        for i, op in enumerate(ops):
            label = "%s seed %d cap %d op %d %s" % (mode, seed, cap, i, op[0])
            assert _apply(eng, c.a, c.b, op) == _apply(c.model, c.ma, c.mb, op), label
            _check_conn(c, label, dirs=(0,))
    finally:
        c.close()
    assert L.b200_launch_count() == launches  # every op ran in the resident kernels


# ---- 2. many connections, deterministic passes

# pass -> [9, 16384] pairs per Send, every Send from plain memory: each of these passes stages more than every pass
# before it (the last one more than any single call of a 16 MiB ring stages), so the shared bounce is reallocated
GROW = {2: 2, 5: 10, 8: 25}


@pytest.mark.parametrize("svc", [dict(owners=1, workers=2), dict(owners=2, workers=16), dict(owners=None, workers=0)],
                         indirect=True, ids=["owners1-workers2", "owners2-workers16", "defaults"])
def test_many_connections_deterministic_passes(svc, models):
    """48 connections (reference, coalesced and stamped in the same pass), every memory kind in every pass.  With
    one owner a pass posts far more than one queue's 16 entries and far more than its 8 pool boxes."""
    pkg = svc.pkg
    rng = np.random.default_rng(4242)
    conns = [Conn(pkg, models, MODES[i % 3], (1024, 4096, 8192)[(i // 3) % 3]) for i in range(48)]
    try:
        staged = 0
        for p in range(10):
            plan = _plan(rng, conns, GROW.get(p, 0))
            if p in GROW:
                assert _unregistered(plan) > staged
            staged = max(staged, _unregistered(plan))
            _check_pass(pkg, conns, plan, svc.arena, "pass %d" % p)
    finally:
        for c in conns:
            c.close()


# ---- 3. both ends of one direction in one pass (the endpoint's steady state): invariants

@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cap", [64 << 10, 16 << 20], ids=["64k", "16m"])
def test_both_ends_of_one_direction_in_one_pass(svc, models, mode, cap):
    """A 4 MiB chttp2-shaped message in non-adjacent pinned slices; every pass is {A sends the rest, B receives}."""
    pkg, a = svc.pkg, svc.arena
    lens = pkg.chttp2_slice_lens(4 << 20)
    total = sum(lens)
    bufs = trace.make_bufs(lens, 61)
    msg = np.concatenate(bufs)
    dkind = DST_KINDS[MODES.index(mode)]
    c = Conn(pkg, models, mode, cap)
    try:
        a.reset()
        sl = a.place(bufs, ["host"] * len(lens))
        ptrs = [(sl[i].ptr, sl[i].len) for i in range(len(lens))]
        dst = a.alloc(dkind, total)
        idx = bidx = sent = got = passes = 0
        while got < total:
            passes += 1
            assert passes < 20000, "no progress: sent %d, delivered %d" % (sent, got)
            sends = []
            if idx < len(lens):
                rest = pkg.make_slices(ptrs[idx:])
                sends = [(c.a.h, rest, len(lens) - idx, bidx)]
            rc, acc, dlv = submit(pkg, sends, [(c.b.h, dst + got, total - got)], UB)
            assert rc == 0, pkg.last_error()
            n = dlv[0]
            if not sends:  # everything sent landed in an earlier pass: one rdma_do_read loop takes all of it
                assert n == sent - got, (passes, n, sent, got)
            if sends:
                sent += acc[0]
                idx, bidx = _advance(lens, idx, bidx, acc[0])
            assert got + n <= sent
            assert np.array_equal(a.get(dkind, dst + got, n), msg[got:got + n]), "pass %d" % passes
            got += n
        assert sent == got == total and idx == len(lens)
        tx, rx = c.a.state(), c.b.state()
        assert rx["head"] == tx["remote_tail"] and tx["partial_write"] == 0 and not c.b.has_message()
        if mode != "stamp":
            assert not c.b.ring_image().any(), "the reference format clears what it reads"
    finally:
        c.close()


# ---- 4. eager frames and the owed Retire

@pytest.mark.parametrize("variant", ["rides_on_a_send", "drain_retire", "peer_sends_first"])
@pytest.mark.parametrize("mode", MODES)
def test_eager_frames_and_the_owed_retire(svc, models, mode, variant):
    """A unary-shaped message with single calls; B's b200_pair_recv takes it from its eager host slot, which leaves
    a Retire owed.  Then a submit pass: a Send on B that carries the Retire, or B's Recv alone (drain_retire first),
    or A's Send of a second frame (B's Retire is drained first).  Nothing may look at B in between: every query
    drains the owed Retire."""
    pkg, L, a = svc.pkg, svc.L, svc.arena
    c = Conn(pkg, models, mode, 65536)
    m = c.model
    hits = L.b200_service_eager_hits()
    try:
        for k in range(12):
            label = "%s %s round %d" % (mode, variant, k)
            bufs = trace.make_bufs([9, 5, 100 + 37 * k], 40 + k)
            assert c.a.send(bufs) == m.send(c.ma, bufs), label
            out = c.b.recv(1 << 16)
            assert trace.sha(out) == trace.sha(m.recv(c.mb, 1 << 16)), label
            a.reset()
            if variant != "drain_retire":
                tx, mtx = (c.b, c.mb) if variant == "rides_on_a_send" else (c.a, c.ma)
                more = trace.make_bufs([9, 5, 50 + 11 * k], 90 + k)
                sl = a.place(more, [Arena.KINDS[(k + i) % 4] for i in range(3)], k)
                rc, acc, _ = submit(pkg, [(tx.h, sl, 3, 0)], (), UB)
                assert rc == 0 and acc[0] == m.send_all(mtx, more, 0)[0], label
            dst = a.alloc(DST_KINDS[k % 3], 1 << 16, k)
            rc, _, dlv = submit(pkg, (), [(c.b.h, dst, 1 << 16)], UB)
            want, _ = m.recv_drain(c.mb, 1 << 16)
            assert rc == 0 and trace.sha(a.get(DST_KINDS[k % 3], dst, dlv[0])) == trace.sha(want), label
            if variant == "rides_on_a_send":  # A takes B's reply
                dst = a.alloc("device", 1 << 16)
                rc, _, dlv = submit(pkg, (), [(c.a.h, dst, 1 << 16)], UB)
                want, _ = m.recv_drain(c.ma, 1 << 16)
                assert rc == 0 and trace.sha(a.get("device", dst, dlv[0])) == trace.sha(want), label
            _check_conn(c, label)
    finally:
        c.close()
    assert L.b200_service_eager_hits() > hits, "no Recv was an eager hit: the owed Retire was never exercised"


# ---- 5. more than kSvcSliceArea - 1 slices in one until-blocked op

@pytest.mark.parametrize("kind", ["plain", "device"])
@pytest.mark.parametrize("mode", ["ref", "coal"])
def test_more_slices_than_one_op_takes(svc, models, mode, kind):
    """An until-blocked op dereferences the first 1023 slices; the rest is folded into a pseudo-slice that only
    counts towards the call's total (pair.cc:661-664).  So the op accepts what the model's rdma_flush loop over
    those 1023 slices accepts, and reports the write as partial; the endpoint re-submits from the returned
    position and the stream completes intact."""
    pkg, a = svc.pkg, svc.arena
    rng = np.random.default_rng(5100 + MODES.index(mode))
    lens = [int(x) for x in rng.integers(1, 4, int(rng.integers(1200, 1501)))]
    bidx = int(rng.integers(0, lens[0]))
    bufs = trace.make_bufs(lens, 77)
    c = Conn(pkg, models, mode, 65536)
    m = c.model
    try:
        a.reset()
        sl = a.place(bufs, [kind] * len(lens))
        rc, acc, _ = submit(pkg, [(c.a.h, sl, len(lens), bidx)], (), UB)
        assert rc == 0, pkg.last_error()
        window = sum(lens[:SLICE_AREA - 1]) - bidx
        assert acc[0] == m.send_all(c.ma, bufs[:SLICE_AREA - 1], bidx)[0] == window
        g, w = _views(c, False)[0], _views(c, True)[0]
        assert g["tx"]["partial_write"] == 1 and g["ready"][2] == 1, g  # the folded rest is still to be written
        w["tx"]["partial_write"] = 1
        w["ready"] = w["ready"][:2] + (1,) + w["ready"][3:]
        assert g == w
        _check_image(c, 0, "first op")
        idx, b2 = _advance(lens, 0, bidx, acc[0])
        assert (idx, b2) == (SLICE_AREA - 1, 0)
        rest = pkg.make_slices([(sl[i].ptr, sl[i].len) for i in range(idx, len(lens))])
        rc, acc2, _ = submit(pkg, [(c.a.h, rest, len(lens) - idx, 0)], (), UB)
        assert rc == 0 and acc2[0] == m.send_all(c.ma, bufs[idx:], 0)[0] == sum(lens) - bidx - acc[0]
        _check_conn(c, "re-submitted", dirs=(0,))
        dst = a.alloc("host", 1 << 16)
        rc, _, dlv = submit(pkg, (), [(c.b.h, dst, 1 << 16)], UB)
        want, _ = m.recv_drain(c.mb, 1 << 16)
        got = a.get("host", dst, dlv[0])
        assert rc == 0 and np.array_equal(got, want)
        assert np.array_equal(got, np.concatenate(bufs)[bidx:]), "the stream is intact"
        _check_conn(c, "drained", dirs=(0,))
    finally:
        c.close()


# ---- 6. errors and the lifecycle

def test_errors_and_the_lifecycle(svc, models):
    pkg, a = svc.pkg, svc.arena
    conns = [Conn(pkg, models, MODES[i], 4096) for i in range(3)]
    try:
        a.reset()
        for i, c in enumerate(conns):
            bufs = trace.make_bufs([100 + i, 9], 7 + i)
            rc, acc, _ = submit(pkg, [(c.a.h, a.place(bufs, ["host", "plain"]), 2, 0)], (), UB)
            assert rc == 0 and acc[0] == c.model.send_all(c.ma, bufs, 0)[0]
        # one Recv of the pass has an unregistered destination: that op fails, the others run
        before = (_views(conns[1], False), conns[1].b.ring_image())
        plain = np.zeros(4096, np.uint8)
        dsts = [a.alloc("device", 4096), plain.ctypes.data, a.alloc("host", 4096)]
        rc, _, dlv = submit(pkg, (), [(c.b.h, d, 4096) for c, d in zip(conns, dsts)], UB)
        assert rc == -1 and "GPU-addressable" in pkg.last_error()
        assert dlv[1] == 0 and not plain.any()
        for i in (0, 2):
            want, _ = conns[i].model.recv_drain(conns[i].mb, 4096)
            assert np.array_equal(a.get(("device", None, "host")[i], dsts[i], dlv[i]), want)
        assert _views(conns[1], False) == before[0] and np.array_equal(conns[1].b.ring_image(), before[1])
        for c in conns:
            _check_conn(c, "after the failed op")
        # ops that move nothing: a pair that is not connected, no slices, no room, no pair
        lone = pkg.Pair("sub-lone")
        sl = a.place(trace.make_bufs([50], 3), ["host"])
        dst = a.alloc("host", 100)
        c = conns[1]
        rc, acc, dlv = submit(pkg, [(lone.h, sl, 1, 0), (c.b.h, sl, 0, 0), (None, sl, 1, 0)],
                              [(lone.h, dst, 100), (c.b.h, dst, 0), (None, dst, 100)], UB)
        assert rc == 0 and acc == [0, 0, 0] and dlv == [0, 0, 0]
        lone.disconnect()  # back to the pool Disconnected: the next Take re-initialises it
        lone.putback()
        _check_conn(c, "ops that move nothing")
        # after the peer's Disconnect the ring still drains
        bufs = trace.make_bufs([300, 9, 1000], 11)
        rc, acc, _ = submit(pkg, [(c.a.h, a.place(bufs, ["device"] * 3), 3, 0)], (), UB)
        assert rc == 0 and acc[0] == c.model.send_all(c.ma, bufs, 0)[0]
        c.a.disconnect()
        assert c.b.status() == 3  # HalfClosed
        dst = a.alloc("registered", 8192)
        rc, _, dlv = submit(pkg, (), [(c.b.h, dst, 8192)], UB)
        want, _ = c.model.recv_drain(c.mb, 8192)
        got = a.get("registered", dst, dlv[0])
        assert rc == 0 and np.array_equal(got, want) and np.array_equal(got[-1309:], np.concatenate(bufs))
        rc, _, dlv = submit(pkg, (), [(c.b.h, dst, 8192)], UB)
        assert rc == 0 and dlv == [0]
    finally:
        for c in conns:
            c.close()


# ---- 7. threads

@pytest.mark.parametrize("svc", [dict(owners=1, workers=4)], indirect=True, ids=["owners1-workers4"])
def test_threads_share_one_owner_queue(svc, models):
    """Four threads drive disjoint connection sets through one owner queue (per-queue posting sections, per-thread
    bounce buffers; a thread never blocks on a full queue while it holds answers of its own).  Each thread records
    its passes; the records are compared with the models afterwards.  A deadlock would surface as the service's
    30 s command timeout (rc -1)."""
    pkg = svc.pkg
    nthreads, per, npasses = 4, 6, 8
    rng = np.random.default_rng(777)
    conns = [[Conn(pkg, models, MODES[(t + i) % 3], (1024, 4096, 8192)[i % 3]) for i in range(per)]
             for t in range(nthreads)]
    try:
        plans = [[_plan(rng, conns[t], 3 if p == 4 else 0) for p in range(npasses)] for t in range(nthreads)]
        arenas = [svc.arena.part(t, nthreads) for t in range(nthreads)]
        recs = [[] for _ in range(nthreads)]
        errors = []

        def drive(t):
            try:
                for plan in plans[t]:
                    recs[t].append(_run_pass(pkg, conns[t], plan, arenas[t]))
            except BaseException as ex:  # reported by the main thread
                errors.append((t, repr(ex)))

        threads = [threading.Thread(target=drive, args=(t,)) for t in range(nthreads)]
        for th in threads:
            th.start()
        for th in threads:
            th.join(600)
        assert not any(th.is_alive() for th in threads), "a thread did not finish"
        assert not errors, errors
        for t in range(nthreads):
            assert len(recs[t]) == npasses
            for p, plan in enumerate(plans[t]):
                _compare_pass(conns[t], plan, recs[t][p], _model_pass(conns[t], plan), "thread %d pass %d" % (t, p))
            for c in conns[t]:
                for d in (0, 1):
                    _check_image(c, d, "thread %d at the end" % t)
    finally:
        for cs in conns:
            for c in cs:
                c.close()


# ---- 8. the benchmark's shape

@pytest.mark.parametrize("svc", [dict(workers=0, arena={"host": 540 << 20})], indirect=True, ids=["defaults"])
def test_benchmark_shape(svc, oracle):
    """bench.py's endpoint leg: 64 connections with 16 MiB rings, one 4 MiB chttp2-shaped message each in
    non-adjacent pinned slices; a pass of all Sends, then a pass of all Recvs, five rounds (more than a lap).  The
    connections carry different bytes in the same shapes, so one model connection gives every op's count and the
    cursors; the delivered bytes are checked against each connection's own stream."""
    pkg, a = svc.pkg, svc.arena
    nconn, cap = 64, 16 << 20
    lens = pkg.chttp2_slice_lens(4 << 20)
    total = sum(lens)
    _config(pkg, cap, "ref")
    pairs = [pkg.connected_pair("bsh-a%d" % i, "bsh-b%d" % i) for i in range(nconn)]
    mtx, mrx = oracle.pair_pair(cap)
    try:
        a.reset()
        msgs, slices, dsts = [], [], []
        for i in range(nconn):
            bufs = trace.make_bufs(lens, 1000 + i)
            msgs.append(np.concatenate(bufs))
            sl = a.place(bufs, ["host"] * len(lens), i)
            slices.append([(sl[j].ptr, sl[j].len) for j in range(len(lens))])
            dsts.append(a.alloc("host", total, i))
        mbufs = trace.make_bufs(lens, 999)
        idx = bidx = pos = 0  # the message position (the same on every connection) and the stream position
        for r in range(5):
            keep = [pkg.make_slices(s[idx:]) for s in slices]
            rc, acc, _ = submit(pkg, [(p[0].h, k, len(lens) - idx, bidx) for p, k in zip(pairs, keep)], (), UB)
            want = oracle.send_all(mtx, mbufs[idx:], bidx)[0]
            assert rc == 0 and acc == [want] * nconn, (r, acc[:4], want)
            idx, bidx = _advance(lens, idx, bidx, want)
            if idx == len(lens):
                idx = 0
            rc, _, dlv = submit(pkg, (), [(p[1].h, d, total) for p, d in zip(pairs, dsts)], UB)
            out, _ = oracle.recv_drain(mrx, total)
            assert rc == 0 and dlv == [out.size] * nconn, (r, dlv[:4], out.size)
            at = (pos + np.arange(out.size)) % total
            for i in range(nconn):
                assert np.array_equal(a.get("host", dsts[i], out.size), msgs[i][at]), "round %d connection %d" % (r, i)
            pos += out.size
            w = _view(oracle, mtx, mrx)
            for i, (tx, rx) in enumerate(pairs):
                assert _view(G, tx, rx) == w, "round %d connection %d" % (r, i)
        assert pos > cap
    finally:
        oracle.destroy(mtx)
        oracle.destroy(mrx)
        for tx, rx in pairs:
            for p in (tx, rx):
                p.disconnect()
                p.putback()


# ---- 9. B200_SUBMIT_STAGE_MIN (read once per process): Recv into pinned host memory through device staging

def stage_min_child():
    """run by test_stage_min_in_a_subprocess in a process of its own"""
    import __graft_entry__ as ge
    import orlib
    pkg = ge.load_package()
    pkg.init(0)
    models = _models(orlib.Oracle())
    rng = np.random.default_rng(31337)
    with Service(pkg, workers=4) as s:
        conns = [Conn(pkg, models, MODES[i % 3], (1024, 4096, 8192)[i % 3]) for i in range(12)]
        try:
            for p in range(6):
                _check_pass(pkg, conns, _plan(rng, conns, dst_kinds=("host", "registered")), s.arena,
                            "stage-min pass %d" % p)
        finally:
            for c in conns:
                c.close()
    print("stage-min ok")


def test_stage_min_in_a_subprocess():
    code = "import sys; sys.path[:0] = [%r, %r]; import test_submit_gpu; test_submit_gpu.stage_min_child()" % (ROOT, HERE)
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, B200_SUBMIT_STAGE_MIN="1"),
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "stage-min ok" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]
