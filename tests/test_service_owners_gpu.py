"""GPU: the service owners' single calls (b200_pair_send / b200_pair_recv with the service running) against the CPU
models, with more connections than an owner's cache holds, at the owner's routing limits, from many threads and with
prepared batches launched beside the owners.

An owner warp (k_svc_owner, b200_kernels.cu) keeps state across commands and connections: a first-in first-out
cache of kConnCache = 8 connections (both pairs' lines, PairSvc and PairSeq, written through, dropped whole when the
host's generation changes), a queue of kOwnQ = 16 commands, kOwnBoxes = 8 pool mailboxes reaped lazily, the eager
slot records and the owed Retire that rides on a pair's next Send.  A stale line in that cache does not fail loudly:
a frame lands at a stale tail, or a Recv starts from a stale head.  So every op's count and delivered bytes are
compared with the connection's model, and after every round both directions' cursors, readiness answers and ring
images with pads masked (test_submit_gpu._check_conn).

Slices come from plain numpy memory, b200_mem_alloc_host, registered and device memory, destinations from the same
four kinds, mixed across connections and ops.  Nothing here synchronises the whole device while the service runs: a
batch's results are collected on its own stream, and torch's stream, event and sleep kernel are used once before the
first service start (a kernel's first launch beside the resident kernels waits for them, DESIGN.md section 7)."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

import trace
from submit_lib import Arena
from test_submit_gpu import MODES, Conn, Service, _check_conn, _models, _views

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

CACHE = 8         # kConnCache: connections one owner warp keeps
INLINE = 5        # kSvcInline: slices a small Send takes
SMALL_MAX = 8192  # kSmallMax: bytes one owner warp moves by itself
EAGER_MAX = 2048  # kEagerMax: frames pushed to the receiver's host slot
DST = ("plain", "host", "registered", "device")


@pytest.fixture(scope="module")
def models(oracle):
    return _models(oracle)


class Gate:
    """Orders a prepared batch behind the single calls without retries: the batch is launched on its own stream
    behind a sleep kernel of about 50 ms and an event is recorded behind it.  If the event has not completed once the
    single calls have returned, the owners served them before the batch ran."""
    CYCLES = 100_000_000  # about 50 ms at 1.98 GHz

    def __init__(self, torch):
        self.torch = torch
        self.st, self.free = torch.cuda.Stream(), torch.cuda.Stream()
        self.h, self.free_h = C.c_void_p(self.st.cuda_stream), C.c_void_p(self.free.cuda_stream)
        self.ev = torch.cuda.Event()
        for s in (self.st, self.free):  # every kernel and call used beside the service, once before it starts
            with torch.cuda.stream(s):
                torch.cuda._sleep(1000)
            self.ev.record(s)
            self.ev.query()
            s.synchronize()

    def launch(self, batch):
        with self.torch.cuda.stream(self.st):
            self.torch.cuda._sleep(self.CYCLES)
        batch.launch(self.h)
        self.ev.record(self.st)

    def held(self, label):
        assert not self.ev.query(), "%s: the batch finished before the single calls were answered: the gate did not " \
                                    "hold, so the order these checks assume is unknown" % label

    def results(self, batch):
        return batch.results(self.h)


@pytest.fixture(scope="module")
def gate(gpu):
    import torch
    return Gate(torch)


@pytest.fixture
def svc(gpu, gate, request):
    p = dict(workers=4, arena=16 << 20)
    p.update(getattr(request, "param", {}))
    with Service(gpu, **p) as s:
        yield s


# ---- ops: ("send", conn, direction, lens, seed, byte_idx, slice kinds) / ("recv", conn, direction, cap, dst kind)

def _desc(op):
    if op[0] == "send":
        return "send %s dir %d lens %s byte_idx %d from %s" % (op[1].name, op[2], op[3], op[5], op[6])
    return "recv %s dir %d cap %d into %s" % (op[1].name, op[2], op[3], op[4])


def _gpu(L, arena, op):
    """one single call: accepted bytes, or (delivered bytes, SHA-1)"""
    arena.reset()
    c, d = op[1], op[2]
    if op[0] == "send":
        tx = c.ends(d)[0]
        sl = arena.place(trace.make_bufs(op[3], op[4]), op[6], op[4])
        return int(L.b200_pair_send(tx.h, sl, len(op[3]), op[5]))
    rx, cap, kind = c.ends(d)[1], op[3], op[4]
    if kind == "plain":
        out = rx.recv(cap)
    else:
        dst = arena.alloc(kind, cap, cap % 16)
        out = arena.get(kind, dst, int(L.b200_pair_recv(rx.h, dst, cap)))
    return int(out.size), trace.sha(out)


def _model(op):
    c = op[1]
    mtx, mrx = c.ends(op[2])[2:]
    if op[0] == "send":
        return int(c.model.send(mtx, trace.make_bufs(op[3], op[4]), op[5]))
    out = c.model.recv(mrx, op[3])
    return int(out.size), trace.sha(out)


def _step(L, arena, op, label):
    g, w = _gpu(L, arena, op), _model(op)
    assert g == w, "%s: %s\n got  %s\n want %s" % (label, _desc(op), g, w)
    return g


def _send(rng, c, d, lens, bidx=None, kinds=None):
    if bidx is None:
        bidx = int(rng.integers(0, lens[0])) if lens[0] else 0
    if kinds is None:
        kinds = [Arena.KINDS[int(x)] for x in rng.integers(0, 4, len(lens))]
    return ("send", c, d, [int(x) for x in lens], int(rng.integers(0, 1 << 16)), bidx, kinds)


def _recv(rng, c, d, cap=None, kind=None):
    if cap is None:
        cap = [int(rng.integers(1, 64)), int(rng.integers(1, 4096)), 1 << 17][int(rng.integers(0, 3))]
    return ("recv", c, d, cap, kind or DST[int(rng.integers(0, 4))])


def _small_lens(rng):
    """<= kSvcInline slices of <= kSmallMax bytes in all: the owner moves the Send itself"""
    n = int(rng.integers(1, INLINE + 1))
    s = int(rng.integers(0, 3))
    if s == 0:  # unary-shaped
        return [9] + [int(x) for x in rng.integers(1, 2000, n - 1)]
    if s == 1:  # tiny, zero-length slices included
        return [int(x) for x in rng.integers(0, 64, n)]
    return [int(x) for x in rng.integers(1, SMALL_MAX // n + 1, n)]


def _pool_lens(rng, cap):
    """more than kSvcInline slices, or more than kSmallMax bytes: the owner hands the Send to the pool"""
    if rng.integers(0, 2):
        return [int(x) for x in rng.integers(1, 700, int(rng.integers(INLINE + 1, 13)))]
    return [9, int(rng.integers(SMALL_MAX, max(2 * cap, 20000)))]


def _small_visit(rng, c):
    """ops of one visit to a connection that the owner serves itself: small Sends and Recvs of frames <= kSmallMax"""
    ops = []
    for _ in range(int(rng.integers(2, 5))):
        d = int(rng.integers(0, 2))
        ops.append(_send(rng, c, d, _small_lens(rng)) if rng.integers(0, 2) else _recv(rng, c, d))
    return ops


def _mixed_op(rng, c):
    d = int(rng.integers(0, 2))
    k = int(rng.integers(0, 10))
    if k < 4:
        return _send(rng, c, d, _small_lens(rng))
    if k < 6:
        return _send(rng, c, d, _pool_lens(rng, c.cap))
    return _recv(rng, c, d)


def _close(conns):
    for c in conns:
        c.close()


def _check_all(conns, label, images=True):
    for c in conns:
        _check_conn(c, label, images)


# ---- 1. more connections than the cache holds

@pytest.mark.parametrize("svc", [dict(owners=1)], indirect=True, ids=["owners1"])
@pytest.mark.parametrize("nconn", [CACHE, CACHE + 1], ids=["8-all-hits", "9-first-op-misses"])
def test_rotation_over_the_cache(svc, models, nconn):
    """One owner serves every connection.  A fixed rotation over 8 connections hits the cache on every op after
    the first lap; over 9 connections first-in first-out refill evicts the connection visited next, so the first
    op of every visit misses and reloads both lines.  Only small ops: a pool hand-over would drop an entry."""
    pkg, L, arena = svc.pkg, svc.L, svc.arena
    rng = np.random.default_rng(8000 + nconn)
    conns = [Conn(pkg, models, MODES[i % 3], (4096, 16384)[(i // 3) % 2]) for i in range(nconn)]
    try:
        for lap in range(8):
            for i, c in enumerate(conns):
                for j, op in enumerate(_small_visit(rng, c)):
                    _step(L, arena, op, "lap %d visit %d op %d" % (lap, i, j))
            _check_all(conns, "after lap %d" % lap)
    finally:
        _close(conns)


@pytest.mark.parametrize("svc", [dict(owners=1), dict(owners=None)], indirect=True, ids=["owners1", "owners32"])
def test_random_order_over_24_connections(svc, models):
    """24 connections in all three framing modes, both directions, visited in random order: small Sends, Sends the
    owner hands to the pool, partial and whole Recvs (those of frames > kSmallMax go to the pool too)."""
    pkg, L, arena = svc.pkg, svc.L, svc.arena
    rng = np.random.default_rng(8100 + (svc.owners or 0))
    conns = [Conn(pkg, models, MODES[i % 3], (4096, 16384, 65536)[(i // 3) % 3]) for i in range(24)]
    hits = L.b200_service_eager_hits()
    try:
        for r in range(6):
            for i in range(150):
                c = conns[int(rng.integers(0, len(conns)))]
                _step(L, arena, _mixed_op(rng, c), "round %d op %d" % (r, i))
            _check_all(conns, "after round %d" % r)
    finally:
        _close(conns)
    assert L.b200_service_eager_hits() > hits


# ---- 2. the owner's routing limits

@pytest.mark.parametrize("svc", [dict(owners=1)], indirect=True, ids=["owners1"])
@pytest.mark.parametrize("mode", MODES)
def test_routing_limits(svc, models, mode):
    """Each side of kSmallMax (Send total and Recv head frame), kSvcInline (slices) and kEagerMax (eager frames) on
    one connection, with ops on three other connections of the same owner between them; then a pool op followed at
    once by a small op of the same connection, in both orders and on both ends (owner_reap's wait for the job and
    the cache entry dropped at the hand-over)."""
    pkg, L, arena = svc.pkg, svc.L, svc.arena
    rng = np.random.default_rng(8200 + MODES.index(mode))
    c = Conn(pkg, models, mode, 65536)
    others = [Conn(pkg, models, MODES[i], 4096) for i in range(3)]
    hits = L.b200_service_eager_hits()

    def between(label):
        for o in others:
            d = int(rng.integers(0, 2))
            _step(L, arena, _send(rng, o, d, _small_lens(rng)), label + " (between)")
            _step(L, arena, _recv(rng, o, d), label + " (between)")

    try:
        cases = [[SMALL_MAX], [SMALL_MAX + 1], [9, SMALL_MAX - 9], [9, SMALL_MAX - 8],  # total payload
                 [700] * INLINE, [700] * (INLINE + 1), [1] * INLINE, [1] * (INLINE + 1),  # slices
                 [EAGER_MAX], [EAGER_MAX + 1], [EAGER_MAX - 9, 9], [EAGER_MAX]]  # eager frames
        for d in (0, 1):
            for k, lens in enumerate(cases):
                label = "%s dir %d case %d %s" % (mode, d, k, lens)
                _step(L, arena, _send(rng, c, d, lens, 0, [Arena.KINDS[(k + i) % 4] for i in range(len(lens))]), label)
                between(label)
                # the head frame is the case's first frame: <= kSmallMax taken by the owner, beyond by the pool
                for kind in ("host", "plain"):
                    _step(L, arena, _recv(rng, c, d, 1 << 16, kind), label)
                between(label)
                _check_conn(c, label)
            for order in ("pool-small", "small-pool"):
                for k in range(3):
                    label = "%s dir %d %s %d" % (mode, d, order, k)
                    pool, small = _pool_lens(rng, c.cap), _small_lens(rng)
                    for lens in ((pool, small) if order == "pool-small" else (small, pool)):
                        _step(L, arena, _send(rng, c, d, lens), label)
                    # a Recv of each kind of frame, each right before a small op on the other end
                    for kind in ("device", "host"):
                        _step(L, arena, _recv(rng, c, d, 1 << 16, kind), label)
                        _step(L, arena, _send(rng, c, 1 - d, _small_lens(rng)), label)
                    _step(L, arena, _recv(rng, c, 1 - d, 1 << 16), label)
                    _step(L, arena, _recv(rng, c, d, 1 << 17), label)
                    _check_conn(c, label)
                    between(label)
        _check_all(others, "%s others" % mode)
    finally:
        _close([c] + others)
    assert L.b200_service_eager_hits() > hits, "no Recv was an eager hit: the eager path never ran"


# ---- 3. threads on one owner

def _join(threads, errors, what):
    for th in threads:
        th.join(300)
    assert not any(th.is_alive() for th in threads), "%s: a thread did not finish" % what
    assert not errors, errors


@pytest.mark.parametrize("svc", [dict(owners=1)], indirect=True, ids=["owners1"])
@pytest.mark.parametrize("nthreads", [8, 20])
def test_threads_on_one_owner(svc, models, nthreads):
    """Threads drive disjoint connections with single calls through one owner queue; with 20 threads more than
    kOwnQ commands are in flight at once, so posters wait for the queue to wrap.  Recvs into host memory are eager
    hits whose Retires ride on that pair's next Send.  Each thread records its results; the records are compared
    with the models after the join."""
    pkg, L = svc.pkg, svc.L
    rng = np.random.default_rng(8300 + nthreads)
    per, nops = 2, 40
    conns = [[Conn(pkg, models, MODES[(t + i) % 3], (4096, 16384)[i % 2]) for i in range(per)] for t in range(nthreads)]
    try:
        plans = [[_mixed_op(rng, conns[t][int(rng.integers(0, per))]) for _ in range(nops)] for t in range(nthreads)]
        arenas = [svc.arena.part(t, nthreads) for t in range(nthreads)]
        recs = [[] for _ in range(nthreads)]
        errors = []

        def drive(t):
            try:
                for op in plans[t]:
                    recs[t].append(_gpu(L, arenas[t], op))
            except BaseException as ex:  # reported by the main thread
                errors.append((t, repr(ex)))

        threads = [threading.Thread(target=drive, args=(t,)) for t in range(nthreads)]
        for th in threads:
            th.start()
        _join(threads, errors, "single calls")
        for t in range(nthreads):
            for i, (op, g) in enumerate(zip(plans[t], recs[t])):
                w = _model(op)
                assert g == w, "thread %d op %d: %s\n got  %s\n want %s" % (t, i, _desc(op), g, w)
            _check_all(conns[t], "thread %d at the end" % t)
    finally:
        for cs in conns:
            _close(cs)


def _readiness_drained(c, label):
    """both directions once everything sent was received: nothing pending, nothing readable, no stale has_message"""
    g = _views(c, False)
    for d in (0, 1):
        rx = c.ends(d)[1]
        v = g[d]
        assert v["ready"][:3] == (0, 0, 0), "%s: direction %d: readiness %s" % (label, d, v)
        assert v["rx"]["head"] == v["tx"]["remote_tail"] and v["rx"]["remain"] == 0, "%s: direction %d: %s" % (label, d, v)
        assert rx.recv(1 << 16).size == 0, "%s: direction %d: a Recv still delivers" % (label, d)


def _stream(rng, total_slices, seed):
    lens = [int(x) for x in rng.integers(1, 3000, total_slices)]
    lens[::4] = [9] * len(lens[::4])
    bufs = trace.make_bufs(lens, seed)
    return lens, bufs, np.concatenate(bufs)


class _Sender:
    """the endpoint's rdma_flush loop over a stream: Send from the returned position until everything is accepted"""

    def __init__(self, send, lens, deadline):
        self.send, self.lens, self.deadline = send, lens, deadline
        self.idx = self.bidx = self.sent = 0

    def run(self):
        while self.idx < len(self.lens):
            assert time.monotonic() < self.deadline, "sender stuck at %d bytes" % self.sent
            n = self.send(self.idx, self.bidx)
            if n == 0:
                time.sleep(0)  # no credit yet: let the receiver run
            self.sent += n
            while n > 0:
                left = self.lens[self.idx] - self.bidx
                if n >= left:
                    n, self.idx, self.bidx = n - left, self.idx + 1, 0
                else:
                    self.bidx, n = self.bidx + n, 0


def _receiver(recv, total, deadline, what):
    parts, got = [], 0
    while got < total:
        assert time.monotonic() < deadline, "%s: receiver stuck at %d of %d bytes" % (what, got, total)
        out = recv()
        got += out.size
        if out.size:
            parts.append(out)
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8)


@pytest.mark.parametrize("svc", [dict(owners=1)], indirect=True, ids=["owners1"])
@pytest.mark.parametrize("mode", MODES)
def test_sender_and_receiver_threads_on_one_connection(svc, models, mode):
    """Four threads on one connection: a sender and a receiver per direction.  Per-op counts depend on timing; the
    delivered streams must be intact, and once every thread has stopped both directions must read as drained (a
    stale has_message = 0 over a frame in the ring would leave a receiver stuck: the host answers Recv from it)."""
    pkg, L, arena = svc.pkg, svc.L, svc.arena
    rng = np.random.default_rng(8400 + MODES.index(mode))
    c = Conn(pkg, models, mode, 16384)
    try:
        streams = [_stream(rng, 600, 50 + d) for d in (0, 1)]
        parts = [arena.part(i, 4) for i in range(4)]
        srcs = []
        for d in (0, 1):  # the stream's slices in pinned host memory, placed once
            srcs.append(parts[d].place(streams[d][1], ["host"] * len(streams[d][0]), d))
        deadline = time.monotonic() + 30
        errors, got = [], [None, None]

        def send(d):
            tx = c.ends(d)[0]
            lens = streams[d][0]
            ptrs = [(srcs[d][i].ptr, srcs[d][i].len) for i in range(len(lens))]
            try:
                _Sender(lambda idx, bidx: int(L.b200_pair_send(tx.h, pkg.make_slices(ptrs[idx:idx + 8]),
                                                                min(8, len(lens) - idx), bidx)), lens, deadline).run()
            except BaseException as ex:
                errors.append(("send", d, repr(ex)))

        def recv(d):
            rx = c.ends(d)[1]
            r = np.random.default_rng(d)
            dst = parts[2 + d].alloc("host", 1 << 14)
            try:
                got[d] = _receiver(lambda: parts[2 + d].get("host", dst, int(L.b200_pair_recv(rx.h, dst, int(r.integers(1, 1 << 14))))),
                                   streams[d][2].size, deadline, "direction %d" % d)
            except BaseException as ex:
                errors.append(("recv", d, repr(ex)))

        threads = [threading.Thread(target=f, args=(d,)) for d in (0, 1) for f in (send, recv)]
        for th in threads:
            th.start()
        _join(threads, errors, mode)
        for d in (0, 1):
            assert np.array_equal(got[d], streams[d][2]), "%s direction %d: the delivered stream differs" % (mode, d)
        _readiness_drained(c, mode)
    finally:
        c.close()


# ---- 4. prepared batches launched beside the owners

PATHS = {"device": ("device", "device"), "staged": ("host", "host")}  # (batch slice memory, batch Recv destination)


def _batch_send(pkg, arena, rng, c, d, kind):
    lens = [9, int(rng.integers(100, 3000)), 9, int(rng.integers(1, 500))]
    bufs = trace.make_bufs(lens, int(rng.integers(0, 1 << 16)))
    sl = arena.place(bufs, [kind] * len(lens), int(rng.integers(0, 16)))
    return pkg.Batch("send", [(c.ends(d)[0], sl, len(lens), 0)], pkg.UNTIL_BLOCKED), bufs


def _gated_send_batch(svc, gate, models, mode, path, others):
    """F0 single Send on a; batch Send F1 on a, gated; single Recv on b (the owner loads both lines: a's tail is
    the pre-batch one); the batch's results; single Send F2 on a and Recvs on b.  The owner must not write F2 at the
    tail it loaded before the batch ran."""
    pkg, L = svc.pkg, svc.L
    one, bat = svc.arena.part(0, 2), svc.arena.part(1, 2)
    rng = np.random.default_rng(8500 + MODES.index(mode) + 10 * len(others))
    c = Conn(pkg, models, mode, 16384)
    try:
        for k in range(8):
            label = "%s %s round %d" % (mode, path, k)
            _step(L, one, _send(rng, c, 0, _small_lens(rng)), label + " F0")
            bat.reset()
            b, bufs = _batch_send(pkg, bat, rng, c, 0, PATHS[path][0])
            try:
                gate.launch(b)
                for o in others:
                    _step(L, one, _mixed_op(rng, o), label + " (between)")
                _step(L, one, _recv(rng, c, 0, kind=DST[k % 4]), label + " Recv behind the gate")
                for o in others:
                    _step(L, one, _mixed_op(rng, o), label + " (between)")
                gate.held(label)
                acc = gate.results(b)[0]
            finally:
                b.destroy()
            want = int(c.model.send_all(c.ma, bufs, 0)[0])
            assert acc == want, "%s: batch F1 accepted %d, model %d" % (label, acc, want)
            _step(L, one, _send(rng, c, 0, _small_lens(rng)), label + " F2")
            for j in range(3):
                _step(L, one, _recv(rng, c, 0, kind=DST[(k + j) % 4]), label + " Recv %d" % j)
            _check_conn(c, label)
        _check_all(others, "%s %s others" % (mode, path))
    finally:
        c.close()


def _gated_recv_batch(svc, gate, models, mode, path, others):
    """The mirror case: F0 single Send on a; batch Recv on b, gated; single Send F1 on a (the owner loads b's
    pre-batch head); the batch's results; single Send F2 on a and Recvs on b.  The owner must not answer from the
    head, the rx counter or the readiness it loaded before the batch consumed the frames."""
    pkg, L = svc.pkg, svc.L
    one, bat = svc.arena.part(0, 2), svc.arena.part(1, 2)
    rng = np.random.default_rng(8600 + MODES.index(mode) + 10 * len(others))
    c = Conn(pkg, models, mode, 16384)
    kind = PATHS[path][1]
    try:
        for k in range(8):
            label = "%s %s round %d" % (mode, path, k)
            _step(L, one, _send(rng, c, 0, _small_lens(rng)), label + " F0")
            bat.reset()
            cap = [1 << 15, int(rng.integers(1, 3000))][k % 2]
            dst = bat.alloc(kind, cap, k)
            b = pkg.Batch("recv", [(c.b, dst, cap)], pkg.UNTIL_BLOCKED)
            try:
                gate.launch(b)
                for o in others:
                    _step(L, one, _mixed_op(rng, o), label + " (between)")
                _step(L, one, _send(rng, c, 0, _small_lens(rng)), label + " F1 behind the gate")
                for o in others:
                    _step(L, one, _mixed_op(rng, o), label + " (between)")
                gate.held(label)
                n = gate.results(b)[0]
            finally:
                b.destroy()
            out = bat.get(kind, dst, n)
            want, _ = c.model.recv_drain(c.mb, cap)
            assert trace.sha(out) == trace.sha(want), "%s: batch Recv delivered %d bytes, model %d" % (label, n, want.size)
            _step(L, one, _send(rng, c, 0, _small_lens(rng)), label + " F2")
            for j in range(3):
                _step(L, one, _recv(rng, c, 0, kind=DST[(k + j) % 4]), label + " Recv %d" % j)
            _check_conn(c, label)
        _check_all(others, "%s %s others" % (mode, path))
    finally:
        c.close()


@pytest.mark.parametrize("svc", [dict(owners=1)], indirect=True, ids=["owners1"])
@pytest.mark.parametrize("path", sorted(PATHS))
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("batch", ["send", "recv"])
@pytest.mark.parametrize("between", [0, 3], ids=["alone", "others-between"])
def test_batch_beside_the_owner(svc, gate, models, mode, path, batch, between):
    pkg = svc.pkg
    others = [Conn(pkg, models, MODES[i % 3], 4096) for i in range(between)]
    try:
        (_gated_send_batch if batch == "send" else _gated_recv_batch)(svc, gate, models, mode, path, others)
    finally:
        _close(others)


@pytest.mark.parametrize("svc", [dict(owners=1)], indirect=True, ids=["owners1"])
@pytest.mark.parametrize("path", sorted(PATHS))
@pytest.mark.parametrize("mode", MODES)
def test_batch_send_loop_beside_single_recvs(svc, gate, models, mode, path):
    """Unsynchronised: one thread sends a stream on a with prepared batches (launched on a stream of its own,
    results collected there), another takes it on b with single Recvs.  The stream must arrive intact and the
    connection must read as drained afterwards."""
    pkg, L = svc.pkg, svc.L
    rng = np.random.default_rng(8700 + MODES.index(mode))
    c = Conn(pkg, models, mode, 16384)
    src, rcv = svc.arena.part(0, 2), svc.arena.part(1, 2)
    lens, bufs, msg = _stream(rng, 400, 77)
    skind = PATHS[path][0]
    try:
        sl = src.place(bufs, [skind] * len(lens), 3)
        ptrs = [(sl[i].ptr, sl[i].len) for i in range(len(lens))]
        deadline = time.monotonic() + 30
        errors, got = [], [None]

        def send_batch(idx, bidx):
            n = min(16, len(lens) - idx)
            b = pkg.Batch("send", [(c.a, pkg.make_slices(ptrs[idx:idx + n]), n, bidx)], pkg.UNTIL_BLOCKED)
            try:
                b.launch(gate.free_h)
                return int(b.results(gate.free_h)[0])
            finally:
                b.destroy()

        def send():
            try:
                _Sender(send_batch, lens, deadline).run()
            except BaseException as ex:
                errors.append(("send", repr(ex)))

        def recv():
            r = np.random.default_rng(5)
            kinds = ("host", "device", "plain")
            dst = {k: rcv.alloc(k, 1 << 14) for k in kinds if k != "plain"}

            def one():
                k = kinds[int(r.integers(0, 3))]
                cap = int(r.integers(1, 1 << 14))
                if k == "plain":
                    return c.b.recv(cap)
                return rcv.get(k, dst[k], int(L.b200_pair_recv(c.b.h, dst[k], cap)))

            try:
                got[0] = _receiver(one, msg.size, deadline, "%s %s" % (mode, path))
            except BaseException as ex:
                errors.append(("recv", repr(ex)))

        threads = [threading.Thread(target=send), threading.Thread(target=recv)]
        for th in threads:
            th.start()
        _join(threads, errors, "%s %s" % (mode, path))
        assert np.array_equal(got[0], msg), "%s %s: the delivered stream differs" % (mode, path)
        _readiness_drained(c, "%s %s" % (mode, path))
    finally:
        c.close()


# ---- 5. generation changes mid-stream

def _reuse_conn(pkg, models, mode, cap, freed):
    """a new connection on the pool entries of `freed`, a Conn just closed.  The pool is first-in first-out: the
    entries ahead of freed.a are held out of it until the new connection has taken freed.a and freed.b."""
    L = pkg.lib()
    ahead = []
    h = L.b200_pool_take(b"")
    while h != freed.a.h:
        assert h, pkg.last_error()
        ahead.append(h)
        h = L.b200_pool_take(b"")
    orig = pkg.Pair

    class Taken(orig):  # the first end of the new connection is the entry already taken
        def __init__(self, ident=""):
            if Taken.h is None:
                return orig.__init__(self, ident)
            self.L, self.h, Taken.h = L, Taken.h, None
            L.b200_pair_init(self.h)
            assert L.b200_pair_status(self.h) == 1, self.error()
    Taken.h = h
    pkg.Pair = Taken
    try:
        return Conn(pkg, models, mode, cap)
    finally:
        pkg.Pair = orig
        for x in ahead:
            L.b200_pool_putback(x)


@pytest.mark.parametrize("svc", [dict(owners=1)], indirect=True, ids=["owners1"])
def test_generation_changes_mid_stream(svc, models):
    """Ten connections keep running against their models on one owner while unrelated connections are created and
    closed (one of them on the pool entries a connection just freed) and an unrelated end is claimed by and
    released from the device API.  Every change bumps the host's generation and the owner drops its cache."""
    pkg, L, arena = svc.pkg, svc.L, svc.arena
    rng = np.random.default_rng(8800)
    conns = [Conn(pkg, models, MODES[i % 3], (4096, 16384)[i % 2]) for i in range(10)]
    side = Conn(pkg, models, "ref", 4096)
    try:
        for r in range(9):
            label = "round %d" % r
            ev = r % 3
            if ev == 0:  # create, use and close an unrelated connection
                x = Conn(pkg, models, MODES[r % 3], 4096)
                _step(L, arena, _send(rng, x, 0, _small_lens(rng)), label + " new")
            elif ev == 1:  # the entries a connection just freed, reused by a new one
                x = Conn(pkg, models, MODES[r % 3], 4096)
                _step(L, arena, _send(rng, x, 1, _small_lens(rng)), label + " to be freed")
                x.close()
                freed = x
                x = _reuse_conn(pkg, models, MODES[(r + 1) % 3], 16384, freed)
                assert (x.a.h, x.b.h) == (freed.a.h, freed.b.h), "the new connection is not on the freed entries"
                _step(L, arena, _send(rng, x, 0, _small_lens(rng)), label + " reused")
            else:  # claim an unrelated end for the device API
                side.a.device_claim()
            for i in range(40):
                c = conns[int(rng.integers(0, len(conns)))]
                _step(L, arena, _mixed_op(rng, c), "%s op %d" % (label, i))
                if i == 20 and ev != 2:
                    _step(L, arena, _recv(rng, x, 0, 1 << 16), label + " unrelated Recv")
                    x.close()
                    x = None
                if i == 20 and ev == 2:
                    side.a.device_release()
            _check_all(conns, label)
        _check_conn(side, "the released end")
        for d in (0, 1):
            _step(L, arena, _send(rng, side, d, _small_lens(rng)), "the released end")
            _step(L, arena, _recv(rng, side, d, 1 << 16), "the released end")
        _check_conn(side, "the released end, used")
    finally:
        if side.a.device_owned():
            side.a.device_release()
        _close(conns + [side])
