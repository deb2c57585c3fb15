"""GPU: stamped ring frames (B200_RING_STAMPED=1, DESIGN.md §2) at the limits of the frame counters, on every path that
writes or checks a stamp, bit for bit against the stamped model (tests/native/stamp_oracle.c).

Every pair starts at frame 0, so without seeding no GPU test gets near the stamp rollover (2^24 - 1 -> 1) or past
2^32 frames.  Here the sender's and the receiver's counters (PairSeq) are seeded through the b200_dev_pair handle,
the model gets the same values, and each replay compares returns, calls, cursors, readiness and the masked ring
image after every op (test_stamp_gpu._replay).  The seeds and the closed form t(s) = 1 + s mod (2^24 - 1) are
pinned on the CPU in test_stamp_limits_cpu.py.

1. rollover: the stamp-(2^24 - 1) frame at the edges of a call, of the receiver's 32-frame scout and of a footer
   segment, and counters past 2^32, through host calls, batches, the service, b200_pairs_submit, warp and block calls
2. readiness with the head on the stamp-(2^24 - 1) frame, then on the stamp-1 frame
3. mismatched counters: a receiver whose stamp is one bit or one frame off reads nothing, everywhere
4. the largest stamped ring (256 MiB) and the first one too large to offer stamped frames

Not covered here: a full lap of minimum-size frames at 256 MiB (the C/24 < 2^24 - 1 margin, DESIGN.md §2) and the
CUDA-IPC wire (two GPUs)."""
import ctypes as C
import select
import time

import numpy as np
import pytest

import device_block_lib as bl
import device_lib
import device_poll_lib
import stamp_lib
import test_submit_gpu
import trace
from device_block_lib import BlockEngine
from device_lib import DeviceEngine
from submit_lib import SubmitEngine
from test_stamp_gpu import StampedGpuEngine, _replay
from test_stamp_limits_cpu import (LANE_SEEDS, LEN_MASK, MIS_S, MISMATCHED, SEGMENT_SEEDS, WIDE_SEEDS, M,
                                   fresh_counters, seq_address, u64)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

STAMPED = {"B200_RING_STAMPED": 1}
CAP = 1 << 16
EDGE = [M - 1, (1 << 32) - 3]  # every path gets these


def expected_stamp(s):
    """t(s), computed here independently of the model and of the kernels"""
    return 1 + s % (2**24 - 1)


# ---- seeding

def _seq(L, handle, value=None):
    """write (tx, rx) into the PairSeq the handle names, or read it back"""
    v = np.array(value if value is not None else (0, 0), np.uint64)
    d = 0 if value is not None else 1
    if d == 0:
        assert L.b200_memcpy(seq_address(handle), v.ctypes.data, 16, 0, None) == 0
    else:
        assert L.b200_memcpy(v.ctypes.data, seq_address(handle), 16, 1, None) == 0
    assert L.b200_stream_sync(None) == 0
    return int(v[0]), int(v[1])


class Seeded:
    """Engine mixin: right after pair_pair the sender's PairSeq.tx is seeds[0] and the receiver's PairSeq.rx is
    seeds[1].  An end the engine drives from the device is written through its handle; a host end is claimed,
    written and released (the release re-publishes the mirror from the device state, and claim and release both
    make the service's owner warps drop their cached copy of the connection).  After the first Send the receiver's
    ring must hold a frame stamped t(seeds[0]): a seed that did not land fails here, not vacuously later."""

    def __init__(self, *args, seeds, **kw):
        super().__init__(*args, **kw)
        self.seeds = seeds
        self._first = None

    def pair_pair(self, cap, max_sge=30):
        tx, rx = super().pair_pair(cap, max_sge)
        assert tx.stamped() and rx.stamped()
        L = self.pkg.lib()
        for p, value in ((tx, (self.seeds[0], 0)), (rx, (0, self.seeds[1]))):
            h = getattr(self, "handles", {}).get(p.h)
            if h is not None:
                _seq(L, h, value)
                assert _seq(L, h) == value
            else:
                h = p.device_claim()
                _seq(L, h, value)
                assert _seq(L, h) == value
                p.device_release()
        self._first = rx
        return tx, rx

    def _check_first(self, n):
        if self._first is not None and n:
            rx, self._first = self._first, None
            hdr = u64(rx.ring_image(), 0)
            assert hdr & LEN_MASK and hdr >> 40 == expected_stamp(self.seeds[0]), hex(hdr)

    def send(self, p, bufs, byte_idx=0):
        n = super().send(p, bufs, byte_idx)
        self._check_first(n)
        return n

    def send_all(self, p, bufs, byte_idx=0):
        r = super().send_all(p, bufs, byte_idx)
        self._check_first(r[0])
        return r


class SeededHost(Seeded, StampedGpuEngine):
    pass


class SeededDevice(Seeded, DeviceEngine):
    pass


class SeededBlock(Seeded, BlockEngine):
    pass


class SeededSubmit(Seeded, SubmitEngine):
    pass


class SeededModel(stamp_lib.StampedOracle):
    """the stamped model with the same seeds; no_calls: b200_pairs_submit does not count calls (-1)"""

    def __init__(self, coalesced=False):
        super().__init__(coalesced)
        self.seeds, self.no_calls = (0, 0), False

    def pair_pair(self, cap, max_sge=30):
        a, b = super().pair_pair(cap, max_sge)
        fresh_counters(self, a, b)
        self.S.stamp_seq_set(a, self.seeds[0], 0)
        self.S.stamp_seq_set(b, 0, self.seeds[1])
        return a, b

    def send_all(self, p, bufs, byte_idx=0):
        n, calls = super().send_all(p, bufs, byte_idx)
        return n, (-1 if self.no_calls else calls)

    def recv_drain(self, p, cap):
        out, calls = super().recv_drain(p, cap)
        return out, (-1 if self.no_calls else calls)


@pytest.fixture(scope="module")
def sm():
    return SeededModel()


@pytest.fixture(scope="module")
def smc():
    return SeededModel(coalesced=True)


@pytest.fixture
def svc(gpu):
    """the service with an Arena for b200_pairs_submit; the drivers' kernels are loaded before it starts"""
    bl.Runner(gpu)
    device_lib.Runner(gpu)
    device_poll_lib.Runner(gpu).close()
    with test_submit_gpu.Service(gpu) as s:
        yield s


def _run(eng, model, seeds, ops, cap=CAP, images=True, no_calls=False):
    model.seeds, model.no_calls = seeds, no_calls
    try:
        _replay(eng, model, cap, ops, images)
    finally:
        model.no_calls = False


# ---- workloads: short traces whose first op writes frames into the empty ring

def _stream_ops():
    """chttp2-shaped [9, n]: period-two frames put k_recv's scout on its speculative path, at several offsets"""
    return [("send_all", [9, 1200] * 20, 11, 0), ("recv_drain", 1 << 20),
            ("send_all", [9, 700] * 20, 12, 0), ("recv", 100), ("recv_drain", 1 << 20),
            ("send_all", [9, 300] * 20, 13, 5), ("recv", 9), ("recv", 50), ("recv_drain", 1 << 20),
            ("stream", [9, 2500] * 24, 14, 30000)]


def _small_ops():
    """irregular frames of <= 32 B (the sequential walk, frames that bypass the movers)"""
    return [("send", [1, 7, 8, 9, 16, 17, 31, 32, 3, 24] * 3, 21, 0), ("recv", 1), ("recv", 40),
            ("recv_drain", 1 << 16), ("send_all", [5, 32, 12, 1] * 12, 22, 2), ("recv_drain", 100),
            ("recv_drain", 1 << 16), ("send", [32] * 40, 23, 31), ("recv_drain", 1 << 16)]


def _partial_ops():
    """partial reads that straddle the first frames (for M - 1 / M - 2: the stamp-M and the stamp-1 frame)"""
    return [("send", [40, 50, 60, 70], 31, 0), ("recv", 7), ("recv", 100), ("recv", 13), ("recv", 13),
            ("recv", 100), ("recv", 3), ("recv", 100), ("recv", 69), ("recv", 100), ("recv", 100)]


def _segment_ops():
    """one send_all of 1 150 8-byte slices: one op spans two 512-entry footer segments"""
    return [("send_all", [8] * 1150, 41, 3), ("recv_drain", 5000), ("recv_drain", 1 << 20)]


def _owner_ops():
    """calls the service's owner warps run by themselves (<= 5 slices of small frames, single Recv calls), with
    unary-shaped messages received right after (eager push, then the owed Retire)"""
    ops = []
    for k in range(12):
        ops += [("send", [9, 5, 20 + k], 50 + k, 0), ("recv", 1 << 16), ("send", [3, 31, 8, 1, 32], 70 + k, k % 3),
                ("recv", 4), ("recv", 1 << 16), ("recv", 1 << 16), ("recv", 1 << 16), ("recv", 1 << 16)]
    return ops


def _workloads(seed):
    """which traces a seed gets: the lane seeds the reading ones, the segment seeds the long send_all"""
    w = []
    if seed in LANE_SEEDS or seed in WIDE_SEEDS:
        w += [_stream_ops(), _small_ops()]
    if seed in (M - 1, M - 2) or seed in WIDE_SEEDS:
        w += [_partial_ops()]
    if seed in SEGMENT_SEEDS or seed in EDGE:
        w += [_segment_ops()]
    return w


ALL_SEEDS = LANE_SEEDS + SEGMENT_SEEDS + WIDE_SEEDS


# ---- 1. rollover matrix

@pytest.mark.parametrize("seed", ALL_SEEDS)
@pytest.mark.parametrize("mem", [("device", 0), ("pinned", 9)])
def test_rollover_host_calls_and_batches(gpu, sm, seed, mem):
    """b200_pair_send / recv (k_send / k_recv single calls) and prepared batches (send_all / recv_drain)"""
    for ops in _workloads(seed):
        _run(SeededHost(gpu, *mem, seeds=(seed, seed)), sm, (seed, seed), ops)


@pytest.mark.parametrize("seed", LANE_SEEDS[:2] + LANE_SEEDS[4:] + WIDE_SEEDS)
def test_rollover_host_coalesced(gpu, smc, seed):
    """coalesced framing: one frame per Send call, against its own model"""
    for ops in (_stream_ops(), _small_ops()) + ((_partial_ops(),) if seed in (M - 1, M - 2) else ()):
        _run(SeededHost(gpu, "device", 3, coalesced=True, seeds=(seed, seed)), smc, (seed, seed), ops)


@pytest.mark.parametrize("seed", [M - 1, M - 2, M - 17, M - 33, M - 510, M - 513] + WIDE_SEEDS)
def test_rollover_under_the_service(svc, sm, smc, seed):
    """small calls in the owner warps (stamped headers, eager push, owed Retire), the rest in the pool"""
    L = svc.L
    hits = L.b200_service_eager_hits()
    _run(SeededHost(svc.pkg, "pinned", 3, seeds=(seed, seed)), sm, (seed, seed), _owner_ops())
    assert L.b200_service_eager_hits() > hits
    for ops in _workloads(seed):
        _run(SeededHost(svc.pkg, "pinned", 3, seeds=(seed, seed)), sm, (seed, seed), ops)
    if seed in EDGE:
        _run(SeededHost(svc.pkg, "pinned", 3, coalesced=True, seeds=(seed, seed)), smc, (seed, seed), _owner_ops())


@pytest.mark.parametrize("seed", [M - 1, M - 32, M - 511, M - 600] + WIDE_SEEDS)
def test_rollover_through_submit(svc, sm, seed):
    """b200_pairs_submit passes under the service (the endpoint's data path)"""
    for ops in _workloads(seed):
        _run(SeededSubmit(svc.pkg, svc.arena, stamped=True, seeds=(seed, seed)), sm, (seed, seed), ops,
             no_calls=True)


DRIVE_CASES = ([(s, ("tx", "rx")) for s in LANE_SEEDS + WIDE_SEEDS]
               + [(s, d) for s in EDGE for d in (("tx",), ("rx",))])


@pytest.mark.parametrize("seed,drive", DRIVE_CASES)
def test_rollover_warp_calls(gpu, sm, seed, drive):
    """b200_warp_send / recv; with one end on the host, host and device hand each other the counter across the
    rollover"""
    for ops in _workloads(seed):
        _run(SeededDevice(gpu, "device", 0, drive=drive, config=STAMPED, seeds=(seed, seed)), sm, (seed, seed), ops)


BLOCK_CASES = ([(s, 0) for s in LANE_SEEDS + SEGMENT_SEEDS + WIDE_SEEDS] + [(s, 3) for s in EDGE])


@pytest.mark.parametrize("seed,warp_every", BLOCK_CASES)
def test_rollover_block_calls(gpu, sm, seed, warp_every):
    """b200_block_send / recv (warp_every 3: every third single call a warp call on the same pair)"""
    for ops in _workloads(seed):
        _run(SeededBlock(gpu, "device", 1, config=STAMPED, warp_every=warp_every, seeds=(seed, seed)), sm,
             (seed, seed), ops)


# ---- 2. readiness at the rollover, and with mismatched counters

def _host_scan(pkg, p):
    arr = (C.c_void_p * 1)(p.h)
    ev = (C.c_uint32 * 1)()
    n = pkg.lib().b200_poller_scan(arr, 1, ev)
    assert n >= 0, pkg.last_error()
    return n, int(ev[0])


def _check_ready(pkg, eng, R, rx, model, mrx, label):
    """every readiness answer for the receive end equals the model's"""
    rd, hm = int(model.readable(mrx)), int(model.has_message(mrx))
    ev = pkg.EV_READABLE if hm else 0
    h = eng.handles[rx.h]
    got = {"mirror": (int(rx.has_message()), int(rx.readable())), "scan": _host_scan(pkg, rx),
           "warp_poll": R.poll([h])[:2], "device": tuple(int(x) for x in eng.device_ready(rx)[:2])}
    got["warp_poll"] = (got["warp_poll"][0], int(got["warp_poll"][1][0]))
    want = {"mirror": (hm, rd), "scan": (int(ev != 0), ev), "warp_poll": (int(ev != 0), ev), "device": (rd, hm)}
    assert got == want, label
    return hm


@pytest.mark.parametrize("s,r", [(s, s) for s in (M - 1, M - 2) + tuple(WIDE_SEEDS)] + [(MIS_S, MIS_S + M)]
                         + [(MIS_S, x) for x in MISMATCHED])
def test_readiness_answers(gpu, sm, s, r):
    """The receive end device-owned, the sender on the host: frames [9, 20, 9, 33] then one warp Recv at a time.
    With equal stamps the head walks the stamp-M frame, then the stamp-1 frame (seeds M - 1 / M - 2); with a
    mismatched receiver nothing is ever ready.  Asked of the host mirror, b200_poller_scan, b200_warp_poll and
    b200_warp_readable / has_message."""
    R = device_poll_lib.Runner(gpu)
    eng = SeededDevice(gpu, "device", 0, drive=("rx",), config=STAMPED, seeds=(s, r))
    sm.seeds = (s, r)
    tx, rx = eng.pair_pair(4096)
    mtx, mrx = sm.pair_pair(4096)
    try:
        bufs = trace.make_bufs([9, 20, 9, 33], 3)
        assert eng.send(tx, bufs) == sm.send(mtx, bufs) == 71
        ready = []
        for k in range(6):
            ready.append(_check_ready(gpu, eng, R, rx, sm, mrx, (s, r, k)))
            got, want = eng.recv(rx, 100), sm.recv(mrx, 100)
            assert np.array_equal(got, want), (s, r, k)
            assert eng.state(rx) == sm.state(mrx), (s, r, k)
        assert ready == ([1, 1, 1, 1, 0, 0] if expected_stamp(r) == expected_stamp(s) else [0] * 6)
        img = rx.ring_image()
        assert u64(img, 0) == 9 | expected_stamp(s) << 40  # the frames stay in the ring either way
    finally:
        eng.destroy(tx)
        eng.destroy(rx)
        sm.destroy(mtx)
        sm.destroy(mrx)
        R.close()


# ---- 3. mismatched counters on every reader

def _mismatch_ops():
    return [("send", [9, 700, 9, 40], 61, 0), ("recv", 100), ("recv_drain", 1 << 16),
            ("send_all", [9, 300] * 20, 62, 0), ("recv_drain", 1 << 16), ("recv", 1)]


def _owner_mismatch_ops():
    return [("send", [9, 5, 40], 63, 0), ("recv", 1 << 16), ("send", [3, 31, 8], 64, 0), ("recv", 4),
            ("recv", 1 << 16)]


MIS_CASES = MISMATCHED + [MIS_S + M]


@pytest.mark.parametrize("r", MIS_CASES)
def test_mismatched_stamps_host_warp_and_block_readers(gpu, sm, r):
    """Sender at S, receiver at R: with a stamp one bit (k = 0 .. 23) or one frame away every Recv returns 0 and
    nothing is ready while Send takes what credit allows; R = S + (2^24 - 1) delivers everything.  k_recv single
    calls and batches, the warp Recv and the block Recv, each against the model seeded the same way."""
    seeds = (MIS_S, r)
    _run(SeededHost(gpu, "device", 0, seeds=seeds), sm, seeds, _mismatch_ops())
    _run(SeededDevice(gpu, "device", 0, drive=("rx",), config=STAMPED, seeds=seeds), sm, seeds, _mismatch_ops())
    _run(SeededBlock(gpu, "device", 0, drive=("rx",), config=STAMPED, seeds=seeds), sm, seeds, _mismatch_ops())


def test_mismatched_stamps_under_the_service(svc, sm):
    """the owner warps (small Recv, eager push), the pool and b200_pairs_submit as readers"""
    for r in MIS_CASES:
        seeds = (MIS_S, r)
        _run(SeededHost(svc.pkg, "pinned", 3, seeds=seeds), sm, seeds, _owner_mismatch_ops())
        _run(SeededHost(svc.pkg, "pinned", 3, seeds=seeds), sm, seeds, _mismatch_ops())
        _run(SeededSubmit(svc.pkg, svc.arena, stamped=True, seeds=seeds), sm, seeds, _mismatch_ops(), no_calls=True)


def _kicked(p, wait_s):
    fd = p.wakeup_fd()
    end = time.monotonic() + wait_s
    while time.monotonic() < end:
        r, _, _ = select.select([fd], [], [], 0.05)
        if r:
            return True
    return False


def test_service_poller_at_the_rollover_and_with_mismatched_stamps(svc, sm):
    """k_svc_poll (the service's ready ring, turned into eventfd kicks by the background Poller): a frame at the
    head with the expected stamp kicks the receiver -- stamp 2^24 - 1, stamp 1 and R = S + (2^24 - 1) -- and one
    whose stamp is a bit or a frame off does not."""
    pkg, L = svc.pkg, svc.L
    cases = [(M - 1, M - 1), (M, M), (MIS_S, MIS_S + M)] + [(MIS_S, MISMATCHED[k]) for k in (0, 7, 16, 23, 24, 25)]
    for s, r in cases:
        eng = SeededHost(pkg, "pinned", 0, seeds=(s, r))
        sm.seeds = (s, r)
        tx, rx = eng.pair_pair(4096)
        mtx, mrx = sm.pair_pair(4096)
        try:
            L.b200_poller_add(rx.h)
            L.b200_pair_consume_wakeup(rx.h)
            bufs = trace.make_bufs([9, 20], 4)
            assert eng.send(tx, bufs) == sm.send(mtx, bufs) == 29
            want = bool(sm.has_message(mrx))
            assert want == (expected_stamp(r) == expected_stamp(s))
            assert _kicked(rx, 5.0 if want else 0.5) == want, (s, r)
            assert (rx.has_message(), rx.readable()) == (sm.has_message(mrx), sm.readable(mrx)), (s, r)
            assert _host_scan(pkg, rx) == ((1, pkg.EV_READABLE) if want else (0, 0)), (s, r)
            assert np.array_equal(eng.recv(rx, 100), sm.recv(mrx, 100)), (s, r)
        finally:
            L.b200_poller_shutdown()
            L.b200_poller_remove(rx.h)
            eng.destroy(tx)
            eng.destroy(rx)
            sm.destroy(mtx)
            sm.destroy(mrx)


# ---- 4. the largest stamped ring

BIG = 256 << 20  # kStampedMaxCap


def _big_ops():
    C_ = BIG
    return [("send", [C_ // 2 - 24, C_ - 24], 81, 0), ("recv_drain", 1 << 20), ("recv_drain", C_),
            ("send_all", [C_ // 2] * 6, 82, 5), ("recv_drain", C_ // 3 + 5), ("recv_drain", C_),
            ("send_all", [C_ // 2] * 6, 82, 5), ("recv_drain", 1 << 20), ("recv_drain", 2 * C_)]


@pytest.mark.parametrize("kind", ["host", "block"])
def test_largest_stamped_ring(gpu, sm, kind):
    """C = 256 MiB with B200_RING_STAMPED=1: both ends run stamped frames; a C/2 - 24 frame and a C - 24 one (cut),
    send_all of 3C from byte 5 and drains of several sizes match the model (no images).  Seeded at M - 1, so the
    rollover falls on the first big frames."""
    seeds = (M - 1, M - 1)
    if kind == "host":
        eng = SeededHost(gpu, "device", 0, seeds=seeds)
    else:
        eng = SeededBlock(gpu, "device", 0, config=STAMPED, seeds=seeds)
    _run(eng, sm, seeds, _big_ops(), cap=BIG, images=False)


def test_ring_over_the_stamped_limit(gpu):
    """C = 512 MiB: both ends offered stamped frames but the ring is too large, so the connection runs the
    reference format and clears what it reads"""
    pkg = gpu
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 2 * BIG)
    pkg.config_set("B200_RING_STAMPED", 1)
    try:
        a, b = pkg.connected_pair("big-a", "big-b")
    finally:
        pkg.config_set("B200_RING_STAMPED", 0)
    try:
        assert not a.stamped() and not b.stamped()
        bufs = trace.make_bufs([9, 100000, 9, 3], 91)
        assert a.send(bufs) == 100021
        out = np.concatenate([b.recv(1 << 20) for _ in range(4)])
        assert np.array_equal(out, np.concatenate(bufs))
        assert not b.ring_image().any(), "a reference-format connection clears what it reads"
    finally:
        for p in (a, b):
            p.disconnect()
            p.putback()
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", BIG)
    pkg.config_set("B200_RING_STAMPED", 1)
    try:
        a, b = pkg.connected_pair("big-c", "big-d")
    finally:
        pkg.config_set("B200_RING_STAMPED", 0)
    try:
        assert a.stamped() and b.stamped()
    finally:
        for p in (a, b):
            p.disconnect()
            p.putback()
