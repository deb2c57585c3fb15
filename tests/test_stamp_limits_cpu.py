"""CPU: stamped ring frames (B200_RING_STAMPED=1, DESIGN.md §2) at the limits of the frame counters, against a
closed form computed here: t(s) = 1 + s mod (2^24 - 1).

The stamped model (tests/native/stamp_oracle.c) and the stamp arithmetic the kernels run (the B200_HD inlines of
csrc/b200_dev.cuh, compiled for the host in tests/native/stamp_arith.cc) are both checked at the counter values the
GPU tests of test_stamp_limits_gpu.py seed: the stamp rollover 2^24 - 1 -> 1 at the edges of a Send call, of the
receiver's 32-frame scout and of a footer segment, and counters past 2^32.  A reader must compare all 24 bits of
the stamp, so headers one stamp bit away, or one frame away, are not frames."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import stamp_lib
import trace

M = (1 << 24) - 1  # stamps run 1 .. M
LEN_MASK = (1 << 40) - 1
U64 = (1 << 64) - 1
NATIVE = stamp_lib.NATIVE

# Frame-counter seeds: where the frame with stamp M (and the stamp-1 frame after it) falls.
#   M - 1, M - 2                  the first / second frame of a call
#   M - 17, M - 31, M - 32, M - 33  lane 16, 30, 31 of a 32-frame round, then the next round
#   M - 255 .. M - 600            the middle, end and just past the end of the first 512-entry footer segment
#   2^32 - 3, 2^32 + M - 2        counters past 2^32 (2^32 = 256 mod M: a narrowed counter gives other stamps)
LANE_SEEDS = [M - 1, M - 2, M - 17, M - 31, M - 32, M - 33]
SEGMENT_SEEDS = [M - 255, M - 510, M - 511, M - 513, M - 600]
WIDE_SEEDS = [(1 << 32) - 3, (1 << 32) + M - 2]
SEEDS = LANE_SEEDS + SEGMENT_SEEDS + WIDE_SEEDS

# mismatched counters: the sender at S, the receiver at R
MIS_S = 0x5A5A59  # stamp 0x5A5A5A


def stamp(s):
    """the stamp of frame s of a direction"""
    return 1 + s % M


def one_bit_off(k):
    """a receiver counter whose stamp is MIS_S's stamp with bit k flipped (never 0: a valid stamp)"""
    return (stamp(MIS_S) ^ (1 << k)) - 1


MISMATCHED = [one_bit_off(k) for k in range(24)] + [MIS_S - 1, MIS_S + 1]


class DevPair(C.Structure):  # b200_dev_pair, include/b200_pair.h
    _fields_ = [("table", C.c_void_p), ("seq", C.c_void_p), ("mirrors", C.c_void_p), ("slot", C.c_int32),
                ("wire", C.c_uint32), ("_reserved", C.c_uint64 * 4)]


class PairSeq(C.Structure):  # csrc/b200_dev.cuh: one pair's frame counters
    _fields_ = [("tx", C.c_uint64), ("rx", C.c_uint64)]


def seq_address(handle):
    """device address of the PairSeq of the pair a 64-byte b200_dev_pair handle names"""
    h = DevPair.from_buffer_copy(handle)
    return h.seq + C.sizeof(PairSeq) * h.slot


def fresh_counters(so, *pairs):
    """Drop the model's counter entries of `pairs` so that the next lookup starts them afresh.  The model keys its
    side table by pair address, and a pair destroyed without stamp_forget (the endpoint ops tables forget a pair at
    Init, not at putback) leaves an entry behind that a new pair at the same address would inherit, pad map sized for
    the old ring included."""
    for p in pairs:
        so.S.stamp_forget(p)


def u64(img, pos):
    return int(img[pos:pos + 8].view(np.uint64)[0])


@pytest.fixture(scope="module")
def dev():
    subprocess.check_call(["make", "-s", "-C", NATIVE, "-f", "stamp_arith.mk"])
    L = C.CDLL(os.path.join(NATIVE, "libstamp_arith.so"))
    u = C.c_uint64
    for name, res, args in [
            ("sa_stamp_of", C.c_uint32, [u]), ("sa_frame_header", u, [u, C.c_uint32]),
            ("sa_frame_footer", u, [u, C.c_uint32]), ("sa_frame_present", u, [u, u, C.c_uint32]),
            ("sa_frame_complete", u, [u, u, u, C.c_uint32]), ("sa_sizeof_pairseq", u, []),
            ("sa_offset_pair_seq", u, [C.c_int]), ("sa_offset_pair_seq_table", u, [C.c_int]),
            ("sa_offset_seq_tx", u, []), ("sa_offset_seq_rx", u, []), ("sa_sizeof_dev_pair", u, []),
            ("sa_offset_dev_pair_seq", u, []), ("sa_offset_dev_pair_slot", u, []), ("sa_sizeof_pairdev", u, [])]:
        f = getattr(L, name)
        f.restype, f.argtypes = res, args
    return L


@pytest.fixture(scope="module")
def so():
    return stamp_lib.StampedOracle()


def test_seeding_offsets_match_the_handle(dev):
    """The GPU tests seed a pair's counters at b200_dev_pair.seq + 16 * slot: the handle's layout, PairSeq's size and
    pair_seq()'s addressing as the library compiles them."""
    assert C.sizeof(DevPair) == dev.sa_sizeof_dev_pair() == 64
    assert DevPair.seq.offset == dev.sa_offset_dev_pair_seq() == 8
    assert DevPair.slot.offset == dev.sa_offset_dev_pair_slot() == 24
    assert C.sizeof(PairSeq) == dev.sa_sizeof_pairseq() == 16
    assert (PairSeq.tx.offset, PairSeq.rx.offset) == (dev.sa_offset_seq_tx(), dev.sa_offset_seq_rx()) == (0, 8)
    rows = 8192 * dev.sa_sizeof_pairdev()  # the side array follows kMaxPairs rows of the connection table
    for slot in (0, 1, 2, 31, 4095, 8191):
        assert dev.sa_offset_pair_seq(slot) == 16 * slot
        assert dev.sa_offset_pair_seq_table(slot) == rows + 16 * slot
    h = DevPair(seq=0x7000_0000_0000, slot=37)
    assert seq_address(bytes(h)) == 0x7000_0000_0000 + 16 * 37


def test_stamps_at_every_seed(dev, so):
    """t(s) from the kernels' stamp_of and from the model equals the closed form over the first 1 200 frames after
    every seed (each seed reaches the rollover within them), and past 2^32 and 2^64 - 2^24."""
    S = so.S
    for seed in SEEDS + [0, (1 << 40) + 5, U64 - 1200]:
        for s in range(seed, seed + 1200):
            want = stamp(s)
            assert dev.sa_stamp_of(s) == want, (seed, s)
            assert S.stamp_of(s) == want, (seed, s)
            assert dev.sa_frame_header(24, dev.sa_stamp_of(s)) == S.stamp_header(24, s) == 24 | want << 40, s
    assert [stamp(s) for s in (M - 2, M - 1, M, M + 1)] == [M - 1, M, 1, 2]
    assert stamp(1 << 32) == 257 and dev.sa_stamp_of(1 << 32) == 257 and dev.sa_stamp_of((1 << 32) - 1) == 256
    assert dev.sa_stamp_of(U64) == stamp(U64)


def test_present_and_complete_use_all_24_bits_and_the_length_bounds(dev):
    cap = 1 << 16
    for s in SEEDS + [MIS_S]:
        st = stamp(s)
        for p in (1, 8, 9, 100, cap - 24):
            hdr = dev.sa_frame_header(p, st)
            assert hdr == p | st << 40 and dev.sa_frame_footer(hdr, st) == ~hdr & U64
            assert dev.sa_frame_present(hdr, cap, st) == p
            assert dev.sa_frame_complete(hdr, ~hdr & U64, cap, st) == p
            assert dev.sa_frame_complete(hdr, ~hdr & U64 ^ 1, cap, st) == 0
            assert dev.sa_frame_complete(hdr, U64, cap, st) == 0          # a reference-format footer
            for k in range(24):
                other = st ^ (1 << k)
                if other == 0:
                    continue
                # a header one stamp bit away, read with either stamp as the expected one
                assert dev.sa_frame_present(p | other << 40, cap, st) == 0, (s, k)
                assert dev.sa_frame_present(hdr, cap, other) == 0, (s, k)
                assert dev.sa_frame_complete(p | other << 40, ~(p | other << 40) & U64, cap, st) == 0, (s, k)
            for d in (-1, 1):  # one frame away
                other = stamp(s + d)
                assert dev.sa_frame_present(p | other << 40, cap, st) == 0
        for p, want in ((0, 0), (1, 1), (cap - 24, cap - 24), (cap - 23, 0), (LEN_MASK, 0)):
            hdr = dev.sa_frame_header(p, st)
            assert dev.sa_frame_present(hdr, cap, st) == want, (s, p)
            assert dev.sa_frame_complete(hdr, ~hdr & U64, cap, st) == want, (s, p)
    # the reference format (st = 0) is untouched: header = p, footer = ~0
    assert dev.sa_frame_present(100, cap, 0) == 100 and dev.sa_frame_complete(100, U64, cap, 0) == 100
    assert dev.sa_frame_present(100 | 5 << 40, cap, 0) == 0


def _seeded(so, cap, s_tx, s_rx):
    tx, rx = so.pair_pair(cap)
    fresh_counters(so, tx, rx)
    so.S.stamp_seq_set(tx, s_tx, 0)
    so.S.stamp_seq_set(rx, 0, s_rx)
    return tx, rx


@pytest.mark.parametrize("coalesced", [False, True])
@pytest.mark.parametrize("seed", SEEDS)
def test_model_images_at_every_seed(seed, coalesced):
    """1 200 8-byte slices in one send_all: every header and footer word of the ring equals the closed form, the
    receiver reads all of them and ends at seed + frames."""
    so = stamp_lib.StampedOracle(coalesced=coalesced)
    cap = 1 << 16
    tx, rx = _seeded(so, cap, seed, seed)
    try:
        bufs = trace.make_bufs([8] * 1200, 3)
        n, calls = so.send_all(tx, bufs, 0)
        assert n == 9600 and calls == (2 if coalesced else 40)  # 1024 slices / 30 frames per call
        img = so.ring_image(rx)
        at, i, tail = 0, 0, so.state(tx)["remote_tail"]
        while at != tail:  # walk the frames by their length fields
            p = u64(img, at) & LEN_MASK
            hdr = p | stamp(seed + i) << 40
            assert 0 < p <= 8192 and u64(img, at) == hdr, (seed, i)
            assert u64(img, at + 8 + (p + 7) // 8 * 8) == ~hdr & U64, (seed, i)
            at, i = at + 16 + (p + 7) // 8 * 8, i + 1
        assert i == (2 if coalesced else 1200) and so.S.stamp_seq_tx(tx) == seed + i
        out, _ = so.recv_drain(rx, 1 << 20)
        assert np.array_equal(out, np.concatenate(bufs))
        assert so.S.stamp_seq_rx(rx) == seed + i
        assert so.has_message(rx) == 0 and so.readable(rx) == 0
    finally:
        so.destroy(tx)
        so.destroy(rx)


@pytest.mark.parametrize("r", MISMATCHED + [MIS_S + M, MIS_S + 2 * M])
def test_model_reads_only_the_expected_stamp(so, r):
    """Sender at S, receiver at R: only R = S + kM (same stamp, other counter) reads; a stamp one bit or one frame
    away reads nothing, and the frames stay in the ring."""
    cap = 4096
    tx, rx = _seeded(so, cap, MIS_S, r)
    try:
        bufs = trace.make_bufs([9, 700, 9, 40], 5)
        assert so.send(tx, bufs) == 758
        img = so.ring_image(rx)
        assert u64(img, 0) == 9 | stamp(MIS_S) << 40
        same = stamp(r) == stamp(MIS_S)
        assert same == (r >= MIS_S + M)
        assert so.has_message(rx) == int(same) and so.readable(rx) == (9 if same else 0)
        out, calls = so.recv_drain(rx, 1 << 16)
        if same:
            assert np.array_equal(out, np.concatenate(bufs)) and calls == 4
            assert so.S.stamp_seq_rx(rx) == r + 4
        else:
            assert out.size == 0 and calls == 0 and so.S.stamp_seq_rx(rx) == r
            assert so.state(rx)["head"] == 0 and np.array_equal(so.ring_image(rx), img)
    finally:
        so.destroy(tx)
        so.destroy(rx)
