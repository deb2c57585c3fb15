"""CPU: the stamped ring frame model (B200_RING_STAMPED=1, DESIGN.md §2; tests/native/stamp_oracle.c).

The mode may change nothing but the ring image: every golden trace replayed through the model gives the golden
return values, partial_write, cursors and delivered bytes.  Hand-checked images pin the wire format; drained rings
full of old frames and payloads that look like reference-format frames pin the readiness rule."""
import json
import os

import numpy as np
import pytest

import stamp_lib
import trace

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def so():
    return stamp_lib.StampedOracle()


def _golden(name):
    with open(os.path.join(HERE, "golden", name)) as f:
        return json.load(f)


@pytest.mark.parametrize("fixture", ["traces.json", "traces_full.json"])
def test_golden_traces_replay_identically(so, fixture):
    """Everything but the ring image: returns, calls, partial_write, cursors, readiness, delivered SHA-1."""
    data = _golden(fixture)
    for name, t in sorted(data["traces"].items()):
        cap, ops = t["cap"], [tuple(o) for o in t["ops"]]
        got = trace.run_trace(so, cap, ops, data["max_sge"], ring_images=False)
        want = t["records"]
        assert len(got) == len(want), name
        for i, (g, w) in enumerate(zip(got, want)):
            for k in w:
                if k == "ring":
                    continue
                assert g[k] == w[k], "%s op %d %s: %s != %s" % (name, i, k, g[k], w[k])


def _u64(img, pos):
    return int(img[pos:pos + 8].view(np.uint64)[0])


def test_hand_checked_images_wrap_and_stamp_rollover(so):
    """64-byte ring, the sender's counter two frames before 2^24 - 1: stamps 2^24 - 2, 2^24 - 1, then 1."""
    cap = 64
    tx, rx = so.pair_pair(cap)
    try:
        M = (1 << 24) - 1
        so.S.stamp_seq_set(tx, M - 2, 0)
        so.S.stamp_seq_set(rx, 0, M - 2)
        assert so.send(tx, [np.arange(1, 6, dtype=np.uint8)]) == 5           # frame at 0: 24 bytes
        img = so.ring_image(rx)
        h = 5 | (M - 1) << 40
        assert _u64(img, 0) == h and _u64(img, 16) == (~h) & (2**64 - 1)
        assert bytes(img[8:13]) == bytes([1, 2, 3, 4, 5])
        assert so.recv(rx, 100).tolist() == [1, 2, 3, 4, 5]
        assert so.send(tx, [np.full(8, 7, np.uint8)]) == 8                   # frame at 24
        h2 = 8 | M << 40
        img = so.ring_image(rx)
        assert _u64(img, 24) == h2 and _u64(img, 40) == (~h2) & (2**64 - 1)
        assert _u64(img, 0) == h, "Recv stores nothing into the ring"
        assert so.recv(rx, 100).tolist() == [7] * 8
        assert so.send(tx, [np.full(3, 9, np.uint8)]) == 3                   # frame at 48: its footer wraps to 0
        h3 = 3 | 1 << 40                                                     # s = 2^24 - 1 -> t = 1
        img = so.ring_image(rx)
        assert _u64(img, 48) == h3 and _u64(img, 0) == (~h3) & (2**64 - 1)
        assert bytes(img[56:59]) == bytes([9, 9, 9])
        assert so.readable(rx) == 3 and so.has_message(rx) == 1
        assert so.recv(rx, 100).tolist() == [9] * 3
        assert so.has_message(rx) == 0 and so.readable(rx) == 0
    finally:
        so.destroy(tx)
        so.destroy(rx)


def stale_frame_at_head(img, head, cap):
    """The word at `head` is a complete frame of an earlier lap: a valid length and footer == ~header (stamped),
    or a reference-format frame (footer == ~0).  Returns "stamped", "reference" or None."""
    hdr = _u64(img, head)
    p = hdr & ((1 << 40) - 1)
    if p == 0 or p > cap - 24:
        return None
    foot = _u64(img, (head + 8 + (p + 7) // 8 * 8) % cap)
    if foot == (~hdr) & (2**64 - 1):
        return "stamped"
    return "reference" if hdr == p and foot == 2**64 - 1 else None


# message shapes whose ring bytes divide the ring, so that every drain leaves the head on last lap's frame
STALE_SHAPES = {False: [9, 2000], True: [9, 2023]}  # per-slice: 32 + 2016 B; coalesced: one frame of 2048 B


@pytest.mark.parametrize("coalesced", [False, True])
def test_drained_ring_full_of_old_frames_reads_empty(coalesced):
    so = stamp_lib.StampedOracle(coalesced=coalesced)
    cap = 1 << 16
    tx, rx = so.pair_pair(cap)
    try:
        lens = STALE_SHAPES[coalesced]
        sent = got = 0
        for k in range(100):                                                 # > 3 laps
            bufs = trace.make_bufs(lens, k)
            n, _ = so.send_all(tx, bufs, 0)
            out, _ = so.recv_drain(rx, 1 << 20)
            assert out.size == n == sum(lens)
            assert np.array_equal(out, np.concatenate(bufs))
            sent, got = sent + n, got + out.size
            img = so.ring_image(rx)
            if k >= 32:                                                      # from the second lap on
                assert stale_frame_at_head(img, so.state(rx)["head"], cap) == "stamped", k
            assert so.has_message(rx) == 0 and so.readable(rx) == 0
            assert so.recv(rx, 1 << 20).size == 0
        assert sent == got > 3 * cap
    finally:
        so.destroy(tx)
        so.destroy(rx)


def test_reference_format_payloads_are_not_frames(so):
    """Last lap's payload holds a reference-format frame (header 8, footer ~0) exactly where a later head lands."""
    cap = 4096
    tx, rx = so.pair_pair(cap)
    try:
        body = np.zeros(2024, np.uint8)                                     # E = 2040; payload at ring 8
        body[0:8] = np.frombuffer(np.uint64(8).tobytes(), np.uint8)         # ring 8: header 8
        body[16:24] = 0xFF                                                  # ring 24: footer ~0
        for _ in range(2):                                                  # frames at 0 and 2040
            assert so.send(tx, [body]) == 2024 and so.recv(rx, 1 << 20).size == 2024
        assert so.send(tx, [np.full(8, 3, np.uint8)]) == 8                   # frame at 4080, E = 24: wraps
        assert so.recv(rx, 1 << 20).tolist() == [3] * 8
        head = so.state(rx)["head"]
        assert head == 8 and stale_frame_at_head(so.ring_image(rx), head, cap) == "reference"
        assert so.has_message(rx) == 0 and so.readable(rx) == 0 and so.recv(rx, 100).size == 0
    finally:
        so.destroy(tx)
        so.destroy(rx)


def test_frame_hbm_bytes_stamped():
    """DESIGN.md §4: one 4 MiB chttp2-shaped message, k_recv moves 12,609,918 B by default and 8,403,270 B stamped."""
    import sys
    sys.path.insert(0, os.path.dirname(HERE))
    import __graft_entry__ as ge
    pkg = ge.load_package()
    lens = pkg.chttp2_slice_lens(4 << 20)
    tx0, rx0 = pkg.frame_hbm_bytes(lens)
    tx1, rx1 = pkg.frame_hbm_bytes(lens, stamped=True)
    assert rx0 == 12609918 and rx1 == 8403270 and tx1 == tx0
    assert tx0 + rx0 == 21013188 and tx1 + rx1 == 16806540


# ---- the product's endpoint state machine and poll loop over the stamped model (test_endpoint_cpu.py shapes)

@pytest.fixture(scope="module")
def drv(pkg, so):
    import endpoint_lib
    D, _ = endpoint_lib.load(pkg, need_oracle=True)
    return D, so.S


@pytest.mark.parametrize("table", ["single", "batch"])
def test_endpoint_conformance_and_echo_over_stamped_model(drv, table):
    import ctypes as C
    D, L = drv
    ops = L.stamp_pair_ops() if table == "single" else L.stamp_pair_ops_batch()
    for ring in (4096, 65536):
        L.stamp_ops_config(ring)
        assert D.drv_read_and_write(ops, 2_000_000, 100_000, 8192, 0, 50, 0, None) == 0
    L.stamp_ops_config(65536)
    assert D.drv_read_and_write(ops, 60_000, 10_000, 1, 0, 50, 0, None) == 0
    L.stamp_ops_config(1024)
    i = 1
    while i < 1000:
        assert D.drv_read_and_write(ops, 40320, i, i, 0, 50, 0, None) == 0, i
        i = max(i + 1, i * 5 // 4)
    L.stamp_ops_config(4096)
    assert D.drv_read_and_write(ops, 300_000, 300_000, 100_000, 0, 50, 0, None) == 0
    L.stamp_ops_config(65536)
    nbytes = C.c_uint64(0)
    assert D.drv_echo(ops, 40, 300_000, 12345, 50, 0, 0, C.byref(nbytes)) == 0 and nbytes.value > 0
