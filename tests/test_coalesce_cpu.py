"""CPU: the coalesced Send model (B200_SEND_COALESCE=1, DESIGN.md §2; tests/native/coalesce_oracle.c) against the
specification on hand-checked cases, against the per-slice oracle on the delivered stream, through the
reference's own receiver, and under the product's endpoint host logic."""
import ctypes as C

import numpy as np
import pytest

import coalesce_lib
import endpoint_lib
import orlib
import trace


@pytest.fixture(scope="module")
def co():
    return coalesce_lib.CoalescedOracle()


def _u64(img, pos):
    return int(img[pos:pos + 8].view(np.uint64)[0])


def _frame(img, cap, pos):
    """(payload bytes, encoded size) of the complete frame at ring offset pos (wraps)."""
    rot = np.roll(img, -pos)
    hdr = _u64(rot, 0)
    assert 0 < hdr <= cap - 24
    assert _u64(rot, 8 + trace.up8(hdr)) == 0xFFFFFFFFFFFFFFFF
    return rot[8:8 + hdr].copy(), 16 + trace.up8(hdr)


def _spec(cap, staging, rh, rt, lens, bidx):
    """The pseudo-code of DESIGN.md §2, straight: bytes of the look window, staging and credit limits."""
    cws = lambda s: 0 if s <= 24 else (s - 24) // 8 * 8
    free = cap - ((rt + cap - rh) % cap)
    look = sum(lens[:1024]) - bidx
    return min(look, cws(staging), cws(free))


def test_cut_at_a_slice_edge_and_in_the_middle(co):
    cap = 4096                                  # staging C/2 = 2048: CWS = 2024 = C/2 - 24
    tx, rx = co.pair_pair(cap)
    bufs = trace.make_bufs([1000, 1024, 50], 1)
    assert _spec(cap, cap // 2, 0, 0, [1000, 1024, 50], 0) == 2024
    assert co.send(tx, bufs) == 2024            # ends exactly at the end of slice 1
    st = co.state(tx)
    assert st["remote_tail"] == 2040 and st["partial_write"] == 1
    img = co.ring_image(rx)
    pay, enc = _frame(img, cap, 0)
    assert enc == 2040 and np.array_equal(pay, np.concatenate(bufs)[:2024])
    assert not img[enc:].any()                  # one frame, nothing behind it
    out, calls = co.recv_drain(rx, 1 << 16)
    assert calls == 1 and np.array_equal(out, pay)
    co.destroy(tx), co.destroy(rx)
    cap = 8192                                  # CWS(C/2) = 4072: the first call ends inside slice 1 at byte 1072
    tx, rx = co.pair_pair(cap)
    bufs = trace.make_bufs([3000, 1500], 2)
    assert co.send(tx, bufs) == 4072
    assert co.send(tx, [bufs[1]], 1072) == 428  # the rdma_flush cursor: slice 1, byte 1072
    got, calls = co.recv_drain(rx, 1 << 16)
    assert calls == 2 and np.array_equal(got, np.concatenate(bufs))
    co.destroy(tx), co.destroy(rx)
    tx, rx = co.pair_pair(cap)
    assert co.send_all(tx, bufs) == (4500, 2)
    co.destroy(tx), co.destroy(rx)


def test_byte_idx_and_zero_length_slices(co):
    tx, rx = co.pair_pair(4096)
    b = trace.make_bufs([100, 50], 3)
    assert co.send(tx, b, 30) == 120
    assert np.array_equal(co.recv(rx, 4096), np.concatenate([b[0][30:], b[1]]))
    # zero-length slices contribute nothing and do not end the call (the per-slice Send stops there)
    z = trace.make_bufs([5, 0, 7, 0], 4)
    assert co.send(tx, z) == 12 and co.state(tx)["partial_write"] == 0
    assert np.array_equal(co.recv(rx, 4096), np.concatenate(z))
    o = orlib.Oracle()
    ptx, prx = o.pair_pair(4096)
    assert o.send(ptx, z) == 5
    for p in (tx, rx, ptx, prx):
        o.destroy(p)


def test_look_window_is_1024_slices(co):
    tx, rx = co.pair_pair(65536)
    bufs = trace.make_bufs([1] * 1100, 5)
    assert co.send(tx, bufs) == 1024 and co.state(tx)["partial_write"] == 1
    out = co.recv(rx, 1 << 16)
    assert out.size == 1024                     # one frame, one Recv
    n, calls = co.send_all(tx, bufs[1024:])
    assert (n, calls) == (76, 1)
    co.destroy(tx), co.destroy(rx)
    tx, rx = co.pair_pair(65536)
    n, calls = co.send_all(tx, bufs)
    assert (n, calls) == (1100, 2)
    out, rcalls = co.recv_drain(rx, 1 << 16)
    assert rcalls == 2 and np.array_equal(out, np.concatenate(bufs))
    co.destroy(tx), co.destroy(rx)


def test_credit_exhaustion(co):
    cap = 1024
    tx, rx = co.pair_pair(cap)
    big = trace.make_bufs([9, 2000], 6)
    assert co.send(tx, big) == 488              # CWS(C/2) = 488
    assert co.send(tx, big) == 488              # free 520: CWS 496, staging still the limit
    assert co.send(tx, big) == 0                # free 16: nothing fits
    assert co.has_pending_writes(tx) == 1
    assert co.writable(tx) == 0
    out, calls = co.recv_drain(rx, 4096)        # credit comes back at C/2 retired
    assert out.size == 976 and calls == 2
    assert co.send(tx, big) == 488
    co.destroy(tx), co.destroy(rx)


def test_wrap_at_every_8_byte_offset(co):
    cap = 256
    tx, rx = co.pair_pair(cap)
    seen = set()
    for k in range(40):                         # 8 payload bytes: E = 24 per frame, gcd(24, 256) = 8
        lens = [1, 2, 0, 5] if k % 2 else [3, 4, 1]
        bufs = trace.make_bufs(lens, 100 + k)
        rt = co.state(tx)["remote_tail"]
        seen.add(rt)
        p = co.send(tx, bufs)
        assert p == sum(lens)
        img = co.ring_image(rx)
        pay, enc = _frame(img, cap, rt)
        assert np.array_equal(pay, np.concatenate(bufs)) and co.state(tx)["remote_tail"] == (rt + enc) % cap
        out = co.recv(rx, 4096)
        assert np.array_equal(out, pay)
        assert not co.ring_image(rx).any()      # clear-on-read leaves nothing behind, wrapped or not
    assert seen == set(range(0, cap, 8))
    co.destroy(tx), co.destroy(rx)


def _random_lens(rng, cap):
    """No zero-length slices: the per-slice rdma_flush loop never gets past one (pair.cc:683-685)."""
    style = rng.integers(0, 4)
    n = int(rng.integers(1, 1500 if style == 3 else 60))
    if style == 0:
        return [int(x) for x in rng.integers(1, 64, n)]
    if style == 1:
        return [9 if i % 2 == 0 else int(rng.integers(1, min(16385, cap))) for i in range(n)]
    if style == 2:
        return [int(x) for x in rng.integers(1, 2 * cap, max(1, n // 8))]
    return [int(x) for x in rng.integers(1, 4, n)]


@pytest.mark.parametrize("seed", range(12))
def test_delivered_stream_equals_per_slice(co, seed):
    rng = np.random.default_rng(500 + seed)
    cap = [256, 1024, 4096, 65536][seed % 4]
    o = orlib.Oracle()
    for k in range(4):
        lens = _random_lens(rng, cap)
        op = [("stream", lens, seed * 10 + k, int(rng.integers(1, 3 * cap)))]
        want = trace.run_trace(o, cap, op)[0]
        got = trace.run_trace(co, cap, op)[0]
        assert got["intact"] and want["intact"]
        assert got["ret"] == want["ret"] and got["sha"] == want["sha"]
        assert got["ring"] == trace.sha(np.zeros(cap, np.uint8)) or got["has_message"] == 0


def test_chttp2_message_counts(co):
    """Per 4 MiB chttp2-shaped message (514 slices): 1 frame, 1 Send, 1 Recv and 4,196,640 ring bytes in
    coalesced mode, against 514 frames, 18 Sends, 514 Recvs and 4,206,648 ring bytes per slice."""
    lens = coalesce_lib.chttp2_lens(4 << 20)
    assert len(lens) == 514
    cap = 16 << 20
    o = orlib.Oracle()
    for eng, frames, sends, ring_bytes in [(o, 514, 18, 4206648), (co, 1, 1, 4196640)]:
        tx, rx = eng.pair_pair(cap)
        bufs = trace.make_bufs(lens, 9)
        n, calls = eng.send_all(tx, bufs)
        assert n == sum(lens) and calls == sends
        assert eng.state(tx)["remote_tail"] == ring_bytes
        out, rcalls = eng.recv_drain(rx, 8 << 20)
        assert rcalls == frames and np.array_equal(out, np.concatenate(bufs))
        eng.destroy(tx), eng.destroy(rx)


@pytest.mark.skipif(not orlib.ref_available(), reason="needs the reference build (GRPC_RDMA_REFERENCE)")
@pytest.mark.parametrize("cap", [1024, 65536])
def test_reference_receiver_reads_coalesced_frames(co, cap):
    """Frames written by the coalesced model drain through the reference's own RingBufferPollable::Read: the
    same bytes as the oracle's receiver, and an all-zero ring after every drain (wraps included)."""
    R = orlib.Ref()
    buf = np.zeros(cap, np.uint8)
    rr = R.L.ref_ring_create(buf.ctypes.data, cap)
    tx, rx = co.pair_pair(cap)
    rng = np.random.default_rng(cap)
    try:
        for k in range(30):
            lens = _random_lens(rng, cap)
            bufs = trace.make_bufs(lens, 700 + k)
            n, _ = co.send_all(tx, bufs)
            buf[:] = co.ring_image(rx)
            want, _ = co.recv_drain(rx, 1 << 20)
            assert want.size == n
            got = np.zeros(max(n, 1), np.uint8)
            off, internal = 0, C.c_uint64(0)
            while off < n:
                m = R.L.ref_ring_read(rr, got[off:].ctypes.data, n - off, C.byref(internal))
                assert m > 0
                off += m
            assert np.array_equal(got[:n], want)
            assert not buf.any() and not co.ring_image(rx).any()
    finally:
        R.L.ref_ring_destroy(rr)
        co.destroy(tx), co.destroy(rx)


# ---- the product's endpoint state machine and poll loop over the coalesced model (test_endpoint_cpu.py shapes)

@pytest.fixture(scope="module")
def drv(pkg, co):
    D, _ = endpoint_lib.load(pkg, need_oracle=True)
    return D, co.C


@pytest.mark.parametrize("table", ["single", "batch"])
def test_endpoint_conformance_with_coalesced_send(drv, table):
    D, L = drv
    ops = L.coalesce_pair_ops() if table == "single" else L.coalesce_pair_ops_batch()
    for ring in (4096, 65536):
        L.coalesce_ops_config(ring)
        assert D.drv_read_and_write(ops, 2_000_000, 100_000, 8192, 0, 50, 0, None) == 0
    L.coalesce_ops_config(65536)
    assert D.drv_read_and_write(ops, 60_000, 10_000, 1, 0, 50, 0, None) == 0
    L.coalesce_ops_config(1024)
    i = 1
    while i < 1000:
        assert D.drv_read_and_write(ops, 40320, i, i, 0, 50, 0, None) == 0, i
        i = max(i + 1, i * 5 // 4)
    L.coalesce_ops_config(4096)
    assert D.drv_read_and_write(ops, 300_000, 300_000, 100_000, 0, 50, 0, None) == 0
    L.coalesce_ops_config(65536)
    nbytes = C.c_uint64(0)
    assert D.drv_echo(ops, 40, 300_000, 12345, 50, 0, 0, C.byref(nbytes)) == 0 and nbytes.value > 0
