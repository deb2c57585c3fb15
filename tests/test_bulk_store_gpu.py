"""GPU: the movers' bulk-store write path at its edges, against the oracle.

The movers realign each 4 KiB item in shared memory to its destination's phase mod 16 and write the aligned
interior with one bulk store (k_recv's clear-on-read with bulk stores from a zero block); the <16-byte edges are
byte stores.  These traces force every destination phase, items that wrap at the ring end, frames one byte off a
multiple of 16, and a credit point while the sender runs concurrently on another stream.
"""
import ctypes as C

import numpy as np
import pytest

import trace
from gpu_engine import GpuEngine

pytestmark = pytest.mark.gpu


def _compare(got, want, label):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, "%s: op %d (%s)\n got  %s\n want %s" % (label, i, w["op"], g, w)


@pytest.mark.parametrize("phase", range(16))
def test_every_destination_phase(gpu, oracle, phase):
    """Send: slices at every source phase into ring payloads at 8 and 0 mod 16 (a 1-byte or 9-byte frame first).
    Recv: destinations at every phase, with partial reads that move the next item's phase as well."""
    cap = 65536
    lens = [9, 12000 + phase, 37, 4096 * 3 + 16 - phase]
    ops = [("send_all", [1 + 8 * (phase & 1)], 10 + phase, 0), ("recv_drain", 64),
           ("send_all", lens, 20 + phase, phase % 9), ("recv", 5000 + phase), ("recv_drain", 1 << 16),
           ("send_all", lens[::-1], 30 + phase, 0), ("recv", 4096 + 7), ("recv", 3 + phase), ("recv_drain", 1 << 16)]
    want = trace.run_trace(oracle, cap, ops)
    got = trace.run_trace(GpuEngine(gpu, "device", phase), cap, ops)
    _compare(got, want, "phase %d" % phase)


@pytest.mark.parametrize("shift", [0, 3, 8, 13])
def test_wrap_inside_an_item(gpu, oracle, shift):
    """A frame that crosses the ring end in the middle of a 4 KiB item: the send side writes both parts from one
    stage, the receive side loads both parts into one stage and clears both."""
    cap = 16384
    ops = [("send_all", [cap - 6000 + 8 * shift], 40 + shift, 0), ("recv_drain", cap),
           ("send_all", [9, 9000 + shift, 9, 2500], 50 + shift, 0), ("recv", 4100 + shift), ("recv_drain", cap)]
    want = trace.run_trace(oracle, cap, ops)
    got = trace.run_trace(GpuEngine(gpu, "device", shift), cap, ops)
    _compare(got, want, "wrap shift %d" % shift)


@pytest.mark.parametrize("mis", [0, 5, 8])
def test_frames_one_byte_off_a_multiple_of_16(gpu, oracle, mis):
    cap = 1 << 17
    lens = [4096 * k + d for k in (1, 2, 5) for d in (-1, 1, 0)] + [33, 31, 47, 49]
    ops = [("send_all", lens, 60 + mis, 0), ("recv", 4095), ("recv", 8193), ("recv_drain", cap),
           ("send_all", lens[::-1], 61 + mis, 1), ("recv_drain", cap)]
    want = trace.run_trace(oracle, cap, ops)
    got = trace.run_trace(GpuEngine(gpu, "device", mis), cap, ops)
    _compare(got, want, "frames off by one, mis %d" % mis)


def test_credit_mid_op_with_concurrent_sender(gpu):
    """k_send and k_recv of one connection on two streams at once (B200_BATCH_CONCURRENT), a 64 KiB ring and
    4 MiB of chttp2-shaped slices: the receiver returns credit in the middle of its op while the sender may be
    writing into the space it just freed.  The zeros must be complete before the credit is visible, or the
    sender's new frames would be cleared under it: the delivered stream must be intact and the ring all zero."""
    import torch
    pkg, L = gpu, gpu.lib()
    cap = 1 << 16
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", cap)
    pkg.config_set("GRPC_RDMA_MAX_SGE", 30)
    lens = pkg.chttp2_slice_lens(4 << 20)
    total = sum(lens)
    tx, rx = pkg.connected_pair("bulk-cc-tx", "bulk-cc-rx")
    rng = np.random.default_rng(5)
    host = rng.integers(0, 256, total, dtype=np.uint8)
    src = L.b200_mem_alloc_device(total + 16)
    dst = L.b200_mem_alloc_device(total + 16)
    assert src and dst
    assert L.b200_memcpy(src + 3, host.ctypes.data, total, 0, None) == 0
    L.b200_stream_sync(None)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    h1, h2 = C.c_void_p(s1.cuda_stream), C.c_void_p(s2.cuda_stream)
    flags = pkg.UNTIL_BLOCKED | 0x8  # B200_BATCH_CONCURRENT
    sent = got = idx = bidx = rounds = 0
    while got < total and rounds < 5000:
        rounds += 1
        bs = None
        if idx < len(lens):
            sl = pkg.make_slices([(src + 3 + int(offs[i]), lens[i]) for i in range(idx, len(lens))])
            bs = pkg.Batch("send", [(tx, sl, len(lens) - idx, bidx)], flags)
        br = pkg.Batch("recv", [(rx, dst + 5 + got, total - got)], flags)
        if bs:
            bs.launch(h1)
        br.launch(h2)
        torch.cuda.synchronize()
        if bs:
            n = bs.results(h1)[0]
            bs.destroy()
            sent += n
            pos = int(offs[idx]) + bidx + n
            idx = int(np.searchsorted(offs, pos, side="right")) - 1
            bidx = pos - int(offs[idx])
        got += br.results(h2)[0]
        br.destroy()
    assert got == sent == total, (got, sent, total, rounds)
    out = np.zeros(total, dtype=np.uint8)
    assert L.b200_memcpy(out.ctypes.data, dst + 5, total, 1, None) == 0
    L.b200_stream_sync(None)
    assert np.array_equal(out, host), "delivered bytes differ"
    assert not rx.ring_image().any(), "ring must read as all zero after a full drain"
    L.b200_mem_free_device(src)
    L.b200_mem_free_device(dst)
    for p in (tx, rx):
        p.disconnect()
        p.putback()
