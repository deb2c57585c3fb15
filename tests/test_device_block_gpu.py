"""GPU: block-level device Send / Recv (include/b200_device_block.cuh) driven from a user kernel's CTAs
(tests/native/device_block.cu).

Bar of test_gpu_parity.py: every return value and `calls`, partial_write, both pairs' cursors and readiness answers,
the SHA-1 of the delivered bytes and the receiver's ring image with pads masked -- here with every op of a claimed end
run by a CTA (single calls as B200_BATCH_ONE_CALL, the rdma_flush / rdma_do_read loops as one B200_BATCH_UNTIL_BLOCKED
call), against the golden records and the CPU models (reference, coalesced, stamped).  Then warp and block calls on one
pair, one end on the host, sender and receiver CTAs side by side, the benchmark's shape, the refusals and the
CUDA-IPC wire."""
import ctypes as C
import json
import os
import time

import numpy as np
import pytest

import coalesce_lib
import device_block_lib as bl
import device_lib
import stamp_lib
import test_coalesce_gpu
import test_gpu_parity
import test_stamp_gpu
import trace
from device_block_lib import BlockEngine

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "traces.json")))
_compare = test_gpu_parity._compare


def _ops(raw):
    return [tuple(o) for o in raw]


@pytest.fixture(scope="module")
def co():
    return coalesce_lib.CoalescedOracle()


@pytest.fixture(scope="module")
def so():
    return stamp_lib.StampedOracle()


@pytest.fixture(scope="module")
def soc():
    return stamp_lib.StampedOracle(coalesced=True)


@pytest.fixture
def svc(gpu):
    bl.Runner(gpu)  # the drivers' kernels are loaded before the resident kernels start
    device_lib.Runner(gpu)
    L = gpu.lib()
    assert L.b200_service_start(4) == 0, gpu.last_error()
    yield gpu
    L.b200_service_stop()


# ---- both ends block-driven, against the golden records and the models

@pytest.mark.parametrize("name", sorted(GOLDEN["traces"]))
@pytest.mark.parametrize("mem,mis", [("device", 0), ("device", 5), ("pinned", 9)])
def test_golden_traces_block_driven(gpu, name, mem, mis):
    t = GOLDEN["traces"][name]
    recs = trace.run_trace(BlockEngine(gpu, mem, mis), t["cap"], _ops(t["ops"]), GOLDEN["max_sge"])
    _compare(recs, t["records"], "golden %s [%s+%d]" % (name, mem, mis))


def test_golden_full_size_block_driven(gpu):
    full = json.load(open(os.path.join(HERE, "golden", "traces_full.json")))
    for name, t in sorted(full["traces"].items()):
        recs = trace.run_trace(BlockEngine(gpu, "device", 3), t["cap"], _ops(t["ops"]), full["max_sge"],
                               ring_images=False)
        _compare(recs, t["records"], "golden full %s" % name)


@pytest.mark.parametrize("seed", range(10))
def test_random_traces_vs_oracle(gpu, oracle, seed):
    rng = np.random.default_rng(5400 + seed)
    cap = [64, 1024, 2048, 4096, 65536][seed % 5]
    ops = test_gpu_parity._random_ops(rng, cap, 80)
    want = trace.run_trace(oracle, cap, ops)
    mem, mis = [("device", 0), ("device", 7), ("pinned", 13)][seed % 3]
    got = trace.run_trace(BlockEngine(gpu, mem, mis), cap, ops)
    _compare(got, want, "random seed %d cap %d [%s+%d]" % (seed, cap, mem, mis))


@pytest.mark.parametrize("max_sge", [1, 4, 32])
def test_other_max_sge(gpu, oracle, max_sge):
    ops = [("send", [7] * 50, 1, 0), ("send_all", [9, 100] * 30, 2, 3), ("recv_drain", 1 << 16),
           ("send_all", [9, 100] * 30, 3, 0), ("recv_drain", 1 << 16), ("send", [5] * 40, 4, 2), ("recv", 3)]
    want = trace.run_trace(oracle, 16384, ops, max_sge)
    got = trace.run_trace(BlockEngine(gpu, "device", 1), 16384, ops, max_sge)
    _compare(got, want, "max_sge %d" % max_sge)


@pytest.mark.parametrize("seed", range(6))
def test_coalesced_vs_model(gpu, co, seed):
    rng = np.random.default_rng(5500 + seed)
    cap = [64, 1024, 4096, 65536, 2048, 1 << 20][seed]
    ops = test_coalesce_gpu._random_ops(rng, cap, 60)
    want = trace.run_trace(co, cap, ops)
    mem, mis = [("device", 0), ("device", 5), ("pinned", 9)][seed % 3]
    got = trace.run_trace(BlockEngine(gpu, mem, mis, config={"B200_SEND_COALESCE": 1}), cap, ops)
    _compare(got, want, "coalesced seed %d cap %d" % (seed, cap))


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("coalesced", [False, True])
def test_stamped_vs_model(gpu, so, soc, seed, coalesced):
    rng = np.random.default_rng(5600 + seed)
    cap = [64, 1024, 4096, 65536][seed % 4]
    mem, mis = [("device", 0), ("device", 3), ("pinned", 11)][seed % 3]
    eng = BlockEngine(gpu, mem, mis, config={"B200_RING_STAMPED": 1, "B200_SEND_COALESCE": int(coalesced)})
    test_stamp_gpu._replay(eng, soc if coalesced else so, cap, test_stamp_gpu._random_ops(rng, cap, 80))


# ---- warp and block calls on one pair

@pytest.mark.parametrize("seed", range(4))
def test_warp_and_block_calls_interleaved(gpu, oracle, seed):
    """every 2nd or 3rd single call of each end is a warp call from warp 0 of the CTA, the others block calls"""
    rng = np.random.default_rng(5700 + seed)
    cap = [1024, 4096, 65536, 2048][seed]
    ops = test_gpu_parity._random_ops(rng, cap, 80)
    got = trace.run_trace(BlockEngine(gpu, "device", seed, warp_every=2 + seed % 2), cap, ops)
    _compare(got, trace.run_trace(oracle, cap, ops), "warp + block seed %d cap %d" % (seed, cap))


# ---- one end on the device, the other on the host

@pytest.mark.parametrize("drive", [("tx",), ("rx",)])
@pytest.mark.parametrize("name", sorted(GOLDEN["traces"]))
def test_mixed_drivers_golden(gpu, drive, name):
    t = GOLDEN["traces"][name]
    recs = trace.run_trace(BlockEngine(gpu, "device", 3, drive=drive), t["cap"], _ops(t["ops"]), GOLDEN["max_sge"])
    _compare(recs, t["records"], "golden %s driven by %s" % (name, drive))


@pytest.mark.parametrize("drive", [("tx",), ("rx",), ("tx", "rx")])
def test_mixed_drivers_under_the_service(svc, oracle, drive):
    """Host ends go through the owner warps and the pool; block-driven ends run beside them.  The 1 KiB ring returns
    credit across C/2 many times."""
    for seed, cap in enumerate((1024, 65536)):
        rng = np.random.default_rng(5800 + seed)
        ops = test_gpu_parity._random_ops(rng, cap, 60)
        ops += [op for k in range(20) for op in (("send", [9, 5, 100 + 37 * k], 40 + k, 0), ("recv", 1 << 16))]
        _compare(trace.run_trace(BlockEngine(svc, "pinned", 3, drive=drive), cap, ops),
                 trace.run_trace(oracle, cap, ops), "service, %s block-driven, cap %d" % (drive, cap))


def _pinned_bytes(L, n):
    p = L.b200_mem_alloc_host(n)
    assert p
    return p, np.ctypeslib.as_array((C.c_uint8 * n).from_address(p))


@pytest.mark.parametrize("service", [False, True])
@pytest.mark.parametrize("device_end", ["tx", "rx"])
def test_block_and_host_ends_concurrently(gpu, service, device_end):
    """One end streams from a device CTA while the other is driven by host calls at the same time, over a dozen laps
    of a 16 KiB ring (credit crosses C/2 every few frames).  Every wait is bounded; the stream arrives whole with the
    cursors and mirrors consistent."""
    pkg, L = gpu, gpu.lib()
    R = bl.Runner(pkg)
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 16384)
    tx, rx = pkg.connected_pair("bc-tx-%s-%d" % (device_end, service), "bc-rx-%s-%d" % (device_end, service))
    lens = [9, 1000, 9, 3000, 9, 500, 17, 2048] * 30
    total = sum(lens)
    src, s_np = _pinned_bytes(L, total)
    dst, d_np = _pinned_bytes(L, total)
    s_np[:] = np.random.default_rng(12).integers(0, 256, total, dtype=np.uint8)
    d_np[:] = 0
    slp = L.b200_mem_alloc_host(16 * len(lens))
    arr = (pkg.Slice * len(lens)).from_address(slp)
    offs = [0]
    for n in lens[:-1]:
        offs.append(offs[-1] + n)
    for k, n in enumerate(lens):
        arr[k].ptr, arr[k].len = src + offs[k], n
    if service:
        assert L.b200_service_start(4) == 0, pkg.last_error()
    try:
        dev = tx if device_end == "tx" else rx
        h = dev.device_claim()
        deadline = time.time() + 60
        if device_end == "tx":
            R.launch([h], [[dict(kind=bl.STREAM_SEND, pair=0, slices=slp, n=len(lens))]], budget_s=60.0)
            moved = 0
            while moved < total and time.time() < deadline:
                moved += rx.recv_into(dst + moved, total - moved)
        else:
            R.launch([h], [[dict(kind=bl.STREAM_RECV, pair=0, dst=dst, n=total)]], budget_s=60.0)
            idx = bidx = moved = 0
            while idx < len(lens) and time.time() < deadline:
                window = [(src + offs[j], lens[j]) for j in range(idx, min(idx + 4, len(lens)))]
                sent = tx.send_raw(window, bidx)
                moved += sent
                while sent > 0:
                    left = lens[idx] - bidx
                    if sent >= left:
                        sent, idx, bidx = sent - left, idx + 1, 0
                    else:
                        bidx, sent = bidx + sent, 0
        res = R.wait()[0][0]
        assert moved == total, "host end stalled at %d of %d bytes" % (moved, total)
        assert res["status"] == bl.OK and res["ret"] == total, res
        assert np.array_equal(d_np, s_np)
        st, sr = tx.state(), rx.state()
        assert sr["head"] == sr["moving_head"] == st["remote_tail"] and sr["remain"] == 0
        assert st["partial_write"] == 0
        assert not rx.has_message() and rx.readable() == 0 and not tx.has_pending_writes()
        dev.device_release()
    finally:
        if service:
            L.b200_service_stop()
        for p in (tx, rx):
            p.disconnect()
            p.putback()
        for p in (src, dst, slp):
            L.b200_mem_free_host(p)


# ---- many connections: streams, and the benchmark's shape

def _setup_streams(pkg, nconn, ring_kb, msg, rounds, name):
    L = pkg.lib()
    pkg.config_set("GRPC_RDMA_RING_BUFFER_SIZE_KB", ring_kb)
    pkg.config_set("GRPC_RDMA_MAX_SGE", 30)
    lens = pkg.chttp2_slice_lens(msg)
    total = sum(lens)
    pairs = [pkg.connected_pair("%s-tx%d" % (name, c), "%s-rx%d" % (name, c)) for c in range(nconn)]
    src = L.b200_mem_alloc_device(nconn * total)
    dst = L.b200_mem_alloc_device(nconn * total * rounds)
    slp = L.b200_mem_alloc_host(16 * len(lens) * nconn)
    assert src and dst and slp
    i = np.arange(total, dtype=np.uint64)
    host = np.zeros((nconn, total), np.uint8)
    for c in range(nconn):
        host[c] = ((i * np.uint64(2654435761) >> np.uint64(13)) + np.uint64(171 * c)) & np.uint64(255)
    assert L.b200_memcpy(src, host.ctypes.data, host.size, 0, None) == 0
    L.b200_stream_sync(None)
    arr = (pkg.Slice * (len(lens) * nconn)).from_address(slp)
    for c in range(nconn):
        off = 0
        for k, n in enumerate(lens):
            arr[c * len(lens) + k].ptr, arr[c * len(lens) + k].len = src + c * total + off, n
            off += n
    return dict(L=L, lens=lens, total=total, pairs=pairs, src=src, dst=dst, slp=slp, host=host)


def _check_and_free(S, rounds, ring_zero):
    L, total, host = S["L"], S["total"], S["host"]
    for c, (tx, rx) in enumerate(S["pairs"]):
        st, sr = tx.state(), rx.state()
        assert sr["head"] == sr["moving_head"] == st["remote_tail"] and sr["remain"] == 0, c
        assert st["partial_write"] == 0 and not rx.has_message() and rx.readable() == 0, c
        out = np.zeros(total * rounds, np.uint8)
        assert L.b200_memcpy(out.ctypes.data, S["dst"] + c * rounds * total, out.size, 1, None) == 0
        L.b200_stream_sync(None)
        for r in range(rounds):
            assert np.array_equal(out[r * total:(r + 1) * total], host[c]), (c, r)
        if ring_zero:
            assert not rx.ring_image().any(), c  # everything read was cleared
    for tx, rx in S["pairs"]:
        for p in (tx, rx):
            if p.device_owned():
                p.device_release()
            p.disconnect()
            p.putback()
    L.b200_mem_free_device(S["src"])
    L.b200_mem_free_device(S["dst"])
    L.b200_mem_free_host(S["slp"])


def test_sender_and_receiver_ctas_concurrently(gpu):
    """8 connections, 256 KiB rings, 3 chttp2-shaped 1 MiB messages each: a sender CTA and a receiver CTA per
    connection in one kernel, each ring lapped a dozen times while both ends run."""
    R = bl.Runner(gpu)
    rounds = 3
    S = _setup_streams(gpu, 8, 256, 1 << 20, rounds, "bcc")
    handles, lists, nl = [], [], len(S["lens"])
    for c, (tx, rx) in enumerate(S["pairs"]):
        handles += [tx.device_claim(), rx.device_claim()]
        lists.append([dict(kind=bl.STREAM_SEND, pair=2 * c, slices=S["slp"] + 16 * c * nl, n=nl)] * rounds)
        lists.append([dict(kind=bl.STREAM_RECV, pair=2 * c + 1, dst=S["dst"] + (c * rounds + r) * S["total"],
                           n=S["total"]) for r in range(rounds)])
    res = R.run(handles, lists, budget_s=120.0)
    for lst in res:
        assert all(o["status"] == bl.OK and o["ret"] == S["total"] for o in lst), lst
    _check_and_free(S, rounds, ring_zero=True)


def test_benchmark_shape_256_connections(gpu):
    """256 connections, 16 MiB rings, one chttp2-shaped 4 MiB message each: one kernel of block sends
    (UNTIL_BLOCKED), then one of block receives; a prepared k_send / k_recv batch moves a message first, on the
    same pairs and buffers.  The bytes, the calls, the frames (the block Send's tail advances exactly as k_send's did),
    and every ring all-zero after the drain."""
    pkg, L = gpu, gpu.lib()
    R = bl.Runner(pkg)
    n = 256
    S = _setup_streams(pkg, n, 16384, 4 << 20, 1, "bbs")
    nl, total = len(S["lens"]), S["total"]
    # the same op through the library's batches first, on the same buffers
    sl = [pkg.make_slices([(S["src"] + c * total + sum(S["lens"][:k]), S["lens"][k]) for k in range(nl)])
          for c in range(n)]
    bs = pkg.Batch("send", [(S["pairs"][c][0], sl[c], nl, 0) for c in range(n)], pkg.UNTIL_BLOCKED)
    br = pkg.Batch("recv", [(S["pairs"][c][1], S["dst"] + c * total, total) for c in range(n)], pkg.UNTIL_BLOCKED)
    bs.launch()
    assert bs.results() == [total] * n
    br.launch()
    assert br.results() == [total] * n
    tail1 = [S["pairs"][c][0].state()["remote_tail"] for c in range(n)]
    bs.destroy()
    br.destroy()
    handles = []
    for tx, rx in S["pairs"]:
        handles += [tx.device_claim(), rx.device_claim()]
    sres = R.run(handles, [[dict(kind=bl.SEND, pair=2 * c, slices=S["slp"] + 16 * c * nl, n=nl,
                                 flags=bl.UNTIL_BLOCKED)] for c in range(n)], budget_s=120.0)
    rres = R.run(handles, [[dict(kind=bl.RECV, pair=2 * c + 1, dst=S["dst"] + c * total, cap=total,
                                 flags=bl.UNTIL_BLOCKED)] for c in range(n)], budget_s=120.0)
    for c in range(n):
        assert sres[c][0]["ret"] == total and rres[c][0]["ret"] == total, (c, sres[c], rres[c])
        # per-slice framing, no credit stop: every slice is one call's frame, max_sge (30) slices per call
        assert sres[c][0]["calls"] == (nl + 29) // 30, sres[c]
        assert rres[c][0]["calls"] == nl, rres[c]
    # the second message's frames follow the first's in each ring: the tails moved by the same encoded size
    for c in range(n):
        assert S["pairs"][c][0].state()["remote_tail"] == (2 * tail1[c]) % (16 << 20), c
    _check_and_free(S, 1, ring_zero=True)


# ---- refusals

def test_refusals_change_nothing(gpu):
    pkg, L = gpu, gpu.lib()
    R = bl.Runner(pkg)
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 4096)
    a, b = pkg.connected_pair("bref-a", "bref-b")
    dev = L.b200_mem_alloc_device(4096)
    slp = L.b200_mem_alloc_host(16)
    (pkg.Slice * 1).from_address(slp)[0].ptr = dev
    (pkg.Slice * 1).from_address(slp)[0].len = 100
    msg = np.arange(100, dtype=np.uint8)
    assert b.send([msg]) == 100  # a frame waits in a's ring
    ha, hb = a.device_claim(), b.device_claim()
    before = (a.state(), b.state(), a.ring_image().copy(), b.ring_image().copy())

    def unchanged():
        assert (a.state(), b.state()) == before[:2]
        assert np.array_equal(a.ring_image(), before[2]) and np.array_equal(b.ring_image(), before[3])

    send = dict(kind=bl.SEND, pair=1, slices=slp, n=1)
    recv = dict(kind=bl.RECV, pair=0, dst=dev, cap=4096)
    # a block of another shape
    for threads in (256, 320, 32):
        assert R.wrong_shape([ha, hb], send, recv, threads) == [(0, 0), (0, 0)], threads
    unchanged()
    # flag bits other than B200_BATCH_UNTIL_BLOCKED
    for fl in (0x2, 0x4, 0x8, 0x9, 0x100):
        res = R.run([ha, hb], [[dict(send, flags=fl)], [dict(recv, flags=fl)]])
        assert [r[0]["ret"] for r in res] == [0, 0] and [r[0]["calls"] for r in res] == [0, 0], fl
    unchanged()
    # n == 0, cap == 0
    res = R.run([ha, hb], [[dict(send, n=0)], [dict(recv, cap=0)]])
    assert [r[0]["ret"] for r in res] == [0, 0]
    unchanged()
    # the calls work on the same handles
    res = R.run([ha, hb], [[recv]])
    assert res[0][0]["ret"] == 100
    out = np.zeros(100, np.uint8)
    L.b200_memcpy(out.ctypes.data, dev, 100, 1, None)
    L.b200_stream_sync(None)
    assert np.array_equal(out, msg)
    a.device_release()
    # the peer has gone: a disconnects, b is HalfClosed with peer_exit; b's block calls answer 0 and change nothing
    a.disconnect()
    assert b.status() == 3 and b.state()["peer_exit"] == 1
    st_b, img_b = b.state(), b.ring_image().copy()
    res = R.run([ha, hb], [[send], [dict(recv, pair=1)]])
    assert [r[0]["ret"] for r in res] == [0, 0] and [r[0]["calls"] for r in res] == [0, 0]
    assert b.state() == st_b and np.array_equal(b.ring_image(), img_b)
    b.device_release()
    b.disconnect()
    for p in (a, b):
        p.putback()
    L.b200_mem_free_device(dev)
    L.b200_mem_free_host(slp)


# ---- the CUDA-IPC wire: a block-driven sender in one process, a host-driven receiver in another (one GPU)

def test_block_sender_over_the_ipc_wire():
    """3 x 1 MiB chttp2-shaped messages through a 256 KiB ring: the device CTA's frames land in the other process's
    ring and it needs the credit that comes back over the wire (system scope) to go on."""
    import subprocess
    import sys
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        procs = [subprocess.Popen([sys.executable, os.path.join(HERE, "device_block_ipc_worker.py"), role, "0", d,
                                   "256", str(1 << 20), "3"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                  text=True)
                 for role in ("server", "client")]
        outs = [p.communicate(timeout=500)[0] for p in procs]
        assert all(p.returncode == 0 for p in procs), "\n".join(outs)
        cli, srv = [json.load(open(os.path.join(d, r + ".json"))) for r in ("client", "server")]
    assert cli["ok"] and cli["released"] and not cli["pending"] and min(cli["calls"]) > 1
    assert srv["ok"] and srv["ring_empty"] and srv["half_closed"]
    assert cli["state"]["remote_tail"] == srv["state"]["head"] == srv["state"]["moving_head"]
