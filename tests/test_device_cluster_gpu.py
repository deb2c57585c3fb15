"""GPU: cluster-level device Send / Recv (b200_cluster_send / b200_cluster_recv, include/b200_device_block.cuh) driven
from a user kernel's thread-block clusters (tests/native/device_cluster.cu), for clusters of K = 1, 2, 8 and 16 CTAs.

Bar of test_device_block_gpu.py: every return value and `calls`, partial_write, both pairs' cursors and readiness
answers, the SHA-1 of the delivered bytes and the receiver's ring image with pads masked, against the golden records and
the CPU models (reference, coalesced, stamped).  Then cluster, block and warp calls on one pair, one end on the host,
sender and receiver clusters side by side, 1 / 4 / 16 connections with 4 MiB messages, the refusals and the CUDA-IPC
wire.  K = 16 is skipped where the device cannot place such a cluster."""
import json
import os
import time

import numpy as np
import pytest

import coalesce_lib
import device_block_lib as bl
import device_cluster_lib as cl
import device_lib
import stamp_lib
import test_coalesce_gpu
import test_device_block_gpu as tb
import test_gpu_parity
import test_stamp_gpu
import trace
from device_cluster_lib import ClusterEngine

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "traces.json")))
_compare = test_gpu_parity._compare
_ops = tb._ops
KS = [1, 2, 8, 16]
MEMS = [("device", 0), ("device", 5), ("pinned", 9)]


@pytest.fixture
def k(gpu, request):
    kk = request.param
    if cl.max_clusters(kk) < 1:
        pytest.skip("this device cannot place a cluster of %d CTAs of %d threads with %d bytes of shared memory each"
                    % (kk, cl.THREADS, cl.SMEM_BYTES))
    return kk


def by_k(f):
    return pytest.mark.parametrize("k", KS, indirect=True)(f)


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
    cl.Runner(gpu)  # the drivers' kernels are loaded before the resident kernels start
    bl.Runner(gpu)
    device_lib.Runner(gpu)
    L = gpu.lib()
    assert L.b200_service_start(4) == 0, gpu.last_error()
    yield gpu
    L.b200_service_stop()


# ---- both ends cluster-driven, against the golden records and the models

@by_k
@pytest.mark.parametrize("name", sorted(GOLDEN["traces"]))
def test_golden_traces_cluster_driven(gpu, k, name):
    t = GOLDEN["traces"][name]
    mem, mis = MEMS[sorted(GOLDEN["traces"]).index(name) % 3]
    recs = trace.run_trace(ClusterEngine(gpu, k, mem, mis), t["cap"], _ops(t["ops"]), GOLDEN["max_sge"])
    _compare(recs, t["records"], "golden %s K=%d [%s+%d]" % (name, k, mem, mis))


@by_k
def test_golden_full_size_cluster_driven(gpu, k):
    full = json.load(open(os.path.join(HERE, "golden", "traces_full.json")))
    for name, t in sorted(full["traces"].items()):
        recs = trace.run_trace(ClusterEngine(gpu, k, "device", 3), t["cap"], _ops(t["ops"]), full["max_sge"],
                               ring_images=False)
        _compare(recs, t["records"], "golden full %s K=%d" % (name, k))


@by_k
@pytest.mark.parametrize("seed", range(4))
def test_random_traces_vs_oracle(gpu, oracle, k, seed):
    rng = np.random.default_rng(6400 + 10 * k + seed)
    cap = [64, 1024, 4096, 65536][seed]
    ops = test_gpu_parity._random_ops(rng, cap, 80)
    mem, mis = MEMS[seed % 3]
    _compare(trace.run_trace(ClusterEngine(gpu, k, mem, mis), cap, ops), trace.run_trace(oracle, cap, ops),
             "random seed %d cap %d K=%d [%s+%d]" % (seed, cap, k, mem, mis))


@by_k
@pytest.mark.parametrize("max_sge", [1, 4, 32])
def test_other_max_sge(gpu, oracle, k, max_sge):
    ops = [("send", [7] * 50, 1, 0), ("send_all", [9, 100] * 30, 2, 3), ("recv_drain", 1 << 16),
           ("send_all", [9, 100] * 30, 3, 0), ("recv_drain", 1 << 16), ("send", [5] * 40, 4, 2), ("recv", 3),
           ("send_all", [9, 20000] * 8, 5, 0), ("recv_drain", 1 << 18)]
    want = trace.run_trace(oracle, 1 << 18, ops, max_sge)
    got = trace.run_trace(ClusterEngine(gpu, k, "device", 1), 1 << 18, ops, max_sge)
    _compare(got, want, "max_sge %d K=%d" % (max_sge, k))


@by_k
@pytest.mark.parametrize("seed", range(3))
def test_coalesced_vs_model(gpu, co, k, seed):
    rng = np.random.default_rng(6500 + 10 * k + seed)
    cap = [1024, 65536, 1 << 20][seed]
    ops = test_coalesce_gpu._random_ops(rng, cap, 60)
    mem, mis = MEMS[seed % 3]
    got = trace.run_trace(ClusterEngine(gpu, k, mem, mis, config={"B200_SEND_COALESCE": 1}), cap, ops)
    _compare(got, trace.run_trace(co, cap, ops), "coalesced seed %d cap %d K=%d" % (seed, cap, k))


@by_k
@pytest.mark.parametrize("seed", range(2))
@pytest.mark.parametrize("coalesced", [False, True])
def test_stamped_vs_model(gpu, so, soc, k, seed, coalesced):
    rng = np.random.default_rng(6600 + 10 * k + seed)
    cap = [4096, 65536][seed]
    mem, mis = MEMS[seed % 3]
    eng = ClusterEngine(gpu, k, mem, mis, config={"B200_RING_STAMPED": 1, "B200_SEND_COALESCE": int(coalesced)})
    test_stamp_gpu._replay(eng, soc if coalesced else so, cap, test_stamp_gpu._random_ops(rng, cap, 80))


# ---- cluster, block and warp calls on one pair

@by_k
@pytest.mark.parametrize("seed", range(2))
def test_cluster_block_and_warp_calls_interleaved(gpu, oracle, k, seed):
    """single calls of each end cycle through cluster calls, a block call from CTA rank 0 and a warp call from its
    warp 0"""
    rng = np.random.default_rng(6700 + 10 * k + seed)
    cap = [1024, 65536][seed]
    ops = test_gpu_parity._random_ops(rng, cap, 80)
    got = trace.run_trace(ClusterEngine(gpu, k, "device", seed, mix_every=2 + seed), cap, ops)
    _compare(got, trace.run_trace(oracle, cap, ops), "cluster + block + warp seed %d cap %d K=%d" % (seed, cap, k))


# ---- one end on the device, the other on the host

@by_k
@pytest.mark.parametrize("drive", [("tx",), ("rx",)])
def test_mixed_drivers_golden(gpu, k, drive):
    for name in ("chttp2_300k_128k", "credit_2k", "max_sge_cut_64k"):
        t = GOLDEN["traces"][name]
        recs = trace.run_trace(ClusterEngine(gpu, k, "device", 3, drive=drive), t["cap"], _ops(t["ops"]),
                               GOLDEN["max_sge"])
        _compare(recs, t["records"], "golden %s driven by %s, K=%d" % (name, drive, k))


@by_k
@pytest.mark.parametrize("drive", [("tx",), ("rx",), ("tx", "rx")])
def test_mixed_drivers_under_the_service(svc, oracle, k, drive):
    """host ends go through the owner warps and the pool; cluster-driven ends run beside them"""
    cap = 1024
    rng = np.random.default_rng(6800 + k)
    ops = test_gpu_parity._random_ops(rng, cap, 60)
    ops += [op for j in range(20) for op in (("send", [9, 5, 100 + 37 * j], 40 + j, 0), ("recv", 1 << 16))]
    _compare(trace.run_trace(ClusterEngine(svc, k, "pinned", 3, drive=drive), cap, ops),
             trace.run_trace(oracle, cap, ops), "service, %s cluster-driven, K=%d" % (drive, k))


@pytest.mark.parametrize("service", [False, True])
@pytest.mark.parametrize("device_end", ["tx", "rx"])
@pytest.mark.parametrize("k", [2, 8, 16], indirect=True)
def test_cluster_and_host_ends_concurrently(gpu, k, service, device_end):
    """One end streams from a device cluster while the other is driven by host calls at the same time, over a dozen
    laps of a 16 KiB ring.  Every wait is bounded; the stream arrives whole with the cursors and mirrors consistent."""
    pkg, L = gpu, gpu.lib()
    R = cl.Runner(pkg, k)
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 16384)
    tx, rx = pkg.connected_pair("cc-tx-%s-%d-%d" % (device_end, service, k), "cc-rx-%s-%d-%d" % (device_end, service, k))
    lens = [9, 1000, 9, 3000, 9, 500, 17, 2048] * 30
    total = sum(lens)
    src, s_np = tb._pinned_bytes(L, total)
    dst, d_np = tb._pinned_bytes(L, total)
    s_np[:] = np.random.default_rng(13).integers(0, 256, total, dtype=np.uint8)
    d_np[:] = 0
    slp = L.b200_mem_alloc_host(16 * len(lens))
    arr = (pkg.Slice * len(lens)).from_address(slp)
    offs = [0]
    for n in lens[:-1]:
        offs.append(offs[-1] + n)
    for j, n in enumerate(lens):
        arr[j].ptr, arr[j].len = src + offs[j], n
    if service:
        assert L.b200_service_start(4) == 0, pkg.last_error()
    try:
        dev = tx if device_end == "tx" else rx
        h = dev.device_claim()
        deadline = time.time() + 60
        if device_end == "tx":
            R.launch([h], [[dict(kind=cl.STREAM_SEND, pair=0, slices=slp, n=len(lens))]], budget_s=60.0)
            moved = 0
            while moved < total and time.time() < deadline:
                moved += rx.recv_into(dst + moved, total - moved)
        else:
            R.launch([h], [[dict(kind=cl.STREAM_RECV, pair=0, dst=dst, n=total)]], budget_s=60.0)
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
        assert res["status"] == cl.OK and res["ret"] == total, res
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


# ---- streams: sender and receiver clusters side by side, and 1 / 4 / 16 connections

@by_k
def test_sender_and_receiver_clusters_concurrently(gpu, k):
    """A sender cluster and a receiver cluster per connection in one kernel, 3 chttp2-shaped 1 MiB messages each
    through 256 KiB rings: every message is larger than the ring, which is lapped a dozen times while both ends run."""
    nconn = max(1, min(4, cl.max_clusters(k) // 2))
    R = cl.Runner(gpu, k)
    rounds = 3
    S = tb._setup_streams(gpu, nconn, 256, 1 << 20, rounds, "ccc%d" % k)
    handles, lists, nl = [], [], len(S["lens"])
    for c, (tx, rx) in enumerate(S["pairs"]):
        handles += [tx.device_claim(), rx.device_claim()]
        lists.append([dict(kind=cl.STREAM_SEND, pair=2 * c, slices=S["slp"] + 16 * c * nl, n=nl)] * rounds)
        lists.append([dict(kind=cl.STREAM_RECV, pair=2 * c + 1, dst=S["dst"] + (c * rounds + r) * S["total"],
                           n=S["total"]) for r in range(rounds)])
    res = R.run(handles, lists, budget_s=120.0)
    for lst in res:
        assert all(o["status"] == cl.OK and o["ret"] == S["total"] for o in lst), lst
    tb._check_and_free(S, rounds, ring_zero=True)


@by_k
@pytest.mark.parametrize("nconn", [1, 4, 16])
def test_connections_with_4mib_messages(gpu, k, nconn):
    """nconn connections, 16 MiB rings, one chttp2-shaped 4 MiB message each: a kernel of cluster sends
    (UNTIL_BLOCKED), then a kernel of cluster receives.  The bytes, the calls (max_sge 30 slices per Send call, one Recv
    call per frame), every delivered byte and every ring all-zero after the drain."""
    R = cl.Runner(gpu, k)
    S = tb._setup_streams(gpu, nconn, 16384, 4 << 20, 1, "c4m%d-%d" % (k, nconn))
    nl, total = len(S["lens"]), S["total"]
    handles = []
    for tx, rx in S["pairs"]:
        handles += [tx.device_claim(), rx.device_claim()]
    sres = R.run(handles, [[dict(kind=cl.SEND, pair=2 * c, slices=S["slp"] + 16 * c * nl, n=nl,
                                 flags=cl.UNTIL_BLOCKED)] for c in range(nconn)], budget_s=120.0)
    rres = R.run(handles, [[dict(kind=cl.RECV, pair=2 * c + 1, dst=S["dst"] + c * total, cap=total,
                                 flags=cl.UNTIL_BLOCKED)] for c in range(nconn)], budget_s=120.0)
    for c in range(nconn):
        assert sres[c][0]["ret"] == total and rres[c][0]["ret"] == total, (c, sres[c], rres[c])
        assert sres[c][0]["calls"] == (nl + 29) // 30, sres[c]
        assert rres[c][0]["calls"] == nl, rres[c]
    tb._check_and_free(S, 1, ring_zero=True)


# ---- refusals

def test_refusals_change_nothing(gpu):
    pkg, L = gpu, gpu.lib()
    R = cl.Runner(pkg, 2)
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 4096)
    a, b = pkg.connected_pair("cref-a", "cref-b")
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

    send = dict(kind=cl.SEND, pair=1, slices=slp, n=1)
    recv = dict(kind=cl.RECV, pair=0, dst=dev, cap=4096)
    # a CTA of another shape, with and without clusters
    for threads, grid, cluster in ((256, (1, 1), (1, 1)), (320, (2, 1), (2, 1)), (32, (4, 1), (4, 1))):
        assert R.wrong_shape([ha, hb], send, recv, threads, grid, cluster) == [(0, 0), (0, 0)], (threads, cluster)
    unchanged()
    # a cluster that is not K x 1 x 1
    for grid, cluster in (((2, 2), (2, 2)), ((1, 2), (1, 2)), ((2, 4), (2, 4))):
        assert R.wrong_shape([ha, hb], send, recv, cl.THREADS, grid, cluster) == [(0, 0), (0, 0)], cluster
    unchanged()
    for kk in (1, 2, 8):
        R.k = kk
        # flag bits other than B200_BATCH_UNTIL_BLOCKED
        for fl in (0x2, 0x4, 0x8, 0x9, 0x100):
            res = R.run([ha, hb], [[dict(send, flags=fl)], [dict(recv, flags=fl)]])
            assert [r[0]["ret"] for r in res] == [0, 0] and [r[0]["calls"] for r in res] == [0, 0], (kk, fl)
        unchanged()
        # n == 0, cap == 0
        res = R.run([ha, hb], [[dict(send, n=0)], [dict(recv, cap=0)]])
        assert [r[0]["ret"] for r in res] == [0, 0], kk
        unchanged()
    # the calls work on the same handles
    R.k = 2
    res = R.run([ha, hb], [[recv]])
    assert res[0][0]["ret"] == 100 and res[0][0]["calls"] == 1
    out = np.zeros(100, np.uint8)
    L.b200_memcpy(out.ctypes.data, dev, 100, 1, None)
    L.b200_stream_sync(None)
    assert np.array_equal(out, msg)
    a.device_release()
    # the peer has gone: a disconnects, b is HalfClosed with peer_exit; b's cluster calls answer 0 and change nothing
    a.disconnect()
    assert b.status() == 3 and b.state()["peer_exit"] == 1
    st_b, img_b = b.state(), b.ring_image().copy()
    for kk in (1, 2):
        R.k = kk
        res = R.run([ha, hb], [[send], [dict(recv, pair=1)]])
        assert [r[0]["ret"] for r in res] == [0, 0] and [r[0]["calls"] for r in res] == [0, 0], kk
        assert b.state() == st_b and np.array_equal(b.ring_image(), img_b)
    b.device_release()
    b.disconnect()
    for p in (a, b):
        p.putback()
    L.b200_mem_free_device(dev)
    L.b200_mem_free_host(slp)


# ---- the CUDA-IPC wire: a cluster-driven sender in one process, a host-driven receiver in another (one GPU)

@pytest.mark.parametrize("k", [2, 16], indirect=True)
def test_cluster_sender_over_the_ipc_wire(k):
    """3 x 1 MiB chttp2-shaped messages through a 256 KiB ring: the device cluster's frames land in the other
    process's ring and it needs the credit that comes back over the wire (system scope) to go on."""
    import subprocess
    import sys
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        procs = [subprocess.Popen([sys.executable, os.path.join(HERE, "device_cluster_ipc_worker.py"), str(k), role,
                                   "0", d, "256", str(1 << 20), "3"], stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT, text=True)
                 for role in ("server", "client")]
        outs = [p.communicate(timeout=500)[0] for p in procs]
        assert all(p.returncode == 0 for p in procs), "\n".join(outs)
        cli, srv = [json.load(open(os.path.join(d, r + ".json"))) for r in ("client", "server")]
    assert cli["ok"] and cli["released"] and not cli["pending"] and min(cli["calls"]) > 1
    assert srv["ok"] and srv["ring_empty"] and srv["half_closed"]
    assert cli["state"]["remote_tail"] == srv["state"]["head"] == srv["state"]["moving_head"]
