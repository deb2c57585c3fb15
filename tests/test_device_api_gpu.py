"""GPU: device-side Send / Recv (include/b200_device.cuh) driven from a user kernel (tests/native/device_api.cu).

Bar of test_gpu_parity.py: every return value and `calls`, partial_write, both pairs' cursors and readiness answers,
the SHA-1 of the delivered bytes and the receiver's ring image with pads masked -- here with every op of a claimed end
run by a device warp, against the golden records and the CPU models (reference, coalesced, stamped).  Then the mixed
drivers (one end on the device, the other on the host, with and without the service), the ownership rules, the
benchmark's shape with one sender and one receiver warp per connection, and the Poller."""
import ctypes as C
import json
import os
import select

import numpy as np
import pytest

import coalesce_lib
import device_lib
import stamp_lib
import test_coalesce_gpu
import test_gpu_parity
import test_stamp_gpu
import trace
from device_lib import DeviceEngine

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
    device_lib.load()
    device_lib.Runner(gpu)  # the driver's kernel is loaded before the resident kernels start
    L = gpu.lib()
    assert L.b200_service_start(4) == 0, gpu.last_error()
    yield gpu
    L.b200_service_stop()


# ---- both ends device-driven, against the golden records and the models

@pytest.mark.parametrize("name", sorted(GOLDEN["traces"]))
@pytest.mark.parametrize("mem,mis", [("device", 0), ("device", 5), ("pinned", 9)])
def test_golden_traces_device_driven(gpu, name, mem, mis):
    t = GOLDEN["traces"][name]
    recs = trace.run_trace(DeviceEngine(gpu, mem, mis), t["cap"], _ops(t["ops"]), GOLDEN["max_sge"])
    _compare(recs, t["records"], "golden %s [%s+%d]" % (name, mem, mis))


def test_golden_full_size_device_driven(gpu):
    full = json.load(open(os.path.join(HERE, "golden", "traces_full.json")))
    for name, t in sorted(full["traces"].items()):
        recs = trace.run_trace(DeviceEngine(gpu, "device", 3), t["cap"], _ops(t["ops"]), full["max_sge"],
                               ring_images=False)
        _compare(recs, t["records"], "golden full %s" % name)


@pytest.mark.parametrize("seed", range(10))
def test_random_traces_vs_oracle(gpu, oracle, seed):
    rng = np.random.default_rng(4400 + seed)
    cap = [64, 1024, 2048, 4096, 65536][seed % 5]
    ops = test_gpu_parity._random_ops(rng, cap, 80)
    want = trace.run_trace(oracle, cap, ops)
    mem, mis = [("device", 0), ("device", 7), ("pinned", 13)][seed % 3]
    got = trace.run_trace(DeviceEngine(gpu, mem, mis), cap, ops)
    _compare(got, want, "random seed %d cap %d [%s+%d]" % (seed, cap, mem, mis))


@pytest.mark.parametrize("max_sge", [1, 4, 32])
def test_other_max_sge(gpu, oracle, max_sge):
    ops = [("send", [7] * 50, 1, 0), ("send_all", [9, 100] * 30, 2, 3), ("recv_drain", 1 << 16),
           ("send_all", [9, 100] * 30, 3, 0), ("recv_drain", 1 << 16), ("send", [5] * 40, 4, 2), ("recv", 3)]
    want = trace.run_trace(oracle, 16384, ops, max_sge)
    got = trace.run_trace(DeviceEngine(gpu, "device", 1), 16384, ops, max_sge)
    _compare(got, want, "max_sge %d" % max_sge)


@pytest.mark.parametrize("seed", range(6))
def test_coalesced_vs_model(gpu, co, seed):
    rng = np.random.default_rng(4500 + seed)
    cap = [64, 1024, 4096, 65536, 2048, 1 << 20][seed]
    ops = test_coalesce_gpu._random_ops(rng, cap, 60)
    want = trace.run_trace(co, cap, ops)
    mem, mis = [("device", 0), ("device", 5), ("pinned", 9)][seed % 3]
    got = trace.run_trace(DeviceEngine(gpu, mem, mis, config={"B200_SEND_COALESCE": 1}), cap, ops)
    _compare(got, want, "coalesced seed %d cap %d" % (seed, cap))


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("coalesced", [False, True])
def test_stamped_vs_model(gpu, so, soc, seed, coalesced):
    rng = np.random.default_rng(4600 + seed)
    cap = [64, 1024, 4096, 65536][seed % 4]
    mem, mis = [("device", 0), ("device", 3), ("pinned", 11)][seed % 3]
    eng = DeviceEngine(gpu, mem, mis, config={"B200_RING_STAMPED": 1, "B200_SEND_COALESCE": int(coalesced)})
    test_stamp_gpu._replay(eng, soc if coalesced else so, cap, test_stamp_gpu._random_ops(rng, cap, 80))


def test_stamped_golden_and_full_size(gpu, so):
    for name, t in sorted(GOLDEN["traces"].items()):
        test_stamp_gpu._replay(DeviceEngine(gpu, "device", 5, config={"B200_RING_STAMPED": 1}), so, t["cap"],
                               _ops(t["ops"]), images=t["cap"] <= 1 << 17)
    lens = gpu.chttp2_slice_lens(4 << 20)
    ops = []
    for k in range(10):
        ops += [("send_all", lens, 600 + k, 0), ("recv_drain", [1 << 20, 5 << 20][k % 2]), ("recv_drain", 1 << 25)]
    test_stamp_gpu._replay(DeviceEngine(gpu, "device", 0, config={"B200_RING_STAMPED": 1}), so, 16 << 20, ops,
                           images=False)


class _HalfStampedEngine(DeviceEngine):
    """tx offers stamped frames, rx does not: the connection runs the reference format"""

    def pair_pair(self, cap, max_sge=30):
        self.pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", cap)
        self.pkg.config_set("GRPC_RDMA_MAX_SGE", max_sge)
        self.n += 1
        self.pkg.config_set("B200_RING_STAMPED", 1)
        try:
            tx = self.pkg.Pair("hs-tx%d" % self.n)
        finally:
            self.pkg.config_set("B200_RING_STAMPED", 0)
        rx = self.pkg.Pair("hs-rx%d" % self.n)
        assert tx.connect(rx.address()) and rx.connect(tx.address())
        assert not tx.stamped() and not rx.stamped()
        for p in (tx, rx):
            self.handles[p.h] = p.device_claim()
        return tx, rx


def test_stamped_offer_with_reference_peer(gpu, oracle):
    rng = np.random.default_rng(4700)
    ops = test_gpu_parity._random_ops(rng, 4096, 80)
    _compare(trace.run_trace(_HalfStampedEngine(gpu, "device", 2), 4096, ops), trace.run_trace(oracle, 4096, ops),
             "stamped offer, reference peer")


# ---- mixed drivers: one end on the device, the other on the host

@pytest.mark.parametrize("drive", [("tx",), ("rx",)])
@pytest.mark.parametrize("name", sorted(GOLDEN["traces"]))
def test_mixed_drivers_golden(gpu, drive, name):
    t = GOLDEN["traces"][name]
    recs = trace.run_trace(DeviceEngine(gpu, "device", 3, drive=drive), t["cap"], _ops(t["ops"]), GOLDEN["max_sge"])
    _compare(recs, t["records"], "golden %s driven by %s" % (name, drive))


@pytest.mark.parametrize("drive", [("tx",), ("rx",), ("tx", "rx")])
def test_mixed_drivers_under_the_service(svc, oracle, drive):
    """Host ends go through the owner warps (small calls, eager push, owed Retire) and the pool; device ends run
    beside them.  Every op matches the model."""
    L = svc.lib()
    hits = L.b200_service_eager_hits()
    for seed, cap in enumerate((1024, 65536)):
        rng = np.random.default_rng(4800 + seed)
        ops = test_gpu_parity._random_ops(rng, cap, 60)
        ops += [op for k in range(20) for op in (("send", [9, 5, 100 + 37 * k], 40 + k, 0), ("recv", 1 << 16))]
        _compare(trace.run_trace(DeviceEngine(svc, "pinned", 3, drive=drive), cap, ops),
                 trace.run_trace(oracle, cap, ops), "service, %s on the device, cap %d" % (drive, cap))
    if drive == ("tx", "rx"):
        assert L.b200_service_eager_hits() == hits  # no host Recv at all


def test_claim_and_release_under_the_service(svc, oracle):
    """Eager hits and an owed Retire before the claim; device ops; after the release the host calls (owner cache,
    eager path, mirrors) continue exactly as the model does."""
    L = svc.lib()
    eng = DeviceEngine(svc, "pinned", 1, drive=())
    cap = 4096
    tx, rx = eng.pair_pair(cap)
    otx, orx = oracle.pair_pair(cap)
    try:
        def both(fn_dev, fn_ora):
            g, w = fn_dev(), fn_ora()
            if isinstance(g, np.ndarray):
                assert np.array_equal(g, w)
            else:
                assert g == w
            assert tx.state() == oracle.state(otx) and rx.state() == oracle.state(orx)
            assert (rx.has_message(), rx.readable(), tx.has_pending_writes(), tx.writable()) == \
                (oracle.has_message(orx), oracle.readable(orx), oracle.has_pending_writes(otx), oracle.writable(otx))

        hits = L.b200_service_eager_hits()
        for k in range(3):
            bufs = trace.make_bufs([9, 200 + k], 70 + k)
            both(lambda: eng.send(tx, bufs), lambda: oracle.send(otx, bufs))
            both(lambda: eng.recv(rx, 1 << 12), lambda: oracle.recv(orx, 1 << 12))
        assert L.b200_service_eager_hits() > hits  # the last Recv owes its Retire: the claim drains it
        bufs = trace.make_bufs([9, 300], 80)
        both(lambda: eng.send(tx, bufs), lambda: oracle.send(otx, bufs))
        for p in (tx, rx):
            eng.handles[p.h] = p.device_claim()
        both(lambda: eng.recv(rx, 100), lambda: oracle.recv(orx, 100))
        for k in range(4):
            bufs = trace.make_bufs([9, 700 + k], 90 + k)
            both(lambda: eng.send(tx, bufs), lambda: oracle.send(otx, bufs))
        both(lambda: eng.recv(rx, 1 << 12), lambda: oracle.recv(orx, 1 << 12))
        for p in (tx, rx):
            del eng.handles[p.h]
            p.device_release()
        hits = L.b200_service_eager_hits()
        for k in range(6):
            bufs = trace.make_bufs([9, 100 + k], 110 + k)
            both(lambda: eng.recv(rx, 1 << 12), lambda: oracle.recv(orx, 1 << 12))
            both(lambda: eng.send(tx, bufs), lambda: oracle.send(otx, bufs))
        both(lambda: eng.recv_drain(rx, 1 << 16)[0], lambda: oracle.recv_drain(orx, 1 << 16)[0])
        assert L.b200_service_eager_hits() > hits  # the eager path works again
    finally:
        eng.destroy(tx)
        eng.destroy(rx)
        oracle.destroy(otx)
        oracle.destroy(orx)


# ---- ownership

def test_ownership_rules(gpu):
    pkg, L = gpu, gpu.lib()
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 4096)
    a = pkg.Pair("own-a")
    with pytest.raises(RuntimeError, match="not connected"):
        a.device_claim()
    b = pkg.Pair("own-b")
    assert a.connect(b.address()) and b.connect(a.address())
    h = a.device_claim()
    assert len(h) == 64 and a.device_owned() and not b.device_owned()
    with pytest.raises(RuntimeError, match="already"):
        a.device_claim()
    msg = np.arange(100, dtype=np.uint8)
    # host calls on the claimed end are refused, with the reason
    assert a.send([msg]) == 0 and "device-owned" in a.error()
    assert a.recv(100).size == 0
    dev = L.b200_mem_alloc_device(4096)
    slp = L.b200_mem_alloc_host(16)  # the device reads the slice array: pinned
    sl = (pkg.Slice * 1).from_address(slp)
    sl[0].ptr, sl[0].len = dev, 100
    sop = (pkg.SendOp * 1)()
    sop[0].pair, sop[0].slices, sop[0].nslices, sop[0].byte_idx = a.h, sl, 1, 0
    rop = (pkg.RecvOp * 1)()
    rop[0].pair, rop[0].dst, rop[0].cap = a.h, dev, 4096
    acc = (C.c_uint64 * 1)()
    assert L.b200_pairs_send(sop, 1, pkg.UNTIL_BLOCKED, acc, None) == -1
    assert L.b200_pairs_recv(rop, 1, pkg.UNTIL_BLOCKED, acc, None) == -1
    assert L.b200_batch_prepare_send(sop, 1, 0) is None
    assert L.b200_pairs_submit(sop, 1, acc, None, 0, None, 0) == -1 and "device-owned" in pkg.last_error()
    # the peer end keeps working: host Send -> device Recv, device Send -> host Recv
    R = device_lib.Runner(pkg)
    assert b.send([msg]) == 100 and a.has_message() and a.readable() == 100
    r = R.run([h], [[dict(kind=device_lib.RECV, pair=0, dst=dev, cap=4096)]])[0][0]
    assert r["ret"] == 100 and not a.has_message()
    out = np.zeros(100, np.uint8)
    L.b200_memcpy(out.ctypes.data, dev, 100, 1, None)
    L.b200_stream_sync(None)
    assert np.array_equal(out, msg)
    r = R.run([h], [[dict(kind=device_lib.SEND, pair=0, slices=slp, n=1, byte_idx=0)]])[0][0]
    assert r["ret"] == 100 and b.has_message()
    assert np.array_equal(b.recv(4096), msg)
    # Disconnect releases the claim and the peer sees peer_exit
    a.disconnect()
    assert not a.device_owned() and a.status() == 4 and b.status() == 3
    assert b.state()["peer_exit"] == 1
    b.disconnect()
    with pytest.raises(RuntimeError):
        a.device_release()
    L.b200_mem_free_device(dev)
    L.b200_mem_free_host(slp)
    a.putback()
    b.putback()


def test_claim_refused_while_a_posted_op_is_in_flight(svc):
    """A posted op counts as in flight until b200_async_poll has reported it finished."""
    pkg, L = svc, svc.lib()
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 4096)
    a, b = pkg.connected_pair("inf-a", "inf-b")
    dst = L.b200_mem_alloc_host(4096)
    again, n = C.c_int(0), C.c_uint64(0)
    op = L.b200_pair_post_recv(a.h, dst, 4096, 0, C.byref(again))
    assert op, pkg.last_error()
    with pytest.raises(RuntimeError, match="in flight"):
        a.device_claim()
    assert not a.device_owned()
    assert L.b200_async_poll(op, C.byref(n)) == 1 and n.value == 0
    a.device_claim()
    assert L.b200_pair_post_recv(a.h, dst, 4096, 0, C.byref(again)) is None and again.value == 0
    assert "device-owned" in pkg.last_error()
    for p in (a, b):
        p.disconnect()
        p.putback()
    L.b200_mem_free_host(dst)


def test_device_readiness_queries(gpu, oracle):
    eng = DeviceEngine(gpu, "device", 0)
    tx, rx = eng.pair_pair(1024)
    otx, orx = oracle.pair_pair(1024)
    try:
        for lens, rcap in (([100], 50), ([2000], 1 << 12), ([9, 9], 9), ([], 0)):
            if lens:
                bufs = trace.make_bufs(lens, 5)
                assert eng.send(tx, bufs) == oracle.send(otx, bufs)
            if rcap:
                assert np.array_equal(eng.recv(rx, rcap), oracle.recv(orx, rcap))
            assert eng.device_ready(rx)[:2] == (oracle.readable(orx), oracle.has_message(orx))
            assert eng.device_ready(tx)[2] == oracle.has_pending_writes(otx)
    finally:
        for p in (tx, rx):
            eng.destroy(p)
        oracle.destroy(otx)
        oracle.destroy(orx)


# ---- scale: one sender warp and one receiver warp per connection, all in one kernel

def _stream_many(gpu, nconn, rounds, ring_kb=16384, msg=4 << 20):
    pkg, L = gpu, gpu.lib()
    pkg.config_set("GRPC_RDMA_RING_BUFFER_SIZE_KB", ring_kb)
    pkg.config_set("GRPC_RDMA_MAX_SGE", 30)
    lens = pkg.chttp2_slice_lens(msg)
    total = sum(lens)
    pairs = [pkg.connected_pair("sc-tx%d" % c, "sc-rx%d" % c) for c in range(nconn)]
    handles = []
    for tx, rx in pairs:
        handles += [tx.device_claim(), rx.device_claim()]
    src = L.b200_mem_alloc_device(nconn * total)
    dst = L.b200_mem_alloc_device(nconn * total * rounds)
    slp = L.b200_mem_alloc_host(16 * len(lens) * nconn)
    assert src and dst and slp
    i = np.arange(total, dtype=np.uint64)
    host = np.zeros((nconn, total), np.uint8)
    for c in range(nconn):
        host[c] = ((i * np.uint64(2654435761) >> np.uint64(13)) + np.uint64(131 * c)) & np.uint64(255)
    assert L.b200_memcpy(src, host.ctypes.data, host.size, 0, None) == 0
    L.b200_stream_sync(None)
    arr = (pkg.Slice * (len(lens) * nconn)).from_address(slp)
    for c in range(nconn):
        off = 0
        for k, n in enumerate(lens):
            arr[c * len(lens) + k].ptr, arr[c * len(lens) + k].len = src + c * total + off, n
            off += n
    lists = []
    for c in range(nconn):
        lists.append([dict(kind=device_lib.STREAM_SEND, pair=2 * c, slices=slp + 16 * c * len(lens), n=len(lens))
                      for _ in range(rounds)])
        lists.append([dict(kind=device_lib.STREAM_RECV, pair=2 * c + 1, dst=dst + (c * rounds + r) * total, n=total)
                      for r in range(rounds)])
    res = device_lib.Runner(pkg).run(handles, lists, budget_s=120.0)
    for c in range(nconn):
        for r in range(rounds):
            assert res[2 * c][r] == dict(ret=total, calls=res[2 * c][r]["calls"], status=device_lib.OK), (c, r)
            assert res[2 * c + 1][r]["ret"] == total and res[2 * c + 1][r]["status"] == device_lib.OK, (c, r)
    enc = sum(16 + (n + 7) // 8 * 8 for n in lens)
    cap = ring_kb << 10
    for c, (tx, rx) in enumerate(pairs):
        st, sr = tx.state(), rx.state()
        # (cuts where credit ran out add frames: the tail is not a closed form of the message shape)
        assert sr["head"] == sr["moving_head"] == st["remote_tail"] and sr["remain"] == 0
        assert st["partial_write"] == 0 and not rx.has_message() and rx.readable() == 0
        out = np.zeros(total * rounds, np.uint8)
        assert L.b200_memcpy(out.ctypes.data, dst + c * rounds * total, out.size, 1, None) == 0
        L.b200_stream_sync(None)
        for r in range(rounds):
            assert np.array_equal(out[r * total:(r + 1) * total], host[c]), (c, r)
    for tx, rx in pairs:
        assert not rx.ring_image().any()  # everything read was cleared
        for p in (tx, rx):
            p.device_release()
            p.disconnect()
            p.putback()
    L.b200_mem_free_device(src)
    L.b200_mem_free_device(dst)
    L.b200_mem_free_host(slp)
    return enc * rounds // cap  # laps: at least this many, each message written as at least its unsplit frames


def test_many_connections_concurrent_warps(gpu):
    """64 connections, 16 MiB rings, 9 chttp2-shaped 4 MiB messages each: every ring wraps twice while the
    sender and receiver warps of all connections run side by side."""
    assert _stream_many(gpu, 64, 9) >= 2


def test_benchmark_shape_256_connections(gpu):
    _stream_many(gpu, 256, 1)


# ---- the Poller sees device-driven frames

def test_poller_sees_device_frames(gpu):
    pkg, L = gpu, gpu.lib()
    eng = DeviceEngine(gpu, "pinned", 0, drive=("tx",))
    pairs = [eng.pair_pair(1024) for _ in range(6)]
    rx = [p[1] for p in pairs]
    arr = (C.c_void_p * len(rx))(*[p.h for p in rx])
    ev = (C.c_uint32 * len(rx))()
    assert L.b200_poller_scan(arr, len(rx), ev) == 0
    for i in (1, 4):
        assert eng.send(pairs[i][0], [np.full(20, i, np.uint8)]) == 20
    assert L.b200_poller_scan(arr, len(rx), ev) == 2
    assert [bool(ev[i] & pkg.EV_READABLE) for i in range(len(rx))] == [i in (1, 4) for i in range(len(rx))]
    # background Poller over the service's ready ring: an eventfd kick with no host call on the pair
    assert L.b200_service_start(4) == 0, pkg.last_error()
    try:
        for p in rx:
            L.b200_poller_add(p.h)
        for p in rx:
            L.b200_pair_consume_wakeup(p.h)
        assert eng.send(pairs[2][0], [np.full(30, 2, np.uint8)]) == 30
        seen = set()
        for _ in range(50):
            r, _, _ = select.select([rx[2].wakeup_fd()], [], [], 0.1)
            seen |= set(r)
            if seen:
                break
        assert seen == {rx[2].wakeup_fd()}
        L.b200_poller_shutdown()
        for p in rx:
            L.b200_poller_remove(p.h)
    finally:
        L.b200_service_stop()
    for tx, r in pairs:
        eng.destroy(tx)
        eng.destroy(r)


# ---- the CUDA-IPC / NVLink wire: a device-driven sender in one process, a host-driven receiver in another

def test_device_sender_over_the_ipc_wire():
    """3 x 1 MiB chttp2-shaped messages through a 256 KiB ring: the device warp's frames land in the other
    process's HBM and it needs the credit that comes back over the wire (system scope) to go on."""
    import subprocess
    import sys
    import tempfile
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs on one machine")
    with tempfile.TemporaryDirectory() as d:
        procs = [subprocess.Popen([sys.executable, os.path.join(HERE, "device_ipc_worker.py"), role, str(dev), d,
                                   "256", str(1 << 20), "3"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                  text=True)
                 for role, dev in (("server", 1), ("client", 0))]
        outs = [p.communicate(timeout=500)[0] for p in procs]
        assert all(p.returncode == 0 for p in procs), "\n".join(outs)
        cli, srv = [json.load(open(os.path.join(d, r + ".json"))) for r in ("client", "server")]
    assert cli["ok"] and cli["released"] and not cli["pending"] and min(cli["calls"]) > 1
    assert srv["ok"] and srv["ring_empty"] and srv["half_closed"]
    assert cli["state"]["remote_tail"] == srv["state"]["head"] == srv["state"]["moving_head"]


# ---- a device-driven end and a host-driven end at the same time, over many laps of a small ring

def _pinned_bytes(L, n):
    p = L.b200_mem_alloc_host(n)
    assert p
    return p, np.ctypeslib.as_array((C.c_uint8 * n).from_address(p))


@pytest.mark.parametrize("service", [False, True])
@pytest.mark.parametrize("device_end", ["tx", "rx"])
def test_device_and_host_ends_concurrently(gpu, service, device_end):
    """One end streams from a device warp while the other is driven by host calls (single calls, through the owner
    warps under the service) at the same time.  The host end decides from its mirror whether a call can do anything
    (the no-credit Send, the empty-ring Recv), so a readiness or credit update lost between the two would stall it:
    every wait here is bounded, and the stream must arrive whole with the cursors and mirrors consistent."""
    import time
    pkg, L = gpu, gpu.lib()
    R = device_lib.Runner(pkg)
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 16384)
    tx, rx = pkg.connected_pair("cc-tx-%s-%d" % (device_end, service), "cc-rx-%s-%d" % (device_end, service))
    lens = [9, 1000, 9, 3000, 9, 500, 17, 2048] * 30  # ~200 KB: a dozen laps of the 16 KiB ring
    total = sum(lens)
    src, s_np = _pinned_bytes(L, total)
    dst, d_np = _pinned_bytes(L, total)
    s_np[:] = np.random.default_rng(11).integers(0, 256, total, dtype=np.uint8)
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
            R.launch([h], [[dict(kind=device_lib.STREAM_SEND, pair=0, slices=slp, n=len(lens))]], budget_s=60.0)
            moved = 0
            while moved < total and time.time() < deadline:
                moved += rx.recv_into(dst + moved, total - moved)
        else:
            R.launch([h], [[dict(kind=device_lib.STREAM_RECV, pair=0, dst=dst, n=total)]], budget_s=60.0)
            idx = bidx = moved = 0
            while idx < len(lens) and time.time() < deadline:
                window = [(src + offs[j], lens[j]) for j in range(idx, min(idx + 4, len(lens)))]
                sent = tx.send_raw(window, bidx)  # <= 4 slices, <= 8 KiB: the owner warps' small Send
                moved += sent
                while sent > 0:
                    left = lens[idx] - bidx
                    if sent >= left:
                        sent, idx, bidx = sent - left, idx + 1, 0
                    else:
                        bidx, sent = bidx + sent, 0
        res = R.wait()[0][0]
        assert moved == total, "host end stalled at %d of %d bytes" % (moved, total)
        assert res["status"] == device_lib.OK and res["ret"] == total, res
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


def test_prepared_batches_and_the_claim(gpu):
    """A launched batch is a host op until its results are collected; a batch prepared before the claim cannot be
    launched on the claimed end; the peer's batches keep working (their kernels publish under the mirror locks)."""
    pkg, L = gpu, gpu.lib()
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 4096)
    a, b = pkg.connected_pair("pb-a", "pb-b")
    dev = L.b200_mem_alloc_device(4096)
    out = L.b200_mem_alloc_device(4096)
    sl = pkg.make_slices([(dev, 100)])
    bs = pkg.Batch("send", [(a, sl, 1, 0)], pkg.ONE_CALL)
    br = pkg.Batch("recv", [(b, out, 4096)], pkg.UNTIL_BLOCKED)
    bs.launch()
    with pytest.raises(RuntimeError, match="in flight"):
        a.device_claim()
    assert bs.results() == [100]
    a.device_claim()
    with pytest.raises(RuntimeError, match="device-owned"):
        bs.launch()
    br.launch()  # the peer end: prepared before the claim, launched after it
    assert br.results() == [100] and not b.has_message()
    a.device_release()
    bs.launch()
    assert bs.results() == [100] and b.has_message() and b.readable() == 100
    bs.destroy()
    br.destroy()
    for p in (a, b):
        p.disconnect()
        p.putback()
    L.b200_mem_free_device(dev)
    L.b200_mem_free_device(out)
