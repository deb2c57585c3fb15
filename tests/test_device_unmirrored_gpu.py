"""GPU: device claims without a host mirror (b200_pair_device_claim_ex with B200_CLAIM_UNMIRRORED).

Twins: one connection claimed mirrored and one claimed unmirrored run the same golden and random traces with warp,
block and cluster (K = 2, 4) calls, per-slice, coalesced and stamped; the records (return values, calls, cursors,
credit, readiness, delivered bytes, ring images) must agree with each other and with the CPU models, and the mirror
bytes of every unmirrored end must stay those the claim left (tests/unmirrored_lib.py).  Then: a host-driven peer with
and without the service, mirrored and unmirrored ends mixed on one connection, no host write through polling, status,
writable and a device Disconnect, the release finishing that Disconnect, a host peer's Disconnect during the claim,
the claim's refusals, and an unmirrored end on the CUDA-IPC wire with and without the service."""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import coalesce_lib
import device_lib
import device_poll_lib as dpl
import stamp_lib
import test_coalesce_gpu
import test_gpu_parity
import test_stamp_gpu
import trace
from unmirrored_lib import UnmirroredDeviceEngine, engines, mirror_bytes, writable_size

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "traces.json")))
_compare = test_gpu_parity._compare
KINDS = ["warp", "block", "cluster2", "cluster4"]


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
    dpl.load()
    dpl.Runner(gpu)
    device_lib.Runner(gpu)  # the drivers' kernels are loaded before the resident kernels start
    L = gpu.lib()
    assert L.b200_service_start(4) == 0, gpu.last_error()
    yield gpu
    L.b200_service_stop()


# ---- twins against the golden records and the models

@pytest.mark.parametrize("kind", KINDS)
def test_twins_golden(gpu, kind):
    for name, t in sorted(GOLDEN["traces"].items()):
        mir, unm = engines(gpu, kind, "device", 3)
        want = trace.run_trace(mir, t["cap"], _ops(t["ops"]), GOLDEN["max_sge"])
        got = trace.run_trace(unm, t["cap"], _ops(t["ops"]), GOLDEN["max_sge"])
        _compare(got, want, "%s unmirrored vs mirrored, golden %s" % (kind, name))
        _compare(got, t["records"], "%s unmirrored, golden %s" % (kind, name))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", range(2))
def test_twins_random_vs_oracle(gpu, oracle, kind, seed):
    rng = np.random.default_rng(7100 + seed)
    cap = [1024, 65536][seed]
    ops = test_gpu_parity._random_ops(rng, cap, 60)
    mem, mis = [("device", 5), ("pinned", 9)][seed]
    mir, unm = engines(gpu, kind, mem, mis)
    got = trace.run_trace(unm, cap, ops)
    _compare(got, trace.run_trace(mir, cap, ops), "%s twins seed %d" % (kind, seed))
    _compare(got, trace.run_trace(oracle, cap, ops), "%s unmirrored vs model seed %d" % (kind, seed))


@pytest.mark.parametrize("kind", KINDS)
def test_twins_coalesced_vs_model(gpu, co, kind):
    rng = np.random.default_rng(7200)
    cap = 4096
    ops = test_coalesce_gpu._random_ops(rng, cap, 50)
    mir, unm = engines(gpu, kind, "device", 3, config={"B200_SEND_COALESCE": 1})
    got = trace.run_trace(unm, cap, ops)
    _compare(got, trace.run_trace(mir, cap, ops), "%s coalesced twins" % kind)
    _compare(got, trace.run_trace(co, cap, ops), "%s coalesced unmirrored vs model" % kind)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("coalesced", [False, True])
def test_twins_stamped_vs_model(gpu, so, soc, kind, coalesced):
    rng = np.random.default_rng(7300 + int(coalesced))
    cap = 4096
    ops = test_stamp_gpu._random_ops(rng, cap, 60)
    for eng in engines(gpu, kind, "device", 3, config={"B200_RING_STAMPED": 1, "B200_SEND_COALESCE": int(coalesced)}):
        test_stamp_gpu._replay(eng, soc if coalesced else so, cap, ops)


# ---- mixed ends

@pytest.mark.parametrize("drive", [("tx",), ("rx",)])
def test_host_driven_peer(gpu, oracle, drive):
    """The host end's answers, readiness and writable come from its own mirror, published by the unmirrored end's
    device calls: they follow the model."""
    for seed, cap in enumerate((1024, 65536)):
        ops = test_gpu_parity._random_ops(np.random.default_rng(7400 + seed), cap, 60)
        got = trace.run_trace(UnmirroredDeviceEngine(gpu, "device", 1, drive=drive), cap, ops)
        _compare(got, trace.run_trace(oracle, cap, ops), "unmirrored %s, host peer, cap %d" % (drive, cap))


@pytest.mark.parametrize("drive", [("tx",), ("rx",), ("tx", "rx")])
def test_under_the_service(svc, oracle, drive):
    for seed, cap in enumerate((1024, 65536)):
        ops = test_gpu_parity._random_ops(np.random.default_rng(7500 + seed), cap, 60)
        ops += [op for k in range(10) for op in (("send", [9, 5, 100 + 37 * k], 40 + k, 0), ("recv", 1 << 16))]
        got = trace.run_trace(UnmirroredDeviceEngine(svc, "pinned", 3, drive=drive), cap, ops)
        _compare(got, trace.run_trace(oracle, cap, ops), "service, unmirrored %s, cap %d" % (drive, cap))


@pytest.mark.parametrize("unmirrored", [("tx",), ("rx",)])
@pytest.mark.parametrize("kind", ["warp", "block"])
def test_mirrored_and_unmirrored_ends_on_one_connection(gpu, oracle, kind, unmirrored):
    cap = 4096
    ops = test_gpu_parity._random_ops(np.random.default_rng(7600), cap, 60)
    _, unm = engines(gpu, kind, "device", 0, unmirrored=unmirrored)
    _compare(trace.run_trace(unm, cap, ops), trace.run_trace(oracle, cap, ops), "%s, unmirrored %s" % (kind, unmirrored))


# ---- no host writes, the release, the claim's rules

def _dev_buf(L, data):
    p = L.b200_mem_alloc_device(max(1, data.size))
    assert L.b200_memcpy(p, data.ctypes.data, data.size, 0, None) == 0 and L.b200_stream_sync(None) == 0
    return p


@pytest.mark.parametrize("service", [False, True])
def test_no_host_writes_then_release_finishes_the_disconnect(gpu, service):
    """An unmirrored device end streams both ways with a host-driven peer, polls, asks status and writable and
    disconnects: its PairMirror bytes never change until the release, while the peer's readiness and status follow.
    The release publishes and finishes the Disconnect; Init, Connect and putback work afterwards."""
    pkg, L = gpu, gpu.lib()
    R = dpl.Runner(pkg)
    if service:
        assert L.b200_service_start(4) == 0, pkg.last_error()
    bufs = []
    try:
        pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 4096)
        a, b = pkg.connected_pair("nhw-a", "nhw-b")
        h = a.device_claim(mirrored=False)
        snap = mirror_bytes(h)
        assert a.device_owned()
        msg = np.arange(700, dtype=np.uint8)
        src = _dev_buf(L, msg)
        bufs.append(src)
        slp = L.b200_mem_alloc_host(16)
        sl = (pkg.Slice * 1).from_address(slp)
        sl[0].ptr, sl[0].len = src, msg.size
        dst = L.b200_mem_alloc_device(4096)
        bufs.append(dst)
        for k in range(8):  # laps the 4 KiB ring: credit flows both ways
            assert R.one(h, kind=dpl.SEND, slices=slp, n=1) == msg.size
            assert mirror_bytes(h) == snap
            assert b.has_message() == 1 and b.readable() == msg.size  # the peer's mirror is published
            assert np.array_equal(b.recv(4096), msg)
            assert b.send([msg[:100 + k]]) == 100 + k
            c, ev, ready = R.poll([h])
            assert c == 1 and ev[0] == dpl.EV_READABLE
            assert R.one(h, kind=dpl.RECV, dst=dst, cap=4096) == 100 + k
            assert R.one(h, kind=dpl.STATUS) == dpl.CONNECTED
            st = a.state()
            assert R.one(h, kind=dpl.WRITABLE) == writable_size(4096, st["credit_remote_head"], st["remote_tail"])
            assert mirror_bytes(h) == snap
        assert R.one(h, kind=dpl.DISCONNECT) == 1
        assert mirror_bytes(h) == snap
        assert b.status() == dpl.HALF_CLOSED
        assert a.status() == dpl.CONNECTED  # frozen until the release
        a.device_release()
        assert not a.device_owned() and a.status() == dpl.DISCONNECTED
        assert mirror_bytes(h) != snap
        b.disconnect()
        L.b200_pair_init(a.h)
        assert a.status() == dpl.INITIALIZED
        c = pkg.Pair("nhw-c")
        assert a.connect(c.address()) and c.connect(a.address())
        assert a.status() == dpl.CONNECTED and c.status() == dpl.CONNECTED
        assert c.send([msg]) == msg.size and np.array_equal(a.recv(4096), msg)
        for p in (a, b, c):
            p.disconnect()
            p.putback()
        L.b200_mem_free_host(slp)
    finally:
        for p in bufs:
            L.b200_mem_free_device(p)
        if service:
            L.b200_service_stop()
        R.close()


def test_both_ends_unmirrored_write_no_mirror(gpu):
    """Two device warps stream through one connection claimed unmirrored at both ends: neither mirror changes; after
    the release both mirrors equal those of the same stream run with mirrored claims."""
    pkg, L = gpu, gpu.lib()
    D = device_lib.Runner(pkg)
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 1 << 16)
    data = np.random.default_rng(7700).integers(0, 256, 1 << 20, dtype=np.uint8)
    src = _dev_buf(L, data)
    dst = L.b200_mem_alloc_device(data.size)
    slp = L.b200_mem_alloc_host(16)
    sl = (pkg.Slice * 1).from_address(slp)
    sl[0].ptr, sl[0].len = src, data.size
    mirrors = []
    try:
        for mirrored in (True, False):
            a, b = pkg.connected_pair("bu-a%d" % mirrored, "bu-b%d" % mirrored)
            ha, hb = a.device_claim(mirrored), b.device_claim(mirrored)
            sa, sb = mirror_bytes(ha), mirror_bytes(hb)
            res = D.run([ha, hb], [[dict(kind=device_lib.STREAM_SEND, pair=0, slices=slp, n=1)],
                                   [dict(kind=device_lib.STREAM_RECV, pair=1, dst=dst, n=data.size)]], budget_s=60.0)
            assert all(o[0]["status"] == device_lib.OK and o[0]["ret"] == data.size for o in res), res
            got = np.zeros_like(data)
            assert L.b200_memcpy(got.ctypes.data, dst, data.size, 1, None) == 0 and L.b200_stream_sync(None) == 0
            assert np.array_equal(got, data)
            if not mirrored:
                assert mirror_bytes(ha) == sa and mirror_bytes(hb) == sb
            else:
                assert mirror_bytes(ha) != sa and mirror_bytes(hb) != sb
            a.device_release()
            b.device_release()
            mirrors.append((mirror_bytes(ha), mirror_bytes(hb), a.state(), b.state()))
            for p in (a, b):
                p.disconnect()
                p.putback()
        assert mirrors[0] == mirrors[1]
    finally:
        L.b200_mem_free_device(src)
        L.b200_mem_free_device(dst)
        L.b200_mem_free_host(slp)


def test_claim_refused_while_the_peer_has_a_host_op_in_flight(svc):
    pkg, L = svc, svc.lib()
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 4096)
    a, b = pkg.connected_pair("pin-a", "pin-b")
    dst = L.b200_mem_alloc_host(4096)
    again, n = C.c_int(0), C.c_uint64(0)
    op = L.b200_pair_post_recv(b.h, dst, 4096, 0, C.byref(again))
    assert op, pkg.last_error()
    with pytest.raises(RuntimeError, match="peer end"):
        a.device_claim(mirrored=False)
    assert not a.device_owned()
    a.device_claim()  # a mirrored claim does not care about the peer's ops
    a.device_release()
    assert L.b200_async_poll(op, C.byref(n)) == 1 and n.value == 0
    a.device_claim(mirrored=False)
    a.device_release()
    for p in (a, b):
        p.disconnect()
        p.putback()
    L.b200_mem_free_host(dst)


def test_batches_refuse_an_unmirrored_end(gpu):
    pkg, L = gpu, gpu.lib()
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 4096)
    a, b = pkg.connected_pair("br-a", "br-b")
    a.device_claim(mirrored=False)
    src = _dev_buf(L, np.ones(64, np.uint8))
    try:
        sl = pkg.make_slices([(src, 64)])
        ops = (pkg.SendOp * 1)()
        ops[0].pair, ops[0].slices, ops[0].nslices, ops[0].byte_idx = a.h, sl, 1, 0
        acc = (C.c_uint64 * 1)()
        for flags in (0, 2 << 4):  # one CTA per op, and B200_BATCH_CLUSTER(3)
            assert L.b200_pairs_send(ops, 1, flags, acc, None) == -1
            assert "device-owned" in pkg.last_error()
        assert a.send([np.ones(8, np.uint8)]) == 0 and "device-owned" in a.error()
    finally:
        a.device_release()
        for p in (a, b):
            p.disconnect()
            p.putback()
        L.b200_mem_free_device(src)


def test_host_peer_disconnects_during_the_claim(gpu):
    """The host peer's Disconnect writes the unmirrored end's credit block and not its mirror: the mirror bytes and the
    end's host status stay as the claim left them, the device sees HALF_CLOSED at once, and the release publishes the
    peer_exit: b200_pair_status says HALF_CLOSED."""
    pkg, L = gpu, gpu.lib()
    R = dpl.Runner(pkg)
    try:
        pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 4096)
        a, b = pkg.connected_pair("pdc-a", "pdc-b")
        assert b.send([np.arange(300, dtype=np.uint8)]) == 300
        h = a.device_claim(mirrored=False)
        snap = mirror_bytes(h)
        b.disconnect()
        assert mirror_bytes(h) == snap
        assert a.status() == dpl.CONNECTED  # frozen until the release
        assert R.one(h, kind=dpl.STATUS) == dpl.HALF_CLOSED
        assert a.state()["peer_exit"] == 1
        a.device_release()
        assert mirror_bytes(h) != snap
        assert a.status() == dpl.HALF_CLOSED
        assert np.frombuffer(mirror_bytes(h), np.uint32)[15] == 1  # PairMirror::peer_exit
        assert np.array_equal(a.recv(4096), np.arange(300, dtype=np.uint8))  # what was sent before the close
        for p in (a, b):
            p.disconnect()
            p.putback()
    finally:
        R.close()


@pytest.mark.parametrize("service", [False, True])
def test_unmirrored_end_over_the_ipc_wire(service):
    """An unmirrored device end streams 3 x 1 MiB through a 256 KiB ring into another process, polls for and receives
    that process's frame and disconnects.  Its mirror bytes and its host queries (each of which scans the end when the
    service is stopped; the device poller scans it when it runs) stay as the claim left them; the release publishes."""
    with tempfile.TemporaryDirectory() as d:
        procs = [subprocess.Popen([sys.executable, os.path.join(HERE, "device_unmirrored_ipc_worker.py"), role, "0", d,
                                   "256", str(1 << 20), "3", str(int(service))], stdout=subprocess.PIPE,
                                  stderr=subprocess.STDOUT, text=True)
                 for role in ("server", "client")]
        outs = [p.communicate(timeout=500)[0] for p in procs]
        assert all(p.returncode == 0 for p in procs), "\n".join(outs)
        cli, srv = [json.load(open(os.path.join(d, r + ".json"))) for r in ("client", "server")]
    assert cli["ok"] and cli["hello_seen"] and cli["hello_ok"] and cli["closed"] == 1, cli
    assert all(cli["frozen"]) and len(cli["frozen"]) == 7, cli
    assert cli["at_claim"][0] == dpl.CONNECTED, cli
    assert cli["republished"] and cli["released"], cli
    assert srv["ok"] and srv["half_closed"] and srv["drained"] == 3 << 20, srv
