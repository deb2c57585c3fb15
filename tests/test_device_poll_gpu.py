"""GPU: the device-side poll loop (include/b200_device.cuh: b200_warp_poll, b200_warp_status, b200_warp_writable,
b200_warp_disconnect) driven from user kernels (tests/native/device_poll.cu).

b200_warp_poll answers what b200_poller_scan answers for the same ends in the same state, in every framing mode;
status and writable follow b200_pair_status / b200_pair_writable through random traces; a device Disconnect plus the
release is observable for observable a host Disconnect; one polling server warp serves 64 connections and closes them;
and the CUDA-IPC wire carries a device end's stream, its close and its credit."""
import contextlib
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import device_poll_lib as dpl
from device_poll_lib import Runner

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
HERE = os.path.dirname(os.path.abspath(__file__))
MODES = {"reference": {}, "coalesced": {"B200_SEND_COALESCE": 1}, "stamped": {"B200_RING_STAMPED": 1}}


def _pairs(pkg, n, cap, config, tag):
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", cap)
    pkg.config_set("GRPC_RDMA_MAX_SGE", 30)
    for k, v in config.items():
        pkg.config_set(k, v)
    try:
        return [pkg.connected_pair("%s-a%d" % (tag, i), "%s-b%d" % (tag, i)) for i in range(n)]
    finally:
        for k in config:
            pkg.config_set(k, 0)


def _drop(conns):
    for a, b in conns:
        for p in (a, b):
            p.disconnect()  # (releases a claim first)
            p.putback()


def _host_scan(pkg, pairs):
    arr = (C.c_void_p * max(1, len(pairs)))(*[p.h for p in pairs])
    ev = np.zeros(max(1, len(pairs)), np.uint32)
    cnt = pkg.lib().b200_poller_scan(arr, len(pairs), ev.ctypes.data_as(C.POINTER(C.c_uint32)))
    assert cnt >= 0, pkg.last_error()
    return cnt, ev[:len(pairs)]


class _Payload:
    """pinned source bytes, pinned slice arrays, a pinned destination"""

    def __init__(self, R, nbytes, seed):
        self.R = R
        self.src_p, self.src = R.mem.array("src", np.uint8, nbytes)
        self.src[:] = np.random.default_rng(seed).integers(0, 256, nbytes, dtype=np.uint8)
        self.dst_p, self.dst = R.mem.array("dst", np.uint8, 1 << 16)
        self.k = 0

    def slices(self, lens, off=0):
        """a pinned slice array over consecutive stretches of the source"""
        self.k += 1
        sp, arr = self.R.mem.array("sl%d" % self.k, np.uint64, 2 * len(lens))
        for i, n in enumerate(lens):
            arr[2 * i], arr[2 * i + 1] = self.src_p + off, n
            off += n
        return sp


@contextlib.contextmanager
def _service(pkg, on):
    if not on:
        yield
        return
    L = pkg.lib()
    assert L.b200_service_start(4) == 0, pkg.last_error()
    try:
        yield
    finally:
        L.b200_service_stop()


# ---- 1. poll parity with the host poller

EMPTY, FRAME, PARTLY_READ, NO_CREDIT, PEER_LEFT, TORN = range(6)


@pytest.mark.parametrize("mode", sorted(MODES))
def test_poll_matches_the_host_poller(gpu, mode):
    R = Runner(gpu)
    cap = 4096
    conns = _pairs(gpu, 64, cap, MODES[mode], "pp-" + mode)
    try:
        handles = [h for a, b in conns for h in (a.device_claim(), b.device_claim())]
        ends = [p for a, b in conns for p in (a, b)]
        P = _Payload(R, 4 * cap, 11)
        lists = []
        for i in range(len(conns)):
            a, b, s = 2 * i, 2 * i + 1, i % 6
            ops = []
            if s == FRAME:
                ops = [dict(kind=dpl.SEND, pair=a, slices=P.slices([100 + i]), n=1)]
            elif s == PARTLY_READ:
                ops = [dict(kind=dpl.SEND, pair=a, slices=P.slices([1000]), n=1),
                       dict(kind=dpl.RECV, pair=b, dst=P.dst_p + 1024 * (i % 32), cap=300)]
            elif s == NO_CREDIT:
                ops = [dict(kind=dpl.SEND_ALL, pair=a, slices=P.slices([3 * cap]), n=1)]
            elif s == PEER_LEFT:
                ops = [dict(kind=dpl.DISCONNECT, pair=b)]
            elif s == TORN:
                ops = [dict(kind=dpl.TORN, pair=a, n=200)]
            lists.append(ops)
        res = R.run(handles, lists)
        assert all(r["status"] == dpl.OK for lst in res for r in lst), res
        hc, hev = _host_scan(gpu, ends)
        c, ev, rd = R.poll(handles)
        assert (c, ev.tolist()) == (hc, hev.tolist())
        assert rd.tolist() == np.nonzero(hev)[0].tolist()
        # the states are the ones meant: every rule of the scan has a witness
        R_, W_ = dpl.EV_READABLE, dpl.EV_WRITABLE
        want = {EMPTY: (0, 0), FRAME: (0, R_), PARTLY_READ: (0, R_), NO_CREDIT: (W_, R_), PEER_LEFT: (R_, 0),
                TORN: (0, 0 if mode == "stamped" else R_)}
        for i in range(len(conns)):
            assert (ev[2 * i], ev[2 * i + 1]) == want[i % 6], (mode, i, ev[2 * i], ev[2 * i + 1])
        # any n, handles repeated; NULL events / ready
        for n in (0, 1, 31, 32, 33, 97, 4096):
            idx = [k % len(handles) for k in range(n)]
            hs = [handles[k] for k in idx]
            c, ev, rd = R.poll(hs)
            if n == 0:
                assert c == 0 and rd.size == 0
                continue
            hc, hev = _host_scan(gpu, [ends[k] for k in idx])
            assert c == hc and ev.tolist() == hev.tolist(), n
            assert rd.tolist() == np.nonzero(hev)[0].tolist() and all(np.diff(rd) > 0), n
            c2, _, rd2 = R.poll(hs, with_events=False)
            c3, ev3, _ = R.poll(hs, with_ready=False)
            c4, _, _ = R.poll(hs, with_events=False, with_ready=False)
            assert c2 == c3 == c4 == c and rd2.tolist() == rd.tolist() and ev3.tolist() == ev.tolist(), n
    finally:
        _drop(conns)
        R.close()


# ---- 2. status and writable against the host answers

@pytest.mark.parametrize("svc", [False, True])
def test_status_and_writable_follow_the_host(gpu, svc):
    R = Runner(gpu)
    with _service(gpu, svc):
        for seed, cap in enumerate((1024, 4096, 65536)):
            rng = np.random.default_rng(5100 + seed + 10 * svc)
            (a, b), = conns = _pairs(gpu, 1, cap, {}, "sw%d%d" % (svc, seed))
            try:
                ha = a.device_claim()
                P = _Payload(R, 3 * cap + 4096, seed)

                def check(what):
                    hs, hw = a.status(), a.writable()  # (the host calls first: they settle an owed Retire)
                    ds, dw = R.one(ha, kind=dpl.STATUS), R.one(ha, kind=dpl.WRITABLE)
                    assert (ds, dw) == (hs, hw), (what, ds, dw, hs, hw)

                check("connected")
                for step in range(60):
                    op = int(rng.integers(4))
                    if op == 0:
                        lens = [int(x) for x in rng.integers(1, cap // 2, int(rng.integers(1, 4)))]
                        R.one(ha, kind=dpl.SEND, slices=P.slices(lens), n=len(lens))
                    elif op == 1:
                        b.recv(int(rng.integers(1, cap)))
                    elif op == 2:
                        b.send([rng.integers(0, 256, int(rng.integers(1, cap // 2)), dtype=np.uint8)])
                    else:
                        R.one(ha, kind=dpl.RECV, dst=P.dst_p, cap=int(rng.integers(1, cap)))
                    check("step %d op %d" % (step, op))
                b.disconnect()
                check("peer left")
                assert a.status() == dpl.HALF_CLOSED
            finally:
                _drop(conns)
    R.close()


# ---- 3. a device Disconnect is a host Disconnect

def _close_run(pkg, R, mode, peer, how, tag):
    L = pkg.lib()
    (c, p), = _pairs(pkg, 1, 4096, MODES[mode], tag)
    P = _Payload(R, 8192, 7)
    hc = c.device_claim()
    hp = p.device_claim() if peer == "device" else None
    rng = np.random.default_rng(77)
    back = [rng.integers(0, 256, n, dtype=np.uint8) for n in (300, 170)]
    # frames in flight both ways, a frame read in part on each side
    assert R.one(hc, kind=dpl.SEND, slices=P.slices([100, 200, 300]), n=3) == 600
    if hp:
        sp = P.slices([300, 170], off=1000)
        P.src[1000:1300], P.src[1300:1470] = back
        assert R.one(hp, kind=dpl.SEND, slices=sp, n=2) == 470
        assert R.one(hp, kind=dpl.RECV, dst=P.dst_p, cap=50) == 50
    else:
        assert p.send(back) == 470
        assert p.recv(50).size == 50
    assert R.one(hc, kind=dpl.RECV, dst=P.dst_p, cap=30) == 30
    obs = {}
    if how == "host":
        c.disconnect()
    else:
        assert R.one(hc, kind=dpl.DISCONNECT) == 1
        assert c.status() == dpl.DISCONNECTED and c.device_owned()  # before the release
        before = (c.state(), p.state(), p.status(), c.ring_image().tobytes(), p.ring_image().tobytes())
        assert R.one(hc, kind=dpl.DISCONNECT) == 0  # a second close changes nothing
        assert R.one(hc, kind=dpl.SEND, slices=P.slices([10]), n=1) == 0
        assert R.one(hc, kind=dpl.RECV, dst=P.dst_p, cap=4096) == 0
        assert R.one(hc, kind=dpl.STATUS) == dpl.DISCONNECTED
        assert before == (c.state(), p.state(), p.status(), c.ring_image().tobytes(), p.ring_image().tobytes())
        c.device_release()
    obs["peer_status"] = p.status()
    obs["peer_state"] = p.state()
    obs["rings"] = (p.ring_image().tobytes(), c.ring_image().tobytes())
    obs["scan"] = [int(x) for x in _host_scan(pkg, [p, c])[1]]
    drained = []
    for _ in range(64):
        if hp:
            n = R.one(hp, kind=dpl.RECV, dst=P.dst_p, cap=4096)
            got = P.dst[:n].copy()
        else:
            got = p.recv(4096)
        if got.size == 0:
            break
        drained.append(got.tobytes())
    obs["drained"] = drained
    if hp:
        obs["send"] = R.one(hp, kind=dpl.SEND, slices=P.slices([10]), n=1)
    else:
        obs["send"] = (p.send([np.ones(10, np.uint8)]), p.error())
    obs["peer_after"] = (p.status(), p.state())
    obs["closed"] = (c.status(), c.state(), c.device_owned())
    if how == "device":  # b200_pair_disconnect after the release writes nothing to the peer
        st = p.state()
        c.disconnect()
        assert p.state() == st and c.status() == dpl.DISCONNECTED
    # the pair lives on: Init, Connect, traffic
    if hp:
        p.device_release()
    p.disconnect()
    for x in (c, p):
        L.b200_pair_init(x.h)
        assert x.status() == dpl.INITIALIZED, x.error()
    assert c.connect(p.address()) and p.connect(c.address())
    msg = rng.integers(0, 256, 999, dtype=np.uint8)
    assert c.send([msg]) == 999 and np.array_equal(p.recv(4096), msg)
    assert p.send([msg[:5]]) == 5 and np.array_equal(c.recv(4096), msg[:5])
    _drop([(c, p)])
    return obs


@pytest.mark.parametrize("peer", ["host", "service", "device"])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_device_disconnect_is_a_host_disconnect(gpu, mode, peer):
    R = Runner(gpu)
    with _service(gpu, peer == "service"):
        host = _close_run(gpu, R, mode, peer, "host", "dh-%s-%s" % (mode, peer))
        dev = _close_run(gpu, R, mode, peer, "device", "dd-%s-%s" % (mode, peer))
    R.close()
    for k in host:
        assert host[k] == dev[k], (k, host[k] if k != "rings" else "", dev[k] if k != "rings" else "")
    assert host["peer_status"] == dpl.HALF_CLOSED and host["scan"] == [dpl.EV_READABLE, 0]
    assert sum(len(x) for x in host["drained"]) == 600 - 50  # what the closed end sent, less what was read before


# ---- 4. a device server

def _serve(pkg, R, n, rounds, msg, device_clients, tag):
    L, D = pkg.lib(), R.D
    conns = _pairs(pkg, n, 16384, {}, tag)
    bufs = []

    def dev(nbytes):
        p = L.b200_mem_alloc_device(nbytes)
        assert p, pkg.last_error()
        bufs.append(p)
        return p

    try:
        srv = R.handles("srv", [a.device_claim() for a, b in conns])
        cli = R.handles("cli", [b.device_claim() for a, b in conns]) if device_clients else None
        state = dev(12 * n)
        zeros = np.zeros(3 * n, np.uint32)
        assert L.b200_memcpy(state, zeros.ctypes.data, zeros.nbytes, 0, None) == 0 and L.b200_stream_sync(None) == 0
        tp, times = R.mem.array("times", np.uint64, n * rounds)
        op, out = R.mem.array("out", np.uint64, 4 * n + 4)
        out[:] = 0
        s = dpl.DpServe(srv=srv, cli=cli, n=n, rounds=rounds, msg=msg, mode=0, sbuf=dev(n * msg),
                        cbuf=dev(2 * n * msg), state=state, times=tp, out=op, budget_ns=int(120e9),
                        max_iters=1 << 40)
        assert D.dp_serve_launch(C.byref(s)) == 0, D.dp_error().decode()
        if not device_clients:  # host clients: one request per connection in flight, every reply checked
            rng = np.random.default_rng(900)
            bad = 0
            for r in range(rounds):
                reqs = [rng.integers(0, 256, msg, dtype=np.uint8) for _ in range(n)]
                for (a, b), q in zip(conns, reqs):
                    sent = 0
                    for _ in range(100000):
                        sent += b.send([q[sent:]])
                        if sent == msg:
                            break
                    assert sent == msg
                for (a, b), q in zip(conns, reqs):
                    got = []
                    for _ in range(100000):
                        got.append(b.recv(msg - sum(x.size for x in got)))
                        if sum(x.size for x in got) == msg:
                            break
                    bad += not np.array_equal(np.concatenate(got), q)
            assert bad == 0
            for a, b in conns:
                for _ in range(100000):
                    if b.status() == dpl.HALF_CLOSED:
                        break
                assert b.status() == dpl.HALF_CLOSED
        assert D.dp_wait() == 0, D.dp_error().decode()
        assert out[4 * n] == dpl.OK and out[4 * n + 1] == n, out[4 * n:].tolist()
        if device_clients:
            per = out[:4 * n].reshape(n, 4)
            assert (per[:, 0] == dpl.OK).all(), per.tolist()
            assert (per[:, 1] == 0).all(), "replies differ from their requests"
            assert (per[:, 2] == rounds).all() and (per[:, 3] == dpl.HALF_CLOSED).all(), per.tolist()
            assert (times > 0).all()
            for a, b in conns:
                assert b.status() == dpl.HALF_CLOSED
        for a, b in conns:
            assert a.status() == dpl.DISCONNECTED
        return out[4 * n + 2], out[4 * n + 3]
    finally:
        _drop(conns)
        for p in bufs:
            L.b200_mem_free_device(p)


def test_device_server_with_device_clients(gpu):
    R = Runner(gpu)
    scans, empty = _serve(gpu, R, 64, 100, 1024, True, "ds")
    assert scans > empty
    R.close()


def test_device_server_with_host_clients_under_the_service(gpu):
    R = Runner(gpu)
    with _service(gpu, True):
        _serve(gpu, R, 64, 100, 1024, False, "dsh")
    R.close()


# ---- 5. the CUDA-IPC wire, two processes on one GPU

def test_device_end_over_the_ipc_wire():
    """A device end streams 3 x 1 MiB through a 256 KiB ring into the other process (it needs the credit that comes
    back over the wire), sees the other process's frame with b200_warp_poll, receives it, and disconnects; the other
    process drains everything and sees HALF_CLOSED."""
    with tempfile.TemporaryDirectory() as d:
        procs = [subprocess.Popen([sys.executable, os.path.join(HERE, "device_poll_ipc_worker.py"), role, "0", d,
                                   "256", str(1 << 20), "3"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                  text=True)
                 for role in ("server", "client")]
        outs = [p.communicate(timeout=500)[0] for p in procs]
        assert all(p.returncode == 0 for p in procs), "\n".join(outs)
        cli, srv = [json.load(open(os.path.join(d, r + ".json"))) for r in ("client", "server")]
    assert cli["ok"] and cli["hello_seen"] and cli["hello_ok"] and cli["closed"] == 1, cli
    assert cli["status_before_release"] == dpl.DISCONNECTED and cli["released"], cli
    assert srv["ok"] and srv["half_closed"] and srv["drained"] == 3 << 20, srv
    assert srv["scan"] == [dpl.EV_READABLE], srv
