"""GPU: parking a device ready set (b200_warp_ready_park / b200_ready_set_park, DESIGN.md §13 "Parking"), driven by
tests/native/device_ready_park.cu: an echo server whose last idle warp parks the set and exits, and device client
warps.
  - a host park of an empty set, then a host Send: one ring, a readable fd, and a server that answers the request;
  - 64 device client warps sending at once to a parked set: exactly one ring;
  - a park over a non-empty queue returns 1 and rings nothing;
  - an add and a host Disconnect of a member's peer ring a parked set, a release of a member does not;
  - launch on demand, per framing mode, with and without the service: a host loop polls the set's fd and launches a
    server of 1 or 8 warps; bursts of device clients, host single calls, batches and host Disconnects with idle gaps
    between them.  Every request is answered once with its bytes; rings never exceed the parks that returned 0; at
    the end the set is parked, its queue empty and its fd not readable;
  - a set that is never parked never rings.
Each case runs in a process of its own (tests/device_ready_park_worker.py)."""
import contextlib
import ctypes as C
import os
import select
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

import device_ready_lib as drl
import device_ready_park_lib as dpl

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1500)]
HERE = os.path.dirname(os.path.abspath(__file__))
MODES = {"reference": {}, "coalesced": {"B200_SEND_COALESCE": 1}, "stamped": {"B200_RING_STAMPED": 1}}
MSG = 256


def _pairs(pkg, n, config, tag, cap=1 << 14):
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", cap)
    for k, v in config.items():
        pkg.config_set(k, v)
    try:
        return [pkg.connected_pair("%s-a%d" % (tag, i), "%s-b%d" % (tag, i)) for i in range(n)]
    finally:
        for k in config:
            pkg.config_set(k, 0)


@contextlib.contextmanager
def _service(pkg, on):
    if on:
        assert pkg.lib().b200_service_start(4) == 0, pkg.last_error()
    try:
        yield
    finally:
        if on:
            pkg.lib().b200_service_stop()


def readable(fd, timeout_ms=0):
    p = select.poll()
    p.register(fd, select.POLLIN)
    return bool(p.poll(timeout_ms))


def wait_for(cond, seconds=10.0):
    t_end = time.time() + seconds
    while time.time() < t_end:
        if cond():
            return True
        time.sleep(0.002)
    return cond()


def host_request(pair, src, conn, rnd):
    """one request through a host single call; returns the reply once it is all there"""
    req = dpl.pattern(conn, rnd, MSG)
    src[:MSG] = req
    assert pair.send_raw([(src.ctypes.data, MSG)]) == MSG
    assert np.array_equal(recv_all(pair), req), ("reply of host client", conn, rnd)


def recv_all(pair):
    """MSG bytes from a host-driven end, polling (30 s at most)"""
    got = []
    t_end = time.time() + 30
    while sum(g.size for g in got) < MSG and time.time() < t_end:
        g = pair.recv(MSG - sum(x.size for x in got))
        if g.size:
            got.append(g)
        else:
            time.sleep(0.0005)
    return np.concatenate(got) if got else np.zeros(0, np.uint8)


class _Rig:
    """n connections whose a ends (claimed) are the members of one set; the first `dev` b ends are claimed by device
    clients, the others are host-driven"""

    def __init__(self, pkg, n, dev, config, tag, mirrored=True):
        self.pkg = pkg
        self.conns = _pairs(pkg, n, config, tag)
        self.mem = drl.Pinned(pkg.lib())
        self.srv_h = [a.device_claim(mirrored=mirrored) for a, b in self.conns]
        self.cli_h = [self.conns[i][1].device_claim() for i in range(dev)]
        self.rs = pkg.ReadySet(n)
        for i, (a, b) in enumerate(self.conns):
            self.rs.add(a, i)
        self.server = dpl.Server(pkg, self.rs, self.srv_h, MSG, self.mem)
        self.clients = dpl.Clients(pkg, self.cli_h, MSG, self.mem) if dev else None
        self.zero_parks = 0
        self.replies = 0

    def serve(self, warps, **kw):
        self.server.launch(warps, **kw)
        r = self.server.wait()
        assert r["status"] == 0, r
        self.replies += r["replies"]
        if not kw.get("no_park"):
            self.zero_parks += 1  # the server exits only once its last warp's park returned 0
        return r

    def close(self):
        for a, b in self.conns:
            for p in (a, b):
                if p.device_owned():
                    p.device_release()
        self.rs.destroy()
        self.server.free()
        if self.clients:
            self.clients.free()
        self.mem.free()
        for a, b in self.conns:
            for p in (a, b):
                p.disconnect()
                p.putback()


def host_park_then_send(pkg):
    R = _Rig(pkg, 4, 0, {}, "pk1")
    try:
        fd = R.rs.wakeup_fd()
        assert R.rs.park() == 1  # the adds' initial entries are queued
        R.serve(1)
        assert R.rs.park() == 0 and R.rs.rings() == 0
        time.sleep(0.05)
        assert not readable(fd)
        _, src = R.mem.array("src", np.uint8, MSG)
        req = dpl.pattern(2, 0, MSG)
        src[:] = req
        assert R.conns[2][1].send_raw([(src.ctypes.data, MSG)]) == MSG
        assert wait_for(lambda: R.rs.rings() == 1)
        assert readable(fd, 5000)
        R.rs.consume_wakeup()
        assert not readable(fd)
        r = R.serve(1)
        assert r["taken"] >= 1 and r["replies"] == 1, r
        assert np.array_equal(recv_all(R.conns[2][1]), req)
        assert R.rs.rings() == 1
    finally:
        R.close()


def many_clients_one_ring(pkg):
    R = _Rig(pkg, 64, 64, {}, "pk2")
    try:
        fd = R.rs.wakeup_fd()
        R.serve(8)  # the initial entries; ends parked
        assert R.rs.rings() == 0
        R.clients.launch(1)
        assert wait_for(lambda: R.rs.rings() >= 1)
        time.sleep(0.1)  # every client has sent by now
        assert R.rs.rings() == 1
        assert readable(fd, 5000)
        R.rs.consume_wakeup()
        while R.clients.running():
            R.serve(8)
        R.clients.wait(1)
        assert R.replies == 64
        assert R.rs.rings() <= R.zero_parks
    finally:
        R.close()


def park_nonempty(pkg):
    R = _Rig(pkg, 8, 0, {}, "pk3")
    try:
        assert R.rs.park() == 1 and R.rs.park() == 1
        time.sleep(0.05)
        assert R.rs.rings() == 0
        r = R.serve(1)
        assert r["taken"] == 8, r
        assert R.rs.rings() == 0 and R.rs.park() == 0
    finally:
        R.close()


def add_disconnect_release(pkg):
    conns = _pairs(pkg, 3, {}, "pk4")
    mem = drl.Pinned(pkg.lib())
    rs = pkg.ReadySet(4)
    handles = [a.device_claim() for a, b in conns]
    server = dpl.Server(pkg, rs, handles, MSG, mem)
    try:
        fd = rs.wakeup_fd()
        rs.add(conns[0][0], 0)
        server.launch(1)
        assert server.wait()["status"] == 0
        assert rs.rings() == 0
        rs.add(conns[1][0], 1)  # an add to a parked set rings
        assert wait_for(lambda: rs.rings() == 1) and readable(fd, 5000)
        rs.consume_wakeup()
        server.launch(1)
        assert server.wait()["taken"] == 1
        conns[0][1].disconnect()  # a host Disconnect of a member's peer rings
        assert wait_for(lambda: rs.rings() == 2) and readable(fd, 5000)
        rs.consume_wakeup()
        server.launch(1)
        assert server.wait()["status"] == 0
        assert server.closed_flags()[0] == 1
        conns[1][0].device_release()  # a release of a member rings nothing
        time.sleep(0.1)
        assert rs.rings() == 2 and not readable(fd)
        conns[0][0].device_release()
        rs.destroy()  # a parked set can be destroyed
        rs = None
    finally:
        for a, b in conns:
            if a.device_owned():
                a.device_release()
        if rs is not None:
            rs.destroy()
        server.free()
        mem.free()
        for a, b in conns:
            a.disconnect()
            b.disconnect()
            a.putback()
            b.putback()


def launch_on_demand(pkg, mode, service, warps):
    n, dev = 96, 64
    R = _Rig(pkg, n, dev, MODES[mode], "pko-%s-%d-%d" % (mode, service, warps), mirrored=bool(warps % 2))
    L = pkg.lib()
    try:
        with _service(pkg, service):
            fd = R.rs.wakeup_fd()
            if R.rs.park() == 1:
                R.serve(warps)
            else:
                R.zero_parks += 1
            host = list(range(dev, n))
            live = list(host)
            srcs = {i: R.mem.array("hsrc%d" % i, np.uint8, MSG)[1] for i in host}
            rounds = {i: 0 for i in host}
            state = dict(requests=0, done=False, error=None)
            rng = np.random.default_rng(17)

            def traffic():
                try:
                    for burst in range(8):
                        kind = ("device", "single", "batch", "device", "single", "disconnect", "batch", "device")[burst]
                        if kind == "device":
                            R.clients.launch(2)
                            R.clients.wait(2)
                            state["requests"] += 2 * dev
                        elif kind == "single":
                            for i in rng.permutation(live)[:16]:
                                host_request(R.conns[i][1], srcs[i], i, rounds[i])
                                rounds[i] += 1
                                state["requests"] += 1
                        elif kind == "batch":
                            idx = [int(i) for i in rng.permutation(live)[:16]]
                            sl = []
                            ops = (pkg.SendOp * len(idx))()
                            for k, i in enumerate(idx):
                                srcs[i][:] = dpl.pattern(i, rounds[i], MSG)
                                sl.append(pkg.make_slices([(srcs[i].ctypes.data, MSG)]))
                                ops[k].pair, ops[k].slices, ops[k].nslices, ops[k].byte_idx = \
                                    R.conns[i][1].h, sl[-1], 1, 0
                            res = (C.c_uint64 * len(idx))()
                            assert L.b200_pairs_send(ops, len(idx), 0, res, None) == 0, pkg.last_error()
                            assert list(res) == [MSG] * len(idx), list(res)
                            for i in idx:
                                want = dpl.pattern(i, rounds[i], MSG)
                                assert np.array_equal(recv_all(R.conns[i][1]), want), ("batch reply", i)
                                rounds[i] += 1
                                state["requests"] += 1
                        else:
                            for i in live[:4]:
                                R.conns[i][1].disconnect()
                            del live[:4]
                        time.sleep(0.05 + 0.05 * rng.random())  # idle: the server parks and exits
                except Exception as e:  # reported by the main thread
                    state["error"] = e
                finally:
                    state["done"] = True

            t = threading.Thread(target=traffic)
            t.start()
            try:
                quiet = 0
                while quiet < 3:
                    if readable(fd, 20):
                        R.rs.consume_wakeup()
                        R.serve(warps)
                        quiet = 0
                    elif state["done"]:
                        quiet += 1
                    assert R.rs.rings() <= R.zero_parks, (R.rs.rings(), R.zero_parks)
            finally:
                t.join()
            if state["error"] is not None:
                raise state["error"]
            assert R.replies == state["requests"], (R.replies, state["requests"])
            assert R.rs.rings() <= R.zero_parks and R.rs.rings() >= 4
            # the end: parked with an empty queue (a host park finds nothing), and no wakeup pending
            assert R.rs.park() == 0
            time.sleep(0.05)
            assert not readable(fd)
            closed = R.server.closed_flags()
            assert all(closed[i] == 1 for i in host if i not in live)
    finally:
        R.close()


def never_parked(pkg):
    R = _Rig(pkg, 96, 64, {}, "pkn")
    try:
        fd = R.rs.wakeup_fd()
        _, src = R.mem.array("src", np.uint8, MSG)
        for burst in range(4):
            R.clients.launch(2)
            R.server.launch(4, idle_takes=1 << 17, no_park=True)
            for i in range(64, 96, 4):
                host_request(R.conns[i][1], src, i, burst)
            R.clients.wait(2)
            r = R.server.wait()
            assert r["status"] == 0, r
            R.replies += r["replies"]
        assert R.replies == 4 * (2 * 64 + 8)
        assert R.rs.rings() == 0 and not readable(fd)
    finally:
        R.close()


def run_case(pkg, case):
    if case == "host-park":
        host_park_then_send(pkg)
    elif case == "one-ring":
        many_clients_one_ring(pkg)
    elif case == "nonempty":
        park_nonempty(pkg)
    elif case == "add-disconnect-release":
        add_disconnect_release(pkg)
    elif case == "never-parked":
        never_parked(pkg)
    elif case.startswith("demand-"):
        _, mode, svc, warps = case.split("-")
        launch_on_demand(pkg, mode, svc == "svc", int(warps))
    else:
        raise ValueError("unknown case " + case)


# Each case runs in a process of its own, as in test_device_ready_shared_gpu.py: the runtime keeps every pair it
# created, with its eventfd, in a pool; run here the cases would leave the pytest process with eventfds above
# select()'s limit for the tests after them.
def _worker(case):
    out = subprocess.run([sys.executable, os.path.join(HERE, "device_ready_park_worker.py"), case],
                         capture_output=True, text=True, timeout=1400)
    assert out.returncode == 0 and ("case %s ok" % case) in out.stdout, out.stdout[-6000:] + out.stderr[-4000:]


@pytest.mark.parametrize("case", ["host-park", "one-ring", "nonempty", "add-disconnect-release", "never-parked"])
def test_park_cases(pkg, case):
    _worker(case)


@pytest.mark.parametrize("warps", [1, 8])
@pytest.mark.parametrize("service", ["svc", "nosvc"])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_launch_on_demand(pkg, mode, service, warps):
    _worker("demand-%s-%s-%d" % (mode, service, warps))
