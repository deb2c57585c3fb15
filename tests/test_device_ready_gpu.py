"""GPU: device ready sets (b200_ready_set_*, include/b200_device.cuh: b200_warp_ready_take / b200_warp_ready_rearm)
consumed by a user kernel (tests/native/device_ready.cu).

After every step of a trace whose peers are driven by every producer path (host single calls with and without the
service, small and pool-sized, prepared batches with one CTA and with B200_BATCH_CLUSTER(2), b200_pairs_submit, posted
ops, device warp and block calls, host and device Disconnect), a consumer kernel drains the set.  Every member that
was READY before the drain was returned by take or rearm, none is READY after it, no member had two entries queued,
no foreign key came back, and each member received exactly the byte stream its peer's calls accepted."""
import contextlib
import ctypes as C

import numpy as np
import pytest

import device_ready_lib as drl

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
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
            p.disconnect()
            p.putback()


@contextlib.contextmanager
def _service(pkg):
    L = pkg.lib()
    assert L.b200_service_start(4) == 0, pkg.last_error()
    try:
        yield
    finally:
        L.b200_service_stop()


def _check_drain(cons, before, res):
    assert res["status"] == 0, res
    assert res["dups"] == 0 and res["foreign"] == 0, res
    returned = (cons.taken + cons.kept) > 0
    missed = [i for i in range(cons.n) if before[i] and not returned[i]]
    assert not missed, ("ready members not returned", missed)
    after = cons.ready()
    left = [i for i in range(cons.n) if after[i] and not cons.closed[i]]
    assert not left, ("members still ready after the drain", left)


class _Trace:
    """n connections; member i = b end (claimed, mirrored when i is even), its peer = a end, host-driven for even i
    and device-claimed for odd i.  Sources are pinned; accepted bytes advance each connection's stream."""

    def __init__(self, pkg, conns, src_bytes, rcap, seed):
        self.pkg, self.L, self.conns = pkg, pkg.lib(), conns
        self.n = len(conns)
        self.mem = drl.Pinned(self.L)
        self.rng = np.random.default_rng(seed)
        self.src_p, self.src = self.mem.array("src", np.uint8, self.n * src_bytes)
        self.src[:] = self.rng.integers(0, 256, self.src.size, dtype=np.uint8)
        self.sb = src_bytes
        self.off = [0] * self.n
        self.left = [False] * self.n  # the peer has disconnected
        self.members = [b.device_claim(mirrored=(i % 2 == 0)) for i, (a, b) in enumerate(conns)]
        self.peers = [a.device_claim() if i % 2 else None for i, (a, b) in enumerate(conns)]
        self.rs = pkg.ReadySet(self.n)
        for i, (a, b) in enumerate(conns):
            self.rs.add(b, i)
        self.cons = drl.Consumer(pkg, self.rs, self.members, rcap)
        self.k = 0

    def slice_arr(self, i, length):
        self.k += 1
        p, arr = self.mem.array("sl%d" % (self.k % 256), np.uint64, 2)
        arr[0], arr[1] = self.src_p + i * self.sb + self.off[i], length
        return p

    def pick(self, host, count):
        idx = [i for i in range(self.n) if (i % 2 == 0) == host and not self.left[i]]
        self.rng.shuffle(idx)
        return idx[:count]

    def length(self, i, big):
        n = int(self.rng.integers(9000, 20000)) if big else int(self.rng.integers(1, 3000))
        return max(0, min(n, self.sb - self.off[i]))

    def step(self, kind):
        pkg, L = self.pkg, self.L
        if kind in ("warp", "block"):
            ops, idx = [], []
            for i in self.pick(False, 12):
                n = self.length(i, kind == "block")
                if n:
                    ops.append((self.peers[i], self.slice_arr(i, n), 1))
                    idx.append(i)
            rets = drl.device_ops(pkg, drl.WARP_SEND if kind == "warp" else drl.BLOCK_SEND, ops, self.mem)
            for i, r in zip(idx, rets):
                self.off[i] += r
        elif kind == "device-disconnect":
            idx = self.pick(False, 3)
            drl.device_ops(pkg, drl.WARP_DISC, [(self.peers[i], 0, 0) for i in idx], self.mem)
            for i in idx:
                self.left[i] = True
        elif kind == "host-disconnect":
            for i in self.pick(True, 3):
                self.conns[i][0].disconnect()
                self.left[i] = True
        elif kind in ("single", "single-big"):
            for i in self.pick(True, 12):
                n = self.length(i, kind == "single-big")
                if n:
                    self.off[i] += self.conns[i][0].send_raw([(int(self.src_p + i * self.sb + self.off[i]), n)])
        elif kind in ("batch", "batch-cluster"):
            ops, idx = [], []
            for i in self.pick(True, 12):
                n = self.length(i, True)
                if n:
                    ops.append((self.conns[i][0], C.cast(self.slice_arr(i, n), C.POINTER(pkg.Slice)), 1, 0))
                    idx.append(i)
            if ops:
                flags = pkg.UNTIL_BLOCKED | (pkg.cluster_flag(2) if kind == "batch-cluster" else 0)
                b = pkg.Batch("send", ops, flags)
                b.launch()
                for i, r in zip(idx, b.results()):
                    self.off[i] += r
                b.destroy()
        elif kind == "submit":
            idx = [i for i in self.pick(True, 12) if self.length(i, False)]
            so = (pkg.SendOp * max(1, len(idx)))()
            for j, i in enumerate(idx):
                so[j].pair, so[j].nslices, so[j].byte_idx = self.conns[i][0].h, 1, 0
                so[j].slices = C.cast(self.slice_arr(i, self.length(i, False)), C.POINTER(pkg.Slice))
            acc = (C.c_uint64 * max(1, len(idx)))()
            assert L.b200_pairs_submit(so, len(idx), acc, None, 0, None, pkg.ONE_CALL) == 0, pkg.last_error()
            for j, i in enumerate(idx):
                self.off[i] += acc[j]
        elif kind == "posted":
            for i in self.pick(True, 6):
                n = self.length(i, False)
                if not n:
                    continue
                again = C.c_int(0)
                op = L.b200_pair_post_send(self.conns[i][0].h, C.cast(self.slice_arr(i, n), C.POINTER(pkg.Slice)),
                                           1, 0, pkg.ONE_CALL, C.byref(again))
                assert op, (again.value, pkg.last_error())
                got = C.c_uint64(0)
                for _ in range(1 << 22):
                    rc = L.b200_async_poll(op, C.byref(got))
                    if rc != 0:
                        break
                assert rc == 1, pkg.last_error()
                self.off[i] += got.value
        else:
            raise ValueError(kind)

    def check(self):
        before = self.cons.ready()
        res = self.cons.drain()
        _check_drain(self.cons, before, res)
        for i in range(self.n):
            want = self.src[i * self.sb:i * self.sb + self.off[i]]
            assert np.array_equal(self.cons.received(i), want), ("bytes of connection", i)
            if self.left[i]:
                assert self.cons.closed[i] == 1, i

    def close(self):
        for i, (a, b) in enumerate(self.conns):
            b.device_release()
            if self.peers[i] is not None:
                a.device_release()
        self.rs.destroy()
        self.cons.close()
        self.mem.free()


@pytest.mark.parametrize("mode", sorted(MODES))
def test_random_traces(gpu, mode):
    drl.load()
    assert drl.load().dr_prepare() == 0
    conns = _pairs(gpu, 64, 1 << 16, MODES[mode], "rt-" + mode)
    T = None
    try:
        T = _Trace(gpu, conns, 1 << 18, 1 << 18, seed=hash(mode) & 0xFFFF)
        T.check()  # the initial entries of the adds
        for kind in ("single", "batch", "warp", "batch-cluster", "block", "single-big", "warp", "single"):
            T.step(kind)
            T.check()
        with _service(gpu):
            for kind in ("single", "single-big", "submit", "posted", "warp", "block", "submit", "single"):
                T.step(kind)
                T.check()
        for kind in ("host-disconnect", "single", "device-disconnect", "warp"):
            T.step(kind)
            T.check()
        assert sum(T.off) > 0
    finally:
        if T is not None:
            T.close()
        _drop(conns)


def test_credit_wakes_a_blocked_sender(gpu):
    """A member owes its peer more than the ring holds: the consumer's Send blocks (a pending write without credit is
    not READY), and each host Recv of the peer that returns credit queues the member again until all is sent."""
    cap = 4096
    conns = _pairs(gpu, 4, cap, {}, "cw")
    rs = gpu.ReadySet(4)
    cons = None
    try:
        members = [b.device_claim(mirrored=(i % 2 == 0)) for i, (a, b) in enumerate(conns)]
        for i, (a, b) in enumerate(conns):
            rs.add(b, i)
        cons = drl.Consumer(gpu, rs, members, 64, scap=6 * cap)
        cons.sbuf[:] = np.random.default_rng(3).integers(0, 256, cons.sbuf.size, dtype=np.uint8)
        cons.owe[:] = 6 * cap
        res = cons.drain()
        assert res["status"] == 0 and res["dups"] == 0
        assert all(0 < cons.sent[i] < 6 * cap for i in range(4))
        got = [bytearray() for _ in range(4)]
        for _ in range(400):
            for i, (a, b) in enumerate(conns):
                while True:
                    r = a.recv(cap)
                    if r.size == 0:
                        break
                    got[i] += r.tobytes()
            before = cons.ready()
            res = cons.drain()
            _check_drain(cons, before, res)
            if all(cons.sent[i] == 6 * cap for i in range(4)) and all(len(g) == 6 * cap for g in got):
                break
        for i in range(4):
            assert bytes(got[i]) == cons.sbuf[i * 6 * cap:(i + 1) * 6 * cap].tobytes()
    finally:
        for a, b in conns:
            b.device_release()
        rs.destroy()
        if cons:
            cons.close()
        _drop(conns)


def test_add_with_a_frame_waiting_and_while_a_consumer_runs(gpu):
    conns = _pairs(gpu, 3, 1 << 16, {}, "aw")
    rs = gpu.ReadySet(8)
    mem = drl.Pinned(gpu.lib())
    cons = None
    try:
        src_p, src = mem.array("src", np.uint8, 3 * 4096)
        src[:] = np.random.default_rng(4).integers(0, 256, src.size, dtype=np.uint8)
        members = [b.device_claim(mirrored=False) for a, b in conns]
        # a frame arrives before the add: the add's initial entry reports it
        assert conns[0][0].send_raw([(src_p, 1000)]) == 1000
        rs.add(conns[0][1], 0)
        cons = drl.Consumer(gpu, rs, members, 8192)
        cons.launch(with_stop=True, max_iters=1 << 26)
        try:
            # members join while the consumer runs, one of them with a frame already waiting
            assert conns[1][0].send_raw([(src_p + 4096, 2000)]) == 2000
            rs.add(conns[1][1], 1)
            rs.add(conns[2][1], 2)
            assert conns[2][0].send_raw([(src_p + 8192, 3000)]) == 3000
            assert conns[0][0].send_raw([(src_p + 1000, 500)]) == 500
            import time
            t_end = time.time() + 20
            while time.time() < t_end and not (cons.got[0] == 1500 and cons.got[1] == 2000 and cons.got[2] == 3000):
                time.sleep(0.01)
        finally:
            cons.stop[0] = 1
            res = cons.wait()
        assert res["status"] == 0 and res["foreign"] == 0, res
        assert np.array_equal(cons.received(0), src[:1500])
        assert np.array_equal(cons.received(1), src[4096:6096])
        assert np.array_equal(cons.received(2), src[8192:11192])
    finally:
        for a, b in conns:
            b.device_release()
        rs.destroy()
        if cons:
            cons.close()
        mem.free()
        _drop(conns)


def test_refusals_and_release(gpu):
    conns = _pairs(gpu, 6, 4096, {}, "rf")
    L = gpu.lib()
    rs = gpu.ReadySet(4)
    other = gpu.ReadySet(4)
    mem = drl.Pinned(L)
    cons = None
    try:
        src_p, src = mem.array("src", np.uint8, 4096)
        src[:] = np.random.default_rng(5).integers(0, 256, 4096, dtype=np.uint8)
        for cap in (0, 8193):
            assert not L.b200_ready_set_create(cap)
            assert "capacity" in gpu.last_error()
        with pytest.raises(RuntimeError, match="not device-owned"):
            rs.add(conns[0][1], 0)
        hs = [b.device_claim(mirrored=(i % 2 == 0)) for i, (a, b) in enumerate(conns)]
        rs.add(conns[0][1], 0)
        with pytest.raises(RuntimeError, match="already a member"):
            rs.add(conns[0][1], 9)
        with pytest.raises(RuntimeError, match="already a member"):
            other.add(conns[0][1], 9)
        for i in (1, 2, 3):
            rs.add(conns[i][1], i)
        with pytest.raises(RuntimeError, match="full"):
            rs.add(conns[4][1], 4)
        with pytest.raises(RuntimeError, match="has 4 members"):
            rs.destroy()
        # release members without taking: their initial entries go stale and fill the queue (4 members, 8 entries)
        for i in (0, 1, 2, 3):
            conns[i][1].device_release()
        hs[0] = conns[0][1].device_claim()
        rs.add(conns[0][1], 0)  # 4 stale + 1 queued + 1 member < 8
        hs[1] = conns[1][1].device_claim()
        rs.add(conns[1][1], 1)
        hs[2] = conns[2][1].device_claim()
        with pytest.raises(RuntimeError, match="overflow"):
            rs.add(conns[2][1], 2)  # 6 queued + 2 members
        # nothing is queued for a released end: its peer's Send lands no entry
        assert conns[3][0].send_raw([(src_p, 100)]) == 100
        cons = drl.Consumer(gpu, rs, hs[:4], 4096)
        cons.closed[3] = 1  # the server's own table: key 3 names a released end, its stale entry is skipped
        res = cons.drain()
        assert res["status"] == 0 and res["foreign"] == 0, res
        assert res["takes"] == 6, res  # 4 stale entries, then the initial entries of the two members
        assert list(cons.got) == [0, 0, 0, 0]
        # after the drain there is room again; a re-claimed end re-joins and its waiting frame is reported
        rs.add(conns[2][1], 2)
        hs[3] = conns[3][1].device_claim()
        rs.add(conns[3][1], 3)
        cons.set_handles(hs[:4])
        cons.closed[3] = 0
        res = cons.drain()
        assert res["status"] == 0 and res["dups"] == 0
        assert np.array_equal(cons.received(3), src[:100])
    finally:
        for a, b in conns:
            if b.device_owned():
                b.device_release()
        rs.destroy()
        other.destroy()
        if cons:
            cons.close()
        mem.free()
        _drop(conns)


def test_one_server_warp_serves_1024_ends_over_the_set(gpu):
    n, active, rounds, msg = 1024, 64, 20, 256
    conns = _pairs(gpu, n, 4096, {}, "sv")
    rs = gpu.ReadySet(n)
    mem = drl.Pinned(gpu.lib())
    try:
        srv = [a.device_claim(mirrored=False) for a, b in conns]
        cli = [b.device_claim(mirrored=False) for a, b in conns[:active]]
        for i, (a, b) in enumerate(conns):
            rs.add(a, i)
        D = drl.load()
        setp = mem.blob("set", [rs.device()])
        sp = mem.blob("srv", srv)
        cp = mem.blob("cli", cli)
        sbuf, _ = mem.array("sbuf", np.uint8, n * msg)
        cbuf, _ = mem.array("cbuf", np.uint8, active * 2 * msg)
        state, _ = mem.array("state", np.uint32, 3 * n)
        outp, out = mem.array("out", np.uint64, 2 * active + 5)
        s = drl.DrServe(setp, sp, cp, n, active, rounds, msg, sbuf, cbuf, state, outp, 1 << 26)
        rc = D.dr_serve_launch(C.byref(s))
        assert rc == 0, D.dr_error().decode()
        srv_out = out[2 * active:]
        assert srv_out[0] == 0 and srv_out[1] == active * rounds, srv_out
        assert all(out[2 * i] == 0 and out[2 * i + 1] == rounds for i in range(active)), out[:2 * active]
    finally:
        for a, b in conns:
            a.device_release()
        for a, b in conns[:active]:
            b.device_release()
        rs.destroy()
        mem.free()
        _drop(conns)
