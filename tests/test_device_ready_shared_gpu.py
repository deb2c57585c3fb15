"""GPU: many consumer warps take from one device ready set (include/b200_device.cuh: b200_warp_ready_take /
b200_warp_ready_rearm; DESIGN.md §13 "Many consumers"), driven by tests/native/device_ready_shared.cu.

Every consumer keeps a holder word per member: a take or a kept rearm CASes it from 0 to the warp's id, and the warp
clears it just before its rearm.  A failed CAS is a violation: two warps held one member.
  - random traces, per framing mode, 256 members (both claim forms): consumers of 1, 2, 8 and 32 warps over several
    CTAs, and two 8-warp kernels on two streams, run while device warp and block Sends, host single calls under the
    service, and host and device Disconnect drive the peers.  Then a drain after the producers stopped.  No violation,
    no second entry, no foreign key; each member received exactly the bytes its peer's calls accepted; no member is
    READY afterwards;
  - an echo server of 1, 4 and 16 warps on one set of 1024 claimed ends with 256 active device clients;
  - members added while an 8-warp consumer runs: each initial entry is served once.
Each case runs in a process of its own (tests/device_ready_shared_worker.py)."""
import contextlib
import os
import subprocess
import sys
import time

import ctypes as C
import numpy as np
import pytest

import device_ready_lib as drl
import device_ready_shared_lib as dsl

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1500)]
HERE = os.path.dirname(os.path.abspath(__file__))
MAX_WARPS = 32
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


class _Consumers:
    """Multi-warp consumers of one set over n members (key = index): what each member received, the holder words
    (device memory) and the per-member counters of ds_drain_kernel."""

    def __init__(self, pkg, rs, handles, rcap, take_max=8):
        self.D = dsl.load()
        assert self.D.ds_prepare() == 0, self.D.ds_error().decode()
        assert drl.load().dr_prepare() == 0
        self.mem, self.dev = drl.Pinned(pkg.lib()), dsl.Device(pkg)
        self.n, self.rcap, self.take_max = len(handles), rcap, take_max
        m = self.mem
        self.setp = m.blob("set", [rs.device()])
        self.hp = m.blob("members", handles)
        self.rbuf_p, self.rbuf = m.array("rbuf", np.uint8, self.n * rcap)
        self.got_p, self.got = m.array("got", np.uint64, self.n)
        self.taken_p, self.taken = m.array("taken", np.uint32, self.n)
        self.kept_p, self.kept = m.array("kept", np.uint32, self.n)
        self.idle_p, self.idle = m.array("idle", np.uint32, self.n)
        self.closed_p, self.closed = m.array("closed", np.uint32, self.n)
        self.stop_p, self.stop = m.array("stop", np.uint32, 1)
        self.holder_p = self.dev.array("holder", np.uint32, self.n)
        # everything a launch uses is allocated here: freeing memory waits for an idle device, and a consumer with a
        # stop flag runs until the host raises it
        self.keys = [self.dev.array("keys%d" % s, np.uint32, MAX_WARPS * take_max) for s in (0, 1)]
        self.outs = [m.array("out%d" % s, np.uint32, 8 * MAX_WARPS) for s in (0, 1)]
        self.running = {}

    def launch(self, warps, stream=0, warp_base=0, with_stop=False, mark_idle=False, max_iters=1 << 26):
        assert warps <= MAX_WARPS
        keys_p = self.keys[stream]
        out_p, out = self.outs[stream]
        out[:] = 0
        d = dsl.DsDrain(self.setp, self.hp, self.n, self.take_max, warp_base, 1 if mark_idle else 0, self.rbuf_p,
                        self.rcap, self.got_p, self.holder_p, self.taken_p, self.kept_p, self.idle_p, self.closed_p,
                        keys_p, out_p, self.stop_p if with_stop else None, max_iters)
        self.running[stream] = (d, out, warps)
        rc = self.D.ds_drain_launch(C.byref(d), warps, stream)
        assert rc == 0, (rc, self.D.ds_error().decode())

    def wait(self, stream=0):
        assert self.D.ds_wait(stream) == 0, self.D.ds_error().decode()
        _, out, warps = self.running.pop(stream)
        rows = out[:8 * warps].reshape(warps, 8)
        return dict(status=int(rows[:, 0].max()), violations=int(rows[:, 1].sum()), dups=int(rows[:, 2].sum()),
                    foreign=int(rows[:, 3].sum()), takes=int(rows[:, 4].sum()), retries=int(rows[:, 5].sum()))

    def ready(self):
        """READY members now (b200_warp_poll's READABLE, or a pending write with credit for one frame)"""
        ep, _ = self.mem.array("ev", np.uint32, self.n)
        rp, r = self.mem.array("rd", np.uint32, self.n)
        D = drl.load()
        assert D.dr_poll(self.hp, self.n, ep, rp) == 0, D.dr_error().decode()
        return r.copy()

    def holders(self):
        return self.dev.read("holder")

    def received(self, k):
        return self.rbuf[k * self.rcap:k * self.rcap + int(self.got[k])].copy()

    def close(self):
        self.mem.free()
        self.dev.free()


def _clean(res, final=False):
    assert res["status"] == 0, res
    assert res["violations"] == 0 and res["foreign"] == 0, res
    if final:
        assert res["dups"] == 0, res


class _Trace:
    """n connections; member i = b end (claimed, mirrored when i is even), its peer = a end, host-driven for even i
    and device-claimed for odd i.  Sources are pinned; accepted bytes advance each connection's stream."""

    def __init__(self, pkg, conns, src_bytes, seed):
        self.pkg, self.L, self.conns = pkg, pkg.lib(), conns
        self.n = len(conns)
        self.mem = drl.Pinned(self.L)
        self.rng = np.random.default_rng(seed)
        self.src_p, self.src = self.mem.array("src", np.uint8, self.n * src_bytes)
        self.src[:] = self.rng.integers(0, 256, self.src.size, dtype=np.uint8)
        self.sb = src_bytes
        self.off = [0] * self.n
        self.left = [False] * self.n
        self.members = [b.device_claim(mirrored=(i % 2 == 0)) for i, (a, b) in enumerate(conns)]
        self.peers = [a.device_claim() if i % 2 else None for i, (a, b) in enumerate(conns)]
        self.rs = pkg.ReadySet(self.n)
        for i, (a, b) in enumerate(conns):
            self.rs.add(b, i)
        self.cons = _Consumers(pkg, self.rs, self.members, src_bytes)
        # slices and device-op descriptors, allocated once (no free while a consumer runs)
        self.sl_p, self.sl = self.mem.array("slices", np.uint64, 2 * 1024)
        self.oph_p, self.oph = self.mem.array("oph", np.uint8, 64 * 64)
        self.ops_p, _ = self.mem.array("ops", np.uint8, C.sizeof(drl.DrOp) * 64)
        self.k = 0

    def slice_arr(self, i, length):
        self.k = (self.k + 1) % 1024
        self.sl[2 * self.k], self.sl[2 * self.k + 1] = self.src_p + i * self.sb + self.off[i], length
        return self.sl_p + 16 * self.k

    def device_ops(self, kind, ops):
        """ops: (handle bytes, slice array pointer, nslices) -> per-op returns (drl.device_ops without allocating)"""
        arr = (drl.DrOp * 64).from_address(self.ops_p)
        for i, (h, sl, n) in enumerate(ops):
            self.oph[64 * i:64 * (i + 1)] = np.frombuffer(h, np.uint8)
            arr[i].h, arr[i].slices, arr[i].n, arr[i].ret = self.oph_p + 64 * i, sl, n, 0
        D = drl.load()
        assert D.dr_ops(kind, self.ops_p, len(ops)) == 0, D.dr_error().decode()
        return [int(arr[i].ret) for i in range(len(ops))]

    def pick(self, host, count):
        idx = [i for i in range(self.n) if (i % 2 == 0) == host and not self.left[i]]
        self.rng.shuffle(idx)
        return idx[:count]

    def length(self, i, big):
        n = int(self.rng.integers(9000, 20000)) if big else int(self.rng.integers(1, 3000))
        return max(0, min(n, self.sb - self.off[i]))

    def step(self, kind):
        if kind in ("warp", "block"):
            ops, idx = [], []
            for i in self.pick(False, 48 if kind == "warp" else 16):
                n = self.length(i, kind == "block")
                if n:
                    ops.append((self.peers[i], self.slice_arr(i, n), 1))
                    idx.append(i)
            rets = self.device_ops(drl.WARP_SEND if kind == "warp" else drl.BLOCK_SEND, ops)
            for i, r in zip(idx, rets):
                self.off[i] += r
        elif kind == "device-disconnect":
            idx = self.pick(False, 6)
            self.device_ops(drl.WARP_DISC, [(self.peers[i], 0, 0) for i in idx])
            for i in idx:
                self.left[i] = True
        elif kind == "host-disconnect":
            for i in self.pick(True, 6):
                self.conns[i][0].disconnect()
                self.left[i] = True
        elif kind in ("single", "single-big"):
            for i in self.pick(True, 24):
                n = self.length(i, kind == "single-big")
                if n:
                    self.off[i] += self.conns[i][0].send_raw([(int(self.src_p + i * self.sb + self.off[i]), n)])
        else:
            raise ValueError(kind)

    def phase(self, kinds, kernels):
        """kernels: consumer warps per kernel (one stream each), running while the producers run; then a drain"""
        c = self.cons
        c.idle[:] = 0
        c.stop[0] = 0
        base = 0
        for s, w in enumerate(kernels):
            c.launch(w, stream=s, warp_base=base, with_stop=True)
            base += w
        try:
            for kind in kinds:
                self.step(kind)
        finally:
            c.stop[0] = 1
            results = [c.wait(s) for s in range(len(kernels))]
        for r in results:
            _clean(r)
        c.launch(kernels[0], mark_idle=True)
        final = c.wait()
        _clean(final, final=True)
        self.check()
        return results, final

    def check(self):
        c = self.cons
        after = c.ready()
        left = [i for i in range(self.n) if after[i] and not c.closed[i]]
        assert not left, ("members still ready after the drain", left)
        held = c.holders()
        assert all(held[i] == 0 for i in range(self.n) if not c.closed[i]), "a member is still held after the drain"
        for i in range(self.n):
            want = self.src[i * self.sb:i * self.sb + self.off[i]]
            assert np.array_equal(c.received(i), want), ("bytes of connection", i)
            if self.left[i]:
                assert c.closed[i] == 1, i

    def close(self):
        for i, (a, b) in enumerate(self.conns):
            b.device_release()
            if self.peers[i] is not None:
                a.device_release()
        self.rs.destroy()
        self.cons.close()
        self.mem.free()


def random_traces(gpu, mode):
    conns = _pairs(gpu, 256, 1 << 16, MODES[mode], "ds-" + mode)
    T = None
    try:
        T = _Trace(gpu, conns, 1 << 17, seed=101 + sorted(MODES).index(mode))
        with _service(gpu):
            for kernels in ([1], [2], [8], [32], [8, 8]):
                T.phase(("single", "warp", "block", "single-big", "warp", "single"), kernels)
            T.phase(("host-disconnect", "single", "device-disconnect", "warp"), [8])
        assert sum(T.off) > 0 and any(T.left)
        # every member was taken at least once: the initial entries of the adds
        assert all(T.cons.taken[i] >= 1 for i in range(T.n))
    finally:
        if T is not None:
            T.close()
        _drop(conns)


def echo_server(gpu, warps):
    n, active, rounds, msg, take_max = 1024, 256, 100, 256, 4
    conns = _pairs(gpu, n, 4096, {}, "dse")
    D = dsl.load()
    assert D.ds_prepare() == 0
    mem, dev = drl.Pinned(gpu.lib()), dsl.Device(gpu)
    stride = n // active
    rs = gpu.ReadySet(n)
    try:
        srv = [a.device_claim(mirrored=False) for a, b in conns]
        cli = [conns[stride * i][1].device_claim(mirrored=False) for i in range(active)]
        for i, (a, b) in enumerate(conns):
            rs.add(a, i)
        outp, out = mem.array("out", np.uint64, 2 * active + 8 * warps)
        s = dsl.DsServe(mem.blob("set", [rs.device()]), mem.blob("srv", srv), mem.blob("cli", cli), n, active, rounds,
                        msg, warps, 1, take_max, dsl.FENCE if warps > 1 else 0,
                        dev.array("sbuf", np.uint8, n * msg), dev.array("cbuf", np.uint8, active * 2 * msg),
                        dev.array("state", np.uint32, 2 * n), dev.array("keys", np.uint32, warps * take_max),
                        dev.array("done", np.uint64, 1), outp, 1 << 26)
        rc = D.ds_serve_launch(C.byref(s))
        assert rc == 0, (rc, D.ds_error().decode())
        assert all(out[2 * i] == 0 and out[2 * i + 1] == rounds for i in range(active)), out[:2 * active]
        rows, _ = dsl.serve_totals(out, active, warps)
        assert (rows[:, 0] == 0).all(), rows
        assert int(rows[:, 1].sum()) == active * rounds, rows[:, 1]
        assert int(rows[:, 5].sum()) == 0, ("holder violations", rows[:, 5])
        assert int(dev.read("done")[0]) == active * rounds
    finally:
        for i, (a, b) in enumerate(conns):
            if a.device_owned():
                a.device_release()
            if b.device_owned():
                b.device_release()
        rs.destroy()
        mem.free()
        dev.free()
        _drop(conns)


def members_added(gpu):
    n = 72
    conns = _pairs(gpu, n, 1 << 16, {}, "dsa")
    rs = gpu.ReadySet(128)
    mem = drl.Pinned(gpu.lib())
    cons = None
    try:
        src_p, src = mem.array("src", np.uint8, n * 4096)
        src[:] = np.random.default_rng(6).integers(0, 256, src.size, dtype=np.uint8)
        members = [b.device_claim(mirrored=(i % 2 == 0)) for i, (a, b) in enumerate(conns)]
        for i in range(8):
            rs.add(conns[i][1], i)
        cons = _Consumers(gpu, rs, members, 4096)
        cons.launch(8, with_stop=True)
        want = {}
        try:
            # members join while the consumer runs, every other one with a frame already waiting
            for i in range(8, n):
                if i % 2:
                    ln = 100 + 37 * i
                    assert conns[i][0].send_raw([(src_p + 4096 * i, ln)]) == ln
                    want[i] = ln
                rs.add(conns[i][1], i)
            t_end = time.time() + 30
            while time.time() < t_end and not all(cons.taken[i] >= 1 for i in range(n)):
                time.sleep(0.01)
        finally:
            cons.stop[0] = 1
            res = cons.wait()
        _clean(res)
        assert list(cons.taken) == [1] * n, cons.taken
        for i in range(n):
            assert np.array_equal(cons.received(i), src[4096 * i:4096 * i + want.get(i, 0)]), i
        assert not cons.ready().any()
    finally:
        for a, b in conns:
            b.device_release()
        rs.destroy()
        if cons:
            cons.close()
        mem.free()
        _drop(conns)


# Each case runs in a process of its own (device_ready_shared_worker.py).  The cases hold up to 2048 pairs at once, and
# the runtime keeps every pair it created, with its eventfd, in a pool that later takes cycle through: run here, they
# would leave the pytest process handing out pairs whose eventfds lie above select()'s limit.
def _worker(case):
    out = subprocess.run([sys.executable, os.path.join(HERE, "device_ready_shared_worker.py"), case],
                         capture_output=True, text=True, timeout=1400)
    assert out.returncode == 0 and ("case %s ok" % case) in out.stdout, out.stdout[-6000:] + out.stderr[-4000:]


@pytest.mark.parametrize("mode", sorted(MODES))
def test_random_traces_many_consumers(pkg, mode):
    _worker("traces-" + mode)


@pytest.mark.parametrize("warps", [1, 4, 16])
def test_echo_server_warps_share_one_set(pkg, warps):
    _worker("echo-%d" % warps)


def test_members_added_while_many_warps_take(pkg):
    _worker("added")
