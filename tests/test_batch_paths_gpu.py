"""GPU: batches the library launches itself -- device memory, the host-staged lanes and B200_BATCH_ZEROCOPY -- against
the CPU models, launch by launch, with guarded destinations.

Memory paths (one parametrized fixture):
  device             b200_mem_alloc_device: one launch per batch, on the library's stream or the given one
  staged             b200_mem_alloc_host: the host-staged lanes (H2D -> k_send, k_recv -> D2H per lane)
  staged-registered  page-aligned anonymous memory passed to b200_mem_register_host: push_h2d widens the H2D copy
                     inside the registered range
  staged-foreign     torch pinned memory: the library does not know its base, so the copy is not widened
  zerocopy           b200_mem_alloc_host + B200_BATCH_ZEROCOPY: the kernels dereference pinned memory over PCIe

Guards: every source slice and every Recv window sits between canary bytes (a pattern of period 255 that never
holds 0), windows at every phase mod 16 and some packed back to back.  Each arena keeps a shadow of what every byte
must hold and the whole used span is compared with it after every launch: sources unchanged; outside the windows
the canary; inside a window [0, delivered) the model's bytes and the rest unchanged -- except on the host-staged path,
which copies the whole window back from the batch's staging arena: there [0, cap) equals a per-op stage image that
starts at zero and takes each launch's delivered bytes over [0, delivered).

Determinism: a send batch holds at most one Send per direction of a connection and a recv batch at most one Recv,
and a recv batch only runs once the send batch before it finished (or, relaunched without host syncs, after it in
stream / lane order), so per-op counts do not depend on timing.
"""
import ctypes as C
import mmap
import os
import subprocess
import sys

import numpy as np
import pytest

import trace
from submit_lib import submit
from test_submit_gpu import MODES, Conn, _check_conn, _config, _lens, _models, _view, G

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PATHS = ("device", "staged", "staged-registered", "staged-foreign", "zerocopy")
CAPS = (1024, 4096, 16384, 65536)
GUARD = 64
PATTERN = ((np.arange(255) * 151 + 89) % 255 + 1).astype(np.uint8)


@pytest.fixture(scope="module")
def models(oracle):
    return _models(oracle)


@pytest.fixture(params=PATHS)
def path(request):
    return request.param


class Mem:
    """One allocation of a memory path and a shadow of what every byte of it must hold (canary bytes at first).
    `skew` (staged-registered only): the registered range starts that many bytes into a page."""

    def __init__(self, pkg, path, nbytes, skew=0):
        self.pkg, self.L, self.path, self.n = pkg, pkg.lib(), path, nbytes
        self.staged = path.startswith("staged")
        self.flags = pkg.ZEROCOPY if path == "zerocopy" else 0
        L, self._keep = self.L, None
        if path == "device":
            self.base = L.b200_mem_alloc_device(nbytes)
        elif path in ("staged", "zerocopy"):
            self.base = L.b200_mem_alloc_host(nbytes)
        elif path == "staged-registered":
            self._keep = mmap.mmap(-1, nbytes + 2 * mmap.PAGESIZE)
            self.base = np.frombuffer(self._keep, np.uint8).ctypes.data + mmap.PAGESIZE + skew
            assert L.b200_mem_register_host(self.base, nbytes) == 0, pkg.last_error()
        else:
            import torch
            self._keep = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
            self.base = self._keep.data_ptr()
        assert self.base, pkg.last_error()
        self.view = None if path == "device" else np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(self.base))
        self.want = np.resize(PATTERN, nbytes)
        self.dirty = (0, nbytes)
        self.upload()
        self.off = self.hi = 0

    def ptr(self, o):
        return self.base + o

    def reset(self):
        self.off = 0

    def alloc(self, n, phase=None, at=None):
        """offset of n bytes: at `at`; else GUARD bytes past the previous allocation at `phase` mod 16; else
        (phase None) right after the previous allocation"""
        if at is not None:
            o = at
        elif phase is None:
            o = self.off
        else:
            o = (self.off + GUARD + 15) // 16 * 16 + phase
        self.off = max(self.off, o + n)
        self.hi = max(self.hi, self.off + GUARD)
        assert self.hi <= self.n, "%s: arena full" % self.path
        return o

    def put(self, o, arr):
        self.want[o:o + arr.size] = arr
        self.dirty = (min(self.dirty[0], o), max(self.dirty[1], o + arr.size))

    def upload(self):
        lo, hi = self.dirty
        if hi > lo:
            if self.view is None:
                assert self.L.b200_memcpy(self.base + lo, self.want[lo:].ctypes.data, hi - lo, 0, None) == 0
                assert self.L.b200_stream_sync(None) == 0
            else:
                self.view[lo:hi] = self.want[lo:hi]
        self.dirty = (self.n, 0)

    def read(self, o, n):
        if self.view is not None:
            return self.view[o:o + n].copy()
        out = np.zeros(max(n, 1), np.uint8)
        if n:
            assert self.L.b200_memcpy(out.ctypes.data, self.base + o, n, 1, None) == 0
            assert self.L.b200_stream_sync(None) == 0
        return out[:n]

    def land(self, o, cap, data, image):
        """what a Recv that delivered `data` into the window [o, o + cap) leaves there"""
        if self.staged:
            image[:data.size] = data
            self.want[o:o + cap] = image
        else:
            self.want[o:o + data.size] = data

    def check(self, label):
        bad = np.flatnonzero(self.read(0, self.hi) != self.want[:self.hi])
        assert bad.size == 0, "%s: %s arena: %d bytes differ from the shadow, first at offsets %s" % (
            label, self.path, bad.size, bad[:16])

    def free(self):
        if self.path == "device":
            self.L.b200_mem_free_device(self.base)
        elif self.path in ("staged", "zerocopy"):
            self.L.b200_mem_free_host(self.base)
        elif self.path == "staged-registered":
            self.L.b200_mem_unregister_host(self.base)
        self.view = self._keep = None


# ---- running ops: prepared batches, b200_pairs_send / recv, b200_pairs_submit (service stopped)

def _batch(pkg, kind, ops, flags):
    bt = pkg.Batch(kind, ops, flags)
    try:
        bt.launch()
        return bt.results(), bt.calls()
    finally:
        bt.destroy()


def _raw(ops):
    return [(op[0].h,) + tuple(op[1:]) for op in ops]


def _pairs(pkg, kind, ops, flags):
    L, n = pkg.lib(), len(ops)
    out = (C.c_uint64 * max(1, n))()
    if kind == "send":
        arr = (pkg.SendOp * max(1, n))()
        for i, (h, sl, nsl, bidx) in enumerate(_raw(ops)):
            arr[i].pair, arr[i].slices, arr[i].nslices, arr[i].byte_idx = h, sl, nsl, bidx
        rc = L.b200_pairs_send(arr, n, flags, out, None)
    else:
        arr = (pkg.RecvOp * max(1, n))()
        for i, (h, dst, cap) in enumerate(_raw(ops)):
            arr[i].pair, arr[i].dst, arr[i].cap = h, dst, cap
        rc = L.b200_pairs_recv(arr, n, flags, out, None)
    assert rc == 0, pkg.last_error()
    return list(out)[:n], None


def _submit(pkg, kind, ops, flags):
    rc, acc, dlv = submit(pkg, _raw(ops) if kind == "send" else (), _raw(ops) if kind == "recv" else (), flags)
    assert rc == 0, pkg.last_error()
    return (acc if kind == "send" else dlv), None


RUNNERS = {"batch": _batch, "pairs": _pairs, "submit": _submit}


def _model_send(op, ub):
    c, d, bufs, bidx = op
    mtx = c.ends(d)[2]
    if ub:
        n, calls = c.model.send_all(mtx, bufs, bidx)
        return int(n), int(calls)
    n = int(c.model.send(mtx, bufs, bidx))
    return n, int(n > 0)


def _model_recv(op, ub):
    c, d, cap = op[:3]
    mrx = c.ends(d)[3]
    if ub:
        out, calls = c.model.recv_drain(mrx, cap)
        return out, int(calls)
    out = c.model.recv(mrx, cap)
    return out, int(out.size > 0)


def _desc(op, kind):
    return "%s %s dir %d" % (kind, op[0].name, op[1])


def _check_all(conns, mems, label):
    for c in conns:
        _check_conn(c, label)
    for m in mems:
        m.check(label)


def _send_phase(pkg, conns, sends, sls, flags, runner, mems, label):
    """sends: [conn, dir, bufs, byte_idx]; sls: their slice arrays"""
    ub = bool(flags & pkg.UNTIL_BLOCKED)
    ops = [(c.ends(d)[0], sl, len(bufs), bidx) for (c, d, bufs, bidx), sl in zip(sends, sls)]
    if ops:
        res, calls = RUNNERS[runner](pkg, "send", ops, flags)
        for i, op in enumerate(sends):
            n, mc = _model_send(op, ub)
            assert res[i] == n, "%s: %s: accepted %d, want %d" % (label, _desc(op, "send"), res[i], n)
            if calls is not None:
                assert calls[i] == mc, "%s: %s: calls %d, want %d" % (label, _desc(op, "send"), calls[i], mc)
    _check_all(conns, mems, label + " after the send batch")


def _recv_phase(pkg, conns, recvs, dmem, offs, flags, runner, mems, label):
    """recvs: [conn, dir, cap, stage image]; windows at dmem offsets `offs`"""
    ub = bool(flags & pkg.UNTIL_BLOCKED)
    ops = [(c.ends(d)[1], dmem.ptr(o), cap) for (c, d, cap, _), o in zip(recvs, offs)]
    if ops:
        res, calls = RUNNERS[runner](pkg, "recv", ops, flags)
        for i, op in enumerate(recvs):
            out, mc = _model_recv(op, ub)
            got = dmem.read(offs[i], res[i])
            assert (res[i], trace.sha(got)) == (out.size, trace.sha(out)), "%s: %s: delivered %d, want %d" % (
                label, _desc(op, "recv"), res[i], out.size)
            if calls is not None:
                assert calls[i] == mc, "%s: %s: calls %d, want %d" % (label, _desc(op, "recv"), calls[i], mc)
            dmem.land(offs[i], op[2], out, op[3])
    _check_all(conns, mems, label + " after the recv batch")


def _place_sends(mem, sends, adjacent, rng):
    """slice arrays: every slice between guards at a random phase, or (adjacent) every slice of every op back to
    back -- the last slice of one op right before the first slice of the next"""
    out = []
    if adjacent:
        o = mem.alloc(sum(b.size for op in sends for b in op[2]), int(rng.integers(0, 16)))
    for op in sends:
        sl = []
        for b in op[2]:
            if not adjacent:
                o = mem.alloc(b.size, int(rng.integers(0, 16)))
            mem.put(o, b)
            sl.append((mem.ptr(o), b.size))
            if adjacent:
                o += b.size
        out.append(mem.pkg.make_slices(sl))
    return out


def _place_recvs(mem, recvs, rng):
    """window offsets: phase i mod 16 between guards, or packed right after the previous window"""
    return [mem.alloc(op[2], None if i and rng.random() < 0.3 else i % 16) for i, op in enumerate(recvs)]


# ---- 1. random rounds, launch by launch

def _conns(pkg, models, n):
    return [Conn(pkg, models, MODES[i % 3], CAPS[(i // 3) % len(CAPS)]) for i in range(n)]


def _random_rounds(pkg, models, path, seed, nconn=48, rounds=8, runner="batch", other=None):
    """`rounds` rounds of one send batch then one recv batch over `nconn` connections (every mode and ring size in
    every batch).  Rounds 3, 7, ...: B200_BATCH_ONE_CALL; odd rounds: the Send slices adjacent in memory.  other: a
    second arena of the other memory class, for calls that mix host and device buffers."""
    rng = np.random.default_rng(seed)
    conns = _conns(pkg, models, nconn)
    mem = Mem(pkg, path, 48 << 20)
    try:
        for r in range(rounds):
            label = "%s round %d" % (path, r)
            flags = (pkg.ONE_CALL if r % 4 == 3 else pkg.UNTIL_BLOCKED) | mem.flags
            adjacent = r % 2 == 1
            sends, recvs = [], []
            for c in conns:
                for d in (0, 1):
                    if rng.random() < 0.6:
                        lens, bidx = _lens(rng, c.cap)
                        sends.append([c, d, trace.make_bufs(lens, int(rng.integers(0, 1 << 16))), bidx])
                    if rng.random() < 0.6:
                        cap = int(rng.integers(1, 2 * c.cap))
                        recvs.append([c, d, cap, np.zeros(cap, np.uint8)])
            if not adjacent:  # adjacent: both directions of a connection share a lane and sit next to each other
                sends = [sends[i] for i in rng.permutation(len(sends))]
            recvs = [recvs[i] for i in rng.permutation(len(recvs))]
            mem.reset()
            sls = _place_sends(mem, sends, adjacent, rng)
            offs = _place_recvs(mem, recvs, rng)
            mem.upload()
            if other is not None:
                _mixed_call(pkg, conns, mem, other, runner, label)
            _send_phase(pkg, conns, sends, sls, flags, runner, [mem], label)
            _recv_phase(pkg, conns, recvs, mem, offs, flags, runner, [mem], label)
    finally:
        for c in conns:
            c.close()
        mem.free()


def test_random_rounds(gpu, models, path):
    _random_rounds(gpu, models, path, 7100 + PATHS.index(path))


# ---- 2. one prepared batch, relaunched

def _check_recvs(br, stream, recvs, offs, want, mem, conns, label):
    """the recv batch's last launch: per op (count, calls, SHA-1 of the window's first `count` bytes), then the
    connections and the arena"""
    for i, (r, n) in enumerate(zip(br.results(stream), br.calls())):
        got = (r, n, trace.sha(mem.read(offs[i], r)))
        assert got == want[i], "%s: %s\n got  %s\n want %s" % (label, _desc(recvs[i], "recv"), got, want[i])
    _check_all(conns, [mem], label)


VARIANTS = [(p, v) for p in PATHS for v in
            (("sync", "stream") if p in ("device", "zerocopy") else ("sync", "lanes-null", "lanes-fork"))]


@pytest.mark.parametrize("path,variant", VARIANTS, ids=["%s-%s" % pv for pv in VARIANTS])
def test_prepared_batches_relaunched(gpu, models, path, variant):
    """A send batch per source buffer and one recv batch, prepared once over 12 connections (both directions) and
    launched for several laps of every ring; the steps alternate the two send batches as bench.py does.  sync:
    compared with the models after every launch.  Otherwise K steps back to back without a host sync -- on a user
    stream (device, zerocopy), with the lanes free and b200_lanes_join(NULL) (lanes-null) or forked from and joined
    back into a user stream (lanes-fork) -- then the last launch's results and calls, the cursors, the ring images and
    every arena byte."""
    pkg, L = gpu, gpu.lib()
    rng = np.random.default_rng(7200 + VARIANTS.index((path, variant)))
    conns = _conns(pkg, models, 12)
    mem = Mem(pkg, path, 16 << 20)
    batches = []
    try:
        sends = [[], []]
        recvs = []
        for c in conns:
            for d in (0, 1):
                lens = [9, int(rng.integers(c.cap // 8, c.cap // 2)), 9, int(rng.integers(1, 200))]
                bidx = int(rng.integers(0, 9))
                for k in (0, 1):
                    sends[k].append([c, d, trace.make_bufs(lens, int(rng.integers(0, 1 << 16))), bidx])
                cap = int(rng.integers(c.cap // 4, 2 * c.cap))
                recvs.append([c, d, cap, np.zeros(cap, np.uint8)])
        sls = [_place_sends(mem, sends[k], k == 1, rng) for k in (0, 1)]
        offs = _place_recvs(mem, recvs, rng)
        mem.upload()
        fl = pkg.UNTIL_BLOCKED | mem.flags
        bs = [pkg.Batch("send", [(c.ends(d)[0], sl, len(b), i) for (c, d, b, i), sl in zip(sends[k], sls[k])], fl)
              for k in (0, 1)]
        br = pkg.Batch("recv", [(c.ends(d)[1], mem.ptr(o), cap) for (c, d, cap, _), o in zip(recvs, offs)], fl)
        batches = bs + [br]
        st = sh = None
        if variant in ("stream", "lanes-fork"):
            import torch
            st = torch.cuda.Stream()
            sh = C.c_void_p(st.cuda_stream)
        launch_on = sh if variant == "stream" else None
        K = 12
        if variant == "lanes-fork":
            assert L.b200_lanes_fork(sh) == 0
        for k in range(K):
            label = "%s %s launch %d" % (path, variant, k)
            b = bs[k & 1]
            b.launch(launch_on)
            want_s = [_model_send(op, True) for op in sends[k & 1]]
            if variant == "sync":
                assert list(zip(b.results(), b.calls())) == want_s, label
                _check_all(conns, [mem], label + " after the send batch")
            br.launch(launch_on)
            want_r = []
            for op, o in zip(recvs, offs):
                out, mc = _model_recv(op, True)
                want_r.append((out.size, mc, trace.sha(out)))
                mem.land(o, op[2], out, op[3])
            if variant == "sync":
                _check_recvs(br, None, recvs, offs, want_r, mem, conns, label + " after the recv batch")
        if variant != "sync":
            label = "%s %s after %d launches" % (path, variant, K)
            if variant == "lanes-fork":
                assert L.b200_lanes_join(sh) == 0
            elif variant == "lanes-null":
                assert L.b200_lanes_join(None) == 0
            if st is not None:
                st.synchronize()
            last = bs[(K - 1) & 1]
            res_on = sh if variant == "stream" else None
            assert list(zip(last.results(res_on), last.calls())) == want_s, label
            _check_recvs(br, res_on, recvs, offs, want_r, mem, conns, label)
    finally:
        for b in batches:
            b.destroy()
        for c in conns:
            c.close()
        mem.free()


# ---- 3. the lane count (B200_LANES / B200_LANE_SHIFT are read once per process)

def _lanes_used(pkg):
    """b200_launch_count's step for a staged send batch and a staged recv batch over 48 connections whose lower
    slots are 0..47: one launch per lane that holds an op.  A fresh process hands out slots in creation order, so
    pair k and pair k + 48 make connection k."""
    L = pkg.lib()
    _config(pkg, 4096, "ref")
    ps = [pkg.Pair("lane-%d" % k) for k in range(96)]
    for k in range(48):
        assert ps[k].connect(ps[k + 48].address()) and ps[k + 48].connect(ps[k].address())
    mem = Mem(pkg, "staged", 1 << 20)
    try:
        bufs = trace.make_bufs([100] * 48, 5)
        sls = _place_sends(mem, [[None, 0, [b], 0] for b in bufs], False, np.random.default_rng(0))
        offs = [mem.alloc(4096, k % 16) for k in range(48)]
        mem.upload()
        used = []
        for kind, ops in (("send", [(ps[k], sls[k], 1, 0) for k in range(48)]),
                          ("recv", [(ps[k + 48], mem.ptr(offs[k]), 4096) for k in range(48)])):
            n = L.b200_launch_count()
            res, _ = _batch(pkg, kind, ops, pkg.UNTIL_BLOCKED)
            assert res == [100] * 48, res
            used.append(L.b200_launch_count() - n)
        return used
    finally:
        for p in ps:
            p.disconnect()
            p.putback()
        mem.free()


def lanes_child(lanes):
    """run by test_lane_counts_in_a_subprocess in a process of its own"""
    import __graft_entry__ as ge
    import orlib
    pkg = ge.load_package()
    pkg.init(0)
    used = _lanes_used(pkg)
    assert used == [lanes, lanes], "lanes used by a 48-connection batch: %s, want %d" % (used, lanes)
    _random_rounds(pkg, _models(orlib.Oracle()), "staged", 7300, rounds=6)
    print("lanes ok")


# (environment, lanes a 48-connection batch uses: (lower slot >> shift) % lanes over slots 0..47)
LANE_ENVS = [({"B200_LANES": "1"}, 1), ({"B200_LANES": "16", "B200_LANE_SHIFT": "0"}, 16), ({"B200_LANES": "3"}, 3)]


@pytest.mark.parametrize("env,lanes", LANE_ENVS, ids=["lanes1", "lanes16-shift0", "lanes3"])
def test_lane_counts_in_a_subprocess(env, lanes):
    code = "import sys; sys.path[:0] = [%r, %r]; import test_batch_paths_gpu; test_batch_paths_gpu.lanes_child(%d)" % (
        ROOT, HERE, lanes)
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0 and "lanes ok" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]


# ---- 4. the edges of push_h2d's widening

@pytest.mark.parametrize("path", ["staged", "staged-registered"])
def test_widening_edges(gpu, models, path):
    """Send slices 1..255 bytes from the start of their allocation / registered range (the registered ranges start
    160 bytes into a page, so below offset 96 the enclosing 256-byte block leaves the range and the copy must not be
    widened; from 96 on it may be, down to the block start inside the range), and slices 1..255 bytes past a 256-byte
    boundary inside the range, each followed by a 9-byte slice right behind it (one run) and mixed with the slices of
    other ops of the same lane.

    What this cannot see: a widening that ignores the range start.  The enclosing 256-byte block always lies in the
    page of the range's first byte, cudaHostRegister pins whole pages, and the CUDA 12 driver on an H100 accepts
    such a copy; the lead bytes land in staging that nothing reads.  The check in push_h2d only matters where a driver
    refuses copies that leave the registered bytes."""
    pkg = gpu
    rng = np.random.default_rng(7400 + (path == "staged-registered"))
    skew = 160 if path == "staged-registered" else 0
    blocks = [Mem(pkg, path, 256 << 10, skew) for _ in range(16)]
    dst = Mem(pkg, path, 4 << 20)
    conns = [Conn(pkg, models, MODES[i % 3], (4096, 65536)[(i // 3) % 2]) for i in range(8)]
    try:
        for r in range(6):
            label = "%s round %d" % (path, r)
            for m in blocks + [dst]:
                m.reset()
            sends, sls = [], []
            first = [int(rng.integers(1, 2000)) for _ in range(16)]
            edge = [blocks[j].alloc(first[j], at=1 + (j * 37 + r * 101) % 255) for j in range(16)]
            for j in range(16):
                c, d = conns[j // 2], j % 2
                lens = [first[j]]
                where = [(blocks[j], edge[j])]
                for k in range(int(rng.integers(1, 4))):
                    m = blocks[(j + 1 + k) % 16]
                    where.append((m, (m.off + GUARD + 255) // 256 * 256 + int(rng.integers(1, 256))))
                    lens.append(int(rng.integers(1, 3000)))
                    where.append((m, None))
                    lens.append(9)
                bufs = trace.make_bufs(lens, int(rng.integers(0, 1 << 16)))
                sl = []
                for k, ((m, at), b) in enumerate(zip(where, bufs)):
                    o = at if k == 0 else m.alloc(b.size, None, at)
                    m.put(o, b)
                    sl.append((m.ptr(o), b.size))
                sends.append([c, d, bufs, int(rng.integers(0, lens[0]))])
                sls.append(pkg.make_slices(sl))
            order = rng.permutation(16)
            sends, sls = [sends[i] for i in order], [sls[i] for i in order]
            recvs = [[c, d, 2 * c.cap, np.zeros(2 * c.cap, np.uint8)] for c in conns for d in (0, 1)]
            offs = _place_recvs(dst, recvs, rng)
            for m in blocks + [dst]:
                m.upload()
            _send_phase(pkg, conns, sends, sls, pkg.UNTIL_BLOCKED, "batch", blocks + [dst], label)
            _recv_phase(pkg, conns, recvs, dst, offs, pkg.UNTIL_BLOCKED, "batch", blocks + [dst], label)
    finally:
        for c in conns:
            c.close()
        for m in blocks + [dst]:
            m.free()


# ---- 5. the benchmark's shape on the staged and zero-copy paths

@pytest.mark.parametrize("path", ["staged", "staged-registered", "staged-foreign", "zerocopy"])
def test_benchmark_shape(gpu, oracle, path):
    """bench.py's e2e leg at a third of its width: 32 connections with 16 MiB rings, one 4 MiB chttp2-shaped message
    per connection in back-to-back slices, destinations 256-byte strided; two prepared send batches over two
    different sources alternate, forked from and joined into a user stream (staged) or launched on it (zerocopy):
    six steps with a host sync after each (more than a lap), then six back to back as bench.py's timed loop runs
    them, where a step's Send overlaps the previous step's Recv unless the lanes order them.  One model connection
    gives every op's count and calls and the cursors."""
    import torch
    pkg, L = gpu, gpu.lib()
    nconn, cap = 32, 16 << 20
    lens = pkg.chttp2_slice_lens(4 << 20)
    total = sum(lens)
    dstride = (total + 255) // 256 * 256
    _config(pkg, cap, "ref")
    pairs = [pkg.connected_pair("bp-a%d" % i, "bp-b%d" % i) for i in range(nconn)]
    mtx, mrx = oracle.pair_pair(cap)
    src = Mem(pkg, path, (2 * nconn * total + (1 << 20)) >> 20 << 20)
    dst = Mem(pkg, path, (nconn * dstride + (1 << 20)) >> 20 << 20)
    batches = []
    try:
        i = np.arange(total, dtype=np.uint64)
        base = [src.alloc(nconn * total, 0), src.alloc(nconn * total, 0)]
        msgs = [[(((i * np.uint64(40503)) >> np.uint64(5)) + np.uint64(17 * c + 91 * k)).astype(np.uint8)
                 for c in range(nconn)] for k in (0, 1)]
        for k in (0, 1):
            src.put(base[k], np.concatenate(msgs[k]))
        dbase = dst.alloc(nconn * dstride, at=256)  # every window 256-byte aligned, as bench.py's are
        src.upload()
        fl = pkg.UNTIL_BLOCKED | src.flags
        keep, bs = [], []
        for k in (0, 1):
            ops = []
            for c in range(nconn):
                offs = np.concatenate([[0], np.cumsum(lens)[:-1]]) + base[k] + c * total
                sl = pkg.make_slices([(src.ptr(int(o)), n) for o, n in zip(offs, lens)])
                keep.append(sl)
                ops.append((pairs[c][0], sl, len(lens), 0))
            bs.append(pkg.Batch("send", ops, fl))
        br = pkg.Batch("recv", [(pairs[c][1], dst.ptr(dbase + c * dstride), total) for c in range(nconn)], fl)
        batches = bs + [br]
        st = torch.cuda.Stream()
        sh = C.c_void_p(st.cuda_stream)
        mbufs = trace.make_bufs(lens, 999)

        def steps(first, k):
            """k steps from step `first` on, back to back, then one host sync"""
            if src.staged:
                assert L.b200_lanes_fork(sh) == 0
            for r in range(first, first + k):
                bs[r & 1].launch(None if src.staged else sh)
                br.launch(None if src.staged else sh)
            if src.staged:
                assert L.b200_lanes_join(sh) == 0
            st.synchronize()
            for _ in range(k):
                want_s = tuple(int(x) for x in oracle.send_all(mtx, mbufs, 0))
                out, mc = oracle.recv_drain(mrx, total)
                assert want_s[0] == out.size == total
            return want_s, int(mc)

        # six steps with a host sync after each, then bench.py's timed loop: six more without one
        for r, k in [(r, 1) for r in range(6)] + [(6, 6)]:
            label = "%s steps %d..%d" % (path, r, r + k - 1)
            want_s, mc = steps(r, k)
            last = (r + k - 1) & 1
            assert list(zip(bs[last].results(sh), bs[last].calls())) == [want_s] * nconn, label
            assert list(zip(br.results(sh), br.calls())) == [(total, mc)] * nconn, label
            for c in range(nconn):
                dst.land(dbase + c * dstride, total, msgs[last][c], np.zeros(total, np.uint8))
            dst.check(label)
            w = _view(oracle, mtx, mrx)
            for c, (tx, rx) in enumerate(pairs):
                assert _view(G, tx, rx) == w, "%s connection %d" % (label, c)
        src.check("%s sources at the end" % path)
    finally:
        for b in batches:
            b.destroy()
        oracle.destroy(mtx)
        oracle.destroy(mrx)
        for tx, rx in pairs:
            for p in (tx, rx):
                p.disconnect()
                p.putback()
        src.free()
        dst.free()


def test_staged_send_waits_for_the_previous_recv(gpu, oracle):
    """The host-staged lanes run a Send kernel only after the Recv kernels enqueued before it on its lane, whose
    credit it may need.  Eight connections' 1 MiB rings are filled to the brim.  Then, with no host sync, on the same
    lanes: a recv batch over 64 other connections (empty rings, but 2 MiB windows whose whole-window D2H copies take
    milliseconds), the recv batch that drains the eight rings (queued behind those copies), and a 4 KiB Send on each
    of the eight, which fits only once that drain has returned the credit -- its own H2D is a few microseconds."""
    pkg, L = gpu, gpu.lib()
    nx, ny, cap, wide = 8, 64, 1 << 20, 2 << 20
    _config(pkg, cap, "ref")
    xs = [pkg.connected_pair("sw-a%d" % i, "sw-b%d" % i) for i in range(nx)]
    _config(pkg, 1024, "ref")
    ys = [pkg.connected_pair("sw-c%d" % i, "sw-d%d" % i) for i in range(ny)]
    mtx, mrx = oracle.pair_pair(cap)
    fill, small = trace.make_bufs([cap // 2, cap // 2], 301), trace.make_bufs([4096], 302)
    t, r = oracle.pair_pair(cap)  # the premise: behind a full ring the small Send accepts nothing
    oracle.send_all(t, fill, 0)
    assert oracle.send_all(t, small, 0)[0] == 0
    oracle.destroy(t)
    oracle.destroy(r)
    src = Mem(pkg, "staged", 16 << 20)
    dst = Mem(pkg, "staged", 144 << 20)
    batches = []
    try:
        sls = [_place_sends(src, [[None, 0, bufs, 0] for _ in range(nx)], True, np.random.default_rng(1))
               for bufs in (fill, small)]
        xoffs = [dst.alloc(cap, i % 16) for i in range(nx)]
        yoffs = [dst.alloc(wide, i % 16) for i in range(ny)]
        src.upload()
        ub = pkg.UNTIL_BLOCKED
        b_fill = pkg.Batch("send", [(p[0], sl, 2, 0) for p, sl in zip(xs, sls[0])], ub)
        b_small = pkg.Batch("send", [(p[0], sl, 1, 0) for p, sl in zip(xs, sls[1])], ub)
        r_y = pkg.Batch("recv", [(p[1], dst.ptr(o), wide) for p, o in zip(ys, yoffs)], ub)
        r_x = pkg.Batch("recv", [(p[1], dst.ptr(o), cap) for p, o in zip(xs, xoffs)], ub)
        batches = [b_fill, r_y, r_x, b_small]
        for b in batches:  # in this order
            b.launch(None)
        assert L.b200_lanes_join(None) == 0
        want_fill = tuple(int(x) for x in oracle.send_all(mtx, fill, 0))
        out, mc = oracle.recv_drain(mrx, cap)
        want_small = tuple(int(x) for x in oracle.send_all(mtx, small, 0))
        assert want_small == (4096, 1)
        assert list(zip(b_fill.results(), b_fill.calls())) == [want_fill] * nx
        assert list(zip(r_y.results(), r_y.calls())) == [(0, 0)] * ny
        assert list(zip(r_x.results(), r_x.calls())) == [(out.size, int(mc))] * nx
        assert list(zip(b_small.results(), b_small.calls())) == [want_small] * nx, "a Send ran before the drain"
        w = _view(oracle, mtx, mrx)
        for c, (tx, rx) in enumerate(xs):
            assert _view(G, tx, rx) == w, "connection %d" % c
        for o in xoffs:
            dst.land(o, cap, out, np.zeros(cap, np.uint8))
        for o in yoffs:
            dst.land(o, wide, out[:0], np.zeros(wide, np.uint8))
        dst.check("destinations")
        src.check("sources")
    finally:
        for b in batches:
            b.destroy()
        oracle.destroy(mtx)
        oracle.destroy(mrx)
        for tx, rx in xs + ys:
            for p in (tx, rx):
                p.disconnect()
                p.putback()
        src.free()
        dst.free()


# ---- 6. without the service: b200_pairs_send / recv and b200_pairs_submit (the same two launches)

def _mixed_call(pkg, conns, mem, other, runner, label):
    """a Send call and a Recv call whose ops sit in host and in device memory: -1, the documented error, and nothing
    moves (the caller checks the cursors and both arenas)"""
    ops_s, ops_r = [], []
    for k, m in enumerate((mem, other)):
        b = trace.make_bufs([100 + k], 5 + k)[0]
        o = m.alloc(b.size, k)
        m.put(o, b)
        ops_s.append((conns[k].a.h, pkg.make_slices([(m.ptr(o), b.size)]), 1, 0))
        ops_r.append((conns[k].b.h, m.ptr(m.alloc(4096, 3 + k)), 4096))
        m.upload()
    for kind, ops in (("send", ops_s), ("recv", ops_r)):
        if runner == "submit":
            rc = submit(pkg, ops if kind == "send" else (), ops if kind == "recv" else (),
                        pkg.UNTIL_BLOCKED | mem.flags)[0]
        else:
            n = len(ops)
            arr = ((pkg.SendOp if kind == "send" else pkg.RecvOp) * n)()
            for i, op in enumerate(ops):
                if kind == "send":
                    arr[i].pair, arr[i].slices, arr[i].nslices, arr[i].byte_idx = op
                else:
                    arr[i].pair, arr[i].dst, arr[i].cap = op
            out = (C.c_uint64 * n)()
            f = pkg.lib().b200_pairs_send if kind == "send" else pkg.lib().b200_pairs_recv
            rc = f(arr, n, pkg.UNTIL_BLOCKED | mem.flags, out, None)
        assert rc == -1 and "cannot be mixed" in pkg.last_error(), "%s: mixed %s call: rc %d (%s)" % (
            label, kind, rc, pkg.last_error())
    _check_all(conns, [mem, other], label + " after the mixed calls")


@pytest.mark.parametrize("runner", ["pairs", "submit"])
def test_without_the_service(gpu, models, path, runner):
    """Rounds of test 1 (24 connections) through unprepared b200_pairs_send / b200_pairs_recv, or b200_pairs_submit
    with the service stopped; every round first makes a Send call and a Recv call that mix host and device buffers."""
    pkg = gpu
    assert pkg.lib().b200_service_running() == 0
    other = Mem(pkg, "staged" if path == "device" else "device", 1 << 20)
    try:
        _random_rounds(pkg, models, path, 7500 + PATHS.index(path), nconn=24, rounds=4, runner=runner, other=other)
    finally:
        other.free()
