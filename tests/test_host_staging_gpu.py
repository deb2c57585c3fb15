"""GPU: the host staging of plain (unregistered) Send slices, at its edges and at its limits, on every host Send path,
against the CPU models.

Before a kernel reads a plain host slice, the runtime copies it to pinned memory (stage_send in b200_runtime.cu).  A
one-call op stages only what one call can read, the first C/2 bytes from byte_idx on; an until-blocked op stages the
slices it looks at whole, or a prefix of them when its buffer is too small.  The paths fill different buffers:
  launch                    b200_pair_send with the service stopped (the calling thread's tx bounce)
  service                   b200_pair_send with the service running (the same bounce)
  submit_one / submit_ub    a b200_pairs_submit pass, B200_BATCH_ONE_CALL / UNTIL_BLOCKED (one bounce per pass)
  posted_one / posted_ub    b200_pair_post_send (a pinned block the op owns)
Each op is compared with the model of its connection's framing mode: a one-call op with one Send, an until-blocked op
with the rdma_flush loop over the slices it looks at.  Then both ends' views and the receiver's ring image, and after
a drain the delivered bytes with the source bytes.

The limits (the pass bounce's 1 GiB, the 2^28-byte block of a posted until-blocked op, the whole need of a one-call
op, the largest device staging class of a service Recv) need gigabytes: host_staging_worker.py runs those cases in
a process of its own, so that the pinned buffers the runtime keeps for a thread's or the pool's later use go with it."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import trace
from gpu_engine import GpuEngine
from submit_lib import SLICE_AREA, Arena, submit
from test_post_poll_gpu import _finish
from test_submit_gpu import MODES, Conn, Service, _advance, _check_conn, _models

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

HERE = os.path.dirname(os.path.abspath(__file__))
ONE_CALL, UB = 0, 1  # B200_BATCH_ONE_CALL, B200_BATCH_UNTIL_BLOCKED
PATHS = ("launch", "service", "submit_one", "submit_ub", "posted_one", "posted_ub")
MAX_SGE = 30  # GRPC_RDMA_MAX_SGE of every Conn


@pytest.fixture(scope="module")
def models(oracle):
    return _models(oracle)


def one_call(path):
    return not path.endswith("_ub")


def send_on(pkg, path, tx, sl, n, bidx):
    """one Send op of `path` over sl[:n] from byte bidx of sl[0]: the bytes it accepted"""
    L = pkg.lib()
    if path in ("launch", "service"):
        return L.b200_pair_send(tx.h, sl, n, bidx)
    flags = ONE_CALL if one_call(path) else UB
    if path.startswith("submit"):
        rc, acc, _ = submit(pkg, [(tx.h, sl, n, bidx)], (), flags)
        assert rc == 0, pkg.last_error()
        return acc[0]
    again = C.c_int(-1)
    h = L.b200_pair_post_send(tx.h, sl, n, bidx, flags, C.byref(again))
    assert h and again.value == 0, "post_send refused: %s" % pkg.last_error()
    return _finish(pkg, h, "posted send")


def recv_on(pkg, path, rx, dst, cap):
    """an until-blocked Recv into GPU-addressable dst through the submit or the posted form of `path`"""
    L = pkg.lib()
    if path.startswith("submit"):
        rc, _, dlv = submit(pkg, (), [(rx.h, dst, cap)], UB)
        assert rc == 0, pkg.last_error()
        return dlv[0]
    again = C.c_int(-1)
    h = L.b200_pair_post_recv(rx.h, dst, cap, UB, C.byref(again))
    assert h and again.value == 0, "post_recv refused: %s" % pkg.last_error()
    return _finish(pkg, h, "posted recv")


def send_like_the_endpoint(pkg, path, c, sl, bufs, bidx, label):
    """A one-call path: one op, against one Send of the model.  An until-blocked path: the endpoint's rdma_flush loop,
    which posts the rest again from the returned position while an op accepts bytes; each op against the model's
    rdma_flush loop over the slices the op looks at (SLICE_AREA - 1).  The bytes accepted in all."""
    lens = [b.size for b in bufs]
    idx = total = 0
    while True:
        rest = sl if idx == 0 else pkg.make_slices([(sl[i].ptr, sl[i].len) for i in range(idx, len(lens))])
        n = send_on(pkg, path, c.a, rest, len(lens) - idx, bidx)
        if one_call(path):
            want = c.model.send(c.ma, bufs, bidx)
        else:
            want = c.model.send_all(c.ma, bufs[idx:idx + SLICE_AREA - 1], bidx)[0]
        assert n == want, "%s: the op from slice %d byte %d accepted %d, the model %d" % (label, idx, bidx, n, want)
        total += n
        if one_call(path) or not n:
            return total
        idx, bidx = _advance(lens, idx, bidx, n)
        if idx == len(lens):
            return total


# ---- 1. the stager's edges on every path

MIXED = ("plain", "host", "plain", "registered", "plain", "device")


def _cases(cap):
    """(label, slice lengths, byte_idx, memory kinds) at the edges of what one op stages on a ring of `cap` bytes"""
    h = cap // 2
    out = []
    for n in (h - 1, h, h + 1):  # one call reads at most C/2 bytes
        for b in (0, 15):
            out.append(("one plain slice of %d from byte %d" % (n, b), [n], b, ["plain"]))
    # several slices whose bytes cross C/2 inside a plain slice (coalesced framing gathers them into one frame)
    lens = [h // 3 + 1, h // 3 + 2, h // 2 + 7, 5]
    out.append(("C/2 inside a slice, plain", lens, 3, ["plain"] * 4))
    out.append(("C/2 inside a slice, mixed", lens, 3, ["plain", "host", "plain", "device"]))
    out.append(("a zero-length slice at C/2", [h - 8, 8, 0, 9], 0, ["plain", "registered", "plain", "plain"]))
    # slice counts at the windows: max_sge (per-slice framing), 1024 (coalesced), 1023 (until-blocked)
    for n in (MAX_SGE, MAX_SGE + 1, SLICE_AREA - 1, SLICE_AREA, SLICE_AREA + 1):
        unit = max(1, cap // n)
        lens = [unit + i % 3 for i in range(n)]  # together about C: the C/2 edge falls inside the window
        kinds = ["plain"] * n if n % 2 == 0 else [MIXED[i % len(MIXED)] for i in range(n)]
        out.append(("%d slices" % n, lens, min(15, lens[0] - 1), kinds))
    # zero-length plain slices at every window edge
    for zeros in ((MAX_SGE - 1, MAX_SGE, SLICE_AREA - 2, SLICE_AREA - 1, SLICE_AREA), (0, SLICE_AREA - 1)):
        lens = [7 + i % 5 for i in range(SLICE_AREA + 2)]
        for z in zeros:
            lens[z] = 0
        out.append(("zero-length slices at %s" % (zeros,), lens, 0, ["plain"] * len(lens)))
    return out


def _drain(pkg, path, c, arena):
    """one rdma_do_read loop at c.b (launched, or an until-blocked op of the service) and at the model"""
    if path == "launch":
        got = GpuEngine(pkg).recv_drain(c.b, 2 * c.cap)[0]
    else:
        dst = arena.alloc("host", 2 * c.cap)
        got = arena.get("host", dst, recv_on(pkg, "posted" if path.startswith("posted") else "submit", c.b, dst,
                                             2 * c.cap))
    want, _ = c.model.recv_drain(c.mb, 2 * c.cap)
    return got, want


def _edges(pkg, models, path, mode, arena):
    for cap in (64, 4096, 1 << 20):
        c = Conn(pkg, models, mode, cap)
        try:
            for k, (what, lens, bidx, kinds) in enumerate(_cases(cap)):
                label = "%s %s ring %d: %s" % (path, mode, cap, what)
                bufs = trace.make_bufs(lens, 50 + k)
                arena.reset()
                sl = arena.place(bufs, kinds, k)
                got = send_like_the_endpoint(pkg, path, c, sl, bufs, bidx, label)
                _check_conn(c, label)
                dg, dw = _drain(pkg, path, c, arena)
                assert np.array_equal(dg, dw), "%s: delivered bytes differ from the model's" % label
                assert np.array_equal(dg, np.concatenate(bufs)[bidx:bidx + got]), "%s: not the source bytes" % label
                _check_conn(c, label + ", drained")
        finally:
            c.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("path", PATHS)
def test_stager_edges(gpu, models, path, mode):
    """Rings of 64 B, 4 KiB and 1 MiB; one plain slice of C/2 - 1, C/2 and C/2 + 1 bytes from byte 0 and 15; slices
    whose bytes cross C/2 inside a plain one; max_sge, 1023, 1024 slices and one more, plain alone or mixed with
    pinned, registered and device slices; zero-length plain slices at the window edges."""
    if path == "launch":
        arena = Arena(gpu, 8 << 20)
        try:
            launches = gpu.lib().b200_launch_count()
            _edges(gpu, models, path, mode, arena)
            assert gpu.lib().b200_launch_count() > launches
        finally:
            arena.free()
        return
    with Service(gpu, arena=8 << 20) as s:
        launches = s.L.b200_launch_count()
        _edges(gpu, models, path, mode, s.arena)
        assert s.L.b200_launch_count() == launches  # every op ran in the resident kernels


# ---- 2. the limits, in processes of their own (host_staging_worker.py)

def _worker(cases, env=None):
    out = subprocess.run([sys.executable, os.path.join(HERE, "host_staging_worker.py")] + cases,
                         env=dict(os.environ, **(env or {})), capture_output=True, text=True, timeout=1700)
    ok = all(("case %s ok" % k) in out.stdout for k in cases)
    assert out.returncode == 0 and ok, out.stdout[-6000:] + out.stderr[-4000:]
    print(out.stdout)  # what each case did, and the worker's peak RSS


@pytest.mark.timeout(1800)
def test_staging_limits_in_a_subprocess():
    """a: a posted until-blocked Send of one plain slice of 2^28 + 16 bytes (larger than such an op's block) on a
    4 MiB ring; b: the same through a pass with 2^30 + 16 bytes (larger than the pass's bounce); c: an until-blocked
    pass of six 200 MiB slices (together larger than the bounce); d: a one-call pass of five 256 MiB slices on
    512 MiB rings; e: posted one-call Sends whose need is larger than an until-blocked op's block; f: a service Recv
    into pinned host memory with a 2^40-byte capacity."""
    _worker(["a", "b", "c", "d", "e", "f"])


def test_recv_staging_classes_in_a_subprocess():
    """B200_SUBMIT_STAGE_MIN=1 (read once per process): a service Recv into pinned host memory with a capacity of
    2^31 bytes goes through the largest device staging class, one of 2^31 + 1 bytes writes in place."""
    _worker(["g"], {"B200_SUBMIT_STAGE_MIN": "1"})
