"""GPU: posted ops -- b200_pair_post_send / b200_pair_post_recv, polled to the end with b200_async_poll -- against the
CPU models, pass by pass.

A pass posts one op per planned (connection, direction) with test_submit_gpu's planner, then polls every op it
posted to the end.  When an owner queue has no free entry (again == 1) the ops posted so far are polled to the end
and the op is posted again.  After every pass each op's count and the bytes it delivered, both pairs' cursors, the
readiness answers and the receivers' ring images are compared with the models.  Slices come from plain numpy memory
(staged in pinned memory the op owns), b200_mem_alloc_host, registered memory and device memory; destinations are
pinned host, registered or device memory."""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import trace
from test_submit_gpu import (MODES, Conn, Service, _check_conn, _check_image, _compare_pass, _desc, _model_pass,
                             _models, _plan, _views)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ONE_CALL, UNTIL_BLOCKED = 0, 1  # B200_BATCH_ONE_CALL, B200_BATCH_UNTIL_BLOCKED
FLAGS = {"one_call": ONE_CALL, "until_blocked": UNTIL_BLOCKED}


@pytest.fixture(scope="module")
def models(oracle):
    return _models(oracle)


@pytest.fixture
def svc(gpu, request):
    with Service(gpu, **getattr(request, "param", {})) as s:
        yield s


def _finish(pkg, op, label):
    """poll a posted op to the end: the bytes it moved"""
    L = pkg.lib()
    n = C.c_uint64()
    t0 = time.monotonic()
    while True:
        rc = L.b200_async_poll(op, C.byref(n))
        if rc:
            break
        assert time.monotonic() - t0 < 60, "%s: the op did not finish" % label
    assert rc == 1, "%s: b200_async_poll %d (%s)" % (label, rc, pkg.last_error())
    return n.value


def _run_posted(pkg, conns, plan, arena, flags):
    """post `plan` as posted ops and poll them to the end: per op (count, SHA-1 of the bytes delivered), every
    connection's view of both directions, and how often a post found its owner queue full"""
    L = pkg.lib()
    arena.reset()
    res, posted, full = [None] * len(plan), [], 0

    def finish_posted():
        for i, h, dst in posted:
            n = _finish(pkg, h, _desc(plan[i]))
            op = plan[i]
            res[i] = (int(n), None) if op[0] == "send" else (int(n), trace.sha(arena.get(op[4], dst, n)))
        posted.clear()

    for i, op in enumerate(plan):
        tx, rx = op[1].ends(op[2])[:2]
        dst = None
        if op[0] == "send":
            sl = arena.place(op[3], op[5], i)
        else:
            dst = arena.alloc(op[4], op[3], i % 16)
        while True:
            again = C.c_int(-1)
            if op[0] == "send":
                h = L.b200_pair_post_send(tx.h, sl, len(op[3]), op[4], flags, C.byref(again))
            else:
                h = L.b200_pair_post_recv(rx.h, dst, op[3], flags, C.byref(again))
            if h or again.value != 1:
                break
            full += 1
            finish_posted()
        assert h and again.value == 0, "%s: post refused (%s)" % (_desc(op), pkg.last_error())
        posted.append((i, h, dst))
    finish_posted()
    return {"rc": 0, "err": "", "res": res, "views": [_views(c, False) for c in conns]}, full


def _model_one_call(conns, plan):
    """_model_pass for B200_BATCH_ONE_CALL ops: one Send call, one Recv call"""
    res = []
    for op in plan:
        c = op[1]
        _, _, mtx, mrx = c.ends(op[2])
        if op[0] == "send":
            res.append((int(c.model.send(mtx, op[3], op[4])), None))
        else:
            out = c.model.recv(mrx, op[3])
            res.append((int(out.size), trace.sha(out)))
    return {"rc": 0, "err": "", "res": res, "views": [_views(c, True) for c in conns]}


def _check_posted(pkg, conns, plan, arena, flags, label):
    got, full = _run_posted(pkg, conns, plan, arena, flags)
    want = _model_pass(conns, plan) if flags == UNTIL_BLOCKED else _model_one_call(conns, plan)
    _compare_pass(conns, plan, got, want, label)
    for c in conns:
        for d in (0, 1):
            _check_image(c, d, label)
    return full


def _passes(pkg, models, arena, flags, seed, mode_of, nconn, npasses, dst_kinds=("host", "registered", "device")):
    rng = np.random.default_rng(seed)
    conns = [Conn(pkg, models, mode_of(i), (1024, 4096, 8192)[i % 3]) for i in range(nconn)]
    full = 0
    try:
        for p in range(npasses):
            plan = _plan(rng, conns, dst_kinds=dst_kinds)
            full += _check_posted(pkg, conns, plan, arena, flags, "pass %d" % p)
    finally:
        for c in conns:
            c.close()
    return full


@pytest.mark.parametrize("flags", sorted(FLAGS))
@pytest.mark.parametrize("mode", MODES)
def test_posted_passes(svc, models, mode, flags):
    """9 connections of one framing mode, 8 passes; every memory kind of Send slice and Recv destination."""
    _passes(svc.pkg, models, svc.arena, FLAGS[flags], 6100 + 2 * MODES.index(mode) + FLAGS[flags],
            lambda i: mode, 9, 8)


@pytest.mark.parametrize("svc", [dict(owners=1, workers=2)], indirect=True, ids=["owners1-workers2"])
@pytest.mark.parametrize("flags", sorted(FLAGS))
def test_full_owner_queue(svc, models, flags):
    """One owner queue of 16 entries and 24 connections of all three modes: a pass posts more ops than the queue
    holds, so posts come back with again == 1 and are posted again once the earlier ops are polled."""
    full = _passes(svc.pkg, models, svc.arena, FLAGS[flags], 6200 + FLAGS[flags], lambda i: MODES[i % 3], 24, 6)
    assert full > 0, "no post found the owner queue full"


def test_unregistered_destination_is_refused(svc, models):
    """A posted Recv into unregistered host memory is refused while a frame waits (again == 0, the pair's error
    says why) and changes nothing; the frame is delivered afterwards."""
    pkg, L, a = svc.pkg, svc.L, svc.arena
    c = Conn(pkg, models, "ref", 4096)
    try:
        a.reset()
        bufs = trace.make_bufs([300, 9, 700], 5)
        sl = a.place(bufs, ["plain", "host", "device"])
        again = C.c_int(-1)
        h = L.b200_pair_post_send(c.a.h, sl, 3, 0, UNTIL_BLOCKED, C.byref(again))
        assert h and again.value == 0, pkg.last_error()
        assert _finish(pkg, h, "send") == c.model.send_all(c.ma, bufs, 0)[0]
        before = (_views(c, False), c.b.ring_image())
        plain = np.zeros(4096, np.uint8)
        again = C.c_int(-1)
        assert not L.b200_pair_post_recv(c.b.h, plain.ctypes.data, 4096, UNTIL_BLOCKED, C.byref(again))
        assert again.value == 0 and "GPU-addressable" in pkg.last_error()
        assert not plain.any()
        assert _views(c, False) == before[0] and np.array_equal(c.b.ring_image(), before[1])
        dst = a.alloc("registered", 4096)
        h = L.b200_pair_post_recv(c.b.h, dst, 4096, UNTIL_BLOCKED, C.byref(again))
        assert h and again.value == 0, pkg.last_error()
        n = _finish(pkg, h, "recv")
        want, _ = c.model.recv_drain(c.mb, 4096)
        assert np.array_equal(a.get("registered", dst, n), want)
        _check_conn(c, "after the refusal")
    finally:
        c.close()


# ---- B200_SUBMIT_STAGE_MIN (read once per process): posted Recvs into pinned host memory through device staging

def stage_min_child():
    """run by test_stage_min_in_a_subprocess in a process of its own"""
    import __graft_entry__ as ge
    import orlib
    pkg = ge.load_package()
    pkg.init(0)
    models = _models(orlib.Oracle())
    with Service(pkg, workers=4) as s:
        for flags in (UNTIL_BLOCKED, ONE_CALL):
            _passes(pkg, models, s.arena, flags, 6300 + flags, lambda i: MODES[i % 3], 9, 5,
                    dst_kinds=("host", "registered"))
    print("stage-min ok")


def test_stage_min_in_a_subprocess():
    code = "import sys; sys.path[:0] = [%r, %r]; import test_post_poll_gpu; test_post_poll_gpu.stage_min_child()" % (
        ROOT, HERE)
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, B200_SUBMIT_STAGE_MIN="1"),
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "stage-min ok" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]
