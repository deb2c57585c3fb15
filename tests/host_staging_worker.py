"""The limits of the host staging of the service's Send and Recv paths, for tests/test_host_staging_gpu.py.  The cases
need gigabytes of host and pinned memory; they run in a process of their own so that the pinned buffers the runtime
keeps for later use (a thread's tx bounce, the posted ops' staging blocks) are released when it exits.

    python host_staging_worker.py <case>...

    a  a posted until-blocked Send of one plain slice of 2^28 + 16 bytes on a 4 MiB ring, from byte 0 and 15
    b  the same through b200_pairs_submit with 2^30 + 16 bytes
    c  an until-blocked pass of six Sends of one 200 MiB plain slice each, on 4 MiB rings
    d  a one-call pass of five Sends of one 256 MiB plain slice each, on 512 MiB rings
    e  posted one-call Sends: one 600 MiB plain slice on a 1 GiB ring; 1024 odd-length plain slices of more than
       256 MiB in all on a coalesced 512 MiB ring
    f  a posted and a submitted Recv into pinned host memory with a capacity of 2^40 bytes
    g  (with B200_SUBMIT_STAGE_MIN=1) the same with capacities of 2^31 + 1 and 2^31 bytes

a-c and f are compared with the models op by op.  The CPU model of a 512 MiB or 1 GiB ring costs more host memory
than the GPU twin of the connection, so d and e compare each op with a twin driven by b200_pair_send with the service
running (test_stager_edges checks that path against the models): answers, views, ring images and delivered bytes.
Each case prints "case <x> ok" or "case <x> FAILED: <why>"; the exit status is 1 when one failed.  The process's
peak RSS is printed at the end."""
import ctypes as C
import hashlib
import os
import resource
import sys
import traceback

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import __graft_entry__ as ge  # noqa: E402
import orlib  # noqa: E402
import trace  # noqa: E402
from test_host_staging_gpu import ONE_CALL, UB, recv_on, send_on  # noqa: E402
from test_submit_gpu import G, MODES, Conn, Service, _check_conn, _config, _models, _view  # noqa: E402
from submit_lib import submit  # noqa: E402

MiB, GiB = 1 << 20, 1 << 30


def random_bytes(n, seed):
    return np.frombuffer(np.random.default_rng(seed).bytes(n), np.uint8)


def at(ptr, n):
    """n bytes of host memory at ptr, without a copy"""
    return np.ctypeslib.as_array((C.c_uint8 * n).from_address(ptr)) if n else np.zeros(0, np.uint8)


def stream(pkg, models, arena, path, src, bidx, label):
    """One plain slice through a 4 MiB connection the way the endpoint sends it: an until-blocked op from the current
    position, then a drain, until everything has arrived.  Every op against the model."""
    c = Conn(pkg, models, "ref", 4 * MiB)
    try:
        arena.reset()
        dst = arena.alloc("host", c.cap)
        sl = pkg.make_slices([(src.ctypes.data, src.size)])
        pos, k = bidx, 0
        while pos < src.size:
            n = send_on(pkg, path, c.a, sl, 1, pos)
            want = c.model.send_all(c.ma, [src], pos)[0]
            assert n == want, "%s, op %d from byte %d: accepted %d, the model %d" % (label, k, pos, n, want)
            if k == 0:
                _check_conn(c, label, dirs=(0,))
            m = recv_on(pkg, path, c.b, dst, c.cap)
            out, _ = c.model.recv_drain(c.mb, c.cap)
            assert np.array_equal(at(dst, m), out), "%s, op %d: delivered bytes differ from the model's" % (label, k)
            assert np.array_equal(out, src[pos:pos + n]), "%s, op %d: not the source bytes" % (label, k)
            pos += n
            k += 1
            assert k < 10000, "%s: no progress" % label
        _check_conn(c, label + ", at the end", dirs=(0,))
        print("  %s: %d ops" % (label, k))
    finally:
        c.close()


def case_a(pkg, models):
    src = random_bytes((1 << 28) + 16, 1)
    with Service(pkg, arena={"host": 8 * MiB}) as s:
        for bidx in (0, 15):
            stream(pkg, models, s.arena, "posted_ub", src, bidx, "posted 2^28 + 16 from byte %d" % bidx)


def case_b(pkg, models):
    src = random_bytes(GiB + 16, 2)
    with Service(pkg, arena={"host": 8 * MiB}) as s:
        for bidx in (0, 15):
            stream(pkg, models, s.arena, "submit_ub", src, bidx, "submitted 2^30 + 16 from byte %d" % bidx)


def case_c(pkg, models):
    size = 200 * MiB
    src = random_bytes(size + 6 * 4099, 3)
    bufs = [src[4099 * i:4099 * i + size] for i in range(6)]
    with Service(pkg, arena={"host": 8 * MiB}) as s:
        conns = [Conn(pkg, models, MODES[i % 3], 4 * MiB) for i in range(6)]
        try:
            sends = [(c.a.h, pkg.make_slices([(b.ctypes.data, size)]), 1, i) for i, (c, b) in enumerate(zip(conns, bufs))]
            rc, acc, _ = submit(pkg, sends, (), UB)
            assert rc == 0, pkg.last_error()
            want = [int(c.model.send_all(c.ma, [b], i)[0]) for i, (c, b) in enumerate(zip(conns, bufs))]
            assert acc == want, "accepted %s, the models %s" % (acc, want)
            s.arena.reset()
            dst = s.arena.alloc("host", 4 * MiB)
            for i, c in enumerate(conns):
                label = "op %d (%s)" % (i, c.mode)
                _check_conn(c, label)
                rc, _, dlv = submit(pkg, (), [(c.b.h, dst, 4 * MiB)], UB)
                out, _ = c.model.recv_drain(c.mb, 4 * MiB)
                assert rc == 0 and np.array_equal(at(dst, dlv[0]), out), label
                assert np.array_equal(out, bufs[i][i:i + acc[i]]), label + ": not the source bytes"
                _check_conn(c, label + ", drained")
        finally:
            for c in conns:
                c.close()


def gpu_conn(pkg, mode, cap, name):
    _config(pkg, cap, mode)
    try:
        return pkg.connected_pair(name + "a", name + "b")
    finally:
        _config(pkg, 4096, "ref")


def close(conns):
    for tx, rx in conns:
        for p in (tx, rx):
            p.disconnect()
            p.putback()


def image_sha(p):
    """SHA-1 of p's ring image with the frame pads masked (trace.sha without its copy: the rings here are large)"""
    img = p.ring_image()
    img = trace.mask_pads(img, p.state(), img.size)
    return hashlib.sha1(memoryview(img)).hexdigest()


def twin_check(pkg, arena, conns, twin, acc, src, label):
    """conns against the twin connection, which took the same Send through b200_pair_send; then each one drained
    and its bytes checked against src"""
    (ttx, trx), tacc = twin, acc[-1]
    assert all(a == tacc for a in acc), "%s: accepted %s, the twin (last) %d" % (label, acc, tacc)
    assert tacc > 0, "%s: nothing accepted" % label
    want = [_view(G, ttx, trx), _view(G, trx, ttx)]
    wimg = image_sha(trx)
    arena.reset()
    dst = arena.alloc("host", tacc)
    for i, (tx, rx) in enumerate(conns + [twin]):
        assert [_view(G, tx, rx), _view(G, rx, tx)] == want, "%s: connection %d's views differ from the twin's" % (label, i)
        if i < len(conns):
            assert image_sha(rx) == wimg, "%s: connection %d's ring differs from the twin's" % (label, i)
        rc, _, dlv = submit(pkg, (), [(rx.h, dst, tacc)], UB)
        assert rc == 0 and dlv[0] == tacc, "%s: connection %d delivered %d of %d" % (label, i, dlv[0], tacc)
        assert np.array_equal(at(dst, tacc), src[:tacc]), "%s: connection %d: not the source bytes" % (label, i)
        if i == 0:
            drained = [_view(G, tx, rx), _view(G, rx, tx)]
        assert [_view(G, tx, rx), _view(G, rx, tx)] == drained, "%s: connection %d, drained" % (label, i)


def case_d(pkg, models):
    size, cap = 256 * MiB, 512 * MiB
    src = random_bytes(size, 4)
    with Service(pkg, arena={"host": size + MiB}) as s:
        conns = [gpu_conn(pkg, "ref", cap, "d%d" % i) for i in range(5)]
        twin = gpu_conn(pkg, "ref", cap, "dt")
        try:
            sl = pkg.make_slices([(src.ctypes.data, size)])
            rc, acc, _ = submit(pkg, [(tx.h, sl, 1, 0) for tx, _ in conns], (), ONE_CALL)
            assert rc == 0, pkg.last_error()
            acc.append(send_on(pkg, "service", twin[0], sl, 1, 0))
            twin_check(pkg, s.arena, conns, twin, acc, src, "five 256 MiB one-call ops in one pass")
        finally:
            close(conns + [twin])


def case_e(pkg, models):
    # one slice larger than C/2 of a 1 GiB ring: the call reads C/2 = 512 MiB of it
    src = random_bytes(600 * MiB, 5)
    with Service(pkg, arena={"host": 512 * MiB + MiB}) as s:
        one, twin = gpu_conn(pkg, "ref", GiB, "e1"), gpu_conn(pkg, "ref", GiB, "e1t")
        try:
            sl = pkg.make_slices([(src.ctypes.data, src.size)])
            acc = [send_on(pkg, "posted_one", one[0], sl, 1, 0), send_on(pkg, "service", twin[0], sl, 1, 0)]
            twin_check(pkg, s.arena, [one], twin, acc, src, "posted 600 MiB on a 1 GiB ring")
        finally:
            close([one, twin])
    del src
    # 1024 odd-length slices: the coalesced call reads the first 256 MiB of them, staged in 16-byte steps
    lens = [262145 + 2 * (i % 5) for i in range(1024)]
    offs = np.cumsum([0] + [n + 3 for n in lens[:-1]])
    flat = random_bytes(int(offs[-1]) + lens[-1], 6)
    src = np.concatenate([flat[o:o + n] for o, n in zip(offs, lens)])
    assert src.size > 256 * MiB
    with Service(pkg, arena={"host": 256 * MiB + MiB}) as s:
        one, twin = gpu_conn(pkg, "coal", 512 * MiB, "e2"), gpu_conn(pkg, "coal", 512 * MiB, "e2t")
        try:
            sl = pkg.make_slices([(flat.ctypes.data + int(o), n) for o, n in zip(offs, lens)])
            acc = [send_on(pkg, "posted_one", one[0], sl, len(lens), 0), send_on(pkg, "service", twin[0], sl, len(lens), 0)]
            twin_check(pkg, s.arena, [one], twin, acc, src, "posted coalesced 1024 odd slices on a 512 MiB ring")
        finally:
            close([one, twin])


def recv_caps(pkg, models, caps):
    """a 100-byte frame, then a posted and a submitted Recv of each capacity into pinned host memory"""
    with Service(pkg, arena={"host": MiB}) as s:
        c = Conn(pkg, models, "ref", 4096)
        try:
            s.arena.reset()
            dst = s.arena.alloc("host", 4096)
            for k, cap in enumerate(caps):
                for path in ("posted", "submit"):
                    label = "%s Recv of capacity %d" % (path, cap)
                    bufs = trace.make_bufs([100], 70 + k)
                    assert c.a.send(bufs) == c.model.send(c.ma, bufs) == 100, label
                    n = recv_on(pkg, path, c.b, dst, cap)
                    out, _ = c.model.recv_drain(c.mb, 4096)
                    assert n == out.size == 100 and np.array_equal(at(dst, n), out), label
                    _check_conn(c, label)
        finally:
            c.close()


def case_f(pkg, models):
    recv_caps(pkg, models, [1 << 40])


def case_g(pkg, models):
    assert os.environ.get("B200_SUBMIT_STAGE_MIN") == "1"
    recv_caps(pkg, models, [(1 << 31) + 1, 1 << 31])


def main():
    pkg = ge.load_package()
    pkg.init(0)
    models = _models(orlib.Oracle())
    failed = False
    for name in sys.argv[1:]:
        try:
            globals()["case_" + name](pkg, models)
            print("case %s ok" % name, flush=True)
        except Exception as ex:  # reported, and the next case runs
            failed = True
            print("case %s FAILED: %s" % (name, ex), flush=True)
            traceback.print_exc()
    print("peak RSS %d MiB" % (resource.getrusage(resource.RUSAGE_SELF).ru_maxrss // 1024), flush=True)
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
