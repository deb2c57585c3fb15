"""Mirrored against unmirrored device claims (b200_pair_device_claim_ex, B200_CLAIM_UNMIRRORED): what publishing the
host-visible mirror costs the device calls.  The two claims alternate in one process on the same connections and
buffers, --reps rounds of each; medians (and every round) are printed as one JSON line, with the card's name and power
limit read in the same run.

  pingpong   1 KiB round trips between two device warps on one loopback connection (tests/native/device_api.cu, the
             time is %globaltimer in the ping warp): p50 / p99 over --rounds per round
  serve      one polling server warp (b200_warp_poll -> b200_warp_recv -> b200_warp_send) against one client warp per
             connection, 64 connections, 1 KiB requests (tests/native/device_poll.cu): round trips per second.  The
             clients disconnect at the end, so every round connects the 64 connections afresh
  stream     256 connections x one chttp2-shaped 4 MiB message, 16 MiB rings: one kernel of block sends
             (B200_BATCH_UNTIL_BLOCKED, one CTA per connection, tests/native/device_block.cu), then one kernel of block
             receives; CUDA events, GB/s of payload

    python tools/unmirrored_ab.py [--reps 5] [--rounds 2000] [--serve-rounds 300]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from device_block_stream import _setup, _teardown  # noqa: E402
from device_serve import card, connections, drop  # noqa: E402

MODES = (("mirrored", True), ("unmirrored", False))


def pingpong(pkg, dl, reps, rounds, size=1024):
    L = pkg.lib()
    pkg.config_set("GRPC_RDMA_RING_BUFFER_SIZE_KB", 4096)
    R = dl.Runner(pkg)
    msg, back, got = (L.b200_mem_alloc_device(size) for _ in range(3))
    times = L.b200_mem_alloc_host(8 * rounds)
    slp = L.b200_mem_alloc_host(16)
    s = (pkg.Slice * 1).from_address(slp)
    s[0].ptr, s[0].len = msg, size
    t = np.ctypeslib.as_array((C.c_uint64 * rounds).from_address(times))
    a, b = pkg.connected_pair("uab-pa", "uab-pb")
    out = {m: [] for m, _ in MODES}
    for rep in range(reps + 1):  # round 0 warms both modes up
        for mode, mirrored in MODES:
            ha, hb = a.device_claim(mirrored), b.device_claim(mirrored)
            res = R.run([ha, hb], [[dict(kind=dl.PING, pair=0, slices=slp, n=rounds, byte_idx=1, dst=got, times=times)],
                                   [dict(kind=dl.PONG, pair=1, dst=back, cap=size, n=rounds)]], budget_s=60.0)
            assert all(o[0]["status"] == dl.OK for o in res), res
            a.device_release()
            b.device_release()
            if rep:
                x = np.sort(t[rounds // 10:].astype(np.float64)) / 1e3
                out[mode].append((float(np.percentile(x, 50)), float(np.percentile(x, 99))))
    a.disconnect(); b.disconnect(); a.putback(); b.putback()
    for p in (msg, back, got):
        L.b200_mem_free_device(p)
    for p in (times, slp):
        L.b200_mem_free_host(p)
    return {m: {"p50_us": round(statistics.median(v[0] for v in out[m]), 2),
                "p99_us": round(statistics.median(v[1] for v in out[m]), 2),
                "rounds_p50_us": [round(v[0], 2) for v in out[m]]} for m, _ in MODES}


def serve(pkg, dpl, reps, rounds, n=64, msg=1024):
    L = pkg.lib()
    R = dpl.Runner(pkg)
    bufs = [L.b200_mem_alloc_device(x) for x in (12 * n, n * msg, 2 * n * msg)]
    state, sbuf, cbuf = bufs
    tp, times = R.mem.array("times", np.uint64, n * rounds)
    op, res = R.mem.array("out", np.uint64, 4 * n + 4)
    z = np.zeros(3 * n, np.uint32)
    out = {m: [] for m, _ in MODES}
    try:
        for rep in range(reps + 1):
            for mode, mirrored in MODES:
                conns = connections(pkg, n, 16384, "uab-s")  # (the clients close their connections at the end)
                srv = R.handles("srv", [a.device_claim(mirrored) for a, b in conns])
                cli = R.handles("cli", [b.device_claim(mirrored) for a, b in conns])
                assert L.b200_memcpy(state, z.ctypes.data, z.nbytes, 0, None) == 0 and L.b200_stream_sync(None) == 0
                res[:] = 0
                s = dpl.DpServe(srv=srv, cli=cli, n=n, rounds=rounds, msg=msg, mode=0, sbuf=sbuf, cbuf=cbuf,
                                state=state, times=tp, out=op, budget_ns=int(120e9), max_iters=1 << 40)
                t0 = time.perf_counter()
                assert R.D.dp_serve_launch(C.byref(s)) == 0, R.D.dp_error().decode()
                assert R.D.dp_wait() == 0, R.D.dp_error().decode()
                wall = time.perf_counter() - t0
                per = res[:4 * n].reshape(n, 4)
                assert (per[:, 0] == 0).all() and (per[:, 1] == 0).all() and (per[:, 2] == rounds).all(), per[:4]
                drop(conns)
                if rep:
                    x = np.sort(times.reshape(n, rounds)[:, rounds // 10:].reshape(-1)) / 1e3
                    out[mode].append((n * rounds / wall, float(x[len(x) // 2])))
    finally:
        for p in bufs:
            L.b200_mem_free_device(p)
        R.close()
    return {m: {"conns": n, "round_trips_per_s": round(statistics.median(v[0] for v in out[m])),
                "p50_us": round(statistics.median(v[1] for v in out[m]), 2),
                "rounds_per_s": [round(v[0]) for v in out[m]]} for m, _ in MODES}


def stream(pkg, bl, torch, reps, conns=256, msg=4 << 20):
    S = _setup(pkg, conns, 16384, msg, "uab-b")
    total, nl = S["total"], len(S["lens"])
    st = torch.cuda.Stream()
    sp = st.cuda_stream
    RS, RR = bl.Runner(pkg), bl.Runner(pkg)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]

    def step(mirrored):
        h = []
        for tx, rx in S["pairs"]:
            h += [tx.device_claim(mirrored), rx.device_claim(mirrored)]
        RS.prepare(h, [[dict(kind=bl.SEND, pair=2 * c, slices=S["slp"] + 16 * c * nl, n=nl, flags=bl.UNTIL_BLOCKED)]
                       for c in range(conns)])
        RR.prepare(h, [[dict(kind=bl.RECV, pair=2 * c + 1, dst=S["dst"] + c * total, cap=total,
                             flags=bl.UNTIL_BLOCKED)] for c in range(conns)])
        st.synchronize()
        ev[0].record(st)
        RS.fire(60.0, stream=sp)
        ev[1].record(st)
        RR.fire(60.0, stream=sp)
        ev[2].record(st)
        rs, rr = RS.wait(), RR.wait()
        assert all(o[0]["ret"] == total for o in rs) and all(o[0]["ret"] == total for o in rr)
        for tx, rx in S["pairs"]:
            tx.device_release()
            rx.device_release()
        return ev[0].elapsed_time(ev[2]) * 1e-3

    out = {m: [] for m, _ in MODES}
    try:
        for rep in range(reps + 1):
            for mode, mirrored in MODES:
                t = step(mirrored)
                if rep:
                    out[mode].append(t)
    finally:
        _teardown(S)
    payload = conns * total
    return {m: {"conns": conns, "msg_bytes": msg, "step_ms": round(statistics.median(out[m]) * 1e3, 3),
                "GBps": round(payload / statistics.median(out[m]) / 1e9, 1),
                "steps_ms": [round(t * 1e3, 3) for t in out[m]]} for m, _ in MODES}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2000)
    ap.add_argument("--serve-rounds", type=int, default=300)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    import device_block_lib
    import device_lib
    import device_poll_lib
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    pkg = ge.load_package()
    pkg.init(0)
    torch.cuda.init()
    line = {"card": card(),
            "pingpong_1KiB": pingpong(pkg, device_lib, args.reps, args.rounds),
            "serve_64_conns": serve(pkg, device_poll_lib, args.reps, args.serve_rounds),
            "stream_256x4MiB_block": stream(pkg, device_block_lib, torch, args.reps)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
