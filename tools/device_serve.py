"""The poll loop of a BPEV server on the GPU (include/b200_device.cuh: b200_warp_poll / b200_warp_recv / b200_warp_send /
b200_warp_disconnect): what a readiness scan costs and what a polling server warp answers.  Prints one JSON line, with
the card's name and power limit read in the same run.

  poll     ns per b200_warp_poll scan of N idle claimed ends by one warp (median over batches of scans, %globaltimer in
           the kernel), N = 32 / 256 / 1024 / 4096
  echo     1 KiB round trips at 1 / 64 / 256 connections, one device client warp per connection
           (tests/native/device_poll.cu): against ONE polling server warp (poll -> Recv -> Send), and against one
           dedicated pong warp per connection; p50 / p99 round trip and round trips per second
  unary    bench.py's service unary p50 (1 KiB, 1 connection, host-driven through the resident service), run in the
           same session for scale

    python tools/device_serve.py [--rounds 300] [--no-bench]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def connections(pkg, n, cap, tag):
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", cap)
    return [pkg.connected_pair("%s-a%d" % (tag, i), "%s-b%d" % (tag, i)) for i in range(n)]


def drop(conns):
    for a, b in conns:
        for p in (a, b):
            p.disconnect()
            p.putback()


def poll_cost(pkg, R, sizes=(32, 256, 1024, 4096), batches=200, per=20):
    L, D = pkg.lib(), R.D
    conns = connections(pkg, max(sizes) // 2, 4096, "dsp")
    out = {}
    try:
        hp = R.handles("h", [h for a, b in conns for h in (a.device_claim(), b.device_claim())])
        hd = L.b200_mem_alloc_device(64 * max(sizes))
        assert L.b200_memcpy(hd, hp, 64 * max(sizes), 2, None) == 0 and L.b200_stream_sync(None) == 0
        ready = L.b200_mem_alloc_device(4 * max(sizes))
        tp, times = R.mem.array("t", np.uint64, batches)
        for where, h in (("handles_in_device_memory", hd), ("handles_in_pinned_memory", hp)):
            out[where] = {}
            for n in sizes:
                assert D.dp_poll_time(h, n, ready, batches, per, tp) == 0, D.dp_error().decode()
                t = float(np.median(times[batches // 10:]))  # (the first batches warm the caches)
                out[where]["n_%d" % n] = {"ns_per_scan": t, "ns_per_handle": t / n}
        L.b200_mem_free_device(ready)
        L.b200_mem_free_device(hd)
    finally:
        drop(conns)
    return out


def echo(pkg, R, n, mode, rounds, msg=1024):
    import device_poll_lib as dpl
    L, D = pkg.lib(), R.D
    conns = connections(pkg, n, 16384, "dse%d" % mode)
    bufs = []

    def dev(nbytes):
        p = L.b200_mem_alloc_device(nbytes)
        bufs.append(p)
        return p

    try:
        srv = R.handles("srv", [a.device_claim() for a, b in conns])
        cli = R.handles("cli", [b.device_claim() for a, b in conns])
        state = dev(12 * n)
        z = np.zeros(3 * n, np.uint32)
        assert L.b200_memcpy(state, z.ctypes.data, z.nbytes, 0, None) == 0 and L.b200_stream_sync(None) == 0
        tp, times = R.mem.array("times", np.uint64, n * rounds)
        op, out = R.mem.array("out", np.uint64, 4 * n + 4)
        out[:] = 0
        s = dpl.DpServe(srv=srv, cli=cli, n=n, rounds=rounds, msg=msg, mode=mode, sbuf=dev(n * msg),
                        cbuf=dev(2 * n * msg), state=state, times=tp, out=op, budget_ns=int(120e9), max_iters=1 << 40)
        t0 = time.perf_counter()
        assert D.dp_serve_launch(C.byref(s)) == 0, D.dp_error().decode()
        assert D.dp_wait() == 0, D.dp_error().decode()
        wall = time.perf_counter() - t0
        per = out[:4 * n].reshape(n, 4)
        ok = bool((per[:, 0] == 0).all() and (per[:, 1] == 0).all() and (per[:, 2] == rounds).all())
        r = np.sort(times.reshape(n, rounds)[:, rounds // 10:].reshape(-1)) / 1e3
        return {"ok": ok, "p50_us": float(r[len(r) // 2]), "p99_us": float(r[int(len(r) * 0.99)]),
                "round_trips_per_s": n * rounds / wall}
    finally:
        drop(conns)
        for p in bufs:
            L.b200_mem_free_device(p)


def bench_unary():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "3", "--warmup",
                          "3", "--no-e2e", "--no-endpoint", "--no-cpu-baseline"], capture_output=True, text=True)
    for line in reversed(out.stdout.strip().splitlines()):
        try:
            u = json.loads(line)["unary"]["b200"]["conns_1"]
            return {"p50_us": u["p50_us"], "p99_us": u["p99_us"]}
        except (ValueError, KeyError, TypeError):
            continue
    return {"error": (out.stdout + out.stderr)[-400:]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=300)
    ap.add_argument("--no-bench", action="store_true")
    args = ap.parse_args()
    import __graft_entry__ as ge
    import device_poll_lib as dpl
    pkg = ge.load_package()
    pkg.init(0)
    R = dpl.Runner(pkg)
    res = {"card": card(), "poll": poll_cost(pkg, R), "echo": {}}
    for n in (1, 64, 256):
        res["echo"]["conns_%d" % n] = {"polling_server_warp": echo(pkg, R, n, 0, args.rounds),
                                       "pong_warp_per_connection": echo(pkg, R, n, 1, args.rounds)}
    R.close()
    if not args.no_bench:
        res["bench_service_unary_1KiB_1conn"] = bench_unary()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
