"""Device ready sets against the b200_warp_poll scan (DESIGN.md §13 "Ready sets"): one JSON line.

  empty_take_ns / scan_ns   ns per empty b200_warp_ready_take and per b200_warp_poll scan of N idle claimed ends,
                            N = 32, 256, 1024, 4096 (one warp, alternating in one kernel, median of the rounds)
  serve                     round trips per second of one unmirrored server warp holding N = 64, 1024, 4096 claimed
                            ends, 64 of them with an active device client (256-byte echo), over the set and over the
                            scan, alternating on the same connections; medians of --rounds runs
The card's name and power limit are read in the same run.  Needs an H100 (sm_90a)."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--trips", type=int, default=200, help="round trips per active client per run")
    args = ap.parse_args()
    import __graft_entry__ as ge
    import device_ready_lib as drl
    pkg = ge.load_package()
    pkg.init(0)
    D = drl.load()
    assert D.dr_prepare() == 0
    L = pkg.lib()
    mem = drl.Pinned(L)
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 4096)
    nmax, active, msg = 4096, 64, 256
    conns = [pkg.connected_pair("rs-a%d" % i, "rs-b%d" % i) for i in range(nmax)]
    srv = [a.device_claim(mirrored=False) for a, b in conns]
    cli = [b.device_claim(mirrored=False) for a, b in conns[:active]]
    out = {"card": card()}
    # ---- empty take against a scan of n idle ends
    cost = {}
    for n in (32, 256, 1024, 4096):
        rs = pkg.ReadySet(n)
        for i in range(n):
            rs.add(conns[i][0], i)
        setp = mem.blob("set", [rs.device()])
        hp = mem.blob("h", srv[:n])
        scr, _ = mem.array("scr", np.uint32, n)
        # drain the initial entries and rearm them all (a consumer that served them)
        cons = drl.Consumer(pkg, rs, srv[:n], 64)
        r = cons.drain()
        assert r["status"] == 0 and r["takes"] == n, r
        cons.close()
        batches, per = 2 * args.rounds, max(4, 20000 // n)
        tp, t = mem.array("t", np.uint64, 2 * batches)
        assert D.dr_cost(setp, hp, n, scr, batches, per, tp) == 0, D.dr_error()
        cost[n] = dict(empty_take_ns=float(np.median(t[0::2][1:])), scan_ns=float(np.median(t[1::2][1:])))
        for i in range(n):
            conns[i][0].device_release()
            srv[i] = conns[i][0].device_claim(mirrored=False)
        rs.destroy()
    out["cost"] = cost
    # ---- one server warp, 64 active clients, N claimed ends: set against scan
    serve = {}
    for n in (64, 1024, 4096):
        rs = pkg.ReadySet(n)
        for i in range(n):
            rs.add(conns[i][0], i)
        cons = drl.Consumer(pkg, rs, srv[:n], 64)
        assert cons.drain()["status"] == 0
        cons.close()
        setp = mem.blob("set", [rs.device()])
        sp = mem.blob("srv", srv[:n])
        cp = mem.blob("cli", cli)
        sbuf, _ = mem.array("sbuf", np.uint8, n * msg)
        cbuf, _ = mem.array("cbuf", np.uint8, active * 2 * msg)
        rates = {"set": [], "scan": []}
        for r in range(args.rounds):
            for how in ("set", "scan"):
                state, _ = mem.array("state", np.uint32, 3 * n)
                op, o = mem.array("out", np.uint64, 2 * active + 5)
                s = drl.DrServe(setp if how == "set" else None, sp, cp, n, active, args.trips, msg, sbuf, cbuf, state,
                                op, 1 << 30)
                assert D.dr_serve_launch(C.byref(s)) == 0, D.dr_error()
                so = o[2 * active:]
                assert so[0] == 0 and so[1] == active * args.trips, (how, n, so)
                assert all(o[2 * i] == 0 and o[2 * i + 1] == args.trips for i in range(active))
                rates[how].append(active * args.trips / (so[4] * 1e-9))
        serve[n] = {how: dict(round_trips_per_s=statistics.median(v), min=min(v), max=max(v))
                    for how, v in rates.items()}
        for i in range(n):
            conns[i][0].device_release()
            srv[i] = conns[i][0].device_claim(mirrored=False)
        rs.destroy()
    out["serve"] = serve
    out["card_after"] = card()
    print(json.dumps(out))
    mem.free()


if __name__ == "__main__":
    main()
