"""Many server warps on one device ready set (DESIGN.md §13 "Many consumers"): one JSON line.

  one_consumer   the shared take (atomicCAS on head) against the one-consumer take it replaced (a plain store of
                 head, kept in tests/native/device_ready_shared.cu for this comparison only), alternating in one
                 process on the same connections:
                   empty_take_ns   ns per empty take of one warp on a set of N = 32, 256, 1024, 4096 idle members,
                                   the queue pointer loaded once (not the set's descriptor on every call)
                   serve           round trips/s of one unmirrored server warp holding N = 64, 1024, 4096 claimed
                                   ends, 64 of them with an active device client (256-byte echo; the workload of
                                   tools/device_ready_serve.py)
  scaling        4096 claimed unmirrored server ends, 256 active device clients, 256-byte echo, W = 1 .. 32 server
                 warps, each taking up to --take-max keys:
                   shared    W warps on one set of 4096 members (each fences before its rearm: the holder rule)
                   sharded   W sets of 4096 / W members, one warp each: the split a server could build before
                 balanced: client j talks to end 16 j, so every shard has clients; skewed: client j talks to end j,
                 so the clients sit on the ends 0 .. 255 (one shard for W <= 16, two for W = 32).  Round trips/s
                 and lost CASes per take (a counter in the driver).
Every figure is the median of --rounds runs, with the minimum and maximum.  The card's name and power limit are read
in the same run.  Needs an H100 (sm_90a)."""
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


def stats(v):
    return dict(median=statistics.median(v), min=min(v), max=max(v))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--ab-trips", type=int, default=200, help="round trips per client, one-consumer comparison")
    ap.add_argument("--trips", type=int, default=100, help="round trips per client, scaling")
    ap.add_argument("--take-max", type=int, default=8, help="keys per take, scaling")
    ap.add_argument("--warps", default="1,2,4,8,16,32")
    args = ap.parse_args()
    import __graft_entry__ as ge
    import device_ready_lib as drl
    import device_ready_shared_lib as dsl
    pkg = ge.load_package()
    pkg.init(0)
    D = dsl.load()
    assert D.ds_prepare() == 0, D.ds_error()
    assert drl.load().dr_prepare() == 0
    L = pkg.lib()
    mem, dev = drl.Pinned(L), dsl.Device(pkg)
    pkg.config_set("B200_RING_BUFFER_SIZE_BYTES", 4096)
    nmax, msg = 4096, 256
    conns = [pkg.connected_pair("rss-a%d" % i, "rss-b%d" % i) for i in range(nmax)]
    srv = [a.device_claim(mirrored=False) for a, b in conns]
    cli = [b.device_claim(mirrored=False) for a, b in conns]
    out = {"card": card()}

    def make_sets(nsets, n):
        """nsets sets over server ends 0 .. n-1 (member i in set i // (n / nsets), key i), initial entries drained"""
        per = n // nsets
        sets = []
        for s in range(nsets):
            rs = pkg.ReadySet(per)
            for i in range(s * per, (s + 1) * per):
                rs.add(conns[i][0], i)
            cons = drl.Consumer(pkg, rs, srv[:n], 64)
            r = cons.drain()
            assert r["status"] == 0 and r["takes"] == per, r
            cons.close()
            sets.append(rs)
        return sets

    def drop_sets(sets, n):
        for i in range(n):
            conns[i][0].device_release()
            srv[i] = conns[i][0].device_claim(mirrored=False)
        for rs in sets:
            rs.destroy()

    def serve(sets, n, clients, servers, trips, take_max, flags):
        a = len(clients)
        op, o = mem.array("out", np.uint64, 2 * a + 8 * servers)
        s = dsl.DsServe(mem.blob("sets", [rs.device() for rs in sets]), mem.blob("srv", srv[:n]),
                        mem.blob("cli", [cli[j] for j in clients]), n, a, trips, msg, servers, len(sets), take_max,
                        flags, dev.array("sbuf", np.uint8, n * msg), dev.array("cbuf", np.uint8, a * 2 * msg),
                        dev.array("state", np.uint32, 2 * n), dev.array("keys", np.uint32, servers * take_max),
                        dev.array("done", np.uint64, 1), op, 1 << 30)
        rc = D.ds_serve_launch(C.byref(s))
        assert rc == 0, (rc, D.ds_error())
        assert all(o[2 * i] == 0 and o[2 * i + 1] == trips for i in range(a)), "a client failed"
        rows, span = dsl.serve_totals(o, a, servers)
        assert (rows[:, 0] == 0).all() and int(rows[:, 1].sum()) == a * trips and int(rows[:, 5].sum()) == 0, rows
        return a * trips / (span * 1e-9), int(rows[:, 4].sum()) / max(1, int(rows[:, 3].sum()))

    # ---- one consumer: empty take, shared against baseline
    cost = {}
    for n in (32, 256, 1024, 4096):
        sets = make_sets(1, n)
        scr = dev.array("scr", np.uint32, n)
        batches, per = 2 * args.rounds + 1, max(4, 20000 // n)
        tp, t = mem.array("t", np.uint64, 2 * batches)
        assert D.ds_cost(mem.blob("set", [sets[0].device()]), n, scr, batches, per, tp) == 0, D.ds_error()
        cost[n] = dict(shared=stats([float(x) for x in t[0::2][1:]]), baseline=stats([float(x) for x in t[1::2][1:]]))
        drop_sets(sets, n)
    # ---- one consumer: one server warp, 64 active clients on ends 0 .. 63
    ab = {}
    for n in (64, 1024, 4096):
        sets = make_sets(1, n)
        rates = {"shared": [], "baseline": []}
        for r in range(args.rounds):
            for how in ("shared", "baseline"):
                rate, _ = serve(sets, n, list(range(64)), 1, args.ab_trips, n, dsl.BASELINE if how == "baseline" else 0)
                rates[how].append(rate)
        ab[n] = {how: stats(v) for how, v in rates.items()}
        drop_sets(sets, n)
    out["one_consumer"] = {"empty_take_ns": cost, "serve_round_trips_per_s": ab}
    print("one consumer: %s" % json.dumps(out["one_consumer"]), file=sys.stderr, flush=True)
    # ---- scaling: 4096 ends, 256 clients
    loads = {"balanced": [16 * j for j in range(256)], "skewed": list(range(256))}
    scaling = {}
    for w in [int(x) for x in args.warps.split(",")]:
        row = {}
        for layout in ("shared", "sharded"):
            sets = make_sets(1 if layout == "shared" else w, nmax)
            flags = dsl.FENCE if layout == "shared" and w > 1 else 0
            got = {ld: ([], []) for ld in loads}
            for r in range(args.rounds):
                for ld, clients in loads.items():
                    rate, retries = serve(sets, nmax, clients, w, args.trips, args.take_max, flags)
                    got[ld][0].append(rate)
                    got[ld][1].append(retries)
            for ld, (rates, retries) in got.items():
                row["%s_%s" % (layout, ld)] = dict(round_trips_per_s=stats(rates),
                                                   lost_cas_per_take=statistics.median(retries))
            drop_sets(sets, nmax)
        scaling[w] = row
        print("scaling W=%d: %s" % (w, json.dumps(row)), file=sys.stderr, flush=True)
    out["scaling"] = scaling
    out["card_after"] = card()
    print(json.dumps(out))
    mem.free()
    dev.free()


if __name__ == "__main__":
    main()
