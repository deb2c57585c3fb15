"""A device server that parks its ready set when idle (DESIGN.md §13 "Parking"): one JSON line.

  wake       256-byte requests from a host client to a parked set, one at a time with a pause between them:
             push -> fd readable   host clock from just before the Send call to the fd polling readable
             fd -> launch          from there to the return of the server's launch call (after consuming the fd)
             launch -> answer      from there to the whole reply read back on the host
             total                 push to answer
             resident              the same request's round trip with a server kept resident (never parking)
             p50 / p99 in µs over --wakes requests
  occupancy  host requests at R per second (default 100 and 1000) for --seconds, answered by servers launched on
             demand: the sum of the servers' kernel times (CUDA events around each launch) over wall time; a resident
             server occupies its SMs 100 % of the time
The server is tests/native/device_ready_park.cu's echo server (1 warp, parking after 64 empty takes in a row).  The
card's name and power limit are read in the same run.  Needs an H100 (sm_90a)."""
import argparse
import json
import os
import select
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

MSG = 256


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def pct(xs, p):
    return round(float(np.percentile(np.array(xs) * 1e6, p)), 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--wakes", type=int, default=300)
    ap.add_argument("--rates", default="100,1000")
    ap.add_argument("--seconds", type=float, default=3.0)
    args = ap.parse_args()
    import __graft_entry__ as ge
    import device_ready_park_lib as dpl
    import test_device_ready_park_gpu as T
    pkg = ge.load_package()
    pkg.init(0)
    out = {"card": card()}
    R = T._Rig(pkg, 1, 0, {}, "tool-park", mirrored=False)
    fd = R.rs.wakeup_fd()
    p = select.poll()
    p.register(fd, select.POLLIN)
    cli = R.conns[0][1]
    _, src = R.mem.array("src", np.uint8, MSG)
    if R.rs.park() == 1:
        R.serve(1)
    rep = np.zeros(MSG, np.uint8)

    def reply():
        got = 0
        while got < MSG:
            got += cli.recv_into(rep.ctypes.data + got, MSG - got)

    # wake latency
    stages = {"push_to_fd": [], "fd_to_launch": [], "launch_to_answer": [], "total": []}
    for k in range(args.wakes + 10):
        src[:] = dpl.pattern(0, k, MSG)
        t0 = time.perf_counter()
        assert cli.send_raw([(src.ctypes.data, MSG)]) == MSG
        if not p.poll(10000):
            raise RuntimeError("no wakeup within 10 s of a request to the parked set")
        t1 = time.perf_counter()
        R.rs.consume_wakeup()
        R.server.launch(1)
        t2 = time.perf_counter()
        reply()
        t3 = time.perf_counter()
        r = R.server.wait()
        assert r["status"] == 0 and np.array_equal(rep, src), r
        if k >= 10:
            for key, v in (("push_to_fd", t1 - t0), ("fd_to_launch", t2 - t1), ("launch_to_answer", t3 - t2),
                           ("total", t3 - t0)):
                stages[key].append(v)
        time.sleep(0.002)
    # resident round trip: a server that does not park, busy-polling until 2^20 takes in a row find nothing
    R.server.launch(1, idle_takes=1 << 20, no_park=True, max_iters=1 << 40)
    rt = []
    for k in range(args.wakes + 10):
        src[:] = dpl.pattern(0, 100000 + k, MSG)
        t0 = time.perf_counter()
        assert cli.send_raw([(src.ctypes.data, MSG)]) == MSG
        reply()
        if k >= 10:
            rt.append(time.perf_counter() - t0)
    out["wake_us"] = {k: {"p50": pct(v, 50), "p99": pct(v, 99)} for k, v in stages.items()}
    out["wake_us"]["resident"] = {"p50": pct(rt, 50), "p99": pct(rt, 99)}
    assert R.server.wait()["status"] == 0
    R.close()
    occ = {}
    for rate in [int(x) for x in args.rates.split(",")]:
        Q = T._Rig(pkg, 1, 0, {}, "tool-occ%d" % rate, mirrored=False)
        try:
            fd = Q.rs.wakeup_fd()
            if Q.rs.park() == 1:
                Q.serve(1)
            Q.server.kernel_ms = 0.0
            cli = Q.conns[0][1]
            _, src = Q.mem.array("src", np.uint8, MSG)
            state = {"done": False, "sent": 0}

            def load():
                try:
                    t_next = time.perf_counter()
                    t_end = t_next + args.seconds
                    while t_next < t_end:
                        while time.perf_counter() < t_next:
                            pass
                        src[:] = dpl.pattern(0, state["sent"], MSG)
                        assert cli.send_raw([(src.ctypes.data, MSG)]) == MSG
                        assert np.array_equal(T.recv_all(cli), src)
                        state["sent"] += 1
                        t_next += 1.0 / rate
                finally:
                    state["done"] = True

            th = threading.Thread(target=load)
            w0 = time.perf_counter()
            th.start()
            launches = 0
            while not state["done"]:
                if T.readable(fd, 5):
                    Q.rs.consume_wakeup()
                    Q.serve(1)
                    launches += 1
            th.join()
            wall = time.perf_counter() - w0
            occ[str(rate)] = {"requests": state["sent"], "launches": launches, "wall_s": round(wall, 3),
                              "kernel_ms": round(Q.server.kernel_ms, 2),
                              "gpu_time_share_pct": round(100.0 * Q.server.kernel_ms / 1e3 / wall, 3)}
        finally:
            Q.close()
    out["occupancy"] = occ
    print(json.dumps(out))


if __name__ == "__main__":
    main()
