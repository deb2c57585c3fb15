"""Device-initiated Send / Recv (include/b200_device.cuh): what one warp per end moves, and how long a round trip
takes when the GPU drives the pair.  Prints one JSON line, with the card's name and power limit read in the same run.

  rate        C connections x M chttp2-shaped messages of S bytes (default 256 x 4 MiB, 16 MiB rings), one sender warp
              and one receiver warp per connection in one kernel (tests/native/device_api.cu), alternating with
              k_send + k_recv (prepared B200_BATCH_UNTIL_BLOCKED batches) on the same buffers in the same process
  pingpong    1 KiB round trips, p50 / p99 over --rounds: two device warps on one loopback connection (the time is
              %globaltimer in the ping warp); a device warp against a host-driven peer under the service, the host
              side being b200_pair_recv / b200_pair_send called from Python through ctypes

    python tools/device_stream.py [--conns 256] [--msg-bytes 4194304] [--msgs 2] [--reps 3] [--rounds 2000]
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


def rate(pkg, dl, conns, msg, msgs, reps):
    L = pkg.lib()
    pkg.config_set("GRPC_RDMA_RING_BUFFER_SIZE_KB", 16384)
    lens = pkg.chttp2_slice_lens(msg)
    total = sum(lens)
    pairs = [pkg.connected_pair("ds-tx%d" % c, "ds-rx%d" % c) for c in range(conns)]
    src = L.b200_mem_alloc_device(conns * total)
    dst = L.b200_mem_alloc_device(conns * total)
    slp = L.b200_mem_alloc_host(16 * len(lens) * conns)
    arr = (pkg.Slice * (len(lens) * conns)).from_address(slp)
    sl = []
    for c in range(conns):
        off, one = 0, []
        for k, n in enumerate(lens):
            arr[c * len(lens) + k].ptr, arr[c * len(lens) + k].len = src + c * total + off, n
            one.append((src + c * total + off, n))
            off += n
        sl.append(pkg.make_slices(one))
    bs = pkg.Batch("send", [(pairs[c][0], sl[c], len(lens), 0) for c in range(conns)], pkg.UNTIL_BLOCKED)
    br = pkg.Batch("recv", [(pairs[c][1], dst + c * total, total) for c in range(conns)], pkg.UNTIL_BLOCKED)
    R = dl.Runner(pkg)

    def cta_step():
        t0 = time.perf_counter()
        for _ in range(msgs):
            bs.launch()
            br.launch()
            assert br.results() == [total] * conns and bs.results() == [total] * conns
        return time.perf_counter() - t0

    def warp_step():
        handles = []
        for tx, rx in pairs:
            handles += [tx.device_claim(), rx.device_claim()]
        lists = []
        for c in range(conns):
            lists.append([dict(kind=dl.STREAM_SEND, pair=2 * c, slices=slp + 16 * c * len(lens), n=len(lens))] * msgs)
            lists.append([dict(kind=dl.STREAM_RECV, pair=2 * c + 1, dst=dst + c * total, n=total)] * msgs)
        t0 = time.perf_counter()
        res = R.run(handles, lists, budget_s=300.0)
        dt = time.perf_counter() - t0
        assert all(o["status"] == dl.OK and o["ret"] == total for lst in res for o in lst)
        for tx, rx in pairs:
            tx.device_release()
            rx.device_release()
        return dt

    cta_step()
    warp_step()  # warm-up
    t_cta, t_warp = [], []
    for _ in range(reps):
        t_cta.append(cta_step())
        t_warp.append(warp_step())
    bytes_moved = conns * total * msgs
    bs.destroy()
    br.destroy()
    for tx, rx in pairs:
        tx.disconnect(); rx.disconnect(); tx.putback(); rx.putback()
    for p in (src, dst):
        L.b200_mem_free_device(p)
    L.b200_mem_free_host(slp)
    return {"conns": conns, "msg_bytes": msg, "msgs_per_conn": msgs, "payload_bytes": bytes_moved,
            "device_warps_GBps": round(bytes_moved / min(t_warp) / 1e9, 2),
            "k_send_k_recv_GBps": round(bytes_moved / min(t_cta) / 1e9, 2),
            "device_warps_s": [round(t, 5) for t in t_warp], "k_send_k_recv_s": [round(t, 5) for t in t_cta]}


def _pct(ns):
    a = np.sort(np.asarray(ns, dtype=np.float64)) / 1e3
    return {"p50_us": round(float(np.percentile(a, 50)), 2), "p99_us": round(float(np.percentile(a, 99)), 2),
            "n": int(a.size)}


def pingpong(pkg, dl, rounds, size=1024):
    L = pkg.lib()
    pkg.config_set("GRPC_RDMA_RING_BUFFER_SIZE_KB", 4096)
    R = dl.Runner(pkg)
    msg = L.b200_mem_alloc_device(size)
    back = L.b200_mem_alloc_device(size)
    got = L.b200_mem_alloc_device(size)
    times = L.b200_mem_alloc_host(8 * rounds)
    slp = L.b200_mem_alloc_host(16)
    s = (pkg.Slice * 1).from_address(slp)
    s[0].ptr, s[0].len = msg, size
    t = np.ctypeslib.as_array((C.c_uint64 * rounds).from_address(times))
    out = {}
    # two device warps
    a, b = pkg.connected_pair("pp-a", "pp-b")
    ha, hb = a.device_claim(), b.device_claim()
    res = R.run([ha, hb], [[dict(kind=dl.PING, pair=0, slices=slp, n=rounds, byte_idx=1, dst=got, times=times)],
                           [dict(kind=dl.PONG, pair=1, dst=back, cap=size, n=rounds)]], budget_s=60.0)
    assert all(o[0]["status"] == dl.OK for o in res), res
    out["device_device"] = _pct(t[rounds // 10:])
    a.disconnect(); b.disconnect(); a.putback(); b.putback()
    # a device warp against a host-driven peer under the service
    a, b = pkg.connected_pair("pq-a", "pq-b")
    hbuf = L.b200_mem_alloc_host(size)
    assert L.b200_service_start(16) == 0, pkg.last_error()
    try:
        ha = a.device_claim()
        R.launch([ha], [[dict(kind=dl.PING, pair=0, slices=slp, n=rounds, byte_idx=1, dst=got, times=times)]],
                 budget_s=60.0)
        deadline = time.time() + 60
        for _ in range(rounds):
            n = 0
            while n < size and time.time() < deadline:
                n += b.recv_into(hbuf + n, size - n)
            sent = 0
            while sent < size and time.time() < deadline:
                sent += b.send_raw([(hbuf + sent, size - sent)])
        res = R.wait()
        assert res[0][0]["status"] == dl.OK, res
        out["device_host_service"] = _pct(t[rounds // 10:])
        a.device_release()
    finally:
        L.b200_service_stop()
    a.disconnect(); b.disconnect(); a.putback(); b.putback()
    for p in (msg, back, got):
        L.b200_mem_free_device(p)
    for p in (times, slp, hbuf):
        L.b200_mem_free_host(p)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--conns", type=int, default=256)
    ap.add_argument("--msg-bytes", type=int, default=4 << 20)
    ap.add_argument("--msgs", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2000)
    args = ap.parse_args()
    import __graft_entry__ as ge
    import device_lib
    pkg = ge.load_package()
    pkg.init(0)
    line = {"card": card(), "rate": rate(pkg, device_lib, args.conns, args.msg_bytes, args.msgs, args.reps),
            "pingpong_1k": pingpong(pkg, device_lib, args.rounds)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
