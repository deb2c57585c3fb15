"""Prepared batches with B200_BATCH_CLUSTER(k): how fast few connections with large messages go when each op of the
batch runs on a thread-block cluster of k CTAs (k_cluster_send / k_cluster_recv) instead of one CTA (k_send / k_recv).

C connections (--conns, default 1 4 16 64) x one chttp2-shaped message of S bytes (default 32 MiB) each, through
64 MiB rings, in the reference format and with stamped frames.  A step is a prepared UNTIL_BLOCKED send batch, then a
prepared UNTIL_BLOCKED recv batch, over device memory.  k = 1, 2, 4, 8, 16 alternate in one process on the same
buffers; CUDA events around every launch; medians over --reps rounds after one warm-up round; every step's delivered
bytes are compared with the source.  Payload GB/s, and algorithmic HBM GB/s from frame_hbm_bytes (what the frames must
read and write, over the step's device time).  Prints one JSON line, with the card's name and power limit read in the
same run.

    python tools/batch_cluster_stream.py [--conns 1 4 16 64] [--msg-bytes 33554432] [--reps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KS = (1, 2, 4, 8, 16)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def placeable(pkg, k):
    """the library refuses a batch whose clusters of k CTAs this device cannot place"""
    b = pkg.lib().b200_batch_prepare_recv((pkg.RecvOp * 1)(), 0, pkg.cluster_flag(k))
    if b:
        pkg.lib().b200_batch_destroy(b)
    return bool(b)


def _row(ts, payload, hbm):
    snd, rcv = statistics.median(t[0] for t in ts), statistics.median(t[1] for t in ts)
    step = statistics.median(t[0] + t[1] for t in ts)
    return {"step_ms": round(step * 1e3, 3), "send_ms": round(snd * 1e3, 3), "recv_ms": round(rcv * 1e3, 3),
            "GBps": round(payload / step / 1e9, 2), "hbm_GBps": round(hbm / step / 1e9, 1),
            "steps_ms": [round((a + b) * 1e3, 3) for a, b in ts]}


def rate(pkg, torch, conns, msg, stamped, reps):
    pkg.config_set("GRPC_RDMA_RING_BUFFER_SIZE_KB", 65536)
    pkg.config_set("GRPC_RDMA_MAX_SGE", 30)
    pkg.config_set("B200_RING_STAMPED", int(stamped))
    lens = pkg.chttp2_slice_lens(msg)
    total = sum(lens)
    pairs = [pkg.connected_pair("bc%d%d-tx%d" % (conns, stamped, c), "bc%d%d-rx%d" % (conns, stamped, c))
             for c in range(conns)]
    pkg.config_set("B200_RING_STAMPED", 0)
    i = torch.arange(total, device="cuda", dtype=torch.int64)
    row = (((i * 2654435761) >> 11) & 255).to(torch.uint8)
    offs = (torch.arange(conns, device="cuda", dtype=torch.int64) * 131 & 255).to(torch.uint8)
    src = (row[None, :] + offs[:, None]).reshape(-1)
    dst = torch.zeros(conns * total, dtype=torch.uint8, device="cuda")
    del i, row, offs
    sls = []
    for c in range(conns):
        base, one = src.data_ptr() + c * total, []
        for n in lens:
            one.append((base, n))
            base += n
        sls.append(pkg.make_slices(one))
    batches = {}
    for k in [k for k in KS if placeable(pkg, k)]:
        fl = pkg.UNTIL_BLOCKED | pkg.cluster_flag(k)
        batches[k] = (pkg.Batch("send", [(pairs[c][0], sls[c], len(lens), 0) for c in range(conns)], fl),
                      pkg.Batch("recv", [(pairs[c][1], dst.data_ptr() + c * total, total) for c in range(conns)], fl))
    stream = torch.cuda.Stream()
    sp = stream.cuda_stream
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]

    def step(k):
        bs, br = batches[k]
        ev[0].record(stream)
        bs.launch(sp)
        ev[1].record(stream)
        br.launch(sp)
        ev[2].record(stream)
        stream.synchronize()
        assert bs.results(sp) == [total] * conns and br.results(sp) == [total] * conns, k
        assert torch.equal(src, dst), "k=%d: delivered bytes differ from what was sent" % k
        dst.zero_()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) * 1e-3, ev[1].elapsed_time(ev[2]) * 1e-3

    times = {k: [] for k in batches}
    for k in batches:  # warm-up
        step(k)
    for _ in range(reps):
        for k in batches:
            times[k].append(step(k))
    for bs, br in batches.values():
        bs.destroy()
        br.destroy()
    for tx, rx in pairs:
        for p in (tx, rx):
            p.disconnect()
            p.putback()
    del src, dst
    torch.cuda.empty_cache()
    tx_b, rx_b = pkg.frame_hbm_bytes(lens, stamped=stamped)
    payload, hbm = conns * total, conns * (tx_b + rx_b)
    return {"format": "stamped" if stamped else "reference", "conns": conns, "msg_bytes": total,
            "payload_bytes": payload, "hbm_bytes": hbm,
            "k": {str(k): _row(ts, payload, hbm) for k, ts in times.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--conns", type=int, nargs="+", default=[1, 4, 16, 64])
    ap.add_argument("--msg-bytes", type=int, default=32 << 20)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    pkg = ge.load_package()
    pkg.init(0)
    torch.cuda.init()
    line = {"card": card(), "ring_bytes": 64 << 20, "reps": args.reps,
            "rate": [rate(pkg, torch, c, args.msg_bytes, st, args.reps) for st in (False, True) for c in args.conns]}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
