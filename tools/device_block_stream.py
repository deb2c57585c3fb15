"""Block-level device Send / Recv (include/b200_device_block.cuh) against the library's k_send + k_recv and against the
warp calls.  All modes alternate in one process on the same buffers; CUDA events around every launch; medians over
--reps rounds.  Prints one JSON line, with the card's name and power limit read in the same run.

  rate     C connections (default 256) x one chttp2-shaped message of S bytes (default 4 MiB), 16 MiB rings: one
           kernel of block sends (B200_BATCH_UNTIL_BLOCKED, one CTA per connection, tests/native/device_block.cu),
           then one kernel of block receives; against k_send then k_recv as prepared UNTIL_BLOCKED batches.  Device
           time per step and per kernel, GB/s of payload.
  duplex   D connections (default 128: 256 CTAs, co-resident at two per SM), a sender and a receiver of each
           connection in ONE kernel, messages of M bytes (default 4 MiB) through 1 MiB rings (each message laps its
           ring four times): block calls (a CTA per end; CUDA events) and warp calls (a warp per end,
           tests/native/device_api.cu, which launches on a stream of its own: host clock around launch + synchronise).

    python tools/device_block_stream.py [--conns 256] [--msg-bytes 4194304] [--duplex-conns 128] [--reps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def _setup(pkg, conns, ring_kb, msg, name):
    L = pkg.lib()
    pkg.config_set("GRPC_RDMA_RING_BUFFER_SIZE_KB", ring_kb)
    pkg.config_set("GRPC_RDMA_MAX_SGE", 30)
    lens = pkg.chttp2_slice_lens(msg)
    total = sum(lens)
    pairs = [pkg.connected_pair("%s-tx%d" % (name, c), "%s-rx%d" % (name, c)) for c in range(conns)]
    src = L.b200_mem_alloc_device(conns * total)
    dst = L.b200_mem_alloc_device(conns * total)
    slp = L.b200_mem_alloc_host(16 * len(lens) * conns)
    assert src and dst and slp
    arr = (pkg.Slice * (len(lens) * conns)).from_address(slp)
    sl = []
    for c in range(conns):
        off, one = 0, []
        for k, n in enumerate(lens):
            arr[c * len(lens) + k].ptr, arr[c * len(lens) + k].len = src + c * total + off, n
            one.append((src + c * total + off, n))
            off += n
        sl.append(pkg.make_slices(one))
    # the device calls read the slice descriptors from device memory, as a prepared batch's kernels do
    sld = L.b200_mem_alloc_device(16 * len(lens) * conns)
    assert sld and L.b200_memcpy(sld, slp, 16 * len(lens) * conns, 0, None) == 0 and L.b200_stream_sync(None) == 0
    return dict(L=L, lens=lens, total=total, pairs=pairs, src=src, dst=dst, slp=sld, slp_host=slp, sl=sl)


def _teardown(S):
    L = S["L"]
    for tx, rx in S["pairs"]:
        for p in (tx, rx):
            if p.device_owned():
                p.device_release()
            p.disconnect()
            p.putback()
    L.b200_mem_free_device(S["src"])
    L.b200_mem_free_device(S["dst"])
    L.b200_mem_free_device(S["slp"])
    L.b200_mem_free_host(S["slp_host"])


def _claim(S):
    h = []
    for tx, rx in S["pairs"]:
        h += [tx.device_claim(), rx.device_claim()]
    return h


def _release(S):
    for tx, rx in S["pairs"]:
        tx.device_release()
        rx.device_release()


def rate(pkg, bl, torch, conns, msg, reps):
    S = _setup(pkg, conns, 16384, msg, "bsr")
    total, nl = S["total"], len(S["lens"])
    stream = torch.cuda.Stream()
    sp = stream.cuda_stream
    bs = pkg.Batch("send", [(S["pairs"][c][0], S["sl"][c], nl, 0) for c in range(conns)], pkg.UNTIL_BLOCKED)
    br = pkg.Batch("recv", [(S["pairs"][c][1], S["dst"] + c * total, total) for c in range(conns)], pkg.UNTIL_BLOCKED)
    RS, RR = bl.Runner(pkg), bl.Runner(pkg)  # (each keeps its own op buffers: both kernels are queued at once)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]

    def cta_step():
        ev[0].record(stream)
        bs.launch(sp)
        ev[1].record(stream)
        br.launch(sp)
        ev[2].record(stream)
        stream.synchronize()
        assert bs.results(sp) == [total] * conns and br.results(sp) == [total] * conns
        return ev[0].elapsed_time(ev[1]) * 1e-3, ev[1].elapsed_time(ev[2]) * 1e-3

    def block_step():
        h = _claim(S)
        sends = [[dict(kind=bl.SEND, pair=2 * c, slices=S["slp"] + 16 * c * nl, n=nl, flags=bl.UNTIL_BLOCKED)]
                 for c in range(conns)]
        recvs = [[dict(kind=bl.RECV, pair=2 * c + 1, dst=S["dst"] + c * total, cap=total, flags=bl.UNTIL_BLOCKED)]
                 for c in range(conns)]
        RS.prepare(h, sends)
        RR.prepare(h, recvs)
        stream.synchronize()
        ev[0].record(stream)
        RS.fire(60.0, stream=sp)
        ev[1].record(stream)
        RR.fire(60.0, stream=sp)
        ev[2].record(stream)
        rs, rr = RS.wait(), RR.wait()
        assert all(o[0]["ret"] == total for o in rs) and all(o[0]["ret"] == total for o in rr)
        _release(S)
        return ev[0].elapsed_time(ev[1]) * 1e-3, ev[1].elapsed_time(ev[2]) * 1e-3

    cta_step()
    block_step()  # warm-up
    t_cta, t_blk = [], []
    for _ in range(reps):
        t_cta.append(cta_step())
        t_blk.append(block_step())
    bs.destroy()
    br.destroy()
    _teardown(S)
    payload = conns * total

    def row(ts):
        snd, rcv = statistics.median(t[0] for t in ts), statistics.median(t[1] for t in ts)
        step = statistics.median(t[0] + t[1] for t in ts)
        return {"step_ms": round(step * 1e3, 3), "send_ms": round(snd * 1e3, 3), "recv_ms": round(rcv * 1e3, 3),
                "GBps": round(payload / step / 1e9, 1), "steps_ms": [round((a + b) * 1e3, 3) for a, b in ts]}

    return {"conns": conns, "msg_bytes": msg, "payload_bytes": payload, "block": row(t_blk),
            "k_send_k_recv": row(t_cta)}


def duplex(pkg, bl, dl, torch, conns, msg, reps):
    S = _setup(pkg, conns, 1024, msg, "bsd")
    total, nl = S["total"], len(S["lens"])
    stream = torch.cuda.Stream()
    sp = stream.cuda_stream
    RB, RW = bl.Runner(pkg), dl.Runner(pkg)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def lists(mod):
        out = []
        for c in range(conns):
            out.append([dict(kind=mod.STREAM_SEND, pair=2 * c, slices=S["slp"] + 16 * c * nl, n=nl)])
            out.append([dict(kind=mod.STREAM_RECV, pair=2 * c + 1, dst=S["dst"] + c * total, n=total)])
        return out

    def block_step():
        h = _claim(S)
        RB.prepare(h, lists(bl))
        stream.synchronize()
        ev[0].record(stream)
        RB.fire(120.0, stream=sp)
        ev[1].record(stream)
        res = RB.wait()
        assert all(o[0]["status"] == bl.OK and o[0]["ret"] == total for o in res)
        _release(S)
        return ev[0].elapsed_time(ev[1]) * 1e-3

    def warp_step():  # (the warp driver launches on a stream of its own: a host clock around launch + synchronise)
        h = _claim(S)
        t0 = time.perf_counter()
        res = RW.run(h, lists(dl), budget_s=300.0)  # (the op fill in Python is inside this window: ~1 ms)
        dt = time.perf_counter() - t0
        assert all(o[0]["status"] == dl.OK and o[0]["ret"] == total for o in res)
        _release(S)
        return dt

    block_step()
    warp_step()
    t_b, t_w = [], []
    for _ in range(reps):
        t_b.append(block_step())
        t_w.append(warp_step())
    _teardown(S)
    payload = conns * total
    mb, mw = statistics.median(t_b), statistics.median(t_w)
    return {"conns": conns, "msg_bytes": msg, "ring_bytes": 1 << 20, "payload_bytes": payload,
            "block": {"ms": round(mb * 1e3, 3), "GBps": round(payload / mb / 1e9, 1),
                      "runs_ms": [round(t * 1e3, 3) for t in t_b]},
            "warp": {"ms": round(mw * 1e3, 3), "GBps": round(payload / mw / 1e9, 1),
                     "runs_ms": [round(t * 1e3, 3) for t in t_w]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--conns", type=int, default=256)
    ap.add_argument("--msg-bytes", type=int, default=4 << 20)
    ap.add_argument("--duplex-conns", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    import device_block_lib
    import device_lib
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    pkg = ge.load_package()
    pkg.init(0)
    torch.cuda.init()
    line = {"card": card(),
            "rate": rate(pkg, device_block_lib, torch, args.conns, args.msg_bytes, args.reps),
            "duplex": duplex(pkg, device_block_lib, device_lib, torch, args.duplex_conns, args.msg_bytes, args.reps)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
