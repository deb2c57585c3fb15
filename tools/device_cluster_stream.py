"""Cluster calls (b200_cluster_send / b200_cluster_recv, include/b200_device_block.cuh) with few connections: how fast
one connection goes with a cluster of K CTAs on it, against the block call (K = 1) and the library's k_send + k_recv.
All variants of a configuration alternate in one process on the same buffers; CUDA events around every kernel;
medians over --reps rounds; every step's delivered bytes are compared with the source.  Prints one JSON line, with the
card's name and power limit read in the same run.

  rate     C connections (--conns, default 1 4 16 64) x one chttp2-shaped message of S bytes (default 32 MiB) each,
           through 64 MiB rings: a kernel of sends (B200_BATCH_UNTIL_BLOCKED), then a kernel of receives, with
             block       the block calls, one CTA per connection (tests/native/device_block.cu)
             cluster_K   the cluster calls, a cluster of K = 2, 4, 8, 16 CTAs per connection (device_cluster.cu)
             k_send_k_recv  the library's kernels as prepared UNTIL_BLOCKED batches
           in the reference format and with stamped frames.  Payload GB/s, and algorithmic HBM GB/s from
           frame_hbm_bytes (what the frames must read and write, over the step's device time).
  duplex   D connections (--duplex-conns, default 1 4), a sender and a receiver of each connection in ONE kernel, the
           same messages through 4 MiB rings (each message laps its ring eight times): block calls and clusters of K.

    python tools/device_cluster_stream.py [--conns 1 4 16 64] [--msg-bytes 33554432] [--reps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

KS = (2, 4, 8, 16)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


class Setup:
    """conns connected pairs with rings of ring_kb, a chttp2-shaped message of msg bytes per connection in `src`,
    `dst` of the same size; slice lists for the batches (host) and for the device calls (device memory)"""

    def __init__(self, pkg, torch, conns, ring_kb, msg, stamped, name):
        self.pkg, self.L, self.conns = pkg, pkg.lib(), conns
        pkg.config_set("GRPC_RDMA_RING_BUFFER_SIZE_KB", ring_kb)
        pkg.config_set("GRPC_RDMA_MAX_SGE", 30)
        pkg.config_set("B200_RING_STAMPED", int(stamped))
        self.lens = pkg.chttp2_slice_lens(msg)
        self.total = total = sum(self.lens)
        self.pairs = [pkg.connected_pair("%s-tx%d" % (name, c), "%s-rx%d" % (name, c)) for c in range(conns)]
        pkg.config_set("B200_RING_STAMPED", 0)
        i = torch.arange(total, device="cuda", dtype=torch.int64)
        row = (((i * 2654435761) >> 11) & 255).to(torch.uint8)
        offs = (torch.arange(conns, device="cuda", dtype=torch.int64) * 131 & 255).to(torch.uint8)
        self.src = (row[None, :] + offs[:, None]).reshape(-1)
        self.dst = torch.zeros(conns * total, dtype=torch.uint8, device="cuda")
        del i, row, offs
        nl = len(self.lens)
        slp = self.L.b200_mem_alloc_host(16 * nl * conns)
        arr = (pkg.Slice * (nl * conns)).from_address(slp)
        self.sl = []
        base = self.src.data_ptr()
        for c in range(conns):
            off, one = 0, []
            for k, n in enumerate(self.lens):
                arr[c * nl + k].ptr, arr[c * nl + k].len = base + c * total + off, n
                one.append((base + c * total + off, n))
                off += n
            self.sl.append(pkg.make_slices(one))
        self.sld = self.L.b200_mem_alloc_device(16 * nl * conns)  # the device calls read descriptors from HBM
        assert self.sld and self.L.b200_memcpy(self.sld, slp, 16 * nl * conns, 0, None) == 0
        assert self.L.b200_stream_sync(None) == 0
        self.L.b200_mem_free_host(slp)

    def claim(self):
        h = []
        for tx, rx in self.pairs:
            h += [tx.device_claim(), rx.device_claim()]
        return h

    def release(self):
        for tx, rx in self.pairs:
            tx.device_release()
            rx.device_release()

    def sends(self, mod, stream=False):
        nl = len(self.lens)
        if stream:
            return [[dict(kind=mod.STREAM_SEND, pair=2 * c, slices=self.sld + 16 * c * nl, n=nl)]
                    for c in range(self.conns)]
        return [[dict(kind=mod.SEND, pair=2 * c, slices=self.sld + 16 * c * nl, n=nl, flags=mod.UNTIL_BLOCKED)]
                for c in range(self.conns)]

    def recvs(self, mod, stream=False):
        t, d = self.total, self.dst.data_ptr()
        if stream:
            return [[dict(kind=mod.STREAM_RECV, pair=2 * c + 1, dst=d + c * t, n=t)] for c in range(self.conns)]
        return [[dict(kind=mod.RECV, pair=2 * c + 1, dst=d + c * t, cap=t, flags=mod.UNTIL_BLOCKED)]
                for c in range(self.conns)]

    def teardown(self):
        for tx, rx in self.pairs:
            for p in (tx, rx):
                if p.device_owned():
                    p.device_release()
                p.disconnect()
                p.putback()
        self.L.b200_mem_free_device(self.sld)


def _row(ts, payload, hbm):
    snd, rcv = statistics.median(t[0] for t in ts), statistics.median(t[1] for t in ts)
    step = statistics.median(t[0] + t[1] for t in ts)
    return {"step_ms": round(step * 1e3, 3), "send_ms": round(snd * 1e3, 3), "recv_ms": round(rcv * 1e3, 3),
            "GBps": round(payload / step / 1e9, 2), "hbm_GBps": round(hbm / step / 1e9, 1),
            "steps_ms": [round((a + b) * 1e3, 3) for a, b in ts]}


def rate(pkg, torch, bl, cl, conns, msg, stamped, reps):
    S = Setup(pkg, torch, conns, 65536, msg, stamped, "cr%d%d" % (conns, stamped))
    total, nl = S.total, len(S.lens)
    stream = torch.cuda.Stream()
    sp = stream.cuda_stream
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    bs = pkg.Batch("send", [(S.pairs[c][0], S.sl[c], nl, 0) for c in range(conns)], pkg.UNTIL_BLOCKED)
    br = pkg.Batch("recv", [(S.pairs[c][1], S.dst.data_ptr() + c * total, total) for c in range(conns)],
                   pkg.UNTIL_BLOCKED)

    def check():
        assert torch.equal(S.src, S.dst), "delivered bytes differ from what was sent"
        S.dst.zero_()
        torch.cuda.synchronize()

    def cta_step():
        ev[0].record(stream)
        bs.launch(sp)
        ev[1].record(stream)
        br.launch(sp)
        ev[2].record(stream)
        stream.synchronize()
        assert bs.results(sp) == [total] * conns and br.results(sp) == [total] * conns
        check()
        return ev[0].elapsed_time(ev[1]) * 1e-3, ev[1].elapsed_time(ev[2]) * 1e-3

    def device_step(mod, RS, RR):
        h = S.claim()
        RS.prepare(h, S.sends(mod))
        RR.prepare(h, S.recvs(mod))
        stream.synchronize()
        ev[0].record(stream)
        RS.fire(60.0, stream=sp)
        ev[1].record(stream)
        RR.fire(60.0, stream=sp)
        ev[2].record(stream)
        rs, rr = RS.wait(), RR.wait()
        assert all(o[0]["ret"] == total for o in rs) and all(o[0]["ret"] == total for o in rr), (rs, rr)
        S.release()
        check()
        return ev[0].elapsed_time(ev[1]) * 1e-3, ev[1].elapsed_time(ev[2]) * 1e-3

    variants = {"block": lambda R=(bl.Runner(pkg), bl.Runner(pkg)): device_step(bl, *R)}
    for k in KS:
        if cl.max_clusters(k) >= 1:
            variants["cluster_%d" % k] = lambda R=(cl.Runner(pkg, k), cl.Runner(pkg, k)): device_step(cl, *R)
    variants["k_send_k_recv"] = cta_step
    times = {name: [] for name in variants}
    for f in variants.values():  # warm-up
        f()
    for _ in range(reps):
        for name, f in variants.items():
            times[name].append(f())
    bs.destroy()
    br.destroy()
    S.teardown()
    tx_b, rx_b = pkg.frame_hbm_bytes(S.lens, stamped=stamped)
    payload, hbm = conns * total, conns * (tx_b + rx_b)
    return {"format": "stamped" if stamped else "reference", "conns": conns, "msg_bytes": total,
            "payload_bytes": payload, "hbm_bytes": hbm,
            "variants": {name: _row(ts, payload, hbm) for name, ts in times.items()}}


def duplex(pkg, torch, bl, cl, conns, msg, reps):
    S = Setup(pkg, torch, conns, 4096, msg, False, "cd%d" % conns)
    total = S.total
    stream = torch.cuda.Stream()
    sp = stream.cuda_stream
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def step(mod, R):
        h = S.claim()
        lists = [x for c in range(conns) for x in (S.sends(mod, True)[c], S.recvs(mod, True)[c])]
        R.prepare(h, lists)
        stream.synchronize()
        ev[0].record(stream)
        R.fire(120.0, stream=sp)
        ev[1].record(stream)
        res = R.wait()
        assert all(o[0]["status"] == mod.OK and o[0]["ret"] == total for o in res), res
        S.release()
        assert torch.equal(S.src, S.dst), "delivered bytes differ from what was sent"
        S.dst.zero_()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) * 1e-3

    variants = {"block": lambda R=bl.Runner(pkg): step(bl, R)}
    skipped = {}
    for k in KS:
        if cl.max_clusters(k) >= 2 * conns:  # the sender and receiver clusters wait for each other
            variants["cluster_%d" % k] = lambda R=cl.Runner(pkg, k): step(cl, R)
        else:
            skipped["cluster_%d" % k] = "%d clusters of %d CTAs cannot be resident at once" % (2 * conns, k)
    times = {name: [] for name in variants}
    for f in variants.values():
        f()
    for _ in range(reps):
        for name, f in variants.items():
            times[name].append(f())
    S.teardown()
    payload = conns * total
    out = {}
    for name, ts in times.items():
        m = statistics.median(ts)
        out[name] = {"ms": round(m * 1e3, 3), "GBps": round(payload / m / 1e9, 2),
                     "runs_ms": [round(t * 1e3, 3) for t in ts]}
    return {"conns": conns, "msg_bytes": total, "ring_bytes": 4 << 20, "payload_bytes": payload, "variants": out,
            "not_placed": skipped}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--conns", type=int, nargs="+", default=[1, 4, 16, 64])
    ap.add_argument("--msg-bytes", type=int, default=32 << 20)
    ap.add_argument("--duplex-conns", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    import device_block_lib
    import device_cluster_lib
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    pkg = ge.load_package()
    pkg.init(0)
    torch.cuda.init()
    line = {"card": card(), "ring_bytes": 64 << 20,
            "max_clusters": {k: device_cluster_lib.max_clusters(k) for k in (1,) + KS},
            "rate": [rate(pkg, torch, device_block_lib, device_cluster_lib, c, args.msg_bytes, st, args.reps)
                     for st in (False, True) for c in args.conns],
            "duplex": [duplex(pkg, torch, device_block_lib, device_cluster_lib, c, args.msg_bytes, args.reps)
                       for c in args.duplex_conns]}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
