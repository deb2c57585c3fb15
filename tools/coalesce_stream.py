"""BASELINE configs[1] (256 connections, 16 MiB rings, 4 MiB chttp2-shaped messages, one GPU) with per-slice and
coalesced send framing (B200_SEND_COALESCE), alternating in one process.  Per mode: device time per step and
GB/s from CUDA events, Send / Recv calls and ring bytes per message, and the rate through the endpoint surface
(lib/libb200_epstream.so) with the mode set before its pairs are initialised.  Prints one JSON line.

    python tools/coalesce_stream.py [--steps 20] [--rounds 3] [--conns 256]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        name, power = subprocess.check_output(
            ["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().split(", ")
        return {"name": name, "power_limit": power}
    except Exception as exc:  # the number still stands, but without its card it is not worth much
        return {"error": repr(exc)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--conns", type=int, default=256)
    ap.add_argument("--ring-kb", type=int, default=16384)
    ap.add_argument("--msg-bytes", type=int, default=4 << 20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the two modes")
    ap.add_argument("--endpoint-threads", type=int, default=8)
    ap.add_argument("--endpoint-msgs", type=int, default=8)
    ap.add_argument("--endpoint-pool", type=int, default=128)
    ap.add_argument("--no-endpoint", action="store_true")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    if not torch.cuda.is_available():
        raise SystemExit("coalesce_stream.py: no CUDA device")
    pkg = ge.load_package()
    L = pkg.lib()
    pkg.init(0)
    dev = torch.device("cuda", 0)
    conns, msg, cap = args.conns, args.msg_bytes, args.ring_kb * 1024
    lens = pkg.chttp2_slice_lens(msg)
    total = sum(lens)
    pkg.config_set("GRPC_RDMA_RING_BUFFER_SIZE_KB", args.ring_kb)
    pkg.config_set("GRPC_RDMA_MAX_SGE", 30)
    i = torch.arange(total, device=dev, dtype=torch.int64)
    row = (((i * 2654435761) >> 11) & 255).to(torch.uint8)
    offs = (torch.arange(conns, device=dev, dtype=torch.int64) * 131 & 255).to(torch.uint8)
    src = (row[None, :] + offs[:, None]).reshape(-1)
    del i, row, offs
    dst = torch.zeros(conns * total, dtype=torch.uint8, device=dev)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    sh = C.c_void_p(stream.cuda_stream)

    modes = {}
    for mode in (0, 1):
        pkg.config_set("B200_SEND_COALESCE", mode)
        pairs = [pkg.connected_pair("cs%d-%d-tx" % (mode, c), "cs%d-%d-rx" % (mode, c)) for c in range(conns)]
        sops, rops, keep = [], [], []
        for c in range(conns):
            off, sl = 0, []
            for n in lens:
                sl.append((src.data_ptr() + c * total + off, n))
                off += n
            arr = pkg.make_slices(sl)
            keep.append(arr)
            sops.append((pairs[c][0], arr, len(lens), 0))
            rops.append((pairs[c][1], dst.data_ptr() + c * total, total))
        modes[mode] = {"pairs": pairs, "keep": keep, "bs": pkg.Batch("send", sops, pkg.UNTIL_BLOCKED),
                       "br": pkg.Batch("recv", rops, pkg.UNTIL_BLOCKED), "step_ms": []}
    pkg.config_set("B200_SEND_COALESCE", 0)

    for m in modes.values():  # warm-up, per-message counts, correctness
        for _ in range(args.warmup):
            m["bs"].launch(sh)
            m["br"].launch(sh)
        torch.cuda.synchronize()
        t0 = m["pairs"][0][0].state()["remote_tail"]
        m["bs"].launch(sh)
        m["br"].launch(sh)
        assert m["bs"].results(sh) == [total] * conns and m["br"].results(sh) == [total] * conns
        m["send_calls"], m["recv_calls"] = m["bs"].calls()[0], m["br"].calls()[0]
        m["ring_bytes"] = (m["pairs"][0][0].state()["remote_tail"] - t0) % cap
        assert torch.equal(src, dst), "delivered bytes differ from what was sent"
        dst.zero_()
    for _ in range(args.rounds):
        for m in modes.values():
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
            ev[0].record(stream)
            for k in range(args.steps):
                m["bs"].launch(sh)
                m["br"].launch(sh)
                ev[k + 1].record(stream)
            torch.cuda.synchronize()
            m["step_ms"].append(ev[0].elapsed_time(ev[-1]) / args.steps)
            assert m["bs"].results(sh) == [total] * conns and torch.equal(src, dst)
            dst.zero_()
    out = {"config": "configs[1]: %d connections x %d-byte chttp2-shaped messages (%d slices), ring %d KiB, 1 GPU"
                     % (conns, msg, len(lens), args.ring_kb),
           "card": card(), "steps": args.steps, "rounds": args.rounds}
    for mode, m in modes.items():
        med = statistics.median(m["step_ms"])
        out["coalesced" if mode else "per_slice"] = {
            "device_ms_per_step": med, "device_ms_per_step_all_rounds": m["step_ms"],
            "device_GBps": conns * msg / (med * 1e-3) / 1e9,
            "send_calls_per_msg": m["send_calls"], "recv_calls_per_msg": m["recv_calls"],
            "ring_bytes_per_msg": m["ring_bytes"]}
        m["bs"].destroy()
        m["br"].destroy()
        for tx, rx in m["pairs"]:
            tx.disconnect(); rx.disconnect(); tx.putback(); rx.putback()
    del src, dst
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

    if not args.no_endpoint:
        C.CDLL(pkg.ENDPOINT_LIB_PATH, mode=C.RTLD_GLOBAL)
        ES = C.CDLL(os.path.join(os.path.dirname(pkg.LIB_PATH), "libb200_epstream.so"))
        ES.ep_stream_run.restype = C.c_double
        ES.ep_stream_run.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_int,
                                     C.POINTER(C.c_uint64)]
        ep = {0: [], 1: []}
        if L.b200_service_start(args.endpoint_pool) != 0:
            out["endpoint"] = {"error": "b200_service_start: " + pkg.last_error()}
        else:
            try:
                for _ in range(args.rounds):
                    for mode in (0, 1):
                        pkg.config_set("B200_SEND_COALESCE", mode)  # before the driver initialises its pairs
                        o = (C.c_uint64 * 4)()
                        t = ES.ep_stream_run(None, conns, args.endpoint_threads, args.endpoint_msgs, 2, msg, 0, o)
                        ep[mode].append({"GBps": o[0] / t / 1e9, "bad_bytes": int(o[1])} if t > 0 else {"error": t})
            finally:
                pkg.config_set("B200_SEND_COALESCE", 0)
                L.b200_service_stop()
            for mode in (0, 1):
                rates = [r["GBps"] for r in ep[mode] if "GBps" in r]
                out["coalesced" if mode else "per_slice"]["endpoint"] = {
                    "GBps_median": statistics.median(rates) if rates else None, "runs": ep[mode],
                    "path": "b200_endpoint_write/read + b200_engine_work, service with %d pool CTAs, %d thread pairs"
                            % (args.endpoint_pool, args.endpoint_threads)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
