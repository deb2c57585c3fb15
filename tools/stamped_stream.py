"""BASELINE configs[1] (256 connections, 16 MiB rings, 4 MiB chttp2-shaped messages, one GPU) in three modes,
alternating in one process: the reference format, stamped ring frames (B200_RING_STAMPED) and stamped + coalesced
send framing (B200_SEND_COALESCE).  Per mode: device time per step and GB/s from CUDA events, k_send and k_recv
times (events around each launch), the algorithmic HBM bytes per message of the mode, and the rate through the
endpoint surface (lib/libb200_epstream.so) with the mode set before its pairs are initialised.  Prints one JSON
line with the card's name and power limit read in the same run.  Without a CUDA device it fails.

    python tools/stamped_stream.py [--steps 20] [--rounds 3] [--conns 256]
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
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the three modes")
    ap.add_argument("--endpoint-threads", type=int, default=8)
    ap.add_argument("--endpoint-msgs", type=int, default=8)
    ap.add_argument("--endpoint-pool", type=int, default=128)
    ap.add_argument("--no-endpoint", action="store_true")
    args = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    if not torch.cuda.is_available():
        raise SystemExit("stamped_stream.py: no CUDA device")
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

    MODES = {"default": (0, 0), "stamped": (1, 0), "stamped_coalesced": (1, 1)}  # (RING_STAMPED, SEND_COALESCE)

    def set_mode(stamped, coalesce):
        pkg.config_set("B200_RING_STAMPED", stamped)
        pkg.config_set("B200_SEND_COALESCE", coalesce)

    modes = {}
    for name, (stamped, coalesce) in MODES.items():
        set_mode(stamped, coalesce)
        pairs = [pkg.connected_pair("ss-%s-%d-tx" % (name, c), "ss-%s-%d-rx" % (name, c)) for c in range(conns)]
        assert all(tx.stamped() == bool(stamped) for tx, _ in pairs)
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
        # algorithmic bytes per message: one frame of `total` bytes when coalesced, one per slice otherwise
        tx_b, rx_b = pkg.frame_hbm_bytes([total] if coalesce else lens, stamped=bool(stamped))
        modes[name] = {"pairs": pairs, "keep": keep, "bs": pkg.Batch("send", sops, pkg.UNTIL_BLOCKED),
                       "br": pkg.Batch("recv", rops, pkg.UNTIL_BLOCKED), "step_ms": [], "send_ms": [],
                       "recv_ms": [], "bytes": (tx_b, rx_b)}
    set_mode(0, 0)

    for m in modes.values():  # warm-up, correctness
        for _ in range(args.warmup):
            m["bs"].launch(sh)
            m["br"].launch(sh)
        torch.cuda.synchronize()
        m["bs"].launch(sh)
        m["br"].launch(sh)
        assert m["bs"].results(sh) == [total] * conns and m["br"].results(sh) == [total] * conns
        assert torch.equal(src, dst), "delivered bytes differ from what was sent"
        dst.zero_()
    for _ in range(args.rounds):
        for m in modes.values():
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * args.steps + 1)]
            ev[0].record(stream)
            for k in range(args.steps):
                m["bs"].launch(sh)
                ev[2 * k + 1].record(stream)
                m["br"].launch(sh)
                ev[2 * k + 2].record(stream)
            torch.cuda.synchronize()
            m["step_ms"].append(ev[0].elapsed_time(ev[-1]) / args.steps)
            m["send_ms"].append(sum(ev[2 * k].elapsed_time(ev[2 * k + 1]) for k in range(args.steps)) / args.steps)
            m["recv_ms"].append(sum(ev[2 * k + 1].elapsed_time(ev[2 * k + 2]) for k in range(args.steps)) / args.steps)
            assert m["bs"].results(sh) == [total] * conns and torch.equal(src, dst)
            dst.zero_()
    out = {"config": "configs[1]: %d connections x %d-byte chttp2-shaped messages (%d slices), ring %d KiB, 1 GPU"
                     % (conns, msg, len(lens), args.ring_kb),
           "card": card(), "steps": args.steps, "rounds": args.rounds}
    for name, m in modes.items():
        med = statistics.median(m["step_ms"])
        tx_b, rx_b = m["bytes"]
        out[name] = {
            "device_ms_per_step": med, "device_ms_per_step_all_rounds": m["step_ms"],
            "device_GBps": conns * msg / (med * 1e-3) / 1e9,
            "k_send_ms": statistics.median(m["send_ms"]), "k_recv_ms": statistics.median(m["recv_ms"]),
            "hbm_bytes_per_msg": {"k_send": tx_b, "k_recv": rx_b, "total": tx_b + rx_b,
                                  "per_payload_byte": (tx_b + rx_b) / msg}}
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
        ep = {name: [] for name in MODES}
        if L.b200_service_start(args.endpoint_pool) != 0:
            out["endpoint"] = {"error": "b200_service_start: " + pkg.last_error()}
        else:
            try:
                for _ in range(args.rounds):
                    for name, mode in MODES.items():
                        set_mode(*mode)  # before the driver initialises its pairs
                        o = (C.c_uint64 * 4)()
                        t = ES.ep_stream_run(None, conns, args.endpoint_threads, args.endpoint_msgs, 2, msg, 0, o)
                        ep[name].append({"GBps": o[0] / t / 1e9, "bad_bytes": int(o[1])} if t > 0 else {"error": t})
            finally:
                set_mode(0, 0)
                L.b200_service_stop()
            for name in MODES:
                rates = [r["GBps"] for r in ep[name] if "GBps" in r]
                out[name]["endpoint"] = {
                    "GBps_median": statistics.median(rates) if rates else None, "runs": ep[name],
                    "path": "b200_endpoint_write/read + b200_engine_work, service with %d pool CTAs, %d thread pairs"
                            % (args.endpoint_pool, args.endpoint_threads)}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
