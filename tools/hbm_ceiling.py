"""HBM ceiling for the streaming kernels' two traffic mixes, in one process (experiment helper).

Prints the card's name and power limit, then one line per variant with the traffic rate (bytes read + bytes
written per second), median and spread over --rounds rounds in which the variants alternate:

  ref  copy / copy+clear, vector and TMA    tools/native/hbm_ref.cu over 1 GiB contiguous buffers: what plain
                                            code reaches for the k_send mix (read 1, write 1) and the k_recv mix
                                            (read 1, write 2)
  probe mode 0 / mode 2, mis 0/8/5          the library's movers without framing (b200_probe_copy) at the
                                            benchmark's shape: 256 CTAs x 4 MiB, CTA c at c * stride, stride
                                            16 MiB (the rings) and 16 MiB + 4 KiB (every CTA at another offset)

The real kernels' k_send / k_recv times come from bench.py (roofline.kernels), run next to this.

    python tools/hbm_ceiling.py [--rounds 3] [--reps 10] [--lib PATH]
"""
import argparse
import ctypes as C
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def build_ref(tmp):
    so = os.path.join(tmp, "hbm_ref.so")
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-shared", "-Xcompiler", "-fPIC",
                           "-o", so, os.path.join(ROOT, "tools", "native", "hbm_ref.cu")])
    lib = C.CDLL(so)
    lib.hbm_ref_run.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p]
    return lib


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                                        "--format=csv,noheader"], text=True).strip()
    except Exception as exc:
        return "%s (nvidia-smi: %r)" % (torch.cuda.get_device_name(), exc)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10, help="launches per timed window")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hbm_ceiling.py: no CUDA device")
    pkg = ge.load_package()
    pkg.init(0)
    L = pkg.lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    sh = C.c_void_p(stream.cuda_stream)
    print("card: %s; lib: %s" % (card(), os.environ.get("B200RDMA_LIB", "default")), flush=True)

    def timed(fn, traffic):
        for _ in range(2):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.reps):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return traffic * args.reps / (e0.elapsed_time(e1) * 1e-3) / 1e9

    variants = []
    with tempfile.TemporaryDirectory() as tmp:
        R = build_ref(tmp)
        G = 1 << 30
        a = torch.randint(0, 255, (G,), dtype=torch.uint8, device="cuda")
        b = torch.empty(G, dtype=torch.uint8, device="cuda")
        for v, name, mult in ((0, "ref copy       vec", 2), (1, "ref copy+clear vec", 3),
                              (2, "ref copy       tma", 2), (3, "ref copy+clear tma", 3)):
            variants.append((name, (lambda v=v: R.hbm_ref_run(v, b.data_ptr(), a.data_ptr(), G, sms, sh)), mult * G))
        conns, per_cta = 256, 4 << 20
        strides = (16 << 20, (16 << 20) + 4096)
        span = (conns - 1) * max(strides) + per_cta + 4096
        src = torch.randint(0, 255, (span,), dtype=torch.uint8, device="cuda")
        dst = torch.empty(span, dtype=torch.uint8, device="cuda")
        for stride in strides:
            for mode in (0, 2):
                for mis in (0, 8, 5):
                    # mode 2 clears the source: the bytes it reads the next time are zeros, which costs the same
                    name = "probe %-4s stride=%-9d mis=%d" % ("send" if mode == 0 else "recv", stride, mis)
                    fn = (lambda stride=stride, mode=mode, mis=mis: L.b200_probe_copy(
                        dst.data_ptr(), src.data_ptr(), per_cta, stride, conns, 288, mis, 4096, mode, sh))
                    variants.append((name, fn, (2 if mode == 0 else 3) * conns * per_cta))
        res = {n: [] for n, _, _ in variants}
        for r in range(args.rounds):
            for name, fn, traffic in variants:
                res[name].append(timed(fn, traffic))
        for name, _, _ in variants:
            v = res[name]
            print("%-40s %7.0f GB/s of traffic  (rounds: %s)" % (name, statistics.median(v),
                                                              " ".join("%.0f" % x for x in v)), flush=True)


if __name__ == "__main__":
    main()
