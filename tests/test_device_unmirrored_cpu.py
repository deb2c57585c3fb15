"""CPU: the unmirrored device claim (b200_pair_device_claim_ex, B200_CLAIM_UNMIRRORED): the symbol, the flag and the
binding, the refusal of unknown flag bits, a user kernel with every device call that skips the publication compiles for
sm_90a without spills, and the library kernels keep their registers.  No GPU needed."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]

USER_KERNELS = r'''
#include "b200_device_block.cuh"
__global__ void warp_calls(const b200_dev_pair* h, const b200_slice* s, uint32_t n, uint8_t* dst, uint64_t* out) {
  const uint64_t a = b200_warp_send(&h[0], s, n, 0);
  const uint64_t b = b200_warp_recv(&h[1], dst, 4096);
  const int d = b200_warp_disconnect(&h[0]);
  if ((threadIdx.x & 31) == 0) out[0] = a + b + d + b200_warp_writable(&h[1]) + b200_warp_status(&h[1]);
}
__global__ void __launch_bounds__(B200_BLOCK_THREADS, 2) cluster_send(const b200_dev_pair* h, const b200_slice* s,
                                                                       uint64_t n, uint64_t* out) {
  __shared__ b200_block st;
  b200_block_init(&st);
  const uint64_t a = b200_cluster_send(&st, h, s, n, 0, B200_BATCH_UNTIL_BLOCKED, nullptr);
  if (threadIdx.x == 0) out[0] = a;
}
__global__ void __launch_bounds__(B200_BLOCK_THREADS, 2) block_recv(const b200_dev_pair* h, uint8_t* dst, uint64_t cap,
                                                                     uint64_t* out) {
  __shared__ b200_block st;
  b200_block_init(&st);
  const uint64_t b = b200_block_recv(&st, h, dst, cap, B200_BATCH_ONE_CALL, nullptr);
  if (threadIdx.x == 0) out[0] = b;
}
'''


def _ptxas(args, cwd):
    out = subprocess.run([NVCC] + ARCH + ["-O3", "-std=c++17", "-Xptxas", "-v"] + args, capture_output=True,
                         text=True, cwd=cwd)
    assert out.returncode == 0, out.stdout + out.stderr
    return out.stderr


def _kernels(report):
    """{kernel: (registers, spill stores, spill loads)} from a ptxas -v report (entry functions)"""
    res, name, spills = {}, None, None
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name, spills = m.group(1), None
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name and spills is None:
            spills = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            res[name] = (int(m.group(1)),) + (spills or (0, 0))
    return res


def _pick(ks, part):
    hits = [v for k, v in ks.items() if part in k]
    assert len(hits) == 1, (part, ks)
    return hits[0]


def test_header_declares_the_flag_and_the_call():
    src = open(os.path.join(ROOT, "include", "b200_pair.h")).read()
    assert re.search(r"#define B200_CLAIM_UNMIRRORED 0x1\b", src)
    assert re.search(r"int b200_pair_device_claim_ex\(b200_pair\* p, int flags, b200_dev_pair\* out\);", src)
    assert "frozen" in src.lower()


def test_binding(pkg):
    import inspect
    assert pkg.CLAIM_UNMIRRORED == 0x1
    assert "b200_pair_device_claim_ex" in pkg.exported_symbols()
    assert inspect.signature(pkg.Pair.device_claim).parameters["mirrored"].default is True
    assert hasattr(pkg.lib(), "b200_pair_device_claim_ex")


@pytest.mark.parametrize("flags", [0x2, 0x100, -1])
def test_unknown_flag_bits_are_refused(pkg, flags):
    out = C.create_string_buffer(64)
    assert pkg.lib().b200_pair_device_claim_ex(None, flags, out) == -1
    assert "unknown flag bits" in pkg.last_error()


def test_user_kernels_compile_without_spills():
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "user.cu"), "w") as f:
            f.write(USER_KERNELS)
        ks = _kernels(_ptxas(["-I", os.path.join(ROOT, "include"), "-c", "user.cu", "-o", "user.o"], d))
    for part in ("warp_calls", "cluster_send", "block_recv"):
        regs, st, ld = _pick(ks, part)
        assert st == 0 and ld == 0, (part, ks)


def test_library_kernels_keep_their_registers():
    with tempfile.TemporaryDirectory() as d:
        ks = _kernels(_ptxas(["-Xcompiler", "-fPIC", "-cubin", "-o", os.path.join(d, "k.cubin"),
                              os.path.join(ROOT, "grpc-rdma_b200", "csrc", "b200_kernels.cu")], d))
    assert _pick(ks, "k_send")[0] == 80 and _pick(ks, "k_recv")[0] == 96, ks
    assert _pick(ks, "k_svc_big") == (96, 20, 20), ks
    assert _pick(ks, "k_svc_owner")[0] == 124 and _pick(ks, "k_svc_poll")[0] == 32, ks
    assert _pick(ks, "k_poll_scan")[0] == 28, ks
