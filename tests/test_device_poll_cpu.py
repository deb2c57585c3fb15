"""CPU: the device poll / status / writable / Disconnect calls (include/b200_device.cuh) and their test driver compile for
sm_90a against the public header alone, without spills; a kernel that only polls pulls in nothing of the CTA pipeline;
and sharing the readiness rule with k_poll_scan leaves the library's kernels' -Xptxas -v numbers where they were.
No GPU needed."""
import os
import re
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]

POLL_ONLY = r'''
#include "b200_device.cuh"
__global__ void poll_only(const b200_dev_pair* h, uint32_t n, uint32_t* events, uint32_t* ready, int* st,
                          uint64_t* out) {
  const uint32_t c = b200_warp_poll(h, n, events, ready);
  const int s = b200_warp_status(&h[0]);
  if ((threadIdx.x & 31) == 0) { out[0] = c; st[0] = s; }
}
'''


def _ptxas(args, cwd):
    out = subprocess.run([NVCC] + ARCH + ["-O3", "-std=c++17", "-lineinfo", "-Xptxas", "-v"] + args,
                         capture_output=True, text=True, cwd=cwd)
    assert out.returncode == 0, out.stdout + out.stderr
    return out.stderr


def _kernels(report):
    """{kernel: (registers, spill stores, spill loads)} from a ptxas -v report (entry functions)"""
    res, name, spills = {}, None, (0, 0)
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


def test_driver_compiles_for_sm90a_without_spills():
    with tempfile.TemporaryDirectory() as d:
        so = os.path.join(d, "libdevice_poll.so")
        rep = _ptxas(["-Xcompiler", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "native", "device_poll.cu")], d)
        ks = _kernels(rep)
        for k in ("dp_kernel", "dp_poll_kernel", "dp_serve_kernel", "dp_poll_time_kernel"):
            assert any(k in name for name in ks), (k, rep)
        for k, (regs, st, ld) in ks.items():
            assert st == 0 and ld == 0, (k, regs, st, ld)
        elf = subprocess.run(["cuobjdump", "-lelf", so], capture_output=True, text=True).stdout
        assert "sm_90a" in elf, elf


def test_poll_only_kernel_needs_no_block_header():
    inc = ["-I", os.path.join(ROOT, "include")]
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "user.cu"), "w") as f:
            f.write(POLL_ONLY)
        ks = _kernels(_ptxas(inc + ["-c", "user.cu", "-o", "user.o"], d))
        regs, st, ld = _pick(ks, "poll_only")
        assert st == 0 and ld == 0, ks
        pre = subprocess.run([NVCC] + ARCH + ["-std=c++17", "-E"] + inc + ["user.cu"], capture_output=True,
                             text=True, cwd=d)
        assert pre.returncode == 0, pre.stderr
        assert "b200_block.cuh" not in pre.stdout and "b200_device_block.cuh" not in pre.stdout


def test_library_kernels_keep_their_registers():
    with tempfile.TemporaryDirectory() as d:
        ks = _kernels(_ptxas(["-Xcompiler", "-fPIC", "-cubin", "-o", os.path.join(d, "k.cubin"),
                              os.path.join(ROOT, "grpc-rdma_b200", "csrc", "b200_kernels.cu")], d))
    assert _pick(ks, "k_poll_scan")[0] == 28, ks
    assert _pick(ks, "k_send")[0] == 80 and _pick(ks, "k_recv")[0] == 96, ks
    assert _pick(ks, "k_svc_big") == (96, 20, 20), ks
    assert _pick(ks, "k_svc_owner")[0] == 124 and _pick(ks, "k_svc_poll")[0] == 32, ks
