"""CPU: the block-level device API (include/b200_device_block.cuh) and its test driver compile for sm_90a against the
public header alone; a user kernel's block calls keep the registers of the library's kernels that run the same
bodies, and two such CTAs fit on an SM.  No GPU needed."""
import os
import re
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
SMEM_PER_SM = 228 * 1024     # H100: shared memory per SM
SMEM_PER_CTA_RESERVED = 1024  # the runtime's reservation per resident CTA
BLOCK_SMEM_BYTES = 99072

USER_KERNELS = r'''
#include "b200_device_block.cuh"
__global__ void __launch_bounds__(B200_BLOCK_THREADS, 2) only_send(const b200_dev_pair* h, const b200_slice* s,
                                                                    uint64_t n, uint64_t* out) {
  __shared__ b200_block st;
  b200_block_init(&st);
  uint64_t c;
  const uint64_t r = b200_block_send(&st, h, s, n, 0, B200_BATCH_UNTIL_BLOCKED, &c);
  if (threadIdx.x == 0) { out[0] = r; out[1] = c; }
}
__global__ void __launch_bounds__(B200_BLOCK_THREADS, 2) only_recv(const b200_dev_pair* h, uint8_t* dst, uint64_t cap,
                                                                    uint64_t* out) {
  __shared__ b200_block st;
  b200_block_init(&st);
  uint64_t c;
  const uint64_t r = b200_block_recv(&st, h, dst, cap, B200_BATCH_UNTIL_BLOCKED, &c);
  if (threadIdx.x == 0) { out[0] = r; out[1] = c; }
}
__global__ void __launch_bounds__(B200_BLOCK_THREADS, 2) send_then_recv(const b200_dev_pair* h, const b200_slice* s,
                                                                         uint64_t n, uint8_t* dst, uint64_t* out) {
  __shared__ b200_block st;
  b200_block_init(&st);
  const uint64_t a = b200_block_send(&st, &h[0], s, n, 0, B200_BATCH_ONE_CALL, nullptr);
  const uint64_t b = b200_block_recv(&st, &h[1], dst, a, B200_BATCH_ONE_CALL, nullptr);
  if (threadIdx.x == 0) out[0] = a + b;
}
'''


def _ptxas(args, cwd):
    out = subprocess.run([NVCC] + ARCH + ["-O3", "-std=c++17", "-lineinfo", "-Xptxas", "-v"] + args,
                         capture_output=True, text=True, cwd=cwd)
    assert out.returncode == 0, out.stdout + out.stderr
    return out.stderr


def _kernels(report):
    """{kernel: (registers, spill stores, spill loads, static smem)} from a ptxas -v report (entry functions)"""
    res, name, spills = {}, None, (0, 0)
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name, spills = m.group(1), (0, 0)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name and (name, "seen") not in res:
            spills = (int(m.group(1)), int(m.group(2)))
            res[(name, "seen")] = True
        m = re.search(r"Used (\d+) registers.*?(?:(\d+) bytes smem)?$", line)
        if m and name:
            res[name] = (int(m.group(1)),) + spills + (int(m.group(2) or 0),)
    return {k: v for k, v in res.items() if not isinstance(k, tuple)}


def _pick(ks, part):
    hits = [v for k, v in ks.items() if part in k]
    assert len(hits) == 1, (part, ks)
    return hits[0]


def _library_kernels():
    with tempfile.TemporaryDirectory() as d:
        rep = _ptxas(["-Xcompiler", "-fPIC", "-cubin", "-o", os.path.join(d, "k.cubin"),
                      os.path.join(ROOT, "grpc-rdma_b200", "csrc", "b200_kernels.cu")], d)
    return _kernels(rep)


def _user_kernels():
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "user.cu"), "w") as f:
            f.write(USER_KERNELS)
        rep = _ptxas(["-I", os.path.join(ROOT, "include"), "-c", "user.cu", "-o", "user.o"], d)
    return _kernels(rep)


def test_block_calls_keep_the_library_kernels_registers():
    lib, user = _library_kernels(), _user_kernels()
    k_send, k_recv, k_svc_big = _pick(lib, "k_send"), _pick(lib, "k_recv"), _pick(lib, "k_svc_big")
    only_send, only_recv, both = _pick(user, "only_send"), _pick(user, "only_recv"), _pick(user, "send_then_recv")
    # a kernel with only b200_block_send is k_send: the same registers, no spills; only b200_block_recv: k_recv
    assert only_send[0] == k_send[0] and only_send[1:3] == (0, 0), (only_send, k_send)
    assert only_recv[0] == k_recv[0] and only_recv[1:3] == (0, 0), (only_recv, k_recv)
    # both bodies in one kernel, as in the service pool: no more spilled than k_svc_big
    assert both[0] <= k_svc_big[0] and both[1] <= k_svc_big[1] and both[2] <= k_svc_big[2], (both, k_svc_big)
    # under __launch_bounds__(288, 2), static + dynamic shared memory leaves two CTAs per SM
    for k in (only_send, only_recv, both):
        assert 2 * (k[3] + BLOCK_SMEM_BYTES + SMEM_PER_CTA_RESERVED) <= SMEM_PER_SM, k
        assert k[0] * 288 * 2 <= 65536, k


def test_driver_compiles_for_sm90a_against_the_public_header():
    with tempfile.TemporaryDirectory() as d:
        so = os.path.join(d, "libdevice_block.so")
        rep = _ptxas(["-Xcompiler", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "native", "device_block.cu")], d)
        ks = _kernels(rep)
        assert any("bd_kernel" in k for k in ks), rep
        elf = subprocess.run(["cuobjdump", "-lelf", so], capture_output=True, text=True).stdout
        assert "sm_90a" in elf, elf


def test_public_header_constants():
    src = open(os.path.join(ROOT, "include", "b200_device_block.cuh")).read()
    assert re.search(r"#define B200_BLOCK_THREADS 288\b", src)
    assert re.search(r"#define B200_BLOCK_SMEM_BYTES %d\b" % BLOCK_SMEM_BYTES, src)
    # the warp-only header does not pull the CTA pipeline into kernels that use only the warp calls
    assert "b200_block" not in open(os.path.join(ROOT, "include", "b200_device.cuh")).read()
