"""CPU: the cluster calls (b200_cluster_send / b200_cluster_recv, include/b200_device_block.cuh) and their test driver
compile for sm_90a against the public header alone; a user kernel that calls only one of them keeps two CTAs per SM
with no spills, and the shared memory of two such CTAs fits an SM.  No GPU needed."""
import os
import subprocess
import tempfile

import test_device_block_cpu as tb

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

USER_KERNELS = r'''
#include "b200_device_block.cuh"
__global__ void __launch_bounds__(B200_BLOCK_THREADS, 2) cluster_send_only(const b200_dev_pair* h,
                                                                            const b200_slice* s, uint64_t n,
                                                                            uint64_t* out) {
  __shared__ b200_block st;
  b200_block_init(&st);
  uint64_t c;
  const uint64_t r = b200_cluster_send(&st, h, s, n, 0, B200_BATCH_UNTIL_BLOCKED, &c);
  if (threadIdx.x == 0) { out[0] = r; out[1] = c; }
}
__global__ void __launch_bounds__(B200_BLOCK_THREADS, 2) cluster_recv_only(const b200_dev_pair* h, uint8_t* dst,
                                                                            uint64_t cap, uint64_t* out) {
  __shared__ b200_block st;
  b200_block_init(&st);
  uint64_t c;
  const uint64_t r = b200_cluster_recv(&st, h, dst, cap, B200_BATCH_UNTIL_BLOCKED, &c);
  if (threadIdx.x == 0) { out[0] = r; out[1] = c; }
}
'''

# both calls in one kernel, as a duplex user kernel would have them (compiled on its own: the producers are shared
# non-inlined functions, so a kernel beside them in the translation unit changes how they are allocated)
BOTH_KERNEL = r'''
#include "b200_device_block.cuh"
__global__ void __cluster_dims__(4, 1, 1) __launch_bounds__(B200_BLOCK_THREADS, 2) cluster_both(
    const b200_dev_pair* h, const b200_slice* s, uint64_t n, uint8_t* dst, uint64_t* out) {
  __shared__ b200_block st;
  b200_block_init(&st);
  const uint64_t a = b200_cluster_send(&st, &h[0], s, n, 0, B200_BATCH_ONE_CALL, nullptr);
  const uint64_t b = b200_cluster_recv(&st, &h[1], dst, a, B200_BATCH_ONE_CALL, nullptr);
  if (threadIdx.x == 0) out[0] = a + b;
}
'''


def _user_kernels(src):
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "user.cu"), "w") as f:
            f.write(src)
        rep = tb._ptxas(["-I", os.path.join(ROOT, "include"), "-c", "user.cu", "-o", "user.o"], d)
    return tb._kernels(rep)


def test_cluster_calls_fit_two_ctas_per_sm_without_spills():
    user = _user_kernels(USER_KERNELS)
    user.update(_user_kernels(BOTH_KERNEL))
    for name in ("cluster_send_only", "cluster_recv_only", "cluster_both"):
        regs, st, ld, smem = tb._pick(user, name)
        # two CTAs of 288 threads per SM: the register file holds them, and nothing spills in a kernel with one call
        assert regs * 288 * 2 <= 65536, (name, regs)
        if name != "cluster_both":
            assert (st, ld) == (0, 0), (name, st, ld)
        # static + dynamic shared memory of two CTAs fits an SM
        assert 2 * (smem + tb.BLOCK_SMEM_BYTES + tb.SMEM_PER_CTA_RESERVED) <= tb.SMEM_PER_SM, (name, smem)


def test_driver_compiles_for_sm90a_against_the_public_header():
    with tempfile.TemporaryDirectory() as d:
        so = os.path.join(d, "libdevice_cluster.so")
        rep = tb._ptxas(["-Xcompiler", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "native", "device_cluster.cu")],
                        d)
        assert any("cd_kernel" in k for k in tb._kernels(rep)), rep
        elf = subprocess.run(["cuobjdump", "-lelf", so], capture_output=True, text=True).stdout
        assert "sm_90a" in elf, elf


def test_block_calls_compile_what_they_did():
    """a kernel that calls only the block calls compiles no cluster instruction"""
    src = tb.USER_KERNELS
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "user.cu"), "w") as f:
            f.write(src)
        subprocess.run([tb.NVCC] + tb.ARCH + ["-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-cubin",
                                              "-o", "user.cubin", "user.cu"], check=True, cwd=d, capture_output=True)
        sass = subprocess.run(["cuobjdump", "-sass", os.path.join(d, "user.cubin")], capture_output=True,
                              text=True).stdout
    assert "UCGABAR" not in sass and "MAPA" not in sass, "cluster instructions in a block-call kernel"
