// hbm_ref.cu -- EXPERIMENT HELPER (not product code): reference kernels for the two traffic mixes of the
// streaming kernels, i.e. what plain code reaches on this GPU for
//   copy        read n, write n                 (the k_send mix)
//   copy+clear  read n, write n, zero the source (the k_recv mix)
// over contiguous buffers, each with 16-byte vector loads/stores (grid-stride) and with TMA bulk copies
// (cp.async.bulk global->shared->global).  tools/hbm_ceiling.py builds this into a shared library in a
// temporary directory and drives it through ctypes:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -shared -Xcompiler -fPIC -o hbm_ref.so tools/native/hbm_ref.cu
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

__device__ __forceinline__ uint4 ld16(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st16(uint4* p, uint4 v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

// 4 vectors in flight per thread, grid-stride
template <bool kClear>
__global__ void __launch_bounds__(256) k_vec(uint4* __restrict__ dst, uint4* __restrict__ src, uint64_t nvec) {
  const uint64_t step = (uint64_t)gridDim.x * blockDim.x;
  const uint4 z = make_uint4(0, 0, 0, 0);
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += 4 * step) {
    uint4 v[4];
#pragma unroll
    for (int k = 0; k < 4; k++)
      if (i + k * step < nvec) v[k] = ld16(src + i + k * step);
#pragma unroll
    for (int k = 0; k < 4; k++)
      if (i + k * step < nvec) {
        st16(dst + i + k * step, v[k]);
        if (kClear) st16(src + i + k * step, z);
      }
  }
}

constexpr uint32_t kTmaChunk = 16384;  // bytes per bulk copy
constexpr uint32_t kTmaStages = 4;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// One elected thread per CTA runs a kTmaStages-deep pipeline: bulk load chunk i into stage i % S while the
// store of chunk i - (S - 1) (and, with kClear, a bulk store of zeros over its source) drains.
template <bool kClear>
__global__ void __launch_bounds__(32) k_tma(uint8_t* __restrict__ dst, uint8_t* __restrict__ src, uint64_t nchunks) {
  extern __shared__ __align__(128) uint8_t sm[];
  uint8_t* zero = sm + kTmaStages * kTmaChunk;
  __shared__ __align__(8) uint64_t bars[kTmaStages];
  if (kClear)
    for (uint32_t i = threadIdx.x; i < kTmaChunk / 16; i += 32) reinterpret_cast<uint4*>(zero)[i] = make_uint4(0, 0, 0, 0);
  if (threadIdx.x == 0)
    for (uint32_t s = 0; s < kTmaStages; s++)
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bars[s])) : "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  if (threadIdx.x != 0) return;
  constexpr uint32_t L = kTmaStages - 1;
  const uint64_t mine = nchunks > blockIdx.x ? (nchunks - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  for (uint64_t i = 0; i < mine + L; i++) {
    if (i >= L) {  // store chunk j
      const uint64_t j = i - L;
      const uint32_t s = (uint32_t)(j % kTmaStages), par = (uint32_t)((j / kTmaStages) & 1);
      uint32_t ok = 0;
      while (!ok)
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                     "selp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok)
                     : "r"(smem_u32(&bars[s])), "r"(par)
                     : "memory");
      const uint64_t off = (blockIdx.x + j * gridDim.x) * (uint64_t)kTmaChunk;
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst + off),
                   "r"(smem_u32(sm + s * kTmaChunk)), "r"(kTmaChunk)
                   : "memory");
      if (kClear)
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(src + off),
                     "r"(smem_u32(zero)), "r"(kTmaChunk)
                     : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    if (i < mine) {  // load chunk i into the stage whose store (chunk i - S, committed one group ago) has read it
      asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      const uint32_t s = (uint32_t)(i % kTmaStages);
      const uint64_t off = (blockIdx.x + i * gridDim.x) * (uint64_t)kTmaChunk;
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bars[s])), "r"(kTmaChunk)
                   : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                       smem_u32(sm + s * kTmaChunk)),
                   "l"(src + off), "r"(kTmaChunk), "r"(smem_u32(&bars[s]))
                   : "memory");
    }
  }
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

}  // namespace

extern "C" {

// variant: 0 copy (vector), 1 copy+clear (vector), 2 copy (TMA), 3 copy+clear (TMA).
// bytes: a multiple of 16 KiB; both buffers 16-byte aligned.  Returns a cudaError_t.
int hbm_ref_run(int variant, void* dst, void* src, uint64_t bytes, int sms, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint32_t smem = kTmaStages * kTmaChunk + ((variant & 1) ? kTmaChunk : 0);
  switch (variant) {
    case 0: k_vec<false><<<sms * 8, 256, 0, st>>>((uint4*)dst, (uint4*)src, bytes / 16); break;
    case 1: k_vec<true><<<sms * 8, 256, 0, st>>>((uint4*)dst, (uint4*)src, bytes / 16); break;
    case 2:
      cudaFuncSetAttribute(k_tma<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      k_tma<false><<<sms * 2, 32, smem, st>>>((uint8_t*)dst, (uint8_t*)src, bytes / kTmaChunk);
      break;
    case 3:
      cudaFuncSetAttribute(k_tma<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      k_tma<true><<<sms * 2, 32, smem, st>>>((uint8_t*)dst, (uint8_t*)src, bytes / kTmaChunk);
      break;
    default: return (int)cudaErrorInvalidValue;
  }
  return (int)cudaGetLastError();
}
}
