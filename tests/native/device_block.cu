// device_block.cu -- TEST INFRASTRUCTURE: a user kernel that drives pairs through the public block-level device API
// (include/b200_device_block.cuh), and ctypes-callable launchers for it.  Built by device_block.mk for sm_90a against
// the public header only.
//
// One launch runs `nlists` lists of ops, one CTA (B200_BLOCK_THREADS threads) per list; list w is
// ops[first[w] .. first[w + 1]).  Lists run concurrently (e.g. one sender CTA and one receiver CTA per connection).
// Every loop is bounded by an iteration cap and a %globaltimer deadline: an op that hits either reports BD_TIMEOUT and
// the rest of its list is skipped.  Nothing waits without bound, and a launch whose CTAs wait for each other is refused
// unless they can all be resident at once.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200_device_block.cuh"

enum : uint32_t {
  BD_SEND = 1,         // one b200_block_send with the op's flags (ONE_CALL: one Send call; UNTIL_BLOCKED: rdma_flush)
  BD_RECV = 2,         // one b200_block_recv with the op's flags (ONE_CALL: one Recv call; UNTIL_BLOCKED: rdma_do_read)
  BD_STREAM_SEND = 3,  // send the whole slice list: UNTIL_BLOCKED block calls, retried while there is no credit
  BD_STREAM_RECV = 4,  // receive exactly n bytes into dst: UNTIL_BLOCKED block calls, retried while nothing is complete
  BD_WARP_SEND = 5,    // one b200_warp_send from warp 0 of the CTA (the other warps wait at a barrier)
  BD_WARP_RECV = 6,    // one b200_warp_recv from warp 0
};
enum : uint32_t { BD_OK = 0, BD_TIMEOUT = 1 };

struct bd_op {
  uint32_t kind, pair;  // pair: index into the handle array
  const b200_slice* slices;
  uint64_t n, byte_idx;  // send: slice count / byte_idx.  stream_recv: bytes
  uint8_t* dst;
  uint64_t cap;
  int32_t flags;  // BD_SEND / BD_RECV: passed to the call as it is
  uint32_t _pad0;
  uint64_t ret, calls;  // results
  uint32_t status, _pad;
};
static_assert(sizeof(bd_op) == 80, "bd_op layout is mirrored in tests/device_block_lib.py");

__device__ __forceinline__ uint64_t now_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

struct Bound {  // block-uniform: thread 0 reads the clock, the barrier gives every thread its answer
  uint64_t deadline, left;
  __device__ bool spent() {
    const int late = __syncthreads_or(threadIdx.x == 0 && now_ns() > deadline);
    return late || left-- == 0;
  }
};

// advance the (slice, byte) cursor by `sent` bytes, as rdma_flush does (rdma_bp_posix.cc:480-493)
__device__ __forceinline__ void advance(const b200_slice* s, uint64_t& idx, uint64_t& bidx, uint64_t sent) {
  while (sent > 0) {
    const uint64_t left = s[idx].len - bidx;
    if (sent >= left) {
      sent -= left;
      idx++;
      bidx = 0;
    } else {
      bidx += sent;
      sent = 0;
    }
  }
}

// kKinds: which calls the launch's lists hold (kSend | kRecv | kWarp).  The launcher picks the instantiation with just
// those, so that a launch of block sends only is k_send's code at k_send's registers, one of block receives k_recv's:
// the code of the other calls beside them costs spills in the movers' loop.
enum : uint32_t { kSend = 1, kRecv = 2, kWarp = 4 };
template <uint32_t kKinds>
__global__ void __launch_bounds__(B200_BLOCK_THREADS, 2)
bd_kernel(const b200_dev_pair* pairs, bd_op* ops, const uint32_t* first, int nlists, uint64_t budget_ns,
          uint64_t max_iters) {
  __shared__ b200_block st;
  __shared__ uint64_t s_t0, s_warp_ret;
  const int w = blockIdx.x;
  if (w >= nlists) return;
  b200_block_init(&st);
  if (threadIdx.x == 0) s_t0 = now_ns();
  __syncthreads();
  Bound b{s_t0 + budget_ns, max_iters};
  for (uint32_t i = first[w]; i < first[w + 1]; i++) {
    bd_op& o = ops[i];
    const b200_dev_pair* h = &pairs[o.pair];
    const uint32_t kind = o.kind;
    uint64_t ret = 0, calls = 0;
    uint32_t status = BD_OK;
    if ((kKinds & kSend) && (kind == BD_SEND || kind == BD_STREAM_SEND)) {  // one call site of b200_block_send for both
      const bool stream = kind == BD_STREAM_SEND;
      uint64_t idx = 0, bidx = o.byte_idx;
      while (idx < o.n) {
        uint64_t c = 0;
        const uint64_t sent = b200_block_send(&st, h, o.slices + idx, o.n - idx, bidx,
                                              stream ? B200_BATCH_UNTIL_BLOCKED : o.flags, &c);
        ret += sent;
        calls += c;
        if (!stream) break;
        if (sent) advance(o.slices, idx, bidx, sent);
        else if (b.spent()) {
          status = BD_TIMEOUT;
          break;
        }
      }
    } else if ((kKinds & kRecv) && (kind == BD_RECV || kind == BD_STREAM_RECV)) {
      const bool stream = kind == BD_STREAM_RECV;
      const uint64_t want = stream ? o.n : o.cap;
      do {
        uint64_t c = 0;
        const uint64_t got =
            b200_block_recv(&st, h, o.dst + ret, want - ret, stream ? B200_BATCH_UNTIL_BLOCKED : o.flags, &c);
        ret += got;
        calls += c;
        if (!stream) break;
        if (!got && b.spent()) {
          status = BD_TIMEOUT;
          break;
        }
      } while (ret < want);
    } else if ((kKinds & kWarp) && (kind == BD_WARP_SEND || kind == BD_WARP_RECV)) {
      if (threadIdx.x < 32) {
        const uint64_t r = kind == BD_WARP_SEND ? b200_warp_send(h, o.slices, (uint32_t)o.n, o.byte_idx)
                                                : b200_warp_recv(h, o.dst, o.cap);
        if (threadIdx.x == 0) s_warp_ret = r;
      }
      __syncthreads();
      ret = s_warp_ret;
      calls = ret != 0;
    } else {
      status = 2;
    }
    if (threadIdx.x == 0) {
      o.ret = ret;
      o.calls = calls;
      o.status = status;
    }
    __syncthreads();
    if (status != BD_OK) break;
  }
}

// A kernel that is not the pipeline's shape: every call refuses.  ret = the Send's answer + the Recv's answer.
__global__ void bd_wrong_shape(const b200_dev_pair* pairs, bd_op* ops) {
  __shared__ b200_block st;
  b200_block_init(&st);
  uint64_t c1 = 7, c2 = 7;
  const uint64_t s = b200_block_send(&st, &pairs[ops[0].pair], ops[0].slices, ops[0].n, 0, 0, &c1);
  const uint64_t r = b200_block_recv(&st, &pairs[ops[1].pair], ops[1].dst, ops[1].cap, 0, &c2);
  if (threadIdx.x == 0) {
    ops[0].ret = s;
    ops[0].calls = c1;
    ops[1].ret = r;
    ops[1].calls = c2;
  }
}

static void* kernel_for(uint32_t kinds) {
  switch (kinds) {
    case kSend: return (void*)bd_kernel<kSend>;
    case kRecv: return (void*)bd_kernel<kRecv>;
    case kSend | kRecv: return (void*)bd_kernel<kSend | kRecv>;
    default: return (void*)bd_kernel<kSend | kRecv | kWarp>;
  }
}
static const uint32_t kAllKinds[] = {kSend, kRecv, kSend | kRecv, kSend | kRecv | kWarp};

static cudaStream_t g_stream = nullptr;
static char g_err[256];

extern "C" const char* bd_error(void) { return g_err; }

static int set_err(cudaError_t e) {
  snprintf(g_err, sizeof g_err, "%s", cudaGetErrorString(e));
  return e == cudaSuccess ? 0 : -1;
}

// Load the module, allow the stages and create the stream now: while the library's service kernels are resident, the
// first launch of a kernel would wait for an idle device.
extern "C" int bd_prepare(void) {
  if (!g_stream && cudaStreamCreateWithFlags(&g_stream, cudaStreamNonBlocking) != cudaSuccess) return -1;
  cudaError_t e = cudaSuccess;
  for (uint32_t k : kAllKinds)
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(kernel_for(k), cudaFuncAttributeMaxDynamicSharedMemorySize, B200_BLOCK_SMEM_BYTES);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(bd_wrong_shape, cudaFuncAttributeMaxDynamicSharedMemorySize, B200_BLOCK_SMEM_BYTES);
  if (e != cudaSuccess) return set_err(e);
  bd_kernel<kSend><<<1, B200_BLOCK_THREADS, B200_BLOCK_SMEM_BYTES, g_stream>>>(nullptr, nullptr, nullptr, 0, 0, 0);
  bd_kernel<kRecv><<<1, B200_BLOCK_THREADS, B200_BLOCK_SMEM_BYTES, g_stream>>>(nullptr, nullptr, nullptr, 0, 0, 0);
  bd_kernel<kSend | kRecv><<<1, B200_BLOCK_THREADS, B200_BLOCK_SMEM_BYTES, g_stream>>>(nullptr, nullptr, nullptr, 0, 0,
                                                                                     0);
  bd_kernel<kSend | kRecv | kWarp><<<1, B200_BLOCK_THREADS, B200_BLOCK_SMEM_BYTES, g_stream>>>(nullptr, nullptr,
                                                                                             nullptr, 0, 0, 0);
  return set_err(cudaStreamSynchronize(g_stream));
}

// CTAs that can be resident at once with the stages they need
extern "C" int bd_max_resident(void) {
  int dev = 0, sms = 0, per_sm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bd_kernel<kSend | kRecv | kWarp>, B200_BLOCK_THREADS, B200_BLOCK_SMEM_BYTES) !=
      cudaSuccess)
    return -1;
  return per_sm * sms;
}

// pairs, ops, first: device or pinned (mapped) memory; ops and first must be host-readable too (pinned).  stream: NULL
// = the driver's own.  bd_launch returns once the kernel is queued (the host may then drive the other end), bd_wait
// once it has finished: 0 when it ran to its end (each op's `status` says whether it timed out), -1 on an error.  A
// launch with a streaming op, whose CTAs may wait for each other, is refused (-2) unless every CTA can be resident.
extern "C" int bd_launch(const void* pairs, void* ops, const uint32_t* first, int nlists, uint64_t budget_ns,
                         uint64_t max_iters, void* stream) {
  if (!g_stream && bd_prepare() != 0) return -1;
  const bd_op* o = static_cast<const bd_op*>(ops);
  bool waits = false;
  uint32_t kinds = 0;
  for (uint32_t i = 0; nlists > 0 && i < first[nlists]; i++) {
    const uint32_t k = o[i].kind;
    waits |= nlists > 1 && (k == BD_STREAM_SEND || k == BD_STREAM_RECV);
    kinds |= k == BD_SEND || k == BD_STREAM_SEND ? kSend : k == BD_RECV || k == BD_STREAM_RECV ? kRecv : kWarp;
  }
  if (waits && bd_max_resident() < nlists) {
    snprintf(g_err, sizeof g_err, "%d CTAs that wait for each other, but only %d can be resident", nlists,
             bd_max_resident());
    return -2;
  }
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : g_stream;
  const b200_dev_pair* pp = static_cast<const b200_dev_pair*>(pairs);
  bd_op* op = static_cast<bd_op*>(ops);
  void* args[] = {&pp, &op, &first, &nlists, &budget_ns, &max_iters};
  const cudaError_t e = cudaLaunchKernel(kernel_for(kinds), dim3(nlists), dim3(B200_BLOCK_THREADS), args,
                                         B200_BLOCK_SMEM_BYTES, s);
  if (e != cudaSuccess) return set_err(e);
  return set_err(cudaGetLastError());
}
extern "C" int bd_wait(void* stream) {
  return set_err(cudaStreamSynchronize(stream ? static_cast<cudaStream_t>(stream) : g_stream));
}

// ops[0] = a Send, ops[1] = a Recv, both run by a CTA of `threads` threads (not B200_BLOCK_THREADS: refused)
extern "C" int bd_wrong_shape_run(const void* pairs, void* ops, int threads) {
  if (!g_stream && bd_prepare() != 0) return -1;
  bd_wrong_shape<<<1, threads, B200_BLOCK_SMEM_BYTES, g_stream>>>(static_cast<const b200_dev_pair*>(pairs),
                                                                  static_cast<bd_op*>(ops));
  if (set_err(cudaGetLastError()) != 0) return -1;
  return set_err(cudaStreamSynchronize(g_stream));
}
