// device_cluster.cu -- TEST INFRASTRUCTURE: a user kernel that drives pairs through the cluster calls of the public
// block-level device API (include/b200_device_block.cuh), and ctypes-callable launchers for it.  Built by
// device_cluster.mk for sm_90a against the public header only.
//
// One launch runs `nlists` lists of ops, one thread-block cluster of K CTAs (B200_BLOCK_THREADS threads each) per list;
// list w is ops[first[w] .. first[w + 1]) and runs on cluster w.  K = 1 is a launch without clusters.  Lists run
// concurrently (e.g. one sender cluster and one receiver cluster per connection).  Every loop is bounded by an
// iteration cap and a %globaltimer deadline: an op that hits either reports CD_TIMEOUT and the rest of its list is
// skipped.  Nothing waits without bound, and a launch whose clusters wait for each other is refused unless they can all
// be resident at once (cudaOccupancyMaxActiveClusters).
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200_device_block.cuh"

namespace cg = cooperative_groups;

enum : uint32_t {
  CD_SEND = 1,         // one b200_cluster_send with the op's flags (ONE_CALL: one Send call; UNTIL_BLOCKED: rdma_flush)
  CD_RECV = 2,         // one b200_cluster_recv with the op's flags
  CD_STREAM_SEND = 3,  // send the whole slice list: UNTIL_BLOCKED cluster calls, retried while there is no credit
  CD_STREAM_RECV = 4,  // receive exactly n bytes into dst: UNTIL_BLOCKED cluster calls, retried while nothing is complete
  CD_WARP_SEND = 5,    // one b200_warp_send from warp 0 of CTA rank 0 (the other threads wait at a cluster barrier)
  CD_WARP_RECV = 6,    // one b200_warp_recv from warp 0 of CTA rank 0
  CD_BLOCK_SEND = 7,   // one b200_block_send with the op's flags from CTA rank 0
  CD_BLOCK_RECV = 8,   // one b200_block_recv with the op's flags from CTA rank 0
};
enum : uint32_t { CD_OK = 0, CD_TIMEOUT = 1 };

struct cd_op {
  uint32_t kind, pair;  // pair: index into the handle array
  const b200_slice* slices;
  uint64_t n, byte_idx;  // send: slice count / byte_idx.  stream_recv: bytes
  uint8_t* dst;
  uint64_t cap;
  int32_t flags;  // CD_SEND / CD_RECV / CD_BLOCK_*: passed to the call as it is
  uint32_t _pad0;
  uint64_t ret, calls;  // results
  uint32_t status, _pad;
};
static_assert(sizeof(cd_op) == 80, "cd_op layout is mirrored in tests/device_cluster_lib.py");

__device__ __forceinline__ uint64_t now_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

struct Bound {  // cluster-uniform: thread 0 of rank 0 reads the clock, every CTA takes its answer
  uint64_t deadline, left;
  uint32_t* late;  // a __shared__ word of this CTA
  __device__ bool spent(cg::cluster_group& cl) {
    if (cl.block_rank() == 0 && threadIdx.x == 0) *late = now_ns() > deadline;
    cl.sync();
    const uint32_t l = *cl.map_shared_rank(late, 0);
    cl.sync();  // rank 0 does not rewrite the word before every CTA has read it
    return l || left-- == 0;
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

// kKinds: which calls the launch's lists hold.  The launcher picks the instantiation with just those, so that a launch
// of cluster sends only compiles the Send body alone (the registers the CPU test checks), one of receives the Recv body.
enum : uint32_t { kSend = 1, kRecv = 2, kOther = 4 };
template <uint32_t kKinds>
__global__ void __launch_bounds__(B200_BLOCK_THREADS, 2)
cd_kernel(const b200_dev_pair* pairs, cd_op* ops, const uint32_t* first, int nlists, uint64_t budget_ns,
          uint64_t max_iters) {
  __shared__ b200_block st;
  __shared__ uint64_t s_t0, s_ret, s_calls;
  __shared__ uint32_t s_late;
  cg::cluster_group cl = cg::this_cluster();
  const uint32_t rank = cl.block_rank();
  const int w = (int)(blockIdx.x / cl.num_blocks());  // every CTA of a cluster has the same list
  if (w >= nlists) return;
  b200_block_init(&st);
  if (threadIdx.x == 0) s_t0 = now_ns();
  cl.sync();
  Bound b{*cl.map_shared_rank(&s_t0, 0) + budget_ns, max_iters, &s_late};
  for (uint32_t i = first[w]; i < first[w + 1]; i++) {
    cd_op& o = ops[i];
    const b200_dev_pair* h = &pairs[o.pair];
    const uint32_t kind = o.kind;
    uint64_t ret = 0, calls = 0;
    uint32_t status = CD_OK;
    if ((kKinds & kSend) && (kind == CD_SEND || kind == CD_STREAM_SEND)) {  // one call site for both
      const bool stream = kind == CD_STREAM_SEND;
      uint64_t idx = 0, bidx = o.byte_idx;
      while (idx < o.n) {
        uint64_t c = 0;
        const uint64_t sent = b200_cluster_send(&st, h, o.slices + idx, o.n - idx, bidx,
                                                stream ? B200_BATCH_UNTIL_BLOCKED : o.flags, &c);
        ret += sent;
        calls += c;
        if (!stream) break;
        if (sent) advance(o.slices, idx, bidx, sent);
        else if (b.spent(cl)) {
          status = CD_TIMEOUT;
          break;
        }
      }
    } else if ((kKinds & kRecv) && (kind == CD_RECV || kind == CD_STREAM_RECV)) {
      const bool stream = kind == CD_STREAM_RECV;
      const uint64_t want = stream ? o.n : o.cap;
      do {
        uint64_t c = 0;
        const uint64_t got =
            b200_cluster_recv(&st, h, o.dst + ret, want - ret, stream ? B200_BATCH_UNTIL_BLOCKED : o.flags, &c);
        ret += got;
        calls += c;
        if (!stream) break;
        if (!got && b.spent(cl)) {
          status = CD_TIMEOUT;
          break;
        }
      } while (ret < want);
    } else if ((kKinds & kOther) && kind >= CD_WARP_SEND && kind <= CD_BLOCK_RECV) {
      if (rank == 0) {  // the other CTAs wait at the barrier below
        if (kind == CD_BLOCK_SEND || kind == CD_BLOCK_RECV) {
          uint64_t c = 0;
          const uint64_t r = kind == CD_BLOCK_SEND ? b200_block_send(&st, h, o.slices, o.n, o.byte_idx, o.flags, &c)
                                                   : b200_block_recv(&st, h, o.dst, o.cap, o.flags, &c);
          if (threadIdx.x == 0) {
            s_ret = r;
            s_calls = c;
          }
        } else if (threadIdx.x < 32) {
          const uint64_t r = kind == CD_WARP_SEND ? b200_warp_send(h, o.slices, (uint32_t)o.n, o.byte_idx)
                                                  : b200_warp_recv(h, o.dst, o.cap);
          if (threadIdx.x == 0) {
            s_ret = r;
            s_calls = r != 0;
          }
        }
      }
      cl.sync();
      ret = s_ret;  // (rank 0's: the only one written to ops)
      calls = s_calls;
    } else {
      status = 2;
    }
    if (rank == 0 && threadIdx.x == 0) {
      o.ret = ret;
      o.calls = calls;
      o.status = status;
    }
    cl.sync();
    if (status != CD_OK) break;
  }
}

// A kernel for shapes the calls refuse: every CTA makes a cluster Send, then a cluster Recv.  Block (0, 0) writes
// ret = the answers and calls.
__global__ void cd_wrong_shape(const b200_dev_pair* pairs, cd_op* ops) {
  __shared__ b200_block st;
  b200_block_init(&st);
  uint64_t c1 = 7, c2 = 7;
  const uint64_t s = b200_cluster_send(&st, &pairs[ops[0].pair], ops[0].slices, ops[0].n, 0, 0, &c1);
  const uint64_t r = b200_cluster_recv(&st, &pairs[ops[1].pair], ops[1].dst, ops[1].cap, 0, &c2);
  if (threadIdx.x == 0 && blockIdx.x == 0 && blockIdx.y == 0) {
    ops[0].ret = s;
    ops[0].calls = c1;
    ops[1].ret = r;
    ops[1].calls = c2;
  }
}

static void* kernel_for(uint32_t kinds) {
  switch (kinds) {
    case kSend: return (void*)cd_kernel<kSend>;
    case kRecv: return (void*)cd_kernel<kRecv>;
    case kSend | kRecv: return (void*)cd_kernel<kSend | kRecv>;
    default: return (void*)cd_kernel<kSend | kRecv | kOther>;
  }
}
static const uint32_t kAllKinds[] = {kSend, kRecv, kSend | kRecv, kSend | kRecv | kOther};

static cudaStream_t g_stream = nullptr;
static char g_err[256];

extern "C" const char* cd_error(void) { return g_err; }

static int set_err(cudaError_t e) {
  snprintf(g_err, sizeof g_err, "%s", cudaGetErrorString(e));
  return e == cudaSuccess ? 0 : -1;
}

// grid = nclusters * k CTAs in clusters of k x 1 x 1; k = 1: no cluster attribute
static cudaLaunchConfig_t config(int nclusters, int k, cudaStream_t s, cudaLaunchAttribute* attr) {
  cudaLaunchConfig_t c = {};
  c.gridDim = dim3((unsigned)(nclusters * k));
  c.blockDim = dim3(B200_BLOCK_THREADS);
  c.dynamicSmemBytes = B200_BLOCK_SMEM_BYTES;
  c.stream = s;
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)k;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  c.attrs = attr;
  c.numAttrs = k > 1 ? 1 : 0;
  return c;
}

// Load the module, allow the stages and clusters of up to 16 CTAs and create the stream now: while the library's
// service kernels are resident, the first launch of a kernel would wait for an idle device.
extern "C" int cd_prepare(void) {
  if (!g_stream && cudaStreamCreateWithFlags(&g_stream, cudaStreamNonBlocking) != cudaSuccess) return -1;
  cudaError_t e = cudaSuccess;
  for (uint32_t k : kAllKinds) {
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(kernel_for(k), cudaFuncAttributeMaxDynamicSharedMemorySize, B200_BLOCK_SMEM_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(kernel_for(k), cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  }
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(cd_wrong_shape, cudaFuncAttributeMaxDynamicSharedMemorySize, B200_BLOCK_SMEM_BYTES);
  if (e != cudaSuccess) return set_err(e);
  for (uint32_t k : kAllKinds) {
    const b200_dev_pair* pp = nullptr;
    cd_op* op = nullptr;
    const uint32_t* first = nullptr;
    int n = 0;
    uint64_t z = 0;
    void* args[] = {&pp, &op, &first, &n, &z, &z};
    e = cudaLaunchKernel(kernel_for(k), dim3(1), dim3(B200_BLOCK_THREADS), args, B200_BLOCK_SMEM_BYTES, g_stream);
    if (e != cudaSuccess) return set_err(e);
  }
  return set_err(cudaStreamSynchronize(g_stream));
}

// clusters of k CTAs that can be resident at once with the stages they need (0: the device cannot place one)
extern "C" int cd_max_clusters(int k) {
  if (!g_stream && cd_prepare() != 0) return -1;
  cudaLaunchAttribute attr[1];
  cudaLaunchConfig_t c = config(1, k, g_stream, attr);
  c.numAttrs = 1;  // (k = 1 counts clusters of one CTA)
  int n = 0;
  const cudaError_t e = cudaOccupancyMaxActiveClusters(&n, kernel_for(kSend | kRecv | kOther), &c);
  if (e != cudaSuccess) {
    set_err(e);
    return 0;
  }
  return n;
}

// pairs, ops, first: device or pinned (mapped) memory; ops and first must be host-readable too (pinned).  stream: NULL
// = the driver's own.  cd_launch returns once the kernel is queued (the host may then drive the other end), cd_wait
// once it has finished: 0 when it ran to its end (each op's `status` says whether it timed out), -1 on an error.  A
// launch with a streaming op, whose clusters may wait for each other, is refused (-2) unless every cluster can be
// resident.
extern "C" int cd_launch(const void* pairs, void* ops, const uint32_t* first, int nlists, int k, uint64_t budget_ns,
                         uint64_t max_iters, void* stream) {
  if (!g_stream && cd_prepare() != 0) return -1;
  if (k < 1 || k > 16) {
    snprintf(g_err, sizeof g_err, "cluster size %d", k);
    return -1;
  }
  const cd_op* o = static_cast<const cd_op*>(ops);
  bool waits = false;
  uint32_t kinds = 0;
  for (uint32_t i = 0; nlists > 0 && i < first[nlists]; i++) {
    const uint32_t kd = o[i].kind;
    waits |= nlists > 1 && (kd == CD_STREAM_SEND || kd == CD_STREAM_RECV);
    kinds |= kd == CD_SEND || kd == CD_STREAM_SEND ? kSend : kd == CD_RECV || kd == CD_STREAM_RECV ? kRecv : kOther;
  }
  if (waits && cd_max_clusters(k) < nlists) {
    snprintf(g_err, sizeof g_err, "%d clusters of %d CTAs that wait for each other, but only %d can be resident",
             nlists, k, cd_max_clusters(k));
    return -2;
  }
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : g_stream;
  const b200_dev_pair* pp = static_cast<const b200_dev_pair*>(pairs);
  cd_op* op = static_cast<cd_op*>(ops);
  void* args[] = {&pp, &op, &first, &nlists, &budget_ns, &max_iters};
  cudaLaunchAttribute attr[1];
  const cudaLaunchConfig_t c = config(nlists > 0 ? nlists : 1, k, s, attr);
  const cudaError_t e = cudaLaunchKernelExC(&c, kernel_for(kinds), args);
  if (e != cudaSuccess) return set_err(e);
  return set_err(cudaGetLastError());
}
extern "C" int cd_wait(void* stream) {
  return set_err(cudaStreamSynchronize(stream ? static_cast<cudaStream_t>(stream) : g_stream));
}

// ops[0] = a Send, ops[1] = a Recv, both run by a grid of gx x gy CTAs of `threads` threads in clusters of cx x cy
// (cx * cy = 1: no cluster attribute)
extern "C" int cd_wrong_shape_run(const void* pairs, void* ops, int threads, int gx, int gy, int cx, int cy) {
  if (!g_stream && cd_prepare() != 0) return -1;
  const b200_dev_pair* pp = static_cast<const b200_dev_pair*>(pairs);
  cd_op* op = static_cast<cd_op*>(ops);
  void* args[] = {&pp, &op};
  cudaLaunchAttribute attr[1];
  cudaLaunchConfig_t c = config(1, 1, g_stream, attr);
  c.gridDim = dim3((unsigned)gx, (unsigned)gy);
  c.blockDim = dim3((unsigned)threads);
  attr[0].val.clusterDim.x = (unsigned)cx;
  attr[0].val.clusterDim.y = (unsigned)cy;
  c.numAttrs = cx * cy > 1 ? 1 : 0;
  if (set_err(cudaLaunchKernelExC(&c, (void*)cd_wrong_shape, args)) != 0) return -1;
  return set_err(cudaStreamSynchronize(g_stream));
}
