// device_api.cu -- TEST INFRASTRUCTURE: a user kernel that drives pairs through the public device API
// (include/b200_device.cuh), and ctypes-callable launchers for it.  Built by device_api.mk for sm_90a against the
// public header only.
//
// One launch runs `nlists` lists of ops, one warp per list; list w is ops[first[w] .. first[w + 1]).  Ops of
// different lists run concurrently (e.g. one sender warp and one receiver warp per connection).  Every loop is
// bounded by an iteration cap and a %globaltimer deadline: an op that hits either reports DA_TIMEOUT and the rest
// of its list is skipped.  Nothing waits without bound.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200_device.cuh"

enum : uint32_t {
  DA_SEND = 1,         // one b200_warp_send
  DA_SEND_ALL = 2,     // rdma_flush loop: Send until it accepts nothing (orb_pair_send_all)
  DA_RECV = 3,         // one b200_warp_recv
  DA_RECV_DRAIN = 4,   // rdma_do_read loop: Recv until nothing more or dst full (orb_pair_recv_drain)
  DA_STREAM_SEND = 5,  // send the whole slice list, retrying while there is no credit
  DA_STREAM_RECV = 6,  // receive exactly n bytes into dst, retrying while nothing is complete
  DA_PING = 7,         // n rounds: send the slice list, receive the same number of bytes; times[i] = round trip (ns)
  DA_PONG = 8,         // n rounds: receive cap bytes into dst, send them back
  DA_READY = 9,        // ret = readable, calls = has_message | has_pending_writes << 1
};
enum : uint32_t { DA_OK = 0, DA_TIMEOUT = 1 };

struct da_op {
  uint32_t kind, pair;  // pair: index into the handle array
  const b200_slice* slices;
  uint64_t n, byte_idx;  // send: slice count / byte_idx.  stream_recv: bytes.  ping / pong: rounds (ping:
                         // byte_idx = slice count)
  uint8_t* dst;
  uint64_t cap;
  uint64_t* times;
  uint64_t ret, calls;  // results
  uint32_t status, _pad;
};
static_assert(sizeof(da_op) == 80, "da_op layout is mirrored in tests/device_lib.py");

__device__ __forceinline__ uint64_t now_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

struct Bound {  // warp-uniform: lane 0 reads the clock, every lane gets its answer
  uint64_t deadline, left;
  __device__ bool spent() {
    uint32_t late = 0;
    if ((threadIdx.x & 31) == 0) late = now_ns() > deadline;
    late = __shfl_sync(0xffffffffu, late, 0);
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

__device__ uint32_t stream_send(const b200_dev_pair* h, const b200_slice* s, uint64_t n, uint64_t bidx, Bound& b,
                                uint64_t& ret, uint64_t& calls) {
  uint64_t idx = 0;
  while (idx < n) {
    const uint64_t sent = b200_warp_send(h, s + idx, (uint32_t)(n - idx), bidx);
    if (sent) {
      ret += sent;
      calls++;
      advance(s, idx, bidx, sent);
    } else if (b.spent()) {
      return DA_TIMEOUT;
    }
  }
  return DA_OK;
}

__device__ uint32_t stream_recv(const b200_dev_pair* h, uint8_t* dst, uint64_t n, Bound& b, uint64_t& ret,
                                uint64_t& calls) {
  while (ret < n) {
    const uint64_t got = b200_warp_recv(h, dst + ret, n - ret);
    if (got) {
      ret += got;
      calls++;
    } else if (b.spent()) {
      return DA_TIMEOUT;
    }
  }
  return DA_OK;
}

__global__ void __launch_bounds__(128) da_kernel(const b200_dev_pair* pairs, da_op* ops, const uint32_t* first,
                                                 int nlists, uint64_t budget_ns, uint64_t max_iters) {
  const int w = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (w >= nlists) return;
  const uint32_t lane = threadIdx.x & 31;
  uint64_t t0 = 0;
  if (lane == 0) t0 = now_ns();
  t0 = __shfl_sync(0xffffffffu, t0, 0);
  Bound b{t0 + budget_ns, max_iters};
  for (uint32_t i = first[w]; i < first[w + 1]; i++) {
    da_op& o = ops[i];
    const b200_dev_pair* h = &pairs[o.pair];
    uint64_t ret = 0, calls = 0;
    uint32_t status = DA_OK;
    switch (o.kind) {
      case DA_SEND:
        ret = b200_warp_send(h, o.slices, (uint32_t)o.n, o.byte_idx);
        calls = ret != 0;
        break;
      case DA_SEND_ALL: {
        uint64_t idx = 0, bidx = o.byte_idx;
        while (idx < o.n) {
          const uint64_t sent = b200_warp_send(h, o.slices + idx, (uint32_t)(o.n - idx), bidx);
          if (sent == 0) break;
          ret += sent;
          calls++;
          advance(o.slices, idx, bidx, sent);
          if (b.spent()) {
            status = DA_TIMEOUT;
            break;
          }
        }
        break;
      }
      case DA_RECV:
        ret = b200_warp_recv(h, o.dst, o.cap);
        calls = ret != 0;
        break;
      case DA_RECV_DRAIN:
        while (ret < o.cap) {
          const uint64_t got = b200_warp_recv(h, o.dst + ret, o.cap - ret);
          if (got == 0) break;
          ret += got;
          calls++;
          if (b.spent()) {
            status = DA_TIMEOUT;
            break;
          }
        }
        break;
      case DA_STREAM_SEND:
        status = stream_send(h, o.slices, o.n, o.byte_idx, b, ret, calls);
        break;
      case DA_STREAM_RECV:
        status = stream_recv(h, o.dst, o.n, b, ret, calls);
        break;
      case DA_PING: {
        uint64_t bytes = 0;
        for (uint32_t k = 0; k < o.byte_idx; k++) bytes += o.slices[k].len;  // byte_idx = slice count here
        for (uint64_t r = 0; r < o.n && status == DA_OK; r++) {
          uint64_t s0 = 0, c = 0, got = 0;
          if (lane == 0) s0 = now_ns();
          status = stream_send(h, o.slices, o.byte_idx, 0, b, ret, c);
          if (status == DA_OK) status = stream_recv(h, o.dst, bytes, b, got, calls);
          if (lane == 0) o.times[r] = now_ns() - s0;
        }
        break;
      }
      case DA_PONG: {
        const b200_slice back{o.dst, o.cap};
        for (uint64_t r = 0; r < o.n && status == DA_OK; r++) {
          uint64_t got = 0, c = 0;
          status = stream_recv(h, o.dst, o.cap, b, got, calls);
          if (status == DA_OK) status = stream_send(h, &back, 1, 0, b, ret, c);
        }
        break;
      }
      case DA_READY:
        ret = b200_warp_readable(h);
        calls = (uint64_t)b200_warp_has_message(h) | (uint64_t)b200_warp_has_pending_writes(h) << 1;
        break;
      default:
        status = 2;
    }
    if (lane == 0) {
      o.ret = ret;
      o.calls = calls;
      o.status = status;
    }
    __syncwarp();
    if (status != DA_OK) break;
  }
}

static cudaStream_t g_stream = nullptr;
static char g_err[256];

extern "C" const char* da_error(void) { return g_err; }

// Load the module and create the stream now: while the library's service kernels are resident, the first launch of
// a kernel would wait for an idle device.
extern "C" int da_prepare(void) {
  if (!g_stream && cudaStreamCreateWithFlags(&g_stream, cudaStreamNonBlocking) != cudaSuccess) return -1;
  da_kernel<<<1, 32, 0, g_stream>>>(nullptr, nullptr, nullptr, 0, 0, 0);
  const cudaError_t e = cudaStreamSynchronize(g_stream);
  snprintf(g_err, sizeof g_err, "%s", cudaGetErrorString(e));
  return e == cudaSuccess ? 0 : -1;
}

// pairs, ops, first: device or pinned (mapped) memory.  da_launch returns once the kernel is queued (the host may
// then drive the other end), da_wait once it has finished: 0 when it ran to its end (each op's `status` says
// whether it timed out), -1 on a launch or execution error.  da_run = both.
extern "C" int da_launch(const void* pairs, void* ops, const uint32_t* first, int nlists, uint64_t budget_ns,
                         uint64_t max_iters) {
  if (!g_stream && da_prepare() != 0) return -1;
  const int threads = 128, warps = threads / 32;
  da_kernel<<<(nlists + warps - 1) / warps, threads, 0, g_stream>>>(
      static_cast<const b200_dev_pair*>(pairs), static_cast<da_op*>(ops), first, nlists, budget_ns, max_iters);
  const cudaError_t e = cudaGetLastError();
  snprintf(g_err, sizeof g_err, "%s", cudaGetErrorString(e));
  return e == cudaSuccess ? 0 : -1;
}
extern "C" int da_wait(void) {
  const cudaError_t e = cudaStreamSynchronize(g_stream);
  snprintf(g_err, sizeof g_err, "%s", cudaGetErrorString(e));
  return e == cudaSuccess ? 0 : -1;
}
extern "C" int da_run(const void* pairs, void* ops, const uint32_t* first, int nlists, uint64_t budget_ns,
                      uint64_t max_iters) {
  if (da_launch(pairs, ops, first, nlists, budget_ns, max_iters) != 0) return -1;
  return da_wait();
}
