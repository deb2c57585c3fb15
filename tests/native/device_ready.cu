// device_ready.cu -- TEST INFRASTRUCTURE: user kernels that consume a device ready set (include/b200_device.cuh:
// b200_warp_ready_take / b200_warp_ready_rearm) and drive peers with the device calls, and ctypes-callable launchers.
// Built by device_ready.mk for sm_90a against the public headers only.
//
//   dr_drain_kernel  the consumer: take, serve each key (Recv until nothing is complete, Send what the member still
//                    owes, Disconnect a member whose peer left), rearm; until the queue is empty, or, with a stop flag,
//                    until the host raises it
//   dr_send_kernel   one b200_warp_send per warp (device warp producers)
//   dr_block_kernel  one b200_block_send per CTA (device block producers)
//   dr_disc_kernel   one b200_warp_disconnect per warp
//   dr_poll_kernel   ready members by b200_warp_poll plus the pending-write rule
//   dr_serve_kernel  one server warp (ready set or b200_warp_poll scan) and one client warp per active connection
//   dr_cost_kernel   ns per empty take and per b200_warp_poll scan of n idle ends, alternating
// Every loop is bounded by an iteration cap; launches whose warps wait for each other check co-residency first.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200_device_block.cuh"

__device__ __forceinline__ uint64_t now_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// ---- the consumer

struct dr_drain {
  const b200_dev_ready_set* set;
  const b200_dev_pair* members;  // by key
  uint32_t n, _pad0;
  uint8_t* rbuf;                 // n * rcap: what each member received, in order
  uint64_t rcap;
  uint64_t* got;                 // n: bytes received so far
  const uint8_t* sbuf;           // n * scap: what each member owes its peer
  uint64_t scap;
  uint64_t* owe;                 // n: bytes of sbuf to send in all
  uint64_t* sent;                // n: bytes sent so far
  uint32_t* taken;               // n: returned by take (this launch)
  uint32_t* kept;                // n: returned by rearm (this launch)
  uint32_t* idle;                // n: rearm returned 0 (this launch): a later take of the key is a second entry
  uint32_t* closed;              // n: the consumer disconnected the member after its peer left
  uint32_t* keys;                // scratch, >= n
  uint32_t* out;                 // [0] status (0 ok, 1 iteration cap), [1] second entries, [2] foreign keys, [3] takes
  volatile uint32_t* stop;       // NULL: return once a take finds nothing; else run until *stop != 0
  uint64_t max_iters;
};
static_assert(sizeof(dr_drain) == 144, "dr_drain layout is mirrored in tests/device_ready_lib.py");

__device__ void serve_member(const dr_drain& d, uint32_t k, uint64_t& iters) {
  const uint32_t lane = lane_id();
  const b200_dev_pair* h = &d.members[k];
  for (;;) {
    uint64_t g = d.got[k];
    for (;;) {
      const uint64_t r = b200_warp_recv(h, d.rbuf + k * d.rcap + g, d.rcap - g);
      if (r == 0) break;
      g += r;
    }
    uint64_t s = d.sent[k];
    if (s < d.owe[k]) {
      const b200_slice sl{d.sbuf + k * d.scap + s, d.owe[k] - s};
      s += b200_warp_send(h, &sl, 1, 0);
    }
    if (lane == 0) {
      d.got[k] = g;
      d.sent[k] = s;
    }
    __syncwarp();
    if (b200_warp_status(h) == B200_HALF_CLOSED) {  // the peer left: close the member, it stays READABLE otherwise
      b200_warp_disconnect(h);
      if (lane == 0) d.closed[k] = 1;
      break;
    }
    const uint32_t ev = b200_warp_ready_rearm(d.set, h);
    if (ev == 0) {
      if (lane == 0) d.idle[k] = 1;
      break;
    }
    if (lane == 0) d.kept[k]++;
    if (++iters >= d.max_iters) break;
  }
  __syncwarp();
}

__global__ void dr_drain_kernel(dr_drain d) {
  if (d.n == 0) return;
  const uint32_t lane = lane_id();
  uint64_t iters = 0;
  uint32_t dups = 0, foreign = 0, takes = 0;
  for (;;) {
    const uint32_t c = b200_warp_ready_take(d.set, d.keys, d.n);
    takes += c;
    if (c == 0) {
      if (d.stop == nullptr || *d.stop != 0) break;
      if (++iters >= d.max_iters) break;
      __nanosleep(200);
      continue;
    }
    for (uint32_t j = 0; j < c; j++) {
      const uint32_t k = d.keys[j];
      if (k >= d.n) {
        foreign++;
        continue;
      }
      if (d.idle[k]) dups++;  // (the producers have finished: nothing could have queued it after that rearm)
      if (lane == 0) d.taken[k]++;
      __syncwarp();
      if (d.closed[k]) continue;  // a stale entry of a member the consumer closed
      serve_member(d, k, iters);
    }
    if (iters >= d.max_iters) break;
  }
  if (lane == 0) {
    d.out[0] = iters >= d.max_iters ? 1 : 0;
    d.out[1] = dups;
    d.out[2] = foreign;
    d.out[3] = takes;
  }
}

// ---- device producers

struct dr_op {
  const b200_dev_pair* h;
  const b200_slice* slices;
  uint64_t n;
  uint64_t ret;
};
static_assert(sizeof(dr_op) == 32, "dr_op layout is mirrored in tests/device_ready_lib.py");

__global__ void dr_send_kernel(dr_op* ops, int nops) {
  const int w = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (w >= nops) return;
  const uint64_t r = b200_warp_send(ops[w].h, ops[w].slices, (uint32_t)ops[w].n, 0);
  if (lane_id() == 0) ops[w].ret = r;
}

__global__ void __launch_bounds__(B200_BLOCK_THREADS, 2) dr_block_kernel(dr_op* ops, int nops) {
  __shared__ b200_block st;
  if ((int)blockIdx.x >= nops) return;
  b200_block_init(&st);
  uint64_t calls = 0;
  const uint64_t r = b200_block_send(&st, ops[blockIdx.x].h, ops[blockIdx.x].slices, ops[blockIdx.x].n, 0, 0, &calls);
  if (threadIdx.x == 0) ops[blockIdx.x].ret = r;
}

__global__ void dr_disc_kernel(dr_op* ops, int nops) {
  const int w = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (w >= nops) return;
  const int r = b200_warp_disconnect(ops[w].h);
  if (lane_id() == 0) ops[w].ret = (uint64_t)r;
}

// ready[i] = 1 when member i is READY: READABLE by b200_warp_poll, or a pending write with credit for one frame
__global__ void dr_poll_kernel(const b200_dev_pair* h, uint32_t n, uint32_t* events, uint32_t* ready) {
  b200_warp_poll(h, n, events, nullptr);
  __syncwarp();
  for (uint32_t i = lane_id(); i < n; i += 32) {
    uint32_t r = (events[i] & B200_EV_READABLE) != 0;
    if (!r && b200::pair_status(reinterpret_cast<b200::PairDev*>(h[i].table), h[i].slot) == B200_CONNECTED &&
        *(volatile uint32_t*)&reinterpret_cast<b200::PairDev*>(h[i].table)[h[i].slot].partial_write) {
      const b200::PairDev& P = reinterpret_cast<b200::PairDev*>(h[i].table)[h[i].slot];
      const uint64_t cap = P.cap;
      const uint64_t fr = b200::free_size(cap, *(volatile uint64_t*)&P.credit_head, *(volatile uint64_t*)&P.remote_tail);
      r = b200::calc_writable(fr < cap / 2 ? fr : cap / 2) != 0;
    }
    ready[i] = r;
  }
}

// ---- the server: ready set (set != NULL) or scan, and the clients

struct dr_serve {
  const b200_dev_ready_set* set;
  const b200_dev_pair* srv;  // n server ends (key = index)
  const b200_dev_pair* cli;  // a client ends: client i talks to server end i
  uint32_t n, a, rounds, msg;
  uint8_t* sbuf;             // n * msg
  uint8_t* cbuf;             // a * 2 * msg
  uint32_t* state;           // 3 * n, zeroed: request bytes so far, replies sent, keys / ready list
  uint64_t* out;             // per client i: out[2 i ..] = mismatched replies, rounds done; out[2 a ..] = server
                             // status, replies, takes or scans, empty takes or scans, elapsed ns
  uint64_t max_iters;
};
static_assert(sizeof(dr_serve) == 80, "dr_serve layout is mirrored in tests/device_ready_lib.py");

__device__ __forceinline__ uint64_t pattern_word(uint32_t conn, uint32_t round, uint32_t j) {
  return ((uint64_t)conn << 48) ^ ((uint64_t)round << 24) ^ ((uint64_t)j * 0x9E3779B97F4A7C15ull);
}

// Recv what is there; a whole request is echoed.  Returns false when the echo ran out of its iteration budget.
__device__ bool serve_one(const dr_serve& s, uint32_t i, uint64_t& replies, uint64_t& iters) {
  const uint32_t lane = lane_id();
  const b200_dev_pair* h = &s.srv[i];
  uint8_t* req = s.sbuf + (uint64_t)i * s.msg;
  uint32_t g = s.state[i];
  for (;;) {
    const uint64_t r = b200_warp_recv(h, req + g, s.msg - g);
    if (r == 0) break;
    g += (uint32_t)r;
    if (g == s.msg) {
      const b200_slice back{req, s.msg};
      uint64_t sent = 0;
      while (sent < s.msg) {
        const b200_slice rest{req + sent, s.msg - sent};
        sent += b200_warp_send(h, &rest, 1, 0);
        if (++iters >= s.max_iters) return false;
      }
      (void)back;
      g = 0;
      replies++;
    }
  }
  if (lane == 0) s.state[i] = g;
  __syncwarp();
  return true;
}

__device__ void server(const dr_serve& s) {
  uint32_t* keys = s.state + 2 * s.n;
  const uint64_t want = (uint64_t)s.a * s.rounds;
  uint64_t replies = 0, iters = 0, passes = 0, empty = 0, t0 = 0;
  if (lane_id() == 0) t0 = now_ns();
  uint32_t status = 0;
  while (replies < want && status == 0) {
    const uint32_t c = s.set ? b200_warp_ready_take(s.set, keys, s.n) : b200_warp_poll(s.srv, s.n, nullptr, keys);
    passes++;
    if (c == 0) empty++;
    for (uint32_t k = 0; k < c && status == 0; k++) {
      const uint32_t i = keys[k];
      for (;;) {
        if (!serve_one(s, i, replies, iters)) {
          status = 1;
          break;
        }
        if (!s.set || b200_warp_ready_rearm(s.set, &s.srv[i]) == 0) break;
      }
    }
    if (++iters >= s.max_iters) status = 1;
  }
  if (lane_id() == 0) {
    uint64_t* o = s.out + 2ull * s.a;
    o[0] = status;
    o[1] = replies;
    o[2] = passes;
    o[3] = empty;
    o[4] = now_ns() - t0;
  }
}

__device__ void client(const dr_serve& s, uint32_t i) {
  const uint32_t lane = lane_id();
  const b200_dev_pair* h = &s.cli[i];
  uint8_t* req = s.cbuf + 2ull * i * s.msg;
  uint8_t* rep = req + s.msg;
  const uint32_t words = s.msg / 8;
  uint64_t bad = 0, iters = 0;
  uint32_t r = 0;
  for (; r < s.rounds; r++) {
    for (uint32_t j = lane; j < words; j += 32) reinterpret_cast<uint64_t*>(req)[j] = pattern_word(i, r, j);
    __syncwarp();
    uint64_t sent = 0, got = 0;
    while (sent < s.msg && iters < s.max_iters) {
      const b200_slice rest{req + sent, s.msg - sent};
      sent += b200_warp_send(h, &rest, 1, 0);
      iters++;
    }
    while (got < s.msg && iters < s.max_iters) {
      got += b200_warp_recv(h, rep + got, s.msg - got);
      iters++;
    }
    if (got < s.msg) break;
    bool diff = false;
    for (uint32_t j = lane; j < words; j += 32) diff |= reinterpret_cast<const uint64_t*>(rep)[j] != pattern_word(i, r, j);
    bad += __any_sync(0xffffffffu, diff) ? 1 : 0;
  }
  if (lane == 0) {
    s.out[2 * i + 0] = bad;
    s.out[2 * i + 1] = r;
  }
}

__global__ void __launch_bounds__(128) dr_serve_kernel(dr_serve s) {
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (s.n == 0) return;
  if (w == 0) server(s);
  else if (w <= s.a) client(s, w - 1);
}

// ---- cost of an empty take and of a scan of n idle ends, alternating: times[2 k] / times[2 k + 1] = ns per call
__global__ void dr_cost_kernel(const b200_dev_ready_set* set, const b200_dev_pair* h, uint32_t n, uint32_t* scratch,
                               uint32_t batches, uint32_t per, uint64_t* times) {
  uint32_t sink = 0;
  for (uint32_t k = 0; k < batches; k++) {
    uint64_t t0 = 0;
    if (lane_id() == 0) t0 = now_ns();
    for (uint32_t j = 0; j < per; j++) sink += b200_warp_ready_take(set, scratch, n);
    if (lane_id() == 0) times[2 * k] = (now_ns() - t0) / per;
    if (lane_id() == 0) t0 = now_ns();
    for (uint32_t j = 0; j < per; j++) sink += b200_warp_poll(h, n, nullptr, scratch);
    if (lane_id() == 0) times[2 * k + 1] = (now_ns() - t0) / per;
  }
  if (lane_id() == 0 && sink == 0xffffffffu) times[0] = 0;  // (keeps the calls)
}

static cudaStream_t g_stream = nullptr;
static char g_err[256];

extern "C" const char* dr_error(void) { return g_err; }

static int fin(cudaError_t e) {
  snprintf(g_err, sizeof g_err, "%s", cudaGetErrorString(e));
  return e == cudaSuccess ? 0 : -1;
}

// Load the module and create the stream now: while the library's service kernels are resident, the first launch of
// a kernel would wait for an idle device.  These launches have nothing to do and touch no memory.
extern "C" int dr_prepare(void) {
  if (!g_stream && cudaStreamCreateWithFlags(&g_stream, cudaStreamNonBlocking) != cudaSuccess) return -1;
  if (fin(cudaFuncSetAttribute(dr_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, B200_BLOCK_SMEM_BYTES)))
    return -1;
  dr_drain d{};
  dr_drain_kernel<<<1, 32, 0, g_stream>>>(d);
  dr_send_kernel<<<1, 32, 0, g_stream>>>(nullptr, 0);
  dr_block_kernel<<<1, B200_BLOCK_THREADS, B200_BLOCK_SMEM_BYTES, g_stream>>>(nullptr, 0);
  dr_disc_kernel<<<1, 32, 0, g_stream>>>(nullptr, 0);
  dr_poll_kernel<<<1, 32, 0, g_stream>>>(nullptr, 0, nullptr, nullptr);
  dr_serve s{};
  dr_serve_kernel<<<1, 32, 0, g_stream>>>(s);
  dr_cost_kernel<<<1, 32, 0, g_stream>>>(nullptr, nullptr, 0, nullptr, 0, 0, nullptr);
  return fin(cudaStreamSynchronize(g_stream));
}

extern "C" int dr_wait(void) { return fin(cudaStreamSynchronize(g_stream)); }

// queued when this returns (a consumer with a stop flag runs until the host raises it): dr_wait() for the end
extern "C" int dr_drain_launch(const dr_drain* d) {
  if (!g_stream && dr_prepare() != 0) return -1;
  dr_drain_kernel<<<1, 32, 0, g_stream>>>(*d);
  return fin(cudaGetLastError());
}

// kind 0: warp Send, 1: block Send, 2: warp Disconnect; synchronous
extern "C" int dr_ops(int kind, dr_op* ops, int nops) {
  if (!g_stream && dr_prepare() != 0) return -1;
  if (nops <= 0) return 0;
  if (kind == 0) dr_send_kernel<<<(nops + 3) / 4, 128, 0, g_stream>>>(ops, nops);
  else if (kind == 1) dr_block_kernel<<<nops, B200_BLOCK_THREADS, B200_BLOCK_SMEM_BYTES, g_stream>>>(ops, nops);
  else dr_disc_kernel<<<(nops + 3) / 4, 128, 0, g_stream>>>(ops, nops);
  if (fin(cudaGetLastError())) return -1;
  return dr_wait();
}

extern "C" int dr_poll(const void* h, uint32_t n, uint32_t* events, uint32_t* ready) {
  if (!g_stream && dr_prepare() != 0) return -1;
  dr_poll_kernel<<<1, 32, 0, g_stream>>>(static_cast<const b200_dev_pair*>(h), n, events, ready);
  if (fin(cudaGetLastError())) return -1;
  return dr_wait();
}

// -2: the warps would not all be resident at once (they wait for each other)
extern "C" int dr_serve_launch(const dr_serve* s) {
  if (!g_stream && dr_prepare() != 0) return -1;
  const uint32_t warps = 1 + s->a;
  const int threads = 128, blocks = (int)((warps * 32 + threads - 1) / threads);
  int dev = 0, sms = 0, per_sm = 0;
  if (fin(cudaGetDevice(&dev)) || fin(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)) ||
      fin(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, dr_serve_kernel, threads, 0)))
    return -1;
  if (per_sm * sms < blocks) {
    snprintf(g_err, sizeof g_err, "%d blocks of %d threads are not co-resident", blocks, threads);
    return -2;
  }
  dr_serve_kernel<<<blocks, threads, 0, g_stream>>>(*s);
  if (fin(cudaGetLastError())) return -1;
  return dr_wait();
}

extern "C" int dr_cost(const void* set, const void* h, uint32_t n, uint32_t* scratch, uint32_t batches, uint32_t per,
                       uint64_t* times) {
  if (!g_stream && dr_prepare() != 0) return -1;
  dr_cost_kernel<<<1, 32, 0, g_stream>>>(static_cast<const b200_dev_ready_set*>(set),
                                         static_cast<const b200_dev_pair*>(h), n, scratch, batches, per, times);
  if (fin(cudaGetLastError())) return -1;
  return dr_wait();
}
