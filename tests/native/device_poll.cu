// device_poll.cu -- TEST INFRASTRUCTURE: user kernels that run the poll loop of a BPEV server through the public device
// API (include/b200_device.cuh: b200_warp_poll / status / writable / disconnect beside Send and Recv), and
// ctypes-callable launchers for them.  Built by device_poll.mk for sm_90a against the public header only.
//
//   dp_kernel        lists of single ops, one warp per list (the parity tests)
//   dp_poll          one b200_warp_poll by one warp
//   dp_serve_kernel  a device server over n connections: one polling server warp (poll -> Recv -> Send, then
//                    Disconnect after the last round) or one pong warp per connection, and optionally one client
//                    warp per connection (round trips with distinct payloads, then wait for HALF_CLOSED)
//   dp_poll_time     ns per b200_warp_poll scan of n handles
// Every loop is bounded by an iteration cap and a %globaltimer deadline; launches whose warps wait for each other
// check first that all of them can be resident at once.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200_device.cuh"

enum : uint32_t {
  DP_SEND = 1,        // one b200_warp_send
  DP_SEND_ALL = 2,    // Send until it accepts nothing
  DP_RECV = 3,        // one b200_warp_recv
  DP_STATUS = 4,      // ret = b200_warp_status
  DP_WRITABLE = 5,    // ret = b200_warp_writable
  DP_DISCONNECT = 6,  // ret = b200_warp_disconnect
  DP_TORN = 7,        // a frame header of n payload bytes (stamped: the next stamp) at the end's remote tail in the
                      // peer's ring, through the handle's table row -- no payload, no footer, no cursor moves
  DP_STREAM_SEND = 8, // the whole slice list, retrying while there is no credit
  DP_STREAM_RECV = 9, // exactly n bytes into dst, retrying while nothing is complete
  DP_WAIT_EVENTS = 10,// b200_warp_poll of this one end until (events & n) != 0; ret = events
};
enum : uint32_t { DP_OK = 0, DP_TIMEOUT = 1 };

struct dp_op {
  uint32_t kind, pair;  // pair: index into the handle array
  const b200_slice* slices;
  uint64_t n, byte_idx;
  uint8_t* dst;
  uint64_t cap;
  uint64_t ret, calls;  // results
  uint32_t status, _pad;
};
static_assert(sizeof(dp_op) == 72, "dp_op layout is mirrored in tests/device_poll_lib.py");

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
__device__ __forceinline__ Bound make_bound(uint64_t budget_ns, uint64_t max_iters) {
  uint64_t t0 = 0;
  if ((threadIdx.x & 31) == 0) t0 = now_ns();
  t0 = __shfl_sync(0xffffffffu, t0, 0);
  return Bound{t0 + budget_ns, max_iters};
}

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

__device__ uint32_t stream_send(const b200_dev_pair* h, const b200_slice* s, uint64_t n, Bound& b, uint64_t& ret,
                                uint64_t& calls) {
  uint64_t idx = 0, bidx = 0;
  while (idx < n) {
    const uint64_t sent = b200_warp_send(h, s + idx, (uint32_t)(n - idx), bidx);
    if (sent) {
      ret += sent;
      calls++;
      advance(s, idx, bidx, sent);
    } else if (b.spent()) {
      return DP_TIMEOUT;
    }
  }
  return DP_OK;
}

__device__ uint32_t stream_recv(const b200_dev_pair* h, uint8_t* dst, uint64_t n, Bound& b, uint64_t& ret,
                                uint64_t& calls) {
  while (ret < n) {
    const uint64_t got = b200_warp_recv(h, dst + ret, n - ret);
    if (got) {
      ret += got;
      calls++;
    } else if (b.spent()) {
      return DP_TIMEOUT;
    }
  }
  return DP_OK;
}

// DP_TORN: what a sender's frame looks like between its header store and its footer store
__device__ void torn_header(const b200_dev_pair* h, uint64_t p) {
  b200::PairDev* table = reinterpret_cast<b200::PairDev*>(h->table);
  b200::PairDev* P = table + h->slot;
  const uint32_t st = (P->max_sge & b200::kSgeStamped) ? b200::stamp_of(b200::pair_seq(table, h->slot)->tx) : 0;
  if ((threadIdx.x & 31) == 0) {
    *reinterpret_cast<volatile uint64_t*>(P->peer_ring + P->remote_tail) = b200::frame_header(p, st);
    __threadfence_system();
  }
  __syncwarp();
}

__global__ void __launch_bounds__(128) dp_kernel(const b200_dev_pair* pairs, dp_op* ops, const uint32_t* first,
                                                 int nlists, uint64_t budget_ns, uint64_t max_iters) {
  const int w = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (w >= nlists) return;
  const uint32_t lane = threadIdx.x & 31;
  Bound b = make_bound(budget_ns, max_iters);
  for (uint32_t i = first[w]; i < first[w + 1]; i++) {
    dp_op& o = ops[i];
    const b200_dev_pair* h = &pairs[o.pair];
    uint64_t ret = 0, calls = 0;
    uint32_t status = DP_OK;
    switch (o.kind) {
      case DP_SEND:
        ret = b200_warp_send(h, o.slices, (uint32_t)o.n, o.byte_idx);
        calls = ret != 0;
        break;
      case DP_SEND_ALL: {
        uint64_t idx = 0, bidx = o.byte_idx;
        while (idx < o.n) {
          const uint64_t sent = b200_warp_send(h, o.slices + idx, (uint32_t)(o.n - idx), bidx);
          if (sent == 0) break;
          ret += sent;
          calls++;
          advance(o.slices, idx, bidx, sent);
          if (b.spent()) {
            status = DP_TIMEOUT;
            break;
          }
        }
        break;
      }
      case DP_RECV:
        ret = b200_warp_recv(h, o.dst, o.cap);
        calls = ret != 0;
        break;
      case DP_STATUS:
        ret = (uint64_t)b200_warp_status(h);
        break;
      case DP_WRITABLE:
        ret = b200_warp_writable(h);
        break;
      case DP_DISCONNECT:
        ret = (uint64_t)b200_warp_disconnect(h);
        break;
      case DP_TORN:
        torn_header(h, o.n);
        break;
      case DP_STREAM_SEND:
        status = stream_send(h, o.slices, o.n, b, ret, calls);
        break;
      case DP_STREAM_RECV:
        status = stream_recv(h, o.dst, o.n, b, ret, calls);
        break;
      case DP_WAIT_EVENTS: {  // dst: 4 bytes of scratch for the events word
        uint32_t ev = 0;
        for (;;) {
          b200_warp_poll(h, 1, reinterpret_cast<uint32_t*>(o.dst), nullptr);
          ev = *reinterpret_cast<volatile uint32_t*>(o.dst);
          if (ev & o.n) break;
          if (b.spent()) {
            status = DP_TIMEOUT;
            break;
          }
        }
        ret = ev;
        break;
      }
      default:
        status = 2;
    }
    if (lane == 0) {
      o.ret = ret;
      o.calls = calls;
      o.status = status;
    }
    __syncwarp();
    if (status != DP_OK) break;
  }
}

__global__ void dp_poll_kernel(const b200_dev_pair* handles, uint32_t n, uint32_t* events, uint32_t* ready,
                               uint32_t* count) {
  const uint32_t c = b200_warp_poll(handles, n, events, ready);
  if ((threadIdx.x & 31) == 0 && count) *count = c;
}

// ---- the device server

struct dp_serve {
  const b200_dev_pair* srv;  // n server ends
  const b200_dev_pair* cli;  // n client ends, or NULL (the clients are driven elsewhere)
  uint32_t n, rounds, msg, mode;  // mode 0: one polling server warp; 1: one pong warp per connection
  uint8_t* sbuf;    // n * msg: the server's request buffers (device)
  uint8_t* cbuf;    // n * 2 * msg: the clients' request and reply buffers (device)
  uint32_t* state;  // 3 * n, zeroed: bytes of the request so far, replies sent, poll's ready list
  uint64_t* times;  // n * rounds: the clients' round trips (ns)
  uint64_t* out;    // per client i: out[4 i ..] = status, mismatched replies, rounds done, last b200_warp_status;
                    // out[4 n ..] = server status, connections closed, scans, empty scans
  uint64_t budget_ns, max_iters;
};
static_assert(sizeof(dp_serve) == 88, "dp_serve layout is mirrored in tests/device_poll_lib.py");

__device__ __forceinline__ uint64_t pattern_word(uint32_t conn, uint32_t round, uint32_t j) {
  return ((uint64_t)conn << 48) ^ ((uint64_t)round << 24) ^ ((uint64_t)j * 0x9E3779B97F4A7C15ull);
}

__device__ void serve_polling(const dp_serve& s) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t* got = s.state;
  uint32_t* done = s.state + s.n;
  uint32_t* ready = s.state + 2 * s.n;
  Bound b = make_bound(s.budget_ns, s.max_iters);
  uint32_t closed = 0, status = DP_OK;
  uint64_t scans = 0, empty = 0;
  while (closed < s.n) {
    const uint32_t cnt = b200_warp_poll(s.srv, s.n, nullptr, ready);
    scans++;
    if (cnt == 0) {
      empty++;
      if (b.spent()) {
        status = DP_TIMEOUT;
        break;
      }
      continue;
    }
    for (uint32_t k = 0; k < cnt && status == DP_OK; k++) {
      const uint32_t i = ready[k];
      const b200_dev_pair* h = &s.srv[i];
      uint8_t* req = s.sbuf + (uint64_t)i * s.msg;
      uint32_t g = got[i];
      const uint64_t r = b200_warp_recv(h, req + g, s.msg - g);  // 0: a header without its footer yet, or credit
      g += (uint32_t)r;
      if (g == s.msg) {
        const b200_slice back{req, s.msg};
        uint64_t sent = 0, c = 0;
        status = stream_send(h, &back, 1, b, sent, c);
        g = 0;
        const uint32_t d = done[i] + 1;
        if (lane == 0) done[i] = d;
        if (d == s.rounds) {
          b200_warp_disconnect(h);
          closed++;
        }
      }
      if (lane == 0) got[i] = g;
      __syncwarp();
    }
    if (b.spent()) status = DP_TIMEOUT;
    if (status != DP_OK) break;
  }
  if (lane == 0) {
    s.out[4 * s.n + 0] = status;
    s.out[4 * s.n + 1] = closed;
    s.out[4 * s.n + 2] = scans;
    s.out[4 * s.n + 3] = empty;
  }
}

__device__ void serve_pong(const dp_serve& s, uint32_t i) {
  Bound b = make_bound(s.budget_ns, s.max_iters);
  const b200_dev_pair* h = &s.srv[i];
  uint8_t* req = s.sbuf + (uint64_t)i * s.msg;
  const b200_slice back{req, s.msg};
  uint32_t status = DP_OK;
  for (uint32_t r = 0; r < s.rounds && status == DP_OK; r++) {
    uint64_t got = 0, sent = 0, c = 0;
    status = stream_recv(h, req, s.msg, b, got, c);
    if (status == DP_OK) status = stream_send(h, &back, 1, b, sent, c);
  }
  if (status == DP_OK) b200_warp_disconnect(h);
  if ((threadIdx.x & 31) == 0 && status != DP_OK) s.out[4 * s.n] = status;
}

__device__ void client(const dp_serve& s, uint32_t i) {
  const uint32_t lane = threadIdx.x & 31;
  Bound b = make_bound(s.budget_ns, s.max_iters);
  const b200_dev_pair* h = &s.cli[i];
  uint8_t* req = s.cbuf + 2ull * i * s.msg;
  uint8_t* rep = req + s.msg;
  const uint32_t words = s.msg / 8;
  const b200_slice out{req, s.msg};
  uint32_t status = DP_OK, r = 0;
  uint64_t bad = 0;
  for (; r < s.rounds && status == DP_OK; r++) {
    for (uint32_t j = lane; j < words; j += 32) reinterpret_cast<uint64_t*>(req)[j] = pattern_word(i, r, j);
    __syncwarp();
    uint64_t t0 = 0, sent = 0, got = 0, c = 0;
    if (lane == 0) t0 = now_ns();
    status = stream_send(h, &out, 1, b, sent, c);
    if (status == DP_OK) status = stream_recv(h, rep, s.msg, b, got, c);
    if (lane == 0) s.times[(uint64_t)i * s.rounds + r] = now_ns() - t0;
    bool diff = false;
    for (uint32_t j = lane; j < words; j += 32) diff |= reinterpret_cast<const uint64_t*>(rep)[j] != pattern_word(i, r, j);
    bad += __any_sync(0xffffffffu, diff) ? 1 : 0;
  }
  if (status == DP_OK) r = s.rounds;
  // the server closes the connection after the last reply: wait for it (bounded)
  int st = b200_warp_status(h);
  while (status == DP_OK && st != B200_HALF_CLOSED) {
    if (b.spent()) {
      status = DP_TIMEOUT;
      break;
    }
    st = b200_warp_status(h);
  }
  if (lane == 0) {
    s.out[4 * i + 0] = status;
    s.out[4 * i + 1] = bad;
    s.out[4 * i + 2] = r;
    s.out[4 * i + 3] = (uint64_t)st;
  }
}

__global__ void __launch_bounds__(128) dp_serve_kernel(dp_serve s) {
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (s.n == 0) return;  // (the module-loading launch of dp_prepare)
  const uint32_t nsrv = s.mode == 0 ? 1 : s.n;
  if (w < nsrv) {
    if (s.mode == 0) serve_polling(s);
    else serve_pong(s, w);
  } else if (s.cli && w < nsrv + s.n) {
    client(s, w - nsrv);
  }
}

// ---- poll cost: `batches` x `per` scans of n handles by one warp; times[k] = ns of batch k / per
__global__ void dp_poll_time_kernel(const b200_dev_pair* handles, uint32_t n, uint32_t* ready, uint32_t batches,
                                    uint32_t per, uint64_t* times) {
  uint32_t sink = 0;
  for (uint32_t k = 0; k < batches; k++) {
    uint64_t t0 = 0;
    if ((threadIdx.x & 31) == 0) t0 = now_ns();
    for (uint32_t j = 0; j < per; j++) sink += b200_warp_poll(handles, n, nullptr, ready);
    if ((threadIdx.x & 31) == 0) times[k] = (now_ns() - t0) / per;
  }
  if ((threadIdx.x & 31) == 0 && sink == 0xffffffffu) times[0] = 0;  // (keeps the scans)
}

static cudaStream_t g_stream = nullptr;
static char g_err[256];

extern "C" const char* dp_error(void) { return g_err; }

static int fin(cudaError_t e) {
  snprintf(g_err, sizeof g_err, "%s", cudaGetErrorString(e));
  return e == cudaSuccess ? 0 : -1;
}

// Load the module and create the stream now: while the library's service kernels are resident, the first launch of
// a kernel would wait for an idle device.  These launches have nothing to do and touch no memory.
extern "C" int dp_prepare(void) {
  if (!g_stream && cudaStreamCreateWithFlags(&g_stream, cudaStreamNonBlocking) != cudaSuccess) return -1;
  dp_kernel<<<1, 32, 0, g_stream>>>(nullptr, nullptr, nullptr, 0, 0, 0);
  dp_poll_kernel<<<1, 32, 0, g_stream>>>(nullptr, 0, nullptr, nullptr, nullptr);
  dp_serve s{};
  dp_serve_kernel<<<1, 32, 0, g_stream>>>(s);
  dp_poll_time_kernel<<<1, 32, 0, g_stream>>>(nullptr, 0, nullptr, 0, 0, nullptr);
  return fin(cudaStreamSynchronize(g_stream));
}

extern "C" int dp_launch(const void* pairs, void* ops, const uint32_t* first, int nlists, uint64_t budget_ns,
                         uint64_t max_iters) {
  if (!g_stream && dp_prepare() != 0) return -1;
  const int threads = 128, warps = threads / 32;
  dp_kernel<<<(nlists + warps - 1) / warps, threads, 0, g_stream>>>(
      static_cast<const b200_dev_pair*>(pairs), static_cast<dp_op*>(ops), first, nlists, budget_ns, max_iters);
  return fin(cudaGetLastError());
}
extern "C" int dp_wait(void) { return fin(cudaStreamSynchronize(g_stream)); }

// one scan; handles / events / ready / count: device or pinned memory (events, ready may be NULL)
extern "C" int dp_poll(const void* handles, uint32_t n, uint32_t* events, uint32_t* ready, uint32_t* count) {
  if (!g_stream && dp_prepare() != 0) return -1;
  dp_poll_kernel<<<1, 32, 0, g_stream>>>(static_cast<const b200_dev_pair*>(handles), n, events, ready, count);
  if (fin(cudaGetLastError()) != 0) return -1;
  return dp_wait();
}

// the server (and clients): queued when this returns, dp_wait() for the end.  -2: the warps would not all be resident
// at once (they wait for each other).
extern "C" int dp_serve_launch(const dp_serve* s) {
  if (!g_stream && dp_prepare() != 0) return -1;
  const uint32_t warps = (s->mode == 0 ? 1 : s->n) + (s->cli ? s->n : 0);
  const int threads = 128, blocks = (int)((warps * 32 + threads - 1) / threads);
  int dev = 0, sms = 0, per_sm = 0;
  if (fin(cudaGetDevice(&dev)) || fin(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)) ||
      fin(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, dp_serve_kernel, threads, 0)))
    return -1;
  if (per_sm * sms < blocks) {
    snprintf(g_err, sizeof g_err, "%d blocks of %d threads are not co-resident (%d per SM x %d SMs)", blocks, threads,
             per_sm, sms);
    return -2;
  }
  dp_serve_kernel<<<blocks, threads, 0, g_stream>>>(*s);
  return fin(cudaGetLastError());
}

extern "C" int dp_poll_time(const void* handles, uint32_t n, uint32_t* ready, uint32_t batches, uint32_t per,
                            uint64_t* times) {
  if (!g_stream && dp_prepare() != 0) return -1;
  dp_poll_time_kernel<<<1, 32, 0, g_stream>>>(static_cast<const b200_dev_pair*>(handles), n, ready, batches, per,
                                              times);
  if (fin(cudaGetLastError()) != 0) return -1;
  return dp_wait();
}
