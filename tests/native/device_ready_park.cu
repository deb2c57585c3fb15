// device_ready_park.cu -- TEST INFRASTRUCTURE: an echo server that parks its device ready set when idle
// (include/b200_device.cuh: b200_warp_ready_park), device client warps, and ctypes-callable launchers.  Built by
// device_ready_park.mk for sm_90a against the public headers only.
//
//   dp_server_kernel   W server warps on one set: take, echo every whole request, rearm; a warp that finds the set empty
//                      `idle_takes` times in a row adds one to the idle counter and stops taking.  The last warp to go
//                      idle parks the set; while the park returns non-zero it serves alone and parks again.
//   dp_client_kernel   one warp per client end: `rounds` requests of `msg` bytes, each followed by its reply, checked
// Every loop is bounded by an iteration cap (status 1).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200_device.cuh"

__device__ __forceinline__ uint64_t now_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ uint32_t warp_id() { return (blockIdx.x * blockDim.x + threadIdx.x) >> 5; }

// request word j of round r of connection `conn`: the server echoes it, the client checks the reply
__device__ __forceinline__ uint64_t pattern_word(uint32_t conn, uint32_t round, uint32_t j) {
  return ((uint64_t)conn << 48) ^ ((uint64_t)round << 24) ^ ((uint64_t)j * 0x9E3779B97F4A7C15ull);
}

struct dp_server {
  const b200_dev_ready_set* set;
  const b200_dev_pair* srv;  // n server ends (key = index)
  uint32_t n, msg, warps, idle_takes;
  uint8_t* sbuf;             // n * msg (device memory): the request each member is receiving
  uint32_t* state;           // n + 1 (device memory): request bytes so far; [n] the idle counter, zeroed per launch
  uint32_t* closed;          // n: the server disconnected the member after its peer left
  uint64_t* out;             // 8 (device memory): status, replies, keys taken, parks that returned non-zero, start
                             // ns (initially ~0), end ns
  uint64_t max_iters;
  uint32_t no_park, _pad;    // no_park: the last warp exits without parking (a set that is never parked)
};
static_assert(sizeof(dp_server) == 80, "dp_server layout is mirrored in tests/device_ready_park_lib.py");

// Echo every whole request member i has; then either disconnect it (its peer left) or rearm it, until the rearm
// returns 0.  Returns false when the run ran out of its iteration budget.
__device__ bool serve_member(const dp_server& s, uint32_t i, uint64_t& replies, uint64_t& iters) {
  const uint32_t lane = lane_id();
  const b200_dev_pair* h = &s.srv[i];
  uint8_t* req = s.sbuf + (uint64_t)i * s.msg;
  volatile uint32_t* st = s.state;
  for (;;) {
    uint32_t g = st[i];
    for (;;) {
      const uint64_t r = b200_warp_recv(h, req + g, s.msg - g);
      if (r == 0) break;
      g += (uint32_t)r;
      if (g == s.msg) {
        uint64_t sent = 0;
        while (sent < s.msg) {
          const b200_slice rest{req + sent, s.msg - sent};
          sent += b200_warp_send(h, &rest, 1, 0);
          if (++iters >= s.max_iters) return false;
        }
        g = 0;
        replies++;
      }
    }
    if (lane == 0) st[i] = g;
    __syncwarp();
    if (b200_warp_status(h) == B200_HALF_CLOSED) {  // the peer left: close the member, which ends the hold
      b200_warp_disconnect(h);
      if (lane == 0) ((volatile uint32_t*)s.closed)[i] = 1;
      return true;
    }
    __threadfence();  // (the warps share the set: what this warp wrote before the next holder takes the member)
    if (b200_warp_ready_rearm(s.set, h) == 0) return true;
    if (++iters >= s.max_iters) return false;
  }
}

// take and serve until `limit` takes in a row find nothing
__device__ bool serve_until_idle(const dp_server& s, uint32_t* keys, uint32_t limit, uint64_t& replies,
                                 uint64_t& taken, uint64_t& iters) {
  for (uint32_t empty = 0; empty < limit;) {
    const uint32_t c = b200_warp_ready_take(s.set, keys, 4);
    if (c == 0) {
      empty++;
      if (++iters >= s.max_iters) return false;
      continue;
    }
    empty = 0;
    taken += c;
    for (uint32_t k = 0; k < c; k++) {
      const uint32_t i = keys[k];
      if (i >= s.n || ((volatile uint32_t*)s.closed)[i]) continue;
      if (!serve_member(s, i, replies, iters)) return false;
    }
  }
  return true;
}

__global__ void __launch_bounds__(256) dp_server_kernel(dp_server s) {
  __shared__ uint32_t keys_smem[8][4];
  const uint32_t lane = lane_id(), w = warp_id();
  if (s.n == 0 || w >= s.warps) return;
  uint32_t* keys = keys_smem[threadIdx.x >> 5];
  uint64_t replies = 0, taken = 0, iters = 0, busy = 0, t0 = 0;
  if (lane == 0) t0 = now_ns();
  bool ok = serve_until_idle(s, keys, s.idle_takes, replies, taken, iters);
  uint32_t last = 0;
  if (lane == 0) last = atomicAdd(&s.state[s.n], 1u) == s.warps - 1;
  last = __shfl_sync(0xffffffffu, last, 0);
  if (last && ok && !s.no_park) {
    // every other warp has stopped taking: park, and serve alone while the park finds work
    while (b200_warp_ready_park(s.set) != 0) {
      busy++;
      if (!serve_until_idle(s, keys, 1, replies, taken, iters)) {
        ok = false;
        break;
      }
    }
  }
  if (lane == 0) {
    if (!ok) atomicExch((unsigned long long*)&s.out[0], 1ull);
    atomicAdd((unsigned long long*)&s.out[1], replies);
    atomicAdd((unsigned long long*)&s.out[2], taken);
    atomicAdd((unsigned long long*)&s.out[3], busy);
    atomicMin((unsigned long long*)&s.out[4], t0);
    atomicMax((unsigned long long*)&s.out[5], now_ns());
  }
}

struct dp_clients {
  const b200_dev_pair* cli;  // a client ends
  uint32_t a, rounds, msg, conn_base;  // conn_base: the pattern's connection number of client 0
  uint8_t* cbuf;             // a * 2 * msg (device memory)
  uint64_t* out;             // 2 a: mismatched replies, rounds done
  uint64_t max_iters;
};
static_assert(sizeof(dp_clients) == 48, "dp_clients layout is mirrored in tests/device_ready_park_lib.py");

__global__ void __launch_bounds__(128) dp_client_kernel(dp_clients c) {
  const uint32_t i = warp_id(), lane = lane_id();
  if (i >= c.a) return;
  const b200_dev_pair* h = &c.cli[i];
  uint8_t* req = c.cbuf + 2ull * i * c.msg;
  uint8_t* rep = req + c.msg;
  const uint32_t words = c.msg / 8;
  uint64_t bad = 0, iters = 0;
  uint32_t r = 0;
  for (; r < c.rounds; r++) {
    for (uint32_t j = lane; j < words; j += 32)
      reinterpret_cast<uint64_t*>(req)[j] = pattern_word(c.conn_base + i, r, j);
    __syncwarp();
    uint64_t sent = 0, got = 0;
    while (sent < c.msg && iters < c.max_iters) {
      const b200_slice rest{req + sent, c.msg - sent};
      sent += b200_warp_send(h, &rest, 1, 0);
      iters++;
    }
    while (got < c.msg && iters < c.max_iters) {
      got += b200_warp_recv(h, rep + got, c.msg - got);
      iters++;
    }
    if (got < c.msg) break;
    bool diff = false;
    for (uint32_t j = lane; j < words; j += 32)
      diff |= reinterpret_cast<const uint64_t*>(rep)[j] != pattern_word(c.conn_base + i, r, j);
    bad += __any_sync(0xffffffffu, diff) ? 1 : 0;
  }
  if (lane == 0) {
    c.out[2 * i + 0] = bad;
    c.out[2 * i + 1] = r;
  }
}

static cudaStream_t g_stream[2] = {nullptr, nullptr};  // [0] servers, [1] clients
static cudaEvent_t g_ev[2] = {nullptr, nullptr};       // around the last server launch
static char g_err[256];

extern "C" const char* dp_error(void) { return g_err; }

static int fin(cudaError_t e) {
  snprintf(g_err, sizeof g_err, "%s", cudaGetErrorString(e));
  return e == cudaSuccess ? 0 : -1;
}

// Load the module and create the streams and events now: while a client kernel or the library's service is resident,
// the first launch of a kernel would wait for an idle device.  These launches have nothing to do.
extern "C" int dp_prepare(void) {
  for (auto& st : g_stream)
    if (!st && cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) return fin(cudaGetLastError());
  for (auto& ev : g_ev)
    if (!ev && cudaEventCreate(&ev) != cudaSuccess) return fin(cudaGetLastError());
  dp_server s{};
  dp_server_kernel<<<1, 32, 0, g_stream[0]>>>(s);
  dp_clients c{};
  dp_client_kernel<<<1, 32, 0, g_stream[0]>>>(c);
  return fin(cudaStreamSynchronize(g_stream[0]));
}

// A server of `warps` (1..256) warps; queued when this returns (dp_server_wait).  The idle counter s->state[n] must
// be 0: dp_server_launch zeroes it on the server stream first.
extern "C" int dp_server_launch(const dp_server* s) {
  if (!g_stream[0] && dp_prepare() != 0) return -1;
  if (s->warps < 1 || s->warps > 256) {
    snprintf(g_err, sizeof g_err, "server warps must be 1..256, not %u", s->warps);
    return -1;
  }
  if (fin(cudaMemsetAsync(s->state + s->n, 0, 4, g_stream[0]))) return -1;
  const uint32_t threads = s->warps < 8 ? 32 * s->warps : 256, blocks = (s->warps * 32 + threads - 1) / threads;
  cudaEventRecord(g_ev[0], g_stream[0]);
  dp_server_kernel<<<blocks, threads, 0, g_stream[0]>>>(*s);
  cudaEventRecord(g_ev[1], g_stream[0]);
  return fin(cudaGetLastError());
}
// waits for the last server; *ms (may be NULL) gets its kernel time from the events around it
extern "C" int dp_server_wait(float* ms) {
  if (fin(cudaStreamSynchronize(g_stream[0]))) return -1;
  if (ms && fin(cudaEventElapsedTime(ms, g_ev[0], g_ev[1]))) return -1;
  return 0;
}

// a client warps on the client stream; queued when this returns (dp_clients_wait)
extern "C" int dp_clients_launch(const dp_clients* c) {
  if (!g_stream[0] && dp_prepare() != 0) return -1;
  const uint32_t threads = 128, blocks = (c->a * 32 + threads - 1) / threads;
  dp_client_kernel<<<blocks, threads, 0, g_stream[1]>>>(*c);
  return fin(cudaGetLastError());
}
extern "C" int dp_clients_wait(void) { return fin(cudaStreamSynchronize(g_stream[1])); }
// 1 while the client kernel runs
extern "C" int dp_clients_running(void) { return cudaStreamQuery(g_stream[1]) == cudaErrorNotReady ? 1 : 0; }

// device memory helpers on the server stream (synchronous)
extern "C" int dp_zero(void* p, uint64_t bytes) {
  if (!g_stream[0] && dp_prepare() != 0) return -1;
  if (fin(cudaMemsetAsync(p, 0, bytes, g_stream[0]))) return -1;
  return fin(cudaStreamSynchronize(g_stream[0]));
}
extern "C" int dp_copy(void* dst, const void* src, uint64_t bytes) {
  if (!g_stream[0] && dp_prepare() != 0) return -1;
  if (fin(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, g_stream[0]))) return -1;
  return fin(cudaStreamSynchronize(g_stream[0]));
}
