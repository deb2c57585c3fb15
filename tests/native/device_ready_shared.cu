// device_ready_shared.cu -- TEST INFRASTRUCTURE: user kernels in which many consumer warps take from one device ready
// set (include/b200_device.cuh: b200_warp_ready_take / b200_warp_ready_rearm), and ctypes-callable launchers.  Built
// by device_ready_shared.mk for sm_90a against the public headers only.
//
//   ds_drain_kernel  W consumer warps, two per CTA: take, serve each key (Recv until nothing is
//                    complete, Disconnect a member whose peer left), rearm; until a take finds nothing, or, with a
//                    stop flag, until the host raises it and a take finds nothing
//   ds_serve_kernel  W server warps on one set or on W sets (warp w takes from set w % nsets), and one client warp per
//                    active connection: an echo until every client has its replies
//   ds_cost_kernel   ns per empty take, the shared take and the one-consumer baseline alternating
// Holder check: every consumer keeps a holder word per member in device memory.  On each take or kept rearm it runs
// atomicCAS(holder, 0, warp + 1) and counts a failure as a violation; it clears the word just before its rearm.
// A consumer that shares its set fences before that clear, so that what it wrote while it held the member (its
// Recv / Send cursors, the bookkeeping below) is visible before the rearm's store of armed = 1 can hand the member to
// another warp (DESIGN.md §13 "Many consumers").
// Every loop is bounded by an iteration cap (status 1); launches whose warps wait for each other check co-residency.
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

// The one-consumer take of the parent design (a plain store of head), kept only so that the measurement tool can
// compare one consumer warp on the shared take against it.  Not safe with two consumers.
__device__ uint32_t baseline_take(b200::ReadyQueue* q, uint32_t* keys, uint32_t max, uint32_t lane) {
  const uint32_t head = *(volatile uint32_t*)&q->head, mask = *(volatile uint32_t*)&q->mask;
  uint32_t n = 0;
  while (n < max) {
    const uint32_t i = n + lane;
    bool ok = false;
    uint64_t e = 0;
    if (i < max) {
      const uint32_t pos = head + i;
      const uint64_t* slot = b200::ready_entries(q) + (pos & mask);
      asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(e) : "l"(slot) : "memory");
      ok = b200::ready_entry_at(e, pos);
    }
    const unsigned bad = __ballot_sync(0xffffffffu, !ok);
    const uint32_t run = bad ? __ffs(bad) - 1 : 32;
    if (lane < run) keys[i] = (uint32_t)e;
    n += run;
    if (run < 32) break;
  }
  __syncwarp();
  if (lane == 0 && n) *(volatile uint32_t*)&q->head = head + n;
  __syncwarp();
  return n;
}

// the holder check: 1 when this warp took the member, 0 (a violation) when another warp holds it
__device__ __forceinline__ uint32_t hold(uint32_t* holder, uint32_t me) {
  uint32_t ok = 0;
  if (lane_id() == 0) ok = atomicCAS(holder, 0u, me) == 0u;
  return __shfl_sync(0xffffffffu, ok, 0);
}
__device__ __forceinline__ void unhold(uint32_t* holder) {
  __threadfence();
  __syncwarp();
  if (lane_id() == 0) atomicExch(holder, 0u);
  __threadfence();
}

// ---- the consumers of the random traces

struct ds_drain {
  const b200_dev_ready_set* set;
  const b200_dev_pair* members;  // by key
  uint32_t n, take_max;          // members; keys per take
  uint32_t warp_base, mark_idle; // holder id = warp_base + warp + 1; mark_idle: rearm 0 sets idle[k]
  uint8_t* rbuf;                 // n * rcap: what each member received, in order
  uint64_t rcap;
  uint64_t* got;                 // n: bytes received so far
  uint32_t* holder;              // n (device memory): holder words
  uint32_t* taken;               // n: returned by take
  uint32_t* kept;                // n: returned by rearm
  uint32_t* idle;                // n: rearm returned 0 while mark_idle: a later take of the key is a second entry
  uint32_t* closed;              // n: the consumer disconnected the member after its peer left
  uint32_t* keys;                // warps * take_max
  uint32_t* out;                 // per warp 8: status, violations, second entries, foreign keys, takes, lost CASes
  volatile uint32_t* stop;       // NULL: return once a take finds nothing; else once *stop != 0 and a take finds nothing
  uint64_t max_iters;
};
static_assert(sizeof(ds_drain) == 128, "ds_drain layout is mirrored in tests/device_ready_shared_lib.py");

__device__ void drain_member(const ds_drain& d, uint32_t k, uint32_t me, uint32_t& viol, uint64_t& iters) {
  const uint32_t lane = lane_id();
  const b200_dev_pair* h = &d.members[k];
  volatile uint64_t* got = d.got;
  for (;;) {
    uint64_t g = got[k];
    for (;;) {
      const uint64_t r = b200_warp_recv(h, d.rbuf + k * d.rcap + g, d.rcap - g);
      if (r == 0) break;
      g += r;
    }
    if (lane == 0) got[k] = g;
    __syncwarp();
    if (b200_warp_status(h) == B200_HALF_CLOSED) {  // the peer left: close the member (this warp keeps holding it)
      b200_warp_disconnect(h);
      if (lane == 0) ((volatile uint32_t*)d.closed)[k] = 1;
      break;
    }
    unhold(&d.holder[k]);
    const uint32_t ev = b200_warp_ready_rearm(d.set, h);
    if (ev == 0) {
      if (lane == 0 && d.mark_idle) ((volatile uint32_t*)d.idle)[k] = 1;
      break;
    }
    if (!hold(&d.holder[k], me)) viol++;
    if (lane == 0) ((volatile uint32_t*)d.kept)[k] += 1;
    if (++iters >= d.max_iters) break;
  }
  __syncwarp();
}

__global__ void ds_drain_kernel(ds_drain d) {
  if (d.n == 0) return;
  const uint32_t lane = lane_id(), w = warp_id(), me = d.warp_base + w + 1;
  uint32_t* keys = d.keys + (uint64_t)w * d.take_max;
  uint32_t retries = 0;
  uint64_t iters = 0;
  uint32_t viol = 0, dups = 0, foreign = 0, takes = 0;
  for (;;) {
    const uint32_t c =
        b200::ready_take(static_cast<b200::ReadyQueue*>(d.set->queue), keys, d.take_max, lane, &retries);
    takes += c;
    if (c == 0) {
      if (d.stop == nullptr || *d.stop != 0) break;
      if (++iters >= d.max_iters) break;
      __nanosleep(200);
      continue;
    }
    for (uint32_t j = 0; j < c; j++) {
      const uint32_t k = keys[j];
      if (k >= d.n) {
        foreign++;
        continue;
      }
      if (((volatile uint32_t*)d.idle)[k]) dups++;  // (producers have stopped: nothing could queue it after that rearm)
      if (!hold(&d.holder[k], me)) viol++;
      if (lane == 0) ((volatile uint32_t*)d.taken)[k] += 1;
      __syncwarp();
      if (((volatile uint32_t*)d.closed)[k]) continue;  // (a closed member has no entry: a take of it is a violation)
      drain_member(d, k, me, viol, iters);
    }
    if (iters >= d.max_iters) break;
  }
  if (lane == 0) {
    uint32_t* o = d.out + 8ull * w;
    o[0] = iters >= d.max_iters ? 1 : 0;
    o[1] = viol;
    o[2] = dups;
    o[3] = foreign;
    o[4] = takes;
    o[5] = retries;
  }
}

// ---- the echo server: W server warps, one client warp per active connection

struct ds_serve {
  const b200_dev_ready_set* sets;  // nsets handles; warp w takes from sets[w % nsets]
  const b200_dev_pair* srv;        // n server ends (key = index)
  const b200_dev_pair* cli;        // a client ends
  uint32_t n, a, rounds, msg;
  uint32_t servers, nsets, take_max, flags;  // flags: kBaseline (one consumer), kFence (warps share a set)
  uint8_t* sbuf;                   // n * msg (device memory)
  uint8_t* cbuf;                   // a * 2 * msg (device memory)
  uint32_t* state;                 // 2 n (device memory, zeroed): request bytes so far, holder words
  uint32_t* keys;                  // servers * take_max (device memory)
  unsigned long long* done;        // replies of all server warps (device memory, zeroed)
  uint64_t* out;                   // clients 2 a: mismatched replies, rounds done; then per server warp 8: status,
                                   // replies, keys taken, takes, lost CASes, violations, start ns, end ns
  uint64_t max_iters;
};
static_assert(sizeof(ds_serve) == 112, "ds_serve layout is mirrored in tests/device_ready_shared_lib.py");
constexpr uint32_t kBaseline = 1, kFence = 2;

__device__ __forceinline__ uint64_t pattern_word(uint32_t conn, uint32_t round, uint32_t j) {
  return ((uint64_t)conn << 48) ^ ((uint64_t)round << 24) ^ ((uint64_t)j * 0x9E3779B97F4A7C15ull);
}

// Recv what is there; a whole request is echoed.  Returns false when the echo ran out of its iteration budget.
__device__ bool serve_one(const ds_serve& s, uint32_t i, uint64_t& replies, uint64_t& iters) {
  const uint32_t lane = lane_id();
  const b200_dev_pair* h = &s.srv[i];
  uint8_t* req = s.sbuf + (uint64_t)i * s.msg;
  volatile uint32_t* st = s.state;
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
      if (lane == 0) atomicAdd(s.done, 1ull);
    }
  }
  if (lane == 0) st[i] = g;
  __syncwarp();
  return true;
}

__device__ void server(const ds_serve& s, uint32_t w) {
  const uint32_t lane = lane_id();
  const b200_dev_ready_set* set = &s.sets[w % s.nsets];
  b200::ReadyQueue* q = static_cast<b200::ReadyQueue*>(set->queue);
  uint32_t* keys = s.keys + (uint64_t)w * s.take_max;
  uint32_t* holder = s.state + s.n;
  const uint64_t want = (uint64_t)s.a * s.rounds;
  uint64_t replies = 0, iters = 0, got = 0, takes = 0, t0 = 0;
  uint32_t status = 0, viol = 0, retries = 0;
  if (lane == 0) t0 = now_ns();
  while (status == 0 && *(volatile unsigned long long*)s.done < want) {
    const uint32_t c = (s.flags & kBaseline) ? baseline_take(q, keys, s.take_max, lane)
                                             : b200::ready_take(q, keys, s.take_max, lane, &retries);
    takes++;
    got += c;
    for (uint32_t k = 0; k < c; k++) {  // every key taken is served and rearmed, even past the last reply
      const uint32_t i = keys[k];
      if (!hold(&holder[i], w + 1)) viol++;
      for (;;) {
        if (!serve_one(s, i, replies, iters)) {
          status = 1;  // (the member stays held: the run has failed)
          break;
        }
        if (s.flags & kFence) {
          unhold(&holder[i]);
        } else if (lane == 0) {
          atomicExch(&holder[i], 0u);
        }
        if (b200_warp_ready_rearm(set, &s.srv[i]) == 0) break;
        if (!hold(&holder[i], w + 1)) viol++;
      }
    }
    if (++iters >= s.max_iters) status = 1;
  }
  if (lane == 0) {
    uint64_t* o = s.out + 2ull * s.a + 8ull * w;
    o[0] = status;
    o[1] = replies;
    o[2] = got;
    o[3] = takes;
    o[4] = retries;
    o[5] = viol;
    o[6] = t0;
    o[7] = now_ns();
  }
}

__device__ void client(const ds_serve& s, uint32_t i) {
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

__global__ void __launch_bounds__(128) ds_serve_kernel(ds_serve s) {
  const uint32_t w = warp_id();
  if (s.n == 0) return;
  if (w < s.servers) server(s, w);
  else if (w < s.servers + s.a) client(s, w - s.servers);
}

// ---- ns per empty take: times[2 k] the shared take, times[2 k + 1] the baseline.  Both take the queue pointer loaded
// once, so neither pays the read of the set's descriptor that b200_warp_ready_take makes on every call.
__global__ void ds_cost_kernel(const b200_dev_ready_set* set, uint32_t n, uint32_t* scratch, uint32_t batches,
                               uint32_t per, uint64_t* times) {
  b200::ReadyQueue* q = static_cast<b200::ReadyQueue*>(set->queue);
  uint32_t sink = 0;
  for (uint32_t k = 0; k < batches; k++) {
    uint64_t t0 = 0;
    if (lane_id() == 0) t0 = now_ns();
    for (uint32_t j = 0; j < per; j++) sink += b200::ready_take(q, scratch, n, lane_id());
    if (lane_id() == 0) times[2 * k] = (now_ns() - t0) / per;
    if (lane_id() == 0) t0 = now_ns();
    for (uint32_t j = 0; j < per; j++) sink += baseline_take(q, scratch, n, lane_id());
    if (lane_id() == 0) times[2 * k + 1] = (now_ns() - t0) / per;
  }
  if (lane_id() == 0 && sink == 0xffffffffu) times[0] = 0;  // (keeps the calls)
}

static cudaStream_t g_stream[2] = {nullptr, nullptr};
static char g_err[256];

extern "C" const char* ds_error(void) { return g_err; }

static int fin(cudaError_t e) {
  snprintf(g_err, sizeof g_err, "%s", cudaGetErrorString(e));
  return e == cudaSuccess ? 0 : -1;
}

// Load the module and create the streams now: while the library's service kernels or a consumer are resident, the
// first launch of a kernel would wait for an idle device.  These launches have nothing to do and touch no memory.
extern "C" int ds_prepare(void) {
  for (auto& st : g_stream)
    if (!st && cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) return -1;
  ds_drain d{};
  ds_drain_kernel<<<1, 64, 0, g_stream[0]>>>(d);
  ds_serve s{};
  ds_serve_kernel<<<1, 128, 0, g_stream[0]>>>(s);
  ds_cost_kernel<<<1, 32, 0, g_stream[0]>>>(nullptr, 0, nullptr, 0, 0, nullptr);
  return fin(cudaStreamSynchronize(g_stream[0]));
}

static int co_resident(const void* kernel, int blocks, int threads) {
  int dev = 0, sms = 0, per_sm = 0;
  if (fin(cudaGetDevice(&dev)) || fin(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)) ||
      fin(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0)))
    return -1;
  if (per_sm * sms < blocks) {
    snprintf(g_err, sizeof g_err, "%d blocks of %d threads are not co-resident", blocks, threads);
    return -2;
  }
  return 0;
}

extern "C" int ds_wait(int stream) { return fin(cudaStreamSynchronize(g_stream[stream & 1])); }

// `warps` consumers, two per CTA, on stream 0 or 1; queued when this returns: ds_wait(stream) for the end.  A consumer
// with a stop flag runs beside the producers, so its CTAs must all be resident (-2 otherwise).
extern "C" int ds_drain_launch(const ds_drain* d, uint32_t warps, int stream) {
  if (!g_stream[0] && ds_prepare() != 0) return -1;
  if (warps == 0 || (warps > 1 && warps % 2)) {
    snprintf(g_err, sizeof g_err, "consumer warps must be 1 or even, not %u", warps);
    return -1;
  }
  const int threads = warps == 1 ? 32 : 64, blocks = (int)((warps + 1) / 2);
  const int rc = co_resident((const void*)ds_drain_kernel, blocks, threads);
  if (rc) return rc;
  ds_drain_kernel<<<blocks, threads, 0, g_stream[stream & 1]>>>(*d);
  return fin(cudaGetLastError());
}

// synchronous; -2: the warps would not all be resident at once (they wait for each other)
extern "C" int ds_serve_launch(const ds_serve* s) {
  if (!g_stream[0] && ds_prepare() != 0) return -1;
  const uint32_t warps = s->servers + s->a;
  const int threads = 128, blocks = (int)((warps * 32 + threads - 1) / threads);
  const int rc = co_resident((const void*)ds_serve_kernel, blocks, threads);
  if (rc) return rc;
  ds_serve_kernel<<<blocks, threads, 0, g_stream[0]>>>(*s);
  if (fin(cudaGetLastError())) return -1;
  return ds_wait(0);
}

extern "C" int ds_cost(const void* set, uint32_t n, uint32_t* scratch, uint32_t batches, uint32_t per,
                       uint64_t* times) {
  if (!g_stream[0] && ds_prepare() != 0) return -1;
  ds_cost_kernel<<<1, 32, 0, g_stream[0]>>>(static_cast<const b200_dev_ready_set*>(set), n, scratch, batches, per,
                                            times);
  if (fin(cudaGetLastError())) return -1;
  return ds_wait(0);
}

// device memory helpers on stream 0 (synchronous)
extern "C" int ds_zero(void* p, uint64_t bytes) {
  if (!g_stream[0] && ds_prepare() != 0) return -1;
  if (fin(cudaMemsetAsync(p, 0, bytes, g_stream[0]))) return -1;
  return ds_wait(0);
}
extern "C" int ds_copy(void* dst, const void* src, uint64_t bytes) {
  if (!g_stream[0] && ds_prepare() != 0) return -1;
  if (fin(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, g_stream[0]))) return -1;
  return ds_wait(0);
}
