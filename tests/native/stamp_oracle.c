/*
 * stamp_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * CPU model of stamped ring frames (B200_RING_STAMPED=1, DESIGN.md §2), written over the plain-C restatement
 * of the reference pair (oracle/rb_oracle.c).  The reference has no such mode, so this model is the pin the
 * CUDA path is compared with.  Only the ring image differs from the reference:
 *
 *   frame s of a direction:  header = p | t(s) << 40,  t(s) = 1 + s mod (2^24 - 1),  footer = ~header
 *   present at head:         1 <= header & (2^40 - 1) <= C - 24 and header >> 40 == t(rx)
 *   complete:                present and footer == ~header
 *   Recv:                    retires what the reference retires, stores nothing into the ring
 *   HasMessage / readable:   remain > 0, or a complete stamped frame at head
 *
 * Send is the reference's per-slice Send or the coalesced one (tests/native/coalesce_oracle.c) with stamped
 * headers and footers.  Each pair's frame counters (tx: frames written into the peer's ring, rx: frames opened
 * in its own ring) live in a side table keyed by the pair.  Also here: b200_pair_ops tables over the model for the
 * endpoint host-logic tests.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/b200_endpoint.h"
#include "../../oracle/rb_oracle.h"

#define STAMP_MOD ((1ull << 24) - 1)
#define LEN_MASK ((1ull << 40) - 1)
#define COALESCE_SLICES 1024u

typedef struct {
  const orb_pair* p;
  uint64_t tx, rx;
  uint8_t* pads; /* 1 = pad byte of the frame last written over this byte of the pair's ring */
} seq_ent;
static seq_ent g_seq[256];

static seq_ent* seq_of(const orb_pair* p) {
  seq_ent* free_e = NULL;
  for (int i = 0; i < 256; i++) {
    if (g_seq[i].p == p) return &g_seq[i];
    if (!g_seq[i].p && !free_e) free_e = &g_seq[i];
  }
  if (!free_e) abort();
  free_e->p = p;
  free_e->tx = free_e->rx = 0;
  free(free_e->pads);
  free_e->pads = (uint8_t*)calloc(1, p->ring.capacity);
  return free_e;
}

uint32_t stamp_of(uint64_t s) { return 1u + (uint32_t)(s % STAMP_MOD); }
uint64_t stamp_header(uint64_t p, uint64_t s) { return p | (uint64_t)stamp_of(s) << 40; }

/* counters: set (tests start a pair at a chosen frame number) / get; forget a pair before it is destroyed */
void stamp_seq_set(const orb_pair* p, uint64_t tx, uint64_t rx) {
  seq_ent* e = seq_of(p);
  e->tx = tx;
  e->rx = rx;
}
uint64_t stamp_seq_tx(const orb_pair* p) { return seq_of(p)->tx; }
uint64_t stamp_seq_rx(const orb_pair* p) { return seq_of(p)->rx; }
void stamp_forget(const orb_pair* p) { seq_of(p)->p = NULL; }
/* the pad bytes of every frame image in the ring: retired frames stay, so their pads are part of the image */
const uint8_t* stamp_pads(const orb_pair* p) { return seq_of(p)->pads; }

static void mark_frame(orb_pair* peer, uint64_t at, uint64_t pay) {
  uint8_t* m = seq_of(peer)->pads;
  const uint64_t mask = peer->ring.mask, e = orb_encoded_size(pay);
  for (uint64_t i = 0; i < e; i++) m[(at + i) & mask] = i >= ORB_ALIGN + pay && i < ORB_ALIGN + orb_round_up(pay);
}

static uint64_t ld64(const uint8_t* b) {
  uint64_t v;
  memcpy(&v, b, 8);
  return v;
}

/* ---- receive side */
uint64_t stamp_readable(const orb_pair* p) {
  const orb_ring* r = &p->ring;
  if (r->remain > 0) return r->remain;
  const uint64_t hdr = ld64(r->buf + r->head), len = hdr & LEN_MASK;
  if ((hdr >> 40) != stamp_of(seq_of(p)->rx) || len == 0 || len > r->capacity - ORB_RESERVED) return 0;
  return ld64(r->buf + ((r->head + ORB_ALIGN + orb_round_up(len)) & r->mask)) == ~hdr ? len : 0;
}
int stamp_has_message(const orb_pair* p) { return stamp_readable(p) != 0; }
uint64_t stamp_pair_readable(const orb_pair* p) { return p->status == ORB_CONNECTED ? stamp_readable(p) : 0; }

/* RingBufferPollable::Read without the clear (ring_buffer.cc:122-191) */
static uint64_t stamp_ring_read(orb_pair* p, void* dst, uint64_t cap, uint64_t* internal) {
  orb_ring* r = &p->ring;
  const uint64_t readable = stamp_readable(p);
  const uint64_t n = readable < cap ? readable : cap;
  const uint64_t prev_mh = r->moving_head;
  *internal = 0;
  if (n == 0) return 0;
  if (r->remain == 0) { /* first touch of this frame */
    r->moving_head = (r->head + ORB_ALIGN) & r->mask;
    r->head = (r->head + 2u * ORB_ALIGN + orb_round_up(readable)) & r->mask;
    seq_of(p)->rx++;
  }
  const uint64_t first = r->capacity - r->moving_head < n ? r->capacity - r->moving_head : n;
  memcpy(dst, r->buf + r->moving_head, first);
  if (n > first) memcpy((uint8_t*)dst + first, r->buf, n - first);
  r->moving_head = (r->moving_head + n) & r->mask;
  r->remain = readable - n;
  if (r->remain == 0) r->moving_head = (orb_round_up(r->moving_head) + ORB_ALIGN) & r->mask; /* pad + footer */
  *internal = (r->moving_head + r->capacity - prev_mh) & r->mask;
  return n;
}

/* PairPollable::Recv + updateStatus (pair.cc:264-286, 624-641) */
uint64_t stamp_recv(orb_pair* p, void* dst, uint64_t cap) {
  if (p->status != ORB_CONNECTED) return 0;
  uint64_t internal = 0;
  const uint64_t n = stamp_ring_read(p, dst, cap, &internal);
  p->internal_read_size += internal;
  p->total_read += n;
  if (p->internal_read_size >= p->ring.capacity / 2) {
    p->status_out.remote_head = p->ring.moving_head;
    p->peer->status_in = p->status_out;
    p->n_status_writes++;
    p->internal_read_size = 0;
  }
  return n;
}

uint64_t stamp_recv_drain(orb_pair* p, void* dst, uint64_t cap, uint64_t* calls) {
  uint64_t got = 0, ncalls = 0;
  while (got < cap) {
    const uint64_t n = stamp_recv(p, (uint8_t*)dst + got, cap - got);
    if (n == 0) break;
    got += n;
    ncalls++;
  }
  if (calls) *calls = ncalls;
  return got;
}

/* ---- send side: the reference's Send (pair.cc:645-734), every frame stamped */
static void put_frame(orb_pair* p, uint8_t* f, const uint8_t* src, uint64_t pay) {
  const uint64_t hdr = stamp_header(pay, seq_of(p)->tx++), foot = ~hdr;
  memcpy(f, &hdr, 8);
  if (src) memcpy(f + ORB_ALIGN, src, pay);
  memcpy(f + ORB_ALIGN + orb_round_up(pay), &foot, 8);
}

uint64_t stamp_send(orb_pair* p, const orb_slice* slices, size_t n, size_t byte_idx) {
  if (p->status != ORB_CONNECTED) return 0;
  const uint64_t cap = p->ring.capacity, rh = p->status_in.remote_head;
  uint64_t rt = p->remote_tail, st = 0, total = 0, written = 0;
  int nsge = 0;
  for (size_t i = 0; i < n; i++) total += slices[i].len;
  total -= byte_idx;
  for (size_t i = 0; i < n && nsge < p->max_sge; i++) {
    const uint8_t* ptr = slices[i].ptr + byte_idx;
    const uint64_t len = slices[i].len - byte_idx;
    byte_idx = 0;
    const uint64_t a = orb_calc_writable(p->staging_size - st), b = orb_calc_writable(orb_free_size(cap, rh, rt));
    uint64_t pay = len;
    if (a < pay) pay = a;
    if (b < pay) pay = b;
    if (pay == 0) break;
    put_frame(p, p->staging + st, ptr, pay);
    mark_frame(p->peer, rt, pay);
    const uint64_t e = orb_encoded_size(pay);
    st += e;
    rt = (rt + e) & (cap - 1);
    written += pay;
    nsge++;
  }
  p->partial_write = written < total;
  if (nsge > 0) p->remote_tail = orb_ring_place(p->peer->ring.buf, cap, p->remote_tail, p->staging, st);
  p->total_write += written;
  return written;
}

/* the coalesced Send (coalesce_oracle.c), its one frame stamped */
uint64_t stamp_send_coalesced(orb_pair* p, const orb_slice* slices, size_t n, size_t byte_idx) {
  if (p->status != ORB_CONNECTED) return 0;
  const uint64_t cap = p->ring.capacity, rh = p->status_in.remote_head, rt = p->remote_tail;
  uint64_t total = 0, avail = 0;
  const size_t look = n < COALESCE_SLICES ? n : COALESCE_SLICES;
  for (size_t i = 0; i < n; i++) total += slices[i].len;
  total -= byte_idx;
  for (size_t i = 0; i < look; i++) avail += slices[i].len;
  avail -= look ? byte_idx : 0;
  uint64_t pay = avail;
  const uint64_t a = orb_calc_writable(p->staging_size), b = orb_calc_writable(orb_free_size(cap, rh, rt));
  if (a < pay) pay = a;
  if (b < pay) pay = b;
  p->partial_write = pay < total;
  if (pay == 0) return 0;
  uint8_t* f = p->staging;
  uint64_t off = 0;
  for (size_t i = 0; i < look && off < pay; i++) {
    const uint64_t skip = i == 0 ? byte_idx : 0;
    uint64_t m = slices[i].len - skip;
    if (m > pay - off) m = pay - off;
    if (m) memcpy(f + ORB_ALIGN + off, slices[i].ptr + skip, m);
    off += m;
  }
  put_frame(p, f, NULL, pay);
  mark_frame(p->peer, rt, pay);
  p->remote_tail = orb_ring_place(p->peer->ring.buf, cap, rt, f, orb_encoded_size(pay));
  p->total_write += pay;
  return pay;
}

/* rdma_flush loop (rdma_bp_posix.cc:470-524) over either Send */
uint64_t stamp_send_all(orb_pair* p, const orb_slice* slices, size_t n, size_t byte_idx, int coalesced,
                        uint64_t* calls) {
  uint64_t sent_total = 0, ncalls = 0;
  size_t idx = 0;
  while (idx < n) {
    uint64_t sent = coalesced ? stamp_send_coalesced(p, slices + idx, n - idx, byte_idx)
                              : stamp_send(p, slices + idx, n - idx, byte_idx);
    if (sent == 0) break;
    ncalls++;
    sent_total += sent;
    while (sent > 0) {
      const uint64_t left = slices[idx].len - byte_idx;
      if (sent >= left) {
        sent -= left;
        idx++;
        byte_idx = 0;
      } else {
        byte_idx += sent;
        sent = 0;
      }
    }
  }
  if (calls) *calls = ncalls;
  return sent_total;
}

/* ---- ops tables: tests/native/oracle_pair_ops.c with stamped Send / Recv / readiness, for the endpoint host-logic
 * tests.  Its pair handle starts with the orb_pair pointer; a pair gets fresh counters at every Init. */
const b200_pair_ops* oracle_pair_ops(void);
const b200_pair_ops* oracle_pair_ops_batch(void);
void oracle_ops_config(uint64_t ring_bytes, int max_sge);

static b200_pair_ops g_base, g_base_batch, g_ops, g_ops_batch;
static orb_pair* P(const void* v) { return *(orb_pair* const*)v; }

static void s_init(void* v) {
  if (P(v)) stamp_forget(P(v));
  g_base.init(v);
  if (P(v)) stamp_forget(P(v)); /* the next lookup starts the pair at frame 0 */
}
static uint64_t s_send(void* v, const b200_slice* s, size_t n, size_t b) {
  return stamp_send(P(v), (const orb_slice*)s, n, b);
}
static uint64_t s_recv(void* v, void* d, uint64_t c) { return stamp_recv(P(v), d, c); }
static int s_has_msg(const void* v) { return stamp_has_message(P(v)); }
static uint64_t s_readable(const void* v) { return stamp_pair_readable(P(v)); }
static int s_submit(const b200_send_op* s, size_t ns, uint64_t* acc, const b200_recv_op* r, size_t nr, uint64_t* del,
                    int flags) {
  for (size_t i = 0; i < ns; i++) {
    orb_pair* p = P(s[i].pair);
    acc[i] = (flags & B200_BATCH_UNTIL_BLOCKED)
                 ? stamp_send_all(p, (const orb_slice*)s[i].slices, s[i].nslices, s[i].byte_idx, 0, NULL)
                 : stamp_send(p, (const orb_slice*)s[i].slices, s[i].nslices, s[i].byte_idx);
  }
  for (size_t i = 0; i < nr; i++) {
    orb_pair* p = P(r[i].pair);
    del[i] = (flags & B200_BATCH_UNTIL_BLOCKED) ? stamp_recv_drain(p, r[i].dst, r[i].cap, NULL)
                                                : stamp_recv(p, r[i].dst, r[i].cap);
  }
  return 0;
}

void stamp_ops_config(uint64_t ring_bytes) { oracle_ops_config(ring_bytes, 30); }

static void stamped(b200_pair_ops* o) {
  o->init = s_init;
  o->send = s_send;
  o->recv = s_recv;
  o->has_message = s_has_msg;
  o->readable = s_readable;
}
const b200_pair_ops* stamp_pair_ops(void) {
  g_base = g_ops = *oracle_pair_ops();
  stamped(&g_ops);
  return &g_ops;
}
const b200_pair_ops* stamp_pair_ops_batch(void) {
  g_base = g_base_batch = g_ops_batch = *oracle_pair_ops_batch();
  stamped(&g_ops_batch);
  g_ops_batch.submit = s_submit;
  return &g_ops_batch;
}
