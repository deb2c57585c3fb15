/*
 * coalesce_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * CPU model of coalesced send framing (B200_SEND_COALESCE=1, DESIGN.md §2), written over the plain-C
 * restatement of the reference pair (oracle/rb_oracle.c).  The reference has no coalesced Send, so this
 * model is the pin the CUDA path is compared with.  A coalesced Send writes ONE frame per call:
 *
 *   if status != Connected: return 0
 *   total = sum(len(slices)) - byte_idx                  (all n slices count)
 *   look  = slices[0, min(n, 1024))                      (zero-length slices contribute nothing)
 *   p = min(bytes of look from byte_idx, CWS(staging), CWS(free(remote_head, remote_tail)))
 *   if p == 0: partial_write = total > 0; return 0
 *   ring[rt ..] = u64(p) | gather(look from byte_idx, p bytes) | pad | u64(~0)
 *   remote_tail += E(p); partial_write = p < total; return p
 *
 * The receive side is the reference's, unchanged.  Also here: a b200_pair_ops table whose Send is the
 * coalesced one (everything else is tests/native/oracle_pair_ops.c), for the endpoint host-logic tests.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/b200_endpoint.h"
#include "../../oracle/rb_oracle.h"

#define COALESCE_SLICES 1024u /* kCoalesceSlices, grpc-rdma_b200/csrc/b200_dev.cuh */

uint64_t orb_pair_send_coalesced(orb_pair* p, const orb_slice* slices, size_t n, size_t byte_idx) {
  if (p->status != ORB_CONNECTED) return 0;
  uint64_t cap = p->ring.capacity;
  uint64_t rh = p->status_in.remote_head, rt = p->remote_tail; /* one credit snapshot */
  uint64_t total = 0, avail = 0;
  size_t look = n < COALESCE_SLICES ? n : COALESCE_SLICES;
  for (size_t i = 0; i < n; i++) total += slices[i].len;
  total -= byte_idx;
  for (size_t i = 0; i < look; i++) avail += slices[i].len;
  avail -= look ? byte_idx : 0;
  uint64_t pay = avail;
  uint64_t a = orb_calc_writable(p->staging_size), b = orb_calc_writable(orb_free_size(cap, rh, rt));
  if (a < pay) pay = a;
  if (b < pay) pay = b;
  p->partial_write = pay < total;
  if (pay == 0) return 0;
  /* frame in staging: [len][gathered payload][pad as-is][~0], then one RDMA write of it */
  uint8_t* f = p->staging;
  uint64_t hdr = pay, foot = ORB_FOOTER, off = 0;
  memcpy(f, &hdr, 8);
  for (size_t i = 0; i < look && off < pay; i++) {
    uint64_t skip = i == 0 ? byte_idx : 0;
    uint64_t m = slices[i].len - skip;
    if (m > pay - off) m = pay - off;
    if (m) memcpy(f + ORB_ALIGN + off, slices[i].ptr + skip, m);
    off += m;
  }
  memcpy(f + ORB_ALIGN + orb_round_up(pay), &foot, 8);
  p->remote_tail = orb_ring_place(p->peer->ring.buf, cap, rt, f, orb_encoded_size(pay));
  p->total_write += pay;
  return pay;
}

/* rdma_flush loop over the coalesced Send: the same slice / byte cursor as orb_pair_send_all */
uint64_t orb_pair_send_coalesced_all(orb_pair* p, const orb_slice* slices, size_t n, size_t byte_idx,
                                     uint64_t* calls) {
  uint64_t sent_total = 0, ncalls = 0;
  size_t idx = 0;
  while (idx < n) {
    uint64_t sent = orb_pair_send_coalesced(p, slices + idx, n - idx, byte_idx);
    if (sent == 0) break;
    ncalls++;
    sent_total += sent;
    while (sent > 0) {
      uint64_t left = slices[idx].len - byte_idx;
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

/* ---- ops tables: tests/native/oracle_pair_ops.c with the coalesced Send.  Its pair handle starts with the
 * orb_pair pointer. */
const b200_pair_ops* oracle_pair_ops(void);
const b200_pair_ops* oracle_pair_ops_batch(void);
void oracle_ops_config(uint64_t ring_bytes, int max_sge);

static orb_pair* P(void* v) { return *(orb_pair**)v; }

static uint64_t c_send(void* v, const b200_slice* s, size_t n, size_t b) {
  return orb_pair_send_coalesced(P(v), (const orb_slice*)s, n, b);
}
static int c_submit(const b200_send_op* s, size_t ns, uint64_t* acc, const b200_recv_op* r, size_t nr, uint64_t* del,
                    int flags) {
  for (size_t i = 0; i < ns; i++) {
    orb_pair* p = P(s[i].pair);
    acc[i] = (flags & B200_BATCH_UNTIL_BLOCKED)
                 ? orb_pair_send_coalesced_all(p, (const orb_slice*)s[i].slices, s[i].nslices, s[i].byte_idx, NULL)
                 : orb_pair_send_coalesced(p, (const orb_slice*)s[i].slices, s[i].nslices, s[i].byte_idx);
  }
  for (size_t i = 0; i < nr; i++) {
    orb_pair* p = P(r[i].pair);
    del[i] = (flags & B200_BATCH_UNTIL_BLOCKED) ? orb_pair_recv_drain(p, r[i].dst, r[i].cap, NULL)
                                                : orb_pair_recv(p, r[i].dst, r[i].cap);
  }
  return 0;
}

static b200_pair_ops g_ops, g_ops_batch;

void coalesce_ops_config(uint64_t ring_bytes) { oracle_ops_config(ring_bytes, 30); }

const b200_pair_ops* coalesce_pair_ops(void) {
  g_ops = *oracle_pair_ops();
  g_ops.send = c_send;
  return &g_ops;
}
const b200_pair_ops* coalesce_pair_ops_batch(void) {
  g_ops_batch = *oracle_pair_ops_batch();
  g_ops_batch.send = c_send;
  g_ops_batch.submit = c_submit;
  return &g_ops_batch;
}
