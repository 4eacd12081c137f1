/*
 * cpu_ref.c - CPU restatement of the hot path at the C-ABI level (ORACLE, TEST INFRASTRUCTURE ONLY).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * link or call this file.  The shipped product (swarmdb_b200/) never does.
 *
 * It restates what the reference's path does to a message, with agents/groups as dense
 * indices exactly as include/swarmdb_b200.h numbers them (tag M: = /root/reference/swarmdb/" main.py"):
 *
 *   send_message     M:393-519   one record appended to the topic log; the receiver is the
 *                                only consumer whose filter (M:579-585) accepts it
 *   send_to_group    M:1229-1279 for each member != sender, in list order: send_message
 *                                (M:1267-1277); duplicates deliver twice
 *   broadcast        M:449-463   one record, visible to an explicit agent list
 *   receive_messages M:521-601   walk the log from this consumer's offset, keep matching
 *                                records, stop after max_messages (M:553-556)
 *
 * Because the filter only ever accepts records addressed to (or listing) the agent, walking
 * the single-partition log from the agent's offset is equivalent to popping from a
 * per-agent FIFO of the accepted records in log order; that is the data structure here.
 * Priority receive (SURVEY App. A rule 9, an extension the reference does not define):
 * the first k pending records in (priority desc, arrival asc) order.
 *
 * PINNING: tests/test_oracle_c.py replays the golden scenarios (produced by the unmodified
 * reference class) through this file and requires identical per-agent streams.
 *
 * Sequence numbers, header layout and padding follow the ABI contract in
 * include/swarmdb_b200.h (they are part of the boundary, not of the reference).
 */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/swarmdb_b200.h"

typedef struct {
  sdb_msg_header hdr;
  uint64_t pay_off;     /* offset into the payload store */
} orc_rec;

typedef struct {
  uint64_t* idx;        /* indices into recs[], arrival order */
  uint8_t* done;        /* consumed flag per entry (priority receive leaves holes) */
  uint64_t n, cap, head;
} orc_inbox;

typedef struct orc {
  uint32_t max_agents, max_groups;
  orc_rec* recs; uint64_t n_recs, cap_recs;
  uint8_t* store; uint64_t n_store, cap_store;
  orc_inbox* inbox;
  uint32_t** gmem; uint32_t* gcnt; uint8_t* gdef;
  uint32_t** gposv;       /* optional: position of each kept member in the full (unsharded) list */
  uint64_t next_seq;
  uint32_t watermark;
  void* mt;               /* persistent context of the multi-threaded baseline path */
  uint64_t* digest;       /* optional [max_agents]: order-sensitive digest of every record delivered to the agent */
  /* balancer */
  uint32_t n_backends; uint32_t* weight; uint64_t* load;
  uint32_t logtab[257];
} orc;

static void* xrealloc(void* p, size_t n) { void* q = realloc(p, n ? n : 1); if (!q) abort(); return q; }
static uint32_t pad32(uint32_t x) { return (x + 31u) & ~31u; }

static void build_log2_table(uint32_t* tab) {
  /* log2(1 + i/256) in Q24, integer only: 26 fractional bits by repeated squaring, rounded */
  for (uint32_t i = 0; i < 256; ++i) {
    unsigned __int128 x = (unsigned __int128)(256 + i) << 54;           /* Q62 */
    const unsigned __int128 two = (unsigned __int128)2 << 62;
    uint32_t r = 0;
    for (int k = 0; k < 26; ++k) { x = (x * x) >> 62; r <<= 1; if (x >= two) { r |= 1u; x >>= 1; } }
    tab[i] = (r + 2u) >> 2;
  }
  tab[256] = 1u << 24;
}
void orc_log2_table(uint32_t* tab257) { build_log2_table(tab257); }

/* ---- per-agent stream digest (definition: include/swarmdb_b200.h, "stream digest") -------------------------
 * rec_hash = sum over the 64-bit little-endian words w_k (k = 0..) of [32-byte header | payload padded to 32 bytes]
 *            of fmix64(w_k ^ ((k + 1) * 0x9E3779B97F4A7C15)),  mod 2^64   (position-keyed, so word order matters)
 * chain    : d <- (rotl64(d, 5) ^ rec_hash) * 0x9E3779B97F4A7C15,  d starts at 0   (so delivery order matters)
 * It is how per-agent delivery order + every header field + every payload byte are compared at sizes where
 * keeping both full result sets is impractical (1M agents, 10^7..10^8 records, several GPUs). */
static uint64_t fmix64(uint64_t x) {
  x ^= x >> 33; x *= 0xFF51AFD7ED558CCDull; x ^= x >> 33; x *= 0xC4CEB9FE1A85EC53ull; x ^= x >> 33;
  return x;
}
static uint64_t rec_hash(const sdb_msg_header* h, const uint8_t* payload_padded) {
  uint64_t w[4], acc = 0;
  memcpy(w, h, 32);
  for (uint32_t k = 0; k < 4; ++k) acc += fmix64(w[k] ^ ((uint64_t)(k + 1) * 0x9E3779B97F4A7C15ull));
  const uint32_t nw = pad32(h->len) / 8;
  for (uint32_t k = 0; k < nw; ++k) {
    uint64_t x; memcpy(&x, payload_padded + 8ull * k, 8);
    acc += fmix64(x ^ ((uint64_t)(k + 5) * 0x9E3779B97F4A7C15ull));
  }
  return acc;
}
static uint64_t digest_chain(uint64_t d, uint64_t rh) {
  return (((d << 5) | (d >> 59)) ^ rh) * 0x9E3779B97F4A7C15ull;
}

orc* orc_create(uint32_t max_agents, uint32_t max_groups) {
  orc* o = (orc*)calloc(1, sizeof(orc));
  o->max_agents = max_agents; o->max_groups = max_groups ? max_groups : 1;
  o->inbox = (orc_inbox*)calloc(max_agents, sizeof(orc_inbox));
  o->gmem = (uint32_t**)calloc(o->max_groups, sizeof(uint32_t*));
  o->gcnt = (uint32_t*)calloc(o->max_groups, sizeof(uint32_t));
  o->gdef = (uint8_t*)calloc(o->max_groups, 1);
  o->gposv = (uint32_t**)calloc(o->max_groups, sizeof(uint32_t*));
  o->next_seq = 1;
  build_log2_table(o->logtab);
  return o;
}

static void mt_free_any(void* m);
void orc_destroy(orc* o) {
  if (!o) return;
  mt_free_any(o->mt);
  for (uint32_t a = 0; a < o->max_agents; ++a) { free(o->inbox[a].idx); free(o->inbox[a].done); }
  for (uint32_t g = 0; g < o->max_groups; ++g) { free(o->gmem[g]); free(o->gposv[g]); }
  free(o->gposv); free(o->inbox); free(o->gmem); free(o->gcnt); free(o->gdef); free(o->recs); free(o->store);
  free(o->weight); free(o->load); free(o->digest); free(o);
}

void orc_register(orc* o, uint32_t a) { if (a < o->max_agents && a + 1 > o->watermark) o->watermark = a + 1; }

/* add_agent_group, M:1208-1227: overwrite, no validation, duplicates kept */
int orc_create_group(orc* o, uint32_t g, uint32_t n, const uint32_t* members) {
  if (g >= o->max_groups) return -1;
  o->gmem[g] = (uint32_t*)xrealloc(o->gmem[g], (size_t)n * 4);
  memcpy(o->gmem[g], members, (size_t)n * 4);
  o->gcnt[g] = n; o->gdef[g] = 1;
  for (uint32_t i = 0; i < n; ++i) orc_register(o, members[i]);
  return 0;
}

static uint64_t store_payload(orc* o, const uint8_t* p, uint32_t len) {
  const uint32_t pl = pad32(len);
  if (o->n_store + pl > o->cap_store) {
    o->cap_store = (o->n_store + pl) * 2 + 4096;
    o->store = (uint8_t*)xrealloc(o->store, o->cap_store);
  }
  const uint64_t off = o->n_store;
  memcpy(o->store + off, p, len);
  memset(o->store + off + len, 0, pl - len);
  o->n_store += pl;
  return off;
}

/* sharded restatement: a shard keeps only the members it owns, with their original positions */
int orc_create_group_pos(orc* o, uint32_t g, uint32_t n, const uint32_t* members, const uint32_t* pos) {
  if (orc_create_group(o, g, n, members) != 0) return -1;
  o->gposv[g] = (uint32_t*)xrealloc(o->gposv[g], (size_t)n * 4);
  memcpy(o->gposv[g], pos, (size_t)n * 4);
  return 0;
}
void orc_set_next_seq(orc* o, uint64_t s) { o->next_seq = s; }
uint64_t orc_get_next_seq(orc* o) { return o->next_seq; }

/* one delivery: the record lands in agent a's stream (the consumer whose filter accepts it) */
static void deliver(orc* o, uint32_t a, uint64_t seq, double ts, uint32_t sender, uint32_t receiver_field,
                    uint32_t group, uint16_t len, uint8_t prio, uint8_t type, uint64_t pay_off) {
  if (o->n_recs == o->cap_recs) { o->cap_recs = o->cap_recs * 2 + 1024; o->recs = (orc_rec*)xrealloc(o->recs, o->cap_recs * sizeof(orc_rec)); }
  orc_rec* r = &o->recs[o->n_recs];
  r->hdr.seq = seq; r->hdr.timestamp = ts; r->hdr.sender = sender; r->hdr.receiver = receiver_field;
  r->hdr.group = group; r->hdr.len = len; r->hdr.prio = prio; r->hdr.type = type; r->pay_off = pay_off;
  orc_inbox* in = &o->inbox[a];
  if (in->n == in->cap) {
    in->cap = in->cap * 2 + 8;
    in->idx = (uint64_t*)xrealloc(in->idx, in->cap * 8);
    in->done = (uint8_t*)xrealloc(in->done, in->cap);
  }
  in->idx[in->n] = o->n_recs; in->done[in->n] = 0; in->n++;
  o->n_recs++;
}

/* send_message x n, M:393-519; returns seq base */
uint64_t orc_send_batch(orc* o, uint32_t n, const uint32_t* sender, const uint32_t* receiver, const uint8_t* prio,
                        const uint8_t* type, const uint16_t* len, const uint64_t* payload_off, const uint8_t* payload,
                        const double* ts) {
  const uint64_t base = o->next_seq;
  for (uint32_t i = 0; i < n; ++i) {
    const uint64_t po = store_payload(o, payload + (payload_off ? payload_off[i] : 0), len[i]);
    orc_register(o, sender[i]); orc_register(o, receiver[i]);                 /* auto-registration M:419-427 */
    deliver(o, receiver[i], base + i, ts ? ts[i] : 0.0, sender[i], receiver[i], SDB_NO_GROUP, len[i],
            prio ? prio[i] : 1, type ? type[i] : 0, po);
  }
  o->next_seq += n;
  return base;
}

/* send_to_group x n, M:1229-1279 */
uint64_t orc_send_group_batch(orc* o, uint32_t n, const uint32_t* sender, const uint32_t* group, const uint8_t* prio,
                              const uint8_t* type, const uint16_t* len, const uint64_t* payload_off,
                              const uint8_t* payload, const double* ts, uint64_t* n_routed) {
  const uint64_t base = o->next_seq;
  uint64_t rec = 0, routed = 0;
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t g = group[i];
    if (g >= o->max_groups || !o->gdef[g]) continue;                           /* unknown group -> [] (M:1255-1257) */
    const uint64_t po = store_payload(o, payload + (payload_off ? payload_off[i] : 0), len[i]);
    for (uint32_t j = 0; j < o->gcnt[g]; ++j) {                                 /* member order, M:1267 */
      const uint32_t a = o->gmem[g][j];
      if (a != sender[i]) {                                                     /* M:1268 */
        deliver(o, a, base + rec + j, ts ? ts[i] : 0.0, sender[i], a, g, len[i], prio ? prio[i] : 1,
                type ? type[i] : 0, po);
        ++routed;
      }
    }
    rec += o->gcnt[g];
  }
  o->next_seq += rec;
  if (n_routed) *n_routed = routed;
  return base;
}

/* group sends whose sequence numbers were assigned elsewhere (cross-shard import): member k of
 * the locally kept list gets seq0[i] + original position; the rest is send_to_group (M:1267-1277) */
void orc_send_group_seq(orc* o, uint32_t n, const uint32_t* sender, const uint32_t* group, const uint8_t* prio,
                        const uint8_t* type, const uint16_t* len, const uint64_t* payload_off, const uint8_t* payload,
                        const double* ts, const uint64_t* seq0) {
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t g = group[i];
    if (g >= o->max_groups || !o->gdef[g]) continue;
    const uint64_t po = store_payload(o, payload + (payload_off ? payload_off[i] : 0), len[i]);
    for (uint32_t k = 0; k < o->gcnt[g]; ++k) {
      const uint32_t a = o->gmem[g][k];
      const uint32_t j = o->gposv[g] ? o->gposv[g][k] : k;
      if (a != sender[i])
        deliver(o, a, seq0[i] + j, ts ? ts[i] : 0.0, sender[i], a, g, len[i], prio ? prio[i] : 1, type ? type[i] : 0, po);
    }
  }
}

/* broadcast with explicit visibility list, M:449-463 / M:810-850: ONE message, many readers */
uint64_t orc_send_list_batch(orc* o, uint32_t n, const uint32_t* sender, const uint64_t* list_off, const uint32_t* list_idx,
                             const uint8_t* prio, const uint8_t* type, const uint16_t* len, const uint64_t* payload_off,
                             const uint8_t* payload, const double* ts) {
  const uint64_t base = o->next_seq;
  for (uint32_t i = 0; i < n; ++i) {
    const uint64_t po = store_payload(o, payload + (payload_off ? payload_off[i] : 0), len[i]);
    for (uint64_t k = list_off[i]; k < list_off[i + 1]; ++k)
      deliver(o, list_idx[k], base + i, ts ? ts[i] : 0.0, sender[i], SDB_NO_RECEIVER, SDB_NO_GROUP, len[i],
              prio ? prio[i] : 1, type ? type[i] : 0, po);
  }
  o->next_seq += n;
  return base;
}

/* receive_messages for a list of agents, M:521-601.  Output format of sdb_receive_batch.
 * SDB_RECV_PEEK (extension, include/swarmdb_b200.h): the same selection, nothing is consumed. */
uint64_t orc_receive_batch(orc* o, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages, uint32_t flags,
                           uint32_t* count_out, sdb_msg_header* hdr_out, uint8_t* payload_out, uint64_t* payload_bytes) {
  uint64_t total = 0, pbytes = 0;
  const int peek = (flags & SDB_RECV_PEEK) != 0;
  if (!agent_idx) n_agents = o->watermark;
  for (uint32_t q = 0; q < n_agents; ++q) {
    const uint32_t a = agent_idx ? agent_idx[q] : q;
    orc_inbox* in = &o->inbox[a];
    uint32_t got = 0;
    /* stream order = one pass; priority order = one pass per level, highest first (App. A rule 9) */
    for (int L = (flags & SDB_RECV_PRIORITY) ? 3 : 0; L >= 0 && got < max_messages; --L)
      for (uint64_t p = in->head; p < in->n && got < max_messages; ++p) {
        if (in->done[p]) continue;
        const orc_rec* r = &o->recs[in->idx[p]];
        if ((flags & SDB_RECV_PRIORITY) && r->hdr.prio != (uint8_t)L) continue;
        if (!peek) in->done[p] = 1;
        if (o->digest) o->digest[a] = digest_chain(o->digest[a], rec_hash(&r->hdr, o->store + r->pay_off));
        if (hdr_out) hdr_out[total] = r->hdr;
        if (payload_out) memcpy(payload_out + pbytes, o->store + r->pay_off, pad32(r->hdr.len));
        pbytes += pad32(r->hdr.len); ++total; ++got;
      }
    while (in->head < in->n && in->done[in->head]) in->head++;
    if (count_out) count_out[q] = got;
  }
  if (payload_bytes) *payload_bytes = pbytes;
  return total;
}

uint64_t orc_pending(orc* o, uint32_t a) {
  orc_inbox* in = &o->inbox[a];
  uint64_t c = 0;
  for (uint64_t p = in->head; p < in->n; ++p) c += !in->done[p];
  return c;
}

/* inbox / load queries (include/swarmdb_b200.h sdb_agent_loads; reference: get_agent_load M:1049-1094, get_unread_message_count
 * M:1026-1047): received = records ever enqueued for the agent (len(agent_inbox[a]), M:1076), pending = not yet received */
void orc_agent_loads(orc* o, uint32_t n, const uint32_t* agent_idx, sdb_agent_load* out) {
  for (uint32_t q = 0; q < n; ++q) {
    const uint32_t a = agent_idx ? agent_idx[q] : q;
    sdb_agent_load r; memset(&r, 0, sizeof(r));
    if (a < o->max_agents) {
      const orc_inbox* in = &o->inbox[a];
      r.received = (uint32_t)in->n;
      for (uint64_t p = in->head; p < in->n; ++p) if (!in->done[p]) {
        const orc_rec* rec = &o->recs[in->idx[p]];
        r.pending++; r.pending_by_prio[rec->hdr.prio & 3]++; r.pending_granules += pad32(rec->hdr.len) / 32;
      }
    }
    out[q] = r;
  }
}

/* digests: enable (allocates, zeroed) / reset / read.  Folding happens inside orc_receive_batch and the MT drain. */
void orc_digest_enable(orc* o) {
  if (!o->digest) o->digest = (uint64_t*)calloc(o->max_agents, 8);
  else memset(o->digest, 0, (size_t)o->max_agents * 8);
}
void orc_digest_read(orc* o, uint32_t n, const uint32_t* agent_idx, uint64_t* out) {
  for (uint32_t q = 0; q < n; ++q) { const uint32_t a = agent_idx ? agent_idx[q] : q; out[q] = (o->digest && a < o->max_agents) ? o->digest[a] : 0; }
}

/* ---- balancer (definition in include/swarmdb_b200.h; the reference has none, M:1281-1325) ---- */
void orc_set_backends(orc* o, uint32_t n, const uint32_t* weight, const uint64_t* load0) {
  o->n_backends = n;
  o->weight = (uint32_t*)xrealloc(o->weight, (size_t)n * 4);
  o->load = (uint64_t*)xrealloc(o->load, (size_t)n * 8);
  for (uint32_t b = 0; b < n; ++b) { o->weight[b] = weight[b]; o->load[b] = load0 ? load0[b] : 0; }
}
void orc_get_backend_loads(orc* o, uint64_t* out) { memcpy(out, o->load, (size_t)o->n_backends * 8); }

static uint64_t mix(uint64_t seed, uint32_t t, uint32_t b) {
  uint64_t x = seed ^ ((uint64_t)t + 1ull) * 0x9E3779B97F4A7C15ull;
  x ^= ((uint64_t)b + 1ull) * 0xD1B54A32D192ED03ull;
  x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ull;
  x ^= x >> 27; x *= 0x94D049BB133111EBull;
  x ^= x >> 31;
  return x;
}
static uint32_t neglog2_q24(uint32_t u, const uint32_t* tab) {
  const uint32_t lz = (uint32_t)__builtin_clz(u);
  const uint32_t un = u << lz;
  const uint32_t idx = (un >> 23) & 0xFFu, frac = un & 0x7FFFFFu;
  const uint32_t lg = tab[idx] + (uint32_t)(((uint64_t)(tab[idx + 1] - tab[idx]) * frac) >> 23);
  return ((1u + lz) << 24) - lg;
}

void orc_select_backend_batch(orc* o, uint32_t n_req, const uint32_t* cost, uint32_t mode, uint64_t seed, uint32_t* out) {
  const uint32_t B = o->n_backends;
  if (mode == 0) {
    /* sequential greedy: argmin load/weight, exact rational compare, ties -> lowest index */
    for (uint32_t t = 0; t < n_req; ++t) {
      uint32_t best = 0;
      for (uint32_t b = 1; b < B; ++b)
        if ((unsigned __int128)o->load[b] * o->weight[best] < (unsigned __int128)o->load[best] * o->weight[b]) best = b;
      out[t] = best;
      o->load[best] += cost ? cost[t] : 1u;
    }
  } else {
    for (uint32_t t = 0; t < n_req; ++t) {
      uint32_t best = 0, bw = 1; uint64_t bk = 0; int have = 0;
      for (uint32_t b = 0; b < B; ++b) {
        const uint32_t u = (uint32_t)(mix(seed, t, b) >> 32) | 1u;
        const uint64_t k = neglog2_q24(u, o->logtab);
        if (!have || k * bw < bk * o->weight[b]) { bk = k; bw = o->weight[b]; best = b; have = 1; }
      }
      out[t] = best;
    }
    for (uint32_t t = 0; t < n_req; ++t) o->load[out[t]] += cost ? cost[t] : 1u;
  }
}

/* ---- multi-threaded group fan-out + drain for the CPU baseline --------------------------------
 * A three-phase pipeline over T threads, all buffers persistent across calls (no allocation in the timed path
 * after the first batch):
 *   route        thread k takes the k-th contiguous slice of the sends and, for every member != sender (M:1268),
 *                pushes (send, position) into bucket[k][receiver % T]          - every membership touched once;
 *   materialise  thread d walks bucket[0..T-1][d] in that order (= global send order) and writes each record
 *                (32-byte header + padded payload - the work a CPU queue does per routed message) into its own
 *                arena, appending the record to the receiver's list: every inbox has exactly one writer, in send
 *                order, so the streams equal the single-threaded path - no locks;
 *   drain        thread d copies the first max_messages records of each of its agents to an output buffer
 *                (and folds them into the stream digests when those are enabled). */
typedef struct { uint32_t send, pos; } mt_ref;
typedef struct { mt_ref* v; uint32_t n, cap; } mt_bucket;
typedef struct {
  struct orc_mt* m; uint32_t tid;
  uint8_t* arena; uint64_t arena_cap, arena_used; uint64_t** lists; uint32_t* lcnt; uint32_t* lcap;
  uint64_t routed, drained, checksum; uint8_t* out; uint64_t out_cap;
} mt_task;
typedef struct orc_mt {
  orc* o; uint32_t T, slots;
  mt_task* ts; pthread_t* th; mt_bucket* bucket;         /* bucket[k * T + d] */
  uint64_t* rec0; uint32_t rec0_cap;
  /* the batch being processed */
  uint32_t n; const uint32_t* sender; const uint32_t* group; const uint8_t* prio; const uint8_t* type;
  const uint16_t* len; const uint64_t* payload_off; const uint8_t* payload; uint64_t seq_base; uint32_t max_messages;
} orc_mt;

static void* mt_route(void* p) {
  mt_task* t = (mt_task*)p; orc_mt* m = t->m; orc* o = m->o;
  const uint32_t T = m->T;
  const uint32_t lo = (uint32_t)((uint64_t)m->n * t->tid / T), hi = (uint32_t)((uint64_t)m->n * (t->tid + 1) / T);
  mt_bucket* row = m->bucket + (size_t)t->tid * T;
  for (uint32_t d = 0; d < T; ++d) row[d].n = 0;
  for (uint32_t i = lo; i < hi; ++i) {
    const uint32_t g = m->group[i];
    const uint32_t* mem = o->gmem[g];
    for (uint32_t j = 0; j < o->gcnt[g]; ++j) {
      const uint32_t a = mem[j];
      if (a == m->sender[i]) continue;                             /* M:1268 */
      mt_bucket* b = &row[a % T];
      if (b->n == b->cap) { b->cap = b->cap * 2 + 64; b->v = (mt_ref*)xrealloc(b->v, (size_t)b->cap * sizeof(mt_ref)); }
      b->v[b->n].send = i; b->v[b->n].pos = j; b->n++;
    }
  }
  return NULL;
}

static void* mt_materialise(void* p) {
  mt_task* t = (mt_task*)p; orc_mt* m = t->m; orc* o = m->o;
  const uint32_t T = m->T;
  uint64_t need = 0;
  for (uint32_t k = 0; k < T; ++k) {
    const mt_bucket* b = &m->bucket[(size_t)k * T + t->tid];
    for (uint32_t e = 0; e < b->n; ++e) need += 32 + pad32(m->len[b->v[e].send]);
  }
  if (need > t->arena_cap) { t->arena_cap = need + need / 4 + (1u << 20); t->arena = (uint8_t*)xrealloc(t->arena, t->arena_cap); }
  t->arena_used = 0; t->routed = 0;
  for (uint32_t k = 0; k < T; ++k) {
    const mt_bucket* b = &m->bucket[(size_t)k * T + t->tid];
    for (uint32_t e = 0; e < b->n; ++e) {
      const uint32_t i = b->v[e].send, j = b->v[e].pos, g = m->group[i], a = o->gmem[g][j];
      const uint32_t pl = pad32(m->len[i]);
      uint8_t* rec = t->arena + t->arena_used;
      sdb_msg_header h; h.seq = m->seq_base + m->rec0[i] + j; h.timestamp = 0.0; h.sender = m->sender[i]; h.receiver = a;
      h.group = g; h.len = m->len[i]; h.prio = m->prio[i]; h.type = m->type[i];
      memcpy(rec, &h, 32);
      memcpy(rec + 32, m->payload + m->payload_off[i], m->len[i]);
      memset(rec + 32 + m->len[i], 0, pl - m->len[i]);
      const uint32_t slot = a / T;
      if (t->lcnt[slot] == t->lcap[slot]) {
        t->lcap[slot] = t->lcap[slot] * 2 + 8;
        t->lists[slot] = (uint64_t*)xrealloc(t->lists[slot], (size_t)t->lcap[slot] * 8);
      }
      t->lists[slot][t->lcnt[slot]++] = t->arena_used;
      t->arena_used += 32 + pl;
      t->routed++;
    }
  }
  return NULL;
}

static void* mt_drain(void* p) {
  mt_task* t = (mt_task*)p; orc_mt* m = t->m;
  uint64_t used = 0, sum = 0;
  t->drained = 0;
  for (uint32_t s = 0; s < m->slots; ++s) {
    const uint32_t k = t->lcnt[s] < m->max_messages ? t->lcnt[s] : m->max_messages;
    for (uint32_t e = 0; e < k; ++e) {
      const uint8_t* rec = t->arena + t->lists[s][e];
      const sdb_msg_header* h = (const sdb_msg_header*)rec;
      const uint32_t sz = 32 + pad32(h->len);
      if (used + sz > t->out_cap) used = 0;                       /* ring the output buffer */
      memcpy(t->out + used, rec, sz);
      if (m->o->digest) { uint64_t* d = &m->o->digest[(uint64_t)s * m->T + t->tid]; *d = digest_chain(*d, rec_hash(h, rec + 32)); }
      used += sz; sum += h->seq; t->drained++;
    }
    t->lcnt[s] = 0;
  }
  t->checksum = sum;
  return NULL;
}

static void mt_free(orc_mt* m) {
  if (!m) return;
  for (uint32_t k = 0; k < m->T; ++k) {
    for (uint32_t s = 0; s < m->slots; ++s) free(m->ts[k].lists[s]);
    free(m->ts[k].lists); free(m->ts[k].lcnt); free(m->ts[k].lcap); free(m->ts[k].arena); free(m->ts[k].out);
  }
  for (size_t b = 0; b < (size_t)m->T * m->T; ++b) free(m->bucket[b].v);
  free(m->bucket); free(m->ts); free(m->th); free(m->rec0); free(m);
}

static void mt_run(orc_mt* m, void* (*fn)(void*)) {
  for (uint32_t k = 0; k < m->T; ++k) pthread_create(&m->th[k], NULL, fn, &m->ts[k]);
  for (uint32_t k = 0; k < m->T; ++k) pthread_join(m->th[k], NULL);
}

/* Returns routed records; *drained_out and *checksum_out (sum of seq of drained records) verify the work. */
uint64_t orc_mt_group_roundtrip(orc* o, uint32_t T, uint32_t n, const uint32_t* sender, const uint32_t* group,
                                const uint8_t* prio, const uint8_t* type, const uint16_t* len, const uint64_t* payload_off,
                                const uint8_t* payload, uint32_t max_messages, uint64_t* drained_out, uint64_t* checksum_out) {
  if (T == 0) T = 1;
  orc_mt* m = (orc_mt*)o->mt;
  if (m && m->T != T) { mt_free(m); m = NULL; }
  if (!m) {
    m = (orc_mt*)calloc(1, sizeof(orc_mt));
    m->o = o; m->T = T; m->slots = (o->max_agents + T - 1) / T;
    m->ts = (mt_task*)calloc(T, sizeof(mt_task)); m->th = (pthread_t*)calloc(T, sizeof(pthread_t));
    m->bucket = (mt_bucket*)calloc((size_t)T * T, sizeof(mt_bucket));
    for (uint32_t k = 0; k < T; ++k) {
      mt_task* t = &m->ts[k];
      t->m = m; t->tid = k;
      t->lists = (uint64_t**)calloc(m->slots, sizeof(uint64_t*)); t->lcnt = (uint32_t*)calloc(m->slots, 4); t->lcap = (uint32_t*)calloc(m->slots, 4);
      t->out_cap = 64u << 20; t->out = (uint8_t*)malloc(t->out_cap);
    }
    o->mt = m;
  }
  if (n > m->rec0_cap) { m->rec0_cap = n; m->rec0 = (uint64_t*)xrealloc(m->rec0, (size_t)n * 8); }
  uint64_t rec = 0;
  for (uint32_t i = 0; i < n; ++i) { m->rec0[i] = rec; rec += o->gcnt[group[i]]; }
  m->n = n; m->sender = sender; m->group = group; m->prio = prio; m->type = type; m->len = len;
  m->payload_off = payload_off; m->payload = payload; m->seq_base = o->next_seq; m->max_messages = max_messages;
  mt_run(m, mt_route);
  mt_run(m, mt_materialise);
  mt_run(m, mt_drain);
  uint64_t routed = 0, drained = 0, sum = 0;
  for (uint32_t k = 0; k < T; ++k) { routed += m->ts[k].routed; drained += m->ts[k].drained; sum += m->ts[k].checksum; }
  o->next_seq += rec;
  if (drained_out) *drained_out = drained;
  if (checksum_out) *checksum_out = sum;
  return routed;
}

static void mt_free_any(void* m) { mt_free((orc_mt*)m); }
