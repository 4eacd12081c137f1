/*
 * swarmdb_b200.h - C ABI of the H100-native agent message queue + backend balancer.
 *
 * This is the drop-in boundary for the hot path of The-Swarm-Corporation/SwarmDB
 * (reference class `SwarmsDB` in /root/reference/swarmdb/" main.py", tag `M:`).  The
 * reference has no FFI of its own: its `SwarmsDB` methods call the third-party
 * `confluent_kafka` client (librdkafka) directly.  Each entry point below replaces one
 * reference method body plus the Kafka client calls it makes; the file:line it replaces is
 * cited on every declaration.  INTEGRATION.md shows the ctypes binding a maintainer adds.
 *
 * Conventions
 *   - plain C: opaque handle, POD structs, pointers and sizes; no C++/torch types.
 *   - every function returns 0 (SDB_OK) or a negative sdb_status; sdb_last_error(h)
 *     returns a human-readable string for the last failure on that handle.
 *   - a handle is NOT thread-safe (the reference class has no locks either, SURVEY 8b);
 *     one handle drives one GPU (one shard).  One process per GPU.
 *   - pointer arguments are caller-owned HOST buffers unless the name ends in `_dev`.
 *   - calls are stream-ordered on the handle's CUDA stream; functions that return
 *     data to the host synchronise that stream before returning, others may return early.
 *   - agents, groups and backends are dense uint32 indices; the string ids of the Python
 *     surface are mapped by the caller (swarmdb_b200/core.py keeps the dict, as the
 *     reference keeps `registered_agents`, M:233).
 *   - there is NO CPU fallback: without a CUDA device sdb_create fails with SDB_ECUDA.
 */
#ifndef SWARMDB_B200_H
#define SWARMDB_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SDB_ABI_VERSION 1u
#define SDB_GRANULE 32u                 /* arena allocation unit, bytes (one DRAM sector) */
#define SDB_NO_GROUP 0xFFFFFFFFu        /* header.group when the message was not a group send */
#define SDB_NO_RECEIVER 0xFFFFFFFFu     /* header.receiver for broadcast records (receiver_id=None, M:61) */

typedef struct sdb_ctx* sdb_handle;

typedef enum sdb_status {
  SDB_OK = 0,
  SDB_EINVAL = -1,         /* bad argument (index out of range, misaligned offset, ...) */
  SDB_ECUDA = -2,          /* CUDA runtime failure (incl. no device) */
  SDB_ENOMEM = -3,         /* host or device allocation failed */
  SDB_ERING_OVERFLOW = -4, /* some receiver's ring was full: those records were NOT enqueued (counted) */
  SDB_EARENA_FULL = -5,    /* message arena cannot hold the batch even after reclaiming consumed space */
  SDB_ECAPACITY = -6,      /* batch larger than the configured staging capacity */
  SDB_ENOTFOUND = -7,      /* unknown group / backend */
  SDB_EOUTPUT = -8         /* caller's output buffer too small */
} sdb_status;

/* Message vocabularies, M:23-51.  Device codes; names in swarmdb_b200/core.py. */
enum { SDB_PRIO_LOW = 0, SDB_PRIO_NORMAL = 1, SDB_PRIO_HIGH = 2, SDB_PRIO_CRITICAL = 3 };
enum { SDB_TYPE_CHAT = 0, SDB_TYPE_COMMAND, SDB_TYPE_FUNCTION_CALL, SDB_TYPE_FUNCTION_RESULT,
       SDB_TYPE_SYSTEM, SDB_TYPE_ERROR, SDB_TYPE_STATUS };
#define SDB_TYPE_MASK 0x07u
#define SDB_TYPEF_JSON 0x08u            /* payload content is JSON (dict/list content, M:75) */
#define SDB_TYPEF_EXTRAS 0x10u          /* payload = u32 content_len | content | JSON extras */
#define SDB_TYPEF_SUPERSEDE 0x20u       /* superseding: a newer flagged record with the same (sender, group, type) replaces it (sdb_supersede) */
#define SDB_TYPEF_TOKENS 0x40u          /* payload = u32 token count (little-endian) | the payload without this flag; len counts
                                           the 4 bytes.  The record weighs that many tokens in sdb_receive_tokens (a record
                                           without the flag, or with len < 4, weighs 0) */

/* Replaces KafkaConfig (M:114-127) + SwarmsDB.__init__ kwargs (M:156-165) for the device side. */
typedef struct sdb_config {
  uint32_t struct_bytes;        /* sizeof(sdb_config), ABI check */
  int32_t  device;              /* CUDA ordinal */
  uint32_t shard_id;            /* this process's shard (== rank) */
  uint32_t num_shards;          /* replaces num_partitions (M:121): 1, 2, 4 or 8 */
  uint32_t max_agents;          /* size of the global agent index space */
  uint32_t ring_slots;          /* per-agent ring capacity in messages, power of two */
  uint64_t arena_bytes;         /* message arena, power of two */
  uint32_t max_payload_bytes;   /* largest payload accepted (<= 65504) */
  uint32_t max_groups;
  uint64_t member_pool_entries; /* total group-member slots (groups may be re-created) */
  uint32_t max_backends;
  uint32_t max_batch_sends;     /* staging capacity: sends per batch */
  uint64_t max_batch_payload;   /* staging capacity: payload bytes per batch */
  uint64_t max_recv_records;    /* receive output capacity, records per call */
  uint64_t max_recv_payload;    /* receive output capacity, payload bytes per call (0: records x 256) */
  uint64_t list_pool_entries;   /* per-batch broadcast recipient-list capacity (0: 2 x max_agents) */
  uint32_t fanout_variant;      /* 2 (recommended): warp-per-send, TMA-in / coalesced stores - imports of wire batches use the deep-prefetch form;
                                   3: deep-prefetch warp-per-send everywhere (payloads <= 480 B); 0: CTA-per-send; 1: TMA-in / TMA-out */
  uint32_t flags;               /* reserved, 0 */
} sdb_config;

/* One message as stored in the arena and returned by receive: 32-byte header followed by
 * the payload padded to SDB_GRANULE.  Field set = the device-relevant subset of `Message`
 * (M:54-82): id <-> seq, sender_id, receiver_id, type, priority, timestamp, metadata["group"]. */
typedef struct sdb_msg_header {
  uint64_t seq;        /* message identity; ids are derived from it (replaces uuid4, M:72) */
  double   timestamp;  /* M:78, carried, never compared */
  uint32_t sender;     /* agent index */
  uint32_t receiver;   /* agent index this copy was delivered to */
  uint32_t group;      /* group index (M:1264 metadata["group"]) or SDB_NO_GROUP */
  uint16_t len;        /* payload bytes */
  uint8_t  prio;       /* 0..3, M:35-41 */
  uint8_t  type;       /* SDB_TYPE_* | SDB_TYPEF_* */
} sdb_msg_header;

typedef struct sdb_stats {
  uint64_t next_seq;            /* messages created so far (M:454 message_count analogue) */
  uint64_t enqueued;            /* records appended to rings */
  uint64_t delivered;           /* records returned by receive */
  uint64_t ring_overflow;       /* records dropped because a ring was full (reported, never silent) */
  uint64_t skipped_sender;      /* group members skipped because member == sender (M:1268) */
  uint64_t arena_tail_bytes;    /* monotonic arena write position */
  uint64_t arena_floor_bytes;   /* everything below is reclaimed */
  uint64_t n_agents;            /* registered-index watermark */
  uint64_t kernel_launches;     /* CUDA kernels launched by this handle so far */
  uint64_t backend_picks;
} sdb_stats;

/* ---- lifecycle: SwarmsDB.__init__ (M:156-237), close (M:1367-1394) ---------------------- */
int sdb_abi_version(void);
int sdb_create(const sdb_config* cfg, sdb_handle* out);
int sdb_destroy(sdb_handle h);
/* Run on a caller-provided CUDA stream (e.g. torch's current stream) instead of the internal one. */
int sdb_set_stream(sdb_handle h, void* cuda_stream);
int sdb_sync(sdb_handle h);
const char* sdb_last_error(sdb_handle h);
int sdb_get_stats(sdb_handle h, sdb_stats* out);
/* Test hook: move the (empty) arena's write position, e.g. next to the 2^32-granule boundary where the
 * 32-bit ring handles wrap.  Only valid while no message is pending. */
int sdb_debug_set_arena_pos(sdb_handle h, uint64_t granules);
/* Move the sequence counter FORWARD to `next_seq` (no-op when it is already there or beyond).  A front-end that
 * hands out message ids at send time (ids are derived from sequence numbers, replacing uuid4 M:72) calls this when a
 * batch was refused, so the ids of the failed messages (M:501-519: marked FAILED, kept) are never issued twice. */
int sdb_advance_seq(sdb_handle h, uint64_t next_seq);

/* Per-kernel device timing (CUDA events on the handle's stream), used by bench.py for the
 * roofline: enable, run, then read accumulated milliseconds and launch counts per kernel class. */
enum { SDB_PK_P2P = 0, SDB_PK_FANOUT, SDB_PK_COMMIT, SDB_PK_RECV_COUNT, SDB_PK_RECV_SCAN, SDB_PK_RECV_SELECT,
       SDB_PK_RECV_GATHER, SDB_PK_ARENA_FLOOR, SDB_PK_PICK, SDB_PK_XSHARD, SDB_PK_INDEX, SDB_PK_XWAIT,
       SDB_PK_RECV_COMPACT = 12, SDB_PK_EXPIRE = 13, SDB_PK_WHERE = 14, SDB_PK_RESTORE = 15, SDB_PK_N = 16,
       /* classes past SDB_PK_N: sdb_profile_read fills SDB_PK_N entries (the array size of every ABI-1 caller), so
          these are read with sdb_profile_read_n only */
       SDB_PK_LEASE = 16, SDB_PK_ALL = 17,
       /* classes past SDB_PK_ALL (the array size of callers written before them): read with sdb_profile_read_n, whose
          n asks for them; SDB_PK_CLASSES counts every class */
       SDB_PK_DEDUP = 17, SDB_PK_CLASSES = 18 };
int sdb_profile(sdb_handle h, int enable);
int sdb_profile_read(sdb_handle h, double* ms_out /* [SDB_PK_N] */, uint64_t* count_out /* [SDB_PK_N] */);
/* The same for the first min(n, SDB_PK_CLASSES) classes (entries from there to n are zeroed); like sdb_profile_read it
 * consumes the recorded intervals. */
int sdb_profile_read_n(sdb_handle h, uint32_t n, double* ms_out /* [n] */, uint64_t* count_out /* [n] */);

/* ---- registry: register_agent (M:314-349) / deregister_agent (M:351-372) ------------------
 * Rings exist for every index < max_agents; registration only moves the watermark that
 * bounds the per-batch commit sweep.  Deregistration keeps the ring and its read position
 * (the Kafka consumer-group offset survives Consumer.close(), SURVEY App. A rule 11). */
int sdb_register_agents(sdb_handle h, uint32_t n, const uint32_t* agent_idx);
int sdb_deregister_agents(sdb_handle h, uint32_t n, const uint32_t* agent_idx);

/* ---- groups: add_agent_group (M:1208-1227), overwrite semantics, duplicates kept --------- */
int sdb_create_group(sdb_handle h, uint32_t group_idx, uint32_t n_members, const uint32_t* member_idx);

/* ---- enqueue --------------------------------------------------------------------------
 * All three take a batch of `n` sends in call order (struct-of-arrays).  payload_off[i] is a
 * byte offset into `payload`, 16-byte aligned, with len[i] bytes valid and readable up to
 * the next multiple of 16.  Sequence numbers are assigned in array order starting at the
 * handle's next_seq; *seq_base_out (nullable) receives the first one.
 *
 * sdb_send_batch        point-to-point: send_message (M:393-519) -> Producer.produce (M:476-482);
 *                       send i gets seq_base + i.
 * sdb_send_group_batch  send_to_group (M:1229-1279): one copy per member != sender, in member
 *                       order; member j of send i gets seq_base + sum(size of earlier groups) + j
 *                       (ids of skipped members are left unused).
 * sdb_send_list_batch   broadcast (M:449-463, M:810-850): recipient list i is
 *                       list_idx[list_off[i] .. list_off[i+1]); every copy shares ONE seq
 *                       (one Message, one id), receiver field = SDB_NO_RECEIVER.
 */
int sdb_send_batch(sdb_handle h, uint32_t n,
                   const uint32_t* sender, const uint32_t* receiver,
                   const uint8_t* prio, const uint8_t* type, const uint16_t* len,
                   const uint64_t* payload_off, const uint8_t* payload, uint64_t payload_bytes,
                   const double* timestamp /* [n] or NULL = 0.0 */, uint64_t* seq_base_out);
int sdb_send_group_batch(sdb_handle h, uint32_t n,
                         const uint32_t* sender, const uint32_t* group_idx,
                         const uint8_t* prio, const uint8_t* type, const uint16_t* len,
                         const uint64_t* payload_off, const uint8_t* payload, uint64_t payload_bytes,
                         const double* timestamp, uint64_t* seq_base_out);
int sdb_send_list_batch(sdb_handle h, uint32_t n,
                        const uint32_t* sender, const uint64_t* list_off /* [n+1] */, const uint32_t* list_idx,
                        const uint8_t* prio, const uint8_t* type, const uint16_t* len,
                        const uint64_t* payload_off, const uint8_t* payload, uint64_t payload_bytes,
                        const double* timestamp, uint64_t* seq_base_out);

/* Mixed batch in call order - what a host-side send buffer flushes (the reference's producer
 * also batches, linger.ms = 10, M:197).  kind[i]: 0 = point-to-point (target = receiver index),
 * 1 = group send (target = group index), 2 = broadcast list (target = list number t, recipients
 * list_idx[list_off[t] .. list_off[t+1])).  Sequence numbers advance by 1, group size, 1. */
int sdb_send_mixed_batch(sdb_handle h, uint32_t n,
                         const uint32_t* sender, const uint8_t* kind, const uint32_t* target,
                         uint32_t n_lists, const uint64_t* list_off, const uint32_t* list_idx,
                         const uint8_t* prio, const uint8_t* type, const uint16_t* len,
                         const uint64_t* payload_off, const uint8_t* payload, uint64_t payload_bytes,
                         const double* timestamp, uint64_t* seq_base_out);

/* Staged variant used to keep inputs resident in HBM (bench `value` leg): stage copies the
 * batch to device memory once; submit enqueues it (may be repeated; each submit takes fresh
 * sequence numbers).  kind: 0 = p2p (second index array = receiver), 1 = group. */
typedef struct sdb_staged* sdb_staged_t;
int sdb_stage_batch(sdb_handle h, uint32_t kind, uint32_t n,
                    const uint32_t* sender, const uint32_t* receiver_or_group,
                    const uint8_t* prio, const uint8_t* type, const uint16_t* len,
                    const uint64_t* payload_off, const uint8_t* payload, uint64_t payload_bytes,
                    const double* timestamp, sdb_staged_t* out);
int sdb_submit_staged(sdb_handle h, sdb_staged_t s, uint64_t* seq_base_out);
int sdb_free_staged(sdb_handle h, sdb_staged_t s);

/* ---- dequeue: receive_messages (M:521-601) -> Consumer.poll (M:557-559) ------------------
 * For each listed agent (agent_idx == NULL: every index below the registration watermark)
 * remove up to max_messages pending records and return them, agents in list order, records
 * in delivery order.  An agent may appear only once in agent_idx (SDB_EINVAL otherwise).
 * Records are delivered:
 *   flags == 0                 stream (arrival) order - the reference's behaviour;
 *   flags & SDB_RECV_PRIORITY  (priority desc, arrival asc) - the extension of SURVEY
 *                              App. A rule 9; equals stream order when priorities are equal.
 * Outputs (host pointers, each nullable to skip the copy): count_out[n_agents];
 * hdr_out[total]; payload_out = payloads back to back, each padded to SDB_GRANULE, in the
 * same order (offset of record r = sum of pad32(hdr_out[0..r).len)).  *total_out /
 * *payload_bytes_out receive the totals.
 * Capacity: one call returns at most rec_cap = min(max_recv_records,
 * max_recv_payload / P, hdr_cap, payload_cap / P) records, P = pad32(max_payload_bytes)
 * (hdr_cap / payload_cap count only when the pointer is given), so that rec_cap records of
 * the largest size always fit.  The rule is the same on every path (bulk, few-agent and
 * latency server): records are laid out agent by agent in list order; if an agent's records
 * do not all fit, that agent and every later agent are truncated and stay queued, never
 * dropped.  The only exception is an agent that is first in the output (nothing placed
 * before it): it gets its first rec_cap records, in the call's delivery order, and keeps
 * the rest queued.  So every call on a non-empty queue makes progress.
 * sdb_receive_budget (below) bounds each agent's take by bytes and sizes a call by the bytes
 * it actually selects instead of the worst case.
 */
#define SDB_RECV_PRIORITY 1u
#define SDB_RECV_PEEK 2u                /* return what a receive would deliver, retire nothing (history snapshots, M:852-892) */
#define SDB_RECV_ASYNC 4u               /* device-resident consumers: enqueue the receive and return at once; all host output
                                           pointers must be NULL, results stay in the buffers of sdb_last_receive_dev (valid in
                                           stream order), totals through sdb_last_receive_totals */
#define SDB_RECV_OWNED 8u               /* sharded handles, agent_idx == NULL: the agents THIS shard owns (ascending index; count_out has
                                           one entry per owned agent) instead of every index below the watermark - the other agents'
                                           rings are empty here by construction, so nothing is lost and 1/num_shards of the work is done */
int sdb_receive_batch(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx,
                      uint32_t max_messages, uint32_t flags,
                      uint32_t* count_out, sdb_msg_header* hdr_out, uint64_t hdr_cap,
                      uint8_t* payload_out, uint64_t payload_cap,
                      uint64_t* total_out, uint64_t* payload_bytes_out);
/* Compact receive: the records sdb_receive_batch would select and retire, with each distinct payload image
 * returned once.  For host consumers, whose cost is the bytes that cross PCIe: a group send's m records share one
 * payload in the arena (shared layout), and the full format copies that payload out m times.
 *   count_out[n_agents]  as in sdb_receive_batch;
 *   entry_out[total]     one 16-byte entry per record, in sdb_receive_batch's header order (agent by agent,
 *                        delivery order);
 *   send_out[n_sends]    one 32-byte row per distinct payload image;
 *   payload_out          the distinct payloads back to back, each padded to SDB_GRANULE, in row order.
 * Contract:
 *   1. Expansion equals the full receive byte for byte.  With row = send_out[entry.send], record r's header is
 *      {entry.seq, row.timestamp, row.sender, entry.receiver, row.group, row.len, row.prio, row.type} and its padded
 *      payload is payload_out[row.payload_off, row.payload_off + pad32(row.len)), pad bytes included.
 *   2. Records whose ring entries point at the same arena payload (shared layout: one group send) share one row;
 *      every other record (point-to-point, broadcast copies, SDB_SHARED_PAYLOAD=0) has its own.  A send with only
 *      some of its records in the call still gets exactly one row.  Zero-length payloads of different sends never
 *      share a row.
 *   3. Rows are in order of first appearance in entry_out: the first occurrences of entry.send read 0, 1, 2, ..
 *      and payload_off is the running sum of pad32(len) over the rows.  The result depends neither on timing nor
 *      on the grid.
 *   4. Capacity as in sdb_receive_batch, with rec_cap = min(max_recv_records, max_recv_payload / P, entry_cap,
 *      send_cap, payload_cap / P) (each caller cap counts only when its pointer is given), P = pad32(max_payload_bytes).
 *      The unshared worst case always fits, so which records a call takes never depends on how much they share.
 *   5. SDB_RECV_PRIORITY, SDB_RECV_PEEK and SDB_RECV_OWNED as in sdb_receive_batch; SDB_RECV_ASYNC is refused
 *      (SDB_EINVAL).  The call always runs the bulk plan (never the few-agent or latency-server paths).  It leaves no
 *      full-format device results: sdb_digest_fold after it returns SDB_EINVAL until the next sdb_receive_batch.
 * *total_out, *n_sends_out and *payload_bytes_out (each nullable) receive the totals. */
typedef struct sdb_recv_entry {
  uint64_t seq;        /* header.seq of this record */
  uint32_t send;       /* row of send_out holding the rest of its header and its payload */
  uint32_t receiver;   /* header.receiver of this record */
} sdb_recv_entry;
typedef struct sdb_recv_send {
  double   timestamp;
  uint64_t payload_off; /* byte offset of the padded payload in payload_out */
  uint32_t sender;
  uint32_t group;
  uint16_t len;
  uint8_t  prio;
  uint8_t  type;
  uint32_t reserved;    /* 0 */
} sdb_recv_send;
int sdb_receive_compact(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages, uint32_t flags,
                        uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
                        sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                        uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out);
/* Receive by byte budget (Kafka's max.partition.fetch.bytes per agent and fetch.max.bytes per call): the arguments of
 * sdb_receive_batch / sdb_receive_compact plus max_agent_bytes.
 *   1. Per-agent take: the longest prefix of the agent's delivery order (stream order, or priority order with
 *      SDB_RECV_PRIORITY) with at most max_messages records and sum(pad32(len)) <= max_agent_bytes (0: no byte limit).
 *      An agent whose first record alone is larger takes that one record, so an oversized message never blocks its queue.
 *   2. Call capacity, exact in bytes: rec_cap = min(max_recv_records, hdr_cap) (full format) or min(max_recv_records,
 *      entry_cap, send_cap) (compact format), with no division by pad32(max_payload_bytes); byte capacity
 *      min(max_recv_payload, payload_cap), compared against sum(pad32(len)) of the records selected (each caller cap
 *      counts only when its pointer is given).  Truncation as in sdb_receive_batch: agents in list order, an agent whose
 *      take does not fit either cap stays queued together with every later agent; an agent first in the output takes the
 *      longest prefix of its take that fits both caps.
 *   3. Progress: payload_cap (when payload_out is given) below pad32(max_payload_bytes) is refused (SDB_EINVAL), so every
 *      call on a non-empty queue makes progress.
 *   4. Compact format: bytes are counted per record as in the full format, never per distinct row, so which records a
 *      call takes does not depend on how much they share; the compact payload output is never larger than that count.
 *   5. Equivalence: the result (records, order, bytes, retirement, counters, rings and, after a full-format call,
 *      sdb_digest_fold) is exactly what sdb_receive_batch / sdb_receive_compact return when each agent's max_messages is
 *      its take.  SDB_RECV_PRIORITY, SDB_RECV_PEEK and SDB_RECV_OWNED as there; SDB_RECV_ASYNC is refused (SDB_EINVAL).
 *      Refused calls leave every queue untouched.  A budget call always runs the bulk plan (never the few-agent or
 *      latency-server paths). */
int sdb_receive_budget(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                       uint64_t max_agent_bytes, uint32_t flags,
                       uint32_t* count_out, sdb_msg_header* hdr_out, uint64_t hdr_cap,
                       uint8_t* payload_out, uint64_t payload_cap,
                       uint64_t* total_out, uint64_t* payload_bytes_out);
int sdb_receive_compact_budget(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                               uint64_t max_agent_bytes, uint32_t flags,
                               uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
                               sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                               uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out);
/* Receive by token budget (as many pending messages as fit N tokens of a model's context): the arguments of
 * sdb_receive_budget / sdb_receive_compact_budget plus max_agent_tokens.  A record's weight is the u32 count at the start
 * of its payload when its type carries SDB_TYPEF_TOKENS (and len >= 4), else 0; records of unknown cost are bounded by
 * max_agent_bytes.
 *   1. Per-agent token take: the longest prefix of the agent's delivery order (stream order, or priority order with
 *      SDB_RECV_PRIORITY) whose weights sum to at most max_agent_tokens (64-bit sums), or its first record alone when that
 *      one is heavier.  In priority order that is whole levels from the top while they fit, then the arrival-order
 *      prefix of the level where the limit falls.
 *   2. Equivalence: the result (records, order, bytes, retirement, counters, rings and, after a full-format call,
 *      sdb_digest_fold) is exactly what sdb_receive_budget / sdb_receive_compact_budget return when each agent's
 *      max_messages is the smaller of max_messages and its token take.  Both takes are prefixes of one delivery order, so
 *      the byte limit, the call's capacity and its truncation rule apply on top exactly as there.
 *   3. max_agent_tokens == 0: no token limit; the call is sdb_receive_budget / sdb_receive_compact_budget.
 *   4. SDB_RECV_PRIORITY, SDB_RECV_PEEK and SDB_RECV_OWNED as in the budget call; SDB_RECV_ASYNC is refused (SDB_EINVAL).
 *      Refused calls leave every queue untouched.  The token pass is timed under SDB_PK_RECV_COUNT. */
int sdb_receive_tokens(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                       uint64_t max_agent_bytes, uint64_t max_agent_tokens, uint32_t flags,
                       uint32_t* count_out, sdb_msg_header* hdr_out, uint64_t hdr_cap,
                       uint8_t* payload_out, uint64_t payload_cap,
                       uint64_t* total_out, uint64_t* payload_bytes_out);
int sdb_receive_compact_tokens(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                               uint64_t max_agent_bytes, uint64_t max_agent_tokens, uint32_t flags,
                               uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
                               sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                               uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out);
/* tokens_out[i] = the token weights (as in sdb_receive_tokens) of agent agent_idx[i]'s pending records, summed
 * (agent_idx NULL: agents 0 .. n_agents - 1, as in sdb_agent_loads).  In-flight leases and dead letters are not pending.
 * Synchronising; the kernel is timed under SDB_PK_RECV_COUNT. */
int sdb_pending_tokens(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint64_t* tokens_out);
/* Restore: put records in the compact format back on the device - a queue snapshot (a PEEK compact receive) after a
 * restart, or what a compact receive just took when its consumer failed (requeue).  Input in exactly the shape
 * sdb_receive_compact and sdb_expire's archive mode return: listed agent i owns the next count[i] entries.
 *   1. Effect     each listed agent gets its records appended behind whatever it has pending, in the given order.  Record
 *                 r has the header of entry r and its row (contract point 1 of sdb_receive_compact: seq, timestamp,
 *                 sender, receiver, group, len, prio, type) and the padded payload bytes.  Every later receive (any path,
 *                 any order, digests) delivers what it would deliver had those records been sent in that position.
 *                 Sequence numbers are kept: message ids do not change.
 *   2. Counters   next_seq = max(next_seq, largest restored seq + 1); stats.enqueued += records, delivered stays; in
 *                 sdb_agent_loads `received`, `pending`, `pending_by_prio` and `pending_granules` grow as if the records
 *                 had been sent; the registration watermark covers every listed agent.
 *   3. Arena      rows in row-index order, each as its headers in entry order followed by ONE payload (shared layout; a
 *                 row with more than 65535 records takes consecutive blocks of at most 65535 headers, each with its own
 *                 payload copy).  From an agent's first entry that names a lower row than its previous entry on, that
 *                 agent's entries are private images (header + payload) in a tail region after all rows, in entry order.
 *                 With SDB_SHARED_PAYLOAD=0 every record is a private image.  Rows no restored entry names take no space.
 *                 Arena positions strictly increase along every ring, and the layout is deterministic.  Rows numbered by
 *                 their smallest seq in a stream-order snapshot give no private images.
 *   4. All or nothing: the call validates and plans on the device, synchronises once, then writes.  On any error rings,
 *                 arena, stats and digests are unchanged:
 *                   SDB_ERING_OVERFLOW  some agent's tail - head + count[i] exceeds ring_slots (tombstones count);
 *                   SDB_EARENA_FULL     the region does not fit after a floor reclaim;
 *                   SDB_ECAPACITY       more than one compact receive holds: n_entries or n_sends above rec_cap, or
 *                                       payload_bytes above rec_cap x pad32(max_payload_bytes) (rec_cap of
 *                                       sdb_receive_compact without caller caps) - a chunk one compact receive
 *                                       returned always restores in one call;
 *                   SDB_EINVAL          agent_idx NULL with n_agents > 0, an agent listed twice or >= max_agents,
 *                                       sum(count) != n_entries, entry.send >= n_sends, entry.receiver neither the
 *                                       listed agent nor SDB_NO_RECEIVER, row len > max_payload_bytes or prio > 3,
 *                                       payload_off not 16-byte aligned or payload_off + pad32(len) > payload_bytes,
 *                                       unknown flag bits.
 *                 Every row is checked, whether an entry names it or not.
 *   5. Flags      SDB_RECV_OWNED on a sharded handle skips the entries of agents this shard does not own (unchecked), so
 *                 every rank can be given the whole snapshot: a snapshot of N shards restores onto M.
 *   6. Ordering   stream-ordered on the handle's stream; synchronises.  Works while the latency server runs.  The last
 *                 receive's device results are left alone (sdb_digest_fold is unaffected).
 * *restored_out (nullable) = records enqueued, *seq_end_out (nullable) = next_seq after the call. */
int sdb_restore_compact(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, const uint32_t* count,
                        const sdb_recv_entry* entries, uint64_t n_entries, const sdb_recv_send* sends, uint64_t n_sends,
                        const uint8_t* payload, uint64_t payload_bytes, uint32_t flags, uint64_t* restored_out,
                        uint64_t* seq_end_out);
/* ---- leased receive: at-least-once delivery (mark_message_as_processed, M:654-669; MessageStatus READ / PROCESSED,
 * M:44-51).  A lease store in device memory keeps a copy of every record a leased receive hands out, in the compact format,
 * until the record is acknowledged or redelivered.  Redelivery puts it back behind what its agent has pending.
 *   sdb_lease_reserve   allocates the store: max_records entries (and rows) and max_payload_bytes (rounded up to
 *                       SDB_GRANULE) of payload, double-buffered for compaction.  max_records == 0 frees it.  Refused
 *                       (SDB_EINVAL) while the store holds live leases.  Nobody who does not call it pays the memory.
 *   sdb_receive_leased  selects, retires and returns exactly what sdb_receive_compact would with the same arguments (its
 *                       contract points 1-4), and appends each returned record to the store with `deadline`.  Record r of
 *                       the call, in entry_out order, gets lease id *lease_base_out + r; ids are monotonic per handle.
 *                       Capacity: rec_cap = min(sdb_receive_compact's rec_cap, free store entries, free store payload / P),
 *                       so a call never overfills the store; no room for one maximum-size record: SDB_ECAPACITY ("lease
 *                       store full: settle or sweep").  Flags: SDB_RECV_PRIORITY and SDB_RECV_OWNED; SDB_RECV_PEEK,
 *                       SDB_RECV_ASYNC and other bits are refused (SDB_EINVAL), as is a call without a reserved store.
 *   sdb_lease_settle    op SDB_LEASE_ACK marks live leases done; SDB_LEASE_RENEW sets their deadline (a later one extends,
 *                       -INFINITY makes them due at the next sweep: a nack).  settled_out[i] (nullable) is 1 when lease
 *                       lease_id[i] was live before the call, else 0 (unknown, already acked, already redelivered: a late
 *                       ack after redelivery is visible, not an error); an id repeated in one call reads 1 each time and is
 *                       settled once.  *n_settled_out = requests that read 1.  Acks free no space: the next sweep does.
 *   sdb_lease_sweep     redelivery.  Due: every live lease with deadline <= now (a NaN deadline or NaN `now` makes nothing
 *                       due); with SDB_LEASE_ALL every live lease, deadlines not read.  One call takes at most one compact
 *                       receive's capacity of due records, in lease-id order (*due_left_out = due records beyond it: loop
 *                       until it reads 0).  Each agent's records are appended behind what it has pending, in lease-id
 *                       order - the original delivery order - with sdb_restore_compact's effect (its points 1-3: seq,
 *                       ids and headers kept; enqueued and agent loads move as for a restore).  Rows are numbered by
 *                       their smallest redelivered seq, so a stream-order lease comes back in its sends' arena layout.  An
 *                       agent whose ring cannot take all of its records of the call (tail - head + records > ring_slots,
 *                       tombstones count) keeps them in the store and is counted in *blocked_out; every other agent is
 *                       served.  SDB_EARENA_FULL (after a floor reclaim) fails the call whole: store, rings and stats
 *                       unchanged.  Afterwards the store is compacted: acked and redelivered entries and the rows and
 *                       payloads no live entry names are dropped, in a stable order (lease ids stay ascending).
 *   sdb_lease_stats     host bookkeeping of the store (no synchronisation).
 * All but sdb_lease_stats are stream-ordered on the handle's stream and synchronise. */
#define SDB_LEASE_ACK 0u
#define SDB_LEASE_RENEW 1u
#define SDB_LEASE_ALL 1u                /* sdb_lease_sweep flag: every live lease is due */
typedef struct sdb_lease_summary {
  uint64_t live;                /* leases neither acked nor redelivered */
  uint64_t acked_unreclaimed;   /* acked entries the next sweep drops */
  uint64_t redelivered_total;   /* records redelivered so far */
  uint64_t acked_total;         /* leases acked so far */
  uint64_t entries_used, entries_reserved;
  uint64_t payload_used, payload_reserved;   /* bytes */
} sdb_lease_summary;
int sdb_lease_reserve(sdb_handle h, uint64_t max_records, uint64_t max_payload_bytes);
int sdb_receive_leased(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages, uint32_t flags,
                       double deadline, uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
                       sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                       uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out, uint64_t* lease_base_out);
/* Leased receive by budget and filter (an agent that assembles a model's context from its queue and needs its messages
 * back when the model call fails): sdb_receive_leased's arguments plus max_agent_bytes, max_agent_tokens and a nullable
 * filter (sdb_receive_where's sdb_filter, declared below).
 *   1. Take: per agent, over its pending records that match the filter (NULL: every pending record), in the call's
 *      delivery order, the shortest of max_messages, the byte take (the longest prefix with sum(pad32(len)) <=
 *      max_agent_bytes) and the token take (sdb_receive_tokens' weights and 64-bit sums).  A budget take is the first
 *      record alone when that record is heavier than its limit; a limit of 0 is no limit.
 *   2. Equivalence: the result (records, order, bytes, retirement, counters, rings, lease ids, deadlines, delivery
 *      counts and the dead-letter ledger) is exactly sdb_receive_leased with each agent's max_messages lowered to its
 *      take, on a queue holding only the matching records.  Capacity is sdb_receive_leased's rule (records x
 *      pad32(max_payload_bytes), the store's free room, lead-agent truncation), not sdb_receive_budget's exact bytes.
 *   3. Both limits 0 and a NULL filter: the call is sdb_receive_leased.
 *   4. Flags, SDB_ECAPACITY and lease_base_out as in sdb_receive_leased; the filter's refusals as in sdb_receive_where
 *      (its per-id outputs included).  A refused call leaves queues, store and ledger untouched.  The take pass of a
 *      filtered call is timed under SDB_PK_RECV_COUNT. */
struct sdb_filter;
int sdb_receive_leased_select(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                              uint64_t max_agent_bytes, uint64_t max_agent_tokens, const struct sdb_filter* filter,
                              uint32_t flags, double deadline, uint32_t* count_out, sdb_recv_entry* entry_out,
                              uint64_t entry_cap, sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out,
                              uint64_t payload_cap, uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out,
                              uint64_t* lease_base_out);
int sdb_lease_settle(sdb_handle h, uint64_t n, const uint64_t* lease_id, uint32_t op, double deadline, uint8_t* settled_out,
                     uint64_t* n_settled_out);
int sdb_lease_sweep(sdb_handle h, double now, uint32_t flags, uint64_t* redelivered_out, uint64_t* blocked_out,
                    uint64_t* due_left_out);
int sdb_lease_stats(sdb_handle h, sdb_lease_summary* out);
/* ---- dead letters: delivery counts and a redelivery limit for leased receives (a poison message is redelivered at most
 * max_deliveries times, then parked).  Off by default; nothing below allocates or launches anything until it is set.
 *   Delivery count  a record returned by a leased receive has deliveries = 1, except when a sweep redelivered it from a
 *                   lease with count k and it stayed pending since (no plain, priority, filtered or compact receive took
 *                   it, no expiry, purge or trim retired it): then the next leased receive that returns it gives it k + 1.
 *                   Records put back by sdb_restore_compact (requeue, redrive) start again at 1.  Records are identified by
 *                   (agent, seq); when two pending copies share both, which one inherits the count is unspecified.
 *   Ledger          the counts of redelivered records wait in a device table keyed by (agent, seq) holding the ring
 *                   position and arena handle restore gave the record (56 bytes per entry).  Each leased receive and
 *                   sweep first drops the entries whose record is no longer that one (left the window, consumed, or the
 *                   slot names another handle), so a count is never inherited by a different record.  A sweep redelivers
 *                   at most the ledger's free room: the rest stays leased and is counted in *due_left_out.
 *   sdb_lease_set_policy  max_deliveries = 0 turns the policy off and frees its memory; max_deliveries >= 1 needs
 *                   ledger_entries >= 1 (0xFFFFFFFF: counts without a limit).  Clears the ledger.  SDB_EINVAL without a
 *                   reserved store, while the store holds live leases or dead letters, or for M > 0 with no ledger.
 *                   sdb_lease_reserve turns the policy off.
 *   Sweep           with M > 0, every live due lease (every live lease under SDB_LEASE_ALL) whose deliveries >= M becomes a
 *                   dead letter instead of being redelivered; dead letters are not counted in *redelivered_out,
 *                   *blocked_out or *due_left_out.  They stay in the store (entries_used, payload_used) and shrink a
 *                   leased receive's capacity until they are taken.  Settle reads them as not live.  A sweep that fails
 *                   with SDB_EARENA_FULL leaves store, ledger, rings and stats as they were.
 *   sdb_lease_deliveries  the count of each live or dead lease; 0 for an unknown, acked or redelivered id.
 *   sdb_lease_dead_letters  the dead letters of the listed agents (agent_idx NULL: every index below the watermark; an
 *                   agent listed twice: SDB_EINVAL), agents in list order and lease-id order within an agent, in the
 *                   compact format (sdb_receive_compact's points 1-3: rows shared by records of one store row, numbered by
 *                   first appearance) with its capacity rule (point 4, lead-agent exception included): loop until
 *                   *total_out == 0.  deliveries_out[total] (nullable) = each record's count.  SDB_RECV_PEEK leaves them
 *                   in the store; without it they leave the store and their space is freed.  Other flag bits: SDB_EINVAL.
 *                   The output is valid sdb_restore_compact input as it stands: a redrive is a take and a restore (ids
 *                   kept, counts restart at 1).
 *   sdb_lease_policy_stats  host bookkeeping (no synchronisation): ledger_used as of the last collection or lookup,
 *                   held_by_ledger_total = due leases sweeps left in the store because the ledger was full.
 * All but sdb_lease_policy_stats are stream-ordered and synchronise; refused calls zero their outputs and change nothing. */
typedef struct sdb_lease_policy_summary {
  uint64_t max_deliveries, dead, dead_total, ledger_used, ledger_cap, held_by_ledger_total;
} sdb_lease_policy_summary;
int sdb_lease_set_policy(sdb_handle h, uint32_t max_deliveries, uint64_t ledger_entries);
int sdb_lease_deliveries(sdb_handle h, uint64_t n, const uint64_t* lease_id, uint32_t* deliveries_out);
int sdb_lease_dead_letters(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t flags,
                           uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
                           sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                           uint32_t* deliveries_out, uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out);
int sdb_lease_policy_stats(sdb_handle h, sdb_lease_policy_summary* out);
/* ---- snapshots of in-flight work: the lease store and the redelivery ledger read out and put back, so that a restart
 * keeps at-least-once delivery (leases not yet acked stay owed, dead letters stay parked, delivery counts continue).
 *   sdb_lease_export  reads only: nothing in the store, ledger, rings or stats moves.  Returns the live leases and the dead
 *                   letters with id >= start_id, in lease-id order (acked and not yet reclaimed entries are left out), in
 *                   the compact format (sdb_receive_compact's points 1-3: rows numbered by first appearance, a store row
 *                   named by several records is one row).  At most rec_cap records per call by sdb_receive_compact's
 *                   point 4 (no agent grouping: the first rec_cap records); meta_out[total] (nullable, counted against
 *                   entry_cap) receives each record's sdb_lease_meta.  *next_id_out = the id to pass next (start_id when
 *                   nothing is returned): loop until *total_out == 0.  flags != 0 or no store: SDB_EINVAL.  It reuses the
 *                   compact receive's buffers: sdb_digest_fold returns SDB_EINVAL afterwards until the next
 *                   sdb_receive_batch.
 *   sdb_lease_import  appends n records, in input order, behind whatever the store holds: record r gets lease id
 *                   *lease_base_out + r (ids stay ascending) and keeps meta[r].deadline, .state and .deliveries (with a
 *                   policy, 0 is imported as 1; without one counts are not stored; meta.id is not read).  Counters: live
 *                   and dead grow by state, entries_used and payload_used grow.  Input in sdb_lease_export's shape; every
 *                   row is checked and copied.  All or nothing: the input is validated on the device, the call
 *                   synchronises once, then writes.  Refusals:
 *                     SDB_EINVAL     NULL arrays with n > 0, entry.send >= n_sends, meta.agent >= max_agents,
 *                                    entry.receiver neither meta.agent nor SDB_NO_RECEIVER, row len > max_payload_bytes or
 *                                    prio > 3, payload_off not 16-byte aligned or payload_off + pad32(len) > payload_bytes,
 *                                    a state other than LIVE or DEAD, a DEAD record on a handle without a policy,
 *                                    flags != 0, no store;
 *                     SDB_ECAPACITY  n or n_sends above one compact receive's rec_cap, or payload_bytes above
 *                                    rec_cap x pad32(max_payload_bytes) (a chunk one export returned always imports in one
 *                                    call); not enough free store entries, rows or payload ("lease store full").
 *                   A LIVE lease with deliveries >= max_deliveries of the importing handle becomes a dead letter at its
 *                   next due sweep.  Like sdb_lease_export it reuses the compact receive's buffers.
 *   sdb_lease_ledger_export  runs the ledger's collection (the one every leased receive runs), so only entries whose
 *                   record is still pending are reported, then writes all of them as (agent, seq, count) triples in no
 *                   particular order; *n_out = their number.  cap below it: SDB_EOUTPUT with *n_out set, nothing written.
 *                   No policy: SDB_EINVAL.
 *   sdb_lease_ledger_import  for each triple the oldest pending (not consumed) record of `agent` whose header seq matches
 *                   gets a ledger entry holding its ring position, its arena handle and `count`: the next leased receive
 *                   of that record gives it count + 1, as if a sweep had redelivered it.  A triple with no such record
 *                   is dropped and not counted in *matched_out; for a pair listed twice which entry wins is unspecified.
 *                   SDB_EINVAL: no policy, agent >= max_agents, count == 0, NULL arrays with n > 0.  SDB_ECAPACITY: n
 *                   above the ledger's free room after a collection.  Refusals change nothing.
 * All four are stream-ordered and synchronise; a refused call zeroes its outputs and changes nothing.  Their kernels time
 * under SDB_PK_LEASE. */
#define SDB_LEASE_STATE_LIVE 0u
#define SDB_LEASE_STATE_DEAD 3u
typedef struct sdb_lease_meta {   /* 32 bytes, one per exported record */
  uint64_t id;                    /* lease id on the exporting handle */
  double   deadline;
  uint32_t agent;
  uint32_t deliveries;            /* 0 when the exporting handle has no policy */
  uint32_t state;                 /* SDB_LEASE_STATE_LIVE or SDB_LEASE_STATE_DEAD */
  uint32_t reserved;              /* 0 */
} sdb_lease_meta;
int sdb_lease_export(sdb_handle h, uint64_t start_id, uint32_t flags, sdb_recv_entry* entry_out, uint64_t entry_cap,
                     sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                     sdb_lease_meta* meta_out, uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out,
                     uint64_t* next_id_out);
int sdb_lease_import(sdb_handle h, uint64_t n, const sdb_recv_entry* entries, const sdb_recv_send* sends, uint64_t n_sends,
                     const uint8_t* payload, uint64_t payload_bytes, const sdb_lease_meta* meta, uint32_t flags,
                     uint64_t* lease_base_out);
int sdb_lease_ledger_export(sdb_handle h, uint64_t cap, uint32_t* agent_out, uint64_t* seq_out, uint32_t* count_out,
                            uint64_t* n_out);
int sdb_lease_ledger_import(sdb_handle h, uint64_t n, const uint32_t* agent, const uint64_t* seq, const uint32_t* count,
                            uint64_t* matched_out);
/* Low-latency dequeue server (opt-in): receive_messages (M:521-601) for ONE agent in a few microseconds.
 * enable = 1 starts a persistent single-CTA kernel on its own stream that polls a mailbox in mapped pinned host memory;
 * sdb_receive_batch calls naming exactly one agent with host outputs (what the Python surface's receive_messages makes)
 * then post a request there and read the answer - count, headers and payloads - from pinned host memory the kernel wrote
 * directly: no kernel launch, no cudaStreamSynchronize, no cudaMemcpy on the path.  Results are identical to the
 * ordinary path (same selection code).  Starting it first loads every kernel of the library (under lazy module loading
 * a kernel's first launch would otherwise wait for the server, which never ends; needs a CUDA 12.4 or later driver).
 * enable = 0 stops it (also done by sdb_destroy).  While it runs the handle
 * stops it around its own calls that free device memory (cudaFree waits for running kernels) and restarts it on the
 * next single-agent receive; callers must likewise not call cudaDeviceSynchronize / cudaFree from outside while it runs. */
int sdb_latency_server(sdb_handle h, int enable);

/* Device-resident results of the LAST receive call (valid until the next one). */
int sdb_last_receive_dev(sdb_handle h, const uint32_t** count_dev, const sdb_msg_header** hdr_dev,
                         const uint8_t** payload_dev);
/* Records and payload bytes of the LAST receive call; waits for it (the host side of SDB_RECV_ASYNC). */
int sdb_last_receive_totals(sdb_handle h, uint64_t* total_out, uint64_t* payload_bytes_out);

/* ---- stream digests: per-agent delivery order + content, checkable at any scale ---------------------------------
 * What the reference promises a consumer is the ORDER and CONTENT of its own stream (drain loop M:553-601, filter
 * M:579-585).  A digest per agent captures exactly that without moving the records off the device:
 *   rec_hash = sum over the 64-bit little-endian words w_k (k = 0, 1, ..) of [sdb_msg_header | payload padded to
 *              SDB_GRANULE] of fmix64(w_k ^ ((k + 1) * 0x9E3779B97F4A7C15))  mod 2^64   (fmix64 = MurmurHash3 finaliser)
 *   chain    : d[a] <- (rotl64(d[a], 5) ^ rec_hash) * 0x9E3779B97F4A7C15, for every record delivered to agent a, in
 *              delivery order; d[a] starts at 0.
 * sdb_digest_fold folds the device-resident results of the LAST sdb_receive_batch call (bulk path; not the
 * <= 8-agent latency path) into d[]; it is stream-ordered and does not synchronise.  sdb_digest_read copies
 * d[agent_idx[i]] (agent_idx == NULL: agents 0..n-1) to the host.  Used by tests and by bench.py's parity check
 * (1M agents, 1..8 GPUs) against the same definition in oracle/cpu_ref.c. */
int sdb_digest_reset(sdb_handle h);
int sdb_digest_fold(sdb_handle h);
int sdb_digest_read(sdb_handle h, uint32_t n, const uint32_t* agent_idx, uint64_t* digest_out);

/* ---- cross-shard delivery (one handle per GPU, one process per GPU) ----------------------------
 * Replaces the partitioned topic: _get_partition (M:309-312, salted hash() % num_partitions) and
 * the explicit-partition produce (M:469-482).  Agents are hash-partitioned over num_shards GPUs;
 * sdb_set_agent_shards declares the owner of every agent index (the Python layer uses
 * fnv1a64(utf8(agent_id)) % num_shards).  Group tables are replicated: every shard calls
 * sdb_create_group with the FULL member list and keeps the members it owns plus their positions.
 *
 * A rank exports the group sends it ingested as ONE wire batch in device memory - descriptor +
 * payload per SEND, not per recipient.  The caller moves wire batches between ranks (NCCL
 * all-gather over NVLink through torch.distributed) and every rank imports the wire batches of
 * all ranks, in rank order: each send is expanded into the copies for the members this shard owns.
 * Sequence numbers are global (rank r's sends follow rank r-1's), so per-agent streams are
 * identical to a single-shard run over the concatenated batch.  With num_shards == 1 the same
 * two calls work without any collective.
 */
uint64_t sdb_wire_bytes(sdb_handle h, uint32_t max_sends, uint64_t max_payload_bytes);
int sdb_set_agent_shards(sdb_handle h, uint32_t n, const uint8_t* shard_of);
int sdb_export_group_batch(sdb_handle h, uint32_t n,
                           const uint32_t* sender, const uint32_t* group_idx,
                           const uint8_t* prio, const uint8_t* type, const uint16_t* len,
                           const uint64_t* payload_off, const uint8_t* payload, uint64_t payload_bytes,
                           const double* timestamp, void* wire_dev, uint64_t wire_cap);
/* Same, for a mixed batch in call order (kinds as in sdb_send_mixed_batch): point-to-point sends are
 * delivered only by the shard that owns the receiver, broadcast lists by every shard for the
 * recipients it owns.  Recipient lists travel inside the wire batch (count them in max_payload_bytes). */
int sdb_export_mixed_batch(sdb_handle h, uint32_t n,
                           const uint32_t* sender, const uint8_t* kind, const uint32_t* target,
                           uint32_t n_lists, const uint64_t* list_off, const uint32_t* list_idx,
                           const uint8_t* prio, const uint8_t* type, const uint16_t* len,
                           const uint64_t* payload_off, const uint8_t* payload, uint64_t payload_bytes,
                           const double* timestamp, void* wire_dev, uint64_t wire_cap);
/* Same, but the exporter numbers its sends itself, starting at `seq_base` (non-zero).  Front-ends that must
 * return message ids at send time - before the collective flush - use a composite number
 * (round << 40 | rank << 32 | local index), which keeps the global (round, rank, local) delivery order. */
int sdb_export_mixed_batch_seq(sdb_handle h, uint64_t seq_base, uint32_t n,
                               const uint32_t* sender, const uint8_t* kind, const uint32_t* target,
                               uint32_t n_lists, const uint64_t* list_off, const uint32_t* list_idx,
                               const uint8_t* prio, const uint8_t* type, const uint16_t* len,
                               const uint64_t* payload_off, const uint8_t* payload, uint64_t payload_bytes,
                               const double* timestamp, void* wire_dev, uint64_t wire_cap);
int sdb_import_wire_batches(sdb_handle h, uint32_t n_src, const void* wire_dev_all, uint64_t wire_stride,
                            uint64_t* seq_base_out);
/* Peer-memory transport (no collective): each rank exports into a buffer allocated with
 * sdb_wire_alloc, hands the 64-byte CUDA-IPC handle to the other ranks (any side channel), which
 * map it with sdb_wire_open; after a cross-rank barrier every rank imports from the table of
 * pointers (its own buffer + the mapped peer buffers, rank order).  The import kernels and the
 * fan-out kernel's TMA loads then read descriptors and payloads directly out of the exporting
 * GPU's memory over NVLink, overlapped with the fan-out itself. */
int sdb_wire_alloc(sdb_handle h, uint64_t bytes, void** dev_out, void* ipc_handle_out /* 64 bytes, nullable */);
int sdb_wire_open(sdb_handle h, const void* ipc_handle, void** dev_out);
int sdb_wire_close(sdb_handle h, void* dev, int opened /* 1: from sdb_wire_open, 0: from sdb_wire_alloc */);
int sdb_import_wire_ptrs(sdb_handle h, uint32_t n_src, const void* const* wire_ptrs, uint64_t* seq_base_out);
/* Flag-synchronised, host-asynchronous form of the peer-memory transport: no collective and no host round trip.
 * Every export buffer of `wire_bytes` (as sized by sdb_wire_bytes) ends in a 128-byte control block with two
 * counters: `ready` (last step whose export into the buffer is complete) and `done` (last step for which the
 * buffer's OWNER finished importing every rank's buffer of that parity).  Steps count 1, 2, 3 ...; with two
 * alternating buffers per rank, buffer step & 1 is used for step.
 *   sdb_wire_wait_done     stream-ordered wait until every listed buffer's owner reports done >= step; call it with
 *                          (step - 2) before exporting `step` into a buffer that peers read two steps ago
 *   sdb_wire_publish       stream-ordered: ready = step (after the export's copies, which run on the same stream)
 *   sdb_import_wire_ptrs_async
 *                          waits ON THE DEVICE for ready >= step of every source (peer flags are polled over NVLink),
 *                          then places and expands the import entirely on the device - arena position, sequence base
 *                          and totals never visit the host (a device-resident cursor is the authority until the next
 *                          call that needs them on the host) - and finally reports done = step in this rank's own
 *                          buffer (wire_ptrs[shard_id]).  Three kernels do the work: one fused localize (wire headers,
 *                          descriptors and group buckets read straight out of the exporting GPUs, decoupled
 *                          look-back scan, placement), the fan-out (TMA pulls of the payloads over NVLink), the
 *                          group-parallel index build.  An import that does not fit (arena / list pool) is dropped
 *                          WHOLE and reported by the next host-synchronising call (SDB_EARENA_FULL / SDB_ECAPACITY).
 *                          Traffic outside the fast shape (payloads above 512 bytes, agents in several groups) takes
 *                          the synchronous import between the same flags. */
int sdb_wire_wait_done(sdb_handle h, uint32_t n_src, const void* const* wire_ptrs, uint64_t wire_bytes, uint32_t step);
int sdb_wire_publish(sdb_handle h, void* wire_dev, uint64_t wire_bytes, uint32_t step);
int sdb_import_wire_ptrs_async(sdb_handle h, uint32_t n_src, const void* const* wire_ptrs, uint64_t wire_bytes, uint32_t step);
/* Pipelining across steps: runs the flag wait and the localize pass of step `step` on a second stream of the handle,
 * ordered after everything enqueued on the shard's stream so far and BESIDE what the caller enqueues next (typically
 * the receive of the previous step, which is bound by HBM while the localize pass is bound by NVLink latency).  The
 * following sdb_import_wire_ptrs_async(.., step) finds the batch localized and only places it (one single-thread
 * kernel: arena base and sequence base still come from the device cursor, after the previous step's commit), then
 * fans out and indexes as usual: delivery order and content are those of the unpipelined sequence.  Two buffer sets
 * alternate by step parity.  The export buffers of `step` must not be rewritten and group membership / ownership must
 * not change between the two calls.  A no-op for traffic outside the fast shape. */
int sdb_import_prefetch(sdb_handle h, uint32_t n_src, const void* const* wire_ptrs, uint64_t wire_bytes, uint32_t step);

/* ---- which records were lost to full rings (delivery report, M:374-391 / M:501-519)
 * A ring is full when tail - head = ring_slots.  The window [head, tail) holds tombstones too (records consumed out of
 * stream order by priority receives, sdb_receive_where and sdb_expire), and after every retiring call head is the
 * oldest pending record (tail when none is left): so a ring takes ring_slots - (tail - head) more records, whichever
 * receive, filtered take, expiry or leased receive consumed the earlier ones.
 * `ring_overflow` in sdb_stats says how many records found their receiver's ring full; this call says WHICH: up to
 * `cap` (receiver agent, sequence number) pairs of records dropped since the previous call, in no particular order
 * (the device logs the first 4096 per interval; *dropped_out = how many were dropped in the interval).  Reading
 * clears the log.  Call it right after the batch that overflowed: the sequence number is read from the dropped
 * record's image in the arena log, which is reclaimed like any other record. */
int sdb_overflow_log(sdb_handle h, uint32_t cap, uint32_t* agent_out, uint64_t* seq_out, uint32_t* n_out, uint64_t* dropped_out);

/* ---- inbox / load queries on the device: get_agent_load, get_unread_message_count (M:1026-1094), get_stats (M:973-1024)
 * The reference answers these by walking its host dictionaries (`messages`, `agent_inbox`); the queue itself now lives
 * in HBM, so the same questions are answered from the rings.  Mapping of the reference's fields:
 *   inbox_size    (len(agent_inbox[a]), M:1076)            = received      records ever enqueued for the agent
 *   unread_count  (status == DELIVERED in the inbox, M:1040) = pending       records still queued (not yet received)
 *   READ / PROCESSED side                                   = received - pending
 * sdb_agent_loads fills one sdb_agent_load per listed agent (agent_idx == NULL: agents 0..n-1).
 * sdb_queue_stats reduces over every agent below the watermark: totals, the pending records per priority level (a
 * histogram over the ring metadata), the deepest queue.  Both synchronise (they return data). */
typedef struct sdb_agent_load {
  uint32_t received;             /* records enqueued for the agent so far (mod 2^32) */
  uint32_t pending;              /* records waiting in its ring */
  uint32_t pending_by_prio[4];   /* ... by priority level (M:35-41) */
  uint32_t pending_granules;     /* 32-byte granules of pending payload (without headers) */
  uint32_t reserved;
} sdb_agent_load;
typedef struct sdb_queue_summary {
  uint64_t agents_with_pending;
  uint64_t pending;
  uint64_t pending_by_prio[4];
  uint64_t pending_granules;
  uint64_t received;             /* sum over agents of `received` */
  uint64_t max_pending;          /* deepest queue */
  uint64_t max_pending_agent;
} sdb_queue_summary;
int sdb_agent_loads(sdb_handle h, uint32_t n, const uint32_t* agent_idx, sdb_agent_load* out);
int sdb_queue_stats(sdb_handle h, sdb_queue_summary* out);

/* ---- retention: flush_old_messages (M:1159-1206), retention.ms (M:123, M:254) --------------------------------------
 * The arena is a log: space is reclaimed only behind the oldest pending record of any ring, so an agent that never
 * receives (crashed, deregistered - deregistration keeps the ring - or idle) pins the whole log until sends fail with
 * SDB_EARENA_FULL.  sdb_expire retires pending records on the device without delivering them.
 *   Selection  for each listed agent (agent_idx == NULL: every index below the watermark, or the owned agents with
 *              SDB_RECV_OWNED), every pending record whose header timestamp < older_than (the strict compare of M:1179:
 *              a NaN timestamp or cutoff never expires anything).  Records sent with timestamp == NULL carry 0.0, so any
 *              positive cutoff expires them.  SDB_EXPIRE_ALL: every pending record of the listed agents, timestamps not
 *              read (purge).  An agent may appear only once in agent_idx (SDB_EINVAL otherwise).
 *   Retire     the selected ring entries are tombstoned; the remaining records keep their order, and every later receive
 *              (any order, any path) delivers what it would have delivered had the expired records never been enqueued.
 *              sdb_stats does not move (expired records are neither delivered nor un-enqueued); in sdb_agent_loads
 *              `pending` and `pending_granules` fall and `received` stays.  The arena floor is not moved by the call:
 *              the next send that needs room recomputes it and finds the space.
 *   Archive    (any of entry_out / send_out / payload_out given) the expired records are returned in the compact receive
 *   mode       format with its contract and capacity rule (sdb_receive_compact, points 1-4): agents in list order, stream
 *              order within an agent, one row per distinct payload image.  What does not fit stays queued: loop until
 *              *total_out == 0.  No usable output capacity: SDB_EOUTPUT.
 *   Drop mode  (all three output pointers NULL) no capacity limit and no copy-out: count_out[n_agents] (nullable) and
 *              *total_out are filled, *n_sends_out and *payload_bytes_out read 0.  The at-scale path.
 *   Flags      SDB_RECV_PEEK (dry run: select and report, retire nothing), SDB_RECV_OWNED, SDB_EXPIRE_ALL; any other bit
 *              is refused (SDB_EINVAL).
 *   Ordering   stream-ordered on the handle's stream; synchronises (it returns totals).  It touches rings only, so it
 *              may sit between sdb_import_prefetch(step) and sdb_import_wire_ptrs_async(step): the prefetch stream reads
 *              the wire batches and writes its own buffers, never a ring. */
#define SDB_EXPIRE_ALL 16u              /* every pending record of the listed agents, timestamps not read (purge) */
int sdb_expire(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, double older_than, uint32_t flags,
               uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
               sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
               uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out);

/* ---- bounded queues: x-max-length / x-max-length-bytes with overflow=drop-head, XTRIM MAXLEN, retention.bytes -------
 * sdb_trim caps each listed agent's pending queue by count and bytes and retires what is over the cap, oldest (or
 * lowest priority) first, without delivering it.  It reads ring entries only, never the arena.
 *   1. Limits     max_records caps an agent's live pending records (0: no count limit).  max_agent_bytes caps the sum of
 *                 pad32(len) over them - the units of sdb_receive_budget and of sdb_agent_load.pending_granules x 32 -
 *                 rounded down to granules (0: no byte limit).  Both 0 is SDB_EINVAL (purging is SDB_EXPIRE_ALL's job).
 *   2. Eviction   default: stream order, oldest first.  SDB_RECV_PRIORITY: the lowest level first (0, then 1, 2, 3),
 *      order      oldest first within a level.  Records are retired in eviction order until the agent's remaining live
 *                 records meet both limits: the shortest prefix of the eviction order that does it.  A record larger
 *                 than the byte limit on its own goes.  An agent already within both limits is not written at all.
 *   3. Scope      only pending ring records are counted or retired; in-flight leases and dead letters are neither
 *                 counted nor touched.  agent_idx == NULL and SDB_RECV_OWNED as in sdb_expire; an agent listed twice or
 *                 out of range is SDB_EINVAL.
 *   4. Effect     that of sdb_expire: every later receive (any order, any path, digests included) delivers what it would
 *                 have delivered had the trimmed records never been enqueued.  sdb_stats does not move; in
 *                 sdb_agent_loads `pending` and `pending_granules` fall and `received` stays.  Ring capacity is freed
 *                 (head moves to the first live entry, ntomb stays exact); the next send that needs room recomputes the
 *                 arena floor.  Ledger entries of trimmed records (sdb_lease_set_policy) are collected as expired ones.
 *   5. Archive    (any of entry_out / send_out / payload_out given) the trimmed records come back in the compact receive
 *      mode       format with sdb_expire's capacity rule: agents in list order, stream order within an agent.  An agent
 *                 whose trimmed records do not fit stays whole, except the first agent of the output, which gives the
 *                 first rec_cap records of its eviction order.  Calls repeated until *total_out == 0 retire exactly the
 *                 records one drop-mode call retires.  No usable output capacity: SDB_EOUTPUT.
 *   6. Drop mode  (all three output pointers NULL) no capacity limit: count_out[n_agents] (nullable) and *total_out are
 *                 filled, *n_sends_out and *payload_bytes_out read 0.
 *   7. Flags      SDB_RECV_PEEK (dry run: select and report, retire nothing), SDB_RECV_OWNED, SDB_RECV_PRIORITY; any
 *                 other bit is SDB_EINVAL.
 *   8. Ordering   as sdb_expire: stream-ordered, synchronising, rings only (so it may sit inside an import prefetch
 *                 window).  Kernels are timed under SDB_PK_EXPIRE. */
int sdb_trim(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_records, uint64_t max_agent_bytes,
             uint32_t flags, uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
             sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
             uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out);

/* ---- superseding sends: last-value queues, conflation (RabbitMQ last-value cache, Kafka compaction, MQTT retained) ---
 * sdb_supersede keeps, at each listed agent, only the newest pending record of each key among the records sent with
 * SDB_TYPEF_SUPERSEDE in their type byte, and retires the others without delivering them.  The send calls do not change:
 * the caller sets the bit in type[].  Costs one header read per live pending record when nothing is flagged.
 *   1. Key        two pending records of one agent have the same key when both carry SDB_TYPEF_SUPERSEDE and have equal
 *                 sender, group and type & SDB_TYPE_MASK.  The JSON and extras bits, priority, length and timestamp are
 *                 not part of it.  Point-to-point sends and broadcast copies both have group == SDB_NO_GROUP, so for one
 *                 sender and one type they share a key.
 *   2. Newest     within a key the record with the largest seq is kept; a tie in seq goes to the record later in the
 *                 ring (restoring the output of a PEEK compact receive with sdb_restore_compact makes one: restore does
 *                 not refuse a seq that is still pending).  Ring order is not seq order once a lease sweep, redrive,
 *                 restore or requeue put records back behind newer ones: the rule is by seq, so a redelivered stale
 *                 version is the one that goes.  Every other record of the key is superseded; unflagged records are
 *                 never counted or retired.
 *   3. Scope      only pending ring records are compared, as in sdb_trim: in-flight leases and dead letters are neither
 *                 compared nor touched, so a redelivered version can follow a newer one that was already received.
 *                 agent_idx == NULL and SDB_RECV_OWNED as in sdb_expire; an agent listed twice or out of range is
 *                 SDB_EINVAL.
 *   4. Effect     that of sdb_trim: every later receive (any order, any path, digests included) delivers what it would
 *                 have delivered had the superseded records never been enqueued.  sdb_stats does not move; in
 *                 sdb_agent_loads `pending` and `pending_granules` fall and `received` stays.  The head and ntomb stay
 *                 exact.  Ledger entries of retired records (sdb_lease_set_policy) are collected as expired ones.
 *   5. Archive    as sdb_trim: the superseded records come back in the compact receive format with sdb_expire's
 *      mode       capacity rule: agents in list order, ring order within an agent, the first agent of the output may be
 *                 partial.  The newest record of a key is never selected, so any subset of the superseded set is safe
 *                 to retire: calls repeated until *total_out == 0 retire exactly what one drop-mode call retires.  No
 *                 usable output capacity: SDB_EOUTPUT.
 *   6. Drop mode  as sdb_trim: count_out[n_agents] (nullable) and *total_out are filled, *n_sends_out and
 *                 *payload_bytes_out read 0.
 *   7. Flags      SDB_RECV_PEEK (dry run: select and report, retire nothing), SDB_RECV_OWNED; any other bit is SDB_EINVAL.
 *   8. Ordering   as sdb_trim: stream-ordered, synchronising, rings only; kernels are timed under SDB_PK_EXPIRE.  A
 *                 count pass runs first and the call ends there when no listed agent has a flagged pending record.
 *                 Otherwise it needs a key table of 32 bytes per slot (a power of two >= 2 x the flagged records) and
 *                 24 bytes per flagged record, kept by the handle and grown on demand; when they cannot be allocated the
 *                 call refuses with SDB_ECAPACITY before anything is retired.  A refused call changes nothing. */
int sdb_supersede(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t flags,
                  uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
                  sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                  uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out);

/* ---- relocation of pinned queues: the other remedy for an agent that pins the log.  Where sdb_expire drops its records,
 * sdb_arena_relocate keeps them: it copies the live records of the agents pinning the log to the tail of the arena and
 * rewrites those agents' ring entries in place, so the floor can pass the old region.  Nothing is delivered, dropped,
 * re-sequenced or reordered; every agent's stream stays byte for byte what it was.
 *   1. Selection  an agent below the registration watermark is selected when its oldest live (non-tombstoned) ring entry
 *                 has its header below floor_bytes (compared as the floor reclaim does: distance below the tail, mod 2^32
 *                 granules).  Arena positions strictly increase along every ring, so that is "has a pending record below
 *                 floor_bytes".  Every live entry of a selected agent moves, those above the cut included.  floor_bytes at
 *                 or below the floor selects nothing and moves nothing; floor_bytes >= the tail selects every agent with
 *                 pending records (a full compaction).
 *   2. Layout     the marked granules are the header of every moved record and the payload granules of every distinct
 *                 payload image a moved record names.  They are copied in arena order to a region placed at the tail as a
 *                 send's is (it never straddles the arena's wrap; the padding is skipped_bytes); the k-th goes to base + k.
 *                 A moved ring entry keeps its ring position, prio and record-granule bits; its handle and payload distance
 *                 are rewritten to the copies.  head / tail / ctail / ntomb do not change and tombstones stay as they are.
 *                 So a shared payload is copied once for all the moved members of its send, and
 *                 moved_bytes = 32 x (records + sum over distinct images of pad32(len) / 32) - the images are exactly the
 *                 rows a PEEK sdb_receive_compact of the selected agents returns (its contract point 2).
 *   3. Effect     every receive path (stream, priority, few-agent, latency server, compact, filtered, leased), expiry,
 *                 restore, lease sweeps, dead letters and digests give the records they would have given without the
 *                 call, byte for byte.  One thing differs in the compact format: when only some members of a shared-
 *                 payload group send moved, the moved members name the copy and the others the original, so a compact
 *                 result holding both returns that payload as two rows (its point 2); expanded, it is unchanged.  In
 *                 sdb_stats only arena_tail_bytes and arena_floor_bytes move; sdb_agent_loads and sdb_queue_stats do not
 *                 change.  Afterwards every pending record sits at or above min(floor_bytes, old tail) and
 *                 arena_floor_bytes = floor_after.  Entries of the dead-letter ledger that count a moved record follow it,
 *                 so delivery counts survive; the lease store keeps its own copies.
 *   4. All or nothing: the call plans on the device, synchronises once, then copies and rewrites.  A region that does not
 *                 fit behind the tail (tail + skip + moved - floor > arena, the floor recomputed) is SDB_EARENA_FULL and
 *                 changes nothing.  Copies never overlap a live granule, so a full arena cannot be compacted in place:
 *                 sdb_expire is the tool then.
 *   5. Flags      SDB_RECV_PEEK: a dry run that fills the whole summary, floor_after and tail_after as the call would leave
 *                 them, and writes nothing.  Any other bit: SDB_EINVAL.
 *   6. Ordering   stream-ordered on the handle's stream; synchronises.  The device cursor of the asynchronous import is
 *                 handed over as sdb_restore_compact does, so a later sdb_import_wire_ptrs_async places behind the moved
 *                 region; the call may sit between sdb_import_prefetch(step) and sdb_import_wire_ptrs_async(step).  Works
 *                 while the latency server runs.  Like a send it may overwrite the images sdb_overflow_log resolves: read
 *                 the log first.
 *   7. Memory     a granule bitmap, one u32 popcount and one u32 rank per bitmap word (3 x arena_bytes / 256 bytes: 12 MiB
 *                 for a 1 GiB arena) and one bit per agent, allocated on the first call.
 * The kernels are timed under SDB_PK_ARENA_FLOOR.  *out (nullable) receives the summary; it is zeroed on a refusal. */
typedef struct sdb_relocate_summary {
  uint64_t agents;          /* agents whose pending records moved */
  uint64_t records;         /* ring entries rewritten */
  uint64_t moved_bytes;     /* granules copied x SDB_GRANULE */
  uint64_t skipped_bytes;   /* tail padding of the wrap rule (a region never straddles the arena's wrap) */
  uint64_t floor_before, floor_after, tail_after;   /* bytes, the scale of sdb_stats.arena_*_bytes */
} sdb_relocate_summary;
int sdb_arena_relocate(sdb_handle h, uint64_t floor_bytes, uint32_t flags, sdb_relocate_summary* out);

/* ---- filtered receive: query_messages / search_messages / get_conversation / delete_message (M:671-808, M:1132-1157)
 * on the device queue itself, and selective receives ("my COMMAND messages", "what the coordinator sent me").
 * sdb_receive_where takes, for each listed agent (agent_idx == NULL: as in sdb_receive_batch), the first max_messages
 * pending records that match `filter`, in the call's delivery order (stream, or SDB_RECV_PRIORITY), and leaves every
 * other record queued in its order.
 *   Filter     the SDB_FILTER_* clauses named in `fields` are ANDed; fields == 0 matches every pending record.
 *   Keyword    matched against a record's content bytes: payload [0, len), or with SDB_TYPEF_EXTRAS the slice
 *              [4, 4 + clen), clen = the little-endian u32 at the payload's start clamped to len - 4 (empty when
 *              len < 4).  A keyword in the JSON extras, or across content and extras, does not match.  For JSON content
 *              the bytes are json.dumps(content).  SDB_FILTER_ICASE folds ASCII A-Z/a-z only; every other byte is
 *              compared exactly.  keyword_len == 0 matches every record.  Cost: up to len x keyword_len byte compares
 *              per record that passes the header clauses (a first-byte test skips most start positions).
 *   Contract   1. The result equals, byte for byte, what sdb_receive_batch returns on a queue holding only the matching
 *                 records, in its full format (count_out, 32-byte headers, payloads padded to SDB_GRANULE).
 *              2. Without SDB_RECV_PEEK the returned records are retired: every later receive (any path, any order)
 *                 delivers what it would have delivered had they been received.
 *              3. stats.delivered grows by the records returned; in sdb_agent_loads `pending` falls, `received` stays.
 *              4. Capacity: sdb_receive_batch's rule (lead-agent exception included) applies to the matches; loop
 *                 until *total_out == 0 to drain.
 *              5. Flags: SDB_RECV_PRIORITY, SDB_RECV_PEEK (a query: nothing retired), SDB_RECV_OWNED, SDB_WHERE_DROP.
 *              6. SDB_WHERE_DROP retires the matches without returning them: every output pointer but count_out must be
 *                 NULL, there is no capacity limit (max_messages still applies), stats do not move (as in sdb_expire's
 *                 drop mode) and *payload_bytes_out reads 0.  DROP | PEEK is a dry-run count.
 *              7. SDB_EINVAL: a NULL filter or a wrong struct_bytes, unknown bits in fields or flags, SDB_RECV_ASYNC, a
 *                 NULL keyword with keyword_len > 0, keyword_len > SDB_FILTER_MAX_KEYWORD, drop mode with output
 *                 buffers, an agent listed twice or out of range; SDB_FILTER_IDS with the old struct_bytes, NULL ids (even
 *                 with n_ids == 0), n_ids > SDB_FILTER_MAX_IDS, id_hits or id_agent without SDB_FILTER_IDS.  SDB_EOUTPUT as
 *                 in sdb_receive_batch.
 *              8. The call always runs the bulk kernels (never the few-agent or latency-server paths); sdb_digest_fold
 *                 after it returns SDB_EINVAL until the next sdb_receive_batch.
 *   Ids        SDB_FILTER_IDS matches the records whose seq is one of ids[0, n_ids): get_message / delete_message by id
 *              on the device queue, many ids in one call.  ids is never NULL; duplicates are allowed, n_ids == 0 and id 0
 *              (never a seq) match nothing.  The call builds an open-addressing hash table of the ids on the device (next power of two
 *              >= 2 x n_ids slots of 16 bytes), and every record that passes the other header clauses costs one probe,
 *              O(1) expected reads.  Per-id outputs (host arrays of n_ids, each nullable, only with the clause):
 *                id_hits[i]   pending records of the listed agents with seq == ids[i] that pass every clause, counted
 *                             when the records are evaluated: before max_messages and the capacity cut.  In drop mode
 *                             with max_messages >= ring_slots it is the number of copies dropped.
 *                id_agent[i]  the smallest agent index holding such a record, else SDB_NO_RECEIVER.
 *              Duplicate ids read the same values.  A call that returns before running (no agents, max_messages == 0)
 *              writes 0 and SDB_NO_RECEIVER.  Only pending records are found: a leased (in flight) or dead-lettered
 *              record is not, and a deleted id that is leased elsewhere comes back only through its lease.
 *              struct_bytes == offsetof(sdb_filter, n_ids), the size before this block, is still accepted, without
 *              SDB_FILTER_IDS.
 *   Memory     one verdict bit per ring slot (max_agents x ring_slots bits) and a 256-byte keyword buffer, allocated on
 *              the first call; with SDB_FILTER_IDS the id table, the ids and the per-id outputs (at most 80 bytes per id
 *              at the largest n_ids so far), allocated on the first call that needs them and grown on demand. */
#define SDB_FILTER_SENDER   1u          /* header.sender == sender */
#define SDB_FILTER_RECEIVER 2u          /* header.receiver == receiver (SDB_NO_RECEIVER: broadcast copies) */
#define SDB_FILTER_GROUP    4u          /* header.group == group (SDB_NO_GROUP: non-group sends) */
#define SDB_FILTER_TYPE     8u          /* bit (header.type & SDB_TYPE_MASK) of type_mask set */
#define SDB_FILTER_PRIO     16u         /* bit header.prio of prio_mask set */
#define SDB_FILTER_TIME     32u         /* after < timestamp < before, both strict: a NaN never matches */
#define SDB_FILTER_SEQ      64u         /* seq_lo <= seq < seq_hi */
#define SDB_FILTER_KEYWORD  128u        /* keyword occurs in the content bytes */
#define SDB_FILTER_ICASE    256u        /* keyword compare folds ASCII A-Z/a-z only; every other byte is compared exactly */
#define SDB_FILTER_IDS      512u        /* seq is one of ids[0, n_ids) */
#define SDB_FILTER_MAX_KEYWORD 256u
#define SDB_FILTER_MAX_IDS  4194304u    /* n_ids at most */
#define SDB_WHERE_DROP 32u              /* flag: retire the matches without returning them */
typedef struct sdb_filter {
  uint32_t struct_bytes;    /* sizeof(sdb_filter), or offsetof(sdb_filter, n_ids) without SDB_FILTER_IDS */
  uint32_t fields;          /* SDB_FILTER_* clauses that apply (ANDed); 0 matches every pending record */
  uint32_t sender;          /* SDB_FILTER_SENDER */
  uint32_t receiver;        /* SDB_FILTER_RECEIVER */
  uint32_t group;           /* SDB_FILTER_GROUP */
  uint8_t  type_mask;       /* SDB_FILTER_TYPE */
  uint8_t  prio_mask;       /* SDB_FILTER_PRIO */
  uint16_t keyword_len;     /* SDB_FILTER_KEYWORD: 0 .. SDB_FILTER_MAX_KEYWORD */
  double   after, before;   /* SDB_FILTER_TIME */
  uint64_t seq_lo, seq_hi;  /* SDB_FILTER_SEQ */
  const uint8_t* keyword;   /* host pointer */
  uint64_t n_ids;           /* SDB_FILTER_IDS: 0 .. SDB_FILTER_MAX_IDS */
  const uint64_t* ids;      /* host pointers, [n_ids] each */
  uint32_t* id_hits;
  uint32_t* id_agent;
} sdb_filter;
int sdb_receive_where(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages, uint32_t flags,
                      const sdb_filter* filter,
                      uint32_t* count_out, sdb_msg_header* hdr_out, uint64_t hdr_cap,
                      uint8_t* payload_out, uint64_t payload_cap, uint64_t* total_out, uint64_t* payload_bytes_out);
/* Filtered receive by budget ("the FUNCTION_RESULT messages the coordinator sent me, up to 4k tokens"):
 * sdb_receive_where's arguments plus max_agent_bytes and max_agent_tokens.
 *   1. Take: per agent, over its pending records that match the filter, in the call's delivery order, the shortest of
 *      max_messages, the byte take (the longest prefix with sum(pad32(len)) <= max_agent_bytes) and the token take
 *      (sdb_receive_tokens' weights and 64-bit sums).  A budget take is the first match alone when that match is heavier
 *      than its limit; a limit of 0 is no limit.  In priority order that is whole levels from the top while they fit,
 *      then the arrival-order prefix of the level where a limit falls.
 *   2. Equivalence: the result is exactly sdb_receive_where with each agent's max_messages lowered to its take (records,
 *      order, bytes, retirement, counters, rings, capacity and its lead-agent rule, id_hits / id_agent, which count the
 *      matches before the cut).  Capacity is sdb_receive_where's records x pad32(max_payload_bytes) rule.
 *   3. Both limits 0: the call is sdb_receive_where.
 *   4. Flags and refusals as in sdb_receive_where (SDB_RECV_PEEK, SDB_RECV_OWNED and SDB_WHERE_DROP included).  With a
 *      limit, a pass between the filter's evaluation and the selection walks each agent's matches and cuts its count;
 *      it reads ring entries and verdict bits, and with a token limit the header's last word and the payload's first
 *      word of each match.  It is timed under SDB_PK_RECV_COUNT. */
int sdb_receive_where_budget(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                             uint64_t max_agent_bytes, uint64_t max_agent_tokens, uint32_t flags, const sdb_filter* filter,
                             uint32_t* count_out, sdb_msg_header* hdr_out, uint64_t hdr_cap, uint8_t* payload_out,
                             uint64_t payload_cap, uint64_t* total_out, uint64_t* payload_bytes_out);

/* ---- LLM backend balancer: set_llm_load_balancing / assign_llm_backend / get_llm_backend
 * (M:1281-1325).  The reference stores a flag and a dict and has NO pick algorithm
 * (SURVEY 0.5); the per-agent sticky map stays in the Python layer, and these entry points
 * add the batched pick over live load counters:
 *   mode 0  weighted least-load: requests are served in index order, each goes to
 *           argmin_b load[b]/weight[b] (exact rational compare, ties -> lowest index) and adds
 *           cost[i] (NULL = 1) to that backend's load;
 *   mode 1  weighted random (one-item weighted reservoir, Efraimidis-Spirakis exponential
 *           race in integer fixed point): P(b) proportional to weight[b], keyed by
 *           (seed, request index); loads are then incremented atomically.
 * A handle holds at most SDB_MAX_BACKENDS backends (sdb_create refuses a larger max_backends with SDB_EINVAL).
 * Weights are in [1, 65535] and initial loads below 2^40; loads then grow with the costs of the picks, and the
 * compares stay exact for any 64-bit load.
 */
#define SDB_MAX_BACKENDS 4096u
int sdb_set_backends(sdb_handle h, uint32_t n, const uint32_t* weight, const uint64_t* load0);
int sdb_get_backend_loads(sdb_handle h, uint32_t n, uint64_t* load_out);
int sdb_release_backends(sdb_handle h, uint32_t n, const uint32_t* backend, const uint32_t* cost /* NULL = 1 */);
int sdb_select_backend_batch(sdb_handle h, uint32_t n_req, const uint32_t* cost, uint32_t mode,
                             uint64_t seed, uint32_t* backend_out);
/* "get_agent_load is the only load signal" (SURVEY 8a R10, M:1049-1094): feed the balancer from the queue itself.
 * sdb_assign_agent_backends is the device copy of the sticky agent -> backend map (assign_llm_backend, M:1293-1311;
 * backend index, or 0xFFFFFFFF = none).  sdb_backend_loads_from_queues sets load[b] = sum of the pending records of the
 * agents assigned to b (one pass over the ring headers, stream-ordered, no host round trip); picks then see real
 * backlog.  Call it before sdb_select_backend_batch whenever the loads should track the queues. */
int sdb_assign_agent_backends(sdb_handle h, uint32_t n, const uint32_t* agent_idx, const uint32_t* backend_idx);
int sdb_backend_loads_from_queues(sdb_handle h);

/* ---- deduplicated sends: a producer names a message with a 128-bit key, and a second send with a key the table holds
 * as a live entry is not written (SQS MessageDeduplicationId, NATS Msg-Id).  Off until sdb_dedup_reserve.
 *   sdb_dedup_reserve           a table of `entries` keys (load factor at most 1/2, 32 bytes a slot, two buffers) with
 *                               the given window (> 0 s); 0 entries frees it.  Either clears the table.
 *   sdb_send_mixed_batch_dedup  sdb_send_mixed_batch's arguments up to timestamp, then one key per send (NULL: every key
 *                               {0,0}), and seq_base_out last.  A send
 *                               with key {0,0} bypasses the table unless SDB_DEDUP_CONTENT gives it its content key (the
 *                               hash of sender, kind, target or the list's recipients, len, prio, type and payload; not
 *                               the timestamp; INTEGRATION.md §3.9).  A send is a duplicate when the table holds its key
 *                               as an entry live at `now` (now < inserted_at + window), or when an earlier send of the
 *                               batch has the key.  Accepted sends are written exactly as sdb_send_mixed_batch writes the
 *                               batch without the duplicates, with the sequence numbers the whole batch gives them; a
 *                               duplicate's numbers stay unused, and it writes nothing and is not counted in `enqueued`.
 *                               dup_of_out[i]: the first seq of the original send (0: accepted); key_out[i]: the key
 *                               used; *n_dup_out: duplicates.  Then every accepted keyed send stores (key, its first seq,
 *                               now); when the new keys would take the occupied slots past `entries`, a rebuild first
 *                               drops the entries not live at `now`.  Refusals leave rings, arena, the seq counter, the
 *                               table and sdb_dedup_stats unchanged, and sdb_stats too except kernel_launches, which
 *                               counts the probe (and counting) kernels a refused call ran: SDB_EARENA_FULL,
 *                               SDB_ECAPACITY (the new keys do not fit beside the live entries), SDB_EINVAL (no table, a
 *                               non-finite now, unknown flags, a non-zero key or SDB_DEDUP_CONTENT on a sharded handle,
 *                               or any argument sdb_send_mixed_batch refuses).
 *   sdb_dedup_forget            kill the entries of the given keys; removed_out[i] = 1 where the entry was live at the
 *                               `now` of the last send call.
 *   sdb_dedup_stats             capacity, entries live at the last send call's `now`, occupied slots and totals.
 * Restores, requeues, lease redeliveries, redrives and cross-shard imports neither consult nor fill the table, and
 * expiry or delete-by-id remove no key.  Snapshots do not carry it.  Kernels are timed under SDB_PK_DEDUP. */
typedef struct sdb_dedup_key { uint64_t lo, hi; } sdb_dedup_key;      /* {0,0}: not deduplicated */
#define SDB_DEDUP_CONTENT 1u          /* sends whose key is {0,0} (all of them when key == NULL) get the content key */
typedef struct sdb_dedup_summary {
  uint64_t capacity;            /* entries the table takes */
  uint64_t live;                /* entries live at the last send call's now */
  uint64_t used;                /* occupied slots: live, expired and forgotten entries until a rebuild drops them */
  double window;                /* seconds */
  uint64_t accepted_total;      /* keyed sends accepted (entries stored) */
  uint64_t duplicate_total;     /* sends refused as duplicates */
  uint64_t expired_total;       /* entries dropped by rebuilds (expired or forgotten) */
  uint64_t forgotten_total;     /* entries killed by sdb_dedup_forget */
  uint64_t rebuilds;
} sdb_dedup_summary;
int sdb_dedup_reserve(sdb_handle h, uint64_t entries, double window_seconds);
int sdb_send_mixed_batch_dedup(sdb_handle h, uint32_t n, const uint32_t* sender, const uint8_t* kind, const uint32_t* target,
                               uint32_t n_lists, const uint64_t* list_off, const uint32_t* list_idx, const uint8_t* prio,
                               const uint8_t* type, const uint16_t* len, const uint64_t* payload_off, const uint8_t* payload,
                               uint64_t payload_bytes, const double* timestamp,
                               const sdb_dedup_key* key /* [n], nullable */, uint32_t flags, double now,
                               sdb_dedup_key* key_out /* [n], nullable */, uint64_t* dup_of_out /* [n], nullable */,
                               uint32_t* n_dup_out, uint64_t* seq_base_out);
int sdb_dedup_forget(sdb_handle h, uint64_t n, const sdb_dedup_key* key, uint8_t* removed_out /* [n], nullable */);
int sdb_dedup_stats(sdb_handle h, sdb_dedup_summary* out);

#ifdef __cplusplus
}
#endif
#endif /* SWARMDB_B200_H */
