// sdb_common.cuh - shared device/host definitions for the sm_90a kernels.
//
// HBM layout of one shard (all sizes powers of two where masks are used):
//
//   arena        uint8 [arena_bytes]      packed message records, 32-byte granules, written
//                                         strictly sequentially in global send order (a log).
//                                         record = sdb_msg_header (32 B) | payload pad32.
//                                         position `apos` (granules, monotonic u64);
//                                         byte address = arena + ((apos & gmask) << 5);
//                                         a batch never straddles the wrap point.
//   ring_hdr     16 B   [max_agents]      {head, tail, ctail, ntomb}: monotonic per-agent cursors, ONE 16-byte
//                                         load per agent for every kernel.  {head, tail} is also one aligned 64-bit
//                                         word: an atomicAdd(1<<32) on it claims a slot and returns head in the
//                                         same L2 transaction (enqueue paths that are not rank-ordered).
//                                         ctail = tail as of the last commit; ntomb = consumed entries still
//                                         inside [head, tail) (holes left by priority receives).
//   ring         8 B    [max_agents][R]   one entry per pending record: {handle = (uint32)apos,
//                                         meta = prio<<14 | record_granules, 0xFFFF = consumed}.  Interleaved so
//                                         the few entries an agent gains/loses per batch share one 32-byte sector.
//   members      uint32 [member_pool]     group member lists (CSR kept on the host)
//
// Ordering contract: after `commit`, every ring is sorted by handle, i.e. by arena
// position, i.e. by global send order (the reference's single-partition Kafka log order,
// SURVEY App. A rule 7).  Enqueue kernels claim slots with atomics in arbitrary order;
// the commit kernel sorts the few entries each agent received in the batch.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/swarmdb_b200.h"

#define SDB_META_TOMB 0xFFFFu
#define SDB_META_GLEN_MASK 0x3FFFu

// per-send descriptor staged to the device (64 B, one per send); q1 is all the index-build
// kernel needs, so it reads 16 bytes per (agent, send) pair
struct __align__(16) sdb_send_desc {
  // q0
  uint64_t payload_off;  // byte offset into the batch payload buffer, 16-B aligned
  double   timestamp;
  // q1
  uint32_t gran0;        // arena granule offset of member 0 relative to the batch arena base
  uint32_t sender;
  uint32_t rgran;        // granules per record = 1 + pad32(len)/32
  uint16_t len;
  uint8_t  prio;
  uint8_t  type;
  // q2
  uint32_t rec0;         // seq offset of member 0 relative to the batch seq base
  uint32_t mstart;       // first member in the member pool (group/list) or receiver idx (p2p)
  uint32_t mcount;       // members (1 for p2p)
  uint32_t group;        // group index or SDB_NO_GROUP
  // q3
  uint32_t flags;        // SDB_DESC_*
  uint32_t pad0;
  uint64_t seq_abs;      // SDB_DESC_ABS_SEQ: absolute sequence number of member position 0 (instead of seq_base + rec0)
};
static_assert(sizeof(sdb_send_desc) == 64, "desc must be 64 bytes");
static_assert(sizeof(sdb_msg_header) == 32, "header must be 32 bytes");
static_assert(sizeof(sdb_recv_entry) == 16 && sizeof(sdb_recv_send) == 32, "compact receive entries must be 16 and 32 bytes");

#define SDB_DESC_SKIP_SENDER 1u   // group send: member == sender is skipped (M:1268)
#define SDB_DESC_SHARED_SEQ 2u    // broadcast: every copy carries the same seq (one Message)
#define SDB_DESC_LIST_TEMP 4u     // mstart indexes the per-batch temporary list buffer
#define SDB_DESC_PULL 8u          // ring entries are built by k_pull_index, not by the fan-out kernel
#define SDB_DESC_RANKED 32u       // p2p: pad0 = rank of this send among the batch's sends to the same receiver (ring slot = ctail + rank)
#define SDB_DESC_RANK_LAST 64u    // p2p: highest rank for its receiver (count = rank + 1): this send publishes the ring tail
#define SDB_DESC_POS 16u          // seq offset of member k is member_pos[mstart + k] (sharded: original group position)
#define SDB_DESC_P2P 32u          // wire batches only: point-to-point send, mstart = receiver index
#define SDB_DESC_ABS_SEQ 64u      // seq_abs holds the sequence number (sources that number their own sends)

// cross-shard wire batch (device memory, moved between ranks by the caller):
//   [sdb_wire_header 128 B][n_sends x sdb_send_desc 64 B][group buckets][broadcast lists][payload bytes]
// descriptors use: payload_off (relative to the wire payload), timestamp, sender, group, rgran,
// len, prio, type, rec0 (seq offset inside the source's batch, counted in FULL group sizes)
struct __align__(16) sdb_wire_header {
  uint32_t magic;          // 'SDBW'
  uint32_t n_sends;
  uint64_t total_recs;     // sequence numbers this batch consumes (sum of full group sizes)
  uint64_t payload_bytes;
  uint64_t desc_off;       // byte offsets from the start of the wire batch
  uint64_t payload_off;
  uint32_t max_padlen;
  uint32_t n_other;        // sends that are not group sends (p2p / broadcast lists)
  uint64_t list_off;       // recipient lists of broadcast sends (uint32 agent indices)
  uint32_t n_list;
  uint32_t n_group_sends;
  uint64_t gs_off_off;     // group-send buckets of THIS batch: offsets [max_groups + 1] ...
  uint64_t gs_idx_off;     // ... and send indices, ascending inside a bucket (built by the exporter)
  uint32_t max_groups;
  uint32_t explicit_seq;   // 1: this batch's sends are numbered from seq_base (assigned by the exporter at send time)
  uint64_t seq_base;
  uint32_t pad[8];
};
static_assert(sizeof(sdb_wire_header) == 128, "wire header must be 128 bytes");
#define SDB_WIRE_MAGIC 0x57424453u

// per-batch view for the agent-parallel index build ("pull"): group sends of the batch bucketed
// by group (gs_*), and the inverse of the group table (which groups/positions an agent is in)
struct sdb_pull_view {
  const uint32_t* memb_off;   // [max_agents + 1]
  const uint32_t* memb_grp;   // [memberships]
  const uint32_t* memb_pos;   // [memberships] position of the agent inside that group's member list
  const uint32_t* gs_off;     // [n_src][gs_off_stride] bucket offsets into gs_idx, one table per source
  const uint32_t* gs_idx;     // [n_src][gs_idx_stride] send indices (relative to the source's first send), ascending inside a bucket
  // The group-parallel index build walks the sources' buckets in source order (= global send order), so a
  // cross-shard import never concatenates them.  One source (n_src = 1, first[0] = 0) is the single-GPU case.
  uint32_t n_src, gs_off_stride, gs_idx_stride;
  const uint32_t* first;      // [n_src] global descriptor index of each source's first send (device), or nullptr = {0}
};

struct sdb_dev_counters {   // device-resident, updated with atomics
  unsigned long long enqueued;
  unsigned long long delivered;
  unsigned long long ring_overflow;
  unsigned long long skipped_sender;
  unsigned long long backend_picks;
  unsigned long long ovf_logged;    // records dropped since the overflow log was last read (the first SDB_OVF_LOG are logged)
  unsigned long long pad[2];
};
#define SDB_OVF_LOG 4096u

// everything a kernel needs about the shard, passed by value
struct __align__(16) sdb_ring_hdr { uint32_t head, tail, ctail, ntomb; };
static_assert(sizeof(sdb_ring_hdr) == 16, "ring header must be 16 bytes");

struct sdb_dev_view {
  uint8_t*  arena;
  sdb_ring_hdr* ring_hdr;       // [max_agents]
  uint2*    ring;               // [max_agents][R]  .x = handle, .y = meta (SDB_META_TOMB: consumed)
  const uint32_t* members;
  const uint32_t* member_pos;   // sharded mode: original group position of members[k]; else nullptr
  sdb_dev_counters* ctr;
  uint2*    ovf_log;     // [SDB_OVF_LOG] {agent, arena handle} of records whose ring was full (sdb_overflow_log)
  uint64_t gmask;        // arena granules - 1
  uint32_t ring_slots;   // R
  uint32_t ring_shift;   // log2 R
  uint32_t max_agents;
};

// arguments of one receive call (scratch + outputs), shared by sdb_api.cu and sdb_recv.cu
struct sdb_recv_args {
  const uint32_t* agent_idx;   // [n] or nullptr (identity)
  uint32_t n;
  uint32_t max_messages;
  uint32_t flags;
  uint32_t* cnt;               // [n] records selected per agent                 (multi-kernel path scratch)
  uint32_t* rec_local;         // [n] scan of cnt (block-local part)             (multi-kernel path scratch)
  uint32_t* rec_tops;          // [tiles] scan of cnt (per-block part)           (multi-kernel path scratch)
  uint32_t* rec_off;           // [n] index of the agent's first output record (both paths)
  // per-record plan, indexed by output record number r = rec_off[slot] + rank:
  //   .x arena handle, .y payload offset in the packed output (granules; the multi-kernel path stores the
  //   tile-local part and adds plan_tops[r / tile]), .z payload granules, .w request slot
  uint4* plan;                 // [rec_cap]
  uint32_t* plan_tops;         // [rec tiles] or nullptr (single-pass path: .y is already absolute)
  unsigned long long* totals;  // [0] records delivered, [1] payload granules delivered, [2..] scratch
  uint32_t* big_list;          // [n] request slots that need the warp-per-agent selector
  uint32_t* big_count;         // [1]
  unsigned long long* lb;      // [tiles + 2] single-pass path: decoupled look-back status words (zero between calls),
                               //             then the tile ticket counter and the packed totals (see k_recv_plan)
  // outputs
  uint32_t* count_out;         // [n]
  sdb_msg_header* hdr_out;     // [rec_cap]
  uint8_t* payload_out;        // [rec_cap * pad32(max_payload)]
  uint64_t rec_cap;
};

// scratch + outputs of a compact receive (sdb_receive_compact), all indexed by output record number unless noted
struct sdb_compact_args {
  unsigned long long* table;   // [2^tbits] open addressing: payload position p << 32 | smallest record naming it; ~0 = empty
  uint32_t tbits;
  uint32_t* rec_slot;          // table slot of each record, then (k_compact_heads) the record that owns its image
  uint32_t* head;              // 1 where a record owns its image (first appearance)
  uint32_t* head_local;        // exclusive scan of head = row index (block-local part) ...
  uint32_t* head_tops;         // ... and per-tile part
  uint32_t* gran;              // payload granules of the image at its owner, 0 elsewhere
  uint32_t* gran_local;        // exclusive scan of gran = payload offset in granules (block-local part) ...
  uint32_t* gran_tops;         // ... and per-tile part
  unsigned long long* totals;  // [0] rows, [1] payload granules
  sdb_recv_entry* entry_out;   // [rec_cap]
  sdb_recv_send* send_out;     // [rec_cap]
  uint8_t* payload_out;        // [rec_cap * pad32(max_payload)]
};

// filter of a filtered receive (sdb_receive_where) as the kernels read it, plus the verdict bitmap
struct sdb_where_args {
  uint32_t fields;             // SDB_FILTER_* (KEYWORD only with kw_len > 0)
  uint32_t sender, receiver, group;
  uint32_t type_mask, prio_mask, kw_len;
  double after, before;
  unsigned long long seq_lo, seq_hi;
  const uint8_t* kw;           // [kw_len] device copy of the keyword (unfolded)
  uint32_t* bits;              // [max_agents][stride] bit j of agent a: the record at head + j matches
  uint32_t stride;             // words per agent = ceil(ring_slots / 32)
  struct sdb_id_slot* id_tab;  // SDB_FILTER_IDS: open-addressing table [id_mask + 1] of the listed ids
  uint32_t id_mask;            // table slots - 1 (a power of two >= 2 x the ids)
  uint32_t id_count;           // 1: every match adds to its id's hit counter and first agent
};

// one slot of the id table of SDB_FILTER_IDS: key 0 is an empty slot (seq 0 is never assigned).  nagent holds ~agent so
// that the zeroed table reads SDB_NO_RECEIVER and atomicMax keeps the smallest agent.
struct __align__(16) sdb_id_slot {
  unsigned long long key;
  uint32_t hits, nagent;
};

// superseding (sdb_supersede): one key of the open-addressing table, {0,0} empty (a key has bit 63 of hi set), the
// largest seq of its records and the largest ring offset among the records holding that seq
struct __align__(16) sdb_ss_slot {
  unsigned long long klo, khi;
  unsigned long long seq;
  uint32_t off, pad;
};
// one flagged pending record: its seq, request slot, ring offset from the head and table slot
struct sdb_ss_cand {
  unsigned long long seq;
  uint32_t q, j, slot, pad;
};
struct sdb_ss_args {
  sdb_ss_slot* tab;            // [mask + 1] zeroed, a power of two >= 2 x n_cand
  uint32_t mask;
  sdb_ss_cand* cand;           // [n_cand] in request-slot order
  uint32_t n_cand;
  uint32_t* bits;              // verdict bitmap, the layout of sdb_where_args::bits: bit j of agent a is superseded
  uint32_t stride;
};

// arguments of one restore (sdb_restore_compact): the compact-format input staged in the compact receive's buffers, the
// per-agent tables uploaded by the host, and scratch carved out of the compact receive's scratch (sdb_api.cu)
struct sdb_restore_args {
  const uint32_t* agent;           // [n] listed agents
  const uint32_t* count;           // [n] entries of each
  const uint32_t* first;           // [n] index of the agent's first entry (exclusive scan of count)
  const sdb_recv_entry* ent;       // [n_entries]
  const sdb_recv_send* snd;        // [n_sends]
  const uint8_t* payload;          // [payload_bytes]
  uint64_t payload_bytes;
  uint32_t n, n_entries, n_sends, max_payload;
  uint32_t shared;                 // 1: rows take the shared layout (headers + one payload); 0: every record is a private image
  uint32_t owned, shard_id;        // owned: skip the agents whose shard_of[] is not shard_id
  const uint8_t* shard_of;
  uint32_t* nsh;                   // [n] entries in the agent's shared prefix (before its first row descent)
  uint32_t* pgran;                 // [n] granules of the agent's private images, then its scan (p_local / p_tops)
  uint32_t* p_local; uint32_t* p_tops;
  uint32_t* e_row;                 // [n_entries] row of a shared entry, ~0 for private / skipped entries
  uint32_t* row_cnt;               // [n_sends] shared entries per row, then its scan (rc_local / rc_tops): bucket base
  uint32_t* rc_local; uint32_t* rc_tops;
  uint32_t* row_gran;              // [n_sends] granules of the row's region, then its scan (rg_local / rg_tops): arena offset
  uint32_t* rg_local; uint32_t* rg_tops;
  uint32_t* key_a; uint32_t* key_b;  // [n_entries] stable radix sort of the entries by row (non-shared entries key n_sends) ...
  uint32_t* val_a; uint32_t* val_b;  // ... carrying entry indices: afterwards row r's shared entries sit, in entry order, at
                                     // [rc_local/rc_tops scan of r, + row_cnt[r])
  uint32_t* hist; uint32_t* h_local; uint32_t* h_tops;   // [256 x sort tiles] digit counts per tile (digit-major) and scan
  uint32_t* e_handle;              // [n_entries] arena handle of each shared entry's header ...
  uint32_t* e_y;                   // ... and its ring entry's .y (meta | dm1 << 16)
  unsigned long long* tot;         // [0] row granules [1] private granules [2] largest seq [3] error bits [4] records [5] shared
  unsigned long long base;         // arena position of the region (write phase)
};
#define SDB_RS_EINVAL 1ull         // tot[3]: a bad entry or row
#define SDB_RS_ERING 2ull          // tot[3]: some agent's ring cannot take its records

// ---- deduplication table (sdb_dedup.cu): one 32-byte entry per key, key {0,0} = empty slot
struct __align__(32) sdb_dedup_entry {
  sdb_dedup_key key;
  unsigned long long seq;          // first seq of the send that stored the key
  double at;                       // inserted_at; -inf once forgotten
};
static_assert(sizeof(sdb_dedup_entry) == 32, "dedup entry must be one 32-byte sector");
// what the content key reads of a send (staged by the host, 32 bytes)
struct __align__(16) sdb_dedup_send {
  uint64_t payload_off;
  uint64_t list_b;                 // kind 2: first recipient in `lists`
  uint32_t sender;
  uint32_t target;                 // receiver (kind 0), group (kind 1) or the list's length (kind 2)
  uint32_t lpt;                    // len | prio << 16 | type << 24
  uint32_t kind;
};
#define SDB_DD_BATCH (1ull << 63)  // verdict: SDB_DD_BATCH | index of the earlier send of the batch with the same key
enum : uint32_t { SDB_DD_USED = 0, SDB_DD_NEW = 1, SDB_DD_FORGOT = 2, SDB_DD_LIVE = 3, SDB_DD_CTRS = 4 };
struct sdb_dedup_args {
  sdb_dedup_entry* tab;            // [mask + 1] the current buffer
  unsigned long long mask;
  double window;
  sdb_dedup_key* key;              // [max_batch_sends] keys of the call (content keys filled in on the device)
  const sdb_dedup_send* snd;       // [max_batch_sends]
  const uint8_t* payload;          // the batch payload
  const uint32_t* lists;           // the batch's recipient lists
  sdb_dedup_key* btab;             // [bmask + 1] keys of the batch ...
  uint32_t* bmin;                  // ... and the lowest send index holding each
  unsigned long long bmask;
  uint32_t* bslot;                 // [max_batch_sends] batch-table slot of each send
  unsigned long long* verdict;     // [max_batch_sends]
  const unsigned long long* seq_of;  // [max_batch_sends] first seq of each send (insert)
  unsigned long long* ctr;         // [SDB_DD_CTRS]
};

// ---- lease store (sdb_receive_leased / sdb_lease_settle / sdb_lease_sweep, sdb_lease.cu): one of its two buffers.  Entries
// are in lease-id order (append-only, then stable compaction); rows and payloads in the compact receive format.
#define SDB_LS_LIVE 0u
#define SDB_LS_ACKED 1u
#define SDB_LS_REDELIVERED 2u
#define SDB_LS_DEAD 3u                 // past the redelivery limit (sdb_lease_set_policy): kept until sdb_lease_dead_letters
struct sdb_lease_buf {
  sdb_recv_entry* ent;             // [cap] seq, store row, receiver
  uint32_t* agent;                 // [cap]
  unsigned long long* id;          // [cap] lease ids, ascending
  double* deadline;                // [cap]
  uint32_t* state;                 // [cap] SDB_LS_*
  sdb_recv_send* rows;             // [cap] payload_off into `payload`
  uint8_t* payload;                // [payload cap]
  uint32_t* deliveries;            // [cap] delivery count of each lease; nullptr while no policy is set
};
// ---- redelivery ledger (sdb_lease_set_policy): the delivery count of every record a sweep put back, keyed by
// (agent, seq), with the ring position p and arena handle restore gave it.  Dense entries in any order (a collection
// rebuilds them into `alt` and swaps), plus an open-addressing index over them (load factor <= 1/2).
struct sdb_ledger_ent {
  unsigned long long seq;
  uint32_t agent;
  uint32_t count;                  // delivery count at redelivery; 0: taken by a leased receive
  uint32_t p;                      // absolute ring position
  uint32_t handle;                 // arena handle of the ring entry at p
};
static_assert(sizeof(sdb_ledger_ent) == 24, "ledger entries are 24 bytes");
struct sdb_ledger {
  sdb_ledger_ent* ent;             // [cap]
  sdb_ledger_ent* alt;             // [cap]
  uint32_t* index;                 // [slots] entry numbers, ~0 = empty
  uint32_t slots;                  // 2 x cap
  unsigned long long* tot;         // [2] entries kept by the last collection, entries taken by lookups since
};
// scratch of a dead-letter readout (sdb_lease_dead_letters), allocated with the policy: [cap] sort keys / values and
// staged entries, radix digit tables for cap keys, [max_agents] list positions (~0 between calls) and per-position counts
struct sdb_dl_scratch {
  uint32_t *key_a, *key_b, *val_a, *val_b, *staged;
  uint32_t *hist, *h_local, *h_tops;
  uint32_t *pos, *cnt;
};
// scratch of the store's kernels; S = max(cap, max_recv_records), R = max_recv_records
struct sdb_lease_scratch {
  uint32_t* flag; uint32_t* f_local; uint32_t* f_tops;     // [S] entry or position flags and their scan
  uint32_t* gran; uint32_t* g_local; uint32_t* g_tops;     // [S] row flags / granules and their scan
  uint32_t* rfirst; uint32_t* rmap;                        // [cap] per store row: first seq-sorted position, new index
  uint32_t* rg; uint32_t* rg_local; uint32_t* rg_tops;     // [cap] compaction: granules of each kept row and their scan
  uint32_t* chunk; uint32_t* staged;                       // [R] store entry of each chunk / staged position
  uint32_t* key_a; uint32_t* key_b; uint32_t* val_a; uint32_t* val_b;   // [R] radix sort
  uint32_t* hist; uint32_t* h_local; uint32_t* h_tops;     // radix sort digit tables
  uint32_t* run_begin;                                     // [R + 1] first chunk position of each agent run
  uint32_t* kcnt; uint32_t* k_local; uint32_t* k_tops;     // [R] entries each run keeps, and their scan
  uint32_t* kflag; uint32_t* kf_local; uint32_t* kf_tops;  // [R] 1 for a kept run, and the scan
  uint32_t* a_local; uint32_t* a_tops;                     // [max_agents] append: scan of the receive's counts
  unsigned long long* req;                                 // [SDB_LS_SETTLE_CHUNK] settle: lease ids ...
  uint32_t* at;                                            // ... their store entries ...
  uint8_t* settled;                                        // ... and the verdicts
  unsigned long long* tot;                                 // [16]
};
#define SDB_LS_SETTLE_CHUNK (1u << 20)

// ---- relocation of pinned queues (sdb_arena_relocate, sdb_relocate.cu): the marked granules of one call, as a bitmap over
// arena positions [lo, tail] (bit k = position lo + k, lo a multiple of 32), and the rank of each word (an exclusive scan of
// their popcounts, block-local part in `pre`, per-tile part in `tops`): a marked granule at position x moves to base + rank(x)
struct sdb_reloc_args {
  uint32_t* bits;                  // [words]
  uint32_t* cnt;                   // [words] popcount of each word
  uint32_t* pre;                   // [words] its exclusive scan (block-local part)
  uint32_t* tops;                  // [sdb_scan_tops_len(words)]
  uint32_t* sel;                   // [ceil(n_agents / 32)] bit a: agent a is selected
  unsigned long long* tot;         // [0] marked granules [1] agents [2] records [3] largest distance below the tail of an
                                   // agent's oldest pending record [4] the same over unselected agents (0: none pending)
  unsigned long long lo, tail;     // granules
  uint32_t words;                  // (tail - lo) / 32 + 1
  uint32_t thr;                    // an agent is selected when its oldest pending header lies more than thr below the tail
  uint32_t n_agents;
  unsigned long long base;         // write phase: where the first marked granule goes
};

// ---- asynchronous import (sdb_import_wire_ptrs_async): everything the host used to learn through a sync lives on
// the device.  `sdb_cursor` is the device-resident twin of the host's arena / sequence counters (whoever advanced
// them last marks the other side stale); `sdb_batch_base` carries one import's placement from the kernel that
// computes it (k_import_fused) to the kernels that follow (fan-out, index build, commit).
struct sdb_cursor {
  unsigned long long arena_tail;    // granules, monotonic
  unsigned long long arena_floor;   // granules: everything below is reclaimed
  unsigned long long next_seq;
  unsigned long long error;         // sticky bits: 1 = an import did not fit the arena (dropped whole), 2 = recipient-list pool exhausted
  unsigned long long floor_dist;    // scratch of the floor scan: max distance of a pending record below the tail
  unsigned long long pad[3];
};
struct sdb_batch_base {
  unsigned long long arena_base;    // granule position of the import's first record
  unsigned long long seq_base;      // sequence number the import's relative numbers count from
  uint32_t n_total;                 // localized descriptors (sends) of the import
  uint32_t n_other;                 // point-to-point / broadcast sends among them (their ring entries need the commit sort)
  uint32_t skip;                    // 1: refused (see sdb_cursor.error) - the following kernels do nothing
  uint32_t max_padlen;
  unsigned long long total_grans, total_recs;
};
// grand totals of one localized import, kept between a prefetch (k_import_fused on the prefetch stream, while the previous
// step still runs) and its placement (k_import_place on the shard's stream, after the previous step's commit)
struct sdb_import_totals {
  unsigned long long need, lists, total_recs, explicit_end;
  uint32_t n_total, n_other, maxpad, pad;
};
// mailbox of the low-latency dequeue server (mapped pinned host memory; request and completion words on separate lines)
struct sdb_ls_mailbox {
  uint32_t req_seq, agent, max_messages, flags, quit, pad0[27];
  uint32_t done_seq, pad1[31];
};
static_assert(sizeof(sdb_ls_mailbox) == 256, "latency mailbox must be 256 bytes");

// cross-rank flags of an export buffer (last 128 bytes of the buffer, never touched by an export's copies)
struct sdb_wire_ctrl {
  uint32_t ready;                   // last step whose export into this buffer is complete (written by the owner)
  uint32_t done;                    // last step for which the OWNER, as an importer, finished reading every rank's buffer of this parity
  uint32_t pad[30];
};
static_assert(sizeof(sdb_wire_ctrl) == 128, "wire ctrl block must be 128 bytes");

// arguments of one cross-shard import (sdb_xshard.cu)
#define SDB_MAX_SRC 16
// per-source prefix table built once per import by k_wire_table (so the per-send kernels never
// touch the - possibly remote - wire headers)
struct sdb_src_tab {
  uint32_t first[SDB_MAX_SRC + 1];   // global index of each source's first send
  uint64_t rec_base[SDB_MAX_SRC];    // sequence offset of each source inside the global batch
  uint64_t desc_off[SDB_MAX_SRC], list_off[SDB_MAX_SRC], payload_off[SDB_MAX_SRC];
  uint64_t gs_off_off[SDB_MAX_SRC], gs_idx_off[SDB_MAX_SRC];
  uint32_t explicit_seq[SDB_MAX_SRC];   // rec_base[s] is then an absolute sequence number
};
struct sdb_import_args {
  const sdb_src_tab* tab;
  const uint8_t* meta[SDB_MAX_SRC];   // header + descriptors of each source: a LOCAL copy when the wire batch is remote
  const uint8_t* wire[SDB_MAX_SRC];   // one wire batch per source rank; may point into PEER GPU memory (NVLink)
  uint32_t n_src;
  uint32_t max_sends;         // capacity per wire batch
  const uint32_t* lstart;     // [max_groups] local member list of each group
  const uint32_t* lcount;
  uint32_t max_groups;
  // outputs / scratch
  uint32_t* w;                // [n_src * max_sends] granules written locally per send (scan input)
  uint32_t* gs_cnt;           // [(max_groups + 1) * n_src + 1] bucket sizes per (group, source), then their scan
  sdb_send_desc* descs;       // [n_src * max_sends] localized descriptors
  const uint32_t* w_local;    // scan of w
  const uint32_t* w_tops;
  const uint32_t* gs_off;     // [max_groups + 1] scan of the histogram
  uint32_t* gs_idx;           // [n_src * max_sends]
  // point-to-point and broadcast sends: recipients this shard owns, compacted into a temporary list
  const uint8_t* shard_of;    // [max_agents]
  uint32_t shard_id;
  uint32_t max_agents;
  uint32_t* lw;               // [n_src * max_sends] owned recipients of each non-group send (scan input)
  const uint32_t* lw_local;   // scan of lw
  const uint32_t* lw_tops;
  uint32_t* tmp_list;         // [list_cap]
  uint32_t list_cap;
};

// arguments of the asynchronous import's fused kernel (sdb_xshard.cu: k_import_fused)
struct sdb_import2_args {
  const uint8_t* wire[SDB_MAX_SRC];   // one wire batch per source rank; may point into PEER GPU memory (NVLink)
  uint32_t n_src, max_sends, max_groups, shard_id, max_agents;
  const uint32_t* lcount; const uint32_t* lstart;
  const uint8_t* shard_of;
  sdb_send_desc* descs;               // out [n_src * max_sends]
  uint32_t* gs_off_src;               // out [n_src][max_groups + 1]
  uint32_t* gs_idx_src;               // out [n_src][max_sends]
  uint32_t* first;                    // out [SDB_MAX_SRC + 1]
  uint32_t* tmp_list; uint32_t list_cap;
  unsigned long long* lb;             // [tiles + 2]: look-back status words, tile ticket (zeroed before the launch)
  sdb_cursor* cur; sdb_batch_base* bb;
  unsigned long long arena_grans;
  const sdb_wire_header* hdrs;        // [n_src] local copies of the wire headers (made by k_wire_wait)
  uint32_t* commit_count;             // reset here for the commit sort that follows the fan-out
  sdb_import_totals* totals;          // prefetch mode (non-null): the grand totals go here and k_import_place places the
                                      // import later, on the shard's stream (the cursor is not touched by this kernel)
  uint32_t shared;                    // group sends take the shared-payload layout: lc headers + one payload per send
};

// ---- optional per-kernel timing with CUDA events on the launching stream (bench / roofline) ----
struct sdb_profiler {
  int enabled;
  int n, cap;
  int* kind;
  cudaEvent_t* ev_a;
  cudaEvent_t* ev_b;
};
static inline int sdb_prof_begin(sdb_profiler* p, int kind, cudaStream_t s) {
  if (!p || !p->enabled || p->n >= p->cap) return -1;
  const int i = p->n++;
  p->kind[i] = kind;
  cudaEventRecord(p->ev_a[i], s);
  return i;
}
static inline void sdb_prof_end(sdb_profiler* p, int i, cudaStream_t s) {
  if (i >= 0) cudaEventRecord(p->ev_b[i], s);
}

// ---- two-level exclusive scan (sdb_scan_u32): the prefix of element i is local[i] + tops[i / SDB_SCAN_TILE] ----
#define SDB_SCAN_TILE 4096u   // elements per scan block (1024 threads x 4)
// words of a `tops` array for a scan of up to n elements
static inline size_t sdb_scan_tops_len(size_t n) { return n / SDB_SCAN_TILE + 2; }

// blocks for `items` work items at per_block each, between 1 and max_blocks (kernels grid-stride beyond)
static inline uint32_t sdb_grid(uint64_t items, uint64_t per_block, uint64_t max_blocks) {
  uint64_t g = (items + per_block - 1) / per_block;
  if (g > max_blocks) g = max_blocks;
  return static_cast<uint32_t>(g ? g : 1);
}
// radix-sort key width: bits needed for keys 0 .. max_key, at least 1
static inline uint32_t sdb_key_bits(uint64_t max_key) {
  uint32_t b = 1;
  while (b < 32 && (max_key >> b)) ++b;
  return b;
}

#ifdef __CUDACC__

__device__ __forceinline__ uint8_t* sdb_arena_ptr(const sdb_dev_view& v, uint64_t apos) {
  return v.arena + ((apos & v.gmask) << 5);
}

__device__ __forceinline__ uint32_t sdb_scan_at(const uint32_t* local, const uint32_t* tops, uint32_t i) {
  return local[i] + tops[i / SDB_SCAN_TILE];
}
// inclusive scan of x over each aligned group of W lanes (every lane of the warp calls it); lane: the caller's lane in
// its group
template <uint32_t W = 32>
__device__ __forceinline__ uint32_t sdb_warp_incl_scan(uint32_t x, uint32_t lane) {
#pragma unroll
  for (uint32_t o = 1; o < W; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o, W);
    if (lane >= o) x += y;
  }
  return x;
}
// exclusive scan of one SDB_SCAN_TILE tile held 4 elements per thread by a 1024-thread block (x: zero past the end).
// Returns the tile-local prefix of this thread's x[0]; one thread writes the tile total to *tile_total.
__device__ __forceinline__ uint32_t sdb_block_scan_tile(const uint32_t (&x)[4], uint32_t* tile_total) {
  __shared__ uint32_t s_warp[32];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t tsum = x[0] + x[1] + x[2] + x[3];
  const uint32_t incl = sdb_warp_incl_scan(tsum, lane);
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    const uint32_t w = s_warp[lane], wi = sdb_warp_incl_scan(w, lane);
    s_warp[lane] = wi - w;              // exclusive warp offsets
    if (lane == 31) *tile_total = wi;
  }
  __syncthreads();
  return s_warp[warp] + incl - tsum;
}

// Claim the next slot of agent a's ring and publish (handle, meta) into it.
// Returns false when the ring is full (nothing is written; the commit kernel clamps tail).
// A record whose receiver's ring is full: it exists in the arena but no ring entry refers to it.  The (agent, handle)
// pair is logged so that the host can tell WHICH messages were lost (sdb_overflow_log), not only how many.
__device__ __forceinline__ void sdb_note_overflow(const sdb_dev_view& v, uint32_t a, uint32_t handle) {
  const unsigned long long k = atomicAdd(&v.ctr->ovf_logged, 1ull);
  if (k < SDB_OVF_LOG) v.ovf_log[k] = make_uint2(a, handle);
}
__device__ __forceinline__ bool sdb_ring_append(const sdb_dev_view& v, uint32_t a, uint32_t handle, uint16_t meta) {
  unsigned long long old = atomicAdd(reinterpret_cast<unsigned long long*>(v.ring_hdr + a), 1ull << 32);
  uint32_t e = static_cast<uint32_t>(old >> 32);
  uint32_t head = static_cast<uint32_t>(old);
  if (e - head >= v.ring_slots) { sdb_note_overflow(v, a, handle); return false; }
  size_t slot = (static_cast<size_t>(a) << v.ring_shift) + (e & (v.ring_slots - 1));
  v.ring[slot] = make_uint2(handle, meta);
  return true;
}
__device__ __forceinline__ uint2* sdb_ring_of(const sdb_dev_view& v, uint32_t a) {
  return v.ring + (static_cast<size_t>(a) << v.ring_shift);
}
__device__ __forceinline__ uint32_t sdb_meta(const uint2& e) { return e.y & 0xFFFFu; }
// Shared payloads.  A record is a 32-byte header at `handle` and its payload at handle + 1 + dm1 granules.  dm1 = 0 is
// the classic image (payload right behind its header); group sends above the pull threshold write the members' headers
// back to back and ONE payload behind them (header j of m: dm1 = m - 1 - j), which every member's ring entry points at.
// dm1 travels in the upper half of a ring entry's .y (the lower half is the meta word) and of a plan entry's .z (the
// lower half is the payload size in granules).  The payload sits ABOVE all its headers, so the arena floor - the
// smallest pending handle - never passes a payload that is still referenced.
__device__ __forceinline__ uint32_t sdb_entry_dm1(uint32_t y) { return y >> 16; }
__device__ __forceinline__ uint32_t sdb_plan_z(uint32_t y) { return ((y & SDB_META_GLEN_MASK) - 1u) | (y & 0xFFFF0000u); }   // ring .y -> plan .z
__device__ __forceinline__ const uint8_t* sdb_payload_of(const sdb_dev_view& v, uint32_t handle, uint32_t dm1) {
  return v.arena + (((static_cast<uint64_t>(handle) + 1u + dm1) & v.gmask) << 5);
}

__device__ __forceinline__ uint4 sdb_header_lo(uint64_t seq, double ts) {
  uint4 r;
  r.x = static_cast<uint32_t>(seq);
  r.y = static_cast<uint32_t>(seq >> 32);
  unsigned long long t = __double_as_longlong(ts);
  r.z = static_cast<uint32_t>(t);
  r.w = static_cast<uint32_t>(t >> 32);
  return r;
}
__device__ __forceinline__ uint4 sdb_header_hi(uint32_t sender, uint32_t receiver, uint32_t group,
                                               uint16_t len, uint8_t prio, uint8_t type) {
  uint4 r;
  r.x = sender;
  r.y = receiver;
  r.z = group;
  r.w = static_cast<uint32_t>(len) | (static_cast<uint32_t>(prio) << 16) | (static_cast<uint32_t>(type) << 24);
  return r;
}

// streaming 16-byte accesses: message bytes are touched once, keep them out of L1
__device__ __forceinline__ uint4 sdb_ld_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void sdb_st_stream(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// L2 eviction-priority policies: message bytes stream through once (evict_first) so that the
// small, hot ring metadata (evict_last) stays L2-resident between enqueue and dequeue
__device__ __forceinline__ uint64_t sdb_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t sdb_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint4 sdb_ld_stream_pol(const void* p, uint64_t pol) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ void sdb_st_stream_pol(void* p, const uint4& v, uint64_t pol) {
  asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol) : "memory");
}

// ---- W consecutive 32-byte headers held one per lane, stored as whole sectors -------------------------------------
// Lane l of a group of W lanes (W = 8 or 32, groups aligned in the warp) holds header l of a run as (lo, hi).  Stored
// as held, each 16-byte store instruction writes half of W sectors, and the L2 gets every sector as two partial writes
// from two instructions (scripts/ubench/stores.cu, header stream mode a).  Here the halves change lanes first: in store
// s (0, 1) lane l writes half (l & 1) of header s * W/2 + l/2, so lanes 2k and 2k + 1 fill one sector in ONE
// instruction and the group writes W * 16 contiguous bytes per store.  Two shuffle rounds: lanes below W/2 offer lo in
// the first round and hi in the second, the others the reverse; lane l reads lane l/2 + (l odd ? W/2 : 0) in the first
// round and that lane ^ W/2 in the second, which gives an even lane the lo halves of headers l/2 and W/2 + l/2 and an
// odd lane their hi halves.  A header whose lane passes `valid` false is not written (neither half); all W lanes of
// the group must call this together.
struct sdb_hdr_sectors { uint4 x0, x1; bool w0, w1; };    // store 0 / 1 of this lane: value, and whether it is written
// c ? a : b per component (a select of whole uint4 lvalues can make the compiler address them in local memory)
__device__ __forceinline__ uint4 sdb_sel4(bool c, uint4 a, uint4 b) {
  return make_uint4(c ? a.x : b.x, c ? a.y : b.y, c ? a.z : b.z, c ? a.w : b.w);
}
template <int W>
__device__ __forceinline__ sdb_hdr_sectors sdb_pair_headers(uint4 lo, uint4 hi, bool valid, uint32_t lane) {
  static_assert(W == 8 || W == 16 || W == 32, "header groups are 8 to 32 lanes");
  constexpr uint32_t H = W / 2;
  const uint32_t l = lane & (W - 1u), seg = lane & ~(W - 1u);
  const uint32_t mask = W == 32 ? 0xFFFFFFFFu : ((1u << W) - 1u) << seg;
  const uint32_t vm = __ballot_sync(mask, valid) >> seg;
  const bool odd = l & 1u, low = l < H;
  const uint32_t src = (l >> 1) + (odd ? H : 0u);
  const uint4 p = sdb_sel4(low, lo, hi), q = sdb_sel4(low, hi, lo);
  uint4 y0, y1;
  y0.x = __shfl_sync(mask, p.x, src, W); y0.y = __shfl_sync(mask, p.y, src, W);
  y0.z = __shfl_sync(mask, p.z, src, W); y0.w = __shfl_sync(mask, p.w, src, W);
  y1.x = __shfl_sync(mask, q.x, src ^ H, W); y1.y = __shfl_sync(mask, q.y, src ^ H, W);
  y1.z = __shfl_sync(mask, q.z, src ^ H, W); y1.w = __shfl_sync(mask, q.w, src ^ H, W);
  sdb_hdr_sectors r;
  r.x0 = sdb_sel4(odd, y1, y0); r.x1 = sdb_sel4(odd, y0, y1);
  r.w0 = (vm >> (l >> 1)) & 1u; r.w1 = (vm >> (H + (l >> 1))) & 1u;
  return r;
}
// dst: the group's first header (32-byte aligned)
template <int W>
__device__ __forceinline__ void sdb_st_headers(void* dst, uint4 lo, uint4 hi, bool valid, uint32_t lane) {
  const sdb_hdr_sectors s = sdb_pair_headers<W>(lo, hi, valid, lane);
  uint4* d = reinterpret_cast<uint4*>(dst) + (lane & (W - 1u));
  if (s.w0) sdb_st_stream(d, s.x0);
  if (s.w1) sdb_st_stream(d + W, s.x1);
}
template <int W>
__device__ __forceinline__ void sdb_st_headers_pol(void* dst, uint4 lo, uint4 hi, bool valid, uint32_t lane, uint64_t pol) {
  const sdb_hdr_sectors s = sdb_pair_headers<W>(lo, hi, valid, lane);
  uint4* d = reinterpret_cast<uint4*>(dst) + (lane & (W - 1u));
  if (s.w0) sdb_st_stream_pol(d, s.x0, pol);
  if (s.w1) sdb_st_stream_pol(d + W, s.x1, pol);
}

__device__ __forceinline__ void sdb_st_u32_pol(uint32_t* p, uint32_t v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.u32 [%0], %1, %2;" :: "l"(p), "r"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void sdb_st_u16_pol(uint16_t* p, uint16_t v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.u16 [%0], %1, %2;" :: "l"(p), "h"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void sdb_st_u64_pol(uint64_t* p, uint64_t v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.u64 [%0], %1, %2;" :: "l"(p), "l"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ uint32_t sdb_ld_u32_pol(const uint32_t* p, uint64_t pol) {
  uint32_t r;
  asm volatile("ld.global.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(r) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ uint16_t sdb_ld_u16_pol(const uint16_t* p, uint64_t pol) {
  uint16_t r;
  asm volatile("ld.global.L2::cache_hint.u16 %0, [%1], %2;" : "=h"(r) : "l"(p), "l"(pol));
  return r;
}
__device__ __forceinline__ uint64_t sdb_ld_u64_pol(const uint64_t* p, uint64_t pol) {
  uint64_t r;
  asm volatile("ld.global.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(r) : "l"(p), "l"(pol));
  return r;
}

// ---- mbarrier + TMA (bulk async copy) wrappers ----------------------------------------------
__device__ __forceinline__ uint32_t sdb_smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void sdb_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(sdb_smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void sdb_fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void sdb_fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void sdb_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(sdb_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sdb_mbar_wait_bounded(uint64_t* bar, uint32_t phase) {
  // bounded spin: a phase-accounting bug must surface as a launch failure (trap), never as a hung GPU.  The bound is
  // wall time (30 s on %globaltimer, polled every 4096 spins), not a spin count: under compute-sanitizer or with a
  // payload arriving from a busy peer GPU a legitimate wait can take many more iterations than on an idle device.
  const uint32_t addr = sdb_smem_u32(bar);
  unsigned long long t0 = 0;
  for (uint32_t spins = 0;; ++spins) {
    uint32_t done;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(done) : "r"(addr), "r"(phase) : "memory");
    if (done) return;
    if ((spins & 4095u) == 4095u) {
      unsigned long long t1;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      if (t0 == 0) t0 = t1;
      else if (t1 - t0 > 30ull * 1000000000ull) __trap();
    }
  }
}
// every mbarrier wait in this library is the bounded one: a phase-accounting bug must trap, never hang the GPU
__device__ __forceinline__ void sdb_mbar_wait(uint64_t* bar, uint32_t phase) { sdb_mbar_wait_bounded(bar, phase); }
// global -> shared bulk copy, completion counted on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void sdb_tma_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(sdb_smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(sdb_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void sdb_tma_load_pol(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               :: "r"(sdb_smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(sdb_smem_u32(bar)), "l"(pol) : "memory");
}
// shared -> global bulk copy (bulk_group completion)
__device__ __forceinline__ void sdb_tma_store(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
               :: "l"(gdst), "r"(sdb_smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sdb_tma_store_pol(void* gdst, const void* smem_src, uint32_t bytes, uint64_t pol) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;"
               :: "l"(gdst), "r"(sdb_smem_u32(smem_src)), "r"(bytes), "l"(pol) : "memory");
}
__device__ __forceinline__ void sdb_tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void sdb_tma_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void sdb_tma_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" :: "n"(N) : "memory");
}

// ---- hierarchical decoupled look-back over pairs (a, b) of 31-bit-saturating sums ------------------------------------
// Single-pass kernels (k_recv_plan, k_import_fused) need, per tile, the exclusive prefix of a pair over all earlier
// tiles.  A flat look-back chain advances 32 tiles per L2 round trip, which for thousands of small tiles IS the
// kernel's duration; wider windows drown the L2 in polling.  Two levels instead:
//   * every tile publishes its aggregate at once (no dependency) and bumps its super-tile's counter (32 tiles each);
//   * the tile that completes a super-tile (its "finalizer") sums the 32 aggregates, publishes the super-tile
//     aggregate, looks back over SUPER-TILE words only (tiles / 32 of them: a handful of hops), and publishes the
//     super-tile's exclusive prefix;
//   * a tile's prefix = its super-tile's exclusive prefix + the aggregates of the earlier tiles of its super-tile.
// Words: [63:62] status, [61:31] a, [30:0] b (saturating: a saturated prefix lies beyond every capacity check).
// Layout of the scratch array `lb` (zeroed before the launch), T tiles, S = ceil(T / 32) super-tiles:
//   [0, T) tile aggregates | [T, T+S) super-tile status | [T+S, T+2S) super-tile exclusive prefix | [T+2S, T+3S) counters
//   | [T+3S] tile ticket | [T+3S+1] kernel-specific
// Tiles must be numbered by an atomic ticket (a tile's predecessors are then running or done).  Call with warp 0.
__device__ __forceinline__ unsigned long long sdb_lb_pack(uint32_t st, unsigned long long a, unsigned long long b) {
  const unsigned long long SAT = 0x7FFFFFFFull;
  return (static_cast<unsigned long long>(st) << 62) | ((a < SAT ? a : SAT) << 31) | (b < SAT ? b : SAT);
}
__device__ __forceinline__ unsigned long long sdb_lb_ld(const unsigned long long* p) {
  unsigned long long x;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(x) : "l"(p) : "memory");
  return x;
}
__device__ __forceinline__ void sdb_lb_st(unsigned long long* p, unsigned long long x) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" :: "l"(p), "l"(x) : "memory");
}
__host__ __device__ static inline size_t sdb_lb_words(uint32_t tiles) { return static_cast<size_t>(tiles) + 3 * ((tiles + 31) / 32) + 2; }

// ta/tb: this tile's aggregate.  Returns the exclusive prefix in ea/eb (every lane).  *is_last tells the caller's lane 0
// whether this tile saw the grand total (ga/gb) - exactly one tile does.
__device__ __forceinline__ void sdb_lb_prefix(unsigned long long* lb, uint32_t tile, uint32_t tiles, unsigned long long ta,
                                              unsigned long long tb, uint32_t lane, unsigned long long& ea, unsigned long long& eb,
                                              bool& is_last, unsigned long long& ga, unsigned long long& gb) {
  const unsigned long long SAT = 0x7FFFFFFFull;
  const uint32_t S = (tiles + 31) / 32;
  unsigned long long* agg = lb;
  unsigned long long* sst = lb + tiles;
  unsigned long long* sex = lb + tiles + S;
  unsigned int* scnt = reinterpret_cast<unsigned int*>(lb + tiles + 2 * static_cast<size_t>(S));   // one 64-bit slot per counter
  const uint32_t st = tile >> 5, ti = tile & 31u;
  const uint32_t first = st << 5;
  const uint32_t msize = min(32u, tiles - first);
  is_last = false; ga = 0; gb = 0;
  uint32_t finalizer = 0;
  if (lane == 0) {
    sdb_lb_st(agg + tile, sdb_lb_pack(1u, ta, tb));
    __threadfence();
    finalizer = atomicAdd(scnt + 2 * st, 1u) == msize - 1 ? 1u : 0u;
  }
  finalizer = __shfl_sync(0xFFFFFFFFu, finalizer, 0);
  if (finalizer) {
    __threadfence();
    // every member has published: sum the super-tile
    const unsigned long long w = lane < msize ? sdb_lb_ld(agg + first + lane) : 0ull;
    unsigned long long sa = (w >> 31) & SAT, sb = w & SAT;
    for (int o = 16; o; o >>= 1) { sa += __shfl_xor_sync(0xFFFFFFFFu, sa, o); sb += __shfl_xor_sync(0xFFFFFFFFu, sb, o); }
    unsigned long long xa = 0, xb = 0;
    if (st == 0) {
      if (lane == 0) sdb_lb_st(sst, sdb_lb_pack(2u, sa, sb));
    } else {
      if (lane == 0) sdb_lb_st(sst + st, sdb_lb_pack(1u, sa, sb));
      int32_t idx = static_cast<int32_t>(st) - 1 - static_cast<int32_t>(lane);
      for (;;) {
        unsigned long long w2; uint32_t dm, upto;
        for (;;) {
          w2 = idx >= 0 ? sdb_lb_ld(sst + idx) : sdb_lb_pack(2u, 0, 0);
          const uint32_t s2 = static_cast<uint32_t>(w2 >> 62);
          dm = __ballot_sync(0xFFFFFFFFu, s2 == 2u);
          const uint32_t zm = __ballot_sync(0xFFFFFFFFu, s2 == 0u);
          upto = dm ? static_cast<uint32_t>(__ffs(dm)) : 32u;
          const uint32_t need = upto >= 32u ? 0xFFFFFFFFu : ((1u << upto) - 1u);
          if ((zm & need) == 0) break;
          __nanosleep(40);
        }
        unsigned long long va = lane < upto ? ((w2 >> 31) & SAT) : 0ull, vb = lane < upto ? (w2 & SAT) : 0ull;
        for (int o = 16; o; o >>= 1) { va += __shfl_xor_sync(0xFFFFFFFFu, va, o); vb += __shfl_xor_sync(0xFFFFFFFFu, vb, o); }
        xa += va; xb += vb;
        if (dm) break;
        idx -= 32;
      }
      __threadfence();
      if (lane == 0) sdb_lb_st(sst + st, sdb_lb_pack(2u, xa + sa, xb + sb));
    }
    if (lane == 0) sdb_lb_st(sex + st, sdb_lb_pack(1u, xa, xb));
    if (st == S - 1) { is_last = true; ga = xa + sa; gb = xb + sb; }
  }
  // every tile: super-tile prefix + earlier tiles of the super-tile
  unsigned long long pw = 0;
  for (;;) {
    const unsigned long long w = lane < ti ? sdb_lb_ld(agg + first + lane) : sdb_lb_pack(1u, 0, 0);
    if (lane == 0) pw = sdb_lb_ld(sex + st);
    const bool missing = (w >> 62) == 0 || (lane == 0 && (pw >> 62) == 0);
    if (!__any_sync(0xFFFFFFFFu, missing)) {
      unsigned long long va = (w >> 31) & SAT, vb = w & SAT;
      if (lane == 0) { va += (pw >> 31) & SAT; vb += pw & SAT; }
      for (int o = 16; o; o >>= 1) { va += __shfl_xor_sync(0xFFFFFFFFu, va, o); vb += __shfl_xor_sync(0xFFFFFFFFu, vb, o); }
      ea = va; eb = vb;
      break;
    }
    __nanosleep(40);
  }
  __threadfence();
}

#endif  // __CUDACC__

// ---- launchers and helpers that one source defines and another calls ----
extern "C" {
cudaError_t sdb_launch_p2p(const sdb_dev_view*, const sdb_send_desc*, uint32_t, const uint8_t*, uint64_t, uint64_t, int, cudaStream_t, sdb_profiler*, uint32_t);
cudaError_t sdb_launch_ovf_resolve(const sdb_dev_view*, uint32_t, unsigned long long*, cudaStream_t);
cudaError_t sdb_launch_list_index(const sdb_dev_view*, const sdb_send_desc*, const uint32_t*, const uint32_t*, uint32_t, uint32_t, uint64_t,
                                  cudaStream_t, sdb_profiler*);
cudaError_t sdb_launch_commit_ranked(const sdb_dev_view*, const sdb_send_desc*, uint32_t, uint32_t, cudaStream_t, sdb_profiler*);
cudaError_t sdb_send_prepare_device();
cudaError_t sdb_launch_fanout(const sdb_dev_view*, const sdb_send_desc*, uint32_t, const uint8_t*, const uint32_t*,
                              uint64_t, uint64_t, uint32_t, int, int, cudaStream_t, sdb_profiler*, const sdb_batch_base*, uint32_t);
cudaError_t sdb_launch_fanout_shared(const sdb_dev_view*, const sdb_send_desc*, uint32_t, const uint8_t*, uint64_t, uint64_t, uint32_t, int,
                                     cudaStream_t, sdb_profiler*, const sdb_batch_base*);
cudaError_t sdb_launch_commit(const sdb_dev_view*, uint32_t, uint32_t, uint32_t*, uint32_t*, int, cudaStream_t, sdb_profiler*,
                              const sdb_batch_base*);
cudaError_t sdb_launch_pull(const sdb_dev_view*, const sdb_pull_view*, const sdb_send_desc*, uint32_t, uint32_t, const uint8_t*,
                            uint32_t, uint32_t, const uint32_t*, const uint32_t*, uint64_t, int, cudaStream_t, sdb_profiler*, int*,
                            const sdb_batch_base*, uint32_t);
cudaError_t sdb_launch_receive(const sdb_dev_view*, const sdb_recv_args*, cudaStream_t, int*, sdb_profiler*, int, uint32_t,
                               const sdb_compact_args*, const uint2*, unsigned long long);
cudaError_t sdb_launch_token_take(const sdb_dev_view*, const sdb_recv_args*, unsigned long long, unsigned long long*, cudaStream_t,
                                  int*, sdb_profiler*, int);
cudaError_t sdb_launch_expire(const sdb_dev_view*, const sdb_recv_args*, double, uint32_t, const uint2*, const sdb_compact_args*,
                              cudaStream_t, int*, sdb_profiler*, int);
cudaError_t sdb_launch_supersede(const sdb_dev_view*, const sdb_recv_args*, const sdb_ss_args*, const sdb_compact_args*, cudaStream_t,
                                 int*, sdb_profiler*, int);
cudaError_t sdb_launch_where(const sdb_dev_view*, const sdb_recv_args*, const sdb_where_args*, int, uint32_t, cudaStream_t, int*,
                             sdb_profiler*, int, const sdb_compact_args*, unsigned long long, unsigned long long);
cudaError_t sdb_launch_id_table(const unsigned long long*, uint32_t, sdb_id_slot*, uint32_t, cudaStream_t, int*);
cudaError_t sdb_launch_id_out(const unsigned long long*, uint32_t, const sdb_id_slot*, uint32_t, uint32_t*, cudaStream_t, int*);
cudaError_t sdb_recv_prepare_device();
cudaError_t sdb_balance_prepare_device();
cudaError_t sdb_launch_receive_small(const sdb_dev_view*, const uint32_t*, uint32_t, uint32_t, uint32_t, uint32_t, uint4*,
                                     uint8_t*, cudaStream_t, sdb_profiler*);
cudaError_t sdb_launch_digest(const sdb_recv_args*, uint32_t, unsigned long long*, int, cudaStream_t);
cudaError_t sdb_launch_arena_floor(const sdb_dev_view*, uint32_t, uint32_t, unsigned long long*, cudaStream_t);
cudaError_t sdb_launch_latency_server(const sdb_dev_view*, sdb_ls_mailbox*, uint8_t*, uint32_t, uint4*, cudaStream_t);
const void* sdb_send_kernel_anchor();
const void* sdb_recv_kernel_anchor();
const void* sdb_balance_kernel_anchor();
const void* sdb_xshard_kernel_anchor();
cudaError_t sdb_launch_pick(int mode, uint32_t n_backends, const uint32_t* weight_dev, unsigned long long* load_dev,
                            uint32_t n_req, const uint32_t* cost_dev, uint64_t seed, uint32_t* out_dev,
                            unsigned long long* scratch_dev, const uint32_t* log_tab_dev,
                            cudaStream_t stream, int* n_launches);
void sdb_build_log2_table(uint32_t* tab257);
cudaError_t sdb_launch_agent_loads(const sdb_dev_view*, const uint32_t*, uint32_t, sdb_agent_load*, int, cudaStream_t);
cudaError_t sdb_launch_queue_stats(const sdb_dev_view*, uint32_t, unsigned long long*, cudaStream_t);
cudaError_t sdb_launch_backend_loads_from_queues(const sdb_dev_view*, uint32_t, const uint32_t*, uint32_t, unsigned long long*, cudaStream_t);
cudaError_t sdb_launch_import_measure(const sdb_import_args*, uint32_t, uint32_t*, uint32_t*, uint32_t*, uint32_t*, uint32_t*,
                                      uint32_t*, uint32_t*, unsigned long long*, cudaStream_t, sdb_profiler*, int*);
cudaError_t sdb_launch_import_localize(const sdb_import_args*, uint32_t, const uint32_t*, uint32_t*, cudaStream_t, sdb_profiler*, int*);
cudaError_t sdb_launch_wire_wait(const uint32_t* const*, uint32_t, uint32_t, cudaStream_t, const void* const*, sdb_wire_header*);
cudaError_t sdb_launch_wire_set(uint32_t*, uint32_t, cudaStream_t);
cudaError_t sdb_launch_import_fused(const sdb_import2_args*, cudaStream_t, sdb_profiler*, int*);
cudaError_t sdb_launch_import_place(const sdb_import_totals*, sdb_cursor*, sdb_batch_base*, unsigned long long, uint32_t, uint32_t*, cudaStream_t);
cudaError_t sdb_launch_arena_floor_cur(const sdb_dev_view*, uint32_t, sdb_cursor*, cudaStream_t);
cudaError_t sdb_launch_restore_plan(const sdb_dev_view*, const sdb_restore_args*, cudaStream_t, sdb_profiler*, int*, int);
cudaError_t sdb_launch_restore_write(const sdb_dev_view*, const sdb_restore_args*, unsigned long long, uint32_t, cudaStream_t,
                                     sdb_profiler*, int*, int);
const void* sdb_restore_kernel_anchor();
cudaError_t sdb_launch_lease_append(const sdb_lease_buf*, const sdb_lease_scratch*, const sdb_compact_args*, const uint32_t*,
                                    const unsigned long long*, const uint32_t*, uint32_t, uint32_t, uint32_t, unsigned long long,
                                    unsigned long long, double, uint64_t, uint32_t, cudaStream_t, sdb_profiler*, int*, int);
cudaError_t sdb_launch_lease_settle(const sdb_lease_buf*, const sdb_lease_scratch*, uint32_t, uint32_t, uint32_t, double, cudaStream_t,
                                    sdb_profiler*, int*);
cudaError_t sdb_launch_lease_due(const sdb_lease_buf*, const sdb_lease_scratch*, uint32_t, double, uint32_t, uint32_t, cudaStream_t,
                                 sdb_profiler*, int*);
cudaError_t sdb_launch_lease_select(const sdb_dev_view*, const sdb_lease_buf*, const sdb_lease_scratch*, uint32_t, uint32_t, uint32_t,
                                    uint32_t*, uint32_t*, uint32_t*, cudaStream_t, sdb_profiler*, int*);
cudaError_t sdb_launch_lease_stage(const sdb_lease_buf*, const sdb_lease_scratch*, uint32_t, uint32_t, unsigned long long,
                                   const sdb_compact_args*, cudaStream_t, sdb_profiler*, int*, int);
cudaError_t sdb_launch_lease_compact(const sdb_lease_buf*, const sdb_lease_buf*, const sdb_lease_scratch*, uint32_t, uint32_t, uint32_t,
                                     uint32_t, double, uint32_t, cudaStream_t, sdb_profiler*, int*, int);
cudaError_t sdb_launch_ledger_collect(const sdb_dev_view*, const sdb_ledger*, uint32_t, cudaStream_t, sdb_profiler*, int*);
cudaError_t sdb_launch_ledger_insert(const sdb_dev_view*, const sdb_lease_buf*, const sdb_lease_scratch*, const sdb_ledger*,
                                     const uint32_t*, const uint32_t*, const uint32_t*, uint32_t, uint32_t, cudaStream_t, sdb_profiler*,
                                     int*, int);
cudaError_t sdb_launch_ledger_take(const sdb_lease_buf*, const sdb_ledger*, const sdb_compact_args*, const unsigned long long*, uint32_t,
                                   uint64_t, cudaStream_t, sdb_profiler*, int*, int);
cudaError_t sdb_launch_lease_deliveries(const sdb_lease_buf*, const sdb_lease_scratch*, uint32_t, uint32_t, cudaStream_t, sdb_profiler*,
                                        int*);
cudaError_t sdb_launch_lease_dl_select(const sdb_lease_buf*, const sdb_lease_scratch*, const sdb_dl_scratch*, uint32_t, const uint32_t*,
                                       uint32_t, cudaStream_t, sdb_profiler*, int*);
cudaError_t sdb_launch_lease_dl_emit(const sdb_lease_buf*, const sdb_lease_scratch*, const sdb_dl_scratch*, uint32_t, uint32_t, uint32_t,
                                     uint32_t, uint32_t, const sdb_compact_args*, uint32_t**, cudaStream_t, sdb_profiler*, int*, int);
cudaError_t sdb_launch_lease_x_select(const sdb_lease_buf*, const sdb_lease_scratch*, uint32_t, unsigned long long, cudaStream_t,
                                      sdb_profiler*, int*);
cudaError_t sdb_launch_lease_x_emit(const sdb_lease_buf*, const sdb_lease_scratch*, uint32_t, uint32_t, uint32_t, const sdb_compact_args*,
                                    sdb_lease_meta*, cudaStream_t, sdb_profiler*, int*, int);
cudaError_t sdb_launch_lease_import_check(const sdb_lease_scratch*, const sdb_compact_args*, const sdb_lease_meta*, uint32_t, uint32_t,
                                          unsigned long long, uint32_t, uint32_t, uint32_t, cudaStream_t, sdb_profiler*, int*, int);
cudaError_t sdb_launch_lease_import_write(const sdb_lease_buf*, const sdb_compact_args*, const sdb_lease_meta*, const unsigned long long*,
                                          uint32_t, uint64_t, uint32_t, uint32_t, unsigned long long, unsigned long long, cudaStream_t,
                                          sdb_profiler*, int*, int);
cudaError_t sdb_launch_ledger_import(const sdb_dev_view*, const sdb_ledger*, uint32_t, uint32_t, unsigned long long*, cudaStream_t,
                                     sdb_profiler*, int*, int);
const void* sdb_lease_kernel_anchor();
cudaError_t sdb_launch_reloc_plan(const sdb_dev_view*, const sdb_reloc_args*, cudaStream_t, sdb_profiler*, int*, int);
cudaError_t sdb_launch_reloc_write(const sdb_dev_view*, const sdb_reloc_args*, const sdb_ledger*, uint32_t, cudaStream_t, sdb_profiler*,
                                   int*, int);
const void* sdb_relocate_kernel_anchor();
cudaError_t sdb_scan_u32(const uint32_t* in, uint32_t* local, uint32_t* tops, uint32_t n, unsigned long long* total_out, uint32_t* out,
                         cudaStream_t stream, int* n_launches);
cudaError_t sdb_radix_sort_u32(uint32_t* ka, uint32_t* va, uint32_t* kb, uint32_t* vb, uint32_t n, uint32_t bits, uint32_t* hist,
                               uint32_t* h_local, uint32_t* h_tops, uint32_t** kres, uint32_t** vres, cudaStream_t stream,
                               int* n_launches);
cudaError_t sdb_launch_dedup_probe(const sdb_dedup_args*, uint32_t, uint32_t, double, int, cudaStream_t, sdb_profiler*, int*);
cudaError_t sdb_launch_dedup_insert(const sdb_dedup_args*, uint32_t, double, cudaStream_t, sdb_profiler*);
cudaError_t sdb_launch_dedup_forget(const sdb_dedup_args*, uint32_t, double, uint8_t*, cudaStream_t, sdb_profiler*);
cudaError_t sdb_launch_dedup_rebuild(const sdb_dedup_args*, sdb_dedup_entry*, double, cudaStream_t, sdb_profiler*);
}
