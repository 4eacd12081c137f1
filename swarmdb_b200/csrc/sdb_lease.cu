// sdb_lease.cu - the lease store of leased receives (sdb_receive_leased, sdb_lease_settle, sdb_lease_sweep), sm_90a.
//
// The store holds a copy of every record a leased receive handed out, in the compact receive format: per entry its
// sdb_recv_entry (send = store row), agent, lease id, deadline and state; rows with payload_off into the store's payload.
// Entries stay in lease-id order: appends go to the tail and compaction is stable, so a settle is a binary search.
//
// Append (after the compact receive's back end, same stream)
//   k_lease_append_agents  one warp per listed agent: agent, lease id, deadline, state of its entries (offsets = scan of
//                          the receive's counts)
//   k_lease_append_copy    entries (send rebased), rows (payload_off rebased) and payload granules behind the tail
// Settle
//   k_lease_settle_find    one thread per request: binary search over the ascending ids, verdict = live before the call
//   k_lease_settle_apply   the transition (ack: live -> acked once; renew: new deadline)
// Sweep (the host synchronises between the phases to size the next one)
//   due      k_lease_due + scan: live and due entries
//   select   k_lease_chunk (first C due entries in lease-id order, keyed by agent), stable radix sort by agent
//            (sdb_radix_sort_u32, restore's kernels), k_lease_run_heads + scan + k_lease_run_begin (agent runs),
//            k_lease_ring_check (blocked agents keep their records), scans, k_lease_stage_list (store entries in agent
//            order + the restore's per-agent tables)
//   stage    stable radix sort of the staged entries by seq, k_lease_row_first / k_lease_row_heads + scans (rows numbered
//            by their smallest staged seq), k_lease_stage_rows (rows + payloads into the compact scratch),
//            k_lease_stage_entries
//   (the host then runs restore's plan and write phases on the staged input)
//   compact  k_lease_mark (staged -> redelivered), k_lease_keep + scans, k_lease_keep_rows + scans, k_lease_copy_entries,
//            k_lease_copy_rows into the other buffer
// Snapshots (read out without changing anything, put back behind the tail)
//   export   k_lease_x_flag + scan (held entries with id >= start), k_lease_x_list, the stage's row kernels over store
//            order, k_lease_x_emit (entries + sdb_lease_meta)
//   import   k_lease_import_check (the host synchronises on its verdict), k_lease_import_meta + k_lease_append_copy
//   ledger   k_ledger_import: one warp per (agent, seq, count) triple finds its record in the agent's ring window
#include "sdb_common.cuh"

__device__ __forceinline__ uint32_t ls_pg(uint32_t len) { return ((len + 31u) & ~31u) >> 5; }
// row i as two 16-byte words: {timestamp, payload_off}, {sender, group, len | prio << 16 | type << 24, reserved}
__device__ __forceinline__ void ls_row(const sdb_recv_send* rows, uint32_t i, uint4& lo, uint4& hi) {
  const uint4* p = reinterpret_cast<const uint4*>(rows + i);
  lo = p[0]; hi = p[1];
}
__device__ __forceinline__ void ls_put_row(sdb_recv_send* rows, uint32_t i, uint4 lo, const uint4& hi, unsigned long long off) {
  uint4* p = reinterpret_cast<uint4*>(rows + i);
  lo.z = static_cast<uint32_t>(off); lo.w = static_cast<uint32_t>(off >> 32);
  p[0] = lo; p[1] = hi;
}
// the warp copies the row's padded payload, 16 bytes per lane and step
__device__ __forceinline__ void ls_copy_payload(const uint8_t* base, const uint4& lo, const uint4& hi, uint8_t* dst, uint32_t lane) {
  const uint4* src = reinterpret_cast<const uint4*>(base + ((static_cast<unsigned long long>(lo.w) << 32) | lo.z));
  uint4* d = reinterpret_cast<uint4*>(dst);
  const uint32_t n = 2u * ls_pg(hi.z & 0xFFFFu);
  for (uint32_t c = lane; c < n; c += 32) d[c] = src[c];
}

// ---- append -----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_lease_append_agents(sdb_lease_buf b, const uint32_t* __restrict__ count, const uint32_t* __restrict__ local,
                      const uint32_t* __restrict__ tops, const uint32_t* __restrict__ agents, uint32_t n, uint32_t used,
                      unsigned long long id_base, double deadline) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t q = gw; q < n; q += nw) {
    const uint32_t c = count[q];
    if (!c) continue;
    const uint32_t off = sdb_scan_at(local, tops, q), a = agents ? agents[q] : q;
    for (uint32_t j = lane; j < c; j += 32) {
      const uint32_t e = used + off + j;
      b.agent[e] = a; b.id[e] = id_base + off + j; b.deadline[e] = deadline; b.state[e] = SDB_LS_LIVE;
      if (b.deliveries) b.deliveries[e] = 1u;
    }
  }
}

__global__ void __launch_bounds__(256)
k_lease_append_copy(sdb_lease_buf b, const sdb_recv_entry* __restrict__ ent, const sdb_recv_send* __restrict__ snd,
                    const uint8_t* __restrict__ pay, const unsigned long long* __restrict__ rx_totals,
                    const unsigned long long* __restrict__ cx_totals, uint32_t used, uint32_t rows_used,
                    unsigned long long pay_used) {
  const uint64_t n = rx_totals[0], nr = cx_totals[0], nc = cx_totals[1] * 2;     // 16-byte chunks of payload
  const uint64_t m = n > nr ? (n > nc ? n : nc) : (nr > nc ? nr : nc);
  for (uint64_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    if (i < n) { sdb_recv_entry e = ent[i]; e.send += rows_used; b.ent[used + i] = e; }
    if (i < nr) { sdb_recv_send s = snd[i]; s.payload_off += pay_used; b.rows[rows_used + i] = s; }
    if (i < nc) reinterpret_cast<uint4*>(b.payload + pay_used)[i] = reinterpret_cast<const uint4*>(pay)[i];
  }
}

// ---- settle -----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_lease_settle_find(sdb_lease_buf b, uint32_t used, sdb_lease_scratch s, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool live = false;
  if (i < n) {
    const unsigned long long x = s.req[i];
    uint32_t lo = 0, hi = used;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (b.id[mid] < x) lo = mid + 1; else hi = mid;
    }
    live = lo < used && b.id[lo] == x && b.state[lo] == SDB_LS_LIVE;
    s.at[i] = live ? lo : 0xFFFFFFFFu;
    s.settled[i] = live ? 1 : 0;
  }
  const uint32_t c = __popc(__ballot_sync(0xFFFFFFFFu, live));
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(s.tot + 0, static_cast<unsigned long long>(c));
}

__global__ void __launch_bounds__(256)
k_lease_settle_apply(sdb_lease_buf b, sdb_lease_scratch s, uint32_t n, uint32_t op, double deadline) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool moved = false;
  if (i < n) {
    const uint32_t e = s.at[i];
    if (e != 0xFFFFFFFFu) {
      if (op == 0u) moved = atomicCAS(b.state + e, SDB_LS_LIVE, SDB_LS_ACKED) == SDB_LS_LIVE;
      else b.deadline[e] = deadline;
    }
  }
  const uint32_t c = __popc(__ballot_sync(0xFFFFFFFFu, moved));
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(s.tot + 1, static_cast<unsigned long long>(c));
}

// ---- sweep: due ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_lease_due(sdb_lease_buf b, uint32_t used, double now, uint32_t all, uint32_t max_deliveries, uint32_t* __restrict__ flag) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= used) return;
  bool due = b.state[e] == SDB_LS_LIVE && (all || b.deadline[e] <= now);         // NaN on either side: not due
  if (max_deliveries && due) due = b.deliveries[e] < max_deliveries;              // at the limit: dead-lettered instead
  flag[e] = due ? 1u : 0u;
}

// ---- sweep: select ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_lease_chunk(sdb_lease_buf b, uint32_t used, sdb_lease_scratch s, uint32_t C) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= used || !s.flag[e]) return;
  const uint32_t p = sdb_scan_at(s.f_local, s.f_tops, e);
  if (p >= C) return;
  s.chunk[p] = e; s.key_a[p] = b.agent[e]; s.val_a[p] = p;
}

__global__ void __launch_bounds__(256)
k_lease_run_heads(const uint32_t* __restrict__ key, uint32_t n, uint32_t* __restrict__ head) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) head[i] = (i == 0 || key[i] != key[i - 1]) ? 1u : 0u;
}

__global__ void __launch_bounds__(256)
k_lease_run_begin(sdb_lease_scratch s, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (s.gran[i]) s.run_begin[sdb_scan_at(s.g_local, s.g_tops, i)] = i;
  if (i == 0) s.run_begin[s.tot[1]] = n;
}

// one thread per run: an agent whose ring cannot take all of its records keeps them in the store
__global__ void __launch_bounds__(256)
k_lease_ring_check(sdb_dev_view v, sdb_lease_scratch s, const uint32_t* __restrict__ key, uint32_t n) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t runs = static_cast<uint32_t>(s.tot[1]);
  bool blocked = false;
  if (r < runs) {
    const uint32_t i0 = s.run_begin[r], c = s.run_begin[r + 1] - i0;
    const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + key[i0]);   // {head, tail, ..}
    blocked = static_cast<uint64_t>(h.y - h.x) + c > v.ring_slots;
    s.kcnt[r] = blocked ? 0u : c;
    s.kflag[r] = blocked ? 0u : 1u;
  } else if (r < n) {
    s.kcnt[r] = 0u; s.kflag[r] = 0u;                      // the scans run over n slots
  }
  const uint32_t k = __popc(__ballot_sync(0xFFFFFFFFu, blocked));
  if ((threadIdx.x & 31) == 0 && k) atomicAdd(s.tot + 4, static_cast<unsigned long long>(k));
}

// chunk position i (agent order): its store entry goes to the staged list; a kept run's head fills the restore's tables
__global__ void __launch_bounds__(256)
k_lease_stage_list(sdb_lease_scratch s, const uint32_t* __restrict__ key, const uint32_t* __restrict__ val, uint32_t n,
                   uint32_t* __restrict__ rs_agent, uint32_t* __restrict__ rs_count, uint32_t* __restrict__ rs_first) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t head = s.gran[i];
  const uint32_t r = sdb_scan_at(s.g_local, s.g_tops, i) + head - 1u;
  const uint32_t c = s.kcnt[r];
  if (!c) return;
  const uint32_t base = sdb_scan_at(s.k_local, s.k_tops, r);
  s.staged[base + i - s.run_begin[r]] = s.chunk[val[i]];
  if (head) {
    const uint32_t q = sdb_scan_at(s.kf_local, s.kf_tops, r);
    rs_agent[q] = key[i]; rs_count[q] = c; rs_first[q] = base;
    atomicMax(s.tot + 5, static_cast<unsigned long long>(key[i]) + 1ull);
  }
}

// ---- sweep: stage -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_lease_seq_keys(sdb_lease_buf b, sdb_lease_scratch s, uint32_t n) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  s.key_a[k] = static_cast<uint32_t>(b.ent[s.staged[k]].seq);
  s.val_a[k] = k;
}
// the high words of the seqs in the order of the first pass (sequence numbers of 2^32 and above)
__global__ void __launch_bounds__(256)
k_lease_seq_hi(sdb_lease_buf b, sdb_lease_scratch s, const uint32_t* __restrict__ val, uint32_t* __restrict__ key, uint32_t n) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) key[p] = static_cast<uint32_t>(b.ent[s.staged[val[p]]].seq >> 32);
}

__global__ void __launch_bounds__(256)
k_lease_row_first(sdb_lease_buf b, sdb_lease_scratch s, const uint32_t* __restrict__ sv, uint32_t n) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) atomicMin(s.rfirst + b.ent[s.staged[sv[p]]].send, p);
}

// seq-sorted position p heads its row when it is the row's first: rows are numbered in order of their smallest seq
__global__ void __launch_bounds__(256)
k_lease_row_heads(sdb_lease_buf b, sdb_lease_scratch s, const uint32_t* __restrict__ sv, uint32_t n) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint32_t row = b.ent[s.staged[sv[p]]].send;
  const bool h = s.rfirst[row] == p;
  s.flag[p] = h ? 1u : 0u;
  s.gran[p] = h ? ls_pg(b.rows[row].len) : 0u;
}

// one warp per seq-sorted position: a head writes its row and payload into the compact scratch
__global__ void __launch_bounds__(256)
k_lease_stage_rows(sdb_lease_buf b, sdb_lease_scratch s, const uint32_t* __restrict__ sv, uint32_t n,
                   sdb_recv_send* __restrict__ send_out, uint8_t* __restrict__ payload_out) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t p = gw; p < n; p += nw) {
    if (!s.flag[p]) continue;
    const uint32_t row = b.ent[s.staged[sv[p]]].send;
    const uint32_t nr = sdb_scan_at(s.f_local, s.f_tops, p);
    const unsigned long long off = static_cast<unsigned long long>(sdb_scan_at(s.g_local, s.g_tops, p)) << 5;
    uint4 lo, hi;
    ls_row(b.rows, row, lo, hi);
    ls_copy_payload(b.payload, lo, hi, payload_out + off, lane);
    if (lane == 0) {
      s.rmap[row] = nr;
      ls_put_row(send_out, nr, lo, hi, off);
    }
  }
}

__global__ void __launch_bounds__(256)
k_lease_stage_entries(sdb_lease_buf b, sdb_lease_scratch s, uint32_t n, sdb_recv_entry* __restrict__ entry_out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  sdb_recv_entry e = b.ent[s.staged[k]];
  e.send = s.rmap[e.send];
  entry_out[k] = e;
}

// ---- sweep: compact -----------------------------------------------------------------------------------------------
// the redelivery limit: live due entries (the sweep's rule) with deliveries >= max_deliveries become dead letters.  Runs
// after the redelivery succeeded, so a failed sweep leaves every state as it was.
__global__ void __launch_bounds__(256)
k_lease_kill(sdb_lease_buf b, uint32_t used, double now, uint32_t all, uint32_t max_deliveries, unsigned long long* __restrict__ tot) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  bool dead = false;
  if (e < used && b.state[e] == SDB_LS_LIVE && (all || b.deadline[e] <= now) && b.deliveries[e] >= max_deliveries) {
    b.state[e] = SDB_LS_DEAD;
    dead = true;
  }
  const uint32_t c = __popc(__ballot_sync(0xFFFFFFFFu, dead));
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(tot, static_cast<unsigned long long>(c));
}

__global__ void __launch_bounds__(256)
k_lease_mark(sdb_lease_buf b, sdb_lease_scratch s, uint32_t n) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) b.state[s.staged[k]] = SDB_LS_REDELIVERED;
}

// kept entries (live and dead) and the rows they name
__global__ void __launch_bounds__(256)
k_lease_keep(sdb_lease_buf b, sdb_lease_scratch s, uint32_t used) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= used) return;
  const uint32_t st = b.state[e];
  const bool keep = st == SDB_LS_LIVE || st == SDB_LS_DEAD;
  s.flag[e] = keep ? 1u : 0u;
  if (keep) s.gran[b.ent[e].send] = 1u;
}

__global__ void __launch_bounds__(256)
k_lease_keep_rows(sdb_lease_buf b, sdb_lease_scratch s, uint32_t rows) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows) s.rg[r] = s.gran[r] ? ls_pg(b.rows[r].len) : 0u;
}

__global__ void __launch_bounds__(256)
k_lease_copy_entries(sdb_lease_buf in, sdb_lease_buf out, sdb_lease_scratch s, uint32_t used) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= used || !s.flag[e]) return;
  const uint32_t k = sdb_scan_at(s.f_local, s.f_tops, e);
  sdb_recv_entry en = in.ent[e];
  en.send = sdb_scan_at(s.g_local, s.g_tops, en.send);
  out.ent[k] = en; out.agent[k] = in.agent[e]; out.id[k] = in.id[e]; out.deadline[k] = in.deadline[e];
  out.state[k] = in.state[e];
  if (in.deliveries) out.deliveries[k] = in.deliveries[e];
}

// one warp per row: a kept row and its payload
__global__ void __launch_bounds__(256)
k_lease_copy_rows(sdb_lease_buf in, sdb_lease_buf out, sdb_lease_scratch s, uint32_t rows) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t r = gw; r < rows; r += nw) {
    if (!s.gran[r]) continue;
    const uint32_t k = sdb_scan_at(s.g_local, s.g_tops, r);
    const unsigned long long off = static_cast<unsigned long long>(sdb_scan_at(s.rg_local, s.rg_tops, r)) << 5;
    uint4 lo, hi;
    ls_row(in.rows, r, lo, hi);
    ls_copy_payload(in.payload, lo, hi, out.payload + off, lane);
    if (lane == 0) ls_put_row(out.rows, k, lo, hi, off);
  }
}

// ---- launchers ----------------------------------------------------------------------------------------------------
#define LS_LAUNCH(n_items, kern, ...)                                                        \
  do {                                                                                       \
    if ((n_items) > 0) { kern<<<((n_items) + 255) / 256, 256, 0, stream>>>(__VA_ARGS__); ++nl; } \
  } while (0)

// after a compact receive: its entries, rows and payloads (device totals) go to the store's tail
extern "C" cudaError_t sdb_launch_lease_append(const sdb_lease_buf* b, const sdb_lease_scratch* s, const sdb_compact_args* cx,
                                               const uint32_t* count, const unsigned long long* rx_totals, const uint32_t* agents,
                                               uint32_t n_agents, uint32_t used, uint32_t rows_used, unsigned long long pay_used,
                                               unsigned long long id_base, double deadline, uint64_t rec_cap, uint32_t max_pad,
                                               cudaStream_t stream, sdb_profiler* prof, int* n_launches, int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  cudaError_t e = sdb_scan_u32(count, s->a_local, s->a_tops, n_agents, nullptr, nullptr, stream, &nl);
  k_lease_append_agents<<<sdb_grid(n_agents, 8, 32 * sm_count), 256, 0, stream>>>(*b, count, s->a_local, s->a_tops, agents, n_agents,
                                                                                  used, id_base, deadline);
  const uint64_t items = rec_cap * (max_pad / 16u > 1u ? max_pad / 16u : 1u);
  k_lease_append_copy<<<sdb_grid(items, 256, 32 * sm_count), 256, 0, stream>>>(*b, cx->entry_out, cx->send_out, cx->payload_out,
                                                                               rx_totals, cx->totals, used, rows_used, pay_used);
  nl += 2;
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// s->req[0, n) holds the ids; verdicts to s->settled, s->tot[0] = live requests, s->tot[1] = transitions
extern "C" cudaError_t sdb_launch_lease_settle(const sdb_lease_buf* b, const sdb_lease_scratch* s, uint32_t used, uint32_t n,
                                               uint32_t op, double deadline, cudaStream_t stream, sdb_profiler* prof,
                                               int* n_launches) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  cudaMemsetAsync(s->tot, 0, 2 * sizeof(unsigned long long), stream);
  LS_LAUNCH(n, k_lease_settle_find, *b, used, *s, n);
  LS_LAUNCH(n, k_lease_settle_apply, *b, *s, n, op, deadline);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return cudaGetLastError();
}

// tot[0] = due entries (with a redelivery limit: those below it)
extern "C" cudaError_t sdb_launch_lease_due(const sdb_lease_buf* b, const sdb_lease_scratch* s, uint32_t used, double now,
                                            uint32_t all, uint32_t max_deliveries, cudaStream_t stream, sdb_profiler* prof,
                                            int* n_launches) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  cudaMemsetAsync(s->tot, 0, 16 * sizeof(unsigned long long), stream);
  LS_LAUNCH(used, k_lease_due, *b, used, now, all, max_deliveries, s->flag);
  cudaError_t e = sdb_scan_u32(s->flag, s->f_local, s->f_tops, used, s->tot + 0, nullptr, stream, &nl);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// the first n due entries, sorted by agent, blocked agents dropped; writes s->staged and the restore's per-agent tables.
// tot[1] = agent runs, tot[2] = staged entries, tot[3] = kept runs, tot[4] = blocked agents, tot[5] = largest agent + 1
extern "C" cudaError_t sdb_launch_lease_select(const sdb_dev_view* v, const sdb_lease_buf* b, const sdb_lease_scratch* s,
                                               uint32_t used, uint32_t n, uint32_t max_agents, uint32_t* rs_agent,
                                               uint32_t* rs_count, uint32_t* rs_first, cudaStream_t stream, sdb_profiler* prof,
                                               int* n_launches) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  LS_LAUNCH(used, k_lease_chunk, *b, used, *s, n);
  uint32_t *ks = nullptr, *vs = nullptr;
  cudaError_t e = sdb_radix_sort_u32(s->key_a, s->val_a, s->key_b, s->val_b, n, sdb_key_bits(max_agents - 1u), s->hist, s->h_local,
                                     s->h_tops, &ks, &vs, stream, &nl);
  LS_LAUNCH(n, k_lease_run_heads, ks, n, s->gran);
  if (e == cudaSuccess) e = sdb_scan_u32(s->gran, s->g_local, s->g_tops, n, s->tot + 1, nullptr, stream, &nl);
  LS_LAUNCH(n, k_lease_run_begin, *s, n);
  LS_LAUNCH(n, k_lease_ring_check, *v, *s, ks, n);          // runs <= n: the slots past the run count read 0
  if (e == cudaSuccess) e = sdb_scan_u32(s->kcnt, s->k_local, s->k_tops, n, s->tot + 2, nullptr, stream, &nl);
  if (e == cudaSuccess) e = sdb_scan_u32(s->kflag, s->kf_local, s->kf_tops, n, s->tot + 3, nullptr, stream, &nl);
  LS_LAUNCH(n, k_lease_stage_list, *s, ks, vs, n, rs_agent, rs_count, rs_first);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// the n staged entries into the compact scratch: rows numbered by smallest seq.  tot[6] = rows, tot[7] = payload granules
extern "C" cudaError_t sdb_launch_lease_stage(const sdb_lease_buf* b, const sdb_lease_scratch* s, uint32_t rows_used, uint32_t n,
                                              unsigned long long seq_end, const sdb_compact_args* cx, cudaStream_t stream,
                                              sdb_profiler* prof, int* n_launches, int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  LS_LAUNCH(n, k_lease_seq_keys, *b, *s, n);
  const unsigned long long top = seq_end ? seq_end - 1ull : 0ull;
  uint32_t *ks = nullptr, *vs = nullptr;
  cudaError_t e = sdb_radix_sort_u32(s->key_a, s->val_a, s->key_b, s->val_b, n, top >> 32 ? 32u : sdb_key_bits(top), s->hist,
                                     s->h_local, s->h_tops, &ks, &vs, stream, &nl);
  if (e == cudaSuccess && (top >> 32)) {
    uint32_t* kh = ks == s->key_a ? s->key_b : s->key_a;
    uint32_t* vh = vs == s->val_a ? s->val_b : s->val_a;
    LS_LAUNCH(n, k_lease_seq_hi, *b, *s, vs, ks, n);          // the used keys are rewritten in place
    e = sdb_radix_sort_u32(ks, vs, kh, vh, n, sdb_key_bits(top >> 32), s->hist, s->h_local, s->h_tops, &ks, &vs, stream, &nl);
  }
  if (rows_used) cudaMemsetAsync(s->rfirst, 0xFF, static_cast<size_t>(rows_used) * sizeof(uint32_t), stream);
  LS_LAUNCH(n, k_lease_row_first, *b, *s, vs, n);
  LS_LAUNCH(n, k_lease_row_heads, *b, *s, vs, n);
  if (e == cudaSuccess) e = sdb_scan_u32(s->flag, s->f_local, s->f_tops, n, s->tot + 6, nullptr, stream, &nl);
  if (e == cudaSuccess) e = sdb_scan_u32(s->gran, s->g_local, s->g_tops, n, s->tot + 7, nullptr, stream, &nl);
  if (n) {
    k_lease_stage_rows<<<sdb_grid(n, 8, 32 * sm_count), 256, 0, stream>>>(*b, *s, vs, n, cx->send_out, cx->payload_out);
    ++nl;
  }
  LS_LAUNCH(n, k_lease_stage_entries, *b, *s, n, cx->entry_out);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// marks the n staged entries redelivered and, with a redelivery limit, the due live entries at it dead; then copies the
// live and dead entries and the rows they name into `out`.
// tot[8] = kept entries, tot[9] = kept rows, tot[10] = their payload granules, tot[11] = entries marked dead
extern "C" cudaError_t sdb_launch_lease_compact(const sdb_lease_buf* in, const sdb_lease_buf* out, const sdb_lease_scratch* s,
                                                uint32_t used, uint32_t rows_used, uint32_t n_staged, uint32_t max_deliveries,
                                                double now, uint32_t all, cudaStream_t stream, sdb_profiler* prof,
                                                int* n_launches, int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  cudaMemsetAsync(s->tot + 8, 0, (max_deliveries ? 4 : 3) * sizeof(unsigned long long), stream);
  LS_LAUNCH(n_staged, k_lease_mark, *in, *s, n_staged);
  if (max_deliveries) LS_LAUNCH(used, k_lease_kill, *in, used, now, all, max_deliveries, s->tot + 11);
  if (rows_used) cudaMemsetAsync(s->gran, 0, static_cast<size_t>(rows_used) * sizeof(uint32_t), stream);
  LS_LAUNCH(used, k_lease_keep, *in, *s, used);
  LS_LAUNCH(rows_used, k_lease_keep_rows, *in, *s, rows_used);
  cudaError_t e = sdb_scan_u32(s->flag, s->f_local, s->f_tops, used, s->tot + 8, nullptr, stream, &nl);
  if (e == cudaSuccess) e = sdb_scan_u32(s->gran, s->g_local, s->g_tops, rows_used, s->tot + 9, nullptr, stream, &nl);
  if (e == cudaSuccess) e = sdb_scan_u32(s->rg, s->rg_local, s->rg_tops, rows_used, s->tot + 10, nullptr, stream, &nl);
  LS_LAUNCH(used, k_lease_copy_entries, *in, *out, *s, used);
  if (rows_used) {
    k_lease_copy_rows<<<sdb_grid(rows_used, 8, 32 * sm_count), 256, 0, stream>>>(*in, *out, *s, rows_used);
    ++nl;
  }
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// ---- redelivery ledger (sdb_lease_set_policy) -------------------------------------------------------------------
// restated in tests/deadletter_ref.py::lg_slot, which tests/test_gpu_lease_edges.py uses to make probe chains wrap
__device__ __forceinline__ uint32_t lg_slot(uint32_t a, unsigned long long seq, uint32_t slots) {
  unsigned long long x = seq ^ (static_cast<unsigned long long>(a) * 0x9E3779B97F4A7C15ull);
  x ^= x >> 33; x *= 0xFF51AFD7ED558CCDull; x ^= x >> 33; x *= 0xC4CEB9FE1A85EC53ull; x ^= x >> 33;
  return static_cast<uint32_t>(__umul64hi(x, slots));
}
__device__ __forceinline__ void lg_index(const sdb_ledger& L, uint32_t k, uint32_t a, unsigned long long seq) {
  for (uint32_t i = lg_slot(a, seq, L.slots);; i = i + 1 == L.slots ? 0u : i + 1)
    if (atomicCAS(L.index + i, 0xFFFFFFFFu, k) == 0xFFFFFFFFu) return;
}

// Collection: an entry stays while its record is still the one the sweep put back: p inside the window [head, tail),
// the ring entry at p not consumed and still naming the same arena handle (handles are unique while a record is
// pending).  Kept entries go to L.alt in any order; tot[0] counts them.
__global__ void __launch_bounds__(256)
k_ledger_collect(sdb_dev_view v, sdb_ledger L, uint32_t n) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  bool keep = false;
  sdb_ledger_ent en{};
  if (e < n) {
    en = L.ent[e];
    if (en.count) {
      const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + en.agent);
      if (en.p - h.x < h.y - h.x) {
        const uint2 r = sdb_ring_of(v, en.agent)[en.p & (v.ring_slots - 1)];
        keep = sdb_meta(r) != SDB_META_TOMB && r.x == en.handle;
      }
    }
  }
  const uint32_t m = __ballot_sync(0xFFFFFFFFu, keep);
  uint32_t base = 0;
  if ((threadIdx.x & 31) == 0 && m) base = static_cast<uint32_t>(atomicAdd(L.tot, static_cast<unsigned long long>(__popc(m))));
  base = __shfl_sync(0xFFFFFFFFu, base, 0);
  if (keep) L.alt[base + __popc(m & ((1u << (threadIdx.x & 31)) - 1u))] = en;
}

// the index over the kept entries (L.ent is the collected buffer by now)
__global__ void __launch_bounds__(256)
k_ledger_reindex(sdb_ledger L, uint32_t n_bound) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_bound || k >= L.tot[0]) return;
  const sdb_ledger_ent en = L.ent[k];
  lg_index(L, k, en.agent, en.seq);
}

// after a sweep's restore: one warp per redelivered agent run.  Record j of a run of c sits at tail - c + j (restore
// appends in entry order); its entry takes number n0 + (staged position).
__global__ void __launch_bounds__(256)
k_ledger_insert(sdb_dev_view v, sdb_lease_buf b, sdb_lease_scratch s, sdb_ledger L, const uint32_t* __restrict__ rs_agent,
                const uint32_t* __restrict__ rs_count, const uint32_t* __restrict__ rs_first, uint32_t runs, uint32_t n0) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t q = gw; q < runs; q += nw) {
    const uint32_t a = rs_agent[q], c = rs_count[q], f = rs_first[q];
    const uint32_t tail = v.ring_hdr[a].tail;
    const uint2* ring = sdb_ring_of(v, a);
    for (uint32_t j = lane; j < c; j += 32) {
      const uint32_t e = s.staged[f + j], p = tail - c + j;
      sdb_ledger_ent en;
      en.seq = b.ent[e].seq; en.agent = a; en.count = b.deliveries[e]; en.p = p; en.handle = ring[p & (v.ring_slots - 1)].x;
      L.ent[n0 + f + j] = en;
      lg_index(L, n0 + f + j, a, en.seq);
    }
  }
}

// after a leased receive's append: record i of the call (store entry used + i) inherits count + 1 from its ledger entry,
// which it takes; tot[1] counts the entries taken
__global__ void __launch_bounds__(256)
k_ledger_take(sdb_lease_buf b, sdb_ledger L, const sdb_recv_entry* __restrict__ ent, const unsigned long long* __restrict__ rx_totals,
              uint32_t used) {
  const uint64_t n = rx_totals[0];
  for (uint64_t i0 = static_cast<uint64_t>(blockIdx.x) * blockDim.x; i0 < n; i0 += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    const uint64_t i = i0 + threadIdx.x;
    uint32_t c = 0;
    if (i < n) {
      const uint32_t a = b.agent[used + i];
      const unsigned long long seq = ent[i].seq;
      for (uint32_t t = lg_slot(a, seq, L.slots);; t = t + 1 == L.slots ? 0u : t + 1) {
        const uint32_t k = L.index[t];
        if (k == 0xFFFFFFFFu) break;
        if (L.ent[k].agent == a && L.ent[k].seq == seq && (c = atomicExch(&L.ent[k].count, 0u)) != 0u) break;
      }
      b.deliveries[used + i] = c + 1u;
    }
    const uint32_t m = __popc(__ballot_sync(0xFFFFFFFFu, c != 0u));
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(L.tot + 1, static_cast<unsigned long long>(m));
  }
}

// ---- sdb_lease_deliveries: binary search over the ascending ids; 0 unless the lease is live or dead ---------------
__global__ void __launch_bounds__(256)
k_lease_deliveries(sdb_lease_buf b, uint32_t used, const unsigned long long* __restrict__ req, uint32_t* __restrict__ out, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long x = req[i];
  uint32_t lo = 0, hi = used;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (b.id[mid] < x) lo = mid + 1; else hi = mid;
  }
  const bool held = lo < used && b.id[lo] == x && (b.state[lo] == SDB_LS_LIVE || b.state[lo] == SDB_LS_DEAD);
  out[i] = held ? b.deliveries[lo] : 0u;
}

// ---- sdb_lease_dead_letters --------------------------------------------------------------------------------------
// agent -> position in the caller's list (~0: not listed)
__global__ void __launch_bounds__(256)
k_lease_dl_pos(const uint32_t* __restrict__ agents, uint32_t n, uint32_t* __restrict__ pos, uint32_t clear) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) pos[agents[i]] = clear ? 0xFFFFFFFFu : i;
}
__device__ __forceinline__ uint32_t dl_pos(const uint32_t* pos, uint32_t n_list, uint32_t a) {
  return pos ? pos[a] : (a < n_list ? a : 0xFFFFFFFFu);
}
// dead entries of listed agents, counted per list position
__global__ void __launch_bounds__(256)
k_lease_dl_flag(sdb_lease_buf b, uint32_t used, const uint32_t* __restrict__ pos, uint32_t n_list, uint32_t* __restrict__ flag,
                uint32_t* __restrict__ cnt) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= used) return;
  const uint32_t q = b.state[e] == SDB_LS_DEAD ? dl_pos(pos, n_list, b.agent[e]) : 0xFFFFFFFFu;
  flag[e] = q != 0xFFFFFFFFu ? 1u : 0u;
  if (q != 0xFFFFFFFFu) atomicAdd(cnt + q, 1u);
}
// flagged entry number k (store order = lease-id order): key = list position, value k, staged[k] = store entry
__global__ void __launch_bounds__(256)
k_lease_dl_keys(sdb_lease_buf b, uint32_t used, sdb_lease_scratch s, const uint32_t* __restrict__ pos, uint32_t n_list,
                uint32_t* __restrict__ staged, uint32_t* __restrict__ key, uint32_t* __restrict__ val) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= used || !s.flag[e]) return;
  const uint32_t k = sdb_scan_at(s.f_local, s.f_tops, e);
  key[k] = dl_pos(pos, n_list, b.agent[e]); val[k] = k; staged[k] = e;
}
// sorted position p: its entry (send = output row), its count; a take marks the entry for the compaction to drop
__global__ void __launch_bounds__(256)
k_lease_dl_emit(sdb_lease_buf b, sdb_lease_scratch s, const uint32_t* __restrict__ sv, uint32_t n, uint32_t take,
                sdb_recv_entry* __restrict__ entry_out, uint32_t* __restrict__ deliveries_out) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const uint32_t e = s.staged[sv[p]];
  sdb_recv_entry en = b.ent[e];
  en.send = s.rmap[en.send];
  entry_out[p] = en;
  deliveries_out[p] = b.deliveries[e];
  if (take) b.state[e] = SDB_LS_REDELIVERED;
}

// L->tot[0] = entries kept, L->tot[1] = entries taken since (both reset here); the caller swaps L->ent and L->alt
extern "C" cudaError_t sdb_launch_ledger_collect(const sdb_dev_view* v, const sdb_ledger* L, uint32_t n, cudaStream_t stream,
                                                 sdb_profiler* prof, int* n_launches) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  cudaMemsetAsync(L->tot, 0, 2 * sizeof(unsigned long long), stream);
  cudaMemsetAsync(L->index, 0xFF, static_cast<size_t>(L->slots) * sizeof(uint32_t), stream);
  LS_LAUNCH(n, k_ledger_collect, *v, *L, n);
  sdb_ledger sw = *L;
  sw.ent = L->alt; sw.alt = L->ent;
  LS_LAUNCH(n, k_ledger_reindex, sw, n);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return cudaGetLastError();
}

extern "C" cudaError_t sdb_launch_ledger_insert(const sdb_dev_view* v, const sdb_lease_buf* b, const sdb_lease_scratch* s,
                                                const sdb_ledger* L, const uint32_t* rs_agent, const uint32_t* rs_count,
                                                const uint32_t* rs_first, uint32_t runs, uint32_t n0, cudaStream_t stream,
                                                sdb_profiler* prof, int* n_launches, int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  if (runs) {
    k_ledger_insert<<<sdb_grid(runs, 8, 32 * sm_count), 256, 0, stream>>>(*v, *b, *s, *L, rs_agent, rs_count, rs_first, runs, n0);
    ++nl;
  }
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return cudaGetLastError();
}

extern "C" cudaError_t sdb_launch_ledger_take(const sdb_lease_buf* b, const sdb_ledger* L, const sdb_compact_args* cx,
                                              const unsigned long long* rx_totals, uint32_t used, uint64_t rec_cap,
                                              cudaStream_t stream, sdb_profiler* prof, int* n_launches, int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  k_ledger_take<<<sdb_grid(rec_cap, 256, 32 * sm_count), 256, 0, stream>>>(*b, *L, cx->entry_out, rx_totals, used);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += 1;
  return cudaGetLastError();
}

// the ids in s->req[0, n): counts to s->at
extern "C" cudaError_t sdb_launch_lease_deliveries(const sdb_lease_buf* b, const sdb_lease_scratch* s, uint32_t used, uint32_t n,
                                                   cudaStream_t stream, sdb_profiler* prof, int* n_launches) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  LS_LAUNCH(n, k_lease_deliveries, *b, used, s->req, s->at, n);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return cudaGetLastError();
}

// phase 1: the dead entries of the listed agents (agents == nullptr: every index below n_list), counted per position
// into d->cnt[n_list]; s->tot[0] = their number.  Leaves keys, values and staged entries in store order.
extern "C" cudaError_t sdb_launch_lease_dl_select(const sdb_lease_buf* b, const sdb_lease_scratch* s, const sdb_dl_scratch* d,
                                                  uint32_t used, const uint32_t* agents, uint32_t n_list, cudaStream_t stream,
                                                  sdb_profiler* prof, int* n_launches) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  cudaMemsetAsync(s->tot, 0, 16 * sizeof(unsigned long long), stream);
  cudaMemsetAsync(d->cnt, 0, static_cast<size_t>(n_list) * sizeof(uint32_t), stream);
  const uint32_t* pos = agents ? d->pos : nullptr;
  if (agents) LS_LAUNCH(n_list, k_lease_dl_pos, agents, n_list, d->pos, 0u);
  LS_LAUNCH(used, k_lease_dl_flag, *b, used, pos, n_list, s->flag, d->cnt);
  cudaError_t e = sdb_scan_u32(s->flag, s->f_local, s->f_tops, used, s->tot + 0, nullptr, stream, &nl);
  LS_LAUNCH(used, k_lease_dl_keys, *b, used, *s, pos, n_list, d->staged, d->key_a, d->val_a);
  if (agents) LS_LAUNCH(n_list, k_lease_dl_pos, agents, n_list, d->pos, 1u);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// phase 2: stable sort of the n selected entries by list position (lease-id order within an agent), then the first m of
// them in the compact format: rows numbered by first appearance (the sweep's row kernels over the sorted order), rows
// and payloads to cx, entries to cx->entry_out, counts to *deliveries_dev (a sort buffer the result does not use).  take: the m entries are marked for the
// compaction to drop.  tot[6] = rows, tot[7] = payload granules
extern "C" cudaError_t sdb_launch_lease_dl_emit(const sdb_lease_buf* b, const sdb_lease_scratch* s, const sdb_dl_scratch* d,
                                                uint32_t rows_used, uint32_t n, uint32_t m, uint32_t n_list, uint32_t take,
                                                const sdb_compact_args* cx, uint32_t** deliveries_dev, cudaStream_t stream,
                                                sdb_profiler* prof, int* n_launches, int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  uint32_t *ks = nullptr, *vs = nullptr;
  cudaError_t e = sdb_radix_sort_u32(d->key_a, d->val_a, d->key_b, d->val_b, n, sdb_key_bits(n_list ? n_list - 1u : 0u), d->hist,
                                     d->h_local, d->h_tops, &ks, &vs, stream, &nl);
  uint32_t* dv = ks == d->key_a ? d->key_b : d->key_a;
  *deliveries_dev = dv;
  sdb_lease_scratch t = *s;
  t.staged = d->staged;
  if (rows_used) cudaMemsetAsync(t.rfirst, 0xFF, static_cast<size_t>(rows_used) * sizeof(uint32_t), stream);
  LS_LAUNCH(m, k_lease_row_first, *b, t, vs, m);
  LS_LAUNCH(m, k_lease_row_heads, *b, t, vs, m);
  if (e == cudaSuccess) e = sdb_scan_u32(t.flag, t.f_local, t.f_tops, m, t.tot + 6, nullptr, stream, &nl);
  if (e == cudaSuccess) e = sdb_scan_u32(t.gran, t.g_local, t.g_tops, m, t.tot + 7, nullptr, stream, &nl);
  if (m) {
    k_lease_stage_rows<<<sdb_grid(m, 8, 32 * sm_count), 256, 0, stream>>>(*b, t, vs, m, cx->send_out, cx->payload_out);
    ++nl;
  }
  LS_LAUNCH(m, k_lease_dl_emit, *b, t, vs, m, take, cx->entry_out, dv);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// ---- snapshots: sdb_lease_export / sdb_lease_import / sdb_lease_ledger_import --------------------------------------
static_assert(sizeof(sdb_lease_meta) == 32, "lease meta records are 32 bytes");
// held entries (live or dead) with id >= start_id
__global__ void __launch_bounds__(256)
k_lease_x_flag(sdb_lease_buf b, uint32_t used, unsigned long long start_id, uint32_t* __restrict__ flag) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= used) return;
  const uint32_t st = b.state[e];
  flag[e] = (st == SDB_LS_LIVE || st == SDB_LS_DEAD) && b.id[e] >= start_id ? 1u : 0u;
}
// the first m flagged entries in store (= lease-id) order: staged[p] = store entry, val_a[p] = p (the row kernels' order)
__global__ void __launch_bounds__(256)
k_lease_x_list(sdb_lease_scratch s, uint32_t used, uint32_t m) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= used || !s.flag[e]) return;
  const uint32_t p = sdb_scan_at(s.f_local, s.f_tops, e);
  if (p < m) { s.staged[p] = e; s.val_a[p] = p; }
}
// position p: its entry (send = output row) and its meta; the last position leaves the id to continue from in tot[8]
__global__ void __launch_bounds__(256)
k_lease_x_emit(sdb_lease_buf b, sdb_lease_scratch s, uint32_t m, sdb_recv_entry* __restrict__ entry_out,
               sdb_lease_meta* __restrict__ meta_out) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= m) return;
  const uint32_t e = s.staged[p];
  sdb_recv_entry en = b.ent[e];
  en.send = s.rmap[en.send];
  entry_out[p] = en;
  sdb_lease_meta x;
  x.id = b.id[e]; x.deadline = b.deadline[e]; x.agent = b.agent[e]; x.deliveries = b.deliveries ? b.deliveries[e] : 0u;
  x.state = b.state[e]; x.reserved = 0u;
  meta_out[p] = x;
  if (p == m - 1u) s.tot[8] = x.id + 1ull;
}

// every entry and row of an import before anything is written; a bad one sets tot[0]
__global__ void __launch_bounds__(256)
k_lease_import_check(const sdb_recv_entry* __restrict__ ent, const sdb_lease_meta* __restrict__ meta,
                     const sdb_recv_send* __restrict__ snd, uint32_t n, uint32_t n_sends, unsigned long long payload_bytes,
                     uint32_t max_agents, uint32_t max_payload, uint32_t policy, unsigned long long* __restrict__ tot) {
  const uint32_t m = n > n_sends ? n : n_sends;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    bool bad = false;
    if (i < n) {
      const sdb_recv_entry en = ent[i];
      const sdb_lease_meta x = meta[i];
      bad = en.send >= n_sends || x.agent >= max_agents || (en.receiver != x.agent && en.receiver != SDB_NO_RECEIVER) ||
            !(x.state == SDB_LS_LIVE || (x.state == SDB_LS_DEAD && policy));
    }
    if (i < n_sends) {
      const sdb_recv_send r = snd[i];
      const unsigned long long pad = 32ull * ls_pg(r.len);
      bad = bad || r.len > max_payload || r.prio > 3u || (r.payload_off & 15ull) || r.payload_off > payload_bytes ||
            payload_bytes - r.payload_off < pad;
    }
    if (bad) atomicOr(tot, 1ull);
  }
}
// the import's agent, id, deadline, state and count of each entry (entries, rows and payload: k_lease_append_copy)
__global__ void __launch_bounds__(256)
k_lease_import_meta(sdb_lease_buf b, const sdb_lease_meta* __restrict__ meta, uint32_t n, uint32_t used,
                    unsigned long long id_base) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const sdb_lease_meta x = meta[i];
  const uint32_t e = used + i;
  b.agent[e] = x.agent; b.id[e] = id_base + i; b.deadline[e] = x.deadline; b.state[e] = x.state;
  if (b.deliveries) b.deliveries[e] = x.deliveries ? x.deliveries : 1u;
}

// one warp per triple staged in L.alt[0, n): the oldest pending record of the agent (ring window [head, tail),
// consumed slots skipped) whose header seq matches takes ledger entry n0 + (matches so far); tot counts them
__global__ void __launch_bounds__(256)
k_ledger_import(sdb_dev_view v, sdb_ledger L, uint32_t n, uint32_t n0, unsigned long long* __restrict__ tot) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t q = gw; q < n; q += nw) {
    const sdb_ledger_ent t = L.alt[q];
    const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + t.agent);   // {head, tail, ..}
    const uint2* ring = sdb_ring_of(v, t.agent);
    const uint32_t w = h.y - h.x;
    for (uint32_t o = 0; o < w; o += 32) {
      bool hit = false;
      uint32_t handle = 0;
      if (o + lane < w) {
        const uint2 r = ring[(h.x + o + lane) & (v.ring_slots - 1)];
        handle = r.x;
        hit = sdb_meta(r) != SDB_META_TOMB &&
              *reinterpret_cast<const unsigned long long*>(sdb_arena_ptr(v, r.x)) == t.seq;
      }
      const uint32_t m = __ballot_sync(0xFFFFFFFFu, hit);
      if (!m) continue;
      if (lane == static_cast<uint32_t>(__ffs(m) - 1)) {
        const uint32_t k = n0 + static_cast<uint32_t>(atomicAdd(tot, 1ull));
        sdb_ledger_ent en = t;
        en.p = h.x + o + lane; en.handle = handle;
        L.ent[k] = en;
        lg_index(L, k, t.agent, t.seq);
      }
      break;
    }
  }
}

// phase 1: the held entries with id >= start_id are flagged and counted (tot[0]; leaves the flag scan)
extern "C" cudaError_t sdb_launch_lease_x_select(const sdb_lease_buf* b, const sdb_lease_scratch* s, uint32_t used,
                                                 unsigned long long start_id, cudaStream_t stream, sdb_profiler* prof,
                                                 int* n_launches) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  cudaMemsetAsync(s->tot, 0, 16 * sizeof(unsigned long long), stream);
  LS_LAUNCH(used, k_lease_x_flag, *b, used, start_id, s->flag);
  cudaError_t e = sdb_scan_u32(s->flag, s->f_local, s->f_tops, used, s->tot + 0, nullptr, stream, &nl);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// phase 2: the first m of them in the compact format (rows numbered by first appearance: the sweep's row kernels over
// store order), entries to cx->entry_out, meta to meta_out.  tot[6] = rows, tot[7] = payload granules, tot[8] = next id
extern "C" cudaError_t sdb_launch_lease_x_emit(const sdb_lease_buf* b, const sdb_lease_scratch* s, uint32_t used, uint32_t rows_used,
                                               uint32_t m, const sdb_compact_args* cx, sdb_lease_meta* meta_out,
                                               cudaStream_t stream, sdb_profiler* prof, int* n_launches, int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  LS_LAUNCH(used, k_lease_x_list, *s, used, m);
  if (rows_used) cudaMemsetAsync(s->rfirst, 0xFF, static_cast<size_t>(rows_used) * sizeof(uint32_t), stream);
  LS_LAUNCH(m, k_lease_row_first, *b, *s, s->val_a, m);
  LS_LAUNCH(m, k_lease_row_heads, *b, *s, s->val_a, m);
  cudaError_t e = sdb_scan_u32(s->flag, s->f_local, s->f_tops, m, s->tot + 6, nullptr, stream, &nl);
  if (e == cudaSuccess) e = sdb_scan_u32(s->gran, s->g_local, s->g_tops, m, s->tot + 7, nullptr, stream, &nl);
  if (m) {
    k_lease_stage_rows<<<sdb_grid(m, 8, 32 * sm_count), 256, 0, stream>>>(*b, *s, s->val_a, m, cx->send_out, cx->payload_out);
    ++nl;
  }
  LS_LAUNCH(m, k_lease_x_emit, *b, *s, m, cx->entry_out, meta_out);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// import, phase 1: the input staged in cx (entries, rows, payload) and meta; error bits to s->tot[0]
extern "C" cudaError_t sdb_launch_lease_import_check(const sdb_lease_scratch* s, const sdb_compact_args* cx, const sdb_lease_meta* meta,
                                                     uint32_t n, uint32_t n_sends, unsigned long long payload_bytes,
                                                     uint32_t max_agents, uint32_t max_payload, uint32_t policy,
                                                     cudaStream_t stream, sdb_profiler* prof, int* n_launches, int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  cudaMemsetAsync(s->tot, 0, sizeof(unsigned long long), stream);
  const uint32_t items = n > n_sends ? n : n_sends;
  if (items) {
    k_lease_import_check<<<sdb_grid(items, 256, 32 * sm_count), 256, 0, stream>>>(cx->entry_out, meta, cx->send_out, n, n_sends,
                                                                                 payload_bytes, max_agents, max_payload, policy,
                                                                                 s->tot);
    if (n_launches) *n_launches += 1;
  }
  sdb_prof_end(prof, pi, stream);
  return cudaGetLastError();
}

// import, phase 2: behind the store's tail.  totals = {n} and cx->totals = {n_sends, payload granules} on the device
extern "C" cudaError_t sdb_launch_lease_import_write(const sdb_lease_buf* b, const sdb_compact_args* cx, const sdb_lease_meta* meta,
                                                     const unsigned long long* totals, uint32_t n, uint64_t items, uint32_t used,
                                                     uint32_t rows_used, unsigned long long pay_used, unsigned long long id_base,
                                                     cudaStream_t stream, sdb_profiler* prof, int* n_launches, int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  int nl = 0;
  LS_LAUNCH(n, k_lease_import_meta, *b, meta, n, used, id_base);
  if (items) {
    k_lease_append_copy<<<sdb_grid(items, 256, 32 * sm_count), 256, 0, stream>>>(*b, cx->entry_out, cx->send_out, cx->payload_out,
                                                                                 totals, cx->totals, used, rows_used, pay_used);
    ++nl;
  }
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return cudaGetLastError();
}

// n triples staged in L->alt: matches become entries n0.. of L->ent, *tot counts them (zeroed here)
extern "C" cudaError_t sdb_launch_ledger_import(const sdb_dev_view* v, const sdb_ledger* L, uint32_t n, uint32_t n0,
                                                unsigned long long* tot, cudaStream_t stream, sdb_profiler* prof, int* n_launches,
                                                int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_LEASE, stream);
  cudaMemsetAsync(tot, 0, sizeof(unsigned long long), stream);
  if (n) {
    k_ledger_import<<<sdb_grid(n, 8, 32 * sm_count), 256, 0, stream>>>(*v, *L, n, n0, tot);
    if (n_launches) *n_launches += 1;
  }
  sdb_prof_end(prof, pi, stream);
  return cudaGetLastError();
}

// any kernel of this file: its module is loaded as a whole before the latency server starts (sdb_api.cu)
extern "C" const void* sdb_lease_kernel_anchor() { return reinterpret_cast<const void*>(&k_lease_due); }
