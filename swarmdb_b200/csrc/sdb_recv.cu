// sdb_recv.cu - dequeue kernels (sm_90a): receive_messages (reference M:521-601; the drain
// loop M:553-601 and its filter M:579-585 are replaced by per-agent rings that only ever
// hold records addressed to that agent).
//
// Stream order (the reference's behaviour) takes the SINGLE-PASS path: k_recv_plan + k_recv_gather.
//   k_recv_plan     one thread per requested agent: one 16-byte ring-header load, the agent's entries (8 bytes
//                   each, one sector for the usual handful), then ONE decoupled look-back over 256-agent tiles
//                   carrying {records, payload granules} together gives every record its output index and
//                   payload offset; the per-record plan is written, heads advance.  No separate count / scan /
//                   select / scan kernels and no second read of the ring.
//   k_recv_gather   flat over records: copy header + payload from the arena to the packed output
// Priority order (extension, SURVEY App. A rule 9) keeps the multi-kernel pipeline (all stream-ordered, no host
// round trip inside):
//   k_recv_count    cnt[q]   = min(max_messages, live(agent q))
//   scan            rec_off  = exclusive scan of cnt             (sdb_scan_u32: k_scan_local + k_scan_tops)
//   k_recv_select   per agent: choose WHICH pending entries are delivered, write the per-record
//                   plan (arena handle, payload size) at the record's output index, retire them
//                     stream order      -> the first cnt live entries (contiguous when the
//                                          window holds no consumed entries: nothing to do);
//                     priority order    -> segmented radix-select on the 2-bit priority:
//                                          pass 1 4-bin histogram of the pending window with
//                                          warp ballots/popc, pick the cut level and residual,
//                                          pass 2 stable compaction (ballot prefix ranks) of
//                                          the selected ring positions in (prio desc, arrival);
//   scan            pay_off  = exclusive scan of payload granules over the planned RECORDS
//   k_recv_gather   flat over records: copy header + payload from the arena to the packed output
// A compact receive (sdb_receive_compact) runs either plan and replaces the gather with the compact kernels (below):
// 16-byte entries per record and one row + payload per distinct payload image.
// A byte-budget receive (sdb_receive_budget) runs the single-pass plan in either order (k_recv_plan<SDB_PLAN_BUDGET>,
// <SDB_PLAN_BUDGET_PRIO>), then the gather or the compact kernels.
//
// Roofline: HBM-bound.  Algorithmic bytes per agent-call: P*1 priority bytes scanned (we scan
// 2-byte ring_meta entries) + 2*k*(L+H) gather+emit (SURVEY 8d).
#include <cstdlib>
#include "sdb_common.cuh"

#define SDB_MODE_LIST 0x80000000u


// ------------------------------------------------------------------------------------------
// generic exclusive scan over uint32 (two tiny kernels; consumers add tops[i / TILE])
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
k_scan_local(const uint32_t* __restrict__ in, uint32_t* __restrict__ local, uint32_t* __restrict__ tops, uint32_t n) {
  const uint32_t base = blockIdx.x * SDB_SCAN_TILE + threadIdx.x * 4u;
  uint32_t x[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) x[k] = (base + k < n) ? in[base + k] : 0u;
  uint32_t run = sdb_block_scan_tile(x, tops + blockIdx.x);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (base + k < n) local[base + k] = run;
    run += x[k];
  }
}

__global__ void __launch_bounds__(1024)
k_scan_tops(uint32_t* __restrict__ tops, uint32_t n_tiles, unsigned long long* __restrict__ total_out) {
  // single block; n_tiles is small (n / 4096)
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_carry;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < n_tiles; base += 1024) {
    const uint32_t i = base + tid;
    const uint32_t x = i < n_tiles ? tops[i] : 0u;
    const uint32_t incl = sdb_warp_incl_scan(x, lane);
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      const uint32_t w = s_warp[lane];
      s_warp[lane] = sdb_warp_incl_scan(w, lane) - w;
    }
    __syncthreads();
    const uint32_t carry = s_carry;
    const uint32_t excl = carry + s_warp[warp] + incl - x;
    if (i < n_tiles) tops[i] = excl;
    __syncthreads();
    if (tid == 1023) s_carry = excl + x;
    __syncthreads();
  }
  if (tid == 0 && total_out) *total_out = s_carry;
}

// out[i] = local[i] + tops[i / TILE]: materialise a scan as a plain array
__global__ void __launch_bounds__(256)
k_scan_apply(const uint32_t* __restrict__ local, const uint32_t* __restrict__ tops, uint32_t* __restrict__ out, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = sdb_scan_at(local, tops, i);
}

// exclusive scan of n uint32 (block-local part in `local`, per-block part in `tops`), optional
// grand total and optional materialised output; usable from the other translation units.  Adds its launches to
// *n_launches (when given).
extern "C" cudaError_t sdb_scan_u32(const uint32_t* in, uint32_t* local, uint32_t* tops, uint32_t n,
                                    unsigned long long* total_out, uint32_t* out, cudaStream_t stream, int* n_launches) {
  if (n == 0) return cudaSuccess;
  const uint32_t tiles = (n + SDB_SCAN_TILE - 1) / SDB_SCAN_TILE;
  k_scan_local<<<tiles, 1024, 0, stream>>>(in, local, tops, n);
  k_scan_tops<<<1, 1024, 0, stream>>>(tops, tiles, total_out);
  if (out) k_scan_apply<<<(n + 255) / 256, 256, 0, stream>>>(local, tops, out, n);
  if (n_launches) *n_launches += out ? 3 : 2;
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_recv_count(sdb_dev_view v, sdb_recv_args r) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= r.n) return;
  const uint32_t a = r.agent_idx ? r.agent_idx[q] : q;
  uint32_t c = 0;
  if (a < v.max_agents) {
    const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);      // head, tail, ctail, ntomb
    c = min(h.y - h.x - h.w, r.max_messages);
  }
  r.cnt[q] = c;
}

// ------------------------------------------------------------------------------------------
// select + retire: one warp owns 32 consecutive agents of the request list.  Agents whose
// selection is a short contiguous run are finished by their own lane; the rest are processed
// one at a time by the whole warp (window scans with ballots).  For every selected record the
// plan (arena handle, payload granules) is written at its output index, the ring entry is
// retired (head advanced / tombstoned), and count_out is final.  Agents that would overflow
// the record capacity are left untouched (whole-agent truncation: nothing is ever lost),
// except the first agent in the output (roff == 0), which takes its first rec_cap records.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t lane_prefix(uint32_t ballot, uint32_t lane) {
  return __popc(ballot & ((1u << lane) - 1u));
}

// whole warp: the first live entry of [P, T), or T.  After a retiring selection head goes there, so that head is always
// the oldest pending record and the ring's free slots (R - (tail - head)) never include a tombstone at the window's start.
// Past the selected range only tombstones are walked (at most ntomb of them) before the first live entry.
__device__ __forceinline__ uint32_t first_live_from(const uint2* rs, uint32_t mask, uint32_t P, uint32_t T, uint32_t lane) {
  for (uint32_t q0 = P; static_cast<int32_t>(T - q0) > 0; q0 += 32) {
    const uint32_t p = q0 + lane;
    const bool live = static_cast<int32_t>(T - p) > 0 && (rs[p & mask].y & 0xFFFFu) != SDB_META_TOMB;
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, live);
    if (b) return q0 + (__ffs(b) - 1);
  }
  return T;
}

// one agent, whole warp: choose the C entries to deliver from the window [H, T), write their plan at
// output index RO.., retire them (advance head / tombstone).  Stream order when !prio_mode.  The plan's payload
// offsets (.y) are filled later (record-level scan / fill_offsets_warp).
__device__ __forceinline__ void select_agent_warp(const sdb_dev_view& v, uint4* plan, uint32_t slot,
                                                  bool prio_mode, uint32_t A, uint32_t H, uint32_t T, uint32_t NT,
                                                  uint32_t C, uint32_t RO, uint32_t lane, bool retire) {
  const uint32_t mask = v.ring_slots - 1;
  uint2* rs = sdb_ring_of(v, A);

  if (!prio_mode && NT == 0) {
    // long contiguous run [H, H+C)
    for (uint32_t j = lane; j < C; j += 32) {
      const uint2 e = rs[(H + j) & mask];
      plan[RO + j] = make_uint4(e.x, 0u, sdb_plan_z(e.y), slot);
    }
    if (lane == 0 && retire) v.ring_hdr[A].head = H + C;
    return;
  }
  // ---- pass 1: histogram of live entries per priority level over the window [H, T)
  uint32_t h0 = 0, h1 = 0, h2 = 0, h3 = 0;
  if (prio_mode) {
    // 2 entries (16 bytes) per lane per load, 4 independent loads in flight per lane (256 entries per warp
    // step), aligned pairs of the circular window
    for (uint32_t b2 = (H & ~1u) + (lane << 1); static_cast<int32_t>(T - b2) > 0; b2 += 256) {
      uint4 q[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t p2 = b2 + u * 64;
        q[u] = static_cast<int32_t>(T - p2) > 0 ? *reinterpret_cast<const uint4*>(rs + (p2 & mask)) : make_uint4(0u, ~0u, 0u, ~0u);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t p2 = b2 + u * 64;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const uint32_t p = p2 + k;
          const uint32_t m = (k ? q[u].w : q[u].y) & 0xFFFFu;
          if (static_cast<int32_t>(p - H) >= 0 && static_cast<int32_t>(T - p) > 0 && m != SDB_META_TOMB) {
            const uint32_t L = m >> 14;
            h0 += (L == 0); h1 += (L == 1); h2 += (L == 2); h3 += (L == 3);
          }
        }
      }
    }
    unsigned long long lo = (static_cast<unsigned long long>(h1) << 32) | h0;
    unsigned long long hi = (static_cast<unsigned long long>(h3) << 32) | h2;
    for (int o = 16; o; o >>= 1) {
      lo += __shfl_xor_sync(0xFFFFFFFFu, lo, o);
      hi += __shfl_xor_sync(0xFFFFFFFFu, hi, o);
    }
    h0 = static_cast<uint32_t>(lo); h1 = static_cast<uint32_t>(lo >> 32);
    h2 = static_cast<uint32_t>(hi); h3 = static_cast<uint32_t>(hi >> 32);
  } else {
    h0 = (T - H) - NT;     // single level: every live entry
  }
  // ---- cut: take every entry of the levels above the cut, and the first `quota` of the cut level
  uint32_t hist[4] = {h0, h1, h2, h3};
  uint32_t quota[4] = {0, 0, 0, 0}, basek[4] = {0, 0, 0, 0};
  {
    uint32_t need = C, acc = 0;
    for (int L = 3; L >= 0; --L) {
      const uint32_t take = min(hist[L], need);
      quota[L] = take; basek[L] = acc; acc += take; need -= take;
    }
  }
  // ---- pass 2: stable compaction of the selected positions, window order within a level
  uint32_t taken[4] = {0, 0, 0, 0};
  uint32_t first_unsel = T;      // first live entry left behind
  uint32_t got = 0;
  uint32_t p0 = H;
  for (; static_cast<int32_t>(T - p0) > 0 && got < C; p0 += 32) {
    const uint32_t p = p0 + lane;
    const bool in = static_cast<int32_t>(T - p) > 0;
    const uint2 e = in ? rs[p & mask] : make_uint2(0u, SDB_META_TOMB);
    const uint32_t m = sdb_meta(e);
    const bool live = m != SDB_META_TOMB;
    const uint32_t L = (live && prio_mode) ? (m >> 14) : 0u;
    bool sel = false; uint32_t rank = 0;
#pragma unroll
    for (uint32_t lev = 0; lev < 4; ++lev) {
      const uint32_t b = __ballot_sync(0xFFFFFFFFu, live && L == lev);
      if (live && L == lev) {
        const uint32_t k = taken[lev] + lane_prefix(b, lane);
        if (k < quota[lev]) { sel = true; rank = basek[lev] + k; }
      }
      taken[lev] += __popc(b);
    }
    if (sel) {
      plan[RO + rank] = make_uint4(e.x, 0u, sdb_plan_z(e.y), slot);
      if (retire) rs[p & mask].y = SDB_META_TOMB;
    }
    const uint32_t bs = __ballot_sync(0xFFFFFFFFu, sel);
    got += __popc(bs);
    const uint32_t bu = __ballot_sync(0xFFFFFFFFu, live && !sel);
    if (bu && first_unsel == T) first_unsel = p0 + (__ffs(bu) - 1);
  }
  const uint32_t scan_end = static_cast<int32_t>(T - p0) > 0 ? p0 : T;
  uint32_t nh = first_unsel;
  if (static_cast<int32_t>(nh - scan_end) >= 0 && retire) nh = first_live_from(rs, mask, scan_end, T, lane);
  if (lane == 0 && retire) {
    v.ring_hdr[A].head = nh;
    v.ring_hdr[A].ntomb = NT + got - (nh - H);
  }
}

__global__ void __launch_bounds__(256)
k_recv_select(sdb_dev_view v, sdb_recv_args r) {
  // one lane per requested agent: short contiguous runs are planned and retired here; everything else is
  // queued for k_recv_select_big (one warp per agent)
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = q < r.n;
  const uint32_t R = v.ring_slots, mask = R - 1;

  uint32_t a = 0, head = 0, nt = 0, cnt = 0, roff = 0;
  if (valid) {
    a = r.agent_idx ? r.agent_idx[q] : q;
    cnt = r.cnt[q];
    roff = sdb_scan_at(r.rec_local, r.rec_tops, q);
    if (cnt && static_cast<uint64_t>(roff) + cnt > r.rec_cap) {      // does not fit: stays queued ...
      if (roff == 0) cnt = static_cast<uint32_t>(r.rec_cap);          // ... unless first in the output: its first rec_cap records
      else cnt = 0;
      atomicMin(r.totals, static_cast<unsigned long long>(roff) + cnt);
    }
    r.count_out[q] = cnt;
    r.rec_off[q] = roff;
    if (cnt) {
      const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
      head = h.x; nt = h.w;
    }
  }
  const bool prio_mode = (r.flags & SDB_RECV_PRIORITY) != 0;
  constexpr uint32_t SMALL = 64, CH = 8;
  const bool small = valid && cnt && !prio_mode && nt == 0 && cnt <= SMALL;
  if (small) {
    const uint64_t pol = sdb_policy_evict_last();
    const uint2* rs = sdb_ring_of(v, a);
    for (uint32_t b = 0; b < cnt; b += CH) {
      uint64_t ev[CH];
#pragma unroll
      for (uint32_t j = 0; j < CH; ++j)       // all loads of the chunk first, then the stores
        if (b + j < cnt) ev[j] = sdb_ld_u64_pol(reinterpret_cast<const uint64_t*>(rs + ((head + b + j) & mask)), pol);
#pragma unroll
      for (uint32_t j = 0; j < CH; ++j)
        if (b + j < cnt)
          r.plan[roff + b + j] = make_uint4(static_cast<uint32_t>(ev[j]), 0u, sdb_plan_z(static_cast<uint32_t>(ev[j] >> 32)), q);
    }
    if (!(r.flags & SDB_RECV_PEEK)) v.ring_hdr[a].head = head + cnt;
  }
  // everything else (long runs, holes, priority order) goes to the warp-per-agent kernel
  const bool big = valid && cnt && !small;
  const uint32_t todo = __ballot_sync(0xFFFFFFFFu, big);
  uint32_t n_deliv = (valid && !(r.flags & SDB_RECV_PEEK)) ? cnt : 0;
  if (todo) {
    uint32_t basew = 0;
    if (lane == 0) basew = atomicAdd(r.big_count, static_cast<uint32_t>(__popc(todo)));
    basew = __shfl_sync(0xFFFFFFFFu, basew, 0);
    if (big) r.big_list[basew + lane_prefix(todo, lane)] = q;
  }
  for (int o = 16; o; o >>= 1) n_deliv += __shfl_xor_sync(0xFFFFFFFFu, n_deliv, o);
  if (lane == 0 && n_deliv) atomicAdd(&v.ctr->delivered, static_cast<unsigned long long>(n_deliv));
}

// Single-pass bounded selection (priority order, or stream order with holes) for C <= SDB_CAND:
// walk the window once in arrival order keeping, per level, the first C live positions (stable,
// ballot-prefix ranks) in shared memory; stop as soon as the top level alone fills the quota -
// with mixed priorities that happens after a few hundred entries instead of the whole window.
#define SDB_CAND 128u
__device__ __forceinline__ void select_agent_warp_bounded(const sdb_dev_view& v, uint4* plan, uint32_t slot,
                                                          bool prio_mode, uint32_t A, uint32_t H, uint32_t T, uint32_t NT,
                                                          uint32_t C, uint32_t RO, uint32_t lane, bool retire,
                                                          uint32_t (*cand)[SDB_CAND]) {
  const uint32_t mask = v.ring_slots - 1;
  uint2* rs = sdb_ring_of(v, A);
  const uint32_t top = prio_mode ? 3u : 0u;
  uint32_t cnt[4] = {0, 0, 0, 0};
  uint32_t p0 = H;
  while (static_cast<int32_t>(T - p0) > 0 && cnt[top] < C) {
    // four chunks of 32 entries in flight per step (the loads do not depend on the running counts)
    uint32_t mm[4];
#pragma unroll
    for (uint32_t u = 0; u < 4; ++u) {
      const uint32_t p = p0 + u * 32u + lane;
      mm[u] = static_cast<int32_t>(T - p) > 0 ? (rs[p & mask].y & 0xFFFFu) : SDB_META_TOMB;
    }
#pragma unroll
    for (uint32_t u = 0; u < 4; ++u) {
      if (static_cast<int32_t>(T - p0) <= 0 || cnt[top] >= C) break;       // warp-uniform
      const uint32_t p = p0 + lane;
      const uint32_t m = mm[u];
      const bool live = m != SDB_META_TOMB;
      const uint32_t L = (live && prio_mode) ? (m >> 14) : 0u;
#pragma unroll
      for (uint32_t lev = 0; lev < 4; ++lev) {
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, live && L == lev);
        if (live && L == lev) {
          const uint32_t k = cnt[lev] + lane_prefix(b, lane);
          if (k < C) cand[lev][k] = p;
        }
        cnt[lev] += __popc(b);
      }
      p0 += 32;
    }
  }
  const uint32_t scan_end = static_cast<int32_t>(T - p0) > 0 ? p0 : T;
  __syncwarp();
  // quotas: everything of the higher levels first, then the first entries of the cut level
  uint32_t need = C, acc = 0, got = 0;
  for (int lev = 3; lev >= 0; --lev) {
    const uint32_t have = min(cnt[lev], C);
    const uint32_t take = min(have, need);
    for (uint32_t k = lane; k < take; k += 32) {
      const uint32_t p = cand[lev][k];
      const uint2 e = rs[p & mask];
      plan[RO + acc + k] = make_uint4(e.x, 0u, sdb_plan_z(e.y), slot);
      if (retire) rs[p & mask].y = SDB_META_TOMB;
    }
    acc += take; need -= take; got += take;
  }
  if (!retire) return;
  __syncwarp();
  // new head: the first live entry left (the tombstones just written count as consumed)
  const uint32_t nh = first_live_from(rs, mask, H, T, lane);
  if (lane == 0) {
    v.ring_hdr[A].head = nh;
    v.ring_hdr[A].ntomb = NT + got - (nh - H);
  }
}

// warp per listed agent (persistent grid-stride over the worklist built by k_recv_select)
__global__ void __launch_bounds__(256)
k_recv_select_big(sdb_dev_view v, sdb_recv_args r) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nw = (gridDim.x * blockDim.x) >> 5;
  __shared__ uint32_t s_cand[8][4][SDB_CAND];            // per warp: first C positions of each level
  const uint32_t n_big = *r.big_count;
  const bool prio_mode = (r.flags & SDB_RECV_PRIORITY) != 0;
  const bool retire = !(r.flags & SDB_RECV_PEEK);
  for (uint32_t w = gw; w < n_big; w += nw) {
    const uint32_t q = r.big_list[w];
    const uint32_t a = r.agent_idx ? r.agent_idx[q] : q;
    const uint32_t cnt = r.count_out[q];
    const uint32_t roff = sdb_scan_at(r.rec_local, r.rec_tops, q);
    const uint4 hd = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
    const uint32_t H = hd.x, T = hd.y, NT = hd.w;
    if (cnt <= SDB_CAND && (prio_mode || NT != 0))
      select_agent_warp_bounded(v, r.plan, q, prio_mode, a, H, T, NT, cnt, roff, lane, retire, s_cand[threadIdx.x >> 5]);
    else
      select_agent_warp(v, r.plan, q, prio_mode, a, H, T, NT, cnt, roff, lane, retire);
    __syncwarp();
  }
}

// scan over the per-record payload sizes (plan[].z) of the multi-kernel path; the tile-local exclusive prefix is
// stored back into plan[].y and the per-tile totals into `tops`.  The element count lives on the device (totals[0]).
__global__ void __launch_bounds__(1024)
k_scan_plan(uint4* __restrict__ plan, uint32_t* __restrict__ tops, const unsigned long long* __restrict__ n_dev) {
  const uint32_t n = static_cast<uint32_t>(*n_dev);
  const uint32_t base = blockIdx.x * SDB_SCAN_TILE + threadIdx.x * 4u;
  if (blockIdx.x * SDB_SCAN_TILE >= n) { if (threadIdx.x == 0) tops[blockIdx.x] = 0; return; }
  uint32_t x[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) x[k] = (base + k < n) ? (plan[base + k].z & 0xFFFFu) : 0u;
  uint32_t run = sdb_block_scan_tile(x, tops + blockIdx.x);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (base + k < n) plan[base + k].y = run;
    run += x[k];
  }
}

// ------------------------------------------------------------------------------------------
// SINGLE-PASS receive plan for stream order (the reference's order): count + both scans + select + retire in one
// kernel.  One thread per request slot, 256 slots per tile, tiles ordered by an atomic ticket; one hierarchical
// decoupled look-back (sdb_common.cuh: sdb_lb_prefix) carries {records, payload granules} as a 31+31-bit pair, so a
// record's output index and its payload offset come out of the same pass.
// Agents whose window holds consumed entries (holes left by earlier priority receives) are walked by their warp.
// Capacity: an agent whose records would run past rec_cap is left untouched together with every agent after it
// (whole-agent truncation, nothing is ever lost), except an agent first in the output (exclusive prefix 0), which takes
// its first rec_cap records; the totals are lowered with an atomic min on the packed pair.
//   r.lb               look-back scratch (layout in sdb_common.cuh, zeroed by the launcher), then the tile ticket, then
//                      ~(records << 32 | granules) of the call, maintained with atomicMax (= min of the value)
// ------------------------------------------------------------------------------------------
#ifndef SDB_PLAN_WARPS
#define SDB_PLAN_WARPS 8u
#endif
#define SDB_PLAN_TILE (32u * SDB_PLAN_WARPS)    // request slots per tile (one per thread)
#define SDB_PLAN_STAGE 256u                     // plan entries staged per warp before a coalesced write
// sum of the payload granules of the first C live entries of the window [H, T), whole warp
__device__ __forceinline__ uint32_t holey_sum_warp(const uint2* rs, uint32_t mask, uint32_t H, uint32_t T, uint32_t C, uint32_t lane) {
  uint32_t taken = 0, sum = 0;
  for (uint32_t p0 = H; static_cast<int32_t>(T - p0) > 0 && taken < C; p0 += 32) {
    const uint32_t p = p0 + lane;
    const uint32_t m = static_cast<int32_t>(T - p) > 0 ? (rs[p & mask].y & 0xFFFFu) : SDB_META_TOMB;
    const bool live = m != SDB_META_TOMB;
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, live);
    if (live && taken + lane_prefix(b, lane) < C) sum += (m & SDB_META_GLEN_MASK) - 1u;
    taken += __popc(b);
  }
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, o);
  return sum;
}
// payload offsets of C freshly planned records [RO, RO + C): running sum of .z from g0, whole warp; returns the offset
// after the last one
__device__ __forceinline__ uint32_t fill_offsets_warp(uint4* plan, uint32_t RO, uint32_t C, uint32_t g0, uint32_t lane) {
  uint32_t run = g0;
  for (uint32_t j0 = 0; j0 < C; j0 += 32) {
    const uint32_t j = j0 + lane;
    const uint32_t g = j < C ? (plan[RO + j].z & 0xFFFFu) : 0u;
    const uint32_t incl = sdb_warp_incl_scan(g, lane);
    if (j < C) plan[RO + j].y = run + incl - g;
    run += __shfl_sync(0xFFFFFFFFu, incl, 31);
  }
  return run;
}

// Byte budgets (sdb_receive_budget): an agent's take is the longest prefix of its delivery order with at most C records
// and at most `lim` payload granules, or its first record alone when that one is larger.
// Whole warp over the window [H, T): {records, granules} of the take.  Stream order stops at the first entry that does
// not fit; priority order (PRIO) first counts {records, granules} per level, takes whole levels from the top while they
// fit, then the arrival-order prefix of the level where the limit falls.
template <bool PRIO>
__device__ __forceinline__ uint2 budget_take_warp(const uint2* rs, uint32_t mask, uint32_t H, uint32_t T, uint32_t C,
                                                  uint32_t lim, uint32_t lane) {
  uint32_t acc_c = 0, acc_g = 0, cut = 0;
  if (PRIO) {
    // per level: live records (nc) and their payload granules (hg)
    uint32_t hg0 = 0, hg1 = 0, hg2 = 0, hg3 = 0;
    uint32_t nc0 = 0, nc1 = 0, nc2 = 0, nc3 = 0;
    for (uint32_t p0 = H; static_cast<int32_t>(T - p0) > 0; p0 += 32) {
      const uint32_t p = p0 + lane;
      const uint32_t m = static_cast<int32_t>(T - p) > 0 ? (rs[p & mask].y & 0xFFFFu) : SDB_META_TOMB;
      const bool live = m != SDB_META_TOMB;
      const uint32_t L = m >> 14, g = (m & SDB_META_GLEN_MASK) - 1u;
      nc0 += live && L == 0; nc1 += live && L == 1; nc2 += live && L == 2; nc3 += live && L == 3;
      hg0 += (live && L == 0) ? g : 0u; hg1 += (live && L == 1) ? g : 0u;
      hg2 += (live && L == 2) ? g : 0u; hg3 += (live && L == 3) ? g : 0u;
    }
    cut = 4;                                                  // 4: every level fits
    auto level = [&](uint32_t L, uint32_t nc, uint32_t hg) {
      const uint32_t c = __reduce_add_sync(0xFFFFFFFFu, nc), g = __reduce_add_sync(0xFFFFFFFFu, hg);
      if (cut == 4) {
        if (acc_c + c <= C && acc_g + g <= lim) { acc_c += c; acc_g += g; }
        else cut = L;
      }
    };
    level(3, nc3, hg3); level(2, nc2, hg2); level(1, nc1, hg1); level(0, nc0, hg0);
    if (cut == 4) return make_uint2(acc_c, acc_g);
  }
  uint32_t taken = 0, sum = 0;
  for (uint32_t p0 = H; static_cast<int32_t>(T - p0) > 0 && acc_c + taken < C; p0 += 32) {
    const uint32_t p = p0 + lane;
    const uint32_t m = static_cast<int32_t>(T - p) > 0 ? (rs[p & mask].y & 0xFFFFu) : SDB_META_TOMB;
    const bool sel = m != SDB_META_TOMB && (!PRIO || (m >> 14) == cut);
    const uint32_t g = sel ? (m & SDB_META_GLEN_MASK) - 1u : 0u;
    const uint32_t b = __ballot_sync(0xFFFFFFFFu, sel);
    const uint32_t k = acc_c + taken + lane_prefix(b, lane);                   // rank in the delivery order
    const uint32_t run = acc_g + sum + sdb_warp_incl_scan(g, lane);
    const bool ok = sel && k < C && (run <= lim || k == 0);
    const uint32_t bo = __ballot_sync(0xFFFFFFFFu, ok);
    sum += __reduce_add_sync(0xFFFFFFFFu, ok ? g : 0u);
    taken += __popc(bo);
    if (bo != b) break;                                        // an entry did not fit: the take ends before it
  }
  return make_uint2(acc_c + taken, acc_g + sum);
}
// one thread, the first n (<= 8) entries of a window without holes held in registers: records of the take, granules in gsum
__device__ __forceinline__ uint32_t budget_take_regs(const uint64_t (&ev)[8], uint32_t n, uint32_t lim, uint32_t& gsum) {
  uint32_t take = 0, sum = 0;
  bool open = true;
#pragma unroll
  for (uint32_t j = 0; j < 8; ++j) {
    if (open && j < n) {
      const uint32_t g = (static_cast<uint32_t>(ev[j] >> 32) & SDB_META_GLEN_MASK) - 1u;
      if (j == 0 || sum + g <= lim) { sum += g; take = j + 1; }
      else open = false;
    }
  }
  gsum = sum;
  return take;
}

// MODE: SDB_PLAN_PLAIN (sdb_receive_batch, stream order), SDB_PLAN_BUDGET (byte budgets, stream order),
// SDB_PLAN_BUDGET_PRIO (byte budgets, priority order: every agent is walked and selected by its warp),
// SDB_PLAN_TOKENS / SDB_PLAN_TOKENS_PRIO (token budgets: the budget modes with min(max_messages, cnt[q]) records per
// agent, cnt[q] written by k_token_take).
// budget = {per-agent limit, call capacity} in payload granules, read by the budget and token modes only.
enum { SDB_PLAN_PLAIN = 0, SDB_PLAN_BUDGET = 1, SDB_PLAN_BUDGET_PRIO = 2, SDB_PLAN_TOKENS = 3, SDB_PLAN_TOKENS_PRIO = 4 };
// at most 64 registers (4 CTAs per SM, the shared-memory limit allows 5): with 80, which the compiler picks otherwise,
// the c2 plan ran 13 % slower on an H100 (400 W power limit)
template <int MODE>
__global__ void __launch_bounds__(SDB_PLAN_TILE, 4)
k_recv_plan(sdb_dev_view v, sdb_recv_args r, uint32_t tiles, uint2 budget) {
  constexpr bool BUDGET = MODE != SDB_PLAN_PLAIN, PRIO = MODE == SDB_PLAN_BUDGET_PRIO || MODE == SDB_PLAN_TOKENS_PRIO;
  constexpr bool TOKENS = MODE == SDB_PLAN_TOKENS || MODE == SDB_PLAN_TOKENS_PRIO;
  __shared__ uint32_t s_tile;
  __shared__ unsigned long long s_wr[SDB_PLAN_WARPS], s_wg[SDB_PLAN_WARPS];
  __shared__ unsigned long long s_br, s_bg;
  __shared__ uint4 s_stage[SDB_PLAN_WARPS][SDB_PLAN_STAGE];                // per warp: plan entries on their way out (32 KB)
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const size_t ticket_at = static_cast<size_t>(tiles) + 3 * ((tiles + 31) / 32), totals_at = ticket_at + 1;
  // tile id from a ticket: tiles start in ticket order by construction, so every earlier tile the look-back waits on is
  // resident or finished
  if (tid == 0) s_tile = atomicAdd(reinterpret_cast<unsigned int*>(r.lb + ticket_at), 1u);
  __syncthreads();
  const uint32_t tile = s_tile;
  const uint32_t q = tile * SDB_PLAN_TILE + tid;
  const bool valid = q < r.n;
  const bool retire = !(r.flags & SDB_RECV_PEEK);
  const uint32_t R = v.ring_slots, mask = R - 1;
  constexpr uint32_t KEEP = 8;
  const uint64_t pol = sdb_policy_evict_last();

  uint32_t a = 0, head = 0, tail = 0, nt = 0, cnt = 0;
  uint4 h4 = make_uint4(0, 0, 0, 0);
  if (valid) {
    a = r.agent_idx ? r.agent_idx[q] : q;
    if (a < v.max_agents) {
      h4 = *reinterpret_cast<const uint4*>(v.ring_hdr + a);                 // head, tail, ctail, ntomb
      head = h4.x; tail = h4.y; nt = h4.w;
      cnt = min(tail - head - nt, r.max_messages);
      if constexpr (TOKENS) cnt = min(cnt, r.cnt[q]);                       // both takes are prefixes of one order
    }
  }
  const bool holey = cnt && (PRIO || nt != 0);      // planned by the warp (select_agent_warp)
  const bool simple = cnt && !holey;
  const bool in_regs = simple && cnt <= KEEP;       // entries held in ev[] (decided before any capacity truncation)
  const bool walked = BUDGET ? cnt && !in_regs : holey;   // sized by the warp (long windows too under a byte budget)
  const uint2* rs = sdb_ring_of(v, valid && a < v.max_agents ? a : 0u);
  uint64_t ev[KEEP];
  uint32_t gsum = 0;
  if (simple) {
    if (in_regs) {
#pragma unroll
      for (uint32_t j = 0; j < KEEP; ++j)
        if (j < cnt) ev[j] = sdb_ld_u64_pol(reinterpret_cast<const uint64_t*>(rs + ((head + j) & mask)), pol);
      if constexpr (BUDGET) {
        cnt = budget_take_regs(ev, cnt, budget.x, gsum);
      } else {
#pragma unroll
        for (uint32_t j = 0; j < KEEP; ++j)
          if (j < cnt) gsum += (static_cast<uint32_t>(ev[j] >> 32) & SDB_META_GLEN_MASK) - 1u;
      }
    } else if (!BUDGET) {
      for (uint32_t j = 0; j < cnt; ++j) gsum += (rs[(head + j) & mask].y & SDB_META_GLEN_MASK) - 1u;
    }
  }
  // agents with holes: their warp walks the window (rare: stream-order receive after priority receives)
  for (uint32_t hb = __ballot_sync(0xFFFFFFFFu, walked); hb; hb &= hb - 1) {
    const uint32_t src = __ffs(hb) - 1;
    const uint32_t A_ = __shfl_sync(0xFFFFFFFFu, a, src), H_ = __shfl_sync(0xFFFFFFFFu, head, src);
    const uint32_t T_ = __shfl_sync(0xFFFFFFFFu, tail, src), C_ = __shfl_sync(0xFFFFFFFFu, cnt, src);
    if constexpr (BUDGET) {
      const uint2 t = budget_take_warp<PRIO>(sdb_ring_of(v, A_), mask, H_, T_, C_, budget.x, lane);
      if (lane == src) { cnt = t.x; gsum = t.y; }
    } else {
      const uint32_t sum = holey_sum_warp(sdb_ring_of(v, A_), mask, H_, T_, C_, lane);
      if (lane == src) gsum = sum;
    }
  }

  // ---- tile scan of {records, granules} (two 64-bit sums: a pathological tile may exceed 32 bits before truncation)
  unsigned long long ir = cnt, ig = gsum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long yr = __shfl_up_sync(0xFFFFFFFFu, ir, o), yg = __shfl_up_sync(0xFFFFFFFFu, ig, o);
    if (lane >= o) { ir += yr; ig += yg; }
  }
  if (lane == 31) { s_wr[warp] = ir; s_wg[warp] = ig; }
  __syncthreads();
  if (warp == 0) {
    const unsigned long long wr = lane < SDB_PLAN_WARPS ? s_wr[lane] : 0ull, wg = lane < SDB_PLAN_WARPS ? s_wg[lane] : 0ull;
    unsigned long long cr = wr, cg = wg;
#pragma unroll
    for (int o = 1; o < static_cast<int>(SDB_PLAN_WARPS); o <<= 1) {
      const unsigned long long yr = __shfl_up_sync(0xFFFFFFFFu, cr, o), yg = __shfl_up_sync(0xFFFFFFFFu, cg, o);
      if (lane >= o) { cr += yr; cg += yg; }
    }
    const unsigned long long tr = __shfl_sync(0xFFFFFFFFu, cr, SDB_PLAN_WARPS - 1), tg = __shfl_sync(0xFFFFFFFFu, cg, SDB_PLAN_WARPS - 1);   // tile aggregate
    if (lane < SDB_PLAN_WARPS) { s_wr[lane] = cr - wr; s_wg[lane] = cg - wg; }                                           // exclusive warp offsets
    // ---- hierarchical decoupled look-back (sdb_common.cuh): exclusive prefix of {records, granules} over earlier tiles
    unsigned long long er, eg, ga, gb; bool last;
    sdb_lb_prefix(r.lb, tile, tiles, tr, tg, lane, er, eg, last, ga, gb);
    if (lane == 0) {
      s_br = er; s_bg = eg;
      if (last)                    // grand total of the call (before truncation; truncation only lowers it)
        atomicMax(r.lb + totals_at, ~((min(ga, 0xFFFFFFFFull) << 32) | min(gb, 0xFFFFFFFFull)));
    }
  }
  __syncthreads();
  const unsigned long long pr = s_br + s_wr[warp] + ir - cnt, pg = s_bg + s_wg[warp] + ig - gsum;   // exclusive prefix of this slot
  const uint32_t roff = static_cast<uint32_t>(min(pr, 0xFFFFFFFFull));
  const uint32_t goff = static_cast<uint32_t>(min(pg, 0xFFFFFFFFull));
  const bool over = cnt && (pr + cnt > r.rec_cap || (BUDGET && pg + gsum > budget.y));   // does not fit: stays queued ...
  const bool lead = over && pr == 0;                                            // ... unless first in the output: then it
  if (lead) {                                                                   // takes its first rec_cap records (their
    if constexpr (BUDGET) {                                                     // granules are summed while they are planned)
      cnt = static_cast<uint32_t>(min(static_cast<uint64_t>(cnt), r.rec_cap));  // or, under a byte budget, the longest
    } else {                                                                    // prefix of its take that fits both caps
      cnt = static_cast<uint32_t>(r.rec_cap);
    }
  } else if (over) {
    atomicMax(r.lb + totals_at, ~((static_cast<unsigned long long>(roff) << 32) | goff));
    cnt = 0;
  }
  if constexpr (BUDGET) {
    for (uint32_t hb = __ballot_sync(0xFFFFFFFFu, lead); hb; hb &= hb - 1) {    // at most one in the call
      const uint32_t src = __ffs(hb) - 1;
      const uint32_t A_ = __shfl_sync(0xFFFFFFFFu, a, src), H_ = __shfl_sync(0xFFFFFFFFu, head, src);
      const uint32_t T_ = __shfl_sync(0xFFFFFFFFu, tail, src), C_ = __shfl_sync(0xFFFFFFFFu, cnt, src);
      const uint2 t = budget_take_warp<PRIO>(sdb_ring_of(v, A_), mask, H_, T_, C_, budget.y, lane);
      if (lane == src) cnt = t.x;
    }
  }
  if (valid) { r.count_out[q] = cnt; r.rec_off[q] = roff; }

  uint32_t gend = goff;                                                         // payload granule offset after this slot
  // ---- plan entries of the warp's simple agents: staged in shared memory, written as whole 32-byte sectors
  // (per-thread 16-byte stores to scattered places would make the L2 fetch every sector before merging it)
  {
    const uint32_t mycnt = (cnt && simple) ? cnt : 0u;
    const uint32_t winc = sdb_warp_incl_scan(mycnt, lane);                     // inclusive scan over the warp
    const uint32_t wtotal = __shfl_sync(0xFFFFFFFFu, winc, 31);
    // the warp's simple records are NOT contiguous in the plan when it also holds holey or truncated agents; they are
    // contiguous per agent, so stage (destination, entry) pairs: destination index travels in a side array
    __shared__ uint32_t s_dst[SDB_PLAN_WARPS][SDB_PLAN_STAGE];
    const uint32_t lbase = winc - mycnt;                                        // local index of this lane's first entry
    for (uint32_t c0 = 0; c0 < wtotal; c0 += SDB_PLAN_STAGE) {
      uint32_t g0 = goff;
      if (mycnt) {
        for (uint32_t j = 0; j < mycnt; ++j) {
          uint64_t e;
          if (in_regs) {
            e = ev[0];
#pragma unroll
            for (uint32_t u = 1; u < KEEP; ++u) if (j == u) e = ev[u];
          } else {
            e = sdb_ld_u64_pol(reinterpret_cast<const uint64_t*>(rs + ((head + j) & mask)), pol);
          }
          const uint32_t g = (static_cast<uint32_t>(e >> 32) & SDB_META_GLEN_MASK) - 1u;
          const uint32_t li = lbase + j;
          if (li >= c0 && li < c0 + SDB_PLAN_STAGE) {
            s_stage[warp][li - c0] = make_uint4(static_cast<uint32_t>(e), g0, g | (static_cast<uint32_t>(e >> 32) & 0xFFFF0000u), q);
            s_dst[warp][li - c0] = roff + j;
          }
          g0 += g;
        }
        gend = g0;
      }
      __syncwarp();
      const uint32_t nst = min(SDB_PLAN_STAGE, wtotal - c0);
      for (uint32_t i = lane; i < nst; i += 32) r.plan[s_dst[warp][i]] = s_stage[warp][i];
      __syncwarp();
    }
    // the whole 16-byte header goes back in one store: neighbouring agents' headers then leave as full sectors
    // (a 4-byte store per agent is a partial-sector write the L2 has to merge)
    if (mycnt && retire) { h4.x = head + cnt; *reinterpret_cast<uint4*>(v.ring_hdr + a) = h4; }
  }
  for (uint32_t hb = __ballot_sync(0xFFFFFFFFu, holey && cnt); hb; hb &= hb - 1) {
    const uint32_t src = __ffs(hb) - 1;
    const uint32_t A_ = __shfl_sync(0xFFFFFFFFu, a, src), H_ = __shfl_sync(0xFFFFFFFFu, head, src);
    const uint32_t T_ = __shfl_sync(0xFFFFFFFFu, tail, src), C_ = __shfl_sync(0xFFFFFFFFu, cnt, src);
    const uint32_t N_ = __shfl_sync(0xFFFFFFFFu, nt, src), RO_ = __shfl_sync(0xFFFFFFFFu, roff, src);
    const uint32_t G_ = __shfl_sync(0xFFFFFFFFu, goff, src), Q_ = __shfl_sync(0xFFFFFFFFu, q, src);
    select_agent_warp(v, r.plan, Q_, PRIO, A_, H_, T_, N_, C_, RO_, lane, retire);
    __threadfence_block();
    __syncwarp();
    const uint32_t end = fill_offsets_warp(r.plan, RO_, C_, G_, lane);
    if (lane == src) gend = end;
  }
  if (lead) atomicMax(r.lb + totals_at, ~((static_cast<unsigned long long>(cnt) << 32) | gend));
  uint32_t n_deliv = retire ? cnt : 0u;
  for (int o = 16; o; o >>= 1) n_deliv += __shfl_xor_sync(0xFFFFFFFFu, n_deliv, o);
  if (lane == 0 && n_deliv) atomicAdd(&v.ctr->delivered, static_cast<unsigned long long>(n_deliv));
}

// ------------------------------------------------------------------------------------------
// gather: flat over output records, 8 lanes per record (4 records per warp step), all loads of a
// step issued before its stores.  Pure indexed copy: arena record -> hdr_out[r] + payload_out.
// The first thread also publishes the call's totals where the host (and the digest kernel) read them.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void gather_record(const sdb_dev_view& v, const sdb_recv_args& r, uint32_t rec, uint32_t l8, uint64_t pol) {
  const uint4 pe = __ldg(r.plan + rec);                        // handle, payload offset, payload granules, slot
  const uint32_t g = pe.z & 0xFFFFu;
  const uint64_t po = static_cast<uint64_t>(pe.y) + (r.plan_tops ? r.plan_tops[rec / SDB_SCAN_TILE] : 0u);
  const uint8_t* src = v.arena + ((static_cast<uint64_t>(pe.x) & v.gmask) << 5);
  const uint8_t* psrc = sdb_payload_of(v, pe.x, sdb_entry_dm1(pe.z)) - 32;   // payload chunk c >= 2 comes from psrc + 16 c
  uint8_t* hdst = reinterpret_cast<uint8_t*>(r.hdr_out + rec);
  uint8_t* pdst = r.payload_out + (po << 5) - 32;          // chunk c >= 2 lands at pdst + 16 c
  const uint32_t nchunk = 2u + (g << 1);
  for (uint32_t c = l8; c < nchunk; c += 24) {
    const uint32_t c1 = c + 8, c2 = c + 16;
    uint4 x0 = sdb_ld_stream_pol((c < 2 ? src : psrc) + (c << 4), pol), x1, x2;
    if (c1 < nchunk) x1 = sdb_ld_stream_pol(psrc + (c1 << 4), pol);
    if (c2 < nchunk) x2 = sdb_ld_stream_pol(psrc + (c2 << 4), pol);
    sdb_st_stream_pol((c < 2 ? hdst : pdst) + (c << 4), x0, pol);
    if (c1 < nchunk) sdb_st_stream_pol(pdst + (c1 << 4), x1, pol);
    if (c2 < nchunk) sdb_st_stream_pol(pdst + (c2 << 4), x2, pol);
  }
}
__device__ __forceinline__ uint32_t gather_total(const sdb_recv_args& r, const unsigned long long* packed_inv) {
  if (!packed_inv) return static_cast<uint32_t>(r.totals[0]);
  const unsigned long long pk = ~*packed_inv;
  if (blockIdx.x == 0 && threadIdx.x == 0) { r.totals[0] = pk >> 32; r.totals[1] = pk & 0xFFFFFFFFull; }
  return static_cast<uint32_t>(pk >> 32);
}

__global__ void __launch_bounds__(256)
k_recv_gather(sdb_dev_view v, sdb_recv_args r, const unsigned long long* __restrict__ packed_inv) {
  const uint32_t total = gather_total(r, packed_inv);
  const uint32_t lane = threadIdx.x & 31, sub = lane >> 3, l8 = lane & 7;
  const uint64_t pol = sdb_policy_evict_first();
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nw = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t r0 = gw * 4u; r0 < total; r0 += nw * 4u) {
    const uint32_t rec = r0 + sub;
    if (rec < total) gather_record(v, r, rec, l8, pol);
  }
}

// The same copy with the TMA engine doing the moving: every lane owns one record per step and issues ONE bulk load of the
// whole record (header + padded payload, 32-byte granules) into its shared-memory slot, completion counted on the
// warp's mbarrier; when a step has landed the lane issues two bulk stores (header -> hdr_out[r], payload -> the packed
// stream).  Two stages per warp: while step i is being stored, step i + 1 is already in flight.  A lane never touches
// the bytes, so the kernel needs few registers, and a CTA keeps stage_bytes x 32 lanes x 2 stages x warps in flight -
// several times what 16-byte loads held in registers can.  Used when a record fits the per-lane slot.
// A per-lane bulk copy costs the warp ~12 issue slots (the copy engine takes its operands from uniform registers), which
// looked like the limit with the payloads coming out of the L2.  It is not: a form with the whole warp moving the
// payloads by 16-byte cp.async copies ran the c2 gather in the same 0.775 ms on an H100 (700 W) and was removed.
// L2 policy: a payload shared by a group send is read once per member, at places spread over the whole receiver-ordered
// output, so its loads are evict-last; everything the kernel touches once (plan entries, headers in, headers and
// payloads out) is evict-first.  On an H100 (700 W) the c2 gather went from 0.782 to 0.686 ms.  Splitting the copy into
// a header pass and a payload pass did not pay (scripts/ubench/gather_phases.cu, DESIGN §8 item 19).
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
k_recv_gather_tma(sdb_dev_view v, sdb_recv_args r, const unsigned long long* __restrict__ packed_inv, uint32_t slot_bytes) {
  extern __shared__ __align__(128) uint8_t s_dyn[];          // [WARPS][2][32][slot_bytes]
  __shared__ __align__(8) uint64_t s_bar[WARPS][2];
  const uint32_t total = gather_total(r, packed_inv);
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* const wbase = s_dyn + static_cast<size_t>(warp) * 2u * 32u * slot_bytes;
  if (lane == 0) { sdb_mbar_init(&s_bar[warp][0], 1); sdb_mbar_init(&s_bar[warp][1], 1); sdb_fence_barrier_init(); }
  __syncwarp();
  const uint32_t gw = blockIdx.x * WARPS + warp, nw = gridDim.x * WARPS;
  uint32_t phase = 0;                                        // bit s = parity of stage s
  const uint64_t pol = sdb_policy_evict_first(), keep = sdb_policy_evict_last();
  // per-lane state of the two stages.  The 32-byte header travels through registers (two 16-byte loads now, stored one
  // step later: the lanes' headers are consecutive in hdr_out, and sdb_st_headers swaps halves between lanes so that
  // each of the warp's two store instructions writes 512 contiguous bytes of whole sectors; stored as loaded, every
  // sector would reach the L2 as two partial writes, at about half the write bandwidth); the payload - right
  // behind the header, or shared by all recipients of a group send (sdb_common.cuh) - takes ONE bulk load and ONE
  // bulk store.  Two bulk operations per record instead of three: the copy engine, not DRAM, was the limit once the
  // payloads came out of the L2.
  uint32_t g0 = 0, g1 = 0; uint64_t po0 = 0, po1 = 0; bool hv0 = false, hv1 = false;
  uint4 ha0 = make_uint4(0, 0, 0, 0), hb0 = ha0, ha1 = ha0, hb1 = ha0;
  uint4 pe_ahead = make_uint4(0, 0, 0, 0);                   // plan entry of the step after the one being requested
  auto issue = [&](uint32_t st, uint32_t r0) {               // all lanes: request step r0 into stage st
    const uint32_t rec = r0 + lane;
    const bool have = rec < total;
    uint32_t bytes = 0; uint4 pe = make_uint4(0, 0, 0, 0);
    if (have) { pe = pe_ahead; bytes = (pe.z & 0xFFFFu) << 5; }
    { const uint32_t ra = rec + nw * 32u; if (ra < total) pe_ahead = sdb_ld_stream_pol(r.plan + ra, pol); }   // consumed one step later
    uint32_t sum = bytes;
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, o);
    if (lane == 0) sdb_mbar_expect_tx(&s_bar[warp][st], sum);
    __syncwarp();
    uint4 ha = make_uint4(0, 0, 0, 0), hb = ha;
    if (have) {
      const uint8_t* src = v.arena + ((static_cast<uint64_t>(pe.x) & v.gmask) << 5);
      ha = sdb_ld_stream_pol(src, pol); hb = sdb_ld_stream_pol(src + 16, pol);
      if (bytes) sdb_tma_load_pol(wbase + (static_cast<size_t>(st) * 32u + lane) * slot_bytes, sdb_payload_of(v, pe.x, sdb_entry_dm1(pe.z)), bytes, &s_bar[warp][st], keep);
    }
    const uint64_t po = static_cast<uint64_t>(pe.y) + ((have && r.plan_tops) ? r.plan_tops[rec / SDB_SCAN_TILE] : 0u);
    if (st) { g1 = pe.z & 0xFFFFu; hv1 = have; po1 = po; ha1 = ha; hb1 = hb; }
    else { g0 = pe.z & 0xFFFFu; hv0 = have; po0 = po; ha0 = ha; hb0 = hb; }
  };
  uint32_t r0 = gw * 32u;
  if (r0 + lane < total) pe_ahead = sdb_ld_stream_pol(r.plan + r0 + lane, pol);
  if (r0 < total) issue(0, r0);
  uint32_t st = 0;
  for (; r0 < total; r0 += nw * 32u, st ^= 1u) {
    const uint32_t rn = r0 + nw * 32u;
    // the other stage was last read by the bulk stores of the step before this one: they must have finished reading it
    sdb_tma_wait_read<0>();
    __syncwarp();
    if (rn < total) issue(st ^ 1u, rn);
    sdb_st_headers_pol<32>(r.hdr_out + r0, sdb_sel4(st, ha1, ha0), sdb_sel4(st, hb1, hb0), st ? hv1 : hv0, lane, pol);   // whole sectors
    sdb_mbar_wait_bounded(&s_bar[warp][st], (phase >> st) & 1u);
    phase ^= 1u << st;
    {
      const bool hv = st ? hv1 : hv0;
      const uint32_t g = st ? g1 : g0;
      // payload offsets are cumulative in record order: when all 32 payloads fill their slots exactly, the warp's output
      // is ONE contiguous run and the slots are contiguous too - one bulk store instead of 32
      if (__all_sync(0xFFFFFFFFu, hv && (g << 5) == slot_bytes)) {
        if (lane == 0) sdb_tma_store_pol(r.payload_out + ((st ? po1 : po0) << 5), wbase + static_cast<size_t>(st) * 32u * slot_bytes, 32u * slot_bytes, pol);
      } else if (hv && g) {
        sdb_tma_store_pol(r.payload_out + ((st ? po1 : po0) << 5), wbase + (static_cast<size_t>(st) * 32u + lane) * slot_bytes, g << 5, pol);
      }
    }
    sdb_tma_commit();
  }
  sdb_tma_wait_all<0>();
}

// ------------------------------------------------------------------------------------------
// compact receive (sdb_receive_compact): the same plan, then one 16-byte entry per record and one row + payload per
// distinct payload image.  A record's image is identified by its payload position p = handle + 1 + dm1 (mod 2^32):
// the records of one shared-layout group send all point at the same p, every other record has its own (pending
// images never overlap and the arena holds fewer than 2^32 granules).  Rows are numbered in order of first appearance:
//   k_compact_owner   one thread per record: insert p into an open-addressing table, keep the smallest record naming
//                     it (slot = p << 32 | record; one CAS claims an empty slot, an atomicMin on the same key lowers
//                     the record)
//   k_compact_heads   head flag where a record owns its image, and the image's payload granules at its owner
//   scans             exclusive scans of both (k_scan_local + k_scan_tops): row index and payload offset
//   k_compact_emit    every record writes its entry; owners write the row and copy the payload once
// Record counts come from the plan's totals on the device (as the gathers read them): no host round trip.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_compact_owner(sdb_recv_args r, const unsigned long long* __restrict__ packed_inv, sdb_compact_args c) {
  const uint32_t total = gather_total(r, packed_inv);
  const uint32_t tmask = (1u << c.tbits) - 1u;
  for (uint32_t rec = blockIdx.x * blockDim.x + threadIdx.x; rec < total; rec += gridDim.x * blockDim.x) {
    const uint4 pe = __ldg(r.plan + rec);
    const uint32_t p = pe.x + 1u + sdb_entry_dm1(pe.z);
    const unsigned long long mine = (static_cast<unsigned long long>(p) << 32) | rec;
    uint32_t s = (p * 0x9E3779B1u) >> (32u - c.tbits);            // Fibonacci hash: strided positions spread evenly
    for (;;) {
      unsigned long long cur = __ldcg(c.table + s);
      if (cur == ~0ull) {
        cur = atomicCAS(c.table + s, ~0ull, mine);
        if (cur == ~0ull) break;
      }
      if ((cur >> 32) == p) {                                     // same key: min over the record half only
        if (static_cast<uint32_t>(cur) > rec) atomicMin(c.table + s, mine);
        break;
      }
      s = (s + 1u) & tmask;
    }
    c.rec_slot[rec] = s;
  }
}

__global__ void __launch_bounds__(256)
k_compact_heads(sdb_recv_args r, sdb_compact_args c, uint32_t bound) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= bound) return;
  const uint32_t total = static_cast<uint32_t>(r.totals[0]);
  uint32_t h = 0, g = 0;
  if (i < total) {
    const uint32_t own = static_cast<uint32_t>(c.table[c.rec_slot[i]]);
    c.rec_slot[i] = own;
    h = own == i;
    if (h) g = r.plan[i].z & 0xFFFFu;
  }
  c.head[i] = h;
  c.gran[i] = g;
}

// 8 lanes per record, 4 records per warp step: lane 0 reads the 32-byte header and writes the entry (and, at an owner,
// the row); an owner's 8 lanes copy its padded payload in 16-byte chunks
__global__ void __launch_bounds__(256)
k_compact_emit(sdb_dev_view v, sdb_recv_args r, sdb_compact_args c) {
  const uint32_t total = static_cast<uint32_t>(r.totals[0]);
  const uint32_t lane = threadIdx.x & 31, sub = lane >> 3, l8 = lane & 7;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nw = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t r0 = gw * 4u; r0 < total; r0 += nw * 4u) {
    const uint32_t rec = r0 + sub;
    if (rec >= total) continue;
    const uint4 pe = __ldg(r.plan + rec);
    const uint32_t own = c.rec_slot[rec];
    const bool head = own == rec;
    const uint64_t po = head ? (static_cast<uint64_t>(c.gran_local[rec]) + c.gran_tops[rec / SDB_SCAN_TILE]) << 5 : 0u;
    if (l8 == 0) {
      const uint8_t* src = v.arena + ((static_cast<uint64_t>(pe.x) & v.gmask) << 5);
      const uint4 lo = sdb_ld_stream(src), hi = sdb_ld_stream(src + 16);    // {seq, timestamp}, {sender, receiver, group, len|prio|type}
      const uint32_t row = sdb_scan_at(c.head_local, c.head_tops, own);
      sdb_st_stream(c.entry_out + rec, make_uint4(lo.x, lo.y, row, hi.y));
      if (head) {
        uint4* dst = reinterpret_cast<uint4*>(c.send_out + row);
        sdb_st_stream(dst, make_uint4(lo.z, lo.w, static_cast<uint32_t>(po), static_cast<uint32_t>(po >> 32)));
        sdb_st_stream(dst + 1, make_uint4(hi.x, hi.z, hi.w, 0u));
      }
    }
    if (head) {
      const uint32_t nchunk = (pe.z & 0xFFFFu) << 1;
      const uint8_t* psrc = sdb_payload_of(v, pe.x, sdb_entry_dm1(pe.z));
      uint8_t* pdst = c.payload_out + po;
      for (uint32_t k = l8; k < nchunk; k += 8) sdb_st_stream(pdst + (k << 4), sdb_ld_stream(psrc + (k << 4)));
    }
  }
}

static cudaError_t launch_compact(const sdb_dev_view* v, const sdb_recv_args* r, const sdb_compact_args* c0,
                                  const unsigned long long* packed_inv, uint64_t bound, int sm_count, cudaStream_t stream,
                                  sdb_profiler* prof, int* n_launches) {
  sdb_compact_args c = *c0;
  uint32_t tbits = 10;                                         // at least twice as many slots as records: load <= 1/2
  while ((1ull << tbits) < 2 * bound) ++tbits;
  c.tbits = tbits;
  const uint32_t n = static_cast<uint32_t>(bound);
  const int pi = sdb_prof_begin(prof, SDB_PK_RECV_COMPACT, stream);
  cudaMemsetAsync(c.table, 0xFF, (1ull << tbits) * sizeof(unsigned long long), stream);
  k_compact_owner<<<sdb_grid(bound, 256, 8 * sm_count), 256, 0, stream>>>(*r, packed_inv, c);
  k_compact_heads<<<static_cast<uint32_t>((bound + 255) / 256), 256, 0, stream>>>(*r, c, n);
  cudaError_t e = sdb_scan_u32(c.head, c.head_local, c.head_tops, n, c.totals, nullptr, stream, n_launches);
  if (e == cudaSuccess) e = sdb_scan_u32(c.gran, c.gran_local, c.gran_tops, n, c.totals + 1, nullptr, stream, n_launches);
  k_compact_emit<<<sdb_grid(bound, 32, 32 * sm_count), 256, 0, stream>>>(*v, *r, c);   // 4 records per warp, 8 warps per block
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += 3;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// ------------------------------------------------------------------------------------------
// stream digests (definition in include/swarmdb_b200.h): one warp per request slot folds the records the last
// receive delivered to that agent, in delivery order, into digest[agent].  Lanes hash the 64-bit words of a
// record in parallel (the per-word terms are position-keyed and summed), lane 0 chains the records.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long sdb_fmix64(unsigned long long x) {
  x ^= x >> 33; x *= 0xFF51AFD7ED558CCDull; x ^= x >> 33; x *= 0xC4CEB9FE1A85EC53ull; x ^= x >> 33;
  return x;
}
__global__ void __launch_bounds__(256)
k_recv_digest(sdb_recv_args r, uint32_t max_agents, unsigned long long* __restrict__ digest) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nw = (gridDim.x * blockDim.x) >> 5;
  const unsigned long long K = 0x9E3779B97F4A7C15ull;
  for (uint32_t q = gw; q < r.n; q += nw) {
    const uint32_t cnt = r.count_out[q];
    if (cnt == 0) continue;
    const uint32_t a = r.agent_idx ? r.agent_idx[q] : q;
    if (a >= max_agents) continue;
    const uint32_t roff = r.rec_off[q];
    unsigned long long d = digest[a];
    for (uint32_t j = 0; j < cnt; ++j) {
      const uint32_t rec = roff + j;
      const unsigned long long* hw = reinterpret_cast<const unsigned long long*>(r.hdr_out + rec);
      const uint32_t len = r.hdr_out[rec].len;
      const uint32_t nwords = 4u + (((len + 31u) & ~31u) >> 3);
      const unsigned long long po = (static_cast<unsigned long long>(r.plan[rec].y) + (r.plan_tops ? r.plan_tops[rec / SDB_SCAN_TILE] : 0u)) << 5;
      const unsigned long long* pw = reinterpret_cast<const unsigned long long*>(r.payload_out + po);
      unsigned long long acc = 0;
      for (uint32_t k = lane; k < nwords; k += 32) {
        const unsigned long long w = k < 4u ? hw[k] : pw[k - 4u];
        acc += sdb_fmix64(w ^ (static_cast<unsigned long long>(k + 1u) * K));
      }
      for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xFFFFFFFFu, acc, o);
      d = (((d << 5) | (d >> 59)) ^ acc) * K;
    }
    if (lane == 0) digest[a] = d;
  }
}

extern "C" cudaError_t sdb_launch_digest(const sdb_recv_args* r, uint32_t max_agents, unsigned long long* digest,
                                         int sm_count, cudaStream_t stream) {
  if (r->n == 0) return cudaSuccess;
  uint32_t grid = static_cast<uint32_t>(sm_count) * 8u;
  const uint32_t need = (r->n + 7) / 8;
  if (grid > need) grid = need;
  k_recv_digest<<<grid, 256, 0, stream>>>(*r, max_agents, digest);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// latency path: up to 8 agents, up to 1024 records, ONE launch (count, scan, select, retire, gather).
// Output block: u64 total records | u64 total granules | u32 counts[8] | pad to 64 B | the records
// back to back in arena format (32-B header + padded payload), so the host needs one D2H.
// ------------------------------------------------------------------------------------------
#define SDB_SMALL_AGENTS 8u
#define SDB_SMALL_RECS 1024u
struct sdb_small_agents { uint32_t idx[SDB_SMALL_AGENTS]; };

__global__ void __launch_bounds__(256)
k_recv_small(sdb_dev_view v, sdb_small_agents ag, uint32_t n, uint32_t max_messages, uint32_t flags, uint32_t rec_cap,
             uint4* __restrict__ plan, uint8_t* __restrict__ out) {
  __shared__ uint32_t s_cnt[SDB_SMALL_AGENTS], s_roff[SDB_SMALL_AGENTS + 1], s_goff[SDB_SMALL_RECS + 1];
  __shared__ uint32_t s_total;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool mine = warp < n;
  const uint32_t a = mine ? ag.idx[warp] : 0u;
  uint32_t head = 0, tail = 0, nt = 0;
  if (lane == 0) {
    uint32_t c = 0;
    if (mine && a < v.max_agents) {
      const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
      head = h.x; tail = h.y; nt = h.w;
      c = min(tail - head - nt, max_messages);
    }
    s_cnt[warp] = c;
  }
  __syncthreads();
  if (tid == 0) {
    uint32_t acc = 0, total = 0; bool open = true;
    for (uint32_t w = 0; w < SDB_SMALL_AGENTS; ++w) {
      s_roff[w] = acc;
      const uint32_t c = s_cnt[w];
      if (open && acc + c <= rec_cap) total = acc + c;
      else if (open && acc == 0) { open = false; s_cnt[w] = rec_cap; total = rec_cap; }      // first in the output: its first rec_cap
      else { open = false; s_cnt[w] = 0; }                                                    // whole-agent truncation
      acc += c;
    }
    s_total = total;
  }
  __syncthreads();
  const uint32_t cnt = s_cnt[warp], roff = s_roff[warp];
  if (lane == 0 && mine) reinterpret_cast<uint32_t*>(out + 16)[warp] = cnt;
  if (cnt) {
    const uint32_t H = __shfl_sync(0xFFFFFFFFu, head, 0), T = __shfl_sync(0xFFFFFFFFu, tail, 0);
    const uint32_t NT = __shfl_sync(0xFFFFFFFFu, nt, 0);
    select_agent_warp(v, plan, warp, (flags & SDB_RECV_PRIORITY) != 0, a, H, T, NT, cnt, roff, lane,
                      !(flags & SDB_RECV_PEEK));
  }
  __syncthreads();
  const uint32_t total = s_total;
  if (warp == 0) {                       // record offsets (granules, header included)
    uint32_t run = 0;
    for (uint32_t r0 = 0; r0 < total; r0 += 32) {
      const uint32_t r = r0 + lane;
      const uint32_t g = r < total ? (plan[r].z & 0xFFFFu) + 1u : 0u;
      const uint32_t incl = sdb_warp_incl_scan(g, lane);
      if (r < total) s_goff[r] = run + incl - g;
      run += __shfl_sync(0xFFFFFFFFu, incl, 31);
    }
    if (lane == 0) {
      s_goff[total] = run;
      reinterpret_cast<unsigned long long*>(out)[0] = total;
      reinterpret_cast<unsigned long long*>(out)[1] = run;
      if (total && !(flags & SDB_RECV_PEEK)) atomicAdd(&v.ctr->delivered, static_cast<unsigned long long>(total));
    }
  }
  __syncthreads();
  const uint32_t l8 = tid & 7;
  for (uint32_t r = tid >> 3; r < total; r += 32) {
    const uint4 pe = plan[r];
    const uint32_t g = pe.z & 0xFFFFu;
    const uint8_t* src = v.arena + ((static_cast<uint64_t>(pe.x) & v.gmask) << 5);
    const uint8_t* psrc = sdb_payload_of(v, pe.x, sdb_entry_dm1(pe.z)) - 32;
    uint8_t* dst = out + 64 + (static_cast<size_t>(s_goff[r]) << 5);
    const uint32_t nchunk = 2u + (g << 1);
    for (uint32_t c = l8; c < nchunk; c += 8) sdb_st_stream(dst + (c << 4), sdb_ld_stream((c < 2 ? src : psrc) + (c << 4)));
  }
}

// ------------------------------------------------------------------------------------------
// Low-latency dequeue SERVER: the same single-launch receive as k_recv_small for one agent, as a persistent CTA that
// polls a mailbox in mapped pinned host memory and writes its answer (the k_recv_small output block) into pinned host
// memory.  Request: {req_seq, agent, max_messages, flags}; the host bumps req_seq last.  Answer complete when
// done_seq == req_seq.  quit != 0 ends the kernel.  Mailbox layout: sdb_ls_mailbox (sdb_common.cuh).
// A persistent kernel sees other kernels' writes only through the L2: every request starts with a gpu-scope fence,
// which also invalidates this SM's L1 (a fence of scope >= cluster emits CCTL.IVALL), and the ring header
// is read with volatile loads.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 1)
k_latency_server(sdb_dev_view v, sdb_ls_mailbox* mb, uint8_t* out, uint32_t out_cap_bytes, uint4* plan) {
  __shared__ uint32_t s_req[4];         // seq, agent, max_messages, flags
  __shared__ uint32_t s_quit, s_cnt, s_total;
  __shared__ uint32_t s_goff[SDB_SMALL_RECS + 1];
  __shared__ uint2 s_fast[32];          // fast path: {arena handle, payload granules} of up to 32 records
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t served = 0;
  if (tid == 0) served = *reinterpret_cast<volatile uint32_t*>(&mb->done_seq);
  for (;;) {
    if (tid == 0) {
      // ONE 16-byte read per poll fetches the whole request {req_seq, agent, max_messages, flags}: every access to the
      // mailbox is a PCIe round trip, so the fields must not be fetched one by one.  flags bit 31 = quit.
      uint4 rq;
      for (;;) {
        asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(rq.x), "=r"(rq.y), "=r"(rq.z), "=r"(rq.w) : "l"(mb) : "memory");
        if (rq.x != served || (rq.w & 0x80000000u)) break;
        __nanosleep(20);
      }
      s_req[0] = rq.x; s_req[1] = rq.y; s_req[2] = rq.z; s_req[3] = rq.w & 0x7FFFFFFFu;
      s_quit = rq.w >> 31;
    }
    __syncthreads();
    if (s_quit) return;
    __threadfence();                                    // fresh view of the rings and the arena (L1 invalidated)
    const uint32_t a = s_req[1], max_messages = s_req[2], flags = s_req[3];
    const uint32_t rec_cap = min(SDB_SMALL_RECS, out_cap_bytes / 64u);
    uint32_t head = 0, tail = 0, nt = 0;
    if (tid < 32) {                                     // warp 0: header, then (short stream-order answers) the entries themselves
      uint32_t c = 0;
      if (a < v.max_agents) {
        const uint4 hd = __ldcv(reinterpret_cast<const uint4*>(v.ring_hdr + a));
        head = hd.x; tail = hd.y; nt = hd.w;
        c = min(min(tail - head - nt, max_messages), rec_cap);
      }
      const bool fast = c && c <= 32u && nt == 0 && !(flags & SDB_RECV_PRIORITY);
      if (fast) {
        // lane j owns record j: entry -> arena handle and size; offsets by a shuffle scan; nothing goes through memory
        uint2 e = make_uint2(0u, 1u);
        if (lane < c) e = __ldcv(sdb_ring_of(v, a) + ((head + lane) & (v.ring_slots - 1)));
        const uint32_t g = lane < c ? (sdb_meta(e) & SDB_META_GLEN_MASK) : 0u;       // granules incl. the header
        const uint32_t incl = sdb_warp_incl_scan(g, lane);
        if (lane < c) { s_goff[lane] = incl - g; s_fast[lane] = make_uint2(e.x, (g - 1u) | (e.y & 0xFFFF0000u)); }
        if (lane == c - 1) s_goff[c] = incl;
        if (lane == 0) {
          s_total = c; s_cnt = 0xFFFFFFFFu;                                          // marker: plan lives in shared memory
          if (!(flags & SDB_RECV_PEEK)) v.ring_hdr[a].head = head + c;
        }
      } else if (lane == 0) {
        s_cnt = c;
      }
    }
    __syncthreads();
    const bool fastpath = s_cnt == 0xFFFFFFFFu;
    const uint32_t cnt = fastpath ? 0u : s_cnt;
    if (warp == 0 && cnt) {
      const uint32_t H = __shfl_sync(0xFFFFFFFFu, head, 0), T = __shfl_sync(0xFFFFFFFFu, tail, 0);
      const uint32_t NT = __shfl_sync(0xFFFFFFFFu, nt, 0);
      select_agent_warp(v, plan, 0u, (flags & SDB_RECV_PRIORITY) != 0, a, H, T, NT, cnt, 0u, lane, !(flags & SDB_RECV_PEEK));
      __threadfence_block();
      __syncwarp();
      // record offsets (granules, header included)
      uint32_t run = 0;
      for (uint32_t r0 = 0; r0 < cnt; r0 += 32) {
        const uint32_t r = r0 + lane;
        const uint32_t g = r < cnt ? (plan[r].z & 0xFFFFu) + 1u : 0u;
        const uint32_t incl = sdb_warp_incl_scan(g, lane);
        if (r < cnt) s_goff[r] = run + incl - g;
        run += __shfl_sync(0xFFFFFFFFu, incl, 31);
      }
      if (lane == 0) { s_goff[cnt] = run; s_total = cnt; }
    }
    if (tid == 0 && !cnt && !fastpath) { s_total = 0; s_goff[0] = 0; }
    __syncthreads();
    const uint32_t total = s_total;
    const uint32_t l8 = tid & 7;
    for (uint32_t r = tid >> 3; r < total; r += 32) {
      uint32_t handle, gz;
      if (fastpath) { handle = s_fast[r].x; gz = s_fast[r].y; } else { const uint4 pe = plan[r]; handle = pe.x; gz = pe.z; }
      const uint32_t g = gz & 0xFFFFu;
      const uint8_t* src = v.arena + ((static_cast<uint64_t>(handle) & v.gmask) << 5);
      const uint8_t* psrc = sdb_payload_of(v, handle, sdb_entry_dm1(gz)) - 32;
      uint8_t* dst = out + 64 + (static_cast<size_t>(s_goff[r]) << 5);
      const uint32_t nchunk = 2u + (g << 1);
      for (uint32_t c = l8; c < nchunk; c += 8) *reinterpret_cast<uint4*>(dst + (c << 4)) = sdb_ld_stream((c < 2 ? src : psrc) + (c << 4));
    }
    if (tid == 0) {
      // totals | granules | count: one 32-byte store group at the head of the answer block
      reinterpret_cast<unsigned long long*>(out)[0] = total;
      reinterpret_cast<unsigned long long*>(out)[1] = s_goff[total];
      reinterpret_cast<uint32_t*>(out + 16)[0] = total;
      if (total && !(flags & SDB_RECV_PEEK)) atomicAdd(&v.ctr->delivered, static_cast<unsigned long long>(total));
    }
    __threadfence_system();                              // the answer is in host memory before the completion flag
    __syncthreads();
    if (tid == 0) {
      *reinterpret_cast<volatile uint32_t*>(&mb->done_seq) = s_req[0];
      __threadfence_system();
    }
    served = s_req[0];
    __syncthreads();
  }
}

extern "C" cudaError_t sdb_launch_latency_server(const sdb_dev_view* v, sdb_ls_mailbox* mb_dev, uint8_t* out_dev, uint32_t out_cap,
                                                 uint4* plan, cudaStream_t stream) {
  k_latency_server<<<1, 256, 0, stream>>>(*v, mb_dev, out_dev, out_cap, plan);
  return cudaGetLastError();
}

extern "C" cudaError_t sdb_launch_receive_small(const sdb_dev_view* v, const uint32_t* agents_host, uint32_t n,
                                                uint32_t max_messages, uint32_t flags, uint32_t rec_cap,
                                                uint4* plan, uint8_t* out,
                                                cudaStream_t stream, sdb_profiler* prof) {
  sdb_small_agents ag{};
  for (uint32_t i = 0; i < n && i < SDB_SMALL_AGENTS; ++i) ag.idx[i] = agents_host[i];
  const int pi = sdb_prof_begin(prof, SDB_PK_RECV_GATHER, stream);
  k_recv_small<<<1, 256, 0, stream>>>(*v, ag, n, max_messages, flags, rec_cap < SDB_SMALL_RECS ? rec_cap : SDB_SMALL_RECS,
                                      plan, out);
  sdb_prof_end(prof, pi, stream);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// max_rec_bytes: largest record (32-byte header + padded payload) this handle can hold; the TMA gather keeps one
// shared-memory slot of that size per lane and stage, so it is used for records up to 544 bytes (512-byte payloads)
static cudaError_t launch_gather(const sdb_dev_view* v, const sdb_recv_args* r, const unsigned long long* packed_inv,
                                 uint64_t bound, uint32_t max_rec_bytes, int sm_count, cudaStream_t stream,
                                 sdb_profiler* prof, int* n_launches) {
  const int pi = sdb_prof_begin(prof, SDB_PK_RECV_GATHER, stream);
  if (max_rec_bytes <= 544 && bound >= 4096) {
    constexpr int WARPS = 4;
    const uint32_t slot = max_rec_bytes > 64u ? max_rec_bytes - 32u : 32u;          // a slot stages the payload only
    const size_t smem = static_cast<size_t>(WARPS) * 2u * 32u * slot;
    uint32_t per_sm = static_cast<uint32_t>((226u * 1024u) / (smem + 1024 + 128));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 8) per_sm = 8;
    uint64_t grid = static_cast<uint64_t>(sm_count) * per_sm * 8u;                 // 8 waves: the tail evens out
    const uint64_t need = (bound + WARPS * 32 - 1) / (WARPS * 32);
    if (grid > need) grid = need;
    k_recv_gather_tma<WARPS><<<static_cast<uint32_t>(grid), WARPS * 32, smem, stream>>>(*v, *r, packed_inv, slot);
  } else {
    // 4 records per warp, 8 warps per block; grid-stride beyond ~4 waves
    k_recv_gather<<<sdb_grid(bound, 32, 32 * sm_count), 256, 0, stream>>>(*v, *r, packed_inv);
  }
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += 1;
  return cudaGetLastError();
}

extern "C" cudaError_t sdb_recv_prepare_device() {
  return cudaFuncSetAttribute(k_recv_gather_tma<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 2 * 32 * 544);
}

// ------------------------------------------------------------------------------------------
// token budgets (sdb_receive_tokens, sdb_pending_tokens).  A record whose type byte carries SDB_TYPEF_TOKENS and whose
// len is at least 4 weighs the little-endian u32 at the start of its payload; every other record weighs 0.
// k_token_take<PRIO> writes each request slot's token take to cnt[q]: the longest prefix of its delivery order whose
// token sum is <= lim, or its first record alone when that one is heavier.  Priority order takes whole levels from the
// top while they fit, then the arrival-order prefix of the level where the limit falls (budget_take_warp's rule).
// sums (nullable) receives the token sum of each take (lim = ~0: every pending record).
// k_expire's shape: 8 lanes per request slot, the ring header once, the window's entries coalesced, then per live entry
// the header's last word and the payload's first word - two independent random loads - 4 entries per lane in flight.
// Priority order walks twice: per-level totals, then the entries of the cut level only (none when every level fits).
// ------------------------------------------------------------------------------------------
#define SDB_TK_G 8u      // lanes per request slot
#define SDB_TK_U 4u      // entries per lane in flight

// the token weights of one step's entries (0 where sel is false)
__device__ __forceinline__ void tk_weights(const sdb_dev_view& v, const uint2 (&e)[SDB_TK_U], const bool (&sel)[SDB_TK_U],
                                           uint32_t (&tk)[SDB_TK_U]) {
  uint32_t hw[SDB_TK_U], pw[SDB_TK_U];
#pragma unroll
  for (uint32_t u = 0; u < SDB_TK_U; ++u) {             // all loads issued before any use
    hw[u] = sel[u] ? __ldg(reinterpret_cast<const uint32_t*>(v.arena + ((static_cast<uint64_t>(e[u].x) & v.gmask) << 5) + 28))
                   : 0u;                                 // len | prio << 16 | type << 24
    pw[u] = sel[u] && (sdb_meta(e[u]) & SDB_META_GLEN_MASK) > 1u
                ? __ldg(reinterpret_cast<const uint32_t*>(sdb_payload_of(v, e[u].x, sdb_entry_dm1(e[u].y))))
                : 0u;
  }
#pragma unroll
  for (uint32_t u = 0; u < SDB_TK_U; ++u)
    tk[u] = (((hw[u] >> 24) & SDB_TYPEF_TOKENS) && (hw[u] & 0xFFFFu) >= 4u) ? pw[u] : 0u;
}

// The walk of k_token_take and, with SEL, of k_where_take.  SEL: only the entries whose verdict bit is set (bits: the
// agent's row of f.bits) are walked, the take is also cut where their payload granules would pass glim, and
// cnt[q] = min(cnt[q], take) (cnt[q] as the where eval left it); the walk stops once the take reaches cnt[q].  lim and
// glim are ~0 for no limit; with lim = ~0 under SEL no payload word is read.
template <bool PRIO, bool SEL>
__device__ __forceinline__ void token_take_walk(const sdb_dev_view& v, const sdb_recv_args& r, unsigned long long lim,
                                                unsigned long long* __restrict__ sums, const uint32_t* __restrict__ fbits,
                                                uint32_t stride, unsigned long long glim) {
  const uint32_t lane = threadIdx.x & 31, l8 = lane & (SDB_TK_G - 1), gsh = lane & ~(SDB_TK_G - 1), below = (1u << l8) - 1u;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint32_t mask = v.ring_slots - 1;
  const bool tok = !SEL || lim != ~0ull;                        // token weights are read
  constexpr uint32_t SPW = 32u / SDB_TK_G;                      // request slots per warp
  for (uint32_t qb = gw * SPW; qb < r.n; qb += nw * SPW) {      // warp-uniform
    const uint32_t q = qb + lane / SDB_TK_G;
    const bool valid = q < r.n;
    uint32_t a = 0, H = 0, T = 0, NT = 0, cin = 0;
    if (valid) {
      a = r.agent_idx ? r.agent_idx[q] : q;
      const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);     // one address for the slot's 8 lanes
      H = h.x; T = h.y; NT = h.w;
      if (SEL) cin = r.cnt[q];
    }
    const uint32_t W = valid && T - H - NT && (!SEL || cin) ? T - H : 0u;
    const uint2* rs = sdb_ring_of(v, a);
    const uint32_t* bits = SEL ? fbits + static_cast<size_t>(a) * stride : nullptr;
    uint32_t take = 0, cut = 4;                                 // cut: the level where the limit falls (4: none)
    unsigned long long tsum = 0, gsum = 0;
    if (PRIO) {
      // 1. per level: live records and their tokens (and, SEL, granules)
      uint32_t c[4] = {0u, 0u, 0u, 0u};
      unsigned long long t[4] = {0ull, 0ull, 0ull, 0ull}, gs[4] = {0ull, 0ull, 0ull, 0ull};
      const uint32_t wmax = __reduce_max_sync(0xFFFFFFFFu, W);
      for (uint32_t j0 = 0; j0 < wmax; j0 += SDB_TK_G * SDB_TK_U) {
        const uint32_t word = SEL && j0 < W ? bits[j0 >> 5] : 0u;
        uint2 e[SDB_TK_U];
        bool lv[SDB_TK_U], lt[SDB_TK_U];
        uint32_t tk[SDB_TK_U];
#pragma unroll
        for (uint32_t u = 0; u < SDB_TK_U; ++u) {
          const uint32_t j = j0 + u * SDB_TK_G + l8;
          const bool in = j < W && (!SEL || ((word >> (u * SDB_TK_G + l8)) & 1u));
          e[u] = in ? rs[(H + j) & mask] : make_uint2(0u, SDB_META_TOMB);
          lv[u] = sdb_meta(e[u]) != SDB_META_TOMB;
          lt[u] = lv[u] && tok;
        }
        tk_weights(v, e, lt, tk);
#pragma unroll
        for (uint32_t u = 0; u < SDB_TK_U; ++u) {
          const uint32_t p = sdb_meta(e[u]) >> 14;
#pragma unroll
          for (uint32_t l = 0; l < 4; ++l)
            if (lv[u] && p == l) {
              c[l] += 1; t[l] += tk[u];
              if (SEL) gs[l] += (sdb_meta(e[u]) & SDB_META_GLEN_MASK) - 1u;
            }
        }
      }
#pragma unroll
      for (int l = 3; l >= 0; --l) {
#pragma unroll
        for (int o = 4; o; o >>= 1) {
          c[l] += __shfl_xor_sync(0xFFFFFFFFu, c[l], o);
          t[l] += __shfl_xor_sync(0xFFFFFFFFu, t[l], o);
          if (SEL) gs[l] += __shfl_xor_sync(0xFFFFFFFFu, gs[l], o);
        }
        if (cut == 4) {
          if (tsum + t[l] <= lim && (!SEL || gsum + gs[l] <= glim)) { take += c[l]; tsum += t[l]; gsum += gs[l]; }
          else cut = static_cast<uint32_t>(l);
        }
      }
    }
    // 2. stream order, or the arrival-order prefix of the cut level: entry i is taken while the running sums fit (or it
    // is the first of the delivery order); sums only grow, so the first one that does not fit ends the take
    const uint32_t W2 = (!PRIO || cut < 4) ? W : 0u;
    bool open = W2 != 0 && (!SEL || take < cin);
    const uint32_t wmax = __reduce_max_sync(0xFFFFFFFFu, W2);
    for (uint32_t j0 = 0; j0 < wmax && __any_sync(0xFFFFFFFFu, open); j0 += SDB_TK_G * SDB_TK_U) {
      const uint32_t word = SEL && open && j0 < W2 ? bits[j0 >> 5] : 0u;
      uint2 e[SDB_TK_U];
      bool sel[SDB_TK_U], st[SDB_TK_U];
      uint32_t tk[SDB_TK_U];
#pragma unroll
      for (uint32_t u = 0; u < SDB_TK_U; ++u) {
        const uint32_t j = j0 + u * SDB_TK_G + l8;
        const bool in = open && j < W2 && (!SEL || ((word >> (u * SDB_TK_G + l8)) & 1u));
        e[u] = in ? rs[(H + j) & mask] : make_uint2(0u, SDB_META_TOMB);
        sel[u] = sdb_meta(e[u]) != SDB_META_TOMB && (!PRIO || sdb_meta(e[u]) >> 14 == cut);
        st[u] = sel[u] && tok;
      }
      tk_weights(v, e, st, tk);
#pragma unroll
      for (uint32_t u = 0; u < SDB_TK_U; ++u) {
        const uint32_t bs = (__ballot_sync(0xFFFFFFFFu, sel[u]) >> gsh) & 0xFFu;
        const unsigned long long g = SEL && sel[u] ? (sdb_meta(e[u]) & SDB_META_GLEN_MASK) - 1u : 0u;
        unsigned long long x = tk[u], xg = g;                   // inclusive scans over the slot's 8 lanes
#pragma unroll
        for (uint32_t o = 1; o < SDB_TK_G; o <<= 1) {
          const unsigned long long y = __shfl_up_sync(0xFFFFFFFFu, x, o, SDB_TK_G);
          if (l8 >= o) x += y;
          if (SEL) {
            const unsigned long long yg = __shfl_up_sync(0xFFFFFFFFu, xg, o, SDB_TK_G);
            if (l8 >= o) xg += yg;
          }
        }
        const bool ok = open && sel[u] && (take + __popc(bs & below) == 0 ||
                                           (tsum + x <= lim && (!SEL || gsum + xg <= glim)));
        const uint32_t bo = (__ballot_sync(0xFFFFFFFFu, ok) >> gsh) & 0xFFu;
        unsigned long long s = ok ? tk[u] : 0ull, sg = ok ? g : 0ull;
#pragma unroll
        for (int o = 4; o; o >>= 1) {
          s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
          if (SEL) sg += __shfl_xor_sync(0xFFFFFFFFu, sg, o);
        }
        take += __popc(bo); tsum += s; gsum += sg;
        if (bo != bs) open = false;                             // an entry did not fit: the take ends before it
      }
      if (SEL && take >= cin) open = false;                     // max_messages (or the matches) reached
    }
    if (valid && l8 == 0) {
      r.cnt[q] = SEL ? min(cin, take) : take;
      if (sums) sums[q] = tsum;
    }
  }
}

template <bool PRIO>
__global__ void __launch_bounds__(256)
k_token_take(sdb_dev_view v, sdb_recv_args r, unsigned long long lim, unsigned long long* __restrict__ sums) {
  token_take_walk<PRIO, false>(v, r, lim, sums, nullptr, 0u, ~0ull);
}

// filtered take (sdb_receive_where_budget, sdb_receive_leased_select): between the where eval and the count scan,
// cnt[q] = min(cnt[q], the take of the matching records under the token limit lim and the granule limit glim)
template <bool PRIO>
__global__ void __launch_bounds__(256)
k_where_take(sdb_dev_view v, sdb_recv_args r, const uint32_t* __restrict__ bits, uint32_t stride, unsigned long long lim,
             unsigned long long glim) {
  token_take_walk<PRIO, true>(v, r, lim, nullptr, bits, stride, glim);
}

// cnt[q] = the token take of each request slot under `lim` (~0: everything pending), sums[q] (nullable) its token sum
extern "C" cudaError_t sdb_launch_token_take(const sdb_dev_view* v, const sdb_recv_args* r, unsigned long long lim,
                                             unsigned long long* sums, cudaStream_t stream, int* n_launches,
                                             sdb_profiler* prof, int sm_count) {
  if (r->n == 0) return cudaSuccess;
  const uint32_t blocks = sdb_grid(r->n, 32, 32 * sm_count);                 // 4 slots per warp, 8 warps per block
  const int pi = sdb_prof_begin(prof, SDB_PK_RECV_COUNT, stream);
  if (r->flags & SDB_RECV_PRIORITY)
    k_token_take<true><<<blocks, 256, 0, stream>>>(*v, *r, lim, sums);
  else
    k_token_take<false><<<blocks, 256, 0, stream>>>(*v, *r, lim, sums);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += 1;
  return cudaGetLastError();
}

// ca != nullptr: a compact receive (the same plan; the compact kernels replace the gather)
// budget != nullptr: byte budgets (sdb_receive_budget), {per-agent limit, call capacity} in payload granules; both orders
// take the single-pass plan
// max_tokens != 0 (with budget): token budgets (sdb_receive_tokens), k_token_take first, then the plan's token modes
extern "C" cudaError_t sdb_launch_receive(const sdb_dev_view* v, const sdb_recv_args* r0, cudaStream_t stream,
                                          int* n_launches, sdb_profiler* prof, int sm_count, uint32_t max_rec_bytes,
                                          const sdb_compact_args* ca, const uint2* budget, unsigned long long max_tokens) {
  if (r0->n == 0) return cudaSuccess;
  sdb_recv_args ra = *r0;
  sdb_recv_args* r = &ra;
  const uint32_t n = r->n;
  // upper bound on records: min(rec_cap, n * max_messages); grids sized from it, kernels read the true count
  uint64_t bound = static_cast<uint64_t>(n) * r->max_messages;
  if (bound > r->rec_cap) bound = r->rec_cap;
  int pi;
  if (!(r->flags & SDB_RECV_PRIORITY) || budget) {
    // ---- stream order (and byte budgets): single-pass plan + gather
    const uint32_t tiles = (n + SDB_PLAN_TILE - 1) / SDB_PLAN_TILE;
    r->plan_tops = nullptr;
    if (budget && max_tokens) {
      const cudaError_t e = sdb_launch_token_take(v, r, max_tokens, nullptr, stream, n_launches, prof, sm_count);
      if (e != cudaSuccess) return e;
    }
    pi = sdb_prof_begin(prof, SDB_PK_RECV_SELECT, stream);
    cudaMemsetAsync(r->lb, 0, sdb_lb_words(tiles) * sizeof(unsigned long long), stream);
    if (!budget)
      k_recv_plan<SDB_PLAN_PLAIN><<<tiles, SDB_PLAN_TILE, 0, stream>>>(*v, *r, tiles, make_uint2(0u, 0u));
    else if (max_tokens && (r->flags & SDB_RECV_PRIORITY))
      k_recv_plan<SDB_PLAN_TOKENS_PRIO><<<tiles, SDB_PLAN_TILE, 0, stream>>>(*v, *r, tiles, *budget);
    else if (max_tokens)
      k_recv_plan<SDB_PLAN_TOKENS><<<tiles, SDB_PLAN_TILE, 0, stream>>>(*v, *r, tiles, *budget);
    else if (r->flags & SDB_RECV_PRIORITY)
      k_recv_plan<SDB_PLAN_BUDGET_PRIO><<<tiles, SDB_PLAN_TILE, 0, stream>>>(*v, *r, tiles, *budget);
    else
      k_recv_plan<SDB_PLAN_BUDGET><<<tiles, SDB_PLAN_TILE, 0, stream>>>(*v, *r, tiles, *budget);
    sdb_prof_end(prof, pi, stream);
    if (n_launches) *n_launches += 1;
    if (ca) return launch_compact(v, r, ca, r->lb + sdb_lb_words(tiles) - 1, bound, sm_count, stream, prof, n_launches);
    return launch_gather(v, r, r->lb + sdb_lb_words(tiles) - 1, bound, max_rec_bytes, sm_count, stream, prof, n_launches);
  }
  pi = sdb_prof_begin(prof, SDB_PK_RECV_COUNT, stream);
  k_recv_count<<<(n + 255) / 256, 256, 0, stream>>>(*v, *r);
  sdb_prof_end(prof, pi, stream);
  pi = sdb_prof_begin(prof, SDB_PK_RECV_SCAN, stream);
  // totals[0] = records requested
  const cudaError_t e = sdb_scan_u32(r->cnt, r->rec_local, r->rec_tops, n, r->totals, nullptr, stream, n_launches);
  sdb_prof_end(prof, pi, stream);
  pi = sdb_prof_begin(prof, SDB_PK_RECV_SELECT, stream);
  cudaMemsetAsync(r->big_count, 0, sizeof(uint32_t), stream);
  k_recv_select<<<(n + 255) / 256, 256, 0, stream>>>(*v, *r);                   // may lower totals[0] (capacity)
  {
    uint32_t bg = static_cast<uint32_t>(sm_count) * 8u;                         // 8 warps per CTA, 8 CTAs per SM
    const uint32_t need = (n + 7) / 8;
    if (bg > need) bg = need;
    k_recv_select_big<<<bg, 256, 0, stream>>>(*v, *r);
  }
  sdb_prof_end(prof, pi, stream);
  const uint32_t rtiles = static_cast<uint32_t>((bound + SDB_SCAN_TILE - 1) / SDB_SCAN_TILE);
  pi = sdb_prof_begin(prof, SDB_PK_RECV_SCAN, stream);
  k_scan_plan<<<rtiles, 1024, 0, stream>>>(r->plan, r->plan_tops, r->totals);
  k_scan_tops<<<1, 1024, 0, stream>>>(r->plan_tops, rtiles, r->totals + 1);    // totals[1] = payload granules
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += 5;
  if (e != cudaSuccess) return e;
  if (ca) return launch_compact(v, r, ca, nullptr, bound, sm_count, stream, prof, n_launches);
  return launch_gather(v, r, nullptr, bound, max_rec_bytes, sm_count, stream, prof, n_launches);
}

// ------------------------------------------------------------------------------------------
// expiry (sdb_expire): retire the pending records of the listed agents whose header timestamp is < older_than (every
// pending record with SDB_EXPIRE_ALL) as if they had never been enqueued.  8 lanes per request slot, 4 slots per warp:
// the 16-byte ring header once, the window's 8-byte entries coalesced, then one header-timestamp load per live entry
// (arena granule of the handle + 8 bytes: one random 32-byte sector per record, the kernel's whole cost), 4 entries per
// lane in flight.  Matches are tombstoned, the head moves to the first live entry left and ntomb stays exact (the rule of
// select_agent_warp); an agent without a match gets no store at all.  Modes:
//   EXP_DROP    every match; count_out[q] (nullable) and totals[0] += matches (one atomic per warp)
//   EXP_COUNT   cnt[q] = matches, nothing retired (archive mode, before the scan of cnt)
//   EXP_SELECT  capacity cut of k_recv_select on the scanned counts, then the first count_out[q] matches are planned in
//               stream order at their output index {handle, 0, plan z, slot} and retired; the compact back end follows
// With SDB_EXPIRE_ALL, EXP_DROP and EXP_COUNT read no entries: the count is tail - head - ntomb, the ring is emptied.
// ------------------------------------------------------------------------------------------
enum { SDB_EXP_DROP = 0, SDB_EXP_COUNT = 1, SDB_EXP_SELECT = 2 };
#define SDB_EXP_G 8u     // lanes per request slot
#define SDB_EXP_U 4u     // entries per lane in flight

// The parts of a retiring walk that expiry and trimming share.  exp_cut: in EXP_SELECT, the capacity cut of
// k_recv_select on the scanned counts (an agent that does not fit stays queued, unless it is first in the output: then
// its first rec_cap selections); returns how many the slot may retire, RO = its first output record.
template <int MODE>
__device__ __forceinline__ uint32_t exp_cut(const sdb_recv_args& r, bool valid, uint32_t q, uint32_t l8, uint32_t* RO) {
  *RO = 0;
  if (MODE != SDB_EXP_SELECT || !valid) return 0xFFFFFFFFu;
  uint32_t c = r.cnt[q];
  *RO = sdb_scan_at(r.rec_local, r.rec_tops, q);
  if (c && static_cast<uint64_t>(*RO) + c > r.rec_cap) {
    c = *RO == 0 ? static_cast<uint32_t>(r.rec_cap) : 0u;
    if (l8 == 0) atomicMin(r.totals, static_cast<unsigned long long>(*RO) + c);
  }
  if (l8 == 0) r.count_out[q] = c;
  return c;
}

// exp_retire: one step of 8 entries per slot (entry e at ring position pos).  A selected entry is planned at its stream
// rank among the slot's selections {handle, 0, plan z, slot} (EXP_SELECT) and tombstoned; `got` counts the selections and
// `nh` becomes the first live entry not selected (T while there is none), the head by select_agent_warp's rule.
template <int MODE>
__device__ __forceinline__ void exp_retire(const sdb_recv_args& r, uint2* rs, uint32_t mask, uint2 e, uint32_t pos, bool lv,
                                           bool sel, bool retire, uint32_t q, uint32_t RO, uint32_t l8, uint32_t gsh,
                                           uint32_t T, uint32_t& got, uint32_t& nh) {
  const uint32_t bs = (__ballot_sync(0xFFFFFFFFu, sel) >> gsh) & 0xFFu;
  const uint32_t bk = (__ballot_sync(0xFFFFFFFFu, lv && !sel) >> gsh) & 0xFFu;
  if (sel) {
    if (MODE == SDB_EXP_SELECT) r.plan[RO + got + __popc(bs & ((1u << l8) - 1u))] = make_uint4(e.x, 0u, sdb_plan_z(e.y), q);
    if (retire) rs[pos & mask].y = SDB_META_TOMB;
  }
  got += __popc(bs);
  if (bk && nh == T) nh = pos - l8 + (__ffs(bk) - 1);
}

// exp_store: the end of a slot.  The ring header is stored once, and only when something was retired (ntomb stays
// exact); the count goes to cnt (EXP_COUNT) or count_out and the warp's total (EXP_DROP).
template <int MODE>
__device__ __forceinline__ void exp_store(const sdb_dev_view& v, const sdb_recv_args& r, bool valid, bool retire, uint32_t l8,
                                          uint32_t q, uint32_t a, uint32_t H, uint32_t NT, uint32_t got, uint32_t nh,
                                          unsigned long long& wsum) {
  if (l8 != 0 || !valid) return;
  if (retire && got) {
    v.ring_hdr[a].head = nh;
    v.ring_hdr[a].ntomb = NT + got - (nh - H);
  }
  if (MODE == SDB_EXP_COUNT) r.cnt[q] = got;
  if (MODE == SDB_EXP_DROP) { if (r.count_out) r.count_out[q] = got; wsum += got; }
}

template <int MODE>
__device__ __forceinline__ void exp_total(const sdb_recv_args& r, uint32_t lane, unsigned long long wsum) {
  if (MODE != SDB_EXP_DROP) return;
  for (int o = 16; o; o >>= 1) wsum += __shfl_xor_sync(0xFFFFFFFFu, wsum, o);
  if (lane == 0 && wsum) atomicAdd(r.totals, wsum);
}

template <int MODE>
__global__ void __launch_bounds__(256)
k_expire(sdb_dev_view v, sdb_recv_args r, double older_than, uint32_t all) {
  const uint32_t lane = threadIdx.x & 31, l8 = lane & (SDB_EXP_G - 1), gsh = lane & ~(SDB_EXP_G - 1);
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint32_t mask = v.ring_slots - 1;
  const bool retire = MODE != SDB_EXP_COUNT && !(r.flags & SDB_RECV_PEEK);
  constexpr uint32_t SPW = 32u / SDB_EXP_G;                     // request slots per warp
  unsigned long long wsum = 0;
  for (uint32_t qb = gw * SPW; qb < r.n; qb += nw * SPW) {      // warp-uniform
    const uint32_t q = qb + lane / SDB_EXP_G;
    const bool valid = q < r.n;
    uint32_t a = 0, H = 0, T = 0, NT = 0;
    if (valid) {
      a = r.agent_idx ? r.agent_idx[q] : q;
      const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);     // one address for the slot's 8 lanes
      H = h.x; T = h.y; NT = h.w;
    }
    const uint32_t live = T - H - NT;
    uint32_t RO;
    const uint32_t limit = exp_cut<MODE>(r, valid, q, l8, &RO);
    // entries are walked unless ALL makes the count alone enough (a selection always needs the handles)
    const bool walk = valid && live && (MODE == SDB_EXP_SELECT ? limit != 0 : !all);
    const uint32_t W = walk ? T - H : 0u;
    const uint32_t wmax = __reduce_max_sync(0xFFFFFFFFu, W);
    uint32_t got = walk ? 0u : (valid && MODE != SDB_EXP_SELECT ? live : 0u);
    uint32_t nh = walk ? T : (got ? T : H);
    uint2* rs = sdb_ring_of(v, a);
    for (uint32_t j0 = 0; j0 < wmax; j0 += SDB_EXP_G * SDB_EXP_U) {
      uint2 e[SDB_EXP_U];
      double ts[SDB_EXP_U];
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
        const uint32_t j = j0 + u * SDB_EXP_G + l8;
        e[u] = j < W ? rs[(H + j) & mask] : make_uint2(0u, SDB_META_TOMB);
      }
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u)               // independent random loads, all issued before any use
        ts[u] = (!all && sdb_meta(e[u]) != SDB_META_TOMB)
                    ? __ldg(reinterpret_cast<const double*>(v.arena + ((static_cast<uint64_t>(e[u].x) & v.gmask) << 5) + 8))
                    : 0.0;
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
        const uint32_t j = j0 + u * SDB_EXP_G + l8;
        const bool lv = sdb_meta(e[u]) != SDB_META_TOMB;
        const bool match = lv && (all || ts[u] < older_than);           // NaN never compares below: never expires
        const uint32_t bm = (__ballot_sync(0xFFFFFFFFu, match) >> gsh) & 0xFFu;
        const bool sel = match && got + __popc(bm & ((1u << l8) - 1u)) < limit;
        exp_retire<MODE>(r, rs, mask, e[u], H + j, lv, sel, retire, q, RO, l8, gsh, T, got, nh);
      }
    }
    exp_store<MODE>(v, r, valid, retire, l8, q, a, H, NT, got, nh, wsum);
  }
  exp_total<MODE>(r, lane, wsum);
}

// ------------------------------------------------------------------------------------------
// trimming (sdb_trim): retire the records that take an agent's pending queue past max_records records or max_gran
// payload granules (~0: no limit), in eviction order: stream order (NL = 1), or with SDB_RECV_PRIORITY level 0 first,
// then 1, 2, 3, stream order within a level (NL = 4).  k_expire's shape and modes, and no arena reads: the ring meta
// holds the priority (bits 14-15) and the record's granules (1 + payload granules).
//   walk 1  per level: live records L and payload granules G (8-lane reductions).  Skipped when the header decides:
//           stream order without a byte limit has L = tail - head - ntomb; an agent within both limits has no walk 2.
//   walk 2  record i of level p (in-level rank i, in-level granule prefix pg) is retired iff what is left after every
//           record before it in eviction order is gone still breaks a limit: sum_{l>=p} L_l - i > max_records or
//           sum_{l>=p} G_l - pg > max_gran.  Both sides fall along the order, so the retired records are a prefix of it;
//           the eviction rank of a retired record is sum_{l<p} L_l + i, which the capacity cut of EXP_SELECT compares
//           with the slot's limit.  Ranks come from ballots, granule prefixes from 8-lane shuffle scans.
// ------------------------------------------------------------------------------------------
template <int NL>
__device__ __forceinline__ uint32_t trim_pick(const uint32_t (&x)[NL], uint32_t p) {
  uint32_t y = x[0];
#pragma unroll
  for (int l = 1; l < NL; ++l) if (p == static_cast<uint32_t>(l)) y = x[l];
  return y;
}

template <int MODE, int NL>
__global__ void __launch_bounds__(256)
k_trim(sdb_dev_view v, sdb_recv_args r, uint32_t max_records, uint32_t max_gran) {
  const uint32_t lane = threadIdx.x & 31, l8 = lane & (SDB_EXP_G - 1), gsh = lane & ~(SDB_EXP_G - 1);
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint32_t mask = v.ring_slots - 1, below = (1u << l8) - 1u;
  const bool retire = MODE != SDB_EXP_COUNT && !(r.flags & SDB_RECV_PEEK);
  const bool bytes = max_gran != 0xFFFFFFFFu;
  constexpr uint32_t SPW = 32u / SDB_EXP_G;
  unsigned long long wsum = 0;
  for (uint32_t qb = gw * SPW; qb < r.n; qb += nw * SPW) {      // warp-uniform
    const uint32_t q = qb + lane / SDB_EXP_G;
    const bool valid = q < r.n;
    uint32_t a = 0, H = 0, T = 0, NT = 0;
    if (valid) {
      a = r.agent_idx ? r.agent_idx[q] : q;
      const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
      H = h.x; T = h.y; NT = h.w;
    }
    const uint32_t live = T - H - NT;
    uint32_t RO;
    const uint32_t limit = exp_cut<MODE>(r, valid, q, l8, &RO);
    const bool cand = valid && live && limit && (bytes || live > max_records);
    uint2* rs = sdb_ring_of(v, a);
    // 1. totals per level
    uint32_t L[NL], G[NL];
#pragma unroll
    for (int l = 0; l < NL; ++l) { L[l] = 0; G[l] = 0; }
    const uint32_t W1 = cand && (bytes || NL > 1) ? T - H : 0u;
    for (uint32_t j = l8; j < W1; j += SDB_EXP_G) {
      const uint32_t m = sdb_meta(rs[(H + j) & mask]);
      if (m == SDB_META_TOMB) continue;
      const uint32_t p = NL > 1 ? m >> 14 : 0u;
#pragma unroll
      for (int l = 0; l < NL; ++l)
        if (p == static_cast<uint32_t>(l)) { L[l] += 1; G[l] += (m & SDB_META_GLEN_MASK) - 1u; }
    }
#pragma unroll
    for (int l = 0; l < NL; ++l)
#pragma unroll
      for (int o = 4; o; o >>= 1) {
        L[l] += __shfl_xor_sync(0xFFFFFFFFu, L[l], o);
        G[l] += __shfl_xor_sync(0xFFFFFFFFu, G[l], o);
      }
    if (!W1) L[0] = cand ? live : 0u;            // stream order without a byte limit: the header's count
    // suffix sums: what is left of levels >= l, and LL[l] = the records of the levels below l
    uint32_t SL[NL], SG[NL], LL[NL];
    SL[NL - 1] = L[NL - 1]; SG[NL - 1] = G[NL - 1];
#pragma unroll
    for (int l = NL - 2; l >= 0; --l) { SL[l] = SL[l + 1] + L[l]; SG[l] = SG[l + 1] + G[l]; }
#pragma unroll
    for (int l = 0; l < NL; ++l) LL[l] = SL[0] - SL[l];
    // 2. select
    const bool walk = cand && (SL[0] > max_records || SG[0] > max_gran);
    const uint32_t W = walk ? T - H : 0u;
    const uint32_t wmax = __reduce_max_sync(0xFFFFFFFFu, W);
    uint32_t got = 0, nh = walk ? T : H;
    uint32_t ri[NL], rg[NL];                     // records and granules of each level before this step
#pragma unroll
    for (int l = 0; l < NL; ++l) { ri[l] = 0; rg[l] = 0; }
    for (uint32_t j0 = 0; j0 < wmax; j0 += SDB_EXP_G * SDB_EXP_U) {
      uint2 e[SDB_EXP_U];
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
        const uint32_t j = j0 + u * SDB_EXP_G + l8;
        e[u] = j < W ? rs[(H + j) & mask] : make_uint2(0u, SDB_META_TOMB);
      }
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
        const uint32_t m = sdb_meta(e[u]);
        const bool lv = m != SDB_META_TOMB;
        const uint32_t p = NL > 1 ? (m >> 14) & 3u : 0u;
        const uint32_t g = lv ? (m & SDB_META_GLEN_MASK) - 1u : 0u;
        uint32_t i = 0, pg = 0;
#pragma unroll
        for (int l = 0; l < NL; ++l) {
          const bool mine = lv && p == static_cast<uint32_t>(l);
          const uint32_t bl = (__ballot_sync(0xFFFFFFFFu, mine) >> gsh) & 0xFFu;
          uint32_t x = mine ? g : 0u;            // inclusive scan of the level's granules over the slot's 8 lanes
#pragma unroll
          for (uint32_t o = 1; o < SDB_EXP_G; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o, SDB_EXP_G);
            if (l8 >= o) x += y;
          }
          if (mine) { i = ri[l] + __popc(bl & below); pg = rg[l] + x - g; }
          ri[l] += __popc(bl);
          rg[l] += __shfl_sync(0xFFFFFFFFu, x, SDB_EXP_G - 1, SDB_EXP_G);
        }
        const bool drop = lv && (trim_pick<NL>(SL, p) - i > max_records || trim_pick<NL>(SG, p) - pg > max_gran);
        const bool sel = drop && trim_pick<NL>(LL, p) + i < limit;
        exp_retire<MODE>(r, rs, mask, e[u], H + j0 + u * SDB_EXP_G + l8, lv, sel, retire, q, RO, l8, gsh, T, got, nh);
      }
    }
    exp_store<MODE>(v, r, valid, retire, l8, q, a, H, NT, got, nh, wsum);
  }
  exp_total<MODE>(r, lane, wsum);
}

// One mode of expiry, or of trimming when trim != nullptr ({max_records, max_gran}, ~0: no limit; r->flags picks the
// eviction order).
template <int MODE>
static void launch_retire(const sdb_dev_view* v, const sdb_recv_args* r, double older_than, uint32_t all, const uint2* trim,
                          uint32_t blocks, cudaStream_t stream) {
  if (!trim)
    k_expire<MODE><<<blocks, 256, 0, stream>>>(*v, *r, older_than, all);
  else if (r->flags & SDB_RECV_PRIORITY)
    k_trim<MODE, 4><<<blocks, 256, 0, stream>>>(*v, *r, trim->x, trim->y);
  else
    k_trim<MODE, 1><<<blocks, 256, 0, stream>>>(*v, *r, trim->x, trim->y);
}

// drop mode (ca == nullptr): one launch; totals[0] = records retired.  Archive mode: count, scan, select, then the compact
// back end exactly as a compact receive runs it (totals as there).
extern "C" cudaError_t sdb_launch_expire(const sdb_dev_view* v, const sdb_recv_args* r, double older_than, uint32_t all,
                                         const uint2* trim, const sdb_compact_args* ca, cudaStream_t stream, int* n_launches,
                                         sdb_profiler* prof, int sm_count) {
  if (r->n == 0) return cudaSuccess;
  const uint32_t n = r->n;
  const uint32_t blocks = sdb_grid(n, 32, 32 * sm_count);                    // 4 slots per warp, 8 warps per block
  const int pi = sdb_prof_begin(prof, SDB_PK_EXPIRE, stream);
  if (!ca) {
    cudaMemsetAsync(r->totals, 0, sizeof(unsigned long long), stream);
    launch_retire<SDB_EXP_DROP>(v, r, older_than, all, trim, blocks, stream);
    sdb_prof_end(prof, pi, stream);
    if (n_launches) *n_launches += 1;
    return cudaGetLastError();
  }
  launch_retire<SDB_EXP_COUNT>(v, r, older_than, all, trim, blocks, stream);
  // totals[0] = matches; the cut may lower it
  const cudaError_t e = sdb_scan_u32(r->cnt, r->rec_local, r->rec_tops, n, r->totals, nullptr, stream, n_launches);
  launch_retire<SDB_EXP_SELECT>(v, r, older_than, all, trim, blocks, stream);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += 2;
  if (e != cudaSuccess) return e;
  uint64_t bound = static_cast<uint64_t>(n) * v->ring_slots;               // upper bound on the records planned
  if (bound > r->rec_cap) bound = r->rec_cap;
  return launch_compact(v, r, ca, nullptr, bound, sm_count, stream, prof, n_launches);
}

// ------------------------------------------------------------------------------------------
// superseding (sdb_supersede): of the pending records carrying SDB_TYPEF_SUPERSEDE, keep per key (agent, sender, group,
// type & SDB_TYPE_MASK) the one with the largest seq, the later in the ring on a tie, and retire the others.  The flag is
// in the header (byte 31), not in the ring meta, so the cost is the header reads, at most two per live record:
//   k_supersede_count    k_expire's shape: cnt[q] = flagged live records (the header's last word); scan -> C
//   (the host stops when C = 0, else sizes the table and the candidate array for C records)
//   k_supersede_insert   the same walk: each flagged record's {seq, slot, ring offset, table slot} goes to cand[] at its
//                        scanned position, its key into the table (128-bit CAS, linear probing), atomicMax of its seq;
//                        the verdict words of walked slots are zeroed
//   k_supersede_tie      per candidate: holders of the key's largest seq atomicMax their ring offset
//   k_supersede_verdict  per candidate: superseded unless it is the key's {seq, offset}; the bit of its ring slot is
//                        set (k_where_eval's bitmap) and cnt[q] counts it (one atomic per warp and slot)
//   k_supersede<MODE>    k_expire's retire walk over ring entries and verdict words only: EXP_DROP, or after a scan of
//                        cnt EXP_SELECT with its capacity cut, then the compact back end
// Every record of a key but its newest is superseded, so any subset of them may go: the capacity cut is safe.
// ------------------------------------------------------------------------------------------
struct __align__(16) ss_key { unsigned long long lo, hi; };

__device__ __forceinline__ uint32_t ss_hash(unsigned long long lo, unsigned long long hi) {
  unsigned long long k = lo ^ (hi * 0x9E3779B97F4A7C15ull);
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return static_cast<uint32_t>(k);
}

__device__ __forceinline__ bool ss_flagged(uint32_t w7) { return ((w7 >> 24) & SDB_TYPEF_SUPERSEDE) != 0u; }

__global__ void __launch_bounds__(256)
k_supersede_count(sdb_dev_view v, sdb_recv_args r) {
  const uint32_t lane = threadIdx.x & 31, l8 = lane & (SDB_EXP_G - 1), gsh = lane & ~(SDB_EXP_G - 1);
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint32_t mask = v.ring_slots - 1;
  constexpr uint32_t SPW = 32u / SDB_EXP_G;
  for (uint32_t qb = gw * SPW; qb < r.n; qb += nw * SPW) {      // warp-uniform
    const uint32_t q = qb + lane / SDB_EXP_G;
    const bool valid = q < r.n;
    uint32_t a = 0, H = 0, T = 0, NT = 0;
    if (valid) {
      a = r.agent_idx ? r.agent_idx[q] : q;
      const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
      H = h.x; T = h.y; NT = h.w;
    }
    const uint32_t W = (valid && T - H - NT) ? T - H : 0u;
    const uint32_t wmax = __reduce_max_sync(0xFFFFFFFFu, W);
    const uint2* rs = sdb_ring_of(v, a);
    uint32_t got = 0;
    for (uint32_t j0 = 0; j0 < wmax; j0 += SDB_EXP_G * SDB_EXP_U) {
      uint2 e[SDB_EXP_U];
      uint32_t w7[SDB_EXP_U];
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
        const uint32_t j = j0 + u * SDB_EXP_G + l8;
        e[u] = j < W ? rs[(H + j) & mask] : make_uint2(0u, SDB_META_TOMB);
      }
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u)               // len | prio << 16 | type << 24, one random sector each
        w7[u] = sdb_meta(e[u]) != SDB_META_TOMB
                    ? __ldg(reinterpret_cast<const uint32_t*>(v.arena + ((static_cast<uint64_t>(e[u].x) & v.gmask) << 5)) + 7)
                    : 0u;
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u)
        got += __popc((__ballot_sync(0xFFFFFFFFu, ss_flagged(w7[u])) >> gsh) & 0xFFu);
    }
    if (l8 == 0 && valid) r.cnt[q] = got;
  }
}

__global__ void __launch_bounds__(256)
k_supersede_insert(sdb_dev_view v, sdb_recv_args r, sdb_ss_args s) {
  const uint32_t lane = threadIdx.x & 31, l8 = lane & (SDB_EXP_G - 1), gsh = lane & ~(SDB_EXP_G - 1);
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint32_t mask = v.ring_slots - 1;
  constexpr uint32_t SPW = 32u / SDB_EXP_G;
  for (uint32_t qb = gw * SPW; qb < r.n; qb += nw * SPW) {      // warp-uniform
    const uint32_t q = qb + lane / SDB_EXP_G;
    const bool valid = q < r.n;
    uint32_t a = 0, H = 0, T = 0, c = 0, base = 0;
    if (valid) {
      a = r.agent_idx ? r.agent_idx[q] : q;
      c = r.cnt[q];
      if (c) {
        const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
        H = h.x; T = h.y;
        base = sdb_scan_at(r.rec_local, r.rec_tops, q);
      }
    }
    const uint32_t W = c ? T - H : 0u;
    const uint32_t wmax = __reduce_max_sync(0xFFFFFFFFu, W);
    const uint2* rs = sdb_ring_of(v, a);
    uint32_t* bits = s.bits + static_cast<size_t>(a) * s.stride;
    uint32_t got = 0;
    for (uint32_t j0 = 0; j0 < wmax; j0 += SDB_EXP_G * SDB_EXP_U) {
      uint2 e[SDB_EXP_U];
      uint4 lo[SDB_EXP_U], hi[SDB_EXP_U];
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
        const uint32_t j = j0 + u * SDB_EXP_G + l8;
        e[u] = j < W ? rs[(H + j) & mask] : make_uint2(0u, SDB_META_TOMB);
      }
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {              // independent random loads, all issued before any use
        lo[u] = hi[u] = make_uint4(0u, 0u, 0u, 0u);
        if (sdb_meta(e[u]) != SDB_META_TOMB) {
          const uint4* src = reinterpret_cast<const uint4*>(v.arena + ((static_cast<uint64_t>(e[u].x) & v.gmask) << 5));
          lo[u] = __ldg(src); hi[u] = __ldg(src + 1);
        }
      }
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
        const bool fl = ss_flagged(hi[u].w);
        const uint32_t bm = (__ballot_sync(0xFFFFFFFFu, fl) >> gsh) & 0xFFu;
        if (fl) {
          const unsigned long long seq = (static_cast<unsigned long long>(lo[u].y) << 32) | lo[u].x;
          const ss_key k{a | (static_cast<unsigned long long>(hi[u].x) << 32),
                         hi[u].z | (static_cast<unsigned long long>((hi[u].w >> 24) & SDB_TYPE_MASK) << 32) | (1ull << 63)};
          uint32_t t = ss_hash(k.lo, k.hi) & s.mask;
          for (;; t = (t + 1) & s.mask) {
            const ss_key old = atomicCAS(reinterpret_cast<ss_key*>(s.tab + t), ss_key{0ull, 0ull}, k);
            if ((old.lo == 0ull && old.hi == 0ull) || (old.lo == k.lo && old.hi == k.hi)) break;
          }
          atomicMax(&s.tab[t].seq, seq);
          s.cand[base + got + __popc(bm & ((1u << l8) - 1u))] = sdb_ss_cand{seq, q, j0 + u * SDB_EXP_G + l8, t, 0u};
        }
        got += __popc(bm);
      }
      if (l8 == 0 && j0 < W) bits[j0 >> 5] = 0u;
    }
  }
}

__global__ void __launch_bounds__(256)
k_supersede_tie(sdb_ss_args s) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= s.n_cand) return;
  const sdb_ss_cand c = s.cand[i];
  if (c.seq == s.tab[c.slot].seq) atomicMax(&s.tab[c.slot].off, c.j);
}

__global__ void __launch_bounds__(256)
k_supersede_verdict(sdb_recv_args r, sdb_ss_args s) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
  bool sup = false;
  uint32_t q = 0xFFFFFFFFu;
  if (i < s.n_cand) {                                         // no early return: the warp meets in the aggregation
    const sdb_ss_cand c = s.cand[i];
    const sdb_ss_slot t = s.tab[c.slot];
    sup = !(c.seq == t.seq && c.j == t.off);
    q = c.q;
    if (sup) {
      const uint32_t a = r.agent_idx ? r.agent_idx[q] : q;
      atomicOr(s.bits + static_cast<size_t>(a) * s.stride + (c.j >> 5), 1u << (c.j & 31u));
    }
  }
  const uint32_t b = __ballot_sync(0xFFFFFFFFu, sup) & __match_any_sync(0xFFFFFFFFu, q);
  if (sup && lane == static_cast<uint32_t>(__ffs(b) - 1)) atomicAdd(r.cnt + q, static_cast<uint32_t>(__popc(b)));
}

template <int MODE>
__global__ void __launch_bounds__(256)
k_supersede(sdb_dev_view v, sdb_recv_args r, sdb_ss_args s) {
  const uint32_t lane = threadIdx.x & 31, l8 = lane & (SDB_EXP_G - 1), gsh = lane & ~(SDB_EXP_G - 1);
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint32_t mask = v.ring_slots - 1;
  const bool retire = !(r.flags & SDB_RECV_PEEK);
  constexpr uint32_t SPW = 32u / SDB_EXP_G;
  unsigned long long wsum = 0;
  for (uint32_t qb = gw * SPW; qb < r.n; qb += nw * SPW) {      // warp-uniform
    const uint32_t q = qb + lane / SDB_EXP_G;
    const bool valid = q < r.n;
    uint32_t RO;
    const uint32_t limit = exp_cut<MODE>(r, valid, q, l8, &RO);
    const bool walk = valid && (MODE == SDB_EXP_SELECT ? limit : r.cnt[q]) != 0u;
    uint32_t a = 0, H = 0, T = 0, NT = 0;
    if (valid) {
      a = r.agent_idx ? r.agent_idx[q] : q;
      const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
      H = h.x; T = h.y; NT = h.w;
    }
    const uint32_t W = walk ? T - H : 0u;
    const uint32_t wmax = __reduce_max_sync(0xFFFFFFFFu, W);
    uint32_t got = 0, nh = walk ? T : H;
    uint2* rs = sdb_ring_of(v, a);
    const uint32_t* bits = s.bits + static_cast<size_t>(a) * s.stride;
    for (uint32_t j0 = 0; j0 < wmax; j0 += SDB_EXP_G * SDB_EXP_U) {
      const uint32_t word = j0 < W ? bits[j0 >> 5] : 0u;
      uint2 e[SDB_EXP_U];
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
        const uint32_t j = j0 + u * SDB_EXP_G + l8;
        e[u] = j < W ? rs[(H + j) & mask] : make_uint2(0u, SDB_META_TOMB);
      }
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
        const bool lv = sdb_meta(e[u]) != SDB_META_TOMB;
        const bool match = lv && ((word >> (u * SDB_EXP_G + l8)) & 1u);
        const uint32_t bm = (__ballot_sync(0xFFFFFFFFu, match) >> gsh) & 0xFFu;
        const bool sel = match && got + __popc(bm & ((1u << l8) - 1u)) < limit;
        exp_retire<MODE>(r, rs, mask, e[u], H + j0 + u * SDB_EXP_G + l8, lv, sel, retire, q, RO, l8, gsh, T, got, nh);
      }
    }
    exp_store<MODE>(v, r, valid, retire, l8, q, a, H, NT, got, nh, wsum);
  }
  exp_total<MODE>(r, lane, wsum);
}

// s->tab == nullptr: k_supersede_count and the scan, totals[0] = flagged records C.  Otherwise, with the table and the
// candidate array sized for s->n_cand = C records: insert, tie, verdict, then drop mode (ca == nullptr, totals[0] =
// records retired) or the select walk and the compact back end exactly as a compact receive runs it (totals as there).
extern "C" cudaError_t sdb_launch_supersede(const sdb_dev_view* v, const sdb_recv_args* r, const sdb_ss_args* s,
                                            const sdb_compact_args* ca, cudaStream_t stream, int* n_launches, sdb_profiler* prof,
                                            int sm_count) {
  if (r->n == 0) return cudaSuccess;
  const uint32_t n = r->n;
  const uint32_t blocks = sdb_grid(n, 32, 32 * sm_count);                    // 4 slots per warp, 8 warps per block
  const int pi = sdb_prof_begin(prof, SDB_PK_EXPIRE, stream);
  if (!s->tab) {
    k_supersede_count<<<blocks, 256, 0, stream>>>(*v, *r);
    const cudaError_t e = sdb_scan_u32(r->cnt, r->rec_local, r->rec_tops, n, r->totals, nullptr, stream, n_launches);
    sdb_prof_end(prof, pi, stream);
    if (n_launches) *n_launches += 1;
    return e != cudaSuccess ? e : cudaGetLastError();
  }
  const uint32_t cblocks = (s->n_cand + 255u) / 256u;
  k_supersede_insert<<<blocks, 256, 0, stream>>>(*v, *r, *s);
  cudaMemsetAsync(r->cnt, 0, static_cast<size_t>(n) * sizeof(uint32_t), stream);   // cnt[q] = superseded records
  k_supersede_tie<<<cblocks, 256, 0, stream>>>(*s);
  k_supersede_verdict<<<cblocks, 256, 0, stream>>>(*r, *s);
  if (!ca) {
    cudaMemsetAsync(r->totals, 0, sizeof(unsigned long long), stream);
    k_supersede<SDB_EXP_DROP><<<blocks, 256, 0, stream>>>(*v, *r, *s);
    sdb_prof_end(prof, pi, stream);
    if (n_launches) *n_launches += 4;
    return cudaGetLastError();
  }
  // totals[0] = superseded records; the cut may lower it
  const cudaError_t e = sdb_scan_u32(r->cnt, r->rec_local, r->rec_tops, n, r->totals, nullptr, stream, n_launches);
  k_supersede<SDB_EXP_SELECT><<<blocks, 256, 0, stream>>>(*v, *r, *s);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += 4;
  if (e != cudaSuccess) return e;
  const uint64_t bound = s->n_cand < r->rec_cap ? s->n_cand : r->rec_cap;   // upper bound on the records planned
  return launch_compact(v, r, ca, nullptr, bound, sm_count, stream, prof, n_launches);
}

// ------------------------------------------------------------------------------------------
// filtered receive (sdb_receive_where): the predicate is evaluated once per pending record and kept as one verdict bit
// per ring slot (f.bits, agent a, offset j from the head); the selection then reads bits and ring entries only.
//   k_where_eval    header clauses only, k_expire's shape: 8 lanes per request slot, the ring header once, the window's
//                   entries coalesced, the 32-byte header sector of every live entry with 4 loads per lane in flight
//   k_where_kw      with a keyword: one warp per request slot, a lane per entry for the header clauses, then every
//                   record that passes gets a warp-cooperative substring search of its content bytes
//   both            write the verdict words and cnt[q] = min(matches, max_messages); with SDB_FILTER_IDS the seq of every
//                   record that passes the other header clauses is probed in the id table (k_id_table), and with
//                   per-id outputs every final match adds to its slot, once per warp and slot (k_id_out reads them out)
//   scan            sdb_scan_u32 over cnt (take mode)
//   k_where_select  capacity cut of k_recv_select, then the first count_out[q] set bits in delivery order (priority
//                   order: one walk per level 3..0 over the entries' meta) are planned {handle, -, plan z, slot} and
//                   tombstoned; head / ntomb by select_agent_warp's rule, the ring header stored at most once.  Take
//                   mode adds to `delivered` with one atomic per warp; drop mode adds to totals[0] instead and stops
//   back end        k_scan_plan + k_scan_tops, then the receive gather unchanged
// ------------------------------------------------------------------------------------------
#define SDB_WHERE_HDR_FIELDS (SDB_FILTER_SENDER | SDB_FILTER_RECEIVER | SDB_FILTER_GROUP | SDB_FILTER_TYPE | SDB_FILTER_PRIO | \
                              SDB_FILTER_TIME | SDB_FILTER_SEQ | SDB_FILTER_IDS)
#define SDB_WHERE_STAGE 1024u     // content bytes staged per warp and step of the keyword search
#define SDB_ID_NONE 0xFFFFFFFFu   // "no slot": the record is not a match of the id clause

// id table of SDB_FILTER_IDS: linear probing from a 64-bit mix of the seq (sequence numbers are dense, so the low bits
// alone would fill runs of neighbouring slots).  At most half the slots are used, so a probe ends at an empty slot.
__device__ __forceinline__ uint32_t id_hash(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return static_cast<uint32_t>(k);
}
// the slot holding key s, or SDB_ID_NONE
__device__ __forceinline__ uint32_t id_find(const sdb_id_slot* tab, uint32_t mask, unsigned long long s) {
  if (s == 0) return SDB_ID_NONE;
  for (uint32_t i = id_hash(s) & mask;; i = (i + 1) & mask) {
    const unsigned long long k = __ldg(&tab[i].key);
    if (k == s) return i;
    if (k == 0) return SDB_ID_NONE;
  }
}

// one kernel inserts every id with a 64-bit CAS; duplicates meet in one slot, id 0 (never a seq) is left out
__global__ void __launch_bounds__(256)
k_id_table(const unsigned long long* ids, uint32_t n, sdb_id_slot* tab, uint32_t mask) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n || ids[t] == 0) return;
  const unsigned long long s = ids[t];
  for (uint32_t i = id_hash(s) & mask;; i = (i + 1) & mask) {
    const unsigned long long k = atomicCAS(&tab[i].key, 0ull, s);
    if (k == 0 || k == s) return;
  }
}

// the slots' values in input order: out[0, n) hits, out[n, 2n) first agent
__global__ void __launch_bounds__(256)
k_id_out(const unsigned long long* ids, uint32_t n, const sdb_id_slot* tab, uint32_t mask, uint32_t* out) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const uint32_t i = id_find(tab, mask, ids[t]);
  out[t] = i == SDB_ID_NONE ? 0u : tab[i].hits;
  out[n + t] = i == SDB_ID_NONE ? SDB_NO_RECEIVER : ~tab[i].nagent;
}

// a match of agent a in id slot `slot` (SDB_ID_NONE: no match); whole warp.  The lanes that hit one slot add once: a
// broadcast queued at every agent sends all its hits to one slot.
__device__ __forceinline__ void where_count_id(const sdb_where_args& f, uint32_t slot, uint32_t a) {
  const uint32_t grp = __match_any_sync(0xFFFFFFFFu, slot);
  if (slot == SDB_ID_NONE) return;
  const uint32_t na = __reduce_max_sync(grp, ~a);
  if ((threadIdx.x & 31) == static_cast<uint32_t>(__ffs(grp) - 1)) {
    atomicAdd(&f.id_tab[slot].hits, static_cast<uint32_t>(__popc(grp)));
    atomicMax(&f.id_tab[slot].nagent, na);
  }
}

// lo = {seq lo, seq hi, timestamp lo, timestamp hi}, hi = {sender, receiver, group, len | prio << 16 | type << 24};
// *slot: the record's id-table slot when the id clause was tested (left alone otherwise)
__device__ __forceinline__ bool where_header(const sdb_where_args& f, const uint4& lo, const uint4& hi, uint32_t* slot) {
  const uint32_t fl = f.fields;
  bool ok = true;
  if (fl & SDB_FILTER_SENDER) ok = ok && hi.x == f.sender;
  if (fl & SDB_FILTER_RECEIVER) ok = ok && hi.y == f.receiver;
  if (fl & SDB_FILTER_GROUP) ok = ok && hi.z == f.group;
  if (fl & SDB_FILTER_TYPE) ok = ok && ((f.type_mask >> ((hi.w >> 24) & SDB_TYPE_MASK)) & 1u);
  if (fl & SDB_FILTER_PRIO) { const uint32_t p = (hi.w >> 16) & 0xFFu; ok = ok && p < 8u && ((f.prio_mask >> p) & 1u); }
  if (fl & SDB_FILTER_TIME) {
    const double ts = __hiloint2double(static_cast<int>(lo.w), static_cast<int>(lo.z));
    ok = ok && ts > f.after && ts < f.before;                 // strict: a NaN never matches
  }
  if (fl & SDB_FILTER_SEQ) {
    const unsigned long long s = (static_cast<unsigned long long>(lo.y) << 32) | lo.x;
    ok = ok && s >= f.seq_lo && s < f.seq_hi;
  }
  if ((fl & SDB_FILTER_IDS) && ok) {                          // last: one probe only for records every other clause passed
    *slot = id_find(f.id_tab, f.id_mask, (static_cast<unsigned long long>(lo.y) << 32) | lo.x);
    ok = *slot != SDB_ID_NONE;
  }
  return ok;
}

__device__ __forceinline__ uint32_t where_fold(uint32_t c, bool icase) { return (icase && c - 65u < 26u) ? c + 32u : c; }

__global__ void __launch_bounds__(256)
k_where_eval(sdb_dev_view v, sdb_recv_args r, sdb_where_args f) {
  const uint32_t lane = threadIdx.x & 31, l8 = lane & (SDB_EXP_G - 1), gsh = lane & ~(SDB_EXP_G - 1);
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint32_t mask = v.ring_slots - 1;
  const bool need_hdr = (f.fields & SDB_WHERE_HDR_FIELDS) != 0;
  constexpr uint32_t SPW = 32u / SDB_EXP_G;
  for (uint32_t qb = gw * SPW; qb < r.n; qb += nw * SPW) {      // warp-uniform
    const uint32_t q = qb + lane / SDB_EXP_G;
    const bool valid = q < r.n;
    uint32_t a = 0, H = 0, T = 0, NT = 0;
    if (valid) {
      a = r.agent_idx ? r.agent_idx[q] : q;
      const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
      H = h.x; T = h.y; NT = h.w;
    }
    const uint32_t W = (valid && T - H - NT) ? T - H : 0u;
    const uint32_t wmax = __reduce_max_sync(0xFFFFFFFFu, W);
    const uint2* rs = sdb_ring_of(v, a);
    uint32_t* bits = f.bits + static_cast<size_t>(a) * f.stride;
    uint32_t got = 0;
    for (uint32_t j0 = 0; j0 < wmax; j0 += SDB_EXP_G * SDB_EXP_U) {
      uint2 e[SDB_EXP_U];
      uint4 lo[SDB_EXP_U], hi[SDB_EXP_U];
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
        const uint32_t j = j0 + u * SDB_EXP_G + l8;
        e[u] = j < W ? rs[(H + j) & mask] : make_uint2(0u, SDB_META_TOMB);
      }
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {              // independent random loads, all issued before any use
        lo[u] = hi[u] = make_uint4(0u, 0u, 0u, 0u);
        if (need_hdr && sdb_meta(e[u]) != SDB_META_TOMB) {
          const uint4* src = reinterpret_cast<const uint4*>(v.arena + ((static_cast<uint64_t>(e[u].x) & v.gmask) << 5));
          lo[u] = __ldg(src); hi[u] = __ldg(src + 1);
        }
      }
      uint32_t word = 0;
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
        uint32_t slot = SDB_ID_NONE;
        const bool match = sdb_meta(e[u]) != SDB_META_TOMB && (!need_hdr || where_header(f, lo[u], hi[u], &slot));
        word |= ((__ballot_sync(0xFFFFFFFFu, match) >> gsh) & 0xFFu) << (u * SDB_EXP_G);
        if (f.id_count) where_count_id(f, match ? slot : SDB_ID_NONE, a);
      }
      if (l8 == 0 && j0 < W) bits[j0 >> 5] = word;
      got += __popc(word);
    }
    if (l8 == 0 && valid) r.cnt[q] = min(got, r.max_messages);
  }
}

// does kw[0, K) (folded) occur in the bytes [cs, ce) of the padded payload p[0, plen)?  Whole warp; the content is staged
// through `buf` in chunks that overlap by K - 1 bytes, 16-byte loads; lanes test start positions, first byte first.
__device__ __forceinline__ bool where_find(const uint8_t* p, uint32_t plen, uint32_t cs, uint32_t ce, const uint8_t* kw,
                                           uint32_t K, bool icase, uint8_t* buf, uint32_t lane) {
  if (ce < cs + K) return false;
  const uint32_t last = ce - K;                               // last start position
  const uint32_t k0 = kw[0];
  uint32_t s = cs;                                            // first start position not tested yet
  for (;;) {
    const uint32_t c0 = s & ~15u;                             // staged: payload bytes [c0, min(c0 + STAGE, plen))
    const uint32_t end = min(c0 + SDB_WHERE_STAGE, plen);
    __syncwarp();
    for (uint32_t b = lane << 4; c0 + b < end; b += 512)
      *reinterpret_cast<uint4*>(buf + b) = __ldg(reinterpret_cast<const uint4*>(p + c0 + b));
    __syncwarp();
    const uint32_t hi = min(last, c0 + SDB_WHERE_STAGE - K);  // last start whose K bytes are staged
    for (uint32_t t0 = s; t0 <= hi; t0 += 32) {               // warp-uniform
      const uint32_t t = t0 + lane;
      bool hit = false;
      if (t <= hi) {
        const uint8_t* x = buf + (t - c0);
        if (where_fold(x[0], icase) == k0) {
          uint32_t i = 1;
          while (i < K && where_fold(x[i], icase) == kw[i]) ++i;
          hit = i == K;
        }
      }
      if (__any_sync(0xFFFFFFFFu, hit)) return true;
    }
    if (hi >= last) return false;
    s = hi + 1;
  }
}

__global__ void __launch_bounds__(256)
k_where_kw(sdb_dev_view v, sdb_recv_args r, sdb_where_args f) {
  __shared__ uint8_t s_kw[SDB_FILTER_MAX_KEYWORD];
  __shared__ __align__(16) uint8_t s_buf[8][SDB_WHERE_STAGE];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint32_t mask = v.ring_slots - 1, K = f.kw_len;
  const bool icase = (f.fields & SDB_FILTER_ICASE) != 0;
  for (uint32_t i = threadIdx.x; i < K; i += blockDim.x) s_kw[i] = static_cast<uint8_t>(where_fold(f.kw[i], icase));
  __syncthreads();
  for (uint32_t q = gw; q < r.n; q += nw) {                   // warp-uniform: one request slot per warp
    const uint32_t a = r.agent_idx ? r.agent_idx[q] : q;
    const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
    const uint32_t H = h.x, T = h.y, NT = h.w;
    const uint32_t W = T - H - NT ? T - H : 0u;
    const uint2* rs = sdb_ring_of(v, a);
    uint32_t* bits = f.bits + static_cast<size_t>(a) * f.stride;
    uint32_t got = 0;
    for (uint32_t j0 = 0; j0 < W; j0 += 32) {
      const uint32_t j = j0 + lane;
      const uint2 e = j < W ? rs[(H + j) & mask] : make_uint2(0u, SDB_META_TOMB);
      const bool lv = sdb_meta(e) != SDB_META_TOMB;
      uint4 lo = make_uint4(0u, 0u, 0u, 0u), hi = lo;
      if (lv) {
        const uint4* src = reinterpret_cast<const uint4*>(v.arena + ((static_cast<uint64_t>(e.x) & v.gmask) << 5));
        lo = __ldg(src); hi = __ldg(src + 1);
      }
      uint32_t slot = SDB_ID_NONE;
      uint32_t word = __ballot_sync(0xFFFFFFFFu, lv && where_header(f, lo, hi, &slot));
      for (uint32_t c = word; c; c &= c - 1) {
        const uint32_t src = __ffs(c) - 1;
        const uint32_t hx = __shfl_sync(0xFFFFFFFFu, e.x, src), hy = __shfl_sync(0xFFFFFFFFu, e.y, src);
        const uint32_t hw = __shfl_sync(0xFFFFFFFFu, hi.w, src);
        const uint32_t len = hw & 0xFFFFu;
        const uint8_t* p = sdb_payload_of(v, hx, sdb_entry_dm1(hy));      // shared-layout images: handle + 1 + dm1
        const uint32_t c0 = ((hw >> 24) & SDB_TYPEF_TOKENS) ? 4u : 0u;    // u32 token count first
        uint32_t cs = c0, ce = len;
        if ((hw >> 24) & SDB_TYPEF_EXTRAS) {                               // u32 content length | content | extras
          cs = c0 + 4u;
          ce = len < cs ? cs : cs + min(__ldg(reinterpret_cast<const uint32_t*>(p + c0)), len - cs);
        }
        if (!where_find(p, (len + 31u) & ~31u, cs, ce, s_kw, K, icase, s_buf[warp], lane)) word &= ~(1u << src);
      }
      if (f.id_count) where_count_id(f, ((word >> lane) & 1u) ? slot : SDB_ID_NONE, a);
      if (lane == 0) bits[j0 >> 5] = word;
      got += __popc(word);
    }
    if (lane == 0) r.cnt[q] = min(got, r.max_messages);
  }
}

template <bool PLAN>
__global__ void __launch_bounds__(256)
k_where_select(sdb_dev_view v, sdb_recv_args r, sdb_where_args f) {
  const uint32_t lane = threadIdx.x & 31, l8 = lane & (SDB_EXP_G - 1), gsh = lane & ~(SDB_EXP_G - 1);
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint32_t mask = v.ring_slots - 1;
  const bool retire = !(r.flags & SDB_RECV_PEEK);
  const int top = (r.flags & SDB_RECV_PRIORITY) ? 3 : -1;      // -1: one walk, every level (stream order)
  constexpr uint32_t SPW = 32u / SDB_EXP_G;
  unsigned long long wsum = 0;
  for (uint32_t qb = gw * SPW; qb < r.n; qb += nw * SPW) {      // warp-uniform
    const uint32_t q = qb + lane / SDB_EXP_G;
    const bool valid = q < r.n;
    uint32_t a = 0, H = 0, T = 0, NT = 0, c = 0, RO = 0;
    if (valid) {
      a = r.agent_idx ? r.agent_idx[q] : q;
      c = r.cnt[q];
      if (PLAN) {
        RO = sdb_scan_at(r.rec_local, r.rec_tops, q);
        if (c && static_cast<uint64_t>(RO) + c > r.rec_cap) {   // does not fit: stays queued ...
          c = RO == 0 ? static_cast<uint32_t>(r.rec_cap) : 0u;  // ... unless first in the output: its first rec_cap matches
          if (l8 == 0) atomicMin(r.totals, static_cast<unsigned long long>(RO) + c);
        }
      }
      if (l8 == 0) r.count_out[q] = c;
      if (c) {
        const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
        H = h.x; T = h.y; NT = h.w;
      }
    }
    const uint32_t W = c ? T - H : 0u;
    const uint32_t wmax = __reduce_max_sync(0xFFFFFFFFu, W);
    uint2* rs = sdb_ring_of(v, a);
    const uint32_t* bits = f.bits + static_cast<size_t>(a) * f.stride;
    uint32_t seen = 0;                                          // matches met so far in delivery order
    for (int L = top;; --L) {
      for (uint32_t j0 = 0; j0 < wmax; j0 += SDB_EXP_G * SDB_EXP_U) {
        if (__all_sync(0xFFFFFFFFu, seen >= c)) break;
        const uint32_t word = (j0 < W && seen < c) ? bits[j0 >> 5] : 0u;
        uint2 e[SDB_EXP_U];
#pragma unroll
        for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
          const uint32_t j = j0 + u * SDB_EXP_G + l8;
          e[u] = ((word >> (u * SDB_EXP_G + l8)) & 1u) ? rs[(H + j) & mask] : make_uint2(0u, SDB_META_TOMB);
        }
#pragma unroll
        for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
          const uint32_t m = sdb_meta(e[u]);
          const bool match = m != SDB_META_TOMB && (L < 0 || (m >> 14) == static_cast<uint32_t>(L));
          const uint32_t bm = (__ballot_sync(0xFFFFFFFFu, match) >> gsh) & 0xFFu;
          const uint32_t k = seen + __popc(bm & ((1u << l8) - 1u));
          if (match && k < c) {
            if (PLAN) r.plan[RO + k] = make_uint4(e[u].x, 0u, sdb_plan_z(e[u].y), q);
            if (retire) rs[(H + j0 + u * SDB_EXP_G + l8) & mask].y = SDB_META_TOMB;
          }
          seen += __popc(bm);
        }
      }
      if (L <= 0) break;
    }
    // new head: the first live entry left (each lane re-reads only the slots it may have tombstoned itself)
    const uint32_t took = min(seen, c);
    const bool fix = retire && took;
    const uint32_t W2 = fix ? W : 0u;
    const uint32_t wmax2 = __reduce_max_sync(0xFFFFFFFFu, W2);
    uint32_t nh = T;
    bool found = false;
    for (uint32_t j0 = 0; j0 < wmax2; j0 += SDB_EXP_G * SDB_EXP_U) {
      if (__all_sync(0xFFFFFFFFu, !fix || found)) break;
      uint32_t m[SDB_EXP_U];
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
        const uint32_t j = j0 + u * SDB_EXP_G + l8;
        m[u] = (j < W2 && !found) ? sdb_meta(rs[(H + j) & mask]) : SDB_META_TOMB;
      }
#pragma unroll
      for (uint32_t u = 0; u < SDB_EXP_U; ++u) {
        const uint32_t b = (__ballot_sync(0xFFFFFFFFu, m[u] != SDB_META_TOMB) >> gsh) & 0xFFu;
        if (b && !found) { nh = H + j0 + u * SDB_EXP_G + (__ffs(b) - 1); found = true; }
      }
    }
    if (l8 == 0 && valid) {
      if (fix) {                                                // the ring header, once
        v.ring_hdr[a].head = nh;
        v.ring_hdr[a].ntomb = NT + took - (nh - H);
      }
      if (!PLAN || retire) wsum += took;
    }
  }
  for (int o = 16; o; o >>= 1) wsum += __shfl_xor_sync(0xFFFFFFFFu, wsum, o);
  if (lane == 0 && wsum) atomicAdd(PLAN ? &v.ctr->delivered : r.totals, wsum);
}

// drop mode: eval + select, totals[0] = records selected.  Take mode: eval, scan, select, plan scan, then the receive
// gather exactly as the priority pipeline runs it (totals[0] records, totals[1] payload granules), or with ca the compact
// back end.  glim / tlim (~0: no limit): per-agent limits on the matches' payload granules and token weights; either one
// set runs k_where_take between the eval and the rest (timed under SDB_PK_RECV_COUNT too)
extern "C" cudaError_t sdb_launch_where(const sdb_dev_view* v, const sdb_recv_args* r, const sdb_where_args* f, int drop,
                                        uint32_t max_rec_bytes, cudaStream_t stream, int* n_launches, sdb_profiler* prof,
                                        int sm_count, const sdb_compact_args* ca, unsigned long long glim,
                                        unsigned long long tlim) {
  if (r->n == 0) return cudaSuccess;
  const uint32_t n = r->n;
  const uint32_t blocks = sdb_grid(n, 32, 32 * sm_count);                    // 4 slots per warp, 8 warps per block
  const int pi = sdb_prof_begin(prof, SDB_PK_WHERE, stream);
  if (f->fields & SDB_FILTER_KEYWORD) {
    k_where_kw<<<sdb_grid(n, 8, 8 * sm_count), 256, 0, stream>>>(*v, *r, *f);   // a warp per slot, 8 warps per block
  } else {
    k_where_eval<<<blocks, 256, 0, stream>>>(*v, *r, *f);
  }
  if (glim != ~0ull || tlim != ~0ull) {
    const int pt = sdb_prof_begin(prof, SDB_PK_RECV_COUNT, stream);
    if (r->flags & SDB_RECV_PRIORITY)
      k_where_take<true><<<blocks, 256, 0, stream>>>(*v, *r, f->bits, f->stride, tlim, glim);
    else
      k_where_take<false><<<blocks, 256, 0, stream>>>(*v, *r, f->bits, f->stride, tlim, glim);
    sdb_prof_end(prof, pt, stream);
    if (n_launches) *n_launches += 1;
  }
  if (drop) {
    cudaMemsetAsync(r->totals, 0, 2 * sizeof(unsigned long long), stream);
    k_where_select<false><<<blocks, 256, 0, stream>>>(*v, *r, *f);
    sdb_prof_end(prof, pi, stream);
    if (n_launches) *n_launches += 2;
    return cudaGetLastError();
  }
  // totals[0] = matches; the cut may lower it
  const cudaError_t e = sdb_scan_u32(r->cnt, r->rec_local, r->rec_tops, n, r->totals, nullptr, stream, n_launches);
  k_where_select<true><<<blocks, 256, 0, stream>>>(*v, *r, *f);
  uint64_t bound = static_cast<uint64_t>(n) * (r->max_messages < v->ring_slots ? r->max_messages : v->ring_slots);   // records planned, at most
  if (bound > r->rec_cap) bound = r->rec_cap;
  const uint32_t rtiles = static_cast<uint32_t>((bound + SDB_SCAN_TILE - 1) / SDB_SCAN_TILE);
  k_scan_plan<<<rtiles, 1024, 0, stream>>>(r->plan, r->plan_tops, r->totals);
  k_scan_tops<<<1, 1024, 0, stream>>>(r->plan_tops, rtiles, r->totals + 1);  // totals[1] = payload granules
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += 4;
  if (e != cudaSuccess) return e;
  if (ca) return launch_compact(v, r, ca, nullptr, bound, sm_count, stream, prof, n_launches);
  return launch_gather(v, r, nullptr, bound, max_rec_bytes, sm_count, stream, prof, n_launches);
}

// the id table of SDB_FILTER_IDS from ids[0, n) into the zeroed tab[mask + 1]
extern "C" cudaError_t sdb_launch_id_table(const unsigned long long* ids, uint32_t n, sdb_id_slot* tab, uint32_t mask,
                                           cudaStream_t stream, int* n_launches) {
  if (n) {
    k_id_table<<<(n + 255) / 256, 256, 0, stream>>>(ids, n, tab, mask);
    if (n_launches) ++*n_launches;
  }
  return cudaGetLastError();
}

// per input id, after the filtered receive: out[0, n) hits, out[n, 2n) first agent
extern "C" cudaError_t sdb_launch_id_out(const unsigned long long* ids, uint32_t n, const sdb_id_slot* tab, uint32_t mask,
                                         uint32_t* out, cudaStream_t stream, int* n_launches) {
  if (n) {
    k_id_out<<<(n + 255) / 256, 256, 0, stream>>>(ids, n, tab, mask, out);
    if (n_launches) ++*n_launches;
  }
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------
// arena floor: smallest arena position still referenced by a pending ring entry.
// One thread per agent; distance below the current arena tail is maximised with atomicMax.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_arena_floor(sdb_dev_view v, uint32_t n_agents, uint32_t tail32, unsigned long long* max_dist) {
  const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n_agents) return;
  const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
  const uint32_t head = h.x, tail = h.y;
  const uint32_t mask = v.ring_slots - 1;
  const uint2* rs = sdb_ring_of(v, a);
  for (uint32_t p = head; p != tail; ++p) {
    const uint2 e = rs[p & mask];
    if (sdb_meta(e) != SDB_META_TOMB) {
      const uint32_t dist = tail32 - e.x;               // granules below the arena tail (mod 2^32)
      atomicMax(max_dist, static_cast<unsigned long long>(dist));
      return;                                           // rings are sorted: first live entry is the oldest
    }
  }
}

// same scan for the asynchronous import: the tail comes from the device cursor, the result goes to cursor.floor_dist
__global__ void __launch_bounds__(256)
k_arena_floor_cur(sdb_dev_view v, uint32_t n_agents, sdb_cursor* cur) {
  const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n_agents) return;
  const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
  const uint32_t head = h.x, tail = h.y;
  if (head == tail) return;
  const uint32_t tail32 = static_cast<uint32_t>(cur->arena_tail);
  const uint32_t mask = v.ring_slots - 1;
  const uint2* rs = sdb_ring_of(v, a);
  for (uint32_t p = head; p != tail; ++p) {
    const uint2 e = rs[p & mask];
    if (sdb_meta(e) != SDB_META_TOMB) { atomicMax(&cur->floor_dist, static_cast<unsigned long long>(tail32 - e.x)); return; }
  }
}
extern "C" cudaError_t sdb_launch_arena_floor_cur(const sdb_dev_view* v, uint32_t n_agents, sdb_cursor* cur, cudaStream_t stream) {
  cudaMemsetAsync(&cur->floor_dist, 0, sizeof(unsigned long long), stream);
  if (n_agents) k_arena_floor_cur<<<(n_agents + 255) / 256, 256, 0, stream>>>(*v, n_agents, cur);
  return cudaGetLastError();
}

extern "C" cudaError_t sdb_launch_arena_floor(const sdb_dev_view* v, uint32_t n_agents, uint32_t tail32,
                                              unsigned long long* max_dist_dev, cudaStream_t stream) {
  cudaMemsetAsync(max_dist_dev, 0, sizeof(unsigned long long), stream);
  if (n_agents) k_arena_floor<<<(n_agents + 255) / 256, 256, 0, stream>>>(*v, n_agents, tail32, max_dist_dev);
  return cudaGetLastError();
}

// any kernel of this file: its module is loaded as a whole before the latency server starts (sdb_api.cu)
extern "C" const void* sdb_recv_kernel_anchor() { return reinterpret_cast<const void*>(&k_scan_local); }
