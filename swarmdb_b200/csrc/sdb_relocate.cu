// sdb_relocate.cu - relocation of pinned queues (sdb_arena_relocate), sm_90a.
//
// The arena is a log reclaimed only behind the oldest pending record of any ring, so an agent that stops receiving pins
// it.  A relocation copies the live records of the agents whose oldest pending record lies below a cut to the tail of the
// arena and rewrites their ring entries in place; the floor can then pass the old region.  Nothing is delivered, dropped,
// re-sequenced or reordered.
//
// Layout (include/swarmdb_b200.h, sdb_arena_relocate): the marked granules - the header of every moved record and the
// payload granules of every image a moved record names - keep their arena order; the k-th goes to base + k.  A ring entry
// {handle, dm1} becomes {base + rank(handle), rank(handle + 1 + dm1) - rank(handle) - 1} with rank(x) = marked granules
// below x, so the copies of one shared payload collapse into one and arena positions still increase along every ring.
//
// Plan phase (nothing is written outside scratch):
//   k_reloc_mark     8 lanes per agent: ring header once, the oldest live entry by ballots, then (selected agents) the
//                    header bit and payload run of every live entry into the bitmap; agent / record totals and the
//                    largest distances below the tail (the floor now, and the floor of the unselected agents)
//   k_reloc_count    popcount per bitmap word
//   scan             sdb_scan_u32 (k_scan_local + k_scan_tops) over the popcounts: the rank of every word
// The host reads the totals once and places the region, then the write phase runs:
//   k_reloc_copy     one warp per bitmap word: its marked granules to base + rank, 16-byte chunks, evict-first stores
//   k_reloc_ledger   (dead-letter policy only) one thread per ledger entry: the new handle of a relocated record, before
//                    the ring pass overwrites the old ones
//   k_reloc_ring     8 lanes per selected agent: the new handle and dm1 of every live entry; tombstones keep theirs
// Every kernel is timed under SDB_PK_ARENA_FLOOR.
#include "sdb_common.cuh"

#define SDB_RL_G 8u            // lanes per agent

// arena position of a 32-bit ring handle: handles are positions mod 2^32 and every pending one lies below the tail
__device__ __forceinline__ unsigned long long rl_pos(const sdb_reloc_args& r, uint32_t handle) {
  return r.tail - static_cast<uint32_t>(static_cast<uint32_t>(r.tail) - handle);
}
__device__ __forceinline__ void rl_mark_run(const sdb_reloc_args& r, unsigned long long pos, uint32_t n) {
  unsigned long long k = pos - r.lo;
  while (n) {
    const uint32_t b = static_cast<uint32_t>(k & 31u), take = min(n, 32u - b);
    const uint32_t m = (take == 32u ? 0xFFFFFFFFu : ((1u << take) - 1u)) << b;
    atomicOr(r.bits + (k >> 5), m);
    k += take; n -= take;
  }
}
// marked granules below arena position pos (lo <= pos <= tail)
__device__ __forceinline__ uint32_t rl_rank(const sdb_reloc_args& r, unsigned long long pos) {
  const unsigned long long k = pos - r.lo;
  const uint32_t w = static_cast<uint32_t>(k >> 5);
  return sdb_scan_at(r.pre, r.tops, w) + __popc(r.bits[w] & ((1u << (k & 31u)) - 1u));
}
__device__ __forceinline__ bool rl_selected(const sdb_reloc_args& r, uint32_t a) { return (r.sel[a >> 5] >> (a & 31u)) & 1u; }

__global__ void __launch_bounds__(256)
k_reloc_mark(sdb_dev_view v, sdb_reloc_args r) {
  const uint32_t lane = threadIdx.x & 31, l8 = lane & (SDB_RL_G - 1), gsh = lane & ~(SDB_RL_G - 1);
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint32_t mask = v.ring_slots - 1, tail32 = static_cast<uint32_t>(r.tail);
  constexpr uint32_t SPW = 32u / SDB_RL_G;
  unsigned long long wag = 0, wrec = 0, wdall = 0, wdun = 0;
  for (uint32_t ab = gw * SPW; ab < r.n_agents; ab += nw * SPW) {      // warp-uniform
    const uint32_t a = ab + lane / SDB_RL_G;
    uint32_t head = 0, W = 0;
    if (a < r.n_agents) {
      const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);   // one address for the agent's 8 lanes
      head = h.x; W = h.y - h.x;
    }
    const uint2* rs = sdb_ring_of(v, a < r.n_agents ? a : 0u);
    bool found = false, sel = false;                                    // group-uniform
    uint32_t dist = 0, recs = 0;
    const uint32_t wmax = __reduce_max_sync(0xFFFFFFFFu, W);
    for (uint32_t j0 = 0; j0 < wmax; j0 += SDB_RL_G) {
      const uint32_t j = j0 + l8;
      const bool in = j < W;
      const uint2 e = in ? rs[(head + j) & mask] : make_uint2(0u, SDB_META_TOMB);
      const bool live = in && sdb_meta(e) != SDB_META_TOMB;
      const uint32_t bm = (__ballot_sync(0xFFFFFFFFu, live) >> gsh) & 0xFFu;
      const uint32_t fx = __shfl_sync(0xFFFFFFFFu, e.x, bm ? gsh + __ffs(bm) - 1u : lane);
      if (!found && bm) {                                               // the oldest live entry: rings are sorted
        found = true;
        dist = tail32 - fx;
        sel = dist > r.thr;
      }
      if (sel && live) {
        const unsigned long long pos = rl_pos(r, e.x);
        rl_mark_run(r, pos, 1u);
        rl_mark_run(r, pos + 1u + sdb_entry_dm1(e.y), (e.y & SDB_META_GLEN_MASK) - 1u);
        ++recs;
      }
      if (!__any_sync(0xFFFFFFFFu, j0 + SDB_RL_G < W && !(found && !sel))) break;   // nothing left to find or mark
    }
#pragma unroll
    for (uint32_t o = SDB_RL_G / 2; o; o >>= 1) recs += __shfl_xor_sync(0xFFFFFFFFu, recs, o);
    if (l8 == 0 && found) {
      wdall = dist > wdall ? dist : wdall;
      if (sel) {
        atomicOr(r.sel + (a >> 5), 1u << (a & 31u));
        ++wag; wrec += recs;
      } else {
        wdun = dist > wdun ? dist : wdun;
      }
    }
  }
  for (int o = 16; o; o >>= 1) {
    wag += __shfl_xor_sync(0xFFFFFFFFu, wag, o);
    wrec += __shfl_xor_sync(0xFFFFFFFFu, wrec, o);
    const unsigned long long d1 = __shfl_xor_sync(0xFFFFFFFFu, wdall, o), d2 = __shfl_xor_sync(0xFFFFFFFFu, wdun, o);
    wdall = d1 > wdall ? d1 : wdall;
    wdun = d2 > wdun ? d2 : wdun;
  }
  if (lane == 0) {
    if (wag) { atomicAdd(r.tot + 1, wag); atomicAdd(r.tot + 2, wrec); }
    if (wdall) atomicMax(r.tot + 3, wdall);
    if (wdun) atomicMax(r.tot + 4, wdun);
  }
}

__global__ void __launch_bounds__(256)
k_reloc_count(sdb_reloc_args r) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w < r.words) r.cnt[w] = __popc(r.bits[w]);
}

__global__ void __launch_bounds__(256)
k_reloc_copy(sdb_dev_view v, sdb_reloc_args r) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint64_t pol = sdb_policy_evict_first();
  for (uint32_t w = gw; w < r.words; w += nw) {                         // warp-uniform
    const uint32_t m = r.bits[w];
    if (!m) continue;
    const uint32_t r0 = sdb_scan_at(r.pre, r.tops, w);
    const unsigned long long p0 = r.lo + (static_cast<unsigned long long>(w) << 5);
#pragma unroll
    for (uint32_t c = lane; c < 64u; c += 32u) {                         // 16-byte chunk c of granule c / 2
      const uint32_t g = c >> 1;
      if ((m >> g) & 1u) {
        const uint32_t rank = r0 + __popc(m & ((1u << g) - 1u));
        const uint4 x = sdb_ld_stream(sdb_arena_ptr(v, p0 + g) + ((c & 1u) << 4));
        sdb_st_stream_pol(sdb_arena_ptr(v, r.base + rank) + ((c & 1u) << 4), x, pol);
      }
    }
  }
}

// an entry is moved when its agent is selected and its slot is still the live record it counts (k_ledger_collect's test)
__global__ void __launch_bounds__(256)
k_reloc_ledger(sdb_dev_view v, sdb_ledger L, uint32_t n, sdb_reloc_args r) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const sdb_ledger_ent en = L.ent[e];
  if (en.agent >= r.n_agents || !rl_selected(r, en.agent)) return;
  const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + en.agent);
  if (en.p - h.x >= h.y - h.x) return;
  const uint2 x = sdb_ring_of(v, en.agent)[en.p & (v.ring_slots - 1)];
  if (sdb_meta(x) == SDB_META_TOMB || x.x != en.handle) return;
  L.ent[e].handle = static_cast<uint32_t>(r.base + rl_rank(r, rl_pos(r, en.handle)));
}

__global__ void __launch_bounds__(256)
k_reloc_ring(sdb_dev_view v, sdb_reloc_args r) {
  const uint32_t lane = threadIdx.x & 31, l8 = lane & (SDB_RL_G - 1);
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint32_t mask = v.ring_slots - 1;
  constexpr uint32_t SPW = 32u / SDB_RL_G;
  for (uint32_t ab = gw * SPW; ab < r.n_agents; ab += nw * SPW) {
    const uint32_t a = ab + lane / SDB_RL_G;
    if (a >= r.n_agents || !rl_selected(r, a)) continue;
    const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
    uint2* rs = sdb_ring_of(v, a);
    for (uint32_t j = l8; j < h.y - h.x; j += SDB_RL_G) {
      const uint32_t s = (h.x + j) & mask;
      const uint2 e = rs[s];
      if (sdb_meta(e) == SDB_META_TOMB) continue;
      const unsigned long long pos = rl_pos(r, e.x);
      const uint32_t rh = rl_rank(r, pos);
      const uint32_t dm1 = rl_rank(r, pos + 1u + sdb_entry_dm1(e.y)) - rh - 1u;
      rs[s] = make_uint2(static_cast<uint32_t>(r.base + rh), (e.y & 0xFFFFu) | (dm1 << 16));
    }
  }
}

// plan phase: r->tot ends with the totals the host reads (tot[0] = marked granules)
extern "C" cudaError_t sdb_launch_reloc_plan(const sdb_dev_view* v, const sdb_reloc_args* r, cudaStream_t stream, sdb_profiler* prof,
                                             int* n_launches, int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_ARENA_FLOOR, stream);
  cudaError_t e = cudaMemsetAsync(r->tot, 0, 5 * sizeof(unsigned long long), stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(r->bits, 0, static_cast<size_t>(r->words) * sizeof(uint32_t), stream);
  if (e == cudaSuccess && r->n_agents)
    e = cudaMemsetAsync(r->sel, 0, static_cast<size_t>((r->n_agents + 31) / 32) * sizeof(uint32_t), stream);
  int nl = 0;
  if (e == cudaSuccess) {
    if (r->n_agents) {
      k_reloc_mark<<<sdb_grid(r->n_agents, 32, 32 * sm_count), 256, 0, stream>>>(*v, *r);
      ++nl;
    }
    k_reloc_count<<<(r->words + 255) / 256, 256, 0, stream>>>(*r);
    ++nl;
    e = sdb_scan_u32(r->cnt, r->pre, r->tops, r->words, r->tot, nullptr, stream, &nl);
  }
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// write phase: r->base is the placed region; the ledger (nullptr: no dead-letter policy) holds n_ledger entries
extern "C" cudaError_t sdb_launch_reloc_write(const sdb_dev_view* v, const sdb_reloc_args* r, const sdb_ledger* ledger,
                                              uint32_t n_ledger, cudaStream_t stream, sdb_profiler* prof, int* n_launches,
                                              int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_ARENA_FLOOR, stream);
  int nl = 0;
  k_reloc_copy<<<sdb_grid(r->words, 8, 32 * sm_count), 256, 0, stream>>>(*v, *r);
  ++nl;
  if (ledger && n_ledger) { k_reloc_ledger<<<(n_ledger + 255) / 256, 256, 0, stream>>>(*v, *ledger, n_ledger, *r); ++nl; }
  if (r->n_agents) { k_reloc_ring<<<sdb_grid(r->n_agents, 32, 32 * sm_count), 256, 0, stream>>>(*v, *r); ++nl; }
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return cudaGetLastError();
}

// any kernel of this file: its module is loaded as a whole before the latency server starts (sdb_api.cu)
extern "C" const void* sdb_relocate_kernel_anchor() { return reinterpret_cast<const void*>(&k_reloc_mark); }
