// sdb_xshard.cu - cross-shard delivery of group sends (sm_90a): the receiving half.
//
// Replaces the reference's partitioned Kafka topic (explicit-partition produce M:469-482, one
// consumer per agent over all partitions M:334-345).  Agents are hash-partitioned over the GPUs
// of the box; group tables are replicated, each shard keeping the members it owns and their
// positions in the full list.  A rank exports its batch of group sends ONCE per send
// (descriptor + payload), the caller all-gathers the wire batches over NVLink (NCCL), and
// every shard expands, for every send of every source, the copies for the members it owns:
//
//   k_wire_table      prefix table over the sources (sends, sequence offsets, section offsets)
//   k_wire_measure    per wire send: local member count x record size (scan input)
//   k_bucket_sizes    per (group, source): size of the exporter-built bucket
//   scans             arena offsets of every send's local region; global bucket offsets
//   k_wire_localize   writes the local fan-out descriptor (payload address in the exporter's buffer,
//                     global sequence offset, local member list)
//   k_bucket_fill     concatenates the sources' buckets in rank order (= global send order)
//   then the ordinary fan-out kernel + pull index build run over the localized descriptors.
//
// NVLink carries (64 + payload) bytes per (send, peer) instead of (32 + payload) per recipient:
// 8 x less for 64-way groups on 8 shards.  With the peer-memory transport (sdb_import_wire_ptrs over
// CUDA-IPC mapped export buffers) there is no separate collective at all: these kernels read the
// descriptors, and the fan-out kernel's TMA bulk loads read the payloads, straight out of the
// exporting GPU's memory, so the NVLink transfer overlaps the fan-out send by send and a shard only
// pulls the sends it has recipients for.
#include "sdb_common.cuh"

__device__ __forceinline__ const sdb_wire_header* wire_hdr(const sdb_import_args& a, uint32_t src) {
  return reinterpret_cast<const sdb_wire_header*>(a.meta[src]);
}

// one thread: read the n_src wire headers (remote when the batch lives in a peer GPU) and publish the prefix table
__global__ void k_wire_table(sdb_import_args a, sdb_src_tab* tab) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  uint32_t first = 0; uint64_t rb = 0;
  for (uint32_t s = 0; s < a.n_src; ++s) {
    const sdb_wire_header* h = wire_hdr(a, s);
    const bool ok = h->magic == SDB_WIRE_MAGIC;
    const bool ex = ok && h->explicit_seq;
    tab->first[s] = first; tab->rec_base[s] = ex ? h->seq_base : rb; tab->explicit_seq[s] = ex ? 1u : 0u;
    tab->desc_off[s] = ok ? h->desc_off : 0; tab->list_off[s] = ok ? h->list_off : 0; tab->payload_off[s] = ok ? h->payload_off : 0;
    tab->gs_off_off[s] = (ok && h->max_groups == a.max_groups) ? h->gs_off_off : 0; tab->gs_idx_off[s] = ok ? h->gs_idx_off : 0;
    first += ok ? min(h->n_sends, a.max_sends) : 0u;
    rb += ok ? h->total_recs : 0ull;
  }
  for (uint32_t s = a.n_src; s <= SDB_MAX_SRC; ++s) tab->first[s] = first;
}

// global send index -> (source, index inside the source), sources concatenated in rank order
__device__ __forceinline__ bool locate(const sdb_import_args& a, uint32_t gi, uint32_t& src, uint32_t& i,
                                       uint64_t& rec_base) {
  const sdb_src_tab* t = a.tab;
  if (gi >= t->first[a.n_src]) return false;
  uint32_t s = 0;
  while (s + 1 < a.n_src && gi >= t->first[s + 1]) ++s;
  src = s; i = gi - t->first[s]; rec_base = t->rec_base[s];
  return true;
}

__device__ __forceinline__ const sdb_send_desc* wire_desc(const sdb_import_args& a, uint32_t src, uint32_t i) {
  return reinterpret_cast<const sdb_send_desc*>(a.meta[src] + a.tab->desc_off[src]) + i;
}

__device__ __forceinline__ const uint32_t* wire_list(const sdb_import_args& a, uint32_t src) {
  return reinterpret_cast<const uint32_t*>(a.wire[src] + a.tab->list_off[src]);
}

__global__ void __launch_bounds__(256)
k_wire_measure(sdb_import_args a, uint32_t n_total) {
  const uint32_t gi = blockIdx.x * blockDim.x + threadIdx.x;
  if (gi >= n_total) return;
  uint32_t src, i; uint64_t rb;
  if (!locate(a, gi, src, i, rb)) { a.w[gi] = 0; a.lw[gi] = 0; return; }
  const uint4* dq = reinterpret_cast<const uint4*>(wire_desc(a, src, i));
  sdb_send_desc dd;                                             // one 64-byte read of the (remote) descriptor
  reinterpret_cast<uint4*>(&dd)[0] = __ldg(dq); reinterpret_cast<uint4*>(&dd)[1] = __ldg(dq + 1);
  reinterpret_cast<uint4*>(&dd)[2] = __ldg(dq + 2); reinterpret_cast<uint4*>(&dd)[3] = __ldg(dq + 3);
  const sdb_send_desc* d = &dd;
  uint32_t lc = 0, own = 0;
  if (d->flags & SDB_DESC_P2P) {                                   // delivered by the receiver's owner only
    own = (d->mstart < a.max_agents && a.shard_of[d->mstart] == a.shard_id) ? 1u : 0u;
    lc = own;
  } else if (d->flags & SDB_DESC_LIST_TEMP) {                      // broadcast: the recipients this shard owns
    const uint32_t* l = wire_list(a, src) + d->mstart;
    for (uint32_t k = 0; k < d->mcount; ++k) { const uint32_t x = l[k]; own += (x < a.max_agents && a.shard_of[x] == a.shard_id); }
    lc = own;
  } else {
    const uint32_t g = d->group;
    lc = g < a.max_groups ? a.lcount[g] : 0u;
  }
  a.w[gi] = lc * d->rgran;
  a.lw[gi] = own;
}

__global__ void __launch_bounds__(256)
k_wire_localize(sdb_import_args a, uint32_t n_total) {
  const uint32_t gi = blockIdx.x * blockDim.x + threadIdx.x;
  if (gi >= n_total) return;
  uint32_t src, i; uint64_t rb;
  sdb_send_desc out;
  if (!locate(a, gi, src, i, rb)) {                  // unused capacity: an empty send
    uint4 z = make_uint4(0, 0, 0, 0);
    uint4* o = reinterpret_cast<uint4*>(a.descs + gi);
    o[0] = z; o[1] = z; o[2] = z; o[3] = z;
    return;
  }
  {
    const uint4* dq = reinterpret_cast<const uint4*>(wire_desc(a, src, i));
    reinterpret_cast<uint4*>(&out)[0] = __ldg(dq); reinterpret_cast<uint4*>(&out)[1] = __ldg(dq + 1);
    reinterpret_cast<uint4*>(&out)[2] = __ldg(dq + 2); reinterpret_cast<uint4*>(&out)[3] = __ldg(dq + 3);
  }
  const sdb_send_desc wd = out;
  const sdb_send_desc* d = &wd;
  // absolute address (the fan-out kernel is launched with a null payload base): the payload stays where the
  // source rank exported it - possibly in a peer GPU's memory - and is pulled by the fan-out's TMA loads
  out.payload_off = reinterpret_cast<uint64_t>(a.wire[src]) + a.tab->payload_off[src] + d->payload_off;
  out.gran0 = sdb_scan_at(a.w_local, a.w_tops, gi);
  out.rec0 = static_cast<uint32_t>(rb + d->rec0);
  const bool abs_seq = a.tab->explicit_seq[src] != 0;
  out.seq_abs = abs_seq ? rb + d->rec0 : 0ull;
  if (d->flags & (SDB_DESC_P2P | SDB_DESC_LIST_TEMP)) {
    const uint32_t own = a.lw[gi];
    uint32_t lo = sdb_scan_at(a.lw_local, a.lw_tops, gi);
    const bool fits = static_cast<uint64_t>(lo) + own <= a.list_cap;      // checked on the host before launch
    out.mstart = lo; out.mcount = fits ? own : 0u; out.group = SDB_NO_GROUP;
    if (d->flags & SDB_DESC_P2P) {
      out.flags = SDB_DESC_LIST_TEMP | (abs_seq ? SDB_DESC_ABS_SEQ : 0u);
      if (own && fits) a.tmp_list[lo] = d->mstart;
    } else {
      out.flags = SDB_DESC_LIST_TEMP | SDB_DESC_SHARED_SEQ | (abs_seq ? SDB_DESC_ABS_SEQ : 0u);
      if (fits) {
        const uint32_t* l = wire_list(a, src) + d->mstart;
        for (uint32_t k = 0; k < d->mcount; ++k) { const uint32_t x = l[k]; if (x < a.max_agents && a.shard_of[x] == a.shard_id) a.tmp_list[lo++] = x; }
      }
    }
    a.descs[gi] = out;
    return;
  }
  const uint32_t g = d->group;
  const uint32_t lc = g < a.max_groups ? a.lcount[g] : 0u;
  out.mstart = lc ? a.lstart[g] : 0u;
  out.mcount = lc;
  out.flags = SDB_DESC_SKIP_SENDER | SDB_DESC_PULL | SDB_DESC_POS | (abs_seq ? SDB_DESC_ABS_SEQ : 0u);
  a.descs[gi] = out;
}

// The exporter already bucketed its group sends by group (ascending send index).  The global bucket of a
// group is the concatenation of the sources' buckets in rank order - which is global send order - so no
// atomics and no sort: sizes per (group, source), one scan, one copy.
__device__ __forceinline__ const uint32_t* src_gs_off(const sdb_import_args& a, uint32_t s) {
  return reinterpret_cast<const uint32_t*>(a.meta[s] + a.tab->gs_off_off[s]);
}
__global__ void __launch_bounds__(256)
k_bucket_sizes(sdb_import_args a) {
  const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t n = a.max_groups * a.n_src;
  if (idx > n) return;
  uint32_t c = 0;
  if (idx < n) {
    const uint32_t g = idx / a.n_src, s = idx % a.n_src;
    if (a.lcount[g] && a.tab->gs_off_off[s]) { const uint32_t* o = src_gs_off(a, s); c = o[g + 1] - o[g]; }
  }
  a.gs_cnt[idx] = c;
}
__global__ void __launch_bounds__(256)
k_bucket_fill(sdb_import_args a, const uint32_t* __restrict__ goff, uint32_t* __restrict__ gs_off_out) {
  const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t n = a.max_groups * a.n_src;
  if (idx > n) return;
  if (idx == n) { gs_off_out[a.max_groups] = goff[n]; return; }
  const uint32_t g = idx / a.n_src, s = idx % a.n_src;
  const uint32_t dst = goff[idx];
  if (s == 0) gs_off_out[g] = dst;
  if (!a.lcount[g] || !a.tab->gs_off_off[s]) return;
  const uint32_t* o = src_gs_off(a, s);
  const uint32_t* ix = reinterpret_cast<const uint32_t*>(a.meta[s] + a.tab->gs_idx_off[s]);
  const uint32_t b = o[g], e = o[g + 1], first = a.tab->first[s];
  for (uint32_t k = b; k < e; ++k) a.gs_idx[dst + (k - b)] = first + ix[k];
}

// phase 1: measure + scans.  totals_dev[0] receives the arena granules this import will write.
extern "C" cudaError_t sdb_launch_import_measure(const sdb_import_args* a, uint32_t n_cap, uint32_t* w_local,
                                                 uint32_t* w_tops, uint32_t* gs_local, uint32_t* gs_tops,
                                                 uint32_t* gs_off_out, uint32_t* lw_local, uint32_t* lw_tops,
                                                 unsigned long long* totals_dev,
                                                 cudaStream_t stream, sdb_profiler* prof, int* n_launches) {
  const int pi = sdb_prof_begin(prof, SDB_PK_XSHARD, stream);
  k_wire_table<<<1, 32, 0, stream>>>(*a, const_cast<sdb_src_tab*>(a->tab));
  k_wire_measure<<<(n_cap + 255) / 256, 256, 0, stream>>>(*a, n_cap);
  int nl = 3;                                                  // k_wire_table, k_wire_measure, k_bucket_sizes
  cudaError_t e = sdb_scan_u32(a->w, w_local, w_tops, n_cap, totals_dev, nullptr, stream, &nl);
  const uint32_t nb = a->max_groups * a->n_src + 1;
  k_bucket_sizes<<<(nb + 255) / 256, 256, 0, stream>>>(*a);
  // gs_off_out here is the materialised scan over (group, source) pairs ("goff", nb entries)
  if (e == cudaSuccess) e = sdb_scan_u32(a->gs_cnt, gs_local, gs_tops, nb, nullptr, gs_off_out, stream, &nl);
  if (e == cudaSuccess) e = sdb_scan_u32(a->lw, lw_local, lw_tops, n_cap, totals_dev + 1, nullptr, stream, &nl);   // owned recipients
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return e != cudaSuccess ? e : cudaGetLastError();
}

// phase 2: localized descriptors + ordered buckets
extern "C" cudaError_t sdb_launch_import_localize(const sdb_import_args* a, uint32_t n_cap, const uint32_t* goff,
                                                  uint32_t* gs_off_out, cudaStream_t stream, sdb_profiler* prof,
                                                  int* n_launches) {
  const int pi = sdb_prof_begin(prof, SDB_PK_XSHARD, stream);
  k_wire_localize<<<(n_cap + 255) / 256, 256, 0, stream>>>(*a, n_cap);
  const uint32_t nb = a->max_groups * a->n_src + 1;
  k_bucket_fill<<<(nb + 255) / 256, 256, 0, stream>>>(*a, goff, gs_off_out);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += 2;
  return cudaGetLastError();
}

// ==========================================================================================
// Asynchronous import (sdb_import_wire_ptrs_async): no host round trip, no collective.
//
//   k_wire_wait      one warp: spins until every source's export buffer carries ready >= step (sources in peer GPUs
//                    are polled over NVLink with volatile loads, so every poll reads the exporter's current value)
//   k_arena_floor    (sdb_recv.cu) distance of the oldest pending record below the arena tail -> cursor.floor_dist
//   k_import_fused   everything k_wire_table / k_wire_measure / 3 scans / k_bucket_sizes / k_wire_localize /
//                    k_bucket_fill did in ~15 launches plus a host sync, in ONE pass:
//                      * every block reads the <= 16 wire headers itself (no leader, no table kernel)
//                      * one thread per wire send: reads the 64-byte descriptor where the source exported it
//                        (straight out of the peer GPU), counts this shard's share, and a decoupled look-back over
//                        256-send tiles (wide window, {arena granules, temporary-list entries} as a 31+31-bit
//                        pair) gives the send its place in the arena; the localized descriptor is written
//                      * the sources' group buckets are copied next to the descriptors (the group-parallel
//                        index build walks them source by source: nothing is concatenated or sorted)
//                      * the LAST tile places the whole import: arena base from the device cursor (wrap rule,
//                        floor check), sequence base, totals -> sdb_batch_base for the kernels that follow
//   k_wire_done      publishes done = step in this rank's own buffer (its exporter may then be overwritten by peers'
//                    view: see sdb_wire_ctrl)
// ==========================================================================================
__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) {
  uint32_t x;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(x) : "l"(p) : "memory");
  return x;
}

struct sdb_wait_args { const uint32_t* flag[SDB_MAX_SRC]; const uint8_t* wire[SDB_MAX_SRC]; sdb_wire_header* hdr_out; uint32_t n; };
__global__ void k_wire_wait(sdb_wait_args w, uint32_t step) {
  const uint32_t lane = threadIdx.x;
  if (lane < w.n) {
    // bounded: a peer that never publishes must surface as a launch failure, not as a hung GPU
    unsigned long long t0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (;;) {
      if (static_cast<int32_t>(ld_volatile_u32(w.flag[lane]) - step) >= 0) break;
      unsigned long long t1;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      if (t1 - t0 > 120ull * 1000000000ull) __trap();       // two minutes: the peer is gone
      __nanosleep(100);
    }
  }
  __syncwarp();
  __threadfence_system();
  // the sources' 128-byte wire headers, fetched once here (8 x 16 bytes per source, remote ones over NVLink) so that
  // the thousands of blocks of the import kernel read them from local memory
  if (w.hdr_out) {
    for (uint32_t e = lane; e < w.n * 8u; e += 32) {
      const uint32_t s = e >> 3, k = e & 7u;
      reinterpret_cast<uint4*>(w.hdr_out + s)[k] = __ldcv(reinterpret_cast<const uint4*>(w.wire[s]) + k);
    }
  }
}
__global__ void k_wire_set(uint32_t* flag, uint32_t step) {
  __threadfence_system();                      // everything this stream wrote before is visible to peers first
  *reinterpret_cast<volatile uint32_t*>(flag) = step;
  __threadfence_system();
}

#define SDB_IMP_TILE 256u

// Places one localized import: arena base from the device cursor (wrap rule, floor check), sequence base, totals ->
// sdb_batch_base for the kernels that follow.  One thread; the floor scan ran just before on the same stream.
__device__ __forceinline__ void sdb_place_import(const sdb_import_totals& t, sdb_cursor* c, sdb_batch_base* b,
                                                 unsigned long long G, uint32_t list_cap, uint32_t* commit_count) {
  unsigned long long tail = c->arena_tail;
  const unsigned long long floor_now = tail - c->floor_dist;
  if (floor_now > c->arena_floor) c->arena_floor = floor_now;
  if ((tail & (G - 1)) + t.need > G) tail = (tail + G - 1) & ~(G - 1);      // an import never straddles the wrap
  uint32_t skip = 0;
  if (t.need > G || tail + t.need - c->arena_floor > G) { skip = 1; c->error |= 1ull; }
  if (t.lists > list_cap) { skip = 1; c->error |= 2ull; }
  if (t.maxpad > 512) { skip = 1; c->error |= 4ull; }                       // the asynchronous path only drives the span kernel
  b->arena_base = tail; b->seq_base = c->next_seq; b->n_total = t.n_total; b->n_other = t.n_other; b->skip = skip;
  b->max_padlen = t.maxpad; b->total_grans = t.need; b->total_recs = t.total_recs;
  if (commit_count) *commit_count = 0u;                                     // worklist of the commit sort that follows
  if (!skip) {
    c->arena_tail = tail + t.need;
    const unsigned long long ns = c->next_seq + (t.explicit_end ? 0ull : t.total_recs);
    c->next_seq = ns > t.explicit_end ? ns : t.explicit_end;
  }
}
__global__ void k_import_place(const sdb_import_totals* t, sdb_cursor* c, sdb_batch_base* b, unsigned long long G,
                               uint32_t list_cap, uint32_t* commit_count) {
  if (threadIdx.x == 0 && blockIdx.x == 0) sdb_place_import(*t, c, b, G, list_cap, commit_count);
}

__global__ void __launch_bounds__(256)
k_import_fused(sdb_import2_args a, uint32_t tiles_cap) {
  __shared__ uint32_t s_tile;
  __shared__ uint32_t s_first[SDB_MAX_SRC + 1], s_nsend[SDB_MAX_SRC], s_ok[SDB_MAX_SRC], s_explicit[SDB_MAX_SRC];
  __shared__ uint32_t s_nother[SDB_MAX_SRC], s_ngs[SDB_MAX_SRC], s_maxpad[SDB_MAX_SRC];
  __shared__ unsigned long long s_recbase[SDB_MAX_SRC], s_totalrecs[SDB_MAX_SRC], s_desc_off[SDB_MAX_SRC], s_list_off[SDB_MAX_SRC];
  __shared__ unsigned long long s_pay_off[SDB_MAX_SRC], s_gso_off[SDB_MAX_SRC], s_gsi_off[SDB_MAX_SRC], s_seqbase[SDB_MAX_SRC];
  __shared__ unsigned long long s_wa[8], s_wb[8], s_ba, s_bb;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_tile = atomicAdd(reinterpret_cast<unsigned int*>(a.lb + sdb_lb_words(tiles_cap) - 2), 1u);
  // ---- every block reads the wire headers itself (128 bytes each, from the local copies k_wire_wait made)
  if (tid < a.n_src) {
    const sdb_wire_header* h = a.hdrs + tid;                 // local copies made by k_wire_wait
    const uint4* hq = reinterpret_cast<const uint4*>(h);
    union { uint4 q[8]; sdb_wire_header hd; } u;
#pragma unroll
    for (int k = 0; k < 8; ++k) u.q[k] = hq[k];
    const bool ok = u.hd.magic == SDB_WIRE_MAGIC;
    s_ok[tid] = ok ? 1u : 0u;
    s_nsend[tid] = ok ? min(u.hd.n_sends, a.max_sends) : 0u;
    s_totalrecs[tid] = ok ? u.hd.total_recs : 0ull;
    s_explicit[tid] = (ok && u.hd.explicit_seq) ? 1u : 0u;
    s_seqbase[tid] = u.hd.seq_base;
    s_desc_off[tid] = u.hd.desc_off; s_list_off[tid] = u.hd.list_off; s_pay_off[tid] = u.hd.payload_off;
    s_gso_off[tid] = (ok && u.hd.max_groups == a.max_groups) ? u.hd.gs_off_off : 0ull; s_gsi_off[tid] = u.hd.gs_idx_off;
    s_nother[tid] = ok ? u.hd.n_other : 0u; s_ngs[tid] = ok ? min(u.hd.n_group_sends, a.max_sends) : 0u;
    s_maxpad[tid] = ok ? u.hd.max_padlen : 0u;
  }
  __syncthreads();
  if (tid == 0) {
    uint32_t f = 0; unsigned long long rb = 0;
    for (uint32_t s = 0; s < a.n_src; ++s) {
      s_first[s] = f; s_recbase[s] = s_explicit[s] ? s_seqbase[s] : rb;
      f += s_nsend[s]; rb += s_totalrecs[s];
    }
    s_first[a.n_src] = f;
  }
  __syncthreads();
  const uint32_t tile = s_tile;
  const uint32_t n_total = s_first[a.n_src];
  const uint32_t n_tiles = n_total ? (n_total + SDB_IMP_TILE - 1) / SDB_IMP_TILE : 1u;     // tiles that take part in the scan

  // ---- copies of the sources' group buckets: one flat element space over (source, offsets | indices), every thread
  // issues all its (remote, coalesced) loads before the first store so the NVLink round trips overlap
  {
    const uint32_t G1 = a.max_groups + 1;
    const uint32_t per_src = G1 + a.max_sends;
    const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
    const size_t E = static_cast<size_t>(a.n_src) * per_src;
    const size_t gt = static_cast<size_t>(tile) * blockDim.x + tid;
    constexpr int UN = 4;
    for (size_t e0 = gt; e0 < E; e0 += nthreads * UN) {
      uint32_t val[UN]; uint32_t* dst[UN];
#pragma unroll
      for (int u = 0; u < UN; ++u) {
        const size_t e = e0 + static_cast<size_t>(u) * nthreads;
        dst[u] = nullptr; val[u] = 0;
        if (e < E) {
          const uint32_t s = static_cast<uint32_t>(e / per_src), i = static_cast<uint32_t>(e % per_src);
          const bool usable = s_gso_off[s] != 0;
          if (i < G1) {
            dst[u] = a.gs_off_src + static_cast<size_t>(s) * G1 + i;
            if (usable) val[u] = reinterpret_cast<const uint32_t*>(a.wire[s] + s_gso_off[s])[i];
          } else if (usable && i - G1 < s_ngs[s]) {
            dst[u] = a.gs_idx_src + static_cast<size_t>(s) * a.max_sends + (i - G1);
            val[u] = reinterpret_cast<const uint32_t*>(a.wire[s] + s_gsi_off[s])[i - G1];
          }
        }
      }
#pragma unroll
      for (int u = 0; u < UN; ++u) if (dst[u]) *dst[u] = val[u];
    }
    if (tile == 0 && tid <= a.n_src) a.first[tid] = s_first[tid];
  }
  if (tile >= n_tiles) return;

  // ---- one wire send per thread
  const uint32_t gi = tile * SDB_IMP_TILE + tid;
  sdb_send_desc d;
  uint32_t src = 0, lc = 0, own = 0;
  bool have = gi < n_total;
  if (have) {
    while (src + 1 < a.n_src && gi >= s_first[src + 1]) ++src;
    const uint32_t i = gi - s_first[src];
    const uint4* dq = reinterpret_cast<const uint4*>(a.wire[src] + s_desc_off[src]) + static_cast<size_t>(i) * 4;
    uint4* o = reinterpret_cast<uint4*>(&d);
    o[0] = dq[0]; o[1] = dq[1]; o[2] = dq[2]; o[3] = dq[3];
    if (d.flags & SDB_DESC_P2P) {                                   // delivered by the receiver's owner only
      own = (d.mstart < a.max_agents && a.shard_of[d.mstart] == a.shard_id) ? 1u : 0u;
      lc = own;
    } else if (d.flags & SDB_DESC_LIST_TEMP) {                      // broadcast: the recipients this shard owns
      const uint32_t* l = reinterpret_cast<const uint32_t*>(a.wire[src] + s_list_off[src]) + d.mstart;
      for (uint32_t k = 0; k < d.mcount; ++k) { const uint32_t x = l[k]; own += (x < a.max_agents && a.shard_of[x] == a.shard_id); }
      lc = own;
    } else {
      lc = d.group < a.max_groups ? a.lcount[d.group] : 0u;
    }
  }
  // arena granules written here: lc whole records, or (shared payloads, group sends) lc headers + one payload
  const bool group_send = have && !(d.flags & (SDB_DESC_P2P | SDB_DESC_LIST_TEMP));
  const unsigned long long wa = !have ? 0ull
      : (a.shared && group_send) ? (lc ? static_cast<unsigned long long>(lc) + d.rgran - 1u : 0ull)
      : static_cast<unsigned long long>(lc) * d.rgran;
  const unsigned long long wb = own;                                                            // temporary-list entries

  // ---- tile scan + decoupled look-back of the pair
  unsigned long long ia = wa, ib = wb;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long ya = __shfl_up_sync(0xFFFFFFFFu, ia, o), yb = __shfl_up_sync(0xFFFFFFFFu, ib, o);
    if (lane >= o) { ia += ya; ib += yb; }
  }
  if (lane == 31) { s_wa[warp] = ia; s_wb[warp] = ib; }
  __syncthreads();
  if (warp == 0) {
    const unsigned long long xa = lane < 8 ? s_wa[lane] : 0ull, xb = lane < 8 ? s_wb[lane] : 0ull;
    unsigned long long ca = xa, cb = xb;
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) {
      const unsigned long long ya = __shfl_up_sync(0xFFFFFFFFu, ca, o), yb = __shfl_up_sync(0xFFFFFFFFu, cb, o);
      if (lane >= o) { ca += ya; cb += yb; }
    }
    const unsigned long long ta = __shfl_sync(0xFFFFFFFFu, ca, 7), tb = __shfl_sync(0xFFFFFFFFu, cb, 7);
    if (lane < 8) { s_wa[lane] = ca - xa; s_wb[lane] = cb - xb; }
    unsigned long long ea, eb, ga, gb; bool last;
    sdb_lb_prefix(a.lb, tile, n_tiles, ta, tb, lane, ea, eb, last, ga, gb);
    if (lane == 0) {
      s_ba = ea; s_bb = eb;
      if (last) {
        // ---- the grand totals are known here and only here
        sdb_import_totals t;
        t.need = ga; t.lists = gb; t.total_recs = 0; t.explicit_end = 0; t.n_total = n_total; t.n_other = 0; t.maxpad = 0; t.pad = 0;
        for (uint32_t s = 0; s < a.n_src; ++s) {
          t.total_recs += s_totalrecs[s]; t.n_other += s_nother[s]; t.maxpad = max(t.maxpad, s_maxpad[s]);
          if (s_explicit[s]) t.explicit_end = max(t.explicit_end, s_seqbase[s] + s_totalrecs[s]);
        }
        if (a.totals) *a.totals = t;                                         // prefetched: placed later (k_import_place)
        else sdb_place_import(t, a.cur, a.bb, a.arena_grans, a.list_cap, a.commit_count);
      }
    }
  }
  __syncthreads();
  if (!have) return;
  const unsigned long long pa = s_ba + s_wa[warp] + ia - wa, pb = s_bb + s_wb[warp] + ib - wb;

  // ---- localized descriptor
  const sdb_send_desc w = d;
  sdb_send_desc out = d;
  // absolute address (the fan-out kernel is launched with a null payload base): the payload stays where the source
  // rank exported it - possibly in a peer GPU's memory - and is pulled by the fan-out's TMA loads
  out.payload_off = reinterpret_cast<uint64_t>(a.wire[src]) + s_pay_off[src] + w.payload_off;
  out.gran0 = static_cast<uint32_t>(pa);
  const unsigned long long rb = s_recbase[src];
  out.rec0 = static_cast<uint32_t>(rb + w.rec0);
  const bool abs_seq = s_explicit[src] != 0;
  out.seq_abs = abs_seq ? rb + w.rec0 : 0ull;
  if (w.flags & (SDB_DESC_P2P | SDB_DESC_LIST_TEMP)) {
    uint32_t lo = static_cast<uint32_t>(pb);
    const bool fits = pb + own <= a.list_cap;
    out.mstart = lo; out.mcount = fits ? own : 0u; out.group = SDB_NO_GROUP;
    if (w.flags & SDB_DESC_P2P) {
      out.flags = SDB_DESC_LIST_TEMP | (abs_seq ? SDB_DESC_ABS_SEQ : 0u);
      if (own && fits) a.tmp_list[lo] = w.mstart;
    } else {
      out.flags = SDB_DESC_LIST_TEMP | SDB_DESC_SHARED_SEQ | (abs_seq ? SDB_DESC_ABS_SEQ : 0u);
      if (fits) {
        const uint32_t* l = reinterpret_cast<const uint32_t*>(a.wire[src] + s_list_off[src]) + w.mstart;
        for (uint32_t k = 0; k < w.mcount; ++k) { const uint32_t x = l[k]; if (x < a.max_agents && a.shard_of[x] == a.shard_id) a.tmp_list[lo++] = x; }
      }
    }
  } else {
    const uint32_t g = w.group;
    out.mstart = lc ? a.lstart[g] : 0u;
    out.mcount = lc;
    out.flags = SDB_DESC_SKIP_SENDER | SDB_DESC_PULL | SDB_DESC_POS | (abs_seq ? SDB_DESC_ABS_SEQ : 0u);
  }
  uint4* o4 = reinterpret_cast<uint4*>(a.descs + gi);
  const uint4* i4 = reinterpret_cast<const uint4*>(&out);
  o4[0] = i4[0]; o4[1] = i4[1]; o4[2] = i4[2]; o4[3] = i4[3];
}

// wires / hdr_out (nullable): also copy each source's wire header to hdr_out[i] once the flags are up
extern "C" cudaError_t sdb_launch_wire_wait(const uint32_t* const* flags, uint32_t n, uint32_t step, cudaStream_t stream,
                                            const void* const* wires, sdb_wire_header* hdr_out) {
  sdb_wait_args w{};
  w.n = n; w.hdr_out = wires ? hdr_out : nullptr;
  for (uint32_t i = 0; i < n && i < SDB_MAX_SRC; ++i) { w.flag[i] = flags[i]; w.wire[i] = wires ? static_cast<const uint8_t*>(wires[i]) : nullptr; }
  k_wire_wait<<<1, 32, 0, stream>>>(w, step);
  return cudaGetLastError();
}
extern "C" cudaError_t sdb_launch_wire_set(uint32_t* flag, uint32_t step, cudaStream_t stream) {
  k_wire_set<<<1, 1, 0, stream>>>(flag, step);
  return cudaGetLastError();
}
extern "C" cudaError_t sdb_launch_import_place(const sdb_import_totals* t, sdb_cursor* c, sdb_batch_base* b, unsigned long long G,
                                               uint32_t list_cap, uint32_t* commit_count, cudaStream_t stream) {
  k_import_place<<<1, 32, 0, stream>>>(t, c, b, G, list_cap, commit_count);
  return cudaGetLastError();
}

extern "C" cudaError_t sdb_launch_import_fused(const sdb_import2_args* a, cudaStream_t stream, sdb_profiler* prof, int* n_launches) {
  const uint32_t n_cap = a->n_src * a->max_sends;
  const uint32_t tiles = (n_cap + SDB_IMP_TILE - 1) / SDB_IMP_TILE;
  const int pi = sdb_prof_begin(prof, SDB_PK_XSHARD, stream);
  cudaMemsetAsync(a->lb, 0, sdb_lb_words(tiles) * sizeof(unsigned long long), stream);
  k_import_fused<<<tiles, 256, 0, stream>>>(*a, tiles);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += 1;
  return cudaGetLastError();
}

// any kernel of this file: its module is loaded as a whole before the latency server starts (sdb_api.cu)
extern "C" const void* sdb_xshard_kernel_anchor() { return reinterpret_cast<const void*>(&k_wire_measure); }
