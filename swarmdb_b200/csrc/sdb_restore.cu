// sdb_restore.cu - re-enqueue of records in the compact receive format (sdb_restore_compact), sm_90a.
//
// The input is what a compact receive returns: per listed agent its next count[q] entries, one row + padded payload per
// distinct image.  Every record goes back behind whatever the agent has pending, with its own seq and header fields.
// Arena layout of one call (include/swarmdb_b200.h, sdb_restore_compact): rows in row-index order, each stored as its
// shared headers in entry order + ONE payload (blocks of at most 65535 headers, one payload each, since dm1 is 16
// bits), then the private images (header + payload) in entry order.  An agent's entries are shared up to its first row
// descent; from there on they are private, so arena positions strictly increase along every ring (k_arena_floor relies
// on it).
//
// Plan phase (nothing is written outside scratch):
//   k_restore_plan      8 lanes per agent: ring header once, ring space, entry checks, the first row descent by ballots,
//                       shared entries counted per row, private granules per agent, largest seq, error bits
//   k_restore_rows_gran one thread per row: row checks and the granules of the row's region
//   scans               sdb_scan_u32 (k_scan_local + k_scan_tops) over row counts, row granules and private granules
// The host reads the totals once, reserves the region, then the write phase runs:
//   radix sort          stable LSD sort of the entry indices by row (k_rs_init, then k_rs_hist + scan + k_rs_scatter per
//                       8-bit digit): row r's shared entries land, in entry order, at its bucket base; no atomic order
//   k_restore_headers   one thread per shared entry in sorted order: its rank in the row is its place in the bucket
//   k_restore_payloads  one warp per row: the payload copy behind each block of headers
//   k_restore_ring      8 lanes per agent: private images, ring entries in order, tail = ctail
#include "sdb_common.cuh"

#define SDB_RS_G 8u            // lanes per agent
#define SDB_RS_HDRS 65535u     // headers per payload copy (dm1 = headers - 1 - j must fit 16 bits)

__device__ __forceinline__ uint32_t rs_pg(uint32_t len) { return ((len + 31u) & ~31u) >> 5; }   // payload granules
// row i: {timestamp, payload_off}, {sender, group, len | prio << 16 | type << 24, reserved}
__device__ __forceinline__ void rs_row(const sdb_recv_send* s, uint32_t i, uint4& lo, uint4& hi) {
  const uint4* p = reinterpret_cast<const uint4*>(s + i);
  lo = __ldg(p); hi = __ldg(p + 1);
}

__global__ void __launch_bounds__(256)
k_restore_plan(sdb_dev_view v, sdb_restore_args r) {
  const uint32_t lane = threadIdx.x & 31, l8 = lane & (SDB_RS_G - 1), gsh = lane & ~(SDB_RS_G - 1);
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  constexpr uint32_t SPW = 32u / SDB_RS_G;
  unsigned long long wseq = 0, wrec = 0;
  uint32_t werr = 0;
  for (uint32_t qb = gw * SPW; qb < r.n; qb += nw * SPW) {      // warp-uniform
    const uint32_t q = qb + lane / SDB_RS_G;
    const bool valid = q < r.n;
    uint32_t a = 0, W = 0, e0 = 0;
    if (valid) {
      a = r.agent[q];
      const bool skip = r.owned && r.shard_of[a] != r.shard_id;
      W = skip ? 0u : r.count[q];
      e0 = r.first[q];
      if (W) {
        const uint4 h = *reinterpret_cast<const uint4*>(v.ring_hdr + a);   // one address for the agent's 8 lanes
        if (static_cast<uint64_t>(h.y - h.x) + W > v.ring_slots) werr |= SDB_RS_ERING;
      }
    }
    const uint32_t wmax = __reduce_max_sync(0xFFFFFFFFu, W);
    uint32_t d = r.shared ? W : 0u;                               // first private entry (group-uniform)
    uint32_t carry = 0, pg_sum = 0;
    for (uint32_t j0 = 0; j0 < wmax; j0 += SDB_RS_G) {
      const uint32_t j = j0 + l8;
      const bool in = j < W;
      uint32_t row = 0, len = 0;
      bool row_ok = false;
      if (in) {
        const uint4 e = __ldg(reinterpret_cast<const uint4*>(r.ent + e0 + j));   // {seq lo, seq hi, send, receiver}
        row = e.z;
        row_ok = row < r.n_sends;
        if (!row_ok) werr |= SDB_RS_EINVAL;
        if (e.w != a && e.w != SDB_NO_RECEIVER) werr |= SDB_RS_EINVAL;
        const unsigned long long seq = (static_cast<unsigned long long>(e.y) << 32) | e.x;
        wseq = seq > wseq ? seq : wseq;
        if (row_ok) len = __ldg(reinterpret_cast<const uint32_t*>(r.snd + row) + 6) & 0xFFFFu;
      }
      uint32_t prow = __shfl_up_sync(0xFFFFFFFFu, row, 1, SDB_RS_G);
      if (l8 == 0) prow = carry;
      const bool desc = in && j > 0 && row < prow;
      const uint32_t bm = (__ballot_sync(0xFFFFFFFFu, desc) >> gsh) & 0xFFu;
      if (bm && j0 + __ffs(bm) - 1 < d) d = j0 + __ffs(bm) - 1;
      carry = __shfl_sync(0xFFFFFFFFu, row, SDB_RS_G - 1, SDB_RS_G);
      if (in && row_ok) {
        if (j < d) { r.e_row[e0 + j] = row; atomicAdd(r.row_cnt + row, 1u); }
        else pg_sum += 1u + rs_pg(len);
      }
    }
#pragma unroll
    for (uint32_t o = SDB_RS_G / 2; o; o >>= 1) pg_sum += __shfl_xor_sync(0xFFFFFFFFu, pg_sum, o);
    if (valid && l8 == 0) {
      r.nsh[q] = d < W ? d : W;
      r.pgran[q] = pg_sum;
      wrec += W;
    }
  }
  for (int o = 16; o; o >>= 1) {
    const unsigned long long s2 = __shfl_xor_sync(0xFFFFFFFFu, wseq, o);
    wseq = s2 > wseq ? s2 : wseq;
    wrec += __shfl_xor_sync(0xFFFFFFFFu, wrec, o);
  }
  werr = __reduce_or_sync(0xFFFFFFFFu, werr);
  if (lane == 0) {
    if (wseq) atomicMax(r.tot + 2, wseq);
    if (werr) atomicOr(r.tot + 3, static_cast<unsigned long long>(werr));
    if (wrec) atomicAdd(r.tot + 4, wrec);
  }
}

// every row is checked, referenced or not; row_gran = headers + one payload per block of <= 65535 headers
__global__ void __launch_bounds__(256)
k_restore_rows_gran(sdb_restore_args r) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= r.n_sends) return;
  uint4 lo, hi;
  rs_row(r.snd, i, lo, hi);
  const uint32_t len = hi.z & 0xFFFFu, prio = (hi.z >> 16) & 0xFFu;
  const unsigned long long off = (static_cast<unsigned long long>(lo.w) << 32) | lo.z;
  const uint32_t pg = rs_pg(len);
  if (len > r.max_payload || prio > 3u || (off & 15u) || off > r.payload_bytes || r.payload_bytes - off < (static_cast<uint64_t>(pg) << 5))
    atomicOr(r.tot + 3, SDB_RS_EINVAL);
  const uint32_t n = r.row_cnt[i];
  const uint32_t nb = (n + SDB_RS_HDRS - 1) / SDB_RS_HDRS;
  r.row_gran[i] = n ? n + nb * pg : 0u;
}

__device__ __forceinline__ void rs_write_header(uint8_t* dst, unsigned long long seq, const uint4& lo, const uint4& hi,
                                                uint32_t receiver, uint64_t pol) {
  sdb_st_stream_pol(dst, make_uint4(static_cast<uint32_t>(seq), static_cast<uint32_t>(seq >> 32), lo.x, lo.y), pol);
  sdb_st_stream_pol(dst + 16, make_uint4(hi.x, receiver, hi.y, hi.z), pol);
}

// ---- stable LSD radix sort of the entries by row, 8 bits per pass: tiles of 1024 keys, one warp per tile walking its
// keys 32 at a time in order, so a key's place depends on the keys before it only (deterministic, linear in n)
#define SDB_RS_TILE 1024u

__global__ void __launch_bounds__(256)
k_rs_init(sdb_restore_args r) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= r.n_entries) return;
  const uint32_t row = r.e_row[i];
  r.key_a[i] = row < r.n_sends ? row : r.n_sends;               // private / skipped entries sort behind every row
  r.val_a[i] = i;
}

__global__ void __launch_bounds__(32)
k_rs_hist(const uint32_t* __restrict__ key, uint32_t n, uint32_t shift, uint32_t* __restrict__ hist, uint32_t tiles) {
  __shared__ uint32_t s[256];
  const uint32_t lane = threadIdx.x;
  for (uint32_t d = lane; d < 256; d += 32) s[d] = 0;
  __syncwarp();
  const uint32_t base = blockIdx.x * SDB_RS_TILE;
  for (uint32_t k = 0; k < SDB_RS_TILE; k += 32) {
    const uint32_t i = base + k + lane;
    if (i < n) atomicAdd(s + ((key[i] >> shift) & 255u), 1u);
  }
  __syncwarp();
  for (uint32_t d = lane; d < 256; d += 32) hist[d * tiles + blockIdx.x] = s[d];
}

__global__ void __launch_bounds__(32)
k_rs_scatter(const uint32_t* __restrict__ kin, const uint32_t* __restrict__ vin, uint32_t* __restrict__ kout,
             uint32_t* __restrict__ vout, uint32_t n, uint32_t shift, const uint32_t* __restrict__ hl,
             const uint32_t* __restrict__ ht, uint32_t tiles) {
  __shared__ uint32_t s[256];
  const uint32_t lane = threadIdx.x;
  for (uint32_t d = lane; d < 256; d += 32) s[d] = sdb_scan_at(hl, ht, d * tiles + blockIdx.x);
  __syncwarp();
  const uint32_t base = blockIdx.x * SDB_RS_TILE;
  for (uint32_t k = 0; k < SDB_RS_TILE; k += 32) {
    const uint32_t i = base + k + lane;
    const bool valid = i < n;
    const uint32_t kv = valid ? kin[i] : 0u;
    const uint32_t d = valid ? (kv >> shift) & 255u : 256u + lane;       // invalid lanes match nobody
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, d);
    const uint32_t b = valid ? s[d] : 0u;
    __syncwarp();
    if (valid) {
      const uint32_t at = b + __popc(peers & ((1u << lane) - 1u));
      kout[at] = kv; vout[at] = vin[i];
      if (lane == static_cast<uint32_t>(__ffs(peers)) - 1u) s[d] = b + __popc(peers);
    }
    __syncwarp();
  }
}

// one thread per shared entry, in sorted order: position p of row r's range is the entry's rank in its row (entry
// order), so consecutive threads write consecutive headers of a row block
__global__ void __launch_bounds__(256)
k_restore_headers(sdb_dev_view v, sdb_restore_args r, const uint32_t* __restrict__ sorted, uint32_t n_shared) {
  const uint64_t pol = sdb_policy_evict_first();
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n_shared; p += gridDim.x * blockDim.x) {
    const uint32_t e = sorted[p];
    const uint32_t row = r.e_row[e];
    const uint32_t n = r.row_cnt[row];
    const uint32_t rank = p - sdb_scan_at(r.rc_local, r.rc_tops, row);
    const unsigned long long rb = r.base + sdb_scan_at(r.rg_local, r.rg_tops, row);
    uint4 lo, hi;
    rs_row(r.snd, row, lo, hi);
    const uint32_t pg = rs_pg(hi.z & 0xFFFFu);
    const uint32_t b = rank / SDB_RS_HDRS, jj = rank % SDB_RS_HDRS;
    const uint32_t kb = min(SDB_RS_HDRS, n - b * SDB_RS_HDRS);
    const unsigned long long hpos = rb + static_cast<unsigned long long>(b) * (SDB_RS_HDRS + pg) + jj;
    const uint4 en = __ldg(reinterpret_cast<const uint4*>(r.ent + e));
    rs_write_header(sdb_arena_ptr(v, hpos), (static_cast<unsigned long long>(en.y) << 32) | en.x, lo, hi, en.w, pol);
    r.e_handle[e] = static_cast<uint32_t>(hpos);
    r.e_y[e] = (((hi.z >> 16) & 3u) << 14 | (1u + pg)) | ((kb - 1u - jj) << 16);
  }
}

// one warp per row: the row's payload behind each block of at most 65535 headers
__global__ void __launch_bounds__(256)
k_restore_payloads(sdb_dev_view v, sdb_restore_args r) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint64_t pol = sdb_policy_evict_first();
  for (uint32_t row = gw; row < r.n_sends; row += nw) {
    const uint32_t n = r.row_cnt[row];
    if (n == 0) continue;
    const unsigned long long rb = r.base + sdb_scan_at(r.rg_local, r.rg_tops, row);
    uint4 lo, hi;
    rs_row(r.snd, row, lo, hi);
    const uint32_t pg = rs_pg(hi.z & 0xFFFFu);
    const uint8_t* src = r.payload + ((static_cast<unsigned long long>(lo.w) << 32) | lo.z);
    const uint32_t nb = (n + SDB_RS_HDRS - 1) / SDB_RS_HDRS;
    for (uint32_t b = 0; b < nb; ++b) {
      const uint32_t kb = min(SDB_RS_HDRS, n - b * SDB_RS_HDRS);
      uint8_t* dst = sdb_arena_ptr(v, rb + static_cast<unsigned long long>(b) * (SDB_RS_HDRS + pg) + kb);
      for (uint32_t c = lane; c < 2u * pg; c += 32) sdb_st_stream_pol(dst + (c << 4), sdb_ld_stream(src + (c << 4)), pol);
    }
  }
}

// 8 lanes per agent: entries in order; shared ones take the handle k_restore_headers gave them, private ones are written
// here (a running offset inside the agent's part of the private region, the 8 lanes copy each image together); then the
// ring entries and tail = ctail
__global__ void __launch_bounds__(256)
k_restore_ring(sdb_dev_view v, sdb_restore_args r, unsigned long long priv_base) {
  const uint32_t lane = threadIdx.x & 31, l8 = lane & (SDB_RS_G - 1), gsh = lane & ~(SDB_RS_G - 1);
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint32_t mask = v.ring_slots - 1;
  constexpr uint32_t SPW = 32u / SDB_RS_G;
  const uint64_t pol = sdb_policy_evict_first();
  unsigned long long wrec = 0;
  for (uint32_t qb = gw * SPW; qb < r.n; qb += nw * SPW) {      // warp-uniform
    const uint32_t q = qb + lane / SDB_RS_G;
    const bool valid = q < r.n;
    uint32_t a = 0, W = 0, e0 = 0, nsh = 0, T = 0;
    unsigned long long pbase = 0;
    if (valid) {
      a = r.agent[q];
      const bool skip = r.owned && r.shard_of[a] != r.shard_id;
      W = skip ? 0u : r.count[q];
      e0 = r.first[q];
      nsh = r.nsh[q];
      pbase = priv_base + sdb_scan_at(r.p_local, r.p_tops, q);
      if (W) T = v.ring_hdr[a].tail;
    }
    const uint32_t wmax = __reduce_max_sync(0xFFFFFFFFu, W);
    uint2* rs = sdb_ring_of(v, a);
    uint32_t pcarry = 0;
    for (uint32_t j0 = 0; j0 < wmax; j0 += SDB_RS_G) {
      const uint32_t j = j0 + l8;
      const bool in = j < W;
      const bool priv = in && j >= nsh;
      uint32_t handle = 0, y = 0, g = 0;
      uint4 lo = make_uint4(0, 0, 0, 0), hi = lo, en = lo;
      if (in && !priv) { handle = r.e_handle[e0 + j]; y = r.e_y[e0 + j]; }
      if (priv) {
        en = __ldg(reinterpret_cast<const uint4*>(r.ent + e0 + j));
        rs_row(r.snd, en.z, lo, hi);
        g = 1u + rs_pg(hi.z & 0xFFFFu);
      }
      const uint32_t incl = sdb_warp_incl_scan<SDB_RS_G>(g, l8);
      const unsigned long long apos = pbase + pcarry + incl - g;
      pcarry += __shfl_sync(0xFFFFFFFFu, incl, SDB_RS_G - 1, SDB_RS_G);
      if (priv) {
        handle = static_cast<uint32_t>(apos);
        y = ((hi.z >> 16) & 3u) << 14 | g;
        rs_write_header(sdb_arena_ptr(v, apos), (static_cast<unsigned long long>(en.y) << 32) | en.x, lo, hi, en.w, pol);
      }
      // the group's private payloads, one image at a time, 16-byte chunks spread over the 8 lanes
      const uint32_t pw = __ballot_sync(0xFFFFFFFFu, priv);
      const uint32_t pm = (pw >> gsh) & 0xFFu;
      for (uint32_t k = 0; pw && k < SDB_RS_G; ++k) {            // warp-uniform; skipped when every entry is shared
        const uint32_t src_lane = gsh + k;
        const unsigned long long d = __shfl_sync(0xFFFFFFFFu, apos, src_lane);
        const uint32_t offlo = __shfl_sync(0xFFFFFFFFu, lo.z, src_lane), offhi = __shfl_sync(0xFFFFFFFFu, lo.w, src_lane);
        const uint32_t gk = __shfl_sync(0xFFFFFFFFu, g, src_lane);
        if ((pm >> k) & 1u) {
          const uint8_t* src = r.payload + ((static_cast<unsigned long long>(offhi) << 32) | offlo);
          uint8_t* dst = sdb_arena_ptr(v, d) + 32;
          for (uint32_t c = l8; c < 2u * (gk - 1u); c += SDB_RS_G) sdb_st_stream_pol(dst + (c << 4), sdb_ld_stream(src + (c << 4)), pol);
        }
      }
      if (in) rs[(T + j) & mask] = make_uint2(handle, y);
    }
    if (valid && l8 == 0 && W) {
      v.ring_hdr[a].tail = T + W;
      v.ring_hdr[a].ctail = T + W;
      wrec += W;
    }
  }
  for (int o = 16; o; o >>= 1) wrec += __shfl_xor_sync(0xFFFFFFFFu, wrec, o);
  if (lane == 0 && wrec) atomicAdd(&v.ctr->enqueued, wrec);
}

// plan phase: validation, row counts, the three scans; r->tot ends with the totals the host reads
extern "C" cudaError_t sdb_launch_restore_plan(const sdb_dev_view* v, const sdb_restore_args* r, cudaStream_t stream,
                                               sdb_profiler* prof, int* n_launches, int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_RESTORE, stream);
  cudaMemsetAsync(r->tot, 0, 6 * sizeof(unsigned long long), stream);
  if (r->n_entries) cudaMemsetAsync(r->e_row, 0xFF, static_cast<size_t>(r->n_entries) * sizeof(uint32_t), stream);
  if (r->n_sends) cudaMemsetAsync(r->row_cnt, 0, static_cast<size_t>(r->n_sends) * sizeof(uint32_t), stream);
  int nl = 0;
  if (r->n) { k_restore_plan<<<sdb_grid(r->n, 32, 32 * sm_count), 256, 0, stream>>>(*v, *r); ++nl; }
  if (r->n_sends) { k_restore_rows_gran<<<(r->n_sends + 255) / 256, 256, 0, stream>>>(*r); ++nl; }
  cudaError_t e = sdb_scan_u32(r->row_cnt, r->rc_local, r->rc_tops, r->n_sends, r->tot + 5, nullptr, stream, &nl);
  if (e == cudaSuccess) e = sdb_scan_u32(r->row_gran, r->rg_local, r->rg_tops, r->n_sends, r->tot + 0, nullptr, stream, &nl);
  if (e == cudaSuccess) e = sdb_scan_u32(r->pgran, r->p_local, r->p_tops, r->n, r->tot + 1, nullptr, stream, &nl);
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// write phase: r->base is the reserved region, rows first, then `row_grans` later the private images; n_shared entries
// are shared (the scan total of the row counts)
extern "C" cudaError_t sdb_launch_restore_write(const sdb_dev_view* v, const sdb_restore_args* r, unsigned long long row_grans,
                                                uint32_t n_shared, cudaStream_t stream, sdb_profiler* prof, int* n_launches,
                                                int sm_count) {
  const int pi = sdb_prof_begin(prof, SDB_PK_RESTORE, stream);
  int nl = 0;
  cudaError_t e = cudaSuccess;
  if (n_shared) {
    k_rs_init<<<(r->n_entries + 255) / 256, 256, 0, stream>>>(*r);
    ++nl;
    uint32_t *ks = nullptr, *vs = nullptr;                               // keys are 0 .. n_sends
    e = sdb_radix_sort_u32(r->key_a, r->val_a, r->key_b, r->val_b, r->n_entries, sdb_key_bits(r->n_sends), r->hist, r->h_local,
                           r->h_tops, &ks, &vs, stream, &nl);
    k_restore_headers<<<sdb_grid(n_shared, 256, 32 * sm_count), 256, 0, stream>>>(*v, *r, vs, n_shared);
    k_restore_payloads<<<sdb_grid(r->n_sends, 8, 32 * sm_count), 256, 0, stream>>>(*v, *r);
    nl += 2;
  }
  if (r->n) { k_restore_ring<<<sdb_grid(r->n, 32, 32 * sm_count), 256, 0, stream>>>(*v, *r, r->base + row_grans); ++nl; }
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches += nl;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// The radix sort above, for the restore and the lease sweep: stable sort of n (key, value) pairs by the low `bits` bits of
// the keys.  hist / h_local take 256 x ceil(n / 1024) words, h_tops that / 4096 + 1.  *kres / *vres name the buffers
// holding the result: the a pair or the b pair.
extern "C" cudaError_t sdb_radix_sort_u32(uint32_t* ka, uint32_t* va, uint32_t* kb, uint32_t* vb, uint32_t n, uint32_t bits,
                                          uint32_t* hist, uint32_t* h_local, uint32_t* h_tops, uint32_t** kres, uint32_t** vres,
                                          cudaStream_t stream, int* n_launches) {
  uint32_t *kin = ka, *vin = va, *kout = kb, *vout = vb;
  cudaError_t e = cudaSuccess;
  const uint32_t tiles = (n + SDB_RS_TILE - 1) / SDB_RS_TILE;
  int nl = 0;
  for (uint32_t shift = 0; n && shift < bits && e == cudaSuccess; shift += 8) {
    k_rs_hist<<<tiles, 32, 0, stream>>>(kin, n, shift, hist, tiles);
    e = sdb_scan_u32(hist, h_local, h_tops, 256u * tiles, nullptr, nullptr, stream, &nl);
    k_rs_scatter<<<tiles, 32, 0, stream>>>(kin, vin, kout, vout, n, shift, h_local, h_tops, tiles);
    nl += 2;
    uint32_t* t = kin; kin = kout; kout = t;
    t = vin; vin = vout; vout = t;
  }
  *kres = kin; *vres = vin;
  if (n_launches) *n_launches += nl;
  return e == cudaSuccess ? cudaGetLastError() : e;
}

// any kernel of this file: its module is loaded as a whole before the latency server starts (sdb_api.cu)
extern "C" const void* sdb_restore_kernel_anchor() { return reinterpret_cast<const void*>(&k_restore_plan); }
