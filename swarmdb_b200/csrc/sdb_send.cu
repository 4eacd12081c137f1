// sdb_send.cu - enqueue kernels (sm_90a).
//
//   k_enqueue_p2p     K1: send_message      (reference M:393-519, produce M:476-482)
//   k_group_fanout    K2: send_to_group     (reference M:1229-1279, the per-member loop M:1267-1277)
//                         and broadcast lists (M:449-463 / M:810-850)
//   k_commit          publishes a batch: sorts each agent's newly claimed ring entries into
//                     arena (= global send) order and clamps overflowed rings
//                     (role of the delivery report, M:374-391: PENDING -> DELIVERED)
//
// Roofline: all three are pure data movement (HBM-bound).  Algorithmic bytes per routed
// message for K2 at L=256, H=16 essential header bytes, F=64: (L+H) written + 4 member id
// read + (L+H)/F source read = 280.25 B (SURVEY 8d); the kernel physically writes a 32-byte
// header (288 B/record) plus 6 B of ring entry.
#include <cstdlib>

#include "sdb_common.cuh"

namespace {

__device__ __forceinline__ sdb_send_desc load_desc(const sdb_send_desc* p) {
  // 64-byte descriptor, same address for the whole CTA -> L1 broadcast
  const uint4* q = reinterpret_cast<const uint4*>(p);
  union { uint4 v[4]; sdb_send_desc d; } u;
  u.v[0] = __ldg(q); u.v[1] = __ldg(q + 1); u.v[2] = __ldg(q + 2); u.v[3] = __ldg(q + 3);
  return u.d;
}

// zero the pad bytes [len, padlen) of a staged payload so arena contents are deterministic
__device__ __forceinline__ void zero_pad(uint8_t* s_payload, uint32_t len, uint32_t padlen, uint32_t tid) {
  uint32_t b = len + tid;
  if (tid < 32 && b < padlen) s_payload[b] = 0;
}

}  // namespace

// ------------------------------------------------------------------------------------------
// K2 (variant A): one CTA per send, payload staged once in shared memory by a TMA bulk load,
// then every member's copy is written with coalesced 16-byte streaming stores.
// Thread j of a 256-member tile owns member j: builds its 32-byte header, stores it and
// claims the ring slot; the 8 warps then stream the payload copies (warp w -> members w, w+8, ..).
// ------------------------------------------------------------------------------------------
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
k_group_fanout_st(sdb_dev_view v, const sdb_send_desc* __restrict__ descs, uint32_t n,
                  const uint8_t* __restrict__ payload, const uint32_t* __restrict__ tmp_list,
                  uint64_t seq_base, uint64_t arena_base) {
  extern __shared__ __align__(128) uint8_t s_payload[];
  __shared__ __align__(8) uint64_t s_bar;
  __shared__ uint32_t s_deliver[THREADS / 32];
  constexpr int NW = THREADS / 32;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid == 0) { sdb_mbar_init(&s_bar, 1); sdb_fence_barrier_init(); }
  __syncthreads();
  uint32_t phase = 0;
  uint32_t n_enq = 0, n_ovf = 0, n_skip = 0;

  for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
    const sdb_send_desc d = load_desc(descs + i);
    if (d.mcount == 0) continue;                       // nobody to deliver to (uniform across the CTA)
    const uint32_t padlen = (d.rgran - 1u) * SDB_GRANULE;
    if (tid == 0 && padlen) {
      sdb_mbar_expect_tx(&s_bar, padlen);
      sdb_tma_load(s_payload, payload + d.payload_off, padlen, &s_bar);
    }
    const uint32_t* mem = (d.flags & SDB_DESC_LIST_TEMP) ? tmp_list + d.mstart : v.members + d.mstart;
    const uint16_t meta = static_cast<uint16_t>((static_cast<uint32_t>(d.prio) << 14) | d.rgran);
    const uint64_t apos0 = arena_base + d.gran0;

    for (uint32_t tile = 0; tile < d.mcount; tile += THREADS) {
      const uint32_t j = tile + tid;
      const bool valid = j < d.mcount;
      const uint32_t a = valid ? __ldg(mem + j) : 0xFFFFFFFFu;
      const bool skip = valid && (d.flags & SDB_DESC_SKIP_SENDER) && a == d.sender;
      const bool deliver = valid && !skip && a < v.max_agents;
      const uint32_t bal = __ballot_sync(0xFFFFFFFFu, deliver);
      if (lane == 0) s_deliver[warp] = bal;
      if (deliver) {
        const uint64_t apos = apos0 + static_cast<uint64_t>(j) * d.rgran;
        const uint32_t pj = (d.flags & SDB_DESC_POS) ? __ldg(v.member_pos + d.mstart + j) : j;
        const uint64_t seq = ((d.flags & SDB_DESC_ABS_SEQ) ? d.seq_abs : seq_base + d.rec0) + ((d.flags & SDB_DESC_SHARED_SEQ) ? 0u : pj);
        const uint32_t rcv = (d.flags & SDB_DESC_SHARED_SEQ) ? SDB_NO_RECEIVER : a;
        uint4* dst = reinterpret_cast<uint4*>(sdb_arena_ptr(v, apos));
        sdb_st_stream(dst, sdb_header_lo(seq, d.timestamp));
        sdb_st_stream(dst + 1, sdb_header_hi(d.sender, rcv, d.group, d.len, d.prio, d.type));
        if (!(d.flags & SDB_DESC_PULL)) { if (sdb_ring_append(v, a, static_cast<uint32_t>(apos), meta)) ++n_enq; else ++n_ovf; }
      }
      n_skip += skip;
      if (tile == 0 && padlen) {
        sdb_mbar_wait(&s_bar, phase);
        zero_pad(s_payload, d.len, padlen, tid);
      }
      __syncthreads();
      const uint32_t in_tile = min(static_cast<uint32_t>(THREADS), d.mcount - tile);
      const uint32_t nchunk = padlen >> 4;
      for (uint32_t jj = warp; jj < in_tile; jj += NW) {
        if (!((s_deliver[jj >> 5] >> (jj & 31)) & 1u)) continue;
        uint8_t* dst = sdb_arena_ptr(v, apos0 + static_cast<uint64_t>(tile + jj) * d.rgran) + 32;
        for (uint32_t c = lane; c < nchunk; c += 32)
          sdb_st_stream(dst + (c << 4), reinterpret_cast<const uint4*>(s_payload)[c]);
      }
      __syncthreads();
    }
    if (padlen) phase ^= 1;
  }
  // one atomic per warp for the counters
  for (int o = 16; o; o >>= 1) {
    n_enq += __shfl_xor_sync(0xFFFFFFFFu, n_enq, o);
    n_ovf += __shfl_xor_sync(0xFFFFFFFFu, n_ovf, o);
    n_skip += __shfl_xor_sync(0xFFFFFFFFu, n_skip, o);
  }
  if (lane == 0) {
    if (n_enq) atomicAdd(&v.ctr->enqueued, n_enq);
    if (n_ovf) atomicAdd(&v.ctr->ring_overflow, n_ovf);
    if (n_skip) atomicAdd(&v.ctr->skipped_sender, n_skip);
  }
}

// ------------------------------------------------------------------------------------------
// K2 (variant B): TMA in, TMA out.  One small CTA (64 threads) per send; the payload is
// bulk-loaded into one of two shared-memory stages, and thread j issues ONE bulk store
// (cp.async.bulk.global.shared::cta) of the whole padded payload into member j's record,
// after writing that record's 32-byte header with two vector stores and claiming the ring
// slot.  No per-chunk store instructions: the LSU only sees headers, ring entries and atomics.
// ------------------------------------------------------------------------------------------
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
k_group_fanout_tma(sdb_dev_view v, const sdb_send_desc* __restrict__ descs, uint32_t n,
                   const uint8_t* __restrict__ payload, const uint32_t* __restrict__ tmp_list,
                   uint64_t seq_base, uint64_t arena_base, uint32_t stage_bytes) {
  extern __shared__ __align__(128) uint8_t s_stage[];   // 2 stages of stage_bytes
  __shared__ __align__(8) uint64_t s_bar[2];
  const uint32_t tid = threadIdx.x, lane = tid & 31;

  if (tid == 0) { sdb_mbar_init(&s_bar[0], 1); sdb_mbar_init(&s_bar[1], 1); sdb_fence_barrier_init(); }
  __syncthreads();
  uint32_t phase[2] = {0, 0};
  uint32_t n_enq = 0, n_ovf = 0, n_skip = 0;

  // prologue: prefetch the first send's payload into stage 0
  uint32_t i = blockIdx.x;
  if (i < n && tid == 0) {
    const sdb_send_desc d0 = load_desc(descs + i);
    const uint32_t pl = (d0.rgran - 1u) * SDB_GRANULE;
    if (pl) { sdb_mbar_expect_tx(&s_bar[0], pl); sdb_tma_load(s_stage, payload + d0.payload_off, pl, &s_bar[0]); }
  }
  uint32_t st = 0;
  for (; i < n; i += gridDim.x, st ^= 1) {
    const sdb_send_desc d = load_desc(descs + i);
    const uint32_t padlen = (d.rgran - 1u) * SDB_GRANULE;
    uint8_t* s_payload = s_stage + st * stage_bytes;
    // prefetch the next send into the other stage; its previous bulk stores must have
    // finished READING that stage (every issuing thread waits on its own bulk groups)
    sdb_tma_wait_read<0>();
    __syncthreads();
    const uint32_t inext = i + gridDim.x;
    if (inext < n && tid == 0) {
      const sdb_send_desc dn = load_desc(descs + inext);
      const uint32_t pl = (dn.rgran - 1u) * SDB_GRANULE;
      if (pl) {
        sdb_mbar_expect_tx(&s_bar[st ^ 1], pl);
        sdb_tma_load(s_stage + (st ^ 1) * stage_bytes, payload + dn.payload_off, pl, &s_bar[st ^ 1]);
      }
    }
    if (padlen) {
      sdb_mbar_wait(&s_bar[st], phase[st]);
      phase[st] ^= 1;
      zero_pad(s_payload, d.len, padlen, tid);
      sdb_fence_proxy_async();        // generic-proxy writes (pad zeroing) -> visible to the bulk store
      __syncthreads();
    }
    const uint32_t* mem = (d.flags & SDB_DESC_LIST_TEMP) ? tmp_list + d.mstart : v.members + d.mstart;
    const uint16_t meta = static_cast<uint16_t>((static_cast<uint32_t>(d.prio) << 14) | d.rgran);
    const uint64_t apos0 = arena_base + d.gran0;
    for (uint32_t j = tid; j < d.mcount; j += THREADS) {
      const uint32_t a = __ldg(mem + j);
      const bool skip = (d.flags & SDB_DESC_SKIP_SENDER) && a == d.sender;
      n_skip += skip;
      if (skip || a >= v.max_agents) continue;
      const uint64_t apos = apos0 + static_cast<uint64_t>(j) * d.rgran;
      const uint32_t pj = (d.flags & SDB_DESC_POS) ? __ldg(v.member_pos + d.mstart + j) : j;
      const uint64_t seq = ((d.flags & SDB_DESC_ABS_SEQ) ? d.seq_abs : seq_base + d.rec0) + ((d.flags & SDB_DESC_SHARED_SEQ) ? 0u : pj);
      const uint32_t rcv = (d.flags & SDB_DESC_SHARED_SEQ) ? SDB_NO_RECEIVER : a;
      uint8_t* rec = sdb_arena_ptr(v, apos);
      if (padlen) sdb_tma_store(rec + 32, s_payload, padlen);
      sdb_st_stream(rec, sdb_header_lo(seq, d.timestamp));
      sdb_st_stream(rec + 16, sdb_header_hi(d.sender, rcv, d.group, d.len, d.prio, d.type));
      if (!(d.flags & SDB_DESC_PULL)) { if (sdb_ring_append(v, a, static_cast<uint32_t>(apos), meta)) ++n_enq; else ++n_ovf; }
    }
    sdb_tma_commit();
  }
  sdb_tma_wait_all<0>();
  for (int o = 16; o; o >>= 1) {
    n_enq += __shfl_xor_sync(0xFFFFFFFFu, n_enq, o);
    n_ovf += __shfl_xor_sync(0xFFFFFFFFu, n_ovf, o);
    n_skip += __shfl_xor_sync(0xFFFFFFFFu, n_skip, o);
  }
  if (lane == 0) {
    if (n_enq) atomicAdd(&v.ctr->enqueued, n_enq);
    if (n_ovf) atomicAdd(&v.ctr->ring_overflow, n_ovf);
    if (n_skip) atomicAdd(&v.ctr->skipped_sender, n_skip);
  }
}

// ------------------------------------------------------------------------------------------
// K2 (variant C, default): one WARP per send, no block-wide barriers.
//   lane 0 issues ONE TMA bulk load of the padded payload into this warp's shared-memory stage
//   (completion on a per-warp mbarrier); while it is in flight the 32 lanes fetch the member ids
//   (2 per lane per 64-member tile), claim ring slots (one 64-bit atomic each) and write the
//   32-byte record headers; then the warp streams the payload copies with fully coalesced
//   16-byte stores, walking the (record, chunk) space flat so all 32 lanes stay busy for any
//   payload size.  When the chunk count divides 32 the lane's chunk never changes and is held in
//   a register.  ~3 warp-instructions per routed message instead of ~75 for variant A.
// ------------------------------------------------------------------------------------------
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 6)
k_group_fanout_warp(sdb_dev_view v, const sdb_send_desc* __restrict__ descs, uint32_t n,
                    const uint8_t* __restrict__ payload, const uint32_t* __restrict__ tmp_list,
                    uint64_t seq_base, uint64_t arena_base, uint32_t stage_bytes) {
  extern __shared__ __align__(128) uint8_t s_stage[];      // WARPS x 2 stages of stage_bytes
  __shared__ __align__(8) uint64_t s_bar[WARPS][2];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* const my_base = s_stage + static_cast<size_t>(warp) * 2u * stage_bytes;
  if (lane == 0) { sdb_mbar_init(&s_bar[warp][0], 1); sdb_mbar_init(&s_bar[warp][1], 1); sdb_fence_barrier_init(); }
  __syncwarp();
  uint32_t phase0 = 0, phase1 = 0;
  uint32_t n_enq = 0, n_ovf = 0, n_skip = 0;
  const uint32_t gw = blockIdx.x * WARPS + warp, nw = gridDim.x * WARPS;
  const uint64_t pol_stream = sdb_policy_evict_first();

  // two-stage software pipeline per warp: while send i is being written out, the descriptor of
  // send i + nw is already loaded and its payload is in flight (TMA) into the other stage - the
  // payload may live in a peer GPU's memory (cross-shard import reads it over NVLink)
  uint32_t i = gw, st = 0;
  bool have = i < n;
  sdb_send_desc d;
  uint32_t pa0 = 0xFFFFFFFFu, pa1 = 0xFFFFFFFFu, pp0 = 0, pp1 = 0;      // first-tile members of the current send
  uint32_t pc_c = 0, q32_c = 0, r32_c = 0, rec_c = 0, ch_c = 0;         // cached (record, chunk) walk parameters
  auto member_list = [&](const sdb_send_desc& x) { return (x.flags & SDB_DESC_LIST_TEMP) ? tmp_list + x.mstart : v.members + x.mstart; };
  auto fetch_members = [&](const sdb_send_desc& x, uint32_t& a0, uint32_t& a1, uint32_t& q0, uint32_t& q1) {
    const uint32_t* m = member_list(x);
    const uint32_t j0 = lane, j1 = lane + 32;
    a0 = j0 < x.mcount ? __ldg(m + j0) : 0xFFFFFFFFu;
    a1 = j1 < x.mcount ? __ldg(m + j1) : 0xFFFFFFFFu;
    if (x.flags & SDB_DESC_POS) {
      const uint32_t* mp = v.member_pos + x.mstart;
      q0 = j0 < x.mcount ? __ldg(mp + j0) : 0u; q1 = j1 < x.mcount ? __ldg(mp + j1) : 0u;
    } else { q0 = j0; q1 = j1; }
  };
  if (have) {
    d = load_desc(descs + i);
    const uint32_t pl = (d.rgran - 1u) * SDB_GRANULE;
    if (lane == 0 && d.mcount && pl) { sdb_mbar_expect_tx(&s_bar[warp][0], pl); sdb_tma_load(my_base, payload + d.payload_off, pl, &s_bar[warp][0]); }
    fetch_members(d, pa0, pa1, pp0, pp1);
  }
  while (have) {
    const uint32_t inext = i + nw;
    const bool have_next = inext < n;
    sdb_send_desc dn;
    uint32_t na0 = 0xFFFFFFFFu, na1 = 0xFFFFFFFFu, np0 = 0, np1 = 0;
    if (have_next) {
      dn = load_desc(descs + inext);
      const uint32_t pl = (dn.rgran - 1u) * SDB_GRANULE;
      if (lane == 0 && dn.mcount && pl) {
        uint8_t* dst = my_base + (st ^ 1u) * stage_bytes;
        sdb_mbar_expect_tx(&s_bar[warp][st ^ 1u], pl);
        sdb_tma_load(dst, payload + dn.payload_off, pl, &s_bar[warp][st ^ 1u]);
      }
      fetch_members(dn, na0, na1, np0, np1);                           // member ids of the next send, in flight with its payload
    }
    uint8_t* const my = my_base + st * stage_bytes;
    const uint4* const my4 = reinterpret_cast<const uint4*>(my);
    const uint32_t padlen = (d.rgran - 1u) * SDB_GRANULE;
    const uint32_t P = padlen >> 4;                        // 16-byte chunks per payload
    const uint32_t* mem = member_list(d);
    const uint16_t meta = static_cast<uint16_t>((static_cast<uint32_t>(d.prio) << 14) | d.rgran);
    const uint64_t apos0 = arena_base + d.gran0;
    uint8_t* const base = sdb_arena_ptr(v, apos0);         // the batch region never wraps: plain pointer math below
    const uint32_t rbytes = d.rgran * SDB_GRANULE;
    const bool shared_seq = (d.flags & SDB_DESC_SHARED_SEQ) != 0;
    const bool skip_sender = (d.flags & SDB_DESC_SKIP_SENDER) != 0;
    const bool pull = (d.flags & SDB_DESC_PULL) != 0;
    const uint32_t* mpos = (d.flags & SDB_DESC_POS) ? v.member_pos + d.mstart : nullptr;

    for (uint32_t tile = 0; tile < d.mcount; tile += 64) {
      const uint32_t j0 = tile + lane, j1 = j0 + 32;
      uint32_t a0, a1, p0, p1;                               // member ids and their sequence offsets (group positions)
      if (tile == 0) { a0 = pa0; a1 = pa1; p0 = pp0; p1 = pp1; }
      else {
        a0 = j0 < d.mcount ? __ldg(mem + j0) : 0xFFFFFFFFu;
        a1 = j1 < d.mcount ? __ldg(mem + j1) : 0xFFFFFFFFu;
        p0 = mpos ? (j0 < d.mcount ? __ldg(mpos + j0) : 0u) : j0;
        p1 = mpos ? (j1 < d.mcount ? __ldg(mpos + j1) : 0u) : j1;
      }
      const bool s0 = j0 < d.mcount && skip_sender && a0 == d.sender;
      const bool s1 = j1 < d.mcount && skip_sender && a1 == d.sender;
      const bool d0 = j0 < d.mcount && !s0 && a0 < v.max_agents;
      const bool d1 = j1 < d.mcount && !s1 && a1 < v.max_agents;
      n_skip += s0 + s1;
      if (!pull) {            // small / non-group batches: claim ring slots here (sorted later by k_commit)
        if (d0) { if (sdb_ring_append(v, a0, static_cast<uint32_t>(apos0 + static_cast<uint64_t>(j0) * d.rgran), meta)) ++n_enq; else ++n_ovf; }
        if (d1) { if (sdb_ring_append(v, a1, static_cast<uint32_t>(apos0 + static_cast<uint64_t>(j1) * d.rgran), meta)) ++n_enq; else ++n_ovf; }
      }
      const uint32_t m0 = __ballot_sync(0xFFFFFFFFu, d0), m1 = __ballot_sync(0xFFFFFFFFu, d1);
      if (tile == 0 && padlen) {
        sdb_mbar_wait(&s_bar[warp][st], st ? phase1 : phase0);
        if (st) phase1 ^= 1; else phase0 ^= 1;
        if (d.len + lane < padlen) my[d.len + lane] = 0;   // deterministic pad bytes
        __syncwarp();
      }
      // flat walk over (record, chunk): PC = 2 header chunks + P payload chunks per record, so every
      // warp store instruction covers 512 contiguous bytes of the send's region
      const uint32_t nrec = min(64u, d.mcount - tile);
      const uint32_t PC = P + 2u;
      const uint32_t total = nrec * PC;
      if (PC != pc_c) {                                     // the divisions are redone only when the record size changes
        pc_c = PC; q32_c = 32u / PC; r32_c = 32u % PC; rec_c = lane / PC; ch_c = lane % PC;
      }
      const uint32_t q32 = q32_c, r32 = r32_c;
      uint32_t rec = rec_c, ch = ch_c;
      uint8_t* const tb = base + static_cast<size_t>(tile) * rbytes;
      const uint64_t seq0 = (d.flags & SDB_DESC_ABS_SEQ) ? d.seq_abs : seq_base + d.rec0;
      const uint4 hdr_hi = sdb_header_hi(d.sender, SDB_NO_RECEIVER, d.group, d.len, d.prio, d.type);
      // record j occupies chunks [j*PC, (j+1)*PC) of the send's region, so flat chunk f lands at tb + 16 f
      uint8_t* dst = tb + (static_cast<size_t>(lane) << 4);
      const bool all_in = (nrec <= 32u) ? (m0 == (nrec == 32u ? 0xFFFFFFFFu : ((1u << nrec) - 1u)))
                                        : (m0 == 0xFFFFFFFFu && m1 == (nrec == 64u ? 0xFFFFFFFFu : ((1u << (nrec - 32u)) - 1u)));
      if (nrec <= 32u) {
        // narrow sends (few local members, e.g. one shard's share of a group): one shuffle pair per step
        for (uint32_t done = 0; done < total; done += 32, dst += 512) {
          const uint32_t src = rec & 31u;
          const uint32_t ra = __shfl_sync(0xFFFFFFFFu, a0, src), rp = __shfl_sync(0xFFFFFFFFu, p0, src);
          if (rec < nrec && (all_in || ((m0 >> src) & 1u))) {
            uint4 x;
            if (ch >= 2u) x = my4[ch - 2u];
            else if (ch == 0) x = sdb_header_lo(seq0 + (shared_seq ? 0u : rp), d.timestamp);
            else { x = hdr_hi; if (!shared_seq) x.y = ra; }
            sdb_st_stream_pol(dst, x, pol_stream);
          }
          ch += r32; rec += q32;
          if (ch >= PC) { ch -= PC; ++rec; }
        }
      } else {
        for (uint32_t done = 0; done < total; done += 32, dst += 512) {
          const uint32_t src = rec & 31u;
          const uint32_t ra0 = __shfl_sync(0xFFFFFFFFu, a0, src), ra1 = __shfl_sync(0xFFFFFFFFu, a1, src);
          const uint32_t rp0 = __shfl_sync(0xFFFFFFFFu, p0, src), rp1 = __shfl_sync(0xFFFFFFFFu, p1, src);
          const bool lo_half = rec < 32u;
          if (rec < nrec && (all_in || (((lo_half ? m0 : m1) >> src) & 1u))) {
            uint4 x;
            if (ch >= 2u) x = my4[ch - 2u];
            else if (ch == 0) x = sdb_header_lo(seq0 + (shared_seq ? 0u : (lo_half ? rp0 : rp1)), d.timestamp);
            else { x = hdr_hi; if (!shared_seq) x.y = lo_half ? ra0 : ra1; }
            sdb_st_stream_pol(dst, x, pol_stream);
          }
          ch += r32; rec += q32;
          if (ch >= PC) { ch -= PC; ++rec; }
        }
      }
      __syncwarp();
    }
    d = dn; i = inext; have = have_next; st ^= 1u;
    pa0 = na0; pa1 = na1; pp0 = np0; pp1 = np1;
  }
  for (int o = 16; o; o >>= 1) {
    n_enq += __shfl_xor_sync(0xFFFFFFFFu, n_enq, o);
    n_ovf += __shfl_xor_sync(0xFFFFFFFFu, n_ovf, o);
    n_skip += __shfl_xor_sync(0xFFFFFFFFu, n_skip, o);
  }
  if (lane == 0) {
    if (n_enq) atomicAdd(&v.ctr->enqueued, n_enq);
    if (n_ovf) atomicAdd(&v.ctr->ring_overflow, n_ovf);
    if (n_skip) atomicAdd(&v.ctr->skipped_sender, n_skip);
  }
}

// ------------------------------------------------------------------------------------------
// K2, variant D ("span"): for batches of many small sends (a shard's share of a group at N = 8
// is ~8 records; payloads up to 512 bytes), where variant C's ~400 warp-instructions of per-send
// bookkeeping - not HBM - set the pace.  Two ideas:
//   * everything a send needs arrives through shared-memory rings filled by TMA well ahead of
//     its use: a 16-deep descriptor ring and an 8-deep payload ring per warp, refilled FOUR sends
//     at a time by four lanes in parallel.  5-8 payloads are in flight per warp, which covers the
//     NVLink round trip when the wire batch lives in a peer GPU, and no descriptor field is held
//     in registers across iterations;
//   * the unit of work is a TILE of up to 32 records that may span several sends (whole sends of
//     one refill group, or 32 members of a wide send).  Lane r prepares record r - descriptor
//     fields, member id, ring claim, the 32-byte header, destination - IN PARALLEL and parks it in
//     a per-warp table; the copy loop then walks the tile's 16-byte chunks flat, one LDS.128 for
//     the table entry, one for the data (header table or staged payload), one STG.128.  The
//     per-send scalar work of variant C becomes per-tile SIMD work.
// The next tile's plan and member ids are computed/loaded while the current tile is written.
// Output bytes are identical to variants A-C.
// ------------------------------------------------------------------------------------------
constexpr uint32_t SDB_SPAN_PAY = 8, SDB_SPAN_DESC = 16, SDB_SPAN_GROUP = 4;
constexpr uint32_t SDB_SPAN_TABLES = 32 * 32 + 32 * 16;          // header table + record table, bytes per warp

__device__ __forceinline__ uint4 sdb_lds128(uint32_t saddr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(saddr) : "memory");
  return r;
}
__device__ __forceinline__ uint32_t sdb_lds32(uint32_t saddr) {
  uint32_t r;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r) : "r"(saddr) : "memory");
  return r;
}

template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 8)
k_group_fanout_span(sdb_dev_view v, const sdb_send_desc* __restrict__ descs, uint32_t n,
                    const uint8_t* __restrict__ payload, const uint32_t* __restrict__ tmp_list,
                    uint64_t seq_base, uint64_t arena_base, uint32_t stage_bytes, const sdb_batch_base* __restrict__ bb,
                    uint32_t skip_pull) {
  // skip_pull: the group sends of this batch (SDB_DESC_PULL) are written by k_group_fanout_shared; only point-to-point
  // and broadcast descriptors are served here - usually none (the import's totals say so: return at once)
  if (bb) {                                                  // asynchronous import: placement computed on the device
    if (bb->skip || (skip_pull && bb->n_other == 0)) return;
    n = bb->n_total; seq_base = bb->seq_base; arena_base = bb->arena_base;
  }
  auto mcnt = [&](const sdb_send_desc& x) -> uint32_t { return (skip_pull && (x.flags & SDB_DESC_PULL)) ? 0u : x.mcount; };
  constexpr uint32_t PAY = SDB_SPAN_PAY, DESC = SDB_SPAN_DESC, GROUP = SDB_SPAN_GROUP, NONE = 0xFFFFFFFFu;
  static_assert(DESC == 4 * GROUP && PAY == 2 * GROUP, "refill schedule below assumes these distances");
  extern __shared__ __align__(128) uint8_t s_dyn[];          // per warp: descriptors | header table | record table | payload stages
  __shared__ __align__(8) uint64_t s_dbar[WARPS][DESC];
  __shared__ __align__(8) uint64_t s_pbar[WARPS][PAY];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t per_warp = DESC * sizeof(sdb_send_desc) + SDB_SPAN_TABLES + static_cast<size_t>(PAY) * stage_bytes;
  uint8_t* const wbase = s_dyn + warp * per_warp;
  const sdb_send_desc* const s_desc = reinterpret_cast<const sdb_send_desc*>(wbase);
  uint4* const s_hdr = reinterpret_cast<uint4*>(wbase + DESC * sizeof(sdb_send_desc));            // [32][2]
  uint4* const s_rec = s_hdr + 64;                                                                  // [32] {dst lo, dst hi, payload smem addr, chunks}
  uint8_t* const s_pay = wbase + DESC * sizeof(sdb_send_desc) + SDB_SPAN_TABLES;
  const uint32_t hdr_sa = sdb_smem_u32(s_hdr), rec_sa = sdb_smem_u32(s_rec), pay_sa = sdb_smem_u32(s_pay);
  if (lane < DESC) sdb_mbar_init(&s_dbar[warp][lane], 1);
  if (lane < PAY) sdb_mbar_init(&s_pbar[warp][lane], 1);
  sdb_fence_barrier_init();
  __syncwarp();
  const uint32_t gw = blockIdx.x * WARPS + warp, nw = gridDim.x * WARPS;
  const uint64_t pol_stream = sdb_policy_evict_first();
  uint32_t n_enq = 0, n_ovf = 0, n_skip = 0;
  if (gw >= n) return;
  const uint32_t mine = (n - gw + nw - 1) / nw;              // sends this warp handles: gw, gw + nw, ...

  auto want_desc = [&](uint32_t t) {                         // one lane: request descriptor t into its ring slot
    uint64_t* bar = &s_dbar[warp][t & (DESC - 1)];
    sdb_mbar_expect_tx(bar, sizeof(sdb_send_desc));
    sdb_tma_load(wbase + (t & (DESC - 1)) * sizeof(sdb_send_desc), descs + (gw + static_cast<size_t>(t) * nw), sizeof(sdb_send_desc), bar);
  };
  auto wait_desc = [&](uint32_t t) { sdb_mbar_wait_bounded(&s_dbar[warp][t & (DESC - 1)], (t / DESC) & 1u); };
  auto want_payload = [&](uint32_t t) {                      // one lane: descriptor t is in shared memory
    const sdb_send_desc& x = s_desc[t & (DESC - 1)];
    const uint32_t pl = (x.rgran - 1u) * SDB_GRANULE;
    if (mcnt(x) && pl) {
      uint64_t* bar = &s_pbar[warp][t & (PAY - 1)];
      sdb_mbar_expect_tx(bar, pl);
      sdb_tma_load(s_pay + (t & (PAY - 1)) * static_cast<size_t>(stage_bytes), payload + x.payload_off, pl, bar);
    }
  };

  // ---- tile plan: (t, joff) uniform -> this lane's record (send ts, member j), the tile's record count, the next tile's start
  uint32_t ts, j, a = NONE, q = 0, nrec, t_next, joff_next;
  auto plan = [&](uint32_t t, uint32_t joff) {
    ts = NONE; j = 0; nrec = 0; a = NONE; q = 0;
    if (t >= mine) { t_next = t; joff_next = 0; return; }
    const uint32_t gend = min((t & ~(GROUP - 1)) + GROUP, mine);
    if ((t & (GROUP - 1)) == 0 && joff == 0)                  // first tile of a refill group: its descriptors were requested >= 8 sends ago
      for (uint32_t u = t; u < gend; ++u) wait_desc(u);
    uint32_t tt = t;
    const uint32_t rem = mcnt(s_desc[tt & (DESC - 1)]) - joff;
    if (rem > 32u) { ts = tt; j = joff + lane; nrec = 32u; t_next = tt; joff_next = joff + 32u; }
    else {
      if (lane < rem) { ts = tt; j = joff + lane; }
      nrec = rem; ++tt;
      while (tt < gend) {                                    // whole following sends of the group while they fit
        const uint32_t m = mcnt(s_desc[tt & (DESC - 1)]);
        if (nrec + m > 32u) break;
        if (lane >= nrec && lane < nrec + m) { ts = tt; j = lane - nrec; }
        nrec += m; ++tt;
      }
      t_next = tt; joff_next = 0;
    }
    if (ts != NONE) {                                        // member id (and original group position) of this lane's record
      const sdb_send_desc& x = s_desc[ts & (DESC - 1)];
      const uint32_t fl = x.flags, ms = x.mstart;
      a = __ldg(((fl & SDB_DESC_LIST_TEMP) ? tmp_list : v.members) + ms + j);
      q = (fl & SDB_DESC_POS) ? __ldg(v.member_pos + ms + j) : j;
    }
  };

  // prologue: lanes request the first descriptors / payloads in parallel
  if (lane < DESC && lane < mine) want_desc(lane);
  if (lane < PAY && lane < mine) { wait_desc(lane); want_payload(lane); }
  uint32_t pay_phase = 0;           // bit s = parity of payload slot s: a slot's phase advances only for sends that have a payload AND recipients
  uint32_t pc_c = 0, q32_c = 0, r32_c = 0, rec_c = 0, ch_c = 0;         // cached walk parameters of uniform tiles
  uint32_t t_first = 0, joff_first = 0;
  plan(0, 0);

  while (t_first < mine) {
    // this tile: lanes [0, c_nrec) hold (c_ts, c_j, c_a, c_q); it ends before send c_tnext (or inside it when c_jnext != 0)
    const uint32_t c_ts = ts, c_j = j, c_a = a, c_q = q, c_nrec = nrec, c_tnext = t_next, c_jnext = joff_next;
    const uint32_t t_last = c_jnext ? c_tnext : c_tnext - 1u;

    // 1. payloads of the sends that start in this tile must have landed; zero their pad bytes
    for (uint32_t u = t_first + (joff_first ? 1u : 0u); u <= t_last && u < mine; ++u) {
      const sdb_send_desc& x = s_desc[u & (DESC - 1)];
      const uint32_t padlen = (x.rgran - 1u) * SDB_GRANULE;
      if (mcnt(x) && padlen) {
        sdb_mbar_wait_bounded(&s_pbar[warp][u & (PAY - 1)], (pay_phase >> (u & (PAY - 1))) & 1u);
        pay_phase ^= 1u << (u & (PAY - 1));
        const uint32_t b = x.len + lane;
        if (b < padlen) s_pay[(u & (PAY - 1)) * static_cast<size_t>(stage_bytes) + b] = 0;
      }
    }

    // 2. every lane prepares its record and parks it in the tables
    uint32_t PC = 0;
    if (c_ts != NONE) {
      const uint4* dq = reinterpret_cast<const uint4*>(s_desc + (c_ts & (DESC - 1)));
      const uint4 q0 = dq[0], q1 = dq[1], q2 = dq[2], q3 = dq[3];
      const uint32_t flags = q3.x, rgran = q1.z, sender = q1.y;
      const uint32_t lpt = q1.w;                              // len | prio << 16 | type << 24
      const bool shared_seq = (flags & SDB_DESC_SHARED_SEQ) != 0;
      const bool skip = (flags & SDB_DESC_SKIP_SENDER) && c_a == sender;
      const bool deliver = !skip && c_a < v.max_agents;
      n_skip += skip;
      const uint64_t apos = arena_base + q1.x + static_cast<uint64_t>(c_j) * rgran;
      if (!(flags & SDB_DESC_PULL) && deliver) {              // small / non-group batches: ring slots claimed here, sorted by k_commit
        const uint16_t meta = static_cast<uint16_t>((((lpt >> 16) & 0xFFu) << 14) | rgran);
        if (sdb_ring_append(v, c_a, static_cast<uint32_t>(apos), meta)) ++n_enq; else ++n_ovf;
      }
      const uint64_t seq0 = (flags & SDB_DESC_ABS_SEQ) ? ((static_cast<uint64_t>(q3.w) << 32) | q3.z) : seq_base + q2.x;
      const uint64_t seq = seq0 + (shared_seq ? 0u : c_q);
      s_hdr[2 * lane] = make_uint4(static_cast<uint32_t>(seq), static_cast<uint32_t>(seq >> 32), q0.z, q0.w);
      s_hdr[2 * lane + 1] = make_uint4(sender, shared_seq ? SDB_NO_RECEIVER : c_a, q2.w, lpt);
      PC = ((rgran - 1u) << 1) + 2u;                          // 16-byte chunks: 2 header + 2 per payload granule
      const unsigned long long dst = deliver ? reinterpret_cast<unsigned long long>(sdb_arena_ptr(v, apos)) : 0ull;
      s_rec[lane] = make_uint4(static_cast<uint32_t>(dst), static_cast<uint32_t>(dst >> 32),
                               pay_sa + (c_ts & (PAY - 1)) * stage_bytes, PC);
    }
    const uint32_t PC0 = __shfl_sync(0xFFFFFFFFu, PC, 0);
    const bool uniform = __all_sync(0xFFFFFFFFu, lane >= c_nrec || PC == PC0);
    uint32_t total = c_nrec * PC0;
    if (!uniform) {
      total = PC;
      for (int o = 16; o; o >>= 1) total += __shfl_xor_sync(0xFFFFFFFFu, total, o);
    }
    __syncwarp();

    // 3. plan the next tile now: its member ids travel while this tile is written
    plan(c_tnext, c_jnext);

    // 4. flat walk over the tile's chunks, 512 bytes per warp step
    if (c_nrec) {
      uint32_t rec, ch;
      auto advance = [&](uint32_t adv) {                     // generic (record, chunk) += adv for tiles with mixed record sizes
        while (rec < c_nrec) {
          const uint32_t pc = sdb_lds32(rec_sa + rec * 16u + 12u);
          if (ch + adv < pc) { ch += adv; return; }
          adv -= pc - ch; ++rec; ch = 0;
        }
      };
      if (uniform) {
        if (PC0 != pc_c) { pc_c = PC0; q32_c = 32u / PC0; r32_c = 32u % PC0; rec_c = lane / PC0; ch_c = lane % PC0; }
        rec = rec_c; ch = ch_c;
      } else { rec = 0; ch = 0; advance(lane); }
      for (uint32_t done = 0; done < total; done += 32) {
        if (rec < c_nrec) {
          const uint4 e = sdb_lds128(rec_sa + rec * 16u);
          if (e.x | e.y) {
            const uint32_t src = ch < 2u ? hdr_sa + rec * 32u + ch * 16u : e.z + (ch - 2u) * 16u;
            const uint4 x = sdb_lds128(src);
            uint8_t* dst = reinterpret_cast<uint8_t*>((static_cast<unsigned long long>(e.y) << 32) | e.x) + ch * 16u;
            sdb_st_stream_pol(dst, x, pol_stream);
          }
        }
        if (uniform) { ch += r32_c; rec += q32_c; if (ch >= PC0) { ch -= PC0; ++rec; } }
        else advance(32u);
      }
    }
    __syncwarp();                                           // tables and (at a group end) stages are free again

    // 5. a refill group has retired: its payload stages take sends g+8..g+11, its descriptor slots g+16..g+19
    if (c_jnext == 0 && ((c_tnext & (GROUP - 1)) == 0 || c_tnext >= mine) && lane < GROUP) {
      const uint32_t g0 = t_first & ~(GROUP - 1);
      const uint32_t u = g0 + PAY + lane, w = g0 + DESC + lane;
      sdb_fence_proxy_async();                              // the stages were written (pad bytes) and read through the generic proxy
      if (u < mine) { wait_desc(u); want_payload(u); }
      if (w < mine) want_desc(w);
    }
    t_first = c_tnext; joff_first = c_jnext;
  }
  for (int o = 16; o; o >>= 1) {
    n_enq += __shfl_xor_sync(0xFFFFFFFFu, n_enq, o);
    n_ovf += __shfl_xor_sync(0xFFFFFFFFu, n_ovf, o);
    n_skip += __shfl_xor_sync(0xFFFFFFFFu, n_skip, o);
  }
  if (lane == 0) {
    if (n_enq) atomicAdd(&v.ctr->enqueued, n_enq);
    if (n_ovf) atomicAdd(&v.ctr->ring_overflow, n_ovf);
    if (n_skip) atomicAdd(&v.ctr->skipped_sender, n_skip);
  }
}

// ------------------------------------------------------------------------------------------
// K2, shared-payload form (group sends above the pull threshold, payloads up to 512 bytes).
// The reference gives every recipient of a group message its own copy (M:1267-1277); the copies differ in 12 header
// bytes.  Here a send writes its members' 32-byte headers back to back and the padded payload ONCE behind them
// (sdb_common.cuh "shared payloads"); the index build points every member's ring entry at its header and records the
// distance to the payload, and the receive gather reads header + payload from the two places.  For the c2 shape
// (64 recipients, 256-byte payloads) a send writes 2.3 KB instead of 18.4 KB.
// LPS lanes per send (32: wide sends; 8: a shard's narrow share of a group at N = 8).  No shared memory; three
// sends of a sub-warp are in flight: descriptor loads two ahead, member ids + payload chunks one ahead, stores now.
// ------------------------------------------------------------------------------------------
template <int LPS>
__global__ void __launch_bounds__(256)
k_group_fanout_shared(sdb_dev_view v, const sdb_send_desc* __restrict__ descs, uint32_t n,
                      const uint8_t* __restrict__ payload, uint64_t seq_base, uint64_t arena_base,
                      const sdb_batch_base* __restrict__ bb) {
  if (bb) {
    if (bb->skip) return;
    n = bb->n_total; seq_base = bb->seq_base; arena_base = bb->arena_base;
  }
  constexpr int NCH = 32 / LPS;                                  // 16-byte payload chunks per lane (512 bytes at most)
  const uint32_t lane = threadIdx.x & 31, sl = lane & (LPS - 1);
  const uint32_t gsw = (blockIdx.x * blockDim.x + threadIdx.x) / LPS, nsw = (gridDim.x * blockDim.x) / LPS;
  const uint64_t pol = sdb_policy_evict_first();
  uint32_t n_skip = 0;
  struct Desc { uint4 q0, q1, q2, q3; };
  struct Work { uint32_t a0, a1, p0, p1; uint4 pc[NCH]; };
  auto load_desc = [&](uint32_t i) {
    Desc d; d.q0 = d.q1 = d.q2 = d.q3 = make_uint4(0, 0, 0, 0);
    if (i < n) {
      const uint4* dq = reinterpret_cast<const uint4*>(descs + i);
      d.q0 = __ldg(dq); d.q1 = __ldg(dq + 1); d.q2 = __ldg(dq + 2); d.q3 = __ldg(dq + 3);
    }
    return d;
  };
  auto fetch = [&](const Desc& d, uint32_t i) {                  // member ids of the first two tiles + this lane's payload chunks
    Work w; w.a0 = w.a1 = 0xFFFFFFFFu; w.p0 = sl; w.p1 = sl + LPS;
#pragma unroll
    for (int c = 0; c < NCH; ++c) w.pc[c] = make_uint4(0, 0, 0, 0);
    if (i >= n) return w;
    const uint32_t mstart = d.q2.y, mcount = d.q2.z, flags = d.q3.x;
    if (!(flags & SDB_DESC_PULL) || mcount == 0) return w;
    if (sl < mcount) w.a0 = __ldg(v.members + mstart + sl);
    if (sl + LPS < mcount) w.a1 = __ldg(v.members + mstart + sl + LPS);
    if (flags & SDB_DESC_POS) {
      if (sl < mcount) w.p0 = __ldg(v.member_pos + mstart + sl);
      if (sl + LPS < mcount) w.p1 = __ldg(v.member_pos + mstart + sl + LPS);
    }
    const uint32_t padlen = (d.q1.z - 1u) * SDB_GRANULE, len = d.q1.w & 0xFFFFu;
    const uint8_t* src = payload + ((static_cast<uint64_t>(d.q0.y) << 32) | d.q0.x);
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const uint32_t b0 = (static_cast<uint32_t>(c) * LPS + sl) << 4;
      if (b0 < padlen) {
        uint4 x = sdb_ld_stream(src + b0);                       // (may be a peer GPU's export buffer: NVLink)
        if (b0 + 16u > len) {                                    // deterministic pad bytes
          uint8_t* xb = reinterpret_cast<uint8_t*>(&x);
#pragma unroll
          for (int k = 0; k < 16; ++k) if (b0 + k >= len) xb[k] = 0;
        }
        w.pc[c] = x;
      }
    }
    return w;
  };
  uint32_t i = gsw;
  Desc d = load_desc(i);
  Work w = fetch(d, i);
  Desc dn = load_desc(i + nsw);
  for (; i < n; i += nsw) {
    const Work wn = fetch(dn, i + nsw);                          // next send's loads are in flight while this one is written
    const Desc dnn = load_desc(i + 2u * nsw);
    const uint32_t mstart = d.q2.y, mcount = d.q2.z, flags = d.q3.x;
    if ((flags & SDB_DESC_PULL) && mcount) {
      const uint32_t sender = d.q1.y, rgran = d.q1.z, lpt = d.q1.w;
      const bool shared_seq = (flags & SDB_DESC_SHARED_SEQ) != 0, skip_sender = (flags & SDB_DESC_SKIP_SENDER) != 0;
      const uint64_t seq0 = (flags & SDB_DESC_ABS_SEQ) ? ((static_cast<uint64_t>(d.q3.w) << 32) | d.q3.z) : seq_base + d.q2.x;
      const double ts = __longlong_as_double((static_cast<long long>(d.q0.w) << 32) | d.q0.z);
      uint8_t* const base = sdb_arena_ptr(v, arena_base + d.q1.x);                // the batch region never wraps
      const uint4 hdr_hi = make_uint4(sender, SDB_NO_RECEIVER, d.q2.w, lpt);
      for (uint32_t tile = 0; tile < mcount; tile += 2u * LPS) {
        uint32_t a0, a1, p0, p1;
        const uint32_t j0 = tile + sl, j1 = j0 + LPS;
        if (tile == 0) { a0 = w.a0; a1 = w.a1; p0 = w.p0; p1 = w.p1; }
        else {
          a0 = j0 < mcount ? __ldg(v.members + mstart + j0) : 0xFFFFFFFFu;
          a1 = j1 < mcount ? __ldg(v.members + mstart + j1) : 0xFFFFFFFFu;
          p0 = (flags & SDB_DESC_POS) ? (j0 < mcount ? __ldg(v.member_pos + mstart + j0) : 0u) : j0;
          p1 = (flags & SDB_DESC_POS) ? (j1 < mcount ? __ldg(v.member_pos + mstart + j1) : 0u) : j1;
        }
        const bool s0 = j0 < mcount && skip_sender && a0 == sender, s1 = j1 < mcount && skip_sender && a1 == sender;
        n_skip += s0 + s1;
        // headers tile..tile+LPS-1 (one per lane), then the next LPS: each run stored as whole sectors (sdb_st_headers),
        // skipped senders and out-of-range agents left unwritten
        uint4 hi0 = hdr_hi, hi1 = hdr_hi;
        if (!shared_seq) { hi0.y = a0; hi1.y = a1; }
        uint8_t* const dst = base + (static_cast<size_t>(tile) << 5);
        sdb_st_headers_pol<LPS>(dst, sdb_header_lo(seq0 + (shared_seq ? 0u : p0), ts), hi0,
                                j0 < mcount && !s0 && a0 < v.max_agents, lane, pol);
        sdb_st_headers_pol<LPS>(dst + LPS * 32, sdb_header_lo(seq0 + (shared_seq ? 0u : p1), ts), hi1,
                                j1 < mcount && !s1 && a1 < v.max_agents, lane, pol);
      }
      // the one payload of the send, behind its mcount headers
      uint8_t* const pdst = base + (static_cast<size_t>(mcount) << 5);
      const uint32_t padlen = (rgran - 1u) * SDB_GRANULE;
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const uint32_t b0 = (static_cast<uint32_t>(c) * LPS + sl) << 4;
        if (b0 < padlen) sdb_st_stream_pol(reinterpret_cast<uint4*>(pdst + b0), w.pc[c], pol);
      }
    }
    d = dn; dn = dnn; w = wn;
  }
  for (int o = 16; o; o >>= 1) n_skip += __shfl_xor_sync(0xFFFFFFFFu, n_skip, o);
  if (lane == 0 && n_skip) atomicAdd(&v.ctr->skipped_sender, n_skip);
}

// ------------------------------------------------------------------------------------------
// K1: point-to-point enqueue.  One warp per record: lanes 0-1 build the header, lanes 2.. copy
// payload chunks global -> global with streaming 16-byte accesses; lane 0 claims the ring slot.
// Algorithmic bytes: 2 (L+H) per record.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_enqueue_p2p(sdb_dev_view v, const sdb_send_desc* __restrict__ descs, uint32_t n,
              const uint8_t* __restrict__ payload, uint64_t seq_base, uint64_t arena_base) {
  // 8 lanes per record, 4 records per warp step; every lane keeps up to three 16-byte chunks in flight
  const uint32_t lane = threadIdx.x & 31, sub = lane >> 3, l8 = lane & 7;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nw = (gridDim.x * blockDim.x) >> 5;
  const uint64_t pol = sdb_policy_evict_first();
  uint32_t n_enq = 0, n_ovf = 0;
  for (uint32_t i0 = gw * 4u; i0 < n; i0 += nw * 4u) {
    const uint32_t i = i0 + sub;
    if (i >= n) continue;
    // the 8 lanes of a record read its descriptor: q0 (payload_off, timestamp), q1 (gran0, sender, rgran, len|prio|type), q2 (rec0, receiver, ..)
    const uint4* dq = reinterpret_cast<const uint4*>(descs + i);
    const uint4 q0 = __ldg(dq), q1 = __ldg(dq + 1), q2 = __ldg(dq + 2);
    const uint32_t a = q2.y;                       // mstart = receiver index
    if (a >= v.max_agents) continue;
    const uint64_t payload_off = (static_cast<uint64_t>(q0.y) << 32) | q0.x;
    const double ts = __longlong_as_double((static_cast<long long>(q0.w) << 32) | q0.z);
    const uint32_t rgran = q1.z, len = q1.w & 0xFFFFu, prio = (q1.w >> 16) & 0xFFu, type = q1.w >> 24;
    const uint32_t padlen = (rgran - 1u) * SDB_GRANULE;
    const uint32_t nchunk = 2u + (padlen >> 4);
    const uint64_t apos = arena_base + q1.x;
    uint8_t* rec = sdb_arena_ptr(v, apos);
    const uint8_t* src = payload + payload_off;
    for (uint32_t c = l8; c < nchunk; c += 24) {
      uint4 x[3]; uint32_t cc[3] = {c, c + 8, c + 16};
#pragma unroll
      for (int u = 0; u < 3; ++u) {
        if (cc[u] >= nchunk) continue;
        if (cc[u] == 0) x[u] = sdb_header_lo(seq_base + q2.x, ts);
        else if (cc[u] == 1) x[u] = sdb_header_hi(q1.y, a, SDB_NO_GROUP, static_cast<uint16_t>(len), static_cast<uint8_t>(prio), static_cast<uint8_t>(type));
        else {
          x[u] = sdb_ld_stream(src + ((cc[u] - 2u) << 4));
          const uint32_t b0 = (cc[u] - 2u) << 4;               // zero the pad bytes beyond len
          if (b0 + 16u > len) {
            uint8_t* xb = reinterpret_cast<uint8_t*>(&x[u]);
#pragma unroll
            for (int k = 0; k < 16; ++k) if (b0 + k >= len) xb[k] = 0;
          }
        }
      }
#pragma unroll
      for (int u = 0; u < 3; ++u) if (cc[u] < nchunk) sdb_st_stream_pol(rec + (cc[u] << 4), x[u], pol);
    }
    if (l8 == 0) {
      const uint16_t meta = static_cast<uint16_t>((prio << 14) | rgran);
      const uint4 q3 = __ldg(dq + 3);
      if (q3.x & SDB_DESC_RANKED) {                    // ranked at staging time: slot = ctail + rank, no atomics (see the bulk-copy form)
        const uint4 hd = __ldcg(reinterpret_cast<const uint4*>(v.ring_hdr + a));
        const uint32_t room = v.ring_slots - (hd.z - hd.x);
        if (q3.y < room) { sdb_ring_of(v, a)[(hd.z + q3.y) & (v.ring_slots - 1)] = make_uint2(static_cast<uint32_t>(apos), meta); ++n_enq; }
        else { ++n_ovf; sdb_note_overflow(v, a, static_cast<uint32_t>(apos)); }
        if (q3.x & SDB_DESC_RANK_LAST) v.ring_hdr[a].tail = hd.z + min(q3.y + 1u, room);
      } else if (sdb_ring_append(v, a, static_cast<uint32_t>(apos), meta)) ++n_enq; else ++n_ovf;
    }
  }
  for (int o = 16; o; o >>= 1) {
    n_enq += __shfl_xor_sync(0xFFFFFFFFu, n_enq, o);
    n_ovf += __shfl_xor_sync(0xFFFFFFFFu, n_ovf, o);
  }
  if (lane == 0) {
    if (n_enq) atomicAdd(&v.ctr->enqueued, n_enq);
    if (n_ovf) atomicAdd(&v.ctr->ring_overflow, n_ovf);
  }
}

// ------------------------------------------------------------------------------------------
// K1, bulk-copy form (default for payloads up to 512 bytes): one LANE per record, 32 records per warp step, two
// steps in flight per warp.
//   * the lane reads its 64-byte descriptor (consecutive lanes -> consecutive descriptors), issues ONE TMA bulk load
//     of the padded payload into its shared-memory slot, writes the 32-byte record header and the ring entry while
//     the load is in flight, then zeroes the pad bytes in the slot and issues ONE bulk store into the arena record
//   * ring slots are NOT claimed with atomics when the batch was ranked at staging time (SDB_DESC_RANKED: the host
//     numbers the sends of one receiver 0, 1, 2 .. in send order): slot = ctail + rank, read-only on the ring header
//     (nobody writes ctail during the kernel); the highest-ranked send publishes tail = ctail + count.  Entries land
//     in send order, so the commit is k_commit_ranked (ctail = tail for the touched receivers): no sort.
// The LSU form above kept one record's descriptor -> payload -> atomic chain per 8 lanes and was latency-bound
// (few instructions issued per cycle, warps waiting on that chain of dependent loads).
// ------------------------------------------------------------------------------------------
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
k_enqueue_p2p_tma(sdb_dev_view v, const sdb_send_desc* __restrict__ descs, uint32_t n,
                  const uint8_t* __restrict__ payload, uint64_t seq_base, uint64_t arena_base, uint32_t slot_bytes) {
  extern __shared__ __align__(128) uint8_t s_dyn[];          // [WARPS][2][32][slot_bytes]
  __shared__ __align__(8) uint64_t s_bar[WARPS][2];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* const wbase = s_dyn + static_cast<size_t>(warp) * 2u * 32u * slot_bytes;
  if (lane == 0) { sdb_mbar_init(&s_bar[warp][0], 1); sdb_mbar_init(&s_bar[warp][1], 1); sdb_fence_barrier_init(); }
  __syncwarp();
  const uint32_t gw = blockIdx.x * WARPS + warp, stride = gridDim.x * WARPS * 32u;
  uint32_t phase = 0;
  uint32_t n_enq = 0, n_ovf = 0;
  // Three steps of a warp are in flight, so that no load is consumed in the step that issues it:
  //   A(k+2) descriptor loads   B(k+1) TMA payload load + record header + ring-header load   C(k) ring entry + bulk store
  struct Desc { uint4 q0, q1, q2, q3; bool have; };
  struct Rec { uint8_t* rec; uint4 hd; uint32_t padlen, len, a, apos32, rank, flags; uint16_t meta; bool valid; };
  auto load_desc = [&](uint32_t i0) {
    Desc d; d.q0 = d.q1 = d.q2 = d.q3 = make_uint4(0, 0, 0, 0);
    const uint32_t i = i0 + lane;
    d.have = i < n;
    if (d.have) {
      const uint4* dq = reinterpret_cast<const uint4*>(descs + i);
      d.q0 = __ldg(dq); d.q1 = __ldg(dq + 1); d.q2 = __ldg(dq + 2); d.q3 = __ldg(dq + 3);
    }
    return d;
  };
  auto start = [&](const Desc& d, uint32_t st) {
    Rec r; r.rec = nullptr; r.hd = make_uint4(0, 0, 0, 0); r.padlen = 0; r.len = 0; r.a = 0; r.apos32 = 0; r.rank = 0; r.flags = 0; r.meta = 0;
    r.valid = d.have && d.q2.y < v.max_agents;
    if (r.valid) { r.padlen = (d.q1.z - 1u) * SDB_GRANULE; r.len = d.q1.w & 0xFFFFu; }
    uint32_t sum = r.padlen;
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, o);
    if (lane == 0) sdb_mbar_expect_tx(&s_bar[warp][st], sum);
    __syncwarp();
    if (r.valid) {
      const uint64_t payload_off = (static_cast<uint64_t>(d.q0.y) << 32) | d.q0.x;
      if (r.padlen) sdb_tma_load(wbase + (static_cast<size_t>(st) * 32u + lane) * slot_bytes, payload + payload_off, r.padlen, &s_bar[warp][st]);
      r.a = d.q2.y; r.flags = d.q3.x; r.rank = d.q3.y;
      if (r.flags & SDB_DESC_RANKED) r.hd = __ldcg(reinterpret_cast<const uint4*>(v.ring_hdr + r.a));   // {head, tail, ctail, ntomb}: L2, not L1
      const uint32_t prio = (d.q1.w >> 16) & 0xFFu, type = d.q1.w >> 24;
      const double ts = __longlong_as_double((static_cast<long long>(d.q0.w) << 32) | d.q0.z);
      const uint64_t apos = arena_base + d.q1.x;
      r.apos32 = static_cast<uint32_t>(apos);
      r.meta = static_cast<uint16_t>((prio << 14) | d.q1.z);
      r.rec = sdb_arena_ptr(v, apos);
      sdb_st_stream(reinterpret_cast<uint4*>(r.rec), sdb_header_lo(seq_base + d.q2.x, ts));
      sdb_st_stream(reinterpret_cast<uint4*>(r.rec) + 1, sdb_header_hi(d.q1.y, r.a, SDB_NO_GROUP, static_cast<uint16_t>(r.len), static_cast<uint8_t>(prio), static_cast<uint8_t>(type)));
    }
    return r;
  };
  uint32_t i0 = gw * 32u;
  if (i0 >= n) return;
  Desc dn = load_desc(i0);
  Rec cur = start(dn, 0);
  dn = load_desc(i0 + stride);
  uint32_t st = 0;
  for (; i0 < n; i0 += stride, st ^= 1u) {
    sdb_tma_wait_read<0>();                                   // the other stage's bulk stores have finished reading it
    __syncwarp();
    Rec nxt; nxt.valid = false; nxt.padlen = 0; nxt.len = 0; nxt.rec = nullptr;
    if (i0 + stride < n) {                                    // (unsigned overflow impossible: n < 2^31 sends per batch)
      nxt = start(dn, st ^ 1u);
      dn = load_desc(i0 + 2u * stride);
    }
    if (cur.valid) {
      if (cur.flags & SDB_DESC_RANKED) {
        const uint32_t room = v.ring_slots - (cur.hd.z - cur.hd.x);                       // free slots at batch start
        if (cur.rank < room) {
          sdb_ring_of(v, cur.a)[(cur.hd.z + cur.rank) & (v.ring_slots - 1)] = make_uint2(cur.apos32, cur.meta);
          ++n_enq;
        } else { ++n_ovf; sdb_note_overflow(v, cur.a, cur.apos32); }
        if (cur.flags & SDB_DESC_RANK_LAST) v.ring_hdr[cur.a].tail = cur.hd.z + min(cur.rank + 1u, room);
      } else {
        if (sdb_ring_append(v, cur.a, cur.apos32, cur.meta)) ++n_enq; else ++n_ovf;
      }
    }
    sdb_mbar_wait_bounded(&s_bar[warp][st], (phase >> st) & 1u);
    phase ^= 1u << st;
    if (cur.padlen) {
      uint8_t* slot = wbase + (static_cast<size_t>(st) * 32u + lane) * slot_bytes;
      for (uint32_t b = cur.len; b < cur.padlen; ++b) slot[b] = 0;     // < 32 bytes: arena contents stay deterministic
      sdb_fence_proxy_async();
      sdb_tma_store(cur.rec + 32, slot, cur.padlen);
    }
    sdb_tma_commit();
    cur = nxt;
  }
  sdb_tma_wait_all<0>();
  for (int o = 16; o; o >>= 1) {
    n_enq += __shfl_xor_sync(0xFFFFFFFFu, n_enq, o);
    n_ovf += __shfl_xor_sync(0xFFFFFFFFu, n_ovf, o);
  }
  if (lane == 0) {
    if (n_enq) atomicAdd(&v.ctr->enqueued, n_enq);
    if (n_ovf) atomicAdd(&v.ctr->ring_overflow, n_ovf);
  }
}

// commit of a ranked point-to-point batch: the entries are in send order already; publish ctail = tail for the
// receivers the batch touched (one thread per send; only the highest-ranked send of a receiver acts)
__global__ void __launch_bounds__(256)
k_commit_ranked(sdb_dev_view v, const sdb_send_desc* __restrict__ descs, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint4* dq = reinterpret_cast<const uint4*>(descs + i);
  const uint4 q3 = __ldg(dq + 3);
  if (!(q3.x & SDB_DESC_RANK_LAST)) return;
  const uint32_t a = __ldg(dq + 2).y;
  if (a >= v.max_agents) return;
  v.ring_hdr[a].ctail = v.ring_hdr[a].tail;
}

// ------------------------------------------------------------------------------------------
// pull index build.  For large group batches the ring entries are not claimed by the fan-out kernel (4 M random
// atomics + small scattered stores rival the payload stream in DRAM time); they are appended in global send order by
// kernels that own whole rings, from the batch's sends bucketed by group (ascending send index inside a bucket,
// built by the exporter): no atomics, no sort.
//
//   k_pull_index_group  one WARP per group whose members all belong to that group only ("exclusive" groups - the
//                       usual case: teams).  Every member of such a group receives the same sends, so the warp
//                       loads the bucket's descriptors once (coalesced), each lane owns members lane, lane + 32, ..
//                       (ONE 16-byte ring-header load per member) and appends one 8-byte entry per send: the
//                       entries of a member are consecutive (one sector for the usual handful).  The dependent
//                       chain bucket -> descriptor is paid once per group instead of once per (agent, send).
//   k_pull_index        four lanes per agent, for agents with several memberships (merged by (send, position)) or
//                       in groups that are not exclusive.
// ------------------------------------------------------------------------------------------

// Whole-sector appends.  A quad of lanes appends one agent's new entries in slot order, up to four per step.  A
// partial-sector store into rings far larger than L2 makes L2 fetch the sector before it merges the write
// (scripts/ubench/stores.cu), so when no live entry shares the sectors the entries land in - the tail is
// sector-aligned, or the ring is drained (head == tail) - and the rounded-up end stays within R of head, the quad
// assembles each 32-byte sector in its four lanes and stores it whole.  Slots of a sector that get no entry take a
// consumed filler (SDB_META_TOMB): they lie outside [head, tail), which is all any reader of a ring looks at.  Otherwise
// (live entries left by a partial drain, tombstoned windows, a ring about to fill, rings of 2 slots) the caller stores
// each entry where it belongs.  Nothing overflows on the fast path: n_max bounds the entries the agent can take.
struct sdb_sector_append {
  uint32_t S;      // first slot of the open sector
  uint64_t cur;    // this lane's slot S + sub of the open sector
  bool fast;
  __device__ __forceinline__ sdb_sector_append(bool ok, uint32_t R, uint32_t head, uint32_t tail, uint32_t n_max)
      : S(tail & ~3u), cur(static_cast<uint64_t>(SDB_META_TOMB) << 32),
        fast(ok && R >= 4u && ((tail & 3u) == 0u || head == tail) && ((tail + n_max + 3u) & ~3u) - head <= R) {}
  // one step: the quad's lanes set in `qbits` hold (in lane order) the entries for slots [p, p + popc(qbits)); e is
  // this lane's.  Every sector the step completes is stored.  Whole warp (shuffles).
  __device__ __forceinline__ void step(uint2* rs, uint32_t mask, uint32_t p, uint32_t qbits, uint64_t e,
                                       uint32_t sub, uint32_t qb, uint64_t pol) {
    const uint32_t cnt = __popc(qbits);
    const uint32_t j = (sub - p) & 3u;                   // the step's entry that falls on a slot = sub (mod 4), if any
    uint32_t m = qbits;                                  // its lane: the j-th set bit of qbits
    if (j > 0) m &= m - 1u;
    if (j > 1) m &= m - 1u;
    if (j > 2) m &= m - 1u;
    const uint64_t x = __shfl_sync(0xFFFFFFFFu, e, qb + (m ? __ffs(m) - 1u : 0u));
    if (!fast) return;
    const bool has = j < cnt;
    const uint32_t s = p + j;
    if (has && s - S < 4u) cur = x;
    if (p + cnt - S >= 4u) {                             // sector S is complete (quad-uniform)
      sdb_st_u64_pol(reinterpret_cast<uint64_t*>(rs + ((S + sub) & mask)), cur, pol);
      S += 4u;
      cur = (has && s - S < 4u) ? x : static_cast<uint64_t>(SDB_META_TOMB) << 32;
    }
  }
  // the open sector, filled up with filler; p = the agent's new tail
  __device__ __forceinline__ void finish(uint2* rs, uint32_t mask, uint32_t p, uint32_t sub, uint64_t pol) {
    if (fast && p != S) sdb_st_u64_pol(reinterpret_cast<uint64_t*>(rs + ((S + sub) & mask)), cur, pol);
  }
};

__global__ void __launch_bounds__(128)
k_pull_index_group(sdb_dev_view v, sdb_pull_view pv, const sdb_send_desc* __restrict__ descs, uint32_t n_groups,
                   const uint8_t* __restrict__ gexcl, const uint32_t* __restrict__ lstart, const uint32_t* __restrict__ lcount,
                   uint64_t arena_base, uint32_t set_ctail, const sdb_batch_base* __restrict__ bb, uint32_t shared) {
  // Dependent-load depth 3: {bucket bounds of every source, member table} -> {send indices, member ids} ->
  // {descriptors, ring headers} (the kernel is latency-bound: every level is issued for the whole warp - 2 members
  // per lane - at once).  The group's bucket is the concatenation of the sources' buckets in source order.
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  uint32_t n_enq = 0, n_ovf = 0;
  if (bb) {
    if (bb->skip) return;
    arena_base = bb->arena_base;
    set_ctail = bb->n_other == 0 ? 1u : 0u;            // with p2p / broadcast sends in the import the commit sort publishes ctail
  }
  if (g < n_groups && gexcl[g]) {
    // level 1: lane s holds source s's bucket [o, e) and the global index of its first send
    uint32_t o = 0, e = 0, f = 0;
    if (lane < pv.n_src) {
      const uint32_t* go = pv.gs_off + static_cast<size_t>(lane) * pv.gs_off_stride;
      o = go[g]; e = go[g + 1];
      f = pv.first ? pv.first[lane] : 0u;
    }
    const uint32_t mstart = __ldg(lstart + g), mcount = __ldg(lcount + g);
    const uint32_t incl = sdb_warp_incl_scan<SDB_MAX_SRC>(e - o, lane);   // prefix over sources: where each source's sends start in the bucket
    const uint32_t total = __shfl_sync(0xFFFFFFFFu, incl, SDB_MAX_SRC - 1 < 31 ? SDB_MAX_SRC - 1 : 31);
    const uint32_t excl = incl - (e - o);
    if (total && mcount) {
      const uint64_t pol = sdb_policy_evict_first();        // the entries are read once, a kernel later
      const uint32_t R = v.ring_slots, mask = R - 1;
      auto send_of = [&](uint32_t p) -> uint32_t {           // bucket position -> global descriptor index (warp-uniform shuffles)
        uint32_t idx = 0xFFFFFFFFu;
        for (uint32_t s = 0; s < pv.n_src; ++s) {
          const uint32_t xs = __shfl_sync(0xFFFFFFFFu, excl, s), cs = __shfl_sync(0xFFFFFFFFu, e - o, s);
          const uint32_t os = __shfl_sync(0xFFFFFFFFu, o, s), fs = __shfl_sync(0xFFFFFFFFu, f, s);
          if (p >= xs && p < xs + cs) idx = fs + pv.gs_idx[static_cast<size_t>(s) * pv.gs_idx_stride + os + (p - xs)];
        }
        return idx;
      };
      for (uint32_t m0 = 0; m0 < mcount; m0 += 64) {
        const uint32_t j0 = m0 + lane, j1 = j0 + 32;      // positions in the (local) member list = record slots in a send's region
        // level 2
        uint32_t sidx = send_of(lane);
        const uint32_t a0 = j0 < mcount ? __ldg(v.members + mstart + j0) : 0xFFFFFFFFu;
        const uint32_t a1 = j1 < mcount ? __ldg(v.members + mstart + j1) : 0xFFFFFFFFu;
        // level 3
        uint4 q1 = make_uint4(0, 0, 0, 0);
        if (sidx != 0xFFFFFFFFu) q1 = __ldg(reinterpret_cast<const uint4*>(descs + sidx) + 1);   // gran0, sender, rgran, len|prio|type
        const bool ok0 = a0 < v.max_agents, ok1 = a1 < v.max_agents;
        uint4 hd0 = make_uint4(0, 0, 0, 0), hd1 = make_uint4(0, 0, 0, 0);
        if (ok0) hd0 = *reinterpret_cast<const uint4*>(v.ring_hdr + a0);                     // head, tail, ctail, ntomb
        if (ok1) hd1 = *reinterpret_cast<const uint4*>(v.ring_hdr + a1);
        uint32_t t0 = hd0.y, t1 = hd1.y;
        // Stores: a QUAD of lanes appends ONE member's entries, four sends per step, in whole sectors where the ring
        // allows it (sdb_sector_append), else up to four consecutive entries in one instruction.  Eight members per
        // warp step; the members' ids / heads / tails travel by shuffle from the lanes that loaded them.
        const uint32_t quad = lane >> 2, sub = lane & 3u, qb = lane & ~3u;
        for (uint32_t k0 = 0; k0 < total; k0 += 32) {
          if (k0) {                                                                          // buckets deeper than 32 sends
            sidx = send_of(k0 + lane);
            q1 = make_uint4(0, 0, 0, 0);
            if (sidx != 0xFFFFFFFFu) q1 = __ldg(reinterpret_cast<const uint4*>(descs + sidx) + 1);
          }
          const uint32_t nk = min(32u, total - k0);
          for (uint32_t mb = 0; mb < 64; mb += 8) {                                          // eight members per step
            const uint32_t mi = mb + quad;                                                   // member slot 0..63 of this block of 64
            const uint32_t srcl = mi & 31u;
            const uint32_t am = __shfl_sync(0xFFFFFFFFu, mi < 32 ? a0 : a1, srcl);
            const uint32_t hm = __shfl_sync(0xFFFFFFFFu, mi < 32 ? hd0.x : hd1.x, srcl);
            const uint32_t tm = __shfl_sync(0xFFFFFFFFu, mi < 32 ? t0 : t1, srcl);
            const bool okm = am < v.max_agents;
            uint2* rs = sdb_ring_of(v, okm ? am : 0u);
            // record slot jm of the send's region: a whole record, or (shared payloads) its header, the one payload
            // sitting behind the region's mcount headers
            const uint32_t jm = m0 + mi;
            sdb_sector_append sa(okm, R, hm, tm, nk);
            uint32_t p = tm;                                                                 // the member's running tail
            for (uint32_t c0 = 0; c0 < nk; c0 += 4) {                                        // four sends per step
              const uint32_t t = c0 + sub;
              const uint32_t gran0 = __shfl_sync(0xFFFFFFFFu, q1.x, t & 31u), sender = __shfl_sync(0xFFFFFFFFu, q1.y, t & 31u);
              const uint32_t rgran = __shfl_sync(0xFFFFFFFFu, q1.z, t & 31u), lpt = __shfl_sync(0xFFFFFFFFu, q1.w, t & 31u);
              const bool keep = t < nk && okm && sender != am;                               // member == sender (M:1268)
              const uint32_t qbits = (__ballot_sync(0xFFFFFFFFu, keep) >> qb) & 0xFu;
              const uint32_t pos = p + __popc(qbits & ((1u << sub) - 1u));
              const uint32_t handle = static_cast<uint32_t>(arena_base + gran0 + (shared ? static_cast<uint64_t>(jm) : static_cast<uint64_t>(jm) * rgran));
              const uint64_t meta_hi = static_cast<uint64_t>((((lpt >> 16) & 0xFFu) << 14) | rgran | (shared ? (mcount - 1u - jm) << 16 : 0u)) << 32;
              if (keep) {
                if (sa.fast) ++n_enq;
                else if (pos - hm >= R) { ++n_ovf; sdb_note_overflow(v, am, handle); }
                else { sdb_st_u64_pol(reinterpret_cast<uint64_t*>(rs + (pos & mask)), meta_hi | handle, pol); ++n_enq; }
              }
              sa.step(rs, mask, p, qbits, meta_hi | handle, sub, qb, pol);
              p += __popc(qbits);
            }
            sa.finish(rs, mask, p, sub, pol);
            // member slot mb + q (quad q) is owned by lane (mb + q) & 31, in half (mb + q) >> 5: it takes the new tail
            const uint32_t pq = __shfl_sync(0xFFFFFFFFu, p, (lane & 7u) << 2);
            if ((lane >> 3) == ((mb >> 3) & 3u)) {                                           // lanes [mb & 31, (mb & 31) + 8) own the 8 members
              if (mb < 32) t0 = pq; else t1 = pq;
            }
          }
        }
        if (ok0 && t0 != hd0.y) {
          if (t0 - hd0.x > R) t0 = hd0.x + R;                                               // dropped entries were counted, never written
          hd0.y = t0; if (set_ctail) hd0.z = t0; *reinterpret_cast<uint4*>(v.ring_hdr + a0) = hd0;
        }
        if (ok1 && t1 != hd1.y) {
          if (t1 - hd1.x > R) t1 = hd1.x + R;
          hd1.y = t1; if (set_ctail) hd1.z = t1; *reinterpret_cast<uint4*>(v.ring_hdr + a1) = hd1;
        }
      }
    }
  }
  for (int o2 = 16; o2; o2 >>= 1) {
    n_enq += __shfl_xor_sync(0xFFFFFFFFu, n_enq, o2);
    n_ovf += __shfl_xor_sync(0xFFFFFFFFu, n_ovf, o2);
  }
  if (lane == 0) {
    if (n_enq) atomicAdd(&v.ctr->enqueued, n_enq);
    if (n_ovf) atomicAdd(&v.ctr->ring_overflow, n_ovf);
  }
}

// ------------------------------------------------------------------------------------------
// k_list_index: owner-computes index build for broadcast batches (M:449-463 / M:810-850).  A pure list batch whose
// recipient lists are pairwise disjoint (the usual case is ONE list - "everybody" - shared by all broadcasts of the
// batch) is the group case with temporary groups: every member of list d receives exactly the sends that name d, in
// send order.  The fan-out kernel then writes records only (SDB_DESC_PULL) and this kernel appends the ring entries:
// one warp per 64 members of a list, four consecutive entries of one member per quad store (full sectors), the
// ring header of a member read and written once.  No atomics, no commit sort: the batch publishes ctail here.
//   lists  [nd] {start in the batch's list pool, count}      bucket  off[nd + 1], idx[] = first-chunk descriptor
//   of every send of the list in send order (record of member j of a send: gran0 + j * rgran: chunks are contiguous)
// ------------------------------------------------------------------------------------------
struct sdb_list_view { const uint32_t* pool; const uint32_t* start; const uint32_t* count; const uint32_t* off; const uint32_t* idx; uint32_t nd; };

__global__ void __launch_bounds__(128)
k_list_index(sdb_dev_view v, sdb_list_view lv, const sdb_send_desc* __restrict__ descs, uint64_t arena_base) {
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t d = blockIdx.y;
  uint32_t n_enq = 0, n_ovf = 0;
  const uint32_t mcount = __ldg(lv.count + d), mstart = __ldg(lv.start + d);
  const uint32_t b0 = __ldg(lv.off + d), total = __ldg(lv.off + d + 1) - b0;
  const uint32_t m0 = (blockIdx.x * 4u + warp) * 64u;
  if (m0 < mcount && total) {
    const uint64_t pol = sdb_policy_evict_first();
    const uint32_t R = v.ring_slots, mask = R - 1;
    const uint32_t j0 = m0 + lane, j1 = j0 + 32;
    const uint32_t a0 = j0 < mcount ? __ldg(lv.pool + mstart + j0) : 0xFFFFFFFFu;
    const uint32_t a1 = j1 < mcount ? __ldg(lv.pool + mstart + j1) : 0xFFFFFFFFu;
    const bool ok0 = a0 < v.max_agents, ok1 = a1 < v.max_agents;
    uint4 hd0 = make_uint4(0, 0, 0, 0), hd1 = make_uint4(0, 0, 0, 0);
    if (ok0) hd0 = *reinterpret_cast<const uint4*>(v.ring_hdr + a0);                       // head, tail, ctail, ntomb
    if (ok1) hd1 = *reinterpret_cast<const uint4*>(v.ring_hdr + a1);
    uint32_t t0 = hd0.y, t1 = hd1.y;
    const uint32_t quad = lane >> 2, sub = lane & 3u, qb = lane & ~3u;
    for (uint32_t k0 = 0; k0 < total; k0 += 32) {
      uint4 q1 = make_uint4(0, 0, 0, 0);
      if (k0 + lane < total) q1 = __ldg(reinterpret_cast<const uint4*>(descs + __ldg(lv.idx + b0 + k0 + lane)) + 1);   // gran0, sender, rgran, len|prio|type
      const uint32_t nk = min(32u, total - k0);
      for (uint32_t mb = 0; mb < 64; mb += 8) {                                            // eight members per step
        const uint32_t mi = mb + quad, srcl = mi & 31u;
        const uint32_t am = __shfl_sync(0xFFFFFFFFu, mi < 32 ? a0 : a1, srcl);
        const uint32_t hm = __shfl_sync(0xFFFFFFFFu, mi < 32 ? hd0.x : hd1.x, srcl);
        const uint32_t tm = __shfl_sync(0xFFFFFFFFu, mi < 32 ? t0 : t1, srcl);
        const bool okm = am < v.max_agents;
        uint2* rs = sdb_ring_of(v, okm ? am : 0u);
        sdb_sector_append sa(okm, R, hm, tm, nk);
        for (uint32_t c0 = 0; c0 < nk; c0 += 4) {                                          // four sends per step
          const uint32_t t = c0 + sub;
          const uint32_t gran0 = __shfl_sync(0xFFFFFFFFu, q1.x, t & 31u);
          const uint32_t rgran = __shfl_sync(0xFFFFFFFFu, q1.z, t & 31u), lpt = __shfl_sync(0xFFFFFFFFu, q1.w, t & 31u);
          const uint32_t pos = tm + c0 + sub;                                              // every member takes every send
          const uint32_t handle = static_cast<uint32_t>(arena_base + gran0 + static_cast<uint64_t>(m0 + mi) * rgran);
          const uint64_t meta_hi = static_cast<uint64_t>((((lpt >> 16) & 0xFFu) << 14) | rgran) << 32;
          if (t < nk && okm) {
            if (sa.fast) ++n_enq;
            else if (pos - hm >= R) { ++n_ovf; sdb_note_overflow(v, am, handle); }
            else { sdb_st_u64_pol(reinterpret_cast<uint64_t*>(rs + (pos & mask)), meta_hi | handle, pol); ++n_enq; }
          }
          sa.step(rs, mask, tm + c0, okm ? (1u << min(4u, nk - c0)) - 1u : 0u, meta_hi | handle, sub, qb, pol);
        }
        sa.finish(rs, mask, tm + nk, sub, pol);
      }
      t0 += nk; t1 += nk;                                                                  // (members that do not exist never store their tail)
    }
    if (ok0) { if (t0 - hd0.x > R) t0 = hd0.x + R; hd0.y = t0; hd0.z = t0; *reinterpret_cast<uint4*>(v.ring_hdr + a0) = hd0; }
    if (ok1) { if (t1 - hd1.x > R) t1 = hd1.x + R; hd1.y = t1; hd1.z = t1; *reinterpret_cast<uint4*>(v.ring_hdr + a1) = hd1; }
  }
  for (int o2 = 16; o2; o2 >>= 1) {
    n_enq += __shfl_xor_sync(0xFFFFFFFFu, n_enq, o2);
    n_ovf += __shfl_xor_sync(0xFFFFFFFFu, n_ovf, o2);
  }
  if (lane == 0) {
    if (n_enq) atomicAdd(&v.ctr->enqueued, n_enq);
    if (n_ovf) atomicAdd(&v.ctr->ring_overflow, n_ovf);
  }
}

__device__ __forceinline__ void pull_emit(const sdb_dev_view& v, const sdb_send_desc* descs, uint32_t s, uint32_t j,
                                          uint32_t a, uint64_t arena_base, uint32_t head, uint32_t& tail,
                                          uint32_t& n_enq, uint32_t& n_ovf, uint64_t pol) {
  const uint4 q1 = __ldg(reinterpret_cast<const uint4*>(descs + s) + 1);   // gran0, sender, rgran, len|prio|type
  if (q1.y == a) return;                                                     // member == sender (M:1268)
  const uint32_t handle = static_cast<uint32_t>(arena_base + q1.x + static_cast<uint64_t>(j) * q1.z);
  if (tail - head >= v.ring_slots) { ++n_ovf; sdb_note_overflow(v, a, handle); return; }
  const uint32_t prio = (q1.w >> 16) & 0xFFu;
  sdb_st_u64_pol(reinterpret_cast<uint64_t*>(sdb_ring_of(v, a) + (tail & (v.ring_slots - 1))),
                 (static_cast<uint64_t>((prio << 14) | q1.z) << 32) | handle, pol);
  ++tail; ++n_enq;
}

// Four lanes per agent ("quad"): the lanes of a quad take consecutive sends of the agent's bucket,
// so the dependent loads (bucket entry -> descriptor) of one agent run in parallel and its new
// ring entries leave in one coalesced store.  Agents with several memberships are merged serially by the
// quad's first lane.  `gexcl` (nullable): agents whose single group is exclusive were served by k_pull_index_group.
__global__ void __launch_bounds__(256)
k_pull_index(sdb_dev_view v, sdb_pull_view pv, const sdb_send_desc* __restrict__ descs, uint32_t n_agents,
             const uint8_t* __restrict__ gexcl, uint64_t arena_base, uint32_t set_ctail) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t a = t >> 2, sub = t & 3u, lane = threadIdx.x & 31, qb = lane & ~3u;
  uint32_t n_enq = 0, n_ovf = 0;
  const uint64_t pol = sdb_policy_evict_last();
  const bool valid = a < n_agents;
  uint32_t k0 = 0, k1 = 0;
  if (valid) { k0 = pv.memb_off[a]; k1 = pv.memb_off[a + 1]; }
  uint32_t nk = k1 - k0;
  if (nk == 1 && gexcl && gexcl[pv.memb_grp[k0]]) nk = 0;            // done by the group-parallel kernel
  uint32_t head = 0, tail = 0, tail0 = 0;
  if (nk) {
    const uint4 hd = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
    head = hd.x; tail = tail0 = hd.y;
  }
  // ---- single membership: quad-parallel
  uint32_t b0 = 0, b1 = 0, j = 0;
  if (nk == 1) { const uint32_t g = pv.memb_grp[k0]; j = pv.memb_pos[k0]; b0 = pv.gs_off[g]; b1 = pv.gs_off[g + 1]; }
  const uint32_t R = v.ring_slots;
  uint2* rs = sdb_ring_of(v, valid ? a : 0u);
  for (uint32_t p = b0 + sub; __any_sync(0xFFFFFFFFu, p - sub < b1); p += 4) {
    const bool act = p < b1;
    uint4 q1 = make_uint4(0, 0, 0, 0);
    if (act) q1 = __ldg(reinterpret_cast<const uint4*>(descs + pv.gs_idx[p]) + 1);     // gran0, sender, rgran, len|prio|type
    const bool keep = act && q1.y != a;                                                 // member == sender (M:1268)
    const uint32_t bal = __ballot_sync(0xFFFFFFFFu, keep);
    const uint32_t qbits = (bal >> qb) & 0xFu;
    const uint32_t pos = tail + __popc(qbits & ((1u << sub) - 1u));
    if (keep) {
      if (pos - head >= R) { ++n_ovf; sdb_note_overflow(v, a, static_cast<uint32_t>(arena_base + q1.x + static_cast<uint64_t>(j) * q1.z)); }
      else {
        const uint32_t handle = static_cast<uint32_t>(arena_base + q1.x + static_cast<uint64_t>(j) * q1.z);
        sdb_st_u64_pol(reinterpret_cast<uint64_t*>(rs + (pos & (R - 1))),
                       (static_cast<uint64_t>((((q1.w >> 16) & 0xFFu) << 14) | q1.z) << 32) | handle, pol);
        ++n_enq;
      }
    }
    tail += __popc(qbits);
  }
  if (nk == 1 && tail - head > R) tail = head + R;           // dropped entries were counted, never written
  // ---- several memberships: serial merge by (send index, member position) on the quad's first lane
  if (nk > 1 && sub == 0) {
    long long last_s = -1; uint32_t last_j = 0;
    for (;;) {
      uint32_t best_s = 0xFFFFFFFFu, best_j = 0xFFFFFFFFu;
      for (uint32_t k = k0; k < k1; ++k) {
        const uint32_t g = pv.memb_grp[k], jj = pv.memb_pos[k];
        uint32_t lo = pv.gs_off[g], hi = pv.gs_off[g + 1];
        const long long need = (last_s >= 0 && jj <= last_j) ? last_s + 1 : last_s;   // first s with (s, jj) > (last_s, last_j)
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          if (static_cast<long long>(pv.gs_idx[mid]) < need) lo = mid + 1; else hi = mid;
        }
        if (lo < pv.gs_off[g + 1]) {
          const uint32_t s2 = pv.gs_idx[lo];
          if (s2 < best_s || (s2 == best_s && jj < best_j)) { best_s = s2; best_j = jj; }
        }
      }
      if (best_s == 0xFFFFFFFFu) break;
      pull_emit(v, descs, best_s, best_j, a, arena_base, head, tail, n_enq, n_ovf, pol);
      last_s = best_s; last_j = best_j;
    }
  }
  if (sub == 0 && tail != tail0) {
    v.ring_hdr[a].tail = tail;
    if (set_ctail) v.ring_hdr[a].ctail = tail;
  }
  for (int o = 16; o; o >>= 1) {
    n_enq += __shfl_xor_sync(0xFFFFFFFFu, n_enq, o);
    n_ovf += __shfl_xor_sync(0xFFFFFFFFu, n_ovf, o);
  }
  if (lane == 0) {
    if (n_enq) atomicAdd(&v.ctr->enqueued, n_enq);
    if (n_ovf) atomicAdd(&v.ctr->ring_overflow, n_ovf);
  }
}

// ------------------------------------------------------------------------------------------
// commit: one thread per agent below the registration watermark.  Entries claimed since the
// last commit sit in [ctail, tail) in atomic-arrival order; sort them by arena position
// relative to the batch base (all of them belong to this batch), clamp an overflowed tail,
// publish ctail = tail.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void commit_agent(const sdb_dev_view& v, uint32_t a, uint32_t batch_base32,
                                             uint32_t* __restrict__ big_list, uint32_t* __restrict__ big_count) {
  const uint4 hd = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
  uint32_t tail = hd.y;
  const uint32_t head = hd.x, ct = hd.z;
  if (tail == ct) return;
  const uint32_t R = v.ring_slots, mask = R - 1;
  if (tail - head > R) {                       // overflowed claims were never written
    tail = head + R;
    v.ring_hdr[a].tail = tail;
  }
  const uint32_t cnt = tail - ct;
  uint2* rs = sdb_ring_of(v, a);
  if (cnt > 1) {
    constexpr uint32_t LOCAL = 16;
    if (cnt <= LOCAL) {
      uint32_t k[LOCAL]; uint32_t m[LOCAL];
#pragma unroll
      for (uint32_t i = 0; i < LOCAL; ++i)
        if (i < cnt) { const uint2 e = rs[(ct + i) & mask]; k[i] = e.x - batch_base32; m[i] = e.y; }
      bool sorted = true;
#pragma unroll
      for (uint32_t i = 1; i < LOCAL; ++i) if (i < cnt && k[i] < k[i - 1]) sorted = false;
      if (!sorted) {
        // odd-even transposition network, fully unrolled so k[]/m[] stay in registers
#pragma unroll
        for (uint32_t r = 0; r < LOCAL; ++r) {
#pragma unroll
          for (uint32_t i = (r & 1); i + 1 < LOCAL; i += 2) {
            if (i + 1 < cnt && k[i + 1] < k[i]) {
              uint32_t tk = k[i]; k[i] = k[i + 1]; k[i + 1] = tk;
              uint32_t tm = m[i]; m[i] = m[i + 1]; m[i + 1] = tm;
            }
          }
        }
#pragma unroll
        for (uint32_t i = 0; i < LOCAL; ++i)
          if (i < cnt) rs[(ct + i) & mask] = make_uint2(k[i] + batch_base32, m[i]);
      }
    } else {
      // many records for one agent in one batch: a whole CTA sorts them (k_commit_big); ctail is published there
      const uint32_t slot = atomicAdd(big_count, 1u);
      big_list[slot] = a;
      return;
    }
  }
  v.ring_hdr[a].ctail = tail;
}


// grid-stride over the agents: with a device-side batch record (asynchronous import) the grid is small and every
// thread returns after ONE load when the import carried no point-to-point / broadcast sends
__global__ void __launch_bounds__(256)
k_commit(sdb_dev_view v, uint32_t n_agents, uint32_t batch_base32, uint32_t* __restrict__ big_list,
         uint32_t* __restrict__ big_count, const sdb_batch_base* __restrict__ bb) {
  if (bb) {
    if (bb->skip || bb->n_other == 0) return;
    batch_base32 = static_cast<uint32_t>(bb->arena_base);
  }
  for (uint32_t a = blockIdx.x * blockDim.x + threadIdx.x; a < n_agents; a += gridDim.x * blockDim.x)
    commit_agent(v, a, batch_base32, big_list, big_count);
}

// one CTA per agent that received more than 16 records in the batch: bitonic sort of (arena position, meta)
// pairs, in shared memory up to 4096 entries, in place in the ring (L2-resident) beyond that
#define SDB_COMMIT_SMEM 4096u
__global__ void __launch_bounds__(256)
k_commit_big(sdb_dev_view v, uint32_t batch_base32, const uint32_t* __restrict__ big_list,
             const uint32_t* __restrict__ big_count, const sdb_batch_base* __restrict__ bb) {
  if (bb) batch_base32 = static_cast<uint32_t>(bb->arena_base);
  __shared__ uint32_t s_key[SDB_COMMIT_SMEM];
  __shared__ uint32_t s_meta[SDB_COMMIT_SMEM];                 // whole .y: meta word and the distance to a shared payload
  const uint32_t n_big = *big_count;
  const uint32_t R = v.ring_slots, mask = R - 1;
  for (uint32_t w = blockIdx.x; w < n_big; w += gridDim.x) {
    const uint32_t a = big_list[w];
    const uint4 hd = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
    const uint32_t tail = hd.y, ct = hd.z;
    const uint32_t cnt = tail - ct;
    uint2* rs = sdb_ring_of(v, a);
    uint32_t N = 1; while (N < cnt) N <<= 1;
    if (N <= SDB_COMMIT_SMEM) {
      for (uint32_t i = threadIdx.x; i < N; i += blockDim.x) {
        const uint2 e = i < cnt ? rs[(ct + i) & mask] : make_uint2(0u, 0u);
        s_key[i] = i < cnt ? e.x - batch_base32 : 0xFFFFFFFFu;
        s_meta[i] = e.y;
      }
      __syncthreads();
      for (uint32_t k = 2; k <= N; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
          for (uint32_t i = threadIdx.x; i < N; i += blockDim.x) {
            const uint32_t l = i ^ j;
            if (l > i) {
              const bool up = (i & k) == 0;
              const uint32_t ki = s_key[i], kl = s_key[l];
              if ((ki > kl) == up) { s_key[i] = kl; s_key[l] = ki; const uint32_t t = s_meta[i]; s_meta[i] = s_meta[l]; s_meta[l] = t; }
            }
          }
          __syncthreads();
        }
      for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x)
        rs[(ct + i) & mask] = make_uint2(s_key[i] + batch_base32, s_meta[i]);
    } else {
      // rare (more than 4096 records for one agent in one batch): odd-even transposition sort in place in the
      // ring (works for any length; the segment is L2-resident)
      for (uint32_t round = 0; round < cnt; ++round) {
        for (uint32_t i = (round & 1u) + 2u * threadIdx.x; i + 1 < cnt; i += 2u * blockDim.x) {
          const uint32_t x = (ct + i) & mask, y = (ct + i + 1) & mask;
          const uint2 ex = rs[x], ey = rs[y];
          if (ex.x - batch_base32 > ey.x - batch_base32) { rs[x] = ey; rs[y] = ex; }
        }
        __syncthreads();
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) v.ring_hdr[a].ctail = tail;
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// host-side launchers (called from sdb_api.cu)
// ------------------------------------------------------------------------------------------
extern "C" cudaError_t sdb_launch_p2p(const sdb_dev_view* v, const sdb_send_desc* descs, uint32_t n,
                                      const uint8_t* payload, uint64_t seq_base, uint64_t arena_base,
                                      int sm_count, cudaStream_t stream, sdb_profiler* prof, uint32_t max_padlen) {
  if (n == 0) return cudaSuccess;
  // 8 warps x 4 records per step; ~4 waves of 8 CTAs/SM, grid-stride beyond
  const uint32_t grid = sdb_grid(n, 8 * 4, 32 * sm_count);
  const int pi = sdb_prof_begin(prof, SDB_PK_P2P, stream);
  if (max_padlen <= 512u) {
    constexpr int WARPS = 4;
    const uint32_t slot = max_padlen < 32u ? 32u : max_padlen;
    const size_t smem = static_cast<size_t>(WARPS) * 2u * 32u * slot;
    uint32_t per_sm = static_cast<uint32_t>((226u * 1024u) / (smem + 1152u));
    if (per_sm > 8u) per_sm = 8u;
    if (per_sm == 0) per_sm = 1;
    uint64_t g = static_cast<uint64_t>(sm_count) * per_sm * 4u;
    const uint64_t need = (static_cast<uint64_t>(n) + WARPS * 32 - 1) / (WARPS * 32);
    if (g > need) g = need;
    k_enqueue_p2p_tma<WARPS><<<static_cast<uint32_t>(g), WARPS * 32, smem, stream>>>(*v, descs, n, payload, seq_base, arena_base, slot);
  } else {
    k_enqueue_p2p<<<grid, 256, 0, stream>>>(*v, descs, n, payload, seq_base, arena_base);
  }
  sdb_prof_end(prof, pi, stream);
  return cudaGetLastError();
}

// the same for batches that touch a large share of the agents: a coalesced sweep over the ring headers (16 bytes per
// agent) instead of one random header access per receiver
__global__ void __launch_bounds__(256)
k_commit_ranked_sweep(sdb_dev_view v, uint32_t n_agents) {
  const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= n_agents) return;
  const uint4 hd = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
  if (hd.y != hd.z) v.ring_hdr[a].ctail = hd.y;
}

extern "C" cudaError_t sdb_launch_commit_ranked(const sdb_dev_view* v, const sdb_send_desc* descs, uint32_t n, uint32_t n_agents,
                                                cudaStream_t stream, sdb_profiler* prof) {
  if (n == 0) return cudaSuccess;
  const int pi = sdb_prof_begin(prof, SDB_PK_COMMIT, stream);
  if (static_cast<uint64_t>(n) * 8u >= n_agents) k_commit_ranked_sweep<<<(n_agents + 255) / 256, 256, 0, stream>>>(*v, n_agents);
  else k_commit_ranked<<<(n + 255) / 256, 256, 0, stream>>>(*v, descs, n);
  sdb_prof_end(prof, pi, stream);
  return cudaGetLastError();
}

// dynamic shared memory limits are per device and per function: set once for the device a handle is created on
extern "C" cudaError_t sdb_send_prepare_device() {
  cudaError_t e;
  if ((e = cudaFuncSetAttribute(k_group_fanout_span<4>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                4 * (SDB_SPAN_DESC * 64 + SDB_SPAN_TABLES + SDB_SPAN_PAY * 512))) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(k_group_fanout_warp<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 4 * 4096 + 512)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(k_enqueue_p2p_tma<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 2 * 32 * 512)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(k_group_fanout_st<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536 + 1024)) != cudaSuccess) return e;
  return cudaFuncSetAttribute(k_group_fanout_tma<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 65536 + 1024);
}

// bb (nullable): the import's placement lives on the device (asynchronous import) - span kernel only
extern "C" cudaError_t sdb_launch_fanout(const sdb_dev_view* v, const sdb_send_desc* descs, uint32_t n,
                                         const uint8_t* payload, const uint32_t* tmp_list,
                                         uint64_t seq_base, uint64_t arena_base, uint32_t max_padlen,
                                         int variant, int sm_count, cudaStream_t stream, sdb_profiler* prof,
                                         const sdb_batch_base* bb, uint32_t skip_pull) {
  if ((bb || skip_pull) && !(variant == 3 && max_padlen <= 512)) return cudaErrorInvalidValue;
  if (n == 0) return cudaSuccess;
  const int pi = sdb_prof_begin(prof, SDB_PK_FANOUT, stream);
  if (variant == 3 && max_padlen <= 512) {
    constexpr int WARPS = 4;
    const uint32_t stage = ((max_padlen ? max_padlen : 16) + 127u) & ~127u;
    const size_t smem = static_cast<size_t>(WARPS) * (SDB_SPAN_DESC * sizeof(sdb_send_desc) + SDB_SPAN_TABLES + static_cast<size_t>(SDB_SPAN_PAY) * stage);
    uint32_t per_sm = 8;
    while (per_sm > 1 && per_sm * (smem + 1024) > 200 * 1024) --per_sm;
    // 4 CTA waves per SM slot: more than one lets the block scheduler even out the tail
    uint32_t grid = static_cast<uint32_t>(sm_count) * per_sm * 4u;
    const uint32_t need = (n + WARPS - 1) / WARPS;
    if (grid > need) grid = need;
    k_group_fanout_span<WARPS><<<grid, WARPS * 32, smem, stream>>>(*v, descs, n, payload, tmp_list, seq_base, arena_base, stage, bb, skip_pull);
  } else if ((variant == 2 || variant == 3) && max_padlen <= 4096) {
    constexpr int WARPS = 4;
    const uint32_t stage = ((max_padlen ? max_padlen : 16) + 127u) & ~127u;
    const size_t smem = static_cast<size_t>(WARPS) * 2 * stage;
    uint32_t per_sm = 16;
    while (per_sm > 1 && per_sm * (smem + 256) > 200 * 1024) per_sm >>= 1;
    uint32_t grid = static_cast<uint32_t>(sm_count) * per_sm;
    const uint32_t need = (n + WARPS - 1) / WARPS;
    if (grid > need) grid = need;
    k_group_fanout_warp<WARPS><<<grid, WARPS * 32, smem, stream>>>(*v, descs, n, payload, tmp_list, seq_base, arena_base, stage);
  } else if (variant == 0 || variant == 2 || variant == 3) {
    constexpr int T = 256;
    const size_t smem = max_padlen ? max_padlen : 16;
    uint32_t grid = static_cast<uint32_t>(sm_count) * 8u;           // persistent: 8 CTAs of 256 threads per SM
    if (grid > n) grid = n;
    k_group_fanout_st<T><<<grid, T, smem, stream>>>(*v, descs, n, payload, tmp_list, seq_base, arena_base);
  } else {
    constexpr int T = 64;
    const uint32_t stage = ((max_padlen ? max_padlen : 16) + 127u) & ~127u;
    uint32_t per_sm = 16;
    const size_t smem = 2ull * stage;
    while (per_sm > 1 && per_sm * (smem + 1024) > 200 * 1024) per_sm >>= 1;
    uint32_t grid = static_cast<uint32_t>(sm_count) * per_sm;
    if (grid > n) grid = n;
    k_group_fanout_tma<T><<<grid, T, smem, stream>>>(*v, descs, n, payload, tmp_list, seq_base, arena_base, stage);
  }
  sdb_prof_end(prof, pi, stream);
  return cudaGetLastError();
}

// shared-payload fan-out (see k_group_fanout_shared): every descriptor of the batch that carries SDB_DESC_PULL
extern "C" cudaError_t sdb_launch_fanout_shared(const sdb_dev_view* v, const sdb_send_desc* descs, uint32_t n, const uint8_t* payload,
                                                uint64_t seq_base, uint64_t arena_base, uint32_t narrow, int sm_count,
                                                cudaStream_t stream, sdb_profiler* prof, const sdb_batch_base* bb) {
  if (n == 0) return cudaSuccess;
  const int pi = sdb_prof_begin(prof, SDB_PK_FANOUT, stream);
  const uint32_t lps = narrow ? 8u : 32u;
  const uint32_t grid = sdb_grid(static_cast<uint64_t>(n) * lps, 256, 32 * sm_count);
  if (narrow) k_group_fanout_shared<8><<<grid, 256, 0, stream>>>(*v, descs, n, payload, seq_base, arena_base, bb);
  else k_group_fanout_shared<32><<<grid, 256, 0, stream>>>(*v, descs, n, payload, seq_base, arena_base, bb);
  sdb_prof_end(prof, pi, stream);
  return cudaGetLastError();
}

// gexcl: per-group "exclusive" flags; n_groups: groups covered by the bucket table; n_shared: how many agents sit in
// non-exclusive groups or in several groups (0: the agent-parallel kernel is not needed at all)
extern "C" cudaError_t sdb_launch_pull(const sdb_dev_view* v, const sdb_pull_view* pv, const sdb_send_desc* descs,
                                       uint32_t n_agents, uint32_t n_groups, const uint8_t* gexcl, uint32_t n_excl_groups,
                                       uint32_t n_shared, const uint32_t* lstart, const uint32_t* lcount,
                                       uint64_t arena_base, int set_ctail, cudaStream_t stream,
                                       sdb_profiler* prof, int* n_launches, const sdb_batch_base* bb, uint32_t shared_payload) {
  if ((bb || shared_payload) && (n_shared || !n_excl_groups)) return cudaErrorInvalidValue;      // group-parallel build only
  if (n_agents == 0) return cudaSuccess;
  const int pi = sdb_prof_begin(prof, SDB_PK_INDEX, stream);
  if (n_excl_groups && n_groups) {
    const uint64_t threads = static_cast<uint64_t>(n_groups) * 32;
    k_pull_index_group<<<static_cast<uint32_t>((threads + 127) / 128), 128, 0, stream>>>(*v, *pv, descs, n_groups, gexcl, lstart, lcount, arena_base, set_ctail ? 1u : 0u, bb, shared_payload);
    if (n_launches) *n_launches += 1;
  }
  if (n_shared || !n_excl_groups) {
    const uint64_t threads = static_cast<uint64_t>(n_agents) * 4;
    k_pull_index<<<static_cast<uint32_t>((threads + 255) / 256), 256, 0, stream>>>(*v, *pv, descs, n_agents, n_excl_groups ? gexcl : nullptr, arena_base, set_ctail ? 1u : 0u);
    if (n_launches) *n_launches += 1;
  }
  sdb_prof_end(prof, pi, stream);
  return cudaGetLastError();
}

// tab: device array {start[nd], count[nd], off[nd + 1], idx[...]} (uint32) as staged by the host
extern "C" cudaError_t sdb_launch_list_index(const sdb_dev_view* v, const sdb_send_desc* descs, const uint32_t* list_pool,
                                             const uint32_t* tab, uint32_t nd, uint32_t max_count, uint64_t arena_base,
                                             cudaStream_t stream, sdb_profiler* prof) {
  if (nd == 0 || max_count == 0) return cudaSuccess;
  if (nd > 65535u) return cudaErrorInvalidValue;
  sdb_list_view lv{list_pool, tab, tab + nd, tab + 2u * nd, tab + 3u * nd + 1u, nd};
  const int pi = sdb_prof_begin(prof, SDB_PK_INDEX, stream);
  dim3 grid((max_count + 255u) / 256u, nd);
  k_list_index<<<grid, 128, 0, stream>>>(*v, lv, descs, arena_base);
  sdb_prof_end(prof, pi, stream);
  return cudaGetLastError();
}

// overflow log -> (agent, sequence number): the dropped records still sit in the arena (nothing refers to them), so the
// sequence number is read from the record header
__global__ void k_ovf_resolve(sdb_dev_view v, uint32_t n, unsigned long long* __restrict__ seq_out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint2 e = v.ovf_log[i];
  // the log keeps the low 32 bits of the arena position; arenas are at most 2^32 granules, so masking recovers the slot
  seq_out[i] = *reinterpret_cast<const unsigned long long*>(v.arena + ((static_cast<uint64_t>(e.y) & v.gmask) << 5));
}
extern "C" cudaError_t sdb_launch_ovf_resolve(const sdb_dev_view* v, uint32_t n, unsigned long long* seq_out, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  k_ovf_resolve<<<(n + 127) / 128, 128, 0, stream>>>(*v, n, seq_out);
  return cudaGetLastError();
}

extern "C" cudaError_t sdb_launch_commit(const sdb_dev_view* v, uint32_t n_agents, uint32_t batch_base32,
                                         uint32_t* big_list, uint32_t* big_count, int sm_count,
                                         cudaStream_t stream, sdb_profiler* prof, const sdb_batch_base* bb) {
  if (n_agents == 0) return cudaSuccess;
  const int pi = sdb_prof_begin(prof, SDB_PK_COMMIT, stream);
  if (!bb) cudaMemsetAsync(big_count, 0, sizeof(uint32_t), stream);     // asynchronous import: k_import_fused reset it
  uint32_t cg = (n_agents + 255) / 256;
  if (bb && cg > static_cast<uint32_t>(sm_count) * 8u) cg = static_cast<uint32_t>(sm_count) * 8u;
  k_commit<<<cg, 256, 0, stream>>>(*v, n_agents, batch_base32, big_list, big_count, bb);
  uint32_t bg = static_cast<uint32_t>(sm_count) * (bb ? 1u : 4u);
  if (bg > n_agents) bg = n_agents;
  k_commit_big<<<bg, 256, 0, stream>>>(*v, batch_base32, big_list, big_count, bb);
  sdb_prof_end(prof, pi, stream);
  return cudaGetLastError();
}

// any kernel of this file: its module is loaded as a whole before the latency server starts (sdb_api.cu)
extern "C" const void* sdb_send_kernel_anchor() { return reinterpret_cast<const void*>(&k_commit_ranked_sweep); }
