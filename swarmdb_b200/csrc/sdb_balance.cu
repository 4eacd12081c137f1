// sdb_balance.cu - K6: batched LLM-backend selection over live load counters (sm_90a).
//
// The reference only stores a flag and a per-agent dict (set_llm_load_balancing /
// assign_llm_backend / get_llm_backend, M:1281-1325) - it has no pick algorithm, so parity
// here is against the definition in include/swarmdb_b200.h, restated by oracle/cpu_ref.c.
//
// mode 0, weighted least-load.  Sequential definition: request t goes to
//   argmin_b (load[b] / weight[b])   (exact rational compare, ties -> lowest index)
// and adds its cost to that backend.  For unit costs the greedy sequence is exactly the
// sorted merge of the per-backend progressions {(L_b + j) / w_b : j >= 0} (each progression
// is increasing, so the smallest remaining element is always a progression head).  Hence
//   pick[t] = backend of the element of global rank t,
//   rank(b, j) = j + sum_{b' != b} #{ j' >= 0 : (L_b' + j')/w_b'  <  (L_b + j)/w_b   [<= if b' < b] }
// which every element computes independently with integer divisions:
//   k_ll_plan     one thread per backend: binary-search n_b = #{j : rank(b, j) < T}
//   k_ll_scatter  one thread per element (b, j): pick[rank(b, j)] = b
// Arbitrary costs have a true sequential dependence; they run on one warp (k_ll_seq).
//
// mode 1, weighted random = one-item weighted reservoir (Efraimidis-Spirakis): backend b
// draws u_b = hash(seed, t, b) and the exponential-race key -log2(u_b)/w_b; the smallest key
// wins, so P(b) ~ w_b.  -log2 is evaluated in Q24 fixed point from a 257-entry table built
// with integer arithmetic only, and keys are compared by cross-multiplication, so results
// are bit-identical on any machine.  Loads are then bumped with shared-memory histograms +
// one global atomic per (CTA, backend).
//
// Not HBM-bound: the table is < 10 KB (L1/shared-resident); report picks/s (SURVEY 8d).
#include "sdb_common.cuh"

// every pick kernel keeps the backend table in shared memory: at SDB_MAX_BACKENDS (include/swarmdb_b200.h) that is up to
// 20 x 4096 + 8 bytes, above the 48 KB a launch gets without opting in (sdb_balance_prepare_device)
static size_t ll_plan_smem(uint32_t B) { return (2 * static_cast<size_t>(B)) * 8 + static_cast<size_t>(B) * 4; }
static size_t ll_scatter_smem(uint32_t B) { return (2 * static_cast<size_t>(B) + 1) * 8 + static_cast<size_t>(B) * 4; }
static size_t ll_seq_smem(uint32_t B) { return static_cast<size_t>(B) * 12; }
static size_t wr_pick_smem(uint32_t B) { return static_cast<size_t>(B) * 12 + 257 * 4; }

// ---- fixed-point -log2 table (host, integer only) --------------------------------------------
extern "C" void sdb_build_log2_table(uint32_t* tab257) {
  for (uint32_t i = 0; i <= 256; ++i) {
    if (i == 256) { tab257[i] = 1u << 24; break; }
    // x = 1 + i/256 in Q62; extract 26 fractional bits of log2(x) by repeated squaring
    unsigned __int128 x = static_cast<unsigned __int128>(256 + i) << 54;
    const unsigned __int128 two = static_cast<unsigned __int128>(2) << 62;
    uint32_t r = 0;
    for (int k = 0; k < 26; ++k) {
      x = (x * x) >> 62;
      r <<= 1;
      if (x >= two) { r |= 1u; x >>= 1; }
    }
    tab257[i] = (r + 2u) >> 2;     // round Q26 -> Q24
  }
}

__device__ __forceinline__ uint64_t sdb_mix(uint64_t seed, uint32_t t, uint32_t b) {
  uint64_t x = seed ^ (static_cast<uint64_t>(t) + 1ull) * 0x9E3779B97F4A7C15ull;
  x ^= (static_cast<uint64_t>(b) + 1ull) * 0xD1B54A32D192ED03ull;
  x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ull;
  x ^= x >> 27; x *= 0x94D049BB133111EBull;
  x ^= x >> 31;
  return x;
}

// -log2(u / 2^32) in Q24 for u in [1, 2^32)
__device__ __forceinline__ uint32_t sdb_neglog2_q24(uint32_t u, const uint32_t* tab) {
  const uint32_t lz = __clz(u);
  const uint32_t un = u << lz;                       // bit 31 set
  const uint32_t idx = (un >> 23) & 0xFFu;
  const uint32_t frac = un & 0x7FFFFFu;
  const uint32_t t0 = tab[idx], t1 = tab[idx + 1];
  const uint32_t lg = t0 + static_cast<uint32_t>((static_cast<uint64_t>(t1 - t0) * frac) >> 23);   // log2(mantissa), Q24
  // log2(u) = (31 - lz) + lg ; -log2(u/2^32) = 32 - log2(u) = (1 + lz) - lg
  return ((1u + lz) << 24) - lg;
}

// ---- mode 0 -----------------------------------------------------------------------------------
// Loads are 64-bit and weights up to 2^16, so load x weight needs up to 80 bits: every cross-multiplication below is
// exact in 128 bits, as in the definition (oracle/cpu_ref.c).  Ranks are only compared with the batch size T < 2^32,
// so each per-backend count saturates at SDB_RANK_SAT: a sum of B <= 4096 of them cannot wrap, and every rank >= T
// stays >= T.
#define SDB_RANK_SAT (1ull << 40)

// a * x < b * y, exactly
__device__ __forceinline__ bool mul_lt(unsigned long long a, uint32_t x, unsigned long long b, uint32_t y) {
  const unsigned long long ah = __umul64hi(a, x), bh = __umul64hi(b, y);
  return ah < bh || (ah == bh && a * x < b * y);
}
__device__ __forceinline__ bool mul_eq(unsigned long long a, uint32_t x, unsigned long long b, uint32_t y) {
  return __umul64hi(a, x) == __umul64hi(b, y) && a * x == b * y;
}

// number of progression elements of backend bp that precede element (b, j) in pick order (bp == b counts j itself)
__device__ __forceinline__ unsigned long long ll_before(unsigned long long Lb_j, uint32_t wb, uint32_t b,
                                                        unsigned long long Lbp, uint32_t wbp, uint32_t bp) {
  unsigned long long n;
  if (__umul64hi(Lb_j, wbp) == 0) {
    const unsigned long long X = Lb_j * wbp;
    const unsigned long long fl = X / wb;
    if (bp < b) {                       // ties go to the lower index: count (L'+j')*w <= X
      const unsigned long long d = fl - Lbp;          // saturated before the + 1: fl - Lbp can be 2^64 - 1
      n = fl >= Lbp ? (d < SDB_RANK_SAT ? d + 1ull : SDB_RANK_SAT) : 0ull;
    } else {                            // strict: (L'+j')*w < X  <=>  L'+j' <= ceil(X/w) - 1
      const unsigned long long ce = fl + ((X % wb) ? 1ull : 0ull);
      n = ce > Lbp ? ce - Lbp : 0ull;
    }
  } else {                              // loads of 2^48 and more: the same in 128 bits
    const unsigned __int128 X = static_cast<unsigned __int128>(Lb_j) * wbp;
    const unsigned __int128 fl = X / wb;
    unsigned __int128 m;
    if (bp < b) m = fl >= Lbp ? fl - Lbp + 1u : 0u;
    else {
      const unsigned __int128 ce = fl + ((X % wb) ? 1u : 0u);
      m = ce > Lbp ? ce - Lbp : 0u;
    }
    n = m < SDB_RANK_SAT ? static_cast<unsigned long long>(m) : SDB_RANK_SAT;
  }
  return n < SDB_RANK_SAT ? n : SDB_RANK_SAT;
}

// global pick-order rank of element (b, j): elements of every progression that precede it, its own included
__device__ unsigned long long ll_rank(uint32_t b, unsigned long long j, uint32_t B, const unsigned long long* L,
                                      const uint32_t* w) {
  unsigned long long r = 0;
  const unsigned long long Lb_j = L[b] + j;
  const uint32_t wb = w[b];
  for (uint32_t bp = 0; bp < B; ++bp) r += ll_before(Lb_j, wb, b, L[bp], w[bp], bp);
  return r;
}

// scratch layout (unsigned long long): [0,B) start offsets, [B,2B) L0 (loads before the batch), [2B] total
__global__ void __launch_bounds__(1024)
k_ll_plan(uint32_t B, const uint32_t* __restrict__ weight, unsigned long long* __restrict__ load, uint32_t T,
          unsigned long long* __restrict__ scratch) {
  extern __shared__ unsigned long long s_mem[];
  unsigned long long* sL = s_mem;                       // [B]
  unsigned long long* sN = s_mem + B;                   // [B]
  uint32_t* sW = reinterpret_cast<uint32_t*>(s_mem + 2 * B);   // [B]
  for (uint32_t b = threadIdx.x; b < B; b += blockDim.x) { sL[b] = load[b]; sW[b] = weight[b]; }
  __syncthreads();
  for (uint32_t b = threadIdx.x; b < B; b += blockDim.x) {
    // smallest j with rank(b, j) >= T  ==  number of picks of backend b
    unsigned long long lo = 0, hi = T;
    while (lo < hi) {
      const unsigned long long mid = (lo + hi) >> 1;
      if (ll_rank(b, mid, B, sL, sW) >= T) hi = mid; else lo = mid + 1;
    }
    sN[b] = lo;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long acc = 0;
    for (uint32_t b = 0; b < B; ++b) { scratch[b] = acc; acc += sN[b]; }
    scratch[2 * B] = acc;
  }
  for (uint32_t b = threadIdx.x; b < B; b += blockDim.x) {
    scratch[B + b] = sL[b];
    load[b] = sL[b] + sN[b];
  }
}

__global__ void __launch_bounds__(256)
k_ll_scatter(uint32_t B, const uint32_t* __restrict__ weight, const unsigned long long* __restrict__ scratch,
             uint32_t T, uint32_t* __restrict__ out) {
  extern __shared__ unsigned long long s_mem[];
  unsigned long long* sL = s_mem;                       // [B]
  unsigned long long* sS = s_mem + B;                   // [B+1]
  uint32_t* sW = reinterpret_cast<uint32_t*>(s_mem + 2 * B + 1);
  for (uint32_t b = threadIdx.x; b < B; b += blockDim.x) { sL[b] = scratch[B + b]; sS[b] = scratch[b]; sW[b] = weight[b]; }
  if (threadIdx.x == 0) sS[B] = scratch[2 * B];
  __syncthreads();
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= T || e >= sS[B]) return;
  uint32_t lo = 0, hi = B;                              // largest b with start[b] <= e
  while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (sS[mid] <= e) lo = mid; else hi = mid; }
  // skip empty backends that share the same start
  uint32_t b = lo;
  while (b + 1 < B && sS[b + 1] <= e) ++b;
  const unsigned long long j = e - sS[b];
  const unsigned long long t = ll_rank(b, j, B, sL, sW);
  if (t < T) out[t] = b;
}

// arbitrary costs: one warp, backends strided over lanes, exact sequential greedy
__global__ void __launch_bounds__(32)
k_ll_seq(uint32_t B, const uint32_t* __restrict__ weight, unsigned long long* __restrict__ load, uint32_t T,
         const uint32_t* __restrict__ cost, uint32_t* __restrict__ out) {
  extern __shared__ unsigned long long s_mem[];
  unsigned long long* sL = s_mem;
  uint32_t* sW = reinterpret_cast<uint32_t*>(s_mem + B);
  const uint32_t lane = threadIdx.x;
  for (uint32_t b = lane; b < B; b += 32) { sL[b] = load[b]; sW[b] = weight[b]; }
  __syncwarp();
  for (uint32_t t = 0; t < T; ++t) {
    unsigned long long bl = ~0ull; uint32_t bw = 1, bi = 0xFFFFFFFFu;
    for (uint32_t b = lane; b < B; b += 32) {
      const unsigned long long l = sL[b]; const uint32_t w = sW[b];
      // l/w < bl/bw  <=>  l*bw < bl*w   (bi == ~0 means "none yet")
      if (bi == 0xFFFFFFFFu || mul_lt(l, bw, bl, w)) { bl = l; bw = w; bi = b; }
    }
    for (int o = 16; o; o >>= 1) {
      const unsigned long long ol = __shfl_xor_sync(0xFFFFFFFFu, bl, o);
      const uint32_t ow = __shfl_xor_sync(0xFFFFFFFFu, bw, o);
      const uint32_t oi = __shfl_xor_sync(0xFFFFFFFFu, bi, o);
      if (oi != 0xFFFFFFFFu) {
        bool better;
        if (bi == 0xFFFFFFFFu) better = true;
        else better = mul_lt(ol, bw, bl, ow) || (mul_eq(ol, bw, bl, ow) && oi < bi);
        if (better) { bl = ol; bw = ow; bi = oi; }
      }
    }
    if (lane == 0) out[t] = bi;
    if ((bi & 31u) == lane) sL[bi] += cost[t];
    __syncwarp();
  }
  for (uint32_t b = lane; b < B; b += 32) load[b] = sL[b];
}

// ---- mode 1 -----------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_wr_pick(uint32_t B, const uint32_t* __restrict__ weight, unsigned long long* __restrict__ load, uint32_t T,
          const uint32_t* __restrict__ cost, uint64_t seed, const uint32_t* __restrict__ logtab,
          uint32_t* __restrict__ out) {
  extern __shared__ unsigned long long s_mem[];
  unsigned long long* sH = s_mem;                                   // [B] cost histogram of this CTA
  uint32_t* sW = reinterpret_cast<uint32_t*>(s_mem + B);            // [B]
  uint32_t* sT = sW + B;                                            // [257]
  for (uint32_t b = threadIdx.x; b < B; b += blockDim.x) { sH[b] = 0; sW[b] = weight[b]; }
  for (uint32_t i = threadIdx.x; i < 257; i += blockDim.x) sT[i] = logtab[i];
  __syncthreads();
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < T) {
    uint32_t best = 0, bw = 1; unsigned long long bk = 0; bool have = false;
    for (uint32_t b = 0; b < B; ++b) {
      const uint32_t u = static_cast<uint32_t>(sdb_mix(seed, t, b) >> 32) | 1u;
      const unsigned long long k = sdb_neglog2_q24(u, sT);
      const uint32_t w = sW[b];
      // k/w < bk/bw  <=>  k*bw < bk*w ; strict, so ties keep the lower index
      if (!have || k * bw < bk * w) { bk = k; bw = w; best = b; have = true; }
    }
    out[t] = best;
    atomicAdd(&sH[best], static_cast<unsigned long long>(cost ? cost[t] : 1u));
  }
  __syncthreads();
  for (uint32_t b = threadIdx.x; b < B; b += blockDim.x)
    if (sH[b]) atomicAdd(&load[b], sH[b]);
}

extern "C" cudaError_t sdb_balance_prepare_device() {
  const uint32_t B = SDB_MAX_BACKENDS;
  cudaError_t e;
  if ((e = cudaFuncSetAttribute(k_ll_plan, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(ll_plan_smem(B)))) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(k_ll_scatter, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(ll_scatter_smem(B)))) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(k_ll_seq, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(ll_seq_smem(B)))) != cudaSuccess) return e;
  return cudaFuncSetAttribute(k_wr_pick, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(wr_pick_smem(B)));
}

extern "C" cudaError_t sdb_launch_pick(int mode, uint32_t B, const uint32_t* weight_dev, unsigned long long* load_dev,
                                       uint32_t n_req, const uint32_t* cost_dev, uint64_t seed, uint32_t* out_dev,
                                       unsigned long long* scratch_dev, const uint32_t* log_tab_dev,
                                       cudaStream_t stream, int* n_launches) {
  if (B > SDB_MAX_BACKENDS) return cudaErrorInvalidValue;
  if (mode == 0) {
    if (cost_dev == nullptr) {
      k_ll_plan<<<1, 1024, ll_plan_smem(B), stream>>>(B, weight_dev, load_dev, n_req, scratch_dev);
      k_ll_scatter<<<(n_req + 255) / 256, 256, ll_scatter_smem(B), stream>>>(B, weight_dev, scratch_dev, n_req, out_dev);
      if (n_launches) *n_launches += 2;
    } else {
      k_ll_seq<<<1, 32, ll_seq_smem(B), stream>>>(B, weight_dev, load_dev, n_req, cost_dev, out_dev);
      if (n_launches) *n_launches += 1;
    }
  } else {
    k_wr_pick<<<(n_req + 255) / 256, 256, wr_pick_smem(B), stream>>>(B, weight_dev, load_dev, n_req, cost_dev, seed, log_tab_dev, out_dev);
    if (n_launches) *n_launches += 1;
  }
  return cudaGetLastError();
}


// ------------------------------------------------------------------------------------------
// N3: inbox / load queries answered from the rings (get_agent_load M:1049-1094, get_unread_message_count
// M:1026-1047, get_stats M:973-1024) and the balancer fed by the queue backlog.
// ------------------------------------------------------------------------------------------
// one warp per listed agent: header fields + a histogram of the pending window's ring metadata
__global__ void __launch_bounds__(256)
k_agent_loads(sdb_dev_view v, const uint32_t* __restrict__ agent_idx, uint32_t n, sdb_agent_load* __restrict__ out) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t q = gw; q < n; q += nw) {
    const uint32_t a = agent_idx ? agent_idx[q] : q;
    uint32_t h[4] = {0, 0, 0, 0}, gran = 0, head = 0, tail = 0;
    if (a < v.max_agents) {
      const uint4 hd = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
      head = hd.x; tail = hd.y;
      const uint2* rs = sdb_ring_of(v, a);
      const uint32_t mask = v.ring_slots - 1;
      for (uint32_t p = head + lane; static_cast<int32_t>(tail - p) > 0; p += 32) {
        const uint32_t m = rs[p & mask].y & 0xFFFFu;
        if (m != SDB_META_TOMB) { h[m >> 14] += 1; gran += (m & SDB_META_GLEN_MASK) - 1u; }
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) for (int o = 16; o; o >>= 1) h[k] += __shfl_xor_sync(0xFFFFFFFFu, h[k], o);
    for (int o = 16; o; o >>= 1) gran += __shfl_xor_sync(0xFFFFFFFFu, gran, o);
    if (lane == 0) {
      sdb_agent_load r;
      r.received = tail; r.pending = h[0] + h[1] + h[2] + h[3];
      r.pending_by_prio[0] = h[0]; r.pending_by_prio[1] = h[1]; r.pending_by_prio[2] = h[2]; r.pending_by_prio[3] = h[3];
      r.pending_granules = gran; r.reserved = 0;
      out[q] = r;
    }
  }
}

// every agent below the watermark: thread per agent for the header part; agents with pending entries walk their
// window (short in the steady state); block-level reduction, one atomic per block and field
__global__ void __launch_bounds__(256)
k_queue_stats(sdb_dev_view v, uint32_t n_agents, unsigned long long* __restrict__ acc /* [10] */) {
  __shared__ unsigned long long s_acc[9];
  __shared__ unsigned long long s_max;
  if (threadIdx.x < 9) s_acc[threadIdx.x] = 0;
  if (threadIdx.x == 0) s_max = 0;
  __syncthreads();
  const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a < n_agents) {
    const uint4 hd = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
    const uint32_t live = hd.y - hd.x - hd.w;
    atomicAdd(&s_acc[7], static_cast<unsigned long long>(hd.y));
    if (live) {
      uint32_t h[4] = {0, 0, 0, 0}, gran = 0;
      const uint2* rs = sdb_ring_of(v, a);
      const uint32_t mask = v.ring_slots - 1;
      for (uint32_t p = hd.x; p != hd.y; ++p) {
        const uint32_t m = rs[p & mask].y & 0xFFFFu;
        if (m != SDB_META_TOMB) { h[m >> 14] += 1; gran += (m & SDB_META_GLEN_MASK) - 1u; }
      }
      atomicAdd(&s_acc[0], 1ull); atomicAdd(&s_acc[1], static_cast<unsigned long long>(live));
      for (int k = 0; k < 4; ++k) if (h[k]) atomicAdd(&s_acc[2 + k], static_cast<unsigned long long>(h[k]));
      atomicAdd(&s_acc[6], static_cast<unsigned long long>(gran));
      atomicMax(&s_max, (static_cast<unsigned long long>(live) << 32) | (0xFFFFFFFFu - a));   // deepest queue, lowest index on ties
    }
  }
  __syncthreads();
  if (threadIdx.x < 8 && s_acc[threadIdx.x]) atomicAdd(acc + threadIdx.x, s_acc[threadIdx.x]);
  if (threadIdx.x == 8 && s_max) atomicMax(acc + 8, s_max);
}

// load[b] = pending records of the agents assigned to b (thread per agent, shared-memory histogram per block)
__global__ void __launch_bounds__(256)
k_backend_loads_from_queues(sdb_dev_view v, uint32_t n_agents, const uint32_t* __restrict__ agent_backend, uint32_t B,
                            unsigned long long* __restrict__ load) {
  extern __shared__ unsigned long long s_load[];
  for (uint32_t b = threadIdx.x; b < B; b += blockDim.x) s_load[b] = 0;
  __syncthreads();
  const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a < n_agents) {
    const uint32_t b = agent_backend[a];
    if (b < B) {
      const uint4 hd = *reinterpret_cast<const uint4*>(v.ring_hdr + a);
      const uint32_t live = hd.y - hd.x - hd.w;
      if (live) atomicAdd(&s_load[b], static_cast<unsigned long long>(live));
    }
  }
  __syncthreads();
  for (uint32_t b = threadIdx.x; b < B; b += blockDim.x) if (s_load[b]) atomicAdd(load + b, s_load[b]);
}

extern "C" cudaError_t sdb_launch_agent_loads(const sdb_dev_view* v, const uint32_t* agent_idx_dev, uint32_t n, sdb_agent_load* out_dev,
                                              int sm_count, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  uint32_t grid = static_cast<uint32_t>(sm_count) * 8u;
  if (grid > (n + 7) / 8) grid = (n + 7) / 8;
  k_agent_loads<<<grid, 256, 0, stream>>>(*v, agent_idx_dev, n, out_dev);
  return cudaGetLastError();
}
extern "C" cudaError_t sdb_launch_queue_stats(const sdb_dev_view* v, uint32_t n_agents, unsigned long long* acc_dev, cudaStream_t stream) {
  cudaMemsetAsync(acc_dev, 0, 10 * sizeof(unsigned long long), stream);
  if (n_agents) k_queue_stats<<<(n_agents + 255) / 256, 256, 0, stream>>>(*v, n_agents, acc_dev);
  return cudaGetLastError();
}
extern "C" cudaError_t sdb_launch_backend_loads_from_queues(const sdb_dev_view* v, uint32_t n_agents, const uint32_t* agent_backend_dev,
                                                            uint32_t B, unsigned long long* load_dev, cudaStream_t stream) {
  cudaMemsetAsync(load_dev, 0, static_cast<size_t>(B) * sizeof(unsigned long long), stream);
  if (n_agents && B) k_backend_loads_from_queues<<<(n_agents + 255) / 256, 256, B * sizeof(unsigned long long), stream>>>(*v, n_agents, agent_backend_dev, B, load_dev);
  return cudaGetLastError();
}

// any kernel of this file: its module is loaded as a whole before the latency server starts (sdb_api.cu)
extern "C" const void* sdb_balance_kernel_anchor() { return reinterpret_cast<const void*>(&k_ll_seq); }
