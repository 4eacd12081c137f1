// Micro-benchmark (H100): where the receive gather's time goes at the c2 shape.  The bulk gather copies, per output
// record, one random 32-byte header and one 256-byte payload (shared by the 64 members of a group send) to packed
// outputs.  This times that copy as one kernel with both access patterns interleaved in every warp step, and as two
// passes that each keep one pattern: the headers alone, then the payloads alone.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/ubench/gather_phases scripts/ubench/gather_phases.cu
// The c2 arena is generated on the device from a seeded hash: 65,536 sends, each 64 back-to-back 32-byte headers and
// one 256-byte payload (72 granules); 1,000,000 agents in 15,625 random groups of 64, every send to a random group.
// Plan entries {handle, payload granule offset, granules | dm1 << 16, slot} in receiver order, as k_recv_plan writes
// them (sdb_recv.cu).  Modes:
//   A     today's kernel: header through registers, TMA payload load, merged bulk store
//   H     header pass alone: plan entry -> two 16-byte loads -> hdr_out as whole sectors (U steps in flight per lane)
//   P     payload pass alone: plan entry -> TMA load -> merged bulk store
//   W     a pure 1.21 GB whole-sector write stream (the floor)
//   ef    evict-first L2 hint on the header loads and stores (H), on the output bulk stores (P, A) or on all output (A)
// Algorithmic bytes per record: 16 B plan entry + 32 B header + 32 B header out + 256 B payload out; the shared payload
// read counted once per send (256 B / 64).  Every complete copy is checked byte for byte against the arena.
// NVIDIA H100 80GB HBM3, 700 W power limit, 1980 MHz max SM clock, 9 rounds of every mode, median (best - worst) ms:
//   A 0.7575 (0.7551-0.7613)   A, ef bulk stores 0.7149 (0.7129-0.7196)   A, ef bulk + header stores 0.7130
//   H (U=4) 0.2210   H (U=8) 0.2230   H ef 0.2191   P 0.5660   P ef 0.5140   W 0.3857 (3132 GB/s)
//   H+P 0.7813 (0.7776-0.7845)   H+P (U=8) 0.7852   H+P ef 0.7315 (0.7277-0.7317)   H ef + P ef 0.7308
// The passes cost about their sum whether apart or interleaved: the split is slower than A, with or without the hint.
// The evict-first hint on the payload bulk stores is what gains (0.043 ms on A, 0.052 ms on P alone).  That fits the
// evict-normal output stream pushing the 16.7 MB of shared payloads out of the L2 between their 64 reads; the L2 hit
// rate itself was not measured.
#include <algorithm>
#include <cstdio>
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); return 1; } } while (0)

constexpr uint32_t SENDS = 65536, FAN = 64, GROUPS = 15625, AGENTS = GROUPS * FAN;
constexpr uint32_t PG = 8, SEND_G = FAN + PG, RECS = SENDS * FAN;
constexpr uint32_t SLOT = PG * 32;            // one 256-byte payload per lane and stage
constexpr int WARPS = 4;

__host__ __device__ __forceinline__ uint32_t hash32(uint32_t x) { x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; return x; }

__device__ __forceinline__ uint64_t pol_evict_first() {
  uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p;
}
template <bool EF>
__device__ __forceinline__ uint4 ld_stream(const void* p, uint64_t pol) {
  uint4 r;
  if (EF) asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                       : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
  else asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
template <bool EF>
__device__ __forceinline__ void st_stream(void* p, const uint4& v, uint64_t pol) {
  if (EF) asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;"
                       :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "l"(pol) : "memory");
  else asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 sel4(bool c, uint4 a, uint4 b) {
  return make_uint4(c ? a.x : b.x, c ? a.y : b.y, c ? a.z : b.z, c ? a.w : b.w);
}
// 32 consecutive headers, one per lane, stored as whole sectors: lane pairs exchange halves so that each of the two
// store instructions writes 512 contiguous bytes (the library's sdb_st_headers<32>)
template <bool EF>
__device__ __forceinline__ void st_headers32(uint4* dst, uint4 lo, uint4 hi, bool valid, uint32_t lane, uint64_t pol) {
  const uint32_t vm = __ballot_sync(0xFFFFFFFFu, valid);
  const bool odd = lane & 1u, low = lane < 16u;
  const uint32_t src = (lane >> 1) + (odd ? 16u : 0u);
  const uint4 p = sel4(low, lo, hi), q = sel4(low, hi, lo);
  uint4 y0, y1;
  y0.x = __shfl_sync(0xFFFFFFFFu, p.x, src); y0.y = __shfl_sync(0xFFFFFFFFu, p.y, src);
  y0.z = __shfl_sync(0xFFFFFFFFu, p.z, src); y0.w = __shfl_sync(0xFFFFFFFFu, p.w, src);
  y1.x = __shfl_sync(0xFFFFFFFFu, q.x, src ^ 16u); y1.y = __shfl_sync(0xFFFFFFFFu, q.y, src ^ 16u);
  y1.z = __shfl_sync(0xFFFFFFFFu, q.z, src ^ 16u); y1.w = __shfl_sync(0xFFFFFFFFu, q.w, src ^ 16u);
  if ((vm >> (lane >> 1)) & 1u) st_stream<EF>(dst + lane, sel4(odd, y1, y0), pol);
  if ((vm >> (16u + (lane >> 1))) & 1u) st_stream<EF>(dst + 32 + lane, sel4(odd, y0, y1), pol);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  for (;;) {
    uint32_t done;
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                 : "=r"(done) : "r"(smem_u32(bar)), "r"(phase) : "memory");
    if (done) return;
  }
}
__device__ __forceinline__ void tma_load(void* s, const void* g, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(s)), "l"(g), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
template <bool EF>
__device__ __forceinline__ void tma_store(void* g, const void* s, uint32_t bytes, uint64_t pol) {
  if (EF) asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;"
                       :: "l"(g), "r"(smem_u32(s)), "r"(bytes), "l"(pol) : "memory");
  else asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" :: "l"(g), "r"(smem_u32(s)), "r"(bytes) : "memory");
}

struct args { const uint8_t* arena; const uint4* plan; uint4* hdr_out; uint8_t* payload_out; uint32_t total; };
__device__ __forceinline__ const uint8_t* payload_of(const uint8_t* arena, uint32_t handle, uint32_t dm1) {
  return arena + ((static_cast<uint64_t>(handle) + 1u + dm1) << 5);
}

// A (HDR = true) and P (HDR = false), EF: evict-first bulk stores, HEF: evict-first header stores; lane per record, two stages per warp, one TMA load of the payload per lane,
// one 8 KB bulk store per warp step when all 32 payloads fill their slots
template <bool HDR, bool EF, bool HEF = false>
__global__ void __launch_bounds__(WARPS * 32) k_gather(args a) {
  extern __shared__ __align__(128) uint8_t s_dyn[];
  __shared__ __align__(8) uint64_t s_bar[WARPS][2];
  const uint32_t total = a.total, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* const wbase = s_dyn + static_cast<size_t>(warp) * 2u * 32u * SLOT;
  if (lane == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(&s_bar[warp][0])));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(&s_bar[warp][1])));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  const uint64_t pol = (EF || HEF) ? pol_evict_first() : 0ull;
  const uint32_t gw = blockIdx.x * WARPS + warp, nw = gridDim.x * WARPS;
  uint32_t phase = 0, g0 = 0, g1 = 0; uint64_t po0 = 0, po1 = 0; bool hv0 = false, hv1 = false;
  uint4 ha0 = make_uint4(0, 0, 0, 0), hb0 = ha0, ha1 = ha0, hb1 = ha0, pe_ahead = ha0;
  auto issue = [&](uint32_t st, uint32_t r0) {
    const uint32_t rec = r0 + lane;
    const bool have = rec < total;
    uint32_t bytes = 0; uint4 pe = make_uint4(0, 0, 0, 0);
    if (have) { pe = pe_ahead; bytes = (pe.z & 0xFFFFu) << 5; }
    { const uint32_t ra = rec + nw * 32u; if (ra < total) pe_ahead = __ldg(a.plan + ra); }
    uint32_t sum = bytes;
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, o);
    if (lane == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(&s_bar[warp][st])), "r"(sum) : "memory");
    __syncwarp();
    uint4 ha = make_uint4(0, 0, 0, 0), hb = ha;
    if (have) {
      if (HDR) { const uint8_t* src = a.arena + (static_cast<uint64_t>(pe.x) << 5); ha = ld_stream<false>(src, 0); hb = ld_stream<false>(src + 16, 0); }
      if (bytes) tma_load(wbase + (static_cast<size_t>(st) * 32u + lane) * SLOT, payload_of(a.arena, pe.x, pe.z >> 16), bytes, &s_bar[warp][st]);
    }
    if (st) { g1 = pe.z & 0xFFFFu; hv1 = have; po1 = pe.y; ha1 = ha; hb1 = hb; }
    else { g0 = pe.z & 0xFFFFu; hv0 = have; po0 = pe.y; ha0 = ha; hb0 = hb; }
  };
  uint32_t r0 = gw * 32u, st = 0;
  if (r0 + lane < total) pe_ahead = __ldg(a.plan + r0 + lane);
  if (r0 < total) issue(0, r0);
  for (; r0 < total; r0 += nw * 32u, st ^= 1u) {
    const uint32_t rn = r0 + nw * 32u;
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    __syncwarp();
    if (rn < total) issue(st ^ 1u, rn);
    if (HDR) st_headers32<HEF>(a.hdr_out + r0 * 2u, sel4(st, ha1, ha0), sel4(st, hb1, hb0), st ? hv1 : hv0, lane, 0);
    mbar_wait(&s_bar[warp][st], (phase >> st) & 1u);
    phase ^= 1u << st;
    const bool hv = st ? hv1 : hv0;
    const uint32_t g = st ? g1 : g0;
    if (__all_sync(0xFFFFFFFFu, hv && (g << 5) == SLOT)) {
      if (lane == 0) tma_store<EF>(a.payload_out + ((st ? po1 : po0) << 5), wbase + static_cast<size_t>(st) * 32u * SLOT, 32u * SLOT, pol);
    } else if (hv && g) {
      tma_store<EF>(a.payload_out + ((st ? po1 : po0) << 5), wbase + (static_cast<size_t>(st) * 32u + lane) * SLOT, g << 5, pol);
    }
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  }
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// H: flat over output records, lane per record, U warp steps of loads in flight before their stores
template <int U, bool EF>
__global__ void __launch_bounds__(256) k_headers(args a) {
  const uint32_t total = a.total, lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const uint64_t pol = EF ? pol_evict_first() : 0ull;
  for (uint32_t r0 = gw * 32u * U; r0 < total; r0 += nw * 32u * U) {
    uint32_t h[U]; uint4 lo[U], hi[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { const uint32_t rec = r0 + u * 32u + lane; h[u] = rec < total ? __ldg(&a.plan[rec].x) : 0u; }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint8_t* src = a.arena + (static_cast<uint64_t>(h[u]) << 5);
      lo[u] = make_uint4(0, 0, 0, 0); hi[u] = lo[u];
      if (r0 + u * 32u + lane < total) { lo[u] = ld_stream<EF>(src, pol); hi[u] = ld_stream<EF>(src + 16, pol); }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) st_headers32<EF>(a.hdr_out + (r0 + u * 32u) * 2u, lo[u], hi[u], r0 + u * 32u + lane < total, lane, pol);
  }
}

// W: the same 1.21 GB of output as whole sectors, coalesced
__global__ void __launch_bounds__(256) k_write(uint4* p0, size_t n0, uint4* p1, size_t n1) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n0 + n1; i += stride) {
    const uint4 v = make_uint4(static_cast<uint32_t>(i), 1u, 2u, 3u);
    if (i < n0) st_stream<false>(p0 + i, v, 0); else st_stream<false>(p1 + (i - n0), v, 0);
  }
}

__global__ void k_fill(uint32_t* p, size_t n, uint32_t seed) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    p[i] = hash32(static_cast<uint32_t>(i) ^ seed) ^ hash32(static_cast<uint32_t>(i >> 32) + seed);
}

// every output record against the arena: header at handle, payload at handle + 1 + dm1
__global__ void k_check(args a, unsigned long long* bad) {
  unsigned long long c = 0;
  for (uint32_t rec = blockIdx.x * blockDim.x + threadIdx.x; rec < a.total; rec += gridDim.x * blockDim.x) {
    const uint4 pe = a.plan[rec];
    const uint4* h = reinterpret_cast<const uint4*>(a.arena + (static_cast<uint64_t>(pe.x) << 5));
    for (uint32_t k = 0; k < 2; ++k) {
      const uint4 x = a.hdr_out[2 * rec + k], y = h[k];
      c += (x.x != y.x) | (x.y != y.y) | (x.z != y.z) | (x.w != y.w);
    }
    const uint4* p = reinterpret_cast<const uint4*>(payload_of(a.arena, pe.x, pe.z >> 16));
    const uint4* o = reinterpret_cast<const uint4*>(a.payload_out + (static_cast<uint64_t>(pe.y) << 5));
    for (uint32_t k = 0; k < 2 * (pe.z & 0xFFFFu); ++k) c += (o[k].x != p[k].x) | (o[k].y != p[k].y) | (o[k].z != p[k].z) | (o[k].w != p[k].w);
  }
  if (c) atomicAdd(bad, c);
}

int main() {
  int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  // ---- the c2 arena and its plan (seeded): agents into random groups of 64, sends to random groups
  const uint32_t seed = 0x5EEDu;
  std::vector<uint32_t> perm(AGENTS);
  for (uint32_t i = 0; i < AGENTS; ++i) perm[i] = i;
  for (uint32_t i = AGENTS - 1; i > 0; --i) std::swap(perm[i], perm[hash32(i ^ seed) % (i + 1)]);
  std::vector<uint32_t> grp(SENDS), cnt(AGENTS + 1, 0);
  for (uint32_t s = 0; s < SENDS; ++s) {
    grp[s] = hash32(s * 0x9E3779B1u + seed) % GROUPS;
    for (uint32_t j = 0; j < FAN; ++j) ++cnt[perm[grp[s] * FAN + j]];
  }
  std::vector<uint32_t> off(AGENTS + 1, 0);
  for (uint32_t a = 0; a < AGENTS; ++a) off[a + 1] = off[a] + cnt[a];
  std::vector<uint4> plan(RECS);
  for (uint32_t s = 0; s < SENDS; ++s)                                     // each agent's records in send order
    for (uint32_t j = 0; j < FAN; ++j) {
      const uint32_t a = perm[grp[s] * FAN + j], rec = off[a]++;
      plan[rec] = make_uint4(s * SEND_G + j, rec * PG, PG | ((FAN - 1u - j) << 16), a);
    }
  const size_t arena_bytes = static_cast<size_t>(SENDS) * SEND_G * 32, hdr_bytes = static_cast<size_t>(RECS) * 32,
               pay_bytes = static_cast<size_t>(RECS) * PG * 32;
  uint8_t *arena, *pay; uint4 *dplan, *hdr; unsigned long long* bad;
  CK(cudaMalloc(&arena, arena_bytes)); CK(cudaMalloc(&dplan, RECS * sizeof(uint4)));
  CK(cudaMalloc(&hdr, hdr_bytes)); CK(cudaMalloc(&pay, pay_bytes)); CK(cudaMalloc(&bad, 8));
  k_fill<<<4 * sms, 256>>>(reinterpret_cast<uint32_t*>(arena), arena_bytes / 4, seed);
  CK(cudaMemcpy(dplan, plan.data(), RECS * sizeof(uint4), cudaMemcpyHostToDevice));
  const args ga{arena, dplan, hdr, pay, RECS};

  // launch shapes of the library (launch_gather): 4 warps, 64 KB of slots per CTA, 8 waves; headers 8 warps per CTA
  const size_t smem = static_cast<size_t>(WARPS) * 2u * 32u * SLOT;
  uint32_t per_sm = static_cast<uint32_t>((226u * 1024u) / (smem + 1024 + 128));
  per_sm = std::min(8u, std::max(1u, per_sm));
  const uint32_t tma_grid = std::min<uint64_t>(static_cast<uint64_t>(sms) * per_sm * 8u, (RECS + WARPS * 32 - 1) / (WARPS * 32));
  CK(cudaFuncSetAttribute(k_gather<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  CK(cudaFuncSetAttribute(k_gather<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  CK(cudaFuncSetAttribute(k_gather<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  CK(cudaFuncSetAttribute(k_gather<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  CK(cudaFuncSetAttribute(k_gather<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  auto hgrid = [&](int u) { return std::min<uint32_t>(32u * sms, (RECS + 256u * u - 1) / (256u * u)); };

  struct mode { const char* name; int id; };
  const mode modes[] = {{"A  interleaved (today)", 0}, {"H  headers, U=4", 1}, {"H  headers, U=8", 2}, {"H  headers, U=4, ef", 3},
                        {"P  payloads", 4}, {"P  payloads, ef store", 5}, {"H+P      (U=4)", 6}, {"H+P ef store (U=4)", 7},
                        {"H ef + P ef (U=4)", 8}, {"H+P      (U=8)", 9}, {"W  write stream 1.21 GB", 10},
                        {"A  ef bulk store", 11}, {"A  ef bulk + header store", 12}};
  const int NM = sizeof(modes) / sizeof(modes[0]);
  auto launch = [&](int id) {
    switch (id) {
      case 0: k_gather<true, false><<<tma_grid, WARPS * 32, smem>>>(ga); break;
      case 1: k_headers<4, false><<<hgrid(4), 256>>>(ga); break;
      case 2: k_headers<8, false><<<hgrid(8), 256>>>(ga); break;
      case 3: k_headers<4, true><<<hgrid(4), 256>>>(ga); break;
      case 4: k_gather<false, false><<<tma_grid, WARPS * 32, smem>>>(ga); break;
      case 5: k_gather<false, true><<<tma_grid, WARPS * 32, smem>>>(ga); break;
      case 6: k_headers<4, false><<<hgrid(4), 256>>>(ga); k_gather<false, false><<<tma_grid, WARPS * 32, smem>>>(ga); break;
      case 7: k_headers<4, false><<<hgrid(4), 256>>>(ga); k_gather<false, true><<<tma_grid, WARPS * 32, smem>>>(ga); break;
      case 8: k_headers<4, true><<<hgrid(4), 256>>>(ga); k_gather<false, true><<<tma_grid, WARPS * 32, smem>>>(ga); break;
      case 9: k_headers<8, false><<<hgrid(8), 256>>>(ga); k_gather<false, false><<<tma_grid, WARPS * 32, smem>>>(ga); break;
      case 11: k_gather<true, true><<<tma_grid, WARPS * 32, smem>>>(ga); break;
      case 12: k_gather<true, true, true><<<tma_grid, WARPS * 32, smem>>>(ga); break;
      case 10: k_write<<<4 * sms, 256>>>(reinterpret_cast<uint4*>(pay), pay_bytes / 16, hdr, hdr_bytes / 16); break;
    }
  };
  // correctness of every complete copy (A and the splits) before timing
  for (int id : {0, 6, 7, 8, 9, 11, 12}) {
    CK(cudaMemset(hdr, 0, hdr_bytes)); CK(cudaMemset(pay, 0, pay_bytes)); CK(cudaMemset(bad, 0, 8));
    launch(id);
    k_check<<<4 * sms, 256>>>(ga, bad);
    unsigned long long nb = 0; CK(cudaMemcpy(&nb, bad, 8, cudaMemcpyDeviceToHost));
    CK(cudaGetLastError());
    printf("check %-24s: %llu mismatching words\n", modes[id].name, nb);
    if (nb) return 1;
  }
  // timing: ROUNDS rounds, every mode once per round (drift on a shared host shows as spread, not as a bias)
  const int ROUNDS = 9;
  std::vector<std::vector<float>> t(NM);
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  for (int id = 0; id < NM; ++id) launch(id);                                // warm-up
  for (int r = 0; r < ROUNDS; ++r)
    for (int id = 0; id < NM; ++id) {
      CK(cudaEventRecord(e0)); launch(id); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); t[id].push_back(ms);
    }
  CK(cudaGetLastError());
  // algorithmic bytes: plan 16 B + header in 32 B + header out 32 B + payload out 256 B per record, the shared payload once
  const double b_plan = RECS * 16.0, b_hin = RECS * 32.0, b_hout = hdr_bytes, b_pout = pay_bytes, b_pin = SENDS * PG * 32.0;
  const double bytes[] = {b_plan + b_hin + b_hout + b_pout + b_pin, b_plan + b_hin + b_hout, b_plan + b_hin + b_hout,
                          b_plan + b_hin + b_hout, b_plan + b_pout + b_pin, b_plan + b_pout + b_pin,
                          2 * b_plan + b_hin + b_hout + b_pout + b_pin, 2 * b_plan + b_hin + b_hout + b_pout + b_pin,
                          2 * b_plan + b_hin + b_hout + b_pout + b_pin, 2 * b_plan + b_hin + b_hout + b_pout + b_pin,
                          b_hout + b_pout, b_plan + b_hin + b_hout + b_pout + b_pin, b_plan + b_hin + b_hout + b_pout + b_pin};
  printf("%s, %d SMs; c2 gather: %u records, %u sends x %u members; %d rounds\n", prop.name, sms, RECS, SENDS, FAN, ROUNDS);
  printf("%-26s %9s %9s %9s %9s\n", "mode", "best ms", "median", "worst", "GB/s");
  for (int id = 0; id < NM; ++id) {
    std::vector<float> s = t[id]; std::sort(s.begin(), s.end());
    printf("%-26s %9.4f %9.4f %9.4f %9.0f\n", modes[id].name, s[0], s[s.size() / 2], s.back(), bytes[id] / (s[s.size() / 2] * 1e6));
  }
  return 0;
}
