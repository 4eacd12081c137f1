// Micro-benchmark (H100): cost of scattered small stores vs full-sector stores into a large (512 MiB) array,
// of dependent random loads, and of the ways a warp can write a stream of 32-byte headers.  Informs the ring-entry
// append design (sdb_send.cu: index build) and the header stores of the group fan-out and the receive gathers.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/ubench/stores scripts/ubench/stores.cu
// NVIDIA H100 80GB HBM3, 400 W power limit, best of 5 launches: a quad writing one aligned full sector per agent
// (mode 3) 0.0167 ms, the same quad writing 4 entries from an unaligned slot, i.e. two partial sectors (mode 5),
// 0.0271 ms; 4 separate 8-byte stores per agent (mode 0) 0.1765 ms.  Mode 2 (one 32-byte store per thread) needs sm_100.
// NVIDIA H100 80GB HBM3, 700 W power limit, 1980 MHz max SM clock, best of 5 launches: mode 3 0.0169 ms, mode 5
// 0.0266 ms, two 16-byte stores per agent (mode 1) 0.0604 ms, mode 0 0.1770 ms.
// Header streams on the same card (1 GiB of 32-byte records, 1 KB per warp step, equal bytes, best of 7): two 16-byte
// stores per lane, i.e. every sector written as two halves by two instructions (mode a), 0.693 ms = 1549 GB/s; the
// halves shuffled so that a lane pair writes each sector in one instruction (mode b) 0.340 ms = 3155 GB/s; one 1 KB
// bulk store from shared memory per warp step (mode c) 0.341 ms = 3151 GB/s.  A sector that reaches the L2 in two
// partial writes costs about twice its bytes: consistent with the L2 filling the sector from DRAM before merging.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); return 1; } } while (0)

__device__ __forceinline__ uint32_t hash32(uint32_t x) { x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; return x; }

// n agents, each owns a 512-byte ring (64 x 8 B); thread per agent writes K consecutive 8-byte entries at slot `pos`
template <int MODE>
__global__ void k_store(uint8_t* ring, uint32_t n, uint32_t pos, uint32_t K) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const uint32_t a = hash32(t) % n;                       // random agent per thread (a permutation is not needed)
  uint8_t* base = ring + (size_t)a * 512;
  if (MODE == 0) {                                        // K separate 8-byte stores (partial sector each)
    for (uint32_t k = 0; k < K; ++k) *reinterpret_cast<uint64_t*>(base + ((pos + k) & 63) * 8) = ((uint64_t)t << 32) | k;
  } else if (MODE == 1) {                                 // two 16-byte stores (aligned slot pairs), K = 4
    uint4 v = make_uint4(t, 0, t, 1);
    const uint32_t p = pos & ~1u;
    *reinterpret_cast<uint4*>(base + (p & 63) * 8) = v;
    *reinterpret_cast<uint4*>(base + ((p + 2) & 63) * 8) = v;
  } else if (MODE == 2) {                                 // one 32-byte store (full sector), K = 4: sm_100 and later only
#if __CUDA_ARCH__ >= 1000
    const uint32_t p = pos & ~3u;
    uint8_t* d = base + (p & 63) * 8;
    asm volatile("st.global.v8.b32 [%0], {%1,%2,%3,%4,%5,%6,%7,%8};" :: "l"(d), "r"(t), "r"(0), "r"(t), "r"(1), "r"(t), "r"(2), "r"(t), "r"(3) : "memory");
#endif
  } else if (MODE == 3) {                                 // full sector written by 4 lanes x 8 B in ONE instruction (quad per agent)
    const uint32_t q = t >> 2, sub = t & 3;
    const uint32_t a2 = hash32(q) % n;
    const uint32_t p = pos & ~3u;
    *reinterpret_cast<uint64_t*>(ring + (size_t)a2 * 512 + ((p + sub) & 63) * 8) = ((uint64_t)t << 32) | sub;
  } else if (MODE == 5) {                                 // quad per agent, 4 x 8B in ONE instruction from an unaligned slot:
    const uint32_t q = t >> 2, sub = t & 3;               // two partial sectors (the index build's append before whole sectors)
    const uint32_t a2 = hash32(q) % n;
    const uint32_t p = (pos & ~3u) + 1u;
    *reinterpret_cast<uint64_t*>(ring + (size_t)a2 * 512 + ((p + sub) & 63) * 8) = ((uint64_t)t << 32) | sub;
  } else if (MODE == 4) {                                 // read-modify-write of the sector: 2 x 16 B load, 2 x 16 B store
    const uint32_t p = pos & ~3u;
    uint4* d = reinterpret_cast<uint4*>(base + (p & 63) * 8);
    uint4 x = d[0], y = d[1];
    x.x = t; y.w = t;
    d[0] = x; d[1] = y;
  }
}

// A contiguous stream of 32-byte records (the receive gather's hdr_out, a group send's headers), one record per lane, so
// a warp step covers 1 KB.  MODE 'a': each lane stores its record as two 16-byte halves (lo, then hi): every store
// instruction writes half of each of 32 sectors.  MODE 'b': the halves are exchanged with __shfl_sync so that lanes
// 2k, 2k+1 store the two halves of one record in the same instruction: two instructions of 512 contiguous bytes, whole
// sectors.  MODE 'c': the lanes put their records into a 1 KB shared-memory slot and one lane issues one bulk (TMA)
// store of it (two slots per warp, the older store must have read its slot before the slot is refilled).
template <char MODE>
__global__ void __launch_bounds__(256) k_hdr_stream(uint4* out, uint32_t steps) {
  __shared__ __align__(128) uint4 s_slot[8][2][64];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t gw = blockIdx.x * 8 + warp, nw = gridDim.x * 8;
  uint32_t k = 0;
  for (uint32_t s = gw; s < steps; s += nw, k ^= 1u) {
    const uint32_t rec = s * 32u + lane;
    const uint4 lo = make_uint4(rec, s, ~rec, 1u), hi = make_uint4(rec * 3u, lane, s ^ rec, 2u);
    uint4* w = out + static_cast<size_t>(s) * 64u;                   // the warp's 1 KB
    if (MODE == 'a') {
      w[2 * lane] = lo; w[2 * lane + 1] = hi;
    } else if (MODE == 'b') {
      const bool odd = lane & 1u, low = lane < 16u;
      const uint32_t src = (lane >> 1) + (odd ? 16u : 0u);
      const uint4 p = low ? lo : hi, q = low ? hi : lo;
      uint4 y0, y1;
      y0.x = __shfl_sync(0xFFFFFFFFu, p.x, src); y0.y = __shfl_sync(0xFFFFFFFFu, p.y, src);
      y0.z = __shfl_sync(0xFFFFFFFFu, p.z, src); y0.w = __shfl_sync(0xFFFFFFFFu, p.w, src);
      y1.x = __shfl_sync(0xFFFFFFFFu, q.x, src ^ 16u); y1.y = __shfl_sync(0xFFFFFFFFu, q.y, src ^ 16u);
      y1.z = __shfl_sync(0xFFFFFFFFu, q.z, src ^ 16u); y1.w = __shfl_sync(0xFFFFFFFFu, q.w, src ^ 16u);
      w[lane] = odd ? y1 : y0; w[32 + lane] = odd ? y0 : y1;
    } else if (MODE == 'c') {
      if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      __syncwarp();
      s_slot[warp][k][2 * lane] = lo; s_slot[warp][k][2 * lane + 1] = hi;
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) {
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], 1024;"
                     :: "l"(w), "r"(static_cast<uint32_t>(__cvta_generic_to_shared(&s_slot[warp][k][0]))) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
    }
  }
  if (MODE == 'c' && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

template <char MODE>
float run_hdr(uint4* out, uint32_t steps, int blocks) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  float best = 1e9;
  for (int it = 0; it < 8; ++it) {
    cudaEventRecord(a);
    k_hdr_stream<MODE><<<blocks, 256>>>(out, steps);
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    if (it > 0 && ms < best) best = ms;
  }
  return best;
}

__global__ void k_diff(const uint4* x, const uint4* y, size_t n, unsigned long long* bad) {
  unsigned long long c = 0;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const uint4 a = x[i], b = y[i];
    c += (a.x != b.x) | (a.y != b.y) | (a.z != b.z) | (a.w != b.w);
  }
  if (c) atomicAdd(bad, c);
}

// dependent random loads: chain of depth D through a table
__global__ void k_chain(const uint32_t* tab, uint32_t n, uint32_t D, uint32_t* out) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  uint32_t x = hash32(t) % n;
  for (uint32_t d = 0; d < D; ++d) x = tab[x];
  out[t] = x;
}

template <int MODE>
float run(uint8_t* ring, uint32_t n, uint32_t threads_per_agent, uint32_t K) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  const uint32_t nt = n * threads_per_agent;
  float best = 1e9;
  for (int it = 0; it < 6; ++it) {
    cudaEventRecord(a);
    k_store<MODE><<<(nt + 255) / 256, 256>>>(ring, n, 4 * it + 1, K);
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    if (it > 0 && ms < best) best = ms;
  }
  return best;
}

int main() {
  const uint32_t n = 1u << 20;
  uint8_t* ring; CK(cudaMalloc(&ring, (size_t)n * 512)); CK(cudaMemset(ring, 0, (size_t)n * 512));
  printf("1M agents x 512 B rings (512 MiB), 4 entries per agent per launch\n");
  printf("mode0 4 x 8B stores (partial)        : %.4f ms\n", run<0>(ring, n, 1, 4));
  printf("mode0 1 x 8B store  (partial)        : %.4f ms\n", run<0>(ring, n, 1, 1));
  printf("mode1 2 x 16B stores (half sectors)  : %.4f ms\n", run<1>(ring, n, 1, 4));
  printf("mode3 4 lanes x 8B one instr (quad)  : %.4f ms\n", run<3>(ring, n, 4, 4));
  printf("mode5 quad, unaligned (2 partial)    : %.4f ms\n", run<5>(ring, n, 4, 4));
  printf("mode3 again (after mode5)            : %.4f ms\n", run<3>(ring, n, 4, 4));
  printf("mode4 RMW 2x16B load + 2x16B store   : %.4f ms\n", run<4>(ring, n, 1, 4));
  uint32_t* tab; uint32_t* out; CK(cudaMalloc(&tab, (size_t)n * 64 * 4)); CK(cudaMalloc(&out, n * 4));
  // table of 64M entries (256 MiB) filled with pseudo-random indices
  {
    uint32_t* h = (uint32_t*)malloc((size_t)n * 64 * 4);
    uint32_t s = 12345; for (size_t i = 0; i < (size_t)n * 64; ++i) { s = s * 1664525u + 1013904223u; h[i] = (s >> 6) % (n * 64); }
    CK(cudaMemcpy(tab, h, (size_t)n * 64 * 4, cudaMemcpyHostToDevice)); free(h);
  }
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  for (uint32_t D : {1u, 2u, 4u, 8u}) {
    float best = 1e9;
    for (int it = 0; it < 4; ++it) {
      cudaEventRecord(a); k_chain<<<n / 256, 256>>>(tab, n * 64, D, out); cudaEventRecord(b); cudaEventSynchronize(b);
      float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms;
    }
    printf("chain depth %u, 1M threads, 256 MiB table: %.4f ms\n", D, best);
  }
  // wait: chain uses n*64 as modulus but launches n threads
  CK(cudaFree(tab)); CK(cudaFree(out)); CK(cudaFree(ring));

  // header streams: 1 GiB of 32-byte records, far larger than the L2; every mode writes the same bytes
  const uint32_t steps = 1u << 20;                                      // 1 KB per warp step
  const size_t bytes = static_cast<size_t>(steps) << 10;
  int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  uint4 *h0, *h1; CK(cudaMalloc(&h0, bytes)); CK(cudaMalloc(&h1, bytes));
  unsigned long long* bad; CK(cudaMalloc(&bad, 8));
  printf("header stream: %u MiB of 32-byte records, one per lane, 1 KB per warp step, %d x 256 threads\n",
         static_cast<uint32_t>(bytes >> 20), 4 * sms);
  const float ta = run_hdr<'a'>(h0, steps, 4 * sms);
  printf("a 2 x 16B per lane (half sectors)    : %.4f ms  %.0f GB/s\n", ta, bytes / (ta * 1e6));
  const char* names[2] = {"b shuffled pairs (whole sectors)    ", "c 1 KB bulk store from shared       "};
  for (int m = 0; m < 2; ++m) {
    CK(cudaMemset(h1, 0, bytes)); CK(cudaMemset(bad, 0, 8));
    const float t = m == 0 ? run_hdr<'b'>(h1, steps, 4 * sms) : run_hdr<'c'>(h1, steps, 4 * sms);
    k_diff<<<4 * sms, 256>>>(h0, h1, bytes / 16, bad);
    unsigned long long nb = 0; CK(cudaMemcpy(&nb, bad, 8, cudaMemcpyDeviceToHost));
    printf("%s: %.4f ms  %.0f GB/s  (%llu 16-byte words differ from a)\n", names[m], t, bytes / (t * 1e6), nb);
  }
  const float ta2 = run_hdr<'a'>(h0, steps, 4 * sms);
  printf("a again                              : %.4f ms  %.0f GB/s\n", ta2, bytes / (ta2 * 1e6));
  CK(cudaGetLastError());
  return 0;
}
