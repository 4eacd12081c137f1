// Micro-benchmark (H100): cost of scattered small stores vs full-sector stores into a large (512 MiB) array,
// and of dependent random loads.  Informs the ring-entry append design (sdb_send.cu: index build).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/ubench/stores scripts/ubench/stores.cu
// NVIDIA H100 80GB HBM3, 400 W power limit, best of 5 launches: a quad writing one aligned full sector per agent
// (mode 3) 0.0167 ms, the same quad writing 4 entries from an unaligned slot, i.e. two partial sectors (mode 5),
// 0.0271 ms; 4 separate 8-byte stores per agent (mode 0) 0.1765 ms.  Mode 2 (one 32-byte store per thread) needs sm_100.
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
  return 0;
}
