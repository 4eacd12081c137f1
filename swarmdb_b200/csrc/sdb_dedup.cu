// sdb_dedup.cu - deduplication of sends (sdb_send_mixed_batch_dedup, sdb_dedup_forget, sdb_dedup_stats).
//
// The table is open addressing with linear probing over 128-bit keys, one 32-byte entry (one DRAM sector) per key:
// {key_lo, key_hi, seq, inserted_at}.  Key {0,0} marks an empty slot.  An entry is live while now < inserted_at +
// window; sdb_dedup_forget kills an entry in place by setting inserted_at to -inf, so a forgotten key is an expired one.
// A key has at most one entry: an insert reuses the slot its key already holds.  Dead entries keep their slot (probe
// chains stay intact) until the host rebuilds the table into its second buffer with the live entries only.
//
// Content keys (SDB_DEDUP_CONTENT) hash the identity of a send as a sequence of 64-bit words w_0 .. w_{m-1}:
//   w_0 = sender | kind << 32,  w_1 = target (kind 0, 1) or the list's length (kind 2),
//   then for a list send its recipients, one word each,  then len | prio << 16 | type << 24,
//   then the payload as little-endian words, bytes past len zero.
// Two lanes: S_x = sum_j mix64(w_j + SEED_x + (j + 1) * PHI) mod 2^64, key = {mix64(S_a ^ m), mix64(S_b ^ (m << 32))},
// {0,0} replaced by {1,0}.  mix64 is the splitmix64 finaliser.  The position term makes the key order-sensitive and the
// sum lets one warp reduce it.  tests/dedup_ref.py reproduces it in numpy.
#include <cuda_runtime.h>
#include <math.h>

#include <algorithm>

#include "sdb_common.cuh"

namespace {

constexpr unsigned long long PHI = 0x9E3779B97F4A7C15ull;
constexpr unsigned long long SEED_A = 0x243F6A8885A308D3ull;
constexpr unsigned long long SEED_B = 0x13198A2E03707344ull;

__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

struct __align__(16) key128 { unsigned long long lo, hi; };

// 128-bit compare-and-swap of a 16-byte aligned key (sm_90)
__device__ __forceinline__ sdb_dedup_key cas_key(sdb_dedup_key* p, const sdb_dedup_key& k) {
  const key128 old = atomicCAS(reinterpret_cast<key128*>(p), key128{0ull, 0ull}, key128{k.lo, k.hi});
  return sdb_dedup_key{old.lo, old.hi};
}

__device__ __forceinline__ bool key_zero(const sdb_dedup_key& k) { return (k.lo | k.hi) == 0ull; }
__device__ __forceinline__ bool key_eq(const sdb_dedup_key& a, const sdb_dedup_key& b) { return a.lo == b.lo && a.hi == b.hi; }
__device__ __forceinline__ unsigned long long slot_hash(const sdb_dedup_key& k) { return mix64(k.lo ^ ((k.hi << 32) | (k.hi >> 32))); }
__device__ __forceinline__ bool live(double at, double now, double window) { return now < at + window; }

__device__ __forceinline__ void term(unsigned long long w, unsigned long long j, unsigned long long& a, unsigned long long& b) {
  const unsigned long long p = (j + 1ull) * PHI;
  a += mix64(w + SEED_A + p);
  b += mix64(w + SEED_B + p);
}

// one warp per send: content key of every send whose key is {0,0}
__global__ void __launch_bounds__(256) k_dedup_content(const sdb_dedup_send* __restrict__ snd, uint32_t n,
                                                       const uint8_t* __restrict__ payload, const uint32_t* __restrict__ lists,
                                                       sdb_dedup_key* key) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
    const sdb_dedup_key k0 = key[i];
    if (!key_zero(k0)) continue;
    const sdb_dedup_send s = snd[i];
    const uint32_t kind = s.kind, len = s.lpt & 0xFFFFu;
    const uint64_t cnt = kind == 2 ? s.target : 0;
    unsigned long long a = 0, b = 0;
    if (lane == 0) term(s.sender | (static_cast<unsigned long long>(kind) << 32), 0, a, b);
    if (lane == 1) term(s.target, 1, a, b);
    for (uint64_t x = lane; x < cnt; x += 32) term(lists[s.list_b + x], 2 + x, a, b);
    if (lane == 2) term(s.lpt, 2 + cnt, a, b);
    const unsigned long long j0 = 3 + cnt;
    const uint8_t* p = payload + s.payload_off;          // 16-byte aligned
    for (uint32_t q = lane; q * 16u < len; q += 32) {    // coalesced 16-byte loads, two words each
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(p) + q);
      unsigned long long w0 = (static_cast<unsigned long long>(v.y) << 32) | v.x;
      unsigned long long w1 = (static_cast<unsigned long long>(v.w) << 32) | v.z;
      const uint32_t b0 = q * 16u;
      if (len - b0 < 8u) w0 &= (1ull << (8u * (len - b0))) - 1ull;
      term(w0, j0 + 2ull * q, a, b);
      if (b0 + 8u < len) {
        if (len - b0 - 8u < 8u) w1 &= (1ull << (8u * (len - b0 - 8u))) - 1ull;
        term(w1, j0 + 2ull * q + 1ull, a, b);
      }
    }
    for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xFFFFFFFFu, a, o); b += __shfl_xor_sync(0xFFFFFFFFu, b, o); }
    if (lane == 0) {
      const unsigned long long m = j0 + (len + 7u) / 8u;
      sdb_dedup_key k{mix64(a ^ m), mix64(b ^ (m << 32))};
      if (key_zero(k)) k.lo = 1;
      key[i] = k;
    }
  }
}

// thread per send: look the key up in the table (read-only) and claim its slot in the batch table, where the lowest
// send index holding the key wins (atomicMin)
__global__ void k_dedup_probe(const sdb_dedup_entry* __restrict__ tab, unsigned long long mask, double now, double window,
                              const sdb_dedup_key* __restrict__ key, uint32_t n, sdb_dedup_key* btab, uint32_t* bmin,
                              unsigned long long bmask, uint32_t* bslot, unsigned long long* verdict) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const sdb_dedup_key k = key[i];
  unsigned long long v = 0;
  uint32_t bs = 0xFFFFFFFFu;
  if (!key_zero(k)) {
    const unsigned long long h = slot_hash(k);
    for (unsigned long long s = h & mask;; s = (s + 1) & mask) {
      const sdb_dedup_entry e = tab[s];
      if (key_zero(e.key)) break;
      if (key_eq(e.key, k)) { if (live(e.at, now, window)) v = e.seq; break; }
    }
    for (unsigned long long s = h & bmask;; s = (s + 1) & bmask) {
      const sdb_dedup_key old = cas_key(&btab[s], k);
      if (key_zero(old) || key_eq(old, k)) { atomicMin(&bmin[s], i); bs = static_cast<uint32_t>(s); break; }
    }
  }
  verdict[i] = v;
  bslot[i] = bs;
}

// verdict[i]: 0 accepted (new key or no key), a table entry's seq, or SDB_DD_BATCH | index of the earlier send of the
// batch with the same key.  ctr[SDB_DD_NEW] counts the new keys.
__global__ void k_dedup_verdict(const uint32_t* __restrict__ bmin, const uint32_t* __restrict__ bslot, uint32_t n,
                                unsigned long long* verdict, unsigned long long* ctr) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool fresh = false;
  if (i < n && bslot[i] != 0xFFFFFFFFu && verdict[i] == 0) {
    const uint32_t first = bmin[bslot[i]];
    if (first != i) verdict[i] = SDB_DD_BATCH | first;
    else fresh = true;
  }
  const uint32_t m = __ballot_sync(0xFFFFFFFFu, fresh);
  if ((threadIdx.x & 31u) == 0 && m) atomicAdd(&ctr[SDB_DD_NEW], static_cast<unsigned long long>(__popc(m)));
}

__device__ __forceinline__ void insert(sdb_dedup_entry* tab, unsigned long long mask, const sdb_dedup_key& k,
                                       unsigned long long seq, double at, unsigned long long* used) {
  for (unsigned long long s = slot_hash(k) & mask;; s = (s + 1) & mask) {
    const sdb_dedup_key old = cas_key(&tab[s].key, k);
    if (key_zero(old) || key_eq(old, k)) {
      tab[s].seq = seq; tab[s].at = at;
      if (key_zero(old)) atomicAdd(used, 1ull);
      return;
    }
  }
}

// thread per send: the accepted keyed sends of the batch store (key, first seq, now)
__global__ void k_dedup_insert(sdb_dedup_entry* tab, unsigned long long mask, const sdb_dedup_key* __restrict__ key,
                               const unsigned long long* __restrict__ verdict, const unsigned long long* __restrict__ seq_of,
                               uint32_t n, double now, unsigned long long* ctr) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const sdb_dedup_key k = key[i];
  if (key_zero(k) || verdict[i] != 0) return;
  insert(tab, mask, k, seq_of[i], now, &ctr[SDB_DD_USED]);
}

// thread per key: kill the entry of each key that is live at `now`; removed[i] = 1 where one was
__global__ void k_dedup_forget(sdb_dedup_entry* tab, unsigned long long mask, double now, double window,
                               const sdb_dedup_key* __restrict__ key, uint32_t n, uint8_t* removed, unsigned long long* ctr) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const sdb_dedup_key k = key[i];
  uint8_t r = 0;
  if (!key_zero(k)) {
    for (unsigned long long s = slot_hash(k) & mask;; s = (s + 1) & mask) {
      const sdb_dedup_key e = tab[s].key;
      if (key_zero(e)) break;
      if (key_eq(e, k)) {
        const double old = __longlong_as_double(atomicExch(reinterpret_cast<unsigned long long*>(&tab[s].at),
                                                           static_cast<unsigned long long>(__double_as_longlong(-INFINITY))));
        r = live(old, now, window) ? 1 : 0;
        break;
      }
    }
  }
  removed[i] = r;
  if (r) atomicAdd(&ctr[SDB_DD_FORGOT], 1ull);
}

// slot per thread: copy the entries live at `now` into the cleared table `dst` (rebuild), or only count them
__global__ void k_dedup_rebuild(const sdb_dedup_entry* __restrict__ src, sdb_dedup_entry* dst, unsigned long long mask,
                                double now, double window, unsigned long long* ctr) {
  const unsigned long long s = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  bool keep = false;
  if (s <= mask) {
    const sdb_dedup_entry e = src[s];
    keep = !key_zero(e.key) && live(e.at, now, window);
    if (keep && dst) insert(dst, mask, e.key, e.seq, e.at, &ctr[SDB_DD_USED]);
  }
  const uint32_t m = __ballot_sync(0xFFFFFFFFu, keep);
  if ((threadIdx.x & 31u) == 0 && m) atomicAdd(&ctr[SDB_DD_LIVE], static_cast<unsigned long long>(__popc(m)));
}

inline unsigned blocks(unsigned long long n, unsigned t) { return static_cast<unsigned>((n + t - 1) / t); }

}  // namespace

// The memsets of each launcher are enqueued before its profiler interval opens, so a failure returns with none open.
cudaError_t sdb_launch_dedup_probe(const sdb_dedup_args* a, uint32_t n, uint32_t content, double now, int sm_count,
                                   cudaStream_t stream, sdb_profiler* prof, int* n_launches) {
  const unsigned long long bmask = a->bmask;
  cudaError_t e = cudaMemsetAsync(a->btab, 0, (bmask + 1) * sizeof(sdb_dedup_key), stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(a->bmin, 0xFF, (bmask + 1) * sizeof(uint32_t), stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(a->ctr + SDB_DD_NEW, 0, sizeof(unsigned long long), stream);
  if (e != cudaSuccess) return e;
  const int pi = sdb_prof_begin(prof, SDB_PK_DEDUP, stream);
  int nl = 0;
  if (content) {      // one warp per send, 8 warps a block, at most 8 blocks an SM (grid-stride beyond)
    const unsigned grid = std::min(blocks(n, 8), 8u * static_cast<unsigned>(std::max(sm_count, 1)));
    k_dedup_content<<<grid, 256, 0, stream>>>(a->snd, n, a->payload, a->lists, a->key);
    ++nl;
  }
  k_dedup_probe<<<blocks(n, 256), 256, 0, stream>>>(a->tab, a->mask, now, a->window, a->key, n, a->btab, a->bmin, bmask,
                                                    a->bslot, a->verdict);
  k_dedup_verdict<<<blocks(n, 256), 256, 0, stream>>>(a->bmin, a->bslot, n, a->verdict, a->ctr);
  nl += 2;
  sdb_prof_end(prof, pi, stream);
  if (n_launches) *n_launches = nl;
  return cudaGetLastError();
}

cudaError_t sdb_launch_dedup_insert(const sdb_dedup_args* a, uint32_t n, double now, cudaStream_t stream, sdb_profiler* prof) {
  const int pi = sdb_prof_begin(prof, SDB_PK_DEDUP, stream);
  k_dedup_insert<<<blocks(n, 256), 256, 0, stream>>>(a->tab, a->mask, a->key, a->verdict, a->seq_of, n, now, a->ctr);
  sdb_prof_end(prof, pi, stream);
  return cudaGetLastError();
}

cudaError_t sdb_launch_dedup_forget(const sdb_dedup_args* a, uint32_t n, double now, uint8_t* removed, cudaStream_t stream,
                                    sdb_profiler* prof) {
  cudaError_t e = cudaMemsetAsync(a->ctr + SDB_DD_FORGOT, 0, sizeof(unsigned long long), stream);
  if (e != cudaSuccess) return e;
  const int pi = sdb_prof_begin(prof, SDB_PK_DEDUP, stream);
  k_dedup_forget<<<blocks(n, 256), 256, 0, stream>>>(a->tab, a->mask, now, a->window, a->key, n, removed, a->ctr);
  sdb_prof_end(prof, pi, stream);
  return cudaGetLastError();
}

// dst == nullptr: count the entries live at `now` into ctr[SDB_DD_LIVE]; else also rebuild them into dst (cleared here)
// and recount ctr[SDB_DD_USED]
cudaError_t sdb_launch_dedup_rebuild(const sdb_dedup_args* a, sdb_dedup_entry* dst, double now, cudaStream_t stream,
                                     sdb_profiler* prof) {
  const unsigned long long slots = a->mask + 1;
  cudaError_t e = cudaMemsetAsync(a->ctr + SDB_DD_LIVE, 0, sizeof(unsigned long long), stream);
  if (e == cudaSuccess && dst) e = cudaMemsetAsync(dst, 0, slots * sizeof(sdb_dedup_entry), stream);
  if (e == cudaSuccess && dst) e = cudaMemsetAsync(a->ctr + SDB_DD_USED, 0, sizeof(unsigned long long), stream);
  if (e != cudaSuccess) return e;
  const int pi = sdb_prof_begin(prof, SDB_PK_DEDUP, stream);
  k_dedup_rebuild<<<blocks(slots, 256), 256, 0, stream>>>(a->tab, dst, a->mask, now, a->window, a->ctr);
  sdb_prof_end(prof, pi, stream);
  return cudaGetLastError();
}
