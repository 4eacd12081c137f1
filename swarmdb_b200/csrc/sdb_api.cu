// sdb_api.cu - host side of the C ABI declared in include/swarmdb_b200.h.
//
// Owns: device memory of one shard, the host mirror of the group table (CSR), the global
// sequence counter, arena space accounting (tail / floor / reclaim), pinned staging for
// per-send descriptors, and the launch sequence of every entry point.  No CPU data path:
// every routed byte goes through the kernels in sdb_send.cu / sdb_recv.cu / sdb_balance.cu.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "sdb_common.cuh"

struct sdb_staged {
  uint32_t kind = 0;          // 0 p2p, 1 group, 2 list
  uint32_t n = 0;
  uint64_t total_recs = 0;    // sequence numbers consumed
  uint64_t total_grans = 0;   // arena granules consumed
  uint32_t max_padlen = 0;
  sdb_send_desc* descs_dev = nullptr;
  uint8_t* payload_dev = nullptr;
  uint32_t* list_dev = nullptr;
  uint32_t* gs_off_dev = nullptr;   // [max_groups + 1] group-send buckets (pull index build)
  uint32_t* gs_idx_dev = nullptr;   // [n]
  bool has_pull = false;      // group sends indexed by k_pull_index
  bool has_atomic = false;    // some sends claim ring slots with atomics -> k_commit must sort
  bool ranked = false;        // pure point-to-point batch ranked per receiver at staging time: no atomics, no sort
  bool shared = false;        // group sends laid out as headers + ONE payload per send (sdb_common.cuh "shared payloads")
  bool list_pull = false;     // pure broadcast batch over pairwise disjoint lists: ring entries built by k_list_index
  uint32_t lp_nd = 0, lp_max_count = 0, lp_words = 0;
  bool owns = false;          // device buffers owned by this object (else the handle's staging)
};

// group batches at least this large build ring entries with the agent-parallel pull kernel
static const uint64_t SDB_PULL_THRESHOLD = 16384;

// slots of the receive totals: rx_totals on the device and its pinned host mirror totals_host
enum : uint32_t {
  TOT_RECORDS = 0,            // records delivered
  TOT_GRANULES = 1,           // payload granules delivered
  TOT_FLOOR = 2,              // arena reclaim: granules from the oldest pending record to the tail
  TOT_IMPORT_GRANULES = 4,    // import: arena granules of the batch
  TOT_IMPORT_OWNED = 5,       // import: recipients this shard owns
  TOT_CX_SENDS = 6,           // compact receive: rows (host mirror of cx.totals[0])
  TOT_CX_GRANULES = 7,        // compact receive: payload granules (host mirror of cx.totals[1])
  TOT_SLOTS = 8
};

struct sdb_ctx {
  sdb_config cfg{};
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  sdb_dev_view view{};
  // device buffers
  uint8_t* arena = nullptr;
  sdb_ring_hdr* ring_hdr = nullptr;
  uint2* ring = nullptr;
  uint32_t* members = nullptr;
  sdb_dev_counters* ctr = nullptr;
  // staging for non-staged sends
  sdb_send_desc* descs_host = nullptr;   // pinned [desc_cap]
  uint64_t desc_cap = 0;                 // max_batch_sends + room for the chunks of long broadcast lists
  sdb_staged scratch;                    // device descs/payload/list owned by the handle
  uint32_t* list_host = nullptr;         // pinned
  uint32_t* gs_host = nullptr;           // pinned [max_groups + 1 + max_batch_sends]
  // inverse group table (agent -> memberships), rebuilt lazily from `ghost`
  uint32_t* memb_off_dev = nullptr; uint32_t* memb_grp_dev = nullptr; uint32_t* memb_pos_dev = nullptr;
  bool memb_dirty = true;
  uint8_t* gexcl_dev = nullptr;          // [max_groups] 1: every member of the group belongs to that group only
  uint32_t n_excl_groups = 0, n_shared_agents = 0;
  std::vector<uint32_t> rank_cnt;              // per-agent scratch table, all zero between calls: point-to-point ranking, the
                                               // disjointness check of broadcast lists, the repeated-agent check of receives
  bool shared_cfg = false;                     // SDB_SHARED_PAYLOAD: group sends above the pull threshold share one payload per send
  uint32_t max_lcount = 0;                     // largest local member count of a group (shared payloads need <= 65535)
  std::vector<uint32_t> lp_first;              // broadcast batches: first chunk descriptor of every send
  std::vector<uint64_t> lp_begin, lp_end;      // broadcast batches: where each send's / list's recipients sit in the pool
  uint32_t* lp_host = nullptr; uint32_t* lp_dev = nullptr; uint64_t lp_cap = 0;   // list-parallel index tables (pinned / device)
  uint2* ovf_log = nullptr; unsigned long long* ovf_seq = nullptr;                  // overflow log + resolved sequence numbers
  // sharding (one handle = one shard): owner of each agent, full group lists, local positions
  std::vector<uint8_t> shard_of; bool sharded = false;
  std::vector<std::vector<uint32_t>> gfull;    // full member lists as given by the caller
  std::vector<std::vector<uint32_t>> gpos;     // position in the full list of each kept member
  std::vector<uint32_t> gcount_full;
  uint32_t* member_pos_dev = nullptr;          // [member_pool] parallel to `members`
  uint32_t* lstart_dev = nullptr; uint32_t* lcount_dev = nullptr; bool ltab_dirty = true;
  // import scratch (capacity xs_cap = num_shards * max_batch_sends sends)
  uint32_t xs_cap = 0;
  uint32_t* xs_w = nullptr; uint32_t* xs_w_local = nullptr; uint32_t* xs_w_tops = nullptr;
  uint32_t* xs_gs_cnt = nullptr; uint32_t* xs_gs_local = nullptr; uint32_t* xs_gs_tops = nullptr; uint32_t* xs_gs_cur = nullptr;
  uint32_t* xs_gs_off = nullptr; uint32_t* xs_gs_idx = nullptr; sdb_send_desc* xs_descs = nullptr;
  uint32_t* xs_lw = nullptr; uint32_t* xs_lw_local = nullptr; uint32_t* xs_lw_tops = nullptr;
  sdb_src_tab* xs_tab = nullptr;
  uint8_t* xs_meta = nullptr; uint64_t xs_meta_stride = 0;   // local copies of remote headers + descriptors
  uint8_t* shard_of_dev = nullptr;
  uint32_t* owned_dev = nullptr; uint32_t n_owned = 0;     // agents this shard owns, ascending (SDB_RECV_OWNED)
  // asynchronous import: device-resident twin of {arena_tail, arena_floor, next_seq} + one import's placement
  sdb_cursor* cursor_dev = nullptr; sdb_batch_base* bb_dev = nullptr;
  sdb_cursor* cursor_host = nullptr;          // pinned
  bool host_stale = false;                     // the device cursor moved (async import): host counters must be refreshed first
  bool dev_stale = true;                       // the host counters moved: push them before the next async import
  uint32_t* xs_gs_off_src = nullptr; uint32_t* xs_gs_idx_src = nullptr; uint32_t* xs_first = nullptr;
  unsigned long long* xs_lb = nullptr; sdb_wire_header* xs_hdrs = nullptr;
  // localized-import buffer sets: set 0 aliases the buffers above; set 1 exists once sdb_import_prefetch was used (an
  // import of step k+1 is localized on `pf_stream` while step k's kernels still read the set of the other parity)
  struct XsSet {
    sdb_send_desc* descs = nullptr; uint32_t* gs_off_src = nullptr; uint32_t* gs_idx_src = nullptr; uint32_t* first = nullptr;
    unsigned long long* lb = nullptr; sdb_wire_header* hdrs = nullptr; uint32_t* tmp_list = nullptr;
    sdb_import_totals* totals = nullptr; cudaEvent_t ready = nullptr; uint32_t step = 0; bool pending = false;
    bool shared = false;            // layout the set's descriptors were localized for
  } xset[2];
  cudaStream_t pf_stream = nullptr; cudaEvent_t ev_pf_fork = nullptr;
  uint8_t* wire_host = nullptr;                // pinned: header + descriptors of an export
  sdb_wire_header* hdrs_host = nullptr;        // pinned [num_shards]
  cudaEvent_t staging_free = nullptr;    // previous H2D of pinned staging has completed
  // receive scratch + outputs
  uint32_t* rx_agent = nullptr; uint32_t* rx_cnt = nullptr; uint32_t* rx_rec_local = nullptr; uint32_t* rx_rec_tops = nullptr;
  uint4* rx_plan = nullptr; uint32_t* rx_rec_off = nullptr; unsigned long long* rx_lb = nullptr;
  uint32_t* rx_plan_tops = nullptr; unsigned long long* rx_totals = nullptr;
  uint32_t* rx_big_list = nullptr; uint32_t* rx_big_count = nullptr;
  uint32_t* rx_count = nullptr; sdb_msg_header* rx_hdr = nullptr; uint8_t* rx_payload = nullptr;
  unsigned long long* totals_host = nullptr;   // pinned [TOT_SLOTS]
  uint8_t* rx_small = nullptr;                 // device output block of the latency path
  uint8_t* small_host = nullptr;               // pinned mirror
  uint64_t small_bytes = 0;
  uint64_t pay_cap_gran = 0;
  // low-latency dequeue server (sdb_latency_server): mailbox + answer block in mapped pinned host memory
  sdb_ls_mailbox* ls_mbox = nullptr; uint8_t* ls_out = nullptr; uint32_t ls_out_cap = 0; uint4* ls_plan = nullptr;
  cudaStream_t ls_stream = nullptr; bool ls_wanted = false, ls_running = false; uint32_t ls_seq = 0;
  bool stream_busy = false;                    // work was enqueued on `stream` since the last synchronisation
  sdb_recv_args last_rx{}; bool last_rx_valid = false;   // the last bulk receive (sdb_digest_fold reads its device results)
  bool last_rx_compact = false;                          // the last receive was compact: no full-format device results
  sdb_compact_args cx{};                                 // compact receive scratch + outputs, allocated on first use
  uint32_t* where_bits = nullptr;                        // filtered receive: verdict bitmap [max_agents][ceil(R / 32)] ...
  uint8_t* where_kw = nullptr;                           // ... and the keyword [SDB_FILTER_MAX_KEYWORD], allocated on first use
  sdb_id_slot* id_tab = nullptr;                         // SDB_FILTER_IDS: id table [id_slots], the ids [id_cap] and the
  unsigned long long* id_in = nullptr;                   // per-id outputs [2 x id_cap], allocated on the first call with
  uint32_t* id_out = nullptr;                            // the clause and grown on demand
  uint64_t id_cap = 0, id_slots = 0;
  sdb_ss_slot* ss_tab = nullptr;                         // sdb_supersede: key table [ss_slots] and candidates [ss_cap],
  sdb_ss_cand* ss_cand = nullptr;                        // allocated on the first call with a flagged record and grown on
  uint64_t ss_slots = 0, ss_cap = 0;                     // demand
  unsigned long long* digest = nullptr;                  // [max_agents] stream digests, allocated on first use
  uint32_t* rs_agent = nullptr;                          // restore: per-agent tables [6][max_agents] + scan tops, allocated
  unsigned long long* rs_tot = nullptr;                  // on first use; totals [8]
  uint32_t* rs_sort = nullptr;                           // restore: radix-sort keys / values [4][max_recv_records] + digit tables
  uint32_t* rl_bits = nullptr;                           // relocation: granule bitmap [G / 32 + 2], its word popcounts and
  uint32_t* rl_cnt = nullptr; uint32_t* rl_pre = nullptr; uint32_t* rl_tops = nullptr;   // their scan (same size) ...
  uint32_t* rl_sel = nullptr;                            // ... selected agents [max_agents / 32 + 1], totals [8]; allocated on
  unsigned long long* rl_tot = nullptr;                  // the first sdb_arena_relocate
  // lease store (sdb_lease_reserve): two buffers (a sweep compacts one into the other), scratch, host bookkeeping
  struct LeaseStore {
    sdb_lease_buf buf[2]{}; int cur = 0;
    sdb_lease_scratch s{};
    unsigned long long* th = nullptr;                    // pinned mirror of s.tot
    std::vector<void*> mem;                              // every device allocation of the store
    uint64_t cap = 0, pay_cap = 0;                       // entries (and rows), payload bytes
    uint64_t used = 0, rows = 0, pay = 0;                // in buf[cur]
    uint64_t next_id = 0;                                // lease ids, monotonic per handle
    uint64_t live = 0, acked = 0, redelivered_total = 0, acked_total = 0;
    // redelivery policy (sdb_lease_set_policy): delivery counts, the ledger and the dead-letter scratch, or nothing
    std::vector<void*> pmem;                             // every device allocation of the policy
    uint32_t max_deliveries = 0;                         // 0: no policy
    bool policy = false;
    sdb_ledger led{}; uint64_t led_cap = 0;
    uint64_t led_n = 0, led_live = 0;                    // dense entries (taken ones included until a collection), held
    unsigned long long* lth = nullptr;                   // pinned mirror of led.tot
    sdb_dl_scratch dl{};
    uint64_t dead = 0, dead_total = 0, held_total = 0;
  } lease;
  // backends
  uint32_t* be_weight = nullptr; unsigned long long* be_load = nullptr; uint32_t n_backends = 0;
  uint32_t* be_req_cost = nullptr; uint32_t* be_out = nullptr; unsigned long long* be_scratch = nullptr;
  uint32_t* be_logtab = nullptr; uint32_t be_req_cap = 0;
  uint32_t* agent_backend_dev = nullptr;      // [max_agents] sticky agent -> backend map on the device (0xFFFFFFFF = none)
  // host state
  uint64_t next_seq = 1;       // ids start at 1 like the deterministic-uuid reference counter
  uint64_t arena_tail = 0;     // granules, monotonic
  uint64_t arena_floor = 0;    // granules
  uint64_t arena_grans = 0;
  uint32_t n_agents = 0;       // watermark
  std::vector<uint64_t> gstart; std::vector<uint32_t> gcount; std::vector<uint8_t> gdefined;
  uint64_t member_used = 0;
  std::vector<std::vector<uint32_t>> ghost;   // authoritative member lists (for pool compaction)
  uint64_t launches = 0;
  uint64_t picks = 0;
  uint64_t seen_overflow = 0;
  // deduplication table (sdb_dedup_reserve): two buffers (a rebuild copies the live entries into the other), per-batch
  // scratch for max_batch_sends sends, pinned mirrors, host bookkeeping
  struct Dedup {
    sdb_dedup_entry* tab[2] = {nullptr, nullptr}; int cur = 0;
    sdb_dedup_args a{};
    sdb_dedup_send* snd_dev = nullptr;
    uint32_t* lists_dev = nullptr; uint64_t lists_cap = 0;
    std::vector<void*> mem;                              // every device allocation but lists_dev
    sdb_dedup_key* key_host = nullptr; sdb_dedup_send* snd_host = nullptr;      // pinned [max_batch_sends]
    unsigned long long* verdict_host = nullptr; unsigned long long* seq_host = nullptr;
    unsigned long long* ctr_host = nullptr;              // pinned [SDB_DD_CTRS]
    std::vector<uint8_t> keep;
    uint64_t entries = 0, used = 0;
    double last_now = -INFINITY;
    uint64_t accepted = 0, dups = 0, expired = 0, forgotten = 0, rebuilds = 0;
  } dd;
  sdb_profiler prof{};
  std::string err;
};

namespace {

int fail(sdb_ctx* h, int code, const std::string& msg) {
  if (h) h->err = msg;
  return code;
}
#define CUDA_TRY(h, expr)                                                                       \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess)                                                                      \
      return fail(h, SDB_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));            \
  } while (0)

// Host -> device upload ordered on the handle's stream, like every kernel that reads the data, and complete when it
// returns.  A plain cudaMemcpy runs on the legacy default stream, which the handle's non-blocking stream is not ordered
// after, and from pageable memory it may return before the data has reached device memory.
cudaError_t upload(sdb_ctx* h, void* dst, const void* src, size_t bytes) {
  const cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, h->stream);
  return e == cudaSuccess ? cudaStreamSynchronize(h->stream) : e;
}
bool is_pow2(uint64_t x) { return x && !(x & (x - 1)); }
// header + descriptors + group buckets of a wire batch (the part a remote importer copies locally)
uint64_t wire_meta_bytes(uint32_t max_sends, uint32_t max_groups) {
  const uint64_t b = sizeof(sdb_wire_header) + static_cast<uint64_t>(max_sends) * (sizeof(sdb_send_desc) + 4) + (static_cast<uint64_t>(max_groups) + 1) * 4 + 64;
  return (b + 127) & ~127ull;                         // wire batches are laid out back to back: keep them 128-byte aligned
}
uint32_t ilog2(uint64_t x) { uint32_t r = 0; while ((1ull << r) < x) ++r; return r; }
inline uint32_t pad32(uint32_t len) { return (len + 31u) & ~31u; }

template <typename T>
cudaError_t dmalloc(T** p, size_t n) { return cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)); }

// ---- low-latency dequeue server ----------------------------------------------------------------------------------
int ls_stop(sdb_ctx* h) {
  if (!h->ls_running) return SDB_OK;
  __atomic_store_n(&h->ls_mbox->flags, 0x80000000u, __ATOMIC_RELEASE);     // quit bit, fetched with the request words
  CUDA_TRY(h, cudaStreamSynchronize(h->ls_stream));
  h->ls_running = false;
  return SDB_OK;
}
// one device buffer of a set allocated on first use: where its pointer goes and how many elements it holds
struct dbuf {
  void** p; size_t bytes;
  template <typename T> dbuf(T** q, size_t n) : p(reinterpret_cast<void**>(q)), bytes(n * sizeof(T)) {}
};
// Allocates a set of device buffers on first use, in order.  The latency server is stopped first (an allocation may wait
// for the kernels running on the device), and a set that cannot be allocated whole is freed again: SDB_ENOMEM, `what`.
int dmalloc_set(sdb_ctx* h, std::initializer_list<dbuf> set, const char* what) {
  { const int rc = ls_stop(h); if (rc != SDB_OK) return rc; }
  bool ok = true;
  for (const dbuf& b : set) ok = ok && cudaMalloc(b.p, b.bytes) == cudaSuccess;
  if (ok) return SDB_OK;
  for (const dbuf& b : set) { if (*b.p) cudaFree(*b.p); *b.p = nullptr; }
  cudaGetLastError();
  return fail(h, SDB_ENOMEM, what);
}
// Under lazy module loading (the CUDA 12 default) the first launch of a kernel loads its code into the context, and that
// load waits for the kernels running there: with the persistent latency server running it would wait forever.  So every
// kernel of the library is loaded before the server starts.  The driver functions come through the runtime's entry
// point query; cuModuleEnumerateFunctions and cuFuncLoad need a CUDA 12.4 driver.
cudaError_t load_all_kernels() {
  using get_module_t = CUresult (*)(CUmodule*, CUfunction);
  using count_t = CUresult (*)(unsigned int*, CUmodule);
  using enumerate_t = CUresult (*)(CUfunction*, unsigned int, CUmodule);
  using load_t = CUresult (*)(CUfunction);
  void *gm = nullptr, *cn = nullptr, *en = nullptr, *ld = nullptr;
  cudaDriverEntryPointQueryResult q;
  for (auto [name, fp] : {std::pair<const char*, void**>{"cuFuncGetModule", &gm}, {"cuModuleGetFunctionCount", &cn},
                          {"cuModuleEnumerateFunctions", &en}, {"cuFuncLoad", &ld}}) {
    const cudaError_t e = cudaGetDriverEntryPoint(name, fp, cudaEnableDefault, &q);
    if (e != cudaSuccess) return e;
    if (q != cudaDriverEntryPointSuccess || !*fp) return cudaErrorNotSupported;
  }
  for (const void* anchor : {sdb_send_kernel_anchor(), sdb_recv_kernel_anchor(), sdb_balance_kernel_anchor(), sdb_xshard_kernel_anchor(),
                              sdb_restore_kernel_anchor(), sdb_lease_kernel_anchor(), sdb_relocate_kernel_anchor()}) {
    cudaFunction_t f = nullptr;
    cudaError_t e = cudaGetFuncBySymbol(&f, anchor);
    if (e != cudaSuccess) return e;
    CUmodule mod = nullptr;
    unsigned int n = 0;
    if (reinterpret_cast<get_module_t>(gm)(&mod, reinterpret_cast<CUfunction>(f)) != CUDA_SUCCESS ||
        reinterpret_cast<count_t>(cn)(&n, mod) != CUDA_SUCCESS) return cudaErrorUnknown;
    std::vector<CUfunction> fs(n);
    if (n && reinterpret_cast<enumerate_t>(en)(fs.data(), n, mod) != CUDA_SUCCESS) return cudaErrorUnknown;
    for (CUfunction fn : fs) if (reinterpret_cast<load_t>(ld)(fn) != CUDA_SUCCESS) return cudaErrorUnknown;
  }
  return cudaSuccess;
}

int ls_start(sdb_ctx* h) {
  if (h->ls_running) return SDB_OK;
  CUDA_TRY(h, load_all_kernels());
  if (!h->ls_mbox) {
    h->ls_out_cap = 64u + 1024u * 64u;                                       // k_recv_small's block: 64-byte head + records
    const uint64_t need = 64ull + 1024ull * (32ull + pad32(h->cfg.max_payload_bytes));
    if (need < (4ull << 20)) h->ls_out_cap = static_cast<uint32_t>(need); else h->ls_out_cap = 4u << 20;
    CUDA_TRY(h, cudaHostAlloc(reinterpret_cast<void**>(&h->ls_mbox), sizeof(sdb_ls_mailbox), cudaHostAllocMapped));
    CUDA_TRY(h, cudaHostAlloc(reinterpret_cast<void**>(&h->ls_out), h->ls_out_cap, cudaHostAllocMapped));
    CUDA_TRY(h, dmalloc(&h->ls_plan, 1024 + 4));
    CUDA_TRY(h, cudaStreamCreateWithFlags(&h->ls_stream, cudaStreamNonBlocking));
    std::memset(h->ls_mbox, 0, sizeof(sdb_ls_mailbox));
  }
  h->ls_mbox->quit = 0; h->ls_mbox->flags = 0; h->ls_mbox->req_seq = h->ls_seq; h->ls_mbox->done_seq = h->ls_seq;
  __sync_synchronize();
  sdb_ls_mailbox* mb_dev = nullptr; uint8_t* out_dev = nullptr;
  CUDA_TRY(h, cudaHostGetDevicePointer(reinterpret_cast<void**>(&mb_dev), h->ls_mbox, 0));
  CUDA_TRY(h, cudaHostGetDevicePointer(reinterpret_cast<void**>(&out_dev), h->ls_out, 0));
  CUDA_TRY(h, sdb_launch_latency_server(&h->view, mb_dev, out_dev, h->ls_out_cap, h->ls_plan, h->ls_stream));
  h->launches += 1;
  h->ls_running = true;
  return SDB_OK;
}

// The asynchronous import advances arena / sequence counters on the device.  Before host code uses its own copies
// it pulls the device's (one small D2H + sync), and reports an import the device had to refuse.
int cursor_to_host(sdb_ctx* h) {
  if (!h->host_stale) return SDB_OK;
  CUDA_TRY(h, cudaMemcpyAsync(h->cursor_host, h->cursor_dev, sizeof(sdb_cursor), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->host_stale = false;
  h->arena_tail = h->cursor_host->arena_tail; h->next_seq = h->cursor_host->next_seq;
  if (h->cursor_host->arena_floor > h->arena_floor) h->arena_floor = h->cursor_host->arena_floor;
  if (h->cursor_host->error) {
    const unsigned long long err = h->cursor_host->error;
    CUDA_TRY(h, cudaMemsetAsync(&h->cursor_dev->error, 0, sizeof(unsigned long long), h->stream));
    if (err & 1ull) return fail(h, SDB_EARENA_FULL, "an asynchronous import did not fit the message arena and was dropped whole "
                                                    "(unconsumed messages pin the log: receive or enlarge arena_bytes)");
    if (err & 2ull) return fail(h, SDB_ECAPACITY, "an asynchronous import's owned recipients exceeded list_pool_entries; it was dropped whole");
    return fail(h, SDB_ECAPACITY, "an asynchronous import carried payloads above 512 bytes (use the synchronous import)");
  }
  return SDB_OK;
}
int cursor_to_dev(sdb_ctx* h) {
  if (!h->dev_stale) return SDB_OK;
  h->cursor_host->arena_tail = h->arena_tail; h->cursor_host->arena_floor = h->arena_floor; h->cursor_host->next_seq = h->next_seq;
  CUDA_TRY(h, cudaMemcpyAsync(h->cursor_dev, h->cursor_host, 3 * sizeof(unsigned long long), cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaEventRecord(h->staging_free, h->stream));
  h->dev_stale = false;
  return SDB_OK;
}

// Make room for `need` granules in the arena; may run the floor-reclaim kernel (synchronises).
int arena_reserve(sdb_ctx* h, uint64_t need, uint64_t* base_out) {
  const uint64_t G = h->arena_grans;
  if (need > G) return fail(h, SDB_EARENA_FULL, "batch larger than the whole arena");
  uint64_t tail = h->arena_tail;
  if ((tail & (G - 1)) + need > G) tail = (tail + G - 1) & ~(G - 1);     // a batch never straddles the wrap
  if (tail + need - h->arena_floor > G) {
    // reclaim: recompute the floor from the oldest pending record of every ring
    cudaError_t e = sdb_launch_arena_floor(&h->view, h->n_agents, static_cast<uint32_t>(h->arena_tail),
                                           h->rx_totals + TOT_FLOOR, h->stream);
    h->launches += 1;
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->totals_host + TOT_FLOOR, h->rx_totals + TOT_FLOOR, sizeof(unsigned long long),
                                             cudaMemcpyDeviceToHost, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("arena floor: ") + cudaGetErrorString(e));
    h->arena_floor = h->arena_tail - h->totals_host[TOT_FLOOR];
    if (tail + need - h->arena_floor > G)
      return fail(h, SDB_EARENA_FULL, "message arena full: unconsumed messages pin the log (receive or enlarge arena_bytes)");
  }
  *base_out = tail;
  return SDB_OK;
}

struct SendArrays {
  const uint32_t* sender; const uint32_t* second; const uint8_t* prio; const uint8_t* type; const uint16_t* len;
  const uint64_t* payload_off; const double* timestamp;
  const uint8_t* kind = nullptr;      // mixed batches only
  uint32_t n_lists = 0;               // mixed batches only
  uint32_t* p2p_list = nullptr;       // mixed batches: where single receivers are appended (pinned list staging)
  uint64_t p2p_list_base = 0, p2p_list_cap = 0, p2p_list_used = 0;
  // list batches: recipients of list li are list_pool[lbegin[li] .. lend[li]) (identical lists of a batch are stored once)
  const uint64_t* lbegin = nullptr; const uint64_t* lend = nullptr;
  const uint32_t* list_pool = nullptr;
  uint32_t* lp_out = nullptr; uint64_t lp_cap = 0;     // staging of the list-parallel index tables (nullptr: not offered)
  const uint8_t* keep = nullptr;      // mixed batches: keep[i] == 0 leaves send i out, its sequence numbers unused
};

// Build descriptors into `out` (host).  kind 0: second = receiver; 1: second = group idx;
// 2: list (list_off/list base offsets supplied).  Returns totals through the staged object.
// A broadcast list longer than SDB_LIST_CHUNK recipients is emitted as several descriptors (same payload, same
// sequence number, consecutive arena regions) so that one warp never owns a million-record fan-out; `out` therefore
// holds s->n >= n descriptors, bounded by `out_cap`.
static const uint32_t SDB_LIST_CHUNK = 1024;
int rebuild_inverse(sdb_ctx* h);

int build_descs(sdb_ctx* h, uint32_t batch_kind, uint32_t n, SendArrays& a, const uint64_t* list_off,
                uint64_t payload_bytes, sdb_send_desc* out, uint64_t out_cap, sdb_staged* s, uint32_t* gs_out = nullptr,
                uint32_t* n_gs_out = nullptr) {
  uint64_t rec = 0, gran = 0, group_recs = 0, list_copies = 0;
  uint32_t n_list_sends = 0;
  std::vector<uint32_t>& first_desc = h->lp_first;    // list sends: index of the send's first chunk descriptor
  uint64_t o = 0;                      // output cursor (descriptors emitted)
  uint32_t max_padlen = 0;
  uint32_t n_group_sends = 0, n_other = 0;
  uint32_t n_kept = n;                 // sends written (all but the duplicates a.keep leaves out)
  const uint32_t A = h->cfg.max_agents;
  if (h->sharded) return fail(h, SDB_EINVAL, "sharded handle: sends go through sdb_export_*_batch + sdb_import_wire_*");
  // shared payloads (pure group batches above the pull threshold, exclusive groups, payloads <= 512 bytes, groups of at
  // most 65535 members): a send's region is mcount headers + ONE payload; decided before any arena offset is handed out
  bool shared = false;
  if (h->shared_cfg && batch_kind == 1 && gs_out && h->cfg.fanout_variant >= 2) {
    if (h->memb_dirty) { int rc0 = rebuild_inverse(h); if (rc0 != SDB_OK) return rc0; }
    uint64_t recs = 0; bool ok = h->n_shared_agents == 0 && h->n_excl_groups != 0;
    for (uint32_t i = 0; i < n && ok; ++i) {
      const uint32_t g = a.second[i];
      if (g >= h->cfg.max_groups || !h->gdefined[g] || h->gcount[g] > 65535u || a.len[i] > 512u) ok = false;
      else recs += h->gcount[g];
    }
    shared = ok && recs >= SDB_PULL_THRESHOLD;
  }
  for (uint32_t i = 0; i < n; ++i) {
    sdb_send_desc d;
    std::memset(&d, 0, sizeof(d));
    const uint32_t len = a.len[i];
    if (len > h->cfg.max_payload_bytes) return fail(h, SDB_EINVAL, "payload longer than max_payload_bytes");
    const uint64_t off = a.payload_off ? a.payload_off[i] : 0;
    if (off & 15u) return fail(h, SDB_EINVAL, "payload_off must be 16-byte aligned");
    if (off + len > payload_bytes) return fail(h, SDB_EINVAL, "payload_off + len beyond payload_bytes");
    if (a.sender[i] >= A) return fail(h, SDB_EINVAL, "sender index out of range");
    if ((a.prio ? a.prio[i] : 1) > 3) return fail(h, SDB_EINVAL, "priority out of range");
    const uint32_t pl = pad32(len);
    max_padlen = std::max(max_padlen, pl);
    d.payload_off = off;
    d.timestamp = a.timestamp ? a.timestamp[i] : 0.0;
    d.sender = a.sender[i];
    d.len = static_cast<uint16_t>(len);
    d.prio = a.prio ? a.prio[i] : 1;
    d.type = a.type ? a.type[i] : 0;
    d.rgran = 1u + pl / SDB_GRANULE;
    d.group = SDB_NO_GROUP;
    if (rec > 0xFFFFFFFFull || gran > 0xFFFFFFFFull) return fail(h, SDB_ECAPACITY, "batch exceeds 2^32 records/granules");
    d.rec0 = static_cast<uint32_t>(rec);
    d.gran0 = static_cast<uint32_t>(gran);
    uint32_t kind = batch_kind;
    if (batch_kind == 3) {
      kind = a.kind[i];
      if (kind > 2) return fail(h, SDB_EINVAL, "kind must be 0, 1 or 2");
      if (a.keep && !a.keep[i]) {     // a duplicate: it takes its sequence numbers and writes nothing
        if (kind == 1) {
          const uint32_t g = a.second[i];
          if (g >= h->cfg.max_groups || !h->gdefined[g]) return fail(h, SDB_ENOTFOUND, "unknown group index");
          rec += h->gcount[g];
        } else {
          rec += 1;
        }
        --n_kept;
        continue;
      }
      if (kind == 0) {      // p2p inside a mixed batch: a one-entry temporary list through the fan-out kernel
        if (a.second[i] >= A) return fail(h, SDB_EINVAL, "receiver index out of range");
        if (a.p2p_list_used >= a.p2p_list_cap) return fail(h, SDB_ECAPACITY, "recipient lists exceed list_pool_entries");
        a.p2p_list[a.p2p_list_used] = a.second[i];
        h->n_agents = std::max(h->n_agents, a.second[i] + 1);
        d.mstart = static_cast<uint32_t>(a.p2p_list_base + a.p2p_list_used); d.mcount = 1; d.flags = SDB_DESC_LIST_TEMP;
        a.p2p_list_used++;
        rec += 1; gran += d.rgran;
        ++n_other;
        if (o >= out_cap) return fail(h, SDB_ECAPACITY, "descriptor staging exhausted");
        out[o++] = d;
        continue;
      }
      if (kind == 2 && a.second[i] >= a.n_lists) return fail(h, SDB_EINVAL, "list number out of range");
    }
    if (kind == 0) {
      if (a.second[i] >= A) return fail(h, SDB_EINVAL, "receiver index out of range");
      h->n_agents = std::max(h->n_agents, a.second[i] + 1);     // auto-registration of the receiver (M:423-427)
      d.mstart = a.second[i]; d.mcount = 1; d.flags = 0;
      rec += 1; gran += d.rgran;
    } else if (kind == 1) {
      const uint32_t g = a.second[i];
      if (g >= h->cfg.max_groups || !h->gdefined[g]) return fail(h, SDB_ENOTFOUND, "unknown group index");
      if (h->sharded) return fail(h, SDB_EINVAL, "sharded handle: use sdb_export_group_batch + sdb_import_wire_batches");
      d.mstart = static_cast<uint32_t>(h->gstart[g]); d.mcount = h->gcount[g]; d.group = g;
      d.flags = SDB_DESC_SKIP_SENDER;
      rec += d.mcount;
      gran += shared ? (d.mcount ? static_cast<uint64_t>(d.mcount) + d.rgran - 1u : 0ull) : static_cast<uint64_t>(d.mcount) * d.rgran;
      group_recs += d.mcount; ++n_group_sends;
    } else {
      const uint32_t li = batch_kind == 3 ? a.second[i] : i;
      const uint64_t b = a.lbegin ? a.lbegin[li] : list_off[li], e = a.lend ? a.lend[li] : list_off[li + 1];
      list_copies += e - b; ++n_list_sends;
      if (first_desc.size() < n) first_desc.resize(n);
      first_desc[i] = static_cast<uint32_t>(o);
      if (e < b || e - b > 0xFFFFFFFFull) return fail(h, SDB_EINVAL, "bad list_off");
      d.flags = SDB_DESC_SHARED_SEQ | SDB_DESC_LIST_TEMP;
      const uint64_t cnt = e - b;
      rec += 1; ++n_other;
      for (uint64_t c0 = 0; c0 == 0 || c0 < cnt; c0 += SDB_LIST_CHUNK) {      // at least one descriptor, even for an empty list
        if (gran > 0xFFFFFFFFull) return fail(h, SDB_ECAPACITY, "batch exceeds 2^32 granules");
        d.mstart = static_cast<uint32_t>(b + c0);
        d.mcount = static_cast<uint32_t>(std::min<uint64_t>(SDB_LIST_CHUNK, cnt - c0));
        d.gran0 = static_cast<uint32_t>(gran);
        gran += static_cast<uint64_t>(d.mcount) * d.rgran;
        if (o >= out_cap) return fail(h, SDB_ECAPACITY, "descriptor staging exhausted");
        out[o++] = d;
      }
      continue;
    }
    if (kind != 1) ++n_other;
    if (o >= out_cap) return fail(h, SDB_ECAPACITY, "descriptor staging exhausted");
    out[o++] = d;
  }
  const uint32_t n_out = static_cast<uint32_t>(o);
  s->kind = batch_kind; s->n = n_out; s->total_recs = rec; s->total_grans = gran; s->max_padlen = max_padlen;
  s->has_pull = false; s->has_atomic = true; s->ranked = false; s->list_pull = false; s->shared = shared;
  if (n_list_sends == n_kept && n_kept && list_copies >= SDB_PULL_THRESHOLD && a.lp_out && a.lbegin && a.list_pool) {
    // pure broadcast batch: if the lists it names are pairwise disjoint (and free of repeats), every member of a list
    // receives exactly the sends naming it, in send order -> owner-computes index build (k_list_index), no atomics.
    // Lists are identified by where they start in the pool (identical lists were stored once by the caller).
    std::vector<std::pair<uint64_t, uint32_t>> key;                       // (list begin, send)
    key.reserve(n_kept);
    for (uint32_t i = 0; i < n; ++i) {
      if (a.keep && !a.keep[i]) continue;
      const uint32_t li = batch_kind == 3 ? a.second[i] : i; key.push_back({a.lbegin[li], i});
    }
    const uint32_t n = n_kept;
    std::stable_sort(key.begin(), key.end(), [](const auto& x, const auto& y) { return x.first < y.first; });
    uint32_t nd = 0;
    for (uint32_t k = 0; k < n; ++k) if (k == 0 || key[k].first != key[k - 1].first) ++nd;
    const uint64_t words = 3ull * nd + 1 + n;
    bool ok = nd <= 65535u && words <= a.lp_cap;
    if (ok) {
      uint32_t* start = a.lp_out; uint32_t* count = start + nd; uint32_t* off = count + nd; uint32_t* idx = off + nd + 1;
      if (h->rank_cnt.size() != A) h->rank_cnt.assign(A, 0u);
      std::vector<uint32_t>& seen = h->rank_cnt;                            // all zero between batches
      uint32_t dcur = 0, max_count = 0;
      std::vector<std::pair<uint64_t, uint64_t>> marked;
      for (uint32_t k = 0; k < n && ok; ++k) {
        const uint32_t i = key[k].second, li = batch_kind == 3 ? a.second[i] : i;
        if (k == 0 || key[k].first != key[k - 1].first) {
          const uint64_t b = a.lbegin[li], e = a.lend[li];
          if (k) ++dcur;
          start[dcur] = static_cast<uint32_t>(b); count[dcur] = static_cast<uint32_t>(e - b); off[dcur] = k;
          max_count = std::max(max_count, count[dcur]);
          marked.push_back({b, e});
          for (uint64_t x = b; x < e; ++x) { uint32_t& c = seen[a.list_pool[x]]; if (c) { ok = false; marked.back().second = x; break; } c = 1; }
        } else if (a.lend[li] - a.lbegin[li] != count[dcur]) ok = false;     // same start, different length: not the same list
        idx[k] = first_desc[i];
      }
      off[nd] = n;
      for (const auto& m : marked) for (uint64_t x = m.first; x < m.second; ++x) seen[a.list_pool[x]] = 0;
      if (ok) {
        for (uint32_t i = 0; i < n_out; ++i) out[i].flags |= SDB_DESC_PULL;
        s->list_pull = true; s->has_atomic = false; s->lp_nd = nd; s->lp_max_count = max_count; s->lp_words = static_cast<uint32_t>(words);
      }
    }
  }
  if (batch_kind == 0 && n_out) {
    // pure point-to-point batch: number the sends of every receiver 0, 1, 2 .. in send order, so that the enqueue
    // kernel places ring entries at ctail + rank without atomics and in final order (no commit sort)
    if (h->rank_cnt.size() != A) h->rank_cnt.assign(A, 0u);
    std::vector<uint32_t>& cnt = h->rank_cnt;
    for (uint32_t i = 0; i < n_out; ++i) { out[i].pad0 = cnt[out[i].mstart]++; out[i].flags |= SDB_DESC_RANKED; }
    for (uint32_t i = n_out; i-- > 0;) {
      uint32_t& c = cnt[out[i].mstart];
      if (c) { out[i].flags |= SDB_DESC_RANK_LAST; c = 0; }      // first seen from the back = highest rank; resets the table
    }
    s->ranked = true;
  }
  if (gs_out && group_recs >= SDB_PULL_THRESHOLD) {
    // bucket the group sends by group (counting sort, ascending send index inside a bucket)
    const uint32_t G = h->cfg.max_groups;
    uint32_t* off = gs_out;            // [G + 1]
    uint32_t* idx = gs_out + G + 1;    // [n_group_sends]
    std::memset(off, 0, (static_cast<size_t>(G) + 1) * sizeof(uint32_t));
    for (uint32_t i = 0; i < n_out; ++i) if (out[i].flags & SDB_DESC_SKIP_SENDER) off[out[i].group + 1]++;
    for (uint32_t g = 0; g < G; ++g) off[g + 1] += off[g];
    std::vector<uint32_t> cur(off, off + G);
    for (uint32_t i = 0; i < n_out; ++i) if (out[i].flags & SDB_DESC_SKIP_SENDER) { idx[cur[out[i].group]++] = i; out[i].flags |= SDB_DESC_PULL; }
    s->has_pull = true; s->has_atomic = n_other != 0;
    *n_gs_out = n_group_sends;
  }
  return SDB_OK;
}

// agent -> (group, position) lists, CSR over agents, from the authoritative host group table
int rebuild_inverse(sdb_ctx* h) {
  const uint32_t A = h->cfg.max_agents, G = h->cfg.max_groups;
  std::vector<uint32_t> off(static_cast<size_t>(A) + 1, 0);
  uint64_t total = 0;
  for (uint32_t g = 0; g < G; ++g) if (h->gdefined[g]) { for (uint32_t m : h->ghost[g]) off[m + 1]++; total += h->ghost[g].size(); }
  if (total > h->cfg.member_pool_entries) return fail(h, SDB_ECAPACITY, "memberships exceed member_pool_entries");
  for (uint32_t a = 0; a < A; ++a) off[a + 1] += off[a];
  std::vector<uint32_t> grp(total ? total : 1), pos(total ? total : 1), cur(off.begin(), off.end() - 1);
  for (uint32_t g = 0; g < G; ++g) if (h->gdefined[g]) {
    const std::vector<uint32_t>& ms = h->ghost[g];
    for (uint32_t j = 0; j < ms.size(); ++j) { const uint32_t c = cur[ms[j]]++; grp[c] = g; pos[c] = j; }
  }
  // a group is "exclusive" when each of its members belongs to that group only (and appears in it once): all members
  // then receive exactly the group's sends and the index build runs group-parallel (k_pull_index_group)
  std::vector<uint8_t> excl(G, 0);
  uint32_t n_excl = 0, n_shared = 0;
  for (uint32_t g = 0; g < G; ++g) if (h->gdefined[g]) {
    bool ex = true;
    for (uint32_t m : h->ghost[g]) if (off[m + 1] - off[m] != 1) { ex = false; break; }
    excl[g] = ex ? 1 : 0; n_excl += ex ? 1 : 0;
  }
  for (uint32_t a = 0; a < A; ++a) {
    const uint32_t nk = off[a + 1] - off[a];
    if (nk > 1 || (nk == 1 && !excl[grp[off[a]]])) ++n_shared;
  }
  h->n_excl_groups = n_excl; h->n_shared_agents = n_shared;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, upload(h, h->gexcl_dev, excl.data(), G));
  CUDA_TRY(h, upload(h, h->memb_off_dev, off.data(), off.size() * sizeof(uint32_t)));
  if (total) {
    CUDA_TRY(h, upload(h, h->memb_grp_dev, grp.data(), total * sizeof(uint32_t)));
    CUDA_TRY(h, upload(h, h->memb_pos_dev, pos.data(), total * sizeof(uint32_t)));
  }
  h->memb_dirty = false;
  return SDB_OK;
}

// device copy of the local group table (start, count per group): index build and cross-shard import read it
int ensure_ltab(sdb_ctx* h) {
  if (!h->ltab_dirty) return SDB_OK;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  std::vector<uint32_t> st(h->cfg.max_groups), ct(h->cfg.max_groups);
  h->max_lcount = 0;
  for (uint32_t g = 0; g < h->cfg.max_groups; ++g) {
    st[g] = static_cast<uint32_t>(h->gstart[g]); ct[g] = h->gdefined[g] ? h->gcount[g] : 0;
    h->max_lcount = std::max(h->max_lcount, ct[g]);
  }
  CUDA_TRY(h, upload(h, h->lstart_dev, st.data(), st.size() * sizeof(uint32_t)));
  CUDA_TRY(h, upload(h, h->lcount_dev, ct.data(), ct.size() * sizeof(uint32_t)));
  h->ltab_dirty = false;
  return SDB_OK;
}

int submit(sdb_ctx* h, const sdb_staged* s, uint64_t* seq_base_out) {
  { int rcc = cursor_to_host(h); if (rcc != SDB_OK) return rcc; }
  if (seq_base_out) *seq_base_out = h->next_seq;
  if (s->n == 0) return SDB_OK;
  if (s->has_pull && h->memb_dirty) { int rc0 = rebuild_inverse(h); if (rc0 != SDB_OK) return rc0; }
  if (s->shared && (h->n_shared_agents != 0 || h->n_excl_groups == 0))
    return fail(h, SDB_EINVAL, "batch staged before a membership change (its groups are no longer exclusive): stage it again");
  if (s->has_pull) { int rc1 = ensure_ltab(h); if (rc1 != SDB_OK) return rc1; }
  uint64_t base = 0;
  int rc = arena_reserve(h, s->total_grans, &base);
  if (rc != SDB_OK) return rc;
  cudaError_t e;
  if (s->kind == 0) {
    e = sdb_launch_p2p(&h->view, s->descs_dev, s->n, s->payload_dev, h->next_seq, base, h->sm_count, h->stream, &h->prof, s->max_padlen);
    if (e == cudaSuccess && s->ranked) {      // entries are in send order already: publish them, nothing to sort
      e = sdb_launch_commit_ranked(&h->view, s->descs_dev, s->n, h->n_agents, h->stream, &h->prof);
      h->launches += 1;
    }
  } else if (s->shared) {
    e = sdb_launch_fanout_shared(&h->view, s->descs_dev, s->n, s->payload_dev, h->next_seq, base, 0u, h->sm_count, h->stream, &h->prof, nullptr);
  } else {
    e = sdb_launch_fanout(&h->view, s->descs_dev, s->n, s->payload_dev, s->list_dev, h->next_seq, base,
                          s->max_padlen, static_cast<int>(h->cfg.fanout_variant), h->sm_count, h->stream, &h->prof, nullptr, 0u);
  }
  h->launches += 1;
  // the index build (rings) follows the payload fan-out (arena) on the same stream.  Beside it on a second stream the
  // two contend for issue slots and HBM: on an H100 (400 W) the fan-out took 12 % and the index 53 % longer, and the
  // c2 step was only 1 % shorter (1.234 against 1.246 ms)
  if (e == cudaSuccess && s->has_pull) {
    sdb_pull_view pv{h->memb_off_dev, h->memb_grp_dev, h->memb_pos_dev, s->gs_off_dev, s->gs_idx_dev, 1u, 0u, 0u, nullptr};
    int nlp = 0;
    e = sdb_launch_pull(&h->view, &pv, s->descs_dev, h->n_agents, h->cfg.max_groups, h->gexcl_dev, h->n_excl_groups,
                        h->n_shared_agents, h->lstart_dev, h->lcount_dev, base, s->has_atomic ? 0 : 1, h->stream, &h->prof, &nlp, nullptr,
                        s->shared ? 1u : 0u);
    h->launches += nlp;
  }
  if (e == cudaSuccess && s->list_pull) {
    e = sdb_launch_list_index(&h->view, s->descs_dev, s->list_dev, h->lp_dev, s->lp_nd, s->lp_max_count, base, h->stream, &h->prof);
    h->launches += 1;
  }
  if (e == cudaSuccess && s->has_atomic && !s->ranked) {
    e = sdb_launch_commit(&h->view, h->n_agents, static_cast<uint32_t>(base), h->rx_big_list, h->rx_big_count + 1, h->sm_count, h->stream, &h->prof, nullptr);
    h->launches += 2;
  }
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("enqueue launch: ") + cudaGetErrorString(e));
  h->next_seq += s->total_recs;
  h->arena_tail = base + s->total_grans;
  h->dev_stale = true;
  h->stream_busy = true;
  return SDB_OK;
}

// payload_staged: the payload is in the handle's payload staging already (deduplicated sends hash it first)
int send_common(sdb_ctx* h, uint32_t kind, uint32_t n, SendArrays& a, const uint64_t* list_off,
                const uint32_t* list_idx, const uint8_t* payload, uint64_t payload_bytes, uint64_t* seq_base_out,
                bool payload_staged = false) {
  if (!h) return SDB_EINVAL;
  if (n == 0) { int rcc = cursor_to_host(h); if (seq_base_out) *seq_base_out = h->next_seq; return rcc; }
  if (!a.sender || !a.len || (kind != 2 && !a.second) || (kind == 3 && !a.kind)) return fail(h, SDB_EINVAL, "null array");
  if (n > h->cfg.max_batch_sends) return fail(h, SDB_ECAPACITY, "n exceeds max_batch_sends");
  if (payload_bytes > h->cfg.max_batch_payload) return fail(h, SDB_ECAPACITY, "payload_bytes exceeds max_batch_payload");
  if (payload_bytes && !payload) return fail(h, SDB_EINVAL, "null payload");
  CUDA_TRY(h, cudaEventSynchronize(h->staging_free));     // pinned descriptor staging is reusable
  sdb_staged* s = &h->scratch;
  uint64_t list_total = 0;
  if (kind == 2 || kind == 3) {
    const uint32_t nl = kind == 2 ? n : a.n_lists;
    list_total = (nl && list_off) ? list_off[nl] : 0;
    const uint64_t cap = h->cfg.list_pool_entries;
    // identical consecutive lists (the same "everybody" list passed with every broadcast) are stored and uploaded once
    h->lp_begin.assign(nl, 0); h->lp_end.assign(nl, 0);
    uint64_t used = 0, prev_b = 0, prev_n = 0; bool have_prev = false;
    for (uint32_t li = 0; li < nl; ++li) {
      const uint64_t b = list_off[li], e = list_off[li + 1];
      if (e < b || e > list_total) return fail(h, SDB_EINVAL, "bad list_off");
      const uint64_t cnt = e - b;
      if (have_prev && cnt == prev_n && cnt && std::memcmp(list_idx + b, h->list_host + prev_b, cnt * sizeof(uint32_t)) == 0) {
        h->lp_begin[li] = prev_b; h->lp_end[li] = prev_b + cnt;
        continue;
      }
      for (uint64_t k = b; k < e; ++k) {
        if (list_idx[k] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "recipient index out of range");
        h->n_agents = std::max(h->n_agents, list_idx[k] + 1);
      }
      if (used + cnt > cap) return fail(h, SDB_ECAPACITY, "recipient lists exceed list_pool_entries");
      if (cnt) std::memcpy(h->list_host + used, list_idx + b, cnt * sizeof(uint32_t));
      h->lp_begin[li] = used; h->lp_end[li] = used + cnt;
      prev_b = used; prev_n = cnt; have_prev = true;
      used += cnt;
    }
    list_total = used;
    a.lbegin = h->lp_begin.data(); a.lend = h->lp_end.data(); a.list_pool = h->list_host;
    if (!h->lp_host) {
      h->lp_cap = 4ull * h->cfg.max_batch_sends + 8;
      CUDA_TRY(h, cudaHostAlloc(reinterpret_cast<void**>(&h->lp_host), h->lp_cap * sizeof(uint32_t), cudaHostAllocDefault));
      CUDA_TRY(h, dmalloc(&h->lp_dev, h->lp_cap));
    }
    a.lp_out = h->lp_host; a.lp_cap = h->lp_cap;
    a.p2p_list = h->list_host + list_total; a.p2p_list_base = list_total; a.p2p_list_cap = cap - list_total;
  }
  uint32_t n_gs = 0;
  int rc = build_descs(h, kind, n, a, list_off, payload_bytes, h->descs_host, h->desc_cap, s, h->gs_host, &n_gs);
  if (rc != SDB_OK) return rc;
  if (s->has_pull) {
    const size_t G1 = static_cast<size_t>(h->cfg.max_groups) + 1;
    CUDA_TRY(h, cudaMemcpyAsync(s->gs_off_dev, h->gs_host, G1 * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(s->gs_idx_dev, h->gs_host + G1, static_cast<size_t>(n_gs) * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  }
  if (s->list_pull)
    CUDA_TRY(h, cudaMemcpyAsync(h->lp_dev, h->lp_host, static_cast<size_t>(s->lp_words) * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  list_total += a.p2p_list_used;
  if (list_total)
    CUDA_TRY(h, cudaMemcpyAsync(s->list_dev, h->list_host, list_total * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(s->descs_dev, h->descs_host, static_cast<size_t>(s->n) * sizeof(sdb_send_desc),
                              cudaMemcpyHostToDevice, h->stream));
  if (payload_bytes && !payload_staged)   // straight from the caller's buffer (pinned memory makes this a true async DMA)
    CUDA_TRY(h, cudaMemcpyAsync(s->payload_dev, payload, payload_bytes, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaEventRecord(h->staging_free, h->stream));
  return submit(h, s, seq_base_out);
}

// n elements (at least one) of device memory for *p, recorded in `owned` (the store's or the policy's allocations)
template <typename T>
bool lease_alloc(std::vector<void*>& owned, T** p, size_t n) {
  void* q = nullptr;
  if (cudaMalloc(&q, std::max<size_t>(n, 1) * sizeof(T)) != cudaSuccess) return false;
  owned.push_back(q);
  *p = static_cast<T*>(q);
  return true;
}

}  // namespace

// =============================================================================================
extern "C" {

int sdb_abi_version(void) { return static_cast<int>(SDB_ABI_VERSION); }

const char* sdb_last_error(sdb_handle h) { return h ? h->err.c_str() : "null handle"; }

int sdb_create(const sdb_config* cfg, sdb_handle* out) {
  if (!cfg || !out) return SDB_EINVAL;
  *out = nullptr;
  if (cfg->struct_bytes != sizeof(sdb_config)) return SDB_EINVAL;
  sdb_ctx* h = new (std::nothrow) sdb_ctx();
  if (!h) return SDB_ENOMEM;
  *out = h;                       // returned even on failure so sdb_last_error works; caller destroys
  h->cfg = *cfg;
  sdb_config& c = h->cfg;
  if (c.num_shards == 0) c.num_shards = 1;
  if (!is_pow2(c.ring_slots) || c.ring_slots < 2 || c.ring_slots > (1u << 24)) return fail(h, SDB_EINVAL, "ring_slots must be a power of two in [2, 2^24]");
  if (!is_pow2(c.arena_bytes) || c.arena_bytes < (1u << 16) || c.arena_bytes > (1ull << 37)) return fail(h, SDB_EINVAL, "arena_bytes must be a power of two in [64 KiB, 128 GiB]");
  if (c.max_agents == 0 || c.max_agents > (1u << 30)) return fail(h, SDB_EINVAL, "max_agents out of range");
  if (c.max_payload_bytes == 0 || c.max_payload_bytes > 65504) return fail(h, SDB_EINVAL, "max_payload_bytes must be in [1, 65504]");
  if (c.max_groups == 0) c.max_groups = 1;
  if (c.member_pool_entries == 0) c.member_pool_entries = 1;
  if (c.max_backends == 0) c.max_backends = 256;
  if (c.max_backends > SDB_MAX_BACKENDS) return fail(h, SDB_EINVAL, "max_backends must be at most SDB_MAX_BACKENDS (4096)");
  if (c.max_batch_sends == 0) c.max_batch_sends = 65536;
  if (c.max_batch_payload == 0) c.max_batch_payload = static_cast<uint64_t>(c.max_batch_sends) * pad32(std::min(c.max_payload_bytes, 256u));
  if (c.max_recv_records == 0) c.max_recv_records = 1u << 20;
  if (c.max_recv_records >= 0x7FFFFFF0ull) return fail(h, SDB_EINVAL, "max_recv_records too large (< 2^31)");
  if (c.max_recv_payload == 0) c.max_recv_payload = c.max_recv_records * 256ull;
  if (c.list_pool_entries == 0) c.list_pool_entries = 2ull * c.max_agents + 1024;
  if (c.fanout_variant > 3) return fail(h, SDB_EINVAL, "fanout_variant must be 0, 1, 2 or 3");

  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(h, SDB_ECUDA, "no CUDA device: swarmdb_b200 has no CPU fallback");
  if (c.device < 0 || c.device >= ndev) return fail(h, SDB_EINVAL, "device ordinal out of range");
  CUDA_TRY(h, cudaSetDevice(c.device));
  // L2 fetch granularity 64 bytes (device-wide limit of this process).  The receive gather reads 288-byte records at
  // 32-byte alignment in receiver order: with the default 128-byte granularity every record costs three full lines
  // (1.37x its bytes).  On an H100 (700 W) the c2 step measured the same with 64 and 128 (1.229 ms); 64 is kept
  // because it never moves more bytes.
  cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 64);
  {
    // shared payloads for group sends above the pull threshold (sdb_common.cuh): SDB_SHARED_PAYLOAD=0 keeps one
    // payload copy per recipient in the arena log
    const char* sp = getenv("SDB_SHARED_PAYLOAD");
    h->shared_cfg = sp ? atoi(sp) != 0 : true;
  }
  CUDA_TRY(h, sdb_send_prepare_device());
  CUDA_TRY(h, sdb_recv_prepare_device());
  CUDA_TRY(h, sdb_balance_prepare_device());
  cudaDeviceProp prop;
  CUDA_TRY(h, cudaGetDeviceProperties(&prop, c.device));
  h->sm_count = prop.multiProcessorCount;
  CUDA_TRY(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  h->own_stream = true;
  CUDA_TRY(h, cudaEventCreateWithFlags(&h->staging_free, cudaEventDisableTiming));

  const size_t A = c.max_agents, R = c.ring_slots;
  h->arena_grans = c.arena_bytes / SDB_GRANULE;
  CUDA_TRY(h, dmalloc(&h->arena, c.arena_bytes));
  CUDA_TRY(h, dmalloc(&h->ring_hdr, A));
  CUDA_TRY(h, dmalloc(&h->ring, A * R));
  CUDA_TRY(h, dmalloc(&h->members, c.member_pool_entries));
  CUDA_TRY(h, dmalloc(&h->ctr, 1));
  CUDA_TRY(h, cudaMemsetAsync(h->ring_hdr, 0, A * sizeof(sdb_ring_hdr), h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->ring, 0xFF, A * R * sizeof(uint2), h->stream));          // every slot "consumed"
  CUDA_TRY(h, cudaMemsetAsync(h->ctr, 0, sizeof(sdb_dev_counters), h->stream));
  CUDA_TRY(h, dmalloc(&h->ovf_log, SDB_OVF_LOG)); CUDA_TRY(h, dmalloc(&h->ovf_seq, SDB_OVF_LOG));

  // send staging
  h->desc_cap = static_cast<uint64_t>(c.max_batch_sends) + c.list_pool_entries / SDB_LIST_CHUNK + 1;
  CUDA_TRY(h, cudaHostAlloc(reinterpret_cast<void**>(&h->descs_host), static_cast<size_t>(h->desc_cap) * sizeof(sdb_send_desc), cudaHostAllocDefault));
  CUDA_TRY(h, cudaHostAlloc(reinterpret_cast<void**>(&h->list_host), c.list_pool_entries * sizeof(uint32_t), cudaHostAllocDefault));
  CUDA_TRY(h, dmalloc(&h->scratch.descs_dev, h->desc_cap));
  CUDA_TRY(h, dmalloc(&h->scratch.payload_dev, c.max_batch_payload + 64));
  CUDA_TRY(h, dmalloc(&h->scratch.list_dev, c.list_pool_entries));
  CUDA_TRY(h, dmalloc(&h->scratch.gs_off_dev, static_cast<size_t>(c.max_groups) + 1));
  CUDA_TRY(h, dmalloc(&h->scratch.gs_idx_dev, c.max_batch_sends));
  CUDA_TRY(h, cudaHostAlloc(reinterpret_cast<void**>(&h->gs_host), (static_cast<size_t>(c.max_groups) + 1 + c.max_batch_sends) * sizeof(uint32_t), cudaHostAllocDefault));
  CUDA_TRY(h, dmalloc(&h->memb_off_dev, static_cast<size_t>(c.max_agents) + 1));
  CUDA_TRY(h, dmalloc(&h->memb_grp_dev, c.member_pool_entries));
  CUDA_TRY(h, dmalloc(&h->memb_pos_dev, c.member_pool_entries));
  CUDA_TRY(h, dmalloc(&h->gexcl_dev, c.max_groups));
  CUDA_TRY(h, cudaMemsetAsync(h->gexcl_dev, 0, c.max_groups, h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->scratch.payload_dev, 0, c.max_batch_payload + 64, h->stream));

  // receive scratch
  const size_t tiles = sdb_scan_tops_len(A);
  CUDA_TRY(h, dmalloc(&h->rx_agent, A)); CUDA_TRY(h, dmalloc(&h->rx_cnt, A));
  CUDA_TRY(h, dmalloc(&h->rx_rec_local, A)); CUDA_TRY(h, dmalloc(&h->rx_rec_tops, tiles));
  const size_t rtiles = sdb_scan_tops_len(c.max_recv_records);
  CUDA_TRY(h, dmalloc(&h->rx_plan, c.max_recv_records + 4)); CUDA_TRY(h, dmalloc(&h->rx_rec_off, A));
  CUDA_TRY(h, dmalloc(&h->rx_plan_tops, rtiles));
  CUDA_TRY(h, dmalloc(&h->rx_lb, sdb_lb_words(static_cast<uint32_t>(A / 64 + 2)) + 4));
  CUDA_TRY(h, dmalloc(&h->rx_totals, TOT_SLOTS));
  CUDA_TRY(h, dmalloc(&h->rx_big_list, A)); CUDA_TRY(h, dmalloc(&h->rx_big_count, 4));
  CUDA_TRY(h, dmalloc(&h->rx_count, A));
  CUDA_TRY(h, dmalloc(&h->rx_hdr, c.max_recv_records));
  h->pay_cap_gran = (c.max_recv_payload + SDB_GRANULE - 1) / SDB_GRANULE;
  if (h->pay_cap_gran >= 0x7FFFFFF0ull) return fail(h, SDB_EINVAL, "max_recv_payload too large (< 64 GiB per call)");
  CUDA_TRY(h, dmalloc(&h->rx_payload, h->pay_cap_gran * SDB_GRANULE));
  CUDA_TRY(h, cudaHostAlloc(reinterpret_cast<void**>(&h->totals_host), TOT_SLOTS * sizeof(unsigned long long), cudaHostAllocDefault));
  h->small_bytes = 64 + 1024ull * (32 + pad32(c.max_payload_bytes));
  CUDA_TRY(h, dmalloc(&h->rx_small, h->small_bytes));
  CUDA_TRY(h, cudaHostAlloc(reinterpret_cast<void**>(&h->small_host), h->small_bytes, cudaHostAllocDefault));

  // backends
  CUDA_TRY(h, dmalloc(&h->be_weight, c.max_backends));
  CUDA_TRY(h, dmalloc(&h->be_load, c.max_backends));
  CUDA_TRY(h, dmalloc(&h->be_scratch, static_cast<size_t>(c.max_backends) * 4 + 16));
  CUDA_TRY(h, dmalloc(&h->be_logtab, 257));
  {
    uint32_t tab[257];
    sdb_build_log2_table(tab);
    CUDA_TRY(h, cudaMemcpyAsync(h->be_logtab, tab, sizeof(tab), cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }

  h->gstart.assign(c.max_groups, 0); h->gcount.assign(c.max_groups, 0); h->gdefined.assign(c.max_groups, 0);
  h->ghost.resize(c.max_groups); h->gfull.resize(c.max_groups); h->gpos.resize(c.max_groups);
  h->gcount_full.assign(c.max_groups, 0);
  h->shard_of.assign(c.max_agents, static_cast<uint8_t>(c.shard_id));
  if (c.shard_id >= c.num_shards || c.num_shards > 255) return fail(h, SDB_EINVAL, "shard_id / num_shards out of range");
  CUDA_TRY(h, dmalloc(&h->member_pos_dev, c.member_pool_entries));
  CUDA_TRY(h, dmalloc(&h->lstart_dev, c.max_groups)); CUDA_TRY(h, dmalloc(&h->lcount_dev, c.max_groups));
  CUDA_TRY(h, cudaMemsetAsync(h->lcount_dev, 0, static_cast<size_t>(c.max_groups) * sizeof(uint32_t), h->stream));
  CUDA_TRY(h, cudaMemsetAsync(h->lstart_dev, 0, static_cast<size_t>(c.max_groups) * sizeof(uint32_t), h->stream));
  {
    const uint64_t cap64 = static_cast<uint64_t>(c.num_shards) * c.max_batch_sends;
    if (cap64 > 0x7FFFFFFFull) return fail(h, SDB_EINVAL, "num_shards * max_batch_sends too large");
    h->xs_cap = static_cast<uint32_t>(cap64);
    const size_t n = h->xs_cap, G1 = static_cast<size_t>(c.max_groups) + 1;
    const size_t GB = G1 * c.num_shards + 2;                 // (group, source) pairs
    const size_t wt = sdb_scan_tops_len(n), gt = sdb_scan_tops_len(GB);
    CUDA_TRY(h, dmalloc(&h->xs_w, n)); CUDA_TRY(h, dmalloc(&h->xs_w_local, n)); CUDA_TRY(h, dmalloc(&h->xs_w_tops, wt));
    CUDA_TRY(h, dmalloc(&h->xs_gs_cnt, GB)); CUDA_TRY(h, dmalloc(&h->xs_gs_local, GB)); CUDA_TRY(h, dmalloc(&h->xs_gs_tops, gt));
    CUDA_TRY(h, dmalloc(&h->xs_gs_cur, GB)); CUDA_TRY(h, dmalloc(&h->xs_gs_off, G1)); CUDA_TRY(h, dmalloc(&h->xs_gs_idx, n));
    CUDA_TRY(h, dmalloc(&h->xs_descs, n));
    CUDA_TRY(h, dmalloc(&h->xs_lw, n)); CUDA_TRY(h, dmalloc(&h->xs_lw_local, n)); CUDA_TRY(h, dmalloc(&h->xs_lw_tops, wt));
    CUDA_TRY(h, dmalloc(&h->xs_tab, 1));
    CUDA_TRY(h, dmalloc(&h->xs_gs_off_src, G1 * c.num_shards)); CUDA_TRY(h, dmalloc(&h->xs_gs_idx_src, n));
    CUDA_TRY(h, dmalloc(&h->xs_first, SDB_MAX_SRC + 1)); CUDA_TRY(h, dmalloc(&h->xs_lb, sdb_lb_words(static_cast<uint32_t>(n / 256 + 2)) + 4));
    CUDA_TRY(h, dmalloc(&h->cursor_dev, 1)); CUDA_TRY(h, dmalloc(&h->bb_dev, 1)); CUDA_TRY(h, dmalloc(&h->xs_hdrs, SDB_MAX_SRC));
    CUDA_TRY(h, cudaMemsetAsync(h->cursor_dev, 0, sizeof(sdb_cursor), h->stream)); CUDA_TRY(h, cudaMemsetAsync(h->bb_dev, 0, sizeof(sdb_batch_base), h->stream));
    {
      auto& S0 = h->xset[0];
      S0.descs = h->xs_descs; S0.gs_off_src = h->xs_gs_off_src; S0.gs_idx_src = h->xs_gs_idx_src; S0.first = h->xs_first;
      S0.lb = h->xs_lb; S0.hdrs = h->xs_hdrs; S0.tmp_list = h->scratch.list_dev;
      CUDA_TRY(h, dmalloc(&S0.totals, 1));
      CUDA_TRY(h, cudaEventCreateWithFlags(&S0.ready, cudaEventDisableTiming));
    }
    CUDA_TRY(h, cudaHostAlloc(reinterpret_cast<void**>(&h->cursor_host), sizeof(sdb_cursor), cudaHostAllocDefault));
    std::memset(h->cursor_host, 0, sizeof(sdb_cursor));
    h->xs_meta_stride = wire_meta_bytes(c.max_batch_sends, c.max_groups);
    CUDA_TRY(h, dmalloc(&h->xs_meta, h->xs_meta_stride * c.num_shards));
    CUDA_TRY(h, dmalloc(&h->shard_of_dev, c.max_agents));
    CUDA_TRY(h, cudaMemsetAsync(h->shard_of_dev, static_cast<int>(c.shard_id), c.max_agents, h->stream));
    CUDA_TRY(h, cudaHostAlloc(reinterpret_cast<void**>(&h->wire_host), wire_meta_bytes(c.max_batch_sends, c.max_groups), cudaHostAllocDefault));
    CUDA_TRY(h, cudaHostAlloc(reinterpret_cast<void**>(&h->hdrs_host), static_cast<size_t>(c.num_shards) * sizeof(sdb_wire_header), cudaHostAllocDefault));
  }

  sdb_dev_view& v = h->view;
  v.arena = h->arena; v.ring_hdr = h->ring_hdr; v.ring = h->ring; v.members = h->members; v.member_pos = h->member_pos_dev; v.ctr = h->ctr;
  v.ovf_log = h->ovf_log;
  v.gmask = h->arena_grans - 1; v.ring_slots = c.ring_slots; v.ring_shift = ilog2(c.ring_slots); v.max_agents = c.max_agents;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return SDB_OK;
}

static void lease_free(sdb_ctx* h);
static void dedup_free(sdb_ctx* h);

int sdb_destroy(sdb_handle h) {
  if (!h) return SDB_EINVAL;
  cudaSetDevice(h->cfg.device);
  ls_stop(h);
  if (h->ls_stream) cudaStreamDestroy(h->ls_stream);
  if (h->ls_mbox) cudaFreeHost(h->ls_mbox);
  if (h->ls_out) cudaFreeHost(h->ls_out);
  if (h->ls_plan) cudaFree(h->ls_plan);
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->pf_stream) { cudaStreamSynchronize(h->pf_stream); cudaStreamDestroy(h->pf_stream); }
  if (h->ev_pf_fork) cudaEventDestroy(h->ev_pf_fork);
  {
    auto& S1 = h->xset[1];
    void* own[] = {S1.descs, S1.gs_off_src, S1.gs_idx_src, S1.first, S1.lb, S1.hdrs, S1.tmp_list, S1.totals, h->xset[0].totals};
    for (void* p : own) if (p) cudaFree(p);
    for (auto& S : h->xset) if (S.ready) cudaEventDestroy(S.ready);
  }
  void* dev[] = {h->arena, h->ring_hdr, h->ring, h->members, h->ctr, h->gexcl_dev, h->rx_rec_off, h->rx_lb,
                 h->xs_gs_off_src, h->xs_gs_idx_src, h->xs_first, h->xs_lb, h->cursor_dev, h->bb_dev, h->xs_hdrs, h->owned_dev, h->agent_backend_dev,
                 h->scratch.descs_dev, h->scratch.payload_dev, h->scratch.list_dev, h->scratch.gs_off_dev,
                 h->scratch.gs_idx_dev, h->memb_off_dev, h->memb_grp_dev, h->memb_pos_dev, h->member_pos_dev,
                 h->lstart_dev, h->lcount_dev, h->xs_w, h->xs_w_local, h->xs_w_tops, h->xs_gs_cnt, h->xs_gs_local,
                 h->xs_gs_tops, h->xs_gs_cur, h->xs_gs_off, h->xs_gs_idx, h->xs_descs, h->xs_lw, h->xs_lw_local,
                 h->xs_lw_tops, h->xs_tab, h->xs_meta, h->shard_of_dev, h->rx_agent, h->rx_cnt,
                 h->rx_rec_local, h->rx_rec_tops, h->rx_plan, h->rx_plan_tops,
                 h->rx_totals, h->rx_big_list, h->rx_big_count, h->rx_count, h->rx_hdr, h->rx_payload,
                 h->be_weight, h->be_load, h->be_scratch, h->be_logtab, h->be_req_cost, h->be_out, h->digest,
                 h->cx.table, h->cx.rec_slot, h->cx.head, h->cx.head_local, h->cx.head_tops, h->cx.gran, h->cx.gran_local,
                 h->cx.gran_tops, h->cx.totals, h->cx.entry_out, h->cx.send_out, h->cx.payload_out, h->where_bits, h->where_kw,
                 h->id_tab, h->id_in, h->id_out, h->ss_tab, h->ss_cand,
                 h->rs_agent, h->rs_tot, h->rs_sort, h->rl_bits, h->rl_cnt, h->rl_pre, h->rl_tops, h->rl_sel, h->rl_tot};
  for (void* p : dev) if (p) cudaFree(p);
  lease_free(h);
  dedup_free(h);
  if (h->descs_host) cudaFreeHost(h->descs_host);
  if (h->list_host) cudaFreeHost(h->list_host);
  if (h->lp_host) cudaFreeHost(h->lp_host);
  if (h->lp_dev) cudaFree(h->lp_dev);
  if (h->ovf_log) cudaFree(h->ovf_log);
  if (h->ovf_seq) cudaFree(h->ovf_seq);
  if (h->gs_host) cudaFreeHost(h->gs_host);
  if (h->wire_host) cudaFreeHost(h->wire_host);
  if (h->hdrs_host) cudaFreeHost(h->hdrs_host);
  if (h->cursor_host) cudaFreeHost(h->cursor_host);
  if (h->totals_host) cudaFreeHost(h->totals_host);
  if (h->small_host) cudaFreeHost(h->small_host);
  if (h->rx_small) cudaFree(h->rx_small);
  if (h->staging_free) cudaEventDestroy(h->staging_free);
  if (h->prof.cap) {
    for (int i = 0; i < h->prof.cap; ++i) { cudaEventDestroy(h->prof.ev_a[i]); cudaEventDestroy(h->prof.ev_b[i]); }
    delete[] h->prof.kind; delete[] h->prof.ev_a; delete[] h->prof.ev_b;
  }
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return SDB_OK;
}

int sdb_set_stream(sdb_handle h, void* cuda_stream) {
  if (!h) return SDB_EINVAL;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (h->own_stream) { cudaStreamDestroy(h->stream); h->own_stream = false; }
  h->stream = static_cast<cudaStream_t>(cuda_stream);
  return SDB_OK;
}

int sdb_sync(sdb_handle h) {
  if (!h) return SDB_EINVAL;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->stream_busy = false;
  return SDB_OK;
}

int sdb_profile(sdb_handle h, int enable) {
  if (!h) return SDB_EINVAL;
  sdb_profiler& p = h->prof;
  if (enable && !p.cap) {
    p.cap = 8192;
    p.kind = new int[p.cap]; p.ev_a = new cudaEvent_t[p.cap]; p.ev_b = new cudaEvent_t[p.cap];
    for (int i = 0; i < p.cap; ++i) { CUDA_TRY(h, cudaEventCreate(&p.ev_a[i])); CUDA_TRY(h, cudaEventCreate(&p.ev_b[i])); }
  }
  p.enabled = enable ? 1 : 0;
  if (enable) p.n = 0;
  return SDB_OK;
}

int sdb_profile_read_n(sdb_handle h, uint32_t n, double* ms_out, uint64_t* count_out) {
  if (!h || !ms_out || !count_out) return SDB_EINVAL;
  for (uint32_t k = 0; k < n; ++k) { ms_out[k] = 0.0; count_out[k] = 0; }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  const int classes = static_cast<int>(std::min<uint32_t>(n, SDB_PK_CLASSES));
  sdb_profiler& p = h->prof;
  for (int i = 0; i < p.n; ++i) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, p.ev_a[i], p.ev_b[i]) == cudaSuccess && p.kind[i] < classes) {
      ms_out[p.kind[i]] += ms; count_out[p.kind[i]] += 1;
    }
  }
  p.n = 0;
  return SDB_OK;
}

// ABI-1 callers pass arrays of SDB_PK_N entries: the classes past it are left out
int sdb_profile_read(sdb_handle h, double* ms_out, uint64_t* count_out) {
  return sdb_profile_read_n(h, SDB_PK_N, ms_out, count_out);
}

int sdb_get_stats(sdb_handle h, sdb_stats* out) {
  if (!h || !out) return SDB_EINVAL;
  { int rcc = cursor_to_host(h); if (rcc != SDB_OK) return rcc; }
  sdb_dev_counters c;
  CUDA_TRY(h, cudaMemcpyAsync(&c, h->ctr, sizeof(c), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  out->next_seq = h->next_seq; out->enqueued = c.enqueued; out->delivered = c.delivered;
  out->ring_overflow = c.ring_overflow; out->skipped_sender = c.skipped_sender;
  out->arena_tail_bytes = h->arena_tail * SDB_GRANULE; out->arena_floor_bytes = h->arena_floor * SDB_GRANULE;
  out->n_agents = h->n_agents; out->kernel_launches = h->launches; out->backend_picks = h->picks;
  return SDB_OK;
}

int sdb_debug_set_arena_pos(sdb_handle h, uint64_t granules) {
  if (!h) return SDB_EINVAL;
  sdb_stats st;
  int rc = sdb_get_stats(h, &st);
  if (rc != SDB_OK) return rc;
  if (st.enqueued != st.delivered + 0 && st.enqueued - st.delivered != 0) return fail(h, SDB_EINVAL, "messages pending");
  h->arena_tail = granules; h->arena_floor = granules;
  h->dev_stale = true;
  return SDB_OK;
}

int sdb_advance_seq(sdb_handle h, uint64_t next_seq) {
  if (!h) return SDB_EINVAL;
  { int rcc = cursor_to_host(h); if (rcc != SDB_OK) return rcc; }
  if (next_seq > h->next_seq) { h->next_seq = next_seq; h->dev_stale = true; }
  return SDB_OK;
}

int sdb_register_agents(sdb_handle h, uint32_t n, const uint32_t* agent_idx) {
  if (!h || (n && !agent_idx)) return SDB_EINVAL;
  for (uint32_t i = 0; i < n; ++i) {
    if (agent_idx[i] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "agent index >= max_agents");
    h->n_agents = std::max(h->n_agents, agent_idx[i] + 1);
  }
  return SDB_OK;
}

int sdb_deregister_agents(sdb_handle h, uint32_t n, const uint32_t* agent_idx) {
  if (!h || (n && !agent_idx)) return SDB_EINVAL;
  for (uint32_t i = 0; i < n; ++i)
    if (agent_idx[i] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "agent index >= max_agents");
  return SDB_OK;   // ring and read position are kept (consumer-group offsets survive close, App. A rule 11)
}

// (re)compute the members this shard owns for group g and their positions in the full list
static void localize_group(sdb_ctx* h, uint32_t g) {
  const std::vector<uint32_t>& full = h->gfull[g];
  std::vector<uint32_t>& loc = h->ghost[g];
  std::vector<uint32_t>& pos = h->gpos[g];
  loc.clear(); pos.clear();
  for (uint32_t j = 0; j < full.size(); ++j)
    if (!h->sharded || h->shard_of[full[j]] == h->cfg.shard_id) { loc.push_back(full[j]); pos.push_back(j); }
  h->gcount_full[g] = static_cast<uint32_t>(full.size());
}

// write every defined group's local list into the device pools from scratch
static int upload_all_groups(sdb_ctx* h) {
  uint64_t used = 0;
  for (uint32_t k = 0; k < h->cfg.max_groups; ++k) if (h->gdefined[k]) used += h->ghost[k].size();
  if (used > h->cfg.member_pool_entries) return fail(h, SDB_ECAPACITY, "member pool exhausted");
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  std::vector<uint32_t> flat, fpos; flat.reserve(used); fpos.reserve(used);
  for (uint32_t k = 0; k < h->cfg.max_groups; ++k) if (h->gdefined[k]) {
    h->gstart[k] = flat.size(); h->gcount[k] = static_cast<uint32_t>(h->ghost[k].size());
    flat.insert(flat.end(), h->ghost[k].begin(), h->ghost[k].end());
    fpos.insert(fpos.end(), h->gpos[k].begin(), h->gpos[k].end());
  }
  if (!flat.empty()) {
    CUDA_TRY(h, upload(h, h->members, flat.data(), flat.size() * sizeof(uint32_t)));
    CUDA_TRY(h, upload(h, h->member_pos_dev, fpos.data(), fpos.size() * sizeof(uint32_t)));
  }
  h->member_used = flat.size();
  h->memb_dirty = true; h->ltab_dirty = true;
  return SDB_OK;
}

int sdb_create_group(sdb_handle h, uint32_t g, uint32_t n_members, const uint32_t* member_idx) {
  if (!h || (n_members && !member_idx)) return SDB_EINVAL;
  if (g >= h->cfg.max_groups) return fail(h, SDB_EINVAL, "group index >= max_groups");
  for (uint32_t i = 0; i < n_members; ++i)
    if (member_idx[i] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "member index >= max_agents");
  h->memb_dirty = true; h->ltab_dirty = true;
  h->gfull[g].assign(member_idx, member_idx + n_members);
  localize_group(h, g);
  h->gdefined[g] = 1;
  const std::vector<uint32_t>& loc = h->ghost[g];
  for (uint32_t m : loc) h->n_agents = std::max(h->n_agents, m + 1);   // members will receive: keep them inside the sweeps
  if (h->member_used + loc.size() > h->cfg.member_pool_entries) return upload_all_groups(h);   // compact the pool
  h->gstart[g] = h->member_used; h->gcount[g] = static_cast<uint32_t>(loc.size());
  if (!loc.empty()) {
    // pageable source: cudaMemcpyAsync stages it before returning, ordered after earlier kernels on the stream
    CUDA_TRY(h, cudaMemcpyAsync(h->members + h->member_used, loc.data(), loc.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(h->member_pos_dev + h->member_used, h->gpos[g].data(), loc.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  }
  h->member_used += loc.size();
  if (h->member_used > 0xFFFFFFFFull) return fail(h, SDB_ECAPACITY, "member pool beyond 2^32 entries");
  return SDB_OK;
}

uint64_t sdb_wire_bytes(sdb_handle h, uint32_t max_sends, uint64_t max_payload_bytes) {
  // header + descriptors + group buckets + payload (+ slack); broadcast recipient lists count towards max_payload_bytes
  const uint32_t G = h ? h->cfg.max_groups : 0;
  // ... + the cross-rank control block (sdb_wire_ctrl) in the last 128 bytes, outside everything an export writes
  return wire_meta_bytes(max_sends, G) + ((max_payload_bytes + 256 + 127) & ~127ull) + sizeof(sdb_wire_ctrl);
}

int sdb_set_agent_shards(sdb_handle h, uint32_t n, const uint8_t* shard_of) {
  if (!h || (n && !shard_of)) return SDB_EINVAL;
  if (n > h->cfg.max_agents) return fail(h, SDB_EINVAL, "n > max_agents");
  for (uint32_t i = 0; i < n; ++i) {
    if (shard_of[i] >= h->cfg.num_shards) return fail(h, SDB_EINVAL, "shard id >= num_shards");
    h->shard_of[i] = shard_of[i];
  }
  h->sharded = h->cfg.num_shards > 1;
  if (h->sharded) h->n_agents = h->cfg.max_agents;   // receivers are named by other ranks: sweeps cover the whole index space
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, upload(h, h->shard_of_dev, h->shard_of.data(), h->cfg.max_agents));
  {
    std::vector<uint32_t> owned;
    for (uint32_t i = 0; i < h->cfg.max_agents; ++i) if (h->shard_of[i] == h->cfg.shard_id) owned.push_back(i);
    if (!h->owned_dev) CUDA_TRY(h, dmalloc(&h->owned_dev, h->cfg.max_agents));
    if (!owned.empty()) CUDA_TRY(h, upload(h, h->owned_dev, owned.data(), owned.size() * sizeof(uint32_t)));
    h->n_owned = static_cast<uint32_t>(owned.size());
  }
  // groups created earlier are re-filtered against the new ownership map
  bool any = false;
  for (uint32_t g = 0; g < h->cfg.max_groups; ++g) if (h->gdefined[g]) { localize_group(h, g); any = true; }
  return any ? upload_all_groups(h) : SDB_OK;
}

// kind == nullptr: every send is a group send (target = group index)
static int export_common(sdb_ctx* h, uint32_t n, const uint32_t* sender, const uint8_t* kind, const uint32_t* target,
                         uint32_t n_lists, const uint64_t* list_off, const uint32_t* list_idx, const uint8_t* prio,
                         const uint8_t* type, const uint16_t* len, const uint64_t* payload_off, const uint8_t* payload,
                         uint64_t payload_bytes, const double* timestamp, void* wire_dev, uint64_t wire_cap,
                         uint64_t explicit_seq_base = 0) {
  if (!h || !wire_dev) return SDB_EINVAL;
  if (n && (!sender || !target || !len)) return fail(h, SDB_EINVAL, "null array");
  if (n > h->cfg.max_batch_sends) return fail(h, SDB_ECAPACITY, "n exceeds max_batch_sends");
  if (payload_bytes && !payload) return fail(h, SDB_EINVAL, "null payload");
  const uint64_t n_list = (n_lists && list_off) ? list_off[n_lists] : 0;
  if (n_list > h->cfg.list_pool_entries) return fail(h, SDB_ECAPACITY, "recipient lists exceed list_pool_entries");
  const uint32_t G = h->cfg.max_groups;
  const uint64_t desc_off = sizeof(sdb_wire_header);
  const uint64_t gso_off = desc_off + static_cast<uint64_t>(n) * sizeof(sdb_send_desc);
  const uint64_t gsi_off = gso_off + (static_cast<uint64_t>(G) + 1) * 4;
  const uint64_t l_off = gsi_off + static_cast<uint64_t>(n) * 4;            // room for every send being a group send
  const uint64_t pay_off = (l_off + n_list * sizeof(uint32_t) + 63) & ~63ull;
  if (pay_off + payload_bytes + 64 + sizeof(sdb_wire_ctrl) > wire_cap) return fail(h, SDB_ECAPACITY, "wire buffer too small (sdb_wire_bytes)");
  CUDA_TRY(h, cudaEventSynchronize(h->staging_free));
  sdb_wire_header* wh = reinterpret_cast<sdb_wire_header*>(h->wire_host);
  sdb_send_desc* wd = reinterpret_cast<sdb_send_desc*>(h->wire_host + desc_off);
  uint32_t* gso = reinterpret_cast<uint32_t*>(h->wire_host + gso_off);
  uint32_t* gsi = reinterpret_cast<uint32_t*>(h->wire_host + gsi_off);
  std::memset(gso, 0, (static_cast<size_t>(G) + 1) * 4);
  uint32_t n_group = 0;
  std::memset(wh, 0, sizeof(*wh));
  uint64_t rec = 0; uint32_t max_padlen = 0, n_other = 0;
  for (uint64_t k = 0; k < n_list; ++k) if (list_idx[k] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "recipient index out of range");
  for (uint32_t i = 0; i < n; ++i) {
    sdb_send_desc d; std::memset(&d, 0, sizeof(d));
    const uint32_t k = kind ? kind[i] : 1u;
    if (sender[i] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "sender index out of range");
    if (len[i] > h->cfg.max_payload_bytes) return fail(h, SDB_EINVAL, "payload longer than max_payload_bytes");
    const uint64_t off = payload_off ? payload_off[i] : 0;
    if ((off & 15u) || off + len[i] > payload_bytes) return fail(h, SDB_EINVAL, "bad payload_off");
    if ((prio ? prio[i] : 1) > 3) return fail(h, SDB_EINVAL, "priority out of range");
    if (rec > 0xFFFFFFFFull) return fail(h, SDB_ECAPACITY, "batch exceeds 2^32 records");
    const uint32_t pl = pad32(len[i]);
    max_padlen = std::max(max_padlen, pl);
    d.payload_off = off; d.timestamp = timestamp ? timestamp[i] : 0.0;
    d.sender = sender[i]; d.group = SDB_NO_GROUP; d.len = len[i]; d.prio = prio ? prio[i] : 1; d.type = type ? type[i] : 0;
    d.rgran = 1u + pl / SDB_GRANULE; d.rec0 = static_cast<uint32_t>(rec);
    if (k == 1) {
      const uint32_t g = target[i];
      if (g >= h->cfg.max_groups || !h->gdefined[g]) return fail(h, SDB_ENOTFOUND, "unknown group index");
      d.group = g; rec += h->gcount_full[g];
      gso[g + 1]++; ++n_group;
    } else if (k == 0) {
      if (target[i] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "receiver index out of range");
      d.mstart = target[i]; d.mcount = 1; d.flags = SDB_DESC_P2P; rec += 1; ++n_other;
    } else if (k == 2) {
      if (target[i] >= n_lists) return fail(h, SDB_EINVAL, "list number out of range");
      const uint64_t b = list_off[target[i]], e = list_off[target[i] + 1];
      if (e < b || e > n_list) return fail(h, SDB_EINVAL, "bad list_off");
      d.mstart = static_cast<uint32_t>(b); d.mcount = static_cast<uint32_t>(e - b); d.flags = SDB_DESC_LIST_TEMP; rec += 1; ++n_other;
    } else return fail(h, SDB_EINVAL, "kind must be 0, 1 or 2");
    wd[i] = d;
  }
  // bucket the group sends by group: counting sort, ascending send index inside a bucket
  for (uint32_t g = 0; g < G; ++g) gso[g + 1] += gso[g];
  {
    std::vector<uint32_t> cur(gso, gso + G);
    for (uint32_t i = 0; i < n; ++i) if (wd[i].group != SDB_NO_GROUP) gsi[cur[wd[i].group]++] = i;
  }
  wh->magic = SDB_WIRE_MAGIC; wh->n_sends = n; wh->total_recs = rec; wh->payload_bytes = payload_bytes;
  wh->desc_off = desc_off; wh->payload_off = pay_off; wh->max_padlen = max_padlen; wh->n_other = n_other;
  wh->list_off = l_off; wh->n_list = static_cast<uint32_t>(n_list);
  wh->n_group_sends = n_group; wh->gs_off_off = gso_off; wh->gs_idx_off = gsi_off; wh->max_groups = G;
  wh->explicit_seq = explicit_seq_base ? 1u : 0u; wh->seq_base = explicit_seq_base;
  uint8_t* w = static_cast<uint8_t*>(wire_dev);
  CUDA_TRY(h, cudaMemcpyAsync(w, h->wire_host, l_off, cudaMemcpyHostToDevice, h->stream));
  if (n_list) {
    std::memcpy(h->list_host, list_idx, n_list * sizeof(uint32_t));
    CUDA_TRY(h, cudaMemcpyAsync(w + l_off, h->list_host, n_list * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  }
  if (payload_bytes) CUDA_TRY(h, cudaMemcpyAsync(w + pay_off, payload, payload_bytes, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaEventRecord(h->staging_free, h->stream));
  return SDB_OK;
}

int sdb_export_group_batch(sdb_handle h, uint32_t n, const uint32_t* sender, const uint32_t* group_idx, const uint8_t* prio,
                           const uint8_t* type, const uint16_t* len, const uint64_t* payload_off, const uint8_t* payload,
                           uint64_t payload_bytes, const double* timestamp, void* wire_dev, uint64_t wire_cap) {
  return export_common(h, n, sender, nullptr, group_idx, 0, nullptr, nullptr, prio, type, len, payload_off, payload, payload_bytes,
                       timestamp, wire_dev, wire_cap);
}

int sdb_export_mixed_batch(sdb_handle h, uint32_t n, const uint32_t* sender, const uint8_t* kind, const uint32_t* target,
                           uint32_t n_lists, const uint64_t* list_off, const uint32_t* list_idx, const uint8_t* prio,
                           const uint8_t* type, const uint16_t* len, const uint64_t* payload_off, const uint8_t* payload,
                           uint64_t payload_bytes, const double* timestamp, void* wire_dev, uint64_t wire_cap) {
  if (h && n && !kind) return fail(h, SDB_EINVAL, "null kind array");
  return export_common(h, n, sender, kind, target, n_lists, list_off, list_idx, prio, type, len, payload_off, payload, payload_bytes,
                       timestamp, wire_dev, wire_cap);
}

int sdb_export_mixed_batch_seq(sdb_handle h, uint64_t seq_base, uint32_t n, const uint32_t* sender, const uint8_t* kind,
                               const uint32_t* target, uint32_t n_lists, const uint64_t* list_off, const uint32_t* list_idx,
                               const uint8_t* prio, const uint8_t* type, const uint16_t* len, const uint64_t* payload_off,
                               const uint8_t* payload, uint64_t payload_bytes, const double* timestamp, void* wire_dev,
                               uint64_t wire_cap) {
  if (h && n && !kind) return fail(h, SDB_EINVAL, "null kind array");
  if (h && seq_base == 0) return fail(h, SDB_EINVAL, "explicit seq_base must be non-zero");
  return export_common(h, n, sender, kind, target, n_lists, list_off, list_idx, prio, type, len, payload_off, payload, payload_bytes,
                       timestamp, wire_dev, wire_cap, seq_base);
}

// ---- peer-memory transport: export buffers that other ranks map with CUDA IPC ---------------------
int sdb_wire_alloc(sdb_handle h, uint64_t bytes, void** dev_out, void* ipc_handle_out) {
  if (!h || !dev_out || bytes == 0) return SDB_EINVAL;
  void* p = nullptr;
  CUDA_TRY(h, cudaMalloc(&p, bytes));
  CUDA_TRY(h, cudaMemsetAsync(p, 0, bytes, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (ipc_handle_out) {
    cudaIpcMemHandle_t hd;
    CUDA_TRY(h, cudaIpcGetMemHandle(&hd, p));
    static_assert(sizeof(hd) == 64, "cudaIpcMemHandle_t is 64 bytes");
    std::memcpy(ipc_handle_out, &hd, sizeof(hd));
  }
  *dev_out = p;
  return SDB_OK;
}

int sdb_wire_open(sdb_handle h, const void* ipc_handle, void** dev_out) {
  if (!h || !ipc_handle || !dev_out) return SDB_EINVAL;
  cudaIpcMemHandle_t hd;
  std::memcpy(&hd, ipc_handle, sizeof(hd));
  CUDA_TRY(h, cudaIpcOpenMemHandle(dev_out, hd, cudaIpcMemLazyEnablePeerAccess));
  return SDB_OK;
}

int sdb_wire_close(sdb_handle h, void* dev, int opened) {
  if (!h || !dev) return SDB_EINVAL;
  ls_stop(h);
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (opened) CUDA_TRY(h, cudaIpcCloseMemHandle(dev)); else CUDA_TRY(h, cudaFree(dev));
  return SDB_OK;
}

int sdb_import_wire_batches(sdb_handle h, uint32_t n_src, const void* wire_dev_all, uint64_t wire_stride, uint64_t* seq_base_out) {
  if (!h || !wire_dev_all || n_src == 0 || n_src > SDB_MAX_SRC) return SDB_EINVAL;
  const void* ptrs[SDB_MAX_SRC];
  for (uint32_t s = 0; s < n_src; ++s) ptrs[s] = static_cast<const uint8_t*>(wire_dev_all) + static_cast<uint64_t>(s) * wire_stride;
  return sdb_import_wire_ptrs(h, n_src, ptrs, seq_base_out);
}

int sdb_import_wire_ptrs(sdb_handle h, uint32_t n_src, const void* const* wire_ptrs, uint64_t* seq_base_out) {
  if (!h || !wire_ptrs || n_src == 0) return SDB_EINVAL;
  { int rcc = cursor_to_host(h); if (rcc != SDB_OK) return rcc; }
  if (seq_base_out) *seq_base_out = h->next_seq;
  if (n_src > h->cfg.num_shards || n_src > SDB_MAX_SRC) return fail(h, SDB_EINVAL, "n_src > num_shards (or > 16)");
  { int rc1 = ensure_ltab(h); if (rc1 != SDB_OK) return rc1; }
  if (h->memb_dirty) { int rc0 = rebuild_inverse(h); if (rc0 != SDB_OK) return rc0; }
  const uint32_t n_cap = n_src * h->cfg.max_batch_sends;
  sdb_import_args a{};
  for (uint32_t k = 0; k < n_src; ++k) {
    if (!wire_ptrs[k]) return fail(h, SDB_EINVAL, "null wire pointer");
    a.wire[k] = static_cast<const uint8_t*>(wire_ptrs[k]);
    a.meta[k] = a.wire[k];
    cudaPointerAttributes pa;
    if (cudaPointerGetAttributes(&pa, wire_ptrs[k]) == cudaSuccess && pa.type == cudaMemoryTypeDevice && pa.device != h->cfg.device) {
      // header + descriptors of a peer's batch: one DMA copy over NVLink instead of per-thread remote reads;
      // the payload (the bulk) stays remote and is pulled by the fan-out kernel's TMA loads
      uint8_t* dst = h->xs_meta + static_cast<uint64_t>(k) * h->xs_meta_stride;
      CUDA_TRY(h, cudaMemcpyAsync(dst, wire_ptrs[k], h->xs_meta_stride, cudaMemcpyDeviceToDevice, h->stream));
      a.meta[k] = dst;
    }
  }
  a.n_src = n_src; a.max_sends = h->cfg.max_batch_sends; a.tab = h->xs_tab;
  a.lstart = h->lstart_dev; a.lcount = h->lcount_dev; a.max_groups = h->cfg.max_groups;
  a.w = h->xs_w; a.gs_cnt = h->xs_gs_cnt; a.descs = h->xs_descs; a.w_local = h->xs_w_local; a.w_tops = h->xs_w_tops;
  a.gs_off = h->xs_gs_off; a.gs_idx = h->xs_gs_idx;
  a.shard_of = h->shard_of_dev; a.shard_id = h->cfg.shard_id; a.max_agents = h->cfg.max_agents;
  a.lw = h->xs_lw; a.lw_local = h->xs_lw_local; a.lw_tops = h->xs_lw_tops;
  a.tmp_list = h->scratch.list_dev; a.list_cap = static_cast<uint32_t>(std::min<uint64_t>(h->cfg.list_pool_entries, 0xFFFFFFFFull));
  int nl = 0;
  cudaError_t e = sdb_launch_import_measure(&a, n_cap, h->xs_w_local, h->xs_w_tops, h->xs_gs_local, h->xs_gs_tops,
                                            h->xs_gs_cur /* goff */, h->xs_lw_local, h->xs_lw_tops, h->rx_totals + TOT_IMPORT_GRANULES, h->stream, &h->prof, &nl);
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("import measure: ") + cudaGetErrorString(e));
  // the host needs the arena footprint and the sequence numbers consumed: one small sync
  CUDA_TRY(h, cudaMemcpyAsync(h->totals_host + TOT_IMPORT_GRANULES, h->rx_totals + TOT_IMPORT_GRANULES, 2 * sizeof(unsigned long long),
                              cudaMemcpyDeviceToHost, h->stream));
  for (uint32_t k = 0; k < n_src; ++k)
    CUDA_TRY(h, cudaMemcpyAsync(h->hdrs_host + k, wire_ptrs[k], sizeof(sdb_wire_header), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  uint64_t total_recs = 0, n_other = 0, explicit_end = 0; uint32_t max_padlen = 0;
  if (h->totals_host[TOT_IMPORT_OWNED] > a.list_cap) return fail(h, SDB_ECAPACITY, "owned recipients of this import exceed list_pool_entries");
  for (uint32_t s = 0; s < n_src; ++s) {
    const sdb_wire_header& wh = h->hdrs_host[s];
    n_other += wh.n_other;
    if (wh.magic == SDB_WIRE_MAGIC && wh.explicit_seq) explicit_end = std::max<uint64_t>(explicit_end, wh.seq_base + wh.total_recs);
    if (wh.magic != SDB_WIRE_MAGIC) return fail(h, SDB_EINVAL, "wire batch without magic (not exported by sdb_export_group_batch?)");
    if (wh.n_sends > h->cfg.max_batch_sends) return fail(h, SDB_ECAPACITY, "wire batch larger than max_batch_sends");
    total_recs += wh.total_recs; max_padlen = std::max(max_padlen, wh.max_padlen);
  }
  const uint64_t total_grans = h->totals_host[TOT_IMPORT_GRANULES];
  uint64_t base = 0;
  int rc = arena_reserve(h, total_grans, &base);
  if (rc != SDB_OK) return rc;
  e = sdb_launch_import_localize(&a, n_cap, h->xs_gs_cur /* goff */, h->xs_gs_off, h->stream, &h->prof, &nl);
  if (e == cudaSuccess)
    e = sdb_launch_fanout(&h->view, h->xs_descs, n_cap, nullptr, h->scratch.list_dev, h->next_seq, base, max_padlen,
                          h->cfg.fanout_variant >= 2 ? 3 : static_cast<int>(h->cfg.fanout_variant), h->sm_count, h->stream, &h->prof, nullptr, 0u);
  if (e == cudaSuccess) {
    sdb_pull_view pv{h->memb_off_dev, h->memb_grp_dev, h->memb_pos_dev, h->xs_gs_off, h->xs_gs_idx, 1u, 0u, 0u, nullptr};
    e = sdb_launch_pull(&h->view, &pv, h->xs_descs, h->n_agents, h->cfg.max_groups, h->gexcl_dev, h->n_excl_groups,
                        h->n_shared_agents, h->lstart_dev, h->lcount_dev, base, n_other ? 0 : 1, h->stream, &h->prof, &nl, nullptr, 0u);
  }
  if (e == cudaSuccess && n_other) {     // p2p / broadcast copies claimed their slots with atomics: sort them into place
    e = sdb_launch_commit(&h->view, h->n_agents, static_cast<uint32_t>(base), h->rx_big_list, h->rx_big_count + 1, h->sm_count, h->stream, &h->prof, nullptr);
    h->launches += 2;
  }
  h->launches += nl + 1;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("import launch: ") + cudaGetErrorString(e));
  h->next_seq = std::max<uint64_t>(h->next_seq + (explicit_end ? 0 : total_recs), explicit_end);
  h->arena_tail = base + total_grans;
  h->dev_stale = true;
  h->stream_busy = true;
  return SDB_OK;
}

// ---- flags + asynchronous import -------------------------------------------------------------------------------
static uint32_t* ctrl_word(const void* wire, uint64_t wire_bytes, int which) {
  uint8_t* c = static_cast<uint8_t*>(const_cast<void*>(wire)) + wire_bytes - sizeof(sdb_wire_ctrl);
  return reinterpret_cast<uint32_t*>(c) + which;           // 0 = ready, 1 = done
}

int sdb_wire_publish(sdb_handle h, void* wire_dev, uint64_t wire_bytes, uint32_t step) {
  if (!h || !wire_dev || wire_bytes < sizeof(sdb_wire_ctrl)) return SDB_EINVAL;
  CUDA_TRY(h, sdb_launch_wire_set(ctrl_word(wire_dev, wire_bytes, 0), step, h->stream));
  h->launches += 1;
  return SDB_OK;
}

int sdb_wire_wait_done(sdb_handle h, uint32_t n_src, const void* const* wire_ptrs, uint64_t wire_bytes, uint32_t step) {
  if (!h || !wire_ptrs || n_src == 0 || n_src > SDB_MAX_SRC || wire_bytes < sizeof(sdb_wire_ctrl)) return SDB_EINVAL;
  const uint32_t* flags[SDB_MAX_SRC];
  for (uint32_t k = 0; k < n_src; ++k) flags[k] = ctrl_word(wire_ptrs[k], wire_bytes, 1);
  CUDA_TRY(h, sdb_launch_wire_wait(flags, n_src, step, h->stream, nullptr, nullptr));
  h->launches += 1;
  return SDB_OK;
}

// traffic shapes the device-only import handles (everything else takes the synchronous body between the same flags)
static bool async_fast(const sdb_ctx* h) {
  return pad32(h->cfg.max_payload_bytes) <= 512 && h->n_shared_agents == 0 && h->n_excl_groups != 0 && h->cfg.fanout_variant >= 2;
}

// wait for the sources' flags + fused localize into buffer set S, on stream `st`; `defer`: leave the placement to
// k_import_place (the cursor belongs to the shard's stream)
static int xs_localize(sdb_ctx* h, sdb_ctx::XsSet& S, uint32_t n_src, const void* const* wire_ptrs, uint64_t wire_bytes,
                       uint32_t step, cudaStream_t st, bool defer) {
  const uint32_t* ready[SDB_MAX_SRC];
  for (uint32_t k = 0; k < n_src; ++k) ready[k] = ctrl_word(wire_ptrs[k], wire_bytes, 0);
  const int pw = sdb_prof_begin(&h->prof, SDB_PK_XWAIT, st);
  CUDA_TRY(h, sdb_launch_wire_wait(ready, n_src, step, st, wire_ptrs, S.hdrs));
  sdb_prof_end(&h->prof, pw, st);
  sdb_import2_args a{};
  for (uint32_t k = 0; k < n_src; ++k) a.wire[k] = static_cast<const uint8_t*>(wire_ptrs[k]);
  a.n_src = n_src; a.max_sends = h->cfg.max_batch_sends; a.max_groups = h->cfg.max_groups; a.shard_id = h->cfg.shard_id;
  a.max_agents = h->cfg.max_agents; a.lcount = h->lcount_dev; a.lstart = h->lstart_dev; a.shard_of = h->shard_of_dev;
  a.descs = S.descs; a.gs_off_src = S.gs_off_src; a.gs_idx_src = S.gs_idx_src; a.first = S.first;
  a.tmp_list = S.tmp_list; a.list_cap = static_cast<uint32_t>(std::min<uint64_t>(h->cfg.list_pool_entries, 0x7FFFFFF0ull));
  a.lb = S.lb; a.cur = h->cursor_dev; a.bb = h->bb_dev; a.arena_grans = h->arena_grans;
  a.hdrs = S.hdrs; a.commit_count = h->rx_big_count + 1; a.totals = defer ? S.totals : nullptr;
  // shared payloads: a send's local region is lc headers + one payload (the fast shape already guarantees payloads
  // <= 512 bytes and exclusive groups; local groups must fit the 16-bit header-to-payload distance)
  S.shared = h->shared_cfg && h->max_lcount <= 65535u;
  a.shared = S.shared ? 1u : 0u;
  int nl = 1;
  cudaError_t e = sdb_launch_import_fused(&a, st, &h->prof, &nl);
  h->launches += nl;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("import localize launch: ") + cudaGetErrorString(e));
  return SDB_OK;
}

static int import_args_check(sdb_handle h, uint32_t n_src, const void* const* wire_ptrs, uint64_t wire_bytes) {
  if (!h || !wire_ptrs || n_src == 0 || wire_bytes < sizeof(sdb_wire_ctrl)) return SDB_EINVAL;
  if (n_src > h->cfg.num_shards || n_src > SDB_MAX_SRC) return fail(h, SDB_EINVAL, "n_src > num_shards (or > 16)");
  for (uint32_t k = 0; k < n_src; ++k) if (!wire_ptrs[k]) return fail(h, SDB_EINVAL, "null wire pointer");
  { int rc1 = ensure_ltab(h); if (rc1 != SDB_OK) return rc1; }
  if (h->memb_dirty) { int rc0 = rebuild_inverse(h); if (rc0 != SDB_OK) return rc0; }
  return SDB_OK;
}

int sdb_import_prefetch(sdb_handle h, uint32_t n_src, const void* const* wire_ptrs, uint64_t wire_bytes, uint32_t step) {
  { int rc = import_args_check(h, n_src, wire_ptrs, wire_bytes); if (rc != SDB_OK) return rc; }
  if (!async_fast(h)) return SDB_OK;                  // the synchronous body has nothing to run ahead
  if (!h->pf_stream) {
    auto& S1 = h->xset[1];
    const size_t n = h->xs_cap, G1 = static_cast<size_t>(h->cfg.max_groups) + 1;
    CUDA_TRY(h, cudaStreamCreateWithFlags(&h->pf_stream, cudaStreamNonBlocking));
    CUDA_TRY(h, cudaEventCreateWithFlags(&h->ev_pf_fork, cudaEventDisableTiming));
    CUDA_TRY(h, dmalloc(&S1.descs, n)); CUDA_TRY(h, dmalloc(&S1.gs_off_src, G1 * h->cfg.num_shards)); CUDA_TRY(h, dmalloc(&S1.gs_idx_src, n));
    CUDA_TRY(h, dmalloc(&S1.first, SDB_MAX_SRC + 1)); CUDA_TRY(h, dmalloc(&S1.lb, sdb_lb_words(static_cast<uint32_t>(n / 256 + 2)) + 4));
    CUDA_TRY(h, dmalloc(&S1.hdrs, SDB_MAX_SRC)); CUDA_TRY(h, dmalloc(&S1.tmp_list, h->cfg.list_pool_entries));
    CUDA_TRY(h, dmalloc(&S1.totals, 1));
    CUDA_TRY(h, cudaEventCreateWithFlags(&S1.ready, cudaEventDisableTiming));
  }
  auto& S = h->xset[step & 1u];
  if (S.pending) return S.step == step ? SDB_OK : fail(h, SDB_EINVAL, "a prefetched import of this parity has not been imported yet");
  // the set's previous user (the import two steps ago) and the table uploads above are ordered before the prefetch;
  // what the caller enqueues on the shard's stream AFTER this call (the receive of the current step) runs beside it
  CUDA_TRY(h, cudaEventRecord(h->ev_pf_fork, h->stream));
  CUDA_TRY(h, cudaStreamWaitEvent(h->pf_stream, h->ev_pf_fork, 0));
  { int rc = xs_localize(h, S, n_src, wire_ptrs, wire_bytes, step, h->pf_stream, true); if (rc != SDB_OK) return rc; }
  CUDA_TRY(h, cudaEventRecord(S.ready, h->pf_stream));
  h->launches += 1;
  S.pending = true; S.step = step;
  return SDB_OK;
}

int sdb_import_wire_ptrs_async(sdb_handle h, uint32_t n_src, const void* const* wire_ptrs, uint64_t wire_bytes, uint32_t step) {
  { int rc = import_args_check(h, n_src, wire_ptrs, wire_bytes); if (rc != SDB_OK) return rc; }
  uint32_t* my_done = ctrl_word(wire_ptrs[h->cfg.shard_id < n_src ? h->cfg.shard_id : 0], wire_bytes, 1);
  if (!async_fast(h)) {
    // general traffic shapes (payloads above 512 bytes, agents in several groups): the synchronous import body
    // 1. wait (on the stream, not on the host) until every source's export of this step is complete
    const uint32_t* ready[SDB_MAX_SRC];
    for (uint32_t k = 0; k < n_src; ++k) ready[k] = ctrl_word(wire_ptrs[k], wire_bytes, 0);
    const int pw = sdb_prof_begin(&h->prof, SDB_PK_XWAIT, h->stream);
    CUDA_TRY(h, sdb_launch_wire_wait(ready, n_src, step, h->stream, wire_ptrs, h->xs_hdrs));
    sdb_prof_end(&h->prof, pw, h->stream);
    h->launches += 1;
    int rc = sdb_import_wire_ptrs(h, n_src, wire_ptrs, nullptr);
    if (rc != SDB_OK) return rc;
    CUDA_TRY(h, sdb_launch_wire_set(my_done, step, h->stream));
    h->launches += 1;
    return SDB_OK;
  }
  auto& S = h->xset[h->pf_stream ? (step & 1u) : 0u];
  const bool prefetched = S.pending && S.step == step;
  // everything happens on the device
  { int rc2 = cursor_to_dev(h); if (rc2 != SDB_OK) return rc2; }
  CUDA_TRY(h, sdb_launch_arena_floor_cur(&h->view, h->n_agents, h->cursor_dev, h->stream));
  if (S.pending) { CUDA_TRY(h, cudaStreamWaitEvent(h->stream, S.ready, 0)); S.pending = false; }
  if (prefetched) {
    // 1. the flags were awaited and the batch localized ahead of time (sdb_import_prefetch): place it now
    CUDA_TRY(h, sdb_launch_import_place(S.totals, h->cursor_dev, h->bb_dev, h->arena_grans,
                                        static_cast<uint32_t>(std::min<uint64_t>(h->cfg.list_pool_entries, 0x7FFFFFF0ull)),
                                        h->rx_big_count + 1, h->stream));
    h->launches += 1;
  } else {
    // 1. wait (on the stream, not on the host) until every source's export of this step is complete; 2. localize + place
    int rc = xs_localize(h, S, n_src, wire_ptrs, wire_bytes, step, h->stream, false);
    if (rc != SDB_OK) return rc;
    h->launches += 1;
  }
  int nl = 0;
  const uint32_t n_cap = n_src * h->cfg.max_batch_sends;
  cudaError_t e = cudaSuccess;
  if (S.shared) {            // group sends: headers + one payload per send; the span kernel only serves p2p / broadcast descriptors
    e = sdb_launch_fanout_shared(&h->view, S.descs, n_cap, nullptr, 0, 0, h->cfg.num_shards >= 4 ? 1u : 0u, h->sm_count, h->stream,
                                 &h->prof, h->bb_dev);
    ++nl;
  }
  if (e == cudaSuccess)
    e = sdb_launch_fanout(&h->view, S.descs, n_cap, nullptr, S.tmp_list, 0, 0, pad32(h->cfg.max_payload_bytes), 3,
                          h->sm_count, h->stream, &h->prof, h->bb_dev, S.shared ? 1u : 0u);
  if (e == cudaSuccess) {
    sdb_pull_view pv{h->memb_off_dev, h->memb_grp_dev, h->memb_pos_dev, S.gs_off_src, S.gs_idx_src, n_src,
                     h->cfg.max_groups + 1, h->cfg.max_batch_sends, S.first};
    e = sdb_launch_pull(&h->view, &pv, S.descs, h->n_agents, h->cfg.max_groups, h->gexcl_dev, h->n_excl_groups, 0,
                        h->lstart_dev, h->lcount_dev, 0, 0, h->stream, &h->prof, &nl, h->bb_dev, S.shared ? 1u : 0u);
  }
  // point-to-point / broadcast copies claimed their slots with atomics: sort them into place (the kernels return at
  // once when the import carried none); the group-parallel build leaves ctail to the commit
  if (e == cudaSuccess)
    e = sdb_launch_commit(&h->view, h->n_agents, 0, h->rx_big_list, h->rx_big_count + 1, h->sm_count, h->stream, &h->prof, h->bb_dev);
  h->launches += nl + 3;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("async import launch: ") + cudaGetErrorString(e));
  h->host_stale = true; h->stream_busy = true;
  // 3. tell the exporters that this rank is done reading their buffers of this parity
  CUDA_TRY(h, sdb_launch_wire_set(my_done, step, h->stream));
  h->launches += 1;
  return SDB_OK;
}

int sdb_overflow_log(sdb_handle h, uint32_t cap, uint32_t* agent_out, uint64_t* seq_out, uint32_t* n_out, uint64_t* dropped_out) {
  if (!h || !n_out || (cap && (!agent_out || !seq_out))) return SDB_EINVAL;
  *n_out = 0;
  if (dropped_out) *dropped_out = 0;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  unsigned long long logged = 0;
  CUDA_TRY(h, cudaMemcpyAsync(&logged, &h->ctr->ovf_logged, sizeof(logged), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (dropped_out) *dropped_out = logged;
  if (logged == 0) return SDB_OK;
  const uint32_t n = static_cast<uint32_t>(std::min<unsigned long long>(std::min<unsigned long long>(logged, SDB_OVF_LOG), cap));
  if (n) {
    cudaError_t e = sdb_launch_ovf_resolve(&h->view, n, h->ovf_seq, h->stream);
    if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("overflow log: ") + cudaGetErrorString(e));
    std::vector<uint2> log(n);
    CUDA_TRY(h, cudaMemcpyAsync(log.data(), h->ovf_log, n * sizeof(uint2), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(seq_out, h->ovf_seq, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    for (uint32_t i = 0; i < n; ++i) agent_out[i] = log[i].x;
  }
  CUDA_TRY(h, cudaMemsetAsync(&h->ctr->ovf_logged, 0, sizeof(unsigned long long), h->stream));
  *n_out = n;
  return SDB_OK;
}

int sdb_send_batch(sdb_handle h, uint32_t n, const uint32_t* sender, const uint32_t* receiver, const uint8_t* prio,
                   const uint8_t* type, const uint16_t* len, const uint64_t* payload_off, const uint8_t* payload,
                   uint64_t payload_bytes, const double* timestamp, uint64_t* seq_base_out) {
  SendArrays a{sender, receiver, prio, type, len, payload_off, timestamp};
  return send_common(h, 0, n, a, nullptr, nullptr, payload, payload_bytes, seq_base_out);
}

int sdb_send_group_batch(sdb_handle h, uint32_t n, const uint32_t* sender, const uint32_t* group_idx, const uint8_t* prio,
                         const uint8_t* type, const uint16_t* len, const uint64_t* payload_off, const uint8_t* payload,
                         uint64_t payload_bytes, const double* timestamp, uint64_t* seq_base_out) {
  SendArrays a{sender, group_idx, prio, type, len, payload_off, timestamp};
  return send_common(h, 1, n, a, nullptr, nullptr, payload, payload_bytes, seq_base_out);
}

int sdb_send_list_batch(sdb_handle h, uint32_t n, const uint32_t* sender, const uint64_t* list_off, const uint32_t* list_idx,
                        const uint8_t* prio, const uint8_t* type, const uint16_t* len, const uint64_t* payload_off,
                        const uint8_t* payload, uint64_t payload_bytes, const double* timestamp, uint64_t* seq_base_out) {
  if (n && (!list_off || (list_off[n] && !list_idx))) return fail(h, SDB_EINVAL, "null list arrays");
  SendArrays a{sender, nullptr, prio, type, len, payload_off, timestamp};
  return send_common(h, 2, n, a, list_off, list_idx, payload, payload_bytes, seq_base_out);
}

int sdb_send_mixed_batch(sdb_handle h, uint32_t n, const uint32_t* sender, const uint8_t* kind, const uint32_t* target,
                         uint32_t n_lists, const uint64_t* list_off, const uint32_t* list_idx, const uint8_t* prio,
                         const uint8_t* type, const uint16_t* len, const uint64_t* payload_off, const uint8_t* payload,
                         uint64_t payload_bytes, const double* timestamp, uint64_t* seq_base_out) {
  if (!h) return SDB_EINVAL;
  if (n_lists && (!list_off || (list_off[n_lists] && !list_idx))) return fail(h, SDB_EINVAL, "null list arrays");
  SendArrays a{sender, target, prio, type, len, payload_off, timestamp};
  a.kind = kind; a.n_lists = n_lists;
  return send_common(h, 3, n, a, list_off, list_idx, payload, payload_bytes, seq_base_out);
}

// ---- deduplicated sends (include/swarmdb_b200.h "deduplicated sends", kernels in sdb_dedup.cu)
static void dedup_free(sdb_ctx* h) {
  sdb_ctx::Dedup& D = h->dd;
  for (void* p : D.mem) cudaFree(p);
  if (D.lists_dev) cudaFree(D.lists_dev);
  for (void* p : {static_cast<void*>(D.key_host), static_cast<void*>(D.snd_host), static_cast<void*>(D.verdict_host),
                  static_cast<void*>(D.seq_host), static_cast<void*>(D.ctr_host)})
    if (p) cudaFreeHost(p);
  D = sdb_ctx::Dedup{};
}

static uint64_t pow2_at_least(uint64_t x) {
  uint64_t p = 64;
  while (p < x) p <<= 1;
  return p;
}

int sdb_dedup_reserve(sdb_handle h, uint64_t entries, double window_seconds) {
  if (!h) return SDB_EINVAL;
  if (entries && !(window_seconds > 0.0)) return fail(h, SDB_EINVAL, "sdb_dedup_reserve: the window must be > 0 seconds");
  if (entries > (1ull << 31)) return fail(h, SDB_EINVAL, "sdb_dedup_reserve: more than 2^31 entries");
  { const int rc = ls_stop(h); if (rc != SDB_OK) return rc; }        // cudaFree / cudaMalloc wait for running kernels
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->stream_busy = false;
  dedup_free(h);
  if (!entries) return SDB_OK;
  sdb_ctx::Dedup& D = h->dd;
  const size_t slots = pow2_at_least(2 * entries), B = h->cfg.max_batch_sends, bslots = pow2_at_least(2ull * B);
  std::vector<void*>& m = D.mem;
  sdb_dedup_args& a = D.a;
  unsigned long long* seq_of = nullptr;
  bool ok = lease_alloc(m, &D.tab[0], slots) && lease_alloc(m, &D.tab[1], slots) && lease_alloc(m, &a.key, B) &&
            lease_alloc(m, &D.snd_dev, B) && lease_alloc(m, &a.btab, bslots) && lease_alloc(m, &a.bmin, bslots) &&
            lease_alloc(m, &a.bslot, B) && lease_alloc(m, &a.verdict, B) && lease_alloc(m, &seq_of, B) &&
            lease_alloc(m, &a.ctr, SDB_DD_CTRS);
  ok = ok && cudaHostAlloc(reinterpret_cast<void**>(&D.key_host), B * sizeof(sdb_dedup_key), cudaHostAllocDefault) == cudaSuccess &&
       cudaHostAlloc(reinterpret_cast<void**>(&D.snd_host), B * sizeof(sdb_dedup_send), cudaHostAllocDefault) == cudaSuccess &&
       cudaHostAlloc(reinterpret_cast<void**>(&D.verdict_host), B * sizeof(unsigned long long), cudaHostAllocDefault) == cudaSuccess &&
       cudaHostAlloc(reinterpret_cast<void**>(&D.seq_host), B * sizeof(unsigned long long), cudaHostAllocDefault) == cudaSuccess &&
       cudaHostAlloc(reinterpret_cast<void**>(&D.ctr_host), SDB_DD_CTRS * sizeof(unsigned long long), cudaHostAllocDefault) == cudaSuccess;
  ok = ok && cudaMemsetAsync(D.tab[0], 0, slots * sizeof(sdb_dedup_entry), h->stream) == cudaSuccess &&
       cudaMemsetAsync(a.ctr, 0, SDB_DD_CTRS * sizeof(unsigned long long), h->stream) == cudaSuccess &&
       cudaStreamSynchronize(h->stream) == cudaSuccess;
  if (!ok) {
    dedup_free(h);
    cudaGetLastError();
    return fail(h, SDB_ENOMEM, "sdb_dedup_reserve: allocation failed");
  }
  a.tab = D.tab[0]; a.mask = slots - 1; a.window = window_seconds; a.snd = D.snd_dev; a.bmask = bslots - 1; a.seq_of = seq_of;
  D.entries = entries;
  D.keep.assign(B, 1);
  return SDB_OK;
}

// Entries live at `now` (a counting pass, one synchronisation); the table is not touched
static int dedup_count_live(sdb_ctx* h, double now, uint64_t* live) {
  sdb_ctx::Dedup& D = h->dd;
  cudaError_t e = sdb_launch_dedup_rebuild(&D.a, nullptr, now, h->stream, &h->prof);
  h->launches += 1;
  if (e == cudaSuccess) e = cudaMemcpyAsync(D.ctr_host, D.a.ctr, SDB_DD_CTRS * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("dedup count: ") + cudaGetErrorString(e));
  *live = D.ctr_host[SDB_DD_LIVE];
  return SDB_OK;
}

int sdb_send_mixed_batch_dedup(sdb_handle h, uint32_t n, const uint32_t* sender, const uint8_t* kind, const uint32_t* target,
                               uint32_t n_lists, const uint64_t* list_off, const uint32_t* list_idx, const uint8_t* prio,
                               const uint8_t* type, const uint16_t* len, const uint64_t* payload_off, const uint8_t* payload,
                               uint64_t payload_bytes, const double* timestamp, const sdb_dedup_key* key, uint32_t flags,
                               double now, sdb_dedup_key* key_out, uint64_t* dup_of_out, uint32_t* n_dup_out,
                               uint64_t* seq_base_out) {
  if (!h) return SDB_EINVAL;
  sdb_ctx::Dedup& D = h->dd;
  if (n_dup_out) *n_dup_out = 0;
  if (!D.entries) return fail(h, SDB_EINVAL, "no deduplication table (sdb_dedup_reserve)");
  if (!std::isfinite(now)) return fail(h, SDB_EINVAL, "now must be finite");
  if (flags & ~SDB_DEDUP_CONTENT) return fail(h, SDB_EINVAL, "unknown deduplication flags");
  const bool content = (flags & SDB_DEDUP_CONTENT) != 0;
  if (h->sharded) {
    if (content) return fail(h, SDB_EINVAL, "sharded handle: no content deduplication");
    for (uint32_t i = 0; key && i < n; ++i)
      if (key[i].lo | key[i].hi) return fail(h, SDB_EINVAL, "sharded handle: no deduplication keys");
  }
  if (n == 0 || h->sharded)
    return sdb_send_mixed_batch(h, n, sender, kind, target, n_lists, list_off, list_idx, prio, type, len, payload_off, payload,
                                payload_bytes, timestamp, seq_base_out);
  if (!sender || !len || !target || !kind) return fail(h, SDB_EINVAL, "null array");
  if (n > h->cfg.max_batch_sends) return fail(h, SDB_ECAPACITY, "n exceeds max_batch_sends");
  if (payload_bytes > h->cfg.max_batch_payload) return fail(h, SDB_ECAPACITY, "payload_bytes exceeds max_batch_payload");
  if (payload_bytes && !payload) return fail(h, SDB_EINVAL, "null payload");
  if (n_lists && (!list_off || (list_off[n_lists] && !list_idx))) return fail(h, SDB_EINVAL, "null list arrays");
  // what the content key and the sequence numbers read is checked before anything is staged
  { int rcc = cursor_to_host(h); if (rcc != SDB_OK) return rcc; }
  CUDA_TRY(h, cudaEventSynchronize(h->staging_free));
  uint64_t rec = h->next_seq;
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t k = kind[i], l = len[i];
    const uint64_t off = payload_off ? payload_off[i] : 0;
    if (k > 2) return fail(h, SDB_EINVAL, "kind must be 0, 1 or 2");
    if (l > h->cfg.max_payload_bytes) return fail(h, SDB_EINVAL, "payload longer than max_payload_bytes");
    if ((off & 15u) || off + l > payload_bytes) return fail(h, SDB_EINVAL, "bad payload_off");
    if (sender[i] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "sender index out of range");
    sdb_dedup_send& d = D.snd_host[i];
    d.payload_off = off; d.list_b = 0; d.sender = sender[i]; d.target = target[i]; d.kind = k;
    d.lpt = l | static_cast<uint32_t>(prio ? prio[i] : 1) << 16 | static_cast<uint32_t>(type ? type[i] : 0) << 24;
    D.seq_host[i] = rec;
    if (k == 1) {
      if (target[i] >= h->cfg.max_groups || !h->gdefined[target[i]]) return fail(h, SDB_ENOTFOUND, "unknown group index");
      rec += h->gcount[target[i]];
    } else {
      if (k == 2) {
        if (target[i] >= n_lists || list_off[target[i] + 1] < list_off[target[i]] || list_off[target[i] + 1] > list_off[n_lists])
          return fail(h, SDB_EINVAL, "bad list number or list_off");
        d.list_b = list_off[target[i]]; d.target = static_cast<uint32_t>(list_off[target[i] + 1] - list_off[target[i]]);
      }
      rec += 1;
    }
  }
  if (key) std::memcpy(D.key_host, key, n * sizeof(sdb_dedup_key));
  else std::memset(D.key_host, 0, n * sizeof(sdb_dedup_key));
  CUDA_TRY(h, cudaMemcpyAsync(D.a.key, D.key_host, n * sizeof(sdb_dedup_key), cudaMemcpyHostToDevice, h->stream));
  if (content) {
    const uint64_t nl = n_lists ? list_off[n_lists] : 0;
    if (nl > D.lists_cap) {
      if (D.lists_dev) { CUDA_TRY(h, cudaStreamSynchronize(h->stream)); cudaFree(D.lists_dev); D.lists_dev = nullptr; D.lists_cap = 0; }
      CUDA_TRY(h, dmalloc(&D.lists_dev, nl));
      D.lists_cap = nl;
    }
    if (nl) CUDA_TRY(h, cudaMemcpyAsync(D.lists_dev, list_idx, nl * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(h, cudaMemcpyAsync(D.snd_dev, D.snd_host, n * sizeof(sdb_dedup_send), cudaMemcpyHostToDevice, h->stream));
    if (payload_bytes)
      CUDA_TRY(h, cudaMemcpyAsync(h->scratch.payload_dev, payload, payload_bytes, cudaMemcpyHostToDevice, h->stream));
    D.a.payload = h->scratch.payload_dev; D.a.lists = D.lists_dev;
  }
  int nl = 0;
  cudaError_t e = sdb_launch_dedup_probe(&D.a, n, content ? 1u : 0u, now, h->sm_count, h->stream, &h->prof, &nl);
  h->launches += nl;
  if (e == cudaSuccess) e = cudaMemcpyAsync(D.verdict_host, D.a.verdict, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(D.ctr_host, D.a.ctr, SDB_DD_CTRS * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess && key_out) e = cudaMemcpyAsync(key_out, D.a.key, n * sizeof(sdb_dedup_key), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);       // the one synchronisation: verdicts to the host
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("dedup probe: ") + cudaGetErrorString(e));
  const uint64_t n_new = D.ctr_host[SDB_DD_NEW];
  D.used = D.ctr_host[SDB_DD_USED];
  uint32_t n_dup = 0;
  for (uint32_t i = 0; i < n; ++i) {
    const unsigned long long v = D.verdict_host[i];
    const uint64_t dup_of = (v & SDB_DD_BATCH) ? D.seq_host[v & ~SDB_DD_BATCH] : v;
    D.keep[i] = dup_of == 0;
    n_dup += dup_of != 0;
    if (dup_of_out) dup_of_out[i] = dup_of;
  }
  // the new keys must fit beside the occupied slots; when they do not, the entries that are not live at `now` are
  // dropped by a rebuild, which runs only once the enqueue is accepted (a refused call leaves the table as it was)
  uint64_t live = D.used;
  const bool rebuild = D.used + n_new > D.entries;
  if (rebuild) {
    int rc = dedup_count_live(h, now, &live);
    if (rc != SDB_OK) return rc;
    if (live + n_new > D.entries) return fail(h, SDB_ECAPACITY, "deduplication table full of live entries");
  }
  CUDA_TRY(h, cudaMemcpyAsync(const_cast<unsigned long long*>(D.a.seq_of), D.seq_host, n * sizeof(unsigned long long),
                              cudaMemcpyHostToDevice, h->stream));
  SendArrays a{sender, target, prio, type, len, payload_off, timestamp};
  a.kind = kind; a.n_lists = n_lists; a.keep = D.keep.data();
  uint64_t base = 0;
  int rc = send_common(h, 3, n, a, list_off, list_idx, payload, payload_bytes, &base, content);
  if (rc != SDB_OK) return rc;
  if (h->scratch.n == 0) {             // every send was a duplicate: the batch still takes its sequence numbers
    h->next_seq += h->scratch.total_recs;
    h->dev_stale = true;
  }
  if (rebuild) {                       // stream-ordered before the insert; keeps exactly the `live` entries counted above
    e = sdb_launch_dedup_rebuild(&D.a, D.tab[D.cur ^ 1], now, h->stream, &h->prof);
    h->launches += 1;
    if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("dedup rebuild: ") + cudaGetErrorString(e));
    D.cur ^= 1; D.a.tab = D.tab[D.cur];
    D.expired += D.used - live; D.used = live; D.rebuilds += 1;
  }
  e = sdb_launch_dedup_insert(&D.a, n, now, h->stream, &h->prof);
  h->launches += 1;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("dedup insert: ") + cudaGetErrorString(e));
  h->stream_busy = true;
  D.used += n_new;                     // at most; the next probe reads the exact count
  D.accepted += n_new; D.dups += n_dup; D.last_now = now;
  if (n_dup_out) *n_dup_out = n_dup;
  if (seq_base_out) *seq_base_out = base;
  return SDB_OK;
}

int sdb_dedup_forget(sdb_handle h, uint64_t n, const sdb_dedup_key* key, uint8_t* removed_out) {
  if (!h) return SDB_EINVAL;
  sdb_ctx::Dedup& D = h->dd;
  if (!D.entries) return fail(h, SDB_EINVAL, "no deduplication table (sdb_dedup_reserve)");
  if (n && !key) return fail(h, SDB_EINVAL, "null keys");
  CUDA_TRY(h, cudaEventSynchronize(h->staging_free));
  const uint64_t B = h->cfg.max_batch_sends;
  uint8_t* removed_dev = reinterpret_cast<uint8_t*>(D.a.bslot);       // [B] bytes of the batch scratch
  for (uint64_t c = 0; c < n; c += B) {
    const uint32_t m = static_cast<uint32_t>(std::min(B, n - c));
    std::memcpy(D.key_host, key + c, m * sizeof(sdb_dedup_key));
    cudaError_t e = cudaMemcpyAsync(D.a.key, D.key_host, m * sizeof(sdb_dedup_key), cudaMemcpyHostToDevice, h->stream);
    if (e == cudaSuccess) e = sdb_launch_dedup_forget(&D.a, m, D.last_now, removed_dev, h->stream, &h->prof);
    h->launches += 1;
    if (e == cudaSuccess && removed_out) e = cudaMemcpyAsync(removed_out + c, removed_dev, m, cudaMemcpyDeviceToHost, h->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(D.ctr_host, D.a.ctr, SDB_DD_CTRS * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("dedup forget: ") + cudaGetErrorString(e));
    D.forgotten += D.ctr_host[SDB_DD_FORGOT];
  }
  return SDB_OK;
}

int sdb_dedup_stats(sdb_handle h, sdb_dedup_summary* out) {
  if (!h || !out) return SDB_EINVAL;
  std::memset(out, 0, sizeof(*out));
  sdb_ctx::Dedup& D = h->dd;
  if (!D.entries) return SDB_OK;
  cudaError_t e = sdb_launch_dedup_rebuild(&D.a, nullptr, D.last_now, h->stream, &h->prof);      // count only
  h->launches += 1;
  if (e == cudaSuccess) e = cudaMemcpyAsync(D.ctr_host, D.a.ctr, SDB_DD_CTRS * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("dedup stats: ") + cudaGetErrorString(e));
  D.used = D.ctr_host[SDB_DD_USED];
  out->capacity = D.entries; out->live = D.ctr_host[SDB_DD_LIVE]; out->used = D.used; out->window = D.a.window;
  out->accepted_total = D.accepted; out->duplicate_total = D.dups; out->expired_total = D.expired;
  out->forgotten_total = D.forgotten; out->rebuilds = D.rebuilds;
  return SDB_OK;
}

int sdb_stage_batch(sdb_handle h, uint32_t kind, uint32_t n, const uint32_t* sender, const uint32_t* second,
                    const uint8_t* prio, const uint8_t* type, const uint16_t* len, const uint64_t* payload_off,
                    const uint8_t* payload, uint64_t payload_bytes, const double* timestamp, sdb_staged_t* out) {
  if (!h || !out || kind > 1) return SDB_EINVAL;
  *out = nullptr;
  if (n == 0 || !sender || !second || !len) return fail(h, SDB_EINVAL, "empty or null batch");
  sdb_staged* s = new (std::nothrow) sdb_staged();
  if (!s) return SDB_ENOMEM;
  s->owns = true;
  std::vector<sdb_send_desc> descs(n);
  std::vector<uint32_t> gs(static_cast<size_t>(h->cfg.max_groups) + 1 + n);
  uint32_t n_gs = 0;
  SendArrays a{sender, second, prio, type, len, payload_off, timestamp};
  int rc = build_descs(h, kind, n, a, nullptr, payload_bytes, descs.data(), n, s, gs.data(), &n_gs);
  if (rc != SDB_OK) { delete s; return rc; }
  cudaError_t e = dmalloc(&s->descs_dev, n);
  if (e == cudaSuccess && s->has_pull) {
    const size_t G1 = static_cast<size_t>(h->cfg.max_groups) + 1;
    e = dmalloc(&s->gs_off_dev, G1);
    if (e == cudaSuccess) e = dmalloc(&s->gs_idx_dev, n_gs ? n_gs : 1);
    if (e == cudaSuccess) e = upload(h, s->gs_off_dev, gs.data(), G1 * sizeof(uint32_t));
    if (e == cudaSuccess && n_gs) e = upload(h, s->gs_idx_dev, gs.data() + G1, static_cast<size_t>(n_gs) * sizeof(uint32_t));
  }
  if (e == cudaSuccess) e = dmalloc(&s->payload_dev, payload_bytes + 64);
  if (e == cudaSuccess) e = cudaMemsetAsync(s->payload_dev, 0, payload_bytes + 64, h->stream);
  if (e == cudaSuccess) e = upload(h, s->descs_dev, descs.data(), static_cast<size_t>(n) * sizeof(sdb_send_desc));
  if (e == cudaSuccess && payload_bytes) e = upload(h, s->payload_dev, payload, payload_bytes);
  if (e != cudaSuccess) {
    if (s->descs_dev) cudaFree(s->descs_dev);
    if (s->payload_dev) cudaFree(s->payload_dev);
    if (s->gs_off_dev) cudaFree(s->gs_off_dev);
    if (s->gs_idx_dev) cudaFree(s->gs_idx_dev);
    delete s;
    return fail(h, SDB_ECUDA, std::string("stage: ") + cudaGetErrorString(e));
  }
  *out = s;
  return SDB_OK;
}

int sdb_submit_staged(sdb_handle h, sdb_staged_t s, uint64_t* seq_base_out) {
  if (!h || !s) return SDB_EINVAL;
  return submit(h, s, seq_base_out);
}

int sdb_free_staged(sdb_handle h, sdb_staged_t s) {
  if (!h || !s) return SDB_EINVAL;
  ls_stop(h);
  cudaStreamSynchronize(h->stream);
  if (s->owns) {
    cudaFree(s->descs_dev); cudaFree(s->payload_dev);
    if (s->gs_off_dev) cudaFree(s->gs_off_dev);
    if (s->gs_idx_dev) cudaFree(s->gs_idx_dev);
  }
  delete s;
  return SDB_OK;
}

int sdb_latency_server(sdb_handle h, int enable) {
  if (!h) return SDB_EINVAL;
  h->ls_wanted = enable != 0;
  return enable ? ls_start(h) : ls_stop(h);
}

// unpack the latency paths' output block (u64 total | u64 granules | u32 counts[8] | pad to 64 B | records) into the caller's arrays
static void unpack_small(const uint8_t* block, uint32_t n_agents, uint32_t* count_out, sdb_msg_header* hdr_out, uint8_t* payload_out,
                         uint64_t* total_out, uint64_t* payload_bytes_out) {
  const unsigned long long* t = reinterpret_cast<const unsigned long long*>(block);
  const uint64_t total = t[0];
  if (count_out) std::memcpy(count_out, block + 16, static_cast<size_t>(n_agents) * sizeof(uint32_t));
  const uint8_t* p = block + 64;
  uint64_t poff = 0;
  for (uint64_t r = 0; r < total; ++r) {
    const sdb_msg_header* hd = reinterpret_cast<const sdb_msg_header*>(p);
    hdr_out[r] = *hd;
    const uint32_t pl = pad32(hd->len);
    std::memcpy(payload_out + poff, p + 32, pl);
    poff += pl; p += 32 + pl;
  }
  if (total_out) *total_out = total;
  if (payload_bytes_out) *payload_bytes_out = poff;
}

// agent list of a receive: within the index space, and no agent twice
static int check_recv_agents(sdb_ctx* h, uint32_t n_agents, const uint32_t* agent_idx) {
  if (n_agents > h->cfg.max_agents) return fail(h, SDB_EINVAL, "n_agents > max_agents");
  if (agent_idx) {
    for (uint32_t i = 0; i < n_agents; ++i)
      if (agent_idx[i] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "agent index out of range");
    if (n_agents > 1) {
      // every slot of a listed agent reads the same ring header, so a repeated index would return the same records
      // twice: refused
      const size_t A = h->cfg.max_agents;
      if (h->rank_cnt.size() != A) h->rank_cnt.assign(A, 0u);
      std::vector<uint32_t>& seen = h->rank_cnt;                            // all zero between calls
      uint32_t i = 0;
      for (; i < n_agents && !seen[agent_idx[i]]; ++i) seen[agent_idx[i]] = 1;
      for (uint32_t k = 0; k < i; ++k) seen[agent_idx[k]] = 0;
      if (i < n_agents) return fail(h, SDB_EINVAL, "agent index listed twice");
    }
  }
  return SDB_OK;
}

// Without a list a receive serves every agent below the registration watermark, or, with SDB_RECV_OWNED on a sharded
// handle, the agents this shard owns; returns whether it serves the owned agents.
static bool recv_agents(const sdb_ctx* h, uint32_t flags, const uint32_t* agent_idx, uint32_t* n_agents) {
  const bool owned = (flags & SDB_RECV_OWNED) && !agent_idx && h->sharded && h->owned_dev;
  if (!agent_idx) *n_agents = owned ? h->n_owned : h->n_agents;
  return owned;
}

// Record capacity of one receive call, the same on every path: the device buffers hold this many records of the maximum
// size (what does not fit stays queued: include/swarmdb_b200.h).
static uint64_t recv_rec_cap(const sdb_ctx* h) {
  return std::min<uint64_t>(h->cfg.max_recv_records, h->pay_cap_gran * SDB_GRANULE / pad32(h->cfg.max_payload_bytes));
}
// room of an optional caller buffer: no bound when it is not given
static uint64_t room(const void* buf, uint64_t cap) { return buf ? cap : ~0ull; }
// ... and bounded by the caller's buffers: `rec_room` records in each record array, `payload_room` payload bytes
static int out_rec_cap(sdb_ctx* h, uint64_t rec_room, uint64_t payload_room, uint64_t* rec_cap) {
  *rec_cap = std::min({recv_rec_cap(h), rec_room, payload_room / pad32(h->cfg.max_payload_bytes)});
  if (*rec_cap == 0) return fail(h, SDB_EOUTPUT, "output buffers cannot hold a single maximum-size record");
  return SDB_OK;
}

// The arguments of a receive over the handle's receive scratch and device outputs, after the agent list (if any) is
// uploaded to rx_agent.  Callers override what their call uses differently.
static int recv_args(sdb_ctx* h, uint32_t n_agents, const uint32_t* agent_idx, bool owned, uint32_t max_messages,
                     uint32_t flags, uint64_t rec_cap, sdb_recv_args* out) {
  if (agent_idx) {
    CUDA_TRY(h, cudaMemcpyAsync(h->rx_agent, agent_idx, static_cast<size_t>(n_agents) * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  }
  sdb_recv_args r{};
  r.agent_idx = agent_idx ? h->rx_agent : (owned ? h->owned_dev : nullptr); r.n = n_agents; r.max_messages = max_messages;
  r.flags = flags;
  r.cnt = h->rx_cnt; r.rec_local = h->rx_rec_local; r.rec_tops = h->rx_rec_tops;
  r.rec_off = h->rx_rec_off; r.plan = h->rx_plan; r.lb = h->rx_lb;
  r.plan_tops = h->rx_plan_tops; r.totals = h->rx_totals; r.big_list = h->rx_big_list; r.big_count = h->rx_big_count;
  r.count_out = h->rx_count; r.hdr_out = h->rx_hdr; r.payload_out = h->rx_payload;
  r.rec_cap = rec_cap;
  *out = r;
  return SDB_OK;
}

// Full-format results to the caller: totals and counts, one synchronisation, then headers and payload and, if any was
// asked for, a second one.
static int copy_full(sdb_ctx* h, uint32_t n_agents, uint32_t* count_out, sdb_msg_header* hdr_out, uint8_t* payload_out,
                     uint64_t* total_out, uint64_t* payload_bytes_out) {
  CUDA_TRY(h, cudaMemcpyAsync(h->totals_host, h->rx_totals, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  if (count_out)
    CUDA_TRY(h, cudaMemcpyAsync(count_out, h->rx_count, static_cast<size_t>(n_agents) * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->stream_busy = false;
  const uint64_t total = h->totals_host[TOT_RECORDS], pbytes = h->totals_host[TOT_GRANULES] * SDB_GRANULE;
  if (total_out) *total_out = total;
  if (payload_bytes_out) *payload_bytes_out = pbytes;
  if (total) {
    if (hdr_out) CUDA_TRY(h, cudaMemcpyAsync(hdr_out, h->rx_hdr, total * sizeof(sdb_msg_header), cudaMemcpyDeviceToHost, h->stream));
    if (payload_out && pbytes) CUDA_TRY(h, cudaMemcpyAsync(payload_out, h->rx_payload, pbytes, cudaMemcpyDeviceToHost, h->stream));
    if (hdr_out || payload_out) CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  return SDB_OK;
}

// Compact-format results to the caller: totals, the compact totals and counts, one synchronisation, then entries, sends
// and payload and, if any was asked for, a second one.
static int copy_compact(sdb_ctx* h, uint32_t n_agents, uint32_t* count_out, sdb_recv_entry* entry_out, sdb_recv_send* send_out,
                        uint8_t* payload_out, uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out) {
  CUDA_TRY(h, cudaMemcpyAsync(h->totals_host, h->rx_totals, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(h->totals_host + TOT_CX_SENDS, h->cx.totals, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  if (count_out)
    CUDA_TRY(h, cudaMemcpyAsync(count_out, h->rx_count, static_cast<size_t>(n_agents) * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->stream_busy = false;
  const uint64_t total = h->totals_host[TOT_RECORDS], n_sends = h->totals_host[TOT_CX_SENDS];
  const uint64_t pbytes = h->totals_host[TOT_CX_GRANULES] * SDB_GRANULE;
  if (total_out) *total_out = total;
  if (n_sends_out) *n_sends_out = n_sends;
  if (payload_bytes_out) *payload_bytes_out = pbytes;
  if (total) {
    if (entry_out) CUDA_TRY(h, cudaMemcpyAsync(entry_out, h->cx.entry_out, total * sizeof(sdb_recv_entry), cudaMemcpyDeviceToHost, h->stream));
    if (send_out) CUDA_TRY(h, cudaMemcpyAsync(send_out, h->cx.send_out, n_sends * sizeof(sdb_recv_send), cudaMemcpyDeviceToHost, h->stream));
    if (payload_out && pbytes) CUDA_TRY(h, cudaMemcpyAsync(payload_out, h->cx.payload_out, pbytes, cudaMemcpyDeviceToHost, h->stream));
    if (entry_out || send_out || payload_out) CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  return SDB_OK;
}

int sdb_receive_batch(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages, uint32_t flags,
                      uint32_t* count_out, sdb_msg_header* hdr_out, uint64_t hdr_cap, uint8_t* payload_out,
                      uint64_t payload_cap, uint64_t* total_out, uint64_t* payload_bytes_out) {
  if (!h) return SDB_EINVAL;
  if (total_out) *total_out = 0;
  if (payload_bytes_out) *payload_bytes_out = 0;
  const bool owned = recv_agents(h, flags, agent_idx, &n_agents);
  if (n_agents == 0 || max_messages == 0) return SDB_OK;
  { const int rc = check_recv_agents(h, n_agents, agent_idx); if (rc != SDB_OK) return rc; }
  uint64_t rec_cap = 0;
  { const int rc = out_rec_cap(h, room(hdr_out, hdr_cap), room(payload_out, payload_cap), &rec_cap); if (rc != SDB_OK) return rc; }
  // ---- latency path: few agents, host outputs -> one launch, one D2H, one sync
  if (agent_idx && n_agents <= 8 && hdr_out && payload_out &&
      static_cast<uint64_t>(n_agents) * max_messages <= 1024) {
    rec_cap = std::min<uint64_t>(rec_cap, 1024);
    h->last_rx_valid = false; h->last_rx_compact = false;
    bool served = false;
    if (h->ls_wanted && n_agents == 1) {
      { int rcl = ls_start(h); if (rcl != SDB_OK) return rcl; }
      const uint64_t want = std::min<uint64_t>(max_messages, rec_cap);
      served = 64ull + want * (32 + pad32(h->cfg.max_payload_bytes)) <= h->ls_out_cap;   // the whole answer must fit the pinned block
    }
    if (served) {
      // ---- the persistent server: post the request in mapped pinned memory, read the answer from pinned memory
      if (h->stream_busy) { CUDA_TRY(h, cudaStreamSynchronize(h->stream)); h->stream_busy = false; }   // earlier sends are complete and visible
      sdb_ls_mailbox* mb = h->ls_mbox;
      mb->agent = agent_idx[0]; mb->max_messages = static_cast<uint32_t>(std::min<uint64_t>(max_messages, rec_cap));
      mb->flags = flags & 0x7FFFFFFFu;
      const uint32_t seq = ++h->ls_seq;
      __atomic_store_n(&mb->req_seq, seq, __ATOMIC_RELEASE);
      uint64_t spins = 0;
      while (__atomic_load_n(&mb->done_seq, __ATOMIC_ACQUIRE) != seq) {
        if (++spins > (1ull << 33)) return fail(h, SDB_ECUDA, "latency server did not answer");
        __builtin_ia32_pause();
      }
      unpack_small(h->ls_out, 1, count_out, hdr_out, payload_out, total_out, payload_bytes_out);
      return SDB_OK;
    }
    cudaError_t e = sdb_launch_receive_small(&h->view, agent_idx, n_agents, max_messages, flags, static_cast<uint32_t>(rec_cap),
                                             h->rx_plan, h->rx_small, h->stream, &h->prof);
    h->launches += 1;
    if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("receive launch: ") + cudaGetErrorString(e));
    const uint64_t window = std::min<uint64_t>(h->small_bytes, 16384);
    CUDA_TRY(h, cudaMemcpyAsync(h->small_host, h->rx_small, window, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    const unsigned long long* t = reinterpret_cast<const unsigned long long*>(h->small_host);
    const uint64_t total = t[0], bytes = 64 + t[1] * SDB_GRANULE;
    if (bytes > window) {
      CUDA_TRY(h, cudaMemcpyAsync(h->small_host + window, h->rx_small + window, bytes - window, cudaMemcpyDeviceToHost, h->stream));
      CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    }
    unpack_small(h->small_host, n_agents, count_out, hdr_out, payload_out, total_out, payload_bytes_out);
    (void)total;
    return SDB_OK;
  }
  sdb_recv_args r{};
  { const int rc = recv_args(h, n_agents, agent_idx, owned, max_messages, flags & (SDB_RECV_PRIORITY | SDB_RECV_PEEK), rec_cap, &r);
    if (rc != SDB_OK) return rc; }
  const bool async = (flags & SDB_RECV_ASYNC) != 0;
  if (async && (count_out || hdr_out || payload_out)) return fail(h, SDB_EINVAL, "SDB_RECV_ASYNC takes no host output buffers");
  int nl = 0;
  cudaError_t e = sdb_launch_receive(&h->view, &r, h->stream, &nl, &h->prof, h->sm_count, 32u + pad32(h->cfg.max_payload_bytes),
                                     nullptr, nullptr, 0ull);
  h->launches += nl;
  if (!(r.flags & SDB_RECV_PRIORITY)) r.plan_tops = nullptr;       // single-pass path: plan offsets are absolute
  h->last_rx = r; h->last_rx_valid = (e == cudaSuccess); h->last_rx_compact = false;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("receive launch: ") + cudaGetErrorString(e));
  if (async) { h->stream_busy = true; return SDB_OK; }   // the caller consumes on the device (stream order) or asks sdb_last_receive_totals later
  return copy_full(h, n_agents, count_out, hdr_out, payload_out, total_out, payload_bytes_out);
}

// verdict bitmap of filtered receives and superseding, [max_agents][where_stride] words, and the keyword buffer; allocated
// once, on first use
static uint32_t where_stride(const sdb_ctx* h) { return (h->cfg.ring_slots + 31) / 32; }
static int where_ensure(sdb_ctx* h) {
  if (h->where_bits) return SDB_OK;
  return dmalloc_set(h, {{&h->where_bits, static_cast<size_t>(h->cfg.max_agents) * where_stride(h)}, {&h->where_kw, SDB_FILTER_MAX_KEYWORD}},
                     "filtered receive: device allocation failed");
}

// compact receive scratch and outputs, sized for max_recv_records; allocated once, on the first compact call
static int compact_ensure(sdb_ctx* h) {
  sdb_compact_args& c = h->cx;
  if (c.table) return SDB_OK;
  const size_t R = h->cfg.max_recv_records, tiles = sdb_scan_tops_len(R);
  uint32_t tbits = 10;
  while ((1ull << tbits) < 2 * R) ++tbits;
  return dmalloc_set(h, {{&c.rec_slot, R}, {&c.head, R}, {&c.head_local, R}, {&c.head_tops, tiles}, {&c.gran, R},
                         {&c.gran_local, R}, {&c.gran_tops, tiles}, {&c.totals, 2}, {&c.entry_out, R}, {&c.send_out, R},
                         {&c.payload_out, h->pay_cap_gran * SDB_GRANULE},
                         {&c.table, static_cast<size_t>(1) << tbits}},          // last: marks the set complete
                     "compact receive: device allocation failed");
}

int sdb_receive_compact(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages, uint32_t flags,
                        uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
                        sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                        uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out) {
  if (!h) return SDB_EINVAL;
  if (total_out) *total_out = 0;
  if (n_sends_out) *n_sends_out = 0;
  if (payload_bytes_out) *payload_bytes_out = 0;
  if (flags & SDB_RECV_ASYNC) return fail(h, SDB_EINVAL, "sdb_receive_compact returns host results: SDB_RECV_ASYNC is not accepted");
  const bool owned = recv_agents(h, flags, agent_idx, &n_agents);
  if (n_agents == 0 || max_messages == 0) return SDB_OK;
  { const int rc = check_recv_agents(h, n_agents, agent_idx); if (rc != SDB_OK) return rc; }
  // sdb_receive_batch's capacity: rec_cap unshared records of the maximum size fit every buffer
  uint64_t rec_cap = 0;
  { const int rc = out_rec_cap(h, std::min(room(entry_out, entry_cap), room(send_out, send_cap)), room(payload_out, payload_cap), &rec_cap);
    if (rc != SDB_OK) return rc; }
  { const int rc = compact_ensure(h); if (rc != SDB_OK) return rc; }
  sdb_recv_args r{};
  { const int rc = recv_args(h, n_agents, agent_idx, owned, max_messages, flags & (SDB_RECV_PRIORITY | SDB_RECV_PEEK), rec_cap, &r);
    if (rc != SDB_OK) return rc; }
  int nl = 0;
  cudaError_t e = sdb_launch_receive(&h->view, &r, h->stream, &nl, &h->prof, h->sm_count, 32u + pad32(h->cfg.max_payload_bytes),
                                     &h->cx, nullptr, 0ull);
  h->launches += nl;
  h->last_rx_valid = false; h->last_rx_compact = true;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("compact receive launch: ") + cudaGetErrorString(e));
  return copy_compact(h, n_agents, count_out, entry_out, send_out, payload_out, total_out, n_sends_out, payload_bytes_out);
}

// Capacity of a byte-budget receive (include/swarmdb_b200.h: sdb_receive_budget), exact in bytes: `rec_room` records and
// the payload buffer's granules, which must hold one record of the maximum size.  budget = {per-agent limit, call
// capacity} in payload granules.
static int budget_caps(sdb_ctx* h, uint64_t rec_room, const void* payload_out, uint64_t payload_cap, uint64_t max_agent_bytes,
                       uint64_t* rec_cap, uint2* budget) {
  const uint64_t P = pad32(h->cfg.max_payload_bytes);
  if (payload_out && payload_cap < P) return fail(h, SDB_EINVAL, "payload_cap below pad32(max_payload_bytes): a call could not make progress");
  const uint64_t gran_cap = std::min<uint64_t>(h->pay_cap_gran, room(payload_out, payload_cap) / SDB_GRANULE);
  *rec_cap = std::min<uint64_t>(h->cfg.max_recv_records, rec_room);
  if (*rec_cap == 0 || gran_cap * SDB_GRANULE < P) return fail(h, SDB_EOUTPUT, "output buffers cannot hold a single maximum-size record");
  const uint64_t agent_gran = max_agent_bytes ? max_agent_bytes / SDB_GRANULE : ~0ull;     // sum(pad32(len)) <= max_agent_bytes
  *budget = make_uint2(static_cast<uint32_t>(std::min<uint64_t>(agent_gran, 0xFFFFFFFFull)), static_cast<uint32_t>(gran_cap));
  return SDB_OK;
}

// sdb_receive_budget and sdb_receive_tokens (max_agent_tokens 0: the budget call); `name` and `what` name the call in
// error messages
static int receive_budget_full(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                               uint64_t max_agent_bytes, uint64_t max_agent_tokens, uint32_t flags, uint32_t* count_out,
                               sdb_msg_header* hdr_out, uint64_t hdr_cap, uint8_t* payload_out, uint64_t payload_cap,
                               uint64_t* total_out, uint64_t* payload_bytes_out, const char* name, const char* what) {
  if (!h) return SDB_EINVAL;
  if (total_out) *total_out = 0;
  if (payload_bytes_out) *payload_bytes_out = 0;
  if (flags & SDB_RECV_ASYNC) return fail(h, SDB_EINVAL, std::string(name) + " returns host results: SDB_RECV_ASYNC is not accepted");
  uint64_t rec_cap = 0;
  uint2 budget;
  { const int rc = budget_caps(h, room(hdr_out, hdr_cap), payload_out, payload_cap, max_agent_bytes, &rec_cap, &budget);
    if (rc != SDB_OK) return rc; }
  const bool owned = recv_agents(h, flags, agent_idx, &n_agents);
  if (n_agents == 0 || max_messages == 0) return SDB_OK;
  { const int rc = check_recv_agents(h, n_agents, agent_idx); if (rc != SDB_OK) return rc; }
  sdb_recv_args r{};
  { const int rc = recv_args(h, n_agents, agent_idx, owned, max_messages, flags & (SDB_RECV_PRIORITY | SDB_RECV_PEEK), rec_cap, &r);
    if (rc != SDB_OK) return rc; }
  int nl = 0;
  cudaError_t e = sdb_launch_receive(&h->view, &r, h->stream, &nl, &h->prof, h->sm_count, 32u + pad32(h->cfg.max_payload_bytes),
                                     nullptr, &budget, max_agent_tokens);
  h->launches += nl;
  r.plan_tops = nullptr;                                        // single-pass plan in both orders: offsets are absolute
  h->last_rx = r; h->last_rx_valid = (e == cudaSuccess); h->last_rx_compact = false;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string(what) + " launch: " + cudaGetErrorString(e));
  return copy_full(h, n_agents, count_out, hdr_out, payload_out, total_out, payload_bytes_out);
}

int sdb_receive_budget(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages, uint64_t max_agent_bytes,
                       uint32_t flags, uint32_t* count_out, sdb_msg_header* hdr_out, uint64_t hdr_cap, uint8_t* payload_out,
                       uint64_t payload_cap, uint64_t* total_out, uint64_t* payload_bytes_out) {
  return receive_budget_full(h, n_agents, agent_idx, max_messages, max_agent_bytes, 0, flags, count_out, hdr_out, hdr_cap,
                             payload_out, payload_cap, total_out, payload_bytes_out, "sdb_receive_budget", "budget receive");
}

int sdb_receive_tokens(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages, uint64_t max_agent_bytes,
                       uint64_t max_agent_tokens, uint32_t flags, uint32_t* count_out, sdb_msg_header* hdr_out, uint64_t hdr_cap,
                       uint8_t* payload_out, uint64_t payload_cap, uint64_t* total_out, uint64_t* payload_bytes_out) {
  return receive_budget_full(h, n_agents, agent_idx, max_messages, max_agent_bytes, max_agent_tokens, flags, count_out, hdr_out,
                             hdr_cap, payload_out, payload_cap, total_out, payload_bytes_out, "sdb_receive_tokens", "token receive");
}

// sdb_receive_compact_budget and sdb_receive_compact_tokens (max_agent_tokens 0: the budget call)
static int receive_budget_compact(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                                  uint64_t max_agent_bytes, uint64_t max_agent_tokens, uint32_t flags, uint32_t* count_out,
                                  sdb_recv_entry* entry_out, uint64_t entry_cap, sdb_recv_send* send_out, uint64_t send_cap,
                                  uint8_t* payload_out, uint64_t payload_cap, uint64_t* total_out, uint64_t* n_sends_out,
                                  uint64_t* payload_bytes_out, const char* name, const char* what) {
  if (!h) return SDB_EINVAL;
  if (total_out) *total_out = 0;
  if (n_sends_out) *n_sends_out = 0;
  if (payload_bytes_out) *payload_bytes_out = 0;
  if (flags & SDB_RECV_ASYNC) return fail(h, SDB_EINVAL, std::string(name) + " returns host results: SDB_RECV_ASYNC is not accepted");
  // bytes are counted per record, so the compact payload (one copy per distinct image) never exceeds the count
  uint64_t rec_cap = 0;
  uint2 budget;
  { const int rc = budget_caps(h, std::min(room(entry_out, entry_cap), room(send_out, send_cap)), payload_out, payload_cap,
                               max_agent_bytes, &rec_cap, &budget);
    if (rc != SDB_OK) return rc; }
  const bool owned = recv_agents(h, flags, agent_idx, &n_agents);
  if (n_agents == 0 || max_messages == 0) return SDB_OK;
  { const int rc = check_recv_agents(h, n_agents, agent_idx); if (rc != SDB_OK) return rc; }
  { const int rc = compact_ensure(h); if (rc != SDB_OK) return rc; }
  sdb_recv_args r{};
  { const int rc = recv_args(h, n_agents, agent_idx, owned, max_messages, flags & (SDB_RECV_PRIORITY | SDB_RECV_PEEK), rec_cap, &r);
    if (rc != SDB_OK) return rc; }
  int nl = 0;
  cudaError_t e = sdb_launch_receive(&h->view, &r, h->stream, &nl, &h->prof, h->sm_count, 32u + pad32(h->cfg.max_payload_bytes),
                                     &h->cx, &budget, max_agent_tokens);
  h->launches += nl;
  h->last_rx_valid = false; h->last_rx_compact = true;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string(what) + " launch: " + cudaGetErrorString(e));
  return copy_compact(h, n_agents, count_out, entry_out, send_out, payload_out, total_out, n_sends_out, payload_bytes_out);
}

int sdb_receive_compact_budget(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                               uint64_t max_agent_bytes, uint32_t flags, uint32_t* count_out, sdb_recv_entry* entry_out,
                               uint64_t entry_cap, sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out,
                               uint64_t payload_cap, uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out) {
  return receive_budget_compact(h, n_agents, agent_idx, max_messages, max_agent_bytes, 0, flags, count_out, entry_out, entry_cap,
                                send_out, send_cap, payload_out, payload_cap, total_out, n_sends_out, payload_bytes_out,
                                "sdb_receive_compact_budget", "compact budget receive");
}

int sdb_receive_compact_tokens(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                               uint64_t max_agent_bytes, uint64_t max_agent_tokens, uint32_t flags, uint32_t* count_out,
                               sdb_recv_entry* entry_out, uint64_t entry_cap, sdb_recv_send* send_out, uint64_t send_cap,
                               uint8_t* payload_out, uint64_t payload_cap, uint64_t* total_out, uint64_t* n_sends_out,
                               uint64_t* payload_bytes_out) {
  return receive_budget_compact(h, n_agents, agent_idx, max_messages, max_agent_bytes, max_agent_tokens, flags, count_out,
                                entry_out, entry_cap, send_out, send_cap, payload_out, payload_cap, total_out, n_sends_out,
                                payload_bytes_out, "sdb_receive_compact_tokens", "compact token receive");
}

int sdb_pending_tokens(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint64_t* tokens_out) {
  if (!h || (n_agents && !tokens_out)) return SDB_EINVAL;
  if (n_agents == 0) return SDB_OK;
  if (n_agents > h->cfg.max_agents) return fail(h, SDB_EINVAL, "n_agents > max_agents");
  if (agent_idx)
    for (uint32_t i = 0; i < n_agents; ++i)
      if (agent_idx[i] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "agent index out of range");
  sdb_recv_args r{};
  { const int rc = recv_args(h, n_agents, agent_idx, false, 0xFFFFFFFFu, 0, 0, &r); if (rc != SDB_OK) return rc; }
  unsigned long long* sums = nullptr;
  CUDA_TRY(h, cudaMallocAsync(reinterpret_cast<void**>(&sums), static_cast<size_t>(n_agents) * sizeof(unsigned long long), h->stream));
  int nl = 0;
  cudaError_t e = sdb_launch_token_take(&h->view, &r, ~0ull, sums, h->stream, &nl, &h->prof, h->sm_count);
  h->launches += nl;
  if (e == cudaSuccess) e = cudaMemcpyAsync(tokens_out, sums, static_cast<size_t>(n_agents) * sizeof(uint64_t), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaFreeAsync(sums, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("pending tokens: ") + cudaGetErrorString(e));
  h->stream_busy = false;
  return SDB_OK;
}

// The first step of sdb_supersede: count the flagged pending records of r's agents (one synchronisation) and, when there
// are any, size the key table (a power of two >= 2 x the records) and the candidate array, zero the table and fill *s.
// s->n_cand == 0: nothing can be superseded.  Scratch that cannot be allocated refuses the call before anything retires.
static int supersede_prepare(sdb_ctx* h, const sdb_recv_args& r, sdb_ss_args* s, int* nl) {
  *s = sdb_ss_args{};
  const cudaError_t e = sdb_launch_supersede(&h->view, &r, s, nullptr, h->stream, nl, &h->prof, h->sm_count);
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("supersede count launch: ") + cudaGetErrorString(e));
  CUDA_TRY(h, cudaMemcpyAsync(h->totals_host, h->rx_totals, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->stream_busy = false;
  const uint64_t C = h->totals_host[TOT_RECORDS];
  if (C == 0) return SDB_OK;
  if (C > (1ull << 30)) return fail(h, SDB_ECAPACITY, "sdb_supersede: more than 2^30 flagged pending records");
  uint64_t slots = 1024;
  while (slots < 2 * C) slots <<= 1;
  if (where_ensure(h) != SDB_OK) return fail(h, SDB_ECAPACITY, "sdb_supersede: verdict bitmap allocation failed");
  if (slots > h->ss_slots || C > h->ss_cap) {
    const uint64_t cap = std::max(C, h->ss_cap), sl = std::max(slots, h->ss_slots);
    { const int rc = ls_stop(h); if (rc != SDB_OK) return rc; }   // cudaFree waits for the kernels on the device
    for (void* p : {static_cast<void*>(h->ss_tab), static_cast<void*>(h->ss_cand)}) if (p) cudaFree(p);
    h->ss_tab = nullptr; h->ss_cand = nullptr; h->ss_slots = h->ss_cap = 0;
    if (dmalloc_set(h, {{&h->ss_tab, sl}, {&h->ss_cand, cap}}, "sdb_supersede: scratch allocation failed") != SDB_OK)
      return fail(h, SDB_ECAPACITY, "sdb_supersede: no device memory for the key table of " + std::to_string(C) + " records");
    h->ss_slots = sl; h->ss_cap = cap;
  }
  CUDA_TRY(h, cudaMemsetAsync(h->ss_tab, 0, slots * sizeof(sdb_ss_slot), h->stream));
  s->tab = h->ss_tab; s->mask = static_cast<uint32_t>(slots - 1);
  s->cand = h->ss_cand; s->n_cand = static_cast<uint32_t>(C);
  s->bits = h->where_bits; s->stride = where_stride(h);
  return SDB_OK;
}

// The body of sdb_expire, sdb_trim and sdb_supersede: `flags` were checked by the caller; trim == nullptr without
// `supersede` is an expiry.  Archive mode takes sdb_receive_compact's capacity rule and copy-out; drop mode returns the
// count and the per-agent counts.
static int retire_call(sdb_ctx* h, uint32_t n_agents, const uint32_t* agent_idx, double older_than, const uint2* trim,
                       bool supersede, uint32_t flags, uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
                       sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                       uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out) {
  const bool owned = recv_agents(h, flags, agent_idx, &n_agents);
  const bool archive = entry_out || send_out || payload_out;
  uint64_t rec_cap = 0;
  if (archive) {      // sdb_receive_compact's capacity rule
    const int rc = out_rec_cap(h, std::min(room(entry_out, entry_cap), room(send_out, send_cap)), room(payload_out, payload_cap), &rec_cap);
    if (rc != SDB_OK) return rc;
  }
  if (n_agents == 0) return SDB_OK;
  { const int rc = check_recv_agents(h, n_agents, agent_idx); if (rc != SDB_OK) return rc; }
  if (archive) { const int rc = compact_ensure(h); if (rc != SDB_OK) return rc; }
  sdb_recv_args r{};
  { const int rc = recv_args(h, n_agents, agent_idx, owned, 0, flags & (SDB_RECV_PEEK | SDB_RECV_PRIORITY), rec_cap, &r);
    if (rc != SDB_OK) return rc; }
  if (!archive && !count_out) r.count_out = nullptr;           // nobody reads the counts
  int nl = 0;
  cudaError_t e;
  if (supersede) {
    sdb_ss_args s;
    const int rc = supersede_prepare(h, r, &s, &nl);
    h->last_rx_valid = false; h->last_rx_compact = false;
    if (rc != SDB_OK || s.n_cand == 0) {                        // refused, or no flagged record: nothing more to launch
      h->launches += nl;
      if (rc == SDB_OK && count_out) std::fill(count_out, count_out + n_agents, 0u);
      return rc;
    }
    e = sdb_launch_supersede(&h->view, &r, &s, archive ? &h->cx : nullptr, h->stream, &nl, &h->prof, h->sm_count);
  } else {
    e = sdb_launch_expire(&h->view, &r, older_than, (flags & SDB_EXPIRE_ALL) ? 1u : 0u, trim, archive ? &h->cx : nullptr,
                          h->stream, &nl, &h->prof, h->sm_count);
  }
  h->launches += nl;
  h->last_rx_valid = false; h->last_rx_compact = false;       // the receive scratch was reused: nothing left to fold
  if (e != cudaSuccess)
    return fail(h, SDB_ECUDA, std::string(supersede ? "supersede" : trim ? "trim" : "expire") + " launch: " + cudaGetErrorString(e));
  if (archive) return copy_compact(h, n_agents, count_out, entry_out, send_out, payload_out, total_out, n_sends_out, payload_bytes_out);
  // drop mode: the number of records retired and the counts
  CUDA_TRY(h, cudaMemcpyAsync(h->totals_host, h->rx_totals, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  if (count_out)
    CUDA_TRY(h, cudaMemcpyAsync(count_out, h->rx_count, static_cast<size_t>(n_agents) * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->stream_busy = false;
  if (total_out) *total_out = h->totals_host[TOT_RECORDS];
  return SDB_OK;
}

int sdb_expire(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, double older_than, uint32_t flags,
               uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
               sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
               uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out) {
  if (!h) return SDB_EINVAL;
  if (total_out) *total_out = 0;
  if (n_sends_out) *n_sends_out = 0;
  if (payload_bytes_out) *payload_bytes_out = 0;
  if (flags & ~(SDB_RECV_PEEK | SDB_RECV_OWNED | SDB_EXPIRE_ALL))
    return fail(h, SDB_EINVAL, "sdb_expire accepts SDB_RECV_PEEK, SDB_RECV_OWNED and SDB_EXPIRE_ALL only");
  return retire_call(h, n_agents, agent_idx, older_than, nullptr, false, flags, count_out, entry_out, entry_cap, send_out, send_cap,
                     payload_out, payload_cap, total_out, n_sends_out, payload_bytes_out);
}

int sdb_trim(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_records, uint64_t max_agent_bytes,
             uint32_t flags, uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
             sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
             uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out) {
  if (!h) return SDB_EINVAL;
  if (total_out) *total_out = 0;
  if (n_sends_out) *n_sends_out = 0;
  if (payload_bytes_out) *payload_bytes_out = 0;
  if (flags & ~(SDB_RECV_PEEK | SDB_RECV_OWNED | SDB_RECV_PRIORITY))
    return fail(h, SDB_EINVAL, "sdb_trim accepts SDB_RECV_PEEK, SDB_RECV_OWNED and SDB_RECV_PRIORITY only");
  if (max_records == 0 && max_agent_bytes == 0)
    return fail(h, SDB_EINVAL, "sdb_trim: max_records and max_agent_bytes are both 0 (SDB_EXPIRE_ALL purges a queue)");
  // limits in records and payload granules, ~0 for none (a queue's granules are counted in 32 bits, as in sdb_agent_loads)
  const uint2 lim = make_uint2(max_records ? max_records : 0xFFFFFFFFu,
                               max_agent_bytes ? static_cast<uint32_t>(std::min<uint64_t>(max_agent_bytes / SDB_GRANULE, 0xFFFFFFFEull))
                                               : 0xFFFFFFFFu);
  return retire_call(h, n_agents, agent_idx, 0.0, &lim, false, flags, count_out, entry_out, entry_cap, send_out, send_cap,
                     payload_out, payload_cap, total_out, n_sends_out, payload_bytes_out);
}

int sdb_supersede(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t flags,
                  uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
                  sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                  uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out) {
  if (!h) return SDB_EINVAL;
  if (total_out) *total_out = 0;
  if (n_sends_out) *n_sends_out = 0;
  if (payload_bytes_out) *payload_bytes_out = 0;
  if (flags & ~(SDB_RECV_PEEK | SDB_RECV_OWNED))
    return fail(h, SDB_EINVAL, "sdb_supersede accepts SDB_RECV_PEEK and SDB_RECV_OWNED only");
  return retire_call(h, n_agents, agent_idx, 0.0, nullptr, true, flags, count_out, entry_out, entry_cap, send_out, send_cap,
                     payload_out, payload_cap, total_out, n_sends_out, payload_bytes_out);
}

static int restore_ensure(sdb_ctx* h);
static int restore_staged(sdb_ctx* h, uint32_t n_agents, uint64_t n_entries, uint64_t n_sends, uint64_t payload_bytes, bool owned,
                          uint64_t* records_out);

int sdb_restore_compact(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, const uint32_t* count,
                        const sdb_recv_entry* entries, uint64_t n_entries, const sdb_recv_send* sends, uint64_t n_sends,
                        const uint8_t* payload, uint64_t payload_bytes, uint32_t flags, uint64_t* restored_out,
                        uint64_t* seq_end_out) {
  if (!h) return SDB_EINVAL;
  if (restored_out) *restored_out = 0;
  { int rcc = cursor_to_host(h); if (rcc != SDB_OK) return rcc; }      // a host-placed write, like a send
  if (seq_end_out) *seq_end_out = h->next_seq;
  if (flags & ~SDB_RECV_OWNED) return fail(h, SDB_EINVAL, "sdb_restore_compact accepts SDB_RECV_OWNED only");
  if (n_agents && (!agent_idx || !count)) return fail(h, SDB_EINVAL, "sdb_restore_compact: agent_idx and count are required");
  if ((n_entries && !entries) || (n_sends && !sends) || (payload_bytes && !payload))
    return fail(h, SDB_EINVAL, "sdb_restore_compact: null input array");
  { const int rc = check_recv_agents(h, n_agents, agent_idx); if (rc != SDB_OK) return rc; }
  uint64_t sum = 0;
  for (uint32_t i = 0; i < n_agents; ++i) sum += count[i];
  if (sum != n_entries) return fail(h, SDB_EINVAL, "sdb_restore_compact: sum(count) != n_entries");
  // one compact receive's capacity: the input is staged in its device buffers
  const uint64_t rec_cap = recv_rec_cap(h);
  if (n_entries > rec_cap || n_sends > rec_cap || payload_bytes > rec_cap * pad32(h->cfg.max_payload_bytes))
    return fail(h, SDB_ECAPACITY, "sdb_restore_compact: input larger than one compact receive's capacity");
  if (n_agents == 0) return SDB_OK;
  { const int rc = restore_ensure(h); if (rc != SDB_OK) return rc; }
  const size_t A = h->cfg.max_agents;
  std::vector<uint32_t> first(n_agents);
  { uint32_t run = 0; for (uint32_t i = 0; i < n_agents; ++i) { first[i] = run; run += count[i]; } }
  uint32_t* t = h->rs_agent;
  const size_t n = n_agents;
  CUDA_TRY(h, cudaMemcpyAsync(t, agent_idx, n * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(t + A, count, n * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(t + 2 * A, first.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  sdb_compact_args& c = h->cx;
  if (n_entries) CUDA_TRY(h, cudaMemcpyAsync(c.entry_out, entries, n_entries * sizeof(sdb_recv_entry), cudaMemcpyHostToDevice, h->stream));
  if (n_sends) CUDA_TRY(h, cudaMemcpyAsync(c.send_out, sends, n_sends * sizeof(sdb_recv_send), cudaMemcpyHostToDevice, h->stream));
  if (payload_bytes) CUDA_TRY(h, cudaMemcpyAsync(c.payload_out, payload, payload_bytes, cudaMemcpyHostToDevice, h->stream));
  uint64_t records = 0;
  { const int rc = restore_staged(h, n_agents, n_entries, n_sends, payload_bytes, (flags & SDB_RECV_OWNED) && h->sharded, &records);
    if (rc != SDB_OK) return rc; }
  for (uint32_t i = 0; i < n_agents; ++i) h->n_agents = std::max(h->n_agents, agent_idx[i] + 1);
  h->stream_busy = false;
  if (restored_out) *restored_out = records;
  if (seq_end_out) *seq_end_out = h->next_seq;
  return SDB_OK;
}

// restore's per-agent tables and radix-sort scratch (and the compact receive buffers its input is staged in), allocated on
// the first restore or lease sweep
static int restore_ensure(sdb_ctx* h) {
  { const int rc = compact_ensure(h); if (rc != SDB_OK) return rc; }
  if (h->rs_agent) return SDB_OK;
  const size_t A = h->cfg.max_agents, tiles = sdb_scan_tops_len(A);
  const size_t R = h->cfg.max_recv_records, H = 256 * (R / 1024 + 1);
  return dmalloc_set(h, {{&h->rs_sort, 4 * R + 2 * H + sdb_scan_tops_len(H)}, {&h->rs_tot, 8}, {&h->rs_agent, 6 * A + tiles}},
                     "restore: device allocation failed");
}

// Plans and writes a restore whose input is staged on the device: the records in the compact receive's entry_out /
// send_out / payload_out and the per-agent tables (agent, count, first) in rs_agent.  Validates and plans, synchronises
// once, reserves arena space and writes; on any error nothing was written.  *records_out = records enqueued.
static int restore_staged(sdb_ctx* h, uint32_t n_agents, uint64_t n_entries, uint64_t n_sends, uint64_t payload_bytes, bool owned,
                          uint64_t* records_out) {
  const size_t A = h->cfg.max_agents;
  const size_t R = h->cfg.max_recv_records, H = 256 * (R / 1024 + 1);
  sdb_restore_args r{};
  uint32_t* t = h->rs_agent;
  r.agent = t; r.count = t + A; r.first = t + 2 * A; r.nsh = t + 3 * A; r.pgran = t + 4 * A; r.p_local = t + 5 * A; r.p_tops = t + 6 * A;
  sdb_compact_args& c = h->cx;
  r.ent = c.entry_out; r.snd = c.send_out; r.payload = c.payload_out; r.payload_bytes = payload_bytes;
  r.n = n_agents; r.n_entries = static_cast<uint32_t>(n_entries); r.n_sends = static_cast<uint32_t>(n_sends);
  r.max_payload = h->cfg.max_payload_bytes;
  r.shared = h->shared_cfg ? 1u : 0u;
  r.owned = owned ? 1u : 0u; r.shard_id = h->cfg.shard_id; r.shard_of = h->shard_of_dev;
  // scratch of the compact receive (max_recv_records entries each; the hash table holds >= 4 x that many words) and of
  // the restore's radix sort
  uint32_t* tw = reinterpret_cast<uint32_t*>(c.table);
  r.e_row = c.rec_slot;
  r.row_cnt = c.head; r.rc_local = c.head_local; r.rc_tops = c.head_tops;
  r.row_gran = c.gran; r.rg_local = c.gran_local; r.rg_tops = c.gran_tops;
  r.e_handle = tw; r.e_y = tw + R;
  {
    uint32_t* q = h->rs_sort;
    r.key_a = q; r.key_b = q + R; r.val_a = q + 2 * R; r.val_b = q + 3 * R;
    r.hist = q + 4 * R; r.h_local = q + 4 * R + H; r.h_tops = q + 4 * R + 2 * H;
  }
  r.tot = h->rs_tot;
  int nl = 0;
  cudaError_t e = sdb_launch_restore_plan(&h->view, &r, h->stream, &h->prof, &nl, h->sm_count);
  h->launches += nl;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("restore plan launch: ") + cudaGetErrorString(e));
  // the plan's totals come back through totals_host and are kept apart: arena_reserve reuses its TOT_FLOOR slot
  unsigned long long tot[6];
  static_assert(sizeof(tot) <= TOT_SLOTS * sizeof(unsigned long long), "totals_host holds the restore plan's totals");
  CUDA_TRY(h, cudaMemcpyAsync(h->totals_host, h->rs_tot, sizeof(tot), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  std::memcpy(tot, h->totals_host, sizeof(tot));
  if (tot[3] & SDB_RS_EINVAL)
    return fail(h, SDB_EINVAL, "sdb_restore_compact: bad entry (send index, receiver) or row (len, prio, payload_off)");
  if (tot[3] & SDB_RS_ERING) return fail(h, SDB_ERING_OVERFLOW, "sdb_restore_compact: a ring cannot take the agent's records");
  const uint64_t records = tot[4], need = tot[0] + tot[1];
  if (records) {
    uint64_t base = 0;
    { const int rc = arena_reserve(h, need, &base); if (rc != SDB_OK) return rc; }
    r.base = base;
    nl = 0;
    e = sdb_launch_restore_write(&h->view, &r, tot[0], static_cast<uint32_t>(tot[5]), h->stream, &h->prof, &nl, h->sm_count);
    h->launches += nl;
    if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("restore write launch: ") + cudaGetErrorString(e));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    h->arena_tail = base + need;
    if (tot[2] + 1 > h->next_seq) h->next_seq = tot[2] + 1;
    h->dev_stale = true;
  }
  *records_out = records;
  return SDB_OK;
}

// ---- relocation of pinned queues -------------------------------------------------------------------------------------
int sdb_arena_relocate(sdb_handle h, uint64_t floor_bytes, uint32_t flags, sdb_relocate_summary* out) {
  if (!h) return SDB_EINVAL;
  if (out) *out = sdb_relocate_summary{};
  if (flags & ~SDB_RECV_PEEK) return fail(h, SDB_EINVAL, "sdb_arena_relocate accepts SDB_RECV_PEEK only");
  { int rcc = cursor_to_host(h); if (rcc != SDB_OK) return rcc; }      // a host-placed write, like a send
  const uint64_t G = h->arena_grans, tail = h->arena_tail;
  if (!h->rl_bits) {
    const size_t W = G / 32 + 2, A = h->cfg.max_agents;
    const int rc = dmalloc_set(h, {{&h->rl_bits, W}, {&h->rl_cnt, W}, {&h->rl_pre, W}, {&h->rl_tops, sdb_scan_tops_len(W)}, {&h->rl_sel, A / 32 + 1},
                                   {&h->rl_tot, 8}}, "sdb_arena_relocate: device allocation failed");
    if (rc != SDB_OK) return rc;
  }
  // every pending record lies in [arena_floor, tail), at most G granules below the tail
  const uint64_t lo = std::max<uint64_t>(h->arena_floor, tail > G ? tail - G : 0) & ~31ull;
  const uint64_t cut = std::min(floor_bytes / SDB_GRANULE + ((floor_bytes % SDB_GRANULE) ? 1u : 0u), tail);
  sdb_reloc_args r{};
  r.bits = h->rl_bits; r.cnt = h->rl_cnt; r.pre = h->rl_pre; r.tops = h->rl_tops; r.sel = h->rl_sel; r.tot = h->rl_tot;
  r.lo = lo; r.tail = tail;
  r.words = static_cast<uint32_t>((tail - lo) / 32 + 1);
  r.thr = static_cast<uint32_t>(std::min<uint64_t>(tail - cut, 0xFFFFFFFFull));
  r.n_agents = h->n_agents;
  int nl = 0;
  cudaError_t e = sdb_launch_reloc_plan(&h->view, &r, h->stream, &h->prof, &nl, h->sm_count);
  h->launches += nl;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("relocate plan launch: ") + cudaGetErrorString(e));
  unsigned long long tot[5];
  static_assert(sizeof(tot) <= TOT_SLOTS * sizeof(unsigned long long), "totals_host holds the relocation plan's totals");
  CUDA_TRY(h, cudaMemcpyAsync(h->totals_host, h->rl_tot, sizeof(tot), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->stream_busy = false;
  std::memcpy(tot, h->totals_host, sizeof(tot));
  const uint64_t moved = tot[0];
  const uint64_t floor_now = tail - tot[3];                            // what k_arena_floor would find now
  uint64_t base = tail;
  if (moved) {                                                         // arena_reserve's placement and fit test
    if ((tail & (G - 1)) + moved > G) base = (tail + G - 1) & ~(G - 1);
    if (moved > G || base + moved - floor_now > G)
      return fail(h, SDB_EARENA_FULL, "sdb_arena_relocate: the moved records do not fit behind the arena tail (the arena is too "
                                      "full of live records to relocate them: receive, expire, or choose a lower cut)");
  }
  const uint64_t tail_after = base + moved;
  uint64_t floor_after = tot[4] ? tail - tot[4] : tail_after;          // the unselected agents' oldest records ...
  if (moved) floor_after = std::min(floor_after, base);                // ... and the moved region
  sdb_relocate_summary s{};
  s.agents = tot[1]; s.records = tot[2];
  s.moved_bytes = moved * SDB_GRANULE; s.skipped_bytes = (base - tail) * SDB_GRANULE;
  s.floor_before = floor_now * SDB_GRANULE; s.floor_after = floor_after * SDB_GRANULE; s.tail_after = tail_after * SDB_GRANULE;
  if (flags & SDB_RECV_PEEK) {
    if (out) *out = s;
    return SDB_OK;
  }
  if (moved) {
    r.base = base;
    const sdb_ctx::LeaseStore& L = h->lease;
    const bool ledger = L.policy && L.led_n;
    nl = 0;
    e = sdb_launch_reloc_write(&h->view, &r, ledger ? &L.led : nullptr, static_cast<uint32_t>(ledger ? L.led_n : 0), h->stream,
                               &h->prof, &nl, h->sm_count);
    h->launches += nl;
    if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("relocate write launch: ") + cudaGetErrorString(e));
    const int pi = sdb_prof_begin(&h->prof, SDB_PK_ARENA_FLOOR, h->stream);
    e = sdb_launch_arena_floor(&h->view, h->n_agents, static_cast<uint32_t>(tail_after), h->rx_totals + TOT_FLOOR, h->stream);
    sdb_prof_end(&h->prof, pi, h->stream);
    h->launches += 1;
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->totals_host + TOT_FLOOR, h->rx_totals + TOT_FLOOR, sizeof(unsigned long long),
                                             cudaMemcpyDeviceToHost, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("relocate: ") + cudaGetErrorString(e));
    h->arena_tail = tail_after;
    h->arena_floor = tail_after - h->totals_host[TOT_FLOOR];
  } else {
    h->arena_floor = std::max(h->arena_floor, floor_now);
  }
  h->dev_stale = true;
  s.floor_after = h->arena_floor * SDB_GRANULE;
  if (out) *out = s;
  return SDB_OK;
}

// ---- lease store: leased receive, settle, sweep ----------------------------------------------------------------------
static void lease_policy_free(sdb_ctx* h) {
  sdb_ctx::LeaseStore& L = h->lease;
  for (void* p : L.pmem) cudaFree(p);
  if (L.lth) cudaFreeHost(L.lth);
  L.pmem.clear(); L.lth = nullptr;
  L.buf[0].deliveries = L.buf[1].deliveries = nullptr;
  L.led = sdb_ledger{}; L.dl = sdb_dl_scratch{};
  L.policy = false; L.max_deliveries = 0; L.led_cap = L.led_n = L.led_live = 0;
  L.dead = 0;
}
static void lease_free(sdb_ctx* h) {
  sdb_ctx::LeaseStore& L = h->lease;
  lease_policy_free(h);
  for (void* p : L.mem) cudaFree(p);
  if (L.th) cudaFreeHost(L.th);
  L.mem.clear(); L.th = nullptr;
  L.buf[0] = L.buf[1] = sdb_lease_buf{}; L.s = sdb_lease_scratch{};
  L.cap = L.pay_cap = L.used = L.rows = L.pay = L.acked = 0; L.cur = 0;
}
int sdb_lease_reserve(sdb_handle h, uint64_t max_records, uint64_t max_payload_bytes) {
  if (!h) return SDB_EINVAL;
  sdb_ctx::LeaseStore& L = h->lease;
  if (L.live) return fail(h, SDB_EINVAL, "sdb_lease_reserve: the store holds live leases (ack them or sweep them back first)");
  if (L.dead) return fail(h, SDB_EINVAL, "sdb_lease_reserve: the store holds dead letters (sdb_lease_dead_letters first)");
  if (max_records > 0xFFFFFFF0ull) return fail(h, SDB_EINVAL, "sdb_lease_reserve: max_records above 2^32 - 16");
  { const int rc = ls_stop(h); if (rc != SDB_OK) return rc; }        // cudaFree / cudaMalloc wait for running kernels
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->stream_busy = false;
  lease_free(h);
  if (!max_records) return SDB_OK;
  const uint64_t P = (max_payload_bytes + SDB_GRANULE - 1) & ~static_cast<uint64_t>(SDB_GRANULE - 1);
  const size_t cap = max_records, R = h->cfg.max_recv_records, S = std::max(cap, R), A = h->cfg.max_agents;
  const size_t tS = sdb_scan_tops_len(S), tR = sdb_scan_tops_len(R), tC = sdb_scan_tops_len(cap), tA = sdb_scan_tops_len(A);
  const size_t H = 256 * (R / 1024 + 1);
  std::vector<void*>& m = L.mem;
  bool ok = true;
  for (sdb_lease_buf& b : L.buf)
    ok = ok && lease_alloc(m, &b.ent, cap) && lease_alloc(m, &b.agent, cap) && lease_alloc(m, &b.id, cap) &&
         lease_alloc(m, &b.deadline, cap) && lease_alloc(m, &b.state, cap) && lease_alloc(m, &b.rows, cap) &&
         lease_alloc(m, &b.payload, P);
  sdb_lease_scratch& s = L.s;
  ok = ok && lease_alloc(m, &s.flag, S) && lease_alloc(m, &s.f_local, S) && lease_alloc(m, &s.f_tops, tS) &&
       lease_alloc(m, &s.gran, S) && lease_alloc(m, &s.g_local, S) && lease_alloc(m, &s.g_tops, tS) &&
       lease_alloc(m, &s.rfirst, cap) && lease_alloc(m, &s.rmap, cap) &&
       lease_alloc(m, &s.rg, cap) && lease_alloc(m, &s.rg_local, cap) && lease_alloc(m, &s.rg_tops, tC) &&
       lease_alloc(m, &s.chunk, R) && lease_alloc(m, &s.staged, R) && lease_alloc(m, &s.key_a, R) && lease_alloc(m, &s.key_b, R) &&
       lease_alloc(m, &s.val_a, R) && lease_alloc(m, &s.val_b, R) &&
       lease_alloc(m, &s.hist, H) && lease_alloc(m, &s.h_local, H) && lease_alloc(m, &s.h_tops, sdb_scan_tops_len(H)) &&
       lease_alloc(m, &s.run_begin, R + 1) && lease_alloc(m, &s.kcnt, R) && lease_alloc(m, &s.k_local, R) &&
       lease_alloc(m, &s.k_tops, tR) && lease_alloc(m, &s.kflag, R) && lease_alloc(m, &s.kf_local, R) && lease_alloc(m, &s.kf_tops, tR) &&
       lease_alloc(m, &s.a_local, A) && lease_alloc(m, &s.a_tops, tA) &&
       lease_alloc(m, &s.req, SDB_LS_SETTLE_CHUNK) && lease_alloc(m, &s.at, SDB_LS_SETTLE_CHUNK) &&
       lease_alloc(m, &s.settled, SDB_LS_SETTLE_CHUNK) && lease_alloc(m, &s.tot, 16);
  ok = ok && cudaHostAlloc(reinterpret_cast<void**>(&L.th), 16 * sizeof(unsigned long long), cudaHostAllocDefault) == cudaSuccess;
  if (!ok) {
    lease_free(h);
    cudaGetLastError();
    return fail(h, SDB_ENOMEM, "sdb_lease_reserve: device allocation failed");
  }
  L.cap = cap; L.pay_cap = P;
  return SDB_OK;
}

// What a filtered call reads from its sdb_filter besides the clauses: the id block and whether a keyword applies
struct where_req {
  uint64_t n_ids = 0;
  uint32_t* id_hits = nullptr;
  uint32_t* id_agent = nullptr;
  bool use_ids = false, use_kw = false;
};
// A filter's refusals (sdb_receive_where's), checked before anything runs; `name` names the call in error messages
static int where_check(sdb_ctx* h, const sdb_filter* filter, const char* name, where_req* w) {
  constexpr uint32_t all_fields = SDB_FILTER_SENDER | SDB_FILTER_RECEIVER | SDB_FILTER_GROUP | SDB_FILTER_TYPE | SDB_FILTER_PRIO |
                                  SDB_FILTER_TIME | SDB_FILTER_SEQ | SDB_FILTER_KEYWORD | SDB_FILTER_ICASE | SDB_FILTER_IDS;
  constexpr uint32_t v1_bytes = offsetof(sdb_filter, n_ids);  // the struct before the id block: callers built against it
  const std::string n(name);
  if (!filter || (filter->struct_bytes != sizeof(sdb_filter) && filter->struct_bytes != v1_bytes))
    return fail(h, SDB_EINVAL, n + ": struct_bytes is neither sizeof(sdb_filter) nor offsetof(sdb_filter, n_ids)");
  if (filter->fields & ~all_fields) return fail(h, SDB_EINVAL, n + ": unknown filter fields");
  // the id block is read only with the full struct_bytes
  w->use_ids = (filter->fields & SDB_FILTER_IDS) != 0;
  w->n_ids = w->use_ids ? filter->n_ids : 0;
  w->id_hits = filter->struct_bytes == v1_bytes ? nullptr : filter->id_hits;
  w->id_agent = filter->struct_bytes == v1_bytes ? nullptr : filter->id_agent;
  if (w->use_ids) {
    if (filter->struct_bytes == v1_bytes) return fail(h, SDB_EINVAL, n + ": SDB_FILTER_IDS needs struct_bytes == sizeof(sdb_filter)");
    if (w->n_ids > SDB_FILTER_MAX_IDS) return fail(h, SDB_EINVAL, n + ": n_ids > SDB_FILTER_MAX_IDS");
    if (!filter->ids) return fail(h, SDB_EINVAL, n + ": NULL ids (an empty set takes any other pointer)");
  } else if (w->id_hits || w->id_agent) {
    return fail(h, SDB_EINVAL, n + ": id_hits / id_agent without SDB_FILTER_IDS");
  }
  w->use_kw = (filter->fields & SDB_FILTER_KEYWORD) && filter->keyword_len;
  if (filter->fields & SDB_FILTER_KEYWORD) {
    if (filter->keyword_len > SDB_FILTER_MAX_KEYWORD) return fail(h, SDB_EINVAL, n + ": keyword_len > SDB_FILTER_MAX_KEYWORD");
    if (filter->keyword_len && !filter->keyword) return fail(h, SDB_EINVAL, n + ": NULL keyword");
  }
  return SDB_OK;
}

// the per-id outputs before the call: no hits, no agent
static void where_id_reset(const where_req& w) {
  if (w.id_hits) std::fill(w.id_hits, w.id_hits + w.n_ids, 0u);
  if (w.id_agent) std::fill(w.id_agent, w.id_agent + w.n_ids, SDB_NO_RECEIVER);
}

// After where_check: the verdict bitmap allocated, the keyword and the id table on the device, *f filled
static int where_setup(sdb_ctx* h, const sdb_filter* filter, const where_req& w, sdb_where_args* f, int* nl) {
  const uint32_t stride = where_stride(h);
  { const int rc = where_ensure(h); if (rc != SDB_OK) return rc; }
  if (w.use_kw) CUDA_TRY(h, cudaMemcpyAsync(h->where_kw, filter->keyword, filter->keyword_len, cudaMemcpyHostToDevice, h->stream));
  const uint64_t n_ids = w.n_ids;
  uint64_t id_slots = 64;                                     // a power of two >= 2 x n_ids (an empty table matches nothing)
  while (id_slots < 2 * n_ids) id_slots <<= 1;
  if (w.use_ids) {
    if (id_slots > h->id_slots || n_ids > h->id_cap) {
      const uint64_t cap = std::max(n_ids, h->id_cap), slots = std::max(id_slots, h->id_slots);
      { const int rc = ls_stop(h); if (rc != SDB_OK) return rc; }   // cudaFree waits for the kernels on the device
      for (void* p : {static_cast<void*>(h->id_tab), static_cast<void*>(h->id_in), static_cast<void*>(h->id_out)}) if (p) cudaFree(p);
      h->id_tab = nullptr; h->id_in = nullptr; h->id_out = nullptr; h->id_cap = h->id_slots = 0;
      const int rc = dmalloc_set(h, {{&h->id_tab, slots}, {&h->id_in, cap}, {&h->id_out, 2 * cap}},
                                 "filtered receive: id table allocation failed");
      if (rc != SDB_OK) return rc;
      h->id_cap = cap; h->id_slots = slots;
    }
    CUDA_TRY(h, cudaMemsetAsync(h->id_tab, 0, id_slots * sizeof(sdb_id_slot), h->stream));
    if (n_ids) CUDA_TRY(h, cudaMemcpyAsync(h->id_in, filter->ids, n_ids * sizeof(uint64_t), cudaMemcpyHostToDevice, h->stream));
    const cudaError_t e = sdb_launch_id_table(h->id_in, static_cast<uint32_t>(n_ids), h->id_tab, static_cast<uint32_t>(id_slots - 1),
                                              h->stream, nl);
    if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("id table launch: ") + cudaGetErrorString(e));
  }
  *f = sdb_where_args{};
  f->fields = w.use_kw ? filter->fields : (filter->fields & ~SDB_FILTER_KEYWORD);
  f->sender = filter->sender; f->receiver = filter->receiver; f->group = filter->group;
  f->type_mask = filter->type_mask; f->prio_mask = filter->prio_mask; f->kw_len = w.use_kw ? filter->keyword_len : 0u;
  f->after = filter->after; f->before = filter->before; f->seq_lo = filter->seq_lo; f->seq_hi = filter->seq_hi;
  f->kw = h->where_kw; f->bits = h->where_bits; f->stride = stride;
  f->id_tab = h->id_tab; f->id_mask = static_cast<uint32_t>(id_slots - 1); f->id_count = (w.id_hits || w.id_agent) && n_ids ? 1u : 0u;
  return SDB_OK;
}

// After the filtered launch: the per-id outputs read out and their copies queued (the caller's synchronisation covers them)
static cudaError_t where_id_out(sdb_ctx* h, const where_req& w, const sdb_where_args& f, int* nl) {
  if (!f.id_count) return cudaSuccess;
  cudaError_t e = sdb_launch_id_out(h->id_in, static_cast<uint32_t>(w.n_ids), h->id_tab, f.id_mask, h->id_out, h->stream, nl);
  if (e == cudaSuccess && w.id_hits)
    e = cudaMemcpyAsync(w.id_hits, h->id_out, w.n_ids * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess && w.id_agent)
    e = cudaMemcpyAsync(w.id_agent, h->id_out + w.n_ids, w.n_ids * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream);
  return e;
}

// the take limits of sdb_launch_where (~0: none): sum(pad32(len)) <= max_agent_bytes in payload granules, and tokens
static unsigned long long agent_gran_limit(uint64_t max_agent_bytes) { return max_agent_bytes ? max_agent_bytes / SDB_GRANULE : ~0ull; }
static unsigned long long token_limit(uint64_t max_agent_tokens) { return max_agent_tokens ? max_agent_tokens : ~0ull; }

// Collection pass of the redelivery ledger (stream-ordered, no synchronisation): the entries whose record is still the
// one a sweep put back are rebuilt into the other buffer and re-indexed; led.tot[0] counts them.
static cudaError_t ledger_collect(sdb_ctx* h) {
  sdb_ctx::LeaseStore& L = h->lease;
  int nl = 0;
  cudaError_t e = sdb_launch_ledger_collect(&h->view, &L.led, static_cast<uint32_t>(L.led_n), h->stream, &h->prof, &nl);
  h->launches += nl;
  std::swap(L.led.ent, L.led.alt);
  return e;
}

// sdb_receive_leased and sdb_receive_leased_select (both limits 0 and no filter: the plain leased call); `name` names the
// call in errors.  Without a filter the limits run the receive's budget or token plan, with a granule capacity that the
// records capacity always reaches first; with one, the filtered pipeline with its take pass and the compact back end.
static int receive_leased_full(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                               uint64_t max_agent_bytes, uint64_t max_agent_tokens, const sdb_filter* filter, uint32_t flags,
                               double deadline, uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
                               sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                               uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out, uint64_t* lease_base_out,
                               const char* name) {
  if (!h) return SDB_EINVAL;
  sdb_ctx::LeaseStore& L = h->lease;
  const std::string nm(name);
  if (total_out) *total_out = 0;
  if (n_sends_out) *n_sends_out = 0;
  if (payload_bytes_out) *payload_bytes_out = 0;
  if (lease_base_out) *lease_base_out = L.next_id;
  if (flags & ~(SDB_RECV_PRIORITY | SDB_RECV_OWNED))
    return fail(h, SDB_EINVAL, nm + " accepts SDB_RECV_PRIORITY and SDB_RECV_OWNED only");
  if (!L.cap) return fail(h, SDB_EINVAL, nm + ": no lease store (sdb_lease_reserve)");
  where_req w;
  if (filter) { const int rc = where_check(h, filter, name, &w); if (rc != SDB_OK) return rc; }
  const bool owned = recv_agents(h, flags, agent_idx, &n_agents);
  where_id_reset(w);
  if (n_agents == 0 || max_messages == 0) return SDB_OK;
  { const int rc = check_recv_agents(h, n_agents, agent_idx); if (rc != SDB_OK) return rc; }
  uint64_t rec_cap = 0;
  { const int rc = out_rec_cap(h, std::min(room(entry_out, entry_cap), room(send_out, send_cap)), room(payload_out, payload_cap), &rec_cap);
    if (rc != SDB_OK) return rc; }
  const uint32_t P = pad32(h->cfg.max_payload_bytes);
  rec_cap = std::min({rec_cap, L.cap - L.used, (L.pay_cap - L.pay) / P});     // the store takes every record of the call
  if (rec_cap == 0) return fail(h, SDB_ECAPACITY, "lease store full: settle or sweep");
  { const int rc = compact_ensure(h); if (rc != SDB_OK) return rc; }
  sdb_recv_args r{};
  { const int rc = recv_args(h, n_agents, agent_idx, owned, max_messages, flags & SDB_RECV_PRIORITY, rec_cap, &r); if (rc != SDB_OK) return rc; }
  int nl = 0;
  sdb_where_args f{};
  if (filter) { const int rc = where_setup(h, filter, w, &f, &nl); if (rc != SDB_OK) return rc; }
  const bool ledger = L.policy && L.led_n;      // the ledger holds entries: collect before anything is retired, look up after
  cudaError_t e = ledger ? ledger_collect(h) : cudaSuccess;
  if (e == cudaSuccess) {
    if (filter) {
      e = sdb_launch_where(&h->view, &r, &f, 0, 32u + P, h->stream, &nl, &h->prof, h->sm_count, &h->cx,
                           agent_gran_limit(max_agent_bytes), token_limit(max_agent_tokens));
      if (e == cudaSuccess) e = where_id_out(h, w, f, &nl);
    } else if (max_agent_bytes || max_agent_tokens) {
      // granule capacity rec_cap x P / 32: a plan within rec_cap records never reaches it, so the records capacity and
      // its truncation rule are sdb_receive_leased's
      const uint64_t agent_gran = agent_gran_limit(max_agent_bytes), gran_cap = rec_cap * (P / SDB_GRANULE);
      const uint2 budget = make_uint2(static_cast<uint32_t>(std::min<uint64_t>(agent_gran, 0xFFFFFFFFull)),
                                      static_cast<uint32_t>(std::min<uint64_t>(gran_cap, 0xFFFFFFFFull)));
      e = sdb_launch_receive(&h->view, &r, h->stream, &nl, &h->prof, h->sm_count, 32u + P, &h->cx, &budget, max_agent_tokens);
    } else {
      e = sdb_launch_receive(&h->view, &r, h->stream, &nl, &h->prof, h->sm_count, 32u + P, &h->cx, nullptr, 0ull);
    }
  }
  h->last_rx_valid = false; h->last_rx_compact = true;
  if (e == cudaSuccess)
    e = sdb_launch_lease_append(&L.buf[L.cur], &L.s, &h->cx, h->rx_count, h->rx_totals, r.agent_idx, n_agents,
                                static_cast<uint32_t>(L.used), static_cast<uint32_t>(L.rows), L.pay, L.next_id, deadline, rec_cap,
                                P, h->stream, &h->prof, &nl, h->sm_count);
  if (e == cudaSuccess && ledger)
    e = sdb_launch_ledger_take(&L.buf[L.cur], &L.led, &h->cx, h->rx_totals, static_cast<uint32_t>(L.used), rec_cap, h->stream,
                               &h->prof, &nl, h->sm_count);
  if (e == cudaSuccess && ledger)
    e = cudaMemcpyAsync(L.lth, L.led.tot, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream);
  h->launches += nl;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("leased receive launch: ") + cudaGetErrorString(e));
  uint64_t total = 0, n_sends = 0, pbytes = 0;
  { const int rc = copy_compact(h, n_agents, count_out, entry_out, send_out, payload_out, &total, &n_sends, &pbytes);
    if (rc != SDB_OK) return rc; }
  if (ledger) { L.led_n = L.lth[0]; L.led_live = L.lth[0] - L.lth[1]; }
  L.used += total; L.rows += n_sends; L.pay += pbytes; L.live += total; L.next_id += total;
  if (total_out) *total_out = total;
  if (n_sends_out) *n_sends_out = n_sends;
  if (payload_bytes_out) *payload_bytes_out = pbytes;
  return SDB_OK;
}

int sdb_receive_leased(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages, uint32_t flags,
                       double deadline, uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
                       sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                       uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out, uint64_t* lease_base_out) {
  return receive_leased_full(h, n_agents, agent_idx, max_messages, 0, 0, nullptr, flags, deadline, count_out, entry_out, entry_cap,
                             send_out, send_cap, payload_out, payload_cap, total_out, n_sends_out, payload_bytes_out,
                             lease_base_out, "sdb_receive_leased");
}

int sdb_receive_leased_select(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                              uint64_t max_agent_bytes, uint64_t max_agent_tokens, const sdb_filter* filter, uint32_t flags,
                              double deadline, uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
                              sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                              uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out, uint64_t* lease_base_out) {
  return receive_leased_full(h, n_agents, agent_idx, max_messages, max_agent_bytes, max_agent_tokens, filter, flags, deadline,
                             count_out, entry_out, entry_cap, send_out, send_cap, payload_out, payload_cap, total_out,
                             n_sends_out, payload_bytes_out, lease_base_out, "sdb_receive_leased_select");
}

int sdb_lease_settle(sdb_handle h, uint64_t n, const uint64_t* lease_id, uint32_t op, double deadline, uint8_t* settled_out,
                     uint64_t* n_settled_out) {
  if (!h) return SDB_EINVAL;
  if (n_settled_out) *n_settled_out = 0;
  if (op != SDB_LEASE_ACK && op != SDB_LEASE_RENEW) return fail(h, SDB_EINVAL, "sdb_lease_settle: op is SDB_LEASE_ACK or SDB_LEASE_RENEW");
  if (n && !lease_id) return fail(h, SDB_EINVAL, "sdb_lease_settle: lease_id is NULL");
  sdb_ctx::LeaseStore& L = h->lease;
  if (!L.cap) return fail(h, SDB_EINVAL, "sdb_lease_settle: no lease store (sdb_lease_reserve)");
  uint64_t settled = 0, moved = 0;
  for (uint64_t o = 0; o < n; o += SDB_LS_SETTLE_CHUNK) {
    const uint32_t m = static_cast<uint32_t>(std::min<uint64_t>(SDB_LS_SETTLE_CHUNK, n - o));
    CUDA_TRY(h, cudaMemcpyAsync(L.s.req, lease_id + o, m * sizeof(uint64_t), cudaMemcpyHostToDevice, h->stream));
    int nl = 0;
    cudaError_t e = sdb_launch_lease_settle(&L.buf[L.cur], &L.s, static_cast<uint32_t>(L.used), m, op, deadline, h->stream, &h->prof, &nl);
    h->launches += nl;
    if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("lease settle launch: ") + cudaGetErrorString(e));
    CUDA_TRY(h, cudaMemcpyAsync(L.th, L.s.tot, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
    if (settled_out) CUDA_TRY(h, cudaMemcpyAsync(settled_out + o, L.s.settled, m, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    settled += L.th[0]; moved += L.th[1];
  }
  h->stream_busy = false;
  L.live -= moved; L.acked += moved; L.acked_total += moved;
  if (n_settled_out) *n_settled_out = settled;
  return SDB_OK;
}

// reads s.tot[lo, lo + k) into the store's pinned mirror, synchronising
static int lease_totals(sdb_ctx* h, uint32_t lo, uint32_t k) {
  CUDA_TRY(h, cudaMemcpyAsync(h->lease.th + lo, h->lease.s.tot + lo, k * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return SDB_OK;
}

int sdb_lease_sweep(sdb_handle h, double now, uint32_t flags, uint64_t* redelivered_out, uint64_t* blocked_out,
                    uint64_t* due_left_out) {
  if (!h) return SDB_EINVAL;
  if (redelivered_out) *redelivered_out = 0;
  if (blocked_out) *blocked_out = 0;
  if (due_left_out) *due_left_out = 0;
  if (flags & ~SDB_LEASE_ALL) return fail(h, SDB_EINVAL, "sdb_lease_sweep accepts SDB_LEASE_ALL only");
  sdb_ctx::LeaseStore& L = h->lease;
  if (!L.cap) return fail(h, SDB_EINVAL, "sdb_lease_sweep: no lease store (sdb_lease_reserve)");
  { int rcc = cursor_to_host(h); if (rcc != SDB_OK) return rcc; }      // redelivery is a host-placed write, like a send
  if (L.used == 0) return SDB_OK;
  { const int rc = restore_ensure(h); if (rc != SDB_OK) return rc; }
  const sdb_lease_buf& b = L.buf[L.cur];
  const uint32_t used = static_cast<uint32_t>(L.used), rows = static_cast<uint32_t>(L.rows);
  const uint32_t M = L.max_deliveries;
  if (L.policy && L.led_n) {                    // the ledger's free room is known exactly after a collection
    cudaError_t ec = ledger_collect(h);
    if (ec == cudaSuccess) ec = cudaMemcpyAsync(L.lth, L.led.tot, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream);
    if (ec != cudaSuccess) return fail(h, SDB_ECUDA, std::string("lease sweep launch: ") + cudaGetErrorString(ec));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    L.led_n = L.led_live = L.lth[0];
  }
  int nl = 0;
  cudaError_t e = sdb_launch_lease_due(&b, &L.s, used, now, flags & SDB_LEASE_ALL, M, h->stream, &h->prof, &nl);
  h->launches += nl;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("lease sweep launch: ") + cudaGetErrorString(e));
  { const int rc = lease_totals(h, 0, 1); if (rc != SDB_OK) return rc; }
  const uint64_t due = L.th[0];
  uint64_t n64 = std::min<uint64_t>(due, recv_rec_cap(h));                             // one compact receive's capacity
  const uint64_t held = L.policy ? n64 - std::min<uint64_t>(n64, L.led_cap - L.led_n) : 0;   // the ledger's free room
  n64 -= held;
  const uint32_t n = static_cast<uint32_t>(n64);
  uint64_t staged = 0, blocked = 0, redelivered = 0;
  if (n) {
    const size_t A = h->cfg.max_agents;
    nl = 0;
    e = sdb_launch_lease_select(&h->view, &b, &L.s, used, n, h->cfg.max_agents, h->rs_agent, h->rs_agent + A, h->rs_agent + 2 * A,
                                h->stream, &h->prof, &nl);
    h->launches += nl;
    if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("lease sweep launch: ") + cudaGetErrorString(e));
    { const int rc = lease_totals(h, 1, 5); if (rc != SDB_OK) return rc; }
    staged = L.th[2]; blocked = L.th[4];
    const uint32_t kept_runs = static_cast<uint32_t>(L.th[3]), agent_end = static_cast<uint32_t>(L.th[5]);
    if (staged) {
      nl = 0;
      e = sdb_launch_lease_stage(&b, &L.s, rows, static_cast<uint32_t>(staged), h->next_seq, &h->cx, h->stream, &h->prof, &nl, h->sm_count);
      h->launches += nl;
      if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("lease sweep launch: ") + cudaGetErrorString(e));
      { const int rc = lease_totals(h, 6, 2); if (rc != SDB_OK) return rc; }
      { const int rc = restore_staged(h, kept_runs, staged, L.th[6], L.th[7] * SDB_GRANULE, false, &redelivered);
        if (rc != SDB_OK) return rc; }                                     // SDB_EARENA_FULL: nothing written, store unchanged
      h->n_agents = std::max(h->n_agents, agent_end);
      if (L.policy) {                                                      // the counts follow the records into the ledger
        nl = 0;
        e = sdb_launch_ledger_insert(&h->view, &b, &L.s, &L.led, h->rs_agent, h->rs_agent + A, h->rs_agent + 2 * A, kept_runs,
                                     static_cast<uint32_t>(L.led_n), h->stream, &h->prof, &nl, h->sm_count);
        h->launches += nl;
        if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("lease sweep launch: ") + cudaGetErrorString(e));
        L.led_n += staged; L.led_live += staged;
      }
    }
  }
  // compaction: redelivered and acked entries are dropped, with the rows and payloads no live entry names
  nl = 0;
  e = sdb_launch_lease_compact(&b, &L.buf[L.cur ^ 1], &L.s, used, rows, static_cast<uint32_t>(staged), M, now, flags & SDB_LEASE_ALL,
                               h->stream, &h->prof, &nl, h->sm_count);
  h->launches += nl;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("lease sweep launch: ") + cudaGetErrorString(e));
  { const int rc = lease_totals(h, 8, M ? 4 : 3); if (rc != SDB_OK) return rc; }
  h->stream_busy = false;
  L.cur ^= 1;
  L.used = L.th[8]; L.rows = L.th[9]; L.pay = L.th[10] * SDB_GRANULE;
  const uint64_t killed = M ? L.th[11] : 0;
  L.live -= staged + killed; L.redelivered_total += staged; L.acked = 0;
  L.dead += killed; L.dead_total += killed; L.held_total += held;
  if (redelivered_out) *redelivered_out = staged;
  if (blocked_out) *blocked_out = blocked;
  if (due_left_out) *due_left_out = due - n;
  return SDB_OK;
}

int sdb_lease_stats(sdb_handle h, sdb_lease_summary* out) {
  if (!h || !out) return SDB_EINVAL;
  const sdb_ctx::LeaseStore& L = h->lease;
  out->live = L.live; out->acked_unreclaimed = L.acked;
  out->redelivered_total = L.redelivered_total; out->acked_total = L.acked_total;
  out->entries_used = L.used; out->entries_reserved = L.cap;
  out->payload_used = L.pay; out->payload_reserved = L.pay_cap;
  return SDB_OK;
}

int sdb_lease_set_policy(sdb_handle h, uint32_t max_deliveries, uint64_t ledger_entries) {
  if (!h) return SDB_EINVAL;
  sdb_ctx::LeaseStore& L = h->lease;
  if (!L.cap) return fail(h, SDB_EINVAL, "sdb_lease_set_policy: no lease store (sdb_lease_reserve)");
  if (L.live || L.dead) return fail(h, SDB_EINVAL, "sdb_lease_set_policy: the store holds live leases or dead letters");
  if (max_deliveries && !ledger_entries) return fail(h, SDB_EINVAL, "sdb_lease_set_policy: a redelivery limit needs ledger entries");
  if (ledger_entries > 0x7FFFFFF0ull) return fail(h, SDB_EINVAL, "sdb_lease_set_policy: ledger_entries above 2^31 - 16");
  { const int rc = ls_stop(h); if (rc != SDB_OK) return rc; }        // cudaFree / cudaMalloc wait for running kernels
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->stream_busy = false;
  lease_policy_free(h);
  if (!max_deliveries) return SDB_OK;
  const size_t cap = L.cap, N = ledger_entries, A = h->cfg.max_agents, H = 256 * (cap / 1024 + 1);
  sdb_dl_scratch& d = L.dl;
  std::vector<void*>& m = L.pmem;
  bool ok = lease_alloc(m, &L.buf[0].deliveries, cap) && lease_alloc(m, &L.buf[1].deliveries, cap) && lease_alloc(m, &L.led.ent, N) &&
            lease_alloc(m, &L.led.alt, N) && lease_alloc(m, &L.led.index, 2 * N) && lease_alloc(m, &L.led.tot, 2) &&
            lease_alloc(m, &d.key_a, cap) && lease_alloc(m, &d.key_b, cap) && lease_alloc(m, &d.val_a, cap) &&
            lease_alloc(m, &d.val_b, cap) && lease_alloc(m, &d.staged, cap) && lease_alloc(m, &d.hist, H) &&
            lease_alloc(m, &d.h_local, H) && lease_alloc(m, &d.h_tops, sdb_scan_tops_len(H)) && lease_alloc(m, &d.pos, A) &&
            lease_alloc(m, &d.cnt, A);
  ok = ok && cudaHostAlloc(reinterpret_cast<void**>(&L.lth), 2 * sizeof(unsigned long long), cudaHostAllocDefault) == cudaSuccess;
  ok = ok && cudaMemsetAsync(d.pos, 0xFF, A * sizeof(uint32_t), h->stream) == cudaSuccess &&
       cudaMemsetAsync(L.led.index, 0xFF, 2 * N * sizeof(uint32_t), h->stream) == cudaSuccess &&
       cudaStreamSynchronize(h->stream) == cudaSuccess;
  if (!ok) {
    lease_policy_free(h);
    cudaGetLastError();
    return fail(h, SDB_ENOMEM, "sdb_lease_set_policy: device allocation failed");
  }
  L.led.slots = static_cast<uint32_t>(2 * N);
  L.policy = true; L.max_deliveries = max_deliveries; L.led_cap = N;
  return SDB_OK;
}

int sdb_lease_deliveries(sdb_handle h, uint64_t n, const uint64_t* lease_id, uint32_t* deliveries_out) {
  if (!h) return SDB_EINVAL;
  if (deliveries_out) std::memset(deliveries_out, 0, n * sizeof(uint32_t));
  sdb_ctx::LeaseStore& L = h->lease;
  if (!L.policy) return fail(h, SDB_EINVAL, "sdb_lease_deliveries: no redelivery policy (sdb_lease_set_policy)");
  if (n && (!lease_id || !deliveries_out)) return fail(h, SDB_EINVAL, "sdb_lease_deliveries: lease_id or deliveries_out is NULL");
  for (uint64_t o = 0; o < n; o += SDB_LS_SETTLE_CHUNK) {
    const uint32_t m = static_cast<uint32_t>(std::min<uint64_t>(SDB_LS_SETTLE_CHUNK, n - o));
    CUDA_TRY(h, cudaMemcpyAsync(L.s.req, lease_id + o, m * sizeof(uint64_t), cudaMemcpyHostToDevice, h->stream));
    int nl = 0;
    cudaError_t e = sdb_launch_lease_deliveries(&L.buf[L.cur], &L.s, static_cast<uint32_t>(L.used), m, h->stream, &h->prof, &nl);
    h->launches += nl;
    if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("lease deliveries launch: ") + cudaGetErrorString(e));
    CUDA_TRY(h, cudaMemcpyAsync(deliveries_out + o, L.s.at, m * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  h->stream_busy = false;
  return SDB_OK;
}

int sdb_lease_dead_letters(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t flags,
                           uint32_t* count_out, sdb_recv_entry* entry_out, uint64_t entry_cap,
                           sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                           uint32_t* deliveries_out, uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out) {
  if (!h) return SDB_EINVAL;
  if (total_out) *total_out = 0;
  if (n_sends_out) *n_sends_out = 0;
  if (payload_bytes_out) *payload_bytes_out = 0;
  sdb_ctx::LeaseStore& L = h->lease;
  recv_agents(h, 0, agent_idx, &n_agents);
  if (count_out && n_agents <= h->cfg.max_agents) std::memset(count_out, 0, static_cast<size_t>(n_agents) * sizeof(uint32_t));
  if (flags & ~SDB_RECV_PEEK) return fail(h, SDB_EINVAL, "sdb_lease_dead_letters accepts SDB_RECV_PEEK only");
  if (!L.policy) return fail(h, SDB_EINVAL, "sdb_lease_dead_letters: no redelivery policy (sdb_lease_set_policy)");
  uint64_t rec_cap = 0;
  { const int rc = out_rec_cap(h, std::min(room(entry_out, entry_cap), room(send_out, send_cap)), room(payload_out, payload_cap), &rec_cap);
    if (rc != SDB_OK) return rc; }
  { const int rc = check_recv_agents(h, n_agents, agent_idx); if (rc != SDB_OK) return rc; }
  if (n_agents == 0 || L.dead == 0) return SDB_OK;
  { const int rc = compact_ensure(h); if (rc != SDB_OK) return rc; }
  const sdb_lease_buf& b = L.buf[L.cur];
  const uint32_t used = static_cast<uint32_t>(L.used), rows = static_cast<uint32_t>(L.rows);
  if (agent_idx)
    CUDA_TRY(h, cudaMemcpyAsync(h->rx_agent, agent_idx, static_cast<size_t>(n_agents) * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  int nl = 0;
  cudaError_t e = sdb_launch_lease_dl_select(&b, &L.s, &L.dl, used, agent_idx ? h->rx_agent : nullptr, n_agents, h->stream, &h->prof, &nl);
  h->launches += nl;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("dead-letter launch: ") + cudaGetErrorString(e));
  std::vector<uint32_t> cnt(n_agents);
  CUDA_TRY(h, cudaMemcpyAsync(cnt.data(), L.dl.cnt, static_cast<size_t>(n_agents) * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  { const int rc = lease_totals(h, 0, 1); if (rc != SDB_OK) return rc; }
  const uint64_t n_dead = L.th[0];
  // the receive capacity rule: agents in list order while they fit, or the lead agent alone with its first rec_cap
  uint64_t m = 0;
  uint32_t q = 0;
  for (; q < n_agents && m + cnt[q] <= rec_cap; ++q) m += cnt[q];
  if (q < n_agents && m == 0) { cnt[q] = static_cast<uint32_t>(rec_cap); m = rec_cap; ++q; }
  for (; q < n_agents; ++q) cnt[q] = 0;
  if (count_out) std::memcpy(count_out, cnt.data(), static_cast<size_t>(n_agents) * sizeof(uint32_t));
  if (m == 0) { h->stream_busy = false; return SDB_OK; }
  const bool take = !(flags & SDB_RECV_PEEK);
  uint32_t* dv = nullptr;
  nl = 0;
  e = sdb_launch_lease_dl_emit(&b, &L.s, &L.dl, rows, static_cast<uint32_t>(n_dead), static_cast<uint32_t>(m), n_agents, take ? 1u : 0u,
                               &h->cx, &dv, h->stream, &h->prof, &nl, h->sm_count);
  h->launches += nl;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("dead-letter launch: ") + cudaGetErrorString(e));
  { const int rc = lease_totals(h, 6, 2); if (rc != SDB_OK) return rc; }
  const uint64_t n_sends = L.th[6], pbytes = L.th[7] * SDB_GRANULE;
  if (entry_out) CUDA_TRY(h, cudaMemcpyAsync(entry_out, h->cx.entry_out, m * sizeof(sdb_recv_entry), cudaMemcpyDeviceToHost, h->stream));
  if (send_out) CUDA_TRY(h, cudaMemcpyAsync(send_out, h->cx.send_out, n_sends * sizeof(sdb_recv_send), cudaMemcpyDeviceToHost, h->stream));
  if (payload_out && pbytes) CUDA_TRY(h, cudaMemcpyAsync(payload_out, h->cx.payload_out, pbytes, cudaMemcpyDeviceToHost, h->stream));
  if (deliveries_out) CUDA_TRY(h, cudaMemcpyAsync(deliveries_out, dv, m * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  if (take) {                                   // the taken entries leave the store: compaction, as after a sweep
    nl = 0;
    e = sdb_launch_lease_compact(&b, &L.buf[L.cur ^ 1], &L.s, used, rows, 0u, 0u, 0.0, 0u, h->stream, &h->prof, &nl, h->sm_count);
    h->launches += nl;
    if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("dead-letter launch: ") + cudaGetErrorString(e));
    { const int rc = lease_totals(h, 8, 3); if (rc != SDB_OK) return rc; }
    L.cur ^= 1;
    L.used = L.th[8]; L.rows = L.th[9]; L.pay = L.th[10] * SDB_GRANULE;
    L.dead -= m; L.acked = 0;
  } else {
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  h->stream_busy = false;
  h->last_rx_valid = false; h->last_rx_compact = true;            // the compact receive's buffers were reused
  if (total_out) *total_out = m;
  if (n_sends_out) *n_sends_out = n_sends;
  if (payload_bytes_out) *payload_bytes_out = pbytes;
  return SDB_OK;
}

int sdb_lease_policy_stats(sdb_handle h, sdb_lease_policy_summary* out) {
  if (!h || !out) return SDB_EINVAL;
  const sdb_ctx::LeaseStore& L = h->lease;
  out->max_deliveries = L.max_deliveries; out->dead = L.dead; out->dead_total = L.dead_total;
  out->ledger_used = L.led_live; out->ledger_cap = L.led_cap; out->held_by_ledger_total = L.held_total;
  return SDB_OK;
}

// ---- snapshots of the lease store and the ledger -----------------------------------------------------------------
int sdb_lease_export(sdb_handle h, uint64_t start_id, uint32_t flags, sdb_recv_entry* entry_out, uint64_t entry_cap,
                     sdb_recv_send* send_out, uint64_t send_cap, uint8_t* payload_out, uint64_t payload_cap,
                     sdb_lease_meta* meta_out, uint64_t* total_out, uint64_t* n_sends_out, uint64_t* payload_bytes_out,
                     uint64_t* next_id_out) {
  if (!h) return SDB_EINVAL;
  if (total_out) *total_out = 0;
  if (n_sends_out) *n_sends_out = 0;
  if (payload_bytes_out) *payload_bytes_out = 0;
  if (next_id_out) *next_id_out = 0;
  sdb_ctx::LeaseStore& L = h->lease;
  if (flags) return fail(h, SDB_EINVAL, "sdb_lease_export: flags must be 0");
  if (!L.cap) return fail(h, SDB_EINVAL, "sdb_lease_export: no lease store (sdb_lease_reserve)");
  uint64_t rec_cap = 0;
  { const int rc = out_rec_cap(h, std::min({room(entry_out, entry_cap), room(meta_out, entry_cap), room(send_out, send_cap)}),
                               room(payload_out, payload_cap), &rec_cap);
    if (rc != SDB_OK) return rc; }
  if (next_id_out) *next_id_out = start_id;
  if (L.used == 0) return SDB_OK;
  { const int rc = compact_ensure(h); if (rc != SDB_OK) return rc; }
  const sdb_lease_buf& b = L.buf[L.cur];
  const uint32_t used = static_cast<uint32_t>(L.used), rows = static_cast<uint32_t>(L.rows);
  int nl = 0;
  cudaError_t e = sdb_launch_lease_x_select(&b, &L.s, used, start_id, h->stream, &h->prof, &nl);
  h->launches += nl;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("lease export launch: ") + cudaGetErrorString(e));
  { const int rc = lease_totals(h, 0, 1); if (rc != SDB_OK) return rc; }
  h->stream_busy = false;
  const uint64_t m = std::min<uint64_t>(L.th[0], rec_cap);
  if (m == 0) return SDB_OK;
  sdb_lease_meta* meta_dev = reinterpret_cast<sdb_lease_meta*>(h->rx_hdr);     // [max_recv_records] x 32 bytes
  nl = 0;
  e = sdb_launch_lease_x_emit(&b, &L.s, used, rows, static_cast<uint32_t>(m), &h->cx, meta_dev, h->stream, &h->prof, &nl, h->sm_count);
  h->launches += nl;
  h->last_rx_valid = false; h->last_rx_compact = true;            // the receive's buffers were reused
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("lease export launch: ") + cudaGetErrorString(e));
  { const int rc = lease_totals(h, 6, 3); if (rc != SDB_OK) return rc; }
  const uint64_t n_sends = L.th[6], pbytes = L.th[7] * SDB_GRANULE, next = L.th[8];
  if (entry_out) CUDA_TRY(h, cudaMemcpyAsync(entry_out, h->cx.entry_out, m * sizeof(sdb_recv_entry), cudaMemcpyDeviceToHost, h->stream));
  if (send_out) CUDA_TRY(h, cudaMemcpyAsync(send_out, h->cx.send_out, n_sends * sizeof(sdb_recv_send), cudaMemcpyDeviceToHost, h->stream));
  if (payload_out && pbytes) CUDA_TRY(h, cudaMemcpyAsync(payload_out, h->cx.payload_out, pbytes, cudaMemcpyDeviceToHost, h->stream));
  if (meta_out) CUDA_TRY(h, cudaMemcpyAsync(meta_out, meta_dev, m * sizeof(sdb_lease_meta), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->stream_busy = false;
  if (total_out) *total_out = m;
  if (n_sends_out) *n_sends_out = n_sends;
  if (payload_bytes_out) *payload_bytes_out = pbytes;
  if (next_id_out) *next_id_out = next;
  return SDB_OK;
}

int sdb_lease_import(sdb_handle h, uint64_t n, const sdb_recv_entry* entries, const sdb_recv_send* sends, uint64_t n_sends,
                     const uint8_t* payload, uint64_t payload_bytes, const sdb_lease_meta* meta, uint32_t flags,
                     uint64_t* lease_base_out) {
  if (!h) return SDB_EINVAL;
  if (lease_base_out) *lease_base_out = 0;
  sdb_ctx::LeaseStore& L = h->lease;
  if (flags) return fail(h, SDB_EINVAL, "sdb_lease_import: flags must be 0");
  if (!L.cap) return fail(h, SDB_EINVAL, "sdb_lease_import: no lease store (sdb_lease_reserve)");
  if ((n && (!entries || !meta)) || (n_sends && !sends) || (payload_bytes && !payload))
    return fail(h, SDB_EINVAL, "sdb_lease_import: null input array");
  const uint64_t rec_cap = recv_rec_cap(h);                  // the input is staged in one compact receive's buffers
  if (n > rec_cap || n_sends > rec_cap || payload_bytes > rec_cap * pad32(h->cfg.max_payload_bytes))
    return fail(h, SDB_ECAPACITY, "sdb_lease_import: input larger than one compact receive's capacity");
  const uint64_t grans = (payload_bytes + SDB_GRANULE - 1) / SDB_GRANULE;
  if (L.used + n > L.cap || L.rows + n_sends > L.cap || L.pay + grans * SDB_GRANULE > L.pay_cap)
    return fail(h, SDB_ECAPACITY, "lease store full: settle or sweep");
  if (n == 0) {
    if (lease_base_out) *lease_base_out = L.next_id;
    return SDB_OK;
  }
  { const int rc = compact_ensure(h); if (rc != SDB_OK) return rc; }
  sdb_compact_args& c = h->cx;
  sdb_lease_meta* meta_dev = reinterpret_cast<sdb_lease_meta*>(h->rx_hdr);
  h->last_rx_valid = false; h->last_rx_compact = true;            // the receive's buffers are reused
  CUDA_TRY(h, cudaMemcpyAsync(c.entry_out, entries, n * sizeof(sdb_recv_entry), cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(meta_dev, meta, n * sizeof(sdb_lease_meta), cudaMemcpyHostToDevice, h->stream));
  if (n_sends) CUDA_TRY(h, cudaMemcpyAsync(c.send_out, sends, n_sends * sizeof(sdb_recv_send), cudaMemcpyHostToDevice, h->stream));
  if (payload_bytes) CUDA_TRY(h, cudaMemcpyAsync(c.payload_out, payload, payload_bytes, cudaMemcpyHostToDevice, h->stream));
  int nl = 0;
  cudaError_t e = sdb_launch_lease_import_check(&L.s, &c, meta_dev, static_cast<uint32_t>(n), static_cast<uint32_t>(n_sends),
                                                payload_bytes, h->cfg.max_agents, h->cfg.max_payload_bytes, L.policy ? 1u : 0u,
                                                h->stream, &h->prof, &nl, h->sm_count);
  h->launches += nl;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("lease import launch: ") + cudaGetErrorString(e));
  { const int rc = lease_totals(h, 0, 1); if (rc != SDB_OK) return rc; }
  h->stream_busy = false;
  if (L.th[0])
    return fail(h, SDB_EINVAL, "sdb_lease_import: bad entry (send index, agent, receiver, state) or row (len, prio, payload_off)");
  const unsigned long long tot[3] = {n, n_sends, grans};          // the copy kernel reads its counts on the device
  CUDA_TRY(h, cudaMemcpyAsync(h->rx_totals, tot, sizeof(unsigned long long), cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(c.totals, tot + 1, 2 * sizeof(unsigned long long), cudaMemcpyHostToDevice, h->stream));
  nl = 0;
  e = sdb_launch_lease_import_write(&L.buf[L.cur], &c, meta_dev, h->rx_totals, static_cast<uint32_t>(n),
                                    std::max({n, n_sends, 2 * grans}), static_cast<uint32_t>(L.used), static_cast<uint32_t>(L.rows),
                                    L.pay, L.next_id, h->stream, &h->prof, &nl, h->sm_count);
  h->launches += nl;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("lease import launch: ") + cudaGetErrorString(e));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  uint64_t dead = 0;
  for (uint64_t i = 0; i < n; ++i) dead += meta[i].state == SDB_LEASE_STATE_DEAD ? 1 : 0;
  if (lease_base_out) *lease_base_out = L.next_id;
  L.used += n; L.rows += n_sends; L.pay += grans * SDB_GRANULE; L.next_id += n;
  L.live += n - dead; L.dead += dead;
  return SDB_OK;
}

// a collection of the ledger, synchronised: afterwards led_n = led_live = entries whose record is still pending
static int ledger_collect_sync(sdb_ctx* h) {
  sdb_ctx::LeaseStore& L = h->lease;
  if (!L.led_n) return SDB_OK;
  cudaError_t e = ledger_collect(h);
  if (e == cudaSuccess) e = cudaMemcpyAsync(L.lth, L.led.tot, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream);
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("ledger collection launch: ") + cudaGetErrorString(e));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  h->stream_busy = false;
  L.led_n = L.led_live = L.lth[0];
  return SDB_OK;
}

int sdb_lease_ledger_export(sdb_handle h, uint64_t cap, uint32_t* agent_out, uint64_t* seq_out, uint32_t* count_out,
                            uint64_t* n_out) {
  if (!h) return SDB_EINVAL;
  if (n_out) *n_out = 0;
  sdb_ctx::LeaseStore& L = h->lease;
  if (!L.policy) return fail(h, SDB_EINVAL, "sdb_lease_ledger_export: no redelivery policy (sdb_lease_set_policy)");
  { const int rc = ledger_collect_sync(h); if (rc != SDB_OK) return rc; }
  const uint64_t n = L.led_n;
  if (n_out) *n_out = n;
  if (n > cap) return fail(h, SDB_EOUTPUT, "sdb_lease_ledger_export: cap below the ledger's entries (*n_out)");
  if (n && (!agent_out || !seq_out || !count_out)) {
    if (n_out) *n_out = 0;
    return fail(h, SDB_EINVAL, "sdb_lease_ledger_export: null output array");
  }
  std::vector<sdb_ledger_ent> ent(n);
  if (n) {
    CUDA_TRY(h, cudaMemcpyAsync(ent.data(), L.led.ent, n * sizeof(sdb_ledger_ent), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  }
  for (uint64_t i = 0; i < n; ++i) { agent_out[i] = ent[i].agent; seq_out[i] = ent[i].seq; count_out[i] = ent[i].count; }
  return SDB_OK;
}

int sdb_lease_ledger_import(sdb_handle h, uint64_t n, const uint32_t* agent, const uint64_t* seq, const uint32_t* count,
                            uint64_t* matched_out) {
  if (!h) return SDB_EINVAL;
  if (matched_out) *matched_out = 0;
  sdb_ctx::LeaseStore& L = h->lease;
  if (!L.policy) return fail(h, SDB_EINVAL, "sdb_lease_ledger_import: no redelivery policy (sdb_lease_set_policy)");
  if (n && (!agent || !seq || !count)) return fail(h, SDB_EINVAL, "sdb_lease_ledger_import: null input array");
  for (uint64_t i = 0; i < n; ++i) {
    if (agent[i] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "sdb_lease_ledger_import: agent index out of range");
    if (!count[i]) return fail(h, SDB_EINVAL, "sdb_lease_ledger_import: a count of 0");
  }
  { const int rc = ledger_collect_sync(h); if (rc != SDB_OK) return rc; }
  if (n > L.led_cap - L.led_n) return fail(h, SDB_ECAPACITY, "sdb_lease_ledger_import: more triples than the ledger's free room");
  if (!n) return SDB_OK;
  std::vector<sdb_ledger_ent> t(n);                         // staged in the ledger's spare buffer (a collection rewrites it)
  for (uint64_t i = 0; i < n; ++i) t[i] = sdb_ledger_ent{seq[i], agent[i], count[i], 0u, 0u};
  CUDA_TRY(h, cudaMemcpyAsync(L.led.alt, t.data(), n * sizeof(sdb_ledger_ent), cudaMemcpyHostToDevice, h->stream));
  int nl = 0;
  cudaError_t e = sdb_launch_ledger_import(&h->view, &L.led, static_cast<uint32_t>(n), static_cast<uint32_t>(L.led_n), L.s.tot,
                                           h->stream, &h->prof, &nl, h->sm_count);
  h->launches += nl;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("ledger import launch: ") + cudaGetErrorString(e));
  { const int rc = lease_totals(h, 0, 1); if (rc != SDB_OK) return rc; }
  h->stream_busy = false;
  const uint64_t matched = L.th[0];
  L.led_n += matched; L.led_live += matched;
  if (matched_out) *matched_out = matched;
  return SDB_OK;
}

// sdb_receive_where and sdb_receive_where_budget (both limits 0: the plain filtered call); `name` names the call in errors
static int receive_where_full(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                              uint64_t max_agent_bytes, uint64_t max_agent_tokens, uint32_t flags, const sdb_filter* filter,
                              uint32_t* count_out, sdb_msg_header* hdr_out, uint64_t hdr_cap, uint8_t* payload_out,
                              uint64_t payload_cap, uint64_t* total_out, uint64_t* payload_bytes_out, const char* name) {
  if (!h) return SDB_EINVAL;
  if (total_out) *total_out = 0;
  if (payload_bytes_out) *payload_bytes_out = 0;
  const std::string n(name);
  where_req w;
  { const int rc = where_check(h, filter, name, &w); if (rc != SDB_OK) return rc; }
  if (flags & SDB_RECV_ASYNC) return fail(h, SDB_EINVAL, n + " returns host results: SDB_RECV_ASYNC is not accepted");
  if (flags & ~(SDB_RECV_PRIORITY | SDB_RECV_PEEK | SDB_RECV_OWNED | SDB_WHERE_DROP))
    return fail(h, SDB_EINVAL, n + " accepts SDB_RECV_PRIORITY, SDB_RECV_PEEK, SDB_RECV_OWNED and SDB_WHERE_DROP only");
  const bool drop = (flags & SDB_WHERE_DROP) != 0;
  if (drop && (hdr_out || payload_out)) return fail(h, SDB_EINVAL, n + ": drop mode takes no output buffers but count_out");
  const bool owned = recv_agents(h, flags, agent_idx, &n_agents);
  where_id_reset(w);
  if (n_agents == 0 || max_messages == 0) return SDB_OK;
  { const int rc = check_recv_agents(h, n_agents, agent_idx); if (rc != SDB_OK) return rc; }
  uint64_t rec_cap = ~0ull;
  if (!drop) {        // sdb_receive_batch's capacity rule
    const int rc = out_rec_cap(h, room(hdr_out, hdr_cap), room(payload_out, payload_cap), &rec_cap);
    if (rc != SDB_OK) return rc;
  }
  sdb_recv_args r{};
  { const int rc = recv_args(h, n_agents, agent_idx, owned, max_messages, flags & (SDB_RECV_PRIORITY | SDB_RECV_PEEK), rec_cap, &r);
    if (rc != SDB_OK) return rc; }
  int nl = 0;
  sdb_where_args f;
  { const int rc = where_setup(h, filter, w, &f, &nl); if (rc != SDB_OK) return rc; }
  cudaError_t e = sdb_launch_where(&h->view, &r, &f, drop ? 1 : 0, 32u + pad32(h->cfg.max_payload_bytes), h->stream, &nl,
                                   &h->prof, h->sm_count, nullptr, agent_gran_limit(max_agent_bytes), token_limit(max_agent_tokens));
  if (e == cudaSuccess) e = where_id_out(h, w, f, &nl);
  h->launches += nl;
  h->last_rx_valid = false; h->last_rx_compact = false;       // no full receive to fold: the plan belongs to a filtered call
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("filtered receive launch: ") + cudaGetErrorString(e));
  // drop mode has no output buffers, and its payload byte count stays 0; the synchronisation covers the id outputs
  return copy_full(h, n_agents, count_out, hdr_out, payload_out, total_out, drop ? nullptr : payload_bytes_out);
}

int sdb_receive_where(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages, uint32_t flags,
                      const sdb_filter* filter, uint32_t* count_out, sdb_msg_header* hdr_out, uint64_t hdr_cap,
                      uint8_t* payload_out, uint64_t payload_cap, uint64_t* total_out, uint64_t* payload_bytes_out) {
  return receive_where_full(h, n_agents, agent_idx, max_messages, 0, 0, flags, filter, count_out, hdr_out, hdr_cap, payload_out,
                            payload_cap, total_out, payload_bytes_out, "sdb_receive_where");
}

int sdb_receive_where_budget(sdb_handle h, uint32_t n_agents, const uint32_t* agent_idx, uint32_t max_messages,
                             uint64_t max_agent_bytes, uint64_t max_agent_tokens, uint32_t flags, const sdb_filter* filter,
                             uint32_t* count_out, sdb_msg_header* hdr_out, uint64_t hdr_cap, uint8_t* payload_out,
                             uint64_t payload_cap, uint64_t* total_out, uint64_t* payload_bytes_out) {
  return receive_where_full(h, n_agents, agent_idx, max_messages, max_agent_bytes, max_agent_tokens, flags, filter, count_out,
                            hdr_out, hdr_cap, payload_out, payload_cap, total_out, payload_bytes_out, "sdb_receive_where_budget");
}

int sdb_last_receive_dev(sdb_handle h, const uint32_t** count_dev, const sdb_msg_header** hdr_dev, const uint8_t** payload_dev) {
  if (!h) return SDB_EINVAL;
  if (count_dev) *count_dev = h->rx_count;
  if (hdr_dev) *hdr_dev = h->rx_hdr;
  if (payload_dev) *payload_dev = h->rx_payload;
  return SDB_OK;
}

int sdb_last_receive_totals(sdb_handle h, uint64_t* total_out, uint64_t* payload_bytes_out) {
  if (!h) return SDB_EINVAL;
  CUDA_TRY(h, cudaMemcpyAsync(h->totals_host, h->rx_totals, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (total_out) *total_out = h->totals_host[TOT_RECORDS];
  if (payload_bytes_out) *payload_bytes_out = h->totals_host[TOT_GRANULES] * SDB_GRANULE;
  return SDB_OK;
}

// ---- N3: inbox / load queries from the rings ---------------------------------------------------
int sdb_agent_loads(sdb_handle h, uint32_t n, const uint32_t* agent_idx, sdb_agent_load* out) {
  if (!h || (n && !out)) return SDB_EINVAL;
  if (n == 0) return SDB_OK;
  if (n > h->cfg.max_agents) return fail(h, SDB_EINVAL, "n > max_agents");
  if (agent_idx) {
    for (uint32_t i = 0; i < n; ++i) if (agent_idx[i] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "agent index out of range");
    CUDA_TRY(h, cudaMemcpyAsync(h->rx_agent, agent_idx, static_cast<size_t>(n) * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  }
  // the receive plan buffer doubles as scratch (32 bytes per agent; it holds max_recv_records + 4 16-byte entries)
  sdb_agent_load* tmp = nullptr;
  CUDA_TRY(h, cudaMallocAsync(reinterpret_cast<void**>(&tmp), static_cast<size_t>(n) * sizeof(sdb_agent_load), h->stream));
  cudaError_t e = sdb_launch_agent_loads(&h->view, agent_idx ? h->rx_agent : nullptr, n, tmp, h->sm_count, h->stream);
  h->launches += 1;
  if (e == cudaSuccess) e = cudaMemcpyAsync(out, tmp, static_cast<size_t>(n) * sizeof(sdb_agent_load), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaFreeAsync(tmp, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("agent loads: ") + cudaGetErrorString(e));
  return SDB_OK;
}

int sdb_queue_stats(sdb_handle h, sdb_queue_summary* out) {
  if (!h || !out) return SDB_EINVAL;
  unsigned long long* acc = h->be_scratch;                 // >= 16 words, free between picks
  cudaError_t e = sdb_launch_queue_stats(&h->view, h->n_agents, acc, h->stream);
  h->launches += 1;
  unsigned long long host[10];
  if (e == cudaSuccess) e = cudaMemcpyAsync(host, acc, sizeof(host), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("queue stats: ") + cudaGetErrorString(e));
  out->agents_with_pending = host[0]; out->pending = host[1];
  for (int k = 0; k < 4; ++k) out->pending_by_prio[k] = host[2 + k];
  out->pending_granules = host[6]; out->received = host[7];
  out->max_pending = host[8] >> 32; out->max_pending_agent = host[8] ? 0xFFFFFFFFull - (host[8] & 0xFFFFFFFFull) : 0;
  return SDB_OK;
}

int sdb_assign_agent_backends(sdb_handle h, uint32_t n, const uint32_t* agent_idx, const uint32_t* backend_idx) {
  if (!h || (n && (!agent_idx || !backend_idx))) return SDB_EINVAL;
  if (!h->agent_backend_dev) {
    CUDA_TRY(h, dmalloc(&h->agent_backend_dev, h->cfg.max_agents));
    CUDA_TRY(h, cudaMemsetAsync(h->agent_backend_dev, 0xFF, static_cast<size_t>(h->cfg.max_agents) * sizeof(uint32_t), h->stream));
  }
  for (uint32_t i = 0; i < n; ++i) {
    if (agent_idx[i] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "agent index out of range");
    if (backend_idx[i] != 0xFFFFFFFFu && backend_idx[i] >= h->cfg.max_backends) return fail(h, SDB_ENOTFOUND, "backend index out of range");
    // assignments are rare and small (one per agent when it first asks): element-wise stream-ordered copies
    CUDA_TRY(h, cudaMemcpyAsync(h->agent_backend_dev + agent_idx[i], backend_idx + i, sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  }
  if (n) CUDA_TRY(h, cudaStreamSynchronize(h->stream));     // the source array is the caller's
  return SDB_OK;
}

int sdb_backend_loads_from_queues(sdb_handle h) {
  if (!h) return SDB_EINVAL;
  if (h->n_backends == 0) return fail(h, SDB_ENOTFOUND, "no backends configured (sdb_set_backends)");
  if (!h->agent_backend_dev) return fail(h, SDB_ENOTFOUND, "no agent is assigned to a backend (sdb_assign_agent_backends)");
  cudaError_t e = sdb_launch_backend_loads_from_queues(&h->view, h->n_agents, h->agent_backend_dev, h->n_backends, h->be_load, h->stream);
  h->launches += 1;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("backend loads: ") + cudaGetErrorString(e));
  return SDB_OK;
}

// ---- stream digests -------------------------------------------------------------------------
static int digest_ensure(sdb_ctx* h) {
  if (h->digest) return SDB_OK;
  { const int rc = dmalloc_set(h, {{&h->digest, h->cfg.max_agents}}, "stream digests: device allocation failed"); if (rc != SDB_OK) return rc; }
  CUDA_TRY(h, cudaMemsetAsync(h->digest, 0, static_cast<size_t>(h->cfg.max_agents) * sizeof(unsigned long long), h->stream));
  return SDB_OK;
}

int sdb_digest_reset(sdb_handle h) {
  if (!h) return SDB_EINVAL;
  int rc = digest_ensure(h);
  if (rc != SDB_OK) return rc;
  CUDA_TRY(h, cudaMemsetAsync(h->digest, 0, static_cast<size_t>(h->cfg.max_agents) * sizeof(unsigned long long), h->stream));
  return SDB_OK;
}

int sdb_digest_fold(sdb_handle h) {
  if (!h) return SDB_EINVAL;
  if (h->last_rx_compact) return fail(h, SDB_EINVAL, "sdb_digest_fold: the last receive was compact (sdb_receive_compact writes no full-format device results)");
  if (!h->last_rx_valid) return fail(h, SDB_EINVAL, "sdb_digest_fold: no bulk receive to fold (the <= 8-agent latency path keeps no device results)");
  int rc = digest_ensure(h);
  if (rc != SDB_OK) return rc;
  cudaError_t e = sdb_launch_digest(&h->last_rx, h->cfg.max_agents, h->digest, h->sm_count, h->stream);
  h->launches += 1;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("digest launch: ") + cudaGetErrorString(e));
  return SDB_OK;
}

int sdb_digest_read(sdb_handle h, uint32_t n, const uint32_t* agent_idx, uint64_t* digest_out) {
  if (!h || (n && !digest_out)) return SDB_EINVAL;
  if (n == 0) return SDB_OK;
  int rc = digest_ensure(h);
  if (rc != SDB_OK) return rc;
  if (!agent_idx) {
    if (n > h->cfg.max_agents) return fail(h, SDB_EINVAL, "n > max_agents");
    CUDA_TRY(h, cudaMemcpyAsync(digest_out, h->digest, static_cast<size_t>(n) * sizeof(uint64_t), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    return SDB_OK;
  }
  std::vector<unsigned long long> all(h->cfg.max_agents);
  CUDA_TRY(h, cudaMemcpyAsync(all.data(), h->digest, all.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  for (uint32_t i = 0; i < n; ++i) {
    if (agent_idx[i] >= h->cfg.max_agents) return fail(h, SDB_EINVAL, "agent index out of range");
    digest_out[i] = all[agent_idx[i]];
  }
  return SDB_OK;
}

// ---- backends -----------------------------------------------------------------------------
int sdb_set_backends(sdb_handle h, uint32_t n, const uint32_t* weight, const uint64_t* load0) {
  if (!h || !weight || n == 0) return SDB_EINVAL;
  if (n > h->cfg.max_backends) return fail(h, SDB_ECAPACITY, "n > max_backends");
  std::vector<unsigned long long> l(n, 0);
  for (uint32_t i = 0; i < n; ++i) {
    if (weight[i] == 0 || weight[i] > 65535) return fail(h, SDB_EINVAL, "backend weight must be in [1, 65535]");
    if (load0) { if (load0[i] >= (1ull << 40)) return fail(h, SDB_EINVAL, "backend load must be < 2^40"); l[i] = load0[i]; }
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  CUDA_TRY(h, upload(h, h->be_weight, weight, n * sizeof(uint32_t)));
  CUDA_TRY(h, upload(h, h->be_load, l.data(), n * sizeof(unsigned long long)));
  h->n_backends = n;
  return SDB_OK;
}

int sdb_get_backend_loads(sdb_handle h, uint32_t n, uint64_t* load_out) {
  if (!h || !load_out || n > h->n_backends) return SDB_EINVAL;
  CUDA_TRY(h, cudaMemcpyAsync(load_out, h->be_load, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return SDB_OK;
}

static int ensure_req_cap(sdb_ctx* h, uint32_t n) {
  if (n <= h->be_req_cap) return SDB_OK;
  { int rcl = ls_stop(h); if (rcl != SDB_OK) return rcl; }      // cudaFree below waits for running kernels
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (h->be_req_cost) cudaFree(h->be_req_cost);
  if (h->be_out) cudaFree(h->be_out);
  h->be_req_cost = nullptr; h->be_out = nullptr; h->be_req_cap = 0;
  CUDA_TRY(h, dmalloc(&h->be_req_cost, n));
  CUDA_TRY(h, dmalloc(&h->be_out, n));
  h->be_req_cap = n;
  return SDB_OK;
}

int sdb_release_backends(sdb_handle h, uint32_t n, const uint32_t* backend, const uint32_t* cost) {
  if (!h || (n && !backend)) return SDB_EINVAL;
  if (n == 0) return SDB_OK;
  // completion reports are rare and small: fold them on the host, apply as one device update
  std::vector<unsigned long long> l(h->n_backends);
  CUDA_TRY(h, cudaMemcpyAsync(l.data(), h->be_load, h->n_backends * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  for (uint32_t i = 0; i < n; ++i) {
    if (backend[i] >= h->n_backends) return fail(h, SDB_ENOTFOUND, "backend index out of range");
    const unsigned long long c = cost ? cost[i] : 1;
    l[backend[i]] = l[backend[i]] >= c ? l[backend[i]] - c : 0;
  }
  CUDA_TRY(h, upload(h, h->be_load, l.data(), h->n_backends * sizeof(unsigned long long)));
  return SDB_OK;
}

int sdb_select_backend_batch(sdb_handle h, uint32_t n_req, const uint32_t* cost, uint32_t mode, uint64_t seed, uint32_t* backend_out) {
  if (!h || !backend_out) return SDB_EINVAL;
  if (mode > 1) return fail(h, SDB_EINVAL, "mode must be 0 (least-load) or 1 (weighted random)");
  if (h->n_backends == 0) return fail(h, SDB_ENOTFOUND, "no backends configured (sdb_set_backends)");
  if (n_req == 0) return SDB_OK;
  int rc = ensure_req_cap(h, n_req);
  if (rc != SDB_OK) return rc;
  if (cost) CUDA_TRY(h, cudaMemcpyAsync(h->be_req_cost, cost, static_cast<size_t>(n_req) * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
  int nl = 0;
  cudaError_t e = sdb_launch_pick(static_cast<int>(mode), h->n_backends, h->be_weight, h->be_load, n_req,
                                  cost ? h->be_req_cost : nullptr, seed, h->be_out, h->be_scratch, h->be_logtab,
                                  h->stream, &nl);
  h->launches += nl;
  h->picks += n_req;
  if (e != cudaSuccess) return fail(h, SDB_ECUDA, std::string("backend pick: ") + cudaGetErrorString(e));
  CUDA_TRY(h, cudaMemcpyAsync(backend_out, h->be_out, static_cast<size_t>(n_req) * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return SDB_OK;
}

}  // extern "C"
