// host.cuh -- what the units of libdint_b200.so share on the host side: the error state, the size tables, the engine,
// the ranks of the multi-GPU step and the cluster, and the internals one unit calls in another.  Everything else is
// static in its unit.  The units:
//   engine.cu   the engine: create / destroy, the chunk launches, the host ring, submit / sync, snapshots, stats
//   step.cu     the C routing ABI, the multi-GPU step (dint_shard_*) and clusters (dint_cluster_*)
//   derive.cu   shards filled from other shards: re-shard and rebuild
//   image.cu    engine and cluster state images
//   kv_host.cu  load, populate and inspection of the KV tables, lock state and the log
//   clients.cu  the closed-loop clients on the GPU (dint_clients_*, dint_txn_clients_*, dint_cluster_clients_*)
#pragma once
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/dint_b200.h"
#include "kv.cuh"

using namespace dint;

extern thread_local std::string g_last_error;        // dint_last_error (engine.cu)
inline int set_err(int code, const char* what, cudaError_t ce = cudaSuccess) {
  char buf[1024];
  if (ce != cudaSuccess) snprintf(buf, sizeof buf, "%s: %s", what, cudaGetErrorString(ce));
  else snprintf(buf, sizeof buf, "%s", what);
  g_last_error = buf;
  return code;
}
template <typename... Args>
int set_errf(int code, const char* fmt, Args... args) {
  char buf[1024];
  snprintf(buf, sizeof buf, fmt, args...);
  return set_err(code, buf);
}
#define CU(call)                                                              \
  do {                                                                        \
    cudaError_t _e = (call);                                                  \
    if (_e != cudaSuccess) return set_err(_e == cudaErrorMemoryAllocation ? DINT_ENOMEM : DINT_EIO, #call, _e); \
  } while (0)

// returns rc after cleanup(), with dint_last_error left as the failure set it (the cleanup may overwrite it)
template <class F>
int keep_error(int rc, F&& cleanup) {
  std::string keep = g_last_error;
  cleanup();
  g_last_error = keep;
  return rc;
}

// seconds on the steady clock: the timers of dint_image_times, dint_reshard_times and dint_rebuild_times
inline double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

constexpr uint32_t kMsgSize[DINT_NUM_KINDS] = {6, 9, 53, 53, 55, 23};
constexpr uint32_t kLogEntry[DINT_NUM_KINDS] = {0, 0, 56, 0, 64, 32};
constexpr uint32_t kValSize[DINT_NUM_KINDS] = {0, 0, 0, 40, 40, 8};

// Kernel kind of a store engine with the eBPF cache tier: not a public dint_kind, so the store's own kernels are
// instantiated exactly as before and the tier's only when an engine asks for it (see exec_kind).
constexpr int kExecStoreEbpf = DINT_NUM_KINDS;
// ... and of a tatp engine with the eBPF cache tier (DINT_CFG_TATP_EBPF)
constexpr int kExecTatpEbpf = DINT_NUM_KINDS + 1;
// ... and of a smallbank engine with the eBPF cache tier (DINT_CFG_SMALLBANK_EBPF)
constexpr int kExecSmallbankEbpf = DINT_NUM_KINDS + 2;

// The one place where an engine's run-time kind picks the kernel templates: calls f(std::integral_constant<int, K>{})
// and returns what f returns.  Record-size-keyed kernels are instantiated with Wire<K>::MSG.
template <class F>
int with_kind(int kind, F&& f) {
  switch (kind) {
    case DINT_LOCK2PL: return f(std::integral_constant<int, K_LOCK2PL>{});
    case DINT_FASST: return f(std::integral_constant<int, K_FASST>{});
    case DINT_LOG: return f(std::integral_constant<int, K_LOG>{});
    case DINT_STORE: return f(std::integral_constant<int, K_STORE>{});
    case DINT_TATP: return f(std::integral_constant<int, K_TATP>{});
    case DINT_SMALLBANK: return f(std::integral_constant<int, K_SMALLBANK>{});
    case kExecStoreEbpf: return f(std::integral_constant<int, K_STORE_EBPF>{});
    case kExecTatpEbpf: return f(std::integral_constant<int, K_TATP_EBPF>{});
    case kExecSmallbankEbpf: return f(std::integral_constant<int, K_SMALLBANK_EBPF>{});
  }
  return set_err(DINT_EINVAL, "bad kind");
}

// Where the replies of one run_device call go when they are not one contiguous array: inside the multi-GPU step the
// batch is W source slabs of seg_tiles tiles each, and the replies of slab s go straight into source s's return buffer.
struct StepTarget {
  uint32_t seg_tiles;                 // tiles per source slab
  uint64_t seg_resp[kMaxShards];      // reply slab of source s (device address, possibly peer memory)
  bool pad_ok;                        // type 0xFE records are slab padding (else: invalid)
  const uint32_t* skip;               // non-zero: a slab overflowed, serve nothing more (see k_p2p_wait)
};

enum { KT_CLASSIFY = 0, KT_LOGSCAN, KT_APPLY, KT_ORDERED, KT_LOAD, KT_NUM };

struct EvPair { cudaEvent_t a, b; int which; };
constexpr int kHostBufs = 4;      // staging sets of dint_submit, and the most any host-path caller uses
// Device staging of the host paths, dint_submit's slices and the multi-GPU step's batches: batch j of a call uses set
// b = j % sets, with H2D on s_in and D2H on s_out next to the compute.  The caller records released[b] behind the last
// launch that reads in[b] / aux[b], and makes the launch that writes out[b] wait for d2h[b] once j >= sets.
// dint_submit and the step share the ring because one engine never has both in flight: dint_submit begins with a
// device synchronise, and shard_run with host buffers ends by synchronising its copy and main streams.
struct HostRing {
  struct Buf { uint8_t* p = nullptr; size_t cap = 0; };
  Buf in[kHostBufs], aux[kHostBufs], out[kHostBufs];   // requests | client-chosen destination bytes (the step) | replies
  cudaEvent_t h2d[kHostBufs]{}, released[kHostBufs]{}, ready[kHostBufs]{}, d2h[kHostBufs]{};
  cudaStream_t s_in = nullptr, s_out = nullptr;
  uint32_t sets = 0;                                    // of the current call (buffers are allocated on first use, then only grow)
};

struct dint_engine {
  int kind = 0;
  int device = 0;
  dint_cfg cfg{};
  uint32_t msg = 0;
  uint32_t chunk = 0;
  uint32_t max_tiles = 0;
  bool has_log = false;
  Ctx ctx{};                       // device pointers + constants; per-launch fields filled per chunk
  std::vector<void*> allocs;       // everything to cudaFree
  cudaStream_t stream = nullptr;
  HostRing ring;                             // host-path staging of dint_submit and the multi-GPU step
  uint32_t host_chunk = 0;                   // requests per host-path slice
  bool plain_launches = false;               // inside the multi-GPU step: no cooperative launches (see GridBar)
  uint32_t host_min_slice = 0;               // smallest slice of the pyramid a host-path call is cut into
  bool host_ramp_up = true;
  unsigned long long* h_counters = nullptr;  // pinned mirror of ctx.counters (host path reads it without a blocking copy)
  unsigned long long* h_kvcnt = nullptr;     // pinned mirror of every table's {live, used} (kv_maintain)
  cudaEvent_t ev_kvcnt = nullptr;
  int coop_grid = 0;
  int sms = 0;
  int grid_classify = 0, grid_apply = 0;     // persistent CTAs (SMs x resident CTAs per SM)
  uint32_t smem_stage = 0;                   // dynamic shared memory of K1/K2: kStages staged tiles
  uint64_t total_groups = 0;
  uint32_t* d_flags[2] = {nullptr, nullptr}; // flag-nibble sets, alternating per chunk
  uint32_t* d_grp[2] = {nullptr, nullptr};   // group ids of the current / previous chunk
  uint64_t chunk_seq = 0;
  uint32_t prev_n = 0;                       // requests of the previous chunk whose flags are still set
  bool ord_pending = false;                  // the previous chunk's listed requests await their replay
  uint8_t* ord_resp = nullptr;               //   ... and live in this reply array
  const uint8_t* ord_req = nullptr;          //   ... their request bytes in this one
  uint32_t ord_tile0 = 0;                    //   ... which starts at this tile of its batch
  uint32_t smem_classify = 0;                // K1: max(stages, ordered-replay slices)
  uint32_t* d_nc = nullptr;                  // [2 chunks][2]: listed / overflow counters
  uint32_t* d_route = nullptr;               // multi-GPU dispatch scratch (per-tile per-shard counts)
  uint32_t route_tiles = 0;
  uint32_t* d_route2 = nullptr;              // dispatch scratch: counters, totals, look-back descriptors
  uint32_t route_desc_tiles = 0, route_seq = 0;
  int grid_route = 0;                        // CTAs of k_route_dispatch: 4 per SM are resident (64 registers x 256 threads)
                                             // (tiles are drawn by ticket, so any grid is correct)
  // L2 persistence: the flag sets (+ lock_fasst lock bits) live in one arena that every launch maps
  // with a persisting access-policy window, so the streaming request/reply traffic cannot evict it
  uint8_t* hot_arena = nullptr;
  size_t hot_bytes = 0;
  bool use_window = false;
  cudaAccessPolicyWindow window{};
  // stats
  dint_stats stats{};
  // profiling
  uint32_t profiling = 0;          // bit k set: bracket launches of kernel k (KT_*) with CUDA events
  std::vector<EvPair> ev_pool;
  size_t ev_used = 0;
  double kt_ms[KT_NUM] = {0};
  uint64_t kt_n[KT_NUM] = {0};
  // KV host mirrors
  KvHost kv[kMaxTables];
};

// a smallbank engine with the eBPF cache tier (its sets live in ctx.ecache, as the store's do)
inline bool sbe_on(const dint_engine* e) { return e->kind == DINT_SMALLBANK && e->ctx.ecache; }
// the kind whose kernels serve this engine: its public kind, or the store's / tatp's / smallbank's cache-tier kind
inline int exec_kind(const dint_engine* e) {
  return e->ctx.tchain ? kExecTatpEbpf : sbe_on(e) ? kExecSmallbankEbpf : e->ctx.ecache ? kExecStoreEbpf : e->kind;
}

int prof_flush(dint_engine* e);
struct ProfScope {
  dint_engine* e; cudaStream_t s; EvPair* p = nullptr;
  ProfScope(dint_engine* e_, cudaStream_t s_, int which) : e(e_), s(s_) {
    e->stats.kernel_launches++;
    if (!((e->profiling >> which) & 1u)) return;
    if (e->ev_used == e->ev_pool.size()) {
      if (e->ev_pool.size() >= 8192) { prof_flush(e); }
      else {
        EvPair np{}; cudaEventCreate(&np.a); cudaEventCreate(&np.b);
        e->ev_pool.push_back(np);
      }
    }
    p = &e->ev_pool[e->ev_used++];
    p->which = which;
    cudaEventRecord(p->a, s);
  }
  ~ProfScope() { if (p) cudaEventRecord(p->b, s); }
};

template <typename... Args>
cudaError_t launch_ex(dint_engine* e, void (*kern)(Args...), int grid, int block, size_t smem, cudaStream_t s,
                             bool coop, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid < 1 ? 1 : grid);
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[3];
  int na = 0;
  if (coop) { at[na].id = cudaLaunchAttributeCooperative; at[na].val.cooperative = 1; na++; }
  if (e->use_window) { at[na].id = cudaLaunchAttributeAccessPolicyWindow; at[na].val.accessPolicyWindow = e->window; na++; }
  cfg.attrs = at;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kern, args...);
}

// an engine being made from state held elsewhere (an image, a re-shard, a rebuild): destroyed unless released
struct EngineOwner {
  dint_engine* e;
  ~EngineOwner() { if (e) dint_destroy(e); }
};

// ---- engine.cu ----------------------------------------------------------------------------------------------
// DINT_EINVAL unless each DINT_CFG_* flag of `flags` is an option of `kind`
int check_kind_flags(int kind, uint32_t flags);
int kv_publish_counts(dint_engine* e, cudaStream_t s);
int engine_ready(dint_engine* e);
int run_device(dint_engine* e, const uint8_t* req, uint64_t n, uint8_t* resp, cudaStream_t s, const StepTarget* tgt = nullptr);
int pull_counters(dint_engine* e);
int ring_reserve(dint_engine* e, uint32_t sets, size_t in_bytes, size_t aux_bytes, size_t out_bytes);
int ring_stage_in(dint_engine* e, uint64_t j, const void* host_in, size_t in_bytes, const void* host_aux, size_t aux_bytes, cudaStream_t consumer);
int ring_drain_out(dint_engine* e, uint64_t j, void* host_out, size_t out_bytes, cudaStream_t producer);
void snapshot_regions(dint_engine* e, std::vector<std::pair<void*, size_t>>& r);

// ---- step.cu ------------------------------------------------------------------------------------------------
// one rank of the multi-GPU step: one engine and its view of every rank's exchange buffers
constexpr int kMaxSets = 4;
static_assert(kMaxSets <= kHostBufs, "the host path stages batch j in set j % n_sets of the engine's HostRing");
struct dint_shard_ctx {
  dint_engine* e = nullptr;
  uint32_t W = 0, me = 0, cap = 0, S = 0;
  uint64_t inbox[kMaxSets][kMaxShards]{}, retbox[kMaxSets][kMaxShards]{};
  PeerPtrs sigreq{}, sigrsp{};
  uint32_t *my_req = nullptr, *my_rsp = nullptr;
  uint32_t epoch = 0;
  cudaStream_t side = nullptr, ret = nullptr;
  cudaEvent_t ev_disp[kMaxSets]{}, ev_comb[kMaxSets]{}, ev_fork = nullptr;
  uint8_t* owner[kMaxSets]{};
  uint32_t* tilebase[kMaxSets]{};
  uint32_t* flags = nullptr;
  uint64_t max_n = 0;
  bool one_stream = false;                 // ranks sharing a device: dispatch, engine and combine on ONE stream, in dependency order
  bool trace = false;                      // DINT_SHARD_TRACE: per-phase CUDA-event timing, printed at destroy
  std::vector<cudaEvent_t> tev;            // 6 events per batch
  double tsum[4]{};
  uint64_t tcount = 0;
};

struct ShardBatch { const void* req; const uint8_t* dst; void* out; uint64_t n; uint32_t cap = 0; };   // cap: slab records of this batch (0 = the full capacity)
struct HostBatch { const uint8_t* req; const uint8_t* dst; uint8_t* out; uint64_t n; };
int shard_run(dint_shard_ctx* const* ranks, uint32_t R, uint32_t k, std::vector<std::vector<ShardBatch>>& b, cudaStream_t const* mains,
              const std::vector<std::vector<HostBatch>>* host = nullptr);

// ---- dint_cluster_*: G shards driven by ONE process (SURVEY.md 8(b): dint_create(kind, cfg, n_gpus) / dint_submit(..., dst_shard, ...)) ----
struct dint_cluster {
  int kind = 0;
  uint32_t G = 0, cap = 0;
  uint64_t max_n = 0;
  bool by_dst = false, shared_device = false;
  std::vector<int> dev;
  std::vector<dint_engine*> eng;
  std::vector<dint_shard_ctx*> sh;
  std::vector<void*> bufs;                  // per rank: one allocation {inbox sets | return-buffer sets | signal block}
  uint64_t overflow_retries = 0;            // submit calls that met a slab overflow and served the rest in small rounds
  dint_cfg base{};                          // the configuration the shards were made from (the image manifest keeps it)
  uint32_t txn_clients = 0;                 // dint_txn_clients attached (dint_cluster_rebuild refuses while there are any)
};

uint64_t cluster_sig_block(const dint_cluster* cl, uint32_t r);
dint_cfg cluster_shard_cfg(const dint_cluster* cl, uint32_t r);
int cluster_ranks(const dint_cluster* cl, const std::vector<dint_engine*>& eng, std::vector<dint_shard_ctx*>& out);
// the shards a re-shard or rebuild reads
struct DeriveFrom {
  std::vector<dint_engine*> src;                    // per source shard: its engine (nullptr where a rebuild lost it)
  uint64_t rows[kMaxShards][kMaxTables] = {};        // the rows each destination shard receives, per table (count_rows)
};
int cluster_make(int kind, const dint_cfg* cfg, int n_gpus, const int* devices, uint64_t max_batch, const char* image_dir,
                 const DeriveFrom* from, uint32_t* rebuild, dint_cluster** out);

// ---- derive.cu ----------------------------------------------------------------------------------------------
extern thread_local double g_rebuild_times[3];
int peer_enable(int device, int peer);
int cluster_quiesce(const dint_cluster* cl);
int reshard_engine(const DeriveFrom& f, uint32_t j, uint32_t G2, int kind, const dint_cfg& c, int device, dint_engine** out);
std::string mask_names(uint32_t mask);
int rebuild_check(int kind, const dint_cfg& cfg, uint32_t G, uint32_t lost);
int rebuild_shards(dint_cluster* cl, uint32_t lost);

// ---- image.cu -----------------------------------------------------------------------------------------------
int image_open_impl(const char* path, int device, const dint_cfg* want, dint_engine** out);
std::string img_shard_path(const char* dir, uint32_t r);
