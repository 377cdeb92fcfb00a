// engine.cu -- host side of libdint_b200.so: state allocation in HBM, the per-chunk launch sequence,
// host<->device pipelining for dint_submit(), state inspection, and the extern "C" ABI of
// include/dint_b200.h.  No CPU implementation of the request path exists here: without a CUDA
// device every compute entry point returns DINT_ENODEV.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <algorithm>
#include <chrono>
#include <type_traits>
#include <vector>
#include <cerrno>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include "../../include/dint_b200.h"
#include "kernels.cuh"
#include "route.cuh"
#include "kv.cuh"
#include "clients.cuh"
#include "txn_clients.cuh"
#include "image.cuh"
#include "reshard.cuh"
#include "rebuild.cuh"

using namespace dint;

static thread_local std::string g_last_error;
static int set_err(int code, const char* what, cudaError_t ce = cudaSuccess) {
  char buf[1024];
  if (ce != cudaSuccess) snprintf(buf, sizeof buf, "%s: %s", what, cudaGetErrorString(ce));
  else snprintf(buf, sizeof buf, "%s", what);
  g_last_error = buf;
  return code;
}
template <typename... Args>
static int set_errf(int code, const char* fmt, Args... args) {
  char buf[1024];
  snprintf(buf, sizeof buf, fmt, args...);
  return set_err(code, buf);
}
#define CU(call)                                                              \
  do {                                                                        \
    cudaError_t _e = (call);                                                  \
    if (_e != cudaSuccess) return set_err(_e == cudaErrorMemoryAllocation ? DINT_ENOMEM : DINT_EIO, #call, _e); \
  } while (0)

static const uint32_t kMsgSize[DINT_NUM_KINDS] = {6, 9, 53, 53, 55, 23};
static const uint32_t kLogEntry[DINT_NUM_KINDS] = {0, 0, 56, 0, 64, 32};
static const uint32_t kValSize[DINT_NUM_KINDS] = {0, 0, 0, 40, 40, 8};

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
static int with_kind(int kind, F&& f) {
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
static const char* kKernelNames[KT_NUM] = {"k_classify", "k_log_scan", "k_apply", "k_ordered", "k_kv_load"};

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
static bool sbe_on(const dint_engine* e) { return e->kind == DINT_SMALLBANK && e->ctx.ecache; }
// the kind whose kernels serve this engine: its public kind, or the store's / tatp's / smallbank's cache-tier kind
static int exec_kind(const dint_engine* e) {
  return e->ctx.tchain ? kExecTatpEbpf : sbe_on(e) ? kExecSmallbankEbpf : e->ctx.ecache ? kExecStoreEbpf : e->kind;
}

template <typename T>
static int dalloc(dint_engine* e, T** p, size_t count, bool zero = true) {
  size_t bytes = count * sizeof(T);
  if (bytes == 0) bytes = sizeof(T);
  void* q = nullptr;
  CU(cudaMalloc(&q, bytes));
  e->allocs.push_back(q);
  if (zero) CU(cudaMemsetAsync(q, 0, bytes, e->stream));
  *p = (T*)q;
  return DINT_OK;
}

// ---- profiling helpers ------------------------------------------------------------------------------
static int prof_flush(dint_engine* e) {
  for (size_t i = 0; i < e->ev_used; i++) {
    float ms = 0;
    CU(cudaEventSynchronize(e->ev_pool[i].b));
    CU(cudaEventElapsedTime(&ms, e->ev_pool[i].a, e->ev_pool[i].b));
    e->kt_ms[e->ev_pool[i].which] += ms;
    e->kt_n[e->ev_pool[i].which]++;
  }
  e->ev_used = 0;
  return DINT_OK;
}
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

// ---- per-chunk launch sequence ------------------------------------------------------------------------
template <typename... Args>
static cudaError_t launch_ex(dint_engine* e, void (*kern)(Args...), int grid, int block, size_t smem, cudaStream_t s,
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

// One chunk: K1 (classify this chunk + replay the previous chunk's listed requests), K2 (apply), and the
// fallback launch that only does work when one of THIS chunk's buckets overflowed.  c.n == 0 = flush: K1
// alone, replaying the last chunk's listed requests.
template <int KIND>
static int launch_chunk_t(dint_engine* e, const Ctx& c, cudaStream_t s) {
  {
    ProfScope ps(e, s, KT_CLASSIFY);
    int want = (int)c.n_tiles, clr = (int)((c.prev_n + 4 * kTile - 1) / (4 * kTile));
    if (clr > want) want = clr;
    int grid = (want < e->grid_classify && !c.ord_pending) ? want : e->grid_classify;
    if (c.n == 0 && e->sms > 0 && grid > 8 * e->sms) grid = 8 * e->sms;     // a flush launch only replays: 32 warps per SM are plenty
    CU(launch_ex(e, k_classify<KIND>, grid, kTile, e->smem_classify, s, false, c));
  }
  if (c.n == 0) { CU(cudaGetLastError()); return DINT_OK; }
  if (kHasLog<KIND>) {
    ProfScope ps(e, s, KT_LOGSCAN);
    k_log_scan<<<1, kThreads, 0, s>>>(c);
  }
  {
    ProfScope ps(e, s, KT_APPLY);
    int grid = (int)c.n_tiles < e->grid_apply ? (int)c.n_tiles : e->grid_apply;
    CU(launch_ex(e, k_apply<KIND>, grid, kTile, e->smem_stage, s, false, c));
  }
  if ((KIND == K_TATP || KIND == K_TATP_EBPF) && c.n > c.ring_n) {                // (a chunk appends at most n entries: none can be skipped otherwise)
    int grid = (int)((c.ring_n + kThreads - 1) / kThreads);   // the last ring_n appends end every slot's history
    if (e->sms > 0 && grid > 4 * e->sms) grid = 4 * e->sms;
    k_log_vals<<<grid, kThreads, 0, s>>>(c);
    e->stats.kernel_launches++;
  }
  if (KIND != K_LOG) {   // the log server has no per-key state: nothing to order
    ProfScope ps(e, s, KT_ORDERED);
    Ctx f = c;           // this chunk's own counters / replies
    f.nc_ord = c.nc_cur;
    f.ord_resp = c.resp;
    f.ord_req = c.req;
    f.ord_tile0 = c.tile0;
    f.coop_launch = e->plain_launches ? 0u : 1u;
    int g3 = e->coop_grid;
    if (e->plain_launches && e->sms > 0) {             // leave room for the one-warp flag-polling kernels of the other streams
      const int per = g3 / e->sms;
      g3 = (per > 1 ? per - 1 : 1) * e->sms;
    }
    CU(launch_ex(e, k_ordered<KIND>, g3, kThreads, 0, s, !e->plain_launches, f));
  }
  CU(cudaGetLastError());
  return DINT_OK;
}

static int launch_chunk(dint_engine* e, const Ctx& c, cudaStream_t s) {
  return with_kind(exec_kind(e), [&](auto k) { return launch_chunk_t<decltype(k)::value>(e, c, s); });
}

template <int KIND>
static int grids_for(dint_engine* e) {
  int per_sm = 0, sms = 0;
  CU(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, e->device));
  e->sms = sms;
  e->grid_route = 4 * sms;
  e->smem_stage = Stage<Wire<KIND>::MSG>::N * Stage<Wire<KIND>::MSG>::BYTES;
  if (e->smem_stage > 48 * 1024) {
    CU(cudaFuncSetAttribute(k_classify<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->smem_stage));
    CU(cudaFuncSetAttribute(k_apply<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)e->smem_stage));
  }
  e->smem_classify = e->smem_stage;
  if (KIND != K_LOG && (kTile / 32) * OrdSlice<KIND>::BYTES > e->smem_classify) e->smem_classify = (kTile / 32) * OrdSlice<KIND>::BYTES;
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_classify<KIND>, kTile, e->smem_classify));
  if (per_sm < 1) return set_err(DINT_EIO, "k_classify cannot be resident");
  e->grid_classify = per_sm * sms;
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_apply<KIND>, kTile, e->smem_stage));
  if (per_sm < 1) return set_err(DINT_EIO, "k_apply cannot be resident");
  e->grid_apply = per_sm * sms;
  if (KIND == K_LOG) { e->coop_grid = 1; return DINT_OK; }
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_ordered<KIND>, kThreads, 0));
  if (per_sm < 1) return set_err(DINT_EIO, "k_ordered cannot be resident");
  if (per_sm > 4) per_sm = 4;
  e->coop_grid = per_sm * sms;
  return DINT_OK;
}

static void fill_chunk_ctx(dint_engine* e, Ctx& c, const StepTarget* tgt) {
  const int cur = (int)(e->chunk_seq & 1);
  c.grp = e->d_grp[cur];
  c.grp_prev = e->d_grp[cur ^ 1];
  c.flags = e->d_flags[cur];
  c.flags_prev = e->d_flags[cur ^ 1];
  c.prev_n = e->prev_n;
  // whole-set clear once there is at least one request per 128-byte line of the set (2^20-request chunks: 8 per line)
  c.clear_set = (uint64_t)(c.flags_mask + 1) / 256 <= e->prev_n ? 1u : 0u;
  c.nc_cur = e->d_nc + 4 * cur;          // {listed, overflow, a writer exists, -}
  c.nc_ord = e->d_nc + 4 * (cur ^ 1);
  c.ord_pending = e->ord_pending ? 1u : 0u;
  c.ord_resp = e->ord_resp;
  c.ord_req = e->ord_req;
  c.ord_tile0 = e->ord_tile0;
  if (tgt) {                             // else e->ctx's zeros: contiguous replies in c.resp, no padding, no skip word
    c.seg_tiles = tgt->seg_tiles;
    c.pad_ok = tgt->pad_ok ? 1u : 0u;
    c.skip = tgt->skip;
    for (int i = 0; i < kMaxShards; i++) c.seg_resp[i] = tgt->seg_resp[i];
  }
}

// one chunk (n <= e->chunk); leaves its listed requests pending until the next chunk or flush_ordered()
static int submit_chunk(dint_engine* e, const uint8_t* req, uint32_t n, uint8_t* resp, cudaStream_t s, uint32_t tile0 = 0,
                        const StepTarget* tgt = nullptr) {
  Ctx c = e->ctx;
  c.n = n;
  c.n_tiles = (n + kTile - 1) / kTile;
  c.req = req;
  c.resp = resp;
  c.tile0 = tile0;
  fill_chunk_ctx(e, c, tgt);
  int rc = launch_chunk(e, c, s);
  if (rc) return rc;
  e->chunk_seq++;
  e->prev_n = n;
  e->ord_pending = e->kind != DINT_LOG;
  e->ord_resp = resp;
  e->ord_req = req;
  e->ord_tile0 = tile0;
  e->stats.chunks++;
  e->stats.requests += n;
  return DINT_OK;
}

// replays the last chunk's listed requests (and retires its flags); after this every reply is final
static int flush_ordered(dint_engine* e, cudaStream_t s, const StepTarget* tgt = nullptr) {
  if (!e->ord_pending) return DINT_OK;
  Ctx c = e->ctx;
  c.n = 0;
  c.n_tiles = 0;
  c.req = nullptr;
  c.resp = nullptr;
  fill_chunk_ctx(e, c, tgt);
  c.prev_n = 0;                  // replay only: that chunk's flags are retired by the NEXT chunk's K1 as usual (next to its tile
                                 // loads), not by this launch, which a caller is waiting for
  int rc = launch_chunk(e, c, s);
  if (rc) return rc;
  e->ord_pending = false;
  return DINT_OK;
}

// Tombstone reclamation (kv.cuh): after every call the per-table {live, used} counters travel to a pinned mirror;
// before the next call a table whose FULL + TOMB entries exceed 70 % of its capacity is rehashed into a fresh
// array (doubled when the live keys alone exceed 35 %).  Synchronous and rare: at load <= 0.5 it takes an
// insert / delete churn of 20 % of the capacity to get there.
static int kv_maintain(dint_engine* e, cudaStream_t s) {
  if (e->ctx.n_tables == 0) return DINT_OK;
  if (!e->h_kvcnt) {
    CU(cudaHostAlloc((void**)&e->h_kvcnt, 2 * kMaxTables * sizeof(unsigned long long), cudaHostAllocDefault));
    memset(e->h_kvcnt, 0, 2 * kMaxTables * sizeof(unsigned long long));
    CU(cudaEventCreateWithFlags(&e->ev_kvcnt, cudaEventDisableTiming));
    return DINT_OK;
  }
  if (cudaEventQuery(e->ev_kvcnt) != cudaSuccess) { cudaGetLastError(); return DINT_OK; }   // mirror not refreshed yet
  for (uint32_t t = 0; t < e->ctx.n_tables; t++) {
    KvTable& T = e->ctx.tbl[t];
    const unsigned long long live = e->h_kvcnt[2 * t], used = e->h_kvcnt[2 * t + 1];
    const unsigned long long cap = T.cap_mask + 1;
    if (used * 10 < cap * 7) continue;
    KvTable N = T;
    if (live * 20 > cap * 7) { N.cap_log2++; N.cap_mask = (1ULL << N.cap_log2) - 1; }
    void* fresh = nullptr;
    const size_t bytes = (size_t)(N.cap_mask + 1) << N.ent_shift;
    CU(cudaMalloc(&fresh, bytes));
    CU(cudaMemsetAsync(fresh, 0, bytes, s));
    CU(cudaMemsetAsync(T.live, 0, 16, s));                   // the rehash re-counts both
    N.entries = (uint8_t*)fresh;
    {
      ProfScope ps(e, s, KT_LOAD);
      with_kind(exec_kind(e), [&](auto k) {
        constexpr int K = decltype(k)::value;
        if constexpr (K == K_STORE || K == K_STORE_EBPF || K == K_TATP || K == K_SMALLBANK || K == K_SMALLBANK_EBPF) k_kv_move<Wire<K>::VALSZ><<<e->sms * 8, 256, 0, s>>>(T, N, KeepAll{});
        return DINT_OK;
      });
    }
    CU(cudaStreamSynchronize(s));
    for (auto& p : e->allocs) if (p == (void*)T.entries) p = fresh;
    CU(cudaFree(T.entries));
    T = N;
    e->kv[t].capacity = N.cap_mask + 1;
    e->h_kvcnt[2 * t + 1] = live;
    e->stats.kv_rebuilds++;
  }
  return DINT_OK;
}
static int kv_publish_counts(dint_engine* e, cudaStream_t s) {
  if (e->ctx.n_tables == 0 || !e->h_kvcnt) return DINT_OK;
  CU(cudaMemcpyAsync(e->h_kvcnt, e->ctx.tbl[0].live, 16 * e->ctx.n_tables, cudaMemcpyDeviceToHost, s));   // (the tables' counters are contiguous)
  CU(cudaEventRecord(e->ev_kvcnt, s));
  return DINT_OK;
}

// an engine being made from state held elsewhere (an image, a re-shard, a rebuild): destroyed unless released
struct EngineOwner {
  dint_engine* e;
  ~EngineOwner() { if (e) dint_destroy(e); }
};
// The last step of making such an engine.  Its KV tables' {live, used} counters were written with the state: set up
// and refresh their host mirror, as dint_snapshot_restore does, so that the next call's kv_maintain decides on them.
static int engine_ready(dint_engine* e) {
  { int rc = kv_maintain(e, e->stream); if (rc) return rc; }
  { int rc = kv_publish_counts(e, e->stream); if (rc) return rc; }
  CU(cudaStreamSynchronize(e->stream));
  e->stats = dint_stats{};
  return DINT_OK;
}

// One call of n requests on stream s.  The replies go to `resp`, or, with a target, where `tgt` says (the multi-GPU
// step; resp is then null).  The target belongs to this call alone: K1 of a chunk also replays the previous chunk's
// listed requests under the CURRENT chunk's target, and that is right only because every call ends in flush_ordered,
// so no chunk of this call is left to be replayed by the next call under another target.  Keep it that way.
static int run_device(dint_engine* e, const uint8_t* req, uint64_t n, uint8_t* resp, cudaStream_t s, const StepTarget* tgt = nullptr) {
  { int rc = kv_maintain(e, s); if (rc) return rc; }
  for (uint64_t off = 0; off < n; off += e->chunk) {
    uint32_t cn = (uint32_t)((n - off < e->chunk) ? (n - off) : e->chunk);
    int rc = submit_chunk(e, req + off * e->msg, cn, resp ? resp + off * e->msg : nullptr, s, (uint32_t)(off / kTile), tgt);
    if (rc) return rc;
  }
  int rc = flush_ordered(e, s, tgt);
  return rc ? rc : kv_publish_counts(e, s);
}

static void stats_from_counters(dint_engine* e, const unsigned long long* h) {
  e->stats.errors = h[0];
  e->stats.conflicted = h[1];
  e->stats.max_run = h[2];
  e->stats.ordered_fallbacks = h[3];
  e->stats.bucket_split_tasks = h[4];
  e->stats.writerless_chunks = h[5];
}
static int pull_counters(dint_engine* e) {
  unsigned long long h[kNumCounters];
  CU(cudaMemcpy(h, e->ctx.counters, sizeof h, cudaMemcpyDeviceToHost));
  stats_from_counters(e, h);
  return DINT_OK;
}

// Host-path slice sizes for a call of n requests (see dint_submit): slices double from `mn` up to the plateau
// `mx`, the body moves in plateau slices (a remainder first), and the end halves back down to `mn`.
struct HostSlices {
  uint32_t lvl[32];          // pyramid levels below the plateau, smallest first
  uint32_t n_lvl = 0, i_up = 0, i_down = 0;
  uint64_t body = 0, plateau = 0, pending = 0;
  bool ramp_up;
  HostSlices(uint64_t n, uint32_t mn, uint32_t mx, bool ramp_up_) : ramp_up(ramp_up_) {
    if (mn > mx) mn = mx;
    uint64_t used = 0;
    for (uint64_t s = mn; s < mx && n_lvl < 32; s <<= 1) {
      const uint64_t cost = ramp_up ? 2 * s : s;
      if (used + cost > n) break;
      lvl[n_lvl++] = (uint32_t)s;
      used += cost;
    }
    body = n - used;
    plateau = n_lvl ? (uint64_t)lvl[n_lvl - 1] * 2 : mx;
    if (plateau > mx) plateau = mx;
    i_down = n_lvl;
    if (!ramp_up) i_up = n_lvl;
  }
  uint32_t next() {          // 0 = done
    if (i_up < n_lvl) return lvl[i_up++];
    if (body) {
      const uint64_t rem = body % plateau;
      uint64_t c = rem ? rem : plateau;
      if (pending) { c = pending; pending = 0; }
      else if (rem && body > rem) {                        // a remainder is shared with one plateau slice: two
        c = (plateau + rem + 1) / 2;                       // mid-size slices instead of a tiny one and a full one
        pending = plateau + rem - c;
      }
      body -= c;
      return (uint32_t)c;
    }
    if (i_down) return lvl[--i_down];
    return 0;
  }
};

// ---- the host staging ring (HostRing) -----------------------------------------------------------------------------
static int ring_reserve(dint_engine* e, uint32_t sets, size_t in_bytes, size_t aux_bytes, size_t out_bytes) {
  HostRing& R = e->ring;
  for (uint32_t b = 0; b < sets; b++) {
    const std::pair<HostRing::Buf*, size_t> want[] = {{&R.in[b], in_bytes}, {&R.aux[b], aux_bytes}, {&R.out[b], out_bytes}};
    for (auto [buf, bytes] : want)
      if (bytes && buf->cap < bytes + 16) {
        CU(cudaFree(buf->p));                 // too small for this call: no earlier call is in flight
        *buf = HostRing::Buf{};
        CU(cudaMalloc(&buf->p, bytes + 16));
        buf->cap = bytes + 16;
      }
  }
  R.sets = sets;
  return DINT_OK;
}
static int ring_stage_in(dint_engine* e, uint64_t j, const void* host_in, size_t in_bytes, const void* host_aux, size_t aux_bytes, cudaStream_t consumer) {
  HostRing& R = e->ring;
  const uint32_t b = (uint32_t)(j % R.sets);
  if (j >= R.sets) CU(cudaStreamWaitEvent(R.s_in, R.released[b], 0));
  if (in_bytes) CU(cudaMemcpyAsync(R.in[b].p, host_in, in_bytes, cudaMemcpyHostToDevice, R.s_in));
  if (aux_bytes) CU(cudaMemcpyAsync(R.aux[b].p, host_aux, aux_bytes, cudaMemcpyHostToDevice, R.s_in));
  CU(cudaEventRecord(R.h2d[b], R.s_in));
  CU(cudaStreamWaitEvent(consumer, R.h2d[b], 0));
  e->stats.h2d_bytes += in_bytes + aux_bytes;
  return DINT_OK;
}
// batch j's replies are final behind what `producer` has enqueued so far
static int ring_drain_out(dint_engine* e, uint64_t j, void* host_out, size_t out_bytes, cudaStream_t producer) {
  HostRing& R = e->ring;
  const uint32_t b = (uint32_t)(j % R.sets);
  CU(cudaEventRecord(R.ready[b], producer));
  CU(cudaStreamWaitEvent(R.s_out, R.ready[b], 0));
  if (out_bytes) CU(cudaMemcpyAsync(host_out, R.out[b].p, out_bytes, cudaMemcpyDeviceToHost, R.s_out));
  CU(cudaEventRecord(R.d2h[b], R.s_out));
  e->stats.d2h_bytes += out_bytes;
  return DINT_OK;
}

// ---- fused dispatch / combine (route.cuh) ---------------------------------------------------------------
template <int KIND>
static int route_dispatch_t(dint_engine* e, const RouteArgs& a, cudaStream_t s) {
  using RT = RTile<Wire<KIND>::MSG>;
  // scratch: [0] finished-CTA counter, [1] the dispatch tile ticket, [4..12] totals + valid word, then the look-back descriptors
  if (!e->d_route2 || a.n_tiles > e->route_desc_tiles) {
    if (e->d_route2) { CU(cudaStreamSynchronize(s)); CU(cudaFree(e->d_route2)); e->d_route2 = nullptr; }
    e->route_desc_tiles = a.n_tiles + a.n_tiles / 2 + 64;
    const size_t bytes = 64 + (size_t)(e->route_desc_tiles + e->route_desc_tiles / 32 + 1) * 4 * sizeof(unsigned long long);
    CU(cudaMalloc(&e->d_route2, bytes));
    CU(cudaMemsetAsync(e->d_route2, 0, bytes, s));
    e->route_seq = 0;
  }
  e->route_seq = e->route_seq % 255u + 1u;              // 1..255; when the number wraps every descriptor is cleared, so a word
  if (e->route_seq == 1)                                 // left by an earlier launch can never carry the current number
    CU(cudaMemsetAsync(e->d_route2, 0, 64 + (size_t)(e->route_desc_tiles + e->route_desc_tiles / 32 + 1) * 4 * sizeof(unsigned long long), s));
  RouteArgs b = a;
  b.done = e->d_route2;
  b.ticket = e->d_route2 + 1;
  b.totals = e->d_route2 + 4;
  b.desc = (unsigned long long*)(e->d_route2 + 16);
  b.gdesc = b.desc + (size_t)e->route_desc_tiles * 4;
  b.seq = e->route_seq;
  if (CUDART_VERSION >= 11000 && RT::SMEM > 48 * 1024) CU(cudaFuncSetAttribute(k_route_dispatch<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RT::SMEM));
  int grid = (int)b.n_tiles < e->grid_route ? (int)b.n_tiles : e->grid_route;
  if (grid < 1) grid = 1;
  k_route_dispatch<KIND><<<grid, kThreads, RT::SMEM, s>>>(e->ctx, b);
  CU(cudaGetLastError());
  return DINT_OK;
}
template <int MSG>
static int route_combine_t(dint_engine* e, const RouteArgs& a, cudaStream_t s) {
  using RT = RTile<MSG>;
  int grid = (int)a.n_tiles;
  if (grid > e->grid_route) grid = e->grid_route;
  k_route_combine<MSG><<<grid, kThreads, RT::SMEM, s>>>(a);
  CU(cudaGetLastError());
  return DINT_OK;
}
static uint32_t route_tile_records(const dint_engine* e) { return e->msg <= 12 ? kThreads * 8u : (uint32_t)kThreads; }

// ======================================================================================================
extern "C" {

uint32_t dint_msg_size(int kind) { return (kind >= 0 && kind < DINT_NUM_KINDS) ? kMsgSize[kind] : 0; }
uint32_t dint_log_entry_size(int kind) { return (kind >= 0 && kind < DINT_NUM_KINDS) ? kLogEntry[kind] : 0; }
const char* dint_last_error(void) { return g_last_error.c_str(); }
uint64_t dint_test_fasthash64(uint64_t x, int len) { return len == 4 ? fasthash64_u32((uint32_t)x) : fasthash64_u64(x); }
uint32_t dint_test_fastmod(uint64_t n, uint32_t d) { FastMod f = make_fastmod(d); return fast_mod(n, f); }
int dint_test_rebuild_source(uint64_t key, uint32_t G, uint32_t lost_mask) {
  return G == 0 || G > kMaxShards ? -1 : rebuild_source((uint32_t)(key % G), G, lost_mask);
}
uint32_t dint_test_txn_reshard_dests(uint64_t key, uint32_t G, uint32_t G2, uint32_t src) {
  if (G == 0 || G > kMaxShards || G2 == 0 || G2 > kMaxShards) return 0;
  return ReplicaDests{make_fastmod(G), make_fastmod(G2), G2, (1u << G2) - 1, src}(key, 0);
}
uint32_t dint_test_host_slices(uint64_t n, uint32_t min_slice, uint32_t max_slice, int ramp_up, uint32_t* out, uint32_t cap) {
  HostSlices sched(n, min_slice, max_slice, ramp_up != 0);
  uint32_t k = 0;
  for (uint32_t cn; (cn = sched.next()) != 0; k++)
    if (k < cap) out[k] = cn;
  return k;
}

void dint_default_cfg(int kind, dint_cfg* cfg) {
  memset(cfg, 0, sizeof *cfg);
  cfg->lock_slots = 36000000u;
  cfg->log_ring = 1000000u;
  cfg->subs_sizing = (kind == DINT_TATP) ? 7000000u : 2000000u;
  cfg->subs_populate = cfg->subs_sizing;
  cfg->accts_sizing = 24000000u;
  cfg->accts_populate = cfg->accts_sizing;
  cfg->n_shards = 1;
  cfg->shard_id = 0;
  cfg->chunk = 1u << 20;
}

void* dint_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  return p;
}
void dint_host_free(void* p) { if (p) cudaFreeHost(p); }

void dint_destroy(dint_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  for (void* p : e->allocs) cudaFree(p);
  if (e->d_route) cudaFree(e->d_route);
  if (e->d_route2) cudaFree(e->d_route2);
  if (e->h_counters) cudaFreeHost(e->h_counters);
  if (e->h_kvcnt) cudaFreeHost(e->h_kvcnt);
  if (e->ev_kvcnt) cudaEventDestroy(e->ev_kvcnt);
  for (auto& ep : e->ev_pool) { cudaEventDestroy(ep.a); cudaEventDestroy(ep.b); }
  HostRing& R = e->ring;
  for (int i = 0; i < kHostBufs; i++) {
    for (HostRing::Buf* b : {&R.in[i], &R.aux[i], &R.out[i]}) cudaFree(b->p);
    for (cudaEvent_t ev : {R.h2d[i], R.released[i], R.ready[i], R.d2h[i]}) if (ev) cudaEventDestroy(ev);
  }
  for (cudaStream_t s : {e->stream, R.s_in, R.s_out}) if (s) cudaStreamDestroy(s);
  delete e;
}

static int create_impl(dint_engine* e) {
  const dint_cfg& cf = e->cfg;
  Ctx& c = e->ctx;
  CU(cudaSetDevice(e->device));
  CU(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
  HostRing& R = e->ring;
  for (cudaStream_t* s : {&R.s_in, &R.s_out}) CU(cudaStreamCreateWithFlags(s, cudaStreamNonBlocking));
  for (int i = 0; i < kHostBufs; i++)
    for (cudaEvent_t* ev : {&R.h2d[i], &R.released[i], &R.ready[i], &R.d2h[i]}) CU(cudaEventCreateWithFlags(ev, cudaEventDisableTiming));
  c.n_shards = cf.n_shards;
  c.shard_id = cf.shard_id;
  c.shard_div = make_fastmod(cf.n_shards);
  c.slot_mod = make_fastmod(cf.lock_slots);
  c.ring_n = cf.log_ring ? cf.log_ring : 1;

  // ---- per-kind state in HBM ----
  uint64_t groups = 0;
  auto local_groups = [&](uint64_t global) { return (global + cf.n_shards - 1) / cf.n_shards; };
  int rc;
  switch (e->kind) {
    case DINT_LOCK2PL:
      groups = local_groups(cf.lock_slots);
      if ((rc = dalloc(e, &c.cnt2, groups))) return rc;
      break;
    case DINT_FASST:
      groups = local_groups(cf.lock_slots);
      if ((rc = dalloc(e, &c.ver, groups))) return rc;     // lock bits: in the hot arena, below
      break;
    case DINT_LOG:
      groups = 0;
      break;
    default:
      if ((rc = kv_create_tables(e->kind, cf, c, e->kv, &groups,
                                 [&](void** p, size_t bytes) -> int {
                                   uint8_t* q = nullptr;
                                   int r = dalloc(e, &q, bytes);
                                   *p = q;
                                   return r;
                                 },
                                 (cf.flags & DINT_CFG_TATP_EBPF) != 0)))
        return rc == DINT_EINVAL ? set_err(rc, "bad KV configuration") : rc;
      break;
  }
  e->total_groups = groups;
  if (groups >= 0xffffffffULL) return set_err(DINT_EINVAL, "too many groups");
  // holder keys: plain HBM, outside the persisting window below -- only lock requests touch them, and the window is
  // for what every request touches
  if ((cf.flags & DINT_CFG_LOCK_HOLDER_KEYS) && (rc = dalloc(e, &c.holder, groups))) return rc;
  // the eBPF store's cache sets, one per bucket (store/ebpf/store_kern.c:25-30): plain HBM, zeroed = every slot invalid
  if (cf.flags & DINT_CFG_STORE_EBPF_MASK) {
    c.ecache_variant = (cf.flags & DINT_CFG_STORE_EBPF_MASK) >> 1;
    if ((rc = dalloc(e, &c.ecache, groups * kEcSetBytes))) return rc;
    if ((rc = dalloc(e, &c.ecache_stats, EC_NSTATS))) return rc;
  }
  // the eBPF TATP server's cache sets (tatp/ebpf/shard_kern.c:61-94) and chained tables: one set and one {head, free}
  // pair per bucket (groups / 4: four lock slots per bucket), and a pool of 1.5 chain entries per bucket.  A chain
  // entry per bucket holds the 2.7 rows per bucket of the reference's population; cache-only rows take none.
  if (cf.flags & DINT_CFG_TATP_EBPF) {
    const uint64_t buckets = groups / 4;
    for (uint32_t t = 0; t < c.n_tables; t++) c.tbkt_mod[t] = make_fastmod(e->kv[t].hash_size);
    c.tpool_cap = (uint32_t)(buckets + buckets / 2 + 4096);
    if ((rc = dalloc(e, &c.ecache, buckets * kEcSetBytes))) return rc;
    if ((rc = dalloc(e, &c.ecache_stats, EC_NSTATS_TATP))) return rc;
    if ((rc = dalloc(e, &c.tchain, buckets))) return rc;
    if ((rc = dalloc(e, &c.tpool, (size_t)c.tpool_cap * kTeEntBytes))) return rc;
    if ((rc = dalloc(e, &c.tpool_top, 1))) return rc;
  }
  // the eBPF SmallBank server's cache sets (smallbank/ebpf/shard_kern.c:40-52): one 128-byte set per bucket of both
  // tables (groups / 4: four lock slots per bucket), zeroed = every slot invalid, as the reference's cache starts
  if (cf.flags & DINT_CFG_SMALLBANK_EBPF) {
    for (uint32_t t = 0; t < c.n_tables; t++) c.tbkt_mod[t] = make_fastmod(e->kv[t].hash_size);
    if ((rc = dalloc(e, &c.ecache, groups / 4 * kSbeSetBytes))) return rc;
    if ((rc = dalloc(e, &c.ecache_stats, SBE_NSTATS))) return rc;
  }
  {
    uint32_t fl = 25;                                  // 2^25 nibbles = 16 MB per set: L2-resident
    while (fl > 10 && (1ULL << (fl - 1)) >= groups * 2 + 2048) fl--;   // tiny group spaces need less
    c.flags_mask = (1u << fl) - 1;
    const size_t set_bytes = (size_t)4 << (fl - 3);
    const size_t lock_bytes = (e->kind == DINT_FASST) ? (((groups + 31) / 32) * 4 + 255) / 256 * 256 : 0;
    e->hot_bytes = 2 * set_bytes + lock_bytes;
    if ((rc = dalloc(e, &e->hot_arena, e->hot_bytes))) return rc;
    e->d_flags[0] = (uint32_t*)e->hot_arena;
    e->d_flags[1] = (uint32_t*)(e->hot_arena + set_bytes);
    if (lock_bytes) c.lockbits = (uint32_t*)(e->hot_arena + 2 * set_bytes);
    // reserve L2 for it
    int max_persist = 0, max_win = 0;
    cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, e->device);
    cudaDeviceGetAttribute(&max_win, cudaDevAttrMaxAccessPolicyWindowSize, e->device);
    if (max_persist > 0 && max_win > 0) {
      size_t want = e->hot_bytes < (size_t)max_persist ? e->hot_bytes : (size_t)max_persist;
      if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want) == cudaSuccess) {
        e->window.base_ptr = e->hot_arena;
        e->window.num_bytes = e->hot_bytes < (size_t)max_win ? e->hot_bytes : (size_t)max_win;
        e->window.hitRatio = (float)((double)want / (double)e->window.num_bytes > 1.0 ? 1.0 : (double)want / (double)e->window.num_bytes);
        e->window.hitProp = cudaAccessPropertyPersisting;
        e->window.missProp = cudaAccessPropertyStreaming;
        e->use_window = true;
      } else cudaGetLastError();
    }
  }
  uint32_t bits = 1;
  while ((1ULL << bits) < groups) bits++;
  c.sort_passes = (bits + 7) / 8;

  if (e->has_log) {
    if ((rc = dalloc(e, &c.ring, (size_t)c.ring_n * kLogEntry[e->kind]))) return rc;
  }
  // ---- chunk scratch ----
  const uint32_t ch = e->chunk;
  e->max_tiles = (ch + kTile - 1) / kTile;
  for (int i = 0; i < 2; i++)
    if ((rc = dalloc(e, &e->d_grp[i], ch))) return rc;
  if ((rc = dalloc(e, &c.clist, (size_t)e->max_tiles * kTile))) return rc;
  if ((rc = dalloc(e, &c.ccnt, e->max_tiles))) return rc;
  if ((rc = dalloc(e, &c.cprefix, e->max_tiles + 1))) return rc;
  if ((rc = dalloc(e, &e->d_nc, 8))) return rc;
  {
    uint32_t lg = 0;
    while (((uint64_t)kBucketFill << lg) < ch) lg++;
    c.bucket_log2 = lg;
    if ((rc = dalloc(e, &c.buckets, ((size_t)1 << lg) * kBucketCap, false))) return rc;
    if ((rc = dalloc(e, &c.bcnt, (size_t)1 << lg))) return rc;
  }
  if ((rc = dalloc(e, &c.sortA, ch))) return rc;
  if ((rc = dalloc(e, &c.sortB, ch))) return rc;
  if ((rc = dalloc(e, &c.ghist, (size_t)256 * ((ch + kSortTile - 1) / kSortTile)))) return rc;
  if ((rc = dalloc(e, &c.rowtot, 256))) return rc;
  if ((rc = dalloc(e, &c.log_tilecnt, e->max_tiles))) return rc;
  if ((rc = dalloc(e, &c.log_tilebase, e->max_tiles))) return rc;
  if ((rc = dalloc(e, &c.log_total, 2))) return rc;
  if (e->kind == DINT_TATP && (rc = dalloc(e, &c.log_src, ch))) return rc;
  if ((rc = dalloc(e, &c.counters, kNumCounters))) return rc;
  if ((rc = dalloc(e, &c.gbar, 4))) return rc;

  if ((rc = with_kind(exec_kind(e), [&](auto k) { return grids_for<decltype(k)::value>(e); }))) return rc;
  int coop = 0;
  CU(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, e->device));
  if (!coop) return set_err(DINT_ENODEV, "device lacks cooperative launch");
  CU(cudaStreamSynchronize(e->stream));
  return DINT_OK;
}

int dint_create(int kind, const dint_cfg* cfg, int device, dint_engine** out) {
  if (!out || kind < 0 || kind >= DINT_NUM_KINDS) return set_err(DINT_EINVAL, "bad kind/out");
  *out = nullptr;
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return set_err(DINT_ENODEV, "no CUDA device: dint_b200 has no CPU fallback");
  }
  if (device < 0 || device >= ndev) return set_err(DINT_EINVAL, "bad device ordinal");
  dint_engine* e = new dint_engine();
  e->kind = kind;
  e->device = device;
  if (cfg) e->cfg = *cfg; else dint_default_cfg(kind, &e->cfg);
  dint_cfg& cf = e->cfg;
  if (cf.n_shards == 0) cf.n_shards = 1;
  if (cf.shard_id >= cf.n_shards || cf.lock_slots == 0) { delete e; return set_err(DINT_EINVAL, "bad shard/lock_slots"); }
  if ((cf.flags & DINT_CFG_LOCK_HOLDER_KEYS) && kind != DINT_TATP) { delete e; return set_err(DINT_EINVAL, "DINT_CFG_LOCK_HOLDER_KEYS is a tatp option"); }
  if ((cf.flags & DINT_CFG_STORE_EBPF_MASK) && kind != DINT_STORE) { delete e; return set_err(DINT_EINVAL, "DINT_CFG_STORE_EBPF_* is a store option"); }
  if ((cf.flags & DINT_CFG_TATP_EBPF) && kind != DINT_TATP) { delete e; return set_err(DINT_EINVAL, "DINT_CFG_TATP_EBPF is a tatp option"); }
  if ((cf.flags & DINT_CFG_TATP_EBPF) && cf.n_shards != 1) { delete e; return set_err(DINT_EINVAL, "DINT_CFG_TATP_EBPF needs n_shards = 1 (place tatp shards with txn_shards)"); }
  if ((cf.flags & DINT_CFG_SMALLBANK_EBPF) && kind != DINT_SMALLBANK) { delete e; return set_err(DINT_EINVAL, "DINT_CFG_SMALLBANK_EBPF is a smallbank option"); }
  if ((cf.flags & DINT_CFG_SMALLBANK_EBPF) && cf.n_shards != 1) { delete e; return set_err(DINT_EINVAL, "DINT_CFG_SMALLBANK_EBPF needs n_shards = 1 (place smallbank shards with txn_shards)"); }
  if (cf.chunk == 0) cf.chunk = 1u << 20;
  e->chunk = (cf.chunk + kTile - 1) / kTile * kTile;
  {
    // host-path slice schedule: 128 K requests doubling up to 256 K (see dint_submit)
    const uint32_t want = 1u << 18;
    e->host_chunk = want < e->chunk ? want : e->chunk;
    e->host_min_slice = 131072u;
    e->host_ramp_up = true;
  }
  e->msg = kMsgSize[kind];
  e->has_log = kLogEntry[kind] != 0;
  int rc = create_impl(e);
  if (rc) { dint_destroy(e); return rc; }
  *out = e;
  return DINT_OK;
}

int dint_route_owner(dint_engine* e, const void* req_dev, uint64_t n, uint8_t* owner_dev, void* cuda_stream) {
  if (!e || (n && (!req_dev || !owner_dev)) || n > 0xffffffffULL) return set_err(DINT_EINVAL, "bad argument");
  if (n == 0) return DINT_OK;
  CU(cudaSetDevice(e->device));
  cudaStream_t s = (cudaStream_t)cuda_stream;
  const uint32_t blocks = (uint32_t)((n + kThreads - 1) / kThreads);
  const uint8_t* rq = (const uint8_t*)req_dev;
  e->stats.kernel_launches++;
  with_kind(exec_kind(e), [&](auto k) {
    k_route_owner<decltype(k)::value><<<blocks, kThreads, 0, s>>>(e->ctx, rq, (uint32_t)n, owner_dev);
    return DINT_OK;
  });
  CU(cudaGetLastError());
  return DINT_OK;
}

int dint_route_partition(dint_engine* e, const void* req_dev, const uint8_t* owner_dev, uint64_t n, uint32_t n_shards,
                         void* sorted_dev, uint32_t* perm_dev, uint32_t* counts_dev, void* cuda_stream) {
  if (!e || n_shards == 0 || n_shards > kMaxShards || n > 0xffffffffULL) return set_err(DINT_EINVAL, "bad argument");
  CU(cudaSetDevice(e->device));
  cudaStream_t s = (cudaStream_t)cuda_stream;
  const uint32_t tiles = (uint32_t)((n + kThreads - 1) / kThreads);
  if (tiles > e->route_tiles) {                          // scratch: per-tile per-shard counts + totals
    if (e->d_route) { CU(cudaFree(e->d_route)); e->d_route = nullptr; }
    e->route_tiles = tiles + tiles / 2 + 64;
    CU(cudaMalloc(&e->d_route, ((size_t)e->route_tiles * kMaxShards + 3 * kMaxShards) * sizeof(uint32_t)));
  }
  uint32_t* totals = e->d_route;                         // [0..8) records per shard
  uint32_t* tilecnt = e->d_route + 3 * kMaxShards;
  if (n == 0) { CU(cudaMemsetAsync(counts_dev, 0, n_shards * sizeof(uint32_t), s)); return DINT_OK; }
  e->stats.kernel_launches += 3;
  k_exact_count<<<tiles, kThreads, 0, s>>>(owner_dev, (uint32_t)n, n_shards, tilecnt);
  k_exact_scan<<<n_shards, kThreads, 0, s>>>(tilecnt, tiles, totals);
  const uint8_t* rq = (const uint8_t*)req_dev;
  uint8_t* out = (uint8_t*)sorted_dev;
  with_kind(exec_kind(e), [&](auto k) {
    k_exact_scatter<Wire<decltype(k)::value>::MSG><<<tiles, kThreads, 0, s>>>(rq, owner_dev, (uint32_t)n, n_shards, tilecnt, totals, out, perm_dev);
    return DINT_OK;
  });
  CU(cudaMemcpyAsync(counts_dev, totals, n_shards * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  CU(cudaGetLastError());
  return DINT_OK;
}

uint32_t dint_route_tile_records(dint_engine* e) { return e ? route_tile_records(e) : 0; }

int dint_route_dispatch(dint_engine* e, const void* req_dev, const uint8_t* owner_in_dev, uint64_t n, uint32_t n_shards, uint32_t rank,
                        uint32_t cap, const dint_peer_ptrs* slab_ptrs, const dint_peer_ptrs* sig_ptrs, uint32_t epoch,
                        uint8_t* owner_dev, uint32_t* tilebase_dev, uint32_t* flags_dev, void* cuda_stream) {
  if (!e || !slab_ptrs || !flags_dev || n_shards == 0 || n_shards > kMaxShards || rank >= n_shards || cap == 0 || n >= (1ULL << 27) ||
      (n && (!req_dev || !owner_dev || !tilebase_dev)))
    return set_err(DINT_EINVAL, "bad argument");
  if ((uintptr_t)req_dev & 15) return set_err(DINT_EINVAL, "device buffers must be 16-byte aligned");
  if (!owner_in_dev && n_shards != e->ctx.n_shards) return set_err(DINT_EINVAL, "owner computation needs n_shards == cfg.n_shards");
  CU(cudaSetDevice(e->device));
  RouteArgs a{};
  a.req = (const uint8_t*)req_dev;
  a.owner_in = owner_in_dev;
  a.owner = owner_dev;
  a.tilebase = tilebase_dev;
  a.flags = flags_dev;
  a.n = (uint32_t)n;
  a.n_tiles = (uint32_t)((n + route_tile_records(e) - 1) / route_tile_records(e));
  a.world = n_shards;
  a.me = rank;
  a.cap = cap;
  a.epoch = epoch;
  for (uint32_t i = 0; i < kMaxShards; i++) { a.slab.p[i] = slab_ptrs->p[i]; a.sig.p[i] = sig_ptrs ? sig_ptrs->p[i] : 0; }
  cudaStream_t s = (cudaStream_t)cuda_stream;
  e->stats.kernel_launches += 1;
  return with_kind(exec_kind(e), [&](auto k) { return route_dispatch_t<decltype(k)::value>(e, a, s); });
}

int dint_route_combine(dint_engine* e, const dint_peer_ptrs* reply_slab_ptrs, const uint8_t* owner_dev, const uint32_t* tilebase_dev,
                       uint64_t n, uint32_t n_shards, uint32_t cap, void* out_dev, void* cuda_stream) {
  if (!e || !reply_slab_ptrs || n_shards == 0 || n_shards > kMaxShards || cap == 0 || n > 0xffffffffULL ||
      (n && (!owner_dev || !tilebase_dev || !out_dev)))
    return set_err(DINT_EINVAL, "bad argument");
  if ((uintptr_t)out_dev & 15) return set_err(DINT_EINVAL, "device buffers must be 16-byte aligned");
  if (n == 0) return DINT_OK;
  CU(cudaSetDevice(e->device));
  RouteArgs a{};
  a.owner = (uint8_t*)owner_dev;
  a.tilebase = (uint32_t*)tilebase_dev;
  a.out = (uint8_t*)out_dev;
  a.n = (uint32_t)n;
  a.n_tiles = (uint32_t)((n + route_tile_records(e) - 1) / route_tile_records(e));
  a.world = n_shards;
  a.cap = cap;
  for (uint32_t i = 0; i < kMaxShards; i++) a.slab.p[i] = reply_slab_ptrs->p[i];
  cudaStream_t s = (cudaStream_t)cuda_stream;
  e->stats.kernel_launches++;
  return with_kind(exec_kind(e), [&](auto k) { return route_combine_t<Wire<decltype(k)::value>::MSG>(e, a, s); });
}

int dint_p2p_wait(dint_engine* e, const uint32_t* local_sig_dev, uint32_t n_shards, uint32_t epoch, uint32_t* flags_dev, void* cuda_stream) {
  if (!e || !local_sig_dev || n_shards == 0 || n_shards > kMaxShards) return set_err(DINT_EINVAL, "bad argument");
  CU(cudaSetDevice(e->device));
  e->stats.kernel_launches++;
  k_p2p_wait<<<1, 32, 0, (cudaStream_t)cuda_stream>>>(local_sig_dev, n_shards, epoch, flags_dev + 1, nullptr);
  CU(cudaGetLastError());
  return DINT_OK;
}

int dint_p2p_signal(dint_engine* e, const dint_peer_ptrs* sig_ptrs, uint32_t n_shards, uint32_t rank, uint32_t epoch, void* cuda_stream) {
  if (!e || !sig_ptrs || n_shards == 0 || n_shards > kMaxShards || rank >= n_shards) return set_err(DINT_EINVAL, "bad argument");
  CU(cudaSetDevice(e->device));
  PeerPtrs sg{};
  for (uint32_t i = 0; i < kMaxShards; i++) sg.p[i] = sig_ptrs->p[i];
  e->stats.kernel_launches++;
  k_p2p_signal<<<1, 32, 0, (cudaStream_t)cuda_stream>>>(sg, n_shards, rank, epoch);
  CU(cudaGetLastError());
  return DINT_OK;
}

int dint_route_unpermute(dint_engine* e, const void* sorted_dev, const uint32_t* perm_dev, uint64_t n, void* out_dev, void* cuda_stream) {
  if (!e || n > 0xffffffffULL) return set_err(DINT_EINVAL, "bad argument");
  if (n == 0) return DINT_OK;
  CU(cudaSetDevice(e->device));
  cudaStream_t s = (cudaStream_t)cuda_stream;
  e->stats.kernel_launches++;
  const uint8_t* in = (const uint8_t*)sorted_dev;
  uint8_t* out = (uint8_t*)out_dev;
  with_kind(exec_kind(e), [&](auto k) {
    k_exact_unpermute<Wire<decltype(k)::value>::MSG><<<(uint32_t)((n + kThreads - 1) / kThreads), kThreads, 0, s>>>(in, perm_dev, (uint32_t)n, out);
    return DINT_OK;
  });
  CU(cudaGetLastError());
  return DINT_OK;
}

int dint_sync(dint_engine* e) {
  if (!e) return DINT_EINVAL;
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  int rc = prof_flush(e);
  if (rc) return rc;
  unsigned long long before = e->stats.errors;
  if ((rc = pull_counters(e))) return rc;
  return e->stats.errors != before ? DINT_EPROTO : DINT_OK;
}

int dint_submit_device(dint_engine* e, const void* req_dev, uint64_t n, void* resp_dev, void* cuda_stream) {
  if (!e || (n && (!req_dev || !resp_dev))) return set_err(DINT_EINVAL, "null argument");
  if (((uintptr_t)req_dev | (uintptr_t)resp_dev) & 15) return set_err(DINT_EINVAL, "device buffers must be 16-byte aligned");
  CU(cudaSetDevice(e->device));
  cudaStream_t s = (cudaStream_t)cuda_stream;        // NULL = the legacy default stream, as in every CUDA API
  return run_device(e, (const uint8_t*)req_dev, n, (uint8_t*)resp_dev, s);
}

int dint_submit(dint_engine* e, const void* req, uint64_t n, void* resp) {
  if (!e || (n && (!req || !resp))) return set_err(DINT_EINVAL, "null argument");
  CU(cudaSetDevice(e->device));
  // the host path moves data in slices of `hchunk` requests through the engine's ring of kHostBufs staging sets:
  // small slices keep the PCIe fill/drain bubbles short, the ring keeps both copy engines and the SMs busy
  const uint32_t hchunk = e->host_chunk;
  static const bool trace = getenv("DINT_HOST_TRACE") != nullptr;
  const auto t_begin = std::chrono::steady_clock::now();
  CU(cudaDeviceSynchronize());     // order after anything submitted on user streams
  { int rc = ring_reserve(e, kHostBufs, (size_t)hchunk * e->msg, 0, (size_t)hchunk * e->msg); if (rc) return rc; }
  { int rc = kv_maintain(e, e->stream); if (rc) return rc; }
  const uint8_t* rq = (const uint8_t*)req;
  uint8_t* rs = (uint8_t*)resp;
  unsigned long long err_before = e->stats.errors;
  // three-stage pipeline: H2D (ring s_in) | kernels (stream) | D2H (ring s_out).  Slice k's replies are final only
  // after the launch that replays its listed requests -- K1 of slice k+1, or the flush after the last
  // slice -- so D2H(k) is ordered behind that.  That launch is also the last to read slice k's requests.
  uint64_t k = 0;
  uint64_t prev_off = 0, prev_bytes = 0;
  auto copy_out_prev = [&](uint64_t kk) -> int {          // D2H of slice kk-1
    CU(cudaEventRecord(e->ring.released[(kk - 1) % kHostBufs], e->stream));
    return ring_drain_out(e, kk - 1, rs + prev_off, prev_bytes, e->stream);
  };
  // Slice schedule.  PCIe moves large copies better than small ones (tools/pcie_probe.cu measures it), but the
  // first slice's H2D and the last two slices' kernels + D2H overlap with nothing.  So a call is cut as a
  // pyramid: slices double from host_min_slice up to host_chunk, stay there, and halve back down at the end.
  HostSlices sched(n, e->host_min_slice, hchunk, e->host_ramp_up);
  uint64_t off = 0;
  for (uint64_t cn; (cn = sched.next()) != 0; k++) {
    int b = (int)(k % kHostBufs);
    size_t bytes = (size_t)cn * e->msg;
    if (k >= (uint64_t)kHostBufs) CU(cudaStreamWaitEvent(e->stream, e->ring.d2h[b], 0));     // slice k-kHostBufs's replies have left out[b]
    int rc = ring_stage_in(e, k, rq + off * e->msg, bytes, nullptr, 0, e->stream);
    if (!rc) rc = submit_chunk(e, e->ring.in[b].p, (uint32_t)cn, e->ring.out[b].p, e->stream);
    if (rc) return rc;
    if (k >= 1 && (rc = copy_out_prev(k))) return rc;                   // slice k-1 is final now
    prev_off = off * e->msg;
    prev_bytes = bytes;
    off += cn;
  }
  {
    int rc = flush_ordered(e, e->stream);
    if (rc) return rc;
    if (k >= 1 && (rc = copy_out_prev(k))) return rc;
  }
  if (!e->h_counters) CU(cudaHostAlloc((void**)&e->h_counters, kNumCounters * sizeof(unsigned long long), cudaHostAllocDefault));
  CU(cudaMemcpyAsync(e->h_counters, e->ctx.counters, kNumCounters * sizeof(unsigned long long), cudaMemcpyDeviceToHost, e->stream));
  { int rc2 = kv_publish_counts(e, e->stream); if (rc2) return rc2; }
  const auto t_enq = std::chrono::steady_clock::now();
  CU(cudaStreamSynchronize(e->ring.s_out));
  CU(cudaStreamSynchronize(e->stream));
  int rc = prof_flush(e);
  if (rc) return rc;
  if (trace) {
    const auto t_end = std::chrono::steady_clock::now();
    fprintf(stderr, "[dint_submit] n=%llu slices=%llu enqueue=%.1f us total=%.1f us\n", (unsigned long long)n, (unsigned long long)k,
            std::chrono::duration<double, std::micro>(t_enq - t_begin).count(),
            std::chrono::duration<double, std::micro>(t_end - t_begin).count());
  }
  stats_from_counters(e, e->h_counters);
  return e->stats.errors != err_before ? DINT_EPROTO : DINT_OK;
}

// ---- state snapshots (checkpoint / restore of one engine's whole server state, device to device) --------------
struct dint_snapshot {
  dint_engine* e = nullptr;
  std::vector<std::pair<void*, size_t>> live;   // the engine's state arrays
  std::vector<void*> copy;
  uint64_t kv_cap[kMaxTables]{};                 // table capacities at snapshot time (a rehash in between invalidates it)
};
static void snapshot_regions(dint_engine* e, std::vector<std::pair<void*, size_t>>& r) {
  const Ctx& c = e->ctx;
  const uint64_t g = e->total_groups;
  if (e->kind == DINT_LOCK2PL || e->kind == DINT_SMALLBANK) r.push_back({c.cnt2, g * sizeof(uint2)});
  if (e->kind == DINT_FASST) { r.push_back({c.ver, g * sizeof(uint32_t)}); r.push_back({c.lockbits, ((g + 31) / 32) * 4}); }
  if (e->kind == DINT_TATP) r.push_back({c.lockbits, ((g + 31) / 32) * 4});
  if (c.holder) r.push_back({c.holder, g * sizeof(uint64_t)});
  if (c.tchain) {
    r.push_back({c.ecache, g / 4 * kEcSetBytes});
    r.push_back({c.tchain, g / 4 * sizeof(uint2)});
    r.push_back({c.tpool, (size_t)c.tpool_cap * kTeEntBytes});
    r.push_back({c.tpool_top, sizeof(uint32_t)});
  } else if (sbe_on(e)) r.push_back({c.ecache, g / 4 * kSbeSetBytes});
  else if (c.ecache) r.push_back({c.ecache, g * kEcSetBytes});
  for (uint32_t t = 0; t < c.n_tables; t++) {
    r.push_back({c.tbl[t].entries, (size_t)(c.tbl[t].cap_mask + 1) << c.tbl[t].ent_shift});
    r.push_back({c.tbl[t].live, 16});
  }
  if (e->has_log) { r.push_back({c.ring, (size_t)c.ring_n * kLogEntry[e->kind]}); r.push_back({c.log_total, 2 * sizeof(unsigned long long)}); }
}
int dint_snapshot_create(dint_engine* e, dint_snapshot** out) {
  if (!e || !out) return set_err(DINT_EINVAL, "null argument");
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  dint_snapshot* s = new dint_snapshot();
  s->e = e;
  snapshot_regions(e, s->live);
  for (uint32_t t = 0; t < e->ctx.n_tables; t++) s->kv_cap[t] = e->ctx.tbl[t].cap_mask + 1;
  for (auto& r : s->live) {
    void* p = nullptr;
    cudaError_t ce = cudaMalloc(&p, r.second ? r.second : 1);
    if (ce != cudaSuccess) { for (void* q : s->copy) cudaFree(q); delete s; return set_err(DINT_ENOMEM, "snapshot", ce); }
    s->copy.push_back(p);
    CU(cudaMemcpyAsync(p, r.first, r.second, cudaMemcpyDeviceToDevice, e->stream));
  }
  CU(cudaStreamSynchronize(e->stream));
  *out = s;
  return DINT_OK;
}
int dint_snapshot_restore(dint_snapshot* s, void* cuda_stream) {
  if (!s) return set_err(DINT_EINVAL, "null argument");
  dint_engine* e = s->e;
  CU(cudaSetDevice(e->device));
  for (uint32_t t = 0; t < e->ctx.n_tables; t++)
    if (s->kv_cap[t] != e->ctx.tbl[t].cap_mask + 1) return set_err(DINT_EINVAL, "a KV table was rehashed since the snapshot");
  std::vector<std::pair<void*, size_t>> now;
  snapshot_regions(e, now);
  if (now.size() != s->live.size()) return set_err(DINT_EINVAL, "snapshot does not match the engine");
  for (size_t i = 0; i < now.size(); i++) {
    if (now[i].second != s->live[i].second) return set_err(DINT_EINVAL, "snapshot does not match the engine");
    CU(cudaMemcpyAsync(now[i].first, s->copy[i], now[i].second, cudaMemcpyDeviceToDevice, (cudaStream_t)cuda_stream));
  }
  // the KV tables' {live, used} counters went back too: refresh their host mirror, or the next call's kv_maintain
  // would rehash a restored table on the occupancy it had before the restore
  return kv_publish_counts(e, (cudaStream_t)cuda_stream);
}
void dint_snapshot_destroy(dint_snapshot* s) {
  if (!s) return;
  cudaSetDevice(s->e->device);
  for (void* p : s->copy) cudaFree(p);
  delete s;
}

}  // extern "C"

// ---- state images: the regions of snapshot_regions in a file, zero lines left out (image.cuh; layout in dint_b200.h) ----
static const char kImgMagic[8] = {'D', 'I', 'N', 'T', 'I', 'M', 'G', '1'};
static const char kCluMagic[8] = {'D', 'I', 'N', 'T', 'C', 'L', 'U', '1'};
constexpr uint32_t kImgVersion = 1;
constexpr uint32_t kImgMaxRegions = 32;
constexpr uint32_t kCfgKnownFlags = DINT_CFG_LOCK_HOLDER_KEYS | DINT_CFG_STORE_EBPF_MASK | DINT_CFG_TATP_EBPF | DINT_CFG_SMALLBANK_EBPF;
constexpr uint32_t kImgSets = 3;                     // blocks in flight: pack | copy | file
struct ImgHeader {
  char magic[8];
  uint32_t version, kind;
  dint_cfg cfg;
  uint32_t n_regions;
  uint64_t kv_capacity[kMaxTables];
  uint32_t tpool_cap, n_tables;
};
struct ImgRegion { uint32_t index, reserved; uint64_t bytes, blocks; };
struct CluManifest {
  char magic[8];
  uint32_t version, kind, shards, reserved;
  dint_cfg cfg;
  uint32_t reserved2;
};
static_assert(sizeof(dint_cfg) == 76 && sizeof(ImgHeader) == 144 && sizeof(ImgRegion) == 24 && sizeof(CluManifest) == 104,
              "the image layout of include/dint_b200.h");

static thread_local double g_img_times[4];           // dint_image_times: wall, kernels, copies, file (s)

struct ImgFd {
  int fd = -1;
  ~ImgFd() { if (fd >= 0) close(fd); }
};
static bool img_read(int fd, void* p, size_t n) {
  uint8_t* q = (uint8_t*)p;
  while (n) {
    const ssize_t k = read(fd, q, n);
    if (k < 0 && errno == EINTR) continue;
    if (k <= 0) return false;
    q += k;
    n -= (size_t)k;
  }
  return true;
}
static bool img_write(int fd, const void* p, size_t n) {
  const uint8_t* q = (const uint8_t*)p;
  while (n) {
    const ssize_t k = write(fd, q, n);
    if (k < 0 && errno == EINTR) continue;
    if (k <= 0) return false;
    q += k;
    n -= (size_t)k;
  }
  return true;
}
// writes `bytes` to path.tmp, fsyncs it and renames it to path: a crash never leaves a half file under the final name
// fsyncs the directory holding `path`, so that a rename or unlink in it is durable
static int img_sync_dir(const char* path) {
  std::string dir(path);
  const size_t slash = dir.find_last_of('/');
  dir = slash == std::string::npos ? std::string(".") : slash == 0 ? std::string("/") : dir.substr(0, slash);
  ImgFd d;
  d.fd = open(dir.c_str(), O_RDONLY | O_DIRECTORY);
  if (d.fd < 0 || fsync(d.fd) != 0) return set_errf(DINT_EIO, "image directory %s: fsync: %s", dir.c_str(), strerror(errno));
  return DINT_OK;
}
static int img_publish(const char* tmp, const char* path, int fd) {
  if (fsync(fd) != 0) return set_errf(DINT_EIO, "image %s: fsync: %s", tmp, strerror(errno));
  if (rename(tmp, path) != 0) return set_errf(DINT_EIO, "image %s: rename: %s", path, strerror(errno));
  return img_sync_dir(path);
}

// one block of a region: its device range
struct ImgBlock { uint32_t region; uint64_t index; uint8_t* p; uint64_t bytes; };
static std::vector<ImgBlock> img_blocks(const std::vector<std::pair<void*, size_t>>& regs) {
  std::vector<ImgBlock> out;
  for (uint32_t r = 0; r < regs.size(); r++)
    for (uint64_t off = 0, k = 0; off < regs[r].second; off += kImgBlock, k++)
      out.push_back({r, k, (uint8_t*)regs[r].first + off, std::min<uint64_t>(kImgBlock, regs[r].second - off)});
  return out;
}
// bytes a block stores for its lines: whole lines, except a partial last line, which keeps its in-range bytes
static uint64_t img_stored_bytes(uint64_t raw, const uint32_t* bitmap, uint64_t n_set) {
  const uint64_t L = img_lines(raw), rem = raw % kImgLine;
  uint64_t b = n_set * kImgLine;
  if (rem && ((bitmap[(L - 1) >> 5] >> ((L - 1) & 31)) & 1u)) b -= kImgLine - rem;
  return b;
}

// What both directions share: device scratch of the kernels, pinned host buffers, the ring's device staging, timing.
struct ImgPipe {
  dint_engine* e = nullptr;
  uint8_t* scratch = nullptr;                         // {ticket, tilebase[], sums, desc[], gdesc[]} of one launch
  uint32_t* bad = nullptr;                            // unpack verdict per block
  uint8_t* host[kImgSets] = {};
  unsigned long long* meta = nullptr;                 // pinned: {checksum, stored lines} per set (save)
  cudaEvent_t ev[kImgSets][4] = {};                   // kernel begin / end, copy begin / end
  size_t stage = 0;
  size_t ring_cap[kImgSets] = {};                     // the ring's staging before this call
  ~ImgPipe() {
    if (!e) return;
    cudaSetDevice(e->device);
    cudaDeviceSynchronize();
    // the 64 MiB staging buffers this call added to the ring go again: the ring allocates what a later call needs
    for (uint32_t b = 0; b < kImgSets; b++)
      if (e->ring.in[b].cap > ring_cap[b]) { cudaFree(e->ring.in[b].p); e->ring.in[b] = HostRing::Buf{}; }
    cudaFree(scratch);
    cudaFree(bad);
    for (uint8_t* h : host) if (h) cudaFreeHost(h);
    if (meta) cudaFreeHost(meta);
    for (auto& s : ev) for (cudaEvent_t x : s) if (x) cudaEventDestroy(x);
  }
  static constexpr size_t kTicket = 0, kSums = 16, kTilebase = 64, kDesc = kTilebase + 4 * kImgMaxTiles;
  static constexpr size_t kGdesc = kDesc + 8 * kImgMaxTiles, kBytes = kGdesc + 8 * (kImgMaxTiles / 32);
  int init(dint_engine* e_, uint64_t n_blocks) {
    e = e_;
    stage = img_words(kImgBlock) * 4 + kImgBlock;
    for (uint32_t b = 0; b < kImgSets; b++) ring_cap[b] = e->ring.in[b].cap;
    { int rc = ring_reserve(e, kImgSets, stage, 0, 0); if (rc) return rc; }
    CU(cudaMalloc(&scratch, kBytes));
    CU(cudaMalloc(&bad, 4 * (n_blocks ? n_blocks : 1)));
    CU(cudaMemsetAsync(bad, 0, 4 * (n_blocks ? n_blocks : 1), e->stream));
    for (uint32_t b = 0; b < kImgSets; b++) {
      CU(cudaHostAlloc((void**)&host[b], stage, cudaHostAllocDefault));
      for (cudaEvent_t& x : ev[b]) CU(cudaEventCreate(&x));
    }
    CU(cudaHostAlloc((void**)&meta, 2 * kImgSets * sizeof(unsigned long long), cudaHostAllocDefault));
    return DINT_OK;
  }
  ImgArgs args(const ImgBlock& k, uint8_t* staged) const {
    ImgArgs a{};
    a.raw = k.p;
    a.bytes = k.bytes;
    a.n_words = (uint32_t)img_words(k.bytes);
    a.n_tiles = (uint32_t)((img_lines(k.bytes) + kImgTileLines - 1) / kImgTileLines);
    a.bitmap = (uint32_t*)staged;
    a.lines = staged + (size_t)a.n_words * 4;
    a.ticket = (uint32_t*)(scratch + kTicket);
    a.sum = (unsigned long long*)(scratch + kSums);
    a.tilebase = (uint32_t*)(scratch + kTilebase);
    a.desc = (unsigned long long*)(scratch + kDesc);
    a.gdesc = (unsigned long long*)(scratch + kGdesc);
    return a;
  }
  // kernel and copy time of the block that used set b (its events are complete)
  int account(uint32_t b) {
    float k = 0, c = 0;
    CU(cudaEventElapsedTime(&k, ev[b][0], ev[b][1]));
    CU(cudaEventElapsedTime(&c, ev[b][2], ev[b][3]));
    g_img_times[1] += k * 1e-3;
    g_img_times[2] += c * 1e-3;
    return DINT_OK;
  }
};

static double img_now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

static int image_save_impl(dint_engine* e, const char* path) {
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());                        // quiesce, as dint_snapshot_create
  std::vector<std::pair<void*, size_t>> regs;
  snapshot_regions(e, regs);
  for (auto& r : regs)
    if ((uintptr_t)r.first & 15) return set_err(DINT_EIO, "internal: a state region is not 16-byte aligned");
  const std::vector<ImgBlock> blocks = img_blocks(regs);
  ImgHeader h{};
  memcpy(h.magic, kImgMagic, 8);
  h.version = kImgVersion;
  h.kind = (uint32_t)e->kind;
  h.cfg = e->cfg;
  h.n_regions = (uint32_t)regs.size();
  h.n_tables = e->ctx.n_tables;
  for (uint32_t t = 0; t < e->ctx.n_tables; t++) h.kv_capacity[t] = e->ctx.tbl[t].cap_mask + 1;
  h.tpool_cap = e->ctx.tpool_cap;
  std::vector<ImgRegion> rec(regs.size());
  for (uint32_t r = 0; r < regs.size(); r++) rec[r] = {r, 0, regs[r].second, (regs[r].second + kImgBlock - 1) / kImgBlock};

  ImgPipe P;
  { int rc = P.init(e, blocks.size()); if (rc) return rc; }
  int grid = 0;
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&grid, k_image_pack, kThreads, 0));
  grid *= e->sms;
  const std::string tmp = std::string(path) + ".tmp";
  ImgFd f;
  f.fd = open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
  if (f.fd < 0) return set_errf(DINT_EIO, "image %s: %s", tmp.c_str(), strerror(errno));
  auto fail = [&](int rc) { unlink(tmp.c_str()); return rc; };
  double t0 = img_now();
  if (!img_write(f.fd, &h, sizeof h) || !img_write(f.fd, rec.data(), rec.size() * sizeof(ImgRegion)))
    return fail(set_errf(DINT_EIO, "image %s: write: %s", tmp.c_str(), strerror(errno)));
  g_img_times[3] += img_now() - t0;
  HostRing& R = e->ring;
  const uint64_t N = blocks.size();
  std::vector<unsigned long long> sum(N), nset(N);
  // block j: packed on e->stream, copied to host set j % 3 on s_out, written to the file -- three blocks in flight
  for (uint64_t j = 0; j < N + 2; j++) {
    if (j < N) {
      const uint32_t b = (uint32_t)(j % kImgSets);
      if (j >= kImgSets) CU(cudaStreamWaitEvent(e->stream, R.d2h[b], 0));     // the set's previous block has left
      CU(cudaMemsetAsync(P.scratch, 0, ImgPipe::kBytes, e->stream));
      const ImgArgs a = P.args(blocks[j], R.in[b].p);
      CU(cudaEventRecord(P.ev[b][0], e->stream));
      k_image_pack<<<grid < (int)a.n_tiles ? grid : (int)a.n_tiles, kThreads, 0, e->stream>>>(a);
      CU(cudaGetLastError());
      CU(cudaEventRecord(P.ev[b][1], e->stream));
      e->stats.kernel_launches++;
      CU(cudaMemcpyAsync(P.meta + 2 * b, a.sum, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, e->stream));
      CU(cudaEventRecord(R.ready[b], e->stream));
    }
    if (j >= 1 && j - 1 < N) {
      const uint64_t k = j - 1;
      const uint32_t b = (uint32_t)(k % kImgSets);
      CU(cudaEventSynchronize(R.ready[b]));
      sum[k] = P.meta[2 * b];
      nset[k] = P.meta[2 * b + 1];
      CU(cudaStreamWaitEvent(R.s_out, R.ready[b], 0));
      CU(cudaEventRecord(P.ev[b][2], R.s_out));
      CU(cudaMemcpyAsync(P.host[b], R.in[b].p, img_words(blocks[k].bytes) * 4 + nset[k] * kImgLine, cudaMemcpyDeviceToHost, R.s_out));
      CU(cudaEventRecord(P.ev[b][3], R.s_out));
      CU(cudaEventRecord(R.d2h[b], R.s_out));
    }
    if (j >= 2) {
      const uint64_t k = j - 2;
      const uint32_t b = (uint32_t)(k % kImgSets);
      CU(cudaEventSynchronize(R.d2h[b]));
      { int rc = P.account(b); if (rc) return fail(rc); }
      const uint64_t words = img_words(blocks[k].bytes);
      const uint64_t bytes = words * 4 + img_stored_bytes(blocks[k].bytes, (const uint32_t*)P.host[b], nset[k]);
      t0 = img_now();
      if (!img_write(f.fd, P.host[b], bytes) || !img_write(f.fd, &sum[k], 8))
        return fail(set_errf(DINT_EIO, "image %s: write: %s", tmp.c_str(), strerror(errno)));
      g_img_times[3] += img_now() - t0;
    }
  }
  t0 = img_now();
  int rc = img_publish(tmp.c_str(), path, f.fd);
  g_img_times[3] += img_now() - t0;
  return rc ? fail(rc) : DINT_OK;
}

// Reads and checks an image's header and region table; touches no CUDA state.
static int image_read_header(int fd, const char* path, ImgHeader& h, std::vector<ImgRegion>& rec) {
  if (!img_read(fd, &h, sizeof h)) return set_errf(DINT_EIO, "image %s: truncated header", path);
  if (memcmp(h.magic, kImgMagic, 8) != 0) return set_errf(DINT_EINVAL, "image %s: bad magic (not a dint_b200 state image)", path);
  if (h.version != kImgVersion) return set_errf(DINT_EINVAL, "image %s: format version %u, this build reads %u", path, h.version, kImgVersion);
  if (h.kind >= DINT_NUM_KINDS) return set_errf(DINT_EINVAL, "image %s: unknown kind %u", path, h.kind);
  if (h.cfg.flags & ~kCfgKnownFlags) return set_errf(DINT_EINVAL, "image %s: unknown option flags 0x%x", path, h.cfg.flags & ~kCfgKnownFlags);
  if (h.n_regions > kImgMaxRegions || h.n_tables > kMaxTables) return set_errf(DINT_EINVAL, "image %s: %u regions, %u tables", path, h.n_regions, h.n_tables);
  for (uint32_t t = 0; t < h.n_tables; t++)
    if (h.kv_capacity[t] < 2 || h.kv_capacity[t] > (1ULL << 34) || (h.kv_capacity[t] & (h.kv_capacity[t] - 1)))
      return set_errf(DINT_EINVAL, "image %s: table %u has capacity %llu", path, t, (unsigned long long)h.kv_capacity[t]);
  rec.resize(h.n_regions);
  if (!img_read(fd, rec.data(), rec.size() * sizeof(ImgRegion))) return set_errf(DINT_EIO, "image %s: truncated region table", path);
  for (uint32_t r = 0; r < h.n_regions; r++)
    if (rec[r].index != r || rec[r].blocks != (rec[r].bytes + kImgBlock - 1) / kImgBlock)
      return set_errf(DINT_EINVAL, "image %s: region %u: bad record", path, r);
  return DINT_OK;
}

// want: the configuration a cluster gives this shard (the image must hold the same one; its chunk is the cluster's)
static int image_open_impl(const char* path, int device, const dint_cfg* want, dint_engine** out) {
  *out = nullptr;
  ImgFd f;
  f.fd = open(path, O_RDONLY);
  if (f.fd < 0) return set_errf(DINT_EIO, "image %s: %s", path, strerror(errno));
  ImgHeader h;
  std::vector<ImgRegion> rec;
  double t0 = img_now();
  { int rc = image_read_header(f.fd, path, h, rec); if (rc) return rc; }
  g_img_times[3] += img_now() - t0;
  dint_cfg cfg = h.cfg;
  for (uint32_t t = 0; t < h.n_tables; t++) {
    uint32_t lg = 0;
    while ((1ULL << lg) < h.kv_capacity[t]) lg++;
    cfg.kv_capacity_log2[t] = lg;                   // (a tatp engine with the eBPF tier keeps its unused tables at 2^10)
  }
  if (want) {
    dint_cfg a = h.cfg, b = *want;
    a.chunk = b.chunk = 0;
    memset(a.kv_capacity_log2, 0, sizeof a.kv_capacity_log2);
    memset(b.kv_capacity_log2, 0, sizeof b.kv_capacity_log2);
    if (memcmp(&a, &b, sizeof a) != 0) return set_errf(DINT_EINVAL, "image %s: its configuration is not this shard's", path);
    cfg.chunk = want->chunk;
  }
  dint_engine* e = nullptr;
  { int rc = dint_create((int)h.kind, &cfg, device, &e); if (rc) return rc; }
  EngineOwner own{e};
  std::vector<std::pair<void*, size_t>> regs;
  snapshot_regions(e, regs);
  if (regs.size() != h.n_regions || e->ctx.tpool_cap != h.tpool_cap)
    return set_errf(DINT_EINVAL, "image %s: %u regions, this build lays the engine out in %u", path, h.n_regions, (uint32_t)regs.size());
  for (uint32_t r = 0; r < regs.size(); r++)
    if (regs[r].second != rec[r].bytes)
      return set_errf(DINT_EINVAL, "image %s: region %u holds %llu bytes, this build lays out %llu", path, r,
                      (unsigned long long)rec[r].bytes, (unsigned long long)regs[r].second);
  const std::vector<ImgBlock> blocks = img_blocks(regs);
  const uint64_t N = blocks.size();
  ImgPipe P;
  { int rc = P.init(e, N); if (rc) return rc; }
  int grid = 0;
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&grid, k_image_unpack, kThreads, 0));
  grid *= e->sms;
  HostRing& R = e->ring;
  // block j: read into host set j % 3, copied to the device on s_in, checked and unpacked on e->stream
  for (uint64_t j = 0; j < N; j++) {
    const uint32_t b = (uint32_t)(j % kImgSets);
    const ImgBlock& k = blocks[j];
    if (j >= kImgSets) {                                // the set's previous block is unpacked
      CU(cudaEventSynchronize(R.released[b]));
      int rc = P.account(b);
      if (rc) return rc;
    }
    const uint64_t words = img_words(k.bytes);
    uint32_t* bm = (uint32_t*)P.host[b];
    uint8_t* lines = P.host[b] + words * 4;
    unsigned long long expect = 0;
    t0 = img_now();
    if (!img_read(f.fd, bm, words * 4)) return set_errf(DINT_EIO, "image %s: region %u block %llu: short read", path, k.region, (unsigned long long)k.index);
    uint64_t n_set = 0;
    for (uint64_t w = 0; w < words; w++) n_set += (uint64_t)__builtin_popcount(bm[w]);
    if (n_set > img_lines(k.bytes)) return set_errf(DINT_EIO, "image %s: region %u block %llu: checksum mismatch (bitmap)", path, k.region, (unsigned long long)k.index);
    const uint64_t stored = img_stored_bytes(k.bytes, bm, n_set);
    if (!img_read(f.fd, lines, stored) || !img_read(f.fd, &expect, 8))
      return set_errf(DINT_EIO, "image %s: region %u block %llu: short read", path, k.region, (unsigned long long)k.index);
    memset(lines + stored, 0, n_set * kImgLine - stored);   // a partial last line is hashed and staged zero-padded
    g_img_times[3] += img_now() - t0;
    if (j >= kImgSets) CU(cudaStreamWaitEvent(R.s_in, R.released[b], 0));
    CU(cudaEventRecord(P.ev[b][2], R.s_in));
    CU(cudaMemcpyAsync(R.in[b].p, P.host[b], words * 4 + n_set * kImgLine, cudaMemcpyHostToDevice, R.s_in));
    CU(cudaEventRecord(P.ev[b][3], R.s_in));
    CU(cudaEventRecord(R.h2d[b], R.s_in));
    CU(cudaStreamWaitEvent(e->stream, R.h2d[b], 0));
    CU(cudaMemsetAsync(P.scratch, 0, ImgPipe::kBytes, e->stream));
    ImgArgs a = P.args(k, R.in[b].p);
    a.expect = expect;
    a.bad = P.bad + j;
    CU(cudaEventRecord(P.ev[b][0], e->stream));
    CU(launch_ex(e, k_image_unpack, grid, kThreads, 0, e->stream, true, a));
    CU(cudaEventRecord(P.ev[b][1], e->stream));
    CU(cudaEventRecord(R.released[b], e->stream));
    e->stats.kernel_launches++;
  }
  {
    uint8_t extra;
    if (read(f.fd, &extra, 1) != 0) return set_errf(DINT_EINVAL, "image %s: bytes after the last block", path);
  }
  CU(cudaStreamSynchronize(e->stream));
  for (uint64_t j = N > kImgSets ? N - kImgSets : 0; j < N; j++) { int rc = P.account((uint32_t)(j % kImgSets)); if (rc) return rc; }
  std::vector<uint32_t> bad(N);
  if (N) CU(cudaMemcpy(bad.data(), P.bad, 4 * N, cudaMemcpyDeviceToHost));
  for (uint64_t j = 0; j < N; j++)
    if (bad[j]) return set_errf(DINT_EIO, "image %s: region %u block %llu: checksum mismatch", path, blocks[j].region, (unsigned long long)blocks[j].index);
  { int rc = engine_ready(e); if (rc) return rc; }
  own.e = nullptr;
  *out = e;
  return DINT_OK;
}

static std::string img_shard_path(const char* dir, uint32_t r) { return std::string(dir) + "/shard-" + std::to_string(r) + ".img"; }
static std::string img_manifest_path(const char* dir) { return std::string(dir) + "/manifest"; }

extern "C" {

int dint_image_save(dint_engine* e, const char* path) {
  if (!e || !path) return set_err(DINT_EINVAL, "null argument");
  for (double& t : g_img_times) t = 0;
  const double t0 = img_now();
  const int rc = image_save_impl(e, path);
  g_img_times[0] = img_now() - t0;
  return rc;
}

int dint_image_open(const char* path, int device, dint_engine** out) {
  if (!path || !out) return set_err(DINT_EINVAL, "null argument");
  *out = nullptr;
  for (double& t : g_img_times) t = 0;
  const double t0 = img_now();
  const int rc = image_open_impl(path, device, nullptr, out);
  g_img_times[0] = img_now() - t0;
  return rc;
}

int dint_image_times(double out[4]) {
  if (!out) return DINT_EINVAL;
  for (int i = 0; i < 4; i++) out[i] = g_img_times[i];
  return DINT_OK;
}

// lock position of lock slot `slot` (= b + H j) of a table of the eBPF TATP / SmallBank tier: 4 b + j (kv.cuh, te_lock_pos)
static uint32_t te_lock_pos_host(const Ctx& c, int table, uint32_t slot) {
  const uint32_t H = c.tbkt_mod[table].d;
  return c.tbl[table].grp_base + 4 * (slot % H) + slot / H;
}

int dint_lock_state(dint_engine* e, int table, uint32_t slot, uint32_t out[2]) {
  if (!e || !out) return DINT_EINVAL;
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  out[0] = out[1] = 0;
  const Ctx& c = e->ctx;
  uint32_t g = slot;
  if (e->kind == DINT_TATP || e->kind == DINT_SMALLBANK) {
    if (table < 0 || table >= (int)c.n_tables) return DINT_EINVAL;
    if (slot % c.n_shards != c.shard_id) return DINT_EINVAL;
    g = c.tbl[table].grp_base + slot / c.n_shards;
    if (c.tchain || sbe_on(e)) {
      if (slot >= c.tbl[table].n_groups) return DINT_EINVAL;   // 4H lock slots per table
      g = te_lock_pos_host(c, table, slot);
    }
  } else if (e->kind == DINT_LOCK2PL || e->kind == DINT_FASST) {
    if (slot % c.n_shards != c.shard_id) return DINT_EINVAL;
    g = slot / c.n_shards;
  } else return DINT_EINVAL;
  if (g >= e->total_groups) return DINT_EINVAL;
  if (e->kind == DINT_LOCK2PL || e->kind == DINT_SMALLBANK) {
    uint2 v;
    CU(cudaMemcpy(&v, c.cnt2 + g, sizeof v, cudaMemcpyDeviceToHost));
    out[0] = v.x; out[1] = v.y;
  } else {
    uint32_t w;
    CU(cudaMemcpy(&w, c.lockbits + (g >> 5), 4, cudaMemcpyDeviceToHost));
    out[0] = (w >> (g & 31)) & 1u;
    if (e->kind == DINT_FASST) CU(cudaMemcpy(&out[1], c.ver + g, 4, cudaMemcpyDeviceToHost));
  }
  return DINT_OK;
}

int dint_lock_holder(dint_engine* e, int table, uint32_t slot, uint64_t* key) {
  if (!e || !key || !e->ctx.holder) return DINT_EINVAL;
  const Ctx& c = e->ctx;
  if (table < 0 || table >= (int)c.n_tables || slot % c.n_shards != c.shard_id || slot / c.n_shards >= c.tbl[table].n_groups) return DINT_EINVAL;
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  const uint32_t g = c.tchain ? te_lock_pos_host(c, table, slot) : c.tbl[table].grp_base + slot / c.n_shards;
  CU(cudaMemcpy(key, c.holder + g, sizeof *key, cudaMemcpyDeviceToHost));
  return DINT_OK;
}

uint32_t dint_lock_slot(dint_engine* e, int table, uint64_t k) {
  if (!e) return 0;
  const Ctx& c = e->ctx;
  if (e->kind == DINT_LOCK2PL || e->kind == DINT_FASST) return fast_mod(fasthash64_u32((uint32_t)k), c.slot_mod);
  if ((e->kind == DINT_TATP || e->kind == DINT_SMALLBANK) && table >= 0 && table < (int)c.n_tables)
    return fast_mod(fasthash64_u64(k), c.tbl[table].lock_mod);
  return 0;
}

int dint_dump_log(dint_engine* e, void* out, uint64_t* appended) {
  if (!e || !e->has_log) return DINT_EINVAL;
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  if (out) CU(cudaMemcpy(out, e->ctx.ring, (size_t)e->ctx.ring_n * kLogEntry[e->kind], cudaMemcpyDeviceToHost));
  if (appended) {
    unsigned long long t[2];
    CU(cudaMemcpy(t, e->ctx.log_total, sizeof t, cudaMemcpyDeviceToHost));
    *appended = t[0];
  }
  return DINT_OK;
}

int dint_get_stats(dint_engine* e, dint_stats* s) {
  if (!e || !s) return DINT_EINVAL;
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  int rc = pull_counters(e);
  if (rc) return rc;
  *s = e->stats;
  return DINT_OK;
}
void dint_reset_stats(dint_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  cudaMemset(e->ctx.counters, 0, kNumCounters * sizeof(unsigned long long));
  e->stats = dint_stats{};
  for (int i = 0; i < KT_NUM; i++) { e->kt_ms[i] = 0; e->kt_n[i] = 0; }
}
int dint_profile(dint_engine* e, int enable) {
  if (!e) return DINT_EINVAL;
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  int rc = prof_flush(e);
  e->profiling = enable < 0 ? 0u : (uint32_t)enable == 1u ? 0xffffffffu : (uint32_t)enable;   // 1 = all kernels; else a bit mask
  return rc;
}
int dint_kernel_times(dint_engine* e, dint_kernel_time* out, int max_entries) {
  if (!e || !out) return DINT_EINVAL;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  prof_flush(e);
  int k = 0;
  for (int i = 0; i < KT_NUM && k < max_entries; i++) {
    if (!e->kt_n[i]) continue;
    memset(&out[k], 0, sizeof out[k]);
    snprintf(out[k].name, sizeof out[k].name, "%s", kKernelNames[i]);
    out[k].launches = e->kt_n[i];
    out[k].total_ms = e->kt_ms[i];
    k++;
  }
  return k;
}

// ---- KV entry points (store / tatp / smallbank) -------------------------------------------------------
// With the eBPF cache tier a (key, value) pair enters as the client's kInsert would (store/caladan/client_ebpf.cc:137-180):
// through the tier, so the cache sets, dirty bits and bloom words are the ones the reference server would hold.  Keys
// of another shard's buckets are skipped, as k_kv_load skips them.
static int ec_serve_inserts(dint_engine* e, const uint64_t* keys, const uint8_t* vals, uint64_t n) {
  using W = Wire<K_STORE_EBPF>;
  const Ctx& c = e->ctx;
  const uint64_t batch = 1u << 20;
  std::vector<uint8_t> buf((size_t)batch * W::MSG);
  for (uint64_t off = 0; off < n;) {
    uint64_t m = 0;
    for (; off < n && m < batch; off++) {
      const uint32_t g = fast_mod(fasthash64_u64(keys[off]), c.tbl[0].lock_mod);
      if (g % c.n_shards != c.shard_id) continue;
      uint8_t* r = buf.data() + (size_t)m++ * W::MSG;
      memset(r, 0, W::MSG);
      r[W::TYPE] = 2;                                   // kInsert, ver 0
      memcpy(r + W::KEY, &keys[off], 8);
      memcpy(r + W::VAL, vals + (size_t)off * W::VALSZ, W::VALSZ);
    }
    if (m == 0) continue;
    int rc = dint_submit(e, buf.data(), m, buf.data());
    if (rc) return rc;
  }
  return DINT_OK;
}

// With the eBPF TATP tier a row enters as its client's insert would (tatp/caladan/client_ebpf_shard.cc:96-339): through
// the tier.  `placed` (dint_populate): kInsertPrim where this engine is the row's primary (key % 3 == txn_shard_id with
// the reference's three shards, key % G with G = txn_shards > 3), kInsertBck where it is a backup -- KvBatch already
// dropped the rows of which it is no replica.  Otherwise (dint_load) kInsertBck throughout, which leaves the lock words
// alone.
static int te_serve_inserts(dint_engine* e, int table, const uint64_t* keys, const uint8_t* vals, uint64_t n, bool placed) {
  using W = Wire<K_TATP_EBPF>;
  const uint32_t G = e->cfg.txn_shards > 3 ? e->cfg.txn_shards : 3, me = e->cfg.txn_shard_id;
  const uint64_t batch = 1u << 20;
  std::vector<uint8_t> buf((size_t)(n < batch ? n : batch) * W::MSG);
  for (uint64_t off = 0; off < n;) {
    uint64_t m = 0;
    for (; off < n && m < batch; off++) {
      uint8_t* r = buf.data() + (size_t)m++ * W::MSG;
      memset(r, 0, W::MSG);
      r[W::TYPE] = placed && keys[off] % G == me ? 18 : 19;
      r[W::TABLE] = (uint8_t)table;
      memcpy(r + W::KEY, &keys[off], 8);
      memcpy(r + W::VAL, vals + (size_t)off * W::VALSZ, W::VALSZ);
    }
    int rc = dint_submit(e, buf.data(), m, buf.data());
    if (rc) return rc;
  }
  return DINT_OK;
}

int dint_load(dint_engine* e, int table, const uint64_t* keys, const void* vals, uint64_t n) {
  if (!e || table < 0 || table >= (int)e->ctx.n_tables || (n && (!keys || !vals))) return set_err(DINT_EINVAL, "bad table/arguments");
  CU(cudaSetDevice(e->device));
  if (e->ctx.tchain) return te_serve_inserts(e, table, keys, (const uint8_t*)vals, n, false);
  if (e->ctx.ecache && e->kind == DINT_STORE) return ec_serve_inserts(e, keys, (const uint8_t*)vals, n);
  const uint32_t vs = kValSize[e->kind];
  const uint64_t batch = 1u << 20;
  uint64_t* dk = nullptr;
  uint8_t* dv = nullptr;
  CU(cudaMalloc(&dk, batch * 8));
  cudaError_t ce = cudaMalloc(&dv, batch * vs);
  if (ce != cudaSuccess) { cudaFree(dk); return set_err(DINT_ENOMEM, "cudaMalloc", ce); }
  int rc = pull_counters(e);                      // failures are counted in counters[0]: compare against its value NOW, not against 0
  const unsigned long long err_before = e->stats.errors;
  for (uint64_t off = 0; off < n && rc == DINT_OK; off += batch) {
    uint64_t m = (n - off < batch) ? (n - off) : batch;
    if (cudaMemcpyAsync(dk, keys + off, m * 8, cudaMemcpyHostToDevice, e->stream) != cudaSuccess ||
        cudaMemcpyAsync(dv, (const uint8_t*)vals + off * vs, m * vs, cudaMemcpyHostToDevice, e->stream) != cudaSuccess) {
      rc = set_err(DINT_EIO, "load copy", cudaGetLastError());
      break;
    }
    {
      ProfScope ps(e, e->stream, KT_LOAD);
      kv_launch_load(e->kind, e->ctx, table, dk, dv, (uint32_t)m, e->stream);
    }
    if (cudaStreamSynchronize(e->stream) != cudaSuccess) rc = set_err(DINT_EIO, "k_kv_load", cudaGetLastError());
  }
  cudaFree(dk);
  cudaFree(dv);
  if (rc == DINT_OK) {
    kv_publish_counts(e, e->stream);
    cudaStreamSynchronize(e->stream);
    int r2 = pull_counters(e);
    if (r2) return r2;
    if (e->stats.errors != err_before) return set_err(DINT_ENOMEM, "KV table full during load");
  }
  return rc;
}

// The eBPF SmallBank client's warm-up (smallbank/caladan/client_ebpf_shard.cc:88-169, 1526-1545): kWarmupRead of
// (saving, a) then (checking, a) for every account a < accts_populate this shard replicates (all of them with
// txn_shards <= 3; a % G in {I - 2, I - 1, I} with G = txn_shards > 3), ascending -- the 600 warm-up threads' slices
// taken in thread order.  Generated on the device (k_sbe_warmup) and served in batches through dint_submit_device.
static int sbe_warmup(dint_engine* e) {
  const uint64_t A = e->cfg.accts_populate;
  const uint32_t G = e->cfg.txn_shards, me = e->cfg.txn_shard_id;
  uint32_t per = 1, blk = 1;
  uint32_t r[3] = {0, 0, 0};
  uint64_t accts = A;
  if (G > 3) {
    per = 3; blk = G;
    for (uint32_t k = 0; k < 3; k++) r[k] = (me + G - 2 + k) % G;
    std::sort(r, r + 3);
    accts = A / G * 3;
    for (uint32_t k = 0; k < 3; k++) accts += r[k] < A % G;
  }
  const uint64_t n = 2 * accts, batch = 1u << 22;
  if (n == 0) return DINT_OK;
  using W = Wire<K_SMALLBANK_EBPF>;
  uint8_t *d_req = nullptr, *d_resp = nullptr;
  CU(cudaMalloc(&d_req, batch * W::MSG));
  cudaError_t ce = cudaMalloc(&d_resp, batch * W::MSG);
  if (ce != cudaSuccess) { cudaFree(d_req); return set_err(DINT_ENOMEM, "cudaMalloc", ce); }
  int rc = DINT_OK;
  for (uint64_t off = 0; off < n && rc == DINT_OK; off += batch) {
    const uint32_t m = (uint32_t)(n - off < batch ? n - off : batch);
    k_sbe_warmup<<<(m + 255) / 256, 256>>>(d_req, off, m, per, blk, make_uint4(r[0], r[1], r[2], 0));
    rc = dint_submit_device(e, d_req, m, d_resp, nullptr);
  }
  if (rc == DINT_OK && cudaDeviceSynchronize() != cudaSuccess) rc = set_err(DINT_EIO, "warm-up", cudaGetLastError());
  cudaFree(d_req);
  cudaFree(d_resp);
  return rc;
}

int dint_populate(dint_engine* e) {
  if (!e) return DINT_EINVAL;
  if (e->ctx.n_tables == 0) return DINT_OK;       // lock / log servers start from zeroed arrays
  if (e->ctx.tchain) {                            // so does the eBPF TATP server
    return tatp_ebpf_populate(e->cfg, [&](int table, const uint64_t* k, const void* v, uint64_t n) {
      return te_serve_inserts(e, table, k, (const uint8_t*)v, n, true);
    });
  }
  if (sbe_on(e)) {                                // the eBPF SmallBank server: kvs_insert of every account, then
    int rc = kv_populate(e->kind, e->cfg, [&](int table, const uint64_t* k, const void* v, uint64_t n) {
      return dint_load(e, table, k, v, n);
    });
    return rc ? rc : sbe_warmup(e);               // ... its client's warm-up through the tier
  }
  if (e->ctx.ecache) {                            // the eBPF store starts empty and is filled over the wire
    return store_ebpf_populate(e->cfg, [&](int, const uint64_t* k, const void* v, uint64_t n) {
      return ec_serve_inserts(e, k, (const uint8_t*)v, n);
    });
  }
  return kv_populate(e->kind, e->cfg, [&](int table, const uint64_t* k, const void* v, uint64_t n) {
    return dint_load(e, table, k, v, n);
  });
}

// a 256-byte cache set as the reference's struct cache_entry (store/ebpf/utils.h:58-66 and tatp/ebpf/utils.h:103-111
// are the same 232 bytes)
static void ec_host_cache_entry(const uint8_t* s, uint8_t* o) {
  memset(o, 0, DINT_STORE_CACHE_ENTRY_BYTES);
  memcpy(o, s, 32);                                // key[4]
  memcpy(o + 32, s + 64, 160);                     // val[4][40]
  memcpy(o + 192, s + 32, 16);                     // ver[4]
  for (int i = 0; i < 4; i++) {
    o[208 + i] = (s[56] >> i) & 1;                 // valid[4]
    o[212 + i] = (s[57] >> i) & 1;                 // dirty[4]
  }
  memcpy(o + 216, s + 48, 8);                      // bloom_filter; lock (+224) = 0
}

// the chain of bucket `b` of `table`, head first: whole 256-byte entries, walked from the host
static int te_host_chain(dint_engine* e, int table, uint32_t b, std::vector<uint8_t>& out) {
  const Ctx& c = e->ctx;
  uint2 hd;
  CU(cudaMemcpy(&hd, c.tchain + c.tbl[table].grp_base / 4 + b, sizeof hd, cudaMemcpyDeviceToHost));
  for (uint32_t x = hd.x; x; ) {
    if (out.size() >= (size_t)c.tpool_cap * kTeEntBytes) return set_err(DINT_EIO, "chain does not end");
    out.resize(out.size() + kTeEntBytes);
    uint8_t* p = out.data() + out.size() - kTeEntBytes;
    CU(cudaMemcpy(p, c.tpool + (size_t)(x - 1) * kTeEntBytes, kTeEntBytes, cudaMemcpyDeviceToHost));
    memcpy(&x, p + 52, 4);
  }
  return DINT_OK;
}

int dint_kv_get(dint_engine* e, int table, uint64_t key, void* val, uint32_t* ver) {
  if (!e || table < 0 || table >= (int)e->ctx.n_tables) return DINT_EINVAL;
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  if (e->ctx.tchain) {                             // kvs_get on the chain (tatp/ebpf/kvs.h:38-53)
    const uint32_t b = fast_mod(fasthash64_u64(key), e->ctx.tbkt_mod[table]);
    std::vector<uint8_t> ch;
    int rc = te_host_chain(e, table, b, ch);
    if (rc) return rc;
    for (size_t o = 0; o < ch.size(); o += kTeEntBytes)
      for (int i = 0; i < 4; i++) {
        uint64_t k;
        memcpy(&k, &ch[o + 8 * i], 8);
        if (k != key || !((ch[o + 48] >> i) & 1)) continue;
        if (ver) memcpy(ver, &ch[o + 32 + 4 * i], 4);
        if (val) memcpy(val, &ch[o + 64 + 40 * i], 40);
        return 0;
      }
    return 1;
  }
  return kv_host_get(e->ctx, table, key, kValSize[e->kind], val, ver);
}

int dint_tatp_cache_set(dint_engine* e, int table, uint32_t bucket, void* out) {
  if (!e || !out || !e->ctx.tchain) return set_err(DINT_EINVAL, "not a tatp engine with the eBPF cache tier");
  const Ctx& c = e->ctx;
  if (table < 0 || table >= (int)c.n_tables || bucket >= c.tbkt_mod[table].d) return set_err(DINT_EINVAL, "bad table / bucket");
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  uint8_t s[kEcSetBytes];
  CU(cudaMemcpy(s, c.ecache + (size_t)(c.tbl[table].grp_base / 4 + bucket) * kEcSetBytes, sizeof s, cudaMemcpyDeviceToHost));
  ec_host_cache_entry(s, (uint8_t*)out);
  return DINT_OK;
}

int dint_tatp_chain(dint_engine* e, int table, uint32_t bucket, void* out, uint32_t max, uint32_t* n) {
  if (!e || !n || (max && !out) || !e->ctx.tchain) return set_err(DINT_EINVAL, "not a tatp engine with the eBPF cache tier");
  const Ctx& c = e->ctx;
  if (table < 0 || table >= (int)c.n_tables || bucket >= c.tbkt_mod[table].d) return set_err(DINT_EINVAL, "bad table / bucket");
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  std::vector<uint8_t> ch;
  int rc = te_host_chain(e, table, bucket, ch);
  if (rc) return rc;
  *n = (uint32_t)(ch.size() / kTeEntBytes);
  uint8_t* o = (uint8_t*)out;
  for (uint32_t k = 0; k < *n && k < max; k++, o += DINT_TATP_CHAIN_REC_BYTES) {
    const uint8_t* p = &ch[(size_t)k * kTeEntBytes];
    memcpy(o, p, 48);                              // key[4], ver[4]
    for (int i = 0; i < 4; i++) o[48 + i] = (p[48] >> i) & 1;   // valid[4]
    memcpy(o + 52, p + 64, 160);                   // val[4][40]
  }
  return DINT_OK;
}

int dint_tatp_cache_stats(dint_engine* e, uint64_t out[9]) {
  if (!e || !out || !e->ctx.tchain) return set_err(DINT_EINVAL, "not a tatp engine with the eBPF cache tier");
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpy(out, e->ctx.ecache_stats, EC_NSTATS_TATP * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  return DINT_OK;
}

int dint_smallbank_cache_set(dint_engine* e, int table, uint32_t bucket, void* out) {
  if (!e || !out || !sbe_on(e)) return set_err(DINT_EINVAL, "not a smallbank engine with the eBPF cache tier");
  const Ctx& c = e->ctx;
  if (table < 0 || table >= (int)c.n_tables || bucket >= c.tbkt_mod[table].d) return set_err(DINT_EINVAL, "bad table / bucket");
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  uint8_t s[kSbeSetBytes];
  CU(cudaMemcpy(s, c.ecache + (size_t)(c.tbl[table].grp_base / 4 + bucket) * kSbeSetBytes, sizeof s, cudaMemcpyDeviceToHost));
  uint8_t* o = (uint8_t*)out;                      // struct cache_entry, smallbank/ebpf/utils.h:82-89
  memset(o, 0, DINT_SMALLBANK_CACHE_ENTRY_BYTES);
  memcpy(o, s, 32);                                // key[4]
  memcpy(o + 32, s + 64, 32);                      // val[4][8]
  memcpy(o + 64, s + 32, 16);                      // ver[4]
  for (int i = 0; i < 4; i++) {
    o[80 + i] = (s[48] >> i) & 1;                  // valid[4]
    o[84 + i] = (s[49] >> i) & 1;                  // dirty[4]; lock (+88) = 0
  }
  return DINT_OK;
}

int dint_smallbank_cache_stats(dint_engine* e, uint64_t out[4]) {
  if (!e || !out || !sbe_on(e)) return set_err(DINT_EINVAL, "not a smallbank engine with the eBPF cache tier");
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpy(out, e->ctx.ecache_stats, SBE_NSTATS * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  return DINT_OK;
}

int dint_store_cache_set(dint_engine* e, uint32_t bucket, void* out) {
  if (!e || !out || !e->ctx.ecache || e->kind != DINT_STORE) return set_err(DINT_EINVAL, "not a store engine with the eBPF cache tier");
  const Ctx& c = e->ctx;
  if (bucket % c.n_shards != c.shard_id || bucket / c.n_shards >= e->total_groups) return set_err(DINT_EINVAL, "bucket of another shard");
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  uint8_t s[kEcSetBytes];
  CU(cudaMemcpy(s, c.ecache + (size_t)(bucket / c.n_shards) * kEcSetBytes, sizeof s, cudaMemcpyDeviceToHost));
  ec_host_cache_entry(s, (uint8_t*)out);
  return DINT_OK;
}

int dint_store_cache_stats(dint_engine* e, uint64_t out[5]) {
  if (!e || !out || !e->ctx.ecache || e->kind != DINT_STORE) return set_err(DINT_EINVAL, "not a store engine with the eBPF cache tier");
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpy(out, e->ctx.ecache_stats, EC_NSTATS * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  return DINT_OK;
}

int64_t dint_kv_count(dint_engine* e, int table) {
  if (!e || table < 0 || table >= (int)e->ctx.n_tables) return DINT_EINVAL;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  unsigned long long v = 0;
  if (e->ctx.tchain) {                             // valid slots of the table's chains
    unsigned long long* d = nullptr;
    uint32_t top = 0;
    if (cudaMemcpy(&top, e->ctx.tpool_top, 4, cudaMemcpyDeviceToHost) != cudaSuccess) return DINT_EIO;
    if (top > e->ctx.tpool_cap) top = e->ctx.tpool_cap;
    if (cudaMalloc(&d, 8) != cudaSuccess) return DINT_ENOMEM;
    cudaMemset(d, 0, 8);
    k_tchain_count<<<e->sms > 0 ? e->sms * 4 : 64, 256>>>(e->ctx, (uint32_t)table, top, d);
    cudaError_t ce = cudaMemcpy(&v, d, 8, cudaMemcpyDeviceToHost);
    cudaFree(d);
    return ce == cudaSuccess ? (int64_t)v : DINT_EIO;
  }
  if (cudaMemcpy(&v, e->ctx.tbl[table].live, 8, cudaMemcpyDeviceToHost) != cudaSuccess) return DINT_EIO;
  return (int64_t)v;
}

}  // extern "C"

// ---- the whole sharded step over NVLink peer memory ---------------------------------------------------------
// A "rank" = one engine (one shard of the key space) with three streams: `side` partitions batch j+1 into the
// OWNERS' inboxes (dispatch), the caller's stream runs the engine on batch j -- K2 stores every reply tile
// straight into its SOURCE's return buffer (Ctx::seg_resp; posted stores over NVLink) -- and `ret` reassembles
// the replies of batch j-1 from the local return buffer (combine).  Cross-GPU synchronisation: two arrays of
// epoch words per rank (requests written / replies written; st.release.sys / ld.acquire.sys, bounded spin);
// buffer reuse needs no third flag: a source re-fills inbox set s only after its combine of the batch that used
// it, i.e. after every owner's "replies written", and an owner re-fills return-buffer set s only after the
// source's next dispatch into that set arrived, which the source ordered behind its combine.
// Ranks may live in different processes (one per GPU, buffers mapped through CUDA IPC / torch symmetric memory:
// dint_shard_*) or in ONE process (dint_cluster_*: cudaMalloc + peer access; several ranks may even share a
// device, then everything runs on one stream in dependency order).
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

static int shard_make(dint_engine* e, uint32_t n_shards, uint32_t rank, uint32_t cap, uint32_t n_sets, const dint_peer_ptrs* inbox_sets,
                      const dint_peer_ptrs* retbox_sets, const dint_peer_ptrs* sig_blocks, uint64_t max_n, bool one_stream,
                      dint_shard_ctx** out) {
  if (!e || !out || !inbox_sets || !retbox_sets || !sig_blocks || n_shards == 0 || n_shards > kMaxShards || rank >= n_shards || cap == 0 ||
      cap % kTile != 0 || n_sets < 2 || n_sets > (uint32_t)kMaxSets || max_n == 0 || max_n > 0xffffffffULL)
    return set_err(DINT_EINVAL, "bad argument (cap must be a multiple of 128, 2 <= n_sets <= 4)");
  CU(cudaSetDevice(e->device));
  dint_shard_ctx* c = new dint_shard_ctx();
  e->plain_launches = true;
  c->e = e; c->W = n_shards; c->me = rank; c->cap = cap; c->S = n_sets; c->max_n = max_n; c->one_stream = one_stream;
  for (uint32_t s = 0; s < n_sets; s++)
    for (uint32_t o = 0; o < n_shards; o++) {
      c->inbox[s][o] = inbox_sets[s].p[o];
      c->retbox[s][o] = retbox_sets[s].p[o];
    }
  for (uint32_t o = 0; o < n_shards; o++) {
    c->sigreq.p[o] = sig_blocks->p[o];
    c->sigrsp.p[o] = sig_blocks->p[o] + 128;          // signal block: request flags [n_sets][8] at +0, reply flags [8] at +128
  }
  c->my_req = (uint32_t*)sig_blocks->p[rank];
  c->my_rsp = (uint32_t*)(sig_blocks->p[rank] + 128);
  if (!c->one_stream) {
    CU(cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&c->ret, cudaStreamNonBlocking));
  }
  CU(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
  const uint32_t tr = route_tile_records(e);
  const size_t tiles = (size_t)((max_n + tr - 1) / tr);
  for (uint32_t s = 0; s < n_sets; s++) {
    CU(cudaEventCreateWithFlags(&c->ev_disp[s], cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&c->ev_comb[s], cudaEventDisableTiming));
    CU(cudaMalloc(&c->owner[s], max_n + 16));
    CU(cudaMalloc(&c->tilebase[s], tiles * kMaxShards * sizeof(uint32_t)));
  }
  CU(cudaMalloc(&c->flags, 4 * sizeof(uint32_t)));        // [0] records that did not fit, [1] timed-out waits, [2] first epoch left unserved
  CU(cudaMemset(c->flags, 0, 4 * sizeof(uint32_t)));
  c->trace = getenv("DINT_SHARD_TRACE") != nullptr;
  *out = c;
  return DINT_OK;
}

// ---- the three phases of one batch on one rank (all asynchronous) -------------------------------------------
static void shard_mark(dint_shard_ctx* c, uint32_t slot, int which, cudaStream_t st) {
  if (!c->trace) return;
  const size_t need = (size_t)6 * (slot + 1);
  while (c->tev.size() < need) { cudaEvent_t ev; cudaEventCreate(&ev); c->tev.push_back(ev); }
  cudaEventRecord(c->tev[(size_t)6 * slot + which], st);
}
// dispatch: partition n records of this rank into the owners' inbox set (epoch ep)
// (cap: the slab capacity THIS batch uses, <= the capacity the buffers were laid out for and the same on every rank: a
//  batch much smaller than max_n then does not make the owners wade through padding)
static int shard_dispatch(dint_shard_ctx* c, uint32_t slot, uint32_t ep, const void* req_dev, const uint8_t* dst_dev, uint64_t n, uint32_t cap, cudaStream_t st) {
  dint_engine* e = c->e;
  CU(cudaSetDevice(e->device));
  const uint32_t s = ep % c->S;
  const size_t slab = (size_t)cap * e->msg;
  if (ep > c->S && !c->one_stream) CU(cudaStreamWaitEvent(st, c->ev_comb[s], 0));   // my combine of batch ep - S: every owner is done with inbox set s
  shard_mark(c, slot, 0, st);
  dint_peer_ptrs in{}, sg{};
  // one request-flag word per (buffer set, source): the flag of epoch ep -- which may carry the overflow bit -- is not
  // overwritten before the owner has consumed it (the source reuses set s only after the owners' replies of ep)
  for (uint32_t o = 0; o < c->W; o++) { in.p[o] = c->inbox[s][o] + (uint64_t)c->me * slab; sg.p[o] = c->sigreq.p[o] + (uint64_t)s * 32; }
  int rc = dint_route_dispatch(e, req_dev, dst_dev, n, c->W, c->me, cap, &in, &sg, ep, c->owner[s], c->tilebase[s], c->flags, st);
  if (rc) return rc;
  shard_mark(c, slot, 1, st);
  if (!c->one_stream) CU(cudaEventRecord(c->ev_disp[s], st));
  return DINT_OK;
}
// engine: this rank's shard serves inbox set (epoch ep); every reply tile goes to its source's return buffer
static int shard_engine(dint_shard_ctx* c, uint32_t slot, uint32_t ep, uint32_t cap, cudaStream_t st) {
  dint_engine* e = c->e;
  CU(cudaSetDevice(e->device));
  const uint32_t s = ep % c->S;
  const size_t slab = (size_t)cap * e->msg;
  k_p2p_wait<<<1, 32, 0, st>>>(c->my_req + s * 8, c->W, ep, c->flags + 1, c->flags + 2);     // every source's slab has arrived (or one did not fit)
  shard_mark(c, slot, 2, st);
  StepTarget tgt{cap / kTile, {}, true, c->flags + 2};
  for (uint32_t r = 0; r < c->W; r++) tgt.seg_resp[r] = c->retbox[s][r] + (uint64_t)c->me * slab;   // my slab inside source r's return buffer
  int rc = run_device(e, (const uint8_t*)c->inbox[s][c->me], (uint64_t)c->W * cap, nullptr, st, &tgt);
  if (rc) return rc;
  k_p2p_signal<<<1, 32, 0, st>>>(c->sigrsp, c->W, c->me, ep);
  shard_mark(c, slot, 3, st);
  e->stats.kernel_launches += 2;
  return DINT_OK;
}
// combine: the replies of batch ep are in my return-buffer set; put them back in request order
static int shard_combine(dint_shard_ctx* c, uint32_t slot, uint32_t ep, void* out_dev, uint64_t n, uint32_t cap, cudaStream_t st) {
  dint_engine* e = c->e;
  CU(cudaSetDevice(e->device));
  const uint32_t s = ep % c->S;
  const size_t slab = (size_t)cap * e->msg;
  if (!c->one_stream) CU(cudaStreamWaitEvent(st, c->ev_disp[s], 0));
  k_p2p_wait<<<1, 32, 0, st>>>(c->my_rsp, c->W, ep, c->flags + 1, nullptr);
  shard_mark(c, slot, 4, st);
  dint_peer_ptrs rb{};
  for (uint32_t o = 0; o < c->W; o++) rb.p[o] = c->retbox[s][c->me] + (uint64_t)o * slab;
  int rc = dint_route_combine(e, &rb, c->owner[s], c->tilebase[s], n, c->W, cap, out_dev, st);
  if (rc) return rc;
  shard_mark(c, slot, 5, st);
  if (!c->one_stream) CU(cudaEventRecord(c->ev_comb[s], st));
  e->stats.kernel_launches += 1;
  return DINT_OK;
}
static void shard_trace_collect(dint_shard_ctx* c, uint32_t k) {
  if (!c->trace) return;
  cudaSetDevice(c->e->device);
  cudaDeviceSynchronize();
  static const int pairs[4][2] = {{0, 1}, {2, 3}, {4, 5}, {0, 5}};
  for (uint32_t j = 0; j < k && (size_t)6 * (j + 1) <= c->tev.size(); j++)
    for (int q = 0; q < 4; q++) {
      float ms = 0;
      if (cudaEventElapsedTime(&ms, c->tev[(size_t)6 * j + pairs[q][0]], c->tev[(size_t)6 * j + pairs[q][1]]) == cudaSuccess) c->tsum[q] += ms;
    }
  c->tcount += k;
}

// One pipelined sequence of k batches over the ranks of THIS process (1 in the one-process-per-GPU deployment,
// G in a cluster).  Host enqueue order per batch: every rank's dispatch of j+1, every rank's engine of j, every
// rank's combine of j (of j-1 when the ranks share one stream) -- each phase only waits for phases enqueued
// before it, on this or another GPU, so one host thread can drive all ranks without blocking.
struct ShardBatch { const void* req; const uint8_t* dst; void* out; uint64_t n; uint32_t cap = 0; };   // cap: slab records of this batch (0 = the full capacity)
struct HostBatch { const uint8_t* req; const uint8_t* dst; uint8_t* out; uint64_t n; };
// `host` given: the batches come from / go to HOST memory through S sets of each rank's engine ring (HostRing) --
// H2D of batch j+1 and D2H of batch j-1 run on the ring's copy streams next to the exchange of batch j.
static int shard_run(dint_shard_ctx* const* ranks, uint32_t R, uint32_t k, std::vector<std::vector<ShardBatch>>& b, cudaStream_t const* mains,
                     const std::vector<std::vector<HostBatch>>* host = nullptr) {
  if (k == 0) return DINT_OK;
  const bool one = ranks[0]->one_stream;
  const uint32_t lag = one ? 1u : 0u;
  int rc;
  for (uint32_t r = 0; r < R; r++) {
    dint_shard_ctx* c = ranks[r];
    CU(cudaSetDevice(c->e->device));
    if (host && (rc = ring_reserve(c->e, c->S, c->max_n * c->e->msg, c->max_n, c->max_n * c->e->msg))) return rc;
    if (one) continue;
    CU(cudaEventRecord(c->ev_fork, mains[r]));
    CU(cudaStreamWaitEvent(c->side, c->ev_fork, 0));
    CU(cudaStreamWaitEvent(c->ret, c->ev_fork, 0));
  }
  auto side = [&](uint32_t r) { return one ? mains[r] : ranks[r]->side; };
  auto retS = [&](uint32_t r) { return one ? mains[r] : ranks[r]->ret; };
  auto dispatch = [&](uint32_t r, uint32_t j) -> int {
    dint_shard_ctx* c = ranks[r];
    if (host) {                                          // stage batch j: H2D on the ring's copy stream, the dispatch waits for it
      const HostBatch& h = (*host)[r][j];
      dint_engine* e = c->e;
      const uint32_t s = j % c->S;
      if (h.n > c->max_n) return set_err(DINT_EINVAL, "batch size");
      CU(cudaSetDevice(e->device));
      if (int rc2 = ring_stage_in(e, j, h.req, h.n * e->msg, h.dst, h.dst ? h.n : 0, side(r))) return rc2;
      b[r][j] = ShardBatch{e->ring.in[s].p, h.dst ? e->ring.aux[s].p : nullptr, e->ring.out[s].p, h.n, 0};
    }
    int rc2 = shard_dispatch(c, j, c->epoch + 1 + j, b[r][j].req, b[r][j].dst, b[r][j].n, b[r][j].cap ? b[r][j].cap : c->cap, side(r));
    if (!rc2 && host) CU(cudaEventRecord(c->e->ring.released[j % c->S], side(r)));   // nothing after the dispatch reads in / aux
    return rc2;
  };
  auto combine = [&](uint32_t r, uint32_t j) -> int {
    dint_shard_ctx* c = ranks[r];
    if (host && j >= c->S) CU(cudaStreamWaitEvent(retS(r), c->e->ring.d2h[j % c->S], 0));   // batch j - S's replies have left out[j % S]
    int rc2 = shard_combine(c, j, c->epoch + 1 + j, b[r][j].out, b[r][j].n, b[r][j].cap ? b[r][j].cap : c->cap, retS(r));
    if (rc2 || !host) return rc2;
    return ring_drain_out(c->e, j, (*host)[r][j].out, (*host)[r][j].n * c->e->msg, retS(r));
  };
  for (uint32_t r = 0; r < R; r++)
    if ((rc = dispatch(r, 0))) return rc;
  for (uint32_t j = 0; j < k; j++) {
    if (j + 1 < k)
      for (uint32_t r = 0; r < R; r++)
        if ((rc = dispatch(r, j + 1))) return rc;
    for (uint32_t r = 0; r < R; r++)
      if ((rc = shard_engine(ranks[r], j, ranks[r]->epoch + 1 + j, b[r][j].cap ? b[r][j].cap : ranks[r]->cap, mains[r]))) return rc;
    if (j >= lag)
      for (uint32_t r = 0; r < R; r++)
        if ((rc = combine(r, j - lag))) return rc;
  }
  for (uint32_t j = k - (lag < k ? lag : k); j < k; j++)
    for (uint32_t r = 0; r < R; r++)
      if ((rc = combine(r, j))) return rc;
  for (uint32_t r = 0; r < R; r++) {
    dint_shard_ctx* c = ranks[r];
    const uint32_t last = c->epoch + k;
    c->epoch = last;
    if (one) continue;
    CU(cudaSetDevice(c->e->device));
    for (uint32_t s = 0; s < c->S && s < k; s++) CU(cudaStreamWaitEvent(mains[r], c->ev_comb[(last - s) % c->S], 0));   // join
    CU(cudaStreamWaitEvent(mains[r], c->ev_disp[last % c->S], 0));
  }
  CU(cudaGetLastError());
  if (host)
    for (uint32_t r = 0; r < R; r++) {                   // returns when every reply is in host memory
      CU(cudaSetDevice(ranks[r]->e->device));
      CU(cudaStreamSynchronize(ranks[r]->e->ring.s_out));
      CU(cudaStreamSynchronize(mains[r]));
    }
  for (uint32_t r = 0; r < R; r++) shard_trace_collect(ranks[r], k);
  return DINT_OK;
}

static int shard_run_host(dint_shard_ctx* const* ranks, uint32_t R, uint32_t k, const std::vector<std::vector<HostBatch>>& hb) {
  std::vector<cudaStream_t> mains(R);
  for (uint32_t r = 0; r < R; r++) mains[r] = ranks[0]->one_stream ? ranks[0]->e->stream : ranks[r]->e->stream;   // ranks sharing a device: one stream
  std::vector<std::vector<ShardBatch>> b(R, std::vector<ShardBatch>(k));
  return shard_run(ranks, R, k, b, mains.data(), &hb);
}

extern "C" {

int dint_shard_create(dint_engine* e, uint32_t n_shards, uint32_t rank, uint32_t cap, uint32_t n_sets, const dint_peer_ptrs* inbox_sets,
                      const dint_peer_ptrs* retbox_sets, const dint_peer_ptrs* sig_blocks, uint64_t max_n, dint_shard_ctx** out) {
  return shard_make(e, n_shards, rank, cap, n_sets, inbox_sets, retbox_sets, sig_blocks, max_n, false, out);
}

void dint_shard_destroy(dint_shard_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->e->device);
  cudaDeviceSynchronize();
  if (c->trace && c->tcount) {
    static const char* names[4] = {"dispatch", "engine", "combine", "dispatch start -> combine end"};
    fprintf(stderr, "[dint_shard rank %u] %llu batches, us per batch:", c->me, (unsigned long long)c->tcount);
    for (int q = 0; q < 4; q++) fprintf(stderr, " | %s %.1f", names[q], c->tsum[q] * 1e3 / (double)c->tcount);
    fprintf(stderr, "\n");
  }
  for (cudaEvent_t ev : c->tev) cudaEventDestroy(ev);
  for (uint32_t s = 0; s < c->S; s++) {
    if (c->ev_disp[s]) cudaEventDestroy(c->ev_disp[s]);
    if (c->ev_comb[s]) cudaEventDestroy(c->ev_comb[s]);
    if (c->owner[s]) cudaFree(c->owner[s]);
    if (c->tilebase[s]) cudaFree(c->tilebase[s]);
  }
  if (c->ev_fork) cudaEventDestroy(c->ev_fork);
  if (c->flags) cudaFree(c->flags);
  if (c->side) cudaStreamDestroy(c->side);
  if (c->ret) cudaStreamDestroy(c->ret);
  c->e->plain_launches = false;
  delete c;
}

int dint_shard_flags(dint_shard_ctx* c, uint32_t out[2]) {
  if (!c || !out) return DINT_EINVAL;
  CU(cudaSetDevice(c->e->device));
  CU(cudaDeviceSynchronize());
  CU(cudaMemcpy(out, c->flags, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  CU(cudaMemset(c->flags, 0, 2 * sizeof(uint32_t)));
  return DINT_OK;
}

// After a slab overflow: *first_unserved = index, inside the LAST submit call (of k batches), of the first batch that
// no shard served (it and every later batch left the state untouched; their replies are garbage), or 0xffffffff when
// nothing was skipped.  Clears the condition and the engine's inter-chunk bookkeeping; call it on every rank before the
// next submit, then serve the unserved batches again in pieces of at most `cap` records per rank (which cannot overflow).
int dint_shard_recover(dint_shard_ctx* c, uint32_t k_last, uint32_t* first_unserved) {
  if (!c || !first_unserved) return DINT_EINVAL;
  dint_engine* e = c->e;
  CU(cudaSetDevice(e->device));
  CU(cudaDeviceSynchronize());
  uint32_t bad = 0;
  CU(cudaMemcpy(&bad, c->flags + 2, sizeof bad, cudaMemcpyDeviceToHost));
  *first_unserved = 0xffffffffu;
  if (!bad) return DINT_OK;
  const uint32_t first_epoch = c->epoch - k_last + 1;
  *first_unserved = bad >= first_epoch ? bad - first_epoch : 0;
  CU(cudaMemset(c->flags, 0, 4 * sizeof(uint32_t)));
  // the skipped launches changed nothing on the device, but the host-side chunk bookkeeping advanced: start clean
  e->ord_pending = false;
  e->prev_n = 0;
  CU(cudaMemset(e->d_nc, 0, 8 * sizeof(uint32_t)));
  CU(cudaMemset(e->d_flags[0], 0, (size_t)((char*)e->d_flags[1] - (char*)e->d_flags[0]) * 2));
  CU(cudaDeviceSynchronize());
  return DINT_OK;
}

int dint_shard_submit_many(dint_shard_ctx* c, uint32_t k, const void* const* req_dev, const uint8_t* const* dst_dev, uint64_t n,
                           void* const* out_dev, void* cuda_stream) {
  if (!c || !req_dev || !out_dev || n == 0 || n > c->max_n) return set_err(DINT_EINVAL, "bad argument");
  if (k == 0) return DINT_OK;
  std::vector<std::vector<ShardBatch>> b(1, std::vector<ShardBatch>(k));
  for (uint32_t j = 0; j < k; j++) b[0][j] = ShardBatch{req_dev[j], dst_dev ? dst_dev[j] : nullptr, out_dev[j], n};
  cudaStream_t main = (cudaStream_t)cuda_stream;
  return shard_run(&c, 1, k, b, &main);
}

}  // extern "C"

extern "C" {

int dint_shard_submit_many_v(dint_shard_ctx* c, uint32_t k, const void* const* req_dev, const uint8_t* const* dst_dev, const uint64_t* n,
                             const uint32_t* cap, void* const* out_dev, void* cuda_stream) {
  if (!c || !req_dev || !out_dev || !n) return set_err(DINT_EINVAL, "bad argument");
  if (k == 0) return DINT_OK;
  std::vector<std::vector<ShardBatch>> b(1, std::vector<ShardBatch>(k));
  for (uint32_t j = 0; j < k; j++) {
    const uint32_t cj = cap ? cap[j] : 0;
    if (n[j] > c->max_n || cj > c->cap || cj % kTile != 0) return set_err(DINT_EINVAL, "batch size / slab capacity (a multiple of 128, <= the capacity of dint_shard_create)");
    b[0][j] = ShardBatch{req_dev[j], dst_dev ? dst_dev[j] : nullptr, out_dev[j], n[j], cj};
  }
  cudaStream_t main = (cudaStream_t)cuda_stream;
  return shard_run(&c, 1, k, b, &main);
}

int dint_shard_submit_host(dint_shard_ctx* c, uint32_t k, const void* const* req_host, const uint8_t* const* dst_host, uint64_t n,
                           void* const* out_host) {
  if (!c || !req_host || !out_host || n == 0 || n > c->max_n) return set_err(DINT_EINVAL, "bad argument");
  std::vector<std::vector<HostBatch>> hb(1, std::vector<HostBatch>(k));
  for (uint32_t j = 0; j < k; j++) hb[0][j] = HostBatch{(const uint8_t*)req_host[j], dst_host ? dst_host[j] : nullptr, (uint8_t*)out_host[j], n};
  return shard_run_host(&c, 1, k, hb);
}

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

// The exchange buffers of a cluster: per rank one allocation {inbox sets | return-buffer sets | signal block}
constexpr uint32_t kClusterSets = 3;
static size_t cluster_region(const dint_cluster* cl) { return ((size_t)cl->G * cl->cap * kMsgSize[cl->kind] + 255) / 256 * 256; }
static uint64_t cluster_sig_block(const dint_cluster* cl, uint32_t r) { return (uint64_t)cl->bufs[r] + 2 * kClusterSets * cluster_region(cl); }

// the configuration shard r of a cluster is created with (cl->base, cap and G set)
static dint_cfg cluster_shard_cfg(const dint_cluster* cl, uint32_t r) {
  dint_cfg c = cl->base;
  if (cl->by_dst) { c.n_shards = 1; c.shard_id = 0; c.txn_shards = cl->G; c.txn_shard_id = r; }
  else { c.n_shards = cl->G; c.shard_id = r; }
  const uint32_t chunk_need = (uint32_t)(((uint64_t)cl->G * cl->cap + kTile - 1) / kTile * kTile);
  if (c.chunk == 0 || c.chunk < chunk_need) c.chunk = chunk_need;        // one batch of the exchange = one engine chunk
  return c;
}

// one shard context per rank over the cluster's exchange buffers, engine r = eng[r]; every epoch starts at 0, so the
// signal blocks must be zero before the first batch
static int cluster_ranks(const dint_cluster* cl, const std::vector<dint_engine*>& eng, std::vector<dint_shard_ctx*>& out) {
  const uint32_t G = cl->G, S = kClusterSets;
  const size_t region = cluster_region(cl);
  for (uint32_t r = 0; r < G; r++) {
    dint_peer_ptrs in[kMaxSets]{}, rb[kMaxSets]{}, sig{};
    for (uint32_t s = 0; s < S; s++)
      for (uint32_t o = 0; o < G; o++) {
        in[s].p[o] = (uint64_t)cl->bufs[o] + (2 * s) * region;
        rb[s].p[o] = (uint64_t)cl->bufs[o] + (2 * s + 1) * region;
      }
    for (uint32_t o = 0; o < G; o++) sig.p[o] = cluster_sig_block(cl, o);
    dint_shard_ctx* c = nullptr;
    int rc = shard_make(eng[r], G, r, cl->cap, S, in, rb, &sig, cl->max_n, cl->shared_device, &c);
    if (rc) return rc;
    out.push_back(c);
  }
  return DINT_OK;
}

void dint_cluster_destroy(dint_cluster* cl) {
  if (!cl) return;
  for (auto* c : cl->sh) dint_shard_destroy(c);
  for (size_t r = 0; r < cl->bufs.size(); r++) { cudaSetDevice(cl->dev[r]); cudaFree(cl->bufs[r]); }
  for (auto* e : cl->eng) dint_destroy(e);
  delete cl;
}

}  // extern "C"

// ---- shards derived from other shards' state (dint_cluster_reshard, dint_cluster_rebuild) ---------------------------
static thread_local double g_reshard_times[3];       // dint_reshard_times: wall, re-shard kernels, count + allocation (s)
static thread_local double g_rebuild_times[3];       // dint_rebuild_times: wall, rebuild kernels, count + allocation (s)

// lets `device` (the current device) read `peer`'s memory; nothing to do when they are the same
static int peer_enable(int device, int peer) {
  if (peer == device) return DINT_OK;
  int can = 0;
  cudaDeviceCanAccessPeer(&can, device, peer);
  if (!can) return set_err(DINT_ENODEV, "GPUs without peer access");
  cudaError_t ce = cudaDeviceEnablePeerAccess(peer, 0);
  if (ce != cudaSuccess && ce != cudaErrorPeerAccessAlreadyEnabled) return set_err(DINT_EIO, "cudaDeviceEnablePeerAccess", ce);
  cudaGetLastError();
  return DINT_OK;
}

// waits for every device of cl
static int cluster_quiesce(const dint_cluster* cl) {
  for (uint32_t r = 0; r < cl->G; r++) {
    CU(cudaSetDevice(cl->dev[r]));
    CU(cudaDeviceSynchronize());
  }
  return DINT_OK;
}

// the shards a re-shard or rebuild reads
struct DeriveFrom {
  std::vector<dint_engine*> src;                    // per source shard: its engine (nullptr where a rebuild lost it)
  uint64_t rows[kMaxShards][kMaxTables] = {};        // the rows each destination shard receives, per table (count_rows)
};

// f.rows[d][t] += the FULL rows of table t of each engine of `read` (nullptr: not read) that go to destination shard d;
// dests_of(s, table) is k_kv_count_rows's filter for source s.  One small copy per source.
template <class DestsOf>
static int count_rows(DeriveFrom& f, const std::vector<dint_engine*>& read, DestsOf dests_of, const char* what) {
  for (uint32_t s = 0; s < read.size(); s++) {
    const dint_engine* e = read[s];
    if (!e || e->ctx.n_tables == 0) continue;
    CU(cudaSetDevice(e->device));
    unsigned long long* d = nullptr;
    unsigned long long h[kMaxTables][kMaxShards] = {};
    CU(cudaMalloc(&d, sizeof h));
    cudaError_t ce = cudaMemset(d, 0, sizeof h);
    for (uint32_t t = 0; t < e->ctx.n_tables && ce == cudaSuccess; t++) {
      k_kv_count_rows<<<e->sms * 4, kThreads>>>(e->ctx.tbl[t], dests_of(s, e->ctx.tbl[t]), d + t * kMaxShards);
      ce = cudaGetLastError();
    }
    if (ce == cudaSuccess) ce = cudaMemcpy(h, d, sizeof h, cudaMemcpyDeviceToHost);
    cudaFree(d);
    if (ce != cudaSuccess) return set_err(DINT_EIO, what, ce);
    for (uint32_t t = 0; t < kMaxTables; t++)
      for (uint32_t j = 0; j < kMaxShards; j++) f.rows[j][t] += h[t][j];
  }
  return DINT_OK;
}

// Shard j of a derived cluster, of `kind` on `device` with configuration c: created as dint_create would, with every KV
// table at least large enough to keep the rows[t] it receives at <= 35 % load (so kv_maintain leaves it as it is),
// given peer access to the engines of `read` (nullptr: not read), filled by fill(e) on its own stream, and made ready.
// What the fill does not write (a rebuild's lock words, holder keys and log ring) is that of a new engine.
// times[1] += the fill's CUDA-event time; times[2] += the sizing, allocation and peer set-up.
template <class Fill>
static int derive_engine(int kind, dint_cfg c, int device, uint32_t j, const uint64_t* rows, const std::vector<dint_engine*>& read,
                         double* times, Fill fill, dint_engine** out) {
  *out = nullptr;
  const double t0 = img_now();
  if (kind == DINT_STORE || kind == DINT_TATP || kind == DINT_SMALLBANK) {
    KvPlan P;
    if (kv_plan(kind, c, false, P) != DINT_OK) return set_err(DINT_EINVAL, "bad KV configuration");
    for (uint32_t t = 0; t < P.nt; t++) {
      const uint32_t lg = kv_fit_log2(P.lg[t], rows[t]);
      if (lg > 34)
        return kind == DINT_STORE ? set_errf(DINT_EINVAL, "re-shard: shard %u would receive %llu keys", j, (unsigned long long)rows[t])
                                  : set_errf(DINT_EINVAL, "%s: shard %u table %u would receive %llu rows",
                                             times == g_rebuild_times ? "rebuild" : "re-shard", j, t, (unsigned long long)rows[t]);
      c.kv_capacity_log2[t] = lg;
    }
  }
  dint_engine* e = nullptr;
  { int rc = dint_create(kind, &c, device, &e); if (rc) return rc; }
  EngineOwner own{e};
  for (const dint_engine* s : read)                    // the fill reads the sources' arrays where they are
    if (s) { int rc = peer_enable(device, s->device); if (rc) return rc; }
  times[2] += img_now() - t0;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  struct Events { cudaEvent_t* ev; ~Events() { for (int i = 0; i < 2; i++) if (ev[i]) cudaEventDestroy(ev[i]); } } evs{ev};
  for (cudaEvent_t& x : ev) CU(cudaEventCreate(&x));
  CU(cudaEventRecord(ev[0], e->stream));
  fill(e);
  CU(cudaGetLastError());
  CU(cudaEventRecord(ev[1], e->stream));
  CU(cudaEventSynchronize(ev[1]));
  float ms = 0;
  CU(cudaEventElapsedTime(&ms, ev[0], ev[1]));
  times[1] += ms * 1e-3;
  { int rc = engine_ready(e); if (rc) return rc; }
  own.e = nullptr;
  *out = e;
  return DINT_OK;
}

// Destination shard j of G2, filled from every source shard by the kernels of reshard.cuh (which has the ownership
// arithmetic); tatp / smallbank with ReplicaKeep (rebuild.cuh, which has the replica arithmetic)
static int reshard_engine(const DeriveFrom& f, uint32_t j, uint32_t G2, int kind, const dint_cfg& c, int device, dint_engine** out) {
  const uint32_t G = (uint32_t)f.src.size();
  return derive_engine(kind, c, device, j, f.rows[j], f.src, g_reshard_times, [&](dint_engine* e) {
    const Ctx& d = e->ctx;
    const cudaStream_t s = e->stream;
    ReshardArgs a{};
    a.G = G; a.G2 = G2; a.j = j; a.src_div = make_fastmod(G);
    a.n_local = (uint32_t)e->total_groups;
    a.n_global = kind == DINT_STORE ? e->kv[0].hash_size : e->cfg.lock_slots;
    const int grid = e->sms * 4;
    if (kind == DINT_LOCK2PL) {
      for (uint32_t r = 0; r < G; r++) a.src[r] = (uint64_t)f.src[r]->ctx.cnt2;
      a.dst = d.cnt2;
      k_reshard_lock<K_LOCK2PL><<<grid, kThreads, 0, s>>>(a);
    } else if (kind == DINT_FASST) {
      for (uint32_t r = 0; r < G; r++) { a.src[r] = (uint64_t)f.src[r]->ctx.ver; a.src_bits[r] = (uint64_t)f.src[r]->ctx.lockbits; }
      a.dst = d.ver;
      a.dst_bits = d.lockbits;
      k_reshard_lock<K_FASST><<<grid, kThreads, 0, s>>>(a);
    } else if (kind == DINT_TATP || kind == DINT_SMALLBANK) {
      for (uint32_t r = 0; r < G; r++)
        for (uint32_t t = 0; t < d.n_tables; t++) {
          const ReplicaKeep keep{make_fastmod(G), make_fastmod(G2), G2, r, j};
          if (kind == DINT_SMALLBANK) k_kv_move<8><<<e->sms * 8, 256, 0, s>>>(f.src[r]->ctx.tbl[t], d.tbl[t], keep);
          else k_kv_move<40><<<e->sms * 8, 256, 0, s>>>(f.src[r]->ctx.tbl[t], d.tbl[t], keep);
        }
    } else {
      for (uint32_t r = 0; r < G; r++)
        k_kv_move<40><<<e->sms * 8, 256, 0, s>>>(f.src[r]->ctx.tbl[0], d.tbl[0], KeepOwner{d.tbl[0].lock_mod, G2, j});
      if (d.ecache) {                                  // the eBPF tier: its sets move whole; its counters start at zero
        for (uint32_t r = 0; r < G; r++) a.src[r] = (uint64_t)f.src[r]->ctx.ecache;
        a.dst = d.ecache;
        k_reshard_sets<<<grid, kThreads, 0, s>>>(a);
      }
    }
  }, out);
}

// ---- rebuilding lost tatp / smallbank shards (rebuild.cuh has the placement arithmetic) ----------------------------
static std::string mask_names(uint32_t mask) {
  std::string s;
  for (uint32_t r = 0; r < 32; r++)
    if ((mask >> r) & 1u) s += (s.empty() ? "" : ", ") + std::to_string(r);
  return "{" + s + "}";
}

// DINT_EINVAL, with the reason, unless the shards of `lost` of a G-shard cluster of this kind and configuration can be
// rebuilt from the others
static const char kEbpfRows[] = "the eBPF cache tiers hold dirty and cache-only rows whose wire-visible versions depend on "
                                "each shard's own hit history";
static int rebuild_check(int kind, const dint_cfg& cfg, uint32_t G, uint32_t lost) {
  if (kind != DINT_TATP && kind != DINT_SMALLBANK)
    return set_err(DINT_EINVAL, "rebuild: lock_2pl, lock_fasst, store and log_server clusters keep no replicas");
  if (cfg.flags & (DINT_CFG_TATP_EBPF | DINT_CFG_SMALLBANK_EBPF))
    return set_errf(DINT_EINVAL, "rebuild: %s, so no peer's copy is that shard's state", kEbpfRows);
  if (G < 3) return set_err(DINT_EINVAL, "rebuild: a one-shard cluster has no replica to rebuild from");
  if (lost == 0 || (lost >> G) != 0) return set_errf(DINT_EINVAL, "rebuild: lost mask 0x%x is empty or names shards outside [0, %u)", lost, G);
  for (uint32_t p = 0; p < G; p++)
    if (rebuild_source(p, G, lost) < 0)
      return set_errf(DINT_EINVAL, "rebuild: losing shards %s leaves the keys k with k %% %u == %u without a replica",
                      mask_names(lost).c_str(), G, p);
  return DINT_OK;
}

struct RebuildFrom : DeriveFrom {
  uint32_t G = 0, lost = 0;
  RebuildFrom(const std::vector<dint_engine*>& eng, uint32_t G_, uint32_t lost_) : G(G_), lost(lost_) {
    src = eng;
    for (uint32_t r = 0; r < G; r++) if ((lost >> r) & 1u) src[r] = nullptr;
  }
  // the surviving shards that may hold keys of a lost shard of `dsts`: within two positions of it, either way round
  std::vector<dint_engine*> near(uint32_t dsts) const {
    std::vector<dint_engine*> out(G, nullptr);
    for (uint32_t s = 0; s < G; s++)
      for (uint32_t d = 0; d < G; d++) {
        const uint32_t a = (s + G - d) % G;
        if (((dsts >> d) & 1u) && (a <= 2 || a >= G - 2)) out[s] = src[s];
      }
    return out;
  }
  // rows: every surviving source's rows per (lost shard, table)
  int count() {
    return count_rows(*this, near(lost), [&](uint32_t s, const KvTable&) { return RebuildDests{make_fastmod(G), G, lost, s}; },
                      "rebuild row count");
  }
  RebuildKeep keep(uint32_t s, uint32_t d) const { return RebuildKeep{make_fastmod(G), G, lost, s, d}; }
};

// Lost shard j, filled from the surviving sources within two positions of it
static int rebuild_engine(const RebuildFrom& f, uint32_t j, int kind, const dint_cfg& c, int device, dint_engine** out) {
  const std::vector<dint_engine*> read = f.near(1u << j);
  return derive_engine(kind, c, device, j, f.rows[j], read, g_rebuild_times, [&](dint_engine* e) {
    for (uint32_t s = 0; s < f.G; s++) {
      if (!read[s]) continue;
      for (uint32_t t = 0; t < e->ctx.n_tables; t++) {
        if (kind == DINT_SMALLBANK) k_kv_move<8><<<e->sms * 8, 256, 0, e->stream>>>(read[s]->ctx.tbl[t], e->ctx.tbl[t], f.keep(s, j));
        else k_kv_move<40><<<e->sms * 8, 256, 0, e->stream>>>(read[s]->ctx.tbl[t], e->ctx.tbl[t], f.keep(s, j));
      }
    }
  }, out);
}

// dint_cluster_create; with image_dir dint_cluster_image_open: then shard r's engine is opened from its image; with
// `from` dint_cluster_reshard: then shard r's engine is filled from the source cluster's shards.  With image_dir and
// `rebuild` (dint_cluster_image_open_rebuild): the shards of *rebuild (known missing) and those whose image fails with
// DINT_EIO are rebuilt from the others once those are open; *rebuild is then set to every shard rebuilt.
static int cluster_make(int kind, const dint_cfg* cfg, int n_gpus, const int* devices, uint64_t max_batch, const char* image_dir,
                        const DeriveFrom* from, uint32_t* rebuild, dint_cluster** out) {
  if (!out || kind < 0 || kind >= DINT_NUM_KINDS || n_gpus < 1 || n_gpus > kMaxShards) return set_err(DINT_EINVAL, "bad kind / n_gpus");
  *out = nullptr;
  const bool by_dst = kind == DINT_TATP || kind == DINT_SMALLBANK;
  if (by_dst && n_gpus == 2) return set_err(DINT_EINVAL, "tatp / smallbank placement needs 1 or >= 3 shards (primary + 2 backups)");
  if (cfg && (cfg->flags & DINT_CFG_LOCK_HOLDER_KEYS) && kind != DINT_TATP) return set_err(DINT_EINVAL, "DINT_CFG_LOCK_HOLDER_KEYS is a tatp option");
  if (cfg && (cfg->flags & DINT_CFG_STORE_EBPF_MASK) && kind != DINT_STORE) return set_err(DINT_EINVAL, "DINT_CFG_STORE_EBPF_* is a store option");
  if (cfg && (cfg->flags & DINT_CFG_TATP_EBPF) && kind != DINT_TATP) return set_err(DINT_EINVAL, "DINT_CFG_TATP_EBPF is a tatp option");
  if (cfg && (cfg->flags & DINT_CFG_SMALLBANK_EBPF) && kind != DINT_SMALLBANK) return set_err(DINT_EINVAL, "DINT_CFG_SMALLBANK_EBPF is a smallbank option");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return set_err(DINT_ENODEV, "no CUDA device: dint_b200 has no CPU fallback"); }
  dint_cluster* cl = new dint_cluster();
  cl->kind = kind; cl->G = (uint32_t)n_gpus; cl->by_dst = by_dst;
  for (int r = 0; r < n_gpus; r++) {
    const int d = devices ? devices[r] : r % ndev;
    if (d < 0 || d >= ndev) { delete cl; return set_err(DINT_EINVAL, "bad device ordinal"); }
    cl->dev.push_back(d);
    for (int q = 0; q < r; q++) if (cl->dev[q] == d) cl->shared_device = true;
  }
  if (cl->shared_device)
    for (int r = 1; r < n_gpus; r++)
      if (cl->dev[r] != cl->dev[0]) { delete cl; return set_err(DINT_EINVAL, "devices must be all distinct or all the same"); }
  const uint32_t G = cl->G;
  if (max_batch == 0) max_batch = 1u << 18;
  cl->max_n = max_batch;
  {
    // slab capacity per (source, owner): hashing spreads records evenly (mean + 25 % + 8 sigma); a client-chosen
    // placement is pre-counted on the host by dint_cluster_submit, which cuts a round where a slab would overflow
    const double mean = (double)max_batch / G;
    uint64_t cap = (uint64_t)(mean * (by_dst ? 2.0 : 1.25) + 8.0 * sqrt(mean) + 64);
    if (G == 1) cap = max_batch;
    cl->cap = (uint32_t)((cap + kTile - 1) / kTile * kTile);
  }
  int rc = DINT_OK;
  dint_cfg& base = cl->base;
  if (cfg) base = *cfg; else dint_default_cfg(kind, &base);
  uint32_t failed = 0;                                  // rebuild: shards whose image failed with DINT_EIO
  for (uint32_t r = 0; r < G && rc == DINT_OK; r++) {
    const dint_cfg c = cluster_shard_cfg(cl, r);
    dint_engine* e = nullptr;
    if (rebuild && ((*rebuild >> r) & 1u)) { failed |= 1u << r; cl->eng.push_back(nullptr); continue; }   // known missing
    rc = image_dir ? image_open_impl(img_shard_path(image_dir, r).c_str(), cl->dev[r], &c, &e)
         : from    ? reshard_engine(*from, r, G, kind, c, cl->dev[r], &e)
                   : dint_create(kind, &c, cl->dev[r], &e);
    if (rc == DINT_EIO && rebuild) {                    // a short, unreadable or corrupt image: rebuilt below
      failed |= 1u << r;
      rc = DINT_OK;
    }
    if (rc == DINT_OK) cl->eng.push_back(e);
  }
  if (rc == DINT_OK && failed) {                        // the present shards are open: fill the failed ones from them
    rc = rebuild_check(kind, base, G, failed);
    if (rc) rc = set_errf(DINT_EIO, "image %s: shard image(s) %s failed and cannot be rebuilt: %s", image_dir,
                          mask_names(failed).c_str(), g_last_error.c_str());
    RebuildFrom f(cl->eng, G, failed);
    if (rc == DINT_OK) rc = f.count();
    for (uint32_t r = 0; r < G && rc == DINT_OK; r++)
      if ((failed >> r) & 1u) rc = rebuild_engine(f, r, kind, cluster_shard_cfg(cl, r), cl->dev[r], &cl->eng[r]);
    if (rc == DINT_OK) *rebuild = failed;
  }
  const uint32_t S = kClusterSets;
  const size_t region = cluster_region(cl);
  for (uint32_t r = 0; r < G && rc == DINT_OK; r++) {
    void* p = nullptr;
    if (cudaSetDevice(cl->dev[r]) != cudaSuccess || cudaMalloc(&p, 2 * S * region + 4096) != cudaSuccess) { rc = set_err(DINT_ENOMEM, "cluster buffers", cudaGetLastError()); break; }
    cudaMemset(p, 0, 2 * S * region + 4096);
    cl->bufs.push_back(p);
    for (uint32_t q = 0; q < G && rc == DINT_OK; q++) rc = peer_enable(cl->dev[r], cl->dev[q]);
  }
  if (rc == DINT_OK) cluster_quiesce(cl);
  if (rc == DINT_OK) rc = cluster_ranks(cl, cl->eng, cl->sh);
  if (rc != DINT_OK) { std::string keep = g_last_error; dint_cluster_destroy(cl); g_last_error = keep; return rc; }
  *out = cl;
  return DINT_OK;
}

extern "C" {

int dint_cluster_create(int kind, const dint_cfg* cfg, int n_gpus, const int* devices, uint64_t max_batch, dint_cluster** out) {
  return cluster_make(kind, cfg, n_gpus, devices, max_batch, nullptr, nullptr, nullptr, out);
}

int dint_cluster_image_save(dint_cluster* cl, const char* dir) {
  if (!cl || !dir) return set_err(DINT_EINVAL, "null argument");
  for (double& t : g_img_times) t = 0;
  const double t0 = img_now();
  if (mkdir(dir, 0755) != 0 && errno != EEXIST) return set_errf(DINT_EIO, "image directory %s: %s", dir, strerror(errno));
  // a manifest names shard images of one moment: an earlier one goes (durably) before the first shard is replaced, so a
  // save that stops part-way leaves a directory that opens as nothing rather than as shards of two moments
  const std::string manifest = img_manifest_path(dir);
  if (unlink(manifest.c_str()) != 0 && errno != ENOENT) return set_errf(DINT_EIO, "image %s: unlink: %s", manifest.c_str(), strerror(errno));
  { int rc = img_sync_dir(manifest.c_str()); if (rc) return rc; }
  int rc = DINT_OK;
  for (uint32_t r = 0; r < cl->G && rc == DINT_OK; r++) rc = image_save_impl(cl->eng[r], img_shard_path(dir, r).c_str());
  if (rc == DINT_OK) {                                  // the manifest last: a directory with one names complete shard images
    CluManifest m{};
    memcpy(m.magic, kCluMagic, 8);
    m.version = kImgVersion;
    m.kind = (uint32_t)cl->kind;
    m.shards = cl->G;
    m.cfg = cl->base;
    const std::string path = img_manifest_path(dir), tmp = path + ".tmp";
    ImgFd f;
    f.fd = open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
    if (f.fd < 0 || !img_write(f.fd, &m, sizeof m)) rc = set_errf(DINT_EIO, "image %s: %s", tmp.c_str(), strerror(errno));
    else rc = img_publish(tmp.c_str(), path.c_str(), f.fd);
  }
  g_img_times[0] = img_now() - t0;
  return rc;
}

}  // extern "C"

// dint_cluster_image_open; with `rebuilt` dint_cluster_image_open_rebuild
static int cluster_image_open(const char* dir, int n_gpus, const int* devices, uint64_t max_batch, uint32_t* rebuilt,
                              dint_cluster** out) {
  if (!dir || !out) return set_err(DINT_EINVAL, "null argument");
  *out = nullptr;
  if (rebuilt) *rebuilt = 0;
  for (double& t : g_img_times) t = 0;
  const double t0 = img_now();
  const std::string path = img_manifest_path(dir);
  CluManifest m;
  {
    ImgFd f;
    f.fd = open(path.c_str(), O_RDONLY);
    if (f.fd < 0) return set_errf(DINT_EIO, "image %s: %s", path.c_str(), strerror(errno));
    if (!img_read(f.fd, &m, sizeof m)) return set_errf(DINT_EIO, "image %s: truncated manifest", path.c_str());
  }
  if (memcmp(m.magic, kCluMagic, 8) != 0) return set_errf(DINT_EINVAL, "image %s: bad magic (not a dint_b200 cluster manifest)", path.c_str());
  if (m.version != kImgVersion) return set_errf(DINT_EINVAL, "image %s: format version %u, this build reads %u", path.c_str(), m.version, kImgVersion);
  if (m.kind >= DINT_NUM_KINDS || (m.cfg.flags & ~kCfgKnownFlags)) return set_errf(DINT_EINVAL, "image %s: unknown kind or option flags", path.c_str());
  if ((uint32_t)n_gpus != m.shards) return set_errf(DINT_EINVAL, "image %s: %u shards, not %d", path.c_str(), m.shards, n_gpus);
  uint32_t missing = 0;
  for (uint32_t r = 0; r < m.shards; r++) {
    struct stat st;
    if (stat(img_shard_path(dir, r).c_str(), &st) == 0) continue;
    if (!rebuilt) return set_errf(DINT_EIO, "image %s: %s", img_shard_path(dir, r).c_str(), strerror(errno));
    missing |= 1u << r;
  }
  if (missing && rebuild_check((int)m.kind, m.cfg, m.shards, missing))   // refused before any CUDA call
    return set_errf(DINT_EIO, "image %s: shard image(s) %s missing and cannot be rebuilt: %s", dir, mask_names(missing).c_str(),
                    g_last_error.c_str());
  if (rebuilt) { for (double& t : g_rebuild_times) t = 0; *rebuilt = missing; }
  const int rc = cluster_make((int)m.kind, &m.cfg, n_gpus, devices, max_batch, dir, nullptr, rebuilt, out);
  if (rc && rebuilt) *rebuilt = 0;
  g_img_times[0] = img_now() - t0;
  if (rebuilt) g_rebuild_times[0] = g_img_times[0];
  return rc;
}

extern "C" {

int dint_cluster_image_open(const char* dir, int n_gpus, const int* devices, uint64_t max_batch, dint_cluster** out) {
  return cluster_image_open(dir, n_gpus, devices, max_batch, nullptr, out);
}

int dint_cluster_image_open_rebuild(const char* dir, int n_gpus, const int* devices, uint64_t max_batch, uint32_t* rebuilt_mask,
                                    dint_cluster** out) {
  if (!rebuilt_mask) return set_err(DINT_EINVAL, "null argument");
  return cluster_image_open(dir, n_gpus, devices, max_batch, rebuilt_mask, out);
}

int dint_cluster_rebuild(dint_cluster* cl, uint32_t lost_mask) {
  if (!cl) return set_err(DINT_EINVAL, "null argument");
  { int rc = rebuild_check(cl->kind, cl->base, cl->G, lost_mask); if (rc) return rc; }
  if (cl->txn_clients)
    return set_errf(DINT_EINVAL, "rebuild: %u dint_txn_clients are attached; clients mid-transaction hold locks the rebuilt "
                                 "shards do not, so destroy them first", cl->txn_clients);
  for (double& t : g_rebuild_times) t = 0;
  const double t0 = img_now();
  { int rc = cluster_quiesce(cl); if (rc) return rc; }
  const uint32_t G = cl->G;
  RebuildFrom f(cl->eng, G, lost_mask);
  { int rc = f.count(); if (rc) return rc; }
  g_rebuild_times[2] += img_now() - t0;
  // the new engines and rank contexts are made next to the old ones, so a failure leaves the cluster as it was
  std::vector<dint_engine*> eng = cl->eng;
  std::vector<dint_shard_ctx*> sh;
  auto fail = [&](int code) {
    std::string keep = g_last_error;
    for (auto* c : sh) dint_shard_destroy(c);
    for (uint32_t r = 0; r < G; r++) {
      if (eng[r] != cl->eng[r]) dint_destroy(eng[r]);
      cl->eng[r]->plain_launches = true;               // (dint_shard_destroy cleared it; the old contexts stay)
    }
    g_last_error = keep;
    return code;
  };
  for (uint32_t r = 0; r < G; r++)
    if ((lost_mask >> r) & 1u) {
      eng[r] = nullptr;
      int rc = rebuild_engine(f, r, cl->kind, cluster_shard_cfg(cl, r), cl->dev[r], &eng[r]);
      if (rc) { if (!eng[r]) eng[r] = cl->eng[r]; return fail(rc); }
    }
  { int rc = cluster_ranks(cl, eng, sh); if (rc) return fail(rc); }
  // commit: every rank's epoch restarts at 0 over zeroed signal blocks
  for (auto* c : cl->sh) dint_shard_destroy(c);
  for (uint32_t r = 0; r < G; r++) {
    CU(cudaSetDevice(cl->dev[r]));
    CU(cudaMemset((void*)cluster_sig_block(cl, r), 0, 4096));
  }
  for (uint32_t r = 0; r < G; r++) {
    if (eng[r] != cl->eng[r]) dint_destroy(cl->eng[r]);
    eng[r]->plain_launches = true;
  }
  cl->eng = eng;
  cl->sh = sh;
  { int rc = cluster_quiesce(cl); if (rc) return rc; }
  g_rebuild_times[0] = img_now() - t0;
  return DINT_OK;
}

int dint_rebuild_times(double out[3]) {
  if (!out) return set_err(DINT_EINVAL, "null argument");
  for (int i = 0; i < 3; i++) out[i] = g_rebuild_times[i];
  return DINT_OK;
}

int dint_cluster_reshard(dint_cluster* src, int n_gpus, const int* devices, uint64_t max_batch, dint_cluster** out) {
  if (!src || !out) return set_err(DINT_EINVAL, "null argument");
  *out = nullptr;
  if (src->kind == DINT_TATP || src->kind == DINT_SMALLBANK)
    return set_err(DINT_EINVAL, "tatp / smallbank: the shard count is the clients' replica placement (primary key % G, backups "
                                "+1 and +2); another count moves which shard is primary for a key, so there is no one-server "
                                "state to move");
  if (src->kind == DINT_LOG) return set_err(DINT_EINVAL, "log_server: a record belongs to the rank that received it, no key decides ownership");
  if (n_gpus < 1 || n_gpus > kMaxShards) return set_err(DINT_EINVAL, "bad n_gpus");
  for (double& t : g_reshard_times) t = 0;
  const double t0 = img_now();
  { int rc = cluster_quiesce(src); if (rc) return rc; }   // as dint_snapshot_create quiesces an engine
  DeriveFrom f;
  f.src = src->eng;
  const uint32_t G2 = (uint32_t)n_gpus;
  { int rc = count_rows(f, f.src, [&](uint32_t, const KvTable& t) { return OwnerDests{t.lock_mod, G2, (1u << G2) - 1}; }, "re-shard key count"); if (rc) return rc; }
  g_reshard_times[2] += img_now() - t0;
  const int rc = cluster_make(src->kind, &src->base, n_gpus, devices, max_batch, nullptr, &f, nullptr, out);
  g_reshard_times[0] = img_now() - t0;
  return rc;
}

int dint_cluster_reshard_txn(dint_cluster* src, int n_gpus, const int* devices, uint64_t max_batch, dint_cluster** out) {
  if (!src || !out) return set_err(DINT_EINVAL, "null argument");
  *out = nullptr;
  if (src->kind != DINT_TATP && src->kind != DINT_SMALLBANK)
    return set_err(DINT_EINVAL, "re-shard: dint_cluster_reshard_txn re-places tatp and smallbank replicas; lock_2pl, lock_fasst "
                                "and store clusters re-shard with dint_cluster_reshard, and a log_server record has no key");
  if (src->base.flags & (DINT_CFG_TATP_EBPF | DINT_CFG_SMALLBANK_EBPF))
    return set_errf(DINT_EINVAL, "re-shard: %s, so no one shard's table holds a key's row", kEbpfRows);
  if (n_gpus < 1 || n_gpus == 2 || n_gpus > (int)kMaxShards)
    return set_errf(DINT_EINVAL, "re-shard: %d shards; tatp / smallbank placement needs 1 or 3..8 (primary + 2 backups)", n_gpus);
  for (double& t : g_reshard_times) t = 0;
  const double t0 = img_now();
  { int rc = cluster_quiesce(src); if (rc) return rc; }
  const uint32_t G = src->G, G2 = (uint32_t)n_gpus;
  // a held lock means a client is mid-transaction: its rows may differ between replicas, and the lock would be lost
  for (uint32_t r = 0; r < G; r++) {
    const dint_engine* e = src->eng[r];
    CU(cudaSetDevice(e->device));
    unsigned long long* d = nullptr;
    unsigned long long held = 0;
    CU(cudaMalloc(&d, sizeof held));
    cudaError_t ce = cudaMemset(d, 0, sizeof held);
    if (ce == cudaSuccess) {
      k_locks_held<<<e->sms * 4, kThreads>>>(src->kind == DINT_TATP ? e->ctx.lockbits : nullptr,
                                             src->kind == DINT_SMALLBANK ? e->ctx.cnt2 : nullptr, e->total_groups, d);
      ce = cudaGetLastError();
    }
    if (ce == cudaSuccess) ce = cudaMemcpy(&held, d, sizeof held, cudaMemcpyDeviceToHost);
    cudaFree(d);
    if (ce != cudaSuccess) return set_err(DINT_EIO, "re-shard lock count", ce);
    if (held)
      return set_errf(DINT_EINVAL, "re-shard: shard %u holds %llu locks: clients are mid-transaction, drain them first "
                                   "(dint_txn_clients_drain)", r, held);
  }
  DeriveFrom f;
  f.src = src->eng;
  { int rc = count_rows(f, f.src, [&](uint32_t s, const KvTable&) { return ReplicaDests{make_fastmod(G), make_fastmod(G2), G2, (1u << G2) - 1, s}; },
                        "re-shard row count"); if (rc) return rc; }
  g_reshard_times[2] += img_now() - t0;
  const int rc = cluster_make(src->kind, &src->base, n_gpus, devices, max_batch, nullptr, &f, nullptr, out);
  g_reshard_times[0] = img_now() - t0;
  return rc;
}

int dint_reshard_times(double out[3]) {
  if (!out) return set_err(DINT_EINVAL, "null argument");
  for (int i = 0; i < 3; i++) out[i] = g_reshard_times[i];
  return DINT_OK;
}

int dint_cluster_populate(dint_cluster* cl) {
  if (!cl) return DINT_EINVAL;
  for (auto* e : cl->eng) { int rc = dint_populate(e); if (rc) return rc; }
  return DINT_OK;
}
dint_engine* dint_cluster_engine(dint_cluster* cl, int shard) { return (cl && shard >= 0 && shard < (int)cl->G) ? cl->eng[shard] : nullptr; }
uint32_t dint_cluster_size(dint_cluster* cl) { return cl ? cl->G : 0; }

// rounds over [from, to): a round hands rank r the r-th of G contiguous pieces of at most `lim` records (rank-major
// order = index order, SURVEY.md 8(e)); for a client-chosen placement the pieces are cut so that no slab can overflow.
// Returns the first record index that was NOT served (to = everything served), or a negative error.
static int64_t cluster_run(dint_cluster* cl, const uint8_t* rq, const uint8_t* dst_shard, uint8_t* rs, uint64_t from, uint64_t to, uint64_t lim) {
  const uint32_t G = cl->G, msg = kMsgSize[cl->kind];
  std::vector<std::vector<HostBatch>> hb(G);
  std::vector<uint64_t> round_off;
  uint64_t off = from;
  while (off < to) {
    uint64_t m = to - off < (uint64_t)G * lim ? to - off : (uint64_t)G * lim;
    for (;;) {
      const uint64_t q = (m + G - 1) / G;
      bool fits = true;
      if (dst_shard && G > 1) {
        for (uint32_t r = 0; r < G && fits; r++) {
          const uint64_t lo = off + (uint64_t)r * q, hi = lo + q < off + m ? lo + q : off + m;
          uint32_t cnt[kMaxShards] = {0};
          for (uint64_t i = lo; i < hi; i++) { const uint8_t o = dst_shard[i]; if (o < G) cnt[o]++; }
          for (uint32_t o = 0; o < G; o++) if (cnt[o] > cl->cap) fits = false;
        }
      }
      if (fits || m <= G) break;
      m = (m + 1) / 2;
    }
    const uint64_t q = (m + G - 1) / G;
    round_off.push_back(off);
    for (uint32_t r = 0; r < G; r++) {
      const uint64_t lo = off + (uint64_t)r * q;
      const uint64_t hi = lo + q < off + m ? lo + q : off + m;
      // (a rank without records in a tail round still takes part in the exchange: its slabs are all padding)
      hb[r].push_back(HostBatch{rq + lo * msg, dst_shard ? dst_shard + lo : nullptr, rs + lo * msg, lo < hi ? hi - lo : 0});
    }
    off += m;
  }
  const uint32_t k = (uint32_t)round_off.size();
  int rc = shard_run_host(cl->sh.data(), G, k, hb);
  if (rc) return rc;
  uint32_t first_unserved = 0xffffffffu;
  for (uint32_t r = 0; r < G; r++) {
    uint32_t fl[2] = {0, 0}, fu = 0xffffffffu;
    if ((rc = dint_shard_flags(cl->sh[r], fl))) return rc;
    if (fl[1]) return set_err(DINT_EIO, "exchange timed out");
    if ((rc = dint_shard_recover(cl->sh[r], k, &fu))) return rc;
    if (fu < first_unserved) first_unserved = fu;
  }
  return first_unserved == 0xffffffffu ? (int64_t)to : (int64_t)round_off[first_unserved];
}

int dint_cluster_submit(dint_cluster* cl, const void* req, uint64_t n, const uint8_t* dst_shard, void* resp) {
  if (!cl || (n && (!req || !resp))) return set_err(DINT_EINVAL, "null argument");
  if (cl->by_dst && cl->G > 1 && !dst_shard) return set_err(DINT_EINVAL, "tatp / smallbank: the client names the shard of every record (dst_shard)");
  if (n == 0) return DINT_OK;
  unsigned long long err_before = 0;
  for (auto* e : cl->eng) err_before += e->stats.errors;
  // Normal rounds; if a slab overflowed (keys skewed beyond the slack of the slabs) every shard stopped serving AT that
  // round, nothing behind it touched the state: serve the rest in rounds of at most `cap` records per rank, which fit
  // any slab whatever the keys are.
  int64_t done = cluster_run(cl, (const uint8_t*)req, dst_shard, (uint8_t*)resp, 0, n, cl->max_n);
  if (done < 0) return (int)done;
  if ((uint64_t)done < n) {
    cl->overflow_retries++;
    done = cluster_run(cl, (const uint8_t*)req, dst_shard, (uint8_t*)resp, (uint64_t)done, n, cl->cap < cl->max_n ? cl->cap : cl->max_n);
    if (done < 0) return (int)done;
    if ((uint64_t)done < n) return set_err(DINT_EIO, "internal: a round of at most cap records per rank overflowed");
  }
  unsigned long long err_after = 0;
  for (uint32_t r = 0; r < cl->G; r++) {
    dint_engine* e = cl->eng[r];
    int rc = pull_counters(e);
    if (rc) return rc;
    err_after += e->stats.errors;
  }
  return err_after != err_before ? DINT_EPROTO : DINT_OK;
}
uint64_t dint_cluster_overflow_retries(dint_cluster* cl) { return cl ? cl->overflow_retries : 0; }

}  // extern "C"

// ---- lock_2pl / lock_fasst / log_server / store closed-loop clients on the GPU (clients.cuh) ------------------
// One block of clients on one device: their state, the requests of the pending round and the replies they absorb next.
// dint_clients holds one next to its engine; dint_cluster_clients holds one per cluster rank.
struct ClientBlock {
  ClientCtx cc{};
  uint8_t *req = nullptr, *resp = nullptr;
  double* cdf = nullptr;
};

static void client_block_free(ClientBlock& b) {
  cudaFree(b.req); cudaFree(b.resp); cudaFree(b.cdf);
  cudaFree(b.cc.hdr); cudaFree(b.cc.rng); cudaFree(b.cc.lcg); cudaFree(b.cc.rk); cudaFree(b.cc.rv); cudaFree(b.cc.stats);
  b = ClientBlock{};
}

// The argument checks of every lock / store / log client handle, then the state of clients [id0, id0 + n) of the family
// `cfg` on `device` (n may be 0: a cluster rank without clients).  On an error nothing stays allocated.
static int client_block_make(int kind, const dint_clients_cfg* cfg, int device, uint32_t id0, uint32_t n, ClientBlock* out) {
  const bool lock = kind == DINT_LOCK2PL || kind == DINT_FASST;
  if (kind == DINT_TATP || kind == DINT_SMALLBANK)
    return set_err(DINT_EINVAL, "tatp / smallbank: their clients are dint_txn_clients_*");
  if (cfg->n_clients == 0) return set_err(DINT_EINVAL, "n_clients must be > 0");
  if ((lock || (kind == DINT_STORE && cfg->store_hot)) && cfg->n_keys == 0)
    return set_err(DINT_EINVAL, "n_keys must be > 0 for lock clients and HOT store clients");
  if (cfg->read_pct > 100) return set_err(DINT_EINVAL, "read_pct must be <= 100");
  if (cfg->set_pct > 100) return set_err(DINT_EINVAL, "set_pct must be <= 100");
  if (kind == DINT_STORE && !cfg->store_hot && cfg->store_subscribers == 0)
    return set_err(DINT_EINVAL, "store_subscribers must be > 0 for REF store clients");
  CU(cudaSetDevice(device));
  ClientBlock b;
  ClientCtx& cc = b.cc;
  const uint32_t msg = kMsgSize[kind];
  cc.n_clients = n; cc.id0 = id0; cc.n_keys = cfg->n_keys; cc.read_pct = cfg->read_pct;
  cc.set_pct = cfg->set_pct; cc.subscribers = cfg->store_subscribers; cc.store_hot = kind == DINT_STORE && cfg->store_hot ? 1u : 0u;
  const size_t na = n ? n : 1;                          // an empty block still gets valid pointers
  const bool ref_store = kind == DINT_STORE && !cc.store_hot;
  bool ok = cudaMalloc(&b.req, na * msg + 16) == cudaSuccess && cudaMalloc(&b.resp, na * msg + 16) == cudaSuccess &&
            cudaMalloc(&cc.stats, 8 * sizeof(unsigned long long)) == cudaSuccess;
  if (ok && !ref_store) ok = cudaMalloc(&cc.rng, na * 8) == cudaSuccess;
  if (ok && ref_store) ok = cudaMalloc(&cc.lcg, na * 8) == cudaSuccess;
  if (ok && lock) ok = cudaMalloc(&cc.hdr, na * 8) == cudaSuccess && cudaMalloc(&cc.rk, na * 40) == cudaSuccess;
  if (ok && kind == DINT_FASST) ok = cudaMalloc(&cc.rv, na * 40) == cudaSuccess && cudaMemset(cc.rv, 0, na * 40) == cudaSuccess;
  if (ok) ok = cudaMemset(cc.stats, 0, 8 * sizeof(unsigned long long)) == cudaSuccess;
  if (!ok) {
    cudaError_t ce = cudaGetLastError();
    client_block_free(b);
    return set_err(DINT_ENOMEM, "client state", ce);
  }
  if (cfg->zipf_theta > 0 && (lock || cc.store_hot)) {  // workloads.cc Zipf::init
    const uint32_t n_keys = cfg->n_keys;
    std::vector<double> cdf(n_keys);
    double acc = 0;
    for (uint32_t k = 0; k < n_keys; k++) { acc += 1.0 / std::pow((double)(k + 1), cfg->zipf_theta); cdf[k] = acc; }
    for (auto& v : cdf) v /= acc;
    if (cudaMalloc(&b.cdf, (size_t)n_keys * sizeof(double)) != cudaSuccess ||
        cudaMemcpy(b.cdf, cdf.data(), (size_t)n_keys * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess) {
      cudaError_t ce = cudaGetLastError();
      client_block_free(b);
      return set_err(DINT_ENOMEM, "Zipf table", ce);
    }
    cc.cdf = b.cdf;
    cc.zipf_n = n_keys;
  }
  *out = b;
  return DINT_OK;
}

// one kernel of a block of clients on s: first = every client starts and emits its first request; otherwise absorb the
// replies in resp and emit the next round's requests
static void clients_launch(int kind, uint64_t seed, const ClientBlock& b, bool first, cudaStream_t s) {
  const uint32_t blocks = (b.cc.n_clients + 255) / 256;
  if (!blocks) return;
  switch (kind) {
    case DINT_FASST:
      if (first) k_clients_init<K_FASST><<<blocks, 256, 0, s>>>(b.cc, seed, b.req);
      else k_clients_step<K_FASST><<<blocks, 256, 0, s>>>(b.cc, b.resp, b.req);
      break;
    case DINT_LOCK2PL:
      if (first) k_clients_init<K_LOCK2PL><<<blocks, 256, 0, s>>>(b.cc, seed, b.req);
      else k_clients_step<K_LOCK2PL><<<blocks, 256, 0, s>>>(b.cc, b.resp, b.req);
      break;
    case DINT_LOG: k_log_clients<<<blocks, 256, 0, s>>>(b.cc, seed, first ? 1u : 0u, b.req); break;
    default: k_store_clients<<<blocks, 256, 0, s>>>(b.cc, seed, first ? 1u : 0u, b.resp, b.req); break;
  }
}

extern "C" {
struct dint_clients {
  dint_engine* e = nullptr;
  int kind = 0;
  uint32_t msg = 0;
  ClientBlock b;
  uint64_t seed = 0;
  bool started = false;
};

void dint_clients_destroy(dint_clients* c) {
  if (!c) return;
  cudaSetDevice(c->e->device);
  cudaDeviceSynchronize();
  client_block_free(c->b);
  delete c;
}

int dint_clients_create_cfg(dint_engine* e, const dint_clients_cfg* cfg, dint_clients** out) {
  if (!e || !cfg || !out) return set_err(DINT_EINVAL, "null argument");
  ClientBlock b;
  int rc = client_block_make(e->kind, cfg, e->device, 0, cfg->n_clients, &b);
  if (rc) return rc;
  dint_clients* c = new dint_clients();
  c->e = e;
  c->kind = e->kind;
  c->msg = kMsgSize[e->kind];
  c->seed = cfg->seed;
  c->b = b;
  *out = c;
  return DINT_OK;
}

int dint_clients_create(dint_engine* e, uint32_t n_clients, uint64_t seed, uint32_t n_keys, double zipf_theta, uint32_t read_pct,
                        dint_clients** out) {
  if (!e || !out || e->kind != DINT_FASST || n_clients == 0 || n_keys == 0) return set_err(DINT_EINVAL, "lock_fasst engine, n_clients > 0, n_keys > 0");
  dint_clients_cfg cfg{};
  cfg.n_clients = n_clients; cfg.n_keys = n_keys; cfg.seed = seed; cfg.zipf_theta = zipf_theta;
  cfg.read_pct = read_pct < 100 ? read_pct : 100;        // every read_pct >= 100 means "no key is written"
  return dint_clients_create_cfg(e, &cfg, out);
}

// `rounds` closed-loop rounds, asynchronous on cuda_stream: every round = the engine on the clients' request buffer
// (dint_submit_device) + ONE kernel that absorbs the replies and emits the next round's requests
int dint_clients_run(dint_clients* c, uint32_t rounds, void* cuda_stream) {
  if (!c) return set_err(DINT_EINVAL, "null argument");
  dint_engine* e = c->e;
  CU(cudaSetDevice(e->device));
  cudaStream_t s = (cudaStream_t)cuda_stream;
  if (!c->started) {
    clients_launch(c->kind, c->seed, c->b, true, s);
    c->started = true;
    e->stats.kernel_launches++;
  }
  for (uint32_t r = 0; r < rounds; r++) {
    int rc = run_device(e, c->b.req, c->b.cc.n_clients, c->b.resp, s);
    if (rc) return rc;
    clients_launch(c->kind, c->seed, c->b, false, s);
    e->stats.kernel_launches++;
  }
  CU(cudaGetLastError());
  return DINT_OK;
}

// out: requests served, committed transactions, validation aborts, lock rejects, rounds (synchronises)
int dint_clients_stats(dint_clients* c, uint64_t out[5]) {
  if (!c || !out) return set_err(DINT_EINVAL, "null argument");
  CU(cudaSetDevice(c->e->device));
  CU(cudaDeviceSynchronize());
  unsigned long long h[5];
  CU(cudaMemcpy(h, c->b.cc.stats, sizeof h, cudaMemcpyDeviceToHost));
  for (int i = 0; i < 5; i++) out[i] = h[i];
  return DINT_OK;
}

// out: requests served, committed transactions, validation aborts, lock rejects, not-exist replies, rounds (the order of
// dint_wl_stats; synchronises)
int dint_clients_stats_all(dint_clients* c, uint64_t out[6]) {
  if (!c || !out) return set_err(DINT_EINVAL, "null argument");
  CU(cudaSetDevice(c->e->device));
  CU(cudaDeviceSynchronize());
  unsigned long long h[6];
  CU(cudaMemcpy(h, c->b.cc.stats, sizeof h, cudaMemcpyDeviceToHost));
  out[0] = h[0]; out[1] = h[1]; out[2] = h[2]; out[3] = h[3]; out[4] = h[5]; out[5] = h[4];
  return DINT_OK;
}

// test hook: the requests the clients will send next and the replies they absorbed last (host buffers of
// n_clients * dint_msg_size(kind) bytes)
int dint_clients_peek(dint_clients* c, void* next_req_host, void* last_resp_host) {
  if (!c) return set_err(DINT_EINVAL, "null argument");
  CU(cudaSetDevice(c->e->device));
  CU(cudaDeviceSynchronize());
  if (!c->started) {
    clients_launch(c->kind, c->seed, c->b, true, 0);
    c->started = true;
    CU(cudaDeviceSynchronize());
  }
  const size_t bytes = (size_t)c->b.cc.n_clients * c->msg;
  if (next_req_host) CU(cudaMemcpy(next_req_host, c->b.req, bytes, cudaMemcpyDeviceToHost));
  if (last_resp_host) CU(cudaMemcpy(last_resp_host, c->b.resp, bytes, cudaMemcpyDeviceToHost));
  return DINT_OK;
}

}  // extern "C"

// ---- closed-loop clients on the GPU against a shard cluster: the round loop of dint_txn_clients_* and ---------------
// ---- dint_cluster_clients_* ------------------------------------------------------------------------------------------
// The clients are split over the cluster's ranks in contiguous blocks, rank r's block on rank r's device, so rank-major
// order is global client order.  A round: every rank's kernels leave the round in its req[] (and, for client-chosen
// placements, dst[]) and its size and per-shard counts in a mapped pinned block; ONE event synchronise per rank hands
// those G x (G + 1) words to the host, which sizes the exchange slabs exactly from them and serves the round with one
// shard_run on device buffers; the clients' next emission absorbs the replies straight from out[].  No record crosses
// PCIe.  Serving K rounds without a host round trip is not done: a closed-loop round needs the previous round's replies,
// and exact slabs need the counts on the host.
struct RoundRank {
  const uint8_t* req = nullptr;  // the pending round, contiguous (device)
  const uint8_t* dst = nullptr;  // its records' owner shards, or null: computed on the device (route_owner_of)
  uint8_t* out = nullptr;        // replies of the round, in the order of req[]
  uint32_t* pub = nullptr;       // host view of the pinned block: [0] records, [1 + o] records for shard o, [9..10] exchange flags
  cudaEvent_t ev = nullptr;      // this rank's emission of the pending round is done
  uint64_t last_n = 0;           // records of the last round served
};
struct RoundLoop {
  dint_cluster* cl = nullptr;
  uint32_t msg = 0;
  bool local = false;            // every rank serves its own batch on its own engine, without the exchange (log_server)
  std::vector<cudaStream_t> mains;
  bool started = false;
  uint64_t requests = 0, rounds = 0, fallback_rounds = 0;
  cudaEvent_t t_beg = nullptr, t_end = nullptr;   // on rank 0's stream: the device work of one round
  uint64_t timed = 0;
  double wall_s = 0, dev_s = 0;
};

// records of one fallback piece: at most min(cap, max_n), a multiple of 16 so that every device batch stays 16-byte aligned
static uint32_t fallback_piece(const dint_cluster* cl) { return (uint32_t)((cl->cap < cl->max_n ? cl->cap : cl->max_n) & ~15ull); }

// wait for every rank's pending emission; the exchange flags of the round before it must read zero
template <class Rank>
static int round_wait(RoundLoop& L, std::vector<Rank>& rk) {
  for (uint32_t r = 0; r < L.cl->G; r++) {
    CU(cudaSetDevice(L.cl->dev[r]));
    CU(cudaEventSynchronize(rk[r].ev));
  }
  for (uint32_t r = 0; r < L.cl->G; r++)
    if (rk[r].pub[9] || rk[r].pub[10]) return set_err(DINT_EIO, "internal: an exchange slab overflowed or a wait timed out");
  return DINT_OK;
}
static int round_errors(dint_cluster* cl, unsigned long long* sum) {
  *sum = 0;
  for (auto* e : cl->eng) {
    CU(cudaSetDevice(e->device));
    int rc = pull_counters(e);
    if (rc) return rc;
    *sum += e->stats.errors;
  }
  return DINT_OK;
}

// `rounds` rounds, blocking.  emit(first) enqueues one emission on every rank and records each rank's event.
template <class Rank, class Emit>
static int serve_rounds(RoundLoop& L, std::vector<Rank>& rk, uint32_t rounds, Emit&& emit) {
  dint_cluster* cl = L.cl;
  const uint32_t G = cl->G, msg = L.msg;
  unsigned long long err_before = 0, err_after = 0;
  int rc = round_errors(cl, &err_before);
  if (rc) return rc;
  if (!L.started && (rc = emit(1))) return rc;
  if ((rc = round_wait(L, rk))) return rc;
  const uint32_t piece = fallback_piece(cl);
  auto round_up = [](uint64_t x) { return (uint32_t)(x ? (x + kTile - 1) / kTile * kTile : kTile); };
  std::vector<uint64_t> n(G);
  std::vector<std::vector<ShardBatch>> b;
  auto t_prev = std::chrono::steady_clock::now();
  for (uint32_t i = 0; i < rounds; i++) {
    // the slab capacity of the round: the largest (source, owner) count, so no slab can overflow
    uint64_t maxc = 0, total = 0;
    bool fits = true;
    for (uint32_t r = 0; r < G; r++) {
      n[r] = rk[r].pub[0];
      total += n[r];
      if (n[r] > cl->max_n) fits = false;
      for (uint32_t o = 0; o < G; o++) maxc = rk[r].pub[1 + o] > maxc ? rk[r].pub[1 + o] : maxc;
    }
    if (total == 0) break;                      // the end of a drain (dint_txn_clients_drain): not served, not counted
    if (maxc > cl->cap) fits = false;
    b.assign(G, {});
    if (L.local) {
      // (served below, without the exchange)
    } else if (fits) {
      for (uint32_t r = 0; r < G; r++) b[r].push_back(ShardBatch{rk[r].req, rk[r].dst, rk[r].out, n[r], round_up(maxc)});
    } else {
      // one source rank at a time sends pieces of at most min(cap, max_n) records, the others send empty batches:
      // every shard still sees rank-major order, and a piece this small cannot overflow a slab
      L.fallback_rounds++;
      for (uint32_t src = 0; src < G; src++)
        for (uint64_t from = 0; from < n[src]; from += piece) {
          const uint64_t len = n[src] - from < piece ? n[src] - from : piece;
          for (uint32_t r = 0; r < G; r++) {
            const Rank& k = rk[r];
            b[r].push_back(r == src ? ShardBatch{k.req + from * msg, k.dst ? k.dst + from : nullptr, k.out + from * msg, len, round_up(len)}
                                    : ShardBatch{k.req, k.dst, k.out, 0, round_up(len)});
          }
        }
    }
    CU(cudaSetDevice(cl->dev[0]));
    CU(cudaEventRecord(L.t_beg, L.mains[0]));
    if (L.local) {
      // log_server: a log record touches no keyed state, so its owner is the rank that received it (route_owner_of);
      // serving each rank's batch on its own engine gives every shard the order the exchange would, without making
      // each owner scan G - 1 slabs of padding
      for (uint32_t r = 0; r < G; r++)
        if (n[r]) {
          CU(cudaSetDevice(cl->dev[r]));
          if ((rc = run_device(cl->eng[r], rk[r].req, n[r], rk[r].out, L.mains[r]))) return rc;
        }
    } else {
      const uint32_t k = (uint32_t)b[0].size();
      if (k && (rc = shard_run(cl->sh.data(), G, k, b, L.mains.data()))) return rc;
      for (uint32_t r = 0; r < G; r++) {          // the exchange flags of this round (dint_shard_flags, without its synchronise)
        CU(cudaSetDevice(cl->dev[r]));
        CU(cudaMemcpyAsync(rk[r].pub + 9, cl->sh[r]->flags, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, L.mains[r]));
        CU(cudaMemsetAsync(cl->sh[r]->flags, 0, 2 * sizeof(uint32_t), L.mains[r]));
      }
    }
    for (uint32_t r = 0; r < G; r++) { rk[r].last_n = n[r]; L.requests += n[r]; }
    L.rounds++;
    if ((rc = emit(0))) return rc;
    CU(cudaSetDevice(cl->dev[0]));
    CU(cudaEventRecord(L.t_end, L.mains[0]));
    if ((rc = round_wait(L, rk))) return rc;
    CU(cudaSetDevice(cl->dev[0]));
    CU(cudaEventSynchronize(L.t_end));
    float ms = 0;
    CU(cudaEventElapsedTime(&ms, L.t_beg, L.t_end));
    const auto now = std::chrono::steady_clock::now();
    L.wall_s += std::chrono::duration<double>(now - t_prev).count();
    L.dev_s += ms * 1e-3;
    L.timed++;
    t_prev = now;
  }
  if ((rc = round_errors(cl, &err_after))) return rc;
  return err_after != err_before ? set_err(DINT_EPROTO, "an engine answered a request with an error reply") : DINT_OK;
}

extern "C" {
// ---- TATP / SmallBank closed-loop clients on the GPU against a shard cluster (txn_clients.cuh) ---------------
// Every shard sees its records in the order one host TxnWorkload would send them.  A round's emission is three kernels
// per rank: step / scan / compact leave the round in req[] / dst[] and its size and per-shard counts in pub.
struct TxnRank : RoundRank {
  txn::DevClients d{};
  uint32_t tiles = 0;
};
struct dint_txn_clients : RoundLoop {
  uint32_t n = 0;
  bool drained = false;          // the pending round is empty after a drain: the next run / peek / stats resumes
  std::vector<TxnRank> rk;
};

void dint_txn_clients_destroy(dint_txn_clients* t) {
  if (!t) return;
  for (size_t r = 0; r < t->rk.size(); r++) {
    TxnRank& k = t->rk[r];
    cudaSetDevice(t->cl->dev[r]);
    cudaDeviceSynchronize();
    cudaFree(k.d.cl); cudaFree(k.d.stg); cudaFree(k.d.stg_dst); cudaFree(k.d.cnt); cudaFree(k.d.off); cudaFree(k.d.tile_sum);
    cudaFree(k.d.owner_cnt); cudaFree(k.d.stats); cudaFree(k.d.req); cudaFree(k.d.dst); cudaFree(k.out);
    if (k.pub) cudaFreeHost(k.pub);
    if (k.ev) cudaEventDestroy(k.ev);
  }
  if (!t->rk.empty()) cudaSetDevice(t->cl->dev[0]);
  if (t->t_beg) cudaEventDestroy(t->t_beg);
  if (t->t_end) cudaEventDestroy(t->t_end);
  t->cl->txn_clients--;
  delete t;
}

int dint_txn_clients_create(dint_cluster* cl, uint32_t n_clients, uint32_t gid0, uint32_t subscribers, dint_txn_clients** out) {
  if (!cl || !out) return set_err(DINT_EINVAL, "null argument");
  *out = nullptr;
  if ((cl->kind != DINT_TATP && cl->kind != DINT_SMALLBANK) || n_clients == 0 || subscribers < 3)
    return set_err(DINT_EINVAL, "a tatp or smallbank cluster, n_clients > 0, subscribers >= 3");
  if (fallback_piece(cl) == 0) return set_err(DINT_EINVAL, "the cluster's max_batch must be >= 16");
  const uint32_t G = cl->G, msg = kMsgSize[cl->kind];
  dint_txn_clients* t = new dint_txn_clients();
  t->cl = cl; t->msg = msg; t->n = n_clients;
  cl->txn_clients++;                                   // (dint_txn_clients_destroy counts it down, also on failure below)
  txn::Cfg w{G, subscribers, 0};
  if (cl->kind == DINT_SMALLBANK) {
    w.hot = (uint32_t)((uint64_t)subscribers * 960000 / 24000000);   // kHotAccountNum / kAccountNum, as txn_workloads.cc
    if (w.hot < 2) w.hot = 2;
  }
  const size_t csz = cl->kind == DINT_TATP ? sizeof(txn::TatpClient) : sizeof(txn::SbClient);
  auto fail = [&](int code, const char* what, cudaError_t ce) { std::string keep; set_err(code, what, ce); keep = g_last_error;
                                                               dint_txn_clients_destroy(t); g_last_error = keep; return code; };
  t->rk.resize(G);
  for (uint32_t r = 0; r < G; r++) {
    TxnRank& k = t->rk[r];
    const uint32_t lo = (uint32_t)((uint64_t)n_clients * r / G), hi = (uint32_t)((uint64_t)n_clients * (r + 1) / G);
    const size_t n = hi - lo;
    k.d.n = (uint32_t)n; k.d.gid0 = (uint64_t)gid0 + lo; k.d.w = w;
    k.tiles = (uint32_t)((n + kThreads - 1) / kThreads);
    t->mains.push_back(cl->shared_device ? cl->eng[0]->stream : cl->eng[r]->stream);
    cudaError_t ce = cudaSetDevice(cl->dev[r]);
    const size_t rec = n * txn::kMaxRecords;
    if (ce == cudaSuccess) ce = cudaMalloc(&k.d.cl, n * csz + 16);
    if (ce == cudaSuccess) ce = cudaMalloc(&k.d.stg, rec * msg + 16);
    if (ce == cudaSuccess) ce = cudaMalloc(&k.d.stg_dst, rec + 16);
    if (ce == cudaSuccess) ce = cudaMalloc(&k.d.cnt, n * 4 + 16);
    if (ce == cudaSuccess) ce = cudaMalloc(&k.d.off, n * 4 + 16);
    if (ce == cudaSuccess) ce = cudaMalloc(&k.d.tile_sum, (size_t)k.tiles * 4 + 16);
    if (ce == cudaSuccess) ce = cudaMalloc(&k.d.owner_cnt, 8 * sizeof(uint32_t));
    if (ce == cudaSuccess) ce = cudaMalloc(&k.d.stats, txn::kDevStats * sizeof(unsigned long long));
    if (ce == cudaSuccess) ce = cudaMalloc(&k.d.req, rec * msg + 16);
    if (ce == cudaSuccess) ce = cudaMalloc(&k.d.dst, rec + 16);
    if (ce == cudaSuccess) ce = cudaMalloc(&k.out, rec * msg + 16);
    if (ce == cudaSuccess) ce = cudaHostAlloc(&k.pub, 16 * sizeof(uint32_t), cudaHostAllocMapped | cudaHostAllocPortable);
    if (ce != cudaSuccess) return fail(DINT_ENOMEM, "txn client state", ce);
    memset(k.pub, 0, 16 * sizeof(uint32_t));
    k.req = k.d.req; k.dst = k.d.dst;
    if (ce == cudaSuccess) ce = cudaHostGetDevicePointer((void**)&k.d.pub, k.pub, 0);
    if (ce == cudaSuccess) ce = cudaMemset(k.d.cl, 0, n * csz + 16);
    if (ce == cudaSuccess) ce = cudaMemset(k.d.owner_cnt, 0, 8 * sizeof(uint32_t));
    if (ce == cudaSuccess) ce = cudaMemset(k.d.stats, 0, txn::kDevStats * sizeof(unsigned long long));
    if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&k.ev, cudaEventDisableTiming);
    if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
    if (ce != cudaSuccess) return fail(DINT_EIO, "txn client setup", ce);
  }
  cudaError_t ce = cudaSetDevice(cl->dev[0]);
  if (ce == cudaSuccess) ce = cudaEventCreate(&t->t_beg);
  if (ce == cudaSuccess) ce = cudaEventCreate(&t->t_end);
  if (ce != cudaSuccess) return fail(DINT_EIO, "txn client events", ce);
  *out = t;
  return DINT_OK;
}

// enqueue one emission (step, scan, compact) on every rank; first = the clients start their first transactions
static int txn_emit(dint_txn_clients* t, int first) {
  dint_cluster* cl = t->cl;
  for (uint32_t r = 0; r < cl->G; r++) {
    TxnRank& k = t->rk[r];
    CU(cudaSetDevice(cl->dev[r]));
    const cudaStream_t s = t->mains[r];
    if (k.d.n) {
      if (cl->kind == DINT_TATP) txn::k_txn_step<DINT_TATP><<<k.tiles, kThreads, 0, s>>>(k.d, k.out, first);
      else txn::k_txn_step<DINT_SMALLBANK><<<k.tiles, kThreads, 0, s>>>(k.d, k.out, first);
      txn::k_txn_scan<<<1, kThreads, 0, s>>>(k.d, k.tiles);
      if (cl->kind == DINT_TATP) txn::k_txn_compact<txn::TM><<<k.tiles, kThreads, 0, s>>>(k.d);
      else txn::k_txn_compact<txn::SMSZ><<<k.tiles, kThreads, 0, s>>>(k.d);
      cl->eng[r]->stats.kernel_launches += 3;
    }
    CU(cudaEventRecord(k.ev, s));
  }
  CU(cudaGetLastError());
  t->started = true;
  return DINT_OK;
}

// the first emission (every client starts), or after a drain the one that resumes the clients: every idle client
// begins its next transaction and emits its first records
static int txn_start(dint_txn_clients* t) {
  if (!t->started) return txn_emit(t, 1);
  if (!t->drained) return DINT_OK;
  t->drained = false;
  return txn_emit(t, 0);
}

int dint_txn_clients_run(dint_txn_clients* t, uint32_t rounds) {
  if (!t) return set_err(DINT_EINVAL, "null argument");
  { int rc = txn_start(t); if (rc) return rc; }
  return serve_rounds(*t, t->rk, rounds, [t](int first) { return txn_emit(t, first); });
}

int dint_txn_clients_drain(dint_txn_clients* t, uint32_t max_rounds, uint32_t* rounds) {
  if (!t) return set_err(DINT_EINVAL, "null argument");
  if (rounds) *rounds = 0;
  if (!t->started || t->drained) return DINT_OK;       // nothing pending
  for (TxnRank& k : t->rk) k.d.w.drain = 1;
  const uint64_t before = t->rounds;
  int rc = serve_rounds(*t, t->rk, max_rounds, [t](int first) { return txn_emit(t, first); });
  for (TxnRank& k : t->rk) k.d.w.drain = 0;            // (an idle client resumes at the next emission)
  if (rounds) *rounds = (uint32_t)(t->rounds - before);
  if (rc && rc != DINT_EPROTO) return rc;
  uint64_t pending = 0;                                // serve_rounds waited for the last emission
  for (const TxnRank& k : t->rk) pending += k.pub[0];
  if (pending == 0) {
    t->drained = true;
    return rc;
  }
  uint64_t busy = 0;                                   // a client is busy while it emits records
  for (uint32_t r = 0; r < t->cl->G; r++) {
    std::vector<uint32_t> cnt(t->rk[r].d.n);
    CU(cudaSetDevice(t->cl->dev[r]));
    if (!cnt.empty()) CU(cudaMemcpy(cnt.data(), t->rk[r].d.cnt, cnt.size() * 4, cudaMemcpyDeviceToHost));
    for (uint32_t c : cnt) busy += c != 0;
  }
  return set_errf(DINT_EINVAL, "drain: %llu clients are still mid-transaction after %u rounds", (unsigned long long)busy, max_rounds);
}

int dint_txn_clients_rebind(dint_txn_clients* t, dint_cluster* c) {
  if (!t || !c) return set_err(DINT_EINVAL, "null argument");
  if (c->kind != t->cl->kind) return set_err(DINT_EINVAL, "rebind: the cluster serves another kind than these clients");
  if (t->started && !t->drained)
    return set_err(DINT_EINVAL, "rebind: the clients are mid-transaction (their pending round holds records): drain them first");
  dint_txn_clients* n = nullptr;
  { int rc = dint_txn_clients_create(c, t->n, (uint32_t)t->rk[0].d.gid0, t->rk[0].d.w.keys, &n); if (rc) return rc; }
  auto fail = [&](int code) { std::string keep = g_last_error; dint_txn_clients_destroy(n); g_last_error = keep; return code; };
  dint_cluster* old = t->cl;
  for (uint32_t r = 0; r < old->G; r++)                // the last emission is done
    if (cudaSetDevice(old->dev[r]) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess)
      return fail(set_err(DINT_EIO, "rebind: synchronise", cudaGetLastError()));
  // each client's record moves block by block: every (old rank, new rank) pair's common range of client ids.  The
  // pending round is empty, so no record of a round moves.
  const size_t csz = c->kind == DINT_TATP ? sizeof(txn::TatpClient) : sizeof(txn::SbClient);
  unsigned long long sum[txn::kDevStats] = {0};
  for (uint32_t r = 0; r < old->G; r++) {
    const txn::DevClients& f = t->rk[r].d;
    unsigned long long h[txn::kDevStats];
    if (cudaSetDevice(old->dev[r]) != cudaSuccess || cudaMemcpy(h, f.stats, sizeof h, cudaMemcpyDeviceToHost) != cudaSuccess)
      return fail(set_err(DINT_EIO, "rebind: counters", cudaGetLastError()));
    for (uint32_t i = 0; i < txn::kDevStats; i++) sum[i] += h[i];
    for (uint32_t q = 0; q < c->G; q++) {
      const txn::DevClients& to = n->rk[q].d;
      const uint64_t lo = std::max(f.gid0, to.gid0), hi = std::min(f.gid0 + f.n, to.gid0 + to.n);
      if (lo < hi && cudaMemcpyPeer((uint8_t*)to.cl + (lo - to.gid0) * csz, c->dev[q], (const uint8_t*)f.cl + (lo - f.gid0) * csz,
                                    old->dev[r], (hi - lo) * csz) != cudaSuccess)
        return fail(set_err(DINT_EIO, "rebind: client state", cudaGetLastError()));
    }
  }
  // the counters carry over: the stats sum the ranks, so the new rank 0 holds the old sums
  if (cudaSetDevice(c->dev[0]) != cudaSuccess || cudaMemcpy(n->rk[0].d.stats, sum, sizeof sum, cudaMemcpyHostToDevice) != cudaSuccess)
    return fail(set_err(DINT_EIO, "rebind: counters", cudaGetLastError()));
  // t takes the new ranks; n takes the old ones and releases them, and its attachment, on the old cluster
  std::swap(t->cl, n->cl);
  std::swap(t->rk, n->rk);
  std::swap(t->mains, n->mains);
  std::swap(t->t_beg, n->t_beg);
  std::swap(t->t_end, n->t_end);
  dint_txn_clients_destroy(n);
  return DINT_OK;
}

// the ranks' DevClients::stats words, summed (synchronises)
static int txn_dev_stats(dint_txn_clients* t, unsigned long long by[txn::kDevStats]) {
  { int rc = txn_start(t); if (rc) return rc; }
  for (uint32_t i = 0; i < txn::kDevStats; i++) by[i] = 0;
  for (uint32_t r = 0; r < t->cl->G; r++) {
    unsigned long long h[txn::kDevStats];
    CU(cudaSetDevice(t->cl->dev[r]));
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpy(h, t->rk[r].d.stats, sizeof h, cudaMemcpyDeviceToHost));
    for (uint32_t i = 0; i < txn::kDevStats; i++) by[i] += h[i];
  }
  return DINT_OK;
}

// out: dint_txn_stats' 18 words (requests and rounds served, transactions started, committed, started-by-type[7],
// committed-by-type[7]), then rounds served through the fallback
int dint_txn_clients_stats(dint_txn_clients* t, uint64_t out[19]) {
  if (!t || !out) return set_err(DINT_EINVAL, "null argument");
  unsigned long long by[txn::kDevStats];
  int rc = txn_dev_stats(t, by);
  if (rc) return rc;
  out[0] = t->requests; out[1] = 0; out[2] = 0; out[3] = t->rounds;
  for (int i = 0; i < 7; i++) {
    out[4 + i] = by[i]; out[11 + i] = by[7 + i];
    out[1] += by[i]; out[2] += by[7 + i];
  }
  out[18] = t->fallback_rounds;
  return DINT_OK;
}

// out: kAcquireLock replies absorbed, of them kRejectLock (false sharing) and kRejectLockSameKey, as
// tatp/caladan/client_lock.cc counts them
int dint_txn_clients_lock_stats(dint_txn_clients* t, uint64_t out[3]) {
  if (!t || !out) return set_err(DINT_EINVAL, "null argument");
  unsigned long long by[txn::kDevStats];
  int rc = txn_dev_stats(t, by);
  if (rc) return rc;
  for (int i = 0; i < 3; i++) out[i] = by[14 + i];
  return DINT_OK;
}

// test hook, global client order: the pending round (its requests and destination shards) and the replies the clients
// absorbed last; buffers of n_clients * 9 records
int dint_txn_clients_peek(dint_txn_clients* t, void* next_req, uint8_t* next_dst, uint64_t* n_next, void* last_resp, uint64_t* n_last) {
  if (!t) return set_err(DINT_EINVAL, "null argument");
  int rc;
  if ((rc = txn_start(t))) return rc;
  if ((rc = round_wait(*t, t->rk))) return rc;
  uint64_t a = 0, z = 0;
  for (uint32_t r = 0; r < t->cl->G; r++) {
    const TxnRank& k = t->rk[r];
    const uint64_t n = k.pub[0];
    CU(cudaSetDevice(t->cl->dev[r]));
    if (next_req) CU(cudaMemcpy((uint8_t*)next_req + a * t->msg, k.d.req, n * t->msg, cudaMemcpyDeviceToHost));
    if (next_dst) CU(cudaMemcpy(next_dst + a, k.d.dst, n, cudaMemcpyDeviceToHost));
    if (last_resp) CU(cudaMemcpy((uint8_t*)last_resp + z * t->msg, k.out, k.last_n * t->msg, cudaMemcpyDeviceToHost));
    a += n;
    z += k.last_n;
  }
  if (n_next) *n_next = a;
  if (n_last) *n_last = z;
  return DINT_OK;
}

// out: rounds timed, their wall time on the host (s), and the CUDA-event time of their device work on rank 0 (s)
int dint_txn_clients_times(dint_txn_clients* t, double out[3]) {
  if (!t || !out) return set_err(DINT_EINVAL, "null argument");
  out[0] = (double)t->timed; out[1] = t->wall_s; out[2] = t->dev_s;
  return DINT_OK;
}

// ---- lock_2pl / lock_fasst / store / log_server closed-loop clients on the GPU against a shard cluster -------------
// Rank r's block of clients (clients.cuh, ClientCtx::id0 = its first global id) emits one record per client into its
// request buffer; k_clients_owner_count publishes the round's per-owner counts; the round loop above serves it; the
// replies land in the block's reply buffer, in request order, where the next step absorbs them.  A cluster of these kinds
// answers like ONE sequential server fed the rank-major concatenation, so the clients take, round for round, the
// decisions of dint_clients with the same clients on one engine.
struct ClusterClientRank : RoundRank {
  ClientBlock b;                 // req = b.req, out = b.resp
  uint32_t* acc = nullptr;       // k_clients_owner_count's per-shard sums [8] and CTA ticket [1]
  uint32_t* pub_dev = nullptr;   // device view of pub
};
struct dint_cluster_clients : RoundLoop {
  int kind = 0;
  uint64_t seed = 0;
  dint_clients_cfg cfg{};        // the family the clients were made from (dint_cluster_clients_rebind makes new blocks of it)
  std::vector<ClusterClientRank> rk;
};

void dint_cluster_clients_destroy(dint_cluster_clients* t) {
  if (!t) return;
  for (size_t r = 0; r < t->rk.size(); r++) {
    ClusterClientRank& k = t->rk[r];
    cudaSetDevice(t->cl->dev[r]);
    cudaDeviceSynchronize();
    client_block_free(k.b);
    cudaFree(k.acc);
    if (k.pub) cudaFreeHost(k.pub);
    if (k.ev) cudaEventDestroy(k.ev);
  }
  if (!t->rk.empty()) cudaSetDevice(t->cl->dev[0]);
  if (t->t_beg) cudaEventDestroy(t->t_beg);
  if (t->t_end) cudaEventDestroy(t->t_end);
  delete t;
}

int dint_cluster_clients_create(dint_cluster* cl, const dint_clients_cfg* cfg, dint_cluster_clients** out) {
  if (!cl || !cfg || !out) return set_err(DINT_EINVAL, "null argument");
  *out = nullptr;
  const uint32_t G = cl->G, n_clients = cfg->n_clients;
  auto lo_of = [&](uint32_t r) { return (uint32_t)((uint64_t)n_clients * r / G); };
  for (uint32_t r = 0; r < G; r++)                     // otherwise every round would be served in pieces
    if (lo_of(r + 1) - lo_of(r) > cl->max_n) return set_err(DINT_EINVAL, "a rank's block of clients exceeds the cluster's max_batch");
  if (fallback_piece(cl) == 0) return set_err(DINT_EINVAL, "the cluster's max_batch must be >= 16");
  dint_cluster_clients* t = new dint_cluster_clients();
  t->cl = cl; t->kind = cl->kind; t->msg = kMsgSize[cl->kind]; t->seed = cfg->seed; t->local = cl->kind == DINT_LOG; t->cfg = *cfg;
  t->rk.resize(G);
  auto fail = [&](int code) { std::string keep = g_last_error; dint_cluster_clients_destroy(t); g_last_error = keep; return code; };
  for (uint32_t r = 0; r < G; r++) {
    ClusterClientRank& k = t->rk[r];
    const uint32_t lo = lo_of(r), n = lo_of(r + 1) - lo;
    t->mains.push_back(cl->shared_device ? cl->eng[0]->stream : cl->eng[r]->stream);
    if (int rc = client_block_make(cl->kind, cfg, cl->dev[r], lo, n, &k.b)) return fail(rc);
    k.req = k.b.req; k.out = k.b.resp;
    cudaError_t ce = cudaSetDevice(cl->dev[r]);
    if (ce == cudaSuccess) ce = cudaMalloc(&k.acc, 16 * sizeof(uint32_t));
    if (ce == cudaSuccess) ce = cudaMemset(k.acc, 0, 16 * sizeof(uint32_t));
    if (ce == cudaSuccess) ce = cudaHostAlloc(&k.pub, 16 * sizeof(uint32_t), cudaHostAllocMapped | cudaHostAllocPortable);
    if (ce != cudaSuccess) return fail(set_err(DINT_ENOMEM, "cluster client state", ce));
    memset(k.pub, 0, 16 * sizeof(uint32_t));
    k.pub[0] = n;                                      // (log_server rounds are not counted: their size is the block's)
    if (ce == cudaSuccess) ce = cudaHostGetDevicePointer((void**)&k.pub_dev, k.pub, 0);
    if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&k.ev, cudaEventDisableTiming);
    if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
    if (ce != cudaSuccess) return fail(set_err(DINT_EIO, "cluster client setup", ce));
  }
  cudaError_t ce = cudaSetDevice(cl->dev[0]);
  if (ce == cudaSuccess) ce = cudaEventCreate(&t->t_beg);
  if (ce == cudaSuccess) ce = cudaEventCreate(&t->t_end);
  if (ce != cudaSuccess) return fail(set_err(DINT_EIO, "cluster client events", ce));
  *out = t;
  return DINT_OK;
}

// enqueue one emission on every rank: the clients' kernel, then (except log_server) the per-owner count.  count_only:
// the per-owner count of the pending round alone (after a rebind, for the new cluster's owners).
static int cluster_clients_emit(dint_cluster_clients* t, int first, bool count_only = false) {
  dint_cluster* cl = t->cl;
  for (uint32_t r = 0; r < cl->G; r++) {
    ClusterClientRank& k = t->rk[r];
    dint_engine* e = cl->eng[r];
    CU(cudaSetDevice(cl->dev[r]));
    const cudaStream_t s = t->mains[r];
    const uint32_t n = k.b.cc.n_clients, blocks = (n + kThreads - 1) / kThreads;
    if (n) {
      if (!count_only) {
        clients_launch(t->kind, t->seed, k.b, first != 0, s);
        e->stats.kernel_launches++;
      }
      if (!t->local) {
        switch (t->kind) {
          case DINT_FASST: k_clients_owner_count<K_FASST><<<blocks, kThreads, 0, s>>>(e->ctx, k.b.req, n, k.acc, k.pub_dev); break;
          case DINT_LOCK2PL: k_clients_owner_count<K_LOCK2PL><<<blocks, kThreads, 0, s>>>(e->ctx, k.b.req, n, k.acc, k.pub_dev); break;
          default: k_clients_owner_count<K_STORE><<<blocks, kThreads, 0, s>>>(e->ctx, k.b.req, n, k.acc, k.pub_dev); break;
        }
        e->stats.kernel_launches++;
      }
    }
    CU(cudaEventRecord(k.ev, s));
  }
  CU(cudaGetLastError());
  t->started = true;
  return DINT_OK;
}

int dint_cluster_clients_run(dint_cluster_clients* t, uint32_t rounds) {
  if (!t) return set_err(DINT_EINVAL, "null argument");
  return serve_rounds(*t, t->rk, rounds, [t](int first) { return cluster_clients_emit(t, first); });
}

// Clients [lo, lo + n) of block `from` copied into block `to` (first global id to_lo): the per-client state, the pending
// round's requests and the last replies.  Arrays are per client, or [10][n_clients] rows (rk, rv).
static int client_block_copy(int kind, const ClientBlock& from, int from_dev, const ClientBlock& to, int to_dev, uint32_t lo,
                             uint32_t n) {
  const uint32_t fo = lo - from.cc.id0, to_off = lo - to.cc.id0, msg = kMsgSize[kind];
  auto cp = [&](const void* f, void* t, size_t es, size_t rows) -> int {
    if (!f || !t) return DINT_OK;
    for (size_t i = 0; i < rows; i++)
      CU(cudaMemcpyPeer((uint8_t*)t + (i * to.cc.n_clients + to_off) * es, to_dev, (const uint8_t*)f + (i * from.cc.n_clients + fo) * es,
                        from_dev, (size_t)n * es));
    return DINT_OK;
  };
  int rc;
  if ((rc = cp(from.req, to.req, msg, 1)) || (rc = cp(from.resp, to.resp, msg, 1))) return rc;
  if ((rc = cp(from.cc.hdr, to.cc.hdr, 8, 1)) || (rc = cp(from.cc.rng, to.cc.rng, 8, 1)) || (rc = cp(from.cc.lcg, to.cc.lcg, 8, 1))) return rc;
  if ((rc = cp(from.cc.rk, to.cc.rk, 4, 10)) || (rc = cp(from.cc.rv, to.cc.rv, 4, 10))) return rc;
  return DINT_OK;
}

int dint_cluster_clients_rebind(dint_cluster_clients* t, dint_cluster* c) {
  if (!t || !c) return set_err(DINT_EINVAL, "null argument");
  if (c->kind != t->kind) return set_err(DINT_EINVAL, "the cluster serves another kind than these clients");
  if (c->G > kMaxShards) return set_err(DINT_EINVAL, "bad shard count");
  dint_cluster_clients* n = nullptr;
  { int rc = dint_cluster_clients_create(c, &t->cfg, &n); if (rc) return rc; }   // refuses a max_batch below a rank's block
  auto fail = [&](int code) { std::string keep = g_last_error; dint_cluster_clients_destroy(n); g_last_error = keep; return code; };
  dint_cluster* old = t->cl;
  for (uint32_t r = 0; r < old->G; r++) {              // the pending emission and any copy of it are done
    if (cudaSetDevice(old->dev[r]) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess)
      return fail(set_err(DINT_EIO, "rebind: synchronise", cudaGetLastError()));
  }
  // the clients move block by block: every (old rank, new rank) pair's common range of client ids
  unsigned long long sum[8] = {0};
  for (uint32_t r = 0; r < old->G; r++) {
    const ClientBlock& f = t->rk[r].b;
    unsigned long long h[8];
    if (cudaSetDevice(old->dev[r]) != cudaSuccess || cudaMemcpy(h, f.cc.stats, sizeof h, cudaMemcpyDeviceToHost) != cudaSuccess)
      return fail(set_err(DINT_EIO, "rebind: counters", cudaGetLastError()));
    for (int i = 0; i < 8; i++) sum[i] += h[i];
    for (uint32_t q = 0; q < c->G; q++) {
      const ClientBlock& to = n->rk[q].b;
      const uint32_t lo = std::max(f.cc.id0, to.cc.id0), hi = std::min(f.cc.id0 + f.cc.n_clients, to.cc.id0 + to.cc.n_clients);
      if (lo < hi) { int rc = client_block_copy(t->kind, f, old->dev[r], to, c->dev[q], lo, hi - lo); if (rc) return fail(rc); }
    }
  }
  // the counters carry over: dint_cluster_clients_stats sums the blocks, so the new rank 0 holds the old sums
  if (cudaSetDevice(c->dev[0]) != cudaSuccess || cudaMemcpy(n->rk[0].b.cc.stats, sum, sizeof sum, cudaMemcpyHostToDevice) != cudaSuccess)
    return fail(set_err(DINT_EIO, "rebind: counters", cudaGetLastError()));
  // t takes the new blocks; n takes the old ones and releases them on the old cluster's devices
  std::swap(t->cl, n->cl);
  std::swap(t->rk, n->rk);
  std::swap(t->mains, n->mains);
  std::swap(t->t_beg, n->t_beg);
  std::swap(t->t_end, n->t_end);
  dint_cluster_clients_destroy(n);
  if (t->started) {                                    // the pending round, counted for the new cluster's owners
    int rc = cluster_clients_emit(t, 0, true);
    if (rc) return rc;
  }
  return DINT_OK;
}

// out: dint_clients_stats_all's 6 words (rounds counted once, not once per rank), then rounds served in pieces
int dint_cluster_clients_stats(dint_cluster_clients* t, uint64_t out[7]) {
  if (!t || !out) return set_err(DINT_EINVAL, "null argument");
  unsigned long long s[6] = {0};
  for (uint32_t r = 0; r < t->cl->G; r++) {
    unsigned long long h[6];
    CU(cudaSetDevice(t->cl->dev[r]));
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpy(h, t->rk[r].b.cc.stats, sizeof h, cudaMemcpyDeviceToHost));
    for (int i = 0; i < 6; i++) s[i] += h[i];
  }
  out[0] = s[0]; out[1] = s[1]; out[2] = s[2]; out[3] = s[3]; out[4] = s[5]; out[5] = t->rounds; out[6] = t->fallback_rounds;
  return DINT_OK;
}

// test hook, global client order: the requests the clients send next and the replies they absorbed last (host buffers
// of n_clients * dint_msg_size(kind) bytes)
int dint_cluster_clients_peek(dint_cluster_clients* t, void* next_req, void* last_resp) {
  if (!t) return set_err(DINT_EINVAL, "null argument");
  int rc;
  if (!t->started && (rc = cluster_clients_emit(t, 1))) return rc;
  if ((rc = round_wait(*t, t->rk))) return rc;
  uint64_t a = 0;
  for (uint32_t r = 0; r < t->cl->G; r++) {
    const ClusterClientRank& k = t->rk[r];
    const size_t bytes = (size_t)k.b.cc.n_clients * t->msg;
    CU(cudaSetDevice(t->cl->dev[r]));
    if (next_req && bytes) CU(cudaMemcpy((uint8_t*)next_req + a, k.b.req, bytes, cudaMemcpyDeviceToHost));
    if (last_resp && bytes) CU(cudaMemcpy((uint8_t*)last_resp + a, k.b.resp, bytes, cudaMemcpyDeviceToHost));
    a += bytes;
  }
  return DINT_OK;
}

// out: rounds timed, their wall time on the host (s), and the CUDA-event time of their device work on rank 0 (s)
int dint_cluster_clients_times(dint_cluster_clients* t, double out[3]) {
  if (!t || !out) return set_err(DINT_EINVAL, "null argument");
  out[0] = (double)t->timed; out[1] = t->wall_s; out[2] = t->dev_s;
  return DINT_OK;
}

}  // extern "C"
