// engine.cu -- the engine of libdint_b200.so: state allocation in HBM, the per-chunk launch sequence, host<->device
// pipelining for dint_submit(), snapshots and statistics.  No CPU implementation of the request path exists here:
// without a CUDA device every compute entry point returns DINT_ENODEV.  host.cuh lists the other units.
#include "host.cuh"

thread_local std::string g_last_error;

namespace dint {

// K1b: absolute append ordinal of every tile's first log append (single CTA).
__global__ void __launch_bounds__(kThreads) k_log_scan(const Ctx c) {
  if (c.skip && __ldcg(c.skip)) return;
  __shared__ uint32_t wsum[kThreads / 32];
  const unsigned long long end =
      cta_exclusive_scan<unsigned long long>(c.log_tilecnt, c.log_tilebase, c.n_tiles, threadIdx.x == 0 ? c.log_total[0] : 0ull, wsum);
  if (threadIdx.x == 0) {
    c.log_total[1] = end;                 // end ordinal of this chunk
    c.log_total[0] = end;                 // base of the next chunk
  }
}

// K2b (tatp): a kDeleteLog append leaves the value bytes of its ring slot as the slot's last kCommitLog wrote them
// (tatp/udp/server_shard.cc:196-203).  When a chunk appends more than ring_n entries, K2 writes only the last append to
// every slot (log_keep), so a kDeleteLog it wrote gets its value bytes here: from the last kCommitLog of this chunk to
// the same slot, or, when there is none, they are already in the ring.
__global__ void __launch_bounds__(kThreads) k_log_vals(const Ctx c) {
  using W = Wire<K_TATP>;
  if (c.skip && __ldcg(c.skip)) return;
  const unsigned long long base = c.log_tilebase[0], end = c.log_total[1];
  if (end - base <= c.ring_n) return;
  for (unsigned long long ord = end - c.ring_n + blockIdx.x * kThreads + threadIdx.x; ord < end; ord += (unsigned long long)gridDim.x * kThreads) {
    if (c.log_src[ord - base] & 1u) continue;            // a kCommitLog: K2 wrote the whole entry
    for (unsigned long long o = ord; o >= base + c.ring_n;) {
      o -= c.ring_n;
      const uint32_t s = c.log_src[o - base];
      if (s & 1u) {
        const uint8_t* src = c.req + (size_t)(s >> 1) * W::MSG + W::VAL;
        uint8_t* e = c.ring + (size_t)(ord % c.ring_n) * W::LOGENT + 16;
        for (int b = 0; b < 40; b++) e[b] = src[b];
        break;
      }
    }
  }
}

}  // namespace dint

static const char* kKernelNames[KT_NUM] = {"k_classify", "k_log_scan", "k_apply", "k_ordered", "k_kv_load"};

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
int prof_flush(dint_engine* e) {
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

// ---- per-chunk launch sequence ------------------------------------------------------------------------
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
int kv_publish_counts(dint_engine* e, cudaStream_t s) {
  if (e->ctx.n_tables == 0 || !e->h_kvcnt) return DINT_OK;
  CU(cudaMemcpyAsync(e->h_kvcnt, e->ctx.tbl[0].live, 16 * e->ctx.n_tables, cudaMemcpyDeviceToHost, s));   // (the tables' counters are contiguous)
  CU(cudaEventRecord(e->ev_kvcnt, s));
  return DINT_OK;
}

// The last step of making an engine from state held elsewhere (an image, a re-shard, a rebuild).  Its KV tables' {live, used} counters were written with the state: set up
// and refresh their host mirror, as dint_snapshot_restore does, so that the next call's kv_maintain decides on them.
int engine_ready(dint_engine* e) {
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
int run_device(dint_engine* e, const uint8_t* req, uint64_t n, uint8_t* resp, cudaStream_t s, const StepTarget* tgt) {
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
int pull_counters(dint_engine* e) {
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
int ring_reserve(dint_engine* e, uint32_t sets, size_t in_bytes, size_t aux_bytes, size_t out_bytes) {
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
int ring_stage_in(dint_engine* e, uint64_t j, const void* host_in, size_t in_bytes, const void* host_aux, size_t aux_bytes, cudaStream_t consumer) {
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
int ring_drain_out(dint_engine* e, uint64_t j, void* host_out, size_t out_bytes, cudaStream_t producer) {
  HostRing& R = e->ring;
  const uint32_t b = (uint32_t)(j % R.sets);
  CU(cudaEventRecord(R.ready[b], producer));
  CU(cudaStreamWaitEvent(R.s_out, R.ready[b], 0));
  if (out_bytes) CU(cudaMemcpyAsync(host_out, R.out[b].p, out_bytes, cudaMemcpyDeviceToHost, R.s_out));
  CU(cudaEventRecord(R.d2h[b], R.s_out));
  e->stats.d2h_bytes += out_bytes;
  return DINT_OK;
}

int check_kind_flags(int kind, uint32_t flags) {
  if ((flags & DINT_CFG_LOCK_HOLDER_KEYS) && kind != DINT_TATP) return set_err(DINT_EINVAL, "DINT_CFG_LOCK_HOLDER_KEYS is a tatp option");
  if ((flags & DINT_CFG_STORE_EBPF_MASK) && kind != DINT_STORE) return set_err(DINT_EINVAL, "DINT_CFG_STORE_EBPF_* is a store option");
  if ((flags & DINT_CFG_TATP_EBPF) && kind != DINT_TATP) return set_err(DINT_EINVAL, "DINT_CFG_TATP_EBPF is a tatp option");
  if ((flags & DINT_CFG_SMALLBANK_EBPF) && kind != DINT_SMALLBANK) return set_err(DINT_EINVAL, "DINT_CFG_SMALLBANK_EBPF is a smallbank option");
  return DINT_OK;
}

// ======================================================================================================
extern "C" {

uint32_t dint_msg_size(int kind) { return (kind >= 0 && kind < DINT_NUM_KINDS) ? kMsgSize[kind] : 0; }
uint32_t dint_log_entry_size(int kind) { return (kind >= 0 && kind < DINT_NUM_KINDS) ? kLogEntry[kind] : 0; }
const char* dint_last_error(void) { return g_last_error.c_str(); }
uint64_t dint_test_fasthash64(uint64_t x, int len) { return len == 4 ? fasthash64_u32((uint32_t)x) : fasthash64_u64(x); }
uint32_t dint_test_fastmod(uint64_t n, uint32_t d) { FastMod f = make_fastmod(d); return fast_mod(n, f); }
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
  if (int rc = check_kind_flags(kind, cf.flags)) { delete e; return rc; }
  if ((cf.flags & DINT_CFG_TATP_EBPF) && cf.n_shards != 1) { delete e; return set_err(DINT_EINVAL, "DINT_CFG_TATP_EBPF needs n_shards = 1 (place tatp shards with txn_shards)"); }
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

}  // extern "C"

// ---- state snapshots (checkpoint / restore of one engine's whole server state, device to device) --------------
struct dint_snapshot {
  dint_engine* e = nullptr;
  std::vector<std::pair<void*, size_t>> live;   // the engine's state arrays
  std::vector<void*> copy;
  uint64_t kv_cap[kMaxTables]{};                 // table capacities at snapshot time (a rehash in between invalidates it)
};
void snapshot_regions(dint_engine* e, std::vector<std::pair<void*, size_t>>& r) {
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

extern "C" {
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

}  // extern "C"
