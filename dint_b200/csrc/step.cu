// step.cu -- the multi-GPU step of libdint_b200.so: the C routing ABI (dint_route_*, dint_p2p_*), the pipelined
// exchange of one process's ranks over NVLink peer memory (dint_shard_*), and clusters of G shards driven by one
// process (dint_cluster_*).
#include <cmath>

#include "host.cuh"
#include "route.cuh"

namespace dint {

// owner shard of every request (multi-GPU routing; see dint_route_owner)
template <int KIND>
__global__ void __launch_bounds__(kThreads) k_route_owner(const Ctx c, const uint8_t* req, uint32_t n, uint8_t* owner) {
  const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
  if (i < n) owner[i] = (uint8_t)route_owner_of<KIND>(c, req + (size_t)i * Wire<KIND>::MSG);
}

// ---- multi-GPU dispatch: stable partition of a batch by owner shard -------------------------------------
// (1) k_exact_count: per 256-record tile, how many records go to each shard;  (2) k_exact_scan (one CTA per shard):
// exclusive offsets -- shard-major, then tile order -- and the per-shard totals;  (3) k_exact_scatter: every
// record is copied to its slot (stable inside a shard: tile order, then thread order) and the inverse
// permutation is recorded.  Afterwards the wire records sit grouped by destination, ready for the exchange.
__global__ void __launch_bounds__(kThreads) k_exact_count(const uint8_t* owner, uint32_t n, uint32_t world, uint32_t* tilecnt) {
  __shared__ uint32_t cnt[kMaxShards];
  if (threadIdx.x < kMaxShards) cnt[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
  const uint32_t o = i < n ? owner[i] : 0xffu;
  const uint32_t peers = __match_any_sync(0xffffffffu, o);
  if (o < world && (int)lane_id() == __ffs(peers) - 1) atomicAdd(&cnt[o], (uint32_t)__popc(peers));
  __syncthreads();
  if (threadIdx.x < world) tilecnt[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = cnt[threadIdx.x];   // shard-major
}
__global__ void __launch_bounds__(kThreads) k_exact_scan(uint32_t* tilecnt, uint32_t n_tiles, uint32_t* totals) {
  // one CTA per shard: exclusive scan of that shard's row of per-tile counts, row total -> totals[shard]
  __shared__ uint32_t wsum[kThreads / 32];
  uint32_t* row = tilecnt + (size_t)blockIdx.x * n_tiles;
  const uint32_t total = cta_exclusive_scan<uint32_t>(row, row, n_tiles, 0u, wsum);
  if (threadIdx.x == 0) totals[blockIdx.x] = total;
}
template <int MSG>
__global__ void __launch_bounds__(kThreads) k_exact_scatter(const uint8_t* req, const uint8_t* owner, uint32_t n, uint32_t world,
                                                            const uint32_t* tilebase, const uint32_t* totals, uint8_t* out,
                                                            uint32_t* perm) {
  __shared__ uint32_t wcnt[kThreads / 32][kMaxShards];
  const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
  if (threadIdx.x < (kThreads / 32) * kMaxShards) ((uint32_t*)wcnt)[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t o = i < n ? owner[i] : 0xffu;
  const uint32_t peers = __match_any_sync(0xffffffffu, o);
  const uint32_t before = __popc(peers & ((1u << lane_id()) - 1u));
  if (o < world && before == 0) wcnt[warp_id()][o] = __popc(peers);
  __syncthreads();
  if (o < world) {
    uint32_t pos = tilebase[(size_t)o * gridDim.x + blockIdx.x] + before;
    for (uint32_t w = 0; w < warp_id(); w++) pos += wcnt[w][o];
    for (uint32_t q = 0; q < o; q++) pos += totals[q];                 // start of shard o's segment
    copy_record<MSG>(out + (size_t)pos * MSG, req + (size_t)i * MSG);
    perm[pos] = i;
  }
}

// ---- exchange over NVLink peer memory: epoch flags (PeerPtrs, kernels.cuh) ---------------------------------------
// after the data: tell every peer that epoch `e` of this rank's slab is complete
__global__ void k_p2p_signal(PeerPtrs sig, uint32_t world, uint32_t me, uint32_t epoch) {
  if (threadIdx.x < world) {
    __threadfence_system();
    volatile uint32_t* flag = (volatile uint32_t*)sig.p[threadIdx.x] + me;
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(epoch) : "memory");
  }
}
// before consuming: wait until every peer has signalled epoch `e` (bounded spin: ~4 s, then *timeout = 1).
// Bit 31 of a request flag = "this source could not fit one of its slabs": the first epoch for which any source says so
// is recorded in *bad (0 = none), and from then on every engine launch of the step returns at once (Ctx::skip): the
// batch and everything behind it is left unserved on EVERY shard -- all owners see all sources' flags -- so the server
// state stays consistent and the host can serve those records again in smaller rounds.
__global__ void k_p2p_wait(const uint32_t* my_sig, uint32_t world, uint32_t epoch, uint32_t* timeout, uint32_t* bad) {
  if (threadIdx.x < world) {
    const long long t0 = clock64();
    uint32_t v;
    do {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(my_sig + threadIdx.x) : "memory");
      if (clock64() - t0 > 8000000000LL) { atomicExch(timeout, 1u); break; }
    } while ((int32_t)((v & ~kSigOverflow) - epoch) < 0);
    if (bad && (v & kSigOverflow) && (v & ~kSigOverflow) == epoch) atomicCAS(bad, 0u, epoch);
  }
  __syncthreads();
  __threadfence_system();
}

// combine: replies arrive in partition order; put each back at its original index
template <int MSG>
__global__ void __launch_bounds__(kThreads) k_exact_unpermute(const uint8_t* sorted, const uint32_t* perm, uint32_t n, uint8_t* out) {
  const uint32_t pos = blockIdx.x * kThreads + threadIdx.x;
  if (pos >= n) return;
  const uint32_t idx = perm[pos];
  if (idx == 0xffffffffu) return;                        // padding slot of a slab
  copy_record<MSG>(out + (size_t)idx * MSG, sorted + (size_t)pos * MSG);
}

}  // namespace dint

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

extern "C" {

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
// `host` given: the batches come from / go to HOST memory through S sets of each rank's engine ring (HostRing) --
// H2D of batch j+1 and D2H of batch j-1 run on the ring's copy streams next to the exchange of batch j.
int shard_run(dint_shard_ctx* const* ranks, uint32_t R, uint32_t k, std::vector<std::vector<ShardBatch>>& b, cudaStream_t const* mains,
              const std::vector<std::vector<HostBatch>>* host) {
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

}  // extern "C"

// ---- dint_cluster_*: G shards driven by ONE process (SURVEY.md 8(b): dint_create(kind, cfg, n_gpus) / dint_submit(..., dst_shard, ...)) ----
// The exchange buffers of a cluster: per rank one allocation {inbox sets | return-buffer sets | signal block}
constexpr uint32_t kClusterSets = 3;
static size_t cluster_region(const dint_cluster* cl) { return ((size_t)cl->G * cl->cap * kMsgSize[cl->kind] + 255) / 256 * 256; }
uint64_t cluster_sig_block(const dint_cluster* cl, uint32_t r) { return (uint64_t)cl->bufs[r] + 2 * kClusterSets * cluster_region(cl); }

// the configuration shard r of a cluster is created with (cl->base, cap and G set)
dint_cfg cluster_shard_cfg(const dint_cluster* cl, uint32_t r) {
  dint_cfg c = cl->base;
  if (cl->by_dst) { c.n_shards = 1; c.shard_id = 0; c.txn_shards = cl->G; c.txn_shard_id = r; }
  else { c.n_shards = cl->G; c.shard_id = r; }
  const uint32_t chunk_need = (uint32_t)(((uint64_t)cl->G * cl->cap + kTile - 1) / kTile * kTile);
  if (c.chunk == 0 || c.chunk < chunk_need) c.chunk = chunk_need;        // one batch of the exchange = one engine chunk
  return c;
}

// one shard context per rank over the cluster's exchange buffers, engine r = eng[r]; every epoch starts at 0, so the
// signal blocks must be zero before the first batch
int cluster_ranks(const dint_cluster* cl, const std::vector<dint_engine*>& eng, std::vector<dint_shard_ctx*>& out) {
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

extern "C" {

void dint_cluster_destroy(dint_cluster* cl) {
  if (!cl) return;
  for (auto* c : cl->sh) dint_shard_destroy(c);
  for (size_t r = 0; r < cl->bufs.size(); r++) { cudaSetDevice(cl->dev[r]); cudaFree(cl->bufs[r]); }
  for (auto* e : cl->eng) dint_destroy(e);
  delete cl;
}

}  // extern "C"


// dint_cluster_create; with image_dir dint_cluster_image_open: then shard r's engine is opened from its image; with
// `from` dint_cluster_reshard: then shard r's engine is filled from the source cluster's shards.  With image_dir and
// `rebuild` (dint_cluster_image_open_rebuild): the shards of *rebuild (known missing) and those whose image fails with
// DINT_EIO are rebuilt from the others once those are open; *rebuild is then set to every shard rebuilt.
int cluster_make(int kind, const dint_cfg* cfg, int n_gpus, const int* devices, uint64_t max_batch, const char* image_dir,
                 const DeriveFrom* from, uint32_t* rebuild, dint_cluster** out) {
  if (!out || kind < 0 || kind >= DINT_NUM_KINDS || n_gpus < 1 || n_gpus > kMaxShards) return set_err(DINT_EINVAL, "bad kind / n_gpus");
  *out = nullptr;
  const bool by_dst = kind == DINT_TATP || kind == DINT_SMALLBANK;
  if (by_dst && n_gpus == 2) return set_err(DINT_EINVAL, "tatp / smallbank placement needs 1 or >= 3 shards (primary + 2 backups)");
  if (cfg) { int rc = check_kind_flags(kind, cfg->flags); if (rc) return rc; }
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
    if (rc == DINT_OK) rc = rebuild_shards(cl, failed);
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
  if (rc != DINT_OK) return keep_error(rc, [&] { dint_cluster_destroy(cl); });
  *out = cl;
  return DINT_OK;
}

extern "C" {

int dint_cluster_create(int kind, const dint_cfg* cfg, int n_gpus, const int* devices, uint64_t max_batch, dint_cluster** out) {
  return cluster_make(kind, cfg, n_gpus, devices, max_batch, nullptr, nullptr, nullptr, out);
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
