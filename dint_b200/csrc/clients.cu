// clients.cu -- closed-loop clients on the GPU: lock_2pl / lock_fasst / store / log_server clients against one engine
// (dint_clients_*) or a shard cluster (dint_cluster_clients_*), and TATP / SmallBank clients against a shard cluster
// (dint_txn_clients_*).  clients.cuh and txn_clients.cuh hold their state machines.
#include <algorithm>
#include <cmath>

#include "host.cuh"
#include "clients.cuh"
#include "txn_clients.cuh"

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
  // the pinned block, zeroed (a family's client state); with pub_map its device view and the event (its setup)
  cudaError_t pub_alloc() {
    cudaError_t ce = cudaHostAlloc(&pub, 16 * sizeof(uint32_t), cudaHostAllocMapped | cudaHostAllocPortable);
    if (ce == cudaSuccess) memset(pub, 0, 16 * sizeof(uint32_t));
    return ce;
  }
  cudaError_t pub_map(uint32_t** pub_dev) {
    cudaError_t ce = cudaHostGetDevicePointer((void**)pub_dev, pub, 0);
    return ce == cudaSuccess ? cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) : ce;
  }
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
  cudaError_t make_timers() {                     // t_beg / t_end, on rank 0's device
    cudaError_t ce = cudaSetDevice(cl->dev[0]);
    if (ce == cudaSuccess) ce = cudaEventCreate(&t_beg);
    if (ce == cudaSuccess) ce = cudaEventCreate(&t_end);
    return ce;
  }
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

// releases every rank, free_rank(k) its family's state on its device once that device is idle, and the round timers
template <class Rank, class FreeRank>
static void round_release(RoundLoop& L, std::vector<Rank>& rk, FreeRank&& free_rank) {
  for (size_t r = 0; r < rk.size(); r++) {
    Rank& k = rk[r];
    cudaSetDevice(L.cl->dev[r]);
    cudaDeviceSynchronize();
    free_rank(k);
    if (k.pub) cudaFreeHost(k.pub);
    if (k.ev) cudaEventDestroy(k.ev);
  }
  if (!rk.empty()) cudaSetDevice(L.cl->dev[0]);
  if (L.t_beg) cudaEventDestroy(L.t_beg);
  if (L.t_end) cudaEventDestroy(L.t_end);
}

// The rebind of a family of clients: n is a new handle of the same clients on the cluster they move to.  Once the old
// devices are done, the ranks' NSTATS counters are summed, copy(from, from_dev, to, to_dev, lo, hi) moves clients
// [lo, hi) for every (old rank, new rank) pair whose blocks share some, and the sums go to the new rank 0 (the stats sum
// the ranks).  Then t takes the new ranks and n the old ones, which destroy(n) releases on the old cluster.  On a
// failure destroy(n) releases the new ranks and t is as it was.
template <uint32_t NSTATS, class T, class Copy, class Destroy>
static int round_rebind(T* t, T* n, Copy&& copy, Destroy&& destroy) {
  auto fail = [&](int code) { return keep_error(code, [&] { destroy(n); }); };
  dint_cluster *old = t->cl, *c = n->cl;
  for (uint32_t r = 0; r < old->G; r++)                // the last emission is done
    if (cudaSetDevice(old->dev[r]) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess)
      return fail(set_err(DINT_EIO, "rebind: synchronise", cudaGetLastError()));
  unsigned long long sum[NSTATS] = {0};
  for (uint32_t r = 0; r < old->G; r++) {
    const auto& f = t->rk[r];
    unsigned long long h[NSTATS];
    if (cudaSetDevice(old->dev[r]) != cudaSuccess || cudaMemcpy(h, f.stats(), sizeof h, cudaMemcpyDeviceToHost) != cudaSuccess)
      return fail(set_err(DINT_EIO, "rebind: counters", cudaGetLastError()));
    for (uint32_t i = 0; i < NSTATS; i++) sum[i] += h[i];
    for (uint32_t q = 0; q < c->G; q++) {
      const auto& to = n->rk[q];
      const uint64_t lo = std::max(f.id0(), to.id0()), hi = std::min(f.id0() + f.n_ids(), to.id0() + to.n_ids());
      if (lo < hi) { int rc = copy(f, old->dev[r], to, c->dev[q], lo, hi); if (rc) return fail(rc); }
    }
  }
  if (cudaSetDevice(c->dev[0]) != cudaSuccess || cudaMemcpy(n->rk[0].stats(), sum, sizeof sum, cudaMemcpyHostToDevice) != cudaSuccess)
    return fail(set_err(DINT_EIO, "rebind: counters", cudaGetLastError()));
  std::swap(t->cl, n->cl);
  std::swap(t->rk, n->rk);
  std::swap(t->mains, n->mains);
  std::swap(t->t_beg, n->t_beg);
  std::swap(t->t_end, n->t_end);
  destroy(n);
  return DINT_OK;
}

extern "C" {
// ---- TATP / SmallBank closed-loop clients on the GPU against a shard cluster (txn_clients.cuh) ---------------
// Every shard sees its records in the order one host TxnWorkload would send them.  A round's emission is three kernels
// per rank: step / scan / compact leave the round in req[] / dst[] and its size and per-shard counts in pub.
struct TxnRank : RoundRank {
  txn::DevClients d{};
  uint32_t tiles = 0;
  unsigned long long* stats() const { return d.stats; }
  uint64_t id0() const { return d.gid0; }
  uint64_t n_ids() const { return d.n; }
};
struct dint_txn_clients : RoundLoop {
  uint32_t n = 0;
  bool drained = false;          // the pending round is empty after a drain: the next run / peek / stats resumes
  std::vector<TxnRank> rk;
};

void dint_txn_clients_destroy(dint_txn_clients* t) {
  if (!t) return;
  round_release(*t, t->rk, [](TxnRank& k) {
    cudaFree(k.d.cl); cudaFree(k.d.stg); cudaFree(k.d.stg_dst); cudaFree(k.d.cnt); cudaFree(k.d.off); cudaFree(k.d.tile_sum);
    cudaFree(k.d.owner_cnt); cudaFree(k.d.stats); cudaFree(k.d.req); cudaFree(k.d.dst); cudaFree(k.out);
  });
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
  auto fail = [&](int code, const char* what, cudaError_t ce) {
    set_err(code, what, ce);
    return keep_error(code, [&] { dint_txn_clients_destroy(t); });
  };
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
    if (ce == cudaSuccess) ce = k.pub_alloc();
    if (ce != cudaSuccess) return fail(DINT_ENOMEM, "txn client state", ce);
    k.req = k.d.req; k.dst = k.d.dst;
    if (ce == cudaSuccess) ce = k.pub_map(&k.d.pub);
    if (ce == cudaSuccess) ce = cudaMemset(k.d.cl, 0, n * csz + 16);
    if (ce == cudaSuccess) ce = cudaMemset(k.d.owner_cnt, 0, 8 * sizeof(uint32_t));
    if (ce == cudaSuccess) ce = cudaMemset(k.d.stats, 0, txn::kDevStats * sizeof(unsigned long long));
    if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
    if (ce != cudaSuccess) return fail(DINT_EIO, "txn client setup", ce);
  }
  if (cudaError_t ce = t->make_timers()) return fail(DINT_EIO, "txn client events", ce);
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
  // each client's record moves; the pending round is empty, so no record of a round moves.  n releases the old ranks
  // and their attachment on the old cluster.
  const size_t csz = c->kind == DINT_TATP ? sizeof(txn::TatpClient) : sizeof(txn::SbClient);
  return round_rebind<txn::kDevStats>(t, n, [&](const TxnRank& f, int f_dev, const TxnRank& to, int to_dev, uint64_t lo, uint64_t hi) -> int {
    if (cudaMemcpyPeer((uint8_t*)to.d.cl + (lo - to.d.gid0) * csz, to_dev, (const uint8_t*)f.d.cl + (lo - f.d.gid0) * csz, f_dev,
                       (hi - lo) * csz) != cudaSuccess)
      return set_err(DINT_EIO, "rebind: client state", cudaGetLastError());
    return DINT_OK;
  }, dint_txn_clients_destroy);
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
  unsigned long long* stats() const { return b.cc.stats; }
  uint64_t id0() const { return b.cc.id0; }
  uint64_t n_ids() const { return b.cc.n_clients; }
};
struct dint_cluster_clients : RoundLoop {
  int kind = 0;
  uint64_t seed = 0;
  dint_clients_cfg cfg{};        // the family the clients were made from (dint_cluster_clients_rebind makes new blocks of it)
  std::vector<ClusterClientRank> rk;
};

void dint_cluster_clients_destroy(dint_cluster_clients* t) {
  if (!t) return;
  round_release(*t, t->rk, [](ClusterClientRank& k) {
    client_block_free(k.b);
    cudaFree(k.acc);
  });
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
  auto fail = [&](int code) { return keep_error(code, [&] { dint_cluster_clients_destroy(t); }); };
  for (uint32_t r = 0; r < G; r++) {
    ClusterClientRank& k = t->rk[r];
    const uint32_t lo = lo_of(r), n = lo_of(r + 1) - lo;
    t->mains.push_back(cl->shared_device ? cl->eng[0]->stream : cl->eng[r]->stream);
    if (int rc = client_block_make(cl->kind, cfg, cl->dev[r], lo, n, &k.b)) return fail(rc);
    k.req = k.b.req; k.out = k.b.resp;
    cudaError_t ce = cudaSetDevice(cl->dev[r]);
    if (ce == cudaSuccess) ce = cudaMalloc(&k.acc, 16 * sizeof(uint32_t));
    if (ce == cudaSuccess) ce = cudaMemset(k.acc, 0, 16 * sizeof(uint32_t));
    if (ce == cudaSuccess) ce = k.pub_alloc();
    if (ce != cudaSuccess) return fail(set_err(DINT_ENOMEM, "cluster client state", ce));
    k.pub[0] = n;                                      // (log_server rounds are not counted: their size is the block's)
    if (ce == cudaSuccess) ce = k.pub_map(&k.pub_dev);
    if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
    if (ce != cudaSuccess) return fail(set_err(DINT_EIO, "cluster client setup", ce));
  }
  if (cudaError_t ce = t->make_timers()) return fail(set_err(DINT_EIO, "cluster client events", ce));
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
  // each client moves with its pending request and its last reply
  int rc = round_rebind<8>(t, n, [&](const ClusterClientRank& f, int f_dev, const ClusterClientRank& to, int to_dev, uint64_t lo,
                                     uint64_t hi) { return client_block_copy(t->kind, f.b, f_dev, to.b, to_dev, (uint32_t)lo, (uint32_t)(hi - lo)); },
                           dint_cluster_clients_destroy);
  if (rc) return rc;
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
