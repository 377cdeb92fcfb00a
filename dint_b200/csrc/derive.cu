// derive.cu -- shards filled from other shards' state: dint_cluster_reshard / dint_cluster_reshard_txn move every row
// or lock word to its owner under a new shard count, dint_cluster_rebuild fills lost tatp / smallbank shards from their
// replicas.  reshard.cuh and rebuild.cuh hold the placement arithmetic and the gathers.
#include "host.cuh"
#include "rebuild.cuh"
#include "reshard.cuh"

extern "C" {

int dint_test_rebuild_source(uint64_t key, uint32_t G, uint32_t lost_mask) {
  return G == 0 || G > kMaxShards ? -1 : rebuild_source((uint32_t)(key % G), G, lost_mask);
}
uint32_t dint_test_txn_reshard_dests(uint64_t key, uint32_t G, uint32_t G2, uint32_t src) {
  if (G == 0 || G > kMaxShards || G2 == 0 || G2 > kMaxShards) return 0;
  return ReplicaDests{make_fastmod(G), make_fastmod(G2), G2, (1u << G2) - 1, src}(key, 0);
}

}  // extern "C"

// ---- shards derived from other shards' state (dint_cluster_reshard, dint_cluster_rebuild) ---------------------------
static thread_local double g_reshard_times[3];       // dint_reshard_times: wall, re-shard kernels, count + allocation (s)
thread_local double g_rebuild_times[3];              // dint_rebuild_times: wall, rebuild kernels, count + allocation (s)

// lets `device` (the current device) read `peer`'s memory; nothing to do when they are the same
int peer_enable(int device, int peer) {
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
int cluster_quiesce(const dint_cluster* cl) {
  for (uint32_t r = 0; r < cl->G; r++) {
    CU(cudaSetDevice(cl->dev[r]));
    CU(cudaDeviceSynchronize());
  }
  return DINT_OK;
}

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
// times[1] += the fill's CUDA-event time; times[2] += the sizing, allocation and peer set-up.  `what` names the
// operation in a refusal.
template <class Fill>
static int derive_engine(int kind, dint_cfg c, int device, uint32_t j, const uint64_t* rows, const std::vector<dint_engine*>& read,
                         double* times, const char* what, Fill fill, dint_engine** out) {
  *out = nullptr;
  const double t0 = now_s();
  if (kind == DINT_STORE || kind == DINT_TATP || kind == DINT_SMALLBANK) {
    KvPlan P;
    if (kv_plan(kind, c, false, P) != DINT_OK) return set_err(DINT_EINVAL, "bad KV configuration");
    for (uint32_t t = 0; t < P.nt; t++) {
      const uint32_t lg = kv_fit_log2(P.lg[t], rows[t]);
      if (lg > 34)
        return kind == DINT_STORE ? set_errf(DINT_EINVAL, "re-shard: shard %u would receive %llu keys", j, (unsigned long long)rows[t])
                                  : set_errf(DINT_EINVAL, "%s: shard %u table %u would receive %llu rows",
                                             what, j, t, (unsigned long long)rows[t]);
      c.kv_capacity_log2[t] = lg;
    }
  }
  dint_engine* e = nullptr;
  { int rc = dint_create(kind, &c, device, &e); if (rc) return rc; }
  EngineOwner own{e};
  for (const dint_engine* s : read)                    // the fill reads the sources' arrays where they are
    if (s) { int rc = peer_enable(device, s->device); if (rc) return rc; }
  times[2] += now_s() - t0;
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
int reshard_engine(const DeriveFrom& f, uint32_t j, uint32_t G2, int kind, const dint_cfg& c, int device, dint_engine** out) {
  const uint32_t G = (uint32_t)f.src.size();
  return derive_engine(kind, c, device, j, f.rows[j], f.src, g_reshard_times, "re-shard", [&](dint_engine* e) {
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
std::string mask_names(uint32_t mask) {
  std::string s;
  for (uint32_t r = 0; r < 32; r++)
    if ((mask >> r) & 1u) s += (s.empty() ? "" : ", ") + std::to_string(r);
  return "{" + s + "}";
}

// DINT_EINVAL, with the reason, unless the shards of `lost` of a G-shard cluster of this kind and configuration can be
// rebuilt from the others
static const char kEbpfRows[] = "the eBPF cache tiers hold dirty and cache-only rows whose wire-visible versions depend on "
                                "each shard's own hit history";
int rebuild_check(int kind, const dint_cfg& cfg, uint32_t G, uint32_t lost) {
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
  return derive_engine(kind, c, device, j, f.rows[j], read, g_rebuild_times, "rebuild", [&](dint_engine* e) {
    for (uint32_t s = 0; s < f.G; s++) {
      if (!read[s]) continue;
      for (uint32_t t = 0; t < e->ctx.n_tables; t++) {
        if (kind == DINT_SMALLBANK) k_kv_move<8><<<e->sms * 8, 256, 0, e->stream>>>(read[s]->ctx.tbl[t], e->ctx.tbl[t], f.keep(s, j));
        else k_kv_move<40><<<e->sms * 8, 256, 0, e->stream>>>(read[s]->ctx.tbl[t], e->ctx.tbl[t], f.keep(s, j));
      }
    }
  }, out);
}

// The shards of `lost` of a cluster being made, whose engines are null, filled from the others (cluster_make)
int rebuild_shards(dint_cluster* cl, uint32_t lost) {
  RebuildFrom f(cl->eng, cl->G, lost);
  int rc = f.count();
  for (uint32_t r = 0; r < cl->G && rc == DINT_OK; r++)
    if ((lost >> r) & 1u) rc = rebuild_engine(f, r, cl->kind, cluster_shard_cfg(cl, r), cl->dev[r], &cl->eng[r]);
  return rc;
}

extern "C" {

int dint_cluster_rebuild(dint_cluster* cl, uint32_t lost_mask) {
  if (!cl) return set_err(DINT_EINVAL, "null argument");
  { int rc = rebuild_check(cl->kind, cl->base, cl->G, lost_mask); if (rc) return rc; }
  if (cl->txn_clients)
    return set_errf(DINT_EINVAL, "rebuild: %u dint_txn_clients are attached; clients mid-transaction hold locks the rebuilt "
                                 "shards do not, so destroy them first", cl->txn_clients);
  for (double& t : g_rebuild_times) t = 0;
  const double t0 = now_s();
  { int rc = cluster_quiesce(cl); if (rc) return rc; }
  const uint32_t G = cl->G;
  RebuildFrom f(cl->eng, G, lost_mask);
  { int rc = f.count(); if (rc) return rc; }
  g_rebuild_times[2] += now_s() - t0;
  // the new engines and rank contexts are made next to the old ones, so a failure leaves the cluster as it was
  std::vector<dint_engine*> eng = cl->eng;
  std::vector<dint_shard_ctx*> sh;
  auto fail = [&](int code) {
    return keep_error(code, [&] {
      for (auto* c : sh) dint_shard_destroy(c);
      for (uint32_t r = 0; r < G; r++) {
        if (eng[r] != cl->eng[r]) dint_destroy(eng[r]);
        cl->eng[r]->plain_launches = true;             // (dint_shard_destroy cleared it; the old contexts stay)
      }
    });
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
  g_rebuild_times[0] = now_s() - t0;
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
  const double t0 = now_s();
  { int rc = cluster_quiesce(src); if (rc) return rc; }   // as dint_snapshot_create quiesces an engine
  DeriveFrom f;
  f.src = src->eng;
  const uint32_t G2 = (uint32_t)n_gpus;
  { int rc = count_rows(f, f.src, [&](uint32_t, const KvTable& t) { return OwnerDests{t.lock_mod, G2, (1u << G2) - 1}; }, "re-shard key count"); if (rc) return rc; }
  g_reshard_times[2] += now_s() - t0;
  const int rc = cluster_make(src->kind, &src->base, n_gpus, devices, max_batch, nullptr, &f, nullptr, out);
  g_reshard_times[0] = now_s() - t0;
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
  const double t0 = now_s();
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
  g_reshard_times[2] += now_s() - t0;
  const int rc = cluster_make(src->kind, &src->base, n_gpus, devices, max_batch, nullptr, &f, nullptr, out);
  g_reshard_times[0] = now_s() - t0;
  return rc;
}

int dint_reshard_times(double out[3]) {
  if (!out) return set_err(DINT_EINVAL, "null argument");
  for (int i = 0; i < 3; i++) out[i] = g_reshard_times[i];
  return DINT_OK;
}

}  // extern "C"
