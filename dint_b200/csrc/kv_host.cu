// kv_host.cu -- the host side of the KV tables, lock state and log of one engine: dint_load / dint_populate (through the
// eBPF cache tiers where an engine has one), dint_kv_get / dint_kv_count, the cache-set and chain inspection of the tiers,
// dint_lock_* and dint_dump_log.
#include <algorithm>

#include "host.cuh"

namespace dint {

// valid slots of table `table`'s chain entries (dint_kv_count with the eBPF tier): freed entries hold none
__global__ void __launch_bounds__(256) k_tchain_count(const Ctx c, uint32_t table, uint32_t n, unsigned long long* out) {
  uint32_t cnt = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint8_t* p = c.tpool + (size_t)i * kTeEntBytes;
    if (__ldcg((const uint32_t*)(p + 56)) == table) cnt += __popc(__ldcg((const uint32_t*)(p + 48)) & 15u);
  }
  if (cnt) atomicAdd(out, (unsigned long long)cnt);
}

// The eBPF SmallBank client's warm-up stream (smallbank/caladan/client_ebpf_shard.cc:88-169) as one shard sees it:
// record j (from `first`) is kWarmupRead of table j % 2 for the (j / 2)-th account the shard replicates, ascending --
// account (i / per) * blk + res[i % per]: every account (per = blk = 1, res = {0}), or with G = txn_shards > 3 the
// accounts whose a % G is one of the three residues res (per = 3, blk = G).
__global__ void __launch_bounds__(256) k_sbe_warmup(uint8_t* out, uint64_t first, uint32_t n, uint32_t per, uint32_t blk, uint4 res) {
  using W = Wire<K_SMALLBANK_EBPF>;
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint64_t i = (first + j) >> 1;
  const uint32_t r = (uint32_t)(i % per);
  const uint64_t a = i / per * blk + (r == 0 ? res.x : r == 1 ? res.y : res.z);
  uint8_t* p = out + (size_t)j * W::MSG;
  p[0] = 0;
  p[W::TYPE] = 17;
  p[W::TABLE] = (uint8_t)((first + j) & 1);
#pragma unroll
  for (int k = 0; k < 8; k++) p[W::KEY + k] = (uint8_t)(a >> (8 * k));
#pragma unroll
  for (int k = W::VAL; k < W::MSG; k++) p[k] = 0;
}

}  // namespace dint

static void kv_launch_load(int kind, const Ctx& c, int table, const uint64_t* dk, const uint8_t* dv, uint32_t n, cudaStream_t s) {
  if (n == 0) return;
  uint32_t blocks = (n + 255) / 256;
  if (kind == DINT_SMALLBANK) k_kv_load<8><<<blocks, 256, 0, s>>>(c, table, dk, dv, n);
  else k_kv_load<40><<<blocks, 256, 0, s>>>(c, table, dk, dv, n);
}

static int kv_host_get(const Ctx& c, int table, uint64_t key, uint32_t valsz, void* val, uint32_t* ver) {
  uint32_t* d = nullptr;
  if (cudaMalloc(&d, 64) != cudaSuccess) return DINT_ENOMEM;
  if (valsz == 8) k_kv_get1<8><<<1, 1>>>(c, table, key, d);
  else k_kv_get1<40><<<1, 1>>>(c, table, key, d);
  uint32_t h[12] = {0};
  cudaError_t ce = cudaMemcpy(h, d, sizeof h, cudaMemcpyDeviceToHost);
  cudaFree(d);
  if (ce != cudaSuccess) return DINT_EIO;
  if (!h[0]) return 1;
  if (ver) *ver = h[1];
  if (val) memcpy(val, &h[2], valsz);
  return 0;
}

extern "C" {

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
