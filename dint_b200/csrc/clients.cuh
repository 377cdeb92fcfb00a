// clients.cuh -- the closed-loop clients of the lock_fasst, lock_2pl, store and log_server servers ON the GPU
// (SURVEY.md section 8(f) rank 2).
//
// The reference's clients are Caladan uthreads on other machines (lock_fasst/caladan/client.cc:183-280,
// lock_2pl/caladan/client.cc:181-230, store/caladan/client_udp.cc:135-208, log_server/caladan/trace_init.sh).
// workloads.cc restates them as round-based state machines on host cores (one request outstanding per client and
// round); these are the same state machines, decision for decision and draw for draw (same per-client xorshift64*
// stream, same store LCG), as ONE kernel per round: a thread absorbs its client's reply of round r and emits the
// request of round r + 1 straight into the engine's device request buffer.  With it "committed txn/s" and the abort
// rate are produced live, for as long as one likes, instead of replayed from a host-recorded trace.  Parity:
// tests/test_gpu_clients.py (lock_fasst) and tests/test_gpu_clients_kinds.py (the others) compare every round's
// request stream and the final counters with workloads.cc driving the oracle.
//
// Lock kinds (k_clients_init / k_clients_step, templated on the kind): state layout (structure of arrays; a round
// touches a header word, one key and, for lock_fasst, one version per client):
//   hdr[c]    u64  {phase:8, pos:8, nr:8, nw:8, lim:8, wmask:16}    wmask bit i = rk[i] is also written (lock_2pl:
//                                                                    locked exclusive)
//   rng[c]    u64  xorshift64* state
//   rk[i][c]  u32  read set, ascending (i < nr)          rv[i][c]  u32  version read for rk[i] (lock_fasst only)
// store / log_server (k_store_clients / k_log_clients): one request is one transaction; the only state is the draw
// stream (rng[c], or the reference's LCG lcg[c] for the REF store family).
// Against a shard cluster (dint_cluster_clients_*) each rank holds a contiguous block of the clients, offset by id0, and
// k_clients_owner_count tells the host how many of the rank's records each shard owns before the round is exchanged.
#pragma once
#include "common.cuh"
#include "engine.cuh"
#include "kernels.cuh"

namespace dint {

// the phases of workloads.cc (PH_*), same numbering
enum : uint32_t { CPH_READ = 0, CPH_ACQ, CPH_VALIDATE, CPH_ABORT, CPH_COMMIT, CPH_RELEASE, CPH_REL_ABORT };

struct ClientCtx {
  uint32_t n_clients, n_keys, read_pct, zipf_n;     // zipf_n != 0: keys are Zipf ranks, cdf[zipf_n]
  uint32_t set_pct, subscribers, store_hot;         // store: percent of kSet, kSubscriberNum, HOT family
  uint32_t id0;                                     // global id of client 0 of this block (0 on one engine; a cluster
                                                    // rank's first client): seeds the draw streams, never indexes state
  const double* cdf;
  unsigned long long* hdr;                          // lock kinds
  unsigned long long* rng;                          // lock kinds, log_server, HOT store
  unsigned long long* lcg;                          // REF store
  uint32_t* rk;                                     // [10][n_clients]
  uint32_t* rv;                                     // [10][n_clients], lock_fasst
  unsigned long long* stats;                        // [0] requests [1] committed [2] validation aborts [3] lock rejects [4] rounds
                                                    // [5] not-exist replies
};

#ifdef __CUDACC__
struct CRng {                                       // workloads.cc Rng
  unsigned long long s;
  DINT_D unsigned long long next() {
    s ^= s >> 12; s ^= s << 25; s ^= s >> 27;
    return s * 0x2545F4914F6CDD1DULL;
  }
  DINT_D uint32_t below(uint32_t n) { return (uint32_t)(((next() >> 32) * (unsigned long long)n) >> 32); }
  DINT_D double unit() { return (double)(next() >> 11) * (1.0 / 9007199254740992.0); }
};
DINT_HD unsigned long long crng_seed(unsigned long long seed) {
  unsigned long long z = seed + 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return (z ^ (z >> 31)) | 1;
}
// client id's stream (workloads.cc dint_wl_create)
DINT_D CRng client_rng(unsigned long long seed, uint32_t id) { return CRng{crng_seed(seed * 0x100000001B3ULL + id)}; }

struct CHdr { uint32_t phase, pos, nr, nw, lim, wmask; };
DINT_D CHdr chdr_unpack(unsigned long long h) {
  return CHdr{(uint32_t)(h & 255u), (uint32_t)(h >> 8) & 255u, (uint32_t)(h >> 16) & 255u, (uint32_t)(h >> 24) & 255u,
              (uint32_t)(h >> 32) & 255u, (uint32_t)(h >> 40) & 0xffffu};
}
DINT_D unsigned long long chdr_pack(const CHdr& h) {
  return (unsigned long long)h.phase | ((unsigned long long)h.pos << 8) | ((unsigned long long)h.nr << 16) |
         ((unsigned long long)h.nw << 24) | ((unsigned long long)h.lim << 32) | ((unsigned long long)h.wmask << 40);
}
// index into rk[] of the k-th written key
DINT_D uint32_t nth_set_bit(uint32_t mask, uint32_t k) {
  for (uint32_t i = 0; i < k; i++) mask &= mask - 1;
  return (uint32_t)__ffs((int)mask) - 1;
}

DINT_D uint32_t client_draw_key(const ClientCtx& c, CRng& r) {
  if (!c.zipf_n) return r.below(c.n_keys);
  const double u = r.unit();                        // std::lower_bound over the cdf
  uint32_t lo = 0, hi = c.zipf_n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (c.cdf[mid] < u) lo = mid + 1; else hi = mid;
  }
  return lo < c.zipf_n - 1 ? lo : c.zipf_n - 1;
}

// lock_fasst/caladan/trace_init.sh:12-24 and lock_2pl/caladan/trace_init.sh:9-24 through workloads.cc new_txn():
// 5-10 distinct ids, sorted, each also written (lock_2pl: locked exclusive) with probability 1 - read_pct
DINT_D void client_new_txn(const ClientCtx& c, uint32_t id, CRng& r, CHdr& h) {
  uint32_t want = 5 + r.below(6);
  if (want > c.n_keys) want = c.n_keys;
  uint32_t k[10];
  uint32_t n = 0;
  while (n < want) {
    const uint32_t x = client_draw_key(c, r);
    bool dup = false;
    for (uint32_t i = 0; i < n; i++) dup |= (k[i] == x);
    if (!dup) k[n++] = x;
  }
  for (uint32_t i = 1; i < n; i++) {                // insertion sort (n <= 10)
    const uint32_t x = k[i];
    uint32_t j = i;
    while (j > 0 && k[j - 1] > x) { k[j] = k[j - 1]; j--; }
    k[j] = x;
  }
  uint32_t wmask = 0, nw = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (r.below(100) >= c.read_pct) { wmask |= 1u << i; nw++; }
    c.rk[(size_t)i * c.n_clients + id] = k[i];
  }
  h.nr = n; h.nw = nw; h.wmask = wmask; h.pos = 0; h.phase = CPH_READ; h.lim = 0;
}

// one lock request of client id: lock_fasst {type@0, lid@1, ver@5 = 0} (9 B), lock_2pl {action@0, lid@1, type@5} (6 B)
template <int KIND>
DINT_D void lock_emit(uint8_t* req, uint32_t id, uint32_t t, uint32_t lid, uint32_t b5) {
  if constexpr (KIND == K_FASST) {
    uint8_t* m = req + (size_t)id * 9;
    m[0] = (uint8_t)t;
    st_u32_unaligned(m + 1, lid);
    st_u32_unaligned(m + 5, 0u);
  } else {                                          // 6-byte records are 2-byte aligned: three u16 stores
    uint16_t* m = (uint16_t*)(req + (size_t)id * 6);
    m[0] = (uint16_t)(t | (lid << 8));
    m[1] = (uint16_t)(lid >> 8);
    m[2] = (uint16_t)((lid >> 24) | (b5 << 8));
  }
}

// a new transaction and its first request: lock_fasst reads rk[0], lock_2pl (no read phase) acquires it
template <int KIND>
DINT_D void client_start_txn(const ClientCtx& c, uint32_t id, CRng& r, uint8_t* req) {
  CHdr h{};
  client_new_txn(c, id, r, h);
  if constexpr (KIND == K_LOCK2PL) h.phase = CPH_ACQ;
  c.hdr[id] = chdr_pack(h);
  lock_emit<KIND>(req, id, 0u, c.rk[id], h.wmask & 1u);
}

// first round: every client starts a transaction and emits its first request
template <int KIND>
__global__ void __launch_bounds__(256) k_clients_init(const ClientCtx c, unsigned long long seed, uint8_t* req) {
  const uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= c.n_clients) return;
  CRng r = client_rng(seed, c.id0 + id);
  client_start_txn<KIND>(c, id, r, req);
  c.rng[id] = r.s;
}

// one round: absorb the reply (workloads.cc absorb(): lock_fasst/caladan/client.cc:183-280,
// lock_2pl/caladan/client.cc:181-230), emit the next request
template <int KIND>
__global__ void __launch_bounds__(256) k_clients_step(const ClientCtx c, const uint8_t* resp, uint8_t* req) {
  constexpr uint32_t MSG = KIND == K_FASST ? 9 : 6;
  const uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t committed = 0, vaborts = 0, rejects = 0;
  __shared__ uint32_t s_list[256];
  __shared__ uint32_t s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  if (id < c.n_clients) {
    CHdr h = chdr_unpack(c.hdr[id]);
    const uint8_t* a = resp + (size_t)id * MSG;
    bool fresh = false;
    if constexpr (KIND == K_FASST) {
      const uint32_t type = a[0], ver = ld_u32_unaligned(a + 5);
      switch (h.phase) {
        case CPH_READ:
          c.rv[(size_t)h.pos * c.n_clients + id] = ver;
          if (++h.pos == h.nr) { h.pos = 0; h.phase = h.nw ? CPH_ACQ : CPH_VALIDATE; }
          break;
        case CPH_ACQ:
          if (type == 5) {                                      // kGrantLock
            if (++h.pos == h.nw) { h.pos = 0; h.phase = CPH_VALIDATE; }
          } else {                                              // kRejectLock: abort the locks taken so far, restart
            rejects = 1;
            if (h.pos) { h.lim = h.pos; h.pos = 0; h.phase = CPH_ABORT; }
            else { h.pos = 0; h.phase = CPH_READ; }
          }
          break;
        case CPH_VALIDATE:
          if (ver != c.rv[(size_t)h.pos * c.n_clients + id]) {  // client.cc:209-212 roll back
            vaborts = 1;
            if (h.nw) { h.lim = h.nw; h.pos = 0; h.phase = CPH_ABORT; }
            else { h.pos = 0; h.phase = CPH_READ; }
          } else if (++h.pos == h.nr) {
            if (h.nw) { h.pos = 0; h.phase = CPH_COMMIT; }
            else { committed = 1; fresh = true; }
          }
          break;
        case CPH_ABORT:
          if (++h.pos == h.lim) { h.pos = 0; h.phase = CPH_READ; }
          break;
        default:                                                // CPH_COMMIT
          if (++h.pos == h.nw) { committed = 1; fresh = true; }
          break;
      }
    } else {                                                    // lock_2pl
      switch (h.phase) {
        case CPH_ACQ:
          if (a[0] == 2) {                                      // kGrantLock: after the last grant, release in reverse
            if (++h.pos == h.nr) { h.pos = h.nr - 1; h.phase = CPH_RELEASE; }
          } else {                                              // kRejectLock: release [0, pos) ascending, retry
            rejects = 1;
            if (h.pos) { h.lim = h.pos; h.pos = 0; h.phase = CPH_REL_ABORT; }
          }
          break;
        case CPH_RELEASE:
          if (h.pos == 0) { committed = 1; fresh = true; }
          else h.pos--;
          break;
        default:                                                // CPH_REL_ABORT
          if (++h.pos == h.lim) { h.pos = 0; h.phase = CPH_ACQ; }
          break;
      }
    }
    if (fresh) {                                          // (new transactions are drawn below, by converged warps)
      s_list[atomicAdd(&s_cnt, 1u)] = id;
    } else {
      c.hdr[id] = chdr_pack(h);
      // ---- emit (workloads.cc emit()) ----
      uint32_t t, lid, b5 = 0;
      if constexpr (KIND == K_FASST) {
        if (h.phase == CPH_READ || h.phase == CPH_VALIDATE) { t = 0; lid = c.rk[(size_t)h.pos * c.n_clients + id]; }
        else {
          t = h.phase == CPH_ACQ ? 1u : h.phase == CPH_ABORT ? 2u : 3u;
          lid = c.rk[(size_t)nth_set_bit(h.wmask, h.pos) * c.n_clients + id];
        }
      } else {                                            // acquire in CPH_ACQ, release otherwise; b5 = lock type
        t = h.phase == CPH_ACQ ? 0u : 1u;
        lid = c.rk[(size_t)h.pos * c.n_clients + id];
        b5 = (h.wmask >> h.pos) & 1u;
      }
      lock_emit<KIND>(req, id, t, lid, b5);
    }
  }
  // ---- clients that finished a transaction (about 1 in 25 per round) start the next one: drawing 5-10 distinct keys,
  //      sorting them and choosing the write set is ~600 instructions, so the few clients of a CTA that need it are
  //      compacted into its first warps instead of dragging every warp through the divergent path ----
  __syncthreads();
  if (threadIdx.x < s_cnt) {
    const uint32_t id2 = s_list[threadIdx.x];
    CRng r{c.rng[id2]};
    client_start_txn<KIND>(c, id2, r, req);
    c.rng[id2] = r.s;
  }
  // counters: one atomic per warp and counter
  const uint32_t all = 0xffffffffu;
  const uint32_t nc = __popc(__ballot_sync(all, committed)), nv = __popc(__ballot_sync(all, vaborts)), nj = __popc(__ballot_sync(all, rejects));
  if ((threadIdx.x & 31) == 0) {
    if (nc) atomicAdd(&c.stats[1], (unsigned long long)nc);
    if (nv) atomicAdd(&c.stats[2], (unsigned long long)nv);
    if (nj) atomicAdd(&c.stats[3], (unsigned long long)nj);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { atomicAdd(&c.stats[0], (unsigned long long)c.n_clients); atomicAdd(&c.stats[4], 1ULL); }
}

// ---- store and log_server: 53-byte records {type@0, key@1, val@9, ver@49} ------------------------------------------
// A CTA of 256 clients owns a 16-byte-aligned slice of 256 x 53 = 13,568 bytes of the request buffer: its threads
// assemble their records in shared memory and the CTA stores the slice with 16-byte stores.
constexpr uint32_t kKvMsg = 53;
constexpr uint32_t kKvSlice = 256 * kKvMsg;
static_assert(kKvSlice % 16 == 0, "a CTA's slice must be 16-byte aligned");

// record {type, payload} into shared memory at s; p[] = the 52 payload bytes (key, val, ver) as little-endian words
DINT_D void kv_stage(uint8_t* s, uint32_t type, const uint32_t (&p)[13]) {
  uint32_t w[13];                                   // record word i = payload bytes 4i-1 .. 4i+2
  w[0] = type | (p[0] << 8);
#pragma unroll
  for (int i = 1; i < 13; i++) w[i] = __funnelshift_l(p[i - 1], p[i], 8);
  st_words_unaligned<13>(s, w);
  s[52] = (uint8_t)(p[12] >> 24);
}

// the CTA's staged records -> its slice of the request buffer (the tail CTA's slice may end in < 16 loose bytes)
DINT_D void kv_flush(const uint8_t* s, uint8_t* req, uint32_t n_clients) {
  const uint32_t first = blockIdx.x * 256, n = n_clients - first < 256 ? n_clients - first : 256;
  const uint32_t bytes = n * kKvMsg, n16 = bytes / 16;
  uint8_t* g = req + (size_t)blockIdx.x * kKvSlice;
  for (uint32_t i = threadIdx.x; i < n16; i += blockDim.x) ((uint4*)g)[i] = ((const uint4*)s)[i];
  for (uint32_t i = n16 * 16 + threadIdx.x; i < bytes; i += blockDim.x) g[i] = s[i];
}

// store/caladan/client_udp.cc:135-147 (store/udp/tatp.h:31-42): the reference's LCG
DINT_D uint32_t store_fastrand(unsigned long long& l) { l = l * 1103515245ULL + 12345ULL; return (uint32_t)(l >> 32); }

// store (workloads.cc emit() / absorb(), store/caladan/client_udp.cc:135-171,199-208): first = the clients' first
// round (seed the streams, nothing to absorb); otherwise absorb the reply (type 7 = not found) and draw the next request
__global__ void __launch_bounds__(256) k_store_clients(const ClientCtx c, unsigned long long seed, uint32_t first,
                                                       const uint8_t* resp, uint8_t* req) {
  __shared__ __align__(16) uint8_t s_rec[kKvSlice];
  const uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t committed = 0, missing = 0;
  if (id < c.n_clients) {
    if (!first) { if (resp[(size_t)id * kKvMsg] == 7) missing = 1; else committed = 1; }
    bool is_set;
    uint32_t s_id, sf, st, end_time = 0;
    if (c.store_hot) {                              // HOT: the first n_keys of the population, xorshift + Zipf
      CRng r = first ? client_rng(seed, c.id0 + id) : CRng{c.rng[id]};
      is_set = r.below(100) < c.set_pct;
      const uint32_t k = client_draw_key(c, r);
      s_id = k / 12; sf = (k % 12) / 3 + 1; st = (k % 3) * 8;
      end_time = r.below(24);
      c.rng[id] = r.s;
    } else {                                        // REF: lcg = 0xdeadbeef + client index (client_udp.cc:201)
      unsigned long long l = first ? 0xdeadbeefULL + c.id0 + id : c.lcg[id];
      is_set = store_fastrand(l) % 100 >= 100 - c.set_pct;   // workgen_arr: reads first, sets last
      const uint32_t x = store_fastrand(l), y = store_fastrand(l);
      s_id = ((x % c.subscribers) | (y & 1048575u)) % c.subscribers;   // NURand
      sf = store_fastrand(l) % 4 + 1;
      st = (store_fastrand(l) % 3) * 8;
      if (is_set) end_time = store_fastrand(l) % 24;
      c.lcg[id] = l;
    }
    uint32_t p[13] = {};
    p[0] = s_id; p[1] = sf | (st << 8);             // key = s_id | sf << 32 | start_time << 40
    if (is_set) p[2] = end_time | (0x5au << 8);     // kSet: val[0] = end_time, val[1] = 0x5a
    kv_stage(s_rec + threadIdx.x * kKvMsg, is_set ? 1u : 0u, p);
  }
  __syncthreads();
  kv_flush(s_rec, req, c.n_clients);
  const uint32_t all = 0xffffffffu;
  const uint32_t nc = __popc(__ballot_sync(all, committed)), nm = __popc(__ballot_sync(all, missing));
  if ((threadIdx.x & 31) == 0) {
    if (nc) atomicAdd(&c.stats[1], (unsigned long long)nc);
    if (nm) atomicAdd(&c.stats[5], (unsigned long long)nm);
  }
  if (!first && blockIdx.x == 0 && threadIdx.x == 0) { atomicAdd(&c.stats[0], (unsigned long long)c.n_clients); atomicAdd(&c.stats[4], 1ULL); }
}

// log_server (log_server/caladan/trace_init.sh:15-19 through workloads.cc emit()): key U[0, 7009999], 40 random value
// bytes, ver U[0, 127]; every reply counts as committed, so the replies are not read
__global__ void __launch_bounds__(256) k_log_clients(const ClientCtx c, unsigned long long seed, uint32_t first, uint8_t* req) {
  __shared__ __align__(16) uint8_t s_rec[kKvSlice];
  const uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id < c.n_clients) {
    CRng r = first ? client_rng(seed, c.id0 + id) : CRng{c.rng[id]};
    uint32_t p[13];
    p[0] = r.below(7010000); p[1] = 0;
#pragma unroll
    for (int i = 0; i < 5; i++) { const unsigned long long v = r.next(); p[2 + 2 * i] = (uint32_t)v; p[3 + 2 * i] = (uint32_t)(v >> 32); }
    p[12] = r.below(128);
    c.rng[id] = r.s;
    kv_stage(s_rec + threadIdx.x * kKvMsg, 0u, p);
  }
  __syncthreads();
  kv_flush(s_rec, req, c.n_clients);
  if (!first && blockIdx.x == 0 && threadIdx.x == 0) {
    atomicAdd(&c.stats[0], (unsigned long long)c.n_clients);
    atomicAdd(&c.stats[1], (unsigned long long)c.n_clients);
    atomicAdd(&c.stats[4], 1ULL);
  }
}

// ---- a cluster rank's round, counted per owner shard (dint_cluster_clients_*) ----------------------------------------
// route_owner_of is what k_route_dispatch computes, so the counts are exact.  Every CTA adds its counts to acc[0, 8); the
// last CTA to finish (ticket acc[8]) publishes them to the mapped pinned block pub -- [0] records, [1 + o] records for
// shard o, the layout of the txn clients' -- and resets acc for the next round.
template <int KIND>
__global__ void __launch_bounds__(kThreads) k_clients_owner_count(const Ctx c, const uint8_t* req, uint32_t n, uint32_t* acc,
                                                                  uint32_t* pub) {
  __shared__ uint32_t s_cnt[kMaxShards];
  __shared__ bool s_last;
  if (threadIdx.x < kMaxShards) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t i = blockIdx.x * kThreads + threadIdx.x;
  const uint32_t o = i < n ? route_owner_of<KIND>(c, req + (size_t)i * Wire<KIND>::MSG) : 0xffu;
  const uint32_t peers = __match_any_sync(0xffffffffu, o);
  if (o < kMaxShards && (int)lane_id() == __ffs(peers) - 1) atomicAdd(&s_cnt[o], (uint32_t)__popc(peers));
  __syncthreads();
  if (threadIdx.x < kMaxShards && s_cnt[threadIdx.x]) atomicAdd(&acc[threadIdx.x], s_cnt[threadIdx.x]);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(&acc[kMaxShards], 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (threadIdx.x == 0) pub[0] = n;
  if (threadIdx.x < kMaxShards) {
    pub[1 + threadIdx.x] = ((volatile uint32_t*)acc)[threadIdx.x];
    acc[threadIdx.x] = 0;
  }
  if (threadIdx.x == 0) acc[kMaxShards] = 0;
}
#endif  // __CUDACC__

}  // namespace dint
