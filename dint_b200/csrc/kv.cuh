// kv.cuh -- the KV side of the hot path: the HBM-resident table that stands in for the reference's
// chained `kvs` (store/udp/kvs.h:13-136; tatp/udp/kvs.h and smallbank/udp/kvs.h are the same code with
// panics on missing keys), and the request semantics of the three servers built on it
// (store/udp/server.cc:75-97, tatp/udp/server_shard.cc:113-210, smallbank/udp/server_shard.cc:107-189).
//
// Layout.  The wire-visible behaviour of `kvs` is the map key -> (val, ver, exists); the reference's
// physical layout (bucket-head pointer array -> 224-byte 4-slot entries -> next pointers) costs two
// dependent DRAM misses per lookup.  Here a table is ONE open-addressing array of naturally aligned
// 64-byte entries (32-byte for smallbank's 8-byte values) at a load factor <= 0.5, so a GET that hits
// on its first probe is exactly one aligned 64-byte HBM access:
//     { u64 key; u32 ver; u32 meta; u8 val[VALSZ]; pad }
// meta: EMPTY (never used) / FULL / TOMB (deleted) / BUSY (insert in flight).  Entries never return to
// EMPTY inside a launch, so a probe sequence that reaches EMPTY proves absence.  Deletes leave tombstones
// (an insert reuses the first one on its probe path); the engine counts the entries that have left EMPTY
// (`live[1]`) and, between calls, rehashes a table into a fresh array once FULL + TOMB passes 70 % of its
// capacity (k_kv_move, engine.cu kv_maintain) -- the reference's chained kvs frees entries on delete
// (store/udp/kvs.h:124-133), so without this a long insert/delete churn would grow the probe chains without
// bound.  Requests on the same key are never
// concurrent (same group -> K3 replays them in one thread); requests on different keys only meet on
// the `meta` word, which is claimed with atomicCAS.
#pragma once
#include <functional>
#include "engine.cuh"
#ifdef __CUDACC__
#include <cooperative_groups.h>
#include "kernels.cuh"
#endif

namespace dint {

template <int VALSZ> struct Ent {
  static constexpr int BYTES = (VALSZ == 40) ? 64 : 32;
  static constexpr int NW = VALSZ / 4;          // value words
  static constexpr int NV = BYTES / 16;         // 16-byte vectors per entry
};
constexpr uint64_t kKvMix = 0x9E3779B97F4A7C15ULL;

#ifdef __CUDACC__
DINT_D uint64_t kv_home(const KvTable& t, uint64_t h) { return (h * kKvMix) >> (64 - t.cap_log2); }

template <int VALSZ>
DINT_D void kv_load_entry(const uint8_t* e, uint4 (&v)[Ent<VALSZ>::NV]) {
#pragma unroll
  for (int k = 0; k < Ent<VALSZ>::NV; k++) v[k] = __ldcg((const uint4*)e + k);   // one aligned entry, L1 bypass
}

// Probe for `key`.  `v` arrives holding the HOME entry (fetched by prefetch()); on a hit returns the
// entry and leaves its 16-byte vectors in `v` (v[0] = key lo/hi, ver, meta; v[1..] = value).
template <int VALSZ>
DINT_D uint8_t* kv_find(const KvTable& t, uint64_t key, uint64_t h, uint4 (&v)[Ent<VALSZ>::NV]) {
  uint64_t i = kv_home(t, h);
  for (uint64_t probe = 0; probe <= t.cap_mask; probe++) {
    uint8_t* e = t.entries + (i << t.ent_shift);
    if (probe) kv_load_entry<VALSZ>(e, v);
    uint32_t meta = v[0].w;
    if (meta == ENT_EMPTY) return nullptr;
    if (meta == ENT_FULL && v[0].x == (uint32_t)key && v[0].y == (uint32_t)(key >> 32)) return e;
    i = (i + 1) & t.cap_mask;
  }
  return nullptr;
}

// kvs_get (kvs.h:37-55): on a hit copy val and ver into the wire record.
template <int VALSZ>
DINT_D bool kv_get_into(const KvTable& t, uint64_t key, uint64_t h, uint4 (&v)[Ent<VALSZ>::NV], uint8_t* wire_val,
                        uint8_t* wire_ver) {
  if (!kv_find<VALSZ>(t, key, h, v)) return false;
  uint32_t w[Ent<VALSZ>::NW];
#pragma unroll
  for (int k = 0; k < Ent<VALSZ>::NW; k++) {
    const uint4& q = v[1 + k / 4];
    w[k] = (k % 4 == 0) ? q.x : (k % 4 == 1) ? q.y : (k % 4 == 2) ? q.z : q.w;
  }
  st_words_unaligned<Ent<VALSZ>::NW>(wire_val, w);
  st_u32_unaligned(wire_ver, v[0].z);
  return true;
}

template <int VALSZ>
DINT_D void kv_write_val(uint8_t* e, const uint32_t (&w)[Ent<VALSZ>::NW]) {
  if constexpr (VALSZ == 40) {
    *((uint4*)(e + 16)) = make_uint4(w[0], w[1], w[2], w[3]);
    *((uint4*)(e + 32)) = make_uint4(w[4], w[5], w[6], w[7]);
    *((uint2*)(e + 48)) = make_uint2(w[8], w[9]);
  } else {
    *((uint2*)(e + 16)) = make_uint2(w[0], w[1]);
  }
}

// kvs_set (kvs.h:57-75): overwrite val, ver++.
template <int VALSZ>
DINT_D bool kv_set_from(const KvTable& t, uint64_t key, uint64_t h, uint4 (&v)[Ent<VALSZ>::NV], const uint8_t* wire_val) {
  uint8_t* e = kv_find<VALSZ>(t, key, h, v);
  if (!e) return false;
  uint32_t w[Ent<VALSZ>::NW];
  ld_words_unaligned<Ent<VALSZ>::NW>(wire_val, w);
  kv_write_val<VALSZ>(e, w);
  *((uint32_t*)(e + 8)) = v[0].z + 1;
  return true;
}
// kvs_set of the eBPF servers (smallbank/ebpf/kvs.h:55-74): overwrite val; ver = `ver` when non-zero, else ver + 1.
// `nv` = the new version.  Probes afresh (earlier calls of the same request may have written).
template <int VALSZ>
DINT_D bool kv_set_ver(const KvTable& t, uint64_t key, uint64_t h, const uint32_t (&w)[Ent<VALSZ>::NW], uint32_t ver,
                       uint32_t& nv) {
  uint4 v[Ent<VALSZ>::NV];
  kv_load_entry<VALSZ>(t.entries + (kv_home(t, h) << t.ent_shift), v);
  uint8_t* e = kv_find<VALSZ>(t, key, h, v);
  if (!e) return false;
  kv_write_val<VALSZ>(e, w);
  nv = ver != 0 ? ver : v[0].z + 1;
  *((uint32_t*)(e + 8)) = nv;
  return true;
}

// kvs_insert (kvs.h:77-104): take the first free entry on the probe path, ver = 0.  Like the
// reference it does not look for an existing copy of the key.
template <int VALSZ>
DINT_D bool kv_insert_words(const KvTable& t, uint64_t key, uint64_t h, const uint32_t (&w)[Ent<VALSZ>::NW], uint32_t ver0 = 0) {
  uint64_t i = kv_home(t, h);
  for (uint64_t probe = 0; probe <= t.cap_mask; probe++) {
    uint8_t* e = t.entries + (i << t.ent_shift);
    uint32_t* meta = (uint32_t*)(e + 12);
    uint32_t m = __ldcg(meta);
    while (m == ENT_EMPTY || m == ENT_TOMB) {
      uint32_t old = atomicCAS(meta, m, (uint32_t)ENT_BUSY);
      if (old == m) {
        *((uint64_t*)e) = key;
        *((uint32_t*)(e + 8)) = ver0;
        kv_write_val<VALSZ>(e, w);
        __threadfence();
        *((volatile uint32_t*)meta) = ENT_FULL;
        atomicAdd(t.live, 1ULL);
        if (m == ENT_EMPTY) atomicAdd(t.live + 1, 1ULL);   // one more entry that can never prove absence again
        return true;
      }
      m = old;
    }
    i = (i + 1) & t.cap_mask;
  }
  return false;    // table full
}
template <int VALSZ>
DINT_D bool kv_insert_from(const KvTable& t, uint64_t key, uint64_t h, const uint8_t* wire_val) {
  uint32_t w[Ent<VALSZ>::NW];
  ld_words_unaligned<Ent<VALSZ>::NW>(wire_val, w);
  return kv_insert_words<VALSZ>(t, key, h, w);
}

// kvs_delete (kvs.h:106-136)
template <int VALSZ>
DINT_D bool kv_delete(const KvTable& t, uint64_t key, uint64_t h, uint4 (&v)[Ent<VALSZ>::NV]) {
  uint8_t* e = kv_find<VALSZ>(t, key, h, v);
  if (!e) return false;
  *((volatile uint32_t*)(e + 12)) = ENT_TOMB;
  atomicAdd(t.live, (unsigned long long)-1LL);
  return true;
}

// group of a KV key: the reference's bucket (store) or lock_hash (tatp.h:12-14, smallbank.h:12-14)
DINT_D uint32_t kv_group(const Ctx& c, uint32_t table, uint64_t h) {
  const KvTable& t = c.tbl[table];
  uint32_t gl;
  if (!to_local_group(c, fast_mod(h, t.lock_mod), gl)) return kNoGroup;
  return t.grp_base + gl;
}
// the home entry of (table, key): the one access a first-probe hit needs
template <int VALSZ>
DINT_D void kv_prefetch_home(const Ctx& c, uint32_t table, uint64_t h, uint4 (&v)[Ent<VALSZ>::NV]) {
  const KvTable& t = c.tbl[table];
  kv_load_entry<VALSZ>(t.entries + (kv_home(t, h) << t.ent_shift), v);
}

// Warp-cooperative fetch of every lane's home entry: NV adjacent lanes read one entry with a single
// coalesced request (64 B = 4 lanes x 16 B, 32 B = 2 lanes), then the 16-byte pieces are handed to the
// owning lane with shuffles.  Must be executed by all 32 lanes; `need` = this lane wants its entry.
template <int VALSZ>
DINT_D void kv_prefetch_home_coop(const uint8_t* entry, bool need, uint4 (&v)[Ent<VALSZ>::NV]) {
  constexpr int LPE = Ent<VALSZ>::NV;        // lanes per entry
  constexpr int EPR = 32 / LPE;              // entries fetched per round
  const uint32_t lane = threadIdx.x & 31;
  const unsigned long long a = (unsigned long long)entry;
#pragma unroll
  for (int r = 0; r < LPE; r++) {
    const int src = r * EPR + (int)(lane / LPE);
    const unsigned long long sa = __shfl_sync(0xffffffffu, a, src);
    const int sneed = __shfl_sync(0xffffffffu, need ? 1 : 0, src);
    uint4 piece = make_uint4(0, 0, 0, 0);
    if (sneed) piece = __ldcg((const uint4*)sa + (lane % LPE));
#pragma unroll
    for (int k = 0; k < LPE; k++) {
      const int from = (int)(lane % EPR) * LPE + k;
      uint4 got;
      got.x = __shfl_sync(0xffffffffu, piece.x, from);
      got.y = __shfl_sync(0xffffffffu, piece.y, from);
      got.z = __shfl_sync(0xffffffffu, piece.z, from);
      got.w = __shfl_sync(0xffffffffu, piece.w, from);
      if ((int)(lane / EPR) == r) v[k] = got;
    }
  }
}
template <int VALSZ>
DINT_D const uint8_t* kv_home_ptr(const Ctx& c, uint32_t table, uint64_t h) {
  const KvTable& t = c.tbl[table];
  return t.entries + (kv_home(t, h) << t.ent_shift);
}

// =================================== store ==========================================================
template <> DINT_D TypeInfo type_info<K_STORE>(const uint8_t* rec) {
  uint8_t t = rec[Wire<K_STORE>::TYPE];
  if (t == 0) return TypeInfo{C_RA, false, false};          // kRead  store/udp/server.cc:79-84
  if (t == 1 || t == 2) return TypeInfo{C_WA, false, false};  // kSet :86-91; kInsert: the eBPF server's
                                                            // population path (store/ebpf/store_user.c)
  return TypeInfo{0, true, false};                          // :93-94
}
template <> DINT_D KeyInfo key_info<K_STORE>(const Ctx& c, const uint8_t* rec) {
  KeyInfo k;
  k.key = ld_u64_unaligned(rec + Wire<K_STORE>::KEY);
  k.h = fasthash64_u64(k.key);                              // kvs.h:33-35
  k.grp = kv_group(c, 0, k.h);
  return k;
}
template <> struct Pre<K_STORE> { uint4 v[4]; };
template <> DINT_D Pre<K_STORE> prefetch<K_STORE>(const Ctx& c, const uint8_t* rec, const KeyInfo& ki, const TypeInfo&) {
  Pre<K_STORE> p;
  if (rec[Wire<K_STORE>::TYPE] != 2) kv_prefetch_home<40>(c, 0, ki.h, p.v);
  return p;
}
template <> DINT_D Pre<K_STORE> prefetch_coop<K_STORE>(const Ctx& c, const uint8_t* rec, const KeyInfo& ki, const TypeInfo&, bool active) {
  Pre<K_STORE> p;
  const bool need = active && rec[Wire<K_STORE>::TYPE] != 2;
  kv_prefetch_home_coop<40>(need ? kv_home_ptr<40>(c, 0, ki.h) : nullptr, need, p.v);
  return p;
}
template <>
DINT_D void apply_one<K_STORE>(const Ctx& c, uint8_t* rec, const KeyInfo& ki, const Pre<K_STORE>& pf, unsigned long long, bool) {
  using W = Wire<K_STORE>;
  const uint8_t t = rec[W::TYPE];
  uint4 v[4] = {pf.v[0], pf.v[1], pf.v[2], pf.v[3]};
  if (t == 0) {
    rec[W::TYPE] = kv_get_into<40>(c.tbl[0], ki.key, ki.h, v, rec + W::VAL, rec + W::VER) ? 3 : 7;   // kGrantRead / kNotExist
  } else if (t == 1) {
    rec[W::TYPE] = kv_set_from<40>(c.tbl[0], ki.key, ki.h, v, rec + W::VAL) ? 5 : 7;                 // kSetAck / kNotExist
  } else {
    if (kv_insert_from<40>(c.tbl[0], ki.key, ki.h, rec + W::VAL)) rec[W::TYPE] = 8;                  // kInsertAck
    else mark_invalid<K_STORE>(c, rec);
  }
}

// ============================ store, eBPF cache tier (DINT_CFG_STORE_EBPF_*) =======================
// The reference's eBPF store server: an XDP program keeps a 4-slot cache set per bucket in front of the user-space
// `kvs` (store/ebpf/store_kern.c:25-30, utils.h:58-66), answers hits and bloom negatives itself, passes misses to
// user space (store_user.c:127-165) and installs the table's answer from a TC egress program (store_kern.c:302-373).
// apply_one<K_STORE_EBPF> is that whole path for one request.  Variants: 1 = store_kern.c (write-back + bloom word),
// 2 = store_wb_kern.c (write-back, no bloom), 3 = store_wt_kern.c + store_wt_user.c (write-through).
// Cache set, 256 bytes: tag block {u64 key[4]; u32 ver[4]; u64 bloom; u8 valid_mask; u8 dirty_mask; pad} at +0 (one
// 64-byte fetch decides hit / bloom / victim), u8 val[4][40] at +64.
// Every request is a writer of its group (a READ miss installs and may write back), so two of one set in a chunk are
// replayed in index order.  Every table access of a request concerns its own bucket: the requested key or a victim of
// the same set.
enum : uint32_t { EC_WB_BLOOM = 1, EC_WB = 2, EC_WT = 3 };
constexpr uint32_t kEcSetBytes = 256;
enum : uint32_t { EC_HIT = 0, EC_BLOOM_NEG = 1, EC_TABLE = 2, EC_WRITEBACK = 3, EC_INSTALL = 4, EC_NSTATS = 5 };

template <> DINT_D TypeInfo type_info<K_STORE_EBPF>(const uint8_t* rec) {
  if (rec[Wire<K_STORE_EBPF>::TYPE] <= 2) return TypeInfo{C_WA, false, false};   // kRead / kSet / kInsert
  return TypeInfo{0, true, false};                                                // store_user.c:164
}
template <> DINT_D KeyInfo key_info<K_STORE_EBPF>(const Ctx& c, const uint8_t* rec) { return key_info<K_STORE>(c, rec); }
template <> struct Pre<K_STORE_EBPF> { uint4 t[4]; };   // the set's tag block
DINT_D uint8_t* ec_set(const Ctx& c, uint32_t g) { return c.ecache + (size_t)g * kEcSetBytes; }
template <> DINT_D Pre<K_STORE_EBPF> prefetch<K_STORE_EBPF>(const Ctx& c, const uint8_t*, const KeyInfo& ki, const TypeInfo&) {
  Pre<K_STORE_EBPF> p;
  kv_load_entry<40>(ec_set(c, ki.grp), p.t);
  return p;
}
template <>
DINT_D Pre<K_STORE_EBPF> prefetch_coop<K_STORE_EBPF>(const Ctx& c, const uint8_t*, const KeyInfo& ki, const TypeInfo&, bool active) {
  Pre<K_STORE_EBPF> p;
  kv_prefetch_home_coop<40>(active ? ec_set(c, ki.grp) : nullptr, active, p.t);
  return p;
}
// warp-aggregated counter bump: the lanes that arrive together are partitioned by counter, one atomic per partition
DINT_D void ec_count(const Ctx& c, uint32_t which) {
  namespace cg = cooperative_groups;
  const cg::coalesced_group arrived = cg::coalesced_threads();
  const cg::coalesced_group peers = cg::labeled_partition(arrived, which);
  if (peers.thread_rank() == 0) atomicAdd(&c.ecache_stats[which], (unsigned long long)peers.size());
}
DINT_D void ec_load_val(const uint8_t* set, int i, uint32_t (&w)[10]) {
  const uint2* p = (const uint2*)(set + 64 + 40 * i);
#pragma unroll
  for (int k = 0; k < 5; k++) { const uint2 q = __ldcg(p + k); w[2 * k] = q.x; w[2 * k + 1] = q.y; }
}
DINT_D void ec_store_val(uint8_t* set, int i, const uint32_t (&w)[10]) {
  uint2* p = (uint2*)(set + 64 + 40 * i);
#pragma unroll
  for (int k = 0; k < 5; k++) p[k] = make_uint2(w[2 * k], w[2 * k + 1]);
}
// the table side (store/ebpf/kvs.h), each call probing afresh: earlier calls of the same request may have written
DINT_D uint8_t* ec_tbl_find(const Ctx& c, uint64_t key, uint64_t h, uint4 (&v)[4]) {
  kv_prefetch_home<40>(c, 0, h, v);
  return kv_find<40>(c.tbl[0], key, h, v);
}
// false: the table is full (the reference's chained table never is) and the pair was lost
DINT_D bool ec_set_evict(const Ctx& c, uint64_t key, const uint32_t (&w)[10], uint32_t ver) {   // kvs.h:103-121
  uint4 v[4];
  const uint64_t h = fasthash64_u64(key);
  uint8_t* e = ec_tbl_find(c, key, h, v);
  if (e) { kv_write_val<40>(e, w); *((uint32_t*)(e + 8)) = ver; return true; }
  return kv_insert_words<40>(c.tbl[0], key, h, w);   // kvs_insert: version 0, not `ver`
}

template <>
DINT_D void apply_one<K_STORE_EBPF>(const Ctx& c, uint8_t* rec, const KeyInfo& ki, const Pre<K_STORE_EBPF>& pf, unsigned long long,
                                    bool) {
  using W = Wire<K_STORE_EBPF>;
  const uint8_t t = rec[W::TYPE];
  const uint32_t var = c.ecache_variant;
  const bool wt = var == EC_WT, bloom_on = var == EC_WB_BLOOM;
  uint8_t* set = ec_set(c, ki.grp);
  uint32_t tw[16];                                    // tag block words: key[4] (0..7), ver[4] (8..11), bloom (12..13), masks (14)
#pragma unroll
  for (int k = 0; k < 4; k++) { tw[4 * k] = pf.t[k].x; tw[4 * k + 1] = pf.t[k].y; tw[4 * k + 2] = pf.t[k].z; tw[4 * k + 3] = pf.t[k].w; }
  uint32_t valid = tw[14] & 15u, dirty = (tw[14] >> 8) & 15u;
  uint64_t bloom = ((uint64_t)tw[13] << 32) | tw[12];
  const uint64_t bit = 1ull << (ki.h >> 58);          // bf_hash, store_kern.c:80
  const uint64_t key = ki.key;
  int hit = -1;                                       // :69-72
#pragma unroll
  for (int i = 3; i >= 0; i--)
    if (((valid >> i) & 1u) && tw[2 * i] == (uint32_t)key && tw[2 * i + 1] == (uint32_t)(key >> 32)) hit = i;
  // victim slot of a miss: first invalid, else (write-back variants) first clean, else 0 (:116-125; store_wt_kern.c:104-108)
  int vic = 0;
  {
    const uint32_t inv = ~valid & 15u, cln = ~dirty & 15u;
    if (inv) vic = __ffs(inv) - 1;
    else if (!wt && cln) vic = __ffs(cln) - 1;
  }
  const bool evict = !wt && ((valid >> vic) & 1u) && ((dirty >> vic) & 1u);
  uint32_t rw[10];                                    // the request's value
  ld_words_unaligned<10>(rec + W::VAL, rw);
  bool tags_changed = false;
  bool stored = true;                                 // false: the table was full and a pair was lost (answered 0xFF)
  auto put_slot = [&](int i, uint64_t k, uint32_t ver) {
    tw[2 * i] = (uint32_t)k; tw[2 * i + 1] = (uint32_t)(k >> 32); tw[8 + i] = ver; tags_changed = true;
  };
  // store_user.c:135,146,158: kvs_set_evict of the victim, which travelled in ext_message.{key2,val2,ver2}.  `first` runs
  // between reading the victim and writing it back (the insert path's kvs_insert of the new key, :157-158).
  auto write_back = [&](auto&& first) {
    uint32_t ow[10];
    ec_load_val(set, vic, ow);
    const uint64_t ok = ((uint64_t)tw[2 * vic + 1] << 32) | tw[2 * vic];
    const uint32_t over = tw[8 + vic];
    first();
    stored &= ec_set_evict(c, ok, ow, over);
    ec_count(c, EC_WRITEBACK);
  };
  uint4 v[4];
  if (t == 2) {                                       // kInsert
    if (wt) {                                         // store_wt_kern.c:165-176, store_wt_user.c: kvs_insert
      const uint32_t inv = ~valid & 15u;
      if (inv) {
        const int i = __ffs(inv) - 1;
        put_slot(i, key, ld_u32_unaligned(rec + W::VER));   // the client's version, while the table holds 0
        ec_store_val(set, i, rw);
        valid |= 1u << i; dirty &= ~(1u << i);
        ec_count(c, EC_INSTALL);
      }
      stored &= kv_insert_words<40>(c.tbl[0], key, ki.h, rw);
      ec_count(c, EC_TABLE);
    } else {
      if (bloom_on) bloom |= bit;                     // store_kern.c:238-239
      if (evict) {                                    // :252-283, then store_user.c:155-161 and the TC INSERT_ACK path
        write_back([&] { stored &= kv_insert_words<40>(c.tbl[0], key, ki.h, rw); });
        ec_count(c, EC_TABLE);
        dirty &= ~(1u << vic);
      } else {                                        // :284-295: cached dirty, the table does not hold it yet
        valid |= 1u << vic; dirty |= 1u << vic;
      }
      put_slot(vic, key, 0);
      ec_store_val(set, vic, rw);
      ec_count(c, EC_INSTALL);
    }
    rec[W::TYPE] = 8;                                 // kInsertAck, the request's key / val / ver echoed
  } else if (hit >= 0 && (t == 0 || !wt)) {
    ec_count(c, EC_HIT);
    if (t == 0) {                                     // :74-86
      uint32_t w[10];
      ec_load_val(set, hit, w);
      st_words_unaligned<10>(rec + W::VAL, w);
      st_u32_unaligned(rec + W::VER, tw[8 + hit]);
      rec[W::TYPE] = 3;                               // kGrantRead
    } else {                                          // :157-172: the reply keeps the client's ver
      ec_store_val(set, hit, rw);
      tw[8 + hit]++; tags_changed = true;
      dirty |= 1u << hit;
      rec[W::TYPE] = 5;                               // kSetAck
    }
    if (bloom_on) bloom |= bit;
  } else if (bloom_on && !(bloom & bit)) {            // :88-94, :174-180: the bloom word says absent
    ec_count(c, EC_BLOOM_NEG);
    rec[W::TYPE] = 7;                                 // kNotExist, ver echoed
  } else {
    // XDP_PASS to user space; ext_message.ver1 carries the eviction flag (write-back variants)
    ec_count(c, EC_TABLE);
    if (evict) write_back([] {});
    if (t == 0) {                                     // store_user.c:133-142
      uint8_t* e = ec_tbl_find(c, key, ki.h, v);
      if (e) {
        const uint32_t* flat = (const uint32_t*)v;
        uint32_t w[10];
#pragma unroll
        for (int k = 0; k < 10; k++) w[k] = flat[4 + k];
        st_words_unaligned<10>(rec + W::VAL, w);
        st_u32_unaligned(rec + W::VER, v[0].z);
        rec[W::TYPE] = 3;
        put_slot(vic, key, v[0].z);                   // TC install, store_kern.c:325-342 (wt: dirty untouched, :223-235)
        ec_store_val(set, vic, w);
        valid |= 1u << vic;
        if (!wt) dirty &= ~(1u << vic);
        if (bloom_on) bloom |= bit;
        ec_count(c, EC_INSTALL);
      } else {
        if (!wt) { st_u32_unaligned(rec + W::VER, evict ? 1u : 0u); dirty &= ~(1u << vic); }   // :128-133, TC :345-352
        rec[W::TYPE] = 7;
      }
    } else {                                          // kSet, store_user.c:144-153 (kvs.h:54-73)
      if (wt && hit >= 0) valid &= ~(1u << hit);      // store_wt_kern.c:132: invalidated, never re-installed by TC
      uint8_t* e = ec_tbl_find(c, key, ki.h, v);
      uint32_t nv = 0;
      if (e) {
        kv_write_val<40>(e, rw);
        nv = v[0].z + 1;
        *((uint32_t*)(e + 8)) = nv;
      }
      st_u32_unaligned(rec + W::VER, nv);
      rec[W::TYPE] = nv != 0 ? 5 : 7;
      if (!wt) {
        if (nv != 0) {                                // TC install of the table's new version
          put_slot(vic, key, nv);
          ec_store_val(set, vic, rw);
          valid |= 1u << vic;
          if (bloom_on) bloom |= bit;
          ec_count(c, EC_INSTALL);
        }
        dirty &= ~(1u << vic);
      }
    }
  }
  if (!stored) mark_invalid<K_STORE_EBPF>(c, rec);   // as apply_one<K_STORE> answers an insert into a full table
  const uint32_t masks = valid | (dirty << 8);
  if (tags_changed || masks != (tw[14] & 0xF0Fu) || bloom != (((uint64_t)tw[13] << 32) | tw[12])) {
    uint4* tp = (uint4*)set;
    tp[0] = make_uint4(tw[0], tw[1], tw[2], tw[3]);
    tp[1] = make_uint4(tw[4], tw[5], tw[6], tw[7]);
    tp[2] = make_uint4(tw[8], tw[9], tw[10], tw[11]);
    tp[3] = make_uint4((uint32_t)bloom, (uint32_t)(bloom >> 32), masks, 0u);
  }
}

// =================================== tatp ===========================================================
template <> DINT_D TypeInfo type_info<K_TATP>(const uint8_t* rec) {
  using W = Wire<K_TATP>;
  // kCommitLog / kDeleteLog never index tables[]: they log msg.table verbatim (tatp/udp/server_shard.cc:182-207)
  if (rec[W::TYPE] == 14 || rec[W::TYPE] == 24) return TypeInfo{0, false, true};
  if (rec[W::TABLE] >= 5) return TypeInfo{0, true, false};
  switch (rec[W::TYPE]) {
    case 0: return TypeInfo{C_RA, false, false};                    // kRead
    case 1: case 2: return TypeInfo{C_WL, false, false};            // kAcquireLock, kAbort
    case 12: case 18: case 22: return TypeInfo{C_WA | C_WL, false, false};  // kCommitPrim, kInsertPrim, kDeletePrim
    case 13: case 19: case 23: return TypeInfo{C_WA, false, false};         // kCommitBck, kInsertBck, kDeleteBck
    default: return TypeInfo{0, true, false};                       // tatp/udp/server_shard.cc:209
  }
}
template <> DINT_D KeyInfo key_info<K_TATP>(const Ctx& c, const uint8_t* rec) {
  using W = Wire<K_TATP>;
  KeyInfo k;
  k.key = ld_u64_unaligned(rec + W::KEY);
  k.h = fasthash64_u64(k.key);
  k.grp = kv_group(c, rec[W::TABLE], k.h);                          // lock_hash, tatp/udp/tatp.h:12-14
  return k;
}
// v: the key's home entry; for a kAcquireLock of an engine that keeps holder keys, v[0].x/.y = the group's holder word
template <> struct Pre<K_TATP> { uint4 v[4]; };
// The holder word (tatp/ebpf/lock_kern.c:12-16 `txn_lock.key`) belongs to resource L of its group: written by a granted
// kAcquireLock, read by a refused one, both WL.  A solo acquire is the only WL request of its group in the chunk, so the
// word fetched beside the flag lookup is the one its reply needs; two acquires of one group raise W2 and are replayed in
// index order, each fetching the word after its predecessor was applied.
DINT_D bool tatp_wants_holder(const Ctx& c, uint8_t type) { return type == 1 && c.holder != nullptr; }
DINT_D uint2 tatp_load_holder(const Ctx& c, uint32_t g) { return __ldcg((const uint2*)(c.holder + g)); }
DINT_D bool tatp_touches_row(uint8_t type) {   // request types that look a row up (not insert / lock / log)
  return type == 0 || type == 12 || type == 13 || type == 22 || type == 23;
}
template <> DINT_D Pre<K_TATP> prefetch<K_TATP>(const Ctx& c, const uint8_t* rec, const KeyInfo& ki, const TypeInfo&) {
  using W = Wire<K_TATP>;
  Pre<K_TATP> p;
  if (tatp_touches_row(rec[W::TYPE])) kv_prefetch_home<40>(c, rec[W::TABLE], ki.h, p.v);
  else if (tatp_wants_holder(c, rec[W::TYPE])) { const uint2 k = tatp_load_holder(c, ki.grp); p.v[0].x = k.x; p.v[0].y = k.y; }
  return p;
}
template <> DINT_D Pre<K_TATP> prefetch_coop<K_TATP>(const Ctx& c, const uint8_t* rec, const KeyInfo& ki, const TypeInfo&, bool active) {
  using W = Wire<K_TATP>;
  Pre<K_TATP> p;
  const bool need = active && tatp_touches_row(rec[W::TYPE]);
  const bool lock = active && tatp_wants_holder(c, rec[W::TYPE]);
  uint2 k = make_uint2(0, 0);
  if (lock) k = tatp_load_holder(c, ki.grp);        // issued before the row fetch: the two latencies overlap
  kv_prefetch_home_coop<40>(need ? kv_home_ptr<40>(c, rec[W::TABLE], ki.h) : nullptr, need, p.v);
  if (lock) { p.v[0].x = k.x; p.v[0].y = k.y; }
  return p;
}
// kCommitLog (tatp/udp/server_shard.cc:182-194) / kDeleteLog (:196-207); the eBPF server's XDP path
// (tatp/ebpf/shard_kern.c:914-936) writes the same entry
DINT_D void tatp_log_append(const Ctx& c, uint8_t* rec, uint8_t type, uint8_t table, unsigned long long ord, bool keep) {
  using W = Wire<K_TATP>;
  if (keep) {                              // log_entry {is_del@0 table@1 key@8 val@16 ver@56} tatp/udp/kvs.h:23-29
    uint8_t* e = c.ring + (size_t)(ord % c.ring_n) * W::LOGENT;
    uint32_t w[13];
    ld_words_unaligned<13>(rec + W::KEY, w);          // key, val, ver are contiguous on the wire
    e[0] = (type == 24);
    e[1] = table;
    *((uint2*)(e + 8)) = make_uint2(w[0], w[1]);
    if (type == 14) {
      *((uint4*)(e + 16)) = make_uint4(w[2], w[3], w[4], w[5]);
      *((uint4*)(e + 32)) = make_uint4(w[6], w[7], w[8], w[9]);
      *((uint2*)(e + 48)) = make_uint2(w[10], w[11]);
    }
    *((uint32_t*)(e + 56)) = w[12];
  }
  rec[W::TYPE] = (type == 14) ? 17 : 27;
}
template <>
DINT_D void apply_one<K_TATP>(const Ctx& c, uint8_t* rec, const KeyInfo& ki, const Pre<K_TATP>& pf, unsigned long long ord,
                              bool keep) {
  using W = Wire<K_TATP>;
  const uint8_t type = rec[W::TYPE], table = rec[W::TABLE];
  if (type == 14 || type == 24) { tatp_log_append(c, rec, type, table, ord, keep); return; }
  const KvTable& t = c.tbl[table];
  const uint64_t key = ki.key, h = ki.h;
  const uint32_t g = ki.grp;
  uint4 v[4] = {pf.v[0], pf.v[1], pf.v[2], pf.v[3]};
  bool ok = true;
  switch (type) {
    case 0: rec[W::TYPE] = kv_get_into<40>(t, key, h, v, rec + W::VAL, rec + W::VER) ? 4 : 6; break;  // :116-121
    case 1:                                                                                           // :123-132
      if (!bm_fetch_set(c.lockbits, g)) {                    // granted; with holder keys, tatp/ebpf/lock_kern.c:290-293
        if (c.holder) __stcg((uint2*)(c.holder + g), make_uint2((uint32_t)key, (uint32_t)(key >> 32)));
        rec[W::TYPE] = 7;
      } else {                                               // :294-298: kRejectLockSameKey when the holder's key is ours
        rec[W::TYPE] = (c.holder && v[0].x == (uint32_t)key && v[0].y == (uint32_t)(key >> 32)) ? 28 : 8;
      }
      break;
    case 2: bm_clear_bit(c.lockbits, g); rec[W::TYPE] = 9; break;                                     // :134-138
    // a would-panic request (kvs_set / kvs_delete on a missing key) applies NOTHING: the reference dies before the unlock
    case 12: ok = kv_set_from<40>(t, key, h, v, rec + W::VAL); if (ok) bm_clear_bit(c.lockbits, g); rec[W::TYPE] = 15; break;  // :140-146
    case 18: ok = kv_insert_from<40>(t, key, h, rec + W::VAL); if (ok) bm_clear_bit(c.lockbits, g); rec[W::TYPE] = 20; break;  // :148-154
    case 22: ok = kv_delete<40>(t, key, h, v); if (ok) bm_clear_bit(c.lockbits, g); rec[W::TYPE] = 25; break;                  // :156-162
    case 13: ok = kv_set_from<40>(t, key, h, v, rec + W::VAL); rec[W::TYPE] = 16; break;              // :164-168
    case 19: ok = kv_insert_from<40>(t, key, h, rec + W::VAL); rec[W::TYPE] = 21; break;              // :170-174
    default: ok = kv_delete<40>(t, key, h, v); rec[W::TYPE] = 26; break;                              // 23 :176-180
  }
  if (!ok) mark_invalid<K_TATP>(c, rec);   // kvs_set / kvs_delete on a missing key: tatp/udp/kvs.h:91,152 panic
}

// ============================ tatp, eBPF cache tier (DINT_CFG_TATP_EBPF) ============================
// The reference's eBPF TATP shard server (tatp/ebpf/shard_kern.c; lock_kern.c = the same with holder keys): an XDP
// program keeps a 4-slot write-back cache set with a bloom word per bucket of every table, answers hits and the lock
// traffic itself, passes misses to a user-space chained `kvs` (shard_user.c:171-247, tatp/ebpf/kvs.h) and installs the
// answer from a TC egress program (shard_kern.c:941-1289).  apply_one<K_TATP_EBPF> is that whole path for one request.
// Cache sets use the store tier's 256-byte layout (EC_*, ec_set / ec_load_val / ec_store_val).  The table side is the
// reference's chained table itself, so that chain order (which of two copies of a key a lookup finds) and the stale keys
// of invalid slots (which the bloom word rebuilt after a delete hashes, shard_user.c:94-104) are what the reference has:
// a {head, free list} pair per bucket and 256-byte chain entries {u64 key[4]; u32 ver[4]; u32 valid; u32 next;
// u32 table; pad} + u8 val[4][40] at +64, drawn from one pool by a bump allocator, or from the entries the bucket freed.
// Conflict group = (table, bucket): every table access of a request concerns its own bucket, and a lock slot h % 4H
// lies in bucket h % H.  Lock words (and holder words) stay one per lock slot, at position grp_base + 4 b + j for slot
// b + H j; the group id of a bucket is that position / 4 (grp_base / 4 + b), which is also the index of its cache set
// and chain head, so consecutive buckets use consecutive flag nibbles.
enum : uint32_t { EC_ALLOC = 5, EC_REUSE = 6, EC_FREE = 7, EC_FAILED = 8, EC_NSTATS_TATP = 9 };
constexpr uint32_t kTeEntBytes = 256;

template <> DINT_D TypeInfo type_info<K_TATP_EBPF>(const uint8_t* rec) {
  using W = Wire<K_TATP_EBPF>;
  if (rec[W::TYPE] == 14 || rec[W::TYPE] == 24) return TypeInfo{0, false, true};   // shard_kern.c:914-936
  if (rec[W::TABLE] >= 5) return TypeInfo{0, true, false};
  switch (rec[W::TYPE]) {
    case 0: case 13: case 19: case 23: return TypeInfo{C_WA, false, false};      // kRead (a hit may set a bloom bit), *Bck
    case 1: case 2: return TypeInfo{C_WL, false, false};                         // kAcquireLock, kAbort
    case 12: case 18: case 22: return TypeInfo{C_WA | C_WL, false, false};       // kCommitPrim, kInsertPrim, kDeletePrim
    default: return TypeInfo{0, true, false};                                    // shard_user.c:247 panics
  }
}
// position of the lock word of (table, h): slot s = h % 4H (shard_kern.c:256) = b + H j with b = h % H
DINT_D uint32_t te_lock_pos(const Ctx& c, uint32_t table, uint64_t h) {
  const uint32_t s = fast_mod(h, c.tbl[table].lock_mod);
  const uint32_t j = (uint32_t)fast_div(s, c.tbkt_mod[table]);
  return c.tbl[table].grp_base + 4 * (s - j * c.tbkt_mod[table].d) + j;
}
template <> DINT_D KeyInfo key_info<K_TATP_EBPF>(const Ctx& c, const uint8_t* rec) {
  using W = Wire<K_TATP_EBPF>;
  KeyInfo k;
  k.key = ld_u64_unaligned(rec + W::KEY);
  k.h = fasthash64_u64(k.key);
  k.grp = te_lock_pos(c, rec[W::TABLE], k.h) >> 2;     // one engine owns the whole key space (n_shards = 1)
  return k;
}
template <> struct Pre<K_TATP_EBPF> { uint4 t[4]; };   // the set's tag block
DINT_D bool te_touches_set(uint8_t type) { return type != 1 && type != 2 && type != 14 && type != 24; }
template <> DINT_D Pre<K_TATP_EBPF> prefetch<K_TATP_EBPF>(const Ctx& c, const uint8_t* rec, const KeyInfo& ki, const TypeInfo&) {
  Pre<K_TATP_EBPF> p;
  if (te_touches_set(rec[Wire<K_TATP_EBPF>::TYPE])) kv_load_entry<40>(ec_set(c, ki.grp), p.t);
  return p;
}
template <>
DINT_D Pre<K_TATP_EBPF> prefetch_coop<K_TATP_EBPF>(const Ctx& c, const uint8_t* rec, const KeyInfo& ki, const TypeInfo&, bool active) {
  Pre<K_TATP_EBPF> p;
  const bool need = active && te_touches_set(rec[Wire<K_TATP_EBPF>::TYPE]);
  kv_prefetch_home_coop<40>(need ? ec_set(c, ki.grp) : nullptr, need, p.t);
  return p;
}

// ---- the chained table (tatp/ebpf/kvs.h) of bucket `si` --------------------------------------------------------
DINT_D uint8_t* te_ent(const Ctx& c, uint32_t e1) { return c.tpool + (size_t)(e1 - 1) * kTeEntBytes; }
DINT_D void te_load_tag(const uint8_t* e, uint32_t (&w)[16]) {
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const uint4 q = __ldcg((const uint4*)e + k);
    w[4 * k] = q.x; w[4 * k + 1] = q.y; w[4 * k + 2] = q.z; w[4 * k + 3] = q.w;
  }
}
// the first valid copy of `key`, head first (kvs.h:38-53): its entry (index + 1, 0 = absent), slot, predecessor, tags
DINT_D uint32_t te_find(const Ctx& c, uint32_t si, uint64_t key, int& slot, uint32_t& prev, uint32_t (&tw)[16]) {
  prev = 0;
  for (uint32_t e = __ldcg(&c.tchain[si].x); e;) {
    te_load_tag(te_ent(c, e), tw);
    for (int i = 0; i < 4; i++)
      if (((tw[12] >> i) & 1u) && tw[2 * i] == (uint32_t)key && tw[2 * i + 1] == (uint32_t)(key >> 32)) { slot = i; return e; }
    prev = e;
    e = tw[13];
  }
  return 0;
}
// a zeroed entry (as calloc leaves it) for bucket si: one the bucket freed, else a fresh one of the pool; 0 = exhausted
DINT_D uint32_t te_alloc(const Ctx& c, uint32_t si, uint32_t table) {
  uint32_t e = __ldcg(&c.tchain[si].y);
  uint8_t* p;
  if (e) {
    p = te_ent(c, e);
    c.tchain[si].y = __ldcg((const uint32_t*)(p + 52));
#pragma unroll
    for (int k = 0; k < 16; k++) ((uint4*)p)[k] = make_uint4(0, 0, 0, 0);
    ec_count(c, EC_REUSE);
  } else {
    // fresh pool entries were zeroed at create; once the pool is spent the counter stops (overshoot <= concurrent lanes)
    if (__ldcg(c.tpool_top) >= c.tpool_cap || (e = atomicAdd(c.tpool_top, 1u) + 1) > c.tpool_cap) {
      ec_count(c, EC_FAILED);
      return 0;
    }
    p = te_ent(c, e);
    ec_count(c, EC_ALLOC);
  }
  *(uint32_t*)(p + 56) = table;
  return e;
}
// kvs_insert (kvs.h:56-82): the first invalid slot walking from the head, else slot 0 of a new head entry
DINT_D bool te_insert(const Ctx& c, uint32_t si, uint32_t table, uint64_t key, const uint32_t (&w)[10]) {
  uint32_t tw[16];
  uint32_t e = __ldcg(&c.tchain[si].x);
  int slot = 0;
  for (; e; e = tw[13]) {
    te_load_tag(te_ent(c, e), tw);
    const uint32_t inv = ~tw[12] & 15u;
    if (inv) { slot = __ffs(inv) - 1; break; }
  }
  uint32_t valid;
  if (e) {
    valid = tw[12] | (1u << slot);
  } else {
    e = te_alloc(c, si, table);
    if (!e) return false;
    valid = 1;
    *(uint32_t*)(te_ent(c, e) + 52) = __ldcg(&c.tchain[si].x);
    c.tchain[si].x = e;
  }
  uint8_t* p = te_ent(c, e);
  *(uint2*)(p + 8 * slot) = make_uint2((uint32_t)key, (uint32_t)(key >> 32));
  *(uint32_t*)(p + 32 + 4 * slot) = 0;
  *(uint32_t*)(p + 48) = valid;
  ec_store_val(p, slot, w);
  return true;
}
// kvs_set (kvs.h:84-104): overwrite val, ver = `ver` when non-zero else ver + 1; an absent key is inserted with
// version 0.  Returns the new version (0 after an insert); `ok` turns false when the insert found no entry.
DINT_D uint32_t te_set(const Ctx& c, uint32_t si, uint32_t table, uint64_t key, const uint32_t (&w)[10], uint32_t ver, bool& ok) {
  uint32_t tw[16], prev;
  int slot = 0;
  const uint32_t e = te_find(c, si, key, slot, prev, tw);
  if (!e) { ok &= te_insert(c, si, table, key, w); return 0; }
  uint8_t* p = te_ent(c, e);
  ec_store_val(p, slot, w);
  const uint32_t nv = ver != 0 ? ver : tw[8 + slot] + 1;
  *(uint32_t*)(p + 32 + 4 * slot) = nv;
  return nv;
}
// kvs_delete (kvs.h:106-133): the key bytes stay; an entry whose slots are all invalid leaves the chain for the
// bucket's free list
DINT_D void te_delete(const Ctx& c, uint32_t si, uint64_t key) {
  uint32_t tw[16], prev;
  int slot = 0;
  const uint32_t e = te_find(c, si, key, slot, prev, tw);
  if (!e) return;
  uint8_t* p = te_ent(c, e);
  const uint32_t valid = tw[12] & ~(1u << slot);
  *(uint32_t*)(p + 48) = valid;
  if (valid) return;
  if (prev) *(uint32_t*)(te_ent(c, prev) + 52) = tw[13];
  else c.tchain[si].x = tw[13];
  *(uint32_t*)(p + 52) = __ldcg(&c.tchain[si].y);
  c.tchain[si].y = e;
  ec_count(c, EC_FREE);
}
// calculate_bloom_filter (shard_user.c:94-104): one bit per chain entry, of fasthash64 over its whole key[4] array
DINT_D uint64_t te_bloom(const Ctx& c, uint32_t si) {
  uint64_t bf = 0;
  uint32_t tw[16];
  for (uint32_t e = __ldcg(&c.tchain[si].x); e; e = tw[13]) {
    te_load_tag(te_ent(c, e), tw);
    uint64_t h = kFhSeed ^ (32ULL * kFhM);
#pragma unroll
    for (int k = 0; k < 4; k++) {
      h ^= fh_mix(((uint64_t)tw[2 * k + 1] << 32) | tw[2 * k]);
      h *= kFhM;
    }
    bf |= 1ull << (fh_mix(h) >> 58);
  }
  return bf;
}

template <>
DINT_D void apply_one<K_TATP_EBPF>(const Ctx& c, uint8_t* rec, const KeyInfo& ki, const Pre<K_TATP_EBPF>& pf,
                                   unsigned long long ord, bool keep) {
  using W = Wire<K_TATP_EBPF>;
  const uint8_t type = rec[W::TYPE], table = rec[W::TABLE];
  if (type == 14 || type == 24) { tatp_log_append(c, rec, type, table, ord, keep); return; }
  const uint64_t key = ki.key;
  const uint32_t lp = te_lock_pos(c, table, ki.h);
  if (type == 1) {                                    // shard_kern.c:251-296; lock_kern.c:289-298
    if (!bm_fetch_set(c.lockbits, lp)) {
      if (c.holder) __stcg((uint2*)(c.holder + lp), make_uint2((uint32_t)key, (uint32_t)(key >> 32)));
      rec[W::TYPE] = 7;
    } else {
      const uint2 hk = c.holder ? __ldcg((const uint2*)(c.holder + lp)) : make_uint2(0, 0);
      rec[W::TYPE] = (c.holder && hk.x == (uint32_t)key && hk.y == (uint32_t)(key >> 32)) ? 28 : 8;
    }
    return;
  }
  if (type == 2) { bm_clear_bit(c.lockbits, lp); rec[W::TYPE] = 9; return; }   // :298-336
  const bool prim = type == 12 || type == 18 || type == 22;
  const uint32_t si = ki.grp;
  uint8_t* set = ec_set(c, si);
  uint32_t tw[16];                                    // tag block words: key[4] (0..7), ver[4] (8..11), bloom (12..13), masks (14)
#pragma unroll
  for (int k = 0; k < 4; k++) { tw[4 * k] = pf.t[k].x; tw[4 * k + 1] = pf.t[k].y; tw[4 * k + 2] = pf.t[k].z; tw[4 * k + 3] = pf.t[k].w; }
  uint32_t valid = tw[14] & 15u, dirty = (tw[14] >> 8) & 15u;
  uint64_t bloom = ((uint64_t)tw[13] << 32) | tw[12];
  const uint64_t bit = 1ull << (ki.h >> 58);          // shard_kern.c:191
  int hit = -1;
#pragma unroll
  for (int i = 3; i >= 0; i--)
    if (((valid >> i) & 1u) && tw[2 * i] == (uint32_t)key && tw[2 * i + 1] == (uint32_t)(key >> 32)) hit = i;
  int vic = 0;                                        // victim of a miss: first invalid, else first clean, else 0 (:227-236)
  {
    const uint32_t inv = ~valid & 15u, cln = ~dirty & 15u;
    if (inv) vic = __ffs(inv) - 1;
    else if (cln) vic = __ffs(cln) - 1;
  }
  const bool evict = ((valid >> vic) & 1u) && ((dirty >> vic) & 1u);
  // the dirty victim, as XDP copies it into ext_message.{key2,val2,ver2} before the slot is reused
  uint32_t ow[10];
  const uint64_t okey = ((uint64_t)tw[2 * vic + 1] << 32) | tw[2 * vic];
  const uint32_t over = tw[8 + vic];
  if (evict) ec_load_val(set, vic, ow);
  uint32_t rw[10];                                    // the request's value
  ld_words_unaligned<10>(rec + W::VAL, rw);
  // false: the chain-entry pool was exhausted.  The request is answered 0xFF, but what it did before the failed
  // allocation stays (the cache set's new tags and values, a write-back that found its entry): the reference's calloc
  // cannot fail, so there is no reference behaviour to follow, and keeping the set consistent with the table matters more.
  bool ok = true;
  bool tags_changed = false;
  auto put_slot = [&](int i, uint64_t k, uint32_t ver) {
    tw[2 * i] = (uint32_t)k; tw[2 * i + 1] = (uint32_t)(k >> 32); tw[8 + i] = ver; tags_changed = true;
  };
  auto write_back = [&]() {                           // shard_user.c:181,191,226: kvs_set(key2, val2, ver2)
    (void)te_set(c, si, table, okey, ow, over, ok);
    ec_count(c, EC_WRITEBACK);
  };
  if (type == 0) {                                    // kRead :140-249, TC GRANT_READ :964-1010 / NOT_EXIST :1012-1045
    if (hit >= 0) {
      ec_count(c, EC_HIT);
      uint32_t w[10];
      ec_load_val(set, hit, w);
      st_words_unaligned<10>(rec + W::VAL, w);
      st_u32_unaligned(rec + W::VER, tw[8 + hit]);
      bloom |= bit;
      rec[W::TYPE] = 4;                               // kGrantRead
    } else if (!(bloom & bit)) {
      ec_count(c, EC_BLOOM_NEG);
      rec[W::TYPE] = 6;                               // kNotExist, ver echoed
    } else {
      ec_count(c, EC_TABLE);
      if (evict) write_back();
      uint32_t ct[16], prev;
      int slot = 0;
      const uint32_t e = te_find(c, si, key, slot, prev, ct);
      if (e) {
        uint32_t w[10];
        ec_load_val(te_ent(c, e), slot, w);
        st_words_unaligned<10>(rec + W::VAL, w);
        st_u32_unaligned(rec + W::VER, ct[8 + slot]);
        put_slot(vic, key, ct[8 + slot]);
        ec_store_val(set, vic, w);
        valid |= 1u << vic;
        dirty &= ~(1u << vic);
        bloom |= bit;
        ec_count(c, EC_INSTALL);
        rec[W::TYPE] = 4;
      } else {
        st_u32_unaligned(rec + W::VER, evict ? 1u : 0u);   // ext_message.ver1: the eviction flag (:239-244)
        rec[W::TYPE] = 6;
      }
    }
  } else if (type == 12 || type == 13) {              // kCommitPrim :338-474 / kCommitBck :659-761
    if (hit >= 0) {
      ec_count(c, EC_HIT);
      if (prim) bm_clear_bit(c.lockbits, lp);
      ec_store_val(set, hit, rw);
      tw[8 + hit]++; tags_changed = true;
      dirty |= 1u << hit;                             // the reply echoes the client's ver
    } else {
      ec_count(c, EC_TABLE);
      if (evict) write_back();
      const uint32_t nv = te_set(c, si, table, key, rw, 0, ok);   // shard_user.c:192,227
      if (prim) bm_clear_bit(c.lockbits, lp);         // TC COMMIT_PRIM_ACK :1112
      put_slot(vic, key, nv);                         // XDP :469-471 (key, val, clean), TC :1116-1117 (ver, valid)
      ec_store_val(set, vic, rw);
      valid |= 1u << vic;
      dirty &= ~(1u << vic);
      st_u32_unaligned(rec + W::VER, nv);
      ec_count(c, EC_INSTALL);
    }
    rec[W::TYPE] = prim ? 15 : 16;
  } else if (type == 18 || type == 19) {              // kInsertPrim :476-608 / kInsertBck :763-863
    bloom |= bit;
    if (evict) {                                      // XDP overwrites the slot (ver 0, clean), user space inserts the
      ec_count(c, EC_TABLE);                          // row and writes the victim back (shard_user.c:199-200,233-234)
      ok &= te_insert(c, si, table, key, rw);
      write_back();
      dirty &= ~(1u << vic);
    } else {                                          // cache only, dirty: the table never sees the row
      valid |= 1u << vic;
      dirty |= 1u << vic;
    }
    put_slot(vic, key, 0);
    ec_store_val(set, vic, rw);
    ec_count(c, EC_INSTALL);
    if (prim) bm_clear_bit(c.lockbits, lp);
    rec[W::TYPE] = prim ? 20 : 21;
  } else {                                            // kDeletePrim :610-657 / kDeleteBck :865-912
    ec_count(c, EC_TABLE);
    if (hit >= 0) valid &= ~(1u << hit);
    te_delete(c, si, key);                            // shard_user.c:207-213,236-242
    bloom = te_bloom(c, si);                          // TC :1186-1187 installs the rebuilt word
    if (prim) bm_clear_bit(c.lockbits, lp);
    const uint32_t bw[2] = {(uint32_t)bloom, (uint32_t)(bloom >> 32)};
    st_words_unaligned<2>(rec + W::VAL, bw);          // *(u64 *)val1 = new_bf
    rec[W::TYPE] = prim ? 25 : 26;
  }
  if (!ok) mark_invalid<K_TATP_EBPF>(c, rec);
  const uint32_t masks = valid | (dirty << 8);
  if (tags_changed || masks != (tw[14] & 0xF0Fu) || bloom != (((uint64_t)tw[13] << 32) | tw[12])) {
    uint4* tp = (uint4*)set;
    tp[0] = make_uint4(tw[0], tw[1], tw[2], tw[3]);
    tp[1] = make_uint4(tw[4], tw[5], tw[6], tw[7]);
    tp[2] = make_uint4(tw[8], tw[9], tw[10], tw[11]);
    tp[3] = make_uint4((uint32_t)bloom, (uint32_t)(bloom >> 32), masks, 0u);
  }
}

// =================================== smallbank ======================================================
template <> DINT_D TypeInfo type_info<K_SMALLBANK>(const uint8_t* rec) {
  using W = Wire<K_SMALLBANK>;
  if (rec[W::TABLE] >= 2) return TypeInfo{0, true, false};
  switch (rec[W::TYPE]) {
    case 0: case 1: return TypeInfo{C_WL | C_RA, false, false};     // kAcquireShared / kAcquireExclusive (+kvs_get)
    case 2: case 3: return TypeInfo{C_WL, false, false};            // kReleaseShared / kReleaseExclusive
    case 4: case 5: return TypeInfo{C_WA, false, false};            // kCommitPrim / kCommitBck
    case 6: return TypeInfo{0, false, true};                        // kCommitLog
    default: return TypeInfo{0, true, false};                       // smallbank/udp/server_shard.cc:188
  }
}
template <> DINT_D KeyInfo key_info<K_SMALLBANK>(const Ctx& c, const uint8_t* rec) {
  using W = Wire<K_SMALLBANK>;
  KeyInfo k;
  k.key = ld_u64_unaligned(rec + W::KEY);
  k.h = fasthash64_u64(k.key);
  k.grp = kv_group(c, rec[W::TABLE], k.h);                          // :109 lock_hash
  return k;
}
template <> struct Pre<K_SMALLBANK> { uint4 v[2]; uint2 s; };
template <> DINT_D Pre<K_SMALLBANK> prefetch<K_SMALLBANK>(const Ctx& c, const uint8_t* rec, const KeyInfo& ki, const TypeInfo&) {
  using W = Wire<K_SMALLBANK>;
  Pre<K_SMALLBANK> p;
  const uint8_t type = rec[W::TYPE];
  if (type <= 3) p.s = __ldcg(&c.cnt2[ki.grp]);
  if (type != 2 && type != 3) kv_prefetch_home<8>(c, rec[W::TABLE], ki.h, p.v);
  return p;
}
template <> DINT_D Pre<K_SMALLBANK> prefetch_coop<K_SMALLBANK>(const Ctx& c, const uint8_t* rec, const KeyInfo& ki, const TypeInfo&, bool active) {
  using W = Wire<K_SMALLBANK>;
  Pre<K_SMALLBANK> p;
  const uint8_t type = active ? rec[W::TYPE] : 2;
  if (active && type <= 3) p.s = __ldcg(&c.cnt2[ki.grp]);
  const bool need = active && type != 2 && type != 3;
  kv_prefetch_home_coop<8>(need ? kv_home_ptr<8>(c, rec[W::TABLE], ki.h) : nullptr, need, p.v);
  return p;
}
// kCommitLog (smallbank/udp/server_shard.cc:175-186); the eBPF server's XDP path (smallbank/ebpf/shard_kern.c:566-583)
// writes the same entry, whatever the table byte
DINT_D void smallbank_log_append(const Ctx& c, uint8_t* rec, uint8_t table, unsigned long long ord, bool keep) {
  using W = Wire<K_SMALLBANK>;
  if (keep) {                              // log_entry {table@0 key@8 val@16 ver@24}
    uint8_t* e = c.ring + (size_t)(ord % c.ring_n) * W::LOGENT;
    uint32_t w[5];
    ld_words_unaligned<5>(rec + W::KEY, w);
    e[0] = table;
    *((uint2*)(e + 8)) = make_uint2(w[0], w[1]);
    *((uint2*)(e + 16)) = make_uint2(w[2], w[3]);
    *((uint32_t*)(e + 24)) = w[4];
  }
  rec[W::TYPE] = 15;
}
template <>
DINT_D void apply_one<K_SMALLBANK>(const Ctx& c, uint8_t* rec, const KeyInfo& ki, const Pre<K_SMALLBANK>& pf,
                                   unsigned long long ord, bool keep) {
  using W = Wire<K_SMALLBANK>;
  const uint8_t type = rec[W::TYPE], table = rec[W::TABLE];
  if (type == 6) { smallbank_log_append(c, rec, table, ord, keep); return; }
  const KvTable& t = c.tbl[table];
  const uint64_t key = ki.key, h = ki.h;
  const uint32_t g = ki.grp;
  uint4 v[2] = {pf.v[0], pf.v[1]};
  bool ok = true;
  if (type <= 3) {
    uint2 s = pf.s;                        // x = num_ex, y = num_sh
    if (type == 0) {                       // :121-133
      if (s.x == 0) { s.y++; c.cnt2[g] = s; ok = kv_get_into<8>(t, key, h, v, rec + W::VAL, rec + W::VER); rec[W::TYPE] = 7; }
      else rec[W::TYPE] = 8;
    } else if (type == 1) {                // :135-147
      if (s.x == 0 && s.y == 0) { s.x++; c.cnt2[g] = s; ok = kv_get_into<8>(t, key, h, v, rec + W::VAL, rec + W::VER); rec[W::TYPE] = 9; }
      else rec[W::TYPE] = 10;
    } else if (type == 2) { s.y--; c.cnt2[g] = s; rec[W::TYPE] = 11; }   // :149-154
    else { s.x--; c.cnt2[g] = s; rec[W::TYPE] = 12; }                    // :156-161
  } else {                                 // kCommitPrim :163-167 / kCommitBck :169-173
    ok = kv_set_from<8>(t, key, h, v, rec + W::VAL);
    rec[W::TYPE] = (type == 4) ? 13 : 14;
  }
  if (!ok) mark_invalid<K_SMALLBANK>(c, rec);   // smallbank/udp/kvs.h:67,86 panic
}

// ============================ smallbank, eBPF cache tier (DINT_CFG_SMALLBANK_EBPF) ==================
// The reference's eBPF SmallBank shard server (smallbank/ebpf/shard_kern.c): an XDP program keeps the lock units and a
// 4-slot write-back cache set per bucket of both tables, answers lock traffic and cache hits itself, passes misses to
// user space (shard_user.c:139-189, over smallbank/ebpf/kvs.h) and installs the table's answer from a TC egress program
// (shard_kern.c:671-741).  apply_one<K_SMALLBANK_EBPF> is that whole path for one request.  There is no bloom word, no
// insert and no delete, so the table side is the open-addressing table of K_SMALLBANK: population inserts a key once,
// and kvs_get / kvs_set find that one copy whatever the chain layout is.
// Cache set, 128 bytes: tag block {u64 key[4]; u32 ver[4]; u32 valid_mask | dirty_mask << 8; pad} at +0 (one 64-byte
// fetch decides hit / victim), u64 val[4] at +64.  Conflict group = (table, bucket), numbered and laid out as
// K_TATP_EBPF's (te_lock_pos): the {num_ex, num_sh} counters stay one per lock slot h % 4H, at grp_base + 4 b + j.
enum : uint32_t { SBE_HIT = 0, SBE_TABLE = 1, SBE_WRITEBACK = 2, SBE_INSTALL = 3, SBE_NSTATS = 4 };
constexpr uint32_t kSbeSetBytes = 128;

template <> DINT_D TypeInfo type_info<K_SMALLBANK_EBPF>(const uint8_t* rec) {
  using W = Wire<K_SMALLBANK_EBPF>;
  if (rec[W::TYPE] == 6) return TypeInfo{0, false, true};          // kCommitLog: the table byte is never checked
  if (rec[W::TABLE] >= 2) return TypeInfo{0, true, false};         // XDP passes it up unextended: shard_user.c:142 panics
  switch (rec[W::TYPE]) {
    case 0: case 1: return TypeInfo{C_WL | C_WA, false, false};    // kAcquire*: the counters, then the set (a miss installs)
    case 2: case 3: return TypeInfo{C_WL, false, false};           // kRelease*
    case 4: case 5: case 17: return TypeInfo{C_WA, false, false};  // kCommitPrim / kCommitBck / kWarmupRead
    default: return TypeInfo{0, true, false};                      // shard_user.c:142,188 panic
  }
}
template <> DINT_D KeyInfo key_info<K_SMALLBANK_EBPF>(const Ctx& c, const uint8_t* rec) {
  using W = Wire<K_SMALLBANK_EBPF>;
  KeyInfo k;
  k.key = ld_u64_unaligned(rec + W::KEY);
  k.h = fasthash64_u64(k.key);
  k.grp = te_lock_pos(c, rec[W::TABLE], k.h) >> 2;     // one engine owns the whole key space (n_shards = 1)
  return k;
}
template <> struct Pre<K_SMALLBANK_EBPF> { uint4 t[4]; uint2 s; };   // the set's tag block; the lock unit's counters
DINT_D uint8_t* sbe_set(const Ctx& c, uint32_t g) { return c.ecache + (size_t)g * kSbeSetBytes; }
template <>
DINT_D Pre<K_SMALLBANK_EBPF> prefetch<K_SMALLBANK_EBPF>(const Ctx& c, const uint8_t* rec, const KeyInfo& ki, const TypeInfo&) {
  using W = Wire<K_SMALLBANK_EBPF>;
  Pre<K_SMALLBANK_EBPF> p;
  const uint8_t type = rec[W::TYPE];
  if (type <= 3) p.s = __ldcg(&c.cnt2[te_lock_pos(c, rec[W::TABLE], ki.h)]);
  if (type != 2 && type != 3) kv_load_entry<40>(sbe_set(c, ki.grp), p.t);
  return p;
}
template <>
DINT_D Pre<K_SMALLBANK_EBPF> prefetch_coop<K_SMALLBANK_EBPF>(const Ctx& c, const uint8_t* rec, const KeyInfo& ki,
                                                             const TypeInfo&, bool active) {
  using W = Wire<K_SMALLBANK_EBPF>;
  Pre<K_SMALLBANK_EBPF> p;
  const uint8_t type = active ? rec[W::TYPE] : 2;
  if (active && type <= 3) p.s = __ldcg(&c.cnt2[te_lock_pos(c, rec[W::TABLE], ki.h)]);
  const bool need = active && type != 2 && type != 3;
  kv_prefetch_home_coop<40>(need ? sbe_set(c, ki.grp) : nullptr, need, p.t);
  return p;
}

template <>
DINT_D void apply_one<K_SMALLBANK_EBPF>(const Ctx& c, uint8_t* rec, const KeyInfo& ki, const Pre<K_SMALLBANK_EBPF>& pf,
                                        unsigned long long ord, bool keep) {
  using W = Wire<K_SMALLBANK_EBPF>;
  const uint8_t type = rec[W::TYPE], table = rec[W::TABLE];
  if (type == 6) { smallbank_log_append(c, rec, table, ord, keep); return; }   // shard_kern.c:566-583
  if (type <= 3) {                                    // the lock unit (:96-392): a refusal changes nothing
    uint2 s = pf.s;                                   // x = num_ex, y = num_sh
    // struct lock_unit's counters are ints tested with > 0 (:138, :255): a count that a stray release took below zero
    // refuses nothing, where the UDP server's unsigned == 0 test refuses
    if (type == 0) {
      if ((int32_t)s.x > 0) { rec[W::TYPE] = 8; return; }   // kRejectShared
      s.y++;
    } else if (type == 1) {
      if ((int32_t)s.x > 0 || (int32_t)s.y > 0) { rec[W::TYPE] = 10; return; }   // kRejectExclusive
      s.x++;
    } else if (type == 2) s.y--;                      // no floor, as the UDP server
    else s.x--;
    c.cnt2[te_lock_pos(c, table, ki.h)] = s;          // a grant counts BEFORE the cache is looked at
    if (type >= 2) { rec[W::TYPE] = type == 2 ? 11 : 12; return; }
  }
  const KvTable& t = c.tbl[table];
  const uint64_t key = ki.key;
  const bool commit = type == 4 || type == 5;
  uint8_t* set = sbe_set(c, ki.grp);
  uint32_t tw[13];                                    // tag block words: key[4] (0..7), ver[4] (8..11), masks (12)
#pragma unroll
  for (int k = 0; k < 3; k++) { tw[4 * k] = pf.t[k].x; tw[4 * k + 1] = pf.t[k].y; tw[4 * k + 2] = pf.t[k].z; tw[4 * k + 3] = pf.t[k].w; }
  tw[12] = pf.t[3].x;
  const uint32_t valid = tw[12] & 15u, dirty = (tw[12] >> 8) & 15u;
  int hit = -1;
#pragma unroll
  for (int i = 3; i >= 0; i--)
    if (((valid >> i) & 1u) && tw[2 * i] == (uint32_t)key && tw[2 * i + 1] == (uint32_t)(key >> 32)) hit = i;
  uint32_t rw[2];                                     // the request's value
  ld_words_unaligned<2>(rec + W::VAL, rw);
  const uint8_t ack = type == 0 ? 7 : type == 1 ? 9 : type == 4 ? 13 : type == 5 ? 14 : 18;
  uint32_t* tag = (uint32_t*)set;
  if (hit >= 0) {
    ec_count(c, SBE_HIT);
    uint2* vp = (uint2*)(set + 64) + hit;
    if (commit) {                                     // :424-435 / :510-521: the reply echoes the client's ver
      *vp = make_uint2(rw[0], rw[1]);
      tag[8 + hit] = tw[8 + hit] + 1;
      if (!((dirty >> hit) & 1u)) tag[12] = tw[12] | (0x100u << hit);
      rec[W::TYPE] = ack;
    } else {                                          // :159-167, :276-284, :615-623: a warm-up hit is kGrantShared
      const uint2 v = __ldcg(vp);
      const uint32_t w[2] = {v.x, v.y};
      st_words_unaligned<2>(rec + W::VAL, w);
      st_u32_unaligned(rec + W::VER, tw[8 + hit]);
      rec[W::TYPE] = type == 1 ? 9 : 7;
    }
    return;
  }
  // a miss: XDP picks the victim (first invalid, else first clean, else 0: :189-198) and passes the request up
  ec_count(c, SBE_TABLE);
  int vic = 0;
  {
    const uint32_t inv = ~valid & 15u, cln = ~dirty & 15u;
    if (inv) vic = __ffs(inv) - 1;
    else if (cln) vic = __ffs(cln) - 1;
  }
  if (((valid & dirty) >> vic) & 1u) {                // shard_user.c:145,154,163,172,180: kvs_set(key2, val2, ver2)
    const uint2 ov = __ldcg((const uint2*)(set + 64) + vic);
    const uint32_t ow[2] = {ov.x, ov.y};
    const uint64_t okey = ((uint64_t)tw[2 * vic + 1] << 32) | tw[2 * vic];
    uint32_t ignored;                                 // a cached key came from the table: it is there
    (void)kv_set_ver<8>(t, okey, fasthash64_u64(okey), ow, tw[8 + vic], ignored);
    ec_count(c, SBE_WRITEBACK);
  }
  uint32_t w[2] = {rw[0], rw[1]}, ver = 0;
  bool found;
  if (commit) {                                       // :165,173: kvs_set(key, val, 0) -> the table's new version
    found = kv_set_ver<8>(t, key, ki.h, w, 0, ver);
  } else {                                            // :147,156,182: kvs_get
    uint4 v[2];
    kv_prefetch_home<8>(c, table, ki.h, v);
    found = kv_find<8>(t, key, ki.h, v) != nullptr;
    w[0] = v[1].x; w[1] = v[1].y; ver = v[0].z;
    if (found) st_words_unaligned<2>(rec + W::VAL, w);
  }
  // A key the table lacks: the reference's kvs_get / kvs_set panic and the server stops.  Answered 0xFF; the counter
  // increment and the write-back above stay, and nothing is installed.
  if (!found) { mark_invalid<K_SMALLBANK_EBPF>(c, rec); return; }
  st_u32_unaligned(rec + W::VER, ver);
  rec[W::TYPE] = ack;
  *(uint2*)(set + 8 * vic) = make_uint2((uint32_t)key, (uint32_t)(key >> 32));   // TC install (:714-720), clean
  tag[8 + vic] = ver;
  *((uint2*)(set + 64) + vic) = make_uint2(w[0], w[1]);
  tag[12] = (valid | (1u << vic)) | ((dirty & ~(1u << vic)) << 8);
  ec_count(c, SBE_INSTALL);
}

// ---- bulk load (dint_load / dint_populate) and single-key inspection ------------------------------
template <int VALSZ>
__global__ void __launch_bounds__(256) k_kv_load(const Ctx c, int table, const uint64_t* keys, const uint8_t* vals, uint32_t n) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const KvTable& t = c.tbl[table];
  uint64_t key = keys[i];
  uint64_t h = fasthash64_u64(key);
  if (kv_group(c, table, h) == kNoGroup) return;   // another shard's key
  uint32_t w[Ent<VALSZ>::NW];
  const uint32_t* src = (const uint32_t*)(vals + (size_t)i * VALSZ);
#pragma unroll
  for (int k = 0; k < Ent<VALSZ>::NW; k++) w[k] = src[k];
  if (!kv_insert_words<VALSZ>(t, key, h, w)) atomicAdd(&c.counters[0], 1ULL);
}

// Every FULL entry of `from` for which keep(key, fasthash64(key)) holds is inserted into `to` with its version;
// tombstones vanish.  `from` may sit in a peer device's memory, and the caller sizes `to` for every key it receives.
// Filters: KeepAll (the tombstone rehash, kv_maintain), KeepOwner (a re-shard, reshard.cuh), RebuildKeep (a rebuild,
// rebuild.cuh).
template <int VALSZ, class Keep>
__global__ void __launch_bounds__(256) k_kv_move(const KvTable from, const KvTable to, const Keep keep) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= from.cap_mask; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t* e = from.entries + (i << from.ent_shift);
    uint4 v[Ent<VALSZ>::NV];
    kv_load_entry<VALSZ>(e, v);
    if (v[0].w != ENT_FULL) continue;
    const uint64_t key = ((uint64_t)v[0].y << 32) | v[0].x;
    const uint64_t h = fasthash64_u64(key);
    if (!keep(key, h)) continue;
    uint32_t w[Ent<VALSZ>::NW];
    const uint32_t* flat = (const uint32_t*)v;
#pragma unroll
    for (int k = 0; k < Ent<VALSZ>::NW; k++) w[k] = flat[4 + k];
    kv_insert_words<VALSZ>(to, key, h, w, v[0].z);   // (`to` has room for every key it receives: cannot fail)
  }
}
struct KeepAll {
  DINT_D bool operator()(uint64_t, uint64_t) const { return true; }
};

// out[d] += the FULL entries of table t that go to destination shard d, for every d of dests.all: dests(key,
// fasthash64(key)) is the bit mask of a row's destinations (OwnerDests, reshard.cuh; RebuildDests, rebuild.cuh).
// Destination tables are sized from these counts before a single row is inserted.
template <class Dests>
__global__ void __launch_bounds__(kThreads) k_kv_count_rows(const KvTable t, const Dests dests, unsigned long long* out) {
  __shared__ unsigned long long s_cnt[kMaxShards];
  if (threadIdx.x < kMaxShards) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t end = (t.cap_mask + 32) / 32 * 32;              // whole warps: the ballots below need every lane
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t m = 0;
    if (i <= t.cap_mask) {
      const uint4 v = __ldcg((const uint4*)(t.entries + (i << t.ent_shift)));   // {key, ver, meta}
      const uint64_t key = ((uint64_t)v.y << 32) | v.x;
      if (v.w == ENT_FULL) m = dests(key, fasthash64_u64(key));
    }
    for (uint32_t a = dests.all; a; a &= a - 1) {
      const uint32_t d = __ffs(a) - 1;
      const uint32_t n = __popc(__ballot_sync(0xffffffffu, (m >> d) & 1u));
      if (n && lane_id() == 0) atomicAdd(&s_cnt[d], (unsigned long long)n);
    }
  }
  __syncthreads();
  if (threadIdx.x < kMaxShards && s_cnt[threadIdx.x]) atomicAdd(&out[threadIdx.x], s_cnt[threadIdx.x]);
}

template <int VALSZ>
__global__ void k_kv_get1(const Ctx c, int table, uint64_t key, uint32_t* out /* [0]=found [1]=ver [2..]=val */) {
  uint4 v[Ent<VALSZ>::NV];
  const uint64_t h = fasthash64_u64(key);
  kv_prefetch_home<VALSZ>(c, table, h, v);
  uint8_t* e = kv_find<VALSZ>(c.tbl[table], key, h, v);
  out[0] = e ? 1u : 0u;
  if (e) {
    out[1] = v[0].z;
    const uint32_t* flat = (const uint32_t*)v;
    for (int k = 0; k < Ent<VALSZ>::NW; k++) out[2 + k] = flat[4 + k];
  }
}
#endif  // __CUDACC__

// =================================== host side ======================================================
struct KvHost {
  uint64_t capacity = 0;
  uint32_t hash_size = 0;     // the reference's bucket count for this table
};

inline uint32_t next_log2(uint64_t x) {
  uint32_t l = 0;
  while ((1ULL << l) < x) l++;
  return l;
}

// Sizes follow the reference: store kvs_init(kSubscriberNum*18/4) (store/udp/server.cc:113); tatp
// kvs_init(S*3/2/4, S*3/2/4, S*15/4/4, S*15/4/4, S*45/8/4) (tatp/udp/server_shard.cc:75-79); smallbank
// kvs_init(A*3/2/4) x2 (smallbank/udp/server_shard.cc:72-73).  The group modulus is the bucket count
// for store and kKeysPerEntry*hash_size (lock_hash) for tatp / smallbank.
// tatp_ebpf: the eBPF server's sizes (tatp/ebpf/utils.h:17-21: call_forwarding has S*15/4/4 buckets); its rows live in
// chained tables (kv.cuh, K_TATP_EBPF), so the open-addressing tables are left at their minimum size, unused.
struct KvPlan {
  uint32_t nt = 0, valsz = 40, lock_mul = 4;
  uint32_t hs[kMaxTables] = {0};     // bucket counts
  uint32_t lg[kMaxTables] = {0};     // log2 capacities a shard of `cf` is created with
};
inline int kv_plan(int kind, const dint_cfg& cf, bool tatp_ebpf, KvPlan& p) {
  const uint64_t S = cf.subs_sizing, Sp = cf.subs_populate, A = cf.accts_sizing, Ap = cf.accts_populate;
  double expect[kMaxTables] = {0};
  if (kind == DINT_STORE) {
    p.nt = 1; p.hs[0] = (uint32_t)(S * 18 / 4); expect[0] = 12.0 * Sp; p.lock_mul = 1;
  } else if (kind == DINT_TATP) {
    p.nt = 5;
    p.hs[0] = p.hs[1] = (uint32_t)(S * 3 / 2 / 4);
    p.hs[2] = p.hs[3] = (uint32_t)(S * 15 / 4 / 4);
    p.hs[4] = tatp_ebpf ? (uint32_t)(S * 15 / 4 / 4) : (uint32_t)(S * 45 / 8 / 4);
    expect[0] = expect[1] = 1.0 * Sp; expect[2] = expect[3] = 2.5 * Sp; expect[4] = 3.75 * Sp;
  } else if (kind == DINT_SMALLBANK) {
    p.nt = 2; p.valsz = 8;
    p.hs[0] = p.hs[1] = (uint32_t)(A * 3 / 2 / 4);
    expect[0] = expect[1] = 1.0 * Ap;
  } else return DINT_EINVAL;
  for (uint32_t t = 0; t < p.nt; t++) {
    if (p.hs[t] == 0) return DINT_EINVAL;
    uint32_t lg = tatp_ebpf ? 10 : cf.kv_capacity_log2[t];
    if (lg == 0) {
      double need = 2.0 * expect[t] / cf.n_shards * 1.05 + 1024;
      lg = next_log2((uint64_t)need);
      if (lg < 10) lg = 10;
    }
    if (lg > 34) return DINT_EINVAL;
    p.lg[t] = lg;
  }
  return DINT_OK;
}
// log2 capacity of a table filled with `keys` keys at once (re-shard, rebuild): at least lg, and large enough that the
// keys load it to <= 35 %, so kv_maintain does not rehash it on the next call; > 34 = too many keys
inline uint32_t kv_fit_log2(uint32_t lg, uint64_t keys) {
  while (lg <= 34 && keys * 20 > (7ULL << lg)) lg++;
  return lg;
}

template <typename AllocFn>
int kv_create_tables(int kind, const dint_cfg& cf, Ctx& c, KvHost* kv, uint64_t* groups_out, AllocFn alloc, bool tatp_ebpf = false) {
  KvPlan P;
  if (kv_plan(kind, cf, tatp_ebpf, P) != DINT_OK) return DINT_EINVAL;
  const uint32_t nt = P.nt, valsz = P.valsz, lock_mul = P.lock_mul;
  const uint32_t* hs = P.hs;
  c.n_tables = nt;
  uint64_t base = 0;
  for (uint32_t t = 0; t < nt; t++) {
    KvTable& T = c.tbl[t];
    const uint32_t lg = P.lg[t];
    T.cap_log2 = lg;
    T.cap_mask = (1ULL << lg) - 1;
    T.ent_shift = (valsz == 40) ? 6 : 5;
    uint64_t mod = (uint64_t)hs[t] * lock_mul;
    if (mod >= 0xffffffffULL) return DINT_EINVAL;
    T.lock_mod = make_fastmod((uint32_t)mod);
    T.grp_base = (uint32_t)base;
    T.n_groups = (uint32_t)((mod + cf.n_shards - 1) / cf.n_shards);
    base += T.n_groups;
    void* p = nullptr;
    int rc = alloc(&p, (size_t)(1ULL << lg) << T.ent_shift);
    if (rc) return rc;
    T.entries = (uint8_t*)p;
    if (t == 0) {                                    // {live, used} of every table side by side: one copy publishes them all
      rc = alloc(&p, 16 * kMaxTables);
      if (rc) return rc;
      c.tbl[0].live = (unsigned long long*)p;
    }
    T.live = c.tbl[0].live + 2 * t;
    kv[t].capacity = 1ULL << lg;
    kv[t].hash_size = hs[t];
  }
  // group state: tatp = one lock bit per group; smallbank = {num_ex, num_sh} per group
  void* p = nullptr;
  if (kind == DINT_TATP) {
    int rc = alloc(&p, ((base + 31) / 32) * 4);
    if (rc) return rc;
    c.lockbits = (uint32_t*)p;
  } else if (kind == DINT_SMALLBANK) {
    int rc = alloc(&p, base * sizeof(uint2));
    if (rc) return rc;
    c.cnt2 = (uint2*)p;
  }
  *groups_out = base;
  return DINT_OK;
}

// ---- deterministic population: the reference's populate_* generators, emitted as (key, val) batches --
inline uint32_t kv_fastrand(uint64_t* seed) {       // store/udp/tatp.h:31-34, tatp/udp/tatp.h:32-35
  *seed = *seed * 1103515245ULL + 12345ULL;
  return (uint32_t)(*seed >> 32);
}
inline uint64_t tatp_sub_nbr_of(uint32_t s_id) {    // tatp/udp/tatp.h:17-25,132-144: 3 x 12-bit BCD groups
  uint64_t r = 0;
  for (int g = 0; g < 3; g++) {
    uint32_t i = s_id % 1000;
    s_id /= 1000;
    r |= ((uint64_t)(((i / 100) % 10) << 8 | ((i / 10) % 10) << 4 | (i % 10))) << (12 * g);
  }
  return r;
}
inline int tatp_select_types(uint64_t* seed, uint8_t out[4]) {   // tatp/udp/tatp.h:254-282 with values {1,2,3,4}
  bool used[8] = {false};
  int want = (int)(kv_fastrand(seed) % 4) + 1, got = 0;
  while (got < want) {
    uint8_t v = (uint8_t)((kv_fastrand(seed) % 4) + 1);
    if (used[v]) continue;
    used[v] = true;
    out[got++] = v;
  }
  return got;
}

// ---- tatp / smallbank replica placement (txn_clients.cuh: primary p = key % G, backups (p + 1) % G and (p + 2) % G) -----
// G is the placement's shard count: dint_cfg.txn_shards > 3 ? txn_shards : 3 for one engine (with three shards or fewer
// every shard holds every key), the shard count for a cluster.  p = key % G.
// The role of `shard` for the keys of residue p: 0 primary, 1 or 2 backup, > 2 not one of their replicas.
DINT_HD uint32_t txn_role(uint32_t p, uint32_t G, uint32_t shard) { return (shard + G - p) % G; }
// The shard a rebuild copies the rows of residue p from when the shards of bit mask `lost` are lost: the surviving
// replica with the lowest role, or -1 when every replica is lost (dint_cluster_rebuild).
DINT_HD int rebuild_source(uint32_t p, uint32_t G, uint32_t lost) {
  for (uint32_t i = 0; i < 3; i++) {
    const uint32_t s = (p + i) % G;                  // the shard of role i: txn_role(p, G, s) == i
    if (!((lost >> s) & 1u)) return (int)s;
  }
  return -1;
}

struct KvBatch {
  std::vector<uint64_t> keys;
  std::vector<uint8_t> vals;
  uint32_t valsz;
  int table;
  std::function<int(int, const uint64_t*, const void*, uint64_t)> sink;
  int rc = 0;
  KvBatch(int table_, uint32_t valsz_, std::function<int(int, const uint64_t*, const void*, uint64_t)> s, const dint_cfg& cf)
      : valsz(valsz_), table(table_), sink(std::move(s)), G(cf.txn_shards), gid(cf.txn_shard_id) {
    keys.reserve(1 << 20);
    vals.reserve((size_t)valsz << 20);
  }
  uint32_t G = 0, gid = 0;                           // replica filter (dint_cfg.txn_shards / txn_shard_id)
  std::vector<uint8_t> dummy;
  uint8_t* add(uint64_t key) {                       // returns the zeroed value slot
    if (G > 3 && txn_role((uint32_t)(key % G), G, gid) > 2) {   // not one of this key's three replica holders: drop it
      dummy.assign(valsz, 0);
      return dummy.data();
    }
    if (keys.size() == (1u << 20)) flush();
    keys.push_back(key);
    vals.resize(vals.size() + valsz, 0);
    return vals.data() + vals.size() - valsz;
  }
  void flush() {
    if (!keys.empty() && rc == 0) rc = sink(table, keys.data(), vals.data(), keys.size());
    keys.clear();
    vals.clear();
  }
};

// Bytes the reference never assigns (stack structs copied whole: store_val_t.numberx[1..],
// tatp_sub_val_t.sub_nbr_unused, tatp_accinf_val_t.data2.., tatp_specfac_val_t.error_cntl/data_a/
// data_b[1..], tatp_callfwd_val_t.numberx[1..]) are zero here -- as they read back from oracle/_ref.
inline int kv_populate(int kind, const dint_cfg& cf, std::function<int(int, const uint64_t*, const void*, uint64_t)> sink) {
  if (kind == DINT_STORE) {                          // store/udp/tatp.h:45-66
    KvBatch b(0, 40, sink, cf);
    uint64_t seed = 0xdeadbeef;
    for (uint32_t s = 0; s < cf.subs_populate; s++)
      for (uint64_t sf = 1; sf <= 4; sf++)
        for (uint64_t st = 0; st <= 16; st += 8) {
          uint8_t* v = b.add((uint64_t)s | (sf << 32) | (st << 40));
          v[0] = (uint8_t)((kv_fastrand(&seed) % 24) + 1);   // end_time
          v[1] = 0x5a;                                       // numberx[0] = kValMagic
        }
    b.flush();
    return b.rc;
  }
  if (kind == DINT_SMALLBANK) {                      // smallbank/udp/smallbank.h:105-127
    KvBatch sav(0, 8, sink, cf), chk(1, 8, sink, cf);
    const float bal = 1000000000.0f;
    for (uint32_t a = 0; a < cf.accts_populate; a++) {
      uint8_t* v = sav.add(a);
      uint32_t magic = 97;
      memcpy(v, &magic, 4); memcpy(v + 4, &bal, 4);
      v = chk.add(a);
      magic = 98;
      memcpy(v, &magic, 4); memcpy(v + 4, &bal, 4);
    }
    sav.flush(); chk.flush();
    return sav.rc ? sav.rc : chk.rc;
  }
  if (kind != DINT_TATP) return DINT_OK;
  const uint32_t N = cf.subs_populate;
  {                                                  // tatp/udp/tatp.h:285-311 subscriber
    KvBatch b(0, 40, sink, cf);
    uint64_t seed = 0xdeadbeef;
    for (uint32_t s = 0; s < N; s++) {
      uint8_t* v = b.add(s);
      uint64_t nbr = tatp_sub_nbr_of(s);
      memcpy(v, &nbr, 8);
      for (int i = 0; i < 5; i++) v[15 + i] = (uint8_t)kv_fastrand(&seed);    // hex[5]
      for (int i = 0; i < 10; i++) v[20 + i] = (uint8_t)kv_fastrand(&seed);   // bytes[10]
      uint16_t bits = (uint16_t)kv_fastrand(&seed);
      memcpy(v + 30, &bits, 2);
      uint32_t msc = 97, vlr = kv_fastrand(&seed);
      memcpy(v + 32, &msc, 4); memcpy(v + 36, &vlr, 4);
    }
    b.flush();
    if (b.rc) return b.rc;
  }
  {                                                  // :314-329 secondary subscriber
    KvBatch b(1, 40, sink, cf);
    for (uint32_t s = 0; s < N; s++) {
      uint8_t* v = b.add(tatp_sub_nbr_of(s));
      memcpy(v, &s, 4);
      v[4] = 98;
    }
    b.flush();
    if (b.rc) return b.rc;
  }
  {                                                  // :332-357 access info
    KvBatch b(2, 40, sink, cf);
    uint64_t seed = 0xdeadbeef;
    for (uint32_t s = 0; s < N; s++) {
      uint8_t ty[4];
      int n = tatp_select_types(&seed, ty);
      for (int i = 0; i < n; i++) b.add((uint64_t)s | ((uint64_t)ty[i] << 32))[0] = 99;
    }
    b.flush();
    if (b.rc) return b.rc;
  }
  {                                                  // :360-412 special facility + call forwarding
    KvBatch sf(3, 40, sink, cf), cfw(4, 40, sink, cf);
    uint64_t seed = 0xdeadbeef;
    for (uint32_t s = 0; s < N; s++) {
      uint8_t ty[4];
      int n = tatp_select_types(&seed, ty);
      for (int i = 0; i < n; i++) {
        uint64_t t = ty[i];
        uint8_t* v = sf.add((uint64_t)s | (t << 32));
        v[3] = 100;
        v[0] = (kv_fastrand(&seed) % 100 < 85) ? 1 : 0;
        for (uint64_t st = 0; st <= 16; st += 8) {
          if (kv_fastrand(&seed) % 2 == 0) continue;
          uint8_t* w = cfw.add((uint64_t)s | (t << 32) | (st << 40));
          w[1] = 101;
          w[0] = (uint8_t)((kv_fastrand(&seed) % 24) + 1);
        }
      }
    }
    sf.flush(); cfw.flush();
    return sf.rc ? sf.rc : cfw.rc;
  }
}

// The eBPF store's population: its client's kInsert stream (store/caladan/client_ebpf.cc:137-180), as ONE sequential
// server sees it -- 600 populate threads (:282) in thread order, each over its slice of the subscribers with fastrand
// restarting at 0xdeadbeef (:138).  Same keys and value bytes as kv_populate's store, in another order and other draws.
inline int store_ebpf_populate(const dint_cfg& cf, std::function<int(int, const uint64_t*, const void*, uint64_t)> sink) {
  KvBatch b(0, 40, sink, cf);
  const uint32_t S = cf.subs_populate, threads = 600, slice = S / threads;
  for (uint32_t w = 0; w < threads; w++) {
    uint64_t seed = 0xdeadbeef;
    const uint32_t lo = w * slice, hi = (w == threads - 1) ? S : (w + 1) * slice;
    for (uint32_t s = lo; s < hi; s++)
      for (uint64_t sf = 1; sf <= 4; sf++)
        for (uint64_t st = 0; st <= 16; st += 8) {
          uint8_t* v = b.add((uint64_t)s | (sf << 32) | (st << 40));
          v[1] = 0x5a;                                       // numberx[0] = kValMagic
          v[0] = (uint8_t)((kv_fastrand(&seed) % 24) + 1);   // end_time
        }
  }
  b.flush();
  return b.rc;
}

// The eBPF TATP server's population: its client's insert stream (tatp/caladan/client_ebpf_shard.cc:96-339) as ONE
// sequential server sees it -- 600 populate threads (:1658) in thread order, each over its slice of the subscribers with
// fastrand restarting at 0xdeadbeef (:97) and running on through the four tables of the slice.  Same keys and value
// layouts as kv_populate's tatp, in another order and with other draws.  Rows of different (table, bucket) pairs never
// interact, so each table's rows are handed to `sink` in their own batches, in stream order.
inline int tatp_ebpf_populate(const dint_cfg& cf, std::function<int(int, const uint64_t*, const void*, uint64_t)> sink) {
  const uint32_t S = cf.subs_populate, threads = 600, slice = S / threads;
  KvBatch b0(0, 40, sink, cf), b1(1, 40, sink, cf), b2(2, 40, sink, cf), b3(3, 40, sink, cf), b4(4, 40, sink, cf);
  for (uint32_t w = 0; w < threads; w++) {
    uint64_t seed = 0xdeadbeef;
    const uint32_t lo = w * slice, hi = (w == threads - 1) ? S : (w + 1) * slice;
    for (uint32_t s = lo; s < hi; s++) {             // subscriber
      uint8_t* v = b0.add(s);
      uint64_t nbr = tatp_sub_nbr_of(s);
      memcpy(v, &nbr, 8);
      for (int i = 0; i < 5; i++) v[15 + i] = (uint8_t)kv_fastrand(&seed);
      for (int i = 0; i < 10; i++) v[20 + i] = (uint8_t)kv_fastrand(&seed);
      uint16_t bits = (uint16_t)kv_fastrand(&seed);
      memcpy(v + 30, &bits, 2);
      uint32_t msc = 97, vlr = kv_fastrand(&seed);
      memcpy(v + 32, &msc, 4); memcpy(v + 36, &vlr, 4);
    }
    for (uint32_t s = lo; s < hi; s++) {             // secondary subscriber
      uint8_t* v = b1.add(tatp_sub_nbr_of(s));
      memcpy(v, &s, 4);
      v[4] = 98;
    }
    for (uint32_t s = lo; s < hi; s++) {             // access info
      uint8_t ty[4];
      int n = tatp_select_types(&seed, ty);
      for (int i = 0; i < n; i++) b2.add((uint64_t)s | ((uint64_t)ty[i] << 32))[0] = 99;
    }
    for (uint32_t s = lo; s < hi; s++) {             // special facility, each followed by its call forwarding rows
      uint8_t ty[4];
      int n = tatp_select_types(&seed, ty);
      for (int i = 0; i < n; i++) {
        const uint64_t t = ty[i];
        uint8_t* v = b3.add((uint64_t)s | (t << 32));
        v[3] = 100;
        v[0] = (kv_fastrand(&seed) % 100 < 85) ? 1 : 0;
        for (uint64_t st = 0; st <= 16; st += 8) {
          if (kv_fastrand(&seed) % 2 == 0) continue;
          uint8_t* x = b4.add((uint64_t)s | (t << 32) | (st << 40));
          x[1] = 101;
          x[0] = (uint8_t)((kv_fastrand(&seed) % 24) + 1);
        }
      }
    }
  }
  for (KvBatch* b : {&b0, &b1, &b2, &b3, &b4}) b->flush();
  return b0.rc ? b0.rc : b1.rc ? b1.rc : b2.rc ? b2.rc : b3.rc ? b3.rc : b4.rc;
}

}  // namespace dint
