// Re-sharding a lock_2pl, lock_fasst or store cluster onto another shard count (dint_cluster_reshard,
// include/dint_b200.h): the device half.
//
// Ownership.  A cluster of G shards answers like ONE server: shard r owns the global lock slots / buckets s with
// s % G == r and keeps s at local index s / G (to_local_group).  A destination of G' shards splits the same global
// numbering the other way, so destination shard j, local g', is global s = g' G' + j, read from source shard s % G at
// local s / G.  Every destination element is found from its own global id: the gathers below write each destination
// word exactly once, need no atomics and give the same bytes whatever the launch order.  The only atomics are those of
// the KV inserts (kv_insert_words, through k_kv_move), which claim free table entries.
//
//   k_reshard_lock    lock_2pl {num_ex, num_sh} per group, or lock_fasst's version per group and its lock bits: one
//                     bit per local group, gathered 32 destination groups per warp and stored as one word (ballot).
//                     A lock held before the move is held after it.
//   k_reshard_sets    the store's eBPF cache tier: one 256-byte set per bucket moves whole (keys, versions, valid and
//                     dirty masks, bloom word, values), 16 threads per set.
//   the store's table entries are first counted per destination shard (bucket % G') by k_kv_count_rows (kv.cuh) with
//   OwnerDests, so that every destination table is sized to hold its keys before a single one is inserted, then move
//   through k_kv_move (kv.cuh) with KeepOwner: one pass per (source table, destination), each FULL entry inserted with
//   its version; tombstones are dropped and {live, used} recounted.
//
// The gathers and k_kv_move run on the destination's device; a source shard on another GPU is read through peer memory.
#pragma once
#include "kernels.cuh"
#include "kv.cuh"

namespace dint {

struct ReshardArgs {
  uint64_t src[kMaxShards];        // the source shards' array (device addresses; peer memory when on another GPU)
  uint64_t src_bits[kMaxShards];   // lock_fasst: the source shards' lock bits
  FastMod src_div;                 // G, the source shard count
  uint32_t G, G2, j;               // source / destination shard counts, this destination shard
  uint32_t n_local;                // the destination shard's local groups
  uint64_t n_global;               // global lock slots (lock kinds) or buckets (store)
  void* dst;
  uint32_t* dst_bits;              // lock_fasst
};

// A store key's bucket is fasthash64(key) % the table's bucket count (bucket_mod); destination shard bucket % n owns it.
struct KeepOwner {                 // k_kv_move: the keys destination shard `owner` of n receives
  FastMod bucket_mod;
  uint32_t n, owner;
#ifdef __CUDACC__
  DINT_D bool operator()(uint64_t, uint64_t h) const { return fast_mod(h, bucket_mod) % n == owner; }
#endif
};
struct OwnerDests {                // k_kv_count_rows: every key to its owner of n; all = (1 << n) - 1
  FastMod bucket_mod;
  uint32_t n, all;
#ifdef __CUDACC__
  DINT_D uint32_t operator()(uint64_t, uint64_t h) const { return 1u << (fast_mod(h, bucket_mod) % n); }
#endif
};

#ifdef __CUDACC__
// the source shard and local index of destination local group g (global g G' + j); false past the global range
DINT_D bool reshard_src(const ReshardArgs& a, uint64_t g, uint32_t& r, uint64_t& l) {
  const uint64_t s = g * a.G2 + a.j;
  if (g >= a.n_local || s >= a.n_global) return false;
  l = fast_div(s, a.src_div);
  r = (uint32_t)(s - l * a.G);
  return true;
}

template <int KIND>
__global__ void __launch_bounds__(kThreads) k_reshard_lock(const ReshardArgs a) {
  const uint64_t end = ((uint64_t)a.n_local + 31) / 32 * 32;   // whole warps: the ballot needs every lane
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < end; g += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t r = 0, bit = 0;
    uint64_t l = 0;
    if (reshard_src(a, g, r, l)) {
      if constexpr (KIND == K_LOCK2PL) {
        ((uint2*)a.dst)[g] = __ldcg((const uint2*)a.src[r] + l);
      } else {
        ((uint32_t*)a.dst)[g] = __ldcg((const uint32_t*)a.src[r] + l);
        bit = (__ldcg((const uint32_t*)a.src_bits[r] + (l >> 5)) >> (l & 31)) & 1u;
      }
    }
    if constexpr (KIND == K_FASST) {
      const uint32_t word = __ballot_sync(0xffffffffu, bit);
      if (lane_id() == 0 && g < a.n_local) a.dst_bits[g >> 5] = word;
    }
  }
}

__global__ void __launch_bounds__(kThreads) k_reshard_sets(const ReshardArgs a) {
  constexpr uint32_t kVecs = kEcSetBytes / 16;
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < (uint64_t)a.n_local * kVecs;
       t += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t r;
    uint64_t l;
    if (!reshard_src(a, t / kVecs, r, l)) continue;
    ((uint4*)a.dst)[t] = __ldcg((const uint4*)a.src[r] + l * kVecs + t % kVecs);
  }
}
#endif  // __CUDACC__

}  // namespace dint
