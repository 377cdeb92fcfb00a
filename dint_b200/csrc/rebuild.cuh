// Rebuilding lost tatp / smallbank shards from their replicas (dint_cluster_rebuild, include/dint_b200.h): the device
// half.
//
// Placement.  The clients write every row of key k to its three replicas, shards (k % G + i) % G of roles i = 0, 1, 2
// (txn_role / rebuild_source, kv.cuh), and population places rows the same way, so each shard holds every row of the
// keys it is a replica of.  For a set of lost shards, the source of key k is its surviving replica with the lowest role
// (rebuild_source).  That depends on (k, G, lost) alone, so every row reaches every lost replica of its key exactly
// once, from one source, and the result does not depend on the launch order.
//
//   RebuildDests   k_kv_count_rows's filter (kv.cuh): the lost shards one source gives a row to, so that every
//                  destination table is sized to hold its rows before a single one is inserted.
//   RebuildKeep    k_kv_move's filter (kv.cuh): one source table's rows for one lost shard; each row is inserted with
//                  its version, tombstones are not copied.
//
// k_kv_move runs on the destination's device; a source shard on another GPU is read through peer memory.  Only the
// sources within two positions of a lost shard hold its keys, and only those are read.
//
// Re-placing onto another shard count (dint_cluster_reshard_txn).  At a drained point every replica of a key holds the
// same row; the source of key k is its old primary, shard k % G, so the result does not depend on the launch order.
// Destination shard j of G' receives every key it replicates under G', (k % G' + i) % G' for i = 0, 1, 2 (for G' = 1
// only shard 0; each key still gets one row).
//
//   ReplicaDests   k_kv_count_rows's filter: the destinations of one source's primary rows.
//   ReplicaKeep    k_kv_move's filter: one source's primary rows that destination dst replicates.
//   k_locks_held   the held lock groups of one shard: the call refuses a source with any, since a client that holds a
//                  lock is mid-transaction and its replicas may differ.
#pragma once
#include "kernels.cuh"
#include "kv.cuh"

namespace dint {

struct RebuildKeep {
  FastMod gmod;                    // G, the cluster's shard count
  uint32_t G, lost, src, dst;      // lost: bit mask; src: the shard read; dst: the lost shard filled
#ifdef __CUDACC__
  // key's row goes from src to dst: src is its source and dst one of its replicas
  DINT_D bool operator()(uint64_t key, uint64_t) const {
    const uint32_t p = fast_mod(key, gmod);
    return rebuild_source(p, G, lost) == (int)src && txn_role(p, G, dst) <= 2;
  }
#endif
};
struct RebuildDests {
  FastMod gmod;
  uint32_t G, all, src;            // all: the lost shards (bit mask); src: the shard read
#ifdef __CUDACC__
  // the lost replicas of key's row, when src is its source
  DINT_D uint32_t operator()(uint64_t key, uint64_t) const {
    const uint32_t p = fast_mod(key, gmod);
    uint32_t dests = 0;
    if (rebuild_source(p, G, all) == (int)src)
      for (uint32_t m = all; m; m &= m - 1) {
        const uint32_t d = __ffs(m) - 1;
        if (txn_role(p, G, d) <= 2) dests |= 1u << d;
      }
    return dests;
  }
#endif
};

struct ReplicaKeep {
  FastMod gmod, g2mod;             // G, G': the source and destination shard counts
  uint32_t G2, src, dst;           // src: the shard read; dst: the destination shard filled
#ifdef __CUDACC__
  DINT_D bool operator()(uint64_t key, uint64_t) const {
    return fast_mod(key, gmod) == src && txn_role(fast_mod(key, g2mod), G2, dst) <= 2;
  }
#endif
};
struct ReplicaDests {
  FastMod gmod, g2mod;
  uint32_t G2, all, src;           // all = (1 << G') - 1; src: the shard read
  // the destinations of key's row when src is its old primary (also the host test hook's answer)
  DINT_HD uint32_t operator()(uint64_t key, uint64_t) const {
    if (fast_mod(key, gmod) != src) return 0;
    const uint32_t p = fast_mod(key, g2mod);
    uint32_t dests = 0;
    for (uint32_t i = 0; i < 3; i++) dests |= 1u << ((p + i) % G2);
    return dests;
  }
};

#ifdef __CUDACC__
// out += the held lock groups of one tatp / smallbank shard: the set bits of `bits` (tatp, one bit per group), or the
// groups of `cnt2` (smallbank, {num_ex, num_sh}) that are not {0, 0}; n groups.  One atomic per CTA.
__global__ void __launch_bounds__(kThreads) k_locks_held(const uint32_t* bits, const uint2* cnt2, uint64_t n, unsigned long long* out) {
  __shared__ uint32_t wsum[kThreads / 32];
  uint32_t held = 0;
  const uint64_t m = bits ? (n + 31) / 32 : n;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t)gridDim.x * blockDim.x) {
    if (bits) held += __popc(__ldcg(bits + i));
    else { const uint2 v = __ldcg(cnt2 + i); held += (v.x | v.y) != 0; }
  }
  held = __reduce_add_sync(0xffffffffu, held);
  if (lane_id() == 0) wsum[threadIdx.x / 32] = held;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long sum = 0;
    for (uint32_t w = 0; w < kThreads / 32; w++) sum += wsum[w];
    if (sum) atomicAdd(out, sum);
  }
}
#endif

}  // namespace dint
