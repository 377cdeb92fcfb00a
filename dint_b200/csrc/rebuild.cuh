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

}  // namespace dint
