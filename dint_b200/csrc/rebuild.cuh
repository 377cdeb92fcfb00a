// Rebuilding lost tatp / smallbank shards from their replicas (dint_cluster_rebuild, include/dint_b200.h): the device
// half.
//
// Placement.  The clients write every row of key k to its three replicas, shards (k % G + i) % G of roles i = 0, 1, 2
// (txn_role / rebuild_source, kv.cuh), and population places rows the same way, so each shard holds every row of the
// keys it is a replica of.  For a set of lost shards, the source of key k is its surviving replica with the lowest role
// (rebuild_source).  That depends on (k, G, lost) alone, so every row reaches every lost replica of its key exactly
// once, from one source, and the result does not depend on the launch order.
//
//   k_rebuild_count   the FULL entries of one source table that this source gives each lost shard, so that every
//                     destination table is sized to hold its rows before a single one is inserted.
//   k_rebuild_rows    one source table's rows for one lost shard: k_kv_rehash's loop (kv_move_rows) with the rebuild's
//                     filter (RebuildKeep); each row is inserted with its version, tombstones are not copied.
//
// The kernels run on the destination's device; a source shard on another GPU is read through peer memory.  Only the
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
  DINT_D bool operator()(uint64_t key) const {
    const uint32_t p = fast_mod(key, gmod);
    return rebuild_source(p, G, lost) == (int)src && txn_role(p, G, dst) <= 2;
  }
#endif
};

#ifdef __CUDACC__
// out[d] += the FULL entries of table t that shard k.src sources for lost shard d (k.dst unused)
__global__ void __launch_bounds__(kThreads) k_rebuild_count(const KvTable t, const RebuildKeep k, unsigned long long* out) {
  __shared__ unsigned long long s_cnt[kMaxShards];
  if (threadIdx.x < kMaxShards) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  const uint64_t end = (t.cap_mask + 32) / 32 * 32;              // whole warps: the ballots below need every lane
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t dests = 0;
    if (i <= t.cap_mask) {
      const uint4 v = __ldcg((const uint4*)(t.entries + (i << t.ent_shift)));   // {key, ver, meta}
      if (v.w == ENT_FULL) {
        const uint32_t p = fast_mod(((uint64_t)v.y << 32) | v.x, k.gmod);
        if (rebuild_source(p, k.G, k.lost) == (int)k.src)
          for (uint32_t m = k.lost; m; m &= m - 1) {
            const uint32_t d = __ffs(m) - 1;
            if (txn_role(p, k.G, d) <= 2) dests |= 1u << d;
          }
      }
    }
    for (uint32_t m = k.lost; m; m &= m - 1) {
      const uint32_t d = __ffs(m) - 1;
      const uint32_t n = __popc(__ballot_sync(0xffffffffu, (dests >> d) & 1u));
      if (n && lane_id() == 0) atomicAdd(&s_cnt[d], (unsigned long long)n);
    }
  }
  __syncthreads();
  if (threadIdx.x < kMaxShards && s_cnt[threadIdx.x]) atomicAdd(&out[threadIdx.x], s_cnt[threadIdx.x]);
}

template <int VALSZ>
__global__ void __launch_bounds__(256) k_rebuild_rows(const KvTable from, const KvTable to, const RebuildKeep k) {
  kv_move_rows<VALSZ, RebuildKeep>(from, to, 0, 0, &k);
}
#endif  // __CUDACC__

}  // namespace dint
