// Multi-GPU dispatch / combine: stable partition of a batch of wire records by owner shard, written straight
// into fixed-capacity slabs (local memory, or the owners' receive buffers over NVLink), and its inverse.
//
//   k_route_dispatch  ONE launch, ONE pass over the batch.  Tiles (2048 records; 256 for the 23/53/55-byte kinds) are
//            handed out in index order by a ticket counter.  Per tile: owner shard of every record (hash of the key,
//            the slot ONE server would compute, modulo the shard count -- or the client-chosen shard), the tile's
//            per-shard counts, and the first slot of the tile's run in every slab from a two-level LOOK-BACK over
//            the preceding tiles' published counts (single-pass prefix sum: a tile publishes its counts at once, sums
//            those of the tiles before it in its group of 32 and those of the groups before its own -- two windows of
//            32 loads, never a wait for somebody else's prefix).  The tile is partitioned in
//            shared memory into one run per shard, each run placed at the alignment of its destination so that it
//            leaves with 16-byte stores.  Slots past a slab's total become padding records; the last CTA to finish
//            raises the epoch flags of the peers (release, system scope) when the slabs live in peer memory.
//
// The combine reads, per tile, one contiguous run per shard from the reply slabs and reassembles the tile in
// request order; its only per-record state is the owner byte and, per tile, the first slot of each run.
//
// The reference does this on the CLIENT (key % 3 / lock-id hashing before sendto, e.g.
// tatp/caladan/client_ebpf_shard.cc: `key % kNumServers`); here any rank may receive any request.
#pragma once
#include "kernels.cuh"

namespace dint {
template <int MSG> struct RTile {
  // records per thread.  Small records: 8, i.e. 2048-record tiles, so that a batch of 2^20 records is 512 tiles = ONE wave
  // of the 4 CTAs per SM the kernels' 64 registers allow (with 1024-record tiles half of the CTAs had to take a second
  // tile after the first: the dispatch is a chain of latencies per tile, and its time was two chains)
  static constexpr int PER = MSG <= 12 ? 8 : 1;
  static constexpr int RECS = kThreads * PER;                    // records per tile
  static constexpr int BYTES = RECS * MSG;                       // a multiple of 16
  static constexpr int RUNS = BYTES + 16 * kMaxShards + 16;      // the partitioned copy: alignment gaps between runs
  static constexpr int SMEM = BYTES + 16 + RUNS;
};

struct RouteArgs {
  const uint8_t* req;        // dispatch: [n * MSG] wire records, 16-byte aligned
  const uint8_t* owner_in;   // dispatch: client-chosen shard per record, or nullptr = computed from the keys
  uint8_t* owner;            // [n] owner byte per record (dispatch writes, combine reads); 0xff = undeliverable
  uint32_t* tilebase;        // [n_tiles][kMaxShards] first slot of each tile's run in each slab
  unsigned long long* desc;  // dispatch scratch [n_tiles][4]: per-tile counts, self-validating words tagged with `seq`
  unsigned long long* gdesc; // dispatch scratch [n_tiles / 32][4]: the same per group of 32 tiles
  uint32_t* totals;          // dispatch scratch [kMaxShards + 1]: per-shard totals of this launch, [8] = seq once they are valid
  uint32_t* ticket;          // dispatch scratch: tile ticket counter, zero between launches
  uint32_t* done;            // dispatch scratch: finished-CTA counter, zero between launches
  uint32_t seq;              // launch sequence number (1..255): stale descriptors of earlier launches read as "not yet"
  uint32_t* flags;           // [0] += records that did not fit their slab
  uint8_t* out;              // combine: [n * MSG] replies in request order, 16-byte aligned
  uint32_t n, n_tiles, world, me, cap, epoch;
  PeerPtrs slab;             // slab of THIS source at shard o (request slabs for dispatch, reply slabs for combine)
  PeerPtrs sig;              // dispatch: epoch word array of shard o (word `me` is written); 0 = no signalling
};

// eight 16-bit counters (one per shard); a tile holds at most 2048 records, so fields never carry
struct Cnt8 { uint64_t lo, hi; };
DINT_D Cnt8 operator+(Cnt8 a, Cnt8 b) { return Cnt8{a.lo + b.lo, a.hi + b.hi}; }
DINT_D Cnt8 operator-(Cnt8 a, Cnt8 b) { return Cnt8{a.lo - b.lo, a.hi - b.hi}; }
DINT_D uint32_t cnt8_get(Cnt8 a, uint32_t o) { return (uint32_t)(((o < 4 ? a.lo : a.hi) >> (16 * (o & 3))) & 0xffffu); }
DINT_D void cnt8_inc(Cnt8& a, uint32_t o) {
  const uint64_t one = 1ull << (16 * (o & 3));
  if (o < 4) a.lo += one; else a.hi += one;
}
// exclusive prefix of `mine` over the CTA's threads, and the CTA total (all threads get both)
DINT_D void block_scan_cnt8(Cnt8 mine, Cnt8& excl, Cnt8& total, Cnt8* s_w) {
  Cnt8 x = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    Cnt8 y{__shfl_up_sync(0xffffffffu, x.lo, o), __shfl_up_sync(0xffffffffu, x.hi, o)};
    if ((int)lane_id() >= o) x = x + y;
  }
  if (lane_id() == 31) s_w[warp_id()] = x;
  __syncthreads();
  Cnt8 woff{0, 0}, tot{0, 0};
#pragma unroll
  for (int w = 0; w < kThreads / 32; w++) {
    if (w < (int)warp_id()) woff = woff + s_w[w];
    tot = tot + s_w[w];
  }
  excl = woff + x - mine;
  total = tot;
  __syncthreads();
}

// All threads of the CTA: copy nbytes; src and dst have the SAME address modulo 16.
DINT_D void coop_copy16(uint8_t* dst, const uint8_t* src, uint32_t nbytes) {
  uint32_t head = (16u - (uint32_t)((uintptr_t)dst & 15u)) & 15u;
  if (head > nbytes) head = nbytes;
  if (threadIdx.x < head) dst[threadIdx.x] = src[threadIdx.x];
  const uint32_t body = (nbytes - head) >> 4;
  const uint4* s4 = (const uint4*)(src + head);
  uint4* d4 = (uint4*)(dst + head);
  for (uint32_t i = threadIdx.x; i < body; i += kThreads) d4[i] = s4[i];
  const uint32_t done = head + (body << 4);
  if (threadIdx.x < nbytes - done) dst[done + threadIdx.x] = src[done + threadIdx.x];
}
// The same by ONE warp.
DINT_D void warp_copy16(uint8_t* dst, const uint8_t* src, uint32_t nbytes) {
  const uint32_t lane = lane_id();
  uint32_t head = (16u - (uint32_t)((uintptr_t)dst & 15u)) & 15u;
  if (head > nbytes) head = nbytes;
  if (lane < head) dst[lane] = src[lane];
  const uint32_t body = (nbytes - head) >> 4;
  const uint4* s4 = (const uint4*)(src + head);
  uint4* d4 = (uint4*)(dst + head);
  for (uint32_t i = lane; i < body; i += 32) d4[i] = s4[i];
  const uint32_t done = head + (body << 4);
  if (lane < nbytes - done) dst[done + lane] = src[done + lane];
}
// All threads of the CTA: fill nbytes at any alignment with the padding byte.
DINT_D void coop_fill_pad(uint8_t* dst, uint64_t nbytes) {
  uint64_t head = (16u - (uint32_t)((uintptr_t)dst & 15u)) & 15u;
  if (head > nbytes) head = nbytes;
  if (threadIdx.x < head) dst[threadIdx.x] = kPadType;
  const uint64_t body = (nbytes - head) >> 4;
  uint4* d4 = (uint4*)(dst + head);
  const uint32_t p = 0x01010101u * kPadType;
  for (uint64_t i = threadIdx.x; i < body; i += kThreads) d4[i] = make_uint4(p, p, p, p);
  const uint64_t done = head + (body << 4);
  if (threadIdx.x < nbytes - done) dst[done + threadIdx.x] = kPadType;
}

// owners of this thread's records of tile t, as bytes (0xff = none) and as a counter vector
template <int PER>
DINT_D Cnt8 load_owners(const RouteArgs& a, uint32_t t, uint32_t (&own)[PER]) {
  const uint32_t i0 = (t * kThreads + threadIdx.x) * PER;
  Cnt8 mine{0, 0};
  if (PER == 8 && i0 + 7 < a.n) {
    const uint2 w = *(const uint2*)(a.owner + i0);
#pragma unroll
    for (int j = 0; j < PER; j++) own[j] = ((j < 4 ? w.x : w.y) >> (8 * (j & 3))) & 0xffu;
  } else {
#pragma unroll
    for (int j = 0; j < PER; j++) own[j] = i0 + j < a.n ? a.owner[i0 + j] : 0xffu;
  }
#pragma unroll
  for (int j = 0; j < PER; j++)
    if (own[j] < a.world) cnt8_inc(mine, own[j]);
  return mine;
}

// look-back descriptor word: bits 63..56 seq, 55..54 status (1 = the tile's own counts, 2 = inclusive prefix), then two
// 27-bit counters (shards 2k and 2k+1 in word k).  Every word validates itself, so the four words of a descriptor need
// no common publication point.
DINT_D unsigned long long lb_pack(uint32_t seq, uint32_t status, uint32_t lo, uint32_t hi) {
  return ((unsigned long long)seq << 56) | ((unsigned long long)status << 54) | ((unsigned long long)hi << 27) | lo;
}
DINT_D unsigned long long lb_load(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
DINT_D void lb_store(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Two-level look-back by ONE whole warp for tile t: publishes the tile's two counts (c0, c1) in desc[t * stride] and
// returns their sums over tiles 0 .. t-1.  (1) the tiles before t inside its group of 32 -- one window; (2) the last tile
// of a group publishes the group's counts in gdesc[g * stride]; (3) the groups before t's -- one window per 32 groups.
// Nothing ever waits for a prefix, only for counts, so all tiles of a wave finish together.  Tiles must be drawn in
// index order (a ticket), so that a tile only waits for tiles that running CTAs hold.  Every word validates itself
// (launch number `seq` + "present" bit); counts stay below 2^27.
DINT_D uint2 lb_exclusive(unsigned long long* desc, unsigned long long* gdesc, uint32_t stride, uint32_t seq, uint32_t t,
                          uint32_t c0, uint32_t c1) {
  const uint32_t lane = lane_id();
  const uint32_t g = t >> 5, j = t & 31u;
  if (lane == 0) lb_store(desc + (size_t)t * stride, lb_pack(seq, 1, c0, c1));
  uint32_t x0 = 0, x1 = 0;
  if (lane < j) {                                        // (1) tiles g*32 .. t-1
    const unsigned long long* p = desc + (size_t)(g * 32 + lane) * stride;
    unsigned long long v;
    do { v = lb_load(p); } while ((uint32_t)(v >> 56) != seq || ((v >> 54) & 3u) == 0);
    x0 = (uint32_t)v & 0x7ffffffu;
    x1 = (uint32_t)(v >> 27) & 0x7ffffffu;
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) { x0 += __shfl_xor_sync(0xffffffffu, x0, d); x1 += __shfl_xor_sync(0xffffffffu, x1, d); }
  if (j == 31 && lane == 0) lb_store(gdesc + (size_t)g * stride, lb_pack(seq, 1, x0 + c0, x1 + c1));   // (2)
  uint32_t e0 = x0, e1 = x1;
  for (uint32_t base = 0; base < g; base += 32) {        // (3) groups 0 .. g-1
    uint32_t y0 = 0, y1 = 0;
    if (base + lane < g) {
      const unsigned long long* p = gdesc + (size_t)(base + lane) * stride;
      unsigned long long v;
      do { v = lb_load(p); } while ((uint32_t)(v >> 56) != seq || ((v >> 54) & 3u) == 0);
      y0 = (uint32_t)v & 0x7ffffffu;
      y1 = (uint32_t)(v >> 27) & 0x7ffffffu;
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) { y0 += __shfl_xor_sync(0xffffffffu, y0, d); y1 += __shfl_xor_sync(0xffffffffu, y1, d); }
    e0 += y0;
    e1 += y1;
  }
  return make_uint2(e0, e1);
}

// dispatch: owner bytes, stable partition into the slabs, padding, epoch flags -- one launch, one pass
template <int KIND>
__global__ void __launch_bounds__(kThreads, 4) k_route_dispatch(const Ctx c, const RouteArgs a) {
  using W = Wire<KIND>;
  using RT = RTile<W::MSG>;
  constexpr int MSG = W::MSG, PER = RT::PER;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* s_in = smem;                                  // the tile as it arrived
  uint8_t* s_out = smem + RT::BYTES + 16;                // the tile partitioned into runs
  __shared__ Cnt8 s_w[kThreads / 32];
  __shared__ uint32_t s_base[kMaxShards], s_total[kMaxShards], s_off[kMaxShards], s_len[kMaxShards];
  __shared__ uint32_t s_tile, s_last;
  const uint32_t G = gridDim.x, b = blockIdx.x;

  for (;;) {
    if (threadIdx.x == 0) s_tile = atomicAdd(a.ticket, 1u);          // tiles in index order: a tile only ever waits for
    __syncthreads();                                                  // tiles drawn before it, i.e. by CTAs that are running
    const uint32_t t = s_tile;
    if (t >= a.n_tiles) break;
    const uint32_t first = t * RT::RECS;
    const uint32_t nrec = a.n - first < (uint32_t)RT::RECS ? a.n - first : (uint32_t)RT::RECS;
    const uint32_t valid = nrec * MSG;
    {
      const uint8_t* src = a.req + (size_t)t * RT::BYTES;
      const uint32_t body = valid >> 4;
      for (uint32_t i = threadIdx.x; i < body; i += kThreads) ((uint4*)s_in)[i] = __ldcg((const uint4*)src + i);
      if (threadIdx.x < valid - (body << 4)) s_in[(body << 4) + threadIdx.x] = src[(body << 4) + threadIdx.x];
    }
    __syncthreads();
    // ---- owners of this thread's records ----
    uint32_t own[PER];
    Cnt8 mine{0, 0};
    const uint32_t r0 = threadIdx.x * PER;
#pragma unroll
    for (int j = 0; j < PER; j++) {
      uint32_t o = 0xffu;
      if (r0 + j < nrec) {
        o = a.owner_in ? a.owner_in[first + r0 + j] : route_owner_of<KIND>(c, s_in + (size_t)(r0 + j) * MSG);
        if (o >= a.world) o = 0xffu;
      }
      own[j] = o;
      if (o < a.world) cnt8_inc(mine, o);
    }
    if (PER == 8 && r0 + 7 < nrec) {
      *(uint2*)(a.owner + first + r0) = make_uint2(own[0] | (own[1 % PER] << 8) | (own[2 % PER] << 16) | (own[3 % PER] << 24),
                                                   own[4 % PER] | (own[5 % PER] << 8) | (own[6 % PER] << 16) | (own[7 % PER] << 24));
    } else {
#pragma unroll
      for (int j = 0; j < PER; j++)
        if (r0 + j < nrec) a.owner[first + r0 + j] = (uint8_t)own[j];
    }
    Cnt8 excl, total;
    block_scan_cnt8(mine, excl, total, s_w);
    // ---- look-back over the published counts (lb_exclusive): warp k (< 4) owns descriptor word k (two shards per word) ----
    if (warp_id() < 4) {
      const uint32_t k = warp_id(), lane = lane_id();
      const uint32_t c0 = cnt8_get(total, 2 * k), c1 = cnt8_get(total, 2 * k + 1);
      const uint2 ex = lb_exclusive(a.desc + k, a.gdesc + k, 4, a.seq, t, c0, c1);
      const uint32_t e0 = ex.x, e1 = ex.y;
      if (lane == 0) {
        s_base[2 * k] = e0;
        s_base[2 * k + 1] = e1;
        if (t == a.n_tiles - 1) {                        // the slabs' totals, for the padding and the overflow count
          a.totals[2 * k] = e0 + c0;
          a.totals[2 * k + 1] = e1 + c1;
        }
      }
    }
    __syncthreads();
    if (t == a.n_tiles - 1 && threadIdx.x == 0) {
      __threadfence();
      asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(a.totals + kMaxShards), "r"(a.seq) : "memory");
    }
    if (threadIdx.x == 0) {
      uint32_t off = 0;
      for (uint32_t o = 0; o < a.world; o++) {
        const uint32_t cnt = cnt8_get(total, o), base = s_base[o];
        const uint32_t room = base < a.cap ? a.cap - base : 0u;
        const uint32_t take = cnt < room ? cnt : room;
        const uint32_t daddr = (uint32_t)((a.slab.p[o] + (uint64_t)base * MSG) & 15u);
        off += (daddr - off) & 15u;                      // the run starts at its destination's alignment
        s_off[o] = off;
        s_len[o] = take * MSG;
        off += cnt * MSG;
        a.tilebase[(size_t)t * kMaxShards + o] = base;
      }
    }
    __syncthreads();
    {
      Cnt8 seen = excl;
#pragma unroll
      for (int j = 0; j < PER; j++) {
        const uint32_t o = own[j];
        if (o < a.world) {
          const uint32_t r = cnt8_get(seen, o);
          cnt8_inc(seen, o);
          if (r * MSG < s_len[o]) copy_record<MSG>(s_out + s_off[o] + r * MSG, s_in + (threadIdx.x * PER + j) * MSG);
        }
      }
    }
    __syncthreads();
    if (a.world <= 2) {
      for (uint32_t o = 0; o < a.world; o++)
        if (s_len[o]) coop_copy16((uint8_t*)a.slab.p[o] + (uint64_t)s_base[o] * MSG, s_out + s_off[o], s_len[o]);
    } else {                                             // one warp per run: the runs leave side by side
      for (uint32_t o = warp_id(); o < a.world; o += kThreads / 32)
        if (s_len[o]) warp_copy16((uint8_t*)a.slab.p[o] + (uint64_t)s_base[o] * MSG, s_out + s_off[o], s_len[o]);
    }
    __syncthreads();                                     // (s_in / s_out / s_tile are reused by the next tile)
  }

  // ---- the slabs' totals: published by whoever handled the last tile ----
  if (a.n_tiles == 0) {
    if (threadIdx.x < kMaxShards) s_total[threadIdx.x] = 0;
  } else {
    if (threadIdx.x == 0) {
      uint32_t v;
      do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(a.totals + kMaxShards) : "memory"); } while (v != a.seq);
    }
    __syncthreads();
    if (threadIdx.x < kMaxShards) s_total[threadIdx.x] = __ldcg(&a.totals[threadIdx.x]);
  }
  __syncthreads();
  if (b == 0 && threadIdx.x < a.world && s_total[threadIdx.x] > a.cap) atomicAdd(&a.flags[0], s_total[threadIdx.x] - a.cap);
  // ---- padding: slots [total, cap) of every slab, shared out over the CTAs ----
  for (uint32_t o = 0; o < a.world; o++) {
    const uint32_t tot = s_total[o] < a.cap ? s_total[o] : a.cap;
    const uint64_t len = (uint64_t)(a.cap - tot) * MSG;
    const uint64_t lo = len * b / G, hi = len * (b + 1) / G;
    if (hi > lo) coop_fill_pad((uint8_t*)a.slab.p[o] + (uint64_t)tot * MSG + lo, hi - lo);
  }
  // ---- the last CTA to finish tells the peers that this source's slabs of epoch `epoch` are complete ----
  // (one system-scope fence per CTA, by the thread that counts the CTA as done, after the CTA barrier: cumulative over the
  //  other threads' stores, instead of a fence in every thread)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const uint32_t prev = atomicAdd(a.done, 1u);
    s_last = prev == G - 1;
    if (s_last) { *a.done = 0; *a.ticket = 0; }          // for the next launch (stream-ordered behind this one)
  }
  __syncthreads();
  if (s_last && threadIdx.x < a.world && a.sig.p[threadIdx.x]) {
    bool over = false;                                   // any slab of this source too small: every owner is told (bit 31)
    for (uint32_t o = 0; o < a.world; o++) over |= s_total[o] > a.cap;
    __threadfence_system();
    uint32_t* flag = (uint32_t*)a.sig.p[threadIdx.x] + a.me;
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(a.epoch | (over ? kSigOverflow : 0u)) : "memory");
  }
}

// combine: the replies of tile t are one contiguous run per shard in the reply slabs; put them back in order
template <int MSG>
__global__ void __launch_bounds__(kThreads, 4) k_route_combine(const RouteArgs a) {
  using RT = RTile<MSG>;
  constexpr int PER = RT::PER;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* s_out = smem;                                 // the tile in request order
  uint8_t* s_in = smem + RT::BYTES + 16;                 // the runs as they sit in the slabs
  __shared__ Cnt8 s_w[kThreads / 32];
  __shared__ uint32_t s_off[kMaxShards], s_len[kMaxShards], s_base[kMaxShards];
  for (uint32_t t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
    uint32_t own[PER];
    const Cnt8 mine = load_owners<PER>(a, t, own);
    Cnt8 excl, total;
    if (threadIdx.x < kMaxShards) s_base[threadIdx.x] = a.tilebase[(size_t)t * kMaxShards + threadIdx.x];   // one latency, not eight
    block_scan_cnt8(mine, excl, total, s_w);
    if (threadIdx.x == 0) {
      uint32_t off = 0;
      for (uint32_t o = 0; o < a.world; o++) {
        const uint32_t cnt = cnt8_get(total, o), base = s_base[o];
        const uint32_t room = base < a.cap ? a.cap - base : 0u;
        const uint32_t take = cnt < room ? cnt : room;
        const uint32_t saddr = (uint32_t)((a.slab.p[o] + (uint64_t)base * MSG) & 15u);
        off += (saddr - off) & 15u;
        s_off[o] = off;
        s_len[o] = take * MSG;
        off += cnt * MSG;
      }
    }
    __syncthreads();
    if (a.world <= 2) {
      for (uint32_t o = 0; o < a.world; o++)
        if (s_len[o]) coop_copy16(s_in + s_off[o], (const uint8_t*)a.slab.p[o] + (uint64_t)s_base[o] * MSG, s_len[o]);
    } else {
      for (uint32_t o = warp_id(); o < a.world; o += kThreads / 32)
        if (s_len[o]) warp_copy16(s_in + s_off[o], (const uint8_t*)a.slab.p[o] + (uint64_t)s_base[o] * MSG, s_len[o]);
    }
    __syncthreads();
    {
      Cnt8 seen = excl;
#pragma unroll
      for (int j = 0; j < PER; j++) {
        const uint32_t o = own[j];
        uint8_t* dst = s_out + (threadIdx.x * PER + j) * MSG;
        bool have = false;
        if (o < a.world) {
          const uint32_t r = cnt8_get(seen, o);
          cnt8_inc(seen, o);
          if (r * MSG < s_len[o]) { copy_record<MSG>(dst, s_in + s_off[o] + r * MSG); have = true; }
        }
        if (!have)                                       // undeliverable or dropped by a full slab: error reply
          for (int q = 0; q < MSG; q++) dst[q] = 0xff;
      }
    }
    __syncthreads();
    {
      const uint32_t first = t * RT::RECS;
      const uint32_t valid = (a.n - first < (uint32_t)RT::RECS ? a.n - first : (uint32_t)RT::RECS) * MSG;
      uint8_t* dst = a.out + (size_t)t * RT::BYTES;
      const uint32_t body = valid >> 4;
      for (uint32_t i = threadIdx.x; i < body; i += kThreads) ((uint4*)dst)[i] = ((const uint4*)s_out)[i];
      if (threadIdx.x < valid - (body << 4)) dst[(body << 4) + threadIdx.x] = s_out[(body << 4) + threadIdx.x];
    }
    __syncthreads();
  }
}

}  // namespace dint
