// State images (dint_image_save / dint_image_open, include/dint_b200.h): the device half.  An engine's state regions
// (snapshot_regions in engine.cu) are cut into blocks of kImgBlock raw bytes; a block is stored as a bitmap with one
// bit per 128-byte line (set when the line holds any non-zero byte), the non-zero lines in order, and a checksum.
//
//   k_image_pack    ONE pass over a block: 16-byte streaming loads, one line per thread, a warp ballot per 32 lines
//                   makes a bitmap word; each line's packed slot comes from the two-level look-back over per-tile
//                   counts (route.cuh, lb_exclusive); the lines go to a device staging buffer and the checksum is
//                   reduced in the same kernel.
//   k_image_unpack  cooperative: recomputes the block's checksum from the staged bytes (the same look-back gives
//                   every tile its first packed slot), and only when it equals the file's -- after a grid barrier --
//                   writes every line of the block's range: the staged line where the bit is set, zeros elsewhere.
//
// Checksum of a block: the sum mod 2^64 of fasthash64 of every bitmap word (its 4 bytes, seed 2 * word index) and of
// every stored line (its 128 bytes, a partial last line padded with zeros; seed 2 * line index + 1, the line's raw
// position in the block).  A sum does not depend on the order of the reduction.
#pragma once
#include "route.cuh"

namespace dint {

constexpr uint64_t kImgBlock = 64ull << 20;         // raw bytes per block (the last block of a region is shorter)
constexpr uint32_t kImgLine = 128;                   // bytes per bitmap bit
constexpr uint32_t kImgTileLines = kThreads;         // one line per thread, a tile per CTA iteration
constexpr uint32_t kImgMaxTiles = (uint32_t)(kImgBlock / kImgLine / kImgTileLines);

// lines / bitmap words of a block of `bytes` raw bytes (the bitmap is padded with zero words to a multiple of 16 bytes)
DINT_HD uint64_t img_lines(uint64_t bytes) { return (bytes + kImgLine - 1) / kImgLine; }
DINT_HD uint64_t img_words(uint64_t bytes) { return (img_lines(bytes) + 127) / 128 * 4; }

struct ImgArgs {
  uint8_t* raw;                 // the block's range in the engine's state (16-byte aligned)
  uint64_t bytes;               // its length
  uint32_t* bitmap;             // staging: img_words(bytes) words, then the packed lines
  uint8_t* lines;
  uint32_t n_words, n_tiles;
  unsigned long long* desc;     // look-back scratch [kImgMaxTiles], gdesc [kImgMaxTiles / 32]; zero before the launch
  unsigned long long* gdesc;
  uint32_t* ticket;             // zero before the launch
  uint32_t* tilebase;           // unpack: [kImgMaxTiles] first packed slot of every tile
  unsigned long long* sum;      // [0] checksum, [1] stored lines; zero before the launch
  unsigned long long expect;    // unpack: the checksum the file holds
  uint32_t* bad;                // unpack: set to 1 when the checksum differs (nothing was written)
};

DINT_HD uint64_t img_hash_word(uint32_t w, uint64_t index) {
  uint64_t h = (2 * index) ^ (4ULL * kFhM);
  h ^= fh_mix((uint64_t)w);
  h *= kFhM;
  return fh_mix(h);
}
DINT_D uint64_t img_hash_line(const uint4 (&v)[8], uint64_t line) {
  uint64_t h = (2 * line + 1) ^ ((uint64_t)kImgLine * kFhM);
#pragma unroll
  for (int k = 0; k < 8; k++) {
    h ^= fh_mix(((uint64_t)v[k].y << 32) | v[k].x);
    h *= kFhM;
    h ^= fh_mix(((uint64_t)v[k].w << 32) | v[k].z);
    h *= kFhM;
  }
  return fh_mix(h);
}

// the first n (< 16) bytes at p, zero-extended (a region may end inside a 16-byte piece)
DINT_D uint4 img_ld_partial(const uint8_t* p, uint32_t n) {
  uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
  for (int i = 0; i < 16; i++)
    if ((uint32_t)i < n) w[i >> 2] |= (uint32_t)p[i] << (8 * (i & 3));
  return make_uint4(w[0], w[1], w[2], w[3]);
}
DINT_D void img_st_partial(uint8_t* p, uint4 v, uint32_t n) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 16; i++)
    if ((uint32_t)i < n) p[i] = (uint8_t)(w[i >> 2] >> (8 * (i & 3)));
}

// line `line` of the block: zeros past its end
DINT_D bool img_load_raw(const ImgArgs& a, uint64_t line, uint4 (&v)[8]) {
  const uint64_t off = line * kImgLine;
  uint32_t any = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const uint64_t po = off + 16 * k;
    if (po + 16 <= a.bytes) v[k] = __ldcs((const uint4*)(a.raw + po));
    else if (po < a.bytes) v[k] = img_ld_partial(a.raw + po, (uint32_t)(a.bytes - po));
    else v[k] = make_uint4(0, 0, 0, 0);
    any |= v[k].x | v[k].y | v[k].z | v[k].w;
  }
  return any != 0;
}
DINT_D void img_store_raw(const ImgArgs& a, uint64_t line, const uint4 (&v)[8]) {
  const uint64_t off = line * kImgLine;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const uint64_t po = off + 16 * k;
    if (po + 16 <= a.bytes) __stcs((uint4*)(a.raw + po), v[k]);
    else if (po < a.bytes) img_st_partial(a.raw + po, v[k], (uint32_t)(a.bytes - po));
  }
}

// CTA-wide: each warp's bitmap word popcount -> the warp's offset in the tile and the tile's total
DINT_D uint32_t img_warp_offset(uint32_t word, uint32_t* s_w, uint32_t& total) {
  if (lane_id() == 0) s_w[warp_id()] = __popc(word);
  __syncthreads();
  uint32_t off = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; w++) {
    const uint32_t c = s_w[w];
    if (w < (int)warp_id()) off += c;
    tot += c;
  }
  total = tot;
  return off;
}

DINT_D void img_add_sum(unsigned long long* sum, unsigned long long acc) {
#pragma unroll
  for (int d = 16; d; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
  if (lane_id() == 0 && acc) atomicAdd(sum, acc);
}

__global__ void __launch_bounds__(kThreads) k_image_pack(const ImgArgs a) {
  __shared__ uint32_t s_w[kThreads / 32], s_tile, s_base;
  unsigned long long acc = 0;
  for (;;) {
    if (threadIdx.x == 0) s_tile = atomicAdd(a.ticket, 1u);   // tiles in index order (the look-back needs it)
    __syncthreads();
    const uint32_t t = s_tile;
    if (t >= a.n_tiles) break;
    const uint64_t line = (uint64_t)t * kImgTileLines + threadIdx.x;
    uint4 v[8];
    const bool nz = img_load_raw(a, line, v);
    const uint32_t word = __ballot_sync(0xffffffffu, nz);
    const uint64_t wi = line >> 5;
    if (lane_id() == 0 && wi < a.n_words) {
      a.bitmap[wi] = word;
      acc += img_hash_word(word, wi);
    }
    uint32_t total;
    const uint32_t woff = img_warp_offset(word, s_w, total);
    if (warp_id() == 0) {
      const uint2 ex = lb_exclusive(a.desc, a.gdesc, 1, 1, t, total, 0);
      if (lane_id() == 0) {
        s_base = ex.x;
        if (total) atomicAdd(&a.sum[1], (unsigned long long)total);
      }
    }
    __syncthreads();
    if (nz) {
      const uint32_t pos = s_base + woff + __popc(word & ((1u << lane_id()) - 1u));
      uint4* d = (uint4*)(a.lines + (size_t)pos * kImgLine);
#pragma unroll
      for (int k = 0; k < 8; k++) __stcs(d + k, v[k]);
      acc += img_hash_line(v, line);
    }
    __syncthreads();                                   // s_w / s_tile / s_base are reused by the next tile
  }
  img_add_sum(&a.sum[0], acc);
}

// Launched cooperatively with every CTA resident (a grid barrier separates the check from the writes).
__global__ void __launch_bounds__(kThreads) k_image_unpack(const ImgArgs a) {
  __shared__ uint32_t s_w[kThreads / 32], s_tile, s_base;
  unsigned long long acc = 0;
  // ---- 1: the checksum of the staged bytes, and every tile's first packed slot ----
  for (;;) {
    if (threadIdx.x == 0) s_tile = atomicAdd(a.ticket, 1u);
    __syncthreads();
    const uint32_t t = s_tile;
    if (t >= a.n_tiles) break;
    const uint64_t line = (uint64_t)t * kImgTileLines + threadIdx.x;
    const uint64_t wi = line >> 5;
    const uint32_t word = wi < a.n_words ? a.bitmap[wi] : 0u;
    if (lane_id() == 0 && wi < a.n_words) acc += img_hash_word(word, wi);
    uint32_t total;
    const uint32_t woff = img_warp_offset(word, s_w, total);
    if (warp_id() == 0) {
      const uint2 ex = lb_exclusive(a.desc, a.gdesc, 1, 1, t, total, 0);
      if (lane_id() == 0) { s_base = ex.x; a.tilebase[t] = ex.x; }
    }
    __syncthreads();
    if ((word >> lane_id()) & 1u) {
      const uint32_t pos = s_base + woff + __popc(word & ((1u << lane_id()) - 1u));
      const uint4* s = (const uint4*)(a.lines + (size_t)pos * kImgLine);
      uint4 v[8];
#pragma unroll
      for (int k = 0; k < 8; k++) v[k] = __ldcs(s + k);
      acc += img_hash_line(v, line);
    }
    __syncthreads();
  }
  img_add_sum(&a.sum[0], acc);
  cg::this_grid().sync();
  // ---- 2: refuse, or write every line of the range ----
  if (__ldcg(&a.sum[0]) != a.expect) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *a.bad = 1u;
    return;
  }
  for (uint32_t t = blockIdx.x; t < a.n_tiles; t += gridDim.x) {
    const uint64_t line = (uint64_t)t * kImgTileLines + threadIdx.x;
    const uint64_t wi = line >> 5;
    const uint32_t word = wi < a.n_words ? a.bitmap[wi] : 0u;
    uint32_t total;
    const uint32_t woff = img_warp_offset(word, s_w, total);
    uint4 v[8];
    if ((word >> lane_id()) & 1u) {
      const uint32_t pos = a.tilebase[t] + woff + __popc(word & ((1u << lane_id()) - 1u));
      const uint4* s = (const uint4*)(a.lines + (size_t)pos * kImgLine);
#pragma unroll
      for (int k = 0; k < 8; k++) v[k] = __ldcs(s + k);
    } else {
#pragma unroll
      for (int k = 0; k < 8; k++) v[k] = make_uint4(0, 0, 0, 0);
    }
    img_store_raw(a, line, v);
    __syncthreads();                                   // s_w is reused by the next tile
  }
}

}  // namespace dint
