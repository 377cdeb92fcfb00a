// ubench.cu -- development microbenchmark: what can this chip do on random 64-byte (and 32-byte)
// gathers?  (The random-access ceiling the store GET path is compared with; not part of the product.)
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint64_t mix(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33; return x; }
template <int VEC, int ILP>
__global__ void gather(const uint4* __restrict__ tbl, uint64_t mask_entries, uint32_t* out, uint32_t iters) {
  uint64_t tid = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint32_t acc = 0;
  for (uint32_t it = 0; it < iters; it++) {
    uint4 v[ILP][VEC];
#pragma unroll
    for (int j = 0; j < ILP; j++) {
      uint64_t e = mix(tid * 1315423911ULL + it * 2654435761ULL + j * 97) & mask_entries;
#pragma unroll
      for (int k = 0; k < VEC; k++) v[j][k] = __ldcg(tbl + e * VEC + k);
    }
#pragma unroll
    for (int j = 0; j < ILP; j++)
#pragma unroll
      for (int k = 0; k < VEC; k++) acc += v[j][k].x ^ v[j][k].w;
  }
  if (acc == 0x12345678) out[0] = acc;
}
template <int VEC, int ILP>
void run(const char* name, uint4* tbl, uint64_t entries, int blocks, int threads, uint32_t iters, uint32_t* out) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  gather<VEC, ILP><<<blocks, threads>>>(tbl, entries - 1, out, 2);
  cudaEventRecord(a);
  gather<VEC, ILP><<<blocks, threads>>>(tbl, entries - 1, out, iters);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  double n = (double)blocks * threads * iters * ILP;
  printf("%-28s entries=%.0fM x %dB  blocks=%d thr=%d ilp=%d : %.2f G gathers/s  %.2f TB/s\n", name, entries / 1e6, VEC * 16, blocks, threads,
         ILP, n / ms / 1e6, n * VEC * 16 / ms / 1e9);
}
int main() {
  size_t bytes = 4ULL << 30;
  uint4* tbl; cudaMalloc(&tbl, bytes); cudaMemset(tbl, 1, bytes);
  uint32_t* out; cudaMalloc(&out, 4);
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  for (size_t tb : {512ULL << 20, 4ULL << 30}) {
    run<4, 1>("64B ilp1 8cta", tbl, tb / 64, sms * 8, 256, 64, out);
    run<4, 2>("64B ilp2 8cta", tbl, tb / 64, sms * 8, 256, 32, out);
    run<4, 4>("64B ilp4 4cta", tbl, tb / 64, sms * 4, 256, 32, out);
    run<2, 1>("32B ilp1 8cta", tbl, tb / 32, sms * 8, 256, 64, out);
    run<2, 4>("32B ilp4 8cta", tbl, tb / 32, sms * 8, 256, 32, out);
    run<1, 4>("16B ilp4 8cta", tbl, tb / 16, sms * 8, 256, 32, out);
  }
  return 0;
}
