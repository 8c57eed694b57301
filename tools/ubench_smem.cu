// Micro-benchmark: shared-memory atomics and gathers at random addresses on sm_90a (H100, 132 SMs).
// Decides the design of the shared-memory-resident segment fold (bw_segfold.cuh): how many
// native 32-bit ATOMS / LDS.64 per event can a block afford?
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/ubench_smem tools/ubench_smem.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
typedef uint64_t u64;
typedef uint32_t u32;
__device__ __forceinline__ u64 mix64(u64 z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
// MODE 0: atomicAdd u32 no return (ATOMS.ADD / RED-like)   1: atomicAdd u32 with return (rank)
//      2: atomicMax u32                                     3: LDS.64 gather
//      4: atomicAdd u64 (CAS loop)                          5: LDS.64 gather + atomicAdd u32 + atomicMax u32 (fold-like)
//      6: plain STS.32 scatter                              7: atomicCAS u64 (claim-like)
template <int MODE>
__global__ void k(u32 words, int iters, u64* sink, unsigned long long* cycles) {
  extern __shared__ __align__(16) unsigned char raw[];
  u32* w = (u32*)raw;
  u64* w64 = (u64*)raw;
  for (u32 i = threadIdx.x; i < words; i += blockDim.x) w[i] = 0;
  __syncthreads();
  const u32 mask = words - 1, mask64 = words / 2 - 1;
  u64 acc = 0;
  u64 seed = ((u64)blockIdx.x << 32) | threadIdx.x;
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
    u64 h[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) h[u] = mix64(seed + (u64)(it * 4 + u) * 0x9E3779B97F4A7C15ULL);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const u32 a = (u32)(h[u] >> 20);
      if (MODE == 0) atomicAdd(&w[a & mask], 1u);
      if (MODE == 1) acc += atomicAdd(&w[a & mask], 1u);
      if (MODE == 2) atomicMax(&w[a & mask], (u32)h[u]);
      if (MODE == 3) acc += w64[a & mask64];
      if (MODE == 4) atomicAdd((unsigned long long*)&w64[a & mask64], 1ULL);
      if (MODE == 5) {
        const u32 s = a & (mask64 / 2);  // first half: keys (u64); second half: two u32 arrays
        acc += w64[s];
        atomicAdd(&w[words / 2 + s], 1u);
        atomicMax(&w[words / 2 + words / 4 + s], (u32)h[u]);
      }
      if (MODE == 6) w[a & mask] = (u32)h[u];
      if (MODE == 7) acc += atomicCAS((unsigned long long*)&w64[a & mask64], 0ULL, h[u] | 1ULL);
    }
  }
  long long t1 = clock64();
  __syncthreads();
  if (acc == 0x1234567) *sink = acc + w[threadIdx.x & mask];
  if (threadIdx.x == 0) atomicMax(cycles, (unsigned long long)(t1 - t0));
}
int main() {
  u64* sink;
  unsigned long long* cyc;
  cudaMalloc(&sink, 8);
  cudaMalloc(&cyc, 8);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  const char* names[] = {"atomicAdd.u32 (no ret)", "atomicAdd.u32 (ret)", "atomicMax.u32", "LDS.64 gather", "atomicAdd.u64 (CAS loop)",
                         "LDS.64 + add.u32 + max.u32", "STS.32 scatter", "atomicCAS.u64"};
  const int iters = 2048;
  for (int kb : {16, 64}) {
    const u32 words = kb * 256;
    for (int threads : {256, 512, 1024}) {
      for (int bps : {1, 2}) {
        if (threads * bps > 2048 || kb * bps > 200) continue;
        for (int mode = 0; mode < 8; ++mode) {
          void (*fn)(u32, int, u64*, unsigned long long*) = nullptr;
          switch (mode) {
            case 0: fn = k<0>; break; case 1: fn = k<1>; break; case 2: fn = k<2>; break; case 3: fn = k<3>; break;
            case 4: fn = k<4>; break; case 5: fn = k<5>; break; case 6: fn = k<6>; break; default: fn = k<7>;
          }
          cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kb * 1024);
          float best = 1e9;
          unsigned long long bc = 0;
          for (int rep = 0; rep < 3; ++rep) {
            cudaMemset(cyc, 0, 8);
            cudaEventRecord(e0);
            fn<<<132 * bps, threads, kb * 1024>>>(words, iters, sink, cyc);
            cudaEventRecord(e1);
            cudaEventSynchronize(e1);
            float ms;
            cudaEventElapsedTime(&ms, e0, e1);
            if (ms < best) {
              best = ms;
              cudaMemcpy(&bc, cyc, 8, cudaMemcpyDeviceToHost);
            }
          }
          const double ops = (double)132 * bps * threads * iters * 4;  // lane-ops
          const double warp_ops_per_sm = (double)bps * threads / 32 * iters * 4;
          printf("smem %3d KB  %4d thr x %d blk/SM  %-28s %.3f ms  %7.1f Gop/s chip  %.2f cyc per warp-op per SM\n", kb, threads, bps,
                 names[mode], best, ops / best / 1e6, (double)bc / warp_ops_per_sm);
        }
      }
    }
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) printf("CUDA error: %s\n", cudaGetErrorString(e));
  return 0;
}
