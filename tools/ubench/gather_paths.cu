// gather_paths.cu -- microbenchmark: which on-chip paths can carry a data-dependent 4-byte /
// 16-byte table lookup per lane, and do they add up?  (Design input for the slice kernel's
// corner gather, which ncu shows bound by shared-memory wavefronts.)
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench/bin/gather_paths tools/ubench/gather_paths.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

constexpr int ITERS = 512;
constexpr int THREADS = 256;

// mode bits: 1 = LDS.128 random z, 2 = SHFL x4 (16 B) random src lane, 4 = LDG.128 (L1 hit) random,
// 8 = LDS.128 warp-uniform address, 16 = LDS.32 x4 random z (multicast), 32 = tex1Dfetch float4
template <int MODE>
__global__ void __launch_bounds__(THREADS) k(const float4* __restrict__ gtab, cudaTextureObject_t tex,
                                             const int* __restrict__ zs, float* out, long long* cycles) {
  __shared__ float4 tab[8 * 3 * 16];  // 8 z-levels x 3 chunks, x 16 "cells"
  for (int i = threadIdx.x; i < 8 * 3 * 16; i += THREADS) tab[i] = gtab[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  int z = zs[(blockIdx.x * THREADS + threadIdx.x) & 4095];
  float4 acc = make_float4(0, 0, 0, 0);
  float4 reg = gtab[lane];  // "table in registers": lane l holds entry l
  long long t0 = clock64();
#pragma unroll 4
  for (int it = 0; it < ITERS; ++it) {
    const int zz = (z + it) & 7;
    if (MODE & 1) {
      const float4 v = tab[zz * 3 + (it & 1)];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (MODE & 2) {
      const int src = zz * 4 + (it & 3);
      acc.x += __shfl_sync(0xffffffffu, reg.x, src);
      acc.y += __shfl_sync(0xffffffffu, reg.y, src);
      acc.z += __shfl_sync(0xffffffffu, reg.z, src);
      acc.w += __shfl_sync(0xffffffffu, reg.w, src);
    }
    if (MODE & 4) {
      const float4 v = __ldg(gtab + zz * 3 + (it & 1));
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (MODE & 8) {
      const float4 v = tab[((it * 7) & 127)];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (MODE & 16) {
      const float* t = reinterpret_cast<const float*>(tab) + zz * 12 + (it & 1) * 4;
      acc.x += t[0]; acc.y += t[1]; acc.z += t[2]; acc.w += t[3];
    }
    if (MODE & 64) {   // second LDS.128 (different chunk)
      const float4 v = tab[zz * 3 + 2];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (MODE & 128) {  // third LDS.128 (neighbour cell)
      const float4 v = tab[24 + zz * 3 + (it & 1)];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (MODE & 256) {  // fourth LDS.128
      const float4 v = tab[24 + zz * 3 + 2];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (MODE & 32) {
      const float4 v = tex1Dfetch<float4>(tex, zz * 3 + (it & 1));
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  long long t1 = clock64();
  out[blockIdx.x * THREADS + threadIdx.x] = acc.x + acc.y + acc.z + acc.w;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int MODE>
void run(const char* name, const float4* gtab, cudaTextureObject_t tex, const int* zs, float* out, long long* cyc, int ctas_per_sm) {
  int sms; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  const int grid = sms * ctas_per_sm;
  k<MODE><<<grid, THREADS>>>(gtab, tex, zs, out, cyc);
  CK(cudaDeviceSynchronize());
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  cudaEventRecord(a);
  k<MODE><<<grid, THREADS>>>(gtab, tex, zs, out, cyc);
  cudaEventRecord(b); CK(cudaDeviceSynchronize());
  float ms; cudaEventElapsedTime(&ms, a, b);
  std::vector<long long> h(grid); CK(cudaMemcpy(h.data(), cyc, grid * sizeof(long long), cudaMemcpyDeviceToHost));
  double avg = 0; for (auto v : h) avg += v; avg /= grid;
  // per SM: warps = ctas_per_sm * 8; each does ITERS lookups of 16 B per lane
  const double lookups_per_sm = double(ctas_per_sm) * 8 * ITERS;
  printf("%-44s ctas/SM=%d  %.1f cycles/CTA  -> %.2f clk per warp-wide 16B-lookup per SM (%.1f B/clk/SM delivered)  [%.3f ms]\n",
         name, ctas_per_sm, avg, avg / lookups_per_sm, 512.0 * lookups_per_sm / avg, ms);
}

int main() {
  float4* gtab; int* zs; float* out; long long* cyc;
  CK(cudaMalloc(&gtab, 8 * 3 * 16 * sizeof(float4)));
  CK(cudaMalloc(&zs, 4096 * sizeof(int)));
  CK(cudaMalloc(&out, 132 * 8 * THREADS * sizeof(float) * 2));
  CK(cudaMalloc(&cyc, 132 * 8 * sizeof(long long) * 2));
  std::vector<float4> h(8 * 3 * 16); for (size_t i = 0; i < h.size(); ++i) h[i] = make_float4(i, i + 1, i + 2, i + 3);
  std::vector<int> hz(4096); srand(1); for (auto& v : hz) v = rand() & 7;
  CK(cudaMemcpy(gtab, h.data(), h.size() * sizeof(float4), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(zs, hz.data(), hz.size() * sizeof(int), cudaMemcpyHostToDevice));
  cudaResourceDesc rd = {}; rd.resType = cudaResourceTypeLinear; rd.res.linear.devPtr = gtab;
  rd.res.linear.desc = cudaCreateChannelDesc<float4>(); rd.res.linear.sizeInBytes = h.size() * sizeof(float4);
  cudaTextureDesc td = {}; td.readMode = cudaReadModeElementType;
  cudaTextureObject_t tex; CK(cudaCreateTextureObject(&tex, &rd, &td, nullptr));
  for (int c : {2, 4}) {
    run<1>("LDS.128 random z (8 addrs/warp)", gtab, tex, zs, out, cyc, c);
    run<8>("LDS.128 warp-uniform address", gtab, tex, zs, out, cyc, c);
    run<16>("4 x LDS.32 random z (multicast)", gtab, tex, zs, out, cyc, c);
    run<2>("4 x SHFL.IDX random src", gtab, tex, zs, out, cyc, c);
    run<4>("LDG.128 L1-hit random z", gtab, tex, zs, out, cyc, c);
    run<32>("tex1Dfetch<float4> random z", gtab, tex, zs, out, cyc, c);
    run<1 | 2>("LDS.128 + 4xSHFL (2 lookups/iter)", gtab, tex, zs, out, cyc, c);
    run<1 | 4>("LDS.128 + LDG.128 (2 lookups/iter)", gtab, tex, zs, out, cyc, c);
    run<1 | 32>("LDS.128 + tex float4 (2 lookups/iter)", gtab, tex, zs, out, cyc, c);
    run<1 | 2 | 32>("LDS.128 + 4xSHFL + tex (3 lookups/iter)", gtab, tex, zs, out, cyc, c);
    run<1 | 64>("2 x LDS.128 (per iter)", gtab, tex, zs, out, cyc, c);
    run<1 | 64 | 32>("2 x LDS.128 + tex (per iter)", gtab, tex, zs, out, cyc, c);
    run<1 | 64 | 128>("3 x LDS.128 (per iter)", gtab, tex, zs, out, cyc, c);
    run<1 | 64 | 128 | 32>("3 x LDS.128 + tex (per iter)", gtab, tex, zs, out, cyc, c);
    run<1 | 64 | 128 | 256>("4 x LDS.128 (per iter)", gtab, tex, zs, out, cyc, c);
    run<1 | 64 | 128 | 256 | 32>("4 x LDS.128 + tex (per iter)", gtab, tex, zs, out, cyc, c);
  }
  return 0;
}
