// conv_wgmma.cu -- 3x3 / 1x1 convolution of the coefficient network as an implicit GEMM on
// Hopper's warpgroup tensor-core instructions (wgmma.mma_async, accumulator in registers), with
// fp32 parity.
//
// A plain TF32 (10-bit mantissa) product would lose the float32 parity the rest of the path
// keeps, so every operand is split
//     a = a_hi + a_lo,  a_hi = a with the low 13 mantissa bits cleared (exactly a TF32 value),
//                       a_lo = a - a_hi (exact in fp32; its own TF32 truncation is 2^-21 of a)
// and three MMAs accumulate a_hi*b_hi + a_hi*b_lo + a_lo*b_hi ("3xTF32"): relative error ~1e-6
// per product, i.e. float32-grade results from the tensor pipe at 3x the MMA count -- irrelevant
// here, the network is latency-bound.  The tensor cores' fp32 additions do not round to nearest,
// so an accumulator that runs over the whole reduction (576 k-values for a 3x3x64 layer) drifts by
// ~1e-5 of its magnitude.  Each 32-k chunk therefore accumulates into a fresh partial (12 MMAs),
// and the partials are summed by the CUDA cores with round-to-nearest.
//
// Shape: out[m][n] = sum_k A[m][k] * W[k][n] with m = output pixel (b, oy, ox), n = output
// channel, k = (ky, kx, ci).  One CTA (two warpgroups, 256 threads) owns a 128-pixel x N tile,
// N <= 128 (partial + total: N registers per thread); warpgroup g computes pixels 64g .. 64g + 63
// of it with m64nTWk8 instructions over N / TW column tiles (TW = 64, 32 or 16, the widest that
// divides N).  A layer with 128 < Cout <= 256 runs as two launches over output columns
// [0, 128) and [128, Cout).
//   * A chunks (32 k-values) are gathered by the threads (im2col with TF SAME padding), split
//     hi/lo and written to shared memory in the K-major no-swizzle core-matrix layout (8-row x
//     16-byte core matrices; SBO = 128 B between 8-row groups, LBO = rows * 16 B between 16-byte
//     k-chunks).  The gather of chunk c + 1 is in flight in registers while chunk c is staged
//     and its MMAs run.
//   * B chunks are either gathered from an HWIO weight buffer by the threads (launch_conv_wgmma,
//     any weights), or -- weights PRE-PACKED per 32-k chunk into the same layout and already split
//     hi/lo (hdrnet_conv2d_tc_pack_f32, once per model) -- one TMA bulk copy per chunk, issued by
//     one thread a chunk ahead of its use and completed on an mbarrier.
//   * A chunk's MMAs are retired (wgmma.wait_group 0) before its partial is added, and a CTA
//     barrier opens the next chunk, so a stage is free again once its chunk ended.  Three stages
//     (they fit for every N <= 128) let the packed weights arrive a chunk ahead of their use.
//   * epilogue: accumulator fragments + bias + ReLU, float2 stores.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "common.cuh"

namespace hdrnet_b200 {

constexpr int kTcThreads = 256;  // two warpgroups
constexpr int kTcM = 128;        // pixels per CTA
constexpr int kTcKc = 32;        // k-values per staged chunk (8 x 16-byte k-chunks, 4 MMA k-steps)
constexpr int kTcMaxN = 128;     // output columns per launch
constexpr int kTcMaxCout = 256;  // Cout of a layer (unpacked form; the packed form takes <= 128)
constexpr int kTcMaxStages = 3;

struct TcConvArgs {
  const float* in;
  const float* w;     // HWIO [k][k][Cin][Cout], or conv_tc_pack_kernel output (kPacked)
  const float* bias;  // [Cout] or nullptr
  float* out;
  int B, H, W, Cin, OH, OW, Cout, k, stride, pad_t, pad_l, relu;
  int n_off;          // first output column of this launch (the kernel's N columns follow it)
  int stages;         // 2 or 3
};

// wgmma shared-memory matrix descriptor, no swizzle (layout type 0), base offset 0.
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t smem_addr, uint32_t lbo_bytes,
                                                     uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr >> 4) & 0x3fffu);          // start address   [0,14)
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3fffu) << 16;    // leading offset  [16,30)
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3fffu) << 32;    // stride offset   [32,46)
  return d;
}

__device__ __forceinline__ void split_tf32(float v, float& hi, float& lo) {
  hi = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
  lo = v - hi;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs.
template <int R>
__device__ __forceinline__ void fence_operands(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x TW] = A[64 x 8] * B[8 x TW] + (scale_d ? D : 0), tf32 inputs from shared memory, fp32 D.
template <int TW>
__device__ __forceinline__ void wgmma_tf32(float (&d)[TW / 2], uint64_t da, uint64_t db, int scale_d);

template <>
__device__ __forceinline__ void wgmma_tf32<16>(float (&d)[8], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(scale_d));
}

template <>
__device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d));
}

template <>
__device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}

template <int N>
__host__ __device__ constexpr int tile_width() { return (N % 64 == 0) ? 64 : (N % 32 == 0) ? 32 : 16; }

template <int N>
__host__ __device__ constexpr size_t stage_bytes() { return static_cast<size_t>(2) * (kTcM + N) * kTcKc * sizeof(float); }

template <int N, bool kPacked>
__global__ void __launch_bounds__(kTcThreads, 1)
conv2d_wgmma_kernel(const TcConvArgs a) {
  constexpr int TW = tile_width<N>();
  constexpr int NT = N / TW;
  constexpr int kAFloats = kTcM * kTcKc;  // one half (hi or lo) of a stage's A
  constexpr int kBFloats = N * kTcKc;
  constexpr int kStageFloats = 2 * kAFloats + 2 * kBFloats;
  constexpr uint32_t kALbo = kTcM * 16, kBLbo = N * 16, kSbo = 128;
  constexpr uint32_t kBBytes = 2 * kBFloats * 4;
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ uint64_t b_full[kTcMaxStages];  // TMA: the packed weights of the stage have landed

  const int tid = threadIdx.x, wg = tid >> 7, row = tid & (kTcM - 1), half = tid >> 7;
  const int S = a.stages;
  float* ring = reinterpret_cast<float*>(smem);
  if (kPacked && tid == 0) {
    for (int s = 0; s < S; ++s) mbar_init(&b_full[s], 1);
    fence_mbar_init();
  }
  __syncthreads();

  // This thread's gather row = output pixel; it gathers k-chunks 4*half .. 4*half + 3 of a chunk.
  const long long total_px = static_cast<long long>(a.B) * a.OH * a.OW;
  const long long q = static_cast<long long>(blockIdx.x) * kTcM + row;
  const bool pv = q < total_px;
  const long long qq = pv ? q : 0;
  const int ox = static_cast<int>(qq % a.OW);
  const int oy = static_cast<int>((qq / a.OW) % a.OH);
  const int ob = static_cast<int>(qq / (static_cast<long long>(a.OW) * a.OH));
  const int K = a.k * a.k * a.Cin;
  const int nchunks = (K + kTcKc - 1) / kTcKc;

  // (ky, kx, ci) of the next k-chunk this thread gathers.  It advances incrementally, 4 channels
  // per step, because runtime integer divisions in the chunk loop cost far more than the loads.
  int g_ci, g_kx, g_ky;
  {
    const int k0 = 16 * half, t = k0 / a.Cin;
    g_ci = k0 - t * a.Cin;
    g_kx = t % a.k;
    g_ky = t / a.k;  // == k: past K, zero-fill
  }
  const auto step = [&]() {
    g_ci += 4;
    if (g_ci >= a.Cin) {
      g_ci = 0;
      if (++g_kx == a.k) { g_kx = 0; ++g_ky; }
    }
  };
  const int iy0 = oy * a.stride - a.pad_t, ix0 = ox * a.stride - a.pad_l;
  const float* in_b = a.in + static_cast<size_t>(ob) * a.H * a.W * a.Cin;
  const auto gather = [&](float4 (&v)[4]) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      v[c] = make_float4(0.f, 0.f, 0.f, 0.f);
      const int iy = iy0 + g_ky, ix = ix0 + g_kx;
      if (pv && g_ky < a.k && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W)
        v[c] = __ldg(reinterpret_cast<const float4*>(in_b + (static_cast<size_t>(iy) * a.W + ix) * a.Cin + g_ci));
      step();
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) step();  // the other warpgroup's half of the chunk
  };
  const auto stage_b = [&](int st) { return ring + static_cast<size_t>(st) * kStageFloats + 2 * kAFloats; };
  const auto issue_b = [&](int ch) {  // one thread: packed weights of chunk `ch` -> its stage
    const int st = ch % S;
    mbar_expect_tx(&b_full[st], kBBytes);
    tma_load_1d(stage_b(st), a.w + static_cast<size_t>(ch) * 2 * kBFloats, kBBytes, &b_full[st]);
  };

  float acc[NT][TW / 2], part[NT][TW / 2];  // the sum of the retired chunks; the current chunk
#pragma unroll
  for (int t = 0; t < NT; ++t)
#pragma unroll
    for (int i = 0; i < TW / 2; ++i) acc[t][i] = part[t][i] = 0.0f;

  // Packed weights run S - 2 chunks ahead of the chunk being staged.
  if (kPacked && tid == 0)
    for (int c = 0; c < S - 2 && c < nchunks; ++c) issue_b(c);
  float4 cur[4], nxt[4];
  gather(cur);
  for (int ch = 0; ch < nchunks; ++ch) {
    const int s = ch % S;
    float* a_hi = ring + static_cast<size_t>(s) * kStageFloats;
    float* a_lo = a_hi + kAFloats;
    float* b_hi = stage_b(s);
    // every warpgroup has retired chunk ch - 1 (wgmma_wait<0> below): every stage but the one
    // issue_b filled a chunk ago is free
    __syncthreads();
    if (kPacked && tid == 0 && ch + S - 2 < nchunks) issue_b(ch + S - 2);
    if (ch + 1 < nchunks) gather(nxt);  // loads in flight across the stores, barrier and MMAs
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float4 h, l;
      split_tf32(cur[c].x, h.x, l.x); split_tf32(cur[c].y, h.y, l.y);
      split_tf32(cur[c].z, h.z, l.z); split_tf32(cur[c].w, h.w, l.w);
      const int off = (4 * half + c) * (kTcM * 4) + (row >> 3) * 32 + (row & 7) * 4;  // floats
      *reinterpret_cast<float4*>(a_hi + off) = h;
      *reinterpret_cast<float4*>(a_lo + off) = l;
    }
    if (!kPacked) {  // B element (n, k) = W[k][n]; thread -> (n = e % N, k-chunk = e / N)
      float* b_lo = b_hi + kBFloats;
      const int k0 = ch * kTcKc;
      for (int e = tid; e < N * (kTcKc / 4); e += kTcThreads) {
        const int n = e % N, c = e / N;
        float4 v;
        float* vp = reinterpret_cast<float*>(&v);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int kk = k0 + 4 * c + j;
          vp[j] = (kk < K) ? __ldg(a.w + static_cast<size_t>(kk) * a.Cout + a.n_off + n) : 0.0f;
        }
        float4 h, l;
        split_tf32(v.x, h.x, l.x); split_tf32(v.y, h.y, l.y);
        split_tf32(v.z, h.z, l.z); split_tf32(v.w, h.w, l.w);
        const int off = c * (N * 4) + (n >> 3) * 32 + (n & 7) * 4;
        *reinterpret_cast<float4*>(b_hi + off) = h;
        *reinterpret_cast<float4*>(b_lo + off) = l;
      }
    }
    fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the tensor core
    __syncthreads();
    if (kPacked) mbar_wait(&b_full[s], static_cast<uint32_t>(ch / S) & 1u);

    const uint32_t ah = smem_u32(a_hi) + wg * 8 * kSbo;  // this warpgroup's 64 rows
    const uint32_t al = smem_u32(a_lo) + wg * 8 * kSbo;
    const uint32_t bh = smem_u32(b_hi), bl = bh + kBFloats * 4;
#pragma unroll
    for (int t = 0; t < NT; ++t) fence_operands(part[t]);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < kTcKc / 8; ++ks) {
      const uint64_t dah = make_kmajor_desc(ah + ks * 2 * kALbo, kALbo, kSbo);
      const uint64_t dal = make_kmajor_desc(al + ks * 2 * kALbo, kALbo, kSbo);
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        const uint32_t nb = t * (TW / 8) * kSbo;  // column tile t: TW / 8 groups of 8 rows of B
        const uint64_t dbh = make_kmajor_desc(bh + nb + ks * 2 * kBLbo, kBLbo, kSbo);
        const uint64_t dbl = make_kmajor_desc(bl + nb + ks * 2 * kBLbo, kBLbo, kSbo);
        wgmma_tf32<TW>(part[t], dah, dbh, ks > 0);  // a fresh partial per chunk
        wgmma_tf32<TW>(part[t], dah, dbl, 1);
        wgmma_tf32<TW>(part[t], dal, dbh, 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      fence_operands(part[t]);
#pragma unroll
      for (int i = 0; i < TW / 2; ++i) acc[t][i] = __fadd_rn(acc[t][i], part[t][i]);
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) cur[c] = nxt[c];
  }

  // ---- epilogue: fragment (row r0 + 8i, column 8c + 2(lane % 4) + j) is acc[t][4c + 2i + j] ----
  const int lane = tid & 31, warp_in_wg = (tid >> 5) & 3;
  const int r0 = wg * 64 + warp_in_wg * 16 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const long long p = static_cast<long long>(blockIdx.x) * kTcM + r0 + 8 * i;
    if (p >= total_px) continue;
    float* dst = a.out + static_cast<size_t>(p) * a.Cout + a.n_off;
#pragma unroll
    for (int t = 0; t < NT; ++t) {
#pragma unroll
      for (int c = 0; c < TW / 8; ++c) {
        const int n = t * TW + 8 * c + 2 * (lane & 3);
        float2 o = make_float2(acc[t][4 * c + 2 * i], acc[t][4 * c + 2 * i + 1]);
        if (a.bias) { o.x += __ldg(a.bias + a.n_off + n); o.y += __ldg(a.bias + a.n_off + n + 1); }
        if (a.relu) { o.x = fmaxf(o.x, 0.0f); o.y = fmaxf(o.y, 0.0f); }
        *reinterpret_cast<float2*>(dst + n) = o;
      }
    }
  }
}

// packed[chunk][half: hi, lo][kchunk 0..7][n 0..N-1][4]: chunk c's B operand (both halves) is one
// contiguous block of 2 * N * 32 floats in exactly the shared-memory layout the MMA reads.
__global__ void __launch_bounds__(256)
conv_tc_pack_kernel(const float* __restrict__ w, float* __restrict__ packed, int K, int N,
                    int nchunks) {
  const long long total = static_cast<long long>(nchunks) * 8 * N;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int n = static_cast<int>(e % N);
    const int c = static_cast<int>((e / N) % 8);
    const int ch = static_cast<int>(e / (static_cast<long long>(N) * 8));
    float4 h, l;
    float* hp = reinterpret_cast<float*>(&h);
    float* lp = reinterpret_cast<float*>(&l);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int kk = ch * kTcKc + 4 * c + j;
      const float v = (kk < K) ? __ldg(w + static_cast<size_t>(kk) * N + n) : 0.0f;
      split_tf32(v, hp[j], lp[j]);
    }
    float* base = packed + static_cast<size_t>(ch) * 2 * N * kTcKc;
    const int off = c * (N * 4) + (n >> 3) * 32 + (n & 7) * 4;
    *reinterpret_cast<float4*>(base + off) = h;
    *reinterpret_cast<float4*>(base + N * kTcKc + off) = l;
  }
}

static bool tc_shape_ok(int Cin, int Cout) {
  return Cin % 4 == 0 && Cout % 16 == 0 && Cout <= kTcMaxCout && Cout >= 16;
}

template <int N, bool kPacked>
static int launch_n(TcConvArgs a, cudaStream_t stream) {
  auto kern = conv2d_wgmma_kernel<N, kPacked>;
  int dev = 0, max_smem = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (e != cudaSuccess) return static_cast<int>(e);
  // 1 KB left for the static shared memory (the stage barriers)
  a.stages = (kTcMaxStages * stage_bytes<N>() + 1024 <= static_cast<size_t>(max_smem)) ? kTcMaxStages : 2;
  const size_t smem = a.stages * stage_bytes<N>();
  e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return static_cast<int>(e);
  const long long total_px = static_cast<long long>(a.B) * a.OH * a.OW;
  kern<<<static_cast<unsigned>((total_px + kTcM - 1) / kTcM), kTcThreads, smem, stream>>>(a);
  return static_cast<int>(cudaGetLastError());
}

// One launch over output columns [a.n_off, a.n_off + n_cols), n_cols a multiple of 16 <= 128.
template <bool kPacked>
static int launch_any_n(const TcConvArgs& a, int n_cols, cudaStream_t stream) {
  switch (n_cols) {
#define HDRNET_TC_CASE(N) case N: return launch_n<N, kPacked>(a, stream);
    HDRNET_TC_CASE(16) HDRNET_TC_CASE(32) HDRNET_TC_CASE(48) HDRNET_TC_CASE(64)
    HDRNET_TC_CASE(80) HDRNET_TC_CASE(96) HDRNET_TC_CASE(112) HDRNET_TC_CASE(128)
#undef HDRNET_TC_CASE
    default: return HDRNET_E_UNSUPPORTED;
  }
}

// Returns HDRNET_E_UNSUPPORTED when the shapes do not suit this path (the caller then runs the
// CUDA-core kernel in cnn.cu).
int launch_conv_wgmma(const float* in, const float* w, const float* bias, float* out, int B,
                      int H, int W, int Cin, int Cout, int k, int stride, int relu, int OH,
                      int OW, int pad_t, int pad_l, cudaStream_t stream) {
  if (!tc_shape_ok(Cin, Cout)) return HDRNET_E_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(in) & 15u) || (reinterpret_cast<uintptr_t>(out) & 15u))
    return HDRNET_E_UNSUPPORTED;
  TcConvArgs a;
  a.in = in; a.w = w; a.bias = bias; a.out = out;
  a.B = B; a.H = H; a.W = W; a.Cin = Cin; a.OH = OH; a.OW = OW; a.Cout = Cout; a.k = k;
  a.stride = stride; a.pad_t = pad_t; a.pad_l = pad_l; a.relu = relu; a.stages = 2;
  for (a.n_off = 0; a.n_off < Cout; a.n_off += kTcMaxN) {
    const int rc = launch_any_n<false>(a, std::min(kTcMaxN, Cout - a.n_off), stream);
    if (rc != 0) return rc;
  }
  return 0;
}

}  // namespace hdrnet_b200

using namespace hdrnet_b200;

extern "C" {

size_t hdrnet_conv2d_tc_packed_bytes(int k, int Cin, int Cout) {
  if ((k != 1 && k != 3) || !tc_shape_ok(Cin, Cout)) return 0;
  const int K = k * k * Cin;
  const size_t nchunks = (K + kTcKc - 1) / kTcKc;
  return nchunks * 2 * static_cast<size_t>(Cout) * kTcKc * sizeof(float);
}

int hdrnet_conv2d_tc_pack_f32(const float* w, float* packed, int k, int Cin, int Cout,
                              void* stream) {
  if (hdrnet_conv2d_tc_packed_bytes(k, Cin, Cout) == 0) return HDRNET_E_UNSUPPORTED;
  if (!w || !packed) return HDRNET_E_NULL_POINTER;
  const int K = k * k * Cin, nchunks = (K + kTcKc - 1) / kTcKc;
  const long long total = static_cast<long long>(nchunks) * 8 * Cout;
  conv_tc_pack_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0,
                        static_cast<cudaStream_t>(stream)>>>(w, packed, K, Cout, nchunks);
  return static_cast<int>(cudaGetLastError());
}

int hdrnet_conv2d_nhwc_tc_f32(const float* in, const float* packed_w, const float* bias,
                              float* out, int B, int H, int W, int Cin, int Cout, int k,
                              int stride, int relu, void* stream) {
  if (B < 0 || H < 1 || W < 1 || Cin < 1 || Cout < 1) return HDRNET_E_BAD_SHAPE;
  if ((k != 1 && k != 3) || (stride != 1 && stride != 2) || !tc_shape_ok(Cin, Cout))
    return HDRNET_E_UNSUPPORTED;
  if (Cout > kTcMaxN) return HDRNET_E_UNSUPPORTED;  // a chunk's packed tile holds every column
  if (B == 0) return HDRNET_OK;
  if (!in || !packed_w || !out) return HDRNET_E_NULL_POINTER;
  if ((reinterpret_cast<uintptr_t>(in) & 15u) || (reinterpret_cast<uintptr_t>(out) & 15u) ||
      (reinterpret_cast<uintptr_t>(packed_w) & 15u))
    return HDRNET_E_UNSUPPORTED;
  TcConvArgs a;
  a.in = in; a.w = packed_w; a.bias = bias; a.out = out;
  a.B = B; a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.k = k; a.stride = stride; a.relu = relu;
  a.OH = (H + stride - 1) / stride;
  a.OW = (W + stride - 1) / stride;
  int tot = (a.OH - 1) * stride + k - H; if (tot < 0) tot = 0; a.pad_t = tot / 2;
  tot = (a.OW - 1) * stride + k - W; if (tot < 0) tot = 0; a.pad_l = tot / 2;
  a.stages = 2;
  a.n_off = 0;
  return launch_any_n<true>(a, Cout, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
