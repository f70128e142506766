// ws_traffic.cu -- speed-of-light probe for the memory traffic of the issuer-warp slice-apply kernel
// (slice_apply_rows_async_kernel<5, lean, 384, 2, slab warp>) at the headline shape: 8 x 3840 x 2160
// float32 pixels, grid 16x16x8.  The probe keeps the kernel's plan and control flow -- 264 CTAs x 384
// threads (10 math warps, the issuer, the slab warp), a 4-stage ring of 1280-pixel items, the same
// bulk loads and bulk store, the same mbarriers -- and replaces the corner gather by a trivial
// per-pixel op.  Forms:
//   a  ring only: input + guide in, output out (28 B/px)
//   b  a + the slab warp writing every row's y-blended slab to the workspace (grid rows read from L2)
//   c  b + the texture fetches the real kernel makes (the 5 texture chunks of every pixel, at the
//      real texel addresses), read back from the workspace
//   d  c with L2 hints: pixels evict_first, workspace stores evict_last, released rows discarded
// and, in the same interleaved bursts, a device-to-device cudaMemcpyAsync moving the same bytes
// (14 B/px read + 14 B/px written) and the real kernel of every library given on the command line.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I include -o tools/ubench/bin/ws_traffic \
//        tools/ubench/ws_traffic.cu -ldl
//   tools/ubench/bin/ws_traffic [lib.so ...]      (prints one line per form: median / min / max ms)
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../hdrnet_b200/csrc/common.cuh"

using namespace hdrnet_b200;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at line %d\n", cudaGetErrorString(e_), __LINE__); exit(2); } } while (0)

constexpr int B = 8, H = 2160, W = 3840, GH = 16, GW = 16, GD = 8;
// make_tma_plan at this shape (tex_mode, 352 threads - the issuer, 2 grid rows): checked against the
// library's hdrnet_slice_apply_plan_ws in main()
constexpr int kThreads = 384, kMathWarps = 10, kSegPx = 1280, kNseg = 3, kStages = 4, kCtas = 264;
constexpr int kRowFloats = GW * GD * 12;              // one slab row: 6144 bytes = 48 lines
constexpr int kOffGuide = kSegPx * 12, kStageBytes = kSegPx * 16, kOffStage = 256;
constexpr int kSmem = kOffStage + kStages * kStageBytes;
enum { kRing = 0, kSlab = 1, kTex = 2, kHinted = 3 };

template <int F>
__global__ void __launch_bounds__(kThreads, 2)
probe_kernel(const float* __restrict__ in, const float* __restrict__ guide, float* __restrict__ out,
             float* ws, const float* __restrict__ grid, cudaTextureObject_t tex) {
  constexpr bool kSlabWarp = F >= kSlab;
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  uint64_t* done = full + kStages;
  uint64_t* slab_full = done + kStages;
  uint64_t* row_free = slab_full + 2;
  unsigned char* stage_base = smem + kOffStage;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long total_items = static_cast<long long>(B) * H * kNseg;
  const long long i_begin = total_items * blockIdx.x / gridDim.x;
  const long long i_end = total_items * (blockIdx.x + 1) / gridDim.x;
  if (i_end <= i_begin) return;
  const long long r_begin = i_begin / kNseg, r_end = (i_end - 1) / kNseg + 1;
  const int x_first = static_cast<int>(i_begin - r_begin * kNseg) * kSegPx;
  const int x_last = min(W, (static_cast<int>((i_end - 1) - (r_end - 1) * kNseg) + 1) * kSegPx);
  auto row_x0 = [&](long long row) { return row == r_begin ? x_first : 0; };
  auto row_x1 = [&](long long row) { return row == r_end - 1 ? x_last : W; };
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&done[s], kMathWarps); }
    for (int i = 0; i < 2; ++i) { mbar_init(&slab_full[i], 1); mbar_init(&row_free[i], 1); }
    fence_mbar_init();
  }
  __syncthreads();
  auto arrive = [&](uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
  };

  if (warp == kMathWarps + 1) {   // ---- slab warp
    if constexpr (kSlabWarp) {
      constexpr int n4 = kRowFloats / 4;
      float4* ws4 = reinterpret_cast<float4*>(ws);
      const float4* g4 = reinterpret_cast<const float4*>(grid);
      const uint64_t ws_pol = l2_policy_evict_last();
      auto discard_row = [&](long long r) {
        if (row_x0(r) != 0 || row_x1(r) != W) return;
        const unsigned char* base = reinterpret_cast<const unsigned char*>(ws4 + static_cast<size_t>(r) * n4);
        for (int l = lane; l < kRowFloats * 4 / 128; l += 32) l2_discard_line(base + 128 * l);
      };
      for (long long row = r_begin; row < r_end; ++row) {
        const int rowk = static_cast<int>(row - r_begin), rb = rowk & 1;
        if (rowk >= 2) mbar_wait(&row_free[rb], static_cast<uint32_t>((rowk >> 1) - 1) & 1u);
        const int b = static_cast<int>(row / H), y = static_cast<int>(row - static_cast<long long>(b) * H);
        const Axis ay = spatial_axis(y, static_cast<float>(GH) / H);
        const float4* a4 = g4 + static_cast<size_t>(b * GH + clampi(ay.i0, 0, GH - 1)) * n4;
        const float4* b4 = g4 + static_cast<size_t>(b * GH + clampi(ay.i0 + 1, 0, GH - 1)) * n4;
        float4* wrow = ws4 + static_cast<size_t>(row) * n4;
        for (int e = lane; e < n4; e += 32) {
          const float4 u = __ldg(a4 + e), v = __ldg(b4 + e);
          const float4 r = make_float4(u.x + ay.f * (v.x - u.x), u.y + ay.f * (v.y - u.y),
                                       u.z + ay.f * (v.z - u.z), u.w + ay.f * (v.w - u.w));
          if constexpr (F == kHinted) st_global_hint(wrow + e, r, ws_pol);
          else wrow[e] = r;
        }
        __threadfence();
        __syncwarp();
        if (lane == 0) arrive(&slab_full[rb]);
        if constexpr (F == kHinted) if (rowk >= 2) discard_row(row - 2);
      }
      if constexpr (F == kHinted)
        for (long long row = max(r_begin, r_end - 2); row < r_end; ++row) {
          const int rowk = static_cast<int>(row - r_begin);
          mbar_wait(&row_free[rowk & 1], static_cast<uint32_t>(rowk >> 1) & 1u);
          discard_row(row);
        }
    }
    return;
  }

  if (warp == kMathWarps) {   // ---- issuer (lane 0)
    if (lane != 0) return;
    const uint64_t px_pol = l2_policy_evict_first();
    long long l_row = r_begin;
    int l_x0 = x_first, l_s = 0;
    auto issue_next_load = [&]() {
      if (l_row >= r_end) return;
      const int npx = min(kSegPx, W - l_x0);
      unsigned char* st = stage_base + static_cast<size_t>(l_s) * kStageBytes;
      const size_t pix = static_cast<size_t>(l_row) * W + l_x0;
      mbar_expect_tx(&full[l_s], static_cast<uint32_t>(npx) * 16u);
      if constexpr (F == kHinted) {
        tma_load_1d(st, in + pix * 3, static_cast<uint32_t>(npx) * 12u, &full[l_s], px_pol);
        tma_load_1d(st + kOffGuide, guide + pix, static_cast<uint32_t>(npx) * 4u, &full[l_s], px_pol);
      } else {
        tma_load_1d(st, in + pix * 3, static_cast<uint32_t>(npx) * 12u, &full[l_s]);
        tma_load_1d(st + kOffGuide, guide + pix, static_cast<uint32_t>(npx) * 4u, &full[l_s]);
      }
      if (++l_s == kStages) l_s = 0;
      l_x0 += kSegPx;
      if (l_x0 >= row_x1(l_row)) { l_x0 = 0; ++l_row; }
    };
    for (int i = 0; i < kStages - 1; ++i) issue_next_load();
    int s = 0;
    uint32_t ph = 0;
    for (long long row = r_begin; row < r_end; ++row) {
      for (int x0 = row_x0(row); x0 < row_x1(row); x0 += kSegPx) {
        mbar_wait(&done[s], ph);
        const int npx = min(kSegPx, W - x0);
        unsigned char* st = stage_base + static_cast<size_t>(s) * kStageBytes;
        const size_t pix = static_cast<size_t>(row) * W + x0;
        if constexpr (F == kHinted) tma_store_1d(out + pix * 3, st, static_cast<uint32_t>(npx) * 12u, px_pol);
        else tma_store_1d(out + pix * 3, st, static_cast<uint32_t>(npx) * 12u);
        tma_store_commit();
        if (l_row < r_end) {
          tma_store_wait_read<1>();
          issue_next_load();
        }
        if (++s == kStages) { s = 0; ph ^= 1u; }
      }
      if constexpr (kSlabWarp) arrive(&row_free[static_cast<int>(row - r_begin) & 1]);
    }
    tma_store_wait_all<0>();
    return;
  }

  // ---- math warps: out = in * guide (+ the texture chunks' sum)
  const int q = warp * 32 + lane;
  const float scale_x = static_cast<float>(GW) / W;
  int s = 0;
  uint32_t ph = 0;
  for (long long row = r_begin; row < r_end; ++row) {
    const int rowk = static_cast<int>(row - r_begin);
    if constexpr (kSlabWarp) mbar_wait(&slab_full[rowk & 1], static_cast<uint32_t>(rowk >> 1) & 1u);
    const int tex_base = static_cast<int>(row) * GW * GD * 3;
    for (int x0 = row_x0(row); x0 < row_x1(row); x0 += kSegPx) {
      const int npx = min(kSegPx, W - x0);
      unsigned char* st = stage_base + static_cast<size_t>(s) * kStageBytes;
      mbar_wait(&full[s], ph);
      if (q * 4 < npx) {
        float4* t4 = reinterpret_cast<float4*>(st) + 3 * q;
        float v[12];
        *reinterpret_cast<float4*>(v) = t4[0];
        *reinterpret_cast<float4*>(v + 4) = t4[1];
        *reinterpret_cast<float4*>(v + 8) = t4[2];
        const float4 gq = lds128(reinterpret_cast<const float4*>(st + kOffGuide) + q);
        const float gv[4] = {gq.x, gq.y, gq.z, gq.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float acc = 0.0f;
          if constexpr (F >= kTex) {   // the real kernel's texture chunks: corners (z0, x1) parts 1-2, (z1, x1) parts 0-2
            const Axis ax = spatial_axis(x0 + 4 * q + i, scale_x);
            const int xc = clampi(ax.i0 + 1, 0, GW - 1);
            const Axis az = range_axis(gv[i], static_cast<float>(GD));
            const int t2 = tex_base + (xc * GD + clampi(az.i0, 0, GD - 1)) * 3;
            const int t3 = tex_base + (xc * GD + clampi(az.i0 + 1, 0, GD - 1)) * 3;
            const float4 c1 = tex1Dfetch<float4>(tex, t2 + 1), c2 = tex1Dfetch<float4>(tex, t2 + 2);
            const float4 d0 = tex1Dfetch<float4>(tex, t3), d1 = tex1Dfetch<float4>(tex, t3 + 1),
                         d2 = tex1Dfetch<float4>(tex, t3 + 2);
            acc = c1.x + c2.y + d0.z + d1.w + d2.x;
          }
#pragma unroll
          for (int c = 0; c < 3; ++c) v[3 * i + c] = fmaf(v[3 * i + c], gv[i], acc);
        }
        t4[0] = *reinterpret_cast<float4*>(v);
        t4[1] = *reinterpret_cast<float4*>(v + 4);
        t4[2] = *reinterpret_cast<float4*>(v + 8);
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) arrive(&done[s]);
      if (++s == kStages) { s = 0; ph ^= 1u; }
    }
  }
}

__global__ void fill_kernel(float* p, size_t n, unsigned seed) {   // hashed uniform [0, 1)
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    unsigned h = static_cast<unsigned>(i) * 0x9E3779B1u ^ seed;
    h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
    p[i] = (h >> 8) * (1.0f / 16777216.0f);
  }
}

typedef int (*apply_ws_fn)(const float*, const float*, const float*, float*, int, int, int, int, int, int,
                           int, int, int, int, void*, size_t, void*);
typedef int (*plan_ws_fn)(int, int, int, int, int, int, int, int, int, int, int*, int*, int*, int*);

int main(int argc, char** argv) {
  const size_t npix = static_cast<size_t>(B) * H * W, ngrid = static_cast<size_t>(B) * GH * GW * GD * 12;
  const size_t nws = static_cast<size_t>(B) * H * kRowFloats * 4;
  float *in, *gd, *out, *ws, *grid, *cpy_src, *cpy_dst;
  CK(cudaMalloc(&in, npix * 12)); CK(cudaMalloc(&gd, npix * 4)); CK(cudaMalloc(&out, npix * 12));
  CK(cudaMalloc(&ws, nws)); CK(cudaMalloc(&grid, ngrid * 4));
  CK(cudaMalloc(&cpy_src, npix * 14)); CK(cudaMalloc(&cpy_dst, npix * 14));
  fill_kernel<<<1024, 256>>>(in, npix * 3, 1u);
  fill_kernel<<<1024, 256>>>(gd, npix, 2u);
  fill_kernel<<<1024, 256>>>(grid, ngrid, 3u);
  CK(cudaMemset(cpy_src, 0, npix * 14));
  CK(cudaDeviceSynchronize());
  cudaResourceDesc rd = {};
  rd.resType = cudaResourceTypeLinear;
  rd.res.linear.devPtr = ws;
  rd.res.linear.desc = cudaCreateChannelDesc<float4>();
  rd.res.linear.sizeInBytes = nws;
  cudaTextureDesc td = {};
  td.readMode = cudaReadModeElementType;
  cudaTextureObject_t tex = 0;
  CK(cudaCreateTextureObject(&tex, &rd, &td, nullptr));
  CK(cudaFuncSetAttribute(probe_kernel<kRing>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  CK(cudaFuncSetAttribute(probe_kernel<kSlab>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  CK(cudaFuncSetAttribute(probe_kernel<kTex>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  CK(cudaFuncSetAttribute(probe_kernel<kHinted>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));

  struct Form { std::string name; apply_ws_fn apply; int form; };
  std::vector<Form> forms = {{"a ring only", nullptr, kRing}, {"b + slab rows to the workspace", nullptr, kSlab},
                             {"c + texture fetches of the workspace", nullptr, kTex},
                             {"d = c with L2 hints and discards", nullptr, kHinted},
                             {"cudaMemcpyAsync D2D, 14 B/px each way", nullptr, -1}};
  for (int i = 1; i < argc; ++i) {
    void* h = dlopen(argv[i], RTLD_NOW | RTLD_LOCAL);
    if (!h) { printf("cannot load %s: %s\n", argv[i], dlerror()); return 2; }
    auto apply = reinterpret_cast<apply_ws_fn>(dlsym(h, "hdrnet_slice_apply_f32_ws"));
    auto plan = reinterpret_cast<plan_ws_fn>(dlsym(h, "hdrnet_slice_apply_plan_ws"));
    if (!apply || !plan) { printf("%s: missing symbols\n", argv[i]); return 2; }
    int variant = 0, ctas = 0, threads = 0, smem = 0;
    plan(B, H, W, GH, GW, GD, 3, 3, 1, 1, &variant, &ctas, &threads, &smem);
    printf("%s plans variant %d, %d CTAs x %d threads, %d B smem (probe: %d x %d)\n", argv[i], variant, ctas,
           threads, smem, kCtas, kThreads);
    forms.push_back({std::string("real kernel, ") + argv[i], apply, -2});
  }
  auto launch = [&](const Form& f) {
    switch (f.form) {
      case kRing: probe_kernel<kRing><<<kCtas, kThreads, kSmem>>>(in, gd, out, ws, grid, tex); break;
      case kSlab: probe_kernel<kSlab><<<kCtas, kThreads, kSmem>>>(in, gd, out, ws, grid, tex); break;
      case kTex: probe_kernel<kTex><<<kCtas, kThreads, kSmem>>>(in, gd, out, ws, grid, tex); break;
      case kHinted: probe_kernel<kHinted><<<kCtas, kThreads, kSmem>>>(in, gd, out, ws, grid, tex); break;
      case -1: CK(cudaMemcpyAsync(cpy_dst, cpy_src, npix * 14, cudaMemcpyDeviceToDevice)); break;
      default: {
        const int rc = f.apply(grid, gd, in, out, B, H, W, GH, GW, GD, 3, 3, 1, 0, ws, nws, nullptr);
        if (rc) { printf("%s: rc %d\n", f.name.c_str(), rc); exit(1); }
      }
    }
  };
  for (const Form& f : forms) { launch(f); CK(cudaGetLastError()); CK(cudaDeviceSynchronize()); }
  const int rounds = 9, iters = 40;
  std::vector<std::vector<float>> t(forms.size());
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  for (int r = 0; r < rounds; ++r)
    for (size_t k = 0; k < forms.size(); ++k) {
      for (int i = 0; i < 3; ++i) launch(forms[k]);
      CK(cudaEventRecord(a));
      for (int i = 0; i < iters; ++i) launch(forms[k]);
      CK(cudaEventRecord(b));
      CK(cudaEventSynchronize(b));
      CK(cudaGetLastError());
      float ms = 0;
      CK(cudaEventElapsedTime(&ms, a, b));
      t[k].push_back(ms / iters);
    }
  printf("8 x 3840 x 2160, grid 16x16x8; median / min / max of %d interleaved bursts of %d launches\n", rounds, iters);
  for (size_t k = 0; k < forms.size(); ++k) {
    std::vector<float> v = t[k];
    std::sort(v.begin(), v.end());
    const float med = v[v.size() / 2];
    printf("%-60s %.4f ms  (min %.4f max %.4f)  %.3f TB/s at 28 B/px\n", forms[k].name.c_str(), med, v.front(),
           v.back(), npix * 28.0 / med / 1e9);
  }
  return 0;
}
