// cabi_check.cu -- torch-free check of a slice-apply kernel variant through the C-ABI: a few
// seconds on a GPU machine instead of a Python start-up (meant for the first runs of an untested
// variant).
//   nvcc -O2 -std=c++17 -I include -o tools/ubench/bin/cabi_check tools/cabi_check.cu -ldl
//   tools/ubench/bin/cabi_check [variant=8] [B=2] [H=64] [W=3840] [gh=16] [gw=16] [gd=8] [iters=20]
// Compares `variant` with HDRNET_VARIANT_GENERIC (one thread per pixel, the reference's own
// summation order) on seeded random inputs -- max |diff| / max |ref|, bar 1e-5 -- runs it twice
// (barrier phases of a second launch), then times `iters` launches with CUDA events.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "hdrnet_b200.h"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at line %d\n", cudaGetErrorString(e_), __LINE__); return 2; } } while (0)

typedef int (*apply_ws_fn)(const float*, const float*, const float*, float*, int, int, int, int, int, int,
                           int, int, int, int, void*, size_t, void*);
typedef size_t (*ws_bytes_fn)(int, int, int, int);

int main(int argc, char** argv) {
  const int variant = argc > 1 ? atoi(argv[1]) : 8;
  const int B = argc > 2 ? atoi(argv[2]) : 2, H = argc > 3 ? atoi(argv[3]) : 64, W = argc > 4 ? atoi(argv[4]) : 3840;
  const int gh = argc > 5 ? atoi(argv[5]) : 16, gw = argc > 6 ? atoi(argv[6]) : 16, gd = argc > 7 ? atoi(argv[7]) : 8;
  const int iters = argc > 8 ? atoi(argv[8]) : 20;
  const char* path = getenv("HDRNET_B200_LIB") ? getenv("HDRNET_B200_LIB") : "hdrnet_b200/lib/libhdrnet_b200.so";
  void* h = dlopen(path, RTLD_NOW);
  if (!h) { printf("cannot load %s: %s\n", path, dlerror()); return 2; }
  auto apply_ws = reinterpret_cast<apply_ws_fn>(dlsym(h, "hdrnet_slice_apply_f32_ws"));
  auto ws_bytes = reinterpret_cast<ws_bytes_fn>(dlsym(h, "hdrnet_slice_apply_workspace_bytes"));
  if (!apply_ws || !ws_bytes) { printf("missing symbols\n"); return 2; }

  const size_t npix = static_cast<size_t>(B) * H * W, ngrid = static_cast<size_t>(B) * gh * gw * gd * 12;
  std::mt19937 rng(1234);
  std::normal_distribution<float> nd(0.f, 1.f);
  std::uniform_real_distribution<float> ud(0.f, 1.f);
  std::vector<float> hg(ngrid), hu(npix), hi(npix * 3), ho(npix * 3), hr(npix * 3);
  for (auto& v : hg) v = nd(rng);
  for (auto& v : hu) v = ud(rng);
  for (auto& v : hi) v = nd(rng);
  hu[0] = 0.f; hu[1] = 1.f; hu[2] = -0.3f; hu[3] = 1.7f;   // clamped depth cells
  float *dg, *du, *di, *dout, *dref;
  void* ws;
  const size_t nws = ws_bytes(B, H, gw, gd);
  CK(cudaMalloc(&dg, ngrid * 4)); CK(cudaMalloc(&du, npix * 4)); CK(cudaMalloc(&di, npix * 12));
  CK(cudaMalloc(&dout, npix * 12)); CK(cudaMalloc(&dref, npix * 12)); CK(cudaMalloc(&ws, nws));
  CK(cudaMemcpy(dg, hg.data(), ngrid * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(du, hu.data(), npix * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(di, hi.data(), npix * 12, cudaMemcpyHostToDevice));
  int rc = apply_ws(dg, du, di, dref, B, H, W, gh, gw, gd, 3, 3, 1, HDRNET_VARIANT_GENERIC, ws, nws, nullptr);
  if (rc) { printf("generic kernel: rc %d\n", rc); return 2; }
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(hr.data(), dref, npix * 12, cudaMemcpyDeviceToHost));
  double refmax = 0;
  for (float v : hr) refmax = std::fmax(refmax, std::fabs(v));
  int status = 0;
  for (int rep = 0; rep < 2; ++rep) {
    CK(cudaMemset(dout, 0xff, npix * 12));
    rc = apply_ws(dg, du, di, dout, B, H, W, gh, gw, gd, 3, 3, 1, variant, ws, nws, nullptr);
    if (rc) { printf("variant %d: rc %d (%s)\n", variant, rc, rc < 0 ? "library code" : cudaGetErrorString((cudaError_t)rc)); return 1; }
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("variant %d: launch %d failed: %s\n", variant, rep, cudaGetErrorString(e)); return 1; }
    CK(cudaMemcpy(ho.data(), dout, npix * 12, cudaMemcpyDeviceToHost));
    double worst = 0; size_t at = 0, bad = 0;
    for (size_t i = 0; i < ho.size(); ++i) {
      const double d = std::fabs(static_cast<double>(ho[i]) - hr[i]);
      if (!(d <= 1e-5 * refmax)) ++bad;
      if (!(d <= worst)) { worst = d; at = i; }
    }
    printf("variant %d launch %d: max|diff|/max|ref| = %.3e at element %zu (pixel %zu of row %zu), %zu of %zu over 1e-5\n",
           variant, rep, worst / refmax, at, (at / 3) % W, at / 3 / W, bad, ho.size());
    if (bad) {
      status = 1;
      for (size_t i = 0, shown = 0; i < ho.size() && shown < 8; ++i)
        if (!(std::fabs(static_cast<double>(ho[i]) - hr[i]) <= 1e-5 * refmax)) {
          printf("   [%zu] row %zu x %zu c %zu: got %g want %g\n", i, i / 3 / W, (i / 3) % W, i % 3, ho[i], hr[i]);
          ++shown;
        }
    }
  }
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  for (int i = 0; i < 3; ++i) apply_ws(dg, du, di, dout, B, H, W, gh, gw, gd, 3, 3, 1, variant, ws, nws, nullptr);
  CK(cudaEventRecord(a));
  for (int i = 0; i < iters; ++i) apply_ws(dg, du, di, dout, B, H, W, gh, gw, gd, 3, 3, 1, variant, ws, nws, nullptr);
  CK(cudaEventRecord(b));
  CK(cudaEventSynchronize(b));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, a, b));
  ms /= iters;
  printf("variant %d: %.4f ms per call, %.1f MP/s, %.1f GB/s at 28 B/px\n", variant, ms, npix / ms / 1e3, npix * 28.0 / ms / 1e6);
  return status;
}
