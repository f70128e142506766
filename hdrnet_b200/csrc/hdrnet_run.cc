// hdrnet_run -- runs a frozen model (hdrnet_b200.bin.freeze_model) on one image through the C-ABI
// alone: the deployment counterpart of the reference's benchmark/ program (benchmark/src/main.cc,
// processor.cc), with the same flags.  It reads the image from a .npy file (H x W x 3 uint8 or
// uint16, C order, as np.save writes it), runs --burn_iters untimed calls and --iters calls timed
// one by one with CUDA events, and writes <model>.npy (the result of the last call) and <model>.json
// (model kind, image size, mean and min milliseconds per call) to --output_directory, <model> being
// the checkpoint file's name without its extension.  No image codecs: decode and encode elsewhere.
//
//   hdrnet_run --checkpoint_path M.hdrnet --input_path X.npy --output_directory D
//              [--burn_iters 3] [--iters 10] [--output_bit_depth 8|16]
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "hdrnet_b200.h"

namespace {

[[noreturn]] void fail(const std::string& msg) {
  std::fprintf(stderr, "hdrnet_run: %s\n", msg.c_str());
  std::exit(1);
}

void check_cuda(cudaError_t e, const char* what) {
  if (e != cudaSuccess) fail(std::string(what) + ": " + cudaGetErrorString(e));
}

void check(int rc, const char* what) {
  if (rc != HDRNET_OK) fail(std::string(what) + ": " + hdrnet_b200_error_string(rc));
}

std::vector<char> read_file(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  if (!f) fail("cannot open " + path);
  return std::vector<char>(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}

// A plain .npy image: version 1.0 / 2.0 header, descr '|u1' or '<u2', fortran_order False,
// shape (H, W, 3).  Anything else is refused with a message.
struct Npy { int bits = 0, H = 0, W = 0; std::vector<char> data; };

Npy read_npy(const std::string& path) {
  const std::vector<char> f = read_file(path);
  if (f.size() < 10 || std::memcmp(f.data(), "\x93NUMPY", 6) != 0) fail(path + ": not a .npy file");
  const int major = static_cast<unsigned char>(f[6]);
  size_t hlen = 0, start = 0;
  if (major == 1) {
    hlen = static_cast<unsigned char>(f[8]) | (static_cast<size_t>(static_cast<unsigned char>(f[9])) << 8);
    start = 10;
  } else if (major == 2 || major == 3) {
    if (f.size() < 12) fail(path + ": truncated .npy header");
    for (int i = 0; i < 4; ++i) hlen |= static_cast<size_t>(static_cast<unsigned char>(f[8 + i])) << (8 * i);
    start = 12;
  } else {
    fail(path + ": unknown .npy version");
  }
  if (f.size() < start + hlen) fail(path + ": truncated .npy header");
  std::string header(f.data() + start, hlen);
  header.erase(std::remove(header.begin(), header.end(), ' '), header.end());
  Npy n;
  if (header.find("'descr':'|u1'") != std::string::npos || header.find("'descr':'<u1'") != std::string::npos)
    n.bits = 8;
  else if (header.find("'descr':'<u2'") != std::string::npos)
    n.bits = 16;
  else
    fail(path + ": only uint8 ('|u1') and little-endian uint16 ('<u2') images are read, header " + header);
  if (header.find("'fortran_order':False") == std::string::npos) fail(path + ": only C-order arrays are read");
  const size_t s = header.find("'shape':(");
  if (s == std::string::npos || std::sscanf(header.c_str() + s + 9, "%d,%d,3)", &n.H, &n.W) != 2 ||
      header.compare(header.find(')', s) - 2, 2, ",3") != 0 || n.H < 1 || n.W < 1)
    fail(path + ": the image must have shape (H, W, 3), header " + header);
  const size_t bytes = static_cast<size_t>(n.H) * n.W * 3 * (n.bits / 8);
  if (f.size() - start - hlen != bytes) fail(path + ": data size does not match the header's shape");
  n.data.assign(f.begin() + start + hlen, f.end());
  return n;
}

void write_npy(const std::string& path, const void* data, int bits, int H, int W) {
  std::string header = std::string("{'descr': '") + (bits == 8 ? "|u1" : "<u2") +
                       "', 'fortran_order': False, 'shape': (" + std::to_string(H) + ", " +
                       std::to_string(W) + ", 3), }";
  const size_t total = 10 + header.size() + 1;
  header.append((64 - total % 64) % 64, ' ');
  header.push_back('\n');
  std::ofstream f(path, std::ios::binary);
  if (!f) fail("cannot write " + path);
  const unsigned short hlen = static_cast<unsigned short>(header.size());
  f.write("\x93NUMPY\x01\x00", 8);
  const char len[2] = {static_cast<char>(hlen & 0xff), static_cast<char>(hlen >> 8)};
  f.write(len, 2);
  f.write(header.data(), static_cast<std::streamsize>(header.size()));
  f.write(static_cast<const char*>(data), static_cast<std::streamsize>(static_cast<size_t>(H) * W * 3 * (bits / 8)));
  if (!f) fail("writing " + path + " failed");
}

std::string stem(const std::string& path) {
  std::string name = path.substr(path.find_last_of('/') == std::string::npos ? 0 : path.find_last_of('/') + 1);
  const size_t dot = name.find_last_of('.');
  return dot == std::string::npos || dot == 0 ? name : name.substr(0, dot);
}

const char* kind_name(int kind) {
  switch (kind) {
    case HDRNET_MODEL_CURVES: return "HDRNetCurves";
    case HDRNET_MODEL_POINTWISE_NN: return "HDRNetPointwiseNNGuide";
    case HDRNET_MODEL_GAUSSIAN_PYR_NN: return "HDRNetGaussianPyrNN";
    case HDRNET_MODEL_GAUSSIAN_PYR: return "HDRNetGaussianPyr";
    default: return "unknown";
  }
}

}  // namespace

int main(int argc, char** argv) {
  std::map<std::string, std::string> a = {{"burn_iters", "3"}, {"iters", "10"}, {"output_bit_depth", "8"}};
  for (int i = 1; i < argc; ++i) {
    std::string k = argv[i];
    if (k.rfind("--", 0) != 0) fail("unexpected argument " + k);
    k = k.substr(2);
    const size_t eq = k.find('=');
    if (eq != std::string::npos) { a[k.substr(0, eq)] = k.substr(eq + 1); continue; }
    if (i + 1 >= argc) fail("--" + k + " needs a value");
    a[k] = argv[++i];
  }
  for (const auto& kv : a)
    if (kv.first != "checkpoint_path" && kv.first != "input_path" && kv.first != "output_directory" &&
        kv.first != "burn_iters" && kv.first != "iters" && kv.first != "output_bit_depth")
      fail("unknown flag --" + kv.first);
  for (const char* req : {"checkpoint_path", "input_path", "output_directory"})
    if (!a.count(req)) fail(std::string("--") + req + " is required");
  const int burn = std::atoi(a["burn_iters"].c_str()), iters = std::atoi(a["iters"].c_str());
  const int out_bits = std::atoi(a["output_bit_depth"].c_str());
  if (burn < 0 || iters < 1) fail("--burn_iters must be >= 0 and --iters >= 1");
  if (out_bits != 8 && out_bits != 16) fail("--output_bit_depth must be 8 or 16");

  const std::vector<char> blob = read_file(a["checkpoint_path"]);
  const Npy img = read_npy(a["input_path"]);
  hdrnet_model* model = nullptr;
  check(hdrnet_model_create(blob.data(), blob.size(), &model), "loading the frozen model");
  int kind = -1;
  check(hdrnet_model_info(model, &kind, nullptr, nullptr, nullptr, nullptr, nullptr), "model info");

  const int in_fmt = img.bits == 8 ? HDRNET_PX_U8 : HDRNET_PX_U16;
  const int out_fmt = out_bits == 8 ? HDRNET_PX_U8 : HDRNET_PX_U16;
  const size_t out_bytes = static_cast<size_t>(img.H) * img.W * 3 * (out_bits / 8);
  const size_t ws_bytes = hdrnet_model_workspace_bytes(model, 1, img.H, img.W, in_fmt, out_fmt);
  void *d_in = nullptr, *d_out = nullptr, *d_ws = nullptr;
  cudaStream_t st = nullptr;
  check_cuda(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking), "stream");
  check_cuda(cudaMalloc(&d_in, img.data.size()), "cudaMalloc");
  check_cuda(cudaMalloc(&d_out, out_bytes), "cudaMalloc");
  check_cuda(cudaMalloc(&d_ws, ws_bytes), "cudaMalloc");
  check_cuda(cudaMemcpy(d_in, img.data.data(), img.data.size(), cudaMemcpyHostToDevice), "upload");
  const auto run = [&] {
    check(hdrnet_model_run_px(model, d_in, in_fmt, nullptr, 0, 0, 0, d_out, out_fmt, 1, img.H, img.W, d_ws,
                              ws_bytes, st),
          "running the model");
  };
  for (int i = 0; i < burn; ++i) run();
  cudaEvent_t t0, t1;
  check_cuda(cudaEventCreate(&t0), "event");
  check_cuda(cudaEventCreate(&t1), "event");
  double sum = 0.0, best = 1e30;
  for (int i = 0; i < iters; ++i) {
    check_cuda(cudaEventRecord(t0, st), "event record");
    run();
    check_cuda(cudaEventRecord(t1, st), "event record");
    check_cuda(cudaEventSynchronize(t1), "synchronise");
    float ms = 0.0f;
    check_cuda(cudaEventElapsedTime(&ms, t0, t1), "event time");
    sum += ms;
    best = std::min(best, static_cast<double>(ms));
  }
  std::vector<char> out(out_bytes);
  check_cuda(cudaMemcpy(out.data(), d_out, out_bytes, cudaMemcpyDeviceToHost), "download");

  const std::string dir = a["output_directory"], name = stem(a["checkpoint_path"]);
  write_npy(dir + "/" + name + ".npy", out.data(), out_bits, img.H, img.W);
  std::ostringstream js;
  js << "{\"model\": \"" << kind_name(kind) << "\", \"height\": " << img.H << ", \"width\": " << img.W
     << ", \"input_bit_depth\": " << img.bits << ", \"output_bit_depth\": " << out_bits
     << ", \"burn_iters\": " << burn << ", \"iters\": " << iters << ", \"mean_ms\": " << sum / iters
     << ", \"min_ms\": " << best << "}\n";
  std::ofstream jf(dir + "/" + name + ".json");
  if (!(jf << js.str())) fail("cannot write " + dir + "/" + name + ".json");
  std::printf("%s", js.str().c_str());

  cudaEventDestroy(t0);
  cudaEventDestroy(t1);
  cudaFree(d_in);
  cudaFree(d_out);
  cudaFree(d_ws);
  cudaStreamDestroy(st);
  check(hdrnet_model_destroy(model), "destroying the model");
  return 0;
}
