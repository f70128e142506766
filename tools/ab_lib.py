"""Same-box A/B of builds and kernel variants of libhdrnet_b200.so at the headline shape (box-to-box
spread is +-4 %, larger than most kernel changes).
    python tools/ab_lib.py SPEC [SPEC ...]      SPEC = path.so[:variant]
Every configuration is driven directly through the C-ABI (hdrnet_slice_apply_f32_ws) in
interleaved bursts; all burst times and the SM clock sampled after each burst are printed, the
median is reported.  Outputs of all configurations must be bitwise equal.  Every library path is
loaded from a private copy, so two builds at the same path name stay apart."""
import ctypes, os, shutil, statistics, sys, tempfile, torch
try:
    import pynvml
    pynvml.nvmlInit()
    _h = pynvml.nvmlDeviceGetHandleByIndex(0)
    sm_clock = lambda: pynvml.nvmlDeviceGetClockInfo(_h, pynvml.NVML_CLOCK_SM)
except Exception:
    sm_clock = lambda: 0

B, H, W, GH, GW, GD = 8, 2160, 3840, 16, 16, 8
if os.environ.get("AB_GRID"):   # e.g. AB_GRID=32,32,16
    GH, GW, GD = (int(v) for v in os.environ["AB_GRID"].split(","))
gen = torch.Generator(device="cuda").manual_seed(1234)
grid = torch.rand(B, GH, GW, GD, 12, device="cuda", generator=gen)
guide = torch.rand(B, H, W, device="cuda", generator=gen)
inp = torch.rand(B, H, W, 3, device="cuda", generator=gen)
libs, cfgs = {}, []
_tmp = tempfile.mkdtemp(prefix="ab_lib_")
for spec in sys.argv[1:]:
    parts = spec.split(":")
    path = parts[0]
    variant = int(parts[1]) if len(parts) > 1 and parts[1] else 0
    if path not in libs:
        private = os.path.join(_tmp, f"lib{len(libs)}.so")
        shutil.copy(os.path.abspath(path), private)
        lib = ctypes.CDLL(private)
        lib.hdrnet_slice_apply_workspace_bytes.restype = ctypes.c_size_t
        lib.hdrnet_slice_apply_workspace_bytes.argtypes = [ctypes.c_int] * 4
        lib.hdrnet_slice_apply_f32_ws.restype = ctypes.c_int
        lib.hdrnet_slice_apply_f32_ws.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int] * 10 + [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
        libs[path] = lib
    cfgs.append((spec, libs[path], variant))
n_ws = next(iter(libs.values())).hdrnet_slice_apply_workspace_bytes(B, H, GW, GD)
ws = torch.empty(n_ws, dtype=torch.uint8, device="cuda")
out = torch.empty_like(inp)
ref = None
stream = torch.cuda.current_stream().cuda_stream

def run(cfg):
    _, lib, variant = cfg
    rc = lib.hdrnet_slice_apply_f32_ws(grid.data_ptr(), guide.data_ptr(), inp.data_ptr(), out.data_ptr(),
                                       B, H, W, GH, GW, GD, 3, 3, 1, variant, ws.data_ptr(), n_ws, stream)
    assert rc == 0, (cfg[0], rc)

def burst(cfg, iters=40):
    for _ in range(3): run(cfg)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters): run(cfg)
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / iters, sm_clock()

equal = True
for cfg in cfgs:   # correctness first: every configuration produces the same bits
    out.zero_(); run(cfg); torch.cuda.synchronize()
    if ref is None: ref = out.clone()
    elif not torch.equal(ref, out): equal = False; print("MISMATCH:", cfg[0], float((ref - out).abs().max()))
res = {c[0]: [] for c in cfgs}
rounds = int(os.environ.get("AB_ROUNDS", "9"))
for r in range(rounds):
    for cfg in cfgs: res[cfg[0]].append(burst(cfg))
lines = []
for spec, v in res.items():
    t = [x[0] for x in v]
    med = statistics.median(t)
    lines.append(f"{spec:70s} median {med:.4f} ms  min {min(t):.4f}  max {max(t):.4f}  frac {B*H*W*28/med/1e6/3350.0:.4f}")
    lines.append("    bursts " + " ".join(f"{x[0]:.4f}@{x[1]}" for x in v))
lines.append(f"all outputs bitwise equal: {equal}")
print("\n".join(lines))
os.makedirs("tools_out", exist_ok=True)
open("tools_out/ab_lib.txt", "w").write("# tools/ab_lib.py " + " ".join(sys.argv[1:]) + "\n" + "\n".join(lines) + "\n")
