"""Per-layer time of the coefficient network's convs (CUDA-graph replay of 20 launches), by batch.

Run once per setting of HDRNET_CONV_PATCH (read once per process):
    HDRNET_CONV_PATCH=0 python tools/time_conv_layers.py   # conv2d_nhwc_kernel<1,4> / <2,8>
    HDRNET_CONV_PATCH=1 python tools/time_conv_layers.py   # patch form, 4 channels per CTA
    HDRNET_CONV_PATCH=2 python tools/time_conv_layers.py   # patch form, 8 channels per CTA
Also prints max |diff| against the tensor-core-free HDRNET_CONV_PATCH=0 result when
tools_out/conv_ref.pt exists (written by the =0 run).
"""
import os, sys, statistics, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hdrnet_b200 import _lib

LAYERS = [  # name, H, Cin, Cout, stride
    ("splat1", 256, 3, 8, 2),
    ("splat2", 128, 8, 16, 2), ("splat3", 64, 16, 32, 2), ("splat4", 32, 32, 64, 2),
    ("gconv1", 16, 64, 64, 2), ("gconv2", 8, 64, 64, 2), ("lconv", 16, 64, 64, 1),
]
mode = os.environ.get("HDRNET_CONV_PATCH", "auto")
lib = _lib.load()
ref_path = "tools_out/conv_ref.pt"
ref = torch.load(ref_path) if (mode != "0" and os.path.exists(ref_path)) else {}
save = {}
for B in (1, 2, 8):
    line = []
    for name, H, ci, co, s in LAYERS:
        g = torch.Generator(device="cuda").manual_seed(1)
        x = torch.randn(B, H, H, ci, device="cuda", generator=g)
        w = torch.randn(3, 3, ci, co, device="cuda", generator=g) * 0.1
        b = torch.randn(co, device="cuda", generator=g)
        oh = -(-H // s)
        out = torch.empty(B, oh, oh, co, device="cuda")
        st = torch.cuda.Stream()
        def call():
            rc = lib.hdrnet_conv2d_nhwc_f32(x.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(), B, H, H,
                                            ci, co, 3, s, 1, torch.cuda.current_stream().cuda_stream)
            assert rc == 0, rc
        with torch.cuda.stream(st):
            call(); torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                for _ in range(20): call()
            ts = []
            for _ in range(5):
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); gr.replay(); e.record(); torch.cuda.synchronize()
                ts.append(a.elapsed_time(e) / 20 * 1e3)
        key = f"{name}_{B}"
        save[key] = out.cpu()
        d = f" d={float((out.cpu() - ref[key]).abs().max()):.1e}" if key in ref else ""
        line.append(f"{name} {statistics.median(ts):.1f}{d}")
    print(f"PATCH={mode} batch {B}: " + "  ".join(line), flush=True)
if mode == "0":
    os.makedirs("tools_out", exist_ok=True)
    torch.save(save, ref_path)
