"""Per-layer time of the coefficient network's convs (CUDA-graph replay of 20 launches), by batch,
in the form the library selects for each layer:
    python tools/time_conv_layers.py
"""
import os, sys, statistics, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hdrnet_b200 import _lib

LAYERS = [  # name, H, Cin, Cout, stride
    ("splat1", 256, 3, 8, 2),
    ("splat2", 128, 8, 16, 2), ("splat3", 64, 16, 32, 2), ("splat4", 32, 32, 64, 2),
    ("gconv1", 16, 64, 64, 2), ("gconv2", 8, 64, 64, 2), ("lconv", 16, 64, 64, 1),
]
lib = _lib.load()
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
        line.append(f"{name} {statistics.median(ts):.1f}")
    print(f"batch {B}: " + "  ".join(line), flush=True)
