import sys, torch
sys.path.insert(0, ".")
from hdrnet_b200 import _lib, models
def t(fn, iters=50):
    for _ in range(5): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3
lib, st = _lib.load(), torch.cuda.current_stream().cuda_stream
for B in (1, 8, 64):
    for (H, cin, cout, k, s) in [(16, 64, 64, 3, 1), (32, 32, 64, 3, 2), (64, 16, 32, 3, 2), (16, 64, 96, 1, 1)]:
        x = torch.rand(B, H, H, cin, device="cuda"); w = torch.rand(k, k, cin, cout, device="cuda"); b = torch.rand(cout, device="cuda")
        out = torch.empty(B, H // s, H // s, cout, device="cuda")
        packed = models.pack_conv_weights(w)
        tc = lambda: lib.hdrnet_conv2d_nhwc_tc_f32(x.data_ptr(), packed.data_ptr(), b.data_ptr(), out.data_ptr(),
                                                   B, H, H, cin, cout, k, s, 1, st)
        _lib.check(tc(), "conv2d (packed)")
        res = [t(lambda: models._conv(x, (w, b), stride=s)), t(tc)]   # the library's own choice, the packed entry
        tiles = (B * (H // s) ** 2 + 127) // 128
        flops = 2 * B * (H // s) ** 2 * cout * k * k * cin
        print(f"B={B} {H}x{H}x{cin}->{cout} k{k}s{s} ({tiles} tiles): library's choice {res[0]:.1f} us, tensor cores pipelined+packed {res[1]:.1f} us ({flops/res[1]/1e6:.2f} TFLOP/s eff.)")
