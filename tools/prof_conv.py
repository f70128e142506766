import sys, torch
sys.path.insert(0, ".")
from hdrnet_b200 import _lib, models
B = 8
x = torch.rand(B, 16, 16, 64, device="cuda"); w = torch.rand(3, 3, 64, 64, device="cuda"); b = torch.rand(64, device="cuda")
out = torch.empty(B, 16, 16, 64, device="cuda")
packed = models.pack_conv_weights(w)
for _ in range(4):   # the packed tensor-core entry, whatever the layer's tile count
    _lib.check(_lib.load().hdrnet_conv2d_nhwc_tc_f32(x.data_ptr(), packed.data_ptr(), b.data_ptr(), out.data_ptr(),
                                                     B, 16, 16, 64, 64, 3, 1, 1, torch.cuda.current_stream().cuda_stream),
               "conv2d (packed)")
torch.cuda.synchronize()
