"""Integer pixel I/O on the model path (SURVEY.md section 8 row f-3): the decoded uint8 / uint16
image goes through img_as_float -> nearest-neighbour network input -> guide + slice + apply ->
uint8(255 * clip(out, 0, 1)) on the device (hdrnet/bin/run.py:145-169, :95).

What is checked, and to what bar:
  * the code -> float conversion is BIT-EXACT with float32(float64(v) / D) for every code value;
  * the nearest-neighbour gather equals the host restatement of run.py exactly;
  * the integer-I/O kernels equal the float32 kernels fed the converted image, quantised on the
    host with the reference's cast: exactly when both run the same kernel family, within one
    code value (and < 0.1 % of samples) when the float path runs a different family;
  * the whole image path against the oracle model: within one code value.
"""
import numpy as np
import pytest
import torch

import oracle
from hdrnet_b200 import _lib, hdrnet_ops, models
from hdrnet_b200.bin import run
from oracle import model_np as M

pytestmark = pytest.mark.gpu

PX = {np.dtype(np.float32): _lib.PX_F32, np.dtype(np.uint8): _lib.PX_U8, np.dtype(np.uint16): _lib.PX_U16}


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def quantize(x):
    """tf.cast(255.0 * tf.clip_by_value(x, 0, 1), tf.uint8): float32 product, truncation."""
    return (np.float32(255.0) * np.clip(x.astype(np.float32), 0, 1)).astype(np.uint8)


def params_for(kind):
    p = dict(M.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8, luma_bins=8)
    if kind == "nn":
        p.update(model_name="HDRNetPointwiseNNGuide", batch_norm=True)
    if kind == "pyramid":
        p.update(model_name="HDRNetGaussianPyrNN")
    p["weights"] = models.init_weights(p, seed=3)
    return p


def rand_image(rng, B, H, W, dtype):
    hi = 256 if dtype == np.uint8 else 65536
    return rng.randint(0, hi, size=(B, H, W, 3)).astype(dtype)


@pytest.mark.parametrize("dtype,D", [(np.uint8, 255.0), (np.uint16, 65535.0)])
def test_code_to_float_is_bit_exact_for_every_code(dtype, D):
    """Identity-size 'resize' of an image holding every code value."""
    n = 256 if dtype == np.uint8 else 65536
    H, W = 64, (n * 2) // (64 * 3) + 1
    codes = (np.arange(H * W * 3) % n).astype(dtype).reshape(1, H, W, 3)
    out = torch.empty((1, H, W, 3), dtype=torch.float32, device="cuda")
    rc = _lib.load().hdrnet_lowres_nearest_f32(cuda(codes).data_ptr(), PX[np.dtype(dtype)], out.data_ptr(),
                                               1, H, W, H, W, 0)
    _lib.check(rc, "lowres")
    torch.cuda.synchronize()
    want = (codes.astype(np.float64) / D).astype(np.float32)      # skimage.img_as_float -> f32 feed
    assert np.array_equal(out.cpu().numpy(), want)
    assert set(np.unique(codes)) == set(range(n))


@pytest.mark.parametrize("H,W,S", [(37, 53, 16), (256, 256, 256), (1080, 1920, 256), (7, 5, 16)])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.float32])
def test_lowres_nearest_matches_run_py_restatement(H, W, S, dtype):
    rng = np.random.RandomState(H + W)
    im = rng.rand(2, H, W, 3).astype(np.float32) if dtype == np.float32 else rand_image(rng, 2, H, W, dtype)
    got = models.lowres_from_image(cuda(im), S).cpu().numpy()
    want = np.stack([run.nearest_resize(run.img_as_float(im[b]), S) for b in range(2)])
    assert got.dtype == np.float32 and np.array_equal(got, want)


def _float_reference(cls, params, im_f, coeffs):
    return cls._fullres(coeffs, cuda(im_f), params, torch.float32).cpu().numpy()


@pytest.mark.parametrize("kind", ["curves", "nn"])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
@pytest.mark.parametrize("B,H,W", [
    (2, 24, 256),      # row kernel, shared-memory slab (no workspace below 2 Mi pixels)
    (1, 548, 3840),    # row kernel, texture-assisted form (>= 2 Mi pixels, workspace lent)
    (1, 9, 1104),      # ragged last segment, W % 16 == 0
    (2, 11, 100),      # W % 16 != 0: per-pixel fused kernel
])
def test_integer_io_equals_float_kernels_quantised(kind, dtype, B, H, W):
    """Same kernel family on both sides -> the bytes are identical."""
    cls = models.HDRNetCurves if kind == "curves" else models.HDRNetPointwiseNNGuide
    p = params_for(kind)
    rng = np.random.RandomState(B * H + W)
    im = rand_image(rng, B, H, W, dtype)
    im_f = np.stack([run.img_as_float(im[b]) for b in range(B)])
    low = models.lowres_from_image(cuda(im), p["net_input_size"])
    coeffs = cls._coefficients(low, p)
    got = cls._fullres(coeffs, cuda(im), p, torch.uint8).cpu().numpy()
    ref_f = _float_reference(cls, p, im_f, coeffs)
    assert got.dtype == np.uint8 and got.shape == im.shape
    assert np.array_equal(got, quantize(ref_f))


@pytest.mark.parametrize("in_dtype,out_dtype", [(np.float32, torch.uint8), (np.uint8, torch.float32),
                                                (np.uint16, torch.float32)])
def test_mixed_format_combinations(in_dtype, out_dtype):
    """Combinations without a row-kernel form run the per-pixel fused kernel; the float path of
    this shape runs the row kernel (different summation order): one code value / 1e-5."""
    cls, p = models.HDRNetCurves, params_for("curves")
    rng = np.random.RandomState(5)
    B, H, W = 2, 16, 256
    im = rng.rand(B, H, W, 3).astype(np.float32) if in_dtype == np.float32 else rand_image(rng, B, H, W, in_dtype)
    im_f = np.stack([run.img_as_float(im[b]) for b in range(B)])
    low = models.lowres_from_image(cuda(im), p["net_input_size"])
    coeffs = cls._coefficients(low, p)
    got = cls._fullres(coeffs, cuda(im), p, out_dtype).cpu().numpy()
    ref_f = _float_reference(cls, p, im_f, coeffs)
    if out_dtype == torch.uint8:
        d = np.abs(got.astype(int) - quantize(ref_f).astype(int))
        assert d.max() <= 1 and (d > 0).mean() < 1e-3
    else:
        assert np.abs(got - ref_f).max() <= 1e-5 * np.abs(ref_f).max()


@pytest.mark.parametrize("kind", ["curves", "nn", "pyramid"])
def test_inference_image_matches_oracle_model(kind):
    """End to end (decode format in, uint8 out) against the numpy restatement of the model fed
    run.py's host-side preprocessing: at most one code value apart, rarely."""
    cls = getattr(models, params_for(kind)["model_name"])
    p = params_for(kind)
    rng = np.random.RandomState(17)
    im = rand_image(rng, 1, 96, 128, np.uint8)
    got = cls.inference_image(cuda(im), p).cpu().numpy()
    im_f = run.img_as_float(im[0])[None]
    low = run.nearest_resize(im_f[0], p["net_input_size"])[None]
    ref_fn = M.gaussian_pyr_inference if kind == "pyramid" else M.inference
    ref = ref_fn(low, im_f, p["weights"], p, oracle.best().bilateral_slice_apply)[0]
    d = np.abs(got.astype(int) - quantize(ref).astype(int))
    assert got.dtype == np.uint8 and d.max() <= 1 and (d > 0).mean() < 5e-3
    # the unquantised prediction from the same integer pixels
    got_f = cls.inference_image(cuda(im), p, out_dtype=torch.float32).cpu().numpy()
    assert np.abs(got_f - ref).max() <= 1e-4 * np.abs(ref).max()


def test_debug_guide_dump_with_integer_pixels():
    cls, p = models.HDRNetCurves, dict(params_for("curves"), debug=True)
    rng = np.random.RandomState(2)
    im = rand_image(rng, 1, 32, 256, np.uint8)
    cls.inference_image(cuda(im), p)
    guide = cls.last_debug["guide"].cpu().numpy()
    want = cls._guide(cuda(run.img_as_float(im[0])[None]), p).cpu().numpy()
    assert np.array_equal(guide, want)


def test_unsupported_formats_are_refused():
    lib = _lib.load()
    z = torch.zeros(64, device="cuda")
    host = np.zeros(64, np.float32)                              # guide parameters are HOST arrays
    args = (host.ctypes.data,) * 5
    rc = lib.hdrnet_slice_apply_curves_px_ws(z.data_ptr(), z.data_ptr(), 7, z.data_ptr(), _lib.PX_U8, 0,
                                             1, 1, 4, 1, 1, 1, *args, 0.0, 0, 0, 0)
    assert rc == -5                                               # HDRNET_E_UNSUPPORTED
    rc = lib.hdrnet_slice_apply_curves_px_ws(z.data_ptr(), z.data_ptr(), _lib.PX_U8, z.data_ptr(), _lib.PX_U16, 0,
                                             1, 1, 4, 1, 1, 1, *args, 0.0, 0, 0, 0)
    assert rc == -5
    assert lib.hdrnet_lowres_nearest_f32(z.data_ptr(), 9, z.data_ptr(), 1, 1, 1, 1, 1, 0) == -5
    with pytest.raises(TypeError):
        models.lowres_from_image(torch.zeros(1, 4, 4, 3, dtype=torch.int32, device="cuda"), 2)


# ---- fused-guide texture-assisted forms against the un-fused composition -------------------------
def test_fused_guide_issuer_warp_form_is_bitwise_equal():
    """At >= 2 Mi pixels the model's full-resolution stage runs the texture-assisted fused-guide forms:
    the issuer-warp form for the curves guide, the block-synchronous one for the pointwise-NN guide.
    For both guides and all three pixel formats they must give the bits of the un-fused composition:
    the standalone guide kernel, then the op API's block-synchronous texture form
    (HDRNET_VARIANT_TEX) on the float image; integer pixels are compared with that float result
    quantised on the host."""
    B, H, W = 2, 300, 3840
    for kind in ("curves", "nn"):
        cls = models.HDRNetCurves if kind == "curves" else models.HDRNetPointwiseNNGuide
        p = params_for(kind)
        for dtype in (np.float32, np.uint8, np.uint16):
            rng = np.random.RandomState(5)
            if dtype == np.float32:
                im = rng.rand(B, H, W, 3).astype(np.float32)
                im_f = im
                low = cuda(rng.rand(B, 64, 64, 3).astype(np.float32))
            else:
                im = rand_image(rng, B, H, W, dtype)
                im_f = np.stack([run.img_as_float(im[b]) for b in range(B)])
                low = models.lowres_from_image(cuda(im), p["net_input_size"])
            coeffs = cls._coefficients(low, p)
            out_dtype = torch.float32 if dtype == np.float32 else torch.uint8
            got = cls._fullres(coeffs, cuda(im), p, out_dtype).cpu().numpy()
            f = cuda(im_f)
            guide = cls._guide(f, p)
            gh, gw, gd = coeffs.shape[1:4]
            want = hdrnet_ops.bilateral_slice_apply(coeffs.reshape(B, gh, gw, gd, 12), guide, f, True,
                                                    variant=_lib.VARIANT_TEX).cpu().numpy()
            if dtype != np.float32:
                want = quantize(want)
            assert np.array_equal(got, want), f"{kind} guide, {np.dtype(dtype).name} pixels"


@pytest.mark.parametrize("kind,dtype,pinned", [("curves", torch.uint8, True), ("nn", torch.uint16, True),
                                              ("curves", torch.uint8, False), ("pyramid", torch.uint8, True)])
def test_host_frame_pipeline_equals_inference_image(kind, dtype, pinned):
    """inference_image_host (upload | model | download of consecutive frames on three streams,
    host_pipeline.py) against inference_image on the same frames, frame by frame: bitwise.  Five
    frames through two device buffers exercise the buffer-reuse events; a second call with
    different content reuses the pipeline object."""
    p = params_for(kind)
    wts = M.make_weights(p, seed=5)
    cls = getattr(models, p["model_name"])
    prm = dict(p, weights=wts)
    g = torch.Generator().manual_seed(11)
    hi = 256 if dtype == torch.uint8 else 65536
    for rep in range(2):
        frames = torch.randint(0, hi, (5, 48, 192, 3), generator=g, dtype=torch.int32).to(dtype)
        if pinned:
            frames = frames.pin_memory()
        got = cls.inference_image_host(frames, prm)
        assert got.dtype == torch.uint8 and not got.is_cuda and tuple(got.shape) == tuple(frames.shape)
        for i in range(frames.shape[0]):
            want = cls.inference_image(frames[i:i + 1].cuda(), prm).cpu()
            assert torch.equal(got[i:i + 1], want), f"{kind}: frame {i} of call {rep} differs"
    with pytest.raises(TypeError):
        cls.inference_image_host(frames.cuda(), prm)
    assert cls.inference_image_host(frames[:0], prm).shape[0] == 0
