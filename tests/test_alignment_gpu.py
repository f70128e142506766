"""Every kernel's unaligned-buffer path against float64 references.

Almost every dispatcher takes its fast form (bulk copies / TMA, texture-assisted rows, float4 and
16-byte cp.async staging, tensor-core convs, the fc cluster forms) only when its base pointers are
16-byte aligned, and a slower form otherwise.  Buffers from torch's allocator always are, but a
caller's need not be: frames carved out of one packed buffer behind a header (torch.frombuffer,
memory-mapped files), ``out=`` tensors taken from a pool, fine-tuning weights held as views into one
flat parameter buffer.  Here every argument is given at 1-3 float32 elements (or 1-15 uint8 /
1-7 uint16 elements) past a 16-byte boundary, one at a time and all at once, at shapes where the
aligned call takes the fast form, so each case crosses the dispatch boundary.

Bars, as in the rest of the suite: outputs within 1e-5 of range of a float64 reference (model
outputs: of the pinned slice oracle fed the CUDA stage's own coefficients and guide, as in
tests/test_models.py); VJPs at the bars of tests/test_grad_scale_gpu.py and
tests/test_cnn_grad_gpu.py; integer gathers bit-exact.  Run with -s to see the worst error of each
group.
"""
import functools

import numpy as np
import pytest
import torch

import oracle
from hdrnet_b200 import _lib, hdrnet_ops, layers, models
from hdrnet_b200.bin import run
from oracle import cnn_grad_f64 as G
from oracle import model_np as M
from oracle import slice_f64
from test_grad_scale_gpu import Case, check as check_vjps, errors as vjp_errors
from util import assert_parity, rand_case, rel_err

pytestmark = pytest.mark.gpu

RTOL = 1e-5
CNN_BAR = 1e-5                        # tests/test_cnn_grad_gpu.py BAR
F32_SHIFTS = (1, 2, 3)
OP_SHAPE = (2, 96, 256, 16, 16, 8)    # B, H, W, gh, gw, gd: W >= 128, W % 4 == 0 -> row kernels
TEX_SHAPE = (1, 1024, 2048, 16, 16, 8)   # B * H * W = 2^21 -> texture-assisted forms

_worst = {}


def note(group, err):
    _worst[group] = max(_worst.get(group, 0.0), float(err))
    return err


@pytest.fixture(scope="module", autouse=True)
def _print_worst_errors():
    yield
    for group, err in sorted(_worst.items()):
        print(f"MEASURE alignment {group}: worst {err:.2e}", flush=True)


# ---- shifted buffers ---------------------------------------------------------------------------
def shifted(t, k, pin=False):
    """A contiguous tensor with the values of ``t`` whose data_ptr() is ``k`` elements past a 16-byte
    boundary: a view at offset ``k`` into a buffer of numel + 16 / itemsize elements.  ``pin``: the
    buffer is page-locked host memory (``t`` on the CPU)."""
    t = torch.as_tensor(t)
    item = t.element_size()
    assert 0 <= k < 16 // item
    buf = torch.empty(t.numel() + 16 // item, dtype=t.dtype, device=t.device, pin_memory=pin)
    assert buf.data_ptr() % 16 == 0
    with torch.no_grad():
        buf[k:k + t.numel()].copy_(t.detach().reshape(-1))
    view = buf[k:k + t.numel()].view(t.shape)
    assert view.is_contiguous() and view.data_ptr() % 16 == k * item
    return view


def shift_args(args, which, k, pin=False):
    """``args`` (name -> tensor) with the argument ``which`` shifted by ``k`` elements, or every
    argument when ``which`` is "all"."""
    return {n: shifted(t, k, pin) if which in (n, "all") else t for n, t in args.items()}


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def np_(t):
    return t.detach().cpu().numpy()


def test_shifted_helper_offsets_and_values():
    for dtype, ks in ((np.float32, F32_SHIFTS), (np.uint8, range(1, 16)), (np.uint16, range(1, 8))):
        a = (np.arange(1000) % 251).astype(dtype).reshape(10, 100)
        for k in ks:
            s = shifted(dev(a), k)
            assert np.array_equal(np_(s), a) and s.data_ptr() % 16 == k * a.itemsize


# ---- op API: bilateral_slice_apply / bilateral_slice --------------------------------------------
@functools.lru_cache(maxsize=None)
def apply_case(shape, seed):
    B, H, W, gh, gw, gd = shape
    grid, guide, inp = rand_case(seed, B, H, W, gh, gw, gd, signed=True)
    return grid, guide, inp, slice_f64.bilateral_slice_apply(grid, guide, inp, True)


def run_apply(shape, which, k, seed=60):
    grid, guide, inp, want = apply_case(shape, seed)
    B, H, W = shape[:3]
    a = shift_args(dict(grid=dev(grid), guide=dev(guide), input=dev(inp),
                        out=torch.empty((B, H, W, 3), device="cuda")), which, k)
    got = hdrnet_ops.bilateral_slice_apply(a["grid"], a["guide"], a["input"], True, out=a["out"])
    assert got.data_ptr() == a["out"].data_ptr()
    got = np_(got)
    note("slice_apply", rel_err(got, want))
    assert_parity(got, want, rtol=RTOL, what=f"slice_apply {which} +{k}")


@pytest.mark.parametrize("k", F32_SHIFTS)
@pytest.mark.parametrize("which", ["grid", "guide", "input", "out", "all"])
def test_slice_apply_shifted(which, k):
    """Row kernel when aligned; the any-shape row kernel otherwise."""
    run_apply(OP_SHAPE, which, k)


@pytest.mark.parametrize("which,k", [("input", 2), ("out", 3), ("all", 1)])
def test_slice_apply_shifted_at_texture_sizes(which, k):
    """Texture-assisted issuer-warp form when aligned (a workspace is lent); the any-shape row
    kernel otherwise."""
    run_apply(TEX_SHAPE, which, k, seed=61)


@pytest.mark.parametrize("which,k", [("guide", 1), ("input", 2), ("out", 3), ("all", 1)])
def test_slice_apply_rows_band_shifted(which, k):
    """hdrnet_slice_apply_rows_f32_ws: rows 24..63 of 96-row images against the same rows of the
    whole-image float64 reference."""
    grid, guide, inp, want = apply_case(OP_SHAPE, 62)
    B, H, W = OP_SHAPE[:3]
    y0, rows = 24, 40
    a = shift_args(dict(guide=dev(guide[:, y0:y0 + rows]), input=dev(inp[:, y0:y0 + rows]),
                        out=torch.empty((B, rows, W, 3), device="cuda")), which, k)
    with torch.no_grad():
        got = hdrnet_ops.bilateral_slice_apply_rows(dev(grid), a["guide"], a["input"], True, y0, H, out=a["out"])
    got = np_(got)
    note("slice_apply rows", rel_err(got, want[:, y0:y0 + rows]))
    assert_parity(got, want[:, y0:y0 + rows], rtol=RTOL, what=f"rows {which} +{k}")


@pytest.mark.parametrize("k", F32_SHIFTS)
@pytest.mark.parametrize("which", ["grid", "guide", "out", "all"])
def test_slice_shifted(which, k):
    """Un-fused slice with 12 channels: TMA row kernel when aligned; the any-shape row kernel
    (float4 stores only to an aligned out) otherwise.  ``out`` goes through the C-ABI directly:
    hdrnet_ops.bilateral_slice always allocates its result."""
    B, H, W, gh, gw, gd = OP_SHAPE
    rng = np.random.RandomState(63 + k)
    grid = rng.randn(B, gh, gw, gd, 12).astype(np.float32)
    guide = rng.rand(B, H, W).astype(np.float32)
    want = slice_f64.bilateral_slice(grid, guide)
    a = shift_args(dict(grid=dev(grid), guide=dev(guide), out=torch.empty((B, H, W, 12), device="cuda")),
                   which, k)
    if which in ("grid", "guide"):
        got = hdrnet_ops.bilateral_slice(a["grid"], a["guide"])
    else:
        rc = _lib.load().hdrnet_slice_f32(a["grid"].data_ptr(), a["guide"].data_ptr(), a["out"].data_ptr(),
                                          B, H, W, gh, gw, gd, 12, torch.cuda.current_stream().cuda_stream)
        _lib.check(rc, "BilateralSlice")
        got = a["out"]
    got = np_(got)
    note("slice", rel_err(got, want))
    assert_parity(got, want, rtol=RTOL, what=f"slice {which} +{k}")


@pytest.mark.parametrize("variant", [_lib.VARIANT_TMA, _lib.VARIANT_TEX, _lib.VARIANT_TEX_ASYNC])
def test_forced_fast_variants_refuse_shifted_buffers(variant):
    """A forced bulk-copy / texture form runs on aligned buffers and refuses shifted ones with the
    existing error, before any launch: the sentinel in ``out`` survives."""
    grid, guide, inp, _ = apply_case(TEX_SHAPE, 61)
    B, H, W = TEX_SHAPE[:3]
    args = dict(grid=dev(grid), guide=dev(guide), input=dev(inp), out=torch.empty((B, H, W, 3), device="cuda"))
    with torch.no_grad():
        forced = hdrnet_ops.bilateral_slice_apply(args["grid"], args["guide"], args["input"], True, variant=variant)
        auto = hdrnet_ops.bilateral_slice_apply(args["grid"], args["guide"], args["input"], True)
    assert_parity(np_(forced), np_(auto), rtol=RTOL, what=f"aligned variant {variant}")
    for which in ("grid", "guide", "input", "out"):
        a = shift_args(args, which, 1)
        a["out"].fill_(float("nan"))
        with pytest.raises(ValueError, match="cannot run these shapes"):
            hdrnet_ops.bilateral_slice_apply(a["grid"], a["guide"], a["input"], True, out=a["out"],
                                             variant=variant)
        torch.cuda.synchronize()
        assert torch.isnan(a["out"]).all(), f"variant {variant} with {which} shifted wrote its output"


# ---- slice VJPs through autograd ---------------------------------------------------------------
@pytest.mark.parametrize("k", F32_SHIFTS)
@pytest.mark.parametrize("op", ["apply", "slice"])
def test_slice_vjps_with_shifted_buffers(op, k):
    c = Case(2, 96, 256, 16, 16, 8, op=op, gc=12, seed=70 + k)
    grid, guide, inp, ct = c.arrays()
    leaves = [shifted(dev(a), k).requires_grad_() for a in ((grid, guide, inp) if op == "apply" else (grid, guide))]
    if op == "apply":
        out = hdrnet_ops.bilateral_slice_apply(*leaves, True)
    else:
        out = hdrnet_ops.bilateral_slice(*leaves)
    out.backward(shifted(dev(ct), k))
    got = [np_(t.grad) for t in leaves] + ([] if op == "apply" else [None])
    e = vjp_errors(got, c.f64(grid, guide, inp, ct))
    for name, v in e.items():
        note(f"{op} vjp {name}", v)
    check_vjps(e, f"{op} VJPs +{k}")


# ---- guides ------------------------------------------------------------------------------------
GUIDE_PARAMS = {"curves": dict(M.DEFAULT_PARAMS),
                "nn": dict(M.DEFAULT_PARAMS, model_name="HDRNetPointwiseNNGuide", batch_norm=True)}


def guide_f64(kind, x, wts):
    """hdrnet/models.py:145-190 (curves) and :199-210 (pointwise NN, conv1 batch-normed), float64."""
    g = "inference/guide"
    x = np.asarray(x, np.float64)
    w = {k: np.asarray(v, np.float64) for k, v in wts.items() if k.startswith(g)}
    if kind == "curves":
        t = x @ w[g + "/ccm"] + w[g + "/ccm_bias"]
        u = (w[g + "/slopes"].reshape(3, -1) * np.maximum(t[..., None] - w[g + "/shifts"].reshape(3, -1), 0)).sum(-1)
        return np.clip(u @ w[g + "/channel_mixing/weights"].reshape(3) + w[g + "/channel_mixing/biases"].reshape(-1)[0],
                       0.0, 1.0)
    c1 = g + "/conv1"
    h = x @ w[c1 + "/weights"].reshape(3, -1)
    h = (h - w[c1 + "/BatchNorm/moving_mean"]) / np.sqrt(w[c1 + "/BatchNorm/moving_variance"] + M.BN_EPS) \
        + w[c1 + "/BatchNorm/beta"]
    y = np.maximum(h, 0) @ w[g + "/conv2/weights"].reshape(-1) + w[g + "/conv2/biases"].reshape(-1)[0]
    return 1.0 / (1.0 + np.exp(-y))


@pytest.mark.parametrize("npix_mod4", [0, 1, 2, 3])
@pytest.mark.parametrize("kind", ["curves", "nn"])
def test_guides_on_shifted_input(kind, npix_mod4):
    """guide.cu: float4 quads + scalar tail when aligned, all scalar otherwise; the same per-pixel
    function, so every shift gives the aligned call's bits."""
    p = GUIDE_PARAMS[kind]
    wts = M.make_weights(p, seed=80)
    params = dict(p, weights=wts)
    cls = models.HDRNetCurves if kind == "curves" else models.HDRNetPointwiseNNGuide
    H, W = 17, 256 + npix_mod4                                      # npix % 4 == npix_mod4
    full = np.random.RandomState(81 + npix_mod4).rand(1, H, W, 3).astype(np.float32)
    want = guide_f64(kind, full, wts)
    t = dev(full)
    aligned = cls._guide(t, params)
    for k in F32_SHIFTS:
        got = cls._guide(shifted(t, k), params)
        note(f"guide {kind}", np.abs(np_(got) - want).max())
        assert np.abs(np_(got) - want).max() <= RTOL, f"{kind} guide +{k}"
        assert torch.equal(got, aligned), f"{kind} guide +{k} differs from the aligned call"


# ---- model path --------------------------------------------------------------------------------
def stage_reference(cls, coeffs, guide, full):
    """The pinned slice oracle fed the CUDA stage's own coefficients and guide."""
    c = np_(coeffs)
    return oracle.best().bilateral_slice_apply(np.ascontiguousarray(c.reshape(c.shape[:4] + (12,))),
                                               np_(guide), np.ascontiguousarray(full, np.float32), True)


@pytest.mark.parametrize("H,W", [(48, 128), (64, 1920), (2160, 3840)])
@pytest.mark.parametrize("kind", ["curves", "nn"])
def test_model_inference_with_shifted_fullres(kind, H, W):
    """The float32 guide-fused call: fused row kernel (texture-assisted at 4K) when aligned; the
    guide kernel into a guide buffer + the any-shape row kernel otherwise."""
    p = GUIDE_PARAMS[kind]
    cls = getattr(models, p["model_name"])
    params = dict(p, weights=M.make_weights(p, seed=82))
    B = 1 if H * W >= (1 << 21) else 2
    rng = np.random.RandomState(83)
    S = p["net_input_size"]
    low = dev(rng.rand(B, S, S, 3).astype(np.float32))
    full = rng.rand(B, H, W, 3).astype(np.float32)
    tfull = dev(full)
    with torch.no_grad():
        aligned = cls.inference(low, tfull, params)
        stage = stage_reference(cls, cls._coefficients(low, params), cls._guide(tfull, params), full)
        for k in (F32_SHIFTS if B > 1 else (1,)):
            got = cls.inference(low, shifted(tfull, k), params)
            note(f"model {kind} stage", rel_err(np_(got), stage))
            assert_parity(np_(got), stage, rtol=RTOL, what=f"{kind} {H}x{W} +{k} full-resolution stage")
            note(f"model {kind} vs aligned", rel_err(np_(got), np_(aligned)))
            assert_parity(np_(got), np_(aligned), rtol=1e-6, elem_rtol=None, what=f"{kind} +{k} vs aligned")


def quantize(x):
    """tf.cast(255.0 * tf.clip_by_value(x, 0, 1), tf.uint8) (hdrnet/bin/run.py:95)."""
    return (np.float32(255.0) * np.clip(x.astype(np.float32), 0, 1)).astype(np.uint8)


@pytest.mark.parametrize("dtype", [torch.uint8, torch.uint16])
@pytest.mark.parametrize("kind", ["curves", "nn"])
def test_inference_image_with_shifted_integer_image(kind, dtype):
    """Integer pixels at every byte offset a 16-byte vector could straddle: the u8 / u16 row kernel
    when aligned (W % 16 == 0), the per-pixel fused kernel otherwise, for float32 and uint8 out."""
    p = dict(GUIDE_PARAMS[kind], net_input_size=64, spatial_bin=8)
    cls = getattr(models, p["model_name"])
    params = dict(p, weights=M.make_weights(p, seed=84))
    B, H, W = 2, 24, 256
    npt = np.uint8 if dtype == torch.uint8 else np.uint16
    im = dev(np.random.RandomState(85).randint(0, np.iinfo(npt).max + 1, size=(B, H, W, 3)).astype(npt))
    with torch.no_grad():
        coeffs = cls._coefficients(models.lowres_from_image(im, p["net_input_size"]), params)
        im_f = models.image_to_float(im)
        stage = stage_reference(cls, coeffs, cls._guide(im_f, params), np_(im_f))
        aligned_u8 = np_(cls.inference_image(im, params)).astype(int)
        for k in range(1, 16 // im.element_size()):
            s = shifted(im, k)
            f = np_(cls.inference_image(s, params, out_dtype=torch.float32))
            u = np_(cls.inference_image(s, params, out_dtype=torch.uint8))
            note(f"image {kind} {dtype}", rel_err(f, stage))
            assert_parity(f, stage, rtol=RTOL, what=f"{kind} {dtype} +{k} float32 out")
            assert np.array_equal(u, quantize(f)), f"{kind} {dtype} +{k}: uint8 out != quantised float32 out"
            assert np.abs(u.astype(int) - aligned_u8).max() <= 1, f"{kind} {dtype} +{k} vs aligned"


def test_pyramid_inference_with_shifted_fullres():
    """HDRNetGaussianPyrNN: level 0 is the caller's image; its guide-fused slice-apply needs the
    guide buffer when that image is shifted."""
    p = dict(M.DEFAULT_PARAMS, model_name="HDRNetGaussianPyrNN", net_input_size=128, spatial_bin=16)
    wts = M.make_weights(p, seed=86)
    params = dict(p, weights=wts)
    cls = models.HDRNetGaussianPyrNN
    rng = np.random.RandomState(87)
    low = dev(rng.rand(2, 128, 128, 3).astype(np.float32))
    full = rng.rand(2, 128, 256, 3).astype(np.float32)
    with torch.no_grad():
        cls.inference(low, dev(full), dict(params, debug=True))
        dbg = cls.last_debug
        aligned = np_(cls.inference(low, dev(full), params))
        c = np_(dbg["bilateral_coefficients"])
        lvls = [full]
        for _ in range(2):
            lvls.append(M.resize_bilinear_ac(lvls[-1], lvls[-1].shape[1] // 2, lvls[-1].shape[2] // 2))
        stage = None
        for il in range(3):                                     # as tests/test_models.py
            src = 2 - il
            ci = np.ascontiguousarray(c[:, :, :, :, il * 3:(il + 1) * 3, :]).reshape(c.shape[:4] + (12,))
            o = oracle.best().bilateral_slice_apply(ci, np_(dbg["guide"][src]), lvls[src], True)
            stage = o if il == 0 else M.resize_bilinear_ac(stage, o.shape[1], o.shape[2]) + o
        for k in F32_SHIFTS:
            got = np_(cls.inference(low, shifted(dev(full), k), params))
            note("pyramid stage", rel_err(got, stage))
            assert_parity(got, stage, rtol=RTOL, elem_rtol=None, what=f"pyramid +{k}")
            assert_parity(got, aligned, rtol=1e-6, elem_rtol=None, what=f"pyramid +{k} vs aligned")


# ---- coefficient network -----------------------------------------------------------------------
TRAIN = dict(models.DEFAULT_PARAMS)


def flat_weights(wts, params, grad=False):
    """The coefficient-network variables as views into ONE flat float32 CUDA buffer, each 1-3
    elements past a 16-byte boundary; the guide variables stay host arrays.  Returns the buffer, the
    weights dict and {name: (offset, shape)}."""
    names = G.variable_names(params)
    where, pos = {}, 0
    for i, n in enumerate(names):
        pos = (pos + 3) // 4 * 4 + 1 + i % 3
        where[n] = (pos, np.asarray(wts[n]).shape)
        pos += np.asarray(wts[n]).size
    flat = torch.zeros(pos + 4, device="cuda")
    for n, (o, shape) in where.items():
        flat[o:o + int(np.prod(shape))] = torch.from_numpy(np.asarray(wts[n], np.float32).reshape(-1))
    flat.requires_grad_(grad)
    out = dict(wts)
    for n, (o, shape) in where.items():
        out[n] = flat[o:o + int(np.prod(shape))].view(shape)
        assert out[n].data_ptr() % 16 != 0
    return flat, out, where


@functools.lru_cache(maxsize=None)
def network_case(B):
    wts = M.make_weights(TRAIN, seed=90)
    low = np.random.RandomState(91 + B).rand(B, 256, 256, 3).astype(np.float32)
    return wts, low, G.Network(wts, TRAIN).forward(low)


@pytest.mark.parametrize("per_layer", [False, True], ids=["chain", "per-layer"])
@pytest.mark.parametrize("B", [1, 4, 8, 16])
def test_coefficients_with_flat_buffer_weights(B, per_layer, monkeypatch):
    """B = 1 / 4: the launch chain with the fc cluster chain, 8: the split-K fc cluster, 16: the
    tensor-core convs -- when the weights are aligned.  Views at odd offsets take the CUDA-core
    convs with scalar weight staging and the plain fc kernel."""
    wts, low, want = network_case(B)
    _, views, _ = flat_weights(wts, TRAIN)
    if per_layer:
        monkeypatch.setattr(models, "CHAIN_CNN_MAX_BATCH", 0)
    with torch.no_grad():
        got = np_(models.HDRNetCurves._coefficients(shifted(dev(low), 1 + B % 3), dict(TRAIN, weights=views)))
        aligned = np_(models.HDRNetCurves._coefficients(dev(low), dict(TRAIN, weights=wts)))
    group = "coefficients " + ("per-layer" if per_layer else "chain")
    note(group, rel_err(got, want))
    assert rel_err(got, want) <= CNN_BAR, f"B={B} {group}: {rel_err(got, want):.3e}"
    assert_parity(got, aligned, rtol=5e-6, elem_rtol=None, what=f"B={B} {group} vs aligned")


def test_coefficient_backward_with_flat_buffer_weights():
    """Gradients into a flat parameter buffer whose views sit at odd offsets, from a shifted upstream
    gradient, against the float64 network's backward."""
    B = 4
    wts, low, _ = network_case(B)
    flat, views, where = flat_weights(wts, TRAIN, grad=True)
    tl = shifted(dev(low), 3).requires_grad_()
    grid = models.HDRNetCurves._coefficients(tl, dict(TRAIN, weights=views))
    dgrid = np.random.RandomState(92).randn(*grid.shape).astype(np.float32)
    grid.backward(shifted(dev(dgrid), 2))
    net = G.Network(wts, TRAIN)
    net.forward(low)
    want = net.backward(dgrid)
    for name, ref in want.items():
        if name == "lowres_input":
            got = np_(tl.grad)
        else:
            o, shape = where[name]
            got = np_(flat.grad[o:o + int(np.prod(shape))]).reshape(shape)
        e = note("coefficient backward", rel_err(got, ref))
        assert e <= CNN_BAR, f"{name}: {e:.3e}"


# ---- small kernels -----------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,cin,cout,stride", [
    (1, 16, 64, 64, 1),      # shared-memory patch form
    (2, 64, 3, 8, 2),        # patch form, 3 input channels (4-byte copies)
    (4, 64, 16, 36, 1),      # CUDA-core kernel, float4 inputs + cp.async weight staging
    (4, 64, 16, 32, 1),      # tensor-core (wgmma) form: 128 tiles of 128 pixels
])
def test_layers_conv_shifted(B, H, cin, cout, stride):
    rng = np.random.RandomState(B * 100 + cout)
    x = rng.randn(B, H, H, cin).astype(np.float32)
    w = (rng.randn(3, 3, cin, cout) / np.sqrt(9 * cin)).astype(np.float32)
    b = rng.randn(cout).astype(np.float32)
    want = np.maximum(M.conv2d_same(x, w, stride) + b, 0)
    for which in ("input", "weights", "bias", "all"):
        for k in F32_SHIFTS:
            a = shift_args(dict(input=dev(x), weights=dev(w), bias=dev(b)), which, k)
            with torch.no_grad():
                got = np_(layers.conv(a["input"], cout, 3, stride=stride, scope="t/c",
                                      weights={"t/c/weights": a["weights"], "t/c/biases": a["bias"]}))
            note("layers.conv", rel_err(got, want))
            assert_parity(got, want, rtol=RTOL, elem_rtol=None, what=f"conv {which} +{k}")


def test_tensor_core_weight_packing_refuses_a_shifted_buffer():
    """hdrnet_conv2d_tc_pack_f32 stores float4s into the caller's buffer: a shifted one is refused
    before any launch (the sentinel survives), a shifted source is read as is."""
    lib = _lib.load()
    w = (np.random.RandomState(96).randn(3, 3, 16, 32) / 12).astype(np.float32)
    nfloats = lib.hdrnet_conv2d_tc_packed_bytes(3, 16, 32) // 4
    stream = torch.cuda.current_stream().cuda_stream
    ref = torch.empty(nfloats, device="cuda")
    _lib.check(lib.hdrnet_conv2d_tc_pack_f32(dev(w).data_ptr(), ref.data_ptr(), 3, 16, 32, stream), "pack")
    for k in F32_SHIFTS:
        packed = shifted(torch.full((nfloats,), float("nan"), device="cuda"), k)
        rc = lib.hdrnet_conv2d_tc_pack_f32(dev(w).data_ptr(), packed.data_ptr(), 3, 16, 32, stream)
        torch.cuda.synchronize()
        assert rc == _lib.E_UNSUPPORTED and torch.isnan(packed).all()
        got = torch.empty(nfloats, device="cuda")
        src = shifted(dev(w), k)
        _lib.check(lib.hdrnet_conv2d_tc_pack_f32(src.data_ptr(), got.data_ptr(), 3, 16, 32, stream), "pack")
        assert torch.equal(got, ref)


@pytest.mark.parametrize("B,I,O", [(8, 1024, 256), (3, 256, 128), (11, 70, 36)])
def test_layers_fc_shifted(B, I, O):
    """(8, 1024, 256) and (3, 256, 128): the split-K cluster form when aligned."""
    rng = np.random.RandomState(I + O)
    x = rng.randn(B, I).astype(np.float32)
    w = (rng.randn(I, O) / np.sqrt(I)).astype(np.float32)
    b = rng.randn(O).astype(np.float32)
    want = np.maximum(x.astype(np.float64) @ w + b, 0)
    for which in ("input", "weights", "bias", "all"):
        for k in F32_SHIFTS:
            a = shift_args(dict(input=dev(x), weights=dev(w), bias=dev(b)), which, k)
            with torch.no_grad():
                got = np_(layers.fc(a["input"], O, scope="t/f",
                                    weights={"t/f/weights": a["weights"], "t/f/biases": a["bias"]}))
            note("layers.fc", rel_err(got, want))
            assert_parity(got, want, rtol=RTOL, elem_rtol=None, what=f"fc {which} +{k}")


@pytest.mark.parametrize("B,H,W,oh,ow", [(2, 64, 96, 32, 48), (1, 33, 50, 16, 25)])
def test_resize_shifted(B, H, W, oh, ow):
    rng = np.random.RandomState(H)
    x = rng.rand(B, H, W, 3).astype(np.float32)
    add = rng.rand(B, oh, ow, 3).astype(np.float32)
    want = M.resize_bilinear_ac(x, oh, ow).astype(np.float64) + add
    for which in ("in", "add", "out", "all"):
        for k in F32_SHIFTS:
            a = shift_args({"in": dev(x), "add": dev(add), "out": torch.empty((B, oh, ow, 3), device="cuda")},
                           which, k)
            rc = _lib.load().hdrnet_resize_bilinear_f32(a["in"].data_ptr(), a["add"].data_ptr(), a["out"].data_ptr(),
                                                        B, H, W, 3, oh, ow, torch.cuda.current_stream().cuda_stream)
            _lib.check(rc, "resize_bilinear")
            err = np.abs(np_(a["out"]) - want).max()
            note("resize", err)
            assert err < 2e-6, f"resize {which} +{k}: {err:.3e}"


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.float32])
def test_lowres_from_shifted_image_is_bit_exact(dtype):
    rng = np.random.RandomState(93)
    B, H, W, S = 2, 120, 256, 64
    if dtype == np.float32:
        im = rng.rand(B, H, W, 3).astype(np.float32)
    else:
        im = rng.randint(0, np.iinfo(dtype).max + 1, size=(B, H, W, 3)).astype(dtype)
    want = np.stack([run.nearest_resize(run.img_as_float(im[b]), S) for b in range(B)])
    t = dev(im)
    for k in range(1, 16 // t.element_size()):
        got = np_(models.lowres_from_image(shifted(t, k), S))
        assert np.array_equal(got, want), f"{dtype} +{k}"


# ---- host paths --------------------------------------------------------------------------------
@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_host_slice_apply_on_shifted_host_buffers(pinned):
    grid, guide, inp, want = apply_case(OP_SHAPE, 64)
    B, H, W = OP_SHAPE[:3]
    for k in F32_SHIFTS:
        a = shift_args(dict(grid=torch.from_numpy(grid), guide=torch.from_numpy(guide), input=torch.from_numpy(inp),
                            out=torch.empty((B, H, W, 3))), "all", k, pin=pinned)
        got = hdrnet_ops.bilateral_slice_apply(a["grid"], a["guide"], a["input"], True, out=a["out"])
        assert got.data_ptr() == a["out"].data_ptr()
        note("host slice_apply", rel_err(got.numpy(), want))
        assert_parity(got.numpy(), want, rtol=RTOL, what=f"host {'pinned' if pinned else 'pageable'} +{k}")


def test_inference_image_host_on_shifted_pinned_frames():
    """Frames at an odd byte offset in page-locked memory, and an output at one: the same bytes as
    inference_image on each frame."""
    p = dict(GUIDE_PARAMS["curves"], net_input_size=64, spatial_bin=8)
    params = dict(p, weights=M.make_weights(p, seed=94))
    cls = models.HDRNetCurves
    frames = torch.from_numpy(np.random.RandomState(95).randint(0, 256, size=(3, 64, 256, 3)).astype(np.uint8))
    want = torch.cat([cls.inference_image(frames[i:i + 1].cuda(), params) for i in range(3)]).cpu()
    src = shifted(frames, 5, pin=True)
    out = shifted(torch.empty_like(frames), 11, pin=True)
    got = cls.inference_image_host(src, params, out=out)
    assert got.data_ptr() == out.data_ptr()
    assert torch.equal(got, want)
