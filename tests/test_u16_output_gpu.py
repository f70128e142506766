"""uint16 results from the model path: the fused slice-apply kernels' uint16 epilogue,
``inference_image(out_dtype=torch.uint16)``, ``inference_image_host`` and ``run.py --output_bit_depth 16``.

What is checked, and to what bar:
  * every kernel form's uint16 result equals np.rint(np.clip(f, 0, 1) * 65535), computed in float32,
    of the float32 result of the same kernel form on the same pixels -- bit for bit.  The float form
    is the call with a float32 ``out`` where that runs the same kernel (the per-pixel kernel reading
    integer pixels), else the float32 call on the img_as_float image (the row and texture-assisted
    forms: same per-pixel arithmetic) or, for float32 pixels in the per-pixel kernel, the standalone
    guide kernel + the generic slice-apply kernel (same summation order).  The img_as_float image is
    converted on the host (run.img_as_float, IEEE division, which the kernels reproduce bit for bit);
  * a grid of [I | 0] returns a uint16 image holding every code value in every channel unchanged
    (under a constant guide that keeps the smoothed depth weights' sum within 1e-7 of one);
  * outputs below 0, above 1 and NaN give 0, 65535 and 0;
  * the buffer contract: every output element written, nothing written outside the output, the
    input unchanged, no dependence on what a lent workspace held;
  * an output past 2^31 bytes: the straddling image equals the call on that image alone;
  * the host frame pipeline and run.py give what inference_image gives.
"""
import functools
import math

import cv2
import numpy as np
import pytest
import torch

from hdrnet_b200 import _lib, models
from hdrnet_b200.bin import run
from oracle import model_np as M

pytestmark = pytest.mark.gpu

FMT = {torch.float32: _lib.PX_F32, torch.uint8: _lib.PX_U8, torch.uint16: _lib.PX_U16}
DTYPES = {"u8": torch.uint8, "u16": torch.uint16, "f32": torch.float32}
KINDS = {"curves": ("HDRNetCurves", 16), "nn-f16": ("HDRNetPointwiseNNGuide", 16),
         "nn-f32": ("HDRNetPointwiseNNGuide", 32)}


def q16(f):
    """The 16-bit result restated in numpy: rint(65535 * clip(f, 0, 1)) in float32."""
    f = np.asarray(f, dtype=np.float32)
    return np.rint(np.clip(f, np.float32(0.0), np.float32(1.0)) * np.float32(65535.0)).astype(np.uint16)


def np_(t):
    return t.detach().cpu().numpy()


def i32(t):
    """uint16 tensors have few CUDA operators: compare them as int32."""
    return t.to(torch.int32)


@functools.lru_cache(maxsize=None)
def params_for(kind):
    name, feats = KINDS[kind] if kind in KINDS else ("HDRNetGaussianPyrNN", 16)
    p = dict(M.DEFAULT_PARAMS, model_name=name, net_input_size=64, spatial_bin=8, guide_complexity=feats)
    if name == "HDRNetPointwiseNNGuide":
        p["batch_norm"] = True
    p["weights"] = M.make_weights(p, seed=40 + feats)
    return p


def cls_of(kind):
    return getattr(models, params_for(kind)["model_name"])


def rand_image(seed, B, H, W, dtype, device="cuda"):
    g = torch.Generator(device=device).manual_seed(seed)
    if dtype == torch.float32:
        return torch.rand(B, H, W, 3, generator=g, device=device)
    hi = 256 if dtype == torch.uint8 else 65536
    return torch.randint(0, hi, (B, H, W, 3), generator=g, device=device, dtype=torch.int32).to(dtype)


def rand_coeffs(seed, B, gh=16, gw=16, gd=8, device="cuda"):
    """[B, gh, gw, gd, 3, 4]: near the identity, so that most outputs fall inside [0, 1]."""
    g = torch.Generator(device=device).manual_seed(seed)
    c = 0.15 * torch.randn(B, gh, gw, gd, 3, 4, generator=g, device=device)
    c[..., [0, 1, 2], [0, 1, 2]] += 1.0
    return c


def at_offset(shape, dtype, offset):
    """A contiguous [shape] view of `dtype` starting `offset` bytes past a 512-byte boundary."""
    item = torch.empty((), dtype=dtype).element_size()
    nbytes = math.prod(shape) * item
    buf = torch.zeros(nbytes + offset + 1024, dtype=torch.uint8, device="cuda")
    lo = (-buf.data_ptr()) % 512 + offset
    v = buf[lo:lo + nbytes].view(dtype).view(shape)
    assert v.data_ptr() % 512 == offset
    return v


def fused_call(kind, coeffs, x, out, ws=None):
    """hdrnet_slice_apply_{curves,nn}_px_ws into the caller's `out` (what models._slice_apply_fused
    launches), with the caller's workspace or none."""
    B, H, W, _ = x.shape
    gh, gw, gd = coeffs.shape[1:4]
    p = params_for(kind)
    guide = models._prepare(models._resolve_weights(p), p, x.device, cls_of(kind)._nn_guide).guides[0]
    lib = _lib.load()
    launch = lib.hdrnet_slice_apply_nn_px_ws if isinstance(guide, models._NNGuide) else lib.hdrnet_slice_apply_curves_px_ws
    rc = launch(coeffs.data_ptr(), x.data_ptr(), FMT[x.dtype], out.data_ptr(), FMT[out.dtype], 0, B, H, W, gh, gw,
                gd, *guide.args, 0 if ws is None else ws.data_ptr(), 0 if ws is None else ws.numel(),
                torch.cuda.current_stream().cuda_stream)
    return rc


def row_kernel_runs(in_dtype, W, aligned=True):
    """Whether the persistent row kernels (or their texture-assisted forms) take an integer -> uint16
    call: 16-byte aligned buffers, W >= 128 and W % 16 == 0 (W % 8 when both sides are uint16)."""
    return in_dtype != torch.float32 and aligned and W >= 128 and W % (8 if in_dtype == torch.uint16 else 16) == 0


def float_form(kind, coeffs, x, row_form):
    """The float32 result of the kernel form the uint16 call ran (module docstring)."""
    cls, p = cls_of(kind), params_for(kind)
    with torch.no_grad():
        if row_form:
            imf = torch.from_numpy(run.img_as_float(np_(x))).to(x.device)
            return cls._fullres(coeffs, imf, p, torch.float32)
        if x.dtype != torch.float32:
            return cls._fullres(coeffs, x, p, torch.float32)
        from hdrnet_b200 import hdrnet_ops
        B, gh, gw, gd = coeffs.shape[:4]
        return hdrnet_ops.bilateral_slice_apply(coeffs.reshape(B, gh, gw, gd, 12), cls._guide(x, p), x, True,
                                                variant=_lib.VARIANT_GENERIC)


def assert_u16_equals_float(got, f, what, min_inside=0.5):
    got, want = np_(got), q16(np_(f))
    assert got.dtype == np.uint16 and got.shape == want.shape, what
    bad = got != want
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} samples differ from rint(65535 * clip(f)), first "
                           f"at {np.argwhere(bad)[0].tolist()}: {got[bad][0]} vs {want[bad][0]}")
    inside = np_(f)
    frac = float(((inside > 0) & (inside < 1)).mean())
    assert frac >= min_inside, f"{what}: only {frac:.2f} of the samples are inside (0, 1)"


# ---- bit for bit against the float form ----------------------------------------------------------
SIZES = {
    "row-2x24x256": (2, 24, 256),            # row kernel, shared-memory slab
    "row-ragged-1x9x1104": (1, 9, 1104),     # two segments per row, the last one ragged
    "w1000-2x5x1000": (2, 5, 1000),          # W % 16 == 8: row kernel for uint16 in, per-pixel for uint8 in
    "per-pixel-2x11x101": (2, 11, 101),      # odd W: the per-pixel kernel
}


@pytest.mark.parametrize("size", list(SIZES))
@pytest.mark.parametrize("in_name", list(DTYPES))
@pytest.mark.parametrize("kind", list(KINDS))
def test_u16_result_is_the_float_result_rounded(kind, in_name, size):
    B, H, W = SIZES[size]
    dt = DTYPES[in_name]
    x = rand_image(len(size) + W, B, H, W, dt)
    coeffs = rand_coeffs(W, B)
    with torch.no_grad():
        got = cls_of(kind)._fullres(coeffs, x, params_for(kind), torch.uint16)
    row = row_kernel_runs(dt, W)
    assert_u16_equals_float(got, float_form(kind, coeffs, x, row), f"{kind} {in_name} {size} ({'row' if row else 'px'})")


@pytest.mark.parametrize("offset", [2, 4, 6])
@pytest.mark.parametrize("in_name", list(DTYPES))
@pytest.mark.parametrize("kind", ["curves", "nn-f16"])
def test_u16_result_at_unaligned_offsets(kind, in_name, offset):
    """Input and output views 2, 4 or 6 bytes past a 16-byte boundary at W = 256: the per-pixel kernel."""
    dt = DTYPES[in_name]
    if dt == torch.float32 and offset % 4:
        pytest.skip("float32 pixels sit on 4-byte boundaries")
    B, H, W = 2, 8, 256
    x = at_offset((B, H, W, 3), dt, offset)
    x.copy_(rand_image(offset, B, H, W, dt))
    coeffs = rand_coeffs(offset, B)
    out = at_offset((B, H, W, 3), torch.uint16, offset)
    _lib.check(fused_call(kind, coeffs, x, out), "fused slice-apply, uint16 out")
    assert_u16_equals_float(out, float_form(kind, coeffs, x, False), f"{kind} {in_name} +{offset}")


@pytest.mark.parametrize("in_name", ["u8", "u16"])
@pytest.mark.parametrize("kind", ["curves", "nn-f16", "nn-f32"])
def test_u16_result_of_the_8x4k_call(kind, in_name):
    """8 x 4K with a lent workspace, what AUTO runs there: the texture-assisted forms (the issuer-warp
    form for the curves guide, the block-synchronous one for the pointwise-NN guide)."""
    B, H, W = 8, 2160, 3840
    x = rand_image(7, B, H, W, DTYPES[in_name])
    coeffs = rand_coeffs(8, B)
    with torch.no_grad():
        got = np_(cls_of(kind)._fullres(coeffs, x, params_for(kind), torch.uint16))
    f = float_form(kind, coeffs, x, True)
    for b in range(B):
        assert_u16_equals_float(torch.from_numpy(got[b]), f[b], f"{kind} {in_name} 8 x 4K image {b}")


@pytest.mark.parametrize("in_name", ["u8", "u16"])
def test_pyramid_u16_result_is_its_float_result_rounded(in_name):
    cls, p = models.HDRNetGaussianPyrNN, params_for("pyramid")
    x = rand_image(9, 2, 100, 260, DTYPES[in_name])
    with torch.no_grad():
        got = cls.inference_image(x, p, out_dtype=torch.uint16)
        f = cls.inference_image(x, p, out_dtype=torch.float32)
    assert got.dtype == torch.uint16 and got.is_cuda
    assert_u16_equals_float(got, f, f"pyramid {in_name}", min_inside=0.0)
    assert torch.equal(i32(got), i32(models.quantize_u16(f)))


# ---- identity round trip and saturation ----------------------------------------------------------
IDENTITY_SIZES = {"row-1x256x256": (1, 256, 256), "texture-1x1024x2048": (1, 1024, 2048),
                  "per-pixel-1x128x515": (1, 128, 515)}


def every_code(H, W):
    """[1, H, W, 3] uint16 whose channels each run through all 65,536 codes (in different orders)."""
    n = np.arange(H * W, dtype=np.int64)
    ch = [(n * k + o) % 65536 for k, o in ((1, 0), (40503, 17), (65521, 999))]      # odd strides
    return torch.from_numpy(np.stack(ch, axis=1).astype(np.uint16).reshape(1, H, W, 3)).cuda()


def affine_coeffs(B, A, offset, gh=16, gw=16, gd=8):
    c = torch.zeros(B, gh, gw, gd, 3, 4, device="cuda")
    c[..., :3] = torch.tensor(A, dtype=torch.float32, device="cuda")
    c[..., 3] = torch.tensor(offset, dtype=torch.float32, device="cuda")
    return c


def constant_guide(kind, value=0.3):
    """params_for(kind) with the guide's output layer zeroed and its bias set so that the guide is
    `value` everywhere.  At 0.3 and 8 depth bins the depth coordinate's fraction is 0.9, where the
    smoothed tent weights max(1 - sqrt(d * d + 1e-8), 0) sum to one within 1e-7; near a fraction of 0
    or 1 they sum to up to 1e-4 less, and an identity grid is no identity there."""
    p = dict(params_for(kind))
    w = dict(p["weights"])
    if kind == "curves":
        w["inference/guide/channel_mixing/weights"] = np.zeros_like(w["inference/guide/channel_mixing/weights"])
        w["inference/guide/channel_mixing/biases"] = np.full_like(w["inference/guide/channel_mixing/biases"], value)
    else:
        w["inference/guide/conv2/weights"] = np.zeros_like(w["inference/guide/conv2/weights"])
        w["inference/guide/conv2/biases"] = np.full_like(w["inference/guide/conv2/biases"],
                                                         np.log(value / (1 - value)))
    p["weights"] = w
    return p


@pytest.mark.parametrize("size", list(IDENTITY_SIZES))
@pytest.mark.parametrize("kind", ["curves", "nn-f16"])
def test_identity_grid_returns_every_code_value(kind, size):
    _, H, W = IDENTITY_SIZES[size]
    p = constant_guide(kind)
    x = every_code(H, W)
    xn = np_(x)
    for c in range(3):
        assert len(np.unique(xn[..., c])) == 65536
    with torch.no_grad():
        got = np_(cls_of(kind)._fullres(affine_coeffs(1, np.eye(3), [0, 0, 0]), x, p, torch.uint16))
        guide = np_(cls_of(kind)._guide(x[:, :1, :64].to(torch.float32), p))
    assert np.abs(guide - 0.3).max() < 1e-3
    bad = got != xn
    assert not bad.any(), f"{kind} {size}: {int(bad.sum())} codes changed, e.g. {xn[bad][0]} -> {got[bad][0]}"


@pytest.mark.parametrize("size", list(IDENTITY_SIZES))
@pytest.mark.parametrize("kind", ["curves", "nn-f16"])
def test_saturation_and_nan(kind, size):
    """Below 0 -> 0, above 1 -> 65535, NaN -> 0; and an in-range value rounds to nearest (under the
    constant guide of the identity test, where the blend weights sum to one within 1e-7)."""
    _, H, W = IDENTITY_SIZES[size]
    x = rand_image(3, 1, H, W, torch.uint16)
    p = constant_guide(kind)
    for offset, want in (([-0.5, 1.5, float("nan")], [0, 65535, 0]), ([-1e30, 1e30, 0.25], [0, 65535, 16384])):
        with torch.no_grad():
            got = cls_of(kind)._fullres(affine_coeffs(1, np.zeros((3, 3)), offset), x, p, torch.uint16)
        got = np_(got)
        for c in range(3):
            vals = np.unique(got[..., c]).tolist()
            assert vals == [want[c]], f"{kind} {size} offset {offset[c]}: {vals[:5]}, want {want[c]}"


# ---- buffer contract -----------------------------------------------------------------------------
PAT_A, PAT_B = 0xFF, 0x5A
GUARD = 64 << 10


class Guarded:
    """A [shape] view of `dtype` with a guard band of >= 64 KiB (and >= one image row) on each side,
    `offset` bytes past a 512-byte boundary; the view holds `fill`, the guards `guard_fill`."""

    def __init__(self, shape, dtype, fill, guard_fill, offset=0):
        item = torch.empty((), dtype=dtype).element_size()
        self.nbytes = math.prod(shape) * item
        row = self.nbytes // max(math.prod(shape[:2]), 1) if len(shape) >= 3 else 0
        guard = -(-max(GUARD, row) // 512) * 512
        self.buf = torch.full((2 * guard + 512 + offset + self.nbytes,), guard_fill, dtype=torch.uint8, device="cuda")
        self.lo = guard + (-(self.buf.data_ptr() + guard)) % 512 + offset
        self.hi = self.lo + self.nbytes
        self.guard_fill = guard_fill
        self.buf[self.lo:self.hi].fill_(fill)
        self.view = self.buf[self.lo:self.hi].view(dtype).view(shape)

    def guards_intact(self):
        return bool((self.buf[:self.lo] == self.guard_fill).all()) and bool((self.buf[self.hi:] == self.guard_fill).all())


CONTRACT_CASES = {
    # id: (B, H, W, input dtype, input / output offset, lend a workspace)
    "row-u16-2x24x256": (2, 24, 256, torch.uint16, 0, False),
    "row-u8-1x9x1104": (1, 9, 1104, torch.uint8, 0, False),
    "texture-u16-1x1024x2048": (1, 1024, 2048, torch.uint16, 0, True),
    "texture-u8-ragged-1x1024x2064": (1, 1024, 2064, torch.uint8, 0, True),
    "per-pixel-f32-2x11x101": (2, 11, 101, torch.float32, 4, False),
    "per-pixel-u16-+2-2x9x256": (2, 9, 256, torch.uint16, 2, False),
}


@pytest.mark.parametrize("name", list(CONTRACT_CASES))
@pytest.mark.parametrize("kind", ["curves", "nn-f16"])
def test_buffer_contract(kind, name):
    """Under two fills of the output and of a workspace lent at exactly its queried size: the same
    bytes, no guard byte changed, the input unchanged, and the float form's result rounded."""
    B, H, W, dt, off, lend = CONTRACT_CASES[name]
    src = rand_image(11, B, H, W, dt)
    coeffs = rand_coeffs(12, B)
    gh, gw, gd = coeffs.shape[1:4]
    ws_bytes = _lib.load().hdrnet_slice_apply_workspace_bytes(B, H, gw, gd) if lend else 0
    runs = []
    for fill in (PAT_A, PAT_B):
        x = Guarded((B, H, W, 3), dt, 0, PAT_A, offset=off)
        x.view.copy_(src)
        before = x.buf.clone()
        out = Guarded((B, H, W, 3), torch.uint16, fill, fill, offset=off)
        ws = Guarded((ws_bytes,), torch.uint8, fill, fill) if lend else None
        _lib.check(fused_call(kind, coeffs, x.view, out.view, None if ws is None else ws.view), name)
        torch.cuda.synchronize()
        assert out.guards_intact(), f"{kind} {name} [fill {fill:#x}]: a write outside the output"
        assert ws is None or ws.guards_intact(), f"{kind} {name} [fill {fill:#x}]: a write outside the workspace"
        assert torch.equal(x.buf, before), f"{kind} {name} [fill {fill:#x}]: the input or its guards changed"
        runs.append(out.view.clone())
    diff = i32(runs[0]) != i32(runs[1])
    assert not bool(diff.any()), f"{kind} {name}: {int(diff.sum())} samples depend on what the buffers held"
    row = row_kernel_runs(dt, W, aligned=off % 16 == 0)
    assert_u16_equals_float(runs[0], float_form(kind, coeffs, src, row), f"{kind} {name}")


# ---- large extents -------------------------------------------------------------------------------
def test_output_past_2_31_bytes():
    """44 x 4K uint16 -> uint16 (2.19 GB each way): image 43 straddles byte 2^31 of the output (and
    of the input); it and image 0 equal the calls on those images alone."""
    B, H, W = 44, 2160, 3840
    per = H * W * 3 * 2
    assert (B - 1) * per < 2 ** 31 < B * per
    cls, p = cls_of("curves"), params_for("curves")
    x = torch.empty(B, H, W, 3, dtype=torch.uint16, device="cuda")
    for b in range(B):
        x[b] = rand_image(100 + b, 1, H, W, torch.uint16)[0]
    coeffs = rand_coeffs(13, B)
    with torch.no_grad():
        got = cls._fullres(coeffs, x, p, torch.uint16)
        for b in (B - 1, 0):
            alone = cls._fullres(coeffs[b:b + 1].contiguous(), x[b:b + 1], p, torch.uint16)
            assert torch.equal(i32(got[b:b + 1]), i32(alone)), f"image {b} of 44 x 4K differs from the call on it alone"
    del x, got


# ---- host pipeline and run.py --------------------------------------------------------------------
@pytest.mark.parametrize("kind,in_name", [("curves", "u8"), ("nn-f16", "u16"), ("pyramid", "u16")])
def test_host_frame_pipeline_u16(kind, in_name):
    cls, p = cls_of(kind), params_for(kind)
    frames = rand_image(21, 5, 48, 192, DTYPES[in_name], device="cpu").pin_memory()
    got = cls.inference_image_host(frames, p, out_dtype=torch.uint16)
    assert got.dtype == torch.uint16 and not got.is_cuda and got.is_pinned()
    assert tuple(got.shape) == tuple(frames.shape)
    for i in range(frames.shape[0]):
        want = cls.inference_image(frames[i:i + 1].cuda(), p, out_dtype=torch.uint16).cpu()
        assert np.array_equal(np_(got[i:i + 1]), np_(want)), f"{kind}: frame {i}"


def test_run_cli_output_bit_depth(tmp_path):
    """--output_bit_depth 16 writes 16-bit PNGs equal to inference_image(out_dtype=torch.uint16); the
    default writes the uint8 result; the --debug pictures stay 8-bit."""
    p = params_for("curves")
    ckpt = tmp_path / "ckpt"
    run.save_checkpoint(str(ckpt), {k: v for k, v in p.items() if k != "weights"}, p["weights"])
    (tmp_path / "in").mkdir()
    images = {"a16.png": np_(rand_image(31, 1, 72, 200, torch.uint16))[0],
              "b8.png": np_(rand_image(32, 1, 64, 256, torch.uint8))[0]}
    for name, im in images.items():
        assert cv2.imwrite(str(tmp_path / "in" / name), im[:, :, ::-1])
    for depth, flags in ((16, ["--output_bit_depth", "16", "--debug"]), (8, [])):
        out_dir = tmp_path / f"out{depth}"
        run.main(run.build_parser().parse_args([str(ckpt), str(tmp_path / "in"), str(out_dir), *flags]))
        for name, im in images.items():
            got = cv2.imread(str(out_dir / name), -1)
            assert got is not None and got.dtype == (np.uint16 if depth == 16 else np.uint8), (depth, name)
            with torch.no_grad():
                want = models.HDRNetCurves.inference_image(
                    torch.from_numpy(np.ascontiguousarray(im[None])).cuda(), p,
                    out_dtype=torch.uint16 if depth == 16 else torch.uint8)[0]
            assert np.array_equal(got[:, :, ::-1], np_(want)), f"{name} at {depth} bits"
            if depth == 16:
                stem = name[:-4]
                for suffix in ("_coeffs.png", "_guide_0.png"):
                    dbg = cv2.imread(str(out_dir / (stem + suffix)), -1)
                    assert dbg is not None and dbg.dtype == np.uint8, stem + suffix
