"""Every kernel on buffers past 2^31 and 2^32 bytes, and across the texture-width limit of the
slab workspace.

The rest of the suite runs each kernel at up to 8 x 4K (796 MB per buffer).  Users reach a 32-bit
byte offset with ordinary calls: 24 float32 4K frames are 2.4 GB in and 2.4 GB out, 88 uint8 4K
frames 2.2 GB.  A pixel offset formed in 32 bits wraps there, and a wrapped offset reads or writes
another image's pixels.  So each case here:

  * draws every image from its own seed on the device, so that reading the wrong image, or the
    right one at a wrapped offset, changes the output;
  * places its large buffers between guard bands of 1 MiB (NaN for float32 buffers, 0xA5 bytes for
    integer ones) and an output pre-filled with them: afterwards the guards are untouched and the
    output is finite;
  * compares, bitwise, each image whose input, output or guide bytes straddle a multiple of 2^31
    bytes, and the first and last image, with the same entry point called on that image alone.
    The row-kernel forms compute the same bits per pixel whatever the batch or the CTA partition
    (tests/test_slice_apply_gpu.py::test_row_kernels_are_bitwise_equal), so this is exact;
  * holds the image rows around each straddled byte to the float64 reference (oracle/slice_f64.py
    computed for those rows only) at the suite's bars.

``hdrnet_slice_apply_plan_ws`` asserts the slice-apply form wherever AUTO chooses it.  Cases run one
at a time and skip, saying why, when the device has less free memory than they need plus 2 GiB.
The last case passes 2^31 float32 elements in one buffer (about 21 GB in all) and skips unless
24 GB are free.  Run with -s to see each case's peak device memory and time.
"""
import ctypes
import gc
import time

import numpy as np
import pytest
import torch

from hdrnet_b200 import _lib, hdrnet_ops, models
from oracle import guide_f64
from oracle import model_np as M
from oracle import slice_f64
from test_guide_grad_gpu import DX_BAR, P_BAR, guide_weights, safe_dguide, vjp_cuda
from util import assert_parity

pytestmark = pytest.mark.gpu

GiB = 1 << 30
GUARD = 1 << 20
NAN_BYTE, INT_GUARD = 0xFF, 0xA5     # 0xFFFFFFFF is a float32 NaN
H4K, W4K = 2160, 3840
RTOL = 1e-5
GUIDE_BAR = 2e-6                     # tests/test_buffer_contract_gpu.py, guide kernels vs model_np
V = _lib


# ---- harness -----------------------------------------------------------------------------------
@pytest.fixture(autouse=True)
def _one_case_at_a_time(request):
    """Frees the previous case's memory first; reports this case's peak device memory and time."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / GiB
    print(f"\n[large extents] {request.node.name}: peak {peak:.2f} GiB, {time.perf_counter() - t0:.1f} s")
    gc.collect()
    torch.cuda.empty_cache()


def need(nbytes, what):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + 2 * GiB:
        pytest.skip(f"{what} needs {nbytes / GiB:.1f} GiB + 2 GiB of device memory; {free / GiB:.1f} GiB free")


class Guarded:
    """A contiguous ``shape`` / ``dtype`` view into a uint8 allocation with GUARD bytes on each side;
    everything, the view included, starts as the guard byte."""

    def __init__(self, shape, dtype):
        self.fill = NAN_BYTE if dtype.is_floating_point else INT_GUARD
        self.nbytes = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
        self.raw = torch.full((2 * GUARD + self.nbytes,), self.fill, dtype=torch.uint8, device="cuda")
        self.t = self.raw[GUARD:GUARD + self.nbytes].view(dtype).view(shape)

    def check(self, what):
        for side, g in (("front", self.raw[:GUARD]), ("back", self.raw[GUARD + self.nbytes:])):
            assert bool((g == self.fill).all()), f"{what}: {side} guard overwritten"


def fill_rand(t, seed, kind="rand"):
    """Image b of ``t`` from seed (seed, b) on the device: float32 uniform [0, 1) / normal, or uniform
    bytes for integer pixels (every uint16 value as two random bytes)."""
    gen = torch.Generator(device="cuda")
    for b in range(t.shape[0]):
        gen.manual_seed(seed * 100003 + b)
        if t.dtype == torch.float32:
            (torch.rand if kind == "rand" else torch.randn)(t[b].shape, generator=gen, device="cuda", out=t[b])
        else:
            u = t[b].view(torch.uint8)
            torch.randint(0, 256, u.shape, generator=gen, device="cuda", dtype=torch.uint8, out=u)
    return t


def rand_grid(B, gh, gw, gd, gc, seed):
    g = fill_rand(torch.empty((B, gh, gw, gd, gc), device="cuda"), seed, "randn")
    g.view(B, gh, gw, gd, gc // 4, 4)[..., [0, 1, 2], [0, 1, 2]] += 1.0    # near identity: outputs in range
    return g


def straddlers(B, *image_bytes):
    """{b: [byte offsets inside image b that are multiples of 2^31]} for every buffer's bytes per
    image, plus the first and last image."""
    out = {0: [], B - 1: []}
    for n in image_bytes:
        for k in range(1, (B * n) // (1 << 31) + 1):
            b, off = divmod(k * (1 << 31), n)
            if b < B:
                out.setdefault(b, []).append((n, off))
    return out


def band_rows(offsets, px_bytes, W, H, halo=1):
    """Row bands [y0, y1) around each straddled byte of the buffer with ``px_bytes`` per pixel
    (``offsets`` from straddlers: (bytes per image, byte in image)); the last rows of the image when
    that buffer has none in it."""
    bands = [(max(0, off // (W * px_bytes) - halo), min(H, off // (W * px_bytes) + halo + 1))
             for n, off in offsets if n == H * W * px_bytes]
    return bands or [(H - 2, H)]


def all_finite(t):
    """Image by image: isfinite of a whole multi-GB buffer would take temporaries of its size."""
    return all(bool(torch.isfinite(t[b]).all()) for b in range(t.shape[0]))


def np_(t):
    return t.detach().cpu().numpy()


def plan(B, H, W, gh, gw, gd, ws=True):
    """(variant, threads) hdrnet_slice_apply_plan_ws reports for AUTO on the float32 3 -> 3 op."""
    v, c, t, s = (ctypes.c_int() for _ in range(4))
    _lib.check(_lib.load().hdrnet_slice_apply_plan_ws(B, H, W, gh, gw, gd, 3, 3, 1, int(ws), ctypes.byref(v),
                                                      ctypes.byref(c), ctypes.byref(t), ctypes.byref(s)), "plan")
    return v.value, t.value


def f64_rows(grid_b, guide_b, inp_b, y0, y1):
    """float64 slice-apply of rows [y0, y1) of one image."""
    H = guide_b.shape[0]
    return slice_f64.bilateral_slice_apply(np_(grid_b)[None], np_(guide_b[y0:y1])[None], np_(inp_b[y0:y1])[None],
                                           True, y_off=y0, height=H)[0]


# ---- slice-apply, op API -----------------------------------------------------------------------
APPLY_CASES = {
    # name: (B, (gh, gw, gd), variants, AUTO's (variant, threads) for the batch and for one image)
    "24x4k-16x16x8-issuer-warp": (24, (16, 16, 8), (V.VARIANT_AUTO,), (V.VARIANT_TEX_ASYNC, 384)),
    "45x4k-16x16x8-past-4GiB": (45, (16, 16, 8), (V.VARIANT_AUTO,), (V.VARIANT_TEX_ASYNC, 384)),
    "24x4k-32x32x16-pre-pass-tma-tex": (24, (32, 32, 16), (V.VARIANT_AUTO, V.VARIANT_TMA, V.VARIANT_TEX),
                                        (V.VARIANT_TEX_ASYNC, 352)),
}


def run_apply_case(B, gdims, variants, form, seed):
    gh, gw, gd = gdims
    npx = H4K * W4K
    ws = B * H4K * gw * gd * 48
    need(B * npx * 28 + ws + 64 * npx, f"{B} x 4K slice-apply")
    assert plan(B, H4K, W4K, gh, gw, gd) == form and plan(1, H4K, W4K, gh, gw, gd) == form
    grid = rand_grid(B, gh, gw, gd, 12, seed)
    guide = Guarded((B, H4K, W4K), torch.float32)
    inp = Guarded((B, H4K, W4K, 3), torch.float32)
    out = Guarded((B, H4K, W4K, 3), torch.float32)
    fill_rand(guide.t, seed + 1)
    fill_rand(inp.t, seed + 2, "randn")
    picks = straddlers(B, npx * 12, npx * 4)
    first = {}
    for variant in variants:
        with torch.no_grad():
            hdrnet_ops.bilateral_slice_apply(grid, guide.t, inp.t, True, out=out.t, variant=variant)
        torch.cuda.synchronize()
        what = f"{B} x 4K {gdims} variant {variant}"
        for g in (guide, inp, out):
            g.check(what)
        assert all_finite(out.t), f"{what}: output not finite (unwritten or wrong pixels)"
        for b, offs in sorted(picks.items()):
            with torch.no_grad():
                one = hdrnet_ops.bilateral_slice_apply(grid[b:b + 1], guide.t[b:b + 1], inp.t[b:b + 1], True,
                                                       variant=variant)
            assert torch.equal(out.t[b], one[0]), f"{what}: image {b} differs from the call on it alone"
            if variant == variants[0]:
                first[b] = one[0].clone()
                for y0, y1 in sorted(set(band_rows(offs, 12, W4K, H4K) + band_rows(offs, 4, W4K, H4K))):
                    assert_parity(np_(out.t[b, y0:y1]), f64_rows(grid[b], guide.t[b], inp.t[b], y0, y1),
                                  what=f"{what} image {b} rows {y0}:{y1}")
            else:   # every row-kernel form computes the same bits
                assert torch.equal(out.t[b], first[b]), f"{what}: image {b} differs from variant {variants[0]}"
    return grid, guide, inp, out


@pytest.mark.parametrize("name", list(APPLY_CASES))
def test_slice_apply_batches_past_2_31_bytes(name):
    B, gdims, variants, form = APPLY_CASES[name]
    run_apply_case(B, gdims, variants, form, seed=10 + B)


def test_slice_apply_host_buffers_past_2_31_bytes():
    """The host-buffer path (pageable tensors, row bands copied at byte offsets past 2^31) equals the
    device call bitwise: both run row-kernel forms."""
    B = 24
    grid, guide, inp, out = run_apply_case(B, (16, 16, 8), (V.VARIANT_AUTO,), (V.VARIANT_TEX_ASYNC, 384), seed=40)
    h_grid, h_guide, h_inp = grid.cpu(), guide.t.cpu(), inp.t.cpu()
    del guide, inp
    h_out = torch.full((B, H4K, W4K, 3), float("nan"))
    with torch.no_grad():
        hdrnet_ops.bilateral_slice_apply(h_grid, h_guide, h_inp, True, out=h_out)
    assert torch.equal(h_out, out.t.cpu()), "host-buffer path differs from the device call"


# ---- the texture-width limit of the slab workspace ---------------------------------------------
# A 32x32x16 slab row is 24 KiB = 1536 float4 texels; a texture over linear memory holds at most 2^27
# texels, so the texture-assisted forms take B * H <= 87,381 rows of such a grid and AUTO runs the
# TMA row kernel from 87,382 rows on.
TEX_W, TEX_G = 128, (32, 32, 16)
TEX_ROWS_MAX = (1 << 27) // (TEX_G[1] * TEX_G[2] * 3)


def tex_case(H, seed):
    grid = rand_grid(1, *TEX_G, 12, seed)
    guide = fill_rand(torch.empty((1, H, TEX_W), device="cuda"), seed + 1)
    inp = fill_rand(torch.empty((1, H, TEX_W, 3), device="cuda"), seed + 2, "randn")
    return grid, guide, inp


def c_abi_call(grid, guide, inp, variant, ws):
    B, H, W, _ = inp.shape
    out = Guarded(tuple(inp.shape), torch.float32)
    ptr, nbytes = (ws.t.data_ptr(), ws.nbytes) if ws is not None else (0, 0)
    rc = _lib.load().hdrnet_slice_apply_f32_ws(grid.data_ptr(), guide.data_ptr(), inp.data_ptr(), out.t.data_ptr(),
                                               B, H, W, *TEX_G, 3, 3, 1, int(variant), ptr, nbytes,
                                               torch.cuda.current_stream().cuda_stream)
    return rc, out


@pytest.mark.parametrize("H", [TEX_ROWS_MAX, TEX_ROWS_MAX + 1], ids=["last-texture-row", "first-tma-row"])
def test_texture_width_limit(H):
    assert TEX_ROWS_MAX == 87381
    lib = _lib.load()
    ws_bytes = lib.hdrnet_slice_apply_workspace_bytes(1, H, TEX_G[1], TEX_G[2])
    assert (ws_bytes // 16 <= (1 << 27)) == (H == TEX_ROWS_MAX)
    need(2 * ws_bytes + H * TEX_W * 64, "texture-width case")
    variant, _ = plan(1, H, TEX_W, *TEX_G)
    if H == TEX_ROWS_MAX:
        assert variant in (V.VARIANT_TEX, V.VARIANT_TEX_ASYNC), variant
    else:
        assert variant == V.VARIANT_TMA, variant
    # the op API and the model path lend the workspace only where the texture forms will use it
    assert hdrnet_ops._texture_form_runs(torch.cuda.current_device(), 1, H, TEX_W, *TEX_G) == (H == TEX_ROWS_MAX)
    grid, guide, inp = tex_case(H, 70)
    ws = Guarded((ws_bytes // 4,), torch.float32)
    rc, auto = c_abi_call(grid, guide, inp, V.VARIANT_AUTO, ws)
    _lib.check(rc, "AUTO")
    rc_tma, tma = c_abi_call(grid, guide, inp, V.VARIANT_TMA, None)
    _lib.check(rc_tma, "TMA")
    rc_tex, tex = c_abi_call(grid, guide, inp, V.VARIANT_TEX, ws)
    if H == TEX_ROWS_MAX:
        _lib.check(rc_tex, "TEX")
    else:
        assert rc_tex == V.E_UNSUPPORTED, f"TEX past the texture limit: rc {rc_tex}"
    torch.cuda.synchronize()
    for name, o in (("AUTO", auto), ("TMA", tma), ("ws", ws)) + ((("TEX", tex),) if rc_tex == 0 else ()):
        o.check(f"H={H} {name}")
    assert all_finite(auto.t), f"H={H}: AUTO output not finite"
    assert torch.equal(auto.t, tma.t), f"H={H}: AUTO differs from the TMA row kernel"
    if rc_tex == 0:
        assert torch.equal(tex.t, tma.t), f"H={H}: TEX differs from the TMA row kernel"
    with torch.no_grad():
        op = hdrnet_ops.bilateral_slice_apply(grid, guide, inp, True)
    assert torch.equal(op, auto.t), f"H={H}: the op API differs from the C-ABI call"
    # the rows whose slab texels lie just below 2^27, the last rows, and the first rows
    for y0, y1 in ((TEX_ROWS_MAX - 6, TEX_ROWS_MAX - 2), (H - 3, H), (0, 3)):
        assert_parity(np_(auto.t[0, y0:y1]), f64_rows(grid[0], guide[0], inp[0], y0, y1), what=f"H={H} rows {y0}:{y1}")


def test_row_bands_past_the_texture_limit():
    """Bands of the 87,382-row image: one of 16,384 rows ending at the last row (2 Mi px: a texture
    form over its own workspace), and short ones starting past texel 2^27 of the whole image's
    workspace; each equals the whole-image rows bitwise."""
    H = TEX_ROWS_MAX + 1
    need(8 * H * TEX_W * 12, "row bands")
    grid, guide, inp = tex_case(H, 80)
    with torch.no_grad():
        whole = hdrnet_ops.bilateral_slice_apply(grid, guide, inp, True)
        for y0, rows, form in ((H - 16384, 16384, (V.VARIANT_TEX, V.VARIANT_TEX_ASYNC)),
                               (TEX_ROWS_MAX - 1, 2, (V.VARIANT_TMA,)), (H - 1, 1, (V.VARIANT_TMA,))):
            assert plan(1, rows, TEX_W, *TEX_G)[0] in form
            band = hdrnet_ops.bilateral_slice_apply_rows(grid, guide[:, y0:y0 + rows].contiguous(),
                                                         inp[:, y0:y0 + rows].contiguous(), True, y0, H)
            assert torch.equal(band, whole[:, y0:y0 + rows]), f"band at row {y0} ({rows} rows)"


# ---- VJPs ---------------------------------------------------------------------------------------
def test_slice_apply_vjps_past_2_31_bytes():
    """The grid, guide and input VJPs of 24 x 4K: image b of each equals the call on image b alone
    (the grid VJP sums per image, in a fixed order); the input and guide VJPs of the rows around
    the straddled bytes meet the float64 VJPs."""
    B, (gh, gw, gd) = 24, (16, 16, 8)
    npx = H4K * W4K
    need(B * npx * 44, "24 x 4K VJPs")
    grid = rand_grid(B, gh, gw, gd, 12, 90).requires_grad_(True)
    guide = Guarded((B, H4K, W4K), torch.float32)
    inp = Guarded((B, H4K, W4K, 3), torch.float32)
    ct = Guarded((B, H4K, W4K, 3), torch.float32)
    fill_rand(guide.t, 91)
    fill_rand(inp.t, 92, "randn")
    fill_rand(ct.t, 93, "randn")
    gt, it = guide.t.requires_grad_(True), inp.t.requires_grad_(True)
    out = hdrnet_ops.bilateral_slice_apply(grid, gt, it, True)
    dgrid, dguide, dinp = torch.autograd.grad(out, (grid, gt, it), ct.t)
    del out
    torch.cuda.synchronize()
    for g in (guide, inp, ct):
        g.check("VJP inputs")
    for name, d in (("grid", dgrid), ("guide", dguide), ("input", dinp)):
        assert all_finite(d), f"{name} VJP not finite"
    for b, offs in sorted(straddlers(B, npx * 12, npx * 4).items()):
        leaves = [t[b:b + 1].detach().requires_grad_(True) for t in (grid, gt, it)]
        one = hdrnet_ops.bilateral_slice_apply(*leaves, True)
        ones = torch.autograd.grad(one, leaves, ct.t[b:b + 1])
        for name, d, o in (("grid", dgrid, ones[0]), ("guide", dguide, ones[1]), ("input", dinp, ones[2])):
            assert torch.equal(d[b], o[0]), f"{name} VJP of image {b} differs from the call on it alone"
        for y0, y1 in band_rows(offs, 12, W4K, H4K):
            r = slice_f64.bilateral_slice_apply_grad(np_(grid[b])[None], np_(gt[b, y0:y1])[None],
                                                     np_(it[b, y0:y1])[None], np_(ct.t[b, y0:y1])[None], True,
                                                     y_off=y0, height=H4K)
            assert_parity(np_(dinp[b, y0:y1]), r.input[0], elem_rtol=None, what=f"input VJP image {b} rows {y0}:{y1}")
            scale = np.maximum(np.abs(r.guide).max(), r.guide_abs)[0]
            err = float((np.abs(np_(dguide[b, y0:y1]) - r.guide[0]) / np.maximum(scale, 1e-30)).max())
            assert err <= RTOL, f"guide VJP image {b} rows {y0}:{y1}: {err:.3e}"


# ---- the model path -----------------------------------------------------------------------------
GUIDE_PARAMS = {"curves": dict(M.DEFAULT_PARAMS),
                "nn": dict(M.DEFAULT_PARAMS, model_name="HDRNetPointwiseNNGuide", batch_norm=True)}


def model(kind):
    p = GUIDE_PARAMS[kind]
    return getattr(models, p["model_name"]), dict(p, weights=M.make_weights(p, seed=100))


def check_fullres(cls, params, coeffs, x, out, out_dtype, what):
    """Images straddling 2^31 bytes of x or out: bitwise against _fullres on the image alone, and their
    straddled rows against the staged reference (the float64 slice oracle fed the coefficients and
    the standalone guide kernel's guide)."""
    B, H, W, _ = x.shape
    npx = H * W
    in_bpp, out_bpp = 3 * x.element_size(), 3 * out.element_size()
    for b, offs in sorted(straddlers(B, npx * in_bpp, npx * out_bpp).items()):
        with torch.no_grad():
            one = cls._fullres(coeffs[b:b + 1], x[b:b + 1], params, out_dtype)
        assert torch.equal(out[b], one[0]), f"{what}: image {b} differs from the call on it alone"
        for y0, y1 in sorted(set(band_rows(offs, in_bpp, W, H) + band_rows(offs, out_bpp, W, H))):
            with torch.no_grad():
                imf = models.image_to_float(x[b:b + 1, y0:y1].contiguous())
                guide = cls._guide(imf, params)
            stage = slice_f64.bilateral_slice_apply(np_(coeffs[b]).reshape(1, 16, 16, 8, 12), np_(guide), np_(imf),
                                                    True, y_off=y0, height=H)[0]
            got = np_(out[b, y0:y1])
            if out_dtype == torch.float32:
                assert_parity(got, stage, rtol=RTOL, what=f"{what} image {b} rows {y0}:{y1}")
            else:
                q = (np.float32(255.0) * np.clip(stage.astype(np.float32), 0, 1)).astype(np.uint8)
                assert np.abs(got.astype(int) - q.astype(int)).max() <= 1, f"{what} image {b} rows {y0}:{y1}"


@pytest.mark.parametrize("kind", list(GUIDE_PARAMS))
def test_model_inference_past_2_31_bytes(kind):
    """24 x 4K float32 through inference: coefficients layer by layer (B > 16), guide fused into the
    texture-assisted slice-apply."""
    B, S = 24, 256
    npx = H4K * W4K
    need(B * npx * 40, f"{kind} inference")
    assert plan(B, H4K, W4K, 16, 16, 8)[0] in (V.VARIANT_TEX, V.VARIANT_TEX_ASYNC)
    cls, params = model(kind)
    low = fill_rand(torch.empty((B, S, S, 3), device="cuda"), 101)
    x = Guarded((B, H4K, W4K, 3), torch.float32)
    fill_rand(x.t, 102)
    with torch.no_grad():
        out = cls.inference(low, x.t, params)
        coeffs = cls._coefficients(low, params)
        staged = cls._fullres(coeffs, x.t, params, torch.float32)
    torch.cuda.synchronize()
    x.check(kind)
    assert all_finite(out), f"{kind}: output not finite"
    assert torch.equal(out, staged), f"{kind}: inference differs from its own stages"
    del staged
    check_fullres(cls, params, coeffs, x.t, out, torch.float32, f"{kind} inference")


@pytest.mark.parametrize("in_dtype, B", [(torch.uint8, 88), (torch.uint16, 44)], ids=["u8-88x4k", "u16-44x4k"])
def test_inference_image_past_2_31_bytes(in_dtype, B):
    """Integer pixels in, uint8 out: 2.2 GB of 8- or 16-bit pixels, and lowres_from_image at the same batch."""
    S = 256
    npx = H4K * W4K
    in_bpp = 3 * torch.empty((), dtype=in_dtype).element_size()
    need(B * npx * (in_bpp + 8), "inference_image")
    cls, params = model("curves")
    x = Guarded((B, H4K, W4K, 3), in_dtype)
    fill_rand(x.t, 110 + in_bpp)
    with torch.no_grad():
        out = cls.inference_image(x.t, params)
        low = models.lowres_from_image(x.t, S)
        coeffs = cls._coefficients(low, params)
        staged = cls._fullres(coeffs, x.t, params, torch.uint8)
    torch.cuda.synchronize()
    x.check("inference_image input")
    assert out.dtype == torch.uint8 and torch.equal(out, staged), "inference_image differs from its own stages"
    del staged
    for b in straddlers(B, npx * in_bpp, npx * 3):
        with torch.no_grad():
            assert torch.equal(low[b], models.lowres_from_image(x.t[b:b + 1], S)[0]), f"lowres of image {b}"
    check_fullres(cls, params, coeffs, x.t, out, torch.uint8, f"inference_image {in_dtype}")


@pytest.mark.parametrize("kind", list(GUIDE_PARAMS))
def test_guide_kernels_past_2_31_bytes(kind):
    """The standalone guide kernels over 24 x 4K float32 pixels (2.4 GB)."""
    B = 24
    npx = H4K * W4K
    need(B * npx * 16, f"{kind} guide")
    cls, params = model(kind)
    x = Guarded((B, H4K, W4K, 3), torch.float32)
    fill_rand(x.t, 120)
    with torch.no_grad():
        guide = cls._guide(x.t, params)
    torch.cuda.synchronize()
    x.check(f"{kind} guide input")
    assert all_finite(guide)
    ref = M.guide_curves if kind == "curves" else M.guide_nn
    for b, offs in sorted(straddlers(B, npx * 12, npx * 4).items()):
        with torch.no_grad():
            assert torch.equal(guide[b], cls._guide(x.t[b:b + 1], params)[0]), f"{kind} guide of image {b}"
        for y0, y1 in band_rows(offs, 12, W4K, H4K):
            err = np.abs(np_(guide[b, y0:y1]) - ref(np_(x.t[b:b + 1, y0:y1]), params["weights"])[0]).max()
            assert err < GUIDE_BAR, f"{kind} guide image {b} rows {y0}:{y1}: {err:.3e}"


def test_curves_guide_vjp_past_2_31_bytes():
    """hdrnet_guide_curves_grad_f32 over 24 x 4K (2.4 GB of pixels and of dinput), built from 3
    distinct frames (with their own upstream gradients) in a fixed pattern: dinput of the images
    around 2^31 bytes, and the first and last, equal the call on the image alone bitwise and meet
    their frame's float64 VJP; each parameter gradient meets the sum over frames of count x that
    frame's float64 gradient.  The parameter sums are chunked by pixel count, so they are not
    bitwise across batch sizes.  Each frame tiles a 240 x 480 patch of its own 9 x 8 times, so that
    the float64 VJP (seconds per megapixel) is computed on the patch only."""
    B = 24
    npx = H4K * W4K
    need(B * npx * 28, "curves guide VJP")
    pattern = [b % 4 % 3 for b in range(B)]                  # frame 0 twelve times, 1 and 2 six times each
    rng = np.random.RandomState(140)
    w = guide_weights(rng)
    ph, pw = H4K // 9, W4K // 8
    tiles = (H4K // ph) * (W4K // pw)
    frames = []
    for _ in range(3):
        xp = (rng.rand(ph, pw, 3) * 1.2 - 0.1).astype(np.float32)
        gp, near = safe_dguide(xp, rng.randn(ph, pw), w)
        assert near <= ph * pw // 2000
        frames.append((xp, gp, guide_f64.vjp(xp, gp, w)))
    x = Guarded((B, H4K, W4K, 3), torch.float32)
    g = Guarded((B, H4K, W4K), torch.float32)
    dev = [(torch.from_numpy(f[0]).cuda().repeat(9, 8, 1), torch.from_numpy(f[1]).cuda().repeat(9, 8))
           for f in frames]
    for b, f in enumerate(pattern):
        x.t[b].copy_(dev[f][0])
        g.t[b].copy_(dev[f][1])
    del dev
    dx, dp = vjp_cuda(x.t, g.t, w)
    for t in (x, g):
        t.check("guide VJP inputs")
    assert all_finite(dx)
    for b in sorted(straddlers(B, npx * 12, npx * 4)):
        one, _ = vjp_cuda(x.t[b:b + 1], g.t[b:b + 1], w, want_p=False)
        assert torch.equal(dx[b], one[0]), f"dinput of image {b} differs from the call on it alone"
        ref = np.tile(frames[pattern[b]][2].dinput, (9, 8, 1))
        e = np.abs(np_(dx[b]).astype(np.float64) - ref).max() / np.abs(ref).max()
        assert e <= DX_BAR, f"dinput of image {b}: {e:.3e} of range"
    counts = [tiles * pattern.count(f) for f in range(3)]
    want = sum(c * guide_f64.flat(f[2].dparams) for c, f in zip(counts, frames))
    terms = sum(c * guide_f64.flat(f[2].dparams_abs) for c, f in zip(counts, frames))
    got = np_(dp).astype(np.float64)
    e = np.abs(got - want) / np.maximum(terms, 1e-30)
    e[(terms == 0) & (got == 0)] = 0.0
    assert e.max() <= P_BAR, f"dparams[{int(e.argmax())}]: {e.max():.3e} of sum |terms|"


def test_pyramid_inference_past_2_31_bytes():
    """HDRNetGaussianPyrNN at 24 x 4K: level 0 (2.4 GB) through the fused NN-guide slice-apply, the
    resizes reading and writing it; image by image equal to the model on that image alone, given
    the batch's coefficients."""
    B = 24
    npx = H4K * W4K
    need(B * npx * 48, "pyramid")
    p = dict(M.DEFAULT_PARAMS, model_name="HDRNetGaussianPyrNN", net_input_size=128, spatial_bin=16)
    params = dict(p, weights=M.make_weights(p, seed=150))
    cls = models.HDRNetGaussianPyrNN
    low = fill_rand(torch.empty((B, 128, 128, 3), device="cuda"), 151)
    x = Guarded((B, H4K, W4K, 3), torch.float32)
    fill_rand(x.t, 152)
    with torch.no_grad():
        out = cls.inference(low, x.t, params)
        coeffs = cls._coefficients(low, params)
        staged = cls._output(cls._multiscale_input(x.t), None, coeffs, params)
        torch.cuda.synchronize()
        x.check("pyramid input")
        assert all_finite(out)
        assert torch.equal(out, staged), "pyramid inference differs from its own stages"
        del staged
        for b in sorted(straddlers(B, npx * 12)):
            one = cls._output(cls._multiscale_input(x.t[b:b + 1]), None, coeffs[b:b + 1], params)
            assert torch.equal(out[b], one[0]), f"pyramid image {b} differs from the model on it alone"


# ---- past 2^31 float32 elements -----------------------------------------------------------------
def test_slice_apply_past_2_31_elements():
    """87 x 4K: 2.17 Gi float32 elements in the input and in the output, 8.7 GB each; guide bytes past
    2^31 too.  Needs about 22 GB of device memory."""
    free, _ = torch.cuda.mem_get_info()
    if free < 24 * GiB:
        pytest.skip(f"87 x 4K needs 24 GiB free; {free / GiB:.1f} GiB free")
    assert 87 * H4K * W4K * 3 > (1 << 31)
    run_apply_case(87, (16, 16, 8), (V.VARIANT_AUTO,), (V.VARIANT_TEX_ASYNC, 384), seed=130)
