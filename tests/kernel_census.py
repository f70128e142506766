"""Every CUDA entry function the library compiles, the smallest public call that launches it, and the
float64 (or exact) reference that call is held to.

`ROWS` maps (source file, kernel) to the id of a case in `CASES`.  The kernel is the demangled name,
normalised by `normalise`: no return type, no parameter list, no `hdrnet_b200::` and no
`(anonymous namespace)::`, no blanks.  The source file is part of the key because two objects may
define kernels of one name (bn_train.cu and guide_nn_grad.cu each have a `stats_partial_kernel`).
tests/test_kernel_census.py holds the keys to the library's symbols in both directions;
tests/test_kernel_census_gpu.py runs each case under the profiler (it must launch every kernel whose
row names it) and holds its results to its reference.

A case is a function of no arguments: it makes its seeded inputs, launches, and returns a check.  The
check computes the reference and returns [(what, error, bar)].  Cases stay small: one call, one or
two images, the smallest shape that reaches the form; the edge-case matrices live in the files of
their features.
"""
import re
import shutil
import subprocess

import numpy as np
import torch

import oracle
from hdrnet_b200 import _lib, data_pipeline, hdrnet_ops, models
from hdrnet_b200.bin import run
from oracle import bn_train_f64, cnn_grad_f64, guide_f64, resize_f64, slice_f64
from oracle import model_np as M

import nn_guide_f64
from test_slice_apply_gpu import ISSUER_WARP_CASES

# ---- names ----------------------------------------------------------------------------------------


def normalise(raw):
    """A kernel's demangled name as cuobjdump | c++filt or torch.profiler spell it -> the census key,
    e.g. 'void hdrnet_b200::conv2d_patch_kernel<2, 4>(hdrnet_b200::ConvArgs)' -> 'conv2d_patch_kernel<2,4>'."""
    name = raw.strip()
    name = name.replace("(anonymous namespace)::", "").replace("hdrnet_b200::", "")
    if name.startswith("void "):
        name = name[5:]
    depth = 0
    for i, ch in enumerate(name):
        depth += ch == "<"
        depth -= ch == ">"
        if ch == "(" and depth == 0:
            name = name[:i]
            break
    return re.sub(r"\s+", "", name)


def cuobjdump():
    """The toolkit's cuobjdump, or None."""
    import os
    for cand in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"),
                                                         "bin", "cuobjdump")):
        if cand and os.path.exists(cand):
            return cand
    return None


def library_kernels(lib_path, tool):
    """{(source file, kernel)} of the entry functions in the library's sm_90a code."""
    out = subprocess.run([tool, "-symbols", lib_path], check=True, capture_output=True, text=True).stdout
    mangled, source = [], None
    for line in out.splitlines():
        if line.startswith("identifier = "):
            source = line.split("=", 1)[1].strip().rsplit("/", 1)[-1]
        elif "STO_ENTRY" in line:
            mangled.append((source, line.split()[-1]))
    names = subprocess.run(["c++filt"], input="\n".join(m for _, m in mangled), check=True,
                           capture_output=True, text=True).stdout.splitlines()
    return {(src, normalise(n)) for (src, _), n in zip(mangled, names)}


# ---- inputs and bars ------------------------------------------------------------------------------
def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.detach().cpu().numpy()


def rel(got, want):
    """max |got - want| / max |want| (float64)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    if not np.isfinite(got).all():
        return float("inf")
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def rel_terms(got, want, terms):
    """max |got - want| / Σ|terms| per reduced element (the scale its float32 sum rounds against)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    if not np.isfinite(got).all():
        return float("inf")
    return float((np.abs(got - want) / np.maximum(np.asarray(terms, np.float64), 1e-30)).max())


CODE_MAX = {torch.uint8: 255.0, torch.uint16: 65535.0}
OUTPUT_BAR = 1e-5          # the float result's bar, of range


def f32_bound(gh, gw, gd):
    """How far a float32 slice-apply result may lie from float64, per unit of Σ|terms| (the sum of its
    terms' magnitudes): the rounding of the sums and products, and of the cell positions x gw / W,
    y gh / H and guide x gd, which move weight between corners by a few float32 units per cell of
    the axis.  Measured over the census: at most 3.4 units (2^-24) per cell of the longest axis plus
    a constant; this allows 6 per cell plus 8."""
    return 2.0 ** -24 * (8 + 6 * max(gh, gw, gd))


def code_err(got, want_f64, err_bound, dtype):
    """Pixels of an integer result off the quantised float64 value: floor(255 clip) for uint8,
    rint(65535 clip) for uint16.  A pixel may be one code off only where the float64 value, scaled to
    codes, lies within its float32 error bound `err_bound` (per pixel, f32_bound Σ|terms|) or 1e-3 of a
    code of a rounding boundary.  Returns the number of other pixels."""
    D = CODE_MAX[dtype]
    s = D * np.clip(np.asarray(want_f64, np.float64), 0.0, 1.0)
    want = np.floor(s) if dtype == torch.uint8 else np.rint(s)
    bound = np.abs(s - np.round(s)) if dtype == torch.uint8 else np.abs(np.abs(s - np.floor(s)) - 0.5)
    window = np.maximum(1e-3, D * np.asarray(err_bound, np.float64))
    d = np.abs(np.asarray(got, np.float64) - want)
    return int(((d > 1) | ((d == 1) & (bound > window))).sum())


def img_as_float(im):
    """skimage.img_as_float of a code image, as float32 (float32(float64(v) / D)); float32 as is."""
    if im.dtype == np.uint8:
        return (im.astype(np.float64) / 255.0).astype(np.float32)
    if im.dtype == np.uint16:
        return (im.astype(np.float64) / 65535.0).astype(np.float32)
    return im


def rand_image(seed, shape, dtype):
    rng = np.random.RandomState(seed)
    if dtype == torch.float32:
        return rng.rand(*shape).astype(np.float32)
    hi = 256 if dtype == torch.uint8 else 65536
    return rng.randint(0, hi, size=shape).astype(np.uint8 if dtype == torch.uint8 else np.uint16)


# ---- cases ---------------------------------------------------------------------------------------
CASES = {}
ROWS = {}


def case(case_id, fn):
    CASES[case_id] = fn
    return case_id


def row(source, kernel, case_id):
    assert (source, kernel) not in ROWS, (source, kernel)
    ROWS[(source, kernel)] = case_id


VARIANT = {"auto": _lib.VARIANT_AUTO, "generic": _lib.VARIANT_GENERIC, "tma": _lib.VARIANT_TMA,
           "tex": _lib.VARIANT_TEX, "tex_async": _lib.VARIANT_TEX_ASYNC}


# -- the op API: slice-apply with the guide as an input, slice, indices ----------------------------
def op_apply(seed, shape, n_in=3, n_out=3, has_offset=True, variant="auto", edge=False):
    B, H, W, gh, gw, gd = shape

    def fn():
        rng = np.random.RandomState(seed)
        J = n_in + int(has_offset)
        grid = rng.randn(B, gh, gw, gd, n_out * J).astype(np.float32)
        guide = rng.rand(B, H, W).astype(np.float32)
        if edge:
            guide[0, :, ::5] = 1.75
            guide[0, :, 1::5] = -0.6
        inp = rng.randn(B, H, W, n_in).astype(np.float32)
        out = hdrnet_ops.bilateral_slice_apply(cuda(grid), cuda(guide), cuda(inp), has_offset,
                                               variant=VARIANT[variant])
        return lambda: [("slice-apply", rel(host(out), slice_f64.bilateral_slice_apply(grid, guide, inp, has_offset)), 1e-5)]
    return case(f"op_apply[{variant},{'x'.join(map(str, shape))},{n_in}->{n_out},{int(has_offset)}]", fn)


def op_slice(seed, shape, gc, variant="auto"):
    B, H, W, gh, gw, gd = shape

    def fn():
        rng = np.random.RandomState(seed)
        grid = rng.randn(B, gh, gw, gd, gc).astype(np.float32)
        guide = rng.rand(B, H, W).astype(np.float32)
        out = hdrnet_ops.bilateral_slice(cuda(grid), cuda(guide), variant=VARIANT[variant])
        return lambda: [("slice", rel(host(out), slice_f64.bilateral_slice(grid, guide)), 1e-5)]
    return case(f"op_slice[{variant},{'x'.join(map(str, shape))},gc={gc}]", fn)


def _indices():
    rng = np.random.RandomState(21)
    guide = rng.rand(2, 9, 70).astype(np.float32)
    guide[0, 0, :6] = [0.0, 1.0, -0.25, 1.5, 0.5, 0.125]
    idx = hdrnet_ops.slice_indices(cuda(guide), (5, 7, 8))
    want = oracle.port().slice_indices(guide, 5, 7, 8)
    return lambda: [("cell indices", float(np.count_nonzero(host(idx) != want)), 0.0)]


def _slice_grads(apply):
    """The slice-apply VJP (slice_grad_pixel_kernel: guide and input; slice_grad_grid_kernel: grid) or the
    slice VJP, through autograd."""
    def fn():
        rng = np.random.RandomState(22)
        B, H, W, gh, gw, gd = 2, 12, 40, 4, 5, 8
        gc = 12
        grid = rng.randn(B, gh, gw, gd, gc).astype(np.float32)
        guide = rng.rand(B, H, W).astype(np.float32)
        inp = rng.randn(B, H, W, 3).astype(np.float32)
        tg, tu, ti = (cuda(a).requires_grad_() for a in (grid, guide, inp))
        if apply:
            out = hdrnet_ops.bilateral_slice_apply(tg, tu, ti, True)
        else:
            out = hdrnet_ops.bilateral_slice(tg, tu)
        ct = rng.randn(*out.shape).astype(np.float32)
        out.backward(cuda(ct))

        def check():
            if apply:
                r = slice_f64.bilateral_slice_apply_grad(grid, guide, inp, ct, True)
            else:
                r = slice_f64.bilateral_slice_grad(grid, guide, ct)
            res = [("d grid", rel_terms(host(tg.grad), r.grid, r.grid_abs), 4e-6),
                   ("d guide", rel(host(tu.grad), r.guide), 1e-5)]
            if apply:
                res.append(("d input", rel(host(ti.grad), r.input), 1e-5))
            return res
        return check
    return fn


# -- the model path: guide-fused slice-apply -------------------------------------------------------
GUIDES = {"curves": ("HDRNetCurves", 16), "nn16": ("HDRNetPointwiseNNGuide", 16),
          "nn32": ("HDRNetPointwiseNNGuide", 32)}
_PARAMS = {}


def model_params(kind, **extra):
    key = (kind, tuple(sorted(extra.items())))
    if key not in _PARAMS:
        name, feats = GUIDES[kind] if kind in GUIDES else (kind, 16)
        p = dict(M.DEFAULT_PARAMS, model_name=name, net_input_size=64, spatial_bin=8, luma_bins=8,
                 guide_complexity=feats, batch_norm=name != "HDRNetCurves")
        p.update(extra)
        p["weights"] = M.make_weights(p, seed=3)
        _PARAMS[key] = p
    return _PARAMS[key]


def guide_f64_of(kind, x, p):
    """The guide of float image(s) x [..., 3] in float64."""
    if kind == "curves":
        return guide_f64.guide(np.asarray(x, np.float64), p["weights"])
    return M.guide_nn(np.asarray(x, np.float64), p["weights"]).astype(np.float64)


def _rows_to_check(H):
    """Row bands the float64 reference is computed on: all rows of a small image; the first, last and
    some middle rows of a large one."""
    if H <= 64:
        return [(0, H)]
    mid = H // 2
    return [(0, 8), (mid - 4, 8), (H - 8, 8)]


def fused_check(kind, p, coeffs, codes, outs, out_dtype):
    """Image i of `codes` (numpy, [H, W, 3]) with grid row i of `coeffs`: its float image, the standalone
    guide kernel's guide map (held to float64 at 2e-6), slice_f64 fed that map at 1e-5 of range, or
    the quantised float64 value for integer results."""
    cls = getattr(models, p["model_name"])
    res = []
    B, gh, gw, gd = coeffs.shape[:4]
    c = host(coeffs).reshape(B, gh, gw, gd, 12)
    for i, (im, out) in enumerate(zip(codes, outs)):
        f = img_as_float(im)[None]
        g = host(cls._guide(cuda(f), p))
        got = host(out)[None]
        H = f.shape[1]
        want_g, want, terms, have = [], [], [], []
        for y0, h in _rows_to_check(H):
            gb, fb = g[:, y0:y0 + h], f[:, y0:y0 + h]
            want_g.append(guide_f64_of(kind, fb, p))
            have.append(gb)
            want.append(slice_f64.bilateral_slice_apply(c[i:i + 1], gb, fb, True, y_off=y0, height=H))
            terms.append(slice_f64.bilateral_slice_apply(np.abs(c[i:i + 1]), gb, np.abs(fb), True, y_off=y0, height=H))
        res.append((f"image {i}: guide", float(np.abs(np.concatenate(have, 1) - np.concatenate(want_g, 1)).max()), 2e-6))
        want, terms = np.concatenate(want, 1), np.concatenate(terms, 1)
        got = np.concatenate([got[:, y0:y0 + h] for y0, h in _rows_to_check(H)], 1)
        if out_dtype == torch.float32:
            res.append((f"image {i}: output", rel(got, want), OUTPUT_BAR))
            res.append((f"image {i}: output / sum|terms|", rel_terms(got, want, terms), f32_bound(gh, gw, gd)))
        else:
            err_bound = f32_bound(gh, gw, gd) * terms
            res.append((f"image {i}: output codes off", float(code_err(got, want, err_bound, out_dtype)), 0.0))
    return res


def coefficients_for(p, B, seed):
    cls = getattr(models, p["model_name"])
    low = torch.from_numpy(np.random.RandomState(seed).rand(B, 64, 64, 3).astype(np.float32)).cuda()
    with torch.no_grad():
        return cls._coefficients(low, p)


def fused(kind, in_dtype, out_dtype, shape, lend_workspace=False, grid=None):
    """One guide-fused slice-apply call (models._slice_apply_fused, what inference_image runs)."""
    B, H, W = shape
    extra = {} if grid is None else dict(spatial_bin=grid[0], luma_bins=grid[1])

    def fn():
        p = model_params(kind, **extra)
        cls = getattr(models, p["model_name"])
        codes = rand_image(31, (B, H, W, 3), in_dtype)
        coeffs = coefficients_for(p, B, 32)
        prep = models._prepare(p["weights"], p, torch.device("cuda"), cls._nn_guide)
        out, _ = models._slice_apply_fused(coeffs, cuda(codes), prep.guides[0], out_dtype, False, lend_workspace)
        return lambda: fused_check(kind, p, coeffs, list(codes), list(out), out_dtype)
    tag = "" if grid is None else f",grid{grid[0]}x{grid[1]}"
    return case(f"fused[{kind},{str(in_dtype)[6:]}->{str(out_dtype)[6:]},{B}x{H}x{W}{',ws' if lend_workspace else ''}{tag}]", fn)


def ragged(kind, in_dtype, out_dtype):
    """inference_images on two images of different sizes: the ragged fused kernel, on one image the
    single-image row kernels take (its quad path) and one they do not (its per-pixel path)."""
    def fn():
        p = model_params(kind)
        cls = getattr(models, p["model_name"])
        codes = [rand_image(33, (20, 256, 3), in_dtype), rand_image(34, (36, 70, 3), in_dtype)]
        outs = cls.inference_images([cuda(c) for c in codes], p, out_dtype=out_dtype)

        def check():
            coeffs = cls._coefficients(models.lowres_from_images([cuda(c) for c in codes], 64), p)
            return fused_check(kind, p, coeffs, codes, outs, out_dtype)
        return check
    return case(f"ragged[{kind},{str(in_dtype)[6:]}->{str(out_dtype)[6:]}]", fn)


def _guide_kernel(kind):
    def fn():
        p = model_params(kind)
        cls = getattr(models, p["model_name"])
        x = np.random.RandomState(35).rand(1, 20, 70, 3).astype(np.float32)
        g = cls._guide(cuda(x), p)
        return lambda: [("guide", float(np.abs(host(g) - guide_f64_of(kind, x, p)).max()), 2e-6)]
    return fn


# -- the coefficient network's layers ----------------------------------------------------------------
def conv(cin, cout, B, H, stride=1, form="auto", relu=True, tensor_cores=False):
    """One conv layer through models._conv: form 'auto' (conv dispatch: CUDA-core, patch or unpacked
    tensor cores), 'packed' (packed weights from PACKED_CONV_MIN_TILES tiles) or 'fp32' (CUDA cores at
    every size).  `tensor_cores`: the row's kernel is a wgmma form (bar 5e-5, else 2e-5); the launch
    census holds the case to that kernel."""
    def fn():
        rng = np.random.RandomState(cin * 1000 + cout + B)
        x = rng.randn(B, H, H, cin).astype(np.float32)
        w = (rng.randn(3, 3, cin, cout) / np.sqrt(9 * cin)).astype(np.float32)
        b = rng.randn(cout).astype(np.float32) * 0.1
        wd, bd = cuda(w), cuda(b)
        wb = (wd, bd, models.pack_conv_weights(wd)) if form == "packed" else (wd, bd)
        out = models._conv(cuda(x), wb, stride=stride, relu=relu, tensor_cores=form != "fp32")

        def check():
            want = M.conv2d_same(x.astype(np.float64), w.astype(np.float64), stride) + b
            want = np.maximum(want, 0) if relu else want
            return [("conv", max(rel(host(out)[i], want[i]) for i in range(B)), 5e-5 if tensor_cores else 2e-5)]
        return check
    return case(f"conv[{form},{B}x{H}x{H}x{cin}->{cout},s{stride}]", fn)


def fc(B, I, O, relu=True):
    def fn():
        rng = np.random.RandomState(I + O + B)
        x = rng.randn(B, I).astype(np.float32)
        w = (rng.randn(I, O) / np.sqrt(I)).astype(np.float32)
        b = rng.randn(O).astype(np.float32) * 0.1
        out = models._fc(cuda(x), (cuda(w), cuda(b)), relu=relu)

        def check():
            want = x.astype(np.float64) @ w.astype(np.float64) + b
            want = np.maximum(want, 0) if relu else want
            return [("fc", max(rel(host(out)[i], want[i]) for i in range(B)), 2e-5)]
        return check
    return case(f"fc[{B}x{I}->{O}]", fn)


def coefficients(B):
    """The whole coefficient network (launch chain up to CHAIN_CNN_MAX_BATCH images), per image."""
    def fn():
        p = model_params("curves")
        low = np.random.RandomState(36).rand(B, 64, 64, 3).astype(np.float32)
        with torch.no_grad():
            got = models.HDRNetCurves._coefficients(cuda(low), p)

        def check():
            want = M.coefficients(low.astype(np.float64), p["weights"], p)
            return [("coefficients", max(rel(host(got)[i], want[i]) for i in range(B)), 2e-5)]
        return check
    return case(f"coefficients[B={B}]", fn)


def _pack():
    """conv_tc_pack_kernel: the packed weights give the unpacked tensor-core result bit for bit."""
    rng = np.random.RandomState(37)
    x = cuda(rng.randn(1, 128, 96, 16).astype(np.float32))
    wd = cuda((rng.randn(3, 3, 16, 32) / 12.0).astype(np.float32))
    packed = models.pack_conv_weights(wd)
    a = models._conv(x, (wd, None, packed), relu=False)
    bb = models._conv(x, (wd, None), relu=False)
    return lambda: [("packed == unpacked", float((a != bb).sum().item()), 0.0)]


# -- coefficient-network VJPs ------------------------------------------------------------------------
def conv_grad(cin, cout, B, H, stride):
    def fn():
        rng = np.random.RandomState(cin + cout + 7)
        x = rng.randn(B, H, H, cin).astype(np.float32)
        w = (rng.randn(3, 3, cin, cout) / np.sqrt(9 * cin)).astype(np.float32)
        b = (rng.randn(cout) * 0.1).astype(np.float32)
        tx, tw, tb = (cuda(a).requires_grad_() for a in (x, w, b))
        y = models._ConvFn.apply(tx, tw, tb, stride, True)
        dy = rng.randn(*y.shape).astype(np.float32)
        y.backward(cuda(dy))

        def check():
            xr, wr = cnn_grad_f64._t(x), cnn_grad_f64._t(w)
            out = (cnn_grad_f64.conv_same(xr, wr, stride) + torch.from_numpy(b.astype(np.float64))).numpy()
            r = cnn_grad_f64.conv_vjp(x, w, np.maximum(out, 0), dy, stride, True)
            return [("d x", rel(host(tx.grad), r.dx), 1e-5), ("d w", rel_terms(host(tw.grad), r.dw, r.dw_abs), 4e-6),
                    ("d b", rel(host(tb.grad), r.db), 1e-5)]
        return check
    return case(f"conv_grad[{B}x{H}x{H}x{cin}->{cout},s{stride}]", fn)


def fc_grad():
    rng = np.random.RandomState(38)
    x = rng.randn(3, 64).astype(np.float32)
    w = (rng.randn(64, 32) / 8).astype(np.float32)
    b = (rng.randn(32) * 0.1).astype(np.float32)
    tx, tw, tb = (cuda(a).requires_grad_() for a in (x, w, b))
    y = models._FcFn.apply(tx, tw, tb, True)
    dy = rng.randn(*y.shape).astype(np.float32)
    y.backward(cuda(dy))

    def check():
        out = np.maximum(x.astype(np.float64) @ w + b, 0)
        r = cnn_grad_f64.fc_vjp(x, w, out, dy, True)
        return [("d x", rel(host(tx.grad), r.dx), 1e-5), ("d w", rel_terms(host(tw.grad), r.dw, r.dw_abs), 4e-6),
                ("d b", rel(host(tb.grad), r.db), 1e-5)]
    return check


def fuse_grad():
    rng = np.random.RandomState(39)
    gd, n_out, n_in, C, B, s = 4, 3, 4, 16, 2, 4
    local = np.maximum(rng.randn(B, s, s, C), 0).astype(np.float32)
    glob = np.maximum(rng.randn(B, C), 0).astype(np.float32)
    w = (rng.randn(C, gd * n_out * n_in) / 4).astype(np.float32)
    b = (rng.randn(gd * n_out * n_in) * 0.1).astype(np.float32)
    tl, tg, tw, tb = (cuda(a).requires_grad_() for a in (local, glob, w, b))
    y = models._FusePredictFn.apply(tl, tg, tw, tb, gd, n_out, n_in)
    dy = rng.randn(*y.shape).astype(np.float32)
    y.backward(cuda(dy))

    def check():
        want = cnn_grad_f64.fuse_predict(*(cnn_grad_f64._t(a) for a in (local, glob, w, b)), gd, n_out, n_in).numpy()
        r = cnn_grad_f64.fuse_predict_vjp(local, glob, w, dy, gd, n_out, n_in)
        return [("forward", rel(host(y), want), 2e-5), ("d local", rel(host(tl.grad), r.dlocal), 1e-5),
                ("d global", rel(host(tg.grad), r.dglobal), 1e-5),
                ("d w", rel_terms(host(tw.grad), r.dw, r.dw_abs), 4e-6), ("d b", rel_terms(host(tb.grad), r.db, r.db_abs), 4e-6)]
    return check


# -- batch norm in training mode -----------------------------------------------------------------------
def bn(N, C):
    def fn():
        rng = np.random.RandomState(N + C)
        z = (rng.randn(N, C) * 2 + 0.5).astype(np.float32)
        beta = (rng.randn(C) * 0.3).astype(np.float32)
        moving = (torch.zeros(C, device="cuda"), torch.ones(C, device="cuda"))
        tz, tb = cuda(z).requires_grad_(), cuda(beta).requires_grad_()
        y = models._BatchNormReluFn.apply(tz, tb, moving)
        dy = rng.randn(N, C).astype(np.float32)
        y.backward(cuda(dy))

        def check():
            want, _, _ = bn_train_f64.bn_relu(z, beta)
            r = bn_train_f64.bn_relu_vjp(z, beta, dy)
            return [("y", rel(host(y), want), 1e-5), ("d z", rel(host(tz.grad), r.dz), 1e-5),
                    ("d beta", rel_terms(host(tb.grad), r.dbeta, r.dbeta_abs), 4e-6)]
        return check
    return case(f"bn[{N}x{C}]", fn)


# -- the guides' VJPs ----------------------------------------------------------------------------------
def _curves_guide_grad(want_x, want_p):
    def fn():
        p = model_params("curves")
        wts = {k: (cuda(np.asarray(v, np.float32)).requires_grad_(want_p) if k.startswith("inference/guide/")
                   else v) for k, v in p["weights"].items()}
        x = np.random.RandomState(40).rand(1, 12, 40, 3).astype(np.float32)
        tx = cuda(x).requires_grad_(want_x)
        g = models.HDRNetCurves._guide(tx, dict(p, weights=wts, guide_grad=True))
        dg = np.random.RandomState(41).randn(*g.shape).astype(np.float32)
        g.backward(cuda(dg))

        def check():
            r = guide_f64.vjp(x, dg, p["weights"])
            res = []
            if want_x:
                res.append(("d input", rel_terms(host(tx.grad), r.dinput, r.dinput_abs), 4e-6))
            if want_p:
                for n in guide_f64.NAMES:
                    got = host(wts["inference/guide/" + n].grad).reshape(r.dparams[n].shape)
                    res.append((f"d {n}", rel_terms(got, r.dparams[n], r.dparams_abs[n]), 4e-6))
            return res
        return check
    return case(f"curves_guide_grad[x={int(want_x)},params={int(want_p)}]", fn)


def nn_guide_grad(feats):
    def fn():
        p = model_params("nn16" if feats == 16 else "nn32", guide_batch_stats=True)
        scope = "inference/guide"
        wts = {k: (cuda(np.asarray(v, np.float32)).requires_grad_(k.split(scope + "/")[-1] in nn_guide_f64.NAMES)
                   if k.startswith(scope + "/") else v) for k, v in p["weights"].items()}
        wts_host = {k: np.asarray(v, np.float32).copy() for k, v in p["weights"].items()}
        x = np.random.RandomState(42).rand(1, 12, 40, 3).astype(np.float32)
        tx = cuda(x).requires_grad_()
        g = models.HDRNetPointwiseNNGuide._guide(tx, dict(p, weights=wts, guide_grad=True), is_training=True)
        dg = np.random.RandomState(43).randn(*g.shape).astype(np.float32)
        g.backward(cuda(dg))

        def check():
            r = nn_guide_f64.vjp(x, dg, wts_host)
            res = [("guide", float(np.abs(host(g) - nn_guide_f64.guide(x, wts_host)).max()), 2e-6),
                   ("d input", rel(host(tx.grad), r.dinput), 1e-5)]
            for n in nn_guide_f64.NAMES:
                got = host(wts[f"{scope}/{n}"].grad).reshape(r.dparams[n].shape)
                res.append((f"d {n}", rel_terms(got, r.dparams[n], r.dparams_abs[n]), 4e-6))
            return res
        return check
    return case(f"nn_guide_grad[F={feats}]", fn)


# -- resize, network inputs, frozen pyramid, training batches ---------------------------------------
def _resize_grad():
    rng = np.random.RandomState(44)
    x = rng.randn(2, 9, 13, 3).astype(np.float32)
    tx = cuda(x).requires_grad_()
    y = models._ResizeFn.apply(tx, 17, 25, None)
    dy = rng.randn(2, 17, 25, 3).astype(np.float32)
    y.backward(cuda(dy))

    def check():
        r = resize_f64.resize_vjp(dy, 9, 13)
        return [("resize", rel(host(y), resize_f64.resize(x, 17, 25)), 1e-6),
                ("d input", rel_terms(host(tx.grad), r.din, r.din_abs), 4e-6)]
    return check


def lowres(in_dtype, ragged_call):
    def fn():
        shapes = [(37, 53), (20, 90)]
        codes = [rand_image(45 + i, s + (3,), in_dtype) for i, s in enumerate(shapes)]
        if ragged_call:
            got = models.lowres_from_images([cuda(c) for c in codes], 16)
        else:
            codes = codes[:1]
            got = models.lowres_from_image(cuda(codes[0][None]), 16)

        def check():
            want = np.stack([run.nearest_resize(run.img_as_float(c), 16) for c in codes])
            return [("network input", float(np.count_nonzero(host(got) != want)), 0.0)]
        return check
    return case(f"lowres[{str(in_dtype)[6:]},{'ragged' if ragged_call else 'batch'}]", fn)


def frozen_pyramid(in_dtype, out_dtype):
    """The frozen pyramid model: img_as_float of the image, the levels' resizes (the last quantised by
    the resize epilogue) and the split of the grid rows.  Bitwise inference_image, and within one code
    of the float64 model."""
    def fn():
        import tempfile
        from hdrnet_b200 import checkpoint
        from hdrnet_b200.frozen import FrozenModel
        p = model_params("HDRNetGaussianPyrNN")
        cls = models.HDRNetGaussianPyrNN
        codes = rand_image(46, (1, 24, 40, 3), in_dtype)
        with tempfile.TemporaryDirectory() as d:
            path = checkpoint.freeze_model(p["weights"], p, d + "/pyr.hdrnet")
            with FrozenModel(path) as model:
                got = model(cuda(codes), out_dtype=out_dtype)
        py = cls.inference_image(cuda(codes), p, out_dtype=out_dtype)

        def check():
            f = img_as_float(codes[0])[None]
            low = run.nearest_resize(f[0], 64)[None]
            want = M.gaussian_pyr_inference(low, f, p["weights"], p, oracle.best().bilateral_slice_apply)[0]
            s = CODE_MAX[out_dtype] * np.clip(want, 0, 1)
            d = np.abs(host(got).astype(np.float64) - (np.floor(s) if out_dtype == torch.uint8 else np.rint(s)))
            return [("frozen != inference_image", float((host(got) != host(py)).sum()), 0.0),
                    ("codes more than one off the model", float((d > 1).sum()), 0.0)]
        return check
    return case(f"frozen_pyramid[{str(in_dtype)[6:]}->{str(out_dtype)[6:]}]", fn)


def _augment(im, d, oh, ow):
    x = np.flip(im, 1) if d.fliplr else im
    x = np.rot90(np.flip(x, 0) if d.flipud else x, d.rot90)
    return x[d.crop_y:d.crop_y + oh, d.crop_x:d.crop_x + ow]


def _nearest_tf1(crop, S):
    oh, ow = crop.shape[:2]
    ys = np.minimum(np.floor(np.arange(S, dtype=np.float32) * (np.float32(oh) / np.float32(S))).astype(np.int64), oh - 1)
    xs = np.minimum(np.floor(np.arange(S, dtype=np.float32) * (np.float32(ow) / np.float32(S))).astype(np.int64), ow - 1)
    return crop[ys][:, xs]


def _train_batch():
    from hdrnet_b200.data_pipeline import Draw
    rng = np.random.RandomState(47)
    srcs = [rng.randint(0, 256, size=(20, 24, 3)).astype(np.uint8), rng.rand(20, 24, 3).astype(np.float32)]
    tgts = [rng.randint(0, 65536, size=(20, 24, 3)).astype(np.uint16), rng.rand(20, 24, 3).astype(np.float32)]
    draws = [Draw(0, True, False, 1, 2, 3), Draw(1, False, True, 3, 0, 1)]
    out = data_pipeline.train_batch([cuda(s) for s in srcs], [cuda(t) for t in tgts], draws, (16, 16), 8)

    def check():
        fin = np.stack([img_as_float(_augment(a, d, 16, 16)) for a, d in zip(srcs, draws)])
        fout = np.stack([img_as_float(_augment(b, d, 16, 16)) for b, d in zip(tgts, draws)])
        want = (fin, fout, np.stack([_nearest_tf1(f, 8) for f in fin]))
        return [(name, float(np.count_nonzero(host(g) != w)), 0.0) for name, g, w in
                zip(("input", "target", "network input"), out, want)]
    return check


def _usm():
    from hdrnet_b200.data_pipeline import Draw
    from scipy.ndimage import gaussian_filter1d
    rng = np.random.RandomState(48)
    src = rng.randint(0, 256, size=(30, 34, 3)).astype(np.uint8)
    sigma, sharpen = 2.0, 1.5
    draws = [Draw(0, False, False, 0, 0, 0)]
    out = data_pipeline.usm_batch([cuda(src)], draws, (30, 34), None, sigma, sharpen)

    def check():
        x = img_as_float(src).astype(np.float64)
        blur = gaussian_filter1d(gaussian_filter1d(x, sigma, axis=0, mode="reflect", truncate=4.0),
                                 sigma, axis=1, mode="reflect", truncate=4.0)
        want = np.clip(x + sharpen * (x - blur), 0, 1)
        return [("input", float(np.count_nonzero(host(out[0])[0] != img_as_float(src))), 0.0),
                ("target", float(np.abs(host(out[1])[0] - want).max()), 4e-6 * (1 + sharpen))]
    return check


# ---- the table -----------------------------------------------------------------------------------
F32, U8, U16 = torch.float32, torch.uint8, torch.uint16
FMT = {F32: 0, U8: 1, U16: 2}
GUIDE_T = {"curves": "GuideCurves", "nn16": "GuideNN<16>", "nn32": "GuideNN<32>"}

# op API, slice_apply.cu
row("slice_apply.cu", "slice_apply_rows_tma_kernel<GuideFromInput,0,2,256,0,0>",
    op_apply(1, (1, 8, 256, 8, 8, 8), variant="tma"))
_tex = op_apply(2, (1, 8, 256, 8, 8, 8), variant="tex")
row("slice_apply.cu", "slice_apply_rows_tma_kernel<GuideFromInput,4,2,512,0,0>", _tex)
row("slice_apply.cu", "yblend_rows_kernel", _tex)
row("slice_apply.cu", "slice_generic_kernel<true>", op_apply(3, (2, 7, 33, 3, 4, 5), variant="generic"))
row("slice_apply.cu", "slice_rows_any_kernel<true,12,3,3>", op_apply(4, (1, 8, 100, 8, 8, 8)))
row("slice_apply.cu", "slice_rows_any_kernel<true,9,3,3>", op_apply(5, (1, 8, 100, 8, 8, 8), has_offset=False))
row("slice_apply.cu", "slice_rows_any_kernel<true,36,3,9>", op_apply(6, (1, 8, 100, 8, 8, 8), n_out=9))
row("slice_apply.cu", "slice_rows_any_kernel<true,0,0,0>", op_apply(7, (1, 8, 100, 4, 4, 4), n_in=2, n_out=2))
row("slice_apply.cu", "slice_rows_tma_kernel", op_slice(8, (1, 8, 256, 8, 8, 8), 12, "tma"))
row("slice_apply.cu", "slice_generic_kernel<false>", op_slice(9, (2, 7, 33, 3, 4, 5), 5, "generic"))
row("slice_apply.cu", "slice_rows_any_kernel<false,12,0,0>", op_slice(10, (1, 8, 100, 8, 8, 8), 12))
row("slice_apply.cu", "slice_rows_any_kernel<false,0,0,0>", op_slice(11, (1, 8, 100, 8, 8, 8), 5))
row("slice_apply.cu", "slice_indices_kernel", case("slice_indices", _indices))

# issuer-warp forms, slice_apply_async.cu: the first shape of each (slab warp, lean) in
# tests/test_slice_apply_gpu.py, which checks that form against the block-synchronous one bitwise
_issuer = {}
for (seed, *shape, edge), form in ISSUER_WARP_CASES.items():
    _issuer.setdefault(form, (seed, tuple(shape), edge))
for (slab, lean), (seed, shape, edge) in sorted(_issuer.items()):
    row("slice_apply_async.cu",
        f"slice_apply_rows_async_kernel<5,{str(lean).lower()},{384 if slab else 352},2,{str(slab).lower()}>",
        op_apply(seed, shape, variant="tex_async", edge=edge))

# guide-fused forms
_ROW_FMTS = [(F32, F32), (U8, U8), (U8, U16), (U16, U8), (U16, U16)]
for kind, gt in GUIDE_T.items():
    for i, o in _ROW_FMTS:
        W = 256
        row("slice_apply.cu", f"slice_apply_rows_tma_kernel<{gt},0,2,256,{FMT[i]},{FMT[o]}>", fused(kind, i, o, (1, 16, W)))
        # texture-assisted (>= 2 Mi pixels, workspace lent); the curves guide runs its issuer-warp form
        # there, and the block-synchronous one where that form cannot keep two CTAs per SM
        if kind == "curves":
            row("slice_apply_async.cu", f"slice_apply_rows_async_fused_kernel<GuideCurves,4,{FMT[i]},{FMT[o]}>",
                fused(kind, i, o, (1, 548, 3840), lend_workspace=True))
            row("slice_apply.cu", f"slice_apply_rows_tma_kernel<{gt},4,2,256,{FMT[i]},{FMT[o]}>",
                fused(kind, i, o, (1, 548, 3840), lend_workspace=True, grid=(32, 32)))
        else:
            row("slice_apply.cu", f"slice_apply_rows_tma_kernel<{gt},4,2,256,{FMT[i]},{FMT[o]}>",
                fused(kind, i, o, (1, 548, 3840), lend_workspace=True))
    for i, o in [(U8, U8), (U16, U8), (F32, U8), (U8, F32), (U16, F32), (U8, U16), (U16, U16), (F32, U16)]:
        W = 256 if F32 in (i, o) else 100        # no row form for these formats / W % 16 != 0
        row("slice_apply.cu", f"slice_apply_px_generic_kernel<{gt},{FMT[i]},{FMT[o]}>", fused(kind, i, o, (2, 11, W)))
    for i in (F32, U8, U16):
        for o in (F32, U8, U16):
            row("slice_apply_ragged.cu", f"slice_apply_ragged_kernel<{gt},{FMT[i]},{FMT[o]}>", ragged(kind, i, o))

# standalone guides, guide.cu
row("guide.cu", "guide_kernel<CurvesFn>", case("guide[curves]", _guide_kernel("curves")))
row("guide.cu", "guide_kernel<NNFn<16>>", case("guide[nn16]", _guide_kernel("nn16")))
row("guide.cu", "guide_kernel<NNFn<32>>", case("guide[nn32]", _guide_kernel("nn32")))

# slice VJPs, slice_grad.cu
_sag = case("slice_apply_grad", _slice_grads(True))
row("slice_grad.cu", "slice_grad_pixel_kernel", _sag)
row("slice_grad.cu", "slice_grad_grid_kernel<12>", _sag)

# coefficient network, cnn.cu and conv_wgmma.cu
row("cnn.cu", "conv2d_nhwc_kernel<1,4>", conv(3, 6, 1, 8))
row("cnn.cu", "conv2d_nhwc_kernel<2,8>", conv(3, 6, 2, 96))
row("cnn.cu", "conv2d_patch_kernel<1,1>", conv(4, 8, 1, 8))
row("cnn.cu", "conv2d_patch_kernel<1,4>", conv(16, 8, 1, 8))
row("cnn.cu", "conv2d_patch_kernel<2,1>", conv(4, 8, 1, 64))
row("cnn.cu", "conv2d_patch_kernel<2,4>", conv(16, 8, 1, 64))
for n in (16, 32, 48, 64, 80, 96, 112, 128):
    row("conv_wgmma.cu", f"conv2d_wgmma_kernel<{n},false>", conv(8, n, 1, 112, tensor_cores=True))
    row("conv_wgmma.cu", f"conv2d_wgmma_kernel<{n},true>", conv(8, n, 1, 96, form="packed", tensor_cores=True))
row("conv_wgmma.cu", "conv_tc_pack_kernel", case("conv_tc_pack", _pack))
row("cnn.cu", "fc_kernel", fc(2, 48, 30))
row("cnn.cu", "fc_cluster_kernel", fc(6, 512, 64))
_coef = coefficients(2)
row("cnn.cu", "fc_chain_kernel", _coef)
row("cnn.cu", "fuse_predict_kernel", _coef)

# coefficient-network VJPs, cnn_grad.cu
_cg = conv_grad(8, 16, 2, 8, 2)
for k in ("conv_dgrad_kernel", "wgrad_partial_kernel<0>", "wgrad_reduce_kernel"):
    row("cnn_grad.cu", k, _cg)
_fg = case("fuse_grad", fuse_grad)
row("cnn_grad.cu", "fuse_dglobal_kernel", _fg)
row("cnn_grad.cu", "fuse_dlocal_kernel", _fg)
row("cnn_grad.cu", "wgrad_partial_kernel<1>", _fg)

# batch norm in training mode, bn_train.cu
_bn = bn(40, 24)
for k in ("stats_partial_kernel", "stats_reduce_kernel", "bn_relu_kernel", "grad_partial_kernel",
          "grad_reduce_kernel", "grad_kernel"):
    row("bn_train.cu", k, _bn)

# guide VJPs, guide_grad.cu and guide_nn_grad.cu
row("guide_grad.cu", "guide_grad_partial_kernel<true,true>", _curves_guide_grad(True, True))
row("guide_grad.cu", "guide_grad_partial_kernel<true,false>", _curves_guide_grad(True, False))
_cgp = _curves_guide_grad(False, True)
row("guide_grad.cu", "guide_grad_partial_kernel<false,true>", _cgp)
row("guide_grad.cu", "guide_grad_reduce_kernel", _cgp)
_nn16, _nn32 = nn_guide_grad(16), nn_guide_grad(32)
row("guide_nn_grad.cu", "stats_partial_kernel", _nn16)
row("guide_nn_grad.cu", "stats_reduce_kernel", _nn16)
row("guide_nn_grad.cu", "vjp_finish_kernel", _nn16)
for F, c in ((16, _nn16), (32, _nn32)):
    row("guide_nn_grad.cu", f"vjp_partial_kernel<{F}>", c)
    row("guide_nn_grad.cu", f"vjp_dx_kernel<{F}>", c)

# resize, network inputs and the frozen pyramid, resize.cu and model.cu
_rz = case("resize_grad", _resize_grad)
row("resize.cu", "resize_bilinear_ac_kernel", _rz)
row("resize.cu", "resize_bilinear_ac_grad_kernel", _rz)
for fmt, dt in ((0, F32), (1, U8), (2, U16)):
    row("resize.cu", f"lowres_nearest_kernel<{fmt}>", lowres(dt, False))
    row("resize.cu", f"lowres_nearest_ragged_kernel<{fmt}>", lowres(dt, True))
_fp8 = frozen_pyramid(U8, U8)
row("resize.cu", "image_to_float_kernel<1>", _fp8)
row("resize.cu", "resize_bilinear_ac_quantize_kernel<1>", _fp8)
row("model.cu", "split_level_rows_kernel", _fp8)
_fp16 = frozen_pyramid(U16, U16)
row("resize.cu", "image_to_float_kernel<2>", _fp16)
row("resize.cu", "resize_bilinear_ac_quantize_kernel<2>", _fp16)

# training batches, train_batch.cu and usm_batch.cu
row("train_batch.cu", "train_batch_kernel", case("train_batch", _train_batch))
_u = case("usm_batch", _usm)
row("usm_batch.cu", "usm_rows_kernel", _u)
row("usm_batch.cu", "usm_target_kernel", _u)
