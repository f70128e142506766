"""Ragged batches on an H100: images of different sizes in one call.  Each image of the ragged
network input, the ragged fused slice-apply and the ragged model calls is compared, bit for bit, with
the single-image call on that image (and its grid row): every format pair, both guides at F = 16
and 32, mixed sizes from 1 x 1 to 4032 x 3024 in both orientations, unaligned bases, the
texture-assisted single-image forms, past 2^31 bytes and across the per-launch image cap; the
buffer contract; FrozenModel, CUDA-graph replay and run.py --batch_size."""
import os

import cv2
import numpy as np
import pytest
import torch

from hdrnet_b200 import _lib, checkpoint, models
from hdrnet_b200.bin import run as run_cli
from hdrnet_b200.frozen import FrozenModel
from oracle import slice_f64

pytestmark = pytest.mark.gpu

U8, U16, F32 = torch.uint8, torch.uint16, torch.float32
DTYPES = {"u8": U8, "u16": U16, "f32": F32}
GH, GW, GD = 16, 16, 8
# 4032 x 3024 in both orientations, 1080p, tiny and odd widths (W % 16 != 0), narrow and wide
MIXED = [(3024, 4032), (4032, 3024), (1080, 1920), (7, 5), (1, 1), (37, 250), (300, 17), (13, 500), (64, 1104)]


def _image(shape, dtype, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if dtype == F32:
        return torch.rand(shape, generator=g, device="cuda")
    top = 256 if dtype == U8 else 65536
    return torch.randint(0, top, shape, generator=g, device="cuda", dtype=torch.int32).to(dtype)


def _coeffs(B, seed=1, gh=GH, gw=GW, gd=GD):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randn((B, gh, gw, gd, 3, 4), generator=g, device="cuda") * 0.3
    c[..., 0, 0] += 1.0
    c[..., 1, 1] += 1.0
    c[..., 2, 2] += 1.0
    return c


def _guide(kind, seed=3):
    rng = np.random.RandomState(seed)
    if kind == "curves":
        p = dict(models.DEFAULT_PARAMS, model_name="HDRNetCurves")
        return models._CurvesGuide.from_weights(models.init_weights(p, seed=seed, model_name="HDRNetCurves"))
    F = 16 if kind == "nn16" else 32
    return models._NNGuide((rng.randn(3, F) * 0.5).astype(np.float32), (rng.randn(F) * 0.1).astype(np.float32),
                           (rng.randn(F) * 0.3 / F ** 0.5).astype(np.float32), np.float32([0.5]))


def _bits(t):
    return t.view(torch.int16) if t.dtype == U16 else t.view(torch.int32) if t.dtype == F32 else t


def _same(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, what
    assert torch.equal(_bits(a), _bits(b)), f"{what}: {int((a.double() != b.double()).sum())} values differ"


def _single(coeffs_row, x, guide, out_dtype):
    """The single-image fused call on one image and its grid row, lending the slab workspace as the
    model path does (so 12 MP images take the texture-assisted form)."""
    return models._slice_apply_fused(coeffs_row[None].contiguous(), x[None], guide, out_dtype, False, True)[0][0]


def _f32_reordered(x, coeffs_row):
    """float32 -> float32 images the row kernels do not take at W >= 64: the single-image call runs the
    guide kernel and the any-shape row kernel, whose apply sums in another order (DESIGN.md row f-13)."""
    W = x.shape[1]
    return x.dtype == F32 and W >= 64 and not models._fused_row_kernel_takes(W, x, x, coeffs_row)


def _check_ragged(images, coeffs, guide, out_dtype, what):
    outs = models._slice_apply_fused_ragged(coeffs.reshape(len(images), GH, GW, GD, 12), images, guide, out_dtype)
    for i, (x, o) in enumerate(zip(images, outs)):
        want = _single(coeffs[i], x, guide, out_dtype)
        if out_dtype == F32 and _f32_reordered(x, coeffs[i]):
            torch.testing.assert_close(o, want, rtol=0, atol=1e-5, msg=f"{what} image {i} {tuple(x.shape)}")
        else:
            _same(o, want, f"{what} image {i} {tuple(x.shape)}")


@pytest.mark.parametrize("dt", list(DTYPES))
def test_ragged_lowres_equals_single(dt):
    sizes = [(1, 1), (7, 5), (900, 31), (29, 1200), (101, 203), (3024, 4032)]
    ims = [_image((h, w, 3), DTYPES[dt], seed=i) for i, (h, w) in enumerate(sizes)]
    low = models.lowres_from_images(ims, 256)
    for i, im in enumerate(ims):
        _same(low[i], models.lowres_from_image(im[None], 256)[0], f"{dt} {sizes[i]}")


@pytest.mark.parametrize("out_name", list(DTYPES))
@pytest.mark.parametrize("in_name", list(DTYPES))
@pytest.mark.parametrize("kind", ["curves", "nn16", "nn32"])
def test_ragged_fused_equals_single(kind, in_name, out_name):
    ims = [_image((h, w, 3), DTYPES[in_name], seed=i) for i, (h, w) in enumerate(MIXED)]
    _check_ragged(ims, _coeffs(len(ims)), _guide(kind), DTYPES[out_name], f"{kind} {in_name}->{out_name}")


def _at_offset(shape, dtype, off, src):
    n = int(np.prod(shape)) * src.element_size()
    buf = torch.zeros(n + 32, dtype=U8, device="cuda")
    v = buf[off:off + n].view(dtype).view(shape)
    v.copy_(src)
    return v


@pytest.mark.parametrize("pair", ["u8-u8", "u16-u16", "u8-u16", "f32-u8"])
@pytest.mark.parametrize("kind", ["curves", "nn16"])
def test_ragged_fused_at_unaligned_offsets(kind, pair):
    i_n, o_n = pair.split("-")
    offs = (4, 8, 12) if i_n == "f32" else (2, 4, 6)
    shapes = [(40, 1024), (33, 777), (9, 256)]
    ims = [_at_offset((h, w, 3), DTYPES[i_n], off, _image((h, w, 3), DTYPES[i_n], seed=h))
           for (h, w), off in zip(shapes, offs)]
    _check_ragged(ims, _coeffs(len(ims)), _guide(kind), DTYPES[o_n], f"{kind} {pair} offsets {offs}")


def test_ragged_fused_against_float64_oracle():
    guide = _guide("curves")
    shapes = [(31, 257), (64, 128), (5, 3)]
    ims = [_image((h, w, 3), F32, seed=i) for i, (h, w) in enumerate(shapes)]
    coeffs = _coeffs(len(ims))
    outs = models._slice_apply_fused_ragged(coeffs.reshape(len(ims), GH, GW, GD, 12), ims, guide, F32)
    for i, (x, o) in enumerate(zip(ims, outs)):
        g = guide.run(x[None].contiguous())
        want = slice_f64.bilateral_slice_apply(coeffs[i:i + 1].reshape(1, GH, GW, GD, 12).double().cpu().numpy(),
                                               g.double().cpu().numpy(), x[None].double().cpu().numpy(), True)
        err = np.abs(o.double().cpu().numpy() - want[0]).max()
        assert err <= 1e-5, f"{shapes[i]}: {err}"


def _prep(name, seed=5, **over):
    params = dict(models.DEFAULT_PARAMS, model_name=name, **over)
    params["weights"] = models.init_weights(params, seed=seed, model_name=name)
    return getattr(models, name), params


MODELS = ["HDRNetCurves", "HDRNetPointwiseNNGuide", "HDRNetGaussianPyrNN"]


@pytest.mark.parametrize("with_lowres", [False, True])
@pytest.mark.parametrize("name", MODELS)
def test_inference_images_equals_fullres_of_the_stacked_grid(name, with_lowres):
    cls, params = _prep(name)
    ims = [_image((h, w, 3), U8, seed=i) for i, (h, w) in enumerate([(120, 200), (200, 120), (7, 9), (64, 1104)])]
    lows = [_image((50 + i, 60, 3), U8, seed=10 + i) for i in range(len(ims))] if with_lowres else None
    with torch.no_grad():
        outs = cls.inference_images(ims, params, lowres_images=lows)
        low = torch.cat([models.lowres_from_image(x[None], 256) for x in (lows or ims)])
        _same(models.lowres_from_images(lows or ims, 256), low, "ragged network input")
        coeffs = cls._coefficients(low, params, False)
        for i, x in enumerate(ims):
            if name == "HDRNetGaussianPyrNN":
                want = models.quantize_u8(cls._output(cls._multiscale_input(models.image_to_float(x[None])), None,
                                                      coeffs[i:i + 1], params))[0]
            else:
                want = cls._fullres(coeffs[i:i + 1].contiguous(), x[None], params, U8)[0]
            _same(outs[i], want, f"{name} image {i}")


@pytest.mark.parametrize("out_dtype", [U8, U16])
@pytest.mark.parametrize("name", MODELS)
def test_same_size_list_equals_stacked_inference_image(name, out_dtype):
    cls, params = _prep(name)
    batch = _image((4, 96, 256, 3), U16, seed=2)
    with torch.no_grad():
        want = cls.inference_image(batch, params, out_dtype=out_dtype)
        outs = cls.inference_images(list(batch.unbind(0)), params, out_dtype=out_dtype)
    for i in range(4):
        _same(outs[i], want[i], f"{name} image {i}")


# ---- buffer contract -----------------------------------------------------------------------------
def _packed(shapes, dtype, fill, gap=64):
    """Views [H_i, W_i, 3] into one buffer with `gap` guard bytes before, between and after them."""
    es = torch.empty((), dtype=dtype).element_size()
    sizes = [h * w * 3 * es for h, w in shapes]
    buf = torch.full((sum(sizes) + gap * (len(shapes) + 1),), fill, dtype=U8, device="cuda")
    views, spans, off = [], [], gap
    for (h, w), n in zip(shapes, sizes):
        views.append(buf[off:off + n].view(dtype).view(h, w, 3))
        spans.append((off, off + n))
        off += n + gap
    return buf, views, spans


def _guards_intact(buf, spans, fill):
    mask = torch.ones(buf.numel(), dtype=torch.bool, device=buf.device)
    for a, b in spans:
        mask[a:b] = False
    return bool((buf[mask] == fill).all())


@pytest.mark.parametrize("out_dtype", [U8, U16, F32])
@pytest.mark.parametrize("name", ["HDRNetCurves", "HDRNetPointwiseNNGuide", "HDRNetGaussianPyrNN"])
def test_model_buffer_contract(tmp_path, name, out_dtype):
    _, params = _prep(name)
    path = tmp_path / "m.hdrnet"
    checkpoint.freeze_model(params["weights"], params, str(path))
    shapes = [(33, 250), (120, 1024), (9, 13), (256, 96)]
    with FrozenModel(str(path)) as model:
        src = [_image((h, w, 3), U8, seed=i) for i, (h, w) in enumerate(shapes)]
        ibuf, ims, _ = _packed(shapes, U8, 0x11)
        for v, s in zip(ims, src):
            v.copy_(s)
        before = ibuf.clone()
        nbytes = model.workspace_bytes_images(ims, out_dtype)
        runs = []
        for fill in (0xFF, 0x5A):
            obuf, outs, spans = _packed(shapes, out_dtype, fill)
            wbuf = torch.full((nbytes + 128,), fill, dtype=U8, device="cuda")
            model.run_images(ims, outs, wbuf[64:64 + nbytes])
            torch.cuda.synchronize()
            assert _guards_intact(obuf, spans, fill), f"fill {fill:#x}: a write outside the outputs"
            assert bool((wbuf[:64] == fill).all()) and bool((wbuf[64 + nbytes:] == fill).all()), "workspace guards"
            assert torch.equal(ibuf, before), "the inputs changed"
            runs.append([o.clone() for o in outs])
        for a, b in zip(*runs):
            _same(a, b, "two fills")
            if out_dtype == F32:
                assert bool(torch.isfinite(a).all())
        # one byte short: refused, nothing written
        obuf, outs, spans = _packed(shapes, out_dtype, 0x77)
        with pytest.raises(ValueError, match="invalid dimension"):
            model.run_images(ims, outs, torch.empty(nbytes - 1, dtype=U8, device="cuda"))
        torch.cuda.synchronize()
        assert bool((obuf == 0x77).all())


# ---- large and capture ---------------------------------------------------------------------------
def test_past_2_31_bytes():
    """45 x 4K uint16 in and out: 2.2 GB each side; the first and last images and those straddling
    a multiple of 2^31 bytes equal their own calls."""
    n, H, W = 45, 2160, 3840
    img_bytes = H * W * 6
    src = torch.empty((n, H, W, 3), dtype=U16, device="cuda")
    for i in range(n):
        src[i].copy_(_image((H, W, 3), U16, seed=i) if i in (0, n - 1) else src[0])
    src[1:n - 1].random_(0, 65536)
    ims = list(src.unbind(0))
    coeffs = _coeffs(n)
    guide = _guide("curves")
    outs_buf = torch.empty_like(src)
    outs = list(outs_buf.unbind(0))
    lib = _lib.load()
    rc = lib.hdrnet_slice_apply_curves_ragged_px_ws(coeffs.data_ptr(), _lib.image_descs(ims, outs), n, _lib.PX_U16,
                                                    _lib.PX_U16, GH, GW, GD, *guide.args, None, 0,
                                                    torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "ragged")
    straddle = {i for i in range(n) if (i * img_bytes) // 2 ** 31 != ((i + 1) * img_bytes - 1) // 2 ** 31}
    for i in sorted({0, n - 1} | straddle):
        _same(outs[i], _single(coeffs[i], ims[i], guide, U16), f"image {i}")
    del src, outs_buf


def test_cap_split():
    n = _lib.RAGGED_MAX_IMAGES + 3
    rng = np.random.RandomState(0)
    ims = [_image((int(rng.randint(1, 40)), int(rng.randint(1, 300)), 3), U8, seed=i) for i in range(n)]
    coeffs = _coeffs(n)
    _check_ragged(ims, coeffs, _guide("nn16"), U8, "cap + 3")
    low = models.lowres_from_images(ims, 64)
    for i in (0, _lib.RAGGED_MAX_IMAGES - 1, _lib.RAGGED_MAX_IMAGES, n - 1):
        _same(low[i], models.lowres_from_image(ims[i][None], 64)[0], f"lowres {i}")


@pytest.mark.parametrize("name", MODELS)
def test_frozen_model_ragged_equals_inference_images(tmp_path, name):
    _, params = _prep(name)
    cls = getattr(models, name)
    path = tmp_path / "m.hdrnet"
    checkpoint.freeze_model(params["weights"], params, str(path))
    # the pyramid from float32 pixels: from integer pixels the C path converts with the bit-exact
    # img_as_float where inference_images divides through torch (DESIGN.md row f-11)
    dt = F32 if name == "HDRNetGaussianPyrNN" else U8
    ims = [_image((h, w, 3), dt, seed=i) for i, (h, w) in enumerate([(300, 401), (401, 300), (1080, 1920), (8, 8)])]
    with FrozenModel(str(path)) as model, torch.no_grad():
        for out_dtype in (U8, U16):
            want = cls.inference_images(ims, params, out_dtype=out_dtype)
            got = model(ims, out_dtype=out_dtype)
            for i in range(len(ims)):
                _same(got[i], want[i], f"{name} {out_dtype} image {i}")


def test_graph_replay_of_a_mixed_set(tmp_path):
    _, params = _prep("HDRNetCurves")
    path = tmp_path / "m.hdrnet"
    checkpoint.freeze_model(params["weights"], params, str(path))
    shapes = [(3024, 4032), (4032, 3024), (7, 5), (1080, 1920)]
    with FrozenModel(str(path)) as model:
        ims = [torch.zeros((h, w, 3), dtype=U8, device="cuda") for h, w in shapes]
        outs = [torch.empty_like(x) for x in ims]
        ws = torch.empty(model.workspace_bytes_images(ims), dtype=U8, device="cuda")
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            model.run_images(ims, outs, ws)      # warm-up outside the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            model.run_images(ims, outs, ws)
        for seed in (1, 2):
            for i, x in enumerate(ims):
                x.copy_(_image(x.shape, U8, seed=seed * 10 + i))
            graph.replay()
            torch.cuda.synchronize()
            want = model([x.clone() for x in ims])
            for i in range(len(ims)):
                _same(outs[i], want[i], f"replay {seed} image {i}")


@pytest.mark.parametrize("bits", [8, 16])
def test_run_cli_batch_size(tmp_path, bits):
    """--batch_size 4 writes every file that --batch_size 1 writes, each the result of inference_images
    on its group, bit for bit.  Against --batch_size 1 the pixels agree to a few code values only: the
    coefficient network chooses some layers' kernels by batch size (the packed tensor-core conv from 64
    output tiles), so a grid computed in a batch of four differs from the batch-of-one grid in its
    last bits (DESIGN.md row f-13)."""
    cls, params = _prep("HDRNetCurves")
    ckpt = tmp_path / "ckpt"
    run_cli.save_checkpoint(str(ckpt), params, params["weights"])
    src = tmp_path / "in"
    src.mkdir()
    rng = np.random.RandomState(0)
    shapes = [(120, 160), (160, 120), (33, 250), (64, 64), (7, 5), (90, 128)]
    for i, (h, w) in enumerate(shapes):
        cv2.imwrite(str(src / f"im{i}.png"), rng.randint(0, 256, (h, w, 3)).astype(np.uint8))
    got = {}
    for n in (1, 4):
        out = tmp_path / f"out{n}"
        args = run_cli.build_parser().parse_args([str(ckpt), str(src), str(out), "--batch_size", str(n),
                                                  "--output_bit_depth", str(bits)])
        run_cli.main(args)
        got[n] = {f: cv2.imread(str(out / f), -1) for f in sorted(os.listdir(out))}
    assert got[1].keys() == got[4].keys() and len(got[1]) == 6
    dt = U8 if bits == 8 else U16
    names = sorted(got[1])
    for g0 in (0, 4):
        group = names[g0:g0 + 4]
        ims = [torch.from_numpy(np.ascontiguousarray(cv2.imread(str(src / f), -1)[:, :, ::-1])).cuda() for f in group]
        with torch.no_grad():
            want = cls.inference_images(ims, params, out_dtype=dt)
        for f, w in zip(group, want):
            assert np.array_equal(got[4][f][:, :, ::-1], w.cpu().numpy()), f
    tol = 3 if bits == 8 else 3 * 257
    for f in names:
        d = np.abs(got[1][f].astype(np.int64) - got[4][f].astype(np.int64)).max()
        assert d <= tol, f"{f}: {d} code values apart"
