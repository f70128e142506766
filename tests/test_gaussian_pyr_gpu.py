"""GPU tests of HDRNetGaussianPyr, the Gaussian pyramid with a curves guide at every level.

Forward: the full-resolution stage fed the CUDA coefficients against the float64 chain (resize_f64,
guide_f64, slice_f64); inference_image from every pixel format to every output format against the
quantised float inference; inference_images against per-image calls.  Gradients: every coefficient
variable, every level's six curves variables, fullres_input and lowres_input against the float64
chain, bitwise repeatable.  CLI: a student fits a teacher with other curves guides (better with
--train_guide), 10 + resume + 10 steps equal 20 bitwise, bin/run.py writes the in-memory model's
PNGs, the usm/train_gpyr.sh flags train at 2048², two gloo ranks train what one process trains.
Frozen: FrozenModel and hdrnet_run against the Python model, ragged, the buffer contract and CUDA
graphs."""
import argparse
import json
import os
import subprocess

import cv2
import numpy as np
import pytest
import torch

from hdrnet_b200 import checkpoint, models
from hdrnet_b200.bin import freeze_model as freeze_cli
from hdrnet_b200.bin import run as run_cli
from hdrnet_b200.bin import train
from hdrnet_b200.frozen import FrozenModel
from oracle import cnn_grad_f64 as C
from oracle import guide_f64
from oracle import resize_f64 as R
from oracle import slice_f64
from test_frozen_model_gpu import RUNNER, _contract, _host_img_as_float, _image, _same
from test_pyramid_grad_gpu import coefficient_grads_f64, footprint
from test_train_dp_gpu import COMMON, STEPS, assert_equivalent, run_ranks

pytestmark = pytest.mark.gpu

NAME = "HDRNetGaussianPyr"
PYR = models.HDRNetGaussianPyr
G = "inference/guide"
LEVELS = [f"{G}/level_{l}" for l in range(3)]
U8, U16, F32 = torch.uint8, torch.uint16, torch.float32
FWD_BAR = 1e-5      # the full-resolution stage: max |diff| / max |ref|
GRAD_BAR = 1e-5     # the model's gradients: max |diff| / max |ref|


def report(what, **vals):
    print("MEASURE", what, " ".join(f"{k}={v:.3g}" if isinstance(v, float) else f"{k}={v}"
                                    for k, v in vals.items()), flush=True)


def np_(t):
    return t.detach().cpu().numpy()


def cuda(a, grad=False):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float32))).cuda().requires_grad_(grad)


def curves_guides(rng):
    """Three different curves guides (float32, model shapes), away from the initial curve."""
    w = {}
    for scope in LEVELS:
        w[f"{scope}/ccm"] = np.eye(3) + 0.15 * rng.randn(3, 3)
        w[f"{scope}/ccm_bias"] = 0.1 * rng.randn(3)
        w[f"{scope}/shifts"] = np.sort(rng.rand(1, 1, 3, 16), axis=-1) * 0.9
        w[f"{scope}/slopes"] = np.abs(rng.randn(1, 1, 1, 3, 16)) * 0.3
        w[f"{scope}/channel_mixing/weights"] = rng.rand(1, 1, 3, 1) * 0.6
        w[f"{scope}/channel_mixing/biases"] = np.array([0.1])
    return {k: np.asarray(v, np.float32) for k, v in w.items()}


def model_weights(params, seed, grad=True):
    rng = np.random.RandomState(seed)
    w = models.init_weights(params, seed=seed, model_name=NAME)
    w.update(curves_guides(rng))
    out = {}
    for k, v in w.items():
        if k.endswith("/biases") and k.startswith(C.P):
            v = (0.05 * rng.randn(*v.shape)).astype(np.float32)
        out[k] = torch.from_numpy(v).cuda().requires_grad_(grad)
    return out


def f64_levels(full):
    lv = [np.asarray(full, np.float64)]
    for _ in range(2):
        lv.append(R.resize(lv[-1], lv[-1].shape[1] // 2, lv[-1].shape[2] // 2))
    return lv


def f64_fullres(grid, full, wn):
    """The full-resolution stage in float64: levels, each level's curves guide and slice-apply with its
    three coefficient rows (coarsest rows 0..2), coarse-to-fine upsample-and-add."""
    B, gh, gw, gd = grid.shape[:4]
    lv = f64_levels(full)
    cur = None
    for il in range(3):
        src = 2 - il
        c = np.asarray(grid[:, :, :, :, il * 3:(il + 1) * 3, :], np.float64).reshape(B, gh, gw, gd, 12)
        out = slice_f64.bilateral_slice_apply(c, guide_f64.guide(lv[src], wn, LEVELS[src]), lv[src], True)
        cur = out if il == 0 else R.resize(cur, *lv[src].shape[1:3]) + out
    return cur


TRAIN = dict(models.DEFAULT_PARAMS, model_name=NAME)


# ---- forward ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,cm", [(1, 2048, 2048, 1), (1, 2048, 2048, 4), (4, 512, 512, 1), (2, 301, 455, 1),
                                      (3, 7, 5, 1)], ids=["1x2048", "1x2048_cm4", "4x512", "2x301x455", "3x7x5"])
def test_fullres_stage_against_float64(B, H, W, cm):
    params = dict(TRAIN, channel_multiplier=cm)
    wts = model_weights(params, 11 + cm, grad=False)
    wn = {k: np_(v) for k, v in wts.items()}
    rng = np.random.RandomState(H + W)
    low, full = rng.rand(B, 256, 256, 3), rng.rand(B, H, W, 3)
    p = dict(params, weights=wts)
    with torch.no_grad():
        got = np_(PYR.inference(cuda(low), cuda(full), p))
        grid = np_(PYR._coefficients(cuda(low), p))
    want = f64_fullres(grid, np.asarray(full, np.float32), wn)
    e = float(np.abs(got - want).max() / np.abs(want).max())
    report(f"curves pyramid fullres {B}x{H}x{W} cm={cm}", err_of_range=e)
    assert e <= FWD_BAR, e


@pytest.mark.parametrize("in_dtype", [U8, U16, F32])
def test_inference_image_equals_the_quantised_float_inference(in_dtype):
    params = dict(TRAIN, net_input_size=128, spatial_bin=8)
    p = dict(params, weights={k: np_(v) for k, v in model_weights(params, 3, grad=False).items()})
    img = _image((2, 540, 960, 3), in_dtype, seed=4)
    with torch.no_grad():
        f = PYR.inference(models.lowres_from_image(img, 128), models.image_to_float(img), p)
        for out_dtype, q in ((U8, models.quantize_u8), (U16, models.quantize_u16), (F32, lambda x: x)):
            _same(PYR.inference_image(img, p, out_dtype=out_dtype), q(f), f"{in_dtype}->{out_dtype}")


def test_inference_images_equal_per_image_calls():
    params = dict(TRAIN, net_input_size=128, spatial_bin=8)
    p = dict(params, weights={k: np_(v) for k, v in model_weights(params, 5, grad=False).items()})
    images = [_image(s, U8, seed=i) for i, s in enumerate([(300, 401, 3), (64, 64, 3), (1080, 1920, 3), (9, 17, 3)])]
    for out_dtype in (U8, U16, F32):
        with torch.no_grad():
            got = PYR.inference_images(images, p, out_dtype=out_dtype)
            for i, im in enumerate(images):
                _same(got[i], PYR.inference_image(im[None], p, out_dtype=out_dtype)[0], f"image {i} {out_dtype}")


def test_debug_collections():
    params = dict(TRAIN, net_input_size=64, spatial_bin=8)
    p = dict(params, weights={k: np_(v) for k, v in model_weights(params, 6, grad=False).items()}, debug=True)
    full = cuda(np.random.RandomState(1).rand(1, 96, 128, 3))
    with torch.no_grad():
        out = PYR.inference(cuda(np.random.RandomState(2).rand(1, 64, 64, 3)), full, p)
        fast = PYR.inference(cuda(np.random.RandomState(2).rand(1, 64, 64, 3)), full, dict(p, debug=False))
    dbg = PYR.last_debug
    assert [tuple(g.shape) for g in dbg["guide"]] == [(1, 96, 128), (1, 48, 64), (1, 24, 32)]
    assert [tuple(m.shape) for m in dbg["multiscale"]] == [(1, 96, 128, 3), (1, 48, 64, 3), (1, 24, 32, 3)]
    assert dbg["output"] is out and tuple(dbg["bilateral_coefficients"].shape) == (1, 8, 8, 8, 9, 4)
    for g, m, scope in zip(dbg["guide"], dbg["multiscale"], LEVELS):
        assert np.abs(np_(g) - guide_f64.guide(np_(m), p["weights"], scope)).max() <= 2e-6
    assert float((out - fast).abs().max()) <= 1e-5 * float(fast.abs().max())


# ---- gradients -------------------------------------------------------------------------------------
def near_ties(x, wn, scope, gmap, gd):
    """Pixels where a float32 mask may differ from the float64 one: t within rounding of a curve knot,
    the guide's pre-clip value within rounding of 0 or 1, or the guide within rounding of a depth-cell
    centre of the slice (where its depth weight has its kink)."""
    a, t = guide_f64.preclip(x, wn, scope)
    s = np.asarray(wn[f"{scope}/shifts"], np.float64).reshape(3, 16)
    near = (np.abs(t[..., None] - s) <= 1e-6 * np.maximum(1.0, np.abs(t[..., None]))).any(axis=(-1, -2))
    near |= (np.abs(a) <= 1e-5) | (np.abs(a - 1.0) <= 1e-5)
    z = np.asarray(gmap, np.float64) * gd - 0.5
    return near | (np.abs(z - np.rint(z)) <= 1e-5)


def model_gradients(params, B, S, full_hw, seed):
    """One L2 loss of inference with guide_grad back to every variable, fullres_input and lowres_input;
    returns (wts, grads, masks, the float32 pieces) for the float64 comparison."""
    wts = model_weights(params, seed)
    rng = np.random.RandomState(seed + 1)
    low = rng.rand(B, S, S, 3).astype(np.float32)
    full = rng.rand(B, *full_hw, 3).astype(np.float32)
    p = dict(params, weights=wts, guide_grad=True)
    wn = {k: np_(v) for k, v in wts.items()}
    with torch.no_grad():
        lv = [np_(t) for t in PYR._multiscale_input(cuda(full))]
        guides = [np_(t) for t in PYR._guide([cuda(x) for x in lv], dict(p, guide_grad=False))]
        grid = np_(PYR._coefficients(cuda(low), p))
    gd = params["luma_bins"]
    near = [near_ties(x, wn, scope, g, gd) for x, scope, g in zip(lv, LEVELS, guides)]
    keep = np.where(near[0], 0.0, 1.0).astype(np.float32)
    target = rng.rand(*full.shape).astype(np.float32)
    tl, tf = cuda(low, True), cuda(full, True)
    out = PYR.inference(tl, tf, p)
    loss = (((out - cuda(target)) * cuda(keep[..., None])) ** 2).sum()
    loss.backward()
    grads = {k: np_(v.grad) for k, v in wts.items()}
    grads["fullres_input"], grads["lowres_input"] = np_(tf.grad), np_(tl.grad)
    return wts, wn, grads, dict(low=low, full=full, lv=lv, guides=guides, grid=grid, near=near, keep=keep,
                                target=target, out=np_(out))


def check_model_gradients(params, B, S, full_hw, seed):
    wts, wn, grads, f = model_gradients(params, B, S, full_hw, seed)
    near, lv, guides, grid = f["near"], f["lv"], f["guides"], f["grid"]
    report("curves pyramid near-tie pixels", **{f"level_{l}": int(n.sum()) for l, n in enumerate(near)},
           of=int(near[0].size))
    assert all(n.sum() <= max(2, n.size // 1000) for n in near)
    # float64 backward, coarse-to-fine output reversed: il = 0 is level 2 (rows 0..2) ... il = 2 level 0
    gh, gw, gd = grid.shape[1:4]
    dgrid = np.zeros(grid.shape)
    dcur = 2.0 * (f["out"].astype(np.float64) - f["target"]) * f["keep"][..., None] ** 2
    dx_own, gvs = [None] * 3, [None] * 3
    for il in reversed(range(3)):
        lvl = 2 - il
        c = grid[:, :, :, :, il * 3:(il + 1) * 3, :].reshape(B, gh, gw, gd, 12)
        sv = slice_f64.bilateral_slice_apply_grad(c, guides[lvl], lv[lvl], dcur, True)
        dgrid[:, :, :, :, il * 3:(il + 1) * 3, :] = sv.grid.reshape(B, gh, gw, gd, 3, 4)
        gvs[lvl] = guide_f64.vjp(lv[lvl], sv.guide, wn, LEVELS[lvl])
        dx_own[lvl] = sv.input + gvs[lvl].dinput
        if il > 0:
            dcur = R.resize_vjp(dcur, *lv[lvl + 1].shape[1:3]).din
    dx = dx_own[2]
    for lvl in (1, 0):
        dx = dx_own[lvl] + R.resize_vjp(dx, *lv[lvl].shape[1:3]).din
    want = coefficient_grads_f64(cuda(f["low"]), wts, params, dgrid)

    def rel(got, ref, mask=None):
        d = np.abs(np.asarray(got, np.float64) - ref)
        if mask is not None:
            d = d[~mask]
        return float(d.max() / max(np.abs(ref).max(), 1e-30))

    errs = {}
    for k in C.variable_names(params):
        errs[k.replace(C.P + "/", "")] = e = rel(grads[k], want[k])
        assert e <= GRAD_BAR, f"{k}: {e:.3e}"
    for lvl, scope in enumerate(LEVELS):
        for n in guide_f64.NAMES:
            errs[f"level_{lvl}/{n}"] = e = rel(grads[f"{scope}/{n}"], gvs[lvl].dparams[n])
            assert e <= GRAD_BAR, f"{scope}/{n}: {e:.3e}"
    H0, W0 = full_hw
    affected = near[0] | footprint(near[1], H0, W0) | footprint(footprint(near[2], *lv[1].shape[1:3]), H0, W0)
    errs["fullres_input"] = e = rel(grads["fullres_input"], dx, np.broadcast_to(affected[..., None], dx.shape))
    assert e <= GRAD_BAR, f"fullres_input: {e:.3e}"
    # lowres_input: the first layer's VJP from the float64 gradient of its output
    errs["lowres_input"] = e = lowres_err(wts, params, f["low"], dgrid, grads["lowres_input"])
    assert e <= GRAD_BAR, f"lowres_input: {e:.3e}"
    report(f"curves pyramid grads {B}x{full_hw} cm={params['channel_multiplier']}", masked_fullres=int(affected.sum()),
           worst=max(errs.values()), **{k: v for k, v in errs.items() if "/" not in k or k.startswith("level")})
    return wts, grads


def lowres_err(wts, params, low, dgrid, got):
    """lowres_input's gradient against the float64 network's (cnn_grad_f64.Network) for the float64 dgrid."""
    net = C.Network({k: np_(v) for k, v in wts.items()}, params, n_out=9)
    net.forward(low)
    ref = net.backward(dgrid)["lowres_input"]
    return float(np.abs(np.asarray(got, np.float64) - ref).max() / max(np.abs(ref).max(), 1e-30))


def test_model_gradients_at_the_recipes_size():
    """1 x 2048², network input 256: the size the reference's gpyr recipes train at."""
    check_model_gradients(TRAIN, 1, 256, (2048, 2048), 2)


def test_model_gradients_with_channel_multiplier_4_are_bitwise_repeatable():
    params = dict(TRAIN, channel_multiplier=4)
    _, first = check_model_gradients(params, 4, 256, (512, 512), 5)
    _, _, again, _ = model_gradients(params, 4, 256, (512, 512), 5)
    for k, v in first.items():
        assert np.array_equal(np.asarray(v).view(np.uint32), np.asarray(again[k]).view(np.uint32)), k


def test_forward_is_unchanged_without_gradients():
    """Tensor weights, with or without guide_grad, under no_grad or with nothing requiring grad: the
    guide-fused path's bits."""
    params = dict(TRAIN, net_input_size=64, spatial_bin=8)
    wts = model_weights(params, 4, grad=False)
    rng = np.random.RandomState(5)
    low, full = cuda(rng.rand(2, 64, 64, 3)), cuda(rng.rand(2, 96, 160, 3))
    with torch.no_grad():
        today = PYR.inference(low, full, dict(params, weights={k: np_(v) for k, v in wts.items()}))
        assert torch.equal(PYR.inference(low, full, dict(params, weights=wts, guide_grad=True)), today)
    assert torch.equal(PYR.inference(low, full, dict(params, weights=wts, guide_grad=True)), today)


# ---- the training CLI ----------------------------------------------------------------------------
MODEL = ["--net_input_size", "64", "--spatial_bin", "8", "--output_resolution", "128", "128", "--batch_size", "4",
         "--model_name", NAME, "--nobatch_norm"]
PARAMS = dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8, output_resolution=[128, 128], model_name=NAME)
N_IMAGES, H, W = 6, 144, 176


def teacher_weights(params, seed=1):
    """init_weights with three curves guides far from the initial one (the mean of RGB): each level's
    guide follows mostly one channel, through a curve that rises at twice the initial slope to
    t = 0.5 and then at 0.4, so per pixel it is not a function of the initial guide that the
    coefficients could absorb."""
    w = models.init_weights(params, seed=seed, model_name=NAME)
    ccm = np.array([[0.2, 0.7, 0.1], [0.1, 0.2, 0.7], [0.7, 0.1, 0.2]])
    for l, scope in enumerate(LEVELS):
        slopes = np.zeros((1, 1, 1, 3, 16))
        slopes[..., 0], slopes[..., 8] = 2.0, -1.6          # knots 0 and 0.5 of the initial linspace
        w[f"{scope}/ccm"] = np.roll(ccm, l, axis=1).astype(np.float32)
        w[f"{scope}/slopes"] = slopes.astype(np.float32)
        w[f"{scope}/channel_mixing/weights"] = np.roll([0.8, 0.1, 0.1], l).reshape(1, 1, 3, 1).astype(np.float32)
    return w


def render(root, n, h, w, teacher, seed, targets=True):
    os.makedirs(root / "input", exist_ok=True)
    os.makedirs(root / "output", exist_ok=True)
    rng = np.random.RandomState(seed)
    names = []
    for i in range(n):
        yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
        base = np.stack([np.sin(3 * xx + i), np.cos(2 * yy - i), xx * yy], axis=2) * 0.4 + 0.5
        im8 = (np.clip(base + 0.1 * rng.randn(h, w, 3), 0, 1) * 255).astype(np.uint8)
        name = f"im{i:02d}.png"
        assert cv2.imwrite(str(root / "input" / name), im8[:, :, ::-1])
        if targets:
            with torch.no_grad():
                out = PYR.inference_image(torch.from_numpy(im8[None]).cuda(), teacher,
                                          out_dtype=torch.float32)[0].cpu().numpy()
            assert cv2.imwrite(str(root / "output" / name),
                               np.rint(np.clip(out, 0, 1) * 65535).astype(np.uint16)[:, :, ::-1])
        names.append(name)
    (root / "filelist.txt").write_text("\n".join(names) + "\n")
    return root


@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    return render(tmp_path_factory.mktemp("gpyr_pairs"), N_IMAGES, H, W,
                  dict(PARAMS, weights=teacher_weights(PARAMS)), 3)


def trainer(ckpt, data, *flags, model=MODEL):
    parser = train.build_parser()
    args = parser.parse_args([str(ckpt), str(data), *model, "--summary_interval", "0",
                              "--checkpoint_interval", "100000", *flags])
    train.check_data_flags(parser, args)
    params = train.model_params(parser, args)
    train.refuse_untrainable(params, args.train_guide, args.guide_batch_stats, args.coefficient_batch_stats)
    return train.Trainer(args, params)


def logged_losses(ckpt_dir):
    return [json.loads(line)["loss"] for line in open(ckpt_dir / "train_log.jsonl") if '"loss"' in line]


def test_student_fits_the_teacher_better_with_the_guides_trained(dataset, tmp_path):
    """200 CLI steps each way.  Measured on an H100: the loss fell 55x with the guides fixed and
    54.7x with them trained, to 0.0707 and 0.0702; the coefficient network absorbs most of the other
    guides, so the trained guides' gain is small (0.7 %), and the bar asks only that it is a gain."""
    final = {}
    for guide in (False, True):
        flags = ["--seed", "5", "--learning_rate", "2e-3", "--max_steps", "200"] + (["--train_guide"] if guide else [])
        trainer(tmp_path / f"fit_{guide}", dataset, *flags).run()
        losses = logged_losses(tmp_path / f"fit_{guide}")
        assert np.isfinite(losses).all()
        first, last = float(np.mean(losses[:3])), float(np.mean(losses[-10:]))
        final[guide] = (first, last)
        report(f"curves pyramid CLI fit train_guide={guide}", first3=first, last10=last, factor=first / last)
    assert final[True][1] * 10 <= final[True][0]
    assert final[True][1] < final[False][1], final


def test_trains_resumes_bitwise_and_run_reproduces_it(dataset, tmp_path):
    flags = ["--fliplr", "--rotate", "--seed", "5", "--learning_rate", "1e-3", "--train_guide"]
    straight = trainer(tmp_path / "straight", dataset, *flags, "--max_steps", "20")
    straight.run()
    trainer(tmp_path / "resumed", dataset, *flags, "--max_steps", "10").run()
    t = trainer(tmp_path / "resumed", dataset, *flags, "--max_steps", "20")
    assert t.step == 10
    t.run()
    a = checkpoint.read_tf_checkpoint(str(tmp_path / "straight"))
    b = checkpoint.read_tf_checkpoint(str(tmp_path / "resumed"))
    assert int(a["global_step"]) == int(b["global_step"]) == 20
    init = models.init_weights(PARAMS, seed=5, model_name=NAME)
    guide = [k for k in init if k.startswith(train.GUIDE)]
    assert len(guide) == 18
    for k in guide:
        assert not np.array_equal(a[k], init[k]), f"{k} did not move"
        assert k + "/Adam" in a and np.abs(a[k + "/Adam_1"]).sum() > 0, k
    keys = [k for k in a if k.startswith("inference/")]
    assert sorted(keys) == sorted(k for k in b if k.startswith("inference/"))
    for k in keys:
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), k

    names = sorted(os.listdir(dataset / "input"))
    for bits, dtype in ((8, U8), (16, U16)):
        for batch in (1, 3):
            out_dir = tmp_path / f"out{bits}_{batch}"
            run_cli.main(argparse.Namespace(checkpoint_dir=str(tmp_path / "straight"), input=str(dataset / "input"),
                                            output=str(out_dir), lowres_input=None, hdrp=False, debug=False,
                                            limit=None, output_bit_depth=bits, batch_size=batch))
            for name in names:
                im8 = cv2.imread(str(dataset / "input" / name), -1)[:, :, ::-1]
                with torch.no_grad():
                    want = PYR.inference_image(torch.from_numpy(np.ascontiguousarray(im8[None])).cuda(), straight.p,
                                               out_dtype=dtype)[0].cpu().numpy()
                assert np.array_equal(cv2.imread(str(out_dir / name), -1)[:, :, ::-1], want), (bits, batch, name)
    # --debug: the reference's pictures, one guide and one level picture per level
    out_dir = tmp_path / "debug"
    run_cli.main(argparse.Namespace(checkpoint_dir=str(tmp_path / "straight"), input=str(dataset / "input"),
                                    output=str(out_dir), lowres_input=None, hdrp=False, debug=True, limit=1))
    stem = os.path.splitext(names[0])[0]
    for suffix in (".png", "_guide.npy", "_coefficients.npy", "_coeffs.png", "_guide_0.png", "_guide_1.png",
                   "_guide_2.png", "_ms_0.png", "_ms_1.png", "_ms_2.png"):
        assert os.path.exists(out_dir / (stem + suffix)), stem + suffix
    assert np.load(out_dir / (stem + "_coefficients.npy")).shape == (8, 8, 8, 9, 4)


def test_the_usm_recipe_trains_at_2048(tmp_path):
    """scripts/usm/train_gpyr.sh's flags: batch 1 at 2048², UnsharpMaskDataPipeline, --nobatch_norm."""
    data = render(tmp_path / "big", 2, 2064, 2080, None, 4, targets=False)
    model = ["--learning_rate", "1e-4", "--batch_size", "1", "--model_name", NAME, "--data_pipeline",
             "UnsharpMaskDataPipeline", "--blur_sigma", "4", "--sharpen", "2", "--nobatch_norm",
             "--output_resolution", "2048", "2048"]
    trainer(tmp_path / "ckpt", data, "--max_steps", "4", model=model).run()
    losses = logged_losses(tmp_path / "ckpt")
    report("curves pyramid usm 2048^2 losses", first=losses[0], last=losses[-1])
    assert len(losses) == 4 and np.isfinite(losses).all()


def test_two_ranks_on_one_card_train_what_one_process_trains(tmp_path, dataset):
    argv = [str(dataset), *COMMON, "--model_name", NAME, "--max_steps", str(STEPS)]
    one, many = tmp_path / "one", tmp_path / "ranks"
    trainer(one, *argv, model=[]).run()
    digests = run_ranks([str(many), *argv])
    assert len(digests[0]) == STEPS and all(d == digests[0] for d in digests), "ranks drifted apart"
    assert len(set(digests[0])) == STEPS
    a, _ = assert_equivalent(str(many), str(one), f"{NAME} 2 ranks (gloo)")
    assert sum(k.startswith(LEVELS[2]) and k.endswith("/Adam") for k in a) == 6


# ---- the frozen model ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def frozen(tmp_path_factory):
    params = dict(TRAIN, channel_multiplier=4)
    w = {k: np_(v) for k, v in model_weights(params, 7, grad=False).items()}
    params["weights"] = w
    path = tmp_path_factory.mktemp("frozen") / "gpyr.hdrnet"
    checkpoint.freeze_model(w, params, str(path))
    model = FrozenModel(str(path))
    assert model.model_name == NAME and model.guide_width == 16
    yield params, model
    model.close()


@pytest.mark.parametrize("B,S", [(1, 2048), (4, 512)])
@pytest.mark.parametrize("in_dtype", [U8, U16, F32])
def test_frozen_model_equals_inference(frozen, B, S, in_dtype):
    params, model = frozen
    img = _image((B, S, S, 3), in_dtype, seed=S)
    with torch.no_grad():
        if in_dtype == F32:
            wants = {d: PYR.inference_image(img, params, out_dtype=d) for d in (U8, U16, F32)}
        else:
            f = PYR.inference(models.lowres_from_image(img, params["net_input_size"]), _host_img_as_float(img), params)
            wants = {U8: models.quantize_u8(f), U16: models.quantize_u16(f), F32: f}
    for d, want in wants.items():
        _same(model(img, out_dtype=d), want, f"{B}x{S}^2 {in_dtype}->{d}")


def test_ragged_run_images_equals_inference_images(frozen):
    params, model = frozen
    images = [_image(s, F32, seed=i) for i, s in enumerate([(300, 401, 3), (1080, 1920, 3), (64, 80, 3)])]
    outs = [torch.empty(im.shape, dtype=U16, device="cuda") for im in images]
    ws = torch.empty(model.workspace_bytes_images(images, U16), dtype=U8, device="cuda")
    model.run_images(images, outs, ws)
    with torch.no_grad():
        want = PYR.inference_images(images, params, out_dtype=U16)
    for i, (o, w_) in enumerate(zip(outs, want)):
        _same(o, w_, f"ragged image {i}")


@pytest.mark.parametrize("out_dtype", [U8, U16, F32])
def test_buffer_contract(frozen, out_dtype):
    params, model = frozen
    img = _image((2, 1080, 1920, 3), U8, seed=3)
    a = _contract(model, img, out_dtype, 0x00)
    _same(a, _contract(model, img, out_dtype, 0xFF), "two fills")
    with torch.no_grad():
        f = PYR.inference(models.lowres_from_image(img, params["net_input_size"]), _host_img_as_float(img), params)
    _same(a, {U8: models.quantize_u8, U16: models.quantize_u16, F32: lambda x: x}[out_dtype](f), "fully written")
    B, H_, W_, _ = img.shape
    ws = torch.full((model.workspace_bytes(B, H_, W_, U8, out_dtype) - 1,), 0x5A, dtype=U8, device="cuda")
    out_bytes = torch.zeros(B * H_ * W_ * 3 * out_dtype.itemsize, dtype=U8, device="cuda")
    with pytest.raises(ValueError, match="invalid dimension"):
        model.run(img, out_bytes.view(out_dtype).view(B, H_, W_, 3), ws)
    torch.cuda.synchronize()
    assert bool((ws == 0x5A).all()) and not bool(out_bytes.any())


@pytest.mark.parametrize("H_,W_", [(1080, 1920), (2160, 3840)])
def test_cuda_graph_replay(frozen, H_, W_):
    _, model = frozen
    static_in = _image((1, H_, W_, 3), U8, seed=0)
    out = torch.empty((1, H_, W_, 3), dtype=U8, device="cuda")
    ws = torch.empty(model.workspace_bytes(1, H_, W_), dtype=U8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        model.run(static_in, out, ws)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        model.run(static_in, out, ws)
    for seed in (1, 2, 3):
        frame = _image((1, H_, W_, 3), U8, seed=seed)
        static_in.copy_(frame)
        graph.replay()
        _same(out, model(frame), f"replay {seed}")


@pytest.fixture(scope="module")
def trained(tmp_path_factory, dataset):
    ckpt = tmp_path_factory.mktemp("gpyr_ckpt")
    trainer(ckpt, dataset, "--max_steps", "5", "--train_guide", "--seed", "2").run()
    return ckpt


@pytest.mark.parametrize("bits", [8, 16])
def test_hdrnet_run_writes_what_run_py_writes(trained, tmp_path, bits):
    """hdrnet_run converts integer pixels with the bit-exact img_as_float, bin/run.py through torch
    (DESIGN.md row f-11): the runner equals the model on the host's img_as_float bit for bit, and
    bin/run.py's PNG within one code."""
    frozen_path = freeze_cli.main(freeze_cli.build_parser().parse_args([str(trained), "--output",
                                                                        str(tmp_path / "model.hdrnet")]))
    rng = np.random.RandomState(bits)
    im = rng.randint(0, 65536, (120, 200, 3)).astype(np.uint16) if bits == 16 else \
        rng.randint(0, 256, (120, 200, 3)).astype(np.uint8)
    np.save(tmp_path / "im.npy", im)
    assert cv2.imwrite(str(tmp_path / "im.png"), im[:, :, ::-1])
    out_dir = tmp_path / "out"
    os.makedirs(out_dir)
    proc = subprocess.run([RUNNER, "--checkpoint_path", frozen_path, "--input_path", str(tmp_path / "im.npy"),
                           "--output_directory", str(out_dir), "--burn_iters", "1", "--iters", "3",
                           "--output_bit_depth", str(bits)], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    got = np.load(out_dir / "model.npy")
    rep = json.loads((out_dir / "model.json").read_text())
    assert rep["model"] == NAME and (rep["height"], rep["width"]) == (120, 200)
    run_dir = tmp_path / "run_py"
    run_cli.main(argparse.Namespace(checkpoint_dir=str(trained), input=str(tmp_path / "im.png"), output=str(run_dir),
                                    lowres_input=None, hdrp=False, debug=False, limit=None, output_bit_depth=bits))
    want = cv2.imread(str(run_dir / "im.png"), -1)[:, :, ::-1]
    params, weights = run_cli.load_checkpoint(str(trained))
    img = torch.from_numpy(im[None]).cuda()
    with torch.no_grad():
        f = PYR.inference(models.lowres_from_image(img, params["net_input_size"]), _host_img_as_float(img),
                          dict(params, weights=weights))
    exact = (models.quantize_u8(f) if bits == 8 else models.quantize_u16(f))[0].cpu().numpy()
    d = np.abs(got.astype(np.int64) - want.astype(np.int64))
    report(f"hdrnet_run vs bin/run.py {bits}-bit", codes_differing=int((d > 0).sum()), of=int(d.size))
    assert got.dtype == want.dtype and np.array_equal(got, exact)
    assert d.max() <= 1
