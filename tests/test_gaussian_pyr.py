"""CPU tests of HDRNetGaussianPyr, the Gaussian pyramid with a curves guide at every level: its
variables, the curves pyramid in the numpy restatement against the torch one (gaussian_pyr_f64), the training
CLI's accepted and refused flag sets (refusals before any data is read), the model's CPU refusals,
and the frozen model file (kind 3) against models._Prepared, with the C side's validation."""
import ctypes

import numpy as np
import pytest
import torch

import oracle
from hdrnet_b200 import _lib, checkpoint, frozen, models
from gaussian_pyr_f64 import inference as pyr_f64
from hdrnet_b200.bin import train
from oracle import model_np as M
from oracle import model_torch as T

NAME = "HDRNetGaussianPyr"
PYR = models.HDRNetGaussianPyr
G = "inference/guide"
LEVELS = [f"{G}/level_{l}" for l in range(3)]
CURVES = ("ccm", "ccm_bias", "shifts", "slopes", "channel_mixing/weights", "channel_mixing/biases")
SHAPES = {"ccm": (3, 3), "ccm_bias": (3,), "shifts": (1, 1, 3, 16), "slopes": (1, 1, 1, 3, 16),
          "channel_mixing/weights": (1, 1, 3, 1), "channel_mixing/biases": (1,)}


def test_public_surface():
    assert models.__all__[:4] == ["HDRNetCurves", "HDRNetPointwiseNNGuide", "HDRNetGaussianPyrNN", NAME]
    assert issubclass(PYR, models.HDRNetCurves) and not issubclass(PYR, models.HDRNetPointwiseNNGuide)
    assert (PYR.n_scales(), PYR.n_out(), PYR.n_in()) == (3, 9, 4)
    assert (models.HDRNetGaussianPyrNN.n_out(), models.HDRNetGaussianPyrNN._nn_guide) == (9, "pyramid")


# ---- init_weights --------------------------------------------------------------------------------
def test_init_weights_names_shapes_and_per_level_jitter():
    p = dict(models.DEFAULT_PARAMS, model_name=NAME)
    w = models.init_weights(p, seed=4)
    nn = models.init_weights(p, seed=4, model_name="HDRNetGaussianPyrNN")
    coeff = {k for k in nn if k.startswith("inference/coefficients/")}
    assert set(w) == coeff | {f"{s}/{n}" for s in LEVELS for n in CURVES}
    for k in coeff:                      # the coefficient network is the NN pyramid's, draw for draw
        assert w[k].tobytes() == nn[k].tobytes(), k
    assert w["inference/coefficients/prediction/conv1/weights"].shape == (1, 1, 64, 8 * 9 * 4)
    curves = models.init_weights(dict(models.DEFAULT_PARAMS), seed=4)
    jitters = []
    for s in LEVELS:
        for n in CURVES:
            assert w[f"{s}/{n}"].shape == SHAPES[n] and w[f"{s}/{n}"].dtype == np.float32, (s, n)
        d = w[f"{s}/ccm"].astype(np.float64) - np.identity(3)
        # identity + one randn(1) * 1e-4, rounded to float32 (the diagonal's rounding is 1 + j's)
        assert np.all(d[~np.eye(3, dtype=bool)] == d[0, 1]) and np.abs(d - d[0, 1]).max() <= 1e-7
        assert 0 < abs(d[0, 1]) < 1e-3
        jitters.append(float(d[0, 1]))
        for n in CURVES[1:]:                                       # the rest is HDRNetCurves' initial curve
            assert w[f"{s}/{n}"].tobytes() == curves[f"{G}/{n}"].tobytes(), (s, n)
    assert len(set(jitters)) == 3                                  # drawn once per level


# ---- the oracle ----------------------------------------------------------------------------------
def oracle_weights(p, seed):
    """The NN pyramid's coefficient network from make_weights, and three different trained-like curves
    guides (make_weights' HDRNetCurves guide at three seeds) under level_{0,1,2}."""
    w = {k: v for k, v in M.make_weights(dict(p, model_name="HDRNetGaussianPyrNN"), seed=seed).items()
         if not k.startswith(G)}
    for l, scope in enumerate(LEVELS):
        c = M.make_weights(dict(p, model_name="HDRNetCurves"), seed=seed + 10 + l)
        w.update({f"{scope}/{n}": c[f"{G}/{n}"] for n in CURVES})
    return w


def _rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max() / max(np.abs(b).max(), 1e-30))


def test_oracle_curves_pyramid_agrees_with_the_torch_restatement():
    """The numpy and torch restatements share no layer code.  Each level's curves guide, fed the same
    level, and the coefficients agree to 1e-6 of range; the levels themselves come from each one's own
    float32 resize, whose last-bit differences the curves' slopes amplify in the guides of levels 1
    and 2 and, through the depth coordinate, in the output: that is held at the pyramid's bar of
    1e-5 of range (tests/test_model_kats.py)."""
    p = dict(M.DEFAULT_PARAMS, model_name=NAME, net_input_size=64, spatial_bin=16)
    wts = oracle_weights(p, 5)
    rng = np.random.RandomState(6)
    low = rng.rand(2, 64, 64, 3).astype(np.float32)
    full = rng.rand(2, 37, 52, 3).astype(np.float32)
    sa = oracle.port().bilateral_slice_apply
    a, ca, ga = pyr_f64(M, low, full, wts, p, sa, M.guide_curves)
    b, cb, gb = pyr_f64(T, low, full, wts, p, sa, T.guide_curves)
    assert [g.shape for g in ga] == [(2, 37, 52), (2, 18, 26), (2, 9, 13)]
    lvls = [full, M.resize_bilinear_ac(full, 18, 26)]
    lvls.append(M.resize_bilinear_ac(lvls[1], 9, 13))
    for lvl, scope, g in zip(lvls, LEVELS, ga):
        assert np.array_equal(M.guide_curves(lvl, wts, scope), g)
        assert np.abs(M.guide_curves(lvl, wts, scope) - T.guide_curves(lvl, wts, scope)).max() <= 1e-6
    assert np.abs(ga[0] - gb[0]).max() <= 1e-6          # level 0 is the input itself
    assert ca.shape == cb.shape == (2, 16, 16, 8, 9, 4) and _rel(ca, cb) <= 1e-6, _rel(ca, cb)
    assert _rel(a, b) <= 1e-5, _rel(a, b)
    # each level runs its own guide: the levels' curves differ, so do their maps on one image
    same = M.guide_curves(full, wts, LEVELS[0])
    assert np.abs(same - M.guide_curves(full, wts, LEVELS[1])).max() > 1e-3


@pytest.mark.parametrize("O", [M, T], ids=["numpy", "torch"])
def test_pyramid_composition_is_the_restatements_own(O):
    """With the pointwise-NN guide, gaussian_pyr_f64 is each restatement's own gaussian_pyr_inference,
    bit for bit: only the guide differs for HDRNetGaussianPyr."""
    p = dict(M.DEFAULT_PARAMS, model_name="HDRNetGaussianPyrNN", net_input_size=64, spatial_bin=16)
    wts = M.make_weights(p, seed=5)
    rng = np.random.RandomState(7)
    low = rng.rand(2, 64, 64, 3).astype(np.float32)
    full = rng.rand(2, 37, 52, 3).astype(np.float32)
    sa = oracle.port().bilateral_slice_apply
    got = pyr_f64(O, low, full, wts, p, sa, O.guide_nn)
    want = O.gaussian_pyr_inference(low, full, wts, p, sa)
    for x, y in zip((got[0], got[1], *got[2]), (want[0], want[1], *want[2])):
        assert x.dtype == y.dtype and x.tobytes() == y.tobytes()


# ---- the training CLI ----------------------------------------------------------------------------
def parse(*argv):
    parser = train.build_parser()
    args = parser.parse_args(["ckpt", "data", "--model_name", NAME, *argv])
    train.check_data_flags(parser, args)
    return args, train.model_params(parser, args)


def refuse(*argv):
    args, params = parse(*argv)
    train.refuse_untrainable(params, args.train_guide, args.guide_batch_stats, args.coefficient_batch_stats)
    return params


USM_GPYR = ["--learning_rate", "1e-4", "--batch_size", "1", "--data_pipeline", "UnsharpMaskDataPipeline",
            "--blur_sigma", "4", "--sharpen", "2", "--nobatch_norm", "--output_resolution", "2048", "2048"]
LL_GPYR = ["--learning_rate", "1e-4", "--batch_size", "1", "--nobatch_norm", "--output_resolution", "2048", "2048",
           "--luma_bins", "8", "--spatial_bin", "16", "--channel_multiplier", "1"]
LL_STRONG_CM4 = ["--learning_rate", "1e-4", "--batch_size", "4", "--nobatch_norm", "--output_resolution", "1024",
                 "1024", "--luma_bins", "8", "--spatial_bin", "16", "--channel_multiplier", "4"]


@pytest.mark.parametrize("flags", [[], ["--train_guide"], USM_GPYR, USM_GPYR + ["--train_guide"], LL_GPYR,
                                   LL_STRONG_CM4, ["--batch_norm", "--coefficient_batch_stats"],
                                   ["--batch_norm", "--coefficient_batch_stats", "--train_guide"]],
                         ids=["plain", "train_guide", "usm_gpyr", "usm_gpyr_guide", "ll_gpyr", "ll_strong_cm4",
                              "coefficient_bn", "coefficient_bn_guide"])
def test_accepted_flag_sets(flags):
    params = refuse(*flags)
    assert params["model_name"] == NAME and "guide_batch_stats" not in params


def test_default_model_is_unchanged():
    parser = train.build_parser()
    assert parser.parse_args(["c", "d"]).model_name == "HDRNetCurves"
    with pytest.raises(SystemExit):
        parser.parse_args(["c", "d", "--model_name", "HDRNetBogus"])


@pytest.mark.parametrize("flags,exc,match", [
    (["--guide_batch_stats"], ValueError, "HDRNetGaussianPyr's guides are curves, with no batch norm"),
    (["--guide_batch_stats", "--train_guide"], ValueError, "no batch norm"),
    (["--batch_norm"], NotImplementedError, "--coefficient_batch_stats runs it in training mode"),
    (["--coefficient_batch_stats"], ValueError, "it needs --batch_norm"),
], ids=["stats", "stats_guide", "batch_norm", "coefficient_stats_alone"])
def test_refused_flag_sets(flags, exc, match):
    with pytest.raises(exc, match=match):
        refuse(*flags)


def test_guide_batch_stats_is_refused_before_any_data_is_read(tmp_path):
    ckpt = tmp_path / "ckpt"
    with pytest.raises(ValueError, match="HDRNetGaussianPyr's guides are curves") as e:
        train.main([str(ckpt), str(tmp_path / "no_such_data"), "--model_name", NAME, "--guide_batch_stats",
                    *USM_GPYR])
    assert "--guide_batch_stats runs the pointwise-NN guide's batch norm" in str(e.value)
    assert not ckpt.exists()


def test_accepted_flags_get_past_the_refusals_to_the_data(tmp_path):
    with pytest.raises(Exception) as e:
        train.main([str(tmp_path / "ckpt"), str(tmp_path / "no_such_data"), "--model_name", NAME, "--train_guide",
                    *USM_GPYR])
    assert not isinstance(e.value, (NotImplementedError, ValueError)) or "guide" not in str(e.value)


def test_trained_names_cover_the_three_curves_guides():
    p = dict(models.DEFAULT_PARAMS, net_input_size=32, spatial_bin=8, luma_bins=4, model_name=NAME)
    w = models.init_weights(p)
    names = train.trained_names(w, train_guide=True)
    assert {f"{s}/{n}" for s in LEVELS for n in CURVES} <= set(names)
    assert not any(k.startswith(G) for k in train.trained_names(w, train_guide=False))


# ---- the model's refusals, on the CPU --------------------------------------------------------------
SMALL_P = dict(models.DEFAULT_PARAMS, net_input_size=32, spatial_bin=8, luma_bins=4, model_name=NAME)


def test_guide_gradients_need_guide_grad_and_name_the_model():
    w = {k: torch.from_numpy(v) for k, v in models.init_weights(SMALL_P).items()}
    w[f"{LEVELS[1]}/slopes"].requires_grad_(True)
    with pytest.raises(NotImplementedError, match="level_1/slopes") as e:
        PYR.inference(torch.zeros(1, 32, 32, 3), torch.zeros(1, 8, 8, 3), dict(SMALL_P, weights=w))
    assert str(e.value).endswith("params['guide_grad'] computes them for HDRNetGaussianPyr")
    with pytest.raises(NotImplementedError, match="fullres_input"):
        PYR.inference(torch.zeros(1, 32, 32, 3), torch.zeros(1, 8, 8, 3, requires_grad=True),
                      dict(SMALL_P, weights=models.init_weights(SMALL_P)))
    with pytest.raises(NotImplementedError, match="inference path only"):
        PYR.inference(torch.zeros(1, 32, 32, 3), torch.zeros(1, 8, 8, 3), dict(SMALL_P, weights=w), is_training=True)


# ---- the frozen model file -------------------------------------------------------------------------
SMALL = dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8)
ODD = dict(models.DEFAULT_PARAMS, net_input_size=32, spatial_bin=8, luma_bins=16, channel_multiplier=2,
           guide_complexity=32, batch_norm=True)
SB3 = dict(models.DEFAULT_PARAMS, net_input_size=48, spatial_bin=3, guide_complexity=8)


def frozen_weights(params, seed=3):
    """init_weights with non-trivial batch-norm statistics and three different curves guides."""
    w = models.init_weights(params, seed=seed, model_name=NAME)
    rng = np.random.RandomState(seed)
    for k in sorted(w):
        if k.endswith("moving_mean") or k.endswith("BatchNorm/beta"):
            w[k] = rng.randn(*w[k].shape).astype(np.float32) * 0.1
        elif k.endswith("moving_variance"):
            w[k] = rng.rand(*w[k].shape).astype(np.float32) + 0.5
        elif k.startswith(G):
            w[k] = (w[k] + 0.05 * rng.randn(*w[k].shape)).astype(np.float32)
    return w


def _create(blob: bytes) -> int:
    lib = _lib.load()
    handle = ctypes.c_void_p()
    rc = lib.hdrnet_model_create(blob, len(blob), ctypes.byref(handle))
    if rc == _lib.OK:
        lib.hdrnet_model_destroy(handle)
    return rc


def test_kind_names():
    assert checkpoint.FROZEN_KINDS == ("HDRNetCurves", "HDRNetPointwiseNNGuide", "HDRNetGaussianPyrNN")
    assert checkpoint.FROZEN_MODEL_NAMES == checkpoint.FROZEN_KINDS + (NAME,)
    assert frozen.FROZEN_MODEL_NAMES is checkpoint.FROZEN_MODEL_NAMES


@pytest.mark.parametrize("params", [SMALL, ODD, SB3], ids=["default", "nondefault", "spatial_bin3"])
def test_round_trip_equals_prepared_bitwise(built_lib, tmp_path, params):
    params = dict(params, model_name=NAME)
    w = frozen_weights(params)
    path = checkpoint.freeze_model(w, params, str(tmp_path / "m.hdrnet"))
    with open(path, "rb") as f:
        blob = f.read()
    assert np.frombuffer(blob, "<u4", 1, 12)[0] == 3      # HDRNET_MODEL_GAUSSIAN_PYR
    got = checkpoint.read_frozen_model(path)
    assert got["model_name"] == NAME and got["guide_width"] == 16
    for k in ("net_input_size", "spatial_bin", "luma_bins", "channel_multiplier"):
        assert got[k] == params[k]
    prep = models._Prepared(w, params, torch.device("cpu"), PYR._nn_guide)
    want = []
    for scope, _, _ in models._coefficient_specs(params):
        wd, bd, _ = prep.layers[scope]
        want += [wd.numpy(), np.zeros(0, np.float32) if bd is None else bd.numpy()]
    assert len(prep.guides) == 3 and all(isinstance(g, models._CurvesGuide) for g in prep.guides)
    for g in prep.guides:
        want += [g.ccm, g.ccm_bias, g.shifts, g.slopes, g.mix, np.float32([g.mix_bias])]
    assert len(got["arrays"]) == len(want) == 2 * len(models._coefficient_specs(params)) + 18
    for a, b in zip(got["arrays"], want):
        assert a.shape == b.shape and a.dtype == np.float32
        assert a.tobytes() == np.ascontiguousarray(b, np.float32).tobytes()
    # level l's arrays are its own variables
    for l, scope in enumerate(LEVELS):
        base = 2 * len(models._coefficient_specs(params)) + 6 * l
        assert got["arrays"][base].tobytes() == w[f"{scope}/ccm"].tobytes()
        assert got["arrays"][base + 3].tobytes() == w[f"{scope}/slopes"].reshape(3, 16).tobytes()
    assert _create(blob) != _lib.E_BAD_MODEL


@pytest.mark.parametrize("case", ["shifts_transposed", "ccm_wide", "mix_bias_missing", "guide_width",
                                  "too_few_levels", "nn_guides"])
def test_wrong_guide_shapes_are_refused_without_a_gpu(built_lib, case):
    params = dict(SMALL, model_name=NAME)
    arrays = checkpoint.frozen_arrays(frozen_weights(params), params)
    hyper = [64, 8, 8, 1, 16]
    n = len(arrays)
    if case == "shifts_transposed":        # level 1's shifts [16, 3]
        arrays[n - 12 + 2] = np.ascontiguousarray(arrays[n - 12 + 2].T)
    elif case == "ccm_wide":               # level 2's ccm [3, 4]
        arrays[n - 6] = np.zeros((3, 4), np.float32)
    elif case == "mix_bias_missing":       # level 0's mix_bias [0]
        arrays[n - 18 + 5] = np.zeros(0, np.float32)
    elif case == "guide_width":            # the curves have 16 knots, whatever the header says
        hyper[4] = 8
    elif case == "too_few_levels":         # HDRNetCurves' single guide under kind 3
        arrays = arrays[:-12]
    else:                                  # the NN pyramid's guides under kind 3
        nn = dict(SMALL, model_name="HDRNetGaussianPyrNN")
        arrays = checkpoint.frozen_arrays(models.init_weights(nn, seed=3, model_name=nn["model_name"]), nn)
    assert _create(checkpoint._frozen_bytes(3, hyper, arrays)) == _lib.E_BAD_MODEL
    good = checkpoint.frozen_arrays(frozen_weights(params), params)
    assert _create(checkpoint._frozen_bytes(3, [64, 8, 8, 1, 16], good)) != _lib.E_BAD_MODEL
    # the same arrays under the NN pyramid's kind are refused too
    assert _create(checkpoint._frozen_bytes(2, [64, 8, 8, 1, 16], good)) == _lib.E_BAD_MODEL


def test_guide_dumps_stay_refused():
    params = dict(SMALL, model_name=NAME)
    with pytest.raises(ValueError, match="no guide dumps"):
        checkpoint.guide_bins(frozen_weights(params), NAME)
