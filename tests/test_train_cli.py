"""CPU tests of the training CLI (hdrnet_b200/bin/train.py) and its data pipeline: the reference's
flag defaults, the refusals before any data is read, the file list and pair checks, the sampler as a
pure function of (seed, step), and the checkpoint layout (Adam slots, global_step) through the
tensor-bundle reader and model_weights."""
import os

import cv2
import numpy as np
import pytest

from hdrnet_b200 import checkpoint, data_pipeline as dp, models
from hdrnet_b200.bin import train

# hdrnet/bin/train.py:188-244
REFERENCE_DEFAULTS = dict(
    eval_data_dir=None, learning_rate=1e-4, log_interval=1, summary_interval=120, checkpoint_interval=600,
    eval_interval=3600, profiling=False, batch_size=16, data_threads=2, rotate=False, flipud=False, fliplr=False,
    random_crop=True, model_name="HDRNetCurves", data_pipeline="ImageFilesDataPipeline", net_input_size=256,
    output_resolution=[512, 512], batch_norm=False, channel_multiplier=1, guide_complexity=16, luma_bins=8,
    spatial_bin=16)
REFERENCE_MODEL_PARAMS = ["model_name", "data_pipeline", "net_input_size", "output_resolution", "batch_norm",
                          "channel_multiplier", "guide_complexity", "luma_bins", "spatial_bin"]


def parse(*argv):
    parser = train.build_parser()
    args = parser.parse_args(["ckpt", "data", *argv])
    return args, train.model_params(parser, args)


def test_parsing_reproduces_the_reference_defaults():
    args, params = parse()
    for k, v in REFERENCE_DEFAULTS.items():
        assert getattr(args, k) == v, k
    assert (args.checkpoint_dir, args.data_dir, args.max_steps, args.seed) == ("ckpt", "data", None, 0)
    assert sorted(params) == sorted(REFERENCE_MODEL_PARAMS)
    assert all(params[k] == models.DEFAULT_PARAMS[k] for k in params if k in models.DEFAULT_PARAMS)


def test_flag_pairs_and_values_parse():
    args, params = parse("--fliplr", "--flipud", "--rotate", "--norandom_crop", "--batch_norm", "--nobatch_norm",
                         "--output_resolution", "300", "200", "--net_input_size", "128", "--max_steps", "7",
                         "--model_name", "HDRNetPointwiseNNGuide", "--learning_rate", "3e-3")
    assert (args.fliplr, args.flipud, args.rotate, args.random_crop, args.batch_norm) == (True, True, True, False, False)
    assert params["output_resolution"] == [300, 200] and params["net_input_size"] == 128 and args.max_steps == 7
    assert params["model_name"] == "HDRNetPointwiseNNGuide" and args.learning_rate == 3e-3


def test_tfrecord_pipelines_and_unknown_models_are_not_accepted():
    for bad in (["--data_pipeline", "HDRpDataPipeline"], ["--data_pipeline", "StyleTransferDataPipeline"],
                ["--model_name", "NoSuchModel"]):
        with pytest.raises(SystemExit):
            parse(*bad)


@pytest.mark.parametrize("flags,match", [(["--batch_norm"], "batch-norm"),
                                         (["--model_name", "HDRNetGaussianPyrNN"], "resize"),
                                         (["--model_name", "HDRNetPointwiseNNGuide", "--batch_norm"], "batch-norm")])
def test_untrainable_configurations_are_refused_before_data_is_read(tmp_path, flags, match):
    ckpt, data = tmp_path / "ckpt", tmp_path / "no_such_data"
    with pytest.raises(NotImplementedError, match=match):
        train.main([str(ckpt), str(data), *flags])
    assert not ckpt.exists()


def test_refusal_text_is_the_models_own():
    _, params = parse("--model_name", "HDRNetGaussianPyrNN")
    with pytest.raises(NotImplementedError) as e:
        train.refuse_untrainable(params)
    assert str(e.value).startswith("HDRNetGaussianPyrNN.inference (needs the VJP of the align-corners resize)")
    _, params = parse("--batch_norm")
    with pytest.raises(NotImplementedError) as e:
        train.refuse_untrainable(params)
    assert str(e.value).startswith("gradients through a batch-norm layer are not implemented")
    train.refuse_untrainable(parse()[1])                                       # the defaults train
    train.refuse_untrainable(parse("--model_name", "HDRNetPointwiseNNGuide")[1])


# ---- file list, decoding and pair checks ---------------------------------------------------------
def write_pair(root, name, im_in, im_out):
    for sub, im in (("input", im_in), ("output", im_out)):
        os.makedirs(os.path.join(root, sub), exist_ok=True)
        assert cv2.imwrite(os.path.join(root, sub, name), im)


def test_filelist_is_read_from_the_directory_or_the_file(tmp_path):
    rng = np.random.RandomState(0)
    for n in ("a.png", "b b.png"):
        write_pair(tmp_path, n, rng.randint(0, 256, (20, 30, 3), dtype=np.uint8),
                   rng.randint(0, 65536, (20, 30, 3)).astype(np.uint16))
    (tmp_path / "filelist.txt").write_text("a.png\n\n  b b.png  \n")
    for path in (str(tmp_path), str(tmp_path / "filelist.txt")):
        names, ins, outs, d = dp.load_pairs(path, nthreads=2)
        assert names == ["a.png", "b b.png"] and os.path.samefile(d, tmp_path)
        assert [a.dtype for a in ins] == [np.uint8] * 2 and [a.dtype for a in outs] == [np.uint16] * 2
    with pytest.raises(ValueError, match="filelist"):
        dp.load_pairs(str(tmp_path / "input"))
    (tmp_path / "filelist.txt").write_text("a.png\nmissing.png\n")
    with pytest.raises(ValueError, match="missing.png"):
        dp.load_pairs(str(tmp_path))
    (tmp_path / "filelist.txt").write_text("\n\n")
    with pytest.raises(ValueError, match="names no images"):
        dp.load_pairs(str(tmp_path))


def test_decoding_gives_rgb_in_the_storage_format(tmp_path):
    bgr = np.zeros((4, 5, 3), np.uint8)
    bgr[..., 0], bgr[..., 1], bgr[..., 2] = 10, 20, 30
    cv2.imwrite(str(tmp_path / "c.png"), bgr)
    assert dp.decode_image(str(tmp_path / "c.png"))[0, 0].tolist() == [30, 20, 10]
    bgra = np.concatenate([bgr.astype(np.uint16) * 257, np.full((4, 5, 1), 7, np.uint16)], axis=2)
    cv2.imwrite(str(tmp_path / "a.png"), bgra)
    im = dp.decode_image(str(tmp_path / "a.png"))
    assert im.dtype == np.uint16 and im.shape == (4, 5, 3) and im[1, 2].tolist() == [30 * 257, 20 * 257, 10 * 257]
    grey = np.arange(20, dtype=np.uint8).reshape(4, 5)
    cv2.imwrite(str(tmp_path / "g.png"), grey)
    im = dp.decode_image(str(tmp_path / "g.png"))
    assert im.shape == (4, 5, 3) and all(np.array_equal(im[..., c], grey) for c in range(3))


def test_pair_size_and_crop_errors_name_the_file(tmp_path):
    a = np.zeros((300, 600, 3), np.uint8)
    with pytest.raises(ValueError, match=r"input/x\.png is 300x600 but .*output/x\.png is 300x500"):
        dp.check_pairs(["x.png"], [a], [np.zeros((300, 500, 3), np.uint8)], "d", (256, 512), rotate=False)
    dp.check_pairs(["x.png"], [a], [a], "d", (256, 512), rotate=False)
    with pytest.raises(ValueError, match=r"input/x\.png is 300x600, smaller when rotated than the output resolution 256x512"):
        dp.check_pairs(["x.png"], [a], [a], "d", (256, 512), rotate=True)
    with pytest.raises(ValueError, match=r"input/y\.png is 300x600, smaller than the output resolution 512x512"):
        dp.check_pairs(["y.png"], [a], [a], "d", (512, 512), rotate=False)
    dp.check_pairs(["x.png"], [a], [a], "d", (300, 300), rotate=True)


# ---- the sampler ---------------------------------------------------------------------------------
SIZES = [(600, 800), (512, 512), (700, 530), (530, 700), (900, 1200)]


def sampler(**kw):
    args = dict(batch_size=4, output_resolution=(512, 512), shuffle=True, fliplr=True, flipud=True, rotate=True,
                random_crop=True, seed=3)
    args.update(kw)
    return dp.Sampler(SIZES, **args)


def test_sampler_is_a_pure_function_of_seed_and_step():
    a, b = sampler(), sampler()
    steps = [0, 1, 2, 50, 7, 3]
    got_a = {s: a.draws(s) for s in steps}
    got_b = {s: b.draws(s) for s in reversed(steps)}               # another instance, another order
    assert got_a == got_b
    assert a.draws(50) == got_a[50]                                  # and again
    assert sampler(seed=4).draws(0) != got_a[0]
    assert len({tuple(d) for s in steps for d in got_a[s]}) > 10     # the draws vary


def test_sampler_epochs_are_permutations_and_crops_fit():
    s = sampler(batch_size=5)
    for epoch in range(4):
        assert sorted(d.index for d in s.draws(epoch)) == list(range(len(SIZES)))
    seen = set()
    for step in range(200):
        for d in s.draws(step):
            H, W = SIZES[d.index]
            rh, rw = (W, H) if d.rot90 % 2 else (H, W)
            assert 0 <= d.crop_y <= rh - 512 and 0 <= d.crop_x <= rw - 512
            seen.add((d.fliplr, d.flipud, d.rot90))
    assert len(seen) == 16                                           # every flip / rotation combination


def test_sampler_without_augmentation_takes_the_centre_crop_in_order():
    s = sampler(shuffle=False, fliplr=False, flipud=False, rotate=False, random_crop=False, batch_size=3)
    got = s.draws(0) + s.draws(1)
    assert [d.index for d in got] == [0, 1, 2, 3, 4, 0]
    for d in got:
        H, W = SIZES[d.index]
        assert (d.fliplr, d.flipud, d.rot90) == (False, False, 0)
        assert (d.crop_y, d.crop_x) == (int((H - 512) / 2), int((W - 512) / 2))
    assert (got[2].crop_y, got[2].crop_x) == (94, 9)                 # 700x530: truncation of 94.0, 9.0
    assert (got[3].crop_y, got[3].crop_x) == (9, 94)


def test_only_the_enabled_augmentations_change_the_draws():
    full, no_flip = sampler(), sampler(fliplr=False, flipud=False)
    for step in range(10):
        for d, e in zip(full.draws(step), no_flip.draws(step)):
            assert (d.index, d.rot90, d.crop_y, d.crop_x) == (e.index, e.rot90, e.crop_y, e.crop_x)
            assert not e.fliplr and not e.flipud


# ---- checkpoints -----------------------------------------------------------------------------------
def test_checkpoint_with_slots_and_global_step_round_trips(tmp_path):
    params = dict(models.DEFAULT_PARAMS, net_input_size=32, spatial_bin=8, luma_bins=4)
    variables = models.init_weights(params, seed=2)
    trained = sorted(k for k in variables if k.startswith(train.COEFFS))
    rng = np.random.RandomState(1)
    moments = {k: (rng.randn(*variables[k].shape).astype(np.float32),
                   rng.rand(*variables[k].shape).astype(np.float32)) for k in trained}
    t = train.checkpoint_tensors(variables, moments, 1234, {"loss": 0.25, "psnr": 17.5})
    checkpoint.write_tf_checkpoint(str(tmp_path / "model.ckpt-1234"), t)
    saved = checkpoint.read_tf_checkpoint(str(tmp_path))
    assert saved["global_step"].dtype == np.int64 and saved["global_step"].shape == () and saved["global_step"] == 1234
    for k in trained:
        assert np.array_equal(saved[k + "/Adam"], moments[k][0]) and np.array_equal(saved[k + "/Adam_1"], moments[k][1])
    assert np.float32(saved["beta1_power"]) == np.float32(0.9 ** 1235)
    values, got_moments, step, ema = train.restored_state(saved, variables, trained)
    assert step == 1234 and ema == {"loss": 0.25, "psnr": 17.5}
    assert all(np.array_equal(values[k], variables[k]) for k in variables)
    assert all(np.array_equal(got_moments[k][i], moments[k][i]) for k in trained for i in (0, 1))
    w = checkpoint.model_weights(saved)
    assert sorted(w) == sorted(variables)                            # slots, step and accumulators dropped
    del saved[trained[0] + "/Adam_1"]
    with pytest.raises(ValueError, match="Adam_1"):
        train.restored_state(saved, variables, trained)
