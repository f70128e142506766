"""CPU tests of ``--data_pipeline UnsharpMaskDataPipeline``: the flags, every refusal (all before
any data is read), the checkpoint scalars and the resume-mismatch refusal, the input-only loading
(``output/`` is not needed), and the kernel's error codes, which it returns before any launch."""
import ctypes
import os

import cv2
import numpy as np
import pytest

from hdrnet_b200 import _lib, checkpoint, data_pipeline as dp
from hdrnet_b200.bin import train

USM = ["--data_pipeline", "UnsharpMaskDataPipeline"]


def parse(*argv):
    parser = train.build_parser()
    args = parser.parse_args(["ckpt", "data", *argv])
    return parser, args


def test_flags_default_off_and_are_not_model_parameters():
    parser, args = parse()
    assert args.blur_sigma is None and args.sharpen is None and train.usm_values(args) is None
    train.check_data_flags(parser, args)
    parser, args = parse(*USM, "--blur_sigma", "2", "--sharpen", "1.5")
    train.check_data_flags(parser, args)
    assert train.usm_values(args) == (2.0, 1.5)
    params = train.model_params(parser, args)
    assert "blur_sigma" not in params and "sharpen" not in params
    assert params["data_pipeline"] == "UnsharpMaskDataPipeline"
    assert "UnsharpMaskDataPipeline" in dp.__all__


@pytest.mark.parametrize("flags,match", [
    (USM, "needs --blur_sigma and --sharpen"),
    (USM + ["--blur_sigma", "2"], "needs --blur_sigma and --sharpen"),
    (USM + ["--sharpen", "1"], "needs --blur_sigma and --sharpen"),
    (["--blur_sigma", "2"], "--blur_sigma sets the unsharp-mask target"),
    (["--sharpen", "1"], "--sharpen sets the unsharp-mask target"),
    (["--blur_sigma", "2", "--sharpen", "1"], "ImageFilesDataPipeline reads its targets"),
    (USM + ["--blur_sigma", "0", "--sharpen", "1"], "blur_sigma must be in"),
    (USM + ["--blur_sigma", "-1", "--sharpen", "1"], "blur_sigma must be in"),
    (USM + ["--blur_sigma", "32.5", "--sharpen", "1"], "blur_sigma must be in"),
    (USM + ["--blur_sigma", "nan", "--sharpen", "1"], "blur_sigma must be in"),
    (USM + ["--blur_sigma", "2", "--sharpen", "inf"], "sharpen must be a finite"),
    (USM + ["--blur_sigma", "2", "--sharpen", "nan"], "sharpen must be a finite"),
])
def test_refusals_come_before_any_data_is_read(tmp_path, capsys, flags, match):
    ckpt = tmp_path / "ckpt"
    with pytest.raises(SystemExit) as e:
        train.main([str(ckpt), str(tmp_path / "no_such_data"), *flags])
    assert e.value.code == 2
    assert match in capsys.readouterr().err
    assert not ckpt.exists()


def test_pipeline_refuses_bad_values_before_reading_files(tmp_path):
    for sigma, sharpen, match in ((None, 1.0, "numbers"), (2.0, None, "numbers"), (0.0, 1.0, "blur_sigma"),
                                  (33.0, 1.0, "blur_sigma"), (2.0, float("inf"), "sharpen")):
        with pytest.raises(ValueError, match=match):
            dp.UnsharpMaskDataPipeline(str(tmp_path / "no_such_data"), blur_sigma=sigma, sharpen=sharpen)
    assert dp.check_usm(32, -0.5) == (32.0, -0.5)
    assert dp.usm_radius(32.0) == 128 and dp.usm_radius(0.5) == 2 and dp.usm_radius(2.5) == 10


def _checkpoint(path, usm=None):
    variables = {"inference/coefficients/splat/conv1/weights": np.zeros((3, 3, 3, 8), np.float32)}
    moments = {k: (v, v) for k, v in variables.items()}
    checkpoint.write_tf_checkpoint(str(path / "model.ckpt-3"), train.checkpoint_tensors(variables, moments, 3, {}, usm))
    return checkpoint.read_tf_checkpoint(str(path / "model.ckpt-3"))


def test_checkpoint_records_the_values_and_resume_checks_them(tmp_path):
    saved = _checkpoint(tmp_path, (2.0, 1.5))
    assert float(saved["train/usm_blur_sigma"]) == 2.0 and float(saved["train/usm_sharpen"]) == 1.5
    train.refuse_resume_mismatch(saved, False, (2.0, 1.5))
    for usm, match in ((None, "resume it with those flags"), ((2.0, 1.0), "not 2.0 and 1.0"),
                       ((4.0, 1.5), "not 4.0 and 1.5")):
        with pytest.raises(ValueError, match=match):
            train.refuse_resume_mismatch(saved, False, usm)
    # the restored state ignores the scalars
    _, _, step, ema = train.restored_state(saved, {"inference/coefficients/splat/conv1/weights": 0},
                                           ["inference/coefficients/splat/conv1/weights"])
    assert step == 3 and ema == {}


def test_checkpoint_readers_ignore_the_scalars(tmp_path):
    """bin/run.py, freeze_model and import_checkpoint read a training directory through
    import_checkpoint, which keeps only inference/* variables."""
    _checkpoint(tmp_path, (2.0, 1.5))
    params, weights = checkpoint.import_checkpoint(str(tmp_path))
    assert sorted(weights) == ["inference/coefficients/splat/conv1/weights"] and params is None
    pairs = tmp_path / "pairs"
    pairs.mkdir()
    paired = _checkpoint(pairs)
    assert not any(k.startswith("train/usm") for k in paired)
    with pytest.raises(ValueError, match="trained on image pairs"):
        train.refuse_resume_mismatch(paired, False, (2.0, 1.5))
    train.refuse_resume_mismatch(paired, False, None)


@pytest.mark.parametrize("saved_usm,flags,match", [
    ((2.0, 1.0), [], "resume it with those flags"),
    ((2.0, 1.0), USM + ["--blur_sigma", "3", "--sharpen", "1"], "not 3.0 and 1.0"),
    (None, USM + ["--blur_sigma", "2", "--sharpen", "1"], "trained on image pairs")])
def test_resume_mismatch_is_refused_before_any_data_is_read(tmp_path, saved_usm, flags, match):
    ckpt = tmp_path / "ckpt"
    ckpt.mkdir()
    _checkpoint(ckpt, saved_usm)
    with pytest.raises(ValueError, match=match):
        train.main([str(ckpt), str(tmp_path / "no_such_data"), *flags])


def test_inputs_load_without_output_folder(tmp_path):
    rng = np.random.RandomState(0)
    os.makedirs(tmp_path / "input")
    for n, dt in (("a.png", np.uint8), ("b.png", np.uint16)):
        im = rng.randint(0, np.iinfo(dt).max + 1, (20, 30, 3)).astype(dt)
        assert cv2.imwrite(str(tmp_path / "input" / n), im)
    (tmp_path / "filelist.txt").write_text("a.png\nb.png\n")
    assert not (tmp_path / "output").exists()
    names, ins, d = dp.load_inputs(str(tmp_path / "filelist.txt"), nthreads=2)
    assert names == ["a.png", "b.png"] and [a.dtype for a in ins] == [np.uint8, np.uint16]
    dp.check_inputs(names, ins, d, (20, 30), rotate=False)
    with pytest.raises(ValueError, match="smaller when rotated"):
        dp.check_inputs(names, ins, d, (20, 30), rotate=True)
    with pytest.raises(ValueError, match="a.png"):
        dp.check_inputs(names, ins, d, (21, 30), rotate=False)


def test_grown_window_and_slot_bytes():
    d = dp.Draw(0, False, False, 0, 5, 7)
    assert dp.grown_window(40, 50, d, 10, 12, 3) == (2, 4, 16, 18)
    assert dp.grown_window(40, 50, d, 10, 12, 30) == (0, 0, 40, 49)
    for lr, ud, k in [(a, b, c) for a in (0, 1) for b in (0, 1) for c in range(4)]:
        d = dp.Draw(0, bool(lr), bool(ud), k, 2, 3)
        y, x, h, w = dp.source_window(40, 50, d, 10, 12)
        y0, x0, gh, gw = dp.grown_window(40, 50, d, 10, 12, 4)
        assert (y0, x0) == (max(0, y - 4), max(0, x - 4))
        assert (y0 + gh, x0 + gw) == (min(40, y + h + 4), min(50, x + w + 4))
    ims = [np.zeros((40, 50, 3), np.uint8), np.zeros((30, 30, 3), np.uint16)]
    assert dp.usm_slot_bytes(ims, 3, (10, 12), 4, False) == 3 * dp._aligned(18 * 20 * 3 * 2)
    assert dp.usm_slot_bytes(ims, 2, (10, 12), 100, True) == 2 * dp._aligned(40 * 50 * 3)


# ---- the kernel's error codes (no launch, no device) --------------------------------------------
def sample(**kw):
    s = dict(input=16, input_fmt=_lib.PX_U8, H=40, W=50, y0=0, x0=0, h=40, w=50, fliplr=0, flipud=0, rot90=0,
             crop_y=10, crop_x=10)
    s.update(kw)
    return _lib.UsmSample(**s)


def call(samples, B, outs=(16, 32, 48), oh=8, ow=8, S=4, sigma=1.0, sharpen=1.0, ws=64, ws_bytes=1 << 30):
    arr = None if samples is None else (_lib.UsmSample * len(samples))(*samples)
    ptr = None if arr is None else ctypes.cast(arr, ctypes.c_void_p)
    return _lib.load().hdrnet_train_batch_usm_f32(ptr, B, *outs, oh, ow, S, sigma, sharpen, ws, ws_bytes, None)


def ws_bytes(samples, oh=8, ow=8, sigma=1.0):
    arr = (_lib.UsmSample * len(samples))(*samples)
    return _lib.load().hdrnet_train_batch_usm_workspace_bytes(ctypes.cast(arr, ctypes.c_void_p), len(samples),
                                                              oh, ow, sigma)


def test_error_codes(built_lib):
    assert call(None, 0) == _lib.OK
    assert call(None, 1) == _lib.E_NULL_POINTER
    assert call([sample()], 1, (16, 0, 48)) == _lib.E_NULL_POINTER       # fullres_out is required
    assert call([sample()], 1, ws=None) == _lib.E_NULL_POINTER
    assert call([sample(), sample(input=None)], 2) == _lib.E_NULL_POINTER
    for bad in (dict(H=0), dict(rot90=4), dict(crop_y=-1), dict(crop_x=43), dict(rot90=1, crop_y=43),
                dict(h=41), dict(y0=1), dict(x0=-1), dict(w=0),
                # a window that does not cover the crop grown by r = 4 (rows 6..21, columns 6..21)
                dict(y0=7, h=33), dict(x0=7, w=43), dict(h=21), dict(w=21)):
        assert call([sample(**bad)], 1) == _lib.E_BAD_SHAPE, bad
    assert call([sample()], -1) == _lib.E_BAD_SHAPE
    for shape in (dict(oh=0), dict(ow=-1), dict(S=0), dict(sigma=0.0), dict(sigma=32.01), dict(sigma=float("nan")),
                  dict(sharpen=float("inf")), dict(sharpen=float("nan"))):
        assert call([sample()], 1, **shape) == _lib.E_BAD_SHAPE, shape
    assert call([sample(input_fmt=3)], 1) == _lib.E_UNSUPPORTED
    # the workspace: exact size from the query, one byte short refused, misaligned refused
    need = ws_bytes([sample(), sample(rot90=1, fliplr=1)])
    assert need == 2 * dp._aligned(16 * 8 * 3 * 4)           # rows 6..21 of 8 crop columns, per sample
    assert call([sample(), sample(rot90=1, fliplr=1)], 2, ws_bytes=need - 1) == _lib.E_BAD_SHAPE
    assert call([sample()], 1, ws=66) == _lib.E_BAD_SHAPE
    assert ws_bytes([sample(H=0)]) == 0 and ws_bytes([sample()], sigma=40.0) == 0
    # a clipped window: the crop at the source's corner grows only inward
    corner = sample(crop_y=0, crop_x=0, h=12, w=12)
    assert ws_bytes([corner]) == dp._aligned(12 * 8 * 3 * 4)
    assert call([sample(crop_y=0, crop_x=0, h=11)], 1) == _lib.E_BAD_SHAPE
    # 17 samples: two launches share the workspace, so it is the larger launch's
    assert ws_bytes([sample()] * 17) == 16 * dp._aligned(16 * 8 * 3 * 4)
