"""uint16 results from the model path, the parts that need no GPU: run.py's --output_bit_depth flag,
the refusal of any other out_dtype before any device work, and quantize_u16 (the pyramid's
quantisation on the device) against its numpy restatement."""
import numpy as np
import pytest
import torch

from hdrnet_b200 import _lib, host_pipeline, models
from hdrnet_b200.bin import run


def test_output_bit_depth_flag():
    parse = run.build_parser().parse_args
    assert parse(["ckpt", "in", "out"]).output_bit_depth == 8
    assert parse(["ckpt", "in", "out", "--output_bit_depth", "16"]).output_bit_depth == 16
    assert parse(["ckpt", "in", "out", "--output_bit_depth", "8"]).output_bit_depth == 8
    for bad in ("12", "32", "sixteen"):
        with pytest.raises(SystemExit):
            parse(["ckpt", "in", "out", "--output_bit_depth", bad])
    assert run.OUTPUT_DTYPES == {8: torch.uint8, 16: torch.uint16}


@pytest.fixture
def no_device(monkeypatch):
    """Any library load or CUDA query fails the test: the refusal must come first."""
    def device_work(*a, **k):
        raise AssertionError("device work before the out_dtype check")
    monkeypatch.setattr(_lib, "load", device_work)
    monkeypatch.setattr(torch.cuda, "is_available", device_work)
    monkeypatch.setattr(torch.cuda, "current_device", device_work)


BAD_DTYPES = [torch.int16, torch.int32, torch.float16, torch.bfloat16, torch.float64, np.uint16, "uint16", None]


@pytest.mark.parametrize("bad", BAD_DTYPES, ids=str)
def test_other_out_dtypes_are_refused_before_device_work(no_device, bad):
    im = torch.zeros(1, 8, 8, 3, dtype=torch.uint16)
    params = dict(models.DEFAULT_PARAMS)
    calls = [lambda: models.HDRNetCurves.inference_image(im, params, out_dtype=bad),
             lambda: models.HDRNetPointwiseNNGuide.inference_image(im, params, out_dtype=bad),
             lambda: models.HDRNetGaussianPyrNN.inference_image(im, params, out_dtype=bad),
             lambda: models.HDRNetCurves.inference_image_host(im, params, out_dtype=bad),
             lambda: host_pipeline.HostImagePipeline(models.HDRNetCurves, params, out_dtype=bad)]
    for call in calls:
        with pytest.raises(TypeError, match=r"torch\.uint8, torch\.uint16 or torch\.float32"):
            call()


def test_accepted_out_dtypes():
    assert models.OUT_DTYPES == (torch.uint8, torch.uint16, torch.float32)
    for dt in models.OUT_DTYPES:
        models._check_out_dtype(dt)


def test_quantize_u16_equals_numpy_restatement():
    """Bitwise np.rint(np.clip(x, 0, 1) * 65535) in float32 (round half to even): every code value's
    img_as_float, the float32 neighbours of every half-way point, random values around [0, 1], and
    the specials (NaN -> 0, as in the kernels)."""
    codes = (np.arange(65536, dtype=np.float64) / 65535).astype(np.float32)
    half = ((np.arange(65535, dtype=np.float64) + 0.5) / 65535).astype(np.float32)
    x = np.concatenate([codes, half, np.nextafter(half, np.float32(0)), np.nextafter(half, np.float32(1)),
                        np.random.RandomState(0).uniform(-0.2, 1.2, 200000).astype(np.float32),
                        np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1.0, 1e30, -1e30], np.float32)])
    got = models.quantize_u16(torch.from_numpy(x))
    assert got.dtype == torch.uint16
    finite = np.nan_to_num(x, nan=0.0)
    want = np.rint(np.clip(finite, np.float32(0), np.float32(1)) * np.float32(65535)).astype(np.uint16)
    assert np.array_equal(got.numpy(), want)
    assert np.array_equal(got.numpy()[:65536], np.arange(65536))        # every code round-trips
    assert got.numpy()[-8:].tolist() == [0, 65535, 0, 0, 0, 65535, 65535, 0]
