"""Ragged batches without a GPU: the C entry points refuse malformed descriptor arrays with their
error codes before touching a device, inference_images refuses mixed dtypes and devices, and
run.py's --batch_size parses and refuses --debug with more than one image per call."""
import ctypes

import numpy as np
import pytest
import torch

from hdrnet_b200 import _lib, models
from hdrnet_b200.bin import run as run_cli

CURVES = models._CurvesGuide.from_weights(
    models.init_weights(dict(models.DEFAULT_PARAMS, model_name="HDRNetCurves"), seed=0, model_name="HDRNetCurves"))


def _descs(*hw, image=0x1000, out=0x100000):
    arr = (_lib.ImageDesc * max(len(hw), 1))()
    for i, (h, w) in enumerate(hw):
        arr[i] = _lib.ImageDesc(image and image + i * 0x10000, out and out + i * 0x10000, h, w)
    return arr


def _curves(lib, descs, B, in_fmt=_lib.PX_U8, out_fmt=_lib.PX_U8, grid=0x7000000, gd=8):
    return lib.hdrnet_slice_apply_curves_ragged_px_ws(grid, descs, B, in_fmt, out_fmt, 16, 16, gd, *CURVES.args,
                                                      None, 0, None)


def test_slice_apply_ragged_refusals(built_lib):
    lib = built_lib
    assert _curves(lib, None, 0) == _lib.OK                                   # B == 0: nothing to do
    assert _curves(lib, _descs((4, 4)), 0) == _lib.OK
    assert _curves(lib, None, 2) == _lib.E_NULL_POINTER
    assert _curves(lib, _descs((4, 4)), -1) == _lib.E_BAD_SHAPE
    assert _curves(lib, _descs((4, 4), (0, 5)), 2) == _lib.E_BAD_SHAPE
    assert _curves(lib, _descs((4, 4), (5, -1)), 2) == _lib.E_BAD_SHAPE
    assert _curves(lib, _descs((4, 4), (5, 5), image=0), 2) == _lib.E_NULL_POINTER
    assert _curves(lib, _descs((4, 4), (5, 5), out=0), 2) == _lib.E_NULL_POINTER
    assert _curves(lib, _descs((4, 4)), 1, grid=0) == _lib.E_NULL_POINTER
    assert _curves(lib, _descs((4, 4)), 1, gd=0) == _lib.E_BAD_SHAPE
    assert _curves(lib, _descs((4, 4)), 1, in_fmt=7) == _lib.E_UNSUPPORTED
    assert _curves(lib, _descs((4, 4)), 1, out_fmt=-1) == _lib.E_UNSUPPORTED
    # a uint16 result over any image of the call
    d = _descs((4, 4), (4, 4))
    d[1].out = d[0].image
    assert _curves(lib, d, 2, out_fmt=_lib.PX_U16) == _lib.E_UNSUPPORTED
    assert lib.hdrnet_slice_apply_ragged_workspace_bytes(d, 2, 16, 16, 8) == 0


def test_nn_and_lowres_ragged_refusals(built_lib):
    lib = built_lib
    rng = np.random.RandomState(0)
    nn = models._NNGuide(rng.randn(3, 16).astype(np.float32), rng.randn(16).astype(np.float32),
                         rng.randn(16).astype(np.float32), np.float32([0.1]))
    call = lambda d, B, fmt=_lib.PX_U8: lib.hdrnet_slice_apply_nn_ragged_px_ws(
        0x7000000, d, B, fmt, _lib.PX_U8, 16, 16, 8, *nn.args, None, 0, None)
    assert call(None, 0) == _lib.OK
    assert call(None, 1) == _lib.E_NULL_POINTER
    assert call(_descs((3, 0)), 1) == _lib.E_BAD_SHAPE
    assert call(_descs((3, 3)), 1, fmt=9) == _lib.E_UNSUPPORTED
    low = lambda d, B, fmt=_lib.PX_U8, out=0x9000000, S=64: lib.hdrnet_lowres_nearest_ragged_f32(d, B, fmt, out, S, S, None)
    assert low(None, 0) == _lib.OK
    assert low(None, 3) == _lib.E_NULL_POINTER
    assert low(_descs((3, 3), (0, 3)), 2) == _lib.E_BAD_SHAPE
    assert low(_descs((3, 3), image=0), 1) == _lib.E_NULL_POINTER
    assert low(_descs((3, 3)), 1, out=0) == _lib.E_NULL_POINTER
    assert low(_descs((3, 3)), 1, fmt=5) == _lib.E_UNSUPPORTED
    assert low(_descs((3, 3)), 1, S=0) == _lib.E_BAD_SHAPE


def test_model_ragged_refuses_a_bad_handle(built_lib):
    lib = built_lib
    bogus = ctypes.c_void_p(0x1234)
    assert lib.hdrnet_model_run_ragged_px(None, _descs((4, 4)), 1, 1, 1, None, 0, None, 0, None) == _lib.E_BAD_CONTEXT
    assert lib.hdrnet_model_run_ragged_px(bogus, None, 0, 1, 1, None, 0, None, 0, None) == _lib.E_BAD_CONTEXT
    assert lib.hdrnet_model_workspace_bytes_ragged(None, _descs((4, 4)), 1, 1, 1) == 0


def test_inference_images_refuses_mixed_dtypes_and_devices():
    a = torch.zeros((4, 4, 3), dtype=torch.uint8)
    for cls in (models.HDRNetCurves, models.HDRNetPointwiseNNGuide, models.HDRNetGaussianPyrNN):
        with pytest.raises(TypeError, match="mixes dtypes"):
            cls.inference_images([a, torch.zeros((5, 4, 3), dtype=torch.uint16)], {})
        with pytest.raises(ValueError, match="spans devices"):
            cls.inference_images([a, torch.zeros((5, 4, 3), dtype=torch.uint8, device="meta")], {})
        with pytest.raises(TypeError, match="list"):
            cls.inference_images(a, {})
        with pytest.raises(ValueError, match=r"\[H, W, 3\]"):
            cls.inference_images([torch.zeros((4, 4), dtype=torch.uint8)], {})
        with pytest.raises(TypeError, match="out_dtype"):
            cls.inference_images([a], {}, out_dtype=torch.int32)
        with pytest.raises(_lib.HdrnetLibraryError, match="no CPU path"):
            cls.inference_images([a], {})
        assert cls.inference_images([], {}) == []


def test_run_cli_batch_size_flag():
    parser = run_cli.build_parser()
    assert parser.parse_args(["c", "i", "o"]).batch_size == 1
    assert parser.parse_args(["c", "i", "o", "--batch_size", "8"]).batch_size == 8
    with pytest.raises(ValueError, match="--batch_size 1"):
        run_cli.main(parser.parse_args(["c", "i", "o", "--batch_size", "2", "--debug"]))
    with pytest.raises(ValueError, match="at least 1"):
        run_cli.main(parser.parse_args(["c", "i", "o", "--batch_size", "0"]))
