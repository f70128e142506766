"""The frozen model file on the CPU: checkpoint.freeze_model and read_frozen_model round-trip every
model kind at default and non-default hyperparameters, the arrays are bit for bit what
models._Prepared folds and keeps, hdrnet_model_create refuses every malformed file with
HDRNET_E_BAD_MODEL before any CUDA call, and the freeze CLI writes where its flags say."""
import ctypes
import json
import os
import struct

import numpy as np
import pytest
import torch

from hdrnet_b200 import _lib, checkpoint, models
from hdrnet_b200.bin import freeze_model as freeze_cli
from hdrnet_b200.bin.run import save_checkpoint

KINDS = checkpoint.FROZEN_KINDS
SMALL = dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8)
# every hyperparameter away from its default, batch norm folded into the coefficient layers
ODD = dict(models.DEFAULT_PARAMS, net_input_size=32, spatial_bin=8, luma_bins=16, channel_multiplier=2,
           guide_complexity=32, batch_norm=True)


def _weights(params, name, seed=3):
    w = models.init_weights(params, seed=seed, model_name=name)
    rng = np.random.RandomState(seed)
    for k in w:   # non-trivial batch-norm statistics, so that the fold shows
        if k.endswith("moving_mean") or k.endswith("BatchNorm/beta"):
            w[k] = rng.randn(*w[k].shape).astype(np.float32) * 0.1
        elif k.endswith("moving_variance"):
            w[k] = rng.rand(*w[k].shape).astype(np.float32) + 0.5
    return w


def _prepared_arrays(w, params, name):
    """What models._Prepared keeps, independently listed: the layers in _coefficient_specs order,
    then the guides' host arrays."""
    prep = models._Prepared(w, params, torch.device("cpu"), getattr(models, name)._nn_guide)
    out = []
    for scope, _, _ in models._coefficient_specs(params):
        wd, bd, _ = prep.layers[scope]
        out += [wd.numpy(), np.zeros(0, np.float32) if bd is None else bd.numpy()]
    for g in prep.guides:
        if name == "HDRNetCurves":
            out += [g.ccm, g.ccm_bias, g.shifts, g.slopes, g.mix, np.float32([g.mix_bias])]
        else:
            out += [g.w1, g.b1, g.w2, np.float32([g.b2])]
    return out


# spatial_bin 3: a grid whose side is no power of two
SB3 = dict(models.DEFAULT_PARAMS, net_input_size=48, spatial_bin=3, guide_complexity=8)


@pytest.mark.parametrize("params", [SMALL, ODD, SB3], ids=["default", "nondefault", "spatial_bin3"])
@pytest.mark.parametrize("name", KINDS)
def test_round_trip_equals_prepared_bitwise(built_lib, tmp_path, name, params):
    params = dict(params, model_name=name)
    w = _weights(params, name)
    path = checkpoint.freeze_model(w, params, str(tmp_path / "m.hdrnet"))
    got = checkpoint.read_frozen_model(path)
    assert got["model_name"] == name
    for k in ("net_input_size", "spatial_bin", "luma_bins", "channel_multiplier"):
        assert got[k] == params[k]
    assert got["guide_width"] == (16 if name == "HDRNetCurves" else params["guide_complexity"])
    want = _prepared_arrays(w, params, name)
    assert len(got["arrays"]) == len(want)
    for a, b in zip(got["arrays"], want):
        assert a.shape == b.shape and a.dtype == np.float32
        assert a.tobytes() == np.ascontiguousarray(b, np.float32).tobytes()
    # the C side's validation accepts the file (without a GPU the device is reached next)
    with open(path, "rb") as f:
        assert _create(f.read()) != _lib.E_BAD_MODEL


def test_batch_norm_is_folded_as_fold_does(tmp_path):
    params = dict(ODD, model_name="HDRNetPointwiseNNGuide")
    w = _weights(params, params["model_name"])
    arrays = checkpoint.read_frozen_model(checkpoint.freeze_model(w, params, str(tmp_path / "m")))["arrays"]
    fw, fb = models._fold(w, "inference/coefficients/splat/conv2", True, False)
    assert arrays[2].tobytes() == fw.tobytes() and arrays[3].tobytes() == fb.tobytes()
    w1, b1 = models._fold(w, "inference/guide/conv1", True, False)
    assert arrays[-4].tobytes() == w1.reshape(3, -1).tobytes() and arrays[-3].tobytes() == b1.tobytes()
    assert arrays[-5].size == 3 * params["luma_bins"] * 4   # prediction bias
    # local conv2 has no bias: an empty array
    assert arrays[2 * (len(models._coefficient_specs(params)) - 2) + 1].size == 0


def _create(blob: bytes) -> int:
    lib = _lib.load()
    handle = ctypes.c_void_p()
    rc = lib.hdrnet_model_create(blob, len(blob), ctypes.byref(handle))
    if rc == _lib.OK:
        lib.hdrnet_model_destroy(handle)
    return rc


def _with_crc(body: bytes) -> bytes:
    return body + struct.pack("<I", checkpoint.crc32c(body))


@pytest.fixture(scope="module")
def good_blob(tmp_path_factory):
    params = dict(SMALL, model_name="HDRNetPointwiseNNGuide")
    path = tmp_path_factory.mktemp("frozen") / "m.hdrnet"
    checkpoint.freeze_model(_weights(params, params["model_name"]), params, str(path))
    return path.read_bytes()


def test_a_valid_file_passes_validation(built_lib, good_blob):
    # with a GPU the object is created; without one the validation passes and the device is reached
    assert _create(good_blob) != _lib.E_BAD_MODEL


def _mutations(blob):
    body = blob[:-4]
    flipped = bytearray(blob)
    flipped[len(blob) // 2] ^= 0x10
    yield "truncated", blob[:-100]
    yield "empty", b""
    yield "flipped byte", bytes(flipped)
    yield "wrong magic", _with_crc(b"HDRNETXX" + body[8:])
    yield "future version", _with_crc(body[:8] + struct.pack("<I", checkpoint.FROZEN_VERSION + 1) + body[12:])
    yield "unknown kind", _with_crc(body[:12] + struct.pack("<I", 7) + body[16:])
    yield "too few arrays", _with_crc(body[:36] + struct.pack("<I", struct.unpack_from("<I", body, 36)[0] - 1)
                                      + body[40:])
    yield "trailing bytes", _with_crc(body + b"\0\0\0\0")
    yield "too many arrays", _with_crc(body[:36] + struct.pack("<I", struct.unpack_from("<I", body, 36)[0] + 1)
                                       + body[40:])


def test_malformed_files_are_refused_without_a_gpu(built_lib, good_blob):
    for what, blob in _mutations(good_blob):
        assert _create(blob) == _lib.E_BAD_MODEL, what
    assert "frozen model" in _lib.error_string(_lib.E_BAD_MODEL)


@pytest.mark.parametrize("case", ["layer", "guide", "hyperparameter"])
def test_shape_mismatches_are_refused(built_lib, case):
    params = dict(SMALL, model_name="HDRNetPointwiseNNGuide")
    arrays = checkpoint.frozen_arrays(_weights(params, params["model_name"]), params)
    hyper = [64, 8, 8, 1, 16]
    if case == "layer":      # splat conv2 with one output channel too many
        arrays[2] = np.zeros(arrays[2].shape[:3] + (arrays[2].shape[3] + 1,), np.float32)
    elif case == "guide":    # w1 transposed
        arrays[-4] = np.ascontiguousarray(arrays[-4].T)
    else:                    # luma_bins that the arrays do not have
        hyper[2] = 16
    assert _create(checkpoint._frozen_bytes(1, hyper, arrays)) == _lib.E_BAD_MODEL
    assert _create(checkpoint._frozen_bytes(1, [64, 8, 8, 1, 16], checkpoint.frozen_arrays(
        _weights(params, params["model_name"]), params))) != _lib.E_BAD_MODEL


def test_reader_refuses_what_the_writer_did_not_write(tmp_path, good_blob):
    for what, blob in _mutations(good_blob):
        if what in ("unknown kind", "too few arrays"):
            continue   # CRC-valid and readable: the shapes are the C side's to check
        p = tmp_path / "bad"
        p.write_bytes(blob)
        with pytest.raises(ValueError):
            checkpoint.read_frozen_model(str(p))


def test_unknown_model_name_is_refused(tmp_path):
    params = dict(SMALL, model_name="HDRNetBogus")
    with pytest.raises(ValueError, match="model_name"):
        checkpoint.freeze_model(models.init_weights(SMALL, seed=0), params, str(tmp_path / "m"))


def test_freeze_cli(tmp_path):
    params = dict(SMALL, model_name="HDRNetGaussianPyrNN")
    w = _weights(params, params["model_name"])
    ckpt = tmp_path / "ckpt"
    save_checkpoint(str(ckpt), params, w)
    out = freeze_cli.main(freeze_cli.build_parser().parse_args([str(ckpt)]))
    assert out == os.path.join(str(ckpt), "frozen_model.hdrnet") and os.path.exists(out)
    other = str(tmp_path / "elsewhere.hdrnet")
    assert freeze_cli.main(freeze_cli.build_parser().parse_args([str(ckpt), "--output", other])) == other
    a, b = checkpoint.read_frozen_model(out), checkpoint.read_frozen_model(other)
    assert a["model_name"] == "HDRNetGaussianPyrNN" and len(a["arrays"]) == len(b["arrays"])
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a["arrays"], b["arrays"]))
    with open(ckpt / "params.json") as f:
        assert json.load(f)["model_name"] == "HDRNetGaussianPyrNN"
    empty = tmp_path / "empty"
    empty.mkdir()
    with pytest.raises(SystemExit, match="no weights.npz"):
        freeze_cli.main(freeze_cli.build_parser().parse_args([str(empty)]))

