"""Weight import / export formats (SURVEY.md section 8 row f-4): the TensorFlow V2 checkpoint
reader, the variable-name maps and the freeze step's raw guide dumps.

Parity status: the reference holds no checkpoint and TensorFlow is not installed, so the reader
is checked against the writer in the same module (which follows the published table / bundle
format, CRC-32C included) -- "parity unpinned" against a TensorFlow-produced file.  The guide
dumps are checked against the layout freeze_graph.py:105-185 spells out and against the
parameters the CUDA guide kernels are fed.
"""
import os
import struct

import numpy as np
import pytest
import torch

from hdrnet_b200 import checkpoint as C
from hdrnet_b200 import models
from oracle import model_np as M


def test_crc32c_known_answers():
    assert C.crc32c(b"") == 0
    assert C.crc32c(b"123456789") == 0xE3069283                    # the standard check value
    assert C.crc32c(bytes(32)) == 0x8A9136AA                       # RFC 3720 B.4: 32 zero bytes
    assert C.crc32c(bytes([0xFF] * 32)) == 0x62A8AB43              # RFC 3720 B.4: 32 0xFF bytes
    assert C.crc32c(b"6789", C.crc32c(b"12345")) == 0xE3069283     # incremental


def _assorted(rng):
    t = {f"inference/coefficients/splat/conv{i}/weights": rng.randn(3, 3, 8, 16).astype(np.float32)
         for i in range(1, 5)}
    t.update({f"inference/coefficients/splat/conv{i}/weights/Adam": rng.randn(3, 3, 8, 16).astype(np.float32)
              for i in range(1, 5)})
    t["global_step"] = np.array(12345, np.int64)                   # scalar
    t["beta1_power"] = np.array(0.5, np.float32)
    t["inference/guide/ccm"] = rng.randn(3, 3).astype(np.float32)
    t["misc/bytes"] = rng.randint(0, 255, size=(7, 5)).astype(np.uint8)
    t["misc/empty"] = np.zeros((0, 4), np.float32)
    t["misc/f64"] = rng.randn(11)
    t["misc/i32"] = rng.randint(-9, 9, size=(2, 2, 2)).astype(np.int32)
    for i in range(300):                                           # many keys: several index blocks
        t[f"pad/variable_{i:04d}/weights"] = np.full((2,), i, np.float32)
    return t


def test_checkpoint_round_trip(tmp_path):
    rng = np.random.RandomState(0)
    tensors = _assorted(rng)
    prefix = str(tmp_path / "model.ckpt-42")
    C.write_tf_checkpoint(prefix, tensors)
    assert os.path.exists(prefix + ".index") and os.path.exists(prefix + ".data-00000-of-00001")
    assert C.latest_checkpoint(str(tmp_path)) == prefix
    for src in (prefix, str(tmp_path)):                            # by prefix, or by directory
        got = C.read_tf_checkpoint(src)
        assert sorted(got) == sorted(tensors)
        for k, v in tensors.items():
            assert got[k].dtype == np.asarray(v).dtype and got[k].shape == np.asarray(v).shape, k
            assert np.array_equal(got[k], v), k
    # table framing: magic number in the footer, more than one data block
    idx = open(prefix + ".index", "rb").read()
    assert struct.unpack("<Q", idx[-8:])[0] == 0xDB4775248B80FB57 and len(idx) > 2 * 4096


def test_checkpoint_corruption_is_detected(tmp_path):
    rng = np.random.RandomState(1)
    prefix = str(tmp_path / "model.ckpt-1")
    C.write_tf_checkpoint(prefix, {"inference/a": rng.randn(64).astype(np.float32)})
    data = bytearray(open(prefix + ".data-00000-of-00001", "rb").read())
    data[10] ^= 0x40
    open(prefix + ".data-00000-of-00001", "wb").write(bytes(data))
    with pytest.raises(ValueError, match="tensor checksum"):
        C.read_tf_checkpoint(prefix)
    assert C.read_tf_checkpoint(prefix, verify=False)["inference/a"].shape == (64,)
    idx = bytearray(open(prefix + ".index", "rb").read())
    idx[3] ^= 0x01
    open(prefix + ".index", "wb").write(bytes(idx))
    with pytest.raises(ValueError, match="checksum"):
        C.read_tf_checkpoint(prefix)
    open(prefix + ".index", "wb").write(b"not a table")
    with pytest.raises(ValueError, match="magic"):
        C.read_tf_checkpoint(prefix)
    assert C.latest_checkpoint(str(tmp_path / "nowhere")) is None


def test_model_weights_filter_and_model_round_trip(tmp_path):
    """A model's variables (+ the clutter a training run leaves) through a checkpoint and back:
    the inference weights come out identical, the clutter is gone."""
    p = dict(M.DEFAULT_PARAMS)
    wts = models.init_weights(p, seed=5)
    clutter = {k + "/Adam": v for k, v in wts.items()}
    clutter.update({k + "/Adam_1": v for k, v in wts.items()})
    clutter.update({"global_step": np.array(7, np.int64), "beta1_power": np.array(0.9, np.float32),
                    "train/inference/unused": np.zeros(3, np.float32)})
    prefix = str(tmp_path / "model.ckpt-7")
    C.write_tf_checkpoint(prefix, {**wts, **clutter})
    got = C.model_weights(C.read_tf_checkpoint(prefix, verify=False))
    assert sorted(got) == sorted(wts)
    for k in wts:
        assert np.array_equal(got[k], np.asarray(wts[k], np.float32)), k
    assert C.model_weights({"inference/x:0": np.ones(2)})["inference/x"].dtype == np.float32


def test_legacy_name_upgrade():
    m = C.legacy_name_map()
    assert m["conv2/biases"] == "inference/coefficients/splat/conv2/BatchNorm/beta"   # upgrade.py:33-34
    assert m["conv1/biases"] == "inference/coefficients/splat/conv1/biases"           # first layer: no BN
    assert m["guide/guide/ccm"] == "inference/guide/ccm"
    assert len(m) == 28                                                                # upgrade.py:29-61
    old = {k: np.full((2,), i, np.float32) for i, k in enumerate(m)}
    old["grid_conv2/biases"] = np.array([1.0, 2.0], np.float32)
    old["global_fc3/biases"] = np.array([10.0, 20.0], np.float32)
    new = C.upgrade_legacy_names(old)
    assert np.array_equal(new["inference/coefficients/global/fc3/biases"], [11.0, 22.0])  # upgrade.py:63-67
    # 28 transferred + the summed fc3 bias + (moving_mean, moving_variance) for the 8 batch-normed layers
    assert len(new) == 29 + 16 and all(k.startswith("inference/") for k in new)


def test_upgraded_legacy_weights_load_into_the_model():
    """ADVICE r01: the upgraded dict must be a complete batch-norm checkpoint -- every layer whose
    old bias became BatchNorm/beta needs moving_mean = 0 / moving_variance = 1 (what the reference's
    freshly initialised graph holds, scripts/upgrade.py:88-100) or models._fold raises KeyError."""
    p = dict(M.DEFAULT_PARAMS, batch_norm=True)
    ref = models.init_weights(p, seed=1)
    inv = {v: k for k, v in C.legacy_name_map().items()}
    old = {inv[k]: v for k, v in ref.items() if k in inv}
    old["grid_conv2/biases"] = np.zeros_like(ref["inference/coefficients/global/fc3/biases"])
    old["global_fc3/biases"] = np.asarray(ref["inference/coefficients/global/fc3/biases"])
    new = C.upgrade_legacy_names(old)
    assert sorted(new) == sorted(ref)                      # exactly the variables the BN graph has
    pre = "inference/coefficients"
    for scope, bn in ((f"{pre}/splat/conv1", False), (f"{pre}/splat/conv2", True), (f"{pre}/global/fc1", True),
                      (f"{pre}/local/conv1", True), (f"{pre}/global/fc3", False)):
        w, b = models._fold(new, scope, bn, not bn)
        assert w.shape == np.asarray(ref[scope + "/weights"]).shape and b is not None
    # the fresh statistics fold to (x / sqrt(1 + eps) + beta): no NaNs, scale just under 1
    w, b = models._fold(new, f"{pre}/splat/conv2", True, False)
    ratio = w / np.asarray(ref[f"{pre}/splat/conv2/weights"])
    assert np.allclose(ratio[np.isfinite(ratio)], 1.0 / np.sqrt(1.0 + 1e-3), rtol=1e-6)


@pytest.mark.parametrize("model_name", ["HDRNetCurves", "HDRNetPointwiseNNGuide", "HDRNetGaussianPyrNN"])
def test_guide_bins_layout_and_round_trip_to_the_guide_objects(tmp_path, model_name):
    p = dict(M.DEFAULT_PARAMS, model_name=model_name, batch_norm=True)
    wts = models.init_weights(p, seed=2, model_name=model_name)
    paths = C.export_guide_bins(wts, model_name, str(tmp_path))
    names = sorted(os.path.basename(q) for q in paths)
    g = "inference/guide"
    if model_name == "HDRNetCurves":
        assert names == ["guide_ccm_f32_3x4.bin", "guide_mix_matrix_f32_1x4.bin",
                         "guide_shifts_f32_16x3.bin", "guide_slopes_f32_16x3.bin"]
        sizes = {n: os.path.getsize(tmp_path / n) for n in names}
        assert sizes == {"guide_ccm_f32_3x4.bin": 48, "guide_mix_matrix_f32_1x4.bin": 16,
                         "guide_shifts_f32_16x3.bin": 192, "guide_slopes_f32_16x3.bin": 192}
        raw = np.fromfile(tmp_path / "guide_ccm_f32_3x4.bin", "<f4").reshape(3, 4)
        assert np.array_equal(raw[:, :3], np.asarray(wts[f"{g}/ccm"]).T)              # [out][in | bias]
        assert np.array_equal(raw[:, 3], np.asarray(wts[f"{g}/ccm_bias"]))
        back = C.load_guide_bins(str(tmp_path), model_name)
        (guide,) = models._Prepared(wts, p, torch.device("cpu"), False).guides                      # what the kernels get
        for k in ("ccm", "ccm_bias", "shifts", "slopes", "mix"):
            assert np.array_equal(back[k], getattr(guide, k)), k
        assert back["mix_bias"] == guide.mix_bias
    else:
        levels = [f"{g}/level_{l}" for l in range(3)] if model_name == "HDRNetGaussianPyrNN" else [g]
        assert len(names) == 2 * len(levels)
        back = C.load_guide_bins(str(tmp_path), model_name)
        prep = models._Prepared(wts, p, torch.device("cpu"), "pyramid" if len(levels) == 3 else True)
        assert len(prep.guides) == len(levels)
        for l, (scope, guide) in enumerate(zip(levels, prep.guides)):
            b = back[f"level_{l}"] if len(levels) == 3 else back
            w1, b1, w2, b2, feats = guide.w1, guide.b1, guide.w2, guide.b2, guide.feats
            assert feats == 16 and b["w1"].shape == (3, 16)
            # the freeze step folds in float32, the kernels' packer in float64: 1 ulp apart at most
            np.testing.assert_allclose(b["w1"], w1, rtol=3e-7, atol=0)
            np.testing.assert_allclose(b["b1"], b1, rtol=3e-6, atol=1e-7)
            assert np.array_equal(b["w2"], w2) and b["b2"] == b2


# ---- model_params from a .meta file, and the import CLI -------------------------------------------
def _pb(field, wt, payload):
    key = C._put_varint((field << 3) | wt)
    return key + (C._put_varint(len(payload)) + payload if wt == 2 else payload)


def _const_node(name, dtype, tensor_fields):
    tensor = _pb(1, 0, C._put_varint(dtype)) + tensor_fields
    attr_value = _pb(8, 2, tensor)
    attr = _pb(5, 2, _pb(1, 2, b"value") + _pb(2, 2, attr_value))
    dtype_attr = _pb(5, 2, _pb(1, 2, b"dtype") + _pb(2, 2, _pb(6, 0, C._put_varint(dtype))))
    return _pb(1, 2, _pb(1, 2, name.encode()) + _pb(2, 2, b"Const") + dtype_attr + attr)


def _fake_meta(params):
    nodes = b"" + _pb(1, 2, _pb(1, 2, b"unrelated") + _pb(2, 2, b"NoOp"))
    for k, v in params.items():
        if isinstance(v, bool):
            nodes += _const_node(k, 10, _pb(11, 0, C._put_varint(int(v))) if v else b"")
        elif isinstance(v, int):
            nodes += _const_node(k, 3, _pb(7, 0, C._put_varint(v)))
        elif isinstance(v, float):
            nodes += _const_node(k, 1, _pb(5, 5, struct.pack("<f", v)))
        elif isinstance(v, list):                            # output_resolution: int32 [2]
            shape = _pb(2, 2, _pb(2, 2, _pb(1, 0, C._put_varint(len(v)))))
            if len(set(v)) == 1:                             # TensorFlow stores a repeated value once
                nodes += _const_node(k, 3, shape + _pb(7, 0, C._put_varint(v[0])))
            else:
                nodes += _const_node(k, 3, shape + _pb(4, 2, np.asarray(v, "<i4").tobytes()))
        else:
            nodes += _const_node(k, 7, _pb(8, 2, v.encode()))
    node_list = b"".join(_pb(1, 2, (k + ":0").encode()) for k in params)
    coll = _pb(4, 2, _pb(1, 2, b"model_params") + _pb(2, 2, _pb(1, 2, node_list)))
    other = _pb(4, 2, _pb(1, 2, b"trainable_variables") + _pb(2, 2, _pb(2, 2, _pb(1, 2, b"xyz"))))
    return _pb(1, 2, _pb(1, 2, b"meta_graph_version")) + _pb(2, 2, nodes) + other + coll


def test_model_params_from_meta_and_import_cli(tmp_path):
    p = dict(M.DEFAULT_PARAMS, model_name="HDRNetPointwiseNNGuide", batch_norm=True, learning_rate=1e-4)
    p.pop("weights", None)
    wts = models.init_weights(p, seed=4, model_name=p["model_name"])
    src, dst = tmp_path / "tf", tmp_path / "out"
    prefix = str(src / "model.ckpt-9")
    C.write_tf_checkpoint(prefix, {**wts, "global_step": np.array(9, np.int64)})
    with open(prefix + ".meta", "wb") as f:
        f.write(_fake_meta(p))
    got = C.read_meta_model_params(prefix + ".meta")
    assert got.keys() == p.keys()
    for k, v in p.items():
        assert got[k] == pytest.approx(v) and type(got[k]) is type(v), k
    from hdrnet_b200.bin import import_checkpoint, run
    import argparse
    import_checkpoint.main(argparse.Namespace(checkpoint_dir=str(src), out_dir=str(dst), params=None,
                                              legacy=False, verify=True, guide_bins=True))
    params, loaded = run.load_checkpoint(str(dst))
    assert params["model_name"] == "HDRNetPointwiseNNGuide" and params["batch_norm"] is True
    assert sorted(loaded) == sorted(wts)
    assert all(np.array_equal(loaded[k], np.asarray(wts[k], np.float32)) for k in wts)
    assert os.path.getsize(dst / "guide_conv1.bin") == 16 * 4 * 4
    with pytest.raises(ValueError, match="model_params"):
        open(prefix + ".meta", "wb").write(_pb(2, 2, b""))
        C.read_meta_model_params(prefix + ".meta")


def test_run_py_reads_a_tensorflow_directory_and_debug_pictures(tmp_path):
    from hdrnet_b200.bin import run
    p = dict(M.DEFAULT_PARAMS, crop=[384, 512])
    wts = models.init_weights(p, seed=6)
    prefix = str(tmp_path / "model.ckpt-3")
    C.write_tf_checkpoint(prefix, wts)
    with pytest.raises(FileNotFoundError, match="model_params"):
        run.load_checkpoint(str(tmp_path))                          # no .meta, no params.json
    with open(prefix + ".meta", "wb") as f:
        f.write(_fake_meta(p))
    params, loaded = run.load_checkpoint(str(tmp_path))             # as the reference: run.py:70-85
    assert params == p and sorted(loaded) == sorted(wts)
    assert models._resolve_weights({}) is loaded or sorted(models._resolve_weights({})) == sorted(wts)
    # --debug pictures (run.py:98-133): mosaic geometry and the symmetric normalisation
    rng = np.random.RandomState(0)
    coeffs = rng.randn(16, 16, 8, 3, 4).astype(np.float32)
    guide = rng.rand(20, 30).astype(np.float32)
    im = rng.randint(0, 255, size=(20, 30, 3)).astype(np.uint8)
    pics = run.debug_images(im, coeffs, [guide])
    assert sorted(pics) == ["_coeffs.png", "_guide_0.png", "_input.png"]
    mosaic = pics["_coeffs.png"]
    assert mosaic.shape == (16 * 8, 16 * 4 * 3) and mosaic.dtype == np.uint8
    m = np.abs(coeffs).max()
    z, y, o, i, x = 5, 3, 2, 1, 7                                   # [gd, gh, no, ni, gw] ordering
    want = np.rint(np.clip((coeffs[y, x, z, o, i] + m) / (2 * m), 0, 1) * 255)
    assert mosaic[z * 16 + y, (o * 4 + i) * 16 + x] == want
    assert pics["_guide_0.png"].max() == 255 and pics["_guide_0.png"].min() >= 127   # guide >= 0
    assert np.array_equal(pics["_input.png"], im[:, :, ::-1])
    # the pyramid model's 'multiscale' pictures (run.py:108-117): channels side by side, [H, C * W]
    level = rng.rand(10, 15, 3).astype(np.float32)
    pics = run.debug_images(im, coeffs, [guide], [level])
    assert "_ms_0.png" in pics and pics["_ms_0.png"].shape == (10, 45)
    mm = np.abs(level).max()
    assert pics["_ms_0.png"][4, 2 * 15 + 7] == np.rint(np.clip((level[4, 7, 2] + mm) / (2 * mm), 0, 1) * 255)


# ---- a checkpoint assembled byte by byte from the format specifications ---------------------------
BUNDLE_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tf_bundle")
INDEX_SHA = "ff14f7a6014e328bf5ef23e6f1a8fa2a2a66b4cb3da8491bc22d5f4b93fcaa4e"
DATA_SHA = "82e81f7c01f0ab8f0b4d08920d53698ac4ffa77d25d2457f1c51e62c1a28f71b"


def test_reads_the_hand_assembled_tensor_bundle():
    """tests/golden/tf_bundle/ is written by tests/golden/make_tf_bundle_fixture.py, an independent
    statement of the LevelDB table + tensor-bundle formats (bit-wise CRC-32C, literal protobuf bytes,
    prefix-compressed keys, two data blocks) that shares no code with hdrnet_b200/checkpoint.py.
    The committed bytes are pinned by their SHA-256; the reader must return exactly the values the
    generator lists, with every block and tensor checksum verified."""
    import hashlib
    with open(os.path.join(BUNDLE_DIR, "model.ckpt-7.index"), "rb") as f:
        index = f.read()
    with open(os.path.join(BUNDLE_DIR, "model.ckpt-7.data-00000-of-00001"), "rb") as f:
        data = f.read()
    assert len(index) == 272 and len(data) == 76
    assert index[-8:] == bytes.fromhex("57fb808b247547db")                    # table magic, little-endian
    assert hashlib.sha256(index).hexdigest() == INDEX_SHA and hashlib.sha256(data).hexdigest() == DATA_SHA
    v = C.read_tf_checkpoint(BUNDLE_DIR, verify=True)                         # via the `checkpoint` state file
    assert sorted(v) == ["global_step", "inference/coefficients/splat/conv1/biases", "inference/guide/ccm"]
    assert v["global_step"].dtype == np.int64 and v["global_step"].shape == () and int(v["global_step"]) == 1234567
    assert v["inference/coefficients/splat/conv1/biases"].tolist() == [0.5, -0.25, 1.0, 2.0, -3.5, 0.125, 100.0, -0.0078125]
    assert v["inference/guide/ccm"].dtype == np.float32
    assert v["inference/guide/ccm"].tolist() == [[1.0, 0.0625, -0.0625], [0.03125, 0.96875, 0.0], [-0.015625, 0.25, 0.75]]
    w = C.model_weights(v)                                                     # run.py:92 scope filter
    assert sorted(w) == ["inference/coefficients/splat/conv1/biases", "inference/guide/ccm"]


META_SHA = "b1eccc63d615d9eb5f7d37487fdc6dc1a891a102cc98dcc914a2721879f06a4b"


def test_reads_the_hand_assembled_meta_graph():
    """tests/golden/tf_bundle/model.ckpt-7.meta is written by tests/golden/make_tf_meta_fixture.py from
    the public .proto definitions (its own varint / tag arithmetic; no code shared with the module):
    train.py's model_params (hdrnet/bin/train.py:60-63, :224-252) as Const nodes the way
    tensor_util.make_tensor_proto encodes python values -- PACKED int_val / float_val / bool_val,
    string_val, an empty shape message for scalars, tensor_content for the 2-vector, a negative int32
    as a ten-byte varint, a False flag -- between a placeholder, other constants, an op with inputs,
    meta_info_def, saver_def and two other collections.  The reader must return exactly these
    values with these python types (what utils.get_model_params returns, hdrnet/utils.py:19-23)."""
    import hashlib
    path = os.path.join(BUNDLE_DIR, "model.ckpt-7.meta")
    with open(path, "rb") as f:
        raw = f.read()
    assert len(raw) == 1414 and hashlib.sha256(raw).hexdigest() == META_SHA
    got = C.read_meta_model_params(path)
    want = {"model_name": "HDRNetPointwiseNNGuide", "data_pipeline": "ImageFilesDataPipeline",
            "net_input_size": 256, "output_resolution": [512, 768], "batch_norm": True,
            "channel_multiplier": 1, "guide_complexity": 16, "luma_bins": 8, "spatial_bin": 16,
            "learning_rate": float(np.float32(0.0001)), "crop_offset": -3, "use_hdrp": False}
    assert list(got) == list(want)                                  # collection order
    for k, v in want.items():
        assert got[k] == v and type(got[k]) is type(v), (k, got[k])
    params, weights = C.import_checkpoint(BUNDLE_DIR, verify=True)  # the directory as run.py takes it (:70-85)
    assert params == want and sorted(weights) == ["inference/coefficients/splat/conv1/biases", "inference/guide/ccm"]
    from hdrnet_b200 import models
    assert hasattr(models, params["model_name"])                    # run.py:82-85


def test_hand_assembled_bundle_corruption_is_detected(tmp_path):
    import shutil
    for victim, offset, what in (("model.ckpt-7.data-00000-of-00001", 20, "tensor checksum"),
                                 ("model.ckpt-7.index", 30, "checksum")):
        d = tmp_path / victim.replace(".", "_")
        shutil.copytree(BUNDLE_DIR, d)
        raw = bytearray((d / victim).read_bytes())
        raw[offset] ^= 0x40
        (d / victim).write_bytes(bytes(raw))
        with pytest.raises(ValueError, match=what):
            C.read_tf_checkpoint(str(d), verify=True)
