"""The training-batch kernel (hdrnet_train_batch_f32, csrc/train_batch.cu) against a numpy
restatement of the reference's _augment_data (hdrnet/data_pipeline.py:126-171): np.flip, np.rot90,
slicing and TF1's nearest-neighbour map src = min(floor(dst * (float32)in / out), in - 1).  Every
comparison is bit-exact.  Hand-checked pixels pin each mapping before the restatement is trusted;
a buffer-contract case checks that the kernel writes all of its output and nothing else; the error
codes are checked without a device."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

from hdrnet_b200 import _lib
from hdrnet_b200.data_pipeline import Draw, train_batch

gpu = pytest.mark.gpu


# ---- the numpy restatement ----------------------------------------------------------------------
def to_float(a):
    """tf.to_float(x) / wl in float32."""
    if a.dtype == np.uint8:
        return a.astype(np.float32) / np.float32(255.0)
    if a.dtype == np.uint16:
        return a.astype(np.float32) / np.float32(65535.0)
    return a.astype(np.float32)


def augment(im, d, oh, ow):
    x = im
    if d.fliplr:
        x = np.flip(x, 1)
    if d.flipud:
        x = np.flip(x, 0)
    x = np.rot90(x, d.rot90)
    assert 0 <= d.crop_y <= x.shape[0] - oh and 0 <= d.crop_x <= x.shape[1] - ow
    return x[d.crop_y:d.crop_y + oh, d.crop_x:d.crop_x + ow]


def nearest_tf1(crop, S):
    oh, ow = crop.shape[:2]
    ys = np.minimum(np.floor(np.arange(S, dtype=np.float32) * (np.float32(oh) / np.float32(S))).astype(np.int64), oh - 1)
    xs = np.minimum(np.floor(np.arange(S, dtype=np.float32) * (np.float32(ow) / np.float32(S))).astype(np.int64), ow - 1)
    return crop[ys][:, xs]


def expected(inputs, targets, draws, oh, ow, S):
    fin = np.stack([to_float(augment(a, d, oh, ow)) for a, d in zip(inputs, draws)])
    fout = np.stack([to_float(augment(b, d, oh, ow)) for b, d in zip(targets, draws)])
    low = np.stack([nearest_tf1(f, S) for f in fin])
    return fin, fout, low


def run(inputs, targets, draws, oh, ow, S):
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in inputs]
    devt = [torch.from_numpy(np.ascontiguousarray(b)).cuda() for b in targets]
    return [t.cpu().numpy() for t in train_batch(dev, devt, draws, (oh, ow), S)]


def check(inputs, targets, draws, oh, ow, S):
    got = run(inputs, targets, draws, oh, ow, S)
    for name, g, w in zip(("image_input", "image_output", "lowres_input"), got, expected(inputs, targets, draws, oh, ow, S)):
        assert g.shape == w.shape, name
        bad = g.view(np.uint32) != w.view(np.uint32)
        assert not bad.any(), f"{name}: {int(bad.sum())} elements differ, first at {np.argwhere(bad)[0].tolist()}"
    return got


def image(rng, H, W, dtype):
    if dtype == np.float32:
        return rng.rand(H, W, 3).astype(np.float32)
    return rng.randint(0, np.iinfo(dtype).max + 1, size=(H, W, 3)).astype(dtype)


def draw(fliplr=False, flipud=False, rot90=0, crop_y=0, crop_x=0):
    return Draw(0, fliplr, flipud, rot90, crop_y, crop_x)


# ---- hand-checked pixels ------------------------------------------------------------------------
@gpu
def test_hand_checked_mappings():
    H, W = 5, 7
    y, x, c = np.meshgrid(np.arange(H), np.arange(W), np.arange(3), indexing="ij")
    src = (100 * y + 10 * x + c).astype(np.float32)          # every value names its pixel
    cases = {  # (draw, rotated extent, out[i, j] -> in[...])
        "identity": (draw(), (H, W), lambda i, j: (i, j)),
        "fliplr": (draw(fliplr=True), (H, W), lambda i, j: (i, W - 1 - j)),
        "flipud": (draw(flipud=True), (H, W), lambda i, j: (H - 1 - i, j)),
        "rot90 k=1": (draw(rot90=1), (W, H), lambda i, j: (j, W - 1 - i)),
        "rot90 k=2": (draw(rot90=2), (H, W), lambda i, j: (H - 1 - i, W - 1 - j)),
        "rot90 k=3": (draw(rot90=3), (W, H), lambda i, j: (H - 1 - j, i)),
        "fliplr then k=1": (draw(fliplr=True, rot90=1), (W, H), lambda i, j: (j, i)),
    }
    for name, (d, (rh, rw), m) in cases.items():
        fin, fout, _ = run([src], [src + 0.5], [d], rh, rw, 4)
        for i, j in ((0, 0), (1, 2), (rh - 1, 0), (0, rw - 1), (rh - 1, rw - 1)):
            sy, sx = m(i, j)
            assert fin[0, i, j].tolist() == src[sy, sx].tolist(), (name, i, j)
            assert fout[0, i, j].tolist() == (src[sy, sx] + 0.5).tolist(), (name, i, j)
    # a crop on the rotated extent: k = 1, origin (2, 1) of the 7 x 5 rotated image
    fin, _, _ = run([src], [src], [draw(rot90=1, crop_y=2, crop_x=1)], 3, 2, 2)
    assert fin[0, 0, 0].tolist() == src[1, W - 1 - 2].tolist() and fin[0, 2, 1].tolist() == src[2, W - 1 - 4].tolist()


@gpu
def test_hand_checked_nearest_network_input_and_normalisation():
    rng = np.random.RandomState(0)
    im = image(rng, 512, 512, np.uint16)
    fin, _, low = run([im], [im], [draw()], 512, 512, 256)
    for dy, dx in ((0, 0), (1, 1), (100, 37), (255, 255)):        # 512 -> 256: src = 2 dst
        assert low[0, dy, dx].tolist() == fin[0, 2 * dy, 2 * dx].tolist()
    assert fin[0, 3, 4, 1] == np.float32(im[3, 4, 1]) / np.float32(65535.0)
    # 300 -> 256 (S does not divide the crop): src = floor(dst * 1.171875)
    im8 = image(rng, 300, 300, np.uint8)
    fin, _, low = run([im8], [im8], [draw()], 300, 300, 256)
    for dst, src in ((0, 0), (1, 1), (6, 7), (7, 8), (255, 298)):
        assert low[0, dst, dst].tolist() == fin[0, src, src].tolist()
    assert fin[0, 0, 0, 0] == np.float32(im8[0, 0, 0]) / np.float32(255.0)


# ---- against the restatement --------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.float32])
def test_all_flip_rotate_combinations(dtype):
    """Every one of the 16 flip / rotation combinations on an odd-sized, non-square source, random
    crops, S not dividing the crop."""
    rng = np.random.RandomState(1)
    H, W, oh, ow, S = 37, 53, 20, 30, 16
    inputs, targets, draws = [], [], []
    for lr, ud, k in itertools.product((False, True), (False, True), range(4)):
        rh, rw = (W, H) if k % 2 else (H, W)
        oh_k, ow_k = oh, ow
        if oh_k > rh or ow_k > rw:
            continue
        inputs.append(image(rng, H, W, dtype))
        targets.append(image(rng, H, W, dtype))
        draws.append(draw(lr, ud, k, int(rng.randint(rh - oh + 1)), int(rng.randint(rw - ow + 1))))
    assert len(draws) == 16
    check(inputs, targets, draws, oh, ow, S)


@gpu
def test_centre_random_and_whole_image_crops():
    rng = np.random.RandomState(2)
    oh, ow, S = 24, 40, 8
    cases = []
    for k in range(4):
        for H, W in ((oh, ow), (ow, oh), (31, 45), (45, 61)):
            rh, rw = (W, H) if k % 2 else (H, W)
            if oh > rh or ow > rw:
                continue
            cases.append((H, W, draw(rot90=k, crop_y=int((rh - oh) / 2), crop_x=int((rw - ow) / 2))))   # centre
            cases.append((H, W, draw(fliplr=True, rot90=k, crop_y=int(rng.randint(rh - oh + 1)),
                                     crop_x=int(rng.randint(rw - ow + 1)))))
    whole = [c for c in cases if ((c[1], c[0]) if c[2].rot90 % 2 else (c[0], c[1])) == (oh, ow)]
    assert len(whole) >= 8                                          # the crop equal to the rotated image
    ims = [image(rng, H, W, np.uint8) for H, W, _ in cases]
    check(ims, [image(rng, H, W, np.uint16) for H, W, _ in cases], [c[2] for c in cases], oh, ow, S)


@gpu
def test_ragged_batch_of_mixed_formats():
    """40 samples (two launches of the kernel's 32-descriptor blocks), each with its own extent and
    its own input and target formats; the network input larger than the crop."""
    rng = np.random.RandomState(3)
    oh, ow, S = 33, 47, 64
    dtypes = [np.uint8, np.uint16, np.float32]
    inputs, targets, draws = [], [], []
    for b in range(40):
        H, W = int(rng.randint(48, 90)), int(rng.randint(48, 90))
        k = int(rng.randint(4))
        rh, rw = (W, H) if k % 2 else (H, W)
        inputs.append(image(rng, H, W, dtypes[b % 3]))
        targets.append(image(rng, H, W, dtypes[(b // 3) % 3]))
        draws.append(draw(bool(rng.randint(2)), bool(rng.randint(2)), k, int(rng.randint(rh - oh + 1)),
                          int(rng.randint(rw - ow + 1))))
    check(inputs, targets, draws, oh, ow, S)


@gpu
def test_training_size_batch():
    """The reference's training size: 16 x 512² crops of larger u8 / u16 sources, 256² network input."""
    rng = np.random.RandomState(4)
    inputs, targets, draws = [], [], []
    for b in range(16):
        H, W = 600 + 7 * b, 700 - 5 * b
        k = b % 4
        rh, rw = (W, H) if k % 2 else (H, W)
        inputs.append(image(rng, H, W, np.uint8))
        targets.append(image(rng, H, W, np.uint16))
        draws.append(draw(b % 2 == 1, b % 3 == 1, k, int(rng.randint(rh - 511)), int(rng.randint(rw - 511))))
    check(inputs, targets, draws, 512, 512, 256)


# ---- buffer contract ----------------------------------------------------------------------------
@gpu
def test_buffer_contract():
    """Outputs are guarded views, filled with NaN bytes in one run and 0x5A in the other: they must
    be bitwise equal across the runs, the guards and the sources untouched."""
    from test_buffer_contract_gpu import PAT_A, PAT_B, Harness

    rng = np.random.RandomState(5)
    oh, ow, S = 29, 37, 19
    srcs = [(image(rng, 40, 50, np.uint8), image(rng, 40, 50, np.uint16)),
            (image(rng, 61, 43, np.float32), image(rng, 61, 43, np.uint8)),
            (image(rng, 45, 45, np.uint16), image(rng, 45, 45, np.float32))]
    draws = [draw(True, False, 1, 3, 2), draw(False, True, 2, 10, 1), draw(True, True, 3, 4, 0)]
    runs = []
    for fill in (PAT_A, PAT_B):
        h = Harness(fill)
        ins = [h.input(a) for a, _ in srcs]
        tgs = [h.input(b) for _, b in srcs]
        out = (h.alloc((3, oh, ow, 3), what="image_input"), h.alloc((3, oh, ow, 3), what="image_output"),
               h.alloc((3, S, S, 3), what="lowres_input"))
        train_batch(ins, tgs, draws, (oh, ow), S, out=out)
        h.check(f"train_batch [fill {fill:#04x}]")
        runs.append([t.cpu().numpy() for t in out])
    for a, b in zip(*runs):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and np.isfinite(a).all()
    want = expected([a for a, _ in srcs], [b for _, b in srcs], draws, oh, ow, S)
    for g, w in zip(runs[0], want):
        assert np.array_equal(g.view(np.uint32), w.view(np.uint32))


# ---- error codes (validation runs before any device work) ---------------------------------------
def call(samples, B, outs=(16, 16, 16), oh=8, ow=8, S=4):
    arr = None
    if samples is not None:
        arr = (_lib.TrainSample * len(samples))(*samples)
    return _lib.load().hdrnet_train_batch_f32(None if arr is None else ctypes.cast(arr, ctypes.c_void_p), B,
                                              *outs, oh, ow, S, None)


def sample(**kw):
    s = dict(input=16, target=32, input_fmt=_lib.PX_U8, target_fmt=_lib.PX_U16, H=10, W=12, fliplr=0, flipud=0,
             rot90=0, crop_y=0, crop_x=0)
    s.update(kw)
    return _lib.TrainSample(**s)


def test_error_codes(built_lib):
    assert call(None, 0) == _lib.OK                                   # empty batch: nothing to do
    assert call(None, 1) == _lib.E_NULL_POINTER
    for outs in ((0, 16, 16), (16, 0, 16), (16, 16, 0)):
        assert call([sample()], 1, outs) == _lib.E_NULL_POINTER
    assert call([sample(), sample(input=None)], 2) == _lib.E_NULL_POINTER
    assert call([sample(target=None)], 1) == _lib.E_NULL_POINTER
    for bad in (dict(H=0), dict(W=-3), dict(rot90=4), dict(rot90=-1), dict(crop_y=-1), dict(crop_x=5),
                dict(crop_y=3), dict(rot90=1, crop_x=3), dict(rot90=3, crop_y=5), dict(H=7)):
        assert call([sample(**bad)], 1) == _lib.E_BAD_SHAPE, bad   # 10x12 source, 8x8 crop
    assert call([sample()], -1) == _lib.E_BAD_SHAPE
    for shape in (dict(oh=0), dict(ow=-1), dict(S=0)):
        assert call([sample()], 1, **shape) == _lib.E_BAD_SHAPE
    for fmt in (dict(input_fmt=3), dict(target_fmt=-1)):
        assert call([sample(**fmt)], 1) == _lib.E_UNSUPPORTED
    assert "NULL" in _lib.error_string(call(None, 1))


def test_python_wrapper_refuses_bad_sources():
    cpu = torch.zeros(10, 12, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA"):
        train_batch([cpu], [cpu], [draw()], (8, 8), 4)
    with pytest.raises(ValueError, match=r"\[H, W, 3\]"):
        train_batch([torch.zeros(10, 12, 4, dtype=torch.uint8)], [cpu], [draw()], (8, 8), 4)
    with pytest.raises(ValueError, match="one input and one target"):
        train_batch([cpu], [], [draw()], (8, 8), 4)
