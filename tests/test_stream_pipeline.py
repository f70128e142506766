"""CPU tests of the streamed tier's host side (hdrnet_b200/data_pipeline.py): ``source_window``
against a numpy restatement of the reference's _augment_data (np.flip, np.rot90, slicing) on index
images, the choice between the device and streamed tiers with a substituted ``device_budget``, and
the staging slots' size for mixed pixel formats."""
import itertools

import numpy as np
import pytest

from hdrnet_b200 import data_pipeline as dp
from hdrnet_b200.data_pipeline import Draw, source_window


def augment(im, d, oh, ow):
    x = im
    if d.fliplr:
        x = np.flip(x, 1)
    if d.flipud:
        x = np.flip(x, 0)
    x = np.rot90(x, d.rot90)
    assert 0 <= d.crop_y <= x.shape[0] - oh and 0 <= d.crop_x <= x.shape[1] - ow
    return x[d.crop_y:d.crop_y + oh, d.crop_x:d.crop_x + ow]


def check_window(H, W, d, oh, ow):
    im = np.arange(H * W, dtype=np.int64).reshape(H, W)           # every value names its pixel
    y0, x0, h, w = source_window(H, W, d, oh, ow)
    assert (h, w) == ((ow, oh) if d.rot90 % 2 else (oh, ow))
    assert 0 <= y0 and 0 <= x0 and y0 + h <= H and x0 + w <= W
    window = im[y0:y0 + h, x0:x0 + w]
    whole = augment(im, d, oh, ow)
    assert np.array_equal(augment(window, d._replace(crop_y=0, crop_x=0), oh, ow), whole), (H, W, d)
    # the window is exactly the set of pixels the crop reads
    assert sorted(window.ravel()) == sorted(whole.ravel())


def extents(H, W, k):
    return (W, H) if k % 2 else (H, W)


@pytest.mark.parametrize("H,W", [(37, 53), (53, 37), (41, 41), (30, 40)])
def test_every_flip_and_rotation_with_random_and_edge_crops(H, W):
    rng = np.random.RandomState(H * W)
    oh, ow = 20, 30
    n = 0
    for lr, ud, k in itertools.product((False, True), (False, True), range(4)):
        rh, rw = extents(H, W, k)
        if oh > rh or ow > rw:
            continue
        origins = {(0, 0), (rh - oh, rw - ow), (0, rw - ow), (rh - oh, 0),
                   (int((rh - oh) / 2), int((rw - ow) / 2))}                      # corners and the centre
        origins |= {(int(rng.randint(rh - oh + 1)), int(rng.randint(rw - ow + 1))) for _ in range(6)}
        for cy, cx in origins:
            check_window(H, W, Draw(0, lr, ud, k, cy, cx), oh, ow)
        n += 1
    assert n == 16 or (H, W) == (30, 40)         # 30x40 is too short for a 30-column crop when rotated


@pytest.mark.parametrize("H,W", [(20, 30), (30, 20), (25, 25)])
def test_whole_image_crops(H, W):
    for lr, ud, k in itertools.product((False, True), (False, True), range(4)):
        oh, ow = extents(H, W, k)
        assert source_window(H, W, Draw(0, lr, ud, k, 0, 0), oh, ow) == (0, 0, H, W)
        check_window(H, W, Draw(0, lr, ud, k, 0, 0), oh, ow)


def test_sampler_draws_map_to_windows():
    sizes = [(600, 800), (512, 512), (701, 531), (531, 701), (901, 1203)]
    s = dp.Sampler(sizes, 5, (512, 512), shuffle=True, fliplr=True, flipud=True, rotate=True, random_crop=True,
                   seed=3)
    seen = set()
    for step in range(40):
        for d in s.draws(step):
            H, W = sizes[d.index]
            check_window(H, W, d, 512, 512)
            seen.add((d.fliplr, d.flipud, d.rot90))
    assert len(seen) == 16


def test_a_crop_outside_the_source_is_refused():
    with pytest.raises(ValueError, match="outside"):
        source_window(20, 30, Draw(0, False, False, 1, 11, 0), 20, 20)  # rows 11..30 of a 30x20 extent
    with pytest.raises(ValueError, match="rot90"):
        source_window(20, 30, Draw(0, False, False, 4, 0, 0), 10, 10)


# ---- tier selection --------------------------------------------------------------------------------
MARGIN = 2 << 30


def budget(monkeypatch, free):
    calls = []

    def fake(device):
        calls.append(device)
        return free
    monkeypatch.setattr(dp, "device_budget", fake)
    return calls


def test_a_dataset_that_fits_is_device_resident(monkeypatch):
    calls = budget(monkeypatch, MARGIN + 1000)
    assert dp.choose_tier(1000, 10, "cuda:0", MARGIN) == "device"
    assert calls == ["cuda:0"]


def test_a_dataset_that_does_not_fit_is_streamed(monkeypatch):
    budget(monkeypatch, MARGIN + 1000)
    assert dp.choose_tier(1001, 1000, "cuda:0", MARGIN) == "stream"
    assert dp.choose_tier(10 ** 12, 10, "cuda:0", MARGIN) == "stream"


def test_staging_slots_that_do_not_fit_raise_memory_error_with_the_byte_counts(monkeypatch):
    budget(monkeypatch, MARGIN + 1000)
    with pytest.raises(MemoryError, match=r"5000 bytes of device memory .* 1001 bytes of staging slots; "
                                          rf"{MARGIN + 1000} bytes are free and {MARGIN} are kept .* 1000 are available"):
        dp.choose_tier(5000, 1001, "cuda:0", MARGIN)
    budget(monkeypatch, 100)                               # less free than the margin
    with pytest.raises(MemoryError, match=r"so 0 are available"):
        dp.choose_tier(5000, 1, "cuda:0", MARGIN)


def test_cache_bytes_align_every_image():
    ims = [np.zeros((3, 5, 3), np.uint8), np.zeros((3, 5, 3), np.uint16), np.zeros((16, 16, 3), np.float32)]
    assert dp.cache_bytes(ims) == 256 + 256 + 3072


def test_slot_size_takes_the_widest_format_pair():
    oh, ow = 33, 47                                       # 4653 values a window
    a8, a16, a32 = (-(-oh * ow * 3 * n // 256) * 256 for n in (1, 2, 4))
    assert (a8, a16, a32) == (4864, 9472, 18688)
    u8, u16, f32 = np.dtype(np.uint8), np.dtype(np.uint16), np.dtype(np.float32)
    assert dp.slot_bytes({(u8, u8)}, 4, (oh, ow)) == 4 * 2 * a8
    assert dp.slot_bytes({(u8, u16)}, 16, (oh, ow)) == 16 * (a8 + a16)
    assert dp.slot_bytes({(u8, u16), (u16, u8)}, 16, (oh, ow)) == 16 * (a8 + a16)
    assert dp.slot_bytes({(u8, f32), (u16, u16), (u8, u8)}, 3, (oh, ow)) == 3 * (a8 + a32)
    assert dp.slot_bytes({(f32, f32), (u8, u16)}, 3, (ow, oh)) == 3 * 2 * a32
    # the reference's training shapes move 4.19 Mpx a batch: 37.7 MB of u8 / u16 windows
    for B, n in ((16, 512), (4, 1024), (1, 2048)):
        assert dp.slot_bytes({(u8, u16)}, B, (n, n)) == 16 * 512 * 512 * 9
