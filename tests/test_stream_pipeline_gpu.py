"""The streamed tier of ImageFilesDataPipeline (hdrnet_b200/data_pipeline.py) against the device
tier: the decoded pairs stay on the host and each batch's crop windows are staged to the device, and
every batch must be bitwise the device tier's.  The tiers are forced by substituting
``data_pipeline.device_budget``; the pairs are handed in through ``load_pairs``.  Covered: a ragged
set of u8 / u16 / f32 sources of odd, non-square sizes with shuffling and every augmentation, B not
dividing n and B > 32; steps out of order (resume, going back, repeats); a slow consumer; a side
stream; the device memory the tier takes; the threads after ``close()``; and the training CLI
(20 steps, and 10 + resume + 10, equal to the device tier's checkpoint)."""
import math
import os
import threading

import cv2
import numpy as np
import pytest
import torch

from hdrnet_b200 import checkpoint, data_pipeline as dp, models
from hdrnet_b200.bin import train

pytestmark = pytest.mark.gpu

OH, OW, S = 24, 40, 16
N = 37
DTYPES = [np.uint8, np.uint16, np.float32]


def image(rng, H, W, dtype):
    if dtype == np.float32:
        return rng.rand(H, W, 3).astype(np.float32)
    return rng.randint(0, np.iinfo(dtype).max + 1, size=(H, W, 3)).astype(dtype)


@pytest.fixture(scope="module")
def pairs():
    """N pairs of odd, non-square sizes; each pair's input and target formats vary independently."""
    rng = np.random.RandomState(11)
    inputs, targets = [], []
    for i in range(N):
        H, W = 2 * int(rng.randint(23, 60)) + 1, 2 * int(rng.randint(23, 60)) + 1
        if H == W:
            W += 2
        inputs.append(image(rng, H, W, DTYPES[i % 3]))
        targets.append(image(rng, H, W, DTYPES[(i // 3) % 3]))
    return [f"{i:02d}" for i in range(N)], inputs, targets, "pairs"


def staging(data, B):
    _, inputs, targets, _ = data
    return dp.STREAM_SLOTS * dp.slot_bytes({(a.dtype, b.dtype) for a, b in zip(inputs, targets)}, B, (OH, OW))


def force(monkeypatch, tier, staging_bytes):
    free = (1 << 50) if tier == "device" else dp.MEMORY_MARGIN + staging_bytes
    monkeypatch.setattr(dp, "device_budget", lambda device: free)


def pipeline(monkeypatch, data, tier, B, nthreads=3, **kw):
    monkeypatch.setattr(dp, "load_pairs", lambda path, nthreads=1: data)
    force(monkeypatch, tier, staging(data, B))
    args = dict(batch_size=B, output_resolution=(OH, OW), shuffle=True, fliplr=True, flipud=True, rotate=True,
                random_crop=True, params={"net_input_size": S}, nthreads=nthreads, seed=4)
    args.update(kw)
    p = dp.ImageFilesDataPipeline("unused", **args)
    assert p.tier == tier
    return p


def assert_same(got, want, what):
    for k in ("image_input", "image_output", "lowres_input"):
        a, b = got[k], want[k]
        assert a.shape == b.shape, (what, k)
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (what, k)


@pytest.mark.parametrize("B", [36, 5])
def test_streamed_batches_equal_the_device_tier_for_three_epochs(monkeypatch, pairs, B):
    dev = pipeline(monkeypatch, pairs, "device", B)
    with pipeline(monkeypatch, pairs, "stream", B) as st:
        assert st.dataset_bytes > st.staging_bytes
        steps = math.ceil(3 * N / B) + 1
        for step in range(steps):
            assert_same(st.batch(step), dev.batch(step), step)


def test_steps_out_of_order(monkeypatch, pairs):
    B = 6
    dev = pipeline(monkeypatch, pairs, "device", B)
    want = {}
    with pipeline(monkeypatch, pairs, "stream", B) as st:
        order = list(range(11)) + [0, 1, 2, 10, 10, 10, 5, 4, 3, 30, 31, 32, 31, 7, 8, 9]
        for step in order:
            want.setdefault(step, dev.batch(step))
            assert_same(st.batch(step), want[step], step)
    with pipeline(monkeypatch, pairs, "stream", B) as st:          # a resumed run: first request at 17
        for step in range(17, 25):
            assert_same(st.batch(step), dev.batch(step), step)


def test_slow_consumer(monkeypatch, pairs):
    B = 33
    dev = pipeline(monkeypatch, pairs, "device", B)
    with pipeline(monkeypatch, pairs, "stream", B) as st:
        for step in range(8):
            torch.cuda._sleep(20_000_000)                            # ~10 ms of the current stream
            got = st.batch(step)
            assert_same(got, dev.batch(step), step)


def test_side_stream(monkeypatch, pairs):
    B = 7
    dev = pipeline(monkeypatch, pairs, "device", B)
    want = [dev.batch(s) for s in range(12)]
    side = torch.cuda.Stream()
    with pipeline(monkeypatch, pairs, "stream", B) as st, torch.cuda.stream(side):
        got = []
        for step in range(12):
            torch.cuda._sleep(2_000_000)
            got.append(st.batch(step))
        for step in range(12):
            assert_same(got[step], want[step], step)
    side.synchronize()


def test_the_dataset_is_not_uploaded(monkeypatch, pairs):
    B = 36
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    slots = dp.STREAM_SLOTS * (-(-(staging(pairs, B) // dp.STREAM_SLOTS) // 512) * 512)   # allocator rounding
    with pipeline(monkeypatch, pairs, "stream", B) as st:
        grown = torch.cuda.memory_allocated() - before
        assert 0 < grown <= slots < st.dataset_bytes
        for step in range(4):
            out = st.batch(step)
        del out
        torch.cuda.synchronize()
        assert torch.cuda.memory_allocated() - before <= slots
    print(f"MEASURE streamed tier: {grown} bytes of device memory for a {st.dataset_bytes}-byte dataset")


def stream_threads():
    return [t for t in threading.enumerate() if t.name.startswith("hdrnet-stream") and t.is_alive()]


def test_close_stops_every_worker_thread(monkeypatch, pairs):
    assert not stream_threads()
    st = pipeline(monkeypatch, pairs, "stream", 5, nthreads=4)
    st.batch(0)
    st.batch(1)
    assert len(stream_threads()) >= 2                               # the producer and at least one packer
    st.close()
    assert not stream_threads()
    st.close()                                                      # idempotent
    with pytest.raises(RuntimeError, match="closed"):
        st.batch(2)
    with pipeline(monkeypatch, pairs, "stream", 5) as st:
        st.batch(0)
    assert not stream_threads()
    dev = pipeline(monkeypatch, pairs, "device", 5)
    dev.close()                                                     # nothing to stop
    assert not stream_threads()


# ---- the training CLI ------------------------------------------------------------------------------
MODEL = ["--net_input_size", "64", "--spatial_bin", "8", "--output_resolution", "128", "128", "--batch_size", "4"]
CLI_FLAGS = ["--fliplr", "--flipud", "--rotate", "--seed", "5"]


@pytest.fixture(scope="module")
def png_dataset(tmp_path_factory):
    root = tmp_path_factory.mktemp("stream_pairs")
    os.makedirs(root / "input")
    os.makedirs(root / "output")
    rng = np.random.RandomState(3)
    names = []
    for i in range(9):
        H, W = 141 + 6 * i, 187 - 4 * i
        name = f"im{i:02d}.png"
        assert cv2.imwrite(str(root / "input" / name), rng.randint(0, 256, size=(H, W, 3)).astype(np.uint8))
        assert cv2.imwrite(str(root / "output" / name), rng.randint(0, 65536, size=(H, W, 3)).astype(np.uint16))
        names.append(name)
    (root / "filelist.txt").write_text("\n".join(names) + "\n")
    return root


def run_cli(monkeypatch, tier, ckpt, data, *flags):
    u8, u16 = np.dtype(np.uint8), np.dtype(np.uint16)
    force(monkeypatch, tier, dp.STREAM_SLOTS * dp.slot_bytes({(u8, u16)}, 4, (128, 128)))
    parser = train.build_parser()
    args = parser.parse_args([str(ckpt), str(data), *MODEL, "--summary_interval", "0",
                              "--checkpoint_interval", "100000", *CLI_FLAGS, *flags])
    t = train.Trainer(args, train.model_params(parser, args))
    assert t.train_data.tier == tier
    t.run()
    assert not stream_threads()
    return checkpoint.read_tf_checkpoint(str(ckpt))


def test_cli_streamed_checkpoints_equal_the_device_tier(monkeypatch, png_dataset, tmp_path):
    want = run_cli(monkeypatch, "device", tmp_path / "device", png_dataset, "--max_steps", "20")
    straight = run_cli(monkeypatch, "stream", tmp_path / "stream", png_dataset, "--max_steps", "20")
    run_cli(monkeypatch, "stream", tmp_path / "resumed", png_dataset, "--max_steps", "10")
    resumed = run_cli(monkeypatch, "stream", tmp_path / "resumed", png_dataset, "--max_steps", "20")
    keys = sorted(k for k in want if k.startswith("inference/"))
    assert sum(k.endswith("/Adam") for k in keys) > 10 and int(want["global_step"]) == 20
    for got in (straight, resumed):
        assert sorted(k for k in got if k.startswith("inference/")) == keys
        assert int(got["global_step"]) == 20
        for k in keys:
            assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), k
