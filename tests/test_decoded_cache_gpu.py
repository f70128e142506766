"""The pipelines and the training CLI over the on-disk decoded cache (``decoded_cache`` /
``--decoded_cache``) against the same runs without it: the batches for three epochs, on both tiers
(forced by substituting ``data_pipeline.device_budget``), for both pipelines, from a ragged set of
uint8 / uint16 / float32 files of odd, non-square sizes with every augmentation, whole and as
``shard=(1, 2)``; the device memory each tier takes; the process memory the streamed tier takes
over an epoch; the CLI's checkpoints after 20 steps, after 10 + a resume that decodes nothing + 10,
and after a resume that adds the flag; and two gloo ranks sharing the card."""
import math
import os

import cv2
import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from hdrnet_b200 import checkpoint, data_pipeline as dp
from hdrnet_b200.bin import train

pytestmark = pytest.mark.gpu

OH, OW, S = 24, 40, 16
N = 13
USM = {"blur_sigma": 2.0, "sharpen": 1.5}


def _write(path, im):
    assert cv2.imwrite(str(path), im[:, :, ::-1] if im.ndim == 3 else im)


@pytest.fixture(scope="module")
def ragged(tmp_path_factory):
    """N pairs of odd, non-square sizes: PNG uint8 / uint16 and TIFF float32, input and target formats
    varying independently (a pair's two files share the name, so each pair has one extension)."""
    root = tmp_path_factory.mktemp("ragged")
    os.makedirs(root / "input")
    os.makedirs(root / "output")
    rng = np.random.RandomState(12)
    names = []
    for i in range(N):
        H, W = 2 * int(rng.randint(23, 50)) + 1, 2 * int(rng.randint(23, 50)) + 1
        if H == W:
            W += 2
        ext = ".tiff" if i % 3 == 2 else ".png"
        name = f"im{i:02d}{ext}"
        for sub, k in (("input", i), ("output", i + 1)):
            if ext == ".tiff":
                im = rng.rand(H, W, 3).astype(np.float32)
            elif k % 2:
                im = rng.randint(0, 65536, (H, W, 3)).astype(np.uint16)
            else:
                im = rng.randint(0, 256, (H, W, 3)).astype(np.uint8)
            _write(root / sub / name, im)
        names.append(name)
    (root / "filelist.txt").write_text("\n".join(names) + "\n")
    return root


def force(monkeypatch, tier, staging_bytes):
    free = (1 << 50) if tier == "device" else dp.MEMORY_MARGIN + staging_bytes
    monkeypatch.setattr(dp, "device_budget", lambda device: free)


def pipeline(monkeypatch, kind, data, tier, B, shard, **kw):
    cls = dp.UnsharpMaskDataPipeline if kind == "usm" else dp.ImageFilesDataPipeline
    args = dict(batch_size=B, output_resolution=(OH, OW), shuffle=True, fliplr=True, flipud=True, rotate=True,
                random_crop=True, params={"net_input_size": S}, nthreads=3, seed=4, shard=shard,
                **(USM if kind == "usm" else {}))
    force(monkeypatch, "device", 0)
    staging = cls(str(data), **args).staging_bytes
    force(monkeypatch, tier, staging)
    p = cls(str(data), **args, **kw)
    assert p.tier == tier
    return p


def assert_same(got, want, what):
    for k in ("image_input", "image_output", "lowres_input"):
        assert got[k].shape == want[k].shape, (what, k)
        assert torch.equal(got[k].view(torch.int32), want[k].view(torch.int32)), (what, k)


@pytest.mark.parametrize("shard", [(0, 1), (1, 2)])
@pytest.mark.parametrize("tier", ["device", "stream"])
@pytest.mark.parametrize("kind", ["files", "usm"])
def test_batches_equal_the_run_without_the_cache(monkeypatch, tmp_path, ragged, kind, tier, shard):
    B = 4
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    with pipeline(monkeypatch, kind, ragged, tier, B, shard) as ram:
        grown_ram = torch.cuda.memory_allocated() - base
        with pipeline(monkeypatch, kind, ragged, tier, B, shard, decoded_cache=tmp_path / "cache") as mapped:
            grown_mapped = torch.cuda.memory_allocated() - base - grown_ram
            assert mapped.decoded_cache.built == (N if kind == "usm" else 2 * N)
            assert all(isinstance(a, np.memmap) for a in (mapped.stream.inputs if tier == "stream" else []))
            assert grown_mapped == grown_ram, (grown_mapped, grown_ram)
            for step in range(math.ceil(3 * N / B) + 1):
                assert_same(mapped.batch(step), ram.batch(step), step)


# ---- process memory of the streamed tier -----------------------------------------------------------
def rss_anon():
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("RssAnon:"):
                return int(line.split()[1]) * 1024
    return None                              # not reported by this kernel


def _epoch_rss(data, cache, q):
    """In a process of its own (a heap holding no memory freed earlier): the RssAnon an
    ImageFilesDataPipeline forced onto the streamed tier grows by from before it is made to after
    one epoch of batches."""
    try:
        src = torch.zeros(8, 8, 3, dtype=torch.uint8, device="cuda")     # CUDA and the library loaded first
        dp.train_batch([src], [src], [dp.Draw(0, False, False, 0, 0, 0)], (8, 8), 4)
        torch.cuda.synchronize()
        B, res = 4, (256, 256)
        u16, u8 = np.dtype(np.uint16), np.dtype(np.uint8)
        staging = dp.STREAM_SLOTS * dp.slot_bytes({(u16, u8)}, B, res)
        dp.device_budget = lambda device: dp.MEMORY_MARGIN + staging
        before = rss_anon()
        with dp.ImageFilesDataPipeline(data, batch_size=B, output_resolution=res, shuffle=True, fliplr=True,
                                       rotate=True, nthreads=4, decoded_cache=cache) as p:
            assert p.tier == "stream" and p.staging_bytes == staging
            for step in range(math.ceil(p.nsamples / B)):
                out = p.batch(step)
            torch.cuda.synchronize()
            del out
            q.put((rss_anon() - before, p.dataset_bytes, staging))
    except BaseException as e:
        q.put(repr(e))
        raise


def _in_fresh_process(data, cache):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=_epoch_rss, args=(data, cache, q))
    p.start()
    try:
        got = q.get(timeout=300)
    finally:
        p.join(timeout=60)
    assert isinstance(got, tuple), got
    return got


def test_streamed_tier_over_the_cache_takes_no_dataset_memory(tmp_path):
    if rss_anon() is None:
        pytest.skip("this kernel does not report RssAnon in /proc/self/status")
    root = tmp_path / "big"
    os.makedirs(root / "input")
    os.makedirs(root / "output")
    rng = np.random.RandomState(2)
    names = []
    for i in range(16):
        name = f"{i:02d}.png"
        H, W = 1200 + 8 * i, 1400
        base = rng.randint(0, 65536, (H, 1, 3)).astype(np.uint16) + np.arange(W, dtype=np.uint16)[None, :, None]
        assert cv2.imwrite(str(root / "input" / name), base, [cv2.IMWRITE_PNG_COMPRESSION, 1])
        assert cv2.imwrite(str(root / "output" / name), (base >> 8).astype(np.uint8), [cv2.IMWRITE_PNG_COMPRESSION, 1])
        names.append(name)
    (root / "filelist.txt").write_text("\n".join(names) + "\n")
    cache = str(tmp_path / "cache")
    dp.DecodedCache(cache).open([str(root / sub / n) for n in names for sub in ("input", "output")], 4)
    mapped, dataset, staging = _in_fresh_process(str(root), cache)
    ram, _, _ = _in_fresh_process(str(root), None)
    margin = 48 << 20
    print(f"MEASURE RssAnon over an epoch of the streamed tier, {dataset}-byte dataset, {staging} bytes of "
          f"staging: {mapped} bytes from the decoded cache, {ram} bytes in memory")
    assert mapped <= staging + margin < dataset
    assert ram >= dataset


# ---- the training CLI ------------------------------------------------------------------------------
MODEL = ["--net_input_size", "64", "--spatial_bin", "8", "--output_resolution", "128", "128", "--batch_size", "4"]
CLI_FLAGS = ["--fliplr", "--flipud", "--rotate", "--seed", "5", "--model_name", "HDRNetCurves"]
CLI_USM = ["--data_pipeline", "UnsharpMaskDataPipeline", "--blur_sigma", "2", "--sharpen", "1"]


@pytest.fixture(scope="module")
def png_dataset(tmp_path_factory):
    root = tmp_path_factory.mktemp("cli_pairs")
    os.makedirs(root / "input")
    os.makedirs(root / "output")
    rng = np.random.RandomState(3)
    names = []
    for i in range(9):
        H, W = 141 + 6 * i, 187 - 4 * i
        name = f"im{i:02d}.png"
        _write(root / "input" / name, rng.randint(0, 256, size=(H, W, 3)).astype(np.uint8))
        _write(root / "output" / name, rng.randint(0, 65536, size=(H, W, 3)).astype(np.uint16))
        names.append(name)
    (root / "filelist.txt").write_text("\n".join(names) + "\n")
    return root


def _fail(*args, **kwargs):
    raise AssertionError("decoded on a resume from a warm cache")


def run_cli(ckpt, data, *flags):
    parser = train.build_parser()
    args = parser.parse_args([str(ckpt), str(data), *MODEL, "--summary_interval", "0", "--checkpoint_interval",
                              "100000", "--eval_data_dir", str(data), "--eval_interval", "100000", *CLI_FLAGS,
                              *flags])
    train.check_data_flags(parser, args)
    t = train.Trainer(args, train.model_params(parser, args))
    t.run()
    with open(os.path.join(ckpt, "params.json")) as f:
        assert "decoded_cache" not in f.read()
    return checkpoint.read_tf_checkpoint(str(ckpt))


def assert_checkpoints_equal(got, want, what):
    keys = sorted(k for k in want if k.startswith("inference/"))
    assert sum(k.endswith("/Adam") for k in keys) > 10 and int(want["global_step"]) == 20
    assert sorted(got) == sorted(want) and int(got["global_step"]) == 20, what
    for k in keys:
        assert np.array_equal(np.asarray(got[k]).view(np.uint8), np.asarray(want[k]).view(np.uint8)), (what, k)


@pytest.mark.parametrize("kind", ["files", "usm"])
def test_cli_checkpoints_equal_the_run_without_the_cache(monkeypatch, png_dataset, tmp_path, kind):
    usm = CLI_USM if kind == "usm" else []
    cache = ["--decoded_cache", str(tmp_path / "cache")]
    want = run_cli(tmp_path / "ram", png_dataset, *usm, "--max_steps", "20")
    straight = run_cli(tmp_path / "straight", png_dataset, *usm, *cache, "--max_steps", "20")
    run_cli(tmp_path / "resumed", png_dataset, *usm, *cache, "--max_steps", "10")
    with monkeypatch.context() as m:
        m.setattr(dp, "decode_image", _fail)
        m.setattr(cv2, "imread", _fail)
        resumed = run_cli(tmp_path / "resumed", png_dataset, *usm, *cache, "--max_steps", "20")
    run_cli(tmp_path / "added", png_dataset, *usm, "--max_steps", "10")
    added = run_cli(tmp_path / "added", png_dataset, *usm, *cache, "--max_steps", "20")
    for got, what in ((straight, "straight"), (resumed, "resumed"), (added, "flag added on resume")):
        assert_checkpoints_equal(got, want, what)


def test_two_gloo_ranks_with_the_cache_train_what_they_train_without(png_dataset, tmp_path):
    from test_train_dp_gpu import COMMON, run_ranks
    argv = [str(png_dataset), *COMMON, "--model_name", "HDRNetCurves", "--max_steps", "3"]
    cache = ["--decoded_cache", str(tmp_path / "cache")]
    d_ram = run_ranks([str(tmp_path / "ram"), *argv])
    d_mapped = run_ranks([str(tmp_path / "mapped"), *argv, "--eval_data_dir", str(png_dataset), *cache])
    assert d_mapped == d_ram and len(d_ram[0]) == 3
    a = checkpoint.read_tf_checkpoint(str(tmp_path / "mapped" / "on_stop.ckpt"))
    b = checkpoint.read_tf_checkpoint(str(tmp_path / "ram" / "on_stop.ckpt"))
    assert sorted(a) == sorted(b)
    for k in b:
        if k.startswith("inference/"):
            assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k
    assert len([f for f in os.listdir(tmp_path / "cache") if f.endswith(".px")]) == 18
