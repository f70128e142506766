"""Data-parallel training on the CPU (gloo, world 2): each rank's shard of a batch, the refusal of a
batch the world size does not divide, the flat-gradient all-reduce, the merge of the guide's batch
moments over ranks, and the divergence guard."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from hdrnet_b200 import data_pipeline as dp
from hdrnet_b200 import parallel
from hdrnet_b200.bin import train

SIZES = [(600, 700), (512, 512), (900, 520), (530, 800), (640, 640)]


def test_shards_tile_the_global_batch():
    for B, N in ((1, 1), (4, 2), (6, 3), (16, 4), (16, 8), (8, 8), (12, 2)):
        args = dict(shuffle=True, fliplr=True, flipud=True, rotate=True, random_crop=True, seed=7)
        whole = dp.Sampler(SIZES, B, (512, 512), **args)
        shards = [dp.Sampler(SIZES, B, (512, 512), shard=(r, N), **args) for r in range(N)]
        for step in (0, 1, 5, 40):
            parts = [s.shard_draws(step) for s in shards]
            assert all(len(p) == B // N for p in parts)
            assert [d for p in parts for d in p] == whole.draws(step), (B, N, step)


def test_batch_not_divisible_by_the_world_is_refused_before_any_data_is_read(tmp_path, monkeypatch):
    missing = tmp_path / "no_such_data"
    with pytest.raises(ValueError, match="not a multiple of the world size 2"):
        dp.ImageFilesDataPipeline(str(missing), batch_size=3, shard=(1, 2))
    for shard in ((2, 2), (-1, 2), (0, 0)):
        with pytest.raises(ValueError, match="0 <= rank < world"):
            dp.Sampler(SIZES, 4, (512, 512), shard=shard)
    monkeypatch.setenv("WORLD_SIZE", "4")
    with pytest.raises(ValueError, match="batch size 6 is not a multiple of the world size 4"):
        train.main([str(tmp_path / "ckpt"), str(missing), "--batch_size", "6"])
    assert not (tmp_path / "ckpt").exists()


def test_merge_moments_is_the_moments_of_the_union():
    rng = np.random.RandomState(0)
    parts = [0.9 + 1e-3 * rng.randn(n, 3) @ rng.randn(3, 3) for n in (5, 1, 300, 77)]
    counts, moms = [], []
    for p in parts:
        counts.append(len(p))
        moms.append(_moments(p))
    got, want = parallel.merge_moments(counts, moms), _moments(np.concatenate(parts))
    # float64 round-off of sums over ~400 pixels, relative to the largest variance (a covariance
    # near 0 cannot hold its own digits)
    np.testing.assert_allclose(got[:3], want[:3], rtol=1e-14)
    np.testing.assert_allclose(got[3:], want[3:], rtol=0, atol=1e-10 * np.abs(want[3:]).max())
    assert np.array_equal(parallel.merge_moments([0, 0], [np.ones(9), np.ones(9)]), np.zeros(9))


def test_without_a_process_group_the_collectives_do_nothing():
    t = [torch.arange(5, dtype=torch.float32)]
    parallel.all_reduce_mean_(t)
    assert torch.equal(t[0], torch.arange(5, dtype=torch.float32))
    m = np.arange(9, dtype=np.float64)
    got, n = parallel.moments_over_ranks(m, 17)
    assert np.array_equal(got, m) and n == 17
    assert np.array_equal(parallel.sum_over_ranks([1.5, 2.0]), [1.5, 2.0])
    parallel.check_ranks_agree([np.ones(3)])


def _moments(px):
    """[mean (3), biased covariance c00 c01 c02 c11 c12 c22], in float64."""
    px = np.asarray(px, np.float64)
    c = np.cov(px.T, bias=True)
    return np.concatenate([px.mean(0), c[np.triu_indices(3)]])


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


# rank r's pixels: 0.9 + 1e-3 noise (a small variance about a large mean), shards of unequal size
PIXELS = 0.9 + 1e-3 * np.random.RandomState(5).randn(2500, 3) @ np.array([[1, 0.3, 0], [0, 1, 0.2], [0, 0, 0.5]])
SPLIT = 1100


def _worker(rank, world, port, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank),
                      MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    parallel.init_distributed("gloo")
    try:
        rng = np.random.RandomState(10 + rank)
        grads = [torch.from_numpy(rng.randn(*s).astype(np.float32)) for s in ((3, 4), (7,), (2, 2, 2))]
        mine = [g.clone() for g in grads]
        parallel.all_reduce_mean_(grads)
        px = PIXELS[:SPLIT] if rank == 0 else PIXELS[SPLIT:]
        mom, n = parallel.moments_over_ranks(_moments(px), len(px))
        sums = parallel.sum_over_ranks([1.0 + rank, 0.0, float(rank == 0)])
        parallel.check_ranks_agree([np.arange(4.0)])
        try:
            parallel.check_ranks_agree([np.arange(4.0) + rank])
            drift = None
        except RuntimeError as e:
            drift = str(e)
        q.put((rank, [g.numpy().tobytes() for g in grads], [m.numpy() for m in mine], mom, n, sums, drift))
    finally:
        parallel.finalize()


def test_collectives_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        results = sorted((q.get(timeout=120) for _ in procs), key=lambda r: r[0])
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join(timeout=10)
    assert all(p.exitcode == 0 for p in procs)
    (_, g0, m0, mom0, n0, s0, d0), (_, g1, m1, mom1, n1, s1, d1) = results
    # the averaged gradients: the same bits on both ranks, and the mean of the two ranks' gradients
    assert g0 == g1
    for got, a, b in zip(g0, m0, m1):
        np.testing.assert_array_equal(np.frombuffer(got, np.float32).reshape(a.shape), (a + b) / 2)
    # the moments of the whole batch, in float64, the same bits on both ranks
    assert n0 == n1 == len(PIXELS)
    assert mom0.tobytes() == mom1.tobytes()
    want = _moments(PIXELS)
    np.testing.assert_allclose(mom0[:3], PIXELS.mean(0), rtol=1e-14)
    np.testing.assert_allclose(mom0[3:], want[3:], rtol=0, atol=1e-10 * np.abs(want[3:]).max())
    assert np.array_equal(s0, [3.0, 0.0, 1.0]) and np.array_equal(s1, s0)
    # the divergence guard: both ranks raise when one rank's state differs
    assert d0 is not None and d1 is not None and "ranks [1] disagree with rank 0" in d0
