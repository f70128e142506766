"""Data-parallel training against one process: two ranks, each building half of every batch of 4
(``shard=(rank, 2)``), must train what one process with the whole batch trains from the same seed.

The ranks share one card over gloo (the gradient all-reduce staged through the host), so the
equivalence runs on a single GPU; the same test over NCCL on two cards runs when two are visible.

What can differ is only the order of float32 sums: a rank's loss is the mean over its 2 images and
the two ranks' gradients are averaged, where one process takes the mean over 4 images; the guide's
batch moments are merged over the ranks in float64.  Reordering a float32 sum changes it by a few
ulps (~1e-6 relative here).  Adam divides each component's first moment by the root of its second,
so every component moves by about the learning rate per step whatever its gradient's scale, and a
relative change e of the gradients changes that step by about e * lr: ~1e-9 over 3 steps at
lr = 1e-3.  That is below the rounding of the variables themselves (values up to ~1 in float32, one
ulp up to 1.2e-7), so the variables differ by a few ulps; the bound, 1e-3 * lr * steps = 3e-6 per
element, is ~25 ulps at 1.0.  (A gradient component within rounding of zero could flip the sign of
its step and move by 2 lr: the bound would catch that, and the seeds here have none.)  The moments m
and v, the moving averages and the logged losses are held to 1e-4 of their own scale.  On an H100
the runs differed by at most 3.7e-7 in the variables, 1.2e-6 of scale in the moments, 0 in the
moving averages and 2.3e-7 in the losses.
"""
import argparse
import hashlib
import json
import os
import socket

import cv2
import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from hdrnet_b200 import checkpoint, models, parallel
from hdrnet_b200.bin import run as run_cli
from hdrnet_b200.bin import train

pytestmark = pytest.mark.gpu

NN, CURVES = "HDRNetPointwiseNNGuide", "HDRNetCurves"
LR, STEPS = 1e-3, 3
COMMON = ["--net_input_size", "64", "--spatial_bin", "8", "--output_resolution", "128", "128", "--batch_size", "4",
          "--summary_interval", "0", "--checkpoint_interval", "100000", "--learning_rate", str(LR),
          "--fliplr", "--rotate", "--seed", "5", "--train_guide"]
FLAGS = {NN: ["--model_name", NN, "--guide_batch_stats"], CURVES: ["--model_name", CURVES]}
N_IMAGES, H, W = 6, 144, 176
G = "inference/guide/"
VAR_ATOL = 1e-3 * LR * STEPS
REL = 1e-4


@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    """u8 inputs and u16 targets rendered by an NN-guide teacher that is not the initial model."""
    root = tmp_path_factory.mktemp("dp_pairs")
    os.makedirs(root / "input")
    os.makedirs(root / "output")
    params = dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8, output_resolution=[128, 128], model_name=NN)
    w = models.init_weights(params, seed=1, model_name=NN)
    rng = np.random.RandomState(3)
    w[G + "conv1/weights"] = (rng.randn(1, 1, 3, 16) * 2.0).astype(np.float32)
    w[G + "conv1/BatchNorm/beta"] = (rng.randn(16) * 0.5).astype(np.float32)
    w[G + "conv2/weights"] = (rng.randn(1, 1, 16, 1) * 0.5).astype(np.float32)
    teacher = dict(params, weights=w)
    names = []
    for i in range(N_IMAGES):
        yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
        base = np.stack([np.sin(3 * xx + i), np.cos(2 * yy - i), xx * yy], axis=2) * 0.4 + 0.5
        im8 = (np.clip(base + 0.1 * rng.randn(H, W, 3), 0, 1) * 255).astype(np.uint8)
        with torch.no_grad():
            out = models.HDRNetPointwiseNNGuide.inference_image(torch.from_numpy(im8[None]).cuda(), teacher,
                                                                out_dtype=torch.float32)[0].cpu().numpy()
        name = f"im{i:02d}.png"
        assert cv2.imwrite(str(root / "input" / name), im8[:, :, ::-1])
        assert cv2.imwrite(str(root / "output" / name), np.rint(np.clip(out, 0, 1) * 65535).astype(np.uint16)[:, :, ::-1])
        names.append(name)
    (root / "filelist.txt").write_text("\n".join(names) + "\n")
    return root


def trainer(argv):
    parser = train.build_parser()
    args = parser.parse_args(argv)
    params = train.model_params(parser, args)
    train.refuse_untrainable(params, args.train_guide, args.guide_batch_stats)
    return train.Trainer(args, params)


def digest(t):
    h = hashlib.sha256()
    for k in sorted(t.weights):
        h.update(t.weights[k].detach().cpu().numpy().tobytes())
    return h.hexdigest()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank(rank, world, port, backend, argv, q):
    """One rank: joins the group, trains (recording a digest of the variables after every step)."""
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank),
                      MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank % torch.cuda.device_count())
    parallel.init_distributed(backend)
    try:
        t = trainer(argv)
        digests, step = [], t.train_step

        def recorded():
            out = step()
            digests.append(digest(t))
            return out

        t.train_step = recorded
        t.run()
        q.put((rank, digests))
    except BaseException as e:
        q.put((rank, repr(e)))
        raise
    finally:
        parallel.finalize()


def run_ranks(argv, world=2, backend="gloo"):
    """Train under ``world`` spawned ranks; returns each rank's per-step digests."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank, args=(r, world, port, backend, argv, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        results = dict(q.get(timeout=600) for _ in procs)
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join(timeout=10)
    for r in range(world):
        assert isinstance(results[r], list), f"rank {r}: {results[r]}"
    assert all(p.exitcode == 0 for p in procs)
    return [results[r] for r in range(world)]


def losses(ckpt_dir):
    with open(os.path.join(ckpt_dir, "train_log.jsonl")) as f:
        return [(rec["step"], rec["loss"]) for rec in map(json.loads, f) if "loss" in rec]


def assert_equivalent(a_dir, b_dir, what):
    """The two runs' on_stop.ckpt and logged losses agree within the module's bounds."""
    a = checkpoint.read_tf_checkpoint(os.path.join(a_dir, "on_stop.ckpt"))
    b = checkpoint.read_tf_checkpoint(os.path.join(b_dir, "on_stop.ckpt"))
    assert sorted(a) == sorted(b)
    assert int(a["global_step"]) == int(b["global_step"])
    worst = {"var": 0.0, "slot": 0.0, "moving": 0.0}
    for k in a:
        if not k.startswith("inference/"):
            continue
        x, y = np.asarray(a[k], np.float64), np.asarray(b[k], np.float64)
        diff = float(np.abs(x - y).max())
        if k.endswith(("/Adam", "/Adam_1")) or "/moving_" in k:
            kind = "moving" if "/moving_" in k else "slot"
            err = diff / max(float(np.abs(y).max()), 1e-30)
            assert err <= REL, f"{what}: {k} differs by {err:.3g} of its scale"
        else:
            kind, err = "var", diff
            assert err <= VAR_ATOL, f"{what}: {k} differs by {err:.3g} > {VAR_ATOL:.3g}"
        worst[kind] = max(worst[kind], err)
    la, lb = losses(a_dir), losses(b_dir)
    assert [s for s, _ in la] == [s for s, _ in lb] and la
    loss_err = max(abs(x - y) / abs(y) for (_, x), (_, y) in zip(la, lb))
    assert loss_err <= REL, f"{what}: logged losses differ by {loss_err:.3g}"
    print(f"MEASURE dp equivalence {what}: variables max|diff| {worst['var']:.3g}, Adam slots {worst['slot']:.3g}, "
          f"moving averages {worst['moving']:.3g} (of scale), losses {loss_err:.3g}", flush=True)
    return a, b


def equivalence(tmp_path, dataset, model, world=2, backend="gloo"):
    argv = [str(dataset), *COMMON, *FLAGS[model], "--max_steps", str(STEPS)]
    one = tmp_path / f"{model}_one"
    many = tmp_path / f"{model}_ranks"
    trainer([str(one), *argv]).run()
    digests = run_ranks([str(many), *argv], world, backend)
    assert len(digests[0]) == STEPS and all(d == digests[0] for d in digests), "ranks drifted apart"
    assert len(set(digests[0])) == STEPS            # and the variables moved every step
    assert_equivalent(str(many), str(one), f"{model} {world} ranks ({backend})")
    return one, many


@pytest.mark.parametrize("model", [NN, CURVES])
def test_two_ranks_on_one_card_train_what_one_process_trains(tmp_path, dataset, model):
    one, many = equivalence(tmp_path, dataset, model)
    with open(many / "params.json") as f:
        assert "world" not in json.dumps(json.load(f))
    if model != NN:
        return
    # bin/run.py on the two-rank checkpoint renders the one-process run's images
    outs = {}
    for d in (one, many):
        outs[d] = tmp_path / (d.name + "_out")
        run_cli.main(argparse.Namespace(checkpoint_dir=str(d), input=str(dataset / "input"), output=str(outs[d]),
                                        lowres_input=None, hdrp=False, debug=False, limit=None))
    names = sorted(os.listdir(outs[one]))
    assert len(names) == N_IMAGES
    for name in names:
        x = cv2.imread(str(outs[one] / name), -1).astype(np.int32)
        y = cv2.imread(str(outs[many] / name), -1).astype(np.int32)
        # uint8 outputs: a float difference far below 1/255 can only move a value across a rounding edge
        assert np.abs(x - y).max() <= 1, name
        assert (x != y).mean() <= 1e-3, name


def test_resume_on_another_world_size(tmp_path, dataset):
    """2 steps on 2 ranks, then 2 more on one process, equal 4 straight steps on one process."""
    argv = [str(dataset), *COMMON, *FLAGS[NN]]
    straight, mixed = tmp_path / "straight", tmp_path / "mixed"
    trainer([str(straight), *argv, "--max_steps", "4"]).run()
    run_ranks([str(mixed), *argv, "--max_steps", "2"])
    t = trainer([str(mixed), *argv, "--max_steps", "4"])
    assert t.step == 2
    t.run()
    assert_equivalent(str(mixed), str(straight), "resume 2 ranks -> 1")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="the NCCL path needs two GPUs; fewer are visible")
def test_nccl_ranks_on_distinct_cards_train_what_one_process_trains(tmp_path, dataset):
    equivalence(tmp_path, dataset, NN, world=2, backend="nccl")
