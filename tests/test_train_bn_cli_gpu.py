"""The training CLI with --batch_norm --coefficient_batch_stats, end to end on a small synthetic dataset
(u8 PNG inputs, u16 PNG targets rendered by a batch-norm HDRNetCurves teacher): a curves student fits
the teacher; 10 steps + resume + 10 steps equal 20 straight steps bit for bit, moving averages and the
betas' Adam slots included; bin/run.py and the frozen model reproduce the in-memory model; the NN and
pyramid models train with all their flags and resume bitwise; two ranks on one card over gloo train
what one process trains.

The bounds are test_train_dp_gpu.py's (1e-4 of scale for Adam's moments and the moving averages), but
the variables are held to 1e-4 rather than 3e-6: the global batch is 4, so fc1 and fc2 normalise over 4
rows, and the two runs' float32 sums, reordered, reach the batch norm's output divided by a spread
taken over 4 values.  On an H100 the variables differed by up to 2.4e-5 (global/fc1/weights)."""
import argparse
import hashlib
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
from hdrnet_b200.frozen import FrozenModel

pytestmark = pytest.mark.gpu

MODEL = ["--net_input_size", "64", "--spatial_bin", "8", "--output_resolution", "128", "128", "--batch_size", "4",
         "--summary_interval", "0", "--checkpoint_interval", "100000", "--batch_norm", "--coefficient_batch_stats"]
PARAMS = dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8, output_resolution=[128, 128], batch_norm=True)
N_IMAGES, H, W = 8, 144, 176
LR, STEPS = 1e-3, 3
VAR_ATOL, REL = 1e-4, 1e-4


@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    root = tmp_path_factory.mktemp("bn_pairs")
    os.makedirs(root / "input")
    os.makedirs(root / "output")
    w = models.init_weights(PARAMS, seed=1)
    rng = np.random.RandomState(7)
    for k in w:       # a teacher whose batch norm is not the identity
        if k.endswith("/moving_mean"):
            w[k] = (0.2 * rng.randn(*w[k].shape)).astype(np.float32)
        elif k.endswith("/moving_variance"):
            w[k] = rng.uniform(0.5, 2.0, w[k].shape).astype(np.float32)
        elif k.endswith("/beta"):
            w[k] = (0.1 * rng.randn(*w[k].shape)).astype(np.float32)
    teacher = dict(PARAMS, weights=w)
    names = []
    for i in range(N_IMAGES):
        yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
        base = np.stack([np.sin(3 * xx + i), np.cos(2 * yy - i), xx * yy], axis=2) * 0.4 + 0.5
        im8 = (np.clip(base + 0.1 * rng.randn(H, W, 3), 0, 1) * 255).astype(np.uint8)
        with torch.no_grad():
            out = models.HDRNetCurves.inference_image(torch.from_numpy(im8[None]).cuda(), teacher,
                                                      out_dtype=torch.float32)[0].cpu().numpy()
        name = f"im{i:02d}.png"
        assert cv2.imwrite(str(root / "input" / name), im8[:, :, ::-1])
        assert cv2.imwrite(str(root / "output" / name), np.rint(np.clip(out, 0, 1) * 65535).astype(np.uint16)[:, :, ::-1])
        names.append(name)
    (root / "filelist.txt").write_text("\n".join(names) + "\n")
    return root


def trainer(argv):
    parser = train.build_parser()
    args = parser.parse_args([str(a) for a in argv])
    params = train.model_params(parser, args)
    train.refuse_untrainable(params, args.train_guide, args.guide_batch_stats, args.coefficient_batch_stats)
    return train.Trainer(args, params)


def losses(ckpt):
    import json
    with open(os.path.join(ckpt, "train_log.jsonl")) as f:
        return [r["loss"] for r in map(json.loads, f) if "loss" in r]


@pytest.fixture(scope="module")
def student(dataset, tmp_path_factory):
    ckpt = tmp_path_factory.mktemp("bn_student")
    t = trainer([ckpt, dataset, *MODEL, "--norandom_crop", "--max_steps", "300"])
    t.run()
    return t, ckpt


def test_student_fits_the_teacher(student):
    _, ckpt = student
    ls = losses(ckpt)
    assert len(ls) == 300 and np.isfinite(ls).all()
    first, last = ls[0], float(np.mean(ls[-10:]))
    print(f"MEASURE train-cli bn student: first {first:.4g} last-10 mean {last:.4g} factor {first / last:.1f}")
    assert first / last >= 10.0


def test_checkpoint_holds_moving_averages_and_beta_slots(student):
    _, ckpt = student
    saved = checkpoint.read_tf_checkpoint(str(ckpt))
    init = models.init_weights(PARAMS, seed=0)
    moving = [k for k in init if "/moving_" in k and k.startswith(train.COEFFS)]
    assert len(moving) == 2 * 7                                  # 7 batch-norm layers at 64^2 / 8
    for k in moving:
        assert not np.array_equal(saved[k], init[k]), k            # they moved
        assert k + "/Adam" not in saved
    betas = [k for k in init if k.endswith("/BatchNorm/beta") and k.startswith(train.COEFFS)]
    assert all(k + "/Adam" in saved and k + "/Adam_1" in saved for k in betas)
    assert all(not np.array_equal(saved[k], init[k]) for k in betas)


def test_run_cli_and_frozen_model_match_the_model_in_memory(student, dataset, tmp_path):
    t, ckpt = student
    out_dir = tmp_path / "out"
    run_cli.main(argparse.Namespace(checkpoint_dir=str(ckpt), input=str(dataset / "input"), output=str(out_dir),
                                    lowres_input=None, hdrp=False, debug=False, limit=None))
    weights = {k: v.detach().cpu().numpy() for k, v in t.weights.items()}
    checkpoint.freeze_model(weights, t.params, str(tmp_path / "m.hdrnet"))
    frozen = FrozenModel(str(tmp_path / "m.hdrnet"))
    for name in sorted(os.listdir(dataset / "input")):
        im8 = torch.from_numpy(np.ascontiguousarray(cv2.imread(str(dataset / "input" / name), -1)[None, :, :, ::-1])).cuda()
        with torch.no_grad():
            want = models.HDRNetCurves.inference_image(im8, t.p)
        assert np.array_equal(cv2.imread(str(out_dir / name), -1)[:, :, ::-1], want[0].cpu().numpy()), name
        assert torch.equal(frozen(im8), want), name
    frozen.close()


def bitwise_resume(tmp_path, dataset, flags):
    trainer([tmp_path / "straight", dataset, *flags, "--max_steps", "20"]).run()
    trainer([tmp_path / "resumed", dataset, *flags, "--max_steps", "10"]).run()
    t = trainer([tmp_path / "resumed", dataset, *flags, "--max_steps", "20"])
    assert t.step == 10
    t.run()
    a = checkpoint.read_tf_checkpoint(str(tmp_path / "straight"))
    b = checkpoint.read_tf_checkpoint(str(tmp_path / "resumed"))
    keys = [k for k in a if k.startswith("inference/")]
    assert sorted(keys) == sorted(k for k in b if k.startswith("inference/"))
    assert any("/BatchNorm/beta/Adam" in k for k in keys) and any("/moving_" in k for k in keys)
    for k in keys:
        assert np.array_equal(np.asarray(a[k]).view(np.uint32), np.asarray(b[k]).view(np.uint32)), k
    ls = losses(tmp_path / "straight")
    assert ls == losses(tmp_path / "resumed") and np.isfinite(ls).all()


@pytest.mark.parametrize("model", ["HDRNetCurves", "HDRNetPointwiseNNGuide", "HDRNetGaussianPyrNN"])
def test_resume_gives_the_uninterrupted_run_bitwise(tmp_path, dataset, model):
    flags = [*MODEL, "--fliplr", "--rotate", "--seed", "5", "--model_name", model]
    if model == "HDRNetPointwiseNNGuide":
        flags += ["--guide_batch_stats"]
    elif model == "HDRNetGaussianPyrNN":
        flags += ["--train_guide", "--guide_batch_stats"]
    bitwise_resume(tmp_path, dataset, flags)


def digest(t):
    h = hashlib.sha256()
    for k in sorted(t.weights):
        h.update(t.weights[k].detach().cpu().numpy().tobytes())
    return h.hexdigest()


def _rank(rank, world, port, argv, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank),
                      MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank % torch.cuda.device_count())
    parallel.init_distributed("gloo")
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


def test_two_ranks_on_one_card_train_what_one_process_trains(tmp_path, dataset):
    argv = [dataset, *MODEL, "--learning_rate", str(LR), "--fliplr", "--rotate", "--seed", "5",
            "--max_steps", str(STEPS)]
    trainer([tmp_path / "one", *argv]).run()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs = [ctx.Process(target=_rank, args=(r, 2, port, [str(tmp_path / "many"), *map(str, argv)], q))
             for r in range(2)]
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
    assert all(isinstance(results[r], list) for r in range(2)), results
    assert len(results[0]) == STEPS and results[0] == results[1], "ranks drifted apart"
    a = checkpoint.read_tf_checkpoint(str(tmp_path / "many" / "on_stop.ckpt"))
    b = checkpoint.read_tf_checkpoint(str(tmp_path / "one" / "on_stop.ckpt"))
    assert sorted(a) == sorted(b)
    worst = {}
    for k in a:
        if not k.startswith("inference/"):
            continue
        x, y = np.asarray(a[k], np.float64), np.asarray(b[k], np.float64)
        diff = float(np.abs(x - y).max())
        if k.endswith(("/Adam", "/Adam_1")) or "/moving_" in k:
            err = diff / max(float(np.abs(y).max()), 1e-30)
            assert err <= REL, f"{k} differs by {err:.3g} of its scale"
        else:
            err = diff
            assert err <= VAR_ATOL, f"{k} differs by {err:.3g}"
        worst[k] = err
    print(f"MEASURE bn dp equivalence: worst {max(worst, key=worst.get)} {max(worst.values()):.3g}")
