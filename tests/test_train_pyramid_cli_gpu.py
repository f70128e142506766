"""The training CLI on HDRNetGaussianPyrNN with --train_guide --guide_batch_stats, on a small
synthetic dataset (u8 PNG inputs, u16 PNG targets rendered by a pyramid teacher whose three guides
are not the initial ones): the student fits the teacher; 10 steps + resume + 10 steps equal 20
straight steps bit for bit, the three levels' moving averages included; bin/run.py on the checkpoint
directory writes the in-memory model's images; the recipes' size (batch 1 at 2048², channel
multiplier 4) trains; two ranks sharing one card over gloo train what one process trains."""
import argparse
import json
import os

import cv2
import numpy as np
import pytest
import torch

from hdrnet_b200 import checkpoint, models
from hdrnet_b200.bin import run as run_cli
from hdrnet_b200.bin import train
from test_train_dp_gpu import COMMON, STEPS, assert_equivalent, run_ranks

pytestmark = pytest.mark.gpu

PYR = "HDRNetGaussianPyrNN"
MODEL = ["--net_input_size", "64", "--spatial_bin", "8", "--output_resolution", "128", "128", "--batch_size", "4",
         "--model_name", PYR]
PARAMS = dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8, output_resolution=[128, 128], model_name=PYR)
N_IMAGES, H, W = 6, 144, 176
LEVELS = [f"inference/guide/level_{l}/" for l in range(3)]


def render(root, n, h, w, teacher, seed):
    os.makedirs(root / "input", exist_ok=True)
    os.makedirs(root / "output", exist_ok=True)
    rng = np.random.RandomState(seed)
    names = []
    for i in range(n):
        yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
        base = np.stack([np.sin(3 * xx + i), np.cos(2 * yy - i), xx * yy], axis=2) * 0.4 + 0.5
        im8 = (np.clip(base + 0.1 * rng.randn(h, w, 3), 0, 1) * 255).astype(np.uint8)
        with torch.no_grad():
            out = models.HDRNetGaussianPyrNN.inference_image(torch.from_numpy(im8[None]).cuda(), teacher,
                                                             out_dtype=torch.float32)[0].cpu().numpy()
        name = f"im{i:02d}.png"
        assert cv2.imwrite(str(root / "input" / name), im8[:, :, ::-1])
        assert cv2.imwrite(str(root / "output" / name), np.rint(np.clip(out, 0, 1) * 65535).astype(np.uint16)[:, :, ::-1])
        names.append(name)
    (root / "filelist.txt").write_text("\n".join(names) + "\n")
    return root


def teacher_weights(params, seed=1):
    w = models.init_weights(params, seed=seed, model_name=PYR)
    rng = np.random.RandomState(3)
    F = params["guide_complexity"]
    for g in LEVELS:
        w[g + "conv1/weights"] = (rng.randn(1, 1, 3, F) * 2.0).astype(np.float32)
        w[g + "conv1/BatchNorm/beta"] = (rng.randn(F) * 0.5).astype(np.float32)
        w[g + "conv1/BatchNorm/moving_mean"] = (rng.rand(F) * 0.5).astype(np.float32)
        w[g + "conv1/BatchNorm/moving_variance"] = (rng.rand(F) * 0.2 + 0.05).astype(np.float32)
        w[g + "conv2/weights"] = (rng.randn(1, 1, F, 1) * 0.5).astype(np.float32)
    return w


@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    return render(tmp_path_factory.mktemp("pyramid_pairs"), N_IMAGES, H, W,
                  dict(PARAMS, weights=teacher_weights(PARAMS)), 3)


def trainer(ckpt, data, *flags, model=MODEL):
    parser = train.build_parser()
    args = parser.parse_args([str(ckpt), str(data), *model, "--summary_interval", "0",
                              "--checkpoint_interval", "100000", "--train_guide", "--guide_batch_stats", *flags])
    params = train.model_params(parser, args)
    train.refuse_untrainable(params, args.train_guide, args.guide_batch_stats)
    return train.Trainer(args, params)


def logged_losses(ckpt_dir):
    return [json.loads(line)["loss"] for line in open(ckpt_dir / "train_log.jsonl") if '"loss"' in line]


def test_student_fits_the_teacher(dataset, tmp_path):
    t = trainer(tmp_path / "fit", dataset, "--seed", "5", "--learning_rate", "2e-3", "--max_steps", "150")
    t.run()
    losses = logged_losses(tmp_path / "fit")
    first, last = float(np.mean(losses[:3])), float(np.mean(losses[-3:]))
    print("MEASURE pyramid CLI fit", f"first3={first:.4g} last3={last:.4g} factor={first / last:.3g}", flush=True)
    assert np.isfinite(losses).all()
    assert last * 10 <= first


def test_pyramid_trains_resumes_bitwise_and_run_reproduces_it(dataset, tmp_path):
    flags = ["--fliplr", "--rotate", "--seed", "5", "--learning_rate", "1e-3"]
    straight = trainer(tmp_path / "straight", dataset, *flags, "--max_steps", "20")
    straight.run()
    trainer(tmp_path / "resumed", dataset, *flags, "--max_steps", "10").run()
    t = trainer(tmp_path / "resumed", dataset, *flags, "--max_steps", "20")
    assert t.step == 10
    t.run()
    a = checkpoint.read_tf_checkpoint(str(tmp_path / "straight"))
    b = checkpoint.read_tf_checkpoint(str(tmp_path / "resumed"))
    assert int(a["global_step"]) == int(b["global_step"]) == 20
    init = models.init_weights(PARAMS, seed=5, model_name=PYR)
    guide = [k for k in init if k.startswith(train.GUIDE)]
    assert len(guide) == 18
    for k in guide:
        assert not np.array_equal(a[k], init[k]), f"{k} did not move"
        if "/moving_" in k:
            assert k + "/Adam" not in a and k + "/Adam_1" not in a, k
        else:
            assert k + "/Adam" in a and np.abs(a[k + "/Adam_1"]).sum() > 0, k
    keys = [k for k in a if k.startswith("inference/")]
    assert sorted(keys) == sorted(k for k in b if k.startswith("inference/"))
    for k in keys:
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), k

    out_dir = tmp_path / "out"
    run_cli.main(argparse.Namespace(checkpoint_dir=str(tmp_path / "straight"), input=str(dataset / "input"),
                                    output=str(out_dir), lowres_input=None, hdrp=False, debug=False, limit=None))
    for name in sorted(os.listdir(dataset / "input")):
        im8 = cv2.imread(str(dataset / "input" / name), -1)[:, :, ::-1]
        with torch.no_grad():
            want = models.HDRNetGaussianPyrNN.inference_image(
                torch.from_numpy(np.ascontiguousarray(im8[None])).cuda(), straight.p)[0].cpu().numpy()
        assert np.array_equal(cv2.imread(str(out_dir / name), -1)[:, :, ::-1], want), name


def test_the_recipes_size_trains(tmp_path):
    """train_gpyrnn_cm4.sh's shape: --batch_size 1 --output_resolution 2048 2048 --channel_multiplier 4."""
    params = dict(models.DEFAULT_PARAMS, model_name=PYR, output_resolution=[2048, 2048])
    data = render(tmp_path / "big", 2, 2064, 2080, dict(params, weights=teacher_weights(params)), 4)
    model = ["--batch_size", "1", "--output_resolution", "2048", "2048", "--channel_multiplier", "4",
             "--model_name", PYR, "--nobatch_norm"]
    trainer(tmp_path / "ckpt", data, "--max_steps", "4", model=model).run()
    losses = logged_losses(tmp_path / "ckpt")
    print("MEASURE pyramid 2048^2 cm4 losses", losses, flush=True)
    assert len(losses) == 4 and np.isfinite(losses).all()


def test_two_ranks_on_one_card_train_what_one_process_trains(tmp_path, dataset):
    argv = [str(dataset), *COMMON, "--model_name", PYR, "--guide_batch_stats", "--max_steps", str(STEPS)]
    one, many = tmp_path / "one", tmp_path / "ranks"
    trainer(one, *argv[:1], *argv[1:], model=[]).run()
    digests = run_ranks([str(many), *argv])
    assert len(digests[0]) == STEPS and all(d == digests[0] for d in digests), "ranks drifted apart"
    assert len(set(digests[0])) == STEPS
    a, _ = assert_equivalent(str(many), str(one), f"{PYR} 2 ranks (gloo)")
    assert sum(k.startswith(LEVELS[2]) and "/moving_" in k for k in a) == 2
