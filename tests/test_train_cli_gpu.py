"""The training CLI end to end on a synthetic dataset: u8 PNG inputs and u16 PNG targets rendered
by a teacher HDRNetCurves (init_weights(seed=1)).  A student run without augmentation fits the
teacher; N steps straight equal N/2 + resume + N/2 bit for bit; the guide stays at its initial
values; bin/run.py on the checkpoint directory reproduces the in-memory model; a run with every
augmentation flag (and an eval set) completes with finite losses."""
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

pytestmark = pytest.mark.gpu

MODEL = ["--net_input_size", "64", "--spatial_bin", "8", "--output_resolution", "128", "128", "--batch_size", "4"]
PARAMS = dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8, output_resolution=[128, 128])
N_IMAGES, H, W = 8, 144, 176


@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    root = tmp_path_factory.mktemp("pairs")
    os.makedirs(root / "input")
    os.makedirs(root / "output")
    teacher = dict(PARAMS, weights=models.init_weights(PARAMS, seed=1))
    rng = np.random.RandomState(7)
    names = []
    for i in range(N_IMAGES):
        # smooth colour fields plus noise: a natural-ish spread of guide values
        yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
        base = np.stack([np.sin(3 * xx + i) , np.cos(2 * yy - i), xx * yy], axis=2) * 0.4 + 0.5
        im = np.clip(base + 0.1 * rng.randn(H, W, 3), 0, 1)
        im8 = (im * 255).astype(np.uint8)
        with torch.no_grad():
            out = models.HDRNetCurves.inference_image(torch.from_numpy(im8[None]).cuda(), teacher,
                                                      out_dtype=torch.float32)[0].cpu().numpy()
        out16 = np.rint(np.clip(out, 0, 1) * 65535).astype(np.uint16)
        name = f"im{i:02d}.png"
        assert cv2.imwrite(str(root / "input" / name), im8[:, :, ::-1])
        assert cv2.imwrite(str(root / "output" / name), out16[:, :, ::-1])
        names.append(name)
    (root / "filelist.txt").write_text("\n".join(names) + "\n")
    return root


def trainer(ckpt, data, *flags):
    parser = train.build_parser()
    args = parser.parse_args([str(ckpt), str(data), *MODEL, "--summary_interval", "0",
                              "--checkpoint_interval", "100000", *flags])
    params = train.model_params(parser, args)
    train.refuse_untrainable(params)
    return train.Trainer(args, params)


def log_records(ckpt):
    with open(os.path.join(ckpt, "train_log.jsonl")) as f:
        return [json.loads(line) for line in f]


@pytest.fixture(scope="module")
def student(dataset, tmp_path_factory):
    ckpt = tmp_path_factory.mktemp("student")
    t = trainer(ckpt, dataset, "--norandom_crop", "--max_steps", "300")
    t.run()
    return t, ckpt


def test_student_fits_the_teacher(student):
    _, ckpt = student
    losses = [r["loss"] for r in log_records(ckpt) if "loss" in r]
    assert len(losses) == 300 and all(np.isfinite(losses))
    first, last = losses[0], float(np.mean(losses[-10:]))
    print(f"MEASURE train-cli student: first {first:.4g} last-10 mean {last:.4g} factor {first / last:.1f}")
    assert first / last >= 10.0


def test_guide_variables_keep_their_initial_values(student):
    _, ckpt = student
    saved = checkpoint.read_tf_checkpoint(str(ckpt))
    init = models.init_weights(PARAMS, seed=0)
    guide = [k for k in init if k.startswith("inference/guide/")]
    assert guide and int(saved["global_step"]) == 300
    for k in guide:
        assert np.array_equal(saved[k].view(np.uint32), init[k].view(np.uint32)), k
    assert not any(k.startswith("inference/guide/") and k.endswith(("/Adam", "/Adam_1")) for k in saved)
    moved = [k for k in init if k.startswith("inference/coefficients/") and not np.array_equal(saved[k], init[k])]
    assert len(moved) > 10


def test_run_cli_on_the_checkpoint_matches_the_model_in_memory(student, dataset, tmp_path):
    t, ckpt = student
    out_dir = tmp_path / "out"
    run_cli.main(argparse.Namespace(checkpoint_dir=str(ckpt), input=str(dataset / "input"), output=str(out_dir),
                                    lowres_input=None, hdrp=False, debug=False, limit=None))
    names = sorted(os.listdir(dataset / "input"))
    assert sorted(os.listdir(out_dir)) == names
    for name in names:
        im8 = cv2.imread(str(dataset / "input" / name), -1)[:, :, ::-1]
        with torch.no_grad():
            want = models.HDRNetCurves.inference_image(torch.from_numpy(np.ascontiguousarray(im8[None])).cuda(),
                                                       t.p)[0].cpu().numpy()
        got = cv2.imread(str(out_dir / name), -1)[:, :, ::-1]
        assert np.array_equal(got, want), name


def test_resume_gives_the_uninterrupted_run_bitwise(dataset, tmp_path):
    flags = ["--fliplr", "--flipud", "--rotate", "--seed", "5"]
    trainer(tmp_path / "straight", dataset, *flags, "--max_steps", "20").run()
    trainer(tmp_path / "resumed", dataset, *flags, "--max_steps", "10").run()
    t = trainer(tmp_path / "resumed", dataset, *flags, "--max_steps", "20")
    assert t.step == 10
    t.run()
    a = checkpoint.read_tf_checkpoint(str(tmp_path / "straight"))
    b = checkpoint.read_tf_checkpoint(str(tmp_path / "resumed"))
    assert int(a["global_step"]) == int(b["global_step"]) == 20
    keys = [k for k in a if k.startswith("inference/")]
    assert sorted(keys) == sorted(k for k in b if k.startswith("inference/"))
    assert sum(k.endswith("/Adam") for k in keys) == sum(k.endswith("/Adam_1") for k in keys) > 10
    for k in keys:
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), k
    la = [r["loss"] for r in log_records(tmp_path / "straight") if "loss" in r]
    lb = [r["loss"] for r in log_records(tmp_path / "resumed") if "loss" in r]
    assert la == lb


def test_every_augmentation_flag_with_an_eval_set(dataset, tmp_path):
    t = trainer(tmp_path / "aug", dataset, "--fliplr", "--flipud", "--rotate", "--random_crop",
                "--eval_data_dir", str(dataset), "--eval_interval", "0", "--max_steps", "12",
                "--model_name", "HDRNetPointwiseNNGuide")
    t.run()
    recs = log_records(tmp_path / "aug")
    losses = [r["loss"] for r in recs if "loss" in r]
    evals = [r["eval_psnr"] for r in recs if "eval_psnr" in r]
    assert len(losses) == 12 and np.isfinite(losses).all()
    assert len(evals) == 12 and np.isfinite(evals).all()
    assert os.path.exists(tmp_path / "aug" / "on_stop.ckpt.index")
    with open(tmp_path / "aug" / "params.json") as f:
        assert json.load(f)["model_name"] == "HDRNetPointwiseNNGuide"
