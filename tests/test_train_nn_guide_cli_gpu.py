"""The training CLI with --train_guide --guide_batch_stats on HDRNetPointwiseNNGuide, on a small
synthetic dataset (u8 PNG inputs, u16 PNG targets rendered by a teacher whose NN guide is not the
initial one): 10 steps + resume + 10 steps equal 20 straight steps bit for bit, moving averages
included; the moving averages left 0 / 1 and carry no Adam slots; bin/run.py on the checkpoint
directory reproduces the in-memory model in its inference form; the loss falls."""
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

NN = "HDRNetPointwiseNNGuide"
MODEL = ["--net_input_size", "64", "--spatial_bin", "8", "--output_resolution", "128", "128", "--batch_size", "4",
         "--model_name", NN]
PARAMS = dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8, output_resolution=[128, 128], model_name=NN)
N_IMAGES, H, W = 6, 144, 176
G = "inference/guide/"


@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    root = tmp_path_factory.mktemp("nn_guide_pairs")
    os.makedirs(root / "input")
    os.makedirs(root / "output")
    w = models.init_weights(PARAMS, seed=1, model_name=NN)
    rng = np.random.RandomState(3)
    w[G + "conv1/weights"] = (rng.randn(1, 1, 3, 16) * 2.0).astype(np.float32)
    w[G + "conv1/BatchNorm/beta"] = (rng.randn(16) * 0.5).astype(np.float32)
    w[G + "conv1/BatchNorm/moving_mean"] = (rng.rand(16) * 0.5).astype(np.float32)
    w[G + "conv1/BatchNorm/moving_variance"] = (rng.rand(16) * 0.2 + 0.05).astype(np.float32)
    w[G + "conv2/weights"] = (rng.randn(1, 1, 16, 1) * 0.5).astype(np.float32)
    teacher = dict(PARAMS, weights=w)
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


def trainer(ckpt, data, *flags):
    parser = train.build_parser()
    args = parser.parse_args([str(ckpt), str(data), *MODEL, "--summary_interval", "0",
                              "--checkpoint_interval", "100000", "--train_guide", "--guide_batch_stats", *flags])
    params = train.model_params(parser, args)
    train.refuse_untrainable(params, args.train_guide, args.guide_batch_stats)
    return train.Trainer(args, params)


def test_nn_guide_trains_resumes_bitwise_and_run_reproduces_it(dataset, tmp_path):
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
    init = models.init_weights(PARAMS, seed=5, model_name=NN)
    guide = [k for k in init if k.startswith(G)]
    assert len(guide) == 6
    for k in guide:
        assert not np.array_equal(a[k], init[k]), f"{k} did not move"
        if "/moving_" in k:
            assert k + "/Adam" not in a and k + "/Adam_1" not in a, k
        else:
            assert k + "/Adam" in a and np.abs(a[k + "/Adam_1"]).sum() > 0, k
    assert not any("/moving_" in k and "/Adam" in k for k in a)
    keys = [k for k in a if k.startswith("inference/")]
    assert sorted(keys) == sorted(k for k in b if k.startswith("inference/"))
    for k in keys:
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), k
    with open(tmp_path / "straight" / "params.json") as f:
        assert "guide_batch_stats" not in json.load(f)

    losses = [json.loads(line)["loss"] for line in open(tmp_path / "straight" / "train_log.jsonl")
              if '"loss"' in line]
    first, last = float(np.mean(losses[:3])), float(np.mean(losses[-3:]))
    print("MEASURE nn-guide CLI loss", f"first3={first:.4g} last3={last:.4g} factor={first / last:.3g}", flush=True)
    assert last * 1.5 <= first

    out_dir = tmp_path / "out"
    run_cli.main(argparse.Namespace(checkpoint_dir=str(tmp_path / "straight"), input=str(dataset / "input"),
                                    output=str(out_dir), lowres_input=None, hdrp=False, debug=False, limit=None))
    for name in sorted(os.listdir(dataset / "input")):
        im8 = cv2.imread(str(dataset / "input" / name), -1)[:, :, ::-1]
        with torch.no_grad():
            want = models.HDRNetPointwiseNNGuide.inference_image(
                torch.from_numpy(np.ascontiguousarray(im8[None])).cuda(), straight.p)[0].cpu().numpy()
        assert np.array_equal(cv2.imread(str(out_dir / name), -1)[:, :, ::-1], want), name
