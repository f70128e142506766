"""CPU tests of the training CLI's --train_guide: off by default and outside the model parameters,
refused for the pointwise-NN guide, and a resume whose checkpoint disagrees with the flag refused
before any data is read; plus the models' own refusals with params['guide_grad']."""
import numpy as np
import pytest
import torch

from hdrnet_b200 import checkpoint, models
from hdrnet_b200.bin import train

P = dict(models.DEFAULT_PARAMS, net_input_size=32, spatial_bin=8, luma_bins=4)


def parse(*argv):
    parser = train.build_parser()
    args = parser.parse_args(["ckpt", "data", *argv])
    return args, train.model_params(parser, args)


def test_train_guide_defaults_off_and_is_not_a_model_parameter():
    args, params = parse()
    assert args.train_guide is False and "train_guide" not in params
    assert parse("--train_guide")[0].train_guide is True
    assert parse("--train_guide", "--notrain_guide")[0].train_guide is False


def test_train_guide_with_the_nn_guide_is_refused_before_data_is_read(tmp_path):
    ckpt = tmp_path / "ckpt"
    with pytest.raises(NotImplementedError, match="training mode"):
        train.main([str(ckpt), str(tmp_path / "no_such_data"), "--train_guide", "--model_name",
                    "HDRNetPointwiseNNGuide"])
    assert not ckpt.exists()
    train.refuse_untrainable(parse("--train_guide")[1], train_guide=True)          # the curves guide trains
    train.refuse_untrainable(parse("--model_name", "HDRNetPointwiseNNGuide")[1])   # without the flag it trains


def write_checkpoint(ckpt, with_guide_slots):
    params = dict(models.DEFAULT_PARAMS, net_input_size=32, spatial_bin=8, luma_bins=4)
    variables = models.init_weights(params, seed=2)
    prefixes = (train.COEFFS, train.GUIDE) if with_guide_slots else (train.COEFFS,)
    trained = sorted(k for k in variables if k.startswith(prefixes))
    moments = {k: (np.zeros_like(variables[k]), np.zeros_like(variables[k])) for k in trained}
    ckpt.mkdir()
    checkpoint.write_tf_checkpoint(str(ckpt / "model.ckpt-3"), train.checkpoint_tensors(variables, moments, 3, {}))


@pytest.mark.parametrize("flag,slots", [("--train_guide", False), ("--notrain_guide", True)])
def test_resume_that_disagrees_with_the_flag_is_refused_before_data_is_read(tmp_path, flag, slots):
    ckpt = tmp_path / "ckpt"
    write_checkpoint(ckpt, slots)
    with pytest.raises(ValueError, match="--train_guide"):
        train.main([str(ckpt), str(tmp_path / "no_such_data"), flag])
    assert sorted(p.name for p in ckpt.iterdir()) == ["checkpoint", "model.ckpt-3.data-00000-of-00001",
                                                      "model.ckpt-3.index"]


def test_resume_that_agrees_with_the_flag_passes_the_check(tmp_path):
    for slots in (False, True):
        ckpt = tmp_path / f"ckpt{int(slots)}"
        write_checkpoint(ckpt, slots)
        train.refuse_resume_mismatch(checkpoint.read_tf_checkpoint(str(ckpt)), slots)


def tensor_weights(model_name=None, grad=()):
    w = {k: torch.from_numpy(v) for k, v in models.init_weights(P, model_name=model_name).items()}
    for k in grad:
        w[k].requires_grad_(True)
    return w


def test_guide_grad_refusals_name_what_is_missing():
    low, full = torch.rand(1, 32, 32, 3), torch.rand(1, 16, 16, 3)
    # without the key: today's refusals, now with a hint naming it
    with pytest.raises(NotImplementedError, match="guide variables.*guide_grad"):
        models.HDRNetCurves.inference(low, full, dict(P, weights=tensor_weights(grad=["inference/guide/ccm"])))
    with pytest.raises(NotImplementedError, match="fullres_input.*guide_grad"):
        models.HDRNetCurves.inference(low, full.clone().requires_grad_(True), dict(P, weights=tensor_weights()))
    # the pointwise-NN guide: refused with the key, naming training-mode batch norm
    nn = tensor_weights("HDRNetPointwiseNNGuide", grad=["inference/guide/conv1/weights"])
    with pytest.raises(NotImplementedError, match="batch norm, which training runs in training mode"):
        models.HDRNetPointwiseNNGuide.inference(low, full, dict(P, weights=nn, guide_grad=True))
    with pytest.raises(NotImplementedError, match="fullres_input"):
        models.HDRNetPointwiseNNGuide.inference(low, full.clone().requires_grad_(True),
                                                dict(P, weights=tensor_weights("HDRNetPointwiseNNGuide"),
                                                     guide_grad=True))
    # the pyramid keeps its refusal
    pyr = tensor_weights("HDRNetGaussianPyrNN", grad=["inference/guide/level_0/conv2/weights"])
    with pytest.raises(NotImplementedError, match="resize"):
        models.HDRNetGaussianPyrNN.inference(low, full, dict(P, weights=pyr, guide_grad=True))
    # the curves guide with the key is not refused: the call gets as far as the device check
    with pytest.raises(Exception) as e:
        models.HDRNetCurves.inference(low, full.clone().requires_grad_(True),
                                      dict(P, weights=tensor_weights(grad=["inference/guide/ccm"]), guide_grad=True))
    assert not isinstance(e.value, NotImplementedError)
