"""CPU tests of --coefficient_batch_stats (the coefficient network's batch norm in training mode): the
flag, the combinations it is accepted in, its refusals before any data is read, and the models'
checks of params['coefficient_batch_stats'] before any device work."""
import pytest
import torch

from hdrnet_b200 import models
from hdrnet_b200.bin import train

BN = ["--batch_norm", "--coefficient_batch_stats"]


def parse(*argv):
    parser = train.build_parser()
    args = parser.parse_args(["ckpt", "data", *argv])
    return args, train.model_params(parser, args)


def refuse(*argv):
    args, params = parse(*argv)
    train.refuse_untrainable(params, args.train_guide, args.guide_batch_stats, args.coefficient_batch_stats)


def test_flag_pair_defaults_off_and_is_not_a_model_parameter():
    args, params = parse()
    assert args.coefficient_batch_stats is False and "coefficient_batch_stats" not in params
    assert parse("--coefficient_batch_stats")[0].coefficient_batch_stats is True
    assert parse("--coefficient_batch_stats", "--nocoefficient_batch_stats")[0].coefficient_batch_stats is False


@pytest.mark.parametrize("flags", [BN, BN + ["--train_guide"],
                                   BN + ["--model_name", "HDRNetPointwiseNNGuide", "--guide_batch_stats"],
                                   BN + ["--model_name", "HDRNetPointwiseNNGuide", "--guide_batch_stats", "--train_guide"],
                                   BN + ["--model_name", "HDRNetGaussianPyrNN", "--train_guide", "--guide_batch_stats"]])
def test_accepted_combinations(flags):
    refuse(*flags)


@pytest.mark.parametrize("flags,error,match", [
    (["--coefficient_batch_stats"], ValueError, "--batch_norm"),
    (BN + ["--model_name", "HDRNetPointwiseNNGuide"], ValueError, "--guide_batch_stats"),
    (BN + ["--model_name", "HDRNetGaussianPyrNN", "--train_guide"], ValueError, "--guide_batch_stats"),
    (BN + ["--model_name", "HDRNetGaussianPyrNN", "--guide_batch_stats"], NotImplementedError, "resize"),
    (["--batch_norm"], NotImplementedError, "^gradients through a batch-norm layer are not implemented.*"
                                            "--coefficient_batch_stats")])
def test_refusals_come_before_any_data_is_read(tmp_path, flags, error, match):
    ckpt = tmp_path / "ckpt"
    with pytest.raises(error, match=match):
        train.main([str(ckpt), str(tmp_path / "no_such_data"), *flags])
    assert not ckpt.exists()


def test_accepted_flags_get_past_the_refusals_to_the_data(tmp_path):
    with pytest.raises(Exception) as e:
        train.main([str(tmp_path / "ckpt"), str(tmp_path / "no_such_data"), *BN])
    assert not isinstance(e.value, NotImplementedError) and "batch" not in str(e.value)


P = dict(models.DEFAULT_PARAMS, net_input_size=32, spatial_bin=8, luma_bins=4, batch_norm=True)


def tensor_weights(params=P, model_name=None, grad=True):
    w = {k: torch.from_numpy(v) for k, v in models.init_weights(params, model_name=model_name).items()}
    for k in w:
        if k.startswith("inference/coefficients") and "/moving_" not in k:
            w[k].requires_grad_(grad)
    return w


def test_models_check_the_key_before_any_device_work():
    low, full = torch.rand(1, 32, 32, 3), torch.rand(1, 16, 16, 3)
    w = tensor_weights()
    with pytest.raises(ValueError, match="batch_norm"):
        models.HDRNetCurves._coefficients(low, dict(P, batch_norm=False, weights=w, coefficient_batch_stats=True),
                                          is_training=True)
    with pytest.raises(ValueError, match="batch_norm"):
        models.HDRNetCurves.inference(low, full, dict(P, batch_norm=False, weights=w, coefficient_batch_stats=True))
    mm = "inference/coefficients/global/fc1/BatchNorm/moving_mean"
    with pytest.raises(TypeError, match="moving_mean"):
        models.HDRNetCurves._coefficients(low, dict(P, weights=dict(w, **{mm: w[mm].numpy()}),
                                                    coefficient_batch_stats=True), is_training=True)
    with pytest.raises(ValueError, match="not trainable"):
        models.HDRNetCurves._coefficients(low, dict(P, weights=dict(w, **{mm: w[mm].clone().requires_grad_(True)}),
                                                    coefficient_batch_stats=True), is_training=True)
    # accepted: every model gets as far as the device check
    for cls, name in ((models.HDRNetCurves, None), (models.HDRNetPointwiseNNGuide, "HDRNetPointwiseNNGuide"),
                      (models.HDRNetGaussianPyrNN, "HDRNetGaussianPyrNN")):
        with pytest.raises(Exception) as e:
            cls.inference(low, full, dict(P, weights=tensor_weights(model_name=name), coefficient_batch_stats=True),
                          is_training=True)
        assert not isinstance(e.value, (NotImplementedError, ValueError, TypeError)), (cls, e.value)
    # without the key, today's refusals
    with pytest.raises(NotImplementedError, match="inference path only"):
        models.HDRNetCurves.inference(low, full, dict(P, weights=w), is_training=True)
    with pytest.raises(NotImplementedError, match="batch-norm"):
        models.HDRNetCurves._coefficients(low, dict(P, weights=w))
