"""CPU tests of the training CLI's --guide_batch_stats and of the training-mode refusals of
HDRNetPointwiseNNGuide.inference: off by default and outside the model parameters, refused for
HDRNetCurves, the moving averages outside the trained names, and the moving averages checked before
any device work."""
import pytest
import torch

from hdrnet_b200 import models
from hdrnet_b200.bin import train

P = dict(models.DEFAULT_PARAMS, net_input_size=32, spatial_bin=8, luma_bins=4)
NN = "HDRNetPointwiseNNGuide"


def parse(*argv):
    parser = train.build_parser()
    args = parser.parse_args(["ckpt", "data", *argv])
    return args, train.model_params(parser, args)


def test_flag_defaults_off_and_is_not_a_model_parameter():
    args, params = parse()
    assert args.guide_batch_stats is False and "guide_batch_stats" not in params
    assert parse("--guide_batch_stats")[0].guide_batch_stats is True
    assert parse("--guide_batch_stats", "--noguide_batch_stats")[0].guide_batch_stats is False


def test_flag_with_curves_is_refused_before_data_is_read(tmp_path):
    ckpt = tmp_path / "ckpt"
    with pytest.raises(ValueError, match="no batch norm"):
        train.main([str(ckpt), str(tmp_path / "no_such_data"), "--guide_batch_stats"])
    assert not ckpt.exists()


def test_pyramid_keeps_its_refusal_with_the_flag(tmp_path):
    with pytest.raises(NotImplementedError, match="resize"):
        train.main([str(tmp_path / "ckpt"), str(tmp_path / "no_such_data"), "--guide_batch_stats",
                    "--model_name", "HDRNetGaussianPyrNN"])


def test_train_guide_on_the_nn_guide_needs_the_flag():
    params = parse("--model_name", NN)[1]
    with pytest.raises(NotImplementedError, match="training mode.*--guide_batch_stats"):
        train.refuse_untrainable(params, train_guide=True)
    train.refuse_untrainable(params, train_guide=True, guide_batch_stats=True)
    train.refuse_untrainable(params, guide_batch_stats=True)


def test_trained_names_exclude_the_moving_averages():
    w = models.init_weights(dict(P, model_name=NN), model_name=NN)
    moving = [k for k in w if "/BatchNorm/moving_" in k]
    assert len(moving) == 2
    names = train.trained_names(w, train_guide=True)
    assert not set(moving) & set(names)
    assert {"inference/guide/conv1/weights", "inference/guide/conv1/BatchNorm/beta", "inference/guide/conv2/weights",
            "inference/guide/conv2/biases"} <= set(names)
    assert not any(k.startswith(train.GUIDE) for k in train.trained_names(w))


def nn_weights(grad=(), **over):
    w = {k: torch.from_numpy(v) for k, v in models.init_weights(P, model_name=NN).items()}
    for k in grad:
        w[k].requires_grad_(True)
    w.update(over)
    return w


def test_training_mode_refusals_come_before_device_work():
    low, full = torch.rand(1, 32, 32, 3), torch.rand(1, 16, 16, 3)
    mm = "inference/guide/conv1/BatchNorm/moving_mean"
    w = nn_weights()
    with pytest.raises(TypeError, match="moving_mean"):
        models.HDRNetPointwiseNNGuide.inference(low, full, dict(P, weights=dict(w, **{mm: w[mm].numpy()})),
                                                is_training=True)
    with pytest.raises(TypeError, match="moving_mean"):
        models.HDRNetPointwiseNNGuide._guide(full, dict(P, weights=dict(w, **{mm: w[mm].numpy()})),
                                             is_training=True)
    with pytest.raises(ValueError, match="not trainable"):
        models.HDRNetPointwiseNNGuide.inference(low, full, dict(P, weights=nn_weights(grad=[mm])), is_training=True)
    with pytest.raises(NotImplementedError, match="coefficient network"):
        models.HDRNetPointwiseNNGuide.inference(low, full, dict(P, batch_norm=True, weights=w), is_training=True)
    # without guide_grad the guide's variables keep today's refusal
    with pytest.raises(NotImplementedError, match="guide variables"):
        models.HDRNetPointwiseNNGuide.inference(
            low, full, dict(P, weights=nn_weights(grad=["inference/guide/conv1/weights"])), is_training=True)
    # with it the call is not refused: it gets as far as the device check
    with pytest.raises(Exception) as e:
        models.HDRNetPointwiseNNGuide.inference(
            low, full.clone().requires_grad_(True),
            dict(P, weights=nn_weights(grad=["inference/guide/conv1/weights"]), guide_grad=True), is_training=True)
    assert not isinstance(e.value, (NotImplementedError, TypeError))
    # the other models keep "inference path only"
    with pytest.raises(NotImplementedError, match="inference path only"):
        models.HDRNetCurves.inference(low, full, dict(P, weights=w), is_training=True)
