"""CPU tests of training HDRNetGaussianPyrNN: the CLI trains it only with --train_guide
--guide_batch_stats, refuses every other configuration before any data is read with the model's own
text and the flags that do train it; inference(..., is_training=True) refuses on the CPU, before any
device work; the trained names cover the three levels' guide variables and none of their moving
averages."""
import pytest
import torch

from hdrnet_b200 import models
from hdrnet_b200.bin import train

P = dict(models.DEFAULT_PARAMS, net_input_size=32, spatial_bin=8, luma_bins=4, model_name="HDRNetGaussianPyrNN")
PYR = models.HDRNetGaussianPyrNN
LEVELS = [f"inference/guide/level_{l}" for l in range(3)]
PREFIX = "HDRNetGaussianPyrNN.inference (needs the VJP of the align-corners resize)"


def parse(*argv):
    parser = train.build_parser()
    args = parser.parse_args(["ckpt", "data", "--model_name", "HDRNetGaussianPyrNN", *argv])
    return args, train.model_params(parser, args)


@pytest.mark.parametrize("flags", [[], ["--guide_batch_stats"], ["--train_guide"]], ids=["none", "stats", "guide"])
def test_other_flag_combinations_are_refused_before_data_is_read(tmp_path, flags):
    ckpt = tmp_path / "ckpt"
    with pytest.raises(NotImplementedError, match="resize") as e:
        train.main([str(ckpt), str(tmp_path / "no_such_data"), "--model_name", "HDRNetGaussianPyrNN", *flags])
    assert str(e.value).startswith(PREFIX)
    assert str(e.value).endswith("--train_guide --guide_batch_stats trains the pyramid: its three guides, in "
                                 "training mode")
    assert "is_training=True" in str(e.value)
    assert not ckpt.exists()


def test_train_guide_with_batch_stats_is_accepted():
    args, params = parse("--train_guide", "--guide_batch_stats")
    train.refuse_untrainable(params, args.train_guide, args.guide_batch_stats)
    # the accepted flags do not lift the coefficient network's batch-norm refusal
    args, params = parse("--train_guide", "--guide_batch_stats", "--batch_norm")
    with pytest.raises(NotImplementedError, match="batch-norm"):
        train.refuse_untrainable(params, args.train_guide, args.guide_batch_stats)


def test_accepted_flags_get_past_the_refusals_to_the_data(tmp_path):
    """With the training flags the CLI goes past the refusals: it fails only later, on the missing data
    directory (or, without a device, on the device check)."""
    with pytest.raises(Exception) as e:
        train.main([str(tmp_path / "ckpt"), str(tmp_path / "no_such_data"), "--model_name", "HDRNetGaussianPyrNN",
                    "--train_guide", "--guide_batch_stats"])
    assert not isinstance(e.value, NotImplementedError)


def test_trained_names_cover_the_three_levels_without_moving_averages():
    w = models.init_weights(P, model_name="HDRNetGaussianPyrNN")
    names = train.trained_names(w, train_guide=True)
    for scope in LEVELS:
        assert {f"{scope}/conv1/weights", f"{scope}/conv1/BatchNorm/beta", f"{scope}/conv2/weights",
                f"{scope}/conv2/biases"} <= set(names)
        assert not {f"{scope}/conv1/BatchNorm/moving_mean", f"{scope}/conv1/BatchNorm/moving_variance"} & set(names)
    assert sum(k.startswith(train.GUIDE) for k in names) == 12
    assert not any(k.startswith(train.GUIDE) for k in train.trained_names(w))


def tensor_weights(grad=(), **over):
    w = {k: torch.from_numpy(v) for k, v in models.init_weights(P, model_name="HDRNetGaussianPyrNN").items()}
    w.update(over)
    for k in grad:
        w[k].requires_grad_(True)
    return w


def inputs():
    return torch.rand(1, 32, 32, 3), torch.rand(1, 16, 16, 3)


def test_training_mode_refusals_come_before_device_work():
    """CPU tensors: each refusal is raised before anything would reach the device."""
    coeff = "inference/coefficients/splat/conv1/weights"
    with pytest.raises(NotImplementedError, match="params\\['batch_norm'\\]"):
        PYR.inference(*inputs(), dict(P, batch_norm=True, weights=tensor_weights()), is_training=True)
    for scope in LEVELS:
        bad = tensor_weights(**{f"{scope}/conv1/BatchNorm/moving_mean": torch.zeros(16, dtype=torch.float64)})
        with pytest.raises(TypeError, match=f"{scope}/conv1/BatchNorm/moving_mean must be a float32"):
            PYR.inference(*inputs(), dict(P, weights=bad), is_training=True)
        numpy_ma = tensor_weights(**{f"{scope}/conv1/BatchNorm/moving_variance": torch.ones(16).numpy()})
        with pytest.raises(TypeError, match="moving_variance must be a float32 torch.Tensor"):
            PYR.inference(*inputs(), dict(P, weights=numpy_ma), is_training=True)
        with pytest.raises(ValueError, match="requires grad: moving averages are not trainable"):
            PYR.inference(*inputs(), dict(P, weights=tensor_weights([f"{scope}/conv1/BatchNorm/moving_mean"])),
                          is_training=True)
        with pytest.raises(NotImplementedError, match="guide variables"):
            PYR.inference(*inputs(), dict(P, weights=tensor_weights([f"{scope}/conv2/weights"])), is_training=True)
    low, full = inputs()
    with pytest.raises(NotImplementedError, match="fullres_input"):
        PYR.inference(low, full.requires_grad_(True), dict(P, weights=tensor_weights([coeff])), is_training=True)
    # with guide_grad nothing is refused: the call gets as far as the device check
    with pytest.raises(Exception) as e:
        PYR.inference(*inputs(), dict(P, weights=tensor_weights([coeff, f"{LEVELS[2]}/conv1/weights"]),
                                      guide_grad=True), is_training=True)
    assert not isinstance(e.value, (NotImplementedError, TypeError))


def test_inference_form_keeps_its_refusal_with_the_new_reason():
    for grad in (["inference/coefficients/splat/conv1/weights"], [f"{LEVELS[1]}/conv2/weights"]):
        with pytest.raises(NotImplementedError) as e:
            PYR.inference(*inputs(), dict(P, weights=tensor_weights(grad), guide_grad=True))
        msg = str(e.value)
        assert msg.startswith(PREFIX) and grad[0] in msg
        assert "batch norm folded from the moving averages, is not differentiated" in msg
        assert "inference(..., is_training=True), the training graph, is" in msg
