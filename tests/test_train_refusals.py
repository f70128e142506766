"""CPU tests: the gradients the package does not compute are refused with NotImplementedError
before any device work (guide variables, fullres_input, batch-norm layers, the pyramid model), and
is_training=True still raises."""
import pytest
import torch

from hdrnet_b200 import layers, models

P = dict(models.DEFAULT_PARAMS, net_input_size=32, spatial_bin=8, luma_bins=4)


def tensor_weights(params=P, model_name=None, grad=()):
    w = {k: torch.from_numpy(v) for k, v in models.init_weights(params, model_name=model_name).items()}
    for k in grad:
        w[k].requires_grad_(True)
    return w


def inputs(grad_full=False):
    low = torch.rand(1, 32, 32, 3)
    full = torch.rand(1, 16, 16, 3).requires_grad_(grad_full)
    return low, full


@pytest.mark.parametrize("model", [models.HDRNetCurves, models.HDRNetPointwiseNNGuide])
def test_guide_variable_requiring_grad_is_refused(model):
    name = "inference/guide/ccm" if model is models.HDRNetCurves else "inference/guide/conv2/weights"
    w = tensor_weights(model_name=model.__name__, grad=[name])
    with pytest.raises(NotImplementedError, match="guide variables"):
        model.inference(*inputs(), dict(P, weights=w))


def test_fullres_input_requiring_grad_is_refused():
    with pytest.raises(NotImplementedError, match="fullres_input"):
        models.HDRNetCurves.inference(*inputs(grad_full=True), dict(P, weights=tensor_weights()))


def test_batch_norm_variable_requiring_grad_is_refused():
    bn = dict(P, batch_norm=True)
    w = tensor_weights(bn, grad=["inference/coefficients/global/fc1/BatchNorm/beta"])
    with pytest.raises(NotImplementedError, match="batch-norm"):
        models.HDRNetCurves._coefficients(inputs()[0], dict(bn, weights=w))
    with pytest.raises(NotImplementedError, match="batch-norm"):
        models.HDRNetCurves.inference(*inputs(), dict(bn, weights=w))
    with pytest.raises(NotImplementedError, match="batch-norm"):
        layers.fc(torch.rand(1, 128), 128, batch_norm=True, scope="inference/coefficients/global/fc1", weights=w)


def test_pyramid_model_gradient_is_refused():
    w = tensor_weights(model_name="HDRNetGaussianPyrNN", grad=["inference/coefficients/splat/conv1/weights"])
    with pytest.raises(NotImplementedError, match="resize"):
        models.HDRNetGaussianPyrNN.inference(*inputs(), dict(P, weights=w))
    low, full = inputs()
    with pytest.raises(NotImplementedError, match="resize"):
        models.HDRNetGaussianPyrNN.inference(low.requires_grad_(True), full,
                                             dict(P, weights=tensor_weights(model_name="HDRNetGaussianPyrNN")))


def test_refusals_are_off_without_grad():
    """Under torch.no_grad() nothing is differentiated, so nothing is refused: the call gets as far
    as the device check."""
    w = tensor_weights(grad=["inference/guide/ccm"])
    with torch.no_grad(), pytest.raises(Exception) as e:
        models.HDRNetCurves.inference(*inputs(grad_full=True), dict(P, weights=w))
    assert not isinstance(e.value, NotImplementedError)


def test_is_training_still_raises():
    w = tensor_weights(grad=["inference/coefficients/splat/conv1/weights"])
    with pytest.raises(NotImplementedError, match="inference path only"):
        models.HDRNetCurves.inference(*inputs(), dict(P, weights=w), is_training=True)
    with pytest.raises(NotImplementedError, match="inference path only"):
        layers.conv(torch.rand(1, 8, 8, 3), 4, 3, is_training=True, scope="s", weights=w)
