"""Image metrics of the training loop: drop-in for the reference's ``hdrnet/metrics.py:21-33``."""
from __future__ import annotations

import math

import torch


def l2_loss(target: torch.Tensor, prediction: torch.Tensor) -> torch.Tensor:
    """mean((target - prediction)^2) over every element."""
    return torch.mean(torch.square(target - prediction))


def psnr(target: torch.Tensor, prediction: torch.Tensor) -> torch.Tensor:
    """PSNR of each image, -10 log10(mean squared error), averaged over the batch."""
    squares = torch.square(target - prediction).reshape(target.shape[0], -1)
    return torch.mean((-10.0 / math.log(10.0)) * torch.log(torch.mean(squares, dim=1)))
