"""HDRNetGaussianPyr's graph in the two float64-summing model restatements -- TEST INFRASTRUCTURE ONLY.

oracle/model_np.py and oracle/model_torch.py restate HDRNetGaussianPyrNN (hdrnet/models.py:213-289)
with the pointwise-NN guide at every level.  ``inference(O, ..., guide)`` is that pyramid, step for
step as ``O.gaussian_pyr_inference`` runs it, with each level's guide chosen by the caller:
``O.guide_curves`` gives HDRNetGaussianPyr (DESIGN.md row f-17).  ``O`` is either restatement module,
so its own coefficient network, resize and guide do the work, and the two stay independent of each
other.  With ``guide=O.guide_nn`` the result is ``O.gaussian_pyr_inference``'s bit for bit
(tests/test_gaussian_pyr.py), which pins the composition here to the restatements' own.
"""
from __future__ import annotations

import numpy as np


def inference(O, lowres, fullres, wts, params, slice_apply, guide):
    """(output, coefficients [B,gh,gw,gd,9,4], the three levels' guides) of the pyramid with
    ``guide(level, wts, prefix)`` under ``inference/guide/level_{l}``; the COARSEST level uses output
    rows 0..2 (the reference's Python-2 ``reversed(zip())``)."""
    coeffs = O.coefficients(lowres, wts, params, n_out=9)
    lvls = [np.asarray(fullres, np.float32)]
    h, w = lvls[0].shape[1:3]
    for _ in range(2):
        h, w = h // 2, w // 2
        lvls.append(O.resize_bilinear_ac(lvls[-1], h, w))
    guides = [guide(lvl, wts, f"inference/guide/level_{i}") for i, lvl in enumerate(lvls)]
    B, gh, gw, gd = coeffs.shape[:4]
    current = None
    for il in range(3):
        src = 2 - il
        c = np.ascontiguousarray(coeffs[:, :, :, :, il * 3:(il + 1) * 3, :]).reshape(B, gh, gw, gd, 12)
        out_lvl = slice_apply(c, guides[src], lvls[src], True)
        current = out_lvl if il == 0 else O.resize_bilinear_ac(current, out_lvl.shape[1], out_lvl.shape[2]) + out_lvl
    return current.astype(np.float32), coeffs, guides
