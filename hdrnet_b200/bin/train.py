#!/usr/bin/env python
"""Training CLI: counterpart of the reference's ``hdrnet/bin/train.py`` with the same positional
arguments, flags and defaults (train.py:188-244):

    python -m hdrnet_b200.bin.train <checkpoint_dir> <data_dir> [--eval_data_dir DIR]
        [--learning_rate 1e-4] [--batch_size 16] [--[no]fliplr|flipud|rotate|random_crop]
        [--model_name HDRNetCurves] [--net_input_size 256] [--output_resolution 512 512] ...
        [--max_steps N] [--seed S] [--[no]train_guide] [--[no]guide_batch_stats]
        [--[no]coefficient_batch_stats] [--data_pipeline UnsharpMaskDataPipeline --blur_sigma S --sharpen A]

``data_dir`` holds ``filelist.txt`` and the ``input/`` and ``output/`` folders (or is that
``filelist.txt``); hdrnet_b200/data_pipeline.py decodes the pairs once and builds each batch in one
kernel.  When the decoded pairs fit in the free device memory (less 2 GiB kept for the step) they
are uploaded once and each batch is gathered on the device; otherwise they stay on the host, and
each batch's crop windows are streamed to the device one to two steps ahead, with the same batches.
``--data_threads`` threads decode the files and, when streaming, pack the windows.  Each step runs ``inference`` with the coefficient-network variables
requiring grad, ``metrics.l2_loss`` and the per-image-mean ``metrics.psnr``, the backward and
``torch.optim.Adam(learning_rate)``.  An exponential moving average (0.99, zero-debiased as TF's
averages of tensors are) of loss and PSNR is logged every ``--log_interval`` seconds, and the
scalars go to ``checkpoint_dir/train_log.jsonl``.

Checkpoints (``model.ckpt-<step>`` every ``--checkpoint_interval`` seconds, ``on_stop.ckpt`` when
the run stops, as train.py:181) are TF V2 bundles written by ``checkpoint.write_tf_checkpoint``:
every ``inference/*`` variable (guide included), Adam's moments under TF's slot names
``<var>/Adam`` and ``<var>/Adam_1``, ``beta1_power`` / ``beta2_power`` and ``global_step``, with
``params.json`` beside them, so ``python -m hdrnet_b200.bin.run <checkpoint_dir> ...`` reads the
directory as it is.  A ``checkpoint_dir`` that already holds a checkpoint is resumed: variables,
moments and step are restored, and the batches continue where they would have (the sampler is a
function of ``(seed, step)``).

What is trained: the coefficient network, and with ``--train_guide`` the curves guide of
``HDRNetCurves`` too (``ccm``, ``ccm_bias``, ``shifts``, ``slopes``, ``channel_mixing/*``), in the
same Adam at the same learning rate, as the reference's single ``opt.minimize`` does
(train.py:92-94, :115); their Adam slots then go into each checkpoint.  Without the flag (the
default) the guide variables are held fixed at their initial (or restored) values.  A resume whose
checkpoint was written with the other setting of the flag is refused before any data is read.

``HDRNetPointwiseNNGuide``'s guide has batch norm after conv1, which the reference trains in training
mode.  ``--guide_batch_stats`` runs each step's forward that way (``inference(..., is_training=True)``):
conv1 is normalised with the batch's statistics, and ``conv1/BatchNorm/moving_mean`` and
``moving_variance`` move toward them once per step (decay 0.999), as the reference's ``UPDATE_OPS``
do (train.py:110-115).  The evaluation, and ``bin/run.py`` on the checkpoints, use the moving
averages, as the reference's eval graph does.  ``--train_guide --guide_batch_stats`` trains the whole
model as the reference's ``*_nn.sh`` scripts do.  The moving averages are not trainable: they get no
Adam slots, but go into every checkpoint and are restored on resume.  The flag is not a model
parameter and is not written to ``params.json``; a checkpoint does not record it, so a resume with the
other setting is not refused: it only changes the guide's forward from then on.  ``--train_guide``
with this model needs the flag; ``--guide_batch_stats`` with ``HDRNetCurves`` (no batch norm) is
refused with ``ValueError``.

``HDRNetGaussianPyrNN`` has one pointwise-NN guide per pyramid level (``inference/guide/level_{0,1,2}``)
and trains only as the reference's ``*_gpyrnn*.sh`` scripts train it: ``--nobatch_norm --train_guide
--guide_batch_stats``.  Each step then runs ``inference(..., is_training=True)``: each level's conv1
is normalised with that level's batch statistics, the three levels' moving averages move toward
them, and the coefficient network and all three guides are trained in the same Adam, their
gradients reaching the coarser levels through the VJP of the align-corners resize.  The three
levels' moving averages get no Adam slots, go into every checkpoint and are restored on resume;
evaluation and ``bin/run.py`` run the guide-fused inference form on them.  The pyramid without both
flags would train through its inference form, which is not differentiated, so it is refused.

``HDRNetGaussianPyr`` is that pyramid with ``HDRNetCurves``' guide at every level
(``inference/guide/level_{0,1,2}/{ccm, ccm_bias, shifts, slopes, channel_mixing/*}``), the model the
reference's ``*_gpyr*.sh`` recipes name (models.HDRNetGaussianPyr defines it).  It trains as
``HDRNetCurves`` does: ``--nobatch_norm``, with ``--train_guide`` its three curves guides too, without it
the three held fixed.  Its guides have no batch norm, so ``--guide_batch_stats`` is refused with
``ValueError`` and ``--batch_norm --coefficient_batch_stats`` does not need it.

``--batch_norm --coefficient_batch_stats`` trains the coefficient network's batch norm as the
reference's ``--batch_norm`` does (train.py:92-115): each step runs ``inference(..., is_training=True)``
with the batch-norm layers normalised by the batch's statistics (the whole batch's under a process
group) and their ``moving_mean`` / ``moving_variance`` moved once per step, on the device, with no host
synchronisation; each ``BatchNorm/beta`` is trained with Adam, the moving averages get no Adam slots but
go into every checkpoint and are restored on resume.  The flag is not a model parameter and is not
written to ``params.json``.  It needs ``--batch_norm`` (``ValueError``), and with
``HDRNetPointwiseNNGuide`` and ``HDRNetGaussianPyrNN`` also ``--guide_batch_stats`` (``ValueError``): the
reference runs every batch norm of the model in training mode.  ``--batch_norm`` without it, the
pyramid without ``--train_guide --guide_batch_stats``, and ``--train_guide`` with
``HDRNetPointwiseNNGuide`` without ``--guide_batch_stats`` are refused before any data is read,
with the models' own ``NotImplementedError``.

Data-parallel training on one host: ``torchrun --nproc-per-node N -m hdrnet_b200.bin.train ...``
(``WORLD_SIZE`` > 1) runs one process per GPU, rank r on ``cuda:(LOCAL_RANK % device_count)``, and
trains what one process with the same flags trains, up to the order of float32 sums.
``--batch_size`` is the global batch, as in the reference; N must divide it (``ValueError`` before
any data is read), and rank r builds rows ``[r B / N, (r + 1) B / N)`` of each batch on either data
tier.  The initial variables are broadcast from rank 0.  After ``backward`` the gradients are
averaged over the ranks with one all-reduce of a flat float32 buffer, so every rank takes the same
Adam step; with ``--guide_batch_stats`` the guide's batch norm uses the whole batch's statistics
(models merges the ranks' moments).  One small all-reduce per step averages the logged loss and PSNR
and carries rank 0's decisions to evaluate and to checkpoint, so no rank decides from its own clock.
Rank 0 alone logs, writes ``train_log.jsonl`` and writes the checkpoints (``on_stop.ckpt`` after an
interrupt included); before each checkpoint the ranks compare a digest of their variables and Adam
moments and raise if they have drifted apart.  The evaluation splits the eval set by index over the
ranks.  The world size is not a model parameter and is not written to ``params.json``: a checkpoint
resumes with any world size, since the batches depend only on ``(seed, step)`` and the global batch.
Without ``WORLD_SIZE`` (or with 1) no process group is made and no collective runs.

``--data_pipeline UnsharpMaskDataPipeline --blur_sigma S --sharpen A`` trains from input images alone,
as the reference's ``scripts/usm/*.sh`` recipes do: ``data_dir`` (and ``--eval_data_dir``) needs
``filelist.txt`` and ``input/`` only, and each target is the unsharp mask
``clip(x + A (x - G_S * x), 0, 1)`` of its input, computed on the device in source coordinates
(data_pipeline.UnsharpMaskDataPipeline defines it).  Both flags are required with that pipeline and
refused with ``ImageFilesDataPipeline``; 0 < S <= 32 and a finite A, else the parser refuses.  The two
values go into every checkpoint as the scalars ``train/usm_blur_sigma`` and ``train/usm_sharpen``
(``bin/run.py``, ``freeze_model`` and ``import_checkpoint`` read only ``inference/*``), and a resume
with other values, or with the other pipeline, is refused before any data is read.

Deliberate differences from the reference:

* ``--max_steps`` (the reference runs until interrupted), ``--seed``, ``--train_guide`` and
  ``--guide_batch_stats`` are added (the reference always trains the guide, in training mode; here
  both are opt-in);
  ``--data_pipeline`` takes ``ImageFilesDataPipeline`` and ``UnsharpMaskDataPipeline`` (the tfrecord
  pipelines need TF).  The reference's ``data_pipeline.py`` does not define ``UnsharpMaskDataPipeline``
  and its parser has no ``--blur_sigma`` or ``--sharpen``, though its ``usm/`` scripts pass them; the
  pipeline and both flags are this project's definition (data_pipeline.py);
  ``--profiling`` is accepted and ignored.
* The evaluation reads ``--eval_data_dir``.  The reference builds the eval pipeline but then
  evaluates the training samples (train.py:86 takes ``train_data_pipeline.samples``, and :105
  scores the training ``prediction``); that is not copied.
* The network input is ``--net_input_size``; the reference's pipeline hard-codes 256
  (data_pipeline.py:166).  The two are equal at the default.
* ``torch.optim.Adam`` adds eps to sqrt(v_hat), the bias-corrected second moment; TF1's
  AdamOptimizer adds its epsilon (``eps-hat``) to sqrt(v) and folds the bias correction into the
  step size.  With eps = 1e-8 the two differ only while sqrt(v) is of the order of eps.
* No queue runners, summaries or TF event files: batches are built on the device when needed and
  the scalars go to ``train_log.jsonl``.  The random streams are not TF's (data_pipeline.py).
* Every file is decoded once at start-up.  By default the decoded dataset is held in host memory, so
  it must fit there, and every rank holds its own copy.  ``--decoded_cache DIR`` instead decodes each
  file once into an on-disk cache at DIR (``data_pipeline.DecodedCache``) and maps its entries: the
  page cache holds one copy for all ranks, a dataset larger than RAM is paged in from disk as the
  crops read it, and a later run or resume opens the entries without decoding.  Under ``torchrun``
  the ranks split the decoding of missing entries, for the training and the eval set.  It applies
  to ``data_dir`` and ``--eval_data_dir`` with either pipeline, gives the same batches and so the
  same checkpoints, and is not a model parameter: it is not written to ``params.json`` or to the
  checkpoints, and a resume may add or drop it.
"""
from __future__ import annotations

import argparse
import json
import logging
import os
import sys
import time

import numpy as np
import torch

import torch.distributed as dist

from hdrnet_b200 import checkpoint, data_pipeline, metrics, models, parallel

logging.basicConfig(format="[%(process)d] %(levelname)s %(filename)s:%(lineno)s | %(message)s")
log = logging.getLogger("train")
log.setLevel(logging.INFO)

COEFFS = "inference/coefficients/"
GUIDE = "inference/guide/"
EMA_DECAY = 0.99
BETA1, BETA2 = 0.9, 0.999       # tf.train.AdamOptimizer's and torch.optim.Adam's defaults


def build_parser() -> argparse.ArgumentParser:
    """train.py:188-244, plus --max_steps and --seed."""
    parser = argparse.ArgumentParser(description="Train an HDRNet model from image pairs.")
    req_grp = parser.add_argument_group("required")
    req_grp.add_argument("checkpoint_dir", default=None, help="directory to save checkpoints to.")
    req_grp.add_argument("data_dir", default=None, help="directory with filelist.txt, input/ and output/ (or that filelist.txt).")
    req_grp.add_argument("--eval_data_dir", default=None, type=str, help="directory with the validation data.")

    train_grp = parser.add_argument_group("training")
    train_grp.add_argument("--learning_rate", default=1e-4, type=float, help="learning rate for the stochastic gradient update.")
    train_grp.add_argument("--log_interval", type=int, default=1, help="interval between log messages (in s).")
    train_grp.add_argument("--summary_interval", type=int, default=120, help="interval between scalar records in train_log.jsonl (in s)")
    train_grp.add_argument("--checkpoint_interval", type=int, default=600, help="interval between model checkpoints (in s)")
    train_grp.add_argument("--eval_interval", type=int, default=3600, help="interval between evaluations (in s)")
    train_grp.add_argument("--max_steps", type=int, default=None, help="stop when the global step reaches this (default: run until interrupted).")
    train_grp.add_argument("--seed", type=int, default=0, help="seed of the initial variables and of the data sampler.")
    train_grp.add_argument("--train_guide", dest="train_guide", action="store_true",
                           help="train the guide's variables too, as the reference does (the pointwise-NN guide "
                                "and the pyramid's guides need --guide_batch_stats).")
    train_grp.add_argument("--notrain_guide", dest="train_guide", action="store_false")
    train_grp.add_argument("--guide_batch_stats", dest="guide_batch_stats", action="store_true",
                           help="run the pointwise-NN guides' batch norm in training mode (batch statistics, "
                                "moving averages updated), as the reference does (HDRNetPointwiseNNGuide and "
                                "HDRNetGaussianPyrNN).")
    train_grp.add_argument("--noguide_batch_stats", dest="guide_batch_stats", action="store_false")
    train_grp.add_argument("--coefficient_batch_stats", dest="coefficient_batch_stats", action="store_true",
                           help="run the coefficient network's batch norm (--batch_norm) in training mode (batch "
                                "statistics, moving averages updated) and train its betas, as the reference does.")
    train_grp.add_argument("--nocoefficient_batch_stats", dest="coefficient_batch_stats", action="store_false")

    debug_grp = parser.add_argument_group("debug and profiling")
    debug_grp.add_argument("--profiling", dest="profiling", action="store_true", help="accepted for compatibility; ignored.")
    debug_grp.add_argument("--noprofiling", dest="profiling", action="store_false")

    data_grp = parser.add_argument_group("data pipeline")
    data_grp.add_argument("--batch_size", default=16, type=int, help="size of a batch for each gradient update.")
    data_grp.add_argument("--data_threads", default=2, type=int,
                          help="number of threads that decode the images at start-up (and pack streamed batches).")
    data_grp.add_argument("--rotate", dest="rotate", action="store_true", help="rotate data augmentation.")
    data_grp.add_argument("--norotate", dest="rotate", action="store_false")
    data_grp.add_argument("--flipud", dest="flipud", action="store_true", help="flip up/down data augmentation.")
    data_grp.add_argument("--noflipud", dest="flipud", action="store_false")
    data_grp.add_argument("--fliplr", dest="fliplr", action="store_true", help="flip left/right data augmentation.")
    data_grp.add_argument("--nofliplr", dest="fliplr", action="store_false")
    data_grp.add_argument("--random_crop", dest="random_crop", action="store_true", help="random crop data augmentation.")
    data_grp.add_argument("--norandom_crop", dest="random_crop", action="store_false")
    data_grp.add_argument("--blur_sigma", default=None, type=float,
                          help="UnsharpMaskDataPipeline: standard deviation of the target's Gaussian blur, in source "
                               "pixels (0 < S <= 32).")
    data_grp.add_argument("--sharpen", default=None, type=float,
                          help="UnsharpMaskDataPipeline: the target is clip(x + sharpen * (x - blur(x)), 0, 1).")
    data_grp.add_argument("--decoded_cache", default=None, type=str, metavar="DIR",
                          help="decode each image once into this on-disk cache and map it, instead of holding the "
                               "decoded dataset in memory (data_dir and --eval_data_dir; shared by ranks and runs).")

    model_grp = parser.add_argument_group("model_params")
    model_grp.add_argument("--model_name", default=models.__all__[0], type=str, help="classname of the model to use.",
                           choices=models.__all__[:4])
    model_grp.add_argument("--data_pipeline", default="ImageFilesDataPipeline", help="classname of the data pipeline to use.",
                           choices=data_pipeline.__all__)
    model_grp.add_argument("--net_input_size", default=256, type=int, help="size of the network's lowres image input.")
    model_grp.add_argument("--output_resolution", default=[512, 512], type=int, nargs=2, help="resolution of the output image.")
    model_grp.add_argument("--batch_norm", dest="batch_norm", action="store_true", help="normalize batches. If False, uses the moving averages.")
    model_grp.add_argument("--nobatch_norm", dest="batch_norm", action="store_false")
    model_grp.add_argument("--channel_multiplier", default=1, type=int, help="Factor to control net throughput (number of intermediate channels).")
    model_grp.add_argument("--guide_complexity", default=16, type=int, help="Control complexity of the guide network.")
    model_grp.add_argument("--luma_bins", default=8, type=int, help="Number of BGU bins for the luminance.")
    model_grp.add_argument("--spatial_bin", default=16, type=int, help="Size of the spatial BGU bins (pixels).")

    parser.set_defaults(profiling=False, flipud=False, fliplr=False, rotate=False, random_crop=True, batch_norm=False,
                        train_guide=False, guide_batch_stats=False, coefficient_batch_stats=False)
    parser.model_group = model_grp
    return parser


def model_params(parser, args) -> dict:
    """The model_params group, as train.py:250-252 collects it (and params.json stores it)."""
    return {a.dest: getattr(args, a.dest, None) for a in parser.model_group._group_actions}


def check_data_flags(parser, args) -> None:
    """parser.error unless ``--blur_sigma`` and ``--sharpen`` are given exactly with
    ``--data_pipeline UnsharpMaskDataPipeline``, with values ``data_pipeline.check_usm`` accepts."""
    given = [f for f in ("blur_sigma", "sharpen") if getattr(args, f, None) is not None]
    if args.data_pipeline == "UnsharpMaskDataPipeline":
        if len(given) != 2:
            parser.error("--data_pipeline UnsharpMaskDataPipeline needs --blur_sigma and --sharpen")
        try:
            data_pipeline.check_usm(args.blur_sigma, args.sharpen)
        except ValueError as e:
            parser.error(f"--blur_sigma / --sharpen: {e}")
    elif given:
        parser.error(f"--{given[0]} sets the unsharp-mask target of --data_pipeline UnsharpMaskDataPipeline; "
                     f"{args.data_pipeline} reads its targets from output/")


def usm_values(args):
    """``(blur_sigma, sharpen)`` of an UnsharpMaskDataPipeline run, else None."""
    if getattr(args, "data_pipeline", "ImageFilesDataPipeline") != "UnsharpMaskDataPipeline":
        return None
    return float(args.blur_sigma), float(args.sharpen)


USM_KEYS = ("train/usm_blur_sigma", "train/usm_sharpen")


PYRAMID_FLAGS = "--train_guide --guide_batch_stats"
CURVES_MODELS = ("HDRNetCurves", "HDRNetGaussianPyr")   # their guides have no batch norm


def refuse_untrainable(params, train_guide=False, guide_batch_stats=False, coefficient_batch_stats=False) -> None:
    """NotImplementedError, with the models' own text, for what cannot be trained: the pyramid model
    other than with ``train_guide`` and ``guide_batch_stats`` together, the coefficient network's batch
    norm without ``coefficient_batch_stats`` and (with ``train_guide``) the pointwise-NN guide without
    ``guide_batch_stats``.  Asks the models themselves, on the CPU, with a stand-in variable that
    requires grad (they refuse before any device work).  ValueError for ``guide_batch_stats`` on
    ``HDRNetCurves`` and ``HDRNetGaussianPyr``, whose guides have no batch norm, for ``coefficient_batch_stats`` without
    ``batch_norm``, and for ``coefficient_batch_stats`` on the models with a batch-normed guide without
    ``guide_batch_stats`` (the reference runs every batch norm of the model in training mode)."""
    S = int(params["net_input_size"])
    if coefficient_batch_stats and not params["batch_norm"]:
        raise ValueError("--coefficient_batch_stats runs the coefficient network's batch norm in training mode; "
                         "it needs --batch_norm")
    if coefficient_batch_stats and params["model_name"] not in CURVES_MODELS and not guide_batch_stats:
        raise ValueError(f"--coefficient_batch_stats with {params['model_name']} needs --guide_batch_stats: the "
                         "reference runs every batch norm of the model, the guide's included, in training mode")
    if params["model_name"] == "HDRNetGaussianPyrNN" and not (train_guide and guide_batch_stats):
        # the pyramid trains only as the reference's recipes train it: all three guides, in training mode
        probe = {COEFFS + "splat/conv1/weights": torch.zeros(1, requires_grad=True)}
        try:
            models.HDRNetGaussianPyrNN.inference(torch.zeros(1, S, S, 3), torch.zeros(1, 1, 1, 3),
                                                 dict(params, weights=probe))
        except NotImplementedError as e:
            raise NotImplementedError(f"{e}; {PYRAMID_FLAGS} trains the pyramid: its three guides, in "
                                      "training mode") from None
    if params["batch_norm"] and not coefficient_batch_stats:
        probe = {f"{scope}/BatchNorm/beta": torch.zeros(1, requires_grad=True)
                 for scope, use_bn, _ in models._coefficient_specs(params) if use_bn}
        try:
            getattr(models, params["model_name"])._coefficients(torch.zeros(1, S, S, 3), dict(params, weights=probe))
        except NotImplementedError as e:
            raise NotImplementedError(f"{e}; --coefficient_batch_stats runs it in training mode and trains it") from None
    if guide_batch_stats and params["model_name"] == "HDRNetCurves":
        raise ValueError("--guide_batch_stats runs the pointwise-NN guide's batch norm in training mode; "
                         "HDRNetCurves' guide has no batch norm")
    if guide_batch_stats and params["model_name"] == "HDRNetGaussianPyr":
        raise ValueError("--guide_batch_stats runs the pointwise-NN guide's batch norm in training mode; "
                         "HDRNetGaussianPyr's guides are curves, with no batch norm")
    if train_guide and not guide_batch_stats and params["model_name"] == "HDRNetPointwiseNNGuide":
        probe = {GUIDE + "conv2/weights": torch.zeros(1, requires_grad=True)}
        try:
            models.HDRNetPointwiseNNGuide.inference(torch.zeros(1, S, S, 3), torch.zeros(1, 1, 1, 3),
                                                    dict(params, weights=probe, guide_grad=True))
        except NotImplementedError as e:
            raise NotImplementedError(f"{e}; --guide_batch_stats runs it in training mode and trains it") from None


def refuse_resume_mismatch(saved: dict, train_guide: bool, usm=None) -> None:
    """ValueError when a checkpoint to resume was written with the other --[no]train_guide (its guide
    variables have Adam slots exactly when it trained them), or with another data pipeline or other
    unsharp-mask values than ``usm`` (``usm_values``: the checkpoint's ``train/usm_*`` scalars)."""
    saved_usm = tuple(float(saved[k]) for k in USM_KEYS) if all(k in saved for k in USM_KEYS) else None
    if usm is None and saved_usm is not None:
        raise ValueError("the checkpoint to resume was trained with --data_pipeline UnsharpMaskDataPipeline "
                         f"--blur_sigma {saved_usm[0]:g} --sharpen {saved_usm[1]:g}: resume it with those flags")
    if usm is not None and saved_usm is None:
        raise ValueError("the checkpoint to resume was trained on image pairs (ImageFilesDataPipeline): resume it "
                         "without --data_pipeline UnsharpMaskDataPipeline, or start a new checkpoint_dir")
    if usm is not None and tuple(float(v) for v in usm) != saved_usm:
        raise ValueError(f"the checkpoint to resume was trained with --blur_sigma {saved_usm[0]!r} --sharpen "
                         f"{saved_usm[1]!r}, not {float(usm[0])!r} and {float(usm[1])!r}: resume it with its own "
                         "values, or start a new checkpoint_dir")
    has_slots = any(k.startswith(GUIDE) and k.endswith(("/Adam", "/Adam_1")) for k in saved)
    if train_guide and not has_slots:
        raise ValueError("the checkpoint to resume was trained with the guide held fixed (no Adam slots for "
                         "inference/guide/*): resume it without --train_guide, or start a new checkpoint_dir")
    if has_slots and not train_guide:
        raise ValueError("the checkpoint to resume was trained with --train_guide (it holds Adam slots for "
                         "inference/guide/*): resume it with --train_guide")


def trained_names(variables, train_guide=False):
    """The variables Adam trains: the coefficient network's, and with ``train_guide`` the guide's;
    never a batch norm's ``moving_mean`` / ``moving_variance``, which the training-mode forward
    updates (TF does not train them)."""
    prefixes = (COEFFS, GUIDE) if train_guide else (COEFFS,)
    return sorted(k for k in variables if k.startswith(prefixes) and "/BatchNorm/moving_" not in k)


def slot_names(name):
    """TF's names of Adam's first and second moment of variable ``name``."""
    return name + "/Adam", name + "/Adam_1"


def checkpoint_tensors(variables: dict, moments: dict, step: int, ema: dict, usm=None) -> dict:
    """What a checkpoint holds, as numpy arrays: the variables, Adam's moments ``{name: (m, v)}``
    under TF's slot names, ``global_step`` (int64), TF's ``beta1_power`` / ``beta2_power``
    accumulators (beta^(step + 1)), the logged moving averages and, for an UnsharpMaskDataPipeline
    run, ``usm = (blur_sigma, sharpen)`` as float64 scalars ``train/usm_blur_sigma`` and
    ``train/usm_sharpen``."""
    t = {k: np.asarray(v) for k, v in variables.items()}
    for k, (m, v) in moments.items():
        sm, sv = slot_names(k)
        t[sm], t[sv] = np.asarray(m, np.float32), np.asarray(v, np.float32)
    t["global_step"] = np.array(step, np.int64)
    t["beta1_power"] = np.array(BETA1 ** (step + 1), np.float32)
    t["beta2_power"] = np.array(BETA2 ** (step + 1), np.float32)
    for key, val in ema.items():
        t[f"train/{key}_ema"] = np.array(val, np.float64)
    if usm is not None:
        for key, val in zip(USM_KEYS, usm):
            t[key] = np.array(val, np.float64)
    return t


def restored_state(saved: dict, variables, trained):
    """(variables, moments, step, ema) of a checkpoint read by read_tf_checkpoint: ``variables``
    names every variable the model needs, ``trained`` those with Adam moments."""
    missing = [k for k in list(variables) + [s for k in trained for s in slot_names(k)] + ["global_step"]
               if k not in saved]
    if missing:
        raise ValueError(f"the checkpoint lacks {missing[0]} ({len(missing)} missing): not a training checkpoint "
                         "of this model")
    values = {k: np.asarray(saved[k], np.float32) for k in variables}
    moments = {k: tuple(np.asarray(saved[s], np.float32) for s in slot_names(k)) for k in trained}
    ema = {key[len("train/"):-len("_ema")]: float(v) for key, v in saved.items()
           if key.startswith("train/") and key.endswith("_ema")}
    return values, moments, int(saved["global_step"]), ema


class Trainer:
    """The training state of one run: variables, Adam, the data pipelines, the step counter."""

    def __init__(self, args, params):
        self.args, self.params = args, params
        os.makedirs(args.checkpoint_dir, exist_ok=True)
        self.mdl = getattr(models, params["model_name"])
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.world = parallel.world_size()
        self.rank = dist.get_rank() if self.world > 1 else 0
        if self.rank:
            log.setLevel(logging.WARNING)           # rank 0 speaks for the run
        init = parallel.broadcast_weights(models.init_weights(params, seed=args.seed,
                                                              model_name=params["model_name"]))
        self.weights = {k: torch.from_numpy(v).to(self.device) for k, v in init.items()}
        self.names = trained_names(self.weights, args.train_guide)
        for k in self.names:
            self.weights[k].requires_grad_(True)
        self.opt = torch.optim.Adam([self.weights[k] for k in self.names], lr=args.learning_rate,
                                    betas=(BETA1, BETA2))
        self.step = 0
        self.ema = {"loss": 0.0, "psnr": 0.0}
        self._resume()
        if args.train_guide:
            log.info("%s: training the %d coefficient-network and guide variables (the guide is trained)",
                     params["model_name"], len(self.names))
        else:
            log.info("%s: training the %d coefficient-network variables; the guide variables (%s*) are held fixed "
                     "at their %s values", params["model_name"], len(self.names), GUIDE,
                     "restored" if self.step else "initial")
        self.usm = usm_values(args)
        if self.usm is None:
            pipeline, data_kw = data_pipeline.ImageFilesDataPipeline, {}
        else:
            pipeline = data_pipeline.UnsharpMaskDataPipeline
            data_kw = {"blur_sigma": self.usm[0], "sharpen": self.usm[1]}
            log.info("targets: unsharp masks of the inputs (blur_sigma %g, sharpen %g)", *self.usm)
        if getattr(args, "decoded_cache", None) is not None:
            data_kw["decoded_cache"] = args.decoded_cache
        self.train_data = pipeline(
            args.data_dir, batch_size=args.batch_size, output_resolution=args.output_resolution, shuffle=True,
            fliplr=args.fliplr, flipud=args.flipud, rotate=args.rotate, random_crop=args.random_crop,
            params=params, nthreads=args.data_threads, seed=args.seed, device=self.device,
            shard=(self.rank, self.world), **data_kw)
        self.eval_data = None
        if args.eval_data_dir is not None:
            self.eval_data = pipeline(
                args.eval_data_dir, batch_size=1, output_resolution=args.output_resolution, shuffle=False,
                params=params, nthreads=args.data_threads if "decoded_cache" in data_kw else 1, device=self.device,
                **data_kw)
        for data in (self.train_data, self.eval_data):
            dc = getattr(data, "decoded_cache", None)
            if dc is not None:
                log.info("%s: decoded cache %s: %d entries valid, %d built, %.1f MB mapped", data.path,
                         dc.directory, dc.valid, dc.built, dc.nbytes / 1e6)
        self.p = dict(params, weights=self.weights)
        if args.train_guide:
            self.p["guide_grad"] = True
        coefficient_batch_stats = bool(getattr(args, "coefficient_batch_stats", False))
        if coefficient_batch_stats:
            self.p["coefficient_batch_stats"] = True
        self.is_training = bool(getattr(args, "guide_batch_stats", False)) or coefficient_batch_stats
        if getattr(args, "guide_batch_stats", False):
            log.info("%s: the guide's batch norm runs in training mode (batch statistics; moving averages "
                     "updated each step)", params["model_name"])
        if coefficient_batch_stats:
            log.info("%s: the coefficient network's batch norm runs in training mode (batch statistics; moving "
                     "averages updated each step)", params["model_name"])

    # ---- checkpoints ---------------------------------------------------------------------------
    def _resume(self):
        prefix = checkpoint.latest_checkpoint(self.args.checkpoint_dir)
        if prefix is None:
            return
        saved = checkpoint.read_tf_checkpoint(prefix)
        refuse_resume_mismatch(saved, self.args.train_guide, usm_values(self.args))
        values, moments, step, ema = restored_state(saved, self.weights, self.names)
        with torch.no_grad():
            for k, v in self.weights.items():
                v.copy_(torch.from_numpy(values[k]).reshape(v.shape))
        for k in self.names:
            var = self.weights[k]
            m, v = (torch.from_numpy(a).reshape(var.shape).to(self.device) for a in moments[k])
            self.opt.state[var] = {"step": torch.tensor(float(step)), "exp_avg": m, "exp_avg_sq": v}
        self.step = step
        self.ema.update(ema)
        log.info("resumed %s at step %d", prefix, step)

    def save(self, name=None, check_ranks=True):
        """Write ``model.ckpt-<step>`` (or ``name``) and params.json; returns the prefix.  Under a
        process group every rank calls it: with ``check_ranks`` the ranks first compare a digest of
        their variables and Adam moments (RuntimeError when they have drifted apart), then rank 0
        alone writes, since every rank holds the same state."""
        prefix = os.path.join(self.args.checkpoint_dir, name or f"model.ckpt-{self.step}")
        moments = {}
        for k in self.names:
            st = self.opt.state.get(self.weights[k])
            zero = torch.zeros_like(self.weights[k])
            moments[k] = (st["exp_avg"] if st else zero).cpu().numpy(), (st["exp_avg_sq"] if st else zero).cpu().numpy()
        variables = {k: v.detach().cpu().numpy() for k, v in self.weights.items()}
        if check_ranks:
            parallel.check_ranks_agree([variables[k] for k in sorted(variables)]
                                       + [a for k in self.names for a in moments[k]],
                                       f"the variables and Adam moments at step {self.step}")
        if self.rank:
            return prefix
        checkpoint.write_tf_checkpoint(prefix, checkpoint_tensors(variables, moments, self.step, self.ema,
                                                                  usm_values(self.args)))
        with open(os.path.join(self.args.checkpoint_dir, "params.json"), "w") as f:
            json.dump(self.params, f)
        log.info("saved %s", prefix)
        return prefix

    # ---- steps ---------------------------------------------------------------------------------
    def train_step(self):
        """One gradient step on batch ``self.step`` (this rank's shard of it); returns (loss, psnr)
        over the shard as device scalars.  Under a process group the gradients are averaged over the
        ranks (parallel.all_reduce_mean_, one all-reduce) before Adam, so every rank takes the step of
        the whole batch's mean loss."""
        batch = self.train_data.batch(self.step)
        self.opt.zero_grad(set_to_none=True)
        pred = self.mdl.inference(batch["lowres_input"], batch["image_input"], self.p,
                                  is_training=self.is_training)
        loss = metrics.l2_loss(batch["image_output"], pred)
        with torch.no_grad():
            psnr = metrics.psnr(batch["image_output"], pred)
        loss.backward()
        if self.world > 1:
            for k in self.names:
                if self.weights[k].grad is None:
                    self.weights[k].grad = torch.zeros_like(self.weights[k])
            parallel.all_reduce_mean_([self.weights[k].grad for k in self.names])
        self.opt.step()
        self.step += 1
        return loss.detach(), psnr

    def evaluate(self) -> float:
        """Mean PSNR over the eval set (batch 1, no augmentation, centre crop).  Under a process group
        rank r scores images r, r + world, ... and the sums are added over the ranks."""
        total = 0.0
        with torch.no_grad():
            for i in range(self.rank, self.eval_data.nsamples, self.world):
                b = self.eval_data.batch(i)
                total += float(metrics.psnr(b["image_output"],
                                            self.mdl.inference(b["lowres_input"], b["image_input"], self.p)))
        return float(parallel.sum_over_ranks([total])[0]) / self.eval_data.nsamples

    def record(self, rec):
        with open(os.path.join(self.args.checkpoint_dir, "train_log.jsonl"), "a") as f:
            f.write(json.dumps(rec) + "\n")

    def close(self):
        """Stop the data pipelines' threads (those of a streamed tier)."""
        for data in (self.train_data, self.eval_data):
            if data is not None:
                data.close()

    def run(self):
        a = self.args
        t0 = time.time()
        last_log = last_summary = last_ckpt = last_eval = t0
        interrupted = False
        try:
            while a.max_steps is None or self.step < a.max_steps:
                loss_t, psnr_t = self.train_step()
                loss, psnr = float(loss_t), float(psnr_t)
                now = time.time()
                lead = self.rank == 0       # rank 0's clock decides what every rank does this step
                evaluate = lead and self.eval_data is not None and now - last_eval >= a.eval_interval
                save = lead and now - last_ckpt >= a.checkpoint_interval
                if self.world > 1:          # one all-reduce: the shards' mean scalars and rank 0's decisions
                    loss, psnr, evaluate, save = parallel.sum_over_ranks([loss, psnr, evaluate, save])
                    loss, psnr, evaluate, save = loss / self.world, psnr / self.world, evaluate > 0, save > 0
                for key, val in (("loss", loss), ("psnr", psnr)):
                    self.ema[key] = EMA_DECAY * self.ema[key] + (1.0 - EMA_DECAY) * val
                debias = 1.0 - EMA_DECAY ** self.step
                loss_ema, psnr_ema = self.ema["loss"] / debias, self.ema["psnr"] / debias
                if lead and now - last_log >= a.log_interval:
                    log.info("Step %d | loss = %.4f | psnr = %.1f dB", self.step, loss_ema, psnr_ema)
                    last_log = now
                if lead and now - last_summary >= a.summary_interval:
                    self.record({"step": self.step, "time": now - t0, "loss": loss, "psnr": psnr,
                                 "loss_ema": loss_ema, "psnr_ema": psnr_ema,
                                 "learning_rate": a.learning_rate, "batch_size": a.batch_size})
                    last_summary = now
                if evaluate:
                    log.info("Evaluating on %d images at step %d", self.eval_data.nsamples, self.step)
                    p = self.evaluate()
                    log.info("  Evaluation PSNR = %.1f dB", p)
                    if lead:
                        self.record({"step": self.step, "time": time.time() - t0, "eval_psnr": p})
                    last_eval = time.time()
                if save:
                    self.save()
                    last_ckpt = time.time()
        except KeyboardInterrupt:
            log.info("interrupted at step %d", self.step)
            interrupted = True
        finally:
            self.close()
        log.info("Training complete, saving chkpt %s", os.path.join(a.checkpoint_dir, "on_stop.ckpt"))
        # after an interrupt the other ranks may be anywhere in a step: no collective, rank 0 writes its state
        return self.save("on_stop.ckpt", check_ranks=not interrupted)


def main(argv=None):
    parser = build_parser()
    args = parser.parse_args(argv)
    check_data_flags(parser, args)
    params = model_params(parser, args)
    refuse_untrainable(params, args.train_guide, args.guide_batch_stats,      # before any data is read
                       args.coefficient_batch_stats)
    world = parallel.world_size() if dist.is_initialized() else int(os.environ.get("WORLD_SIZE", "1"))
    data_pipeline.check_shard((0, world), args.batch_size)
    prefix = checkpoint.latest_checkpoint(args.checkpoint_dir)
    if prefix is not None:
        refuse_resume_mismatch(checkpoint.read_tf_checkpoint(prefix), args.train_guide, usm_values(args))
    if args.profiling:
        log.warning("--profiling is accepted for compatibility and ignored")
    if not torch.cuda.is_available():
        raise RuntimeError("training needs a CUDA device; hdrnet_b200 has no CPU path")
    joined = False
    if world > 1:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")) % torch.cuda.device_count())
        joined = not dist.is_initialized()
        parallel.init_distributed()
    try:
        return Trainer(args, params).run()
    finally:
        if joined:
            parallel.finalize()


if __name__ == "__main__":
    try:
        main()
    except NotImplementedError as e:
        sys.exit(f"train.py: {e}")
