#!/usr/bin/env python
"""Freeze a trained model for deployment without Python: one file holding exactly the arrays the
kernels consume (batch norm folded), which ``hdrnet_model_create`` of the C-ABI, the ``hdrnet_run``
program and ``hdrnet_b200.frozen.FrozenModel`` load.  The counterpart of the reference's
hdrnet/bin/freeze_graph.py, for this project's kernels rather than a TF graph:

    python -m hdrnet_b200.bin.freeze_model <checkpoint_dir> [--output PATH]

``checkpoint_dir`` is anything ``hdrnet_b200.bin.run`` reads: ``weights.npz`` + ``params.json``, or a
TensorFlow training directory.  The default output is ``<checkpoint_dir>/frozen_model.hdrnet``.
"""
from __future__ import annotations

import argparse
import logging
import os

from hdrnet_b200 import checkpoint
from hdrnet_b200.bin.run import load_checkpoint

log = logging.getLogger("freeze_model")


def main(args):
    has_npz = os.path.exists(os.path.join(args.checkpoint_dir, "weights.npz"))
    if not (has_npz or checkpoint.latest_checkpoint(args.checkpoint_dir)):
        raise SystemExit(f"{args.checkpoint_dir}: no weights.npz and no TensorFlow checkpoint to freeze")
    params, weights = load_checkpoint(args.checkpoint_dir)
    out = args.output or os.path.join(args.checkpoint_dir, "frozen_model.hdrnet")
    checkpoint.freeze_model(weights, params, out)
    log.info("froze %s (%s) to %s", args.checkpoint_dir, params.get("model_name", "HDRNetCurves"), out)
    return out


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(description="freeze a trained model into one file for the C-ABI")
    ap.add_argument("checkpoint_dir", help="weights.npz + params.json, or a TensorFlow training directory")
    ap.add_argument("--output", default=None, help="output file (default <checkpoint_dir>/frozen_model.hdrnet)")
    return ap


if __name__ == "__main__":
    logging.basicConfig(level=logging.INFO)
    main(build_parser().parse_args())
