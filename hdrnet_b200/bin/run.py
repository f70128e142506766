#!/usr/bin/env python
"""Inference CLI: drop-in for the reference's ``hdrnet/bin/run.py`` (same positional
arguments and flags, hdrnet/bin/run.py:219-238):

    python -m hdrnet_b200.bin.run <checkpoint_dir> <input> <output> [--lowres_input X]
                                  [--hdrp] [--debug] [--limit N] [--output_bit_depth {8,16}]
                                  [--batch_size N]

``checkpoint_dir`` holds ``weights.npz`` (reference variable names, '/' written as '__') and
``params.json`` (the model_params the reference stores as graph constants, train.py:60-63,
read back by utils.get_model_params) instead of a TF checkpoint + meta graph.

Host-side pre/post processing follows the reference (run.py:139-190):
  cv2.imread(-1) -> drop alpha -> BGR->RGB -> img_as_float (u8 /255, u16 /65535; --hdrp only
  logs, both branches of run.py:156-164 call img_as_float) -> nearest-neighbour S x S lowres
  (skimage.transform.resize(order=0), run.py:168-169) -> model -> uint8(255 * clip(out, 0, 1))
  (truncating cast, run.py:95) -> PNG.  Everything after the decode runs on the device, on the
  integer pixels (models.*.inference_image).

``--output_bit_depth 16`` is an addition to the reference's CLI: the result is written as a 16-bit
PNG, rint(65535 * clip(out, 0, 1)) from the same fused kernel, instead of the 8-bit cast that drops
half the bits a model trained on 16-bit targets produces.  The default, 8, writes what the reference
writes; the ``--debug`` pictures are 8-bit either way.

``--batch_size N`` is another addition: with N > 1, N consecutive files of the listing (of one pixel
dtype) go through one ``inference_images`` call, whatever their sizes, and each file's PNG holds the
same bytes as with N = 1 (the default, which runs one ``inference_image`` call per file as before).
``--limit`` still counts files; ``--debug`` needs N = 1.
"""
from __future__ import annotations

import argparse
import json
import logging
import os
import re

import numpy as np
import torch

from hdrnet_b200 import models

logging.basicConfig(format="[%(process)d] %(levelname)s %(filename)s:%(lineno)s | %(message)s")
log = logging.getLogger("run")
log.setLevel(logging.INFO)


def get_input_list(path):
    """hdrnet/bin/run.py:42-58: a .txt file list, a directory of images, or one image."""
    regex = re.compile(r".*\.(png|jpeg|jpg|tif|tiff)$", re.IGNORECASE)
    if os.path.isdir(path):
        return sorted(os.path.join(path, f) for f in os.listdir(path) if regex.match(f))
    if os.path.splitext(path)[-1] == ".txt":
        dirname = os.path.dirname(path)
        with open(path) as fid:
            return [os.path.join(dirname, "input", line.strip()) for line in fid if line.strip()]
    return [path]


def img_as_float(im: np.ndarray) -> np.ndarray:
    """skimage.img_as_float for the dtypes run.py feeds it (run.py:162/164)."""
    if im.dtype == np.uint8:
        return im.astype(np.float32) / np.float32(255.0)
    if im.dtype == np.uint16:
        return im.astype(np.float32) / np.float32(65535.0)
    return im.astype(np.float32)


def nearest_resize(im: np.ndarray, size: int) -> np.ndarray:
    """skimage.transform.resize(im, [S, S], order=0) without anti-aliasing: output sample i
    reads input round((i + 0.5) * H / S - 0.5) (run.py:168-169)."""
    H, W = im.shape[:2]
    ys = np.clip(np.floor((np.arange(size) + 0.5) * H / size).astype(np.int64), 0, H - 1)
    xs = np.clip(np.floor((np.arange(size) + 0.5) * W / size).astype(np.int64), 0, W - 1)
    return im[ys][:, xs]


def load_checkpoint(checkpoint_dir):
    """``weights.npz`` + ``params.json``; or, like the reference (run.py:70-85, :136-142), a
    TensorFlow training directory: latest ``model.ckpt-N`` + its ``.meta`` model_params (read by
    hdrnet_b200.checkpoint, no TensorFlow needed; ``params.json`` there overrides the .meta)."""
    npz = os.path.join(checkpoint_dir, "weights.npz")
    pjson = os.path.join(checkpoint_dir, "params.json")
    if os.path.exists(npz):
        with open(pjson) as f:
            params = json.load(f)
        return params, models.load_weights(npz)
    from hdrnet_b200 import checkpoint
    params, weights = checkpoint.import_checkpoint(checkpoint_dir)
    if os.path.exists(pjson):
        with open(pjson) as f:
            params = json.load(f)
    if params is None:
        raise FileNotFoundError(f"{checkpoint_dir}: no params.json and no .meta file to read model_params from")
    models.set_weights(weights)
    return params, weights


def save_checkpoint(checkpoint_dir, params, weights):
    os.makedirs(checkpoint_dir, exist_ok=True)
    with open(os.path.join(checkpoint_dir, "params.json"), "w") as f:
        json.dump({k: v for k, v in params.items() if k != "weights"}, f)
    np.savez(os.path.join(checkpoint_dir, "weights.npz"),
             **{k.replace("/", "__"): np.asarray(v) for k, v in weights.items()})


def process(mdl, params, im_u: np.ndarray, lowres_u: np.ndarray | None = None, hdrp=False,
            out_dtype=torch.uint8):
    """One image through the model; returns uint8 HxWx3 -- uint16 with ``out_dtype=torch.uint16``
    -- (and the float output when params['debug'] asks for the collections).

    The decoded uint8 / uint16 pixels go to the device as they are (3 or 6 bytes per pixel);
    img_as_float, the nearest-neighbour network input, the model and the uint8 cast all run
    there (models.*.inference_image).  ``--hdrp`` only logs a notice in the reference: both of
    its branches call skimage.img_as_float (run.py:156-164), so it changes nothing here."""
    if im_u.ndim == 2:
        im_u = np.repeat(im_u[..., None], 3, axis=2)
    if im_u.shape[2] > 3:
        im_u = im_u[:, :, :3]                                      # run.py:146-148
    if hdrp and im_u.dtype == np.uint16:
        log.info("Using HDR+ hack for uint16 input. Assuming input white level is 32767.")

    def to_dev(a):
        if a.dtype not in (np.uint8, np.uint16):
            a = a.astype(np.float32)
        return torch.from_numpy(np.ascontiguousarray(a[None])).cuda()

    full_t = to_dev(im_u)
    low_t = None
    if lowres_u is not None:
        if lowres_u.ndim == 2:
            lowres_u = np.repeat(lowres_u[..., None], 3, axis=2)
        low_t = to_dev(lowres_u[:, :, :3])
    out_q = mdl.inference_image(full_t, params, lowres_image=low_t, out_dtype=out_dtype)  # run.py:95 cast included
    out = mdl.last_debug["output"] if params.get("debug") and hasattr(mdl, "last_debug") else None
    return out_q[0].cpu().numpy(), out


def _to_png(x01: np.ndarray) -> np.ndarray:
    """A [0, 1] float image as skimage.io.imsave stores it (uint8, round to nearest)."""
    return np.clip(np.rint(x01 * 255.0), 0, 255).astype(np.uint8)


def debug_images(im_rgb: np.ndarray, coeffs: np.ndarray, guides: list, multiscale=()) -> dict:
    """The --debug pictures of the reference (run.py:98-133, :192-215) as {file suffix: image}:
    the input, the coefficient mosaic ([gh*gd, gw*n_in*n_out], symmetric normalisation
    (x + m) / 2m with m = max |x|), one normalised picture per guide map and -- for the pyramid
    model's 'multiscale' collection (run.py:108-117, :201-205) -- one picture per level with its
    channels side by side ([H, C*W])."""
    out = {"_input.png": np.ascontiguousarray(im_rgb[:, :, ::-1])}
    gh, gw, gd, no, ni = coeffs.shape
    c = np.transpose(coeffs, (2, 0, 3, 4, 1)).reshape(gh * gd, gw * ni * no)   # tf.transpose [0,3,1,4,5,2]
    m = float(np.abs(c).max()) or 1.0
    out["_coeffs.png"] = _to_png(np.clip((c + m) / (2 * m), 0, 1))
    for i, g in enumerate(guides):
        mg = float(np.abs(g).max()) or 1.0
        out[f"_guide_{i}.png"] = _to_png(np.clip((g + mg) / (2 * mg), 0, 1))
    for i, m in enumerate(multiscale):                               # [H, W, C] -> [H, C * W]
        mm = float(np.abs(m).max()) or 1.0
        m = np.clip((m + mm) / (2 * mm), 0, 1)
        out[f"_ms_{i}.png"] = _to_png(np.transpose(m, (0, 2, 1)).reshape(m.shape[0], -1))
    return out


def _rgb3(im: np.ndarray) -> np.ndarray:
    """process()'s channel handling: grey to three channels, alpha dropped."""
    if im.ndim == 2:
        im = np.repeat(im[..., None], 3, axis=2)
    return np.ascontiguousarray(im[:, :, :3])


def process_batch(mdl, params, ims: list, lowres: list, out_dtype=torch.uint8) -> list:
    """Several decoded images of one dtype, each of its own size, through one ``inference_images``
    call; ``lowres`` holds each image's network-input image or None (the image itself).  Returns
    one HxWx3 array per image, the bytes ``process`` returns for it."""
    def to_dev(a):
        if a.dtype not in (np.uint8, np.uint16):
            a = a.astype(np.float32)
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()

    full = [to_dev(_rgb3(im)) for im in ims]
    low = None
    if any(lo is not None for lo in lowres):
        low = [full[i] if lo is None else to_dev(_rgb3(lo)) for i, lo in enumerate(lowres)]
    return [o.cpu().numpy() for o in mdl.inference_images(full, params, lowres_images=low, out_dtype=out_dtype)]


def main(args):
    # callers that build the namespace themselves may leave the flag out: 8, as the parser's default
    out_dtype = OUTPUT_DTYPES[int(getattr(args, "output_bit_depth", 8))]
    batch_size = int(getattr(args, "batch_size", 1))
    if batch_size < 1:
        raise ValueError(f"--batch_size must be at least 1, got {batch_size}")
    if batch_size > 1 and args.debug:
        raise ValueError("--debug writes one image's collections: it needs --batch_size 1")
    import cv2
    params, _ = load_checkpoint(args.checkpoint_dir)
    mdl = getattr(models, params["model_name"])                     # run.py:82-85
    params["debug"] = bool(args.debug)
    paths = get_input_list(args.input)
    if args.limit is not None:
        paths = paths[:args.limit]
    os.makedirs(args.output, exist_ok=True)
    if batch_size > 1:
        _run_batches(cv2, mdl, params, args, paths, batch_size, out_dtype)
        return
    for i, path in enumerate(paths):
        log.info("Processing %s (%d/%d)", path, i + 1, len(paths))
        bgr = cv2.imread(path, -1)
        if bgr is None:
            log.warning("could not read %s", path)
            continue
        rgb = bgr[:, :, :3][:, :, ::-1] if bgr.ndim == 3 else bgr   # run.py:150
        low_u = None
        if args.lowres_input is not None:
            lp = os.path.join(args.lowres_input, os.path.basename(path))
            lb = cv2.imread(lp, -1)
            low_u = lb[:, :, :3][:, :, ::-1] if lb is not None and lb.ndim == 3 else lb
        out_q, _ = process(mdl, params, np.ascontiguousarray(rgb), low_u, hdrp=args.hdrp, out_dtype=out_dtype)
        name = os.path.splitext(os.path.basename(path))[0]
        cv2.imwrite(os.path.join(args.output, name + ".png"), out_q[:, :, ::-1])
        if args.debug:                                              # run.py:192-215
            dbg = mdl.last_debug
            guides = dbg["guide"] if isinstance(dbg["guide"], (list, tuple)) else [dbg["guide"]]
            coeffs = dbg["bilateral_coefficients"][0].cpu().numpy()
            np.save(os.path.join(args.output, name + "_guide.npy"), guides[0][0].cpu().numpy())
            np.save(os.path.join(args.output, name + "_coefficients.npy"), coeffs)
            ms = [m[0].cpu().numpy() for m in dbg.get("multiscale", ())]
            for fname, img in debug_images(rgb, coeffs, [g[0].cpu().numpy() for g in guides], ms).items():
                cv2.imwrite(os.path.join(args.output, name + fname), img)


def _run_batches(cv2, mdl, params, args, paths, batch_size, out_dtype):
    """main() with --batch_size > 1: batch_size consecutive files per inference_images call (split
    where the pixel dtype changes, since one call takes one dtype)."""
    for start in range(0, len(paths), batch_size):
        group = []
        for j, path in enumerate(paths[start:start + batch_size]):
            log.info("Processing %s (%d/%d)", path, start + j + 1, len(paths))
            bgr = cv2.imread(path, -1)
            if bgr is None:
                log.warning("could not read %s", path)
                continue
            rgb = bgr[:, :, :3][:, :, ::-1] if bgr.ndim == 3 else bgr   # run.py:150
            if args.hdrp and rgb.dtype == np.uint16:
                log.info("Using HDR+ hack for uint16 input. Assuming input white level is 32767.")
            low_u = None
            if args.lowres_input is not None:
                lb = cv2.imread(os.path.join(args.lowres_input, os.path.basename(path)), -1)
                low_u = lb[:, :, :3][:, :, ::-1] if lb is not None and lb.ndim == 3 else lb
            group.append((path, rgb, low_u))
        while group:
            n = 1
            while n < len(group) and group[n][1].dtype == group[0][1].dtype:
                n += 1
            run, group = group[:n], group[n:]
            outs = process_batch(mdl, params, [g[1] for g in run], [g[2] for g in run], out_dtype)
            for (path, _, _), out_q in zip(run, outs):
                name = os.path.splitext(os.path.basename(path))[0]
                cv2.imwrite(os.path.join(args.output, name + ".png"), out_q[:, :, ::-1])


# --output_bit_depth -> the dtype inference_image returns and cv2.imwrite stores
OUTPUT_DTYPES = {8: torch.uint8, 16: torch.uint16}


def build_parser() -> argparse.ArgumentParser:
    parser = argparse.ArgumentParser()
    parser.add_argument("checkpoint_dir", type=str, help="directory with weights.npz + params.json")
    parser.add_argument("input", type=str, help="image, directory of images, or filelist.txt")
    parser.add_argument("output", type=str, help="output directory")
    parser.add_argument("--lowres_input", default=None, type=str)
    parser.add_argument("--hdrp", dest="hdrp", action="store_true", help="HDR+ inputs: 16-bit linear, white level 32767")
    parser.add_argument("--nohdrp", dest="hdrp", action="store_false")
    parser.add_argument("--debug", dest="debug", action="store_true")
    parser.add_argument("--limit", type=int)
    parser.add_argument("--output_bit_depth", type=int, choices=sorted(OUTPUT_DTYPES), default=8,
                        help="8: uint8 PNGs, as the reference writes; 16: 16-bit PNGs, rint(65535 * clip)")
    parser.add_argument("--batch_size", type=int, default=1,
                        help="files per model call; images of different sizes batch together (default 1)")
    parser.set_defaults(hdrp=False, debug=False)
    return parser


if __name__ == "__main__":
    main(build_parser().parse_args())
