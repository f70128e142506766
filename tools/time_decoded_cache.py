"""Time the training data path with and without the on-disk decoded cache (``--decoded_cache``).

In one run, with the card's name and power limit read in the same run, on a PNG dataset generated
from a seed in a temporary directory (``--pairs`` pairs of ``--width`` x ``--height`` uint16 inputs
and uint8 targets):
  1. start-up without the cache (every pair decoded into memory) against a cold cache build, with the
     same ``--data_threads``;
  2. a warm start: every entry valid, nothing decoded;
  3. the CLI's streamed-tier step (Trainer.train_step, then the loss read on the host) from the cache
     against from memory, at 16 x 512² and 1 x 2048², the cache resident in the page cache; windows
     alternated;
  4. the same step from the cache with the tool's own entry files evicted from the page cache before
     each window (their pages dropped from the maps with madvise(MADV_DONTNEED), then
     posix_fadvise(POSIX_FADV_DONTNEED) on each file): the larger-than-RAM case, with the bytes read
     from storage (``read_bytes`` of /proc/self/io), with and without madvise(MADV_RANDOM) on the
     maps, alternated.
The tool only touches its own files; it changes no system setting.  Prints one JSON object; --out
also writes it.

    python tools/time_decoded_cache.py [--pairs 64 --width 4032 --height 3024 --data_threads 4]
        [--steps 10 --warmup 3 --reps 3 --tmp DIR --out tools_out/decoded_cache.json]
"""
from __future__ import annotations

import argparse
import json
import mmap
import os
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from hdrnet_b200 import data_pipeline as dp  # noqa: E402
from hdrnet_b200.bin import train  # noqa: E402
from time_train_step import gpu_identity, timed  # noqa: E402

SHAPES = ((16, 512), (1, 2048))


def generate(root, n, H, W):
    """n pairs of uint16 inputs and uint8 targets: a per-pair ramp plus per-row noise, PNG level 1."""
    import cv2
    os.makedirs(os.path.join(root, "input"))
    os.makedirs(os.path.join(root, "output"))
    rng = np.random.RandomState(0)
    names = []
    for i in range(n):
        im = (np.arange(W, dtype=np.uint16)[None, :, None] * np.uint16(7 + i)
              + rng.randint(0, 4096, (H, 1, 3)).astype(np.uint16))
        name = f"{i:03d}.png"
        cv2.imwrite(os.path.join(root, "input", name), im, [cv2.IMWRITE_PNG_COMPRESSION, 1])
        cv2.imwrite(os.path.join(root, "output", name), (im >> 8).astype(np.uint8), [cv2.IMWRITE_PNG_COMPRESSION, 1])
        names.append(name)
    with open(os.path.join(root, "filelist.txt"), "w") as f:
        f.write("\n".join(names) + "\n")


def read_bytes():
    try:
        with open("/proc/self/io") as f:
            for line in f:
                if line.startswith("read_bytes:"):
                    return int(line.split()[1])
    except OSError:
        return None
    return None


def filesystem(path):
    """(mount point, type) of the filesystem holding ``path``."""
    best = ("", "unknown")
    with open("/proc/self/mounts") as f:
        for line in f:
            _, mnt, kind = line.split()[:3]
            if os.path.abspath(path).startswith(mnt.rstrip("/") + "/") and len(mnt) > len(best[0]):
                best = (mnt, kind)
    return best


def stream_trainer(tmp, data, B, oh, threads, cache=None, ram=None):
    """A Trainer on the streamed tier (a substituted device_budget lets only the staging slots fit),
    reading the maps of ``cache`` or, with ``ram``, the decoded arrays ``ram`` (load_pairs substituted)."""
    staging = dp.STREAM_SLOTS * dp.slot_bytes({(np.dtype(np.uint16), np.dtype(np.uint8))}, B, (oh, oh))
    keep = dp.device_budget, dp.load_pairs
    dp.device_budget = lambda device: dp.MEMORY_MARGIN + staging
    if ram is not None:
        dp.load_pairs = lambda path, nthreads=1: ram
    try:
        parser = train.build_parser()
        argv = [os.path.join(tmp, f"ckpt_{B}x{oh}_{'cache' if cache else 'ram'}"), data, "--fliplr", "--flipud",
                "--rotate", "--batch_size", str(B), "--output_resolution", str(oh), str(oh), "--data_threads",
                str(threads)] + (["--decoded_cache", cache] if cache else [])
        args = parser.parse_args(argv)
        t = train.Trainer(args, train.model_params(parser, args))
    finally:
        dp.device_budget, dp.load_pairs = keep
    assert t.train_data.tier == "stream"
    return t


def synced_step(t):
    def step():
        loss, psnr = t.train_step()
        float(loss), float(psnr)
    return step


def evict(maps, advice=None):
    """Drop ``maps``' pages from this process and their files' pages from the page cache; then give
    the maps ``advice`` (an madvise constant) when not None."""
    for m in maps:
        m._mmap.madvise(mmap.MADV_DONTNEED)
    for path in {m.filename for m in maps}:
        fd = os.open(path, os.O_RDONLY)
        try:
            os.posix_fadvise(fd, 0, 0, os.POSIX_FADV_DONTNEED)
        finally:
            os.close(fd)
    if advice is not None:
        for m in maps:
            m._mmap.madvise(advice)


def evicted_window(t, maps, steps, advice):
    evict(maps, advice)
    step = synced_step(t)
    r0 = read_bytes()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    ms = 1e3 * (time.perf_counter() - t0) / steps
    r1 = read_bytes()
    for m in maps:
        m._mmap.madvise(mmap.MADV_NORMAL)
    return ms, None if r0 is None else r1 - r0


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--width", type=int, default=4032)
    ap.add_argument("--height", type=int, default=3024)
    ap.add_argument("--data_threads", type=int, default=4)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--tmp", default=None, help="directory for the generated dataset and the cache")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_decoded_cache.py needs a CUDA device")
    res = {"gpu": gpu_identity(), "host_cpus": len(os.sched_getaffinity(0)), "pairs": a.pairs,
           "source": [a.height, a.width], "formats": "uint16 input, uint8 target", "data_threads": a.data_threads,
           "steps": a.steps, "warmup": a.warmup, "reps": a.reps}
    with tempfile.TemporaryDirectory(dir=a.tmp) as tmp:
        data, cache = os.path.join(tmp, "data"), os.path.join(tmp, "cache")
        res["filesystem"] = filesystem(tmp)
        t0 = time.perf_counter()
        generate(data, a.pairs, a.height, a.width)
        res["generate_s"] = time.perf_counter() - t0
        res["png_bytes"] = sum(os.path.getsize(os.path.join(data, s, n)) for s in ("input", "output")
                               for n in os.listdir(os.path.join(data, s)))

        # 1, 2: start-up
        t0 = time.perf_counter()
        ram = dp.load_pairs(data, a.data_threads)
        res["startup_in_memory_s"] = time.perf_counter() - t0
        res["decoded_bytes"] = sum(im.nbytes for im in ram[1] + ram[2])
        for key in ("cold", "warm"):
            dc = dp.DecodedCache(cache)
            t0 = time.perf_counter()
            dp.load_pairs(data, a.data_threads, cache=dc)
            res[f"startup_{key}_cache_s"] = time.perf_counter() - t0
            res[f"startup_{key}_cache_entries"] = {"valid": dc.valid, "built": dc.built}
        res["free_disk_bytes_after_build"] = shutil.disk_usage(tmp).free

        # 3, 4: the streamed tier's step
        for B, oh in SHAPES:
            key = f"{B}x{oh}"
            trainers = {"cache": stream_trainer(tmp, data, B, oh, a.data_threads, cache=cache),
                        "ram": stream_trainer(tmp, data, B, oh, a.data_threads, ram=ram)}
            try:
                for tag in ("a", "b"):
                    for name, t in trainers.items():
                        res[f"step_{key}_{name}_resident_{tag}"] = timed(synced_step(t), a.steps, a.warmup, a.reps)
                st = trainers["cache"].train_data.stream
                maps = [m for m in st.inputs + st.targets]
                for rep in range(a.reps):
                    for advice, label in ((None, "normal"), (mmap.MADV_RANDOM, "madv_random")):
                        ms, nread = evicted_window(trainers["cache"], maps, a.steps, advice)
                        res.setdefault(f"step_{key}_cache_evicted_{label}", []).append(
                            {"ms": ms, "read_bytes": nread})
            finally:
                for t in trainers.values():
                    t.close()
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
