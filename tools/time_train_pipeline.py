"""Time the training CLI's data path and step on the device (hdrnet_b200/bin/train.py).

In one run, with the card's name and power limit read in the same run:
  * CUDA-event time of the batch-assembly kernel (hdrnet_train_batch_f32) at the reference's training
    size -- 16 crops of 512² with flips, rotations and random crops, plus the 256² network input --
    from a cache of uint8 sources and from one of uint16 sources (u8 / u16 / u8 / u16), with the
    bytes the kernel must move and the bandwidth that implies;
  * the CLI's steady-state step (train.Trainer.train_step: batch kernel, forward, L2 loss, PSNR,
    backward, Adam.step) on a synthetic dataset, alternated with tools/time_train_step.py's whole
    step plus Adam.step on fixed tensors (A / B / A / B);
  * the CLI's step on each data tier -- decoded pairs resident on the device, or kept on the host
    with each batch's crop windows streamed (forced by substituting data_pipeline.device_budget) --
    at the reference's three training shapes, 16 x 512², 4 x 1024² and 1 x 2048², from uint8 inputs
    and uint16 targets with flips, rotations and random crops.  Each step ends with the loss and
    PSNR read on the host, as Trainer.run does; the tiers alternate (device / stream / device /
    stream) per shape;
  * with --trace DIR, a torch.profiler run of its own of the streamed tier at 16 x 512²: the host
    time packing a batch's windows, the host-to-device copies, the training thread's wait in
    batch(), how long the compute stream sat idle waiting for an upload, and the step's
    cudaLaunchKernel times while a batch is being packed and otherwise; the Chrome trace goes to DIR.
Prints one JSON object; --out also writes it.

    python tools/time_train_pipeline.py [--steps 20 --warmup 5 --reps 5 --out tools_out/train_pipeline.json]
        [--trace tools_out/stream_trace]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from hdrnet_b200 import data_pipeline as dp, metrics, models  # noqa: E402
from hdrnet_b200.bin import train  # noqa: E402
from time_train_step import gpu_identity, timed  # noqa: E402

B, OH, S = 16, 512, 256
SRC_H, SRC_W, N_SRC = 600, 700, 32


def kernel_record(dtype, steps, warmup, reps):
    rng = np.random.RandomState(0)
    hi = np.iinfo(dtype).max + 1
    srcs = [torch.from_numpy(rng.randint(0, hi, size=(SRC_H, SRC_W, 3)).astype(dtype)).cuda() for _ in range(2 * B)]
    sampler = dp.Sampler([(SRC_H, SRC_W)] * B, B, (OH, OH), shuffle=True, fliplr=True, flipud=True, rotate=True,
                         random_crop=True, seed=0)
    draws = sampler.draws(0)
    out = (torch.empty(B, OH, OH, 3, device="cuda"), torch.empty(B, OH, OH, 3, device="cuda"),
           torch.empty(B, S, S, 3, device="cuda"))

    def call():
        dp.train_batch([srcs[d.index] for d in draws], [srcs[B + d.index] for d in draws], draws, (OH, OH), S, out=out)

    t = timed(call, steps, warmup, reps)
    item = np.dtype(dtype).itemsize
    nbytes = B * (2 * OH * OH * 3 * item + 2 * OH * OH * 3 * 4 + S * S * 3 * (item + 4))
    t.update(bytes=nbytes, tb_per_s=nbytes / (t["ms"] * 1e-3) / 1e12)
    return t


def synthetic_dataset(root, n=N_SRC):
    import cv2
    os.makedirs(os.path.join(root, "input"))
    os.makedirs(os.path.join(root, "output"))
    rng = np.random.RandomState(1)
    names = []
    for i in range(n):
        name = f"{i:03d}.png"
        cv2.imwrite(os.path.join(root, "input", name), rng.randint(0, 256, size=(SRC_H, SRC_W, 3)).astype(np.uint8))
        cv2.imwrite(os.path.join(root, "output", name), rng.randint(0, 65536, size=(SRC_H, SRC_W, 3)).astype(np.uint16))
        names.append(name)
    with open(os.path.join(root, "filelist.txt"), "w") as f:
        f.write("\n".join(names) + "\n")


def kernel_and_step_records(res, steps, warmup, reps):
    for tag in ("a", "b"):          # alternated: the first window also pays for the clock ramp
        res[f"batch_kernel_u8_{tag}"] = kernel_record(np.uint8, steps, warmup, reps)
        res[f"batch_kernel_u16_{tag}"] = kernel_record(np.uint16, steps, warmup, reps)

    with tempfile.TemporaryDirectory() as tmp:
        synthetic_dataset(os.path.join(tmp, "data"))
        parser = train.build_parser()
        args = parser.parse_args([os.path.join(tmp, "ckpt"), os.path.join(tmp, "data"), "--fliplr", "--flipud", "--rotate"])
        cli = train.Trainer(args, train.model_params(parser, args))

        # tools/time_train_step.py's step on fixed tensors, plus Adam.step
        params = dict(models.DEFAULT_PARAMS)
        rng = np.random.RandomState(0)
        wts = {k: torch.from_numpy(v).cuda().requires_grad_(k.startswith(train.COEFFS))
               for k, v in models.init_weights(params, seed=0).items()}
        p = dict(params, weights=wts)
        low = torch.from_numpy(rng.rand(B, S, S, 3).astype(np.float32)).cuda()
        full = torch.from_numpy(rng.rand(B, OH, OH, 3).astype(np.float32)).cuda()
        target = torch.from_numpy(rng.rand(B, OH, OH, 3).astype(np.float32)).cuda()
        opt = torch.optim.Adam([v for v in wts.values() if v.requires_grad], lr=1e-4)

        def fixed_step():
            opt.zero_grad(set_to_none=True)
            metrics.l2_loss(target, models.HDRNetCurves.inference(low, full, p)).backward()
            opt.step()

        for tag in ("a", "b"):
            res[f"cli_step_{tag}"] = timed(cli.train_step, steps, warmup, reps)
            res[f"fixed_step_adam_{tag}"] = timed(fixed_step, steps, warmup, reps)
        cli.close()


TIER_SHAPES = ((16, 512), (4, 1024), (1, 2048))        # 4.19 Mpx per batch each


def synthetic_pairs(root, n, H, W):
    """n pairs of uint8 inputs and uint16 targets, PNGs without compression (fast to write and decode)."""
    import cv2
    os.makedirs(os.path.join(root, "input"))
    os.makedirs(os.path.join(root, "output"))
    rng = np.random.RandomState(2)
    names = []
    for i in range(n):
        name = f"{i:03d}.png"
        cv2.imwrite(os.path.join(root, "input", name), rng.randint(0, 256, size=(H, W, 3)).astype(np.uint8),
                    [cv2.IMWRITE_PNG_COMPRESSION, 0])
        cv2.imwrite(os.path.join(root, "output", name), rng.randint(0, 65536, size=(H, W, 3)).astype(np.uint16),
                    [cv2.IMWRITE_PNG_COMPRESSION, 0])
        names.append(name)
    with open(os.path.join(root, "filelist.txt"), "w") as f:
        f.write("\n".join(names) + "\n")


def tier_trainer(tmp, data, tier, B, oh, data_threads=2):
    """A Trainer on ``tier``, chosen by a substituted device_budget (the dataset fits, or only the
    staging slots do)."""
    u8, u16 = np.dtype(np.uint8), np.dtype(np.uint16)
    staging = dp.STREAM_SLOTS * dp.slot_bytes({(u8, u16)}, B, (oh, oh))
    free = torch.cuda.mem_get_info()[0] if tier == "device" else dp.MEMORY_MARGIN + staging
    keep = dp.device_budget
    dp.device_budget = lambda device: free
    try:
        parser = train.build_parser()
        args = parser.parse_args([os.path.join(tmp, f"ckpt_{tier}"), data, "--fliplr", "--flipud", "--rotate",
                                  "--batch_size", str(B), "--output_resolution", str(oh), str(oh),
                                  "--data_threads", str(data_threads)])
        t = train.Trainer(args, train.model_params(parser, args))
    finally:
        dp.device_budget = keep
    assert t.train_data.tier == tier, (t.train_data.tier, tier)
    return t


def synced_step(t):
    """Trainer.run's step: train_step, then the loss and PSNR read on the host."""
    def step():
        loss, psnr = t.train_step()
        float(loss), float(psnr)
    return step


def tier_records(res, steps, warmup, reps, data_threads):
    for B, oh in TIER_SHAPES:
        n = max(2 * B, 4)
        with tempfile.TemporaryDirectory() as tmp:
            data = os.path.join(tmp, "data")
            synthetic_pairs(data, n, oh + 88, oh + 188)
            trainers = {tier: tier_trainer(tmp, data, tier, B, oh, data_threads) for tier in ("device", "stream")}
            try:
                key = f"{B}x{oh}"
                res[f"tier_{key}"] = {"pairs": n, "data_threads": data_threads, "source": [oh + 88, oh + 188],
                                      "dataset_bytes": trainers["device"].train_data.dataset_bytes,
                                      "streamed_bytes_per_batch": B * oh * oh * 3 * (1 + 2),
                                      "staging_bytes": trainers["stream"].train_data.staging_bytes}
                for tag in ("a", "b"):
                    for tier, t in trainers.items():
                        res[f"cli_step_{key}_{tier}_{tag}"] = timed(synced_step(t), steps, warmup, reps)
                st = trainers["stream"].train_data.stream
                res[f"tier_{key}"]["pack_ms_per_batch"] = 1e3 * st.pack_seconds / max(st.packed, 1)
            finally:
                for t in trainers.values():
                    t.close()


def device_intervals(prof):
    """(name, start µs, end µs) of the device-side activities in a profile."""
    out = []
    for e in prof.events():
        if getattr(e, "device_type", None) == torch.autograd.DeviceType.CUDA:
            out.append((e.name, e.time_range.start, e.time_range.end))
    return sorted(out, key=lambda x: x[1])


def launch_slowdown(trace_path):
    """The training step's cudaLaunchKernel times (forward and autograd threads) while the producer
    thread packs a batch (from the end of its cudaEventSynchronize on the pinned slot to its
    cudaMemcpyAsync) and otherwise."""
    with open(trace_path) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("ph") == "X"]
    by_tid = {}
    for e in ev:
        by_tid.setdefault(e.get("tid"), []).append(e)
    producer = [v for v in by_tid.values() if any(e["name"] == "cudaMemcpyAsync" for e in v)
                and not any(e["name"].startswith("aten::") for e in v)]
    if len(producer) != 1:
        return {}
    launches = [e for v in by_tid.values() if v is not producer[0] for e in v if e["name"] == "cudaLaunchKernel"]
    windows, synced = [], None
    for e in sorted(producer[0], key=lambda e: e["ts"]):
        if e["name"] == "cudaEventSynchronize":
            synced = e["ts"] + e["dur"]
        elif e["name"] == "cudaMemcpyAsync" and synced is not None:
            windows.append((synced, e["ts"]))
            synced = None
    inside, outside = [], []
    for e in launches:
        (inside if any(a <= e["ts"] <= b for a, b in windows) else outside).append(e["dur"])
    return {"pack_windows": len(windows), "pack_window_ms": float(np.mean([b - a for a, b in windows])) / 1e3,
            "launches_while_packing": len(inside), "launch_us_median_while_packing": float(np.median(inside)),
            "launches_otherwise": len(outside), "launch_us_median_otherwise": float(np.median(outside))}


def profile_record(trace_dir, steps, data_threads):
    """The streamed tier at 16 x 512² under torch.profiler: host time per region, the uploads, and
    the compute stream's idle time ahead of each batch kernel that an upload still running explains."""
    from torch.profiler import ProfilerActivity, profile
    B, oh = TIER_SHAPES[0]
    with tempfile.TemporaryDirectory() as tmp:
        data = os.path.join(tmp, "data")
        synthetic_pairs(data, 2 * B, oh + 88, oh + 188)
        t = tier_trainer(tmp, data, "stream", B, oh, data_threads)
        try:
            step = synced_step(t)
            for _ in range(5):
                step()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                t0 = time.perf_counter()
                for _ in range(steps):
                    step()
                torch.cuda.synchronize()
                elapsed = time.perf_counter() - t0
        finally:
            t.close()
    os.makedirs(trace_dir, exist_ok=True)
    prof_trace = os.path.join(trace_dir, "stream_16x512.json")
    prof.export_chrome_trace(prof_trace)
    st = t.train_data.stream
    rec = {"steps": steps, "step_ms": 1e3 * elapsed / steps, "pack_ms_per_batch": 1e3 * st.pack_seconds / st.packed}
    for ev in prof.key_averages():
        if ev.key.startswith("data_pipeline.stream.") or ev.key.startswith("Memcpy HtoD") \
                or "train_batch_kernel" in ev.key:
            rec[ev.key] = {"count": ev.count, "cpu_ms_per_call": ev.cpu_time_total / 1e3 / max(ev.count, 1),
                           "device_ms_per_call": getattr(ev, "device_time_total", 0.0) / 1e3 / max(ev.count, 1)}
    dev = device_intervals(prof)
    uploads = [(s, e) for n, s, e in dev if n.startswith("Memcpy HtoD")]
    idle, waited = [], 0
    for i, (name, start, _) in enumerate(dev):
        if "train_batch_kernel" not in name:
            continue
        prev_end = max((e for n, s, e in dev[:i] if not n.startswith("Memcpy")), default=start)
        up_end = max((e for s, e in uploads if e <= start + 1), default=None)
        gap = max(0.0, start - prev_end)
        if up_end is not None and up_end > prev_end:           # the compute stream waited for this upload
            waited += 1
            idle.append(min(gap, up_end - prev_end))
        else:
            idle.append(0.0)
    rec.update(launch_slowdown(prof_trace))
    rec["batch_kernels"] = len(idle)
    rec["batches_waiting_for_upload"] = waited
    rec["compute_idle_for_upload_ms_per_step"] = float(np.sum(idle)) / 1e3 / max(len(idle), 1)
    return rec


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--trace", default=None, help="directory for the streamed tier's profile (a run of its own)")
    ap.add_argument("--data_threads", type=int, default=2, help="the CLI's --data_threads for the tier records")
    ap.add_argument("--only-tiers", action="store_true", help="skip the batch-kernel and fixed-tensor records")
    ap.add_argument("--no-tiers", dest="tiers", action="store_false", help="skip the device / streamed tier records")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_train_pipeline.py needs a CUDA device")
    res = {"gpu": gpu_identity(), "host_cpus": len(os.sched_getaffinity(0)), "batch": B, "crop": OH, "lowres": S,
           "source": [SRC_H, SRC_W], "steps": a.steps, "warmup": a.warmup, "reps": a.reps}
    if not a.only_tiers:
        kernel_and_step_records(res, a.steps, a.warmup, a.reps)
    if a.tiers:
        tier_records(res, a.steps, a.warmup, a.reps, a.data_threads)
    if a.trace:
        res["stream_profile_16x512"] = profile_record(a.trace, a.steps, a.data_threads)
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
