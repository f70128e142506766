"""Time a whole model per frame three ways: the Python path (``inference_image``), the frozen model
through the whole-model C-ABI (``FrozenModel``: one ctypes call, output and workspace from torch's
allocator), and that same call captured once in a CUDA graph and replayed.

For HDRNetCurves and HDRNetPointwiseNNGuide (default hyperparameters, synthetic weights), uint8 ->
uint8, at batch 1 for 1080p and 4K and at batch 8 for 4K.  CUDA-event times on the current stream
over windows of --steps calls, so host time between launches counts where the GPU waits for it; the
three paths alternate round by round (--rounds), after --warmup calls each.  Reports the median and
the min-max spread per path in ms per call, and each path's time over inference_image's.  The
outputs of the three paths are checked equal first.  Reads the card's name, power limit and maximum
SM clock in the same run.  Prints one JSON object; --out also writes it.

    python tools/time_frozen_model.py [--steps 20 --warmup 5 --rounds 5 --out tools_out/frozen_model.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hdrnet_b200 import checkpoint, models  # noqa: E402
from hdrnet_b200.frozen import FrozenModel  # noqa: E402
from time_train_step import gpu_identity, timed  # noqa: E402

SHAPES = {"1080p_x1": (1, 1080, 1920), "4k_x1": (1, 2160, 3840), "4k_x8": (8, 2160, 3840)}
GUIDES = ("HDRNetCurves", "HDRNetPointwiseNNGuide")


def case(model_name, B, H, W, a, tmp):
    p = dict(models.DEFAULT_PARAMS, model_name=model_name)
    p["weights"] = models.init_weights(p, seed=0, model_name=model_name)
    cls = getattr(models, model_name)
    model = FrozenModel(checkpoint.freeze_model(p["weights"], p, os.path.join(tmp, model_name + ".hdrnet")))
    gen = torch.Generator(device="cuda").manual_seed(5)
    img = torch.randint(0, 256, (B, H, W, 3), device="cuda", generator=gen, dtype=torch.int32).to(torch.uint8)
    out = torch.empty_like(img)
    ws = torch.empty(model.workspace_bytes(B, H, W), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        model.run(img, out, ws)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        model.run(img, out, ws)
    calls = {"inference_image": lambda: cls.inference_image(img, p), "frozen": lambda: model(img),
             "graph_replay": graph.replay}
    want = calls["inference_image"]()
    graph.replay()
    assert torch.equal(calls["frozen"](), want) and torch.equal(out, want), "the three paths differ"
    for fn in calls.values():
        timed(fn, 1, a.warmup, 1)
    per = {name: [] for name in calls}
    for _ in range(a.rounds):                                  # interleaved: A B C A B C ...
        for name, fn in calls.items():
            per[name].append(timed(fn, a.steps, 0, 1)["ms"])
    res = {name: {"ms": float(np.median(v)), "min": min(v), "max": max(v)} for name, v in per.items()}
    base = res["inference_image"]["ms"]
    for name in calls:
        res[name]["over_inference_image"] = res[name]["ms"] / base
    model.close()
    del img, out, ws, graph
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_frozen_model.py needs a CUDA device")
    res = {"gpu": gpu_identity(), "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds}
    with torch.no_grad(), tempfile.TemporaryDirectory() as tmp:
        for key, (B, H, W) in SHAPES.items():
            res[key] = {name: case(name, B, H, W, a, tmp) for name in GUIDES}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
