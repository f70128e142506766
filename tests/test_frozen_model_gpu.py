"""The whole-model C-ABI on an H100: a frozen model run through hdrnet_model_run_px (FrozenModel)
gives bit for bit what the Python path gives on the same weights -- inference_image for the curves
and NN models over every pixel-format pair, both coefficient paths, the row-kernel, per-pixel and
texture-assisted shapes, unaligned images and a separate network input; for the pyramid, its float
inference on the host's img_as_float followed by the quantisation -- keeps the buffer contract,
replays from a CUDA graph, runs on side streams and past 2^31 bytes, refuses destroyed objects and
short workspaces, and hdrnet_run writes what bin/run.py writes."""
import argparse
import json
import os
import subprocess

import cv2
import numpy as np
import pytest
import torch

from hdrnet_b200 import _lib, checkpoint, models
from hdrnet_b200.bin import freeze_model as freeze_cli
from hdrnet_b200.bin import run as run_cli
from hdrnet_b200.bin import train
from hdrnet_b200.frozen import FrozenModel

pytestmark = pytest.mark.gpu

U8, U16, F32 = torch.uint8, torch.uint16, torch.float32
RUNNER = os.path.join(os.path.dirname(_lib.LIB_PATH), "hdrnet_run")


def _image(shape, dtype, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if dtype == F32:
        return torch.rand(shape, generator=g, device="cuda")
    top = 256 if dtype == U8 else 65536
    return torch.randint(0, top, shape, generator=g, device="cuda", dtype=torch.int32).to(dtype)


def _frozen(tmp_path_factory, name, seed, **over):
    params = dict(models.DEFAULT_PARAMS, model_name=name, **over)
    w = models.init_weights(params, seed=seed, model_name=name)
    rng = np.random.RandomState(seed)
    for k in w:   # non-zero biases and batch-norm statistics, so that every array matters
        if k.endswith(("/biases", "BatchNorm/beta", "moving_mean")):
            w[k] = (rng.randn(*w[k].shape) * 0.05).astype(np.float32)
    params["weights"] = w
    path = tmp_path_factory.mktemp("frozen") / f"{name}.hdrnet"
    checkpoint.freeze_model(w, params, str(path))
    return params, FrozenModel(str(path))


@pytest.fixture(scope="module", params=["HDRNetCurves", "HDRNetPointwiseNNGuide"])
def guided(request, tmp_path_factory):
    params, model = _frozen(tmp_path_factory, request.param, 5)
    yield getattr(models, request.param), params, model
    model.close()


@pytest.fixture(scope="module")
def pyramid(tmp_path_factory):
    params, model = _frozen(tmp_path_factory, "HDRNetGaussianPyrNN", 6, channel_multiplier=4)
    yield params, model
    model.close()


def _same(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, what
    ok = torch.equal(a.view(torch.int16) if a.dtype == U16 else a.view(torch.int32) if a.dtype == F32 else a,
                     b.view(torch.int16) if b.dtype == U16 else b.view(torch.int32) if b.dtype == F32 else b)
    assert ok, f"{what}: {int((a.to(torch.float64) != b.to(torch.float64)).sum())} values differ"


@pytest.mark.parametrize("in_dtype", [U8, U16, F32])
@pytest.mark.parametrize("out_dtype", [U8, U16, F32])
def test_every_format_pair(guided, in_dtype, out_dtype):
    cls, params, model = guided
    img = _image((3, 48, 256, 3), in_dtype)
    with torch.no_grad():
        want = cls.inference_image(img, params, out_dtype=out_dtype)
    _same(model(img, out_dtype=out_dtype), want, f"{in_dtype}->{out_dtype}")


@pytest.mark.parametrize("B,H,W", [(1, 72, 512), (3, 40, 128), (17, 32, 256), (2, 33, 97), (1, 20, 130)])
@pytest.mark.parametrize("fmt", [(U8, U8), (U16, U16), (F32, F32), (U8, F32)])
def test_batches_and_shapes(guided, B, H, W, fmt):
    """B = 17 takes the per-layer coefficient path, the others the launch chain; odd W and W % 16 != 0
    the per-pixel kernel."""
    cls, params, model = guided
    img = _image((B, H, W, 3), fmt[0], seed=B + W)
    with torch.no_grad():
        want = cls.inference_image(img, params, out_dtype=fmt[1])
    _same(model(img, out_dtype=fmt[1]), want, f"{B}x{H}x{W} {fmt}")


@pytest.mark.parametrize("offset_bytes", [2, 4, 6])
@pytest.mark.parametrize("dtype", [U8, U16])
def test_unaligned_images(guided, dtype, offset_bytes):
    cls, params, model = guided
    shape = (2, 24, 256, 3)
    n = int(np.prod(shape))
    off = offset_bytes // (1 if dtype == U8 else 2)
    buf = _image((n + off,), dtype, seed=offset_bytes)
    img = buf[off:off + n].view(shape)
    assert img.data_ptr() % 16 == offset_bytes % 16
    with torch.no_grad():
        want = cls.inference_image(img, params, out_dtype=U8)
    _same(model(img, out_dtype=U8), want, f"offset {offset_bytes}")


@pytest.mark.parametrize("out_dtype", [U8, U16])
def test_8x4k_texture_forms(guided, out_dtype):
    cls, params, model = guided
    img = _image((8, 2160, 3840, 3), U8, seed=11)
    with torch.no_grad():
        want = cls.inference_image(img, params, out_dtype=out_dtype)
    _same(model(img, out_dtype=out_dtype), want, "8 x 4K")


def test_lowres_image(guided):
    cls, params, model = guided
    img, low = _image((2, 64, 256, 3), U16, seed=1), _image((2, 100, 150, 3), U8, seed=2)
    with torch.no_grad():
        want = cls.inference_image(img, params, lowres_image=low, out_dtype=U16)
    got = model(img, lowres_image=low, out_dtype=U16)
    _same(got, want, "lowres_image")
    assert not torch.equal(got.view(torch.int16), model(img, out_dtype=U16).view(torch.int16))


def _host_img_as_float(img):
    return torch.from_numpy(run_cli.img_as_float(img.cpu().numpy())).cuda()


@pytest.mark.parametrize("B,S", [(1, 2048), (4, 512)])
@pytest.mark.parametrize("in_dtype", [U8, U16, F32])
def test_pyramid(pyramid, B, S, in_dtype):
    params, model = pyramid
    cls = models.HDRNetGaussianPyrNN
    img = _image((B, S, S, 3), in_dtype, seed=S)
    with torch.no_grad():
        if in_dtype == F32:
            wants = {d: cls.inference_image(img, params, out_dtype=d) for d in (U8, U16, F32)}
        else:
            low = models.lowres_from_image(img, params["net_input_size"])
            f = cls.inference(low, _host_img_as_float(img), params)
            wants = {U8: models.quantize_u8(f), U16: models.quantize_u16(f), F32: f}
    for d, want in wants.items():
        _same(model(img, out_dtype=d), want, f"pyramid {B}x{S}^2 {in_dtype}->{d}")


def _contract(model, img, out_dtype, fill):
    """One run with `out` and the workspace (lent at exactly workspace_bytes) inside guarded byte
    buffers filled with `fill`; returns a copy of the output and asserts that nothing outside `out`
    or the workspace changed."""
    B, H, W, _ = img.shape
    nbytes = model.workspace_bytes(B, H, W, img.dtype, out_dtype)
    guard, size = 4096, out_dtype.itemsize
    ws_buf = torch.full((nbytes + 2 * guard,), fill, dtype=U8, device="cuda")
    n_out = B * H * W * 3
    out_buf = torch.full(((n_out + 2 * guard) * size,), fill, dtype=U8, device="cuda")
    out = out_buf.view(out_dtype)[guard:guard + n_out].view(B, H, W, 3)
    model.run(img, out, ws_buf[guard:guard + nbytes])
    torch.cuda.synchronize()
    for buf, g, what in ((ws_buf, guard, "workspace"), (out_buf, guard * size, "out")):
        assert bool((buf[:g] == fill).all()) and bool((buf[-g:] == fill).all()), f"written outside {what}"
    return out.clone()


def _check_buffer_contract(cls, params, model, out_dtype, pyramid):
    img = _image((2, 1080, 1920, 3), U8, seed=3)
    a = _contract(model, img, out_dtype, 0x00)
    b = _contract(model, img, out_dtype, 0xFF)   # garbage in out and the workspace changes nothing
    _same(a, b, "two fills")
    with torch.no_grad():
        if not pyramid:
            want = cls.inference_image(img, params, out_dtype=out_dtype)
        else:
            f = cls.inference(models.lowres_from_image(img, params["net_input_size"]), _host_img_as_float(img), params)
            want = {U8: models.quantize_u8, U16: models.quantize_u16, F32: lambda x: x}[out_dtype](f)
    _same(a, want, "fully written")
    # one byte short: refused, nothing written
    B, H, W, _ = img.shape
    nbytes = model.workspace_bytes(B, H, W, U8, out_dtype)
    ws = torch.full((nbytes - 1,), 0x5A, dtype=U8, device="cuda")
    out_bytes = torch.zeros(B * H * W * 3 * out_dtype.itemsize, dtype=U8, device="cuda")
    with pytest.raises(ValueError, match="invalid dimension"):
        model.run(img, out_bytes.view(out_dtype).view(B, H, W, 3), ws)
    torch.cuda.synchronize()
    assert bool((ws == 0x5A).all()) and not bool(out_bytes.any())


@pytest.mark.parametrize("out_dtype", [U8, U16, F32])
def test_buffer_contract(guided, out_dtype):
    _check_buffer_contract(*guided, out_dtype, False)


@pytest.mark.parametrize("out_dtype", [U8, U16, F32])
def test_buffer_contract_pyramid(pyramid, out_dtype):
    _check_buffer_contract(models.HDRNetGaussianPyrNN, *pyramid, out_dtype, True)


def test_uint16_output_over_the_input_is_refused(guided):
    _, _, model = guided
    buf = _image((2 * 64 * 256 * 3,), U16)
    img = buf.view(2, 64, 256, 3)
    ws = torch.empty(model.workspace_bytes(2, 64, 256, U16, U16), dtype=U8, device="cuda")
    with pytest.raises(ValueError, match="cannot run"):
        model.run(img, img, ws)


@pytest.mark.parametrize("H,W", [(1080, 1920), (2160, 3840)])
def test_cuda_graph_replay(guided, pyramid, H, W):
    for model in (guided[2], pyramid[1]):
        static_in = _image((1, H, W, 3), U8, seed=0)
        out = torch.empty((1, H, W, 3), dtype=U8, device="cuda")
        ws = torch.empty(model.workspace_bytes(1, H, W), dtype=U8, device="cuda")
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            model.run(static_in, out, ws)       # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            model.run(static_in, out, ws)
        for seed in (1, 2, 3):
            frame = _image((1, H, W, 3), U8, seed=seed)
            static_in.copy_(frame)
            graph.replay()
            _same(out, model(frame), f"{model.model_name} replay {seed}")


def test_graph_outlives_the_texture_cache(guided):
    """A graph captured at 4K (the texture-assisted forms) owns the texture it fetches the slab
    through: running the same workspace directly, then more distinct workspaces than the library's
    texture cache holds (16), leaves every replay equal to direct calls."""
    model = guided[2]
    H, W = 2160, 3840
    static_in = _image((1, H, W, 3), U8, seed=0)
    out = torch.empty((1, H, W, 3), dtype=U8, device="cuda")
    nbytes = model.workspace_bytes(1, H, W)
    ws = torch.empty(nbytes, dtype=U8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        model.run(static_in, out, ws)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        model.run(static_in, out, ws)
    model.run(static_in, torch.empty_like(out), ws)          # the graph's workspace, run directly
    others = [torch.empty(nbytes, dtype=U8, device="cuda") for _ in range(20)]   # all alive: distinct bases
    scratch = torch.empty_like(out)
    for other in others:
        model.run(static_in, scratch, other)
    torch.cuda.synchronize()
    model.run(static_in, scratch, others[0])                 # evicted textures are destroyed by now
    torch.cuda.synchronize()
    for seed in (4, 5):
        frame = _image((1, H, W, 3), U8, seed=seed)
        static_in.copy_(frame)
        graph.replay()
        _same(out, model(frame), f"{model.model_name} replay {seed} after 20 other workspaces")
    del graph
    torch.cuda.synchronize()
    _same(model(frame), model.run(frame, scratch, ws), "the workspace after the graph is gone")


def test_side_streams_and_two_objects(guided, pyramid):
    a, b = guided[2], pyramid[1]
    img = _image((2, 256, 512, 3), U8, seed=9)
    want_a, want_b = a(img), b(img)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for s in (s1, s2):
        s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s1):
        got_a = a(img)
    with torch.cuda.stream(s2):
        got_b = b(img)
    torch.cuda.synchronize()
    _same(got_a, want_a, "side stream 1")
    _same(got_b, want_b, "side stream 2")


def test_destroyed_object_and_wrong_device(tmp_path):
    params = dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8)
    path = checkpoint.freeze_model(models.init_weights(params, seed=0), params, str(tmp_path / "m.hdrnet"))
    lib = _lib.load()
    img = _image((1, 16, 128, 3), U8)
    out = torch.empty_like(img)
    ws = torch.empty(1 << 20, dtype=U8, device="cuda")

    def run(handle):
        return lib.hdrnet_model_run_px(handle, img.data_ptr(), _lib.PX_U8, None, 0, 0, 0, out.data_ptr(), _lib.PX_U8,
                                       1, 16, 128, ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)

    model = FrozenModel(path)
    handle = model.handle
    assert run(handle) == _lib.OK
    if torch.cuda.device_count() > 1:
        with torch.cuda.device(1):
            assert run(handle) == _lib.E_BAD_CONTEXT
    model.close()
    assert run(handle) == _lib.E_BAD_CONTEXT
    assert lib.hdrnet_model_destroy(handle) == _lib.E_BAD_CONTEXT
    assert lib.hdrnet_model_workspace_bytes(handle, 1, 16, 128, 1, 1) == 0
    with pytest.raises(ValueError, match="closed"):
        model(img)


def _exact_coefficients(tmp_path_factory, name):
    """A model whose coefficient network computes its grid without rounding: every conv and fc weight
    zero, so each layer's output is exactly its bias and the grid is the prediction bias (near the
    identity, varying with depth), whatever order a kernel sums in.  Calls on different batch sizes
    (launch chain or per-layer convs) then share one grid, and single-image calls are a reference
    for any image of a batch."""
    params = dict(models.DEFAULT_PARAMS, model_name=name)
    w = models.init_weights(params, seed=7, model_name=name)
    rng = np.random.RandomState(7)
    for k in w:
        if k.startswith("inference/coefficients/") and k.endswith("/weights"):
            w[k] = np.zeros_like(w[k])
        elif k.startswith("inference/coefficients/") and k.endswith("/biases"):
            w[k] = (rng.rand(*w[k].shape) * 0.1).astype(np.float32)
    gd, n_out = params["luma_bins"], getattr(models, name).n_out()
    o = np.arange(gd * n_out * 4)
    z, i, j = o % gd, (o // gd) % n_out, o // (gd * n_out)
    scale = 1.0 / 3.0 if name == "HDRNetGaussianPyrNN" else 1.0
    bias = np.where(j == i % 3, scale, 0.0) + 0.05 * np.sin(z + 3 * i + 7 * j)
    w["inference/coefficients/prediction/conv1/biases"] = bias.astype(np.float32)
    params["weights"] = w
    path = tmp_path_factory.mktemp("exact") / f"{name}.hdrnet"
    checkpoint.freeze_model(w, params, str(path))
    return params, FrozenModel(str(path))


@pytest.mark.parametrize("name", checkpoint.FROZEN_KINDS)
def test_44x4k_uint16_past_2_31_bytes(tmp_path_factory, name):
    """44 x 4K uint16 in and out (2.19 GB each): the first image, the ones straddling 2^31 bytes (of the
    uint16 buffers, and of the pyramid's float32 levels) and the last equal calls on those images alone; curves and NN also equal inference_image on the batch."""
    params, model = _exact_coefficients(tmp_path_factory, name)
    B, H, W = 44, 2160, 3840
    img = _image((B, H, W, 3), U16, seed=4)
    assert img.numel() * 2 > 2 ** 31
    got = model(img, out_dtype=U16)
    straddle = (2 ** 31) // (H * W * 6)              # of the uint16 image and result
    straddle_f32 = (2 ** 31) // (H * W * 12)         # of the pyramid's float32 intermediates
    for b in (0, straddle_f32, straddle, B - 1):
        _same(got[b:b + 1], model(img[b:b + 1].clone(), out_dtype=U16), f"image {b}")
    assert int(got.view(torch.int16)[straddle].ne(0).sum()) > H * W   # not a blank result
    if name != "HDRNetGaussianPyrNN":
        with torch.no_grad():
            want = getattr(models, name).inference_image(img, params, out_dtype=U16)
        _same(got, want, "44 x 4K")
    model.close()


# ---- end to end: training CLI -> freeze_model -> hdrnet_run, against bin/run.py -----------------
MODEL = ["--net_input_size", "64", "--spatial_bin", "8", "--output_resolution", "64", "64", "--batch_size", "2"]


@pytest.fixture(scope="module")
def trained(tmp_path_factory):
    root = tmp_path_factory.mktemp("pairs")
    for d in ("input", "output"):
        os.makedirs(root / d)
    rng = np.random.RandomState(0)
    names = []
    for i in range(4):
        im8 = rng.randint(0, 256, (80, 96, 3)).astype(np.uint8)
        out16 = (im8.astype(np.uint16) * 200)[:, :, ::-1]
        name = f"im{i}.png"
        assert cv2.imwrite(str(root / "input" / name), im8)
        assert cv2.imwrite(str(root / "output" / name), np.ascontiguousarray(out16))
        names.append(name)
    (root / "filelist.txt").write_text("\n".join(names) + "\n")
    ckpt = tmp_path_factory.mktemp("ckpt")
    parser = train.build_parser()
    args = parser.parse_args([str(ckpt), str(root), *MODEL, "--summary_interval", "0", "--checkpoint_interval",
                              "100000", "--max_steps", "5"])
    params = train.model_params(parser, args)
    train.refuse_untrainable(params)
    train.Trainer(args, params).run()
    return ckpt


@pytest.mark.parametrize("bits", [8, 16])
def test_hdrnet_run_writes_what_run_py_writes(trained, tmp_path, bits):
    frozen = freeze_cli.main(freeze_cli.build_parser().parse_args([str(trained), "--output",
                                                                   str(tmp_path / "model.hdrnet")]))
    rng = np.random.RandomState(bits)
    im = rng.randint(0, 65536, (120, 200, 3)).astype(np.uint16) if bits == 16 else \
        rng.randint(0, 256, (120, 200, 3)).astype(np.uint8)
    np.save(tmp_path / "im.npy", im)
    assert cv2.imwrite(str(tmp_path / "im.png"), im[:, :, ::-1])
    out_dir = tmp_path / "out"
    os.makedirs(out_dir)
    proc = subprocess.run([RUNNER, "--checkpoint_path", frozen, "--input_path", str(tmp_path / "im.npy"),
                           "--output_directory", str(out_dir), "--burn_iters", "1", "--iters", "3",
                           "--output_bit_depth", str(bits)], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    got = np.load(out_dir / "model.npy")
    report = json.loads((out_dir / "model.json").read_text())
    assert report["model"] == "HDRNetCurves" and (report["height"], report["width"]) == (120, 200)
    assert report["iters"] == 3 and 0 < report["min_ms"] <= report["mean_ms"]
    run_dir = tmp_path / "run_py"
    run_cli.main(argparse.Namespace(checkpoint_dir=str(trained), input=str(tmp_path / "im.png"), output=str(run_dir),
                                    lowres_input=None, hdrp=False, debug=False, limit=None, output_bit_depth=bits))
    want = cv2.imread(str(run_dir / "im.png"), -1)[:, :, ::-1]
    assert got.dtype == (np.uint8 if bits == 8 else np.uint16) and np.array_equal(got, want)


def test_hdrnet_run_refuses_other_npy_files(tmp_path):
    params = dict(models.DEFAULT_PARAMS, net_input_size=64, spatial_bin=8)
    path = checkpoint.freeze_model(models.init_weights(params, seed=0), params, str(tmp_path / "m.hdrnet"))
    np.save(tmp_path / "f.npy", np.zeros((8, 8, 3), np.float32))
    proc = subprocess.run([RUNNER, "--checkpoint_path", path, "--input_path", str(tmp_path / "f.npy"),
                           "--output_directory", str(tmp_path)], capture_output=True, text=True)
    assert proc.returncode != 0 and "uint8" in proc.stderr
