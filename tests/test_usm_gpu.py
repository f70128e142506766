"""UnsharpMaskDataPipeline's batch kernel (hdrnet_train_batch_usm_f32, csrc/usm_batch.cu) on the
device.  The float64 oracle is scipy's ``gaussian_filter1d(mode="reflect", truncate=4.0)`` along x,
then y, of the same float32 input, and ``x + sharpen * (x - b)``; the augmentation is
test_train_batch_gpu's numpy restatement, applied to the oracle's whole-source target (the target is
a function of the source pixel).  Covered: accuracy for every sigma / sharpen / format / size / flip
and rotation / crop kind the definition names; known answers (sharpen 0, a constant image, an
impulse); the input and network input against train_batch; draw invariance; the streamed tier
against the device tier; the buffer contract; a batch past 2^31 bytes; the public ``unsharp_mask``."""

import numpy as np
import pytest
import torch
from scipy.ndimage import gaussian_filter1d

from hdrnet_b200 import _lib, data_pipeline as dp
from hdrnet_b200.data_pipeline import Draw, train_batch, unsharp_mask, usm_batch

from test_train_batch_gpu import augment, image, to_float

pytestmark = pytest.mark.gpu

SIGMAS = [0.5, 1.0, 2.5, 8.0, 32.0]
SHARPENS = [0.0, 0.5, 1.0, 4.0, -0.5]
DTYPES = [np.uint8, np.uint16, np.float32]
AUGS = [(lr, ud, k) for lr in (False, True) for ud in (False, True) for k in range(4)]
WORST = {}


def tol(sharpen):
    return 4e-6 * (1.0 + abs(sharpen))


def blur64(x, sigma):
    """G_sigma * x in float64: along x, then along y."""
    b = gaussian_filter1d(x.astype(np.float64), sigma, axis=1, mode="reflect", truncate=4.0)
    return gaussian_filter1d(b, sigma, axis=0, mode="reflect", truncate=4.0)


def target64(x, b, sharpen):
    """The pre-clip target of float32 input x with blur b."""
    x = x.astype(np.float64)
    return x + sharpen * (x - b)


def draws_for(rng, H, W, oh, ow, kind):
    out = []
    for lr, ud, k in AUGS:
        rh, rw = (W, H) if k % 2 else (H, W)
        if kind == "centre":
            cy, cx = (rh - oh) // 2, (rw - ow) // 2
        elif kind == "random":
            cy, cx = int(rng.randint(0, rh - oh + 1)), int(rng.randint(0, rw - ow + 1))
        else:                                  # corner: a different corner per draw
            cy, cx = (rh - oh) * (len(out) % 2), (rw - ow) * ((len(out) // 2) % 2)
        out.append(Draw(0, lr, ud, k, cy, cx))
    return out


def run(srcs, draws, oh, ow, S, sigma, sharpen, windows=None):
    dev = [s if isinstance(s, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(s)).cuda() for s in srcs]
    out = usm_batch(dev, draws, (oh, ow), S, sigma, sharpen, windows=windows)
    return [None if t is None else t.cpu().numpy() for t in out]


def check_against_oracle(src, draws, oh, ow, sigma, b64, what):
    """The target under every sharpen against clip(oracle); returns the worst error over tol."""
    x = to_float(src)
    worst = 0.0
    for sharpen in SHARPENS:
        got = run([src] * len(draws), draws, oh, ow, None, sigma, sharpen)[1]
        want = np.clip(target64(x, b64, sharpen), 0.0, 1.0)
        for g, d in zip(got, draws):
            err = float(np.abs(g - augment(want, d, oh, ow)).max())
            assert err <= tol(sharpen), f"{what} sigma {sigma} sharpen {sharpen} {d}: {err:.3e}"
            worst = max(worst, err / (1.0 + abs(sharpen)))
    WORST[what] = max(WORST.get(what, 0.0), worst)
    return worst


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, v in sorted(WORST.items()):
        print(f"usm worst |target - oracle| / (1 + |sharpen|): {k}: {v:.3e}")


@pytest.mark.parametrize("H,W,oh,ow", [(7, 5, 3, 2), (33, 50, 20, 24), (600, 700, 256, 320)])
def test_accuracy_against_scipy(H, W, oh, ow):
    rng = np.random.RandomState(H * 1000 + W)
    for dt in DTYPES:
        src = image(rng, H, W, dt)
        x = to_float(src)
        for sigma in SIGMAS:
            b64 = blur64(x, sigma)
            for kind in ("centre", "random", "corner"):
                check_against_oracle(src, draws_for(rng, H, W, oh, ow, kind), oh, ow, sigma, b64, f"{H}x{W}")
            # whole-image crops: the rotated extent is the crop
            for odd in (0, 1):
                d = [Draw(0, lr, ud, k, 0, 0) for lr, ud, k in AUGS if k % 2 == odd]
                check_against_oracle(src, d, *((W, H) if odd else (H, W)), sigma, b64, f"{H}x{W}")


def test_accuracy_training_shapes():
    """16 x 512^2 from 600 x 700 sources, and 1 x 2048^2 from 2136 x 2236 (the train_std.sh shape)."""
    rng = np.random.RandomState(3)
    srcs = [image(rng, 600, 700, DTYPES[i % 3]) for i in range(16)]
    for sigma in SIGMAS:
        draws = [Draw(0, lr, ud, k, int(rng.randint(0, 89)), int(rng.randint(0, 89)))
                 for lr, ud, k in AUGS]
        for sharpen in (1.0, 4.0):
            got = run(srcs, draws, 512, 512, None, sigma, sharpen)[1]
            for s, g, d in zip(srcs, got, draws):
                x = to_float(s)
                want = augment(np.clip(target64(x, blur64(x, sigma), sharpen), 0, 1), d, 512, 512)
                err = float(np.abs(g - want).max())
                assert err <= tol(sharpen), (sigma, sharpen, d, err)
                WORST["16 x 512^2"] = max(WORST.get("16 x 512^2", 0.0), err / (1 + sharpen))
    for dt in DTYPES:
        src = image(rng, 2136, 2236, dt)
        x = to_float(src)
        for sigma in (1.0, 32.0):
            b64 = blur64(x, sigma)
            d = [Draw(0, bool(rng.randint(2)), bool(rng.randint(2)), int(rng.randint(4)), 0, 0)]
            rh, rw = (2236, 2136) if d[0].rot90 % 2 else (2136, 2236)
            d = [d[0]._replace(crop_y=int(rng.randint(0, rh - 2047)), crop_x=int(rng.randint(0, rw - 2047)))]
            check_against_oracle(src, d, 2048, 2048, sigma, b64, "1 x 2048^2")


# ---- known answers ------------------------------------------------------------------------------
def test_sharpen_zero_gives_the_input():
    rng = np.random.RandomState(1)
    for dt in (np.uint8, np.uint16):
        srcs = [image(rng, 61, 47, dt) for _ in range(4)]
        draws = [Draw(0, lr, ud, k, 3, 5) for lr, ud, k in AUGS[::4]]
        for sigma in (0.5, 32.0):
            fin, fout, _ = run(srcs, draws, 30, 20, 8, sigma, 0.0)
            assert np.array_equal(fin.view(np.uint32), fout.view(np.uint32))


def test_constant_image_within_a_few_ulp():
    for value in (0.25, 0.7, 1.0 / 3.0):
        src = np.full((45, 38, 3), value, np.float32)
        for sigma in SIGMAS:
            for sharpen in (1.0, 4.0, -0.5):
                fout = run([src] * 4, [Draw(0, False, False, k, 0, 0) for k in (0, 2)] * 2, 20, 20, None,
                           sigma, sharpen)[1]
                ulps = np.abs(fout.view(np.int32).astype(np.int64) - np.float32(value).view(np.int32))
                assert ulps.max() <= 4, (value, sigma, sharpen, int(ulps.max()))


def test_impulse_gives_the_weights_outer_product():
    for sigma in (1.0, 2.5, 8.0):
        r = dp.usm_radius(sigma)
        n = 4 * r + 21
        src = np.zeros((n, n, 3), np.float32)
        c = n // 2
        src[c, c] = (1.0, 0.5, 0.25)
        k = np.arange(-r, r + 1)
        w = np.exp(-0.5 / sigma ** 2 * k.astype(np.float64) ** 2)
        w /= w.sum()
        fout = run([src], [Draw(0, False, False, 0, 0, 0)], n, n, None, sigma, -1.0)[1][0]   # t = b
        want = np.zeros((n, n, 3))
        for ch, v in enumerate((1.0, 0.5, 0.25)):
            want[c - r:c + r + 1, c - r:c + r + 1, ch] = v * np.outer(w, w)
        err = np.abs(fout - want)
        assert (err <= 3e-7 * np.abs(want)).all(), (sigma, float(err.max()))   # two float32 roundings


# ---- the other outputs and draw invariance ------------------------------------------------------
def test_input_and_network_input_equal_train_batch():
    rng = np.random.RandomState(2)
    srcs = [image(rng, 70 + 3 * i, 90 - 2 * i, DTYPES[i % 3]) for i in range(16)]
    draws = []
    for (lr, ud, k), s in zip(AUGS, srcs):
        rh, rw = (s.shape[1], s.shape[0]) if k % 2 else s.shape[:2]
        draws.append(Draw(0, lr, ud, k, int(rng.randint(0, rh - 40 + 1)), int(rng.randint(0, rw - 52 + 1))))
    dev = [torch.from_numpy(s).cuda() for s in srcs]
    want = [t.cpu().numpy() for t in train_batch(dev, dev, draws, (40, 52), 17)]
    got = run(dev, draws, 40, 52, 17, 2.5, 1.0)
    for i in (0, 2):
        assert np.array_equal(got[i].view(np.uint32), want[i].view(np.uint32))


def test_target_of_a_source_pixel_does_not_depend_on_the_draw():
    rng = np.random.RandomState(4)
    H, W = 53, 41
    src = image(rng, H, W, np.uint16)
    index = np.arange(H * W).reshape(H, W, 1)
    for sigma, oh, ow in ((2.5, 41, 41), (8.0, 30, 17)):
        seen = np.full((H * W, 3), np.nan, np.float32)
        for kind in ("centre", "random", "corner"):
            draws = draws_for(rng, H, W, oh, ow, kind)
            fout = run([src] * 16, draws, oh, ow, None, sigma, 4.0)[1]
            for g, d in zip(fout, draws):
                where = augment(index, d, oh, ow)[..., 0].reshape(-1)
                vals = g.reshape(-1, 3)
                known = ~np.isnan(seen[where, 0])
                assert np.array_equal(seen[where][known].view(np.uint32), vals[known].view(np.uint32)), (sigma, d)
                seen[where] = vals


# ---- the streamed tier --------------------------------------------------------------------------
N = 37
OH, OW, S = 24, 40, 16


@pytest.fixture(scope="module")
def inputs():
    rng = np.random.RandomState(11)
    ims = []
    for i in range(N):
        H, W = 2 * int(rng.randint(23, 60)) + 1, 2 * int(rng.randint(23, 60)) + 1
        ims.append(image(rng, H, W, DTYPES[i % 3]))
    return [f"{i:02d}" for i in range(N)], ims, "inputs"


def pipeline(monkeypatch, data, tier, B, sigma):
    monkeypatch.setattr(dp, "load_inputs", lambda path, nthreads=1: data)
    r = dp.usm_radius(sigma)
    staging = dp.STREAM_SLOTS * dp.usm_slot_bytes(data[1], B, (OH, OW), r, True)
    free = (1 << 50) if tier == "device" else dp.MEMORY_MARGIN + staging
    monkeypatch.setattr(dp, "device_budget", lambda device: free)
    p = dp.UnsharpMaskDataPipeline("unused", batch_size=B, output_resolution=(OH, OW), shuffle=True, fliplr=True,
                                   flipud=True, rotate=True, random_crop=True, params={"net_input_size": S},
                                   nthreads=3, seed=7, blur_sigma=sigma, sharpen=1.5)
    assert p.tier == tier
    return p


@pytest.mark.parametrize("B,sigma", [(5, 2.5), (36, 1.0)])
def test_streamed_tier_equals_device_tier(monkeypatch, inputs, B, sigma):
    # (at B = 36 two slots of sigma 2.5's grown windows would hold the whole set: no stream)
    r = dp.usm_radius(sigma)
    dev = pipeline(monkeypatch, inputs, "device", B, sigma)
    assert dev.dataset_bytes == dp.cache_bytes(inputs[1])
    steps = list(range(3 * N // B + 1))
    order = steps + [2, 1] + steps[:3] + [steps[-1], 0]
    want = {s: {k: v.cpu().numpy() for k, v in dev.batch(s).items()} for s in steps}
    with pipeline(monkeypatch, inputs, "stream", B, sigma) as st:
        staged = []
        take = st.stream.take

        def spy(step):
            item = take(step)
            staged.append(item)
            return item

        st.stream.take = spy
        for s in order:
            got = st.batch(s)
            for k, v in want[s].items():
                assert np.array_equal(got[k].cpu().numpy().view(np.uint32), v.view(np.uint32)), (B, s, k)
        for item in staged:                    # the grown input windows alone were staged
            assert item.targets is None
            nbytes = 0
            for x, d, win in zip(item.inputs, item.draws, item.windows):
                a = inputs[1][d.index]
                y0, x0, h, w = dp.grown_window(a.shape[0], a.shape[1], d, OH, OW, r)
                assert win == (a.shape[0], a.shape[1], y0, x0) and tuple(x.shape) == (h, w, 3)
                nbytes += dp._aligned(h * w * 3 * a.itemsize)
            assert item.nbytes == nbytes
    dev.close()


# ---- buffer contract, refusal, large batch --------------------------------------------------------
def _descs(srcs, draws):
    arr = (_lib.UsmSample * len(srcs))()
    for i, (s, d) in enumerate(zip(srcs, draws)):
        arr[i] = _lib.UsmSample(s.data_ptr(), dp._TORCH_FMT[s.dtype], s.shape[0], s.shape[1], 0, 0, s.shape[0],
                                s.shape[1], int(d.fliplr), int(d.flipud), d.rot90, d.crop_y, d.crop_x)
    return arr


def test_buffer_contract():
    """Outputs and the workspace between guard bands (test_buffer_contract_gpu's Harness): under the
    0xFF and 0x5A fills the outputs are bitwise equal and finite and no guard is touched; a workspace
    of exactly the queried size works and one byte short is refused with nothing written."""
    import ctypes

    from test_buffer_contract_gpu import PAT_A, PAT_B, Harness

    rng = np.random.RandomState(5)
    oh, ow, S, sigma = 29, 37, 19, 8.0
    srcs = [image(rng, 40, 50, np.uint8), image(rng, 61, 43, np.float32), image(rng, 45, 45, np.uint16)]
    draws = [Draw(0, True, False, 1, 3, 2), Draw(0, False, True, 2, 10, 1), Draw(0, True, True, 3, 4, 0)]
    lib = _lib.load()
    runs = []
    for fill in (PAT_A, PAT_B):
        h = Harness(fill)
        ins = [h.input(a) for a in srcs]
        descs = _descs(ins, draws)
        need = lib.hdrnet_train_batch_usm_workspace_bytes(ctypes.cast(descs, ctypes.c_void_p), 3, oh, ow, sigma)
        assert need > 0
        out = (h.alloc((3, oh, ow, 3), what="image_input"), h.alloc((3, oh, ow, 3), what="image_output"),
               h.alloc((3, S, S, 3), what="lowres_input"))
        ws = h.alloc((need,), dtype=torch.uint8, what="workspace")
        args = [ctypes.cast(descs, ctypes.c_void_p), 3] + [t.data_ptr() for t in out] + [oh, ow, S, sigma, 1.0,
                                                                                         ws.data_ptr()]
        stream = torch.cuda.current_stream().cuda_stream
        assert lib.hdrnet_train_batch_usm_f32(*args, need - 1, stream) == _lib.E_BAD_SHAPE
        torch.cuda.synchronize()
        for t in out:
            assert (t.view(torch.uint8) == fill).all()          # nothing written
        assert lib.hdrnet_train_batch_usm_f32(*args, need, stream) == _lib.OK
        h.check(f"usm_batch [fill {fill:#04x}]")
        runs.append([t.cpu().numpy() for t in out])
    for a, b in zip(*runs):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and np.isfinite(a).all()
    want = run(srcs, draws, oh, ow, S, sigma, 1.0)
    for g, w in zip(runs[0], want):
        assert np.array_equal(g.view(np.uint32), w.view(np.uint32))


def test_batch_past_2_31_bytes():
    """44 x 2048^2: fullres_out is 2.2e9 bytes.  The first, the last and the image that straddles
    byte 2^31 equal calls on each alone."""
    rng = np.random.RandomState(6)
    B, oh = 44, 2048
    srcs = [torch.from_numpy(image(rng, 2136, 2236, dt)).cuda() for dt in DTYPES]
    draws = []
    for i in range(B):
        lr, ud, k = AUGS[i % 16]
        rh, rw = (2236, 2136) if k % 2 else (2136, 2236)
        draws.append(Draw(0, lr, ud, k, int(rng.randint(0, rh - oh + 1)), int(rng.randint(0, rw - oh + 1))))
    batch = [srcs[i % 3] for i in range(B)]
    fin, fout, low = usm_batch(batch, draws, (oh, oh), 256, 4.0, 1.0)
    assert fout.numel() * 4 > 2 ** 31
    straddle = (2 ** 31) // (oh * oh * 3 * 4)
    for i in (0, straddle, B - 1):
        one = usm_batch([batch[i]], [draws[i]], (oh, oh), 256, 4.0, 1.0)
        for a, b in zip((fin, fout, low), one):
            assert torch.equal(a[i].view(torch.int32), b[0].view(torch.int32)), i


# ---- the public helper --------------------------------------------------------------------------
def test_unsharp_mask_helper():
    rng = np.random.RandomState(8)
    for dt, (H, W) in zip(DTYPES, ((37, 52), (120, 90), (64, 64))):
        src = image(rng, H, W, dt)
        for sigma, sharpen in ((1.0, 1.0), (8.0, 4.0), (32.0, -0.5)):
            got = unsharp_mask(torch.from_numpy(src).cuda(), sigma, sharpen)
            assert got.shape == (H, W, 3) and got.dtype == torch.float32
            got = got.cpu().numpy()
            x = to_float(src)
            want = np.clip(target64(x, blur64(x, sigma), sharpen), 0, 1)
            assert float(np.abs(got - want).max()) <= tol(sharpen)
            pipe = run([src], [Draw(0, False, False, 0, 0, 0)], H, W, 16, sigma, sharpen)[1][0]
            assert np.array_equal(got.view(np.uint32), pipe.view(np.uint32))
    with pytest.raises(ValueError, match="blur_sigma"):
        unsharp_mask(torch.zeros(8, 8, 3, dtype=torch.uint8, device="cuda"), 33.0, 1.0)
