"""The buffer contract of every entry point: each call writes all of its output, writes nothing
outside the buffers it was given, never depends on what a lent workspace (or any buffer it
allocates) held when the call began, and leaves its inputs unchanged.

torch's caching allocator usually hands a call the block the previous call of the same shape just
freed, and that block often already holds the right answer; a kernel that skipped a ragged segment,
a last row or a tail tile would then pass a plain parity test.  Here every buffer is a view into a
larger one with a guard band on each side (>= 64 KiB and >= one image row):

* outputs, VJP buffers, lent workspaces, network-chain scratch, guide buffers and packed weights that
  the package allocates come from a proxy of ``torch`` installed in ``hdrnet_ops``, ``models`` and
  ``host_pipeline``, whose ``empty`` / ``empty_like`` return such views filled with one byte pattern;
* buffers the test lends (``out=``, C-ABI workspaces at exactly the size their query returns, host
  ``out``) are filled the same way;
* inputs sit between guards of 0xFF bytes (NaN), so a read past an input's end that reaches an
  output shows as NaN.

Each case runs twice, under pattern A (0xFF in every byte: NaN / 255 / 65535 / -1) and pattern B
(0x5A: ~1.5e16 in float32).  Then: every output is bitwise equal between the two runs; no float
output is non-finite under A; every guard still holds its pattern; every input is bitwise
unchanged; and the result meets the float64 reference at the bar the suite already holds that kernel
to.  Where AUTO chooses the form, ``hdrnet_slice_apply_plan_ws`` asserts which one it is.  Run with
-s to see the worst error of each group.
"""
import contextlib
import ctypes
import functools
import math
import types

import numpy as np
import pytest
import torch

import oracle
from hdrnet_b200 import _lib, hdrnet_ops, host_pipeline, models
from hdrnet_b200.bin import run
from oracle import cnn_grad_f64 as G
from oracle import model_np as M
from oracle import slice_f64
from test_cnn_grad_gpu import EXTRA
from test_grad_scale_gpu import CASES as VJP_CASES, check as check_vjps, errors as vjp_errors
from util import assert_parity, rand_case, rel_err

gpu = pytest.mark.gpu

PAT_A, PAT_B = 0xFF, 0x5A
GUARD_MIN = 64 << 10
ALIGN = 512                 # torch's allocator aligns blocks to 512 bytes
RTOL = 1e-5
CNN_BAR = 1e-5              # tests/test_cnn_grad_gpu.py BAR

_worst = {}


def note(group, err):
    _worst[group] = max(_worst.get(group, 0.0), float(err))
    return err


@pytest.fixture(scope="module", autouse=True)
def _print_worst_errors():
    yield
    for group, err in sorted(_worst.items()):
        print(f"MEASURE buffer-contract {group}: worst {err:.2e}", flush=True)


# ---- the harness -------------------------------------------------------------------------------
class Guarded:
    """A contiguous view of ``shape`` / ``dtype`` into a larger uint8 buffer, with a guard band on
    each side: at least 64 KiB and at least one image row.  The view starts ``offset`` bytes past a
    512-byte boundary.  The view is filled with ``fill``, the guards with ``guard_fill``."""

    def __init__(self, shape, dtype, device, fill, guard_fill=None, offset=0, pin=False):
        self.shape = tuple(int(s) for s in shape)
        item = torch.empty((), dtype=dtype).element_size()
        self.nbytes = math.prod(self.shape) * item
        lead = math.prod(self.shape[:2]) if len(self.shape) >= 3 else (self.shape[0] if self.shape else 1)
        row = self.nbytes // max(lead, 1)
        guard = -(-max(GUARD_MIN, row) // ALIGN) * ALIGN
        self.buf = torch.empty(2 * guard + ALIGN + offset + self.nbytes, dtype=torch.uint8, device=device,
                               pin_memory=pin)
        self.lo = guard + (-(self.buf.data_ptr() + guard)) % ALIGN + offset
        self.hi = self.lo + self.nbytes
        self.guard_fill = fill if guard_fill is None else guard_fill
        self.buf.fill_(self.guard_fill)
        if fill != self.guard_fill:
            self.buf[self.lo:self.hi].fill_(fill)
        self.view = self.buf[self.lo:self.hi].view(dtype).view(self.shape)
        assert self.view.data_ptr() % ALIGN == offset

    def guard_damage(self):
        """Byte offsets (relative to the view's start) of the first damaged byte below and above
        the view, or None."""
        below = (self.buf[:self.lo] != self.guard_fill).nonzero()
        above = (self.buf[self.hi:] != self.guard_fill).nonzero()
        if len(below) == 0 and len(above) == 0:
            return None
        return (int(below[0]) - self.lo if len(below) else None,
                int(above[0]) + self.nbytes if len(above) else None)


class Harness:
    """The guarded buffers of one run of a case under one fill pattern."""

    def __init__(self, fill):
        self.fill = fill
        self.bufs = []      # (what, Guarded): outputs, scratch and workspaces
        self.inputs = []    # (what, Guarded, bytes at the start)

    def alloc(self, shape, dtype=torch.float32, device="cuda", pin=False, offset=0, what="lent buffer"):
        g = Guarded(shape, dtype, device, self.fill, offset=offset, pin=pin)
        self.bufs.append((what, g))
        return g.view

    def input(self, a, device="cuda", pin=False, what="input"):
        t = torch.from_numpy(np.ascontiguousarray(a)) if isinstance(a, np.ndarray) else a.detach()
        g = Guarded(t.shape, t.dtype, device, PAT_A, pin=pin)
        g.view.copy_(t)
        self.inputs.append((what, g, g.buf[g.lo:g.hi].clone()))
        return g.view

    def lent_sizes(self):
        return [g.nbytes for _, g in self.bufs]

    def check(self, case):
        _sync()
        for what, g in self.bufs + [(w, g) for w, g, _ in self.inputs]:
            bad = g.guard_damage()
            assert bad is None, (f"{case}: a write outside {what} {g.shape} ({g.nbytes} bytes): first "
                                 f"damaged byte below / above the view at {bad}")
        for what, g, before in self.inputs:
            changed = (g.buf[g.lo:g.hi] != before).nonzero()
            assert len(changed) == 0, f"{case}: {what} {g.shape} changed (first byte {int(changed[0])})"


class _PoisonedTorch(types.ModuleType):
    """``torch`` as the package modules see it under the harness: ``empty`` / ``empty_like`` return
    guarded buffers under the current pattern; everything else is torch's own."""

    def __init__(self, harness):
        super().__init__("torch")
        self._h = harness

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *size, dtype=None, device=None, pin_memory=False, **kw):
        if len(size) == 1 and not isinstance(size[0], int):
            size = tuple(size[0])
        return self._h.alloc(size, dtype or torch.get_default_dtype(), torch.device("cpu") if device is None else device,
                             pin=pin_memory, what=f"package allocation {tuple(size)}")

    def empty_like(self, t, dtype=None, device=None, **kw):
        return self._h.alloc(t.shape, dtype or t.dtype, t.device if device is None else device,
                             what=f"package allocation like {tuple(t.shape)}")


POISONED_MODULES = (hdrnet_ops, models, host_pipeline)


@contextlib.contextmanager
def poisoned(harness):
    proxy = _PoisonedTorch(harness)
    saved = [m.torch for m in POISONED_MODULES]
    for m in POISONED_MODULES:
        m.torch = proxy
    try:
        yield
    finally:
        for m, t in zip(POISONED_MODULES, saved):
            m.torch = t


def _sync():
    if torch.cuda.is_available():
        torch.cuda.synchronize()


def _bytes(t):
    return t.detach().contiguous().reshape(-1).view(torch.uint8)


def contract(case, fn):
    """Runs ``fn(harness) -> {name: tensor}`` under pattern A and under pattern B and checks the
    buffer contract; returns the outputs of the run under A."""
    runs = []
    for fill in (PAT_A, PAT_B):
        h = Harness(fill)
        models.invalidate_prepared()          # packed weights are rebuilt under this fill
        models._host_pipelines.clear()        # and so are the host pipeline's frame buffers
        with poisoned(h):
            outs = fn(h)
        h.check(f"{case} [fill {fill:#04x}]")
        runs.append(outs)
    a, b = runs
    assert a.keys() == b.keys()
    for k in a:
        ba, bb = _bytes(a[k]), _bytes(b[k])
        if not torch.equal(ba, bb):
            n = int((ba != bb).sum())
            first = int((ba != bb).nonzero()[0]) // a[k].element_size()
            raise AssertionError(f"{case}: {k} {tuple(a[k].shape)} depends on what its buffers held: {n} bytes "
                                 f"differ between fills, first at element {first}")
        if a[k].is_floating_point():
            bad = ~torch.isfinite(a[k].detach())
            assert not bool(bad.any()), (f"{case}: {k} has {int(bad.sum())} non-finite elements under the NaN fill "
                                         f"(first at {int(bad.reshape(-1).nonzero()[0])})")
    return a


def np_(t):
    return t.detach().cpu().numpy()


# ---- harness self-test (CPU) -------------------------------------------------------------------
def _fake_kernel(defect):
    """A float32 'kernel' written in torch on CPU tensors: out = 2 * x, its output allocated through
    the package's (proxied) torch, with one of three defects."""
    def fn(h):
        x = h.input(np.arange(1000, dtype=np.float32), device="cpu")
        out = hdrnet_ops.torch.empty(x.shape, dtype=torch.float32)
        n = x.numel() - (1 if defect == "last unwritten" else 0)
        out[:n] = 2.0 * x[:n]
        if defect == "one past the end":
            torch.as_strided(out, (x.numel() + 1,), (1,), out.storage_offset())[-1] = 0.0
        if defect == "input modified":
            x[7] = -1.0
        return {"out": out}
    return fn


def test_harness_flags_each_broken_fake_kernel():
    got = contract("correct fake", _fake_kernel(None))
    assert torch.equal(got["out"], 2.0 * torch.arange(1000, dtype=torch.float32))
    for defect, msg in (("last unwritten", "depends on what its buffers held"),
                        ("one past the end", "a write outside"),
                        ("input modified", "changed")):
        with pytest.raises(AssertionError, match=msg):
            contract(defect, _fake_kernel(defect))
    assert all(m.torch is torch for m in POISONED_MODULES)


def test_guarded_buffer_layout():
    for shape, dtype, offset in (((3, 5, 7, 3), torch.float32, 0), ((2, 4, 4000, 3), torch.uint8, 16),
                                 ((9,), torch.int32, 0), ((4, 3), torch.uint16, 16)):
        g = Guarded(shape, dtype, "cpu", PAT_B, guard_fill=PAT_A, offset=offset)
        assert g.view.shape == shape and g.view.dtype == dtype and g.view.is_contiguous()
        assert g.view.data_ptr() % ALIGN == offset
        row = g.nbytes // math.prod(shape[:2]) if len(shape) >= 3 else g.nbytes // shape[0]
        assert min(g.lo, len(g.buf) - g.hi) >= max(GUARD_MIN, row)
        assert bool((g.buf[:g.lo] == PAT_A).all()) and bool((g.buf[g.lo:g.hi] == PAT_B).all())
        assert g.guard_damage() is None
        g.buf[g.hi] = 0
        assert g.guard_damage() == (None, g.nbytes)


# ---- what AUTO picks ---------------------------------------------------------------------------
def plan(B, H, W, gh, gw, gd, n_in=3, n_out=3, has_offset=True, ws=True):
    """(variant, threads) of hdrnet_slice_apply_plan_ws.  threads 384: the issuer-warp form with the
    slab warp; 352: the same form fed by the pre-pass."""
    v, c, t, s = (ctypes.c_int() for _ in range(4))
    rc = _lib.load().hdrnet_slice_apply_plan_ws(B, H, W, gh, gw, gd, n_in, n_out, int(has_offset), int(ws),
                                                ctypes.byref(v), ctypes.byref(c), ctypes.byref(t), ctypes.byref(s))
    _lib.check(rc, "plan")
    return v.value, t.value


def stream():
    return torch.cuda.current_stream().cuda_stream


# ---- bilateral_slice_apply, float32 3 -> 3 -----------------------------------------------------
@functools.lru_cache(maxsize=4)
def apply_case(shape, seed):
    grid, guide, inp = rand_case(seed, *shape, signed=True)
    return grid, guide, inp, slice_f64.bilateral_slice_apply(grid, guide, inp, True)


V = _lib
APPLY_CASES = {
    # id: (shape B, H, W, gh, gw, gd; variant; the form AUTO must pick (variant, threads or None))
    "generic-forced": ((3, 30, 25, 16, 12, 8), V.VARIANT_GENERIC, None),
    "any-shape-30x25": ((3, 30, 25, 16, 12, 8), V.VARIANT_AUTO, (V.VARIANT_GENERIC, None)),
    "any-shape-157x1023": ((2, 157, 1023, 7, 9, 5), V.VARIANT_AUTO, (V.VARIANT_GENERIC, None)),
    "tma-two-ragged-segments": ((2, 7, 1028, 5, 7, 3), V.VARIANT_AUTO, (V.VARIANT_TMA, None)),
    "tex-forced-1080p-rows": ((1, 300, 1920, 16, 16, 8), V.VARIANT_TEX, None),
    "tex-async-non-lean": ((3, 9, 128, 8, 64, 4), V.VARIANT_TEX_ASYNC, None),      # W < 4 gw
    "auto-slab-warp": ((1, 1100, 2048, 16, 16, 8), V.VARIANT_AUTO, (V.VARIANT_TEX_ASYNC, 384)),
    "auto-pre-pass-1008-byte-rows": ((1, 1024, 2052, 5, 7, 3), V.VARIANT_AUTO, (V.VARIANT_TEX_ASYNC, 352)),
}


@gpu
@pytest.mark.parametrize("lend_out", [False, True], ids=["package-out", "lent-out"])
@pytest.mark.parametrize("name", list(APPLY_CASES))
def test_slice_apply(name, lend_out):
    shape, variant, form = APPLY_CASES[name]
    B, H, W = shape[:3]
    if form is not None:
        v, t = plan(*shape)
        assert v == form[0] and (form[1] is None or t == form[1]), f"{name}: AUTO plans ({v}, {t}), not {form}"
    grid, guide, inp, want = apply_case(shape, 100 + list(APPLY_CASES).index(name))

    def fn(h):
        out = h.alloc((B, H, W, 3), what="out") if lend_out else None
        with torch.no_grad():
            got = hdrnet_ops.bilateral_slice_apply(h.input(grid), h.input(guide), h.input(inp), True, out=out,
                                                   variant=variant)
        assert out is None or got.data_ptr() == out.data_ptr()
        return {"out": got}

    got = np_(contract(name, fn)["out"])
    note("slice_apply", rel_err(got, want))
    assert_parity(got, want, rtol=RTOL, what=name)


@gpu
@pytest.mark.parametrize("offset", [0, 16, 128], ids=["aligned", "+16", "+128"])
def test_slice_apply_c_abi_workspace(offset):
    """The C-ABI call with the workspace lent at exactly hdrnet_slice_apply_workspace_bytes.  Aligned:
    the slab-warp form.  The texture-assisted forms read the workspace through a texture object,
    which needs the device's texture alignment (512 bytes): 16 or 128 bytes past it AUTO runs the TMA
    row kernel, and a forced TEX_ASYNC is refused before any launch (the output keeps its fill)."""
    shape = (1, 1100, 2048, 16, 16, 8)
    B, H, W, gh, gw, gd = shape
    assert plan(*shape) == (V.VARIANT_TEX_ASYNC, 384)
    grid, guide, inp, want = apply_case(shape, 120)
    lib = _lib.load()
    nbytes = lib.hdrnet_slice_apply_workspace_bytes(B, H, gw, gd)

    def call(h, variant):
        g, u, i = h.input(grid), h.input(guide), h.input(inp)
        out = h.alloc((B, H, W, 3), what="out")
        ws = h.alloc((nbytes,), torch.uint8, offset=offset, what="workspace")
        rc = lib.hdrnet_slice_apply_f32_ws(g.data_ptr(), u.data_ptr(), i.data_ptr(), out.data_ptr(), B, H, W,
                                           gh, gw, gd, 3, 3, 1, variant, ws.data_ptr(), nbytes, stream())
        return rc, out

    def fn(h):
        rc, out = call(h, V.VARIANT_AUTO)
        _lib.check(rc, "slice_apply_ws")
        return {"out": out}

    got = np_(contract(f"workspace +{offset}", fn)["out"])
    note("slice_apply", rel_err(got, want))
    assert_parity(got, want, rtol=RTOL, what=f"workspace +{offset}")
    if offset:
        h = Harness(PAT_A)
        rc, out = call(h, V.VARIANT_TEX_ASYNC)
        h.check(f"forced TEX_ASYNC, workspace +{offset}")
        assert rc == _lib.E_UNSUPPORTED and bool((_bytes(out) == PAT_A).all())


@gpu
def test_slice_apply_pre_pass_form_on_the_4k_32x32x16_grid():
    """Two more 24 KB grid rows would not leave the slab warp a ring of >= 3 stages: the pre-pass."""
    shape = (1, 2160, 3840, 32, 32, 16)
    assert plan(*shape) == (V.VARIANT_TEX_ASYNC, 352)
    grid, guide, inp, want = apply_case(shape, 121)

    def fn(h):
        with torch.no_grad():
            return {"out": hdrnet_ops.bilateral_slice_apply(h.input(grid), h.input(guide), h.input(inp), True)}

    got = np_(contract("4K 32x32x16", fn)["out"])
    note("slice_apply", rel_err(got, want))
    assert_parity(got, want, rtol=RTOL, what="4K 32x32x16")


# The benchmarked call: 8 x 4K, 16 x 16 x 8 (bench.py's shape and tests/test_slice_apply_gpu.py's seed)
BIG = (8, 2160, 3840, 16, 16, 8)


@functools.lru_cache(maxsize=1)
def big_case():
    return rand_case(1234, *BIG)


@functools.lru_cache(maxsize=None)
def big_f64(b):
    grid, guide, inp = big_case()
    return slice_f64.bilateral_slice_apply(grid[b:b + 1], guide[b:b + 1], inp[b:b + 1], True)[0]


@gpu
def test_slice_apply_benchmarked_call():
    """Images 0 and 7 against the float64 reference; the two-fill equality covers all 8
    (tests/test_slice_apply_gpu.py holds all 66 MP to the compiled reference loops)."""
    assert plan(*BIG) == (V.VARIANT_TEX_ASYNC, 384)
    grid, guide, inp = big_case()

    def fn(h):
        with torch.no_grad():
            return {"out": hdrnet_ops.bilateral_slice_apply(h.input(grid), h.input(guide), h.input(inp), True)}

    out = contract("8 x 4K", fn)["out"]
    for b in (0, 7):
        got = np_(out[b])
        note("slice_apply 8x4K", rel_err(got, big_f64(b)))
        assert_parity(got, big_f64(b), rtol=RTOL, what=f"8 x 4K image {b}")


# ---- bilateral_slice_apply, general channel counts (the any-shape row kernel) -------------------
@gpu
@pytest.mark.parametrize("n_in,n_out,has_offset,W", [(3, 3, False, 1000), (3, 4, True, 1026), (2, 5, False, 777),
                                                      (3, 3, True, 1023), (3, 9, True, 640), (1, 1, True, 65)])
def test_slice_apply_general_channels(n_in, n_out, has_offset, W):
    shape = (2, 157, W, 7, 9, 5)
    assert plan(*shape, n_in, n_out, has_offset)[0] == V.VARIANT_GENERIC
    grid, guide, inp = rand_case(23, *shape, n_in, n_out, has_offset, signed=True)
    want = slice_f64.bilateral_slice_apply(grid, guide, inp, has_offset)

    def fn(h):
        with torch.no_grad():
            return {"out": hdrnet_ops.bilateral_slice_apply(h.input(grid), h.input(guide), h.input(inp), has_offset)}

    got = np_(contract(f"{n_in}->{n_out} offset={has_offset} W={W}", fn)["out"])
    note("slice_apply channels", rel_err(got, want))
    assert_parity(got, want, rtol=RTOL, what=f"{n_in}->{n_out} offset={has_offset} W={W}")


# ---- bilateral_slice_apply_rows ----------------------------------------------------------------
@gpu
def test_row_bands_of_a_4k_frame():
    """The two 1080-row bands of image 0 of the benchmarked call (4.1 MP each: a lent workspace and
    the issuer-warp form at a non-zero row offset)."""
    grid, guide, inp = big_case()
    H, W = BIG[1:3]
    assert plan(1, 1080, W, 16, 16, 8)[0] == V.VARIANT_TEX_ASYNC
    for y0 in (0, 1080):
        def fn(h):
            with torch.no_grad():
                return {"out": hdrnet_ops.bilateral_slice_apply_rows(
                    h.input(grid[:1]), h.input(guide[:1, y0:y0 + 1080]), h.input(inp[:1, y0:y0 + 1080]), True, y0, H)}
        got = np_(contract(f"4K band at {y0}", fn)["out"])[0]
        want = big_f64(0)[y0:y0 + 1080]
        note("slice_apply rows", rel_err(got, want))
        assert_parity(got, want, rtol=RTOL, what=f"4K band at row {y0}")


@gpu
def test_row_band_of_40_rows_at_row_24():
    shape = (2, 96, 256, 16, 16, 8)
    grid, guide, inp, want = apply_case(shape, 122)
    y0, rows = 24, 40

    def fn(h):
        out = h.alloc((2, rows, 256, 3), what="out")
        with torch.no_grad():
            hdrnet_ops.bilateral_slice_apply_rows(h.input(grid), h.input(guide[:, y0:y0 + rows]),
                                                  h.input(inp[:, y0:y0 + rows]), True, y0, 96, out=out)
        return {"out": out}

    got = np_(contract("40-row band", fn)["out"])
    note("slice_apply rows", rel_err(got, want[:, y0:y0 + rows]))
    assert_parity(got, want[:, y0:y0 + rows], rtol=RTOL, what="40-row band at 24")


# ---- bilateral_slice, slice_indices ------------------------------------------------------------
SLICE_CASES = {
    "tma-gc12": ((2, 96, 256, 16, 16, 8), 12, V.VARIANT_AUTO),
    "any-shape-gc2": ((2, 157, 1023, 7, 9, 5), 2, V.VARIANT_AUTO),
    "any-shape-gc13": ((2, 157, 1023, 7, 9, 5), 13, V.VARIANT_AUTO),
    "any-shape-gc24": ((2, 157, 1023, 7, 9, 5), 24, V.VARIANT_AUTO),
    "generic-forced-gc12": ((3, 30, 25, 16, 12, 8), 12, V.VARIANT_GENERIC),
}


@gpu
@pytest.mark.parametrize("name", list(SLICE_CASES))
def test_slice_and_indices(name):
    (B, H, W, gh, gw, gd), gc, variant = SLICE_CASES[name]
    rng = np.random.RandomState(130 + gc)
    grid = rng.randn(B, gh, gw, gd, gc).astype(np.float32)
    guide = rng.rand(B, H, W).astype(np.float32)
    guide[:, :, ::13] = 1.4                                   # clamped depth corners too
    want = slice_f64.bilateral_slice(grid, guide)

    def fn(h):
        g, u = h.input(grid), h.input(guide)
        with torch.no_grad():
            return {"out": hdrnet_ops.bilateral_slice(g, u, variant=variant),
                    "idx": hdrnet_ops.slice_indices(u, (gh, gw, gd))}

    got = contract(name, fn)
    note("slice", rel_err(np_(got["out"]), want))
    assert_parity(np_(got["out"]), want, rtol=RTOL, what=name)
    assert np.array_equal(np_(got["idx"]), oracle.port().slice_indices(guide, gh, gw, gd)), f"{name}: indices"


# ---- guide-fused model path (_fullres) ---------------------------------------------------------
GUIDE_PARAMS = {"curves": dict(M.DEFAULT_PARAMS),
                "nn": dict(M.DEFAULT_PARAMS, model_name="HDRNetPointwiseNNGuide", batch_norm=True)}
FULLRES_SIZES = {
    "row-kernel-2x24x256": (2, 24, 256),        # the row kernel, no workspace
    "texture-1x548x3840": (1, 548, 3840),       # >= 2 Mi px: issuer-warp (curves) / block-synchronous (NN) forms
    "ragged-1x1024x2052": (1, 1024, 2052),      # the same forms with W % 16 != 0: a ragged last segment
    "per-pixel-2x11x100": (2, 11, 100),         # the per-pixel px kernel / the guide-kernel fallback
}
PX_DTYPES = {"f32": torch.float32, "u8": torch.uint8, "u16": torch.uint16}


def quantize(x):
    """tf.cast(255.0 * tf.clip_by_value(x, 0, 1), tf.uint8) (hdrnet/bin/run.py:95)."""
    return (np.float32(255.0) * np.clip(x.astype(np.float32), 0, 1)).astype(np.uint8)


@functools.lru_cache(maxsize=8)
def fullres_case(kind, in_name, size):
    """Image, coefficients, weights and the staged reference: the pinned slice oracle fed the
    standalone guide kernel's guide (as tests/test_models.py stages it)."""
    B, H, W = FULLRES_SIZES[size]
    p = GUIDE_PARAMS[kind]
    wts = M.make_weights(p, seed=140)
    rng = np.random.RandomState(141)
    if in_name == "f32":
        im = rng.rand(B, H, W, 3).astype(np.float32)
    else:
        npt = np.uint8 if in_name == "u8" else np.uint16
        im = rng.randint(0, np.iinfo(npt).max + 1, size=(B, H, W, 3)).astype(npt)
    coeffs = (0.6 * rng.randn(B, 16, 16, 8, 3, 4)).astype(np.float32)
    coeffs[..., [0, 1, 2], [0, 1, 2]] += 1.0
    cls = getattr(models, p["model_name"])
    params = dict(p, weights=wts)
    with torch.no_grad():
        imf = models.image_to_float(torch.from_numpy(im).cuda())
        guide = cls._guide(imf, params)
    stage = oracle.best().bilateral_slice_apply(coeffs.reshape(B, 16, 16, 8, 12), np_(guide), np_(imf), True)
    return im, coeffs, params, np_(imf), stage


@gpu
@pytest.mark.parametrize("debug", [False, True], ids=["no-debug", "debug"])
@pytest.mark.parametrize("size", list(FULLRES_SIZES))
@pytest.mark.parametrize("in_name", list(PX_DTYPES))
@pytest.mark.parametrize("kind", list(GUIDE_PARAMS))
def test_guide_fused_fullres(kind, in_name, size, debug):
    """Float32 and uint8 output of one call each; with ``debug`` the guide dump (guide_out) too."""
    im, coeffs, params, imf, stage = fullres_case(kind, in_name, size)
    cls = getattr(models, params["model_name"])
    params = dict(params, debug=debug)

    def fn(h):
        x, c = h.input(im), h.input(coeffs)
        outs = {}
        with torch.no_grad():
            for name, dt in (("f32", torch.float32), ("u8", torch.uint8)):
                outs[name] = cls._fullres(c, x, params, dt)
                if debug:
                    outs["guide " + name] = cls.last_debug["guide"]
        return outs

    case = f"{kind} {in_name} {size} debug={debug}"
    got = contract(case, fn)
    f = np_(got["f32"])
    note(f"fullres {kind}", rel_err(f, stage))
    assert_parity(f, stage, rtol=RTOL, what=case + " float32 out")
    u = np_(got["u8"]).astype(int)
    assert np.abs(u - quantize(stage).astype(int)).max() <= 1, case + " uint8 out"
    if debug:
        ref = (M.guide_curves if kind == "curves" else M.guide_nn)(imf, params["weights"])
        for name in ("f32", "u8"):
            err = np.abs(np_(got["guide " + name]) - ref).max()
            note("fullres guide_out", err)
            assert err < 2e-6, f"{case}: guide_out of the {name} call: {err:.3e}"


@gpu
def test_pyramid_inference():
    """HDRNetGaussianPyrNN at 1 x 1088 x 1940: level 0 (2.1 MP, W % 4 == 0) runs the fused NN row
    kernel; the 970- and 485-wide levels take the lent guide scratch; resize with and without add."""
    p = dict(M.DEFAULT_PARAMS, model_name="HDRNetGaussianPyrNN", net_input_size=128, spatial_bin=16)
    params = dict(p, weights=M.make_weights(p, seed=150))
    cls = models.HDRNetGaussianPyrNN
    rng = np.random.RandomState(151)
    low = rng.rand(1, 128, 128, 3).astype(np.float32)
    full = rng.rand(1, 1088, 1940, 3).astype(np.float32)
    with torch.no_grad():
        cls.inference(torch.from_numpy(low).cuda(), torch.from_numpy(full).cuda(), dict(params, debug=True))
    dbg = cls.last_debug
    c = np_(dbg["bilateral_coefficients"])
    lvls = [full]
    for _ in range(2):
        lvls.append(M.resize_bilinear_ac(lvls[-1], lvls[-1].shape[1] // 2, lvls[-1].shape[2] // 2))
    assert [l.shape[2] for l in lvls] == [1940, 970, 485]
    stage = None
    for il in range(3):                                     # as tests/test_models.py
        src = 2 - il
        ci = np.ascontiguousarray(c[:, :, :, :, il * 3:(il + 1) * 3, :]).reshape(c.shape[:4] + (12,))
        o = oracle.best().bilateral_slice_apply(ci, np_(dbg["guide"][src]), lvls[src], True)
        stage = o if il == 0 else M.resize_bilinear_ac(stage, o.shape[1], o.shape[2]) + o

    def fn(h):
        with torch.no_grad():
            return {"out": cls.inference(h.input(low), h.input(full), params)}

    got = np_(contract("pyramid", fn)["out"])
    note("pyramid stage", rel_err(got, stage))
    assert_parity(got, stage, rtol=RTOL, elem_rtol=None, what="pyramid")


# ---- guide, lowres and resize kernels ----------------------------------------------------------
@gpu
@pytest.mark.parametrize("kind", list(GUIDE_PARAMS))
def test_guide_kernels(kind):
    """npix % 4 != 0: float4 quads and a scalar tail."""
    p = GUIDE_PARAMS[kind]
    params = dict(p, weights=M.make_weights(p, seed=160))
    cls = getattr(models, p["model_name"])
    for B, H, W in ((1, 17, 257), (2, 37, 53), (1, 3, 1)):
        full = np.random.RandomState(161 + W).rand(B, H, W, 3).astype(np.float32)
        got = np_(contract(f"{kind} guide {B}x{H}x{W}", lambda h: {"g": cls._guide(h.input(full), params)})["g"])
        err = np.abs(got - (M.guide_curves if kind == "curves" else M.guide_nn)(full, params["weights"])).max()
        note("guide", err)
        assert err < 2e-6, f"{kind} guide {B}x{H}x{W}: {err:.3e}"


@gpu
@pytest.mark.parametrize("in_name", list(PX_DTYPES))
def test_lowres_from_image(in_name):
    rng = np.random.RandomState(170)
    B, H, W, S = 2, 120, 250, 64
    if in_name == "f32":
        im = rng.rand(B, H, W, 3).astype(np.float32)
    else:
        npt = np.uint8 if in_name == "u8" else np.uint16
        im = rng.randint(0, np.iinfo(npt).max + 1, size=(B, H, W, 3)).astype(npt)
    want = np.stack([run.nearest_resize(run.img_as_float(im[b]), S) for b in range(B)])
    got = contract(f"lowres {in_name}", lambda h: {"low": models.lowres_from_image(h.input(im), S)})["low"]
    assert np.array_equal(np_(got), want), f"lowres {in_name}"


@gpu
@pytest.mark.parametrize("B,H,W,oh,ow", [(2, 64, 96, 32, 48), (1, 33, 50, 16, 25), (1, 5, 7, 1, 1)])
def test_resize(B, H, W, oh, ow):
    rng = np.random.RandomState(H)
    x = rng.rand(B, H, W, 3).astype(np.float32)
    add = rng.rand(B, oh, ow, 3).astype(np.float32)
    got = contract(f"resize {H}x{W}->{oh}x{ow}", lambda h: {
        "plain": models._resize(h.input(x), oh, ow), "add": models._resize(h.input(x), oh, ow, add=h.input(add))})
    want = M.resize_bilinear_ac(x, oh, ow).astype(np.float64)
    for name, ref in (("plain", want), ("add", want + add)):
        err = np.abs(np_(got[name]) - ref).max()
        note("resize", err)
        assert err < 2e-6, f"resize {name}: {err:.3e}"


# ---- coefficient network: layers, fusion, the whole network ------------------------------------
CONV_CASES = {
    # id: (B, H, W, Cin, Cout, k, stride, packed)
    "cuda-core-cout100": (2, 48, 64, 16, 100, 3, 1, False),   # Cout % 4 == 0: too many CTAs for the patch form
    "cuda-core-cout18": (2, 33, 50, 5, 18, 3, 2, False),      # Cout % 4 != 0
    "patch-4ch": (1, 16, 16, 64, 64, 3, 1, False),            # 128 CTAs of 4 output channels
    "patch-8ch": (2, 16, 16, 64, 64, 3, 1, False),            # > 1 CTA per SM: 8 channels per CTA
    "wgmma-unpacked": (4, 64, 64, 16, 32, 3, 1, False),       # 128 tiles of 128 pixels
    "wgmma-packed": (2, 64, 64, 32, 64, 3, 1, True),          # 64 tiles, pre-packed weights
    "wgmma-cout192": (1, 112, 112, 64, 192, 3, 1, False),     # 98 tiles; Cout > 128: two launches
}


@gpu
@pytest.mark.parametrize("name", list(CONV_CASES))
def test_conv(name):
    B, H, W, cin, cout, k, s, packed = CONV_CASES[name]
    rng = np.random.RandomState(180 + cout)
    x = rng.randn(B, H, W, cin).astype(np.float32)
    w = (rng.randn(k, k, cin, cout) / np.sqrt(k * k * cin)).astype(np.float32)
    b = rng.randn(cout).astype(np.float32)
    want = np.maximum(M.conv2d_same(x, w, s) + b, 0)
    nbytes = _lib.load().hdrnet_conv2d_tc_packed_bytes(k, cin, cout)

    def fn(h):
        wd = h.input(w)
        outs = {}
        if packed:
            outs["packed"] = models.pack_conv_weights(wd)
            assert outs["packed"].numel() * 4 == nbytes
        with torch.no_grad():
            outs["out"] = models._conv(h.input(x), (wd, h.input(b), outs.get("packed")), stride=s, relu=True)
        return outs

    got = np_(contract(name, fn)["out"])
    note("conv", rel_err(got, want))
    assert_parity(got, want, rtol=RTOL, elem_rtol=None, what=name)


@gpu
@pytest.mark.parametrize("B,I,O", [(8, 1024, 256), (11, 70, 37)], ids=["cluster", "plain"])
def test_fc(B, I, O):
    rng = np.random.RandomState(I + O)
    x = rng.randn(B, I).astype(np.float32)
    w = (rng.randn(I, O) / np.sqrt(I)).astype(np.float32)
    b = rng.randn(O).astype(np.float32)
    want = np.maximum(x.astype(np.float64) @ w + b, 0)
    got = np_(contract(f"fc {B}x{I}->{O}", lambda h: {
        "out": models._fc(h.input(x), (h.input(w), h.input(b)), relu=True)})["out"])
    note("fc", rel_err(got, want))
    assert_parity(got, want, rtol=RTOL, elem_rtol=None, what=f"fc {B}x{I}->{O}")


@gpu
@pytest.mark.parametrize("C,n_out", [(64, 3), (256, 9)], ids=["weights-in-smem", "weights-through-cache"])
def test_fuse_predict(C, n_out):
    rng = np.random.RandomState(190 + C)
    B, gh, gw, gd, n_in = 2, 5, 7, 8, 4
    O = gd * n_out * n_in
    loc = rng.randn(B, gh, gw, C).astype(np.float32)
    glob = rng.randn(B, C).astype(np.float32)
    w = (rng.randn(C, O) / np.sqrt(C)).astype(np.float32)
    b = rng.randn(O).astype(np.float32)
    f = np.maximum(loc + glob[:, None, None, :], 0).astype(np.float64)
    want = (f @ w.astype(np.float64) + b).reshape(B, gh, gw, n_in, n_out, gd).transpose(0, 1, 2, 5, 4, 3)

    def fn(h):
        grid = h.alloc((B, gh, gw, gd, n_out, n_in), what="grid")
        _lib.check(_lib.load().hdrnet_fuse_predict_f32(
            h.input(loc).data_ptr(), h.input(glob).data_ptr(), h.input(w).data_ptr(), h.input(b).data_ptr(),
            grid.data_ptr(), B, gh, gw, C, gd, n_out, n_in, stream()), "fuse_predict")
        return {"grid": grid}

    got = np_(contract(f"fuse_predict C={C}", fn)["grid"])
    note("fuse_predict", rel_err(got, want))
    assert_parity(got, want, rtol=RTOL, elem_rtol=None, what=f"fuse_predict C={C}")


NET = dict(M.DEFAULT_PARAMS, net_input_size=128, spatial_bin=16)


@gpu
@pytest.mark.parametrize("B", [1, 4, 16, 17])
def test_coefficients(B):
    """B <= 16: the whole network behind one call, its scratch allocated at exactly
    hdrnet_coefficients_scratch_bytes; B = 17: layer by layer (tensor-core convs on packed weights)."""
    assert models.CHAIN_CNN_MAX_BATCH == 16
    wts = M.make_weights(NET, seed=200)
    low = np.random.RandomState(201 + B).rand(B, 128, 128, 3).astype(np.float32)
    want = M.coefficients(low, wts, NET)
    scratch = _lib.load().hdrnet_coefficients_scratch_bytes(B, 128, 16, 8, 1, 3, 4)
    sizes = []

    def fn(h):
        with torch.no_grad():
            out = models.HDRNetCurves._coefficients(h.input(low), dict(NET, weights=wts))
        sizes[:] = h.lent_sizes()
        return {"grid": out}

    got = np_(contract(f"coefficients B={B}", fn)["grid"])
    assert (scratch in sizes) == (B <= 16), f"B={B}: chain scratch {scratch} bytes among {sizes}"
    note("coefficients", rel_err(got, want))
    assert_parity(got, want, rtol=2e-5, elem_rtol=None, what=f"coefficients B={B}")


# ---- backward ----------------------------------------------------------------------------------
TRAIN = dict(models.DEFAULT_PARAMS)
P = G.P


@gpu
def test_fine_tuning_step():
    """One step of HDRNetCurves at the reference's training size (16 x 256² network input, 16 x 512²
    output, L2 loss): the gradient of every coefficient variable against slice_f64's grid VJP fed
    through the float64 network's backward (as tests/test_cnn_grad_gpu.py)."""
    w0 = models.init_weights(TRAIN, seed=2)
    rng = np.random.RandomState(210)
    for k in w0:
        if k.endswith("/biases") and k.startswith(P):
            w0[k] = (0.05 * rng.randn(*w0[k].shape)).astype(np.float32)
    low = rng.rand(16, 256, 256, 3).astype(np.float32)
    full = rng.rand(16, 512, 512, 3).astype(np.float32)
    target = rng.rand(16, 512, 512, 3).astype(np.float32)
    names = G.variable_names(TRAIN)

    def fn(h):
        wts = {k: h.input(v).requires_grad_(k.startswith(P)) for k, v in w0.items()}
        out = models.HDRNetCurves.inference(h.input(low), h.input(full), dict(TRAIN, weights=wts))
        ((out - h.input(target)) ** 2).sum().backward()
        return dict({"out": out.detach()}, **{k: wts[k].grad for k in names})

    got = contract("fine-tuning step", fn)
    with torch.no_grad():
        guide = np_(models.HDRNetCurves._guide(torch.from_numpy(full).cuda(), dict(TRAIN, weights=w0)))
    ct = 2.0 * (np_(got["out"]).astype(np.float64) - target)
    gv = slice_f64.bilateral_slice_apply_grad(np.zeros((16, 16, 16, 8, 12)), guide, full, ct, True)[0]
    net = G.Network(w0, TRAIN)
    net.forward(low)
    want = net.backward(gv.reshape(16, 16, 16, 8, 3, 4))
    for k in names:
        e = note("fine-tuning step grads", rel_err(np_(got[k]), want[k]))
        assert e <= CNN_BAR, f"{k}: {e:.3e}"


@gpu
@pytest.mark.parametrize("case", EXTRA, ids=lambda c: "-".join(str(v) for v in c))
def test_layer_vjps_at_odd_shapes(case):
    """tests/test_cnn_grad_gpu.py's EXTRA shapes through the autograd Functions (dx / dw / db and
    the VJPs' partial-sum workspaces from the package)."""
    kind, B, H, W, cin, cout, k, s, relu, bias = case
    rng = np.random.RandomState(220)
    if kind == "fuse":
        C, gd, n_out, n_in = cin, cout, k, s
        O = gd * n_out * n_in
        arrs = dict(x=rng.randn(B, H, W, C), g=rng.randn(B, C), w=rng.randn(C, O) / np.sqrt(C), b=rng.randn(O) * 0.1)
    else:
        x = np.maximum(rng.randn(B, H, W, cin) if kind == "conv" else rng.randn(B, cin), 0)
        w = rng.randn(*((k, k, cin, cout) if kind == "conv" else (cin, cout))) / np.sqrt(k * k * cin)
        arrs = dict(x=x, w=w, b=rng.randn(cout) * 0.1)
    arrs = {n: a.astype(np.float32) for n, a in arrs.items()}
    if kind != "fuse" and not bias:
        del arrs["b"]
    fwd = {}

    def fn(h):
        t = {n: h.input(a).requires_grad_() for n, a in arrs.items()}
        if kind == "fuse":
            y = models._FusePredictFn.apply(t["x"], t["g"], t["w"], t["b"], gd, n_out, n_in)
        elif kind == "conv":
            y = models._ConvFn.apply(t["x"], t["w"], t.get("b"), s, relu)
        else:
            y = models._FcFn.apply(t["x"], t["w"], t.get("b"), relu)
        fwd["dy"] = np.random.RandomState(221).randn(*y.shape).astype(np.float32)
        y.backward(h.input(fwd["dy"]))
        return dict({"y": y.detach()}, **{"d" + n: v.grad for n, v in t.items()})

    got = contract(f"VJP {case}", fn)
    g = {n: np_(v) for n, v in got.items()}
    if kind == "fuse":
        v = G.fuse_predict_vjp(arrs["x"], arrs["g"], arrs["w"], fwd["dy"], gd, n_out, n_in)
        checks = [("dx", v.dlocal, None), ("dg", v.dglobal, None), ("dw", v.dw, v.dw_abs), ("db", v.db, v.db_abs)]
    else:
        v = (G.conv_vjp(arrs["x"], arrs["w"], g["y"], fwd["dy"], s, relu) if kind == "conv"
             else G.fc_vjp(arrs["x"], arrs["w"], g["y"], fwd["dy"], relu))
        checks = [("dx", v.dx, None), ("dw", v.dw, v.dw_abs)] + ([("db", v.db, v.db_abs)] if bias else [])
    for n, ref, terms in checks:
        e = note("layer VJPs", rel_err(g[n], ref))
        assert e <= CNN_BAR, f"{case} {n}: {e:.3e} of max |ref|"
        if terms is not None:
            pe = float((np.abs(g[n].astype(np.float64) - ref) / np.maximum(terms, 1e-30)).max())
            assert pe <= CNN_BAR, f"{case} {n}: {pe:.3e} of Σ|terms|"


GRID_VJP_CASES = ["switch-gd9-column-ztiles", "switch-gc13-slice-column-ctiles", "gd16-column-ztiles-b16",
                  "gc36-column-ctiles", "switch-small-image-column"]


@gpu
@pytest.mark.parametrize("name", GRID_VJP_CASES)
def test_slice_vjps_at_grid_vjp_tile_edges(name):
    c = VJP_CASES[name]
    grid, guide, inp, ct = c.arrays()

    def fn(h):
        leaves = [h.input(a).requires_grad_() for a in ((grid, guide, inp) if c.op == "apply" else (grid, guide))]
        out = (hdrnet_ops.bilateral_slice_apply(*leaves, c.ho) if c.op == "apply"
               else hdrnet_ops.bilateral_slice(*leaves))
        out.backward(h.input(ct))
        return dict({"out": out.detach()}, **{f"vjp{i}": t.grad for i, t in enumerate(leaves)})

    got = contract(name, fn)
    grads = [np_(got[f"vjp{i}"]) for i in range(3 if c.op == "apply" else 2)] + ([] if c.op == "apply" else [None])
    e = vjp_errors(grads, c.f64(grid, guide, inp, ct))
    for k, v in e.items():
        note(f"slice VJP {k}", v)
    check_vjps(e, name, c.elem_bar)


# ---- host paths --------------------------------------------------------------------------------
@functools.lru_cache(maxsize=1)
def device_out_of_3_4k_frames():
    grid, guide, inp = big_case()
    with torch.no_grad():
        return np_(hdrnet_ops.bilateral_slice_apply(*(torch.from_numpy(a[:3]).cuda() for a in (grid, guide, inp)), True))


@gpu
@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_host_path_at_4k(pinned):
    """3 x 4K with the default context (4 Mi px per band): 1092 + 1068 rows per image, 6 bands over
    3 slots.  Equal bit for bit to the device call on the same frames; image 0 against float64."""
    grid, guide, inp = big_case()

    def fn(h):
        args = [h.input(a[:3], device="cpu", pin=pinned) for a in (grid, guide, inp)]
        out = hdrnet_ops.bilateral_slice_apply(*args, True)
        assert not out.is_cuda and out.is_pinned() == pinned
        return {"out": out}

    got = contract(f"host 3 x 4K {'pinned' if pinned else 'pageable'}", fn)["out"].numpy()
    assert np.array_equal(got, device_out_of_3_4k_frames())
    note("host slice_apply", rel_err(got[0], big_f64(0)))
    assert_parity(got[0], big_f64(0), rtol=RTOL, what="host 4K image 0")


@gpu
def test_host_path_with_small_bands():
    """A context of 5000 pixels per slot: bands of 4 rows and a last band of 1 row per 1023-wide image,
    slots reused across bands and images."""
    shape = (2, 157, 1023, 7, 9, 5)
    B, H, W, gh, gw, gd = shape
    grid, guide, inp, want = apply_case(shape, 230)
    lib = _lib.load()
    ctx = ctypes.c_void_p()
    _lib.check(lib.hdrnet_host_ctx_create(ctypes.byref(ctx), 5000), "host context")
    try:
        def fn(h):
            g, u, i = (h.input(a, device="cpu", pin=True) for a in (grid, guide, inp))
            out = h.alloc((B, H, W, 3), device="cpu", pin=True, what="host out")
            _lib.check(lib.hdrnet_slice_apply_host_f32(ctx, g.data_ptr(), u.data_ptr(), i.data_ptr(), out.data_ptr(),
                                                       B, H, W, gh, gw, gd, 3, 3, 1), "host slice_apply")
            return {"out": out}
        got = contract("host small bands", fn)["out"].numpy()
    finally:
        _lib.check(lib.hdrnet_host_ctx_destroy(ctx), "host context destroy")
    note("host slice_apply", rel_err(got, want))
    assert_parity(got, want, rtol=RTOL, what="host small bands")


@gpu
def test_inference_image_host_into_a_lent_out():
    """5 frames through the three-stream pipeline (2 device frame buffers, reused) into a guarded
    page-locked ``out``: the same bytes as inference_image on each frame."""
    p = dict(GUIDE_PARAMS["curves"], net_input_size=64, spatial_bin=8)
    params = dict(p, weights=M.make_weights(p, seed=240))
    cls = models.HDRNetCurves
    frames = np.random.RandomState(241).randint(0, 256, size=(5, 64, 256, 3)).astype(np.uint8)
    want = np.concatenate([np_(cls.inference_image(torch.from_numpy(frames[i:i + 1]).cuda(), params))
                           for i in range(5)])

    def fn(h):
        out = h.alloc(frames.shape, torch.uint8, device="cpu", pin=True, what="host out")
        got = cls.inference_image_host(h.input(frames, device="cpu", pin=True), params, out=out)
        assert got.data_ptr() == out.data_ptr()
        return {"out": out}

    got = contract("inference_image_host", fn)["out"].numpy()
    assert np.array_equal(got, want)
