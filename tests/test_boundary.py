"""CPU tests of the drop-in boundary: the C-ABI library loads and exports every symbol the
header declares, the Python surface mirrors the reference's names / errors, and the product
never touches the oracle."""
import ast
import os
import re
import subprocess

import pytest
import torch

from hdrnet_b200 import _lib, hdrnet_ops, layers

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def header_functions():
    text = open(_lib.HEADER_PATH).read()
    return sorted(set(re.findall(r"HDRNET_API\s+[\w\s\*]+?\b(hdrnet_\w+)\s*\(", text)))


def test_header_declares_the_expected_entry_points():
    names = header_functions()
    for required in ("hdrnet_slice_apply_f32", "hdrnet_slice_f32", "hdrnet_slice_indices_i32",
                     "hdrnet_slice_apply_host_f32"):
        assert required in names


def test_library_exports_every_declared_symbol(built_lib):
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True,
                         text=True, check=True).stdout
    exported = set(re.findall(r"\bT (hdrnet_\w+)", out))
    declared = set(header_functions())
    assert declared <= exported, f"missing from .so: {sorted(declared - exported)}"
    assert exported <= declared, f"exported but undeclared: {sorted(exported - declared)}"


def test_ctypes_table_covers_the_header(built_lib):
    assert sorted(_lib.SIGNATURES) == header_functions()
    for name in _lib.SIGNATURES:
        assert hasattr(built_lib, name)
    assert built_lib.hdrnet_b200_abi_version() == 1
    assert _lib.error_string(0) == "ok"
    assert "NULL" in _lib.error_string(_lib.E_NULL_POINTER)


def test_library_is_built_for_sm_90a(built_lib):
    out = subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True)
    assert "sm_90a" in out.stdout


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "hdrnet_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            path = os.path.join(dirpath, f)
            if f.endswith(".py"):
                tree = ast.parse(open(path).read())
                for node in ast.walk(tree):
                    mods = []
                    if isinstance(node, ast.Import):
                        mods = [a.name for a in node.names]
                    elif isinstance(node, ast.ImportFrom):
                        mods = [node.module or ""]
                    assert not any(m.split(".")[0] == "oracle" for m in mods), path
            elif f.endswith((".cu", ".cuh", ".h", ".cc")):
                assert "oracle/" not in open(path).read(), path


def test_python_surface_mirrors_reference_names():
    # hdrnet/hdrnet_ops.py:30-31, hdrnet/layers.py:99-198
    assert callable(hdrnet_ops.bilateral_slice) and callable(hdrnet_ops.bilateral_slice_apply)
    for name in ("bilateral_slice", "bilateral_slice_apply", "apply", "conv", "fc"):
        assert callable(getattr(layers, name))
    import inspect
    # positional order of the reference's constructors (hdrnet/layers.py:25-29, :62-66)
    assert list(inspect.signature(layers.conv).parameters)[:11] == [
        "inputs", "num_outputs", "kernel_size", "stride", "rate", "use_bias", "batch_norm", "is_training",
        "activation_fn", "scope", "reuse"]
    assert list(inspect.signature(layers.fc).parameters)[:7] == [
        "inputs", "num_outputs", "use_bias", "batch_norm", "is_training", "activation_fn", "scope"]


def _t(*shape):
    return torch.zeros(*shape, dtype=torch.float32)


@pytest.mark.parametrize("grid,guide,inp,msg", [
    (_t(2, 4, 4, 4), _t(2, 8, 8), _t(2, 8, 8, 3), "Input grid should be 5D"),
    (_t(2, 4, 4, 4, 12), _t(2, 8, 8, 1), _t(2, 8, 8, 3), "Guide image should be 3D"),
    (_t(2, 4, 4, 4, 12), _t(2, 8, 8), _t(2, 8, 8), "Input image should be 4D"),
    (_t(2, 4, 4, 4, 12), _t(2, 8, 8), _t(2, 8, 9, 3), "Input and guide size should match."),
    (_t(3, 4, 4, 4, 12), _t(2, 8, 8), _t(2, 8, 8, 3), "Batch sizes should match."),
    (_t(2, 4, 4, 4, 10), _t(2, 8, 8), _t(2, 8, 8, 3), "Slicing with affine offset"),
])
def test_invalid_arguments_raise_reference_messages(built_lib, grid, guide, inp, msg):
    """hdrnet/ops/bilateral_slice_apply_op.cc:147-193 (InvalidArgument -> ValueError)."""
    with pytest.raises(ValueError, match=re.escape(msg)):
        hdrnet_ops.bilateral_slice_apply(grid, guide, inp, has_offset=True)


def test_invalid_channels_without_offset(built_lib):
    with pytest.raises(ValueError, match="Slicing without affine offset"):
        hdrnet_ops.bilateral_slice_apply(_t(2, 4, 4, 4, 10), _t(2, 8, 8), _t(2, 8, 8, 3),
                                         has_offset=False)


def test_slice_rank_errors(built_lib):
    with pytest.raises(ValueError, match="Grid should be 5D"):
        hdrnet_ops.bilateral_slice(_t(2, 4, 4, 4), _t(2, 8, 8))
    with pytest.raises(ValueError, match="Guide image should be 3D"):
        hdrnet_ops.bilateral_slice(_t(2, 4, 4, 4, 2), _t(2, 8, 8, 1))


def test_non_float_dtype_rejected(built_lib):
    with pytest.raises(TypeError):
        hdrnet_ops.bilateral_slice_apply(_t(2, 4, 4, 4, 12).double(), _t(2, 8, 8), _t(2, 8, 8, 3),
                                         has_offset=True)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_fails_loudly_without_a_gpu(built_lib):
    """No CPU fallback: a valid call without CUDA must raise, not compute."""
    with pytest.raises(_lib.HdrnetLibraryError):
        hdrnet_ops.bilateral_slice_apply(_t(1, 4, 4, 4, 12), _t(1, 8, 8), _t(1, 8, 8, 3),
                                         has_offset=True)


def test_row_band_argument_checks(built_lib):
    """bilateral_slice_apply_rows: the reference op's messages for rank / size / batch / channel
    errors, a band that does not fit the image, and no CPU path."""
    f = hdrnet_ops.bilateral_slice_apply_rows
    grid, guide, inp = _t(1, 4, 4, 8, 12), _t(1, 6, 16), _t(1, 6, 16, 3)
    with pytest.raises(ValueError, match="Input grid should be 5D"):
        f(_t(4, 4, 8, 12), guide, inp, True, 0, 6)
    with pytest.raises(ValueError, match="Input and guide size should match"):
        f(grid, _t(1, 5, 16), inp, True, 0, 6)
    with pytest.raises(ValueError, match="Batch sizes should match"):
        f(_t(2, 4, 4, 8, 12), guide, inp, True, 0, 6)
    with pytest.raises(ValueError, match="output_channels \\* \\(input_channels \\+ 1\\)"):
        f(_t(1, 4, 4, 8, 10), guide, inp, True, 0, 6)
    for y_off, height in ((-1, 10), (5, 10), (0, 5)):
        with pytest.raises(ValueError, match="does not fit an image"):
            f(grid, guide, inp, True, y_off, height)
    if not torch.cuda.is_available():
        with pytest.raises(_lib.HdrnetLibraryError):
            f(grid, guide, inp, True, 2, 10)


def test_layers_apply_matches_reference_semantics():
    """hdrnet/layers.py:153-198 on CPU tensors (pure torch ops, no kernel)."""
    torch.manual_seed(0)
    sliced = torch.rand(2, 5, 4, 3, 4)
    im = torch.rand(2, 5, 4, 3)
    out = layers.apply(sliced, im, has_affine_term=True)
    ref = torch.einsum("bhwij,bhwj->bhwi", sliced[..., :3], im) + sliced[..., 3]
    assert torch.allclose(out, ref, atol=1e-6)
    with pytest.raises(ValueError):
        layers.apply(sliced, im[:, :4], has_affine_term=True)


def _plan(lib, B, H, W, gh, gw, gd, with_ws, n_in=3, n_out=3, has_offset=1):
    import ctypes
    v, c, t, sm = (ctypes.c_int() for _ in range(4))
    rc = lib.hdrnet_slice_apply_plan_ws(B, H, W, gh, gw, gd, n_in, n_out, has_offset, with_ws,
                                        ctypes.byref(v), ctypes.byref(c), ctypes.byref(t), ctypes.byref(sm))
    assert rc == 0
    return v.value, c.value, t.value, sm.value


def test_kernel_selection_plan(built_lib):
    """Host-side kernel selection (no launch; without a device the planner assumes an H100: 132 SMs,
    227 KB of opt-in shared memory): which form AUTO runs for BASELINE.json's shapes."""
    from hdrnet_b200 import _lib
    lib = built_lib
    # config 3 (headline): issuer-warp texture-assisted form, 2 CTAs x 132 SMs, 10 math warps + issuer
    # + slab warp (no pre-pass), 4-stage ring of 1280-pixel segments + 2 slab rows + 2 grid rows
    assert _plan(lib, 8, 2160, 3840, 16, 16, 8, 1) == (_lib.VARIANT_TEX_ASYNC, 264, 384, 106752)
    # no workspace lent: the all-LSU TMA row kernel
    v, c, t, _ = _plan(lib, 8, 2160, 3840, 16, 16, 8, 0)
    assert (v, c, t) == (_lib.VARIANT_TMA, 264, 256)
    # config 4 (12 MP, 8 frames per GPU): three 1344-pixel segments per row, 4-stage ring
    v, c, t, sm = _plan(lib, 8, 3024, 4032, 16, 16, 8, 1)
    assert (v, c, t) == (_lib.VARIANT_TEX_ASYNC, 264, 384) and sm <= 115712
    # config 5's 32x32 grids (24 / 48 KB of slab rows) still leave the 20 KB stages a 3-stage ring;
    # 32x32x16 has no room for two more grid rows: pre-pass form (352 threads)
    assert _plan(lib, 8, 2160, 3840, 32, 32, 8, 1)[:3] == (_lib.VARIANT_TEX_ASYNC, 264, 384)
    assert _plan(lib, 8, 2160, 3840, 32, 32, 16, 1)[:3] == (_lib.VARIANT_TEX_ASYNC, 264, 352)
    assert _plan(lib, 8, 2160, 3840, 8, 8, 4, 1)[0] == _lib.VARIANT_TEX_ASYNC
    # config 2 (one 1080p frame, < 2 Mi px): no pre-pass, TMA row kernel
    assert _plan(lib, 1, 1080, 1920, 16, 16, 8, 1)[0] == _lib.VARIANT_TMA
    # shapes the row kernels cannot take: odd width, other channel counts, tiny images
    assert _plan(lib, 8, 2160, 3841, 16, 16, 8, 1)[0] == _lib.VARIANT_GENERIC
    assert _plan(lib, 8, 2160, 3840, 16, 16, 8, 1, n_out=4)[0] == _lib.VARIANT_GENERIC
    assert _plan(lib, 1, 16, 64, 4, 4, 4, 1)[0] == _lib.VARIANT_GENERIC
    # 96 x 16 cells: two 72 KB grid rows leave no room for the all-LSU row kernel's slab and ring, so
    # no row kernel (nor its texture-assisted forms) takes the call, workspace or not
    assert _plan(lib, 2, 1080, 1920, 16, 96, 16, 1)[0] == _lib.VARIANT_GENERIC
