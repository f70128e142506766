"""The census table (tests/kernel_census.py) against the library's entry functions, in both directions:
a kernel the library compiles but the table does not list has no case that launches it, and a row
whose kernel is gone tests nothing.  Runs cuobjdump on the built library; no GPU needed."""
import os

import pytest

import kernel_census as K
from hdrnet_b200 import _lib


# (c++filt of the library's cuobjdump symbol, torch.profiler's kernel name, census key).  Both
# spellings were recorded from the same build, the profiler's on an H100 with torch 2.11.
RECORDED = [
    ("void hdrnet_b200::slice_apply_rows_tma_kernel<hdrnet_b200::GuideFromInput, 4, 2, 512, 0, 0>"
     "(hdrnet_b200::TmaArgs, hdrnet_b200::GuideFromInput)",
     "void hdrnet_b200::slice_apply_rows_tma_kernel<hdrnet_b200::GuideFromInput, 4, 2, 512, 0, 0>"
     "(hdrnet_b200::TmaArgs, hdrnet_b200::GuideFromInput)",
     "slice_apply_rows_tma_kernel<GuideFromInput,4,2,512,0,0>"),
    ("void hdrnet_b200::guide_kernel<hdrnet_b200::NNFn<32> >(float const*, float*, long long, bool, hdrnet_b200::NNFn<32>)",
     "void hdrnet_b200::guide_kernel<hdrnet_b200::NNFn<32> >(float const*, float*, long long, bool, hdrnet_b200::NNFn<32>)",
     "guide_kernel<NNFn<32>>"),
    ("hdrnet_b200::(anonymous namespace)::stats_partial_kernel(float const*, double*, long long, int, long long)",
     "hdrnet_b200::(anonymous namespace)::stats_partial_kernel(float const*, double*, long long, int, long long)",
     "stats_partial_kernel"),
    ("(anonymous namespace)::split_level_rows_kernel(float const*, float*, float*, float*, long long)",
     "(anonymous namespace)::split_level_rows_kernel(float const*, float*, float*, float*, long long)",
     "split_level_rows_kernel"),
    ("void hdrnet_b200::conv2d_wgmma_kernel<32, true>(hdrnet_b200::TcConvArgs)",
     "void hdrnet_b200::conv2d_wgmma_kernel<32, true>(hdrnet_b200::TcConvArgs)",
     "conv2d_wgmma_kernel<32,true>"),
    ("hdrnet_b200::yblend_rows_kernel(float const*, float4*, hdrnet_b200::SliceGeom, int)",
     "hdrnet_b200::yblend_rows_kernel(float const*, float4*, hdrnet_b200::SliceGeom, int)",
     "yblend_rows_kernel"),
]


def test_normalise_gives_one_name_for_both_spellings():
    for cuobj, prof, want in RECORDED:
        assert K.normalise(cuobj) == want
        assert K.normalise(prof) == want


def test_normalise_ignores_what_other_demanglers_spell_differently():
    """Return type, blanks inside template arguments and parameter lists of other tools' spellings."""
    for _, _, want in RECORDED:
        for raw in (want, "void " + want + "()", want.replace(",", ", ").replace(">>", "> >") + "(int)"):
            assert K.normalise(raw) == want
    assert K.normalise("guide_kernel<NNFn<32>>(float const*, NNFn<32>)") == "guide_kernel<NNFn<32>>"


def test_every_row_names_a_case():
    assert set(K.ROWS.values()) <= set(K.CASES)
    assert set(K.CASES) <= set(K.ROWS.values()), "cases no row uses"


def test_census_table_equals_the_library_entry_functions(built_lib):
    tool = K.cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump (CUDA toolkit) not found: the census cannot be read from the library")
    assert os.path.exists(_lib.LIB_PATH)
    have = K.library_kernels(_lib.LIB_PATH, tool)
    assert have, "no entry functions read from the library"
    missing = sorted(have - set(K.ROWS))
    gone = sorted(set(K.ROWS) - have)
    assert not missing, ("kernels in the library with no census row (add a case that launches each): "
                         + "; ".join(f"{s}: {k}" for s, k in missing))
    assert not gone, "census rows whose kernel the library no longer has: " + "; ".join(f"{s}: {k}" for s, k in gone)
