"""The coefficient network at every batch size where one of its layers changes kernel, against float64.

The network's kernels are chosen by batch size in three places: models.py (the launch chain up to
CHAIN_CNN_MAX_BATCH images, the packed tensor-core conv from PACKED_CONV_MIN_TILES tiles), the conv
and fc dispatch in csrc/cnn.cu (thresholds that scale with the SM count), and csrc/model.cu, which
repeats the two Python constants for the frozen model.  `plan` below restates those rules; the census
checks the restatement against the kernels that actually launch (torch.profiler, in a child process:
a hundred profiling sessions in the test process left later sessions in it without kernel records),
so that a change to the rules fails here instead of leaving the sweep on the wrong sizes.

At every batch size of the sweep, each image's coefficients are held to the float64 network
(oracle/model_np.py) over that image's own range, so that a wrong last image of a tile or an fc pass
cannot hide behind the other images' range.  Batch sizes that launch the same kernel for every layer
must give every image bit-for-bit the same coefficients: no kernel's per-element sum order depends on
where the image sits in a tile or a pass.  The sweep runs descending, then ascending, on the same
weights cache and allocator, with the same results.  The frozen model (csrc/model.cu) must equal the
Python path bitwise on both sides of every crossover of the two constants it repeats.
"""
import re

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from hdrnet_b200 import checkpoint, models
from hdrnet_b200.frozen import FrozenModel
from oracle import model_np as M

# The two constants models.py holds and csrc/model.cu repeats.  A change on the Python side shows
# in the census; a change to model.cu's copies that changes a result, in the frozen-model check.
CHAIN_MAX_BATCH = 16          # models.CHAIN_CNN_MAX_BATCH, model.cu kChainMaxBatch
PACKED_MIN_TILES = 64         # models.PACKED_CONV_MIN_TILES, model.cu kPackedMinTiles
# Crossovers are searched up to this batch size.
MAX_SEARCH_B = 4096

SETS = {
    # the default network (S = 256, 16 x 16 x 8 grid): every B from 1 to 40 and around each crossover
    "default": dict(M.DEFAULT_PARAMS),
    # the pyramid's wider prediction layer (n_out 9) and three splat convs
    "pyramid": dict(M.DEFAULT_PARAMS, model_name="HDRNetGaussianPyrNN", net_input_size=128, spatial_bin=16),
    # batch norm folded into the weights; fc3 (64 -> 32) too short for the cluster split-K kernel
    "bn_small": dict(M.DEFAULT_PARAMS, batch_norm=True, net_input_size=64, spatial_bin=8, luma_bins=4),
}
SHORT_LIST = (1, 5, 8, 9, 16, 17)

# bars of test_models.py: test_coefficients_match_oracle, test_coefficients_with_wgmma_convs
BAR_CUDA_CORES = 2e-5
BAR_TENSOR_CORES = 5e-5


# ---- the dispatch rules, restated -----------------------------------------------------------------
class Conv:
    def __init__(self, name, H, cin, cout, stride):
        self.name, self.H, self.cin, self.cout, self.stride, self.k = name, H, cin, cout, stride, 3
        self.K = 9 * cin

    def px(self, B):
        oh = _ceil(self.H, self.stride)
        return B * oh * oh


def network(p, n_out):
    """The layers of the coefficient network as the kernels see them (csrc/cnn.cu coef_plan)."""
    S, sb, gd, cm = p["net_input_size"], p["spatial_bin"], p["luma_bins"], p["channel_multiplier"]
    n_ds = int(np.log2(S // sb))
    splat, cin = [], 3
    for i in range(n_ds):
        splat.append(Conv(f"splat/conv{i + 1}", S >> i, cin, cm * gd << i, 2))
        cin = cm * gd << i
    c8 = 8 * cm * gd
    g1 = (sb + 1) // 2
    g2 = (g1 + 1) // 2
    return dict(splat=splat,
                glob=[Conv("global/conv1", sb, cin, c8, 2), Conv("global/conv2", g1, c8, c8, 2)],
                loc=[Conv("local/conv1", sb, cin, c8, 1), Conv("local/conv2", sb, c8, c8, 1)],
                fc=[g2 * g2 * c8, 32 * cm * gd, 16 * cm * gd, c8],
                fuse=(c8, gd * n_out * 4))


def _ceil(a, b):
    return -(-a // b)


def _tiles128(px):
    return _ceil(px, 128)


def _tc_shape_ok(cin, cout):                     # conv_wgmma.cu tc_shape_ok
    return cin % 4 == 0 and cout % 16 == 0 and 16 <= cout <= 256


def _packable(c):                                # models.pack_conv_weights, model.cu packed[]
    return _tc_shape_ok(c.cin, c.cout) and c.cout <= 128


def _patch_k4(K):
    return (K + 3) // 4 * 4


def _patch_slices(K):
    return 1 if _patch_k4(K) <= 64 else 4


def _patch_smem(K, groups):
    q = _patch_k4(K) // 4
    row = (q if q & 1 else q + 1) * 4
    return (32 * row + _patch_k4(K) * 4 * groups + (_patch_slices(K) - 1) * groups * 32 * 4) * 4


def _patch_ok(c):
    return c.cout % 4 == 0 and _patch_smem(c.K, 1) <= 200 * 1024


def _two_groups(ctas1, cout, K, sms):
    return ctas1 > sms and cout % 8 == 0 and _patch_smem(K, 2) <= 200 * 1024


def conv_dispatch(c, B, sms):
    """cnn.cu conv_dispatch -> kernel names, one per launch."""
    px = c.px(B)
    if _tiles128(px) >= 96 and _tc_shape_ok(c.cin, c.cout):
        return [f"conv2d_wgmma_kernel<{min(128, c.cout - n0)},false>" for n0 in range(0, c.cout, 128)]
    if _patch_ok(c):
        ctas1 = _ceil(px, 32) * (c.cout // 4)
        two = _two_groups(ctas1, c.cout, c.K, sms)
        if (ctas1 // 2 if two else ctas1) <= 32 * sms:
            return [f"conv2d_patch_kernel<{2 if two else 1},{_patch_slices(c.K)}>"]
    big = _ceil(px, 64) * _ceil(c.cout, 32)
    return ["conv2d_nhwc_kernel<2,8>" if big >= 2 * sms else "conv2d_nhwc_kernel<1,4>"]


def conv_dispatch_pair(a, b, B, sms):
    """cnn.cu conv_dispatch_pair: the kernel that runs the local (a) and the global (b) branch in one
    launch when both are small, else None (each then goes through conv_dispatch)."""
    def small(c):
        return _tiles128(c.px(B)) < 96 and _patch_ok(c)
    if a.cout == b.cout and small(a) and small(b) and _patch_slices(a.K) == _patch_slices(b.K):
        ctas1 = (_ceil(a.px(B), 32) + _ceil(b.px(B), 32)) * (a.cout // 4)
        two = _two_groups(ctas1, a.cout, max(a.K, b.K), sms)
        return f"conv2d_patch_kernel<{2 if two else 1},{_patch_slices(a.K)}>"
    return None


def python_conv(c, B, sms):
    """models._conv: the packed tensor-core form from PACKED_MIN_TILES tiles, else conv_dispatch."""
    if _packable(c) and _tiles128(c.px(B)) >= PACKED_MIN_TILES:
        return [f"conv2d_wgmma_kernel<{c.cout},true>"]
    return conv_dispatch(c, B, sms)


def fc_kernel(I, O):
    """cnn.cu hdrnet_fc_f32: split-K over a cluster when K is worth splitting, else the plain kernel."""
    ks = 1
    while ks < 8 and I // (ks * 2) >= 64:
        ks *= 2
    return "fc_cluster_kernel" if O % 4 == 0 and ks >= 2 and _ceil(I, ks) <= 256 else "fc_kernel"


def fc_chain_ok(B, n):
    """cnn.cu fc_chain_ok and launch_fc_chain's shared-memory bound."""
    if not 1 <= B <= 4 or any(v < 32 or v & (v - 1) for v in n) or max(n[1:]) > 1024 or n[0] // 8 > 1024:
        return False
    smem = (4 * max(v // 8 for v in n[:3]) + 2 * 4 * max(n[1:]) + 256 * 4 * 4) * 4
    return smem <= 200 * 1024


def plan(net, B, sms):
    """[(layer, kernel)] in launch order for `_coefficients` on B images."""
    out = []

    def add(layer, names):
        out.extend((layer, k) for k in names)

    fcs = list(zip(("global/fc1", "global/fc2", "global/fc3"), net["fc"][:3], net["fc"][1:]))
    if B <= CHAIN_MAX_BATCH:     # hdrnet_coefficients_f32: the launch chain
        for c in net["splat"]:
            add(c.name, conv_dispatch(c, B, sms))
        for (lc, gc) in zip(net["loc"], net["glob"]):
            pair = conv_dispatch_pair(lc, gc, B, sms)
            if pair:
                add(f"{lc.name}+{gc.name}", [pair])
            else:
                add(lc.name, conv_dispatch(lc, B, sms))
                add(gc.name, conv_dispatch(gc, B, sms))
        if fc_chain_ok(B, net["fc"]):
            add("global/fc1-fc3", ["fc_chain_kernel"])
        else:
            for name, I, O in fcs:
                add(name, [fc_kernel(I, O)])
    else:                        # _coefficients_layers
        for c in net["splat"] + net["glob"]:
            add(c.name, python_conv(c, B, sms))
        for name, I, O in fcs:
            add(name, [fc_kernel(I, O)])
        for c in net["loc"]:
            add(c.name, python_conv(c, B, sms))
    add("fusion+prediction", ["fuse_predict_kernel"])
    return out


def crossovers(net, sms):
    """The batch sizes B (2 <= B <= MAX_SEARCH_B) whose plan differs from B - 1's."""
    prev, found = plan(net, 1, sms), []
    for B in range(2, MAX_SEARCH_B + 1):
        cur = plan(net, B, sms)
        if cur != prev:
            found.append(B)
        prev = cur
    return found


def packed_crossovers(net, sms):
    """Crossovers where the set of layers on the packed tensor-core form changes."""
    def packed(B):
        return {layer for layer, k in plan(net, B, sms) if k.endswith(",true>")}
    return [B for B in crossovers(net, sms) if packed(B) != packed(B - 1)]


def sweep(name, cross):
    near = {b + d for b in cross for d in (-1, 0, 1) if b + d >= 1}
    base = set(range(1, 41)) if name == "default" else set(SHORT_LIST)
    return sorted(base | near)


def test_restatement_on_the_default_network():
    """The crossovers the reading of the rules gives for the default network on a 132-SM H100: the
    splat convs change form at 2, 3, 9 and 12, the fc layers leave the fc chain at 5, the network
    goes layer by layer at 17, and the packed form takes splat conv4 and the local convs at 32,
    global conv1 at 127 and global conv2 at 505.  The thresholds in csrc/cnn.cu scale with the SM
    count: with an H100 PCIe's 114 SMs splat conv1 changes at 8, not 9, and splat conv4 never runs
    one channel group."""
    net = network(SETS["default"], 3)
    assert crossovers(net, 132) == [2, 3, 5, 9, 12, 17, 32, 127, 505]
    assert packed_crossovers(net, 132) == [17, 32, 127, 505]
    assert crossovers(net, 114) == [3, 5, 8, 12, 17, 32, 127, 505]


# ---- running it ---------------------------------------------------------------------------------
def _kernel_name(raw):
    """'void hdrnet_b200::conv2d_patch_kernel<2, 4>(hdrnet_b200::ConvArgs, ...)' -> 'conv2d_patch_kernel<2,4>'."""
    name = raw.replace("(anonymous namespace)::", "")
    name = name[5:] if name.startswith("void ") else name
    depth = 0
    for i, ch in enumerate(name):
        depth += ch == "<"
        depth -= ch == ">"
        if ch == "(" and depth == 0:
            name = name[:i]
            break
    name = re.sub(r"\s+", "", name)
    head, sep, tail = name.partition("<")
    return head.rsplit("::", 1)[-1] + sep + tail


def _launched(fn):
    """Names of the CUDA kernels `fn` launches, in launch order (torch.profiler, CUDA activity only)."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
          and not e.name.startswith(("Memcpy", "Memset"))]
    return [_kernel_name(e.name) for e in sorted(ev, key=lambda e: e.time_range.start)]


def _census_child(name, sizes):
    """{B: kernel names} of `_coefficients` on B images (run in a spawned process).  The kernels
    depend on the shapes only, so the input is zeros."""
    p = SETS[name]
    cls = getattr(models, p["model_name"])
    params = dict(p, weights=M.make_weights(p, seed=3))
    S = p["net_input_size"]
    low = torch.zeros((max(sizes), S, S, 3), device="cuda")
    with torch.no_grad():
        cls._coefficients(low[:1], params)      # prepared weights (and their packing) first
        return {B: _launched(lambda: cls._coefficients(low[:B], params)) for B in sizes}


class Case:
    def __init__(self, name):
        self.name = name
        self.p = SETS[name]
        self.cls = getattr(models, self.p["model_name"])
        self.sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
        self.net = network(self.p, self.cls.n_out())
        self.cross = crossovers(self.net, self.sms)
        self.sizes = sweep(name, self.cross)
        self.wts = M.make_weights(self.p, seed=3)
        self.params = dict(self.p, weights=self.wts)
        S, n = self.p["net_input_size"], max(self.sizes)
        self.low = torch.from_numpy(np.random.RandomState(4).rand(n, S, S, 3).astype(np.float32)).cuda()
        # float64 network once per image, in chunks (bounds its float64 im2col); every B a prefix
        lo = self.low.cpu().numpy()
        ref = [M.coefficients(lo[i:i + 32], self.wts, self.p, n_out=self.cls.n_out()) for i in range(0, n, 32)]
        self.ref = torch.from_numpy(np.concatenate(ref)).cuda()
        self.ref_scale = self.ref.abs().flatten(1).amax(1)
        with mp.get_context("spawn").Pool(1) as pool:
            launched = pool.apply(_census_child, (name, self.sizes))
        self.census = {B: self._layers(B, launched[B]) for B in self.sizes}

    def coefficients(self, B):
        with torch.no_grad():
            return self.cls._coefficients(self.low[:B], self.params)

    def _layers(self, B, names):
        """Launch order maps each kernel to its layer; a count mismatch keeps the raw list for the report."""
        want = plan(self.net, B, self.sms)
        if len(names) != len(want):
            return tuple(("?", k) for k in names)
        return tuple((layer, k) for (layer, _), k in zip(want, names))


@pytest.fixture(scope="module", params=list(SETS))
def case(request):
    return Case(request.param)


def _tensor_cores(census):
    return any("wgmma" in k for _, k in census)


@pytest.mark.gpu
def test_census_matches_the_dispatch_rules(case):
    print(f"\n[{case.name}] {case.sms} SMs; crossovers {case.cross}; swept {case.sizes}")
    prev = None
    for B in case.sizes:
        got = case.census[B]
        if got != prev:
            print(f"  B={B}: " + "  ".join(f"{layer}:{k}" for layer, k in got))
        prev = got
    for B in case.sizes:
        want = tuple(plan(case.net, B, case.sms))
        assert case.census[B] == want, (f"{case.name} B={B}: launched {[k for _, k in case.census[B]]}, "
                                        f"the dispatch rules give {[k for _, k in want]}")
    predicted = {k for B in range(1, max(case.sizes) + 1) for _, k in plan(case.net, B, case.sms)}
    seen = {k for c in case.census.values() for _, k in c}
    assert predicted <= seen, f"{case.name}: kernels never launched: {sorted(predicted - seen)}"
    # the sequence changes exactly at the crossovers, wherever the sweep has both B - 1 and B
    changes = [B for B in case.sizes if B - 1 in case.census and case.census[B] != case.census[B - 1]]
    assert changes == [B for B in case.cross if B - 1 in case.census]


@pytest.mark.gpu
def test_coefficients_against_float64_at_every_batch_size(case):
    results, worst, over = {}, {}, []
    for B in sorted(case.sizes, reverse=True):
        got = case.coefficients(B)
        assert got.shape == case.ref[:B].shape
        assert bool(torch.isfinite(got).all()), f"{case.name} B={B}: non-finite coefficients"
        err = (got.double() - case.ref[:B]).abs().flatten(1).amax(1) / case.ref_scale[:B]
        bar = BAR_TENSOR_CORES if _tensor_cores(case.census[B]) else BAR_CUDA_CORES
        worst[B] = float(err.max())
        over += [f"B={B} image {i}: {float(err[i]):.2e} > {bar:.0e}"
                 for i in torch.nonzero(err > bar).flatten().tolist()]
        results[B] = got
    groups = {}
    for B in case.sizes:
        groups.setdefault(case.census[B], []).append(B)
    print(f"\n[{case.name}] worst per-image error against float64, by kernel sequence:")
    for census, sizes in groups.items():
        print(f"  B {sizes}: {max(worst[B] for B in sizes):.2e}  ({' '.join(k for _, k in census)})")
    assert not over, f"{case.name}: {len(over)} images off the float64 network: " + "; ".join(over[:12])
    # ascending, each call after a smaller one, as descending, each after a larger one
    for B in sorted(case.sizes):
        assert torch.equal(case.coefficients(B), results[B]), f"{case.name} B={B}: ascending != descending"
    # the same kernel for every layer: every image's coefficients bit for bit the same
    for sizes in groups.values():
        top = max(sizes)
        for B in sizes:
            same = (results[B] == results[top][:B]).flatten(1).all(1)
            bad = [i for i in range(B) if not bool(same[i])]
            assert not bad, (f"{case.name}: B={B} and B={top} launch the same kernels, but images {bad[:8]} "
                             f"differ between them")


@pytest.mark.gpu
def test_frozen_model_on_both_sides_of_the_repeated_constants(tmp_path):
    """csrc/model.cu repeats CHAIN_CNN_MAX_BATCH and PACKED_CONV_MIN_TILES: the frozen model must
    equal the Python path bitwise at B - 1 and B of each crossover of either, for stacked and for
    ragged batches."""
    p = SETS["default"]
    cls = models.HDRNetCurves
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    sizes = sorted({CHAIN_MAX_BATCH, CHAIN_MAX_BATCH + 1} |
                   {b + d for b in packed_crossovers(network(p, 3), sms) for d in (-1, 0)})
    wts = M.make_weights(p, seed=3)
    params = dict(p, weights=wts)
    path = tmp_path / "default.hdrnet"
    checkpoint.freeze_model(wts, params, str(path))
    shapes = [(64, 96), (96, 64), (48, 80)]
    g = torch.Generator(device="cuda").manual_seed(7)
    with FrozenModel(str(path)) as model, torch.no_grad():
        for B in sizes:
            img = torch.randint(0, 256, (B, 64, 96, 3), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
            got, want = model(img), cls.inference_image(img, params)
            assert torch.equal(got, want), (f"frozen B={B}: {int((got != want).any(-1).flatten(1).any(1).sum())} "
                                            f"of {B} images differ from inference_image")
            ims = [torch.randint(0, 256, shapes[i % 3] + (3,), generator=g, device="cuda",
                                 dtype=torch.int32).to(torch.uint8) for i in range(B)]
            got, want = model(ims), cls.inference_images(ims, params)
            bad = [i for i in range(B) if not torch.equal(got[i], want[i])]
            assert not bad, f"frozen ragged B={B}: images {bad[:8]} differ from inference_images"
