"""The per-tap convolution's wide tiles (conv_tc.cu, conv_wide_kernel) against its 128 x 128 tile (conv_tc_kernel).

Both accumulate every output element's terms in the same (tap, slab, k16) order, so the fp16 outputs are equal bit
for bit; the GPU tests compare them with torch.equal at the shapes the UNets run them at and at edge cases of the
wide tiles' grid. The CPU tests pin the tile v2e_conv_pick_tile chooses per layer and read the compiled kernels'
SASS (asynchronous wgmma chains, no local-memory spills)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from v2e_b200 import _lib
from v2e_b200 import build as _build

LEGACY, T256x128, T128x256 = 0, 1, 2
AUTO = -1

# (name, cin1, cin2, cout, level) of the layers that run on the per-tap kernel at 1280 px. UNet(12, 5) and UNet(2, 4)
# differ only in their first and last layers (strip kernel), so both networks run these shapes.
TAP_LAYERS = [("down2.c1", 64, 0, 128, 2), ("down2.c2", 128, 0, 128, 2),
              ("down3.c1", 128, 0, 256, 3), ("down3.c2", 256, 0, 256, 3),
              ("down4.c1", 256, 0, 512, 4), ("down4.c2", 512, 0, 512, 4),
              ("down5.c1", 512, 0, 512, 5), ("down5.c2", 512, 0, 512, 5),
              ("up1.c1", 512, 0, 512, 4), ("up1.c2", 512, 512, 512, 4),
              ("up2.c1", 512, 0, 256, 3), ("up2.c2", 256, 256, 256, 3),
              ("up3.c1", 256, 0, 128, 2), ("up3.c2", 128, 128, 128, 2)]

# the headline (1280x720 -> 1280x704 network input, batch 8) and the 346x260 secondary (320x256, all 30 pairs)
SIZES = {"1280": (8, 704, 1280), "320": (30, 256, 320)}


def wide_tile(cout):
    return T256x128 if cout == 128 else T128x256


def plan(size, n_sms=132):
    lib = _lib.load()
    N, H, W = SIZES[size]
    return {name: lib.v2e_conv_pick_tile(c1, c2, co, 3, 3, N, H >> lvl, W >> lvl, n_sms)
            for name, c1, c2, co, lvl in TAP_LAYERS}


def test_tile_plan_at_1280():
    # down5 at 40x22 x 8 images: 288 CTAs of 128 x 128 (3 waves on 132 SMs) or 144 of 128 x 256 (2 waves of 1.5x the
    # bytes per stage): a tie, which goes to the narrow tile
    assert plan("1280") == {"down2.c1": T256x128, "down2.c2": T256x128, "down3.c1": T128x256, "down3.c2": T128x256,
                            "down4.c1": T128x256, "down4.c2": T128x256, "down5.c1": LEGACY, "down5.c2": LEGACY,
                            "up1.c1": T128x256, "up1.c2": T128x256, "up2.c1": T128x256, "up2.c2": T128x256,
                            "up3.c1": T256x128, "up3.c2": T256x128}


def test_tile_plan_at_320():
    # down5 at 10x8 x 30 images: 120 CTAs of 128 x 128 or 60 of 128 x 256, one wave either way
    assert plan("320") == {"down2.c1": T256x128, "down2.c2": T256x128, "down3.c1": T128x256, "down3.c2": T128x256,
                           "down4.c1": T128x256, "down4.c2": T128x256, "down5.c1": LEGACY, "down5.c2": LEGACY,
                           "up1.c1": T128x256, "up1.c2": T128x256, "up2.c1": T128x256, "up2.c2": T128x256,
                           "up3.c1": T256x128, "up3.c2": T256x128}


def test_narrow_or_small_layers_keep_the_legacy_tile():
    lib = _lib.load()
    assert lib.v2e_conv_pick_tile(64, 0, 64, 3, 3, 8, 352, 640, 132) == LEGACY      # Cout_pad 64
    assert lib.v2e_conv_pick_tile(32, 0, 128, 3, 3, 8, 176, 320, 132) == LEGACY     # 32-channel slabs
    assert lib.v2e_conv_pick_tile(512, 0, 512, 3, 3, 1, 8, 10, 132) == LEGACY       # one wave either way


# ---- SASS of the built library (no GPU) -------------------------------------------------------------------------
def _wide_sass():
    lib = _build.build()
    nvcc = _build._nvcc()
    cand = os.path.join(os.path.dirname(nvcc), "cuobjdump") if os.path.isabs(nvcc) else None
    tool = cand if cand and os.path.exists(cand) else shutil.which("cuobjdump")
    if tool is None:
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([tool, "-sass", lib], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if "conv_wide_kernel" in m.group(1) else None
            if cur:
                funcs[cur] = {"hgmma": 0, "depbar": 0, "local": 0}
            continue
        if cur:
            if "HGMMA" in line:
                funcs[cur]["hgmma"] += 1
            elif "WARPGROUP.DEPBAR" in line:
                funcs[cur]["depbar"] += 1
            elif re.search(r"\b(STL|LDL)(\.\S+)?\s", line):
                funcs[cur]["local"] += 1
    return funcs


def test_both_wide_kernels_chain_their_wgmmas_and_do_not_spill():
    funcs = _wide_sass()
    assert len(funcs) == 2, sorted(funcs)          # 256x128, 128x256
    bad = {k: v for k, v in funcs.items() if v["depbar"] >= v["hgmma"] or v["local"]}
    assert not bad, "serialised wgmma chains or local-memory spills: %r" % bad


# ---- GPU: wide tiles equal the 128 x 128 tile bit for bit ---------------------------------------------------------
def _run(case, tiles, seed):
    """One random layer (N, H, W, C1, C2, Cout) through each tile of `tiles`; the fp16 outputs."""
    import torch
    N, H, W, C1, C2, Cout = case
    L = _lib.load()
    g = torch.Generator(device="cuda:0").manual_seed(seed)
    x1 = torch.randn((N, H, W, C1), generator=g, device="cuda:0").half()
    x2 = torch.randn((N, H, W, C2), generator=g, device="cuda:0").half() if C2 else None
    K = 9 * (C1 + C2)
    w = (torch.randn((Cout, K), generator=g, device="cuda:0") / K ** 0.5).half()
    b = torch.randn((Cout,), generator=g, device="cuda:0") * 0.1
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    outs = []
    for tile in tiles:
        out = torch.full((N, H, W, Cout), float("nan"), dtype=torch.float16, device="cuda:0")
        _lib.check(L.v2e_conv2d_lrelu_sm100_tile(p(x1), C1, p(x2), C2, p(w), p(b), Cout, 3, 3, N, H, W, p(out), Cout,
                                                 0, Cout, ctypes.c_float(0.1), tile, st))
        outs.append(out)
    torch.cuda.synchronize()
    return outs


def _assert_all_equal(case, tiles, seed=0):
    import torch
    outs = _run(case, tiles, seed)
    assert not torch.isnan(outs[0]).any()
    for tile, o in zip(tiles[1:], outs[1:]):
        assert torch.equal(o, outs[0]), "tile %d differs from the 128 x 128 tile at %r" % (tile, case)


@pytest.mark.gpu
@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("layer", TAP_LAYERS, ids=[l[0] for l in TAP_LAYERS])
def test_wide_tiles_equal_the_legacy_tile_at_production_shapes(layer, size):
    name, c1, c2, co, lvl = layer
    N, H, W = SIZES[size]
    case = (N, H >> lvl, W >> lvl, c1, c2, co)
    wt = wide_tile(co)
    _assert_all_equal(case, [LEGACY, wt, AUTO], seed=lvl * 131 + co + c2)


EDGE_CASES = [
    # N, H, W, C1, C2, Cout
    (1, 24, 48, 256, 0, 256),        # 3 x 3 = 9 tiles of 8x16, one output-channel block
    (1, 40, 48, 128, 0, 128),        # 3 x 3 = 9 tiles of 16x16 (H not a multiple of 16), one output-channel block
    (3, 36, 36, 64, 64, 128),        # concatenated inputs, 16x16 tiles cut at both edges, 3 x 9 tiles
    (1, 9, 23, 256, 256, 512),       # concatenated inputs, 8x16 tiles cut at both edges, two channel blocks
    (1, 16, 32, 512, 0, 512),        # one wave: 2 tiles x 2 channel blocks
    (1, 8, 16, 128, 0, 256),         # a single tile
    (2, 5, 7, 64, 0, 128),           # smaller than one tile
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", EDGE_CASES)
def test_wide_tiles_equal_the_legacy_tile_at_edge_cases(case):
    _assert_all_equal(case, [LEGACY, wide_tile(case[5])])


@pytest.mark.gpu
def test_128x256_tile_at_cout_128_is_refused_and_256x128_runs_at_cout_512():
    """Cout_pad must be a multiple of the tile width; the 16x16 tile also runs where the pick does not choose it."""
    with pytest.raises(Exception):
        _run((1, 8, 16, 64, 0, 128), [T128x256], 0)
    _assert_all_equal((2, 44, 80, 256, 0, 512), [LEGACY, T256x128])
