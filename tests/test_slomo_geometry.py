"""The SloMo engine against float64 at the frame sizes, batch sizes and SM counts that real videos reach.

The source size, the batch and the device's SM count decide which kernel runs each layer (strip, pooled strip, fused
up-sampling or per-tap: v2e_conv_strip_pick_kc, v2e_conv_up2_supported_c), which tile a per-tap layer gets
(v2e_conv_pick_tile) and how strips are cut into items (seg_h of v2e_strip_prepare / v2e_conv_up2_prepare). The
geometries below reach partial column strips, odd and 1-row last segments, odd deepest levels, strip layers a few
rows high, 1x1 pools and the resize copy path; tests/test_slomo_layers.py covers the production shapes. The checks and
bars are tests/slomo_checks.py's.

Bit-for-bit invariances: every output element of a convolution is summed in an order fixed by the layer, whatever
the tile, segment or grid (DESIGN.md 4.2), and the pools and up-samplings are order-exact, so an image's result does
not depend on its batch, on the engine's max_batch, or on the SM count the launches are planned for
(v2e_slomo_set_option(h, 3, n)).

CPU tests pin, through the host pick functions, that the sweep covers what it claims."""
import ctypes

import numpy as np
import pytest
import torch

import slomo_ref
from helpers import err_ratio, ulp32
from slomo_checks import (DEV, KMEAN, NAMES, check_every_layer, crafted_flows, layer_ratio, make_weights,
                          post_interp_reference, pre_interp_bar, pre_interp_reference, snapshot, textured,
                          warp_engine)
from test_layer_plan import LAYERS, cout_pad, pad16
from v2e_b200 import _lib

T256x128 = 1                         # v2e_conv_pick_tile: the 16 x 16-pixel tile
ROW_TILE = 128                       # columns of a strip (conv_tc.cu kRowTile)

# non-tap layers of the plan (index: kernel); the rest run on the per-tap kernel
WIDE = {0: "strip", 1: "strip_pool", 2: "strip", 3: "strip_pool", 18: "strip", 19: "strip", 20: "up2", 21: "strip",
        22: "strip"}                                   # network width >= 512: strips at levels 0 and 1, fused up5.conv1
NARROW = {0: "strip", 1: "strip_pool", 20: "strip", 21: "strip", 22: "strip"}   # 256 <= width < 512: level 0 only
TAP = {}

# source frame size, batch, the engine's plan
CONFIGS = {
    # 1920x1056: 7.5 strips at half resolution, up5.conv1 fused over 7.5 low strips, deepest level 33x60, LANCZOS
    # vertical pass only; batch 4: up4.conv2's last segment is 1 row; batch 1: conv1 in segments of 17 rows
    "1920x1080_b4": ((1920, 1080), 4, WIDE),
    "1920x1080_b1": ((1920, 1080), 1, WIDE),
    # 832x480: 6.5 and 3.25 strips, fused up-sampling over 3.25 low strips, deepest level 15x26, horizontal pass only
    "854x480_b3": ((854, 480), 3, WIDE),
    # just above the fused up-sampling threshold (a 16-px last low strip); pooled down1.conv2 on 2.125 strips
    "544x416_b2": ((544, 416), 2, WIDE),
    # the narrowest strip layers (2.25 strips), deepest level 7x9
    "288x224_b2": ((288, 224), 2, NARROW),
    # strip and fused up-sampling layers 32 / 16 rows high, deepest level 1x32
    "1024x32_b2": ((1024, 32), 2, WIDE),
    # DAVIS240 (224x160 network): all per-tap, LANCZOS in both passes, deepest level 5x7
    "240x180_b5": ((240, 180), 5, TAP),
    # the smallest accepted frame: pools to 1x1, up-sampling from 1x1, the resize copy path
    "32x32_b1": ((32, 32), 1, TAP),
}


def net_size(src):
    return src[0] // 32 * 32, src[1] // 32 * 32


def full_plan(nontap):
    return [nontap.get(i, "tap") for i in range(23)]


def layer_level(li):
    if li < 2 or li == 22:
        return 0
    return (li - 2) // 2 + 1 if li < 12 else 4 - (li - 12) // 2


# ---- the host's picks (no GPU) ---------------------------------------------------------------------------------------
def host_plan(W, H):
    """Per layer "strip", "up2" or "tap" from the host pick functions (the pooled epilogue is not exported: the GPU
    tests read it from the engine)."""
    lib = _lib.load()
    out = []
    for li, (name, c1, c2, co, k, lvl) in enumerate(LAYERS):
        c1p, c2p, cp = pad16(c1), pad16(c2) if c2 else 0, cout_pad(co)
        if 12 <= li < 22 and li % 2 == 0 and lib.v2e_conv_up2_supported_c(c1p, cp, W >> lvl):
            out.append("up2")
        else:
            out.append("strip" if lib.v2e_conv_strip_pick_kc(c1p, c2p, cp, k, k, W >> lvl) else "tap")
    return out


def tap_tiles(W, H, B, n_sms):
    """{layer: tile} of the per-tap layers at network size W x H, batch B, planned for n_sms SMs."""
    lib = _lib.load()
    plan = host_plan(W, H)
    return {name: lib.v2e_conv_pick_tile(pad16(c1), pad16(c2) if c2 else 0, cout_pad(co), k, k, B, H >> lvl, W >> lvl,
                                         n_sms)
            for li, (name, c1, c2, co, k, lvl) in enumerate(LAYERS) if plan[li] == "tap"}


def strip_seg_h(h, w, KH, B, n_sms, pool):
    """Rows per item of a strip layer (v2e_strip_prepare): halved from h while there are fewer than 6 items per SM
    and more than 4 KH rows, even when the pool rides in the epilogue."""
    strips = -(-w // ROW_TILE) * B
    s = h
    while s > 4 * KH and strips * -(-h // s) < 6 * n_sms:
        s = (s + 1) // 2
    return (s + 1) & ~1 if pool else s


def up2_seg_h(hl, wl, B, n_sms):
    """Low-resolution rows per item of the fused up-sampling (v2e_conv_up2_prepare)."""
    strips = -(-wl // ROW_TILE) * B
    n_seg = max(1, -(-6 * n_sms // strips))
    s = -(-hl // n_seg)
    return s if s >= 8 else min(hl, 8)


@pytest.mark.parametrize("config", list(CONFIGS))
def test_host_plan_of_each_geometry(config):
    src, B, nontap = CONFIGS[config]
    W, H = net_size(src)
    assert host_plan(W, H) == [p.replace("strip_pool", "strip") for p in full_plan(nontap)]


def test_sweep_reaches_partial_strips_and_short_segments():
    """Strip layers whose width is not a multiple of 128 at levels 0 and 1, a fused up-sampling whose low-resolution
    width is not, a segment of an odd number of rows and a 1-row last segment (planned for 132 SMs)."""
    partial = {0: set(), 1: set()}
    up2_partial, odd_seg, one_row = set(), set(), set()
    for config, (src, B, nontap) in CONFIGS.items():
        W, H = net_size(src)
        for li, p in enumerate(full_plan(nontap)):
            lvl = layer_level(li)
            if p.startswith("strip"):
                w, h = W >> lvl, H >> lvl
                if w % ROW_TILE:
                    partial[lvl].add(config)
                s = strip_seg_h(h, w, LAYERS[li][4], B, 132, p == "strip_pool")
                if s % 2:
                    odd_seg.add(config)
                if h % s == 1:
                    one_row.add(config)
            if p == "up2" and (W // 2) % ROW_TILE:
                up2_partial.add(config)
    assert {"854x480_b3", "544x416_b2", "288x224_b2"} <= partial[0], partial
    assert {"1920x1080_b4", "854x480_b3", "544x416_b2"} <= partial[1], partial
    assert {"1920x1080_b4", "854x480_b3", "544x416_b2"} <= up2_partial, up2_partial
    assert "1920x1080_b1" in odd_seg and "1920x1080_b4" in one_row, (odd_seg, one_row)
    # 544x416: the fused up-sampling's low strips are 272 wide, the last one 16 px
    assert (544 // 2) % ROW_TILE == 16


def test_sweep_reaches_a_256x128_tile_with_a_ragged_height():
    """A per-tap layer on the 256 x 128 tile (16 x 16 pixels) whose height is not a multiple of 16."""
    hits = []
    for config, (src, B, nontap) in CONFIGS.items():
        W, H = net_size(src)
        for name, tile in tap_tiles(W, H, B, 132).items():
            lvl = [l[5] for l in LAYERS if l[0] == name][0]
            if tile == T256x128 and (H >> lvl) % 16:
                hits.append((config, name, H >> lvl))
    assert hits, "no 256x128-tile layer with a ragged height"


def test_plans_of_the_smallest_and_flattest_frames():
    assert host_plan(32, 32) == ["tap"] * 23
    assert host_plan(1024, 32) == [p.replace("strip_pool", "strip") for p in full_plan(WIDE)]
    assert host_plan(224, 160) == ["tap"] * 23


SM_COUNTS = (132, 114, 66, 7, 1)


@pytest.mark.parametrize("src,B", [((346, 260), 3), ((544, 416), 2)])
def test_sm_counts_change_some_tile(src, B):
    """The SM-count invariance test below must move at least one per-tap layer to another tile."""
    W, H = net_size(src)
    picks = [tap_tiles(W, H, B, n) for n in SM_COUNTS]
    assert any(p != picks[0] for p in picks[1:]), picks


# ---- GPU: every layer against float64 --------------------------------------------------------------------------------
def device_sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def ragged_regions(W, H, B, plan, n_sms):
    """regions(li) for check_every_layer: the columns of the last partial strip ("last_strip") and the rows of the
    last segment ("last_segment") of every strip and fused up-sampling layer."""
    def regions(li):
        p, lvl = plan[li], layer_level(li)
        if p == "tap":
            return {}
        w, h = W >> lvl, H >> lvl
        out = {}
        if p == "up2":
            wl, hl = w // 2, h // 2
            s = up2_seg_h(hl, wl, B, n_sms)
            if wl % ROW_TILE:
                out["last_strip"] = (slice(None), slice(2 * (wl // ROW_TILE * ROW_TILE), None))
            out["last_segment"] = (slice(2 * ((hl - 1) // s * s), None), slice(None))
        else:
            s = strip_seg_h(h, w, LAYERS[li][4], B, n_sms, p == "strip_pool")
            if w % ROW_TILE:
                out["last_strip"] = (slice(None), slice(w // ROW_TILE * ROW_TILE, None))
            out["last_segment"] = (slice((h - 1) // s * s, None), slice(None))
        return out
    return regions


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(CONFIGS))
def test_every_layer_matches_float64_at_other_geometries(config):
    """All 23 layers of both networks, every image, every pool and separate up-sampling, within the bars of
    tests/slomo_checks.py; the worst ratio of the last partial strip and of the last segment is reported apart."""
    src, B, nontap = CONFIGS[config]
    snap = snapshot(src, B)
    H, W = snap["hw"]
    assert (W, H) == net_size(src)
    plan = full_plan(nontap)
    assert snap["flow"]["plan"] == plan and snap["interp"]["plan"] == plan, snap["flow"]["plan"]
    worst = check_every_layer(snap, ragged_regions(W, H, B, plan, device_sms()))
    worst.report("%s (network %dx%d, batch %d)" % (config, W, H, B))
    assert not worst.bad(), worst.bad()


@pytest.mark.gpu
@pytest.mark.parametrize("config,li,perturb", [
    ("544x416_b2", 20, dict(drop_channel=5)),
    ("544x416_b2", 20, dict(drop_tap=(0, 2))),
    ("854x480_b3", 0, dict(drop_tap=(6, 6))),
    ("854x480_b3", 19, dict(drop_channel=70)),          # the skip half of a concatenated input
    ("854x480_b3", 1, dict(drop_tap=(3, 0))),
    ("854x480_b3", 3, dict(drop_channel=9)),
])
def test_last_partial_strip_comparison_fails_on_perturbed_reference(config, li, perturb):
    """Restricted to the columns of the last partial strip, the comparison passes against the true reference and fails
    when one tap or one input channel is dropped from it; for the fused up-sampling in the interior and in the frame."""
    src, B, nontap = CONFIGS[config]
    snap = snapshot(src, B)
    net = snap["interp"]
    H, W = snap["hw"]
    assert net["plan"][li] == full_plan(nontap)[li] and net["plan"][li] != "tap"
    w = W >> layer_level(li)
    x0 = 2 * ((w // 2) // ROW_TILE * ROW_TILE) if net["plan"][li] == "up2" else w // ROW_TILE * ROW_TILE
    assert 0 < x0 < w
    b = B - 1
    assert max(layer_ratio(net, li, b, x0=x0).values()) <= 1.0
    bad = layer_ratio(net, li, b, x0=x0, **perturb)
    print("\n%s %s %s, columns >= %d: ratio against the perturbed reference %s" % (config, NAMES[li], perturb, x0, bad))
    assert all(r > 1.0 for r in bad.values()), bad


# ---- GPU: batch and SM-count invariance ------------------------------------------------------------------------------
def run_engine(src, max_batch, frames, n_sms=None):
    """set_pairs + interp(0.3) of frames [B+1, H, W] on a fresh engine: flow_out, intrp_out, float32 Ft and the uint8
    frames, and the plan."""
    from v2e_b200.slomo import SloMoEngine
    sd_fc, sd_at = make_weights(11)
    eng = SloMoEngine(sd_fc, sd_at, src, max_batch, DEV)
    try:
        if n_sms is not None:
            _lib.check(eng.lib.v2e_slomo_set_option(eng._h, 3, n_sms))
        B = frames.shape[0] - 1
        eng.set_pairs(frames)
        flow = eng.flow_out().clone()
        out = torch.empty((B, src[1], src[0]), dtype=torch.uint8, device=DEV)
        ft = torch.empty((B, eng.h, eng.w), dtype=torch.float32, device=DEV)
        eng.interp(0.3, out, ft)
        res = dict(flow=flow, intrp=eng.intrp_out().clone(), ft=ft, u8=out)
        plan = eng.layer_kernels()
        eng.check_finite()
    finally:
        eng.close()
    return res, plan


def assert_image_equal(a, ia, b, ib, what):
    for k in ("flow", "intrp", "ft", "u8"):
        assert torch.equal(a[k][ia], b[k][ib]), "%s: %s of the image differs (%d vs %d differing elements)" % (
            what, k, int((a[k][ia] != b[k][ib]).sum()), a[k][ia].numel())


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["1920x1080_b4", "854x480_b3", "544x416_b2"])
def test_image_result_does_not_depend_on_its_batch(config):
    """Image b's heads, float32 Ft and uint8 frame are identical in a batch of B, in a short batch of fewer pairs on an
    engine sized for 8, and alone on an engine sized for 1 (segmentation and tiles follow the batch)."""
    src, B, _ = CONFIGS[config]
    frames = torch.from_numpy(textured(B + 1, src[1], src[0], 17)).to(DEV)
    full, _ = run_engine(src, B, frames)
    a = max(0, B - 2) if B >= 3 else B - 1
    short, _ = run_engine(src, 8, frames[a:].contiguous())
    for b in range(a, B):
        assert_image_equal(full, b, short, b - a, "%s image %d, short batch of %d" % (config, b, B - a))
    for b in range(B):
        alone, _ = run_engine(src, 1, frames[b:b + 2].contiguous())
        assert_image_equal(full, b, alone, 0, "%s image %d alone" % (config, b))


@pytest.mark.gpu
@pytest.mark.parametrize("src,B", [((346, 260), 3), ((544, 416), 2)])
def test_result_does_not_depend_on_the_sm_count(src, B):
    """Planned for n in {device count, 114, 66, 7, 1} SMs (option 3), the heads and frames are identical; at 1 and 7
    SMs every persistent CTA walks dozens of items."""
    n_dev = device_sms()
    frames = torch.from_numpy(textured(B + 1, src[1], src[0], 23)).to(DEV)
    ref, plan = run_engine(src, B, frames)
    for n in [n_dev] + [n for n in SM_COUNTS[1:] if n < n_dev]:
        got, p = run_engine(src, B, frames, n_sms=n)
        assert p == plan
        for b in range(B):
            assert_image_equal(ref, b, got, b, "%s batch %d planned for %d SMs, image %d" % (src, B, n, b))


@pytest.mark.gpu
def test_sm_count_option_refuses_values_outside_the_device():
    from v2e_b200.slomo import SloMoEngine
    sd_fc, sd_at = make_weights(11)
    eng = SloMoEngine(sd_fc, sd_at, (64, 64), 1, DEV)
    try:
        for bad in (-1, device_sms() + 1):
            assert eng.lib.v2e_slomo_set_option(eng._h, 3, bad) == _lib.V2E_E_INVALID
        for ok in (1, device_sms(), 0):
            _lib.check(eng.lib.v2e_slomo_set_option(eng._h, 3, ok))
    finally:
        eng.close()


# ---- GPU: warps at sizes that are not powers of two -----------------------------------------------------------------
WARP_SIZES = [(320, 256, 2), (832, 480, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("t", [0.5, 0.3])
@pytest.mark.parametrize("size", WARP_SIZES, ids=["%dx%d" % s[:2] for s in WARP_SIZES])
def test_pre_interp_warps_at_other_sizes(size, t):
    """pre_interp_kernel on the crafted flows (samples on -1, 0, n-1, n and fully outside) within 1 fp16 ulp of the
    float32 reference, plus the position allowance on the two warp channels at both t.

    W and H are not powers of two, so grid_sample's float32 round trip x + u, / W, - 0.5, * 2, + 1, * W, - 1, / 2 is
    not exact on either side (at t = 0.5 too): each of its roundings moves the position by at most 2^-24 of a value
    of at most |F| + 2W pixels, and the kernel contracts multiply-adds the reference rounds twice; delta_x = 2^-21 *
    (|F_x| + 2W) bounds the difference, likewise along y. A bilinear sample of values within +-m changes by at most 2m
    per pixel of movement along an axis: bar ulp16 + 2m (delta_x + delta_y) (slomo_checks.position_delta)."""
    W, H, B = size
    eng = warp_engine(W, H, B)
    f, ax, ay = crafted_flows(1, B, H, W)
    eng.flow_out().copy_(f)
    eng.interp(t, torch.empty((B, H, W), dtype=torch.uint8, device=DEV))
    a = eng.activations()
    got = a["in16"].double()
    want = pre_interp_reference(a["img"], eng.flow_out(), t).double()
    bar = pre_interp_bar(want, a["img"], exact_positions=False)
    r = [err_ratio(got[..., c], want[..., c], bar[..., c]) for c in range(12)]
    print("\npre_interp %dx%d t=%.1f: largest |got - ref| / bar per channel %s" % (W, H, t, ["%.3f" % v for v in r]))
    assert max(r) <= 1.0
    assert (a["in16"][..., 12:] == 0).all()
    if t == 0.5:
        out0 = torch.from_numpy((np.abs(ax) > W + 1) | (np.abs(ay) > H + 1)).to(DEV)
        assert out0.any() and (got[..., 11][out0] == 0).all() and (got[..., 10][out0] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("t", [0.5, 0.3])
@pytest.mark.parametrize("size", WARP_SIZES, ids=["%dx%d" % s[:2] for s in WARP_SIZES])
def test_post_interp_blend_at_other_sizes(size, t):
    """post_interp_kernel vs slomo.py:421-437 in float64: 16 float32 ulps of M (test_slomo_layers) plus the position
    allowance 2m * delta of the warps (the blend is a convex combination of the two warps: the larger delta of the
    two). The uint8 frame equals the reference's float32 expression of the kernel's own Ft everywhere, and the
    truncation of the float64 (Ft + 0.428) * 255 wherever that value is farther than 255 bars from an integer (at
    832x480 the allowance is ~0.36 DN, so only part of the frame is decided that way)."""
    W, H, B = size
    eng = warp_engine(W, H, B)
    f, _, _ = crafted_flows(2, B, H, W)
    eng.flow_out().copy_(f)
    out = torch.empty((B, H, W), dtype=torch.uint8, device=DEV)
    ft = torch.empty((B, H, W), dtype=torch.float32, device=DEV)
    eng.interp(t, out, ft)
    img = eng.activations()["img"]
    want, M, delta = post_interp_reference(img, eng.flow_out(), eng.intrp_out(), t)
    bar = 16 * ulp32(M) + 2 * img.abs().max().item() * delta
    r = err_ratio(ft, want, bar)
    print("\npost_interp %dx%d t=%.1f: largest |got - ref| / bar = %.4f" % (W, H, t, r))
    assert r <= 1.0
    s = (want + KMEAN) * 255.0
    ok = (s - torch.round(s)).abs() > 255.0 * bar          # truncation decided by the float64 value
    assert ok.any()
    assert torch.equal(out.long()[ok], (torch.trunc(s).long() & 255)[ok])
    assert torch.equal(out.cpu(), slomo_ref.to_u8(ft.cpu()))


@pytest.mark.gpu
def test_max_speed_at_1920x1056_last_pixel():
    """max_speed_kernel over a 1920x1056 batch of 1 (2 M pixels, a grid-stride loop of several rounds) finds the
    maximum planted at the batch's last pixel exactly."""
    from v2e_b200.slomo import SloMoEngine
    sd_fc, sd_at = make_weights(21)
    eng = SloMoEngine(sd_fc, sd_at, (1920, 1056), 1, DEV)
    try:
        eng.set_pairs(torch.from_numpy(textured(2, 1056, 1920, 5)).to(DEV))
        rng = np.random.default_rng(4)
        f = torch.from_numpy(rng.uniform(-3, 3, (1, 1056, 1920, 8)).astype(np.float32)).to(DEV)
        f[..., 4:] = 0
        f[-1, -1, -1, 2:4] = torch.tensor([-30.0, 40.0])
        eng.flow_out().copy_(f)
        assert eng.max_flow() == 50.0
    finally:
        eng.close()


# ---- GPU: resizes against Pillow -------------------------------------------------------------------------------------
RESIZE_SOURCES = [src for src, _, _ in CONFIGS.values()] + [(33, 47)]


def _resizer(sw, sh, dw, dh, filt, n):
    L = _lib.load()
    r = ctypes.c_void_p()
    _lib.check(L.v2e_resize_create(sw, sh, dw, dh, filt, n, ctypes.byref(r)))
    return L, r


def _images(n, h, w, seed):
    rng = np.random.default_rng(seed)
    imgs = rng.integers(0, 256, (n, h, w), dtype=np.uint8)
    imgs[1] = np.kron(rng.integers(0, 256, (h // 4 + 1, w // 4 + 1), dtype=np.uint8), np.ones((4, 4), np.uint8))[:h, :w]
    return imgs


def _pillow(img, size, filt):
    from PIL import Image
    return np.asarray(Image.fromarray(img).resize(size, Image.LANCZOS if filt else Image.BILINEAR))


@pytest.mark.gpu
@pytest.mark.parametrize("src", sorted(set(RESIZE_SOURCES)), ids=lambda s: "%dx%d" % s)
def test_resizes_are_pillow_exact_at_every_source_size(src):
    """LANCZOS down to the network size (33x47 shrinks to 32x32) and BILINEAR back, bit for bit with Pillow; where
    a size does not change, Pillow skips that pass (32x32 is a plain copy)."""
    sw, sh = src
    dw, dh = max(32, sw // 32 * 32), max(32, sh // 32 * 32)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for (aw, ah), (bw, bh), filt in (((sw, sh), (dw, dh), 1), ((dw, dh), (sw, sh), 0)):
        imgs = _images(3, ah, aw, aw * 7 + bh)
        L, r = _resizer(aw, ah, bw, bh, filt, 3)
        try:
            s = torch.from_numpy(imgs).to(DEV)
            d = torch.zeros((3, bh, bw), dtype=torch.uint8, device=DEV)
            _lib.check(L.v2e_resize_run(r, ctypes.c_void_p(s.data_ptr()), ctypes.c_void_p(d.data_ptr()), 3, st))
            got = d.cpu().numpy()
        finally:
            L.v2e_resize_destroy(r)
        for i in range(3):
            want = _pillow(imgs[i], (bw, bh), filt)
            assert np.array_equal(got[i], want), "%s -> %s image %d: %d pixels differ" % (
                (aw, ah), (bw, bh), i, int((got[i] != want).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("src", [(1920, 1080), (854, 480), (240, 180), (32, 32)], ids=lambda s: "%dx%d" % s)
def test_strided_resize_leaves_the_other_frames_untouched(src):
    """v2e_resize_run_strided into the U-interleaved clip interp writes (frame of pair b at step k at index U*b + k):
    the B frames of step k equal Pillow's BILINEAR up-resize, every other byte of the sentinel-filled clip is
    unchanged (vertical pass only, horizontal pass, both passes, and the copy path)."""
    sw, sh = src
    nw, nh = sw // 32 * 32, sh // 32 * 32
    B, U, k = 3, 4, 2
    imgs = _images(B, nh, nw, sw + sh)
    L, r = _resizer(nw, nh, sw, sh, 0, B)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    try:
        clip = torch.full((B * U, sh, sw), 0xA5, dtype=torch.uint8, device=DEV)
        s = torch.from_numpy(imgs).to(DEV)
        blk = clip[k:U * B:U]
        _lib.check(L.v2e_resize_run_strided(r, ctypes.c_void_p(s.data_ptr()), ctypes.c_void_p(blk.data_ptr()), B,
                                            blk.stride(0), st))
        got = clip.cpu().numpy()
    finally:
        L.v2e_resize_destroy(r)
    for i in range(B * U):
        if i % U == k:
            want = _pillow(imgs[i // U], (sw, sh), 0)
            assert np.array_equal(got[i], want), "frame %d: %d pixels differ from Pillow" % (
                i, int((got[i] != want).sum()))
        else:
            assert (got[i] == 0xA5).all(), "frame %d was written" % i
