"""GPU: every convolution of both SuperSloMo UNets, the average pools, the bilinear up-samplings, the warps, the blend
and the frame preparation against float64 references, layer by layer.

Each kernel is fed the engine's OWN fp16 inputs (SloMoEngine.activations), so errors do not compound through the
network and every kernel is judged alone in its production configuration: the engine's buffers, concatenated inputs,
batch, grid and items per CTA. Every test asserts from the engine's own record (SloMoEngine.layer_kernels) which
kernels it covered. Frames are textured (independent random uint8 pixels), where a half-pixel sampling error or a
dropped filter tap is far above every bar.

Bars (tests/helpers.py): fp16 outputs |got - ref| <= ulp16(ref) + 2^-16 * S with S = conv2d(|x|, |w|) + |b|; fp32
heads 2^-16 * S; pools and separate up-samplings 1 fp16 ulp of the float64 value computed from the engine's input
plus their float32 rounding (pool_ratio, up_ratio); fused up-sampling convolutions ulp16(ref) + 2^-10 * S'
(tests/slomo_checks.py, layer_error). The sensitivity tests at the end show that each comparison fails when the
float64 reference, and only the reference, is perturbed."""
import numpy as np
import pytest
import torch

import slomo_ref
from helpers import err_ratio, ulp16, ulp32
from slomo_checks import (DEV, KMEAN, NAMES, R_FLOW, check_every_layer, crafted_flows, layer_ratio, pool_ratio,
                          post_interp_reference, pre_interp_bar, pre_interp_reference, snapshot, warp_engine)

pytestmark = pytest.mark.gpu


# source frame size, batch, weight scale. Items per CTA of the strip kernels at 1280x704 (132 SMs): conv1 1280 items on
# 264 CTAs (2 per SM), conv2 1280 items on 132 CTAs, down1.conv2 (5x5, 64 channels, output channels split over two CTA
# classes) 320 items on 66 CTAs per class; batch 2 divides these by 4.
CONFIGS = {
    "1280x704_b8": ((1280, 704), 8, None),        # bench headline: strip, pooled epilogues, fused up-sampling
    "346x260_b3": ((346, 260), 3, None),          # 320x256 network: 2.5-strip rows, odd batch, pooled conv2
    "128x96_b2": ((128, 96), 2, None),            # per-tap kernel, separate pool / up-sampling kernels only
    "1280x704_b2_x400": ((1280, 704), 2, 400.0),  # activations in the thousands through strip and fused kernels
}


@pytest.mark.parametrize("config", list(CONFIGS))
def test_every_layer_matches_float64(config):
    """All 23 layers of both networks, on every image of the batch, plus every pool and separate up-sampling.

    Fused up-sampling layers (up5.conv1 at >= 512 px): the reference is conv2d(interpolate(x), w16) in float64, the bar
    ulp16(ref) + 2^-10 * S' with S' = conv2d(interpolate(|x|), |w|) + |b|. The interior kernel multiplies x by the
    up-sampling folded into the filter and rounded to fp16 once (relative error 2^-11 per folded weight, and |folded
    weight| <= the same combination of |w|): at most 2^-11 * S'; the 2-pixel frame kernel rounds each bilinear sample
    to fp16 (2^-11 * S' again) and must meet the same bar."""
    snap = snapshot(*CONFIGS[config])
    B, (H, W) = snap["B"], snap["hw"]
    plans = snap["flow"]["plan"], snap["interp"]["plan"]
    assert plans[0] == plans[1] and None not in plans[0]
    plan = plans[0]
    if config.startswith("1280x704"):
        assert plan[1] == "strip_pool" and plan[3] == "strip_pool" and plan[20] == "up2", plan
        assert {0, 2, 18, 19, 21, 22} <= {i for i, p in enumerate(plan) if p == "strip"}, plan
    elif config == "346x260_b3":
        assert (H, W) == (256, 320) and plan[1] == "strip_pool" and plan[0] == "strip" and "up2" not in plan, plan
    else:
        assert set(plan) == {"tap"}, plan
    worst = check_every_layer(snap)
    worst.report(config)
    assert not worst.bad(), worst.bad()


@pytest.mark.parametrize("config", list(CONFIGS))
def test_prep_pairs_is_exact(config):
    """prep_pairs_kernel: img = float32(u8 / 255 - 0.428) exactly (the reference's float32 ToTensor + Normalize);
    the flow network's input channels 0 / 1 are its fp16 rounding for frames b / b+1, channels 2..15 are zero."""
    snap = snapshot(*CONFIGS[config])
    B = snap["B"]
    net = snap["flow"]
    img = net["acts"]["img"]
    want = torch.from_numpy(net["net_in"].cpu().numpy().astype(np.float32) / 255.0 - 0.428).to(DEV)  # slomo_ref
    assert want.dtype == torch.float32 and torch.equal(img, want)
    in16 = net["acts"]["in16"]
    assert torch.equal(in16[..., 0], want[:B].half()) and torch.equal(in16[..., 1], want[1:].half())
    assert (in16[..., 2:] == 0).all()


# ---- warps, blend, flow maximum: crafted flows on a 128x64 network -------------------------------------------------
# W and H are powers of two and the crafted flows are dyadic, so at t = 0.5 every sampling position of the reference's
# float32 arithmetic (x + u, / W, - 0.5, * 2, + 1, * W, - 1, / 2) is exact: kernel and reference sample at the same
# points whether or not multiply-adds are contracted.
WW, WH, WB = 128, 64, 2


@pytest.mark.parametrize("t", [0.5, 0.3])
def test_pre_interp_warps_crafted_flows(t):
    """pre_interp_kernel: the 12-channel interpolator input (channel order of slomo.py:415-419: I0, I1, F01, F10, F_t1,
    F_t0, g(I1, F_t1), g(I0, F_t0)) within 1 fp16 ulp of the float32 reference, padding channels 12..15 zero, and the
    back-warp of a sample fully outside the image exactly 0. Flows set through the writable flow_out view after
    set_pairs; interp then runs the kernel on them.

    t = 0.5 makes every sampling position exact on both sides. At t = 0.3 F_t is rounded: the kernel contracts
    c00 * F01 + c01 * F10 into a multiply-add where the reference rounds both products, and the float32 normalise /
    un-normalise round trip of grid_sample (six roundings of values up to |F_t| + 2W) moves a position by at most
    delta = 2^-21 * (|F_t| + 2W) per axis. A bilinear sample of values within +-m changes by at most 2m per pixel of
    movement along an axis, so the two warp channels get 2m * (delta_x + delta_y) on top of the fp16 ulp."""
    eng = warp_engine(WW, WH, WB)
    f, ax, ay = crafted_flows(1, WB, WH, WW)
    eng.flow_out().copy_(f)
    eng.interp(t, torch.empty((WB, WH, WW), dtype=torch.uint8, device=DEV))
    a = eng.activations()
    got = a["in16"].double()
    want = pre_interp_reference(a["img"], eng.flow_out(), t).double()
    bar = pre_interp_bar(want, a["img"], exact_positions=t == 0.5)
    r = [err_ratio(got[..., c], want[..., c], bar[..., c]) for c in range(12)]
    print("\npre_interp t=%.1f: largest |got - ref| / bar per channel %s" % (t, ["%.3f" % v for v in r]))
    assert max(r) <= 1.0
    assert (a["in16"][..., 12:] == 0).all()
    if t == 0.5:
        out0 = torch.from_numpy((np.abs(ax) > WW + 1) | (np.abs(ay) > WH + 1)).to(DEV)
        assert out0.any() and (got[..., 11][out0] == 0).all() and (got[..., 10][out0] == 0).all()


def test_post_interp_blend_crafted_flows():
    """post_interp_kernel (refined flows, visibility, two back-warps, blend, uint8 quantisation) vs slomo.py:421-437
    in float64, from the engine's own flow_out (crafted), intrp_out and img. At t = 0.5 with these flows and dyadic
    residuals the sampling positions are exact, so what remains is float32 rounding: four products and sums per
    warp, expf / reciprocal / 1 - V0 for the visibility, the blend and its division -- each at most a few 2^-24 of
    the magnitude M of the terms; the bar is 16 float32 ulps of M. The uint8 frame (truncation toward zero of
    (Ft + 0.428) * 255, wrapped mod 256) must be exact except where that value lies within 1e-4 of an integer."""
    eng = warp_engine(WW, WH, WB)
    f, _, _ = crafted_flows(2, WB, WH, WW)
    eng.flow_out().copy_(f)
    out = torch.empty((WB, WH, WW), dtype=torch.uint8, device=DEV)
    ft = torch.empty((WB, WH, WW), dtype=torch.float32, device=DEV)
    eng.interp(0.5, out, ft)
    intrp = eng.intrp_out()
    assert torch.equal(intrp[..., :4], torch.tensor(R_FLOW, device=DEV).expand_as(intrp[..., :4]))
    assert intrp[..., 4].std() > 0.01
    want, M, _ = post_interp_reference(eng.activations()["img"], eng.flow_out(), intrp, 0.5)
    r = err_ratio(ft, want, 16 * ulp32(M))
    print("\npost_interp: largest |got - ref| / (16 ulp32(M)) = %.4f" % r)
    assert r <= 1.0
    s = (want + KMEAN) * 255.0
    ok = (s - torch.round(s)).abs() >= 1e-4
    u8 = torch.trunc(s).long() & 255
    assert ok.float().mean() > 0.99
    assert torch.equal(out.long()[ok], u8[ok])
    # and everywhere, from the kernel's own float32 Ft with the reference's float32 expression (slomo_ref.to_u8)
    assert torch.equal(out.cpu(), slomo_ref.to_u8(ft.cpu()))


@pytest.mark.parametrize("case", ["last_pixel", "first_pixel", "zero"])
def test_max_speed_crafted_flows(case):
    """max_speed_kernel: max over the batch of |F01| and |F10| (slomo.py:358-366) equals the planted maximum exactly
    (3-4-5 triangles: the float32 square root is exact), including the batch's last pixel and an all-zero field."""
    eng = warp_engine(WW, WH, WB)
    rng = np.random.default_rng(3)
    f = torch.from_numpy(rng.uniform(-3, 3, (WB, WH, WW, 8)).astype(np.float32)).to(DEV)    # |F| <= 3 sqrt(2) < 5
    f[..., 4:] = 0
    if case == "last_pixel":
        f[-1, -1, -1, 2:4] = torch.tensor([-30.0, 40.0])
        want = 50.0
    elif case == "first_pixel":
        f[0, 0, 0, 0:2] = torch.tensor([6.0, -8.0])
        want = 10.0
    else:
        f.zero_()
        want = 0.0
    eng.flow_out().copy_(f)
    assert eng.max_flow() == want


# ---- sensitivity: each comparison above fails when its reference is perturbed -------------------------------------
@pytest.mark.parametrize("config,li,family,perturb", [
    ("128x96_b2", 5, "tap", dict(drop_channel=17)),
    ("128x96_b2", 14, "tap", dict(drop_tap=(2, 0))),
    ("1280x704_b8", 0, "strip", dict(drop_tap=(3, 3))),
    ("1280x704_b8", 21, "strip", dict(drop_channel=40)),          # skip half of a concatenated input
    ("1280x704_b8", 1, "strip_pool", dict(drop_tap=(0, 6))),
    ("1280x704_b8", 3, "strip_pool", dict(drop_channel=3)),
    ("1280x704_b8", 20, "up2", dict(drop_channel=5)),
])
def test_layer_comparison_fails_on_perturbed_reference(config, li, family, perturb):
    """The layer comparison must fail when one input channel or one filter tap is removed from the float64 reference
    (the kernels are unchanged): the bars are tight enough to see a single missing term group. For the fused
    up-sampling both the interior and the separately computed frame must fail."""
    snap = snapshot(*CONFIGS[config])
    net = snap["interp"]
    assert net["plan"][li] == family
    b = snap["B"] - 1
    assert max(layer_ratio(net, li, b).values()) <= 1.0
    bad = layer_ratio(net, li, b, **perturb)
    print("\n%s %s %s: ratio against the perturbed reference %s" % (config, NAMES[li], perturb, bad))
    assert all(r > 1.0 for r in bad.values()), bad


@pytest.mark.parametrize("config", ["1280x704_b8", "128x96_b2"])
def test_pool_comparison_fails_on_shifted_window(config):
    """The pool comparison (fused at 1280x704, separate kernel at 128x96) fails when the reference's 2x2 windows move
    by one pixel."""
    net = snapshot(*CONFIGS[config])["flow"]
    assert pool_ratio(net, 0, 0) <= 1.0
    assert pool_ratio(net, 0, 0, shift=1) > 1.0


def test_warp_comparisons_fail_on_half_pixel_shift():
    """pre_interp and post_interp comparisons fail when the reference's warps move by 0.5 px."""
    eng = warp_engine(WW, WH, WB)
    f, _, _ = crafted_flows(1, WB, WH, WW)
    eng.flow_out().copy_(f)
    ft = torch.empty((WB, WH, WW), dtype=torch.float32, device=DEV)
    eng.interp(0.5, torch.empty((WB, WH, WW), dtype=torch.uint8, device=DEV), ft)
    a = eng.activations()
    want = pre_interp_reference(a["img"], eng.flow_out(), 0.5, shift=0.5).double()
    assert err_ratio(a["in16"][..., 10:12], want[..., 10:12], ulp16(want[..., 10:12])) > 1.0
    want, M, _ = post_interp_reference(a["img"], eng.flow_out(), eng.intrp_out(), 0.5, shift=0.5)
    assert err_ratio(ft, want, 16 * ulp32(M)) > 1.0
