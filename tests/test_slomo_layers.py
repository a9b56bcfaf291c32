"""GPU: every convolution of both SuperSloMo UNets, the average pools, the bilinear up-samplings, the warps, the blend
and the frame preparation against float64 references, layer by layer.

Each kernel is fed the engine's OWN fp16 inputs (SloMoEngine.activations), so errors do not compound through the
network and every kernel is judged alone in its production configuration: the engine's buffers, concatenated inputs,
batch, grid and items per CTA. Every test asserts from the engine's own record (SloMoEngine.layer_kernels) which
kernels it covered. Frames are textured (independent random uint8 pixels), where a half-pixel sampling error or a
dropped filter tap is far above every bar.

Bars (tests/helpers.py): fp16 outputs |got - ref| <= ulp16(ref) + 2^-16 * S with S = conv2d(|x|, |w|) + |b|; fp32
heads 2^-16 * S; pools and separate up-samplings 1 fp16 ulp of the float64 value computed from the engine's input
plus their float32 rounding (pool_ratio, up_ratio); fused up-sampling convolutions ulp16(ref) + 2^-10 * S' (see test docstring). The sensitivity tests at the end show that
each comparison fails when the float64 reference, and only the reference, is perturbed."""
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import slomo_ref
from helpers import conv_bound, conv_ref64, err_ratio, ulp16, ulp32

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES_FC, SHAPES_AT = slomo_ref.layer_shapes(2, 4), slomo_ref.layer_shapes(12, 5)
NAMES = slomo_ref.LAYER_NAMES
UP_BAR = 2.0 ** -10
KMEAN = float(np.float32(0.428))


def _weights(seed):
    return (slomo_ref.make_test_weights(100 + seed, 2, 4, head_gain=25.0),
            slomo_ref.make_test_weights(200 + seed, 12, 5, head_gain=0.3))


def _scaled(sd, first, last):
    """Hidden activations ~first times larger (thousands), head scaled back (as test_slomo_gpu._scaled)."""
    out = {k: v.clone() for k, v in sd.items()}
    out["conv1.weight"] *= first
    out["conv1.bias"] *= first
    out["conv3.weight"] *= last
    return out


def textured(n, H, W, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, H, W), dtype=np.uint8)


# source frame size, batch, weight scale. Items per CTA of the strip kernels at 1280x704 (132 SMs): conv1 1280 items on
# 264 CTAs (2 per SM), conv2 1280 items on 132 CTAs, down1.conv2 (5x5, 64 channels, output channels split over two CTA
# classes) 320 items on 66 CTAs per class; batch 2 divides these by 4.
CONFIGS = {
    "1280x704_b8": ((1280, 704), 8, None),        # bench headline: strip, pooled epilogues, fused up-sampling
    "346x260_b3": ((346, 260), 3, None),          # 320x256 network: 2.5-strip rows, odd batch, pooled conv2
    "128x96_b2": ((128, 96), 2, None),            # per-tap kernel, separate pool / up-sampling kernels only
    "1280x704_b2_x400": ((1280, 704), 2, 400.0),  # activations in the thousands through strip and fused kernels
}


def _clone(a):
    if isinstance(a, dict):
        return {k: _clone(v) for k, v in a.items()}
    return [_clone(v) for v in a] if isinstance(a, list) else a.clone()


@functools.lru_cache(maxsize=1)
def snapshot(name):
    """Runs one set_pairs + one interp(0.3) on textured frames and keeps copies of everything the checks read: the
    flow network's activations (taken between set_pairs and interp: the two networks share the buffers), the
    interpolation network's, both heads and both kernel records. One configuration is held at a time."""
    from v2e_b200.slomo import SloMoEngine
    (W, H), B, scale = CONFIGS[name]
    sd_fc, sd_at = _weights(11)
    if scale:
        sd_fc, sd_at = _scaled(sd_fc, scale, 1 / scale), _scaled(sd_at, scale, 1 / scale)
    eng = SloMoEngine(sd_fc, sd_at, (W, H), B, DEV)
    eng.set_pairs(torch.from_numpy(textured(B + 1, H, W, 7)).to(DEV))
    flow = dict(acts=_clone(eng.activations()), head=eng.flow_out().clone(), sd=sd_fc, shapes=SHAPES_FC,
                net_in=eng._net_in[:B + 1].clone())
    eng.interp(0.3, torch.empty((B, H, W), dtype=torch.uint8, device=DEV))
    interp = dict(acts=_clone(eng.activations()), head=eng.intrp_out().clone(), sd=sd_at, shapes=SHAPES_AT)
    plan = eng.layer_kernels()
    flow["plan"], interp["plan"] = plan["flow"], plan["interp"]
    eng.check_finite()
    eng.close()
    torch.cuda.synchronize()
    return {"flow": flow, "interp": interp, "B": B, "hw": (eng.h, eng.w)}


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def layer_inputs(net, li):
    """The engine's fp16 input(s) of layer li (NHWC, batch first) and its output; for a fused up-sampling layer the
    input is the low-resolution x (up[k] was never written)."""
    a, plan = net["acts"], net["plan"]
    ci = net["shapes"][li][1]
    if li == 0:
        return [a["in16"][..., :ci]], a["x0"]
    if li == 1:
        return [a["x0"]], a["s1"]
    if li < 12:
        l = (li - 2) // 2
        return ([a["pool"][l]], a["da"][l]) if li % 2 == 0 else ([a["da"][l]], a["s"][l])
    if li < 22:
        k = (li - 12) // 2
        if li % 2 == 0:
            x = a["s"][4] if k == 0 else a["ub"][k - 1]
            return ([x] if plan[li] == "up2" else [a["up"][k]]), a["ua"][k]
        return [a["ua"][k], a["s"][3 - k] if k < 4 else a["s1"]], a["ub"][k]
    return [a["ub"][4]], net["head"]


def layer_ratio(net, li, b, drop_channel=None, drop_tap=None):
    """max |got - ref| / bar of layer li on image b: {"all": r} or, for the fused up-sampling, {"interior": r,
    "frame": r} (the 2-pixel frame is computed by a separate kernel). Padded head channels must be exactly 0."""
    co, ci, k = net["shapes"][li]
    sd = net["sd"]
    w = sd[NAMES[li] + ".weight"].to(DEV).half()
    bias = sd[NAMES[li] + ".bias"].to(DEV).float()
    xs, out = layer_inputs(net, li)
    x = _nchw(torch.cat([t[b:b + 1] for t in xs], -1)).double()
    if net["plan"][li] == "up2":
        up = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
        ref, _ = conv_ref64(up, w, bias, 1, drop_channel=drop_channel, drop_tap=drop_tap)
        upa = F.interpolate(x.abs(), scale_factor=2, mode="bilinear", align_corners=False)
        _, S = conv_ref64(upa, w, bias, 1)
        bar = conv_bound(ref, S, acc=UP_BAR)
        got = _nchw(out[b:b + 1, ..., :co])
        frame = torch.ones_like(ref, dtype=torch.bool)
        frame[..., 2:-2, 2:-2] = False
        r = (got.double() - ref).abs() / bar
        assert torch.isfinite(r).all()
        return {"interior": r[~frame].max().item(), "frame": r[frame].max().item()}
    ref, S = conv_ref64(x, w, bias, k // 2, drop_channel=drop_channel, drop_tap=drop_tap)
    if li == 22:                                            # fp32 head [B, H, W, 8]: first co channels
        assert (out[b, ..., co:] == 0).all(), "padded head channels must be exactly lrelu(0) = 0"
        return {"all": err_ratio(_nchw(out[b:b + 1, ..., :co]), ref, conv_bound(ref, S, fp16_out=False))}
    assert out.shape[-1] == co
    return {"all": err_ratio(_nchw(out[b:b + 1]), ref, conv_bound(ref, S))}


def pool_ratio(net, l, b, shift=0):
    """pool[l] vs the float64 mean of the engine's four fp16 values. The kernels add the four in float32 (three
    roundings of at most 2^-24 of the running |sum| <= sum |a_i|: exact unless the four magnitudes span more than
    ~2^13, which the 400x-scaled activations do) and round the quarter to fp16 once: bar ulp16(mean) + 2^-20 * mean|a_i|
    (12 * 2^-24 rounded up). shift moves the reference's 2x2 windows one pixel to the right (sensitivity)."""
    a = net["acts"]
    src = (a["s1"] if l == 0 else a["s"][l - 1])[b].double()
    if shift:
        src = torch.roll(src, -shift, dims=1)
    H, W, C = src.shape
    want = src.view(H // 2, 2, W // 2, 2, C).mean((1, 3))
    A = src.abs().view(H // 2, 2, W // 2, 2, C).mean((1, 3))
    return err_ratio(a["pool"][l][b], want, ulp16(want) + 2.0 ** -20 * A)


def up_ratio(net, k, b):
    """Separate up-sampling up[k] vs float64 F.interpolate(x, 2, bilinear) of the engine's x. The kernel evaluates
    the 0.25 / 0.75 weighted sum of four fp16 values in float32 (at most four roundings along any path, each <= 2^-24
    of a partial sum bounded by A = interpolate(|x|)) and rounds to fp16 once: bar ulp16(ref) + 2^-22 * A. The second
    term matters where the four values nearly cancel (the 400x-scaled activations)."""
    a = net["acts"]
    x = _nchw((a["s"][4] if k == 0 else a["ub"][k - 1])[b:b + 1]).double()
    want = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
    A = F.interpolate(x.abs(), scale_factor=2, mode="bilinear", align_corners=False)
    return err_ratio(_nchw(a["up"][k][b:b + 1]), want, ulp16(want) + 2.0 ** -22 * A)


def _family(plan, li):
    return plan[li] + ("_head" if li == 22 else "")


@pytest.mark.parametrize("config", list(CONFIGS))
def test_every_layer_matches_float64(config):
    """All 23 layers of both networks, on every image of the batch, plus every pool and separate up-sampling.

    Fused up-sampling layers (up5.conv1 at >= 512 px): the reference is conv2d(interpolate(x), w16) in float64, the bar
    ulp16(ref) + 2^-10 * S' with S' = conv2d(interpolate(|x|), |w|) + |b|. The interior kernel multiplies x by the
    up-sampling folded into the filter and rounded to fp16 once (relative error 2^-11 per folded weight, and |folded
    weight| <= the same combination of |w|): at most 2^-11 * S'; the 2-pixel frame kernel rounds each bilinear sample
    to fp16 (2^-11 * S' again) and must meet the same bar."""
    snap = snapshot(config)
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
    worst = {}

    def note(fam, r, what):
        if fam not in worst or r > worst[fam][0]:
            worst[fam] = (r, what)

    for netname in ("flow", "interp"):
        net = snap[netname]
        for li in range(23):
            for b in range(B):
                for region, r in layer_ratio(net, li, b).items():
                    fam = _family(plan, li) + ("" if region == "all" else "_" + region)
                    note(fam, r, "%s %s image %d" % (netname, NAMES[li], b))
        for l in range(5):
            fused = plan[1 if l == 0 else 2 * l + 1] == "strip_pool"
            for b in range(B):
                note("pool_fused" if fused else "pool", pool_ratio(net, l, b), "%s pool[%d] image %d" % (netname, l, b))
        for k in range(5):
            if plan[12 + 2 * k] != "up2":
                for b in range(B):
                    note("upsample", up_ratio(net, k, b), "%s up[%d] image %d" % (netname, k, b))
    print("\n%s: largest |got - ref| / bar per kernel family" % config)
    for fam, (r, what) in sorted(worst.items()):
        print("  %-18s %.4f  (%s)" % (fam, r, what))
    bad = {f: v for f, v in worst.items() if not v[0] <= 1.0}
    assert not bad, bad


@pytest.mark.parametrize("config", list(CONFIGS))
def test_prep_pairs_is_exact(config):
    """prep_pairs_kernel: img = float32(u8 / 255 - 0.428) exactly (the reference's float32 ToTensor + Normalize);
    the flow network's input channels 0 / 1 are its fp16 rounding for frames b / b+1, channels 2..15 are zero."""
    snap = snapshot(config)
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
R_FLOW = (0.25, 0.5, 0.75, 0.125)          # residual flows of the interpolation head (dyadic: exact positions)


def _offsets(n, pos, rng):
    """Per-pixel sampling offsets u along one axis of size n at coordinates pos: zero, integer and half-integer
    shifts, negative fractions, samples landing exactly on -1, 0, n-1 and n (x + u - 0.5 = target), and shifts
    beyond +-n (fully outside: the sample is 0)."""
    fixed = np.array([0, 1, -1, 3, -2, 0.5, -0.5, 2.5, -1.5, -0.25, -0.75, -1.625, 0.375,
                      n + 3.25, -(n + 2.5), 2 * n, -3 * n], np.float64)
    land = np.stack([t - pos + 0.5 for t in (-1, 0, n - 1, n)], -1)
    k = rng.integers(0, len(fixed) + 4, pos.shape)
    u = np.where(k < len(fixed), fixed[np.minimum(k, len(fixed) - 1)],
                 np.take_along_axis(land, np.clip(k - len(fixed), 0, 3)[..., None], -1)[..., 0])
    return u.astype(np.float32)


def crafted_flows(seed):
    """flow_out [B, H, W, 8]: F01 = -2a, F10 = 2a per pixel, so that at t = 0.5 F_t0 = a and F_t1 = -a exactly."""
    rng = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.arange(WH), np.arange(WW), indexing="ij")
    ax = _offsets(WW, np.broadcast_to(xs, (WB, WH, WW)), rng)
    ay = _offsets(WH, np.broadcast_to(ys, (WB, WH, WW)), rng)
    f = np.zeros((WB, WH, WW, 8), np.float32)
    f[..., 0], f[..., 1], f[..., 2], f[..., 3] = -2 * ax, -2 * ay, 2 * ax, 2 * ay
    return torch.from_numpy(f).to(DEV), ax, ay


@functools.lru_cache(maxsize=1)
def warp_engine():
    """128x64 engine on textured frames whose interpolation head returns the constant residual flows R_FLOW (conv3
    weights of channels 0..3 zero, biases R_FLOW: LeakyReLU passes them unchanged) and a per-pixel visibility logit."""
    from v2e_b200.slomo import SloMoEngine
    sd_fc, sd_at = _weights(21)
    sd_at = {k: v.clone() for k, v in sd_at.items()}
    sd_at["conv3.weight"][:4] = 0
    sd_at["conv3.bias"][:4] = torch.tensor(R_FLOW)
    eng = SloMoEngine(sd_fc, sd_at, (WW, WH), WB, DEV)
    eng.set_pairs(torch.from_numpy(textured(WB + 1, WH, WW, 5)).to(DEV))
    return eng


def _coef(t):
    """slomo.py:405-410, 428 as the kernels receive them: Python doubles rounded to float32."""
    temp = -t * (1 - t)
    return [float(np.float32(v)) for v in (temp, t * t, (1 - t) * (1 - t), temp, 1 - t, t)]


def pre_interp_reference(img, flow, t, shift=0.0):
    """slomo.py:405-419 with the reference's own float32 arithmetic (slomo_ref.backwarp): the 12 interpolator input
    channels [B, H, W, 12]. shift moves both warps by that many pixels along x (sensitivity)."""
    I0, I1 = img[:-1, None].cpu(), img[1:, None].cpu()
    F01, F10 = _nchw(flow[..., 0:2]).cpu(), _nchw(flow[..., 2:4]).cpu()
    temp = -t * (1 - t)
    Ft0 = temp * F01 + (t * t) * F10
    Ft1 = ((1 - t) * (1 - t)) * F01 + temp * F10
    sh = torch.tensor([shift, 0.0]).view(1, 2, 1, 1)
    g0 = slomo_ref.backwarp(I0, Ft0 + sh)
    g1 = slomo_ref.backwarp(I1, Ft1 + sh)
    return torch.cat((I0, I1, F01, F10, Ft1, Ft0, g1, g0), 1).permute(0, 2, 3, 1).to(DEV)


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
    eng = warp_engine()
    f, ax, ay = crafted_flows(1)
    eng.flow_out().copy_(f)
    eng.interp(t, torch.empty((WB, WH, WW), dtype=torch.uint8, device=DEV))
    a = eng.activations()
    got = a["in16"].double()
    want = pre_interp_reference(a["img"], eng.flow_out(), t).double()
    bar = ulp16(want)
    if t != 0.5:
        m = a["img"].abs().max().item()
        for ch, fx in ((10, 6), (11, 8)):       # g(I1, F_t1), g(I0, F_t0)
            delta = 2.0 ** -21 * (want[..., fx].abs() + want[..., fx + 1].abs() + 2 * (WW + WH))
            bar[..., ch] += 2 * m * delta
    r = [err_ratio(got[..., c], want[..., c], bar[..., c]) for c in range(12)]
    print("\npre_interp t=%.1f: largest |got - ref| / bar per channel %s" % (t, ["%.3f" % v for v in r]))
    assert max(r) <= 1.0
    assert (a["in16"][..., 12:] == 0).all()
    if t == 0.5:
        out0 = torch.from_numpy((np.abs(ax) > WW + 1) | (np.abs(ay) > WH + 1)).to(DEV)
        assert out0.any() and (got[..., 11][out0] == 0).all() and (got[..., 10][out0] == 0).all()


def _bilinear64(I, ix, iy):
    """grid_sample(bilinear, zeros, align_corners=False) of I [B, H, W] (float64) at pixel coordinates ix, iy."""
    B, H, W = I.shape
    x0, y0 = torch.floor(ix), torch.floor(iy)
    acc = torch.zeros_like(ix)
    bi = torch.arange(B, device=I.device).view(B, 1, 1).expand_as(ix)
    for dy in (0, 1):
        for dx in (0, 1):
            xx, yy = x0 + dx, y0 + dy
            wgt = (1 - (ix - xx).abs()) * (1 - (iy - yy).abs())
            ok = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
            v = I[bi, yy.clamp(0, H - 1).long(), xx.clamp(0, W - 1).long()]
            acc = acc + torch.where(ok, wgt * v, torch.zeros_like(v))
    return acc


def post_interp_reference(img, flow, intrp, t, shift=0.0):
    """slomo.py:421-437 in float64 from the engine's float32 flows, head and frames: (Ft, M) with M the blend of the
    absolute values (w0 G0 + w1 G1) / (w0 V0 + w1 V1), G = bilinear sample of |I|, which bounds every term's size."""
    c00, c01, c10, c11, w0, w1 = _coef(t)
    f, r = flow.double(), intrp.double()
    I0, I1 = img[:-1].double(), img[1:].double()
    B, H, W = I0.shape
    ys, xs = torch.meshgrid(torch.arange(H, device=DEV, dtype=torch.float64),
                            torch.arange(W, device=DEV, dtype=torch.float64), indexing="ij")
    ft0x = c00 * f[..., 0] + c01 * f[..., 2] + r[..., 0] + shift
    ft0y = c00 * f[..., 1] + c01 * f[..., 3] + r[..., 1]
    ft1x = c10 * f[..., 0] + c11 * f[..., 2] + r[..., 2] + shift
    ft1y = c10 * f[..., 1] + c11 * f[..., 3] + r[..., 3]
    v0 = torch.sigmoid(r[..., 4])
    v1 = 1 - v0
    p0 = (xs + ft0x - 0.5, ys + ft0y - 0.5)
    p1 = (xs + ft1x - 0.5, ys + ft1y - 0.5)
    g0, g1 = _bilinear64(I0, *p0), _bilinear64(I1, *p1)
    den = w0 * v0 + w1 * v1
    ft = (w0 * v0 * g0 + w1 * v1 * g1) / den
    M = (w0 * _bilinear64(I0.abs(), *p0) + w1 * _bilinear64(I1.abs(), *p1)) / den
    return ft, M


def test_post_interp_blend_crafted_flows():
    """post_interp_kernel (refined flows, visibility, two back-warps, blend, uint8 quantisation) vs slomo.py:421-437
    in float64, from the engine's own flow_out (crafted), intrp_out and img. At t = 0.5 with these flows and dyadic
    residuals the sampling positions are exact, so what remains is float32 rounding: four products and sums per
    warp, expf / reciprocal / 1 - V0 for the visibility, the blend and its division -- each at most a few 2^-24 of
    the magnitude M of the terms; the bar is 16 float32 ulps of M. The uint8 frame (truncation toward zero of
    (Ft + 0.428) * 255, wrapped mod 256) must be exact except where that value lies within 1e-4 of an integer."""
    eng = warp_engine()
    f, _, _ = crafted_flows(2)
    eng.flow_out().copy_(f)
    out = torch.empty((WB, WH, WW), dtype=torch.uint8, device=DEV)
    ft = torch.empty((WB, WH, WW), dtype=torch.float32, device=DEV)
    eng.interp(0.5, out, ft)
    intrp = eng.intrp_out()
    assert torch.equal(intrp[..., :4], torch.tensor(R_FLOW, device=DEV).expand_as(intrp[..., :4]))
    assert intrp[..., 4].std() > 0.01
    want, M = post_interp_reference(eng.activations()["img"], eng.flow_out(), intrp, 0.5)
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
    eng = warp_engine()
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
    snap = snapshot(config)
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
    net = snapshot(config)["flow"]
    assert pool_ratio(net, 0, 0) <= 1.0
    assert pool_ratio(net, 0, 0, shift=1) > 1.0


def test_warp_comparisons_fail_on_half_pixel_shift():
    """pre_interp and post_interp comparisons fail when the reference's warps move by 0.5 px."""
    eng = warp_engine()
    f, _, _ = crafted_flows(1)
    eng.flow_out().copy_(f)
    ft = torch.empty((WB, WH, WW), dtype=torch.float32, device=DEV)
    eng.interp(0.5, torch.empty((WB, WH, WW), dtype=torch.uint8, device=DEV), ft)
    a = eng.activations()
    want = pre_interp_reference(a["img"], eng.flow_out(), 0.5, shift=0.5).double()
    assert err_ratio(a["in16"][..., 10:12], want[..., 10:12], ulp16(want[..., 10:12])) > 1.0
    want, M = post_interp_reference(a["img"], eng.flow_out(), eng.intrp_out(), 0.5, shift=0.5)
    assert err_ratio(ft, want, 16 * ulp32(M)) > 1.0
