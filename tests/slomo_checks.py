"""Float64 references of the SuperSloMo engine's kernels and their error bars, judged layer by layer on the engine's
own inputs: shared by tests/test_slomo_layers.py (production shapes) and tests/test_slomo_geometry.py (the frame
sizes, batch sizes and SM counts that reach the other kernel paths).

Each kernel is fed the engine's OWN fp16 inputs (SloMoEngine.activations), so errors do not compound through the
network and every kernel is judged alone in its production configuration: the engine's buffers, concatenated inputs,
batch, grid and items per CTA. Frames are textured (independent random uint8 pixels), where a half-pixel sampling
error or a dropped filter tap is far above every bar.

Bars (tests/helpers.py): fp16 outputs |got - ref| <= ulp16(ref) + 2^-16 * S with S = conv2d(|x|, |w|) + |b|; fp32
heads 2^-16 * S; pools and separate up-samplings 1 fp16 ulp of the float64 value computed from the engine's input
plus their float32 rounding (pool_ratio, up_ratio); fused up-sampling convolutions ulp16(ref) + 2^-10 * S' (see
layer_error)."""
import functools

import numpy as np
import torch
import torch.nn.functional as F

import slomo_ref
from helpers import conv_bound, conv_ref64, err_ratio, ulp16

DEV = "cuda:0"
SHAPES_FC, SHAPES_AT = slomo_ref.layer_shapes(2, 4), slomo_ref.layer_shapes(12, 5)
NAMES = slomo_ref.LAYER_NAMES
UP_BAR = 2.0 ** -10
KMEAN = float(np.float32(0.428))


def make_weights(seed):
    return (slomo_ref.make_test_weights(100 + seed, 2, 4, head_gain=25.0),
            slomo_ref.make_test_weights(200 + seed, 12, 5, head_gain=0.3))


def scaled(sd, first, last):
    """Hidden activations ~first times larger (thousands), head scaled back (as test_slomo_gpu._scaled)."""
    out = {k: v.clone() for k, v in sd.items()}
    out["conv1.weight"] *= first
    out["conv1.bias"] *= first
    out["conv3.weight"] *= last
    return out


def textured(n, H, W, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, H, W), dtype=np.uint8)


def _clone(a):
    if isinstance(a, dict):
        return {k: _clone(v) for k, v in a.items()}
    return [_clone(v) for v in a] if isinstance(a, list) else a.clone()


@functools.lru_cache(maxsize=1)
def snapshot(src, B, scale=None):
    """Runs one set_pairs + one interp(0.3) on textured source frames of size src = (W, H) and keeps copies of
    everything the checks read: the flow network's activations (taken between set_pairs and interp: the two networks
    share the buffers), the interpolation network's, both heads and both kernel records. One configuration is held at
    a time."""
    from v2e_b200.slomo import SloMoEngine
    W, H = src
    sd_fc, sd_at = make_weights(11)
    if scale:
        sd_fc, sd_at = scaled(sd_fc, scale, 1 / scale), scaled(sd_at, scale, 1 / scale)
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


def nchw(t):
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


def layer_error(net, li, b, drop_channel=None, drop_tap=None):
    """|got - ref| / bar of layer li on image b, per element [co, H, W] (float64), and for the fused up-sampling the
    mask [H, W] of its 2-pixel frame (computed by a separate kernel), else None. Padded head channels must be exactly 0.

    Fused up-sampling layers (up5.conv1 at >= 512 px): the reference is conv2d(interpolate(x), w16) in float64, the bar
    ulp16(ref) + 2^-10 * S' with S' = conv2d(interpolate(|x|), |w|) + |b|. The interior kernel multiplies x by the
    up-sampling folded into the filter and rounded to fp16 once (relative error 2^-11 per folded weight, and |folded
    weight| <= the same combination of |w|): at most 2^-11 * S'; the 2-pixel frame kernel rounds each bilinear sample
    to fp16 (2^-11 * S' again) and must meet the same bar."""
    co, ci, k = net["shapes"][li]
    sd = net["sd"]
    w = sd[NAMES[li] + ".weight"].to(DEV).half()
    bias = sd[NAMES[li] + ".bias"].to(DEV).float()
    xs, out = layer_inputs(net, li)
    x = nchw(torch.cat([t[b:b + 1] for t in xs], -1)).double()
    frame = None
    if net["plan"][li] == "up2":
        up = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
        ref, _ = conv_ref64(up, w, bias, 1, drop_channel=drop_channel, drop_tap=drop_tap)
        del up
        upa = F.interpolate(x.abs(), scale_factor=2, mode="bilinear", align_corners=False)
        _, S = conv_ref64(upa, w, bias, 1)
        del upa
        bar = conv_bound(ref, S, acc=UP_BAR)
        frame = torch.ones(ref.shape[-2:], dtype=torch.bool, device=ref.device)
        frame[2:-2, 2:-2] = False
    else:
        ref, S = conv_ref64(x, w, bias, k // 2, drop_channel=drop_channel, drop_tap=drop_tap)
        bar = conv_bound(ref, S, fp16_out=li != 22)
    del S
    if li == 22:                                            # fp32 head [B, H, W, 8]: first co channels
        assert (out[b, ..., co:] == 0).all(), "padded head channels must be exactly lrelu(0) = 0"
        got = out[b, ..., :co]
    else:
        assert out.shape[-1] == co
        got = out[b]
    r = (got.permute(2, 0, 1).double() - ref[0]).abs() / bar[0]
    r[~torch.isfinite(r)] = float("inf")
    return r, frame


def layer_ratio(net, li, b, drop_channel=None, drop_tap=None, x0=0):
    """max |got - ref| / bar of layer li on image b over the columns x >= x0: {"all": r} or, for the fused
    up-sampling, {"interior": r, "frame": r}."""
    r, frame = layer_error(net, li, b, drop_channel, drop_tap)
    r = r[..., x0:]
    if frame is None:
        return {"all": r.max().item()}
    frame = frame[:, x0:]
    return {"interior": r[:, ~frame].max().item(), "frame": r[:, frame].max().item()}


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
    x = nchw((a["s"][4] if k == 0 else a["ub"][k - 1])[b:b + 1]).double()
    want = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
    A = F.interpolate(x.abs(), scale_factor=2, mode="bilinear", align_corners=False)
    return err_ratio(nchw(a["up"][k][b:b + 1]), want, ulp16(want) + 2.0 ** -22 * A)


def family(plan, li):
    return plan[li] + ("_head" if li == 22 else "")


class Worst:
    """Largest ratio per key, with what produced it."""

    def __init__(self):
        self.d = {}

    def note(self, key, r, what):
        if key not in self.d or r > self.d[key][0]:
            self.d[key] = (r, what)

    def report(self, title):
        print("\n%s: largest |got - ref| / bar" % title)
        for key, (r, what) in sorted(self.d.items()):
            print("  %-26s %.4f  (%s)" % (key, r, what))

    def bad(self):
        return {k: v for k, v in self.d.items() if not v[0] <= 1.0}


def check_every_layer(snap, regions=None):
    """All 23 layers of both networks on every image of the batch, every pool and every separate up-sampling: the
    largest ratio per kernel family (Worst). regions(li) -> {name: (rows, cols)} (slices of layer li's output) adds the
    largest ratio inside each such region of each layer as the key "<family> <name>"."""
    B = snap["B"]
    plan = snap["flow"]["plan"]
    worst = Worst()
    for netname in ("flow", "interp"):
        net = snap[netname]
        for li in range(23):
            fam = family(plan, li)
            for b in range(B):
                what = "%s %s image %d" % (netname, NAMES[li], b)
                r, frame = layer_error(net, li, b)
                if frame is None:
                    worst.note(fam, r.max().item(), what)
                else:
                    worst.note(fam + "_interior", r[:, ~frame].max().item(), what)
                    worst.note(fam + "_frame", r[:, frame].max().item(), what)
                for name, (rows, cols) in (regions(li) if regions else {}).items():
                    worst.note("%s %s" % (fam, name), r[:, rows, cols].max().item(), what)
                del r
        for l in range(5):
            fused = plan[1 if l == 0 else 2 * l + 1] == "strip_pool"
            for b in range(B):
                worst.note("pool_fused" if fused else "pool", pool_ratio(net, l, b),
                           "%s pool[%d] image %d" % (netname, l, b))
        for k in range(5):
            if plan[12 + 2 * k] != "up2":
                for b in range(B):
                    worst.note("upsample", up_ratio(net, k, b), "%s up[%d] image %d" % (netname, k, b))
    return worst


# ---- warps, blend, flow maximum: crafted flows ----------------------------------------------------------------------
def sample_offsets(n, pos, rng):
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


def crafted_flows(seed, B, H, W):
    """flow_out [B, H, W, 8]: F01 = -2a, F10 = 2a per pixel, so that at t = 0.5 F_t0 = a and F_t1 = -a exactly."""
    rng = np.random.default_rng(seed)
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    ax = sample_offsets(W, np.broadcast_to(xs, (B, H, W)), rng)
    ay = sample_offsets(H, np.broadcast_to(ys, (B, H, W)), rng)
    f = np.zeros((B, H, W, 8), np.float32)
    f[..., 0], f[..., 1], f[..., 2], f[..., 3] = -2 * ax, -2 * ay, 2 * ax, 2 * ay
    return torch.from_numpy(f).to(DEV), ax, ay


R_FLOW = (0.25, 0.5, 0.75, 0.125)          # residual flows of the interpolation head (dyadic: exact positions)


_WARP_ENGINE = {}


def warp_engine(W, H, B):
    """W x H engine (network size) on textured frames whose interpolation head returns the constant residual flows
    R_FLOW (conv3 weights of channels 0..3 zero, biases R_FLOW: LeakyReLU passes them unchanged) and a per-pixel
    visibility logit. One engine is kept at a time (the previous one is closed)."""
    from v2e_b200.slomo import SloMoEngine
    key = (W, H, B)
    if key not in _WARP_ENGINE:
        for e in _WARP_ENGINE.values():
            e.close()
        _WARP_ENGINE.clear()
        sd_fc, sd_at = make_weights(21)
        sd_at = {k: v.clone() for k, v in sd_at.items()}
        sd_at["conv3.weight"][:4] = 0
        sd_at["conv3.bias"][:4] = torch.tensor(R_FLOW)
        eng = SloMoEngine(sd_fc, sd_at, (W, H), B, DEV)
        eng.set_pairs(torch.from_numpy(textured(B + 1, H, W, 5)).to(DEV))
        _WARP_ENGINE[key] = eng
    return _WARP_ENGINE[key]


def flow_coef(t):
    """slomo.py:405-410, 428 as the kernels receive them: Python doubles rounded to float32."""
    temp = -t * (1 - t)
    return [float(np.float32(v)) for v in (temp, t * t, (1 - t) * (1 - t), temp, 1 - t, t)]


def pre_interp_reference(img, flow, t, shift=0.0):
    """slomo.py:405-419 with the reference's own float32 arithmetic (slomo_ref.backwarp): the 12 interpolator input
    channels [B, H, W, 12]. shift moves both warps by that many pixels along x (sensitivity)."""
    I0, I1 = img[:-1, None].cpu(), img[1:, None].cpu()
    F01, F10 = nchw(flow[..., 0:2]).cpu(), nchw(flow[..., 2:4]).cpu()
    temp = -t * (1 - t)
    Ft0 = temp * F01 + (t * t) * F10
    Ft1 = ((1 - t) * (1 - t)) * F01 + temp * F10
    sh = torch.tensor([shift, 0.0]).view(1, 2, 1, 1)
    g0 = slomo_ref.backwarp(I0, Ft0 + sh)
    g1 = slomo_ref.backwarp(I1, Ft1 + sh)
    return torch.cat((I0, I1, F01, F10, Ft1, Ft0, g1, g0), 1).permute(0, 2, 3, 1).to(DEV)


def position_delta(fx, fy, H, W):
    """Allowed movement (pixels, x plus y) of a back-warp's sampling position between the kernel's and the
    reference's float32 evaluations at flow (fx, fy). grid_sample's normalise / un-normalise round trip
    (x + u, / W, - 0.5, * 2, + 1, * W, - 1, / 2) rounds six values whose size in pixels is at most |u| + 2W; each
    rounding moves the position by at most 2^-24 of that, and the kernel may contract a multiply-add where the
    reference rounds twice. delta_x = 2^-21 * (|fx| + 2W) covers them with room; the same along y."""
    return 2.0 ** -21 * (fx.abs() + fy.abs() + 2 * (W + H))


def pre_interp_bar(want, img, exact_positions):
    """Bar of pre_interp against pre_interp_reference: 1 fp16 ulp of every channel, and on the two warp channels
    (10: g(I1, F_t1), 11: g(I0, F_t0)) the position allowance 2m * (delta_x + delta_y) (position_delta, from the
    reference's F_t1 / F_t0 in channels 6-7 / 8-9): a bilinear sample of values within +-m changes by at most 2m per
    pixel of movement along an axis. exact_positions: both sides sample at the same points (no allowance)."""
    bar = ulp16(want)
    if not exact_positions:
        m = img.abs().max().item()
        H, W = want.shape[1:3]
        for ch, fx in ((10, 6), (11, 8)):
            bar[..., ch] += 2 * m * position_delta(want[..., fx], want[..., fx + 1], H, W)
    return bar


def bilinear64(I, ix, iy):
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
    """slomo.py:421-437 in float64 from the engine's float32 flows, head and frames: (Ft, M, delta) with M the blend
    of the absolute values (w0 G0 + w1 G1) / (w0 V0 + w1 V1), G = bilinear sample of |I|, which bounds every term's
    size, and delta the larger position_delta of the two warps."""
    c00, c01, c10, c11, w0, w1 = flow_coef(t)
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
    g0, g1 = bilinear64(I0, *p0), bilinear64(I1, *p1)
    den = w0 * v0 + w1 * v1
    ft = (w0 * v0 * g0 + w1 * v1 * g1) / den
    M = (w0 * bilinear64(I0.abs(), *p0) + w1 * bilinear64(I1.abs(), *p1)) / den
    delta = torch.maximum(position_delta(ft0x, ft0y, H, W), position_delta(ft1x, ft1y, H, W))
    return ft, M, delta
