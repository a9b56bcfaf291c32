"""Shared test helpers: golden-fixture loading, the RNG tape, event comparators."""
import json
import os

import numpy as np
import torch

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

EMU_GOLDENS = ["emu_class_default", "emu_cli_noisy", "emu_clean", "emu_scalar_thres_f64",
               "emu_refractory_multi", "emu_float_frames", "emu_static_leak_shot",
               "emu_ragged_13x37", "emu_csdvs", "emu_csdvs_120x176", "emu_hdr", "emu_hdr_nolp"]
# optional pixel models: SCIDVS (emulator.py:58-80, 719-725), photoreceptor noise (emulator.py:694-703)
EMU_GOLDENS_OPT = ["emu_scidvs", "emu_scidvs_f32", "emu_prnoise", "emu_prnoise_scidvs_csdvs"]


def load_golden(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False)
    g = {k: z[k] for k in z.files if not k.startswith("tape_0")}
    g["kwargs"] = json.loads(str(z["kwargs_json"]))
    if "tape_kinds" in z.files:
        g["tape"] = [(str(k), z["tape_%05d" % i]) for i, k in enumerate(z["tape_kinds"])]
    return g


class TapeRNG:
    """Replays the random draws the reference made when the golden was recorded
    (oracle/make_golden.py::Recorder), checking that the consumer asks for the same
    kind and size of draw in the same order."""

    def __init__(self, tape):
        self.tape = list(tape)
        self.pos = 0

    def _next(self, kind, shape=None):
        assert self.pos < len(self.tape), "RNG tape exhausted (asked for %s)" % kind
        k, arr = self.tape[self.pos]
        self.pos += 1
        assert k == kind, "draw %d: reference drew %s, consumer asked %s" % (self.pos - 1, k, kind)
        if shape is not None:
            assert tuple(arr.shape) == tuple(shape), (kind, arr.shape, shape)
        return torch.from_numpy(np.array(arr))

    def normal(self, mean, std, shape):
        return self._next("normal", shape)

    def randn(self, shape):
        return self._next("randn", shape)

    def rand(self, shape):
        return self._next("rand", shape)

    def randperm(self, n):
        t = self._next("randperm", (n,))
        return t.long()

    def exhausted(self):
        return self.pos == len(self.tape)


class DeviceDrawRNG:
    """Draw source for OracleEmulator(rng=..., shuffle=False) that hands the oracle the device RNG's own per-frame draws,
    so that rng_mode="device" can be compared with the oracle bit for bit.

    draws_for_frame(k) -> {"leak_randn", "shot_u01", "pr_randn"} ([H, W] float32, numpy or torch) for frame k >= 1 of
    the clip; `frame` must hold the number of the frame being generated (run_oracle_with_draws sets it). Frame 0's
    initial draws (thresholds, SCIDVS tau, noise-rate field) come from torch's global generator, as in device mode.
    After that: randn gives the photoreceptor normals (when that model is on), then the leak normals; rand the shot
    uniforms; randperm(n) the identity (device rows of one (frame, iteration, polarity) group have no order)."""

    def __init__(self, draws_for_frame, photoreceptor_noise=False):
        self.draws_for_frame = draws_for_frame
        self.photoreceptor_noise = photoreceptor_noise
        self.frame = 0
        self._loaded = None
        self.calls = []            # (frame, kind) of every per-frame draw served

    def _load(self, kind, shape):
        assert self.frame >= 1
        if self._loaded != self.frame:
            d = self.draws_for_frame(self.frame)
            host = {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in d.items()}
            self._randn = ([host["pr_randn"]] if self.photoreceptor_noise else []) + [host["leak_randn"]]
            self._rand = [host["shot_u01"]]
            self._loaded = self.frame
        q = self._randn if kind == "randn" else self._rand
        assert q, "frame %d: more %s draws than the device makes" % (self.frame, kind)
        a = q.pop(0)
        assert a.shape == tuple(shape) and a.dtype == np.float32, (a.shape, a.dtype, shape)
        self.calls.append((self.frame, kind))
        return torch.from_numpy(np.array(a))

    def normal(self, mean, std, shape):
        assert self.frame == 0, "normal() after the first frame"
        return torch.normal(mean, std, size=shape, dtype=torch.float32)

    def randn(self, shape):
        if self.frame == 0:
            return torch.randn(shape, dtype=torch.float32)
        return self._load("randn", shape)

    def rand(self, shape):
        assert self.frame >= 1, "rand() in the first frame"
        return self._load("rand", shape)

    def randperm(self, n):
        return torch.arange(n)


def run_oracle_with_draws(orc, rng, frames, times):
    """Runs the oracle over a clip with a DeviceDrawRNG, frame k's draws being those of the clip's frame k.
    Returns the per-frame rows (canonical order)."""
    out = []
    for k, (f, t) in enumerate(zip(frames, times)):
        rng.frame = k
        out.append(canonical(orc.generate_events(f, float(t))))
    return out


# ---- float64 references of the SuperSloMo convolutions and their error bars -----------------------------------
# The convolution kernels multiply fp16 operands exactly and accumulate in fp32; fp16 outputs are then rounded once.
# Against conv2d evaluated in float64 on the SAME fp16 operands the error of an output is therefore at most
#   fp16 output rounding   <= ulp16(ref) / 2
#   fp32 accumulation      <= (number of fp32 additions) * 2^-24 * (running |partial sum|) <= K * 2^-24 * S in the
#                             worst case, S = conv2d(|x|, |w|) + |b|. The tensor cores add K = 16 products per step with
#                             wider internal precision and the running sums cancel (|sum| << S), so in practice the
#                             error is ~2^-20 S; 2^-16 * S keeps a large margin and is still far below the cost of
#                             dropping one product out of K <= 9216 (~S / K >= 2^-13.2 * S).
# LeakyReLU is 1-Lipschitz, so the same bar holds after the activation. The fp32 network heads are not rounded to
# fp16: their bar is the accumulation term alone.
SLOPE = float(np.float32(0.1))     # the kernels' LeakyReLU slope: 0.1 rounded to float32
ACC_BAR = 2.0 ** -16


def ulp16(x):
    """Spacing of fp16 numbers at |x| (float64 tensor); 2^-24 in fp16's subnormal range."""
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -14))      # |x| = m * 2^e, m in [0.5, 1)
    return torch.ldexp(torch.ones_like(x), (e - 11).to(torch.int32))


def ulp32(x):
    """Spacing of float32 numbers at |x| (float64 tensor)."""
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x), (e - 24).to(torch.int32))


def conv_ref64(x, w, b, pad, slope=SLOPE, drop_channel=None, drop_tap=None):
    """lrelu(conv2d(x, w, b)) in float64 and S = conv2d(|x|, |w|) + |b|. x: [N, C, H, W], w: [Co, C, K, K] (both already
    rounded to the operand precision), b: [Co]. drop_channel / drop_tap remove one input channel / one filter tap (r, s)
    from the reference only: the perturbations that must make a comparison fail."""
    x64, w64, b64 = x.double(), w.double(), b.double()
    wr = w64.clone()
    if drop_channel is not None:
        wr[:, drop_channel] = 0
    if drop_tap is not None:
        wr[:, :, drop_tap[0], drop_tap[1]] = 0
    ref = torch.nn.functional.leaky_relu(torch.nn.functional.conv2d(x64, wr, b64, padding=pad), slope)
    S = torch.nn.functional.conv2d(x64.abs(), w64.abs(), padding=pad) + b64.abs().view(1, -1, 1, 1)
    return ref, S


def conv_bound(ref, S, fp16_out=True, acc=ACC_BAR):
    """Largest |got - ref| the arithmetic allows (see above): ulp16(ref) + acc * S, or acc * S for fp32 outputs."""
    return (ulp16(ref) if fp16_out else 0.0) + acc * S


def err_ratio(got, ref, bound):
    """max |got - ref| / bound (nan / inf in got count as failures)."""
    r = (got.double() - ref).abs() / bound
    return float("inf") if not torch.isfinite(r).all() else r.max().item()


def split_events(events, counts):
    off = np.concatenate([[0], np.cumsum(counts)])
    return [events[off[i]:off[i + 1]] for i in range(len(counts))]


def canonical(ev):
    """Sort rows by (t, y, x, p) -- the order-insensitive form (SURVEY 8d parity criteria)."""
    if ev is None or len(ev) == 0:
        return np.zeros((0, 4), np.float32)
    k = np.lexsort((ev[:, 3], ev[:, 1], ev[:, 2], ev[:, 0]))
    return np.ascontiguousarray(ev[k])


def assert_events_equal(got, want, exact_order=True, t_tol=0.0, ctx=""):
    got = np.zeros((0, 4), np.float32) if got is None else got
    want = np.zeros((0, 4), np.float32) if want is None else want
    assert got.shape == want.shape, "%s: %s rows vs reference %s" % (ctx, got.shape, want.shape)
    if not exact_order:
        got, want = canonical(got), canonical(want)
    assert np.array_equal(got[:, 1:], want[:, 1:]), "%s: x/y/polarity differ" % ctx
    if t_tol == 0.0:
        assert np.array_equal(got[:, 0], want[:, 0]), "%s: timestamps differ" % ctx
    else:
        assert np.max(np.abs(got[:, 0] - want[:, 0]), initial=0.0) <= t_tol, "%s: timestamps" % ctx
