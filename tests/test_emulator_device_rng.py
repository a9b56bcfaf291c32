"""GPU: rng_mode="device" pinned to the CPU oracle BIT FOR BIT with leak, shot and photoreceptor noise on.

The device draws its per-frame noise from Philox in-kernel, so torch's generator cannot be replayed. Instead the oracle
is fed the device's own draws (EventEmulator.device_draws, helpers.DeviceDrawRNG): per frame, rows (canonical order:
device rows of one (frame, iteration, polarity) group come in no order), counters and final state must be identical.
This checks the leak with Philox normals, the shot-noise prefix fast reject (a pixel whose 12-bit prefix lies
outside pref_lo of either end is never tested; the oracle tests every pixel), and the Philox frame-index contract:
frame k >= 1 of a clip draws with frame_index k - 1, on every call path. The draws themselves are held against an
independent numpy restatement of the streams (oracle/philox.py).
"""
import collections
import ctypes
import math

import numpy as np
import pytest
import torch

import philox
from helpers import DeviceDrawRNG, assert_events_equal, canonical, run_oracle_with_draws

pytestmark = pytest.mark.gpu

# bench.py's workloads (v2e_args.py:150-204; the 'noisy' preset's rates, emulator.py:525-535)
CLI_DEFAULTS = dict(pos_thres=0.2, neg_thres=0.2, sigma_thres=0.03, cutoff_hz=300.0, leak_rate_hz=0.01,
                    shot_noise_rate_hz=0.001, refractory_period_s=0.0005)
C3_PARAMS = dict(pos_thres=0.2, neg_thres=0.2, sigma_thres=0.03, cutoff_hz=300.0, leak_rate_hz=0.1,
                 shot_noise_rate_hz=5.0, refractory_period_s=0.0005)
SEED = 1234


def texture_frames(H, W, T, seed=0, speed=1.0, block=4):
    rng = np.random.default_rng(seed)
    pad = int(T * speed * 1.5) + 8
    base = rng.integers(0, 256, ((H + pad) // block + 2, (W + pad) // block + 2)).astype(np.uint8)
    big = np.kron(base, np.ones((block, block), np.uint8))
    return np.stack([np.ascontiguousarray(big[int(k * speed * 0.5):int(k * speed * 0.5) + H,
                                              int(k * speed):int(k * speed) + W]) for k in range(T)])


def smooth_clip(H, W, T, seed):
    """bench.py's source texture translating 1 px per frame (what the headline's interpolated frames look like)."""
    from bench import source_clip
    return source_clip(H, W, T, seed=seed, px_per_frame=1)


def _emulator(**kw):
    from v2e_b200 import EventEmulator
    return EventEmulator(device="cuda", rng_mode="device", **kw)


def _state(obj, device):
    names = ("base_log_frame", "lp_log_frame", "timestamp_mem", "photoreceptor_noise_arr", "scidvs_highpass")
    if device:
        vals = [getattr(obj, k) for k in names]
        vals = [None if v is None else v.cpu().numpy() for v in vals]
    else:
        vals = [obj.base, obj.lp, obj.tmem, obj.noise_arr, obj.hp]
    return {k: v for k, v in zip(names, vals) if v is not None}


def run_device(kw, frames, ts, seed=SEED, path="batch", mfps=24, fused=True, rows_hint=None):
    """The CUDA path. Returns (emulator, result); the emulator's handle serves the oracle's draws."""
    em = _emulator(seed=seed, max_frames_per_step=mfps, fused=fused, **kw)
    if rows_hint is not None:
        em.event_rows_hint = rows_hint
    shot = [0, 0]
    account = em._account

    def count_shots(fi):            # per-frame control blocks: shot-noise rows are counted apart from the others
        shot[0] += int(fi.n_shot_on)
        shot[1] += int(fi.n_shot_off)
        account(fi)
    em._account = count_shots
    if path == "frames":
        rows = [canonical(em.generate_events(f, t)) for f, t in zip(frames, ts)]
    else:
        r, o = em.generate_events_batch(frames, ts)
        rows = [canonical(r[o[i]:o[i + 1]]) for i in range(len(frames))]
    a, b = ctypes.c_longlong(0), ctypes.c_longlong(0)
    em._lib.v2e_emu_fused_stats(em._h, ctypes.byref(a), ctypes.byref(b))
    return em, dict(rows=rows, counts=(em.num_events_on, em.num_events_off, em.num_events_total),
                    shot=tuple(shot), chunks=a.value, rejected=b.value, state=_state(em, True))


def draws_from(em, shift=0, perturb=None):
    """Frame k's draws for the oracle: Philox frame index k - 1 (+ shift, for the sensitivity tests)."""
    def get(k):
        d = {name: t.cpu().numpy() for name, t in em.device_draws(k - 1 + shift).items()}
        return perturb(d) if perturb is not None else d
    return get


def run_oracle(em, kw, frames, ts, seed=SEED, **how):
    from emu_oracle import OracleEmulator
    rng = DeviceDrawRNG(draws_from(em, **how), photoreceptor_noise=kw.get("photoreceptor_noise", False))
    orc = OracleEmulator(seed=seed, rng=rng, shuffle=False, **kw)
    rows = run_oracle_with_draws(orc, rng, frames, ts)
    return dict(rows=rows, counts=(orc.num_events_on, orc.num_events_off, orc.num_events_total),
                state=_state(orc, False))


HP_TOL = {np.dtype(np.float64): 4e-15, np.dtype(np.float32): 2e-6}     # CUDA sinh vs libm (test_oracle_golden.py)


def assert_same(dev, ref, ctx):
    assert len(dev["rows"]) == len(ref["rows"])
    for i, (a, b) in enumerate(zip(dev["rows"], ref["rows"])):
        assert_events_equal(a, b, exact_order=True, ctx="%s frame %d" % (ctx, i))
    assert dev["counts"] == ref["counts"], ctx
    assert dev["state"].keys() == ref["state"].keys(), ctx
    for k, want in ref["state"].items():
        got = dev["state"][k]
        assert got.dtype == want.dtype, (ctx, k)
        if k == "scidvs_highpass":
            assert np.max(np.abs(got - want)) <= HP_TOL[got.dtype], (ctx, k)
        else:
            assert np.array_equal(got, want), (ctx, k)


def same(dev, ref):
    try:
        assert_same(dev, ref, "")
        return True
    except AssertionError:
        return False


def rows_changed(a_rows, b_rows):
    """Rows in one run and not the other (multiset symmetric difference over all frames)."""
    n = 0
    for a, b in zip(a_rows, b_rows):
        ca, cb = collections.Counter(map(bytes, a)), collections.Counter(map(bytes, b))
        n += sum(((ca - cb) + (cb - ca)).values())
    return n


def neg_leak(d):
    return dict(d, leak_randn=-d["leak_randn"])


# name: (kwargs, frames/times builder, run options, minimum shot ON, shot OFF, leak-dependent rows)
def _wild_frames(H, W, T):
    rng = np.random.default_rng(6)
    base = texture_frames(H, W, T, seed=6, speed=2.0).astype(np.float32)
    return (base * np.float32(1.3) - np.float32(40) + rng.uniform(0, 1, base.shape).astype(np.float32))


def _hdr_frames(H, W, T):
    return np.log1p(texture_frames(H, W, T, seed=8, speed=2.0).astype(np.float32)).astype(np.float32)


def _refractory_times(T):
    ts = [k * 1e-2 for k in range(T - 1)]
    return ts[:6] + ts[5:]             # frames 5 and 6 share a timestamp (delta_time = 0)


CASES = {
    # thousands of shot events per frame through the prefix reject, FAST kernels (float64, per-pixel thresholds)
    "c3_1280x720": (C3_PARAMS, lambda: (smooth_clip(720, 1280, 9, seed=5), [k / 300. for k in range(9)]),
                    dict(mfps=24), 10000, 10000, 1),
    "c3_346x260": (C3_PARAMS, lambda: (texture_frames(260, 346, 13, seed=2), [k / 300. for k in range(13)]),
                   dict(mfps=24), 2000, 2000, 1),
    # pref_lo saturates at 2048: every pixel is a candidate (and ON and OFF can fire together)
    "shot_saturated_346x260": (dict(C3_PARAMS, shot_noise_rate_hz=200.0),
                               lambda: (texture_frames(260, 346, 6, seed=3), [k * 5e-3 for k in range(6)]),
                               dict(mfps=24), 50000, 50000, 1),
    # non-FAST RNG=1 kernels, partial last quad (n % 4 != 0), the fused kernel's slow loads
    "sigma0_37x53": (dict(sigma_thres=0.0, cutoff_hz=300, leak_rate_hz=20.0, shot_noise_rate_hz=40.0),
                     lambda: (texture_frames(37, 53, 14, seed=4), [k * 5e-3 for k in range(14)]),
                     dict(mfps=24), 20, 20, 1),
    "f32state_37x53": (dict(cutoff_hz=0, leak_rate_hz=20.0, shot_noise_rate_hz=40.0),
                       lambda: (texture_frames(37, 53, 14, seed=5), [k * 5e-3 for k in range(14)]),
                       dict(mfps=24), 20, 20, 1),
    "leak_only_13x37": (dict(cutoff_hz=100, leak_rate_hz=20.0, shot_noise_rate_hz=0.0),
                        lambda: (texture_frames(13, 37, 14, seed=6), [k * 5e-3 for k in range(14)]),
                        dict(mfps=24), 0, 0, 1),
    "shot_only_13x37": (dict(cutoff_hz=100, leak_rate_hz=0.0, shot_noise_rate_hz=100.0),
                        lambda: (texture_frames(13, 37, 14, seed=7), [k * 5e-3 for k in range(14)]),
                        dict(mfps=24), 20, 20, 0),
    # refractory filter active: chunks rejected, back-off, filter kernel, frame-by-frame replay; one dt = 0 frame
    "refractory_64x96": (dict(cutoff_hz=200, leak_rate_hz=5.0, refractory_period_s=0.004, pos_thres=0.05,
                              neg_thres=0.05, sigma_thres=0.01, shot_noise_rate_hz=20.0),
                         lambda: (texture_frames(64, 96, 20, seed=9, speed=3.0), _refractory_times(20)),
                         dict(mfps=8), 20, 20, 1),
    # float32 frames outside [0, 255]: every such pixel is a shot candidate ('wild'); lin_log evaluated
    "wild_float_40x56": (dict(cutoff_hz=100, leak_rate_hz=20.0, shot_noise_rate_hz=40.0),
                         lambda: (_wild_frames(40, 56, 10), [k * 5e-3 for k in range(10)]),
                         dict(mfps=24), 20, 20, 1),
    # log-encoded input
    "hdr_40x56": (dict(hdr=True, cutoff_hz=300, leak_rate_hz=20.0, shot_noise_rate_hz=40.0, pos_thres=0.1,
                       neg_thres=0.1, refractory_period_s=0.001),
                  lambda: (_hdr_frames(40, 56, 10), [k * 5e-3 for k in range(10)]), dict(mfps=24), 20, 20, 1),
    "hdr_nolp_40x56": (dict(hdr=True, cutoff_hz=0, leak_rate_hz=20.0, shot_noise_rate_hz=40.0, pos_thres=0.1,
                            neg_thres=0.1, refractory_period_s=0.001),
                       lambda: (_hdr_frames(40, 56, 10), [k * 5e-3 for k in range(10)]), dict(mfps=24), 20, 20, 1),
    # centre-surround model with leak + shot (f_cs with RNG=1)
    "csdvs_60x80": (dict(cs_lambda_pixels=4, cs_tau_p_ms=0.5, cutoff_hz=100, leak_rate_hz=100.0,
                         shot_noise_rate_hz=200.0, refractory_period_s=1e-3),
                    lambda: (texture_frames(60, 80, 10, seed=10), [k * 5e-4 for k in range(10)]),
                    dict(mfps=24), 20, 20, 1),
    # SCIDVS + photoreceptor noise: the front kernel's Philox draw (shot events come from the noise, none injected)
    "scidvs_prnoise_64x96": (dict(scidvs=True, photoreceptor_noise=True, cutoff_hz=100, shot_noise_rate_hz=5.0,
                                  leak_rate_hz=20.0, pr_vrms_tape=[0.05] * 16),
                             lambda: (texture_frames(64, 96, 12, seed=11), [k * 1e-3 for k in range(12)]),
                             dict(mfps=16), 0, 0, 1),
}


def report(name, dev, leak_dep, extra=""):
    print("DEVRNG %-24s rows=%d shot_on=%d shot_off=%d leak_dependent_rows=%s chunks=%d rejected=%d %s" % (
        name, dev["counts"][2], dev["shot"][0], dev["shot"][1], leak_dep, dev["chunks"], dev["rejected"], extra))


def prefix_margins(em, kw, frames, ts):
    """Shot events the exact test fires, from the device's full uniforms (the oracle's decision, restated): the
    largest 12-bit prefix of a firing OFF uniform and the smallest of a firing ON one, against pref_lo as make_params
    computes it. A non-candidate (pref_lo <= prefix < 4096 - pref_lo) must never fire."""
    pos, neg = em.pos_thres.cpu().numpy(), em.neg_thres.cpu().numpy()
    pre_max = max(kw["pos_thres"], kw["neg_thres"]) / float(min(pos.min(), neg.min()))
    off_max, on_min, los, n_on, n_off = -1, 4096, set(), 0, 0
    for k in range(1, len(frames)):
        dt = ts[k] - ts[k - 1]
        shot_c = (kw["shot_noise_rate_hz"] / 2) * dt
        bound = abs(shot_c) * 1.0 * pre_max * 1.0001 + 1e-300       # intensity factor <= max(0.25, 1) on [0, 255]
        pref_lo = min(math.ceil(bound * 4096.0), 2048)
        los.add(pref_lo)
        r = em.device_draws(k - 1)["shot_u01"].cpu().numpy().astype(np.float64)
        factor = shot_c * ((0.25 - 1) * ((frames[k].astype(np.float64) + 20.0) / 275.0) + 1)
        on = r > 1 - factor * (np.float32(kw["pos_thres"]) / pos).astype(np.float64)
        off = r < factor * (np.float32(kw["neg_thres"]) / neg).astype(np.float64)
        pref = np.floor(r * 4096).astype(np.int64)
        n_on, n_off = n_on + int(on.sum()), n_off + int(off.sum())
        if off.any():
            off_max = max(off_max, int(pref[off].max()))
        if on.any():
            on_min = min(on_min, int(pref[on].min()))
        fired = pref[on | off]
        assert not np.any((fired >= pref_lo) & (fired < 4096 - pref_lo)), (off_max, on_min, pref_lo)
    return dict(pref_lo=sorted(los), off_prefix_max=off_max, on_prefix_min=on_min, fired_on=n_on, fired_off=n_off)


@pytest.mark.parametrize("name", list(CASES))
def test_device_rng_equals_oracle_given_device_draws(name):
    kw, make, opts, min_on, min_off, min_leak = CASES[name]
    frames, ts = make()
    em, dev = run_device(kw, frames, ts, **opts)
    ref = run_oracle(em, kw, frames, ts)
    assert_same(dev, ref, name)
    assert dev["shot"][0] >= min_on and dev["shot"][1] >= min_off, dev["shot"]
    leak_dep = "-"
    if kw.get("leak_rate_hz", 0.1) > 0:
        leak_dep = rows_changed(ref["rows"], run_oracle(em, kw, frames, ts, perturb=neg_leak)["rows"])
        assert leak_dep >= min_leak, leak_dep
    extra = ""
    if name.startswith("c3_") or name.startswith("shot_saturated"):
        m = prefix_margins(em, kw, frames, ts)
        assert (m["pref_lo"] == [2048]) == name.startswith("shot_saturated"), m
        extra = str(m)
    if name == "refractory_64x96":
        assert dev["chunks"] >= 1 and dev["rejected"] >= 1, (dev["chunks"], dev["rejected"])
    report(name, dev, leak_dep, extra)


# ---- headline: v2e's CLI defaults at 1280x720, the FAST fused kernel, count / plan / emit -------------------------
@pytest.fixture(scope="module")
def headline():
    frames, ts = smooth_clip(720, 1280, 25, seed=11), [k / 300. for k in range(25)]   # <= 4 events per pixel and frame
    em, dev = run_device(CLI_DEFAULTS, frames, ts, mfps=24)
    ref = run_oracle(em, CLI_DEFAULTS, frames, ts)
    return dict(em=em, dev=dev, ref=ref, frames=frames, ts=ts)


def test_headline_cli_defaults_1280x720(headline):
    dev, ref = headline["dev"], headline["ref"]
    assert_same(dev, ref, "headline")
    assert dev["chunks"] >= 1 and dev["rejected"] == 0, (dev["chunks"], dev["rejected"])
    assert dev["counts"][2] > 500000
    # shot rate 0.001 Hz: about 20 shot events per polarity in the clip; c3_1280x720 runs the same kernels with
    # tens of thousands
    report("headline_cli_1280x720", dev, "-")


# ---- call paths: the frame-index contract --------------------------------------------------------------------------
@pytest.fixture(scope="module")
def c3():
    kw = C3_PARAMS
    frames, ts = texture_frames(260, 346, 16, seed=12), [k / 300. for k in range(16)]
    em, dev = run_device(kw, frames, ts, mfps=24)
    ref = run_oracle(em, kw, frames, ts)
    return dict(em=em, dev=dev, ref=ref, frames=frames, ts=ts, kw=kw)


@pytest.mark.parametrize("path", ["batch_T", "frames", "batch_1", "batch_7", "unfused", "rows_hint_64"])
def test_call_paths_equal_oracle(c3, path):
    """Same seed, same clip: generate_events frame by frame, generate_events_batch at 1, 7 and all frames per step,
    fused=False, and a 64-row initial event buffer (capacity aborts, growth and resume) must all give the oracle's
    output with frame k drawn at Philox frame index k - 1."""
    frames, ts, kw = c3["frames"], c3["ts"], c3["kw"]
    opts = {"batch_T": dict(mfps=len(frames)), "frames": dict(path="frames"), "batch_1": dict(mfps=1),
            "batch_7": dict(mfps=7), "unfused": dict(fused=False), "rows_hint_64": dict(rows_hint=64)}[path]
    em, dev = run_device(kw, frames, ts, **opts)
    assert_same(dev, c3["ref"], path)
    if path in ("batch_T", "batch_7"):
        assert dev["chunks"] >= 1
    if path in ("unfused", "frames", "batch_1"):
        assert dev["chunks"] == 0
    report("c3_346x260_" + path, dev, "-")


@pytest.mark.parametrize("perturb", ["next_frame_index", "negated_leak", "neighbour_shot"])
def test_comparison_fails_when_only_the_oracle_draws_change(c3, perturb):
    """The comparison is sensitive to each draw: perturbing only the oracle's draws must break it."""
    em, frames, ts, kw = c3["em"], c3["frames"], c3["ts"], c3["kw"]
    assert same(c3["dev"], c3["ref"])
    how = {"next_frame_index": dict(shift=1), "negated_leak": dict(perturb=neg_leak),
           "neighbour_shot": dict(perturb=lambda d: dict(d, shot_u01=np.roll(d["shot_u01"].ravel(), 1)
                                                          .reshape(d["shot_u01"].shape)))}[perturb]
    bad = run_oracle(em, kw, frames, ts, **how)
    assert not same(c3["dev"], bad)
    print("DEVRNG sensitivity %s: %d rows differ" % (perturb, rows_changed(c3["dev"]["rows"], bad["rows"])))


# ---- the draws themselves ------------------------------------------------------------------------------------------
def test_pixel_offset_draws_the_matching_slice():
    """A row band of an odd-width frame starts in the middle of a Philox quad (noise_px4_unaligned): its leak and shot
    draws must be exactly the band's slice of the whole frame's. The photoreceptor stream counts LOCAL quads."""
    H, W, y0, y1 = 37, 53, 13, 29                     # rng_pixel_offset 689 = 4 * 172 + 1
    full, band = _emulator(seed=SEED, **C3_PARAMS), _emulator(seed=SEED, **C3_PARAMS)
    full._create(H, W)
    band._create(y1 - y0, W, px_offset=y0 * W)
    for fi in (0, 7):
        a, b = full.device_draws(fi), band.device_draws(fi)
        assert torch.equal(b["leak_randn"], a["leak_randn"][y0:y1])
        assert torch.equal(b["shot_u01"], a["shot_u01"][y0:y1])
        assert torch.equal(b["pr_randn"], a["pr_randn"][:y1 - y0])
        assert np.array_equal(b["shot_u01"].cpu().numpy().ravel(),
                              philox.shot_u01(SEED, (y1 - y0) * W, fi, px_off=y0 * W))


def _polar(nrm):
    """radius^2 and angle in [0, 2pi) of each Box-Muller pair (pixels 0, 1 and 2, 3 of a quad)."""
    q = nrm.astype(np.float64).reshape(-1, 2)
    return (q ** 2).sum(1), np.mod(np.arctan2(q[:, 1], q[:, 0]), 2 * np.pi)


def _assert_polar_close(nrm, u, ang, what):
    r2, a = _polar(nrm)
    r2_ref = -2.0 * np.log(u.reshape(-1, 2)[:, 0].astype(np.float64))
    a_ref = ang.reshape(-1, 2)[:, 0].astype(np.float64)
    assert np.all(np.abs(r2 - r2_ref) <= 1e-5 * np.maximum(r2_ref, 1.0)), what
    ok = r2_ref > 1e-6                                  # the angle of a (near-)zero radius is not recoverable
    da = np.abs(np.mod(a[ok] - a_ref[ok] + np.pi, 2 * np.pi) - np.pi)
    assert np.all(da <= 1e-5 * np.maximum(a_ref[ok], 1.0)), (what, da.max())


def test_device_stream_matches_numpy_restatement_1280x720():
    """Seed above 2^32 (the key's high word matters). Shot uniforms bit for bit; the normals' Box-Muller radius^2
    and angle within 1e-5 relative (floor 1: __logf / __sincosf are accurate in absolute terms); moments of
    3.7 M samples within 5 sigma of N(0, 1) / U(0, 1); frame indices and streams give different fields."""
    H, W = 720, 1280
    n = H * W
    seed = (0x9E3779B9 << 32) | 0x7F4A7C15
    em = _emulator(**CLI_DEFAULTS)
    em.seed = seed                                       # (np.random.seed would refuse it in the constructor)
    em._create(H, W)
    fis = (0, 1, 2, 1000)
    d = {fi: {k: v.cpu().numpy().ravel() for k, v in em.device_draws(fi).items()} for fi in fis}
    for fi in (0, 1000):
        want = philox.shot_u01(seed, n, fi)
        assert np.array_equal(d[fi]["shot_u01"].view(np.uint32), want.view(np.uint32)), fi
    for fi in (0, 1):
        u, ang, _, _ = philox.leak_fields(seed, n, fi)
        _assert_polar_close(d[fi]["leak_randn"], u, ang, "leak %d" % fi)
        u, ang, _ = philox.pr_fields(seed, n, fi)
        _assert_polar_close(d[fi]["pr_randn"], u, ang, "photoreceptor %d" % fi)
    for key in ("leak_randn", "pr_randn"):
        x = np.concatenate([d[fi][key] for fi in fis]).astype(np.float64)
        N = len(x)
        assert N >= 3_600_000
        for m, (mu, var) in zip((x.mean(), (x ** 2).mean(), (x ** 3).mean(), (x ** 4).mean()),
                                ((0, 1), (1, 2), (0, 15), (3, 96))):
            assert abs(m - mu) < 5 * math.sqrt(var / N), (key, m, mu)
    u = np.concatenate([d[fi]["shot_u01"] for fi in fis]).astype(np.float64)
    assert u.min() >= 0 and u.max() < 1
    assert abs(u.mean() - 0.5) < 5 * math.sqrt(1 / 12 / len(u))
    assert abs(((u - 0.5) ** 2).mean() - 1 / 12) < 5 * math.sqrt(1 / 180 / len(u))
    eq = lambda a, b: np.mean(a == b)
    for a, b in ((0, 1), (1, 2), (0, 1000)):
        for key in ("leak_randn", "shot_u01", "pr_randn"):
            assert eq(d[a][key], d[b][key]) < 1e-3, (a, b, key)
    assert eq(d[0]["leak_randn"], d[0]["pr_randn"]) < 1e-3
    shot_bits = (d[0]["shot_u01"].astype(np.float64) * 2.0 ** 32).astype(np.uint64) & np.uint64(0xFFF00)
    leak_w = philox.philox4x32((np.arange(n) >> 2, np.zeros(n), np.zeros(n), np.full(n, philox.TAG_LEAK)),
                               philox.seed_key(seed))
    leak_bits = (np.choose(np.arange(n) & 3, leak_w).astype(np.uint64) >> np.uint64(12)) & np.uint64(0xFFF00)
    assert eq(shot_bits, leak_bits) < 0.01                  # the shot stream is not the leak stream's words
    assert not np.array_equal(d[0]["shot_u01"], philox.shot_u01(seed & 0xFFFFFFFF, n, 0))
