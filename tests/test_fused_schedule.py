"""The multi-frame pixel-model path's control decisions, checked at their edges against the oracle.

generate_events_batch runs a chunk of up to max_frames_per_step frames speculatively through the multi-frame kernels
(per-pixel state in registers), then the plan kernel accepts or rejects it frame by frame: frame f is rejected when its
maximum count max_n exceeds kFusedMaxN (31) or iter_cap, or when the refractory filter would run
(refractory_period_s > dt / max_n). v2e_emu_collect then re-schedules the chunk: rejected frames frame by frame, runs of
two or more good frames through the multi-frame kernels again, a lone good frame with its frame-by-frame neighbours;
the maxima after a rejected frame are predictions from a speculative state, so a run can be rejected again. A chunk
with many bad frames makes the next 1, 2, 4 ... 64 chunks run frame by frame (back-off).

The clips here are a static background with planted pixels whose code jumps give a CHOSEN max_n in chosen frames:
31 / 32 (the accept / reject edge), 63, 64 and 100 (past the 6-bit record clamp), 8 / 9 at refractory_period_s =
dt / 8 on dyadic times, and bad frames first, last, in the middle, adjacent, around a lone good frame, in a 2-frame
chunk and in a trailing 1-frame chunk. The codes are planned with a numpy restatement of the oracle's arithmetic
(lin_log table, float32 / float64 difference, ATen floor division, the refractory filter on the planted pixels);
the CPU tests hold the oracle to that plan. On the GPU the device-RNG path must equal the oracle fed the device's own
Philox draws bit for bit (tests/test_emulator_device_rng.py), report the planned maxima, and run the schedule a Python
restatement of v2e_emu_collect's rule predicts.
"""
import ctypes

import numpy as np
import pytest
import torch

from helpers import DeviceDrawRNG, canonical
from test_emulator_device_rng import assert_same, draws_from, same, _state

H, W = 64, 96
DT = 2.0 ** -8                 # dyadic frame times k * 2^-8 s: dt / max_n is exact for max_n a power of two
SEED = 4321
FUSED_MAX_N = 31               # kFusedMaxN in emu.cu
REC_CLAMP = 63                 # the record's 6-bit event count (make_rec16)

# Thresholds of 0.04 so that one code jump (lin_log(255) = 5.54) reaches ~100 events. Leak (0.2 Hz: at most ~0.1
# threshold of drift over a clip) and shot noise (0.5 Hz) are what the planner does not model: every planned count has
# a quotient at least 0.3 away from an integer. cutoff_hz = 1e4 keeps the state float64 with an exact low-pass:
# eps = inten01 * dt * 2 pi * cutoff >= 17 clamps to 1 at dt = 2^-8, so lp = lin_log(code).
CONFIGS = {
    "f32_scalar": dict(pos_thres=0.04, neg_thres=0.04, sigma_thres=0.0, cutoff_hz=0, leak_rate_hz=0.0,
                       shot_noise_rate_hz=0.0),
    "f32_leak_shot": dict(pos_thres=0.04, neg_thres=0.04, sigma_thres=0.003, cutoff_hz=0, leak_rate_hz=0.2,
                          shot_noise_rate_hz=0.5),
    "f64_fast": dict(pos_thres=0.04, neg_thres=0.04, sigma_thres=0.003, cutoff_hz=1e4, leak_rate_hz=0.2,
                     shot_noise_rate_hz=0.5),
    "f64_scalar": dict(pos_thres=0.04, neg_thres=0.04, sigma_thres=0.0, cutoff_hz=1e4, leak_rate_hz=0.0,
                       shot_noise_rate_hz=0.0),
}


def _heavy(f):
    """Bad frames f and f + 2 of a 4-frame chunk [f, f + 4): the good frames f + 1 and f + 3 are lone, so the whole
    chunk goes frame by frame, and 4 * 2 bad > 4 engages the back-off."""
    return [(f, 40, 1), (f + 2, 40, -1)]


# name: dict(T, mfps, bursts [(frame, events, +1 ON / -1 OFF[, row range])], refr, targets: maxima the clip must
# reach, exact: the speculative maxima are exact (no refractory filter), so the schedule is restated exactly;
# one_round: the speculative maxima after a filtered frame are not exact, but they are bad exactly where the real ones
# are, so every chunk still takes one rejection round and the schedule is restated exactly too)
DESIGNS = {
    # chunks [1, 9) [9, 17): 31 in the first and the last frame of a chunk, all accepted
    "deep_accept": dict(T=17, mfps=8, bursts=[(1, 31, 1), (3, 7, 1), (3, 3, -1), (5, 16, 1), (8, 31, -1),
                                              (10, 30, 1), (12, 3, 1), (14, 31, 1), (16, 31, -1)],
                        targets={3, 7, 16, 30, 31}, exact=True),
    # chunks [1, 9): bad first (32) and last (64) frame; [9, 17): bad middle frame (100); [17, 25): adjacent bad frames
    # 19, 20 and a lone good frame 21 before bad 22; [25, 26): a trailing 1-frame chunk (never multi-frame)
    "count_reject": dict(T=26, mfps=8, bursts=[(1, 32, 1), (5, 31, 1), (8, 64, -1), (10, 30, 1), (12, 100, 1),
                                               (14, 31, -1), (19, 100, 1), (20, 64, -1), (21, 7, 1), (22, 32, 1),
                                               (24, 31, 1), (25, 100, -1)],
                         targets={31, 32, 64, 100}, exact=True),
    # 2-frame chunks [1, 3) [3, 5) ... [11, 13), then a trailing 1-frame chunk [13, 14): a bad last frame (c1) and a
    # bad first frame (c3) send a whole chunk frame by frame (the lone good frame merges) and back off for 1, then 2
    # chunks (c2; c4 and c5)
    "two_frame": dict(T=14, mfps=2, bursts=[(2, 31, 1), (4, 32, -1), (6, 63, 1), (7, 64, -1), (10, 31, 1),
                                            (12, 31, -1), (13, 100, 1)],
                      targets={31, 32, 63, 64, 100}, exact=True),
    # max_n = 25 in a multi-frame chunk: iter_cap = 25 accepts it, iter_cap = 20 must fail
    "iter_cap": dict(T=9, mfps=8, bursts=[(2, 7, 1), (4, 25, -1), (6, 3, 1)], targets={25}, exact=True),
    # H = 64 over 2 ranks: rank 1 owns rows [32, 64). Frame 3: 40 events in rank 1's rows, 31 in rank 0's; frame 9,
    # with refractory_period_s = dt / 8: 9 events in rank 1's rows, 8 in rank 0's. Rank 0's own maxima accept both.
    "band_count": dict(T=13, mfps=6, bursts=[(3, 40, 1, (32, 64)), (3, 31, -1, (0, 32)), (5, 16, 1, (0, 32))],
                       targets={16, 40}, exact=True),
    "band_refr": dict(T=13, mfps=6, refr=2.0 ** -11,
                      bursts=[(9, 9, -1, (32, 64)), (9, 8, 1, (0, 32)), (2, 8, 1, (32, 64))],
                      targets={4, 8, 9}, exact=False, one_round=True),
    # 4-frame chunks c0 .. c13: heavy chunks c0, c2, c5 back off for 1, 2, 4 chunks; the quiet chunk c10 is accepted
    # whole and releases the back-off, so the heavy c11 backs off for 1 chunk only (c12, heavy, is skipped) and the
    # quiet c13 is tried and accepted. Without the release c11 would back off for 8 chunks and c13 be skipped too.
    "backoff": dict(T=57, mfps=4, bursts=_heavy(1) + [(6, 50, 1)] + _heavy(9) + [(14, 50, -1)] + _heavy(21) +
                    [(26, 50, 1), (33, 40, -1)] + [(42, 31, 1)] + _heavy(45) + _heavy(49) + [(54, 31, -1)],
                    targets={31, 40, 50}, exact=True),
    # refractory_period_s = 2^-11 = dt / 8: max_n = 8 leaves the filter off (accepted), max_n = 9 turns it on (rejected,
    # replayed; the filter drops 4 of the 9 events, the next frame emits them)
    "refr_boundary": dict(T=17, mfps=8, refr=2.0 ** -11,
                          bursts=[(2, 8, 1), (5, 9, 1), (10, 8, -1), (12, 9, -1), (15, 8, 1)],
                          targets={4, 8, 9}, exact=False, one_round=True),
    # refractory_period_s = 0.3 dt: frames with max_n >= 4 are bad. Frame 5's 12 events pass 3 at a time; the
    # speculative state predicts nothing after it, the replayed state gives 9, 6, 3 events in frames 6, 7, 8: the
    # chunk is rejected in three rounds
    "second_round": dict(T=17, mfps=16, refr=0.3 * DT, bursts=[(5, 12, 1)], targets={12, 9, 6, 3}, exact=False),
}
# the count-limited clip at other chunk lengths: bursts land on other chunk edges
for _m in (5, 16):
    DESIGNS["count_reject_m%d" % _m] = dict(DESIGNS["count_reject"], mfps=_m)


# ---- the planner: a numpy restatement of the oracle's arithmetic on the planted pixels -----------------------------
def _lut():
    from emu_oracle import linlog_lut
    return linlog_lut()


def div_floor(a, b):
    """ATen's div_floor_floating for a >= 0, b > 0, in the dtype of a and b (emu_oracle.c div_floor_f32 / _f64)."""
    mod = np.fmod(a, b)
    div = (a - mod) / b
    if div == 0:
        return 0
    fl = np.floor(div)
    if div - fl > 0.5:
        fl += 1
    return int(fl)


def thresholds(kw, seed):
    """The per-pixel thresholds the emulator and the oracle draw first from torch's generator seeded with `seed`
    (normal(pos), normal(neg), clamped at 0.01); the nominal ones as float32 fields when sigma_thres = 0."""
    if kw["sigma_thres"] <= 0:
        return (np.full((H, W), kw["pos_thres"], np.float32), np.full((H, W), kw["neg_thres"], np.float32))
    g = torch.Generator().manual_seed(seed)
    pos = torch.clamp(torch.normal(kw["pos_thres"], kw["sigma_thres"], size=(H, W), generator=g), min=0.01)
    neg = torch.clamp(torch.normal(kw["neg_thres"], kw["sigma_thres"], size=(H, W), generator=g), min=0.01)
    return pos.numpy(), neg.numpy()


class _Px:
    """One planted pixel's arithmetic: state dtype S, its float32 thresholds and the divisor the oracle uses."""

    def __init__(self, kw, thp, thn):
        self.S = np.float64 if kw["cutoff_hz"] > 0 else np.float32
        self.thp, self.thn = np.float32(thp), np.float32(thn)
        scalar64 = self.S is np.float64 and kw["sigma_thres"] <= 0     # a Python-float threshold stays float64
        self.bp = self.S(kw["pos_thres"]) if scalar64 else self.S(self.thp)
        self.bn = self.S(kw["neg_thres"]) if scalar64 else self.S(self.thn)

    def count(self, lp, base):
        diff = lp - base
        return (div_floor(diff, self.bp), 1) if diff > 0 else (div_floor(-diff, self.bn), -1) if diff < 0 else (0, 1)

    def moved(self, base, passed, sign):
        """base after `passed` events: int32 * float32 threshold -> float32, then the state's dtype."""
        return base + self.S(np.float32(passed) * (self.thp if sign > 0 else self.thn)) * sign


def pick_codes(px, n, sign, lut):
    """(c0, c1): a jump from code c0 to c1 that gives exactly n events of polarity `sign` from base = lin_log(c0), with
    the quotient's fractional part in [0.3, 0.7] (closest to 0.5)."""
    l = lut.astype(px.S)
    d = (l[None, :] - l[:, None]) * px.S(sign)                      # [c0, c1]
    q = d.astype(np.float64) / float(px.bp if sign > 0 else px.bn)
    frac = q - np.floor(q)
    ok = (np.floor(q) == n) & (frac >= 0.3) & (frac <= 0.7)
    assert ok.any(), "no code jump gives %d events" % n
    c0, c1 = np.unravel_index(np.argmin(np.where(ok, np.abs(frac - 0.5), np.inf)), ok.shape)
    got, s = px.count(l[c1], l[c0])
    assert (got, s) == (n, sign), (n, sign, got, s)
    return int(c0), int(c1)


def simulate(pixels, codes, ts, refr, lut, filter_on=True):
    """Per-frame maxima of the planted pixels (the static background makes none) under the oracle's arithmetic.
    The refractory filter is restated for them in float64 time (the clips' decisions are >= 10 % of the period away
    from a tie). filter_on=False gives what the speculative multi-frame pass predicts."""
    base = [px.S(lut[c[0]]) for px, c in zip(pixels, codes)]
    tmem = [float(np.float32(-refr))] * len(pixels)
    plan = [None]
    for k in range(1, len(ts)):
        dt = ts[k] - ts[k - 1]
        cnt = [px.count(px.S(lut[c[k]]), b) for px, c, b in zip(pixels, codes, base)]
        m = max([n for n, _ in cnt], default=0)
        plan.append(m)
        step = dt / max(m, 1)
        active = filter_on and refr > step
        for i, (px, (n, s)) in enumerate(zip(pixels, cnt)):
            passed = 0
            for it in range(n):
                t = ts[k - 1] + (it + 1) * step
                if not active or t - tmem[i] > refr:
                    passed += 1
                    if active:
                        tmem[i] = t
            base[i] = px.moved(base[i], passed, s)
    return plan


def build(design, config, seed=SEED, rows=(0, H)):
    """-> (emulator / oracle keywords, frames [T, H, W] uint8, times, plan, speculative plan). rows: plant only the
    bursts inside these rows (what one band of a sharded clip sees)."""
    from bench import source_clip
    d = DESIGNS[design]
    kw = dict(CONFIGS[config], refractory_period_s=d.get("refr", 0.0))
    T, lut = d["T"], _lut()
    pos, neg = thresholds(kw, seed)
    frames = np.repeat(source_clip(H, W, 1, seed=7, px_per_frame=0)[0][None], T, 0)
    pixels, codes = [], []
    for k, b in enumerate(d["bursts"]):
        f, n, sign = b[:3]
        r0, r1 = b[3] if len(b) > 3 else (0, H)
        if r0 < rows[0] or r1 > rows[1]:
            continue
        y, x = r0 + 2 + 4 * (k // 15), 3 + 6 * (k % 15)
        px = _Px(kw, pos[y, x], neg[y, x])
        c0, c1 = pick_codes(px, n, sign, lut)
        frames[:f, y, x], frames[f:, y, x] = c0, c1
        pixels.append(px)
        codes.append(frames[:, y, x].copy())
    ts = [k * DT for k in range(T)]
    refr = kw["refractory_period_s"]
    return (kw, frames, ts, simulate(pixels, codes, ts, refr, lut),
            simulate(pixels, codes, ts, refr, lut, filter_on=False))


def bad_frame(m, dt, refr, limit=FUSED_MAX_N, iter_cap=1024):
    """v2e_emu_collect's (and the plan kernel's) predicate."""
    return m > limit or m > iter_cap or (refr > 0 and m > 0 and refr > dt / m)


def restatable(design):
    return DESIGNS[design]["exact"] or DESIGNS[design].get("one_round", False)


def restate_schedule(maxima, ts, mfps, refr=0.0, limit=FUSED_MAX_N, iter_cap=1024, release=True):
    """generate_events_batch + v2e_emu_step + v2e_emu_collect, restated for maxima the speculative pass predicts
    exactly (one rejection round per chunk): frame 0 initialises, then chunks of mfps frames; a chunk of >= 2 frames
    is tried multi-frame unless the back-off skips it; on a rejection, runs of >= 2 good frames go multi-frame, bad
    frames and lone good frames frame by frame; 4 * bad frames > chunk length backs off for 1, 2, 4 ... 64 chunks; a
    chunk accepted whole releases it (release=False: never, for the sensitivity checks).
    -> (chunks, rejected, frames_multi, frames_single)."""
    chunks = rejected = multi = single = 0
    skip = penalty = 0
    f = 1
    while f < len(maxima):
        e = min(len(maxima), f + mfps)
        if e - f >= 2 and skip:
            skip -= 1
        elif e - f >= 2:
            chunks += 1
            bad = [bad_frame(maxima[q], ts[q] - ts[q - 1], refr, limit, iter_cap) for q in range(f, e)]
            if not any(bad):
                multi += e - f
                if release:
                    penalty = 0
            else:
                rejected += 1
                q = 0
                while q < e - f:
                    r = q
                    while r < e - f and bad[r] == bad[q]:
                        r += 1
                    if not bad[q] and r - q >= 2:
                        multi += r - q
                    else:
                        single += r - q
                    q = r
                if 4 * sum(bad) > e - f:
                    penalty = min(2 * penalty, 64) if penalty else 1
                    skip = penalty
        f = e
    return chunks, rejected, multi, single


# ---- CPU: the designs reach their planned maxima in the oracle ----------------------------------------------------
def oracle_maxima(kw, frames, ts, seed=SEED, rng=None):
    from emu_oracle import OracleEmulator
    orc = OracleEmulator(seed=seed, rng=rng, shuffle=False, **kw)
    rows, maxima = [], [None]
    for k, (f, t) in enumerate(zip(frames, ts)):
        if rng is not None:
            rng.frame = k
        rows.append(canonical(orc.generate_events(f, float(t))))
        if k:
            maxima.append(orc.last_max_n)
    return orc, rows, maxima


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("design", list(DESIGNS))
def test_designed_clip_reaches_planned_maxima(design, config):
    kw, frames, ts, plan, spec = build(design, config)
    _, _, maxima = oracle_maxima(kw, frames, ts)
    assert maxima == plan, (design, config, maxima, plan)
    assert DESIGNS[design]["targets"] <= set(plan[1:]), (design, sorted(set(plan[1:])))
    if DESIGNS[design]["exact"]:
        assert spec == plan
    if restatable(design):
        refr = kw["refractory_period_s"]
        assert [bad_frame(m, DT, refr) for m in spec[1:]] == [bad_frame(m, DT, refr) for m in plan[1:]], (plan, spec)
    if design == "refr_boundary":
        dt8 = [k for k in range(1, len(plan)) if plan[k] == 8]
        assert dt8 and all(not bad_frame(8, ts[k] - ts[k - 1], kw["refractory_period_s"]) for k in dt8)
        assert all(bad_frame(9, ts[k] - ts[k - 1], kw["refractory_period_s"]) for k in range(1, len(plan)))
    if design == "second_round":
        assert plan[5:9] == [12, 9, 6, 3] and spec[5:9] == [12, 0, 0, 0], (plan, spec)


def test_schedule_restatement_reaches_every_branch():
    """The restated schedules of the count-limited clips: first / last / middle / adjacent bad frames, lone-frame
    merging, whole frame-by-frame chunks, the back-off doubling and released, the refractory clips; and the 31 / 32
    edge and the release move them."""
    def sched(design, **how):
        kw, frames, ts, plan, _ = build(design, "f32_scalar")
        return restate_schedule(plan, ts, DESIGNS[design]["mfps"], kw["refractory_period_s"], **how)
    assert sched("deep_accept") == (2, 0, 16, 0)
    # [1] [2, 8) [8] | [9, 12) [12] [13, 17) | [17, 19) [19, 23) [23, 25) | trailing [25] (not counted)
    assert sched("count_reject") == (3, 3, 6 + 7 + 4, 2 + 1 + 4)
    # c0 accepted | c1 frame by frame, backs off | c2 skipped | c3 frame by frame, backs off for 2 | c4, c5 skipped
    assert sched("two_frame") == (3, 2, 2, 4)
    # attempted: c0 c2 c5 (heavy), c10 (quiet, accepted), c11 (heavy), c13 (quiet, accepted); skipped: c1, c3 c4,
    # c6 .. c9, c12
    assert sched("backoff") == (6, 4, 8, 16)
    # without the release c11 backs off for 8 chunks: c12 and c13 are skipped
    assert sched("backoff", release=False) == (5, 4, 4, 16)
    # [1, 5) [5] [6, 9) | [9, 12) [12] [13, 17)
    assert sched("refr_boundary") == (2, 2, 14, 2)
    for design in ("count_reject", "two_frame"):
        assert sched(design, limit=30) != sched(design) != sched(design, limit=32)


# ---- GPU: the device-RNG multi-frame path against the oracle ------------------------------------------------------
def _stats(em):
    L, h = em._lib, em._h
    a, b, c, d = (ctypes.c_longlong(0) for _ in range(4))
    L.v2e_emu_fused_stats(h, ctypes.byref(a), ctypes.byref(b))
    L.v2e_emu_fused_frames(h, ctypes.byref(c), ctypes.byref(d))
    fr, mx = ctypes.c_int(-1), ctypes.c_int(-1)
    L.v2e_emu_fused_last_reject(h, ctypes.byref(fr), ctypes.byref(mx))
    return dict(chunks=a.value, rejected=b.value, multi=c.value, single=d.value, last_reject=(fr.value, mx.value))


def run_device(kw, frames, ts, mfps, rows_hint=None, iter_cap=1024, seed=SEED):
    """generate_events_batch on the device RNG; every frame's control block (max_n, filter_active) is kept, and every
    capacity abort: _run_step grows the event buffer with keep= and resumes the step, and whether the step's chunk
    had been rejected (re-scheduled) by then."""
    from v2e_b200 import EventEmulator
    em = EventEmulator(device="cuda", rng_mode="device", seed=seed, max_frames_per_step=mfps, iter_cap=iter_cap, **kw)
    if rows_hint is not None:
        em.event_rows_hint = rows_hint
    seen = []
    account = em._account

    def keep(fi):
        seen.append((int(fi.max_n), int(fi.filter_active)))
        account(fi)
    em._account = keep
    resumes, rejected_before = [], [0]
    run_step, grow = em._run_step, em._grow_event_buffer

    def step_probe(*a, **k):
        rejected_before[0] = _stats(em)["rejected"]
        return run_step(*a, **k)

    def grow_probe(rows, **k):
        if "keep" in k:
            resumes.append(_stats(em)["rejected"] > rejected_before[0])
        return grow(rows, **k)
    em._run_step, em._grow_event_buffer = step_probe, grow_probe
    r, o = em.generate_events_batch(frames, ts)
    rows = [canonical(r[o[i]:o[i + 1]]) for i in range(len(frames))]
    return em, dict(rows=rows, counts=(em.num_events_on, em.num_events_off, em.num_events_total),
                    state=_state(em, True), maxima=[None] + [m for m, _ in seen],
                    filter=[None] + [a for _, a in seen], resumes=resumes, **_stats(em))


def run_oracle(em, kw, frames, ts):
    rng = DeviceDrawRNG(draws_from(em))
    orc, rows, maxima = oracle_maxima(kw, frames, ts, rng=rng)
    return dict(rows=rows, counts=(orc.num_events_on, orc.num_events_off, orc.num_events_total),
                state=_state(orc, False), maxima=maxima)


def report(name, dev, extra=""):
    print("FUSED %-34s maxima=%s chunks=%d rejected=%d frames_multi=%d frames_single=%d last_reject=%s rows=%d %s" % (
        name, sorted(set(dev["maxima"][1:])), dev["chunks"], dev["rejected"], dev["multi"], dev["single"],
        dev["last_reject"], dev["counts"][2], extra))


def check_against_oracle(design, config, **run):
    kw, frames, ts, plan, _ = build(design, config)
    mfps = DESIGNS[design]["mfps"]
    em, dev = run_device(kw, frames, ts, mfps, **run)
    ref = run_oracle(em, kw, frames, ts)
    ctx = "%s/%s" % (design, config)
    assert_same(dev, ref, ctx)
    assert dev["maxima"] == ref["maxima"] == plan, (ctx, dev["maxima"], plan)
    refr = kw["refractory_period_s"]
    want_filter = [None] + [int(refr > (ts[k] - ts[k - 1]) / max(plan[k], 1)) for k in range(1, len(plan))]
    assert dev["filter"] == want_filter, (ctx, dev["filter"])
    return kw, frames, ts, plan, em, dev, ref


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("design", list(DESIGNS))
def test_multi_frame_path_equals_oracle(design, config):
    """Rows (canonical order, per frame), counters and state bit for bit; every frame's max_n and filter_active as
    planned; for the clips that take one rejection round per chunk the schedule v2e_emu_collect ran is the restated
    one."""
    kw, frames, ts, plan, em, dev, ref = check_against_oracle(design, config)
    d = DESIGNS[design]
    if restatable(design):
        assert (dev["chunks"], dev["rejected"], dev["multi"], dev["single"]) == \
            restate_schedule(plan, ts, d["mfps"], kw["refractory_period_s"]), (design, config, dev)
    if design == "count_reject":
        # the last rejection is frame 19 of the step [17, 25) (slot 2): 100 events, the record holds 63
        assert dev["last_reject"] == (2, REC_CLAMP), dev["last_reject"]
    if design == "second_round":
        # one chunk [1, 17), rejected at frame 5, then at 6 and 7 (predicted 0 events, replayed state 9 and 6)
        assert dev["chunks"] == 1 and dev["rejected"] == 3, dev
        assert dev["last_reject"] == (7 - 1, 6), dev["last_reject"]
    report("%s/%s" % (design, config), dev)


@pytest.mark.gpu
def test_schedule_comparison_fails_at_a_neighbouring_limit():
    """The schedule check is sensitive to the limit and to the back-off release: restated with 30 or 32 instead of
    31, the observed schedule of a clip with 31 and 32 events in its frames no longer matches; restated without the
    release, the back-off clip's no longer matches."""
    for design, changes in (("count_reject", [dict(limit=30), dict(limit=32)]),
                            ("two_frame", [dict(limit=30), dict(limit=32)]), ("backoff", [dict(release=False)])):
        kw, frames, ts, plan, _ = build(design, "f64_fast")
        mfps = DESIGNS[design]["mfps"]
        em, dev = run_device(kw, frames, ts, mfps)
        got = (dev["chunks"], dev["rejected"], dev["multi"], dev["single"])
        assert got == restate_schedule(plan, ts, mfps)
        for how in changes:
            assert got != restate_schedule(plan, ts, mfps, **how), (design, how)
        report("sensitivity/%s" % design, dev)


@pytest.mark.gpu
@pytest.mark.parametrize("design", ["count_reject", "second_round", "backoff"])
def test_capacity_growth_inside_rescheduled_chunks(design):
    """A 64-row initial event buffer: capacity aborts land inside re-scheduled segments (resume_emit); the output and
    the schedule equal the unconstrained run's."""
    kw, frames, ts, plan, em, dev, ref = check_against_oracle(design, "f64_fast", rows_hint=64)
    _, full = run_device(kw, frames, ts, DESIGNS[design]["mfps"])
    # the first step's chunk is rejected and its rows exceed 64: a capacity abort after the re-scheduling
    assert any(dev["resumes"]) and not full["resumes"], (dev["resumes"], full["resumes"])
    assert same(dev, full)
    for k in ("chunks", "rejected", "multi", "single", "last_reject", "maxima"):
        assert dev[k] == full[k], (k, dev[k], full[k])
    report("rows_hint_64/%s" % design, dev, "resumes=%d in_rescheduled=%d" % (len(dev["resumes"]),
                                                                            sum(dev["resumes"])))


@pytest.mark.gpu
def test_iter_cap_in_the_batch_path():
    """max_n = 25 in a multi-frame chunk: iter_cap = 25 accepts it (oracle output); iter_cap = 20 rejects the chunk,
    replays the frame and fails with V2E_E_ITER_CAP instead of returning truncated rows."""
    from v2e_b200 import _lib
    kw, frames, ts, plan, em, dev, ref = check_against_oracle("iter_cap", "f64_fast", iter_cap=25)
    assert max(plan[1:]) == 25
    assert (dev["chunks"], dev["rejected"], dev["multi"], dev["single"]) == (1, 0, 8, 0), dev
    report("iter_cap_25", dev)
    with pytest.raises(_lib.V2eError) as e:
        run_device(kw, frames, ts, 8, iter_cap=20)
    assert e.value.code == _lib.V2E_E_ITER_CAP


# ---- GPU: a burst only one band of a pixel-sharded clip sees -------------------------------------------------------
BAND_DESIGNS = ("band_count", "band_refr")


def _sharded_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from v2e_b200 import EventEmulator
        from v2e_b200.parallel import row_band
        out = {}
        for name in BAND_DESIGNS:
            kw, frames, ts, _, _ = build(name, "f64_fast")
            em = EventEmulator(device="cuda:0", seed=SEED, rng_mode="device", shard=(rank, world, None),
                               max_frames_per_step=DESIGNS[name]["mfps"], **kw)
            y0, y1 = row_band(H, rank, world)
            rows, offs = em.generate_events_band_batch(np.ascontiguousarray(frames[:, y0:y1]), ts, H)
            out[name] = (rows, offs, _stats(em))
            em.cleanup()
        q.put((rank, out))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_band_local_burst_rejected_on_every_rank():
    """2 gloo ranks on one GPU. The all-reduced frame maxima, not a band's own, decide: both ranks reject the frame
    that only rank 1's rows make bad, report the same rejection, and their rows together are the single-GPU run's
    (itself equal to the oracle), frame by frame."""
    import socket
    import torch.multiprocessing as mp
    from helpers import assert_events_equal
    from v2e_b200.parallel import row_band
    want = {}
    for name in BAND_DESIGNS:
        kw, frames, ts, plan, em, dev, ref = check_against_oracle(name, "f64_fast")
        refr = kw["refractory_period_s"]
        own0 = build(name, "f64_fast", rows=row_band(H, 0, 2))[3]
        assert not any(bad_frame(m, DT, refr) for m in own0[1:]), (name, own0)
        want[name] = (dev, plan, [k for k in range(1, len(plan)) if bad_frame(plan[k], DT, refr)])
        assert want[name][2], (name, plan)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for name, (dev, plan, bad_at) in want.items():
        for i in range(DESIGNS[name]["T"]):
            got = np.concatenate([res[r][name][0][res[r][name][1][i]:res[r][name][1][i + 1]] for r in (0, 1)])
            assert_events_equal(canonical(got), dev["rows"][i], exact_order=True, ctx="%s frame %d" % (name, i))
        s0, s1 = res[0][name][2], res[1][name][2]
        assert s0["rejected"] == s1["rejected"] == len(bad_at), (name, s0, s1, bad_at)
        assert s0["chunks"] == s1["chunks"], (name, s0, s1)
        # chunks [1, 7) [7, 13): the rejected frame's index in its chunk, with the all-reduced maximum
        assert s0["last_reject"] == s1["last_reject"] == ((bad_at[-1] - 1) % DESIGNS[name]["mfps"], plan[bad_at[-1]]), \
            (name, s0, s1, bad_at)
        print("FUSED sharded/%-26s maxima=%s rank0=%s rank1=%s" % (name, sorted(set(plan[1:])), s0, s1))
