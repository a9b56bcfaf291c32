"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/pixel_states_*.npz by running the UNMODIFIED reference
(device="cpu") with record_single_pixel_states (emulator.py:278-302, 985-1009).

    python oracle/make_golden_pixel_states.py        # needs /root/reference

The reference records one pixel per run. A first run picks the pixels from its output (the busiest pixel, the pixel
with the most events in one frame, the quietest pixel, and for the band cases pixels on the first / last row of a band);
recordings of candidate pixels then add, where the run has one, a pixel whose events the refractory filter cut (its
recorded final count is below floor(|diff| / threshold)) and a pixel a shot-noise event reset (more rows at the pixel
than recorded signal events). Then the reference runs again with the same seed once per pixel. Recording draws nothing, so every run makes the same draws: the tape of the first run (make_golden.Recorder)
replays all of them. Each fixture holds the frames, times, kwargs, seed, tape, photoreceptor-noise amplitudes, the
picked pixels [P, 2] as (row, column), every recorded array as [P, SINGLE_PIXEL_MAX_SAMPLES] (NaN tail included),
the sample counts, the reference's event rows and its final lp / base state.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402
from make_golden import OUT, run_reference, texture_frames  # noqa: E402

NAMES = ("time", "new_frame", "base_log_frame", "lp_log_frame", "log_new_frame", "pos_thres", "neg_thres",
         "diff_frame", "final_neg_evts_frame", "final_pos_evts_frame")


def _pick(frames, per_frame, H, W, band_rows=()):
    """(row, column) pixels chosen from a run's event rows."""
    cnt = np.zeros((len(frames), H, W), np.int64)
    for f, ev in enumerate(per_frame):
        if ev is not None:
            np.add.at(cnt[f], (ev[:, 2].astype(np.int64), ev[:, 1].astype(np.int64)), 1)
    tot = cnt.sum(0)
    px = [tuple(int(v) for v in np.unravel_index(np.argmax(tot), tot.shape)),
          tuple(int(v) for v in np.unravel_index(np.argmax(cnt.max(0)), tot.shape))]
    quiet = np.argwhere(tot == 0)
    # the quietest pixel (no events at all where there is one)
    px.append(tuple(int(v) for v in quiet[len(quiet) // 2]) if len(quiet) else
              tuple(int(v) for v in np.unravel_index(np.argmin(tot), tot.shape)))
    for r in band_rows:
        row = tot[r]
        px.append((int(r), int(np.argmax(row))))
    out = []
    for p in px:
        if p not in out:
            out.append(p)
    return out, cnt


def _record(emu_mod, kwargs, frames, times, seed, p):
    cwd = os.getcwd()
    os.chdir(os.environ.get("TMPDIR", "/tmp"))      # the reference saves pixel-states.dat in the cwd
    try:
        em, _, tape = run_reference(emu_mod, dict(kwargs, record_single_pixel_states=p), frames, times, seed)
        em.cleanup()
    finally:
        os.chdir(cwd)
    em.record_single_pixel_states = None
    return em, tape


def _pick_special(emu_mod, kwargs, frames, times, seed, cnt, have):
    """A refractory-cut pixel and a shot-reset pixel, from recordings of candidates (the busiest pixels)."""
    tot = cnt.sum(0)
    order = [tuple(int(v) for v in np.unravel_index(i, tot.shape)) for i in np.argsort(-tot, axis=None, kind="stable")[:24]]
    found = {}
    for p in order:
        if len(found) == 2:
            break
        em, _ = _record(emu_mod, kwargs, frames, times, seed, p)
        s, n = em.single_pixel_states, em.single_pixel_sample_count
        fin = s["final_pos_evts_frame"][:n] + s["final_neg_evts_frame"][:n]
        thr = np.where(s["diff_frame"][:n] < 0, s["neg_thres"][:n], s["pos_thres"][:n])
        pre = np.floor(np.abs(s["diff_frame"][:n]) / thr)
        if "refractory" not in found and np.any(fin < pre):
            found["refractory"] = p
        if "shot" not in found and np.any(cnt[1:n + 1, p[0], p[1]] > fin):
            found["shot"] = p
    return [p for p in found.values() if p not in have]


def save_pixel_case(name, emu_mod, kwargs, frames, times, seed=42, band_rows=(), max_samples=None):
    em, per_frame, tape = run_reference(emu_mod, kwargs, frames, times, seed)
    H, W = frames.shape[1:3]
    pixels, cnt = _pick(frames, per_frame, H, W, band_rows)
    pixels += _pick_special(emu_mod, kwargs, frames, times, seed, cnt, pixels)
    d = {"frames": frames, "times": np.asarray(times, np.float64), "kwargs_json": np.array(json.dumps(kwargs)),
         "seed": np.array(seed), "pixels": np.asarray(pixels, np.int32),
         "event_counts": np.array([0 if e is None else len(e) for e in per_frame], np.int64),
         "torch_version": np.array(torch.__version__)}
    allev = [e for e in per_frame if e is not None]
    d["events"] = np.concatenate(allev, 0) if allev else np.zeros((0, 4), np.float32)
    if em._pr_vrms_used:
        d["pr_vrms"] = np.asarray(em._pr_vrms_used, np.float64)
    for nm in ("lp_log_frame", "base_log_frame"):
        d["state_" + nm] = getattr(em, nm).detach().cpu().numpy()
    d["tape_kinds"] = np.array([k for k, _ in tape])
    for i, (_, arr) in enumerate(tape):
        d["tape_%05d" % i] = arr.astype(np.int32) if arr.dtype == np.int64 else arr
    if max_samples is not None:
        d["max_samples"] = np.array(max_samples)
    counts = []
    rec = {k: [] for k in NAMES}
    for p in pixels:
        # the overflow case: the limit is lowered while the instance is made (its arrays have that length)
        orig = emu_mod.EventEmulator.SINGLE_PIXEL_MAX_SAMPLES
        if max_samples is not None:
            emu_mod.EventEmulator.SINGLE_PIXEL_MAX_SAMPLES = max_samples
        try:
            em2, tape2 = _record(emu_mod, kwargs, frames, times, seed, p)
        finally:
            emu_mod.EventEmulator.SINGLE_PIXEL_MAX_SAMPLES = orig
        assert len(tape2) == len(tape) and all(np.array_equal(a, b) for (_, a), (_, b) in zip(tape, tape2))
        counts.append(em2.single_pixel_sample_count)
        for k in NAMES:
            rec[k].append(np.asarray(em2.single_pixel_states[k], np.float64))
    d["sample_count"] = np.asarray(counts, np.int64)
    for k in NAMES:
        d["rec_" + k] = np.stack(rec[k])
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **d)
    print("%-34s pixels=%s samples=%s  %.1f KB" % (name, pixels, counts, os.path.getsize(path) / 1024))


def main():
    emu_mod, _, _, _ = ref_shim.load_reference()
    import logging
    logging.disable(logging.WARNING)
    H, W, T = 24, 40, 12
    fr = texture_frames(H, W, T, seed=21, speed=2.0)
    ts = np.arange(T) * 1e-3
    cli = dict(cutoff_hz=300, leak_rate_hz=0.01, shot_noise_rate_hz=0.001, refractory_period_s=0.0005,
               sigma_thres=0.03)
    save_pixel_case("pixel_states_cli", emu_mod, cli, fr, ts)
    save_pixel_case("pixel_states_noisy", emu_mod, dict(cli, leak_rate_hz=0.1, shot_noise_rate_hz=5.0), fr, ts)
    save_pixel_case("pixel_states_class_default", emu_mod, {}, fr, ts)
    save_pixel_case("pixel_states_sigma0", emu_mod, dict(cli, sigma_thres=0.0), fr, ts)
    frh = np.log1p(fr.astype(np.float32)).astype(np.float32)
    save_pixel_case("pixel_states_hdr", emu_mod, dict(cli, hdr=True, pos_thres=0.1, neg_thres=0.1), frh, ts)
    fr4 = texture_frames(20, 36, 6, seed=7)
    cs = dict(cs_lambda_pixels=10, cs_tau_p_ms=0.5, refractory_period_s=1e-3, leak_rate_hz=0.1,
              shot_noise_rate_hz=1.0, sigma_thres=0.03)
    save_pixel_case("pixel_states_cs_f64", emu_mod, dict(cs, cutoff_hz=100), fr4, np.arange(6) * 1e-4,
                    band_rows=(0, 9, 10, 19))
    save_pixel_case("pixel_states_cs_f32", emu_mod, dict(cs, cutoff_hz=0), fr4, np.arange(6) * 1e-4,
                    band_rows=(0, 9, 10, 19))
    save_pixel_case("pixel_states_scidvs", emu_mod,
                    dict(scidvs=True, cutoff_hz=100, leak_rate_hz=0.1, shot_noise_rate_hz=5.0, sigma_thres=0.03,
                         refractory_period_s=0.0005), fr, ts, band_rows=(11, 12))
    save_pixel_case("pixel_states_prnoise", emu_mod,
                    dict(photoreceptor_noise=True, cutoff_hz=100, shot_noise_rate_hz=5.0, leak_rate_hz=0.1,
                         sigma_thres=0.03), fr, ts, band_rows=(11, 12))
    # noise-free: device mode matches bit for bit; the refractory filter engages (refractory > dt / max_n) in the
    # frames where some pixel has >= 3 events, so multi-frame chunks are accepted and rejected
    from scipy.ndimage import gaussian_filter
    big = gaussian_filter(np.random.default_rng(5).uniform(0, 255, (80, 140)), 3)
    big = (big - big.min()) / (big.max() - big.min()) * 200 + 20
    frq = np.stack([big[k // 4:k // 4 + 32, k // 2:k // 2 + 64] for k in range(40)]).round().astype(np.uint8)
    frq[12:14] = np.clip(frq[12:14].astype(np.int64) * 2, 0, 255).astype(np.uint8)
    frq[27] = 255 - frq[27]
    save_pixel_case("pixel_states_noise_free", emu_mod,
                    dict(cutoff_hz=300, leak_rate_hz=0, shot_noise_rate_hz=0, refractory_period_s=0.0004,
                         sigma_thres=0.03, pos_thres=0.15, neg_thres=0.15), frq, np.arange(40) * 1e-3,
                    band_rows=(15, 16))
    save_pixel_case("pixel_states_overflow", emu_mod, cli, fr, ts, max_samples=5)


if __name__ == "__main__":
    main()
