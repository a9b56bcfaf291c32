"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/emu_*.npz by running the
UNMODIFIED reference (device="cpu") in the build container.

    python oracle/make_golden.py            # needs /root/reference
    python oracle/make_golden.py optional   # SCIDVS / photoreceptor-noise fixtures only
    python oracle/make_golden.py hdr        # log-encoded input (hdr=True) fixtures only
    python oracle/make_golden.py cs         # centre-surround fixtures only

Each fixture holds: the input frames and times, the constructor kwargs, the
"tape" of every random draw the reference made (thresholds, noise-rate field,
per-frame leak randn / shot rand, per-iteration randperm) so that parity does not
depend on the host's torch RNG implementation, the reference's per-frame event
rows (exact order), and its final per-pixel state.

The tape is recorded by wrapping torch.normal/randn/rand/randperm while the
reference runs; the wrapped functions return the reference's own values untouched.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


class Recorder:
    """Context manager that logs the outputs of the torch RNG entry points used by
    the reference emulator (emulator.py:460-471, 501-503, 868; emulator_utils.py:122-124, 340-343)."""
    NAMES = ("normal", "randn", "rand", "randperm")

    def __init__(self):
        self.tape = []

    def __enter__(self):
        self._orig = {n: getattr(torch, n) for n in self.NAMES}
        for n in self.NAMES:
            setattr(torch, n, self._wrap(n, self._orig[n]))
        return self

    def _wrap(self, name, fn):
        def inner(*a, **k):
            out = fn(*a, **k)
            self.tape.append((name, out.detach().cpu().numpy().copy()))
            return out
        return inner

    def __exit__(self, *exc):
        for n in self.NAMES:
            setattr(torch, n, self._orig[n])


def texture_frames(H, W, T, seed=0, speed=1.0, block=4):
    rng = np.random.default_rng(seed)
    pad = int(T * speed * 1.5) + 8
    base = rng.integers(0, 256, ((H + pad) // block + 2, (W + pad) // block + 2)).astype(np.uint8)
    big = np.kron(base, np.ones((block, block), np.uint8))
    out = []
    for k in range(T):
        dx, dy = int(k * speed), int(k * speed * 0.5)
        out.append(np.ascontiguousarray(big[dy:dy + H, dx:dx + W]))
    return np.stack(out)


def run_reference(emu_mod, kwargs, frames, times, seed):
    import logging
    logging.disable(logging.WARNING)
    # the photoreceptor-noise amplitude comes from an UNSEEDED numpy generator (emulator_utils.py:234-235,
    # 254): record the values the reference used, frame by frame
    vrms = []
    orig_vn = emu_mod.compute_photoreceptor_noise_voltage

    def vn_wrap(*a, **k):
        v = orig_vn(*a, **k)
        vrms.append(float(v))
        return v
    emu_mod.compute_photoreceptor_noise_voltage = vn_wrap
    try:
        with Recorder() as rec:
            em = emu_mod.EventEmulator(device="cpu", seed=seed, **kwargs)
            per_frame = []
            for f, t in zip(frames, times):
                per_frame.append(em.generate_events(f, float(t)))
    finally:
        emu_mod.compute_photoreceptor_noise_voltage = orig_vn
    em._pr_vrms_used = vrms
    return em, per_frame, rec.tape


def save_case(name, emu_mod, kwargs, frames, times, seed=42, keep_tape=True, keep_events=True):
    em, per_frame, tape = run_reference(emu_mod, kwargs, frames, times, seed)
    counts = np.array([0 if e is None else len(e) for e in per_frame], np.int64)
    d = {
        "frames": frames,
        "times": np.asarray(times, np.float64),
        "kwargs_json": np.array(json.dumps(kwargs)),
        "seed": np.array(seed),
        "event_counts": counts,
        "num_on": np.array(em.num_events_on), "num_off": np.array(em.num_events_off),
        "cpu_capability": np.array(torch.backends.cpu.get_cpu_capability()),
        "torch_version": np.array(torch.__version__),
    }
    allev = [e for e in per_frame if e is not None]
    allev = np.concatenate(allev, 0) if allev else np.zeros((0, 4), np.float32)
    if keep_events:
        d["events"] = allev
    else:
        # canonical digest: per-frame counts + lexicographically sorted rows
        import hashlib
        off = np.concatenate([[0], np.cumsum(counts)])
        h = hashlib.sha1()
        for i in range(len(counts)):
            e = allev[off[i]:off[i + 1]]
            if len(e):
                k = np.lexsort((e[:, 3], e[:, 1], e[:, 2], e[:, 0]))
                h.update(np.ascontiguousarray(e[k]).tobytes())
        d["events_sha1_canonical"] = np.array(h.hexdigest())
    if em._pr_vrms_used:
        d["pr_vrms"] = np.asarray(em._pr_vrms_used, np.float64)
    for nm in ("lp_log_frame", "base_log_frame", "timestamp_mem", "pos_thres", "neg_thres",
               "noise_rate_array", "cs_surround_frame", "scidvs_highpass", "photoreceptor_noise_arr",
               "scidvs_tau_arr"):
        v = getattr(em, nm, None)
        if isinstance(v, torch.Tensor):
            d["state_" + nm] = v.detach().cpu().numpy()
    if getattr(em, "cs_steps_taken", None):
        d["cs_steps_taken"] = np.asarray(em.cs_steps_taken, np.int32)
    if keep_tape:
        d["tape_kinds"] = np.array([k for k, _ in tape])
        for i, (_, arr) in enumerate(tape):
            if arr.dtype == np.int64:
                arr = arr.astype(np.int32)
            d["tape_%05d" % i] = arr
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **d)
    print("%-28s frames=%d events=%d on=%d off=%d  %.1f KB" % (
        name, len(frames), counts.sum(), em.num_events_on, em.num_events_off,
        os.path.getsize(path) / 1024))


def main_optional(emu_mod):
    """SCIDVS (emulator.py:58-80, 719-725) and photoreceptor noise (emulator.py:694-703) fixtures."""
    H, W, T = 24, 40, 10
    fr = texture_frames(H, W, T)
    ts = np.arange(T) * 1e-3
    save_case("emu_scidvs", emu_mod,
              dict(scidvs=True, cutoff_hz=100, leak_rate_hz=0.1, shot_noise_rate_hz=5.0, sigma_thres=0.03,
                   refractory_period_s=0.0005), fr, ts)
    save_case("emu_scidvs_f32", emu_mod,
              dict(scidvs=True, cutoff_hz=0, leak_rate_hz=0.1, shot_noise_rate_hz=0, sigma_thres=0.03,
                   pos_thres=0.4, neg_thres=0.4), fr[:6, :16, :24].copy(), ts[:6])
    save_case("emu_prnoise", emu_mod,
              dict(photoreceptor_noise=True, cutoff_hz=100, shot_noise_rate_hz=5.0, leak_rate_hz=0.1,
                   sigma_thres=0.03), fr, ts)
    fr4 = texture_frames(20, 36, 6, seed=7)
    save_case("emu_prnoise_scidvs_csdvs", emu_mod,
              dict(photoreceptor_noise=True, scidvs=True, cs_lambda_pixels=10, cs_tau_p_ms=0.5, cutoff_hz=100,
                   refractory_period_s=1e-3, leak_rate_hz=0.1, shot_noise_rate_hz=1.0, sigma_thres=0.03,
                   pos_thres=0.05, neg_thres=0.05), fr4, np.arange(6) * 1e-4)


def main_hdr(emu_mod):
    """hdr=True (emulator.py:100, 663-672): the frames are already natural-log intensities, float32."""
    H, W, T = 24, 40, 8
    fr = np.log1p(texture_frames(H, W, T, seed=13, speed=2.0).astype(np.float32)).astype(np.float32)
    ts = np.arange(T) * 1e-3
    save_case("emu_hdr", emu_mod,
              dict(hdr=True, cutoff_hz=300, leak_rate_hz=0.1, shot_noise_rate_hz=5.0, refractory_period_s=0.001,
                   sigma_thres=0.03, pos_thres=0.1, neg_thres=0.1), fr, ts)
    save_case("emu_hdr_nolp", emu_mod,
              dict(hdr=True, cutoff_hz=0, leak_rate_hz=0.1, shot_noise_rate_hz=5.0, refractory_period_s=0.001,
                   sigma_thres=0.03, pos_thres=0.1, neg_thres=0.1), fr, ts)


def main_cs(emu_mod):
    """Centre-surround fixtures (emulator.py:1061-1124). The surround's float32 Laplacian sums its taps in an order
    that depends on the frame size and, below 20 480 padded pixels, on the flattened index (oracle/emu_oracle.c,
    oracle_lap_kernel_order): one fixture on each side of that switch and one whose flattened tail is non-empty."""
    # centre-surround model (scripts/csdvs.sh:7-16: lambda 10 px, tau_p 0.5 ms, dt 1e-4 s, cutoff 100 Hz)
    fr4 = texture_frames(20, 36, 6, seed=7)
    save_case("emu_csdvs", emu_mod,
              dict(cs_lambda_pixels=10, cs_tau_p_ms=0.5, cutoff_hz=100, refractory_period_s=1e-3,
                   leak_rate_hz=0.1, shot_noise_rate_hz=1.0, sigma_thres=0.03), fr4, np.arange(6) * 1e-4)
    # > 20480 padded pixels: the size class of both BASELINE resolutions (different float32 conv2d summation order)
    save_case("emu_csdvs_120x176", emu_mod,
              dict(cs_lambda_pixels=4, cs_tau_p_ms=2.0, cutoff_hz=200, leak_rate_hz=0, shot_noise_rate_hz=0,
                   sigma_thres=0.02), texture_frames(120, 176, 5, seed=9), np.arange(5) * 5e-4)
    # 37x53 = 1961 px: below the switch, the last 1961 mod 16 = 9 pixels take the other summation order; high contrast
    # (1 px blocks, fast motion) so that the surround differs between the two orders
    save_case("emu_csdvs_37x53", emu_mod,
              dict(cs_lambda_pixels=3, cs_tau_p_ms=0.5, cutoff_hz=300, leak_rate_hz=0.1, shot_noise_rate_hz=1.0,
                   sigma_thres=0.03, pos_thres=0.3, neg_thres=0.3),
              texture_frames(37, 53, 6, seed=11, speed=3.0, block=1), np.arange(6) * 2e-4)


def main():
    emu_mod, _, _, _ = ref_shim.load_reference()
    if len(sys.argv) > 1 and sys.argv[1] == "optional":
        return main_optional(emu_mod)
    if len(sys.argv) > 1 and sys.argv[1] == "hdr":
        return main_hdr(emu_mod)
    if len(sys.argv) > 1 and sys.argv[1] == "cs":
        return main_cs(emu_mod)
    H, W, T = 24, 40, 10
    fr = texture_frames(H, W, T)
    ts = np.arange(T) * 1e-3
    # class defaults (emulator.py:88-95): float32 state, leak only
    save_case("emu_class_default", emu_mod, {}, fr, ts)
    # CLI defaults (v2e_args.py:150-204) with a visible shot rate
    save_case("emu_cli_noisy", emu_mod,
              dict(cutoff_hz=300, leak_rate_hz=0.1, shot_noise_rate_hz=5.0,
                   refractory_period_s=0.0005, sigma_thres=0.03), fr, ts)
    # test/v2e-tests.sh:8 "clean" recipe
    save_case("emu_clean", emu_mod,
              dict(sigma_thres=0.0, cutoff_hz=0, leak_rate_hz=0, shot_noise_rate_hz=0), fr, ts)
    # scalar thresholds against float64 state (sigma_thres == 0 keeps Python floats)
    save_case("emu_scalar_thres_f64", emu_mod,
              dict(sigma_thres=0.0, cutoff_hz=100, leak_rate_hz=0.2, shot_noise_rate_hz=10), fr, ts)
    # refractory filter active with many events per pixel per frame
    fr2 = texture_frames(H, W, T, speed=3.0)
    ts2 = np.arange(T) * 1e-2
    save_case("emu_refractory_multi", emu_mod,
              dict(cutoff_hz=200, leak_rate_hz=0.1, refractory_period_s=0.004, pos_thres=0.05,
                   neg_thres=0.05, sigma_thres=0.01, shot_noise_rate_hz=2), fr2, ts2)
    # float32 frames with non-integer values (lin_log evaluated, not looked up)
    rng = np.random.default_rng(3)
    frn = (fr.astype(np.float32) + rng.uniform(0, 0.9, fr.shape).astype(np.float32))
    save_case("emu_float_frames", emu_mod,
              dict(cutoff_hz=300, leak_rate_hz=0.01, shot_noise_rate_hz=0.001,
                   refractory_period_s=0.0005), frn, ts)
    # test/leak_event_test.py:17-32 recipe: static image, leak + shot only
    static = np.repeat(fr[:1], T, axis=0)
    save_case("emu_static_leak_shot", emu_mod,
              dict(pos_thres=0.2, neg_thres=0.2, sigma_thres=0.03, cutoff_hz=200,
                   leak_rate_hz=0.2, shot_noise_rate_hz=10), static, np.arange(T) * 2e-3)
    # ragged size (odd width, not a multiple of the kernel's vector width), empty-event frames
    fr3 = texture_frames(13, 37, 8, seed=5)
    fr3[3] = fr3[2]
    fr3[4] = fr3[2]
    save_case("emu_ragged_13x37", emu_mod,
              dict(cutoff_hz=0, leak_rate_hz=0, shot_noise_rate_hz=0, sigma_thres=0.03), fr3,
              np.arange(8) * 1e-3)
    main_cs(emu_mod)
    # BASELINE config 1: scripts/moving_dot.py 64x64, class defaults, seed 42 -> 27 917 events
    import importlib
    md = importlib.import_module("scripts.moving_dot")
    import cv2
    cv2.destroyAllWindows = lambda: None
    src = md.moving_dot(width=64, height=64, preview=False, parent_args=None, arg_list=[
        "--t_total", "0.05", "--radius", "20", "--dt", "1e-4"])
    mfr, mts = [], []
    while True:
        f, t = src.next_frame()
        if f is None:
            break
        mfr.append(np.array(f, copy=True))
        mts.append(t)
    mfr = np.stack(mfr)
    save_case("emu_moving_dot_c1", emu_mod, {}, mfr, np.array(mts), keep_tape=False, keep_events=False)


if __name__ == "__main__":
    main()
