"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/model_states_*.npz by running the UNMODIFIED reference
(device="cpu") with show_dvs_model_state and save_dvs_model_state (emulator.py:41-50, 365-368, 580-617, 756-767).

    python oracle/make_golden_model_states.py        # needs /root/reference

The reference's GUI calls are stubbed (namedWindow, moveWindow, imshow, waitKey, pollKey) and its video_writer
(imported by name, emulator.py:28) is replaced by a recorder. Each fixture holds the frames, times, kwargs, seed, the
RNG tape, the photoreceptor-noise amplitudes, and, for every shown state: the bytes the reference casts before its
overlay (the float image handed to the first putText of each _show, x255, astype(uint8)) as plane_<name> [k, H, W],
one channel of the BGR frames it wrote (the three are checked equal) as video_<name>, the writer's arguments, the
frame counters and t_previous values of the overlay text, and the names the reference skipped. The SCIDVS case also
keeps the float64 scidvs_highpass / diff_frame it showed (raw_<name>).
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402
from make_golden import OUT, run_reference, texture_frames  # noqa: E402


class _Writer:
    def __init__(self, log, fn, height, width):
        self.fn, self.height, self.width = fn, height, width
        self.frames = []
        self.released = False
        log.append(self)

    def write(self, frame):
        assert frame.dtype == np.uint8 and frame.ndim == 3 and frame.shape[2] == 3
        assert np.array_equal(frame[..., 0], frame[..., 1]) and np.array_equal(frame[..., 0], frame[..., 2])
        self.frames.append(frame[..., 0].copy())

    def release(self):
        self.released = True


def run_shown(emu_mod, kwargs, frames, times, seed, show, keep_raw=()):
    import cv2
    writers, shows = [], []
    cur = {}
    stubs = {k: (lambda *a, **kw: -1) for k in ("namedWindow", "moveWindow", "imshow", "waitKey", "pollKey")}
    saved = {k: getattr(cv2, k) for k in list(stubs) + ["putText"]}
    orig_put, orig_show, orig_vw = cv2.putText, emu_mod.EventEmulator._show, emu_mod.video_writer

    def put(img, text, **kw):
        if kw.get("color") == (0, 0, 0):
            cur["plane"] = (img * 255).astype(np.uint8)
            cur["text"] = text
        return orig_put(img, text, **kw)

    def show_wrap(self, inp, name):
        cur.clear()
        raw = inp.detach().cpu().numpy().astype(np.float64) if name in keep_raw else None
        orig_show(self, inp, name)
        shows.append((name, self.frame_counter, float(self.t_previous), cur["plane"], cur["text"], raw))

    for k, v in stubs.items():
        setattr(cv2, k, v)
    cv2.putText = put
    emu_mod.EventEmulator._show = show_wrap
    emu_mod.video_writer = lambda fn, h, w: _Writer(writers, fn, h, w)
    try:
        with tempfile.TemporaryDirectory() as td:
            em, per_frame, tape = run_reference(
                emu_mod, dict(kwargs, show_dvs_model_state=show, save_dvs_model_state=True, output_folder=td),
                frames, times, seed)
            em.cleanup()
            for w in writers:
                w.fn = os.path.relpath(w.fn, td)
    finally:
        for k, v in saved.items():
            setattr(cv2, k, v)
        emu_mod.EventEmulator._show = orig_show
        emu_mod.video_writer = orig_vw
    return em, per_frame, tape, writers, shows


def save_state_case(name, emu_mod, kwargs, frames, times, show=("all",), seed=42, keep_raw=()):
    # the reference draws its overlay at output_height (the v2e CLI always passes the output size)
    kwargs = dict(kwargs, output_height=int(frames.shape[1]), output_width=int(frames.shape[2]))
    em, per_frame, tape, writers, shows = run_shown(emu_mod, kwargs, frames, times, seed, list(show), keep_raw)
    names = []
    for s in shows:
        if s[0] not in names:
            names.append(s[0])
    d = {"frames": frames, "times": np.asarray(times, np.float64), "kwargs_json": np.array(json.dumps(kwargs)),
         "seed": np.array(seed), "show": np.array(list(show)), "shown": np.array(names),
         "skipped": np.array(list(em.dont_show_list), dtype=str),
         "output_hw": np.array([em.output_height, em.output_width], np.int64),
         "event_counts": np.array([0 if e is None else len(e) for e in per_frame], np.int64),
         "torch_version": np.array(torch.__version__)}
    if em._pr_vrms_used:
        d["pr_vrms"] = np.asarray(em._pr_vrms_used, np.float64)
    d["tape_kinds"] = np.array([k for k, _ in tape])
    for i, (_, arr) in enumerate(tape):
        d["tape_%05d" % i] = arr.astype(np.int32) if arr.dtype == np.int64 else arr
    first = [s for s in shows if s[0] == names[0]]
    d["frame_counter"] = np.array([s[1] for s in first], np.int64)
    d["t_previous"] = np.array([s[2] for s in first], np.float64)
    d["text"] = np.array([s[4] for s in first])
    for nm in names:
        mine = [s for s in shows if s[0] == nm]
        assert [s[1] for s in mine] == list(d["frame_counter"])
        d["plane_" + nm] = np.stack([s[3] for s in mine])
        if nm in keep_raw:
            d["raw_" + nm] = np.stack([s[5] for s in mine])
    for w in writers:
        nm = os.path.splitext(w.fn)[0]
        assert w.released and w.fn == nm + ".avi" and nm in names
        d["video_" + nm] = np.stack(w.frames)
        d["writer_" + nm] = np.array([w.height, w.width], np.int64)
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **d)
    print("%-30s shown=%s skipped=%s frames=%d  %.1f KB" % (name, names, list(em.dont_show_list),
                                                            len(d["frame_counter"]), os.path.getsize(path) / 1024))


def main(only=()):
    """Regenerates every fixture, or only the ones named."""
    emu_mod, _, _, _ = ref_shim.load_reference()

    def case(name, *a, **k):
        if not only or name in only:
            save_state_case(name, emu_mod, *a, **k)
    import logging
    logging.disable(logging.WARNING)
    T = 10
    fa = texture_frames(13, 37, T, seed=21, speed=2.0)
    fb = texture_frames(37, 53, T, seed=22, speed=1.5)
    ts = np.arange(T) * 1e-3
    cli = dict(cutoff_hz=300, leak_rate_hz=0.01, shot_noise_rate_hz=0.001, refractory_period_s=0.0005,
               sigma_thres=0.03)
    case("model_states_cli", cli, fa, ts)
    case("model_states_noisy", dict(cli, leak_rate_hz=0.1, shot_noise_rate_hz=5.0), fb, ts)
    case("model_states_class_default", {}, fa, ts,
         show=("diff_frame", "lp_log_frame", "no_such_state", "base_log_frame", "scidvs_highpass"))
    case("model_states_sigma0", dict(cli, sigma_thres=0.0), fb, ts)
    fah = np.log1p(fa.astype(np.float32)).astype(np.float32)
    case("model_states_hdr", dict(cli, hdr=True, pos_thres=0.1, neg_thres=0.1), fah, ts)
    cs = dict(cs_lambda_pixels=10, cs_tau_p_ms=0.5, refractory_period_s=1e-3, leak_rate_hz=0.1,
              shot_noise_rate_hz=1.0, sigma_thres=0.03)
    fc = texture_frames(37, 53, 6, seed=7)
    case("model_states_cs_f64", dict(cs, cutoff_hz=100), fc, np.arange(6) * 1e-4)
    case("model_states_cs_f32", dict(cs, cutoff_hz=0), fc[:, :13, :37], np.arange(6) * 1e-4)
    case("model_states_scidvs",
         dict(scidvs=True, cutoff_hz=100, leak_rate_hz=0.1, shot_noise_rate_hz=5.0, sigma_thres=0.03,
              refractory_period_s=0.0005), fb, ts, keep_raw=("scidvs_highpass", "diff_frame"))
    case("model_states_prnoise",
         dict(photoreceptor_noise=True, cutoff_hz=100, shot_noise_rate_hz=5.0, leak_rate_hz=0.1,
              sigma_thres=0.03), fa, ts)
    # noise-free: the device RNG matches bit for bit; the refractory filter engages in the frames where some pixel has
    # >= 3 events, so multi-frame chunks are accepted and rejected
    from scipy.ndimage import gaussian_filter
    big = gaussian_filter(np.random.default_rng(5).uniform(0, 255, (80, 140)), 3)
    big = (big - big.min()) / (big.max() - big.min()) * 200 + 20
    frq = np.stack([big[k // 4:k // 4 + 37, k // 2:k // 2 + 53] for k in range(40)]).round().astype(np.uint8)
    frq[12:14] = np.clip(frq[12:14].astype(np.int64) * 2, 0, 255).astype(np.uint8)
    frq[27] = 255 - frq[27]
    case("model_states_noise_free",
         dict(cutoff_hz=300, leak_rate_hz=0, shot_noise_rate_hz=0, refractory_period_s=0.0004,
              sigma_thres=0.03, pos_thres=0.15, neg_thres=0.15), frq, np.arange(40) * 1e-3)
    # a DAVIS346 frame: the overlay text lies inside the frame. Noise-free and smooth, translating 1 px per frame, so
    # that few pixels fire and the replayed randperm tape stays small; 14 grey levels, so that the fixture compresses
    smooth = gaussian_filter(np.random.default_rng(9).uniform(0, 255, (264, 352)), 6)
    smooth = (smooth - smooth.min()) / (smooth.max() - smooth.min()) * 13
    fd = np.stack([smooth[2:262, k:k + 346] for k in range(3)]).round().astype(np.uint8) * 16 + 20
    case("model_states_346x260", dict(cutoff_hz=300, leak_rate_hz=0, sigma_thres=0.0), fd, np.arange(3) * 1e-3,
         show=("new_frame", "diff_frame", "cs_surround_frame"))


if __name__ == "__main__":
    main(sys.argv[1:])
