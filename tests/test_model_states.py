"""Model-state planes (show_dvs_model_state / save_dvs_model_state, emulator.py:41-50, 580-617, 756-767): the uint8
cast and the numpy oracle (oracle/model_state_oracle.py) against numpy and the fixtures made from the unmodified
reference by oracle/make_golden_model_states.py; the keyword checks; and (GPU) the device's planes and written frames
on every path against the fixtures."""
import os
import sys
import types

import numpy as np
import pytest

from helpers import TapeRNG, load_golden

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import model_state_oracle as mso  # noqa: E402

CASES = ["model_states_cli", "model_states_noisy", "model_states_class_default", "model_states_sigma0",
         "model_states_hdr", "model_states_cs_f64", "model_states_cs_f32", "model_states_scidvs",
         "model_states_prnoise", "model_states_noise_free", "model_states_346x260"]


def _shown(g):
    return [str(s) for s in g["shown"]]


# ---- the cast and the oracle (CPU) ---------------------------------------------------------------------------------
def test_cast_rule_equals_numpy_astype():
    edge = np.array([65025, -1, 300.7, -300.2, -0.5, 0.0, -0.0, 255.9, 256, 1e10 + 5, 2.0 ** 31 + 7, 2.0 ** 40 + 9,
                     2.0 ** 31 - 0.5, -2.0 ** 31, -2.0 ** 31 - 0.5, -2.0 ** 31 - 1, np.nan, np.inf, -np.inf, 1e300,
                     -1e300, 5e-324], np.float64)
    want = np.array([1, 255, 44, 212, 0, 0, 0, 255, 0, 0, 0, 0], np.uint8)
    assert np.array_equal(mso.u8(edge[:12]), want)
    with np.errstate(invalid="ignore"):
        assert np.array_equal(mso.u8(edge), edge.astype(np.uint8))
        rng = np.random.default_rng(0)
        for n in list(range(1, 40)) + [63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 999, 1000]:
            scale = rng.choice([1.0, 300.0, 1e5, 3e9, 1e12])
            v = rng.standard_normal(n) * scale
            v[rng.integers(0, n, max(1, n // 10))] = rng.choice(edge, max(1, n // 10))
            assert np.array_equal(mso.u8(v), v.astype(np.uint8)), n


def test_ranges_are_the_references():
    from v2e_b200.emulator import EventEmulator, MODEL_STATE_RANGES
    assert tuple(MODEL_STATE_RANGES) == EventEmulator.MODEL_STATES
    for k, (lo, hi) in MODEL_STATE_RANGES.items():
        assert (lo, hi) == mso.RANGES[k] and (hi - lo) == (mso.RANGES[k][1] - mso.RANGES[k][0]), k


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_fixture(name):
    """The oracle's planes from the inputs (new_frame, log_new_frame with hdr, constant photoreceptor_noise_arr
    without photoreceptor noise, the float64 SCIDVS states) and its overlay from every plane equal the reference's."""
    g = load_golden(name)
    fr = g["frames"][1:].astype(np.float64)
    shown = _shown(g)
    if "new_frame" in shown:
        assert np.array_equal(g["plane_new_frame"], mso.plane(fr, "new_frame"))
    if g["kwargs"].get("hdr") and "log_new_frame" in shown:
        assert np.array_equal(g["plane_log_new_frame"], mso.plane(fr, "log_new_frame"))
    if "photoreceptor_noise_arr" in shown and not g["kwargs"].get("photoreceptor_noise"):
        assert np.all(g["plane_photoreceptor_noise_arr"] == mso.plane(np.zeros(1), "photoreceptor_noise_arr")[0])
    for k in ("scidvs_highpass", "diff_frame"):
        if "raw_" + k in g:
            assert np.array_equal(g["plane_" + k], mso.plane(g["raw_" + k], k)), k
    assert list(g["text"]) == [mso.overlay_text(f, t) for f, t in zip(g["frame_counter"], g["t_previous"])]
    assert list(g["frame_counter"]) == list(range(2, len(g["frames"]) + 1))
    pytest.importorskip("cv2")
    H = int(g["output_hw"][0])
    for k in shown:
        assert np.array_equal(g["writer_" + k], g["output_hw"])
        for j, (f, t) in enumerate(zip(g["frame_counter"], g["t_previous"])):
            assert np.array_equal(g["video_" + k][j], mso.overlay(g["plane_" + k][j], f, t, H)), (k, j)


def test_fixture_regenerates_byte_for_byte():
    import ref_shim
    try:
        emu_mod = ref_shim.load_reference()[0]
    except Exception as e:
        pytest.skip("the reference emulator is not importable here (%s)" % e)
    from make_golden_model_states import run_shown
    g = load_golden("model_states_cli")
    kw = dict(g["kwargs"], output_height=int(g["output_hw"][0]), output_width=int(g["output_hw"][1]))
    em, _, _, writers, shows = run_shown(emu_mod, kw, g["frames"], g["times"], int(g["seed"]), list(g["show"]))
    for k in _shown(g):
        assert np.array_equal(np.stack([s[3] for s in shows if s[0] == k]), g["plane_" + k]), k
        w = next(w for w in writers if w.fn == k + ".avi")
        assert np.array_equal(np.stack(w.frames), g["video_" + k]), k


# ---- keywords (CPU, library stubbed) ---------------------------------------------------------------------------------
def _stub(monkeypatch, **kw):
    from v2e_b200 import emulator as em_mod
    monkeypatch.setattr(em_mod._lib, "load", lambda *a, **k: object())
    e = em_mod.EventEmulator(device="cuda", **kw)
    e._finalizer.detach()
    return e


def test_keywords(monkeypatch, tmp_path):
    from v2e_b200.emulator import EventEmulator
    assert EventEmulator.MODEL_STATES[0] == "new_frame" and len(EventEmulator.MODEL_STATES) == 9
    e = _stub(monkeypatch, show_dvs_model_state=["all"])
    assert e._ms_names == ["new_frame", "log_new_frame", "lp_log_frame", "photoreceptor_noise_arr",
                           "base_log_frame", "diff_frame"]
    e = _stub(monkeypatch, show_dvs_model_state=["all"], scidvs=True, cs_lambda_pixels=5)
    assert e._ms_names == list(EventEmulator.MODEL_STATES)
    e = _stub(monkeypatch, show_dvs_model_state=["diff_frame", "nope", "cs_surround_frame", "new_frame"])
    assert e._ms_names == ["diff_frame", "new_frame"] and e._ms_order() == ["new_frame", "diff_frame"]
    with pytest.raises(ValueError):
        _stub(monkeypatch, show_dvs_model_state=["diff_frame", "pos_thres"])
    with pytest.raises(ValueError):
        _stub(monkeypatch, show_dvs_model_state=["diff_frame"], save_dvs_model_state=True)
    # nothing shown: no folder needed, nothing captured
    e = _stub(monkeypatch, save_dvs_model_state=True)
    assert e._ms_names == [] and e._ms_video_writer is None
    with pytest.raises(RuntimeError):
        e.model_state_frames()


def test_without_video_writer_one_warning_no_files(monkeypatch, tmp_path):
    from v2e_b200 import emulator as em_mod
    monkeypatch.setitem(sys.modules, "v2ecore", None)
    monkeypatch.setitem(sys.modules, "v2ecore.v2e_utils", None)
    warned = []
    monkeypatch.setattr(em_mod.logger, "warning", lambda msg, *a: warned.append(msg % a))
    e = _stub(monkeypatch, show_dvs_model_state=["diff_frame"], save_dvs_model_state=True,
              output_folder=str(tmp_path))
    assert e._ms_video_writer is None
    assert sum("save_dvs_model_state ignored" in m for m in warned) == 1
    assert os.listdir(tmp_path) == []


# ---- GPU ---------------------------------------------------------------------------------------------------------------
class _RecWriter:
    def __init__(self, log, fn, h, w):
        self.fn, self.h, self.w, self.frames, self.released = fn, h, w, [], False
        log.append(self)

    def write(self, frame):
        assert frame.dtype == np.uint8 and frame.shape[2] == 3
        assert np.array_equal(frame[..., 0], frame[..., 1]) and np.array_equal(frame[..., 0], frame[..., 2])
        self.frames.append(frame[..., 0].copy())

    def release(self):
        self.released = True


def _inject_writer(monkeypatch):
    log = []
    pkg = types.ModuleType("v2ecore")
    mod = types.ModuleType("v2ecore.v2e_utils")
    mod.video_writer = lambda fn, h, w: _RecWriter(log, fn, h, w)
    pkg.v2e_utils = mod
    monkeypatch.setitem(sys.modules, "v2ecore", pkg)
    monkeypatch.setitem(sys.modules, "v2ecore.v2e_utils", mod)
    return log


def _kw(g, tmp_path=None, show=True):
    kw = dict(g["kwargs"], output_height=int(g["output_hw"][0]), output_width=int(g["output_hw"][1]))
    if show:
        kw["show_dvs_model_state"] = [str(s) for s in g["show"]]
        if tmp_path is not None:
            kw.update(save_dvs_model_state=True, output_folder=str(tmp_path))
    return kw


def _run_replay(g, **kw):
    from v2e_b200 import EventEmulator
    extra = {"pr_vrms_tape": list(g["pr_vrms"])} if "pr_vrms" in g else {}
    em = EventEmulator(device="cuda", rng=TapeRNG(g["tape"]), **kw, **extra)
    rows, frames = [], {}
    for f, t in zip(g["frames"], g["times"]):
        rows.append(em.generate_events(f, float(t)))
        if em._ms_names and em._ms_chunks:
            ms = em.model_state_frames()
            for k in em._ms_names:
                frames.setdefault(k, []).append(ms[k].cpu().numpy())
            frames.setdefault("frame", []).append(ms["frame"])
            frames.setdefault("t_previous", []).append(ms["t_previous"])
    return em, rows, {k: np.concatenate(v) for k, v in frames.items()}


def _compare_planes(g, got, name):
    exempt = 0
    for k in _shown(g):
        want = g["plane_" + k]
        diff = got[k] != want
        if diff.any() and name == "model_states_scidvs" and k in ("scidvs_highpass", "diff_frame"):
            v = mso.normalise(g["raw_" + k], k) * 255
            assert np.all(np.abs(v - np.round(v))[diff] < 1e-9), k
            exempt += int(diff.sum())
        else:
            assert not diff.any(), (name, k, int(diff.sum()))
    print("%s: %d SCIDVS pixels exempted" % (name, exempt))


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_replay_planes_and_videos_equal_reference(name, tmp_path, monkeypatch):
    g = load_golden(name)
    log = _inject_writer(monkeypatch)
    em, rows, got = _run_replay(g, **_kw(g, tmp_path))
    assert em._ms_names == _shown(g)
    assert np.array_equal(got["frame"], g["frame_counter"]) and np.array_equal(got["t_previous"], g["t_previous"])
    _compare_planes(g, got, name)
    em.cleanup()
    assert sorted(w.fn for w in log) == sorted(os.path.join(str(tmp_path), k + ".avi") for k in _shown(g))
    for w in log:
        k = os.path.basename(w.fn)[:-4]
        assert w.released and (w.h, w.w) == tuple(g["writer_" + k])
        vid = np.stack(w.frames)
        if name == "model_states_scidvs" and k in ("scidvs_highpass", "diff_frame"):
            assert np.array_equal(vid == g["video_" + k], got[k] == g["plane_" + k]) or \
                (vid != g["video_" + k]).sum() <= (got[k] != g["plane_" + k]).sum()
        else:
            assert np.array_equal(vid, g["video_" + k]), k
    # capture changes no row and no counter
    em0, rows0, _ = _run_replay(g, **_kw(g, show=False))
    assert len(rows) == len(rows0)
    for a, b in zip(rows, rows0):
        assert (a is None and b is None) or np.array_equal(a, b)
    assert (em.num_events_on, em.num_events_off, em.num_events_total) == \
        (em0.num_events_on, em0.num_events_off, em0.num_events_total)
    assert em0._lib.v2e_emu_model_state_device(em0._h) == -1


@pytest.mark.gpu
@pytest.mark.parametrize("mfs", [1, 2, 7, 64])
def test_multi_frame_path_equals_reference(mfs):
    """Noise-free fixture, device RNG, through the multi-frame kernels (chunks accepted and rejected) and a capacity
    resume: the planes equal the reference's, every frame exactly once; rows and offsets equal a run without capture."""
    from v2e_b200 import EventEmulator
    g = load_golden("model_states_noise_free")
    for hint in (None, 64):
        em = EventEmulator(device="cuda", rng=TapeRNG(g["tape"]), rng_mode="device", max_frames_per_step=mfs,
                           row_order="canonical", **_kw(g))
        em.event_rows_hint = hint
        rows, offs = em.generate_events_batch(g["frames"], g["times"])
        ms = em.model_state_frames()
        assert np.array_equal(ms["frame"], g["frame_counter"])
        assert np.array_equal(ms["t_previous"], g["t_previous"])
        for k in _shown(g):
            assert np.array_equal(ms[k].cpu().numpy(), g["plane_" + k]), (mfs, hint, k)
        if mfs == 64:
            multi, single = _fused_frames(em)
            assert multi >= 2 and single >= 1, (multi, single)
        em0 = EventEmulator(device="cuda", rng=TapeRNG(g["tape"]), rng_mode="device", max_frames_per_step=mfs,
                            row_order="canonical", **_kw(g, show=False))
        em0.event_rows_hint = hint
        rows0, offs0 = em0.generate_events_batch(g["frames"], g["times"])
        assert np.array_equal(rows, rows0) and np.array_equal(offs, offs0)
        assert em.num_events_total == em0.num_events_total


def _fused_frames(em):
    import ctypes
    multi, single = ctypes.c_longlong(0), ctypes.c_longlong(0)
    em._lib.v2e_emu_fused_frames(em._h, ctypes.byref(multi), ctypes.byref(single))
    return multi.value, single.value


@pytest.mark.gpu
@pytest.mark.parametrize("preset", ["cli", "noisy"])
def test_device_rng_1280x720_paths_agree(preset):
    """A smooth texture translating 1 px per frame, device RNG with noise: the multi-frame planes equal the
    frame-by-frame path's; new_frame is the input, log_new_frame and lp_log_frame the oracle's planes of the input's
    lin_log and of the final low-passed state."""
    import torch
    from v2e_b200 import EventEmulator
    from scipy.ndimage import gaussian_filter
    T, H, W = 10, 720, 1280
    big = gaussian_filter(np.random.default_rng(3).uniform(0, 255, (H + T, W + 2 * T)), 4)
    big = (big - big.min()) / (big.max() - big.min()) * 200 + 20
    frames = np.stack([big[k // 2:k // 2 + H, k:k + W] for k in range(T)]).round().astype(np.uint8)
    ts = np.arange(T) * 1e-3
    kw = dict(cutoff_hz=300, leak_rate_hz=0.01, shot_noise_rate_hz=0.001, refractory_period_s=0.0005,
              sigma_thres=0.03) if preset == "cli" else \
        dict(cutoff_hz=30, leak_rate_hz=0.1, shot_noise_rate_hz=5.0, sigma_thres=0.05)
    kw.update(rng_mode="device", seed=5, show_dvs_model_state=["all"])
    out = []
    for fused in (True, False):
        em = EventEmulator(device="cuda", fused=fused, **kw)
        em.generate_events_batch(frames, ts)
        ms = em.model_state_frames()
        out.append((em, {k: ms[k].cpu().numpy() for k in em._ms_names}))
    (emf, a), (_, b) = out
    assert _fused_frames(emf)[0] >= 2
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    assert np.array_equal(a["new_frame"], frames[1:])
    from v2e_b200.emulator import _linlog_lut
    lut = _linlog_lut().numpy()
    assert np.array_equal(a["log_new_frame"], mso.plane(lut[frames[1:]], "log_new_frame"))
    lp = emf.lp_log_frame.cpu().numpy()
    assert np.array_equal(a["lp_log_frame"][-1], mso.plane(lp, "lp_log_frame"))
    torch.cuda.synchronize()


# ---- pixel-sharded (gloo ranks on the test GPU) -----------------------------------------------------------------------
def _band_worker(rank, world, port, q, name, mode, outdir):
    from test_sharded_options import _init
    import torch.distributed as dist
    _init(rank, world, port)
    try:
        from v2e_b200 import EventEmulator
        log = []
        mod = types.ModuleType("v2ecore.v2e_utils")
        mod.video_writer = lambda fn, h, w: log.append(fn)
        sys.modules["v2ecore"] = types.ModuleType("v2ecore")
        sys.modules["v2ecore.v2e_utils"] = mod
        g = load_golden(name)
        extra = {"pr_vrms_tape": list(g["pr_vrms"])} if "pr_vrms" in g else {}
        if mode == "batch":
            extra["rng_mode"] = "device"
        em = EventEmulator(device="cuda:0", shard=(rank, world, None), rng=TapeRNG(g["tape"]),
                           **_kw(g, outdir), **extra)
        frames, times = g["frames"], g["times"]
        H = frames.shape[1]
        y0, y1 = em.ext_band(H)
        planes = {}
        if mode == "batch":
            em.generate_events_band_batch(frames[:, y0:y1], times, H)
            ms = em.model_state_frames()
            planes = {k: ms[k].cpu().numpy() for k in em._ms_names}
        else:
            for f, t in zip(frames, times):
                em.generate_events_band(f[y0:y1], float(t), H)
                if em._ms_chunks:
                    ms = em.model_state_frames()
                    for k in em._ms_names:
                        planes.setdefault(k, []).append(ms[k].cpu().numpy())
            planes = {k: np.concatenate(v) for k, v in planes.items()}
        em.cleanup()
        q.put((rank, (planes, log)))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("name,world,mode", [
    ("model_states_cs_f64", 2, "band"), ("model_states_cs_f64", 3, "band"), ("model_states_scidvs", 2, "band"),
    ("model_states_prnoise", 3, "band"), ("model_states_noise_free", 2, "batch"),
    ("model_states_noise_free", 3, "batch")])
def test_sharded_bands_concatenate_to_one_gpu_planes(name, world, mode, tmp_path):
    from test_sharded_options import _spawn
    g = load_golden(name)
    res = _spawn(world, _band_worker, name, mode, str(tmp_path))
    got = {k: np.concatenate([res[r][0][k] for r in range(world)], axis=1) for k in _shown(g)}
    _compare_planes(g, got, name)
    for r in range(world):
        assert res[r][1] == []
    assert os.listdir(tmp_path) == []
