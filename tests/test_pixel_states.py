"""Single-pixel recording (record_single_pixel_states, emulator.py:278-302, 985-1009; record_pixels): the fixtures
made by oracle/make_golden_pixel_states.py from the unmodified reference, the recorder's save / overflow logic, the
probe-off build of the multi-frame kernel, and (GPU) the device's samples on every path against the fixtures."""
import os
import pickle
import re
import subprocess

import numpy as np
import pytest

from helpers import TapeRNG, load_golden

NAMES = ("time", "new_frame", "base_log_frame", "lp_log_frame", "log_new_frame", "pos_thres", "neg_thres",
         "diff_frame", "final_neg_evts_frame", "final_pos_evts_frame")
REPLAY = ["pixel_states_cli", "pixel_states_noisy", "pixel_states_class_default", "pixel_states_sigma0",
          "pixel_states_hdr", "pixel_states_cs_f64", "pixel_states_cs_f32", "pixel_states_scidvs",
          "pixel_states_prnoise", "pixel_states_noise_free"]


# ---- fixtures (CPU) -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", REPLAY + ["pixel_states_overflow"])
def test_fixture_counts_and_final_state(name):
    """Per frame, the recorded final counts are the reference's rows at the pixel minus its shot rows (no shot noise:
    equal; with it: at most the rows); the last sample's lp / base are the final state at the pixel."""
    g = load_golden(name)
    counts = g["event_counts"]
    off = np.concatenate([[0], np.cumsum(counts)])
    noisy = g["kwargs"].get("shot_noise_rate_hz", 0) > 0 or g["kwargs"].get("photoreceptor_noise")
    for j, (r, c) in enumerate(g["pixels"]):
        n = int(g["sample_count"][j])
        assert n == min(len(counts) - 1, int(g.get("max_samples", 10000)))
        for k in range(n):
            ev = g["events"][off[k + 1]:off[k + 2]]
            at = ev[(ev[:, 1] == c) & (ev[:, 2] == r)]
            pos, neg = int((at[:, 3] > 0).sum()), int((at[:, 3] < 0).sum())
            got = (g["rec_final_pos_evts_frame"][j, k], g["rec_final_neg_evts_frame"][j, k])
            if noisy:
                assert got[0] <= pos and got[1] <= neg, (name, j, k)
            else:
                assert got == (pos, neg), (name, j, k)
        assert np.all(np.isnan(g["rec_time"][j, n:]))
        if n == len(counts) - 1:
            assert g["rec_lp_log_frame"][j, n - 1] == g["state_lp_log_frame"][r, c]
            assert g["rec_base_log_frame"][j, n - 1] == g["state_base_log_frame"][r, c]


def test_fixtures_are_reproducible():
    """Re-running the generator's reference path gives the same arrays (one fixture, one pixel)."""
    import sys
    here = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle")
    sys.path.insert(0, here)
    import ref_shim
    from make_golden import run_reference
    try:
        emu_mod = ref_shim.load_reference()[0]
    except Exception as e:
        pytest.skip("the reference emulator is not importable here (%s)" % e)
    g = load_golden("pixel_states_cli")
    r, c = (int(v) for v in g["pixels"][0])
    cwd = os.getcwd()
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        os.chdir(d)
        try:
            em, _, _ = run_reference(emu_mod, dict(g["kwargs"], record_single_pixel_states=(r, c)), g["frames"],
                                     g["times"], int(g["seed"]))
        finally:
            os.chdir(cwd)
    for k in NAMES:
        assert np.array_equal(em.single_pixel_states[k], g["rec_" + k][0], equal_nan=True), k
    em.record_single_pixel_states = None


# ---- recorder logic with the library stubbed (CPU) ------------------------------------------------------
def _stub_emulator(monkeypatch, **kw):
    from v2e_b200 import emulator as em_mod
    monkeypatch.setattr(em_mod._lib, "load", lambda *a, **k: object())
    e = em_mod.EventEmulator(device="cuda", **kw)
    e._finalizer.detach()
    return e, em_mod


def _samples(em_mod, nf, value):
    s = np.zeros((nf, 1), dtype=em_mod._PROBE_DTYPE)
    for f in range(nf):
        for name in em_mod._PROBE_DTYPE.names:
            s[f, 0][name] = value + f
    return s


def test_recorder_saves_reference_pickle_at_cleanup(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    e, em_mod = _stub_emulator(monkeypatch, record_single_pixel_states=(5, 17))
    e._spx["col"] = 0
    e._record(_samples(em_mod, 3, 1), [1e-3, 2e-3, 3e-3])
    assert e.single_pixel_sample_count == 3
    assert not os.path.exists("pixel-states.dat")
    e._hbox[0] = None
    e.cleanup()
    with open(tmp_path / "pixel-states.dat", "rb") as fh:
        d = pickle.load(fh)
    assert sorted(d) == sorted(NAMES)
    for k in NAMES:
        assert d[k].dtype == np.float64 and d[k].shape == (10000,)
        assert np.all(np.isnan(d[k][3:]))
    assert list(d["time"][:3]) == [1e-3, 2e-3, 3e-3]
    assert list(d["final_pos_evts_frame"][:3]) == [1.0, 2.0, 3.0]


def test_recorder_overflow_saves_and_stops(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    from v2e_b200 import emulator as em_mod
    monkeypatch.setattr(em_mod.EventEmulator, "SINGLE_PIXEL_MAX_SAMPLES", 4)
    e, em_mod = _stub_emulator(monkeypatch, record_single_pixel_states=(0, 0))
    e._spx["col"] = 0
    e._record(_samples(em_mod, 4, 0), [0.1, 0.2, 0.3, 0.4])
    assert not os.path.exists("pixel-states.dat")
    e._record(_samples(em_mod, 2, 10), [0.5, 0.6])      # the 5th frame saves and stops; the 6th is not recorded
    assert e.record_single_pixel_states is None and e.single_pixel_sample_count == 4
    with open("pixel-states.dat", "rb") as fh:
        d = pickle.load(fh)
    assert list(d["time"]) == [0.1, 0.2, 0.3, 0.4]
    os.remove("pixel-states.dat")
    e._hbox[0] = None
    e.cleanup()
    assert not os.path.exists("pixel-states.dat")


def test_no_keyword_no_file(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    e, _ = _stub_emulator(monkeypatch)
    assert e.single_pixel_states is None
    e._hbox[0] = None
    e.cleanup()
    assert os.listdir(tmp_path) == []


def test_record_pixels_is_validated(monkeypatch):
    with pytest.raises(ValueError):
        _stub_emulator(monkeypatch, record_pixels=[(1, 2)] * 65)
    with pytest.raises(ValueError):
        _stub_emulator(monkeypatch, record_pixels=[(1, 2.0)])


# ---- the probe-off multi-frame kernel is the kernel without probes (CPU) -----------------------------------
# cuobjdump -res-usage of emu_fused_update_kernel<S, FAST> built without probes: registers, stack, shared memory,
# local memory
PROBE_OFF_USAGE = {
    ("f", 0): (96, 96, 5120, 0), ("f", 1): (90, 96, 5120, 0), ("d", 0): (96, 112, 5120, 0), ("d", 1): (96, 96, 5120, 0),
}


def test_probe_off_fused_kernel_resources_unchanged_at_the_4x5_block_shape():
    from test_conv_sass import _cuobjdump
    from v2e_b200 import build as _build
    lib = _build.build()
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    out = subprocess.run([tool, "-res-usage", lib], check=True, capture_output=True, text=True).stdout
    got = {}
    lines = out.splitlines()
    for i, line in enumerate(lines):
        m = re.search(r"emu_fused_update_kernelI([fd])Lb([01])ELb([01])E", line)
        if m and m.group(3) == "0":
            u = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", lines[i + 1])
            got[(m.group(1), int(m.group(2)))] = tuple(int(v) for v in u.groups())
    assert got == PROBE_OFF_USAGE


# ---- GPU ---------------------------------------------------------------------------------------------------
def _emulator(**kw):
    from v2e_b200 import EventEmulator
    return EventEmulator(device="cuda", **kw)


def _replay(g, pixel, **extra):
    kw = dict(g["kwargs"])
    if "pr_vrms" in g:
        extra["pr_vrms_tape"] = list(g["pr_vrms"])
    em = _emulator(rng=TapeRNG(g["tape"]), record_single_pixel_states=pixel, **kw, **extra)
    for f, t in zip(g["frames"], g["times"]):
        em.generate_events(f, float(t))
    return em


@pytest.mark.gpu
@pytest.mark.parametrize("name", REPLAY)
def test_replay_mode_equals_reference(name, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    g = load_golden(name)
    for j, (r, c) in enumerate(g["pixels"]):
        em = _replay(g, (int(r), int(c)))
        assert em.single_pixel_sample_count == int(g["sample_count"][j])
        for k in NAMES:
            assert np.array_equal(em.single_pixel_states[k], g["rec_" + k][j], equal_nan=True), (name, (r, c), k)
        em.record_single_pixel_states = None


@pytest.mark.gpu
def test_overflow_saves_the_file(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    from v2e_b200 import EventEmulator
    g = load_golden("pixel_states_overflow")
    monkeypatch.setattr(EventEmulator, "SINGLE_PIXEL_MAX_SAMPLES", int(g["max_samples"]))
    r, c = (int(v) for v in g["pixels"][0])
    em = _replay(g, (r, c))
    assert em.record_single_pixel_states is None and em.single_pixel_sample_count == int(g["max_samples"])
    with open("pixel-states.dat", "rb") as fh:
        d = pickle.load(fh)
    for k in NAMES:
        assert np.array_equal(d[k], g["rec_" + k][0], equal_nan=True), k


def _device_traces(g, pixels, **kw):
    em = _emulator(rng=TapeRNG(g["tape"]), rng_mode="device", record_pixels=pixels, **g["kwargs"], **kw)
    em.generate_events_batch(g["frames"], g["times"])
    return em, em.pixel_traces()


@pytest.mark.gpu
def test_device_mode_multi_frame_path_equals_reference():
    """Noise-free fixture through the multi-frame kernels: bit for bit, with chunks both accepted and rejected, and
    the same trace for any chunk length and frame by frame."""
    import ctypes
    g = load_golden("pixel_states_noise_free")
    pixels = [(int(r), int(c)) for r, c in g["pixels"]]
    em, tr = _device_traces(g, pixels)
    chunks, rejected = ctypes.c_longlong(0), ctypes.c_longlong(0)
    em._lib.v2e_emu_fused_stats(em._h, ctypes.byref(chunks), ctypes.byref(rejected))
    assert chunks.value >= 1 and rejected.value >= 1, (chunks.value, rejected.value)
    multi, single = ctypes.c_longlong(0), ctypes.c_longlong(0)
    em._lib.v2e_emu_fused_frames(em._h, ctypes.byref(multi), ctypes.byref(single))
    assert multi.value >= 2 and single.value >= 1, (multi.value, single.value)
    n = int(g["sample_count"][0])
    for k in NAMES:
        want = g["rec_" + k][:, :n].T
        assert np.array_equal(tr[k], want[:, 0] if k == "time" else want), k
    for kw in (dict(max_frames_per_step=2), dict(max_frames_per_step=7), dict(fused=False)):
        _, tr2 = _device_traces(g, pixels, **kw)
        for k in NAMES:
            assert np.array_equal(tr2[k], tr[k], equal_nan=True), (kw, k)


def _fused_frames(em):
    import ctypes
    multi, single = ctypes.c_longlong(0), ctypes.c_longlong(0)
    em._lib.v2e_emu_fused_frames(em._h, ctypes.byref(multi), ctypes.byref(single))
    return multi.value, single.value


def _fused_stats(em):
    import ctypes
    chunks, rejected = ctypes.c_longlong(0), ctypes.c_longlong(0)
    em._lib.v2e_emu_fused_stats(em._h, ctypes.byref(chunks), ctypes.byref(rejected))
    return chunks.value, rejected.value


def _smooth_frames(T, H, W, seed):
    from scipy.ndimage import gaussian_filter
    big = gaussian_filter(np.random.default_rng(seed).uniform(0, 255, (H + T, W + 2 * T)), 3)
    big = (big - big.min()) / (big.max() - big.min()) * 200 + 20
    return np.stack([big[k // 2:k // 2 + H, k:k + W] for k in range(T)]).round().astype(np.uint8)


@pytest.mark.gpu
def test_device_mode_noisy_paths_agree():
    """CLI defaults with leak, shot and refractory in device mode (the multi-frame kernel's FAST instantiation): the
    multi-frame path, the frame-by-frame kernels and capacity resumes record the same traces; recording changes no row
    (canonical order, whose key is a function of the row), offset or counter."""
    T, H, W = 24, 48, 64
    frames = _smooth_frames(T, H, W, 1)
    ts = np.arange(T) * 1e-3
    kw = dict(cutoff_hz=300, leak_rate_hz=0.5, shot_noise_rate_hz=20.0, refractory_period_s=0.0005,
              sigma_thres=0.03, seed=7, rng_mode="device", row_order="canonical")
    pixels = [(0, 0), (5, 17), (23, 40), (47, 63), (12, 3), (30, 31)]

    def run(probe, **extra):
        em = _emulator(**kw, **extra, **({"record_pixels": pixels} if probe else {}))
        rows, offs = em.generate_events_batch(frames, ts)
        return em, rows, offs

    em_f, rows_f, offs_f = run(True)
    multi, _ = _fused_frames(em_f)
    assert multi >= T // 2, "the multi-frame kernels must have taken most frames (%d)" % multi
    em_s, rows_s, offs_s = run(True, fused=False)
    assert _fused_frames(em_s) == (0, 0)
    em_c, rows_c, offs_c = run(True, max_frames_per_step=5)
    em_0, rows_0, offs_0 = run(False)
    tf = em_f.pixel_traces()
    for other in (em_s, em_c):
        to = other.pixel_traces()
        for k in NAMES:
            assert np.array_equal(to[k], tf[k], equal_nan=True), k
    counters = lambda e: (e.num_events_on, e.num_events_off, e.num_events_total)
    for em, rows, offs in ((em_s, rows_s, offs_s), (em_c, rows_c, offs_c), (em_f, rows_f, offs_f)):
        assert np.array_equal(offs, offs_0) and np.array_equal(rows, rows_0)
        assert counters(em) == counters(em_0)
    assert np.nansum(tf["final_pos_evts_frame"]) + np.nansum(tf["final_neg_evts_frame"]) > 0
    # capacity resumes: a tiny initial event buffer has to grow (V2E_E_CAPACITY, then resume) during the clip
    em_r = _emulator(**kw, record_pixels=pixels)
    em_r.event_rows_hint = 64
    rows_r, offs_r = em_r.generate_events_batch(frames, ts)
    assert em_r._ev_dev.shape[0] > 64, "no capacity resume happened"
    assert np.array_equal(rows_r, rows_0) and np.array_equal(offs_r, offs_0)
    assert counters(em_r) == counters(em_0)
    tr = em_r.pixel_traces()
    for k in NAMES:
        assert np.array_equal(tr[k], tf[k], equal_nan=True), k


@pytest.mark.gpu
def test_probe_buffers_live_on_the_handles_device():
    """The probe buffers are allocated on the emulator's device even when another device is current."""
    import torch
    n = torch.cuda.device_count()
    dev = n - 1
    from v2e_b200 import EventEmulator
    em = EventEmulator(device="cuda:%d" % dev, record_pixels=[(1, 2)], cutoff_hz=300, sigma_thres=0.03,
                       leak_rate_hz=0)
    fr = _smooth_frames(4, 16, 24, 3)
    with torch.cuda.device(0):
        em.generate_events_batch(fr, np.arange(4) * 1e-3)
    assert em._lib.v2e_emu_probe_device(em._h) == dev
    assert em.pixel_traces()["time"].shape == (3,)


# ---- pixel-sharded (gloo ranks on the test GPU) -------------------------------------------------------------
def _band_worker(rank, world, port, q, name, mode, outdir):
    from test_sharded_options import _init
    import torch.distributed as dist
    _init(rank, world, port)
    try:
        from v2e_b200 import EventEmulator
        g = load_golden(name)
        os.chdir(os.path.join(outdir, str(rank)))
        pixels = [(int(r), int(c)) for r, c in g["pixels"]]
        extra = {"pr_vrms_tape": list(g["pr_vrms"])} if "pr_vrms" in g else {}
        if mode == "batch":
            extra["rng_mode"] = "device"
        em = EventEmulator(device="cuda:0", shard=(rank, world, None), rng=TapeRNG(g["tape"]), record_pixels=pixels,
                           record_single_pixel_states=pixels[0], **extra, **g["kwargs"])
        frames, times = g["frames"], g["times"]
        H = frames.shape[1]
        y0, y1 = em.ext_band(H)
        if mode == "frame":
            for f, t in zip(frames, times):
                em.generate_events(f, float(t))
        elif mode == "band":
            for f, t in zip(frames, times):
                em.generate_events_band(f[y0:y1], float(t), H)
        else:
            em.generate_events_band_batch(frames[:, y0:y1], times, H)
        states = {k: np.array(v) for k, v in em.single_pixel_states.items()}
        res = (em.pixel_traces(), em.single_pixel_sample_count, states, _fused_stats(em) if mode == "batch" else None)
        em.cleanup()
        em.record_single_pixel_states = None
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("name,world,mode", [
    ("pixel_states_cli", 2, "frame"), ("pixel_states_cs_f64", 2, "frame"), ("pixel_states_cs_f64", 3, "band"),
    ("pixel_states_cs_f32", 2, "band"), ("pixel_states_scidvs", 2, "band"), ("pixel_states_prnoise", 3, "frame"),
    ("pixel_states_noise_free", 2, "batch"), ("pixel_states_noise_free", 3, "batch")])
def test_sharded_owner_records_what_one_gpu_records(name, world, mode, tmp_path):
    """Each fixture pixel (band-edge rows among them) is recorded by the rank whose own rows hold it, equal to the
    reference's (centre-surround with halo rows, SCIDVS, photoreceptor noise: replay mode; noise-free: device mode
    through generate_events_band_batch's split multi-frame path); the other ranks record nothing and write no file."""
    from test_sharded_options import _spawn
    from v2e_b200.parallel import row_band

    def row_band_of(H, world, row):
        return next(r for r in range(world) if row_band(H, r, world)[0] <= row < row_band(H, r, world)[1])
    g = load_golden(name)
    for r in range(world):
        os.makedirs(tmp_path / str(r))
    res = _spawn(world, _band_worker, name, mode, str(tmp_path))
    H = g["frames"].shape[1]
    n = int(g["sample_count"][0])
    for j, (r, c) in enumerate(g["pixels"]):
        owner = row_band_of(H, world, int(r))
        for rank in range(world):
            tr = res[rank][0]
            for k in NAMES[1:]:
                got = tr[k][:, j]
                if rank == owner:
                    assert np.array_equal(got, g["rec_" + k][j, :n]), (name, world, (r, c), k)
                else:
                    assert np.all(np.isnan(got)), (name, world, rank, (r, c), k)
    owner0 = row_band_of(H, world, int(g["pixels"][0][0]))
    for rank in range(world):
        _, count, states, ff = res[rank]
        saved = os.listdir(tmp_path / str(rank))
        if rank == owner0:
            assert count == n and saved == ["pixel-states.dat"]
            for k in NAMES:
                assert np.array_equal(states[k], g["rec_" + k][0], equal_nan=True), k
        else:
            assert count == 0 and saved == [] and np.all(np.isnan(states["time"]))
        if ff is not None:          # multi-frame chunks both accepted and rejected (then replayed frame by frame)
            assert ff[1] >= 1 and ff[0] > ff[1], ff
