"""Long clips: the pixel model, the event sinks, the streamed pipeline and the renderer at absolute times of tens of
minutes to ten hours, where float32 time arithmetic changes character. At 2500 s one float32 ulp is 2.4e-4 s, at
36 000 s it is 3.9e-3 s, longer than a 1/300 s frame interval: a frame's linspace of iteration timestamps (make_ts in
emu.cu) then collapses to one value, and the refractory test (t - timestamp_mem) > refractory_period_s in float32
decides on quantised differences. Every comparison here is against the plain references the suite trusts, bit for bit.

A fresh emulator does not advance t_previous on its first frame (the reference returns early, emulator.py:717), so the
second frame's delta_time is its whole absolute time. The noise rates scale with 1 / T0 to keep that one frame bounded,
and the centre-surround time constants scale with T0 to keep its Euler steps within cs_cap (8192).

CPU: the AEDAT-2.0 and HDF5 timestamp rules of oracle/sinks_oracle.py against the reference's writer (fixture) and
numpy; the oracle's sensitivity to time rounding; that the 36 000 s clips collapse frames' timestamp ranges.
GPU: single-frame path (replay RNG), generate_events_batch one and several frames per step and device-RNG draws,
both row orders, the centre-surround model on its cooperative and per-step paths -- all against the CPU oracle at
T0 in {1000, 2147.5, 5000, 36 000} s, 37x53 and 260x346; the sink kernels and the files generate_events and
generate_events_batch write across 2^31 us and 2^32 us; V2EPipeline.run_segments streaming across 2^31 us; the
renderer's long-clip fixtures."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

import row_order
import sinks_oracle
import text_sink_oracle
from helpers import DeviceDrawRNG, GOLDEN_DIR, assert_events_equal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T0S = [1000.0, 2147.5, 5000.0, 36000.0]
SIZES = [(37, 53), (260, 346)]
T = 12
SEED = 21
US31 = np.float32(2147.483648)          # 2^31 us: the AEDAT-2.0 int32 timestamp's range ends here
US32 = np.float32(4294.967296)          # 2^32 us: the HDF5 uint32 timestamp's


def ulp32(t):
    t = np.float32(t)
    return float(np.nextafter(t, np.float32(np.inf)) - t)


def configs(t0):
    """name -> EventEmulator / OracleEmulator keywords for a clip at T0 = t0."""
    noise = dict(leak_rate_hz=0.5 / t0, shot_noise_rate_hz=0.5 / t0)
    return {
        # float64 state; refractory filter active whenever a frame has 2 or more iterations (3.2e-3 > dt / max_n)
        "f64_refractory": dict(cutoff_hz=300.0, refractory_period_s=0.0032, **noise),
        # float32 state (cutoff_hz = 0), no refractory filter: the multi-frame kernels accept every chunk
        "f32_free": dict(cutoff_hz=0.0, refractory_period_s=0.0, **noise),
    }


def cs_config(t0):
    """Centre-surround: tau_h = tau_p / 16 = t0 / 1000 s, so frame 1 (delta_time ~ t0) takes at most ~5000 steps."""
    return dict(cutoff_hz=100.0, refractory_period_s=0.0032, leak_rate_hz=0.0, shot_noise_rate_hz=0.0,
                cs_lambda_pixels=4, cs_tau_p_ms=16.0 * t0)


def clip(H, W, t0, seed=0, contrast="high"):
    """T frames of a texture moving 2 px per frame, 1/300 s apart from t0. "high": values 0..255, up to ~70 events of
    one pixel in a frame; "low": 64..191, at most ~12, below the multi-frame kernels' limit of 31 (kFusedMaxN)."""
    from test_emulator_device_rng import texture_frames
    fr = texture_frames(H, W, T, seed=seed + H, speed=2.0)
    if contrast == "low":
        fr = fr // 2 + 64
    return fr, [t0 + k / 300.0 for k in range(T)]


def _frames(rows, offs):
    return [rows[offs[i]:offs[i + 1]] for i in range(len(offs) - 1)]


def oracle_run(kw, frames, ts, rng=None, seed=SEED, shuffle=True):
    """OracleEmulator over a clip: (per-frame rows as it returns them, per-frame iteration counts [m, 2], oracle)."""
    from emu_oracle import OracleEmulator
    orc = OracleEmulator(seed=seed, rng=rng, shuffle=shuffle, **kw)
    rows, iters = [], []
    for k, (f, t) in enumerate(zip(frames, ts)):
        if isinstance(rng, DeviceDrawRNG):
            rng.frame = k
        ev = orc.generate_events(f, float(t))
        rows.append(np.zeros((0, 4), np.float32) if ev is None else ev)
        iters.append(orc.last_iter_counts if k else np.zeros((0, 2), np.int32))
    return rows, iters, orc


def oracle_state(orc):
    return {k: v for k, v in (("lp_log_frame", orc.lp), ("base_log_frame", orc.base), ("timestamp_mem", orc.tmem))
            if v is not None}


def device_state(em):
    out = {}
    for k in ("lp_log_frame", "base_log_frame", "timestamp_mem"):
        v = getattr(em, k)
        if v is not None:
            out[k] = v.cpu().numpy()
    return out


def assert_state_equal(got, want, ctx):
    assert got.keys() == want.keys(), ctx
    for k in want:
        assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), (ctx, k)


def assert_rows_equal(got_frames, want_frames, ctx):
    """Rows of every frame, values and order, bit for bit."""
    assert len(got_frames) == len(want_frames), ctx
    for i, (g, w) in enumerate(zip(got_frames, want_frames)):
        g = np.zeros((0, 4), np.float32) if g is None else np.asarray(g)
        assert g.shape == w.shape, "%s frame %d: %s rows vs oracle %s" % (ctx, i, g.shape, w.shape)
        assert g.tobytes() == w.tobytes(), "%s frame %d" % (ctx, i)


def stamp_ranges(iters, ts):
    """(start, end) of make_ts for every frame k >= 1 with events: float32(t_prev + dt / max_n), float32(t_frame),
    t_prev = 0 for frame 1 (the first frame does not advance it)."""
    out = []
    for k in range(1, len(ts)):
        m = len(iters[k])
        if m:
            tp = ts[k - 1] if k > 1 else 0.0
            out.append((np.float32(tp + (ts[k] - tp) / m), np.float32(ts[k]), m))
    return out


# ---- CPU: the sink rules --------------------------------------------------------------------------------------------
def test_aedat2_oracle_matches_reference_writer_past_2_31_us():
    """Rows from 2140 s to 36 001 s written by the reference's own AEDat2Output: timestamps at or past 2^31 us are
    INT32_MIN in its file, as the oracle's rule states."""
    g = np.load(os.path.join(GOLDEN_DIR, "sinks_aedat2.npz"))
    ev = g["events_long"]
    words, _ = sinks_oracle.aedat2_words(ev, 346, 260)
    assert words.tobytes() == g["body_long"].tobytes()
    t = words.byteswap()[1::2]
    out = ev[:, 0] * np.float32(1e6) >= np.float32(2.0 ** 31)
    assert out.sum() > 300 and (~out).sum() > 300
    assert np.all(t[out] == np.int32(-2 ** 31)) and np.all(t[~out] >= 2140 * 10 ** 6)
    assert np.float32(np.nextafter(US31, np.float32(0))) in ev[:, 0] and US31 in ev[:, 0]


def test_int32_rule_at_its_edges():
    v = np.array([np.nan, -np.inf, np.inf, -2.0 ** 31, -2.0 ** 31 - 256, 2.0 ** 31, 2.0 ** 31 - 128, -0.5, 2.9, -2.9,
                  3e9], np.float32)
    want = [-2 ** 31, -2 ** 31, -2 ** 31, -2 ** 31, -2 ** 31, -2 ** 31, 2 ** 31 - 128, 0, 2, -2, -2 ** 31]
    assert sinks_oracle.trunc_int32(v).tolist() == want


def test_h5_rule_equals_numpy_below_2_32_us_and_wraps_past_it():
    """Every float32 time whose microseconds lie in [0, 2^32): numpy's exact cast. Sampled over the whole range, and
    the last 4096 float32 times below 2^32 us. Past it, the wrap mod 2^32."""
    rng = np.random.default_rng(1)
    t = np.concatenate([rng.uniform(0, 4294.967296, 200000).astype(np.float32),
                        np.nextafter(US32, np.float32(0)) - np.arange(4096, dtype=np.float32) * ulp32(4294.0)])
    t_us = t * np.float32(1e6)
    keep = t_us < np.float32(2.0 ** 32)
    assert keep.sum() > 200000
    ev = np.stack([t[keep], np.full(keep.sum(), 5, np.float32), np.full(keep.sum(), 7, np.float32),
                   np.where(np.arange(keep.sum()) % 2, 1.0, -1.0).astype(np.float32)], 1)
    want = np.array(ev, np.float32)
    want[:, 0] *= np.float32(1e6)
    want[want[:, 3] == -1, 3] = 0
    assert np.array_equal(sinks_oracle.h5_rows(ev), want.astype(np.uint32))
    t_last = t[keep].max()                       # the last float32 time whose microseconds are below 2^32
    assert np.nextafter(t_last, np.float32(np.inf)) * np.float32(1e6) >= np.float32(2.0 ** 32)
    assert sinks_oracle.h5_rows(ev)[:, 0].max() >= 2 ** 32 - 1024
    past = np.array([[4294.967296, 1, 2, 1], [5000.0, 1, 2, 1], [36000.0, 1, 2, -1]], np.float32)
    got = sinks_oracle.h5_rows(past)[:, 0]
    assert got.tolist() == [int(v) % 2 ** 32 for v in (past[:, 0] * np.float32(1e6)).astype(np.float64)]


# ---- CPU: the oracle sees time rounding -----------------------------------------------------------------------------
def test_clips_at_36000_s_collapse_frames_timestamp_ranges():
    """At 36 000 s a frame's iteration timestamps collapse: make_ts' start (float32 of t_prev + dt / max_n) is not
    below its end for frames with several iterations."""
    t0 = 36000.0
    for H, W in SIZES:
        fr, ts = clip(H, W, t0)
        _, iters, _ = oracle_run(configs(t0)["f64_refractory"], fr, ts)
        r = stamp_ranges(iters, ts)
        assert sum(1 for s, e, m in r if m >= 2 and s >= e) >= 2, r


def test_refractory_decisions_follow_time_rounding():
    """f64_refractory at 5000 s: one frame interval is 6.8 float32 ulps, so the difference of two frames' timestamps
    is 6 or 7 ulps (2.93e-3 or 3.42e-3 s) against a 3.2e-3 s refractory period. Shifting the clip by half an ulp
    changes which differences round to 7, and the events that pass: x / y / polarity change, not only t."""
    from helpers import canonical
    t0 = 5000.0
    kw = configs(t0)["f64_refractory"]
    fr, ts = clip(37, 53, t0)
    a, _, _ = oracle_run(kw, fr, ts, shuffle=False)
    b, _, _ = oracle_run(kw, fr, [t + ulp32(t0) / 2 for t in ts], shuffle=False)
    xyp = lambda rows: sorted(map(bytes, canonical(np.concatenate(rows))[:, 1:]))
    assert xyp(a) != xyp(b)


# ---- GPU: the pixel model -------------------------------------------------------------------------------------------
def _emulator(**kw):
    from v2e_b200 import EventEmulator
    return EventEmulator(device="cuda", **kw)


CASES = [(s, t0, c) for s in SIZES for t0 in T0S for c in ("f64_refractory", "f32_free")]
IDS = ["%dx%d-%g-%s" % (s[1], s[0], t0, c) for s, t0, c in CASES]


@pytest.mark.gpu
@pytest.mark.parametrize("size,t0,cfg", CASES, ids=IDS)
def test_single_frame_path_equals_oracle(size, t0, cfg):
    """generate_events frame by frame, replay RNG: rows in the reference's (shuffled) order, counters, lp / base /
    timestamp_mem, against the oracle on the same seed."""
    kw = configs(t0)[cfg]
    fr, ts = clip(*size, t0)
    want, iters, orc = oracle_run(kw, fr, ts)                # both draw from torch's global generator: one, then the other
    em = _emulator(seed=SEED, **kw)
    got = [em.generate_events(f, t) for f, t in zip(fr, ts)]
    assert_rows_equal(got, want, "single-frame")
    assert (em.num_events_on, em.num_events_off, em.num_events_total) == \
        (orc.num_events_on, orc.num_events_off, orc.num_events_total)
    assert_state_equal(device_state(em), oracle_state(orc), "single-frame")
    assert orc.num_events_total > 50


def _device_oracle(em, kw, fr, ts):
    from test_emulator_device_rng import draws_from
    rng = DeviceDrawRNG(draws_from(em))
    return oracle_run(kw, fr, ts, rng=rng, shuffle=False)


@pytest.mark.gpu
@pytest.mark.parametrize("contrast", ["high", "low"])
@pytest.mark.parametrize("mfps", [1, 8])
@pytest.mark.parametrize("size,t0,cfg", CASES, ids=IDS)
def test_batch_device_rng_equals_oracle(size, t0, cfg, mfps, contrast):
    """generate_events_batch with the device RNG, one frame per step (the frame-by-frame kernels) and 8 (the
    multi-frame kernels: on the low-contrast clip without a refractory period they emit the frames; where the
    refractory filter is active, or a pixel has more than 31 events, they reject the chunk and the frames are replayed
    frame by frame), canonical row order, against the oracle fed the device's draws."""
    import ctypes
    kw = configs(t0)[cfg]
    fr, ts = clip(*size, t0, contrast=contrast)
    em = _emulator(seed=SEED, rng_mode="device", row_order="canonical", max_frames_per_step=mfps, **kw)
    rows, offs = em.generate_events_batch(fr, ts)
    want, iters, orc = _device_oracle(em, kw, fr, ts)
    assert_rows_equal(_frames(rows, offs), want, "batch mfps=%d" % mfps)
    assert (em.num_events_on, em.num_events_off, em.num_events_total) == \
        (orc.num_events_on, orc.num_events_off, orc.num_events_total)
    assert_state_equal(device_state(em), oracle_state(orc), "batch")
    v = [ctypes.c_longlong(0) for _ in range(4)]
    em._lib.v2e_emu_fused_stats(em._h, ctypes.byref(v[0]), ctypes.byref(v[1]))
    em._lib.v2e_emu_fused_frames(em._h, ctypes.byref(v[2]), ctypes.byref(v[3]))
    chunks, rejected, multi, single = (x.value for x in v)
    if mfps == 1:
        assert chunks == 0
    else:
        assert chunks >= 1
        if contrast == "low" and cfg == "f32_free":
            assert multi >= T - 2, (chunks, rejected, multi, single)
        else:
            assert rejected >= 1, (chunks, rejected, multi, single)
    print("LONG %s %g %s %s mfps=%d rows=%d chunks=%d rejected=%d frames multi=%d single=%d" % (
        size, t0, cfg, contrast, mfps, len(rows), chunks, rejected, multi, single))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["canonical", "shuffled"])
@pytest.mark.parametrize("t0", T0S)
@pytest.mark.parametrize("size", SIZES, ids=["53x37", "346x260"])
def test_row_orders_equal_oracle(size, t0, mode):
    """row_order canonical and shuffled, unsorted, against the oracle's rows put in that order by oracle/row_order.py
    from its own per-iteration counts (at 36 000 s iterations share timestamps, so they cannot be told apart by t)."""
    kw = configs(t0)["f64_refractory"]
    H, W = size
    fr, ts = clip(H, W, t0)
    em = _emulator(seed=SEED, rng_mode="device", row_order=mode, max_frames_per_step=8, **kw)
    rows, offs = em.generate_events_batch(fr, ts)
    want, iters, orc = _device_oracle(em, kw, fr, ts)
    woffs = np.concatenate([[0], np.cumsum([len(r) for r in want])])
    assert np.array_equal(offs, woffs)
    counts = [it.sum(axis=1) for it in iters]
    n_shot = [len(r) - int(c.sum()) for r, c in zip(want, counts)]
    flat = np.concatenate(want)
    expect = row_order.order_rows(flat, woffs, counts, n_shot, mode, seed=SEED, W=W)
    assert rows.tobytes() == expect.tobytes()
    assert_state_equal(device_state(em), oracle_state(orc), mode)


@functools.lru_cache(maxsize=None)
def cs_oracle(size, t0):
    fr, ts = clip(*size, t0, seed=3)
    rows, _, orc = oracle_run(cs_config(t0), fr, ts, seed=11)
    return dict(rows=rows, steps=list(orc.cs_steps_taken), cs_surround_frame=orc.surround, **oracle_state(orc))


def cs_device(size, t0):
    fr, ts = clip(*size, t0, seed=3)
    em = _emulator(seed=11, **cs_config(t0))
    rows = [em.generate_events(f, t) for f, t in zip(fr, ts)]
    out = dict(rows=[np.zeros((0, 4), np.float32) if r is None else r for r in rows], steps=list(em.cs_steps_taken),
               paths=em.cs_paths(), cs_surround_frame=em.cs_surround_frame.cpu().numpy(), **device_state(em))
    return out


def _cs_per_step_worker(cases, q):
    os.environ["V2E_CS_COOP"] = "0"     # read once, at the first centre-surround frame of the process
    try:
        for c in cases:
            q.put((c, cs_device(*c)))
    except BaseException as e:          # report instead of leaving the parent waiting
        q.put(("error", repr(e)))


CS_CASES = [(s, t0) for s in SIZES for t0 in T0S]


@functools.lru_cache(maxsize=None)
def cs_per_step_results():
    from test_emulator_centre_surround import _spawn
    return dict(_spawn(_cs_per_step_worker, [(CS_CASES,)], len(CS_CASES)))


def _assert_cs(got, want, ctx):
    assert got["steps"] == want["steps"], (ctx, got["steps"], want["steps"])
    assert len(got["rows"]) == len(want["rows"])
    for i, (g, w) in enumerate(zip(got["rows"], want["rows"])):
        assert_events_equal(g, w, exact_order=False, ctx="%s frame %d" % (ctx, i))
    for k in ("cs_surround_frame", "lp_log_frame", "base_log_frame", "timestamp_mem"):
        assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), (ctx, k)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["coop", "per_step"])
@pytest.mark.parametrize("size,t0", CS_CASES, ids=["%dx%d-%g" % (s[1], s[0], t0) for s, t0 in CS_CASES])
def test_centre_surround_equals_oracle(size, t0, path):
    """The centre-surround model, single-frame path, on its cooperative launch (this process) and one kernel per Euler
    step (a spawned process with V2E_CS_COOP=0): rows of every frame (sorted: without per-frame noise the single-frame
    path does not replay the reference's shuffle), Euler steps, surround, lp, base and timestamp_mem."""
    want = cs_oracle(size, t0)
    got = cs_device(size, t0) if path == "coop" else cs_per_step_results()[(size, t0)]
    n = len(want["steps"])
    assert got["paths"] == ((n, 0) if path == "coop" else (0, n)), got["paths"]
    _assert_cs(got, want, "%s %s %g" % (path, size, t0))
    assert max(want["steps"]) > 100 and sum(len(r) for r in want["rows"]) > 20


@pytest.mark.gpu
def test_device_rows_differ_from_oracle_one_ulp_later():
    """The comparisons see time rounding: the oracle on the same clip shifted by one float32 ulp gives other rows."""
    t0 = 5000.0
    kw = configs(t0)["f64_refractory"]
    fr, ts = clip(37, 53, t0)
    em = _emulator(seed=SEED, rng_mode="device", row_order="canonical", max_frames_per_step=8, **kw)
    rows, offs = em.generate_events_batch(fr, ts)
    want, _, _ = _device_oracle(em, kw, fr, ts)
    shifted, _, _ = _device_oracle(em, kw, fr, [t + ulp32(t0) for t in ts])
    assert_rows_equal(_frames(rows, offs), want, "same clip")
    with pytest.raises(AssertionError):
        assert_rows_equal(_frames(rows, offs), shifted, "one ulp later")


# ---- GPU: the sink kernels ------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_sink_kernels_at_long_times():
    """AEDAT-2.0 words against the reference writer's bytes past 2^31 us; HDF5 rows against the oracle over
    [0, 2^32) us and its wrap past it; the text body against text_sink_oracle, with and without labels."""
    import torch
    from v2e_b200 import sinks
    g = np.load(os.path.join(GOLDEN_DIR, "sinks_aedat2.npz"))
    ev = g["events_long"]
    words, n_on = sinks.events_to_aedat2(torch.from_numpy(ev).cuda(), 346, 260)
    assert words.cpu().numpy().tobytes() == g["body_long"].tobytes()
    assert int(n_on.item()) == int(np.sum(ev[:, 3] > 0))
    odd = np.array([[np.nan, 1, 2, 1], [-3000.0, 1, 2, -1], [np.inf, 1, 2, 1], [1e30, 1, 2, 1]], np.float32)
    w, _ = sinks.events_to_aedat2(torch.from_numpy(odd).cuda(), 346, 260)
    assert w.cpu().numpy().tobytes() == sinks_oracle.aedat2_words(odd)[0].tobytes()
    rng = np.random.default_rng(4)
    n = 300001
    t = np.sort(np.concatenate([rng.uniform(0, 4294.967296, n - 4096 - 2000),
                                np.float64(np.nextafter(US32, np.float32(0))) - np.arange(4096) * ulp32(4294.0),
                                rng.uniform(4294.967296, 40000.0, 2000)]).astype(np.float32))
    rows = np.stack([t, rng.integers(0, 1280, n), rng.integers(0, 720, n), rng.choice([-1.0, 1.0], n)], 1).astype(np.float32)
    d = torch.from_numpy(rows).cuda()
    got = sinks.events_to_h5_rows(d).cpu().numpy().view(np.uint32)
    assert np.array_equal(got, sinks_oracle.h5_rows(rows))
    lab = rng.integers(0, 2, n).astype(np.uint8)
    for labels in (None, lab):
        body = sinks.events_to_text(d, None if labels is None else torch.from_numpy(labels).cuda())
        assert body.cpu().numpy().tobytes() == text_sink_oracle.text_body(rows, labels)


# ---- GPU: the files of the single-frame and batched paths -----------------------------------------------------------
def long_file_clip():
    """A 37x53 clip that crosses 2^31 us between frames and then jumps past 2^32 us (a 2147 s frame interval)."""
    from test_emulator_device_rng import texture_frames
    ts = [2147.40 + 0.01 * k for k in range(14)] + [4294.90 + 0.01 * k for k in range(12)]
    return texture_frames(37, 53, len(ts), seed=8, speed=2.0), ts


_H5_STAND_IN = r"""
import sys, types
import numpy as np
class _Dataset:
    def __init__(self, path):
        self.path, self.a = path, np.zeros((0, 4), np.uint32)
    @property
    def shape(self):
        return self.a.shape
    def resize(self, n, axis=0):
        b = np.zeros((n, 4), np.uint32)
        b[:min(n, len(self.a))] = self.a[:n]
        self.a = b
    def __setitem__(self, k, v):
        self.a[k] = v
class _File:
    def __init__(self, path, mode):
        self.path = path
    def create_dataset(self, name, **kw):
        self.ds = _Dataset(self.path)
        return self.ds
    def close(self):
        np.save(self.path + ".npy", self.ds.a)
sys.modules["h5py"] = types.SimpleNamespace(File=_File)
"""

_FILES = r"""
import os, sys
sys.path[:0] = [{root!r}, os.path.join({root!r}, "oracle"), os.path.join({root!r}, "tests")]
try:
    import h5py
    real_h5 = True
except ImportError:
    exec({stand_in!r})
    real_h5 = False
import numpy as np
import ref_shim
ref_shim.load_reference()
from test_long_clip_times import long_file_clip
from v2e_b200 import EventEmulator
fr, ts = long_file_clip()
out = {out!r}
kw = dict(cutoff_hz=200.0, leak_rate_hz=1e-4, shot_noise_rate_hz=1e-4, refractory_period_s=0.002)
for name in ("frames", "batch"):
    d = os.path.join(out, name)
    os.makedirs(d)
    em = EventEmulator(device="cuda", rng_mode="device", seed=4, row_order="canonical", label_signal_noise=True,
                       max_frames_per_step=5, output_folder=d, dvs_text="ev", dvs_aedat2="ev", dvs_h5="ev",
                       output_width=346, output_height=260, **kw)
    if name == "frames":
        rows, lab = [], []
        for f, t in zip(fr, ts):
            ev = em.generate_events(f, t)
            if ev is not None:
                rows.append(ev)
                lab.append(em.last_signnoise_label)
        rows, lab = np.concatenate(rows), np.concatenate(lab)
    else:
        rows, offs, lab = em.generate_events_batch(fr, ts, return_labels=True)
    em.cleanup()
    np.savez(os.path.join(d, "rows.npz"), rows=rows, labels=lab, real_h5=real_h5)
"""


def _h5(d, real):
    if real:
        import h5py
        with h5py.File(d / "ev.h5", "r") as f:
            return f["events"][:]
    return np.load(str(d / "ev.h5") + ".npy")


@pytest.mark.gpu
def test_single_frame_and_batch_files_are_identical_across_2_31_and_2_32_us(tmp_path):
    """generate_events and generate_events_batch write byte-identical AEDAT-2.0, HDF5 and text files for a clip that
    crosses both boundaries, and those bytes are the oracles' (the HDF5 rows through h5py where it imports, else
    through an in-memory stand-in of the two calls the sink makes)."""
    import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("v2ecore (the reference's writers) does not import")
    from test_sinks_batched import _files, aedat2_body
    subprocess.check_call([sys.executable, "-c", _FILES.format(root=ROOT, out=str(tmp_path), stand_in=_H5_STAND_IN)])
    a, b = tmp_path / "frames", tmp_path / "batch"
    ra, rb = np.load(a / "rows.npz"), np.load(b / "rows.npz")
    rows, labels = ra["rows"], ra["labels"]
    assert rows.tobytes() == rb["rows"].tobytes() and np.array_equal(labels, rb["labels"])
    assert _files(a) == _files(b)
    ha, hb = _h5(a, bool(ra["real_h5"])), _h5(b, bool(rb["real_h5"]))
    assert ha.tobytes() == hb.tobytes()
    text, aedat = _files(b)
    assert text == text_sink_oracle.text_body(rows, labels)
    assert aedat == aedat2_body(rows, 346, 260, labels)
    assert np.array_equal(hb, sinks_oracle.h5_rows(rows))
    t = rows[:, 0] * np.float32(1e6)
    assert np.sum(t < np.float32(2.0 ** 31)) > 100 and np.sum((t >= np.float32(2.0 ** 31)) & (t < 2.0 ** 32)) > 100
    assert np.sum(t >= np.float32(2.0 ** 32)) > 100
    assert (~labels).sum() > 0


# ---- GPU: the pipeline across 2^31 us -------------------------------------------------------------------------------
T_OFFSET = 2147.3
_PIPE = r"""
import os, sys
sys.path[:0] = [{root!r}, os.path.join({root!r}, "oracle"), os.path.join({root!r}, "tests")]
import numpy as np
import ref_shim
ref_shim.load_reference()
from test_long_clip_times import PIPE_NOISE, T_OFFSET
from test_pipeline_segments import _clip, _emulator, _slomo
from v2e_b200 import V2EPipeline
frames = _clip(12, 64, 96, [3] * 11)
sl = _slomo(False)
em = _emulator(row_order="canonical", output_folder={out!r}, dvs_aedat2="ev", output_width=346, output_height=260,
               **PIPE_NOISE)
n = sum(len(r[0]) for r in V2EPipeline(sl, em).run_segments(lambda a, b: frames[a:b], 12, 0.4, t_offset=T_OFFSET,
                                                             segment_pairs=3))
em.cleanup()
sl.cleanup()
np.save(os.path.join({out!r}, "n.npy"), np.array(n))
"""
PIPE_NOISE = dict(cutoff_hz=200, leak_rate_hz=1e-4, shot_noise_rate_hz=1e-4, sigma_thres=0.02,
                  refractory_period_s=0.0005)


@pytest.mark.gpu
def test_pipeline_streams_across_2_31_us(tmp_path):
    """run_segments with t_offset = 2147.3 s over a 0.4 s clip: the AEDAT-2.0 file it streams holds the oracle's
    words of the rows one run call returns, and those rows are the pixel-model oracle's, fed the pipeline's own
    interpolated frames and times and the device's draws."""
    import torch
    import ref_shim
    from test_pipeline_segments import _clip, _emulator, _slomo
    from test_sinks_batched import aedat2_body
    from v2e_b200 import V2EPipeline
    frames = _clip(12, 64, 96, [3] * 11)
    sl = _slomo(False)
    em = _emulator(row_order="canonical", **PIPE_NOISE)
    ev, offs, t, nf = V2EPipeline(sl, em).run(frames, 0.4, t_offset=T_OFFSET, copy=True)
    assert t[0] < US31 < t[-1] and nf == len(t)
    interp, _, _, _ = sl.interpolate_frames(torch.from_numpy(frames), return_ups=True, first_pair=0, clip_frames=12)
    interp = interp.cpu().numpy()
    assert interp.shape[0] == nf
    from test_emulator_device_rng import draws_from
    want, _, orc = oracle_run(PIPE_NOISE, interp, t, rng=DeviceDrawRNG(draws_from(em)), seed=9, shuffle=False)
    assert_rows_equal(_frames(ev, offs), want, "pipeline")
    assert em.num_events_total == orc.num_events_total
    sl.cleanup()
    past = ev[:, 0] * np.float32(1e6) >= np.float32(2.0 ** 31)
    assert past.sum() > 100 and (~past).sum() > 100
    if not ref_shim.reference_available():
        pytest.skip("v2ecore (the reference's writers) does not import")
    subprocess.check_call([sys.executable, "-c", _PIPE.format(root=ROOT, out=str(tmp_path))])
    assert int(np.load(tmp_path / "n.npy")) == len(ev)
    aedat = split_aedat(tmp_path)
    assert aedat == aedat2_body(ev, 346, 260, None)


def split_aedat(d):
    from test_sinks_batched import split_header
    return split_header((d / "ev.aedat").read_bytes(), b"\r\n")[1]


# ---- GPU: the renderer ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_renderer_matches_reference_past_2_31_us():
    """The DURATION and COUNT fixtures whose packets start at 2147.47 s (frame start times accumulated in float32)."""
    from test_render import _golden
    from v2e_b200.renderer import EventRenderer, ExposureMode
    done = 0
    for name, mode, value, H, W, fs, area, pk in _golden():
        if not name.endswith("_long"):
            continue
        assert pk[0][0][0, 0] > 2147.0
        r = EventRenderer(full_scale_count=fs, exposure_mode=ExposureMode(mode), exposure_value=value, area_dimension=area)
        n = 0
        for ev, want in pk:
            got = r.render_events_to_frames(ev, H, W, return_frames=True)
            got = np.zeros((0, H, W)) if got is None else got
            assert got.dtype == np.float64 and got.shape == want.shape and np.array_equal(got, want), name
            n += len(want)
        assert n > 0
        done += 1
    assert done == 2
