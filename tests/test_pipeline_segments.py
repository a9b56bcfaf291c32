"""V2EPipeline.run_segments: a clip of any length through SloMo and the pixel model segment by segment, with the
output of one V2EPipeline.run call on the whole clip.

CPU: the segment plan (pipeline.segment_plan); the time scale from the last batch's U alone (slomo.clip_span) against
the one run takes from the clip's times (slomo.clip_times); the orchestration -- per-segment times, frames, the
pre-pass that picks the last batch's U, the argument checks -- with SloMo's engine and the pixel model replaced by
recording stand-ins; the AEDAT-2.0 leading-'#' rule carried across segments.
GPU: streamed against one run, bit for bit, with device-RNG noise, both row orders, fixed and automatic U and several
segment sizes; rows as per-frame multisets without a row order; a refractory period; the event files; vid_orig /
vid_slomo; the device-memory high-water mark of a long clip."""
import io
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from v2e_b200.pipeline import DEFAULT_SEGMENT_PAIRS, V2EPipeline, segment_plan
from v2e_b200.slomo import clip_span, clip_times

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- CPU: the plan ------------------------------------------------------------------------------------------------
def _check_plan(plan, n_frames, batch_size):
    assert plan[0][0] == 0 and plan[-1][1] == n_frames - 1
    for (a0, a1), (b0, b1) in zip(plan, plan[1:]):
        assert a1 == b0                                  # segment k's last source frame is segment k+1's first
    for p0, p1 in plan:
        assert p1 > p0 and p0 % batch_size == 0          # every segment starts on a batch boundary of the clip


@pytest.mark.parametrize("batch_size", [1, 3, 8])
@pytest.mark.parametrize("n_frames", [2, 3, 4, 10, 25, 26, 200])
@pytest.mark.parametrize("segment_pairs", [1, 2, 5, 8, 24, 1000, None])
def test_segment_plan(n_frames, batch_size, segment_pairs):
    plan = segment_plan(n_frames, batch_size, segment_pairs)
    _check_plan(plan, n_frames, batch_size)
    sp = DEFAULT_SEGMENT_PAIRS if segment_pairs is None else segment_pairs
    sp = -(-sp // batch_size) * batch_size
    assert all(p1 - p0 == sp for p0, p1 in plan[:-1])
    assert 1 <= plan[-1][1] - plan[-1][0] <= sp
    assert len(plan) == -(-(n_frames - 1) // sp)


def test_segment_plan_cases():
    assert segment_plan(2, 1, 1) == [(0, 1)]                                   # n_frames = 2
    assert segment_plan(2, 8, None) == [(0, 1)]
    assert segment_plan(12, 3, 4) == [(0, 6), (6, 11)]                        # 4 pairs round up to 6; short last
    assert segment_plan(12, 3, 3) == [(0, 3), (3, 6), (6, 9), (9, 11)]
    assert segment_plan(12, 3, 100) == [(0, 11)]                              # larger than the clip
    assert segment_plan(10, 1, 4) == [(0, 4), (4, 8), (8, 9)]
    assert segment_plan(17, 8, 16) == [(0, 16)]


@pytest.mark.parametrize("n_frames,segment_pairs", [(1, 4), (0, 4), (5, 0), (5, -3)])
def test_segment_plan_rejects(n_frames, segment_pairs):
    with pytest.raises(ValueError):
        segment_plan(n_frames, 3, segment_pairs)


# ---- CPU: the time scale ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(16))
def test_time_scale_from_the_last_batch_equals_runs(seed):
    """run's f = src / (max - min of the clip's interpTimes) against src / clip_span(...) from the last batch's U, bit
    for bit, and the seconds t_offset + f * times of every segment (times by global pair index) against the clip's."""
    rng = np.random.default_rng(seed)
    n_pairs = int(rng.integers(1, 60))
    batch_size = int(rng.integers(1, 10))
    bs = min(batch_size, n_pairs)
    n_batches = -(-n_pairs // bs)
    fixed = seed % 2 == 0
    ups = [7] * n_batches if fixed else [int(u) for u in rng.integers(2, 40, n_batches)]
    src, t0 = float(rng.uniform(0.01, 100.0)), float(rng.uniform(0, 10))
    times, _ = clip_times(ups, n_pairs, batch_size)
    f = src / (np.max(times) - np.min(times))
    g = src / clip_span(n_pairs, batch_size, ups[-1])
    assert type(g) is type(f) and g == f
    want = t0 + f * times
    from v2e_b200.slomo import batch_times
    got = []
    for p0, p1 in segment_plan(n_pairs + 1, batch_size, int(rng.integers(1, 20))):
        seg = [batch_times(a, min(bs, n_pairs - a), ups[a // bs]) for a in range(p0, p1, bs)]
        got.append(t0 + g * np.concatenate(seg))
    assert np.concatenate(got).tobytes() == want.tobytes()


# ---- CPU: orchestration with stand-ins ---------------------------------------------------------------------------
class _Engine:
    """SloMoEngine stand-in: 'max flow' of a batch is flows[first source frame // batch size]; every interpolated frame
    is its pair's first source frame plus the step k."""

    def __init__(self, flows, bs):
        self.flows, self.bs, self.firsts, self.cur_b = flows, bs, [], 0

    def set_pairs(self, fr):
        self.cur, self.cur_b = fr, fr.shape[0] - 1
        self.firsts.append(int(fr[0, 0, 0]))

    def max_flow(self):
        return self.flows[self.firsts[-1] // self.bs]

    def interp(self, t, out):
        out.copy_(self.cur[:-1] + int(t * 64))

    def check_finite(self):
        pass

    def close(self):
        pass


class _Emulator:
    """EventEmulator stand-in: records what generate_events_batch gets."""
    shard = None

    def __init__(self):
        self.frames, self.t, self.cont, self._sinks_continue = [], [], [], False

    def check_batch_path(self):
        pass

    def generate_events_batch(self, frames, t, return_device=False, copy=True):
        self.frames.append(frames.clone())
        self.t.append(np.asarray(t))
        self.cont.append(self._sinks_continue)
        return np.zeros((0, 4), np.float32), np.zeros(len(t) + 1, np.int64)


def _stand_in_slomo(monkeypatch, auto, batch_size, flows):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    from v2e_b200.slomo import SuperSloMo
    s = SuperSloMo(model=None, auto_upsample=auto, upsampling_factor=None if auto else 3, batch_size=batch_size,
                   device="cpu")
    eng = _Engine(flows, batch_size)
    s._engine = eng
    monkeypatch.setattr(s, "_engine_for", lambda dim, batch: eng)
    return s, eng


def _src(n, H=4, W=5):
    return np.repeat(np.arange(n, dtype=np.uint8)[:, None, None], H * W, 1).reshape(n, H, W)


@pytest.mark.parametrize("auto", [False, True])
@pytest.mark.parametrize("n,batch_size,segment_pairs", [(2, 1, 1), (12, 3, 3), (12, 3, 4), (12, 3, 100), (10, 1, 2),
                                                      (26, 4, 8), (26, 8, 8)])
def test_segments_concatenate_to_run(monkeypatch, auto, n, batch_size, segment_pairs):
    """Per segment: the frames, the times (bit for bit, with the pre-pass scale) and the sinks' continuation flag;
    concatenated: what run gives. With auto_upsample and more than one segment the flow network runs once more, first,
    on the clip's last batch."""
    src = _src(n)
    bs = min(batch_size, n - 1)
    flows = [1.5 + 2.7 * ((7 * i) % 5) for i in range(-(-(n - 1) // bs))]
    s, eng = _stand_in_slomo(monkeypatch, auto, batch_size, flows)
    em_run = _Emulator()
    ev, offs, t_run, nf = V2EPipeline(s, em_run).run(src, 0.37, t_offset=1.25)
    run_firsts = list(eng.firsts)
    eng.firsts.clear()
    em = _Emulator()
    segs = list(V2EPipeline(s, em).run_segments(lambda a, b: src[a:b], n, 0.37, t_offset=1.25,
                                                segment_pairs=segment_pairs))
    plan = segment_plan(n, batch_size, segment_pairs)
    assert len(segs) == len(plan) == len(em.frames)
    assert em.cont == [k > 0 for k in range(len(plan))]
    assert np.concatenate([sg[2] for sg in segs]).tobytes() == t_run.tobytes()
    assert np.concatenate(em.t).tobytes() == t_run.tobytes()
    assert torch.equal(torch.cat(em.frames), em_run.frames[0])
    assert sum(sg[3] for sg in segs) == nf == len(t_run)
    last = (n - 2) // bs * bs
    pre = [last] if auto and len(plan) > 1 else []
    assert eng.firsts == pre + run_firsts
    assert [sg[3] for sg in segs] == [fr.shape[0] for fr in em.frames]


def test_argument_checks(monkeypatch):
    s, _ = _stand_in_slomo(monkeypatch, False, 3, [2.0] * 8)
    pipe = V2EPipeline(s, _Emulator())
    src = _src(12)
    with pytest.raises(ValueError, match="two source frames"):
        next(pipe.run_segments(lambda a, b: src[a:b], 1, 0.2))
    for bad, seg in ((lambda a, b: src[a:b].astype(np.float32) if a else src[a:b], 1),
                     (lambda a, b: src[a:b, :3] if a >= 6 else src[a:b], 2),
                     (lambda a, b: src[a:b + 1], 0),
                     (lambda a, b: src[a:b, 0], 0),
                     (lambda a, b: list(src[a:b]), 0)):
        it = pipe.run_segments(bad, 12, 0.2, segment_pairs=3)
        with pytest.raises(ValueError, match="segment %d of 4" % seg):
            for _ in it:
                pass


def test_refusals_before_any_work(monkeypatch):
    s, eng = _stand_in_slomo(monkeypatch, False, 3, [2.0] * 8)
    em = _Emulator()

    def refuse():
        raise RuntimeError("sharded")
    em.check_batch_path = refuse
    with pytest.raises(RuntimeError, match="sharded"):
        next(V2EPipeline(s, em).run_segments(lambda a, b: _src(12)[a:b], 12, 0.2, segment_pairs=3))
    assert eng.firsts == []


def test_aedat2_drop_rule_continues_across_segments(monkeypatch):
    """While every record written so far was dropped, a continuing write keeps dropping leading '#' records: the bytes
    of one write of the concatenation. A write that does not continue follows the per-call rule."""
    from test_sinks_batched import aedat2_body, hash_rows
    from v2e_b200 import emulator as em_mod
    from v2e_b200 import sinks
    import sinks_oracle

    def fake(ev, w, h, labels=None):
        words, n_on = sinks_oracle.aedat2_words(ev.numpy(), w, h)
        return torch.from_numpy(words.view(np.int32).copy()), torch.tensor([n_on])
    monkeypatch.setattr(sinks, "events_to_aedat2", fake)
    parts = [hash_rows(5, 1, 5), hash_rows(7, 2, 3), hash_rows(6, 3, 2)]
    allrows = np.concatenate(parts)
    for cont, want in ((True, aedat2_body(allrows, 346, 260, None)),
                       (False, b"".join(aedat2_body(p, 346, 260, None, written=k) for k, p in enumerate(parts)))):
        w = types.SimpleNamespace(file=io.BytesIO(), sizex=346, sizey=260, numEventsWritten=0, numOnEvents=0,
                                  numOffEvents=0)
        dropped = False
        for k, p in enumerate(parts):
            dropped = em_mod._append_aedat2(w, torch.from_numpy(p), None, cont and k > 0 and dropped)
        assert w.file.getvalue() == want, cont
        assert w.numEventsWritten == len(allrows)


# ---- GPU ----------------------------------------------------------------------------------------------------------
_NOISE = dict(cutoff_hz=200, leak_rate_hz=0.2, shot_noise_rate_hz=10.0, sigma_thres=0.02)
_SIZES = [(64, 96), (260, 346)]


def _slomo(auto, batch_size=3, **kw):
    from test_slomo_gpu import _weights
    from v2e_b200 import SuperSloMo
    fc, at = _weights(5)
    return SuperSloMo(model=None, auto_upsample=auto, upsampling_factor=None if auto else 3, batch_size=batch_size,
                      state_dicts={"state_dictFC": fc, "state_dictAT": at}, **kw)


def _emulator(**kw):
    from v2e_b200 import EventEmulator
    return EventEmulator(device="cuda:0", seed=9, rng_mode="device", **kw)


def _clip(n, H, W, shifts, seed=0):
    """n frames of a blocky texture; frame k is shifted by shifts[k] px from frame k-1, with a contrast that changes."""
    rng = np.random.default_rng(seed)
    pos = np.concatenate([[0], np.cumsum(shifts[:n - 1])]).astype(int)
    big = np.kron(rng.integers(30, 220, (H // 8 + 2, (W + pos[-1]) // 8 + 2)), np.ones((8, 8))).astype(np.float32)
    gains = 0.6 + 0.4 * np.cos(np.arange(n))
    return np.stack([np.clip(128 + g * (big[3:3 + H, p:p + W] - 128), 0, 255).astype(np.uint8)
                     for p, g in zip(pos, gains)])


_AUTO_CLIPS = {}


def _auto_clip(H, W, sl):
    """A clip of 12 frames (batches of 3, 3, 3, 2 pairs) whose per-batch U differ, the last batch's from the first's."""
    if (H, W) not in _AUTO_CLIPS:
        for seed in range(12):
            rng = np.random.default_rng(seed)
            shifts = np.repeat(rng.choice([1, 2, 6, 10, 14], 4), 3)
            frames = _clip(12, H, W, shifts, seed)
            _, _, _, ups = sl.interpolate_frames(frames, return_ups=True)
            if len(set(ups)) >= 2 and ups[-1] != ups[0]:
                _AUTO_CLIPS[(H, W)] = frames
                break
        assert (H, W) in _AUTO_CLIPS, "no candidate clip whose per-batch U's differ"
    return _AUTO_CLIPS[(H, W)]


def _counters(em):
    return (em.num_events_total, em.num_events_on, em.num_events_off, em.frame_counter, float(em.t_previous))


def _stream(sl, em, frames, seg, **kw):
    rows, offs, times, nf, base = [], [], [], 0, 0
    for ev, o, t, n in V2EPipeline(sl, em).run_segments(lambda a, b: frames[a:b], len(frames), 0.2, t_offset=0.5,
                                                        segment_pairs=seg, copy=True, **kw):
        assert len(o) == n + 1 and o[0] == 0 and o[-1] == len(ev) and len(t) == n
        rows.append(np.array(ev))
        offs.append(o[:-1] + base)
        base += len(ev)
        times.append(t)
        nf += n
    return np.concatenate(rows), np.concatenate(offs + [[base]]), np.concatenate(times), nf


def _frames_as_multisets(rows, offs):
    from helpers import canonical
    return [canonical(rows[a:b]).tobytes() for a, b in zip(offs[:-1], offs[1:])]


@pytest.mark.gpu
@pytest.mark.parametrize("auto", [False, True])
@pytest.mark.parametrize("row_order", ["canonical", "shuffled", None])
@pytest.mark.parametrize("H,W", _SIZES)
def test_streamed_equals_one_run(H, W, row_order, auto):
    """12 source frames in batches of 3: segments of 1 batch, of 2 batches (5 pairs rounded up) and one segment, against
    one run: rows, offsets, times and the emulator's counters bit for bit (without a row order, each frame's rows as a
    multiset)."""
    sl = _slomo(auto)
    frames = _auto_clip(H, W, sl) if auto else _clip(12, H, W, [3] * 11)
    em = _emulator(row_order=row_order, **_NOISE)
    ev, offs, t, nf = V2EPipeline(sl, em).run(frames, 0.2, t_offset=0.5, copy=True)
    want = _counters(em)
    assert len(ev) > 1000 and nf == len(t)
    for seg in (3, 5, 11):
        em2 = _emulator(row_order=row_order, **_NOISE)
        rows, o, tt, n = _stream(sl, em2, frames, seg)
        assert n == nf and tt.tobytes() == t.tobytes(), seg
        assert np.array_equal(o, offs), seg
        if row_order is None:
            assert _frames_as_multisets(rows, o) == _frames_as_multisets(ev, offs), seg
        else:
            assert rows.tobytes() == ev.tobytes(), seg
        assert _counters(em2) == want, seg
    sl.cleanup()


@pytest.mark.gpu
@pytest.mark.parametrize("return_device", [False, True])
def test_streamed_with_refractory_period_equals_one_run(return_device):
    """A refractory period longer than a frame interval rejects multi-frame chunks, which are replayed frame by frame;
    with 4 frames per chunk the chunks straddle the segment boundaries."""
    sl = _slomo(False)
    frames = _clip(12, 96, 128, [4] * 11)
    kw = dict(_NOISE, refractory_period_s=0.02, max_frames_per_step=4, row_order="canonical")
    em = _emulator(**kw)
    ev, offs, t, nf = V2EPipeline(sl, em).run(frames, 0.2, t_offset=0.5, copy=True)
    em2 = _emulator(**kw)
    rows, o, tt, n = [], [], [], 0
    for r, oo, ttt, nn in V2EPipeline(sl, em2).run_segments(lambda a, b: frames[a:b], 12, 0.2, t_offset=0.5,
                                                           segment_pairs=3, return_device=return_device):
        rows.append(r.cpu().numpy() if return_device else r.copy())
        o.append(oo[:-1] + sum(len(x) for x in rows[:-1]))
    rows = np.concatenate(rows)
    assert rows.tobytes() == ev.tobytes() and np.array_equal(np.concatenate(o + [[len(rows)]]), offs)
    assert _counters(em2) == _counters(em)
    sl.cleanup()


_SINKS = r"""
import os, sys
import numpy as np
sys.path[:0] = [{root!r}, os.path.join({root!r}, "oracle"), os.path.join({root!r}, "tests")]
import ref_shim
ref_shim.load_reference()
from test_pipeline_segments import _clip, _emulator, _slomo
from v2e_b200 import V2EPipeline
frames = _clip(12, 260, 346, [3] * 11)
sl = _slomo(False)
for name, seg in (("run", None), ("stream", 3)):
    out = os.path.join({out!r}, name)
    os.makedirs(out)
    em = _emulator(row_order="shuffled", label_signal_noise=True, output_folder=out, dvs_text="ev", dvs_aedat2="ev",
                   output_width=346, output_height=260, cutoff_hz=200, leak_rate_hz=0.2, shot_noise_rate_hz=10.0,
                   sigma_thres=0.02)
    pipe = V2EPipeline(sl, em)
    if seg is None:
        n = len(pipe.run(frames, 0.2, copy=True)[0])
    else:
        n = sum(len(r[0]) for r in pipe.run_segments(lambda a, b: frames[a:b], 12, 0.2, segment_pairs=seg))
    c = (n, em.dvs_text.numEventsWritten, em.dvs_aedat2.numEventsWritten, em.dvs_aedat2.numOnEvents)
    em.cleanup()
    np.save(os.path.join(out, "counters.npy"), np.array(c))
sl.cleanup()
"""


@pytest.mark.gpu
def test_streamed_event_files_equal_runs(tmp_path):
    """dvs_text and dvs_aedat2 (label_signal_noise, shuffled rows) written segment by segment: the bodies after the
    headers byte for byte, and the writers' counters, equal to one run's."""
    import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("v2ecore (the reference's writers) does not import")
    from test_sinks_batched import _files
    subprocess.check_call([sys.executable, "-c", _SINKS.format(root=ROOT, out=str(tmp_path))])
    a, b = tmp_path / "run", tmp_path / "stream"
    assert np.array_equal(np.load(a / "counters.npy"), np.load(b / "counters.npy"))
    assert int(np.load(a / "counters.npy")[0]) > 1000
    assert _files(a) == _files(b)


@pytest.mark.gpu
@pytest.mark.parametrize("auto", [False, True])
def test_streamed_videos_equal_runs(monkeypatch, tmp_path, auto):
    """vid_orig gets every source frame once, in order (the frame two segments share is written once); vid_slomo every
    interpolated frame: the frames run writes."""
    from test_slomo_video import _assert_frames, _inject_writer
    log = _inject_writer(monkeypatch)
    probe = _slomo(auto)
    frames = _auto_clip(64, 96, probe) if auto else _clip(12, 64, 96, [3] * 11)
    probe.cleanup()
    for seg in (None, 3):
        sl = _slomo(auto, video_path=str(tmp_path))
        pipe = V2EPipeline(sl, _emulator(**_NOISE))
        if seg is None:
            pipe.run(frames, 0.2)
        else:
            for _ in pipe.run_segments(lambda a, b: frames[a:b], 12, 0.2, segment_pairs=seg):
                pass
        assert sl.numOrigVideoFramesWritten == 12
        sl.cleanup()
    assert len(log) == 4
    assert len(log[0].frames) == 12
    _assert_frames(log[2].frames, log[0].frames)
    _assert_frames(log[3].frames, log[1].frames)


@pytest.mark.gpu
def test_device_memory_depends_on_the_segment_not_the_clip():
    """torch.cuda.max_memory_allocated streaming 3 and 9 segments of the same repeated content (346x260, U = 10,
    8 pairs per segment) differs by less than one segment's interpolated frames; for 9 segments it is below run's."""
    H, W, U, seg = 260, 346, 10, 8
    from test_slomo_gpu import _weights
    from v2e_b200 import SuperSloMo
    fc, at = _weights(5)
    sl = SuperSloMo(model=None, auto_upsample=False, upsampling_factor=U, batch_size=4,
                    state_dicts={"state_dictFC": fc, "state_dictAT": at})
    base = _clip(seg + 1, H, W, [3] * seg)[:seg]

    def get(a, b):
        return base[np.arange(a, b) % seg]
    seg_bytes = seg * U * H * W

    def peak(n_seg, streamed):
        import gc
        gc.collect()
        em = _emulator(**_NOISE)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        n = n_seg * seg + 1
        if streamed:
            for ev, offs, t, nf in V2EPipeline(sl, em).run_segments(get, n, 0.1 * n_seg, segment_pairs=seg):
                assert nf == seg * U
        else:
            V2EPipeline(sl, em).run(get(0, n), 0.1 * n_seg)
        torch.cuda.synchronize()
        p = torch.cuda.max_memory_allocated()
        em.cleanup()
        del em
        return p
    peak(1, True)                                     # the SloMo engine and its buffers exist before any measurement
    p3, p9, r9 = peak(3, True), peak(9, True), peak(9, False)
    assert abs(p9 - p3) < seg_bytes, (p3, p9, seg_bytes)
    assert p9 < r9, (p9, r9)
    sl.cleanup()
