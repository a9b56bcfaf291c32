"""V2EPipeline without an upsampler: v2e.py's --disable_slomo / no-upsampling mode (source frames straight to the pixel
model at interpTimes = range(n), v2e.py:776-797) through run / run_segments / run_segments_sharded, and its
--synthetic_input loop (v2e.py:580-607) through run_synthetic.

CPU: the frame segment plan; the frame times against v2e.py:794-797 restated in numpy; the synthetic loop's packets
against renderer.cut_packets with the frame index shifted by one; the orchestration with a recording stand-in emulator
(frames, times, sink continuation, render calls, a source that reuses its frame array); the batch_size checks; two gloo
ranks with a stand-in band emulator (every rank's bands are the source frames' rows).
GPU: the pipeline against v2e.py's per-frame loops on a fresh emulator, streamed against one run and one
generate_events_batch call, the event files, the DVS video and frame-times file, and two ranks against one GPU."""
import os

import numpy as np
import pytest
import torch

from test_render_packets import Recorder
from test_render_stream import packets_by_calls
from v2e_b200.pipeline import DEFAULT_BATCH_SIZE, DEFAULT_SEGMENT_FRAMES, DEFAULT_SEGMENT_PAIRS, V2EPipeline, \
    segment_plan


# ---- literal restatements of v2e.py ---------------------------------------------------------------------------------
def v2e_times(n, src_duration, t_offset=0.0):
    """v2e.py:792-797 (the npy2png branch's interpTimes, scaled to the clip), plus the pipeline's t_offset."""
    interpTimes = np.array(range(n))
    f = src_duration / (np.max(interpTimes) - np.min(interpTimes))
    interpTimes = f * interpTimes
    return t_offset + interpTimes


def synthetic_loop(frame_rows, batch_size):
    """v2e.py:580-607, literally, over the rows generate_events returned per frame: the packets render_events_to_frames
    is called with."""
    packets, events = [], np.zeros((0, 4), dtype=np.float32)
    i = 0
    for newEvents in frame_rows:
        i += 1
        if newEvents is not None and newEvents.shape[0] > 0:
            events = np.append(events, newEvents, axis=0)
            events = np.array(events)
            if i % batch_size == 0:
                packets.append(events)
                events = np.zeros((0, 4), dtype=np.float32)
    if len(events) > 0:
        packets.append(events)
    return packets


def stage3_loop(frame_rows, batch_size):
    """v2e.py:826-846, literally."""
    from test_render_stream import v2e_loop
    return v2e_loop(frame_rows, batch_size)


# ---- CPU: the plan and the times ------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("segment_frames", [1, 2, 5, 7, 64, 1000, None])
@pytest.mark.parametrize("n", [2, 3, 4, 10, 64, 65, 641, 1300])
def test_frame_segment_plan(n, segment_frames, world):
    if n < world:
        with pytest.raises(ValueError, match="fewer frames than ranks"):
            segment_plan(n, 1, segment_frames, world=world, upsampler=False)
        return
    plan = segment_plan(n, 1, segment_frames, world=world, upsampler=False)
    assert plan[0][0] == 0 and plan[-1][1] == n
    assert all(a1 == b0 for (_, a1), (b0, _) in zip(plan, plan[1:]))          # disjoint, every frame once
    assert all(b - a >= world for a, b in plan)
    sf = max(DEFAULT_SEGMENT_FRAMES if segment_frames is None else segment_frames, world)
    assert all(b - a == sf for a, b in plan[:-1]) and plan[-1][1] - plan[-1][0] < 2 * sf
    # batch_size and auto_upsample do not enter the plan without an upsampler
    assert segment_plan(n, 7, segment_frames, world=world, auto_upsample=True, upsampler=False) == plan


def test_frame_segment_plan_cases():
    assert DEFAULT_SEGMENT_FRAMES == 10 * DEFAULT_SEGMENT_PAIRS == 640 and DEFAULT_BATCH_SIZE == 8
    assert segment_plan(2, 1, None, upsampler=False) == [(0, 2)]
    assert segment_plan(10, 1, 4, upsampler=False) == [(0, 4), (4, 8), (8, 10)]
    assert segment_plan(10, 1, 4, world=3, upsampler=False) == [(0, 4), (4, 10)]               # 2-frame tail folded
    assert segment_plan(1281, 1, None, upsampler=False) == [(0, 640), (640, 1280), (1280, 1281)]


@pytest.mark.parametrize("n,segment_frames", [(1, 4), (0, 4), (5, 0), (5, -3)])
def test_frame_segment_plan_rejects(n, segment_frames):
    with pytest.raises(ValueError):
        segment_plan(n, 1, segment_frames, upsampler=False)


class _Emulator:
    """EventEmulator stand-in: records what generate_events_batch gets; frame j of the clip gets counts[j] rows whose
    time is j."""
    shard, device, output_height, output_width = None, "cpu", 4, 5

    def __init__(self, counts=None):
        self.frames, self.t, self.cont, self._sinks_continue = [], [], [], False
        self.counts, self.done = counts, 0

    def check_batch_path(self):
        pass

    def generate_events_batch(self, frames, t, return_device=False, copy=True):
        self.frames.append(torch.as_tensor(frames).clone())
        self.t.append(np.asarray(t))
        self.cont.append(self._sinks_continue)
        T = len(t)
        c = np.zeros(T, np.int64) if self.counts is None else np.asarray(self.counts[self.done:self.done + T])
        rows = np.repeat(np.arange(self.done, self.done + T, dtype=np.float32), c)[:, None].repeat(4, 1)
        self.done += T
        self.rows = torch.from_numpy(rows)
        return (self.rows if return_device else rows), np.concatenate([[0], np.cumsum(c)]).astype(np.int64)

    def _rows_to_host(self, n, copy=True):
        return self.rows[:n].numpy()


class _Renderer:
    """EventRenderer stand-in: the packets render_frame_rows renders (cut_packets, rows held across calls)."""

    def __init__(self):
        self.calls = []

    def render_frame_rows(self, rows, offsets, first_frame, packet_frames, end_of_clip=False, height=None, width=None):
        self.calls.append((np.asarray(rows).copy(), np.asarray(offsets), first_frame, packet_frames, end_of_clip))

    def packets(self):
        from v2e_b200.renderer import cut_packets
        out, held = [], np.zeros((0, 4), np.float32)
        for rows, offs, first, pf, end in self.calls:
            allr = np.concatenate([held, rows[offs[0]:offs[-1]]])
            ends, keep = cut_packets(offs, first, pf, len(held), end)
            out += [allr[a:b] for a, b in zip(np.concatenate([[0], ends[:-1]]), ends)]
            held = allr[keep:]
        return out


def _src(n, H=4, W=5):
    return np.repeat(np.arange(n, dtype=np.uint8)[:, None, None], H * W, 1).reshape(n, H, W)


@pytest.mark.parametrize("seed", range(24))
def test_segments_times_and_frames_equal_v2e(seed):
    """Per segment: the source frames themselves and the times of v2e.py:794-797 (with t_offset), bit for bit, the
    sinks' continuation flag, the yielded frame counts; concatenated: what run gives, and the times of the literal
    restatement."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(2, 90))
    src_dur, t0 = float(rng.uniform(1e-3, 5000.0)), [0.0, float(rng.uniform(0, 40000.0))][seed % 2]
    seg = [1, 2, 7, int(rng.integers(1, 100)), None][seed % 5]
    src = _src(n)
    want = v2e_times(n, src_dur, t0)
    em_run = _Emulator()
    ev, offs, t_run, nf = V2EPipeline(None, em_run).run(src, src_dur, t_offset=t0)
    assert len(em_run.frames) == 1 and nf == n and t_run.tobytes() == want.tobytes()
    em = _Emulator()
    segs = list(V2EPipeline(None, em).run_segments(lambda a, b: src[a:b], n, src_dur, t_offset=t0,
                                                   segment_pairs=seg))
    plan = segment_plan(n, 1, seg, upsampler=False)
    assert len(segs) == len(plan) == len(em.frames)
    assert [s[3] for s in segs] == [b - a for a, b in plan]
    assert em.cont == [k > 0 for k in range(len(plan))]
    assert np.concatenate([s[2] for s in segs]).tobytes() == want.tobytes()
    assert np.concatenate(em.t).tobytes() == want.tobytes()
    assert torch.equal(torch.cat(em.frames), torch.from_numpy(src))


def test_times_take_numpy_scalars_as_v2e_does():
    """A float32 duration is divided by numpy's int64 span, as v2e.py divides it (float64), not in float32."""
    em = _Emulator()
    src = _src(11)
    _, _, t, _ = V2EPipeline(None, em).run(src, np.float32(0.3))
    assert t.dtype == np.float64 and t.tobytes() == v2e_times(11, np.float32(0.3)).tobytes()


def test_argument_checks():
    pipe = V2EPipeline(None, _Emulator())
    src = _src(12)
    with pytest.raises(ValueError, match="two source frames"):
        next(pipe.run_segments(lambda a, b: src[a:b], 1, 0.2))
    with pytest.raises(ValueError, match="two source frames"):
        pipe.run(src[:1], 0.2)
    with pytest.raises(ValueError, match="at least one frame"):
        next(pipe.run_segments(lambda a, b: src[a:b], 12, 0.2, segment_pairs=0))
    for bad, seg in ((lambda a, b: src[a:b].astype(np.float32) if a else src[a:b], 1),
                     (lambda a, b: src[a:b, :3] if a >= 6 else src[a:b], 2),
                     (lambda a, b: src[a:b + 1], 0)):
        with pytest.raises(ValueError, match="segment %d of 4" % seg):
            for _ in pipe.run_segments(bad, 12, 0.2, segment_pairs=3):
                pass
    with pytest.raises(ValueError):
        V2EPipeline(None, _Emulator(), batch_size=0)


def test_batch_size_with_an_upsampler(monkeypatch):
    sl, _ = _stand_in(monkeypatch)
    assert V2EPipeline(sl, _Emulator()).batch_size == 3
    assert V2EPipeline(sl, _Emulator(), batch_size=3).batch_size == 3
    for k in (1, 2, 4, 8):
        with pytest.raises(ValueError, match="batch_size"):
            V2EPipeline(sl, _Emulator(), batch_size=k)
    assert V2EPipeline(None, _Emulator()).batch_size == 8
    assert V2EPipeline(None, _Emulator(), batch_size=5).batch_size == 5


def _stand_in(monkeypatch):
    from test_pipeline_segments import _stand_in_slomo
    return _stand_in_slomo(monkeypatch, False, 3, [2.0] * 8)


# ---- CPU: the synthetic loop ----------------------------------------------------------------------------------------
def _counts(seed, T):
    rng = np.random.default_rng(seed)
    c = rng.integers(0, 6, T)
    c[rng.random(T) < 0.35] = 0
    return c


def _restated(counts, batch_size, loop):
    offsets = np.concatenate([[0], np.cumsum(counts)])
    frames = [np.repeat(np.arange(a, b, dtype=np.float32)[:, None], 4, 1) for a, b in zip(offsets[:-1], offsets[1:])]
    return [p[:, 0].astype(np.int64) for p in loop(frames, batch_size)]


@pytest.mark.parametrize("seed", range(16))
@pytest.mark.parametrize("batch_size", [1, 3, 8])
def test_synthetic_packets_are_cut_packets_one_frame_on(seed, batch_size):
    """The synthetic loop's packets are render_frame_rows' with the frames counted from 1, in calls of every length; and
    they are not the stage-3 loop's."""
    T = 29
    counts = _counts(seed, T)
    counts[batch_size - 1] = max(counts[batch_size - 1], 1)        # the first synthetic boundary has rows
    counts[batch_size] = max(counts[batch_size], 1) if batch_size > 1 else counts[batch_size]
    want = _restated(counts, batch_size, synthetic_loop)
    for k in range(1, T + 1):
        calls = [(a, min(T, a + k)) for a in range(0, T, k)]
        got = packets_by_calls(counts, calls, 1, batch_size)
        assert len(got) == len(want) and all(np.array_equal(g, w) for g, w in zip(got, want)), k
    if batch_size > 1:
        stage3 = _restated(counts, batch_size, stage3_loop)
        assert len(stage3) != len(want) or any(not np.array_equal(a, b) for a, b in zip(stage3, want))


class _Source:
    """base_synthetic_input's contract; like the reference's sources it returns the same array, redrawn, every frame."""

    def __init__(self, n, H=4, W=5, dt=1e-3, dtype=np.uint8):
        self.n, self.k, self.dt = n, 0, dt
        self.pix = np.zeros((H, W), dtype)
        self.cleaned = False

    def total_frames(self):
        return self.n

    def next_frame(self):
        if self.k >= self.n:
            return None, self.k * self.dt
        self.pix[:] = self.k % 256
        t = self.k * self.dt
        self.k += 1
        return self.pix, t

    def cleanup(self):
        self.cleaned = True


@pytest.mark.parametrize("dtype", [np.uint8, np.float32, np.float64])
@pytest.mark.parametrize("n,seg", [(1, 4), (2, 1), (12, 3), (12, 5), (12, 12), (12, 100), (40, None), (9, 1)])
def test_run_synthetic_orchestration(n, seg, dtype):
    """Segments of `seg` frames pulled from the source (each frame copied before the source redraws its array), the
    source's times plus t_offset, the sinks' continuation flag, and the renderer called with the frames counted from 1
    and end_of_clip on the last segment only: the synthetic loop's packets. The source is not cleaned up."""
    counts = _counts(n, n)
    em, rd = _Emulator(counts), _Renderer()
    src = _Source(n, dtype=dtype)
    segs = list(V2EPipeline(None, em, renderer=rd, batch_size=3).run_synthetic(src, segment_frames=seg, t_offset=2.5))
    sf = DEFAULT_SEGMENT_FRAMES if seg is None else seg
    assert [s[3] for s in segs] == [min(sf, n - a) for a in range(0, n, sf)]
    assert em.cont == [k > 0 for k in range(len(segs))]
    if n:
        fr = torch.cat(em.frames)
        assert fr.dtype == torch.from_numpy(np.zeros(1, dtype)).dtype
        assert torch.equal(fr[:, 0, 0].double(), torch.arange(n, dtype=torch.float64) % 256)
        t = np.concatenate([s[2] for s in segs])
        assert t.tobytes() == (2.5 + np.array([k * 1e-3 for k in range(n)])).tobytes()
    assert [c[2] for c in rd.calls] == [1 + a for a in range(0, n, sf)]
    assert [c[3] for c in rd.calls] == [3] * len(segs)
    assert [c[4] for c in rd.calls] == [k == len(segs) - 1 for k in range(len(segs))]
    want = _restated(counts, 3, synthetic_loop)
    got = [p[:, 0].astype(np.int64) for p in rd.packets()]
    offs = np.concatenate([[0], np.cumsum(counts)])
    want = [np.repeat(np.arange(n), counts)[w] for w in want]           # row ids -> frame ids, as the stand-in stamps
    assert len(got) == len(want) and all(np.array_equal(g, w) for g, w in zip(got, want))
    assert offs[-1] == sum(len(p) for p in got) and not src.cleaned


def test_run_synthetic_rejects_frames_unlike_the_first():
    class Bad(_Source):
        def next_frame(self):
            fr, t = super().next_frame()
            return (fr[:, :3] if fr is not None and self.k == 4 else fr), t
    with pytest.raises(ValueError, match="frame 3"):
        list(V2EPipeline(None, _Emulator()).run_synthetic(Bad(6), segment_frames=2))
    with pytest.raises(ValueError, match="at least one frame"):
        list(V2EPipeline(None, _Emulator()).run_synthetic(_Source(6), segment_frames=0))


# ---- CPU: two gloo ranks with a stand-in band emulator --------------------------------------------------------------
class _BandEmulator:
    label_signal_noise, row_order, _sinks, device, rng_mode = False, None, None, "cpu", "device"

    def __init__(self, shard):
        self.shard, self.bands, self.t = shard, [], []

    def cs_halo_rows(self, H):
        return 1

    def generate_events_band_batch(self, bands, t, H):
        self.bands.append(bands.clone())
        self.t.append(np.asarray(t))
        return np.zeros((0, 4), np.float32), np.zeros(bands.shape[0] + 1, np.int64)


def _bands_worker(rank, world, port, q, n, seg):
    import torch.distributed as dist
    from test_pipeline_segments_sharded import _init
    _init(rank, world, port)
    try:
        rng = np.random.default_rng(1)
        src = rng.integers(0, 256, (n, 7, 5), dtype=np.uint8)
        asked = []

        def get(a, b):
            asked.append((a, b))
            return src[a:b]
        em = _BandEmulator((rank, world, None))
        res = list(V2EPipeline(None, em).run_segments_sharded(get, n, 0.3, t_offset=1.0, segment_pairs=seg))
        q.put((rank, dict(asked=asked, bands=[b.numpy() for b in em.bands], t=em.t, nf=[r[2] for r in res])))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,n,seg", [(2, 13, 4), (3, 13, 4), (2, 5, None)])
def test_sharded_ranks_fetch_their_runs_and_get_their_bands(world, n, seg):
    from test_pipeline_segments_sharded import _spawn
    from v2e_b200.parallel import band_with_halo, pair_range
    res = _spawn(world, _bands_worker, n, seg, timeout=120)
    src = np.random.default_rng(1).integers(0, 256, (n, 7, 5), dtype=np.uint8)
    plan = segment_plan(n, 1, seg if seg is not None else DEFAULT_SEGMENT_FRAMES * world, world=world,
                        upsampler=False)
    for r in range(world):
        y0, y1 = band_with_halo(7, r, world, 1)
        assert res[r]["asked"] == [tuple(s0 + x for x in pair_range(s1 - s0, r, world)) for s0, s1 in plan]
        assert np.array_equal(np.concatenate(res[r]["bands"]), src[:, y0:y1])
        assert np.concatenate(res[r]["t"]).tobytes() == v2e_times(n, 0.3, 1.0).tobytes()
        assert res[r]["nf"] == [b - a for a, b in plan]


# ---- GPU ------------------------------------------------------------------------------------------------------------
_CLI = dict(pos_thres=0.2, neg_thres=0.2, sigma_thres=0.03, cutoff_hz=300.0, leak_rate_hz=0.01,
            shot_noise_rate_hz=0.001, refractory_period_s=0.0005)              # v2e's CLI defaults
_CLEAN = dict(_CLI, leak_rate_hz=0.0, shot_noise_rate_hz=0.0)
_SIZES = [(260, 346), (720, 1280)]


def _clip(n, H, W, shift=3, seed=0):
    from test_pipeline_segments import _clip as clip
    return clip(n, H, W, [shift] * (n - 1), seed)


def _emulator(device="cuda:0", **kw):
    from v2e_b200 import EventEmulator
    return EventEmulator(device=device, seed=9, **kw)


def _counters(em):
    return (em.num_events_total, em.num_events_on, em.num_events_off, em.frame_counter, float(em.t_previous))


def _per_frame(rows, offs):
    return [rows[a:b] for a, b in zip(offs[:-1], offs[1:])]


def _drop_in_loop(em, frames, times):
    """v2e.py:819-836: generate_events per frame; the rows of each frame ([0, 4] for None)."""
    out = []
    for fr, t in zip(frames, times):
        ev = em.generate_events(fr, t)
        out.append(np.zeros((0, 4), np.float32) if ev is None else np.array(ev))
    return out


def _concat(segs):
    """Consumes the yields one by one (device rows are views valid until the next one): (rows, offsets, times,
    segments)."""
    rows, offs, times, base = [], [], [], 0
    for ev, o, t, n in segs:
        ev = ev.cpu().numpy() if isinstance(ev, torch.Tensor) else np.array(ev)
        assert len(o) == n + 1 and o[0] == 0 and o[-1] == len(ev) and len(t) == n
        rows.append(ev)
        offs.append(np.asarray(o[:-1]) + base)
        base += len(ev)
        times.append(t)
    return np.concatenate(rows), np.concatenate(offs + [[base]]), np.concatenate(times), len(rows)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", _SIZES)
@pytest.mark.parametrize("rng_mode", ["replay", "device"])
def test_run_equals_v2e_drop_in_loop(H, W, rng_mode):
    """No noise. Device RNG with the canonical row order: run's rows, in order, are generate_events' per frame at v2e's
    times f * i on a fresh emulator. Replay RNG (the default, host-drawn thresholds): the same rows per frame; the order
    inside a frame is the reference's randperm shuffle there, which the batched path does not replay."""
    from helpers import canonical
    n, dur = 24, 0.25
    frames = _clip(n, H, W)
    kw = dict(_CLEAN, rng_mode=rng_mode, **({"row_order": "canonical"} if rng_mode == "device" else {}))
    ev, offs, t, nf = V2EPipeline(None, _emulator(**kw)).run(frames, dur, copy=True)
    em = _emulator(**kw)                                 # seeds torch's generator again: the same thresholds
    got = _per_frame(ev, offs)
    want = _drop_in_loop(em, frames, v2e_times(n, dur))
    assert nf == n and t.tobytes() == v2e_times(n, dur).tobytes()
    assert sum(len(w) for w in want) > 1000 and len(want[0]) == 0
    for i, (g, w) in enumerate(zip(got, want)):
        if rng_mode == "device":
            assert g.tobytes() == w.tobytes(), i
        else:
            assert canonical(g).tobytes() == canonical(w).tobytes(), i


class MovingGaussian:
    """base_synthetic_input's contract: a Gaussian spot circling over a grey background, redrawn into one array."""

    def __init__(self, n, H, W, dtype=np.uint8, dt=1 / 1000.0):
        self.n, self.k, self.dt, self.dtype = n, 0, dt, dtype
        self.y, self.x = np.mgrid[0:H, 0:W].astype(np.float64)
        self.H, self.W = H, W
        self.pix = np.zeros((H, W), dtype)

    def total_frames(self):
        return self.n

    def next_frame(self):
        if self.k >= self.n:
            return None, self.k * self.dt
        a = 2 * np.pi * self.k / 40
        cx, cy = self.W / 2 + self.W / 4 * np.cos(a), self.H / 2 + self.H / 4 * np.sin(a)
        g = 40 + 180 * np.exp(-((self.x - cx) ** 2 + (self.y - cy) ** 2) / (2 * (self.H / 10) ** 2))
        self.pix[:] = np.round(g) if self.dtype == np.uint8 else g
        t = self.k * self.dt
        self.k += 1
        return self.pix, t


def _synthetic_drop_in(em, source):
    """v2e.py:580-600's emulation: generate_events on every (frame, time) until the frame is None."""
    out = []
    fr, t = source.next_frame()
    while fr is not None:
        ev = em.generate_events(fr, t)
        out.append(np.zeros((0, 4), np.float32) if ev is None else np.array(ev))
        fr, t = source.next_frame()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
def test_run_synthetic_equals_v2e_synthetic_loop(dtype):
    """Device RNG with v2e's CLI-default noise, canonical row order: run_synthetic in segments of 1, 7, 64 and the
    default equals generate_events frame by frame on the source's frames and times, rows in order and counters."""
    H, W, n = 260, 346, 90
    kw = dict(_CLI, rng_mode="device", row_order="canonical")
    em = _emulator(**kw)
    want = _synthetic_drop_in(em, MovingGaussian(n, H, W, dtype))
    want_counters = _counters(em)
    assert sum(len(w) for w in want) > 1000
    for seg in (1, 7, 64, None):
        em = _emulator(**kw)
        rows, offs, t, _ = _concat(V2EPipeline(None, em).run_synthetic(MovingGaussian(n, H, W, dtype),
                                                                       segment_frames=seg, copy=True))
        assert t.tobytes() == np.array([k * (1 / 1000.0) for k in range(n)]).tobytes(), seg
        assert rows.tobytes() == np.concatenate(want).tobytes(), seg
        assert np.array_equal(np.diff(offs), [len(w) for w in want]), seg
        assert _counters(em) == want_counters, seg


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["host", "pinned", "device"])
def test_segments_equal_one_run_and_one_batch_call(where):
    """Device RNG, v2e's CLI defaults, canonical order: run_segments(None) over segments of 1, 7, 64 and the default
    (640: one segment) concatenates to one run -- rows, offsets, times, counters and t_previous --, and run equals one
    generate_events_batch on the same frames and times; get_frames on the host, in pinned memory and on the device."""
    H, W, n = 260, 346, 80
    frames = _clip(n, H, W)
    src = {"host": torch.from_numpy(frames), "pinned": torch.from_numpy(frames).pin_memory(),
           "device": torch.from_numpy(frames).cuda()}[where]
    kw = dict(_CLI, rng_mode="device", row_order="canonical")
    em = _emulator(**kw)
    ev, offs, t, nf = V2EPipeline(None, em).run(src, 0.4, t_offset=3.0, copy=True)
    want = _counters(em)
    em_b = _emulator(**kw)
    rows_b, offs_b = em_b.generate_events_batch(frames, 3.0 + v2e_times(n, 0.4))
    assert rows_b.tobytes() == ev.tobytes() and np.array_equal(offs_b, offs) and _counters(em_b) == want
    assert len(ev) > 1000 and t.tobytes() == v2e_times(n, 0.4, 3.0).tobytes()
    for seg in (1, 7, 64, None):
        em2 = _emulator(**kw)
        rows, o, tt, m = _concat(V2EPipeline(None, em2).run_segments(lambda a, b: src[a:b], n, 0.4, t_offset=3.0,
                                                                     segment_pairs=seg, return_device=seg == 7,
                                                                     copy=True))
        assert m == len(segment_plan(n, 1, seg, upsampler=False)), seg
        assert rows.tobytes() == ev.tobytes() and np.array_equal(o, offs) and tt.tobytes() == t.tobytes(), seg
        assert _counters(em2) == want, seg


def _files_worker(rank, world, port, q, out):
    """One GPU: dvs_text + dvs_aedat2 with labels from run_segments(None) in segments of 5, and from one
    generate_events_batch call; also run_synthetic against one generate_events_batch call on its frames."""
    import torch.distributed as dist
    from test_pipeline_segments_sharded import _init
    _init(rank, world, port)
    try:
        import ref_shim
        ref_shim.load_reference()
        H, W, n = 260, 346, 30
        frames = _clip(n, H, W)
        src = MovingGaussian(n, H, W)
        syn = np.stack([src.next_frame()[0].copy() for _ in range(n)])
        counts = {}
        for name in ("seg", "batch", "syn", "syn_batch"):
            d = os.path.join(out, name)
            os.makedirs(d)
            em = _emulator(rng_mode="device", row_order="shuffled", label_signal_noise=True, output_folder=d,
                           dvs_text="ev", dvs_aedat2="ev", output_width=W, output_height=H,
                           **dict(_CLI, shot_noise_rate_hz=5.0))
            if name == "seg":
                for _ in V2EPipeline(None, em).run_segments(lambda a, b: frames[a:b], n, 0.3, segment_pairs=5):
                    pass
            elif name == "batch":
                em.generate_events_batch(frames, v2e_times(n, 0.3))
            elif name == "syn":
                for _ in V2EPipeline(None, em).run_synthetic(MovingGaussian(n, H, W), segment_frames=4):
                    pass
            else:
                em.generate_events_batch(syn, np.array([k * (1 / 1000.0) for k in range(n)]))
            counts[name] = (em.dvs_text.numEventsWritten, em.dvs_aedat2.numEventsWritten)
            em.cleanup()
        q.put((rank, counts))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_event_files_equal_one_batch_call(tmp_path):
    import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("v2ecore (the reference's writers) does not import")
    from test_pipeline_segments_sharded import _spawn
    from test_sinks_batched import _files
    counts = _spawn(1, _files_worker, str(tmp_path))[0]
    assert counts["seg"] == counts["batch"] and counts["seg"][0] > 1000
    assert counts["syn"] == counts["syn_batch"] and counts["syn"][0] > 100
    assert _files(tmp_path / "seg") == _files(tmp_path / "batch")
    assert _files(tmp_path / "syn") == _files(tmp_path / "syn_batch")


def _renderer(mode, out_dir):
    from v2e_b200.renderer import EventRenderer, ExposureMode
    opened = []

    def writer(path, height, width, frame_rate=30):
        opened.append(Recorder(path, height, width, frame_rate))
        return opened[-1]
    r = EventRenderer(full_scale_count=2, output_path=str(out_dir), dvs_vid="dvs-video.avi",
                      exposure_mode=ExposureMode[mode], exposure_value=0.01 if mode == "DURATION" else 100,
                      video_writer=writer)
    return r, opened


def _written(r, opened, out_dir):
    """cleanup(), then (the frames the video writer got, the frame-times file's text)."""
    r.cleanup()
    assert len(opened) == 1 and opened[0].released
    with open(os.path.join(str(out_dir), "dvs-video-frame_times.txt")) as f:
        text = f.read()
    return (np.stack(opened[0].frames) if opened[0].frames else np.zeros((0,), np.uint8)), text


def _render_packets(packets, H, W, mode, out_dir):
    os.makedirs(out_dir)
    r, opened = _renderer(mode, out_dir)
    for p in packets:
        r.render_events_to_frames(p, H, W)
    return _written(r, opened, out_dir)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["DURATION", "COUNT"])
@pytest.mark.parametrize("what", ["segments", "synthetic"])
def test_renderer_writes_v2e_loops_video(what, mode, tmp_path):
    """With a renderer (batch_size 3 and the default 8): the DVS video and frame-times file equal the yielded rows fed
    through v2e.py's loop -- stage 3 for run_segments, the synthetic loop for run_synthetic -- into
    render_events_to_frames; the rows equal a run without a renderer."""
    H, W, n = 96, 128, 40
    frames = _clip(n, H, W)
    kw = dict(_CLI, rng_mode="device", row_order="canonical")
    for bs in (3, None):
        for seg in (5, None):
            name = "%s-%s" % (bs, seg)
            d = tmp_path / name
            d.mkdir()
            r, opened = _renderer(mode, d)
            if what == "segments":
                run = lambda p: p.run_segments(lambda a, b: frames[a:b], n, 0.39, segment_pairs=seg, copy=True)
            else:
                run = lambda p: p.run_synthetic(MovingGaussian(n, H, W, dt=0.01), segment_frames=seg, copy=True)
            # each emulator seeds torch's generator when it is built and draws its thresholds on its first frame
            pipe = V2EPipeline(None, _emulator(**kw), renderer=r, batch_size=bs)
            rows, offs, _, _ = _concat(run(pipe))
            rows2, offs2, _, _ = _concat(run(V2EPipeline(None, _emulator(**kw), batch_size=bs)))
            assert rows.tobytes() == rows2.tobytes() and np.array_equal(offs, offs2), name
            vid, text = _written(r, opened, d)
            loop = stage3_loop if what == "segments" else synthetic_loop
            packets = loop(_per_frame(rows, offs), pipe.batch_size)
            want_vid, want_text = _render_packets(packets, H, W, mode, tmp_path / ("want-" + name))
            assert len(packets) >= 3 and len(want_vid) >= 3, name
            assert vid.shape == want_vid.shape and np.array_equal(vid, want_vid) and text == want_text, name


_FILES_KW = dict(rng_mode="device", row_order="canonical", label_signal_noise=True, cutoff_hz=200, sigma_thres=0.02,
                 leak_rate_hz=0.2, shot_noise_rate_hz=5.0)
_CS_KW = dict(rng_mode="device", cs_lambda_pixels=4, cs_tau_p_ms=2.0, cutoff_hz=200,
              leak_rate_hz=0, shot_noise_rate_hz=0, sigma_thres=0.02, refractory_period_s=0.001)


def _sharded_worker(rank, world, port, q, spec, backend="gloo"):
    """world > 1: run_segments_sharded(None) with write_sinks (event files and, on the first rank, the DVS video) or,
    for the centre-surround model, the rows alone. world == 1: one GPU's run_segments(None) with the same outputs."""
    import torch.distributed as dist
    from test_pipeline_segments_sharded import _init
    dev = _init(rank, world, port, backend)
    try:
        frames, n, out = spec["frames"], len(spec["frames"]), spec["out"]
        files = spec["files"]
        if files:
            import ref_shim
            ref_shim.load_reference()
        kw = dict(_FILES_KW if files else _CS_KW)
        r = opened = None
        if rank == 0 and files:
            os.makedirs(out)
            kw.update(output_folder=out, dvs_text="ev", dvs_aedat2="ev", output_width=frames.shape[2],
                      output_height=frames.shape[1])
            r, opened = _renderer("DURATION", out)
        em = _emulator(device=dev, shard=(rank, world, None) if world > 1 else None, **kw)
        pipe = V2EPipeline(None, em, renderer=r, batch_size=3)
        get = lambda a, b: frames[a:b]
        if world > 1:
            res = [(s[0], s[1], s[2]) for s in pipe.run_segments_sharded(get, n, spec["dur"], t_offset=spec["t0"],
                                                                         segment_pairs=spec["seg"], write_sinks=files)]
        else:
            res = [(np.array(s[0]), s[2], s[3]) for s in pipe.run_segments(get, n, spec["dur"], t_offset=spec["t0"],
                                                                           segment_pairs=spec["seg"])]
        video = _written(r, opened, out) if r is not None else None
        counters = _counters(em)
        em.cleanup()
        q.put((rank, dict(rows=np.concatenate([s[0] for s in res]), t=np.concatenate([s[1] for s in res]),
                          nf=[s[2] for s in res], video=video, counters=counters)))
    finally:
        dist.destroy_process_group()


def _assert_sharded_equals_one_gpu(tmp_path, spec, world=2, backend="gloo"):
    from helpers import canonical
    from test_pipeline_segments_sharded import _spawn
    from test_sinks_batched import _files
    one = _spawn(1, _sharded_worker, dict(spec, out=str(tmp_path / "one")))[0]
    res = _spawn(world, _sharded_worker, dict(spec, out=str(tmp_path / "sharded")), backend)
    merged = np.concatenate([res[r]["rows"] for r in range(world)])
    assert len(one["rows"]) > 1000 and len(one["nf"]) >= 3
    assert canonical(merged).tobytes() == canonical(one["rows"]).tobytes()
    for r in range(world):
        assert res[r]["t"].tobytes() == one["t"].tobytes() and res[r]["nf"] == one["nf"], r
        assert res[r]["counters"][3:] == one["counters"][3:], r
    if spec["files"]:
        # the merged stream, in the one-GPU order: the files hold it row by row
        assert _files(tmp_path / "sharded") == _files(tmp_path / "one")
        vid, text = res[0]["video"]
        one_vid, one_text = one["video"]
        assert len(one_vid) >= 5 and vid.shape == one_vid.shape and np.array_equal(vid, one_vid)
        assert text == one_text and res[1]["video"] is None


@pytest.mark.gpu
def test_sharded_equals_one_gpu(tmp_path):
    """Two gloo ranks on one GPU, canonical order, write_sinks: the merged rows, the first rank's event files and DVS
    video equal one GPU's run_segments(None); 23 frames of 346x260 (a size the AEDAT-2.0 writer takes) in segments of 5,
    the last of 3."""
    import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("v2ecore (the reference's writers) does not import")
    _assert_sharded_equals_one_gpu(tmp_path, dict(frames=_clip(23, 260, 346), dur=0.2, t0=0.5, seg=5, files=True))


@pytest.mark.gpu
def test_sharded_centre_surround_equals_one_gpu(tmp_path):
    """The centre-surround model over two ranks (64 rows: bands of 32 with halo rows exchanged) against one GPU, 5 ms
    frame intervals from t = 0 (the first frame only initialises the state, so the second steps from t = 0; a later
    start would take more Euler steps than the model's cap)."""
    _assert_sharded_equals_one_gpu(tmp_path, dict(frames=_clip(41, 64, 96, shift=1), dur=0.2, t0=0.0, seg=7,
                                                  files=False))


@pytest.mark.gpu
def test_sharded_equals_one_gpu_over_nccl(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")
    import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("v2ecore (the reference's writers) does not import")
    _assert_sharded_equals_one_gpu(tmp_path, dict(frames=_clip(23, 260, 346), dur=0.2, t0=0.5, seg=5, files=True),
                                   backend="nccl")
