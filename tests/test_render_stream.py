"""EventRenderer.render_frame_rows and V2EPipeline(..., renderer): the DVS video and its frame-times file from the rows
of consecutive pixel-model frames, cut into the packets v2e.py's stage-3 loop renders (v2e.py:826-846), with every
packet's frame slicing on the device.

CPU: renderer.cut_packets, called on the frames of a clip in calls of every length (with the rows it holds carried from
call to call), against a literal restatement of v2e.py's loop.
GPU (frames bit for bit, the frame-times file byte for byte, the video through a stub v2ecore.v2e_utils):
  * the 18 fixtures of tests/golden/render_ref.npz, one fixture packet per frame, in one call and one call per frame;
  * the pixel model's rows (device RNG, v2e's CLI defaults, 346x260 and 1280x720) in one call and in calls of k frames,
    k coprime to 8, in all four exposure modes, DURATION and COUNT also at long-clip times, against the same rows cut by
    the restatement and fed packet by packet to EventRenderer.render_events_to_frames and to the numpy oracle;
  * V2EPipeline.run / run_segments with a renderer, fixed and automatic U, against the rows they yield fed through
    v2e.py's loop; the rows, offsets and counters of a pipeline without a renderer;
  * run_segments_sharded over two gloo ranks with write_sinks: the first rank's video equals one GPU's; a renderer on
    another rank makes every rank raise;
  * the render's device memory is bounded by its chunk of frames; a DURATION packet over 2^20 intervals inside a
    multi-frame call writes nothing."""
import os
import sys
import types

import numpy as np
import pytest

from render_oracle import AREA_COUNT, COUNT, DURATION, SOURCE, RenderOracle, frame_times_text, video_frames
from test_render_packets import (BATCH_SIZE, CASES, CLI_DEFAULTS, DVS_VID, SIZES, T0S, Recorder, boundary_ties,
                                 exposures, render_with_video, shifted, video)  # noqa: F401 (video: a fixture)
from v2e_b200.renderer import cut_packets


# ---- CPU: the packet cutting ----------------------------------------------------------------------------------------
def v2e_loop(frame_rows, batch_size, first_frame=0):
    """v2e.py:826-846, literally: the packets render_events_to_frames is called with."""
    packets, events = [], np.zeros((0, 4), dtype=np.float32)
    for j, newEvents in enumerate(frame_rows):
        i = first_frame + j
        if newEvents is not None and newEvents.shape[0] > 0:
            events = np.append(events, newEvents, axis=0)
            events = np.array(events)
            if i % batch_size == 0:
                packets.append(events)
                events = np.zeros((0, 4), dtype=np.float32)
    if len(events) > 0:
        packets.append(events)
    return packets


def packets_by_calls(counts, calls, first_frame, packet_frames, base=0):
    """The packets (as row ids) cut_packets gives for frames with `counts` rows, passed in calls [(a, b)] of frames,
    with the rows after each call's last packet held for the next one, as render_frame_rows holds them. Offsets start
    at `base`, as a view into a larger row buffer's would."""
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    out, held = [], np.zeros(0, np.int64)
    for a, b in calls:
        offs = offsets[a:b + 1] + base
        ids = np.concatenate([held, np.arange(offsets[a], offsets[b])])
        ends, keep = cut_packets(offs, first_frame + a, packet_frames, len(held), end_of_clip=b == len(counts))
        assert np.all(np.diff(np.concatenate([[0], ends])) > 0) and keep <= len(ids)
        out += [ids[s:e] for s, e in zip(np.concatenate([[0], ends[:-1]]), ends)]
        held = ids[keep:]
    assert len(held) == 0
    return out


def restated(counts, first_frame, packet_frames):
    offsets = np.concatenate([[0], np.cumsum(counts)])
    frames = [np.repeat(np.arange(a, b, dtype=np.float32)[:, None], 4, 1) for a, b in zip(offsets[:-1], offsets[1:])]
    return [p[:, 0].astype(np.int64) for p in v2e_loop(frames, packet_frames, first_frame)]


def _counts(seed, T):
    rng = np.random.default_rng(seed)
    c = rng.integers(0, 6, T)
    c[rng.random(T) < 0.35] = 0                          # frames without rows, boundary frames among them
    return c


@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("packet_frames", [1, 3, 8])
def test_cut_packets_in_calls_of_every_length_equal_v2e_loop(seed, packet_frames):
    T = 29
    counts = _counts(seed, T)
    counts[0] = seed % 2 * 3                             # frame 0 with and without rows
    first_frame = [0, 0, 5, 16][seed % 4]
    idx = first_frame + np.arange(T)
    b = np.flatnonzero((idx % packet_frames == 0) & (idx > first_frame))
    counts[b[0]] = 0                                     # a boundary frame without rows
    counts[b[1]] = max(counts[b[1]], 1)                  # and one with rows
    want = restated(counts, first_frame, packet_frames)
    for k in range(1, T + 1):
        calls = [(a, min(T, a + k)) for a in range(0, T, k)]
        got = packets_by_calls(counts, calls, first_frame, packet_frames, base=seed)
        assert len(got) == len(want), k
        assert all(np.array_equal(g, w) for g, w in zip(got, want)), k


@pytest.mark.parametrize("seed", range(20))
def test_cut_packets_at_random_call_boundaries(seed):
    rng = np.random.default_rng(100 + seed)
    T = int(rng.integers(1, 60))
    counts = _counts(seed, T)
    pf, first = int(rng.integers(1, 10)), int(rng.integers(0, 20))
    cuts = sorted(set(rng.integers(1, T + 1, int(rng.integers(0, 8))).tolist()) | {T})
    calls = list(zip([0] + cuts[:-1], cuts))
    got = packets_by_calls(counts, calls, first, pf)
    want = restated(counts, first, pf)
    assert len(got) == len(want) and all(np.array_equal(g, w) for g, w in zip(got, want))


def test_cut_packets_cases():
    o = np.array([0, 0, 2, 2, 5, 6])                     # frames 0..4 with 0, 2, 0, 3, 1 rows
    e, keep = cut_packets(o, 0, 2)                       # boundaries 0 and 2 have no rows, 4 has one
    assert list(e) == [6] and keep == 6
    e, keep = cut_packets(o, 1, 2)                       # frames 1..5: boundaries 2 and 4 have rows
    assert list(e) == [2, 5] and keep == 5
    e, keep = cut_packets(o, 1, 2, held=4)
    assert list(e) == [6, 9] and keep == 9
    e, keep = cut_packets(o[:3], 0, 2)                   # frames 0, 1: no packet ends, every row held
    assert len(e) == 0 and keep == 0
    e, keep = cut_packets(o, 0, 3, held=1, end_of_clip=True)   # boundary 3 has rows: cut after row 5; leftover 1 row
    assert list(e) == [6, 7] and keep == 7
    e, keep = cut_packets(np.array([4]), 0, 8, held=3, end_of_clip=True)       # no frames, held rows only
    assert list(e) == [3] and keep == 3
    e, keep = cut_packets(np.array([4]), 0, 8, held=0, end_of_clip=True)
    assert len(e) == 0 and keep == 0
    with pytest.raises(ValueError):
        cut_packets(o, 0, 0)


# ---- GPU helpers ----------------------------------------------------------------------------------------------------
def _renderer(mode, value, area, out_dir, fs=2):
    from v2e_b200.renderer import EventRenderer, ExposureMode
    return EventRenderer(full_scale_count=fs, output_path=str(out_dir), dvs_vid=DVS_VID,
                         exposure_mode=ExposureMode(mode), exposure_value=value, area_dimension=area)


def _written(r, opened, out_dir, H, W):
    """cleanup(), then (the uint8 frames the video writer got, the frame-times file's text)."""
    r.cleanup()
    rec = opened[-1]
    assert rec.released and (rec.height, rec.width) == (H, W)
    with open(os.path.join(str(out_dir), "dvs-video-frame_times.txt"), "rb") as f:
        text = f.read().decode()
    return (np.stack(rec.frames) if rec.frames else np.zeros((0, H, W, 3), np.uint8)), text


def render_in_calls(rows, offsets, k, H, W, mode, value, area, out_dir, opened, fs=2, packet_frames=BATCH_SIZE):
    """rows through render_frame_rows in calls of k frames (None: one call): (frames finished, video, frame times)."""
    r = _renderer(mode, value, area, out_dir, fs)
    T = len(offsets) - 1
    k = k or T
    n = 0
    for a in range(0, T, k):
        b = min(T, a + k)
        n += r.render_frame_rows(rows, offsets[a:b + 1], a, packet_frames, end_of_clip=b == T, height=H, width=W)
    vid, text = _written(r, opened, out_dir, H, W)
    assert n == len(vid)
    return vid, text


def straddling(offsets, packets_ends, k):
    """Packets whose rows come from more than one call of k frames."""
    T = len(offsets) - 1
    call_of_row = np.repeat(np.arange(T) // k, np.diff(offsets))
    s = 0
    out = 0
    for e in packets_ends:
        out += len(set(call_of_row[s:e].tolist())) > 1
        s = e
    return out


# ---- GPU: the fixtures ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_fixture_packets_as_frames_write_the_reference_video(name, video, tmp_path):
    import torch
    c = CASES[name]
    evs = [ev for ev, _ in c["packets"]]
    rows = np.concatenate(evs).astype(np.float32)
    offsets = np.concatenate([[0], np.cumsum([len(e) for e in evs])]).astype(np.int64)
    for k, as_tensor in ((None, False), (1, True), (None, True)):
        d = tmp_path / ("%s-%s" % (k, as_tensor))
        d.mkdir()
        src = torch.from_numpy(rows).cuda() if as_tensor else rows
        vid, text = render_in_calls(src, offsets, k, c["H"], c["W"], c["mode"], c["value"], c["area"], d, video,
                                    fs=c["fs"], packet_frames=1)
        assert vid.shape == c["video"].shape and np.array_equal(vid, c["video"]), k
        assert text == c["times"], k


# ---- GPU: the pixel model's rows ------------------------------------------------------------------------------------
N_FRAMES = 4 * BATCH_SIZE + 5
FRAME_DT = 0.005
EMPTY_BOUNDARIES = (8, 24)         # boundary frames whose rows are taken out: a packet runs on past them


def pixel_model_frames(H, W):
    """(rows, offsets) of generate_events_batch (device RNG, CLI defaults) on a textured clip whose frame times after
    frame 1 are put on 0.01 s DURATION boundaries every other frame (the first row's float32 time plus k intervals,
    accumulated in float32), so that the rows of a frame's last iteration tie with a boundary; the rows of frames
    EMPTY_BOUNDARIES are then taken out."""
    import torch
    from test_emulator_device_rng import texture_frames
    from v2e_b200 import EventEmulator
    fr = torch.from_numpy(texture_frames(H, W, N_FRAMES, seed=3, speed=1.0, block=8) // 2 + 64).cuda()
    mk = lambda: EventEmulator(device="cuda", rng_mode="device", seed=7, row_order="canonical", **CLI_DEFAULTS)
    em = mk()
    rows1, _ = em.generate_events_batch(fr[:2], np.array([0.0, FRAME_DT]))
    em.cleanup()
    bound = rows1[0, 0]
    t = [0.0, FRAME_DT]
    for i in range(2, N_FRAMES):
        if i % 2:
            while float(bound) <= t[-1] + FRAME_DT / 4:
                bound = bound + 0.01                      # float32 + Python float: float32, as the renderer adds
            t.append(float(bound))
        else:
            t.append(t[-1] + FRAME_DT)
    em = mk()
    rows, offs = em.generate_events_batch(fr, np.array(t))
    em.cleanup()
    assert np.array_equal(rows[:len(rows1)], rows1)
    frames = [rows[a:b] for a, b in zip(offs[:-1], offs[1:])]
    assert len(frames[0]) == 0
    for i in EMPTY_BOUNDARIES:
        assert len(frames[i]) > 0
        frames[i] = frames[i][:0]
    rows = np.concatenate(frames)
    offs = np.concatenate([[0], np.cumsum([len(f) for f in frames])]).astype(np.int64)
    assert np.all(np.diff(rows[:, 0]) >= 0)
    return rows, offs


@pytest.fixture(scope="module")
def model_frames():
    cache = {}

    def get(size):
        if size not in cache:
            cache[size] = pixel_model_frames(*SIZES[size])
        return cache[size]
    return get


PM_CASES = [(s, m, t0) for s in SIZES for m in (DURATION, COUNT, AREA_COUNT, SOURCE)
            for t0 in (T0S if m in (DURATION, COUNT) else T0S[:1])]


@pytest.mark.gpu
@pytest.mark.parametrize("size,mode,t0", PM_CASES, ids=["%s-%d-%g" % c for c in PM_CASES])
def test_pixel_model_rows_in_calls_equal_packet_by_packet(size, mode, t0, model_frames, video, tmp_path):
    import torch
    H, W = SIZES[size]
    rows, offs = model_frames(size)
    (rows,) = shifted([rows], t0)
    frames = [rows[a:b] for a, b in zip(offs[:-1], offs[1:])]
    packets = v2e_loop(frames, BATCH_SIZE)
    ends = np.cumsum([len(p) for p in packets])
    assert len(packets) == N_FRAMES // BATCH_SIZE + 1 - len(EMPTY_BOUNDARIES)
    value, area = exposures(size)[mode]
    o = RenderOracle(2, mode, value, area)
    want = [o.render(p, H, W) for p in packets]
    allw = np.concatenate([w for w in want if w is not None])
    assert len(allw) >= 3
    want_vid, want_text = video_frames(allw, H, W), frame_times_text(DVS_VID, o.times)
    d = tmp_path / "pinned"
    d.mkdir()
    _, vid, text = render_with_video(packets, H, W, 2, mode, value, area, d, video)
    assert np.array_equal(vid, want_vid) and text == want_text
    if mode == DURATION:
        assert boundary_ties(packets, 0.01) > 0
    dev = torch.from_numpy(rows).cuda()
    for k in (None, 1, 3, 5, 7, 9):
        if k:
            assert straddling(offs, ends, k) >= 2, k     # packets held across calls
        d = tmp_path / ("k%s" % k)
        d.mkdir()
        vid, text = render_in_calls(dev if k != 5 else rows, offs, k, H, W, mode, value, area, d, video)
        assert vid.shape == want_vid.shape and np.array_equal(vid, want_vid), k
        assert text == want_text, k


# ---- GPU: the pipeline ----------------------------------------------------------------------------------------------
def _pipe_rows(sl, em, frames, seg, renderer=None):
    from test_pipeline_segments import _counters
    from v2e_b200 import V2EPipeline
    pipe = V2EPipeline(sl, em, renderer=renderer)
    if seg is None:
        res = [pipe.run(frames, 0.2, t_offset=0.5, copy=True)]
    else:
        res = list(pipe.run_segments(lambda a, b: frames[a:b], len(frames), 0.2, t_offset=0.5, segment_pairs=seg,
                                     copy=True))
    out = [(np.array(ev), o, t, n) for ev, o, t, n in res]
    return out, _counters(em)


@pytest.mark.gpu
@pytest.mark.parametrize("auto", [False, True])
@pytest.mark.parametrize("mode", [DURATION, COUNT])
def test_pipeline_with_a_renderer_writes_v2e_loops_video(auto, mode, video, tmp_path):
    from test_pipeline_segments import _auto_clip, _clip, _emulator, _slomo
    H, W = 64, 96
    sl = _slomo(auto)
    frames = _auto_clip(H, W, sl) if auto else _clip(14, H, W, [3] * 13, seed=2)
    value = 0.01 if mode == DURATION else 100
    for seg in (None, 1, 3, 6):
        plain, cnt = _pipe_rows(sl, _emulator(row_order="canonical", **CLI_DEFAULTS), frames, seg)
        d = tmp_path / ("seg%s" % seg)
        d.mkdir()
        r = _renderer(mode, value, None, d)
        got, cnt_r = _pipe_rows(sl, _emulator(row_order="canonical", **CLI_DEFAULTS), frames, seg, renderer=r)
        vid, text = _written(r, video, d, H, W)
        assert cnt_r == cnt and len(got) == len(plain) >= (1 if seg is None else 2)
        for (ev, o, t, n), (ev2, o2, t2, n2) in zip(got, plain):
            assert ev.tobytes() == ev2.tobytes() and np.array_equal(o, o2) and t.tobytes() == t2.tobytes() and n == n2
        per_frame = [ev[a:b] for ev, o, _, _ in got for a, b in zip(o[:-1], o[1:])]
        packets = v2e_loop(per_frame, sl.batch_size)
        e = tmp_path / ("want%s" % seg)
        e.mkdir()
        _, want_vid, want_text = render_with_video(packets, H, W, 2, mode, value, None, e, video)
        assert len(want_vid) >= 3 and len(packets) >= 3
        assert np.array_equal(vid, want_vid) and text == want_text, seg
    sl.cleanup()


# ---- GPU: two gloo ranks --------------------------------------------------------------------------------------------
def _stub_modules(opened):
    def checkAddSuffix(path, suffix):
        return path if path.endswith(suffix) else os.path.splitext(path)[0] + suffix

    def video_writer(output_path, height, width, frame_rate=30, fourcc=None):
        opened.append(Recorder(output_path, height, width, frame_rate))
        return opened[-1]
    pkg = types.ModuleType("v2ecore")
    pkg.__path__ = []
    utils = types.ModuleType("v2ecore.v2e_utils")
    utils.checkAddSuffix, utils.video_writer = checkAddSuffix, video_writer
    pkg.v2e_utils = utils
    return {"v2ecore": pkg, "v2ecore.v2e_utils": utils}


def _sharded_worker(rank, world, port, q, frames, out, render_rank):
    import torch.distributed as dist
    from test_pipeline_segments_sharded import _FILES_KW, _init, _slomo
    _init(rank, world, port)
    try:
        from v2e_b200 import EventEmulator, V2EPipeline
        opened = []
        sys.modules.update(_stub_modules(opened))
        sl = _slomo(False, 3)
        em = EventEmulator(device="cuda:0", seed=9, shard=(rank, world, None), **_FILES_KW)
        r = None
        if rank == render_rank:
            os.makedirs(out)
            r = _renderer(DURATION, 0.01, None, out)
        pipe = V2EPipeline(sl, em, renderer=r)
        try:
            for _ in pipe.run_segments_sharded(lambda a, b: frames[a:b], len(frames), 0.2, t_offset=0.5,
                                               segment_pairs=3, write_sinks=True):
                pass
        except ValueError as e:
            q.put((rank, ("ValueError", str(e))))
            return
        res = None
        if r is not None:
            vid, text = _written(r, opened, out, frames.shape[1], frames.shape[2])
            res = (vid, text)
        em.cleanup()
        sl.cleanup()
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_sharded_first_rank_writes_one_gpus_video(video, tmp_path):
    from test_pipeline_segments import _clip, _slomo
    from test_pipeline_segments_sharded import _FILES_KW, _spawn
    from v2e_b200 import EventEmulator, V2EPipeline
    frames = _clip(14, 64, 96, [3] * 13, seed=2)
    res = _spawn(2, _sharded_worker, frames, str(tmp_path / "sharded"), 0)
    vid, text = res[0]
    assert res[1] is None
    sl = _slomo(False)
    d = tmp_path / "one"
    d.mkdir()
    r = _renderer(DURATION, 0.01, None, d)
    segs = list(V2EPipeline(sl, EventEmulator(device="cuda:0", seed=9, **_FILES_KW), renderer=r).run_segments(
        lambda a, b: frames[a:b], len(frames), 0.2, t_offset=0.5, segment_pairs=3))
    one_vid, one_text = _written(r, video, d, 64, 96)
    sl.cleanup()
    assert len(segs) >= 3 and len(one_vid) >= 5
    assert vid.shape == one_vid.shape and np.array_equal(vid, one_vid) and text == one_text


@pytest.mark.gpu
def test_renderer_on_another_rank_raises_on_every_rank(tmp_path):
    from test_pipeline_segments import _clip
    from test_pipeline_segments_sharded import _spawn
    frames = _clip(14, 64, 96, [3] * 13, seed=2)
    res = _spawn(2, _sharded_worker, frames, str(tmp_path / "sharded"), 1)
    for r in (0, 1):
        assert res[r][0] == "ValueError" and "renderer" in res[r][1], res[r]


# ---- GPU: memory and limits -----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_render_memory_is_bounded_by_the_chunk(video, tmp_path):
    """One call whose packets finish ~20 chunks of frames: every frame is written, as the oracle renders it, and the
    render's device memory stays within a few chunks' buffers, far below one buffer per frame."""
    import torch
    from v2e_b200.renderer import RENDER_CHUNK_FRAMES
    H, W, T = 360, 640, 40
    rng = np.random.default_rng(5)
    per = [np.sort(rng.uniform(f * 0.01, (f + 1) * 0.01, 300)).astype(np.float32) for f in range(T)]
    frames = [np.stack([t, rng.integers(0, W, len(t)), rng.integers(0, H, len(t)), rng.choice([-1.0, 1.0], len(t))],
                       1).astype(np.float32) for t in per]
    rows = np.concatenate(frames)
    offs = np.concatenate([[0], np.cumsum([len(f) for f in frames])]).astype(np.int64)
    o = RenderOracle(2, DURATION, 0.001)
    for p in v2e_loop(frames, 16):
        o.render(p, H, W)
    n = len(o.times)
    assert n > 16 * RENDER_CHUNK_FRAMES
    dev = torch.from_numpy(rows).cuda()
    r = _renderer(DURATION, 0.001, None, tmp_path)
    r.render_frame_rows(dev[:1], offs[:1], 0, 16, height=H, width=W)     # opens the video
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    k = r.render_frame_rows(dev, offs, 0, 16, end_of_clip=True, height=H, width=W)
    torch.cuda.synchronize()
    added = torch.cuda.max_memory_allocated() - base
    vid, text = _written(r, video, tmp_path, H, W)
    assert k == n == len(vid) and text == frame_times_text(DVS_VID, o.times)
    assert np.array_equal(vid, video_frames(np.concatenate([f for f in o_frames(frames, H, W)]), H, W))
    chunk = RENDER_CHUNK_FRAMES * H * W * 5
    print("render of %d frames added %.1f MB (one chunk %.1f MB, all frames at once %.1f MB)"
          % (n, added / 1e6, chunk / 1e6, n * H * W * 5 / 1e6))
    assert added < 2 * chunk + 64 * rows.nbytes + (8 << 20)
    assert added < n * H * W * 5 / 4


def o_frames(frames, H, W):
    o = RenderOracle(2, DURATION, 0.001)
    return [f for f in (o.render(p, H, W) for p in v2e_loop(frames, 16)) if f is not None]


@pytest.mark.gpu
def test_duration_packet_past_2_20_intervals_in_a_call_writes_nothing(video, tmp_path):
    """Frames 1..7 are ordinary; frame 9 jumps 2.2 s at 1 us exposure, so the call's second packet spans more than 2^20
    intervals: ValueError, with no frame of the call written and nothing held."""
    import torch
    ts = [np.float32([0.001 * f + 1e-5 * j for j in range(4)]) for f in range(12)]
    ts[9] = ts[9] + np.float32(2.2)
    ts[10], ts[11] = ts[10] + np.float32(2.2), ts[11] + np.float32(2.2)
    frames = [np.stack([t, np.full(4, 1.0), np.full(4, 2.0), np.ones(4)], 1).astype(np.float32) for t in ts]
    frames[0] = frames[0][:0]
    rows = torch.from_numpy(np.concatenate(frames)).cuda()
    offs = np.concatenate([[0], np.cumsum([len(f) for f in frames])]).astype(np.int64)
    r = _renderer(DURATION, 1e-6, None, tmp_path)
    with pytest.raises(ValueError):
        r.render_frame_rows(rows, offs, 0, 4, end_of_clip=True, height=8, width=8)
    assert r.numFramesWritten == 0 and r.currentFrameStartTime is None and r._n_held == 0
    vid, text = _written(r, video, tmp_path, 8, 8)
    assert len(vid) == 0 and text == frame_times_text(DVS_VID, [])
    # the packets before the jump alone render as the oracle renders them
    ok = RenderOracle(2, DURATION, 1e-6)
    want = [ok.render(p, 8, 8) for p in v2e_loop(frames[:8], 4)]
    assert sum(len(w) for w in want if w is not None) > 0
