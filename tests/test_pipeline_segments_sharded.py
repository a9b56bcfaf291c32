"""V2EPipeline.run_segments_sharded: one clip of any length over several ranks, segment by segment, with the output of
one V2EPipeline.run_clip_sharded call on the whole clip.

CPU: the segment plan over ranks (pipeline.segment_plan(..., world, auto_upsample)); the segments' times against the
times run_clip_sharded builds for the whole clip (pipeline.sharded_times / sharded_span); gloo ranks with a stand-in
upsampler and emulator, one of whose get_frames returns wrong frames in a later segment: every rank raises, none hangs.
GPU: gloo ranks sharing the one test GPU (and NCCL ranks on two GPUs where present), streamed against run_clip_sharded
bit for bit: fixed and automatic U, the frame-by-frame pixel-model paths, labels, the event files and the device-memory
high-water mark."""
import os
import socket

import numpy as np
import pytest
import torch

from v2e_b200.pipeline import segment_plan, sharded_span, sharded_times
from v2e_b200.slomo import clip_times

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _spawn(world, target, *args, timeout=300):
    """Runs target(rank, world, port, q, *args) on `world` spawned ranks; returns {rank: what the rank put}. A rank
    that raises reports the error instead; the others, which may then wait in a collective, are terminated."""
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_guarded, args=(target, r, world, port, q) + args) for r in range(world)]
    for p in procs:
        p.start()
    res, err = {}, None
    try:
        for _ in range(world):
            r, ok, payload = q.get(timeout=timeout)
            if not ok:
                err = "rank %d: %s" % (r, payload)
                break
            res[r] = payload
    finally:
        for p in procs:
            if err is not None:
                p.terminate()
            p.join(timeout=60)
    assert err is None, err
    for p in procs:
        assert p.exitcode == 0
    return res


def _guarded(target, rank, world, port, q, *args):
    import traceback

    class _Q:
        def put(self, item):
            q.put((item[0], True, item[1]))
    try:
        target(rank, world, port, _Q(), *args)
    except BaseException:
        q.put((rank, False, traceback.format_exc()))
        raise


def _init(rank, world, port, backend="gloo"):
    """Joins the group; returns this rank's device (gloo ranks share cuda:0, NCCL ranks get one GPU each)."""
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    if backend == "gloo":
        dist.init_process_group("gloo", rank=rank, world_size=world)
        return "cuda:0"
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    return "cuda:%d" % rank


# ---- CPU: the plan ------------------------------------------------------------------------------------------------
def _today(n_frames, batch_size, segment_pairs):
    """segment_plan before it took world / auto_upsample."""
    sp = 64 if segment_pairs is None else segment_pairs
    sp = -(-sp // batch_size) * batch_size
    return [(p0, min(p0 + sp, n_frames - 1)) for p0 in range(0, n_frames - 1, sp)]


@pytest.mark.parametrize("auto", [False, True])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("segment_pairs", [1, 4, 7, 24, None])
@pytest.mark.parametrize("batch_size", [1, 3, 8])
@pytest.mark.parametrize("n_frames", [2, 3, 5, 10, 26, 27, 200])
def test_sharded_segment_plan(n_frames, batch_size, segment_pairs, world, auto):
    n_pairs = n_frames - 1
    unit = batch_size if auto else 1
    units = lambda p0, p1: -(-(p1 - p0) // unit)           # pairs, or batches with auto_upsample
    if units(0, n_pairs) < world:
        with pytest.raises(ValueError, match="fewer"):
            segment_plan(n_frames, batch_size, segment_pairs, world=world, auto_upsample=auto)
        return
    plan = segment_plan(n_frames, batch_size, segment_pairs, world=world, auto_upsample=auto)
    assert plan[0][0] == 0 and plan[-1][1] == n_pairs                     # every pair once, in order
    for (a0, a1), (b0, b1) in zip(plan, plan[1:]):
        assert a1 == b0
    for p0, p1 in plan:
        assert p1 > p0 and p0 % batch_size == 0                           # on the clip's batch boundaries
        assert units(p0, p1) >= world                                     # run_clip_sharded accepts the segment
    sp = 64 if segment_pairs is None else segment_pairs
    sp = -(-max(sp, world * unit) // batch_size) * batch_size
    unfolded = _today(n_frames, batch_size, sp)
    if units(*unfolded[-1]) < world:                                      # a short tail joins the segment before it
        assert plan == unfolded[:-2] + [(unfolded[-2][0], n_pairs)]
    else:
        assert plan == unfolded
    if world == 1 and not auto:
        assert segment_plan(n_frames, batch_size, segment_pairs) == plan == _today(n_frames, batch_size, segment_pairs)


def test_sharded_segment_plan_cases():
    assert segment_plan(14, 3, 3, world=2) == [(0, 3), (3, 6), (6, 9), (9, 13)]             # 1-pair tail folded
    assert segment_plan(14, 3, 3, world=3) == [(0, 3), (3, 6), (6, 9), (9, 13)]
    assert segment_plan(14, 3, 3, world=4) == [(0, 6), (6, 13)]                             # raised to 4, then 6
    assert segment_plan(26, 2, 1, world=2, auto_upsample=True) == [(0, 4), (4, 8), (8, 12), (12, 16), (16, 20),
                                                                  (20, 25)]
    assert segment_plan(6, 2, 1, world=3, auto_upsample=True) == [(0, 5)]                  # 3 batches: 2, 2, 1
    for n, bs, world, auto in ((3, 1, 3, False), (6, 2, 4, True), (4, 8, 2, True), (2, 1, 2, False)):
        with pytest.raises(ValueError):
            segment_plan(n, bs, None, world=world, auto_upsample=auto)


# ---- CPU: the times -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(24))
def test_segment_times_equal_run_clip_sharded_times(seed):
    """The seconds t_offset + f * times of every segment, concatenated, against the ones run_clip_sharded builds for
    the whole clip (np.arange(n_pairs * U) * (1 / U) with a fixed U, slomo.clip_times of the per-batch U's with
    auto_upsample), bit for bit; f from sharded_span when there is more than one segment."""
    rng = np.random.default_rng(seed)
    auto = seed % 2 == 1
    world = int(rng.integers(1, 5))
    batch_size = int(rng.integers(1, 9))
    n_pairs = int(rng.integers(world * (batch_size if auto else 1), 400))
    bs = min(batch_size, n_pairs)
    n_batches = -(-n_pairs // bs)
    U = int(rng.integers(2, 60))
    ups = [int(u) for u in rng.integers(2, 60, n_batches)]
    src, t0 = float(rng.uniform(0.01, 1000.0)), float(rng.uniform(0, 5000))
    times = clip_times(ups, n_pairs, batch_size)[0] if auto else np.arange(n_pairs * U) * (1.0 / U)
    want = t0 + src / (np.max(times) - np.min(times)) * times             # run_clip_sharded, v2e.py:794-797
    plan = segment_plan(n_pairs + 1, batch_size, int(rng.integers(1, 50)), world=world, auto_upsample=auto)
    seg = [sharded_times(n_pairs, batch_size, (p0, p1), ups[p0 // bs:-(-p1 // bs)] if auto else U)
           for p0, p1 in plan]
    if len(plan) > 1:
        f = src / sharded_span(n_pairs, batch_size, ups[-1] if auto else U, auto)
    else:
        f = src / (np.max(seg[0]) - np.min(seg[0]))
    got = np.concatenate([t0 + f * s for s in seg])
    assert got.dtype == np.float64 and np.array_equal(got, want) and got.tobytes() == want.tobytes()
    assert np.concatenate(seg).tobytes() == times.tobytes()


# ---- CPU: every rank raises together ------------------------------------------------------------------------------
class _StubSloMo:
    """Upsampler stand-in: U = 2, every interpolated frame is its pair's first source frame."""
    auto_upsample, upsampling_factor, batch_size = False, 2, 2

    def writes_video(self):
        return False

    def interpolate_frames(self, frames, write_video=True, **kw):
        frames = torch.as_tensor(frames)
        n = frames.shape[0] - 1
        return frames[:-1].repeat_interleave(2, 0), np.arange(2 * n) * 0.5, 2.0


class _StubEmulator:
    """Band-emulator stand-in: records the band frames it gets."""
    label_signal_noise, row_order, _sinks, device, rng_mode = False, None, None, "cpu", "device"

    def __init__(self, shard):
        self.shard, self.frames = shard, []

    def cs_halo_rows(self, H):
        return 0

    def generate_events_band_batch(self, bands, t, H):
        self.frames.append(bands.shape[0])
        return np.zeros((0, 4), np.float32), np.zeros(bands.shape[0] + 1, np.int64)


def _bad_frames_worker(rank, world, port, q, bad_rank, bad_seg, kind):
    import torch.distributed as dist
    _init(rank, world, port)
    try:
        from v2e_b200 import V2EPipeline
        src = np.repeat(np.arange(13, dtype=np.uint8)[:, None, None], 6 * 5, 1).reshape(13, 6, 5)
        plan = segment_plan(13, 2, 4, world=world)

        def get(a, b):
            if rank == bad_rank and plan[bad_seg][0] <= a < plan[bad_seg][1]:
                return src[a:b, :, :4] if kind == "shape" else src[a:b].astype(np.float32)
            return src[a:b]
        em = _StubEmulator((rank, world, None))
        done, msg = 0, None
        try:
            for _ in V2EPipeline(_StubSloMo(), em).run_segments_sharded(get, 13, 0.5, segment_pairs=4):
                done += 1
        except ValueError as e:
            msg = str(e)
        q.put((rank, (done, msg, len(plan))))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,bad_rank,bad_seg,kind", [(2, 1, 1, "shape"), (2, 0, 2, "dtype"), (3, 1, 0, "shape"),
                                                         (3, 2, 1, "dtype")])
def test_wrong_frames_on_one_rank_raise_on_every_rank(world, bad_rank, bad_seg, kind):
    """One rank's get_frames returns frames of the wrong shape or dtype in segment k: every rank yields the segments
    before k, then raises ValueError naming segment k and that rank (none waits in a collective)."""
    res = _spawn(world, _bad_frames_worker, bad_rank, bad_seg, kind, timeout=120)
    for r in range(world):
        done, msg, m = res[r]
        assert m >= 3 and done == bad_seg, (r, done)
        assert msg is not None and ("segment %d of %d" % (bad_seg, m)) in msg and ("rank %d" % bad_rank) in msg, msg


# ---- GPU ----------------------------------------------------------------------------------------------------------
_NOISE = dict(cutoff_hz=200, leak_rate_hz=0.2, shot_noise_rate_hz=10.0, sigma_thres=0.02)
_CLI = dict(pos_thres=0.2, neg_thres=0.2, sigma_thres=0.03, cutoff_hz=300.0, leak_rate_hz=0.01,
            shot_noise_rate_hz=0.001, refractory_period_s=0.0005)          # bench.CLI_DEFAULTS (v2e's CLI)


def _slomo(auto, batch_size, U=3, device="cuda:0"):
    from test_slomo_gpu import _weights
    from v2e_b200 import SuperSloMo
    fc, at = _weights(5)
    return SuperSloMo(model=None, auto_upsample=auto, upsampling_factor=None if auto else U, batch_size=batch_size,
                      device=device, state_dicts={"state_dictFC": fc, "state_dictAT": at})


def _counters(em):
    return (em.num_events_total, em.num_events_on, em.num_events_off, em.frame_counter, float(em.t_previous))


def _both_worker(rank, world, port, q, spec, backend="gloo"):
    """run_clip_sharded and run_segments_sharded on the same clip, each on a fresh emulator; with spec["out"] the first
    rank writes event files (clip/ and seg/ under it)."""
    import torch.distributed as dist
    dev = _init(rank, world, port, backend)
    try:
        if spec.get("out"):
            import ref_shim
            ref_shim.load_reference()
        from v2e_b200 import EventEmulator, V2EPipeline
        frames = spec["frames"]
        sl = _slomo(spec["auto"], spec["batch_size"], spec.get("U", 3), device=dev)
        labels = spec.get("labels", False)
        dur, t0 = spec.get("duration", 0.2), spec.get("t_offset", 0.5)
        out = {}
        for name in ("clip", "seg"):
            kw = dict(spec["em"])
            if spec.get("out") and rank == 0:
                folder = os.path.join(spec["out"], name)
                os.makedirs(folder)
                kw.update(output_folder=folder, dvs_text="ev", dvs_aedat2="ev", output_width=frames.shape[2],
                          output_height=frames.shape[1])
            em = EventEmulator(device=dev, seed=9, shard=(rank, world, None), **kw)
            pipe = V2EPipeline(sl, em)
            sinks = bool(spec.get("out"))
            if name == "clip":
                res = [pipe.run_clip_sharded(frames, dur, t_offset=t0, return_labels=labels, write_sinks=sinks)]
            else:
                res = list(pipe.run_segments_sharded(lambda a, b: frames[a:b], len(frames), dur, t_offset=t0,
                                                     segment_pairs=spec["seg"], return_labels=labels,
                                                     write_sinks=sinks))
            counters = _counters(em)
            files = (em.dvs_text.numEventsWritten, em.dvs_aedat2.numEventsWritten) if sinks and rank == 0 else None
            em.cleanup()
            out[name] = dict(res=res, counters=counters, files=files)
        sl.cleanup()
        q.put((rank, out))
    finally:
        dist.destroy_process_group()


def _assert_equal_to_clip(res, world, exact=True):
    """Per rank: the segments, concatenated, equal the run_clip_sharded call (rows bit for bit, or as a multiset of
    (t, x, y, p) when exact is False; times, frame counts, labels, counters)."""
    from helpers import canonical
    for r in range(world):
        (one,), segs = res[r]["clip"]["res"], res[r]["seg"]["res"]
        assert len(segs) >= 3, (r, len(segs))
        rows = np.concatenate([s[0] for s in segs])
        if exact:
            assert rows.tobytes() == np.asarray(one[0]).tobytes(), r
        else:
            assert canonical(rows).tobytes() == canonical(np.asarray(one[0])).tobytes(), r
        t = np.concatenate([s[1] for s in segs])
        assert t.dtype == np.float64 and t.tobytes() == one[1].tobytes(), r
        assert sum(s[2] for s in segs) == one[2] == len(t), r
        if len(one) > 3:
            assert np.concatenate([s[3] for s in segs]).tobytes() == one[3].tobytes(), r
        assert res[r]["seg"]["counters"] == res[r]["clip"]["counters"], r
        assert all(np.array_equal(res[q]["seg"]["res"][k][1], segs[k][1]) for q in range(world) for k in
                   range(len(segs)))                                     # every rank has the same times
    assert sum(len(res[r]["clip"]["res"][0][0]) for r in range(world)) > 1000


def _clip(n, H, W, shifts, seed=0):
    from test_pipeline_segments import _clip as clip
    return clip(n, H, W, shifts, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_fixed_u_segments_equal_run_clip_sharded(world):
    """(a) U = 3, batches of 3, 13 pairs in segments of 3 (a 1-pair tail folded into the fourth), device RNG with v2e's
    CLI-default noise, canonical row order: every rank's rows, the times and the counters bit for bit."""
    spec = dict(frames=_clip(14, 64, 96, [3] * 13), auto=False, batch_size=3, seg=3,
                em=dict(_CLI, rng_mode="device", row_order="canonical"))
    _assert_equal_to_clip(_spawn(world, _both_worker, spec), world)


def _auto_frames(sl, n=26, H=64, W=96):
    """n frames whose per-batch U's differ, the last batch's from the first's."""
    for seed in range(16):
        rng = np.random.default_rng(seed)
        shifts = np.repeat(rng.choice([1, 2, 6, 10, 14], n), 2)[:n - 1]
        frames = _clip(n, H, W, shifts, seed)
        _, _, _, ups = sl.interpolate_frames(frames, return_ups=True)
        if len(set(ups)) >= 3 and ups[-1] != ups[0]:
            return frames, ups
    raise AssertionError("no candidate clip whose per-batch U's differ")


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_auto_upsampled_segments_equal_run_clip_sharded_and_one_gpu(world):
    """(b) A U chosen per batch (batches of 2, 25 pairs: 13 batches, the last short), segments of `world` batches with
    the tail folded: the time scale comes from the pre-pass over the last batch. Equal to run_clip_sharded bit for bit,
    and, merged over the ranks, to one GPU's run_segments on the same clip."""
    from helpers import canonical
    from v2e_b200 import EventEmulator, V2EPipeline
    sl = _slomo(True, 2)
    frames, ups = _auto_frames(sl)
    kw = dict(_NOISE, rng_mode="device", row_order="canonical")
    em = EventEmulator(device="cuda:0", seed=9, **kw)
    one = list(V2EPipeline(sl, em).run_segments(lambda a, b: frames[a:b], len(frames), 0.2, t_offset=0.5,
                                                segment_pairs=4, copy=True))
    want = np.concatenate([s[0] for s in one])
    want_t = np.concatenate([s[2] for s in one])
    em.cleanup()
    sl.cleanup()
    torch.cuda.empty_cache()
    res = _spawn(world, _both_worker, dict(frames=frames, auto=True, batch_size=2, seg=1, em=kw))
    _assert_equal_to_clip(res, world)
    got = np.concatenate([np.concatenate([s[0] for s in res[r]["seg"]["res"]]) for r in range(world)])
    assert canonical(got).tobytes() == canonical(want).tobytes()
    assert np.concatenate([s[1] for s in res[0]["seg"]["res"]]).tobytes() == want_t.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("case", ["centre_surround", "scidvs_pr_noise", "replay_noise"])
def test_frame_by_frame_paths_equal_run_clip_sharded(world, case):
    """(c) The pixel-model paths that run frame by frame: the centre-surround model (halo rows exchanged per Euler
    chunk), SCIDVS with photoreceptor noise (device RNG), and replay mode with leak and shot noise (generate_events_band
    per frame). Rows as a multiset of (t, x, y, p), times, frame counts and counters equal run_clip_sharded's."""
    n = 14
    em = {"centre_surround": dict(rng_mode="device", cs_lambda_pixels=4, cs_tau_p_ms=2.0, cutoff_hz=200,
                                  leak_rate_hz=0, shot_noise_rate_hz=0, sigma_thres=0.02, refractory_period_s=0.001),
          "scidvs_pr_noise": dict(rng_mode="device", scidvs=True, photoreceptor_noise=True, cutoff_hz=100,
                                  leak_rate_hz=0.5, shot_noise_rate_hz=5.0, sigma_thres=0.03,
                                  pr_vrms_tape=[0.05] * (3 * (n - 1))),
          "replay_noise": dict(_NOISE, rng_mode="replay")}[case]
    # frame intervals for which the Euler-step and event-count caps hold: those of test_multi_gpu's centre-surround
    # case, and 1 ms for the noisy models
    timing = dict(duration=0.2, t_offset=0.0) if case == "centre_surround" else dict(duration=0.039)
    spec = dict(frames=_clip(n, 64, 96, [3] * (n - 1)), auto=False, batch_size=3, seg=3, em=em, **timing)
    _assert_equal_to_clip(_spawn(world, _both_worker, spec), world, exact=False)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_labels_equal_run_clip_sharded(world):
    """(d) return_labels: the signal / noise labels of every rank's rows, segment by segment, equal run_clip_sharded's
    (shot-noise rows present)."""
    spec = dict(frames=_clip(14, 64, 96, [3] * 13), auto=False, batch_size=3, seg=3, labels=True,
                em=dict(_NOISE, rng_mode="device", row_order="canonical", label_signal_noise=True))
    res = _spawn(world, _both_worker, spec)
    _assert_equal_to_clip(res, world)
    lab = np.concatenate([res[r]["clip"]["res"][0][3] for r in range(world)])
    assert lab.sum() > 0 and (~lab).sum() > 0


_FILES_KW = dict(rng_mode="device", row_order="canonical", label_signal_noise=True, cutoff_hz=200, sigma_thres=0.0)


def _hash_clip(lo, hi, thres):
    """346 x 260 frames (U = 3, batches of 3) whose first 4 pairs change only a block in rows 116..119 (between lo and
    hi), then a texture moves over the whole frame; thres: the pixel model's thresholds."""
    n, H, W = 14, 260, 346
    fr = np.full((n, H, W), 128, np.uint8)
    for k in range(5):
        fr[k, 116:120, 100:200] = lo if k % 2 == 0 else hi
    fr[5:] = _clip(n - 5, H, W, [4] * (n - 6), seed=3)
    return fr, dict(_FILES_KW, pos_thres=thres, neg_thres=thres)


def _hash_first_segment():
    """A _hash_clip whose first segment of 3 pairs has events only in rows 116..119 -- records whose first AEDAT-2.0
    byte is '#' (flipped y >> 2 == 35), which the writer drops while it has written nothing -- so that the dropping has
    to continue into segment 1. The warps of the upsampler decide which rows change, so candidates are tried on one
    GPU."""
    from v2e_b200 import EventEmulator, V2EPipeline
    sl = _slomo(False, 3)
    for lo, hi, thres in ((128, 160, 0.2), (128, 200, 0.4), (110, 150, 0.25), (128, 255, 0.6), (100, 140, 0.3)):
        frames, kw = _hash_clip(lo, hi, thres)
        em = EventEmulator(device="cuda:0", seed=9, **kw)
        segs = [np.array(s[0]) for s in V2EPipeline(sl, em).run_segments(lambda a, b: frames[a:b], len(frames), 0.2,
                                                                          segment_pairs=3, copy=True)]
        em.cleanup()
        first = (frames.shape[1] - 1 - segs[0][:, 2].astype(int)) >> 2
        if len(first) and np.all(first == 35):
            sl.cleanup()
            torch.cuda.empty_cache()
            return frames, kw
    sl.cleanup()
    raise AssertionError("no candidate clip whose first segment holds only '#' records")


def _one_gpu_files_worker(rank, world, port, q, out, frames, kw):
    import torch.distributed as dist
    _init(rank, world, port)
    try:
        import ref_shim
        ref_shim.load_reference()
        from v2e_b200 import EventEmulator, V2EPipeline
        os.makedirs(out)
        sl = _slomo(False, 3)
        em = EventEmulator(device="cuda:0", seed=9, output_folder=out, dvs_text="ev", dvs_aedat2="ev",
                           output_width=frames.shape[2], output_height=frames.shape[1], **kw)
        rows = V2EPipeline(sl, em).run(frames, 0.2, t_offset=0.5, copy=True)[0]
        files = (em.dvs_text.numEventsWritten, em.dvs_aedat2.numEventsWritten)
        em.cleanup()
        sl.cleanup()
        q.put((rank, (len(rows), files)))
    finally:
        dist.destroy_process_group()


def _assert_files(tmp_path, world, backend="gloo"):
    import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("v2ecore (the reference's writers) does not import")
    from test_sinks_batched import _files
    frames, kw = _hash_first_segment()
    spec = dict(frames=frames, auto=False, batch_size=3, seg=3, em=kw, out=str(tmp_path / "sharded"))
    res = _spawn(world, _both_worker, spec, backend)
    _assert_equal_to_clip(res, world)
    one = _spawn(1, _one_gpu_files_worker, str(tmp_path / "one"), frames, kw)[0]
    n = sum(len(res[r]["clip"]["res"][0][0]) for r in range(world))
    assert one[0] == n and one[1] == (n, n) == res[0]["clip"]["files"] == res[0]["seg"]["files"]
    for r in range(1, world):
        assert res[r]["seg"]["files"] is None
    clip, seg = _files(tmp_path / "sharded" / "clip"), _files(tmp_path / "sharded" / "seg")
    assert seg == clip == _files(tmp_path / "one")
    # segment 0 wrote only '#' records, all dropped; the drop went on into segment 1
    seg0 = np.concatenate([res[r]["seg"]["res"][0][0] for r in range(world)])
    first_byte = (frames.shape[1] - 1 - seg0[:, 2].astype(int)) >> 2
    assert len(seg0) > 0 and np.all(first_byte == 35)
    assert n - len(seg[1]) // 8 > len(seg0) and not seg[1].startswith(b"#")


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_event_files_equal_run_clip_sharded_and_one_gpu(tmp_path, world):
    """(e) write_sinks with dvs_text and dvs_aedat2, labels on: the first rank's text and AEDAT-2.0 bodies equal
    run_clip_sharded's and one GPU's V2EPipeline.run's byte for byte, the other ranks open no file, and the AEDAT-2.0
    rule that drops leading '#' records carries from segment 0 into segment 1."""
    _assert_files(tmp_path, world)


def _memory_worker(rank, world, port, q, frames, seg):
    import torch.distributed as dist
    dev = _init(rank, world, port)
    try:
        from v2e_b200 import EventEmulator, V2EPipeline
        sl = _slomo(False, 4, U=10)
        n = len(frames)

        def added(streamed):
            em = EventEmulator(device=dev, seed=9, rng_mode="device", shard=(rank, world, None), **_NOISE)
            pipe = V2EPipeline(sl, em)
            torch.cuda.synchronize()
            before = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            if streamed:
                for _ in pipe.run_segments_sharded(lambda a, b: frames[a:b], n, 0.1, segment_pairs=seg):
                    pass
            else:
                pipe.run_clip_sharded(frames, 0.1)
            torch.cuda.synchronize()
            p = torch.cuda.max_memory_allocated() - before
            em.cleanup()
            return p
        added(True)                                  # the SloMo engine and its buffers exist before any measurement
        q.put((rank, (added(True), added(False))))
        sl.cleanup()
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_device_memory_depends_on_the_segment_not_the_clip():
    """(f) 346x260, U = 10, 64 pairs over 2 ranks: with segments of 8 pairs each rank's peak of allocated device memory
    above what it held before stays below a third of what run_clip_sharded adds on the same clip."""
    frames = _clip(65, 260, 346, [3] * 64)
    res = _spawn(2, _memory_worker, frames, 8)
    for r in (0, 1):
        seg, clip = res[r]
        assert 0 < seg < clip / 3, (r, seg, clip)


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["rows", "files"])
def test_segments_equal_run_clip_sharded_over_nccl(tmp_path, what):
    """(a) and (e) over NCCL, one GPU per rank (parallel.exchange_frame_bands' all-to-all)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")
    if what == "files":
        _assert_files(tmp_path, 2, backend="nccl")
        return
    spec = dict(frames=_clip(14, 64, 96, [3] * 13), auto=False, batch_size=3, seg=3,
                em=dict(_CLI, rng_mode="device", row_order="canonical"))
    _assert_equal_to_clip(_spawn(2, _both_worker, spec, "nccl"), 2)
