"""SuperSloMo's two videos (slomo.py:288-303, 468-491): `vid_orig`, the source frames, and `vid_slomo`, the
interpolated frames in output order, written GRAY2BGR through v2ecore.v2e_utils.video_writer; and the constructor
keywords v2e.py passes by default (v2e.py:467-478: video_path, vid_orig, vid_slomo, preview=True).

CPU: construction, the preview warning and the writers' lifecycle, with `video_writer` replaced by a recording stand-in
(or made unimportable). GPU: the frames every path writes -- the file API, the in-memory path, V2EPipeline.run -- and a
round trip through a real cv2.VideoWriter; a sharded clip writes nothing."""
import glob
import logging
import os
import sys
import types

import numpy as np
import pytest
import torch

V2E_DEFAULTS = dict(model="SuperSloMo39.ckpt", auto_upsample=True, upsampling_factor=1, vid_orig="video_orig.avi",
                    vid_slomo="video_slomo.avi", preview=True, batch_size=8)     # v2e.py:467-478, v2e_args.py


class _RecWriter:
    """Stands in for the cv2.VideoWriter that v2ecore.v2e_utils.video_writer returns: keeps every frame."""

    def __init__(self, log, fn, h, w, frame_rate):
        self.fn, self.h, self.w, self.frame_rate = fn, h, w, frame_rate
        self.frames, self.released = [], False
        log.append(self)

    def write(self, frame):
        assert frame.dtype == np.uint8 and frame.shape == (self.h, self.w, 3)
        self.frames.append(frame.copy())

    def release(self):
        self.released = True


def _writer_module(make):
    pkg = types.ModuleType("v2ecore")
    mod = types.ModuleType("v2ecore.v2e_utils")
    mod.video_writer = make
    pkg.v2e_utils = mod
    return pkg, mod


def _inject_writer(monkeypatch, make=None):
    """Replaces v2ecore.v2e_utils.video_writer(output_path, height, width, frame_rate=30) (v2e_utils.py:277);
    returns the list of writers it opened, in order."""
    log = []
    pkg, mod = _writer_module(make or (lambda fn, h, w, frame_rate=30: _RecWriter(log, fn, h, w, frame_rate)))
    monkeypatch.setitem(sys.modules, "v2ecore", pkg)
    monkeypatch.setitem(sys.modules, "v2ecore.v2e_utils", mod)
    return log


def _warnings(caplog, text):
    return [r for r in caplog.records if r.levelno == logging.WARNING and text in r.getMessage()]


def _cpu_slomo(monkeypatch, **kw):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    from v2e_b200.slomo import SuperSloMo
    return SuperSloMo(**kw)


# ---- CPU ---------------------------------------------------------------------------------------------------------------
def test_v2e_default_keywords_construct(monkeypatch, tmp_path):
    """The keywords v2e.py passes without --skip_video_output / --no_preview are accepted; nothing is opened before
    the first batch."""
    s = _cpu_slomo(monkeypatch, video_path=str(tmp_path), **V2E_DEFAULTS)
    assert s.writes_video()
    assert s.ori_writer is None and s.slomo_writer is None
    assert s.numOrigVideoFramesWritten == 0 and s.numSlomoVideoFramesWritten == 0
    assert os.listdir(tmp_path) == []
    s.cleanup()


@pytest.mark.parametrize("preview", [False, True])
def test_preview_is_ignored_with_one_warning(monkeypatch, caplog, preview):
    caplog.set_level(logging.WARNING)
    _cpu_slomo(monkeypatch, model=None, auto_upsample=False, upsampling_factor=2, preview=preview)
    assert len(_warnings(caplog, "preview")) == int(preview)


def test_writers_opened_once_at_output_size(monkeypatch, tmp_path, caplog):
    """slomo.py:288-303: one writer per video name, (path, height, width, frame_rate=avi_frame_rate); later calls
    append to the same writers; cleanup() releases both and nothing reopens a finished file."""
    caplog.set_level(logging.INFO, logger="v2e_b200.slomo")
    log = _inject_writer(monkeypatch)
    s = _cpu_slomo(monkeypatch, video_path=str(tmp_path), avi_frame_rate=25, **V2E_DEFAULTS)
    s._open_writers(72, 100)
    s._open_writers(72, 100)
    assert [(w.fn, w.h, w.w, w.frame_rate) for w in log] == [
        (os.path.join(str(tmp_path), "video_orig.avi"), 72, 100, 25),
        (os.path.join(str(tmp_path), "video_slomo.avi"), 72, 100, 25)]
    assert s.ori_writer is log[0] and s.slomo_writer is log[1]
    s.numOrigVideoFramesWritten, s.numSlomoVideoFramesWritten = 8, 21
    s.cleanup()
    assert all(w.released for w in log) and s.ori_writer is None and s.slomo_writer is None
    closing = [r.getMessage() for r in caplog.records if r.getMessage().startswith("closing")]
    assert closing == ["closing original video AVI video_orig.avi after writing 8 frames",
                       "closing slomo video AVI video_slomo.avi after writing 21 frames"]
    s._open_writers(72, 100)
    assert len(log) == 2


def test_without_video_writer_one_warning_no_files(monkeypatch, tmp_path, caplog):
    caplog.set_level(logging.WARNING)
    monkeypatch.setitem(sys.modules, "v2ecore", None)
    monkeypatch.setitem(sys.modules, "v2ecore.v2e_utils", None)
    s = _cpu_slomo(monkeypatch, video_path=str(tmp_path), **dict(V2E_DEFAULTS, preview=False))
    s._open_writers(72, 100)
    s._open_writers(72, 100)
    assert len(_warnings(caplog, "video_path ignored")) == 1
    assert s.ori_writer is None and s.slomo_writer is None
    assert os.listdir(tmp_path) == []


def test_no_video_names_no_import(monkeypatch, tmp_path, caplog):
    """video_path with both names None (v2e.py's --vid_orig None --vid_slomo None) writes nothing and warns nothing."""
    caplog.set_level(logging.WARNING)
    monkeypatch.setitem(sys.modules, "v2ecore.v2e_utils", None)
    s = _cpu_slomo(monkeypatch, model=None, auto_upsample=False, upsampling_factor=2, video_path=str(tmp_path),
                   vid_orig=None, vid_slomo=None)
    assert not s.writes_video()
    s._open_writers(72, 100)
    assert not caplog.records and os.listdir(tmp_path) == []


# ---- GPU ---------------------------------------------------------------------------------------------------------------
H, W = 72, 100
_EMU_KW = dict(cutoff_hz=200, leak_rate_hz=0, shot_noise_rate_hz=0, refractory_period_s=0.001, sigma_thres=0.02)


def _clip(n, step, seed=3):
    """n frames of a blocky texture translating `step` px per frame."""
    rng = np.random.default_rng(seed)
    big = np.kron(rng.integers(30, 220, (H // 8 + 2, (W + step * n) // 8 + 2)), np.ones((8, 8))).astype(np.uint8)
    return np.stack([big[3:3 + H, step * k:step * k + W] for k in range(n)])


def _slomo(auto=False, batch_size=3, **kw):
    from test_slomo_gpu import _weights
    from v2e_b200 import SuperSloMo
    fc, at = _weights(5)
    return SuperSloMo(model=None, auto_upsample=auto, upsampling_factor=None if auto else 3, batch_size=batch_size,
                      state_dicts={"state_dictFC": fc, "state_dictAT": at}, **kw)


def _bgr(gray):
    import cv2
    return [cv2.cvtColor(np.ascontiguousarray(f), cv2.COLOR_GRAY2BGR) for f in gray]


def _assert_frames(got, want):
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a, b), i


@pytest.mark.gpu
@pytest.mark.parametrize("auto", [False, True])
def test_interpolate_writes_reference_videos(monkeypatch, tmp_path, auto):
    """The file API on 8 frames in batches of 3 pairs (3, 3, 1): vid_orig holds GRAY2BGR(np.load(f)) of every source
    file in order, vid_slomo GRAY2BGR(imread(png, GRAYSCALE)) of the output folder's PNGs in numerical order -- the
    reference's own definitions (slomo.py:471-491, 497-538). A second call appends to the same writers."""
    import cv2
    log = _inject_writer(monkeypatch)
    src, vid = tmp_path / "src", tmp_path / "vid"
    src.mkdir()
    vid.mkdir()
    for i, f in enumerate(_clip(8, 5 if auto else 3)):
        np.save(str(src / ("%08d.npy" % i)), f)
    s = _slomo(auto, video_path=str(vid), vid_orig="video_orig.avi", vid_slomo="video_slomo.avi", avi_frame_rate=25)
    files = sorted(glob.glob(str(src / "*.npy")))
    want_orig, want_slomo, n_times = [], [], 0
    for call in range(2):
        out = tmp_path / ("out%d" % call)
        times, _ = s.interpolate(str(src), str(out), (W, H))
        pngs = sorted(glob.glob(str(out / "*.png")), key=lambda p: int(os.path.basename(p).split(".")[0]))
        assert len(pngs) == len(times)
        want_orig += _bgr(np.load(f) for f in files)
        want_slomo += _bgr(cv2.imread(p, cv2.IMREAD_GRAYSCALE) for p in pngs)
        n_times += len(times)
        assert [(os.path.basename(w.fn), w.h, w.w, w.frame_rate) for w in log] == [
            ("video_orig.avi", H, W, 25), ("video_slomo.avi", H, W, 25)]
        assert all(os.path.dirname(w.fn) == str(vid) for w in log)
        _assert_frames(log[0].frames, want_orig)
        _assert_frames(log[1].frames, want_slomo)
        assert s.numOrigVideoFramesWritten == 8 * (call + 1) and s.numSlomoVideoFramesWritten == n_times
    s.cleanup()
    assert log[0].released and log[1].released


@pytest.mark.gpu
@pytest.mark.parametrize("auto", [False, True])
def test_interpolate_frames_and_pipeline_write_returned_frames(monkeypatch, tmp_path, auto):
    """The in-memory path (frames on the device) and V2EPipeline.run: vid_slomo holds the returned uint8 frames in
    order, vid_orig the frames passed in."""
    from v2e_b200 import EventEmulator, V2EPipeline
    log = _inject_writer(monkeypatch)
    frames = _clip(8, 5 if auto else 3)
    s = _slomo(auto, video_path=str(tmp_path))
    out, times, _ = s.interpolate_frames(torch.from_numpy(frames).cuda())
    assert out.shape[0] == len(times)
    _assert_frames(log[0].frames, _bgr(frames))
    _assert_frames(log[1].frames, _bgr(out.cpu().numpy()))
    assert (s.numOrigVideoFramesWritten, s.numSlomoVideoFramesWritten) == (8, out.shape[0])
    s.cleanup()

    p = _slomo(auto, video_path=str(tmp_path))
    got = []
    run_interp = p.interpolate_frames
    p.interpolate_frames = lambda *a, **k: got.append(run_interp(*a, **k)) or got[-1]
    em = EventEmulator(device="cuda:0", seed=9, rng_mode="device", **_EMU_KW)
    ev, offs, t, nf = V2EPipeline(p, em).run(frames, 0.2)
    assert len(got) == 1 and nf == got[0][0].shape[0] and len(log) == 4
    _assert_frames(log[2].frames, _bgr(frames))
    _assert_frames(log[3].frames, _bgr(got[0][0].cpu().numpy()))
    p.cleanup()
    assert all(w.released for w in log)


@pytest.mark.gpu
@pytest.mark.parametrize("keep", ["vid_orig", "vid_slomo"])
def test_one_video_name_opens_one_writer(monkeypatch, tmp_path, keep):
    log = _inject_writer(monkeypatch)
    frames = _clip(6, 3)
    names = {"vid_orig": None, "vid_slomo": None, keep: keep + ".avi"}
    s = _slomo(video_path=str(tmp_path), **names)
    out, _, _ = s.interpolate_frames(frames)
    assert [os.path.basename(w.fn) for w in log] == [keep + ".avi"]
    assert (s.ori_writer is log[0]) == (keep == "vid_orig") and (s.slomo_writer is log[0]) == (keep == "vid_slomo")
    _assert_frames(log[0].frames, _bgr(frames if keep == "vid_orig" else out.cpu().numpy()))
    s.cleanup()


@pytest.mark.gpu
def test_real_video_writer_round_trip(monkeypatch, tmp_path):
    """Through a real cv2.VideoWriter (MJPG): the files read back with the frame count and size written."""
    cv2 = pytest.importorskip("cv2")
    _inject_writer(monkeypatch, lambda fn, h, w, frame_rate=30:
                   cv2.VideoWriter(fn, cv2.VideoWriter_fourcc(*"MJPG"), frame_rate, (w, h)))
    frames = _clip(6, 3)
    s = _slomo(video_path=str(tmp_path), vid_orig="orig.avi", vid_slomo="slomo.avi")
    out, _, _ = s.interpolate_frames(frames)
    s.cleanup()
    for name, n in (("orig.avi", len(frames)), ("slomo.avi", out.shape[0])):
        cap = cv2.VideoCapture(str(tmp_path / name))
        shapes = []
        while True:
            ok, f = cap.read()
            if not ok:
                break
            shapes.append(f.shape)
        cap.release()
        assert shapes == [(H, W, 3)] * n, name


class _ListHandler(logging.Handler):
    def __init__(self):
        super().__init__(logging.WARNING)
        self.messages = []

    def emit(self, record):
        self.messages.append(record.getMessage())


def _sharded_worker(rank, world, port, q, frames, video_dir):
    import torch.distributed as dist
    from test_sharded_options import _init
    _init(rank, world, port)
    try:
        from v2e_b200 import EventEmulator, V2EPipeline

        def touch(fn, h, w, frame_rate=30):        # a writer that creates its file, as cv2.VideoWriter does
            open(fn, "wb").close()
            return _RecWriter([], fn, h, w, frame_rate)
        sys.modules["v2ecore"], sys.modules["v2ecore.v2e_utils"] = _writer_module(touch)
        rec = _ListHandler()
        logging.getLogger("v2e_b200").addHandler(rec)
        res = []
        for vp in (None, video_dir):
            s = _slomo(video_path=vp)
            em = EventEmulator(device="cuda:0", seed=9, rng_mode="device", shard=(rank, world, None), **_EMU_KW)
            rows, t, nf = V2EPipeline(s, em).run_clip_sharded(frames, 0.2)
            res.append(dict(rows=rows, t=t, nf=nf, n=(s.numOrigVideoFramesWritten, s.numSlomoVideoFramesWritten),
                            open=(s.ori_writer, s.slomo_writer) != (None, None)))
            s.cleanup()
        q.put((rank, dict(res=res, warnings=rec.messages)))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_sharded_clip_writes_no_video(tmp_path):
    """run_clip_sharded over two gloo ranks on the one GPU with video_path set: every rank holds only its own frame
    pairs, so no writer is opened and no file is made; rank 0 warns once; the events are those of the run without
    video_path."""
    from helpers import canonical
    from test_sharded_options import _spawn
    frames = _clip(7, 3)
    res = _spawn(2, _sharded_worker, frames, str(tmp_path))
    assert os.listdir(tmp_path) == []
    warned = [[m for m in res[r]["warnings"] if "video_path ignored" in m] for r in (0, 1)]
    assert [len(w) for w in warned] == [1, 0]
    for r in (0, 1):
        plain, video = res[r]["res"]
        assert video["n"] == (0, 0) and not video["open"]
        assert plain["nf"] == video["nf"] == 18 and np.array_equal(plain["t"], video["t"])
        assert np.array_equal(canonical(plain["rows"]), canonical(video["rows"])), r
    assert sum(len(res[r]["res"][0]["rows"]) for r in (0, 1)) > 0
