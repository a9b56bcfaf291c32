"""The greyscale Motion-JPEG video writer (v2e_b200.video, csrc/mjpeg.cu) and its numpy oracle (oracle/mjpeg_oracle.py).

CPU: the oracle's constants and marker structure; its JPEGs decoded by libjpeg-turbo (cv2.imdecode) and by Pillow at
sizes 1x1 .. 1280x720, qualities 50 / 95 / 100, random, smooth and DVS-like frames, within error bounds measured on the
oracle (constant frames exactly); the AVI container read back through cv2.VideoCapture, in one RIFF and in several
AVIX segments; the writer's refusals; the BGR -> luma rule.
GPU: the CUDA encoder's bytes equal the oracle's for every case, a batch equals its single-frame calls; EventRenderer,
SuperSloMo (interpolate_frames and interpolate) and a two-rank sharded run write, through MjpegWriter, the oracle's
encoding of exactly the frames the default path hands its video writer."""
import io
import os
import struct
import sys
import types

import numpy as np
import pytest

import mjpeg_oracle as mo

SIZES = [(1, 1), (8, 8), (9, 17), (37, 53), (260, 346), (720, 1280)]
QUALITIES = [50, 95, 100]
KINDS = ["random", "smooth", "dvs", "constant"]
# largest |decoded - frame| and mean over frames of at least 1000 pixels, measured on the oracle's JPEGs (cv2 and
# Pillow decode them alike); for comparison Pillow's own q95 encoder gives 9 and 1.3 on the 346x260 DVS-like frame
BOUNDS = {(50, "random"): (94, 14.6), (50, "smooth"): (6, 1.05), (50, "dvs"): (99, 9.93),
          (95, "random"): (10, 1.53), (95, "smooth"): (2, 0.18), (95, "dvs"): (9, 1.28),
          (100, "random"): (1, 0.1), (100, "smooth"): (1, 0.07), (100, "dvs"): (1, 0.07)}


def make_frame(kind, H, W, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, (H, W), dtype=np.uint8)
    if kind == "smooth":
        yy, xx = np.mgrid[0:H, 0:W]
        return (127 + 100 * np.sin(xx / 17.0) * np.cos(yy / 23.0)).astype(np.uint8)
    if kind == "dvs":                                   # v2e's DVS frames: a grey 127 field with 0 / 255 dots
        f = np.full((H, W), 127, np.uint8)
        m = rng.random((H, W)) < 0.03
        f[m] = rng.choice([0, 255], int(m.sum())).astype(np.uint8)
        return f
    return np.full((H, W), 200, np.uint8)


def markers(jpg):
    """[(marker, segment body)] up to SOS, then the scan's RSTn / EOI markers in order."""
    out, k = [], 2
    assert jpg[:2] == b"\xff\xd8"
    while True:
        m, n = jpg[k + 1], int.from_bytes(jpg[k + 2:k + 4], "big")
        out.append((m, jpg[k + 4:k + 2 + n]))
        k += 2 + n
        if m == 0xDA:
            break
    scan = np.frombuffer(jpg[k:], np.uint8)
    ff = np.nonzero(scan[:-1] == 0xFF)[0]
    out += [(int(scan[i + 1]), b"") for i in ff if scan[i + 1] != 0]
    return out


def avi_jpegs(path):
    """The '00dc' chunks of every movi list of an AVI file, in file order."""
    data = open(path, "rb").read()
    out, k = [], 0
    while k < len(data):
        assert data[k:k + 4] == b"RIFF"
        end = k + 8 + struct.unpack("<I", data[k + 4:k + 8])[0]
        j = k + 12
        while j < end:
            tag, n = data[j:j + 4], struct.unpack("<I", data[j + 4:j + 8])[0]
            if tag == b"LIST" and data[j + 8:j + 12] == b"movi":
                i = j + 12
                while i < j + 8 + n:
                    t, m = data[i:i + 4], struct.unpack("<I", data[i + 4:i + 8])[0]
                    if t == b"00dc":
                        out.append(data[i + 8:i + 8 + m])
                    i += 8 + m + m % 2
            j += 8 + n + n % 2
        k = end + (end % 2)
    return out


# ---- CPU: the oracle ------------------------------------------------------------------------------------------------
def test_constants():
    assert np.array_equal(mo.DCT_MATRIX, mo.dct_matrix())
    assert sorted(mo.ZIGZAG.tolist()) == list(range(64))
    assert mo.ZIGZAG[:10].tolist() == [0, 1, 8, 16, 9, 2, 3, 10, 17, 24]
    assert sum(mo.AC_BITS) == len(mo.AC_VALS) == 162 and sum(mo.DC_BITS) == len(mo.DC_VALS) == 12
    assert mo.quant_table(100).tolist() == [1] * 64 and np.array_equal(mo.quant_table(50), mo.K1_LUMA)
    for q in (0, 101):
        with pytest.raises(ValueError):
            mo.quant_table(q)


@pytest.mark.parametrize("H,W", SIZES)
def test_marker_structure(H, W):
    jpg = mo.encode(make_frame("dvs", H, W), 95)
    ms = markers(jpg)
    names = [m for m, _ in ms]
    assert names[:7] == [0xE0, 0xDB, 0xC0, 0xC4, 0xC4, 0xDD, 0xDA]
    sof = dict(ms)[0xC0]
    assert int.from_bytes(sof[1:3], "big") == H and int.from_bytes(sof[3:5], "big") == W
    assert sof[5] == 1 and sof[7] == 0x11
    assert int.from_bytes(dict(ms)[0xDD], "big") == -(-W // 8)
    rst = [m for m in names[7:] if 0xD0 <= m <= 0xD7]
    assert rst == [0xD0 + (i & 7) for i in range(-(-H // 8) - 1)]
    assert names[7:].count(0xD9) == 1 and names[-1] == 0xD9 and jpg.endswith(b"\xff\xd9")


@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("quality", QUALITIES)
def test_independent_decoders(H, W, quality):
    import cv2
    from PIL import Image
    for kind in KINDS:
        f = make_frame(kind, H, W, seed=H + W)
        jpg = mo.encode(f, quality)
        a = cv2.imdecode(np.frombuffer(jpg, np.uint8), cv2.IMREAD_UNCHANGED)
        b = np.asarray(Image.open(io.BytesIO(jpg)))
        for d in (a, b):
            assert d.shape == (H, W) and d.dtype == np.uint8
            e = np.abs(d.astype(np.int64) - f)
            if kind == "constant":
                assert e.max() == 0
                continue
            top, mean = BOUNDS[(quality, kind)]
            assert e.max() <= top, (kind, e.max())
            if H * W >= 1000:
                assert e.mean() <= mean, (kind, e.mean())


def test_luma_rule():
    import cv2
    import torch
    from v2e_b200.video import bgr_to_luma
    g = make_frame("random", 37, 53)
    assert np.array_equal(mo.luma(cv2.cvtColor(g, cv2.COLOR_GRAY2BGR)), g)
    bgr = np.random.default_rng(1).integers(0, 256, (37, 53, 3), dtype=np.uint8)
    assert np.array_equal(bgr_to_luma(torch.from_numpy(bgr)).numpy(), mo.luma(bgr))
    assert np.abs(mo.luma(bgr).astype(int) - cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY)).max() <= 1


# ---- CPU: the container ---------------------------------------------------------------------------------------------
def _read_back(path, jpgs, H, W, fps):
    import cv2
    cap = cv2.VideoCapture(str(path))
    assert cap.isOpened()
    assert cap.get(cv2.CAP_PROP_FPS) == fps and cap.get(cv2.CAP_PROP_FRAME_COUNT) == len(jpgs)
    n = 0
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        want = cv2.imdecode(np.frombuffer(jpgs[n], np.uint8), cv2.IMREAD_GRAYSCALE)
        assert fr.shape == (H, W, 3)
        assert np.array_equal(fr[..., 0], fr[..., 1]) and np.array_equal(fr[..., 0], fr[..., 2])
        # FFmpeg's MJPEG decoder and libjpeg-turbo round their IDCTs differently: at most 1 apart
        assert np.abs(fr[..., 0].astype(int) - want).max() <= 1, n
        n += 1
    assert n == len(jpgs)


def test_container_reads_back(tmp_path, monkeypatch):
    from v2e_b200 import video
    H, W = 37, 53
    jpgs = [mo.encode(make_frame("random", H, W, seed=s), 95) for s in range(13)]
    a = video.AviWriter(str(tmp_path / "one.avi"), W, H, 25)
    for j in jpgs:
        a.add(j)
    a.close()
    data = open(tmp_path / "one.avi", "rb").read()
    assert data.count(b"AVIX") == 0 and avi_jpegs(tmp_path / "one.avi") == jpgs
    _read_back(tmp_path / "one.avi", jpgs, H, W, 25)
    # several OpenDML segments: each RIFF holds about three frames
    monkeypatch.setattr(video, "RIFF_LIMIT", 3 * len(jpgs[0]) + 2000)
    a = video.AviWriter(str(tmp_path / "segs.avi"), W, H, 25)
    for j in jpgs:
        a.add(j)
    a.close()
    data = open(tmp_path / "segs.avi", "rb").read()
    assert data.count(b"AVIX") >= 3 and data.count(b"ix00") == data.count(b"AVIX") + 1
    assert avi_jpegs(tmp_path / "segs.avi") == jpgs
    _read_back(tmp_path / "segs.avi", jpgs, H, W, 25)


def test_writer_refuses_bad_frames(tmp_path):
    import torch
    from v2e_b200 import MjpegWriter
    w = MjpegWriter(str(tmp_path / "v.avi"), 16, 24)
    assert w.isOpened()
    for bad in (np.zeros((16, 25), np.uint8), np.zeros((16, 24), np.float32), np.zeros((16, 24, 4), np.uint8),
                torch.zeros((16, 24), dtype=torch.int16)):
        with pytest.raises(ValueError):
            w.write(bad)
    with pytest.raises(ValueError):
        w.write_frames(np.zeros((2, 16, 23), np.uint8))
    w.release()
    assert not w.isOpened()
    for q in (0, 101):
        with pytest.raises(ValueError):
            MjpegWriter(str(tmp_path / "q.avi"), 16, 24, quality=q)


# ---- GPU: the encoder -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("H,W", SIZES)
def test_encoder_bit_exact(H, W, tmp_path):
    import torch
    from v2e_b200 import MjpegWriter
    for quality in QUALITIES:
        w = MjpegWriter(str(tmp_path / "v.avi"), H, W, quality=quality)
        frames = np.stack([make_frame(k, H, W, seed=H + W) for k in KINDS])
        want = [mo.encode(f, quality) for f in frames]
        for f, jw in zip(frames, want):
            data, sizes = w.encode(torch.from_numpy(f[None]).cuda())
            assert len(sizes) == 1 and data.numpy().tobytes() == jw, (quality, H, W)
        data, sizes = w.encode(torch.from_numpy(frames).cuda())
        assert sizes.tolist() == [len(j) for j in want] and data.numpy().tobytes() == b"".join(want)
        w.release()


@pytest.mark.gpu
def test_writer_file_is_the_oracles(tmp_path):
    """write_frames and write (grey and GRAY2BGR, host and device) in one file: every chunk is the oracle's JPEG."""
    import cv2
    import torch
    from v2e_b200 import MjpegWriter
    H, W = 260, 346
    frames = np.stack([make_frame(k, H, W, seed=s) for s in range(3) for k in KINDS])
    w = MjpegWriter(str(tmp_path / "v.avi"), H, W, frame_rate=30)
    w.write_frames(torch.from_numpy(frames[:5]).cuda())
    w.write(frames[5])
    w.write(cv2.cvtColor(frames[6], cv2.COLOR_GRAY2BGR))
    w.write(torch.from_numpy(cv2.cvtColor(frames[7], cv2.COLOR_GRAY2BGR)).cuda())
    w.write_frames(frames[8:])
    w.release()
    got = avi_jpegs(tmp_path / "v.avi")
    assert got == [mo.encode(f, 95) for f in frames]
    _read_back(tmp_path / "v.avi", got, H, W, 30)


# ---- GPU: the renderer, SuperSloMo and a sharded clip ---------------------------------------------------------------
def _recorded_to_oracle(frames_bgr):
    out = []
    for f in frames_bgr:
        assert np.array_equal(f[..., 0], f[..., 1]) and np.array_equal(f[..., 0], f[..., 2])
        out.append(mo.encode(f[..., 0], 95))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("seg", [None, 3])
def test_renderer_writes_the_default_paths_frames(seg, tmp_path, monkeypatch):
    from test_pipeline_segments import _clip, _emulator, _slomo
    from test_render_packets import CLI_DEFAULTS, DVS_VID, Recorder
    from v2e_b200 import MjpegWriter, V2EPipeline
    from v2e_b200.renderer import EventRenderer, ExposureMode
    opened = []
    pkg, utils = types.ModuleType("v2ecore"), types.ModuleType("v2ecore.v2e_utils")
    pkg.__path__ = []
    utils.checkAddSuffix = lambda p, s: p if p.endswith(s) else os.path.splitext(p)[0] + s
    utils.video_writer = lambda p, h, w, frame_rate=30, fourcc=None: opened.append(Recorder(p, h, w, frame_rate)) \
        or opened[-1]
    pkg.v2e_utils = utils
    monkeypatch.setitem(sys.modules, "v2ecore", pkg)
    monkeypatch.setitem(sys.modules, "v2ecore.v2e_utils", utils)
    H, W = 64, 96
    frames = _clip(14, H, W, [3] * 13, seed=2)
    sl = _slomo(False)
    texts, files = [], []
    for kind in ("default", "mjpeg"):
        d = tmp_path / kind
        d.mkdir()
        r = EventRenderer(full_scale_count=2, output_path=str(d), dvs_vid=DVS_VID, exposure_mode=ExposureMode.DURATION,
                          exposure_value=0.01, video_writer=MjpegWriter if kind == "mjpeg" else None)
        for _ in V2EPipeline(sl, _emulator(row_order="canonical", **CLI_DEFAULTS), renderer=r).run_segments(
                lambda a, b: frames[a:b], len(frames), 0.2, segment_pairs=seg):
            pass
        r.cleanup()
        texts.append(open(d / "dvs-video-frame_times.txt", "rb").read())
        files.append(d / "dvs-video.avi")
    sl.cleanup()
    assert len(opened) == 1 and len(opened[0].frames) >= 5
    assert texts[0] == texts[1]
    assert avi_jpegs(files[1]) == _recorded_to_oracle(opened[0].frames)


@pytest.mark.gpu
@pytest.mark.parametrize("auto", [False, True])
def test_slomo_writes_the_default_paths_frames(auto, tmp_path, monkeypatch):
    from test_slomo_video import _clip, _inject_writer, _slomo
    from v2e_b200 import MjpegWriter
    log = _inject_writer(monkeypatch)
    clip = _clip(8, 5 if auto else 3)
    src = tmp_path / "src"
    src.mkdir()
    for i, f in enumerate(clip):
        np.save(str(src / ("%08d.npy" % i)), f)
    H, W = clip.shape[1:]
    for api in ("frames", "files"):
        got = {}
        for kind in ("default", "mjpeg"):
            vid = tmp_path / ("%s_%s" % (api, kind))
            vid.mkdir()
            s = _slomo(auto, video_path=str(vid), video_writer=MjpegWriter if kind == "mjpeg" else None)
            for call in range(2):
                if api == "frames":
                    s.interpolate_frames(clip)
                else:
                    s.interpolate(str(src), str(tmp_path / ("out_%s_%s_%d" % (api, kind, call))), (W, H))
            got[kind] = (s.numOrigVideoFramesWritten, s.numSlomoVideoFramesWritten)
            s.cleanup()
        rec_orig, rec_slomo = log[-2], log[-1]
        assert got["mjpeg"] == got["default"] == (len(rec_orig.frames), len(rec_slomo.frames))
        vid = tmp_path / ("%s_mjpeg" % api)
        assert avi_jpegs(vid / "original.avi") == _recorded_to_oracle(rec_orig.frames)
        assert avi_jpegs(vid / "slomo.avi") == _recorded_to_oracle(rec_slomo.frames)


def _sharded_worker(rank, world, port, q, frames, out):
    import torch.distributed as dist
    from test_pipeline_segments_sharded import _FILES_KW, _init, _slomo
    _init(rank, world, port)
    try:
        from v2e_b200 import EventEmulator, MjpegWriter, V2EPipeline
        from v2e_b200.renderer import EventRenderer, ExposureMode
        sl = _slomo(False, 3)
        em = EventEmulator(device="cuda:0", seed=9, shard=(rank, world, None), **_FILES_KW)
        r = None
        if rank == 0:
            os.makedirs(out)
            r = EventRenderer(full_scale_count=2, output_path=out, dvs_vid="dvs-video.avi",
                              exposure_mode=ExposureMode.DURATION, exposure_value=0.01, video_writer=MjpegWriter)
        for _ in V2EPipeline(sl, em, renderer=r).run_segments_sharded(
                lambda a, b: frames[a:b], len(frames), 0.2, t_offset=0.5, segment_pairs=3, write_sinks=True):
            pass
        if r is not None:
            r.cleanup()
        em.cleanup()
        sl.cleanup()
        q.put((rank, None))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_sharded_dvs_avi_equals_one_gpus(tmp_path):
    from test_pipeline_segments import _clip, _slomo
    from test_pipeline_segments_sharded import _FILES_KW, _spawn
    from v2e_b200 import EventEmulator, MjpegWriter, V2EPipeline
    from v2e_b200.renderer import EventRenderer, ExposureMode
    frames = _clip(14, 64, 96, [3] * 13, seed=2)
    res = _spawn(2, _sharded_worker, frames, str(tmp_path / "sharded"))
    assert res == {0: None, 1: None}
    d = tmp_path / "one"
    d.mkdir()
    r = EventRenderer(full_scale_count=2, output_path=str(d), dvs_vid="dvs-video.avi",
                      exposure_mode=ExposureMode.DURATION, exposure_value=0.01, video_writer=MjpegWriter)
    sl = _slomo(False)
    for _ in V2EPipeline(sl, EventEmulator(device="cuda:0", seed=9, **_FILES_KW), renderer=r).run_segments(
            lambda a, b: frames[a:b], len(frames), 0.2, t_offset=0.5, segment_pairs=3):
        pass
    r.cleanup()
    sl.cleanup()
    one = open(d / "dvs-video.avi", "rb").read()
    assert len(avi_jpegs(d / "dvs-video.avi")) >= 5
    assert open(tmp_path / "sharded" / "dvs-video.avi", "rb").read() == one
    assert open(tmp_path / "sharded" / "dvs-video-frame_times.txt").read() == \
        open(d / "dvs-video-frame_times.txt").read()
