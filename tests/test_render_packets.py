"""The DVS frame renderer on the packets v2e feeds it, with the DVS video open: the float64 frames, the uint8 BGR frames
handed to the video writer and the frame-times file (v2ecore/renderer.py:161-366).

CPU: the numpy oracle against every case of tests/golden/render_ref.npz (oracle/make_golden_render.py ran the
unmodified class with a recording video writer); each case's edge is checked to occur in its packets. The renderer's
constructor refuses exposures that would never finish a frame.
GPU: v2e_b200.renderer.EventRenderer against the same fixtures with a video open (a stub v2ecore.v2e_utils records
what it writes); against the oracle on the pixel model's own rows (device RNG, v2e's CLI defaults, 346x260 and
1280x720, packets formed as v2e.py:590-606 forms them, fed as numpy arrays and as CUDA tensors), also with the rows
shifted to long-clip times; a 10^6-row packet at a full scale no count reaches, where every frame must be the exact
ON - OFF count; and a DURATION packet longer than the boundary table."""
import os
import sys
import types

import numpy as np
import pytest

from helpers import GOLDEN_DIR
from render_oracle import AREA_COUNT, COUNT, DURATION, SOURCE, RenderOracle, frame_times_text, video_frames
from test_render import _golden

DVS_VID = "dvs-video.avi"
BATCH_SIZE = 8                      # v2e's --batch_size default: frames of events per rendered packet


def _cases():
    z = np.load(os.path.join(GOLDEN_DIR, "render_ref.npz"))
    for name, mode, value, H, W, fs, area, pk in _golden():
        yield dict(name=name, mode=mode, value=value, H=H, W=W, fs=fs, area=area, packets=pk,
                   video=z[name + "_vid"], times=str(z[name + "_times"]))


CASES = {c["name"]: c for c in _cases()}


def boundary_ties(packets, interval):
    """Rows whose time equals a DURATION frame boundary after the first: the reference's frame start times are the
    first row's float32 time plus k intervals, accumulated in float32 (renderer.py:208, 316)."""
    ts = np.concatenate([p[:, 0] for p in packets])
    c, bounds = ts[0] + interval, []
    while c <= ts[-1]:
        bounds.append(c)
        c = c + interval
    return int(np.isin(ts, np.array(bounds, np.float32)).sum())


def clipped(frames):
    """Pixels at +-full scale: 0.0 or 1.0 in a normalised frame."""
    return int(sum(((f == 0.0) | (f == 1.0)).sum() for f in frames if len(f)))


def run_oracle(case):
    o = RenderOracle(case["fs"], case["mode"], case["value"], case["area"])
    frames = []
    for ev, _ in case["packets"]:
        got = o.render(ev, case["H"], case["W"])
        frames.append(np.zeros((0, case["H"], case["W"])) if got is None else got)
    return o, frames


# ---- CPU: the oracle against the reference's output -----------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_video_and_frame_times(name):
    c = CASES[name]
    o, frames = run_oracle(c)
    for (ev, want), got in zip(c["packets"], frames):
        assert got.dtype == np.float64 and got.shape == want.shape and np.array_equal(got, want)
    allf = np.concatenate(frames)
    assert len(allf) > 0
    vid = video_frames(allf, c["H"], c["W"])
    assert c["video"].dtype == np.uint8 and c["video"].shape == vid.shape and np.array_equal(vid, c["video"])
    assert frame_times_text(DVS_VID, o.times) == c["times"]
    assert len(c["times"].splitlines()) == 2 + len(allf)


def test_fixture_cases_reach_their_edges():
    """Each case's packets hold the input it is there for."""
    g = {n: (c, run_oracle(c)) for n, c in CASES.items()}
    for n in ("v2e_default", "v2e_default_t2147"):
        c, _ = g[n]
        assert c["mode"] == DURATION and c["value"] == 0.01 and c["fs"] == 2
        assert boundary_ties([ev for ev, _ in c["packets"]], c["value"]) >= 20, n
        assert clipped([f for _, f in c["packets"]]) > 0, n
    for n in ("duration_gaps", "duration_tiny", "source_tiny"):
        c, (o, _) = g[n]
        assert sum(1 for s, e in o.slices if e == s) >= (1 if n == "source_tiny" else 10), n
    sizes = [len(ev) for ev, _ in g["duration_tiny"][0]["packets"]]
    assert 1 in sizes and 2 in sizes
    assert any(len(fr) for ev, fr in g["duration_tiny"][0]["packets"] if len(ev) == 2)   # empty frames from 2 rows
    c, _ = g["count_short"]
    short = [len(fr) for ev, fr in c["packets"] if len(ev) <= c["value"] + 1]
    assert len(short) >= 5 and not any(short) and sum(len(fr) for _, fr in c["packets"]) > 0
    c, (o, _) = g["area_ragged"]
    d = c["area"]
    assert c["W"] % d and c["H"] % d
    ev = np.concatenate([ev for ev, _ in c["packets"]])
    assert ((ev[:, 1] >= c["W"] // d * d) & (ev[:, 2] >= c["H"] // d * d)).sum() > 50
    assert sum(len(fr) for ev, fr in c["packets"][:1]) == 0 < len(c["packets"][1][1])     # counts carried over
    for a in (2, 3, 10):
        c, (o, _) = g["area_one_cell_%d" % a]
        ev, fr = c["packets"][0]
        cells = np.unique(ev[:, 1:3] // c["area"], axis=0)
        assert len(cells) == 1
        assert len(fr) > len(ev) // a + 2                 # more frames than a slice table of n // area_count + 2
        assert all(e - s == a - 1 for s, e in o.slices[1:len(fr)])
    for n in ("source", "source_tiny"):
        assert g[n][0]["mode"] == SOURCE
    c, _ = g["duration_noclip"]
    frames = np.concatenate([fr for _, fr in c["packets"]])
    counts = frames * (2 * c["fs"]) - c["fs"]
    assert clipped(frames) == 0 and np.abs(counts).max() > 5


def test_constructor_refuses_exposures_that_never_finish_a_frame():
    """COUNT with fewer than 1 event per frame and AREA_COUNT with area_count 1 would loop forever: each frame would
    end where it starts."""
    from v2e_b200.renderer import EventRenderer, ExposureMode
    for v in (0, 0.5, 0.999, -3):
        with pytest.raises(ValueError):
            EventRenderer(exposure_mode=ExposureMode.COUNT, exposure_value=v)
    for v in (1, 1.5, 0, -2):
        with pytest.raises(ValueError):
            EventRenderer(exposure_mode=ExposureMode.AREA_COUNT, exposure_value=v, area_dimension=8)


# ---- GPU: EventRenderer with the DVS video open ---------------------------------------------------------------------
class Recorder:
    """Stands in for the cv2.VideoWriter v2ecore.v2e_utils.video_writer opens."""

    def __init__(self, path, height, width, frame_rate):
        self.path, self.height, self.width, self.frame_rate = path, height, width, frame_rate
        self.frames = []
        self.released = False

    def write(self, frame):
        self.frames.append(np.array(frame, copy=True))

    def release(self):
        self.released = True


@pytest.fixture
def video(monkeypatch):
    """A stub v2ecore package whose v2e_utils has the two functions the renderer takes from it; it replaces any
    v2ecore imported earlier. Returns the list of recorders it opened."""
    opened = []

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
    monkeypatch.setitem(sys.modules, "v2ecore", pkg)
    monkeypatch.setitem(sys.modules, "v2ecore.v2e_utils", utils)
    return opened


def render_with_video(packets, H, W, fs, mode, value, area, out_dir, opened, as_tensor=False):
    """Every packet through one EventRenderer with a DVS video open: (float64 frames per packet, the uint8 frames
    written, the frame-times file's text)."""
    import torch
    from v2e_b200.renderer import EventRenderer, ExposureMode
    r = EventRenderer(full_scale_count=fs, output_path=str(out_dir), dvs_vid=DVS_VID,
                      exposure_mode=ExposureMode(mode), exposure_value=value, area_dimension=area)
    n0 = len(opened)
    frames = []
    for ev in packets:
        if as_tensor:
            got = r.render_events_to_frames(torch.from_numpy(ev).cuda(), H, W, return_device=True)
            got = None if got is None else got.cpu().numpy()
        else:
            got = r.render_events_to_frames(ev, H, W, return_frames=True)
        frames.append(np.zeros((0, H, W)) if got is None else got)
    r.cleanup()
    assert len(opened) == n0 + 1
    rec = opened[-1]
    assert rec.released and rec.path == os.path.join(str(out_dir), DVS_VID) and (rec.height, rec.width) == (H, W)
    with open(os.path.join(str(out_dir), "dvs-video-frame_times.txt"), "rb") as f:
        text = f.read().decode()
    vid = np.stack(rec.frames) if rec.frames else np.zeros((0, H, W, 3), np.uint8)
    return frames, vid, text


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_cuda_renderer_writes_the_reference_video_and_frame_times(name, video, tmp_path):
    c = CASES[name]
    frames, vid, text = render_with_video([ev for ev, _ in c["packets"]], c["H"], c["W"], c["fs"], c["mode"],
                                          c["value"], c["area"], tmp_path, video)
    for (_, want), got in zip(c["packets"], frames):
        assert got.dtype == np.float64 and got.shape == want.shape and np.array_equal(got, want)
    assert vid.dtype == np.uint8 and vid.shape == c["video"].shape and np.array_equal(vid, c["video"])
    assert text == c["times"]


# ---- GPU: the pixel model's rows ------------------------------------------------------------------------------------
CLI_DEFAULTS = dict(pos_thres=0.2, neg_thres=0.2, sigma_thres=0.03, cutoff_hz=300.0, leak_rate_hz=0.01,
                    shot_noise_rate_hz=0.001, refractory_period_s=0.0005)          # v2e_args.py:150-204
SIZES = {"346x260": (260, 346), "1280x720": (720, 1280)}
FRAME_DT = 0.005                    # two source frames per 0.01 s DURATION frame
N_FRAMES = 4 * BATCH_SIZE + 4       # four full packets and a leftover one
T0S = [0.0, 2147.47, 36000.0]


def pixel_model_packets(H, W):
    """Rows of EventEmulator (device RNG, CLI defaults) on a textured clip, appended frame by frame and cut every
    BATCH_SIZE frames as v2e.py:590-606 does, the leftover packet last. After the first frame with events every other
    frame time is put on a 0.01 s frame boundary (the first row's float32 time plus k intervals, accumulated in float32):
    the rows of that frame's last iteration carry that time."""
    from test_emulator_device_rng import texture_frames
    from v2e_b200 import EventEmulator
    em = EventEmulator(device="cuda", rng_mode="device", seed=7, row_order="canonical", **CLI_DEFAULTS)
    fr = texture_frames(H, W, N_FRAMES, seed=3, speed=1.0, block=8) // 2 + 64
    packets, events = [], np.zeros((0, 4), np.float32)
    t, bound = 0.0, None
    for i in range(1, N_FRAMES + 1):
        if bound is None:
            t = (i - 1) * FRAME_DT
        elif i % 2:
            while float(bound) <= t + FRAME_DT / 4:
                bound = bound + 0.01                      # float32 + Python float: float32, as the renderer adds
            t = float(bound)
        else:
            t = t + FRAME_DT
        new = em.generate_events(fr[i - 1], t)
        if new is not None and new.shape[0] > 0:
            if bound is None:
                bound = new[0, 0]
            events = np.append(events, new, axis=0)
            if i % BATCH_SIZE == 0:
                packets.append(events)
                events = np.zeros((0, 4), np.float32)
    if len(events) > 0:
        packets.append(events)
    assert len(packets) == N_FRAMES // BATCH_SIZE + 1
    for p in packets:
        assert p.dtype == np.float32 and np.all(np.diff(p[:, 0]) >= 0)
    return packets


@pytest.fixture(scope="module")
def model_rows():
    cache = {}

    def get(size):
        if size not in cache:
            cache[size] = pixel_model_packets(*SIZES[size])
        return cache[size]
    return get


def shifted(packets, t0):
    """The rows at t0 + t, rounded to float32 as the pixel model's timestamps are."""
    out = []
    for p in packets:
        q = p.copy()
        q[:, 0] = (p[:, 0].astype(np.float64) + t0).astype(np.float32)
        out.append(q)
    return out


def exposures(size):
    """(mode, value, area_dimension) per mode, v2e's --dvs_exposure forms; counts scaled to the frame size."""
    big = size == "1280x720"
    return {DURATION: (0.01, None), COUNT: (200000 if big else 20000, None), AREA_COUNT: (1000 if big else 500, 64),
            SOURCE: (0, None)}


PM_CASES = [(s, m, t0) for s in SIZES for m in (DURATION, COUNT, AREA_COUNT, SOURCE)
            for t0 in (T0S if m in (DURATION, COUNT) else T0S[:1])]


@pytest.mark.gpu
@pytest.mark.parametrize("size,mode,t0", PM_CASES, ids=["%s-%d-%g" % c for c in PM_CASES])
def test_cuda_renderer_matches_oracle_on_pixel_model_rows(size, mode, t0, model_rows, video, tmp_path):
    H, W = SIZES[size]
    packets = shifted(model_rows(size), t0)
    value, area = exposures(size)[mode]
    fs = 2
    o = RenderOracle(fs, mode, value, area)
    want = []
    for p in packets:
        f = o.render(p, H, W)
        want.append(np.zeros((0, H, W)) if f is None else f)
    allw = np.concatenate(want)
    assert len(allw) >= 5
    assert clipped(allw) > 0
    ties = boundary_ties(packets, 0.01)
    if mode == DURATION:
        assert ties > 0
    print("render %s mode %d T0 %g: rows per packet %s, rows tied with a 0.01 s boundary %d, frames %d"
          % (size, mode, t0, [len(p) for p in packets], ties, len(allw)))
    for as_tensor in (False, True):
        d = tmp_path / ("tensor" if as_tensor else "numpy")
        d.mkdir()
        frames, vid, text = render_with_video(packets, H, W, fs, mode, value, area, d, video, as_tensor=as_tensor)
        for w, g in zip(want, frames):
            assert g.dtype == np.float64 and g.shape == w.shape and np.array_equal(g, w), as_tensor
        assert np.array_equal(vid, video_frames(allw, H, W)), as_tensor
        assert text == frame_times_text(DVS_VID, o.times), as_tensor


# ---- GPU: the atomics, with nothing clipped -------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [DURATION, SOURCE])
def test_cuda_renderer_counts_exactly_when_nothing_clips(mode, video, tmp_path):
    """10^6 rows, 80 % of them on four pixels: one all ON, one alternating ON / OFF (the counts cancel), one two ON to
    one OFF, one mostly OFF. At a full scale above every count each float64 frame is (ON - OFF + fs) / (2 fs) of its
    rows, counted here with np.add.at: a lost or doubled atomic add shows."""
    H, W, n, fs = 260, 346, 1_000_000, 1 << 21
    rng = np.random.default_rng(11)
    ts = np.sort(rng.uniform(0, 0.05, n)).astype(np.float32)
    x, y = rng.integers(0, W, n), rng.integers(0, H, n)
    p = np.where(rng.random(n) < 0.5, 1.0, -1.0)
    which = rng.integers(0, 10, n)
    hot = [(17, 3, lambda k: np.ones(k)), (345, 259, lambda k: np.where(np.arange(k) % 2, 1.0, -1.0)),
           (0, 0, lambda k: np.where(np.arange(k) % 3 == 2, -1.0, 1.0)), (200, 100, lambda k: np.where(np.arange(k) % 8, -1.0, 1.0))]
    for j, (hx, hy, pol) in enumerate(hot):
        m = (which == 2 * j) | (which == 2 * j + 1)
        x[m], y[m] = hx, hy
        p[m] = pol(m.sum())
    ev = np.stack([ts, x, y, p], 1).astype(np.float32)
    value = 0.01 if mode == DURATION else 0
    o = RenderOracle(fs, mode, value)
    want = o.render(ev, H, W)
    assert want is not None and len(want) >= (4 if mode == DURATION else 1)
    exact = []
    for s, e in o.slices:
        cnt = np.zeros((H, W), np.int64)
        np.add.at(cnt, (ev[s:e, 2].astype(np.int64), ev[s:e, 1].astype(np.int64)), np.where(ev[s:e, 3] == 1, 1, -1))
        assert np.abs(cnt).max() > 1000 and np.abs(cnt).max() < fs
        exact.append((cnt + fs) / float(2 * fs))
    assert np.array_equal(np.stack(exact), want)
    frames, vid, text = render_with_video([ev], H, W, fs, mode, value, None, tmp_path, video, as_tensor=True)
    assert np.array_equal(frames[0], np.stack(exact))
    assert np.array_equal(vid, video_frames(want, H, W))
    assert text == frame_times_text(DVS_VID, o.times)


# ---- GPU: the DURATION boundary table ------------------------------------------------------------------------------
@pytest.mark.gpu
def test_duration_packet_past_the_boundary_table_is_refused():
    """Three rows 2.2 s apart at 1 us exposure span more than 2^20 frame intervals: refused, not cut short."""
    from v2e_b200.renderer import EventRenderer, ExposureMode
    ev = np.array([[0.5, 1, 1, 1], [1.0, 2, 2, -1], [2.7, 3, 3, 1]], np.float32)
    assert (ev[-1, 0] - ev[0, 0]) / 1e-6 > 1 << 21
    r = EventRenderer(full_scale_count=2, exposure_mode=ExposureMode.DURATION, exposure_value=1e-6)
    with pytest.raises(ValueError):
        r.render_events_to_frames(ev, 8, 8, return_frames=True)


@pytest.mark.gpu
def test_duration_packet_finishing_more_frames_than_a_grid_dimension():
    """A packet 70 s long at 1 ms exposure finishes more than 65 535 frames (the most one grid dimension holds): all of
    them are rendered, the empty ones and the few with rows, as the oracle renders them."""
    from v2e_b200.renderer import EventRenderer, ExposureMode
    ev = np.array([[0.0, 1, 2, 1], [0.0004, 1, 2, 1], [30.0, 3, 0, -1], [30.0003, 3, 0, 1], [30.0004, 3, 0, 1],
                   [68.5005, 0, 3, 1], [68.5006, 0, 3, 1], [70.2, 2, 2, -1]], np.float32)
    o = RenderOracle(2, DURATION, 0.001)
    want = o.render(ev, 4, 4)
    assert len(want) > 65535 and sum(1 for s, e in o.slices if e > s) >= 3
    r = EventRenderer(full_scale_count=2, exposure_mode=ExposureMode.DURATION, exposure_value=0.001)
    got = r.render_events_to_frames(ev, 4, 4, return_frames=True)
    assert got.shape == want.shape and np.array_equal(got, want)
