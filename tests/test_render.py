"""DVS frame rendering (v2ecore/renderer.py:161-430; SURVEY.md 8f rank 4). CPU: the numpy oracle against frames the
UNMODIFIED reference class returned (fixtures by oracle/make_golden_render.py). GPU: v2e_b200.renderer.EventRenderer
against the same fixtures, packet by packet (the state carried between packets matters), and against the oracle on a
larger seeded stream -- float64 frames, bit-exact."""
import os

import numpy as np
import pytest

from helpers import GOLDEN_DIR
from render_oracle import RenderOracle


def _golden():
    z = np.load(os.path.join(GOLDEN_DIR, "render_ref.npz"))
    for name in z["names"]:
        name = str(name)
        mode, value, H, W, fs, npk, area = z[name + "_cfg"]
        pk = [(z["%s_ev_%d" % (name, i)], z["%s_fr_%d" % (name, i)]) for i in range(int(npk))]
        # the exposure value as the reference got it, a Python float: a numpy float64 would make the DURATION frame start
        # times accumulate in float64 instead of float32 (renderer.py:208, 316), which shows past 2^31 us
        yield name, int(mode), (float(value) if int(mode) == 1 else int(value)), int(H), int(W), int(fs), int(area) or None, pk


def test_oracle_matches_reference_fixtures():
    for name, mode, value, H, W, fs, area, pk in _golden():
        o = RenderOracle(fs, mode, value, area)
        n = 0
        for ev, want in pk:
            got = o.render(ev, H, W)
            got = np.zeros((0, H, W)) if got is None else got
            assert got.dtype == np.float64 and got.shape == want.shape and np.array_equal(got, want), name
            n += len(want)
        assert n > 0, name


@pytest.mark.gpu
def test_cuda_renderer_matches_reference_fixtures():
    from v2e_b200.renderer import EventRenderer, ExposureMode
    done = 0
    for name, mode, value, H, W, fs, area, pk in _golden():
        r = EventRenderer(full_scale_count=fs, exposure_mode=ExposureMode(mode), exposure_value=value, area_dimension=area)
        for ev, want in pk:
            got = r.render_events_to_frames(ev, H, W, return_frames=True)
            got = np.zeros((0, H, W)) if got is None else got
            assert got.dtype == np.float64 and got.shape == want.shape and np.array_equal(got, want), name
        done += 1
    assert done == 18


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2, 3, 4])
def test_cuda_renderer_matches_oracle_on_a_dense_stream(mode):
    """346x260, ~200 k events per packet from the pixel model's own output format (CUDA tensor in, device frames out)."""
    import torch
    from v2e_b200.renderer import EventRenderer, ExposureMode
    H, W = 260, 346
    rng = np.random.default_rng(5)
    value = {1: 0.002, 2: 30000, 3: 400, 4: 0}[mode]
    area = 16 if mode == 3 else None
    o = RenderOracle(3, mode, value, area)
    r = EventRenderer(full_scale_count=3, exposure_mode=ExposureMode(mode), exposure_value=value, area_dimension=area)
    t = 0.0
    for _ in range(3):
        n = 40000
        ts = np.sort(t + rng.uniform(0, 0.01, n)).astype(np.float32)
        t += 0.01
        ev = np.stack([ts, rng.integers(0, W, n), rng.integers(0, H, n), np.where(rng.random(n) < 0.5, 1, -1)], 1).astype(np.float32)
        ev[rng.integers(0, n, 3000), 1:3] = (100, 77)            # a hot pixel: the clip engages
        want = o.render(ev, H, W)
        got = r.render_events_to_frames(torch.from_numpy(ev).cuda(), H, W, return_device=True)
        if want is None:
            assert got is None
        else:
            assert np.array_equal(got.cpu().numpy(), want)
