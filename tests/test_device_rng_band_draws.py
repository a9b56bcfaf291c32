"""GPU: the device-RNG draws of a pixel-sharded emulator's row band are the band's slice of the whole frame's -- leak,
shot and photoreceptor streams alike -- also for a band that starts in the middle of a Philox quad."""
import numpy as np
import pytest
import torch

import philox

pytestmark = pytest.mark.gpu

C3_PARAMS = dict(pos_thres=0.2, neg_thres=0.2, sigma_thres=0.03, cutoff_hz=300.0, leak_rate_hz=0.1,
                 shot_noise_rate_hz=5.0, refractory_period_s=0.0005)
SEED = 1234


def test_sharded_band_draws_the_matching_slice():
    """A sharded emulator's handle counts photoreceptor-noise pixels in the whole frame (v2e_emu_set_option(h, 1, 1),
    pr_noise_px4_unaligned for a band starting mid-quad), like its leak and shot pixels; an unsharded handle created
    with the same pixel offset keeps counting its own pixels, as before."""
    from v2e_b200 import EventEmulator
    H, W, y0, y1 = 37, 53, 13, 29                     # rng_pixel_offset 689 = 4 * 172 + 1
    full = EventEmulator(device="cuda", seed=SEED, rng_mode="device", **C3_PARAMS)
    band = EventEmulator(device="cuda", seed=SEED, rng_mode="device", shard=(1, 2, None), **C3_PARAMS)
    plain = EventEmulator(device="cuda", seed=SEED, rng_mode="device", **C3_PARAMS)
    full._create(H, W)
    band._create(y1 - y0, W, px_offset=y0 * W)
    plain._create(y1 - y0, W, px_offset=y0 * W)
    for fi in (0, 7):
        a, b, c = full.device_draws(fi), band.device_draws(fi), plain.device_draws(fi)
        for k in ("leak_randn", "shot_u01", "pr_randn"):
            assert torch.equal(b[k], a[k][y0:y1]), k
        assert not torch.equal(b["pr_randn"], a["pr_randn"][:y1 - y0])
        assert torch.equal(c["pr_randn"], a["pr_randn"][:y1 - y0])
        assert np.array_equal(b["shot_u01"].cpu().numpy().ravel(),
                              philox.shot_u01(SEED, (y1 - y0) * W, fi, px_off=y0 * W))
