"""CPU: the synthetic inputs of bench.py are what SURVEY.md 8(d) / BASELINE.json name. The config-2 clip must be the
reference's own scripts/gradients.py pattern (checked against frames the script itself produced, stored by
oracle/make_golden_gradients.py, and against properties of im_function); the config-3 / config-5 block texture must
be deterministic."""
import os

import numpy as np

import bench
from helpers import GOLDEN_DIR


def test_gradient_clip_properties():
    fr = bench.gradient_clip(260, 346, 31)
    assert fr.shape == (31, 260, 346) and fr.dtype == np.uint8
    low, high = np.uint8((127 * 2) / 3), np.uint8(2 * (127 * 2) / 3)      # contrast 2 around the background 127
    assert fr.min() == low and fr.max() == high
    assert (fr == fr[:, :1, :]).all()                                  # constant along y
    # the bump's peak moves 300 px/s = 10 px per 30 fps frame
    peaks = [int(np.argmax(f[0, :int(0.5 * 346) + 10 * k + 2])) for k, f in enumerate(fr[:10])]
    assert np.all(np.diff(peaks) == 10), peaks


def test_gradient_clip_equals_reference_script():
    ref = np.load(os.path.join(GOLDEN_DIR, "gradients_im_function.npz"))["frames"]     # gradients.py:117-140, 30 fps
    mine = bench.gradient_clip(260, 346, 8)
    assert ref.shape == mine.shape
    for k in range(8):
        assert np.array_equal(mine[k], ref[k]), k


def test_block_texture_clip_is_deterministic_and_translates():
    a = bench.block_texture_clip(64, 96, 5, seed=0)
    b = bench.block_texture_clip(64, 96, 5, seed=0)
    assert np.array_equal(a, b) and a.dtype == np.uint8
    assert np.array_equal(a[1][:-4, :-8], a[0][4:, 8:])                # (+8, +4) px per source frame
    assert len(np.unique(a[0])) > 50


def test_unet_activation_bytes_matches_a_hand_count():
    # one layer by hand: conv2 of UNet(12, 5) at 1280x704, batch 8: 32 channels in + 32 out, fp16
    tot = bench.unet_activation_bytes(12, 5, 704, 1280, 8)
    conv2 = 8 * 704 * 1280 * (32 + 32) * 2
    assert tot > 5 * conv2 and tot < 12 * conv2
