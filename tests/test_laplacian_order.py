"""CPU: the float32 Laplacian of the centre-surround update (emulator.py:1115) as the oracle restates it
(oracle_laplacian_f32 / oracle_lap_kernel_order in oracle/emu_oracle.c) against torch's CPU conv2d, stored by
oracle/make_golden_laplacian.py in tests/golden/laplacian_conv2d.npz. Bit for bit, at frame sizes on both sides of the
summation-order switch, every flattened tail length n mod 16, degenerate widths and heights, and the production
sizes."""
import hashlib
import os

import numpy as np
import pytest
import torch

from emu_oracle import lib
from helpers import GOLDEN_DIR
from make_golden_laplacian import KINDS, SHAPES, field, two_orders

_G = np.load(os.path.join(GOLDEN_DIR, "laplacian_conv2d.npz"), allow_pickle=False)


def oracle_laplacian(h):
    h = np.ascontiguousarray(h, np.float32)
    out = np.empty_like(h)
    lib().oracle_laplacian_f32(h.ctypes.data, h.shape[0], h.shape[1], out.ctypes.data)
    return out


def test_fixture_lists_the_generator_shapes():
    assert [tuple(s) for s in _G["shapes"]] == SHAPES and list(_G["kinds"]) == list(KINDS)


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("i", range(len(SHAPES)), ids=["%dx%d" % s for s in SHAPES])
def test_oracle_laplacian_matches_torch_conv2d(i, kind):
    """Stored elements first, so that a mismatch names pixels; then the sha256 of the whole output."""
    H, W = SHAPES[i]
    got = oracle_laplacian(field(H, W, kind))
    key = "%d_%s" % (i, kind)
    if "out_" + key in _G.files:
        idx, want = np.arange(H * W), _G["out_" + key].ravel()
    else:
        idx, want = _G["sample_idx_" + key], _G["sample_" + key]
    bad = idx[got.ravel()[idx].view(np.uint32) != want.view(np.uint32)]
    assert bad.size == 0, "%dx%d %s: %d stored elements differ, first at flat index %s" % (H, W, kind, bad.size,
                                                                                      bad[:4].tolist())
    assert sha256(got) == str(_G["sha256_" + key]), "%dx%d %s: unstored elements differ" % (H, W, kind)


def test_fixture_tells_the_orders_apart():
    """Each part of the rule decides some pixel of the fixture: the oracle's output is the kernel-order sum where
    oracle_lap_kernel_order says so and the pairwise sum elsewhere (and equals torch's by the test above), and on
    the normal field the two sums differ at many pixels above the switch and in the flattened tail below it."""
    L = lib()
    for H, W in SHAPES:
        if H * W > 30000:
            continue
        h = field(H, W, "normal")
        k, p = (x.ravel().view(np.uint32) for x in two_orders(h))
        got = oracle_laplacian(h).ravel().view(np.uint32)
        kernel = np.array([L.oracle_lap_kernel_order(H, W, j) for j in range(H * W)], bool)
        assert np.array_equal(got[kernel], k[kernel]) and np.array_equal(got[~kernel], p[~kernel])
        if (H + 2) * (W + 2) > 20480:
            assert kernel.all() and (k != p).mean() > 0.3, (H, W)
        else:
            tail = H * W % 16
            assert kernel.sum() == tail and kernel[H * W - tail:].all()
            assert (k[~kernel] != p[~kernel]).any() or H * W - tail < 16, (H, W)
            if tail >= 4:           # a handful of random pixels always tell the sums apart
                assert (k[kernel] != p[kernel]).any(), (H, W)


def test_legacy_rule_is_caught():
    """The rule the oracle stated before (kernel order iff H*W >= 20000, no tail) differs from torch on 20x974
    (19 480 px, padded 21 472), 141x141 (19 881 px, padded 20 449) and 37x53 (tail of 9)."""
    L = lib()
    L.oracle_set_cs_perturbation(1, 0)
    try:
        for H, W in [(20, 974), (141, 141), (37, 53)]:
            i = SHAPES.index((H, W))
            assert sha256(oracle_laplacian(field(H, W, "normal"))) != str(_G["sha256_%d_normal" % i]), (H, W)
    finally:
        L.oracle_set_cs_perturbation(0, 0)


def test_fixture_host_matches_this_torch():
    """The fixture is a record of torch 2.11 on an AVX-512 host. Where this host's torch is the same build, recompute
    every shape and check that the fixture still describes it."""
    if str(_G["cpu_capability"]) != torch.backends.cpu.get_cpu_capability() or \
            str(_G["torch_version"]) != torch.__version__:
        pytest.skip("torch CPU kernels differ from the fixture's host")
    from make_golden_laplacian import torch_laplacian
    for i, (H, W) in enumerate(SHAPES):
        for kind in KINDS:
            assert sha256(torch_laplacian(field(H, W, kind))) == str(_G["sha256_%d_%s" % (i, kind)]), (H, W, kind)
