"""The strip kernel's stacked wgmma chain (conv_tc.cu, strip_stack_mma): one wgmma of N = 2 * BN per input row, slab,
column and 16 channels, over weight tiles stacked in shared memory with zero tiles at both ends of every column. The
extra terms are exact zeros added to accumulators that start at +0, so the outputs must be bit-identical to the paired
chain's (two wgmmas of N = BN), and -- where there is one channel slab, so that the two kernels' term orders
coincide -- to the per-tap kernel's. Elsewhere the float64 reference bounds them as in test_slomo_gpu.py.

CPU: which strip layers run the stacked chain (v2e_conv_strip_pick_chain). GPU: every strip layer of the headline
(1280x704 and its half-resolution layers) and of the 346x260 secondary (320x256), the strip cases of test_slomo_gpu.py
(ragged strips, odd last rows, concatenated inputs, split output channels), and the whole network planned for 1 and
for all SMs. The pooled epilogue under the stacked chain is covered by test_slomo_gpu.py's fused-pool test (conv2)."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import conv_bound, conv_ref64, err_ratio
from test_layer_plan import LAYERS, cout_pad, pad16
from v2e_b200 import _lib

PAIRED, STACKED = 0, 1
DEV = "cuda:0"


def chains(W):
    lib = _lib.load()
    out = {}
    for name, c1, c2, co, k, lvl in LAYERS:
        ch = lib.v2e_conv_strip_pick_chain(pad16(c1), pad16(c2) if c2 else 0, cout_pad(co), k, k, W >> lvl)
        if ch >= 0:
            out[name] = "stacked" if ch == STACKED else "paired"
    return out


def test_stacked_chain_plan_at_1280():
    # every layer with <= 32 output channels per CTA class whose stacked weights fit beside the ring with the paired
    # plan's CTAs per SM and split: not down1.conv1 (64 channels per CTA), down1.conv2 (124 KB of weights per CTA class
    # beside six 17 KB ring rows) and up4.conv1/2
    assert chains(1280) == {"conv1": "stacked", "conv2": "stacked", "down1.c1": "paired", "down1.c2": "paired",
                            "up4.c1": "paired", "up4.c2": "paired", "up5.c1": "stacked", "up5.c2": "stacked",
                            "conv3": "stacked"}


def test_stacked_chain_plan_at_320():
    assert chains(320) == {"conv1": "stacked", "conv2": "stacked", "up5.c1": "stacked", "up5.c2": "stacked",
                           "conv3": "stacked"}


# ---- GPU ---------------------------------------------------------------------------------------------------------
# (N, H, W, C1, C2, Cout, K, out_mode): the strip layers at the headline's network size (batch 1) and at the
# secondary's (batch 2); the layer names are test_layer_plan.py's strip layers at those widths
STRIP_1280 = ("conv1", "conv2", "down1.c1", "down1.c2", "up4.c1", "up4.c2", "up5.c1", "up5.c2", "conv3")
STRIP_320 = ("conv1", "conv2", "up5.c1", "up5.c2", "conv3")
HEADLINE = [(1, 704 >> lvl, 1280 >> lvl, c1, c2, co, k, 1 if name == "conv3" else 0)
            for name, c1, c2, co, k, lvl in LAYERS if name in STRIP_1280]
SECONDARY = [(2, 256, 320, c1, c2, co, k, 1 if name == "conv3" else 0)
             for name, c1, c2, co, k, lvl in LAYERS if name in STRIP_320]


def _cases():
    from test_slomo_gpu import STRIP_CASES
    return HEADLINE + SECONDARY + STRIP_CASES


def _run(case, seed):
    from test_slomo_gpu import pack_w, pack_w_strip, to_nhwc16
    N, H, W, C1, C2, Cout, K, mode = case
    L = _lib.load()
    g = torch.Generator().manual_seed(seed)
    x1 = torch.randn((N, C1, H, W), generator=g).to(DEV)
    x2 = torch.randn((N, C2, H, W), generator=g).to(DEV) if C2 else None
    w = (torch.randn((Cout, C1 + C2, K, K), generator=g) / np.sqrt((C1 + C2) * K * K)).to(DEV)
    b = (torch.randn((Cout,), generator=g) * 0.1).to(DEV)
    a1 = to_nhwc16(x1)
    a2 = to_nhwc16(x2) if C2 else None
    c1p, c2p, Cp = a1.shape[-1], a2.shape[-1] if C2 else 0, cout_pad(Cout)
    KC = L.v2e_conv_strip_pick_kc(c1p, c2p, Cp, K, K, W)
    assert KC in (16, 32, 64), "case must qualify for the strip kernel"
    bp = torch.zeros(Cp, device=DEV)
    bp[:Cout] = b
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())

    def new_out():
        return torch.full((N, H, W, Cp if mode == 0 else 8), float("nan"),
                          dtype=torch.float16 if mode == 0 else torch.float32, device=DEV)

    wrow, _ = pack_w_strip(w, C1, C2, KC)
    outs = {}
    for chain in (PAIRED, STACKED):
        out = new_out()
        rc = L.v2e_conv2d_lrelu_sm100_strip_chain(p(a1), c1p, p(a2), c2p, p(wrow), p(bp), Cp, K, K, N, H, W, p(out), Cp,
                                                  mode, min(Cout, 8), ctypes.c_float(0.1), chain, st)
        if chain == STACKED and rc == _lib.V2E_E_INVALID:
            continue                                      # the stacked weights do not fit beside the ring
        _lib.check(rc)
        outs[chain] = out
    wtap, _ = pack_w(w, C1, C2)
    tap = new_out()
    _lib.check(L.v2e_conv2d_lrelu_sm100(p(a1), c1p, p(a2), c2p, p(wtap), p(bp), Cp, K, K, N, H, W, p(tap), Cp, mode,
                                        min(Cout, 8), ctypes.c_float(0.1), st))
    torch.cuda.synchronize()
    return outs, tap, (c1p + c2p) // KC, (x1, x2, w, b)


@pytest.mark.gpu
@pytest.mark.parametrize("case", _cases())
def test_stacked_chain_is_bit_identical(case):
    N, H, W, C1, C2, Cout, K, mode = case
    outs, tap, slabs, (x1, x2, w, b) = _run(case, hash(case) & 0xFFFF)
    co = min(Cout, outs[PAIRED].shape[-1])
    got = outs.get(STACKED, outs[PAIRED])
    if STACKED in outs:
        assert torch.equal(outs[STACKED].view(torch.uint8), outs[PAIRED].view(torch.uint8)), \
            "stacked and paired chains differ in %d elements" % int((outs[STACKED] != outs[PAIRED]).sum())
    else:
        lib = _lib.load()
        assert lib.v2e_conv_strip_pick_chain(pad16(C1), pad16(C2) if C2 else 0, cout_pad(Cout), K, K, W) == PAIRED
    if slabs == 1:
        assert torch.equal(got[..., :co].contiguous().view(torch.uint8), tap[..., :co].contiguous().view(torch.uint8)), \
            "strip and per-tap kernels differ in %d elements" % int((got[..., :co] != tap[..., :co]).sum())
    else:
        xin = torch.cat([x1, x2], 1) if C2 else x1
        ref, S = conv_ref64(xin.half(), w.half(), b, K // 2)
        ref, S = ref.permute(0, 2, 3, 1), S.permute(0, 2, 3, 1)
        r = err_ratio(got[..., :co], ref[..., :co], conv_bound(ref[..., :co], S[..., :co], fp16_out=mode == 0))
        assert r <= 1.0, r


@pytest.mark.gpu
def test_headline_frames_do_not_depend_on_the_sm_count():
    """The full network at the headline's frame size, planned for 1 SM (option 3) and for all of them: flow heads,
    intermediate heads, float32 and uint8 frames identical (every strip layer's CTAs walk all items at 1 SM)."""
    from test_slomo_geometry import assert_image_equal, device_sms, run_engine, textured
    src, B = (1280, 720), 1
    frames = torch.from_numpy(textured(B + 1, src[1], src[0], 29)).to(DEV)
    ref, plan = run_engine(src, B, frames, n_sms=device_sms())
    got, p = run_engine(src, B, frames, n_sms=1)
    assert p == plan
    assert_image_equal(ref, 0, got, 0, "1280x720 planned for 1 SM")
