"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/laplacian_conv2d.npz: torch's CPU float32 Laplacian

    torch.conv2d(ReplicationPad2d(1)(h), [[0,1,0],[1,-4,1],[0,1,0]])       (emulator.py:1105-1115)

of seeded [1,1,H,W] fields at the frame sizes where its summation order changes. tests/test_laplacian_order.py
checks oracle_laplacian_f32 (oracle/emu_oracle.c) against it bit for bit.

    python oracle/make_golden_laplacian.py            # writes the fixture
    python oracle/make_golden_laplacian.py bisect     # re-measures the order switch

How the rule was found (torch 2.11 CPU, get_cpu_capability() == "AVX512"): at every pixel the result equals one of
two float32 sums of the five taps, kernel order (((u+l)+c)+r)+d or pairwise order (u+l)+(c+(r+d)).
`bisect` classifies every factorisation (H+2)*(W+2) = P of every padded size P in [20400, 20600): all shapes with
P <= 20480 take pairwise order, all with P > 20480 kernel order, whatever their aspect ratio. That is ATen's
use_mkldnn size heuristic (input numel > 20480 selects oneDNN). Below it the native im2col + GEMM path pairs the
taps except in the last n mod 16 elements of the flattened output (its 16-float vector remainder), which take
kernel order. The torch thread count does not change either result.

Two fields per shape: random normal (almost every pixel tells the two orders apart) and a surround-like field of
log intensities with small spatial differences, what the Euler iteration actually convolves. Both are rebuilt by
the test from `field(H, W, kind)`.
"""
import hashlib
import os
import sys

import numpy as np
import torch

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "laplacian_conv2d.npz")
KINDS = ("normal", "surround")
# Every output is stored as a sha256 of its bytes, which pins each pixel. Outputs of up to FULL_MAX_PX pixels are
# stored whole as well; larger ones keep SAMPLE elements (the last 16, where the tail lies, and seeded random ones)
# so that a mismatch can be located.
FULL_MAX_PX = 2048
SAMPLE = 256

SWITCH = [(141, 141), (141, 142), (143, 143), (100, 199), (99, 202), (20, 974), (19, 1050), (200, 100), (120, 176),
          (126, 158), (1, 6825)]        # padded 20449, 20592, 21025, 20502, 20604, 21472, 22092, 20604, 21716, 20480, 20481
TAILS = [(3, w) for w in range(16, 32)]  # n = 3w: every n mod 16 from 0 to 15
EDGES = [(1, 1), (1, 2), (2, 1), (1, 37), (37, 1), (29, 2), (2, 29), (7, 9), (37, 53), (13, 37), (20, 36), (60, 80),
         (2, 9), (2, 23)]
PRODUCTION = [(260, 346), (720, 1280), (704, 1280)]
SHAPES = SWITCH + TAILS + EDGES + PRODUCTION


def field(H, W, kind):
    rng = np.random.default_rng([H, W, KINDS.index(kind)])
    if kind == "normal":
        return rng.standard_normal((H, W)).astype(np.float32)
    # lin_log of a mid-grey scene with a few percent of contrast: log values near 4.8 that differ by ~1e-2
    return (np.log(120.0) + 0.02 * rng.standard_normal((H, W))).astype(np.float32)


def torch_laplacian(h):
    lap = torch.tensor([[0, 1, 0], [1, -4, 1], [0, 1, 0]], dtype=torch.float32).view(1, 1, 3, 3)
    t = torch.from_numpy(h).view(1, 1, *h.shape)
    return torch.conv2d(torch.nn.ReplicationPad2d(1)(t), lap)[0, 0].numpy().copy()


def two_orders(h):
    """(kernel order, pairwise order) sums of the five taps, float32, replicate padding."""
    H, W = h.shape
    p = np.pad(h, 1, mode="edge")
    u, l, c = p[0:H, 1:W + 1], p[1:H + 1, 0:W], np.float32(-4) * p[1:H + 1, 1:W + 1]
    r, d = p[1:H + 1, 2:W + 2], p[2:H + 2, 1:W + 1]
    return (((u + l) + c) + r) + d, (u + l) + (c + (r + d))


def sample_index(n):
    rnd = np.random.default_rng(n).choice(n - 16, size=SAMPLE - 16, replace=False)
    return np.sort(np.concatenate([rnd, np.arange(n - 16, n)])).astype(np.int32)


def bisect():
    for P in range(20400, 20600):
        seen = set()
        for a in range(3, P // 3 + 1):
            if P % a:
                continue
            H, W = a - 2, P // a - 2
            if H < 1 or W < 1:
                continue
            t = torch_laplacian(field(H, W, "normal")).view(np.uint32)
            k, pw = (x.view(np.uint32) for x in two_orders(field(H, W, "normal")))
            if np.array_equal(t, k):
                seen.add("kernel")
            elif np.array_equal(t.ravel()[:H * W // 16 * 16], pw.ravel()[:H * W // 16 * 16]):
                seen.add("pairwise")
            else:
                seen.add("neither: %dx%d" % (H, W))
        print(P, sorted(seen))


def main():
    d = {"torch_version": np.array(torch.__version__),
         "cpu_capability": np.array(torch.backends.cpu.get_cpu_capability()),
         "shapes": np.array(SHAPES, np.int64), "kinds": np.array(KINDS)}
    for i, (H, W) in enumerate(SHAPES):
        for kind in KINDS:
            out = torch_laplacian(field(H, W, kind))
            key = "%d_%s" % (i, kind)
            d["sha256_" + key] = np.array(hashlib.sha256(out.tobytes()).hexdigest())
            if H * W <= FULL_MAX_PX:
                d["out_" + key] = out
            else:
                idx = sample_index(H * W)
                d["sample_idx_" + key] = idx
                d["sample_" + key] = out.ravel()[idx]
    np.savez_compressed(OUT, **d)
    print("%s: %d shapes, %.1f KB" % (OUT, len(SHAPES), os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    bisect() if sys.argv[1:] == ["bisect"] else main()
