"""Per-layer timing of the strip convolution (csrc/conv_tc.cu, conv_strip_kernel) with its two wgmma chains: "paired"
(per input row, two wgmmas of N = BN, one per output row of the pair) against "stacked" (one wgmma of N = 2 * BN over
weight tiles stacked with zero tiles in shared memory), at the shapes the headline runs the strip layers at.

    python bench_strip.py [--size 1280|320] [--iters 100] [--warmup 20] [--layers conv1,conv2]

Every strip layer of the flow / interpolation UNets at the headline (batch 8, 1280x704 and its half-resolution layers)
or at the 346x260 secondary's network size (batch 30, 320x256). conv2 and down1.conv2 are timed without the 2x2 pool
their epilogue writes in the network. For every layer the chains are launched in turn, each timed with CUDA events over
--iters back-to-back launches after --warmup launches; the rounds alternate (--rounds) so that clock drift hits both
alike, and the median round is reported. Per layer and chain: ms per launch, TFLOP/s (2 * pixels * Cout * Cin * K^2
over the real channel counts) and the shared-memory operand bytes the wgmmas read per second, counted from the chain
shape: per output-row pair and 64-pixel half, the paired chain issues 2 * KH wgmmas of N = BN per (slab, s, k16), the
stacked chain KH + 1 of N = 2 * BN, each reading a 64 x 16 A window (2 KB) and an N x 16 weight tile. "auto" names the
chain the network runs (up5.conv1 is left out where the network runs it with its up-sampling folded in). A chain
whose resident weights do not fit is reported as such. The card's name, power limit
and SM clock are read in the same process. One JSON line at the end."""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench_conv import card  # noqa: E402
from v2e_b200 import _lib  # noqa: E402

PAIRED, STACKED = 0, 1
CHAINS = [("paired", PAIRED), ("stacked", STACKED)]
# (name, cin1, cin2, cout, k, level, out_mode) of the UNets' strip layers (tests/test_layer_plan.py)
STRIP_LAYERS = [("conv1", 12, 0, 32, 7, 0, 0), ("conv2", 32, 0, 32, 7, 0, 0),
                ("down1.c1", 32, 0, 64, 5, 1, 0), ("down1.c2", 64, 0, 64, 5, 1, 0),
                ("up4.c1", 128, 0, 64, 3, 1, 0), ("up4.c2", 64, 64, 64, 3, 1, 0),
                ("up5.c1", 64, 0, 32, 3, 0, 0), ("up5.c2", 32, 32, 32, 3, 0, 0), ("conv3", 32, 0, 5, 3, 0, 1)]
SIZES = {"1280": (8, 704, 1280), "320": (30, 256, 320)}
ROW_TILE = 128


def pad16(c):
    return (c + 15) // 16 * 16


def cout_pad(c):
    p = pad16(c)
    return 16 if p <= 16 else 32 if p <= 32 else 64 if p <= 64 else (p + 127) // 128 * 128


def pairs(N, H, W, K, n_sms):
    """Output-row pairs over all items (v2e_strip_prepare's segmentation; an odd last row runs a whole pair)."""
    tiles_x = -(-W // ROW_TILE)
    seg_h, strips = H, tiles_x * N
    while seg_h > 4 * K and strips * -(-H // seg_h) < 6 * n_sms:
        seg_h = (seg_h + 1) // 2
    return strips * sum(-(-min(seg_h, H - y) // 2) for y in range(0, H, seg_h))


def n_split_of(c1p, c2p, Cp, K, kc, stacked):
    """CTA classes of the layer's strip plan (conv_tc.cu, strip_config); None: the chain's weights do not fit."""
    up = lambda x: -(-x // 1024) * 1024
    slabs = (c1p + c2p) // kc
    row = up((ROW_TILE + K - 1) * kc * 2) * slabs
    for split in (1, 2):
        bn = Cp // split
        if bn < 16 or bn % 16:
            break
        wb = up(slabs * (K * (K + 1) + 1 if stacked else K * K) * bn * kc * 2)
        budget = 110 * 1024 if wb + 2048 + (K + 3) * row <= 110 * 1024 else 222 * 1024
        if wb + 2048 + (K + 1) * row <= budget:
            return split
    return None


def smem_operand_bytes(chain, n_pairs, K, C, KC, Cp, n_split):
    """Bytes the wgmmas of a launch read from shared memory (A windows + weight tiles), over all CTA classes."""
    bn = Cp // n_split
    k16 = C // 16                        # slabs x KC / 16
    per = (2 * K, bn) if chain == PAIRED else (K + 1, 2 * bn)
    wgmmas = n_pairs * 2 * n_split * per[0] * K * k16
    return wgmmas * (64 * 16 * 2 + per[1] * 16 * 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="1280", choices=sorted(SIZES))
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--layers", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_strip.py needs a CUDA device")
    L = _lib.load()
    N, H0, W0 = SIZES[a.size]
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    want = set(a.layers.split(",")) if a.layers else None
    st = torch.cuda.current_stream()
    stp = ctypes.c_void_p(st.cuda_stream)
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    rows = []
    card_before = card()
    for name, c1, c2, co, K, lvl, mode in STRIP_LAYERS:
        if want and name not in want:
            continue
        H, W = H0 >> lvl, W0 >> lvl
        c1p, c2p, Cp = pad16(c1), pad16(c2) if c2 else 0, cout_pad(co)
        KC = L.v2e_conv_strip_pick_kc(c1p, c2p, Cp, K, K, W)
        if not KC or (name == "up5.c1" and L.v2e_conv_up2_supported_c(c1p, Cp, W)):
            continue                    # up5.conv1 runs with its up-sampling folded in where that kernel applies
        auto = L.v2e_conv_strip_pick_chain(c1p, c2p, Cp, K, K, W)
        g = torch.Generator(device="cuda:0").manual_seed(lvl * 10 + K)
        x1 = torch.randn((N, H, W, c1p), generator=g, device="cuda:0").half()
        x2 = torch.randn((N, H, W, c2p), generator=g, device="cuda:0").half() if c2 else None
        slabs = (c1p + c2p) // KC
        w = (torch.randn((slabs, K * K, Cp, KC), generator=g, device="cuda:0") / (K * K * (c1p + c2p)) ** 0.5).half()
        b = torch.zeros(Cp, device="cuda:0")
        out = torch.empty((N, H, W, Cp if mode == 0 else 8), dtype=torch.float16 if mode == 0 else torch.float32,
                          device="cuda:0")

        def launch(chain):
            return L.v2e_conv2d_lrelu_sm100_strip_chain(p(x1), c1p, p(x2), c2p, p(w), p(b), Cp, K, K, N, H, W, p(out),
                                                        Cp, mode, min(co, 8), ctypes.c_float(0.1), chain, stp)

        variants = []
        for vn, chain in CHAINS:
            if launch(chain) == 0:
                variants.append((vn, chain))
        torch.cuda.synchronize()
        times = {vn: [] for vn, _ in variants}
        for _ in range(a.rounds):
            for vn, chain in variants:
                for _ in range(a.warmup):
                    launch(chain)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                for _ in range(a.iters):
                    launch(chain)
                e1.record(st)
                e1.synchronize()
                times[vn].append(e0.elapsed_time(e1) / a.iters)
        flops = 2.0 * N * H * W * co * (c1 + c2) * K * K
        npairs = pairs(N, H, W, K, n_sms)
        row = {"layer": name, "shape": [N, H, W, c1 + c2, co, K], "kc": KC,
               "auto": "stacked" if auto == STACKED else "paired"}
        for vn, chain in CHAINS:
            if vn not in times:
                row[vn] = "does not fit"
                continue
            ms = sorted(times[vn])[len(times[vn]) // 2]
            by = smem_operand_bytes(chain, npairs, K, c1p + c2p, KC, Cp, n_split_of(c1p, c2p, Cp, K, KC, chain))
            row[vn] = {"ms": round(ms, 4), "tflops": round(flops / ms / 1e9, 1), "smem_tb_s": round(by / ms / 1e9, 2),
                       "spread_ms": round(max(times[vn]) - min(times[vn]), 4)}
        rows.append(row)
        print("%-9s %-24s auto=%-7s" % (name, "x".join(map(str, row["shape"])), row["auto"]) +
              "".join("  %s %.3f ms %5.0f TF/s %5.2f TB/s" % (vn, row[vn]["ms"], row[vn]["tflops"], row[vn]["smem_tb_s"])
                      if isinstance(row[vn], dict) else "  %s: does not fit" % vn for vn, _ in CHAINS), flush=True)
        del x1, x2, w, out
    res = {"what": "strip convolution chains at %s (batch %d)" % (a.size, N), "card": card_before,
           "card_after": card(), "iters": a.iters, "rounds": a.rounds, "layers": rows}
    for vn, _ in CHAINS:
        res["total_ms_" + vn] = round(sum(r[vn]["ms"] for r in rows if isinstance(r[vn], dict)), 3)
    res["total_ms_auto"] = round(sum(r[r["auto"]]["ms"] for r in rows), 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
