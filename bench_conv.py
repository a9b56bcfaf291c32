"""Per-layer timing of the per-tap convolution's tiles (csrc/conv_tc.cu): the 128 x 128 tile ("legacy") against the
wide tile the layer's shape calls for ("wide": 256 x 128 at 128 output channels, else 128 x 256), at the shapes the
headline runs them at.

    python bench_conv.py [--size 1280|320] [--iters 100] [--warmup 20] [--layers down4.c1,up1.c2]

For every per-tap layer of the UNets the variants are launched in turn, each timed with CUDA events over --iters
back-to-back launches after --warmup launches, and the rounds alternate (--rounds) so that clock drift hits every
variant alike; the median round is reported. Per layer and variant: ms per launch, TFLOP/s (2 * pixels * Cout * Cin *
9 / time) and the bytes the CTAs request from L2 into shared memory per second, counted from the tiling: launched
CTAs x (tap, slab) stages x bytes issued per stage (A window + the weight slab). The
card's name, power limit and SM clock are read in the same process. One JSON line at the end."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from v2e_b200 import _lib  # noqa: E402

LEGACY, T256x128, T128x256 = 0, 1, 2
TAP_LAYERS = [("down2.c1", 64, 0, 128, 2), ("down2.c2", 128, 0, 128, 2),
              ("down3.c1", 128, 0, 256, 3), ("down3.c2", 256, 0, 256, 3),
              ("down4.c1", 256, 0, 512, 4), ("down4.c2", 512, 0, 512, 4),
              ("down5.c1", 512, 0, 512, 5), ("down5.c2", 512, 0, 512, 5),
              ("up1.c1", 512, 0, 512, 4), ("up1.c2", 512, 512, 512, 4),
              ("up2.c1", 512, 0, 256, 3), ("up2.c2", 256, 256, 256, 3),
              ("up3.c1", 256, 0, 128, 2), ("up3.c2", 128, 128, 128, 2)]
SIZES = {"1280": (8, 704, 1280), "320": (30, 256, 320)}


def l2_bytes(tile, N, H, W, C, Cout):
    """CTAs x stages x bytes per stage the producers issue (KC = 64 for every per-tap layer)."""
    mh, bn = {LEGACY: (1, min(Cout, 128)), T256x128: (2, 128), T128x256: (1, 256)}[tile]
    tiles = -(-W // 16) * -(-H // (8 * mh)) * N
    ctas = tiles * (Cout // bn)
    a = 128 * mh * 64 * 2
    b = bn * 64 * 2
    return ctas * 9 * (C // 64) * (a + b), ctas


def card():
    props = torch.cuda.get_device_properties(0)
    info = {"name": props.name, "sms": props.multi_processor_count}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock"], info["sm_clock_max"] = [x.strip() for x in q.split(",")]
    except Exception as e:  # noqa: BLE001
        info["nvidia_smi"] = "unavailable: %s" % e
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="1280", choices=sorted(SIZES))
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--layers", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_conv.py needs a CUDA device")
    L = _lib.load()
    N, H0, W0 = SIZES[a.size]
    want = set(a.layers.split(",")) if a.layers else None
    st = torch.cuda.current_stream()
    stp = ctypes.c_void_p(st.cuda_stream)
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    rows = []
    card_before = card()
    for name, c1, c2, co, lvl in TAP_LAYERS:
        if want and name not in want:
            continue
        H, W = H0 >> lvl, W0 >> lvl
        g = torch.Generator(device="cuda:0").manual_seed(lvl)
        x1 = torch.randn((N, H, W, c1), generator=g, device="cuda:0").half()
        x2 = torch.randn((N, H, W, c2), generator=g, device="cuda:0").half() if c2 else None
        w = (torch.randn((co, 9 * (c1 + c2)), generator=g, device="cuda:0") / (9 * (c1 + c2)) ** 0.5).half()
        b = torch.zeros(co, device="cuda:0")
        out = torch.empty((N, H, W, co), dtype=torch.float16, device="cuda:0")
        wide = T256x128 if co == 128 else T128x256
        variants = [("legacy", LEGACY), ("wide", wide)]

        def launch(tile):
            _lib.check(L.v2e_conv2d_lrelu_sm100_tile(p(x1), c1, p(x2), c2, p(w), p(b), co, 3, 3, N, H, W, p(out), co,
                                                     0, co, ctypes.c_float(0.1), tile, stp))

        times = {v[0]: [] for v in variants}
        for _ in range(a.rounds):
            for vn, tile in variants:
                for _ in range(a.warmup):
                    launch(tile)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                for _ in range(a.iters):
                    launch(tile)
                e1.record(st)
                e1.synchronize()
                times[vn].append(e0.elapsed_time(e1) / a.iters)
        flops = 2.0 * N * H * W * co * (c1 + c2) * 9
        row = {"layer": name, "shape": [N, H, W, c1 + c2, co]}
        for vn, tile in variants:
            ms = sorted(times[vn])[len(times[vn]) // 2]
            by, ctas = l2_bytes(tile, N, H, W, c1 + c2, co)
            row[vn] = {"ms": round(ms, 4), "tflops": round(flops / ms / 1e9, 1), "l2_tb_s": round(by / ms / 1e9, 2),
                       "ctas": ctas, "spread_ms": round(max(times[vn]) - min(times[vn]), 4)}
        rows.append(row)
        print("%-9s %-22s" % (name, "x".join(map(str, row["shape"]))) +
              "".join("  %s %.3f ms %5.0f TF/s %4.2f TB/s" % (vn, row[vn]["ms"], row[vn]["tflops"], row[vn]["l2_tb_s"])
                      for vn, _ in variants), flush=True)
        del x1, x2, w, out
    res = {"what": "per-tap convolution tiles at %s (batch %d)" % (a.size, N), "card": card_before,
           "card_after": card(), "iters": a.iters, "rounds": a.rounds, "layers": rows}
    for vn in ("legacy", "wide"):
        res["total_ms_" + vn] = round(sum(r[vn]["ms"] for r in rows), 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
