#!/usr/bin/env python
"""V2EPipeline without an upsampler (v2e.py's --disable_slomo / no-upsampling mode): every emulated frame is a source
frame, so nothing hides the frames' trip to the device. At 1280x720 and 346x260, v2e's CLI defaults (rng_mode="device"),
a 300 fps clip moving 1 px per frame (bench.source_clip(px_per_frame=1): about the motion per frame of a SloMo-upsampled
clip), --frames source frames (default 1280: two default segments of 640):

  seg_pinned / seg_device   V2EPipeline(None, em).run_segments(get_frames, ...) with the default segment length, frames
                            fetched from pinned host memory / already on the device; host rows (copy=False)
  batch_floor               EventEmulator.generate_events_batch on device-resident frames, one call per 640 frames,
                            host rows (copy=False): the pixel model alone, the floor for the pipeline
  drop_in                   v2e.py's loop today: generate_events(frame_i, f * i) per frame from host uint8 arrays
                            (--drop-in-frames frames)
  h2d                       the copy of one segment of frames from pinned host memory to the device alone

Every arm runs on its own emulator, one warm-up call and then --rounds rounds, alternating arms; each call starts one
frame interval after the previous one. Reported: ms per frame (median, min, max over rounds); for run_segments from
pinned memory at 64, 160 and 640 frames per segment, the device memory its first call added on top of what was
allocated before it (torch.cuda.max_memory_allocated - memory_allocated). Prints one JSON line with the card's name,
power limit and max SM clock, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

SIZES = ((720, 1280), (260, 346))
FPS = 300.0
MEMORY_SEGMENTS = (64, 160, 640)


def bench_size(H, W, a):
    from bench import CLI_DEFAULTS, source_clip
    from v2e_b200 import EventEmulator, V2EPipeline
    from v2e_b200.pipeline import DEFAULT_SEGMENT_FRAMES
    n = a.frames
    loop = source_clip(H, W, 2 * 256 + 1, seed=0, px_per_frame=1)[:512]       # loops: frame 512 is frame 0
    host = torch.from_numpy(loop[np.arange(n) % 512]).pin_memory()
    dev = host.to("cuda:0")
    clip_s = (n - 1) / FPS
    period = n / FPS
    mk = lambda: EventEmulator(device="cuda:0", rng_mode="device", seed=1, **CLI_DEFAULTS)

    def seg_arm(src, seg=None):
        def call(em, t0):
            rows = 0
            for ev, offs, t, k in V2EPipeline(None, em).run_segments(lambda p, q: src[p:q], n, clip_s, t_offset=t0,
                                                                     segment_pairs=seg):
                rows += len(ev)
            return n, rows
        return call

    def batch_floor(em, t0):
        t = t0 + clip_s / np.int64(n - 1) * np.arange(n)
        rows = 0
        for p in range(0, n, DEFAULT_SEGMENT_FRAMES):
            q = min(n, p + DEFAULT_SEGMENT_FRAMES)
            ev, offs = em.generate_events_batch(dev[p:q], t[p:q], copy=False)
            rows += len(ev)
        return n, rows

    nd = min(a.drop_in_frames, n)
    host_np = host.numpy()

    def drop_in(em, t0):
        f = clip_s / np.int64(n - 1)
        rows = 0
        for i in range(nd):
            ev = em.generate_events(host_np[i], t0 + f * i)
            rows += 0 if ev is None else len(ev)
        return nd, rows

    seg_len = min(DEFAULT_SEGMENT_FRAMES, n)
    scratch = torch.empty((seg_len, H, W), dtype=torch.uint8, device="cuda:0")

    def h2d(em, t0):
        scratch.copy_(host[:seg_len], non_blocking=True)
        return seg_len, 0

    arms = dict(seg_pinned=seg_arm(host), seg_device=seg_arm(dev), batch_floor=batch_floor, drop_in=drop_in, h2d=h2d)
    state = {k: dict(em=mk(), calls=0, ms=[]) for k in arms}

    def run(name):
        st = state[name]
        t0 = st["calls"] * period
        st["calls"] += 1
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        nf, rows = arms[name](st["em"], t0)
        torch.cuda.synchronize()
        return (time.perf_counter() - w0) * 1e3 / nf, nf, rows

    res = {}
    for name in arms:
        _, nf, rows = run(name)                           # warm-up
        res[name] = dict(frames_per_call=nf, events_per_frame=round(rows / nf, 1))
    for _ in range(a.rounds):
        for name in arms:
            state[name]["ms"].append(run(name)[0])
    for name in arms:
        v = state[name]["ms"]
        res[name].update(ms_per_frame_median=round(float(np.median(v)), 4), ms_per_frame_min=round(min(v), 4),
                         ms_per_frame_max=round(max(v), 4))
    for st in state.values():
        st["em"].cleanup()
    del state
    mem = {}
    for seg in MEMORY_SEGMENTS:
        em = mk()
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        seg_arm(host, seg)(em, 0.0)
        torch.cuda.synchronize()
        mem[str(seg)] = torch.cuda.max_memory_allocated() - before
        em.cleanup()
        del em
    return dict(size="%dx%d" % (W, H), frames=n, fps=FPS, h2d_bytes_per_frame=H * W, arms=res,
                added_device_bytes_by_segment_frames=mem)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1280)
    ap.add_argument("--drop-in-frames", type=int, default=320)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sizes", default="1280x720,346x260")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_no_upsampler.py needs a CUDA device")
    out = dict(bench="no_upsampler", rounds=a.rounds, results=[])
    for s in a.sizes.split(","):
        W, H = (int(x) for x in s.split("x"))
        out["results"].append(bench_size(H, W, a))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    out["gpu"] = q[0] if q else "unknown"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
