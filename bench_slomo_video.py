#!/usr/bin/env python
"""Cost of SuperSloMo's vid_orig / vid_slomo videos on the in-memory path: interpolated frames/s of
SuperSloMo.interpolate_frames without and with video_path, at 346x260 and 1280x720, U = 10, batch 8, bench.py's
seeded random weights and source clip (17 source frames: two batches, 160 interpolated frames per call).

With video_path the frames go through a real cv2.VideoWriter with the XVID fourcc -- the writer the reference's
v2ecore.v2e_utils.video_writer returns (v2e_utils.py:277) -- into a temporary directory. The two settings alternate
in one process. Per call it reports
  device_ms  CUDA-event time of the call without video (the SloMo kernels; interpolate_frames ends in a synchronise)
  writer_ms  host time in GRAY2BGR + encode (the writes of both videos), with video
  d2h_ms     one synchronised pageable copy of the call's output to host memory (the bytes the per-batch copies move)
  fps_off / fps_video  interpolated frames per second of wall time.
Prints one JSON line with the card's name, power limit and max SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

SIZES = ((346, 260), (1280, 720))
U, BATCH, N_SRC = 10, 8, 17


def install_xvid_writer(cv2):
    """v2ecore.v2e_utils.video_writer as the reference defines it: XVID, (width, height)."""
    mod = types.ModuleType("v2ecore.v2e_utils")
    mod.video_writer = lambda path, height, width, frame_rate=30: cv2.VideoWriter(
        path, cv2.VideoWriter_fourcc(*"XVID"), frame_rate, (width, height))
    pkg = types.ModuleType("v2ecore")
    pkg.v2e_utils = mod
    sys.modules["v2ecore"], sys.modules["v2ecore.v2e_utils"] = pkg, mod


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_slomo_video.py needs a CUDA device")
    import cv2
    from bench import slomo_weights, source_clip
    from v2e_b200 import SuperSloMo
    from v2e_b200 import slomo as slomo_mod
    install_xvid_writer(cv2)
    writer_s = [0.0]
    write_gray = slomo_mod._write_gray

    def timed_write_gray(writer, frames):
        t0 = time.perf_counter()
        n = write_gray(writer, frames)
        writer_s[0] += time.perf_counter() - t0
        return n
    slomo_mod._write_gray = timed_write_gray

    wts = slomo_weights()
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        for W, H in SIZES:
            src = torch.from_numpy(source_clip(H, W, N_SRC, seed=0)).cuda()
            vdir = os.path.join(tmp, "%dx%d" % (W, H))
            os.makedirs(vdir)
            arms = {"off": SuperSloMo(model=None, auto_upsample=False, upsampling_factor=U, batch_size=BATCH,
                                      state_dicts=wts),
                    "video": SuperSloMo(model=None, auto_upsample=False, upsampling_factor=U, batch_size=BATCH,
                                        state_dicts=wts, video_path=vdir)}
            out = None
            for s in arms.values():                     # warm-up: engine, kernels, writers
                out, _, _ = s.interpolate_frames(src)
            nf = out.shape[0]
            wall = {k: [] for k in arms}
            dev, wr, d2h = [], [], []
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(a.rounds):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e0.record()
                out, _, _ = arms["off"].interpolate_frames(src)
                e1.record()
                torch.cuda.synchronize()
                wall["off"].append(time.perf_counter() - t0)
                dev.append(e0.elapsed_time(e1))
                t0 = time.perf_counter()
                out.cpu()
                d2h.append((time.perf_counter() - t0) * 1e3)
                writer_s[0] = 0.0
                t0 = time.perf_counter()
                arms["video"].interpolate_frames(src)
                torch.cuda.synchronize()
                wall["video"].append(time.perf_counter() - t0)
                wr.append(writer_s[0] * 1e3)
            written = arms["video"].numSlomoVideoFramesWritten
            for s in arms.values():
                s.cleanup()
            size = os.path.getsize(os.path.join(vdir, "slomo.avi"))
            med = lambda v: float(np.median(v))
            res["%dx%d" % (W, H)] = {
                "frames_per_call": nf, "fps_off": round(nf / med(wall["off"]), 1),
                "fps_video": round(nf / med(wall["video"]), 1),
                "device_ms": round(med(dev), 2), "writer_ms": round(med(wr), 2), "d2h_ms": round(med(d2h), 2),
                "wall_ms_off": round(med(wall["off"]) * 1e3, 2), "wall_ms_video": round(med(wall["video"]) * 1e3, 2),
                "slomo_frames_written": written, "slomo_avi_bytes": size}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"bench": "slomo_video", "U": U, "batch": BATCH, "source_frames": N_SRC, "rounds": a.rounds,
                      "codec": "XVID (cv2 %s)" % cv2.__version__, "host_cpus": os.cpu_count(),
                      "sizes": res, "gpu": q[0] if q else "unknown"}))


if __name__ == "__main__":
    main()
