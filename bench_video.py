#!/usr/bin/env python
"""v2e's three default videos (vid_orig, vid_slomo and the DVS video) from V2EPipeline.run_segments at 1280x720 and
346x260, U = 10, batch 8, with bench.py's seeded SloMo weights, source clip and pixel-model settings (CLI defaults,
rng_mode="device") and v2e's default DVS video (DURATION 0.01 s, full scale 2).

Arms, alternating in rounds, every call a fresh SuperSloMo / EventRenderer writing into a temporary directory:
  none   no video;
  xvid   the three videos through a stand-in for v2ecore.v2e_utils.video_writer built on cv2.VideoWriter with XVID
         (as bench_slomo_video.py builds it): frames copied to the host and converted GRAY2BGR;
  mjpeg  the three videos through v2e_b200.MjpegWriter: device frames, device encode, compressed bytes to the host.
Reported per size and arm: ms per interpolated frame (median, min, max over the rounds) and the videos' bytes per
frame; for mjpeg also the encoder's kernel time per frame, from CUDA events around v2e_mjpeg_encode on one batch of
U * batch = 80 frames, the size of one SloMo batch. Prints one JSON line with the card's name and power
limit read in the same run."""
import argparse
import ctypes
import json
import os
import shutil
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

SIZES = ((1280, 720), (346, 260))
U, BATCH, SRC_FPS = 10, 8, 30.0


def install_xvid_writer():
    import cv2

    def video_writer(path, height, width, frame_rate=30, fourcc=None):
        w = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"XVID"), frame_rate, (width, height))
        if not w.isOpened():
            raise RuntimeError("cv2.VideoWriter cannot open XVID here")
        return w
    pkg = types.ModuleType("v2ecore")
    pkg.__path__ = []
    utils = types.ModuleType("v2ecore.v2e_utils")
    utils.video_writer = video_writer
    utils.checkAddSuffix = lambda p, s: p if p.endswith(s) else os.path.splitext(p)[0] + s
    pkg.v2e_utils = utils
    sys.modules["v2ecore"], sys.modules["v2ecore.v2e_utils"] = pkg, utils


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=32, help="source frame pairs of the clip")
    ap.add_argument("--segment", type=int, default=16, help="source frame pairs per segment")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_video.py needs a CUDA device")
    import cv2
    from bench import CLI_DEFAULTS, slomo_weights, source_clip
    from v2e_b200 import EventEmulator, MjpegWriter, SuperSloMo, V2EPipeline, _lib
    from v2e_b200.renderer import EventRenderer, ExposureMode
    install_xvid_writer()
    wts = slomo_weights()
    dev = torch.device("cuda", 0)
    tmp = tempfile.mkdtemp(prefix="bench_video_")
    arms = ("none", "xvid", "mjpeg")
    res = {}
    for W, H in SIZES:
        n = a.pairs + 1
        src = torch.from_numpy(source_clip(H, W, n, seed=0)).to(dev)
        clip_s = (n - 1) / SRC_FPS
        period = clip_s * n / (n - 1)
        state = {k: dict(em=EventEmulator(device="cuda:0", rng_mode="device", seed=1, **CLI_DEFAULTS), calls=0,
                         ms=[], bytes=0, frames=0) for k in arms}

        def call(name):
            st = state[name]
            out = os.path.join(tmp, "%dx%d_%s%d" % (W, H, name, st["calls"]))
            os.makedirs(out)
            fac = MjpegWriter if name == "mjpeg" else None
            vid = dict(video_path=out, video_writer=fac) if name != "none" else {}
            sl = SuperSloMo(model=None, auto_upsample=False, upsampling_factor=U, batch_size=BATCH, state_dicts=wts,
                            **vid)
            r = None if name == "none" else EventRenderer(
                full_scale_count=2, output_path=out, dvs_vid="dvs-video.avi", exposure_mode=ExposureMode.DURATION,
                exposure_value=0.01, video_writer=fac)
            t0 = st["calls"] * period
            st["calls"] += 1
            torch.cuda.synchronize()
            w0 = time.perf_counter()
            nf = 0
            for _, _, _, k in V2EPipeline(sl, st["em"], renderer=r).run_segments(
                    lambda p, q: src[p:q], n, clip_s, t_offset=t0, segment_pairs=a.segment):
                nf += k
            if r is not None:
                r.cleanup()
            sl.cleanup()
            torch.cuda.synchronize()
            ms = (time.perf_counter() - w0) * 1e3
            size = sum(os.path.getsize(os.path.join(out, f)) for f in os.listdir(out) if f.endswith(".avi"))
            frames = nf + (sl.numOrigVideoFramesWritten + (r.numFramesWritten if r is not None else 0))
            shutil.rmtree(out, ignore_errors=True)
            return ms, nf, size, frames

        for name in arms:                                 # warm-up
            call(name)
        for _ in range(a.rounds):
            for name in arms:
                ms, nf, size, frames = call(name)
                st = state[name]
                st["ms"].append(ms / nf)
                st["bytes"], st["frames"], st["nf"] = size, frames, nf
        sz = {}
        for name in arms:
            st, v = state[name], state[name]["ms"]
            sz[name] = dict(ms_per_frame_median=round(float(np.median(v)), 4), ms_per_frame_min=round(min(v), 4),
                            ms_per_frame_max=round(max(v), 4), interpolated_frames=st["nf"])
            if name != "none":
                sz[name].update(video_frames=st["frames"], avi_bytes=st["bytes"],
                                bytes_per_video_frame=round(st["bytes"] / max(st["frames"], 1), 1),
                                added_ms_per_frame_vs_none=round(float(np.median(v)) -
                                                                 float(np.median(state["none"]["ms"])), 4))
        # the encoder alone: one call's worth of SloMo-sized batches (U * BATCH frames), CUDA events around encode
        frames = torch.from_numpy(source_clip(H, W, U * BATCH, seed=1)).to(dev)
        w = MjpegWriter(os.path.join(tmp, "enc.avi"), H, W)
        for _ in range(3):
            w.encode(frames)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for _ in range(10):
            e0.record()
            _lib.check(w._lib.v2e_mjpeg_encode(w._enc, ctypes.c_void_p(frames.data_ptr()), frames.shape[0],
                                               ctypes.c_void_p(w._out.data_ptr()), ctypes.c_void_p(w._sizes.data_ptr()),
                                               ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        _, sizes = w.encode(frames)
        w.release()
        sz["mjpeg"]["encoder_kernel_ms_per_frame"] = round(float(np.median(times)) / frames.shape[0], 4)
        sz["mjpeg"]["encoder_batch_frames"] = int(frames.shape[0])
        sz["mjpeg"]["encoder_bytes_per_source_frame"] = round(float(sizes.mean()), 1)
        res["%dx%d" % (W, H)] = sz
    shutil.rmtree(tmp, ignore_errors=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"bench": "video", "U": U, "batch": BATCH, "pairs": a.pairs, "segment_pairs": a.segment,
                      "rounds": a.rounds, "quality": 95, "xvid": "cv2 %s" % cv2.__version__,
                      "host_cpus": os.cpu_count(), "sizes": res, "gpu": q[0] if q else "unknown"}))


if __name__ == "__main__":
    main()
