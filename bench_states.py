"""Cost of show_dvs_model_state on the multi-frame pixel-model path: 1280x720, CLI defaults, device RNG, 64-frame
chunks, timed with v2e_emu_time_fused (K repetitions of one chunk between one CUDA-event pair) with no state shown,
one (diff_frame) and all six that exist there, the settings alternated in one process. Prints one JSON line with the
card's name, power limit and max SM clock read in the same run. Writes nothing."""
import argparse
import ctypes
import json
import subprocess

import numpy as np
import torch

from v2e_b200 import EventEmulator, _lib

CLI = dict(cutoff_hz=300, leak_rate_hz=0.01, shot_noise_rate_hz=0.001, refractory_period_s=0.0005, sigma_thres=0.03)
SETTINGS = {"off": None, "one": ["diff_frame"], "six": ["all"]}


def clip(H, W, T, seed):
    """A smooth texture translating 1 px per frame (a clip the multi-frame kernels accept whole)."""
    from scipy.ndimage import gaussian_filter
    big = gaussian_filter(np.random.default_rng(seed).uniform(0, 255, (H + 8, W + T + 8)), 4)
    big = (big - big.min()) / (big.max() - big.min()) * 200 + 20
    return np.stack([big[4:4 + H, k:k + W] for k in range(T)]).round().astype(np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_states.py needs a CUDA device")
    H, W, T = 720, 1280, 64
    fr = torch.from_numpy(clip(H, W, 2 * T + 1, 3)).cuda()
    ts = np.arange(2 * T + 1) / 300.0
    ems = {}
    for name, show in SETTINGS.items():
        em = EventEmulator(device="cuda:0", rng_mode="device", seed=5, max_frames_per_step=T,
                           show_dvs_model_state=show, **CLI)
        em.event_rows_hint = 16 * 1024 * 1024
        em.generate_events_batch(fr[:T + 1], ts[:T + 1], return_device=True)
        ems[name] = em
    tt = (ctypes.c_double * T)(*ts[T + 1:])
    chunk = fr[T + 1:]
    res = {k: [] for k in SETTINGS}
    upd = {k: [] for k in SETTINGS}
    for _ in range(a.rounds):
        for name, em in ems.items():
            uc, uu = ctypes.c_float(0), ctypes.c_float(0)
            _lib.check(em._lib.v2e_emu_time_fused(em._h, ctypes.c_void_p(chunk.data_ptr()), 0, T, tt,
                                                  float(em.t_previous), ctypes.c_void_p(em._ev_dev.data_ptr()),
                                                  em._ev_dev.shape[0], a.reps, ctypes.byref(uc), ctypes.byref(uu),
                                                  em._stream()))
            res[name].append(round(uc.value / T, 3))
            upd[name].append(round(uu.value / T, 3))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    floor_us = 6 * H * W / 3.35e12 * 1e6
    print(json.dumps({"bench": "model_states", "frame": [W, H], "chunk_frames": T, "reps": a.reps,
                      "us_per_frame_chunk": res, "us_per_frame_update_kernel": upd,
                      "six_state_write_floor_us": round(floor_us, 3), "gpu": q[0] if q else "unknown"}))
    for em in ems.values():
        em.cleanup()


if __name__ == "__main__":
    main()
