"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/emu_cs32_*.npz by running the UNMODIFIED reference
(device="cpu") with the centre-surround model on a float32 photoreceptor state (cutoff_hz = 0: low_pass_filter returns
the float32 log frame, emulator_utils.py:75-77, and the surround is its clone, emulator.py:1063, so every op of the
Euler step is float32).

    python oracle/make_golden_cs32.py       # needs /root/reference

Same fixture contents as oracle/make_golden.py (frames, kwargs, the tape of every random draw, rows in the reference's
order, final state, cs_steps_taken); a fixture of a run that applied a --dvs_params preset after construction
(v2e.py:565-570) also holds "dvs_params". Each clip starts with a uniform pair, so that frame 1's iteration stops after
one step, and ends with a static pair. Not in tests/helpers.EMU_GOLDENS: tests/test_*_csdvs_f32.py load them.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402
from make_golden import OUT, save_case, texture_frames  # noqa: E402


def clip(H, W, seed, block, speed, times_moving, hold, lo=0):
    """uniform, uniform, T moving frames (grey levels lo .. 255 - lo), the last one held for `hold` seconds"""
    mov = texture_frames(H, W, len(times_moving), seed=seed, speed=speed, block=block)
    mov = (lo + mov.astype(np.int32) * (256 - 2 * lo) // 256).astype(np.uint8)
    grey = np.full((1, H, W), 128, np.uint8)
    frames = np.concatenate([grey, grey, mov, mov[-1:]])
    t0 = 1e-3
    times = np.concatenate([[0.0, t0], t0 + np.asarray(times_moving), [t0 + times_moving[-1] + hold]])
    return frames, times


def with_preset(emu_mod, preset):
    """emu_mod whose EventEmulator applies set_dvs_params(preset) right after construction, as v2e.py:565-570 does"""
    def make(*a, **k):
        em = emu_mod.EventEmulator(*a, **k)
        em.set_dvs_params(preset)
        return em
    return types.SimpleNamespace(EventEmulator=make, compute_photoreceptor_noise_voltage=None)


def main():
    emu_mod, _, _, _ = ref_shim.load_reference()
    # .idea/runConfigurations/CSDVS_test.xml: --pos_thres=.15 --neg_thres=.15 --sigma_thres=0 --cutoff=0 --leak_rate=0
    # --shot=0 --cs_lambda_pixels=15 --cs_tau_p_ms=20; 120x176 is above the float32 conv2d summation-order switch
    fr, ts = clip(120, 176, seed=21, block=8, speed=1.0, times_moving=np.arange(1, 3) / 1500., hold=4e-3, lo=96)
    save_case("emu_cs32_120x176", emu_mod,
              dict(pos_thres=0.15, neg_thres=0.15, sigma_thres=0, cutoff_hz=0, leak_rate_hz=0, shot_noise_rate_hz=0,
                   cs_lambda_pixels=15, cs_tau_p_ms=20), fr, ts)
    # 37x53: below the switch with a 9-pixel tail; per-pixel thresholds, leak, shot noise and the refractory filter
    fr, ts = clip(37, 53, seed=23, block=1, speed=3.0, times_moving=np.arange(1, 5) * 2e-4, hold=1e-3)
    save_case("emu_cs32_37x53", emu_mod,
              dict(cs_lambda_pixels=3, cs_tau_p_ms=0.5, cutoff_hz=0, leak_rate_hz=0.1, shot_noise_rate_hz=2.0,
                   refractory_period_s=1e-4, sigma_thres=0.03, pos_thres=0.3, neg_thres=0.3), fr, ts)
    # SCIDVS in front of the change amplifier (photoreceptor = 2 * highpass, float32)
    fr, ts = clip(20, 36, seed=25, block=2, speed=1.0, times_moving=np.arange(1, 4) * 1e-4, hold=5e-4)
    save_case("emu_cs32_scidvs", emu_mod,
              dict(scidvs=True, cs_lambda_pixels=10, cs_tau_p_ms=0.5, cutoff_hz=0, leak_rate_hz=0.1,
                   shot_noise_rate_hz=0, sigma_thres=0.03, pos_thres=0.3, neg_thres=0.3), fr, ts)
    # .idea/runConfigurations/gradients_csdvs.xml: --leak_rate=0 --shot=0 --cutoff_hz=300 --sigma_thr=.05
    # --cs_lambda=5 --cs_tau_p_ms=10 --dvs_params clean; the preset sets cutoff_hz = 0 (v2e.py:565-570)
    fr, ts = clip(30, 44, seed=27, block=4, speed=1.0, times_moving=np.arange(1, 4) * 5e-4, hold=3e-3)
    save_case("emu_cs32_clean", with_preset(emu_mod, "clean"),
              dict(leak_rate_hz=0, shot_noise_rate_hz=0, cutoff_hz=300, sigma_thres=0.05, cs_lambda_pixels=5,
                   cs_tau_p_ms=10), fr, ts)
    path = os.path.join(OUT, "emu_cs32_clean.npz")
    with np.load(path) as z:
        d = {k: z[k] for k in z.files}
    d["dvs_params"] = np.array("clean")
    np.savez_compressed(path, **d)


if __name__ == "__main__":
    main()
