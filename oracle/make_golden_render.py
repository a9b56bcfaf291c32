"""TEST INFRASTRUCTURE ONLY -- tests/golden/render_ref.npz: frames returned by the UNMODIFIED reference
EventRenderer.render_events_to_frames(..., return_frames=True) for seeded event packets, every exposure mode.

    python oracle/make_golden_render.py        # needs /root/reference (or oracle/_ref)
"""
import os
import zlib

import numpy as np

import ref_shim

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "render_ref.npz")


def packets(seed, H, W, n_packets, n_per, dt, t0=0.0):
    rng = np.random.default_rng(seed)
    t, out = t0, []
    for _ in range(n_packets):
        n = int(rng.integers(n_per // 2, n_per))
        ts = np.sort(t + rng.uniform(0, dt, n)).astype(np.float32)
        t += dt
        x = rng.integers(0, W, n); y = rng.integers(0, H, n)
        hot = rng.random(n) < 0.3                      # a hot spot, so that the +-full-scale clip engages
        x[hot] = W // 3 + rng.integers(0, 2, hot.sum()); y[hot] = H // 2
        p = np.where(rng.random(n) < 0.6, 1.0, -1.0)
        out.append(np.stack([ts, x, y, p], 1).astype(np.float32))
    return out


CASES = [dict(name="duration", mode="DURATION", value=0.004, H=24, W=32, fs=3, n_packets=5, n_per=900, dt=0.01, area=None),
         dict(name="duration_fs1", mode="DURATION", value=1 / 300.0, H=20, W=20, fs=1, n_packets=3, n_per=400, dt=0.005, area=None),
         dict(name="count", mode="COUNT", value=250, H=24, W=32, fs=3, n_packets=4, n_per=900, dt=0.01, area=None),
         dict(name="source", mode="SOURCE", value=0, H=16, W=24, fs=2, n_packets=4, n_per=300, dt=0.01, area=None),
         dict(name="area_count", mode="AREA_COUNT", value=40, H=24, W=32, fs=3, n_packets=3, n_per=900, dt=0.01, area=8),
         # packets of a long clip, past 2^31 us: float32 timestamps 2.4e-4 s apart, frame start times accumulated in
         # float32 by the reference (renderer.py:208, 316)
         dict(name="duration_long", mode="DURATION", value=1 / 300.0, H=24, W=32, fs=3, n_packets=5, n_per=900,
              dt=0.01, area=None, t0=2147.47),
         dict(name="count_long", mode="COUNT", value=250, H=24, W=32, fs=3, n_packets=4, n_per=900, dt=0.01, area=None,
              t0=2147.47)]


def main():
    ref_shim.load_reference()
    from v2ecore.renderer import EventRenderer, ExposureMode
    out = {"names": np.array([c["name"] for c in CASES])}
    for c in CASES:
        r = EventRenderer(full_scale_count=c["fs"], output_path=None, dvs_vid=None, preview=False,
                          exposure_mode=getattr(ExposureMode, c["mode"]), exposure_value=c["value"],
                          area_dimension=c["area"])
        pk = packets(zlib.crc32(c["name"].encode()) % 1000, c["H"], c["W"], c["n_packets"], c["n_per"], c["dt"],
                     c.get("t0", 0.0))
        for i, ev in enumerate(pk):
            fr = r.render_events_to_frames(ev, height=c["H"], width=c["W"], return_frames=True)
            out["%s_ev_%d" % (c["name"], i)] = ev
            out["%s_fr_%d" % (c["name"], i)] = np.zeros((0, c["H"], c["W"])) if fr is None else fr
        out[c["name"] + "_cfg"] = np.array([{"DURATION": 1, "COUNT": 2, "AREA_COUNT": 3, "SOURCE": 4}[c["mode"]], c["value"], c["H"],
                                            c["W"], c["fs"], c["n_packets"], c["area"] or 0], dtype=np.float64)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
