"""TEST INFRASTRUCTURE ONLY -- tests/golden/render_ref.npz: what the UNMODIFIED reference
EventRenderer.render_events_to_frames(..., return_frames=True) returns and writes for seeded event packets, every
exposure mode. The class runs with a DVS video open: its output folder is a temporary one, a recorder stands in for
v2ecore.renderer.video_writer and keeps every frame passed to write(), and the class writes its own frame-times file.

Per case: <name>_cfg, and per packet <name>_ev_<i> (float32 rows) and <name>_fr_<i> (the float64 frames returned);
<name>_vid, every uint8 BGR frame written to the video [k, H, W, 3], and <name>_times, the frame-times file's text.

    python oracle/make_golden_render.py        # needs /root/reference (or oracle/_ref)
"""
import os
import tempfile
import zlib

import numpy as np

import ref_shim

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "render_ref.npz")
DVS_VID = "dvs-video.avi"                                  # v2e's --dvs_vid default


def packets(seed, H, W, n_packets, n_per, dt, t0=0.0, sizes=None, gap=None, tie=None, cell=None, hot_cell=None):
    """Seeded packets of float32 rows [t, x, y, p], packet i spanning [t0 + i dt, t0 + (i + 1) dt).
    sizes: the packets' row counts (default: random in [n_per / 2, n_per)).
    gap: (a, b), fractions of dt: no row of a packet lies in [a dt, b dt) of its span.
    tie: interval; a quarter of the rows are moved onto frame boundaries, the times the reference's DURATION exposure
         starts frames at (the first row's float32 time plus k intervals, accumulated in float32).
    cell: (x0, y0, d): every row lies in the d x d cell at (x0, y0).
    hot_cell: (x0, y0, x1, y1): 40 % of the rows lie in that box instead of the default hot spot."""
    rng = np.random.default_rng(seed)
    t, out = t0, []
    for i in range(n_packets):
        n = int(sizes[i]) if sizes is not None else int(rng.integers(n_per // 2, n_per))
        u = rng.uniform(0, dt, n)
        if gap is not None:
            a, b = gap[0] * dt, gap[1] * dt
            u = np.where(u < a, u, a + (u - a) * (dt - b) / (dt - a) + (b - a))
        ts = np.sort(t + u).astype(np.float32)
        t += dt
        x = rng.integers(0, W, n); y = rng.integers(0, H, n)
        if cell is not None:
            x0, y0, d = cell
            x = x0 + rng.integers(0, d, n); y = y0 + rng.integers(0, d, n)
        elif hot_cell is not None:
            hot = rng.random(n) < 0.4
            x[hot] = rng.integers(hot_cell[0], hot_cell[2], hot.sum()); y[hot] = rng.integers(hot_cell[1], hot_cell[3], hot.sum())
        else:
            hot = rng.random(n) < 0.3                  # a hot spot, so that the +-full-scale clip engages
            x[hot] = W // 3 + rng.integers(0, 2, hot.sum()); y[hot] = H // 2
        p = np.where(rng.random(n) < 0.6, 1.0, -1.0)
        out.append(np.stack([ts, x, y, p], 1).astype(np.float32))
    if tie is not None:
        c, bounds = out[0][0, 0], []
        while c <= out[-1][-1, 0]:
            bounds.append(c)
            c = c + tie                                # float32 + Python float: float32, as the reference adds
        bounds = np.array(bounds, np.float32)
        for ev in out:
            inside = bounds[(bounds >= ev[0, 0]) & (bounds <= ev[-1, 0])]
            m = rng.random(len(ev)) < 0.25
            m[0] = False
            if len(inside):
                ev[m, 0] = rng.choice(inside, m.sum())
            ev[:] = ev[np.argsort(ev[:, 0], kind="stable")]
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
              t0=2147.47),
         # v2e's defaults (--dvs_exposure duration 0.01, --dvs_vid_full_scale 2), with rows on frame boundaries
         dict(name="v2e_default", mode="DURATION", value=0.01, H=26, W=34, fs=2, n_packets=5, n_per=1200, dt=0.035,
              area=None, tie=0.01),
         dict(name="v2e_default_t2147", mode="DURATION", value=0.01, H=26, W=34, fs=2, n_packets=4, n_per=1200,
              dt=0.035, area=None, tie=0.01, t0=2147.47),
         # no row in the middle 70 % of every packet: several empty frames per packet
         dict(name="duration_gaps", mode="DURATION", value=0.004, H=20, W=28, fs=2, n_packets=4, n_per=300, dt=0.04,
              area=None, gap=(0.15, 0.85)),
         # packets of one and two rows, between longer ones and across gaps of several intervals
         dict(name="duration_tiny", mode="DURATION", value=0.005, H=12, W=16, fs=2, n_packets=7, n_per=0, dt=0.03,
              area=None, sizes=[1, 2, 200, 2, 1, 2, 150]),
         # COUNT with event_count >= the packet's rows (n <= count + 1: no frame), and just above
         dict(name="count_short", mode="COUNT", value=500, H=16, W=20, fs=2, n_packets=8, n_per=0, dt=0.01, area=None,
              sizes=[1, 2, 499, 500, 501, 502, 1, 1200]),
         # AREA_COUNT, 30 x 21 with 8-pixel cells: the last column and row of cells are partial; 40 % of the rows in the
         # corner cell, counts carried from packet to packet
         dict(name="area_ragged", mode="AREA_COUNT", value=25, H=21, W=30, fs=2, n_packets=5, n_per=60, dt=0.01, area=8,
              hot_cell=(24, 16, 30, 21)),
         # every row in one cell: each frame but the first holds area_count - 1 new rows
         dict(name="area_one_cell_2", mode="AREA_COUNT", value=2, H=16, W=16, fs=2, n_packets=2, n_per=0, dt=0.01,
              area=4, sizes=[100, 37], cell=(4, 8, 4)),
         dict(name="area_one_cell_3", mode="AREA_COUNT", value=3, H=16, W=16, fs=2, n_packets=2, n_per=0, dt=0.01,
              area=4, sizes=[100, 40], cell=(12, 12, 4)),
         dict(name="area_one_cell_10", mode="AREA_COUNT", value=10, H=16, W=16, fs=2, n_packets=2, n_per=0, dt=0.01,
              area=4, sizes=[1000, 95], cell=(0, 0, 4)),
         # SOURCE with packets of one and two rows: a frame per packet, the one-row packet's empty
         dict(name="source_tiny", mode="SOURCE", value=0, H=12, W=16, fs=2, n_packets=5, n_per=0, dt=0.01, area=None,
              sizes=[1, 2, 300, 1, 40]),
         # a full scale above every count: no pixel clips, the frames are the exact ON - OFF counts
         dict(name="duration_noclip", mode="DURATION", value=0.01, H=16, W=24, fs=1000, n_packets=3, n_per=3000,
              dt=0.03, area=None)]

EXTRA = ("t0", "sizes", "gap", "tie", "cell", "hot_cell")


class Recorder:
    """Stands in for cv2.VideoWriter: keeps every frame written."""

    def __init__(self, *args, **kwargs):
        self.frames = []

    def write(self, frame):
        self.frames.append(np.array(frame, copy=True))

    def release(self):
        pass


def main():
    ref_shim.load_reference()
    import v2ecore.renderer as ref_renderer
    from v2ecore.renderer import EventRenderer, ExposureMode
    recorders = []

    def video_writer(*args, **kwargs):
        recorders.append(Recorder(*args, **kwargs))
        return recorders[-1]

    ref_renderer.video_writer = video_writer
    out = {"names": np.array([c["name"] for c in CASES])}
    for c in CASES:
        with tempfile.TemporaryDirectory() as d:
            r = EventRenderer(full_scale_count=c["fs"], output_path=d, dvs_vid=DVS_VID, preview=False,
                              exposure_mode=getattr(ExposureMode, c["mode"]), exposure_value=c["value"],
                              area_dimension=c["area"])
            pk = packets(zlib.crc32(c["name"].encode()) % 1000, c["H"], c["W"], c["n_packets"], c["n_per"], c["dt"],
                         **{k: c[k] for k in EXTRA if k in c})
            for i, ev in enumerate(pk):
                fr = r.render_events_to_frames(ev, height=c["H"], width=c["W"], return_frames=True)
                out["%s_ev_%d" % (c["name"], i)] = ev
                out["%s_fr_%d" % (c["name"], i)] = np.zeros((0, c["H"], c["W"])) if fr is None else fr
            r.cleanup()
            with open(os.path.join(d, "dvs-video-frame_times.txt")) as f:
                out[c["name"] + "_times"] = np.array(f.read())
        rec = recorders.pop()
        out[c["name"] + "_vid"] = np.stack(rec.frames) if rec.frames else np.zeros((0, c["H"], c["W"], 3), np.uint8)
        out[c["name"] + "_cfg"] = np.array([{"DURATION": 1, "COUNT": 2, "AREA_COUNT": 3, "SOURCE": 4}[c["mode"]], c["value"], c["H"],
                                            c["W"], c["fs"], c["n_packets"], c["area"] or 0], dtype=np.float64)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
