"""TEST INFRASTRUCTURE ONLY -- tests/golden/sinks_aedat2.npz: event rows and the bytes the UNMODIFIED
reference writer (v2ecore/output/aedat2_output.py AEDat2Output.appendEvents) put into a file for them.

    python oracle/make_golden_sinks.py        # needs /root/reference
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


def main():
    ref_shim.load_reference()
    from v2ecore.output.aedat2_output import AEDat2Output
    rng = np.random.default_rng(12)
    d = {}
    for (w, h) in ((346, 260), (240, 180), (640, 480)):
        n = 3000
        t = np.sort(rng.uniform(0.0, 35.0, n)).astype(np.float32)      # up to 35 s: int32 microseconds
        ev = np.stack([t, rng.integers(0, w, n).astype(np.float32), rng.integers(0, h, n).astype(np.float32),
                       rng.choice([-1.0, 1.0], n).astype(np.float32)], 1)
        ev[0, 1:3] = (0, 0)
        ev[1, 1:3] = (w - 1, h - 1)
        with tempfile.TemporaryDirectory() as td:
            path = os.path.join(td, "x.aedat")
            o = AEDat2Output(path, output_width=w, output_height=h)
            hdr = o.file.tell()
            o.appendEvents(ev)
            o.file.flush()
            n_on, n_off = o.numOnEvents, o.numOffEvents
            o.close()
            body = open(path, "rb").read()[hdr:]
        assert len(body) == 8 * n
        d["events_%dx%d" % (w, h)] = ev
        d["body_%dx%d" % (w, h)] = np.frombuffer(body, np.uint8)
        d["on_off_%dx%d" % (w, h)] = np.array([n_on, n_off])
    # a clip running past 2^31 us (2147.483648 s): float32 times on both sides of it, the last ones below it and the
    # first ones at or above it, where the writer's int32 cast is out of range
    w, h = 346, 260
    lo = np.float32(2147.483648)
    edge = [np.nextafter(lo, np.float32(0), dtype=np.float32), lo, np.nextafter(lo, np.float32(1e4), dtype=np.float32)]
    t = np.sort(np.concatenate([rng.uniform(2140.0, 2160.0, 1000), rng.uniform(4294.0, 4296.0, 200),
                                rng.uniform(36000.0, 36001.0, 100)]).astype(np.float32))
    t = np.sort(np.concatenate([t, np.array(edge * 3, np.float32)]))
    n = len(t)
    ev = np.stack([t, rng.integers(0, w, n).astype(np.float32), rng.integers(0, h, n).astype(np.float32),
                   rng.choice([-1.0, 1.0], n).astype(np.float32)], 1)
    ev[0, 1:3] = (0, 0)
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "x.aedat")
        o = AEDat2Output(path, output_width=w, output_height=h)
        hdr = o.file.tell()
        o.appendEvents(ev)
        o.file.flush()
        o.close()
        body = open(path, "rb").read()[hdr:]
    assert len(body) == 8 * n
    d["events_long"] = ev
    d["body_long"] = np.frombuffer(body, np.uint8)
    np.savez_compressed(os.path.join(OUT, "sinks_aedat2.npz"), **d)
    print("sinks_aedat2.npz written")


if __name__ == "__main__":
    main()
