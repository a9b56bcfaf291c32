"""TEST INFRASTRUCTURE ONLY -- tests/golden/sinks_labeled.npz: event rows, signal / noise labels and the bytes the
UNMODIFIED reference writers put into files for them:
  text_*     DVSTextOutput.appendEvents (v2ecore/output/ae_text_output.py:68-101), without and with labels; the body
             after the header. The writer calls np.float, the alias numpy removed in 1.24; it is set to float for
             the run only (what the writer was written against).
  aedat2_*   AEDat2Output(label_signal_noise=True).appendEvents(ev, signnoise_label=...) (aedat2_output.py:133-188)
             for the three camera sizes; the body after the header.

    python oracle/make_golden_text.py [OUT.npz]        # needs the reference tree (ref_shim)
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "sinks_labeled.npz")


def text_events(rng):
    """Timestamps below 1e-4 (scientific notation), around it, typical clip times, and the float32 extremes; x and y
    at the corners of the 346x260, 1280x720 and 16-bit address spaces; both polarities."""
    n = 3000
    t = np.concatenate([
        rng.uniform(0.0, 1e-4, 400), 10.0 ** rng.uniform(-12, -4, 200), rng.uniform(1e-4, 1e-2, 400),
        np.sort(rng.uniform(0.0, 35.0, n - 1000 - 24)),
        [0.0, 1e-4, 9.99999974738e-05, 1.00000004749e-04, 1e-5, 0.5, 1.0, 2.0, 33.333, 1e15, 1e16, 3.0e16,
         1.4e-45, 1.17549435e-38, 3.4028235e38, 123456.789, 4.8999998398358e-05, 0.1, 0.2, 0.3, 1e-3, 10.0,
         100.0, 1e7]]).astype(np.float32)
    corners = np.array([(0, 0), (345, 259), (1279, 719), (65535, 65535), (0, 65535), (65535, 0)], np.float32)
    xy = np.stack([rng.integers(0, 1280, n), rng.integers(0, 720, n)], 1).astype(np.float32)
    xy[:len(corners)] = corners
    xy[-len(corners):] = corners
    p = rng.choice([-1.0, 1.0], n).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([t[:, None], xy, p[:, None]], 1))


def write_body(make_writer, append):
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "x")
        o = make_writer(path)
        o.file.flush()
        hdr = o.file.tell()
        append(o)
        o.file.flush()
        o.close()
        with open(path, "rb") as f:
            return f.read()[hdr:]


def main(out=OUT):
    ref_shim.load_reference()
    from v2ecore.output.ae_text_output import DVSTextOutput
    from v2ecore.output.aedat2_output import AEDat2Output
    rng = np.random.default_rng(21)
    d = {}
    ev = text_events(rng)
    lab = rng.random(len(ev)) < 0.8
    d["text_events"], d["text_labels"] = ev, lab
    had = hasattr(np, "float")
    np.float = float
    try:
        plain = write_body(lambda p: DVSTextOutput(p), lambda o: o.appendEvents(ev))
        labelled = write_body(lambda p: DVSTextOutput(p, label_signal_noise=True),
                              lambda o: o.appendEvents(ev, signnoise_label=lab))
    finally:
        if not had:
            del np.float
    d["text_body"] = np.frombuffer(plain, np.uint8)
    d["text_body_labeled"] = np.frombuffer(labelled, np.uint8)
    for (w, h) in ((346, 260), (240, 180), (640, 480)):
        n = 3000
        t = np.sort(rng.uniform(0.0, 35.0, n)).astype(np.float32)
        e = np.stack([t, rng.integers(0, w, n).astype(np.float32), rng.integers(0, h, n).astype(np.float32),
                      rng.choice([-1.0, 1.0], n).astype(np.float32)], 1)
        e[0, 1:3] = (w - 1, h - 1)           # the first address must not start with '#' (aedat2_output.py:166-172)
        e[1, 1:3] = (0, 0)
        e[2, 1:3] = (w - 1, 0)
        e[3, 1:3] = (0, h - 1)
        sl = rng.random(n) < 0.7
        body = write_body(lambda p: AEDat2Output(p, output_width=w, output_height=h, label_signal_noise=True),
                          lambda o: o.appendEvents(e, signnoise_label=sl))
        assert len(body) == 8 * n
        d["aedat2_events_%dx%d" % (w, h)] = e
        d["aedat2_labels_%dx%d" % (w, h)] = sl
        d["aedat2_body_%dx%d" % (w, h)] = np.frombuffer(body, np.uint8)
    np.savez_compressed(out, **d)
    print("%s written" % out)


if __name__ == "__main__":
    main(*sys.argv[1:2])
