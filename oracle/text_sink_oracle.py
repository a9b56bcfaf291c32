"""TEST INFRASTRUCTURE ONLY -- restatements of the DVS text sink and of the signal / noise labels (label_signal_noise).

  text_body(events, labels)            v2ecore/output/ae_text_output.py:89-101 (the DVS text lines, plain Python
                                       formatting: Python itself prints the digits)
  aedat2_words_labeled(ev, w, h, lab)  v2ecore/output/aedat2_output.py:154-158 (noise rows OR in bit 1 << 10) on top of
                                       sinks_oracle.aedat2_words
  LabelCountingRNG, frame_labels       the labels of the rows OracleEmulator.generate_events returns: its signal rows
                                       are the rows it shuffles (one randperm(n) per iteration with n rows), its
                                       shot-noise rows are the rest, appended after them (emulator.py:866-923)

Pinned by tests/test_sinks_text.py against tests/golden/sinks_labeled.npz, whose payload the reference's own
DVSTextOutput and AEDat2Output(label_signal_noise=True) wrote (oracle/make_golden_text.py). Never imported by
v2e_b200/."""
import numpy as np

import sinks_oracle


def text_body(events, labels=None):
    """The bytes DVSTextOutput.appendEvents(events[, signnoise_label=labels]) writes (ae_text_output.py:89-101):
    '{} {} {} {}\\n'.format(t, x, y, p) per row, t the float32 timestamp as a Python float, x, y and (p + 1) / 2
    (float32) cast to int32, and ' {}'.format(int(label)) before the newline with labels."""
    ev = np.asarray(events, dtype=np.float32).reshape(-1, 4)
    t = ev[:, 0].astype(np.float64).tolist()
    x = ev[:, 1].astype(np.int32).tolist()
    y = ev[:, 2].astype(np.int32).tolist()
    p = ((ev[:, 3] + 1) / 2).astype(np.int32).tolist()
    if labels is None:
        lines = ['{} {} {} {}\n'.format(*r) for r in zip(t, x, y, p)]
    else:
        lab = [int(v) for v in np.asarray(labels).tolist()]
        lines = ['{} {} {} {} {}\n'.format(*r) for r in zip(t, x, y, p, lab)]
    return ''.join(lines).encode('ascii')


def aedat2_words_labeled(events, width, height, labels):
    """sinks_oracle.aedat2_words with AEDat2Output(label_signal_noise=True)'s noise marking: the address of every row
    whose label is 0 ORs in the special-event bit 1 << 10 (also where that bit overlaps x, at 640x480)."""
    words, n_on = sinks_oracle.aedat2_words(events, width, height)
    native = words.byteswap()
    addr = native[0::2]
    addr[np.logical_not(np.asarray(labels, bool))] |= 1 << 10       # a view: marks native's addresses
    return native.byteswap(), n_on


class LabelCountingRNG:
    """Draw source for OracleEmulator(rng=...) that passes every draw through to `rng` and counts the rows the oracle
    shuffles since the last reset: one randperm(n) per iteration with n > 0 rows. Those are the frame's signal rows
    (leak events included); the rest of the rows generate_events returns are its shot-noise rows."""

    def __init__(self, rng):
        self.rng = rng
        self.signal_rows = 0

    def normal(self, mean, std, shape):
        return self.rng.normal(mean, std, shape)

    def randn(self, shape):
        return self.rng.randn(shape)

    def rand(self, shape):
        return self.rng.rand(shape)

    def randperm(self, n):
        self.signal_rows += int(n)
        return self.rng.randperm(n)


def frame_labels(orc, frame, t_frame):
    """orc.generate_events(frame, t_frame) for an oracle built with rng=LabelCountingRNG(...). Returns (rows, labels):
    labels a bool array, True for the signal rows (first) and False for the shot-noise rows (last), or (None, None)."""
    rng = orc.rng
    assert isinstance(rng, LabelCountingRNG)
    rng.signal_rows = 0
    ev = orc.generate_events(frame, t_frame)
    if ev is None:
        return None, None
    assert rng.signal_rows <= len(ev)
    lab = np.zeros(len(ev), bool)
    lab[:rng.signal_rows] = True
    return ev, lab
