"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the reference's event-sink row conversions.

  h5_rows(events)        emulator.py:953-959 (uint32 rows of the HDF5 "events" dataset)
  aedat2_words(events)   v2ecore/output/aedat2_output.py:133-165 (big-endian address / timestamp words)

Out-of-range float -> integer casts are stated as rules here rather than left to numpy, whose result for them is
undefined (DESIGN.md 2):
  * AEDAT-2.0 timestamps: 1e6 * t (float32) truncated toward zero inside [-2^31, 2^31), INT32_MIN outside it and for
    NaN -- what numpy's float32 -> int32 cast gives on x86-64 at every array length, and so what the reference writes.
  * HDF5 timestamps: 1e6 * t (float32) truncated toward zero, taken mod 2^32. Inside [0, 2^32) that is numpy's cast;
    past 2^32 numpy's own result depends on the array's length, and the wrap is the port's choice.

Pinned by tests/test_sinks.py against tests/golden/sinks_aedat2.npz, whose payload the reference's own
AEDat2Output wrote (oracle/make_golden_sinks.py). Never imported by v2e_b200/."""
import numpy as np

# aedat2_output.py:38-60: (width, height) -> (yShiftBits, xShiftBits, polShiftBits); flipx = flipy = True
LAYOUTS = {(346, 260): (22, 12, 11), (240, 180): (22, 12, 11), (640, 480): (11, 1, 0)}
INT32_MIN = -2 ** 31


def trunc_int32(v):
    """float32 array -> int32 by the AEDAT-2.0 rule above."""
    v = np.asarray(v, np.float32)
    ok = (v >= np.float32(-2.0 ** 31)) & (v < np.float32(2.0 ** 31))
    return np.where(ok, np.trunc(np.where(ok, v, 0)).astype(np.float64), INT32_MIN).astype(np.int32)


def trunc_uint32_wrap(v):
    """float32 array (|v| < 2^63) -> uint32: truncated toward zero, mod 2^32."""
    v = np.asarray(v, np.float32)
    return (np.trunc(v).astype(np.float64).astype(np.int64) & 0xFFFFFFFF).astype(np.uint32)


def h5_rows(events):
    t = np.array(events, dtype=np.float32)
    t[:, 0] = t[:, 0] * 1e6
    t[t[:, 3] == -1, 3] = 0
    return trunc_uint32_wrap(t)


def aedat2_words(events, width=346, height=260):
    ys, xs, ps = LAYOUTS[(width, height)]
    t = trunc_int32(1e6 * np.asarray(events[:, 0], np.float32))
    x = (width - 1) - events[:, 1].astype(np.int32)
    y = (height - 1) - events[:, 2].astype(np.int32)
    p = ((events[:, 3] + 1) / 2).astype(np.int32)
    a = (x << xs | y << ys | p << ps)
    out = np.empty(2 * events.shape[0], dtype=np.int32)
    out[0::2] = a
    out[1::2] = t
    return out.byteswap(), int(np.count_nonzero(p))
