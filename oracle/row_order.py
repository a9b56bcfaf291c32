"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the row orders of EventEmulator(row_order=...).

Written from the rule, independently of v2e_b200/csrc/order.cuh. Per frame the rows are iteration-major, shot noise
last. "canonical": inside an iteration ON rows then OFF rows, each by pixel index y*W + x; shot ON, then shot OFF, each
by pixel -- the reference's order before its randperm (emulator.py:861-870, 906-919), OracleEmulator(shuffle=False)'s.
"shuffled": the ON and OFF rows of one (frame, iteration) in ascending order of

    key = words 0, 1 (word 0 high) of Philox4x32-7(counter = (2*pixel + (p < 0), Philox frame index, iteration, "rord"),
                                                   key = (seed low word, seed high word))

ties broken by 2*pixel + (p < 0); shot rows as in "canonical". The fourth counter word is the stream's tag, as in the
leak / shot / photoreceptor streams of philox.py ("leak", "shot", "prnz"): it alone keeps the four streams' counters
apart, whatever the other three words hold. pixel is the index in the WHOLE frame (global y), frame k >= 1 of a clip
has Philox frame index k - 1.
"""
import numpy as np

import philox

TAG_ROW_ORDER = 0x726f7264          # "rord"


def counter_words(frame_index, iteration, x, y, p, W):
    """The Philox counter (4 arrays of 32-bit words) of the ROW_ORDER stream for rows (x, y, p); frame_index and
    iteration are scalars or arrays that broadcast against them."""
    x, y, p = (np.asarray(a) for a in (x, y, p))
    ident = 2 * (y.astype(np.uint64) * np.uint64(W) + x.astype(np.uint64)) + (p < 0).astype(np.uint64)
    assert np.all(ident < 2 ** 32)
    frame_index = (np.asarray(frame_index, np.int64) & 0xFFFFFFFF).astype(np.uint64)
    return tuple(np.broadcast_arrays(ident, frame_index, np.asarray(iteration, np.uint64), np.uint64(TAG_ROW_ORDER)))


def keys(seed, frame_index, iteration, x, y, p, W):
    """uint64 sort keys of the shuffled order."""
    w = philox.philox4x32(counter_words(frame_index, iteration, x, y, p, W), philox.seed_key(seed))
    return (w[0].astype(np.uint64) << np.uint64(32)) | w[1].astype(np.uint64)


def pixel_keys(x, y, p, W):
    """uint64 sort keys of the canonical order (and of shot rows in both): (p < 0) << 32 | pixel."""
    x, y, p = (np.asarray(a) for a in (x, y, p))
    return ((p < 0).astype(np.uint64) << np.uint64(32)) | (y.astype(np.uint64) * np.uint64(W) + x.astype(np.uint64))


def row_keys(rows, mode, seed, frame_index, iteration, W):
    """Keys of float32 rows [t, x, y, p] of one segment: iteration None = shot rows."""
    x, y, p = rows[:, 1].astype(np.int64), rows[:, 2].astype(np.int64), rows[:, 3]
    if mode == "canonical" or iteration is None:
        return pixel_keys(x, y, p, W)
    return keys(seed, frame_index, iteration, x, y, p, W)


def order_rows(rows, offsets, iter_counts, n_shot, mode, seed=0, W=None, first_frame_index=-1, return_keys=False):
    """rows [N, 4] float32 with frame f at rows[offsets[f]:offsets[f + 1]], iteration-major, its last n_shot[f] rows
    shot noise; iter_counts[f][i] = signal rows of iteration i of frame f (zeros allowed). Rows inside an iteration
    and inside the shot block may come in any order. Frame f has Philox frame index first_frame_index + f (frame 0 of
    a clip emits nothing: -1 for a clip given whole). Returns the rows in `mode` order (and their keys)."""
    assert mode in ("canonical", "shuffled") and W is not None
    out, out_keys = np.empty_like(rows), np.zeros(len(rows), np.uint64)
    for f in range(len(offsets) - 1):
        a, b = int(offsets[f]), int(offsets[f + 1])
        segs = [(it, int(c)) for it, c in enumerate(iter_counts[f])] + [(None, int(n_shot[f]))]
        assert sum(c for _, c in segs) == b - a, "frame %d: iteration counts and shot rows do not add up" % f
        for it, c in segs:
            blk = rows[a:a + c]
            k = row_keys(blk, mode, seed, first_frame_index + f, it, W)
            ident = 2 * (blk[:, 2].astype(np.int64) * W + blk[:, 1].astype(np.int64)) + (blk[:, 3] < 0)
            o = np.lexsort((ident, k))
            out[a:a + c], out_keys[a:a + c] = blk[o], k[o]
            a += c
    return (out, out_keys) if return_keys else out
