"""CPU: the row orders of EventEmulator(row_order=...) as oracle/row_order.py states them -- the ROW_ORDER Philox
stream's layout, the uniformity of the shuffled order, the canonical order against OracleEmulator(shuffle=False), and
the merge of row bands (v2e_b200.parallel.merge_by_key) against the whole frame's order."""
import itertools

import numpy as np
import pytest

import philox
import row_order
from helpers import TapeRNG, load_golden

SEED = 1234


# ---- shared with tests/test_row_order_gpu.py -------------------------------------------------------------------
def oracle_clip(orc, frames, ts, rng=None):
    """Runs OracleEmulator(shuffle=False) over a clip. Returns (rows, offsets, iter_counts, n_shot): the rows as the
    oracle returns them (its canonical order, NOT re-sorted), and per frame the signal rows of every iteration and the
    shot rows. The oracle reports neither, so: the signal rows of a frame are those its randperm calls cover, and
    iteration i is stamped linspace(t_prev + dt / max_n, t_frame, max_n)[i] (emulator.py:792-796) -- the clip must not
    give two iterations of a frame the same float32 time."""
    from emu_oracle import lib
    L = lib()
    drawn = []
    inner = orc.rng.randperm

    def randperm(n):
        drawn.append(int(n))
        return inner(n)
    orc.rng.randperm = randperm
    rows, offsets, iter_counts, n_shot = [], [0], [], []
    for k, (f, t) in enumerate(zip(frames, ts)):
        if rng is not None:
            rng.frame = k
        del drawn[:]
        tp = float(orc.t_previous)
        ev = orc.generate_events(f, float(t))
        ev = np.zeros((0, 4), np.float32) if ev is None else ev
        n_sig, m = sum(drawn), orc.last_max_n if k else 0
        sig_t = ev[:n_sig, 0]
        stamps = np.array([L.oracle_linspace_f32(tp + (float(t) - tp) / m, float(t), m, i) for i in range(m)], np.float32)
        assert len(set(stamps.tolist())) == m, "frame %d: iterations share a float32 timestamp" % k
        counts = np.array([int(np.sum(sig_t == s)) for s in stamps], np.int64)
        assert counts.sum() == n_sig and np.all(np.diff(sig_t) >= 0), "frame %d" % k
        rows.append(ev)
        offsets.append(offsets[-1] + len(ev))
        iter_counts.append(counts)
        n_shot.append(len(ev) - n_sig)
    return np.concatenate(rows), np.asarray(offsets, np.int64), iter_counts, np.asarray(n_shot, np.int64)


def scramble(rows, offsets, iter_counts, n_shot, seed=0):
    """The same rows with every iteration's rows and every shot block permuted: what an unordered emission may return."""
    g = np.random.default_rng(seed)
    out = rows.copy()
    for f in range(len(offsets) - 1):
        a = int(offsets[f])
        for c in list(iter_counts[f]) + [int(n_shot[f])]:
            out[a:a + c] = rows[a:a + c][g.permutation(int(c))]
            a += int(c)
    return out


# ---- 1. key layout ------------------------------------------------------------------------------------------
def test_row_order_stream_cannot_collide_with_the_noise_streams():
    """Counter word 3 is the stream's tag in all four streams; the ROW_ORDER tag differs from the other three, so no
    (counter, key) pair of it equals one of theirs whatever the other words hold."""
    tags = {philox.TAG_LEAK, philox.TAG_SHOT, philox.TAG_PR}
    assert row_order.TAG_ROW_ORDER == 0x726f7264 and row_order.TAG_ROW_ORDER not in tags
    W, H = 1280, 720
    corners = [(0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1)]
    seen = set()
    for fi, it, (x, y), p in itertools.product((0, 1, 2 ** 20), (0, 30), corners, (1.0, -1.0)):
        c = row_order.counter_words(fi, it, np.array([x]), np.array([y]), np.array([p]), W)
        words = tuple(int(w[0]) for w in c)
        assert words == (2 * (y * W + x) + (p < 0), fi, it, 0x726f7264)
        # the three noise streams count (quad, frame index, stream number, tag): the tag word alone tells them apart
        for stream, tag in enumerate((philox.TAG_LEAK, philox.TAG_SHOT, philox.TAG_PR)):
            assert words != (words[0], fi, stream, tag)
        k = int(row_order.keys(SEED, fi, it, np.array([x]), np.array([y]), np.array([p]), W)[0])
        w = philox.philox4x32(tuple(np.array([v], np.uint64) for v in words), philox.seed_key(SEED))
        assert k == (int(w[0][0]) << 32) | int(w[1][0])
        seen.add(k)
    assert len(seen) == 3 * 2 * 4 * 2                 # every (frame, iteration, pixel, polarity) has its own key
    # and the key is not what the noise streams draw from the same first three words
    other = philox.philox4x32(tuple(np.array([v], np.uint64) for v in (5, 7, 0, philox.TAG_LEAK)), philox.seed_key(SEED))
    mine = philox.philox4x32(tuple(np.array([v], np.uint64) for v in (5, 7, 0, row_order.TAG_ROW_ORDER)),
                             philox.seed_key(SEED))
    assert [int(a[0]) for a in other] != [int(a[0]) for a in mine]


# ---- 2. uniformity ------------------------------------------------------------------------------------------
def test_shuffled_order_of_four_rows_is_uniform_over_the_24_permutations():
    W = 346
    x, y, p = np.array([3, 200, 77, 345]), np.array([0, 12, 259, 100]), np.array([1.0, -1.0, 1.0, -1.0])
    fi, it = np.meshgrid(np.arange(800), np.arange(30), indexing="ij")
    k = row_order.keys(SEED, fi.reshape(-1, 1), it.reshape(-1, 1), x[None], y[None], p[None], W)      # [24000, 4]
    assert k.shape == (24000, 4)
    perms = np.argsort(k, axis=1)
    code = perms[:, 0] * 64 + perms[:, 1] * 16 + perms[:, 2] * 4 + perms[:, 3]
    vals, counts = np.unique(code, return_counts=True)
    assert len(vals) == 24
    sigma = np.sqrt(24000 * (1 / 24) * (23 / 24))
    assert np.all(np.abs(counts - 1000) <= 5 * sigma), counts


def _run_lengths(pol):
    """Lengths of the runs of equal polarity in each row of pol [K, n] as one flat array, and runs per row."""
    change = np.diff(pol.astype(np.int8), axis=1) != 0
    runs_per_row = change.sum(1) + 1
    lengths = []
    for row in change:
        edges = np.concatenate([[-1], np.flatnonzero(row), [len(row)]])
        lengths.append(np.diff(edges))
    return np.concatenate(lengths), runs_per_row


def test_shuffled_order_of_1000_rows_mixes_like_a_random_permutation():
    """n = 1000 (500 ON rows then 500 OFF rows in canonical order) over 300 (frame, iteration) pairs, against numpy's
    permutation: mean displacement |new place - old place|, the number of ON/OFF runs, and how many runs have length
    1, 2, 3, 4 and >= 5 -- each within 5 sigma of the difference of the two samples."""
    W, n, K = 1280, 1000, 300
    g = np.random.default_rng(7)
    pix = np.sort(g.choice(1280 * 720, n // 2, replace=False))
    x, y = np.tile(pix % W, 2), np.tile(pix // W, 2)
    p = np.repeat([1.0, -1.0], n // 2)
    fi, it = np.meshgrid(np.arange(K // 3), np.arange(3), indexing="ij")
    k = row_order.keys(SEED, fi.reshape(-1, 1), it.reshape(-1, 1), x[None], y[None], p[None], W)
    mine = np.argsort(k, axis=1)                       # mine[s, j] = canonical index of the row at place j
    ref = np.stack([g.permutation(n) for _ in range(K)])

    def stats(perm):
        disp = np.abs(perm - np.arange(n)[None]).mean(1)
        lengths, runs = _run_lengths(perm >= n // 2)
        hist = np.array([np.sum(lengths == 1), np.sum(lengths == 2), np.sum(lengths == 3), np.sum(lengths == 4),
                         np.sum(lengths >= 5)])
        return disp, runs, hist
    d1, r1, h1 = stats(mine)
    d2, r2, h2 = stats(ref)
    for a, b in ((d1, d2), (r1, r2)):
        assert abs(a.mean() - b.mean()) <= 5 * np.sqrt(a.var(ddof=1) / K + b.var(ddof=1) / K), (a.mean(), b.mean())
    assert np.all(np.abs(h1 - h2) <= 5 * np.sqrt(h1 + h2)), (h1, h2)
    assert abs(d1.mean() - (n * n - 1) / (3 * n)) < 5 * d1.std(ddof=1) / np.sqrt(K)      # E|i - pi(i)| of a uniform pi


# ---- 3. canonical = the oracle's order before randperm ---------------------------------------------------------
@pytest.mark.parametrize("name", ["emu_cli_noisy", "emu_ragged_13x37"])
def test_canonical_order_is_the_oracles_unshuffled_order(name):
    from emu_oracle import OracleEmulator
    g = load_golden(name)
    orc = OracleEmulator(rng=TapeRNG(g["tape"]), shuffle=False, **g["kwargs"])
    rows, offs, iters, n_shot = oracle_clip(orc, g["frames"], [float(t) for t in g["times"]])
    assert len(rows) > 0 and sum(len(c) for c in iters) > 0
    W = g["frames"].shape[2]
    mixed = scramble(rows, offs, iters, n_shot, seed=3)
    assert not np.array_equal(mixed, rows)
    got = row_order.order_rows(mixed, offs, iters, n_shot, "canonical", W=W)
    assert got.tobytes() == rows.tobytes()
    # the shuffled order holds the same rows per iteration, ON and OFF mixed, shot rows where they were
    sh = row_order.order_rows(mixed, offs, iters, n_shot, "shuffled", seed=SEED, W=W)
    assert not np.array_equal(sh, rows)
    for f in range(len(offs) - 1):
        a, b = int(offs[f]), int(offs[f + 1])
        s = b - int(n_shot[f])
        assert np.array_equal(sh[s:b], rows[s:b]) and np.array_equal(sh[a:b, 0], rows[a:b, 0])


# ---- 4. bands merge into the whole frame's order -------------------------------------------------------------
def _synthetic_clip(H, W, T, seed):
    g = np.random.default_rng(seed)
    rows, offs, iters, n_shot = [], [0], [], []
    for f in range(T):
        m = int(g.integers(1, 4))
        stamps = (np.float32(f) + np.arange(1, m + 1, dtype=np.float32) / np.float32(m)) * np.float32(1e-3)
        fr, counts = [], []
        for it in range(m):
            pix = np.flatnonzero(g.random(H * W) < 0.3 / (it + 1))
            pol = np.where(g.random(len(pix)) < 0.5, 1.0, -1.0)
            blk = np.stack([np.full(len(pix), stamps[it]), pix % W, pix // W, pol], 1).astype(np.float32)
            fr.append(blk)
            counts.append(len(blk))
        shot = []
        for pol in (1.0, -1.0):
            pix = np.flatnonzero(g.random(H * W) < 0.02)
            shot.append(np.stack([np.full(len(pix), stamps[-1]), pix % W, pix // W, np.full(len(pix), pol)], 1))
        shot = np.concatenate(shot).astype(np.float32)
        rows += fr + [shot]
        offs.append(offs[-1] + sum(counts) + len(shot))
        iters.append(np.asarray(counts, np.int64))
        n_shot.append(len(shot))
    return np.concatenate(rows), np.asarray(offs, np.int64), iters, np.asarray(n_shot, np.int64)


@pytest.mark.parametrize("mode", ["canonical", "shuffled"])
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("size", [(13, 37), (120, 176)])
def test_bands_ordered_by_whole_frame_keys_merge_into_the_whole_frames_order(size, world, mode):
    from v2e_b200.parallel import merge_by_key, row_band
    H, W = size
    T = 4
    rows, offs, iters, n_shot = _synthetic_clip(H, W, T, seed=H + world)
    whole = row_order.order_rows(scramble(rows, offs, iters, n_shot, 1), offs, iters, n_shot, mode, seed=SEED, W=W)
    streams, keys, boffs, bshot = [], [], [], []
    for r in range(world):
        y0, y1 = row_band(H, r, world)
        mine = (rows[:, 2] >= y0) & (rows[:, 2] < y1)
        b_rows, b_offs, b_iters, b_shot = [], [0], [], []
        for f in range(T):
            a = int(offs[f])
            cs = []
            for c in list(iters[f]) + [int(n_shot[f])]:
                blk = rows[a:a + c][mine[a:a + c]]
                b_rows.append(blk)
                cs.append(len(blk))
                a += int(c)
            b_iters.append(np.asarray(cs[:-1], np.int64))
            b_shot.append(cs[-1])
            b_offs.append(b_offs[-1] + sum(cs))
        b_rows = scramble(np.concatenate(b_rows), b_offs, b_iters, b_shot, seed=r)
        o, k = row_order.order_rows(b_rows, b_offs, b_iters, b_shot, mode, seed=SEED, W=W, return_keys=True)
        streams.append(o); keys.append(k); boffs.append(np.asarray(b_offs)); bshot.append(np.asarray(b_shot))
    merged, moffs = merge_by_key(streams, keys, boffs, bshot)
    assert np.array_equal(moffs, offs)
    assert merged.tobytes() == whole.tobytes()
    # each band is a subsequence of the whole order
    for s in streams:
        j = 0
        for r in whole:
            if j < len(s) and r.tobytes() == s[j].tobytes():
                j += 1
        assert j == len(s)
