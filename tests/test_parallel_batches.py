"""CPU tests of the pair-sharded auto-upsampling plumbing: how a clip's SloMo batches are dealt to ranks
(parallel.batch_pair_range) and how the clip's interpTimes are rebuilt from the per-batch U's (slomo.clip_times)."""
import numpy as np
import pytest

from v2e_b200.parallel import batch_pair_range, pair_range
from v2e_b200.slomo import clip_times


@pytest.mark.parametrize("n_pairs", [1, 2, 5, 7, 8, 17, 64])
@pytest.mark.parametrize("batch_size", [1, 2, 3, 8])
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_batch_pair_range_deals_whole_batches(n_pairs, batch_size, world):
    n_batches = -(-n_pairs // batch_size)
    if n_batches < world:
        for r in range(world):
            with pytest.raises(ValueError):
                batch_pair_range(n_pairs, batch_size, r, world)
        return
    ranges = [batch_pair_range(n_pairs, batch_size, r, world) for r in range(world)]
    # every pair exactly once, in rank order
    assert ranges[0][0] == 0 and ranges[-1][1] == n_pairs
    for (a0, a1), (b0, b1) in zip(ranges, ranges[1:]):
        assert a1 == b0
    for r, (p0, p1) in enumerate(ranges):
        assert p1 > p0                              # every rank has at least one batch
        assert p0 % batch_size == 0                 # starts on a batch boundary of the clip
        if r < world - 1:
            assert (p1 - p0) % batch_size == 0      # whole batches: only the last rank has the short one
    # the batches are spread as evenly as pair_range spreads pairs
    counts = [-(-(p1 - p0) // batch_size) for p0, p1 in ranges]
    assert counts == [b - a for a, b in (pair_range(n_batches, r, world) for r in range(world))]


def test_batch_pair_range_rejects_bad_arguments():
    with pytest.raises(ValueError):
        batch_pair_range(10, 2, 2, 2)
    with pytest.raises(ValueError):
        batch_pair_range(10, 0, 0, 2)


def _batches_formula(ups, n_pairs, batch_size):
    """SuperSloMo._batches / interpolate_frames (slomo.py:330-400) without the network: per batch the times
    in_ctr + arange(U*b) / U, concatenated, and the mean U."""
    bs = max(1, min(int(batch_size), n_pairs))
    times, used, in_ctr, i = [], [], 0, 0
    while in_ctr < n_pairs:
        b = min(bs, n_pairs - in_ctr)
        U = ups[i]
        times.append(in_ctr + np.array(range(U * b)) * (1 / U))
        used.append(U)
        in_ctr += b
        i += 1
    return np.concatenate(times), sum(used) / len(used)


@pytest.mark.parametrize("seed", range(12))
def test_clip_times_equals_the_single_gpu_formula(seed):
    rng = np.random.default_rng(seed)
    n_pairs = int(rng.integers(1, 40))
    batch_size = int(rng.integers(1, 9))
    n_batches = -(-n_pairs // min(batch_size, n_pairs))
    ups = [int(u) for u in rng.integers(2, 40, n_batches)]
    want_t, want_avg = _batches_formula(ups, n_pairs, batch_size)
    got_t, got_avg = clip_times(ups, n_pairs, batch_size)
    assert got_t.dtype == want_t.dtype and np.array_equal(got_t, want_t)
    assert got_avg == want_avg
    # the time scaling of v2e.py:794-797 then gives identical seconds
    f = 0.37 / (np.max(want_t) - np.min(want_t)) if len(want_t) > 1 else 1.0
    assert np.array_equal(0.1 + f * got_t, 0.1 + f * want_t)


def test_clip_times_needs_one_u_per_batch():
    with pytest.raises(ValueError):
        clip_times([2, 3], 7, 2)
