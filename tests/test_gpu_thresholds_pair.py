"""
gb_thresholds_pair / gb_thresholds_pair_f64 against two gb_thresholds calls, bit for bit, and against pandas'
rolling(window).min().max(): windows from 1 to longer than the jobs, ragged jobs in one launch, NaN patterns, zeros of both signs,
1 and 256 tags, and more jobs than one grid dimension holds.
"""
import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("needs an H100")
    import __graft_entry__ as ge

    ge.build()
    return t


@pytest.fixture(scope="module")
def engine(torch):
    from gordo_components_b200 import engine as e

    return e


def _scores(rng, rows, n_out, dtype):
    """Non-negative scores with scattered NaNs, a NaN run of 300 rows, an all-NaN column, zeros and -0.0."""
    tag = rng.random((rows, n_out)) ** 3
    tag[rng.random(tag.shape) < 0.01] = np.nan
    tag[rng.random(tag.shape) < 0.03] = 0.0
    tag[rng.random(tag.shape) < 0.03] = -0.0
    if rows > 600:
        tag[200:500, n_out // 2] = np.nan
    if n_out > 1:
        tag[:, 0] = np.nan
    tot = rng.random(rows) ** 2
    tot[rng.random(rows) < 0.01] = np.nan
    tot[rng.random(rows) < 0.03] = -0.0
    return tag.astype(dtype), tot.astype(dtype)


def _case(torch, engine, rng, lengths, n_out, dtype):
    """Ragged jobs: slot, output row and job index all differ; rows between the jobs hold values no job may read."""
    lengths = np.asarray(lengths, dtype=np.int64)
    n = len(lengths)
    gap = 3
    order = rng.permutation(n)  # job i's rows sit at position order[i] of the layout
    starts = np.zeros(n, dtype=np.int64)
    pos = 0
    for i in np.argsort(order):
        starts[i] = pos + gap
        pos += gap + lengths[i]
    rows = pos + gap
    tag, tot = _scores(rng, rows, n_out, dtype)
    slots = rng.permutation(n + 2)[:n]  # two slots no job covers
    jobs = engine.jobs_to_device(engine.make_jobs(slots, lengths, np.zeros(n, dtype=np.int64), starts), "cuda")
    td, sd = torch.from_numpy(tag).cuda(), torch.from_numpy(tot).cuda()
    return jobs, n, int(lengths.max()), td, sd, n + 2, (tag, tot, slots, starts, lengths)


def _bits(torch, t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int64).cpu()


def _assert_pair(torch, engine, jobs, n, max_rows, td, sd, n_out, n_slots, w0, w1):
    got = engine.thresholds_pair(jobs, n, max_rows, td, sd, n_out, n_slots, w0, w1, "cuda")
    want = engine.thresholds(jobs, n, max_rows, td, sd, n_out, n_slots, w0, "cuda") + engine.thresholds(jobs, n, max_rows, td, sd, n_out, n_slots, w1, "cuda")
    torch.cuda.synchronize()
    for name, g, w in zip(("feat0", "agg0", "feat1", "agg1"), got, want):
        assert g.dtype == w.dtype and g.shape == w.shape
        assert torch.equal(_bits(torch, g), _bits(torch, w)), (name, w0, w1)
    return got


LENGTHS = [1, 2, 5, 6, 7, 143, 144, 145, 300, 1000, 1001, 2500, 4380]


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("w0,w1", [(6, 1), (6, 2), (6, 6), (6, 144), (6, 1000), (1, 6), (144, 6), (6, 4380), (6, 4381)])
def test_pair_is_two_threshold_launches(torch, engine, dtype, w0, w1):
    rng = np.random.default_rng(w0 * 7919 + w1)
    jobs, n, max_rows, td, sd, n_slots, _ = _case(torch, engine, rng, LENGTHS, 64, dtype)
    _assert_pair(torch, engine, jobs, n, max_rows, td, sd, 64, n_slots, w0, w1)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("n_out", [1, 256])
@pytest.mark.parametrize("w1", [12, 144])
def test_pair_at_the_tag_count_limits(torch, engine, dtype, n_out, w1):
    rng = np.random.default_rng(n_out + w1)
    jobs, n, max_rows, td, sd, n_slots, _ = _case(torch, engine, rng, [3, 150, 700, 2000], n_out, dtype)
    _assert_pair(torch, engine, jobs, n, max_rows, td, sd, n_out, n_slots, 6, w1)


@pytest.mark.parametrize("w1", [6, 144])
def test_pair_equal_to_job_length(torch, engine, w1):
    rng = np.random.default_rng(5)
    jobs, n, max_rows, td, sd, n_slots, _ = _case(torch, engine, rng, [w1 - 1, w1, w1 + 1], 8, np.float32)
    _assert_pair(torch, engine, jobs, n, max_rows, td, sd, 8, n_slots, 6, w1)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_more_jobs_than_one_grid_dimension(torch, engine, dtype):
    rng = np.random.default_rng(11)
    lengths = rng.integers(1, 20, size=70000)
    jobs, n, max_rows, td, sd, n_slots, _ = _case(torch, engine, rng, lengths, 3, dtype)
    _assert_pair(torch, engine, jobs, n, max_rows, td, sd, 3, n_slots, 6, 12)


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("w1", [2, 144, 1000])
def test_pair_against_pandas(torch, engine, dtype, w1):
    rng = np.random.default_rng(w1)
    jobs, n, max_rows, td, sd, n_slots, (tag, tot, slots, starts, lengths) = _case(torch, engine, rng, [100, 999, 1000, 3000], 16, dtype)
    got = [t.cpu().numpy() for t in _assert_pair(torch, engine, jobs, n, max_rows, td, sd, 16, n_slots, 6, w1)]
    for i in range(n):
        blk = slice(starts[i], starts[i] + lengths[i])
        for (feat, agg), w in (((got[0], got[1]), 6), ((got[2], got[3]), w1)):
            want_f = pd.DataFrame(tag[blk].astype(np.float64)).rolling(w).min().max().to_numpy()
            want_a = pd.Series(tot[blk].astype(np.float64)).rolling(w).min().max()
            np.testing.assert_array_equal(feat[slots[i]].astype(np.float64), want_f + 0.0)
            np.testing.assert_array_equal(np.float64(agg[slots[i]]), np.float64(want_a) + 0.0)
            assert not np.signbit(feat[slots[i]][~np.isnan(feat[slots[i]])]).any()
    for s in set(range(n_slots)) - set(slots.tolist()):  # slots no job covers keep what the caller put there
        assert np.isnan(got[0][s]).all() and np.isnan(got[3][s])
