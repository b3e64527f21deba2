"""
gb_smooth_scores: the four anomaly arrays of a ragged batch smoothed in one launch come out bit for bit what four gb_smooth calls
give, for every method, window and tag count, float32 or float64 input, across the split into launches of 65 535 jobs, and within
float32 tolerance of the pandas formulas of the oracle.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KEYS = ("tag-anomaly-scaled", "total-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-unscaled")


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("needs an H100")
    import __graft_entry__ as ge

    ge.build()
    return t


def _batch(torch, lens, T, dtype=np.float32, seed=0, gap=2):
    """Score arrays of jobs of ``lens`` rows, ``gap`` unused rows between jobs; NaNs inside jobs and at the start of some."""
    from gordo_components_b200 import engine

    rng = np.random.default_rng(seed)
    starts = np.concatenate([[0], np.cumsum(np.asarray(lens) + gap)[:-1]]).astype(np.int64)
    rows = int(starts[-1] + lens[-1] + gap)
    tags = [rng.random((rows, T)) * 10 for _ in range(2)]
    totals = [t.mean(1) for t in tags]
    arrays = {"tag-anomaly-scaled": tags[0], "tag-anomaly-unscaled": tags[1], "total-anomaly-scaled": totals[0], "total-anomaly-unscaled": totals[1]}
    for k, a in arrays.items():
        a[rng.random(a.shape) < 0.01] = np.nan
        for j, (s, n) in enumerate(zip(starts, lens)):
            if n and j % 3 == 1:
                a[s] = np.nan  # a NaN on a job's first row
            if n > 4 and j % 3 == 2:
                a[s + n // 2] = np.nan
    jobs_h = engine.make_jobs(np.arange(len(lens)) % 5, lens, starts)
    dev = engine.cuda_device()
    d = {k: torch.from_numpy(np.ascontiguousarray(v, dtype=dtype)).to(dev) for k, v in arrays.items()}
    return jobs_h, engine.jobs_to_device(jobs_h, dev), d


def _four_calls(torch, jobs_h, jobs_d, arrays, window, method):
    from gordo_components_b200 import engine

    max_rows = int(jobs_h["n_rows"].max())
    return {"smooth-" + k: engine.smooth(jobs_d, len(jobs_h), arrays[k].to(torch.float32), window, method, max_rows=max_rows) for k in KEYS}


def _assert_same_bits(got, want):
    for k in want:
        assert got[k].shape == want[k].shape and got[k].dtype == want[k].dtype, k
        assert torch_equal_bits(got[k], want[k]), k


def torch_equal_bits(a, b):
    import torch

    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _lens(window):
    """0 rows, 1 row, fewer rows than the window, exactly the window, several 128-row chunks."""
    return [0, 1, max(window - 1, 0), window, 3 * 128 + 5, 2 * 128, window + 130, 7]


@pytest.mark.parametrize("method", ["smm", "sma", "ewma"])
@pytest.mark.parametrize("window", [1, 2, 144, 145])
@pytest.mark.parametrize("T", [1, 3, 64, 65, 128])
def test_one_launch_equals_four_smooth_calls(torch, method, window, T):
    from gordo_components_b200 import engine

    jobs_h, jobs_d, arrays = _batch(torch, _lens(window), T, seed=window * 7 + T)
    got = engine.smooth_scores(jobs_d, len(jobs_h), int(jobs_h["n_rows"].max()), arrays, window, method)
    _assert_same_bits(got, _four_calls(torch, jobs_h, jobs_d, arrays, window, method))


@pytest.mark.parametrize("method", ["smm", "sma", "ewma"])
@pytest.mark.parametrize("window", [801, 3000])  # 32 and 16 threads per rolling-median CTA
def test_wide_windows(torch, method, window):
    from gordo_components_b200 import engine

    for T in (1, 64):
        jobs_h, jobs_d, arrays = _batch(torch, [window + 300, window, 5, 0, window - 1], T, seed=window + T)
        got = engine.smooth_scores(jobs_d, len(jobs_h), int(jobs_h["n_rows"].max()), arrays, window, method)
        _assert_same_bits(got, _four_calls(torch, jobs_h, jobs_d, arrays, window, method))


@pytest.mark.parametrize("method", ["smm", "sma", "ewma"])
def test_float64_input_equals_float32_rounded_input(torch, method):
    from gordo_components_b200 import engine

    jobs_h, jobs_d, a64 = _batch(torch, _lens(6), 64, dtype=np.float64, seed=5)
    a32 = {k: v.to(torch.float32) for k, v in a64.items()}
    max_rows = int(jobs_h["n_rows"].max())
    got64 = engine.smooth_scores(jobs_d, len(jobs_h), max_rows, a64, 6, method)
    got32 = engine.smooth_scores(jobs_d, len(jobs_h), max_rows, a32, 6, method)
    _assert_same_bits(got64, got32)
    _assert_same_bits(got64, _four_calls(torch, jobs_h, jobs_d, a32, 6, method))


@pytest.mark.parametrize("method", ["smm", "ewma"])
def test_more_jobs_than_one_launch_holds(torch, method):
    from gordo_components_b200 import engine

    lens = list(np.random.default_rng(3).integers(0, 5, 70_000))
    jobs_h, jobs_d, arrays = _batch(torch, lens, 3, seed=11, gap=0)
    got = engine.smooth_scores(jobs_d, len(jobs_h), int(jobs_h["n_rows"].max()), arrays, 2, method)
    _assert_same_bits(got, _four_calls(torch, jobs_h, jobs_d, arrays, 2, method))


@pytest.mark.parametrize("method", ["smm", "sma", "ewma"])
@pytest.mark.parametrize("window", [1, 6, 144])
def test_against_the_pandas_formulas(torch, method, window):
    from gordo_components_b200 import engine
    from oracle import anomaly_math as am

    jobs_h, jobs_d, arrays = _batch(torch, _lens(window), 5, seed=window)
    got = engine.smooth_scores(jobs_d, len(jobs_h), int(jobs_h["n_rows"].max()), arrays, window, method)
    for job in jobs_h:
        s, n = int(job["out_row"]), int(job["n_rows"])
        for k in KEYS:
            src = arrays[k][s:s + n].cpu().numpy().astype(np.float32)
            want = am.smoothing(src, window, method)
            np.testing.assert_allclose(got["smooth-" + k][s:s + n].cpu().numpy(), want, rtol=2e-6, atol=1e-6, equal_nan=True)
    # rows between jobs are not written
    gaps = np.ones(arrays["total-anomaly-scaled"].shape[0], dtype=bool)
    for job in jobs_h:
        gaps[int(job["out_row"]):int(job["out_row"]) + int(job["n_rows"])] = False
    assert torch.isnan(got["smooth-total-anomaly-scaled"][torch.from_numpy(gaps).to(jobs_d.device)]).all()
