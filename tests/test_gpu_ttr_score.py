"""
gb_minmax_inverse_score_f64 on the H100: the TransformedTargetRegressor's MinMax inverse and the float64 scoring in one pass equal,
bit for bit in every output, gb_minmax_inverse_f32 followed by gb_anomaly_score_f64 on the widened result -- across tag counts,
ragged and empty jobs, more jobs than one launch carries, NaN and overflowing values, any subset of outputs, in place or not.  The
inverse also equals sklearn's MinMaxScaler.inverse_transform on the float32 array.
"""
import itertools

import numpy as np
import pytest
from sklearn.preprocessing import MinMaxScaler

pytestmark = pytest.mark.gpu

KEYS = ("tag-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-scaled", "total-anomaly-unscaled", "anomaly-confidence",
        "total-anomaly-confidence")


@pytest.fixture(scope="module")
def torch():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _case(rng, n_out, n_rows, specials=False):
    """Per-slot scalers fitted on float64 targets, a float32 network output in [0, 1]-ish and the float64 targets (rows laid out
    back to back per job)."""
    S = len(n_rows)
    scalers = []
    for s in range(S):
        y = rng.normal(0, 1, (40, n_out)) * rng.uniform(0.1, 300, n_out) + rng.uniform(-500, 500, n_out)
        if specials:
            y[:, 0] = 7.25  # zero-range column: scale_ 1
            if n_out > 1:
                y[:, 1] = np.abs(y[:, 1]) - np.abs(y[:, 1]).min()  # data_min = 0: min_ = -0.0
        scalers.append(MinMaxScaler().fit(y))
    total = int(np.sum(n_rows))
    p = rng.normal(0.5, 0.5, (total, n_out)).astype(np.float32)
    y = rng.normal(0, 200, (total, n_out))
    if specials and total:
        p.flat[rng.integers(p.size, size=3)] = np.nan
        y.flat[rng.integers(y.size, size=3)] = np.nan
        p.flat[rng.integers(p.size)] = np.float32(3.0e38)  # overflows float32 on the inverse of a small scale_
        p.flat[rng.integers(p.size)] = -np.inf
    return scalers, p, y


def _run(torch, scalers, p, y, n_rows, want=KEYS, in_place=False, slots=None):
    from gordo_components_b200 import engine

    dev = engine.cuda_device()
    S, n_out = len(n_rows), p.shape[1]
    starts = np.concatenate([[0], np.cumsum(n_rows)[:-1]]).astype(np.int64)
    slots = np.arange(S) if slots is None else slots
    jobs = engine.jobs_to_device(engine.make_jobs(slots, n_rows, starts), dev)
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    rng = np.random.default_rng(n_out)
    y_scale = f(np.stack([s.scale_ for s in scalers]))
    y_min = f(np.stack([s.min_ for s in scalers]))
    mult = f(rng.uniform(0.1, 3, (len(scalers), n_out)))
    feat = f(rng.uniform(0.5, 2, (len(scalers), n_out)))
    agg = f(rng.uniform(0.5, 2, len(scalers)))
    max_rows = int(max(n_rows)) if len(n_rows) else 0
    pd_, yd = f(p), f(y)
    # the two-launch route
    back = engine.minmax_inverse_f32(jobs, S, max_rows, pd_, y_scale, y_min)
    ref = engine.anomaly_score(jobs, S, max_rows, back["f64"], yd, n_out, mult, feat, agg, want=want)
    # the new entry, optionally writing the inverse over the prediction
    out = {"model-output": pd_} if in_place else None
    got = engine.minmax_inverse_score_f64(jobs, S, max_rows, pd_, yd, y_scale, y_min, mult, feat, agg, want=want, out=out)
    torch.cuda.synchronize()
    return back, ref, got


def _rows(res, n_rows):
    """Only the rows the jobs own: everything else of a freshly allocated output is undefined."""
    idx = np.concatenate([np.arange(s, s + n) for s, n in zip(np.concatenate([[0], np.cumsum(n_rows)[:-1]]), n_rows)] or [np.zeros(0, int)])
    return {k: v.cpu().numpy()[idx] for k, v in res.items()}


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("n_out", [1, 4, 31, 32, 33, 64, 100, 256])
@pytest.mark.parametrize("in_place", [False, True])
def test_equals_inverse_then_float64_scoring(torch, n_out, in_place):
    rng = np.random.default_rng(n_out)
    n_rows = np.array([300, 1, 0, 1500, 77])  # ragged, one empty, one across two row chunks
    scalers, p, y = _case(rng, n_out, n_rows, specials=True)
    back, ref, got = _run(torch, scalers, p, y, n_rows, in_place=in_place)
    b, r, g = _rows(back, n_rows), _rows(ref, n_rows), _rows(got, n_rows)
    assert _same(g["model-output"], b["f32"])
    assert set(g) == set(KEYS) | {"model-output"}
    for k in KEYS:
        assert g[k].dtype == np.float64 and _same(g[k], r[k]), k
    # and the inverse is sklearn's, slot by slot, on the float32 array
    ofs = 0
    for s, n in enumerate(n_rows):
        block = p[ofs:ofs + n]
        with np.errstate(over="ignore", invalid="ignore"):
            want = block.copy()
            want -= scalers[s].min_
            want /= scalers[s].scale_
        if n and np.isfinite(block).all():  # sklearn refuses ±inf and empty arrays
            assert _same(g["model-output"][ofs:ofs + n], scalers[s].inverse_transform(block))
        assert _same(g["model-output"][ofs:ofs + n], want)
        ofs += n


def test_overflow_and_nan_reach_only_their_cells(torch):
    rng = np.random.default_rng(5)
    n_rows = np.array([64])
    scalers, p, y = _case(rng, 8, n_rows)
    scalers[0].scale_[3] = 1e-300  # every prediction of tag 3 overflows float32 on the inverse
    p[5, 1] = np.nan
    y[9, 2] = np.nan
    _, ref, got = _run(torch, scalers, p, y, n_rows)
    g = {k: v.cpu().numpy() for k, v in got.items()}
    assert np.isinf(g["model-output"][:, 3]).all() and np.isfinite(g["model-output"][:, [0, 1, 2, 4]][np.arange(64) != 5]).all()
    assert np.isnan(g["tag-anomaly-unscaled"][5, 1]) and np.isnan(g["tag-anomaly-unscaled"][9, 2])
    for k in KEYS:
        assert _same(g[k], ref[k].cpu().numpy()), k


@pytest.mark.parametrize("subset", [s for r in range(0, 7) for s in itertools.combinations(KEYS, r)][::5] + [(), KEYS])
def test_any_subset_of_outputs(torch, subset):
    rng = np.random.default_rng(len(subset))
    n_rows = np.array([40, 3, 129])
    scalers, p, y = _case(rng, 33, n_rows, specials=True)
    back, ref, got = _run(torch, scalers, p, y, n_rows, want=subset)
    assert set(got) == set(subset) | {"model-output"}
    b, r, g = _rows(back, n_rows), _rows(ref, n_rows), _rows(got, n_rows)
    assert _same(g["model-output"], b["f32"])
    for k in subset:
        assert _same(g[k], r[k]), k


def test_more_jobs_than_one_launch_carries(torch):
    rng = np.random.default_rng(9)
    n_jobs, S = 70000, 7
    n_rows = rng.integers(0, 4, n_jobs)
    scalers, p, y = _case(rng, 5, np.full(S, 1))  # the scalers of S slots
    total = int(n_rows.sum())
    p = rng.normal(0.5, 0.5, (total, 5)).astype(np.float32)
    y = rng.normal(0, 200, (total, 5))
    back, ref, got = _run(torch, scalers, p, y, n_rows, slots=np.arange(n_jobs) % S)
    b, r, g = _rows(back, n_rows), _rows(ref, n_rows), _rows(got, n_rows)
    assert _same(g["model-output"], b["f32"])
    for k in KEYS:
        assert _same(g[k], r[k]), k
