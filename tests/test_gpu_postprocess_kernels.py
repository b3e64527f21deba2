"""
The kernels that run after the network, against plain float64 NumPy and pandas: the column extrema of the target scaler
(gb_minmax_fit, gb_minmax_f64), the alert thresholds (gb_thresholds, gb_thresholds_f64), the score of existing predictions
(gb_anomaly_score, gb_anomaly_score_f64), the K-fold percentile (gb_quantile), the smoothing (gb_smooth) and the scaled copies
of the fleet inputs (gb_affine_f64).

Every case runs ragged jobs whose slot, input row and output row all differ from the job index.  Slots and output rows that no
job covers are pre-filled with a sentinel that must survive, and input rows that no job covers hold values that would change a
result if a kernel read them.  Selections (min, max, abs, a single rounded multiply or divide) are compared exactly, with the
sign of a zero; sums at the tolerances of test_gpu_parity.py.
"""
import warnings
from fractions import Fraction

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

SENT = -12345.0  # pre-filled into every output; none of the data below can produce it


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


# ------------------------------------------------------------------------------------------------ helpers
def layout(engine, lens, shared=()):
    """
    Jobs of the given lengths.  Job i has slot 2J-1-i (slots 0..J-1 and 2J stay unused), reads its inputs from rows stored back
    to front from row 5 with 3-row gaps and its outputs front to back from row 1 with 2-row gaps.  ``shared``: (i, k) pairs that
    give job i the slot of job k.  Returns (jobs, n_slots, input rows, output rows).
    """
    lens = np.asarray(lens, dtype=np.int64)
    J = len(lens)
    slots = 2 * J - 1 - np.arange(J)
    for i, k in shared:
        slots[i] = slots[k]
    x_rows = (5 + np.concatenate([[0], np.cumsum(lens[::-1] + 3)[:-1]]))[::-1]
    out_rows = 1 + np.concatenate([[0], np.cumsum(lens + 2)[:-1]])
    return engine.make_jobs(slots, lens, x_rows, out_rows), 2 * J + 1, int(5 + (lens + 3).sum()), int(1 + (lens + 2).sum())


def covered(jobs, key, total):
    """Rows [key, key + n_rows) of every job."""
    m = np.zeros(total, dtype=bool)
    for j in jobs:
        m[j[key]: j[key] + j["n_rows"]] = True
    return m


def exact(got, want, name=""):
    """Equal values (NaN equal to NaN) and, where the expected value is a zero, the same sign."""
    got, want = np.asarray(got), np.asarray(want)
    np.testing.assert_array_equal(got, want, err_msg=name)
    zero = want == 0
    np.testing.assert_array_equal(np.signbit(got[zero]), np.signbit(want[zero]), err_msg=f"{name}: sign of a zero")


def put(torch, a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to("cuda")


def lib_call(engine, name, *args):
    from gordo_components_b200 import _cabi

    args = [_cabi.ptr(a) if a is None or hasattr(a, "data_ptr") else a for a in args]
    _cabi.check(getattr(_cabi.load_library(), name)(*args, engine._stream_ptr()))


def sentinel(torch, shape, dtype):
    return torch.full(shape, SENT, dtype={np.float32: torch.float32, np.float64: torch.float64}[np.dtype(dtype).type], device="cuda")


# ------------------------------------------------------------------------------------------------ gb_minmax_fit / gb_minmax_f64
def minmax_run(engine, torch, jobs, n_slots, y):
    """gb_minmax_fit (float32 y) or gb_minmax_f64 (float64 y), every output pre-filled with SENT -> dict of numpy arrays."""
    n_out = y.shape[1]
    jd, yd = engine.jobs_to_device(jobs, "cuda"), put(torch, y)
    max_rows = int(jobs["n_rows"].max())
    if y.dtype == np.float32:
        scale, offset, ws = (sentinel(torch, s, y.dtype) for s in ((n_slots, n_out), (n_slots, n_out), (n_slots, 2, n_out)))
        lib_call(engine, "gb_minmax_fit", jd, len(jobs), max_rows, yd, n_out, scale, offset, ws, n_slots)
        return {"lo": ws[:, 0].cpu().numpy(), "hi": ws[:, 1].cpu().numpy(), "scale": scale.cpu().numpy(), "offset": offset.cpu().numpy()}
    mm = sentinel(torch, (n_slots, 2, n_out), y.dtype)
    lib_call(engine, "gb_minmax_f64", jd, len(jobs), max_rows, yd, n_out, mm, n_slots)
    return {"lo": mm[:, 0].cpu().numpy(), "hi": mm[:, 1].cpu().numpy()}


def minmax_ref(jobs, n_slots, y):
    """np.nanmin / np.nanmax over the input rows of all jobs of a slot; an all-NaN column gives +inf / -inf; SENT for unused slots.
    For float32 also sklearn's scale_ / min_ in float32: a range below 10 * eps is a constant column (range 1)."""
    lo = np.full((n_slots, y.shape[1]), SENT, y.dtype)
    hi = lo.copy()
    for s in np.unique(jobs["slot"]):
        rows = np.concatenate([y[j["x_row"]: j["x_row"] + j["n_rows"]] for j in jobs if j["slot"] == s])
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            l, h = np.nanmin(rows, axis=0), np.nanmax(rows, axis=0)
        lo[s], hi[s] = np.where(np.isnan(l), np.inf, l), np.where(np.isnan(h), -np.inf, h)
    want = {"hi": hi, "lo": lo}  # the maximum first: its -0.0 case fails deterministically, the minimum's is a race
    if y.dtype == np.float32:
        used = np.isin(np.arange(n_slots), jobs["slot"])
        with np.errstate(invalid="ignore", over="ignore"):
            rng = hi - lo
            rng = np.where(rng >= np.float32(10) * np.finfo(np.float32).eps, rng, np.float32(1))
            scale = np.float32(1) / rng
            offset = -lo * scale
        want["scale"] = np.where(used[:, None], scale, np.float32(SENT))
        want["offset"] = np.where(used[:, None], offset, np.float32(SENT))
    return want


def check_minmax(engine, torch, jobs, n_slots, y64, name):
    for y in (y64.astype(np.float32), y64):
        got, want = minmax_run(engine, torch, jobs, n_slots, y), minmax_ref(jobs, n_slots, y)
        for k in want:
            exact(got[k], want[k], f"{name} {y.dtype} {k}")


@pytest.mark.parametrize("n_out", [1, 31, 32, 33, 255, 256])
def test_minmax_matches_nanmin_nanmax(engine, torch, n_out):
    """Across the 32-lane column loop and the [warps][256] shared tile; jobs of 1 row, of fewer rows than warps, and around the
    1024-row blocks; the last job merges its extrema into the slot of the 1024-row job (a K-fold slot is a union of test blocks);
    scattered NaNs and an all-NaN column."""
    rng = np.random.default_rng(n_out)
    jobs, n_slots, xt, _ = layout(engine, [1, 7, 1023, 1024, 1025, 5000, 700], shared=[(6, 3)])
    y = rng.normal(size=(xt, n_out)) * 10
    y[rng.random(y.shape) < 0.02] = np.nan
    if n_out > 1:
        y[:, n_out // 2] = np.nan
    outside = ~covered(jobs, "x_row", xt)
    y[outside] = rng.choice([-1e30, 1e30], size=(int(outside.sum()), n_out))
    check_minmax(engine, torch, jobs, n_slots, y, f"n_out={n_out}")


def test_minmax_signed_zeros(engine, torch):
    """
    -0.0 is the largest non-positive value but, as a signed integer, the smallest: the float atomics choose their integer form from
    the sign bit.  A column maximum of -0.0 must replace -inf and beat the negative maximum of another block or job, and a block
    minimum of -0.0 must lose to a negative minimum of another block whichever finishes first.
    """
    rng = np.random.default_rng(3)
    lens = [8 * 1024 + 100, 1000, 1500]
    jobs, n_slots, xt, _ = layout(engine, lens, shared=[(2, 1)])  # job 2 merges into the one-block slot of job 1
    y = np.full((xt, 4), 7.0)  # rows outside the jobs would raise every maximum
    r = [y[j["x_row"]: j["x_row"] + j["n_rows"]] for j in jobs]
    r[0][:] = -rng.uniform(1, 3, r[0].shape)
    blk = np.arange(lens[0]) // 1024
    r[0][:, 0] = -0.0                       # nothing but -0.0, in every block
    r[0][blk == 8, 1] = -0.0                # -0.0 only in the last block, the negative values in the others
    r[0][blk % 2 == 0, 2] = -0.0            # -0.0 blocks next to negative blocks, in both orders
    r[0][blk % 2 == 1, 3] = -0.0
    r[1][:] = -rng.uniform(1, 3, r[1].shape)
    r[1][:, 0] = -0.0                       # one block of -0.0 merging with job 2's -5 (minimum -5)
    r[1][-1, 1] = -0.0                      # [-3, ..., -0.0] in one block, merging with job 2's negative values (maximum -0.0)
    r[1][:, 3] = -0.0
    r[2][:] = -rng.uniform(1, 3, r[2].shape)
    r[2][:, 0] = -5.0
    r[2][:, 2] = -0.0
    check_minmax(engine, torch, jobs, n_slots, y, "signed zeros")


def test_minmax_fit_constant_column_threshold(engine, torch):
    """sklearn's _handle_zeros_in_scale: a float32 range below 10 * eps(float32) is a constant column (scale_ 1).  Ranges of 4, 5 and
    6 ulps of 3.0 sit below, at and above it (5 ulps of 3.0 is exactly 10 * eps), as do the neighbours of 10 * eps above 0."""
    thr = np.float32(10) * np.finfo(np.float32).eps
    u3 = np.spacing(np.float32(3))
    cols = [(3, 3 + k * u3) for k in (0, 1, 4, 5, 6, 50)] + [(0, h) for h in (np.nextafter(thr, np.float32(0)), thr, np.nextafter(thr, np.float32(1)))]
    jobs, n_slots, xt, _ = layout(engine, [600, 1300])
    rng = np.random.default_rng(4)
    y = np.full((xt, len(cols)), 1e6, np.float32)
    for j in jobs:
        part = y[j["x_row"]: j["x_row"] + j["n_rows"]]
        for c, (lo, hi) in enumerate(cols):
            part[:, c] = np.float32(lo) + (np.float32(hi) - np.float32(lo)) * (rng.random(len(part)) < 0.5)
            part[0, c], part[-1, c] = lo, hi
    want = minmax_ref(jobs, n_slots, y)
    s = jobs["slot"][0]
    assert list(want["scale"][s] == 1) == [True, True, True, False, False, False, True, False, False]  # the data straddles 10 * eps
    got = minmax_run(engine, torch, jobs, n_slots, y)
    for k in want:
        exact(got[k], want[k], k)


# ------------------------------------------------------------------------------------------------ gb_thresholds / gb_thresholds_f64
def thresholds_run(engine, torch, jobs, n_slots, tu, ts, window):
    """Feature thresholds from ``tu`` and / or the aggregate threshold from ``ts`` (the other may be None: its pair goes NULL),
    outputs pre-filled with SENT."""
    a = tu if tu is not None else ts
    n_out = tu.shape[1] if tu is not None else 1
    feat = sentinel(torch, (n_slots, n_out), a.dtype) if tu is not None else None
    agg = sentinel(torch, (n_slots,), a.dtype) if ts is not None else None
    name = "gb_thresholds" if a.dtype == np.float32 else "gb_thresholds_f64"
    lib_call(engine, name, engine.jobs_to_device(jobs, "cuda"), len(jobs), int(jobs["n_rows"].max()), put(torch, tu), put(torch, ts), n_out,
             window, feat, agg, n_slots)
    return None if feat is None else feat.cpu().numpy(), None if agg is None else agg.cpu().numpy()


def thresholds_ref(jobs, n_slots, arr, window):
    """pandas rolling(window).min().max() of every job's rows (they start at out_row), at the job's slot; SENT elsewhere."""
    want = np.full((n_slots,) + arr.shape[1:], SENT, arr.dtype)
    for j in jobs:
        part = arr[j["out_row"]: j["out_row"] + j["n_rows"]].astype(np.float64)
        part = part[:, None] if part.ndim == 1 else part
        want[j["slot"]] = pd.DataFrame(part).rolling(window).min().max().values.reshape(arr.shape[1:])
    return want


@pytest.mark.parametrize("n_out", [1, 33, 256])
@pytest.mark.parametrize("window", [1, 2, 6, 144, 1025])
def test_thresholds_match_pandas(engine, torch, window, n_out):
    """Jobs shorter than the window (NaN), exactly the window, one longer, and on both sides of the first block edge (the blocks
    start at t0 = window - 1 + k * 1024); the feature and aggregate paths each alone; NaNs inside windows, a column in which every
    window holds one (NaN) and a zero-residual column of -0.0 (threshold 0)."""
    rng = np.random.default_rng(1000 * window + n_out)
    jobs, n_slots, _, ot = layout(engine, [window - 1, window, window + 1, 1024 + window - 1, 1024 + window, 5000])
    outside = ~covered(jobs, "out_row", ot)
    for dt in (np.float32, np.float64):
        tu, ts = rng.random((ot, n_out)).astype(dt), rng.random(ot).astype(dt)
        tu[rng.random(tu.shape) < 2e-4] = np.nan
        ts[rng.random(ts.shape) < 2e-4] = np.nan
        if n_out > 1:
            tu[np.arange(ot) % window == 0, 0] = np.nan
            tu[:, 1] = -0.0
        tu[outside], ts[outside] = 5, 5  # above every residual: reading them would raise a threshold
        feat, _ = thresholds_run(engine, torch, jobs, n_slots, tu, None, window)
        _, agg = thresholds_run(engine, torch, jobs, n_slots, None, ts, window)
        np.testing.assert_array_equal(feat, thresholds_ref(jobs, n_slots, tu, window), err_msg=f"{dt.__name__} feature thresholds")
        np.testing.assert_array_equal(agg, thresholds_ref(jobs, n_slots, ts, window), err_msg=f"{dt.__name__} aggregate threshold")


def test_thresholds_across_the_launch_split(engine, torch):
    """70 000 jobs of 0 to 4 rows, more than gridDim.y's 65 535: every job has its own slot and is compared exactly, on both sides
    of the split.  Jobs of 0 or 1 row are shorter than the window (NaN)."""
    J, W, T = 70_000, 2, 3
    rng = np.random.default_rng(70)
    lens = rng.integers(0, 5, J)
    jobs, n_slots, _, ot = layout(engine, lens)
    slots, out_rows = jobs["slot"], jobs["out_row"]
    outside = ~covered(jobs, "out_row", ot)
    for dt in (np.float32, np.float64):
        tu, ts = rng.random((ot, T)).astype(dt), rng.random(ot).astype(dt)
        tu[outside], ts[outside] = 5, 5
        feat, agg = thresholds_run(engine, torch, jobs, n_slots, tu, ts, W)
        for got, arr in ((feat, tu), (agg, ts[:, None])):
            pad = np.full((J, 4, arr.shape[1]), np.nan, dt)  # each job's rows, NaN past its end
            for r in range(4):
                pad[lens > r, r] = arr[out_rows[lens > r] + r]
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", RuntimeWarning)
                per_job = np.nanmax(np.minimum(pad[:, :-1], pad[:, 1:]), axis=1)  # rolling(2).min().max()
            want = np.full((n_slots, arr.shape[1]), SENT, dt)
            want[slots] = per_job
            assert np.isfinite(want[slots[65_535:]]).any() and np.isnan(want[slots[65_535:]]).any()
            np.testing.assert_array_equal(got.reshape(n_slots, -1), want, err_msg=dt.__name__)


# ------------------------------------------------------------------------------------------------ gb_anomaly_score / _f64
SCORE_TAGS = ("tag-anomaly-scaled", "tag-anomaly-unscaled", "anomaly-confidence")


def score_run(engine, torch, jobs, yhat, y, scale, feat, agg, out_total, want):
    """gb_anomaly_score(_f64) with the requested outputs (the others NULL) pre-filled with SENT."""
    n_out = y.shape[1]
    outs = {k: sentinel(torch, (out_total, n_out) if k in SCORE_TAGS else (out_total,), y.dtype) if k in want else None for k in engine.SCORE_KEYS}
    name = "gb_anomaly_score" if y.dtype == np.float32 else "gb_anomaly_score_f64"
    lib_call(engine, name, engine.jobs_to_device(jobs, "cuda"), len(jobs), int(jobs["n_rows"].max()), put(torch, yhat), put(torch, y), n_out,
             put(torch, scale), put(torch, feat), put(torch, agg), *(outs[k] for k in engine.SCORE_KEYS))
    return {k: v.cpu().numpy() for k, v in outs.items() if v is not None}


def score_ref(jobs, yhat, y, scale, feat, agg, out_total):
    """Tag columns in the data's precision (|yhat - y|, * scale and / feat_thr are one rounding each); row totals in float64."""
    n_out, dt = y.shape[1], y.dtype
    want = {k: np.full((out_total, n_out) if k in SCORE_TAGS else (out_total,), SENT, dt if k in SCORE_TAGS else np.float64) for k in
            ("tag-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-scaled", "total-anomaly-unscaled", "anomaly-confidence",
             "total-anomaly-confidence")}
    for j in jobs:
        o, x, s = slice(j["out_row"], j["out_row"] + j["n_rows"]), slice(j["x_row"], j["x_row"] + j["n_rows"]), j["slot"]
        d = np.abs(yhat[o] - y[x])
        e = d * scale[s]
        want["tag-anomaly-unscaled"][o], want["tag-anomaly-scaled"][o], want["anomaly-confidence"][o] = d, e, d / feat[s]
        want["total-anomaly-unscaled"][o] = (d.astype(np.float64) ** 2).mean(axis=1)
        want["total-anomaly-scaled"][o] = (e.astype(np.float64) ** 2).mean(axis=1)
        want["total-anomaly-confidence"][o] = want["total-anomaly-scaled"][o] / float(agg[s])
    return want


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n_out", [1, 31, 32, 33, 257, 300])
def test_anomaly_score_matches_numpy(engine, torch, n_out, dtype):
    """yhat and the outputs at out_row, y at x_row, scale and thresholds at the slot; rows across the 1024-row blocks; all six
    outputs at once and each alone.  yhat = -0.0 against y = +0.0 gives +0.0 tag columns, as np.abs."""
    rng = np.random.default_rng(n_out)
    jobs, n_slots, xt, ot = layout(engine, [1, 1500, 2049, 37])
    yhat, y = rng.random((ot, n_out)).astype(dtype), rng.random((xt, n_out)).astype(dtype)
    j1 = jobs[1]
    yhat[j1["out_row"]], y[j1["x_row"]] = -0.0, 0.0
    yhat[j1["out_row"] + 1], y[j1["x_row"] + 1] = 0.0, -0.0
    used = np.isin(np.arange(n_slots), jobs["slot"])
    scale, feat, agg = np.full((n_slots, n_out), np.nan, dtype), np.full((n_slots, n_out), np.nan, dtype), np.full(n_slots, np.nan, dtype)
    scale[used] = rng.uniform(0.5, 2, (used.sum(), n_out))  # unused slots are NaN: reading one shows
    feat[used] = rng.uniform(0.05, 0.3, (used.sum(), n_out))
    agg[used] = rng.uniform(0.01, 0.1, used.sum())
    want = score_ref(jobs, yhat, y, scale, feat, agg, ot)
    zeros = want["tag-anomaly-unscaled"][j1["out_row"]: j1["out_row"] + 2]
    assert (zeros == 0).all() and not np.signbit(zeros).any()  # exact() holds the kernel to the same sign
    rtol = 1e-5 if dtype == np.float32 else 1e-13
    outside = ~covered(jobs, "out_row", ot)
    for keys in [want.keys()] + [(k,) for k in want]:
        got = score_run(engine, torch, jobs, yhat, y, scale, feat, agg, ot, keys)
        assert set(got) == set(keys)
        for k, g in got.items():
            if k in SCORE_TAGS:
                exact(g, want[k], k)
            else:
                assert (g[outside] == SENT).all(), k
                np.testing.assert_allclose(g[~outside], want[k][~outside], rtol=rtol, atol=0, err_msg=k)


# ------------------------------------------------------------------------------------------------ gb_quantile
def test_quantile_matches_pandas_across_ragged_jobs(engine, torch):
    """
    pandas DataFrame.quantile(q) of every job in one launch: lengths 0 (NaN) to 40 000; q of 0, 1, 0.37 and values at which
    (n-1)*q is a whole number for some jobs (compared exactly there); heavy ties and columns that mix -0.0 and +0.0.  The jobs of up
    to 32 768 rows once more, sorted in shared memory (their true max_rows) and selected from L2 (max_rows 32 769, the kernel only
    uses it as an upper bound): the two agree bit for bit.
    """
    rng = np.random.default_rng(8)
    lens = [0, 1, 2, 777, 1025, 32768, 40000]
    jobs, _, _, ot = layout(engine, lens)
    a = rng.normal(size=(ot, 3)).astype(np.float32)
    a[:, 1] = np.round(a[:, 1], 1)
    a[:, 2] = rng.choice(np.float32([-1.5, -0.0, 0.0, 0.0, -0.0, 2.25]), ot)
    a[rng.random(a.shape) < 0.1] = np.nan
    a[~covered(jobs, "out_row", ot)] = 1e30  # would move every quantile
    ad = put(torch, a)
    jd, jd_short = engine.jobs_to_device(jobs, "cuda"), engine.jobs_to_device(jobs[:-1], "cuda")
    n_whole = 0  # exact comparisons at 0 < q < 1 with two or more values
    for q in (0.0, 1.0, 0.37, 0.5, 0.25, 0.75):
        q64 = float(np.float32(q))  # the kernel takes q as a float
        got = engine.quantile(jd, len(jobs), max(lens), ad, q).cpu().numpy()
        sort = engine.quantile(jd_short, len(jobs) - 1, 32768, ad, q).cpu().numpy()
        select = engine.quantile(jd_short, len(jobs) - 1, 32769, ad, q).cpu().numpy()
        np.testing.assert_array_equal(sort.view(np.uint32), select.view(np.uint32), err_msg=f"q={q}: shared-memory sort against L2 selection")
        for res in (got, sort):
            for i, j in enumerate(jobs[:len(res)]):
                part = a[j["out_row"]: j["out_row"] + j["n_rows"]].astype(np.float64)
                want = pd.DataFrame(part).quantile(q64).values
                for c in range(3):
                    n = int((~np.isnan(part[:, c])).sum())
                    if n == 0 or ((n - 1) * q64).is_integer():
                        n_whole += 0 < q < 1 and n >= 2
                        exact(res[i, c], np.float32(want[c]), f"job {i} col {c} q={q}")
                    else:
                        np.testing.assert_allclose(res[i, c], want[c], rtol=1e-6, atol=0, err_msg=f"job {i} col {c} q={q}")
    assert n_whole > 0


# ------------------------------------------------------------------------------------------------ gb_smooth
def smooth_run(engine, torch, jobs, arr, window, method):
    out = sentinel(torch, arr.shape, np.float32)
    lib_call(engine, "gb_smooth", engine.jobs_to_device(jobs, "cuda"), len(jobs), int(jobs["n_rows"].max()), put(torch, arr), arr.shape[1],
             window, engine.SMOOTH_METHODS[method], out)
    return out.cpu().numpy()


def check_smooth(jobs, a, got, window, method):
    """pandas rolling().median() / rolling().mean() / ewm(span=).mean() per job, at test_smoothing_with_interior_nans_matches_pandas'
    tolerance; rows no job covers keep the sentinel."""
    assert (got[~covered(jobs, "out_row", len(a))] == SENT).all()
    for j in jobs:
        o = slice(j["out_row"], j["out_row"] + j["n_rows"])
        frame = pd.DataFrame(a[o].astype(np.float64))
        want = {"smm": lambda: frame.rolling(window).median(), "sma": lambda: frame.rolling(window).mean(),
                "ewma": lambda: frame.ewm(span=window).mean()}[method]().values
        assert np.array_equal(np.isnan(got[o]), np.isnan(want)), (method, window)
        np.testing.assert_allclose(got[o], want, rtol=2e-6, atol=1e-7, err_msg=f"{method} window {window}")


@pytest.mark.parametrize("n_cols", [65, 130])
@pytest.mark.parametrize("method,window", [("smm", 1), ("sma", 1), ("ewma", 1), ("sma", 144), ("ewma", 144), ("smm", 800), ("smm", 801)])
def test_smooth_matches_pandas(engine, torch, n_cols, method, window):
    """More columns than one 64-column block; window 1 for every method; median windows at 64 threads per block (800 values each,
    exactly 200 KB) and at 32 (801).  Interior and leading NaNs."""
    rng = np.random.default_rng(n_cols + window)
    jobs, _, _, ot = layout(engine, [1, 700, 1000, 1900])
    a = rng.random((ot, n_cols)).astype(np.float32)
    a[rng.random(ot) < 0.002, 1] = np.nan
    a[: jobs[2]["out_row"] + 9, 64] = np.nan
    a[~covered(jobs, "out_row", ot)] = 1e30
    check_smooth(jobs, a, smooth_run(engine, torch, jobs, a, window, method), window, method)


def test_smooth_median_at_the_shared_memory_cap(engine, torch):
    """A 51 200-value window, one thread per block, is the widest the median holds (200 KB); 51 201 is refused (GB_E_SMEM).  The data
    ascends with noise, so insertion into the sorted window stays cheap (random data costs O(window^2) per 128-row chunk)."""
    rng = np.random.default_rng(51)
    n = 52_000
    jobs, _, _, ot = layout(engine, [n])
    a = np.full((ot, 1), 1e30, np.float32)
    a[jobs[0]["out_row"]: jobs[0]["out_row"] + n, 0] = np.arange(n) + rng.uniform(-2, 2, n)
    check_smooth(jobs, a, smooth_run(engine, torch, jobs, a, 51_200, "smm"), 51_200, "smm")
    with pytest.raises(ValueError):
        engine.smooth(engine.jobs_to_device(jobs, "cuda"), 1, put(torch, a), 51_201, "smm")


# ------------------------------------------------------------------------------------------------ gb_affine_f64
def affine_case(rng, lens, n_cols):
    """Offset-dominated data: x ~ 1e4 +- 1e-3, a ~ 1e3, b ~ -1e7, so x * a + b cancels to ~1 and the double rounding of x * a shows
    in the float32 result.  Unused slots have NaN coefficients, input rows no job covers are NaN."""
    lens = np.asarray(lens)
    J = len(lens)
    n_slots, xt = 2 * J + 1, int(5 + (lens + 3).sum())
    x = 1e4 + rng.uniform(-1e-3, 1e-3, (xt, n_cols))
    a = np.full((n_slots, n_cols), np.nan)
    a[J:2 * J] = 1e3 * (1 + rng.uniform(-0.1, 0.1, (J, n_cols)))
    return x, a, -1e4 * a


def affine_run(engine, torch, jobs, x, a, b, out_total):
    out = sentinel(torch, (out_total, x.shape[1]), np.float32)
    lib_call(engine, "gb_affine_f64", engine.jobs_to_device(jobs, "cuda"), len(jobs), int(jobs["n_rows"].max()), put(torch, x), x.shape[1],
             put(torch, a), put(torch, b), out)
    return out.cpu().numpy()


def affine_ref(jobs, x, a, b, out_total):
    """((x * a) + b).astype(float32) per job: two float64 roundings, then one to float32."""
    want = np.full((out_total, x.shape[1]), SENT, np.float32)
    for j in jobs:
        want[j["out_row"]: j["out_row"] + j["n_rows"]] = ((x[j["x_row"]: j["x_row"] + j["n_rows"]] * a[j["slot"]]) + b[j["slot"]]).astype(np.float32)
    return want


@pytest.mark.parametrize("n_cols", [1, 7, 256, 300])
def test_affine_f64_matches_numpy(engine, torch, n_cols):
    rng = np.random.default_rng(n_cols)
    lens = [1, 5, 333, 1200]
    jobs, _, xt, ot = layout(engine, lens)
    x, a, b = affine_case(rng, lens, n_cols)
    x[~covered(jobs, "x_row", xt)] = np.nan
    exact(affine_run(engine, torch, jobs, x, a, b, ot), affine_ref(jobs, x, a, b, ot))


def test_affine_f64_grid_stride_and_no_fma(engine, torch):
    """A 2 000 x 200 job has more elements than the grid-stride width (1184 blocks of 256 threads).  On this data a fused
    multiply-add rounds differently from x * a followed by + b: the test checks that it does, so a contracted kernel would fail."""
    rng = np.random.default_rng(2000)
    lens = [2000, 3]
    jobs, _, xt, ot = layout(engine, lens)
    assert lens[0] * 200 > 1184 * 256
    x, a, b = affine_case(rng, lens, 200)
    x[~covered(jobs, "x_row", xt)] = np.nan
    want = affine_ref(jobs, x, a, b, ot)
    j = jobs[0]
    xs, s = x[j["x_row"]: j["x_row"] + 10], j["slot"]
    fused = np.array([[np.float32(float(Fraction(v) * Fraction(a[s, c]) + Fraction(b[s, c]))) for c, v in enumerate(row)] for row in xs])
    assert (fused != want[j["out_row"]: j["out_row"] + 10]).any()
    exact(affine_run(engine, torch, jobs, x, a, b, ot), want)


def test_affine_f64_across_the_launch_split(engine, torch):
    """70 000 one-row jobs, more than gridDim.y's 65 535, each with its own slot."""
    rng = np.random.default_rng(7)
    lens = np.ones(70_000, dtype=np.int64)
    jobs, _, xt, ot = layout(engine, lens)
    x, a, b = affine_case(rng, lens, 3)
    want = np.full((ot, 3), SENT, np.float32)
    s, xr = jobs["slot"], jobs["x_row"]
    want[jobs["out_row"]] = ((x[xr] * a[s]) + b[s]).astype(np.float32)
    exact(affine_run(engine, torch, jobs, x, a, b, ot), want)
