"""
Missing and non-finite sensor values on the GPU path.  A tag that did not report reaches the kernels as NaN (JSON null, a missing
key, a NaN literal or a parquet null all parse to the same float64 NaN frame), and a broken sensor can report ±inf.

* Kernels: a poisoned x or y row changes its own row and nothing else -- Dense variants 1, 2 (T = 32 and a zero-padded T = 36) and 3,
  gb_anomaly_score(_f64), the LSTM kernels and the request coalescer -- against a clean launch of the same layout, bit for bit.
  NaN in x gives an all-NaN row; ±inf in x follows the float64 oracle on the fp32 kernels (tanh(±inf) = ±1, as in Keras) and gives an
  all-NaN row on the tensor-core Dense kernel, whose layer 0 splits x into TF32 + BF16 parts (inf - inf), and NaN windows on the
  tensor-core LSTM kernel; the estimators launch the fp32 kernels for inputs holding ±inf.  Poison in y reaches only its
  own (row, tag) cells; the kernels' row totals are the numpy mean (NaN or inf with the cell), which threshold fitting needs.
* Detector and server: the anomaly frame follows the reference's (tests/golden/ffnet_anomaly_nan.npz, made by the reference's own
  code): totals skip missing tags as pandas does, ±inf in y, in the model output or behind a scaler pipeline is refused with sklearn's
  error, and a bare model with ±inf in x is answered by an fp32 kernel.
"""
import json
import os

import numpy as np
import pandas as pd
import pytest
from parity_helpers import close
from test_gpu_infer_coverage import PER_ROW, SCORE, dense_net, engine, lstm_net, lstm_oracle, run_dense, run_lstm, score_inputs, torch  # noqa: F401
from test_gpu_postprocess_kernels import SENT, covered, layout, score_ref, score_run

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")

# float32 bit patterns: quiet NaN, negative quiet NaN, a NaN whose payload sits only in the 13 bits TF32 drops (trunc_tf32 makes it inf)
POISON = {"nan": 0x7FC00000, "-nan": 0xFFC00000, "nan_low_payload": 0x7F800001, "+inf": 0x7F800000, "-inf": 0xFF800000}
INF = ("+inf", "-inf")


def poison(a, rows, cols, kind):
    """a copy of float32 `a` with the cells (rows x cols) set to the bit pattern of `kind`."""
    a = np.array(a, dtype=np.float32)
    bits = a.view(np.uint32)
    bits[np.ix_(np.atleast_1d(rows), np.atleast_1d(cols))] = POISON[kind]
    return a


def same_class_and_close(got, want, mag, name):
    """NaN, +inf, -inf and finite in exactly the same elements; the finite ones within parity_helpers.close."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    for what, f in (("NaN", np.isnan), ("+inf", np.isposinf), ("-inf", np.isneginf)):
        np.testing.assert_array_equal(f(got), f(want), err_msg=f"{name}: {what} elements differ")
    fin = np.isfinite(want)
    close(got[fin], want[fin], mag, name=name)


def out_map(jobs, out_rows):
    """For every output row: the x row it reads (-1 where no job writes) and its slot."""
    xrow, slot = np.full(out_rows, -1), np.full(out_rows, -1)
    for j in jobs:
        o, n = int(j["out_row"]), int(j["n_rows"])
        xrow[o:o + n] = np.arange(int(j["x_row"]), int(j["x_row"]) + n)
        slot[o:o + n] = int(j["slot"])
    return xrow, slot


def assert_rows_equal(got, clean, rows, variant, name):
    """`rows` of every output bit-identical between two launches."""
    for k in clean:
        np.testing.assert_array_equal(got[k][rows], clean[k][rows], err_msg=f"{name}: {k}")


# ------------------------------------------------------------------------------------------------ Dense kernels
# variant, dims: the generic kernel with 24 tags (column-order row sums, not a shuffle tree) and a hidden width it pads to 24, the row-per-thread kernel, the
# tensor-core kernel at 32 tags and at 36 tags (zero-padded to the next MMA width)
DENSE_CASES = {"v1": (1, [24, 21, 24]), "v3": (3, [8, 6, 8]), "v2_T32": (2, [32, 24, 32]), "v2_T36": (2, [36, 29, 36])}


def dense_layout(engine):
    # slot, n_rows, x_row, out_row: slots 0 and 1 read the overlapping x rows 60..159; jobs end inside a 64-row tile (x 160, 207, 301)
    # and inside a 16-row output box (out 150, 300, 347, 490); x rows 160..169 and 207..210 belong to no job
    return engine.make_jobs([0, 1, 0, 2], [150, 100, 37, 90], [10, 60, 170, 211], [0, 200, 310, 400])


# first row of a job (10, 60: both slots read row 60), last row of a job (206), rows just past a job's end that a tile reads (160, 207),
# a row inside a job (250)
X_POISON_ROWS = [10, 60, 160, 206, 207, 250]


def dense_case(engine, case, seed=0):
    from oracle import keras_math as km

    variant, dims = DENSE_CASES[case]
    acts = ["tanh"] * (len(dims) - 2) + ["linear"]
    nets = [dense_net(km, dims, acts, 40 + s) for s in range(3)]
    rng = np.random.default_rng(seed)
    X = rng.random((320, dims[0])).astype(np.float32)
    y = rng.random((320, dims[-1])).astype(np.float32)
    scale, feat, agg = score_inputs(rng, 3, dims[-1])
    return variant, nets, X, y, scale, feat, agg, dense_layout(engine), 500


@pytest.mark.parametrize("kind", list(POISON))
@pytest.mark.parametrize("case", list(DENSE_CASES))
def test_dense_poisoned_x_rows_stay_in_their_rows(engine, torch, case, kind):
    from oracle import anomaly_math as am
    from oracle import keras_math as km

    variant, nets, X, y, scale, feat, agg, jobs, out_rows = dense_case(engine, case)
    spec, weights = nets[0][0], [w for _, w in nets]
    Xp = poison(X, X_POISON_ROWS, [5], kind)  # one cell per row: two infinities of opposite weight make a NaN in Keras too
    clean = run_dense(engine, torch, spec, weights, X, y, jobs, scale, feat, agg, out_rows, variant, nan_fill=True)
    got = run_dense(engine, torch, spec, weights, Xp, y, jobs, scale, feat, agg, out_rows, variant, nan_fill=True)
    xrow, slot = out_map(jobs, out_rows)
    hit = np.isin(xrow, X_POISON_ROWS)
    assert hit.sum() == 5  # rows 10, 206, 250 once, row 60 by two slots; rows 160 and 207 belong to no job
    assert_rows_equal(got, clean, (xrow >= 0) & ~hit, variant, f"{case} {kind}: rows without poison")
    for k, v in got.items():
        assert np.isnan(v[xrow < 0]).all(), f"{k} written outside the jobs"
    for o in np.flatnonzero(hit):
        name = f"{case} {kind}: out row {o} (x row {xrow[o]})"
        if kind not in INF or variant == 2:
            # NaN in x, and ±inf on the tensor-core kernel (its TF32 + BF16 split of layer 0 computes inf - inf): an all-NaN row
            for k, v in got.items():
                assert np.isnan(v[o]).all(), f"{name}: {k} = {v[o]}"
            continue
        s = slot[o]
        with np.errstate(all="ignore"):
            want_out = km.ff_forward(spec, weights[s], Xp[xrow[o]:xrow[o] + 1], np.float64)
            want = am.anomaly_arrays(want_out, y[xrow[o]:xrow[o] + 1], scale[s].astype(np.float64), np.zeros(scale.shape[1]), feat[s], float(agg[s]))
        assert np.isfinite(want_out).all()  # tanh(±inf) = ±1: Keras answers with a finite row
        finite = lambda a: np.abs(a[np.isfinite(a)]).max(initial=1.0)  # noqa: E731
        m, d, smax = finite(want_out), finite(want["tag-anomaly-unscaled"]), float(scale[s].max())
        tot = 2 * m * d * smax ** 2
        mags = {"model-output": m, "tag-anomaly-unscaled": m, "tag-anomaly-scaled": m * smax, "anomaly-confidence": m / float(feat[s].min()),
                "total-anomaly-unscaled": 2 * m * d, "total-anomaly-scaled": tot, "total-anomaly-confidence": tot / float(agg[s])}
        same_class_and_close(got["model-output"][o:o + 1], want_out, m, f"{name}: model-output")
        for k in SCORE:
            same_class_and_close(got[k][o:o + 1].reshape(want[k].shape), want[k], mags[k], f"{name}: {k}")


@pytest.mark.parametrize("kind", list(POISON))
@pytest.mark.parametrize("case", list(DENSE_CASES))
def test_dense_poisoned_y_cells_stay_in_their_cells(engine, torch, case, kind):
    variant, nets, X, y, scale, feat, agg, jobs, out_rows = dense_case(engine, case, seed=1)
    spec, weights = nets[0][0], [w for _, w in nets]
    cols = [1, y.shape[1] - 1]
    yp = poison(y, X_POISON_ROWS, cols, kind)
    clean = run_dense(engine, torch, spec, weights, X, y, jobs, scale, feat, agg, out_rows, variant, nan_fill=True)
    got = run_dense(engine, torch, spec, weights, X, yp, jobs, scale, feat, agg, out_rows, variant, nan_fill=True)
    xrow, _ = out_map(jobs, out_rows)
    hit = np.isin(xrow, X_POISON_ROWS)
    np.testing.assert_array_equal(got["model-output"], clean["model-output"])
    assert_rows_equal(got, clean, (xrow >= 0) & ~hit, variant, f"{case} {kind}: rows without poison")
    others = np.setdiff1d(np.arange(y.shape[1]), cols)
    inf = kind in INF
    for k in SCORE:
        v = got[k][hit]
        if k in PER_ROW:
            # the numpy mean over every tag: NaN with a NaN cell, +inf with an infinite one
            assert (np.isposinf(v) if inf else np.isnan(v)).all(), f"{case} {kind}: {k} = {v}"
        else:
            np.testing.assert_array_equal(v[:, others], clean[k][hit][:, others], err_msg=f"{case} {kind}: {k}, the row's other tags")
            assert (np.isposinf(v[:, cols]) if inf else np.isnan(v[:, cols])).all(), f"{case} {kind}: {k} = {v[:, cols]}"


# ------------------------------------------------------------------------------------------------ gb_anomaly_score / _f64
@pytest.mark.parametrize("kind", list(POISON))
@pytest.mark.parametrize("side", ["y", "yhat"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_anomaly_score_poison_stays_in_its_cells(engine, torch, dtype, side, kind):
    """Ragged jobs (test_gpu_postprocess_kernels.layout): a poisoned y cell (read at x_row) or yhat cell (read at out_row) changes that
    cell's tag columns and its row's totals, nothing else; a poisoned y row that no job reads changes nothing."""
    T = 33
    rng = np.random.default_rng(9)
    jobs, n_slots, xt, ot = layout(engine, [1, 70, 1100, 37])
    yhat, y = rng.random((ot, T)).astype(np.float32), rng.random((xt, T)).astype(np.float32)
    scale, feat, agg = rng.uniform(0.5, 2, (n_slots, T)), rng.uniform(0.05, 0.3, (n_slots, T)), rng.uniform(0.01, 0.1, n_slots)
    j = jobs
    if side == "y":  # the one-row job, the first and last row of a long job, the first row of the last job, a row between jobs
        rows = [int(j[0]["x_row"]), int(j[2]["x_row"]), int(j[2]["x_row"] + j[2]["n_rows"] - 1), int(j[3]["x_row"]), int(j[3]["x_row"]) - 1]
        assert not covered(jobs, "x_row", xt)[rows[-1]]
        y = poison(y, rows, [0, 31], kind)
    else:
        rows = [int(j[0]["out_row"]), int(j[1]["out_row"] + 35), int(j[2]["out_row"] + j[2]["n_rows"] - 1)]
        yhat = poison(yhat, rows, [0, 31], kind)
    cast = [np.asarray(a, dtype) for a in (yhat, y, scale, feat, agg)]
    keys = tuple(score_ref(jobs, *cast, ot))
    clean_in = [np.asarray(a, dtype) for a in (np.nan_to_num(yhat, nan=0.5, posinf=0.5, neginf=0.5), np.nan_to_num(y, nan=0.5, posinf=0.5, neginf=0.5))]
    got = score_run(engine, torch, jobs, *cast[:2], *cast[2:], ot, keys)
    clean = score_run(engine, torch, jobs, *clean_in, *cast[2:], ot, keys)
    with np.errstate(all="ignore"):
        want = score_ref(jobs, *cast, ot)
    hit_out = np.zeros(ot, bool)
    for jb in jobs:
        o, x, n = int(jb["out_row"]), int(jb["x_row"]), int(jb["n_rows"])
        src = np.arange(x, x + n) if side == "y" else np.arange(o, o + n)
        hit_out[o:o + n] = np.isin(src, rows)
    assert hit_out.sum() == (4 if side == "y" else 3)
    for k in keys:
        g, w = got[k], want[k]
        if k in ("total-anomaly-scaled", "total-anomaly-unscaled", "total-anomaly-confidence"):
            same_class_and_close(g[hit_out], w[hit_out], 0.0, f"{side} {kind}: {k}")
            np.testing.assert_array_equal(g[~hit_out], clean[k][~hit_out], err_msg=k)
        else:
            np.testing.assert_array_equal(g, w, err_msg=k)  # one rounding per cell: NaN where NaN, inf where inf, equal elsewhere
            np.testing.assert_array_equal(g[:, 1:31], clean[k][:, 1:31], err_msg=k)
            np.testing.assert_array_equal(g[~hit_out], clean[k][~hit_out], err_msg=k)
    assert (got["tag-anomaly-unscaled"][~covered(jobs, "out_row", ot)] == SENT).all()


# ------------------------------------------------------------------------------------------------ LSTM kernels
@pytest.mark.parametrize("kind", list(POISON))
@pytest.mark.parametrize("cells", ["tanh", "sigmoid"])
@pytest.mark.parametrize("variant", [1, 2])
def test_lstm_poisoned_x_rows_stay_in_their_windows(engine, torch, variant, cells, kind):
    from oracle import keras_math as km

    L = 4
    nets = [lstm_net(km, 6, [16, 12], [cells, cells], 6, "linear", L, 80 + s) for s in range(2)]
    spec, weights = nets[0][0], [w for _, w in nets]
    X = np.random.default_rng(10).random((300, 6)).astype(np.float32)
    # slot, windows, x_row, out_row: both slots over x rows 30..122, a second job of slot 0 further on
    jobs = engine.make_jobs([0, 1, 0], [120, 90, 50], [0, 30, 200], [0, 130, 240])
    # a job's first row, a row both slots read, the last row both slots' windows read, a row between jobs, a row inside a job
    rows = [0, 31, 122, 150, 230]
    Xp = poison(X, rows, [2], kind)
    clean = run_lstm(engine, torch, spec, weights, X, jobs, 300, variant)
    got = run_lstm(engine, torch, spec, weights, Xp, jobs, 300, variant)
    n_hit = 0
    for jb in jobs:
        s, n, xr, o = (int(jb[k]) for k in ("slot", "n_rows", "x_row", "out_row"))
        start = np.arange(xr, xr + n)
        hit = np.array([any(w <= r < w + L for r in rows) for w in start])
        n_hit += hit.sum()
        np.testing.assert_array_equal(got[o:o + n][~hit], clean[o:o + n][~hit], err_msg=f"slot {s}: windows without poison")
        if kind not in INF or variant == 2:
            # NaN in x, and ±inf on the tensor-core kernel (KerasLSTMBaseEstimator.predict launches the fp32 kernel for ±inf): NaN windows
            assert np.isnan(got[o:o + n][hit]).all(), f"slot {s}: the windows holding the poisoned row must be NaN"
            continue
        with np.errstate(all="ignore"):
            want = lstm_oracle(km, spec, weights[s], Xp, xr, n)[hit]
        same_class_and_close(got[o:o + n][hit], want, 1.0, f"variant {variant} {cells} {kind} slot {s}")
    assert n_hit == (1 + 4 + 1) + (2 + 1) + 4  # row 150 lies in no window


# ------------------------------------------------------------------------------------------------ request coalescer
@pytest.mark.parametrize("kind", list(POISON))
def test_coalescer_poisoned_request_leaves_the_others_alone(engine, torch, kind):
    """One batch of four requests, one of them with poisoned x and y rows: every other request equals its own launch bit for bit."""
    from oracle import keras_math as km

    from gordo_components_b200.serving import AnomalyCoalescer

    spec = km.ff_hourglass_spec(32)
    nets = [dense_net(km, spec.dims, spec.acts, 60 + s)[1] for s in range(3)]
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    params = eng.pack_params(nets)
    rng = np.random.default_rng(11)
    scale, feat, agg = (torch.from_numpy(a).to(eng.device) for a in score_inputs(rng, 3, 32))
    reqs = [(s, rng.random((n, 32)).astype(np.float32), rng.random((n, 32)).astype(np.float32)) for s, n in ((0, 70), (2, 100), (1, 33), (0, 129))]
    s, Xr, yr = reqs[1]
    reqs[1] = (s, poison(Xr, [0, 64, 99], [3], kind), poison(yr, [5, 64], [7], kind))
    co = AnomalyCoalescer(eng, params, scale, feat, agg, max_wait_ms=500.0)
    try:
        futs = [co.submit(s, X, y) for s, X, y in reqs]
        got = [f.result() for f in futs]
        assert co.batches == 1
    finally:
        co.close()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)  # noqa: E731
    for i, (s, X, y) in enumerate(reqs):
        n = len(X)
        own = eng.infer_score(params, engine.jobs_to_device(engine.make_jobs([s], [n], [0], [0]), eng.device), 1, n, t(X), t(y), scale, feat, agg,
                              want=co.want)
        own = {k: v.cpu().numpy() for k, v in own.items()}
        for k in co.want:
            np.testing.assert_array_equal(got[i][k], own[k], err_msg=f"request {i}: {k}")
    bad = got[1]
    assert np.isnan(bad["model-output"][[0, 64, 99]]).all()  # the tensor-core kernel: NaN and ±inf in x give NaN rows
    assert np.isfinite(bad["model-output"][[1, 5, 63, 65, 98]]).all()


# ------------------------------------------------------------------------------------------------ detector and server
def fixture_frames(g):
    cols = [f"tag-{i}" for i in range(g["X"].shape[1])]
    index = pd.date_range("2019-01-01", periods=len(g["X"]), freq="10min", tz="UTC")
    return pd.DataFrame(g["X"], columns=cols, index=index), pd.DataFrame(g["y"], columns=cols, index=index)


def fixture_detector(g, window=None, method=None):
    """This package's detector with the fixture's network weights, error scaler and thresholds."""
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    dims = [int(d) for d in g["net_dims"]]
    ae = KerasAutoEncoder(kind="feedforward_hourglass")
    ae.kwargs.update({"n_features": dims[0], "n_features_out": dims[-1]})
    ae.set_weights([(g[f"W{l}"], g[f"b{l}"]) for l in range(len(dims) - 1)])
    assert list(ae.model.spec.dims) == dims
    X, y = fixture_frames(g)
    det = DiffBasedAnomalyDetector(base_estimator=ae, scaler=MinMaxScaler().fit(y), window=window, smoothing_method=method)
    np.testing.assert_allclose(det.scaler.scale_, g["scale"], rtol=1e-12)
    det.feature_thresholds_ = pd.Series(g["feature_thresholds"], index=X.columns)
    det.aggregate_threshold_ = float(g["aggregate_threshold"])
    return det


def assert_frame_follows_fixture(frame_block, g, smax):
    """Every column block against the reference's frame: the same NaN positions, the rest at the parity tolerances."""
    tot = float(np.nanmax(g["frame_total-anomaly-scaled"]))
    totu = float(np.nanmax(g["frame_total-anomaly-unscaled"]))
    mags = {"model-output": 1.0, "tag-anomaly-scaled": smax, "tag-anomaly-unscaled": 1.0, "total-anomaly-scaled": smax * np.sqrt(tot),
            "total-anomaly-unscaled": np.sqrt(totu), "anomaly-confidence": float((1 / g["feature_thresholds"]).max()),
            "total-anomaly-confidence": smax * np.sqrt(tot) / float(g["aggregate_threshold"])}
    checked = []
    for top in (str(s) for s in g["columns_level0"]):
        base = top[len("smooth-"):] if top.startswith("smooth-") else top
        if base not in mags:
            continue
        got = frame_block(top)
        if got is None:
            continue
        want = g[f"frame_{top}"].reshape(got.shape)
        np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=f"{top}: NaN positions")
        close(got, want, mags[base], name=top)
        checked.append(top)
    return checked


def test_detector_frame_with_missing_values_follows_the_reference(engine, torch):
    g = np.load(os.path.join(GOLDEN, "ffnet_anomaly_nan.npz"))
    det = fixture_detector(g, window=int(g["window"]), method=str(g["method"]))
    X, y = fixture_frames(g)
    frame = det.anomaly(X, y, frequency=pd.Timedelta("10min"))
    assert [str(s) for s in g["columns_level0"]] == list(dict.fromkeys(frame.columns.get_level_values(0)))
    checked = assert_frame_follows_fixture(lambda top: frame[top].values.astype(np.float64), g, float(g["scale"].max()))
    assert len(checked) == 11
    # the totals are finite on every row with at least one target (the row of nothing but NaN targets stays NaN)
    t = frame[("total-anomaly-scaled", "")].values
    assert np.isnan(t).sum() == np.isnan(g["frame_total-anomaly-scaled"]).sum() < np.isnan(np.asarray(g["y"]).sum(axis=1)).sum()


def test_server_frame_with_missing_values_follows_the_reference(engine, torch, tmp_path):
    """The fixture as JSON requests (NaN literals), per request and through a ResidentBucket (whose models have no smoothing window)."""
    from gordo_components_b200 import serializer, server

    g = np.load(os.path.join(GOLDEN, "ffnet_anomaly_nan.npz"))
    X, y = fixture_frames(g)
    meta = {"dataset": {"tag_list": list(X.columns), "resolution": "10min"}}
    serializer.dump(fixture_detector(g, int(g["window"]), str(g["method"])), str(tmp_path / "smoothed"), metadata={"name": "smoothed", **meta})
    serializer.dump(fixture_detector(g), str(tmp_path / "plain"), metadata={"name": "plain", **meta})
    store = server.ModelStore(str(tmp_path))
    payload = json.loads(json.dumps({"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(y)}))
    bucket = server.ResidentBucket(store, names=["plain"])
    try:
        for name, kw in (("smoothed", {}), ("plain", {}), ("plain", {"bucket": bucket})):
            reply = server.anomaly_prediction(store, name, json=payload, all_columns=True, **kw)
            assert reply.status == 200, reply.body
            got = server.dataframe_from_dict(reply.body["data"])
            tops = set(got.columns.get_level_values(0))
            checked = assert_frame_follows_fixture(lambda top: got[top].values.astype(np.float64) if top in tops else None, g, float(g["scale"].max()))
            assert len(checked) == (11 if name == "smoothed" else 7), (name, checked)
        assert bucket.coalescer.requests == 1
    finally:
        bucket.close()


def test_fold_thresholds_with_missing_targets_follow_the_reference(engine, torch):
    """gb_thresholds on the fixture's fold predictions with NaN targets: the numpy row mean (NaN rows) that cross_validate needs,
    rolling minima over windows without a NaN, their maximum -- the reference's per-fold thresholds."""
    g = np.load(os.path.join(GOLDEN, "ffnet_anomaly_nan.npz"))
    dev = engine.cuda_device()
    y = np.ascontiguousarray(g["y"], dtype=np.float32)
    T = y.shape[1]
    tlen = int(g["fold0_test_len"])
    starts = [int(g[f"fold{i}_test_start"]) for i in range(3)]
    pred = np.ascontiguousarray(np.concatenate([g[f"fold{i}_pred"] for i in range(3)]), dtype=np.float32)
    ytest = np.ascontiguousarray(np.concatenate([y[s:s + tlen] for s in starts]))
    assert np.isnan(ytest).any() and np.isnan(pred).any()
    scale = np.ascontiguousarray(np.stack([g[f"fold{i}_scale"] for i in range(3)]), dtype=np.float32)
    jd = engine.jobs_to_device(engine.make_jobs([0, 1, 2], [tlen] * 3, [0, tlen, 2 * tlen]), dev)
    res = engine.anomaly_score(jd, 3, tlen, torch.from_numpy(pred).to(dev), torch.from_numpy(ytest).to(dev), T, torch.from_numpy(scale).to(dev),
                               want=("tag-anomaly-unscaled", "total-anomaly-scaled"))
    feat, agg = engine.thresholds(jd, 3, tlen, res["tag-anomaly-unscaled"], res["total-anomaly-scaled"], T, 3, 6, dev)
    close(feat.cpu().numpy(), g["feature_thresholds_per_fold"], rtol=2e-5, mag=1e-3, name="feature thresholds per fold")
    close(agg.cpu().numpy(), g["aggregate_thresholds_per_fold"], rtol=1e-4, mag=1e-4, name="aggregate thresholds per fold")
    assert np.isfinite(feat.cpu().numpy()).all() and np.isfinite(agg.cpu().numpy()).all()


def _nan_targets(y, rng):
    y = np.array(y, dtype=np.float64)
    y.flat[rng.choice(y.size, size=15, replace=False)] = np.nan
    y[7] = np.nan
    return y


def _check_against_oracle(frame, pred, y, det, name):
    """Every score block of `frame` against oracle/anomaly_math (pandas' totals) at float64 precision."""
    from oracle import anomaly_math as am

    want = am.anomaly_arrays(pred, y, det.scaler.scale_, det.scaler.min_, det.feature_thresholds_.values, det.aggregate_threshold_)
    for k, w in want.items():
        if k == "model-output":
            continue
        got = frame[k].values.astype(np.float64).reshape(w.shape)
        np.testing.assert_array_equal(np.isnan(got), np.isnan(w), err_msg=f"{name}: {k} NaN positions")
        np.testing.assert_allclose(got, w, rtol=1e-9, atol=1e-12, equal_nan=True, err_msg=f"{name}: {k}")
    assert np.isfinite(frame[("total-anomaly-confidence", "")].values).sum() > len(pred) - 3


def test_foreign_estimator_detector_with_missing_targets(engine, torch):
    """A scikit-learn base estimator: float64 scoring (gb_anomaly_score_f64), pandas' totals where targets are missing."""
    from sklearn.linear_model import LinearRegression
    from sklearn.multioutput import MultiOutputRegressor

    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector

    rng = np.random.default_rng(12)
    X, y = pd.DataFrame(rng.random((120, 4))), pd.DataFrame(rng.random((120, 4)) * 3)
    det = DiffBasedAnomalyDetector(base_estimator=MultiOutputRegressor(LinearRegression())).fit(X, y)
    det.feature_thresholds_, det.aggregate_threshold_ = pd.Series(rng.uniform(0.1, 0.5, 4)), 0.2
    yn = _nan_targets(y.values, rng)
    frame = det.anomaly(X, pd.DataFrame(yn))
    _check_against_oracle(frame, det.predict(X), yn, det, "foreign estimator")


def test_lstm_detector_with_missing_targets(engine, torch):
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasLSTMAutoEncoder

    rng = np.random.default_rng(13)
    X = pd.DataFrame(rng.random((90, 4)))
    det = DiffBasedAnomalyDetector(base_estimator=KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=3, epochs=1, encoding_layers=1)).fit(X, X)
    det.feature_thresholds_, det.aggregate_threshold_ = pd.Series(rng.uniform(0.1, 0.5, 4)), 0.2
    yn = _nan_targets(X.values, rng)
    frame = det.anomaly(X, pd.DataFrame(yn))
    pred = det.predict(X)
    assert len(pred) == 88
    _check_against_oracle(frame, pred, yn, det, "LSTM")
    # ±inf in X saturates the gates (the fp32 kernel, as in Keras): finite windows, and the windows before the row are unchanged
    Xi = X.copy()
    Xi.iat[40, 1] = np.inf
    got = det.predict(Xi)
    assert np.isfinite(got).all()
    close(got[:38], pred[:38], 1.0, name="LSTM windows before the infinite row")


def _served_dense(tmp_path, pipeline=False):
    """A detector around a 32-tag hourglass (the tensor-core kernel's range), saved in a model store, and its request frames."""
    from oracle import keras_math as km
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200 import serializer, server
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    spec = km.ff_hourglass_spec(32)
    spec, w = dense_net(km, spec.dims, spec.acts, 70)
    ae = KerasAutoEncoder(kind="feedforward_hourglass")
    ae.kwargs.update({"n_features": 32, "n_features_out": 32})
    ae.set_weights(w)
    rng = np.random.default_rng(14)
    cols = [f"t{i}" for i in range(32)]
    idx = pd.date_range("2020-01-01", periods=150, freq="10min", tz="UTC")
    X, y = pd.DataFrame(rng.random((150, 32)), columns=cols, index=idx), pd.DataFrame(rng.random((150, 32)), columns=cols, index=idx)
    base = Pipeline([("scale", MinMaxScaler().fit(X)), ("ae", ae)]) if pipeline else ae
    det = DiffBasedAnomalyDetector(base_estimator=base, scaler=MinMaxScaler().fit(y))
    det.feature_thresholds_, det.aggregate_threshold_ = pd.Series(rng.uniform(0.2, 0.6, 32), index=cols), 0.1
    name = "pipe" if pipeline else "bare"
    serializer.dump(det, str(tmp_path / name), metadata={"name": name, "dataset": {"tag_list": cols, "resolution": "10min"}})
    return server.ModelStore(str(tmp_path)), name, det, spec, w, X, y


def _payload(X, y):
    from gordo_components_b200 import server

    return json.loads(json.dumps({"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(y)}))


@pytest.mark.parametrize("kind", INF)
def test_infinite_targets_and_scaled_inputs_are_refused(engine, torch, tmp_path, kind):
    """sklearn's scalers refuse ±inf, and the reference scales y, the model output and (behind a scaler pipeline) X with them."""
    from gordo_components_b200 import server

    v = np.inf if kind == "+inf" else -np.inf
    store, name, det, *_, X, y = _served_dense(tmp_path)
    yi = y.copy()
    yi.iloc[40, 3] = v
    bucket = server.ResidentBucket(store, names=[name])
    try:
        with pytest.raises(ValueError, match="infinity"):
            det.anomaly(X, yi)
        with pytest.raises(ValueError, match="infinity"):
            server.anomaly_prediction(store, name, json=_payload(X, yi))
        with pytest.raises(ValueError, match="infinity"):
            server.anomaly_prediction(store, name, json=_payload(X, yi), bucket=bucket)
        assert bucket.coalescer.requests == 0
        assert server.anomaly_prediction(store, name, json=_payload(X, y), bucket=bucket).status == 200  # the bucket still serves
    finally:
        bucket.close()
    pstore, pname, pdet, *_, X, y = _served_dense(tmp_path, pipeline=True)
    Xi = X.copy()
    Xi.iloc[[0, 99], 5] = v
    for call in (lambda: pdet.anomaly(Xi, y), lambda: server.anomaly_prediction(pstore, pname, json=_payload(Xi, y))):
        with pytest.raises(ValueError, match="infinity"):
            call()
    Xn = X.copy()
    Xn.iloc[[0, 99], 5] = np.nan  # NaN passes the scalers: NaN rows
    frame = pdet.anomaly(Xn, y)
    assert np.isnan(frame["model-output"].values[[0, 99]]).all() and np.isfinite(frame["model-output"].values[1:99]).all()


@pytest.mark.parametrize("kind", INF)
def test_bare_model_with_infinite_inputs_answers_like_the_oracle(engine, torch, tmp_path, kind):
    """tanh(±inf) = ±1: the reference's Keras model answers ±inf inputs with finite outputs, and so does this package -- per request
    and through a ResidentBucket, whose coalescer would otherwise hand the rows to the tensor-core kernel."""
    from oracle import anomaly_math as am
    from oracle import keras_math as km

    from gordo_components_b200 import server

    store, name, det, spec, w, X, y = _served_dense(tmp_path)
    Xi = X.copy()
    for r, c in ((3, 0), (64, 17), (149, 31)):  # one per row: two infinities of opposite weight would make a NaN in Keras too
        Xi.iat[r, c] = np.inf if kind == "+inf" else -np.inf
    Xi.iat[70, 9] = np.nan
    with np.errstate(all="ignore"):
        want_out = km.ff_forward(spec, w, Xi.values, np.float64)
    want = am.anomaly_arrays(want_out, y.values, det.scaler.scale_, det.scaler.min_, det.feature_thresholds_.values, det.aggregate_threshold_)
    assert np.isfinite(want_out[[3, 64, 149]]).all() and np.isnan(want_out[70]).all()
    bucket = server.ResidentBucket(store, names=[name])
    try:
        frames = {"detector": det.anomaly(Xi, y)}
        for label, kw in (("per request", {}), ("bucket", {"bucket": bucket})):
            reply = server.anomaly_prediction(store, name, json=_payload(Xi, y), **kw)
            assert reply.status == 200
            frames[label] = server.dataframe_from_dict(reply.body["data"])
    finally:
        bucket.close()
    smax = float(det.scaler.scale_.max())
    for label, frame in frames.items():
        same_class_and_close(frame["model-output"].values, want_out, 1.0, f"{label}: model-output")
        for k, mag in (("tag-anomaly-scaled", smax), ("tag-anomaly-unscaled", 1.0), ("total-anomaly-scaled", 2 * smax ** 2),
                       ("total-anomaly-unscaled", 2.0), ("anomaly-confidence", 1 / float(det.feature_thresholds_.min())),
                       ("total-anomaly-confidence", 2 * smax ** 2 / det.aggregate_threshold_)):
            same_class_and_close(frame[k].values.astype(np.float64).reshape(want[k].shape), want[k], mag, f"{label}: {k}")
