"""
TransformedTargetRegressor LSTM detectors served through the LSTM request coalescer (``ResidentBucket(lstm=True,
target_scaler=True)``): a TTR around a bare autoencoder, a bare forecast, ``Pipeline([MinMaxScaler, autoencoder])`` and
``Pipeline([StandardScaler, forecast])``, smoothed ones (smm and ewma), detectors built by ``FleetModelBuilder(target_scaler=True,
smoothing=True)`` and loaded from disk, and a store that mixes them with feed-forward TTR and plain LSTM detectors.  Replies through
a bucket equal the per-request route's byte for byte, in JSON and parquet, with and without the smoothed columns; the refusals raise
the same exception with the same message on both routes.  Kept in a file of its own that sorts after the kernel tests.
"""
import json
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

T, L = 4, 6
META = {"dataset": {"tag_list": [f"TAG {t}" for t in range(T)], "resolution": "10min"}}


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("needs an H100")
    import __graft_entry__ as ge

    ge.build()
    return t


def _series(rows, seed):
    rng = np.random.default_rng(seed)
    t = np.linspace(0, 25, rows)[:, None]
    values = (0.5 + 0.4 * np.sin(t * rng.uniform(0.5, 2, T) + rng.uniform(0, 3, T)) + rng.normal(0, 0.02, (rows, T))) * rng.uniform(1, 50, T)
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(values, index=idx, columns=[f"TAG {i}" for i in range(T)])


def _ttr(kind, pre=None, transformer=None):
    from sklearn.compose import TransformedTargetRegressor
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import MinMaxScaler, StandardScaler

    from gordo_components_b200.machine.model import models

    net = getattr(models, kind)(kind="lstm_hourglass", lookback_window=L, epochs=1, encoding_layers=2)
    reg = net if pre is None else Pipeline([("scale", {"minmax": MinMaxScaler, "standard": StandardScaler}[pre]()), ("net", net)])
    return TransformedTargetRegressor(transformer=transformer if transformer is not None else MinMaxScaler(), regressor=reg)


FORMS = {  # prefix -> (network, leading step)
    "ae": ("KerasLSTMAutoEncoder", None),
    "fc": ("KerasLSTMForecast", None),
    "pae": ("KerasLSTMAutoEncoder", "minmax"),
    "sfc": ("KerasLSTMForecast", "standard"),
}


@pytest.fixture(scope="module")
def store(torch, tmp_path_factory):
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200 import serializer, server
    from gordo_components_b200.machine.model import models
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector

    root = tmp_path_factory.mktemp("lstm-ttr-store")

    def dump(name, det, seed, patch=None):
        frame = _series(300, seed)
        if det.require_thresholds:
            det.cross_validate(X=frame, y=frame)
        det.fit(frame, frame)
        if patch is not None:
            patch(det.base_estimator)
        serializer.dump(det, str(root / name), metadata=META)

    seed = 0
    for prefix, (kind, pre) in FORMS.items():
        for i in range(2):
            dump(f"{prefix}-{i}", DiffBasedAnomalyDetector(base_estimator=_ttr(kind, pre)), seed)
            seed += 1
    # the inverse is (p - min_) / scale_ whatever the transformer's range
    dump("range-0", DiffBasedAnomalyDetector(base_estimator=_ttr("KerasLSTMAutoEncoder", transformer=MinMaxScaler(feature_range=(-1, 1)))), 20)
    for method in ("smm", "ewma"):
        for i in range(2):
            dump(f"{method}-{i}", DiffBasedAnomalyDetector(base_estimator=_ttr("KerasLSTMForecast", "minmax"), window=12, smoothing_method=method),
                 30 + seed)
            seed += 1

    def infinite_prediction(ttr):  # the dense head answers +inf for every window
        net = ttr.regressor_.steps[-1][1]
        layers, (W, b) = net.model.weights
        net.model.weights = (layers, (np.zeros_like(W), np.full_like(b, np.inf)))

    def overflowing_inverse(ttr):  # tag 0 leaves float32 on the way back to the targets' units
        ttr.transformer_.scale_ = ttr.transformer_.scale_.copy()
        ttr.transformer_.scale_[0] = 1e-300

    dump("bad-infpred", DiffBasedAnomalyDetector(base_estimator=_ttr("KerasLSTMAutoEncoder", "minmax")), 40, infinite_prediction)
    dump("bad-overflow", DiffBasedAnomalyDetector(base_estimator=_ttr("KerasLSTMAutoEncoder", "minmax")), 41, overflowing_inverse)

    # a feed-forward TTR and plain LSTM detectors in the same store
    from sklearn.compose import TransformedTargetRegressor

    for i in range(2):
        ff = TransformedTargetRegressor(transformer=MinMaxScaler(), regressor=models.KerasAutoEncoder(kind="feedforward_hourglass", epochs=1))
        dump(f"ffttr-{i}", DiffBasedAnomalyDetector(base_estimator=ff), 50 + i)
        plain = models.KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=L, epochs=1, encoding_layers=2)
        dump(f"plain-{i}", DiffBasedAnomalyDetector(base_estimator=plain), 60 + i)
    return server.ModelStore(str(root))


def _members(store, *prefixes):
    return [n for n in store.names() if n.split("-")[0] in prefixes]


def _reply(store, name, X, y, all_columns, fmt, bucket=None):
    from gordo_components_b200 import server

    if fmt == "parquet":
        files = {"X": server.dataframe_into_parquet_bytes(X), "y": server.dataframe_into_parquet_bytes(y)}
        r = server.anomaly_prediction(store, name, files=files, fmt="parquet", all_columns=all_columns, bucket=bucket)
        return r.status, r.body
    payload = {"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(y)}
    r = server.anomaly_prediction(store, name, json=payload, all_columns=all_columns, bucket=bucket)
    return r.status, json.dumps(r.body["data"]) if r.status == 200 else r.body


def _requests(names, n_req, seed):
    """Requests over ``names`` in every reply form (JSON / parquet, ``all_columns`` off / on), some with a NaN in X or y."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_req):
        rows = int(rng.integers(L + 2, 200))
        X = _series(rows, 1000 + seed * 100 + k)
        y = X.copy()
        if k % 5 == 0:
            X.iloc[int(rng.integers(rows)), int(rng.integers(T))] = np.nan
        if k % 7 == 3:
            y.iloc[int(rng.integers(rows)), int(rng.integers(T))] = np.nan  # with all_columns and a window: answered per request
        out.append((names[k % len(names)], X, y, (k // 2) % 2 == 0, "parquet" if k % 2 else None))
    return out


def _check_against_per_request(store, buckets, work, threads=8):
    want = [_reply(store, *job) for job in work]
    assert all(status == 200 for status, _ in want)
    with ThreadPoolExecutor(threads) as ex:
        got = list(ex.map(lambda job: _reply(store, *job, bucket=buckets), work))
    for job, g, w in zip(work, got, want):
        assert g == w, (job[0], job[3], job[4])


def test_bucket_holds_the_ttr_lstm_models(store, torch):
    from gordo_components_b200 import server

    plain = server.ResidentBucket(store, lstm=True)  # refuses every TTR, as before
    ttr = server.ResidentBucket(store, lstm=True, target_scaler=True)
    try:
        assert sorted(plain.names) == _members(store, "plain") and not plain.target_scaler and plain.coalescer.y_inverse is None
        assert sorted(ttr.names) == _members(store, "ae", "fc", "pae", "sfc", "range", "bad")  # the largest group
        assert ttr.lstm and ttr.target_scaler and ttr.smoothing is None and ttr.coalescer.y_inverse is not None
    finally:
        plain.close()
        ttr.close()


def test_replies_through_the_buckets_equal_the_per_request_route(store, torch):
    from gordo_components_b200 import server

    plain = _members(store, "ae", "fc", "pae", "sfc", "range")
    buckets = [server.ResidentBucket(store, names=plain, lstm=True, target_scaler=True, max_wait_ms=50)]
    for method in ("smm", "ewma"):
        buckets.append(server.ResidentBucket(store, names=_members(store, method), lstm=True, smoothing=True, target_scaler=True, max_wait_ms=50))
    try:
        assert [b.smoothing for b in buckets] == [None, (12, "smm"), (12, "ewma")] and all(b.target_scaler for b in buckets)
        work = _requests(plain, 64, 1) + _requests(_members(store, "smm", "ewma"), 32, 2)
        _check_against_per_request(store, buckets, work)
        for b in buckets:
            assert 0 < b.coalescer.batches < b.coalescer.requests  # requests of several threads and slots answered from one batch
    finally:
        for b in buckets:
            b.close()


def _outcome(fn):
    try:
        r = fn()
    except Exception as e:  # noqa: BLE001 - the exception itself is what is compared
        return type(e), str(e)
    return r.status, json.dumps(r.body.get("data", r.body))


def test_refusals_match_the_per_request_route(store, torch):
    from gordo_components_b200 import server

    bucket = server.ResidentBucket(store, lstm=True, target_scaler=True)
    try:
        X = _series(60, 7)
        y_inf, X_inf = X.copy(), X.copy()
        y_inf.iloc[3, 1] = np.inf
        X_inf.iloc[4, 2] = -np.inf
        short = X.iloc[:L]
        inf32 = "Input contains infinity or a value too large for dtype('float32')."
        cases = [  # name, X, y, what the per-request route answers
            ("pae-0", X_inf, y_inf, (ValueError, "Input X contains infinity or a value too large for dtype('float64').")),  # y first
            ("ae-0", X, y_inf, (ValueError, "Input X contains infinity or a value too large for dtype('float64').")),
            ("pae-0", X_inf, X, (ValueError, "Input X contains infinity or a value too large for dtype('float64').")),  # the step's own
            ("sfc-0", X_inf, X, (ValueError, "Input X contains infinity or a value too large for dtype('float64').")),
            ("ae-0", short, short, (ValueError, "For KerasLSTMForecast lookback_window must be < size of X")),
            ("pae-1", short, short, (ValueError, "For KerasLSTMForecast lookback_window must be < size of X")),
            ("bad-infpred", X, X, (ValueError, inf32)),  # sklearn's inverse_transform on the raw prediction
            ("bad-overflow", X, X, (ValueError, "Input X contains infinity or a value too large for dtype('float32').")),  # after it
        ]
        before = bucket.coalescer.requests
        for name, Xr, yr, expected in cases:
            payload = {"X": server.dataframe_to_dict(Xr), "y": server.dataframe_to_dict(yr)}
            want = _outcome(lambda: server.anomaly_prediction(store, name, json=payload))
            got = _outcome(lambda: server.anomaly_prediction(store, name, json=payload, bucket=bucket))
            assert want == expected, (name, want)
            assert got == want, name
        assert bucket.coalescer.requests == before + 2  # only the two overflow cases reached the launch
        # the raw prediction comes back beside an infinite inverse, so the two overflows can be told apart
        Xv = np.asarray(X.values, dtype=np.float32)
        raw = bucket.coalescer.anomaly(bucket.slot["bad-infpred"], Xv, X.values[-(len(Xv) - L + 1):])
        assert np.isposinf(raw["raw-model-output"]).all() and np.isinf(raw["model-output"]).all()
        over = bucket.coalescer.anomaly(bucket.slot["bad-overflow"], Xv, X.values[-(len(Xv) - L + 1):])
        assert np.isfinite(over["raw-model-output"]).all() and np.isinf(over["model-output"][:, 0]).all()
        assert "raw-model-output" not in bucket.coalescer.anomaly(bucket.slot["ae-0"], Xv, X.values[-(len(Xv) - L + 1):])
        # ±inf in X before a bare regressor: answered on the per-request route (the fp32 kernel), so the same reply
        n0 = bucket.coalescer.requests
        for all_columns in (False, True):
            for fmt in (None, "parquet"):
                assert _reply(store, "ae-1", X_inf, X, all_columns, fmt, bucket=bucket) == _reply(store, "ae-1", X_inf, X, all_columns, fmt)
        assert bucket.coalescer.requests == n0
        assert _reply(store, "ae-1", X_inf, X, False, None)[0] == 200
    finally:
        bucket.close()


def test_nan_in_x_and_y(store, torch):
    from gordo_components_b200 import server

    buckets = [server.ResidentBucket(store, names=_members(store, "ae", "fc", "pae", "sfc"), lstm=True, target_scaler=True),
               server.ResidentBucket(store, names=_members(store, "smm"), lstm=True, smoothing=True, target_scaler=True)]
    try:
        X = _series(80, 8)
        X_nan, y_nan = X.copy(), X.copy()
        X_nan.iloc[10, 1] = np.nan
        y_nan.iloc[30, 2] = np.nan
        for name in ("ae-0", "fc-1", "pae-0", "sfc-1", "smm-0"):
            for Xr, yr in ((X_nan, X), (X, y_nan), (X_nan, y_nan)):
                for all_columns in (False, True):
                    for fmt in (None, "parquet"):
                        assert _reply(store, name, Xr, yr, all_columns, fmt, bucket=buckets) == _reply(store, name, Xr, yr, all_columns, fmt), name
    finally:
        for b in buckets:
            b.close()


def test_one_store_three_buckets(store, torch):
    """Feed-forward TTR, plain LSTM and TTR LSTM detectors of one store, each answered from its own bucket."""
    from gordo_components_b200 import server

    ff = server.ResidentBucket(store, target_scaler=True)
    lstm = server.ResidentBucket(store, lstm=True)
    lstm_ttr = server.ResidentBucket(store, lstm=True, target_scaler=True)
    buckets = [ff, lstm, lstm_ttr]
    try:
        assert sorted(ff.names) == _members(store, "ffttr") and sorted(lstm.names) == _members(store, "plain")
        names = ["ffttr-0", "plain-1", "ae-0", "sfc-1", "ffttr-1", "plain-0", "range-0", "pae-1"]
        work = []
        for k, name in enumerate(names):
            X = _series(40 + 13 * k, 300 + k)
            for all_columns in (False, True):
                for fmt in (None, "parquet"):
                    work.append((name, X, X, all_columns, fmt))
        _check_against_per_request(store, buckets, work, threads=4)
        assert [b.coalescer.requests for b in buckets] == [4 * 2, 4 * 2, 4 * 4]
    finally:
        for b in buckets:
            b.close()


def test_fleet_built_detectors_serve_through_the_bucket(torch, tmp_path):
    from gordo_components_b200 import builder, serializer, server

    DET = "gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector"

    def definition(cls_name, piped, **kw):
        net = {f"gordo.machine.model.models.{cls_name}": {"kind": "lstm_hourglass", "lookback_window": 5, "epochs": 2, "batch_size": 16}}
        reg = {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", net]}} if piped else net
        return {DET: {"base_estimator": {"sklearn.compose.TransformedTargetRegressor": {
            "transformer": "sklearn.preprocessing.MinMaxScaler", "regressor": reg}}, **kw}}

    models = {"fc": definition("KerasLSTMForecast", True, window=12, smoothing_method="sma"), "ae": definition("KerasLSTMAutoEncoder", False)}
    machines = [{"name": f"{kind}-{i}", "model": models[kind], "dataset": {"X": _series(200, 70 + 10 * j + i), "y": _series(200, 70 + 10 * j + i)}}
                for j, kind in enumerate(models) for i in range(3)]
    builder.FleetModelBuilder(machines, target_scaler=True, smoothing=True).build(str(tmp_path / "built"))
    for m in machines:
        det = serializer.load(str(tmp_path / "built" / m["name"]))
        assert type(det.base_estimator).__name__ == "TransformedTargetRegressor"
        serializer.dump(det, str(tmp_path / "served" / m["name"]), metadata=META)
    store = server.ModelStore(str(tmp_path / "served"))
    fc = server.ResidentBucket(store, names=[f"fc-{i}" for i in range(3)], lstm=True, smoothing=True, target_scaler=True, max_wait_ms=20)
    ae = server.ResidentBucket(store, names=[f"ae-{i}" for i in range(3)], lstm=True, target_scaler=True, max_wait_ms=20)
    try:
        assert len(fc.names) == len(ae.names) == 3 and fc.smoothing == (12, "sma") and fc.target_scaler and ae.target_scaler
        _check_against_per_request(store, [fc, ae], _requests(fc.names + ae.names, 24, 5))
        assert fc.coalescer.requests > 0 and ae.coalescer.requests > 0
    finally:
        fc.close()
        ae.close()
