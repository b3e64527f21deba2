"""
TransformedTargetRegressor detectors served through the request coalescer (``ResidentBucket(target_scaler=True)``): a TTR around a
bare autoencoder and around ``Pipeline([MinMaxScaler, autoencoder])``, as plain detectors and as K-fold detectors (window 144, smm),
and the reference's production definition built by ``FleetModelBuilder(kfcv=True, early_stopping=True)`` and loaded from disk.
Replies through a bucket equal the per-request route's byte for byte, in JSON and parquet, with and without the smoothed columns;
the refusals (±inf in y, in X, in the raw prediction, after the inverse) raise the same exception with the same message on both
routes.  Kept in a file of its own that sorts after the kernel tests.
"""
import json
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

T = 4


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("needs an H100")
    import __graft_entry__ as ge

    ge.build()
    return t


def _series(rows, seed, tags=T):
    rng = np.random.default_rng(seed)
    t = np.linspace(0, 25, rows)[:, None]
    values = (0.5 + 0.4 * np.sin(t * rng.uniform(0.5, 2, tags) + rng.uniform(0, 3, tags)) + rng.normal(0, 0.02, (rows, tags))) * rng.uniform(1, 50, tags)
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(values, index=idx, columns=[f"TAG {i}" for i in range(tags)])


def _ttr(piped):
    from sklearn.compose import TransformedTargetRegressor
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200.machine.model import models

    ae = models.KerasAutoEncoder(kind="feedforward_hourglass", epochs=1)
    reg = Pipeline([("s", MinMaxScaler()), ("m", ae)]) if piped else ae
    return TransformedTargetRegressor(transformer=MinMaxScaler(), regressor=reg)


@pytest.fixture(scope="module")
def store(torch, tmp_path_factory):
    from gordo_components_b200 import builder, serializer, server
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector, DiffBasedKFCVAnomalyDetector

    root = tmp_path_factory.mktemp("ttr-store")
    meta = {"dataset": {"tag_list": [f"TAG {t}" for t in range(T)], "resolution": "10min"}}

    def dump(name, det, seed, patch=None):
        frame = _series(400, seed)
        det.cross_validate(X=frame, y=frame)
        det.fit(frame, frame)
        if patch is not None:
            patch(det.base_estimator)
        serializer.dump(det, str(root / name), metadata=meta)

    for i in range(3):
        dump(f"bare-{i}", DiffBasedAnomalyDetector(base_estimator=_ttr(False)), i)
        dump(f"piped-{i}", DiffBasedAnomalyDetector(base_estimator=_ttr(True)), 10 + i)
        dump(f"kbare-{i}", DiffBasedKFCVAnomalyDetector(base_estimator=_ttr(False), window=144, smoothing_method="smm"), 20 + i)
        dump(f"kpiped-{i}", DiffBasedKFCVAnomalyDetector(base_estimator=_ttr(True), window=144, smoothing_method="smm"), 30 + i)

    def infinite_prediction(ttr):  # the network's last layer answers +inf for every input
        ae = ttr.regressor_.steps[-1][1]
        W, b = ae.model.weights[-1]
        ae.model.weights[-1] = (np.zeros_like(W), np.full_like(b, np.inf))

    def overflowing_inverse(ttr):  # tag 0 leaves float32 on the way back to the targets' units
        ttr.transformer_.scale_ = ttr.transformer_.scale_.copy()
        ttr.transformer_.scale_[0] = 1e-300

    dump("piped-infpred", DiffBasedAnomalyDetector(base_estimator=_ttr(True)), 40, infinite_prediction)
    dump("piped-overflow", DiffBasedAnomalyDetector(base_estimator=_ttr(True)), 41, overflowing_inverse)

    # the production definition, built in one batched bucket and loaded from disk
    ae = {"gordo.machine.model.models.KerasAutoEncoder": {
        "kind": "feedforward_hourglass", "batch_size": 128, "compression_factor": 0.5, "encoding_layers": 1, "func": "tanh", "out_func": "linear",
        "epochs": 4, "validation_split": 0.1,
        "callbacks": [{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "val_loss", "patience": 1, "min_delta": 0.5, "restore_best_weights": True}}]}}
    model = {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {
        "base_estimator": {"sklearn.compose.TransformedTargetRegressor": {
            "transformer": "sklearn.preprocessing.MinMaxScaler",
            "regressor": {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", ae]}}}},
        "scaler": "sklearn.preprocessing.MinMaxScaler", "window": 144, "shuffle": True, "threshold_percentile": 0.975}}
    evaluation = {"cv": {"sklearn.model_selection.KFold": {"n_splits": 5, "shuffle": True, "random_state": 0}}}
    machines = [{"name": f"prod-{i}", "model": model, "dataset": {"X": _series(800, 50 + i), "y": _series(800, 50 + i)}, "evaluation": evaluation}
                for i in range(3)]
    kroot = tmp_path_factory.mktemp("prod")
    builder.FleetModelBuilder(machines, kfcv=True, early_stopping=True).build(str(kroot))
    for m in machines:
        det = serializer.load(str(kroot / m["name"]))
        assert type(det).__name__ == "DiffBasedKFCVAnomalyDetector" and type(det.base_estimator).__name__ == "TransformedTargetRegressor"
        serializer.dump(det, str(root / m["name"]), metadata=meta)
    return server.ModelStore(str(root))


def _requests(names, n_req, seed, min_rows):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_req):
        rows = int(rng.integers(min_rows, 260))
        X = _series(rows, 1000 + seed * 100 + k)
        y = X.copy()
        if k % 5 == 0:
            X.iloc[int(rng.integers(rows)), int(rng.integers(T))] = np.nan
        if k % 7 == 3:
            y.iloc[int(rng.integers(rows)), int(rng.integers(T))] = np.nan  # with all_columns and a window: answered per request
        out.append((names[k % len(names)], X, y, k % 2 == 0, "parquet" if k % 3 == 0 else None))
    return out


def _reply(store, name, X, y, all_columns, fmt, bucket=None):
    from gordo_components_b200 import server

    if fmt == "parquet":
        files = {"X": server.dataframe_into_parquet_bytes(X), "y": server.dataframe_into_parquet_bytes(y)}
        r = server.anomaly_prediction(store, name, files=files, fmt="parquet", all_columns=all_columns, bucket=bucket)
        return r.status, r.body
    payload = {"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(y)}
    r = server.anomaly_prediction(store, name, json=payload, all_columns=all_columns, bucket=bucket)
    return r.status, json.dumps(r.body["data"])


GROUPS = {
    "bare": ({"target_scaler": True}, None),
    "piped": ({"input_scalers": True, "target_scaler": True}, None),
    "kbare": ({"smoothing": True, "target_scaler": True}, (144, "smm")),
    "kpiped": ({"input_scalers": True, "smoothing": True, "target_scaler": True}, (144, "smm")),
    "prod": ({"input_scalers": True, "smoothing": True, "target_scaler": True}, (144, "smm")),
}


def _members(store, prefix):
    return [n for n in store.names() if n.split("-")[0] == prefix and n.split("-")[-1].isdigit()]


def test_buckets_hold_the_ttr_models(store, torch):
    from gordo_components_b200 import server

    with pytest.raises(ValueError, match="no model"):
        server.ResidentBucket(store)  # the default bucket refuses every TTR model, as before
    with pytest.raises(ValueError, match="no model"):
        server.ResidentBucket(store, input_scalers=True, smoothing=True)
    b = server.ResidentBucket(store, input_scalers=True, smoothing=True, target_scaler=True)
    try:
        assert b.target_scaler and b.coalescer.y_inverse is not None and len(b.names) >= 3
    finally:
        b.close()


def test_ttr_replies_through_the_buckets_equal_the_per_request_route(store, torch):
    from gordo_components_b200 import server

    buckets = []
    try:
        for prefix, (kw, smoothing) in GROUPS.items():
            members = _members(store, prefix)
            b = server.ResidentBucket(store, names=members, max_wait_ms=20, **kw)
            buckets.append(b)
            assert sorted(b.names) == sorted(members) and b.smoothing == smoothing and b.target_scaler
        served = [n for b in buckets for n in b.names]
        work = _requests(served, 120, 1, 150) + _requests([n for n in served if n.startswith(("k", "prod"))], 16, 2, 10)
        want = [_reply(store, *job) for job in work]
        for (name, X, y, all_columns, fmt), (status, body) in zip(work, want):
            assert status == 200
            if fmt == "parquet":  # the frames the server parses out of the request
                Xp, yp = (server.dataframe_from_parquet_bytes(server.dataframe_into_parquet_bytes(f)) for f in (X, y))
            else:
                Xp, yp = (server.dataframe_from_dict(server.dataframe_to_dict(f)) for f in (X, y))
            frame = store.model(name).anomaly(Xp, yp, frequency=store.frequency(name))
            if not all_columns:
                frame = frame.drop(columns=[c for c in frame.columns if c[0] in server.DELETED_FROM_RESPONSE_COLUMNS])
            if fmt == "parquet":
                assert body == server.dataframe_into_parquet_bytes(frame)
            else:
                assert body == json.dumps(server.dataframe_to_dict(frame))
        with ThreadPoolExecutor(8) as ex:
            got = list(ex.map(lambda job: _reply(store, *job, bucket=buckets), work))
        for job, g, w in zip(work, got, want):
            assert g == w, job[0]
        for b in buckets:
            assert 0 < b.coalescer.batches < b.coalescer.requests  # several models answered from one batch
    finally:
        for b in buckets:
            b.close()


def _outcome(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001 - the exception itself is what is compared
        return type(e), str(e)
    return None


def test_refusals_match_the_per_request_route(store, torch):
    from gordo_components_b200 import server

    piped = server.ResidentBucket(store, names=_members(store, "piped") + ["piped-infpred", "piped-overflow"], input_scalers=True,
                                  target_scaler=True)
    bare = server.ResidentBucket(store, names=_members(store, "bare"), target_scaler=True)
    try:
        X = _series(50, 7)
        y_inf, X_inf = X.copy(), X.copy()
        y_inf.iloc[3, 1] = np.inf
        X_inf.iloc[4, 2] = -np.inf
        cases = [
            ("piped-0", X_inf, y_inf, piped, ValueError, "Input X contains infinity or a value too large for dtype('float64')."),  # y first
            ("piped-0", X_inf, X, piped, ValueError, "Input X contains infinity or a value too large for dtype('float64')."),
            ("piped-infpred", X, X, piped, ValueError, "Input contains infinity or a value too large for dtype('float32')."),
            ("piped-overflow", X, X, piped, ValueError, "Input X contains infinity or a value too large for dtype('float32')."),
        ]
        for name, Xr, yr, bucket, exc, msg in cases:
            model = store.model(name)
            want = _outcome(lambda: model.anomaly_blocks(Xr, yr, frequency=store.frequency(name)))
            got = _outcome(lambda: bucket.anomaly_blocks(store, name, Xr, yr, store.frequency(name)))
            assert want == (exc, msg), (name, want)
            assert got == want, name
        # ±inf in X before a bare regressor: answered on the per-request route, so the same reply
        assert _reply(store, "bare-1", X_inf, X, True, None, bucket=bare) == _reply(store, "bare-1", X_inf, X, True, None)
        n0 = bare.coalescer.requests
        assert _reply(store, "bare-1", X, X, False, None, bucket=bare) == _reply(store, "bare-1", X, X, False, None)
        assert bare.coalescer.requests == n0 + 1
        # a NaN in y works on both routes
        y_nan = X.copy()
        y_nan.iloc[5, 0] = np.nan
        for all_columns in (False, True):
            assert _reply(store, "piped-2", X, y_nan, all_columns, None, bucket=piped) == _reply(store, "piped-2", X, y_nan, all_columns, None)
    finally:
        piped.close()
        bare.close()
