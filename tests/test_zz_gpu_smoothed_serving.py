"""
Smoothing-window detectors served through the request coalescers (``ResidentBucket(smoothing=True)``): windowed feed-forward models,
bare and behind a scaler Pipeline, windowed LSTM autoencoder and forecast models, and K-fold detectors built by the batched fleet
builder and loaded from disk.  Replies through a bucket equal the per-request route's byte for byte, with and without the smoothed
columns, in JSON and parquet; the per-request replies equal the model's own anomaly frame.  Kept in a file of its own that sorts
after the kernel tests.
"""
import json
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

T, L = 4, 5


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


AE = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 1}}
KFCV = {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {"base_estimator": AE, "window": 144, "smoothing_method": "smm"}}


@pytest.fixture(scope="module")
def store(torch, tmp_path_factory):
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200 import builder, serializer, server
    from gordo_components_b200.machine.model import models
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector

    root = tmp_path_factory.mktemp("smoothed-store")
    meta = {"dataset": {"tag_list": [f"TAG {t}" for t in range(T)], "resolution": "10min"}}

    def dump(name, det, seed):
        frame = _series(400, seed)
        det.cross_validate(X=frame, y=frame)
        det.fit(frame, frame)
        serializer.dump(det, str(root / name), metadata=meta)

    for i in range(3):
        dump(f"ff-smm-{i}", DiffBasedAnomalyDetector(base_estimator=models.KerasAutoEncoder(kind="feedforward_hourglass", epochs=1), window=12), i)
        dump(f"ff-pipe-sma-{i}", DiffBasedAnomalyDetector(
            base_estimator=Pipeline([("s", MinMaxScaler()), ("m", models.KerasAutoEncoder(kind="feedforward_hourglass", epochs=1))]),
            window=7, smoothing_method="sma"), 10 + i)
    for i, kind in enumerate(("KerasLSTMAutoEncoder", "KerasLSTMForecast", "KerasLSTMAutoEncoder")):
        net = getattr(models, kind)(kind="lstm_hourglass", lookback_window=L, epochs=1, encoding_layers=2)
        dump(f"lstm-ewma-{i}", DiffBasedAnomalyDetector(base_estimator=net, window=9, smoothing_method="ewma"), 20 + i)
    dump("ff-plain", DiffBasedAnomalyDetector(base_estimator=models.KerasAutoEncoder(kind="feedforward_hourglass", epochs=1)), 30)
    evaluation = {"cv": {"sklearn.model_selection.KFold": {"n_splits": 5, "shuffle": True, "random_state": 0}}}
    machines = [{"name": f"kfold-{i}", "model": KFCV, "dataset": {"X": _series(600, 40 + i), "y": _series(600, 40 + i)}, "evaluation": evaluation}
                for i in range(3)]
    kroot = tmp_path_factory.mktemp("kfold")
    builder.FleetModelBuilder(machines, kfcv=True).build(str(kroot))
    for m in machines:
        det = serializer.load(str(kroot / m["name"]))
        assert type(det).__name__ == "DiffBasedKFCVAnomalyDetector" and det.window == 144
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
            y.iloc[int(rng.integers(rows)), int(rng.integers(T))] = np.nan  # with all_columns: answered per request
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


def test_buckets_group_the_windowed_models(store, torch):
    from gordo_components_b200 import server

    default = server.ResidentBucket(store)
    try:
        assert default.names == ["ff-plain"] and default.smoothing is None  # windowed models stay out of a default bucket
    finally:
        default.close()
    b = server.ResidentBucket(store, input_scalers=True, smoothing=True)
    try:
        assert len(b.names) == 3 and b.smoothing in ((12, "smm"), (7, "sma"), (144, "smm"))
    finally:
        b.close()


def test_smoothed_replies_through_the_buckets_equal_the_per_request_route(store, torch):
    from gordo_components_b200 import server

    names = store.names()
    groups = {
        "ff": ([n for n in names if n.startswith("ff-smm-")], {}, (12, "smm")),
        "pipe": ([n for n in names if n.startswith("ff-pipe-")], {"input_scalers": True}, (7, "sma")),
        "lstm": ([n for n in names if n.startswith("lstm-")], {"lstm": True}, (9, "ewma")),
        "kfold": ([n for n in names if n.startswith("kfold-")], {}, (144, "smm")),
    }
    buckets = []
    try:
        for members, kw, smoothing in groups.values():
            b = server.ResidentBucket(store, names=members, smoothing=True, max_wait_ms=20, **kw)
            buckets.append(b)
            assert sorted(b.names) == sorted(members) and b.smoothing == smoothing
        served = [n for members, _, _ in groups.values() for n in members]
        work = _requests(served, 96, 1, 150) + _requests([n for n in served if n.startswith("kfold-")], 16, 2, 10)
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
            assert any(c[0].startswith("smooth-") for c in frame.columns) == all_columns
            if fmt == "parquet":
                assert body == server.dataframe_into_parquet_bytes(frame)
            else:
                assert body == json.dumps(server.dataframe_to_dict(frame))
        with ThreadPoolExecutor(8) as ex:
            got = list(ex.map(lambda job: _reply(store, *job, bucket=buckets), work))
        for job, g, w in zip(work, got, want):
            assert g == w, job[0]
        for b in buckets:
            assert 0 < b.coalescer.batches < b.coalescer.requests
    finally:
        for b in buckets:
            b.close()


def test_coalescer_smooths_only_the_requests_that_ask(store, torch):
    from gordo_components_b200 import server

    bucket = server.ResidentBucket(store, names=[n for n in store.names() if n.startswith("ff-smm-")], smoothing=True, max_wait_ms=50)
    try:
        co = bucket.coalescer
        reqs = [(_series(n, 500 + n), k % 2 == 1) for k, n in enumerate((30, 200, 150, 5, 64, 300))]
        futs = [co.submit(k % 3, X.values, X.values, smooth=s) for k, (X, s) in enumerate(reqs)]
        res = [f.result() for f in futs]
        assert co.batches < len(reqs)
        for k, ((X, s), r) in enumerate(zip(reqs, res)):
            assert any(key.startswith("smooth-") for key in r) == s
            if s:
                model = store.model(bucket.names[k % 3])
                for key in ("tag-anomaly-scaled", "total-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-unscaled"):
                    assert r["smooth-" + key].tobytes() == model._smoothing(r[key]).tobytes(), key
    finally:
        bucket.close()
