"""
KerasRawModelRegressor detectors served through the request coalescer (``ResidentBucket``): an autoencoder-shaped raw network and a
one-output regressor.  A reply through the bucket equals the per-request route's byte for byte.  Kept in a file of its own that
sorts after the kernel tests, since the buckets start coalescer threads.
"""
import json

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


def _frame(rows, seed, cols):
    rng = np.random.default_rng(seed)
    t = np.linspace(0, 25, rows)[:, None]
    values = 0.5 + 0.4 * np.sin(t * rng.uniform(0.5, 2, len(cols)) + rng.uniform(0, 3, len(cols))) + rng.normal(0, 0.02, (rows, len(cols)))
    return pd.DataFrame(values, index=pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC"), columns=cols)


def _kind(n_out):
    return {"compile": {"loss": "mse", "optimizer": "adam"}, "spec": {"tensorflow.keras.models.Sequential": {"layers": [
        {"tensorflow.keras.layers.Dense": {"units": 6, "activation": "tanh", "kernel_regularizer": "l2"}},
        {"tensorflow.keras.layers.Dense": {"units": n_out}}]}}}


def test_raw_detectors_reply_through_a_bucket_as_per_request(torch, tmp_path):
    from sklearn.model_selection import TimeSeriesSplit

    from gordo_components_b200 import serializer, server
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasRawModelRegressor

    tags = [f"TAG {i}" for i in range(T)]
    shapes = {"raw-ae-0": tags, "raw-ae-1": tags, "raw-one-0": ["TAG 0"], "raw-one-1": ["TAG 0"]}
    for i, (name, targets) in enumerate(shapes.items()):
        X = _frame(300, i, tags)
        y = X[targets]
        det = DiffBasedAnomalyDetector(base_estimator=KerasRawModelRegressor(_kind(len(targets)), epochs=2))
        det.cross_validate(X=X, y=y, cv=TimeSeriesSplit(n_splits=3))
        det.fit(X, y)
        serializer.dump(det, str(tmp_path / name), metadata={"name": name, "dataset": {"tag_list": tags, "target_tag_list": targets,
                                                                                          "resolution": "10min"}})
    store = server.ModelStore(str(tmp_path))
    buckets = []
    try:
        for prefix in ("raw-ae", "raw-one"):
            names = [n for n in store.names() if n.startswith(prefix)]
            assert all(server.ResidentBucket.eligible(store.model(n)) for n in names)
            b = server.ResidentBucket(store, names=names, max_wait_ms=20)
            assert sorted(b.names) == sorted(names)
            buckets.append(b)
        for b in buckets:
            for i, name in enumerate(b.names):
                X = _frame(120, 50 + i, tags)
                y = X[shapes[name]]
                payload = json.loads(json.dumps({"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(y)}))
                direct = server.anomaly_prediction(store, name, json=payload)
                through = server.anomaly_prediction(store, name, json=payload, bucket=b)
                assert direct.status == through.status == 200
                assert json.dumps(through.body["data"]) == json.dumps(direct.body["data"])
            assert b.coalescer.requests == len(b.names)
    finally:
        for b in buckets:
            b.close()
