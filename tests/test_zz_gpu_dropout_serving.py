"""
KerasRawModelRegressor detectors with Dropout layers served through the request coalescer (``ResidentBucket``).  Inference runs
without dropout, so a dropout detector is served as any raw detector is: a reply through the bucket equals the per-request
route's byte for byte.  Kept in a file of its own that sorts after the kernel tests, since the buckets start coalescer threads.
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


def _kind():
    return {"compile": {"loss": "mse", "optimizer": "adam"}, "spec": {"tensorflow.keras.models.Sequential": {"layers": [
        {"tensorflow.keras.layers.Dropout": {"rate": 0.1}},
        {"tensorflow.keras.layers.Dense": {"units": 6, "activation": "tanh"}},
        {"tensorflow.keras.layers.Dropout": {"rate": 0.4}},
        {"tensorflow.keras.layers.Dense": {"units": T}}]}}}


def test_dropout_detectors_reply_through_a_bucket_as_per_request(torch, tmp_path):
    from sklearn.model_selection import TimeSeriesSplit

    from gordo_components_b200 import serializer, server
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasRawModelRegressor

    tags = [f"TAG {i}" for i in range(T)]
    names = ["drop-0", "drop-1", "drop-2"]
    for i, name in enumerate(names):
        X = _frame(300, i, tags)
        det = DiffBasedAnomalyDetector(base_estimator=KerasRawModelRegressor(_kind(), epochs=2))
        det.cross_validate(X=X, y=X, cv=TimeSeriesSplit(n_splits=3))
        det.fit(X, X)
        assert det.base_estimator.model.spec.dropout == [0.1, 0.4]
        serializer.dump(det, str(tmp_path / name), metadata={"name": name, "dataset": {"tag_list": tags, "target_tag_list": tags,
                                                                                          "resolution": "10min"}})
    store = server.ModelStore(str(tmp_path))
    assert all(server.ResidentBucket.eligible(store.model(n)) for n in names)
    b = server.ResidentBucket(store, names=names, max_wait_ms=20)
    try:
        assert sorted(b.names) == names
        for i, name in enumerate(b.names):
            X = _frame(120, 50 + i, tags)
            payload = json.loads(json.dumps({"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(X)}))
            direct = server.anomaly_prediction(store, name, json=payload)
            through = server.anomaly_prediction(store, name, json=payload, bucket=b)
            assert direct.status == through.status == 200
            assert json.dumps(through.body["data"]) == json.dumps(direct.body["data"])
            again = server.anomaly_prediction(store, name, json=payload, bucket=b)  # no mask in inference: the same reply again
            assert json.dumps(again.body["data"]) == json.dumps(direct.body["data"])
        assert b.coalescer.requests == 2 * len(b.names)
    finally:
        b.close()
