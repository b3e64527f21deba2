"""
Build -> model directory -> ModelStore -> the two POST views, JSON and parquet, on the GPU
(tests/gordo/server/test_anomaly_view.py:14-120, test_gordo_server.py).  Kept in a file of its own that sorts after the
kernel parity tests.
"""
import json

import numpy as np
import pandas as pd
import pytest

from test_gpu_builder import DETECTOR, _series

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


def test_built_models_answer_requests(engine, torch, tmp_path):
    """Build -> directory -> ModelStore -> the two POST views, JSON and parquet (tests/gordo/server/test_anomaly_view.py:14-120)."""
    from gordo_components_b200 import builder, server

    N, T = 240, 4

    class Dataset:
        def __init__(self, frame):
            self.frame = frame

        def get_data(self):
            return self.frame, self.frame

        def get_metadata(self):
            return {"rows": len(self.frame)}

        def to_dict(self):
            return {"type": "TimeSeriesDataset", "tag_list": [{"name": c, "asset": None} for c in self.frame.columns], "resolution": "10min"}

    frames = {n: _series(N, T, seed) for seed, n in enumerate(["m-1", "m-2"])}
    builder.FleetModelBuilder([{"name": n, "model": DETECTOR, "dataset": Dataset(f)} for n, f in frames.items()]).build(str(tmp_path))
    store = server.ModelStore(str(tmp_path))
    assert store.names() == ["m-1", "m-2"] and store.tags("m-2") == list(frames["m-2"].columns)
    assert store.metadata("m-1")["metadata"]["build_metadata"]["dataset"]["dataset_meta"] == {"rows": N}

    X = frames["m-2"].iloc[100:140].astype(np.float64)
    want = store.model("m-2").anomaly(X, X, frequency=store.frequency("m-2"))
    reply = server.anomaly_prediction(store, "m-2", json={"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(X)})
    assert reply.status == 200 and reply.content_type == "application/json" and float(reply.body["time-seconds"]) > 0
    json.dumps(reply.body)
    got = server.dataframe_from_dict(reply.body["data"])
    assert set(got.columns.get_level_values(0)) == set(want.columns.get_level_values(0))
    for block in ("model-output", "tag-anomaly-scaled", "total-anomaly-confidence", "anomaly-confidence"):
        np.testing.assert_array_equal(got[block].values.ravel(), want[block].values.ravel())
    assert list(got["start"].values.ravel()) == list(want["start"].values.ravel())

    # parquet in, parquet out; unlabelled columns are accepted when the width fits (utils.py:206-247)
    unlabelled = X.copy()
    unlabelled.columns = [str(i) for i in range(T)]
    files = {"X": server.dataframe_into_parquet_bytes(unlabelled), "y": server.dataframe_into_parquet_bytes(X)}
    reply = server.anomaly_prediction(store, "m-2", files=files, fmt="parquet")
    assert reply.status == 200 and reply.content_type == "application/octet-stream"
    frame = server.dataframe_from_parquet_bytes(reply.body)
    np.testing.assert_array_equal(frame["total-anomaly-scaled"].values.ravel(), want["total-anomaly-scaled"].values.ravel())
    assert not any(c[0].startswith("smooth-") for c in frame.columns)

    # the plain prediction view
    reply = server.prediction(store, "m-1", json={"X": server.dataframe_to_dict(frames["m-1"].iloc[:10].astype(np.float64))})
    assert reply.status == 200 and set(reply.body["data"]) == {"start", "end", "model-input", "model-output"}
    out = server.dataframe_from_dict(reply.body["data"])
    np.testing.assert_array_equal(out["model-output"].values.ravel(), store.model("m-1").predict(frames["m-1"].iloc[:10]).astype(np.float64).ravel())
    assert server.anomaly_prediction(store, "m-1", json={"X": server.dataframe_to_dict(X[list(X.columns[:2])]), "y": server.dataframe_to_dict(X)}).status == 400


def test_detector_build_equals_the_reference_build(engine, torch):
    """
    ModelBuilder on a DiffBasedAnomalyDetector around a scikit-learn model, against the reference's ModelBuilder._build with the
    reference's own detector (tests/golden/callers.json "build_detector", produced by tests/golden/make_golden.py): the scores come
    from the same CPU predictions (1e-9); thresholds and anomaly columns come from this package's float64 kernels (1e-9).
    """
    import os

    from gordo_components_b200 import builder

    golden = os.path.join(os.path.dirname(__file__), "golden")
    with open(os.path.join(golden, "callers.json")) as f:
        meta = json.load(f)
    arrays = np.load(os.path.join(golden, "callers.npz"))
    info, want = meta["build_frame"], meta["build_detector"]
    frame = pd.DataFrame(arrays["build_frame"], index=pd.date_range(info["start"], periods=info["rows"], freq=info["freq"]), columns=info["columns"])
    model, built = builder.ModelBuilder({"name": "fixture-detector", "model": want["model"], "dataset": (frame, frame),
                                         "evaluation": meta["build"]["default"]["evaluation"]}).build()
    got = built["metadata"]["build_metadata"]["model"]
    assert got["model_offset"] == want["model_offset"] == 0
    assert list(got["cross_validation"]["scores"]) == list(want["scores"])
    for key, stats in want["scores"].items():
        for stat, value in stats.items():
            np.testing.assert_allclose(got["cross_validation"]["scores"][key][stat], value, rtol=1e-9, atol=1e-12, err_msg=f"{key} {stat}")
    mm, ref = got["model_meta"], want["model_meta"]
    assert set(mm) == set(ref)
    # a scikit-learn base estimator: predictions, scaler and every anomaly column are float64 here as in the reference
    # (gb_anomaly_score_f64 / gb_thresholds_f64), although the targets sit at magnitude ~100 with residuals of ~1e-3
    np.testing.assert_allclose(mm["feature-thresholds"], ref["feature-thresholds"], rtol=1e-9)
    np.testing.assert_allclose(mm["aggregate-threshold"], ref["aggregate-threshold"], rtol=1e-9)
    for fold, value in ref["aggregate-thresholds-per-fold"].items():
        np.testing.assert_allclose(mm["aggregate-thresholds-per-fold"][fold], value, rtol=1e-9)
    for tag, folds in ref["feature-thresholds-per-fold"].items():
        for fold, value in folds.items():
            np.testing.assert_allclose(mm["feature-thresholds-per-fold"][tag][fold], value, rtol=1e-9)
    anomaly = model.anomaly(frame.iloc[-50:], frame.iloc[-50:], frequency=pd.Timedelta("10min"))
    np.testing.assert_allclose(np.asarray(anomaly["tag-anomaly-scaled"], dtype=np.float64), arrays["build_detector_tag_scaled"], rtol=1e-9, atol=1e-15)
    np.testing.assert_allclose(np.asarray(anomaly["total-anomaly-confidence"], dtype=np.float64).ravel(), arrays["build_detector_total_confidence"], rtol=1e-9)


def test_bucket_of_resident_models_answers_like_single_requests(engine, torch, tmp_path):
    """server.ResidentBucket: many threads, several models, one coalescer -- every reply equals the model's own answer."""
    from concurrent.futures import ThreadPoolExecutor

    from gordo_components_b200 import builder, server

    N, T = 240, 4
    frames = {f"m-{i}": _series(N, T, 10 + i) for i in range(3)}
    machines = [{"name": n, "model": DETECTOR, "dataset": (f, f)} for n, f in frames.items()]
    machines.append({"name": "lstm", "model": {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": {
        "gordo.machine.model.models.KerasLSTMAutoEncoder": {"kind": "lstm_hourglass", "lookback_window": 3, "epochs": 1, "encoding_layers": 1}}}},
        "dataset": (frames["m-0"], frames["m-0"])})
    builder.FleetModelBuilder(machines).build(str(tmp_path))
    store = server.ModelStore(str(tmp_path))
    bucket = server.ResidentBucket(store)
    try:
        assert bucket.names == ["m-0", "m-1", "m-2"]  # the LSTM model is served on its own path
        payloads = {}
        for n, f in frames.items():
            X = f.iloc[50:90].astype(np.float64)
            payloads[n] = {"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(X)}
        want = {n: json.dumps(server.anomaly_prediction(store, n, json=p).body["data"]) for n, p in payloads.items()}
        order = [n for _ in range(8) for n in payloads]
        with ThreadPoolExecutor(8) as ex:
            got = list(ex.map(lambda n: json.dumps(server.anomaly_prediction(store, n, json=payloads[n], bucket=bucket).body["data"]), order))
        assert got == [want[n] for n in order]
        assert bucket.coalescer.requests == len(order) and bucket.coalescer.batches <= len(order)
        Xl = frames["m-0"].iloc[:20].astype(np.float64)
        lstm = server.anomaly_prediction(store, "lstm", json={"X": server.dataframe_to_dict(Xl), "y": server.dataframe_to_dict(Xl)}, bucket=bucket)
        assert lstm.status == 200 and len(lstm.body["data"]["total-anomaly-scaled"]["total-anomaly-scaled"]) == 18
    finally:
        bucket.close()
