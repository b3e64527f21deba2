"""
Smoothing-window detectors on the serving side, without a GPU: the argument checks of gb_smooth_scores, which detectors a
``ResidentBucket(smoothing=True)`` admits and how it groups them, the coalescers' smoothing options and jobs, and which requests
the bucket sends down the per-request route.
"""
import ctypes as C
import json

import numpy as np
import pandas as pd
import pytest

from gordo_components_b200 import _cabi, server

T = 4
TAGS = [f"tag-{i}" for i in range(T)]


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


# ------------------------------------------------------------------------------------------------ gb_smooth_scores arguments
FAKE = C.c_void_p(256)  # never dereferenced: every call below is refused, or has no job, before any launch


def _call(lib, **kw):
    a = dict(jobs=FAKE, n_jobs=2, max_rows=10, ts=FAKE, tots=FAKE, tu=FAKE, totu=FAKE, in_f64=0, n_tags=T, window=3, method=0,
             o_ts=FAKE, o_tots=FAKE, o_tu=FAKE, o_totu=FAKE)
    a.update(kw)
    return lib.gb_smooth_scores(a["jobs"], a["n_jobs"], a["max_rows"], a["ts"], a["tots"], a["tu"], a["totu"], a["in_f64"], a["n_tags"],
                                a["window"], a["method"], a["o_ts"], a["o_tots"], a["o_tu"], a["o_totu"], None)


@pytest.mark.parametrize("arg", ["jobs", "ts", "tots", "tu", "totu", "o_ts", "o_tots", "o_tu", "o_totu"])
def test_smooth_scores_refuses_null_pointers(lib, arg):
    assert _call(lib, **{arg: None}) == -1 and b"non-NULL" in lib.gb_last_error()


@pytest.mark.parametrize("kw, code, msg", [
    ({"in_f64": 2}, -1, b"in_f64"),
    ({"in_f64": -1}, -1, b"in_f64"),
    ({"n_tags": 0}, -1, b"n_tags"),
    ({"n_tags": (1 << 24) + 1}, -1, b"n_tags"),
    ({"window": 0}, -1, b"window"),
    ({"window": -144}, -1, b"window"),
    ({"method": 3}, -1, b"method"),
    ({"method": -1}, -1, b"method"),
    ({"n_jobs": -1}, -1, b"n_jobs"),
    ({"max_rows": -1}, -1, b"max_rows"),
    ({"max_rows": 65535 * 128 + 1}, -1, b"rows per job"),
    ({"window": 51201, "method": 0}, -4, b"rolling-median window"),
    ({"window": 51201, "method": 0, "n_jobs": 0}, -4, b"rolling-median window"),  # checked even when there is nothing to launch
])
def test_smooth_scores_refuses_bad_arguments(lib, kw, code, msg):
    assert _call(lib, **kw) == code and msg in lib.gb_last_error()
    with pytest.raises(ValueError):
        _cabi.check(code)


@pytest.mark.parametrize("kw", [{"n_jobs": 0}, {"max_rows": 0}, {"n_jobs": 0, "window": 51200}, {"n_jobs": 0, "window": 51201, "method": 1},
                                {"n_jobs": 0, "window": 51201, "method": 2}, {"n_jobs": 0, "in_f64": 1}])
def test_smooth_scores_accepts_empty_batches_without_a_launch(lib, kw):
    assert _call(lib, **kw) == 0


def test_engine_wrapper_checks_its_arrays(lib):
    import torch

    from gordo_components_b200 import engine

    good = {"tag-anomaly-scaled": torch.zeros(5, T), "total-anomaly-scaled": torch.zeros(5), "tag-anomaly-unscaled": torch.zeros(5, T),
            "total-anomaly-unscaled": torch.zeros(5)}
    with pytest.raises(ValueError, match="smoothing_method"):
        engine.smooth_scores(None, 1, 5, good, 3, "median")
    with pytest.raises(ValueError, match="float32 or four float64"):
        engine.smooth_scores(None, 1, 5, {**good, "total-anomaly-scaled": torch.zeros(5, dtype=torch.float64)}, 3, "smm")
    with pytest.raises(ValueError, match="float32 or four float64"):
        engine.smooth_scores(None, 1, 5, {k: v.to(torch.float16) for k, v in good.items()}, 3, "smm")
    with pytest.raises(ValueError, match="shapes"):
        engine.smooth_scores(None, 1, 5, {**good, "total-anomaly-unscaled": torch.zeros(4)}, 3, "smm")


# ------------------------------------------------------------------------------------------------ eligibility and grouping
def _ae(n=T):
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    ae = KerasAutoEncoder(kind="feedforward_hourglass")
    ae.kwargs.update({"n_features": n, "n_features_out": n})
    ae._prepare_model()
    return ae


def _lstm(n=T):
    from gordo_components_b200.machine.model.models import KerasLSTMAutoEncoder

    return KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=3, encoding_layers=1).initialize(n, n)


def _fitted(det, pre=()):
    rng = np.random.default_rng(0)
    for s in pre:
        s.fit(rng.random((8, T)) * 100)
    det.scaler.fit(rng.random((8, T)))
    det.feature_thresholds_, det.aggregate_threshold_ = pd.Series(np.ones(T), index=TAGS), 0.5
    return det


def _diff(est, window=None, method=None, pre=()):
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector

    return _fitted(DiffBasedAnomalyDetector(base_estimator=est, window=window, smoothing_method=method), pre)


def _kfcv(est, window=144, method="smm", pre=()):
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedKFCVAnomalyDetector

    return _fitted(DiffBasedKFCVAnomalyDetector(base_estimator=est, window=window, smoothing_method=method), pre)


def _piped(est):
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import MinMaxScaler

    scaler = MinMaxScaler()
    return Pipeline([("s", scaler), ("m", est)]), [scaler]


def test_feed_forward_eligibility(lib):
    ok = [_diff(_ae(), 144), _diff(_ae(), 6, "sma"), _diff(_ae(), 6, "ewma"), _diff(_ae(), np.int64(12), "smm"), _kfcv(_ae()),
          _kfcv(_ae(), 3, "ewma"), _diff(_ae(), 51200, "smm"), _diff(_ae(), 51201, "sma"), _diff(_ae(), 60000, "ewma")]
    for det in ok:
        assert server.ResidentBucket.eligible(det, smoothing=True), (det.window, det.smoothing_method)
        assert server.ResidentBucket.eligible(det, input_scalers=True, smoothing=True)
        assert not server.ResidentBucket.eligible(det)  # the default bucket takes no smoothing window, as before
        assert not server.ResidentBucket.eligible(det, input_scalers=True)
        assert not server.ResidentBucket.eligible_lstm(det, smoothing=True)
    for make in (_diff, _kfcv):
        est, pre = _piped(_ae())
        det = make(est, 144, "smm", pre=pre)
        assert server.ResidentBucket.eligible(det, input_scalers=True, smoothing=True)
        assert not server.ResidentBucket.eligible(det, smoothing=True)  # a Pipeline needs input_scalers=True, as before
        assert not server.ResidentBucket.eligible(det, input_scalers=True)
    refused = [_diff(_ae(), 12.0), _diff(_ae(), "12"), _diff(_ae(), True), _diff(_ae(), 0), _diff(_ae(), -6, "sma"),
               _diff(_ae(), 51201, "smm"), _kfcv(_ae(), 51201), _diff(_ae(), 6, "median"), _kfcv(_ae(), 6, None), _kfcv(_ae(), 6, "SMM")]
    for det in refused:
        assert not server.ResidentBucket.eligible(det, smoothing=True), (det.window, det.smoothing_method)
        assert not server.ResidentBucket.eligible(det, input_scalers=True, smoothing=True)
    plain = _diff(_ae())
    assert server.ResidentBucket.eligible(plain) and server.ResidentBucket.eligible(plain, smoothing=True)


def test_lstm_eligibility(lib):
    est, pre = _piped(_lstm())
    ok = [_diff(_lstm(), 6), _diff(_lstm(), 6, "ewma"), _kfcv(_lstm(), 144, "sma"), _diff(est, 6, "smm", pre=pre)]
    for det in ok:
        assert server.ResidentBucket.eligible_lstm(det, smoothing=True)
        assert not server.ResidentBucket.eligible_lstm(det)  # the default LSTM bucket is unchanged
        assert not server.ResidentBucket.eligible(det, input_scalers=True, smoothing=True)
    for det in (_diff(_lstm(), 0), _diff(_lstm(), 2.5), _diff(_lstm(), 51201), _diff(_lstm(), 6, "median")):
        assert not server.ResidentBucket.eligible_lstm(det, smoothing=True)
    assert server.ResidentBucket.eligible_lstm(_diff(_lstm()), smoothing=True)


def test_windowed_detectors_are_grouped_by_window_and_method(lib):
    est, pre = _piped(_ae())
    models = {
        "plain": _diff(_ae()),
        "smm-144": _diff(_ae(), 144), "kfcv-144": _kfcv(_ae()), "kfcv-144b": _kfcv(_ae()),  # one window, one method: one group
        "sma-144": _kfcv(_ae(), 144, "sma"),
        "smm-6": _diff(_ae(), 6),
        "piped-144": _kfcv(est, pre=pre),  # bare and Pipeline models never share a group
        "bad": _diff(_ae(), 0),
    }
    groups = server.ResidentBucket.ff_groups(models, input_scalers=True, smoothing=True)
    assert sorted(map(sorted, groups.values())) == [["kfcv-144", "kfcv-144b", "smm-144"], ["piped-144"], ["plain"], ["sma-144"], ["smm-6"]]
    assert max(groups.values(), key=len) == ["smm-144", "kfcv-144", "kfcv-144b"]
    assert {k[-1] for k in groups} == {None, (144, "smm"), (144, "sma"), (6, "smm")}
    assert list(server.ResidentBucket.ff_groups(models).values()) == [["plain"]]  # the default bucket

    lstm_models = {"plain": _diff(_lstm()), "w6": _diff(_lstm(), 6), "w6b": _kfcv(_lstm(), 6), "w6-ewma": _diff(_lstm(), 6, "ewma"),
                   "ff": _diff(_ae(), 6)}
    groups = server.ResidentBucket.lstm_groups(lstm_models, smoothing=True)
    assert sorted(map(sorted, groups.values())) == [["plain"], ["w6", "w6b"], ["w6-ewma"]]
    assert list(server.ResidentBucket.lstm_groups(lstm_models).values()) == [["plain"]]


# ------------------------------------------------------------------------------------------------ coalescer options
def _bare_coalescer(want=None):
    from gordo_components_b200.fleet import PER_ROW, PER_TAG
    from gordo_components_b200.serving import AnomalyCoalescer

    co = AnomalyCoalescer.__new__(AnomalyCoalescer)
    co.want = tuple(want) if want is not None else PER_TAG + PER_ROW
    return co


def test_coalescer_smoothing_option_is_checked():
    co = _bare_coalescer()
    assert co._check_smoothing(None) is None
    assert co._check_smoothing((144, "smm")) == (144, "smm")
    assert co._check_smoothing((np.int32(6), "ewma")) == (6, "ewma")
    assert co._check_smoothing((51201, "sma")) == (51201, "sma")
    for bad in ((0, "smm"), (2.0, "smm"), (True, "sma"), (6, "median"), (6, None), (51201, "smm")):
        with pytest.raises(ValueError):
            co._check_smoothing(bad)
    with pytest.raises(ValueError, match="total-anomaly-unscaled"):
        _bare_coalescer(want=("model-output", "tag-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-scaled"))._check_smoothing((6, "smm"))


def test_smooth_requests_need_a_smoothing_coalescer():
    import queue

    co = _bare_coalescer()
    co.params, co.smoothing, co._q, co._closed = np.zeros((2, 1)), None, queue.Queue(), False
    co._request = lambda X, y: (X, y)
    with pytest.raises(ValueError, match="without smoothing"):
        co.submit(0, np.zeros((3, T)), np.zeros((3, T)), smooth=True)
    co.submit(0, np.zeros((3, T)), np.zeros((3, T)))
    co.smoothing = (3, "smm")
    co.submit(1, np.zeros((3, T)), np.zeros((3, T)), smooth=True)
    assert [item[-2] for item in (co._q.get(), co._q.get())] == [False, True]


def test_smoothing_jobs_cover_exactly_the_requests_that_asked():
    co = _bare_coalescer()
    batch = [(0, None, None, False, None), (3, None, None, True, None), (1, None, None, False, None), (2, None, None, True, None),
             (2, None, None, False, None)]
    starts, counts = np.array([0, 10, 15, 40, 41]), np.array([10, 5, 25, 1, 7])
    jobs, lo, hi = co._smoothing_jobs(batch, starts, counts)
    assert (lo, hi) == (10, 41)
    assert jobs["n_rows"].tolist() == [5, 1] and jobs["out_row"].tolist() == [0, 30] and jobs["x_row"].tolist() == [0, 30]
    assert co._smoothing_jobs([(0, None, None, False, None)], [0], [10]) is None


# ------------------------------------------------------------------------------------------------ routing in the bucket

def _store(tmp_path, det):
    import pickle

    d = tmp_path / "w"
    d.mkdir()
    with open(d / "model.pkl", "wb") as f:
        pickle.dump(det, f)
    (d / "metadata.json").write_text(json.dumps({"dataset": {"tag_list": TAGS, "resolution": "10min"}}))
    return server.ModelStore(str(tmp_path))


def _scores(rows):
    rng = np.random.default_rng(rows)
    tags = rng.random((rows, T)).astype(np.float32)
    return {"model-output": rng.random((rows, T)).astype(np.float32), "tag-anomaly-scaled": tags, "tag-anomaly-unscaled": tags * 2,
            "total-anomaly-scaled": tags.mean(1), "total-anomaly-unscaled": tags.mean(1) * 2, "anomaly-confidence": tags,
            "total-anomaly-confidence": tags.mean(1)}


def _frame(rows, nan=False):
    idx = pd.date_range("2020-01-01", periods=rows, freq="10min", tz="UTC")
    f = pd.DataFrame(np.random.default_rng(1).random((rows, T)), index=idx, columns=TAGS)
    if nan:
        f.iloc[3, 1] = np.nan
    return f


def test_bucket_routes_smoothing_requests(tmp_path, monkeypatch):
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector

    store = _store(tmp_path, _kfcv(_ae(), 6, "smm"))
    rows = 20
    det = store.model("w")
    smoothed = []
    monkeypatch.setattr(DiffBasedAnomalyDetector, "_score", lambda self, *a, **k: _scores(rows))
    monkeypatch.setattr(DiffBasedAnomalyDetector, "_smoothing", lambda self, m: smoothed.append(m.shape) or np.asarray(m, dtype=np.float32) + 1)
    calls = []

    class FakeCoalescer:
        def anomaly(self, slot, X, y, smooth=False):
            calls.append(smooth)
            res = _scores(rows)
            if smooth:
                res.update({"smooth-" + k: np.asarray(res[k], dtype=np.float32) + 1 for k in
                            ("tag-anomaly-scaled", "total-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-unscaled")})
            return res

    bucket = server.ResidentBucket.__new__(server.ResidentBucket)
    bucket.names, bucket.slot, bucket.coalescer, bucket.smoothing = ["w"], {"w": 0}, FakeCoalescer(), (6, "smm")

    def ask(y_nan, all_columns, through):
        X = _frame(rows)
        payload = {"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(_frame(rows, y_nan))}
        return server.anomaly_prediction(store, "w", json=payload, all_columns=all_columns, bucket=bucket if through else None)

    # the default reply: nothing is smoothed on either route
    for y_nan in (False, True):
        assert json.dumps(ask(y_nan, False, True).body["data"]) == json.dumps(ask(y_nan, False, False).body["data"])
    assert calls == [False, False] and smoothed == []
    # the reply with every column: the coalescer smooths (no host smoothing); a NaN target goes on its own route
    got, want = ask(False, True, True), ask(False, True, False)
    assert calls == [False, False, True] and len(smoothed) == 4
    assert json.dumps(got.body["data"]) == json.dumps(want.body["data"]) and "smooth-total-anomaly-scaled" in got.body["data"]
    smoothed.clear()
    got = ask(True, True, True)
    assert calls == [False, False, True] and smoothed == [(rows, T), (rows,), (rows, T), (rows,)]
    assert "smooth-tag-anomaly-unscaled" in got.body["data"]
    # the detector itself: smooth=False leaves the blocks out, smooth-* arrays already given are used as they are
    smoothed.clear()
    X = _frame(rows)
    _, _, cols = det.anomaly_blocks(X, X, smooth=False)
    assert not any(top.startswith("smooth-") for top, _ in cols) and smoothed == []
    _, _, cols = det.blocks_from_scores(FakeCoalescer().anomaly(0, X, X, smooth=True), X, X)
    assert [top for top, _ in cols if top.startswith("smooth-")] and smoothed == []
