"""
Host-side mirror of the reference model API (no GPU needed): factories, registry, estimator protocol, frame assembly.
Modelled on the reference's tests: tests/gordo/machine/model/{test_factories_utils,test_feedforward_autoencoder,
test_lstm_autoencoder,test_register,test_model,test_utils}.py and anomaly/test_anomaly_detectors.py.
"""
import os
import pickle

import numpy as np
import pandas as pd
import pytest
from sklearn.base import clone
from sklearn.preprocessing import MinMaxScaler

from gordo_components_b200.machine.model import utils as model_utils
from gordo_components_b200.machine.model.anomaly.base import AnomalyDetectorBase
from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector, _scaler_multiplier
from gordo_components_b200.machine.model.base import GordoBase
from gordo_components_b200.machine.model.factories import feedforward_autoencoder as ffa
from gordo_components_b200.machine.model.factories import lstm_autoencoder as lsa
from gordo_components_b200.machine.model.factories.utils import check_dim_func_len, hourglass_calc_dims
from gordo_components_b200.machine.model.models import (
    KerasAutoEncoder,
    KerasLSTMAutoEncoder,
    KerasLSTMForecast,
    create_keras_timeseriesgenerator,
)
from gordo_components_b200.machine.model.register import register_model_builder
from oracle import anomaly_math as am

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


# ---------------------------------------------------------------- factories (test_factories_utils.py:8-35)
@pytest.mark.parametrize(
    "test_input,test_expected",
    [((0.2, 4, 5), (4, 3, 2, 1)), ((0.5, 3, 10), (8, 7, 5)), ((0.5, 3, 3), (3, 2, 2)), ((0.3, 3, 10), (8, 5, 3)),
     ((1, 3, 10), (10, 10, 10)), ((0, 3, 100000), (66667, 33334, 1))],
)
def test_hourglass_calc_dims_check_dims(test_input, test_expected):
    assert hourglass_calc_dims(*test_input) == test_expected


def test_check_dim_func_len():
    with pytest.raises(ValueError):
        check_dim_func_len("test", dim=(256, 128), func=("tanh", "tanh", "tanh"))
    with pytest.raises(ValueError):
        check_dim_func_len("test", dim=(256, 128, 56), func=("tanh", "tanh"))


def test_hourglass_topologies():
    # test_feedforward_autoencoder.py:76-180 (dims reaching feedforward_model) + doctests
    assert ffa.feedforward_hourglass(10).units == [8, 7, 5, 5, 7, 8, 10]
    assert ffa.feedforward_hourglass(3).units == [3, 2, 2, 2, 2, 3, 3]
    assert ffa.feedforward_hourglass(10, compression_factor=0.3).units == [8, 5, 3, 3, 5, 8, 10]
    assert ffa.feedforward_hourglass(100, encoding_layers=2, compression_factor=0.0).dims[1:3] == [50, 1]
    s = ffa.feedforward_hourglass(64)
    assert s.dims == [64, 53, 43, 32, 32, 43, 53, 64] and s.n_params == 15438
    assert s.l1 == [0.0, 10e-5, 10e-5, 0, 0, 0, 0] and s.acts == ["tanh"] * 6 + ["linear"]
    assert ffa.feedforward_hourglass(64, n_features_out=3).dims[-1] == 3
    ls = lsa.lstm_hourglass(10, lookback_window=5)
    assert ls.units == [8, 7, 5, 5, 7, 8, 10] and ls.lookback_window == 5
    assert lsa.lstm_symmetric(128, lookback_window=144).n_params == 1199744


def test_factory_errors():
    # test_feedforward_autoencoder.py:182-196, lstm equivalents
    for bad in (dict(compression_factor=1.5), dict(compression_factor=-0.1), dict(encoding_layers=0)):
        with pytest.raises(ValueError):
            ffa.feedforward_hourglass(10, **bad)
        with pytest.raises(ValueError):
            lsa.lstm_hourglass(10, **bad)
    with pytest.raises(ValueError):
        ffa.feedforward_symmetric(5, dims=[])
    with pytest.raises(ValueError):
        lsa.lstm_symmetric(5, dims=[])
    with pytest.raises(ValueError):
        ffa.feedforward_model(5, encoding_dim=(4, 3), encoding_func=("tanh",))
    with pytest.raises(ValueError):
        ffa.feedforward_hourglass(5, optimizer="SGD")  # only what the fit kernel implements is accepted
    with pytest.raises(ValueError):
        ffa.feedforward_hourglass(5, func="swish")


def test_register():
    # test_register.py
    @register_model_builder(type="KerasAutoEncoder")
    def special_keras_model_builder(n_features, **kw):
        return ffa.feedforward_hourglass(n_features)

    assert "special_keras_model_builder" in register_model_builder.factories["KerasAutoEncoder"]
    with pytest.raises(ValueError):

        @register_model_builder(type="KerasAutoEncoder")
        def no_features_arg(n_inputs):
            return None

    for t in ("KerasAutoEncoder", "KerasLSTMAutoEncoder", "KerasLSTMForecast"):
        assert t in register_model_builder.factories
    assert {"lstm_model", "lstm_symmetric", "lstm_hourglass"} <= set(register_model_builder.factories["KerasLSTMForecast"])


# ---------------------------------------------------------------- estimator protocol (test_model.py)
def test_estimator_protocol():
    m = KerasAutoEncoder(kind="feedforward_hourglass", epochs=3, batch_size=16)
    assert isinstance(m, GordoBase)
    assert m.get_params() == {"kind": "feedforward_hourglass", "epochs": 3, "batch_size": 16}
    assert m.into_definition() == {"kind": "feedforward_hourglass", "epochs": 3, "batch_size": 16}
    m2 = KerasAutoEncoder.from_definition({"kind": "feedforward_symmetric", "dims": [4, 2], "funcs": ["tanh", "tanh"]})
    assert m2.kind == "feedforward_symmetric" and m2.kwargs["dims"] == [4, 2]
    c = clone(m)
    assert c is not m and c.get_params() == m.get_params()
    assert m.get_metadata() == {}
    p = pickle.loads(pickle.dumps(m))
    assert p.get_params() == m.get_params()
    from sklearn.exceptions import NotFittedError

    with pytest.raises(NotFittedError):
        m.score(np.zeros((2, 2)), np.zeros((2, 2)))
    with pytest.raises(ValueError):
        KerasAutoEncoder(kind="not_a_factory")
    with pytest.raises(ValueError):
        KerasAutoEncoder(kind="no.such.module.factory")
    with pytest.raises(ValueError):
        KerasAutoEncoder.get_n_features(np.zeros(4))

    def my_builder(n_features, **kw):
        return ffa.feedforward_hourglass(n_features)

    assert KerasAutoEncoder(kind=my_builder).kind == "my_builder"
    dotted = KerasAutoEncoder(kind="gordo_components_b200.machine.model.factories.feedforward_autoencoder.feedforward_hourglass")
    assert dotted._factory() is ffa.feedforward_hourglass


def test_lstm_estimator_protocol():
    m = KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=4, batch_size=8)
    assert m.lookahead == 0 and KerasLSTMForecast(kind="lstm_model").lookahead == 1
    assert m.get_params()["lookback_window"] == 4 and m.get_params()["batch_size"] == 8
    assert m.get_metadata() == {"forecast_steps": 0}
    assert clone(m).get_params() == m.get_params()
    # test_model.py:161-236: lookback_window >= len(X) is a ValueError
    for lb in (5, 6):
        with pytest.raises(ValueError):
            KerasLSTMForecast(kind="lstm_model", lookback_window=lb)._validate_and_fix_size_of_X(np.random.random((5, 2)))


# ---------------------------------------------------------------- windowing goldens (test_model.py:239-321)
def test_timeseries_windows_golden():
    X = np.array([[0, 1], [2, 3], [4, 5], [6, 7], [8, 9]])
    g = create_keras_timeseriesgenerator(X, X.copy(), batch_size=2, lookback_window=3, lookahead=0)
    assert g[0][0].tolist() == [[[0, 1], [2, 3], [4, 5]], [[2, 3], [4, 5], [6, 7]]] and g[0][1].tolist() == [[4, 5], [6, 7]]
    assert g[1][0].tolist() == [[[4, 5], [6, 7], [8, 9]]] and g[1][1].tolist() == [[8, 9]]
    g = create_keras_timeseriesgenerator(X, X.copy(), batch_size=2, lookback_window=2, lookahead=1)
    assert g[0][0].tolist() == [[[0, 1], [2, 3]], [[2, 3], [4, 5]]] and g[0][1].tolist() == [[4, 5], [6, 7]]
    assert g[1][0].tolist() == [[[4, 5], [6, 7]]] and g[1][1].tolist() == [[8, 9]]
    g = create_keras_timeseriesgenerator(X, X.copy(), batch_size=2, lookback_window=2, lookahead=2)
    assert g[0][1].tolist() == [[6, 7], [8, 9]] and g[1][0].tolist() == []
    with pytest.raises(ValueError):
        create_keras_timeseriesgenerator(X, X, batch_size=2, lookback_window=2, lookahead=-1)


# ---------------------------------------------------------------- frames (test_utils.py)
def test_metric_wrapper():
    from sklearn.metrics import mean_squared_error

    y_true = np.arange(20.0).reshape(10, 2)
    y_pred = y_true[2:] + 1.0
    assert model_utils.metric_wrapper(mean_squared_error)(y_true, y_pred) == pytest.approx(1.0)
    sc = MinMaxScaler().fit(y_true)
    assert model_utils.metric_wrapper(mean_squared_error, scaler=sc)(y_true, y_pred) < 1.0


@pytest.mark.parametrize("datetime_index", [True, False])
@pytest.mark.parametrize("offset", [0, 3])
def test_make_base_dataframe_matches_oracle(datetime_index, offset):
    n = 12
    idx = pd.date_range("2019-01-01", periods=n, freq="10min", tz="UTC") if datetime_index else pd.RangeIndex(n)
    X = np.random.default_rng(0).random((n, 3))
    out = np.random.default_rng(1).random((n - offset, 3)).astype(np.float32)
    freq = pd.Timedelta("10min") if datetime_index else None
    got = model_utils.make_base_dataframe(["a", "b", "c"], X, out, index=idx, frequency=freq)
    want = am.base_frame(["a", "b", "c"], X, out, index=idx, frequency=freq)
    assert list(got.columns) == list(want.columns) and len(got) == n - offset
    assert got.index.equals(want.index)
    np.testing.assert_array_equal(got["model-input"].values, X[offset:])
    np.testing.assert_array_equal(got["model-output"].values.astype(np.float32), out)
    assert got[("start", "")].tolist() == want[("start", "")].tolist()
    assert got[("end", "")].tolist() == want[("end", "")].tolist()
    # width mismatch -> numbered second level (model/utils.py:145-151)
    odd = model_utils.make_base_dataframe(["a", "b", "c"], X, np.zeros((n, 2)), index=idx)
    assert list(odd["model-output"].columns) == ["0", "1"]


def test_make_base_dataframe_matches_reference_fixture():
    g = np.load(os.path.join(GOLDEN, "ffnet_anomaly.npz"))
    n, t = g["X"].shape
    idx = pd.date_range("2019-01-01", periods=n, freq="10min", tz="UTC")
    tags = [f"tag-{i}" for i in range(t)]
    f = model_utils.make_base_dataframe(tags, g["X"], g["pred"], target_tag_list=tags, index=idx, frequency=pd.Timedelta("10min"))
    assert ["|".join(c) for c in f.columns] == [str(c) for c in g["columns"]][: len(f.columns)]
    assert f[("start", "")].tolist() == [str(s) for s in g["frame_start"]]
    assert f[("end", "")].tolist() == [str(s) for s in g["frame_end"]]


# ---------------------------------------------------------------- detector bookkeeping (test_anomaly_detectors.py:55-57,166-187,675-732)
def test_detector_protocol():
    base = KerasAutoEncoder(kind="feedforward_hourglass")
    sc = MinMaxScaler()
    d = DiffBasedAnomalyDetector(base_estimator=base, scaler=sc, shuffle=True)
    assert isinstance(d, AnomalyDetectorBase) and isinstance(d, GordoBase)
    assert d.get_params() == dict(base_estimator=base, scaler=sc, shuffle=True)
    dw = DiffBasedAnomalyDetector(base_estimator=base, scaler=sc, window=144)
    assert dw.get_params() == dict(base_estimator=base, scaler=sc, shuffle=False, window=144, smoothing_method="smm")
    assert d.kind == "feedforward_hourglass"  # transparent attribute access
    assert callable(d.predict)
    with pytest.raises(AttributeError):
        d.no_such_attribute
    md = dw.get_metadata()
    assert md["window"] == 144 and md["smoothing-method"] == "smm" and "feature-thresholds" not in md
    c = clone(d)
    assert c.base_estimator is not base and c.base_estimator.get_params() == base.get_params()
    pickle.loads(pickle.dumps(d))
    with pytest.raises(ValueError):  # diff.py:332-333
        DiffBasedAnomalyDetector(base_estimator=base, require_thresholds=False).anomaly(np.zeros((3, 3)), np.zeros((3, 3)))
    frame = pd.DataFrame(np.zeros((3, 3)))
    with pytest.raises(AttributeError):  # diff.py:448-456
        DiffBasedAnomalyDetector(base_estimator=base, require_thresholds=True).anomaly(frame, frame)


def test_kfcv_detector_protocol():
    """test_anomaly_detectors.py:403-424, 675-732: constructor defaults, get_params, metadata keys, clone / pickle."""
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedKFCVAnomalyDetector

    base = KerasAutoEncoder(kind="feedforward_hourglass")
    sc = MinMaxScaler()
    d = DiffBasedKFCVAnomalyDetector(base_estimator=base, scaler=sc)
    assert isinstance(d, DiffBasedAnomalyDetector) and isinstance(d, AnomalyDetectorBase)
    assert d.get_params() == dict(base_estimator=base, scaler=sc, window=144, smoothing_method="smm", shuffle=True, threshold_percentile=0.99)
    assert "feature-thresholds" not in d.get_metadata()
    c = clone(d)
    assert c.threshold_percentile == 0.99 and c.base_estimator is not base
    pickle.loads(pickle.dumps(d))
    frame = pd.DataFrame(np.zeros((3, 3)))
    with pytest.raises(AttributeError):
        d.anomaly(frame, frame)


def test_early_stopping_state_machine():
    """keras 3.3.3 EarlyStopping semantics [3P] (the callback of gordo's model definitions, test_model.py:341-361,
    test_anomaly_detectors.py:531-534), restated for the per-epoch launch loop."""
    from gordo_components_b200.machine.model.models import EarlyStopping, build_callbacks

    (cb,) = build_callbacks([{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "val_loss", "patience": 2, "restore_best_weights": True}}])
    assert cb.monitor == "val_loss" and cb.patience == 2 and cb.mode == "min"
    w = [None]
    stops = []
    for e, v in enumerate([1.0, 0.8, 0.9, 0.85, 0.95]):
        w[0] = e
        stops.append(cb.update(e, {"val_loss": v}, lambda: w[0]))
        if stops[-1]:
            break
    assert stops == [False, False, False, True] and cb.best == 0.8 and cb.best_weights == 1 and cb.stopped_epoch == 3
    # min_delta: an improvement smaller than it does not count; patience 0 stops at the first non-improving epoch after epoch 0
    cb = EarlyStopping(monitor="loss", min_delta=0.1, patience=0)
    assert [cb.update(e, {"loss": v}, lambda: None) for e, v in enumerate([1.0, 0.95])] == [False, True]
    # baseline: wait only restarts when the baseline is beaten too, and the stop test runs on non-improving epochs only
    cb = EarlyStopping(monitor="loss", patience=2, baseline=0.5)
    assert [cb.update(e, {"loss": v}, lambda: None) for e, v in enumerate([1.0, 0.9, 0.8, 0.85])] == [False, False, False, True]
    # a missing metric never stops training; accuracy-like monitors are maximised
    assert EarlyStopping(monitor="val_loss").update(0, {"loss": 1.0}, lambda: None) is False
    assert EarlyStopping(monitor="val_accuracy").mode == "max"
    assert build_callbacks([{"tensorflow.keras.callbacks.TerminateOnNaN": {}}]) == []
    m = KerasAutoEncoder(kind="feedforward_hourglass", batch_size=128, callbacks=[{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "val_loss", "patience": 10}}])
    assert len(m.sk_params["callbacks"]) == 1 and clone(m).get_params() == m.get_params()


def test_scaler_multiplier():
    from sklearn.preprocessing import QuantileTransformer, RobustScaler

    y = np.random.default_rng(0).random((50, 3)) * [1, 5, 10]
    np.testing.assert_allclose(_scaler_multiplier(MinMaxScaler().fit(y), 3), MinMaxScaler().fit(y).scale_, rtol=1e-6)
    np.testing.assert_allclose(_scaler_multiplier(RobustScaler().fit(y), 3), 1 / RobustScaler().fit(y).scale_, rtol=1e-6)
    with pytest.raises(ValueError):
        _scaler_multiplier(QuantileTransformer(n_quantiles=10).fit(y), 3)
    # the slope of a fitted scaler is probed once per fitted state: a refit (new scale_ / min_ arrays) is seen, a repeat request is not re-probed
    sc = MinMaxScaler().fit(y)
    first = _scaler_multiplier(sc, 3)
    calls = []
    real_transform = sc.transform
    sc.transform = lambda X: (calls.append(1), real_transform(X))[1]
    assert _scaler_multiplier(sc, 3) is first and not calls
    sc.fit(y * 2.0)
    np.testing.assert_allclose(_scaler_multiplier(sc, 3), first / 2.0, rtol=1e-12)
    assert len(calls) == 1


# ---------------------------------------------------------------- frame assembly fast paths
def test_isoformat_equals_timestamp_isoformat():
    """The arithmetic ISO formatter against pandas' own ``Timestamp.isoformat`` over the whole 0001..9999 range and the edges."""
    rng = np.random.default_rng(0)
    secs = np.concatenate([rng.integers(-62135596800, 253402300799, 5000),
                           np.array([0, -1, 86399, 86400, -86400, 951782400, 951868800, 4107542400, 1582934400, -62135596800, 253402300799])])
    for tz in (None, "UTC"):
        idx = pd.DatetimeIndex(secs.astype("datetime64[s]"), tz=tz)
        got = model_utils._isoformat(idx)
        assert got.dtype == object and type(got[0]) is str
        assert list(got) == [ts.isoformat() for ts in idx]
    # anything the fast path does not cover falls back to the per-timestamp loop
    for idx in (pd.date_range("2019-01-01", periods=3, freq="1500ms", tz="UTC"), pd.date_range("2019-03-30", periods=3, freq="12h", tz="Europe/Oslo"),
                pd.date_range("2019-01-01", periods=0, freq="1h")):
        assert list(model_utils._isoformat(idx)) == [ts.isoformat() for ts in idx]
    assert model_utils._iso_seconds(np.array([253402300800]), True) is None  # year 10000


@pytest.mark.parametrize("rows,offset,thresholds,window,index_kind", [(1, 0, True, None, "utc"), (40, 3, True, 5, "utc"), (25, 0, False, None, "range"),
                                                                      (30, 2, False, 4, "naive"), (12, 0, True, None, "sub-second")])
def test_anomaly_frame_assembly_with_a_mocked_score(rows, offset, thresholds, window, index_kind):
    """
    ``anomaly()`` builds its frame in one pass (cached column index, one concat); here the GPU score is replaced by fixed arrays and
    the result is compared with the frame spelled out the slow way: base frame + one block per column group, concatenated.
    """
    T = 3
    tags = [f"tag {i}" for i in range(T)]
    idx = {"utc": pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC"), "naive": pd.date_range("2019-01-01", periods=rows, freq="10min"),
           "sub-second": pd.date_range("2019-01-01", periods=rows, freq="1500ms", tz="UTC"), "range": pd.RangeIndex(rows)}[index_kind]
    rng = np.random.default_rng(rows)
    X = pd.DataFrame(rng.random((rows, T)), index=idx, columns=tags)
    det = DiffBasedAnomalyDetector(base_estimator=KerasAutoEncoder(kind="feedforward_hourglass"), require_thresholds=thresholds, window=window,
                                   smoothing_method="sma" if window else None)
    if thresholds:
        det.feature_thresholds_, det.aggregate_threshold_ = pd.Series(np.ones(T), index=tags), 0.5
    n = rows - offset
    res = {"model-output": rng.random((n, T)).astype(np.float32), "tag-anomaly-scaled": rng.random((n, T)).astype(np.float32),
           "total-anomaly-scaled": rng.random(n).astype(np.float32), "tag-anomaly-unscaled": rng.random((n, T)).astype(np.float32),
           "total-anomaly-unscaled": rng.random(n).astype(np.float32)}
    if thresholds:
        res.update({"anomaly-confidence": rng.random((n, T)).astype(np.float32), "total-anomaly-confidence": rng.random(n).astype(np.float32)})
    det._score = lambda *a, **k: dict(res)
    det._smoothing = lambda metric: np.asarray(metric, dtype=np.float32) * 0.5
    freq = pd.Timedelta("10min")
    got = det.anomaly(X, X, frequency=freq)

    order = ["tag-anomaly-scaled", "total-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-unscaled"]
    groups = list(order) + (["smooth-" + k for k in order] if window else []) + (["anomaly-confidence", "total-anomaly-confidence"] if thresholds else [])
    pieces = [model_utils.make_base_dataframe(tags=tags, model_input=X.values, model_output=res["model-output"], target_tag_list=tags, index=idx, frequency=freq)]
    for key in groups:
        v = np.asarray(res[key[len("smooth-"):]] * 0.5 if key.startswith("smooth-") else res[key], dtype=np.float64)
        cols = [(key, t) for t in tags] if v.ndim == 2 else [(key, "")]
        pieces.append(pd.DataFrame(v.reshape(n, -1), index=pieces[0].index, columns=pd.MultiIndex.from_tuples(cols)))
    want = pd.concat(pieces, axis=1)
    assert list(got.columns) == list(want.columns) and list(got.dtypes) == list(want.dtypes) and len(got) == n
    pd.testing.assert_frame_equal(got, want, check_exact=True, check_freq=False)
    assert got.columns is not det.anomaly(X, X, frequency=freq).columns  # the cached column index is handed out as copies


@pytest.mark.parametrize("window", [None, 4])
def test_anomaly_frame_totals_skip_missing_target_tags(window):
    """
    Rows with NaN target tags, as requests with missing sensor values give them: the kernels' totals (numpy mean over every tag) are
    NaN there, and the frame replaces them with pandas' mean over the tags that have a value (diff.py:366, :383) -- NaN only when no
    tag has one -- and recomputes the total confidence from it.  Smoothing sees the corrected totals; every other row is untouched.
    """
    T, n = 4, 30
    tags = [f"tag {i}" for i in range(T)]
    rng = np.random.default_rng(7)
    X = pd.DataFrame(rng.random((n, T)), index=pd.date_range("2019-01-01", periods=n, freq="10min", tz="UTC"), columns=tags)
    det = DiffBasedAnomalyDetector(base_estimator=KerasAutoEncoder(kind="feedforward_hourglass"), window=window,
                                   smoothing_method="sma" if window else None)
    agg = 0.3
    det.feature_thresholds_, det.aggregate_threshold_ = pd.Series(np.full(T, 0.5), index=tags), agg
    tag_s, tag_u = rng.random((n, T)).astype(np.float32), rng.random((n, T)).astype(np.float32)
    for a in (tag_s, tag_u):
        a[3, 1] = a[10, [0, 2]] = a[11] = np.nan  # one tag, two tags, every tag
        a[20:27, 3] = np.nan                      # a run longer than the window
    tot_s, tot_u = np.square(tag_s).mean(axis=1), np.square(tag_u).mean(axis=1)
    res = {"model-output": rng.random((n, T)).astype(np.float32), "tag-anomaly-scaled": tag_s, "total-anomaly-scaled": tot_s,
           "tag-anomaly-unscaled": tag_u, "total-anomaly-unscaled": tot_u, "anomaly-confidence": tag_u / np.float32(0.5),
           "total-anomaly-confidence": tot_s / np.float32(agg)}
    det._score = lambda *a, **k: dict(res)
    smoothed = []
    det._smoothing = lambda metric: (smoothed.append(np.array(metric)), np.asarray(metric, dtype=np.float32) * 0.5)[1]
    got = det.anomaly(X, X)

    missing = np.isnan(tot_s)
    assert missing.sum() == 10
    with np.errstate(all="ignore"), __import__("warnings").catch_warnings():
        __import__("warnings").simplefilter("ignore", RuntimeWarning)
        want_s = pd.DataFrame(np.square(tag_s.astype(np.float64))).mean(axis=1).values
        want_u = pd.DataFrame(np.square(tag_u.astype(np.float64))).mean(axis=1).values
    for key, want, kernel in (("total-anomaly-scaled", want_s, tot_s), ("total-anomaly-unscaled", want_u, tot_u),
                              ("total-anomaly-confidence", want_s / agg, tot_s / np.float32(agg))):
        col = got[(key, "")].values
        np.testing.assert_array_equal(col[~missing], kernel[~missing].astype(np.float64), err_msg=key)  # bit for bit
        np.testing.assert_allclose(col[missing], want[missing], rtol=1e-12, err_msg=key)
        assert np.isnan(col).tolist() == [i == 11 for i in range(n)], key  # NaN only where no tag has a value
    np.testing.assert_array_equal(got["tag-anomaly-scaled"].values, tag_s.astype(np.float64))
    if window:
        # the smoothed totals are the smoothing of the corrected totals
        assert len(smoothed) == 4
        np.testing.assert_array_equal(smoothed[1], got[("total-anomaly-scaled", "")].values)
        np.testing.assert_array_equal(smoothed[3], got[("total-anomaly-unscaled", "")].values)
        corrected = np.where(missing, want_s, tot_s).astype(np.float32)
        np.testing.assert_array_equal(got[("smooth-total-anomaly-scaled", "")].values, (corrected * 0.5).astype(np.float64))
    # without a NaN row the totals pass through as the kernels computed them
    clean = {k: np.nan_to_num(v, nan=0.25) for k, v in res.items()}
    det._score = lambda *a, **k: dict(clean)
    frame = det.anomaly(X, X)
    np.testing.assert_array_equal(frame[("total-anomaly-scaled", "")].values, clean["total-anomaly-scaled"].astype(np.float64))
