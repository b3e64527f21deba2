"""
TransformedTargetRegressor LSTM detectors on the serving side, without a GPU: which of them ``ResidentBucket(lstm=True,
target_scaler=True)`` admits, how it groups them, and that the LSTM bucket without ``target_scaler`` still refuses them.
"""
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


def _lstm(cls="KerasLSTMAutoEncoder", lookback=3, n=T, **kw):
    from gordo_components_b200.machine.model import models

    return getattr(models, cls)(kind="lstm_hourglass", lookback_window=lookback, encoding_layers=1, **kw).initialize(n, n)


def _ttr(reg, transformer=None, fitted=True, **kw):
    """A TransformedTargetRegressor around ``reg`` in the state its fit leaves (what the fleet builder assembles)."""
    from sklearn.base import clone
    from sklearn.compose import TransformedTargetRegressor
    from sklearn.preprocessing import MinMaxScaler

    ttr = TransformedTargetRegressor(regressor=reg, transformer=transformer if transformer is not None else MinMaxScaler(), **kw)
    if fitted:
        ttr._training_dim = 2
        ttr.transformer_ = clone(ttr.transformer).fit(np.random.default_rng(1).random((8, T)) * 50)
        ttr.regressor_ = reg
    return ttr


def _piped(est, *steps):
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import MinMaxScaler

    steps = steps or (MinMaxScaler(),)
    rng = np.random.default_rng(2)
    for s in steps:
        s.fit(rng.random((8, T)) * 100)
    return Pipeline([(f"s{i}", s) for i, s in enumerate(steps)] + [("m", est)])


def _det(est, window=None, method=None, scaler=None, thresholds=True):
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector

    det = DiffBasedAnomalyDetector(base_estimator=est, scaler=scaler if scaler is not None else MinMaxScaler(), window=window,
                                   smoothing_method=method, require_thresholds=thresholds)
    det.scaler.fit(np.random.default_rng(0).random((8, T)))
    if thresholds:
        det.feature_thresholds_, det.aggregate_threshold_ = pd.Series(np.ones(T), index=TAGS), 0.5
    return det


def test_admitted_forms(lib):
    from sklearn.preprocessing import MaxAbsScaler, MinMaxScaler, RobustScaler, StandardScaler

    admitted = {
        "autoencoder": _det(_ttr(_lstm())),
        "forecast": _det(_ttr(_lstm("KerasLSTMForecast"))),
        "MinMaxScaler input": _det(_ttr(_piped(_lstm()))),
        # unlike the feed-forward TTR bucket, any leading steps: they run on the host as Pipeline.predict runs them
        "StandardScaler input": _det(_ttr(_piped(_lstm("KerasLSTMForecast"), StandardScaler()))),
        "RobustScaler input": _det(_ttr(_piped(_lstm(), RobustScaler()))),
        "MaxAbsScaler input": _det(_ttr(_piped(_lstm(), MaxAbsScaler()))),
        "two input scalers": _det(_ttr(_piped(_lstm(), MinMaxScaler(), StandardScaler()))),
        "no thresholds": _det(_ttr(_lstm()), thresholds=False),
        # inverse_transform is (X - min_) / scale_ whatever the range, and so is the launch's inverse; the feed-forward TTR
        # bucket admits it too
        "feature_range (-1, 1)": _det(_ttr(_lstm(), MinMaxScaler(feature_range=(-1, 1)))),
    }
    for why, det in admitted.items():
        assert server.ResidentBucket.eligible_lstm(det, target_scaler=True), why
        assert server.ResidentBucket.eligible_lstm(det, smoothing=True, target_scaler=True), why
        assert not server.ResidentBucket.eligible_lstm(det), why  # the LSTM bucket refuses a TTR without the flag, as before
        assert not server.ResidentBucket.eligible_lstm(det, smoothing=True), why
        assert not server.ResidentBucket.eligible(det, input_scalers=True, smoothing=True, target_scaler=True), why  # never feed-forward
    for method in ("smm", "sma", "ewma"):
        windowed = _det(_ttr(_piped(_lstm())), window=12, method=method)
        assert server.ResidentBucket.eligible_lstm(windowed, smoothing=True, target_scaler=True), method
        assert not server.ResidentBucket.eligible_lstm(windowed, target_scaler=True), method  # a window needs smoothing=True, as before
    # plain LSTM detectors are admitted with the flag as without it
    for det in (_det(_lstm()), _det(_piped(_lstm("KerasLSTMForecast")))):
        assert server.ResidentBucket.eligible_lstm(det, target_scaler=True) and server.ResidentBucket.eligible_lstm(det)


def test_refused_forms(lib):
    from sklearn.preprocessing import MinMaxScaler, QuantileTransformer, StandardScaler

    from gordo_components_b200.machine.model.models import KerasLSTMAutoEncoder

    refused = {
        "StandardScaler transformer": _det(_ttr(_lstm(), StandardScaler())),
        "func": _det(_ttr(_lstm(), transformer=None, func=np.log1p, inverse_func=np.expm1)),
        "relu cells": _det(_ttr(_lstm(func="relu"))),
        "linear cells": _det(_ttr(_lstm(func="linear"))),
        "not fitted": _det(_ttr(_lstm(), fitted=False)),
        "LSTM without weights": _det(_ttr(KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=3))),
        "non-affine error scaler": _det(_ttr(_lstm()), scaler=QuantileTransformer(n_quantiles=5)),
        "thresholds required but missing": _det(_ttr(_lstm()), thresholds=False),
    }
    refused["thresholds required but missing"].require_thresholds = True
    for why, det in refused.items():
        assert not server.ResidentBucket.eligible_lstm(det, smoothing=True, target_scaler=True), why
    # a TTR fitted on a 1-D target predicts 1-D: its reply shape is the per-request route's business
    one_d = _ttr(_lstm())
    one_d._training_dim = 1
    assert not server.ResidentBucket.eligible_lstm(_det(one_d), smoothing=True, target_scaler=True)
    # a transformer fitted on another number of targets than the network predicts
    wide = _ttr(_lstm())
    wide.transformer_ = MinMaxScaler().fit(np.random.default_rng(0).random((8, T + 1)))
    assert not server.ResidentBucket.eligible_lstm(_det(wide), smoothing=True, target_scaler=True)


def test_ttr_and_plain_lstm_models_get_groups_of_their_own(lib):
    from sklearn.preprocessing import StandardScaler

    models = {
        "ae": _det(_lstm()),
        "fc": _det(_lstm("KerasLSTMForecast")),
        "ttr-ae": _det(_ttr(_lstm())),
        "ttr-fc": _det(_ttr(_lstm("KerasLSTMForecast"))),         # autoencoder and forecast TTRs share a group
        "ttr-piped": _det(_ttr(_piped(_lstm()))),                  # so does a TTR around a Pipeline of the same stack
        "ttr-std": _det(_ttr(_piped(_lstm("KerasLSTMForecast"), StandardScaler()))),
        "ttr-lb5": _det(_ttr(_lstm(lookback=5))),                  # another lookback: another architecture
        "ttr-window": _det(_ttr(_lstm()), window=12, method="smm"),
        "ttr-relu": _det(_ttr(_lstm(func="relu"))),                # not eligible at all
    }
    groups = server.ResidentBucket.lstm_groups(models, smoothing=True, target_scaler=True)
    assert sorted(map(sorted, groups.values())) == [["ae", "fc"], ["ttr-ae", "ttr-fc", "ttr-piped", "ttr-std"], ["ttr-lb5"], ["ttr-window"]]
    by_name = {n: k for k, names in groups.items() for n in names}
    assert by_name["ttr-ae"][2] is True and by_name["ae"][2] is False  # the flag; everything else of the key is the same
    assert by_name["ttr-ae"][:2] == by_name["ae"][:2] and by_name["ttr-ae"][3:] == by_name["ae"][3:]
    assert by_name["ttr-window"][-1] == (12, "smm")
    assert max(groups.values(), key=len) == ["ttr-ae", "ttr-fc", "ttr-piped", "ttr-std"]
    # without the flag the groups are what they were
    assert sorted(map(sorted, server.ResidentBucket.lstm_groups(models, smoothing=True).values())) == [["ae", "fc"]]
    assert sorted(map(sorted, server.ResidentBucket.lstm_groups(models).values())) == [["ae", "fc"]]
    assert server.ResidentBucket.ff_groups(models, input_scalers=True, smoothing=True, target_scaler=True) == {}


def test_bucket_passes_the_targets_transformers_to_the_coalescer(lib, monkeypatch, tmp_path):
    """``ResidentBucket(lstm=True, target_scaler=True)`` hands the LSTM coalescer each slot's float64 ``scale_`` / ``min_``; the
    bucket without the flag holds the plain models and passes none."""
    import torch

    from gordo_components_b200 import engine, serializer, serving

    made = []

    class Recorder:
        def __init__(self, eng, params, scale, feat_thr=None, agg_thr=None, **kwargs):
            self.params, self.kwargs = params, kwargs
            made.append(self)

        def close(self):
            pass

    class Eng:
        device = "cpu"

        def __init__(self, spec):
            self.n_out = spec.n_features_out

        def pack_params(self, weights):
            return torch.zeros((len(weights), 1))

    monkeypatch.setattr(serving, "LSTMAnomalyCoalescer", Recorder)
    monkeypatch.setattr(engine, "lstm_engine_for", Eng)
    models = {"ae": _det(_lstm()), "ae-b": _det(_lstm("KerasLSTMForecast")), "ttr-0": _det(_ttr(_piped(_lstm()))),
              "ttr-1": _det(_ttr(_lstm("KerasLSTMForecast"))), "ttr-2": _det(_ttr(_lstm()))}
    models["ttr-1"].base_estimator.transformer_.fit(np.random.default_rng(5).random((8, T)) * 7)
    for name, det in models.items():
        serializer.dump(det, str(tmp_path / name), metadata={"dataset": {"tag_list": TAGS}})
    store = server.ModelStore(str(tmp_path))
    b = server.ResidentBucket(store, lstm=True, target_scaler=True, max_wait_ms=5.0)
    assert b.lstm and b.target_scaler and b.names == ["ttr-0", "ttr-1", "ttr-2"]
    y_scale, y_min = made[-1].kwargs["y_inverse"]
    assert made[-1].kwargs["max_wait_ms"] == 5.0 and y_scale.dtype == y_min.dtype == torch.float64
    for i, name in enumerate(b.names):
        tr = store.model(name).base_estimator.transformer_
        np.testing.assert_array_equal(y_scale[i].numpy(), tr.scale_)
        np.testing.assert_array_equal(y_min[i].numpy(), tr.min_)
    plain = server.ResidentBucket(store, lstm=True)
    assert plain.names == ["ae", "ae-b"] and not plain.target_scaler and "y_inverse" not in made[-1].kwargs
    with pytest.raises(ValueError, match="no LSTM model"):
        server.ResidentBucket(store, names=["ttr-0", "ttr-1"], lstm=True)
