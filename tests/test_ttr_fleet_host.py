"""
Which TransformedTargetRegressor detectors FleetModelBuilder(target_scaler=True) batches under a TimeSeriesSplit cv, how it buckets
them, and that without the flag they still build one machine at a time: host logic, no GPU.
"""
import numpy as np
import pandas as pd
import pytest

from gordo_components_b200 import builder

DET = "gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector"
MINMAX = "sklearn.preprocessing.MinMaxScaler"
AE = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2}}
RAW = {"gordo.machine.model.models.KerasRawModelRegressor": {"kind": {
    "spec": {"tensorflow.keras.models.Sequential": {"layers": [
        {"tensorflow.keras.layers.Dense": {"units": 3, "input_shape": [4]}},
        {"tensorflow.keras.layers.Dense": {"units": 4}}]}},
    "compile": {"loss": "mse", "optimizer": "adam"}}}}
LSTM = {"gordo.machine.model.models.KerasLSTMAutoEncoder": {"kind": "lstm_hourglass", "lookback_window": 6, "epochs": 2, "batch_size": 16}}
FORECAST = {"gordo.machine.model.models.KerasLSTMForecast": {"kind": "lstm_hourglass", "lookback_window": 6, "epochs": 2, "batch_size": 16}}


def _frame(rows=200, tags=4):
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(np.random.default_rng(0).random((rows, tags)), index=idx, columns=[f"tag-{i}" for i in range(tags)])


def _piped(net, scaler=MINMAX):
    return {"sklearn.pipeline.Pipeline": {"steps": [scaler, net]}}


def _ttr(regressor, transformer=MINMAX, **kw):
    return {"sklearn.compose.TransformedTargetRegressor": {"regressor": regressor, "transformer": transformer, **kw}}


def _machine(base, name="m", rows=200, evaluation=None, **detector_kw):
    X = _frame(rows)
    out = {"name": name, "model": {DET: {"base_estimator": base, **detector_kw}}, "dataset": {"X": X, "y": X}}
    if evaluation is not None:
        out["evaluation"] = evaluation
    return out


FF_FORMS = {"bare": AE, "piped": _piped(AE), "raw": RAW, "raw-piped": _piped(RAW)}
LSTM_FORMS = {"bare": LSTM, "piped": _piped(LSTM), "forecast": FORECAST, "forecast-piped": _piped(FORECAST)}


@pytest.mark.parametrize("form", sorted(FF_FORMS))
def test_feed_forward_ttr_is_batched_with_the_flag_only(form):
    machine = _machine(_ttr(FF_FORMS[form]))
    assert not builder._is_lstm_definition(machine)
    assert builder._canonical(0, machine) is None
    c = builder._canonical(0, machine, target_scaler=True)
    assert c is not None and c.target_scaler and c.input_scaler == form.endswith("piped")
    plain = builder._canonical(0, _machine(FF_FORMS[form]), target_scaler=True)
    assert plain is not None and not plain.target_scaler


@pytest.mark.parametrize("form", sorted(LSTM_FORMS))
def test_lstm_ttr_is_batched_with_the_flag_only(form):
    machine = _machine(_ttr(LSTM_FORMS[form]))
    assert builder._is_lstm_definition(machine)  # the LSTM classifier sees through the TTR ...
    assert builder._canonical_lstm(0, machine) is None  # ... and refuses it without the flag
    c = builder._canonical_lstm(0, machine, target_scaler=True)
    assert isinstance(c, builder._CanonicalLSTM) and c.target_scaler and c.input_scaler == form.endswith("piped")
    assert c.lookahead == (1 if form.startswith("forecast") else 0)
    assert builder._canonical(0, machine, target_scaler=True) is None  # the feed-forward classifier still refuses LSTM networks


REFUSED = {
    "standard-transformer": _ttr(AE, transformer="sklearn.preprocessing.StandardScaler"),
    "ranged-transformer": _ttr(AE, transformer={MINMAX: {"feature_range": [-1, 1]}}),
    "clipped-transformer": _ttr(AE, transformer={MINMAX: {"clip": True}}),
    "no-transformer": _ttr(AE, transformer=None),
    "func": {"sklearn.compose.TransformedTargetRegressor": {"regressor": AE, "func": "numpy.log1p", "inverse_func": "numpy.expm1"}},
    "standard-in-regressor": _ttr(_piped(AE, "sklearn.preprocessing.StandardScaler")),
    "nested-ttr": _ttr(_ttr(AE)),
}


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_other_target_regressors_are_refused(name):
    machine = _machine(REFUSED[name])
    assert builder._canonical(0, machine, target_scaler=True) is None


@pytest.mark.parametrize("name", ["standard-transformer", "ranged-transformer", "no-transformer", "func", "standard-in-regressor"])
def test_other_target_regressors_around_an_lstm_are_refused(name):
    swap = {"standard-transformer": _ttr(LSTM, transformer="sklearn.preprocessing.StandardScaler"),
            "ranged-transformer": _ttr(LSTM, transformer={MINMAX: {"feature_range": [-1, 1]}}),
            "no-transformer": _ttr(LSTM, transformer=None),
            "func": {"sklearn.compose.TransformedTargetRegressor": {"regressor": LSTM, "func": "numpy.log1p", "inverse_func": "numpy.expm1"}},
            "standard-in-regressor": _ttr(_piped(LSTM, "sklearn.preprocessing.StandardScaler"))}
    machine = _machine(swap[name])
    assert builder._is_lstm_definition(machine)
    assert builder._canonical_lstm(0, machine, target_scaler=True) is None


def test_the_target_regressor_test_is_shared():
    """All three classifiers take their TTR from one helper: the regressor when it is taken, a reason when it is not."""
    from sklearn.compose import TransformedTargetRegressor
    from sklearn.preprocessing import MinMaxScaler, StandardScaler

    reg = object()
    assert builder._target_regressor(reg) == (None, reg, False)
    ok = TransformedTargetRegressor(regressor=reg, transformer=MinMaxScaler())
    assert builder._target_regressor(ok) == (None, reg, True)
    reason, _, in_ttr = builder._target_regressor(ok, target_scaler=False)
    assert in_ttr and "target_scaler=True" in reason
    for bad in (TransformedTargetRegressor(regressor=reg, transformer=StandardScaler()), TransformedTargetRegressor(regressor=reg),
                TransformedTargetRegressor(regressor=reg, func=np.log1p, inverse_func=np.expm1)):
        reason, _, in_ttr = builder._target_regressor(bad)
        assert in_ttr and reason


def test_kfold_detectors_keep_their_ttr_route():
    kfcv = {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {"base_estimator": _ttr(_piped(AE))}}
    machine = {"name": "k", "model": kfcv, "dataset": {"X": _frame()}, "evaluation": {"cv": {"sklearn.model_selection.KFold": {"n_splits": 3}}}}
    c = builder._canonical_kfcv(0, machine)
    assert c is not None and c.target_scaler and c.input_scaler
    assert c.bucket()[-1] is True and not any(isinstance(e, tuple) and e[:1] == ("target_scaler",) for e in c.bucket())  # key unchanged


def test_bucket_keys_separate_ttr_machines():
    ff, ff_ttr = (builder._canonical(0, _machine(b), target_scaler=True) for b in (_piped(AE), _ttr(_piped(AE))))
    assert ff.bucket() != ff_ttr.bucket() and ff_ttr.bucket()[:-1] == ff.bucket() and ff_ttr.bucket()[-1] == ("target_scaler", True)
    assert ff.bucket() == builder._canonical(0, _machine(_piped(AE))).bucket()  # keys without a TTR are as before
    assert builder._canonical(1, _machine(_ttr(_piped(AE)), name="other"), target_scaler=True).bucket() == ff_ttr.bucket()
    lstm, lstm_ttr = (builder._canonical_lstm(0, _machine(b), target_scaler=True) for b in (LSTM, _ttr(LSTM)))
    assert lstm.bucket() != lstm_ttr.bucket() and lstm_ttr.bucket()[:-1] == lstm.bucket()
    assert lstm.bucket() == builder._canonical_lstm(0, _machine(LSTM)).bucket()
    assert ff_ttr.bucket(ragged=True) != ff.bucket(ragged=True)


def test_ttr_combines_with_the_other_options():
    stop = [{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "val_loss", "patience": 1}}]
    split = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2, "validation_split": 0.1, "callbacks": stop}}
    c = builder._canonical(0, _machine(_ttr(_piped(split)), shuffle=True, window=12), early_stopping=True, smoothing=True, target_scaler=True)
    assert c is not None and c.target_scaler and c.split == (True, 0.1, 32) and c.early_stopping is not None and c.window == 12
    assert builder._canonical(0, _machine(_ttr(_piped(split)), window=12), early_stopping=True, target_scaler=True) is None  # needs smoothing=True
    wide = {"gordo.machine.model.models.KerasLSTMAutoEncoder": {"kind": "lstm_hourglass", "lookback_window": 6, "epochs": 3, "batch_size": 64,
                                                                "callbacks": [{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "loss"}}]}}
    c = builder._canonical_lstm(0, _machine(_ttr(wide), window=6), wide_batches=True, early_stopping=True, smoothing=True, target_scaler=True)
    assert c is not None and c.target_scaler and c.fit["batch_size"] == 64 and c.early_stopping is not None and c.window == 6
    ragged = [builder._canonical(i, _machine(_ttr(AE), name=f"r{i}", rows=r), target_scaler=True) for i, r in enumerate((200, 260))]
    assert ragged[0].bucket() != ragged[1].bucket() and ragged[0].bucket(ragged=True) == ragged[1].bucket(ragged=True)


def test_without_the_flag_ttr_machines_build_one_at_a_time(monkeypatch):
    calls = []

    def fake_single(self, output_dir=None):
        calls.append(self.machine["name"])
        return f"single:{self.machine['name']}", builder._machine_out(self.machine, {"model": {}, "dataset": {}})

    def fake_bucket(members):
        raise AssertionError("no TTR machine is batched without target_scaler=True")

    monkeypatch.setattr(builder.ModelBuilder, "build", fake_single)
    monkeypatch.setattr(builder.FleetModelBuilder, "_build_bucket", staticmethod(fake_bucket))
    machines = [_machine(_ttr(AE), name="ff"), _machine(_ttr(_piped(AE)), name="ff-piped"), _machine(_ttr(LSTM), name="lstm"),
                _machine(_ttr(_piped(FORECAST)), name="forecast-piped")]
    results = builder.FleetModelBuilder(machines, smoothing=True, early_stopping=True, lstm_early_stopping=True, kfcv=True).build()
    assert calls == [m["name"] for m in machines] and [r for r, _ in results] == [f"single:{m['name']}" for m in machines]


def test_with_the_flag_ttr_machines_share_a_bucket_per_family(monkeypatch):
    buckets = []

    def fake_bucket(members):
        buckets.append(([c.machine["name"] for c in members], type(members[0]).__name__, members[0].target_scaler))
        return [(c.machine["name"], builder._machine_out(c.machine, {"model": {}, "dataset": {}})) for c in members]

    monkeypatch.setattr(builder.ModelBuilder, "build", lambda self, output_dir=None: pytest.fail(f"{self.machine['name']} fell back"))
    monkeypatch.setattr(builder.FleetModelBuilder, "_build_bucket", staticmethod(fake_bucket))
    machines = [_machine(_ttr(AE), name=f"ff-{i}") for i in range(3)] + [_machine(_ttr(LSTM), name=f"lstm-{i}") for i in range(3)]
    machines.append(_machine(AE, name="plain"))
    fleet = builder.FleetModelBuilder(machines, target_scaler=True)
    assert fleet.shard(0, 2).target_scaler and fleet.shard(1, 2).target_scaler
    fleet.build()
    assert sorted(buckets) == sorted([([f"ff-{i}" for i in range(3)], "_Canonical", True), ([f"lstm-{i}" for i in range(3)], "_CanonicalLSTM", True),
                                      (["plain"], "_Canonical", False)])
