"""Which LSTM machines FleetModelBuilder batches, how it buckets them and how shard splits them: host logic, no GPU."""
import numpy as np
import pandas as pd
import pytest

from gordo_components_b200 import builder


def _frame(rows=200, tags=4):
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(np.random.default_rng(0).random((rows, tags)), index=idx, columns=[f"tag-{i}" for i in range(tags)])


def _lstm(cls_name="KerasLSTMAutoEncoder", scaler=None, **kwargs):
    est = {f"gordo.machine.model.models.{cls_name}": {"kind": "lstm_hourglass", "lookback_window": 6, "epochs": 2, "batch_size": 16, **kwargs}}
    base = {"sklearn.pipeline.Pipeline": {"steps": [scaler, est]}} if scaler else est
    return base


def _machine(name="m", base=None, rows=200, detector=None, evaluation=None, **detector_kw):
    model = {detector or "gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": base or _lstm(), **detector_kw}}
    out = {"name": name, "model": model, "dataset": {"X": _frame(rows)}}
    if evaluation is not None:
        out["evaluation"] = evaluation
    return out


@pytest.mark.parametrize("machine", [
    _machine(),
    _machine(base=_lstm("KerasLSTMForecast")),
    _machine(base=_lstm(scaler="sklearn.preprocessing.MinMaxScaler")),
    _machine(base=_lstm("KerasLSTMForecast", scaler="sklearn.preprocessing.MinMaxScaler")),
    _machine(evaluation={"metrics": ["r2_score", "sklearn.metrics.mean_squared_error"], "scoring_scaler": None}),
], ids=["autoencoder", "forecast", "autoencoder-minmax", "forecast-minmax", "metrics-subset"])
def test_canonical_lstm_forms_are_accepted(machine):
    assert builder._is_lstm_definition(machine)
    c = builder._canonical_lstm(0, machine)
    assert isinstance(c, builder._CanonicalLSTM)
    assert c.fit == {"epochs": 2, "batch_size": 16, "shuffle": False} and c.n_splits == 3
    assert c.lookahead == (1 if "Forecast" in str(machine["model"]) else 0)
    assert c.input_scaler == ("Pipeline" in str(machine["model"]))
    assert builder._canonical(0, machine) is None  # the feed-forward classifier still refuses LSTM definitions


@pytest.mark.parametrize("machine", [
    _machine(evaluation={"cv_mode": "cross_val_only"}),
    _machine(evaluation={"metrics": ["explained_variance_score", "max_error"]}),
    _machine(evaluation={"scoring_scaler": "sklearn.preprocessing.StandardScaler"}),
    _machine(evaluation={"cv": {"sklearn.model_selection.TimeSeriesSplit": {"n_splits": 3, "gap": 2}}}),
    _machine(evaluation={"cv": {"sklearn.model_selection.KFold": {"n_splits": 3}}}),
    _machine(shuffle=True),
    _machine(window=12),
    _machine(scaler="sklearn.preprocessing.StandardScaler"),
    _machine(detector="gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector"),
    _machine(base=_lstm(scaler="sklearn.preprocessing.StandardScaler")),
    _machine(base=_lstm(callbacks=[{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "loss", "patience": 1}}])),
    _machine(base=_lstm(batch_size=64)),
    _machine(rows=24),   # fold 0 trains on 6 rows: no prediction window at lookback 6
    _machine(rows=27),   # fold 0 has training windows, but test blocks of 6 rows leave no room at lookback 6
    _machine(base={"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass"}}),
], ids=["cross-val-only", "other-metric", "scoring-scaler", "tss-gap", "kfold", "shuffle", "window", "detector-scaler", "kfcv-detector",
        "other-input-scaler", "callbacks", "batch-64", "too-few-rows", "short-test-block", "feed-forward"])
def test_non_canonical_lstm_variations_are_refused(machine):
    assert builder._canonical_lstm(0, machine) is None


def test_lstm_buckets_separate_lookback_lookahead_input_scaler_and_rows():
    base = builder._canonical_lstm(0, _machine())
    same = builder._canonical_lstm(1, _machine(name="n"))
    assert base.bucket() == same.bucket()
    variants = [
        _machine(base=_lstm(lookback_window=8)),
        _machine(base=_lstm("KerasLSTMForecast")),
        _machine(base=_lstm(scaler="sklearn.preprocessing.MinMaxScaler")),
        _machine(rows=240),
        _machine(base=_lstm(epochs=3)),
    ]
    keys = [builder._canonical_lstm(i, m).bucket() for i, m in enumerate(variants)]
    assert len(set(keys) | {base.bucket()}) == len(variants) + 1


def test_shard_covers_every_lstm_machine_once():
    machines = [_machine(name=f"lstm-{i}", base=_lstm("KerasLSTMForecast" if i % 2 else "KerasLSTMAutoEncoder")) for i in range(7)]
    machines.insert(3, _machine(name="ff", base={"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass"}}))
    fleet = builder.FleetModelBuilder(machines)
    seen = []
    for rank in range(3):
        part = fleet.shard(rank, 3)
        for i, m in enumerate(part.machines):
            seen.append(m["name"])
            if m["name"].startswith("lstm"):
                assert isinstance(builder._canonical_lstm(i, m), builder._CanonicalLSTM)
    assert sorted(seen) == sorted(m["name"] for m in machines)
