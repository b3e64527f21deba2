"""
Which smoothing-window detectors FleetModelBuilder(smoothing=True) batches, how their window enters the bucket keys and how shard
carries the flag, and the argument checks of gb_thresholds_pair: host logic, no GPU.
"""
import ctypes as C

import numpy as np
import pandas as pd
import pytest

from gordo_components_b200 import _cabi, builder

DET = "gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector"
AE = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2}}
SCALED_AE = {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", AE]}}
LSTM = {"gordo.machine.model.models.KerasLSTMAutoEncoder": {"kind": "lstm_hourglass", "lookback_window": 6, "epochs": 2, "batch_size": 16}}


def _frame(rows=200, tags=4):
    idx = pd.date_range("2020-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(np.random.default_rng(0).random((rows, tags)), index=idx, columns=[f"tag-{i}" for i in range(tags)])


def _machine(base=AE, name="m", **detector_kw):
    X = _frame()
    return {"name": name, "model": {DET: {"base_estimator": base, **detector_kw}}, "dataset": {"X": X, "y": X}}


def _classify(machine, smoothing):
    if builder._is_lstm_definition(machine):
        return builder._canonical_lstm(0, machine, smoothing=smoothing)
    return builder._canonical(0, machine, smoothing=smoothing)


@pytest.mark.parametrize("base", [AE, SCALED_AE, LSTM], ids=["bare", "minmax-pipeline", "lstm"])
@pytest.mark.parametrize("method", [None, "smm", "sma", "ewma"])
def test_window_detectors_are_batched_with_the_flag_only(base, method):
    kw = {"window": 144} if method is None else {"window": 144, "smoothing_method": method}
    machine = _machine(base, **kw)
    assert _classify(machine, smoothing=False) is None  # as before: the per-machine path
    c = _classify(machine, smoothing=True)
    assert c is not None and c.window == 144
    assert c.model.window == 144 and c.model.smoothing_method == (method or "smm")  # the detector keeps its own window and method
    assert c.input_scaler == (base is SCALED_AE)


@pytest.mark.parametrize("base", [AE, LSTM], ids=["feed-forward", "lstm"])
@pytest.mark.parametrize("kw", [{"window": 0}, {"window": 2.5}, {"window": True}, {"window": 12, "smoothing_method": "median"}],
                         ids=["zero", "float", "bool", "median"])
def test_bad_windows_and_methods_are_refused(base, kw):
    assert _classify(_machine(base, **kw), smoothing=True) is None


def test_other_refusals_stay_with_the_flag():
    assert builder._canonical_lstm(0, _machine(LSTM, window=12, shuffle=True), smoothing=True) is None  # shuffled LSTM detectors
    robust = _machine(AE, window=12, scaler="sklearn.preprocessing.RobustScaler")
    assert builder._canonical(0, robust, smoothing=True) is None
    kfcv = {"name": "k", "model": {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {"base_estimator": AE, "window": 12}},
            "dataset": {"X": _frame()}}
    assert builder._canonical(0, kfcv, smoothing=True) is None


@pytest.mark.parametrize("base", [AE, SCALED_AE, LSTM], ids=["bare", "minmax-pipeline", "lstm"])
def test_bucket_keys_gain_the_window_only_when_set(base):
    plain = _machine(base)
    assert _classify(plain, smoothing=True).bucket() == _classify(plain, smoothing=False).bucket()
    assert _classify(plain, smoothing=True).bucket(ragged=True) == _classify(plain, smoothing=False).bucket(ragged=True)
    w12 = _classify(_machine(base, window=12), smoothing=True)
    w144 = _classify(_machine(base, window=144), smoothing=True)
    assert len({w12.bucket(), w144.bucket(), _classify(plain, smoothing=True).bucket()}) == 3
    # the method does not enter the thresholds: it does not split buckets
    assert _classify(_machine(base, window=12, smoothing_method="ewma"), smoothing=True).bucket() == w12.bucket()


def test_kfold_keys_do_not_change():
    kfcv = {"name": "k", "model": {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {"base_estimator": AE, "window": 12}},
            "dataset": {"X": _frame()}, "evaluation": {"cv": {"sklearn.model_selection.KFold": {"n_splits": 3}}}}
    c = builder._canonical_kfcv(0, kfcv)
    assert c is not None and c.window is None and c.bucket()[-5] == 12


def test_shard_keeps_the_flag():
    fmb = builder.FleetModelBuilder([_machine(name=f"m{i}", window=12) for i in range(4)], smoothing=True)
    assert fmb.smoothing and fmb.shard(1, 2).smoothing and len(fmb.shard(1, 2).machines) == 2
    assert not builder.FleetModelBuilder([_machine()]).smoothing


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


@pytest.mark.parametrize("name", ["gb_thresholds_pair", "gb_thresholds_pair_f64"])
def test_pair_argument_checks_need_no_device(lib, name):
    fn = getattr(lib, name)
    jobs, p = C.c_void_p(16), C.c_void_p(64)  # never dereferenced: every check comes before any launch

    def call(**kw):
        a = dict(jobs=jobs, n_jobs=1, max_rows=10, tag=p, total=p, n_out=4, w0=6, w1=12, f0=p, a0=p, f1=p, a1=p, n_slots=1)
        a.update(kw)
        return fn(a["jobs"], a["n_jobs"], a["max_rows"], a["tag"], a["total"], a["n_out"], a["w0"], a["w1"], a["f0"], a["a0"], a["f1"],
                  a["a1"], a["n_slots"], None)

    for kw, code, field in [
        ({"jobs": None}, -1, b"jobs"),
        ({"f1": None}, -1, b"feat_thr1"),
        ({"tag": None}, -1, b"tag_unscaled"),
        ({"a0": None}, -1, b"agg_thr0"),
        ({"n_out": 0}, -2, b"n_out"),
        ({"n_out": 257}, -2, b"n_out"),
        ({"w0": 0}, -1, b"w0"),
        ({"w1": -3}, -1, b"w1"),
        ({"max_rows": -1}, -1, b"max_rows"),
        ({"n_jobs": -1}, -1, b"n_jobs"),
        ({"n_slots": -1}, -1, b"n_slots"),
    ]:
        assert call(**kw) == code, kw
        assert field in lib.gb_last_error(), (kw, lib.gb_last_error())
    # no jobs: nothing to do, and nothing launched
    assert call(n_jobs=0) == 0
    with pytest.raises(ValueError):
        _cabi.check(call(w1=0))
