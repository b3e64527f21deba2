"""Host side of EarlyStopping inside the LSTM fit launches: the C entry points' argument checks (no device needed), which LSTM
definitions with a callback FleetModelBuilder(lstm_early_stopping=True) batches, how it buckets them and how shard carries the
flag.  No GPU needed."""
import ctypes as C

import numpy as np
import pandas as pd
import pytest

from gordo_components_b200 import _cabi, builder, engine

ES = "tensorflow.keras.callbacks.EarlyStopping"


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


# ------------------------------------------------------------------------------------------------ C ABI
def _net():
    return _cabi.make_lstmnet(4, [8, 3, 8], ["tanh"] * 3, 4, "linear", 6)


def _call(lib, entry, batch, stop, best=C.c_void_p(256), out_epochs=C.c_void_p(512), out_best=C.c_void_p(768), n_jobs=2):
    hp = _cabi.GbLstmFitHParams()
    hp.epochs, hp.batch_size, hp.lookahead, hp.primer = 3, batch, 0, 1
    hp.lr, hp.beta1, hp.beta2, hp.eps = 1e-3, 0.9, 0.999, 1e-7
    p = C.c_void_p(256)  # never dereferenced: every refusal below happens before anything is enqueued
    rec = None if stop is None else stop.ctypes.data_as(C.c_void_p)
    return getattr(lib, entry)(C.byref(_net()), p, p, p, p, p, n_jobs, 10, p, p, C.byref(hp), p, p, p, 0, None, rec, best, out_epochs,
                               out_best, None)


ENTRIES = [("gb_lstm_fit_stop", 16), ("gb_lstm_fit_tc_stop", 100)]


@pytest.mark.parametrize("entry,batch", ENTRIES)
def test_stop_arguments_are_refused_without_a_device(lib, entry, batch):
    good = engine.make_stop([{"monitor": "loss", "patience": 2}, {"monitor": "accuracy", "restore_best_weights": True}])
    for kw in ({"best": None}, {"out_epochs": None}, {"out_best": None}):
        assert _call(lib, entry, batch, good, **kw) == -1 and b"best_params, out_epochs and out_best_epoch" in lib.gb_last_error()
    assert _call(lib, entry, batch, good, best=C.c_void_p(260)) == -1 and b"aligned" in lib.gb_last_error()
    for field, value, word in (("monitor", 4, b"monitor"), ("monitor", -1, b"monitor"), ("mode", 0, b"mode"), ("mode", 2, b"mode"),
                               ("patience", -1, b"patience"), ("min_delta", -0.5, b"min_delta")):
        bad = good.copy()
        bad[1][field] = value
        rc = _call(lib, entry, batch, bad)
        assert rc == -1 and word in lib.gb_last_error(), (field, value)
        with pytest.raises(ValueError):
            _cabi.check(rc)
    # the checks of the entry point without a rule come first, unchanged
    assert _call(lib, entry, 300, good) == -2
    assert _call(lib, entry, batch, good, n_jobs=-1) == -1 and b"n_jobs" in lib.gb_last_error()


def test_fp32_stop_entry_refuses_wide_batches(lib):
    assert _call(lib, "gb_lstm_fit_stop", 64, engine.make_stop([{"monitor": "loss"}] * 2)) == -2


def test_stop_state_bytes(lib):
    size = lib.gb_lstm_fit_stop_state_bytes
    assert size(0) == 16 and size(1) == 16 + 24 + 56 and size(32) == 16 + 32 * 80 and size(-1) == 0
    assert size(7) % 8 == 0


def test_workspace_queries_are_unchanged_by_the_stop_path(lib):
    net = _net()
    ws = lib.gb_lstm_fit_workspace_bytes(C.byref(net), 3)
    assert ws > 0 and ws % 8 == 0  # the rule's state starts right after it
    assert lib.gb_lstm_fit_tc_workspace_bytes(C.byref(net), 3, 100) % 8 == 0


# ------------------------------------------------------------------------------------------------ the builder
def _frame(rows=200, tags=4):
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(np.random.default_rng(0).random((rows, tags)), index=idx, columns=[f"tag-{i}" for i in range(tags)])


def _lstm(cls_name="KerasLSTMAutoEncoder", scaler=None, **kwargs):
    est = {f"gordo.machine.model.models.{cls_name}": {"kind": "lstm_hourglass", "lookback_window": 6, "epochs": 4, "batch_size": 16, **kwargs}}
    return {"sklearn.pipeline.Pipeline": {"steps": [scaler, est]}} if scaler else est


def _machine(name="m", base=None, rows=200):
    model = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": base or _lstm()}}
    return {"name": name, "model": model, "dataset": {"X": _frame(rows)}}


def _es(**kw):
    return [{ES: {"monitor": "loss", "patience": 2, **kw}}]


@pytest.mark.parametrize("base", [
    _lstm(callbacks=_es()),
    _lstm("KerasLSTMForecast", callbacks=_es(restore_best_weights=True)),
    _lstm(scaler="sklearn.preprocessing.MinMaxScaler", callbacks=_es(min_delta=0.01, baseline=0.5)),
    _lstm(callbacks=_es(mode="max", start_from_epoch=1)),
    _lstm(callbacks=_es(patience=0)),
    _lstm(batch_size=64, callbacks=_es()),
], ids=["loss", "forecast-restore", "minmax-baseline", "max-start-from", "patience-0", "wide"])
def test_one_reported_early_stopping_is_accepted_with_the_flag(base):
    m = _machine(base=base)
    c = builder._canonical_lstm(0, m, wide_batches=True, early_stopping=True)
    assert isinstance(c, builder._CanonicalLSTM)
    assert c.early_stopping is not None and c.early_stopping.monitor in ("loss", "accuracy")
    assert builder._canonical_lstm(0, m, wide_batches=True) is None  # without the flag: ModelBuilder, as before


@pytest.mark.parametrize("base", [
    _lstm(callbacks=_es(monitor="val_loss")),
    _lstm(callbacks=_es(monitor="val_accuracy")),
    _lstm(callbacks=_es(monitor="mean_absolute_error")),
    _lstm(callbacks=_es(monitor="accuracy")),  # the LSTM specs report no accuracy unless the metric is named
    _lstm(callbacks=_es() + _es(patience=3)),
    _lstm(callbacks=[{"tensorflow.keras.callbacks.ModelCheckpoint": {"filepath": "x"}}]),
    _lstm(callbacks=_es() + [{"tensorflow.keras.callbacks.ReduceLROnPlateau": {}}]),
    _lstm(callbacks=_es(), validation_split=0.1),
    _lstm(validation_split=0.1),
    _lstm(batch_size=64, callbacks=_es()),  # wide batches still need their own flag
], ids=["val-loss", "val-accuracy", "unreported-metric", "accuracy-without-metric", "two-early-stoppings", "other-callback", "early-stopping-and-other",
        "validation-split-with-callback", "validation-split", "wide-without-flag"])
def test_other_callbacks_and_validation_split_are_refused(base):
    assert builder._canonical_lstm(0, _machine(base=base), early_stopping=True) is None


def test_accuracy_monitor_needs_the_accuracy_metric():
    metrics = builder._canonical_lstm(0, _machine(base=_lstm(callbacks=_es())), early_stopping=True).spec.metrics
    accepted = builder._canonical_lstm(0, _machine(base=_lstm(callbacks=_es(monitor="accuracy"))), early_stopping=True) is not None
    assert accepted == ("accuracy" in metrics)


def test_callback_parameters_do_not_split_a_bucket():
    keys = {builder._canonical_lstm(i, _machine(name=f"m{i}", base=_lstm(callbacks=cb)), early_stopping=True).bucket()
            for i, cb in enumerate([_es(), _es(patience=5), _es(min_delta=0.1, restore_best_weights=True), _es(baseline=0.2, start_from_epoch=2)])}
    assert len(keys) == 1
    plain = builder._canonical_lstm(9, _machine(name="plain"), early_stopping=True)
    assert plain.early_stopping is None and plain.bucket() not in keys  # with and without a callback: separate launches


def test_flag_survives_shard():
    machines = [_machine(name=f"m{i}") for i in range(5)]
    fleet = builder.FleetModelBuilder(machines, lstm_early_stopping=True, lstm_wide_batches=True)
    for rank in range(3):
        part = fleet.shard(rank, 3)
        assert part.lstm_early_stopping and part.lstm_wide_batches
    assert not builder.FleetModelBuilder(machines).shard(0, 2).lstm_early_stopping
