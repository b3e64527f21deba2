"""Host side of EarlyStopping inside the fit kernel: the gb_fit_stop records and their C ABI, how make_stop resolves a callback,
and which definitions with callbacks the fleet builder batches (and how it buckets them).  No GPU needed."""
import ctypes as C
import os
import re

import numpy as np
import pandas as pd
import pytest

from gordo_components_b200 import _cabi, builder, engine
from gordo_components_b200.machine.model.models import EarlyStopping

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
ES = "tensorflow.keras.callbacks.EarlyStopping"
KAE = "gordo.machine.model.models.KerasAutoEncoder"


def production_ae(callbacks=None, **kw):
    """The estimator of the reference's production definition (test_anomaly_detectors.py, DiffBasedKFCVAnomalyDetector example)."""
    ae = {"kind": "feedforward_hourglass", "batch_size": 128, "compression_factor": 0.5, "encoding_layers": 1, "func": "tanh",
          "out_func": "linear", "optimizer": "Adam", "loss": "mse", "epochs": 1000, "validation_split": 0.1,
          "callbacks": [{ES: {"monitor": "val_loss", "patience": 10, "restore_best_weights": True}}] if callbacks is None else callbacks}
    ae.update(kw)
    return {KAE: ae}


def detector(ae, shuffle=True):
    return {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {
        "base_estimator": {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", ae]}},
        "scaler": "sklearn.preprocessing.MinMaxScaler", "shuffle": shuffle}}


EVALUATION = {"cv": {"sklearn.model_selection.TimeSeriesSplit": {"n_splits": 5}}}


def _machine(name="m", model=None, rows=600, tags=6, evaluation=EVALUATION):
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    X = pd.DataFrame(np.random.default_rng(rows).random((rows, tags)), index=idx, columns=[f"tag-{i}" for i in range(tags)])
    return {"name": name, "model": model or detector(production_ae()), "dataset": {"X": X, "y": X}, "evaluation": evaluation}


# ------------------------------------------------------------------------------------------------ C ABI
def header_struct_fields(name):
    text = open(os.path.join(ROOT, "include", "gordo_b200.h")).read()
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), text, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            ctype, names = decl.split(None, 1)
            fields += [(ctype, n.strip()) for n in names.split(",")]
    return fields


def test_stop_record_layout_matches_the_header():
    sizes = {"int32_t": 4, "double": 8}
    ofs, want = 0, []
    for ctype, name in header_struct_fields("gb_fit_stop"):
        ofs = (ofs + sizes[ctype] - 1) // sizes[ctype] * sizes[ctype]
        want.append((name, ofs))
        ofs += sizes[ctype]
    assert [n for n, _ in want] == [n for n, _ in _cabi.GbFitStop._fields_]
    assert ofs == C.sizeof(_cabi.GbFitStop) == _cabi.STOP_DTYPE.itemsize == 40
    for name, o in want:
        assert getattr(_cabi.GbFitStop, name).offset == o == _cabi.STOP_DTYPE.fields[name][1]


def test_fit_stop_is_exported_and_checks_its_arguments():
    import __graft_entry__ as ge

    ge.build()
    lib = _cabi.load_library()
    assert "gb_ffae_fit_stop" in _cabi.EXPORTS and lib.gb_abi_version() == 2
    fn = lib.gb_ffae_fit_stop
    assert fn.restype is C.c_int and len(fn.argtypes) == 23
    assert fn.argtypes[:18] == lib.gb_ffae_fit_split.argtypes[:18]
    net = _cabi.make_ffnet([4, 2, 4], ["tanh", "linear"])
    hp = _cabi.GbFitHParams(epochs=1, batch_size=4)
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    odd = C.c_void_p(p.value + 4)

    def call(stop, best, epochs, best_epoch):  # a host buffer stands in for every device array: nothing reaches the device
        return fn(C.byref(net), p, p, p, p, None, 1, 4, p, p, None, None, C.byref(hp), 4, p, p, None, None, stop, best, epochs, best_epoch, None)

    for args, word in (((p, None, p, p), b"best_params"), ((p, p, None, p), b"out_epochs"), ((p, p, p, None), b"out_best_epoch"),
                       ((p, odd, p, p), b"aligned")):
        assert call(*args) == -1 and word in lib.gb_last_error(), args
    with pytest.raises(ValueError):
        _cabi.check(call(p, None, p, p))
    # the checks of gb_ffae_fit_split still come first
    rc = fn(C.byref(net), p, p, p, p, p, 1, 4, p, p, None, None, C.byref(hp), 0, p, p, p, p, p, p, p, p, None)
    assert rc == -1 and b"val_batch" in lib.gb_last_error()


# ------------------------------------------------------------------------------------------------ make_stop
def test_make_stop_resolves_like_early_stopping():
    cbs = [EarlyStopping(monitor="val_loss", patience=10, restore_best_weights=True),
           {"monitor": "val_accuracy", "min_delta": -0.25, "patience": 3},
           {"monitor": "accuracy", "mode": "auto", "baseline": 0.5, "start_from_epoch": 2},
           {"monitor": "loss", "mode": "max", "min_delta": 1e-3},
           {"monitor": "loss", "mode": "bogus"}]
    rec = engine.make_stop(cbs)
    assert rec.dtype == _cabi.STOP_DTYPE and len(rec) == 5
    assert list(rec["monitor"]) == [2, 3, 1, 0, 0]
    for r, cb in zip(rec, cbs):
        es = cb if isinstance(cb, EarlyStopping) else EarlyStopping(**cb)
        assert r["mode"] == (1 if es.mode == "min" else -1)
        assert r["min_delta"] == es.min_delta >= 0 and r["patience"] == es.patience and r["start_from_epoch"] == es.start_from_epoch
        assert bool(r["restore_best"]) == es.restore_best_weights and bool(r["has_baseline"]) == (es.baseline is not None)
    assert list(rec["mode"]) == [1, -1, -1, -1, 1] and rec["min_delta"][1] == 0.25 and rec["baseline"][2] == 0.5

    class KerasLike:  # a keras object handed over by the caller: its attributes, through EarlyStopping.__init__
        monitor, min_delta, patience, mode, baseline, restore_best_weights, start_from_epoch = "val_loss", -0.1, 4, "auto", None, False, 0

    (r,) = engine.make_stop([KerasLike()])
    assert (r["monitor"], r["mode"], r["min_delta"], r["patience"]) == (2, 1, 0.1, 4)
    raw = engine.make_stop(cbs[:1]).view(np.uint8).tobytes()
    s = _cabi.GbFitStop.from_buffer_copy(raw)
    assert (s.monitor, s.mode, s.patience, s.restore_best) == (2, 1, 10, 1)
    with pytest.raises(ValueError):
        engine.make_stop([{"monitor": "acc"}])


# ------------------------------------------------------------------------------------------------ the builder
def canonical(index, machine):
    return builder._canonical(index, machine, early_stopping=True)


def test_callbacks_keep_the_per_machine_path_by_default():
    # without the opt-in a callback still sends the machine to ModelBuilder, whatever it is
    for callbacks in (None, [{ES: {"monitor": "loss"}}], [EarlyStopping(monitor="val_loss", patience=10, restore_best_weights=True)]):
        assert builder._canonical(0, _machine(model=detector(production_ae(callbacks)))) is None
    assert builder._canonical(0, _machine(model=detector(production_ae([])))) is not None
    assert not builder.FleetModelBuilder([]).early_stopping
    fmb = builder.FleetModelBuilder([_machine(f"m{i}") for i in range(4)], early_stopping=True)
    assert fmb.early_stopping and fmb.shard(1, 2).early_stopping and len(fmb.shard(1, 2).machines) == 2


def test_canonical_takes_the_production_definition():
    c = canonical(0, _machine())
    assert c is not None and c.input_scaler and c.n_splits == 5 and c.split == (True, 0.1, 128)
    assert c.fit == {"epochs": 1000, "batch_size": 128, "shuffle": True}
    es = c.early_stopping
    assert isinstance(es, EarlyStopping) and (es.monitor, es.patience, es.restore_best_weights, es.mode) == ("val_loss", 10, True, "min")
    # the callback as an object, as gordo's serializer may hand it over
    obj = canonical(0, _machine(model=detector(production_ae([EarlyStopping(monitor="val_loss", patience=10, restore_best_weights=True)]))))
    assert obj is not None and obj.early_stopping.patience == 10 and obj.bucket() == c.bucket()
    # without callbacks: the same model, another bucket
    plain = canonical(0, _machine(model=detector(production_ae([]))))
    assert plain is not None and plain.early_stopping is None and plain.bucket() != c.bucket()
    # monitors this fit reports: loss always, val_loss with the split
    for monitor in ("loss", "val_loss"):
        assert canonical(0, _machine(model=detector(production_ae([{ES: {"monitor": monitor}}])))) is not None
    no_split = {KAE: {k: v for k, v in production_ae([{ES: {"monitor": "loss"}}])[KAE].items() if k != "validation_split"}}
    assert canonical(0, _machine(model=detector(no_split))).split == (True, 0.0, None)


def test_canonical_refuses_other_callbacks():
    refused = [
        [{ES: {"monitor": "val_loss"}}, {ES: {"monitor": "loss"}}],          # two callbacks
        [{"tensorflow.keras.callbacks.TerminateOnNaN": {}}],                 # not an EarlyStopping (the estimator ignores it)
        [{ES: {"monitor": "val_loss"}}, {"tensorflow.keras.callbacks.TerminateOnNaN": {}}],
        [{ES: {"monitor": "acc"}}],                                          # a metric the fit does not report
        [{ES: {"monitor": "val_mse"}}],
    ]
    for callbacks in refused:
        assert canonical(0, _machine(model=detector(production_ae(callbacks)))) is None, callbacks
    # val_loss without a validation_split: nothing to monitor
    no_split = {KAE: {k: v for k, v in production_ae()[KAE].items() if k != "validation_split"}}
    assert canonical(0, _machine(model=detector(no_split))) is None


def test_machines_differing_in_the_callback_share_a_bucket():
    defs = [{"monitor": "val_loss", "patience": p, "restore_best_weights": r, "min_delta": d} for p, r, d in ((10, True, 0), (3, False, 1e-4), (0, True, 0.5))]
    cs = [canonical(i, _machine(f"m{i}", model=detector(production_ae([{ES: d}])))) for i, d in enumerate(defs)]
    assert len({c.bucket() for c in cs}) == 1
    assert [c.early_stopping.patience for c in cs] == [10, 3, 0]
    rec = engine.make_stop([c.early_stopping for c in cs])
    assert list(rec["patience"]) == [10, 3, 0] and list(rec["restore_best"]) == [1, 0, 1]
