"""Host side of the batched build of shuffling detectors with a validation split: which definitions the builder batches, the row
maps the fleet hands the fit kernel, and the C ABI of gb_ffae_fit_split.  No GPU needed."""
import ctypes as C

import numpy as np
import pandas as pd
import pytest
from sklearn.utils import shuffle as sk_shuffle

from gordo_components_b200 import _cabi, builder, engine

# the model block of the reference's examples/model-configuration.yaml, with its gordo.* class paths
EXAMPLE_AE = {"gordo.machine.model.models.KerasAutoEncoder": {
    "batch_size": 128, "compression_factor": 0.6, "encoding_layers": 1, "epochs": 100, "func": "tanh", "kind": "feedforward_hourglass",
    "loss": "mse", "optimizer": "Adam", "out_func": "linear", "validation_split": 0.1}}


def example_model(shuffle=True, ae=EXAMPLE_AE):
    return {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {
        "base_estimator": {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", ae]}},
        "scaler": "sklearn.preprocessing.MinMaxScaler", "shuffle": shuffle, "smoothing_method": "smm"}}


EXAMPLE_EVALUATION = {"cv": {"sklearn.model_selection.TimeSeriesSplit": {"n_splits": 5}}}


def _machine(name="m", model=None, rows=600, tags=6, evaluation=EXAMPLE_EVALUATION):
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    X = pd.DataFrame(np.random.default_rng(rows).random((rows, tags)), index=idx, columns=[f"tag-{i}" for i in range(tags)])
    return {"name": name, "model": model or example_model(), "dataset": {"X": X, "y": X}, "evaluation": evaluation}


def _without_split(ae):
    kw = dict(ae["gordo.machine.model.models.KerasAutoEncoder"])
    kw.pop("validation_split")
    return {"gordo.machine.model.models.KerasAutoEncoder": kw}


def test_canonical_takes_the_example_definition():
    c = builder._canonical(0, _machine())
    assert c is not None and c.input_scaler and c.n_splits == 5
    assert c.fit == {"epochs": 100, "batch_size": 128, "shuffle": True}
    assert c.split == (True, 0.1, 128)
    assert c.bucket() == builder._canonical(1, _machine("other")).bucket()
    # the same model without the detector shuffle, or without the split, is another bucket
    unshuffled = builder._canonical(0, _machine(model=example_model(shuffle=False)))
    unsplit = builder._canonical(0, _machine(model=example_model(ae=_without_split(EXAMPLE_AE))))
    assert unshuffled.split == (False, 0.1, 128) and unsplit.split == (True, 0.0, None)
    assert len({c.bucket(), unshuffled.bucket(), unsplit.bucket()}) == 3
    vb = {"gordo.machine.model.models.KerasAutoEncoder": dict(EXAMPLE_AE["gordo.machine.model.models.KerasAutoEncoder"], validation_batch_size=16)}
    small = builder._canonical(0, _machine(model=example_model(ae=vb)))
    assert small.split == (True, 0.1, 16) and small.bucket() != c.bucket()


def test_canonical_refusals_with_a_split():
    # callbacks still take the per-machine loop
    stopping = {"gordo.machine.model.models.KerasAutoEncoder": dict(EXAMPLE_AE["gordo.machine.model.models.KerasAutoEncoder"],
                                                                    callbacks=[{"tensorflow.keras.callbacks.EarlyStopping": {"patience": 1}}])}
    assert builder._canonical(0, _machine(model=example_model(ae=stopping))) is None
    # 12 rows, 5 folds: the first fold has 2 rows, and validation_split 0.6 leaves it floor(2 * 0.4) = 0 training rows
    big = {"gordo.machine.model.models.KerasAutoEncoder": dict(EXAMPLE_AE["gordo.machine.model.models.KerasAutoEncoder"], validation_split=0.6)}
    assert builder._canonical(0, _machine(model=example_model(ae=big), rows=12)) is None
    assert builder._canonical(0, _machine(model=example_model(ae=big), rows=18)) is not None  # first fold: 3 rows, 1 trains
    outside = {"gordo.machine.model.models.KerasAutoEncoder": dict(EXAMPLE_AE["gordo.machine.model.models.KerasAutoEncoder"], validation_split=1.5)}
    assert builder._canonical(0, _machine(model=example_model(ae=outside))) is None


def slot_maps(N, K):
    """What build_fleet hands the kernel for every slot length: the maps concatenated, and each slot length's offset."""
    test = N // (K + 1)
    slot_n = [N] + [N - (K - k) * test for k in range(K)]
    maps = [sk_shuffle(np.arange(n), random_state=0) for n in slot_n]
    return slot_n, np.concatenate(maps), np.cumsum([0] + slot_n[:-1])


@pytest.mark.parametrize("N,K", [(600, 5), (1000, 3), (37, 3)])
def test_row_map_is_the_detectors_shuffle(N, K):
    X = np.random.default_rng(N).random((N, 3))
    y = X * 2
    slot_n, row_map, ofs = slot_maps(N, K)
    for n, o in zip(slot_n, ofs):
        m = row_map[o:o + n]
        Xs, ys = sk_shuffle(X[:n], y[:n], random_state=0)  # DiffBasedAnomalyDetector.fit on the slot's rows
        assert np.array_equal(X[m], Xs) and np.array_equal(y[m], ys)


def test_split_records_match_ctypes():
    assert _cabi.SPLIT_DTYPE.itemsize == C.sizeof(_cabi.GbFitSplit) == 16
    for name in ("n_val", "reserved", "map_ofs"):
        assert _cabi.SPLIT_DTYPE.fields[name][1] == getattr(_cabi.GbFitSplit, name).offset
    split = engine.make_split([3, 0], [10, -1])
    raw = split.view(np.uint8).tobytes()
    rec = (_cabi.GbFitSplit * 2).from_buffer_copy(raw)
    assert (rec[0].n_val, rec[0].map_ofs, rec[1].n_val, rec[1].map_ofs) == (3, 10, 0, -1)


def test_fit_split_is_exported():
    import __graft_entry__ as ge

    ge.build()
    lib = _cabi.load_library()
    assert "gb_ffae_fit_split" in _cabi.EXPORTS
    assert lib.gb_abi_version() == 2
    fn = lib.gb_ffae_fit_split
    assert fn.restype is C.c_int and len(fn.argtypes) == 19
    assert fn.argtypes[5] is _cabi._P and fn.argtypes[12]._type_ is _cabi.GbFitHParams and fn.argtypes[13] is C.c_int32
    # argument checks run before any device work
    net = _cabi.make_ffnet([4, 2, 4], ["tanh", "linear"])
    hp = _cabi.GbFitHParams(epochs=1, batch_size=4)
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    rc = fn(C.byref(net), p, p, p, p, p, 1, 4, p, p, None, None, C.byref(hp), 0, p, p, p, p, None)
    assert rc == -1 and b"val_batch" in lib.gb_last_error()
    rc = fn(C.byref(net), p, p, p, p, p, 1, 4, p, p, None, None, C.byref(hp), 4, p, p, None, None, None)
    assert rc == -1 and b"out_val_loss" in lib.gb_last_error()
