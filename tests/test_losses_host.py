"""
Host side of the training losses (no GPU): which compile_kwargs losses the factories accept and how they resolve, that a spec
pickled before the loss field existed loads as mean squared error, that the fleet builder buckets machines by loss, and the
gb_loss ids of the C ABI.
"""
import ctypes as C
import os
import pickle
import re

import numpy as np
import pandas as pd
import pytest

from gordo_components_b200 import _cabi, builder
from gordo_components_b200.machine.model.factories import feedforward_autoencoder as ffa
from gordo_components_b200.machine.model.factories import lstm_autoencoder as lsa
from gordo_components_b200.machine.model.factories.specs import FFNetSpec, LSTMNetSpec, resolve_loss
from gordo_components_b200.machine.model.models import KerasAutoEncoder, KerasLSTMAutoEncoder

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))

SPELLINGS = {
    "mse": ("mse", "MSE", "mean_squared_error", "MeanSquaredError"),
    "mae": ("mae", "MAE", "mean_absolute_error", "MeanAbsoluteError"),
    "mape": ("mape", "MAPE", "mean_absolute_percentage_error", "MeanAbsolutePercentageError"),
    "msle": ("msle", "MSLE", "mean_squared_logarithmic_error", "MeanSquaredLogarithmicError"),
    "huber": ("huber", "Huber"),
    "log_cosh": ("log_cosh", "LogCosh"),
}
REFUSED = ["binary_crossentropy", "categorical_crossentropy", "sparse_categorical_crossentropy", "hinge", "squared_hinge",
           "poisson", "kld", "kl_divergence", "cosine_similarity", "logcosh", "huber_loss", "Mae", "l1", None, 3,
           {"class_name": "Huber", "config": {"delta": 2.0}}]


@pytest.mark.parametrize("canonical,name", [(c, n) for c, names in SPELLINGS.items() for n in names])
def test_every_keras_spelling_resolves(canonical, name):
    assert resolve_loss({"loss": name}) == canonical
    assert ffa.feedforward_hourglass(10, compile_kwargs={"loss": name}).loss == canonical
    assert ffa.feedforward_model(6, encoding_dim=(4,), encoding_func=("tanh",), decoding_dim=(4,), decoding_func=("tanh",),
                                 compile_kwargs={"loss": name}).loss == canonical
    assert lsa.lstm_hourglass(10, compile_kwargs={"loss": name}).loss == canonical
    assert lsa.lstm_symmetric(4, dims=(3,), funcs=("tanh",), compile_kwargs={"loss": name, "metrics": ["accuracy"]}).loss == canonical


def test_the_default_is_mean_squared_error():
    assert resolve_loss(None) == resolve_loss({}) == resolve_loss({"metrics": ["accuracy"]}) == "mse"
    assert ffa.feedforward_hourglass(10).loss == "mse" and lsa.lstm_model(4).loss == "mse"


@pytest.mark.parametrize("loss", REFUSED, ids=[str(r) for r in REFUSED])
def test_other_losses_are_refused_at_construction(loss):
    with pytest.raises(ValueError, match="implement the losses"):
        ffa.feedforward_hourglass(10, compile_kwargs={"loss": loss})
    with pytest.raises(ValueError, match="implement the losses"):
        lsa.lstm_hourglass(10, compile_kwargs={"loss": loss})
    with pytest.raises(ValueError):
        KerasAutoEncoder(kind="feedforward_hourglass", n_features=6, compile_kwargs={"loss": loss})._build_spec()


def test_a_top_level_loss_key_means_nothing():
    """The reference ignores a `loss:` next to `kind:` (its compile reads compile_kwargs only); so does this code."""
    for loss in ("mae", "binary_crossentropy"):
        assert ffa.feedforward_hourglass(10, loss=loss).loss == "mse"
        assert KerasAutoEncoder(kind="feedforward_hourglass", n_features=6, loss=loss)._build_spec().loss == "mse"
        assert KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=3, n_features=6, loss=loss)._build_spec().loss == "mse"


def test_the_estimator_builds_the_reference_test_definition():
    """tests/gordo/machine/model/test_lstm_autoencoder.py: lstm_hourglass(3, func='tanh', out_func='relu', loss mae)."""
    est = KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=2, n_features=3, func="tanh", out_func="relu",
                               compile_kwargs={"loss": "mae"})
    spec = est._build_spec()
    assert spec.loss == "mae" and spec.out_func == "relu" and spec.units[-1] == 3


def test_a_spec_pickled_before_the_loss_field_loads_as_mse():
    for spec in (ffa.feedforward_hourglass(8), lsa.lstm_hourglass(8)):
        state = dict(spec.__dict__)
        state.pop("loss")  # the attributes a pickle written before this field carries
        old = object.__new__(type(spec))
        old.__dict__.update(state)
        back = pickle.loads(pickle.dumps(old))
        assert "loss" not in back.__dict__ and back.loss == "mse"
    assert FFNetSpec.loss == "mse" and LSTMNetSpec.loss == "mse"


def test_the_loss_does_not_change_the_architecture_key():
    """Engines (and the LSTM fleet's template check) are per architecture; the loss is an argument of each fit."""
    assert ffa.feedforward_hourglass(10, compile_kwargs={"loss": "mae"}).key() == ffa.feedforward_hourglass(10).key()
    assert lsa.lstm_hourglass(10, compile_kwargs={"loss": "huber"}).key() == lsa.lstm_hourglass(10).key()


# ------------------------------------------------------------------------------------------------ bucket keys
def _frame(rows, tags=4):
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(np.random.default_rng(rows).random((rows, tags)), index=idx, columns=[f"tag-{i}" for i in range(tags)])


def _ff_machine(name, loss):
    ae = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2, "batch_size": 32,
                                                          **({"compile_kwargs": {"loss": loss}} if loss else {})}}
    model = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": ae}}
    return {"name": name, "model": model, "dataset": {"X": _frame(300)}}


def _lstm_machine(name, loss):
    est = {"gordo.machine.model.models.KerasLSTMAutoEncoder": {"kind": "lstm_hourglass", "lookback_window": 6, "epochs": 2, "batch_size": 16,
                                                               **({"compile_kwargs": {"loss": loss}} if loss else {})}}
    model = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": est}}
    return {"name": name, "model": model, "dataset": {"X": _frame(200)}}


def _kfold_machine(name, loss):
    ae = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2, "batch_size": 64,
                                                          **({"compile_kwargs": {"loss": loss}} if loss else {})}}
    ttr = {"sklearn.compose.TransformedTargetRegressor": {"transformer": "sklearn.preprocessing.MinMaxScaler", "regressor": ae}}
    model = {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {"base_estimator": ttr, "scaler": "sklearn.preprocessing.MinMaxScaler",
                                                                               "window": 12}}
    return {"name": name, "model": model, "dataset": {"X": _frame(300)},
            "evaluation": {"cv": {"sklearn.model_selection.KFold": {"n_splits": 3}}}}


@pytest.mark.parametrize("make,classify", [(_ff_machine, builder._canonical), (_lstm_machine, builder._canonical_lstm),
                                           (_kfold_machine, builder._canonical_kfcv)], ids=["dense", "lstm", "kfold"])
def test_machines_differing_only_in_loss_get_their_own_buckets(make, classify):
    cs = {loss: classify(i, make(f"m{i}", loss)) for i, loss in enumerate([None, "mse", "mean_squared_error", "mae", "huber", "log_cosh"])}
    assert all(c is not None for c in cs.values())
    assert cs[None].bucket() == cs["mse"].bucket() == cs["mean_squared_error"].bucket()  # the same loss spelled three ways
    keys = {cs[k].bucket() for k in ("mse", "mae", "huber", "log_cosh")}
    assert len(keys) == 4
    assert cs["mae"].spec.loss == "mae"


# ------------------------------------------------------------------------------------------------ C ABI
def test_loss_ids_match_the_header():
    text = open(os.path.join(ROOT, "include", "gordo_b200.h")).read()
    body = re.search(r"typedef enum gb_loss \{(.*?)\} gb_loss;", text, flags=re.S).group(1)
    header = {name: int(v) for name, v in re.findall(r"(GB_LOSS_\w+)\s*=\s*(\d+)", body)}
    assert header == {n: getattr(_cabi, n) for n in header} and len(header) == 6
    assert sorted(_cabi.LOSS_CODES.values()) == list(range(6))
    assert {k: _cabi.loss_code(k) for k in SPELLINGS} == _cabi.LOSS_CODES
    with pytest.raises(ValueError):
        _cabi.loss_code("mean_absolute_error")  # the engine takes canonical names only


def test_fit_hparams_keep_their_layout():
    assert C.sizeof(_cabi.GbFitHParams) == 48
    assert _cabi.GbFitHParams.loss.offset == 44 and _cabi.GbFitHParams.step0.offset == 40
    text = open(os.path.join(ROOT, "include", "gordo_b200.h")).read()
    body = re.search(r"typedef struct gb_fit_hparams \{(.*?)\} gb_fit_hparams;", text, flags=re.S).group(1)
    assert re.search(r"int32_t step0;.*int32_t loss;", body, flags=re.S)
    from gordo_components_b200 import engine

    assert engine._fit_hparams(1, 32, True, None, None, 0, False, 0).loss == 0
    assert engine._fit_hparams(1, 32, True, None, None, 0, False, 0, "log_cosh").loss == 5


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def test_gb_lstm_fit_loss_is_exported(lib):
    assert "gb_lstm_fit_loss" in _cabi.EXPORTS and hasattr(lib, "gb_lstm_fit_loss")


@pytest.mark.parametrize("bad", [-1, 6, 1 << 20])
def test_a_bad_loss_id_is_refused_without_a_gpu(lib, bad):
    """Argument validation runs before anything touches a device, so these return GB_E_ARG on a GPU-less host too."""
    net = _cabi.make_ffnet([4, 3, 4], ["tanh", "linear"])
    hp = _cabi.GbFitHParams(epochs=1, batch_size=8, shuffle=0, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7, loss=bad)
    fake = C.c_void_p(16)  # never dereferenced: validation refuses first
    rc = lib.gb_ffae_fit(C.byref(net), fake, fake, fake, fake, 1, 8, fake, fake, None, C.byref(hp), fake, fake, None)
    assert rc == -1 and b"loss" in lib.gb_last_error()
    rc = lib.gb_ffae_fit_split(C.byref(net), fake, fake, fake, fake, None, 1, 8, fake, fake, None, None, C.byref(hp), 8, fake, fake, None, None, None)
    assert rc == -1 and b"loss" in lib.gb_last_error()
    rc = lib.gb_ffae_fit_stop(C.byref(net), fake, fake, fake, fake, None, 1, 8, fake, fake, None, None, C.byref(hp), 8, fake, fake, None, None,
                              None, None, None, None, None)
    assert rc == -1 and b"loss" in lib.gb_last_error()
    lnet = _cabi.make_lstmnet(4, [3], ["tanh"], 4, "linear", 5)
    lhp = _cabi.GbLstmFitHParams(epochs=1, batch_size=8, lookahead=0, primer=1, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7)
    rc = lib.gb_lstm_fit_loss(C.byref(lnet), fake, fake, fake, fake, fake, 1, 8, fake, fake, C.byref(lhp), fake, fake, fake, bad, None)
    assert rc == -1 and b"loss" in lib.gb_last_error()
    with pytest.raises(ValueError):
        _cabi.check(rc)
