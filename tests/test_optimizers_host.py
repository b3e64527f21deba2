"""
Host side of the training optimizers (no GPU): the optimizer oracle against torch.optim in float64; which optimizers and
optimizer_kwargs the factories accept, their defaults and refusals; that a spec pickled before the optimizer fields existed loads as
the same Adam fit; that the fleet builder buckets machines by optimizer while Adam keys stay as they were; and the gb_optimizer
struct, the new exports and their argument checks in the C ABI.
"""
import ctypes as C
import os
import pickle
import re

import numpy as np
import pandas as pd
import pytest

import optimizer_oracle as oo
from gordo_components_b200 import _cabi, builder
from gordo_components_b200.machine.model.factories import feedforward_autoencoder as ffa
from gordo_components_b200.machine.model.factories import lstm_autoencoder as lsa
from gordo_components_b200.machine.model.factories.specs import (OPTIMIZER_DEFAULTS, FFNetSpec, LSTMNetSpec, fit_optimizer,
                                                                  resolve_optimizer)
from gordo_components_b200.machine.model.models import KerasAutoEncoder, KerasLSTMAutoEncoder

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


# ------------------------------------------------------------------------------------------------ the oracle against torch.optim
def _torch_optimizer(torch, name, cfg, params):
    """torch.optim's form of a Keras record: eps outside the root is set to 0 on both sides (see _case)."""
    lr = cfg["lr"]
    if name == "adam":
        return torch.optim.Adam(params, lr=lr, betas=(cfg["beta1"], cfg["beta2"]), eps=0.0)
    if name == "adamw":  # torch's mul_(1 - lr * wd) is Keras' decay
        return torch.optim.AdamW(params, lr=lr, betas=(cfg["beta1"], cfg["beta2"]), eps=0.0, weight_decay=cfg["weight_decay"])
    if name == "rmsprop":  # torch's buffer is Keras' momentum divided by lr
        return torch.optim.RMSprop(params, lr=lr, alpha=cfg["rho"], eps=0.0, momentum=cfg["momentum"], centered=cfg["centered"])
    if name == "adagrad":
        return torch.optim.Adagrad(params, lr=lr, initial_accumulator_value=cfg["initial_accumulator_value"], eps=0.0)
    if name == "adadelta":  # eps inside the roots on both sides
        return torch.optim.Adadelta(params, lr=lr, rho=cfg["rho"], eps=cfg["eps"])
    if name == "adamax":
        return torch.optim.Adamax(params, lr=lr, betas=(cfg["beta1"], cfg["beta2"]), eps=0.0)
    if name == "nadam":  # 0.96^(t psi) with psi = 1 is Keras' 0.96^t
        return torch.optim.NAdam(params, lr=lr, betas=(cfg["beta1"], cfg["beta2"]), eps=0.0, momentum_decay=1.0)
    raise ValueError(name)


CASES = [("adam", {}), ("adamw", {}), ("rmsprop", {}), ("rmsprop", {"momentum": 0.7}), ("rmsprop", {"centered": True}),
         ("adagrad", {}), ("adadelta", {"learning_rate": 1.0}), ("adamax", {}), ("nadam", {})]


def _case(name, kw):
    kw = dict(kw)
    if name != "adadelta":
        kw["epsilon"] = 0.0
    kw.setdefault("learning_rate", 0.01)
    return resolve_optimizer(name, kw)


@pytest.mark.parametrize("steps", [1, 25])
@pytest.mark.parametrize("name,kw", CASES, ids=[f"{n}{'-' + '-'.join(k) if k else ''}" for n, k in CASES])
def test_the_oracle_takes_torch_optims_steps(name, kw, steps):
    torch = pytest.importorskip("torch")
    o = _case(name, kw)
    rng = np.random.default_rng(len(name) + steps)
    w0 = [rng.normal(size=(5, 4)), rng.normal(size=(4,))]
    grads = [[rng.normal(size=a.shape) * (1 + t % 3) for a in w0] for t in range(steps)]
    tp = [torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in w0]
    default = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)  # torch keeps NAdam's product in the default scalar dtype
    try:
        topt = _torch_optimizer(torch, o[0], o[1], tp)
        st = oo.OptState(w0, np.float64)
        w = [a.copy() for a in w0]
        for g in grads:
            for p, gi in zip(tp, g):
                p.grad = torch.tensor(gi, dtype=torch.float64)
            topt.step()
            w = oo.step(o, w, g, st, np.float64)
    finally:
        torch.set_default_dtype(default)
    for a, p in zip(w, tp):
        np.testing.assert_allclose(a, p.detach().numpy(), rtol=1e-10, atol=1e-13)


def test_the_oracle_clips_before_the_decay_and_decays_before_the_rule():
    """clipvalue then weight decay then the rule, as keras' apply: a clipped gradient is the unclipped one at the bound."""
    o = resolve_optimizer("adagrad", {"learning_rate": 0.1, "clipvalue": 0.5, "weight_decay": 0.2})
    w = [np.array([1.0, -2.0, 3.0])]
    g = [np.array([0.1, -3.0, 9.0])]
    got = oo.step(o, w, g, oo.OptState(w, np.float64), np.float64)[0]
    wd = w[0] - w[0] * 0.2 * 0.1
    gc = np.clip(g[0], -0.5, 0.5)
    want = wd - 0.1 * gc / np.sqrt(0.1 + gc * gc + 1e-7)
    np.testing.assert_allclose(got, want, rtol=1e-14)
    late = oo.step(o, w, g, oo.OptState(w, np.float64), np.float64, decay_after=True)[0]
    assert not np.allclose(late, want, rtol=1e-9)


# ------------------------------------------------------------------------------------------------ resolution
@pytest.mark.parametrize("spelling", ["Adam", "adam", "ADAM", "RMSprop", "rmsprop", "Adagrad", "Adadelta", "Adamax", "Nadam", "AdamW"])
def test_every_spelling_resolves(spelling):
    name, cfg = resolve_optimizer(spelling, None)
    assert name == spelling.lower()
    assert {k: cfg[k] for k in OPTIMIZER_DEFAULTS[name]} == OPTIMIZER_DEFAULTS[name]
    assert cfg["clipvalue"] is None and cfg["weight_decay"] == (0.004 if name == "adamw" else 0.0)


def test_keras_defaults():
    assert resolve_optimizer("RMSprop", {})[1] == {"lr": 1e-3, "rho": 0.9, "momentum": 0.0, "eps": 1e-7, "centered": False,
                                                   "weight_decay": 0.0, "clipvalue": None}
    assert resolve_optimizer("Adagrad", {})[1]["initial_accumulator_value"] == 0.1
    assert resolve_optimizer("Adadelta", {})[1]["rho"] == 0.95
    cfg = resolve_optimizer("Nadam", {"learning_rate": 0.02, "beta_1": 0.8, "beta_2": 0.99, "epsilon": 1e-6, "weight_decay": 0.1,
                                      "clipvalue": 2})[1]
    assert cfg == {"lr": 0.02, "beta1": 0.8, "beta2": 0.99, "eps": 1e-6, "weight_decay": 0.1, "clipvalue": 2.0}
    assert resolve_optimizer("rmsprop", {"lr": 0.5})[1]["lr"] == 0.5
    assert resolve_optimizer("Adam", {"learning_rate": 0.2, "lr": 0.5})[1]["lr"] == 0.2  # learning_rate wins, as it always has
    assert resolve_optimizer("Adam", {"amsgrad": False})[0] == "adam"


def test_an_adam_spec_comes_out_as_before():
    keras_adam = {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7}
    for spec in (ffa.feedforward_hourglass(8), ffa.feedforward_hourglass(8, optimizer="adam", optimizer_kwargs={"amsgrad": False}),
                 ffa.feedforward_hourglass(8, optimizer="AdamW", optimizer_kwargs={"weight_decay": None}), lsa.lstm_hourglass(8)):
        assert spec.adam == keras_adam and spec.optimizer == "adam" and spec.optimizer_config is None and fit_optimizer(spec) is None
    spec = ffa.feedforward_hourglass(8, optimizer_kwargs={"learning_rate": 0.01, "beta_1": 0.8})
    assert spec.adam == {"lr": 0.01, "beta1": 0.8, "beta2": 0.999, "eps": 1e-7} and spec.optimizer_config is None


def test_other_optimizers_reach_the_spec():
    spec = lsa.lstm_hourglass(3, optimizer="RMSprop", optimizer_kwargs={"learning_rate": 0.02, "momentum": 0.001})
    assert spec.optimizer == "rmsprop" and spec.optimizer_config["momentum"] == 0.001 and spec.optimizer_config["lr"] == 0.02
    assert fit_optimizer(spec) == ("rmsprop", spec.optimizer_config)
    assert spec.adam == OPTIMIZER_DEFAULTS["adam"]  # read only by the zero-rate held-out pass
    spec = ffa.feedforward_hourglass(8, optimizer="Adam", optimizer_kwargs={"clipvalue": 1.0})
    assert fit_optimizer(spec)[0] == "adam"
    est = KerasAutoEncoder(kind="feedforward_hourglass", n_features=6, optimizer="Nadam", optimizer_kwargs={"learning_rate": 0.01})
    assert est._build_spec().optimizer == "nadam"
    est = KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=3, n_features=6, optimizer="Adagrad")
    assert est._build_spec().optimizer == "adagrad"


REFUSED = [("SGD", {}), ("sgd", {}), ("Ftrl", {}), ("Lion", {}), ("Lamb", {}), ("adam_w", {}), (None, {}), (3, {}),
           ({"class_name": "Adam", "config": {}}, {}), ("Adam", {"amsgrad": True}), ("AdamW", {"amsgrad": True}),
           ("RMSprop", {"centered": True, "momentum": 0.5}), ("Adam", {"clipnorm": 1.0}), ("Adam", {"global_clipnorm": 1.0}),
           ("Nadam", {"use_ema": True}), ("Adam", {"loss_scale_factor": 2.0}), ("Adam", {"gradient_accumulation_steps": 2}),
           ("Adam", {"momentum": 0.9}), ("Adagrad", {"rho": 0.9}), ("Adam", {"nesterov": True}), ("RMSprop", {"beta_1": 0.9}),
           ("Adam", {"learning_rate": {"class_name": "ExponentialDecay", "config": {}}}), ("Adam", {"beta_1": 1.0}),
           ("RMSprop", {"rho": -0.1}), ("Adam", {"learning_rate": -1.0}), ("Adam", {"clipvalue": 0.0})]


@pytest.mark.parametrize("optimizer,kw", REFUSED, ids=[f"{o}-{sorted(k)}" for o, k in REFUSED])
def test_what_the_kernels_cannot_run_is_refused(optimizer, kw):
    with pytest.raises(ValueError):
        resolve_optimizer(optimizer, kw)
    with pytest.raises(ValueError):
        ffa.feedforward_hourglass(10, optimizer=optimizer, optimizer_kwargs=kw)
    with pytest.raises(ValueError):
        lsa.lstm_hourglass(10, optimizer=optimizer, optimizer_kwargs=kw)


def test_an_unknown_optimizer_names_the_supported_set():
    with pytest.raises(ValueError, match="adadelta.*adagrad.*adam.*adamax.*adamw.*nadam.*rmsprop"):
        ffa.feedforward_hourglass(5, optimizer="SGD")


def test_a_spec_pickled_before_the_optimizer_fields_loads_as_adam():
    for spec in (ffa.feedforward_hourglass(8, optimizer_kwargs={"learning_rate": 0.01}), lsa.lstm_hourglass(8)):
        state = dict(spec.__dict__)
        state.pop("optimizer")
        state.pop("optimizer_config")
        old = object.__new__(type(spec))
        old.__dict__.update(state)
        back = pickle.loads(pickle.dumps(old))
        assert "optimizer" not in back.__dict__ and back.optimizer == "adam" and back.optimizer_config is None
        assert fit_optimizer(back) is None and back.adam == spec.adam
    assert FFNetSpec.optimizer == LSTMNetSpec.optimizer == "adam" and FFNetSpec.optimizer_config is None


# ------------------------------------------------------------------------------------------------ bucket keys
def _frame(rows, tags=4):
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(np.random.default_rng(rows).random((rows, tags)), index=idx, columns=[f"tag-{i}" for i in range(tags)])


def _ff_machine(name, optimizer, kw=None):
    ae = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2, "batch_size": 32,
                                                          **({"optimizer": optimizer} if optimizer else {}),
                                                          **({"optimizer_kwargs": kw} if kw else {})}}
    return {"name": name, "model": {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": ae}},
            "dataset": {"X": _frame(300)}}


def _lstm_machine(name, optimizer, kw=None):
    est = {"gordo.machine.model.models.KerasLSTMAutoEncoder": {"kind": "lstm_hourglass", "lookback_window": 6, "epochs": 2, "batch_size": 16,
                                                               **({"optimizer": optimizer} if optimizer else {}),
                                                               **({"optimizer_kwargs": kw} if kw else {})}}
    return {"name": name, "model": {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": est}},
            "dataset": {"X": _frame(200)}}


def _kfold_machine(name, optimizer, kw=None):
    ae = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2, "batch_size": 64,
                                                          **({"optimizer": optimizer} if optimizer else {}),
                                                          **({"optimizer_kwargs": kw} if kw else {})}}
    ttr = {"sklearn.compose.TransformedTargetRegressor": {"transformer": "sklearn.preprocessing.MinMaxScaler", "regressor": ae}}
    model = {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {"base_estimator": ttr, "scaler": "sklearn.preprocessing.MinMaxScaler",
                                                                               "window": 12}}
    return {"name": name, "model": model, "dataset": {"X": _frame(300)}, "evaluation": {"cv": {"sklearn.model_selection.KFold": {"n_splits": 3}}}}


@pytest.mark.parametrize("make,classify", [(_ff_machine, builder._canonical), (_lstm_machine, builder._canonical_lstm),
                                           (_kfold_machine, builder._canonical_kfcv)], ids=["dense", "lstm", "kfold"])
def test_machines_get_a_bucket_per_optimizer(make, classify):
    cases = {"default": (None, None), "Adam": ("Adam", None), "adam": ("adam", {"amsgrad": False}), "RMSprop": ("RMSprop", None),
             "rmsprop": ("rmsprop", {"rho": 0.9}), "rmsprop_fast": ("rmsprop", {"learning_rate": 0.01}), "Nadam": ("Nadam", None),
             "adam_clip": ("Adam", {"clipvalue": 1.0})}
    cs = {k: classify(i, make(f"m{i}", *v)) for i, (k, v) in enumerate(cases.items())}
    assert all(c is not None for c in cs.values())
    assert cs["default"].bucket() == cs["Adam"].bucket() == cs["adam"].bucket()
    assert cs["RMSprop"].bucket() == cs["rmsprop"].bucket()
    keys = {cs[k].bucket() for k in ("default", "RMSprop", "rmsprop_fast", "Nadam", "adam_clip")}
    assert len(keys) == 5
    # a plain Adam machine's key is the key it had before the optimizer fields existed: no optimizer entry at all
    assert not any(isinstance(e, tuple) and e[:1] == ("optimizer",) for e in cs["default"].bucket())


# ------------------------------------------------------------------------------------------------ C ABI
def test_optimizer_ids_and_struct_match_the_header():
    text = open(os.path.join(ROOT, "include", "gordo_b200.h")).read()
    body = re.search(r"typedef enum gb_opt \{(.*?)\} gb_opt;", text, flags=re.S).group(1)
    header = {name: int(v) for name, v in re.findall(r"(GB_OPT_\w+)\s*=\s*(\d+)", body)}
    assert header == {n: getattr(_cabi, n) for n in header} and len(header) == 7
    assert sorted(_cabi.OPT_CODES.values()) == list(range(7)) and set(_cabi.OPT_CODES) == set(OPTIMIZER_DEFAULTS)
    assert int(re.search(r"#define GB_OPT_CENTERED (\d+)", text).group(1)) == _cabi.GB_OPT_CENTERED
    body = re.search(r"typedef struct gb_optimizer \{(.*?)\} gb_optimizer;", text, flags=re.S).group(1)
    fields = re.findall(r"(int32_t|float)\s+(\w+);", body)
    assert [n for _, n in fields] == [n for n, _ in _cabi.GbOptimizer._fields_]
    assert C.sizeof(_cabi.GbOptimizer) == 40
    assert C.sizeof(_cabi.GbFitHParams) == 48 and C.sizeof(_cabi.GbLstmFitHParams) == 32


def test_make_optimizer_maps_the_record():
    o = _cabi.make_optimizer(*resolve_optimizer("RMSprop", {"rho": 0.8, "centered": True, "clipvalue": 0.5}))
    assert (o.kind, o.flags, o.clipvalue, o.weight_decay, o.momentum) == (_cabi.GB_OPT_RMSPROP, _cabi.GB_OPT_CENTERED, 0.5, 0.0, 0.0)
    assert abs(o.beta1 - 0.8) < 1e-7
    o = _cabi.make_optimizer(*resolve_optimizer("Adagrad", {}))
    assert abs(o.initial_accumulator - 0.1) < 1e-8 and o.flags == 0
    o = _cabi.make_optimizer(*resolve_optimizer("AdamW", {}))
    assert o.kind == _cabi.GB_OPT_ADAMW and abs(o.weight_decay - 0.004) < 1e-9
    with pytest.raises(ValueError):
        _cabi.make_optimizer("sgd", {})


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def test_the_optimizer_entry_points_are_exported(lib):
    for name in ("gb_ffae_fit_opt", "gb_lstm_fit_opt", "gb_lstm_fit_tc_opt"):
        assert name in _cabi.EXPORTS and hasattr(lib, name)


BAD = [dict(kind=7), dict(kind=-1), dict(kind=0, flags=2), dict(kind=0, flags=1), dict(kind=2, flags=1, momentum=0.5),
       dict(kind=2, lr=-1.0), dict(kind=0, beta1=1.0), dict(kind=6, beta2=1.5), dict(kind=4, beta1=-0.5), dict(kind=3, eps=-1e-7),
       dict(kind=1, weight_decay=-0.1), dict(kind=5, clipvalue=-1.0), dict(kind=0, lr=float("nan")), dict(kind=0, lr=float("inf"))]


@pytest.mark.parametrize("bad", BAD, ids=[str(b) for b in BAD])
def test_a_bad_optimizer_is_refused_without_a_gpu(lib, bad):
    """Argument validation runs before anything touches a device, so these return GB_E_ARG on a GPU-less host too."""
    o = _cabi.GbOptimizer(kind=0, flags=0, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7)
    for k, v in bad.items():
        setattr(o, k, v)
    net = _cabi.make_ffnet([4, 3, 4], ["tanh", "linear"])
    hp = _cabi.GbFitHParams(epochs=1, batch_size=8, shuffle=0, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7)
    fake = C.c_void_p(16)  # never dereferenced: validation refuses first
    rc = lib.gb_ffae_fit_opt(C.byref(net), fake, fake, fake, fake, None, 1, 8, fake, fake, None, None, C.byref(hp), 8, fake, fake, None, None,
                             None, None, None, None, C.byref(o), None)
    assert rc == -1 and b"optimizer" in lib.gb_last_error()
    lnet = _cabi.make_lstmnet(4, [3], ["tanh"], 4, "linear", 5)
    lhp = _cabi.GbLstmFitHParams(epochs=1, batch_size=8, lookahead=0, primer=1, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7)
    for entry in (lib.gb_lstm_fit_opt, lib.gb_lstm_fit_tc_opt):
        rc = entry(C.byref(lnet), fake, fake, fake, fake, fake, 1, 8, fake, fake, C.byref(lhp), fake, fake, fake, 0, C.byref(o), None)
        assert rc == -1 and b"optimizer" in lib.gb_last_error()
    with pytest.raises(ValueError):
        _cabi.check(rc)
