"""Network specifications produced by the factories and consumed by the CUDA engine."""
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional

SUPPORTED_ACTIVATIONS = ("tanh", "relu", "sigmoid", "linear")


def _check_act(name):
    if name not in SUPPORTED_ACTIVATIONS:
        raise ValueError(f"activation {name!r} is not supported by the CUDA kernels {SUPPORTED_ACTIVATIONS}")
    return name


# The Keras 3 loss names the fit kernels implement (the spellings keras.losses.get resolves [3P keras 3.3.3]) -> canonical
# name, which is what a spec stores and what engine / _cabi.LOSS_CODES take.  Per-element definitions: include/gordo_b200.h gb_loss.
LOSS_NAMES = {
    **dict.fromkeys(("mse", "MSE", "mean_squared_error", "MeanSquaredError"), "mse"),
    **dict.fromkeys(("mae", "MAE", "mean_absolute_error", "MeanAbsoluteError"), "mae"),
    **dict.fromkeys(("mape", "MAPE", "mean_absolute_percentage_error", "MeanAbsolutePercentageError"), "mape"),
    **dict.fromkeys(("msle", "MSLE", "mean_squared_logarithmic_error", "MeanSquaredLogarithmicError"), "msle"),
    **dict.fromkeys(("huber", "Huber"), "huber"),
    **dict.fromkeys(("log_cosh", "LogCosh"), "log_cosh"),
}


def resolve_loss(compile_kwargs) -> str:
    """
    Canonical name of ``compile_kwargs["loss"]`` (mean squared error when absent, as the reference's factories default it).
    Only names are accepted: a loss object or dict (e.g. a Huber with another delta) and every loss the kernels do not
    implement are refused.
    """
    loss = (compile_kwargs or {}).get("loss", "mse")
    if not isinstance(loss, str) or loss not in LOSS_NAMES:
        raise ValueError(f"loss {loss!r}: the CUDA fit kernels implement the losses {sorted(LOSS_NAMES)}")
    return LOSS_NAMES[loss]


# The Keras 3 optimizers the fit kernels implement (include/gordo_b200.h gb_optimizer; keras 3.3.3 defaults [3P]): lower-cased
# class name -> complete hyperparameter record.  `lr` is the learning rate, `beta1` is also RMSprop's and Adadelta's rho.
OPTIMIZER_DEFAULTS = {
    "adam": {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7},
    "adamw": {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7},
    "rmsprop": {"lr": 1e-3, "rho": 0.9, "momentum": 0.0, "eps": 1e-7, "centered": False},
    "adagrad": {"lr": 1e-3, "initial_accumulator_value": 0.1, "eps": 1e-7},
    "adadelta": {"lr": 1e-3, "rho": 0.95, "eps": 1e-7},
    "adamax": {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7},
    "nadam": {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7},
}
# Keras keyword -> record key, per optimizer (learning_rate / lr, weight_decay and clipvalue are common to all)
_OPT_KWARGS = {
    "adam": {"beta_1": "beta1", "beta_2": "beta2", "epsilon": "eps", "amsgrad": None},
    "adamw": {"beta_1": "beta1", "beta_2": "beta2", "epsilon": "eps", "amsgrad": None},
    "rmsprop": {"rho": "rho", "momentum": "momentum", "epsilon": "eps", "centered": "centered"},
    "adagrad": {"initial_accumulator_value": "initial_accumulator_value", "epsilon": "eps"},
    "adadelta": {"rho": "rho", "epsilon": "eps"},
    "adamax": {"beta_1": "beta1", "beta_2": "beta2", "epsilon": "eps"},
    "nadam": {"beta_1": "beta1", "beta_2": "beta2", "epsilon": "eps"},
}
# Keras optimizer options the kernels cannot honour: a third state slot (amsgrad; RMSprop centered with momentum), a reduction over
# a whole variable before its update (clipnorm, global_clipnorm) or machinery of their own (EMA, loss scaling, accumulation)
_OPT_REFUSED_KWARGS = ("clipnorm", "global_clipnorm", "use_ema", "ema_momentum", "ema_overwrite_frequency", "loss_scale_factor",
                       "gradient_accumulation_steps")


def resolve_optimizer(optimizer, optimizer_kwargs):
    """
    (canonical name, complete hyperparameter record) of a factory's ``optimizer`` / ``optimizer_kwargs``, which the reference
    hands to ``keras.optimizers.get({"class_name": optimizer, "config": optimizer_kwargs})``.  The record holds every key of
    ``OPTIMIZER_DEFAULTS[name]`` plus ``weight_decay`` (0.0 = none; AdamW's default 0.004) and ``clipvalue`` (None = none).
    Names are matched case-insensitively.  Everything the CUDA fit kernels do not implement is refused with a ValueError: other
    optimizers (SGD included), optimizer objects and dicts, learning-rate schedules, the options above and unknown keywords.
    """
    supported = sorted(OPTIMIZER_DEFAULTS)
    if not isinstance(optimizer, str) or optimizer.lower() not in OPTIMIZER_DEFAULTS:
        raise ValueError(f"optimizer {optimizer!r}: the CUDA fit kernels implement the optimizers {supported}")
    name = optimizer.lower()
    kw = dict(optimizer_kwargs or {})
    cfg = dict(OPTIMIZER_DEFAULTS[name], weight_decay=0.004 if name == "adamw" else 0.0, clipvalue=None)
    cfg["lr"] = kw.pop("learning_rate", kw.pop("lr", cfg["lr"]))  # learning_rate wins over the old spelling, as it always has
    refused = sorted(k for k in kw if k in _OPT_REFUSED_KWARGS and kw[k] not in (None, False))
    if refused:
        raise ValueError(f"optimizer_kwargs {refused}: not implemented by the CUDA fit kernels (optimizers {supported} with "
                         "learning_rate, weight_decay, clipvalue and their own Keras keywords)")
    for k in _OPT_REFUSED_KWARGS:
        kw.pop(k, None)
    if "weight_decay" in kw:
        wd = kw.pop("weight_decay")
        cfg["weight_decay"] = 0.0 if wd is None else wd
    if "clipvalue" in kw:
        cfg["clipvalue"] = kw.pop("clipvalue")
    for k in list(kw):
        if k not in _OPT_KWARGS[name]:
            raise ValueError(f"unsupported optimizer_kwargs for {optimizer}: {sorted(kw)}")
        target = _OPT_KWARGS[name][k]
        v = kw.pop(k)
        if target is None:  # amsgrad
            if v:
                raise ValueError("amsgrad=True needs a third optimizer state slot, which the CUDA fit kernels do not have")
            continue
        cfg[target] = v
    if not isinstance(cfg["lr"], (int, float)) or isinstance(cfg["lr"], bool):
        raise ValueError(f"learning_rate {cfg['lr']!r}: the CUDA fit kernels take a constant float learning rate, not a schedule")
    for k, v in cfg.items():
        if k == "centered":
            cfg[k] = bool(v)
        elif not (k == "clipvalue" and v is None):
            cfg[k] = float(v)
    if cfg["lr"] < 0 or cfg["weight_decay"] < 0 or cfg["eps"] < 0 or cfg.get("momentum", 0.0) < 0:
        raise ValueError(f"optimizer {optimizer!r}: negative hyperparameter in {cfg}")
    if cfg["clipvalue"] is not None and not cfg["clipvalue"] > 0:
        raise ValueError(f"clipvalue={cfg['clipvalue']!r} must be > 0")
    for k in ("beta1", "beta2", "rho"):
        if k in cfg and not 0.0 <= cfg[k] < 1.0:
            raise ValueError(f"optimizer {optimizer!r}: {k}={cfg[k]} outside [0, 1)")
    if name == "rmsprop" and cfg["centered"] and cfg["momentum"] > 0:
        raise ValueError("RMSprop with centered=True and momentum > 0 needs a third optimizer state slot, which the CUDA fit kernels "
                         "do not have")
    return name, cfg


def _optimizer(optimizer, optimizer_kwargs):
    """
    (adam, optimizer, optimizer_config) of a factory's arguments: the Adam record every spec carries, and the optimizer when it is
    not plain Adam.  Plain Adam (no weight decay, no clipping) comes out exactly as before the other optimizers existed: its
    hyperparameters in ``adam`` and ``optimizer_config`` None.  For another optimizer, ``adam`` keeps the Keras Adam defaults:
    only the zero-rate held-out pass of the per-epoch fit reads it.
    """
    name, cfg = resolve_optimizer(optimizer, optimizer_kwargs)
    if name in ("adam", "adamw") and cfg["weight_decay"] == 0.0 and cfg["clipvalue"] is None:
        return {k: cfg[k] for k in ("lr", "beta1", "beta2", "eps")}, "adam", None
    return dict(OPTIMIZER_DEFAULTS["adam"]), name, cfg


def fit_optimizer(spec):
    """What the engine's fits take as ``optimizer``: None for plain Adam (``spec.adam``), else (name, record)."""
    cfg = getattr(spec, "optimizer_config", None)
    return None if cfg is None else (spec.optimizer, cfg)


def optimizer_key(spec) -> tuple:
    """A bucket-key suffix that separates machines by optimizer: empty for plain Adam, so that Adam keys are what they were."""
    cfg = getattr(spec, "optimizer_config", None)
    return () if cfg is None else (("optimizer", spec.optimizer, tuple(sorted(cfg.items()))),)


REG_FIELDS = ("kernel_l1", "kernel_l2", "bias_l1", "bias_l2")


def fit_reg(spec):
    """What the engine's Dense fits take as ``reg``: None when the spec has no non-zero weight regularizer, else the per-layer
    coefficients of every field of ``REG_FIELDS`` (zeros where a layer has none)."""
    n = len(spec.dims) - 1
    reg = {k: [float(v) for v in (getattr(spec, k, None) or [0.0] * n)] for k in REG_FIELDS}
    return reg if any(v for vals in reg.values() for v in vals) else None


def reg_key(spec) -> tuple:
    """A bucket-key suffix that separates machines by weight regularizers: empty when there are none, so that other keys are what
    they were."""
    reg = fit_reg(spec)
    return () if reg is None else (("reg", *(tuple(reg[k]) for k in REG_FIELDS)),)


def fit_dropout(spec):
    """What the engine's Dense fits take as ``dropout``: None when the spec has no non-zero Dropout rate, else the per-layer rates
    (``dropout[l]`` on the input of Dense layer l, 0.0 where there is none)."""
    rates = [float(v) for v in (getattr(spec, "dropout", None) or [0.0] * (len(spec.dims) - 1))]
    return rates if any(rates) else None


def dropout_key(spec) -> tuple:
    """A bucket-key suffix that separates machines by Dropout rates: empty when there are none, so that other keys are what they
    were."""
    rates = fit_dropout(spec)
    return () if rates is None else (("dropout", tuple(rates)),)


@dataclass
class FFNetSpec:
    """Dense stack: ``dims[0]`` inputs, ``dims[l+1]`` units / ``acts[l]`` / ``l1[l]`` activity-L1 of layer l.  ``kernel_l1`` ..
    ``bias_l2``: per-layer weight regularizer coefficients (Keras ``kernel_regularizer`` / ``bias_regularizer``), None = none.
    ``dropout``: per-layer Keras Dropout rates, ``dropout[l]`` on the input of layer l (``dropout[0]``: input dropout), None = none."""

    dims: List[int]
    acts: List[str]
    l1: List[float]
    adam: Dict[str, float] = field(default_factory=lambda: {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7})
    metrics: List[str] = field(default_factory=lambda: ["accuracy"])
    loss: str = "mse"  # canonical name (resolve_loss); a plain default, so a spec pickled before the field existed loads as MSE
    # resolve_optimizer's name and record when the fit is not plain Adam; plain defaults, so that a spec pickled before these
    # fields existed loads as the Adam fit of ``adam``
    optimizer: str = "adam"
    optimizer_config: Optional[Dict[str, Any]] = None
    # plain None defaults, so that a spec pickled before these fields existed loads without regularizers
    kernel_l1: Optional[List[float]] = None
    kernel_l2: Optional[List[float]] = None
    bias_l1: Optional[List[float]] = None
    bias_l2: Optional[List[float]] = None
    # likewise: a spec pickled before this field existed loads without dropout
    dropout: Optional[List[float]] = None

    @property
    def n_layers(self):
        return len(self.dims) - 1

    @property
    def units(self):  # what `[layer.units for layer in model.layers]` gives in the reference doctests
        return self.dims[1:]

    @property
    def n_params(self):
        return sum(i * o + o for i, o in zip(self.dims[:-1], self.dims[1:]))

    def key(self):
        return ("ff", tuple(self.dims), tuple(self.acts))


@dataclass
class LSTMNetSpec:
    """LSTM stack (every layer returns sequences except the last) followed by one Dense layer."""

    n_features: int
    lstm_units: List[int]
    acts: List[str]
    n_features_out: int
    out_func: str
    lookback_window: int
    adam: Dict[str, float] = field(default_factory=lambda: {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7})
    metrics: List[str] = field(default_factory=list)
    loss: str = "mse"  # as FFNetSpec.loss
    optimizer: str = "adam"  # as FFNetSpec.optimizer / optimizer_config
    optimizer_config: Optional[Dict[str, Any]] = None

    @property
    def units(self):
        return [*self.lstm_units, self.n_features_out]

    @property
    def n_params(self):
        p, i = 0, self.n_features
        for u in self.lstm_units:
            p += 4 * u * (i + u + 1)
            i = u
        return p + i * self.n_features_out + self.n_features_out

    def key(self):
        return ("lstm", self.n_features, tuple(self.lstm_units), tuple(self.acts), self.n_features_out, self.out_func, self.lookback_window)
