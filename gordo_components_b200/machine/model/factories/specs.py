"""Network specifications produced by the factories and consumed by the CUDA engine."""
from dataclasses import dataclass, field
from typing import Any, Dict, List

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


def _optimizer(optimizer, optimizer_kwargs):
    """Only what the kernels implement is accepted: Adam."""
    if not isinstance(optimizer, str) or optimizer.lower() != "adam":
        raise ValueError(f"optimizer {optimizer!r}: the CUDA fit kernel implements Adam only")
    kw = dict(optimizer_kwargs or {})
    out = {
        "lr": float(kw.pop("learning_rate", kw.pop("lr", 1e-3))),
        "beta1": float(kw.pop("beta_1", 0.9)),
        "beta2": float(kw.pop("beta_2", 0.999)),
        "eps": float(kw.pop("epsilon", 1e-7)),
    }
    if kw:
        raise ValueError(f"unsupported optimizer_kwargs for Adam: {sorted(kw)}")
    return out


@dataclass
class FFNetSpec:
    """Dense stack: ``dims[0]`` inputs, ``dims[l+1]`` units / ``acts[l]`` / ``l1[l]`` activity-L1 of layer l."""

    dims: List[int]
    acts: List[str]
    l1: List[float]
    adam: Dict[str, float] = field(default_factory=lambda: {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7})
    metrics: List[str] = field(default_factory=lambda: ["accuracy"])
    loss: str = "mse"  # canonical name (resolve_loss); a plain default, so a spec pickled before the field existed loads as MSE

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
