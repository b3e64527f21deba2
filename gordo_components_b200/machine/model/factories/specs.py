"""Network specifications produced by the factories and consumed by the CUDA engine."""
from dataclasses import dataclass, field
from typing import Any, Dict, List

SUPPORTED_ACTIVATIONS = ("tanh", "relu", "sigmoid", "linear")


def _check_act(name):
    if name not in SUPPORTED_ACTIVATIONS:
        raise ValueError(f"activation {name!r} is not supported by the CUDA kernels {SUPPORTED_ACTIVATIONS}")
    return name


def _optimizer(optimizer, optimizer_kwargs, compile_kwargs):
    """Only what the kernels implement is accepted: Adam + mean squared error."""
    if not isinstance(optimizer, str) or optimizer.lower() != "adam":
        raise ValueError(f"optimizer {optimizer!r}: the CUDA fit kernel implements Adam only")
    loss = (compile_kwargs or {}).get("loss", "mse")
    if loss not in ("mse", "mean_squared_error"):
        raise ValueError(f"loss {loss!r}: the CUDA fit kernel implements mean squared error only")
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
