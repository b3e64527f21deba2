"""
LSTM autoencoder factories: same names, arguments and validation as
gordo/machine/model/factories/lstm_autoencoder.py:15-263, returning an ``LSTMNetSpec``.
Registered for both wrapper types, like the reference (:15-16, :106-107, :177-178).
"""
from typing import Any, Dict, Optional, Tuple

from ..register import register_model_builder
from .specs import LSTMNetSpec, _check_act, _optimizer, resolve_loss
from .utils import check_dim_func_len, hourglass_calc_dims

__all__ = ["lstm_model", "lstm_symmetric", "lstm_hourglass"]


@register_model_builder(type="KerasLSTMAutoEncoder")
@register_model_builder(type="KerasLSTMForecast")
def lstm_model(
    n_features: int,
    n_features_out: Optional[int] = None,
    lookback_window: int = 1,
    encoding_dim: Tuple[int, ...] = (256, 128, 64),
    encoding_func: Tuple[str, ...] = ("tanh", "tanh", "tanh"),
    decoding_dim: Tuple[int, ...] = (64, 128, 256),
    decoding_func: Tuple[str, ...] = ("tanh", "tanh", "tanh"),
    out_func: str = "linear",
    optimizer: str = "Adam",
    optimizer_kwargs: Optional[Dict[str, Any]] = None,
    compile_kwargs: Optional[Dict[str, Any]] = None,
    **kwargs,
) -> LSTMNetSpec:
    n_features_out = n_features_out or n_features
    check_dim_func_len("encoding", encoding_dim, encoding_func)
    check_dim_func_len("decoding", decoding_dim, decoding_func)
    units = [*map(int, encoding_dim), *map(int, decoding_dim)]
    acts = [_check_act(f) for f in (*encoding_func, *decoding_func)]
    adam, opt, opt_cfg = _optimizer(optimizer, optimizer_kwargs)
    return LSTMNetSpec(int(n_features), units, acts, int(n_features_out), _check_act(out_func), int(lookback_window),
                       adam, list((compile_kwargs or {}).get("metrics", [])), resolve_loss(compile_kwargs), opt, opt_cfg)


@register_model_builder(type="KerasLSTMAutoEncoder")
@register_model_builder(type="KerasLSTMForecast")
def lstm_symmetric(
    n_features: int,
    n_features_out: Optional[int] = None,
    lookback_window: int = 1,
    dims: Tuple[int, ...] = (256, 128, 64),
    funcs: Tuple[str, ...] = ("tanh", "tanh", "tanh"),
    out_func: str = "linear",
    optimizer: str = "Adam",
    optimizer_kwargs: Optional[Dict[str, Any]] = None,
    compile_kwargs: Optional[Dict[str, Any]] = None,
    **kwargs,
) -> LSTMNetSpec:
    if len(dims) == 0:
        raise ValueError("Parameter dims must have len > 0")
    return lstm_model(
        n_features=n_features, n_features_out=n_features_out, lookback_window=lookback_window, encoding_dim=tuple(dims),
        decoding_dim=tuple(dims)[::-1], encoding_func=tuple(funcs), decoding_func=tuple(funcs)[::-1], out_func=out_func,
        optimizer=optimizer, optimizer_kwargs=optimizer_kwargs, compile_kwargs=compile_kwargs, **kwargs,
    )


@register_model_builder(type="KerasLSTMAutoEncoder")
@register_model_builder(type="KerasLSTMForecast")
def lstm_hourglass(
    n_features: int,
    n_features_out: Optional[int] = None,
    lookback_window: int = 1,
    encoding_layers: int = 3,
    compression_factor: float = 0.5,
    func: str = "tanh",
    out_func: str = "linear",
    optimizer: str = "Adam",
    optimizer_kwargs: Optional[Dict[str, Any]] = None,
    compile_kwargs: Optional[Dict[str, Any]] = None,
    **kwargs,
) -> LSTMNetSpec:
    """
    >>> lstm_hourglass(10).units
    [8, 7, 5, 5, 7, 8, 10]
    >>> lstm_hourglass(10, compression_factor=0.2).units
    [7, 5, 2, 2, 5, 7, 10]
    """
    dims = hourglass_calc_dims(compression_factor, encoding_layers, n_features)
    return lstm_symmetric(
        n_features=n_features, n_features_out=n_features_out, lookback_window=lookback_window, dims=dims,
        funcs=tuple([func] * len(dims)), out_func=out_func, optimizer=optimizer, optimizer_kwargs=optimizer_kwargs,
        compile_kwargs=compile_kwargs, **kwargs,
    )
