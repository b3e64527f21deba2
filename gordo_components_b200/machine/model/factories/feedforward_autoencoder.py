"""
Feed-forward autoencoder factories: same names, arguments and validation as
gordo/machine/model/factories/feedforward_autoencoder.py:15-251, returning an ``FFNetSpec``.

Topology (reference :65-104): encoder Dense layers (the first one plain, the following ones with an
l1(10e-5) activity regulariser), decoder Dense layers, then ``Dense(n_features_out, out_func)``;
compiled with Adam / metrics ["accuracy"] and ``compile_kwargs["loss"]``, mean squared error by default (``specs.resolve_loss``).
"""
from typing import Any, Dict, Optional, Tuple

from ..register import register_model_builder
from .specs import FFNetSpec, _check_act, _optimizer, resolve_loss
from .utils import check_dim_func_len, hourglass_calc_dims

__all__ = ["feedforward_model", "feedforward_symmetric", "feedforward_hourglass"]

ACTIVITY_L1 = 10e-5


@register_model_builder(type="KerasAutoEncoder")
def feedforward_model(
    n_features: int,
    n_features_out: Optional[int] = None,
    encoding_dim: Tuple[int, ...] = (256, 128, 64),
    encoding_func: Tuple[str, ...] = ("tanh", "tanh", "tanh"),
    decoding_dim: Tuple[int, ...] = (64, 128, 256),
    decoding_func: Tuple[str, ...] = ("tanh", "tanh", "tanh"),
    out_func: str = "linear",
    optimizer: str = "Adam",
    optimizer_kwargs: Optional[Dict[str, Any]] = None,
    compile_kwargs: Optional[Dict[str, Any]] = None,
    **kwargs,
) -> FFNetSpec:
    n_features_out = n_features_out or n_features
    check_dim_func_len("encoding", encoding_dim, encoding_func)
    check_dim_func_len("decoding", decoding_dim, decoding_func)
    dims = [int(n_features), *map(int, encoding_dim), *map(int, decoding_dim), int(n_features_out)]
    acts = [_check_act(f) for f in (*encoding_func, *decoding_func, out_func)]
    l1 = [0.0 if i == 0 else ACTIVITY_L1 for i in range(len(encoding_dim))] + [0.0] * (len(decoding_dim) + 1)
    metrics = list((compile_kwargs or {}).get("metrics", ["accuracy"]))
    adam, opt, opt_cfg = _optimizer(optimizer, optimizer_kwargs)
    return FFNetSpec(dims, acts, l1, adam, metrics, resolve_loss(compile_kwargs), opt, opt_cfg)


@register_model_builder(type="KerasAutoEncoder")
def feedforward_symmetric(
    n_features: int,
    n_features_out: Optional[int] = None,
    dims: Tuple[int, ...] = (256, 128, 64),
    funcs: Tuple[str, ...] = ("tanh", "tanh", "tanh"),
    optimizer: str = "Adam",
    optimizer_kwargs: Optional[Dict[str, Any]] = None,
    compile_kwargs: Optional[Dict[str, Any]] = None,
    **kwargs,
) -> FFNetSpec:
    if len(dims) == 0:
        raise ValueError("Parameter dims must have len > 0")
    return feedforward_model(
        n_features, n_features_out, encoding_dim=tuple(dims), decoding_dim=tuple(dims)[::-1], encoding_func=tuple(funcs),
        decoding_func=tuple(funcs)[::-1], optimizer=optimizer, optimizer_kwargs=optimizer_kwargs,
        compile_kwargs=compile_kwargs, **kwargs,
    )


@register_model_builder(type="KerasAutoEncoder")
def feedforward_hourglass(
    n_features: int,
    n_features_out: Optional[int] = None,
    encoding_layers: int = 3,
    compression_factor: float = 0.5,
    func: str = "tanh",
    optimizer: str = "Adam",
    optimizer_kwargs: Optional[Dict[str, Any]] = None,
    compile_kwargs: Optional[Dict[str, Any]] = None,
    **kwargs,
) -> FFNetSpec:
    """
    >>> feedforward_hourglass(10).units
    [8, 7, 5, 5, 7, 8, 10]
    >>> feedforward_hourglass(5).units
    [4, 4, 3, 3, 4, 4, 5]
    >>> feedforward_hourglass(10, compression_factor=0.2).units
    [7, 5, 2, 2, 5, 7, 10]
    >>> feedforward_hourglass(10, encoding_layers=1).units
    [5, 5, 10]
    """
    dims = hourglass_calc_dims(compression_factor, encoding_layers, n_features)
    return feedforward_symmetric(
        n_features, n_features_out, dims=dims, funcs=tuple([func] * len(dims)), optimizer=optimizer,
        optimizer_kwargs=optimizer_kwargs, compile_kwargs=compile_kwargs, **kwargs,
    )
