"""
The raw model definitions of ``KerasRawModelRegressor``: ``{"spec": {<Sequential>: {"layers": [...]}}, "compile": {...}}`` (what the
reference hands to ``serializer.from_definition`` and ``model.compile``), translated into the ``FFNetSpec`` of a Dense stack.

Only what the Dense fit and inference kernels run is accepted: a ``Sequential`` of ``Dense`` layers (optionally after one
``Input`` / ``InputLayer``) with bias, the default initialisers, the kernel activations of ``SUPPORTED_ACTIVATIONS``, L1 / L2 / L1L2
kernel and bias regularizers and an L1 activity regularizer, with ``Dropout`` layers between two Dense layers or in front of the
first one.  Everything else is refused with a ValueError naming what is supported.
Regularizer defaults are keras 3.3.3's [3P], restated: ``L1(l1=0.01)``, ``L2(l2=0.01)``, ``L1L2(l1=0.0, l2=0.0)``.

A Dropout's rate becomes ``FFNetSpec.dropout[l]``, the rate on the input of the Dense layer l that follows it; the fit kernel
draws its masks from its own seeded generator (include/gordo_b200.h, gb_dense_dropout), so a Dropout's ``seed`` is taken but
selects nothing.  Prediction runs without dropout, as Keras' does.
"""
import math
from typing import Any, Dict, Optional, Tuple

from ...._cabi import GB_MAX_WIDTH
from .specs import FFNetSpec, _check_act, _optimizer, resolve_loss

__all__ = ["raw_spec", "resolve_regularizer"]

_PREFIXES = ("tensorflow.keras.", "keras.")
_REGULARIZERS = {"L1": ("l1",), "L2": ("l2",), "L1L2": ("l1", "l2")}
_REGULARIZER_DEFAULTS = {"L1": {"l1": 0.01}, "L2": {"l2": 0.01}, "L1L2": {"l1": 0.0, "l2": 0.0}}
_REGULARIZER_NAMES = {"l1": "L1", "l2": "L2", "l1_l2": "L1L2", "L1": "L1", "L2": "L2", "L1L2": "L1L2"}
_DENSE_KEYS = ("units", "activation", "kernel_regularizer", "bias_regularizer", "activity_regularizer", "name", "input_shape",
               "input_dim", "use_bias", "kernel_initializer", "bias_initializer", "kernel_constraint", "bias_constraint")
_DROPOUT_KEYS = ("rate", "noise_shape", "seed", "name", "input_shape")
_COMPILE_IGNORED = ("run_eagerly", "jit_compile", "steps_per_execution")
SUPPORTED = ("a models.Sequential of layers.Dense (units, activation, kernel_regularizer, bias_regularizer, activity_regularizer "
             "with L1 only, name, input_shape / input_dim on the first layer), optionally after one layers.Input / InputLayer; "
             "layers.Dropout (rate, seed, name, input_shape as the first layer) between two Dense layers or before the first one; "
             "regularizers L1, L2, L1L2")


def _name(path: str, module: str) -> Optional[str]:
    """Class name of a Keras path in ``module`` (``tensorflow.keras.layers.Dense``, ``keras.layers.Dense``, ``layers.Dense`` or
    ``Dense``), or None for a path outside it."""
    if not isinstance(path, str):
        return None
    for p in _PREFIXES:
        if path.startswith(p):
            path = path[len(p):]
            break
    mod, _, name = path.rpartition(".")
    return name if mod in ("", module) else None


def _entry(item, what: str) -> Tuple[str, Dict[str, Any]]:
    """(path, kwargs) of a ``{path: kwargs}`` or bare ``path`` definition."""
    if isinstance(item, str):
        return item, {}
    if isinstance(item, dict) and len(item) == 1:
        path, kw = next(iter(item.items()))
        if kw is None:
            kw = {}
        if not isinstance(kw, dict):
            raise ValueError(f"{what} {path!r}: arguments must be a mapping, got {kw!r}")
        return path, dict(kw)
    raise ValueError(f"{what} {item!r} is not a {{path: arguments}} mapping or a path; supported: {SUPPORTED}")


def resolve_regularizer(value, what: str = "regularizer") -> Tuple[float, float]:
    """(l1, l2) of a Keras regularizer definition: None, a name (``"l1"``, ``"l2"``, ``"l1_l2"`` or the class names) or
    ``{...regularizers.L1 | L2 | L1L2: kwargs}``.  Coefficients must be finite and >= 0."""
    if value is None:
        return 0.0, 0.0
    if isinstance(value, str) and value in _REGULARIZER_NAMES:
        cls, kw = _REGULARIZER_NAMES[value], {}
    else:
        path, kw = _entry(value, what)
        name = _name(path, "regularizers")
        cls = _REGULARIZER_NAMES.get(name) if name is not None else None
        if cls is None:
            raise ValueError(f"{what} {path!r} is not supported: the Dense fit kernel implements the regularizers L1, L2 and L1L2")
    unknown = sorted(set(kw) - set(_REGULARIZERS[cls]))
    if unknown:
        raise ValueError(f"{what} {cls}: unsupported arguments {unknown} (it takes {list(_REGULARIZERS[cls])})")
    coef = dict(_REGULARIZER_DEFAULTS[cls], **kw)
    out = []
    for k in ("l1", "l2"):
        v = coef.get(k, 0.0)
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or v < 0:
            raise ValueError(f"{what} {cls}: {k}={v!r} must be a finite float >= 0")
        out.append(float(v))
    return out[0], out[1]


def _input_width(shape, what: str) -> int:
    shape = list(shape) if isinstance(shape, (list, tuple)) else [shape]
    if len(shape) != 1 or isinstance(shape[0], bool) or not isinstance(shape[0], int) or shape[0] < 1:
        raise ValueError(f"{what} {shape!r}: a Dense stack takes one-dimensional rows, [n_features]")
    return int(shape[0])


def _input_layer(name: str, kw: dict) -> int:
    keys = ("shape", "input_shape", "batch_shape", "batch_input_shape")
    unknown = sorted(set(kw) - set(keys) - {"name", "dtype"})
    if unknown or kw.get("dtype") not in (None, "float32"):
        raise ValueError(f"layers.{name}: unsupported arguments {unknown or ['dtype']} (it takes shape and name)")
    given = [k for k in keys if kw.get(k) is not None]
    if len(given) != 1:
        raise ValueError(f"layers.{name} needs exactly one of shape / batch_shape")
    shape = list(kw[given[0]])
    if given[0].startswith("batch"):
        shape = shape[1:]
    return _input_width(shape, f"layers.{name} shape")


def _dense(kw: dict, first: bool, index: int):
    """(units, activation, kernel (l1, l2), bias (l1, l2), activity l1, input width or None) of a Dense layer's arguments."""
    what = f"layer {index} (Dense)"
    unknown = sorted(set(kw) - set(_DENSE_KEYS))
    if unknown:
        raise ValueError(f"{what}: unsupported arguments {unknown}; supported: {SUPPORTED}")
    units = kw.get("units")
    if isinstance(units, bool) or not isinstance(units, int) or not 1 <= units <= GB_MAX_WIDTH:
        raise ValueError(f"{what}: units={units!r} must be an int in [1, {GB_MAX_WIDTH}]")
    if not kw.get("use_bias", True):
        raise ValueError(f"{what}: use_bias=False is not supported, the Dense kernels always add a bias")
    if kw.get("kernel_initializer", "glorot_uniform") not in ("glorot_uniform", "GlorotUniform"):
        raise ValueError(f"{what}: kernel_initializer {kw['kernel_initializer']!r} is not supported (Dense's default glorot_uniform)")
    if kw.get("bias_initializer", "zeros") not in ("zeros", "Zeros"):
        raise ValueError(f"{what}: bias_initializer {kw['bias_initializer']!r} is not supported (Dense's default zeros)")
    for k in ("kernel_constraint", "bias_constraint"):
        if kw.get(k) is not None:
            raise ValueError(f"{what}: {k} is not supported")
    act = kw.get("activation")
    act = _check_act("linear" if act is None else act)
    kernel = resolve_regularizer(kw.get("kernel_regularizer"), f"{what} kernel_regularizer")
    bias = resolve_regularizer(kw.get("bias_regularizer"), f"{what} bias_regularizer")
    activity = resolve_regularizer(kw.get("activity_regularizer"), f"{what} activity_regularizer")
    if activity[1] != 0.0:
        raise ValueError(f"{what}: an L2 activity_regularizer is not supported (the Dense fit kernel implements activity L1 only)")
    width = None
    if kw.get("input_shape") is not None or kw.get("input_dim") is not None:
        if not first:
            raise ValueError(f"{what}: input_shape / input_dim are only taken on the first layer")
        width = _input_width(kw["input_shape"] if kw.get("input_shape") is not None else kw["input_dim"], f"{what} input_shape")
    return units, act, kernel, bias, activity[0], width


def _dropout(kw: dict, first: bool, index: int):
    """(rate, input width or None) of a Dropout layer's arguments."""
    what = f"layer {index} (Dropout)"
    unknown = sorted(set(kw) - set(_DROPOUT_KEYS))
    if unknown:
        raise ValueError(f"{what}: unsupported arguments {unknown}; supported: {SUPPORTED}")
    rate = kw.get("rate")
    if isinstance(rate, bool) or not isinstance(rate, (int, float)) or not math.isfinite(rate) or not 0.0 <= rate < 1.0:
        raise ValueError(f"{what}: rate={rate!r} must be a finite float in [0, 1)")
    if kw.get("noise_shape") is not None:
        raise ValueError(f"{what}: noise_shape is not supported (the fit kernel drops every element independently)")
    seed = kw.get("seed")
    if seed is not None and (isinstance(seed, bool) or not isinstance(seed, int)):
        raise ValueError(f"{what}: seed={seed!r} must be an int or None")
    width = None
    if kw.get("input_shape") is not None:
        if not first:
            raise ValueError(f"{what}: input_shape is only taken on the first layer")
        width = _input_width(kw["input_shape"], f"{what} input_shape")
    return float(rate), width


def raw_spec(kind: dict, n_features: Optional[int], n_features_out: Optional[int] = None) -> FFNetSpec:
    """
    The ``FFNetSpec`` of a raw model definition (``kind["spec"]``, ``kind["compile"]``) for rows of ``n_features`` inputs and
    ``n_features_out`` targets (checked against the spec's input shape and last layer when given).
    """
    spec_def, compile_def = kind["spec"], kind["compile"] or {}
    path, kw = _entry(spec_def, "spec")
    if _name(path, "models") != "Sequential":
        raise ValueError(f"spec {path!r} is not supported: {SUPPORTED}")
    unknown = sorted(set(kw) - {"layers", "name"})
    if unknown:
        raise ValueError(f"models.Sequential: unsupported arguments {unknown} (it takes layers and name)")
    layers = kw.get("layers") or []
    width, dims, acts, l1, dropout = None, [], [], [], []
    reg = {"kernel_l1": [], "kernel_l2": [], "bias_l1": [], "bias_l2": []}
    pending = None  # (index, path, rate) of a Dropout that waits for the Dense layer whose input it drops
    for i, item in enumerate(layers):
        lpath, lkw = _entry(item, f"layer {i}")
        name = _name(lpath, "layers")
        if name in ("Input", "InputLayer"):
            if i != 0:
                raise ValueError(f"layer {i}: layers.{name} must come first")
            width = _input_layer(name, lkw)
            continue
        if name == "Dropout":
            if pending is not None:
                raise ValueError(f"layer {i} {lpath!r} right after the Dropout of layer {pending[0]} is not supported: two Dropout "
                                 f"layers in a row; supported: {SUPPORTED}")
            rate, w = _dropout(lkw, i == 0, i)
            width = w if w is not None else width
            if dims and l1[-1] != 0.0 and rate != 0.0:
                raise ValueError(f"layer {i} {lpath!r} after a Dense layer with an activity_regularizer is not supported: the fit "
                                 f"kernel keeps only the dropped activation; supported: {SUPPORTED}")
            pending = (i, lpath, rate)
            continue
        if name != "Dense":
            raise ValueError(f"layer {i} {lpath!r} is not supported: {SUPPORTED}")
        units, act, kernel, bias, activity, w = _dense(lkw, not dims and width is None, i)
        width = w if w is not None else width
        dims.append(units)
        acts.append(act)
        l1.append(activity)
        dropout.append(0.0 if pending is None else pending[2])
        pending = None
        for k, v in zip(reg, (*kernel, *bias)):
            reg[k].append(v)
    if not dims:
        raise ValueError(f"models.Sequential has no Dense layer: {SUPPORTED}")
    if pending is not None:
        raise ValueError(f"layer {pending[0]} {pending[1]!r} after the last Dense layer is not supported: it would drop the model's "
                         f"output; supported: {SUPPORTED}")
    if width is not None and n_features is not None and width != int(n_features):
        raise ValueError(f"the spec's input shape [{width}] does not match the {int(n_features)} features of X")
    if width is None:
        if n_features is None:
            raise ValueError("the spec has no input shape: fit the model (or pass n_features) to build it")
        width = int(n_features)
    if n_features_out is not None and dims[-1] != int(n_features_out):
        raise ValueError(f"the last Dense layer has {dims[-1]} units, but y has {int(n_features_out)} columns")

    if not isinstance(compile_def, dict):
        raise ValueError(f"compile {compile_def!r} must be a mapping of Model.compile arguments")
    unknown = sorted(set(compile_def) - {"loss", "optimizer", "metrics"} - set(_COMPILE_IGNORED))
    if unknown:
        raise ValueError(f"compile: unsupported arguments {unknown} (supported: loss, optimizer, metrics, and the ignored "
                         f"execution options {list(_COMPILE_IGNORED)})")
    loss = resolve_loss(compile_def)
    opt_def = compile_def.get("optimizer", "rmsprop")  # Model.compile's default
    if isinstance(opt_def, str):
        opt_name, opt_kw = (_name(opt_def, "optimizers") or opt_def), {}
    else:
        opt_path, opt_kw = _entry(opt_def, "compile optimizer")
        opt_name = _name(opt_path, "optimizers") or opt_path
    adam, opt, opt_cfg = _optimizer(opt_name, opt_kw)
    metrics = compile_def.get("metrics") or []
    metrics = [metrics] if isinstance(metrics, str) else list(metrics)
    if metrics not in ([], ["accuracy"]):
        raise ValueError(f"compile metrics {metrics!r}: the fit kernels report accuracy only (metrics: none or ['accuracy'])")
    return FFNetSpec([width, *dims], acts, l1, adam, metrics, loss, opt, opt_cfg, **reg, dropout=dropout if any(dropout) else None)
