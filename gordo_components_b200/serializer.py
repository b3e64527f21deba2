"""
Model definitions (the YAML/dict form of a machine's ``model:`` block) <-> estimator objects, and the on-disk layout of a
built model.  This is the caller side of the hot path: the reference reaches ``KerasAutoEncoder`` & co. only through
``gordo.serializer`` (gordo/serializer/from_definition.py:23-373, into_definition.py:10-190, serializer.py:18-196), so a
builder that runs where gordo itself is not installed needs the same three things:

* ``from_definition``: a definition is a class path (``"sklearn.preprocessing.MinMaxScaler"``) or a one-key mapping
  ``{class path: kwargs}``; kwargs may themselves hold definitions (``base_estimator``, ``scaler`` ...), Pipelines take
  ``steps`` / FeatureUnions ``transformer_list`` (or a bare list), classes exposing ``from_definition`` build themselves,
  strings that resolve to functions become the functions (``FunctionTransformer.func``), tuple-typed parameters given as
  lists are turned back into tuples.
* ``into_definition``: the inverse, through ``into_definition()`` hooks or ``get_params(deep=False)``.
* ``dump`` / ``load`` / ``load_metadata`` / ``load_info``: ``model.pkl`` + ``metadata.json`` + ``info.json``.

Class paths written for the reference (``gordo.machine.model...``, and the pre-1.0 ``gordo_components.model...``) resolve to
this package's classes, so production configs load unchanged; Keras callback paths resolve to the callbacks of the CUDA fit
loop.
"""
import copy
import importlib
import inspect
import json
import os
import pickle
import typing
from typing import Any, Optional, Union

from sklearn.base import BaseEstimator
from sklearn.pipeline import FeatureUnion, Pipeline

_HERE = __name__.rsplit(".", 1)[0]
_PATH_ALIASES = (
    ("gordo.machine.model.", _HERE + ".machine.model."),
    ("gordo_components.model.", _HERE + ".machine.model."),
)
_CALLBACK_MODULES = ("tensorflow.keras.callbacks", "keras.callbacks", "keras.src.callbacks", "tensorflow.python.keras.callbacks")


def resolve_path(path: str) -> str:
    """The import path this package serves ``path`` from (identity for everything that is not a gordo model path)."""
    for old, new in _PATH_ALIASES:
        if path.startswith(old):
            return new + path[len(old):]
    module, _, name = path.rpartition(".")
    if module in _CALLBACK_MODULES:
        return f"{_HERE}.machine.model.models.{name}"
    return path


def locate(path: Any):
    """Import ``pkg.mod.attr``; ``None`` when ``path`` is not an importable dotted path (plain strings stay plain strings)."""
    if not isinstance(path, str) or "." not in path or any(not part.isidentifier() for part in path.split(".")):
        return None
    module, _, name = resolve_path(path).rpartition(".")
    try:
        return getattr(importlib.import_module(module), name, None)
    except ImportError:
        return None


# ---------------------------------------------------------------------------------------------- definition -> object
def _is_tuple_annotation(tp) -> bool:
    if tp is tuple or typing.get_origin(tp) is tuple:
        return True
    if typing.get_origin(tp) is Union or type(tp).__name__ == "UnionType":
        args = [a for a in typing.get_args(tp) if a is not type(None)]
        return bool(args) and all(a is tuple or typing.get_origin(a) is tuple for a in args)
    return False


def create_instance(factory, **kwargs):
    """``factory(**kwargs)`` with list values turned into tuples where the signature says tuple (YAML has no tuples)."""
    try:
        parameters = inspect.signature(factory).parameters.values()
    except (TypeError, ValueError):
        parameters = ()
    for p in parameters:
        if p.name in kwargs and p.kind in (p.KEYWORD_ONLY, p.POSITIONAL_OR_KEYWORD):
            if isinstance(p.default, tuple) or (p.annotation is not p.empty and _is_tuple_annotation(p.annotation)):
                kwargs[p.name] = tuple(kwargs[p.name])
    return factory(**kwargs)


def _named_steps(definitions):
    return [(f"step_{i}", _build(d)) for i, d in enumerate(definitions)]


def _build(node):
    if isinstance(node, str):
        target = locate(node)
        if hasattr(target, "from_definition"):
            return target.from_definition({})
        return target() if target is not None else node
    if not isinstance(node, dict):
        raise ValueError(f"Expected step to be either a string or a dict, found: {type(node)}")
    if len(node) != 1:
        return _resolve_params(node)

    (path, params), = node.items()
    cls = locate(path)
    if cls is None:
        raise ImportError(f'Could not locate path: "{path}"')
    if params is None:
        params = {}
    if hasattr(cls, "from_definition"):
        return cls.from_definition(params)
    if isinstance(params, dict):
        params = _resolve_params(params)
        for key, value in params.items():
            target = locate(value)
            if callable(target):
                params[key] = target
    if cls in (Pipeline, FeatureUnion):
        if isinstance(params, dict) and "transformer_list" in params:
            params["transformer_list"] = _named_steps(params["transformer_list"])
        elif isinstance(params, dict) and "steps" in params:
            params["steps"] = _named_steps(params["steps"])
        elif isinstance(params, (list, tuple)):
            return cls(_named_steps(params))
        else:
            raise ValueError(f"Got {cls} but the supplied parameters seem invalid: {params}")
    return create_instance(cls, **params)


def _resolve_params(params: dict) -> dict:
    """kwargs whose values are class paths / one-key definitions become objects; everything else is left alone."""
    from .machine.model.models import build_callbacks

    out = dict(params)
    for key, value in params.items():
        if isinstance(value, str):
            target = locate(value)
            if hasattr(target, "from_definition"):
                out[key] = target.from_definition({})
            elif isinstance(target, type) and issubclass(target, BaseEstimator):
                out[key] = target()
        elif isinstance(value, dict) and len(value) == 1 and isinstance(next(iter(value.values())), dict):
            (path, sub), = value.items()
            target = locate(path)
            if hasattr(target, "from_definition"):
                out[key] = target.from_definition(sub)
            elif isinstance(target, type):
                out[key] = _build(value) if issubclass(target, Pipeline) else create_instance(target, **_resolve_params(sub))
        elif key == "callbacks" and isinstance(value, list):
            out[key] = build_callbacks(value)
    return out


def from_definition(definition: Union[str, dict]):
    """Build the estimator (Pipeline, detector, bare model ...) a ``model:`` block describes.  The input is not modified."""
    return _build(copy.deepcopy(definition))


def load_params_from_definition(definition: dict) -> dict:
    """Resolve every value of a kwargs mapping (gordo/serializer/from_definition.py:322-334)."""
    if not isinstance(definition, dict):
        raise ValueError(f"Expected definition to be a dict, found: {type(definition)}")
    return _resolve_params(definition)


# ---------------------------------------------------------------------------------------------- object -> definition
def _has_hook(obj, name) -> bool:
    # looked up on the class: the detectors forward unknown attributes to their base estimator, whose hook is not theirs
    return hasattr(type(obj), name)


def _value_definition(value, tuples_to_list):
    if _has_hook(value, "get_params") or _has_hook(value, "into_definition"):
        return _node_definition(value, False, tuples_to_list)
    if isinstance(value, list):
        return [_node_definition(v[1], False, tuples_to_list) if isinstance(v, tuple) else v for v in value]
    if isinstance(value, tuple) and tuples_to_list:
        return list(value)
    if callable(value):
        return f"{value.__module__}.{value.__name__}"
    return value


def _node_definition(obj, prune_default_params, tuples_to_list):
    path = f"{type(obj).__module__}.{type(obj).__name__}"
    if _has_hook(obj, "into_definition"):
        return {path: obj.into_definition()}
    params = obj.get_params(deep=False)
    if prune_default_params:
        defaults = {k: p.default for k, p in inspect.signature(type(obj).__init__).parameters.items() if p.default is not p.empty}
        params = {k: v for k, v in params.items() if not (k in defaults and _same(defaults[k], v))}
    return {path: {k: _value_definition(v, tuples_to_list) for k, v in params.items()}}


def _same(a, b) -> bool:
    try:
        return bool(a == b) or (a is b)
    except Exception:
        return False


def into_definition(pipeline, prune_default_params: bool = False, tuples_to_list: bool = True) -> dict:
    """The definition ``from_definition`` rebuilds ``pipeline`` from: plain dicts, lists, strings and numbers only."""
    return _node_definition(pipeline, prune_default_params, tuples_to_list)


def load_definition_from_params(params: dict, tuples_to_list: bool = True) -> dict:
    return {k: _value_definition(v, tuples_to_list) for k, v in params.items()}


# ---------------------------------------------------------------------------------------------- bytes and directories
def dumps(model) -> bytes:
    return pickle.dumps(model)


def loads(data: bytes):
    return pickle.loads(data)


def _find_json(source_dir, name) -> Optional[str]:
    for candidate in (os.path.join(source_dir, name), os.path.join(source_dir, "..", name)):
        if os.path.exists(candidate):
            return candidate
    return None


def metadata_path(source_dir) -> Optional[str]:
    return _find_json(source_dir, "metadata.json")


def _load_json(source_dir, name) -> dict:
    path = _find_json(source_dir, name)
    if path is None:
        raise FileNotFoundError(f"'{name}' file not found in '{source_dir}'")
    with open(path, "r") as f:
        return json.load(f)


def load_metadata(source_dir) -> dict:
    """``metadata.json`` from ``source_dir`` or its parent (serializer.py:95-115)."""
    return _load_json(source_dir, "metadata.json")


def load_info(source_dir) -> dict:
    return _load_json(source_dir, "info.json")


def load(source_dir) -> Any:
    with open(os.path.join(source_dir, "model.pkl"), "rb") as f:
        return pickle.load(f)


def dump(obj, dest_dir, metadata: Optional[dict] = None, info: Optional[dict] = None) -> None:
    """``model.pkl`` (+ ``metadata.json``, ``info.json`` when given) under ``dest_dir``: what gordo.server loads (serializer.py:149-196)."""
    os.makedirs(dest_dir, exist_ok=True)
    with open(os.path.join(dest_dir, "model.pkl"), "wb") as f:
        pickle.dump(obj, f)
    if info is not None:
        with open(os.path.join(dest_dir, "info.json"), "w") as f:
            json.dump(info, f, default=str)
    if metadata is not None:
        with open(os.path.join(dest_dir, "metadata.json"), "w") as f:
            json.dump(metadata, f, default=str)
