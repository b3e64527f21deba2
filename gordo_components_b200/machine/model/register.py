"""
Factory registry ``{type: {kind: function}}`` (mirror of gordo/machine/model/register.py:10-75).

A registered factory takes ``n_features`` (plus keyword arguments from the model definition)
and returns a network *specification* (``factories.specs.FFNetSpec`` / ``LSTMNetSpec``) -- the
CUDA engine compiles nothing per model, so there is no framework graph object to build.
"""
import inspect
from typing import Callable, Dict


class register_model_builder:
    factories: Dict[str, Dict[str, Callable]] = dict()

    def __init__(self, type: str):
        self.type = type

    def __call__(self, build_fn: Callable):
        self._register(self.type, build_fn)
        return build_fn

    @classmethod
    def _register(cls, type: str, build_fn: Callable):
        cls._validate_func(build_fn)
        cls.factories.setdefault(type, dict())[build_fn.__name__] = build_fn

    @staticmethod
    def _validate_func(func):
        if "n_features" not in inspect.getfullargspec(func).args:
            raise ValueError(f"Build function: {func.__name__} does not have 'n_features' as an argument; it should.")
