"""
sklearn-style model wrappers with the public surface of gordo/machine/model/models.py
(KerasBaseEstimator :36-357, KerasAutoEncoder :360-398, KerasRawModelRegressor :401-460, KerasLSTMBaseEstimator :463-698,
KerasLSTMForecast :701-704, KerasLSTMAutoEncoder :707-710, create_keras_timeseriesgenerator :713-793)
-- same class names, constructor arguments, methods, return types and exceptions -- whose fit and
predict run as CUDA kernels on an H100 through ``gordo_components_b200.engine``.

The class names keep their "Keras" prefix on purpose: gordo model definitions, the factory registry
(``register_model_builder.factories["KerasAutoEncoder"]``) and stored metadata key on them.  There is no
Keras, TensorFlow or scikeras underneath, and no CPU fallback.
"""
from __future__ import annotations

import abc
import importlib
import logging
import math
from copy import copy, deepcopy
from importlib.util import find_spec
from pprint import pformat
from typing import Any, Callable, Dict, Optional, Tuple, Union

import numpy as np
import pandas as pd
from sklearn.base import BaseEstimator, TransformerMixin
from sklearn.exceptions import NotFittedError
from sklearn.metrics import explained_variance_score

from .base import GordoBase
from .factories import *  # noqa: F401,F403  -- executes the @register_model_builder decorators
from .factories.raw import raw_spec
from .factories.specs import FFNetSpec, LSTMNetSpec, fit_dropout, fit_optimizer, fit_reg
from .register import register_model_builder

logger = logging.getLogger(__name__)


class History:
    """What keras leaves in ``model.history``: per-epoch metric lists, the fit params and the epoch index."""

    def __init__(self, history=None, params=None, epoch=None):
        self.history = history or {}
        self.params = params or {}
        self.epoch = epoch or []


class FittedNet:
    """A trained network: its specification plus host copies of the weights (what gets pickled)."""

    def __init__(self, spec, weights):
        self.spec = spec
        self.weights = weights
        self.history: Optional[History] = None

    @property
    def layers(self):
        return self.spec.units

    def get_weights(self):
        return self.weights


def _glorot_uniform(fan_in: int, fan_out: int) -> np.ndarray:
    limit = math.sqrt(6.0 / (fan_in + fan_out))
    return np.random.uniform(-limit, limit, size=(fan_in, fan_out)).astype(np.float32)


def _orthogonal(rows: int, cols: int) -> np.ndarray:
    a = np.random.standard_normal((max(rows, cols), min(rows, cols)))
    q, r = np.linalg.qr(a)
    q = q * np.sign(np.diag(r))
    if rows < cols:
        q = q.T
    return q[:rows, :cols].astype(np.float32)


def _as_2d_values(a):
    a = getattr(a, "values", a)
    return np.asarray(a)


class EarlyStopping:
    """
    The one Keras callback gordo's model definitions use (``tensorflow.keras.callbacks.EarlyStopping``: monitor, min_delta,
    patience, mode, baseline, restore_best_weights, start_from_epoch), restated from keras 3.3.3 [3P]
    ``keras/src/callbacks/early_stopping.py`` -- epochs are kernel launches here, so the callback is host-side bookkeeping
    between them.  ``update(epoch, logs, get_weights)`` returns True when training must stop.
    """

    def __init__(self, monitor="val_loss", min_delta=0, patience=0, verbose=0, mode="auto", baseline=None, restore_best_weights=False,
                 start_from_epoch=0):
        self.monitor, self.patience, self.verbose, self.baseline = monitor, int(patience), verbose, baseline
        self.min_delta = abs(float(min_delta))
        self.restore_best_weights, self.start_from_epoch = bool(restore_best_weights), int(start_from_epoch)
        if mode not in ("auto", "min", "max"):
            mode = "auto"
        if mode == "auto":  # keras: accuracy-like metrics are maximised, everything else minimised
            mode = "max" if any(k in monitor for k in ("acc", "accuracy", "auc")) else "min"
        self.mode = mode
        self.reset()

    def reset(self):
        self.wait, self.stopped_epoch, self.best_epoch = 0, 0, 0
        self.best = float("inf") if self.mode == "min" else -float("inf")
        self.best_weights = None

    def _is_improvement(self, value, reference):
        return value + self.min_delta < reference if self.mode == "min" else value - self.min_delta > reference

    def update(self, epoch: int, logs: Dict[str, float], get_weights: Callable) -> bool:
        current = logs.get(self.monitor)
        if current is None or epoch < self.start_from_epoch:
            if current is None:
                logger.warning("Early stopping conditioned on metric `%s` which is not available. Available metrics are: %s",
                               self.monitor, ",".join(logs))
            return False
        if self.restore_best_weights and self.best_weights is None:
            self.best_weights, self.best_epoch = get_weights(), epoch
        self.wait += 1
        if self._is_improvement(current, self.best):
            self.best, self.best_epoch = current, epoch
            if self.restore_best_weights:
                self.best_weights = get_weights()
            if self.baseline is None or self._is_improvement(current, self.baseline):
                self.wait = 0
            return False
        if self.wait >= self.patience and epoch > 0:
            self.stopped_epoch = epoch
            return True
        return False


def build_callbacks(definitions) -> list:
    """
    ``callbacks`` of a model definition -- ``[{"tensorflow.keras.callbacks.EarlyStopping": {...}}]`` as gordo's serializer
    receives them (gordo/serializer/from_definition.py:337-372) or already-built objects -- to the callbacks this fit loop
    understands.  Anything but EarlyStopping is reported and skipped.
    """
    out = []
    for cb in definitions or []:
        if isinstance(cb, EarlyStopping):
            out.append(cb)
        elif isinstance(cb, dict) and len(cb) == 1 and str(next(iter(cb))).split(".")[-1] == "EarlyStopping":
            out.append(EarlyStopping(**(next(iter(cb.values())) or {})))
        elif isinstance(cb, str) and cb.split(".")[-1] == "EarlyStopping":
            out.append(EarlyStopping())
        elif type(cb).__name__ == "EarlyStopping":  # a real keras object handed over by the caller
            out.append(EarlyStopping(**{k: getattr(cb, k) for k in ("monitor", "min_delta", "patience", "baseline", "restore_best_weights",
                                                                    "start_from_epoch") if hasattr(cb, k)}))
        else:
            logger.warning("callback %s is not supported by the CUDA fit loop and is ignored", cb)
    return out


class KerasBaseEstimator(BaseEstimator, GordoBase):
    # keyword arguments of the model definition that steer fitting rather than the architecture
    supported_fit_args = [
        "batch_size", "epochs", "verbose", "callbacks", "validation_split", "shuffle", "class_weight", "initial_epoch",
        "steps_per_epoch", "validation_batch_size", "max_queue_size", "workers", "use_multiprocessing",
    ]

    def __init__(self, kind: Union[str, Callable], **kwargs) -> None:
        """
        ``kind`` names a registered factory for this class (``feedforward_hourglass`` ...), a dotted path to a
        factory function, or is the factory function itself (it must take ``n_features``).  Every other keyword
        goes to the factory and/or steers ``fit`` (``epochs``, ``batch_size``, ``validation_split``, ``shuffle``).
        """
        self.kind = self.load_kind(kind)
        self.kwargs: Dict[str, Any] = kwargs
        self._history: Optional[History] = None
        self.model: Optional[FittedNet] = None

    # ------------------------------------------------------------------ definition <-> object
    @staticmethod
    def parse_module_path(module_path) -> Tuple[Optional[str], str]:
        parts = module_path.split(".")
        return (None, parts[0]) if len(parts) == 1 else (".".join(parts[:-1]), parts[-1])

    def load_kind(self, kind):
        if callable(kind):
            register_model_builder(type=self.__class__.__name__)(kind)
            return kind.__name__
        module_name, name = self.parse_module_path(kind)
        if module_name is None:
            if name not in register_model_builder.factories.get(self.__class__.__name__, {}):
                raise ValueError(f"kind: {kind} is not an available model for type: {self.__class__.__name__}!")
        else:
            try:
                found = find_spec(module_name) is not None
            except ModuleNotFoundError:
                found = False
            if not found:
                raise ValueError(f"kind: {kind}, unable to find module: '{module_name}'")
        return kind

    @classmethod
    def extract_supported_fit_args(cls, kwargs):
        return {k: kwargs[k] for k in cls.supported_fit_args if k in kwargs}

    @classmethod
    def from_definition(cls, definition: dict):
        """Hook used by gordo.serializer.from_definition (gordo/serializer/from_definition.py:190-191)."""
        definition = copy(definition)
        kind = definition.pop("kind")
        return cls(kind, **definition)

    def into_definition(self) -> dict:
        """Hook used by gordo.serializer.into_definition (gordo/serializer/into_definition.py:92-93)."""
        definition = copy(self.kwargs)
        definition["kind"] = self.kind
        return definition

    @property
    def sk_params(self):
        return self.kwargs

    def get_params(self, **params):
        out = {"kind": self.kind}
        out.update(self.kwargs)
        return out

    def set_params(self, **params):
        if "kind" in params:
            self.kind = self.load_kind(params.pop("kind"))
        self.kwargs.update(params)
        return self

    def __sklearn_clone__(self):
        return self.__class__(self.kind, **deepcopy(self.kwargs))

    def __sklearn_is_fitted__(self) -> bool:
        # no trailing-underscore attributes here: tell sklearn (Pipeline.predict checks its last step) what "fitted" means
        return self.model is not None

    # ------------------------------------------------------------------ pickling: plain numpy state, no device handles
    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop("_dev_cache", None)
        return state

    def __setstate__(self, state):
        self.__dict__.update(state)

    # ------------------------------------------------------------------ shapes
    @staticmethod
    def get_n_features_out(y) -> Union[int, tuple]:
        if len(y.shape) == 1:
            raise ValueError("Unsupported number of the output dataset dimensions %d" % len(y.shape))
        return y.shape[1] if len(y.shape) == 2 else y.shape[1:]

    @staticmethod
    def get_n_features(X) -> Union[int, tuple]:
        if len(X.shape) == 1:
            raise ValueError("Unsupported number of the output dataset dimensions %d" % len(X.shape))
        return X.shape[1] if len(X.shape) == 2 else X.shape[2]

    # ------------------------------------------------------------------ model construction
    def _factory(self):
        module_name, name = self.parse_module_path(self.kind)
        if module_name is None:
            return register_model_builder.factories[self.__class__.__name__][self.kind]
        module = importlib.import_module(module_name)
        if not hasattr(module, name):
            raise ValueError("kind: %s, unable to find class %s in module '%s'" % (self.kind, name, module_name))
        return getattr(module, name)

    def _build_spec(self):
        spec = self._factory()(**self.sk_params)
        if not isinstance(spec, (FFNetSpec, LSTMNetSpec)):
            raise ValueError(
                f"factory {self.kind!r} returned {type(spec).__name__}; factories must return an FFNetSpec or LSTMNetSpec"
            )
        return spec

    def _initial_weights(self, spec):
        """Keras initialisers [3P]: Dense/LSTM kernels glorot_uniform, recurrent kernels orthogonal, biases zero (forget gate 1)."""
        if isinstance(spec, FFNetSpec):
            return [(_glorot_uniform(i, o), np.zeros(o, np.float32)) for i, o in zip(spec.dims[:-1], spec.dims[1:])]
        layers, i = [], spec.n_features
        for u in spec.lstm_units:
            b = np.zeros(4 * u, np.float32)
            b[u : 2 * u] = 1.0
            layers.append((_glorot_uniform(i, 4 * u), _orthogonal(u, 4 * u), b))
            i = u
        return layers, (_glorot_uniform(i, spec.n_features_out), np.zeros(spec.n_features_out, np.float32))

    def _prepare_model(self):
        spec = self._build_spec()
        self.model = FittedNet(spec, self._initial_weights(spec))

    def set_weights(self, weights):
        """Install trained weights (Keras order: per Dense layer (kernel [in,out], bias [out]))."""
        if self.model is None:
            if "n_features" not in self.kwargs:
                raise NotFittedError("set_weights needs n_features: pass it in kwargs or call fit first")
            self._prepare_model()
        self.model.weights = weights
        self.__dict__.pop("_dev_cache", None)
        return self

    # ------------------------------------------------------------------ device plumbing
    def _engine(self):
        from ... import engine

        return engine.ff_engine_for(self.model.spec)

    def _device_params(self):
        cache = self.__dict__.get("_dev_cache")
        if cache is None or cache[0] is not self.model.weights:
            eng = self._engine()
            cache = (self.model.weights, eng.pack_params([self.model.weights]))
            self.__dict__["_dev_cache"] = cache
        return cache[1]

    # ------------------------------------------------------------------ fit / predict
    def fit(self, X, y, **kwargs):
        """
        Train on ``X`` -> ``y`` (numpy arrays or DataFrames).  Keyword arguments override the fit arguments given
        at construction (``epochs``, ``batch_size``, ``shuffle``, ``validation_split``).
        """
        from ... import engine

        if isinstance(y, np.ndarray) and y.ndim == 1:
            y = y.reshape(-1, 1)
        self.kwargs.update({"n_features": self.get_n_features(X), "n_features_out": self.get_n_features_out(y)})
        X, y = _as_2d_values(X), _as_2d_values(y)
        if self.model is None:
            self._prepare_model()
        spec = self.model.spec
        optimizer = fit_optimizer(spec)  # None: Adam from spec.adam
        reg = fit_reg(spec)  # None: no weight regularizers
        dropout = fit_dropout(spec)  # None: no Dropout layers
        if spec.dims[0] != X.shape[1] or spec.dims[-1] != y.shape[1]:
            raise ValueError(f"model was built for {spec.dims[0]}->{spec.dims[-1]} features, got X {X.shape} y {y.shape}")
        fit_args = {**self.extract_supported_fit_args(self.kwargs), **kwargs}
        epochs = int(fit_args.get("epochs", 1))
        batch_size = int(fit_args.get("batch_size") or 32)
        shuffle = bool(fit_args.get("shuffle", True))
        vsplit = float(fit_args.get("validation_split") or 0.0)
        callbacks = build_callbacks(fit_args.get("callbacks"))
        for cb in callbacks:
            cb.reset()
        n_train = len(X)
        if 0.0 < vsplit < 1.0:  # keras holds out the *tail* before shuffling
            n_train = int(math.floor(len(X) * (1.0 - vsplit)))
        if n_train < 1:
            raise ValueError("no training rows")

        eng = engine.ff_engine_for(spec)
        dev = eng.device
        xd, yd = engine.to_device_f32(X, dev), engine.to_device_f32(y, dev)
        params = eng.pack_params([self.model.weights])
        jobs = engine.jobs_to_device(engine.make_jobs([0], [n_train], [0]), dev)
        seed = int(np.random.randint(0, 2**31 - 1))  # follows numpy's global seed, like gordo's builder set_seed
        history: Dict[str, list] = {"loss": []}
        if "accuracy" in spec.metrics:
            history["accuracy"] = []
        n_val = len(X) - n_train
        if n_val or callbacks:
            # one launch per epoch: the validation loss and the callbacks live between epochs
            if n_val:
                history["val_loss"] = []
                if "accuracy" in history:
                    history["val_accuracy"] = []
                vjobs = engine.jobs_to_device(engine.make_jobs([0], [n_val], [n_train]), dev)
                vbatch = int(fit_args.get("validation_batch_size") or batch_size)
            state, step0 = None, 0
            steps = int(math.ceil(n_train / batch_size))
            frozen = dict(spec.adam, lr=0.0)  # an Adam pass at lr 0 whatever the fit's optimizer: it moves nothing
            for e in range(epochs):
                loss, acc, state = eng.fit(params, jobs, 1, n_train, xd, yd, epochs=1, batch_size=batch_size, shuffle=shuffle,
                                           adam=spec.adam, seed=seed + e, state=state, step0=step0, loss=spec.loss, optimizer=optimizer,
                                           reg=reg, dropout=dropout)
                step0 += steps
                logs = {"loss": float(loss[0, 0])}
                if "accuracy" in history:
                    logs["accuracy"] = float(acc[0, 0])
                if n_val:
                    # keras evaluates the *total* loss (the compiled loss + activity and weight regularisation) on the held-out tail in
                    # batches: the fit kernel with a zero learning rate on a throw-away optimizer state computes exactly that and moves nothing
                    # (and, without ``dropout``, runs the network as Keras' evaluation does, undropped)
                    vl, va, _ = eng.fit(params, vjobs, 1, n_val, xd, yd, epochs=1, batch_size=vbatch, shuffle=False, adam=frozen, loss=spec.loss,
                                        reg=reg)
                    logs["val_loss"] = float(vl[0, 0])
                    if "accuracy" in history:
                        logs["val_accuracy"] = float(va[0, 0])
                for k, v in logs.items():
                    history[k].append(v)
                if any([cb.update(e, logs, lambda: params.clone()) for cb in callbacks]):
                    break
            for cb in callbacks:  # keras restores at train end whether or not training stopped early
                if cb.restore_best_weights and cb.best_weights is not None:
                    params = cb.best_weights
            epochs_run = len(history["loss"])
        else:
            loss, acc, _ = eng.fit(params, jobs, 1, n_train, xd, yd, epochs=epochs, batch_size=batch_size, shuffle=shuffle,
                                   adam=spec.adam, seed=seed, loss=spec.loss, optimizer=optimizer, reg=reg, dropout=dropout)
            history["loss"] = [float(v) for v in loss[0].cpu().numpy()]
            if "accuracy" in history:
                history["accuracy"] = [float(v) for v in acc[0].cpu().numpy()]
            epochs_run = epochs
        self.model.weights = eng.unpack_params(params)[0]
        self.__dict__["_dev_cache"] = (self.model.weights, params)
        self._history = History(history, {"verbose": 0, "epochs": epochs, "steps": int(math.ceil(n_train / batch_size))}, list(range(epochs_run)))
        self.model.history = self._history
        return self

    def predict(self, X, **kwargs) -> np.ndarray:
        """Model output for every row of ``X`` as a float32 array ``[len(X), n_features_out]``."""
        from ... import engine

        if self.model is None:
            raise NotFittedError(f"This {self.__class__.__name__} has not been fitted yet.")
        X = _as_2d_values(X)
        if X.ndim != 2 or X.shape[1] != self.model.spec.dims[0]:
            raise ValueError(f"X has shape {X.shape}; the model expects [n, {self.model.spec.dims[0]}]")
        eng = self._engine()
        if len(X) == 0:
            return np.empty((0, eng.n_out), np.float32)
        xd = engine.to_device_f32(X, eng.device)
        jobs = engine.jobs_to_device(engine.make_jobs([0], [len(X)], [0]), eng.device)
        res = eng.infer_score(self._device_params(), jobs, 1, len(X), xd)
        return res["model-output"].cpu().numpy()

    def get_metadata(self):
        """``{"history": {<metric>: [per epoch...], "params": {...}}}`` after fit, ``{}`` before."""
        if self._history is not None:
            history = self._history.history
            history["params"] = self._history.params
            return {"history": history}
        return {}


class KerasAutoEncoder(KerasBaseEstimator, TransformerMixin):
    """Feed-forward autoencoder; ``score`` is the explained variance of the reconstruction."""

    def score(self, X, y, sample_weight=None, **kwargs) -> float:
        if self.model is None:
            raise NotFittedError(f"This {self.__class__.__name__} has not been fitted yet.")
        return explained_variance_score(_as_2d_values(y), self.predict(X, **kwargs))


class KerasRawModelRegressor(KerasAutoEncoder):
    """
    A Dense network from a raw model definition: ``kind`` is the dict itself, ``{"spec": {...models.Sequential: {"layers": [...]}},
    "compile": {"loss": ..., "optimizer": ..., "metrics": ...}}``, as gordo project YAML gives it.  The ``Sequential`` must be a stack
    of ``Dense`` layers, with ``Dropout`` layers between them or in front of the first one (``factories.raw``); it trains and
    predicts on the Dense kernels, its L1 / L2 kernel and bias regularizers and its dropout inside the fit kernel (``predict`` runs
    without dropout, as Keras' does).  Any other graph is refused with a ValueError.  ``score`` is the explained variance, as for
    ``KerasAutoEncoder``.

    >>> model = KerasRawModelRegressor(kind={"compile": {"loss": "mse", "optimizer": "adam"},
    ...     "spec": {"tensorflow.keras.models.Sequential": {"layers": [{"tensorflow.keras.layers.Dense": {"units": 4, "input_shape": [4]}},
    ...                                                                {"tensorflow.keras.layers.Dense": {"units": 1}}]}}})
    >>> model.kwargs.update(n_features=4, n_features_out=1)
    >>> model._build_spec().dims
    [4, 4, 1]
    """

    _expected_keys = ("spec", "compile")

    def load_kind(self, kind):
        return kind

    def __repr__(self):
        return f"{self.__class__.__name__}(kind: {pformat(self.kind)})"

    def __sklearn_clone__(self):
        return self.__class__(deepcopy(self.kind), **deepcopy(self.kwargs))

    def _build_spec(self):
        if not all(k in self.kind for k in self._expected_keys):
            raise ValueError(f"Expected spec to have keys: {self._expected_keys}, but found {self.kind.keys()}")
        return raw_spec(self.kind, self.kwargs.get("n_features"), self.kwargs.get("n_features_out"))


class KerasLSTMBaseEstimator(KerasBaseEstimator, TransformerMixin, metaclass=abc.ABCMeta):
    """Many-to-one LSTM over a sliding ``lookback_window`` (autoencoder: lookahead 0, forecast: lookahead 1)."""

    def __init__(self, kind: Union[Callable, str], lookback_window: int = 1, batch_size: int = 32, **kwargs) -> None:
        self.lookback_window = lookback_window
        self.batch_size = batch_size
        kwargs["lookback_window"] = lookback_window
        kwargs["batch_size"] = batch_size
        super().__init__(kind, **kwargs)

    def __sklearn_clone__(self):
        kw = deepcopy(self.kwargs)
        kw.pop("lookback_window", None)
        kw.pop("batch_size", None)
        return self.__class__(self.kind, lookback_window=self.lookback_window, batch_size=self.batch_size, **kw)

    @property
    @abc.abstractmethod
    def lookahead(self) -> int:
        """Steps ahead in y the model targets."""

    def get_metadata(self):
        metadata = super().get_metadata()
        metadata.update({"forecast_steps": self.lookahead})
        return metadata

    def _validate_and_fix_size_of_X(self, X):
        if X.ndim == 1:
            X = X.reshape(len(X), 1)
        if self.lookback_window >= X.shape[0]:
            raise ValueError("For KerasLSTMForecast lookback_window must be < size of X")
        return X

    def _engine(self):
        from ... import engine

        return engine.lstm_engine_for(self.model.spec)

    def initialize(self, n_features: int, n_features_out: Optional[int] = None):
        """Build the network with freshly initialised weights (what the reference's primer fit does, models.py:585-597)."""
        self.kwargs.update({"n_features": int(n_features), "n_features_out": int(n_features_out or n_features)})
        self._prepare_model()
        return self

    def fit(self, X, y, **kwargs):
        """
        models.py:557-616: the network is built and initialised, takes the reference's primer Adam step on the first window,
        then ``epochs`` passes over the lookback windows in order (``shuffle=False``) in batches of ``self.batch_size``
        (gb_lstm_fit, back-propagation through time on the GPU).  Batches of up to 32 windows train on the fp32 kernel family,
        larger ones (up to 256) on the tensor-core family (``LSTMEngine.fit_tc``).
        """
        from ... import engine

        X = self._validate_and_fix_size_of_X(_as_2d_values(X))
        y = _as_2d_values(y)
        if y.ndim == 1:
            y = y.reshape(-1, 1)
        self.initialize(X.shape[1], y.shape[1])
        spec = self.model.spec
        optimizer = fit_optimizer(spec)  # None: Adam from spec.adam
        fit_args = {**self.extract_supported_fit_args(self.kwargs), **kwargs}
        epochs = int(fit_args.get("epochs", 1))
        callbacks = build_callbacks(fit_args.get("callbacks"))
        for cb in callbacks:
            cb.reset()
        batch_size = int(self.batch_size)
        n_win = len(X) - self.lookback_window + 1 - self.lookahead
        if n_win < 1:
            raise ValueError("no training windows")
        eng = self._engine()
        fit = eng.fit_for_batch(batch_size)
        dev = eng.device
        xd, yd = engine.to_device_f32(X, dev), engine.to_device_f32(y, dev)
        params = eng.pack_params([self.model.weights])
        jobs = engine.jobs_to_device(engine.make_jobs([0], [n_win], [0]), dev)
        want_acc = "accuracy" in getattr(spec, "metrics", ("accuracy",))
        history: Dict[str, list] = {"loss": []}
        if want_acc:
            history["accuracy"] = []
        if callbacks:  # one launch sequence per epoch, the callbacks in between (the generator fit has no validation data)
            state = None
            for e in range(epochs):
                loss, acc, state = fit(params, jobs, 1, n_win, xd, yd, epochs=1, batch_size=batch_size, lookahead=self.lookahead,
                                       primer=(e == 0), adam=getattr(spec, "adam", None), state=state, loss=spec.loss, optimizer=optimizer)
                logs = {"loss": float(loss[0, 0])}
                if want_acc:
                    logs["accuracy"] = float(acc[0, 0])
                for k, v in logs.items():
                    history[k].append(v)
                if any([cb.update(e, logs, lambda: params.clone()) for cb in callbacks]):
                    break
            for cb in callbacks:
                if cb.restore_best_weights and cb.best_weights is not None:
                    params = cb.best_weights
        else:
            loss, acc, _ = fit(params, jobs, 1, n_win, xd, yd, epochs=epochs, batch_size=batch_size, lookahead=self.lookahead,
                               primer=True, adam=getattr(spec, "adam", None), loss=spec.loss, optimizer=optimizer)
            history["loss"] = [float(v) for v in loss[0].cpu().numpy()]
            if want_acc:
                history["accuracy"] = [float(v) for v in acc[0].cpu().numpy()]
        self.model.weights = eng.unpack_params(params)[0]
        self.__dict__["_dev_cache"] = (self.model.weights, params)
        self._history = History(history, {"verbose": 0, "epochs": epochs, "steps": int(math.ceil(n_win / batch_size))}, list(range(len(history["loss"]))))
        self.model.history = self._history
        return self

    def predict(self, X, **kwargs) -> np.ndarray:
        """``[len(X) - lookback_window + 1 - lookahead, n_features_out]`` float32: row j is the net applied to X[j : j+lookback]."""
        from ... import engine

        if self.model is None:
            raise NotFittedError(f"This {self.__class__.__name__} has not been fitted yet.")
        X = self._validate_and_fix_size_of_X(_as_2d_values(X))
        eng = self._engine()
        n_win = len(X) - self.lookback_window + 1 - self.lookahead
        if n_win <= 0:
            return np.empty((0, eng.n_out), np.float32)
        xd = engine.to_device_f32(X, eng.device)
        jobs = engine.jobs_to_device(engine.make_jobs([0], [n_win], [0]), eng.device)
        cache = self.__dict__.get("_dev_cache")
        if cache is None or cache[0] is not self.model.weights:
            cache = (self.model.weights, eng.pack_params([self.model.weights]))
            self.__dict__["_dev_cache"] = cache
        # ±inf in X: the fp32 kernel saturates the gates as Keras does; the tensor-core kernel's windows come out NaN
        variant = 1 if np.asarray(X).dtype.kind == "f" and np.isinf(X).any() else 0
        return eng.infer(cache[1], jobs, 1, n_win, xd, n_win, variant=variant).cpu().numpy()

    def score(self, X, y, sample_weight=None, **kwargs) -> float:
        if self.model is None:
            raise NotFittedError(f"This {self.__class__.__name__} has not been fitted yet.")
        out = self.predict(X, **kwargs)
        return explained_variance_score(_as_2d_values(y)[-len(out):], out)


class KerasLSTMForecast(KerasLSTMBaseEstimator):
    @property
    def lookahead(self) -> int:
        return 1


class KerasLSTMAutoEncoder(KerasLSTMBaseEstimator):
    @property
    def lookahead(self) -> int:
        return 0


class TimeseriesWindows:
    """
    Index form of the reference's generator: sample j is ``X[j : j+lookback]`` with target
    ``y[j + lookback - 1 + lookahead]``.  Batches are materialised only when indexed (host side, for
    inspection/tests); the LSTM kernels read the windows straight out of ``X``.
    """

    def __init__(self, X, y, batch_size, lookback_window, lookahead):
        self.X, self.y = np.asarray(X), (np.asarray(y) if y is not None else None)
        self.batch_size, self.lookback_window, self.lookahead = int(batch_size), int(lookback_window), int(lookahead)
        count = max(len(self.X) - self.lookback_window + 1 - self.lookahead, 0)
        self.starts = np.arange(count)
        self.targets = self.starts + self.lookback_window - 1 + self.lookahead

    def __len__(self):
        return int(math.ceil(len(self.starts) / self.batch_size))

    def __getitem__(self, i):
        js = self.starts[i * self.batch_size : (i + 1) * self.batch_size]
        bx = np.array([self.X[j : j + self.lookback_window] for j in js])
        by = self.y[self.targets[i * self.batch_size : (i + 1) * self.batch_size]] if self.y is not None else None
        return bx, by


def create_keras_timeseriesgenerator(X, y, batch_size: int, lookback_window: int, lookahead: int) -> TimeseriesWindows:
    """
    Windows over ``X`` with the target shifted ``lookahead`` steps past the window's last row.

    >>> import numpy as np
    >>> X, y = np.random.rand(100, 2), np.random.rand(100, 2)
    >>> gen = create_keras_timeseriesgenerator(X, y, batch_size=10, lookback_window=20, lookahead=0)
    >>> len(gen), len(gen[0]), len(gen[0][0]), len(gen[0][0][0]), len(gen[0][0][0][0])
    (9, 2, 10, 20, 2)
    """
    if lookahead < 0:
        raise ValueError(f"Value of `lookahead` can not be negative, is {lookahead}")
    return TimeseriesWindows(X, y, batch_size, lookback_window, lookahead)
