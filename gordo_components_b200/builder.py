"""
The builder side of the hot path: what ``gordo build`` does for one machine (``ModelBuilder``: data -> model from its
definition -> cross validation with the evaluation metrics -> final fit -> offset + metadata -> ``model.pkl`` /
``metadata.json``; gordo/builder/build_model.py:48-340, 345-570) and the same for a whole project at once
(``FleetModelBuilder``).

``FleetModelBuilder`` is where the batched kernels pay off: machines whose definition is the canonical
``DiffBasedAnomalyDetector(base_estimator=KerasAutoEncoder(<feed-forward kind>), scaler=MinMaxScaler())`` -- the network bare or
behind one ``MinMaxScaler`` in a Pipeline, as in gordo's example configs -- are bucketed by architecture and training length (with ``FleetModelBuilder(ragged=True)`` by architecture alone), and every bucket is built by ``fleet.build_fleet`` -- all final fits and all CV folds
in one ``gb_ffae_fit`` launch, fold scoring / thresholds / scaler statistics / metric moments one launch each.  With
``FleetModelBuilder(early_stopping=True)`` an estimator with one Keras ``EarlyStopping`` callback on a metric its fit reports
(loss, accuracy, and their ``val_*`` forms with a ``validation_split``) is batched as well: every fit applies the rule inside the
launch (``gb_ffae_fit_stop``), and machines that differ only in the callback's parameters share a bucket.  The LSTM form
of the same definition (``KerasLSTMAutoEncoder`` / ``KerasLSTMForecast``, ``_canonical_lstm``) is bucketed by architecture,
lookback, lookahead, batch size and training length and built by ``fleet.build_lstm_fleet``: all fits as jobs of ``gb_lstm_fit``
(batches above 32 windows: ``gb_lstm_fit_tc``, with ``FleetModelBuilder(lstm_wide_batches=True)``; in chunks that fit a workspace budget), every fold model's test block in one LSTM inference launch, float64 scoring.
With ``FleetModelBuilder(lstm_early_stopping=True)`` an LSTM estimator with one ``EarlyStopping`` on ``loss`` (or a reported
``accuracy``) is batched too: every fit applies the rule inside its launch (``gb_lstm_fit_stop`` / ``gb_lstm_fit_tc_stop``).  The
cross-validation ``scores`` block of the metadata is then assembled on the host from ``gb_cv_moments``' five sums per
(fold, tag).  Any other definition (other transformers in a Pipeline, callbacks unless batched as above, LSTM fits with
``validation_split``, K-fold detectors unless ``FleetModelBuilder(kfcv=True)`` batches them under a KFold cv through ``fleet.build_kfold_fleet``,
``TransformedTargetRegressor`` estimators unless ``FleetModelBuilder(target_scaler=True)`` batches them, custom metrics ...) goes through ``ModelBuilder``: one machine at a time, still on the GPU through the estimators' own fit / predict.

Machines are plain dicts in the layout of ``Machine.to_dict()`` (gordo/machine/machine.py:226-246): ``name``, ``model`` (a
definition), ``dataset``, and optionally ``project_name``, ``evaluation``, ``metadata``, ``runtime``.  ``dataset`` is
anything with ``get_data() -> (X, y)`` (and optionally ``get_metadata()``), an ``(X, y)`` pair, or ``{"X": ..., "y": ...}`` --
gordo's data providers themselves are outside this path.  Out of scope as well: the model cache / registry arguments of
``ModelBuilder.build`` and the reporters.
"""
import copy
import datetime
import importlib
import logging
import math
import os
import random
import time
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import pandas as pd
from sklearn import metrics as sk_metrics
from sklearn.base import BaseEstimator
from sklearn.compose import TransformedTargetRegressor
from sklearn.model_selection import KFold, TimeSeriesSplit, cross_validate
from sklearn.pipeline import Pipeline
from sklearn.preprocessing import MinMaxScaler

from . import __version__, serializer
from .machine.model.base import GordoBase
from .machine.model.factories.specs import dropout_key, fit_dropout, fit_optimizer, fit_reg, optimizer_key, reg_key
from .machine.model.utils import metric_wrapper

logger = logging.getLogger(__name__)

# NormalizedConfig.DEFAULT_CONFIG_GLOBALS["evaluation"] (gordo/workflow/config_elements/normalized_config.py:97-106)
DEFAULT_EVALUATION: Dict[str, Any] = {
    "cv_mode": "full_build",
    "scoring_scaler": "sklearn.preprocessing.MinMaxScaler",
    "metrics": ["explained_variance_score", "r2_score", "mean_squared_error", "mean_absolute_error"],
}
DEFAULT_CV = {"sklearn.model_selection.TimeSeriesSplit": {"n_splits": 3}}
MOMENT_METRICS = ("explained_variance_score", "r2_score", "mean_squared_error", "mean_absolute_error")


# ------------------------------------------------------------------------------------------------ pieces of ModelBuilder
def metrics_from_list(metric_list: Optional[Sequence[str]] = None) -> List[Callable]:
    """Metric names (looked up in ``sklearn.metrics``) or dotted function paths -> functions (build_model.py:671-707)."""
    funcs = []
    for path in metric_list or DEFAULT_EVALUATION["metrics"]:
        func = None
        if "." in path:
            module, _, name = path.rpartition(".")
            try:
                func = getattr(importlib.import_module(module), name, None)
            except ImportError:
                func = None
        if func is None:
            func = getattr(sk_metrics, path, None)
        if func is None:
            raise AttributeError(f"Could not locate metric function: {path}")
        funcs.append(func)
    return funcs


def _column_label(col) -> str:
    return str(col).replace(" ", "-")


def build_metrics_dict(metrics_list: Sequence[Callable], y: pd.DataFrame, scaler=None) -> dict:
    """
    sklearn scorers keyed ``<metric>-<tag>`` for every target tag and ``<metric>`` for the average over tags
    (build_model.py:378-446).  ``scaler`` (object or definition) is fitted on ``y`` and applied to targets and predictions
    before scoring.
    """
    if scaler:
        if isinstance(scaler, (str, dict)):
            scaler = serializer.from_definition(scaler)
        scaler.fit(y)

    def column_metric(func, index):
        def score(y_true, y_pred):
            y_true = getattr(y_true, "values", y_true)
            y_pred = getattr(y_pred, "values", y_pred)
            return func(y_true[:, index], y_pred[:, index])

        return score

    out = {}
    for func in metrics_list:
        name = func.__name__.replace("_", "-")
        for index, col in enumerate(y.columns):
            out[f"{name}-{_column_label(col)}"] = sk_metrics.make_scorer(metric_wrapper(column_metric(func, index), scaler=scaler))
        out[name] = sk_metrics.make_scorer(metric_wrapper(func, scaler=scaler))
    return out


def build_split_dict(X: pd.DataFrame, split_obj) -> dict:
    """Start / end timestamps and sizes of every CV fold's train and test part (build_model.py:347-376)."""
    out: Dict[str, Any] = {}
    for i, (train, test) in enumerate(split_obj.split(X), start=1):
        out[f"fold-{i}-train-start"] = X.index[train[0]]
        out[f"fold-{i}-train-end"] = X.index[train[-1]]
        out[f"fold-{i}-test-start"] = X.index[test[0]]
        out[f"fold-{i}-test-end"] = X.index[test[-1]]
        out[f"fold-{i}-n-train"] = len(train)
        out[f"fold-{i}-n-test"] = len(test)
    return out


def fold_summary(values) -> dict:
    """``fold-mean/std/max/min`` and ``fold-<i>`` of one metric's per-fold values (build_model.py:274-289)."""
    v = np.asarray(values, dtype=np.float64)
    out = {"fold-mean": float(v.mean()), "fold-std": float(v.std()), "fold-max": float(v.max()), "fold-min": float(v.min())}
    out.update({f"fold-{i + 1}": float(x) for i, x in enumerate(v)})
    return out


def determine_offset(model, X) -> int:
    """Rows the model's output is shorter than its input (LSTM look-back; build_model.py:448-471)."""
    X = getattr(X, "values", X)
    out = model.predict(X) if hasattr(model, "predict") else model.transform(X)
    return len(X) - len(out)


def extract_metadata_from_model(model, metadata: Optional[dict] = None) -> dict:
    """``get_metadata()`` of every GordoBase found in ``model`` (last Pipeline steps, estimator attributes; build_model.py:515-569)."""
    out = dict(metadata or {})
    if isinstance(model, Pipeline):
        out.update(extract_metadata_from_model(model.steps[-1][1]))
        return out
    if isinstance(model, GordoBase):
        out.update(model.get_metadata())
    for key, val in vars(model).items():
        if key == "regressor":  # TransformedTargetRegressor keeps the unfitted original next to regressor_
            continue
        if isinstance(val, Pipeline):
            out.update(extract_metadata_from_model(val.steps[-1][1]))
        elif isinstance(val, (GordoBase, BaseEstimator)):
            out.update(extract_metadata_from_model(val))
    return out


def scores_from_moments(moments: np.ndarray, n_rows, scoring_scale: Optional[np.ndarray] = None,
                        metrics: Sequence[str] = MOMENT_METRICS) -> Dict[str, Tuple[np.ndarray, np.ndarray]]:
    """
    The four evaluation metrics of one machine from ``gb_cv_moments``: ``moments`` is ``[folds, 5, tags]`` (sum e, sum e^2,
    sum |e|, sum (y-y0), sum (y-y0)^2 over the fold's ``n_rows`` test rows, e = prediction - target), ``scoring_scale`` the
    per-tag ``scale_`` of the scoring scaler fitted on all targets (an affine map per tag: errors scale by it, the two
    ratio metrics do not change).  ``n_rows``: the test rows of every fold (an int), or one count per fold (KFold folds differ
    in size by one row).  Returns ``{metric: (per_tag [folds, tags], averaged [folds])}`` with sklearn's
    conventions: uniform average over tags; a constant target scores 1 when predicted exactly and 0 otherwise.
    """
    m = np.asarray(moments, dtype=np.float64)
    n = float(n_rows) if np.ndim(n_rows) == 0 else np.asarray(n_rows, dtype=np.float64).reshape(-1, 1)  # per fold, against [folds, tags]
    se, see, sae, sc, scc = (m[..., q, :] for q in range(5))
    s = 1.0 if scoring_scale is None else np.asarray(scoring_scale, dtype=np.float64)

    def explained(numerator, denominator):
        out = np.ones_like(numerator)
        ok = (numerator != 0) & (denominator != 0)
        out[ok] = 1.0 - numerator[ok] / denominator[ok]
        out[(numerator != 0) & (denominator == 0)] = 0.0
        return out

    tss = np.maximum(scc - sc * sc / n, 0.0)  # sum (y - mean y)^2
    per_tag = {
        "explained_variance_score": lambda: explained(np.maximum(see / n - (se / n) ** 2, 0.0), tss / n),
        "r2_score": lambda: explained(see, tss),
        "mean_squared_error": lambda: see / n * s * s,
        "mean_absolute_error": lambda: sae / n * np.abs(s),
    }
    out = {}
    for name in metrics:
        if name not in per_tag:
            raise ValueError(f"metric {name!r} is not one of {MOMENT_METRICS}")
        values = per_tag[name]()
        out[name] = (values, values.mean(axis=-1))
    return out


def scores_block(moment_scores: Dict[str, Tuple[np.ndarray, np.ndarray]], tags: Sequence) -> dict:
    """``scores`` of the build metadata from ``scores_from_moments``: same keys and summaries as ModelBuilder writes."""
    out = {}
    for name, (per_tag, averaged) in moment_scores.items():
        label = name.replace("_", "-")
        # all tags at once (a thousand machines x 65 keys x 4 metrics is too many tiny numpy calls): rows = folds, last column = the average
        v = np.concatenate([np.asarray(per_tag, dtype=np.float64), np.asarray(averaged, dtype=np.float64)[:, None]], axis=1)
        stats = np.stack([v.mean(axis=0), v.std(axis=0), v.max(axis=0), v.min(axis=0)]).T.tolist()
        folds = v.T.tolist()
        keys = [f"{label}-{_column_label(tag)}" for tag in tags] + [label]
        for key, (mean, std, vmax, vmin), values in zip(keys, stats, folds):
            summary = {"fold-mean": mean, "fold-std": std, "fold-max": vmax, "fold-min": vmin}
            summary.update({f"fold-{i + 1}": x for i, x in enumerate(values)})
            out[key] = summary
    return out


def _get_data(dataset):
    if hasattr(dataset, "get_data"):
        X, y = dataset.get_data()
        meta = dataset.get_metadata() if hasattr(dataset, "get_metadata") else {}
    elif isinstance(dataset, dict) and "X" in dataset:
        X, y, meta = dataset["X"], dataset.get("y"), dataset.get("metadata", {})
    elif isinstance(dataset, (tuple, list)) and len(dataset) == 2:
        (X, y), meta = dataset, {}
    else:
        raise TypeError("dataset must provide get_data(), or be an (X, y) pair or {'X': ..., 'y': ...}; gordo's data providers "
                        "are outside this package")
    if not isinstance(X, pd.DataFrame):
        X = pd.DataFrame(np.asarray(X))
    if y is None:
        y = X
    if not isinstance(y, pd.DataFrame):
        y = pd.DataFrame(np.asarray(y), index=X.index)
    return X, y, meta


def _machine_dict(machine) -> dict:
    machine = machine.to_dict() if hasattr(machine, "to_dict") and not isinstance(machine, dict) else machine
    if "name" not in machine or "model" not in machine or "dataset" not in machine:
        raise ValueError("a machine needs at least 'name', 'model' and 'dataset'")
    return machine


def _machine_out(machine: dict, build_metadata: dict) -> dict:
    """The machine as ``Machine.to_dict()`` would give it after a build: the input plus ``metadata.build_metadata``."""
    out = {k: v for k, v in machine.items() if k != "dataset"}
    ds = machine["dataset"]
    out["dataset"] = ds.to_dict() if hasattr(ds, "to_dict") else (ds if isinstance(ds, dict) and "X" not in ds else {})
    meta = copy.deepcopy(machine.get("metadata") or {})
    meta.setdefault("user_defined", {})
    meta["build_metadata"] = build_metadata
    out["metadata"] = meta
    out["evaluation"] = {**DEFAULT_EVALUATION, **(machine.get("evaluation") or {})}
    return out


def _now() -> str:
    return str(datetime.datetime.now(datetime.timezone.utc).astimezone())


class ModelBuilder:
    """
    Build one machine: ``ModelBuilder(machine).build(output_dir)`` -> ``(model, machine_dict)``; the machine dict carries
    ``metadata.build_metadata.{model,dataset}`` exactly where the reference puts it (build_model.py:291-339).
    """

    def __init__(self, machine):
        self.machine = _machine_dict(machine)

    @property
    def gordo_version(self) -> str:
        return __version__

    @staticmethod
    def set_seed(seed: int):
        # the fit loops draw their shuffling seed and initial weights from numpy's global state
        np.random.seed(seed)
        random.seed(seed)

    def build(self, output_dir: Optional[str] = None):
        model, machine = self._build()
        if output_dir is not None:
            serializer.dump(model, output_dir, metadata=machine)
        return model, machine

    def _build(self):
        machine = self.machine
        evaluation = {**DEFAULT_EVALUATION, **(machine.get("evaluation") or {})}
        self.set_seed(int(evaluation.get("seed", 0)))

        t0 = time.time()
        X, y, dataset_meta = _get_data(machine["dataset"])
        query_sec = time.time() - t0
        model = serializer.from_definition(machine["model"])

        cv_sec, scores, splits = None, {}, {}
        cv_mode = str(evaluation["cv_mode"]).lower()
        if cv_mode in ("cross_val_only", "full_build") and hasattr(model, "predict"):
            t0 = time.time()
            scorers = build_metrics_dict(metrics_from_list(evaluation.get("metrics")), y, scaler=evaluation.get("scoring_scaler"))
            split_obj = serializer.from_definition(evaluation.get("cv", DEFAULT_CV))
            splits = build_split_dict(X, split_obj)
            kw = dict(X=X, y=y, scoring=scorers, return_estimator=True, cv=split_obj)
            cv = model.cross_validate(**kw) if hasattr(model, "cross_validate") else cross_validate(model, **kw)
            scores = {name: fold_summary(cv[f"test_{name}"]) for name in scorers}
            cv_sec = time.time() - t0
        cross_validation = {"scores": scores, "cv_duration_sec": cv_sec, "splits": splits}
        dataset_block = {"query_duration_sec": query_sec, "dataset_meta": dataset_meta}
        if cv_mode == "cross_val_only":
            return model, _machine_out(machine, {"model": {"cross_validation": cross_validation}, "dataset": dataset_block})

        t0 = time.time()
        model.fit(X, y)
        fit_sec = time.time() - t0
        model_block = {
            "model_offset": determine_offset(model, X),
            "model_creation_date": _now(),
            "model_builder_version": self.gordo_version,
            "model_training_duration_sec": fit_sec,
            "cross_validation": cross_validation,
            "model_meta": extract_metadata_from_model(model),
        }
        return model, _machine_out(machine, {"model": model_block, "dataset": dataset_block})


# ------------------------------------------------------------------------------------------------ the whole project at once
class _Canonical:
    """What ``FleetModelBuilder`` needs to know about a machine that can take the batched path."""

    def __init__(self, index, machine, model, spec, X, y, dataset_meta, query_sec, fit, n_splits, evaluation, input_scaler,
                 split=(False, 0.0, None), early_stopping=None):
        self.index, self.machine, self.model, self.spec, self.input_scaler = index, machine, model, spec, input_scaler
        self.split = split  # (detector shuffle, keras validation_split, validation batch size or None without a split)
        self.early_stopping = early_stopping  # the estimator's one EarlyStopping callback, or None
        self.X, self.y, self.dataset_meta, self.query_sec = X, y, dataset_meta, query_sec
        self.fit, self.n_splits, self.evaluation = fit, n_splits, evaluation
        self.window = None  # the plain detector's smoothing window (FleetModelBuilder(smoothing=True)), or None
        self.target_scaler = False  # the estimator is a TransformedTargetRegressor(MinMaxScaler()) (FleetModelBuilder(target_scaler=True))

    def _window_key(self) -> tuple:
        """The smoothing window as a bucket field, only when there is one: keys of machines without a window stay as they were.
        The smoothing method does not enter the thresholds, so it does not split buckets."""
        return () if self.window is None else (("window", self.window),)

    def _target_key(self) -> tuple:
        """The target transformer as a bucket field, only when there is one: keys of machines without one stay as they were."""
        return (("target_scaler", True),) if self.target_scaler else ()

    def bucket(self, ragged: bool = False):
        """The fields machines of one batched build share; ``ragged`` leaves out the row count (``FleetModelBuilder(ragged=True)``)."""
        s = self.spec
        return (tuple(s.dims), tuple(s.acts), tuple(float(v) for v in s.l1), tuple(sorted(s.adam.items())), tuple(s.metrics), s.loss,
                None if ragged else len(self.X), self.fit["epochs"], self.fit["batch_size"], self.fit["shuffle"], self.n_splits, int(self.evaluation.get("seed", 0)),
                self.split, self.early_stopping is not None, self.input_scaler) + optimizer_key(s) + reg_key(s) + dropout_key(s) + self._window_key() + self._target_key()  # EarlyStopping's parameters are per-job records


def _default_minmax(scaler) -> bool:
    return type(scaler) is MinMaxScaler and tuple(scaler.feature_range) == (0, 1) and not getattr(scaler, "clip", False)


def _window_refusal(model) -> Optional[str]:
    """Why the batched builds cannot take this detector's smoothing window (not a positive int, or an unknown method), or None."""
    import numbers

    if model.window is not None and (not isinstance(model.window, numbers.Integral) or isinstance(model.window, bool) or model.window < 1):
        return f"window {model.window!r} is not a positive int"
    if model.window is not None and model.smoothing_method not in ("smm", "sma", "ewma"):
        return f"smoothing_method {model.smoothing_method!r}"
    return None


def _target_regressor(est, target_scaler: bool = True):
    """
    (refusal or None, the regressor, whether it sits in a TransformedTargetRegressor) of a detector's base estimator.  A
    TransformedTargetRegressor is taken only with ``target_scaler`` and a default MinMaxScaler transformer, without ``func`` /
    ``inverse_func``; any other estimator is its own regressor.
    """
    if type(est) is not TransformedTargetRegressor:
        return None, est, False
    if est.func is not None or est.inverse_func is not None or est.transformer is None or not _default_minmax(est.transformer):
        return "TransformedTargetRegressor without a default MinMaxScaler transformer", est, True
    if not target_scaler:
        return "a TransformedTargetRegressor is batched with FleetModelBuilder(target_scaler=True)", est, True
    return None, est.regressor, True


def _refuse(machine, reason: str) -> None:
    """Log why ``machine`` takes the per-machine path; the classifiers return this None."""
    logger.info("machine %s takes the per-machine path: %s", machine["name"], reason)
    return None


def _tss_refusal(split_obj) -> Optional[str]:
    """Why the batched builds cannot take this cv (anything but a plain TimeSeriesSplit), or None."""
    if type(split_obj) is not TimeSeriesSplit or split_obj.max_train_size is not None or split_obj.test_size is not None or split_obj.gap:
        return "cv is not a plain TimeSeriesSplit"
    return None


def _fetch(machine):
    """(X, y, dataset metadata, query seconds) of the machine's dataset."""
    t0 = time.time()
    X, y, dataset_meta = _get_data(machine["dataset"])
    return X, y, dataset_meta, time.time() - t0


def _canonical(index, machine, early_stopping: bool = False, smoothing: bool = False, target_scaler: bool = False) -> Optional[_Canonical]:
    """
    The machine as a candidate for the batched path, or ``None`` with the reason logged.  ``early_stopping``: also take an
    estimator with one Keras ``EarlyStopping`` callback on a metric its fit reports (``FleetModelBuilder(early_stopping=True)``);
    without it any callback sends the machine to ``ModelBuilder``.  ``smoothing``: also take a detector with a smoothing
    ``window`` (a positive int, smm / sma / ewma; ``FleetModelBuilder(smoothing=True)``); without it such a detector goes to
    ``ModelBuilder``.  ``target_scaler``: also take the estimator inside a ``TransformedTargetRegressor`` with a default MinMaxScaler
    transformer (``FleetModelBuilder(target_scaler=True)``); without it such a detector goes to ``ModelBuilder``.
    """
    from .machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from .machine.model.factories.specs import FFNetSpec
    from .machine.model.models import KerasAutoEncoder, KerasRawModelRegressor

    evaluation = {**DEFAULT_EVALUATION, **(machine.get("evaluation") or {})}
    reason = _evaluation_refusal(evaluation)
    if reason:
        return _refuse(machine, reason)
    split_obj = serializer.from_definition(evaluation.get("cv", DEFAULT_CV))
    reason = _tss_refusal(split_obj)
    if reason:
        return _refuse(machine, reason)

    model = serializer.from_definition(machine["model"])
    if type(model) is not DiffBasedAnomalyDetector or (model.window is not None and not smoothing):
        return _refuse(machine, "model is not a plain DiffBasedAnomalyDetector")
    reason = _window_refusal(model)
    if reason:
        return _refuse(machine, reason)
    if not _default_minmax(model.scaler):
        return _refuse(machine, "detector scaler is not a default MinMaxScaler")
    reason, est, in_ttr = _target_regressor(model.base_estimator, target_scaler)
    if reason:
        return _refuse(machine, reason)
    ae, input_scaler = _network(est, (KerasAutoEncoder, KerasRawModelRegressor))
    if ae is None:
        return _refuse(machine, "base_estimator is not a KerasAutoEncoder, bare or behind one default MinMaxScaler")
    reason, fit_args, stopping, vsplit = _ff_fit_arguments(ae, early_stopping)
    if reason:
        return _refuse(machine, reason)

    X, y, dataset_meta, query_sec = _fetch(machine)
    ae.kwargs.update({"n_features": X.shape[1], "n_features_out": y.shape[1]})
    spec = ae._build_spec()
    if not isinstance(spec, FFNetSpec):
        return _refuse(machine, "not a feed-forward network")
    test = len(X) // (split_obj.n_splits + 1)
    if len(X) != len(y) or test == 0:
        return _refuse(machine, "too few rows for the CV folds")
    if vsplit and math.floor((len(X) - split_obj.n_splits * test) * (1.0 - vsplit)) < 1:  # the smallest fold: keras' split (models.py)
        return _refuse(machine, f"validation_split {vsplit} leaves the first CV fold without a training row")
    reason = _monitor_refusal(stopping, spec, vsplit)
    if reason:
        return _refuse(machine, reason)
    fit, split = _ff_fit(fit_args, model.shuffle, vsplit)
    c = _Canonical(index, machine, model, spec, X, y, dataset_meta, query_sec, fit, split_obj.n_splits, evaluation, input_scaler, split, stopping)
    c.window = None if model.window is None else int(model.window)
    c.target_scaler = in_ttr
    return c


def _evaluation_refusal(evaluation: dict) -> Optional[str]:
    """Why the batched path cannot reproduce this evaluation's metadata (cv aside), or None."""
    if str(evaluation["cv_mode"]).lower() != "full_build":
        return f"cv_mode {evaluation['cv_mode']}"
    if any(m.rpartition(".")[2] not in MOMENT_METRICS or ("." in m and not m.startswith("sklearn.metrics.")) for m in evaluation["metrics"]):
        return "evaluation metrics beyond the four moment metrics"
    scoring = evaluation.get("scoring_scaler")
    if scoring:
        scoring = serializer.from_definition(scoring) if isinstance(scoring, (str, dict)) else scoring
        if not _default_minmax(scoring):
            return "scoring_scaler is not a default MinMaxScaler"
    return None


def _network(est, types: tuple):
    """(the network, whether a default MinMaxScaler is in front of it) of a bare network of one of ``types`` or
    ``Pipeline([MinMaxScaler(), network])``; (None, False) otherwise."""
    input_scaler = False
    if type(est) is Pipeline and len(est.steps) == 2 and _default_minmax(est.steps[0][1]):
        est, input_scaler = est.steps[1][1], True  # Pipeline([MinMaxScaler(), KerasAutoEncoder]): gordo's example config
    return (est, input_scaler) if type(est) in types else (None, False)


def _ff_fit(fit_args, detector_shuffle, vsplit: float):
    """The ``fit`` dict (epochs, batch size, shuffle) and ``split`` tuple (detector shuffle, validation_split, validation batch
    size or None without a split) of a feed-forward estimator's fit arguments."""
    fit = {"epochs": int(fit_args.get("epochs", 1)), "batch_size": int(fit_args.get("batch_size") or 32), "shuffle": bool(fit_args.get("shuffle", True))}
    return fit, (bool(detector_shuffle), vsplit, int(fit_args.get("validation_batch_size") or fit["batch_size"]) if vsplit else None)


def _early_stopping(fit_args, early_stopping: bool, flag: str):
    """(refusal or None, the one EarlyStopping callback or None) of an estimator's fit arguments; ``flag`` names the builder option."""
    from .machine.model.models import build_callbacks

    if not fit_args.get("callbacks"):
        return None, None
    if not early_stopping:
        return f"callbacks need the per-epoch loop (FleetModelBuilder({flag}=True) batches one EarlyStopping)", None
    definitions = fit_args["callbacks"]
    definitions = list(definitions) if isinstance(definitions, (list, tuple)) else [definitions]
    callbacks = build_callbacks(definitions)
    if len(definitions) != 1 or len(callbacks) != 1:  # several callbacks, or one the fit loop does not know
        return "callbacks other than one EarlyStopping need the per-epoch loop", None
    return None, callbacks[0]


def _ff_fit_arguments(ae, early_stopping: bool):
    """(refusal or None, fit arguments, the one EarlyStopping callback or None, validation_split) of a feed-forward estimator."""
    fit_args = ae.extract_supported_fit_args(ae.kwargs)
    reason, stopping = _early_stopping(fit_args, early_stopping, "early_stopping")
    if reason:
        return reason, fit_args, None, 0.0
    vsplit = float(fit_args.get("validation_split") or 0.0)
    if vsplit and not 0.0 < vsplit < 1.0:
        return f"validation_split {vsplit} is outside (0, 1)", fit_args, stopping, vsplit
    return None, fit_args, stopping, vsplit


def _monitor_refusal(stopping, spec, vsplit: float) -> Optional[str]:
    """Why the fit cannot apply this EarlyStopping callback (a monitor it does not report), or None."""
    if stopping is None:
        return None
    available = {"loss"} | ({"accuracy"} if "accuracy" in spec.metrics else set())
    if vsplit:
        available |= {"val_" + k for k in available}
    if stopping.monitor not in available:
        return f"EarlyStopping monitors {stopping.monitor!r}, which this fit does not report"
    return None


class _CanonicalLSTM(_Canonical):
    """A machine whose LSTM detector can take the batched path (``fleet.build_lstm_fleet``)."""

    def __init__(self, *args, lookahead: int):
        super().__init__(*args)
        self.lookahead = lookahead

    def bucket(self, ragged: bool = False):
        s = self.spec
        return (s.key(), tuple(sorted(s.adam.items())), tuple(s.metrics), s.loss, self.lookahead, None if ragged else len(self.X), self.fit["epochs"], self.fit["batch_size"],
                self.n_splits, int(self.evaluation.get("seed", 0)), self.input_scaler, self.early_stopping is not None) + optimizer_key(s) + self._window_key() + self._target_key()  # EarlyStopping's parameters are per-job records


def _is_lstm_definition(machine) -> bool:
    """True when the machine's model is a DiffBasedAnomalyDetector around an LSTM estimator (bare or last Pipeline step, either of
    them optionally inside a TransformedTargetRegressor)."""
    from .machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from .machine.model.models import KerasLSTMBaseEstimator

    try:
        model = serializer.from_definition(machine["model"])
    except Exception:  # ModelBuilder raises the definition's own error
        return False
    est = getattr(model, "base_estimator", None) if isinstance(model, DiffBasedAnomalyDetector) else None
    if isinstance(est, TransformedTargetRegressor):
        est = est.regressor
    if isinstance(est, Pipeline) and est.steps:
        est = est.steps[-1][1]
    return isinstance(est, KerasLSTMBaseEstimator)


def _canonical_lstm(index, machine, wide_batches: bool = False, early_stopping: bool = False, smoothing: bool = False,
                    target_scaler: bool = False) -> Optional[_CanonicalLSTM]:
    """
    The LSTM form of the canonical definition -- ``DiffBasedAnomalyDetector(KerasLSTMAutoEncoder | KerasLSTMForecast)``, the network bare
    or behind one default ``MinMaxScaler``, under the evaluation ``_canonical`` accepts -- as a candidate for the batched path, or
    ``None`` with the reason logged.  Machines too short for the CV folds go to ``ModelBuilder``, which raises the reference's errors.
    ``wide_batches``: also take batch sizes above 32, up to ``LSTMEngine.TC_MAX_BATCH`` (the tensor-core fit family;
    ``FleetModelBuilder(lstm_wide_batches=True)``).  ``early_stopping``: also take an estimator with one Keras ``EarlyStopping``
    callback on a metric its fit reports, ``loss`` or (with the accuracy metric) ``accuracy`` (``FleetModelBuilder(lstm_early_stopping=True)``).
    ``smoothing``: also take a detector with a smoothing ``window``, as ``_canonical`` does (``FleetModelBuilder(smoothing=True)``).
    ``target_scaler``: also take the estimator inside a ``TransformedTargetRegressor`` with a default MinMaxScaler transformer, as
    ``_canonical`` does (``FleetModelBuilder(target_scaler=True)``).
    """
    from .machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from .engine import LSTMEngine
    from .machine.model.factories.specs import LSTMNetSpec
    from .machine.model.models import KerasLSTMAutoEncoder, KerasLSTMForecast

    evaluation = {**DEFAULT_EVALUATION, **(machine.get("evaluation") or {})}
    reason = _evaluation_refusal(evaluation)
    if reason:
        return _refuse(machine, reason)
    split_obj = serializer.from_definition(evaluation.get("cv", DEFAULT_CV))
    reason = _tss_refusal(split_obj)
    if reason:
        return _refuse(machine, reason)

    model = serializer.from_definition(machine["model"])
    if type(model) is not DiffBasedAnomalyDetector or (model.window is not None and not smoothing) or model.shuffle:
        return _refuse(machine, "model is not a plain DiffBasedAnomalyDetector")
    reason = _window_refusal(model)
    if reason:
        return _refuse(machine, reason)
    if not _default_minmax(model.scaler):
        return _refuse(machine, "detector scaler is not a default MinMaxScaler")
    reason, est, in_ttr = _target_regressor(model.base_estimator, target_scaler)
    if reason:
        return _refuse(machine, reason)
    est, input_scaler = _network(est, (KerasLSTMAutoEncoder, KerasLSTMForecast))
    if est is None:
        return _refuse(machine, "base_estimator is not a KerasLSTMAutoEncoder / KerasLSTMForecast, bare or behind one default MinMaxScaler")
    fit_args = est.extract_supported_fit_args(est.kwargs)
    if fit_args.get("validation_split"):
        return _refuse(machine, "validation_split needs the per-machine fit")
    reason, stopping = _early_stopping(fit_args, early_stopping, "lstm_early_stopping")
    if reason:
        return _refuse(machine, reason)
    batch_size = int(est.batch_size)
    if not 1 <= batch_size <= LSTMEngine.FP32_MAX_BATCH and not (wide_batches and 1 <= batch_size <= LSTMEngine.TC_MAX_BATCH):
        if wide_batches:
            return _refuse(machine, f"batch_size {batch_size}: the batched LSTM fit takes at most {LSTMEngine.TC_MAX_BATCH} windows per batch")
        return _refuse(machine, f"batch_size {batch_size}: the batched LSTM fit takes at most {LSTMEngine.FP32_MAX_BATCH} windows per batch "
                  "(FleetModelBuilder(lstm_wide_batches=True) batches up to 256)")

    X, y, dataset_meta, query_sec = _fetch(machine)
    est.kwargs.update({"n_features": X.shape[1], "n_features_out": y.shape[1]})
    spec = est._build_spec()
    if not isinstance(spec, LSTMNetSpec):
        return _refuse(machine, "not an LSTM network")
    L, la, K = int(est.lookback_window), int(est.lookahead), split_obj.n_splits
    test = len(X) // (K + 1)
    first_train = len(X) - K * test
    if len(X) != len(y) or test <= L + la or first_train <= L or first_train - L + 1 - la < 1:
        return _refuse(machine, "too few rows for the CV folds at this lookback_window")
    reason = _monitor_refusal(stopping, spec, 0.0)  # the generator fit has no validation data
    if reason:
        return _refuse(machine, reason)
    fit = {"epochs": int(fit_args.get("epochs", 1)), "batch_size": batch_size, "shuffle": False}
    c = _CanonicalLSTM(index, machine, model, spec, X, y, dataset_meta, query_sec, fit, K, evaluation, input_scaler, (False, 0.0, None), stopping,
                       lookahead=la)
    c.window = None if model.window is None else int(model.window)
    c.target_scaler = in_ttr
    return c


class _CanonicalKFold(_Canonical):
    """A machine whose ``DiffBasedKFCVAnomalyDetector`` can take the batched path (``fleet.build_kfold_fleet``)."""

    def __init__(self, *args, cv, target_scaler: bool):
        super().__init__(*args)
        self.cv, self.target_scaler = cv, target_scaler

    def bucket(self, ragged: bool = False):
        m = self.model  # every field below is a scalar of the shared row maps or of the gb_smooth / gb_quantile launches
        return super().bucket(ragged) + ((self.cv.n_splits, bool(self.cv.shuffle), self.cv.random_state), m.window, m.smoothing_method,
                                   float(m.threshold_percentile), bool(m.shuffle), self.target_scaler)

    def _target_key(self) -> tuple:
        return ()  # the K-fold key carries the target transformer in a field of its own


def _is_kfcv_definition(machine) -> bool:
    from .machine.model.anomaly.diff import DiffBasedKFCVAnomalyDetector

    try:
        return type(serializer.from_definition(machine["model"])) is DiffBasedKFCVAnomalyDetector
    except Exception:  # ModelBuilder raises the definition's own error
        return False


def _canonical_kfcv(index, machine, early_stopping: bool = False) -> Optional[_CanonicalKFold]:
    """
    A ``DiffBasedKFCVAnomalyDetector`` machine as a candidate for the batched path (``FleetModelBuilder(kfcv=True)``), or ``None``
    with the reason logged.  The detector has a default MinMaxScaler, an int or no ``window`` and smm / sma / ewma smoothing; its
    estimator is a feed-forward ``KerasAutoEncoder``, bare or behind one default MinMaxScaler, optionally inside a
    ``TransformedTargetRegressor`` with a default MinMaxScaler transformer; the fit arguments are those ``_canonical`` takes; the
    evaluation's cv is a ``KFold`` that is unshuffled or seeded with an int, so every machine of a bucket gets the same folds.
    """
    import numbers

    from .machine.model.factories.specs import FFNetSpec
    from .machine.model.models import KerasAutoEncoder, KerasRawModelRegressor

    evaluation = {**DEFAULT_EVALUATION, **(machine.get("evaluation") or {})}
    reason = _evaluation_refusal(evaluation)
    if reason:
        return _refuse(machine, reason)
    cv = serializer.from_definition(evaluation.get("cv", DEFAULT_CV))
    if type(cv) is not KFold:
        return _refuse(machine, "a K-fold detector is batched under a KFold cv only")
    if cv.shuffle and (not isinstance(cv.random_state, numbers.Integral) or isinstance(cv.random_state, bool)):
        return _refuse(machine, "a shuffled KFold without an int random_state gives every machine other folds")

    model = serializer.from_definition(machine["model"])
    if not _default_minmax(model.scaler):
        return _refuse(machine, "detector scaler is not a default MinMaxScaler")
    reason = _window_refusal(model)
    if reason:
        return _refuse(machine, reason)
    reason, est, target_scaler = _target_regressor(model.base_estimator)
    if reason:
        return _refuse(machine, reason)
    ae, input_scaler = _network(est, (KerasAutoEncoder, KerasRawModelRegressor))
    if ae is None:
        return _refuse(machine, "the estimator is not a KerasAutoEncoder, bare or behind one default MinMaxScaler")
    reason, fit_args, stopping, vsplit = _ff_fit_arguments(ae, early_stopping)
    if reason:
        return _refuse(machine, reason)

    X, y, dataset_meta, query_sec = _fetch(machine)
    ae.kwargs.update({"n_features": X.shape[1], "n_features_out": y.shape[1]})
    spec = ae._build_spec()
    if not isinstance(spec, FFNetSpec):
        return _refuse(machine, "not a feed-forward network")
    if len(X) != len(y) or len(X) < cv.n_splits:
        return _refuse(machine, "too few rows for the CV folds")
    smallest = len(X) - math.ceil(len(X) / cv.n_splits)  # the training rows of the largest test fold
    if vsplit and math.floor(smallest * (1.0 - vsplit)) < 1:
        return _refuse(machine, f"validation_split {vsplit} leaves a CV fold without a training row")
    reason = _monitor_refusal(stopping, spec, vsplit)
    if reason:
        return _refuse(machine, reason)
    fit, split = _ff_fit(fit_args, model.shuffle, vsplit)
    return _CanonicalKFold(index, machine, model, spec, X, y, dataset_meta, query_sec, fit, cv.n_splits, evaluation, input_scaler, split, stopping,
                           cv=cv, target_scaler=target_scaler)


class FleetModelBuilder:
    """
    Build every machine of a project: ``FleetModelBuilder(machines).build(output_dir)`` -> ``[(model, machine_dict), ...]`` in
    input order, each written to ``<output_dir>/<name>/`` when ``output_dir`` is given.  Results per machine are what
    ``ModelBuilder`` gives (same detector attributes and metadata keys); only the launch count differs.

    ``early_stopping``: also batch feed-forward machines whose estimator has one Keras ``EarlyStopping`` callback on a metric its
    fit reports (``loss``, ``accuracy``, their ``val_*`` forms with a ``validation_split``) -- the reference's production
    definition.  Every fit then applies the rule inside the fit launch (``fleet.build_fleet(early_stopping=...)``).  Off by
    default: such machines then build through ``ModelBuilder``, one epoch launch at a time, as they always have.

    ``kfcv``: also batch ``DiffBasedKFCVAnomalyDetector`` machines under a ``KFold`` cv (``_canonical_kfcv``; the reference's
    production definition), built by ``fleet.build_kfold_fleet``.  Off by default for the same reason: the batched fits draw their
    initial weights per fleet, so without the flag these machines build through ``ModelBuilder`` as before.

    ``lstm_wide_batches``: also batch LSTM machines whose batch_size is above 32 (up to 256), trained by the tensor-core fit
    family (``LSTMEngine.fit_tc``).  Off by default for the same reason: without it such machines build through ``ModelBuilder``,
    whose estimator fit runs the same family one machine at a time.

    ``lstm_early_stopping``: also batch LSTM machines whose estimator has one Keras ``EarlyStopping`` callback on ``loss`` or
    ``accuracy`` (``_canonical_lstm``).  Every fit applies the rule inside its launch (``fleet.build_lstm_fleet(early_stopping=...)``)
    and a fit that stops does no further work.  Off by default for the same reason as ``kfcv``: without it such machines build
    through ``ModelBuilder``, one epoch launch at a time.  It combines with ``lstm_wide_batches``.

    ``ragged``: let machines of different lengths share a bucket (the bucket keys leave out the row count; every other field
    still separates buckets).  Each machine keeps its own CV split, fold blocks, scalers and metadata; the batched builds take
    one row count per machine.  Off by default for the same reason as ``kfcv``: the batched fits draw their initial weights per
    bucket, so merging lengths changes which weights a machine starts from.  Without it buckets, builds and artefacts are
    those of equal-length buckets.

    ``smoothing``: also batch plain feed-forward and LSTM detectors with a smoothing ``window`` (a positive int) and smm / sma / ewma
    ``smoothing_method``.  Every fold's 6-row and window thresholds come from one pass over its scores (``gb_thresholds_pair``),
    and the detectors carry the ``smooth_*`` thresholds and metadata ``ModelBuilder`` gives them.  The window is a bucket field;
    the method is not (it does not enter the thresholds).  Off by default for the same reason as ``kfcv``: without it such
    machines build through ``ModelBuilder`` as before.

    ``target_scaler``: also batch plain feed-forward and LSTM detectors whose estimator is a ``TransformedTargetRegressor`` with a
    default MinMaxScaler transformer and no ``func`` / ``inverse_func`` around a network those paths take (bare or behind one default
    MinMaxScaler) -- the reference's production base estimator under the default ``TimeSeriesSplit`` cv.  Every slot trains on its
    own scaled targets, and the fold models' predictions go through sklearn's float32 inverse and float64 scoring in one launch
    (``gb_minmax_inverse_score_f64``).  The target transformer is a bucket field.  Off by default for the same reason as ``kfcv``: without it such
    machines build through ``ModelBuilder`` as before.  K-fold detectors with a TransformedTargetRegressor are ``kfcv``'s.

    ``mixed_widths``: build feed-forward buckets (plain and K-fold) whose keys differ only in the network's ``dims`` -- machines with
    other tag counts -- together, when their nets share the fit's memory plan (``engine.fit_plan``): every bucket prepares its build,
    their fits go out as one gb_ffae_fit_group launch (``fleet.build_joined``), and every bucket finishes on its own.  Buckets, their
    initial weights and every machine's artefacts are those of the default build; only the fit launches are fewer.  If a joined
    build raises, its buckets build one by one as without the flag.  LSTM buckets are untouched.  Off by default.
    """

    def __init__(self, machines: Sequence, early_stopping: bool = False, kfcv: bool = False, lstm_wide_batches: bool = False,
                 lstm_early_stopping: bool = False, ragged: bool = False, smoothing: bool = False, target_scaler: bool = False,
                 mixed_widths: bool = False):
        self.ragged = bool(ragged)
        self.mixed_widths = bool(mixed_widths)
        self.target_scaler = bool(target_scaler)
        self.smoothing = bool(smoothing)
        self.early_stopping = bool(early_stopping)
        self.kfcv = bool(kfcv)
        self.lstm_wide_batches = bool(lstm_wide_batches)
        self.lstm_early_stopping = bool(lstm_early_stopping)
        self.machines = [_machine_dict(m) for m in machines]
        names = [m["name"] for m in self.machines]
        if len(set(names)) != len(names):
            raise ValueError("machine names must be unique")

    def shard(self, rank: int, world: int) -> "FleetModelBuilder":
        """
        This rank's contiguous block of the project (``fleet.partition``): machines are independent, so a multi-GPU build is
        ``FleetModelBuilder(machines).shard(rank, world).build(output_dir)`` in every process, with no collective at all.
        """
        from . import fleet

        return FleetModelBuilder([self.machines[i] for i in fleet.partition(len(self.machines), world)[rank]], early_stopping=self.early_stopping,
                                 kfcv=self.kfcv, lstm_wide_batches=self.lstm_wide_batches, lstm_early_stopping=self.lstm_early_stopping,
                                 ragged=self.ragged, smoothing=self.smoothing, target_scaler=self.target_scaler, mixed_widths=self.mixed_widths)

    def build(self, output_dir: Optional[str] = None) -> List[Tuple[Any, dict]]:
        results: List[Optional[Tuple[Any, dict]]] = [None] * len(self.machines)
        buckets: Dict[tuple, List[_Canonical]] = {}
        for i, machine in enumerate(self.machines):
            if _is_lstm_definition(machine):
                c = _canonical_lstm(i, machine, wide_batches=self.lstm_wide_batches, early_stopping=self.lstm_early_stopping, smoothing=self.smoothing,
                                    target_scaler=self.target_scaler)
            elif self.kfcv and _is_kfcv_definition(machine):
                c = _canonical_kfcv(i, machine, early_stopping=self.early_stopping)
            else:
                c = _canonical(i, machine, early_stopping=self.early_stopping, smoothing=self.smoothing, target_scaler=self.target_scaler)
            if c is None:
                results[i] = ModelBuilder(machine).build()
            else:
                buckets.setdefault(c.bucket(self.ragged), []).append(c)
        for joined in (launch_groups(buckets) if self.mixed_widths else [[members] for members in buckets.values()]):
            built_buckets = None
            if len(joined) > 1:
                try:
                    built_buckets = self._build_buckets_joined(joined)
                except Exception as exc:  # the buckets still get built, each on its own
                    logger.warning("joined build of %d buckets failed (%s: %s); building them one by one", len(joined), type(exc).__name__, exc)
            for i, members in enumerate(joined):
                if built_buckets is not None:
                    built_bucket = built_buckets[i]
                else:
                    try:
                        built_bucket = self._build_bucket(members)
                    except Exception as exc:  # e.g. an architecture the batched fit kernel cannot hold: the machines still get built, one by one
                        logger.warning("batched build of %d machines failed (%s: %s); building them one at a time", len(members), type(exc).__name__, exc)
                        built_bucket = [ModelBuilder(c.machine).build() for c in members]
                for c, built in zip(members, built_bucket):
                    results[c.index] = built
        if output_dir is not None:
            for model, machine in results:
                serializer.dump(model, os.path.join(output_dir, machine["name"]), metadata=machine)
        return results

    @staticmethod
    def _build_bucket(members: List[_Canonical]) -> List[Tuple[Any, dict]]:
        if isinstance(members[0], _CanonicalLSTM):
            return FleetModelBuilder._build_lstm_bucket(members)
        from . import fleet

        return fleet.build_joined([_ff_bucket_steps(members)])[0]

    @staticmethod
    def _build_buckets_joined(joined: List[List[_Canonical]]) -> List[List[Tuple[Any, dict]]]:
        """Feed-forward buckets of one launch group (``launch_groups``), their fits in one launch (``fleet.build_joined``)."""
        from . import fleet

        out = fleet.build_joined([_ff_bucket_steps(members) for members in joined])
        logger.info("built %d buckets of %d machines with their fits in one launch", len(joined), sum(len(m) for m in joined))
        return out

    @staticmethod
    def _build_lstm_bucket(members: List[_CanonicalLSTM]) -> List[Tuple[Any, dict]]:
        from . import engine, fleet

        first = members[0]
        eng = engine.lstm_engine_for(first.spec)
        t0 = time.time()
        xd, yd = _upload(members, eng.device, float64=True)
        fb = fleet.build_lstm_fleet(eng, xd, yd, [len(c.X) for c in members], lookahead=first.lookahead, epochs=first.fit["epochs"],
                                    batch_size=first.fit["batch_size"], n_splits=first.n_splits, seed=int(first.evaluation.get("seed", 0)),
                                    adam=first.spec.adam, input_scaler=first.input_scaler, loss=first.spec.loss, optimizer=fit_optimizer(first.spec),
                                    early_stopping=_stops(members), window=first.window, target_scaler=first.target_scaler)
        # the first prediction answers row lookback_window - 1 + lookahead
        out = _assemble(members, fb, fb.cv_moments, fb.machine_n_test, eng.lookback - 1 + first.lookahead, TimeSeriesSplit(n_splits=first.n_splits), t0)
        logger.info("built %d LSTM machines in one batched bucket", len(members))
        return out


def _ff_bucket_steps(members: List[_Canonical]):
    """The batched build of a feed-forward bucket (plain or K-fold) as ``fleet.build_joined`` takes it: a generator that yields the
    bucket's fit request, receives the fit's result and returns the machines as ``ModelBuilder`` returns them."""
    from . import engine, fleet

    first = members[0]
    eng = engine.ff_engine_for(first.spec)
    t0 = time.time()
    if isinstance(first, _CanonicalKFold):
        xd, yd = _upload(members, eng.device, float64=True)
        det = first.model
        fb = yield from fleet.build_kfold_fleet.steps(
            eng, xd, yd, [len(c.X) for c in members], first.cv, epochs=first.fit["epochs"], batch_size=first.fit["batch_size"],
            seed=int(first.evaluation.get("seed", 0)), adam=first.spec.adam, shuffle=first.fit["shuffle"], input_scaler=first.input_scaler,
            target_scaler=first.target_scaler, detector_shuffle=first.split[0], validation_split=first.split[1],
            validation_batch_size=first.split[2], early_stopping=_stops(members), window=det.window, smoothing_method=det.smoothing_method,
            threshold_percentile=det.threshold_percentile, loss=first.spec.loss, optimizer=fit_optimizer(first.spec), reg=fit_reg(first.spec),
            dropout=fit_dropout(first.spec))
        out = _assemble(members, fb, fb.cv_moments, fb.n_test, 0, first.cv, t0)  # a Dense stack answers every row
        logger.info("built %d K-fold machines in one batched bucket", len(members))
        return out
    xd, yd = _upload(members, eng.device, float64=first.target_scaler)  # TransformedTargetRegressor.fit hands its transformer float64 targets
    fb = yield from fleet.build_fleet.steps(
        eng, xd, yd, [len(c.X) for c in members], epochs=first.fit["epochs"], batch_size=first.fit["batch_size"], n_splits=first.n_splits,
        seed=int(first.evaluation.get("seed", 0)), adam=first.spec.adam, shuffle=first.fit["shuffle"], input_scaler=first.input_scaler,
        detector_shuffle=first.split[0], validation_split=first.split[1], validation_batch_size=first.split[2], early_stopping=_stops(members),
        loss=first.spec.loss, optimizer=fit_optimizer(first.spec), reg=fit_reg(first.spec), window=first.window,
        dropout=fit_dropout(first.spec), target_scaler=first.target_scaler)
    return _assemble(members, fb, fb.cv_moments.cpu().numpy(), fb.n_test, 0, TimeSeriesSplit(n_splits=first.n_splits), t0)  # a Dense stack answers every row


def launch_groups(buckets: Dict[tuple, List[_Canonical]]) -> List[List[List[_Canonical]]]:
    """
    ``FleetModelBuilder(mixed_widths=True)``'s launch groups: the buckets (in key order of first appearance) whose keys differ only
    in the network's ``dims`` and whose nets share the fit's memory plan, as lists of buckets; LSTM buckets, and buckets whose plan
    the fit refuses, stay alone.
    """
    from . import engine

    groups: Dict[tuple, List[List[_Canonical]]] = {}
    for key, members in buckets.items():
        c = members[0]
        plan = None if isinstance(c, _CanonicalLSTM) else engine.fit_plan(c.spec.dims, c.spec.acts, c.spec.l1)
        join = ("alone", key) if plan is None else (type(c).__name__, key[1:], plan)
        groups.setdefault(join, []).append(members)
    return list(groups.values())


def _upload(members: List[_Canonical], device, float64: bool):
    """The machines' X and y stacked on the device, float64 or float32; y is X when every machine's y is its X."""
    from . import engine

    def stacked(frames):
        if float64:
            return engine._torch().from_numpy(np.concatenate([np.ascontiguousarray(f.values, dtype=np.float64) for f in frames])).to(device)
        return engine.to_device_f32(np.concatenate([np.ascontiguousarray(f.values, dtype=np.float32) for f in frames]), device)

    xd = stacked([c.X for c in members])
    return xd, (xd if all(c.y is c.X for c in members) else stacked([c.y for c in members]))


def _stops(members: List[_Canonical]):
    """The bucket's EarlyStopping callbacks, one per machine, or None without them."""
    return None if members[0].early_stopping is None else [c.early_stopping for c in members]


def _assemble(members: List[_Canonical], fb, moments, n_test, model_offset: int, split_obj, t0: float) -> List[Tuple[Any, dict]]:
    """
    Every machine of a built bucket as ``ModelBuilder`` returns it: the detector from ``fb.detector`` and its metadata, the CV
    scores from the host ``moments`` [M, K, 5, T] over ``n_test[m]`` test rows per fold.  The bucket's wall time since ``t0`` is
    spread evenly: there is no per-machine time any more.
    """
    from . import engine

    engine._torch().cuda.synchronize()
    share = (time.time() - t0) / len(members)
    K = members[0].n_splits
    out = []
    for m, c in enumerate(members):
        tags = list(c.y.columns)
        model = fb.detector(m, tags=tags, template=c.model, input_tags=list(c.X.columns))
        names = [s.rpartition(".")[2] for s in c.evaluation["metrics"]]
        scoring_scale = model.scaler.scale_ if c.evaluation.get("scoring_scaler") else None  # the scoring scaler sees all targets too
        scores = scores_block(scores_from_moments(moments[m], n_test[m], scoring_scale, names), tags)
        model_block = {
            "model_offset": model_offset,
            "model_creation_date": _now(),
            "model_builder_version": __version__,
            "model_training_duration_sec": share * 1.0 / (K + 1),
            "cross_validation": {"scores": scores, "cv_duration_sec": share * K / (K + 1), "splits": build_split_dict(c.X, split_obj)},
            "model_meta": extract_metadata_from_model(model),
        }
        dataset_block = {"query_duration_sec": c.query_sec, "dataset_meta": c.dataset_meta}
        out.append((model, _machine_out(c.machine, {"model": model_block, "dataset": dataset_block})))
    return out


# ------------------------------------------------------------------------------------------------ from a project config
MACHINE_YAML_FIELDS = ("model", "dataset", "evaluation", "metadata", "runtime")  # may arrive as YAML text blocks (machine/constants.py)


def patch_dict(original: dict, patch: dict) -> dict:
    """
    ``original`` with every path of ``patch`` added or replaced, nothing removed (workflow_generator/helpers.py:16-45).  Lists are
    replaced as a whole; the reference patches through dictdiffer [3P, not installed here], which walks lists element by element.
    """
    out = copy.deepcopy(original)
    for key, value in (patch or {}).items():
        if isinstance(value, dict) and isinstance(out.get(key), dict):
            out[key] = patch_dict(out[key], value)
        else:
            out[key] = copy.deepcopy(value)
    return out


class RandomDataset:
    """
    Stand-in for gordo-core's ``RandomDataProvider`` datasets [3P, not installed]: seeded uniform noise for the configured tags on
    the regular ``resolution`` grid between ``train_start_date`` and ``train_end_date``.  It exists so that project configs written
    for the reference's tests and docs (``data_provider: {type: RandomDataProvider}``) build here; real data comes from any object
    with ``get_data()`` passed through ``datasets=``.
    """

    def __init__(self, **config):
        self.config = config
        tags = config.get("tag_list") or config.get("tags")
        if not tags:
            raise ValueError("dataset needs 'tag_list' (or 'tags')")
        self.tag_list = [t["name"] if isinstance(t, dict) else str(t) for t in tags]
        targets = config.get("target_tag_list") or tags
        self.target_tag_list = [t["name"] if isinstance(t, dict) else str(t) for t in targets]
        self.resolution = config.get("resolution", "10min")
        self.start, self.end = pd.Timestamp(config["train_start_date"]), pd.Timestamp(config["train_end_date"])
        if self.start.tzinfo is None or self.end.tzinfo is None:
            raise ValueError("train_start_date / train_end_date need a timezone")
        if self.start >= self.end:
            raise ValueError(f"train_end_date ({self.end}) must be after train_start_date ({self.start})")

    def get_data(self):
        import zlib

        index = pd.date_range(self.start, self.end, freq=pd.tseries.frequencies.to_offset(self.resolution), inclusive="left")
        names = list(dict.fromkeys(self.tag_list + self.target_tag_list))
        rng = np.random.default_rng(zlib.crc32("|".join(names).encode()))
        data = pd.DataFrame(rng.random((len(index), len(names))), index=index, columns=names)
        return data[self.tag_list], data[self.target_tag_list]

    def get_metadata(self):
        return {"tag_list": self.tag_list, "target_tag_list": self.target_tag_list, "resolution": self.resolution,
                "train_start_date": str(self.start), "train_end_date": str(self.end)}

    def to_dict(self):
        out = {k: v for k, v in self.config.items() if k != "tags"}
        out.update({"type": "RandomDataset", "tag_list": self.tag_list, "target_tag_list": self.target_tag_list, "resolution": self.resolution})
        return out


def _dataset_from_config(config: dict):
    provider = (config.get("data_provider") or {}).get("type", "") if isinstance(config.get("data_provider"), dict) else ""
    if str(config.get("type", "")).endswith("RandomDataset") or str(provider).endswith("RandomDataProvider"):
        return RandomDataset(**config)
    raise TypeError("only RandomDataset / RandomDataProvider dataset configs can be instantiated here; pass datasets= (name or machine -> an "
                    "object with get_data()) for real data")


def machines_from_config(config, project_name: str = "local-build", datasets=None) -> List[dict]:
    """
    The machines of a project config -- ``{"machines": [...], "globals": {...}}`` as a dict or YAML text -- in the dict form the
    builders take, with the globals folded in the way ``Machine.from_config`` does (gordo/machine/machine.py:78-149: the machine's
    model wins, runtime and evaluation are globals patched by the machine, dataset is the machine patched by the globals) over
    the default evaluation of ``NormalizedConfig``.  ``datasets``: mapping name -> dataset object, or a callable taking the machine.
    """
    import yaml

    if isinstance(config, str):
        config = yaml.safe_load(config)
    if not isinstance(config, dict) or not config.get("machines"):
        raise ValueError("config needs a non-empty 'machines' list")

    def parsed(block: dict) -> dict:
        out = dict(block or {})
        for field in MACHINE_YAML_FIELDS:
            if isinstance(out.get(field), str):
                out[field] = yaml.safe_load(out[field])
        return out

    config_globals = patch_dict({"evaluation": DEFAULT_EVALUATION}, parsed(config.get("globals")))
    machines = []
    for conf in config["machines"]:
        conf = parsed(conf)
        if "name" not in conf:
            raise ValueError("every machine needs a name")
        model = conf.get("model") or config_globals.get("model")
        if model is None:
            raise ValueError("model is empty")
        machine = {
            "name": conf["name"],
            "project_name": conf.get("project_name") or project_name,
            "model": model,
            "runtime": patch_dict(config_globals.get("runtime") or {}, conf.get("runtime") or {}),
            "evaluation": patch_dict(config_globals.get("evaluation") or {}, conf.get("evaluation") or {"cv_mode": "full_build"}),
            "metadata": {"user_defined": {"global-metadata": config_globals.get("metadata") or {}, "machine-metadata": conf.get("metadata") or {}}},
        }
        dataset_config = patch_dict(conf.get("dataset") or {}, config_globals.get("dataset") or {})
        if callable(datasets):
            machine["dataset"] = datasets({**machine, "dataset": dataset_config})
        elif datasets is not None and conf["name"] in datasets:
            machine["dataset"] = datasets[conf["name"]]
        else:
            machine["dataset"] = _dataset_from_config(dataset_config)
        machines.append(machine)
    return machines


def local_build(config_str, datasets=None, batched: bool = True, early_stopping: bool = False, kfcv: bool = False,
                lstm_wide_batches: bool = False):
    """
    Build the model(s) of a bare gordo config locally and yield ``(model, machine)`` per machine, in config order
    (gordo/builder/local_build.py:15-80).  ``batched=False`` builds one machine at a time like the reference does;
    ``early_stopping``, ``kfcv`` and ``lstm_wide_batches`` are ``FleetModelBuilder``'s.
    """
    machines = machines_from_config(config_str, datasets=datasets)
    if batched:
        yield from FleetModelBuilder(machines, early_stopping=early_stopping, kfcv=kfcv, lstm_wide_batches=lstm_wide_batches).build()
    else:
        for machine in machines:
            yield ModelBuilder(machine).build()
