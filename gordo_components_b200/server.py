"""
The serving side of the hot path without the web framework: what ``POST /gordo/v0/<project>/<name>/anomaly/prediction``
and ``.../prediction`` do between the HTTP layer and ``model.anomaly`` (gordo/server/blueprints/anomaly.py:28-122,
base.py:30-120, utils.py:47-330), as plain functions a Flask / ASGI view can call:

* the wire formats: frames as nested JSON dicts or parquet bytes (``dataframe_to_dict`` / ``dataframe_from_dict`` /
  ``dataframe_into_parquet_bytes`` / ``dataframe_from_parquet_bytes``), and the check of request frames against the model's
  tag list (``verify_dataframe``);
* ``ModelStore``: the models of a project directory kept loaded -- the reference unpickles through ``lru_cache(2)``
  (utils.py:334-353) because a TensorFlow model per machine is heavy; here a model is a few hundred KB of numpy weights whose
  device copy is cached on the estimator, so a whole project stays resident (``max_models`` bounds it if needed);
* ``anomaly_prediction`` / ``prediction``: request payload in, ``Reply(status, body)`` out, with the reference's status
  codes and messages (400 without ``X`` / ``y`` or on unexpected features, 422 when the model is not an anomaly detector).

Many small concurrent requests are better served through ``serving.AnomalyCoalescer`` (one launch for everything that is
waiting); this module is the per-request path and the data formats either way.
"""
import io
import os
import threading
import timeit
from collections import OrderedDict
from typing import Any, Dict, List, Optional, Sequence, Union

import dateutil.parser
import numpy as np
import pandas as pd

from . import serializer
from .machine.model import utils as model_utils

DELETED_FROM_RESPONSE_COLUMNS = (
    "smooth-tag-anomaly-scaled",
    "smooth-total-anomaly-scaled",
    "smooth-tag-anomaly-unscaled",
    "smooth-total-anomaly-unscaled",
)


# ------------------------------------------------------------------------------------------------ wire formats
def dataframe_into_parquet_bytes(df: pd.DataFrame, compression: str = "snappy") -> bytes:
    import pyarrow as pa
    import pyarrow.parquet as pq

    sink = pa.BufferOutputStream()
    pq.write_table(pa.Table.from_pandas(df), sink, compression=compression)
    return sink.getvalue().to_pybytes()


def dataframe_from_parquet_bytes(buf: bytes) -> pd.DataFrame:
    import pyarrow.parquet as pq

    return pq.read_table(io.BytesIO(buf)).to_pandas()


def dataframe_to_dict(df: pd.DataFrame) -> dict:
    """
    JSON-able form of a frame: ``{column: {index: value}}``, and for two-level columns (the anomaly frame)
    ``{top: {sub: {index: value}}}``; a DatetimeIndex is written as strings (utils.py:86-143).  Built column by column from
    plain lists: going through ``DataFrame.__getitem__`` / ``to_dict`` per top-level name, as the reference does, costs
    tens of milliseconds per response -- more than everything else in a small request together.
    """
    keys = (df.index.astype(str) if isinstance(df.index, pd.DatetimeIndex) else df.index).tolist()
    if not isinstance(df.columns, pd.MultiIndex):
        if not df.columns.is_unique:
            return df.set_axis(keys, axis=0).to_dict()
        return {col: dict(zip(keys, series.tolist())) for col, series in df.items()}
    out: dict = {}
    for (top, sub), series in df.items():
        # a lone column with an empty second level comes out under its own top-level name, as ``DataFrame(series).to_dict()`` gives it
        out.setdefault(top, {})[sub if sub != "" else top] = dict(zip(keys, series.tolist()))
    return out


def blocks_to_dict(index, blocks, columns, skip=()) -> dict:
    """``dataframe_to_dict(frame_from_blocks(index, blocks, columns))`` without building the frame (top-level names in ``skip`` left out)."""
    keys = (index.astype(str) if isinstance(index, pd.DatetimeIndex) else index).tolist()
    out: dict = {}
    names = iter(columns)
    for block in blocks:
        values = block.to_numpy() if isinstance(block, pd.DataFrame) else np.asarray(block)
        for j in range(values.shape[1]):
            top, sub = next(names)
            if top not in skip:
                out.setdefault(top, {})[sub if sub != "" else top] = dict(zip(keys, values[:, j].tolist()))
    return out


def _fast_frame(data: dict) -> Optional[pd.DataFrame]:
    """The frame of a well-formed payload -- every column over the same keys in the same order -- or None (the general path decides)."""
    first = next(iter(data.values()))
    if not isinstance(first, dict) or not first:
        return None
    nested = isinstance(next(iter(first.values())), dict)
    columns = {}
    for top, block in data.items():
        if not isinstance(block, dict):
            return None
        if nested:
            for sub, col in block.items():
                if not isinstance(col, dict):
                    return None
                columns[(top, sub)] = col
        else:
            columns[top] = block
    cols = iter(columns.values())
    keys = list(next(cols))
    if not keys or any(isinstance(v, dict) for v in next(iter(columns.values())).values()):
        return None
    for col in cols:
        if list(col) != keys:
            return None
    index = _parse_keys(keys)
    if index is None:
        return None
    frame = pd.DataFrame({name: list(col.values()) for name, col in columns.items()}, index=index)
    return frame if index.is_monotonic_increasing else frame.sort_index()


def _parse_keys(keys: List[str]) -> Optional[pd.Index]:
    """ISO timestamps of one offset (or none) -> DatetimeIndex; anything else is left to the general path."""
    first = keys[0]
    if not (isinstance(first, str) and len(first) >= 10 and first[4] == "-" and first[7] == "-"):
        return None
    try:
        index = pd.to_datetime(keys, format="ISO8601")
    except (ValueError, TypeError):
        return None
    return index.as_unit("us") if isinstance(index, pd.DatetimeIndex) else None


def dataframe_from_dict(data: dict) -> pd.DataFrame:
    """Inverse of ``dataframe_to_dict``; the index is parsed as ISO timestamps, else as integers, and sorted (utils.py:146-191)."""
    if isinstance(data, dict) and data:
        fast = _fast_frame(data)
        if fast is not None:
            return fast
    if isinstance(data, dict) and any(isinstance(v, dict) for v in data.values()):
        try:
            keys = list(data.keys())
            df = pd.concat((pd.DataFrame.from_dict(data[k]) for k in keys), axis=1, keys=keys)
        except (ValueError, AttributeError):
            df = pd.DataFrame.from_dict(data)
    else:
        df = pd.DataFrame.from_dict(data)
    try:
        df.index = df.index.map(dateutil.parser.isoparse)
    except (TypeError, ValueError):
        df.index = df.index.map(int)
    return df.sort_index()


class Reply:
    """What a view returns: an HTTP status and a JSON-able dict or raw (parquet) bytes."""

    def __init__(self, status: int, body: Union[dict, bytes]):
        self.status, self.body = status, body

    @property
    def content_type(self) -> str:
        return "application/octet-stream" if isinstance(self.body, (bytes, bytearray)) else "application/json"

    def __repr__(self):
        return f"Reply({self.status}, {self.content_type})"


def verify_dataframe(df: pd.DataFrame, expected_columns: List[str]) -> Union[pd.DataFrame, Reply]:
    """
    The request frame reduced / relabelled to the model's tags, or a 400 ``Reply`` (utils.py:206-247): unlabelled frames of
    the right width get the expected names, frames that carry all expected names are reordered, anything else is refused.
    """
    if isinstance(df.columns, pd.MultiIndex):
        return Reply(400, {"message": f"Server does not support multi-level dataframes at this time: {df.columns.tolist()}"})
    if list(df.columns) == list(expected_columns):
        return df
    if all(col in df.columns for col in expected_columns):
        return df[expected_columns]
    if len(df.columns) != len(expected_columns):
        return Reply(400, {"message": f"Unexpected features: was expecting {expected_columns} length of {len(expected_columns)}, "
                                      f"but got {df.columns} length of {len(df.columns)}"})
    df = df.copy(deep=False)
    df.columns = expected_columns
    return df


# ------------------------------------------------------------------------------------------------ resident models
def _tag_names(tags) -> List[str]:
    return [t["name"] if isinstance(t, dict) else str(getattr(t, "name", t)) for t in tags or []]


class ModelStore:
    """
    ``<directory>/<name>/{model.pkl, metadata.json}`` (what ``serializer.dump`` and the builders write) kept loaded.
    Thread safe; ``max_models=None`` keeps everything, otherwise least-recently-used models are dropped.
    """

    def __init__(self, directory: str, max_models: Optional[int] = None):
        self.directory, self.max_models = directory, max_models
        self._models: "OrderedDict[str, Any]" = OrderedDict()
        self._metadata: Dict[str, dict] = {}
        self._lock = threading.Lock()

    def names(self) -> List[str]:
        return sorted(d for d in os.listdir(self.directory) if os.path.isfile(os.path.join(self.directory, d, "model.pkl")))

    def model(self, name: str):
        with self._lock:
            if name in self._models:
                self._models.move_to_end(name)
                return self._models[name]
        path = os.path.join(self.directory, name)
        if not os.path.isfile(os.path.join(path, "model.pkl")):
            raise FileNotFoundError(f"No such model found: '{name}'")
        model = serializer.load(path)
        with self._lock:
            self._models[name] = model
            while self.max_models is not None and len(self._models) > self.max_models:
                self._models.popitem(last=False)
        return model

    def metadata(self, name: str) -> dict:
        with self._lock:
            if name in self._metadata:
                return self._metadata[name]
        meta = serializer.load_metadata(os.path.join(self.directory, name))
        with self._lock:
            self._metadata[name] = meta
        return meta

    def tags(self, name: str) -> List[str]:
        return _tag_names(self.metadata(name).get("dataset", {}).get("tag_list"))

    def target_tags(self, name: str) -> List[str]:
        dataset = self.metadata(name).get("dataset", {})
        return _tag_names(dataset.get("target_tag_list")) or self.tags(name)

    def frequency(self, name: str):
        resolution = self.metadata(name).get("dataset", {}).get("resolution")
        return None if resolution is None else pd.tseries.frequencies.to_offset(resolution)


class ResidentBucket:
    """
    The models of a store that share one feed-forward architecture, served through ONE ``serving.AnomalyCoalescer``: their weights,
    scaler slopes and thresholds sit packed on the device, and whatever requests are waiting -- from any thread, for any of the
    models -- become one fused launch.  Eligible: this package's ``DiffBasedAnomalyDetector`` around a bare ``KerasAutoEncoder``
    (an affine error scaler, no smoothing window unless ``smoothing=True``); pass ``bucket=`` to ``anomaly_prediction`` and every eligible model is answered
    through it, the rest as before.  The replies are the same bytes either way (rows are independent in the kernel).

    ``input_scalers=True`` also admits the definition the reference's examples deploy, a ``Pipeline`` of per-feature scalers
    (MinMaxScaler, StandardScaler, RobustScaler, MaxAbsScaler) ending in a ``KerasAutoEncoder``: the composed float64 scaler of
    each model rides with its weights, and the launch applies it as it reads X (``serving.AnomalyCoalescer(x_scale=, x_offset=)``).
    Bare and Pipeline models never share a bucket.

    ``lstm=True`` builds a bucket of LSTM detectors instead, served through ``serving.LSTMAnomalyCoalescer``: a
    ``KerasLSTMAutoEncoder`` or ``KerasLSTMForecast``, bare or as the last step of a ``Pipeline``, on a stack the tensor-core LSTM
    kernel runs (tanh and sigmoid cells).  The Pipeline's leading steps run on the host as ``Pipeline.predict`` runs them; autoencoder
    and forecast models of one architecture share a bucket (the lookahead only decides which rows of y a request stages).
    With ``target_scaler=True`` it also admits those networks as the ``regressor_`` of a fitted ``TransformedTargetRegressor`` (the
    same MinMax transformer condition as below); any leading Pipeline steps are admitted, since they run on the host either way.  The
    batch applies each model's target inverse and scores in float64 in one launch (``serving.LSTMAnomalyCoalescer(y_inverse=)``).

    ``smoothing=True`` (with either of the above) also admits detectors with a smoothing window -- ``DiffBasedAnomalyDetector`` with
    ``window`` and ``DiffBasedKFCVAnomalyDetector``, the reference's production definition (``window=144``, smm) -- whose ``window``
    is a positive int and whose ``smoothing_method`` is smm, sma or ewma (a median window of at most ``serving.SMM_MAX_WINDOW``).
    Models are grouped by window and method as well, and windowed and unwindowed models never share a bucket.  A reply that carries
    the ``smooth-*`` columns (``all_columns=True``) gets them from one smoothing launch over the batch's requests that asked; a
    request whose y holds a NaN and that asks for them is answered per request, where pandas' totals of those rows are recomputed
    on the host before they are smoothed.

    ``target_scaler=True`` (with any of the feed-forward flags) also admits detectors whose base estimator is a fitted
    ``TransformedTargetRegressor(transformer=MinMaxScaler(), regressor=...)`` without ``func`` / ``inverse_func`` -- the reference's
    production definition -- around a bare ``KerasAutoEncoder`` or, with ``input_scalers=True``, a ``Pipeline([MinMaxScaler(),
    KerasAutoEncoder])``.  The coalescer predicts, then applies each model's target inverse and scores in float64 in one launch
    (``serving.AnomalyCoalescer(y_inverse=)``), as the per-request route does with sklearn's ``inverse_transform`` and
    gb_anomaly_score_f64.  Other input scalers stay on the per-request route inside a TransformedTargetRegressor: sklearn's
    ``Pipeline.predict`` runs their subtract-and-divide transform there, which the composed affine scaler of the launch does not
    round the same way.  Models with and without a target transformer never share a bucket.
    """

    input_scalers = False  # the bucket holds Pipeline models (set by the constructor)
    lstm = False  # the bucket holds LSTM models (set by the constructor)
    smoothing = None  # (window, method) of the bucket's windowed detectors (set by the constructor)
    target_scaler = False  # the bucket holds TransformedTargetRegressor models (set by the constructor)

    def __init__(self, store: "ModelStore", names: Optional[List[str]] = None, input_scalers: bool = False, lstm: bool = False,
                 smoothing: bool = False, target_scaler: bool = False, **coalescer_kwargs):
        from . import engine, serving
        from .machine.model.anomaly.diff import _compose_affine, _scaler_multiplier

        candidates = {name: store.model(name) for name in (names if names is not None else store.names())}
        groups = (self.lstm_groups(candidates, smoothing, target_scaler) if lstm
                  else self.ff_groups(candidates, input_scalers, smoothing, target_scaler))
        if not groups:
            raise ValueError(f"no {'LSTM ' if lstm else ''}model in the store can be served through a coalescer")
        self.lstm = lstm
        self.names = max(groups.values(), key=len)  # the largest architecture group
        self.slot = {name: i for i, name in enumerate(self.names)}
        models = [store.model(n) for n in self.names]
        parts = [_served_parts(m, lstm) for m in models]
        eng = (engine.lstm_engine_for if lstm else engine.ff_engine_for)(parts[0][1].model.spec)
        torch = engine._torch()
        params = eng.pack_params([net.model.weights for _, net in parts])
        self.target_scaler = _target_minmax(models[0]) is not None
        # LSTM scores, and those of a target inverse, are float64, as on the per-request route
        dt = np.float64 if lstm or self.target_scaler else np.float32
        to_dev = lambda rows, dt=dt: torch.from_numpy(np.ascontiguousarray(np.stack(rows), dtype=dt)).to(eng.device)  # noqa: E731
        scale = to_dev([_scaler_multiplier(m.scaler, eng.n_out) for m in models])
        feat, agg = zip(*(m._thresholds() for m in models))
        feat_thr = to_dev([np.asarray(f, dtype=dt) for f in feat]) if feat[0] is not None else None
        agg_thr = to_dev([dt(a) for a in agg]) if agg[0] is not None else None
        if self.target_scaler:
            y_scale, y_min = zip(*(_target_minmax(m) for m in models))
            coalescer_kwargs.update(y_inverse=(to_dev(y_scale, np.float64), to_dev(y_min, np.float64)))
        self.input_scalers = not lstm and bool(parts[0][0])  # an LSTM Pipeline's leading steps run on the host
        if self.input_scalers:
            a, b = zip(*(_compose_affine(pre, eng.n_in) for pre, _ in parts))
            coalescer_kwargs.update(x_scale=to_dev(a, np.float64), x_offset=to_dev(b, np.float64))
        self.smoothing = _smoothing_of(models[0])
        coalescer = serving.LSTMAnomalyCoalescer if lstm else serving.AnomalyCoalescer
        self.coalescer = coalescer(eng, params, scale, feat_thr, agg_thr, smoothing=self.smoothing, **coalescer_kwargs)

    @classmethod
    def ff_groups(cls, models: Dict[str, Any], input_scalers: bool = False, smoothing: bool = False,
                  target_scaler: bool = False) -> Dict[Any, List[str]]:
        """The eligible feed-forward detectors of ``models`` (name -> model) by (architecture, bare or Pipeline, which thresholds
        are present, with or without a target transformer, smoothing)."""
        def arch(model):
            pre, ae = _served_parts(model)
            spec = ae.model.spec
            return tuple(spec.dims), tuple(spec.acts), tuple(spec.l1), bool(pre)

        return _groups(models, lambda m: cls.eligible(m, input_scalers, smoothing, target_scaler), arch)

    @classmethod
    def lstm_groups(cls, models: Dict[str, Any], smoothing: bool = False, target_scaler: bool = False) -> Dict[Any, List[str]]:
        """The eligible LSTM detectors of ``models`` (name -> model) by (architecture, which thresholds are present, with or without
        a target transformer, smoothing)."""
        return _groups(models, lambda m: cls.eligible_lstm(m, smoothing, target_scaler), lambda m: (_served_parts(m, True)[1].model.spec.key(),))

    @staticmethod
    def eligible_lstm(model, smoothing: bool = False, target_scaler: bool = False) -> bool:
        """True for a detector ``ResidentBucket(lstm=True, smoothing=smoothing, target_scaler=target_scaler)`` serves (no device
        needed)."""
        import ctypes as C

        from . import _cabi

        parts = _admitted_parts(model, True, smoothing, target_scaler)
        if parts is None:
            return False
        spec = parts[1].model.spec
        net = _cabi.make_lstmnet(spec.n_features, spec.lstm_units, spec.acts, spec.n_features_out, spec.out_func, spec.lookback_window)
        if _cabi.load_library().gb_lstm_tc_supported(C.byref(net)) != 0:
            return False  # relu / linear cells: the fp32 kernel, on the per-request route
        return _error_scaler_is_affine(model, spec.n_features_out)

    @staticmethod
    def eligible(model, input_scalers: bool = False, smoothing: bool = False, target_scaler: bool = False) -> bool:
        """True for a detector ``ResidentBucket(input_scalers=input_scalers, smoothing=smoothing, target_scaler=target_scaler)``
        serves (no device needed)."""
        from sklearn.compose import TransformedTargetRegressor
        from sklearn.preprocessing import MinMaxScaler

        from .machine.model.anomaly.diff import _compose_affine

        parts = _admitted_parts(model, False, smoothing, target_scaler)
        if parts is None or (parts[0] and not input_scalers):
            return False
        pre, ae = parts
        if pre and (_compose_affine(pre, ae.model.spec.dims[0]) is None or not _x64_launch_holds(ae.model.spec)):
            return False  # served per request: sklearn's own transform, or the separate gb_affine_f64 pass
        if pre and type(model.base_estimator) is TransformedTargetRegressor and not (len(pre) == 1 and type(pre[0]) is MinMaxScaler):
            return False  # other scalers subtract and divide in sklearn's Pipeline.predict, which the composed affine does not round alike
        return _error_scaler_is_affine(model, ae.model.spec.dims[-1])

    def anomaly_blocks(self, store: "ModelStore", name: str, X: pd.DataFrame, y: pd.DataFrame, frequency=None, smooth: bool = True):
        """``model.anomaly_blocks(X, y, frequency, smooth)`` of the bucket's model ``name``, through the coalescer."""
        from .machine.model.anomaly.diff import _has_inf, _refuse_infinity, _values

        model = store.model(name)
        _refuse_infinity(_values(y))
        smooth = smooth and self.smoothing is not None
        if smooth and np.isnan(np.asarray(_values(y), dtype=np.float64)).any():
            # the rows of a missing target get pandas' totals on the host, and those are what is smoothed: this request goes on its own
            return model.anomaly_blocks(X, y, frequency=frequency, smooth=True)
        if self.lstm:
            return self._lstm_anomaly_blocks(name, model, X, y, frequency, smooth)
        if self.input_scalers:
            # what the Pipeline's sklearn steps raise, as the per-request route does before any launch
            _refuse_infinity(np.ascontiguousarray(_values(X), dtype=np.float64))
        elif _has_inf(_values(X)):
            # the coalescer's launch may run the tensor-core kernel, which does not take ±inf inputs: this request goes on its own
            return model.anomaly_blocks(X, y, frequency=frequency, smooth=smooth)
        scores = self._scores(name, X, y, smooth)
        return model.blocks_from_scores(scores, X, y, frequency, smooth=smooth)

    def _scores(self, name: str, X, y, smooth: bool):
        """The coalescer's result for one request, refused as the per-request route refuses its model output; ``smooth`` is only
        passed when set, the call of a bucket without smoothing stays ``anomaly(slot, X, y)``."""
        from .machine.model.anomaly.diff import _has_inf, _refuse_infinity

        scores = self.coalescer.anomaly(self.slot[name], X, y, smooth=True) if smooth else self.coalescer.anomaly(self.slot[name], X, y)
        raw = scores.pop("raw-model-output", None)
        if raw is not None and _has_inf(raw):
            # what sklearn's inverse_transform raises on the regressor's prediction, before the per-request route's own check
            raise ValueError(f"Input contains infinity or a value too large for {raw.dtype!r}.")
        _refuse_infinity(scores["model-output"])
        return scores

    def _lstm_anomaly_blocks(self, name: str, model, X: pd.DataFrame, y: pd.DataFrame, frequency, smooth: bool):
        """What ``model.anomaly_blocks`` computes, in the order the per-request route raises: the leading steps' transform (which
        refuses ±inf in X), the lookback check; a transformed X holding ±inf goes on its own (the fp32 kernel saturates the gates).
        Around a TransformedTargetRegressor, the inverse's refusals follow the launch (``_scores``)."""
        from .machine.model.anomaly.diff import _has_inf, _values

        pre, net = _served_parts(model, lstm=True)
        Xt = X
        for step in pre:
            if step is not None and step != "passthrough":  # skipped, as Pipeline.predict skips them
                Xt = step.transform(Xt)
        Xv = net._validate_and_fix_size_of_X(np.asarray(_values(Xt)))
        if _has_inf(Xv):
            return model.anomaly_blocks(X, y, frequency=frequency, smooth=smooth)
        n = len(Xv) - net.lookback_window + 1 - net.lookahead
        scores = self._scores(name, Xv, _values(y)[-n:], smooth)
        return model.blocks_from_scores(scores, X, y, frequency, smooth=smooth)

    def close(self):
        self.coalescer.close()


# ------------------------------------------------------------------------------------------------ the two POST views
def _extract_X_y(store: ModelStore, name: str, json: Optional[dict], files: Optional[Dict[str, bytes]]):
    """(X, y) frames of a request -- JSON ``{"X": ..., "y": ...}`` or parquet parts -- or a 400 ``Reply`` (utils.py:250-330)."""
    payload = json if json is not None else (files or {})
    if "X" not in payload:
        return Reply(400, {"message": 'Cannot predict without "X"'})
    load = dataframe_from_dict if json is not None else dataframe_from_parquet_bytes
    X = load(payload["X"])
    y = payload.get("y")
    if y is not None:
        y = load(y)
    tags, targets = store.tags(name), store.target_tags(name)
    X = verify_dataframe(X, tags) if tags else X
    if isinstance(X, Reply):
        return X
    if y is not None and targets:
        y = verify_dataframe(y, targets)
        if isinstance(y, Reply):
            return y
    return X, y


def _served_parts(model, lstm: bool = False):
    """(leading Pipeline steps, network) of a detector whose base estimator is a bare network ([] for the steps) or a ``Pipeline``
    ending in one, else None: a ``KerasAutoEncoder``, or with ``lstm`` a ``KerasLSTMAutoEncoder`` / ``KerasLSTMForecast``.  For a
    fitted ``TransformedTargetRegressor`` these are the parts of its ``regressor_`` (its target transformer: ``_target_minmax``).
    A ``KerasRawModelRegressor`` is served as an autoencoder is: it is a Dense stack too, and inference does not see its weight
    regularizers."""
    from sklearn.compose import TransformedTargetRegressor
    from sklearn.pipeline import Pipeline

    from .machine.model.models import KerasAutoEncoder, KerasLSTMAutoEncoder, KerasLSTMForecast, KerasRawModelRegressor

    served = (KerasLSTMAutoEncoder, KerasLSTMForecast) if lstm else (KerasAutoEncoder, KerasRawModelRegressor)
    est = model.base_estimator
    if type(est) is TransformedTargetRegressor:
        est = getattr(est, "regressor_", None)
    if type(est) in served:
        return [], est
    if type(est) is Pipeline and len(est.steps) > 1 and type(est.steps[-1][1]) in served:
        return [step for _, step in est.steps[:-1]], est.steps[-1][1]
    return None


def _admitted_parts(model, lstm: bool, smoothing: bool, target_scaler: bool):
    """``_served_parts(model, lstm)`` of a detector that passes the checks both kinds of bucket make, else None: this package's
    ``anomaly``, a smoothing window the bucket takes (``_window_served``), the thresholds it requires, a fitted network, and around
    a ``TransformedTargetRegressor`` (only with ``target_scaler``) a MinMax target transformer as wide as the network's output."""
    from sklearn.compose import TransformedTargetRegressor

    if not (_frame_is_from_blocks(model) and _window_served(model, smoothing)
            and not (model.require_thresholds and all(t is None for t in model._thresholds()))):
        return None
    parts = _served_parts(model, lstm)
    if parts is None or parts[1].model is None:
        return None
    if type(model.base_estimator) is TransformedTargetRegressor:
        spec = parts[1].model.spec
        target = _target_minmax(model)
        if not target_scaler or target is None or target[0].shape != ((spec.n_features_out if lstm else spec.dims[-1]),):
            return None
    return parts


def _error_scaler_is_affine(model, n_out: int) -> bool:
    """True when the detector's error scaler is affine per feature.  A detector with any other (clip=True, QuantileTransformer, ...)
    is served on the per-request route, not refused for the whole store."""
    from .machine.model.anomaly.diff import _scaler_multiplier

    try:
        _scaler_multiplier(model.scaler, n_out)
    except (ValueError, AttributeError):
        return False
    return True


def _groups(models: Dict[str, Any], eligible, arch) -> Dict[Any, List[str]]:
    """The names of the ``eligible`` detectors of ``models`` grouped by ``arch(model)`` + (which thresholds are present, with or
    without a target transformer, smoothing), in the order of ``models``."""
    groups: Dict[Any, List[str]] = {}
    for name, model in models.items():
        if eligible(model):
            key = arch(model) + (tuple(t is not None for t in model._thresholds()), _target_minmax(model) is not None, _smoothing_of(model))
            groups.setdefault(key, []).append(name)
    return groups


def _target_minmax(model):
    """(scale_, min_) as float64 arrays of the target transformer of a detector whose base estimator is a fitted
    ``TransformedTargetRegressor`` without ``func`` / ``inverse_func`` whose ``transformer_`` is exactly a ``MinMaxScaler`` (what
    gb_minmax_inverse_score_f64 applies), else None."""
    from sklearn.compose import TransformedTargetRegressor
    from sklearn.preprocessing import MinMaxScaler

    est = model.base_estimator
    if type(est) is not TransformedTargetRegressor or est.func is not None or est.inverse_func is not None:
        return None
    tr = getattr(est, "transformer_", None)
    if type(tr) is not MinMaxScaler or getattr(est, "_training_dim", None) != 2:
        return None  # a 1-D target comes back squeezed from predict
    scale, mn = getattr(tr, "scale_", None), getattr(tr, "min_", None)
    if scale is None or mn is None or np.ndim(scale) != 1 or np.shape(scale) != np.shape(mn):
        return None
    return np.ascontiguousarray(scale, dtype=np.float64), np.ascontiguousarray(mn, dtype=np.float64)


def _smoothing_of(model):
    """None for a detector without a smoothing window; (window, method) for one whose smoothing the coalescers run (a positive int
    window, smm / sma / ewma, a median window the kernel holds); False for any other."""
    from .engine import SMOOTH_METHODS
    from .serving import SMM_MAX_WINDOW

    window, method = model.window, model.smoothing_method
    if window is None:
        return None
    if isinstance(window, bool) or not isinstance(window, (int, np.integer)) or window < 1 or method not in SMOOTH_METHODS \
            or (method == "smm" and window > SMM_MAX_WINDOW):
        return False
    return int(window), method


def _window_served(model, smoothing: bool) -> bool:
    """True when a bucket built with ``smoothing`` takes the detector's smoothing window (or it has none)."""
    s = _smoothing_of(model)
    return s is None or (smoothing and s is not False)


def _x64_launch_holds(spec) -> bool:
    """True when the fused launch with float64 x holds this stack on the kernel the per-request route picks (no device needed)."""
    import ctypes as C

    from . import _cabi

    lib = _cabi.load_library()
    return lib.gb_ffae_infer_plan_x64(C.byref(_cabi.make_ffnet(spec.dims, spec.acts, spec.l1)), 0, None, None) == 0


def _frame_is_from_blocks(model) -> bool:
    """True when ``model.anomaly`` is this package's own (not overridden in a subclass): then ``anomaly_blocks`` is the same result."""
    from .machine.model.anomaly.diff import DiffBasedAnomalyDetector

    return isinstance(model, DiffBasedAnomalyDetector) and type(model).anomaly is DiffBasedAnomalyDetector.anomaly \
        and type(model).anomaly_blocks is DiffBasedAnomalyDetector.anomaly_blocks


def _respond(frame: pd.DataFrame, fmt: Optional[str], start: float) -> Reply:
    if fmt == "parquet":
        return Reply(200, dataframe_into_parquet_bytes(frame))
    return Reply(200, {"data": dataframe_to_dict(frame), "time-seconds": f"{timeit.default_timer() - start:.4f}"})


def anomaly_prediction(store: ModelStore, name: str, json: Optional[dict] = None, files: Optional[Dict[str, bytes]] = None,
                       all_columns: bool = False, fmt: Optional[str] = None,
                       bucket: Union[ResidentBucket, Sequence[ResidentBucket], None] = None) -> Reply:
    """
    ``POST .../<name>/anomaly/prediction`` (anomaly.py:28-122): the anomaly frame of the request's X against its y.  With ``bucket``
    the models it holds are scored through its request coalescer (one launch for everything that is waiting); a sequence of buckets
    (say a feed-forward and an LSTM one over the same store) is asked in order, and the first that holds the model answers.
    """
    start = timeit.default_timer()
    try:
        model = store.model(name)
    except FileNotFoundError as e:
        return Reply(404, {"message": str(e)})
    xy = _extract_X_y(store, name, json, files)
    if isinstance(xy, Reply):
        return xy
    X, y = xy
    if y is None:
        return Reply(400, {"message": "Cannot perform anomaly without 'y' to compare against."})
    not_a_detector = Reply(422, {"message": f"Model is not an AnomalyDetector, it is of type: {type(model)}"})
    if not hasattr(type(model), "anomaly"):
        return not_a_detector
    skip = () if all_columns else DELETED_FROM_RESPONSE_COLUMNS
    try:
        buckets = () if bucket is None else (bucket,) if isinstance(bucket, ResidentBucket) else tuple(bucket)
        holder = next((b for b in buckets if name in b.slot), None)
        if holder is not None or _frame_is_from_blocks(model):
            # this package's detectors: straight from the column blocks (no DataFrame in between for JSON), the smoothed ones only
            # when the reply carries them
            blocks = (holder.anomaly_blocks(store, name, X, y, store.frequency(name), smooth=all_columns) if holder is not None
                      else model.anomaly_blocks(X, y, frequency=store.frequency(name), smooth=all_columns))
            if fmt != "parquet":
                return Reply(200, {"data": blocks_to_dict(*blocks, skip=skip), "time-seconds": f"{timeit.default_timer() - start:.4f}"})
            frame = model_utils.frame_from_blocks(*blocks)
        else:
            frame = model.anomaly(X, y, frequency=store.frequency(name))
    except AttributeError:  # as the reference: also what a detector without its required thresholds answers (anomaly.py:46-52)
        return not_a_detector
    dropped = [c for c in frame.columns if c[0] in skip]
    if dropped:
        frame = frame.drop(columns=dropped)
    return _respond(frame, fmt, start)


def prediction(store: ModelStore, name: str, json: Optional[dict] = None, files: Optional[Dict[str, bytes]] = None,
               fmt: Optional[str] = None) -> Reply:
    """``POST .../<name>/prediction`` (base.py:30-120): model input and output side by side, no scoring."""
    start = timeit.default_timer()
    try:
        model = store.model(name)
    except FileNotFoundError as e:
        return Reply(404, {"message": str(e)})
    xy = _extract_X_y(store, name, json, files)
    if isinstance(xy, Reply):
        return xy
    X, _ = xy
    try:
        output = model.predict(X) if hasattr(type(model), "predict") or hasattr(model, "predict") else model.transform(X)
    except ValueError as err:
        return Reply(400, {"error": f"ValueError: {err}"})
    except Exception:  # the reference answers every other failure of the model the same way (base.py:83-91)
        return Reply(400, {"error": "Something unexpected happened; check your input data"})
    frame = model_utils.make_base_dataframe(tags=store.tags(name) or list(X.columns), model_input=X.values, model_output=output,
                                            target_tag_list=store.target_tags(name) or None, index=X.index)
    return _respond(frame, fmt, start)
