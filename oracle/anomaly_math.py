"""
TEST INFRASTRUCTURE ONLY -- CPU restatement (NumPy/pandas, float64) of the anomaly half
of the gordo hot path.  Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
cpu_baseline / ``--impl reference`` legs may import this module.

PARITY STATUS: **pinned.**  Every function here is checked against outputs of the
reference's own, unmodified ``gordo/machine/model/anomaly/diff.py`` executed from
the reference project (``oracle/reference_loader.py``; fixtures committed under
``tests/golden/`` by ``tests/golden/make_golden.py``), and against the formula pins in
``tests/gordo/machine/model/anomaly/test_anomaly_detectors.py:94-110, 252-348``.

Reference lines restated:
  scaler fit on y after training            diff.py:166-174  (+ sklearn MinMaxScaler [3P 1.5.2])
  per-fold thresholds rolling(6).min().max() diff.py:213-233, final = last fold :257-264
  scaled mse per timestep                   diff.py:268-293
  absolute error                            diff.py:295-300
  smoothing smm / sma / ewma                diff.py:302-308
  anomaly frame arithmetic                  diff.py:350-385, 420-444
  frame assembly + tail alignment           gordo/machine/model/utils.py:49-165
  TimeSeriesSplit geometry                  sklearn [3P] as used at diff.py:181, build_model.py:257-262
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np
import pandas as pd

# ------------------------------------------------------------------ scalers


def minmax_fit(y: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """sklearn MinMaxScaler(feature_range=(0,1)).fit: scale_ = 1/(max-min) with zero ranges -> 1; min_ = -min*scale_."""
    y = np.asarray(y, dtype=np.float64)
    lo, hi = np.nanmin(y, axis=0), np.nanmax(y, axis=0)
    rng = hi - lo
    rng = np.where(rng < 10 * np.finfo(np.float64).eps, 1.0, rng)
    scale = 1.0 / rng
    return scale, -lo * scale


def minmax_transform(v: np.ndarray, scale: np.ndarray, min_: np.ndarray) -> np.ndarray:
    return np.asarray(v) * scale + min_


# ------------------------------------------------------------------ CV geometry


def time_series_split(n_samples: int, n_splits: int = 3) -> List[Tuple[np.ndarray, np.ndarray]]:
    """sklearn TimeSeriesSplit(n_splits) with default test_size/gap: test_size = n // (n_splits+1)."""
    test_size = n_samples // (n_splits + 1)
    if test_size == 0:
        raise ValueError("Too many splits for number of samples")
    idx = np.arange(n_samples)
    out = []
    for test_start in range(n_samples - n_splits * test_size, n_samples, test_size):
        out.append((idx[:test_start], idx[test_start : test_start + test_size]))
    return out


# ------------------------------------------------------------------ rolling statistics (pandas semantics)


def rolling_min_then_max(a: np.ndarray, window: int) -> np.ndarray:
    """column-wise  a.rolling(window).min().max()  (min_periods=window; leading NaNs skipped by max)."""
    a = np.asarray(a, dtype=np.float64)
    one_d = a.ndim == 1
    if one_d:
        a = a[:, None]
    n = a.shape[0]
    if n < window:
        res = np.full(a.shape[1], np.nan)
    else:
        win = np.lib.stride_tricks.sliding_window_view(a, window, axis=0)  # [n-w+1, cols, w]
        mins = win.min(axis=-1)  # a window holding a NaN gives NaN (pandas rolling min with min_periods=window) ...
        with np.errstate(all="ignore"), __import__("warnings").catch_warnings():
            __import__("warnings").simplefilter("ignore", RuntimeWarning)
            res = np.nanmax(mins, axis=0)  # ... which DataFrame.max() skips; a column without one complete window stays NaN
    return res[0] if one_d else res


def smoothing(metric: np.ndarray, window: int, method: str) -> np.ndarray:
    """diff.py:302-308 -- smm rolling median, sma rolling mean (first window-1 rows NaN), ewma ewm(span).mean() (adjust=True)."""
    a = np.asarray(metric, dtype=np.float64)
    one_d = a.ndim == 1
    if one_d:
        a = a[:, None]
    n = a.shape[0]
    out = np.full(a.shape, np.nan)
    if method in ("smm", "sma"):
        if n >= window:
            win = np.lib.stride_tricks.sliding_window_view(a, window, axis=0)
            out[window - 1 :] = np.median(win, axis=-1) if method == "smm" else win.mean(axis=-1)
    elif method == "ewma":
        # pandas/_libs/window/aggregations.pyx ewm() [3P, pandas 1.5.3]: adjust=True, ignore_na=False, min_periods=0 -- a NaN adds no
        # observation but ages the weights, the previous average is carried forward, leading NaNs stay NaN
        alpha = 2.0 / (window + 1.0)
        for c in range(a.shape[1]):
            weighted, old_wt = a[0, c] if n else np.nan, 1.0
            if n:
                out[0, c] = weighted
            for t in range(1, n):
                cur = a[t, c]
                if weighted == weighted:
                    old_wt *= 1.0 - alpha
                    if cur == cur:
                        if weighted != cur:
                            weighted = (old_wt * weighted + cur) / (old_wt + 1.0)
                        old_wt += 1.0
                elif cur == cur:
                    weighted = cur
                out[t, c] = weighted
    else:
        raise ValueError(method)
    return out[:, 0] if one_d else out


# ------------------------------------------------------------------ thresholds (cross_validate)


def fold_thresholds(y_true: np.ndarray, y_pred: np.ndarray, scale: np.ndarray, min_: np.ndarray, window: int = 6):
    """
    One fold of DiffBasedAnomalyDetector.cross_validate (diff.py:213-233):
    returns (feature_thresholds [T], aggregate_threshold scalar).
    ``y_true`` must already be tail-aligned to ``y_pred`` (diff.py:218-219).
    """
    y_true = np.asarray(y_true, dtype=np.float64)
    y_pred64 = np.asarray(y_pred, dtype=np.float64)
    scaled_mse = ((minmax_transform(y_pred64, scale, min_) - minmax_transform(y_true, scale, min_)) ** 2).mean(axis=1)
    mae = np.abs(y_true - y_pred64)
    return rolling_min_then_max(mae, window), float(rolling_min_then_max(scaled_mse, window))


# ------------------------------------------------------------------ anomaly()


def row_mean_skipna(a: np.ndarray) -> np.ndarray:
    """``DataFrame.mean(axis=1)`` (diff.py:366, :383): NaN cells are skipped, a row without any value is NaN.  Only the rows whose
    plain mean is NaN are recomputed, so all-finite data costs one mean and one NaN scan."""
    m = a.mean(axis=1)
    bad = np.isnan(m)
    if bad.any():
        sub = a[bad]
        cnt = (~np.isnan(sub)).sum(axis=1)
        with np.errstate(invalid="ignore", divide="ignore"):
            m[bad] = np.where(cnt > 0, np.nansum(sub, axis=1) / cnt, np.nan)
    return m


def anomaly_arrays(
    y_pred: np.ndarray,
    y: np.ndarray,
    scale: np.ndarray,
    min_: np.ndarray,
    feature_thresholds: Optional[np.ndarray] = None,
    aggregate_threshold: Optional[float] = None,
    window: Optional[int] = None,
    smoothing_method: Optional[str] = None,
) -> Dict[str, np.ndarray]:
    """
    diff.py:350-444 on arrays.  ``y`` is tail-aligned to ``len(y_pred)`` here (:359, :374).
    Note (diff.py:421): anomaly-confidence divides the *unscaled* abs diff by the feature thresholds.
    """
    y_pred = np.asarray(y_pred)
    n = len(y_pred)
    y = np.asarray(y, dtype=np.float64)[-n:]
    pred64 = y_pred.astype(np.float64)
    out: Dict[str, np.ndarray] = {"model-output": y_pred}
    tag_scaled = np.abs(minmax_transform(pred64, scale, min_) - minmax_transform(y, scale, min_))
    out["tag-anomaly-scaled"] = tag_scaled
    out["total-anomaly-scaled"] = row_mean_skipna(np.square(tag_scaled))
    tag_unscaled = np.abs(pred64 - y)
    out["tag-anomaly-unscaled"] = tag_unscaled
    out["total-anomaly-unscaled"] = row_mean_skipna(np.square(tag_unscaled))
    if window is not None and smoothing_method is not None:
        out["smooth-tag-anomaly-scaled"] = smoothing(tag_scaled, window, smoothing_method)
        out["smooth-total-anomaly-scaled"] = smoothing(out["total-anomaly-scaled"], window, smoothing_method)
        out["smooth-tag-anomaly-unscaled"] = smoothing(tag_unscaled, window, smoothing_method)
        out["smooth-total-anomaly-unscaled"] = smoothing(out["total-anomaly-unscaled"], window, smoothing_method)
    if feature_thresholds is not None:
        out["anomaly-confidence"] = tag_unscaled / np.asarray(feature_thresholds, dtype=np.float64)
    if aggregate_threshold is not None:
        out["total-anomaly-confidence"] = out["total-anomaly-scaled"] / aggregate_threshold
    return out


# ------------------------------------------------------------------ frame assembly (model/utils.py:49-165)


def base_frame(tags, model_input, model_output, target_tag_list=None, index=None, frequency=None) -> pd.DataFrame:
    """MultiIndex frame start/end/model-input/model-output, input tail-aligned to the output length."""
    target_tag_list = target_tag_list if target_tag_list is not None else tags
    n = len(model_output)
    model_input = np.asarray(getattr(model_input, "values", model_input))[-n:, :]
    model_output = np.asarray(getattr(model_output, "values", model_output))
    idx = index[-n:] if index is not None else pd.RangeIndex(n)
    if isinstance(idx, pd.DatetimeIndex):
        start = [ts.isoformat() for ts in idx]
        end = [(ts + frequency).isoformat() for ts in idx] if frequency is not None else [None] * n
    else:
        start, end = [None] * n, [None] * n
    blocks = {("start", ""): pd.Series(start, index=idx, dtype=object), ("end", ""): pd.Series(end, index=idx, dtype=object)}
    frame = pd.DataFrame(blocks, index=idx)
    frame.columns = pd.MultiIndex.from_tuples([("start", ""), ("end", "")])
    parts = [frame]
    for name, values, names in (("model-input", model_input, tags), ("model-output", model_output, target_tag_list)):
        names = [str(getattr(t, "name", t)) for t in names]
        second = names if values.shape[1] == len(names) else [str(i) for i in range(values.shape[1])]
        parts.append(pd.DataFrame(values, index=idx, columns=pd.MultiIndex.from_tuples([(name, s) for s in second])))
    return pd.concat(parts, axis=1)


# ------------------------------------------------------------------ DiffBasedKFCVAnomalyDetector (diff.py:461-635)


def kfcv_thresholds(abs_err: np.ndarray, scaled_mse: np.ndarray, window: Optional[int], smoothing_method: Optional[str], percentile: float):
    """
    diff.py:623-635: thresholds = percentile (pandas ``quantile``: linear interpolation, NaNs skipped) of the smoothed validation
    metric, where every row's metric comes from the K-fold model that did not train on it (:598-615).
    Returns (feature_thresholds [T], aggregate_threshold).
    """
    def thr(metric):
        m = smoothing(metric, window, smoothing_method) if (window is not None and smoothing_method is not None) else np.asarray(metric, dtype=np.float64)
        return pd.DataFrame(m).quantile(percentile).values

    return thr(np.asarray(abs_err, dtype=np.float64)), float(thr(np.asarray(scaled_mse, dtype=np.float64).reshape(-1, 1))[0])
