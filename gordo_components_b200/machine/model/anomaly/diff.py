"""
Diff-based anomaly detection with the public contract of
gordo/machine/model/anomaly/diff.py:21-458 (DiffBasedAnomalyDetector) -- constructor arguments,
``get_params`` contents, ``cross_validate`` / ``anomaly`` outputs, threshold attributes, metadata keys and
exceptions -- with every number computed on the GPU:

* ``anomaly``         one fused launch: network forward + abs diffs + row means + confidences (gb_ffae_infer_score),
                      or gb_anomaly_score when the base estimator is not one of ours;
* ``cross_validate``  fold scoring as above followed by the rolling-min/max threshold reduction (gb_thresholds);
* ``fit``             base estimator fit (gb_ffae_fit) and the MinMax scaler statistics (gb_minmax_fit).

Because ``S(yhat) - S(y) = (yhat - y) * scale`` for any per-feature affine scaler, the kernels need only the
scaler's per-tag multiplier; a non-affine ``scaler`` is rejected with ValueError rather than approximated.
"""
from __future__ import annotations

from datetime import timedelta
from typing import Dict, Optional, Sequence, Union

import weakref

import numpy as np
import pandas as pd
from sklearn.base import BaseEstimator, TransformerMixin
from sklearn.exceptions import NotFittedError
from sklearn.model_selection import TimeSeriesSplit
from sklearn.model_selection import cross_validate as sk_cross_validate
from sklearn.pipeline import Pipeline
from sklearn.preprocessing import MinMaxScaler
from sklearn.utils import shuffle as sk_shuffle
from sklearn.utils.validation import check_is_fitted

from .. import utils as model_utils
from ..base import GordoBase
from ..models import KerasAutoEncoder, KerasBaseEstimator, KerasLSTMBaseEstimator
from .base import AnomalyDetectorBase

_SCORE_ALL = ("tag-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-scaled", "total-anomaly-unscaled",
              "anomaly-confidence", "total-anomaly-confidence")


def _values(a) -> np.ndarray:
    return np.asarray(getattr(a, "values", a))


def _has_inf(a: np.ndarray) -> bool:
    return a.dtype.kind in "fc" and bool(np.isinf(a).any())


def _refuse_infinity(a: np.ndarray):
    """The error sklearn's scalers raise on ±inf (NaN passes): the reference scales y, the model output and, behind a scaler
    pipeline, X with them, so a request holding ±inf in any of these is refused there too."""
    if _has_inf(a):
        raise ValueError(f"Input X contains infinity or a value too large for {a.dtype!r}.")


def _total_skipna(total: np.ndarray, per_tag: np.ndarray, rows: np.ndarray) -> np.ndarray:
    """
    ``total`` (float64) with its ``rows`` (the NaN ones) recomputed as the reference computes the anomaly frame's totals,
    ``np.square(tags).mean(axis=1)`` on a DataFrame (diff.py:366, :383): pandas skips NaN tags, and a row with no tag left is NaN.
    The kernels average over every tag, the numpy mean that threshold fitting needs (diff.py:292), so only the frame is corrected.
    """
    sq = np.square(np.asarray(per_tag, dtype=np.float64)[rows])
    cnt = (~np.isnan(sq)).sum(axis=1)
    out = np.array(total, dtype=np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        out[rows] = np.where(cnt > 0, np.nansum(sq, axis=1) / cnt, np.nan)
    return out


_MULTIPLIERS = weakref.WeakKeyDictionary()  # scaler object -> (fitted-state key, slope): a request does not re-probe a fitted scaler


def _scaler_multiplier(scaler, n_features: int) -> np.ndarray:
    """Per-feature slope (float64) of a fitted affine scaler; ValueError if the transform is not affine per feature."""
    # a refit replaces the fitted arrays, so their identities stand for the fitted state (objects without such attributes are probed every time)
    state = tuple(id(getattr(scaler, name)) for name in ("scale_", "min_", "mean_", "center_") if getattr(scaler, name, None) is not None)
    key = (n_features, state)
    try:
        hit = _MULTIPLIERS.get(scaler) if state else None
    except TypeError:  # unhashable / not weak-referenceable scaler object
        hit = None
    if hit is not None and hit[0] == key:
        return hit[1]
    probe = np.vstack([np.zeros(n_features), np.ones(n_features), np.full(n_features, 2.0)])
    t = np.asarray(scaler.transform(probe), dtype=np.float64)
    slope = t[1] - t[0]
    if not np.allclose(t[2] - t[1], slope, rtol=1e-9, atol=1e-12):
        raise ValueError(f"scaler {scaler!r} is not a per-feature affine transform; the fused anomaly kernels cannot use it")
    if state:
        try:
            _MULTIPLIERS[scaler] = (key, slope)
        except TypeError:
            pass
    return slope


def _affine_of(step, n):
    """(a, b) with step.transform(X) == X * a + b per feature, or None when the step is not a plain per-feature scaler."""
    from sklearn.preprocessing import MaxAbsScaler, RobustScaler, StandardScaler

    one, zero = np.ones(n, dtype=np.float64), np.zeros(n, dtype=np.float64)
    try:
        if type(step) is MinMaxScaler and not getattr(step, "clip", False):
            a, b = np.asarray(step.scale_, dtype=np.float64), np.asarray(step.min_, dtype=np.float64)
        elif type(step) is StandardScaler:
            a = 1.0 / np.asarray(step.scale_, dtype=np.float64) if step.with_std else one
            b = -np.asarray(step.mean_, dtype=np.float64) * a if step.with_mean else zero
        elif type(step) is RobustScaler:
            a = 1.0 / np.asarray(step.scale_, dtype=np.float64) if step.with_scaling else one
            b = -np.asarray(step.center_, dtype=np.float64) * a if step.with_centering else zero
        elif type(step) is MaxAbsScaler:
            a, b = 1.0 / np.asarray(step.scale_, dtype=np.float64), zero
        else:
            return None
    except AttributeError:  # not fitted: let the step raise its own NotFittedError on the host path
        return None
    if a.shape != (n,) or b.shape != (n,):
        return None
    return a, b


def _compose_affine(steps, n):
    a, b = np.ones(n, dtype=np.float64), np.zeros(n, dtype=np.float64)
    for step in steps:
        ab = _affine_of(step, n)
        if ab is None:
            return None
        a, b = ab[0] * a, ab[0] * b + ab[1]
    return np.ascontiguousarray(a), np.ascontiguousarray(b)


class DiffBasedAnomalyDetector(AnomalyDetectorBase):
    def __init__(
        self,
        base_estimator: BaseEstimator = KerasAutoEncoder(kind="feedforward_hourglass"),
        scaler: TransformerMixin = MinMaxScaler(),
        require_thresholds: bool = True,
        shuffle: bool = False,
        window: Optional[int] = None,
        smoothing_method: Optional[str] = None,
    ):
        """
        Wraps ``base_estimator``; after training it, fits ``scaler`` on the target purely for the error arithmetic
        (the estimator itself sees unscaled ``y``).  Thresholds come from ``cross_validate`` (rolling minimum over 6
        samples of the validation errors, maximised; the last fold wins).  ``require_thresholds`` makes ``anomaly``
        raise AttributeError when they are missing.  ``shuffle`` shuffles rows in ``fit``.  ``window`` +
        ``smoothing_method`` ('smm' | 'sma' | 'ewma', default 'smm' when only a window is given) add smoothed scores.
        """
        self.base_estimator = base_estimator
        self.scaler = scaler
        self.require_thresholds = require_thresholds
        self.shuffle = shuffle
        self.window = window
        self.smoothing_method = smoothing_method
        if self.window is not None and self.smoothing_method is None:
            self.smoothing_method = "smm"

    def __getattr__(self, item):
        # anything the detector does not own is looked up on the wrapped estimator (this is how .predict exists)
        if item in self.__dict__:
            return getattr(self, item)
        if item == "base_estimator":
            raise AttributeError(item)
        return getattr(self.base_estimator, item)

    # ------------------------------------------------------------------ bookkeeping
    def get_params(self, deep=True):
        params = {"base_estimator": self.base_estimator, "scaler": self.scaler, "shuffle": self.shuffle}
        if self.window is not None:
            params["window"] = self.window
            params["smoothing_method"] = self.smoothing_method
        return params

    def score(self, X, y, sample_weight=None) -> float:
        return self.base_estimator.score(X, y)

    def get_metadata(self):
        metadata = dict()
        if hasattr(self, "feature_thresholds_"):
            metadata["feature-thresholds"] = self.feature_thresholds_.tolist()
        if hasattr(self, "aggregate_threshold_"):
            metadata["aggregate-threshold"] = self.aggregate_threshold_
        if hasattr(self, "feature_thresholds_per_fold_"):
            metadata["feature-thresholds-per-fold"] = self.feature_thresholds_per_fold_.to_dict()
        if hasattr(self, "aggregate_thresholds_per_fold_"):
            metadata["aggregate-thresholds-per-fold"] = self.aggregate_thresholds_per_fold_
        if hasattr(self, "window"):
            metadata["window"] = self.window
        if hasattr(self, "smoothing_method"):
            metadata["smoothing-method"] = self.smoothing_method
        if hasattr(self, "smooth_feature_thresholds_") and self.smooth_aggregate_threshold_ is not None:
            metadata["smooth-feature-thresholds"] = self.smooth_feature_thresholds_.tolist()
        if hasattr(self, "smooth_aggregate_threshold_") and self.smooth_aggregate_threshold_ is not None:
            metadata["smooth-aggregate-threshold"] = self.smooth_aggregate_threshold_
        if hasattr(self, "smooth_feature_thresholds_per_fold_"):
            metadata["smooth-feature-thresholds-per-fold"] = self.smooth_feature_thresholds_per_fold_.to_dict()
        if hasattr(self, "smooth_aggregate_thresholds_per_fold_"):
            metadata["smooth-aggregate-thresholds-per-fold"] = self.smooth_aggregate_thresholds_per_fold_
        if isinstance(self.base_estimator, GordoBase):
            metadata.update(self.base_estimator.get_metadata())
        else:
            metadata.update({"scaler": str(self.scaler), "base_estimator": str(self.base_estimator), "shuffle": self.shuffle})
        return metadata

    # ------------------------------------------------------------------ fit
    def fit(self, X, y):
        if self.shuffle:
            Xs, ys = sk_shuffle(X, y, random_state=0)
            self.base_estimator.fit(Xs, ys)
        else:
            self.base_estimator.fit(X, y)
        self._fit_scaler(y)
        return self

    def _is_b200_network(self) -> bool:
        """True when the predictions come out of one of this package's fp32 networks (bare or last step of a Pipeline)."""
        est = self.base_estimator
        if isinstance(est, Pipeline) and len(est.steps):
            est = est.steps[-1][1]
        return isinstance(est, KerasBaseEstimator)

    def _fit_scaler(self, y):
        """
        Scaler statistics of the targets (diff.py:173 ``self.scaler.fit(y)``).  For a default MinMaxScaler around one of this
        package's networks the column extrema come from the gb_minmax_f64 kernel -- on the float64 targets, as the reference's
        scaler sees them -- and sklearn's float64 attribute arithmetic is applied to them on the host, so every fitted attribute
        equals sklearn's own.  Any other scaler, and any foreign base estimator, is fitted by its own code.
        """
        sc = self.scaler
        plain_minmax = type(sc) is MinMaxScaler and tuple(sc.feature_range) == (0, 1) and not getattr(sc, "clip", False)
        yv = _values(y)
        if not plain_minmax or not self._is_b200_network() or yv.ndim != 2 or yv.shape[1] > 256 or len(yv) == 0 or not np.issubdtype(yv.dtype, np.number):
            sc.fit(y)  # user supplied transformer / foreign estimator: its own code owns its statistics
            return
        from .... import engine

        dev = engine.cuda_device()
        torch = engine._torch()
        yd = torch.from_numpy(np.ascontiguousarray(yv, dtype=np.float64)).to(dev)
        n, t = yd.shape
        jobs = engine.jobs_to_device(engine.make_jobs([0], [n], [0]), dev)
        lo, hi = engine.minmax_f64(jobs, 1, n, yd, 1)
        lo, hi = lo[0].cpu().numpy(), hi[0].cpu().numpy()
        if not (np.isfinite(lo).all() and np.isfinite(hi).all()):
            sc.fit(y)  # all-NaN or infinite columns: sklearn's own error / warning behaviour
            return
        # sklearn.preprocessing.MinMaxScaler.partial_fit [3P]: data_range_ = max - min; scale_ = 1 / range with ranges below
        # 10 * eps taken as 1 (_handle_zeros_in_scale); min_ = 0 - data_min_ * scale_
        data_range = hi - lo
        denom = data_range.copy()
        denom[denom < 10 * np.finfo(np.float64).eps] = 1.0
        sc.n_samples_seen_ = n
        sc.n_features_in_ = t
        sc.data_min_, sc.data_max_, sc.data_range_ = lo, hi, data_range
        sc.scale_ = 1.0 / denom
        sc.min_ = 0.0 - lo * sc.scale_
        if hasattr(y, "columns") and all(isinstance(c, str) for c in y.columns):
            sc.feature_names_in_ = np.asarray(y.columns, dtype=object)
        elif hasattr(sc, "feature_names_in_"):
            del sc.feature_names_in_

    # ------------------------------------------------------------------ scoring core (all GPU)
    def _fused_target(self):
        """(pre-transformers, our feed-forward AE) when the forward pass can be fused with the scoring, else None."""
        est = self.base_estimator
        if isinstance(est, KerasAutoEncoder):
            return [], est
        if isinstance(est, Pipeline) and len(est.steps) and isinstance(est.steps[-1][1], KerasAutoEncoder):
            return [step for _, step in est.steps[:-1]], est.steps[-1][1]
        return None

    def _score(self, estimator_owner, X, y_true, scaler, feat_thr=None, agg_thr=None, want: Sequence[str] = _SCORE_ALL) -> Dict[str, np.ndarray]:
        """
        Model output and the requested anomaly columns as host arrays.  ``estimator_owner`` is the detector whose
        base estimator predicts (``self`` or a CV fold clone); ``y_true`` may be longer than the prediction and is
        tail-aligned to it (LSTM offset).
        """
        from .... import engine

        dev = engine.cuda_device()
        yv = _values(y_true)
        _refuse_infinity(yv)
        n_out = yv.shape[1]
        mult = _scaler_multiplier(scaler, n_out)
        torch = engine._torch()
        fused = estimator_owner._fused_target()
        fused = fused if fused is not None and fused[1].model is not None else None
        # the fused launch is fp32 like the network; predictions that come from elsewhere are scored in float64 like the reference
        dt, npdt = (torch.float32, np.float32) if fused is not None else (torch.float64, np.float64)
        scale_d = torch.from_numpy(np.ascontiguousarray(mult.reshape(1, -1), dtype=npdt)).to(dev)
        ft_d = torch.from_numpy(np.asarray(feat_thr, dtype=npdt).reshape(1, -1)).to(dev) if feat_thr is not None else None
        at_d = torch.tensor([float(agg_thr)], dtype=dt, device=dev) if agg_thr is not None else None
        if fused is not None:
            pre, ae = fused
            eng = ae._engine()
            affine = _compose_affine(pre, eng.n_in)
            variant, x_affine = 0, None
            if pre and affine is not None:
                # per-feature scalers in front of the network, in float64 on the device instead of sklearn on the host: applied by the
                # fused kernel as it reads x (gb_ffae_infer_score_x64), or, for a stack that mode does not hold, as a separate pass
                # (gb_affine_f64) -- the same float32 x' either way, so the same bits out
                Xv = np.ascontiguousarray(_values(X), dtype=np.float64)
                _refuse_infinity(Xv)  # what the sklearn steps would have raised
                n = len(Xv)
                jobs = engine.jobs_to_device(engine.make_jobs([0], [n], [0]), dev)
                a_d, b_d = (torch.from_numpy(v.reshape(1, -1)).to(dev) for v in affine)
                if n and eng.infer_plan_x64(variant) is not None:
                    xd, x_affine = torch.from_numpy(Xv).to(dev), (a_d, b_d)
                else:
                    xd = engine.affine_f64(jobs, 1, n, torch.from_numpy(Xv).to(dev), a_d, b_d) if n else torch.empty((0, eng.n_in), dtype=torch.float32, device=dev)
            else:
                Xt = X
                for step in pre:
                    Xt = step.transform(Xt)
                Xv = _values(Xt)
                n = len(Xv)
                jobs = engine.jobs_to_device(engine.make_jobs([0], [n], [0]), dev)
                xd = engine.to_device_f32(Xv, dev)
                if _has_inf(Xv):
                    # tanh(±inf) = ±1 as in Keras on the fp32 kernels; the tensor-core kernel's split of x into TF32 + BF16 parts
                    # turns ±inf into NaN, so an input holding ±inf is not given to it
                    variant = 1
            yd = engine.to_device_f32(yv, dev)
            res = eng.infer_score(ae._device_params(), jobs, 1, n, xd, yd, scale_d, ft_d, at_d, want=want, variant=variant, x_affine=x_affine)
        else:
            # diff.py:350-385: pandas arithmetic on float64 y and the (float32- or float64-valued) predictions widened to float64
            pred = np.asarray(estimator_owner.predict(X) if hasattr(estimator_owner, "predict") else estimator_owner.transform(X))
            _refuse_infinity(pred)
            n = len(pred)
            p64 = np.ascontiguousarray(pred, dtype=np.float64)
            p64 = p64.reshape(n, -1)
            pd_ = torch.from_numpy(p64).to(dev)
            yd = torch.from_numpy(np.ascontiguousarray(yv[-n:] if n else yv[:0], dtype=np.float64)).to(dev)
            jobs = engine.jobs_to_device(engine.make_jobs([0], [n], [0]), dev)
            res = engine.anomaly_score(jobs, 1, n, pd_, yd, n_out, scale_d, ft_d, at_d, want=want) if n else {}
            res["model-output"] = pred
        res = {k: (v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v)) for k, v in res.items()}
        if fused is not None:
            _refuse_infinity(res["model-output"])
        return res

    # ------------------------------------------------------------------ cross validation -> thresholds
    def cross_validate(self, *, X, y, cv=TimeSeriesSplit(n_splits=3), **kwargs):
        """
        sklearn cross validation of the detector (same return dict), after which the thresholds are derived from
        each fold's validation errors; the final thresholds are the last fold's.
        """
        from .... import engine

        kwargs.update(dict(return_estimator=True, cv=cv))
        cv_output = sk_cross_validate(self, X=X, y=y, **kwargs)

        columns = list(y.columns) if hasattr(y, "columns") else list(range(_values(y).shape[1]))
        per_fold, agg_per_fold = {}, {}
        smooth_per_fold, smooth_agg_per_fold = {}, {}
        feat = agg = sfeat = sagg = None
        dev = engine.cuda_device()
        torch = engine._torch()
        for i, ((_, test_idxs), fold) in enumerate(zip(kwargs["cv"].split(X, y), cv_output["estimator"])):
            X_test = X.iloc[test_idxs] if isinstance(X, pd.DataFrame) else X[test_idxs]
            y_test = y.iloc[test_idxs] if isinstance(y, pd.DataFrame) else y[test_idxs]
            try:
                check_is_fitted(fold.scaler)
            except NotFittedError:
                fold.scaler.fit(y_test)
            res = self._score(fold, X_test, y_test, fold.scaler, want=("tag-anomaly-unscaled", "total-anomaly-scaled"))
            n = len(res["model-output"])
            tu = torch.from_numpy(np.ascontiguousarray(res["tag-anomaly-unscaled"])).to(dev)  # float32 (fused network) or float64
            ts = torch.from_numpy(np.ascontiguousarray(res["total-anomaly-scaled"], dtype=res["tag-anomaly-unscaled"].dtype)).to(dev)
            jobs = engine.jobs_to_device(engine.make_jobs([0], [n], [0]), dev)
            f, a = engine.thresholds(jobs, 1, n, tu, ts, tu.shape[1], 1, 6, dev)
            feat = pd.Series(f[0].cpu().numpy().astype(np.float64), index=columns, name=f"fold-{i}")
            agg = float(a[0])
            per_fold[f"fold-{i}"] = feat
            agg_per_fold[f"fold-{i}"] = agg
            if self.window is not None:
                f, a = engine.thresholds(jobs, 1, n, tu, ts, tu.shape[1], 1, int(self.window), dev)
                sfeat = pd.Series(f[0].cpu().numpy().astype(np.float64), index=columns, name=f"fold-{i}")
                sagg = float(a[0])
                smooth_per_fold[f"fold-{i}"] = sfeat
                smooth_agg_per_fold[f"fold-{i}"] = sagg

        self.feature_thresholds_per_fold_ = pd.DataFrame(list(per_fold.values())) if per_fold else pd.DataFrame()
        self.aggregate_thresholds_per_fold_ = agg_per_fold
        self.smooth_feature_thresholds_per_fold_ = pd.DataFrame(list(smooth_per_fold.values())) if smooth_per_fold else pd.DataFrame()
        self.smooth_aggregate_thresholds_per_fold_ = smooth_agg_per_fold
        self.feature_thresholds_ = feat
        self.aggregate_threshold_ = agg
        self.smooth_aggregate_threshold_ = sagg
        self.smooth_feature_thresholds_ = sfeat
        return cv_output

    # ------------------------------------------------------------------ anomaly frame
    def _smoothing(self, metric: np.ndarray) -> np.ndarray:
        """smm / sma / ewma of every column of ``metric`` (gb_smooth kernel, pandas rolling/ewm semantics)."""
        from .... import engine

        dev = engine.cuda_device()
        torch = engine._torch()
        a = torch.from_numpy(np.ascontiguousarray(metric, dtype=np.float32)).to(dev)
        jobs = engine.jobs_to_device(engine.make_jobs([0], [a.shape[0]], [0]), dev)
        return engine.smooth(jobs, 1, a, int(self.window), self.smoothing_method).cpu().numpy()

    def anomaly(self, X: pd.DataFrame, y: pd.DataFrame, frequency: Optional[timedelta] = None) -> pd.DataFrame:
        """
        Frame with ``start, end, model-input, model-output, tag-anomaly-scaled, total-anomaly-scaled,
        tag-anomaly-unscaled, total-anomaly-unscaled`` [+ ``anomaly-confidence, total-anomaly-confidence`` when
        thresholds exist]; with ``window`` + ``smoothing_method`` the four ``smooth-*`` blocks come before the confidences.
        Rows follow the model output (shorter than X for LSTM models).
        """
        return model_utils.frame_from_blocks(*self.anomaly_blocks(X, y, frequency))

    def anomaly_blocks(self, X: pd.DataFrame, y: pd.DataFrame, frequency: Optional[timedelta] = None, smooth: bool = True):
        """
        The anomaly frame before it becomes a DataFrame: ``(row index, [column blocks], [(top, sub) column names])``.  A caller that
        only serialises the result (``server.anomaly_prediction``) reads the blocks directly and skips the frame.  ``smooth=False``
        leaves out the ``smooth-*`` blocks (and the work behind them), for a reply that drops them anyway.
        """
        if not hasattr(X, "values"):
            raise ValueError("Unable to find X.values property")
        if self.require_thresholds and not any(hasattr(self, a) for a in ("feature_thresholds_", "aggregate_threshold_")):
            raise AttributeError(
                f"`require_thresholds={self.require_thresholds}` however `.cross_validate` needs to be called in order "
                f"to calculate these thresholds before calling `.anomaly`"
            )
        feat_thr, agg_thr = self._thresholds()
        return self.blocks_from_scores(self._score(self, X, y, self.scaler, feat_thr, agg_thr), X, y, frequency, smooth=smooth)

    def _thresholds(self):
        feat_thr = self.feature_thresholds_.values if getattr(self, "feature_thresholds_", None) is not None else None
        agg_thr = self.aggregate_threshold_ if getattr(self, "aggregate_threshold_", None) is not None else None
        return feat_thr, agg_thr

    def blocks_from_scores(self, res: Dict[str, np.ndarray], X, y, frequency: Optional[timedelta] = None, smooth: bool = True):
        """
        ``anomaly_blocks`` for score arrays that already exist (``res`` as ``_score`` returns it, e.g. out of a request coalescer).
        ``smooth-*`` arrays already in ``res`` (a coalescer's smoothing launch) are used as they are; the caller makes sure they were
        smoothed from the same totals, i.e. that no row's total is recomputed here (a target holding NaN).
        """
        feat_thr, agg_thr = self._thresholds()
        res = dict(res)
        # rows with a missing target tag: pandas' totals, and the total confidence from them, before anything is smoothed
        for total, per_tag in (("total-anomaly-scaled", "tag-anomaly-scaled"), ("total-anomaly-unscaled", "tag-anomaly-unscaled")):
            if total not in res or per_tag not in res:
                continue
            rows = np.isnan(res[total])
            if not rows.any():
                continue
            res[total] = _total_skipna(res[total], res[per_tag], rows)
            if total == "total-anomaly-scaled" and "total-anomaly-confidence" in res and agg_thr is not None:
                conf = np.array(res["total-anomaly-confidence"], dtype=np.float64)
                conf[rows] = res[total][rows] / float(agg_thr)
                res["total-anomaly-confidence"] = conf
        out = res["model-output"]
        index, frame_blocks, frame_cols = model_utils.base_blocks(
            tags=X.columns, model_input=X.values, model_output=out, target_tag_list=y.columns,
            index=getattr(X, "index", None), frequency=frequency,
        )
        targets = [sub for top, sub in frame_cols if top == "model-output"]
        blocks, cols = [], []

        def add(name, per_tag):
            if name not in res:
                return
            v = np.asarray(res[name], dtype=np.float64)
            if per_tag:
                blocks.append(v)
                cols.extend((name, t) for t in targets)
            else:
                blocks.append(v.reshape(-1, 1))
                cols.append((name, ""))

        add("tag-anomaly-scaled", True)
        add("total-anomaly-scaled", False)
        add("tag-anomaly-unscaled", True)
        add("total-anomaly-unscaled", False)
        if smooth and self.window is not None and self.smoothing_method is not None:
            for name, per_tag in (("tag-anomaly-scaled", True), ("total-anomaly-scaled", False), ("tag-anomaly-unscaled", True),
                                  ("total-anomaly-unscaled", False)):
                if "smooth-" + name not in res:
                    res["smooth-" + name] = self._smoothing(res[name])
                add("smooth-" + name, per_tag)
        if feat_thr is not None:
            add("anomaly-confidence", True)
        if agg_thr is not None:
            add("total-anomaly-confidence", False)
        if blocks:  # all score columns travel as one float64 block
            frame_blocks.append(np.concatenate(blocks, axis=1))
        return index, frame_blocks, frame_cols + cols


class DiffBasedKFCVAnomalyDetector(DiffBasedAnomalyDetector):
    """
    diff.py:461-635: thresholds are a percentile of the *smoothed* validation errors gathered over K-fold cross-validation
    predictions (every row is predicted by the fold model that did not see it), instead of the rolling-min/max of the last
    TimeSeriesSplit fold.  ``anomaly`` is inherited.  Error columns, smoothing and the percentile run on the GPU
    (gb_anomaly_score / gb_ffae_infer_score, gb_smooth, gb_quantile).
    """

    def __init__(
        self,
        base_estimator: BaseEstimator = KerasAutoEncoder(kind="feedforward_hourglass"),
        scaler: TransformerMixin = MinMaxScaler(),
        require_thresholds: bool = True,
        shuffle: bool = True,
        window: int = 144,
        smoothing_method: str = "smm",
        threshold_percentile: float = 0.99,
    ):
        self.base_estimator = base_estimator
        self.scaler = scaler
        self.require_thresholds = require_thresholds
        self.window = window
        self.shuffle = shuffle
        self.smoothing_method = smoothing_method
        self.threshold_percentile = threshold_percentile

    def get_params(self, deep=True):
        return {
            "base_estimator": self.base_estimator, "scaler": self.scaler, "window": self.window, "smoothing_method": self.smoothing_method,
            "shuffle": self.shuffle, "threshold_percentile": self.threshold_percentile,
        }

    def get_metadata(self):
        metadata = dict()
        if hasattr(self, "feature_thresholds_"):
            metadata["feature-thresholds"] = self.feature_thresholds_.tolist()
        if hasattr(self, "aggregate_threshold_"):
            metadata["aggregate-threshold"] = self.aggregate_threshold_
        if isinstance(self.base_estimator, GordoBase):
            metadata.update(self.base_estimator.get_metadata())
        else:
            metadata.update({
                "scaler": str(self.scaler), "base_estimator": str(self.base_estimator), "shuffle": self.shuffle, "window": self.window,
                "smoothing-method": self.smoothing_method, "threshold-percentile": self.threshold_percentile,
            })
        return metadata

    def cross_validate(self, *, X, y, cv=None, **kwargs):
        from sklearn.model_selection import KFold

        cv = cv if cv is not None else KFold(n_splits=5, shuffle=True, random_state=0)
        kwargs.update(dict(return_estimator=True, cv=cv))
        cv_output = sk_cross_validate(self, X=X, y=y, **kwargs)
        feature_thresholds, self.aggregate_threshold_ = self.kfold_thresholds(X, y, kwargs["cv"], cv_output["estimator"])
        self.feature_thresholds_ = feature_thresholds
        return cv_output

    def kfold_thresholds(self, X, y, cv, fold_estimators):
        """
        ``(feature_thresholds_, aggregate_threshold_)`` from fitted fold detectors (``cross_validate``'s ``estimator`` list, in the
        order of ``cv.split``): every row scored by the fold model that did not see it, smoothed, the ``threshold_percentile``
        quantile.
        """
        from .... import engine

        yv = _values(y)
        n, t = yv.shape
        columns = list(y.columns) if hasattr(y, "columns") else list(range(t))
        abs_err = np.zeros((n, t), dtype=np.float32)
        val_mse = np.full((n,), np.nan, dtype=np.float32)
        for (_, test_idxs), fold in zip(cv.split(X, y), fold_estimators):
            X_test = X.iloc[test_idxs] if isinstance(X, pd.DataFrame) else X[test_idxs]
            y_test = y.iloc[test_idxs] if isinstance(y, pd.DataFrame) else y[test_idxs]
            res = self._score(fold, X_test, y_test, fold.scaler, want=("tag-anomaly-unscaled", "total-anomaly-scaled"))
            if len(res["model-output"]) != len(test_idxs):
                raise ValueError("K-fold thresholds need a base estimator that predicts one row per input row")
            abs_err[test_idxs] = res["tag-anomaly-unscaled"]
            val_mse[test_idxs] = res["total-anomaly-scaled"]

        dev = engine.cuda_device()
        torch = engine._torch()
        jobs = engine.jobs_to_device(engine.make_jobs([0], [n], [0]), dev)
        q = float(self.threshold_percentile)

        def threshold(metric: np.ndarray):
            a = torch.from_numpy(np.ascontiguousarray(metric, dtype=np.float32)).to(dev)
            if self.window is not None and self.smoothing_method is not None:
                a = engine.smooth(jobs, 1, a, int(self.window), self.smoothing_method)
            return engine.quantile(jobs, 1, n, a, q)[0].cpu().numpy().astype(np.float64)

        aggregate = float(threshold(val_mse)[0])
        return pd.Series(threshold(abs_err), index=columns), aggregate
