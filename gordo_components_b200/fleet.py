"""
Fleet API: score (and shard) many machines at once.

``anomaly_many`` is the call a fleet user makes: host arrays in, host arrays out, with the host<->device copies
pipelined against the fused kernel on a few CUDA streams.  ``partition``/``assign_machines``/``gather_summaries`` are
the whole multi-GPU story: machines are independent (the reference runs one Kubernetes pod per machine,
gordo/workflow/workflow_generator/resources/argo-workflow.yml.template:1544-1557), so ranks own disjoint contiguous
blocks of machines and the only communication is the broadcast of the assignment and the gather of per-machine
summaries -- there is no exchange step inside fit, predict or anomaly.
"""
from __future__ import annotations

import functools
import math
import time
from typing import Dict, List, Optional, Sequence

import numpy as np
from sklearn.utils import shuffle as sk_shuffle

from . import engine

PER_TAG = ("model-output", "tag-anomaly-scaled", "tag-anomaly-unscaled", "anomaly-confidence")
PER_ROW = ("total-anomaly-scaled", "total-anomaly-unscaled", "total-anomaly-confidence")


# ------------------------------------------------------------------------------------------------ sharding
def partition(n_machines: int, world: int) -> List[range]:
    """Contiguous, balanced blocks: the first (n % world) ranks get one extra machine."""
    base, extra = divmod(n_machines, world)
    out, start = [], 0
    for r in range(world):
        size = base + (1 if r < extra else 0)
        out.append(range(start, start + size))
        start += size
    return out


def assign_machines(n_machines: int, world: int, rank: int, dist=None) -> np.ndarray:
    """Rank 0 computes the partition and broadcasts it (NCCL/gloo object broadcast); returns this rank's machine ids."""
    if dist is None or world == 1:
        return np.arange(n_machines)
    payload = [[list(r) for r in partition(n_machines, world)] if rank == 0 else None]
    dist.broadcast_object_list(payload, src=0)
    return np.asarray(payload[0][rank], dtype=np.int64)


def gather_summaries(local, world: int, dist=None):
    """all_gather of one fixed-size summary tensor per rank (e.g. max total-anomaly-confidence per machine)."""
    if dist is None or world == 1:
        return local
    torch = engine._torch()
    buf = torch.empty((world * local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(buf, local.contiguous())
    return buf


def random_glorot_params(eng: "engine.FFEngine", n_slots: int, generator):
    """Synthetic fleet: glorot-uniform kernels, small uniform biases, generated on the device (bench/test plumbing)."""
    torch = engine._torch()
    params = torch.zeros((n_slots, eng.param_stride), dtype=torch.float32, device=eng.device)
    ofs = 0
    for i, o in zip(eng.dims[:-1], eng.dims[1:]):
        lim = float(np.sqrt(6.0 / (i + o)))
        params[:, ofs:ofs + i * o] = (torch.rand((n_slots, i * o), generator=generator, device=eng.device) * 2 - 1) * lim
        ofs += i * o
        params[:, ofs:ofs + o] = (torch.rand((n_slots, o), generator=generator, device=eng.device) * 2 - 1) * 0.1
        ofs += o
    return params


# ------------------------------------------------------------------------------------------------ host-buffer scoring
class HostPipeline:
    """Pinned host buffers + per-stream device staging for ``anomaly_many``; reusable across calls of the same shape."""

    def __init__(self, eng: "engine.FFEngine", n_machines: int, rows: int, chunk_machines: int = 50, n_streams: int = 3,
                 want: Sequence[str] = PER_TAG + PER_ROW):
        torch = engine._torch()
        self.eng, self.M, self.R = eng, n_machines, rows
        self.chunk = max(1, min(chunk_machines, n_machines))
        self.want = tuple(want)
        dev = eng.device
        self.streams = [torch.cuda.Stream(device=dev) for _ in range(n_streams)]
        cr = self.chunk * rows
        self.stage = []
        for _ in self.streams:
            st = {"x": torch.empty((cr, eng.n_in), dtype=torch.float32, device=dev), "y": torch.empty((cr, eng.n_out), dtype=torch.float32, device=dev), "out": {}}
            for k in self.want:
                st["out"][k] = torch.empty((cr, eng.n_out) if k in PER_TAG else (cr,), dtype=torch.float32, device=dev)
            self.stage.append(st)
        total = n_machines * rows
        self.host_out = {k: torch.empty((total, eng.n_out) if k in PER_TAG else (total,), dtype=torch.float32).pin_memory() for k in self.want}
        self.chunks = []
        for c0 in range(0, n_machines, self.chunk):
            m = min(self.chunk, n_machines - c0)
            jobs = engine.make_jobs(np.arange(c0, c0 + m), rows, np.arange(m, dtype=np.int64) * rows)
            self.chunks.append((c0, m, engine.jobs_to_device(jobs, dev)))
        self.h2d_bytes = total * (eng.n_in + eng.n_out) * 4
        self.d2h_bytes = sum(v.numel() * 4 for v in self.host_out.values())

    def run(self, params, x_host, y_host, scale, feat_thr, agg_thr, variant: int = 0) -> Dict[str, "object"]:
        """x_host / y_host: pinned float32 host tensors [M*R, T].  Returns pinned host tensors (valid after the sync below)."""
        torch = engine._torch()
        R = self.R
        for i, (c0, m, jobs) in enumerate(self.chunks):
            s = self.streams[i % len(self.streams)]
            st = self.stage[i % len(self.streams)]
            rows = slice(c0 * R, (c0 + m) * R)
            with torch.cuda.stream(s):
                st["x"][: m * R].copy_(x_host[rows], non_blocking=True)
                st["y"][: m * R].copy_(y_host[rows], non_blocking=True)
                self.eng.infer_score(params, jobs, m, R, st["x"], st["y"], scale, feat_thr, agg_thr, out_rows=self.chunk * R,
                                     want=self.want, variant=variant, out=st["out"])
                for k in self.want:
                    self.host_out[k][rows].copy_(st["out"][k][: m * R], non_blocking=True)
        for s in self.streams:
            s.synchronize()
        return self.host_out


def anomaly_many(eng: "engine.FFEngine", params, x_host, y_host, scale, feat_thr=None, agg_thr=None, rows: Optional[int] = None,
                 pipeline: Optional[HostPipeline] = None, variant: int = 0):
    """
    Fleet form of ``DiffBasedAnomalyDetector.anomaly``: machine m owns rows [m*rows, (m+1)*rows) of the host arrays and
    slot m of ``params`` / ``scale`` / thresholds.  Returns a dict of host arrays named like the anomaly frame's blocks.
    """
    torch = engine._torch()
    xh = x_host if hasattr(x_host, "is_pinned") else torch.from_numpy(np.ascontiguousarray(x_host, dtype=np.float32))
    yh = y_host if hasattr(y_host, "is_pinned") else torch.from_numpy(np.ascontiguousarray(y_host, dtype=np.float32))
    n_machines = params.shape[0]
    rows = rows or xh.shape[0] // n_machines
    want = [k for k in PER_TAG + PER_ROW if not ((feat_thr is None and k == "anomaly-confidence") or (agg_thr is None and k == "total-anomaly-confidence"))]
    pipe = pipeline or HostPipeline(eng, n_machines, rows, want=want)
    if not xh.is_pinned():
        xh = xh.pin_memory()
    if not yh.is_pinned():
        yh = yh.pin_memory()
    return pipe.run(params, xh, yh, scale, feat_thr, agg_thr, variant)


def time_e2e(eng, params, jobs_h, x_dev, y_dev, scale, feat_thr, agg_thr, steps: int = 3, variant: int = 0):
    """End-to-end windows/s of ``anomaly_many``: pinned host inputs, H2D + kernel + D2H of every output inside the timed region."""
    torch = engine._torch()
    M = len(jobs_h)
    R = int(jobs_h["n_rows"][0])
    xh = torch.empty(x_dev.shape, dtype=torch.float32).pin_memory()
    yh = torch.empty(y_dev.shape, dtype=torch.float32).pin_memory()
    xh.copy_(x_dev)
    yh.copy_(y_dev)
    pipe = HostPipeline(eng, M, R)
    anomaly_many(eng, params, xh, yh, scale, feat_thr, agg_thr, rows=R, pipeline=pipe, variant=variant)  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        anomaly_many(eng, params, xh, yh, scale, feat_thr, agg_thr, rows=R, pipeline=pipe, variant=variant)
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / steps
    return {"ms_per_step": dt * 1e3, "h2d_bytes": pipe.h2d_bytes, "d2h_bytes": pipe.d2h_bytes}


# ------------------------------------------------------------------------------------------------ fleet build (train + thresholds)
def _fill_history(est, metrics, epochs: int, steps, loss, acc, val_loss=None, val_acc=None, epochs_run=None):
    """
    The Keras ``History`` a fit leaves, as ``est._history`` and ``est.model.history``, from one fit's host per-epoch rows: loss,
    accuracy when ``metrics`` has it, and their ``val_*`` forms with a validation split, in the per-machine History's key order.
    ``epochs_run``: the epochs an EarlyStopping fit ran (None: every row); ``epochs`` / ``steps`` are History.params'.
    """
    from .machine.model.models import History

    ran = len(loss) if epochs_run is None else int(epochs_run)
    rows = {"loss": loss, "accuracy": acc, "val_loss": val_loss, "val_accuracy": val_acc}
    hist = {k: [float(v) for v in r[:ran]] for k, r in rows.items() if r is not None and ("accuracy" in metrics or not k.endswith("accuracy"))}
    est._history = History(hist, {"verbose": 0, "epochs": int(epochs), "steps": steps}, list(range(ran)))
    est.model.history = est._history
    return est


def _fill_thresholds(det, tags, feat, agg, fold_feat=None, fold_agg=None, window=None, fold_smooth_feat=None, fold_smooth_agg=None):
    """
    The thresholds a detector's ``cross_validate`` leaves, from host arrays: ``feature_thresholds_`` / ``aggregate_threshold_``
    (``feat`` [T], ``agg``), and with ``fold_feat`` [K, T] / ``fold_agg`` [K] the per-fold ones (diff.py:257-264) and the four
    smooth-threshold attributes (diff.py:384-391) -- from the per-fold window-``window`` thresholds ``fold_smooth_feat`` [K, T] /
    ``fold_smooth_agg`` [K] when the detector has a window, else the empty values.  Without ``fold_feat`` (a K-fold detector)
    only the first two, the Series unnamed.
    """
    import pandas as pd

    K = None if fold_agg is None else len(fold_agg)
    det.feature_thresholds_ = pd.Series(np.array(feat, dtype=np.float64), index=tags, name=None if K is None else f"fold-{K - 1}")
    det.aggregate_threshold_ = float(agg)
    if K is None:
        return det
    det.feature_thresholds_per_fold_ = pd.DataFrame(np.array(fold_feat, dtype=np.float64), columns=tags, index=[f"fold-{k}" for k in range(K)])
    det.aggregate_thresholds_per_fold_ = {f"fold-{k}": float(fold_agg[k]) for k in range(K)}
    if window is None:
        det.smooth_feature_thresholds_per_fold_ = pd.DataFrame()
        det.smooth_aggregate_thresholds_per_fold_ = {}
        det.smooth_aggregate_threshold_ = None
        det.smooth_feature_thresholds_ = None
        return det
    ff = np.asarray(fold_smooth_feat, dtype=np.float64)
    det.smooth_feature_thresholds_per_fold_ = pd.DataFrame(ff.copy(), columns=tags, index=[f"fold-{k}" for k in range(K)])
    det.smooth_aggregate_thresholds_per_fold_ = {f"fold-{k}": float(fold_smooth_agg[k]) for k in range(K)}
    det.smooth_feature_thresholds_ = pd.Series(ff[K - 1].copy(), index=tags, name=f"fold-{K - 1}")
    det.smooth_aggregate_threshold_ = float(fold_smooth_agg[K - 1])
    return det


def _ff_template(eng, template, target_scaler: bool, input_scaler: bool, params):
    """
    Fill the feed-forward network of ``template`` (an unfitted detector from the machine's own definition) with the fleet's
    architecture and the weights ``params`` [1, stride].  Returns (the TransformedTargetRegressor or None, the estimator inside
    it -- the Pipeline, whose MinMaxScaler the caller fills, or the network -- and the network); ValueError when the template's
    target transformer, input scaler or architecture differ from the fleet's.
    """
    from sklearn.pipeline import Pipeline

    ttr, est = _target_regressor_of(template.base_estimator, target_scaler)
    ae = est.steps[-1][1] if isinstance(est, Pipeline) else est
    if isinstance(est, Pipeline) != bool(input_scaler):
        raise ValueError("the template's input scaler and the fleet's do not match")
    ae.kwargs.update({"n_features": eng.n_in, "n_features_out": eng.n_out})
    ae._prepare_model()
    if list(ae.model.spec.dims) != list(eng.dims) or list(ae.model.spec.acts) != list(eng.acts):
        raise ValueError("template architecture differs from the fleet's")
    ae.model.weights = eng.unpack_params(params)[0]
    return ttr, est, ae


class FleetBuild:
    """
    Result of ``build_fleet``: everything ``ModelBuilder._build`` (gordo/builder/build_model.py:192-339) produces for one
    machine -- final weights, target scaler, CV thresholds (per fold and final), loss histories -- for all machines at once.
    """

    def __init__(self, eng, n_machines, n_splits, params, scale, offset, feat_thr, agg_thr, loss, acc, fold_loss, fold_feat_thr, fold_agg_thr,
                 fold_params=None, cv_moments=None, in_scale=None, in_offset=None, fold_in_scale=None, fold_in_offset=None, steps_per_epoch=None,
                 val_loss=None, val_acc=None, fold_val_loss=None, fold_val_acc=None, epochs=None, epochs_run=None, best_epoch=None,
                 fold_epochs_run=None, fold_best_epoch=None, rows=None, n_test=None, starts=None, init_params=None, window=None,
                 fold_smooth_feat_thr=None, fold_smooth_agg_thr=None, y_min=None, y_max=None, fold_y_min=None, fold_y_max=None):
        # TransformedTargetRegressor(MinMaxScaler()): float64 column extrema of the targets ([M, T]; per CV fold [M, K, T]), which the
        # transformer and the detector's scaler both saw; None without one (scale / offset are then float32)
        self.y_min, self.y_max, self.fold_y_min, self.fold_y_max = y_min, y_max, fold_y_min, fold_y_max
        # the detector's smoothing window and every fold's thresholds at it ([M, K, T], [M, K]); None without a window
        self.window, self.fold_smooth_feat_thr, self.fold_smooth_agg_thr = window, fold_smooth_feat_thr, fold_smooth_agg_thr
        # EarlyStopping: epochs each fit ran and its best epoch (-1: none) ([M]; per CV fold [M, K]); None without the callback.
        # History entries past a fit's epochs_run are NaN.  `epochs` is the configured count (keras History.params["epochs"]).
        self.epochs = epochs
        # per machine: rows [M], test rows of every fold [M], first test row of fold k [M, K] (its TimeSeriesSplit)
        self.rows, self.n_test, self.starts = rows, n_test, starts
        self.init_params = init_params                                         # [S, stride] initial parameters (keep_init_params), or None
        self.epochs_run, self.best_epoch, self.fold_epochs_run, self.fold_best_epoch = epochs_run, best_epoch, fold_epochs_run, fold_best_epoch
        # Keras validation_split: per-epoch loss / accuracy on the held-out tail ([M, epochs]; per CV fold [M, K, epochs]); None without one
        self.val_loss, self.val_acc, self.fold_val_loss, self.fold_val_acc = val_loss, val_acc, fold_val_loss, fold_val_acc
        # optimizer steps per epoch of every machine's final fit (keras History.params["steps"]) [M]; steps_per_epoch: machine 0's
        self.machine_steps = None if steps_per_epoch is None else np.atleast_1d(np.asarray(steps_per_epoch, dtype=np.int64))
        self.steps_per_epoch = None if steps_per_epoch is None else int(self.machine_steps[0])
        # float64 scale_ / min_ of the MinMaxScaler in front of the network ([M, T]; per CV fold [M, K, T]); None without one
        self.in_scale, self.in_offset, self.fold_in_scale, self.fold_in_offset = in_scale, in_offset, fold_in_scale, fold_in_offset
        self.eng, self.n_machines, self.n_splits = eng, n_machines, n_splits
        self.fold_params = fold_params                                         # [M, K, stride]: the CV models (cv["estimator"] of the reference)
        self.cv_moments = cv_moments                                           # [M, K, 5, T] float64: gb_cv_moments of every fold's test block
        self.params, self.scale, self.offset = params, scale, offset          # [M, stride], [M, T], [M, T]
        self.feat_thr, self.agg_thr = feat_thr, agg_thr                        # [M, T], [M]  (last fold, diff.py:257-264)
        self.loss, self.acc = loss, acc                                        # [M, epochs]
        self.fold_loss, self.fold_feat_thr, self.fold_agg_thr = fold_loss, fold_feat_thr, fold_agg_thr  # [M, K, ...]

    @staticmethod
    def _fill_minmax(sc, scale, offset, names):
        """Give a MinMaxScaler the fitted attributes sklearn's ``fit`` would have left (feature_range (0, 1))."""
        sc.scale_, sc.min_ = scale, offset
        sc.data_min_ = -offset / scale
        sc.data_range_ = 1.0 / scale
        sc.data_max_ = sc.data_min_ + sc.data_range_
        sc.n_features_in_, sc.n_samples_seen_ = len(scale), 0
        if names is not None and all(isinstance(n, str) for n in names):
            sc.feature_names_in_ = np.asarray(names, dtype=object)
        return sc

    def detector(self, m: int, tags=None, template=None, input_tags=None):
        """
        Materialise machine ``m`` as a ``DiffBasedAnomalyDetector`` (picklable, servable by gordo.server).  ``template``: an
        unfitted detector built from the machine's own definition (same architecture) to fill in, so that ``kind`` and the
        other constructor arguments survive into ``get_params`` / ``into_definition``.
        """
        from sklearn.preprocessing import MinMaxScaler

        from .machine.model.anomaly.diff import DiffBasedAnomalyDetector
        from .machine.model.factories.specs import FFNetSpec
        from .machine.model.models import FittedNet, KerasAutoEncoder

        eng = self.eng
        T = eng.n_out
        tags = list(tags) if tags is not None else list(range(T))
        host = lambda t: None if t is None else t[m].cpu().numpy()  # noqa: E731
        ttr = None
        if template is not None:
            ttr, est, ae = _ff_template(eng, template, self.y_min is not None, self.in_scale is not None, self.params[m : m + 1])
            if self.in_scale is not None:
                self._fill_minmax(est.steps[0][1], host(self.in_scale), host(self.in_offset), input_tags)
        elif self.y_min is not None:
            raise ValueError("a fleet with a target transformer materialises its detectors from a template")
        else:
            ae = KerasAutoEncoder(kind="feedforward_model", n_features=eng.n_in, n_features_out=T)
            spec = FFNetSpec(list(eng.dims), list(eng.acts), list(eng.l1))
            ae.model = FittedNet(spec, eng.unpack_params(self.params[m : m + 1])[0])
        _fill_history(ae, ae.model.spec.metrics, self.epochs, int(self.machine_steps[m]), host(self.loss), host(self.acc), host(self.val_loss),
                      host(self.val_acc), host(self.epochs_run))
        if ttr is not None:
            _fill_target_regressor(ttr, est, self.y_min[m], self.y_max[m], self.rows[m])
            sc = _fill_minmax_from_extrema(MinMaxScaler(), self.y_min[m], self.y_max[m], self.rows[m], tags)
        else:
            sc = self._fill_minmax(MinMaxScaler(), host(self.scale).astype(np.float64), host(self.offset).astype(np.float64), None)
        if template is not None:
            det = template
            det.scaler = sc
        else:
            det = DiffBasedAnomalyDetector(base_estimator=ae, scaler=sc, **({} if self.window is None else {"window": self.window}))
        return _fill_thresholds(det, tags, host(self.feat_thr), host(self.agg_thr), host(self.fold_feat_thr), host(self.fold_agg_thr), self.window,
                                host(self.fold_smooth_feat_thr), host(self.fold_smooth_agg_thr))


def dump_fleet(fb: "FleetBuild", root: str, names: Sequence[str], tags: Optional[Sequence[Sequence[str]]] = None,
               metadata: Optional[Dict[str, dict]] = None, info: Optional[dict] = None) -> List[str]:
    """
    Writes every machine of a ``FleetBuild`` in the layout ``gordo.serializer.dump`` produces and ``gordo.serializer.load`` /
    ``load_metadata`` / gordo.server read (gordo/serializer/serializer.py:149-196): ``<root>/<name>/model.pkl`` (the pickled
    detector), ``metadata.json`` (user metadata + the model's own ``get_metadata()`` under ``metadata.build_metadata.model.
    model_meta`` -- where ModelBuilder puts it, gordo/builder/build_model.py:291-321) and, when given, ``info.json``.
    Returns the directories written.
    """
    import json
    import os
    import pickle

    out = []
    for m, name in enumerate(names):
        det = fb.detector(m, tags=None if tags is None else tags[m])
        dest = os.path.join(root, name)
        os.makedirs(dest, exist_ok=True)
        with open(os.path.join(dest, "model.pkl"), "wb") as f:
            pickle.dump(det, f)
        meta = dict((metadata or {}).get(name, {}))
        meta.setdefault("name", name)
        meta.setdefault("metadata", {}).setdefault("build_metadata", {}).setdefault("model", {})["model_meta"] = det.get_metadata()
        with open(os.path.join(dest, "metadata.json"), "w") as f:
            json.dump(meta, f, default=str)
        if info is not None:
            with open(os.path.join(dest, "info.json"), "w") as f:
                json.dump(info, f, default=str)
        out.append(dest)
    return out


def _keras_initial_params(eng: "engine.FFEngine", n_slots: int, generator):
    """Fresh Dense stacks for ``n_slots`` fits: glorot-uniform kernels and, as Keras initialises them, zero biases."""
    params = random_glorot_params(eng, n_slots, generator)
    ofs = 0
    for i, o in zip(eng.dims[:-1], eng.dims[1:]):
        ofs += i * o
        params[:, ofs:ofs + o] = 0
        ofs += o
    return params


def _fit_slots(eng, params, fit_jobs, n_jobs, max_rows, x, y, split, row_map, n_machines, epochs, batch_size, shuffle, adam, seed,
               validation_batch_size, early_stopping, loss="mse", optimizer=None, reg=None, dropout=None):
    """
    The one fit launch of a bucket (job j trains a slot of machine j mod n_machines), with held-out positions and a row map where
    ``split`` is given and an EarlyStopping callback (one for all machines or one per machine) where ``early_stopping`` is.
    Returns (loss, acc, val_loss, val_acc, epochs_run, best_epoch): val_* rows NaN for jobs without held-out positions,
    epochs_run / best_epoch None without a callback.
    """
    stop = _slot_stops(early_stopping, n_machines, n_jobs)
    hist, acc, val_loss, val_acc, *ran, _ = eng.fit_split(
        params, fit_jobs, n_jobs, max_rows, x, y, split=split, row_map=row_map, val_batch=validation_batch_size or batch_size, epochs=epochs,
        batch_size=batch_size, shuffle=shuffle, adam=adam, seed=seed, stop=stop, loss=loss, optimizer=optimizer, reg=reg, dropout=dropout)
    epochs_run, best_epoch = ran or (None, None)
    return hist, acc, val_loss, val_acc, epochs_run, best_epoch


class _FitRequest:
    """The arguments of a bucket's one fit launch (``_fit_slots``), as a build hands them to ``build_joined``."""

    def __init__(self, eng, params, fit_jobs, n_jobs, max_rows, x, y, split, row_map, n_machines, epochs, batch_size, shuffle, adam, seed,
                 validation_batch_size, early_stopping, loss="mse", optimizer=None, reg=None, dropout=None):
        self.eng, self.params, self.fit_jobs, self.n_jobs, self.max_rows = eng, params, fit_jobs, n_jobs, max_rows
        self.x, self.y, self.split, self.row_map, self.n_machines, self.early_stopping = x, y, split, row_map, n_machines, early_stopping
        self.fit_kw = dict(val_batch=validation_batch_size or batch_size, epochs=epochs, batch_size=batch_size, shuffle=shuffle, adam=adam,
                           seed=seed, loss=loss, optimizer=optimizer, reg=reg, dropout=dropout)
        self.args = (eng, params, fit_jobs, n_jobs, max_rows, x, y, split, row_map, n_machines, epochs, batch_size, shuffle, adam, seed,
                     validation_batch_size, early_stopping, loss, optimizer, reg, dropout)

    def launch_key(self):
        """What fits of one launch share: the memory plan, every fit argument but the network, and the entry point."""
        return (engine.fit_plan(self.eng.dims, self.eng.acts, self.eng.l1), repr(sorted(self.fit_kw.items())), self.split is None,
                self.early_stopping is None)


def _fit_requests_together(reqs: Sequence[_FitRequest]):
    """The fit launches of ``reqs`` that share a launch key, as one gb_ffae_fit_group launch: ``_fit_slots``'s result for each."""
    groups = [engine.FitGroup(r.eng, r.params, r.fit_jobs, r.n_jobs, r.max_rows, r.x, r.y, split=r.split, row_map=r.row_map,
                              stop=_slot_stops(r.early_stopping, r.n_machines, r.n_jobs)) for r in reqs]
    out = []
    for res in engine.fit_group(groups, **reqs[0].fit_kw):
        hist, acc, val_loss, val_acc, *ran, _ = res
        epochs_run, best_epoch = ran or (None, None)
        out.append((hist, acc, val_loss, val_acc, epochs_run, best_epoch))
    return out


def build_joined(builds: Sequence) -> list:
    """
    Several batched builds (``build_fleet.steps(...)`` / ``build_kfold_fleet.steps(...)`` generators) with their fits joined: every
    build runs up to its fit, the fits that share a memory plan and every fit argument but the network go out as one
    gb_ffae_fit_group launch (a fit alone keeps its own launch), and every build finishes with its own fit's result.  Each build's
    result is exactly what it gives on its own.  Returns the builds' results in order.
    """
    builds = list(builds)
    reqs = [next(b) for b in builds]
    results = [None] * len(reqs)
    launches: Dict[tuple, List[int]] = {}
    for i, r in enumerate(reqs):
        launches.setdefault(r.launch_key(), []).append(i)
    for key, idx in launches.items():
        if len(idx) == 1 or key[0] is None:
            for i in idx:
                results[i] = _fit_slots(*reqs[i].args)
        else:
            for i, res in zip(idx, _fit_requests_together([reqs[i] for i in idx])):
                results[i] = res
    out = []
    for b, res in zip(builds, results):
        try:
            b.send(res)
        except StopIteration as done:
            out.append(done.value)
        else:
            raise RuntimeError("a batched build asked for a second fit")
    return out


def _fit_joined(steps):
    """A batched build from its generator of steps (which yields its one ``_FitRequest`` and receives ``_fit_slots``'s result):
    the build on its own, its fit one launch; ``.steps`` keeps the generator for ``build_joined``."""

    @functools.wraps(steps)
    def build(*args, **kwargs):
        return build_joined([steps(*args, **kwargs)])[0]

    build.steps = steps
    return build


def _slot_stops(early_stopping, n_machines: int, n_slots: int):
    """The stop records of ``n_slots`` fits, slot s applying machine s mod M's EarlyStopping callback (``early_stopping``: one for
    every machine or one per machine), or None without a callback."""
    if early_stopping is None:
        return None
    per_machine = list(early_stopping) if isinstance(early_stopping, (list, tuple)) else [early_stopping] * n_machines
    if len(per_machine) != n_machines:
        raise ValueError(f"early_stopping: {len(per_machine)} callbacks for {n_machines} machines")
    return engine.make_stop([per_machine[s % n_machines] for s in range(n_slots)])


def _keras_train_rows(slot_n, validation_split):
    """Keras' ``validation_split``: the rows each slot of ``slot_n`` rows trains on (int64), the rest held out."""
    vsplit = float(validation_split or 0.0)
    n_train = np.asarray([int(math.floor(v * (1.0 - vsplit))) if 0.0 < vsplit < 1.0 else int(v) for v in slot_n], dtype=np.int64)
    if n_train.min() < 1:
        raise ValueError(f"validation_split {vsplit} leaves the {int(slot_n.min())}-row slot without a training row")
    return n_train


def _slot_copies(n, row0, n_splits: int, device):
    """
    Every slot's own copy of its machine's rows, for slots that scale them on their own: the stacked machines (rows ``n``, first
    rows ``row0``) repeated K + 1 times, slot s (finals, then fold k of machine m at M + k*M + m) at copy0[s].  Returns (copy0,
    the device jobs that copy slot s's machine rows to copy0[s]).
    """
    base = np.tile(row0, n_splits + 1)
    copy0 = np.arange(n_splits + 1, dtype=np.int64).repeat(len(n)) * int(n.sum()) + base
    return copy0, engine.jobs_to_device(engine.make_jobs(np.arange(len(base)), np.tile(n, n_splits + 1), base, copy0), device)


def _machine_rows(x, rows):
    """
    (row counts [M], first rows [M]) of the machines stacked in ``x``: ``rows`` is an int, M = len(x) // rows machines of that
    many rows each, or one count per machine.  Machine m owns rows [row0[m], row0[m] + rows[m]), row0 the prefix sum.
    """
    if np.ndim(rows) == 0:
        n = np.full(x.shape[0] // int(rows), int(rows), dtype=np.int64)
    else:
        n = np.asarray(rows, dtype=np.int64)
        if n.ndim != 1 or len(n) == 0 or (n < 1).any() or int(n.sum()) > x.shape[0]:
            raise ValueError(f"rows: {n.size} per-machine counts (sum {int(n.sum())}) for {x.shape[0]} stacked rows")
    return n, _prefix(n)


def _prefix(counts) -> np.ndarray:
    """Exclusive prefix sums (int64): the first row of every block laid out back to back."""
    return np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)


def tss_layout(rows, n_splits: int):
    """
    Every machine's sklearn ``TimeSeriesSplit(n_splits)`` over its own ``rows[m]`` rows: (test rows [M], starts [M, K]), fold k of
    machine m training on [0, starts[m, k]) and testing the next test[m] rows.
    """
    n, K = np.asarray(rows, dtype=np.int64), int(n_splits)
    test = n // (K + 1)
    if (test == 0).any():
        raise ValueError("Too many splits for number of samples")
    return test, n[:, None] - (K - np.arange(K))[None, :] * test[:, None]


def shuffle_maps(slot_rows):
    """
    The row maps of ``DiffBasedAnomalyDetector(shuffle=True)`` for slots of ``slot_rows`` rows: ``sklearn.utils.shuffle(arange(n),
    random_state=0)`` once per distinct length, back to back (int32), and every slot's offset into them (int64).
    """
    lengths = list(dict.fromkeys(int(v) for v in slot_rows))  # in slot order
    first = dict(zip(lengths, _prefix(lengths)))
    maps = np.concatenate([sk_shuffle(np.arange(v), random_state=0) for v in lengths]).astype(np.int32)
    return maps, np.asarray([first[int(v)] for v in slot_rows], dtype=np.int64)


@_fit_joined
def build_fleet(eng: "engine.FFEngine", x, y, rows, epochs: int = 1, batch_size: int = 32, n_splits: int = 3, seed: int = 0,
                adam: Optional[Dict[str, float]] = None, shuffle: bool = True, generator=None, input_scaler: bool = False,
                detector_shuffle: bool = False, validation_split: float = 0.0, validation_batch_size: Optional[int] = None,
                early_stopping=None, loss: str = "mse", optimizer=None, keep_init_params: bool = False, reg=None,
                window: Optional[int] = None, dropout=None, target_scaler: bool = False) -> FleetBuild:
    """
    The batched form of ``gordo build`` for one architecture bucket: for every machine the 3-fold TimeSeriesSplit
    cross-validation (fit on each prefix, thresholds from the following test block: diff.py:176-266) and the final fit on
    all rows (build_model.py:257-321) -- ``(n_splits + 1) * n_machines`` fits in ONE gb_ffae_fit launch (one CTA per fit),
    then fold scoring, threshold reduction and scaler statistics, each a single launch.

    x, y: device tensors of the machines' rows stacked.  ``rows``: an int, machine m owning rows [m*rows, (m+1)*rows), or one
    count per machine, machine m owning rows [row0[m], row0[m] + rows[m]) with row0 the prefix sum.  Every machine gets its own
    TimeSeriesSplit (``test = rows[m] // (n_splits + 1)``), and each fit, scoring and reduction job covers its own slot's rows.

    ``input_scaler``: the network sits behind a MinMaxScaler (``Pipeline([MinMaxScaler(), KerasAutoEncoder])``, the shape of
    gordo's example configs, examples/config.yaml:74-81).  Inside cross validation every fold clone fits that scaler on its
    own training prefix, so every fit slot gets its own scaled copy of its machine's rows -- sklearn's float64 arithmetic on
    the exact column extrema (``gb_minmax_fit`` finds them, ``gb_affine_f64`` applies them), rounded to float32 once.

    ``detector_shuffle``: ``DiffBasedAnomalyDetector(shuffle=True)``, which hands its estimator its rows in the order of
    ``sklearn.utils.shuffle(X, y, random_state=0)`` (the final fit on all rows, every CV clone on its own prefix).  The fits read
    the rows through that order (a row map; one per distinct slot length, shared by every slot of that length) instead of a
    shuffled copy.
    ``validation_split``: Keras' hold-out of the estimator: of a slot's ``n`` (shuffled) rows it trains on the first
    ``floor(n * (1 - validation_split))`` and reports the loss and accuracy of the rest after every epoch (``val_loss``,
    ``val_accuracy``; in batches of ``validation_batch_size``, default ``batch_size``), computed inside the same fit launch.
    The scalers still see all ``n`` rows of a slot, as the detector's and the Pipeline's do.
    ``early_stopping``: the estimator's Keras ``EarlyStopping`` callback -- one for every machine, or a sequence of one per machine
    (``engine.make_stop`` takes any form).  Every slot of machine m, the final fit and each CV fold, applies m's rule at the end of
    each of its epochs inside the fit launch (gb_ffae_fit_stop), as sklearn's clone hands every fold the same callbacks.  The
    result then carries ``epochs_run`` / ``best_epoch``; history entries past a fit's ``epochs_run`` are NaN.
    ``loss``: the estimator's canonical Keras loss name (``FFNetSpec.loss``), trained on and reported by every fit.
    ``optimizer``: None (Adam from ``adam``) or the estimator's (name, record) (``factories.specs.fit_optimizer``), for every fit.
    ``reg``: None or the estimator's weight regularizers (``factories.specs.fit_reg``), for every fit.
    ``dropout``: None or the estimator's Dropout rates (``factories.specs.fit_dropout``), for every fit; each slot draws its masks
    under its own key (gb_dense_dropout).
    ``keep_init_params``: keep the initial parameters of every slot on the result (``init_params``).
    ``window``: the detector's smoothing window.  Every fold then also gets its thresholds at that window (the detector's
    ``smooth_*`` attributes), from the same pass over the fold scores as its 6-row thresholds (gb_thresholds_pair).
    ``target_scaler``: the estimator is ``TransformedTargetRegressor(transformer=MinMaxScaler(), regressor=...)``; x and y are then
    float64, as the estimator receives them.  Every slot's transformer and the detector's scaler take the float64 extrema of that
    slot's targets (gb_minmax_f64; held-out rows included), and the slot trains on its own float32 copy of its scaled targets
    (gb_affine_f64; one copy serves both scalers when y is x and the network is behind an input scaler).  The fold models'
    predictions go through sklearn's float32 inverse of the fold's transformer and are scored in float64 against the float64
    targets in one launch (gb_minmax_inverse_score_f64), as the per-machine detector scores a foreign estimator, so the fold
    thresholds and the result's ``fold_*_thr`` are float64; the metric moments are in target units.
    """
    torch = engine._torch()
    dev = eng.device
    if target_scaler and (x.dtype != torch.float64 or y.dtype != torch.float64):
        raise ValueError(f"build_fleet(target_scaler=True) takes float64 x and y, got {x.dtype} / {y.dtype}")
    n, row0 = _machine_rows(x, rows)
    M, K = len(n), n_splits
    test, starts = tss_layout(n, K)
    g = generator or torch.Generator(device=dev).manual_seed(seed)
    # slots: [0, M) final models, then fold k of machine m at M + k*M + m
    S = M * (K + 1)
    params = _keras_initial_params(eng, S, g)
    init_params = params.clone() if keep_init_params else None
    N = int(n.max())                                             # the longest slot
    slot_n = np.concatenate([n] + [starts[:, k] for k in range(K)])  # every row of a slot: what its scalers see
    n_train = _keras_train_rows(slot_n, validation_split)
    held_out = bool((n_train != slot_n).any())
    fit_x = np.tile(row0, K + 1)                                 # first row of every slot's machine
    split = row_map = None
    if detector_shuffle or held_out:
        map_ofs = np.full(S, -1, dtype=np.int64)
        if detector_shuffle:
            maps, map_ofs = shuffle_maps(slot_n)
            row_map = torch.from_numpy(maps).to(dev)
        split = engine.make_split(slot_n - n_train, map_ofs)
    in_scale = in_offset = None
    y64 = y_lo = y_hi = None
    if target_scaler:
        y64, same_y, total = y, y is x, int(n.sum())
        prefix_jobs = engine.jobs_to_device(engine.make_jobs(np.arange(S), slot_n, fit_x), dev)
        y_lo, y_hi = _slot_extrema(prefix_jobs, S, N, y)
        t_scale_h, t_offset_h = _minmax_attributes(y_lo, y_hi)
        t_scale, t_offset = _f64(t_scale_h, dev), _f64(t_offset_h, dev)
        copy0, copy_jobs = _slot_copies(n, row0, K, dev)  # slot s works on its own copies of its machine's rows
        if input_scaler:
            in_lo, in_hi = (y_lo, y_hi) if same_y else _slot_extrema(prefix_jobs, S, N, x)
            in_scale, in_offset = (_f64(v, dev) for v in _minmax_attributes(in_lo, in_hi))
            x = engine.affine_f64(copy_jobs, S, N, x, in_scale, in_offset, out_rows=(K + 1) * total)
        else:
            x = x[:total].to(torch.float32).repeat(K + 1, 1)
        # the same extrema and the same arithmetic give the same copy when the input scaler and the transformer see one array
        y = x if (input_scaler and same_y) else engine.affine_f64(copy_jobs, S, N, y64, t_scale, t_offset, out_rows=(K + 1) * total)
        fit_x = copy0
    elif input_scaler:
        prefix_jobs = engine.jobs_to_device(engine.make_jobs(np.arange(S), slot_n, fit_x), dev)
        _, _, lo, hi = engine.minmax_fit(prefix_jobs, S, N, x, eng.n_in, S, dev, return_minmax=True)
        lo, span = lo.double(), hi.double() - lo.double()
        span[~(span >= 10 * np.finfo(np.float64).eps)] = 1.0  # sklearn _handle_zeros_in_scale (also catches all-NaN columns)
        in_scale = 1.0 / span
        in_offset = -lo * in_scale
        total = int(n.sum())
        copy0, copy_jobs = _slot_copies(n, row0, K, dev)  # slot s works on its own copy of its machine's rows
        x = engine.affine_f64(copy_jobs, S, N, x.double(), in_scale.contiguous(), in_offset.contiguous(), out_rows=(K + 1) * total)
        y = y[:total].repeat(K + 1, 1)
        fit_x = copy0
    fit_jobs = engine.jobs_to_device(engine.make_jobs(np.arange(S), n_train, fit_x), dev)
    hist, acc, val_loss, val_acc, epochs_run, best_epoch = yield _FitRequest(
        eng, params, fit_jobs, S, N, x, y, split, row_map, M, epochs, batch_size, shuffle, adam, seed, validation_batch_size, early_stopping,
        loss, optimizer, reg, dropout)
    if not held_out:
        val_loss = val_acc = None
    # scalers: final on all rows, fold k on its training prefix (diff.py:173 inside each CV clone), held-out rows included
    if target_scaler:  # the detector's scaler saw the float64 targets too
        scale, offset = t_scale, t_offset
    else:
        all_jobs = engine.jobs_to_device(engine.make_jobs(np.arange(S), slot_n, fit_x), dev) if held_out else fit_jobs
        scale, offset = eng.minmax_fit(all_jobs, S, N, y, S)
    # fold scoring on the test blocks: job k*M + m scores fold k of machine m, outputs back to back
    KM = K * M
    fk, fm = np.repeat(np.arange(K), M), np.tile(np.arange(M), K)
    sc_n = test[fm]
    sc_jobs = engine.jobs_to_device(engine.make_jobs(M + np.arange(KM), sc_n, fit_x[M:] + starts[fm, fk], _prefix(sc_n)), dev)
    max_test = int(test.max())
    want = ("tag-anomaly-unscaled", "total-anomaly-scaled")
    if target_scaler:
        # the fold models' outputs, then sklearn's float32 inverse of the fold's transformer and float64 scoring against the float64
        # targets (at their own rows, x_row) with the fold detector's multiplier, transform(1) - transform(0)
        pred = eng.infer_score(params, sc_jobs, KM, max_test, x, out_rows=int(sc_n.sum()))["model-output"]
        mom_jobs = engine.jobs_to_device(engine.make_jobs(M + np.arange(KM), sc_n, row0[fm] + starts[fm, fk], _prefix(sc_n)), dev)
        res = engine.minmax_inverse_score_f64(mom_jobs, KM, max_test, pred, y64, t_scale, t_offset, scale=_f64((t_scale_h + t_offset_h) - t_offset_h, dev),
                                              want=want, out_rows=int(sc_n.sum()), out={"model-output": pred})
        y_true = y64.to(torch.float32)
    else:
        res = eng.infer_score(params, sc_jobs, KM, max_test, x, y, scale, out_rows=int(sc_n.sum()), want=want)
        mom_jobs, y_true = sc_jobs, y
    fold_sfeat = fold_sagg = None
    if window is None:
        feat, agg = eng.thresholds(sc_jobs, KM, max_test, res["tag-anomaly-unscaled"], res["total-anomaly-scaled"], S, window=6)
    else:
        feat, agg, sfeat, sagg = eng.thresholds_pair(sc_jobs, KM, max_test, res["tag-anomaly-unscaled"], res["total-anomaly-scaled"], S, 6, int(window))
        fold_sfeat = _device_folds(sfeat[M:], M).contiguous()
        fold_sagg = _device_folds(sagg[M:], M).contiguous()
    # the evaluation metrics of ModelBuilder's cross validation (build_model.py:250-289) reduce to five sums per (fold, tag)
    moments = _device_folds(engine.cv_moments(mom_jobs, KM, res["model-output"], y_true, eng.n_out), M).contiguous()
    finals = lambda t: None if t is None else t[:M]  # noqa: E731
    folds = lambda t: None if t is None else _device_folds(t[M:], M)  # noqa: E731
    finals_c = lambda t: None if t is None else t[:M].contiguous()  # noqa: E731
    folds_c = lambda t: None if t is None else folds(t).contiguous()  # noqa: E731
    fold_params, fold_feat, fold_agg = folds_c(params), folds_c(feat), folds_c(agg)
    return FleetBuild(eng, M, K, params[:M].contiguous(), scale[:M].contiguous(), offset[:M].contiguous(), fold_feat[:, K - 1].contiguous(),
                      fold_agg[:, K - 1].contiguous(), hist[:M], acc[:M], folds(hist), fold_feat, fold_agg,
                      fold_params=fold_params, cv_moments=moments, in_scale=finals_c(in_scale), in_offset=finals_c(in_offset),
                      fold_in_scale=folds_c(in_scale), fold_in_offset=folds_c(in_offset),
                      steps_per_epoch=(n_train[:M] + int(batch_size) - 1) // int(batch_size),
                      val_loss=finals(val_loss), val_acc=finals(val_acc), fold_val_loss=folds(val_loss), fold_val_acc=folds(val_acc), epochs=int(epochs),
                      epochs_run=finals(epochs_run), best_epoch=finals(best_epoch), fold_epochs_run=folds(epochs_run), fold_best_epoch=folds(best_epoch),
                      rows=n, n_test=test, starts=starts, init_params=init_params, window=None if window is None else int(window),
                      fold_smooth_feat_thr=fold_sfeat, fold_smooth_agg_thr=fold_sagg,
                      **({} if y_lo is None else dict(y_min=y_lo[:M], y_max=y_hi[:M], fold_y_min=_folds(y_lo[M:], M), fold_y_max=_folds(y_hi[M:], M))))


def _f64(a, device):
    """A host array as a float64 device tensor."""
    return engine._torch().from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(device)


def _slot_extrema(jobs_dev, n_jobs, max_rows, a64):
    """Float64 column (min, max) of every job's rows as host arrays [n_jobs, cols] (gb_minmax_f64); ValueError when a column has no
    finite value."""
    lo, hi = (t.cpu().numpy() for t in engine.minmax_f64(jobs_dev, n_jobs, max_rows, a64, n_jobs))
    if not (np.isfinite(lo).all() and np.isfinite(hi).all()):
        raise ValueError("a column without finite values in a training block")
    return lo, hi


def _folds(a, n_machines: int):
    """Fold-ordered host rows [K*M, ...] (fold k of machine m at k*M + m: the rows of a slot-ordered array from M on, or one per
    fold job) -> every machine's folds [M, K, ...], contiguous."""
    return np.ascontiguousarray(np.swapaxes(a.reshape((-1, n_machines) + a.shape[1:]), 0, 1))


def _device_folds(t, n_machines: int):
    """``_folds`` of a device tensor, as a view."""
    return t.view((-1, n_machines) + tuple(t.shape[1:])).transpose(0, 1)


# ------------------------------------------------------------------------------------------------ fleet build of LSTM detectors
def _minmax_attributes(lo: np.ndarray, hi: np.ndarray):
    """(scale_, min_) of a MinMaxScaler (feature_range (0, 1)) from float64 column extrema, with sklearn's own arithmetic."""
    denom = hi - lo
    denom[denom < 10 * np.finfo(np.float64).eps] = 1.0  # _handle_zeros_in_scale
    scale = 1.0 / denom
    return scale, 0.0 - lo * scale


def _fill_minmax_from_extrema(sc, lo, hi, n_samples, names):
    """Give a MinMaxScaler exactly the attributes sklearn's ``fit`` leaves for data with column extrema ``lo`` / ``hi``."""
    sc.n_samples_seen_, sc.n_features_in_ = int(n_samples), len(lo)
    sc.data_min_, sc.data_max_, sc.data_range_ = lo.copy(), hi.copy(), hi - lo
    sc.scale_, sc.min_ = _minmax_attributes(lo, hi)
    if names is not None and all(isinstance(n, str) for n in names):
        sc.feature_names_in_ = np.asarray(names, dtype=object)
    return sc


def _target_regressor_of(est, target_scaler: bool):
    """(the TransformedTargetRegressor or None, the estimator to fill: a clone of its regressor, or ``est`` itself) of a template's
    base estimator; ValueError when the template and the fleet disagree on the target transformer."""
    from sklearn.base import clone
    from sklearn.compose import TransformedTargetRegressor

    ttr = est if isinstance(est, TransformedTargetRegressor) else None
    if (ttr is not None) != bool(target_scaler):
        raise ValueError("the template's target transformer and the fleet's do not match")
    return ttr, (clone(ttr.regressor) if ttr is not None else est)


def _fill_target_regressor(ttr, reg, lo, hi, n_samples):
    """What ``TransformedTargetRegressor.fit`` leaves: the transformer fitted on the target array (extrema ``lo`` / ``hi``), the
    fitted regressor clone ``reg``, and the regressor's input names."""
    from sklearn.base import clone

    ttr._training_dim = 2
    ttr.transformer_ = _fill_minmax_from_extrema(clone(ttr.transformer), lo, hi, n_samples, None)
    ttr.regressor_ = reg
    if hasattr(reg, "feature_names_in_"):
        ttr.feature_names_in_ = reg.feature_names_in_
    return ttr


class LSTMFleetBuild:
    """
    Result of ``build_lstm_fleet``: what ``ModelBuilder._build`` produces for one LSTM machine -- final weights, target scaler,
    CV thresholds per fold and final, loss histories, CV metric moments -- for all machines of a bucket.  Slot layout of
    ``init_params``: final models at [0, M), fold k of machine m at M + k*M + m.  Arrays named ``fold_*`` are [M, K, ...].
    """

    def __init__(self, eng, n_machines, n_splits, rows, lookahead, batch_size, starts, n_test, params, fold_params, init_params, loss, acc,
                 fold_loss, fold_acc, y_min, y_max, fold_y_min, fold_y_max, feat_thr, agg_thr, fold_feat_thr, fold_agg_thr, cv_moments,
                 fold_predictions, in_min=None, in_max=None, fold_in_min=None, fold_in_max=None, epochs=None, epochs_run=None, best_epoch=None,
                 fold_epochs_run=None, fold_best_epoch=None, window=None, fold_smooth_feat_thr=None, fold_smooth_agg_thr=None,
                 target_scaler=False):
        # the estimator is a TransformedTargetRegressor(MinMaxScaler()), whose transformer saw the same targets as the detector's
        # scaler (y_min / y_max); fold_predictions are then in target units
        self.target_scaler = bool(target_scaler)
        # the detector's smoothing window and every fold's thresholds at it ([M, K, T], [M, K] float64); None without a window
        self.window, self.fold_smooth_feat_thr, self.fold_smooth_agg_thr = window, fold_smooth_feat_thr, fold_smooth_agg_thr
        # EarlyStopping: epochs each fit ran and its best epoch (-1: none) ([M]; per CV fold [M, K]) as int32 host arrays; None without
        # the callback.  History entries past a fit's epochs_run are NaN.  `epochs` is the configured count (History.params["epochs"]).
        self.epochs = epochs
        self.epochs_run, self.best_epoch, self.fold_epochs_run, self.fold_best_epoch = epochs_run, best_epoch, fold_epochs_run, fold_best_epoch
        self.eng, self.n_machines, self.n_splits = eng, n_machines, n_splits
        self.rows = np.asarray(rows, dtype=np.int64)          # [M] rows of every machine
        self.lookahead, self.batch_size = lookahead, batch_size
        # optimizer steps per epoch of every machine's final fit (History.params["steps"]) [M]; steps_per_epoch: machine 0's
        self.machine_steps = -(-(self.rows - eng.lookback + 1 - lookahead) // batch_size)
        self.steps_per_epoch = int(self.machine_steps[0])
        # per machine: first test row of every fold [M, K] and predictions per test block [M]; starts / n_test: machine 0's
        self.machine_starts, self.machine_n_test = np.asarray(starts, dtype=np.int64), np.asarray(n_test, dtype=np.int64)
        self.starts, self.n_test = [int(v) for v in self.machine_starts[0]], int(self.machine_n_test[0])
        self.params, self.fold_params, self.init_params = params, fold_params, init_params  # device float32 ([S, stride] or None)
        self.loss, self.acc, self.fold_loss, self.fold_acc = loss, acc, fold_loss, fold_acc   # [M, epochs], [M, K, epochs]
        # float64 column extrema of the targets (final fit on all rows, fold k on its training prefix): the detector scalers
        self.y_min, self.y_max, self.fold_y_min, self.fold_y_max = y_min, y_max, fold_y_min, fold_y_max
        # the same for the MinMaxScaler in front of the network (None without one)
        self.in_min, self.in_max, self.fold_in_min, self.fold_in_max = in_min, in_max, fold_in_min, fold_in_max
        self.feat_thr, self.agg_thr = feat_thr, agg_thr                                # [M, T], [M] float64 (last fold)
        self.fold_feat_thr, self.fold_agg_thr = fold_feat_thr, fold_agg_thr            # [M, K, T], [M, K] float64
        self.cv_moments = cv_moments                                                   # [M, K, 5, T] float64
        self.fold_predictions = fold_predictions          # fold_predictions[m, k]: [machine_n_test[m], T] float32 (device)

    def detector(self, m: int, tags=None, template=None, input_tags=None):
        """
        Machine ``m`` as a picklable ``DiffBasedAnomalyDetector`` around a ``KerasLSTMAutoEncoder`` / ``KerasLSTMForecast``, with the
        attributes the per-machine build leaves.  ``template``: an unfitted detector from the machine's own definition, filled in
        so that the estimator class, ``kind`` and the other constructor arguments survive.
        """
        from sklearn.pipeline import Pipeline
        from sklearn.preprocessing import MinMaxScaler

        from .machine.model.anomaly.diff import DiffBasedAnomalyDetector
        from .machine.model.models import FittedNet, KerasLSTMAutoEncoder, KerasLSTMForecast

        eng = self.eng
        T = eng.n_out
        tags = list(tags) if tags is not None else list(range(T))
        ttr = None
        if template is not None:
            det = template
            ttr, est = _target_regressor_of(det.base_estimator, self.target_scaler)
            lstm = est.steps[-1][1] if isinstance(est, Pipeline) else est
            if isinstance(est, Pipeline) != (self.in_min is not None):
                raise ValueError("the template's input scaler and the fleet's do not match")
            if lstm.lookahead != self.lookahead:
                raise ValueError("the template's lookahead differs from the fleet's")
            lstm.kwargs.update({"n_features": eng.n_features, "n_features_out": T})
            spec = lstm._build_spec()
            if spec.key() != ("lstm", eng.n_features, tuple(eng.units), tuple(eng.acts), T, eng.out_func, eng.lookback):
                raise ValueError("template architecture differs from the fleet's")
            if isinstance(est, Pipeline):
                _fill_minmax_from_extrema(est.steps[0][1], self.in_min[m], self.in_max[m], self.rows[m], input_tags)
        elif self.target_scaler:
            raise ValueError("a fleet with a target transformer materialises its detectors from a template")
        else:
            cls = KerasLSTMForecast if self.lookahead else KerasLSTMAutoEncoder
            lstm = cls(kind="lstm_model", lookback_window=eng.lookback, batch_size=self.batch_size, encoding_dim=tuple(eng.units),
                       encoding_func=tuple(eng.acts), decoding_dim=(), decoding_func=(), out_func=eng.out_func, n_features=eng.n_features,
                       n_features_out=T)
            spec = lstm._build_spec()
            det = DiffBasedAnomalyDetector(base_estimator=lstm, scaler=MinMaxScaler(), **({} if self.window is None else {"window": self.window}))
        lstm.model = FittedNet(spec, eng.unpack_params(self.params[m : m + 1])[0])
        _fill_history(lstm, spec.metrics, self.epochs, int(self.machine_steps[m]), self.loss[m], self.acc[m],
                      epochs_run=None if self.epochs_run is None else self.epochs_run[m])
        if ttr is not None:
            _fill_target_regressor(ttr, est, self.y_min[m], self.y_max[m], self.rows[m])
        # a fresh scaler: detectors made from definitions without a scaler share the constructor's default MinMaxScaler object
        det.scaler = _fill_minmax_from_extrema(MinMaxScaler(), self.y_min[m], self.y_max[m], self.rows[m], tags)
        windowed = self.window is not None
        return _fill_thresholds(det, tags, self.feat_thr[m], self.agg_thr[m], self.fold_feat_thr[m], self.fold_agg_thr[m], self.window,
                                self.fold_smooth_feat_thr[m] if windowed else None, self.fold_smooth_agg_thr[m] if windowed else None)


class _FoldBlocks:
    """``blocks[m, k]``: the rows of fold k of machine m in an array of per-job blocks laid out back to back (job k*M + m)."""

    def __init__(self, arr, first, count, n_machines):
        self.arr, self.first, self.count, self.M = arr, first, count, n_machines

    def __getitem__(self, mk):
        m, k = mk
        j = k * self.M + m
        return self.arr[int(self.first[j]) : int(self.first[j] + self.count[j])]


def build_lstm_fleet(eng: "engine.LSTMEngine", x, y, rows, lookahead: int = 0, epochs: int = 1, batch_size: int = 32, n_splits: int = 3,
                     seed: int = 0, adam: Optional[Dict[str, float]] = None, input_scaler: bool = False, memory_budget: int = 8 << 30,
                     keep_init_params: bool = False, generator=None, loss: str = "mse", optimizer=None, early_stopping=None,
                     window: Optional[int] = None, target_scaler: bool = False) -> LSTMFleetBuild:
    """
    The batched ``gordo build`` of one bucket of LSTM machines (``DiffBasedAnomalyDetector(KerasLSTMAutoEncoder | KerasLSTMForecast)``,
    the network bare or behind one MinMaxScaler): for every machine the TimeSeriesSplit cross validation and the final fit, as
    ``(n_splits + 1) * n_machines`` jobs of gb_lstm_fit (primer step, ordered batches), then one gb_lstm_infer(_tc) launch for
    every fold model's test block and float64 scoring, thresholds, scaler extrema and metric moments, one launch each.

    x, y: float64 device tensors of the machines' rows stacked; ``rows`` an int (machine m owns rows [m*rows, (m+1)*rows)) or one
    count per machine (machine m owns rows [row0[m], row0[m] + rows[m]), row0 the prefix sum).  ``y`` may be ``x``.  Every machine
    gets its own TimeSeriesSplit, windows and test blocks; a fit launch steps its jobs in lockstep up to its longest one.

    ``batch_size``: up to 32 windows on gb_lstm_fit, up to 256 on gb_lstm_fit_tc (``LSTMEngine.fit_for_batch``).
    ``memory_budget``: bytes of fit workspace (gb_lstm_fit_workspace_bytes, or gb_lstm_fit_tc_workspace_bytes at the batch size)
    one fit launch may take.  Machines are
    trained in chunks that fit it -- all ``n_splits + 1`` fits of a machine in the same chunk; every job's result is the same
    whatever the chunking.  Chunks take the machines shortest first, so each chunk's lockstep loop runs close to its own
    longest machine.  ``keep_init_params``: keep the initial parameters of every slot on the result (``init_params``).
    ``loss``: the estimator's canonical Keras loss name (``LSTMNetSpec.loss``).  ``optimizer``: as in ``build_fleet``.
    ``early_stopping``: the estimator's Keras ``EarlyStopping`` callback -- one for every machine, or a sequence of one per machine
    (``engine.make_stop`` takes any form).  Every slot of machine m, the final fit and each CV fold, applies m's rule at the end of
    each of its epochs inside the fit launch (``LSTMEngine.fit_stop``), as sklearn's clone hands every fold the same callbacks.  The
    result then carries ``epochs_run`` / ``best_epoch``; history entries past a fit's ``epochs_run`` are NaN.  With
    ``restore_best_weights`` the launch also holds a snapshot of every slot, which ``memory_budget`` counts.
    ``window``: the detector's smoothing window, as in ``build_fleet``: every fold also gets its thresholds at that window, from
    the same pass over its float64 fold scores (gb_thresholds_pair_f64).
    ``target_scaler``: the estimator is ``TransformedTargetRegressor(transformer=MinMaxScaler(), regressor=...)``.  Its transformer
    sees all of a slot's rows of y (the detector scaler's extrema), and every slot trains on its own float32 copy of its scaled
    targets (gb_affine_f64).  The fold predictions go through sklearn's float32 inverse of the fold's transformer and are scored in
    float64 in one launch (gb_minmax_inverse_score_f64), so ``fold_predictions`` and the metric moments are in target units.
    """
    torch = engine._torch()
    dev = eng.device
    if x.dtype != torch.float64 or y.dtype != torch.float64:
        raise ValueError(f"build_lstm_fleet takes float64 x and y, got {x.dtype} / {y.dtype}")
    n, row0 = _machine_rows(x, rows)
    M, K, T = len(n), int(n_splits), eng.n_out
    N = int(n.max())                                 # the longest machine
    L, la = eng.lookback, int(lookahead)
    test, starts = tss_layout(n, K)
    n_test = test - L + 1 - la                       # predictions per test block, per machine
    for m in range(M):
        if starts[m, 0] - L + 1 - la < 1 or starts[m, 0] <= L or n_test[m] < 1:
            raise ValueError(f"{int(n[m])} rows leave fold 0 without a training window or a test block without a prediction at lookback_window {L}, "
                             f"lookahead {la}")
    S = M * (K + 1)
    g = generator or torch.Generator(device=dev).manual_seed(int(seed))
    params = eng.initial_params(S, g)
    init_params = params.clone() if keep_init_params else None
    # per slot (final fits, then fold k of machine m at M + k*M + m): training rows / windows and the first row of its machine
    slot_rows = np.concatenate([n] + [starts[:, k] for k in range(K)])
    slot_windows = slot_rows - L + 1 - la            # the estimator's window count
    x_row = np.tile(row0, K + 1)

    def host(t):
        return t.cpu().numpy()

    # target scalers: final on all rows, fold k on its training prefix (diff.py:173 inside each CV clone), float64 like _fit_scaler
    prefix_jobs = engine.jobs_to_device(engine.make_jobs(np.arange(S), slot_rows, x_row), dev)
    y_lo, y_hi = _slot_extrema(prefix_jobs, S, N, y)
    y32 = y.to(torch.float32)
    in_lo = in_hi = None
    total = int(n.sum())
    if input_scaler or target_scaler:  # slot s trains on its own copy of its machine's rows, at x_row[s]
        x_row, copy_jobs = _slot_copies(n, row0, K, dev)
    if input_scaler:
        # every fold clone fits the Pipeline's MinMaxScaler on its own prefix: slot s trains on its own float64-scaled copy of its
        # machine's rows (gb_affine_f64: sklearn's transform, rounded once)
        in_lo, in_hi = (y_lo, y_hi) if y is x else _slot_extrema(prefix_jobs, S, N, x)
        a, b = (_f64(v, dev) for v in _minmax_attributes(in_lo, in_hi))
        xf = engine.affine_f64(copy_jobs, S, N, x, a, b, out_rows=(K + 1) * total)
        yf = y32[:total].repeat(K + 1, 1)
    else:
        xf = y32 if y is x else x.to(torch.float32)
        yf = y32
    if target_scaler:
        # TransformedTargetRegressor(MinMaxScaler()): the transformer saw the extrema above, and slot s trains on its own float32 copy of
        # its scaled targets at x_row[s], laid out as the input scaler's copies are (one copy for both when they see the same array)
        if not input_scaler:
            xf = xf[:total].repeat(K + 1, 1)
        t_scale, t_offset = _minmax_attributes(y_lo, y_hi)
        yf = xf if (input_scaler and y is x) else engine.affine_f64(copy_jobs, S, N, y, _f64(t_scale, dev), _f64(t_offset, dev), out_rows=(K + 1) * total)

    # fits: chunks of whole machines (final + K folds) whose workspace fits the budget
    # (batches above 32 windows train on the tensor-core family, whose workspace grows with the batch)
    fit = eng.fit_for_batch(batch_size)
    per_machine_bytes = eng.fit_workspace_bytes_for_batch(K + 1, batch_size)
    stop, epochs_run, best_epoch = _slot_stops(early_stopping, M, S), None, None
    if stop is not None:
        per_machine_bytes += int(eng.lib.gb_lstm_fit_stop_state_bytes(K + 1))
        if stop["restore_best"].any():  # the snapshot area
            per_machine_bytes += (K + 1) * eng.param_stride * 4
        epochs_run, best_epoch = np.zeros(S, np.int32), np.zeros(S, np.int32)
    chunk = max(1, min(M, int(memory_budget) // max(per_machine_bytes, 1), 65535 // (K + 1)))
    hist = torch.empty((S, epochs), dtype=torch.float32, device=dev)
    acc = torch.empty_like(hist)
    by_length = np.argsort(n, kind="stable")
    for m0 in range(0, M, chunk):
        ms = by_length[m0:m0 + chunk]
        slots = np.concatenate([j * M + ms for j in range(K + 1)])
        idx = torch.from_numpy(slots).to(dev)
        p = params.index_select(0, idx)
        jobs = engine.jobs_to_device(engine.make_jobs(np.arange(len(slots)), slot_windows[slots], x_row[slots]), dev)
        args = (p, jobs, len(slots), int(slot_windows[slots].max()), xf, yf)
        kw = dict(epochs=epochs, batch_size=batch_size, lookahead=la, primer=True, adam=adam, loss=loss, optimizer=optimizer)
        if stop is None:
            cl, ca, _ = fit(*args, **kw)
        else:
            cl, ca, er, be, _ = eng.fit_stop(*args, stop[slots], **kw)
            epochs_run[slots], best_epoch[slots] = host(er), host(be)
        params.index_copy_(0, idx, p)
        hist.index_copy_(0, idx, cl)
        acc.index_copy_(0, idx, ca)

    # fold scoring: fold k of machine m (job k*M + m) predicts the windows inside its test block, in one launch, outputs back to back
    KM = K * M
    fk, fm = np.repeat(np.arange(K), M), np.tile(np.arange(M), K)
    test_start = starts[fm, fk]
    job_n = n_test[fm]
    out0 = _prefix(job_n)
    max_n = int(n_test.max())
    infer_jobs = engine.jobs_to_device(engine.make_jobs(M + np.arange(KM), job_n, x_row[M:] + test_start, out0), dev)
    if eng.tc_supported:  # the ragged tile layout: each job costs its own windows (the same bits per window as gb_lstm_infer_tc)
        tiles = eng.tile_base(job_n)
        pred = eng.infer(params, infer_jobs, KM, max_n, xf, int(job_n.sum()), tile_base=torch.from_numpy(tiles).to(dev), n_tiles=int(tiles[-1]))
    else:
        pred = eng.infer(params, infer_jobs, KM, max_n, xf, int(job_n.sum()))
    # targets tail-aligned to the predictions, scored in float64 as the per-machine detector scores LSTM output (diff.py:350-385)
    score_jobs = engine.jobs_to_device(engine.make_jobs(np.arange(KM), job_n, row0[fm] + test_start + L - 1 + la, out0), dev)
    y_scale, y_offset = _minmax_attributes(y_lo, y_hi)
    want = ("tag-anomaly-unscaled", "total-anomaly-scaled")
    if target_scaler:  # sklearn's float32 inverse of the fold's transformer, in place, and float64 scoring with transform(1) - transform(0)
        res = engine.minmax_inverse_score_f64(score_jobs, KM, max_n, pred, y, _f64(y_scale[M:], dev), _f64(y_offset[M:], dev),
                                              scale=_f64(((y_scale + y_offset) - y_offset)[M:], dev), want=want, out={"model-output": pred})
    else:
        res = engine.anomaly_score(score_jobs, KM, max_n, pred.to(torch.float64), y, T, scale=_f64(y_scale[M:], dev), want=want)
    fold_sfeat = fold_sagg = None
    if window is None:
        feat, agg = engine.thresholds(score_jobs, KM, max_n, res["tag-anomaly-unscaled"], res["total-anomaly-scaled"], T, KM, 6, dev)
    else:
        feat, agg, sfeat, sagg = engine.thresholds_pair(score_jobs, KM, max_n, res["tag-anomaly-unscaled"], res["total-anomaly-scaled"], T, KM, 6,
                                                        int(window), dev)
        fold_sfeat, fold_sagg = _folds(host(sfeat), M), _folds(host(sagg), M)
    # the evaluation metrics of ModelBuilder's cross validation reduce to five sums per (fold, tag)
    moments = _folds(host(engine.cv_moments(score_jobs, KM, pred, y32, T)), M)
    fold_feat, fold_agg = _folds(host(feat), M), _folds(host(agg), M)
    loss_h, acc_h = host(hist), host(acc)
    finals = lambda a: None if a is None else a[:M]  # noqa: E731
    folds = lambda a: None if a is None else _folds(a[M:], M)  # noqa: E731
    return LSTMFleetBuild(
        eng, M, K, n, la, int(batch_size), starts, n_test, params[:M].contiguous(), _device_folds(params[M:], M).contiguous(),
        init_params, loss_h[:M], acc_h[:M], folds(loss_h), folds(acc_h), y_lo[:M], y_hi[:M], folds(y_lo), folds(y_hi),
        np.ascontiguousarray(fold_feat[:, K - 1]), np.ascontiguousarray(fold_agg[:, K - 1]), fold_feat, fold_agg, moments,
        _FoldBlocks(pred, out0, job_n, M), in_min=finals(in_lo), in_max=finals(in_hi), fold_in_min=folds(in_lo), fold_in_max=folds(in_hi),
        epochs=int(epochs), epochs_run=finals(epochs_run), best_epoch=finals(best_epoch), fold_epochs_run=folds(epochs_run),
        fold_best_epoch=folds(best_epoch), window=None if window is None else int(window), fold_smooth_feat_thr=fold_sfeat,
        fold_smooth_agg_thr=fold_sagg, target_scaler=target_scaler)


# ------------------------------------------------------------------------------------------------ fleet build of K-fold detectors
class KFoldFleetBuild:
    """
    Result of ``build_kfold_fleet``: what ``ModelBuilder._build`` produces for one ``DiffBasedKFCVAnomalyDetector`` machine -- final
    weights, target (and input) scaler extrema, the K-fold percentile thresholds, loss histories, CV metric moments -- for all
    machines of a bucket.  Slot layout of ``params`` / ``init_params`` and of every ``slot_*`` array: final models at [0, M), fold k
    of machine m at M + k*M + m.  Host arrays except ``params`` / ``init_params`` (device float32 [S, stride]).
    """

    def __init__(self, eng, n_machines, n_splits, rows, n_test, params, init_params, loss, acc, val_loss, val_acc, epochs, epochs_run,
                 best_epoch, slot_steps, y_min, y_max, in_min, in_max, target_scaler, feat_thr, agg_thr, cv_moments):
        self.eng, self.n_machines, self.n_splits = eng, n_machines, n_splits
        self.rows = rows                                      # [M] rows of every machine
        self.n_test = n_test                                  # [M, K] test rows of every fold (a machine's KFold folds differ by one row at most)
        self.params, self.init_params = params, init_params
        # per slot [S, epochs] (val_* None without a validation_split; NaN past a fit's epochs_run with EarlyStopping)
        self.loss, self.acc, self.val_loss, self.val_acc = loss, acc, val_loss, val_acc
        self.epochs, self.epochs_run, self.best_epoch = epochs, epochs_run, best_epoch  # epochs_run / best_epoch [S] or None
        self.slot_steps = slot_steps                          # [S] optimizer steps per epoch of every fit (History.params["steps"])
        self.steps_per_epoch = int(slot_steps[0])             # ... of the final fits
        # float64 column extrema per slot [S, T] of the targets (the detector's scaler and the TransformedTargetRegressor's
        # transformer) and of the inputs (the Pipeline's MinMaxScaler; None without one)
        self.y_min, self.y_max, self.in_min, self.in_max = y_min, y_max, in_min, in_max
        self.target_scaler = target_scaler                    # the estimator is a TransformedTargetRegressor(MinMaxScaler)
        self.feat_thr, self.agg_thr = feat_thr, agg_thr       # [M, T], [M] float64: feature_thresholds_ / aggregate_threshold_
        self.cv_moments = cv_moments                          # [M, K, 5, T] float64 (gb_cv_moments of every fold's test block)

    def detector(self, m: int, template, tags=None, input_tags=None):
        """
        Machine ``m`` as its fitted ``DiffBasedKFCVAnomalyDetector``: ``template`` is an unfitted detector from the machine's own
        definition, filled in with the attributes the per-machine build leaves (picklable, servable).
        """
        det = self._fill(m, template, tags, input_tags)
        return _fill_thresholds(det, list(tags) if tags is not None else list(range(self.eng.n_out)), self.feat_thr[m], self.agg_thr[m])

    def fold_detector(self, m: int, k: int, template, tags=None, input_tags=None):
        """Fold k's detector of machine m (a ``cross_validate`` estimator: fitted on fold k's training rows, no thresholds)."""
        return self._fill(self.n_machines + k * self.n_machines + m, template, tags, input_tags)

    def _fill(self, s: int, template, tags, input_tags):
        """``template`` with the fitted state of slot ``s``: scalers, weights, History, the target transformer."""
        from sklearn.preprocessing import MinMaxScaler

        M = self.n_machines
        m = s % M
        n_rows = int(self.rows[m]) if s < M else int(self.rows[m] - self.n_test[m, (s - M) // M])  # the rows the slot's scalers saw
        tags = list(tags) if tags is not None else list(range(self.eng.n_out))
        det = template
        ttr, reg, ae = _ff_template(self.eng, det, self.target_scaler, self.in_min is not None, self.params[s : s + 1])
        if self.in_min is not None:
            _fill_minmax_from_extrema(reg.steps[0][1], self.in_min[s], self.in_max[s], n_rows, input_tags)
        slot = lambda a: None if a is None else a[s]  # noqa: E731
        _fill_history(ae, ae.model.spec.metrics, self.epochs, int(self.slot_steps[s]), self.loss[s], self.acc[s], slot(self.val_loss),
                      slot(self.val_acc), slot(self.epochs_run))
        if ttr is not None:
            _fill_target_regressor(ttr, reg, self.y_min[s], self.y_max[s], n_rows)
        # a fresh scaler: detectors made from definitions without a scaler share the constructor's default MinMaxScaler object
        det.scaler = _fill_minmax_from_extrema(MinMaxScaler(), self.y_min[s], self.y_max[s], n_rows, tags)
        return det


def kfold_layout(cv, rows: int):
    """
    The row layout of a K-fold bucket from ``cv.split`` over ``rows`` rows: (tests, trains, order, inverse), where ``order`` is the
    concatenation of the folds' test rows (fold order: fold k tests a contiguous block) and ``inverse[t]`` is the fold-order
    position of row t.  ValueError unless the folds test every row exactly once.
    """
    folds = [(np.asarray(tr, dtype=np.int64), np.asarray(te, dtype=np.int64)) for tr, te in cv.split(np.arange(rows))]
    trains, tests = [f[0] for f in folds], [f[1] for f in folds]
    order = np.concatenate(tests) if tests else np.zeros(0, np.int64)
    if len(tests) < 2 or len(order) != rows or not np.array_equal(np.sort(order), np.arange(rows)):
        raise ValueError("K-fold thresholds need a cv whose test folds cover every row exactly once (KFold)")
    inverse = np.empty(rows, dtype=np.int64)
    inverse[order] = np.arange(rows)
    return tests, trains, order, inverse


def kfold_row_maps(trains, inverse, rows: int, detector_shuffle: bool):
    """
    The K + 1 row maps of a K-fold bucket, in fold-order rows: the final fit's positions (all rows, in time order) and fold k's
    (its training rows) -- each in the order ``sklearn.utils.shuffle(..., random_state=0)`` gives when the detector shuffles.
    """
    orders = [np.arange(rows)] + list(trains)
    if detector_shuffle:
        orders = [sk_shuffle(t, random_state=0) for t in orders]
    return [inverse[t] for t in orders]


def kfold_bucket_maps(cv, rows, detector_shuffle: bool):
    """
    The row maps of a K-fold bucket whose machines have ``rows[m]`` rows, made once per distinct length (a KFold split depends only
    on the length and ``cv``) and laid out back to back.  Returns (n_test [M, K], to_fold, to_time, machine_ofs [M], fit_maps,
    slot_ofs [S]): machine m's fold-order map (``kfold_layout``'s order) and time-order map (its inverse) start at machine_ofs[m]
    of to_fold / to_time; slot s (finals, then fold k of machine m at M + k*M + m) reads map j of ``kfold_row_maps`` for its
    machine's length (j = 0 for the final fit, k + 1 for fold k) at slot_ofs[s] of fit_maps.  Maps are int32, offsets int64.
    """
    n = np.asarray(rows, dtype=np.int64)
    lengths = list(dict.fromkeys(int(v) for v in n))
    layouts = [kfold_layout(cv, v) for v in lengths]
    of_length = np.asarray([lengths.index(int(v)) for v in n], dtype=np.int64)
    n_test = np.asarray([[len(t) for t in layouts[i][0]] for i in of_length], dtype=np.int64).reshape(len(n), -1)
    maps = [kfold_row_maps(lay[1], lay[3], v, detector_shuffle) for lay, v in zip(layouts, lengths)]
    fit_ofs = _prefix([len(mp) for per_length in maps for mp in per_length]).reshape(len(lengths), -1)
    i32 = lambda parts: np.concatenate(parts).astype(np.int32)  # noqa: E731
    return (n_test, i32([lay[2] for lay in layouts]), i32([lay[3] for lay in layouts]), _prefix(lengths)[of_length],
            i32([mp for per_length in maps for mp in per_length]), fit_ofs[of_length].T.reshape(-1))


def combine_fold_extrema(lo, hi):
    """
    Column extrema per slot from those of the K test blocks (``lo`` / ``hi``: [K, M, T]): the final slot's over all blocks, fold
    k's over every block but k.  Min and max do not depend on order, so these are exactly the extrema of the slot's rows.
    Returns ([S, T], [S, T]) in the slot layout (finals, then fold k of machine m at M + k*M + m).
    """
    K, M = lo.shape[:2]
    s_lo = np.empty(((K + 1) * M,) + lo.shape[2:], dtype=lo.dtype)
    s_hi = np.empty_like(s_lo)
    s_lo[:M], s_hi[:M] = lo.min(axis=0), hi.max(axis=0)
    for k in range(K):
        others = [j for j in range(K) if j != k]
        s_lo[M + k * M : M + (k + 1) * M] = lo[others].min(axis=0)
        s_hi[M + k * M : M + (k + 1) * M] = hi[others].max(axis=0)
    return s_lo, s_hi


@_fit_joined
def build_kfold_fleet(eng: "engine.FFEngine", x, y, rows, cv, epochs: int = 1, batch_size: int = 32, seed: int = 0,
                      adam: Optional[Dict[str, float]] = None, shuffle: bool = True, generator=None, input_scaler: bool = False,
                      target_scaler: bool = False, detector_shuffle: bool = False, validation_split: float = 0.0,
                      validation_batch_size: Optional[int] = None, early_stopping=None, window: Optional[int] = None,
                      smoothing_method: Optional[str] = None, threshold_percentile: float = 0.99,
                      keep_init_params: bool = False, loss: str = "mse", optimizer=None, reg=None, dropout=None) -> KFoldFleetBuild:
    """
    The batched ``gordo build`` of one bucket of ``DiffBasedKFCVAnomalyDetector`` machines (diff.py:566-635 in the reference):
    for every machine the K-fold cross validation under ``cv`` (a KFold) and the final fit -- ``(K + 1) * n_machines`` fits in one
    fit launch -- then every fold model's test block scored in one launch, the errors brought back to time order, smoothed and
    reduced to the ``threshold_percentile`` quantile, and the CV metric moments.

    x, y: float64 device tensors of the machines' rows stacked; ``rows`` an int (machine m owns rows [m*rows, (m+1)*rows)) or one
    count per machine (machine m owns rows [row0[m], row0[m] + rows[m]), row0 the prefix sum).  ``y`` may be ``x``.

    A KFold split depends only on the row count and ``cv``, so the split and its row maps are made once per distinct length and
    shared by every machine of that length.  x and y are laid out once in fold order (each machine's folds' test rows one after
    the other, gb_gather_rows_ragged with each job pointing at its machine's map), where fold k's test rows are one contiguous
    block; the fits read their rows through the K + 1 maps of their machine's length.  ``input_scaler``: the network is behind a MinMaxScaler
    (``Pipeline([MinMaxScaler(), KerasAutoEncoder])``); ``target_scaler``: the estimator is ``TransformedTargetRegressor(transformer=
    MinMaxScaler(), regressor=...)``, so every slot trains on its own MinMax-scaled targets and the fold models' predictions are
    mapped back by sklearn's float32 inverse and scored in float64 in one pass (gb_minmax_inverse_score_f64), as the per-machine
    detector scores a foreign estimator.  Every scaler's extrema come from gb_minmax_f64 over the test blocks (a slot's rows are a union of blocks)
    with sklearn's float64 attribute arithmetic.  ``detector_shuffle``, ``validation_split``, ``early_stopping``, ``loss``, ``optimizer``,
    ``reg``, ``dropout`` as in ``build_fleet``.
    """
    torch = engine._torch()
    dev = eng.device
    if x.dtype != torch.float64 or y.dtype != torch.float64:
        raise ValueError(f"build_kfold_fleet takes float64 x and y, got {x.dtype} / {y.dtype}")
    x, y = x.contiguous(), (None if y is x else y.contiguous())
    y = x if y is None else y
    n, row0 = _machine_rows(x, rows)
    M, N, T = len(n), int(n.max()), eng.n_out
    total = int(n.sum())
    n_test, to_fold, to_time, machine_ofs, fit_maps, slot_map = kfold_bucket_maps(cv, n, detector_shuffle)
    K = n_test.shape[1]
    S, KM = M * (K + 1), M * K
    o = np.cumsum(n_test, axis=1) - n_test                      # first fold-order row of fold k's test block in machine m's rows
    max_test = int(n_test.max())

    def i32(a):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(dev)

    def i64(a):
        return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to(dev)

    def jobs(slots, rows_, x_row, out_row=None):
        return engine.jobs_to_device(engine.make_jobs(slots, rows_, x_row, out_row), dev)

    to_fold, to_time = i32(to_fold), i32(to_time)

    # 1. fold order: one gather per array
    whole = jobs(np.arange(M), n, row0)
    per_machine = i64(machine_ofs)
    xq = engine.gather_rows(whole, M, N, to_fold, x, total, map_ofs=per_machine)
    yq = xq if y is x else engine.gather_rows(whole, M, N, to_fold, y, total, map_ofs=per_machine)

    # 2. scaler extrema: one reduction over the K*M test blocks (job k*M + m), combined per slot on the host
    fk, fm = np.repeat(np.arange(K), M), np.tile(np.arange(M), K)
    blocks = jobs(np.arange(KM), n_test[fm, fk], row0[fm] + o[fm, fk])

    def slot_extrema(a):
        lo, hi = (t.cpu().numpy().reshape(K, M, -1) for t in engine.minmax_f64(blocks, KM, max_test, a, KM))
        s_lo, s_hi = combine_fold_extrema(lo, hi)
        if not (np.isfinite(s_lo).all() and np.isfinite(s_hi).all()):
            raise ValueError("a column without finite values in a training set")
        return s_lo, s_hi

    y_lo, y_hi = slot_extrema(yq)
    y_scale, y_offset = _minmax_attributes(y_lo, y_hi)
    in_lo = in_hi = None
    if input_scaler:
        in_lo, in_hi = (y_lo, y_hi) if y is x else slot_extrema(xq)

    # 3. the fits' inputs: with a scaler in front of the network or on the targets, slot s owns its own copy of its machine's rows
    # (the stacked machines repeated K + 1 times, slot s at slot_x[s])
    per_slot = input_scaler or target_scaler
    slot_x, copy_jobs = _slot_copies(n, row0, K, dev) if per_slot else (np.tile(row0, K + 1), None)  # first row of slot s in x / y
    per_slot_ofs = i64(np.tile(machine_ofs, K + 1))
    if input_scaler:
        a, b = _minmax_attributes(in_lo, in_hi)
        xf = engine.affine_f64(copy_jobs, S, N, xq, _f64(a, dev), _f64(b, dev), out_rows=(K + 1) * total)
    elif per_slot:
        xf = engine.gather_rows(copy_jobs, S, N, to_fold, x, (K + 1) * total, to_f32=True, map_ofs=per_slot_ofs)
    else:
        xf = engine.gather_rows(whole, M, N, to_fold, x, total, to_f32=True, map_ofs=per_machine)
    if target_scaler:
        yf = xf if (input_scaler and y is x) else engine.affine_f64(copy_jobs, S, N, yq, _f64(y_scale, dev), _f64(y_offset, dev), out_rows=(K + 1) * total)
    elif per_slot:
        yf = engine.gather_rows(copy_jobs, S, N, to_fold, y, (K + 1) * total, to_f32=True, map_ofs=per_slot_ofs)
    else:
        yf = xf if y is x else engine.gather_rows(whole, M, N, to_fold, y, total, to_f32=True, map_ofs=per_machine)

    slot_n = np.concatenate([n] + [n - n_test[:, k] for k in range(K)])  # rows each slot's estimator receives
    n_train = _keras_train_rows(slot_n, validation_split)
    split = engine.make_split(slot_n - n_train, slot_map)
    row_map = i32(fit_maps)
    g = generator or torch.Generator(device=dev).manual_seed(seed)
    params = _keras_initial_params(eng, S, g)
    init_params = params.clone() if keep_init_params else None
    fit_jobs = jobs(np.arange(S), n_train, slot_x)
    hist, acc, val_loss, val_acc, epochs_run, best_epoch = yield _FitRequest(
        eng, params, fit_jobs, S, N, xf, yf, split, row_map, M, epochs, batch_size, shuffle, adam, seed, validation_batch_size, early_stopping,
        loss, optimizer, reg, dropout)
    if (n_train == slot_n).all():  # nothing held out
        val_loss = val_acc = None

    # 4. fold errors in fold order, by the route the per-machine detector takes (DiffBasedAnomalyDetector._score)
    sc_slots = M + np.arange(KM)
    sc_n = n_test[fm, fk]
    out0 = row0[fm] + o[fm, fk]                                     # fold-order rows of the test block in machine layout
    sc_jobs = jobs(sc_slots, sc_n, slot_x[sc_slots] + o[fm, fk], out0)
    mult = (y_scale + y_offset) - y_offset                          # _scaler_multiplier: transform(1) - transform(0)
    want = ("tag-anomaly-unscaled", "total-anomaly-scaled")
    if not target_scaler:  # fused predict + score, fp32, with the fold detector's multiplier
        res = eng.infer_score(params, sc_jobs, KM, max_test, xf, yf, torch.from_numpy(mult.astype(np.float32)).to(dev), out_rows=total, want=want)
        pred32, tag_err, tot_err = res["model-output"], res["tag-anomaly-unscaled"], res["total-anomaly-scaled"]
        mom_jobs, y32 = sc_jobs, yf
    else:  # predict, then in one pass sklearn's float32 inverse of the slot's transformer and float64 scoring against the float64 targets
        pred = eng.infer_score(params, sc_jobs, KM, max_test, xf, out_rows=total)["model-output"]
        mom_jobs = jobs(sc_slots, sc_n, out0, out0)
        res = engine.minmax_inverse_score_f64(mom_jobs, KM, max_test, pred, yq, _f64(y_scale, dev), _f64(y_offset, dev), scale=_f64(mult, dev), want=want,
                                              out_rows=total)
        pred32, tag_err, tot_err = res["model-output"], res["tag-anomaly-unscaled"], res["total-anomaly-scaled"]
        y32 = engine.gather_rows(whole, M, N, to_fold, y, total, to_f32=True, map_ofs=per_machine)

    # 5. K-fold thresholds: errors back in time order (float32, as the detector stores them), smoothed, the percentile
    narrow = tag_err.dtype == torch.float64
    tag_t = engine.gather_rows(whole, M, N, to_time, tag_err, total, to_f32=narrow, map_ofs=per_machine)
    tot_t = engine.gather_rows(whole, M, N, to_time, tot_err, total, to_f32=narrow, map_ofs=per_machine)
    if window is not None and smoothing_method is not None:
        tag_t = engine.smooth(whole, M, tag_t, int(window), smoothing_method, max_rows=N)
        tot_t = engine.smooth(whole, M, tot_t, int(window), smoothing_method, max_rows=N)
    q = float(threshold_percentile)
    feat = engine.quantile(whole, M, N, tag_t, q)
    agg = engine.quantile(whole, M, N, tot_t, q)[:, 0]

    # 6. the evaluation metrics of ModelBuilder's cross validation, in the targets' own units
    moments = engine.cv_moments(mom_jobs, KM, pred32, y32, T)

    def host(t):
        return None if t is None else t.cpu().numpy()

    return KFoldFleetBuild(
        eng, M, K, n, n_test, params, init_params, host(hist), host(acc), host(val_loss), host(val_acc), int(epochs), host(epochs_run),
        host(best_epoch), (n_train + int(batch_size) - 1) // int(batch_size), y_lo, y_hi, in_lo, in_hi, bool(target_scaler),
        host(feat).astype(np.float64), host(agg).astype(np.float64), _folds(host(moments), M))
