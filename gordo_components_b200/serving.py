"""
Request coalescer for model servers (SURVEY §8f rank 3, BASELINE configs[4]).

gordo.server answers every ``POST /anomaly/prediction`` on its own: unpickle (lru_cache of 2), ``model.anomaly(X, y)``, JSON
(gordo/server/blueprints/anomaly.py:49-55, gordo/server/utils.py:334-353) -- up to 8 gunicorn threads per worker call into
the models concurrently (gordo/cli/cli.py:288-296).  At 100 rows per request a kernel launch per request wastes the GPU: the
launch, the two small copies and the Python around them cost more than the arithmetic.  ``AnomalyCoalescer`` keeps the
weights, scalers and thresholds of ALL machines of one architecture bucket resident on the device and turns whatever
requests are waiting into ONE ``gb_ffae_infer_score`` launch (a request is just a job ``{slot, n_rows, x_row, out_row}``):

    co  = AnomalyCoalescer(eng, params, scale, feat_thr, agg_thr)
    fut = co.submit(machine_index, X, y)          # any thread; X, y: [rows, tags] arrays
    cols = fut.result()                           # dict of host arrays named like the anomaly frame's blocks

With ``x_scale`` / ``x_offset`` (float64 [n_slots, n_in] device tensors: the composed per-feature input scalers of Pipeline models)
requests' X is staged as float64 and the launch applies each slot's scaler as it reads x (gb_ffae_infer_score_x64), exactly the
float32 batch ``gb_affine_f64`` would have produced.

With ``y_inverse=(y_scale, y_min)`` (float64 [n_slots, n_out] device tensors: the MinMax ``transformer_`` of detectors around a
``TransformedTargetRegressor``) the batch runs the fused launch for the prediction only, then one gb_minmax_inverse_score_f64
launch that applies sklearn's float32 ``inverse_transform`` and scores in float64 against the float64 y, as the per-request route
does on the host and in gb_anomaly_score_f64.  ``scale`` / thresholds are then float64 and so are the score arrays; a request
whose model output holds ±inf also gets the network's raw prediction of its rows under ``raw-model-output``, so the caller can
tell an infinite prediction from an inverse that overflows float32.

Thread-safe, re-entrant, no shared mutable scratch outside the worker thread (the reference's threading convention,
SURVEY §8b).  The per-request results are bit-identical to a per-request launch: rows are independent in the kernel.

``LSTMAnomalyCoalescer`` does the same for LSTM detectors: the waiting requests become one ragged tensor-core LSTM launch
sequence (gb_lstm_infer_tc_ragged, each request a job of its own windows) and one float64 scoring launch (gb_anomaly_score_f64, or
with ``y_inverse`` gb_minmax_inverse_score_f64, as above).

Either coalescer built with ``smoothing=(window, method)`` (the detectors' ``window`` / ``smoothing_method``) also answers the
smoothed columns: ``submit(slot, X, y, smooth=True)`` marks a request whose reply carries them, and a batch holding such requests
runs one more launch (gb_smooth_scores) over exactly their jobs, reading the score arrays the batch's launch left on the device.
Its results come back with the rest of the batch, before the batch's one synchronisation.  Each request is smoothed on its own
rows (its windows start at its first row), as ``DiffBasedAnomalyDetector._smoothing`` smooths it on the per-request route.
"""
from __future__ import annotations

import queue
import threading
import time
from concurrent.futures import Future
from typing import Dict, Optional, Sequence

import numpy as np

from . import engine
from .fleet import PER_ROW, PER_TAG

SMM_MAX_WINDOW = 200 * 1024 // 4  # the rolling median keeps one thread's sorted window in shared memory (gb_smooth / gb_smooth_scores)


class AnomalyCoalescer:
    def __init__(self, eng: "engine.FFEngine", params, scale, feat_thr=None, agg_thr=None, max_batch_rows: int = 1 << 18,
                 max_wait_ms: float = 1.0, want: Optional[Sequence[str]] = None, x_scale=None, x_offset=None, smoothing=None, y_inverse=None):
        torch = engine._torch()
        if (x_scale is None) != (x_offset is None):
            raise ValueError("x_scale and x_offset go together")
        self.max_rows = self.max_cost = int(max_batch_rows)
        self._setup(eng, params, scale, feat_thr, agg_thr, max_wait_ms, want, smoothing, y_inverse)
        self.x_affine = (x_scale, x_offset) if x_scale is not None else None
        x_dtype = torch.float64 if self.x_affine is not None else torch.float32
        self._x_np = np.float64 if self.x_affine is not None else np.float32
        y_dtype, score_dtype = (torch.float64, torch.float64) if self.y_inverse is not None else (torch.float32, torch.float32)
        self._y_np = np.float64 if self.y_inverse is not None else np.float32
        dev = eng.device
        self._xh = torch.empty((self.max_rows, eng.n_in), dtype=x_dtype).pin_memory()
        self._yh = torch.empty((self.max_rows, eng.n_out), dtype=y_dtype).pin_memory()
        self._xd = torch.empty((self.max_rows, eng.n_in), dtype=x_dtype, device=dev)
        self._yd = torch.empty((self.max_rows, eng.n_out), dtype=y_dtype, device=dev)
        self._out_d = {k: torch.empty((self.max_rows, eng.n_out) if k in PER_TAG else (self.max_rows,),
                                      dtype=torch.float32 if k == "model-output" else score_dtype, device=dev) for k in self.want}
        if self.y_inverse is not None:  # the network's raw prediction, kept apart from its inverse
            self._out_d["raw-model-output"] = torch.empty((self.max_rows, eng.n_out), dtype=torch.float32, device=dev)
        self._out_h = {k: torch.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in self._out_d.items()}
        # the batch's jobs, then those of its requests that want the smoothed columns
        self._jobs_h = torch.empty((2 * self.max_jobs * engine._cabi.JOB_DTYPE.itemsize,), dtype=torch.uint8).pin_memory()
        self._start()

    max_jobs = 4096  # requests per batch: the pinned buffer the job records are staged through holds this many

    def _setup(self, eng, params, scale, feat_thr, agg_thr, max_wait_ms, want, smoothing, y_inverse):
        """What both coalescers keep: the bucket's device tensors, the score arrays a reply carries (by default all but the
        confidences whose thresholds are absent), the smoothing option, the batching wait and the stream the batches run on."""
        self.eng, self.params, self.scale, self.feat_thr, self.agg_thr = eng, params, scale, feat_thr, agg_thr
        self.y_inverse = tuple(y_inverse) if y_inverse is not None else None
        self.max_wait = float(max_wait_ms) * 1e-3
        self.want = tuple(want) if want is not None else tuple(
            k for k in PER_TAG + PER_ROW if not ((feat_thr is None and k == "anomaly-confidence") or (agg_thr is None and k == "total-anomaly-confidence")))
        self.smoothing = self._check_smoothing(smoothing)
        self._stream = engine._torch().cuda.Stream(device=eng.device)

    def _check_smoothing(self, smoothing):
        """``smoothing`` as (int window, method name), or None; ValueError for anything the smoothing launch does not take."""
        if smoothing is None:
            return None
        window, method = smoothing
        if isinstance(window, bool) or not isinstance(window, (int, np.integer)) or window < 1:
            raise ValueError(f"smoothing window {window!r} must be a positive int")
        if method not in engine.SMOOTH_METHODS:
            raise ValueError(f"smoothing_method {method!r} must be one of {sorted(engine.SMOOTH_METHODS)}")
        if method == "smm" and window > SMM_MAX_WINDOW:
            raise ValueError(f"a rolling-median window of {window} exceeds the {SMM_MAX_WINDOW} values the kernel holds")
        missing = [k for k in engine.SMOOTH_SCORE_KEYS if k not in self.want]
        if missing:
            raise ValueError(f"smoothing needs the score arrays {missing}, which this coalescer does not compute")
        return int(window), method

    def _start(self):
        self._q: "queue.Queue" = queue.Queue()
        self._closed = False
        self.batches = 0
        self.requests = 0
        self._worker = threading.Thread(target=self._run, name="gordo-b200-coalescer", daemon=True)
        self._worker.start()

    # ------------------------------------------------------------------ client side
    def submit(self, slot: int, X, y, smooth: bool = False) -> Future:
        """Queue one request; the Future resolves to {column block: host array} for exactly these rows.  ``smooth=True`` adds the
        four ``smooth-*`` arrays (float32) of a coalescer built with ``smoothing``."""
        if self._closed:
            raise RuntimeError("coalescer is closed")
        if not (0 <= int(slot) < self.params.shape[0]):
            raise ValueError(f"unknown machine slot {slot}")
        if smooth and self.smoothing is None:
            raise ValueError("smoothed columns asked of a coalescer built without smoothing")
        fut: Future = Future()
        self._q.put((int(slot), *self._request(X, y), bool(smooth), fut))
        return fut

    def _request(self, X, y):
        """The request's staged (X, y) host arrays, or ValueError when they do not fit the bucket."""
        Xv = np.ascontiguousarray(getattr(X, "values", X), dtype=self._x_np)
        yv = np.ascontiguousarray(getattr(y, "values", y), dtype=self._y_np)
        if Xv.ndim != 2 or Xv.shape[1] != self.eng.n_in or yv.shape != (len(Xv), self.eng.n_out):
            raise ValueError(f"request of shape X {Xv.shape} / y {yv.shape} does not fit a {self.eng.n_in}->{self.eng.n_out} model")
        if len(Xv) > self.max_rows:
            raise ValueError(f"a request of {len(Xv)} rows exceeds max_batch_rows={self.max_rows}")
        return Xv, yv

    def _cost(self, item) -> int:
        """What a request adds to a batch, against ``max_cost``: its rows."""
        return len(item[1])

    def anomaly(self, slot: int, X, y, smooth: bool = False) -> Dict[str, np.ndarray]:
        return self.submit(slot, X, y, smooth).result()

    def close(self):
        self._closed = True
        self._q.put(None)
        self._worker.join()

    # ------------------------------------------------------------------ worker
    def _run(self):
        torch = engine._torch()
        pending = None
        while True:
            first = pending if pending is not None else self._q.get()
            pending = None
            if first is None:
                return
            batch, cost = [first], self._cost(first)
            deadline = time.perf_counter() + self.max_wait
            while cost < self.max_cost and len(batch) < self.max_jobs:
                try:
                    item = self._q.get(timeout=max(0.0, deadline - time.perf_counter())) if self._q.empty() else self._q.get_nowait()
                except queue.Empty:
                    break
                if item is None:
                    self._q.put(None)
                    break
                if cost + self._cost(item) > self.max_cost:
                    pending = item
                    break
                batch.append(item)
                cost += self._cost(item)
            try:
                self._launch(torch, batch, cost)
            except BaseException as exc:  # noqa: BLE001 - every waiting caller must hear about it
                for item in batch:
                    if not item[-1].done():
                        item[-1].set_exception(exc)

    def _smoothing_jobs(self, batch, starts, counts):
        """The job records of the batch's requests that want the smoothed columns, on rows ``[starts[i] - lo, + counts[i])`` of the
        score arrays' rows ``[lo, hi)``, the span those requests cover; (jobs, lo, hi), or None when no request asked."""
        sel = np.fromiter((item[-2] for item in batch), dtype=bool, count=len(batch))
        if not sel.any():
            return None
        starts, counts = np.asarray(starts, dtype=np.int64)[sel], np.asarray(counts, dtype=np.int64)[sel]
        lo, hi = int(starts[0]), int(starts[-1] + counts[-1])
        return engine.make_jobs(np.zeros(len(starts), dtype=np.int64), counts, starts - lo), lo, hi

    def _smooth(self, torch, jobs_d, jobs, lo, hi, scores):
        """One gb_smooth_scores launch over ``jobs`` on rows [lo, hi) of the batch's device ``scores``, on the current stream, and
        the copy of its results into pinned host memory: {"smooth-<key>": host tensor of rows [lo, hi)}."""
        window, method = self.smoothing
        if hi == lo:  # only empty requests asked: nothing to launch
            return {"smooth-" + k: torch.empty((0,) + tuple(scores[k].shape[1:]), dtype=torch.float32) for k in engine.SMOOTH_SCORE_KEYS}
        res = engine.smooth_scores(jobs_d, len(jobs), int(jobs["n_rows"].max()), {k: scores[k][lo:hi] for k in engine.SMOOTH_SCORE_KEYS},
                                   window, method)
        host = {k: torch.empty(v.shape, dtype=v.dtype, pin_memory=True) for k, v in res.items()}
        for k, v in res.items():
            host[k].copy_(v, non_blocking=True)
        return host

    @staticmethod
    def _reply(batch, host, starts, counts, smoothed):
        """Resolve each request of ``batch`` to copies of its rows ``[start, start + count)`` of the batch's host tensors ``host``
        and, when it asked for them, of the smoothed arrays (``smoothed``: ``_smooth``'s result and its first row, or None).
        ``host["raw-model-output"]`` (the network's prediction under a target inverse) goes only to a request whose
        ``model-output`` holds ±inf."""
        arrays = {k: v.numpy() for k, v in host.items()}
        raw = arrays.pop("raw-model-output", None)
        smooth, lo = ({k: v.numpy() for k, v in smoothed[0].items()}, smoothed[1]) if smoothed is not None else ({}, 0)
        for item, start, n in zip(batch, starts, counts):
            result = {k: v[start:start + n].copy() for k, v in arrays.items()}
            if raw is not None and np.isinf(result.get("model-output", 0.0)).any():
                result["raw-model-output"] = raw[start:start + n].copy()
            if item[-2]:
                result.update({k: v[start - lo:start - lo + n].copy() for k, v in smooth.items()})
            item[-1].set_result(result)

    def _launch(self, torch, batch, rows):
        jobs = np.empty(len(batch), dtype=engine._cabi.JOB_DTYPE)
        ofs = 0
        xh, yh = self._xh.numpy(), self._yh.numpy()
        for i, (slot, Xv, yv, _, _) in enumerate(batch):
            n = len(Xv)
            xh[ofs:ofs + n] = Xv
            yh[ofs:ofs + n] = yv
            jobs[i] = (slot, n, ofs, ofs)
            ofs += n
        max_rows = int(jobs["n_rows"].max()) if len(jobs) else 0
        smooth = self._smoothing_jobs(batch, jobs["out_row"], jobs["n_rows"]) if rows else None
        staged = jobs if smooth is None else np.concatenate([jobs, smooth[0]])
        jb = self._jobs_h[: staged.nbytes]
        jb.numpy()[:] = staged.view(np.uint8)
        smoothed = None
        with torch.cuda.stream(self._stream):
            jobs_all = jb.to(self.eng.device, non_blocking=True)
            jobs_d = jobs_all[: jobs.nbytes]
            self._xd[:rows].copy_(self._xh[:rows], non_blocking=True)
            self._yd[:rows].copy_(self._yh[:rows], non_blocking=True)
            out = {k: v[:rows] for k, v in self._out_d.items()}
            if rows and self.y_inverse is None:
                self.eng.infer_score(self.params, jobs_d, len(batch), max_rows, self._xd[:rows], self._yd[:rows], self.scale, self.feat_thr,
                                     self.agg_thr, out_rows=rows, want=self.want, out=out, x_affine=self.x_affine)
            elif rows:  # prediction only, then the target inverse and float64 scoring in one pass
                raw = out.pop("raw-model-output")
                self.eng.infer_score(self.params, jobs_d, len(batch), max_rows, self._xd[:rows], out_rows=rows, out={"model-output": raw},
                                     x_affine=self.x_affine)
                engine.minmax_inverse_score_f64(jobs_d, len(batch), max_rows, raw, self._yd[:rows], *self.y_inverse, self.scale, self.feat_thr,
                                                self.agg_thr, want=self.want, out_rows=rows, out=out)
            if smooth is not None:
                smoothed = (self._smooth(torch, jobs_all[jobs.nbytes:], *smooth, self._out_d), smooth[1])
            for k in self._out_d:
                self._out_h[k][:rows].copy_(self._out_d[k][:rows], non_blocking=True)
        self._stream.synchronize()
        self.batches += 1
        self.requests += len(batch)
        self._reply(batch, self._out_h, jobs["out_row"].tolist(), jobs["n_rows"].tolist(), smoothed)


class LSTMAnomalyCoalescer(AnomalyCoalescer):
    """
    ``AnomalyCoalescer`` for the LSTM detectors of one architecture: ``params`` [n_slots, param_stride] float32, ``scale`` /
    ``feat_thr`` [n_slots, n_out] and ``agg_thr`` [n_slots] float64 device tensors.  A request is the model input ``X`` (float32, the
    Pipeline's leading steps already applied) and the float64 targets of its windows, ``y[-n_windows:]``; ``X`` must hold at least
    ``n_windows + lookback - 1`` rows (a forecast's last row is not read).  Per batch: X packed back to back, the batch's distinct
    models gathered into compact tensors (the launch stages the FP16 images of the slots it is given), one ragged tensor-core launch
    sequence, the prediction widened to float64 on the device and scored there, one synchronisation.  A batch closes at
    ``max_batch_tiles`` 128-window tiles or ``max_jobs`` requests.  Results: float32 ``model-output``, float64 scores, as the
    per-request route returns them.

    With ``y_inverse=(y_scale, y_min)`` (float64 [n_slots, n_out] device tensors, the MinMax ``transformer_`` of detectors around a
    ``TransformedTargetRegressor``) the prediction is not widened and scored: one gb_minmax_inverse_score_f64 launch writes its float32
    inverse as ``model-output`` and the float64 scores, and a request whose inverse holds ±inf also gets its raw prediction under
    ``raw-model-output``, as ``AnomalyCoalescer`` does.
    """

    def __init__(self, eng: "engine.LSTMEngine", params, scale, feat_thr=None, agg_thr=None, max_batch_tiles: int = 1024,
                 max_wait_ms: float = 1.0, smoothing=None, y_inverse=None):
        torch = engine._torch()
        self.max_cost = int(max_batch_tiles)
        self._setup(eng, params, scale, feat_thr, agg_thr, max_wait_ms, None, smoothing, y_inverse)
        # staged per batch in one copy: the infer jobs, the score jobs, the gather job, the smoothing jobs, tile_base and the
        # distinct slots
        jb = engine._cabi.JOB_DTYPE.itemsize
        self._stage_h = torch.empty((3 * self.max_jobs * jb + 2 * (self.max_jobs + 1) * 4 + jb,), dtype=torch.uint8).pin_memory()
        self._start()

    def _request(self, X, y):
        Xv = np.ascontiguousarray(getattr(X, "values", X), dtype=np.float32)
        yv = np.ascontiguousarray(getattr(y, "values", y), dtype=np.float64)
        n = len(yv)
        if Xv.ndim != 2 or Xv.shape[1] != self.eng.n_features or yv.ndim != 2 or yv.shape[1] != self.eng.n_out:
            raise ValueError(f"request of shape X {Xv.shape} / y {yv.shape} does not fit a {self.eng.n_features}->{self.eng.n_out} LSTM model")
        if not 1 <= n <= len(Xv) - self.eng.lookback + 1:
            raise ValueError(f"{n} target rows for {len(Xv)} input rows: a lookback of {self.eng.lookback} gives 1 to "
                             f"{len(Xv) - self.eng.lookback + 1} windows")
        if self._tiles(n) > self.max_cost:
            raise ValueError(f"a request of {n} windows exceeds max_batch_tiles={self.max_cost} tiles of {self.eng.TILE}")
        return Xv, yv

    def _tiles(self, n_windows: int) -> int:
        return -(-int(n_windows) // self.eng.TILE)

    def _cost(self, item) -> int:
        return self._tiles(len(item[2]))

    def _launch(self, torch, batch, n_tiles):
        _cabi = engine._cabi
        k = len(batch)
        slots = np.fromiter((item[0] for item in batch), dtype=np.int64, count=k)
        uniq, compact = np.unique(slots, return_inverse=True)
        x_rows = np.fromiter((len(item[1]) for item in batch), dtype=np.int64, count=k)
        windows = np.fromiter((len(item[2]) for item in batch), dtype=np.int64, count=k)
        x_ofs = np.concatenate([[0], np.cumsum(x_rows)])
        w_ofs = np.concatenate([[0], np.cumsum(windows)])
        rows, total = int(x_ofs[-1]), int(w_ofs[-1])
        infer_jobs = engine.make_jobs(compact, windows, x_ofs[:-1], w_ofs[:-1])
        score_jobs = engine.make_jobs(compact, windows, w_ofs[:-1])  # y and the prediction both at the windows' rows
        tile_base = self.eng.tile_base(windows)
        gather_job = engine.make_jobs([0], [len(uniq)], [0])
        smooth = self._smoothing_jobs(batch, w_ofs[:-1], windows)
        smooth_jobs = smooth[0] if smooth is not None else engine.make_jobs([], [], [])
        # job records first: they hold int64 fields and stay 8-byte aligned in the staged buffer
        parts = [infer_jobs.view(np.uint8), score_jobs.view(np.uint8), gather_job.view(np.uint8), smooth_jobs.view(np.uint8),
                 tile_base.view(np.uint8), uniq.astype(np.int32).view(np.uint8)]
        sizes = [p.nbytes for p in parts]
        stage = self._stage_h.numpy()
        ofs = np.concatenate([[0], np.cumsum(sizes)])
        for p, o in zip(parts, ofs[:-1]):
            stage[o:o + p.nbytes] = p
        xh = torch.empty((rows, self.eng.n_features), dtype=torch.float32, pin_memory=True)
        yh = torch.empty((total, self.eng.n_out), dtype=torch.float64, pin_memory=True)
        xn, yn = xh.numpy(), yh.numpy()
        for i, (_, Xv, yv, _, _) in enumerate(batch):
            xn[x_ofs[i]:x_ofs[i + 1]] = Xv
            yn[w_ofs[i]:w_ofs[i + 1]] = yv
        dev = self.eng.device
        with torch.cuda.stream(self._stream):
            staged = self._stage_h[: int(ofs[-1])].to(dev, non_blocking=True)
            view = [staged[int(ofs[i]):int(ofs[i + 1])] for i in range(len(parts))]
            jobs_d, score_d, gjob_d, sjobs_d, tb_d, map_d = view[0], view[1], view[2], view[3], view[4].view(torch.int32), view[5].view(torch.int32)
            xd = xh.to(dev, non_blocking=True)
            yd = yh.to(dev, non_blocking=True)
            gather = lambda t: engine.gather_rows(gjob_d, 1, len(uniq), map_d, t, len(uniq))  # noqa: E731 - the batch's models, compact
            params = gather(self.params)
            scale = gather(self.scale)
            feat_thr = gather(self.feat_thr) if self.feat_thr is not None else None
            agg_thr = gather(self.agg_thr) if self.agg_thr is not None else None
            pred = self.eng.infer(params, jobs_d, k, int(windows.max()), xd, total, tile_base=tb_d, n_tiles=int(tile_base[-1]))
            if self.y_inverse is None:
                res = engine.anomaly_score(score_d, k, int(windows.max()), pred.to(torch.float64), yd, self.eng.n_out, scale, feat_thr,
                                           agg_thr, want=self.want)
                res["model-output"] = pred
            else:
                y_scale, y_min = (gather(t) for t in self.y_inverse)
                res = engine.minmax_inverse_score_f64(score_d, k, int(windows.max()), pred, yd, y_scale, y_min, scale, feat_thr, agg_thr,
                                                      want=self.want)
                res["raw-model-output"] = pred
            smoothed = (self._smooth(torch, sjobs_d, *smooth, res), smooth[1]) if smooth is not None else None
            host = {key: torch.empty(v.shape, dtype=v.dtype, pin_memory=True) for key, v in res.items()}
            for key, v in res.items():
                host[key].copy_(v, non_blocking=True)
        self._stream.synchronize()
        self.batches += 1
        self.requests += k
        self._reply(batch, host, w_ofs[:-1].tolist(), windows.tolist(), smoothed)
