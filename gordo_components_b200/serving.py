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

Thread-safe, re-entrant, no shared mutable scratch outside the worker thread (the reference's threading convention,
SURVEY §8b).  The per-request results are bit-identical to a per-request launch: rows are independent in the kernel.
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


class AnomalyCoalescer:
    def __init__(self, eng: "engine.FFEngine", params, scale, feat_thr=None, agg_thr=None, max_batch_rows: int = 1 << 18,
                 max_wait_ms: float = 1.0, want: Optional[Sequence[str]] = None, x_scale=None, x_offset=None):
        torch = engine._torch()
        self.eng, self.params, self.scale, self.feat_thr, self.agg_thr = eng, params, scale, feat_thr, agg_thr
        if (x_scale is None) != (x_offset is None):
            raise ValueError("x_scale and x_offset go together")
        self.x_affine = (x_scale, x_offset) if x_scale is not None else None
        x_dtype = torch.float64 if self.x_affine is not None else torch.float32
        self._x_np = np.float64 if self.x_affine is not None else np.float32
        self.max_rows, self.max_wait = int(max_batch_rows), float(max_wait_ms) * 1e-3
        self.want = tuple(want) if want is not None else tuple(
            k for k in PER_TAG + PER_ROW if not ((feat_thr is None and k == "anomaly-confidence") or (agg_thr is None and k == "total-anomaly-confidence")))
        dev = eng.device
        self._stream = torch.cuda.Stream(device=dev)
        self._xh = torch.empty((self.max_rows, eng.n_in), dtype=x_dtype).pin_memory()
        self._yh = torch.empty((self.max_rows, eng.n_out), dtype=torch.float32).pin_memory()
        self._xd = torch.empty((self.max_rows, eng.n_in), dtype=x_dtype, device=dev)
        self._yd = torch.empty((self.max_rows, eng.n_out), dtype=torch.float32, device=dev)
        self._out_d = {k: torch.empty((self.max_rows, eng.n_out) if k in PER_TAG else (self.max_rows,), dtype=torch.float32, device=dev) for k in self.want}
        self._out_h = {k: torch.empty(v.shape, dtype=torch.float32).pin_memory() for k, v in self._out_d.items()}
        self._jobs_h = torch.empty((4096 * engine._cabi.JOB_DTYPE.itemsize,), dtype=torch.uint8).pin_memory()
        self._q: "queue.Queue" = queue.Queue()
        self._closed = False
        self.batches = 0
        self.requests = 0
        self._worker = threading.Thread(target=self._run, name="gordo-b200-coalescer", daemon=True)
        self._worker.start()

    # ------------------------------------------------------------------ client side
    def submit(self, slot: int, X, y) -> Future:
        """Queue one request; the Future resolves to {column block: host array} for exactly these rows."""
        if self._closed:
            raise RuntimeError("coalescer is closed")
        Xv = np.ascontiguousarray(getattr(X, "values", X), dtype=self._x_np)
        yv = np.ascontiguousarray(getattr(y, "values", y), dtype=np.float32)
        if Xv.ndim != 2 or Xv.shape[1] != self.eng.n_in or yv.shape != (len(Xv), self.eng.n_out):
            raise ValueError(f"request of shape X {Xv.shape} / y {yv.shape} does not fit a {self.eng.n_in}->{self.eng.n_out} model")
        if len(Xv) > self.max_rows:
            raise ValueError(f"a request of {len(Xv)} rows exceeds max_batch_rows={self.max_rows}")
        if not (0 <= int(slot) < self.params.shape[0]):
            raise ValueError(f"unknown machine slot {slot}")
        fut: Future = Future()
        self._q.put((int(slot), Xv, yv, fut))
        return fut

    def anomaly(self, slot: int, X, y) -> Dict[str, np.ndarray]:
        return self.submit(slot, X, y).result()

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
            batch, rows = [first], len(first[1])
            deadline = time.perf_counter() + self.max_wait
            while rows < self.max_rows and len(batch) < 4096:
                try:
                    item = self._q.get(timeout=max(0.0, deadline - time.perf_counter())) if self._q.empty() else self._q.get_nowait()
                except queue.Empty:
                    break
                if item is None:
                    self._q.put(None)
                    break
                if rows + len(item[1]) > self.max_rows:
                    pending = item
                    break
                batch.append(item)
                rows += len(item[1])
            try:
                self._launch(torch, batch, rows)
            except BaseException as exc:  # noqa: BLE001 - every waiting caller must hear about it
                for _, _, _, fut in batch:
                    if not fut.done():
                        fut.set_exception(exc)

    def _launch(self, torch, batch, rows):
        jobs = np.empty(len(batch), dtype=engine._cabi.JOB_DTYPE)
        ofs = 0
        xh, yh = self._xh.numpy(), self._yh.numpy()
        for i, (slot, Xv, yv, _) in enumerate(batch):
            n = len(Xv)
            xh[ofs:ofs + n] = Xv
            yh[ofs:ofs + n] = yv
            jobs[i] = (slot, n, ofs, ofs)
            ofs += n
        max_rows = int(jobs["n_rows"].max()) if len(jobs) else 0
        jb = self._jobs_h[: jobs.nbytes]
        jb.numpy()[:] = jobs.view(np.uint8)
        with torch.cuda.stream(self._stream):
            jobs_d = jb.to(self.eng.device, non_blocking=True)
            self._xd[:rows].copy_(self._xh[:rows], non_blocking=True)
            self._yd[:rows].copy_(self._yh[:rows], non_blocking=True)
            if rows:
                self.eng.infer_score(self.params, jobs_d, len(batch), max_rows, self._xd[:rows], self._yd[:rows], self.scale, self.feat_thr,
                                     self.agg_thr, out_rows=rows, want=self.want, out={k: v[:rows] for k, v in self._out_d.items()},
                                     x_affine=self.x_affine)
            for k in self.want:
                self._out_h[k][:rows].copy_(self._out_d[k][:rows], non_blocking=True)
        self._stream.synchronize()
        self.batches += 1
        self.requests += len(batch)
        ofs = 0
        for slot, Xv, _, fut in batch:
            n = len(Xv)
            fut.set_result({k: self._out_h[k][ofs:ofs + n].numpy().copy() for k in self.want})
            ofs += n
