"""
Fleet engine: the thin Python layer between gordo-style estimators and the C ABI.

It owns no arithmetic.  PyTorch supplies device memory and the current stream; every
number is produced by a kernel in ``csrc/`` reached through ``_cabi``.  The unit of work is
a *job* (``slot`` = which trained network, a row range of ``x``/``y`` and where the results
go), so one launch scores or trains thousands of machines -- the per-estimator methods in
``machine/model`` are the one-job special case of these functions.

Reference call sites replaced: keras ``Model.predict`` / ``Model.fit`` (gordo/machine/model/
models.py:284,300), sklearn ``MinMaxScaler.fit`` and the pandas arithmetic of
``DiffBasedAnomalyDetector`` (gordo/machine/model/anomaly/diff.py:166-458).
"""
from __future__ import annotations

import ctypes as C
import threading
import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _cabi

SCORE_KEYS = ("tag-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-scaled", "total-anomaly-unscaled",
              "anomaly-confidence", "total-anomaly-confidence")


def _torch():
    import torch

    return torch


def cuda_device(device=None):
    """Resolve a CUDA device or fail loudly -- there is no CPU path."""
    torch = _torch()
    if not torch.cuda.is_available():
        raise _cabi.GordoB200Error("no CUDA device visible: gordo_components_b200 runs on H100 (sm_90a) only, there is no CPU fallback")
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    _cabi.require_device(dev.index)
    return dev


def _stream_ptr():
    return C.c_void_p(_torch().cuda.current_stream().cuda_stream)


def make_jobs(slots, n_rows, x_rows, out_rows=None) -> np.ndarray:
    """Structured array of gb_job records."""
    slots = np.asarray(slots)
    jobs = np.zeros(len(slots), dtype=_cabi.JOB_DTYPE)
    jobs["slot"] = slots
    jobs["n_rows"] = n_rows
    jobs["x_row"] = x_rows
    jobs["out_row"] = x_rows if out_rows is None else out_rows
    return jobs


def uniform_jobs(n_machines: int, rows: int) -> np.ndarray:
    """Machine m owns rows [m*rows, (m+1)*rows) and slot m."""
    start = np.arange(n_machines, dtype=np.int64) * rows
    return make_jobs(np.arange(n_machines), rows, start)


def jobs_to_device(jobs: np.ndarray, device):
    torch = _torch()
    raw = torch.from_numpy(np.ascontiguousarray(jobs).view(np.uint8).copy())
    return raw.to(device, non_blocking=False)


class FFEngine:
    """All machines of one Dense-stack architecture (one bucket of the fleet)."""

    def __init__(self, dims: Sequence[int], acts: Sequence[str], l1: Optional[Sequence[float]] = None, device=None):
        self.lib = _cabi.load_library()
        self.device = cuda_device(device)
        self.dims, self.acts = [int(d) for d in dims], list(acts)
        self.l1 = [float(v) for v in (l1 if l1 is not None else [0.0] * (len(dims) - 1))]
        self.net = _cabi.make_ffnet(self.dims, self.acts, self.l1)
        self.n_params = int(self.lib.gb_ffnet_param_count(C.byref(self.net)))
        if self.n_params == 0:
            _cabi.check(-2)
        self.param_stride = int(self.lib.gb_ffnet_param_stride(C.byref(self.net)))
        self.state_stride = int(self.lib.gb_ffae_fit_state_stride(C.byref(self.net)))
        self.n_in, self.n_out = self.dims[0], self.dims[-1]

    # ------------------------------------------------------------------ parameter packing (host side, layout only)
    def pack_params(self, weights_per_slot: Sequence[Sequence[Tuple[np.ndarray, np.ndarray]]]):
        """[(W [in,out], b [out]) per layer] per slot  ->  device tensor [n_slots, param_stride] in Keras order."""
        torch = _torch()
        host = np.zeros((len(weights_per_slot), self.param_stride), dtype=np.float32)
        for s, layers in enumerate(weights_per_slot):
            ofs = 0
            for (W, b), i, o in zip(layers, self.dims[:-1], self.dims[1:]):
                W = np.asarray(W, dtype=np.float32)
                b = np.asarray(b, dtype=np.float32)
                if W.shape != (i, o) or b.shape != (o,):
                    raise ValueError(f"layer weights of shape {W.shape}/{b.shape} do not match the architecture ({i},{o})")
                host[s, ofs : ofs + i * o] = W.ravel()
                ofs += i * o
                host[s, ofs : ofs + o] = b
                ofs += o
        return torch.from_numpy(host).to(self.device)

    def unpack_params(self, params) -> List[List[Tuple[np.ndarray, np.ndarray]]]:
        host = params.detach().cpu().numpy()
        out = []
        for s in range(host.shape[0]):
            ofs, layers = 0, []
            for i, o in zip(self.dims[:-1], self.dims[1:]):
                W = host[s, ofs : ofs + i * o].reshape(i, o).copy()
                ofs += i * o
                b = host[s, ofs : ofs + o].copy()
                ofs += o
                layers.append((W, b))
            out.append(layers)
        return out

    # ------------------------------------------------------------------ K1 + K4
    def infer_score(self, params, jobs_dev, n_jobs: int, max_rows: int, x, y=None, scale=None, feat_thr=None, agg_thr=None,
                    out_rows: Optional[int] = None, want: Sequence[str] = SCORE_KEYS, variant: int = 0, out: Optional[Dict] = None,
                    x_affine=None):
        """
        One fused launch: model output (+ the requested anomaly columns) for every job.
        ``want`` selects score outputs (names as in the anomaly frame); outputs are float32 device tensors.
        ``x_affine``: None, or (a, b) float64 device tensors [n_slots, n_in], the per-slot input scaler of a Pipeline.  ``x`` is then
        float64 and the kernel applies ``(float)(x * a + b)`` as it reads it (gb_ffae_infer_score_x64): bit for bit ``affine_f64``
        followed by this call with the float32 result, on the same variant, in one launch.
        """
        torch = _torch()
        total = int(out_rows if out_rows is not None else x.shape[0])
        res = out if out is not None else {}

        def buf(name, shape):
            if name not in res:
                res[name] = torch.empty(shape, dtype=torch.float32, device=self.device)
            return res[name]

        o_model = buf("model-output", (total, self.n_out))
        score = y is not None
        sel = set(want) if score else set()
        if scale is None:
            sel -= {"tag-anomaly-scaled", "total-anomaly-scaled", "total-anomaly-confidence"}
        if feat_thr is None:
            sel.discard("anomaly-confidence")
        if agg_thr is None:
            sel.discard("total-anomaly-confidence")
        g = lambda name, shape: buf(name, shape) if name in sel else None  # noqa: E731
        o_ts = g("tag-anomaly-scaled", (total, self.n_out))
        o_tu = g("tag-anomaly-unscaled", (total, self.n_out))
        o_tots = g("total-anomaly-scaled", (total,))
        o_totu = g("total-anomaly-unscaled", (total,))
        o_conf = g("anomaly-confidence", (total, self.n_out))
        o_totc = g("total-anomaly-confidence", (total,))
        p = _cabi.ptr
        outs = (p(o_model), p(o_ts), p(o_tu), p(o_tots), p(o_totu), p(o_conf), p(o_totc), int(variant), _stream_ptr())
        if x_affine is None:
            _cabi.check(self.lib.gb_ffae_infer_score(
                C.byref(self.net), p(params), p(jobs_dev), int(n_jobs), int(max_rows), int(x.shape[0]), total, p(x), p(y), p(scale), p(feat_thr),
                p(agg_thr), *outs))
        else:
            a, b = x_affine
            if x.dtype != torch.float64 or a.dtype != torch.float64 or b.dtype != torch.float64:
                raise ValueError(f"x_affine takes float64 x, scale and offset, got {x.dtype}, {a.dtype}, {b.dtype}")
            _cabi.check(self.lib.gb_ffae_infer_score_x64(
                C.byref(self.net), p(params), p(jobs_dev), int(n_jobs), int(max_rows), int(x.shape[0]), total, p(x), p(a), p(b), p(y), p(scale),
                p(feat_thr), p(agg_thr), *outs))
        return res

    def infer_plan_x64(self, variant: int = 0):
        """(kernel, tensor-core warpgroups) ``infer_score(..., x_affine=...)`` runs on ``variant`` (gb_ffae_infer_plan_x64; no device
        work), or None when it refuses this architecture there."""
        kernel, nwg = C.c_int32(0), C.c_int32(0)
        rc = self.lib.gb_ffae_infer_plan_x64(C.byref(self.net), int(variant), C.byref(kernel), C.byref(nwg))
        return (kernel.value, nwg.value) if rc == 0 else None

    # ------------------------------------------------------------------ K2
    def fit(self, params, jobs_dev, n_jobs: int, max_rows: int, x, y, epochs: int = 1, batch_size: int = 32, shuffle=True,
            perm=None, adam: Optional[Dict[str, float]] = None, seed: int = 0, l1_div_batch: bool = False, state=None,
            step0: int = 0, loss: str = "mse", optimizer=None, reg=None, dropout=None):
        """
        Trains every job's slot in place (``params`` is updated).  Returns (loss [n_jobs, epochs], accuracy, (m, v)).
        ``perm`` (int32 [n_jobs, epochs, max_rows]) pins the visiting order (parity tests).  ``loss``: canonical Keras loss name
        (``_cabi.LOSS_CODES``) the fit minimises and reports.  ``optimizer``: None (Adam from ``adam``) or the (name, record) pair of
        ``factories.specs.resolve_optimizer`` (gb_ffae_fit_opt); (m, v) are then its state slots 0 and 1.  ``reg``: None or the
        per-layer weight regularizer coefficients ``factories.specs.fit_reg`` gives (gb_ffae_fit_reg), added to the loss the fit
        minimises and reports.  ``dropout``: None or the per-layer Dropout rates ``factories.specs.fit_dropout`` gives
        (gb_ffae_fit_drop): ``dropout[l]`` on the input of layer l, in training mini-batches only, masks keyed by ``seed``, the
        slot and the absolute optimizer step (``step0`` counts), so E one-epoch fits that carry ``step0`` draw the masks of one
        E-epoch fit.
        """
        hp = _fit_hparams(epochs, batch_size, shuffle, perm, adam, seed, l1_div_batch, step0, loss)
        hist, acc, *_, mv = self._fit_launch(params, jobs_dev, n_jobs, max_rows, x, y, perm, hp, state, optimizer, reg=reg, dropout=dropout)
        return hist, acc, mv

    def fit_split(self, params, jobs_dev, n_jobs: int, max_rows: int, x, y, split=None, row_map=None, val_batch: Optional[int] = None,
                  epochs: int = 1, batch_size: int = 32, shuffle=True, perm=None, adam: Optional[Dict[str, float]] = None, seed: int = 0,
                  l1_div_batch: bool = False, state=None, step0: int = 0, stop=None, loss: str = "mse", optimizer=None, reg=None,
                  dropout=None):
        """
        ``fit`` over row *positions* with Keras' ``validation_split``, in one launch (gb_ffae_fit_opt with a split).  Job i trains on its
        positions [0, n_rows) exactly as ``fit`` trains on its rows, and after every epoch runs the network forward over the held-out
        positions [n_rows, n_rows + split[i].n_val) in batches of ``val_batch`` (default ``batch_size``) rows -- what Keras reports as
        ``val_loss`` / ``val_accuracy``.  Position p reads row x_row + row_map[map_ofs + p] (x_row + p where map_ofs is -1).

        ``split``: ``make_split`` records [n_jobs] (host array or device bytes), None = no held-out positions and no map.
        ``row_map``: int32 device tensor of row indices relative to a job's x_row, shared by the jobs through map_ofs.
        Returns (loss, accuracy, val_loss, val_accuracy, (m, v)), each [n_jobs, epochs]; val_* rows of jobs without held-out
        positions are NaN.

        ``stop``: ``make_stop`` records [n_jobs] (host array or device bytes): every job applies its Keras EarlyStopping rule at the
        end of each epoch inside the launch (gb_ffae_fit_opt with a stop array) and leaves the kernel when it fires; with ``restore_best_weights``
        its slot of ``params`` ends with the weights of its best epoch.  Returns (loss, accuracy, val_loss, val_accuracy,
        epochs_run, best_epoch, (m, v)): epochs_run / best_epoch are int32 [n_jobs] (best_epoch -1 when no epoch improved and no
        snapshot was taken), and every history entry past a job's epochs_run is NaN.

        ``loss``, ``optimizer``, ``reg``, ``dropout``: as in ``fit``; the held-out statistics report the same loss, without dropout.
        """
        hp = _fit_hparams(epochs, batch_size, shuffle, perm, adam, seed, l1_div_batch, step0, loss)
        vb = int(val_batch if val_batch is not None else batch_size)
        *out, epochs_run, best_epoch, mv = self._fit_launch(params, jobs_dev, n_jobs, max_rows, x, y, perm, hp, state, optimizer, val=True,
                                                            split=split, row_map=row_map, val_batch=vb, stop=stop, reg=reg,
                                                            dropout=dropout)
        return (*out, mv) if stop is None else (*out, epochs_run, best_epoch, mv)

    def _fit_launch(self, params, jobs_dev, n_jobs, max_rows, x, y, perm, hp, state, optimizer, val=False, split=None, row_map=None,
                    val_batch=1, stop=None, reg=None, dropout=None):
        """
        The one gb_ffae_fit_opt launch of ``fit`` and ``fit_split``, with NULL where there is no split, stop rule or optimizer; with a
        ``reg`` that has a non-zero coefficient, the gb_ffae_fit_reg launch instead, and with a ``dropout`` that has a non-zero rate,
        the gb_ffae_fit_drop launch (NULL ``reg`` where it has none).
        Returns (loss, accuracy, val_loss, val_accuracy, epochs_run, best_epoch, (m, v)): val_* (NaN where no held-out pass writes)
        only with ``val``; epochs_run / best_epoch only with ``stop``, which also fills loss / accuracy with NaN first.
        """
        torch = _torch()
        m, v = self._fit_state(params, state)
        if split is not None and isinstance(split, np.ndarray):
            split = jobs_to_device(split, self.device)
        shape = (n_jobs, hp.epochs)
        make = torch.empty if stop is None else (lambda shape, **kw: torch.full(shape, float("nan"), **kw))  # noqa: E731
        out = [make(shape, dtype=torch.float32, device=self.device) for _ in range(2)]
        out += [torch.full(shape, float("nan"), dtype=torch.float32, device=self.device) if val else None for _ in range(2)]
        best = epochs_run = best_epoch = None
        if stop is not None:
            if isinstance(stop, np.ndarray):
                stop = jobs_to_device(stop, self.device)
            best = torch.empty_like(params)  # snapshot area
            epochs_run = torch.zeros((n_jobs,), dtype=torch.int32, device=self.device)
            best_epoch = torch.full((n_jobs,), -1, dtype=torch.int32, device=self.device)
        opt = None if optimizer is None else _cabi.make_optimizer(*optimizer)
        p = _cabi.ptr
        args = (C.byref(self.net), p(params), p(m), p(v), p(jobs_dev), p(split), int(n_jobs), int(max_rows), p(x), p(y), p(row_map), p(perm),
                C.byref(hp), int(val_batch), *(p(t) for t in out), p(stop), p(best), p(epochs_run), p(best_epoch),
                None if opt is None else C.byref(opt))
        has_reg = reg is not None and any(v for vals in reg.values() for v in vals)
        if dropout is not None and any(dropout):
            rec = _cabi.make_dense_reg(**reg) if has_reg else None
            drop = _cabi.make_dense_dropout(dropout)
            _cabi.check(self.lib.gb_ffae_fit_drop(*args, None if rec is None else C.byref(rec), C.byref(drop), _stream_ptr()))
        elif has_reg:
            rec = _cabi.make_dense_reg(**reg)
            _cabi.check(self.lib.gb_ffae_fit_reg(*args, C.byref(rec), _stream_ptr()))
        else:
            _cabi.check(self.lib.gb_ffae_fit_opt(*args, _stream_ptr()))
        return (*out, epochs_run, best_epoch, (m, v))

    def _fit_state(self, params, state):
        """Optimizer state slots (m, v) of every slot: the given pair, or zeros for a fresh fit."""
        if state is not None:
            return state
        torch = _torch()
        m = torch.zeros((params.shape[0], self.state_stride), dtype=torch.float32, device=self.device)
        return m, torch.zeros_like(m)

    # ------------------------------------------------------------------ K7 / K5 / K4-alone (architecture independent)
    def minmax_fit(self, jobs_dev, n_jobs, max_rows, y, n_slots):
        return minmax_fit(jobs_dev, n_jobs, max_rows, y, self.n_out, n_slots, self.device)

    def thresholds(self, jobs_dev, n_jobs, max_rows, tag_unscaled, total_scaled, n_slots, window=6):
        return thresholds(jobs_dev, n_jobs, max_rows, tag_unscaled, total_scaled, self.n_out, n_slots, window, self.device)

    def thresholds_pair(self, jobs_dev, n_jobs, max_rows, tag_unscaled, total_scaled, n_slots, w0, w1):
        return thresholds_pair(jobs_dev, n_jobs, max_rows, tag_unscaled, total_scaled, self.n_out, n_slots, w0, w1, self.device)


def fit_plan(dims: Sequence[int], acts: Sequence[str], l1: Optional[Sequence[float]] = None) -> Optional[Tuple[int, int]]:
    """The memory plan of the Dense fit for this architecture (gb_ffae_fit_plan; no device needed): (weights in L2, dz buffers in
    L2), or None when the fit refuses the architecture.  Nets of one ``fit_group`` launch share it."""
    lib = _cabi.load_library()
    try:
        net = _cabi.make_ffnet([int(d) for d in dims], list(acts), l1)
    except ValueError:
        return None
    w, d = C.c_int32(0), C.c_int32(0)
    return (w.value, d.value) if lib.gb_ffae_fit_plan(C.byref(net), C.byref(w), C.byref(d)) == 0 else None


class FitGroup:
    """One architecture's part of a ``fit_group`` launch, in the form ``FFEngine.fit_split`` takes it: the engine, the slots' params
    (trained in place), the device jobs, their count and longest row range, x and y, and optionally the ``make_split`` records with
    their row map, a pinned visiting order ``perm`` [n_jobs, epochs, max_rows], the optimizer state (m, v) and ``make_stop`` records."""

    def __init__(self, eng: FFEngine, params, jobs_dev, n_jobs: int, max_rows: int, x, y, split=None, row_map=None, perm=None, state=None,
                 stop=None):
        self.eng, self.params, self.jobs_dev, self.n_jobs, self.max_rows = eng, params, jobs_dev, int(n_jobs), int(max_rows)
        self.x, self.y, self.split, self.row_map, self.perm, self.state, self.stop = x, y, split, row_map, perm, state, stop


def _host_records(rec, dtype, n: int) -> np.ndarray:
    """``n`` split or stop records as a host array, from a host array or device bytes."""
    if isinstance(rec, np.ndarray):
        return np.ascontiguousarray(rec[:n])
    return rec.cpu().numpy().view(dtype)[:n].copy()


def fit_group(groups: Sequence[FitGroup], val_batch: Optional[int] = None, epochs: int = 1, batch_size: int = 32, shuffle=True,
              adam: Optional[Dict[str, float]] = None, seed: int = 0, l1_div_batch: bool = False, step0: int = 0, loss: str = "mse",
              optimizer=None, reg=None, dropout=None):
    """
    ``FFEngine.fit_split`` of several architectures in one launch (gb_ffae_fit_group): every group's jobs train its own slots on
    its own rows, and each group gets back exactly what ``fit_split`` with the same arguments returns for it alone -- (loss,
    accuracy, val_loss, val_accuracy, (m, v)), with ``epochs_run, best_epoch`` before (m, v) when the groups carry stop records --
    bit for bit.  The keyword arguments are ``fit_split``'s and apply to every group.  The groups must share a memory plan
    (``fit_plan``) and an entry point: split records for all or none, stop records for all or none, perm for all or none.
    Row maps are laid end to end and each group's ``map_ofs`` moved with its map.
    """
    torch = _torch()
    groups = list(groups)
    if not groups:
        return []
    for what in ("split", "stop", "perm"):
        if len({getattr(g, what) is None for g in groups}) > 1:
            raise ValueError(f"fit_group: {what} for some groups but not all; the groups of one launch share an entry point")
    dev = groups[0].eng.device
    counts = [g.n_jobs for g in groups]
    n, max_rows = sum(counts), max(g.max_rows for g in groups)
    jobs_dev = torch.cat([g.jobs_dev[: c * _cabi.JOB_DTYPE.itemsize] for g, c in zip(groups, counts)])
    job_group = np.repeat(np.arange(len(groups), dtype=np.int32), counts)
    split = row_map = stop = perm = None
    if groups[0].split is not None:
        parts, maps, ofs = [], [], 0
        for g, c in zip(groups, counts):
            s = _host_records(g.split, _cabi.SPLIT_DTYPE, c)
            if g.row_map is None:
                s["map_ofs"] = -1  # without a map the kernel never reads it
            else:
                s["map_ofs"] = np.where(s["map_ofs"] >= 0, s["map_ofs"] + ofs, -1)
                maps.append(g.row_map.reshape(-1))
                ofs += int(g.row_map.numel())
            parts.append(s)
        split = jobs_to_device(np.concatenate(parts), dev)
        row_map = torch.cat(maps) if maps else None
    if groups[0].stop is not None:
        stop = jobs_to_device(np.concatenate([_host_records(g.stop, _cabi.STOP_DTYPE, c) for g, c in zip(groups, counts)]), dev)
    if groups[0].perm is not None:
        perm = torch.zeros((n, int(epochs), max_rows), dtype=torch.int32, device=dev)
        for g, j0, c in zip(groups, np.cumsum([0] + counts[:-1]), counts):
            perm[j0:j0 + c, :, :g.max_rows] = g.perm[:c]
    hp = _fit_hparams(epochs, batch_size, shuffle, perm, adam, seed, l1_div_batch, step0, loss)
    states = [g.eng._fit_state(g.params, g.state) for g in groups]
    shape = (n, hp.epochs)
    make = torch.empty if stop is None else (lambda shape, **kw: torch.full(shape, float("nan"), **kw))  # noqa: E731
    out = [make(shape, dtype=torch.float32, device=dev) for _ in range(2)]
    out += [torch.full(shape, float("nan"), dtype=torch.float32, device=dev) for _ in range(2)]
    bests = [None] * len(groups)
    epochs_run = best_epoch = None
    if stop is not None:
        bests = [torch.empty_like(g.params) for g in groups]
        epochs_run = torch.zeros((n,), dtype=torch.int32, device=dev)
        best_epoch = torch.full((n,), -1, dtype=torch.int32, device=dev)
    p = _cabi.ptr
    recs = (_cabi.GbFitGroup * len(groups))()
    for r, g, (m, v), best in zip(recs, groups, states, bests):
        r.net = g.eng.net
        r.params, r.adam_m, r.adam_v, r.best_params, r.x, r.y = (p(t) for t in (g.params, m, v, best, g.x, g.y))
    opt = None if optimizer is None else _cabi.make_optimizer(*optimizer)
    has_reg = reg is not None and any(v for vals in reg.values() for v in vals)
    rec = _cabi.make_dense_reg(**reg) if has_reg else None
    drop = _cabi.make_dense_dropout(dropout) if dropout is not None and any(dropout) else None
    jg = np.ascontiguousarray(job_group)
    lib = groups[0].eng.lib
    ws = torch.empty((int(lib.gb_ffae_fit_group_workspace_bytes(len(groups), n)),), dtype=torch.uint8, device=dev)  # records + job_group
    _cabi.check(lib.gb_ffae_fit_group(
        recs, len(groups), jg.ctypes.data_as(C.POINTER(C.c_int32)), p(jobs_dev), p(split), n, max_rows, p(row_map), p(perm), C.byref(hp),
        int(val_batch if val_batch is not None else batch_size), *(p(t) for t in out), p(stop), p(epochs_run), p(best_epoch),
        None if opt is None else C.byref(opt), None if rec is None else C.byref(rec), None if drop is None else C.byref(drop), p(ws),
        _stream_ptr()))
    res, j0 = [], 0
    for g, c, mv in zip(groups, counts, states):
        part = tuple(t[j0:j0 + c] for t in out)
        res.append((*part, mv) if stop is None else (*part, epochs_run[j0:j0 + c], best_epoch[j0:j0 + c], mv))
        j0 += c
    return res


def _fit_hparams(epochs, batch_size, shuffle, perm, adam, seed, l1_div_batch, step0, loss="mse") -> "_cabi.GbFitHParams":
    adam = adam or {}
    hp = _cabi.GbFitHParams()
    hp.epochs, hp.batch_size = int(epochs), int(batch_size)
    hp.shuffle = 2 if perm is not None else (1 if shuffle else 0)
    hp.l1_div_batch = int(bool(l1_div_batch))
    hp.lr, hp.beta1 = float(adam.get("lr", 1e-3)), float(adam.get("beta1", 0.9))
    hp.beta2, hp.eps = float(adam.get("beta2", 0.999)), float(adam.get("eps", 1e-7))
    hp.seed, hp.step0 = int(seed) & (2**64 - 1), int(step0)
    hp.loss = _cabi.loss_code(loss)
    return hp


def make_split(n_val, map_ofs=-1) -> np.ndarray:
    """Structured array of gb_fit_split records (per job: held-out positions, offset of its row map or -1)."""
    n_val = np.atleast_1d(np.asarray(n_val))
    split = np.zeros(len(n_val), dtype=_cabi.SPLIT_DTYPE)
    split["n_val"] = n_val
    split["map_ofs"] = map_ofs
    return split


STOP_ARGS = ("monitor", "min_delta", "patience", "mode", "baseline", "restore_best_weights", "start_from_epoch")


def make_stop(callbacks_per_job) -> np.ndarray:
    """
    Structured array of gb_fit_stop records, one per job, from Keras EarlyStopping callbacks: ``EarlyStopping`` objects (ours or
    anything with its attributes) or dicts of its constructor arguments.  Each goes through ``EarlyStopping.__init__``, so
    ``mode="auto"`` and the sign of ``min_delta`` resolve exactly as the per-machine fit loop resolves them.  The monitor must be
    one the fit kernel writes: loss, accuracy, val_loss or val_accuracy.
    """
    from .machine.model.models import EarlyStopping

    stop = np.zeros(len(callbacks_per_job), dtype=_cabi.STOP_DTYPE)
    for j, cb in enumerate(callbacks_per_job):
        kw = dict(cb) if isinstance(cb, dict) else {k: getattr(cb, k) for k in STOP_ARGS if hasattr(cb, k)}
        cb = EarlyStopping(**kw)
        if cb.monitor not in _cabi.STOP_MONITORS:
            raise ValueError(f"EarlyStopping monitor {cb.monitor!r} is not one of {sorted(_cabi.STOP_MONITORS)}")
        stop[j] = (_cabi.STOP_MONITORS[cb.monitor], 1 if cb.mode == "min" else -1, cb.patience, cb.start_from_epoch,
                   int(cb.restore_best_weights), int(cb.baseline is not None), cb.min_delta,
                   0.0 if cb.baseline is None else float(cb.baseline))
    return stop


def minmax_fit(jobs_dev, n_jobs, max_rows, y, n_out, n_slots, device, return_minmax=False):
    """
    MinMaxScaler.fit per job on device: returns (scale_ [n_slots, n_out], min_ [n_slots, n_out]); with ``return_minmax`` also
    the raw (data_min_, data_max_) the kernel found -- exact float32 values, for callers that need sklearn's float64 arithmetic
    on them (a scaler in front of the network, where ``x * scale_ + min_`` cancels for offset-dominated tags).
    """
    torch = _torch()
    lib = _cabi.load_library()
    scale = torch.ones((n_slots, n_out), dtype=torch.float32, device=device)
    offset = torch.zeros((n_slots, n_out), dtype=torch.float32, device=device)
    ws = torch.empty((n_slots, 2, n_out), dtype=torch.float32, device=device)
    p = _cabi.ptr
    _cabi.check(lib.gb_minmax_fit(p(jobs_dev), int(n_jobs), int(max_rows), p(y), int(n_out), p(scale), p(offset), p(ws), int(n_slots), _stream_ptr()))
    if return_minmax:
        return scale, offset, ws[:, 0], ws[:, 1]
    return scale, offset


def minmax_f64(jobs_dev, n_jobs, max_rows, y64, n_slots):
    """Column (min, max) of float64 targets per job: two [n_slots, n_out] float64 tensors (NaNs skipped, +-inf when a column has none)."""
    torch = _torch()
    lib = _cabi.load_library()
    if y64.dtype != torch.float64:
        raise ValueError(f"minmax_f64 takes float64 targets, got {y64.dtype}")
    n_out = y64.shape[1]
    mm = torch.empty((int(n_slots), 2, n_out), dtype=torch.float64, device=y64.device)
    p = _cabi.ptr
    _cabi.check(lib.gb_minmax_f64(p(jobs_dev), int(n_jobs), int(max_rows), p(y64), int(n_out), p(mm), int(n_slots), _stream_ptr()))
    return mm[:, 0], mm[:, 1]


def thresholds(jobs_dev, n_jobs, max_rows, tag_unscaled, total_scaled, n_out, n_slots, window, device):
    """
    rolling(window).min().max() per tag and for the aggregate series: (feat_thr [n_slots, n_out], agg_thr [n_slots]).
    float32 or float64 score arrays (the dtype of ``tag_unscaled`` decides; both arrays must agree).
    """
    torch = _torch()
    lib = _cabi.load_library()
    dtype = tag_unscaled.dtype
    if total_scaled.dtype != dtype or dtype not in (torch.float32, torch.float64):
        raise ValueError(f"thresholds need two float32 or two float64 arrays, got {dtype} / {total_scaled.dtype}")
    feat = torch.full((n_slots, n_out), float("nan"), dtype=dtype, device=device)
    agg = torch.full((n_slots,), float("nan"), dtype=dtype, device=device)
    p = _cabi.ptr
    fn = lib.gb_thresholds if dtype == torch.float32 else lib.gb_thresholds_f64
    _cabi.check(fn(p(jobs_dev), int(n_jobs), int(max_rows), p(tag_unscaled), p(total_scaled), int(n_out), int(window),
                                  p(feat), p(agg), int(n_slots), _stream_ptr()))
    return feat, agg


def thresholds_pair(jobs_dev, n_jobs, max_rows, tag_unscaled, total_scaled, n_out, n_slots, w0, w1, device):
    """
    ``thresholds`` at two windows from one pass over the score arrays (gb_thresholds_pair): (feat_thr0, agg_thr0, feat_thr1,
    agg_thr1), the first pair at ``w0`` and the second at ``w1``, each bit for bit what ``thresholds`` gives at that window.
    """
    torch = _torch()
    lib = _cabi.load_library()
    dtype = tag_unscaled.dtype
    if total_scaled.dtype != dtype or dtype not in (torch.float32, torch.float64):
        raise ValueError(f"thresholds need two float32 or two float64 arrays, got {dtype} / {total_scaled.dtype}")
    out = [torch.full(shape, float("nan"), dtype=dtype, device=device) for shape in ((n_slots, n_out), (n_slots,)) * 2]
    p = _cabi.ptr
    fn = lib.gb_thresholds_pair if dtype == torch.float32 else lib.gb_thresholds_pair_f64
    _cabi.check(fn(p(jobs_dev), int(n_jobs), int(max_rows), p(tag_unscaled), p(total_scaled), int(n_out), int(w0), int(w1),
                   *(p(t) for t in out), int(n_slots), _stream_ptr()))
    return tuple(out)


def cv_moments(jobs_dev, n_jobs, yhat, y, n_out):
    """Per job and column: sums of e, e^2, |e|, (y-y0), (y-y0)^2 over the job's rows (e = yhat - y): [n_jobs, 5, n_out] float64."""
    torch = _torch()
    lib = _cabi.load_library()
    out = torch.zeros((int(n_jobs), 5, int(n_out)), dtype=torch.float64, device=yhat.device)
    if int(n_jobs) == 0:
        return out
    p = _cabi.ptr
    _cabi.check(lib.gb_cv_moments(p(jobs_dev), int(n_jobs), p(yhat), p(y), int(n_out), p(out), _stream_ptr()))
    return out


def anomaly_score(jobs_dev, n_jobs, max_rows, yhat, y, n_out, scale=None, feat_thr=None, agg_thr=None, want=SCORE_KEYS, device=None):
    """
    Anomaly columns for predictions that already exist (base estimators that are not ours, LSTM outputs).  float64 ``yhat`` selects
    the float64 kernel (the reference's own precision, diff.py:268-300, 350-385): every operand must then be float64 and so are the results.
    """
    torch = _torch()
    lib = _cabi.load_library()
    device = yhat.device
    total = yhat.shape[0]
    dtype = yhat.dtype
    for name, t in (("y", y), ("scale", scale), ("feat_thr", feat_thr), ("agg_thr", agg_thr)):
        if t is not None and t.dtype != dtype:
            raise ValueError(f"anomaly_score: {name} is {t.dtype}, yhat is {dtype}")
    fn = {torch.float32: lib.gb_anomaly_score, torch.float64: lib.gb_anomaly_score_f64}.get(dtype)
    if fn is None:
        raise ValueError(f"anomaly_score takes float32 or float64 arrays, not {dtype}")
    sel = set(want)
    if scale is None:
        sel -= {"tag-anomaly-scaled", "total-anomaly-scaled", "total-anomaly-confidence"}
    if feat_thr is None:
        sel.discard("anomaly-confidence")
    if agg_thr is None:
        sel.discard("total-anomaly-confidence")
    res = {}

    def g(name, shape):
        if name in sel:
            res[name] = torch.empty(shape, dtype=dtype, device=device)
            return res[name]
        return None

    o_ts = g("tag-anomaly-scaled", (total, n_out))
    o_tu = g("tag-anomaly-unscaled", (total, n_out))
    o_tots = g("total-anomaly-scaled", (total,))
    o_totu = g("total-anomaly-unscaled", (total,))
    o_conf = g("anomaly-confidence", (total, n_out))
    o_totc = g("total-anomaly-confidence", (total,))
    p = _cabi.ptr
    _cabi.check(fn(p(jobs_dev), int(n_jobs), int(max_rows), p(yhat), p(y), int(n_out), p(scale), p(feat_thr), p(agg_thr),
                                     p(o_ts), p(o_tu), p(o_tots), p(o_totu), p(o_conf), p(o_totc), _stream_ptr()))
    return res


def quantile(jobs_dev, n_jobs, max_rows, arr, q: float):
    """pandas ``.quantile(q)`` (linear interpolation, NaNs skipped) of every column of ``arr`` per job -> [n_jobs, n_cols]."""
    torch = _torch()
    lib = _cabi.load_library()
    a2 = arr if arr.dim() == 2 else arr.reshape(-1, 1)
    out = torch.empty((int(n_jobs), a2.shape[1]), dtype=torch.float32, device=a2.device)
    p = _cabi.ptr
    _cabi.check(lib.gb_quantile(p(jobs_dev), int(n_jobs), int(max_rows), p(a2), int(a2.shape[1]), float(q), p(out), _stream_ptr()))
    return out


def affine_f64(jobs_dev, n_jobs, max_rows, x64, a, b, out_rows=None):
    """Per-feature ``x * a[slot] + b[slot]`` in float64 on the device, rounded once to float32 (sklearn scalers' transform)."""
    torch = _torch()
    lib = _cabi.load_library()
    n_cols = x64.shape[1]
    out = torch.empty((int(out_rows if out_rows is not None else x64.shape[0]), n_cols), dtype=torch.float32, device=x64.device)
    p = _cabi.ptr
    _cabi.check(lib.gb_affine_f64(p(jobs_dev), int(n_jobs), int(max_rows), p(x64), int(n_cols), p(a), p(b), p(out), _stream_ptr()))
    return out


def gather_rows(jobs_dev, n_jobs, max_rows, row_map, src, out_rows: int, to_f32: bool = False, out=None, map_ofs=None):
    """
    Row permutation per job (gb_gather_rows): out[out_row + p] = src[x_row + row_map[p]] for p < n_rows.  ``src``: [rows, cols]
    or [rows] tensor of 4- or 8-byte elements; ``to_f32`` narrows float64 to float32 in the same pass.  ``row_map``: int32 device
    tensor shared by every job.  ``map_ofs``: int64 device tensor [n_jobs] giving each job its own map, row_map[map_ofs[i] + p]
    (gb_gather_rows_ragged).  Returns ``out`` ([out_rows, ...], allocated when not given).
    """
    torch = _torch()
    lib = _cabi.load_library()
    if row_map.dtype != torch.int32:
        raise ValueError(f"gather_rows takes an int32 row map, got {row_map.dtype}")
    if to_f32 and src.dtype != torch.float64:
        raise ValueError(f"gather_rows narrows float64 to float32, got {src.dtype}")
    n_cols = 1 if src.dim() == 1 else int(src.shape[1])
    dtype = torch.float32 if to_f32 else src.dtype
    if out is None:
        out = torch.empty((int(out_rows),) + tuple(src.shape[1:]), dtype=dtype, device=src.device)
    if out.dtype != dtype:
        raise ValueError(f"gather_rows: out is {out.dtype}, expected {dtype}")
    p = _cabi.ptr
    if map_ofs is not None:
        if map_ofs.dtype != torch.int64:
            raise ValueError(f"gather_rows takes int64 map offsets, got {map_ofs.dtype}")
        _cabi.check(lib.gb_gather_rows_ragged(p(jobs_dev), int(n_jobs), int(max_rows), p(row_map), p(map_ofs), p(src), n_cols, int(src.element_size()),
                                              int(bool(to_f32)), p(out), _stream_ptr()))
        return out
    _cabi.check(lib.gb_gather_rows(p(jobs_dev), int(n_jobs), int(max_rows), p(row_map), p(src), n_cols, int(src.element_size()), int(bool(to_f32)),
                                   p(out), _stream_ptr()))
    return out


def minmax_inverse_f32(jobs_dev, n_jobs, max_rows, pred, scale, min_, out_rows=None, want=("f32", "f64")):
    """
    ``MinMaxScaler.inverse_transform`` of float32 predictions as sklearn computes it on a float32 array (gb_minmax_inverse_f32):
    per job, rows of ``pred`` at x_row with the float64 ``scale_`` / ``min_`` of its slot, to rows at out_row.  Returns the
    requested forms, ``{"f32": float32 tensor, "f64": the same values as float64}``.
    """
    torch = _torch()
    lib = _cabi.load_library()
    total = int(out_rows if out_rows is not None else pred.shape[0])
    res = {}
    if "f32" in want:
        res["f32"] = torch.empty((total, pred.shape[1]), dtype=torch.float32, device=pred.device)
    if "f64" in want:
        res["f64"] = torch.empty((total, pred.shape[1]), dtype=torch.float64, device=pred.device)
    p = _cabi.ptr
    _cabi.check(lib.gb_minmax_inverse_f32(p(jobs_dev), int(n_jobs), int(max_rows), p(pred), int(pred.shape[1]), p(scale), p(min_), p(res.get("f32")),
                                          p(res.get("f64")), _stream_ptr()))
    return res


def minmax_inverse_score_f64(jobs_dev, n_jobs, max_rows, pred, y, y_scale, y_min, scale=None, feat_thr=None, agg_thr=None,
                             want=SCORE_KEYS, out_rows=None, out=None):
    """
    The anomaly columns of a ``TransformedTargetRegressor(transformer=MinMaxScaler)`` prediction in one launch
    (gb_minmax_inverse_score_f64): the float32 network output ``pred`` goes through sklearn's float32 ``inverse_transform`` with the
    slot's float64 ``y_scale`` / ``y_min`` ([n_slots, n_out]) and is scored in float64 against the float64 ``y``, bit for bit
    ``minmax_inverse_f32`` followed by ``anomaly_score`` on its float64 form.  ``pred`` and the outputs at out_row, ``y`` at x_row.
    Returns ``{"model-output": float32, <want>: float64}`` keyed as ``anomaly_score`` keys them; ``out`` may hold preallocated
    tensors under those keys (``out["model-output"]`` may be ``pred`` itself: the inverse is then written in place).
    """
    torch = _torch()
    lib = _cabi.load_library()
    n_out = int(pred.shape[1])
    total = int(out_rows if out_rows is not None else pred.shape[0])
    if pred.dtype != torch.float32:
        raise ValueError(f"minmax_inverse_score_f64 takes a float32 prediction, got {pred.dtype}")
    for name, t in (("y", y), ("y_scale", y_scale), ("y_min", y_min), ("scale", scale), ("feat_thr", feat_thr), ("agg_thr", agg_thr)):
        if t is not None and t.dtype != torch.float64:
            raise ValueError(f"minmax_inverse_score_f64: {name} is {t.dtype}, not float64")
    sel = set(want)
    if scale is None:
        sel -= {"tag-anomaly-scaled", "total-anomaly-scaled", "total-anomaly-confidence"}
    if feat_thr is None:
        sel.discard("anomaly-confidence")
    if agg_thr is None:
        sel.discard("total-anomaly-confidence")
    res = {}

    def g(name, shape, dtype=torch.float64):
        if name != "model-output" and name not in sel:
            return None
        if out is not None and name in out:
            res[name] = out[name]
        else:
            res[name] = torch.empty(shape, dtype=dtype, device=pred.device)
        return res[name]

    o_model = g("model-output", (total, n_out), torch.float32)
    o_ts = g("tag-anomaly-scaled", (total, n_out))
    o_tu = g("tag-anomaly-unscaled", (total, n_out))
    o_tots = g("total-anomaly-scaled", (total,))
    o_totu = g("total-anomaly-unscaled", (total,))
    o_conf = g("anomaly-confidence", (total, n_out))
    o_totc = g("total-anomaly-confidence", (total,))
    p = _cabi.ptr
    _cabi.check(lib.gb_minmax_inverse_score_f64(p(jobs_dev), int(n_jobs), int(max_rows), p(pred), p(y), n_out, p(y_scale), p(y_min), p(scale),
                                                p(feat_thr), p(agg_thr), p(o_model), p(o_ts), p(o_tu), p(o_tots), p(o_totu), p(o_conf), p(o_totc),
                                                _stream_ptr()))
    return res


def orthonormal_rows(g, out, out_offset: int, out_stride: int):
    """
    Keras' Orthogonal initialiser for every float64 standard-normal draw ``g`` [n, rows, cols] (overwritten): the rows
    orthonormalised, written as float32 into the dense tensor ``out`` at element ``out_offset + i * out_stride`` for matrix i.
    """
    lib = _cabi.load_library()
    n, rows, cols = (int(d) for d in g.shape)
    if g.dtype != _torch().float64 or out.dtype != _torch().float32:
        raise ValueError(f"orthonormal_rows takes float64 draws and a float32 output, got {g.dtype} / {out.dtype}")
    if n and int(out_offset) + (n - 1) * int(out_stride) + rows * cols > out.numel():
        raise ValueError("orthonormal_rows: the matrices do not fit into out")
    p = _cabi.ptr
    _cabi.check(lib.gb_orthonormal_rows(p(g), n, rows, cols, p(out), int(out_offset), int(out_stride), _stream_ptr()))


SMOOTH_METHODS = {"smm": 0, "sma": 1, "ewma": 2}


def smooth(jobs_dev, n_jobs, arr, window: int, method: str, max_rows: Optional[int] = None):
    """
    Rolling median / mean / EWMA of every column of ``arr`` ([rows] or [rows, cols]) per job (pandas semantics, NaNs included).
    ``max_rows``: longest job (defaults to the length of ``arr``, always an upper bound).
    """
    torch = _torch()
    lib = _cabi.load_library()
    if method not in SMOOTH_METHODS:
        raise ValueError(f"smoothing_method {method!r} must be one of {sorted(SMOOTH_METHODS)}")
    n_cols = 1 if arr.dim() == 1 else arr.shape[1]
    out = torch.full_like(arr, float("nan"))
    p = _cabi.ptr
    _cabi.check(lib.gb_smooth(p(jobs_dev), int(n_jobs), int(max_rows if max_rows is not None else arr.shape[0]), p(arr), int(n_cols), int(window),
                              SMOOTH_METHODS[method], p(out), _stream_ptr()))
    return out


SMOOTH_SCORE_KEYS = ("tag-anomaly-scaled", "total-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-unscaled")


def smooth_scores(jobs_dev, n_jobs, max_rows, scores, window: int, method: str):
    """
    ``smooth`` of the four anomaly arrays of every job in one launch (gb_smooth_scores): ``scores`` holds the SMOOTH_SCORE_KEYS
    arrays ([rows, tags] / [rows], all float32 or all float64; float64 is rounded to float32 as it is read).  Returns
    ``{"smooth-<key>": float32 tensor of the same shape}``; rows outside every job are NaN.
    """
    torch = _torch()
    lib = _cabi.load_library()
    if method not in SMOOTH_METHODS:
        raise ValueError(f"smoothing_method {method!r} must be one of {sorted(SMOOTH_METHODS)}")
    ins = [scores[k] for k in SMOOTH_SCORE_KEYS]
    dtype = ins[0].dtype
    if dtype not in (torch.float32, torch.float64) or any(t.dtype != dtype for t in ins):
        raise ValueError(f"smooth_scores takes four float32 or four float64 arrays, got {[t.dtype for t in ins]}")
    rows, n_tags = ins[0].shape
    if ins[2].shape != (rows, n_tags) or ins[1].shape != (rows,) or ins[3].shape != (rows,):
        raise ValueError(f"smooth_scores: score arrays of shapes {[tuple(t.shape) for t in ins]} are not [rows, tags] / [rows]")
    out = {"smooth-" + k: torch.full(t.shape, float("nan"), dtype=torch.float32, device=t.device) for k, t in zip(SMOOTH_SCORE_KEYS, ins)}
    p = _cabi.ptr
    _cabi.check(lib.gb_smooth_scores(p(jobs_dev), int(n_jobs), int(max_rows), *(p(t) for t in ins), int(dtype == torch.float64), int(n_tags),
                                     int(window), SMOOTH_METHODS[method], *(p(out["smooth-" + k]) for k in SMOOTH_SCORE_KEYS), _stream_ptr()))
    return out


class LSTMEngine:
    """All machines of one LSTM-stack architecture."""

    def __init__(self, n_features, units, acts, n_features_out, out_func, lookback, device=None):
        self.lib = _cabi.load_library()
        self.device = cuda_device(device)
        self.n_features, self.units, self.acts = int(n_features), [int(u) for u in units], list(acts)
        self.n_out, self.out_func, self.lookback = int(n_features_out), out_func, int(lookback)
        self.net = _cabi.make_lstmnet(n_features, units, acts, n_features_out, out_func, lookback)
        self.n_params = int(self.lib.gb_lstm_param_count(C.byref(self.net)))
        if self.n_params == 0:
            _cabi.check(-2)
        self.param_stride = int(self.lib.gb_lstm_param_stride(C.byref(self.net)))

    def pack_params(self, weights_per_slot):
        """([(kernel [in,4u], recurrent [u,4u], bias [4u]) per layer], (Wd, bd)) per slot -> device [n_slots, stride]."""
        torch = _torch()
        host = np.zeros((len(weights_per_slot), self.param_stride), dtype=np.float32)
        for s, (layers, (Wd, bd)) in enumerate(weights_per_slot):
            flat = []
            for K, U, b in layers:
                flat += [np.asarray(K, np.float32).ravel(), np.asarray(U, np.float32).ravel(), np.asarray(b, np.float32).ravel()]
            flat += [np.asarray(Wd, np.float32).ravel(), np.asarray(bd, np.float32).ravel()]
            vec = np.concatenate(flat)
            if vec.size != self.n_params:
                raise ValueError(f"LSTM weights hold {vec.size} values, architecture needs {self.n_params}")
            host[s, : vec.size] = vec
        return torch.from_numpy(host).to(self.device)

    def initial_params(self, n_slots: int, generator, draw_bytes: int = 256 << 20):
        """
        Fresh networks on the device with Keras' LSTM initialisers, as ``KerasBaseEstimator._initial_weights`` draws them: kernels
        glorot-uniform, recurrent kernels orthogonal (gb_orthonormal_rows on standard-normal draws, ``draw_bytes`` of them at a
        time), biases zero except a forget-gate bias of 1.  Returns [n_slots, param_stride] float32.
        """
        torch = _torch()
        params = torch.zeros((int(n_slots), self.param_stride), dtype=torch.float32, device=self.device)
        ofs, i = 0, self.n_features
        for u in self.units:
            lim = math.sqrt(6.0 / (i + 4 * u))
            params[:, ofs:ofs + i * 4 * u].uniform_(-lim, lim, generator=generator)
            ofs += i * 4 * u
            block = max(1, int(draw_bytes) // (u * 4 * u * 8))
            for s0 in range(0, int(n_slots), block):
                n = min(block, int(n_slots) - s0)
                g = torch.randn((n, u, 4 * u), dtype=torch.float64, device=self.device, generator=generator)
                orthonormal_rows(g, params, s0 * self.param_stride + ofs, self.param_stride)
            ofs += u * 4 * u
            params[:, ofs + u:ofs + 2 * u] = 1.0  # gate order i, f, c, o: unit_forget_bias
            ofs += 4 * u
            i = u
        lim = math.sqrt(6.0 / (i + self.n_out))
        params[:, ofs:ofs + i * self.n_out].uniform_(-lim, lim, generator=generator)
        return params

    def unpack_params(self, params):
        """device [n_slots, stride] -> per slot ([(kernel, recurrent, bias) per layer], (Wd, bd)) as host arrays."""
        host = params.detach().cpu().numpy()
        out = []
        for vec in host:
            layers, ofs, i = [], 0, self.n_features
            for u in self.units:
                K = vec[ofs:ofs + i * 4 * u].reshape(i, 4 * u).copy(); ofs += i * 4 * u
                U = vec[ofs:ofs + u * 4 * u].reshape(u, 4 * u).copy(); ofs += u * 4 * u
                b = vec[ofs:ofs + 4 * u].copy(); ofs += 4 * u
                layers.append((K, U, b))
                i = u
            Wd = vec[ofs:ofs + i * self.n_out].reshape(i, self.n_out).copy(); ofs += i * self.n_out
            out.append((layers, (Wd, vec[ofs:ofs + self.n_out].copy())))
        return out

    FP32_MAX_BATCH = 32   # largest batch of the fp32 fit family (gb_lstm_fit_loss)
    TC_MAX_BATCH = 256    # largest batch of the tensor-core fit family (gb_lstm_fit_tc)

    def fit_workspace_bytes(self, n_jobs: int) -> int:
        """Device scratch one ``fit`` launch of ``n_jobs`` jobs allocates (gb_lstm_fit_workspace_bytes)."""
        return int(self.lib.gb_lstm_fit_workspace_bytes(C.byref(self.net), int(n_jobs)))

    def fit_tc_workspace_bytes(self, n_jobs: int, batch_size: int) -> int:
        """Device scratch one ``fit_tc`` launch of ``n_jobs`` jobs at ``batch_size`` allocates (gb_lstm_fit_tc_workspace_bytes)."""
        return int(self.lib.gb_lstm_fit_tc_workspace_bytes(C.byref(self.net), int(n_jobs), int(batch_size)))

    def fit_for_batch(self, batch_size: int):
        """The fit family for ``batch_size``: ``fit`` (fp32) up to FP32_MAX_BATCH windows, ``fit_tc`` above."""
        return self.fit if int(batch_size) <= self.FP32_MAX_BATCH else self.fit_tc

    def fit_workspace_bytes_for_batch(self, n_jobs: int, batch_size: int) -> int:
        """Workspace of the launch ``fit_for_batch(batch_size)`` makes for ``n_jobs`` jobs."""
        if int(batch_size) <= self.FP32_MAX_BATCH:
            return self.fit_workspace_bytes(n_jobs)
        return self.fit_tc_workspace_bytes(n_jobs, batch_size)

    def fit(self, params, jobs_dev, n_jobs, max_windows, x, y, epochs: int = 1, batch_size: int = 32, lookahead: int = 0,
            primer: bool = True, adam: Optional[Dict[str, float]] = None, state=None, loss: str = "mse", optimizer=None):
        """
        Trains every job's slot in place by back-propagation through time (``jobs`` count windows; target of window j is
        y[x_row + j + lookback - 1 + lookahead]).  Returns (loss [n_jobs, epochs], accuracy, (m, v, t)).  ``loss``: canonical
        Keras loss name (``_cabi.LOSS_CODES``), for the primer step too (gb_lstm_fit_loss).  ``optimizer``: None (Adam from
        ``adam``) or the (name, record) pair of ``factories.specs.resolve_optimizer`` (gb_lstm_fit_opt); m and v are its state slots.
        """
        hist, acc, _, _, st = self._fit_launch(False, params, jobs_dev, n_jobs, max_windows, x, y, epochs, batch_size, lookahead, primer,
                                               adam, state, loss, optimizer)
        return hist, acc, st

    def fit_tc(self, params, jobs_dev, n_jobs, max_windows, x, y, epochs: int = 1, batch_size: int = 32, lookahead: int = 0,
               primer: bool = True, adam: Optional[Dict[str, float]] = None, state=None, loss: str = "mse", optimizer=None):
        """
        ``fit`` on the tensor-core family (gb_lstm_fit_tc): the same training for batches of 1 .. TC_MAX_BATCH windows, the
        GEMMs of each step on wgmma in split TF32.  Same arguments, return value and (m, v, t) state, which may be carried
        between calls of either family.  A batch above TC_MAX_BATCH raises ValueError before anything is launched.
        """
        if not 1 <= int(batch_size) <= self.TC_MAX_BATCH:
            raise ValueError(f"batch_size={int(batch_size)}: the LSTM fit handles batches of 1 to {self.TC_MAX_BATCH} windows")
        hist, acc, _, _, st = self._fit_launch(True, params, jobs_dev, n_jobs, max_windows, x, y, epochs, batch_size, lookahead, primer,
                                               adam, state, loss, optimizer)
        return hist, acc, st

    def fit_stop(self, params, jobs_dev, n_jobs, max_windows, x, y, stop, epochs: int = 1, batch_size: int = 32, lookahead: int = 0,
                 primer: bool = True, adam: Optional[Dict[str, float]] = None, state=None, loss: str = "mse", optimizer=None):
        """
        ``fit_for_batch(batch_size)`` with Keras' EarlyStopping inside the launch (gb_lstm_fit_stop, or gb_lstm_fit_tc_stop above
        FP32_MAX_BATCH windows): every job applies its rule at the end of each epoch, a job that stops does no further work, and
        with ``restore_best_weights`` its slot of ``params`` ends with the weights of its best epoch.  ``stop``: ``make_stop``
        records, one per job (a host array).  Returns (loss, accuracy, epochs_run, best_epoch, (m, v, t)): epochs_run / best_epoch
        are int32 [n_jobs] (best_epoch -1 when no epoch improved and no snapshot was taken), and every history entry past a job's
        epochs_run is NaN.  The other arguments and (m, v, t) are ``fit``'s.
        """
        if not 1 <= int(batch_size) <= self.TC_MAX_BATCH:
            raise ValueError(f"batch_size={int(batch_size)}: the LSTM fit handles batches of 1 to {self.TC_MAX_BATCH} windows")
        stop = np.ascontiguousarray(stop, dtype=_cabi.STOP_DTYPE)
        if stop.shape != (int(n_jobs),):
            raise ValueError(f"stop holds {stop.shape} records for {int(n_jobs)} jobs")
        return self._fit_launch(int(batch_size) > self.FP32_MAX_BATCH, params, jobs_dev, n_jobs, max_windows, x, y, epochs, batch_size,
                                lookahead, primer, adam, state, loss, optimizer, stop=stop)

    def _fit_launch(self, tc, params, jobs_dev, n_jobs, max_windows, x, y, epochs, batch_size, lookahead, primer, adam, state, loss,
                    optimizer=None, stop=None):
        """
        The one launch of ``fit`` / ``fit_tc`` / ``fit_stop``: the family's _stop entry (gb_lstm_fit_tc_stop if ``tc``, else
        gb_lstm_fit_stop), with NULL for a missing optimizer and, without ``stop`` records, for the rule and its outputs.  Returns
        (loss, accuracy, epochs_run, best_epoch, (m, v, t)); epochs_run / best_epoch None without ``stop``.
        """
        torch = _torch()
        entry = self.lib.gb_lstm_fit_tc_stop if tc else self.lib.gb_lstm_fit_stop
        ws_bytes = self.fit_tc_workspace_bytes(n_jobs, batch_size) if tc else self.fit_workspace_bytes(n_jobs)
        best = epochs_run = best_epoch = None
        if stop is not None:
            ws_bytes += int(self.lib.gb_lstm_fit_stop_state_bytes(int(n_jobs)))
            epochs_run = torch.zeros((int(n_jobs),), dtype=torch.int32, device=self.device)
            best_epoch = torch.full((int(n_jobs),), -1, dtype=torch.int32, device=self.device)
            best = torch.empty_like(params)  # snapshot area
        opt = None if optimizer is None else _cabi.make_optimizer(*optimizer)
        adam = adam or {}
        hp = _cabi.GbLstmFitHParams()
        hp.epochs, hp.batch_size, hp.lookahead, hp.primer = int(epochs), int(batch_size), int(lookahead), int(bool(primer))
        hp.lr, hp.beta1 = float(adam.get("lr", 1e-3)), float(adam.get("beta1", 0.9))
        hp.beta2, hp.eps = float(adam.get("beta2", 0.999)), float(adam.get("eps", 1e-7))
        if state is None:
            m = torch.zeros_like(params)
            v = torch.zeros_like(params)
            t = torch.zeros((params.shape[0],), dtype=torch.int32, device=self.device)
        else:
            m, v, t = state
        ws = torch.empty((ws_bytes + 3) // 4, dtype=torch.float32, device=self.device)
        # a primer-only fit (epochs = 0) writes no history, but the kernel takes the outputs as non-NULL pointers and a tensor with
        # no elements has none: the buffers keep one column and the caller gets the empty slice
        fill = 0.0 if stop is None else float("nan")  # with a stop rule, the entries past a job's epochs_run stay NaN
        hist = torch.full((n_jobs, max(epochs, 1)), fill, dtype=torch.float32, device=self.device)
        acc = torch.full((n_jobs, max(epochs, 1)), fill, dtype=torch.float32, device=self.device)
        p = _cabi.ptr
        _cabi.check(entry(C.byref(self.net), p(params), p(m), p(v), p(t), p(jobs_dev), int(n_jobs), int(max_windows), p(x), p(y), C.byref(hp),
                          p(ws), p(hist), p(acc), _cabi.loss_code(loss), None if opt is None else C.byref(opt),
                          None if stop is None else stop.ctypes.data_as(C.c_void_p), p(best), p(epochs_run), p(best_epoch), _stream_ptr()))
        return hist[:, :epochs], acc[:, :epochs], epochs_run, best_epoch, (m, v, t)

    @property
    def tc_supported(self) -> bool:
        return self.lib.gb_lstm_tc_supported(C.byref(self.net)) == 0

    TILE = 128  # windows per tile of the tensor-core inference kernels

    @classmethod
    def tile_base(cls, n_windows) -> np.ndarray:
        """int32 [n_jobs + 1] prefix sums of ceil(n_windows_j / 128): the ragged tile layout of ``infer(tile_base=)``."""
        tiles = (np.asarray(n_windows, dtype=np.int64) + cls.TILE - 1) // cls.TILE
        return np.concatenate([[0], np.cumsum(tiles)]).astype(np.int32)

    def tc_workspace_bytes(self, n_slots: int, n_jobs: int, max_windows: int, n_tiles: Optional[int] = None) -> int:
        """Device scratch of one tensor-core ``infer`` launch: every job max_windows' tiles, or with ``n_tiles`` the ragged layout (0: refused)."""
        if n_tiles is None:
            return int(self.lib.gb_lstm_tc_workspace_bytes(C.byref(self.net), int(n_slots), int(n_jobs), int(max_windows), 1))
        return int(self.lib.gb_lstm_tc_ragged_workspace_bytes(C.byref(self.net), int(n_slots), int(n_jobs), int(n_tiles), int(max_windows)))

    def infer(self, params, jobs_dev, n_jobs, max_windows, x, out_rows, variant: int = 0, tile_base=None, n_tiles: Optional[int] = None):
        """
        out[j] = net(x[j : j + lookback]) for every job's windows (jobs' n_rows counts windows).
        variant 0 = tensor-core (wgmma) kernel when the layer widths allow it, 1 = fp32 CUDA-core kernel, 2 = tensor-core kernel (error if unsupported).
        ``tile_base`` (int32 device tensor of ``tile_base(n_rows)``) with ``n_tiles`` = its last entry: the ragged tile layout
        (gb_lstm_infer_tc_ragged), where a batch costs its jobs' own windows; tensor-core kernel only, the same bits per window.
        """
        torch = _torch()
        out = torch.empty((int(out_rows), self.n_out), dtype=torch.float32, device=self.device)
        p = _cabi.ptr
        if tile_base is not None:
            if n_tiles is None or variant == 1:
                raise ValueError("a ragged tile layout takes n_tiles and runs on the tensor-core kernel only")
            _cabi.check(self.lib.gb_lstm_tc_supported(C.byref(self.net)))
            ws_bytes = self.tc_workspace_bytes(params.shape[0], n_jobs, max_windows, n_tiles)
            ws = torch.empty((ws_bytes + 255,), dtype=torch.uint8, device=self.device)
            _cabi.check(self.lib.gb_lstm_infer_tc_ragged(C.byref(self.net), p(params), int(params.shape[0]), p(jobs_dev), int(n_jobs), p(tile_base),
                                                         int(n_tiles), int(max_windows), p(x), int(x.shape[0]), p(out), p(ws), _stream_ptr()))
            return out
        if variant == 2 or (variant == 0 and self.tc_supported):
            ws_bytes = int(self.lib.gb_lstm_tc_workspace_bytes(C.byref(self.net), int(params.shape[0]), int(n_jobs), int(max_windows), int(x.shape[0])))
            if ws_bytes == 0:
                _cabi.check(self.lib.gb_lstm_tc_supported(C.byref(self.net)))
            ws = torch.empty((ws_bytes + 255,), dtype=torch.uint8, device=self.device)
            _cabi.check(self.lib.gb_lstm_infer_tc(C.byref(self.net), p(params), int(params.shape[0]), p(jobs_dev), int(n_jobs), int(max_windows), p(x),
                                                  int(x.shape[0]), p(out), p(ws), _stream_ptr()))
            return out
        _cabi.check(self.lib.gb_lstm_infer(C.byref(self.net), p(params), p(jobs_dev), int(n_jobs), int(max_windows), p(x), p(out), None, _stream_ptr()))
        return out


_ff_engines: Dict[tuple, FFEngine] = {}
_lstm_engines: Dict[tuple, LSTMEngine] = {}
_engine_lock = threading.Lock()  # gordo.server calls into shared models from several gunicorn threads


def ff_engine_for(spec, device=None) -> FFEngine:
    dev = cuda_device(device)
    key = (spec.key(), tuple(spec.l1), dev.index)
    with _engine_lock:
        if key not in _ff_engines:
            _ff_engines[key] = FFEngine(spec.dims, spec.acts, spec.l1, dev)
        return _ff_engines[key]


def lstm_engine_for(spec, device=None) -> LSTMEngine:
    dev = cuda_device(device)
    key = (spec.key(), dev.index)
    with _engine_lock:
        if key not in _lstm_engines:
            _lstm_engines[key] = LSTMEngine(spec.n_features, spec.lstm_units, spec.acts, spec.n_features_out, spec.out_func, spec.lookback_window, dev)
        return _lstm_engines[key]


def to_device_f32(a, device):
    """Host array/frame -> contiguous float32 device tensor (the reference casts to floatx=float32 too [3P scikeras])."""
    torch = _torch()
    arr = np.ascontiguousarray(np.asarray(getattr(a, "values", a), dtype=np.float32))
    if arr.ndim == 1:
        arr = arr.reshape(-1, 1)
    return torch.from_numpy(arr).to(device)
