"""
TEST INFRASTRUCTURE ONLY -- the Keras regression losses the fit kernels train on, restated in NumPy, and the oracle's Dense and
LSTM fit loops (oracle/keras_math.py) with the loss as a parameter.  The loops are those of keras_math with the mean squared
error replaced by ``loss``; every other piece (forward pass, activations, Adam, accuracy, windowing) is keras_math's own.

[3P keras 3.3.3, keras/src/losses/losses.py] restated, not verified against TF.  With e = yhat - y and EPS = 1e-7 (Keras
``backend.epsilon()``), each loss is a per-element f averaged over the batch's elements; its gradient follows TF's: sign(0) = 0
(``abs``), and ``maximum(yhat, EPS)`` passes the gradient to yhat where yhat >= EPS.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import numpy as np

from oracle import keras_math as km

LOSSES = ("mse", "mae", "mape", "msle", "huber", "log_cosh")
EPS = 1e-7


def loss_value(loss: str, yhat, y):
    """Per-element f(yhat, y) in the dtype of the arguments."""
    yhat, y = np.asarray(yhat), np.asarray(y)
    dt = yhat.dtype.type
    e = yhat - y
    eps = dt(EPS)
    if loss == "mse":
        return e * e
    if loss == "mae":
        return np.abs(e)
    if loss == "mape":
        return dt(100) * np.abs(e) / np.maximum(np.abs(y), eps)
    if loss == "msle":
        d = np.log(np.maximum(yhat, eps) + dt(1)) - np.log(np.maximum(y, eps) + dt(1))
        return d * d
    if loss == "huber":
        a = np.abs(e)
        return np.where(a <= dt(1), dt(0.5) * e * e, a - dt(0.5)).astype(dt)
    if loss == "log_cosh":
        return (e + np.logaddexp(dt(0), dt(-2) * e) - dt(math.log(2.0))).astype(dt)
    raise ValueError(loss)


def loss_grad(loss: str, yhat, y):
    """Per-element df/dyhat."""
    yhat, y = np.asarray(yhat), np.asarray(y)
    dt = yhat.dtype.type
    e = yhat - y
    eps = dt(EPS)
    if loss == "mse":
        return dt(2) * e
    if loss == "mae":
        return np.sign(e)
    if loss == "mape":
        return dt(100) * np.sign(e) / np.maximum(np.abs(y), eps)
    if loss == "msle":
        p = np.maximum(yhat, eps) + dt(1)  # = yhat + 1 wherever the gradient passes
        g = dt(2) * (np.log(p) - np.log(np.maximum(y, eps) + dt(1))) / p
        return np.where(yhat >= eps, g, dt(0)).astype(dt)
    if loss == "huber":
        return np.where(np.abs(e) <= dt(1), e, np.sign(e)).astype(dt)
    if loss == "log_cosh":
        return (dt(1) - dt(2) / (dt(1) + np.exp(dt(2) * e))).astype(dt)
    raise ValueError(loss)


def _output_delta(loss, yhat, y, dtype):
    """(batch loss without regularisation, dL/dyhat): mean of f over the batch's elements."""
    if loss == "mse":  # keras_math's arithmetic, so that MSE is its fit to the bit
        diff = yhat - y
        return dtype(np.mean(diff.astype(dtype) ** 2)), (dtype(2.0) / dtype(diff.size)) * diff
    return dtype(np.mean(loss_value(loss, yhat, y))), (dtype(1.0) / dtype(yhat.size)) * loss_grad(loss, yhat, y)


def ff_loss_and_grads(spec, weights, xb, yb, dtype=np.float32, l1_div_batch=False, loss="mse"):
    """keras_math.ff_loss_and_grads on ``loss``: returns (total loss, data loss, grads, yhat)."""
    acts = km.ff_forward(spec, weights, xb, dtype, return_all=True)
    yhat = acts[-1]
    B = xb.shape[0]
    data, delta = _output_delta(loss, yhat, yb.astype(dtype), dtype)
    reg = dtype(0)
    for l in range(spec.n_layers):
        if spec.l1[l] != 0.0:
            r = dtype(spec.l1[l]) * np.sum(np.abs(acts[l + 1]), dtype=dtype)
            reg = reg + (r / dtype(B) if l1_div_batch else r)
    grads = [None] * spec.n_layers
    for l in range(spec.n_layers - 1, -1, -1):
        a_out = acts[l + 1]
        g = delta
        if spec.l1[l] != 0.0:
            c = dtype(spec.l1[l]) / (dtype(B) if l1_div_batch else dtype(1))
            g = g + c * np.sign(a_out)
        dz = (g * km._act_grad_from_output(spec.acts[l], a_out)).astype(dtype)
        grads[l] = ((acts[l].T @ dz).astype(dtype), dz.sum(axis=0).astype(dtype))
        if l > 0:
            delta = (dz @ weights[l][0].astype(dtype).T).astype(dtype)
    return dtype(data + reg), data, grads, yhat


def ff_fit(spec, weights, X, y, epochs=1, batch_size=32, perms: Optional[Sequence[np.ndarray]] = None, validation_split=0.0,
           val_batch: Optional[int] = None, lr=1e-3, b1=0.9, b2=0.999, eps=1e-7, dtype=np.float32, l1_div_batch=False, loss="mse"):
    """
    keras_math.ff_fit on ``loss`` with an injected visiting order.  The held-out tail is evaluated after every epoch in batches
    of ``val_batch`` (default ``batch_size``), sample-weighted like the training history, as Keras' evaluate does.
    Returns (weights, history, adam_state).
    """
    X = np.asarray(X, dtype=dtype)
    y = np.asarray(y, dtype=dtype)
    n_val = 0
    if validation_split and 0.0 < validation_split < 1.0:
        split_at = int(math.floor(len(X) * (1.0 - validation_split)))
        Xv, yv = X[split_at:], y[split_at:]
        X, y = X[:split_at], y[:split_at]
        n_val = len(Xv)
    n = len(X)
    st = km.adam_init(weights)
    weights = [(W.astype(dtype).copy(), b.astype(dtype).copy()) for W, b in weights]
    hist: Dict[str, list] = {"loss": [], "accuracy": []}
    if n_val:
        hist["val_loss"], hist["val_accuracy"] = [], []
    for e in range(epochs):
        order = np.asarray(perms[e]) if perms is not None else np.arange(n)
        loss_sum = hit_sum = 0.0
        for s in range(0, n, batch_size):
            idx = order[s:s + batch_size]
            lo, _, grads, yhat = ff_loss_and_grads(spec, weights, X[idx], y[idx], dtype, l1_div_batch, loss)
            loss_sum += float(lo) * len(idx)
            hit_sum += km.categorical_accuracy(y[idx], yhat) * len(idx)
            weights = km.adam_step(weights, grads, st, lr, b1, b2, eps, dtype)
        hist["loss"].append(loss_sum / n)
        hist["accuracy"].append(hit_sum / n)
        if n_val:
            vb = val_batch or batch_size
            ls = hs = 0.0
            for s in range(0, n_val, vb):
                lo, _, _, yh = ff_loss_and_grads(spec, weights, Xv[s:s + vb], yv[s:s + vb], dtype, l1_div_batch, loss)
                ls += float(lo) * len(yh)
                hs += km.categorical_accuracy(yv[s:s + vb], yh) * len(yh)
            hist["val_loss"].append(ls / n_val)
            hist["val_accuracy"].append(hs / n_val)
    return weights, hist, st


def lstm_loss_and_grads(spec, weights, windows, targets, dtype=np.float32, loss="mse"):
    """keras_math.lstm_loss_and_grads on ``loss``: returns (loss, grads, yhat)."""
    layers, (Wd, bd) = weights
    seq = np.asarray(windows, dtype=dtype)
    tg = np.asarray(targets, dtype=dtype)
    B, L, _ = seq.shape
    saved = []
    for (K, U, b), act in zip(layers, spec.acts):
        u = U.shape[0]
        K, U, b = K.astype(dtype), U.astype(dtype), b.astype(dtype)
        h = np.zeros((B, u), dtype)
        c = np.zeros((B, u), dtype)
        ig, fg, gg, og, cs, hs = (np.empty((B, L, u), dtype) for _ in range(6))
        for t in range(L):
            z = seq[:, t] @ K + b + h @ U
            ig[:, t] = km._sigmoid(z[:, :u])
            fg[:, t] = km._sigmoid(z[:, u:2 * u])
            gg[:, t] = km._act(act, z[:, 2 * u:3 * u])
            og[:, t] = km._sigmoid(z[:, 3 * u:])
            c = (fg[:, t] * c + ig[:, t] * gg[:, t]).astype(dtype)
            h = (og[:, t] * km._act(act, c)).astype(dtype)
            cs[:, t], hs[:, t] = c, h
        saved.append((seq, ig, fg, gg, og, cs, hs))
        seq = hs
    last = seq[:, -1]
    yhat = km._act(spec.out_func, last @ Wd.astype(dtype) + bd.astype(dtype)).astype(dtype)
    value, delta = _output_delta(loss, yhat, tg, dtype)
    dout = (delta * km._act_grad_from_output(spec.out_func, yhat)).astype(dtype)
    g_dense = ((last.T @ dout).astype(dtype), dout.sum(axis=0).astype(dtype))
    dh_seq = np.zeros_like(seq)
    dh_seq[:, -1] = dout @ Wd.astype(dtype).T
    g_layers = [None] * len(layers)
    for li in range(len(layers) - 1, -1, -1):
        K, U, b = (w.astype(dtype) for w in layers[li])
        act = spec.acts[li]
        xs, ig, fg, gg, og, cs, hs = saved[li]
        u = U.shape[0]
        dK, dU, db = np.zeros_like(K), np.zeros_like(U), np.zeros_like(b)
        dx_seq = np.zeros_like(xs)
        dh_next = np.zeros((B, u), dtype)
        dc_next = np.zeros((B, u), dtype)
        for t in range(L - 1, -1, -1):
            dh = dh_seq[:, t] + dh_next
            ac = km._act(act, cs[:, t])
            c_prev = cs[:, t - 1] if t > 0 else np.zeros((B, u), dtype)
            h_prev = hs[:, t - 1] if t > 0 else np.zeros((B, u), dtype)
            dc = dh * og[:, t] * km._act_grad_from_output(act, ac) + dc_next
            dz = np.concatenate([dc * gg[:, t] * ig[:, t] * (1 - ig[:, t]), dc * c_prev * fg[:, t] * (1 - fg[:, t]),
                                 dc * ig[:, t] * km._act_grad_from_output(act, gg[:, t]), dh * ac * og[:, t] * (1 - og[:, t])],
                                axis=1).astype(dtype)
            dK += xs[:, t].T @ dz
            dU += h_prev.T @ dz
            db += dz.sum(axis=0)
            dx_seq[:, t] = dz @ K.T
            dh_next = dz @ U.T
            dc_next = dc * fg[:, t]
        g_layers[li] = (dK.astype(dtype), dU.astype(dtype), db.astype(dtype))
        dh_seq = dx_seq
    return value, (g_layers, g_dense), yhat


def lstm_fit(spec, weights, X, y, epochs=1, batch_size=32, lookahead=0, lr=1e-3, b1=0.9, b2=0.999, eps=1e-7, dtype=np.float32, loss="mse"):
    """keras_math.lstm_fit on ``loss`` (primer step included).  Returns (weights, history, (m, v)) with m / v flat like the weights."""
    X = np.asarray(X, dtype=dtype)
    y = np.asarray(y, dtype=dtype)
    L = spec.lookback_window
    starts, tgt = km.timeseries_windows(len(X), L, lookahead)
    nl = len(spec.units)
    flat = [np.asarray(a, dtype=dtype).copy() for a in km._lstm_flat(weights)]
    m = [np.zeros_like(a) for a in flat]
    v = [np.zeros_like(a) for a in flat]
    t_step = 0

    def step(js):
        nonlocal t_step
        win = np.stack([X[j:j + L] for j in js])
        lo, grads, yhat = lstm_loss_and_grads(spec, km._lstm_unflat(flat, nl), win, y[tgt[js]], dtype, loss)
        t_step += 1
        alpha = dtype(lr * math.sqrt(1.0 - b2**t_step) / (1.0 - b1**t_step))
        for k, g in enumerate(km._lstm_flat(grads)):
            m[k] += (g - m[k]) * dtype(1 - b1)
            v[k] += (g * g - v[k]) * dtype(1 - b2)
            flat[k] = (flat[k] - alpha * m[k] / (np.sqrt(v[k]) + dtype(eps))).astype(dtype)
        return float(lo), km.categorical_accuracy(y[tgt[js]], yhat)

    step(np.array([0]))  # primer
    hist: Dict[str, list] = {"loss": [], "accuracy": []}
    n = len(starts)
    for _ in range(epochs):
        ls = hs = 0.0
        for s in range(0, n, batch_size):
            js = starts[s:s + batch_size]
            lo, ac = step(js)
            ls += lo * len(js)
            hs += ac * len(js)
        hist["loss"].append(ls / n)
        hist["accuracy"].append(hs / n)
    return km._lstm_unflat(flat, nl), hist, (m, v)
