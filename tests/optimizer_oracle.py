"""
TEST INFRASTRUCTURE ONLY -- the Keras optimizers the fit kernels implement, restated in NumPy, and the loss oracle's Dense and LSTM
fit loops (tests/loss_oracle.py) with the optimizer as a parameter: every other piece (forward pass, loss gradients, accuracy,
windowing, primer step) is the loss oracle's own.

[3P keras 3.3.3, keras/src/optimizers/{adam,adamw,rmsprop,adagrad,adadelta,adamax,nadam}.py and base_optimizer.py] restated, not
verified against TensorFlow.  An optimizer is the (name, record) pair of ``factories.specs.resolve_optimizer``.  Per step, on the
summed mini-batch gradient g of each variable: g = clip(g, -clipvalue, clipvalue) when clipvalue is set, then the decoupled weight
decay w -= w * weight_decay * lr, then the rule (include/gordo_b200.h gb_optimizer).  t counts the slot's steps from 1.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import numpy as np

import loss_oracle as lo
from oracle import keras_math as km

OPTIMIZERS = ("adam", "adamw", "rmsprop", "adagrad", "adadelta", "adamax", "nadam")


def resolve(name, **kwargs):
    """(name, record) of ``optimizer=name, optimizer_kwargs=kwargs``, through the package's resolver."""
    from gordo_components_b200.machine.model.factories.specs import resolve_optimizer

    return resolve_optimizer(name, kwargs)


class OptState:
    """The two state slots of every variable (s0 / s1: the kernels' adam_m / adam_v), the step count and Nadam's product."""

    def __init__(self, arrays: Sequence[np.ndarray], dtype):
        self.s0 = [np.zeros_like(a, dtype=dtype) for a in arrays]
        self.s1 = [np.zeros_like(a, dtype=dtype) for a in arrays]
        self.t = 0
        self.pi = dtype(1.0)


def step(optimizer, params: List[np.ndarray], grads: Sequence[np.ndarray], st: OptState, dtype=np.float32,
         decay_after=False) -> List[np.ndarray]:
    """
    One optimizer step of every variable; returns the new variables (st is updated in place).  ``decay_after`` applies the weight
    decay after the rule instead of before it (a deliberately wrong variant for the tests that must tell the two apart).
    """
    name, cfg = optimizer
    d = dtype
    st.t += 1
    t = st.t
    lr, eps = d(cfg["lr"]), d(cfg["eps"])
    wd, clip = cfg.get("weight_decay") or 0.0, cfg.get("clipvalue")
    if name == "nadam":
        b1 = cfg["beta1"]
        u_t = d(b1 * (1.0 - 0.5 * 0.96 ** t))
        u_t1 = d(b1 * (1.0 - 0.5 * 0.96 ** (t + 1)))
        st.pi = d(st.pi * u_t)  # updated before the step's variable updates
    out = []
    for k, (w, g) in enumerate(zip(params, grads)):
        w = np.asarray(w, dtype=d).copy()
        g = np.asarray(g, dtype=d)
        if clip is not None:
            g = np.clip(g, d(-clip), d(clip))
        if wd and not decay_after:
            w = (w - w * d(wd) * lr).astype(d)
        s0, s1 = st.s0[k], st.s1[k]
        if name in ("adam", "adamw"):
            b1, b2 = cfg["beta1"], cfg["beta2"]
            alpha = d(cfg["lr"] * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t))
            s0 += (g - s0) * d(1 - b1)
            s1 += (g * g - s1) * d(1 - b2)
            w = w - (s0 * alpha) / (np.sqrt(s1) + eps)
        elif name == "rmsprop":
            rho = d(cfg["rho"])
            s0[...] = rho * s0 + (d(1) - rho) * (g * g)
            if cfg["centered"]:
                s1[...] = rho * s1 + (d(1) - rho) * g
                den = s0 - s1 * s1 + eps
            else:
                den = s0 + eps
            inc = lr * g / np.sqrt(den)
            if cfg["momentum"] > 0:
                s1[...] = d(cfg["momentum"]) * s1 + inc
                w = w - s1
            else:
                w = w - inc
        elif name == "adagrad":
            acc = (np.full_like(s0, d(cfg["initial_accumulator_value"])) if t == 1 else s0) + g * g
            s0[...] = acc
            w = w - lr * g / np.sqrt(acc + eps)
        elif name == "adadelta":
            rho = d(cfg["rho"])
            s0[...] = rho * s0 + (d(1) - rho) * (g * g)
            dv = -(np.sqrt(s1 + eps) * g / np.sqrt(s0 + eps))
            s1[...] = rho * s1 + (d(1) - rho) * (dv * dv)
            w = w + lr * dv
        elif name == "adamax":
            b1, b2 = cfg["beta1"], cfg["beta2"]
            s0 += (g - s0) * d(1 - b1)
            s1[...] = np.maximum(d(b2) * s1, np.abs(g))
            w = w - (lr * s0) / (d(1.0 - b1 ** t) * (s1 + eps))
        elif name == "nadam":
            b1, b2 = cfg["beta1"], cfg["beta2"]
            s0 += (g - s0) * d(1 - b1)
            s1 += (g * g - s1) * d(1 - b2)
            m_hat = u_t1 * s0 / (d(1) - st.pi * u_t1) + (d(1) - u_t) * g / (d(1) - st.pi)
            v_hat = s1 / d(1.0 - b2 ** t)
            w = w - (m_hat * lr) / (np.sqrt(v_hat) + eps)
        else:
            raise ValueError(name)
        if wd and decay_after:
            w = w - w * d(wd) * lr
        out.append(np.asarray(w, dtype=d))
    return out


def ff_fit(spec, weights, X, y, optimizer, epochs=1, batch_size=32, perms: Optional[Sequence[np.ndarray]] = None, validation_split=0.0,
           val_batch: Optional[int] = None, dtype=np.float32, l1_div_batch=False, loss="mse"):
    """loss_oracle.ff_fit with ``optimizer``.  Returns (weights, history, state) with state.s0 / s1 as [(W, b)] per layer."""
    X = np.asarray(X, dtype=dtype)
    y = np.asarray(y, dtype=dtype)
    n_val = 0
    if validation_split and 0.0 < validation_split < 1.0:
        split_at = int(math.floor(len(X) * (1.0 - validation_split)))
        Xv, yv = X[split_at:], y[split_at:]
        X, y = X[:split_at], y[:split_at]
        n_val = len(Xv)
    n = len(X)
    flat = [a.astype(dtype).copy() for W, b in weights for a in (W, b)]
    st = OptState(flat, dtype)
    hist: Dict[str, list] = {"loss": [], "accuracy": []}
    if n_val:
        hist["val_loss"], hist["val_accuracy"] = [], []

    def pairs(arrs):
        return [(arrs[2 * i], arrs[2 * i + 1]) for i in range(len(arrs) // 2)]

    for e in range(epochs):
        order = np.asarray(perms[e]) if perms is not None else np.arange(n)
        loss_sum = hit_sum = 0.0
        for s in range(0, n, batch_size):
            idx = order[s:s + batch_size]
            lo_, _, grads, yhat = lo.ff_loss_and_grads(spec, pairs(flat), X[idx], y[idx], dtype, l1_div_batch, loss)
            loss_sum += float(lo_) * len(idx)
            hit_sum += km.categorical_accuracy(y[idx], yhat) * len(idx)
            g = [a for gW, gb in grads for a in (gW, gb)]
            flat = step(optimizer, flat, g, st, dtype)
        hist["loss"].append(loss_sum / n)
        hist["accuracy"].append(hit_sum / n)
        if n_val:
            vb = val_batch or batch_size
            ls = hs = 0.0
            for s in range(0, n_val, vb):
                lo_, _, _, yh = lo.ff_loss_and_grads(spec, pairs(flat), Xv[s:s + vb], yv[s:s + vb], dtype, l1_div_batch, loss)
                ls += float(lo_) * len(yh)
                hs += km.categorical_accuracy(yv[s:s + vb], yh) * len(yh)
            hist["val_loss"].append(ls / n_val)
            hist["val_accuracy"].append(hs / n_val)
    st.s0, st.s1 = pairs(st.s0), pairs(st.s1)
    return pairs(flat), hist, st


def lstm_fit(spec, weights, X, y, optimizer, epochs=1, batch_size=32, lookahead=0, dtype=np.float32, loss="mse", primer=True):
    """loss_oracle.lstm_fit with ``optimizer`` (primer step included).  Returns (weights, history, state) with flat state slots."""
    X = np.asarray(X, dtype=dtype)
    y = np.asarray(y, dtype=dtype)
    L = spec.lookback_window
    starts, tgt = km.timeseries_windows(len(X), L, lookahead)
    nl = len(spec.units)
    flat = [np.asarray(a, dtype=dtype).copy() for a in km._lstm_flat(weights)]
    st = OptState(flat, dtype)

    def one(js):
        nonlocal flat
        win = np.stack([X[j:j + L] for j in js])
        lo_, grads, yhat = lo.lstm_loss_and_grads(spec, km._lstm_unflat(flat, nl), win, y[tgt[js]], dtype, loss)
        flat = step(optimizer, flat, km._lstm_flat(grads), st, dtype)
        return float(lo_), km.categorical_accuracy(y[tgt[js]], yhat)

    if primer:
        one(np.array([0]))
    hist: Dict[str, list] = {"loss": [], "accuracy": []}
    n = len(starts)
    for _ in range(epochs):
        ls = hs = 0.0
        for s in range(0, n, batch_size):
            js = starts[s:s + batch_size]
            lo_, ac = one(js)
            ls += lo_ * len(js)
            hs += ac * len(js)
        hist["loss"].append(ls / n)
        hist["accuracy"].append(hs / n)
    return km._lstm_unflat(flat, nl), hist, st
