"""
TEST INFRASTRUCTURE ONLY -- CPU restatement (NumPy) of the neural-network half of the
gordo autoencoder hot path.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s cpu_baseline / ``--impl reference`` legs may import this module; the
product package (``gordo_components_b200``) never does and has no CPU fallback.

PARITY STATUS: **parity unpinned at the TF/Keras boundary.**  The arithmetic restated
here lives in third-party packages that are not vendored in the reference project and
are not installable in this image: tensorflow==2.16.2, keras==3.3.3, scikeras==0.13.0
(reference ``requirements/full_requirements.txt:449,201,406``).  No reference test pins
a numerical output of Keras ``fit``/``predict`` (SURVEY.md section 8c), so this file
restates the published Keras algorithms and is anchored on the reference's call sites:

* topology          gordo/machine/model/factories/feedforward_autoencoder.py:65-104
                    gordo/machine/model/factories/lstm_autoencoder.py:72-103
* layer widths      gordo/machine/model/factories/utils.py:7-41  (pinned exactly by
                    tests/gordo/machine/model/test_factories_utils.py:8-24 -> tests/test_oracle_golden.py)
* fit/predict flow  gordo/machine/model/models.py:243-300, 557-660
* windowing         gordo/machine/model/models.py:713-793 (pinned exactly by
                    tests/gordo/machine/model/test_model.py:239-321)

Everything that *is* pinned by the reference (dims table, timeseries batches, anomaly
formulas via the reference's own diff.py) is checked in tests/test_oracle_golden.py.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

# --------------------------------------------------------------------------------------
# architecture
# --------------------------------------------------------------------------------------


def hourglass_calc_dims(compression_factor: float, encoding_layers: int, n_features: int) -> Tuple[int, ...]:
    """Layer widths of the hourglass encoder (reference factories/utils.py:7-41)."""
    if not (0 <= compression_factor <= 1):
        raise ValueError("compression_factor must be 0 <= compression_factor <= 1")
    if encoding_layers < 1:
        raise ValueError("encoding_layers must be >= 1")
    narrow = max(min(math.ceil(compression_factor * n_features), n_features), 1)
    slope = (n_features - narrow) / encoding_layers
    # Python's round() is round-half-to-even; the reference relies on it (dims 10 -> (8, 7, 5))
    return tuple(round(n_features - i * slope) for i in range(1, encoding_layers + 1))


@dataclass
class FFSpec:
    """A Dense stack: dims[0] inputs, dims[l+1] units of layer l, activation + L1 activity coefficient per layer."""

    dims: List[int]
    acts: List[str]
    l1: List[float] = field(default_factory=list)

    def __post_init__(self):
        if not self.l1:
            self.l1 = [0.0] * (len(self.dims) - 1)
        assert len(self.acts) == len(self.dims) - 1 == len(self.l1)

    @property
    def n_layers(self) -> int:
        return len(self.dims) - 1

    @property
    def n_params(self) -> int:
        return sum(i * o + o for i, o in zip(self.dims[:-1], self.dims[1:]))


def ff_model_spec(
    n_features: int,
    n_features_out: Optional[int] = None,
    encoding_dim: Sequence[int] = (256, 128, 64),
    encoding_func: Sequence[str] = ("tanh", "tanh", "tanh"),
    decoding_dim: Sequence[int] = (64, 128, 256),
    decoding_func: Sequence[str] = ("tanh", "tanh", "tanh"),
    out_func: str = "linear",
) -> FFSpec:
    """feedforward_model (feedforward_autoencoder.py:15-104): encoder layers i>=1 carry l1(10e-5) activity reg."""
    n_features_out = n_features_out or n_features
    if len(encoding_dim) != len(encoding_func) or len(decoding_dim) != len(decoding_func):
        raise ValueError("dims and funcs must have equal length")
    dims = [n_features, *encoding_dim, *decoding_dim, n_features_out]
    acts = [*encoding_func, *decoding_func, out_func]
    l1 = [0.0 if i == 0 else 10e-5 for i in range(len(encoding_dim))] + [0.0] * (len(decoding_dim) + 1)
    return FFSpec(list(map(int, dims)), list(acts), l1)


def ff_symmetric_spec(n_features, n_features_out=None, dims=(256, 128, 64), funcs=("tanh", "tanh", "tanh"), out_func="linear") -> FFSpec:
    """feedforward_symmetric (feedforward_autoencoder.py:107-157)."""
    if len(dims) == 0:
        raise ValueError("Parameter dims must have len > 0")
    return ff_model_spec(n_features, n_features_out, tuple(dims), tuple(funcs), tuple(dims)[::-1], tuple(funcs)[::-1], out_func)


def ff_hourglass_spec(n_features, n_features_out=None, encoding_layers=3, compression_factor=0.5, func="tanh") -> FFSpec:
    """feedforward_hourglass (feedforward_autoencoder.py:160-251)."""
    dims = hourglass_calc_dims(compression_factor, encoding_layers, n_features)
    return ff_symmetric_spec(n_features, n_features_out, dims, tuple([func] * len(dims)))


# --------------------------------------------------------------------------------------
# Keras initialisers [3P keras 3.3.3]
# --------------------------------------------------------------------------------------


def glorot_uniform(rng: np.random.Generator, fan_in: int, fan_out: int) -> np.ndarray:
    limit = math.sqrt(6.0 / (fan_in + fan_out))
    return rng.uniform(-limit, limit, size=(fan_in, fan_out)).astype(np.float32)


def orthogonal(rng: np.random.Generator, rows: int, cols: int) -> np.ndarray:
    a = rng.standard_normal((max(rows, cols), min(rows, cols)))
    q, r = np.linalg.qr(a)
    q = q * np.sign(np.diag(r))
    if rows < cols:
        q = q.T
    return q[:rows, :cols].astype(np.float32)


def init_ff_weights(spec: FFSpec, rng: np.random.Generator) -> List[Tuple[np.ndarray, np.ndarray]]:
    """Dense: kernel [in, out] glorot_uniform, bias zeros."""
    return [(glorot_uniform(rng, i, o), np.zeros(o, np.float32)) for i, o in zip(spec.dims[:-1], spec.dims[1:])]


# --------------------------------------------------------------------------------------
# activations
# --------------------------------------------------------------------------------------


def _act(name: str, z: np.ndarray) -> np.ndarray:
    if name in ("linear", None):
        return z
    if name == "tanh":
        return np.tanh(z)
    if name == "relu":
        return np.maximum(z, 0)
    if name == "sigmoid":
        return 1.0 / (1.0 + np.exp(-z))
    raise ValueError(f"oracle: unsupported activation {name!r}")


def _act_grad_from_output(name: str, a: np.ndarray) -> np.ndarray:
    if name in ("linear", None):
        return np.ones_like(a)
    if name == "tanh":
        return 1.0 - a * a
    if name == "relu":
        return (a > 0).astype(a.dtype)
    if name == "sigmoid":
        return a * (1.0 - a)
    raise ValueError(name)


# --------------------------------------------------------------------------------------
# Dense stack forward / fit  (Keras Dense: act(x @ kernel + bias))
# --------------------------------------------------------------------------------------


def ff_forward(spec: FFSpec, weights, X: np.ndarray, dtype=np.float32, return_all=False):
    a = np.asarray(X, dtype=dtype)
    acts = [a]
    for (W, b), name in zip(weights, spec.acts):
        a = _act(name, a @ W.astype(dtype) + b.astype(dtype)).astype(dtype)
        acts.append(a)
    return acts if return_all else a


def ff_predict(spec: FFSpec, weights, X: np.ndarray, batch_size: int = 32, dtype=np.float32) -> np.ndarray:
    """Model.predict control flow (models.py:289-300): Keras default batch_size=32, batches concatenated."""
    X = np.asarray(X, dtype=dtype)
    out = np.empty((len(X), spec.dims[-1]), dtype=dtype)
    for s in range(0, len(X), batch_size):
        out[s : s + batch_size] = ff_forward(spec, weights, X[s : s + batch_size], dtype)
    return out


@dataclass
class AdamState:
    m: List[Tuple[np.ndarray, np.ndarray]]
    v: List[Tuple[np.ndarray, np.ndarray]]
    t: int = 0


def adam_init(weights) -> AdamState:
    z = lambda: [(np.zeros_like(W), np.zeros_like(b)) for W, b in weights]
    return AdamState(z(), z(), 0)


def ff_loss_and_grads(spec: FFSpec, weights, xb, yb, dtype=np.float32, l1_div_batch=False):
    """
    loss = mean((yhat - y)^2 over all batch elements) + sum_l l1_l * sum|a_l|   [3P keras]
    Returns (loss, mse, grads, yhat).
    """
    acts = ff_forward(spec, weights, xb, dtype, return_all=True)
    yhat = acts[-1]
    B = xb.shape[0]
    diff = yhat - yb.astype(dtype)
    mse = dtype(np.mean(diff.astype(dtype) ** 2))
    reg = dtype(0)
    for l in range(spec.n_layers):
        if spec.l1[l] != 0.0:
            r = dtype(spec.l1[l]) * np.sum(np.abs(acts[l + 1]), dtype=dtype)
            reg = reg + (r / dtype(B) if l1_div_batch else r)
    delta = (dtype(2.0) / dtype(diff.size)) * diff  # dL/dyhat
    grads = [None] * spec.n_layers
    for l in range(spec.n_layers - 1, -1, -1):
        a_out = acts[l + 1]
        g = delta
        if spec.l1[l] != 0.0:
            c = dtype(spec.l1[l]) / (dtype(B) if l1_div_batch else dtype(1))
            g = g + c * np.sign(a_out)
        dz = (g * _act_grad_from_output(spec.acts[l], a_out)).astype(dtype)
        grads[l] = ((acts[l].T @ dz).astype(dtype), dz.sum(axis=0).astype(dtype))
        if l > 0:
            delta = (dz @ weights[l][0].astype(dtype).T).astype(dtype)
    return dtype(mse + reg), mse, grads, yhat


def adam_step(weights, grads, st: AdamState, lr=1e-3, b1=0.9, b2=0.999, eps=1e-7, dtype=np.float32):
    """Keras 3 Adam.update_step [3P]: alpha = lr*sqrt(1-b2^t)/(1-b1^t); m += (g-m)(1-b1); v += (g^2-v)(1-b2); w -= alpha*m/(sqrt(v)+eps)."""
    st.t += 1
    t = st.t
    alpha = dtype(lr * math.sqrt(1.0 - b2**t) / (1.0 - b1**t))
    out = []
    for l, ((W, b), (gW, gb)) in enumerate(zip(weights, grads)):
        new = []
        for k, (p, g) in enumerate(((W, gW), (b, gb))):
            m = st.m[l][k]
            v = st.v[l][k]
            m += (g - m) * dtype(1 - b1)
            v += (g * g - v) * dtype(1 - b2)
            new.append((p - alpha * m / (np.sqrt(v) + dtype(eps))).astype(dtype))
        out.append((new[0], new[1]))
    return out


def categorical_accuracy(y_true, y_pred) -> float:
    """metrics=["accuracy"] on 2-D float targets resolves to categorical accuracy (argmax match) [3P]; width 1 -> binary accuracy."""
    if y_true.shape[-1] == 1:
        return float(np.mean((y_pred > 0.5).astype(np.float32) == y_true))
    return float(np.mean(np.argmax(y_true, axis=-1) == np.argmax(y_pred, axis=-1)))


def ff_fit(
    spec: FFSpec,
    weights,
    X: np.ndarray,
    y: np.ndarray,
    epochs: int = 1,
    batch_size: int = 32,
    shuffle: bool = True,
    perms: Optional[Sequence[np.ndarray]] = None,
    rng: Optional[np.random.Generator] = None,
    validation_split: float = 0.0,
    lr=1e-3,
    b1=0.9,
    b2=0.999,
    eps=1e-7,
    dtype=np.float32,
    l1_div_batch=False,
    state: Optional[AdamState] = None,
):
    """
    Keras Model.fit on arrays [3P]: validation_split holds out the *tail* before shuffling;
    every epoch visits a fresh permutation (``perms[e]`` if injected) in batches of
    ``batch_size`` keeping the last partial batch; history loss = sample-weighted mean of
    the per-batch total loss.  Returns (weights, history, adam_state).
    """
    X = np.asarray(X, dtype=dtype)
    y = np.asarray(y, dtype=dtype)
    if y.ndim == 1:
        y = y.reshape(-1, 1)
    n_val = 0
    if validation_split and 0.0 < validation_split < 1.0:
        split_at = int(math.floor(len(X) * (1.0 - validation_split)))
        Xv, yv = X[split_at:], y[split_at:]
        X, y = X[:split_at], y[:split_at]
        n_val = len(Xv)
    n = len(X)
    st = state or adam_init(weights)
    weights = [(W.astype(dtype).copy(), b.astype(dtype).copy()) for W, b in weights]
    hist: Dict[str, list] = {"loss": [], "accuracy": []}
    if n_val:
        hist["val_loss"], hist["val_accuracy"] = [], []
    for e in range(epochs):
        if perms is not None:
            order = np.asarray(perms[e])
        elif shuffle:
            order = (rng or np.random.default_rng(e)).permutation(n)
        else:
            order = np.arange(n)
        loss_sum = 0.0
        hit_sum = 0.0
        for s in range(0, n, batch_size):
            idx = order[s : s + batch_size]
            xb, yb = X[idx], y[idx]
            loss, _mse, grads, yhat = ff_loss_and_grads(spec, weights, xb, yb, dtype, l1_div_batch)
            loss_sum += float(loss) * len(idx)
            hit_sum += categorical_accuracy(yb, yhat) * len(idx)
            weights = adam_step(weights, grads, st, lr, b1, b2, eps, dtype)
        hist["loss"].append(loss_sum / n)
        hist["accuracy"].append(hit_sum / n)
        if n_val:
            lv, _, _, yh = ff_loss_and_grads(spec, weights, Xv, yv, dtype, l1_div_batch)
            hist["val_loss"].append(float(lv))
            hist["val_accuracy"].append(categorical_accuracy(yv, yh))
    hist["params"] = {"verbose": 0, "epochs": epochs, "steps": int(math.ceil(n / batch_size))}
    return weights, hist, st


# --------------------------------------------------------------------------------------
# LSTM stack  (Keras LSTM: gates i,f,c,o packed in kernel [in,4u], recurrent_kernel [u,4u], bias [4u])
# --------------------------------------------------------------------------------------


@dataclass
class LSTMSpec:
    n_features: int
    units: List[int]  # all LSTM layers, encoder then decoder
    acts: List[str]
    n_features_out: int
    out_func: str = "linear"
    lookback_window: int = 1

    @property
    def n_params(self) -> int:
        p, i = 0, self.n_features
        for u in self.units:
            p += 4 * u * (i + u + 1)
            i = u
        return p + i * self.n_features_out + self.n_features_out

    @property
    def flop_per_window(self) -> int:
        mac, i = 0, self.n_features
        for u in self.units:
            mac += 4 * u * (i + u)
            i = u
        return 2 * mac * self.lookback_window + 2 * i * self.n_features_out


def lstm_model_spec(n_features, n_features_out=None, lookback_window=1, encoding_dim=(256, 128, 64), encoding_func=("tanh",) * 3,
                    decoding_dim=(64, 128, 256), decoding_func=("tanh",) * 3, out_func="linear") -> LSTMSpec:
    """lstm_model (lstm_autoencoder.py:15-103): all LSTMs return sequences except the last, then Dense."""
    if len(encoding_dim) != len(encoding_func) or len(decoding_dim) != len(decoding_func):
        raise ValueError("dims and funcs must have equal length")
    return LSTMSpec(int(n_features), [*map(int, encoding_dim), *map(int, decoding_dim)], [*encoding_func, *decoding_func],
                    int(n_features_out or n_features), out_func, int(lookback_window))


def lstm_symmetric_spec(n_features, n_features_out=None, lookback_window=1, dims=(256, 128, 64), funcs=("tanh",) * 3, out_func="linear") -> LSTMSpec:
    """lstm_symmetric (lstm_autoencoder.py:106-174)."""
    if len(dims) == 0:
        raise ValueError("Parameter dims must have len > 0")
    return lstm_model_spec(n_features, n_features_out, lookback_window, tuple(dims), tuple(funcs), tuple(dims)[::-1], tuple(funcs)[::-1], out_func)


def lstm_hourglass_spec(n_features, n_features_out=None, lookback_window=1, encoding_layers=3, compression_factor=0.5, func="tanh", out_func="linear") -> LSTMSpec:
    """lstm_hourglass (lstm_autoencoder.py:177-263)."""
    dims = hourglass_calc_dims(compression_factor, encoding_layers, n_features)
    return lstm_symmetric_spec(n_features, n_features_out, lookback_window, dims, tuple([func] * len(dims)), out_func)


def init_lstm_weights(spec: LSTMSpec, rng: np.random.Generator):
    """kernel glorot_uniform, recurrent orthogonal, bias zeros with unit forget bias [3P]. Returns ([(K,U,b)...], (Wd,bd))."""
    layers, i = [], spec.n_features
    for u in spec.units:
        K = glorot_uniform(rng, i, 4 * u)
        U = orthogonal(rng, u, 4 * u)
        b = np.zeros(4 * u, np.float32)
        b[u : 2 * u] = 1.0
        layers.append((K, U, b))
        i = u
    return layers, (glorot_uniform(rng, i, spec.n_features_out), np.zeros(spec.n_features_out, np.float32))


def _sigmoid(z):
    return 1.0 / (1.0 + np.exp(-z))


def lstm_forward_windows(spec: LSTMSpec, weights, windows: np.ndarray, dtype=np.float32) -> np.ndarray:
    """windows [B, L, n_features] -> [B, n_features_out]; zero initial state per window."""
    layers, (Wd, bd) = weights
    seq = np.asarray(windows, dtype=dtype)
    B, L, _ = seq.shape
    for li, ((K, U, b), act) in enumerate(zip(layers, spec.acts)):
        u = U.shape[0]
        K, U, b = K.astype(dtype), U.astype(dtype), b.astype(dtype)
        h = np.zeros((B, u), dtype)
        c = np.zeros((B, u), dtype)
        out = np.empty((B, L, u), dtype)
        xk = seq @ K + b  # input projection for all steps
        for t in range(L):
            z = xk[:, t] + h @ U
            i_g = _sigmoid(z[:, :u])
            f_g = _sigmoid(z[:, u : 2 * u])
            c = (f_g * c + i_g * _act(act, z[:, 2 * u : 3 * u])).astype(dtype)
            o_g = _sigmoid(z[:, 3 * u :])
            h = (o_g * _act(act, c)).astype(dtype)
            out[:, t] = h
        seq = out
    last = seq[:, -1]
    return _act(spec.out_func, last @ Wd.astype(dtype) + bd.astype(dtype)).astype(dtype)


# --------------------------------------------------------------------------------------
# windowing  (models.py:713-793 / keras TimeseriesGenerator [3P])
# --------------------------------------------------------------------------------------


def timeseries_windows(n_rows: int, lookback_window: int, lookahead: int):
    """
    Index form of create_keras_timeseriesgenerator: sample j uses rows X[j : j+L] and
    target y[j + L - 1 + lookahead]; there are n_rows - L + 1 - lookahead samples.
    Returns (starts, target_idx).
    """
    if lookahead < 0:
        raise ValueError(f"Value of `lookahead` can not be negative, is {lookahead}")
    count = max(n_rows - lookback_window + 1 - lookahead, 0)
    starts = np.arange(count)
    return starts, starts + lookback_window - 1 + lookahead


def timeseries_batches(X: np.ndarray, y: np.ndarray, batch_size: int, lookback_window: int, lookahead: int):
    """Materialised batches, for checking against the reference's golden batches (test_model.py:239-321)."""
    starts, tgt = timeseries_windows(len(X), lookback_window, lookahead)
    batches = []
    for s in range(0, len(starts), batch_size):
        js = starts[s : s + batch_size]
        bx = np.stack([X[j : j + lookback_window] for j in js]) if len(js) else np.empty((0,))
        by = y[tgt[s : s + batch_size]]
        batches.append((bx, by))
    return batches


def lstm_predict(spec: LSTMSpec, weights, X: np.ndarray, lookahead: int = 0, batch_size: int = 10000, dtype=np.float32) -> np.ndarray:
    """KerasLSTMBaseEstimator.predict (models.py:618-660): generator with batch 10000 over X, y=X."""
    X = np.asarray(X, dtype=dtype)
    if X.ndim == 1:
        X = X.reshape(len(X), 1)
    L = spec.lookback_window
    if L >= X.shape[0]:
        raise ValueError("For KerasLSTMForecast lookback_window must be < size of X")
    starts, _ = timeseries_windows(len(X), L, lookahead)
    outs = []
    for s in range(0, len(starts), batch_size):
        js = starts[s : s + batch_size]
        win = np.lib.stride_tricks.sliding_window_view(X, (L, X.shape[1]))[js, 0]
        outs.append(lstm_forward_windows(spec, weights, win, dtype))
    return np.concatenate(outs, axis=0)


# --------------------------------------------------------------------------------------
# LSTM fit  (KerasLSTMBaseEstimator.fit, models.py:557-616: primer step on one window, then
# Model.fit on the window generator with shuffle=False) -- back-propagation through time [3P keras]
# --------------------------------------------------------------------------------------


def lstm_loss_and_grads(spec: LSTMSpec, weights, windows: np.ndarray, targets: np.ndarray, dtype=np.float32):
    """
    MSE over all batch elements and its gradient for the stacked LSTM + Dense (no activity regulariser in lstm_model,
    lstm_autoencoder.py:72-103).  Returns (loss, grads, yhat); grads mirrors ``weights``: ([(dK, dU, db)...], (dWd, dbd)).
    """
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
            ig[:, t] = _sigmoid(z[:, :u])
            fg[:, t] = _sigmoid(z[:, u : 2 * u])
            gg[:, t] = _act(act, z[:, 2 * u : 3 * u])
            og[:, t] = _sigmoid(z[:, 3 * u :])
            c = (fg[:, t] * c + ig[:, t] * gg[:, t]).astype(dtype)
            h = (og[:, t] * _act(act, c)).astype(dtype)
            cs[:, t], hs[:, t] = c, h
        saved.append((seq, ig, fg, gg, og, cs, hs))
        seq = hs
    last = seq[:, -1]
    yhat = _act(spec.out_func, last @ Wd.astype(dtype) + bd.astype(dtype)).astype(dtype)
    diff = yhat - tg
    loss = dtype(np.mean(diff**2))
    dout = ((dtype(2.0) / dtype(diff.size)) * diff * _act_grad_from_output(spec.out_func, yhat)).astype(dtype)
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
            ac = _act(act, cs[:, t])
            c_prev = cs[:, t - 1] if t > 0 else np.zeros((B, u), dtype)
            h_prev = hs[:, t - 1] if t > 0 else np.zeros((B, u), dtype)
            dc = dh * og[:, t] * _act_grad_from_output(act, ac) + dc_next
            dz = np.concatenate(
                [
                    dc * gg[:, t] * ig[:, t] * (1 - ig[:, t]),
                    dc * c_prev * fg[:, t] * (1 - fg[:, t]),
                    dc * ig[:, t] * _act_grad_from_output(act, gg[:, t]),
                    dh * ac * og[:, t] * (1 - og[:, t]),
                ],
                axis=1,
            ).astype(dtype)
            dK += xs[:, t].T @ dz
            dU += h_prev.T @ dz
            db += dz.sum(axis=0)
            dx_seq[:, t] = dz @ K.T
            dh_next = dz @ U.T
            dc_next = dc * fg[:, t]
        g_layers[li] = (dK.astype(dtype), dU.astype(dtype), db.astype(dtype))
        dh_seq = dx_seq
    return loss, (g_layers, g_dense), yhat


def _lstm_flat(weights):
    layers, dense = weights
    return [a for lay in layers for a in lay] + list(dense)


def _lstm_unflat(flat, n_layers):
    return [tuple(flat[3 * i : 3 * i + 3]) for i in range(n_layers)], tuple(flat[3 * n_layers : 3 * n_layers + 2])


def lstm_fit(spec: LSTMSpec, weights, X: np.ndarray, y: np.ndarray, epochs: int = 1, batch_size: int = 32, lookahead: int = 0,
             lr=1e-3, b1=0.9, b2=0.999, eps=1e-7, dtype=np.float32):
    """
    models.py:557-616.  (1) primer: one Adam step on the single window X[:L] -> y[L-1+lookahead] (``super().fit`` with epochs=1 on
    a batch of one); (2) ``epochs`` passes over the windows IN ORDER (shuffle=False) in batches of ``batch_size``, last partial
    batch kept, the optimizer state carrying on from the primer step.  History = sample-weighted mean loss / accuracy per epoch.
    Returns (weights, history).
    """
    X = np.asarray(X, dtype=dtype)
    y = np.asarray(y, dtype=dtype)
    if X.ndim == 1:
        X = X.reshape(-1, 1)
    if y.ndim == 1:
        y = y.reshape(-1, 1)
    L = spec.lookback_window
    starts, tgt = timeseries_windows(len(X), L, lookahead)
    nl = len(spec.units)
    flat = [np.asarray(a, dtype=dtype).copy() for a in _lstm_flat(weights)]
    m = [np.zeros_like(a) for a in flat]
    v = [np.zeros_like(a) for a in flat]
    t_step = 0

    def step(js):
        nonlocal flat, t_step
        win = np.stack([X[j : j + L] for j in js])
        loss, grads, yhat = lstm_loss_and_grads(spec, _lstm_unflat(flat, nl), win, y[tgt[js]], dtype)
        t_step += 1
        alpha = dtype(lr * math.sqrt(1.0 - b2**t_step) / (1.0 - b1**t_step))
        for k, g in enumerate(_lstm_flat(grads)):
            m[k] += (g - m[k]) * dtype(1 - b1)
            v[k] += (g * g - v[k]) * dtype(1 - b2)
            flat[k] = (flat[k] - alpha * m[k] / (np.sqrt(v[k]) + dtype(eps))).astype(dtype)
        return float(loss), categorical_accuracy(y[tgt[js]], yhat)

    step(np.array([0]))  # primer
    hist: Dict[str, list] = {"loss": [], "accuracy": []}
    n = len(starts)
    for _ in range(epochs):
        ls = hs = 0.0
        for s in range(0, n, batch_size):
            js = starts[s : s + batch_size]
            lo, ac = step(js)
            ls += lo * len(js)
            hs += ac * len(js)
        hist["loss"].append(ls / n)
        hist["accuracy"].append(hs / n)
    hist["params"] = {"verbose": 0, "epochs": epochs, "steps": int(math.ceil(n / batch_size))}
    return _lstm_unflat(flat, nl), hist
