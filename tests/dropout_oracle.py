"""
Dropout in the Dense fit, restated in NumPy: the mask generator of include/gordo_b200.h (gb_dense_dropout) and Keras' fit of a
Dense stack with Dropout layers (keras 3.3.3 layers.Dropout -> tf.nn.dropout, restated) in float64, with those masks.

``rates[l]`` is the rate on the input of Dense layer l (``rates[0]``: input dropout).  In a training mini-batch the input of
layer l becomes ``where(keep, a * s, 0)``, s = float32(1 / (1 - rate)); the next layer and its weight gradient read the dropped
values, the gradient flowing back is ``g * keep * s`` and the batch loss is that of the dropped forward pass.  Held-out batches
run undropped.  Kernel and bias regularizers are the ones of tests/test_gpu_raw_regressor.py.
"""
import numpy as np

import loss_oracle as lo
import optimizer_oracle as oo
from oracle import keras_math as km

M32 = 0xFFFFFFFF
MAX_LAYERS = 16  # GB_MAX_LAYERS


def mix32(h):
    h = np.asarray(h, dtype=np.uint64) & M32
    h ^= h >> np.uint64(16)
    h = (h * np.uint64(0x7FEB352D)) & M32
    h ^= h >> np.uint64(15)
    h = (h * np.uint64(0x846CA68B)) & M32
    h ^= h >> np.uint64(16)
    return h


def job_key(seed: int, slot: int):
    """The key of a job (the keyed shuffle's too): from the fit's 64-bit seed and the job's slot."""
    seed = int(seed) & (2**64 - 1)
    lo_, hi = seed & M32, seed >> 32
    return mix32(np.uint64(lo_) ^ mix32((hi + 0x632BE5AB * (slot + 1)) & M32))


def threshold(rate) -> int:
    """floor(rate * 2^32) of the float32 rate, in double."""
    return int(np.floor(float(np.float32(rate)) * 4294967296.0))


def scale(rate) -> float:
    """The scale of the kept values: float32(1 / (1 - rate)), computed in double."""
    return float(np.float32(1.0 / (1.0 - float(np.float32(rate)))))


def words(seed: int, slot: int, t: int, positions, layer: int, units: int):
    """The 32-bit words u [len(positions), units] of optimizer step t (absolute, 1-based) for the rows at those positions of their
    mini-batch, on the input of ``layer``."""
    kd = mix32(job_key(seed, slot) ^ np.uint64(0x2545F491))
    ks = mix32((kd + np.uint64(t & M32) * np.uint64(0x9E3779B9)) & M32)
    p = np.asarray(positions, dtype=np.uint64)
    kr = mix32((ks + ((p * np.uint64(MAX_LAYERS) + np.uint64(layer)) & M32) * np.uint64(0x85EBCA6B)) & M32)
    k = np.arange(units, dtype=np.uint64)
    return mix32((kr[:, None] + k[None, :] * np.uint64(0x27D4EB2F)) & M32)


def keep_mask(seed, slot, t, n_rows, layer, units, rate):
    """Whether each element of a mini-batch of ``n_rows`` rows is kept (rate 0: all)."""
    if rate == 0:
        return np.ones((n_rows, units), dtype=bool)
    return words(seed, slot, t, np.arange(n_rows), layer, units) >= threshold(rate)


def penalty(flat, reg):
    if reg is None:
        return 0.0
    out = 0.0
    for l in range(len(flat) // 2):
        W, b = flat[2 * l], flat[2 * l + 1]
        out += reg["kernel_l1"][l] * np.abs(W).sum() + reg["kernel_l2"][l] * (W * W).sum()
        out += reg["bias_l1"][l] * np.abs(b).sum() + reg["bias_l2"][l] * (b * b).sum()
    return float(out)


def reg_grads(flat, reg):
    if reg is None:
        return [np.zeros_like(a) for a in flat]
    g = []
    for l in range(len(flat) // 2):
        W, b = flat[2 * l], flat[2 * l + 1]
        g += [reg["kernel_l1"][l] * np.sign(W) + 2 * reg["kernel_l2"][l] * W, reg["bias_l1"][l] * np.sign(b) + 2 * reg["bias_l2"][l] * b]
    return g


def dropped_loss_and_grads(spec, weights, xb, yb, rates, masks, loss="mse"):
    """(data loss + activity term, grads) of one training mini-batch in float64, ``masks[l]`` the keep mask of layer l's input
    (None where its rate is 0)."""
    d = np.float64
    L = spec.n_layers
    a = np.asarray(xb, d)
    if masks[0] is not None:
        a = np.where(masks[0], a * scale(rates[0]), 0.0)
    acts, raw = [a], [a]  # inputs of each layer as stored (dropped), and the undropped activations
    for l in range(L):
        W, b = weights[l]
        o = km._act(spec.acts[l], acts[-1] @ np.asarray(W, d) + np.asarray(b, d))
        raw.append(o)
        if l + 1 < L and masks[l + 1] is not None:
            o = np.where(masks[l + 1], o * scale(rates[l + 1]), 0.0)
        acts.append(o)
    data, delta = lo._output_delta(loss, acts[-1], np.asarray(yb, d), d)
    reg = 0.0
    for l in range(L):
        if spec.l1[l] != 0.0:
            reg += spec.l1[l] * np.abs(acts[l + 1]).sum()
    grads = [None] * L
    for l in range(L - 1, -1, -1):
        g = delta
        if spec.l1[l] != 0.0:
            g = g + spec.l1[l] * np.sign(acts[l + 1])
        if l + 1 < L and masks[l + 1] is not None:
            g = g * masks[l + 1] * scale(rates[l + 1])
        dz = g * km._act_grad_from_output(spec.acts[l], raw[l + 1])
        grads[l] = (acts[l].T @ dz, dz.sum(axis=0))
        if l > 0:
            delta = dz @ np.asarray(weights[l][0], d).T
    return float(data) + float(reg), grads


def fit(spec, weights, X, y, rates, seed=0, slot=0, step0=0, reg=None, optimizer=None, epochs=1, batch_size=32, perms=None,
        n_val=0, val_batch=None, loss="mse", stop=None, state=None):
    """
    Keras' fit with Dropout in float64, the masks of job (``seed``, ``slot``) from optimizer step ``step0`` + 1 on.  ``stop``:
    (monitor, patience) of an EarlyStopping callback.  Returns (weights, history, state); pass ``state`` back with ``step0``
    advanced to continue a fit.
    """
    d = np.float64
    optimizer = optimizer or ("adam", {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7, "weight_decay": 0.0, "clipvalue": None})
    X, y = np.asarray(X, d), np.asarray(y, d)
    n = len(X) - n_val
    Xv, yv = X[n:], y[n:]
    flat = [np.asarray(a, d).copy() for W, b in weights for a in (W, b)]
    st = state if state is not None else oo.OptState(flat, d)
    pairs = lambda a: [(a[2 * i], a[2 * i + 1]) for i in range(len(a) // 2)]  # noqa: E731
    widths = spec.dims[:-1]
    hist = {"loss": [], "val_loss": []}
    best, wait, t = np.inf, 0, step0
    for e in range(epochs):
        order = np.asarray(perms[e])[:n] if perms is not None else np.arange(n)
        ls = 0.0
        for s in range(0, n, batch_size):
            idx = order[s:s + batch_size]
            t += 1
            masks = [None if rates[l] == 0 else keep_mask(seed, slot, t, len(idx), l, widths[l], rates[l]) for l in range(spec.n_layers)]
            l_, grads = dropped_loss_and_grads(spec, pairs(flat), X[idx], y[idx], rates, masks, loss)
            ls += (l_ + penalty(flat, reg)) * len(idx)
            g = [a + r for a, r in zip([a for gW, gb in grads for a in (gW, gb)], reg_grads(flat, reg))]
            flat = oo.step(optimizer, flat, g, st, d)
        hist["loss"].append(ls / n)
        if n_val:
            vb, vs = val_batch or batch_size, 0.0
            for s in range(0, n_val, vb):
                l_, _, _, yh = lo.ff_loss_and_grads(spec, pairs(flat), Xv[s:s + vb], yv[s:s + vb], d, False, loss)
                vs += (float(l_) + penalty(flat, reg)) * len(yh)
            hist["val_loss"].append(vs / n_val)
        if stop is not None:
            v = hist[stop[0]][-1]
            wait += 1
            if v < best:
                best, wait = v, 0
            elif wait >= stop[1] and e > 0:
                break
    return pairs(flat), hist, st
