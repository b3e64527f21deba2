"""
The loss oracle (tests/loss_oracle.py) against PyTorch's CPU autograd in float64, and against central finite differences through
a Dense stack and an LSTM stack -- no GPU needed.  torch's ``l1_loss`` / ``huber_loss(delta=1)`` / ``mse_loss`` and the Keras
expressions of MAPE, MSLE and log-cosh written with torch ops are the witnesses; gradients at the table's edge cases (e = 0,
yhat below eps, |e| at delta) are pinned explicitly.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from loss_oracle import EPS, LOSSES, ff_loss_and_grads, loss_grad, loss_value, lstm_loss_and_grads
from test_oracle_torch_witness import t64, torch_ff

from oracle import keras_math as km


def torch_loss(loss, yh, y):
    """Mean over all elements, as Keras' per-sample mean then sum_over_batch_size gives for equal-width rows."""
    if loss == "mse":
        return F.mse_loss(yh, y)
    if loss == "mae":
        return F.l1_loss(yh, y)
    if loss == "huber":
        return F.huber_loss(yh, y, delta=1.0)
    if loss == "mape":
        return (100.0 * (y - yh).abs() / y.abs().clamp(min=EPS)).mean()
    if loss == "msle":
        return ((yh.clamp(min=EPS) + 1).log() - (y.clamp(min=EPS) + 1).log()).pow(2).mean()
    if loss == "log_cosh":
        e = yh - y
        return (e + F.softplus(-2.0 * e) - math.log(2.0)).mean()
    raise ValueError(loss)


def edge_data(rng):
    """Predictions and targets that reach every branch: e = 0 exactly, |e| on both sides of 1, yhat < 0 and = eps, y near 0."""
    y = rng.uniform(-0.5, 2.0, (9, 7))
    yh = y + rng.uniform(-2.5, 2.5, y.shape)
    yh[0, :3] = y[0, :3]                     # e = 0
    yh[1, 0], yh[1, 1] = y[1, 0] + 1.0, y[1, 1] - 1.0  # |e| = delta
    yh[2, :] = -rng.uniform(0.01, 0.5, 7)    # negative predictions (MSLE clamps them)
    yh[3, 0] = EPS                           # the tie of maximum(yhat, eps)
    y[4, :] = rng.uniform(-1e-4, 1e-4, 7)    # targets near 0 (MAPE divides by max(|y|, eps))
    y[4, 0] = 0.0
    return yh, y


@pytest.mark.parametrize("loss", LOSSES)
def test_loss_values_and_gradients_against_autograd(loss):
    yh, y = edge_data(np.random.default_rng(5))
    tyh = t64(yh, True)
    ref = torch_loss(loss, tyh, t64(y))
    ref.backward()
    np.testing.assert_allclose(np.mean(loss_value(loss, yh, y)), ref.item(), rtol=1e-12)
    np.testing.assert_allclose(loss_grad(loss, yh, y) / yh.size, tyh.grad.numpy(), rtol=1e-12, atol=1e-15)


def test_edge_case_gradients():
    yh, y = edge_data(np.random.default_rng(5))
    assert (loss_grad("mae", yh, y)[0, :3] == 0).all() and (loss_grad("mape", yh, y)[0, :3] == 0).all()  # sign(0) = 0
    assert loss_grad("huber", yh, y)[1, 0] == pytest.approx(1.0) and loss_grad("huber", yh, y)[1, 1] == pytest.approx(-1.0)
    assert (loss_grad("msle", yh, y)[2] == 0).all()  # below eps: maximum passes nothing to yhat
    assert loss_grad("msle", yh, y)[3, 0] != 0       # at eps: the tie goes to yhat
    assert np.abs(loss_grad("mape", yh, y)[4, 0]) == pytest.approx(100.0 / EPS)
    e = np.linspace(-30, 30, 61)
    np.testing.assert_allclose(loss_grad("log_cosh", e, np.zeros_like(e)), np.tanh(e), atol=1e-15)
    np.testing.assert_allclose(loss_value("log_cosh", e, np.zeros_like(e)), np.log(np.cosh(e)), rtol=1e-12, atol=1e-15)


def test_float32_keeps_its_dtype():
    yh, y = (a.astype(np.float32) for a in edge_data(np.random.default_rng(5)))
    for loss in LOSSES:
        assert loss_value(loss, yh, y).dtype == np.float32 and loss_grad(loss, yh, y).dtype == np.float32, loss


def dense_case(rng):
    spec = km.FFSpec([6, 5, 3, 5, 6], ["tanh", "relu", "sigmoid", "linear"], [0.0, 1e-3, 0.0, 0.0])
    w = [(W.astype(np.float64), rng.uniform(-0.3, 0.3, b.shape)) for W, b in km.init_ff_weights(spec, rng)]
    x = rng.random((10, 6))
    y = x * 2.5 - 0.3  # errors on both sides of the Huber delta, some targets below 0
    y[0, 0] = 0.0
    return spec, w, x, y


@pytest.mark.parametrize("loss", LOSSES)
def test_dense_stack_against_autograd(loss):
    spec, w, x, y = dense_case(np.random.default_rng(7))
    total, data, grads, yhat = ff_loss_and_grads(spec, w, x, y, dtype=np.float64, loss=loss)
    tw = [(t64(W, True), t64(b, True)) for W, b in w]
    acts = []
    out = torch_ff(spec, tw, t64(x), acts)
    t_data = torch_loss(loss, out, t64(y))
    t_total = t_data + sum(c * a.abs().sum() for c, a in zip(spec.l1, acts) if c)
    t_total.backward()
    np.testing.assert_allclose([total, data], [t_total.item(), t_data.item()], rtol=1e-12)
    for (gW, gb), (W, b) in zip(grads, tw):
        np.testing.assert_allclose(gW, W.grad.numpy(), rtol=1e-9, atol=1e-13)
        np.testing.assert_allclose(gb, b.grad.numpy(), rtol=1e-9, atol=1e-13)


def central_difference(f, arrays, picks, h=1e-6):
    out = []
    for a, idx in picks:
        a = arrays[a]
        old = a[idx]
        a[idx] = old + h
        up = f()
        a[idx] = old - h
        down = f()
        a[idx] = old
        out.append((up - down) / (2 * h))
    return np.array(out)


@pytest.mark.parametrize("loss", LOSSES)
def test_dense_stack_finite_differences(loss):
    spec, w, x, y = dense_case(np.random.default_rng(9))
    w = [(W.copy(), b.copy()) for W, b in w]
    arrays = [a for pair in w for a in pair]
    _, _, grads, _ = ff_loss_and_grads(spec, w, x, y, dtype=np.float64, loss=loss)
    flat_g = [g for pair in grads for g in pair]
    rng = np.random.default_rng(1)
    picks = [(k, tuple(rng.integers(0, s) for s in arrays[k].shape)) for k in range(len(arrays)) for _ in range(4)]
    fd = central_difference(lambda: float(ff_loss_and_grads(spec, w, x, y, dtype=np.float64, loss=loss)[0]), arrays, picks)
    an = np.array([flat_g[k][idx] for k, idx in picks])
    np.testing.assert_allclose(an, fd, rtol=2e-5, atol=1e-8 + 1e-7 * np.abs(fd).max())  # MAPE's y = 0 element: losses ~1e9, FD noise with them


def torch_lstm(spec, layers, dense, windows):
    """The LSTM stack in torch ops on the given leaves (gate order i, f, c, o; one bias; zero initial state)."""
    seq = windows
    for (K, U, b), act in zip(layers, spec.acts):
        u = U.shape[0]
        h = torch.zeros((seq.shape[0], u), dtype=torch.float64)
        c = torch.zeros_like(h)
        out = []
        for t in range(seq.shape[1]):
            z = seq[:, t] @ K + h @ U + b
            i, f, g, o = torch.sigmoid(z[:, :u]), torch.sigmoid(z[:, u:2 * u]), torch.tanh(z[:, 2 * u:3 * u]), torch.sigmoid(z[:, 3 * u:])
            c = f * c + i * g
            h = o * torch.tanh(c)
            out.append(h)
        seq = torch.stack(out, dim=1)
    return seq[:, -1] @ dense[0] + dense[1]


def lstm_case(rng, out_func="linear"):
    spec = km.LSTMSpec(n_features=4, units=[5, 3], acts=["tanh", "tanh"], n_features_out=4, out_func=out_func, lookback_window=4)
    layers, dense = km.init_lstm_weights(spec, rng)
    layers = [(K.astype(np.float64), U.astype(np.float64), (b + rng.uniform(-0.2, 0.2, b.shape)).astype(np.float64)) for K, U, b in layers]
    weights = (layers, (dense[0].astype(np.float64), rng.uniform(-0.2, 0.2, dense[1].shape)))
    windows, targets = rng.random((6, 4, 4)), rng.uniform(-0.5, 2.5, (6, 4))
    return spec, weights, windows, targets


@pytest.mark.parametrize("loss", LOSSES)
def test_lstm_stack_against_autograd_and_finite_differences(loss):
    spec, weights, windows, targets = lstm_case(np.random.default_rng(11))
    value, grads, _ = lstm_loss_and_grads(spec, weights, windows, targets, dtype=np.float64, loss=loss)
    tl = [(t64(K, True), t64(U, True), t64(b, True)) for K, U, b in weights[0]]
    td = (t64(weights[1][0], True), t64(weights[1][1], True))
    ref = torch_loss(loss, torch_lstm(spec, tl, td, t64(windows)), t64(targets))
    ref.backward()
    np.testing.assert_allclose(value, ref.item(), rtol=1e-11)
    want = [t.grad.numpy() for lay in tl for t in lay] + [t.grad.numpy() for t in td]
    for g, r in zip(km._lstm_flat(grads), want):
        np.testing.assert_allclose(g, r, rtol=1e-8, atol=1e-12)

    arrays = [a.copy() for a in km._lstm_flat(weights)]
    nl = len(spec.units)
    rng = np.random.default_rng(2)
    picks = [(k, tuple(rng.integers(0, s) for s in arrays[k].shape)) for k in range(len(arrays)) for _ in range(3)]
    fd = central_difference(lambda: float(lstm_loss_and_grads(spec, km._lstm_unflat(arrays, nl), windows, targets, np.float64, loss)[0]),
                            arrays, picks)
    flat_g = km._lstm_flat(grads)
    np.testing.assert_allclose([flat_g[k][idx] for k, idx in picks], fd, rtol=2e-5, atol=1e-8)


def test_mse_is_the_oracles_own_fit():
    """With loss="mse" the loss oracle is keras_math's arithmetic to the bit, in float32."""
    spec, w, x, y = dense_case(np.random.default_rng(3))
    w32 = [(W.astype(np.float32), b.astype(np.float32)) for W, b in w]
    a = ff_loss_and_grads(spec, w32, x.astype(np.float32), y.astype(np.float32))
    b = km.ff_loss_and_grads(spec, w32, x.astype(np.float32), y.astype(np.float32))
    assert a[0] == b[0] and all(np.array_equal(p, q) for gp, gq in zip(a[2], b[2]) for p, q in zip(gp, gq))
    spec, weights, windows, targets = lstm_case(np.random.default_rng(4))
    w32 = ([tuple(t.astype(np.float32) for t in lay) for lay in weights[0]], tuple(t.astype(np.float32) for t in weights[1]))
    a = lstm_loss_and_grads(spec, w32, windows, targets)
    b = km.lstm_loss_and_grads(spec, w32, windows, targets)
    assert a[0] == b[0] and all(np.array_equal(p, q) for p, q in zip(km._lstm_flat(a[1]), km._lstm_flat(b[1])))
