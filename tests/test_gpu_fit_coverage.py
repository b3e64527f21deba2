"""
The training kernels across what they accept: gb_ffae_fit (Dense stacks) and gb_lstm_fit (LSTM stacks) against the oracle's
Keras-style fit loops (oracle/keras_math.py) started from the same weights and visiting order.

A default Adam step moves each weight by about lr whatever the size of its gradient, so a gradient off by a constant factor
survives a comparison of trained weights.  The "gradient" cases therefore run Adam with beta1 = beta2 = 0 and eps much larger
than the gradients, with lr = eps: a step is then -g * eps / (|g| + eps), close to -g, and the weight change exposes the raw
gradient sums.
"""
import ctypes as C
import math

import numpy as np
import pytest
from parity_helpers import close, random_net

pytestmark = pytest.mark.gpu

KERAS_ADAM = {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7}
GRAD_ADAM = {"lr": 1.0, "beta1": 0.0, "beta2": 0.0, "eps": 1.0}


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("needs an H100")
    import __graft_entry__ as ge

    ge.build()
    return t


@pytest.fixture(scope="module")
def engine(torch):
    from gordo_components_b200 import engine as e

    return e


@pytest.fixture(scope="module")
def km(torch):
    from oracle import keras_math

    return keras_math


def waves(rng, n, width, lo=0.15, hi=0.85):
    """Smooth multi-sine columns in [lo, hi] (sensor-like data: the fit makes progress, unlike on white noise)."""
    t = np.linspace(0, 12, n)[:, None]
    mid, amp = (lo + hi) / 2, (hi - lo) / 2 * 0.9
    return (mid + amp * np.sin(t * rng.uniform(0.5, 2, width) + rng.uniform(0, 3, width)) + rng.normal(0, 0.01, (n, width))).astype(np.float32)


def device(torch, eng, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)


def ff_plan(spec):
    from gordo_components_b200 import _cabi

    net = _cabi.make_ffnet(spec.dims, spec.acts, spec.l1)
    w, d = C.c_int32(-1), C.c_int32(-1)
    rc = _cabi.load_library().gb_ffae_fit_plan(C.byref(net), C.byref(w), C.byref(d))
    return rc, w.value, d.value


def ff_fit_gpu(engine, torch, spec, w0s, X, Y, jobs_h, epochs, batch, perm=None, **kw):
    """One gb_ffae_fit launch: returns (trained weights per slot, loss [n_jobs, epochs], accuracy [n_jobs, epochs])."""
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    params = eng.pack_params(w0s)
    loss, acc, _ = eng.fit(params, engine.jobs_to_device(jobs_h, eng.device), len(jobs_h), int(jobs_h["n_rows"].max()), device(torch, eng, X),
                           device(torch, eng, Y), epochs=epochs, batch_size=batch, perm=None if perm is None else device(torch, eng, perm), **kw)
    torch.cuda.synchronize()
    return eng.unpack_params(params), loss.cpu().numpy(), acc.cpu().numpy()


def check_ff_fit(km, spec, w0s, Xs, Ys, perm, got, loss, acc, epochs, batch, adam=KERAS_ADAM, l1_div_batch=False, gradients=False):
    """Job j (slot j) against the oracle's fit of the same weights over the same visiting order."""
    for j in range(len(Xs)):
        n = len(Xs[j])
        w_ref, hist, _ = km.ff_fit(spec, w0s[j], Xs[j], Ys[j], epochs=epochs, batch_size=batch, perms=[perm[j, e, :n] for e in range(epochs)],
                                   lr=adam["lr"], b1=adam["beta1"], b2=adam["beta2"], eps=adam["eps"], l1_div_batch=l1_div_batch,
                                   dtype=np.float64 if gradients else np.float32)
        for l, ((Wg, bg), (Wr, br), (W0, b0)) in enumerate(zip(got[j], w_ref, w0s[j])):
            if gradients:  # the weight change is (nearly) minus the summed gradient of every step
                for g_, r_, z_, what in ((Wg, Wr, W0, "W"), (bg, br, b0, "b")):
                    close(g_ - z_, r_ - z_, mag=float(np.abs(r_ - z_).max()), rtol=1e-3, name=f"job {j} raw gradients {what}{l}")
            else:  # weights moved by ~lr*steps; agreement to 1e-4 of the weight scale
                close(Wg, Wr, mag=float(np.abs(Wr).max()), name=f"job {j} W{l}")
                close(bg, br, mag=max(float(np.abs(br).max()), 1e-2), name=f"job {j} b{l}")
        close(loss[j], np.array(hist["loss"]), mag=0.0, rtol=5e-4, name=f"job {j} loss history")
        close(acc[j], np.array(hist["accuracy"]), mag=0, rtol=0, atol=2.0 / n, name=f"job {j} accuracy history")


def uniform_perm(M, E, N, seed):
    return np.stack([[np.random.default_rng(seed + 1000 * m + e).permutation(N) for e in range(E)] for m in range(M)]).astype(np.int32)


# ------------------------------------------------------------------------------------------------ A1: architectures
#   name: (dims, acts, l1, l1_div_batch, targets)   targets: "x" (autoencoder), "waves" (other columns), "binary" (0/1)
FF_GRID = {
    "relu_hidden": ([12, 10, 6, 10, 12], ["relu"] * 3 + ["linear"], None, False, "x"),
    "sigmoid_hidden": ([12, 10, 6, 10, 12], ["sigmoid"] * 3 + ["linear"], None, False, "x"),
    "linear_hidden": ([12, 10, 6, 10, 12], ["linear"] * 4, None, False, "x"),
    "sigmoid_out": ([9, 7, 9], ["tanh", "sigmoid"], None, False, "x"),
    "tanh_out": ([9, 7, 9], ["relu", "tanh"], None, False, "x"),
    "relu_out": ([9, 7, 9], ["sigmoid", "relu"], None, False, "x"),
    "out_narrower": ([12, 8, 7], ["tanh", "linear"], None, False, "waves"),   # n_in a multiple of 4, n_out not
    "out_wider": ([7, 5, 16], ["tanh", "linear"], None, False, "waves"),      # n_out a multiple of 4, n_in not
    "binary": ([8, 5, 1], ["tanh", "sigmoid"], None, False, "binary"),       # n_out == 1: binary accuracy
    "width1": ([8, 1, 8], ["tanh", "linear"], None, False, "x"),
    "width3": ([8, 3, 3, 8], ["tanh", "relu", "linear"], None, False, "x"),
    "l1_every_layer": ([10, 7, 4, 7, 10], ["tanh"] * 3 + ["linear"], [1e-3, 2e-3, 1e-3, 5e-4], False, "x"),
    "l1_div_batch": ([10, 7, 4, 7, 10], ["tanh"] * 3 + ["linear"], [1e-3, 2e-3, 1e-3, 5e-4], True, "x"),
}


def ff_case_data(km, case, M, N, seed):
    dims, acts, l1, div, targets = FF_GRID[case]
    spec = km.FFSpec(list(dims), list(acts), list(l1) if l1 else [])
    rng = np.random.default_rng(seed)
    Xs = [waves(rng, N, dims[0]) for _ in range(M)]
    if targets == "x":
        Ys = Xs
    elif targets == "waves":
        Ys = [waves(rng, N, dims[-1]) for _ in range(M)]
    else:
        Ys = [(rng.random((N, 1)) > 0.5).astype(np.float32) for _ in range(M)]
    w0s = [random_net(km, dims, seed + 7 * m, acts)[1] for m in range(M)]
    return spec, div, Xs, Ys, w0s


@pytest.mark.parametrize("case", list(FF_GRID))
def test_ffae_fit_architecture_grid(engine, torch, km, case):
    M, N, E, B = 3, 150, 2, 32
    spec, div, Xs, Ys, w0s = ff_case_data(km, case, M, N, seed=3)
    perm = uniform_perm(M, E, N, seed=11)
    got, loss, acc = ff_fit_gpu(engine, torch, spec, w0s, np.concatenate(Xs), np.concatenate(Ys), engine.uniform_jobs(M, N), E, B, perm,
                                l1_div_batch=div)
    check_ff_fit(km, spec, w0s, Xs, Ys, perm, got, loss, acc, E, B, l1_div_batch=div)


# ------------------------------------------------------------------------------------------------ A2: raw gradients
#   name: (grid case, rows, batch)
FF_GRAD = {
    "tanh": ("l1_every_layer", 100, 32),
    "relu": ("relu_hidden", 100, 32),
    "sigmoid": ("sigmoid_hidden", 100, 32),
    "linear": ("linear_hidden", 100, 32),
    "heads": ("relu_out", 100, 32),
    "l1": ("l1_every_layer", 100, 32),
    "l1_div_batch": ("l1_div_batch", 100, 32),
    "n_out_ne_n_in": ("out_wider", 100, 32),
    "batch_100": ("out_narrower", 300, 100),  # 4 chunks of 32 rows, the last one ragged (4 rows)
}


@pytest.mark.parametrize("case", list(FF_GRAD))
def test_ffae_fit_raw_gradients(engine, torch, km, case):
    grid_case, N, B = FF_GRAD[case]
    M, E = 2, 1
    spec, div, Xs, Ys, w0s = ff_case_data(km, grid_case, M, N, seed=5)
    if case == "tanh":
        spec.l1 = [0.0] * spec.n_layers
    perm = uniform_perm(M, E, N, seed=13)
    got, loss, acc = ff_fit_gpu(engine, torch, spec, w0s, np.concatenate(Xs), np.concatenate(Ys), engine.uniform_jobs(M, N), E, B, perm,
                                l1_div_batch=div, adam=GRAD_ADAM)
    check_ff_fit(km, spec, w0s, Xs, Ys, perm, got, loss, acc, E, B, adam=GRAD_ADAM, l1_div_batch=div, gradients=True)


# ------------------------------------------------------------------------------------------------ A3: memory plans
# (weights in L2, dz buffers in L2) -> shape; tests/test_fit_plan.py pins the same shapes to the same plans without a GPU
PLAN_CASES = {
    "shared": ((0, 0), "hourglass", 64),
    "weights_in_l2": ((1, 0), "symmetric", 10),
    "one_dz_in_l2": ((1, 1), "symmetric", 64),
    "two_dz_in_l2": ((1, 2), "symmetric", 96),
    "three_dz_in_l2": ((1, 3), "symmetric", 128),
}


def plan_spec(km, kind, T):
    return km.ff_hourglass_spec(T) if kind == "hourglass" else km.ff_symmetric_spec(T)


@pytest.mark.parametrize("case", list(PLAN_CASES))
def test_ffae_fit_every_memory_plan(engine, torch, km, case):
    want, kind, T = PLAN_CASES[case]
    spec = plan_spec(km, kind, T)
    assert ff_plan(spec) == (0, *want)
    M, N, E, B = 2, 150, 2, 50  # 50-row batches: two chunks each, the gradient scratch is used as well
    rng = np.random.default_rng(T)
    Xs = [waves(rng, N, T) for _ in range(M)]
    w0s = [km.init_ff_weights(spec, np.random.default_rng(60 + m)) for m in range(M)]
    perm = uniform_perm(M, E, N, seed=17)
    X = np.concatenate(Xs)
    got, loss, acc = ff_fit_gpu(engine, torch, spec, w0s, X, X, engine.uniform_jobs(M, N), E, B, perm)
    check_ff_fit(km, spec, w0s, Xs, Xs, perm, got, loss, acc, E, B)


def test_ffae_fit_refuses_the_first_width_beyond_the_plans(engine, torch, km):
    """173 tags with the 256-128-64 symmetric default: gb_ffae_fit returns GB_E_SMEM before it launches anything."""
    spec = km.ff_symmetric_spec(173)
    assert ff_plan(spec)[0] == -4
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    params = torch.full((1, eng.param_stride), 0.25, device=eng.device)
    m = torch.zeros((1, eng.state_stride), device=eng.device)
    v = torch.zeros_like(m)
    x = torch.rand((40, 173), device=eng.device)
    with pytest.raises(ValueError, match="shared memory"):
        eng.fit(params, engine.jobs_to_device(engine.uniform_jobs(1, 40), eng.device), 1, 40, x, x, epochs=1, state=(m, v))
    torch.cuda.synchronize()
    assert bool((params == 0.25).all()) and not bool(m.any()) and not bool(v.any())


# ------------------------------------------------------------------------------------------------ A4: on-device shuffle
@pytest.mark.parametrize("batch", [32, 7])
def test_ffae_fit_shuffle_visits_every_row_once(engine, torch, km, batch):
    """
    With lr = 0 the weights stay put, so with l1 = 0 an epoch's loss is (sum over the visited rows of the row's mean squared
    error) / n.  Job j of n reads n copies of the same rows; its targets are 0 except row j, whose error dominates: an epoch that
    skips row j reports about (1 - share) of the expected loss, one that visits it twice about (1 + share).  All jobs share a slot,
    so they walk the same keyed permutation: together they check that every row of it is visited exactly once per epoch.
    """
    spec = km.FFSpec([4, 3, 4], ["tanh", "linear"])
    _, w = random_net(km, [4, 3, 4], 2)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    params = eng.pack_params([w])
    D = 20.0
    for n in (1, 2, 3, 4, 5, 16, 17, 63, 64, 65, 257, 1000, 1025):
        rows = np.random.default_rng(n).random((n, 4)).astype(np.float32)
        base = (km.ff_forward(spec, w, rows, np.float64) ** 2).mean(axis=1)        # targets 0
        dom = ((km.ff_forward(spec, w, rows, np.float64) - D) ** 2).mean(axis=1)   # target D
        want = (base.sum() - base + dom) / n                                        # job j: row j carries the target D
        x = torch.from_numpy(rows).to(dev).repeat(n, 1)
        y = torch.zeros_like(x)
        y.view(n, n, 4)[torch.arange(n), torch.arange(n)] = D
        jobs = engine.jobs_to_device(engine.make_jobs(np.zeros(n, np.int32), n, np.arange(n, dtype=np.int64) * n), dev)
        for seed in (1, 2):
            loss, _, _ = eng.fit(params, jobs, n, n, x, y, epochs=3, batch_size=batch, shuffle=True, seed=seed, adam=dict(KERAS_ADAM, lr=0.0))
            got = loss.cpu().numpy()
            for e in range(3):
                close(got[:, e], want, mag=0.0, rtol=1e-4, name=f"n={n} seed={seed} epoch {e}: per-row coverage")


# ------------------------------------------------------------------------------------------------ A5: one launch per epoch
@pytest.mark.parametrize("kind,T,want,batch,order", [("hourglass", 8, (0, 0), 32, "perm"), ("hourglass", 8, (0, 0), 50, "sequential"),
                                                     ("symmetric", 10, (1, 0), 32, "perm"), ("symmetric", 10, (1, 0), 50, "sequential"),
                                                     ("symmetric", 64, (1, 1), 50, "perm")])
def test_ffae_fit_per_epoch_launches_equal_one_launch(engine, torch, km, kind, T, want, batch, order):
    """The estimators' EarlyStopping / validation_split path trains one launch per epoch, carrying the Adam state and step count
    (models.py): E such launches must be bit-identical to one E-epoch launch, weights and moments -- in the plans that keep the
    weight image and the dz scratch in the same state arrays too."""
    spec = plan_spec(km, kind, T)
    M, N, E = 2, 110, 4
    rng = np.random.default_rng(1)
    X = np.concatenate([waves(rng, N, spec.dims[0]) for _ in range(M)])
    w0s = [km.init_ff_weights(spec, np.random.default_rng(70 + m)) for m in range(M)]
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    xd = device(torch, eng, X)
    jobs = engine.jobs_to_device(engine.uniform_jobs(M, N), dev)
    perm = device(torch, eng, uniform_perm(M, E, N, seed=3)) if order == "perm" else None
    p1 = eng.pack_params(w0s)
    l1, _, (m1, v1) = eng.fit(p1, jobs, M, N, xd, xd, epochs=E, batch_size=batch, perm=perm, shuffle=False)
    p2 = eng.pack_params(w0s)
    state, step0, l2 = None, 0, []
    for e in range(E):
        pe = None if perm is None else perm[:, e:e + 1].contiguous()
        loss, _, state = eng.fit(p2, jobs, M, N, xd, xd, epochs=1, batch_size=batch, perm=pe, shuffle=False, state=state, step0=step0)
        step0 += math.ceil(N / batch)
        l2.append(loss)
    torch.cuda.synchronize()
    assert ff_plan(spec)[1:] == want
    assert torch.equal(p1, p2), "weights"
    assert torch.equal(m1, state[0]), "Adam m (and the gradient scratch / weight image)"
    assert torch.equal(v1, state[1]), "Adam v (and the dz scratch)"
    assert torch.equal(l1, torch.cat(l2, dim=1)), "loss history"


# ------------------------------------------------------------------------------------------------ A6: validation loss, ragged fleets
def test_frozen_validation_loss_in_batches(engine, torch, km):
    """validation_split + validation_batch_size below the tail: the estimator's val_loss is the lr = 0 fit of the tail, which must
    be the sample-weighted mean of the per-batch total losses (MSE + activity l1, not divided by the batch) at the trained weights."""
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    np.random.seed(4)
    X = waves(np.random.default_rng(4), 300, 6)
    m = KerasAutoEncoder(kind="feedforward_hourglass", epochs=2, batch_size=32, validation_split=0.15, validation_batch_size=16)
    m.fit(X, X)
    spec = km.ff_hourglass_spec(6)
    assert any(spec.l1)
    tail = X[255:]
    assert len(tail) == 45
    num = 0.0
    for s in range(0, 45, 16):
        total, _mse, _g, _yh = km.ff_loss_and_grads(spec, m.model.weights, tail[s:s + 16], tail[s:s + 16], np.float64)
        num += float(total) * len(tail[s:s + 16])
    close(m.get_metadata()["history"]["val_loss"][-1], num / 45, mag=0.0, rtol=2e-4, name="val_loss")


@pytest.mark.parametrize("T,batch", [(6, 1), (8, 32), (6, 50)])
def test_ffae_fit_many_ragged_jobs(engine, torch, km, T, batch):
    """About 200 jobs of 1..300 rows in one launch, at row offsets that are not multiples of 4, with their own slots in shuffled
    order; jobs shorter than their batch among them.  Every job against the oracle."""
    rng = np.random.default_rng(T * 100 + batch)
    J = 200
    lens = rng.integers(1, 301, J)
    lens[:6] = [1, 2, max(batch - 1, 1), batch, batch + 1, 300]
    gaps = rng.integers(1, 4, J)
    x_rows = np.cumsum(gaps) + np.concatenate([[0], np.cumsum(lens)[:-1]])
    X = waves(rng, int(x_rows[-1] + lens[-1]), T)
    slots = rng.permutation(J).astype(np.int32)
    nets = [random_net(km, T, 300 + s) for s in range(J)]
    spec = nets[0][0]
    w0s = [w for _, w in nets]
    E = 1 if batch == 1 else 2
    perm = np.zeros((J, E, int(lens.max())), np.int32)
    for j in range(J):
        for e in range(E):
            perm[j, e, :lens[j]] = rng.permutation(lens[j])
    got, loss, acc = ff_fit_gpu(engine, torch, spec, w0s, X, X, engine.make_jobs(slots, lens, x_rows), E, batch, perm)
    Xs = [X[x_rows[j]:x_rows[j] + lens[j]] for j in range(J)]
    check_ff_fit(km, spec, [w0s[s] for s in slots], Xs, Xs, perm, [got[s] for s in slots], loss, acc, E, batch)


# ------------------------------------------------------------------------------------------------ B: LSTM fit
#   name: (n_features, n_features_out, units, cell act, head act, lookback, rows per job, batch, epochs)
LSTM_GRID = {
    "relu_cells_three_jobs": (5, 5, [6, 5], "relu", "tanh", 4, [40, 33, 51], 8, 2),
    "linear_cells": (6, 6, [7, 4, 6], "linear", "sigmoid", 3, [45], 8, 2),
    "sigmoid_cells_wider_out": (4, 9, [8, 5], "sigmoid", "relu", 5, [50], 16, 2),
    "narrower_out_lookback_1_batch_1": (9, 3, [6, 4], "tanh", "linear", 1, [25], 1, 2),
    "widths_65_130_windows_64_65": (20, 20, [65, 130], "tanh", "linear", 3, [66, 67], 32, 2),
}


def lstm_setup(engine, torch, km, F, F_out, units, act, head, lookback, rows, seed):
    spec = km.LSTMSpec(F, list(units), [act] * len(units), F_out, head, lookback)
    rng = np.random.default_rng(seed)
    shrink = 0.5 if act in ("relu", "linear") else 1.0  # keep unbounded cells bounded over the lookback
    ws = []
    for i in range(len(rows)):
        layers, (Wd, bd) = km.init_lstm_weights(spec, np.random.default_rng(seed + 10 + i))
        layers = [(K * shrink, U * shrink, b + rng.uniform(-0.1, 0.1, b.shape).astype(np.float32)) for K, U, b in layers]
        ws.append((layers, (Wd, rng.uniform(-0.1, 0.1, bd.shape).astype(np.float32))))
    Xs = [rng.random((n, F)).astype(np.float32) for n in rows]
    Ys = [rng.random((n, F_out)).astype(np.float32) for n in rows]
    eng = engine.LSTMEngine(F, spec.units, spec.acts, F_out, head, lookback)
    dev = eng.device
    nwin = [n - lookback + 1 for n in rows]
    starts = np.concatenate([[0], np.cumsum(rows)[:-1]])
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(len(rows)), nwin, starts), dev)
    x, y = device(torch, eng, np.concatenate(Xs)), device(torch, eng, np.concatenate(Ys))
    return spec, eng, ws, Xs, Ys, nwin, jobs, x, y


def check_lstm_fit(km, spec, ws, Xs, Ys, got, loss, acc, nwin, epochs, B, adam, gradients):
    for i in range(len(Xs)):
        want_w, hist = km.lstm_fit(spec, ws[i], Xs[i], Ys[i], epochs=epochs, batch_size=B, lr=adam["lr"], b1=adam["beta1"], b2=adam["beta2"],
                                   eps=adam["eps"])
        if epochs:
            close(loss[i], np.array(hist["loss"]), rtol=5e-4, name=f"job {i} loss history")
            assert np.allclose(acc[i], hist["accuracy"], atol=1.5 / nwin[i]), (acc[i], hist["accuracy"])
        steps = 1 + epochs * math.ceil(nwin[i] / B)
        for k, (w0, gl, wl) in enumerate(zip(km._lstm_flat(ws[i]), km._lstm_flat(got[i]), km._lstm_flat(want_w))):
            if gradients:
                close(gl - w0, wl - w0, mag=float(np.abs(wl - w0).max()), rtol=1e-3, name=f"job {i} array {k}: accumulated raw gradients")
            else:  # Adam moves a weight by ~lr per step whatever the gradient's size: compare the distance travelled
                close(gl - w0, wl - w0, mag=adam["lr"] * steps, rtol=2e-2, name=f"job {i} array {k}: trained weights")


@pytest.mark.parametrize("case", list(LSTM_GRID))
def test_lstm_fit_architecture_grid(engine, torch, km, case):
    F, F_out, units, act, head, lookback, rows, B, E = LSTM_GRID[case]
    spec, eng, ws, Xs, Ys, nwin, jobs, x, y = lstm_setup(engine, torch, km, F, F_out, units, act, head, lookback, rows, seed=21)
    params = eng.pack_params(ws)
    loss, acc, _ = eng.fit(params, jobs, len(rows), max(nwin), x, y, epochs=E, batch_size=B, primer=True, adam=KERAS_ADAM)
    torch.cuda.synchronize()
    check_lstm_fit(km, spec, ws, Xs, Ys, eng.unpack_params(params), loss.cpu().numpy(), acc.cpu().numpy(), nwin, E, B, KERAS_ADAM, False)


@pytest.mark.parametrize("act,epochs", [("relu", 1), ("linear", 1), ("relu", 0)])
def test_lstm_fit_raw_gradients(engine, torch, km, act, epochs):
    """beta1 = beta2 = 0, eps = lr = 1 with a sigmoid head; epochs = 0 is the primer step alone."""
    spec, eng, ws, Xs, Ys, nwin, jobs, x, y = lstm_setup(engine, torch, km, 8, 8, [12, 7], act, "sigmoid", 5, [70], seed=23)
    params = eng.pack_params(ws)
    loss, acc, (_, _, t) = eng.fit(params, jobs, 1, max(nwin), x, y, epochs=epochs, batch_size=32, primer=True, adam=GRAD_ADAM)
    torch.cuda.synchronize()
    assert int(t[0]) == 1 + epochs * math.ceil(nwin[0] / 32)
    check_lstm_fit(km, spec, ws, Xs, Ys, eng.unpack_params(params), loss.cpu().numpy(), acc.cpu().numpy(), nwin, epochs, 32, GRAD_ADAM, True)


def test_lstm_fit_per_epoch_launches_equal_one_launch(engine, torch, km):
    """The LSTM estimators' per-epoch path: E one-epoch launches carrying (m, v, t), the primer step in the first only, are
    bit-identical to one E-epoch launch."""
    _, eng, ws, _, _, nwin, jobs, x, y = lstm_setup(engine, torch, km, 6, 6, [9, 5], "tanh", "linear", 4, [60, 47], seed=25)
    E = 3
    p1 = eng.pack_params(ws)
    l1, _, (m1, v1, t1) = eng.fit(p1, jobs, 2, max(nwin), x, y, epochs=E, batch_size=16, primer=True)
    p2 = eng.pack_params(ws)
    state, l2 = None, []
    for e in range(E):
        loss, _, state = eng.fit(p2, jobs, 2, max(nwin), x, y, epochs=1, batch_size=16, primer=e == 0, state=state)
        l2.append(loss)
    torch.cuda.synchronize()
    assert torch.equal(t1, state[2]) and int(t1[0]) == 1 + E * math.ceil(nwin[0] / 16)
    assert torch.equal(p1, p2), "weights"
    assert torch.equal(m1, state[0]) and torch.equal(v1, state[1]), "Adam moments"
    assert torch.equal(l1, torch.cat(l2, dim=1)), "loss history"
