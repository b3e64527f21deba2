"""
The Keras regression losses on the training kernels: gb_ffae_fit in every memory plan at batches of 32 and 80 rows and
gb_ffae_fit_split in every memory plan through a row map with a held-out tail, the split / stop entry points on a small stack, and
gb_lstm_fit_loss, against the loss oracle (tests/loss_oracle.py) from injected weights and visiting order; the edge cases of the
loss table (sign(0) = 0, MSLE below eps, MAPE near 0, Huber on both sides of delta); mean squared error bit-identical to the
default call; and the loss through the estimators and the three batched fleet builds.
"""
import ctypes as C
import math
import pickle

import numpy as np
import pandas as pd
import pytest
from loss_oracle import LOSSES
from parity_helpers import ENTRIES, close, crossed, ff_split_run, random_net

pytestmark = pytest.mark.gpu

KERAS_ADAM = {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7}
GRAD_ADAM = {"lr": 1.0, "beta1": 0.0, "beta2": 0.0, "eps": 1.0}  # a step is ~ -g: the weight change exposes the raw gradients


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


@pytest.fixture(scope="module")
def lo(torch):
    import loss_oracle

    return loss_oracle


def waves(rng, n, width, lo=0.15, hi=0.85):
    t = np.linspace(0, 12, n)[:, None]
    mid, amp = (lo + hi) / 2, (hi - lo) / 2 * 0.9
    return (mid + amp * np.sin(t * rng.uniform(0.5, 2, width) + rng.uniform(0, 3, width)) + rng.normal(0, 0.01, (n, width))).astype(np.float32)


def dev(torch, eng, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)


def perms(M, E, N, seed):
    return np.stack([[np.random.default_rng(seed + 1000 * m + e).permutation(N) for e in range(E)] for m in range(M)]).astype(np.int32)


def unpack_state(eng, state_row):
    """The padded Adam image of one slot (per layer W as [Kp][Np], then bias [Np]; widths padded to 4) in canonical [(W, b)] form."""
    out, ofs = [], 0
    for i, o in zip(eng.dims[:-1], eng.dims[1:]):
        kp, np_ = -(-i // 4) * 4, -(-o // 4) * 4
        W = state_row[ofs:ofs + kp * np_].reshape(kp, np_)[:i, :o]
        ofs += kp * np_
        out.append((W, state_row[ofs:ofs + o]))
        ofs += np_
    return out


def ff_run(engine, torch, spec, w0s, X, Y, N, E, B, perm, adam, loss):
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    params = eng.pack_params(w0s)
    jobs = engine.jobs_to_device(engine.uniform_jobs(len(w0s), N), eng.device)
    hist, acc, (m, v) = eng.fit(params, jobs, len(w0s), N, dev(torch, eng, X), dev(torch, eng, Y), epochs=E, batch_size=B,
                                perm=dev(torch, eng, perm), adam=adam, loss=loss)
    torch.cuda.synchronize()
    return eng, eng.unpack_params(params), hist.cpu().numpy(), acc.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy()


def check_ff(lo, spec, w0s, Xs, Ys, perm, res, E, B, adam, loss, gradients=False, atol_w=0.0, n_val=0):
    """With n_val, Xs / Ys are the jobs' positions (training, then n_val held out) and res ends with val_loss / val_accuracy."""
    eng, got, hist, acc, m, v, *val = res
    for j in range(len(w0s)):
        n = len(Xs[j]) - n_val
        vsplit = n_val / len(Xs[j])
        assert math.floor(len(Xs[j]) * (1.0 - vsplit)) == n  # the oracle's split is the launch's
        w_ref, h_ref, st = lo.ff_fit(spec, w0s[j], Xs[j], Ys[j], epochs=E, batch_size=B, perms=[perm[j, e, :n] for e in range(E)],
                                     lr=adam["lr"], b1=adam["beta1"], b2=adam["beta2"], eps=adam["eps"],
                                     dtype=np.float64 if gradients else np.float32, loss=loss, validation_split=vsplit)
        for l, ((Wg, bg), (Wr, br), (W0, b0)) in enumerate(zip(got[j], w_ref, w0s[j])):
            if gradients:
                for g_, r_, z_, what in ((Wg, Wr, W0, "W"), (bg, br, b0, "b")):
                    close(g_ - z_, r_ - z_, mag=float(np.abs(r_ - z_).max()), rtol=1e-3, name=f"{loss} job {j} raw gradients {what}{l}")
            else:
                close(Wg, Wr, mag=float(np.abs(Wr).max()), atol=atol_w, name=f"{loss} job {j} W{l}")
                close(bg, br, mag=max(float(np.abs(br).max()), 1e-2), atol=atol_w, name=f"{loss} job {j} b{l}")
        if not gradients:  # Adam moments, from the kernel's padded state image
            for what, state, ref in (("m", m, st.m), ("v", v, st.v)):
                for l, ((sW, sb), (rW, rb)) in enumerate(zip(unpack_state(eng, state[j]), ref)):
                    mag = float(max(np.abs(rW).max(), np.abs(rb).max()))
                    close(sW, rW, mag=mag, rtol=1e-3, atol=1e-4 * mag, name=f"{loss} job {j} Adam {what} W{l}")
                    close(sb, rb, mag=mag, rtol=1e-3, atol=1e-4 * mag, name=f"{loss} job {j} Adam {what} b{l}")
        close(hist[j], np.array(h_ref["loss"]), mag=0.0, rtol=5e-4, name=f"{loss} job {j} loss history")
        close(acc[j], np.array(h_ref["accuracy"]), mag=0, rtol=0, atol=2.0 / n, name=f"{loss} job {j} accuracy history")
        if n_val:
            close(val[0][j], np.array(h_ref["val_loss"]), mag=0.0, rtol=5e-4, name=f"{loss} job {j} val_loss history")
            close(val[1][j], np.array(h_ref["val_accuracy"]), mag=0, rtol=0, atol=2.0 / n_val, name=f"{loss} job {j} val_accuracy history")


# (weights in L2, dz buffers in L2) of the five fit plans (tests/test_fit_plan.py pins these shapes to them)
PLANS = {"smem": ("hourglass", 64), "w_l2": ("symmetric", 10), "dz1": ("symmetric", 64), "dz2": ("symmetric", 96), "dz3": ("symmetric", 128)}


@pytest.mark.parametrize("plan,entry", crossed(PLANS, ENTRIES))
@pytest.mark.parametrize("loss", LOSSES)
def test_every_loss_in_every_memory_plan(engine, torch, km, lo, loss, plan, entry):
    """Targets 3x - 0.3 of the inputs (0.12 .. 2.3): errors on both sides of the Huber delta, negative outputs.  Targets near 0, where
    one MAPE term outweighs the rest of the batch, have their own test.  At batch 80 the last mini-batch of an epoch is partial too
    (170 = 80 + 80 + 10 rows); the split launch holds out 40 positions, one held-out batch of two chunks."""
    kind, T = PLANS[plan]
    spec = km.ff_hourglass_spec(T) if kind == "hourglass" else km.ff_symmetric_spec(T)
    split, B = entry
    M, N, E, NV = 2, 70 if B == 32 else 170, 2, 40 if split else 0
    atol_w = 0.0
    if loss in ("mae", "mape"):
        # sign(e) of an element within rounding of 0 can differ from the oracle's: two steps only.  And a gradient that is the
        # small residue of many +-100/|y| terms keeps few digits: a weight may end up to 1/50 of its two Adam steps apart.
        N, E = 2 * B, 1
        atol_w = 0.02 * KERAS_ADAM["lr"] * 2
    rng = np.random.default_rng(T)
    Xs = [waves(rng, N + NV, T) for _ in range(M)]
    Ys = [3 * x - 0.3 for x in Xs]
    w0s = [random_net(km, spec.dims, 5 + m, spec.acts)[1] for m in range(M)]
    perm = perms(M, E, N, seed=T)
    if split:
        maps = [np.random.default_rng(50 + m).permutation(N + NV) for m in range(M)]
        res = ff_split_run(engine, torch, spec, w0s, Xs, Ys, maps, NV, E, B, perm, adam=KERAS_ADAM, loss=loss)
        Xs, Ys = [x[mp] for x, mp in zip(Xs, maps)], [y[mp] for y, mp in zip(Ys, maps)]  # the gathered copies
    else:
        res = ff_run(engine, torch, spec, w0s, np.concatenate(Xs), np.concatenate(Ys), N, E, B, perm, KERAS_ADAM, loss)
    check_ff(lo, spec, w0s, Xs, Ys, perm, res, E, B, KERAS_ADAM, loss, atol_w=atol_w, n_val=NV)


@pytest.mark.parametrize("loss", LOSSES)
def test_raw_gradients(engine, torch, km, lo, loss):
    """beta1 = beta2 = 0, eps = lr = 1: the weight change of each step is ~ minus its gradient, compared to the float64 oracle."""
    spec = km.FFSpec([12, 10, 6, 10, 12], ["relu", "tanh", "sigmoid", "linear"], [0.0, 1e-3, 0.0, 0.0])
    M, N, E, B = 2, 64, 1, 32
    rng = np.random.default_rng(9)
    Xs = [waves(rng, N, 12) for _ in range(M)]
    Ys = [3 * x + 0.2 for x in Xs]  # targets away from 0 (a MAPE gradient there is 1e9), errors on both sides of 1
    w0s = [random_net(km, spec.dims, 31 + m, spec.acts)[1] for m in range(M)]
    perm = perms(M, E, N, seed=3)
    res = ff_run(engine, torch, spec, w0s, np.concatenate(Xs), np.concatenate(Ys), N, E, B, perm, GRAD_ADAM, loss)
    check_ff(lo, spec, w0s, Xs, Ys, perm, res, E, B, GRAD_ADAM, loss, gradients=True)


@pytest.mark.parametrize("loss", LOSSES)
def test_an_output_column_with_zero_error_stays_put(engine, torch, km, loss):
    """Zero kernel column and bias, zero target: the column's error is exactly 0 at every step, and f'(0) = 0 for every loss
    (sign(0) = 0 for MAE / MAPE, and yhat = 0 < eps for MSLE), so the column never moves."""
    spec = km.FFSpec([8, 5, 8], ["tanh", "linear"])
    N, E, B = 96, 3, 32
    rng = np.random.default_rng(4)
    X = waves(rng, N, 8)
    Y = X.copy()
    Y[:, 3] = 0.0
    w0 = random_net(km, spec.dims, 2, spec.acts)[1]
    w0[1][0][:, 3] = 0.0
    w0[1][1][3] = 0.0
    _, got, hist, _, _, _ = ff_run(engine, torch, spec, [w0], X, Y, N, E, B, perms(1, E, N, 8), KERAS_ADAM, loss)
    assert (got[0][1][0][:, 3] == 0).all() and got[0][1][1][3] == 0, "the zero-error column moved"
    assert not np.array_equal(got[0][1][1], w0[1][1]), "the other columns train"


def test_mape_near_zero_targets_and_msle_negative_outputs(engine, torch, km, lo):
    spec = km.FFSpec([6, 5, 6], ["tanh", "linear"])
    M, N, E, B = 2, 64, 1, 32
    rng = np.random.default_rng(12)
    Xs = [waves(rng, N, 6) for _ in range(M)]
    Ys = [x - 0.5 for x in Xs]
    Ys[0][::7, 0] = 0.0
    Ys[0][1::7, 1] = 1e-5
    w0s = [random_net(km, spec.dims, 40 + m, spec.acts)[1] for m in range(M)]
    w0s[1][1] = (w0s[1][1][0], w0s[1][1][1] - 1.0)  # machine 1: most linear outputs below 0
    perm = perms(M, E, N, seed=5)
    for loss in ("mape", "msle"):
        res = ff_run(engine, torch, spec, w0s, np.concatenate(Xs), np.concatenate(Ys), N, E, B, perm, KERAS_ADAM, loss)
        check_ff(lo, spec, w0s, Xs, Ys, perm, res, E, B, KERAS_ADAM, loss)


@pytest.mark.parametrize("plan", list(PLANS))
def test_explicit_mse_is_bit_identical_to_the_default(engine, torch, km, plan):
    kind, T = PLANS[plan]
    spec = km.ff_hourglass_spec(T) if kind == "hourglass" else km.ff_symmetric_spec(T)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    rng = np.random.default_rng(1)
    x = dev(torch, eng, np.concatenate([waves(rng, 80, T) for _ in range(2)]))
    jobs = engine.jobs_to_device(engine.uniform_jobs(2, 80), eng.device)
    w0s = [random_net(km, spec.dims, 5 + m, spec.acts)[1] for m in range(2)]
    p1, p2 = eng.pack_params(w0s), eng.pack_params(w0s)
    l1, a1, (m1, v1) = eng.fit(p1, jobs, 2, 80, x, x, epochs=2, batch_size=32, seed=3)
    l2, a2, (m2, v2) = eng.fit(p2, jobs, 2, 80, x, x, epochs=2, batch_size=32, seed=3, loss="mse")
    torch.cuda.synchronize()
    assert torch.equal(p1, p2) and torch.equal(l1, l2) and torch.equal(a1, a2) and torch.equal(m1, m2) and torch.equal(v1, v2)


# ------------------------------------------------------------------------------------------------ held-out statistics and EarlyStopping
def test_split_and_stop_report_the_loss_of_the_tail(engine, torch, km, lo):
    from gordo_components_b200.machine.model.models import EarlyStopping

    spec = km.FFSpec([8, 6, 8], ["tanh", "linear"])
    M, N, E, B, VB, vsplit = 3, 150, 6, 32, 20, 0.2
    n_train = int(math.floor(N * (1 - vsplit)))
    rng = np.random.default_rng(6)
    Xs = [waves(rng, N, 8) for _ in range(M)]
    w0s = [random_net(km, spec.dims, 60 + m, spec.acts)[1] for m in range(M)]
    perm = perms(M, E, n_train, seed=7)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    x = dev(torch, eng, np.concatenate(Xs))
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(M), n_train, np.arange(M) * N), eng.device)
    split = engine.make_split([N - n_train] * M)
    p = eng.pack_params(w0s)
    hist, _, vl, _, _ = eng.fit_split(p, jobs, M, n_train, x, x, split=split, val_batch=VB, epochs=E, batch_size=B, perm=dev(torch, eng, perm),
                                      adam=KERAS_ADAM, loss="mae")
    vl = vl.cpu().numpy()
    for j in range(M):
        _, h_ref, _ = lo.ff_fit(spec, w0s[j], Xs[j], Xs[j], epochs=E, batch_size=B, perms=[perm[j, e] for e in range(E)], validation_split=vsplit,
                                val_batch=VB, loss="mae")
        close(hist[j].cpu().numpy(), np.array(h_ref["loss"]), mag=0.0, rtol=5e-4, name=f"job {j} loss")
        close(vl[j], np.array(h_ref["val_loss"]), mag=0.0, rtol=5e-4, name=f"job {j} val_loss (MAE of the tail)")
    # the same fits with EarlyStopping(monitor="val_loss") stop where the host rule, applied to the val_loss above, says
    rules = [dict(monitor="val_loss", patience=1, min_delta=1.0), dict(monitor="val_loss", patience=2, min_delta=5e-3), dict(monitor="val_loss", patience=E)]
    p2 = eng.pack_params(w0s)
    _, _, vl2, _, ran, best, _ = eng.fit_split(p2, jobs, M, n_train, x, x, split=split, val_batch=VB, epochs=E, batch_size=B,
                                               perm=dev(torch, eng, perm), adam=KERAS_ADAM, loss="mae", stop=engine.make_stop(rules))
    ran, vl2 = ran.cpu().numpy(), vl2.cpu().numpy()
    for j, r in enumerate(rules):
        cb = EarlyStopping(**r)
        cb.reset()
        want = E
        for e in range(E):
            if cb.update(e, {"val_loss": float(vl[j, e])}, lambda: None):
                want = e + 1
                break
        assert int(ran[j]) == want, (j, ran[j], want)
        assert np.array_equal(vl2[j, :want], vl[j, :want]), "the stopping run computes the same held-out MAE"
    assert (ran < E).any()


# ------------------------------------------------------------------------------------------------ LSTM
def lstm_data(km, F, units, act, head, lookback, rows, seed):
    spec = km.LSTMSpec(F, list(units), [act] * len(units), F, head, lookback)
    rng = np.random.default_rng(seed)
    ws = []
    for i in range(len(rows)):
        layers, (Wd, bd) = km.init_lstm_weights(spec, np.random.default_rng(seed + 10 + i))
        layers = [(K, U, b + rng.uniform(-0.1, 0.1, b.shape).astype(np.float32)) for K, U, b in layers]
        ws.append((layers, (Wd, rng.uniform(-0.1, 0.1, bd.shape).astype(np.float32))))
    Xs = [rng.random((n, F)).astype(np.float32) for n in rows]
    Ys = [(3 * rng.random((n, F)) - 0.5).astype(np.float32) for n in rows]
    return spec, ws, Xs, Ys


def lstm_run(engine, torch, spec, ws, Xs, Ys, E, B, adam, loss):
    eng = engine.LSTMEngine(spec.n_features, spec.units, spec.acts, spec.n_features_out, spec.out_func, spec.lookback_window)
    rows = [len(x) for x in Xs]
    nwin = [n - spec.lookback_window + 1 for n in rows]
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(len(rows)), nwin, np.concatenate([[0], np.cumsum(rows)[:-1]])), eng.device)
    params = eng.pack_params(ws)
    hist, _, (m, v, _) = eng.fit(params, jobs, len(rows), max(nwin), dev(torch, eng, np.concatenate(Xs)), dev(torch, eng, np.concatenate(Ys)),
                                 epochs=E, batch_size=B, primer=True, adam=adam, loss=loss)
    torch.cuda.synchronize()
    return eng, params, hist.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy(), nwin


def check_lstm(km, lo, spec, ws, Xs, Ys, res, E, B, adam, loss):
    eng, params, hist, m, v, nwin = res
    got = eng.unpack_params(params)
    for i in range(len(Xs)):
        want_w, h_ref, (mr, vr) = lo.lstm_fit(spec, ws[i], Xs[i], Ys[i], epochs=E, batch_size=B, lr=adam["lr"], b1=adam["beta1"], b2=adam["beta2"],
                                              eps=adam["eps"], loss=loss)
        close(hist[i], np.array(h_ref["loss"]), rtol=5e-4, name=f"{loss} job {i} loss history")
        steps = 1 + E * math.ceil(nwin[i] / B)
        for k, (w0, gl, wl) in enumerate(zip(km._lstm_flat(ws[i]), km._lstm_flat(got[i]), km._lstm_flat(want_w))):
            close(gl - w0, wl - w0, mag=adam["lr"] * steps, rtol=2e-2, name=f"{loss} job {i} array {k}: trained weights")
        ofs = 0
        for k, (a_m, a_v) in enumerate(zip(mr, vr)):
            n = a_m.size
            for what, got_s, ref in (("m", m[i, ofs:ofs + n], a_m.ravel()), ("v", v[i, ofs:ofs + n], a_v.ravel())):
                mag = float(np.abs(ref).max())
                close(got_s, ref, mag=mag, rtol=1e-2, atol=1e-3 * mag, name=f"{loss} job {i} array {k}: Adam {what}")
            ofs += n


@pytest.mark.parametrize("loss", LOSSES)
def test_lstm_every_loss(engine, torch, km, lo, loss):
    spec, ws, Xs, Ys = lstm_data(km, 5, [6, 4], "tanh", "linear", 4, [60, 45], seed=7)
    res = lstm_run(engine, torch, spec, ws, Xs, Ys, 2, 16, KERAS_ADAM, loss)
    check_lstm(km, lo, spec, ws, Xs, Ys, res, 2, 16, KERAS_ADAM, loss)


def test_lstm_reference_test_shape_with_mae(engine, torch, km, lo):
    """tests/gordo/machine/model/test_lstm_autoencoder.py: lstm_hourglass(3, func="tanh", out_func="relu", compile_kwargs={"loss": "mae"})."""
    hg = km.lstm_hourglass_spec(3, lookback_window=5, func="tanh", out_func="relu")
    spec, ws, Xs, Ys = lstm_data(km, 3, hg.units, "tanh", "relu", 5, [70], seed=3)
    res = lstm_run(engine, torch, spec, ws, Xs, Ys, 2, 32, KERAS_ADAM, "mae")
    check_lstm(km, lo, spec, ws, Xs, Ys, res, 2, 32, KERAS_ADAM, "mae")


def test_gb_lstm_fit_is_gb_lstm_fit_loss_with_mse(engine, torch, km):
    from gordo_components_b200 import _cabi

    spec, ws, Xs, Ys = lstm_data(km, 5, [6, 4], "tanh", "linear", 4, [60, 45], seed=2)
    eng, p_loss, h_loss, m_loss, v_loss, nwin = lstm_run(engine, torch, spec, ws, Xs, Ys, 2, 16, KERAS_ADAM, "mse")
    # the same launch through the entry point without the loss argument
    p = eng.pack_params(ws)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    t = torch.zeros((2,), dtype=torch.int32, device=eng.device)
    rows = [len(x) for x in Xs]
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(2), nwin, np.concatenate([[0], np.cumsum(rows)[:-1]])), eng.device)
    hp = _cabi.GbLstmFitHParams(epochs=2, batch_size=16, lookahead=0, primer=1, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7)
    ws_t = torch.empty((eng.fit_workspace_bytes(2) + 3) // 4, dtype=torch.float32, device=eng.device)
    hist = torch.zeros((2, 2), dtype=torch.float32, device=eng.device)
    acc = torch.zeros_like(hist)
    x, y = dev(torch, eng, np.concatenate(Xs)), dev(torch, eng, np.concatenate(Ys))
    P = _cabi.ptr
    _cabi.check(eng.lib.gb_lstm_fit(C.byref(eng.net), P(p), P(m), P(v), P(t), P(jobs), 2, max(nwin), P(x), P(y), C.byref(hp), P(ws_t), P(hist), P(acc),
                                    C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert torch.equal(p, p_loss) and np.array_equal(hist.cpu().numpy(), h_loss)
    assert np.array_equal(m.cpu().numpy(), m_loss) and np.array_equal(v.cpu().numpy(), v_loss)


# ------------------------------------------------------------------------------------------------ estimators
def test_keras_autoencoder_with_huber(engine, torch, km, lo):
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    rng = np.random.default_rng(0)
    X = waves(rng, 120, 6) * 3 - 0.5
    est = KerasAutoEncoder(kind="feedforward_hourglass", compile_kwargs={"loss": "huber"}, epochs=3, batch_size=32, shuffle=False)
    est.kwargs.update({"n_features": 6, "n_features_out": 6})
    est._prepare_model()
    w0 = [(W.copy(), b.copy()) for W, b in est.model.weights]
    est.fit(X, X)
    assert est.model.spec.loss == "huber"
    spec = km.FFSpec(est.model.spec.dims, est.model.spec.acts, est.model.spec.l1)
    _, h_ref, _ = lo.ff_fit(spec, w0, X, X, epochs=3, batch_size=32, loss="huber")
    meta = est.get_metadata()["history"]
    close(meta["loss"], h_ref["loss"], mag=0.0, rtol=5e-4, name="huber history")
    back = pickle.loads(pickle.dumps(est))
    assert back.model.spec.loss == "huber" and back.get_metadata()["history"]["loss"] == meta["loss"]
    np.testing.assert_array_equal(back.predict(X), est.predict(X))


def test_estimator_per_epoch_loop_uses_the_loss(engine, torch, km, lo):
    """validation_split: the per-epoch launches and the lr = 0 held-out pass both use the compiled loss."""
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    X = waves(np.random.default_rng(1), 100, 6)
    est = KerasAutoEncoder(kind="feedforward_hourglass", compile_kwargs={"loss": "log_cosh"}, epochs=2, batch_size=16, shuffle=False,
                           validation_split=0.2)
    est.kwargs.update({"n_features": 6, "n_features_out": 6})
    est._prepare_model()
    w0 = [(W.copy(), b.copy()) for W, b in est.model.weights]
    est.fit(X, X)
    spec = km.FFSpec(est.model.spec.dims, est.model.spec.acts, est.model.spec.l1)
    _, h_ref, _ = lo.ff_fit(spec, w0, X, X, epochs=2, batch_size=16, validation_split=0.2, loss="log_cosh")
    h = est.get_metadata()["history"]
    close(h["loss"], h_ref["loss"], mag=0.0, rtol=5e-4, name="loss")
    close(h["val_loss"], h_ref["val_loss"], mag=0.0, rtol=5e-4, name="val_loss")


# ------------------------------------------------------------------------------------------------ batched builds
def _initial(fleet, eng, S, seed, torch):
    g = torch.Generator(device=eng.device).manual_seed(seed)
    return fleet._keras_initial_params(eng, S, g)


def test_build_fleet_with_mae_replays(engine, torch, km):
    from gordo_components_b200 import fleet

    spec = km.ff_hourglass_spec(8)
    M, N, K, E, B = 3, 200, 3, 3, 32
    X = np.concatenate([waves(np.random.default_rng(m), N, 8) for m in range(M)])
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    xd = dev(torch, eng, X)
    fb = fleet.build_fleet(eng, xd, xd, N, epochs=E, batch_size=B, n_splits=K, seed=3, adam=KERAS_ADAM, shuffle=False, loss="mae")
    fb_mse = fleet.build_fleet(eng, xd, xd, N, epochs=E, batch_size=B, n_splits=K, seed=3, adam=KERAS_ADAM, shuffle=False)
    torch.cuda.synchronize()
    assert not torch.equal(fb.params, fb_mse.params)
    p0 = _initial(fleet, eng, M * (K + 1), 3, torch)
    test = N // (K + 1)
    for m in range(M):
        for j, n in enumerate([N] + [N - (K - k) * test for k in range(K)]):
            slot = m if j == 0 else M + (j - 1) * M + m
            p = p0[slot:slot + 1].clone()
            jobs = engine.jobs_to_device(engine.make_jobs([0], [n], [m * N]), eng.device)
            hist, _, _ = eng.fit(p, jobs, 1, n, xd, xd, epochs=E, batch_size=B, shuffle=False, adam=KERAS_ADAM, seed=3, loss="mae")
            got_hist = fb.loss[m] if j == 0 else fb.fold_loss[m, j - 1]
            got_p = fb.params[m] if j == 0 else fb.fold_params[m, j - 1]
            assert torch.equal(got_p, p[0]) and torch.equal(got_hist, hist[0]), (m, j)


def test_build_lstm_fleet_with_huber_replays(engine, torch, km):
    from gordo_components_b200 import fleet

    M, N, K, E, B, L = 2, 160, 3, 2, 16, 5
    eng = engine.LSTMEngine(4, [5, 3], ["tanh", "tanh"], 4, "linear", L)
    X = np.concatenate([waves(np.random.default_rng(10 + m), N, 4).astype(np.float64) * 3 for m in range(M)])
    xd = torch.from_numpy(X).to(eng.device)
    fb = fleet.build_lstm_fleet(eng, xd, xd, N, epochs=E, batch_size=B, n_splits=K, seed=4, keep_init_params=True, loss="huber")
    torch.cuda.synchronize()
    x32 = xd.to(torch.float32)
    test = N // (K + 1)
    for m in range(M):
        for j, n in enumerate([N] + [N - (K - k) * test for k in range(K)]):
            slot = j * M + m
            p = fb.init_params[slot:slot + 1].clone()
            jobs = engine.jobs_to_device(engine.make_jobs([0], [n - L + 1], [m * N]), eng.device)
            hist, _, _ = eng.fit(p, jobs, 1, n - L + 1, x32, x32, epochs=E, batch_size=B, primer=True, loss="huber")
            got_p = fb.params[m] if j == 0 else fb.fold_params[m, j - 1]
            got_hist = fb.loss[m] if j == 0 else fb.fold_loss[m, j - 1]
            assert torch.equal(got_p, p[0]), (m, j, "weights")
            assert np.array_equal(got_hist, hist[0].cpu().numpy()), (m, j, "loss")


def test_build_kfold_fleet_ttr_with_log_cosh_replays(engine, torch, km):
    from sklearn.model_selection import KFold
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200 import fleet
    from gordo_components_b200.machine.model.factories.feedforward_autoencoder import feedforward_hourglass

    M, N, T, E, B, K = 2, 150, 6, 3, 32, 3
    spec = feedforward_hourglass(n_features=T, compression_factor=0.5, encoding_layers=1, func="tanh", out_func="linear",
                                 compile_kwargs={"loss": "log_cosh"})
    eng = engine.ff_engine_for(spec)
    X = np.concatenate([waves(np.random.default_rng(20 + m), N, T).astype(np.float64) * 5 for m in range(M)])
    xd = torch.from_numpy(X).to(eng.device)
    cv = KFold(K)
    fb = fleet.build_kfold_fleet(eng, xd, xd, N, cv, epochs=E, batch_size=B, seed=5, adam=spec.adam, shuffle=False, target_scaler=True,
                                 window=6, smoothing_method="smm", keep_init_params=True, loss=spec.loss)
    torch.cuda.synchronize()
    folds = list(cv.split(np.arange(N)))
    for m in range(M):
        Xm = X[m * N:(m + 1) * N]
        for j, rows in enumerate([np.arange(N)] + [tr for tr, _ in folds]):
            slot = m if j == 0 else M + (j - 1) * M + m
            xs = torch.from_numpy(Xm[rows].astype(np.float32)).to(eng.device)
            ys = torch.from_numpy(MinMaxScaler().fit(Xm[rows]).transform(Xm[rows]).astype(np.float32)).to(eng.device)
            p = fb.init_params[slot:slot + 1].clone()
            jobs = engine.jobs_to_device(engine.make_jobs([0], [len(rows)], [0]), eng.device)
            hist, _, _ = eng.fit(p, jobs, 1, len(rows), xs, ys, epochs=E, batch_size=B, shuffle=False, adam=spec.adam, seed=5, loss="log_cosh")
            assert torch.equal(fb.params[slot], p[0]), (m, j, "weights")
            assert np.array_equal(fb.loss[slot], hist[0].cpu().numpy()), (m, j, "loss")


def test_fleet_model_builder_buckets_by_loss(engine, torch, monkeypatch):
    from gordo_components_b200 import builder

    def frame(seed, rows=240, tags=5):
        idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
        return pd.DataFrame(waves(np.random.default_rng(seed), rows, tags).astype(np.float64), index=idx, columns=[f"tag-{i}" for i in range(tags)])

    def machine(name, seed, loss):
        ae = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2, "batch_size": 32,
                                                              **({"compile_kwargs": {"loss": loss}} if loss else {})}}
        return {"name": name, "model": {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": ae}},
                "dataset": {"X": frame(seed)}}

    machines = [machine("a", 1, None), machine("b", 2, "mae"), machine("c", 3, "mse"), machine("d", 4, "mean_absolute_error")]
    seen = []
    real = builder.FleetModelBuilder._build_bucket

    def spy(members):
        seen.append(sorted(c.machine["name"] for c in members))
        return real(members)

    monkeypatch.setattr(builder.FleetModelBuilder, "_build_bucket", staticmethod(spy))
    mixed = builder.FleetModelBuilder(machines).build()
    assert sorted(seen) == [["a", "c"], ["b", "d"]]
    alone = builder.FleetModelBuilder([machines[1], machines[3]]).build()  # the MAE bucket by itself: the same launch
    for (model, _), (ref, _) in zip([mixed[1], mixed[3]], alone):
        est = model.base_estimator
        assert est.model.spec.loss == "mae"
        assert est.get_metadata()["history"]["loss"] == ref.base_estimator.get_metadata()["history"]["loss"]
        for (W, b), (Wr, br) in zip(est.model.weights, ref.base_estimator.model.weights):
            assert np.array_equal(W, Wr) and np.array_equal(b, br)
    assert mixed[0][0].base_estimator.model.spec.loss == "mse"
