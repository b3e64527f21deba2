"""
The Keras optimizers on the training kernels: gb_ffae_fit_opt in every memory plan (plain launches at batches of 32 and 80 rows, and
split launches through a row map with a held-out tail), gb_lstm_fit_opt and gb_lstm_fit_tc_opt against the optimizer oracle
(tests/optimizer_oracle.py) from injected weights and visiting order, on the weights, both state slots and the history; split and stop
launches on a small stack; clipvalue on the summed gradient of a mini-batch above 32 rows; weight decay; padded lanes; per-epoch
launches equal to one launch; NULL and plain Adam equal to the Adam entry points; and the optimizer through the estimators and the
three batched fleet builds.  The stop launches in every memory plan are compared with the split ones in tests/test_gpu_fit_stop.py.
"""
import ctypes as C
import math

import numpy as np
import pandas as pd
import pytest
from optimizer_oracle import OPTIMIZERS
from parity_helpers import ENTRIES, close, crossed, ff_split_run, random_net

pytestmark = pytest.mark.gpu

KERAS_ADAM = {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7}


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
def oo(torch):
    import optimizer_oracle

    return optimizer_oracle


def opt(name, **kw):
    from gordo_components_b200.machine.model.factories.specs import resolve_optimizer

    return resolve_optimizer(name, kw)


# a larger rate than Keras' default, so that every rule moves the weights well beyond their float32 rounding in a few steps (Adadelta,
# whose steps are ~sqrt(eps / (1 - rho)) = 1.4e-3 times the rate, at the rate its users run it with)
def fast_opt(name, **kw):
    return opt(name, learning_rate=1.0 if name == "adadelta" else 0.01, **({"momentum": 0.5} if name == "rmsprop" else {}), **kw)




def waves(rng, n, width, lo=0.15, hi=0.85):
    t = np.linspace(0, 12, n)[:, None]
    mid, amp = (lo + hi) / 2, (hi - lo) / 2 * 0.9
    return (mid + amp * np.sin(t * rng.uniform(0.5, 2, width) + rng.uniform(0, 3, width)) + rng.normal(0, 0.01, (n, width))).astype(np.float32)


def dev(torch, eng, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)


def perms(M, E, N, seed):
    return np.stack([[np.random.default_rng(seed + 1000 * m + e).permutation(N) for e in range(E)] for m in range(M)]).astype(np.int32)


def unpack_state(eng, state_row):
    """The padded state image of one slot (per layer W as [Kp][Np], then bias [Np]) in canonical [(W, b)] form."""
    out, ofs = [], 0
    for i, o in zip(eng.dims[:-1], eng.dims[1:]):
        kp, np_ = -(-i // 4) * 4, -(-o // 4) * 4
        W = state_row[ofs:ofs + kp * np_].reshape(kp, np_)[:i, :o]
        ofs += kp * np_
        out.append((W, state_row[ofs:ofs + o]))
        ofs += np_
    return out


def ff_run(engine, torch, spec, w0s, X, Y, N, E, B, perm, optimizer, loss="mse"):
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    params = eng.pack_params(w0s)
    jobs = engine.jobs_to_device(engine.uniform_jobs(len(w0s), N), eng.device)
    hist, acc, (m, v) = eng.fit(params, jobs, len(w0s), N, dev(torch, eng, X), dev(torch, eng, Y), epochs=E, batch_size=B,
                                perm=dev(torch, eng, perm), loss=loss, optimizer=optimizer)
    torch.cuda.synchronize()
    return eng, eng.unpack_params(params), hist.cpu().numpy(), acc.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy()


def check_ff(oo, spec, w0s, Xs, Ys, perm, res, E, B, optimizer, loss="mse", n_val=0):
    """The tolerances of the loss tests on the weights and the history, with a wider absolute part where the rules normalise g: an
    element whose summed gradient nearly cancels carries its rounding into its step and its state at their own scale.  With n_val,
    Xs / Ys are the jobs' positions (training, then n_val held out) and res ends with val_loss / val_accuracy."""
    eng, got, hist, acc, m, v, *val = res
    for j in range(len(w0s)):
        n = len(Xs[j]) - n_val
        vsplit = n_val / len(Xs[j])
        assert math.floor(len(Xs[j]) * (1.0 - vsplit)) == n  # the oracle's split is the launch's
        w_ref, h_ref, st = oo.ff_fit(spec, w0s[j], Xs[j], Ys[j], optimizer, epochs=E, batch_size=B, perms=[perm[j, e, :n] for e in range(E)],
                                     loss=loss, validation_split=vsplit)
        for l, ((Wg, bg), (Wr, br), (W0, b0)) in enumerate(zip(got[j], w_ref, w0s[j])):
            # plus 0.5 % of the array's largest move: Adam's, Adamax's, Nadam's and RMSprop's steps are normalised, so an element whose
            # summed gradient nearly cancels moves by up to a full step in a direction its rounding decides
            close(Wg, Wr, mag=float(np.abs(Wr).max()), atol=5e-3 * float(np.abs(Wr - W0).max()), name=f"{optimizer[0]} job {j} W{l}")
            close(bg, br, mag=max(float(np.abs(br).max()), 1e-2), atol=5e-3 * float(np.abs(br - b0).max()), name=f"{optimizer[0]} job {j} b{l}")
        for what, state, ref in (("slot 0", m, st.s0), ("slot 1", v, st.s1)):
            for l, ((sW, sb), (rW, rb)) in enumerate(zip(unpack_state(eng, state[j]), ref)):
                mag = float(max(np.abs(rW).max(), np.abs(rb).max(), 1e-12))
                close(sW, rW, mag=mag, rtol=1e-3, atol=1e-2 * mag, name=f"{optimizer[0]} job {j} {what} W{l}")
                close(sb, rb, mag=mag, rtol=1e-3, atol=1e-2 * mag, name=f"{optimizer[0]} job {j} {what} b{l}")
        close(hist[j], np.array(h_ref["loss"]), mag=0.0, rtol=5e-4, name=f"{optimizer[0]} job {j} loss history")
        close(acc[j], np.array(h_ref["accuracy"]), mag=0, rtol=0, atol=2.0 / n, name=f"{optimizer[0]} job {j} accuracy history")
        if n_val:
            close(val[0][j], np.array(h_ref["val_loss"]), mag=0.0, rtol=5e-4, name=f"{optimizer[0]} job {j} val_loss history")
            close(val[1][j], np.array(h_ref["val_accuracy"]), mag=0, rtol=0, atol=2.0 / n_val, name=f"{optimizer[0]} job {j} val_accuracy history")


# (weights in L2, dz buffers in L2) of the five fit plans (tests/test_fit_plan.py pins these shapes to them)
PLANS = {"smem": ("hourglass", 64), "w_l2": ("symmetric", 10), "dz1": ("symmetric", 64), "dz2": ("symmetric", 96), "dz3": ("symmetric", 128)}


def _plan_case(km, plan, M=2, N=70, seed=0):
    kind, T = PLANS[plan]
    spec = km.ff_hourglass_spec(T) if kind == "hourglass" else km.ff_symmetric_spec(T)
    rng = np.random.default_rng(T + seed)
    Xs = [waves(rng, N, T) for _ in range(M)]
    Ys = [3 * x - 0.3 for x in Xs]
    w0s = [random_net(km, spec.dims, 5 + m + seed, spec.acts)[1] for m in range(M)]
    return spec, Xs, Ys, w0s


@pytest.mark.parametrize("plan,entry", crossed(PLANS, ENTRIES))
@pytest.mark.parametrize("name", OPTIMIZERS)
def test_every_optimizer_in_every_memory_plan(engine, torch, km, oo, name, plan, entry):
    """At batch 80 the last mini-batch of an epoch is partial too (170 = 80 + 80 + 10 rows), and clipvalue binds on the gradients the
    three chunks sum in the L2 scratch image; the split launch holds out 40 positions, one held-out batch of two chunks."""
    split, B = entry
    M, N, E, NV = 2, 70 if B == 32 else 170, 2, 40 if split else 0
    spec, Xs, Ys, w0s = _plan_case(km, plan, N=N + NV)
    if B > 32:
        # without the activity term, whose sign(a) jumps by 2 l1 where an activation lies within rounding of 0 (AdamW's second job in
        # the two-dz plan meets one 7.7e-7 from 0 at step 4): the normalised rules carry such a jump into a step-sized difference, and
        # there the float32 oracle stands as far from the float64 one as the kernel does
        spec = km.FFSpec(spec.dims, spec.acts, [0.0] * len(spec.acts))
    perm = perms(M, E, N, seed=11)
    o = fast_opt(name, **({"clipvalue": 0.02} if B > 32 else {}))
    if split:
        maps = [np.random.default_rng(50 + m).permutation(N + NV) for m in range(M)]
        res = ff_split_run(engine, torch, spec, w0s, Xs, Ys, maps, NV, E, B, perm, optimizer=o)
        Xs, Ys = [x[mp] for x, mp in zip(Xs, maps)], [y[mp] for y, mp in zip(Ys, maps)]  # the gathered copies
    else:
        res = ff_run(engine, torch, spec, w0s, np.concatenate(Xs), np.concatenate(Ys), N, E, B, perm, o)
    check_ff(oo, spec, w0s, Xs, Ys, perm, res, E, B, o, n_val=NV)


@pytest.mark.parametrize("name", OPTIMIZERS)
def test_clipvalue_and_weight_decay_on_batches_above_32_rows(engine, torch, km, oo, name):
    """Batches of 80 rows (three 32-row chunks): clipvalue binds on the summed gradient, then the decay, then the rule; and with
    the decay alone.  MAE keeps the summed output gradient well above the clip value."""
    spec = km.FFSpec([12, 8, 12], ["tanh", "linear"])
    M, N, E, B = 2, 160, 2, 80
    rng = np.random.default_rng(21)
    Xs = [waves(rng, N, 12) for _ in range(M)]
    Ys = [3 * x - 0.3 for x in Xs]
    w0s = [random_net(km, spec.dims, 70 + m, spec.acts)[1] for m in range(M)]
    perm = perms(M, E, N, seed=13)
    for kw in ({"clipvalue": 0.02, "weight_decay": 0.05}, {"weight_decay": 0.05}):
        o = opt(name, learning_rate=0.01, **kw)
        res = ff_run(engine, torch, spec, w0s, np.concatenate(Xs), np.concatenate(Ys), N, E, B, perm, o, loss="mae")
        check_ff(oo, spec, w0s, Xs, Ys, perm, res, E, B, o, loss="mae")


@pytest.mark.parametrize("name", OPTIMIZERS)
def test_a_single_raw_step(engine, torch, km, oo, name):
    """One step of 32 rows from a fresh state, against the float64 oracle: the weight change and both state slots."""
    spec = km.FFSpec([12, 10, 6, 10, 12], ["relu", "tanh", "sigmoid", "linear"], [0.0, 1e-3, 0.0, 0.0])
    M, N, E, B = 2, 32, 1, 32
    rng = np.random.default_rng(9)
    Xs = [waves(rng, N, 12) for _ in range(M)]
    Ys = [3 * x + 0.2 for x in Xs]
    w0s = [random_net(km, spec.dims, 31 + m, spec.acts)[1] for m in range(M)]
    perm = perms(M, E, N, seed=3)
    o = fast_opt(name)
    eng, got, _, _, m, v = ff_run(engine, torch, spec, w0s, np.concatenate(Xs), np.concatenate(Ys), N, E, B, perm, o)
    for j in range(M):
        w_ref, _, st = oo.ff_fit(spec, w0s[j], Xs[j], Ys[j], o, epochs=1, batch_size=B, perms=[perm[j, 0]], dtype=np.float64)
        for l, ((Wg, bg), (Wr, br), (W0, b0)) in enumerate(zip(got[j], w_ref, w0s[j])):
            for g_, r_, z_, what in ((Wg, Wr, W0, "W"), (bg, br, b0, "b")):
                close(g_ - z_, r_ - z_, mag=float(np.abs(r_ - z_).max()), rtol=1e-3, name=f"{name} job {j} step {what}{l}")
        for what, state, ref in (("slot 0", m, st.s0), ("slot 1", v, st.s1)):
            for l, ((sW, sb), (rW, rb)) in enumerate(zip(unpack_state(eng, state[j]), ref)):
                mag = float(max(np.abs(rW).max(), np.abs(rb).max(), 1e-30))
                close(sW, rW, mag=mag, rtol=1e-3, atol=1e-4 * mag, name=f"{name} job {j} {what} W{l}")
                close(sb, rb, mag=mag, rtol=1e-3, atol=1e-4 * mag, name=f"{name} job {j} {what} b{l}")


@pytest.mark.parametrize("name", OPTIMIZERS)
def test_padded_lanes_stay_zero(engine, torch, km, name):
    """The 10-tag symmetric stack keeps its weight image in the slot's state area (the w_l2 plan): after a fit with decay and
    clipping, every padded lane of the image is still exactly 0, and the rest is the trained parameter vector."""
    kind, T = PLANS["w_l2"]
    spec = km.ff_symmetric_spec(T)
    assert any(d % 4 for d in spec.dims)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    rng = np.random.default_rng(2)
    w0s = [random_net(km, spec.dims, 3, spec.acts)[1]]
    p = eng.pack_params(w0s)
    x = dev(torch, eng, waves(rng, 90, T))
    jobs = engine.jobs_to_device(engine.uniform_jobs(1, 90), eng.device)
    o = opt(name, learning_rate=0.01, weight_decay=0.1, clipvalue=0.5)
    _, _, (m, _) = eng.fit(p, jobs, 1, 90, x, x, epochs=3, batch_size=40, shuffle=False, optimizer=o)
    torch.cuda.synchronize()
    wfloats = eng.state_stride // 3
    image = m[0, 2 * wfloats:].cpu().numpy()
    ofs = 0
    trained = eng.unpack_params(p)[0]
    for (i, o_), (W, b) in zip(zip(spec.dims[:-1], spec.dims[1:]), trained):
        kp, np_ = -(-i // 4) * 4, -(-o_ // 4) * 4
        Wi = image[ofs:ofs + kp * np_].reshape(kp, np_)
        ofs += kp * np_
        bi = image[ofs:ofs + np_]
        ofs += np_
        assert (Wi[i:, :] == 0).all() and (Wi[:, o_:] == 0).all() and (bi[o_:] == 0).all(), f"{name}: a padded lane moved"
        assert np.array_equal(Wi[:i, :o_], W) and np.array_equal(bi[:o_], b)


@pytest.mark.parametrize("name", OPTIMIZERS)
def test_per_epoch_launches_equal_one_launch(engine, torch, km, name):
    """Three launches of one epoch, the state and step count carried, are the three-epoch launch bit for bit (Nadam's product
    recomputed from step 1, Adagrad's first step read once)."""
    spec = km.FFSpec([8, 6, 8], ["tanh", "linear"])
    N, E, B = 96, 3, 32
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    X = waves(np.random.default_rng(5), N, 8)
    x = dev(torch, eng, X)
    w0s = [random_net(km, spec.dims, 8, spec.acts)[1]]
    perm = perms(1, E, N, seed=4)
    jobs = engine.jobs_to_device(engine.uniform_jobs(1, N), eng.device)
    o = fast_opt(name)
    p1 = eng.pack_params(w0s)
    h1, _, (m1, v1) = eng.fit(p1, jobs, 1, N, x, x, epochs=E, batch_size=B, perm=dev(torch, eng, perm), optimizer=o)
    p2 = eng.pack_params(w0s)
    state, h2 = None, []
    for e in range(E):
        h, _, state = eng.fit(p2, jobs, 1, N, x, x, epochs=1, batch_size=B, perm=dev(torch, eng, perm[:, e:e + 1]), optimizer=o, state=state,
                              step0=e * (N // B))
        h2.append(h[0, 0].item())
    torch.cuda.synchronize()
    assert torch.equal(p1, p2) and torch.equal(m1, state[0]) and torch.equal(v1, state[1])
    assert h1[0].cpu().numpy().tolist() == h2


def test_split_and_stop_with_another_optimizer(engine, torch, km, oo):
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
    o = opt("RMSprop", learning_rate=0.01, centered=True)
    p = eng.pack_params(w0s)
    hist, _, vl, _, _ = eng.fit_split(p, jobs, M, n_train, x, x, split=split, val_batch=VB, epochs=E, batch_size=B, perm=dev(torch, eng, perm),
                                      optimizer=o)
    vl = vl.cpu().numpy()
    for j in range(M):
        _, h_ref, _ = oo.ff_fit(spec, w0s[j], Xs[j], Xs[j], o, epochs=E, batch_size=B, perms=[perm[j, e] for e in range(E)],
                                validation_split=vsplit, val_batch=VB)
        close(hist[j].cpu().numpy(), np.array(h_ref["loss"]), mag=0.0, rtol=5e-4, name=f"job {j} loss")
        close(vl[j], np.array(h_ref["val_loss"]), mag=0.0, rtol=5e-4, name=f"job {j} val_loss")
    rules = [dict(monitor="val_loss", patience=1, min_delta=1.0), dict(monitor="val_loss", patience=2, min_delta=5e-3), dict(monitor="val_loss", patience=E)]
    p2 = eng.pack_params(w0s)
    _, _, vl2, _, ran, _, _ = eng.fit_split(p2, jobs, M, n_train, x, x, split=split, val_batch=VB, epochs=E, batch_size=B,
                                            perm=dev(torch, eng, perm), optimizer=o, stop=engine.make_stop(rules))
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
        assert np.array_equal(vl2[j, :want], vl[j, :want])
    assert (ran < E).any()
    assert torch.equal(p[2], p2[2]), "the job that never stops ends where the split launch ends"


def test_null_and_plain_adam_are_the_adam_entry_points(engine, torch, km):
    from gordo_components_b200 import _cabi

    spec = km.ff_hourglass_spec(16)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    N, NV = 100, 20
    # each job's 20 held-out positions are rows of its own after its N training rows, so no launch reads past x
    x = dev(torch, eng, np.concatenate([waves(np.random.default_rng(m), N + NV, 16) for m in range(2)]))
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(2), N, np.arange(2) * (N + NV)), eng.device)
    w0s = [random_net(km, spec.dims, 5 + m, spec.acts)[1] for m in range(2)]
    split = engine.jobs_to_device(engine.make_split([NV, NV]), eng.device)
    stop = engine.jobs_to_device(engine.make_stop([dict(monitor="val_loss", patience=1)] * 2), eng.device)
    hp = engine._fit_hparams(3, 32, True, None, KERAS_ADAM, 7, False, 0, "huber")
    P = _cabi.ptr
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    plain = _cabi.make_optimizer(*opt("Adam"))

    def run(entry, optimizer, use_split, use_stop):
        p = eng.pack_params(w0s)
        m, v = eng._fit_state(p, None)
        out = [torch.full((2, 3), float("nan"), device=eng.device) for _ in range(4)]
        best, ran, be = torch.zeros_like(p), torch.zeros(2, dtype=torch.int32, device=eng.device), torch.zeros(2, dtype=torch.int32, device=eng.device)
        common = (C.byref(eng.net), P(p), P(m), P(v), P(jobs))
        sp = P(split) if use_split else None
        st = (P(stop), P(best), P(ran), P(be)) if use_stop else (None, None, None, None)
        if entry == "stop":
            rc = eng.lib.gb_ffae_fit_stop(*common, sp, 2, N, P(x), P(x), None, None, C.byref(hp), 20, *(P(t) for t in out), *st, stream)
        elif entry == "fit":
            rc = eng.lib.gb_ffae_fit(*common, 2, N, P(x), P(x), None, C.byref(hp), P(out[0]), P(out[1]), stream)
        elif entry == "split":
            rc = eng.lib.gb_ffae_fit_split(*common, sp, 2, N, P(x), P(x), None, None, C.byref(hp), 20, *(P(t) for t in out), stream)
        else:
            rc = eng.lib.gb_ffae_fit_opt(*common, sp, 2, N, P(x), P(x), None, None, C.byref(hp), 20, *(P(t) for t in out), *st,
                                         None if optimizer is None else C.byref(optimizer), stream)
        _cabi.check(rc)
        torch.cuda.synchronize()
        return [p, m, v, *out, ran]

    def same(a, b):
        return all(torch.equal(torch.nan_to_num(s, nan=-7.0), torch.nan_to_num(t, nan=-7.0)) for s, t in zip(a, b))

    for optimizer in (None, plain):
        assert same(run("stop", None, True, True), run("opt", optimizer, True, True))
        assert same(run("split", None, True, False), run("opt", optimizer, True, False))
        assert same(run("fit", None, False, False), run("opt", optimizer, False, False))
    # the plain Adam of another rate follows that rate, not hp's
    fast = _cabi.make_optimizer(*opt("Adam", learning_rate=0.01))
    assert not same(run("fit", None, False, False), run("opt", fast, False, False))


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


def lstm_run(engine, torch, spec, ws, Xs, Ys, E, B, optimizer, loss="mse", family="fp32"):
    eng = engine.LSTMEngine(spec.n_features, spec.units, spec.acts, spec.n_features_out, spec.out_func, spec.lookback_window)
    rows = [len(x) for x in Xs]
    nwin = [n - spec.lookback_window + 1 for n in rows]
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(len(rows)), nwin, np.concatenate([[0], np.cumsum(rows)[:-1]])), eng.device)
    params = eng.pack_params(ws)
    fit = eng.fit if family == "fp32" else eng.fit_tc
    hist, _, (m, v, t) = fit(params, jobs, len(rows), max(nwin), dev(torch, eng, np.concatenate(Xs)), dev(torch, eng, np.concatenate(Ys)),
                             epochs=E, batch_size=B, primer=True, loss=loss, optimizer=optimizer)
    torch.cuda.synchronize()
    return eng, params, hist.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy(), nwin, t.cpu().numpy()


def check_lstm(km, oo, spec, ws, Xs, Ys, res, E, B, optimizer, loss="mse"):
    eng, params, hist, m, v, nwin, t = res
    got = eng.unpack_params(params)
    lr = optimizer[1]["lr"]  # the loss tests' tolerances: the change on the scale of lr x steps
    for i in range(len(Xs)):
        want_w, h_ref, st = oo.lstm_fit(spec, ws[i], Xs[i], Ys[i], optimizer, epochs=E, batch_size=B, loss=loss)
        steps = 1 + E * math.ceil(nwin[i] / B)
        assert int(t[i]) == steps == st.t
        close(hist[i], np.array(h_ref["loss"]), rtol=5e-4, name=f"{optimizer[0]} job {i} loss history")
        for k, (w0, gl, wl) in enumerate(zip(km._lstm_flat(ws[i]), km._lstm_flat(got[i]), km._lstm_flat(want_w))):
            close(gl - w0, wl - w0, mag=lr * steps, rtol=2e-2, name=f"{optimizer[0]} job {i} array {k}: trained weights")
        ofs = 0
        for k, (a0, a1) in enumerate(zip(st.s0, st.s1)):
            n = a0.size
            for what, got_s, ref in (("slot 0", m[i, ofs:ofs + n], a0.ravel()), ("slot 1", v[i, ofs:ofs + n], a1.ravel())):
                mag = float(max(np.abs(ref).max(), 1e-30))
                close(got_s, ref, mag=mag, rtol=1e-2, atol=1e-2 * mag, name=f"{optimizer[0]} job {i} array {k}: {what}")
            ofs += n


@pytest.mark.parametrize("family,batch", [("fp32", 16), ("tc", 64), ("tc", 256)])
@pytest.mark.parametrize("name", OPTIMIZERS)
def test_lstm_every_optimizer(engine, torch, km, oo, name, family, batch):
    rows = [60, 45] if batch <= 32 else [batch + 40, batch // 2 + 20]
    spec, ws, Xs, Ys = lstm_data(km, 5, [6, 4], "tanh", "linear", 4, rows, seed=7)
    o = fast_opt(name)
    res = lstm_run(engine, torch, spec, ws, Xs, Ys, 2, batch, o, family=family)
    check_lstm(km, oo, spec, ws, Xs, Ys, res, 2, batch, o)


def test_lstm_reference_test_shape_with_rmsprop(engine, torch, km, oo):
    """tests/gordo/machine/model/test_lstm_autoencoder.py's lstm_hourglass(3, out_func="relu", loss mae), with RMSprop(0.02, momentum
    0.001) for its SGD: the factory's spec trained against the oracle, and the estimator built and trained from the definition."""
    from gordo_components_b200.machine.model.factories import lstm_autoencoder as lsa
    from gordo_components_b200.machine.model.factories.specs import fit_optimizer
    from gordo_components_b200.machine.model.models import KerasLSTMAutoEncoder

    kw = dict(func="tanh", out_func="relu", compile_kwargs={"loss": "mae"}, optimizer="RMSprop",
              optimizer_kwargs={"learning_rate": 0.02, "momentum": 0.001})
    fs = lsa.lstm_hourglass(3, lookback_window=5, **kw)
    o = fit_optimizer(fs)
    assert o[0] == "rmsprop" and o[1]["momentum"] == 0.001 and fs.loss == "mae"
    spec, ws, Xs, Ys = lstm_data(km, 3, fs.lstm_units, "tanh", "relu", 5, [70], seed=3)
    res = lstm_run(engine, torch, spec, ws, Xs, Ys, 2, 32, o, loss="mae")
    check_lstm(km, oo, spec, ws, Xs, Ys, res, 2, 32, o, loss="mae")
    est = KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=5, epochs=2, batch_size=32, **kw)
    est.fit(Xs[0], Xs[0])
    assert est.model.spec.optimizer == "rmsprop"
    assert all(np.isfinite(est.get_metadata()["history"]["loss"]))


# ------------------------------------------------------------------------------------------------ estimators
@pytest.mark.parametrize("name,vsplit", [("nadam", 0.0), ("adagrad", 0.2), ("adamw", 0.0)])
def test_keras_autoencoder_with_an_optimizer(engine, torch, km, oo, name, vsplit):
    """The one-launch fit and (validation_split) the per-epoch fit with its lr-0 held-out pass."""
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    X = waves(np.random.default_rng(1), 100, 6) * 3 - 0.5
    est = KerasAutoEncoder(kind="feedforward_hourglass", optimizer=name, optimizer_kwargs={"learning_rate": 0.01}, epochs=3, batch_size=16,
                           shuffle=False, validation_split=vsplit)
    est.kwargs.update({"n_features": 6, "n_features_out": 6})
    est._prepare_model()
    w0 = [(W.copy(), b.copy()) for W, b in est.model.weights]
    est.fit(X, X)
    s = est.model.spec
    spec = km.FFSpec(s.dims, s.acts, s.l1)
    w_ref, h_ref, _ = oo.ff_fit(spec, w0, X, X, (s.optimizer, s.optimizer_config), epochs=3, batch_size=16, validation_split=vsplit)
    h = est.get_metadata()["history"]
    close(h["loss"], h_ref["loss"], mag=0.0, rtol=5e-4, name="loss")
    if vsplit:
        close(h["val_loss"], h_ref["val_loss"], mag=0.0, rtol=5e-4, name="val_loss")
    for l, ((Wg, bg), (Wr, br)) in enumerate(zip(est.model.weights, w_ref)):
        close(Wg, Wr, mag=float(np.abs(Wr).max()), atol=1e-4, name=f"W{l}")


def test_detector_with_an_optimizer(engine, torch):
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    idx = pd.date_range("2019-01-01", periods=240, freq="10min", tz="UTC")
    X = pd.DataFrame(waves(np.random.default_rng(3), 240, 5).astype(np.float64), index=idx, columns=list("abcde"))
    det = DiffBasedAnomalyDetector(base_estimator=KerasAutoEncoder(kind="feedforward_hourglass", optimizer="Adamax", epochs=2, batch_size=32),
                                   require_thresholds=False)
    det.fit(X, X)
    assert det.base_estimator.model.spec.optimizer == "adamax"
    out = det.anomaly(X, X)
    assert np.isfinite(out["total-anomaly-scaled"].to_numpy()).all()


# ------------------------------------------------------------------------------------------------ batched builds
def _initial(fleet, eng, S, seed, torch):
    g = torch.Generator(device=eng.device).manual_seed(seed)
    return fleet._keras_initial_params(eng, S, g)


def test_build_fleet_with_nadam_replays(engine, torch, km):
    from gordo_components_b200 import fleet

    spec = km.ff_hourglass_spec(8)
    M, N, K, E, B = 3, 200, 3, 3, 32
    X = np.concatenate([waves(np.random.default_rng(m), N, 8) for m in range(M)])
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    xd = dev(torch, eng, X)
    o = opt("Nadam", learning_rate=0.005, weight_decay=0.01)
    fb = fleet.build_fleet(eng, xd, xd, N, epochs=E, batch_size=B, n_splits=K, seed=3, shuffle=False, optimizer=o)
    torch.cuda.synchronize()
    p0 = _initial(fleet, eng, M * (K + 1), 3, torch)
    test = N // (K + 1)
    for m in range(M):
        for j, n in enumerate([N] + [N - (K - k) * test for k in range(K)]):
            slot = m if j == 0 else M + (j - 1) * M + m
            p = p0[slot:slot + 1].clone()
            jobs = engine.jobs_to_device(engine.make_jobs([0], [n], [m * N]), eng.device)
            hist, _, _ = eng.fit(p, jobs, 1, n, xd, xd, epochs=E, batch_size=B, shuffle=False, seed=3, optimizer=o)
            got_hist = fb.loss[m] if j == 0 else fb.fold_loss[m, j - 1]
            got_p = fb.params[m] if j == 0 else fb.fold_params[m, j - 1]
            assert torch.equal(got_p, p[0]) and torch.equal(got_hist, hist[0]), (m, j)


def test_build_lstm_fleet_with_adadelta_replays(engine, torch, km):
    from gordo_components_b200 import fleet

    M, N, K, E, B, L = 2, 160, 3, 2, 16, 5
    eng = engine.LSTMEngine(4, [5, 3], ["tanh", "tanh"], 4, "linear", L)
    X = np.concatenate([waves(np.random.default_rng(10 + m), N, 4).astype(np.float64) * 3 for m in range(M)])
    xd = torch.from_numpy(X).to(eng.device)
    o = opt("Adadelta", learning_rate=1.0)
    fb = fleet.build_lstm_fleet(eng, xd, xd, N, epochs=E, batch_size=B, n_splits=K, seed=4, keep_init_params=True, optimizer=o)
    torch.cuda.synchronize()
    x32 = xd.to(torch.float32)
    test = N // (K + 1)
    for m in range(M):
        for j, n in enumerate([N] + [N - (K - k) * test for k in range(K)]):
            slot = j * M + m
            p = fb.init_params[slot:slot + 1].clone()
            jobs = engine.jobs_to_device(engine.make_jobs([0], [n - L + 1], [m * N]), eng.device)
            hist, _, _ = eng.fit(p, jobs, 1, n - L + 1, x32, x32, epochs=E, batch_size=B, primer=True, optimizer=o)
            got_p = fb.params[m] if j == 0 else fb.fold_params[m, j - 1]
            got_hist = fb.loss[m] if j == 0 else fb.fold_loss[m, j - 1]
            assert torch.equal(got_p, p[0]), (m, j, "weights")
            assert np.array_equal(got_hist, hist[0].cpu().numpy()), (m, j, "loss")


def test_build_kfold_fleet_with_rmsprop_replays(engine, torch, km):
    from sklearn.model_selection import KFold
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200 import fleet
    from gordo_components_b200.machine.model.factories.feedforward_autoencoder import feedforward_hourglass
    from gordo_components_b200.machine.model.factories.specs import fit_optimizer

    M, N, T, E, B, K = 2, 150, 6, 3, 32, 3
    spec = feedforward_hourglass(n_features=T, compression_factor=0.5, encoding_layers=1, func="tanh", out_func="linear",
                                 optimizer="rmsprop", optimizer_kwargs={"momentum": 0.3, "clipvalue": 0.05})
    o = fit_optimizer(spec)
    eng = engine.ff_engine_for(spec)
    X = np.concatenate([waves(np.random.default_rng(20 + m), N, T).astype(np.float64) * 5 for m in range(M)])
    xd = torch.from_numpy(X).to(eng.device)
    cv = KFold(K)
    fb = fleet.build_kfold_fleet(eng, xd, xd, N, cv, epochs=E, batch_size=B, seed=5, adam=spec.adam, shuffle=False, target_scaler=True,
                                 window=6, smoothing_method="smm", keep_init_params=True, optimizer=o)
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
            hist, _, _ = eng.fit(p, jobs, 1, len(rows), xs, ys, epochs=E, batch_size=B, shuffle=False, adam=spec.adam, seed=5, optimizer=o)
            assert torch.equal(fb.params[slot], p[0]), (m, j, "weights")
            assert np.array_equal(fb.loss[slot], hist[0].cpu().numpy()), (m, j, "loss")


def test_fleet_model_builder_mixes_adam_rmsprop_and_nadam(engine, torch, monkeypatch):
    """One project, three optimizers: three buckets, and each bucket trains as it does alone."""
    from gordo_components_b200 import builder

    def frame(seed, rows=192, tags=5):
        idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
        return pd.DataFrame(waves(np.random.default_rng(seed), rows, tags).astype(np.float64), index=idx, columns=[f"tag-{i}" for i in range(tags)])

    def machine(name, seed, optimizer):
        ae = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2, "batch_size": 32,
                                                              **({"optimizer": optimizer, "optimizer_kwargs": {"learning_rate": 0.01}} if optimizer else {})}}
        return {"name": name, "model": {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": ae}},
                "dataset": {"X": frame(seed)}}

    machines = [machine("a", 1, None), machine("b", 2, "RMSprop"), machine("c", 3, "Nadam"), machine("d", 4, "rmsprop")]
    seen = []
    real = builder.FleetModelBuilder._build_bucket

    def spy(members):
        seen.append(sorted(c.machine["name"] for c in members))
        return real(members)

    monkeypatch.setattr(builder.FleetModelBuilder, "_build_bucket", staticmethod(spy))
    mixed = builder.FleetModelBuilder(machines).build()
    assert sorted(seen) == [["a"], ["b", "d"], ["c"]]
    names = {"a": "adam", "b": "rmsprop", "c": "nadam", "d": "rmsprop"}
    for (model, _), mach in zip(mixed, machines):
        s = model.base_estimator.model.spec
        assert s.optimizer == names[mach["name"]] and (s.optimizer_config is None) == (mach["name"] == "a")
    for group in ([machines[1], machines[3]], [machines[2]], [machines[0]]):
        alone = builder.FleetModelBuilder(group).build()
        for (ref, _), mach in zip(alone, group):
            est = mixed[machines.index(mach)][0].base_estimator
            assert est.get_metadata()["history"]["loss"] == ref.base_estimator.get_metadata()["history"]["loss"]
            for (W, b), (Wr, br) in zip(est.model.weights, ref.base_estimator.model.weights):
                assert np.array_equal(W, Wr) and np.array_equal(b, br)
