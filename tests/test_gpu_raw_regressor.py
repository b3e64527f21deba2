"""
Weight regularizers in the Dense fit kernel (gb_ffae_fit_reg) and KerasRawModelRegressor on the GPU.

The kernel runs against a float64 restatement of Keras' regularized fit: the loss oracle's forward pass and gradients
(tests/loss_oracle.py) and the optimizer oracle's update rules (tests/optimizer_oracle.py), with the penalty
sum_l kernel_l1 sum|W| + kernel_l2 sum W^2 + bias_l1 sum|b| + bias_l2 sum b^2 of the step's weights added to every mini-batch loss
and its gradient l1 sign(w) + 2 l2 w to every step's summed gradient.  Weights and visiting order are injected, so the two fits
take the same steps.  Then the estimator end to end, and the fleet builder against the per-machine fit.
"""
import ctypes as C

import numpy as np
import pytest
from parity_helpers import close

import loss_oracle as lo
import optimizer_oracle as oo

pytestmark = pytest.mark.gpu

ADAM = ("adam", {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7, "weight_decay": 0.0, "clipvalue": None})


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


def waves(rng, n, width):
    t = np.linspace(0, 12, n)[:, None]
    return (0.5 + 0.3 * np.sin(t * rng.uniform(0.5, 2, width) + rng.uniform(0, 3, width)) + rng.normal(0, 0.01, (n, width))).astype(np.float32)


def penalty(flat, reg):
    out = 0.0
    for l in range(len(flat) // 2):
        W, b = flat[2 * l], flat[2 * l + 1]
        out += reg["kernel_l1"][l] * np.abs(W).sum() + reg["kernel_l2"][l] * (W * W).sum()
        out += reg["bias_l1"][l] * np.abs(b).sum() + reg["bias_l2"][l] * (b * b).sum()
    return float(out)


def reg_grads(flat, reg):
    g = []
    for l in range(len(flat) // 2):
        W, b = flat[2 * l], flat[2 * l + 1]
        g += [reg["kernel_l1"][l] * np.sign(W) + 2 * reg["kernel_l2"][l] * W, reg["bias_l1"][l] * np.sign(b) + 2 * reg["bias_l2"][l] * b]
    return g


def oracle_fit(spec, weights, X, y, reg, optimizer=ADAM, epochs=1, batch_size=32, perms=None, n_val=0, val_batch=None, loss="mse", stop=None):
    """Keras' fit with kernel / bias regularizers in float64.  ``stop``: (patience,) of EarlyStopping(monitor='val_loss')."""
    d = np.float64
    X, y = np.asarray(X, d), np.asarray(y, d)
    n = len(X) - n_val
    Xv, yv = X[n:], y[n:]
    flat = [np.asarray(a, d).copy() for W, b in weights for a in (W, b)]
    st = oo.OptState(flat, d)
    pairs = lambda a: [(a[2 * i], a[2 * i + 1]) for i in range(len(a) // 2)]  # noqa: E731
    hist = {"loss": [], "val_loss": []}
    best, wait = np.inf, 0
    for e in range(epochs):
        order = np.asarray(perms[e])[:n] if perms is not None else np.arange(n)
        ls = 0.0
        for s in range(0, n, batch_size):
            idx = order[s:s + batch_size]
            l_, _, grads, _ = lo.ff_loss_and_grads(spec, pairs(flat), X[idx], y[idx], d, False, loss)
            ls += (float(l_) + penalty(flat, reg)) * len(idx)
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
                v = hist["val_loss"][-1]
                wait += 1
                if v < best:
                    best, wait = v, 0
                elif wait >= stop[0] and e > 0:
                    break
    return pairs(flat), hist


def reg_record(L, kernel_l1=0.0, kernel_l2=0.0, bias_l1=0.0, bias_l2=0.0):
    return {"kernel_l1": [kernel_l1] * L, "kernel_l2": [kernel_l2] * L, "bias_l1": [bias_l1] * L, "bias_l2": [bias_l2] * L}


def gpu_fit(engine, torch, spec, w0s, Xs, Ys, reg, epochs, batch, perm, optimizer=None, loss="mse", n_val=0, stop=None):
    """One launch over len(Xs) jobs (slot j = job j); ``n_val`` held-out tail rows per job (fit_split), ``stop`` a patience."""
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    params = eng.pack_params(w0s)
    N = len(Xs[0])
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)  # noqa: E731
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(len(Xs)), [N - n_val] * len(Xs), np.arange(len(Xs)) * N), eng.device)
    perm = np.pad(perm, ((0, 0), (0, 0), (0, N - perm.shape[2])))  # [n_jobs][epochs][max_rows]: a job's order in its first n_rows entries
    kw = dict(epochs=epochs, batch_size=batch, perm=dev(perm), loss=loss, optimizer=optimizer, reg=reg)
    x, y = dev(np.concatenate(Xs)), dev(np.concatenate(Ys))
    if n_val or stop is not None:
        stops = None if stop is None else engine.make_stop([{"monitor": "val_loss", "patience": stop[0]}] * len(Xs))
        out = eng.fit_split(params, jobs, len(Xs), N, x, y, split=engine.make_split([n_val] * len(Xs)), stop=stops, **kw)
        hist, val = out[0], out[2]
    else:
        hist, _, _ = eng.fit(params, jobs, len(Xs), N, x, y, **kw)
        val = None
    torch.cuda.synchronize()
    return eng.unpack_params(params), hist.cpu().numpy(), None if val is None else val.cpu().numpy()


def check(got, want, loss, hist, name, val=None, E=None):
    for l, ((Wg, bg), (Wr, br)) in enumerate(zip(got, want)):
        close(Wg, Wr, mag=float(np.abs(Wr).max()), name=f"{name} W{l}")
        close(bg, br, mag=max(float(np.abs(br).max()), 1e-2), name=f"{name} b{l}")
    E = E or len(hist["loss"])
    close(loss[:E], np.array(hist["loss"]), mag=0.0, rtol=5e-4, name=f"{name} loss history")
    if val is not None:
        close(val[:E], np.array(hist["val_loss"]), mag=0.0, rtol=5e-4, name=f"{name} val_loss history")


def perms_for(M, E, N, seed):
    return np.stack([[np.random.default_rng(seed + 100 * m + e).permutation(N) for e in range(E)] for m in range(M)]).astype(np.int32)


def case_data(km, dims, M, N, seed, acts=None):
    spec = km.FFSpec(list(dims), acts or ["tanh"] * (len(dims) - 2) + ["linear"])
    rng = np.random.default_rng(seed)
    Xs = [waves(rng, N, dims[0]) for _ in range(M)]
    Ys = Xs if dims[0] == dims[-1] else [waves(rng, N, dims[-1]) for _ in range(M)]
    w0s = []
    for m in range(M):
        w = km.init_ff_weights(spec, np.random.default_rng(seed + m))
        w0s.append([(W, np.random.default_rng(seed + 50 + m).uniform(-0.2, 0.2, b.shape).astype(np.float32)) for W, b in w])
    return spec, Xs, Ys, w0s


# ------------------------------------------------------------------------------------------------ the penalty terms
REGS = {
    "kernel_l1": dict(kernel_l1=0.01),
    "kernel_l2": dict(kernel_l2=0.05),
    "kernel_l1l2": dict(kernel_l1=0.01, kernel_l2=0.02),
    "bias": dict(bias_l1=0.02, bias_l2=0.1),
    "everything": dict(kernel_l1=0.005, kernel_l2=0.01, bias_l1=0.01, bias_l2=0.05),
}


@pytest.mark.parametrize("batch", [32, 80])
@pytest.mark.parametrize("case", list(REGS))
def test_penalty_terms_match_the_oracle(engine, torch, km, case, batch):
    M, N, E = 2, 160, 2
    spec, Xs, Ys, w0s = case_data(km, [10, 7, 5, 7, 10], M, N, seed=3)
    reg = reg_record(spec.n_layers, **REGS[case])
    perm = perms_for(M, E, N, 7)
    got, loss, _ = gpu_fit(engine, torch, spec, w0s, Xs, Ys, reg, E, batch, perm)
    for j in range(M):
        want, hist = oracle_fit(spec, w0s[j], Xs[j], Ys[j], reg, epochs=E, batch_size=batch, perms=perm[j])
        check(got[j], want, loss[j], hist, f"{case} job {j}")
    assert hist["loss"][0] > oracle_fit(spec, w0s[0], Xs[0], Ys[0], reg_record(spec.n_layers), epochs=1, batch_size=batch, perms=perm[0])[1]["loss"][0]


PLAN_CASES = {  # (weights in L2, dz buffers in L2) -> stack, as the coverage tests choose them
    "shared": ((0, 0), "hourglass", 64),
    "weights_in_l2": ((1, 0), "symmetric", 10),
    "one_dz_in_l2": ((1, 1), "symmetric", 64),
    "two_dz_in_l2": ((1, 2), "symmetric", 96),
    "three_dz_in_l2": ((1, 3), "symmetric", 128),
}


@pytest.mark.parametrize("case", list(PLAN_CASES))
def test_every_memory_plan(engine, torch, km, case):
    from gordo_components_b200 import _cabi

    want_plan, kind, T = PLAN_CASES[case]
    spec = km.ff_hourglass_spec(T) if kind == "hourglass" else km.ff_symmetric_spec(T)
    net = _cabi.make_ffnet(spec.dims, spec.acts, spec.l1)
    w, dz = C.c_int32(-1), C.c_int32(-1)
    assert _cabi.load_library().gb_ffae_fit_plan(C.byref(net), C.byref(w), C.byref(dz)) == 0 and (w.value, dz.value) == want_plan
    M, N, E, B = 2, 120, 2, 50
    rng = np.random.default_rng(T)
    Xs = [waves(rng, N, T) for _ in range(M)]
    w0s = [km.init_ff_weights(spec, np.random.default_rng(60 + m)) for m in range(M)]
    reg = reg_record(spec.n_layers, kernel_l1=1e-3, kernel_l2=5e-3, bias_l1=1e-3, bias_l2=1e-2)
    perm = perms_for(M, E, N, 17)
    got, loss, _ = gpu_fit(engine, torch, spec, w0s, Xs, Xs, reg, E, B, perm)
    for j in range(M):
        want, hist = oracle_fit(spec, w0s[j], Xs[j], Xs[j], reg, epochs=E, batch_size=B, perms=perm[j])
        check(got[j], want, loss[j], hist, f"{case} job {j}")


def test_another_loss_and_optimizer_with_clipvalue(engine, torch, km):
    M, N, E, B = 2, 150, 2, 40
    spec, Xs, Ys, w0s = case_data(km, [9, 6, 4], M, N, seed=21, acts=["relu", "linear"])
    reg = reg_record(spec.n_layers, kernel_l1=0.02, kernel_l2=0.03, bias_l2=0.05)
    opt = oo.resolve("rmsprop", learning_rate=3e-3, clipvalue=0.05)
    perm = perms_for(M, E, N, 5)
    got, loss, _ = gpu_fit(engine, torch, spec, w0s, Xs, Ys, reg, E, B, perm, optimizer=opt, loss="huber")
    for j in range(M):
        want, hist = oracle_fit(spec, w0s[j], Xs[j], Ys[j], reg, optimizer=opt, epochs=E, batch_size=B, perms=perm[j], loss="huber")
        check(got[j], want, loss[j], hist, f"rmsprop/huber job {j}")


def test_held_out_loss_carries_the_penalty(engine, torch, km):
    M, N, E, B, V = 2, 140, 3, 32, 30
    spec, Xs, Ys, w0s = case_data(km, [8, 6, 8], M, N, seed=31)
    reg = reg_record(spec.n_layers, kernel_l2=0.05, bias_l1=0.01)
    perm = perms_for(M, E, N - V, 9)
    got, loss, val = gpu_fit(engine, torch, spec, w0s, Xs, Ys, reg, E, B, perm, n_val=V)
    for j in range(M):
        want, hist = oracle_fit(spec, w0s[j], Xs[j], Ys[j], reg, epochs=E, batch_size=B, perms=perm[j], n_val=V)
        check(got[j], want, loss[j], hist, f"split job {j}", val=val[j])
        bare = oracle_fit(spec, w0s[j], Xs[j], Ys[j], reg_record(spec.n_layers), epochs=1, batch_size=B, perms=perm[j], n_val=V)[1]
        assert val[j, 0] > bare["val_loss"][0]


def test_early_stopping_on_val_loss(engine, torch, km):
    M, N, E, B, V = 2, 120, 8, 32, 24
    spec, Xs, Ys, w0s = case_data(km, [6, 4, 6], M, N, seed=41)
    reg = reg_record(spec.n_layers, kernel_l2=0.5)  # a heavy penalty: val_loss turns up within a few epochs
    opt = oo.resolve("adam", learning_rate=0.05)
    perm = perms_for(M, E, N - V, 3)
    got, loss, val = gpu_fit(engine, torch, spec, w0s, Xs, Ys, reg, E, B, perm, optimizer=opt, n_val=V, stop=(1,))
    for j in range(M):
        want, hist = oracle_fit(spec, w0s[j], Xs[j], Ys[j], reg, optimizer=opt, epochs=E, batch_size=B, perms=perm[j], n_val=V, stop=(1,))
        ran = len(hist["loss"])
        check(got[j], want, loss[j], hist, f"stop job {j}", val=val[j], E=ran)
        assert np.isnan(loss[j, ran:]).all()


def test_weights_at_zero_under_l1_stay_there(engine, torch, km):
    """sign(0) = 0: a weight at exactly 0 whose loss gradient is 0 (its input column is 0) feels no L1 pull and stays exactly 0."""
    M, N, E, B = 1, 96, 2, 32
    spec, Xs, Ys, w0s = case_data(km, [6, 5, 6], M, N, seed=51)
    Xs = [x.copy() for x in Xs]
    Xs[0][:, 0] = 0.0
    (W0, b0), rest = w0s[0][0], w0s[0][1:]
    W0 = W0.copy()
    W0[0, :] = 0.0
    W0[1, 2] = 0.0  # a zero weight with a live input: the loss moves it off 0
    w0s = [[(W0, b0), *rest]]
    reg = reg_record(spec.n_layers, kernel_l1=0.1)
    perm = perms_for(M, E, N, 1)
    got, loss, _ = gpu_fit(engine, torch, spec, w0s, Xs, Ys, reg, E, B, perm)
    assert (got[0][0][0][0, :] == 0.0).all()
    assert got[0][0][0][1, 2] != 0.0
    want, hist = oracle_fit(spec, w0s[0], Xs[0], Ys[0], reg, epochs=E, batch_size=B, perms=perm[0])
    check(got[0], want, loss[0], hist, "zeros")


@pytest.mark.parametrize("split", [False, True])
def test_a_null_or_zero_record_is_gb_ffae_fit_opt(engine, torch, km, split):
    from gordo_components_b200 import _cabi

    M, N, E, B = 2, 100, 2, 40
    spec, Xs, Ys, w0s = case_data(km, [12, 8, 12], M, N, seed=61)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    lib = _cabi.load_library()
    p = _cabi.ptr
    x, y = (torch.from_numpy(np.concatenate(a)).to(eng.device) for a in (Xs, Ys))
    jobs = engine.jobs_to_device(engine.uniform_jobs(M, N - 20 * split), eng.device)
    splits = engine.jobs_to_device(engine.make_split([20 * split] * M), eng.device) if split else None
    hp = engine._fit_hparams(E, B, True, None, None, 5, False, 0, "mse")
    results = []
    for rec in ("opt", None, _cabi.make_dense_reg(), _cabi.make_dense_reg(kernel_l1=[0.0] * 2)):
        params = eng.pack_params(w0s)
        m, v = eng._fit_state(params, None)
        out = [torch.full((M, E), float("nan"), device=eng.device) for _ in range(4)]
        args = (C.byref(eng.net), p(params), p(m), p(v), p(jobs), p(splits), M, N, p(x), p(y), None, None, C.byref(hp), B,
                *(p(t) for t in out), None, None, None, None, None)
        if rec == "opt":
            _cabi.check(lib.gb_ffae_fit_opt(*args, None))
        else:
            _cabi.check(lib.gb_ffae_fit_reg(*args, None if rec is None else C.byref(rec), None))
        torch.cuda.synchronize()
        results.append([params.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy()] + [t.cpu().numpy() for t in out])
    for other in results[1:]:
        for a, b in zip(results[0], other):
            assert np.array_equal(a, b, equal_nan=True)


# ------------------------------------------------------------------------------------------------ the estimator
def raw_kind(n_out, reg="l2", input_shape=None, metrics=None):
    first = {"units": 6, "activation": "tanh", "kernel_regularizer": reg}
    if input_shape:
        first["input_shape"] = [input_shape]
    comp = {"loss": "mse", "optimizer": "adam"}
    if metrics:
        comp["metrics"] = metrics
    return {"compile": comp, "spec": {"tensorflow.keras.models.Sequential": {"layers": [
        {"tensorflow.keras.layers.Dense": first},
        {"tensorflow.keras.layers.Dense": {"units": n_out, "bias_regularizer": {"tensorflow.keras.regularizers.L1L2": {"l1": 0.01, "l2": 0.01}}}}]}}}


def test_fit_predict_score(torch, km):
    from gordo_components_b200.machine.model.models import KerasRawModelRegressor

    np.random.seed(0)
    rng = np.random.default_rng(1)
    X = waves(rng, 300, 5)
    y = X[:, :1] * 0.5 + 0.2
    model = KerasRawModelRegressor(raw_kind(1, input_shape=5), epochs=3)
    w0 = None
    model.kwargs.update(n_features=5, n_features_out=1)
    model._prepare_model()
    w0 = [(W.copy(), b.copy()) for W, b in model.model.weights]
    model.fit(X, y, shuffle=False)
    assert list(model._history.history) == ["loss"] and len(model._history.history["loss"]) == 3
    spec = km.FFSpec([5, 6, 1], ["tanh", "linear"])
    reg = {"kernel_l1": [0.0, 0.0], "kernel_l2": [0.01, 0.0], "bias_l1": [0.0, 0.01], "bias_l2": [0.0, 0.01]}
    want, hist = oracle_fit(spec, w0, X, y, reg, epochs=3, batch_size=32)
    check(model.model.weights, want, np.array(model._history.history["loss"]), hist, "estimator")
    out = model.predict(X)
    assert out.shape == (300, 1)
    np.testing.assert_allclose(out, km.ff_forward(spec, model.model.weights, X), rtol=1e-4, atol=1e-5)
    from sklearn.metrics import explained_variance_score

    assert model.score(X, y) == pytest.approx(explained_variance_score(y, out))
    with pytest.raises(ValueError, match="does not match the 4 features"):
        KerasRawModelRegressor(raw_kind(1, input_shape=5)).fit(X[:, :4], y)


def test_inside_a_detector_and_a_pipeline(torch):
    import pandas as pd
    import yaml
    from sklearn.model_selection import TimeSeriesSplit

    from gordo_components_b200 import serializer
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasRawModelRegressor

    rng = np.random.default_rng(2)
    idx = pd.date_range("2020-01-01", periods=400, freq="10min", tz="UTC")
    X = pd.DataFrame(waves(rng, 400, 4), index=idx, columns=[f"in-{i}" for i in range(4)])
    y = pd.DataFrame(X.values[:, :1] * 0.8 + 0.1, index=idx, columns=["target"])
    det = DiffBasedAnomalyDetector(base_estimator=KerasRawModelRegressor(raw_kind(1), epochs=2))
    cv = det.cross_validate(X=X, y=y, cv=TimeSeriesSplit(n_splits=3))
    assert len(cv["estimator"]) == 3 and all(type(e.base_estimator) is KerasRawModelRegressor for e in cv["estimator"])
    det.fit(X, y)
    out = det.anomaly(X, y)
    assert np.isfinite(out["total-anomaly-scaled"].values).all() and out["model-output"].shape == (400, 1)

    pipe = serializer.from_definition(yaml.safe_load("""
    sklearn.pipeline.Pipeline:
      steps:
        - sklearn.decomposition.PCA:
            n_components: 4
        - gordo.machine.model.models.KerasRawModelRegressor:
            kind:
              compile: {loss: mse, optimizer: adam}
              spec:
                tensorflow.keras.models.Sequential:
                  layers:
                    - tensorflow.keras.layers.Dense: {units: 4, input_shape: [4]}
                    - tensorflow.keras.layers.Dense:
                        units: 1
                        kernel_regularizer: {tensorflow.keras.regularizers.L1L2: {l1: 0.2}}
    """))
    for m in range(2):  # one pipeline per machine
        Xm, ym = np.random.default_rng(m).random((100, 4)), np.random.default_rng(10 + m).random((100, 1))
        pipe.fit(Xm, ym)
        assert pipe.predict(Xm).shape == (100, 1)


def test_fleet_builder_matches_the_per_machine_fit(engine, torch, km, tmp_path):
    import pandas as pd

    from gordo_components_b200 import builder, fleet
    from gordo_components_b200.machine.model.factories.specs import fit_reg
    from gordo_components_b200.machine.model.models import KerasRawModelRegressor

    T, N, M, E = 4, 200, 3, 2
    k = raw_kind(T)
    rng = np.random.default_rng(5)
    frames = [waves(rng, N, T) for _ in range(M)]
    proto = KerasRawModelRegressor(k)
    proto.kwargs.update(n_features=T, n_features_out=T)
    spec = proto._build_spec()
    eng = engine.ff_engine_for(spec)
    x = torch.from_numpy(np.concatenate(frames)).to(eng.device)
    fb = fleet.build_fleet(eng, x, x, N, epochs=E, batch_size=32, shuffle=False, keep_init_params=True, reg=fit_reg(spec))
    torch.cuda.synchronize()
    for m in range(M):  # slot m is machine m's final fit on all its rows
        est = KerasRawModelRegressor(k, n_features=T, n_features_out=T)
        est.set_weights(eng.unpack_params(fb.init_params[m:m + 1])[0])
        est.fit(frames[m], frames[m], epochs=E, shuffle=False)
        got = eng.unpack_params(fb.params[m:m + 1])[0]
        for l, ((Wg, bg), (Wr, br)) in enumerate(zip(got, est.model.weights)):
            close(Wg, Wr, mag=float(np.abs(Wr).max()), name=f"machine {m} W{l}")
            close(bg, br, mag=max(float(np.abs(br).max()), 1e-2), name=f"machine {m} b{l}")
        close(fb.loss[m].cpu().numpy(), np.array(est._history.history["loss"]), mag=0.0, rtol=5e-4, name=f"machine {m} loss")

    # a project of raw and hourglass machines: one batched bucket per network, each machine's metadata shaped as ModelBuilder's
    idx = pd.date_range("2020-01-01", periods=N, freq="10min", tz="UTC")
    raw_est = {"gordo.machine.model.models.KerasRawModelRegressor": {"kind": k, "epochs": E}}
    hg_est = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": E}}
    machines = []
    for i, est in enumerate((raw_est, raw_est, hg_est, hg_est)):
        frame = pd.DataFrame(frames[i % M].astype(np.float64), index=idx, columns=[f"tag-{c}" for c in range(T)])
        machines.append({"name": f"m-{i}", "dataset": {"X": frame, "y": frame},
                         "model": {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": est}}})
    calls = []
    orig = builder.FleetModelBuilder._build_bucket
    builder.FleetModelBuilder._build_bucket = staticmethod(lambda members: calls.append(len(members)) or orig(members))
    try:
        out = builder.FleetModelBuilder(machines).build(str(tmp_path))
    finally:
        builder.FleetModelBuilder._build_bucket = staticmethod(orig)
    assert sorted(calls) == [2, 2]
    for i in (0, 2):
        single_model, single_meta = builder.ModelBuilder(dict(machines[i])).build()
        model, meta = out[i]
        assert type(model.base_estimator) is type(single_model.base_estimator)
        hist = meta["metadata"]["build_metadata"]["model"]["model_meta"]["history"]
        want = single_meta["metadata"]["build_metadata"]["model"]["model_meta"]["history"]
        assert list(hist) == list(want)
        assert list(meta["metadata"]["build_metadata"]["model"]["cross_validation"]["scores"]) == \
            list(single_meta["metadata"]["build_metadata"]["model"]["cross_validation"]["scores"])


def test_kfold_fleet_builder_reports_the_loss_alone_without_metrics(engine, torch, monkeypatch):
    """A raw regressor compiled without metrics: its K-fold detector's History has the loss (and val_loss) only, batched as per
    machine."""
    import pandas as pd

    from gordo_components_b200 import builder

    T, N = 4, 300
    idx = pd.date_range("2020-01-01", periods=N, freq="10min", tz="UTC")
    frame = pd.DataFrame(waves(np.random.default_rng(7), N, T), index=idx, columns=[f"tag-{c}" for c in range(T)])
    est = {"gordo.machine.model.models.KerasRawModelRegressor": {"kind": raw_kind(T), "epochs": 2, "validation_split": 0.2}}
    machine = {"name": "raw-kfold", "dataset": {"X": frame, "y": frame}, "evaluation": {"cv": {"sklearn.model_selection.KFold": {"n_splits": 3}}},
               "model": {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {"base_estimator": est}}}
    calls = []
    orig = builder.FleetModelBuilder._build_bucket
    monkeypatch.setattr(builder.FleetModelBuilder, "_build_bucket", staticmethod(lambda members: calls.append(len(members)) or orig(members)))
    batched, batched_meta = builder.FleetModelBuilder([dict(machine)], kfcv=True).build()[0]
    assert calls == [1]
    single, single_meta = builder.ModelBuilder(dict(machine)).build()
    for meta in (batched_meta, single_meta):
        assert list(meta["metadata"]["build_metadata"]["model"]["model_meta"]["history"]) == ["loss", "val_loss", "params"]
    assert batched.base_estimator._history.params == single.base_estimator._history.params


def test_every_regularized_kernel_instantiation_runs(engine, torch):
    """The nine ffae_fit_reg_kernel<WG, DG, SPLIT, STOP> a record reaches, one per (memory plan group, entry point), read back from
    torch.profiler; the same launches without a record reach the MSE-Adam ffae_fit_kernel, never a regularized one."""
    import re

    from test_fit_plan import PLAN_SHAPES
    from torch.profiler import ProfilerActivity, profile

    groups = {(False, False): (0, 0), (True, False): (1, 0), (True, True): (1, 1)}
    entries = {"fit": (False, False), "split": (True, False), "stop": (True, True)}
    expected = {g + e for g in groups for e in entries.values()}
    N, NV = 40, 8
    torch.cuda.synchronize()
    # every cell twice: after a long run of other tests in the same process, the records of a profiling session's first launches
    # were seen to go missing, and the census is about which kernels the dispatch reaches, not about one launch
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for plan in [*groups.values()] * 2:
            spec = PLAN_SHAPES[plan]
            eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
            x = torch.from_numpy(np.random.default_rng(0).random((N + NV, spec.dims[0]), dtype=np.float32)).to(eng.device)
            jobs = engine.jobs_to_device(engine.make_jobs([0], [N], [0]), eng.device)
            for reg in (reg_record(spec.n_layers, kernel_l1=1e-3, bias_l2=1e-3), reg_record(spec.n_layers)):
                for entry in entries:
                    p = torch.zeros((1, eng.param_stride), dtype=torch.float32, device=eng.device)
                    if entry == "fit":
                        eng.fit(p, jobs, 1, N, x, x, epochs=1, batch_size=32, reg=reg)
                    else:
                        stop = engine.make_stop([{"monitor": "loss", "patience": 1}]) if entry == "stop" else None
                        eng.fit_split(p, jobs, 1, N, x, x, split=engine.make_split([NV]), stop=stop, epochs=1, batch_size=32, reg=reg)
        torch.cuda.synchronize()
    keys = [e.key for e in prof.key_averages()]
    if not any("ffae_fit" in k for k in keys):
        pytest.skip("the profiler lists no kernels here")

    def flags(name, kernel):
        m = re.search(kernel + r"<([^>]*)>", name)
        if m:
            return tuple(a.strip() in ("true", "(bool)1") for a in m.group(1).split(","))
        m = re.search(kernel + r"I((?:Lb[01]E)+)", name)
        return tuple(b == "1" for b in re.findall(r"Lb([01])E", m.group(1))) if m else None

    reg_seen = {flags(k, "ffae_fit_reg_kernel") for k in keys if "ffae_fit_reg_kernel" in k}
    plain_seen = {flags(k, "ffae_fit_kernel") for k in keys if "ffae_fit_kernel" in k}
    assert reg_seen == expected, (sorted(expected - reg_seen), sorted(reg_seen - expected))
    assert plain_seen == {e + (False, False) for e in expected}
