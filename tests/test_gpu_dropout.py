"""
Dropout in the Dense fit kernel (gb_ffae_fit_drop) and in KerasRawModelRegressor on the GPU.

The kernel runs against tests/dropout_oracle.py: Keras' fit with Dropout in float64, drawing its masks from a NumPy restatement
of the generator include/gordo_b200.h documents, with kernel / bias regularizers where a case has them.  Weights and visiting
order are injected, so the two fits take the same steps under the same masks.  Then the launch-level identities (one E-epoch
launch against E one-epoch launches; a NULL or all-zero record against gb_ffae_fit_reg), the kernel census, the estimator end to
end and the fleet builder.
"""
import ctypes as C

import numpy as np
import pytest
from parity_helpers import close

import dropout_oracle as do
import optimizer_oracle as oo

pytestmark = pytest.mark.gpu

SEED = 20261018


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


def reg_record(L, **kw):
    return {k: [kw.get(k, 0.0)] * L for k in ("kernel_l1", "kernel_l2", "bias_l1", "bias_l2")}


def gpu_fit(engine, torch, spec, w0s, Xs, Ys, rates, epochs, batch, perm, reg=None, optimizer=None, n_val=0, stop=None):
    """One launch over len(Xs) jobs (slot j = job j) with hp.seed SEED; ``n_val`` held-out tail rows per job, ``stop`` (monitor,
    patience) of an EarlyStopping rule."""
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    params = eng.pack_params(w0s)
    N = len(Xs[0])
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)  # noqa: E731
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(len(Xs)), [N - n_val] * len(Xs), np.arange(len(Xs)) * N), eng.device)
    perm = np.pad(perm, ((0, 0), (0, 0), (0, N - perm.shape[2])))
    kw = dict(epochs=epochs, batch_size=batch, perm=dev(perm), optimizer=optimizer, reg=reg, dropout=rates, seed=SEED)
    x, y = dev(np.concatenate(Xs)), dev(np.concatenate(Ys))
    ran = None
    if n_val or stop is not None:
        stops = None if stop is None else engine.make_stop([{"monitor": stop[0], "patience": stop[1]}] * len(Xs))
        out = eng.fit_split(params, jobs, len(Xs), N, x, y, split=engine.make_split([n_val] * len(Xs)), stop=stops, **kw)
        hist, val = out[0], out[2]
        if stop is not None:
            ran = out[4].cpu().numpy()
    else:
        hist, _, _ = eng.fit(params, jobs, len(Xs), N, x, y, **kw)
        val = None
    torch.cuda.synchronize()
    return eng.unpack_params(params), hist.cpu().numpy(), None if val is None else val.cpu().numpy(), ran


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


# ------------------------------------------------------------------------------------------------ rates and placements
RATES = {  # rates on the inputs of the four layers of [10, 7, 5, 7, 10]
    "hidden_0.1": [0.0, 0.1, 0.0, 0.0],
    "hidden_0.5": [0.0, 0.0, 0.5, 0.0],
    "input": [0.2, 0.0, 0.0, 0.0],
    "two_boundaries": [0.0, 0.3, 0.0, 0.5],
    "everywhere": [0.1, 0.5, 0.25, 0.1],
}


@pytest.mark.parametrize("batch", [32, 80])
@pytest.mark.parametrize("case", list(RATES))
def test_rates_and_placements_match_the_oracle(engine, torch, km, case, batch):
    M, N, E = 2, 160, 2
    spec, Xs, Ys, w0s = case_data(km, [10, 7, 5, 7, 10], M, N, seed=3)
    rates = RATES[case]
    perm = perms_for(M, E, N, 7)
    got, loss, _, _ = gpu_fit(engine, torch, spec, w0s, Xs, Ys, rates, E, batch, perm)
    for j in range(M):
        want, hist, _ = do.fit(spec, w0s[j], Xs[j], Ys[j], rates, seed=SEED, slot=j, epochs=E, batch_size=batch, perms=perm[j])
        check(got[j], want, loss[j], hist, f"{case} job {j}")
    # the masks matter: the undropped fit is another fit
    bare = do.fit(spec, w0s[0], Xs[0], Ys[0], [0.0] * 4, epochs=E, batch_size=batch, perms=perm[0])[1]
    assert abs(loss[0, 0] - bare["loss"][0]) > 1e-3 * bare["loss"][0]


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
    # every hidden boundary but the output of a layer with an activity L1 (the encoder's first layer here), which is refused
    rates = [0.1] + [0.0 if spec.l1[l - 1] else 0.2 if l % 2 else 0.4 for l in range(1, spec.n_layers)]
    assert sum(r > 0 for r in rates) >= 3
    perm = perms_for(M, E, N, 17)
    got, loss, _, _ = gpu_fit(engine, torch, spec, w0s, Xs, Xs, rates, E, B, perm)
    for j in range(M):
        want, hist, _ = do.fit(spec, w0s[j], Xs[j], Xs[j], rates, seed=SEED, slot=j, epochs=E, batch_size=B, perms=perm[j])
        check(got[j], want, loss[j], hist, f"{case} job {j}")


def test_with_weight_regularizers_and_another_optimizer(engine, torch, km):
    M, N, E, B = 2, 150, 2, 40
    spec, Xs, Ys, w0s = case_data(km, [9, 6, 4], M, N, seed=21, acts=["relu", "linear"])
    reg = reg_record(spec.n_layers, kernel_l2=0.03, bias_l2=0.05)
    rates = [0.1, 0.3]
    opt = oo.resolve("rmsprop", learning_rate=3e-3)
    perm = perms_for(M, E, N, 5)
    for optimizer in (None, opt):
        got, loss, _, _ = gpu_fit(engine, torch, spec, w0s, Xs, Ys, rates, E, B, perm, reg=reg, optimizer=optimizer)
        for j in range(M):
            want, hist, _ = do.fit(spec, w0s[j], Xs[j], Ys[j], rates, seed=SEED, slot=j, reg=reg, optimizer=optimizer, epochs=E,
                                   batch_size=B, perms=perm[j])
            check(got[j], want, loss[j], hist, f"l2 {optimizer and optimizer[0]} job {j}")


def test_the_held_out_loss_is_undropped(engine, torch, km):
    M, N, E, B, V = 2, 140, 3, 32, 30
    spec, Xs, Ys, w0s = case_data(km, [8, 6, 8], M, N, seed=31)
    rates = [0.2, 0.5]
    perm = perms_for(M, E, N - V, 9)
    got, loss, val, _ = gpu_fit(engine, torch, spec, w0s, Xs, Ys, rates, E, B, perm, n_val=V)
    for j in range(M):
        want, hist, _ = do.fit(spec, w0s[j], Xs[j], Ys[j], rates, seed=SEED, slot=j, epochs=E, batch_size=B, perms=perm[j], n_val=V)
        check(got[j], want, loss[j], hist, f"split job {j}", val=val[j])


def test_early_stopping_on_the_dropped_loss(engine, torch, km):
    M, N, E, B = 2, 96, 10, 32
    spec, Xs, Ys, w0s = case_data(km, [6, 8, 6], M, N, seed=41)
    rates = [0.0, 0.5]
    opt = oo.resolve("adam", learning_rate=0.05)
    perm = perms_for(M, E, N, 3)
    got, loss, _, ran = gpu_fit(engine, torch, spec, w0s, Xs, Ys, rates, E, B, perm, optimizer=opt, stop=("loss", 1))
    stopped = 0
    for j in range(M):
        want, hist, _ = do.fit(spec, w0s[j], Xs[j], Ys[j], rates, seed=SEED, slot=j, optimizer=opt, epochs=E, batch_size=B, perms=perm[j],
                               stop=("loss", 1))
        n = len(hist["loss"])
        assert ran[j] == n
        check(got[j], want, loss[j], hist, f"stop job {j}", E=n)
        assert np.isnan(loss[j, n:]).all()
        stopped += n < E
    assert stopped >= 1  # the noisy dropped loss turns up: at least one job stops early


# ------------------------------------------------------------------------------------------------ launch-level identities
def test_one_launch_equals_epoch_launches_with_step0_carried(engine, torch, km):
    """The masks are keyed by the absolute step: E one-epoch launches that carry step0 and the optimizer state (sequential order,
    the same seed) draw the masks of one E-epoch launch and end bit-identical."""
    M, N, E, B = 2, 100, 3, 40
    spec, Xs, Ys, w0s = case_data(km, [8, 6, 4, 6, 8], M, N, seed=71)
    rates = [0.2, 0.3, 0.0, 0.5]
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    x, y = (torch.from_numpy(np.concatenate(a)).to(eng.device) for a in (Xs, Ys))
    jobs = engine.jobs_to_device(engine.uniform_jobs(M, N), eng.device)
    one = eng.pack_params(w0s)
    loss1, _, (m1, v1) = eng.fit(one, jobs, M, N, x, y, epochs=E, batch_size=B, shuffle=False, seed=SEED, dropout=rates)
    many = eng.pack_params(w0s)
    state, step0, losses = None, 0, []
    for e in range(E):
        l_, _, state = eng.fit(many, jobs, M, N, x, y, epochs=1, batch_size=B, shuffle=False, seed=SEED, state=state, step0=step0,
                               dropout=rates)
        losses.append(l_.cpu().numpy()[:, 0])
        step0 += -(-N // B)
    torch.cuda.synchronize()
    assert np.array_equal(one.cpu().numpy(), many.cpu().numpy())
    assert np.array_equal(m1.cpu().numpy(), state[0].cpu().numpy()) and np.array_equal(v1.cpu().numpy(), state[1].cpu().numpy())
    assert np.array_equal(loss1.cpu().numpy(), np.stack(losses, axis=1))
    want, hist, _ = do.fit(spec, w0s[1], Xs[1], Ys[1], rates, seed=SEED, slot=1, epochs=E, batch_size=B)
    check(eng.unpack_params(one)[1], want, loss1.cpu().numpy()[1], hist, "one launch")


@pytest.mark.parametrize("split", [False, True])
def test_a_null_or_zero_record_is_gb_ffae_fit_reg(engine, torch, km, split):
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
    for reg in (None, _cabi.make_dense_reg(kernel_l2=[0.01, 0.02])):
        results = []
        for rec in ("reg", None, _cabi.make_dense_dropout(), _cabi.make_dense_dropout([0.0, 0.0])):
            params = eng.pack_params(w0s)
            m, v = eng._fit_state(params, None)
            out = [torch.full((M, E), float("nan"), device=eng.device) for _ in range(4)]
            args = (C.byref(eng.net), p(params), p(m), p(v), p(jobs), p(splits), M, N, p(x), p(y), None, None, C.byref(hp), B,
                    *(p(t) for t in out), None, None, None, None, None, None if reg is None else C.byref(reg))
            if rec == "reg":
                _cabi.check(lib.gb_ffae_fit_reg(*args, None))
            else:
                _cabi.check(lib.gb_ffae_fit_drop(*args, None if rec is None else C.byref(rec), None))
            torch.cuda.synchronize()
            results.append([params.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy()] + [t.cpu().numpy() for t in out])
        for other in results[1:]:
            for a, b in zip(results[0], other):
                assert np.array_equal(a, b, equal_nan=True)


def test_every_dropout_kernel_instantiation_runs(engine, torch):
    """The nine ffae_fit_drop_kernel<WG, DG, SPLIT, STOP> a record reaches, one per (memory plan group, entry point), read back from
    torch.profiler; the same launches with all-zero rates reach the MSE-Adam ffae_fit_kernel, never a dropout one."""
    import re

    from test_fit_plan import PLAN_SHAPES
    from torch.profiler import ProfilerActivity, profile

    groups = {(False, False): (0, 0), (True, False): (1, 0), (True, True): (1, 1)}
    entries = {"fit": (False, False), "split": (True, False), "stop": (True, True)}
    expected = {g + e for g in groups for e in entries.values()}
    N, NV = 40, 8
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for plan in [*groups.values()] * 2:  # every cell twice, as the regularized census does
            spec = PLAN_SHAPES[plan]
            eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
            x = torch.from_numpy(np.random.default_rng(0).random((N + NV, spec.dims[0]), dtype=np.float32)).to(eng.device)
            jobs = engine.jobs_to_device(engine.make_jobs([0], [N], [0]), eng.device)
            for rates in ([0.1] + [0.0] * (spec.n_layers - 1), [0.0] * spec.n_layers):
                for entry in entries:
                    p = torch.zeros((1, eng.param_stride), dtype=torch.float32, device=eng.device)
                    if entry == "fit":
                        eng.fit(p, jobs, 1, N, x, x, epochs=1, batch_size=32, dropout=rates)
                    else:
                        stop = engine.make_stop([{"monitor": "loss", "patience": 1}]) if entry == "stop" else None
                        eng.fit_split(p, jobs, 1, N, x, x, split=engine.make_split([NV]), stop=stop, epochs=1, batch_size=32, dropout=rates)
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

    drop_seen = {flags(k, "ffae_fit_drop_kernel") for k in keys if "ffae_fit_drop_kernel" in k}
    plain_seen = {flags(k, "ffae_fit_kernel") for k in keys if "ffae_fit_kernel" in k}
    assert drop_seen == expected, (sorted(expected - drop_seen), sorted(drop_seen - expected))
    assert plain_seen == {e + (False, False) for e in expected}


# ------------------------------------------------------------------------------------------------ the estimator and the fleet
def raw_kind(n_out, input_shape=None, rate=0.3, input_rate=0.1):
    first = {"units": 6, "activation": "tanh"}
    layers = [{"tensorflow.keras.layers.Dropout": {"rate": input_rate, "seed": 11}}] if input_rate else []
    if input_shape:
        (layers[0]["tensorflow.keras.layers.Dropout"] if layers else first)["input_shape"] = [input_shape]
    layers += [{"tensorflow.keras.layers.Dense": first}, {"tensorflow.keras.layers.Dropout": {"rate": rate}},
               {"tensorflow.keras.layers.Dense": {"units": n_out, "kernel_regularizer": "l2"}}]
    return {"compile": {"loss": "mse", "optimizer": "adam"}, "spec": {"tensorflow.keras.models.Sequential": {"layers": layers}}}


def test_fit_and_an_undropped_predict(torch, km):
    from gordo_components_b200.machine.model.models import KerasRawModelRegressor

    rng = np.random.default_rng(1)
    X = waves(rng, 300, 5)
    y = X[:, :1] * 0.5 + 0.2
    model = KerasRawModelRegressor(raw_kind(1, input_shape=5), epochs=3)
    model.kwargs.update(n_features=5, n_features_out=1)
    model._prepare_model()
    assert model.model.spec.dropout == [0.1, 0.3]
    w0 = [(W.copy(), b.copy()) for W, b in model.model.weights]
    np.random.seed(4)
    seed = int(np.random.randint(0, 2**31 - 1))  # what fit draws from numpy's global state for the launch's seed
    np.random.seed(4)
    model.fit(X, y, shuffle=False)
    spec = km.FFSpec([5, 6, 1], ["tanh", "linear"])
    reg = {"kernel_l1": [0.0, 0.0], "kernel_l2": [0.0, 0.01], "bias_l1": [0.0, 0.0], "bias_l2": [0.0, 0.0]}
    want, hist, _ = do.fit(spec, w0, X, y, [0.1, 0.3], seed=seed, slot=0, reg=reg, epochs=3, batch_size=32)
    check(model.model.weights, want, np.array(model._history.history["loss"]), hist, "estimator")
    out = model.predict(X)
    np.testing.assert_allclose(out, km.ff_forward(spec, model.model.weights, X), rtol=1e-4, atol=1e-5)
    assert np.array_equal(out, model.predict(X))  # no mask in inference: the same rows give the same outputs


def test_the_fleet_builder_matches_the_oracle_under_each_slot_key(engine, torch, km, tmp_path):
    import pandas as pd

    from gordo_components_b200 import builder, fleet
    from gordo_components_b200.machine.model.factories.specs import fit_dropout, fit_reg
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
    fb = fleet.build_fleet(eng, x, x, N, epochs=E, batch_size=32, shuffle=False, seed=SEED, keep_init_params=True, reg=fit_reg(spec),
                           dropout=fit_dropout(spec))
    torch.cuda.synchronize()
    ospec = km.FFSpec(spec.dims, spec.acts)
    for m in range(M):  # slot m is machine m's final fit on all its rows
        w0 = eng.unpack_params(fb.init_params[m:m + 1])[0]
        want, hist, _ = do.fit(ospec, w0, frames[m], frames[m], fit_dropout(spec), seed=SEED, slot=m, reg=fit_reg(spec), epochs=E)
        check(eng.unpack_params(fb.params[m:m + 1])[0], want, fb.loss[m].cpu().numpy(), hist, f"machine {m}")

    # a project of dropout and plain raw machines: one batched bucket per network, each machine's metadata shaped as ModelBuilder's
    plain = raw_kind(T, rate=0.0, input_rate=0.0)
    idx = pd.date_range("2020-01-01", periods=N, freq="10min", tz="UTC")
    machines = []
    for i, kd in enumerate((k, k, plain, plain)):
        frame = pd.DataFrame(frames[i % M].astype(np.float64), index=idx, columns=[f"tag-{c}" for c in range(T)])
        est = {"gordo.machine.model.models.KerasRawModelRegressor": {"kind": kd, "epochs": E}}
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
        assert type(model.base_estimator) is KerasRawModelRegressor
        assert model.base_estimator.model.spec.dropout == single_model.base_estimator.model.spec.dropout
        hist = meta["metadata"]["build_metadata"]["model"]["model_meta"]["history"]
        want = single_meta["metadata"]["build_metadata"]["model"]["model_meta"]["history"]
        assert list(hist) == list(want) and np.isfinite(hist["loss"]).all()
