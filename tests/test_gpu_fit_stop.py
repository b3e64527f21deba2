"""
gb_ffae_fit_stop on the H100: Keras' EarlyStopping applied by every job at the end of each epoch, inside the fit launch.

- A rule that never fires gives gb_ffae_fit_split's results, bit for bit, in every memory plan.
- Jobs that stop after different epochs in one launch end with the weights of a launch of that many epochs (or, restoring, of
  their snapshot's epoch), their Adam state of the last epoch run, and NaN history past their last epoch.
- epochs run and best epoch are those of the host EarlyStopping applied to the full history, over monitors, modes, min_delta,
  baseline, start_from_epoch and restore_best_weights, NaN losses included.
- build_fleet(early_stopping=...) replays the per-machine loop slot by slot, with the weights in shared memory and in L2, and
  FleetModelBuilder builds the reference's production estimator definition in one bucket with the metadata ModelBuilder writes.
- The first three hold for every kernel family of the fit (MSE-Adam, another loss, another optimizer: parity_helpers.FIT_KW); the
  optimizer state checked is then the optimizer's two state slots.
"""
import math

import numpy as np
import pytest
from parity_helpers import FIT_KW, crossed
from sklearn.utils import shuffle as sk_shuffle

pytestmark = pytest.mark.gpu

KERAS_ADAM = {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7}
FROZEN = dict(KERAS_ADAM, lr=0.0)

# (weights in L2, dz buffers in L2) of the five memory plans, with a shape that takes each (tests/test_fit_plan.py)
PLANS = {"shared": ("hourglass", 64), "weights_in_l2": ("symmetric", 10), "one_dz_in_l2": ("symmetric", 64),
         "two_dz_in_l2": ("symmetric", 96), "three_dz_in_l2": ("symmetric", 128)}


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


def plan_spec(km, name):
    kind, T = PLANS[name]
    return km.ff_hourglass_spec(T) if kind == "hourglass" else km.ff_symmetric_spec(T)


def waves(rng, n, width):
    t = np.linspace(0, 12, n)[:, None]
    return (0.5 + 0.3 * np.sin(t * rng.uniform(0.5, 2, width) + rng.uniform(0, 3, width)) + rng.normal(0, 0.01, (n, width))).astype(np.float32)


def dev(torch, eng, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)


def same(torch, a, b):
    """torch.equal with NaN positions compared as positions."""
    na, nb = a.isnan(), b.isnan()
    return torch.equal(na, nb) and torch.equal(torch.where(na, torch.zeros_like(a), a), torch.where(nb, torch.zeros_like(b), b))


def host_rule(cfg, history, E):
    """The host EarlyStopping over a full history: (epochs run, best epoch or -1, epoch whose weights the job keeps)."""
    from gordo_components_b200.machine.model.models import EarlyStopping

    cb = EarlyStopping(**cfg)
    ran = E
    for e in range(E):
        logs = {k: float(v[e]) for k, v in history.items()}
        if cb.update(e, logs, lambda e=e: e):
            ran = e + 1
            break
    improved = cb.best not in (math.inf, -math.inf)
    best = cb.best_epoch if (cb.best_weights is not None or improved) else -1
    keep = cb.best_weights + 1 if (cb.restore_best_weights and cb.best_weights is not None) else ran
    return ran, best, keep


# ------------------------------------------------------------------------------------------------ 1. a rule that never fires
@pytest.mark.parametrize("plan,fit", crossed(PLANS, FIT_KW))
def test_rule_that_never_fires_is_fit_split(engine, torch, km, plan, fit):
    spec = plan_spec(km, plan)
    M, N, NV, E, B = 3, 150, 23, 3, 50
    rng = np.random.default_rng(7)
    X = np.concatenate([waves(rng, N + NV, spec.dims[0]) for _ in range(M)])
    w0s = [km.init_ff_weights(spec, np.random.default_rng(70 + m)) for m in range(M)]
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    xd = dev(torch, eng, X)
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(M), N, np.arange(M) * (N + NV)), eng.device)
    split = engine.make_split(np.full(M, NV))
    kw = dict(split=split, epochs=E, batch_size=B, shuffle=True, seed=13, **fit)
    p1, p2 = eng.pack_params(w0s), eng.pack_params(w0s)
    l1, a1, vl1, va1, (m1, v1) = eng.fit_split(p1, jobs, M, N, xd, xd, **kw)
    stop = engine.make_stop([{"monitor": mon, "patience": E} for mon in ("val_loss", "loss", "val_accuracy")])
    l2, a2, vl2, va2, ran, best, (m2, v2) = eng.fit_split(p2, jobs, M, N, xd, xd, stop=stop, **kw)
    torch.cuda.synchronize()
    for name, g, w in (("weights", p2, p1), ("Adam m", m2, m1), ("Adam v", v2, v1), ("loss", l2, l1), ("accuracy", a2, a1),
                       ("val_loss", vl2, vl1), ("val_accuracy", va2, va1)):
        assert torch.equal(g, w), name
    assert ran.tolist() == [E] * M


# ------------------------------------------------------------------------------------------------ 2. ragged stops in one launch
@pytest.mark.parametrize("plan,fit", crossed(PLANS, FIT_KW))
@pytest.mark.parametrize("batch", [1, 32, 128])
@pytest.mark.parametrize("restore", [False, True])
def test_ragged_stops(engine, torch, km, plan, batch, restore, fit):
    spec = plan_spec(km, plan)
    lens = np.array([150, 97, 64, 33, 140])
    J, E = len(lens), 7
    patience = np.arange(1, J + 1)  # job j runs exactly patience + 1 epochs: epoch 0 improves on inf, nothing after beats 1e30
    rng = np.random.default_rng(batch)
    x_row = np.concatenate([[0], np.cumsum(lens[:-1] + 3)])
    X = waves(rng, int(x_row[-1] + lens[-1]), spec.dims[0])
    w0s = [km.init_ff_weights(spec, np.random.default_rng(90 + j)) for j in range(J)]
    slots = np.array([3, 0, 4, 1, 2])
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    xd = dev(torch, eng, X)
    jobs_h = engine.make_jobs(slots, lens, x_row)
    kw = dict(batch_size=batch, shuffle=True, seed=5, **fit)
    p = eng.pack_params([w0s[s] for s in range(J)])
    stop = engine.make_stop([{"monitor": "loss", "patience": int(pj), "min_delta": 1e30, "restore_best_weights": restore} for pj in patience])
    loss, acc, _, _, ran, best, (m, v) = eng.fit_split(p, engine.jobs_to_device(jobs_h, eng.device), J, int(lens.max()), xd, xd, epochs=E,
                                                      stop=stop, **kw)
    torch.cuda.synchronize()
    assert ran.tolist() == (patience + 1).tolist()
    assert best.tolist() == [0] * J
    for j in range(J):
        s, k = int(slots[j]), int(patience[j] + 1)
        one = engine.jobs_to_device(jobs_h[j:j + 1], eng.device)
        pw = eng.pack_params([w0s[i] for i in range(J)])
        wl, wa, _, _, (wm, wv) = eng.fit_split(pw, one, 1, int(lens[j]), xd, xd, epochs=k, **kw)
        p1 = eng.pack_params([w0s[i] for i in range(J)])
        eng.fit_split(p1, one, 1, int(lens[j]), xd, xd, epochs=1, **kw)
        torch.cuda.synchronize()
        assert torch.equal(p[s], (p1 if restore else pw)[s]), (j, "weights")
        assert torch.equal(m[s], wm[s]) and torch.equal(v[s], wv[s]), (j, "optimizer state of the last epoch run")
        assert torch.equal(loss[j, :k], wl[0]) and torch.equal(acc[j, :k], wa[0]), (j, "history")
        assert bool(loss[j, k:].isnan().all()) and bool(acc[j, k:].isnan().all()), (j, "history past the stop")


# ------------------------------------------------------------------------------------------------ 3. the rule against the host class
RULES = [dict(monitor=mon, patience=pat, min_delta=md, restore_best_weights=rb, **extra)
         for mon, md in (("loss", 0.0), ("loss", 2e-3), ("val_loss", 0.0), ("val_loss", 2e-3), ("accuracy", 0.0), ("val_accuracy", 0.0),
                         ("val_accuracy", 0.05))
         for pat, rb, extra in ((1, False, {}), (2, True, {}), (1, True, {"start_from_epoch": 3}))] + [
    dict(monitor="val_loss", patience=2, baseline=0.01, restore_best_weights=True),
    dict(monitor="val_loss", patience=0, baseline=1e-9, restore_best_weights=False),
    dict(monitor="loss", patience=3, mode="max"),
    dict(monitor="val_accuracy", patience=2, mode="min", restore_best_weights=True),
    dict(monitor="loss", patience=20, start_from_epoch=50, restore_best_weights=True),  # every epoch skipped
]


@pytest.mark.parametrize("plan,fit", crossed(["shared", "weights_in_l2", "three_dz_in_l2"], FIT_KW))
def test_rule_is_the_host_early_stopping(engine, torch, km, plan, fit):
    spec = plan_spec(km, plan)
    J, N, NV, E, B = len(RULES), 120, 30, 10, 32
    rng = np.random.default_rng(31)
    x_row = np.arange(J) * (N + NV)
    X = np.concatenate([waves(rng, N + NV, spec.dims[0]) for _ in range(J)])
    w0s = [km.init_ff_weights(spec, np.random.default_rng(500 + j)) for j in range(J)]
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    xd = dev(torch, eng, X)
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(J), N, x_row), eng.device)
    kw = dict(split=engine.make_split(np.full(J, NV)), batch_size=B, shuffle=True, seed=17, **fit)
    # witnesses: the same launch without the rule, for every epoch count
    ref = {}
    for k in range(1, E + 1):
        pk = eng.pack_params(w0s)
        *hist, (mk, vk) = eng.fit_split(pk, jobs, J, N, xd, xd, epochs=k, **kw)
        ref[k] = (pk, mk, vk, hist)
    full = [h.cpu().numpy() for h in ref[E][3]]
    p = eng.pack_params(w0s)
    loss, acc, vloss, vacc, ran, best, (m, v) = eng.fit_split(p, jobs, J, N, xd, xd, epochs=E, stop=engine.make_stop(RULES), **kw)
    torch.cuda.synchronize()
    fired = 0
    for j, cfg in enumerate(RULES):
        history = {"loss": full[0][j], "accuracy": full[1][j], "val_loss": full[2][j], "val_accuracy": full[3][j]}
        want_ran, want_best, keep = host_rule(cfg, history, E)
        fired += want_ran < E
        assert (int(ran[j]), int(best[j])) == (want_ran, want_best), (j, cfg)
        assert torch.equal(p[j], ref[keep][0][j]), (j, cfg, "weights")
        assert torch.equal(m[j], ref[want_ran][1][j]) and torch.equal(v[j], ref[want_ran][2][j]), (j, cfg, "optimizer state")
        for got, want in zip((loss, acc, vloss, vacc), ref[want_ran][3]):
            assert torch.equal(got[j, :want_ran], want[j]) and bool(got[j, want_ran:].isnan().all()), (j, cfg, "history")
    assert fired >= 3  # the grid exercises early stops, not only full runs


@pytest.mark.parametrize("restore", [False, True])
def test_nan_losses_never_improve(engine, torch, km, restore):
    spec = km.ff_hourglass_spec(8)
    patience = [1, 2, 4]
    J, N, E = len(patience), 64, 8
    rng = np.random.default_rng(3)
    X = waves(rng, J * N, 8)
    X[5::17] = np.nan  # NaN rows: every loss is NaN
    w0s = [km.init_ff_weights(spec, np.random.default_rng(40 + j)) for j in range(J)]
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    xd = dev(torch, eng, X)
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(J), N, np.arange(J) * N), eng.device)
    kw = dict(batch_size=16, shuffle=True, seed=2)
    p = eng.pack_params(w0s)
    stop = engine.make_stop([{"monitor": "loss", "patience": pj, "restore_best_weights": restore} for pj in patience])
    loss, _, _, _, ran, best, (m, v) = eng.fit_split(p, jobs, J, N, xd, xd, epochs=E, stop=stop, **kw)
    torch.cuda.synchronize()
    assert bool(loss[:, 0].isnan().all())
    want = [max(pj - 1, 1) + 1 for pj in patience]  # stops at epoch max(patience - 1, 1): wait counts epoch 0 too
    assert ran.tolist() == want
    assert best.tolist() == ([0] * J if restore else [-1] * J)
    for j in range(J):
        pw = eng.pack_params(w0s)
        _, _, _, _, (wm, _) = eng.fit_split(pw, jobs, J, N, xd, xd, epochs=1 if restore else want[j], **kw)
        pm = eng.pack_params(w0s)
        _, _, _, _, (mm, _) = eng.fit_split(pm, jobs, J, N, xd, xd, epochs=want[j], **kw)
        torch.cuda.synchronize()
        assert same(torch, p[j], pw[j]), (j, "weights")
        assert same(torch, m[j], mm[j]), (j, "Adam m")


# ------------------------------------------------------------------------------------------------ 4. build_fleet, slot by slot
def replay_fleet_with_early_stopping(engine, torch, km, T, fit):
    """build_fleet(early_stopping=...) on T-tag hourglasses against the per-machine loop, slot by slot: the fleet runs the stop kernels,
    the loop the plain ones, one launch per epoch and the frozen Adam tail."""
    from gordo_components_b200 import fleet
    from gordo_components_b200.machine.model.models import EarlyStopping

    spec = km.ff_hourglass_spec(T)
    M, N, K, E, B, vsplit = 3, 230, 3, 10, 32, 0.1
    rng = np.random.default_rng(22)
    X = np.concatenate([waves(rng, N, T) for _ in range(M)])
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    xd = dev(torch, eng, X)
    rules = [dict(monitor="val_loss", patience=1, min_delta=1.0, restore_best_weights=False),  # stops after epoch 1
             dict(monitor="val_loss", patience=2, min_delta=2e-3, restore_best_weights=True),
             dict(monitor="val_loss", patience=E, restore_best_weights=True)]
    fb = fleet.build_fleet(eng, xd, xd, N, epochs=E, batch_size=B, n_splits=K, seed=3, adam=KERAS_ADAM, shuffle=False,
                           detector_shuffle=True, validation_split=vsplit, early_stopping=[EarlyStopping(**r) for r in rules], **fit)
    torch.cuda.synchronize()
    assert fb.epochs == E and tuple(fb.epochs_run.shape) == (M,) and tuple(fb.fold_epochs_run.shape) == (M, K)
    test = N // (K + 1)
    slot_n = [N] + [N - (K - k) * test for k in range(K)]
    g = torch.Generator(device=eng.device).manual_seed(3)
    p0 = fleet.random_glorot_params(eng, M * (K + 1), g)
    ofs = 0
    for i, o in zip(eng.dims[:-1], eng.dims[1:]):
        ofs += i * o
        p0[:, ofs:ofs + o] = 0
        ofs += o
    stopped = 0
    for m in range(M):
        for j, n in enumerate(slot_n):
            slot = m if j == 0 else M + (j - 1) * M + m
            Xs = sk_shuffle(X[m * N:m * N + n], random_state=0)
            n_train = int(math.floor(n * (1 - vsplit)))
            xs = dev(torch, eng, Xs)
            p = p0[slot:slot + 1].clone()
            tj = engine.jobs_to_device(engine.make_jobs([0], [n_train], [0]), eng.device)
            vj = engine.jobs_to_device(engine.make_jobs([0], [n - n_train], [n_train]), eng.device)
            cb = EarlyStopping(**rules[m])
            state, losses, vlosses = None, [], []
            for e in range(E):  # the per-machine loop: one epoch, the frozen tail, the callback
                l, _, state = eng.fit(p, tj, 1, n_train, xs, xs, epochs=1, batch_size=B, shuffle=False, adam=KERAS_ADAM, state=state,
                                      step0=e * math.ceil(n_train / B), **fit)
                vl, _, _ = eng.fit(p.clone(), vj, 1, n - n_train, xs, xs, epochs=1, batch_size=B, shuffle=False, adam=FROZEN,
                                   loss=fit.get("loss", "mse"))
                losses.append(l)
                vlosses.append(vl)
                if cb.update(e, {"loss": float(l[0, 0]), "val_loss": float(vl[0, 0])}, lambda: p.clone()):
                    break
            if cb.restore_best_weights and cb.best_weights is not None:
                p = cb.best_weights
            torch.cuda.synchronize()
            ran = len(losses)
            stopped += ran < E
            got_p = fb.params[m] if j == 0 else fb.fold_params[m, j - 1]
            got_l = fb.loss[m] if j == 0 else fb.fold_loss[m, j - 1]
            got_v = fb.val_loss[m] if j == 0 else fb.fold_val_loss[m, j - 1]
            got_ran = fb.epochs_run[m] if j == 0 else fb.fold_epochs_run[m, j - 1]
            assert int(got_ran) == ran, (m, j, "epochs run")
            assert torch.equal(got_p, p[0]), (m, j, "weights")
            assert torch.equal(got_l[:ran], torch.cat(losses, dim=1)[0]) and bool(got_l[ran:].isnan().all()), (m, j, "loss")
            assert torch.equal(got_v[:ran], torch.cat(vlosses, dim=1)[0]) and bool(got_v[ran:].isnan().all()), (m, j, "val_loss")
    assert stopped >= K + 1
    det = fb.detector(0)
    h = det.base_estimator.get_metadata()["history"]
    ran0 = int(fb.epochs_run[0])
    assert all(len(h[k]) == ran0 for k in ("loss", "accuracy", "val_loss", "val_accuracy"))
    assert h["params"]["epochs"] == E and det.base_estimator._history.epoch == list(range(ran0))


def test_build_fleet_with_early_stopping_replays(engine, torch, km):
    replay_fleet_with_early_stopping(engine, torch, km, 8, FIT_KW["mse-adam"])


# the other stop kernels the batched build reaches: the weight image in L2 (128 tags), and another loss and optimizer (LOSS + OPT)
@pytest.mark.parametrize("T,fit", crossed([8, 128], {k: FIT_KW[k] for k in ("mse-adam", "mae-nadam")})[1:])
def test_build_fleet_with_early_stopping_replays_other_kernels(engine, torch, km, T, fit):
    replay_fleet_with_early_stopping(engine, torch, km, T, fit)


# ------------------------------------------------------------------------------------------------ 5. the production definition
def test_fleet_builder_builds_the_production_definition(torch, tmp_path):
    import pickle

    import pandas as pd

    from gordo_components_b200 import builder, serializer

    E = 6
    ae = {"gordo.machine.model.models.KerasAutoEncoder": {
        "kind": "feedforward_hourglass", "batch_size": 128, "compression_factor": 0.5, "encoding_layers": 1, "func": "tanh", "out_func": "linear",
        "optimizer": "Adam", "loss": "mse", "epochs": E, "validation_split": 0.1,
        "callbacks": [{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "val_loss", "patience": 1, "min_delta": 1e-3, "restore_best_weights": True}}]}}
    model = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {
        "base_estimator": {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", ae]}},
        "scaler": "sklearn.preprocessing.MinMaxScaler", "shuffle": True}}
    evaluation = {"cv": {"sklearn.model_selection.TimeSeriesSplit": {"n_splits": 5}}}
    N, T = 1500, 12
    idx = pd.date_range("2019-01-01", periods=N, freq="10min", tz="UTC")
    rng = np.random.default_rng(9)
    machines = []
    for i in range(3):
        frame = pd.DataFrame(waves(rng, N, T).astype(np.float64), index=idx, columns=[f"tag-{c}" for c in range(T)])
        machines.append({"name": f"prod-{i}", "model": model, "dataset": {"X": frame, "y": frame}, "evaluation": evaluation})
    assert all(builder._canonical(i, m) is None for i, m in enumerate(machines))  # opt-in: ModelBuilder by default
    assert all(builder._canonical(i, m, early_stopping=True) is not None for i, m in enumerate(machines))
    calls = []
    orig = builder.FleetModelBuilder._build_bucket
    builder.FleetModelBuilder._build_bucket = staticmethod(lambda members: calls.append(len(members)) or orig(members))
    try:
        fleet_out = builder.FleetModelBuilder(machines, early_stopping=True).build(str(tmp_path))
    finally:
        builder.FleetModelBuilder._build_bucket = staticmethod(orig)
    assert calls == [3]  # one batched bucket, no fall-back
    single_model, single_meta = builder.ModelBuilder(dict(machines[0])).build()

    def keys(d):
        return {k: keys(v) for k, v in d.items()} if isinstance(d, dict) else None

    for model_, meta in fleet_out:
        assert keys(meta) == keys(single_meta)
        hist = meta["metadata"]["build_metadata"]["model"]["model_meta"]["history"]
        want = single_meta["metadata"]["build_metadata"]["model"]["model_meta"]["history"]
        assert list(hist) == list(want) == ["loss", "accuracy", "val_loss", "val_accuracy", "params"]
        assert hist["params"] == want["params"] and hist["params"]["epochs"] == E
        ae_ = model_.base_estimator.steps[-1][1]
        ran = len(ae_._history.epoch)
        assert 1 <= ran <= E and ae_._history.epoch == list(range(ran))
        assert all(len(hist[k]) == ran for k in ("loss", "accuracy", "val_loss", "val_accuracy"))
        assert np.isfinite(hist["val_loss"]).all()
    for m in machines:
        with open(tmp_path / m["name"] / "model.pkl", "rb") as f:
            det = pickle.load(f)
        frame = m["dataset"]["X"]
        out = det.anomaly(frame.iloc[:200], frame.iloc[:200])
        assert np.isfinite(out["total-anomaly-scaled"].values).all()
        assert serializer.load_metadata(str(tmp_path / m["name"]))["name"] == m["name"]
