"""
gb_ffae_fit_split on the H100: training over row positions through a row map, and the validation pass at the end of every epoch.

- Without a map or held-out positions it is gb_ffae_fit, bit for bit, in every memory plan.
- With a map it is gb_ffae_fit on the gathered copy x[map], bit for bit, in shared memory and in both L2 plan groups.
- Its val_loss / val_accuracy are those of the per-machine estimator's two launches per epoch (one training epoch, then an
  lr = 0 Adam fit of the held-out tail with the same loss), bit for bit, and the float64 oracle's to 2e-4.
- Each of these holds for every kernel family of the fit (MSE-Adam, another loss, another optimizer: parity_helpers.FIT_KW), whose
  split instantiations are then compared with their plain ones.
- build_fleet(detector_shuffle=True, validation_split=0.1) replays slot by slot, and FleetModelBuilder builds the reference's
  example definition through the batched path with the metadata ModelBuilder writes.
"""
import math

import loss_oracle
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


def perms(rng, lens, E, max_rows):
    p = np.zeros((len(lens), E, max_rows), np.int32)
    for j, n in enumerate(lens):
        for e in range(E):
            p[j, e, :n] = rng.permutation(n)
    return p


# ------------------------------------------------------------------------------------------------ 1. no map, nothing held out
@pytest.mark.parametrize("plan,fit", crossed(PLANS, FIT_KW))
@pytest.mark.parametrize("order", ["perm", "keyed"])
def test_split_without_map_is_fit(engine, torch, km, plan, order, fit):
    spec = plan_spec(km, plan)
    M, N, E, B = 2, 150, 2, 50
    rng = np.random.default_rng(5)
    X = np.concatenate([waves(rng, N, spec.dims[0]) for _ in range(M)])
    w0s = [km.init_ff_weights(spec, np.random.default_rng(60 + m)) for m in range(M)]
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    xd = dev(torch, eng, X)
    jobs = engine.jobs_to_device(engine.uniform_jobs(M, N), eng.device)
    perm = dev(torch, eng, perms(rng, [N] * M, E, N)) if order == "perm" else None
    p1, p2 = eng.pack_params(w0s), eng.pack_params(w0s)
    l1, a1, (m1, v1) = eng.fit(p1, jobs, M, N, xd, xd, epochs=E, batch_size=B, perm=perm, shuffle=True, seed=9, **fit)
    split = engine.make_split(np.zeros(M, np.int32), -1)
    l2, a2, vl, va, (m2, v2) = eng.fit_split(p2, jobs, M, N, xd, xd, split=split, epochs=E, batch_size=B, perm=perm, shuffle=True, seed=9, **fit)
    torch.cuda.synchronize()
    for name, g, w in (("weights", p2, p1), ("Adam m", m2, m1), ("Adam v", v2, v1), ("loss", l2, l1), ("accuracy", a2, a1)):
        assert torch.equal(g, w), name
    assert bool(vl.isnan().all()) and bool(va.isnan().all())


# ------------------------------------------------------------------------------------------------ 2. row map = gathered copy
# shared memory, and one shape of each L2 plan group: the weight image alone, and the weight image with dz buffers
ROW_MAP_PLANS = {"hourglass8": ("hourglass", 8), "weights_in_l2": PLANS["weights_in_l2"], "three_dz_in_l2": PLANS["three_dz_in_l2"]}


@pytest.mark.parametrize("plan,fit", crossed(ROW_MAP_PLANS, FIT_KW))
@pytest.mark.parametrize("shuffle", [0, 1, 2])
@pytest.mark.parametrize("batch", [1, 32, 50, 128])
def test_row_map_is_the_gathered_copy(engine, torch, km, shuffle, batch, plan, fit):
    kind, T = ROW_MAP_PLANS[plan]
    spec = km.ff_hourglass_spec(T) if kind == "hourglass" else km.ff_symmetric_spec(T)
    rng = np.random.default_rng(100 * shuffle + batch)
    lens = np.array([200, 200, 129, 129, 7, 1, 60])
    maps = {200: sk_shuffle(np.arange(200), random_state=0), 129: sk_shuffle(np.arange(129), random_state=0), 7: rng.permutation(7)}
    keys = list(maps)
    ofs = dict(zip(keys, np.cumsum([0] + [len(maps[k]) for k in keys[:-1]])))
    row_map = np.concatenate([maps[k] for k in keys]).astype(np.int32)
    map_ofs = np.array([ofs.get(n, -1) if j != 6 else -1 for j, n in enumerate(lens)])  # the 60-row job reads its rows in place
    J = len(lens)
    x_row = np.concatenate([[3], 3 + np.cumsum(lens[:-1] + 5)])  # gaps between the jobs' rows
    X = waves(rng, int(x_row[-1] + lens[-1] + 4), T)
    Y = waves(rng, len(X), T)
    gathered_rows = np.concatenate([x_row[j] + (row_map[map_ofs[j]:map_ofs[j] + lens[j]] if map_ofs[j] >= 0 else np.arange(lens[j])) for j in range(J)])
    g_row = np.concatenate([[0], np.cumsum(lens[:-1])])
    slots = rng.permutation(J).astype(np.int32)
    w0s = [km.init_ff_weights(spec, np.random.default_rng(200 + s)) for s in range(J)]
    E = 2
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    perm = dev(torch, eng, perms(rng, lens, E, int(lens.max()))) if shuffle == 2 else None
    kw = dict(epochs=E, batch_size=batch, shuffle=shuffle == 1, perm=perm, seed=11, **fit)
    p1 = eng.pack_params(w0s)
    l1, a1, (m1, v1) = eng.fit(p1, engine.jobs_to_device(engine.make_jobs(slots, lens, g_row), eng.device), J, int(lens.max()),
                               dev(torch, eng, X[gathered_rows]), dev(torch, eng, Y[gathered_rows]), **kw)
    p2 = eng.pack_params(w0s)
    split = engine.make_split(np.zeros(J, np.int32), map_ofs)
    l2, a2, _, _, (m2, v2) = eng.fit_split(p2, engine.jobs_to_device(engine.make_jobs(slots, lens, x_row), eng.device), J, int(lens.max()),
                                           dev(torch, eng, X), dev(torch, eng, Y), split=split, row_map=dev(torch, eng, row_map), **kw)
    torch.cuda.synchronize()
    for name, g, w in (("weights", p2, p1), ("Adam m", m2, m1), ("Adam v", v2, v1), ("loss", l2, l1), ("accuracy", a2, a1)):
        assert torch.equal(g, w), name


# ------------------------------------------------------------------------------------------------ 3. validation pass
def two_launch_witness(engine, torch, eng, w0s, xd, yd, lens, n_val, x_row, E, B, vb, perm, **fit):
    """The per-machine estimator's method: one training launch per epoch, then an lr = 0 Adam fit of every held-out tail with the
    same loss."""
    J = len(lens)
    params = eng.pack_params(w0s)
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(J), lens, x_row), eng.device)
    vjobs = engine.jobs_to_device(engine.make_jobs(np.arange(J), n_val, x_row + lens), eng.device)
    state, step0, loss, acc, vloss, vacc, weights = None, 0, [], [], [], [], []
    for e in range(E):
        # every job takes ceil(n / B) steps; the jobs differ in n, so each carries its own step count through its own launch
        l_e, a_e = [], []
        for j in range(J):
            jj = engine.jobs_to_device(engine.make_jobs([j], [lens[j]], [x_row[j]]), eng.device)
            st = None if state is None else state[j]
            l, a, s = eng.fit(params, jj, 1, int(lens[j]), xd, yd, epochs=1, batch_size=B, perm=perm[j:j + 1, e:e + 1].contiguous(), shuffle=False,
                              state=st, step0=e * math.ceil(lens[j] / B), **fit)
            l_e.append(l)
            a_e.append(a)
            if state is None:
                state = [None] * J
            state[j] = s
        loss.append(torch.cat(l_e))
        acc.append(torch.cat(a_e))
        vl, va, _ = eng.fit(params.clone(), vjobs, J, int(max(n_val)), xd, yd, epochs=1, batch_size=vb, shuffle=False, adam=FROZEN,
                            loss=fit.get("loss", "mse"))
        vloss.append(vl)
        vacc.append(va)
        weights.append(eng.unpack_params(params))
    cat = lambda v: torch.cat(v, dim=1)  # noqa: E731
    return params, cat(loss), cat(acc), cat(vloss), cat(vacc), weights


@pytest.mark.parametrize("plan,fit", crossed(PLANS, FIT_KW))
@pytest.mark.parametrize("vb", [1, 16, 32, 50, 128])
def test_validation_pass_is_the_frozen_launch(engine, torch, km, plan, vb, fit):
    spec = plan_spec(km, plan)
    T = spec.dims[0]
    rng = np.random.default_rng(vb)
    lens = np.array([100, 90, 80, 41])
    n_val = np.array([1, max(vb - 1, 1), 45, vb + 3])  # one row; fewer rows than a batch; several batches, the last one ragged
    x_row = np.concatenate([[0], np.cumsum(lens + n_val + 3)[:-1]])
    X = waves(rng, int(x_row[-1] + lens[-1] + n_val[-1]), T)
    w0s = [km.init_ff_weights(spec, np.random.default_rng(300 + j)) for j in range(len(lens))]
    E, B = 2, 32
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    xd = dev(torch, eng, X)
    perm_h = perms(rng, lens, E, int(lens.max()))
    perm = dev(torch, eng, perm_h)
    params = eng.pack_params(w0s)
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(len(lens)), lens, x_row), eng.device)
    loss, acc, vloss, vacc, _ = eng.fit_split(params, jobs, len(lens), int(lens.max()), xd, xd, split=engine.make_split(n_val), val_batch=vb,
                                              epochs=E, batch_size=B, perm=perm, **fit)
    wp, wl, wa, wvl, wva, weights = two_launch_witness(engine, torch, eng, w0s, xd, xd, lens, n_val, x_row, E, B, vb, perm, **fit)
    torch.cuda.synchronize()
    assert torch.equal(params, wp), "weights"
    assert torch.equal(loss, wl) and torch.equal(acc, wa), "training loss / accuracy"
    assert torch.equal(vloss, wvl), "val_loss"
    assert torch.equal(vacc, wva), "val_accuracy"
    # the float64 oracle at the weights after each epoch: sample-weighted mean of the per-batch total losses (loss + activity term)
    got = vloss.cpu().numpy()
    for j in range(len(lens)):
        tail = X[x_row[j] + lens[j]: x_row[j] + lens[j] + n_val[j]]
        for e in range(E):
            num = 0.0
            for s in range(0, n_val[j], vb):
                total, _data, _g, _yh = loss_oracle.ff_loss_and_grads(spec, weights[e][j], tail[s:s + vb], tail[s:s + vb], np.float64,
                                                                      loss=fit.get("loss", "mse"))
                num += float(total) * len(tail[s:s + vb])
            want = num / n_val[j]
            assert abs(got[j, e] - want) <= 2e-4 * abs(want), (j, e, got[j, e], want)


# ------------------------------------------------------------------------------------------------ 4. build_fleet, slot by slot
@pytest.mark.parametrize("input_scaler", [False, True])
def test_build_fleet_shuffled_with_validation_split(engine, torch, km, input_scaler):
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200 import fleet

    spec = km.ff_hourglass_spec(8)
    M, N, K, E, B, vsplit = 3, 230, 3, 2, 32, 0.1
    rng = np.random.default_rng(21)
    X = np.concatenate([waves(rng, N, 8) for _ in range(M)])
    Y = np.concatenate([waves(rng, N, 8) for _ in range(M)])
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    xd, yd = dev(torch, eng, X), dev(torch, eng, Y)
    fb = fleet.build_fleet(eng, xd, yd, N, epochs=E, batch_size=B, n_splits=K, seed=3, adam=KERAS_ADAM, shuffle=False, input_scaler=input_scaler,
                           detector_shuffle=True, validation_split=vsplit)
    torch.cuda.synchronize()
    test = N // (K + 1)
    slot_n = [N] + [N - (K - k) * test for k in range(K)]
    assert fb.steps_per_epoch == math.ceil(math.floor(N * (1 - vsplit)) / B)
    assert tuple(fb.val_loss.shape) == (M, E) and tuple(fb.fold_val_loss.shape) == (M, K, E)
    # scalers on all n rows of every slot, held-out ones included
    for m in range(M):
        ym = Y[m * N:(m + 1) * N].astype(np.float64)
        np.testing.assert_allclose(fb.scale[m].cpu().numpy(), MinMaxScaler().fit(ym).scale_, rtol=1e-5)
        if input_scaler:
            xm = X[m * N:(m + 1) * N].astype(np.float64)
            np.testing.assert_allclose(fb.in_scale[m].cpu().numpy(), MinMaxScaler().fit(xm).scale_, rtol=1e-12)
            for k in range(K):
                np.testing.assert_allclose(fb.fold_in_scale[m, k].cpu().numpy(), MinMaxScaler().fit(xm[:slot_n[k + 1]]).scale_, rtol=1e-12)
    if input_scaler:
        return
    # replay: the fleet's initial parameters, the detector's shuffle of the slot's rows, per-epoch fits + the frozen tail
    g = torch.Generator(device=eng.device).manual_seed(3)
    p0 = fleet.random_glorot_params(eng, M * (K + 1), g)
    ofs = 0
    for i, o in zip(eng.dims[:-1], eng.dims[1:]):
        ofs += i * o
        p0[:, ofs:ofs + o] = 0
        ofs += o
    for m in (0, M - 1):
        for j, n in enumerate(slot_n):
            slot = m if j == 0 else M + (j - 1) * M + m
            rows = X[m * N:m * N + n]
            Xs, Ys = sk_shuffle(rows, Y[m * N:m * N + n], random_state=0)
            n_train = int(math.floor(n * (1 - vsplit)))
            xs, ys = dev(torch, eng, Xs), dev(torch, eng, Ys)
            p = p0[slot:slot + 1].clone()
            tj = engine.jobs_to_device(engine.make_jobs([0], [n_train], [0]), eng.device)
            vj = engine.jobs_to_device(engine.make_jobs([0], [n - n_train], [n_train]), eng.device)
            state, losses, vlosses = None, [], []
            for e in range(E):
                l, _, state = eng.fit(p, tj, 1, n_train, xs, ys, epochs=1, batch_size=B, shuffle=False, adam=KERAS_ADAM, state=state,
                                      step0=e * math.ceil(n_train / B))
                vl, _, _ = eng.fit(p.clone(), vj, 1, n - n_train, xs, ys, epochs=1, batch_size=B, shuffle=False, adam=FROZEN)
                losses.append(l)
                vlosses.append(vl)
            torch.cuda.synchronize()
            got_p = fb.params[m] if j == 0 else fb.fold_params[m, j - 1]
            got_l = fb.loss[m] if j == 0 else fb.fold_loss[m, j - 1]
            got_v = fb.val_loss[m] if j == 0 else fb.fold_val_loss[m, j - 1]
            assert torch.equal(got_p, p[0]), (m, j, "weights")
            assert torch.equal(got_l, torch.cat(losses, dim=1)[0]), (m, j, "loss")
            assert torch.equal(got_v, torch.cat(vlosses, dim=1)[0]), (m, j, "val_loss")


# ------------------------------------------------------------------------------------------------ 5. the reference's example definition
def test_fleet_builder_builds_the_example_definition(torch, tmp_path):
    import pickle

    import pandas as pd

    from gordo_components_b200 import builder

    ae = {"gordo.machine.model.models.KerasAutoEncoder": {
        "batch_size": 128, "compression_factor": 0.6, "encoding_layers": 1, "epochs": 4, "func": "tanh", "kind": "feedforward_hourglass",
        "loss": "mse", "optimizer": "Adam", "out_func": "linear", "validation_split": 0.1}}
    model = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {
        "base_estimator": {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", ae]}},
        "scaler": "sklearn.preprocessing.MinMaxScaler", "shuffle": True, "smoothing_method": "smm"}}
    evaluation = {"cv": {"sklearn.model_selection.TimeSeriesSplit": {"n_splits": 5}}}
    N, T = 1500, 12
    idx = pd.date_range("2019-01-01", periods=N, freq="10min", tz="UTC")
    rng = np.random.default_rng(8)
    machines = []
    for i in range(3):
        frame = pd.DataFrame(waves(rng, N, T).astype(np.float64), index=idx, columns=[f"tag-{c}" for c in range(T)])
        machines.append({"name": f"ex-{i}", "model": model, "dataset": {"X": frame, "y": frame}, "evaluation": evaluation})
    assert all(builder._canonical(i, m) is not None for i, m in enumerate(machines))
    calls = []
    orig = builder.FleetModelBuilder._build_bucket
    builder.FleetModelBuilder._build_bucket = staticmethod(lambda members: calls.append(len(members)) or orig(members))
    try:
        fleet_out = builder.FleetModelBuilder(machines).build(str(tmp_path))
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
        assert hist["params"] == want["params"] and hist["params"]["steps"] == math.ceil(math.floor(0.9 * N) / 128)
        assert all(len(hist[k]) == 4 for k in ("loss", "accuracy", "val_loss", "val_accuracy"))
        assert hist["loss"][-1] < hist["loss"][0] and np.isfinite(hist["val_loss"]).all()
    from gordo_components_b200 import serializer

    for m in machines:
        with open(tmp_path / m["name"] / "model.pkl", "rb") as f:
            det = pickle.load(f)
        frame = m["dataset"]["X"]
        out = det.anomaly(frame.iloc[:200], frame.iloc[:200])
        assert np.isfinite(out["total-anomaly-scaled"].values).all()
        assert serializer.load_metadata(str(tmp_path / m["name"]))["name"] == m["name"]
