"""
The grouped Dense fit on the H100 (gb_ffae_fit_group, engine.fit_group, fleet.build_joined, FleetModelBuilder(mixed_widths=True)).

Kernel level: nets of several architectures that share a memory plan, trained in one launch, against a per-net launch of each group
alone (engine.FFEngine.fit_split), bit for bit in params, optimizer state, history, held-out statistics, epochs_run and best_epoch --
in every memory plan, kernel family and entry point.  Builder level: a project of machines over several tag counts built with and
without mixed_widths gives the same detectors bit for bit, with one fit launch per launch group.
"""
import pickle
import zlib

import numpy as np
import pandas as pd
import pytest
from parity_helpers import FIT_KW

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("no CUDA device")
    import __graft_entry__ as ge

    ge.build()
    return t


def _spec(kind, tags):
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    return KerasAutoEncoder(kind=kind, n_features=tags, n_features_out=tags)._build_spec()


def _plan_nets():
    """Per memory plan, the hourglasses of one grouped launch: five tag counts in shared memory, the first two of each L2 plan."""
    from gordo_components_b200 import engine

    nets = {(0, 0): [_spec("feedforward_hourglass", t) for t in (4, 9, 17, 33, 64)]}
    for t in range(65, 197):
        s = _spec("feedforward_hourglass", t)
        plan = engine.fit_plan(s.dims, s.acts, s.l1)
        if plan != (0, 0) and len(nets.setdefault(plan, [])) < 2:
            nets[plan].append(s)
    return nets


PLANS = {"smem": (0, 0), "l2-weights": (1, 0), "l2-dz1": (1, 1), "l2-dz2": (1, 2), "l2-dz3": (1, 3)}
FAMILIES = ["mse", "huber", "nadam", "reg", "dropout"]
ENTRIES = ["plain", "split", "stop"]


def _family_kw(family, n_layers):
    if family == "mse":
        return {}
    if family == "huber":
        return dict(FIT_KW["huber-adam"])
    if family == "nadam":
        return dict(FIT_KW["mae-nadam"])
    if family == "reg":
        zeros = [0.0] * (n_layers - 2)
        return {"reg": {"kernel_l1": [1e-4, 0.0] + zeros, "kernel_l2": [0.0, 1e-3] + zeros, "bias_l1": [0.0] * n_layers,
                        "bias_l2": [1e-3, 0.0] + zeros}}
    return {"dropout": [0.1, 0.2] + [0.0] * (n_layers - 2)}


def _bits(t):
    """The tensor's bits, so that NaN entries compare equal to themselves."""
    import torch

    return t.contiguous().view(torch.int32 if t.dtype in (torch.float32, torch.int32) else torch.int64).cpu()


def _same(a, b, what):
    if a is None or b is None:
        assert a is None and b is None, what
        return
    assert a.shape == b.shape, what
    assert bool((_bits(a) == _bits(b)).all()), what


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("plan", list(PLANS))
def test_grouped_launch_equals_per_net_launches(torch, plan, family, entry):
    from gordo_components_b200 import engine

    key = PLANS[plan]
    specs = _plan_nets()[key]
    assert len(specs) >= 2
    dev = engine.cuda_device()
    rng = np.random.default_rng(zlib.crc32(f"{plan}{family}{entry}".encode()))
    counts = [40, 7, 29, 1, 60][: len(specs)] if key == (0, 0) else [5, 3]  # uneven; more jobs than SMs in shared memory
    E, B = 4, 32
    kw = dict(epochs=E, batch_size=B, seed=11, **_family_kw(family, len(specs[0].dims) - 1))
    groups, alone = [], []
    for spec, n_jobs in zip(specs, counts):
        eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
        T = spec.dims[0]
        n_rows = rng.integers(40, 120, n_jobs)
        n_val = rng.integers(5, 20, n_jobs) if entry != "plain" else np.zeros(n_jobs, int)
        tot = n_rows + n_val
        x_row = np.concatenate([[0], np.cumsum(tot)[:-1]])
        x = torch.from_numpy(rng.normal(size=(int(tot.sum()), T)).astype(np.float32)).to(dev)
        y = torch.from_numpy(rng.normal(size=(int(tot.sum()), spec.dims[-1])).astype(np.float32)).to(dev)
        params = torch.from_numpy(rng.uniform(-0.3, 0.3, (n_jobs, eng.param_stride)).astype(np.float32)).to(dev)
        jobs = engine.jobs_to_device(engine.make_jobs(np.arange(n_jobs), n_rows, x_row), dev)
        split = row_map = stop = None
        if entry != "plain":
            maps = [rng.permutation(int(v)).astype(np.int32) for v in tot]
            row_map = torch.from_numpy(np.concatenate(maps)).to(dev)
            split = engine.make_split(n_val, np.concatenate([[0], np.cumsum(tot)[:-1]]))
        if entry == "stop":
            rules = [{"monitor": "val_loss", "patience": 0, "restore_best_weights": True} if j % 2 == 0 else
                     {"monitor": "loss", "patience": 1, "min_delta": 1.0} for j in range(n_jobs)]  # the odd ones stop after epoch 2
            stop = engine.make_stop(rules)
        groups.append(engine.FitGroup(eng, params.clone(), jobs, n_jobs, int(n_rows.max()), x, y, split=split, row_map=row_map, stop=stop))
        p = params.clone()
        alone.append((p, eng.fit_split(p, jobs, n_jobs, int(n_rows.max()), x, y, split=split, row_map=row_map, stop=stop, **kw)))
    joined = engine.fit_group(groups, **kw)
    torch.cuda.synchronize()
    stopped = 0
    for g, (p, ref), got in zip(groups, alone, joined):
        _same(g.params, p, "params")
        for i, (a, b) in enumerate(zip(got[:-1], ref[:-1])):
            _same(a, b, f"output {i}")
        _same(got[-1][0], ref[-1][0], "m")
        _same(got[-1][1], ref[-1][1], "v")
        if entry == "stop":
            stopped += int((got[4] < E).sum())
    if entry == "stop":
        assert stopped > 0


def test_job_group_map_follows_any_job_order(torch):
    """Jobs of the groups interleaved in the launch: each still computes what its group's per-net launch does."""
    from gordo_components_b200 import _cabi, engine

    dev = engine.cuda_device()
    specs = [_spec("feedforward_hourglass", t) for t in (5, 12)]
    rng = np.random.default_rng(3)
    engs = [engine.FFEngine(s.dims, s.acts, s.l1) for s in specs]
    xs = [torch.from_numpy(rng.normal(size=(400, s.dims[0])).astype(np.float32)).to(dev) for s in specs]
    ps = [torch.from_numpy(rng.uniform(-0.3, 0.3, (3, e.param_stride)).astype(np.float32)).to(dev) for e in engs]
    host_jobs = [engine.make_jobs(np.arange(3), [50, 80, 33], [0, 100, 200]) for _ in specs]
    refs = []
    for e, x, p, hj in zip(engs, xs, ps, host_jobs):
        q = p.clone()
        e.fit(q, engine.jobs_to_device(hj, dev), 3, 80, x, x, epochs=2)
        refs.append(q)
    order = [(1, 0), (0, 0), (1, 1), (0, 1), (0, 2), (1, 2)]  # (group, job)
    jobs = np.concatenate([host_jobs[g][j:j + 1] for g, j in order])
    jg = np.asarray([g for g, _ in order], dtype=np.int32)
    out = torch.empty((6, 2), dtype=torch.float32, device=dev)
    recs = (_cabi.GbFitGroup * 2)()
    states = [e._fit_state(p, None) for e, p in zip(engs, ps)]
    for r, e, p, (m, v), x in zip(recs, engs, ps, states, xs):
        r.net = e.net
        r.params, r.adam_m, r.adam_v, r.x, r.y = (_cabi.ptr(t) for t in (p, m, v, x, x))
    hp = engine._fit_hparams(2, 32, True, None, None, 0, False, 0)
    jd = engine.jobs_to_device(jobs, dev)
    ws = torch.empty((int(engs[0].lib.gb_ffae_fit_group_workspace_bytes(2, 6)),), dtype=torch.uint8, device=dev)
    import ctypes as C

    _cabi.check(engs[0].lib.gb_ffae_fit_group(recs, 2, jg.ctypes.data_as(C.POINTER(C.c_int32)), _cabi.ptr(jd), None, 6, 80, None, None,
                                              C.byref(hp), 1, _cabi.ptr(out), None, None, None, None, None, None, None, None, None,
                                              _cabi.ptr(ws), engine._stream_ptr()))
    torch.cuda.synchronize()
    for p, q in zip(ps, refs):
        _same(p, q, "params")


# ------------------------------------------------------------------------------------------------ builder level
def waves(rng, n, t):
    s = np.linspace(0, 20, n)[:, None]
    return 3.0 + np.sin(s * rng.uniform(0.5, 2, t) + rng.uniform(0, 6, t)) * rng.uniform(0.5, 4, t) + rng.normal(0, 0.05, (n, t))


def _series(rows, tags, seed):
    rng = np.random.default_rng(seed)
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(waves(rng, rows, tags).astype(np.float32), index=idx, columns=[f"TAG {i}" for i in range(tags)])


def _strip(meta):
    if isinstance(meta, dict):
        return {k: _strip(v) for k, v in meta.items() if k != "model_creation_date" and not k.endswith("duration_sec")}
    return meta


def _ae(**kw):
    return {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2, **kw}}


def _det(base, **kw):
    return {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": base, **kw}}


PIPE = {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", _ae()]}}
STOP = [{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "val_loss", "patience": 1, "min_delta": 1e-3, "restore_best_weights": True}}]
DEFS = {
    "bare": _det(_ae()),
    "pipe": _det(PIPE),
    "split": _det(_ae(validation_split=0.1), shuffle=True),
    "stop": _det(_ae(epochs=4, validation_split=0.1, callbacks=STOP)),
    "kfold": {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {"base_estimator": _ae(), "window": 12}},
    "ttr": _det({"sklearn.compose.TransformedTargetRegressor": {"transformer": "sklearn.preprocessing.MinMaxScaler", "regressor": _ae()}}),
    "smooth": _det(_ae(), window=12, smoothing_method="sma"),
}
KFOLD = {"cv": {"sklearn.model_selection.KFold": {"n_splits": 3, "shuffle": True, "random_state": 0}}}


@pytest.mark.parametrize("ragged", [False, True])
def test_mixed_widths_build_equals_the_default_build(torch, monkeypatch, ragged):
    from gordo_components_b200 import builder, engine

    tags = [3, 5, 8, 5, 13, 3, 21, 8, 34, 13, 5, 21, 3, 8]
    kinds = ["bare", "pipe", "split", "stop", "kfold", "ttr", "smooth"]
    machines = []
    for i, t in enumerate(tags):
        kind = kinds[i % len(kinds)] if i < 2 * len(kinds) else "bare"
        rows = 240 + (17 * i if ragged else 0)
        m = {"name": f"m{i}-{kind}-{t}", "model": DEFS[kind], "dataset": {"X": _series(rows, t, i)}}
        if kind == "kfold":
            m["evaluation"] = KFOLD
        machines.append(m)
    flags = dict(kfcv=True, early_stopping=True, smoothing=True, target_scaler=True, ragged=ragged)
    plain = builder.FleetModelBuilder(machines, **flags).build()

    launches, groups = [], []
    real_group, real_split, real_lg = engine.fit_group, engine.FFEngine.fit_split, builder.launch_groups
    monkeypatch.setattr(engine, "fit_group", lambda *a, **k: launches.append("group") or real_group(*a, **k))
    monkeypatch.setattr(engine.FFEngine, "fit_split", lambda self, *a, **k: launches.append("net") or real_split(self, *a, **k))
    monkeypatch.setattr(builder, "launch_groups", lambda b: groups.extend(real_lg(b)) or groups)
    mixed = builder.FleetModelBuilder(machines, mixed_widths=True, **flags).build()
    assert len(launches) == len(groups) and "group" in launches
    assert sum(len(g) > 1 for g in groups) == launches.count("group")
    for (m0, meta0), (m1, meta1) in zip(plain, mixed):
        assert meta0["name"] == meta1["name"]
        assert pickle.dumps(m0) == pickle.dumps(m1), meta0["name"]
        assert _strip(meta0) == _strip(meta1), meta0["name"]
