"""
Host side of the grouped Dense fit (gb_ffae_fit_group) and of FleetModelBuilder(mixed_widths=True), no GPU needed: every refusal
returns before anything is enqueued or dereferenced (placeholder device addresses, as the other fit host tests use), the grouped
kernels keep their static shared memory within the plans' reserve, and the builder's launch groups join exactly the buckets whose
keys differ only in the network's dims and whose nets share the fit's memory plan.
"""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pandas as pd
import pytest

from gordo_components_b200 import _cabi, builder, engine

GB_E_ARG, GB_E_SHAPE, GB_E_ALIGN, GB_E_SMEM = -1, -2, -3, -4
P = 256  # a 16-byte aligned placeholder address


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def hourglass_spec(tags):
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    return KerasAutoEncoder(kind="feedforward_hourglass", n_features=tags, n_features_out=tags)._build_spec()


def hourglass(tags):
    spec = hourglass_spec(tags)
    return _cabi.make_ffnet(spec.dims, spec.acts, spec.l1)


def group(net, params=P, x=P, y=P, best=P):
    g = _cabi.GbFitGroup()
    g.net = net
    g.params, g.adam_m, g.adam_v, g.best_params, g.x, g.y = params, P, P, best, x, y
    return g


def fit_group(lib, groups, job_group, n_jobs=None, stop=None, split=None, reg=None, drop=None, opt=None, workspace=P):
    recs = (_cabi.GbFitGroup * max(len(groups), 1))(*groups)
    hp = _cabi.GbFitHParams()
    hp.epochs, hp.batch_size, hp.shuffle = 1, 32, 1
    hp.lr, hp.beta1, hp.beta2, hp.eps = 1e-3, 0.9, 0.999, 1e-7
    jg = None if job_group is None else (C.c_int32 * len(job_group))(*job_group)
    n = len(job_group) if n_jobs is None else n_jobs
    return lib.gb_ffae_fit_group(recs if groups else None, len(groups), jg, P, split, n, 40, None, None, C.byref(hp), 32, P, P, P, P, stop,
                                 P if stop else None, P if stop else None, None if opt is None else C.byref(opt),
                                 None if reg is None else C.byref(reg), None if drop is None else C.byref(drop), workspace, None)


def refused(lib, rc, code, *words):
    msg = lib.gb_last_error().decode()
    assert rc == code, msg
    for w in words:
        assert w in msg, msg


def test_binding_matches_the_header(lib):
    assert "gb_ffae_fit_group" in _cabi.EXPORTS
    assert C.sizeof(_cabi.GbFitGroup) == C.sizeof(_cabi.GbFFNet) + 6 * 8 == 248  # the net (200 bytes, a multiple of 8), six pointers


def test_arguments_of_the_launch_are_refused_before_any_launch(lib):
    a, b = hourglass(4), hourglass(9)
    refused(lib, fit_group(lib, [], [0]), GB_E_ARG, "n_groups")
    refused(lib, lib.gb_ffae_fit_group(None, 2, None, P, None, 1, 40, None, None, None, 32, P, P, None, None, None, None, None, None,
                                       None, None, P, None), GB_E_ARG, "groups")
    # the library allocates nothing: the caller hands it the device workspace for the records and the job -> group map
    refused(lib, fit_group(lib, [group(a), group(b)], [0, 1], workspace=None), GB_E_ARG, "workspace")
    refused(lib, fit_group(lib, [group(a), group(b)], [0, 1], workspace=P + 8), GB_E_ARG, "workspace")
    size = lib.gb_ffae_fit_group_workspace_bytes(2, 3)
    assert size == 2 * lib.gb_ffae_fit_group_workspace_bytes(1, 0) + 3 * 4 and size > 3 * 4
    refused(lib, fit_group(lib, [group(a), group(b)], None, n_jobs=3), GB_E_ARG, "job_group")
    refused(lib, fit_group(lib, [group(a), group(b)], [0, 1, 2]), GB_E_ARG, "job_group[2]=2")
    refused(lib, fit_group(lib, [group(a), group(b)], [0, -1]), GB_E_ARG, "job_group[1]=-1")
    # a stop array needs every group's snapshot area
    stop = C.c_void_p(P)
    refused(lib, fit_group(lib, [group(a), group(b, best=None)], [0, 1], stop=stop), GB_E_ARG, "group 1", "best_params")
    refused(lib, fit_group(lib, [group(a), group(b, best=P + 4)], [0, 1], stop=stop), GB_E_ARG, "group 1", "aligned")


def test_every_group_is_checked_as_a_per_net_launch(lib):
    a, b = hourglass(4), hourglass(9)
    refused(lib, fit_group(lib, [group(a), group(b, params=None)], [0, 1]), GB_E_ARG, "group 1", "non-NULL")
    refused(lib, fit_group(lib, [group(a, x=None), group(b)], [0, 1]), GB_E_ARG, "group 0", "non-NULL")
    refused(lib, fit_group(lib, [group(a), group(b, y=P + 4)], [0, 1]), GB_E_ALIGN, "group 1", "aligned")
    wide = hourglass(4)
    wide.dims[1] = 300
    refused(lib, fit_group(lib, [group(a), group(wide)], [0, 1]), GB_E_SHAPE, "group 1")
    # past shared memory on its own (tests/test_fit_widths_host.py): refused with the per-net status, naming the group
    big = hourglass(197)
    refused(lib, fit_group(lib, [group(a), group(big)], [0, 1]), GB_E_SMEM, "group 1")


def test_groups_of_different_memory_plans_are_refused(lib):
    w, d = C.c_int32(), C.c_int32()
    plans = {}
    for tags in (4, 64, 128):
        assert lib.gb_ffae_fit_plan(C.byref(hourglass(tags)), C.byref(w), C.byref(d)) == 0
        plans[tags] = (w.value, d.value)
    assert plans[4] == plans[64] == (0, 0) and plans[128] != (0, 0)
    refused(lib, fit_group(lib, [group(hourglass(4)), group(hourglass(128))], [0, 1]), GB_E_ARG, "group 1", "memory plan")


def test_rates_and_coefficients_are_checked_against_every_net(lib):
    deep, short = hourglass(9), _cabi.make_ffnet([9, 9], ["linear"])
    drop = _cabi.make_dense_dropout([0.0, 0.2])  # on the input of layer 1: the one-layer net has none
    refused(lib, fit_group(lib, [group(deep), group(short)], [0, 1], drop=drop), GB_E_ARG, "group 1", "dropout rate[1]")
    bad = _cabi.make_dense_reg(kernel_l1=[0.0, 0.0, 0.0, -0.1])
    refused(lib, fit_group(lib, [group(short), group(deep)], [0, 1], reg=bad), GB_E_ARG, "group 1", "kernel_l1[3]")
    # coefficients on layers one net has and the other has not: the two would run different kernel families
    reg = _cabi.make_dense_reg(kernel_l2=[0.0, 0.0, 0.0, 0.1])
    refused(lib, fit_group(lib, [group(deep), group(short)], [0, 1], reg=reg), GB_E_ARG, "group 1", "kernel families")
    opt = _cabi.GbOptimizer()
    opt.kind = 99
    refused(lib, fit_group(lib, [group(deep), group(short)], [0, 1], opt=opt), GB_E_ARG, "group 0", "optimizer kind")


def test_grouped_kernels_static_shared_memory_fits_the_reserve(lib):
    """The grouped kernels read their record through L1: their static shared memory is the per-net kernels', within the 2 KB the
    plans keep for it (FIT_STATIC_SMEM), so every plan the per-net fit takes holds for a group too."""
    from gordo_components_b200.csrc import build

    obj = os.path.join(build.OBJ, "ffae_fit_group.o")
    tool = os.path.join(os.path.dirname(build._nvcc()), "cuobjdump")
    out = subprocess.run([tool, "-res-usage", obj], capture_output=True, text=True, check=True).stdout
    sizes = [int(v) for v in re.findall(r"SHARED:(\d+)", out)]
    assert len(sizes) == 45, "9 (plan, entry) cells x 5 kernel families"
    assert max(sizes) <= 2048, sorted(set(sizes))


# ------------------------------------------------------------------------------------------------ the builder's launch groups
AE = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2}}
DETECTOR = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": AE}}
KFCV = {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {"base_estimator": AE}}
KFOLD = {"cv": {"sklearn.model_selection.KFold": {"n_splits": 3, "shuffle": True, "random_state": 0}}}


def _frame(rows, tags, seed=0):
    rng = np.random.default_rng(seed)
    idx = pd.date_range("2020-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(rng.random((rows, tags)).astype(np.float32), index=idx, columns=[f"TAG {i}" for i in range(tags)])


def _machine(name, tags=4, rows=200, model=DETECTOR, **extra):
    X = _frame(rows, tags)
    return {"name": name, "model": model, "dataset": {"X": X, "y": X}, **extra}


def _buckets(machines, ragged=False):
    buckets = {}
    for i, m in enumerate(machines):
        c = builder._canonical_kfcv(i, m) if "KFCV" in str(m["model"]) else builder._canonical(i, m)
        buckets.setdefault(c.bucket(ragged), []).append(c)
    return buckets


def _names(groups):
    return [[[c.machine["name"] for c in members] for members in g] for g in groups]


def test_buckets_that_differ_only_in_dims_and_share_a_plan_join():
    assert engine.fit_plan(*_spec(4)) == engine.fit_plan(*_spec(80)) == (0, 0)
    assert engine.fit_plan(*_spec(81)) == engine.fit_plan(*_spec(128)) == (1, 0)
    assert engine.fit_plan(*_spec(150)) == (1, 1) and engine.fit_plan(*_spec(197)) is None
    machines = [_machine("t4", 4), _machine("t9", 9), _machine("t4b", 4), _machine("t17", 17), _machine("t80", 80), _machine("t96", 96),
                _machine("t128", 128), _machine("t150", 150), _machine("t197", 197), _machine("t200", 200)]
    groups = _names(builder.launch_groups(_buckets(machines)))
    assert groups == [[["t4", "t4b"], ["t9"], ["t17"], ["t80"]], [["t96"], ["t128"]], [["t150"]], [["t197"]], [["t200"]]]


@pytest.mark.parametrize("field", ["seed", "epochs", "rows", "kind", "kfcv"])
def test_any_other_key_field_keeps_buckets_apart(field):
    other = {
        "seed": dict(evaluation={"seed": 5}),
        "epochs": dict(model={"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": {
            "gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 3}}}}),
        "rows": dict(rows=240),
        "kind": dict(model={"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": {
            "gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_symmetric", "epochs": 2}}}}),
        "kfcv": dict(model=KFCV, evaluation=KFOLD),
    }[field]
    machines = [_machine("a", 4), _machine("b", 9, **other)]
    assert _names(builder.launch_groups(_buckets(machines))) == [[["a"]], [["b"]]]
    if field == "rows":  # ragged buckets leave the row count out of the key: they join
        assert _names(builder.launch_groups(_buckets(machines, ragged=True))) == [[["a"], ["b"]]]


def test_kfold_buckets_join_among_themselves():
    machines = [_machine("k4", 4, model=KFCV, evaluation=KFOLD), _machine("p4", 4), _machine("k33", 33, model=KFCV, evaluation=KFOLD),
                _machine("p33", 33)]
    assert _names(builder.launch_groups(_buckets(machines))) == [[["k4"], ["k33"]], [["p4"], ["p33"]]]


def _spec(tags):
    s = hourglass_spec(tags)
    return s.dims, s.acts, s.l1


def _fake_builds(monkeypatch, fail_joined=False):
    calls = []

    def fake_bucket(members):
        calls.append(("bucket", [c.machine["name"] for c in members]))
        return [(f"batched:{c.machine['name']}", builder._machine_out(c.machine, {"model": {}, "dataset": {}})) for c in members]

    def fake_joined(joined):
        calls.append(("joined", [[c.machine["name"] for c in members] for members in joined]))
        if fail_joined:
            raise RuntimeError("joined build failed")
        return [[(f"joined:{c.machine['name']}", builder._machine_out(c.machine, {"model": {}, "dataset": {}})) for c in members]
                for members in joined]

    monkeypatch.setattr(builder.FleetModelBuilder, "_build_bucket", staticmethod(fake_bucket))
    monkeypatch.setattr(builder.FleetModelBuilder, "_build_buckets_joined", staticmethod(fake_joined))
    return calls


def test_flagged_builder_builds_launch_groups_together(monkeypatch):
    calls = _fake_builds(monkeypatch)
    machines = [_machine("a", 4), _machine("b", 9), _machine("c", 4), _machine("d", 150)]
    full = builder.FleetModelBuilder(machines, mixed_widths=True)
    assert full.shard(0, 1).mixed_widths
    results = full.build()
    assert [m for m, _ in results] == ["joined:a", "joined:b", "joined:c", "batched:d"]
    assert calls == [("joined", [["a", "c"], ["b"]]), ("bucket", ["d"])]


def test_a_failed_joined_build_falls_back_to_its_buckets(monkeypatch):
    calls = _fake_builds(monkeypatch, fail_joined=True)
    results = builder.FleetModelBuilder([_machine("a", 4), _machine("b", 9)], mixed_widths=True).build()
    assert [m for m, _ in results] == ["batched:a", "batched:b"]
    assert calls == [("joined", [["a"], ["b"]]), ("bucket", ["a"]), ("bucket", ["b"])]


def test_without_the_flag_buckets_and_calls_are_unchanged(monkeypatch):
    calls = _fake_builds(monkeypatch)
    results = builder.FleetModelBuilder([_machine("a", 4), _machine("b", 9), _machine("c", 4)]).build()
    assert [m for m, _ in results] == ["batched:a", "batched:b", "batched:c"]
    assert calls == [("bucket", ["a", "c"]), ("bucket", ["b"])]
