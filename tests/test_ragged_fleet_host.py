"""
Machines of different lengths in one batched build, without a device: the bucket keys with and without
FleetModelBuilder(ragged=True), every machine's own fold layout and row maps against sklearn, the argument checks of
gb_gather_rows_ragged, and how a mixed-length project is grouped.
"""
import ctypes as C

import numpy as np
import pandas as pd
import pytest
from sklearn.model_selection import KFold, TimeSeriesSplit
from sklearn.utils import shuffle as sk_shuffle

from gordo_components_b200 import _cabi, builder, fleet

AE = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2}}
KFOLD = {"sklearn.model_selection.KFold": {"n_splits": 5, "shuffle": True, "random_state": 0}}
LENGTHS = [103, 211, 240, 1000, 211]


def _frame(rows, tags=4, seed=0):
    idx = pd.date_range("2020-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(np.random.default_rng(seed).random((rows, tags)), index=idx, columns=[f"tag-{i}" for i in range(tags)])


def _machine(name, model, rows=200, evaluation=None):
    X = _frame(rows)
    return {"name": name, "model": model, "dataset": {"X": X, "y": X}, **({"evaluation": evaluation} if evaluation else {})}


def _ff(**kw):
    est = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2, **kw}}
    return {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": est}}


def _lstm(**kw):
    est = {"gordo.machine.model.models.KerasLSTMAutoEncoder": {"kind": "lstm_hourglass", "lookback_window": 6, "epochs": 2, "batch_size": 16, **kw}}
    return {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": est}}


def _kfcv(**det):
    return {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {"base_estimator": AE, "window": 12, **det}}


FAMILIES = {
    "feedforward": (lambda m: builder._canonical(0, m), _ff, dict(epochs=3), None),
    "lstm": (lambda m: builder._canonical_lstm(0, m), _lstm, dict(lookback_window=8), None),
    "kfold": (lambda m: builder._canonical_kfcv(0, m), _kfcv, dict(window=24), {"cv": KFOLD}),
}


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_bucket_keys_leave_out_the_length_only_with_the_flag(family):
    canonical, model, other, evaluation = FAMILIES[family]
    a = canonical(_machine("a", model(), 200, evaluation))
    b = canonical(_machine("b", model(), 300, evaluation))
    assert a is not None and b is not None
    assert a.bucket() != b.bucket() and a.bucket(False) == a.bucket()  # the default keys are today's
    assert a.bucket(ragged=True) == b.bucket(ragged=True)
    changed = canonical(_machine("c", model(**other), 300, evaluation))
    assert changed is not None and changed.bucket(ragged=True) != a.bucket(ragged=True)
    seeded = canonical(_machine("d", model(), 300, {**(evaluation or {}), "seed": 7}))
    assert seeded.bucket(ragged=True) != a.bucket(ragged=True)


def test_timeseries_layout_of_every_machine_is_sklearns():
    for K in (3, 5):
        test, starts = fleet.tss_layout(LENGTHS, K)
        assert test.shape == (len(LENGTHS),) and starts.shape == (len(LENGTHS), K)
        for m, n in enumerate(LENGTHS):
            for k, (train, te) in enumerate(TimeSeriesSplit(K).split(np.arange(n))):
                assert len(train) == starts[m, k] and np.array_equal(te, np.arange(starts[m, k], starts[m, k] + test[m]))
    with pytest.raises(ValueError):
        fleet.tss_layout([100, 3], 3)


def test_shuffle_maps_are_sklearns_per_slot_length():
    _, starts = fleet.tss_layout(LENGTHS, 3)
    slot_n = np.concatenate([LENGTHS] + [starts[:, k] for k in range(3)])
    maps, ofs = fleet.shuffle_maps(slot_n)
    assert maps.dtype == np.int32 and ofs.dtype == np.int64 and len(ofs) == len(slot_n)
    assert len(maps) == sum(set(int(v) for v in slot_n))  # one map per distinct length
    for s, n in enumerate(slot_n):
        assert np.array_equal(maps[ofs[s]:ofs[s] + n], sk_shuffle(np.arange(n), random_state=0))
    # equal lengths: the maps of the equal-length build, in the same order
    uniform, u_ofs = fleet.shuffle_maps(np.repeat([240, 60, 120, 180], 4))
    assert np.array_equal(uniform, np.concatenate([sk_shuffle(np.arange(n), random_state=0) for n in (240, 60, 120, 180)]))
    assert np.array_equal(u_ofs, np.repeat([0, 240, 300, 420], 4))


@pytest.mark.parametrize("detector_shuffle", [False, True])
def test_kfold_maps_of_every_machine_are_its_lengths(detector_shuffle):
    cv = KFold(5, shuffle=True, random_state=0)
    M, K = len(LENGTHS), 5
    n_test, to_fold, to_time, machine_ofs, fit_maps, slot_ofs = fleet.kfold_bucket_maps(cv, LENGTHS, detector_shuffle)
    assert n_test.shape == (M, K) and len(slot_ofs) == M * (K + 1)
    assert machine_ofs[1] == machine_ofs[4]  # the repeated length shares its maps
    assert len(to_fold) == len(to_time) == sum(set(LENGTHS))
    for m, n in enumerate(LENGTHS):
        tests, trains, order, inverse = fleet.kfold_layout(cv, n)
        assert list(n_test[m]) == [len(t) for t in tests]
        assert np.array_equal(to_fold[machine_ofs[m]:machine_ofs[m] + n], order)
        assert np.array_equal(to_time[machine_ofs[m]:machine_ofs[m] + n], inverse)
        want = fleet.kfold_row_maps(trains, inverse, n, detector_shuffle)
        for j in range(K + 1):  # the final fit (j = 0), then fold j - 1, of machine m: slot j*M + m
            o = slot_ofs[j * M + m]
            assert np.array_equal(fit_maps[o:o + len(want[j])], want[j]), (m, j)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def test_gather_rows_ragged_refuses_bad_arguments_without_a_device(lib):
    fake = C.c_void_p(256)  # never dereferenced: every check runs before any launch
    good = dict(jobs=fake, n_jobs=2, max_rows=4, row_map=fake, map_ofs=fake, src=fake, n_cols=3, elem_bytes=4, to_f32=0, dst=fake)

    def call(**kw):
        a = {**good, **kw}
        return lib.gb_gather_rows_ragged(a["jobs"], a["n_jobs"], a["max_rows"], a["row_map"], a["map_ofs"], a["src"], a["n_cols"], a["elem_bytes"],
                                         a["to_f32"], a["dst"], None)

    cases = [(dict(map_ofs=None), b"map_ofs"), (dict(map_ofs=None, n_jobs=0), b"map_ofs"), (dict(jobs=None), b"non-NULL"),
             (dict(row_map=None), b"non-NULL"), (dict(src=None), b"non-NULL"), (dict(dst=None), b"non-NULL"), (dict(elem_bytes=2), b"elem_bytes"),
             (dict(to_f32=1), b"to_f32"), (dict(n_cols=0), b"n_cols"), (dict(max_rows=-1), b"max_rows"), (dict(n_jobs=-1), b"n_jobs")]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        assert msg in lib.gb_last_error(), (kw, lib.gb_last_error())
    assert call(n_jobs=0) == 0 and call(max_rows=0) == 0  # nothing to launch


def test_a_mixed_length_project_is_one_bucket_per_family(monkeypatch):
    buckets = []

    def fake_bucket(members):
        buckets.append(sorted(c.machine["name"] for c in members))
        return [(c.machine["name"], builder._machine_out(c.machine, {"model": {}, "dataset": {}})) for c in members]

    monkeypatch.setattr(builder.FleetModelBuilder, "_build_bucket", staticmethod(fake_bucket))
    monkeypatch.setattr(builder.ModelBuilder, "build", lambda self, output_dir=None: pytest.fail(f"{self.machine['name']} built alone"))
    machines = []
    for i, rows in enumerate([120, 300, 200, 421]):
        machines += [_machine(f"ff-{i}", _ff(), rows), _machine(f"lstm-{i}", _lstm(), rows), _machine(f"kf-{i}", _kfcv(), rows, {"cv": KFOLD})]
    ragged = builder.FleetModelBuilder(machines, kfcv=True, ragged=True)
    results = ragged.build()
    assert [name for name, _ in results] == [m["name"] for m in machines]
    assert sorted(buckets) == [[f"{f}-{i}" for i in range(4)] for f in ("ff", "kf", "lstm")]
    buckets.clear()
    builder.FleetModelBuilder(machines, kfcv=True).build()
    assert len(buckets) == 12  # without the flag every length is its own bucket
    assert all(s.ragged for s in (ragged.shard(r, 3) for r in range(3)))
    assert not builder.FleetModelBuilder(machines).shard(0, 2).ragged
