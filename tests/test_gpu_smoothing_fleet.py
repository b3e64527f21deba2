"""
FleetModelBuilder(smoothing=True) end to end: feed-forward and LSTM detectors with windows 6, 12 and 144 (144 is longer than their
test blocks) and every smoothing method.  The smooth thresholds of every fold are what gb_thresholds gives at the window on the
fleet's own fold scores, bit for bit; everything else equals the same bucket built without a window; metadata.json carries
ModelBuilder's smooth keys; the models serve through ResidentBucket(smoothing=True) exactly as through the per-request route.
"""
import json
import os

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

T, ROWS = 4, 400  # test blocks of 100 rows (96 LSTM predictions)
DET = "gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector"
AE = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2}}
LSTM = {"gordo.machine.model.models.KerasLSTMAutoEncoder": {"kind": "lstm_hourglass", "lookback_window": 5, "epochs": 1, "batch_size": 16}}
SMOOTH_KEYS = {"smooth-feature-thresholds", "smooth-aggregate-threshold", "smooth-feature-thresholds-per-fold", "smooth-aggregate-thresholds-per-fold"}


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("needs an H100")
    import __graft_entry__ as ge

    ge.build()
    return t


def _series(seed):
    rng = np.random.default_rng(seed)
    t = np.linspace(0, 25, ROWS)[:, None]
    values = (0.5 + 0.4 * np.sin(t * rng.uniform(0.5, 2, T) + rng.uniform(0, 3, T)) + rng.normal(0, 0.02, (ROWS, T))) * rng.uniform(1, 50, T)
    idx = pd.date_range("2019-01-01", periods=ROWS, freq="10min", tz="UTC")
    return pd.DataFrame(values, index=idx, columns=[f"TAG {i}" for i in range(T)])


def _machine(name, base, seed, window=None, method=None):
    kw = {} if window is None else {"window": window, **({} if method is None else {"smoothing_method": method})}
    X = _series(seed)
    return {"name": name, "model": {DET: {"base_estimator": base, **kw}}, "dataset": {"X": X, "y": X}}


FF_SPECS = [("ff-w12-smm", 12, "smm"), ("ff-w12-sma", 12, "sma"), ("ff-w12-ewma", 12, "ewma"), ("ff-w6-a", 6, None), ("ff-w6-b", 6, "sma"),
            ("ff-w144-a", 144, None), ("ff-w144-b", 144, "ewma")]
LSTM_SPECS = [("lstm-w12-a", 12, "ewma"), ("lstm-w12-b", 12, "ewma"), ("lstm-w6", 6, "smm"), ("lstm-w144", 144, "sma")]


def _machines(windowed=True, only=None):
    """Every machine, or those of the bucket (kind, window) ``only``; without their windows unless ``windowed``."""
    out = []
    for kind, base, specs, seed0 in (("ff", AE, FF_SPECS, 0), ("lstm", LSTM, LSTM_SPECS, 100)):
        for k, (name, w, method) in enumerate(specs):
            if only is None or only == (kind, w):
                out.append(_machine(name, base, seed0 + k, w if windowed else None, method if windowed else None))
    return out


@pytest.fixture(scope="module")
def built(torch, tmp_path_factory):
    """The windowed fleet (with every gb_thresholds_pair call's arguments and results captured) and the same fleet without windows."""
    from gordo_components_b200 import builder, engine

    calls = []
    pair = engine.thresholds_pair

    def capture(*args):
        out = pair(*args)
        calls.append((args, out))
        return out

    root = tmp_path_factory.mktemp("smooth-fleet")
    engine.thresholds_pair = capture
    try:
        fmb = builder.FleetModelBuilder(_machines(), smoothing=True)
        for c in fmb.machines:  # every machine takes the batched path
            canon = builder._canonical_lstm(0, c, smoothing=True) if builder._is_lstm_definition(c) else builder._canonical(0, c, smoothing=True)
            assert canon is not None, c["name"]
        results = fmb.build(str(root))
    finally:
        engine.thresholds_pair = pair
    # each bucket again without its window (buckets draw their initial weights per bucket)
    plain = [r for key in [("ff", w) for w in (6, 12, 144)] + [("lstm", w) for w in (6, 12, 144)]
             for r in builder.FleetModelBuilder(_machines(windowed=False, only=key), smoothing=True).build()]
    return {"results": results, "plain": plain, "calls": calls, "root": str(root)}


def _by_name(results):
    return {m["name"]: det for det, m in results}


def _bits(a):
    a = np.asarray(a, dtype=np.float64)
    return a.view(np.int64)


def test_smooth_thresholds_are_the_window_thresholds_of_the_fold_scores(built, torch):
    from gordo_components_b200 import engine

    dets = _by_name(built["results"])
    # buckets: ff w12 (3 methods), ff w6, ff w144, lstm w12, lstm w6, lstm w144
    assert sorted(int(args[8]) for args, _ in built["calls"]) == [6, 6, 12, 12, 144, 144]
    for args, got in built["calls"]:
        jobs, n_jobs, max_rows, tu, ts, n_out, n_slots, w0, w1, dev = args
        assert w0 == 6
        want6 = engine.thresholds(jobs, n_jobs, max_rows, tu, ts, n_out, n_slots, 6, dev)
        wantw = engine.thresholds(jobs, n_jobs, max_rows, tu, ts, n_out, n_slots, w1, dev)
        for g, w in zip(got, want6 + wantw):
            assert np.array_equal(_bits(g.cpu().numpy()), _bits(w.cpu().numpy()))
        # the detectors of this bucket carry those values: fold k of machine m is job k*M + m
        lstm = tu.dtype == torch.float64
        names = [n for n, w, _ in (LSTM_SPECS if lstm else FF_SPECS) if w == w1]
        M, K = len(names), 3
        ofs = n_slots - K * M  # feed-forward slots start after the M final fits
        feat, agg = wantw[0].cpu().numpy().astype(np.float64), wantw[1].cpu().numpy().astype(np.float64)
        for m, name in enumerate(names):
            det = dets[name]
            assert det.window == w1
            rows = [feat[ofs + k * M + m] for k in range(K)]
            assert np.array_equal(_bits(det.smooth_feature_thresholds_per_fold_.to_numpy()), _bits(np.stack(rows)))
            assert list(det.smooth_feature_thresholds_per_fold_.index) == [f"fold-{k}" for k in range(K)]
            assert list(det.smooth_feature_thresholds_per_fold_.columns) == [f"TAG {i}" for i in range(T)]
            assert np.array_equal(_bits(list(det.smooth_aggregate_thresholds_per_fold_.values())), _bits([agg[ofs + k * M + m] for k in range(K)]))
            assert det.smooth_feature_thresholds_.name == f"fold-{K - 1}"
            assert np.array_equal(_bits(det.smooth_feature_thresholds_.to_numpy()), _bits(rows[-1]))
            assert np.array_equal(_bits(det.smooth_aggregate_threshold_), _bits(agg[ofs + (K - 1) * M + m]))
            assert np.isnan(det.smooth_aggregate_threshold_) == (w1 == 144)  # 100-row test blocks are shorter than the window


def test_everything_else_equals_the_build_without_a_window(built):
    dets, plain = _by_name(built["results"]), _by_name(built["plain"])
    methods = {n: m for n, _, m in FF_SPECS + LSTM_SPECS}
    for name, det in dets.items():
        ref = plain[name]
        assert det.smoothing_method == (methods[name] or "smm") and ref.window is None
        assert np.array_equal(_bits(det.feature_thresholds_per_fold_.to_numpy()), _bits(ref.feature_thresholds_per_fold_.to_numpy()))
        assert np.array_equal(_bits(list(det.aggregate_thresholds_per_fold_.values())), _bits(list(ref.aggregate_thresholds_per_fold_.values())))
        assert np.array_equal(_bits(det.feature_thresholds_.to_numpy()), _bits(ref.feature_thresholds_.to_numpy()))
        est, ref_est = (d.base_estimator for d in (det, ref))
        wa, wb = _leaves(est.model.weights), _leaves(ref_est.model.weights)
        assert len(wa) == len(wb) and all(np.array_equal(x, y) for x, y in zip(wa, wb))
        assert est._history.history == ref_est._history.history


def _leaves(w):
    if isinstance(w, (list, tuple)):
        return [leaf for item in w for leaf in _leaves(item)]
    return [w]


def _model_meta(meta):
    if isinstance(meta, dict):
        if "feature-thresholds" in meta:
            return meta
        for v in meta.values():
            found = _model_meta(v)
            if found is not None:
                return found
    return None


def test_metadata_carries_model_builders_smooth_keys(built):
    from gordo_components_b200 import builder

    for name, base, seed, window, method in (("ff-w12-sma", AE, 1, 12, "sma"), ("lstm-w12-a", LSTM, 100, 12, "ewma")):
        with open(os.path.join(built["root"], name, "metadata.json")) as f:
            fleet_meta = _model_meta(json.load(f))
        _, machine = builder.ModelBuilder(_machine(name, base, seed, window, method)).build()
        ref_meta = _model_meta(machine["metadata"])
        assert SMOOTH_KEYS <= set(ref_meta)
        assert set(fleet_meta) == set(ref_meta), set(fleet_meta) ^ set(ref_meta)
        assert fleet_meta["window"] == window and fleet_meta["smoothing-method"] == method
        assert list(fleet_meta["smooth-aggregate-thresholds-per-fold"]) == [f"fold-{k}" for k in range(3)]
        assert len(fleet_meta["smooth-feature-thresholds"]) == T


def test_fleet_models_serve_through_the_smoothing_bucket(built, torch, tmp_path):
    from gordo_components_b200 import serializer, server

    meta = {"dataset": {"tag_list": [f"TAG {t}" for t in range(T)], "resolution": "10min"}}
    dets = _by_name(built["results"])
    groups = {"ff": (["ff-w12-smm"], {}), "lstm": (["lstm-w12-a", "lstm-w12-b"], {"lstm": True})}
    for members, _ in groups.values():
        for n in members:
            serializer.dump(dets[n], str(tmp_path / n), metadata=meta)
    store = server.ModelStore(str(tmp_path))
    for members, kw in groups.values():
        bucket = server.ResidentBucket(store, names=members, smoothing=True, max_wait_ms=20, **kw)
        try:
            assert sorted(bucket.names) == sorted(members) and bucket.smoothing == (12, dets[members[0]].smoothing_method)
            for k in range(6):
                name = members[k % len(members)]
                X = _series(500 + k).iloc[: 60 + 20 * k]
                payload = {"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(X)}
                want = server.anomaly_prediction(store, name, json=payload, all_columns=True)
                got = server.anomaly_prediction(store, name, json=payload, all_columns=True, bucket=[bucket])
                assert want.status == got.status == 200
                assert json.dumps(got.body["data"]) == json.dumps(want.body["data"])
                assert "smooth-total-anomaly-scaled" in json.dumps(want.body["data"])
        finally:
            bucket.close()
