"""
The batched K-fold build on the H100: gb_gather_rows and gb_minmax_inverse_f32 against NumPy, every fit slot of
fleet.build_kfold_fleet against a one-slot replay on the rows that slot's estimator receives, the K-fold thresholds against the
per-machine code path run on the batched fold models, and the production definition end to end through FleetModelBuilder.
"""
import math
import pickle

import numpy as np
import pandas as pd
import pytest
from sklearn.model_selection import KFold
from sklearn.preprocessing import MinMaxScaler
from sklearn.utils import shuffle as sk_shuffle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def waves(rng, n, t):
    s = np.linspace(0, 20, n)[:, None]
    return 3.0 + np.sin(s * rng.uniform(0.5, 2, t) + rng.uniform(0, 6, t)) * rng.uniform(0.5, 4, t) + rng.normal(0, 0.05, (n, t))


# ------------------------------------------------------------------------------------------------ 1. the row kernels
@pytest.mark.parametrize("kind", ["f32", "f64", "f64-to-f32"])
@pytest.mark.parametrize("cols", [1, 3, 4, 8, 12])
def test_gather_rows_equals_fancy_indexing(torch, kind, cols):
    from gordo_components_b200 import engine

    dev = engine.cuda_device()
    rng = np.random.default_rng(cols)
    rows, total = 97, 5 * 97
    src = rng.normal(size=(total, cols)) * 1e3
    src = src.astype(np.float32) if kind == "f32" else src
    row_map = rng.permutation(rows).astype(np.int32)
    n = np.array([97, 50, 1, 0, 97])  # ragged jobs; one empty
    x_row = np.array([0, 97, 194, 291, 388])
    out_row = np.array([388, 0, 194, 291, 97])
    jobs = engine.jobs_to_device(engine.make_jobs(np.zeros(5, int), n, x_row, out_row), dev)
    s = torch.from_numpy(src).to(dev)
    out = torch.full((total, cols), -7.0, dtype=torch.float32 if kind != "f64" else torch.float64, device=dev)
    engine.gather_rows(jobs, 5, rows, torch.from_numpy(row_map).to(dev), s, total, to_f32=kind == "f64-to-f32", out=out)
    got = out.cpu().numpy()
    want = np.full_like(got, -7.0)
    for j in range(5):
        want[out_row[j]:out_row[j] + n[j]] = src[x_row[j] + row_map[:n[j]]]
    assert np.array_equal(got, want)


def test_gather_rows_beyond_one_launch_of_jobs(torch):
    from gordo_components_b200 import engine

    dev = engine.cuda_device()
    n_jobs, rows = 70000, 3
    src = np.arange(n_jobs * rows, dtype=np.float64).reshape(-1, 1)
    row_map = np.array([2, 0, 1], dtype=np.int32)
    base = np.arange(n_jobs, dtype=np.int64) * rows
    jobs = engine.jobs_to_device(engine.make_jobs(np.zeros(n_jobs, int), rows, base), dev)
    got = engine.gather_rows(jobs, n_jobs, rows, torch.from_numpy(row_map).to(dev), torch.from_numpy(src).to(dev), n_jobs * rows).cpu().numpy()
    assert np.array_equal(got, src[(base[:, None] + row_map[None, :]).ravel()])


def test_minmax_inverse_equals_sklearn_float32(torch):
    from gordo_components_b200 import engine

    dev = engine.cuda_device()
    rng = np.random.default_rng(3)
    T, S, rows = 9, 3, 50
    y = [waves(rng, 200, T) * 100 for _ in range(S)]
    scalers = [MinMaxScaler().fit(v) for v in y]
    pred = rng.normal(0.5, 0.4, (S * rows, T)).astype(np.float32)
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(S), rows, np.arange(S) * rows), dev)
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    res = engine.minmax_inverse_f32(jobs, S, rows, f(pred), f(np.stack([s.scale_ for s in scalers])), f(np.stack([s.min_ for s in scalers])))
    for s, sc in enumerate(scalers):
        want = sc.inverse_transform(pred[s * rows:(s + 1) * rows])
        assert want.dtype == np.float32
        assert np.array_equal(res["f32"][s * rows:(s + 1) * rows].cpu().numpy(), want)
        assert np.array_equal(res["f64"][s * rows:(s + 1) * rows].cpu().numpy(), want.astype(np.float64))


# ------------------------------------------------------------------------------------------------ 2. fit replay, slot by slot
@pytest.mark.parametrize("K", [3, 5])
@pytest.mark.parametrize("detector_shuffle", [True, False])
@pytest.mark.parametrize("form", ["pipeline", "ttr"])
def test_every_fit_slot_replays(torch, K, detector_shuffle, form):
    from gordo_components_b200 import engine, fleet
    from gordo_components_b200.machine.model.factories.feedforward_autoencoder import feedforward_hourglass
    from gordo_components_b200.machine.model.models import EarlyStopping

    M, N, T, E, B, vsplit = 3, 211, 8, 8, 32, 0.1
    spec = feedforward_hourglass(n_features=T, compression_factor=0.5, encoding_layers=1, func="tanh", out_func="linear")
    eng = engine.ff_engine_for(spec)
    rng = np.random.default_rng(K)
    X = np.concatenate([waves(rng, N, T) for _ in range(M)])
    xd = torch.from_numpy(X).to(eng.device)
    rules = [dict(monitor="val_loss", patience=1, min_delta=1.0, restore_best_weights=False),
             dict(monitor="val_loss", patience=2, min_delta=2e-3, restore_best_weights=True),
             dict(monitor="val_loss", patience=E, restore_best_weights=True)]
    cv = KFold(K, shuffle=True, random_state=0)
    input_scaler, target_scaler = form == "pipeline", form == "ttr"
    fb = fleet.build_kfold_fleet(eng, xd, xd, N, cv, epochs=E, batch_size=B, seed=5, adam=spec.adam, shuffle=False, input_scaler=input_scaler,
                                 target_scaler=target_scaler, detector_shuffle=detector_shuffle, validation_split=vsplit,
                                 early_stopping=[EarlyStopping(**r) for r in rules], window=12, smoothing_method="smm", keep_init_params=True)
    folds = list(cv.split(np.arange(N)))
    stopped = 0
    for m in range(M):
        Xm = X[m * N:(m + 1) * N]
        for j, rows in enumerate([np.arange(N)] + [tr for tr, _ in folds]):
            slot = m if j == 0 else M + (j - 1) * M + m
            received = sk_shuffle(Xm[rows], random_state=0) if detector_shuffle else Xm[rows]
            sc = MinMaxScaler().fit(Xm[rows])  # the Pipeline's input scaler, or the target transformer: both see the slot's rows
            xs = torch.from_numpy(sc.transform(received).astype(np.float32) if input_scaler else received.astype(np.float32)).to(eng.device)
            ys = torch.from_numpy(sc.transform(received).astype(np.float32) if target_scaler else received.astype(np.float32)).to(eng.device)
            n = len(rows)
            n_train = int(math.floor(n * (1 - vsplit)))
            p = fb.init_params[slot:slot + 1].clone()
            tj = engine.jobs_to_device(engine.make_jobs([0], [n_train], [0]), eng.device)
            loss, _, vl, _, ran, _, _ = eng.fit_split(p, tj, 1, n, xs, ys, split=engine.make_split([n - n_train]), val_batch=B, epochs=E, batch_size=B,
                                                      shuffle=False, adam=spec.adam, seed=5, stop=engine.make_stop([rules[m]]))
            ran = int(ran[0])
            stopped += ran < E
            assert int(fb.epochs_run[slot]) == ran, (m, j, "epochs run")
            assert torch.equal(fb.params[slot], p[0]), (m, j, "weights")
            assert np.array_equal(fb.loss[slot], loss[0].cpu().numpy(), equal_nan=True), (m, j, "loss")
            assert np.array_equal(fb.val_loss[slot], vl[0].cpu().numpy(), equal_nan=True), (m, j, "val_loss")
    assert stopped >= K + 1


# ------------------------------------------------------------------------------------------------ 3. thresholds against the per-machine path
AE = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "batch_size": 64, "compression_factor": 0.5,
                                                      "encoding_layers": 1, "func": "tanh", "out_func": "linear", "epochs": 3}}
PIPE = {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", AE]}}


def ttr(regressor):
    return {"sklearn.compose.TransformedTargetRegressor": {"transformer": "sklearn.preprocessing.MinMaxScaler", "regressor": regressor}}


FORMS = {"bare": AE, "pipeline": PIPE, "ttr-bare": ttr(AE), "ttr-pipeline": ttr(PIPE)}


@pytest.mark.parametrize("form,method,window,rows", [
    ("bare", "smm", 12, 240), ("pipeline", "sma", 12, 240), ("pipeline", "ewma", 12, 240), ("pipeline", "smm", None, 240),
    ("ttr-bare", "smm", 12, 240), ("ttr-pipeline", "ewma", 12, 240), ("pipeline", "smm", 144, 100),
])
def test_thresholds_equal_the_per_machine_path(torch, form, method, window, rows):
    """
    Exact in every form.  The TransformedTargetRegressor route reproduces sklearn's float32 inverse transform
    (gb_minmax_inverse_f32) and then scores in float64 as the per-machine detector scores a foreign estimator, so it is exact too.
    rows < window: every smoothed value is NaN, and so are the thresholds, as per machine.
    """
    from gordo_components_b200 import engine, fleet, serializer

    definition = {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {
        "base_estimator": FORMS[form], "scaler": "sklearn.preprocessing.MinMaxScaler", "window": window, "smoothing_method": method,
        "shuffle": True, "threshold_percentile": 0.975}}
    M, T, K = 3, 6, 3
    rng = np.random.default_rng(rows)
    frames = [pd.DataFrame(waves(rng, rows, T) * 10, columns=[f"tag-{c}" for c in range(T)]) for _ in range(M)]
    template = serializer.from_definition(definition)
    ae = template.base_estimator
    ae = getattr(ae, "regressor", ae)
    ae = ae.steps[-1][1] if hasattr(ae, "steps") else ae
    ae.kwargs.update({"n_features": T, "n_features_out": T})
    spec = ae._build_spec()
    eng = engine.ff_engine_for(spec)
    xd = torch.from_numpy(np.concatenate([f.values for f in frames])).to(eng.device)  # column-major: the build takes any strides
    cv = KFold(K, shuffle=True, random_state=0)
    fb = fleet.build_kfold_fleet(eng, xd, xd, rows, cv, epochs=3, batch_size=64, seed=1, adam=spec.adam, input_scaler="pipeline" in form,
                                 target_scaler=form.startswith("ttr"), detector_shuffle=True, window=window, smoothing_method=method,
                                 threshold_percentile=0.975)
    tags = list(frames[0].columns)
    for m, frame in enumerate(frames):
        folds = [fb.fold_detector(m, k, serializer.from_definition(definition), tags=tags, input_tags=tags) for k in range(K)]
        feat, agg = serializer.from_definition(definition).kfold_thresholds(frame, frame, cv, folds)
        assert np.array_equal(fb.feat_thr[m], feat.values, equal_nan=True), (m, fb.feat_thr[m], feat.values)
        assert np.array_equal(fb.agg_thr[m], agg, equal_nan=True), (m, fb.agg_thr[m], agg)
        if window is not None and rows < window:
            assert np.isnan(fb.feat_thr[m]).all() and np.isnan(fb.agg_thr[m])
        else:
            assert np.isfinite(fb.feat_thr[m]).all() and np.isfinite(fb.agg_thr[m])
        det = fb.detector(m, serializer.from_definition(definition), tags=tags, input_tags=tags)
        assert det.feature_thresholds_.index.tolist() == tags and det.feature_thresholds_.name is None


# ------------------------------------------------------------------------------------------------ 4. the production definition end to end
def test_fleet_builder_builds_the_kfold_production_definition(torch, tmp_path):
    from gordo_components_b200 import builder, serializer

    E = 6
    ae = {"gordo.machine.model.models.KerasAutoEncoder": {
        "kind": "feedforward_hourglass", "batch_size": 128, "compression_factor": 0.5, "encoding_layers": 1, "func": "tanh", "out_func": "linear",
        "epochs": E, "validation_split": 0.1,
        "callbacks": [{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "val_loss", "patience": 1, "min_delta": 0.5, "restore_best_weights": True}}]}}
    model = {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {
        "base_estimator": {"sklearn.compose.TransformedTargetRegressor": {
            "transformer": "sklearn.preprocessing.MinMaxScaler",
            "regressor": {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", ae]}}}},
        "scaler": "sklearn.preprocessing.MinMaxScaler", "window": 144, "shuffle": True, "threshold_percentile": 0.975}}
    evaluation = {"cv": {"sklearn.model_selection.KFold": {"n_splits": 5, "shuffle": True, "random_state": 0}}}
    N, T = 1500, 12
    idx = pd.date_range("2019-01-01", periods=N, freq="10min", tz="UTC")
    rng = np.random.default_rng(9)
    machines = []
    for i in range(3):
        frame = pd.DataFrame(waves(rng, N, T), index=idx, columns=[f"tag-{c}" for c in range(T)])
        machines.append({"name": f"prod-{i}", "model": model, "dataset": {"X": frame, "y": frame}, "evaluation": evaluation})
    assert all(builder._canonical_kfcv(i, m, early_stopping=True) is not None for i, m in enumerate(machines))
    calls = []
    orig = builder.FleetModelBuilder._build_bucket
    builder.FleetModelBuilder._build_bucket = staticmethod(lambda members: calls.append(len(members)) or orig(members))
    try:
        fleet_out = builder.FleetModelBuilder(machines, early_stopping=True, kfcv=True).build(str(tmp_path))
    finally:
        builder.FleetModelBuilder._build_bucket = staticmethod(orig)
    assert calls == [3]  # one batched bucket, no fall-back
    single_model, single_meta = builder.ModelBuilder(dict(machines[0])).build()

    def keys(d):
        return {k: keys(v) for k, v in d.items()} if isinstance(d, dict) else None

    for (model_, meta), m in zip(fleet_out, machines):
        assert keys(meta) == keys(single_meta)
        cvm = meta["metadata"]["build_metadata"]["model"]["cross_validation"]
        assert cvm["splits"] == builder.build_split_dict(m["dataset"]["X"], KFold(5, shuffle=True, random_state=0))
        assert all(np.isfinite(v["fold-mean"]) for v in cvm["scores"].values())
        assert sorted(vars(model_.base_estimator)) == sorted(vars(single_model.base_estimator))
        assert sorted(vars(model_.base_estimator.transformer_)) == sorted(vars(single_model.base_estimator.transformer_))
        reg = model_.base_estimator.regressor_
        ran = len(reg.steps[-1][1]._history.epoch)
        assert 1 <= ran <= E
        hist = meta["metadata"]["build_metadata"]["model"]["model_meta"]["history"]
        assert list(hist) == ["loss", "accuracy", "val_loss", "val_accuracy", "params"] and hist["params"]["epochs"] == E
        assert all(len(hist[k]) == ran for k in ("loss", "accuracy", "val_loss", "val_accuracy"))
    assert all(len(r.base_estimator.regressor_.steps[-1][1]._history.epoch) < E for r, _ in fleet_out)  # min_delta 0.5: the patience fires
    for m in machines:
        with open(tmp_path / m["name"] / "model.pkl", "rb") as f:
            det = pickle.load(f)
        frame = m["dataset"]["X"]
        out = det.anomaly(frame.iloc[:300], frame.iloc[:300])
        assert np.isfinite(out["total-anomaly-scaled"].values).all()
        assert np.isfinite(out["total-anomaly-confidence"].values).all()
        assert serializer.load_metadata(str(tmp_path / m["name"]))["name"] == m["name"]
