"""
Machines of different lengths in one batched build, on the H100: gb_gather_rows_ragged against NumPy, every fit slot of the
three fleet builds on per-machine row counts against a one-slot replay from its initial parameters, the fold predictions,
thresholds and CV scores against each machine on its own, an equal-length project built alike with and without
FleetModelBuilder(ragged=True), and a project of three machines of different lengths built in one bucket and served.
"""
import math
import os
import pickle

import numpy as np
import pandas as pd
import pytest
from sklearn import metrics as sk_metrics
from sklearn.model_selection import KFold
from sklearn.preprocessing import MinMaxScaler
from sklearn.utils import shuffle as sk_shuffle

pytestmark = pytest.mark.gpu

KERAS_ADAM = {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7}


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("no CUDA device")
    import __graft_entry__ as ge

    ge.build()
    return t


def waves(rng, n, t):
    s = np.linspace(0, 20, n)[:, None]
    return 3.0 + np.sin(s * rng.uniform(0.5, 2, t) + rng.uniform(0, 6, t)) * rng.uniform(0.5, 4, t) + rng.normal(0, 0.05, (n, t))


# ------------------------------------------------------------------------------------------------ 1. the gather kernel
@pytest.mark.parametrize("kind", ["f32", "f64", "f64-to-f32"])
@pytest.mark.parametrize("cols", [1, 3, 4, 8, 12])
def test_gather_rows_ragged_equals_fancy_indexing(torch, kind, cols):
    from gordo_components_b200 import engine

    dev = engine.cuda_device()
    rng = np.random.default_rng(cols)
    n = np.array([97, 50, 1, 0, 61, 97])  # ragged jobs; one empty
    lengths = [97, 50, 61]
    maps = [rng.permutation(v).astype(np.int32) for v in lengths]
    first = np.concatenate([[0], np.cumsum(lengths)[:-1]])
    map_ofs = np.array([first[0], first[1], first[1], first[2], first[2], first[0]], dtype=np.int64)  # jobs share maps
    x_row = np.concatenate([[0], np.cumsum(n)[:-1]])
    out_row = 3 + np.concatenate([np.cumsum(n[::-1])[::-1][1:], [0]])  # the blocks in reverse job order, 3 rows in
    total = int(n.sum()) + 3
    src = rng.normal(size=(total, cols)) * 1e3
    src = src.astype(np.float32) if kind == "f32" else src
    jobs = engine.jobs_to_device(engine.make_jobs(np.zeros(len(n), int), n, x_row, out_row), dev)
    row_map = torch.from_numpy(np.concatenate(maps)).to(dev)
    out = torch.full((total, cols), -7.0, dtype=torch.float32 if kind != "f64" else torch.float64, device=dev)
    engine.gather_rows(jobs, len(n), int(n.max()), row_map, torch.from_numpy(src).to(dev), total, to_f32=kind == "f64-to-f32", out=out,
                       map_ofs=torch.from_numpy(map_ofs).to(dev))
    got = out.cpu().numpy()
    cat = np.concatenate(maps)
    want = np.full_like(got, -7.0)
    for j in range(len(n)):
        want[out_row[j]:out_row[j] + n[j]] = src[x_row[j] + cat[map_ofs[j]:map_ofs[j] + n[j]]]
    assert np.array_equal(got, want)
    # all offsets 0: the bytes of gb_gather_rows
    shared = torch.from_numpy(maps[0]).to(dev)
    same = np.minimum(n, 97)
    jobs = engine.jobs_to_device(engine.make_jobs(np.zeros(len(n), int), same, x_row, out_row), dev)
    a = engine.gather_rows(jobs, len(n), 97, shared, torch.from_numpy(src).to(dev), total, to_f32=kind == "f64-to-f32")
    b = engine.gather_rows(jobs, len(n), 97, shared, torch.from_numpy(src).to(dev), total, to_f32=kind == "f64-to-f32",
                           map_ofs=torch.zeros(len(n), dtype=torch.int64, device=dev))
    torch.cuda.synchronize()
    rows = np.concatenate([np.arange(o, o + k) for o, k in zip(out_row, same)])  # rows outside every job are uninitialised
    assert np.array_equal(a.cpu().numpy()[rows].view(np.uint8), b.cpu().numpy()[rows].view(np.uint8))


def test_gather_rows_ragged_beyond_one_launch_of_jobs(torch):
    from gordo_components_b200 import engine

    dev = engine.cuda_device()
    n_jobs = 70000
    n = np.where(np.arange(n_jobs) % 2 == 0, 3, 2)
    maps = np.array([2, 0, 1, 1, 0], dtype=np.int32)  # a 3-row map at 0, a 2-row map at 3
    map_ofs = np.where(n == 3, 0, 3).astype(np.int64)
    base = np.concatenate([[0], np.cumsum(n)[:-1]])
    src = np.arange(int(n.sum()), dtype=np.float64).reshape(-1, 1)
    jobs = engine.jobs_to_device(engine.make_jobs(np.zeros(n_jobs, int), n, base), dev)
    got = engine.gather_rows(jobs, n_jobs, 3, torch.from_numpy(maps).to(dev), torch.from_numpy(src).to(dev), len(src),
                             map_ofs=torch.from_numpy(map_ofs).to(dev)).cpu().numpy()
    want = np.concatenate([src[b + maps[o:o + k]] for b, o, k in zip(base, map_ofs, n)])
    assert np.array_equal(got, want)


# ------------------------------------------------------------------------------------------------ 2. build_fleet
FF_LENGTHS = [211, 317, 160]


@pytest.mark.parametrize("input_scaler", [False, True])
def test_ragged_build_fleet_replays_every_slot(torch, input_scaler):
    from gordo_components_b200 import builder, engine, fleet
    from gordo_components_b200.machine.model.models import EarlyStopping
    from oracle import keras_math as km

    T, K, E, B, vsplit = 8, 3, 8, 32, 0.1
    spec = km.ff_hourglass_spec(T)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    rng = np.random.default_rng(7)
    Xs = [waves(rng, n, T).astype(np.float32) for n in FF_LENGTHS]
    X = np.concatenate(Xs)
    xd = torch.from_numpy(X).to(eng.device)
    rules = [dict(monitor="val_loss", patience=1, min_delta=1.0, restore_best_weights=False),
             dict(monitor="val_loss", patience=2, min_delta=2e-3, restore_best_weights=True),
             dict(monitor="loss", patience=E, restore_best_weights=True)]
    fb = fleet.build_fleet(eng, xd, xd, FF_LENGTHS, epochs=E, batch_size=B, n_splits=K, seed=3, adam=KERAS_ADAM, shuffle=False,
                           input_scaler=input_scaler, detector_shuffle=True, validation_split=vsplit,
                           early_stopping=[EarlyStopping(**r) for r in rules], keep_init_params=True)
    torch.cuda.synchronize()
    M = len(FF_LENGTHS)
    test, starts = fleet.tss_layout(FF_LENGTHS, K)
    assert list(fb.rows) == FF_LENGTHS and list(fb.n_test) == list(test)
    assert list(fb.machine_steps) == [math.ceil(math.floor(n * (1 - vsplit)) / B) for n in FF_LENGTHS]
    stopped = 0
    for m, Xm in enumerate(Xs):
        for j, n in enumerate([FF_LENGTHS[m]] + list(starts[m])):
            slot = m if j == 0 else M + (j - 1) * M + m
            received = sk_shuffle(Xm[:n], random_state=0)
            xin = MinMaxScaler().fit(Xm[:n].astype(np.float64)).transform(received.astype(np.float64)).astype(np.float32) if input_scaler else received
            n_train = int(math.floor(n * (1 - vsplit)))
            p = fb.init_params[slot:slot + 1].clone()
            tj = engine.jobs_to_device(engine.make_jobs([0], [n_train], [0]), eng.device)
            loss, _, vl, _, ran, _, _ = eng.fit_split(p, tj, 1, n, torch.from_numpy(np.ascontiguousarray(xin)).to(eng.device),
                                                      torch.from_numpy(np.ascontiguousarray(received)).to(eng.device), split=engine.make_split([n - n_train]),
                                                      val_batch=B, epochs=E, batch_size=B, shuffle=False, adam=KERAS_ADAM, seed=3,
                                                      stop=engine.make_stop([rules[m]]))
            ran = int(ran[0])
            stopped += ran < E
            got_p = fb.params[m] if j == 0 else fb.fold_params[m, j - 1]
            got_l = fb.loss[m] if j == 0 else fb.fold_loss[m, j - 1]
            got_v = fb.val_loss[m] if j == 0 else fb.fold_val_loss[m, j - 1]
            got_ran = fb.epochs_run[m] if j == 0 else fb.fold_epochs_run[m, j - 1]
            assert int(got_ran) == ran, (m, j, "epochs run")
            assert torch.equal(got_p, p[0]), (m, j, "weights")
            assert np.array_equal(got_l.cpu().numpy(), loss[0].cpu().numpy(), equal_nan=True), (m, j, "loss")
            assert np.array_equal(got_v.cpu().numpy(), vl[0].cpu().numpy(), equal_nan=True), (m, j, "val_loss")
    assert stopped >= 1

    # fold thresholds and CV scores: each machine's fold models on its own test blocks, one machine at a time
    for m, Xm in enumerate(Xs):
        tm = int(test[m])
        scaler = MinMaxScaler().fit(Xm.astype(np.float64))
        got_scores = builder.scores_from_moments(fb.cv_moments[m].cpu().numpy(), tm, fb.scale[m].cpu().numpy())
        for k in range(K):
            s = int(starts[m, k])
            prefix = Xm[:s]
            xin = Xm if not input_scaler else MinMaxScaler().fit(prefix.astype(np.float64)).transform(Xm.astype(np.float64)).astype(np.float32)
            one = engine.jobs_to_device(engine.make_jobs([0], [s], [0]), eng.device)
            sc, _ = eng.minmax_fit(one, 1, s, torch.from_numpy(np.ascontiguousarray(Xm)).to(eng.device), 1)
            jobs = engine.jobs_to_device(engine.make_jobs([0], [tm], [s], [0]), eng.device)
            res = eng.infer_score(fb.fold_params[m, k:k + 1].contiguous(), jobs, 1, tm, torch.from_numpy(np.ascontiguousarray(xin)).to(eng.device),
                                  torch.from_numpy(np.ascontiguousarray(Xm)).to(eng.device), sc, out_rows=tm)
            out_jobs = engine.jobs_to_device(engine.make_jobs([0], [tm], [0]), eng.device)
            feat, agg = eng.thresholds(out_jobs, 1, tm, res["tag-anomaly-unscaled"], res["total-anomaly-scaled"], 1, window=6)
            assert torch.equal(fb.fold_feat_thr[m, k], feat[0]), (m, k, "feature thresholds")
            assert torch.equal(fb.fold_agg_thr[m, k], agg[0]), (m, k, "aggregate threshold")
            pred = res["model-output"].cpu().numpy()
            yt, yp = scaler.transform(Xm[s:s + tm].astype(np.float64)), scaler.transform(pred.astype(np.float64))
            for name in builder.MOMENT_METRICS:
                func = getattr(sk_metrics, name)
                np.testing.assert_allclose(got_scores[name][1][k], func(yt, yp), rtol=1e-5, atol=1e-7, err_msg=f"{name} machine {m} fold {k}")
        det = fb.detector(m)
        assert det.base_estimator.get_metadata()["history"]["params"]["steps"] == fb.machine_steps[m]


# ------------------------------------------------------------------------------------------------ 3. build_lstm_fleet
LSTM_LENGTHS = [130, 171, 97, 130]


@pytest.mark.parametrize("scaled", [False, True], ids=["bare", "minmax"])
def test_ragged_lstm_fleet_replays_every_slot(torch, scaled):
    from gordo_components_b200 import engine, fleet
    from oracle import anomaly_math as am
    from oracle import keras_math as km

    T, L, K, E, B, la = 4, 6, 3, 2, 16, 0
    spec = km.lstm_model_spec(T, T, lookback_window=L, encoding_dim=(8,), encoding_func=("tanh",), decoding_dim=(8,), decoding_func=("tanh",))
    eng = engine.LSTMEngine(spec.n_features, spec.units, spec.acts, spec.n_features_out, spec.out_func, spec.lookback_window)
    rng = np.random.default_rng(11)
    Xs = [waves(rng, n, T).astype(np.float32).astype(np.float64) for n in LSTM_LENGTHS]
    xd = torch.from_numpy(np.concatenate(Xs)).to(eng.device)
    # a budget of two machines per fit launch: the chunks take the machines shortest first
    budget = eng.fit_workspace_bytes_for_batch(2 * (K + 1), B)
    fb = fleet.build_lstm_fleet(eng, xd, xd, LSTM_LENGTHS, epochs=E, batch_size=B, n_splits=K, seed=4, adam=KERAS_ADAM, input_scaler=scaled,
                                memory_budget=budget, keep_init_params=True)
    torch.cuda.synchronize()
    M = len(LSTM_LENGTHS)
    test, starts = fleet.tss_layout(LSTM_LENGTHS, K)
    assert list(fb.rows) == LSTM_LENGTHS and np.array_equal(fb.machine_starts, starts) and list(fb.machine_n_test) == list(test - L + 1 - la)
    assert list(fb.machine_steps) == [math.ceil((n - L + 1) / B) for n in LSTM_LENGTHS]
    fit = eng.fit_for_batch(B)
    for m, Xm in enumerate(Xs):
        for j, n in enumerate([LSTM_LENGTHS[m]] + list(starts[m])):
            slot = m if j == 0 else M + (j - 1) * M + m
            prefix = Xm[:n]
            x_in = MinMaxScaler().fit(prefix).transform(Xm).astype(np.float32) if scaled else Xm.astype(np.float32)
            p = fb.init_params[slot:slot + 1].clone()
            jobs = engine.jobs_to_device(engine.make_jobs([0], [n - L + 1], [0]), eng.device)
            loss, _, _ = fit(p, jobs, 1, n - L + 1, torch.from_numpy(np.ascontiguousarray(x_in)).to(eng.device),
                             torch.from_numpy(Xm.astype(np.float32)).to(eng.device), epochs=E, batch_size=B, lookahead=la, primer=True, adam=KERAS_ADAM)
            got = fb.params[m] if j == 0 else fb.fold_params[m, j - 1]
            assert torch.equal(got, p[0]), (m, j, "weights")
            assert np.array_equal(fb.loss[m] if j == 0 else fb.fold_loss[m, j - 1], loss[0].cpu().numpy()), (m, j, "loss")
            if j == 0:
                continue
            k, tm, nt = j - 1, int(test[m]), int(fb.machine_n_test[m])
            jobs = engine.jobs_to_device(engine.make_jobs([0], [nt], [0]), eng.device)
            block = torch.from_numpy(np.ascontiguousarray(x_in[n:n + tm])).to(eng.device)
            own = eng.infer(fb.fold_params[m, k:k + 1].contiguous(), jobs, 1, nt, block, nt)  # the fold estimator's own predict
            pred = fb.fold_predictions[m, k]
            assert torch.equal(pred, own), (m, k, "fold predictions")
            y_true = Xm[n + L - 1 + la:n + tm]
            ft, at = am.fold_thresholds(y_true, pred.cpu().numpy(), *am.minmax_fit(prefix))
            np.testing.assert_allclose(fb.fold_feat_thr[m, k], ft, rtol=1e-9, atol=1e-14)
            np.testing.assert_allclose(fb.fold_agg_thr[m, k], at, rtol=1e-9, atol=1e-14)
        det = fb.detector(m)
        assert det.scaler.n_samples_seen_ == LSTM_LENGTHS[m]
        assert det.base_estimator.get_metadata()["history"]["params"]["steps"] == fb.machine_steps[m]


# ------------------------------------------------------------------------------------------------ 4. build_kfold_fleet
AE = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "batch_size": 64, "compression_factor": 0.5,
                                                      "encoding_layers": 1, "func": "tanh", "out_func": "linear", "epochs": 3}}
PIPE = {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", AE]}}
TTR = {"sklearn.compose.TransformedTargetRegressor": {"transformer": "sklearn.preprocessing.MinMaxScaler", "regressor": PIPE}}


@pytest.mark.parametrize("form", ["pipeline", "ttr"])
def test_ragged_kfold_thresholds_equal_the_per_machine_path(torch, form):
    """Machines of 240, 100 (shorter than the window: NaN thresholds), 317 and 240 rows, each against kfold_thresholds on its fold detectors."""
    from gordo_components_b200 import engine, fleet, serializer

    lengths, T, K, window = [240, 100, 317, 240], 6, 3, 144
    definition = {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {
        "base_estimator": PIPE if form == "pipeline" else TTR, "scaler": "sklearn.preprocessing.MinMaxScaler", "window": window,
        "smoothing_method": "smm", "shuffle": True, "threshold_percentile": 0.975}}
    rng = np.random.default_rng(5)
    frames = [pd.DataFrame(waves(rng, n, T) * 10, columns=[f"tag-{c}" for c in range(T)]) for n in lengths]
    template = serializer.from_definition(definition)
    ae = getattr(template.base_estimator, "regressor", template.base_estimator).steps[-1][1]
    ae.kwargs.update({"n_features": T, "n_features_out": T})
    spec = ae._build_spec()
    eng = engine.ff_engine_for(spec)
    xd = torch.from_numpy(np.concatenate([f.values for f in frames])).to(eng.device)
    cv = KFold(K, shuffle=True, random_state=0)
    fb = fleet.build_kfold_fleet(eng, xd, xd, lengths, cv, epochs=3, batch_size=64, seed=1, adam=spec.adam, input_scaler=True,
                                 target_scaler=form == "ttr", detector_shuffle=True, window=window, smoothing_method="smm", threshold_percentile=0.975)
    assert fb.n_test.shape == (len(lengths), K) and list(fb.rows) == lengths
    tags = list(frames[0].columns)
    for m, frame in enumerate(frames):
        folds = [fb.fold_detector(m, k, serializer.from_definition(definition), tags=tags, input_tags=tags) for k in range(K)]
        feat, agg = serializer.from_definition(definition).kfold_thresholds(frame, frame, cv, folds)
        assert np.array_equal(fb.feat_thr[m], feat.values, equal_nan=True), (m, fb.feat_thr[m], feat.values)
        assert np.array_equal(fb.agg_thr[m], agg, equal_nan=True), (m, fb.agg_thr[m], agg)
        assert np.isnan(fb.feat_thr[m]).all() == (lengths[m] < window)
        det = fb.detector(m, serializer.from_definition(definition), tags=tags, input_tags=tags)
        assert det.scaler.n_samples_seen_ == lengths[m]
        for k in range(K):
            assert folds[k].scaler.n_samples_seen_ == lengths[m] - fb.n_test[m, k]


# ------------------------------------------------------------------------------------------------ 5. FleetModelBuilder
FF_DEF = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": {"sklearn.pipeline.Pipeline": {"steps": [
    "sklearn.preprocessing.MinMaxScaler", {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2}}]}}}}
LSTM_DEF = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": {"gordo.machine.model.models.KerasLSTMAutoEncoder": {
    "kind": "lstm_hourglass", "lookback_window": 4, "epochs": 1, "batch_size": 16}}}}
KF_DEF = {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {"base_estimator": AE, "window": 12}}
KFOLD = {"cv": {"sklearn.model_selection.KFold": {"n_splits": 3, "shuffle": True, "random_state": 0}}}


def _series(rows, tags, seed):
    rng = np.random.default_rng(seed)
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(waves(rng, rows, tags).astype(np.float32), index=idx, columns=[f"TAG {i}" for i in range(tags)])


def _strip(meta):
    if isinstance(meta, dict):
        return {k: _strip(v) for k, v in meta.items() if k != "model_creation_date" and not k.endswith("duration_sec")}
    return meta


def test_equal_lengths_build_alike_with_and_without_the_flag(torch, tmp_path):
    from gordo_components_b200 import builder

    N, T = 240, 5
    machines = []
    for i in range(2):
        machines += [{"name": f"ff-{i}", "model": FF_DEF, "dataset": {"X": _series(N, T, i)}},
                     {"name": f"lstm-{i}", "model": LSTM_DEF, "dataset": {"X": _series(N, T, 10 + i)}},
                     {"name": f"kf-{i}", "model": KF_DEF, "dataset": {"X": _series(N, T, 20 + i)}, "evaluation": KFOLD}]
    plain = builder.FleetModelBuilder(machines, kfcv=True).build()
    ragged = builder.FleetModelBuilder(machines, kfcv=True, ragged=True).build()
    for (m0, meta0), (m1, meta1) in zip(plain, ragged):
        assert meta0["name"] == meta1["name"]
        assert pickle.dumps(m0) == pickle.dumps(m1), meta0["name"]
        assert _strip(meta0) == _strip(meta1), meta0["name"]


PROJECT = """
machines:
  - name: plant-a
    dataset: |
      data_provider:
        type: RandomDataProvider
      tags: [GRA-TAG 1, GRA-TAG 2, GRA-TAG 3]
      train_start_date: 2018-01-01T00:00:00+01:00
      train_end_date: 2018-01-04T00:00:00+01:00
  - name: plant-b
    dataset: |
      data_provider:
        type: RandomDataProvider
      resolution: 2min
      tags: [GRA-TAG 1, GRA-TAG 2, GRA-TAG 3]
      train_start_date: 2018-05-20T01:00:04+02:00
      train_end_date: 2018-05-21T15:05:50+02:00
  - name: plant-c
    dataset: |
      data_provider:
        type: RandomDataProvider
      tags: [GRA-TAG 1, GRA-TAG 2, GRA-TAG 3]
      train_start_date: 2018-09-15T13:03:04+02:00
      train_end_date: 2018-09-17T11:05:10+02:00
globals:
  model: |
    gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector:
      base_estimator:
        sklearn.pipeline.Pipeline:
          steps:
            - sklearn.preprocessing.MinMaxScaler
            - gordo.machine.model.models.KerasAutoEncoder:
                kind: feedforward_hourglass
"""


def test_a_project_of_three_lengths_builds_in_one_bucket_and_serves(torch, tmp_path, monkeypatch):
    from gordo_components_b200 import builder, server

    machines = builder.machines_from_config(PROJECT)
    lengths = [len(m["dataset"].get_data()[0]) for m in machines]
    assert len(set(lengths)) == 3
    buckets = []
    real = builder.FleetModelBuilder._build_bucket

    def counted(members):
        buckets.append([c.machine["name"] for c in members])
        return real(members)

    monkeypatch.setattr(builder.FleetModelBuilder, "_build_bucket", staticmethod(counted))
    results = builder.FleetModelBuilder(machines, ragged=True).build(str(tmp_path))
    assert buckets == [["plant-a", "plant-b", "plant-c"]]
    store = server.ModelStore(str(tmp_path))
    for (model, meta), n in zip(results, lengths):
        K = 3
        cv = meta["metadata"]["build_metadata"]["model"]["cross_validation"]
        assert cv["splits"]["fold-1-n-test"] == n // (K + 1) and cv["splits"]["fold-3-n-train"] == n - n // (K + 1)
        assert model.base_estimator.steps[-1][1].get_metadata()["history"]["params"]["steps"] == math.ceil(n / 32)
        X = machines[[m["name"] for m in machines].index(meta["name"])]["dataset"].get_data()[0].iloc[:50]
        payload = {"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(X)}
        reply = server.anomaly_prediction(store, meta["name"], json=payload)
        assert reply.status == 200, reply.body
        frame = server.dataframe_from_dict(reply.body["data"])
        assert len(frame) == 50 and np.isfinite(frame["total-anomaly-confidence"].values.astype(np.float64)).all()
    assert sorted(os.listdir(tmp_path)) == ["plant-a", "plant-b", "plant-c"]
