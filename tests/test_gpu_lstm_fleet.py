"""
The batched LSTM build (fleet.build_lstm_fleet, FleetModelBuilder's LSTM buckets) on the GPU: every slot against the oracle's
restatement of the per-machine fit from the same initial weights, thresholds / scalers / anomaly against oracle.anomaly_math and
sklearn, chunked fits against one launch, and the batched machine against the same machine built by ModelBuilder.
"""
import logging
import pickle

import numpy as np
import pandas as pd
import pytest
from sklearn.preprocessing import MinMaxScaler

pytestmark = pytest.mark.gpu

M, N, T, L, K, EPOCHS, B = 4, 130, 4, 6, 3, 2, 16  # test blocks of 32 rows; 125 / 29 / 61 / 93 training windows: partial last batches


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


def close(got, want, mag=1.0, rtol=1e-4, name="", floor=2e-5):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (name, got.shape, want.shape)
    err = np.abs(got - want)
    bad = ~(err <= rtol * np.abs(want) + floor * mag)
    assert not bad.any(), f"{name}: {bad.sum()} of {bad.size} outside tolerance; max err {err[bad].max():.3e}"


def _frames(n=N, tags=T, count=M):
    out = []
    for seed in range(count):
        rng = np.random.default_rng(100 + seed)
        t = np.linspace(0, 20, n)[:, None]
        v = (0.5 + 0.4 * np.sin(t * rng.uniform(0.5, 2, tags) + rng.uniform(0, 3, tags)) + rng.normal(0, 0.02, (n, tags))) * rng.uniform(1, 5, tags)
        idx = pd.date_range("2019-01-01", periods=n, freq="10min", tz="UTC")
        out.append(pd.DataFrame(v.astype(np.float32).astype(np.float64), index=idx, columns=[f"tag-{i}" for i in range(tags)]))
    return out


def _definition(cls_name, scaled, lookback=L):
    lstm = {f"gordo.machine.model.models.{cls_name}": {"kind": "lstm_hourglass", "lookback_window": lookback, "epochs": EPOCHS, "batch_size": B}}
    base = {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", lstm]}} if scaled else lstm
    return {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": base}}


def _build(engine, torch, frames, lookahead, scaled, **kw):
    from gordo_components_b200 import fleet
    from oracle import keras_math as km

    spec = km.lstm_hourglass_spec(T, lookback_window=L)
    eng = engine.LSTMEngine(spec.n_features, spec.units, spec.acts, spec.n_features_out, spec.out_func, spec.lookback_window)
    x = torch.from_numpy(np.ascontiguousarray(np.concatenate([f.values for f in frames]))).to(eng.device)  # frame values are column-major
    fb = fleet.build_lstm_fleet(eng, x, x, N, lookahead=lookahead, epochs=EPOCHS, batch_size=B, n_splits=K, seed=7, input_scaler=scaled, **kw)
    torch.cuda.synchronize()
    return spec, eng, fb


def test_orthonormal_rows_is_keras_orthogonal(engine, torch):
    """gb_orthonormal_rows gives Q^T of numpy's QR of the transposed draw with diag(R) made positive (Keras' Orthogonal)."""
    dev = engine.cuda_device()
    u = 40
    g = torch.randn((3, u, 4 * u), dtype=torch.float64, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    draw = g.cpu().numpy()
    out = torch.zeros((3, 5 + u * 4 * u), dtype=torch.float32, device=dev)
    engine.orthonormal_rows(g, out, 5, out.shape[1])
    got = out.cpu().numpy()
    assert (got[:, :5] == 0).all()
    for i in range(3):
        q, r = np.linalg.qr(draw[i].T)
        want = (q * np.sign(np.diag(r))).T
        np.testing.assert_allclose(got[i, 5:].reshape(u, 4 * u), want, atol=2e-6)


def test_initial_params_follow_the_keras_initialisers(engine, torch):
    from oracle import keras_math as km

    spec = km.lstm_model_spec(5, 3, lookback_window=4, encoding_dim=(24,), encoding_func=("tanh",), decoding_dim=(8,), decoding_func=("tanh",))
    eng = engine.LSTMEngine(spec.n_features, spec.units, spec.acts, spec.n_features_out, spec.out_func, spec.lookback_window)
    p = eng.initial_params(6, torch.Generator(device=eng.device).manual_seed(3))
    again = eng.initial_params(6, torch.Generator(device=eng.device).manual_seed(3))
    assert torch.equal(p, again)
    for layers, (Wd, bd) in eng.unpack_params(p):
        i = spec.n_features
        for (Kk, U, b), u in zip(layers, spec.units):
            assert np.abs(Kk).max() <= np.sqrt(6.0 / (i + 4 * u)) and Kk.std() > 0
            np.testing.assert_allclose(U @ U.T, np.eye(u), atol=1e-5)
            np.testing.assert_array_equal(b, np.r_[np.zeros(u), np.ones(u), np.zeros(2 * u)].astype(np.float32))
            i = u
        assert np.abs(Wd).max() <= np.sqrt(6.0 / (i + spec.n_features_out)) and (bd == 0).all()


@pytest.mark.parametrize("scaled", [False, True], ids=["bare", "minmax"])
@pytest.mark.parametrize("cls_name", ["KerasLSTMAutoEncoder", "KerasLSTMForecast"])
def test_lstm_fleet_build_matches_per_machine_oracle(engine, torch, cls_name, scaled):
    from gordo_components_b200 import serializer
    from oracle import anomaly_math as am
    from oracle import keras_math as km

    la = 1 if cls_name == "KerasLSTMForecast" else 0
    frames = _frames()
    spec, eng, fb = _build(engine, torch, frames, la, scaled, keep_init_params=True)
    test = N // (K + 1)
    starts = [N - (K - k) * test for k in range(K)]
    assert fb.starts == starts and fb.n_test == test - L + 1 - la
    init = eng.unpack_params(fb.init_params)
    final = eng.unpack_params(fb.params)
    for m, frame in enumerate(frames):
        Xv = frame.values
        for j, n_rows in enumerate([N] + starts):  # slot j*M + m: the final fit, then fold j-1
            prefix = Xv[:n_rows]
            x_in = MinMaxScaler().fit(prefix).transform(Xv).astype(np.float32) if scaled else Xv.astype(np.float32)
            want_w, hist = km.lstm_fit(spec, init[j * M + m], x_in[:n_rows], prefix.astype(np.float32), epochs=EPOCHS, batch_size=B, lookahead=la)
            got_w = final[m] if j == 0 else eng.unpack_params(fb.fold_params[m, j - 1 : j])[0]
            got_loss = fb.loss[m] if j == 0 else fb.fold_loss[m, j - 1]
            close(got_loss, hist["loss"], rtol=5e-4, name=f"machine {m} slot {j} loss history")
            steps = 1 + EPOCHS * int(np.ceil((n_rows - L + 1 - la) / B))
            w0 = km._lstm_flat(init[j * M + m])
            for a0, gl, wl in zip(w0, km._lstm_flat(got_w), km._lstm_flat(want_w)):
                close(gl - a0, wl - a0, mag=1e-3 * steps, rtol=2e-2, name=f"machine {m} slot {j} trained weights")
            if j == 0:
                continue
            # fold j-1: its scaler, predictions on the test block and thresholds
            k = j - 1
            np.testing.assert_array_equal(fb.fold_y_min[m, k], prefix.min(0))
            np.testing.assert_array_equal(fb.fold_y_max[m, k], prefix.max(0))
            pred = fb.fold_predictions[m, k].cpu().numpy()
            close(pred, km.lstm_predict(spec, got_w, x_in[starts[k] : starts[k] + test], lookahead=la), rtol=2e-4, name="fold predictions")
            y_true = Xv[starts[k] + L - 1 + la : starts[k] + test]
            ft, at = am.fold_thresholds(y_true, pred, *am.minmax_fit(prefix))
            np.testing.assert_allclose(fb.fold_feat_thr[m, k], ft, rtol=1e-9, atol=1e-14)
            np.testing.assert_allclose(fb.fold_agg_thr[m, k], at, rtol=1e-9, atol=1e-14)
            e, c = pred.astype(np.float64) - y_true.astype(np.float32), y_true - y_true[0]
            np.testing.assert_allclose(fb.cv_moments[m, k], np.stack([e.sum(0), (e * e).sum(0), np.abs(e).sum(0), c.sum(0), (c * c).sum(0)]), rtol=1e-9, atol=1e-9)
        np.testing.assert_array_equal(fb.feat_thr[m], fb.fold_feat_thr[m, K - 1])
        assert fb.agg_thr[m] == fb.fold_agg_thr[m, K - 1]

        # the detector: sklearn's scalers, the reference's estimator class and attributes, anomaly as the oracle computes it
        template = serializer.from_definition(_definition(cls_name, scaled))
        det = fb.detector(m, tags=list(frame.columns), template=template, input_tags=list(frame.columns))
        lstm = det.base_estimator.steps[-1][1] if scaled else det.base_estimator
        assert type(lstm).__name__ == cls_name and lstm.kind == "lstm_hourglass" and lstm.lookback_window == L and lstm.batch_size == B
        meta = lstm.get_metadata()  # a Pipeline is not a GordoBase: the detector's own metadata then holds only its repr
        assert meta["forecast_steps"] == la and len(meta["history"]["loss"]) == EPOCHS
        assert meta["history"]["params"]["steps"] == int(np.ceil((N - L + 1 - la) / B))
        sk = MinMaxScaler().fit(frame)
        for name in ("scale_", "min_", "data_min_", "data_max_", "data_range_"):
            np.testing.assert_array_equal(getattr(det.scaler, name), getattr(sk, name), err_msg=name)
            if scaled:
                np.testing.assert_array_equal(getattr(det.base_estimator.steps[0][1], name), getattr(sk, name), err_msg=name)
        assert det.scaler.n_samples_seen_ == N and list(det.scaler.feature_names_in_) == list(frame.columns)
        frame_out = det.anomaly(frame, frame)
        x_final = sk.transform(Xv).astype(np.float32) if scaled else Xv.astype(np.float32)
        pred = km.lstm_predict(spec, final[m], x_final, lookahead=la)
        close(frame_out["model-output"].values, pred, rtol=2e-4, name="detector model-output")
        want = am.anomaly_arrays(pred, Xv, sk.scale_, sk.min_, det.feature_thresholds_.values, det.aggregate_threshold_)
        close(frame_out["tag-anomaly-unscaled"].values, want["tag-anomaly-unscaled"], rtol=2e-4, name="tag-anomaly-unscaled")
        close(frame_out["total-anomaly-confidence"].values.ravel(), want["total-anomaly-confidence"], float(want["total-anomaly-confidence"].max()), rtol=2e-4,
              name="total-anomaly-confidence")
        again = pickle.loads(pickle.dumps(det))
        np.testing.assert_array_equal(again.anomaly(frame, frame)["model-output"].values, frame_out["model-output"].values)
        assert again.aggregate_threshold_ == det.aggregate_threshold_


def test_chunked_fits_give_the_same_fleet(engine, torch):
    frames = _frames()
    _, eng, whole = _build(engine, torch, frames, 0, True)
    budget = eng.fit_workspace_bytes(2 * (K + 1))  # two machines per gb_lstm_fit launch: two chunks
    assert budget < eng.fit_workspace_bytes(M * (K + 1))
    _, _, chunked = _build(engine, torch, frames, 0, True, memory_budget=budget)
    assert torch.equal(whole.params, chunked.params) and torch.equal(whole.fold_params, chunked.fold_params)
    for name in ("loss", "fold_loss", "feat_thr", "agg_thr", "fold_feat_thr", "fold_agg_thr", "cv_moments"):
        np.testing.assert_array_equal(getattr(whole, name), getattr(chunked, name), err_msg=name)


def _key_tree(d):
    return {k: _key_tree(v) for k, v in d.items()} if isinstance(d, dict) else None


def test_batched_and_per_machine_lstm_builds_have_the_same_shape(engine, torch, caplog):
    from gordo_components_b200 import builder

    frame = _frames(n=200, count=1)[0]
    definition = _definition("KerasLSTMForecast", True)
    machines = [{"name": "batched", "model": definition, "dataset": {"X": frame, "y": frame}}]
    with caplog.at_level(logging.INFO, logger="gordo_components_b200.builder"):
        (model, batched), = builder.FleetModelBuilder(machines).build()
    assert any("built 1 LSTM machines in one batched bucket" in r.getMessage() for r in caplog.records)
    single_model, single = builder.ModelBuilder({"name": "batched", "model": definition, "dataset": {"X": frame, "y": frame}}).build()
    a, b = batched["metadata"]["build_metadata"]["model"], single["metadata"]["build_metadata"]["model"]
    tree_a, tree_b = _key_tree(batched), _key_tree(single)
    for tree in (tree_a, tree_b):  # the dataset block holds whatever the data source reports
        tree["metadata"]["build_metadata"]["dataset"] = None
    assert tree_a == tree_b
    assert a["model_offset"] == b["model_offset"] == L - 1 + 1
    assert a["cross_validation"]["splits"] == b["cross_validation"]["splits"]
    assert set(a["cross_validation"]["scores"]) == set(b["cross_validation"]["scores"])
    for key, val in a["cross_validation"]["scores"].items():
        assert set(val) == set(b["cross_validation"]["scores"][key])
        assert np.isfinite(list(val.values())).all(), key
        if key.startswith("mean-"):
            assert val["fold-min"] >= 0.0
        else:
            assert val["fold-max"] <= 1.0
    assert set(a["model_meta"]) == set(b["model_meta"])
    assert len(model.anomaly(frame, frame)) == len(single_model.anomaly(frame, frame)) == 200 - a["model_offset"]


def test_the_end_to_end_lstm_machine_takes_the_batched_path(engine, torch, caplog):
    """The lstm machine of test_gpu_builder's project is built by build_lstm_fleet, not one at a time."""
    from gordo_components_b200 import builder

    frame = _frames(n=320, tags=5, count=1)[0]
    lstm = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": {"gordo.machine.model.models.KerasLSTMAutoEncoder": {
        "kind": "lstm_hourglass", "lookback_window": 4, "epochs": 1, "encoding_layers": 1}}}}
    machines = [{"name": "lstm", "model": lstm, "dataset": {"X": frame}, "evaluation": {"metrics": ["r2_score"], "scoring_scaler": None}}]
    with caplog.at_level(logging.INFO, logger="gordo_components_b200.builder"):
        (model, machine), = builder.FleetModelBuilder(machines).build()
    messages = [r.getMessage() for r in caplog.records]
    assert any("built 1 LSTM machines in one batched bucket" in s for s in messages), messages
    assert not any("per-machine path" in s or "one at a time" in s for s in messages), messages
    assert machine["metadata"]["build_metadata"]["model"]["model_offset"] == 3
    assert set(machine["metadata"]["build_metadata"]["model"]["cross_validation"]["scores"]) == {"r2-score"} | {f"r2-score-tag-{i}" for i in range(5)}
