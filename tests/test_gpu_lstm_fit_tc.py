"""
The tensor-core LSTM fit family (gb_lstm_fit_tc, ``LSTMEngine.fit_tc``): batches above 32 windows against the oracle's Keras-style
fit loop (oracle/keras_math.py, tests/loss_oracle.py for the other losses) with the tolerances of the fp32 family's coverage tests,
agreement with the fp32 family where both apply, bit-for-bit replays, and the callers that select it (the LSTM estimators,
fleet.build_lstm_fleet, FleetModelBuilder(lstm_wide_batches=True)).
"""
import json
import logging
import math
import os

import numpy as np
import pandas as pd
import pytest
from parity_helpers import close
from test_gpu_fit_coverage import GRAD_ADAM, KERAS_ADAM, check_lstm_fit, lstm_setup

pytestmark = pytest.mark.gpu


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


def _fit_tc_and_check(engine, torch, km, F, F_out, units, act, head, lookback, rows, B, E, seed, adam=KERAS_ADAM, gradients=False):
    spec, eng, ws, Xs, Ys, nwin, jobs, x, y = lstm_setup(engine, torch, km, F, F_out, units, act, head, lookback, rows, seed=seed)
    params = eng.pack_params(ws)
    loss, acc, (_, _, t) = eng.fit_tc(params, jobs, len(rows), max(nwin), x, y, epochs=E, batch_size=B, primer=True, adam=adam)
    torch.cuda.synchronize()
    assert [int(v) for v in t.cpu()] == [1 + E * math.ceil(n / B) for n in nwin]
    check_lstm_fit(km, spec, ws, Xs, Ys, eng.unpack_params(params), loss.cpu().numpy(), acc.cpu().numpy(), nwin, E, B, adam, gradients)


#   name: (n_features, n_features_out, units, cell act, head act, lookback, rows per job, batch, epochs)
TC_GRID = {
    "relu_cells_tanh_head_ragged_b64": (5, 5, [6, 5], "relu", "tanh", 4, [140, 40, 301, 67], 64, 2),  # 37 windows < one batch; 64 exactly one
    "linear_cells_sigmoid_head_b33": (6, 6, [7, 4, 6], "linear", "sigmoid", 3, [100, 20], 33, 2),
    "sigmoid_cells_relu_head_wider_out_b100": (4, 9, [8, 5], "sigmoid", "relu", 5, [250, 104], 100, 2),
    "tanh_cells_narrower_out_lookback_1_b128": (9, 3, [6, 4], "tanh", "linear", 1, [300, 90, 129], 128, 2),
    "widths_65_130_b256": (20, 20, [65, 130], "tanh", "linear", 3, [300, 522], 256, 2),
    "widths_130_65_b128": (70, 66, [130, 65], "tanh", "sigmoid", 2, [200], 128, 1),
    "lookback_144_b64": (8, 8, [24, 16], "tanh", "linear", 144, [144 + 150], 64, 1),  # error growth over a long BPTT
}


@pytest.mark.parametrize("case", list(TC_GRID))
def test_fit_tc_architecture_grid(engine, torch, km, case):
    F, F_out, units, act, head, lookback, rows, B, E = TC_GRID[case]
    _fit_tc_and_check(engine, torch, km, F, F_out, units, act, head, lookback, rows, B, E, seed=31)


@pytest.mark.parametrize("act,epochs,B", [("relu", 1, 64), ("linear", 1, 128), ("tanh", 0, 64), ("tanh", 0, 128)])
def test_fit_tc_raw_gradients(engine, torch, km, act, epochs, B):
    """beta1 = beta2 = 0, eps = lr = 1 with a sigmoid head: the weight change is the raw gradient sum; epochs = 0 is the primer alone."""
    _fit_tc_and_check(engine, torch, km, 8, 8, [12, 7], act, "sigmoid", 5, [300], B, epochs, seed=33, adam=GRAD_ADAM, gradients=True)


@pytest.mark.parametrize("loss", ["mse", "mae", "mape", "msle", "huber", "log_cosh"])
def test_fit_tc_every_loss(engine, torch, km, loss):
    import loss_oracle as lo

    F, L, rows, B, E = 5, 4, [200, 70], 64, 2
    spec = km.LSTMSpec(F, [6, 4], ["tanh", "tanh"], F, "linear", L)
    rng = np.random.default_rng(7)
    ws = []
    for i in range(len(rows)):
        layers, (Wd, bd) = km.init_lstm_weights(spec, np.random.default_rng(17 + i))
        layers = [(K, U, b + rng.uniform(-0.1, 0.1, b.shape).astype(np.float32)) for K, U, b in layers]
        ws.append((layers, (Wd, rng.uniform(-0.1, 0.1, bd.shape).astype(np.float32))))
    Xs = [rng.random((n, F)).astype(np.float32) for n in rows]
    Ys = [(3 * rng.random((n, F)) - 0.5).astype(np.float32) for n in rows]
    eng = engine.LSTMEngine(F, spec.units, spec.acts, F, "linear", L)
    nwin = [n - L + 1 for n in rows]
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(len(rows)), nwin, np.concatenate([[0], np.cumsum(rows)[:-1]])), eng.device)
    params = eng.pack_params(ws)
    x = torch.from_numpy(np.concatenate(Xs)).to(eng.device)
    y = torch.from_numpy(np.concatenate(Ys)).to(eng.device)
    hist, _, _ = eng.fit_tc(params, jobs, len(rows), max(nwin), x, y, epochs=E, batch_size=B, primer=True, adam=KERAS_ADAM, loss=loss)
    torch.cuda.synchronize()
    hist, got = hist.cpu().numpy(), eng.unpack_params(params)
    for i in range(len(rows)):
        want_w, h_ref, _ = lo.lstm_fit(spec, ws[i], Xs[i], Ys[i], epochs=E, batch_size=B, loss=loss)
        close(hist[i], np.array(h_ref["loss"]), rtol=5e-4, name=f"{loss} job {i} loss history")
        steps = 1 + E * math.ceil(nwin[i] / B)
        for k, (w0, gl, wl) in enumerate(zip(km._lstm_flat(ws[i]), km._lstm_flat(got[i]), km._lstm_flat(want_w))):
            close(gl - w0, wl - w0, mag=KERAS_ADAM["lr"] * steps, rtol=2e-2, name=f"{loss} job {i} array {k}: trained weights")


@pytest.mark.parametrize("B", [1, 8, 32])
def test_fit_tc_agrees_with_the_fp32_family(engine, torch, km, B):
    spec, eng, ws, Xs, Ys, nwin, jobs, x, y = lstm_setup(engine, torch, km, 7, 5, [9, 6], "tanh", "linear", 4, [90, 41], seed=35)
    E = 2
    p32, ptc = eng.pack_params(ws), eng.pack_params(ws)
    l32, a32, (_, _, t32) = eng.fit(p32, jobs, 2, max(nwin), x, y, epochs=E, batch_size=B)
    ltc, atc, (_, _, ttc) = eng.fit_tc(ptc, jobs, 2, max(nwin), x, y, epochs=E, batch_size=B)
    torch.cuda.synchronize()
    assert torch.equal(t32, ttc)
    close(ltc.cpu().numpy(), l32.cpu().numpy(), rtol=5e-4, name="loss history")
    for i in range(2):
        assert np.allclose(atc[i].cpu().numpy(), a32[i].cpu().numpy(), atol=1.5 / nwin[i])
        steps = 1 + E * math.ceil(nwin[i] / B)
        for k, (w0, gt, gf) in enumerate(zip(km._lstm_flat(ws[i]), km._lstm_flat(eng.unpack_params(ptc)[i]), km._lstm_flat(eng.unpack_params(p32)[i]))):
            close(gt - w0, gf - w0, mag=KERAS_ADAM["lr"] * steps, rtol=2e-2, name=f"job {i} array {k}: trained weights")


def test_fit_tc_per_epoch_launches_equal_one_launch_and_runs_repeat(engine, torch, km):
    """E one-epoch launches carrying (m, v, t), the primer in the first only, are bit-identical to one E-epoch launch, and two
    identical launches are bit-identical (the head reduces its slices in a fixed order, without atomics)."""
    _, eng, ws, _, _, nwin, jobs, x, y = lstm_setup(engine, torch, km, 6, 6, [9, 70], "tanh", "linear", 4, [200, 47, 133], seed=37)
    E, B = 3, 64
    p1 = eng.pack_params(ws)
    l1, a1, (m1, v1, t1) = eng.fit_tc(p1, jobs, 3, max(nwin), x, y, epochs=E, batch_size=B)
    p2 = eng.pack_params(ws)
    state, l2 = None, []
    for e in range(E):
        loss, _, state = eng.fit_tc(p2, jobs, 3, max(nwin), x, y, epochs=1, batch_size=B, primer=e == 0, state=state)
        l2.append(loss)
    p3 = eng.pack_params(ws)
    l3, a3, (m3, v3, _) = eng.fit_tc(p3, jobs, 3, max(nwin), x, y, epochs=E, batch_size=B)
    torch.cuda.synchronize()
    assert torch.equal(t1, state[2]) and int(t1[0]) == 1 + E * math.ceil(nwin[0] / B)
    assert torch.equal(p1, p2), "weights"
    assert torch.equal(m1, state[0]) and torch.equal(v1, state[1]), "Adam moments"
    assert torch.equal(l1, torch.cat(l2, dim=1)), "loss history"
    assert torch.equal(p1, p3) and torch.equal(m1, m3) and torch.equal(v1, v3) and torch.equal(l1, l3) and torch.equal(a1, a3), "repeat run"


def test_batches_above_the_cap_are_refused_before_any_launch(engine, torch, km):
    _, eng, ws, _, _, nwin, jobs, x, y = lstm_setup(engine, torch, km, 4, 4, [5], "tanh", "linear", 3, [600], seed=39)
    params = eng.pack_params(ws)
    before = params.clone()
    for B in (257, 1000):
        with pytest.raises(ValueError, match="256"):
            eng.fit_tc(params, jobs, 1, max(nwin), x, y, batch_size=B)
    with pytest.raises(ValueError):
        eng.fit(params, jobs, 1, max(nwin), x, y, batch_size=64)  # the fp32 family keeps its limit
    torch.cuda.synchronize()
    assert torch.equal(params, before)
    from gordo_components_b200.machine.model.models import KerasLSTMAutoEncoder

    with pytest.raises(ValueError):
        KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=3, batch_size=300).fit(np.random.rand(400, 4), np.random.rand(400, 4))


# ------------------------------------------------------------------------------------------------ estimators
def _frame(n, T, seed=1):
    rng = np.random.default_rng(seed)
    t = np.linspace(0, 20, n)[:, None]
    v = 0.5 + 0.4 * np.sin(t * np.linspace(0.5, 2, T)) + rng.normal(0, 0.02, (n, T))
    return pd.DataFrame(v, columns=[f"tag-{i}" for i in range(T)], index=pd.date_range("2019-01-01", periods=n, freq="10min", tz="UTC"))


@pytest.mark.parametrize("cls_name,B,early_stopping", [("KerasLSTMAutoEncoder", 128, False), ("KerasLSTMAutoEncoder", 128, True),
                                                       ("KerasLSTMForecast", 64, False)])
def test_detector_with_wide_batch_lstm(engine, torch, km, cls_name, B, early_stopping):
    from gordo_components_b200.machine.model import models
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from oracle import anomaly_math as am

    n, T, L = 700, 4, 6
    X = _frame(n, T)
    kw = {"callbacks": [{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "loss", "patience": 2}}]} if early_stopping else {}
    det = DiffBasedAnomalyDetector(base_estimator=getattr(models, cls_name)(kind="lstm_hourglass", lookback_window=L, epochs=3, batch_size=B, **kw))
    det.cross_validate(X=X, y=X)
    assert len(det.feature_thresholds_) == T and np.isfinite(det.aggregate_threshold_)
    det.fit(X, X)
    ae = det.base_estimator
    meta = ae.get_metadata()["history"]
    n_win = n - L + 1 - ae.lookahead
    assert meta["params"]["steps"] == math.ceil(n_win / B) and meta["params"]["epochs"] == 3
    assert 1 <= len(meta["loss"]) <= 3 and np.isfinite(meta["loss"]).all()
    frame = det.anomaly(X, X)
    assert len(X) - len(frame) == L - 1 + ae.lookahead
    spec = km.lstm_hourglass_spec(T, lookback_window=L)
    pred = km.lstm_predict(spec, ae.model.weights, X.values.astype(np.float32), lookahead=ae.lookahead)
    close(frame["model-output"].values, pred, rtol=2e-4, name="model-output")
    sc, mn = am.minmax_fit(X.values)
    want = am.anomaly_arrays(pred, X.values, sc, mn, det.feature_thresholds_.values, det.aggregate_threshold_)
    close(frame["tag-anomaly-unscaled"].values, want["tag-anomaly-unscaled"], rtol=2e-4, name="tag-anomaly-unscaled")


def test_estimator_fit_follows_the_oracle_at_batch_128(engine, torch, km):
    """The estimator's one-launch path at batch 128 trains what keras_math.lstm_fit trains from the same initial weights."""
    from gordo_components_b200.machine.model.models import KerasLSTMAutoEncoder

    n, T, L, B, E = 600, 4, 5, 128, 2
    X = _frame(n, T, seed=3).values.astype(np.float32)
    est = KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=L, epochs=E, batch_size=B)
    est.initialize(T, T)
    w0 = est.model.weights
    est.initialize = lambda *a, **k: est  # fit from these weights instead of drawing new ones
    est.fit(X, X)
    spec = km.lstm_hourglass_spec(T, lookback_window=L)
    want_w, hist = km.lstm_fit(spec, w0, X, X, epochs=E, batch_size=B)
    close(est.get_metadata()["history"]["loss"], hist["loss"], rtol=5e-4, name="loss history")
    steps = 1 + E * math.ceil((n - L + 1) / B)
    for a0, gl, wl in zip(km._lstm_flat(w0), km._lstm_flat(est.model.weights), km._lstm_flat(want_w)):
        close(gl - a0, wl - a0, mag=1e-3 * steps, rtol=2e-2, name="trained weights")


# ------------------------------------------------------------------------------------------------ batched builds
M, N, T, L, K, EPOCHS, B = 3, 400, 4, 6, 3, 2, 64  # final fit 395 windows, folds 95 / 195 / 295: partial last batches


def _frames(n=N, tags=T, count=M):
    out = []
    for seed in range(count):
        rng = np.random.default_rng(100 + seed)
        t = np.linspace(0, 20, n)[:, None]
        v = (0.5 + 0.4 * np.sin(t * rng.uniform(0.5, 2, tags) + rng.uniform(0, 3, tags)) + rng.normal(0, 0.02, (n, tags))) * rng.uniform(1, 5, tags)
        idx = pd.date_range("2019-01-01", periods=n, freq="10min", tz="UTC")
        out.append(pd.DataFrame(v.astype(np.float32).astype(np.float64), index=idx, columns=[f"tag-{i}" for i in range(tags)]))
    return out


@pytest.mark.parametrize("cls_name", ["KerasLSTMAutoEncoder", "KerasLSTMForecast"])
def test_lstm_fleet_at_batch_64_matches_per_slot_oracle(engine, torch, km, cls_name):
    from gordo_components_b200 import fleet

    la = 1 if cls_name == "KerasLSTMForecast" else 0
    frames = _frames()
    spec = km.lstm_hourglass_spec(T, lookback_window=L)
    eng = engine.LSTMEngine(spec.n_features, spec.units, spec.acts, spec.n_features_out, spec.out_func, spec.lookback_window)
    x = torch.from_numpy(np.ascontiguousarray(np.concatenate([f.values for f in frames]))).to(eng.device)
    fb = fleet.build_lstm_fleet(eng, x, x, N, lookahead=la, epochs=EPOCHS, batch_size=B, n_splits=K, seed=7, keep_init_params=True)
    torch.cuda.synchronize()
    test = N // (K + 1)
    starts = [N - (K - k) * test for k in range(K)]
    init, final = eng.unpack_params(fb.init_params), eng.unpack_params(fb.params)
    for m, frame in enumerate(frames):
        Xv = frame.values
        for j, n_rows in enumerate([N] + starts):
            x_in = Xv[:n_rows].astype(np.float32)
            want_w, hist = km.lstm_fit(spec, init[j * M + m], x_in, x_in, epochs=EPOCHS, batch_size=B, lookahead=la)
            got_w = final[m] if j == 0 else eng.unpack_params(fb.fold_params[m, j - 1 : j])[0]
            got_loss = fb.loss[m] if j == 0 else fb.fold_loss[m, j - 1]
            close(got_loss, hist["loss"], rtol=5e-4, name=f"machine {m} slot {j} loss history")
            steps = 1 + EPOCHS * int(np.ceil((n_rows - L + 1 - la) / B))
            for a0, gl, wl in zip(km._lstm_flat(init[j * M + m]), km._lstm_flat(got_w), km._lstm_flat(want_w)):
                close(gl - a0, wl - a0, mag=1e-3 * steps, rtol=2e-2, name=f"machine {m} slot {j} trained weights")
    # the memory budget chunks by the batch-aware workspace: two machines per launch give the same fleet
    budget = eng.fit_tc_workspace_bytes(2 * (K + 1), B)
    assert budget > eng.fit_workspace_bytes(2 * (K + 1))
    again = fleet.build_lstm_fleet(eng, x, x, N, lookahead=la, epochs=EPOCHS, batch_size=B, n_splits=K, seed=7, memory_budget=budget)
    torch.cuda.synchronize()
    assert torch.equal(fb.params, again.params) and torch.equal(fb.fold_params, again.fold_params)


def _project():
    lstm = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": {"gordo.machine.model.models.KerasLSTMAutoEncoder": {
        "kind": "lstm_hourglass", "lookback_window": 5, "epochs": 1, "batch_size": 64}}}}
    return [{"name": f"lstm-{i}", "model": lstm, "dataset": {"X": f}, "evaluation": {"metrics": ["r2_score"], "scoring_scaler": None}}
            for i, f in enumerate(_frames(n=360, tags=5, count=2))]


def test_fleet_builder_batches_wide_lstm_machines_with_the_flag(engine, torch, caplog, tmp_path):
    from gordo_components_b200 import builder

    with caplog.at_level(logging.INFO, logger="gordo_components_b200.builder"):
        out = builder.FleetModelBuilder(_project(), lstm_wide_batches=True).build(str(tmp_path))
    messages = [r.getMessage() for r in caplog.records]
    assert any("built 2 LSTM machines in one batched bucket" in s for s in messages), messages
    assert not any("per-machine path" in s for s in messages), messages
    for model, machine in out:
        d = os.path.join(str(tmp_path), machine["name"])
        assert os.path.exists(os.path.join(d, "model.pkl"))
        meta = json.load(open(os.path.join(d, "metadata.json")))
        assert meta["metadata"]["build_metadata"]["model"]["model_offset"] == 4
        hist = model.base_estimator.get_metadata()["history"]
        assert hist["params"]["steps"] == math.ceil((360 - 5 + 1) / 64)


def test_fleet_builder_without_the_flag_builds_wide_lstm_machines_one_at_a_time(engine, torch, caplog, tmp_path):
    from gordo_components_b200 import builder

    with caplog.at_level(logging.INFO, logger="gordo_components_b200.builder"):
        out = builder.FleetModelBuilder(_project()).build(str(tmp_path))
    messages = [r.getMessage() for r in caplog.records]
    assert any("per-machine path" in s and "batch_size 64" in s for s in messages), messages
    assert not any("in one batched bucket" in s for s in messages), messages
    for model, machine in out:
        assert os.path.exists(os.path.join(str(tmp_path), machine["name"], "model.pkl"))
        assert machine["metadata"]["build_metadata"]["model"]["model_offset"] == 4
        assert model.base_estimator.get_metadata()["history"]["params"]["steps"] == math.ceil(356 / 64)
