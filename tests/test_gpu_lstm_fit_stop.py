"""
EarlyStopping inside the LSTM fit launches (gb_lstm_fit_stop / gb_lstm_fit_tc_stop, ``LSTMEngine.fit_stop``): a rule that never
fires changes nothing, jobs that stop match plain launches of the epochs they ran, the decisions are those of the host class
(models.EarlyStopping), stopped jobs run no kernels, and the fleet builder replays the per-machine loop bit for bit.  Both
families: batch 16 on the fp32 kernels, 64 and 100 on the tensor cores.
"""
import logging
import math

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

F, UNITS, LOOKBACK = 5, [8, 6], 4
BATCHES = [16, 64, 100]
HUGE = 1e9  # a min_delta only the first epoch (against +inf) beats: the job stops after epoch max(patience, 1)


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


def _setup(engine, torch, rows, seed=0, nan_job=None):
    eng = engine.LSTMEngine(F, UNITS, ["tanh"] * len(UNITS), F, "linear", LOOKBACK)
    rng = np.random.default_rng(seed)
    X = rng.random((sum(rows), F)).astype(np.float32)
    Y = X.copy()
    starts = np.concatenate([[0], np.cumsum(rows)[:-1]])
    if nan_job is not None:
        Y[starts[nan_job] + LOOKBACK + 3] = np.nan
    nwin = [n - LOOKBACK + 1 for n in rows]
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(len(rows)), nwin, starts), eng.device)
    params = eng.initial_params(len(rows), torch.Generator(device=eng.device).manual_seed(seed))
    return eng, params, jobs, nwin, torch.from_numpy(X).to(eng.device), torch.from_numpy(Y).to(eng.device)


def _plain(eng, params, jobs, nwin, x, y, epochs, B, **kw):
    p = params.clone()
    loss, acc, (m, v, t) = eng.fit_for_batch(B)(p, jobs, len(nwin), max(nwin), x, y, epochs=epochs, batch_size=B, **kw)
    return p, loss, acc, m, v, t


def _stop(engine, eng, params, jobs, nwin, x, y, rules, epochs, B, **kw):
    p = params.clone()
    loss, acc, er, be, (m, v, t) = eng.fit_stop(p, jobs, len(nwin), max(nwin), x, y, engine.make_stop(rules), epochs=epochs, batch_size=B, **kw)
    return p, loss, acc, m, v, t, er.cpu().numpy(), be.cpu().numpy()


FIT_KW = [{}, {"loss": "huber", "optimizer": ("rmsprop", {"lr": 2e-3, "rho": 0.9, "eps": 1e-7})}]


@pytest.mark.parametrize("kw", FIT_KW, ids=["mse-adam", "huber-rmsprop"])
@pytest.mark.parametrize("B", BATCHES)
def test_a_rule_that_never_fires_is_the_opt_entry_bit_for_bit(engine, torch, B, kw):
    eng, params, jobs, nwin, x, y = _setup(engine, torch, [90, 57, 140])
    E = 3
    want = _plain(eng, params, jobs, nwin, x, y, E, B, **kw)
    got = _stop(engine, eng, params, jobs, nwin, x, y, [{"monitor": "loss", "patience": 100}] * 3, E, B, **kw)
    for a, b, name in zip(got[:6], want, ("params", "loss", "accuracy", "state 0", "state 1", "steps")):
        assert torch.equal(a, b), name
    assert (got[6] == E).all() and (got[7] >= 0).all()


@pytest.mark.parametrize("kw", FIT_KW, ids=["mse-adam", "huber-rmsprop"])
@pytest.mark.parametrize("B", BATCHES)
def test_ragged_stops_match_plain_launches_of_the_epochs_run(engine, torch, B, kw):
    eng, params, jobs, nwin, x, y = _setup(engine, torch, [90, 57, 140, 75], seed=1)
    E = 8
    rules = [{"monitor": "loss", "patience": p, "min_delta": HUGE, "restore_best_weights": r} for p, r in ((2, False), (3, True), (5, False), (0, True))]
    p, loss, acc, m, v, t, ran, best = _stop(engine, eng, params, jobs, nwin, x, y, rules, E, B, **kw)
    assert list(ran) == [3, 4, 6, 2] and list(best) == [0, 0, 0, 0]
    loss, acc = loss.cpu().numpy(), acc.cpu().numpy()
    for j, n in enumerate(ran):
        ref = _plain(eng, params, jobs, nwin, x, y, int(n), B, **kw)
        np.testing.assert_array_equal(loss[j, :n], ref[1][j].cpu().numpy())
        np.testing.assert_array_equal(acc[j, :n], ref[2][j].cpu().numpy())
        assert np.isnan(loss[j, n:]).all() and np.isnan(acc[j, n:]).all()
        for got, want, name in ((m, ref[3], "state 0"), (v, ref[4], "state 1"), (t, ref[5], "steps")):
            assert torch.equal(got[j], want[j]), (j, name)
        if rules[j]["restore_best_weights"]:
            assert 0 <= best[j] < n
            assert torch.equal(p[j], _plain(eng, params, jobs, nwin, x, y, int(best[j]) + 1, B, **kw)[0][j]), j
        else:
            assert torch.equal(p[j], ref[0][j]), j


GRID = [
    {"monitor": "loss", "patience": 1},
    {"monitor": "loss", "patience": 0},
    {"monitor": "loss", "patience": 1, "mode": "max"},
    {"monitor": "loss", "patience": 2, "min_delta": 0.01},
    {"monitor": "loss", "patience": 1, "min_delta": 1e-4, "restore_best_weights": True},
    {"monitor": "loss", "patience": 2, "baseline": 10.0},
    {"monitor": "loss", "patience": 2, "baseline": 0.0},
    {"monitor": "loss", "patience": 1, "start_from_epoch": 3},
    {"monitor": "accuracy", "patience": 1},
    {"monitor": "accuracy", "patience": 0, "mode": "min"},
    {"monitor": "accuracy", "patience": 2, "min_delta": 0.05, "restore_best_weights": True},
    {"monitor": "accuracy", "patience": 1, "baseline": 0.99},
    {"monitor": "accuracy", "patience": 1, "start_from_epoch": 2, "mode": "max"},
]


def _host_rule(rule, loss, acc):
    """(epochs_run, best_epoch) of models.EarlyStopping replayed on a full history, with the kernels' -1 for 'no best epoch'."""
    from gordo_components_b200.machine.model.models import EarlyStopping

    cb = EarlyStopping(**rule)
    for e in range(len(loss)):
        if cb.update(e, {"loss": float(loss[e]), "accuracy": float(acc[e])}, lambda: e):
            return e + 1, cb.best_epoch
    seen = cb.best_weights is not None or math.isfinite(cb.best)
    return len(loss), cb.best_epoch if seen else -1


@pytest.mark.parametrize("B", BATCHES)
def test_the_rule_matches_the_host_class(engine, torch, B):
    n = len(GRID)
    eng, params, jobs, nwin, x, y = _setup(engine, torch, [60 + 7 * j for j in range(n)], seed=2)
    E = 8
    _, full_loss, full_acc, *_ = _plain(eng, params, jobs, nwin, x, y, E, B)
    *_, ran, best = _stop(engine, eng, params, jobs, nwin, x, y, GRID, E, B)
    full_loss, full_acc = full_loss.cpu().numpy(), full_acc.cpu().numpy()
    for j, rule in enumerate(GRID):
        assert (int(ran[j]), int(best[j])) == _host_rule(rule, full_loss[j], full_acc[j]), rule
    assert len(set(ran.tolist())) > 2  # the grid does stop at different epochs


@pytest.mark.parametrize("B", BATCHES)
def test_nan_targets_never_improve_and_val_monitors_never_stop(engine, torch, B):
    eng, params, jobs, nwin, x, y = _setup(engine, torch, [80, 80, 80], seed=3, nan_job=0)
    E = 5
    rules = [{"monitor": "loss", "patience": 3}, {"monitor": "val_loss", "patience": 0, "restore_best_weights": True},
             {"monitor": "val_accuracy", "patience": 0}]
    p, loss, _, _, _, _, ran, best = _stop(engine, eng, params, jobs, nwin, x, y, rules, E, B)
    assert np.isnan(loss[0, :3].cpu().numpy()).all()
    assert list(ran) == [3, E, E] and list(best) == [-1, -1, -1]
    ref = _plain(eng, params, jobs, nwin, x, y, E, B)[0]
    assert torch.equal(p[1:], ref[1:])  # no snapshot, so nothing restored
    assert torch.equal(p[0].view(torch.int32), _plain(eng, params, jobs, nwin, x, y, 3, B)[0][0].view(torch.int32))  # NaN weights, bit for bit


@pytest.mark.parametrize("B", [16, 64])
def test_no_step_kernel_runs_once_every_job_has_stopped(engine, torch, B):
    from torch.profiler import ProfilerActivity, profile, schedule

    eng, params, jobs, nwin, x, y = _setup(engine, torch, [90, 90], seed=4)
    rules = [{"monitor": "loss", "patience": 1, "min_delta": HUGE}] * 2  # both stop after epoch 1

    def forward_kernels(run):
        # one warm-up step traced and discarded, then the counted one: the first CUDA trace of a process can come back without
        # kernel records while the activity tracer starts up
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA], schedule=schedule(wait=0, warmup=1, active=1, repeat=1)) as prof:
            for _ in range(2):
                run()
                torch.cuda.synchronize()
                prof.step()
        return sum(e.count for e in prof.key_averages() if "fwd_kernel" in e.key)

    stopped = forward_kernels(lambda: _stop(engine, eng, params, jobs, nwin, x, y, rules, 12, B))
    plain = forward_kernels(lambda: _plain(eng, params, jobs, nwin, x, y, 2, B))
    if plain == 0:
        pytest.skip("the profiler lists no kernels of graph replays here; benchmarks/bench_lstm_fit_stop.py (b) times the stopped steps")
    steps = 1 + 2 * math.ceil(max(nwin) / B)
    assert plain == steps * LOOKBACK * len(UNITS)
    assert stopped == plain


# ------------------------------------------------------------------------------------------------ the fleet and the builder
N, T, M, K, EPOCHS, BF = 160, 4, 3, 3, 6, 16


def _frames(count=M, n=N):
    out = []
    for seed in range(count):
        rng = np.random.default_rng(200 + seed)
        t = np.linspace(0, 20, n)[:, None]
        v = (0.5 + 0.4 * np.sin(t * rng.uniform(0.5, 2, T) + rng.uniform(0, 3, T)) + rng.normal(0, 0.02, (n, T))) * rng.uniform(1, 5, T)
        idx = pd.date_range("2019-01-01", periods=n, freq="10min", tz="UTC")
        out.append(pd.DataFrame(v.astype(np.float32).astype(np.float64), index=idx, columns=[f"tag-{i}" for i in range(T)]))
    return out


FLEET_RULES = [{"monitor": "loss", "patience": 0}, {"monitor": "loss", "patience": 1, "restore_best_weights": True, "min_delta": 1e-3},
               {"monitor": "loss", "patience": 2, "min_delta": HUGE, "restore_best_weights": True}]


@pytest.mark.parametrize("one_per_chunk", [False, True], ids=["one-launch", "one-machine-per-chunk"])
@pytest.mark.parametrize("scaled", [False, True], ids=["bare", "minmax"])
@pytest.mark.parametrize("la", [0, 1], ids=["autoencoder", "forecast"])
def test_lstm_fleet_replays_the_per_machine_loop_bit_for_bit(engine, torch, la, scaled, one_per_chunk):
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200 import fleet
    from gordo_components_b200.machine.model.models import EarlyStopping

    frames = _frames()
    eng = engine.LSTMEngine(T, UNITS, ["tanh"] * len(UNITS), T, "linear", LOOKBACK)
    x = torch.from_numpy(np.ascontiguousarray(np.concatenate([f.values for f in frames]))).to(eng.device)
    kw = {}
    if one_per_chunk:
        kw["memory_budget"] = eng.fit_workspace_bytes(K + 1) + eng.lib.gb_lstm_fit_stop_state_bytes(K + 1) + (K + 1) * eng.param_stride * 4
    fb = fleet.build_lstm_fleet(eng, x, x, N, lookahead=la, epochs=EPOCHS, batch_size=BF, n_splits=K, seed=5, input_scaler=scaled,
                                keep_init_params=True, early_stopping=FLEET_RULES, **kw)
    torch.cuda.synchronize()
    test = N // (K + 1)
    starts = [N - (K - k) * test for k in range(K)]
    ran_any = set()
    for m, frame in enumerate(frames):
        Xv = frame.values
        for j, n_rows in enumerate([N] + starts):
            x_in = MinMaxScaler().fit(Xv[:n_rows]).transform(Xv).astype(np.float32) if scaled else Xv.astype(np.float32)
            xd, yd = (torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(eng.device) for a in (x_in, Xv))
            n_win = n_rows - LOOKBACK + 1 - la
            jobs = engine.jobs_to_device(engine.make_jobs([0], [n_win], [0]), eng.device)
            p = fb.init_params[j * M + m : j * M + m + 1].clone()
            cb, state, hist = EarlyStopping(**FLEET_RULES[m]), None, []
            for e in range(EPOCHS):
                loss, _, state = eng.fit(p, jobs, 1, n_win, xd, yd, epochs=1, batch_size=BF, lookahead=la, primer=(e == 0), state=state)
                hist.append(float(loss[0, 0]))
                if cb.update(e, {"loss": hist[-1]}, lambda: p.clone()):
                    break
            if cb.restore_best_weights and cb.best_weights is not None:
                p = cb.best_weights
            got_p = fb.params[m] if j == 0 else fb.fold_params[m, j - 1]
            got_loss = fb.loss[m] if j == 0 else fb.fold_loss[m, j - 1]
            got_ran = fb.epochs_run[m] if j == 0 else fb.fold_epochs_run[m, j - 1]
            assert got_ran == len(hist), (m, j)
            assert np.array_equal(got_loss[: len(hist)], np.array(hist, np.float32)) and np.isnan(got_loss[len(hist):]).all(), (m, j)
            assert torch.equal(got_p, p[0]), (m, j)
            ran_any.add(len(hist))
        hist_attr = fb.detector(m, tags=list(frame.columns)).base_estimator._history
        assert len(hist_attr.history["loss"]) == fb.epochs_run[m] and hist_attr.params["epochs"] == EPOCHS
    assert len(ran_any) > 1


def _definition(patience, batch_size=BF, cls_name="KerasLSTMAutoEncoder"):
    lstm = {f"gordo.machine.model.models.{cls_name}": {
        "kind": "lstm_hourglass", "lookback_window": LOOKBACK, "epochs": EPOCHS, "batch_size": batch_size,
        "callbacks": [{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "loss", "patience": patience, "min_delta": HUGE}}]}}
    return {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {
        "base_estimator": {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", lstm]}}}}


def _key_tree(d):
    return {k: _key_tree(v) for k, v in d.items()} if isinstance(d, dict) else None


def test_fleet_builder_batches_a_mixed_early_stopping_project(engine, torch, caplog):
    from gordo_components_b200 import builder

    frames = _frames(count=4, n=200)
    patience = [1, 3, 4]
    machines = [{"name": f"m{i}", "model": _definition(p), "dataset": {"X": f, "y": f}} for i, (p, f) in enumerate(zip(patience, frames))]
    machines.append({"name": "wide", "model": _definition(2, batch_size=128), "dataset": {"X": frames[3], "y": frames[3]}})
    with caplog.at_level(logging.INFO, logger="gordo_components_b200.builder"):
        built = builder.FleetModelBuilder(machines, lstm_early_stopping=True, lstm_wide_batches=True).build()
    messages = [r.getMessage() for r in caplog.records]
    assert "built 3 LSTM machines in one batched bucket" in messages and "built 1 LSTM machines in one batched bucket" in messages
    assert not any("takes the per-machine path" in s for s in messages)
    lengths = [len(model.base_estimator.steps[-1][1]._history.history["loss"]) for model, _ in built]
    assert lengths == [max(p, 1) + 1 for p in patience] + [3]
    single_model, single = builder.ModelBuilder(machines[1]).build()
    assert len(single_model.base_estimator.steps[-1][1]._history.history["loss"]) == lengths[1]
    tree_a, tree_b = _key_tree(built[1][1]), _key_tree(single)
    for tree in (tree_a, tree_b):
        tree["metadata"]["build_metadata"]["dataset"] = None
    assert tree_a == tree_b
    assert built[1][0].base_estimator.steps[-1][1]._history.params["epochs"] == EPOCHS  # the configured count, as the estimator leaves it
