"""
TransformedTargetRegressor(MinMaxScaler()) detectors under a TimeSeriesSplit in the batched builds (fleet.build_fleet and
fleet.build_lstm_fleet with target_scaler=True, FleetModelBuilder(target_scaler=True)) on the H100: every fit slot against a one-slot
replay on the scaled targets that slot's estimator receives, the transformers and detector scalers against sklearn, the fold
thresholds against the per-machine cross_validate run on the batched fold models, and the builder end to end, served through
ResidentBucket(target_scaler=True, input_scalers=True).
"""
import json
import logging

import numpy as np
import pandas as pd
import pytest
from sklearn.base import clone
from sklearn.model_selection import TimeSeriesSplit
from sklearn.pipeline import Pipeline
from sklearn.preprocessing import MinMaxScaler

pytestmark = pytest.mark.gpu

K, T = 3, 5
DET = "gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector"
AE = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "batch_size": 32, "compression_factor": 0.5,
                                                      "encoding_layers": 1, "func": "tanh", "out_func": "linear", "epochs": 3}}
ATTRS = ("scale_", "min_", "data_min_", "data_max_", "data_range_", "n_samples_seen_", "n_features_in_")


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("needs an H100")
    import __graft_entry__ as ge

    ge.build()
    return t


def _frame(rows, seed, tags=T):
    rng = np.random.default_rng(seed)
    s = np.linspace(0, 20, rows)[:, None]
    v = 3.0 + np.sin(s * rng.uniform(0.5, 2, tags) + rng.uniform(0, 6, tags)) * rng.uniform(0.5, 40, tags) + rng.normal(0, 0.05, (rows, tags))
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(v, index=idx, columns=[f"tag-{i}" for i in range(tags)])


def _lstm(cls_name, **kw):
    return {f"gordo.machine.model.models.{cls_name}": {"kind": "lstm_hourglass", "lookback_window": 5, "epochs": 2, "batch_size": 16, **kw}}


def _piped(net):
    return {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", net]}}


def _ttr(regressor):
    return {"sklearn.compose.TransformedTargetRegressor": {"transformer": "sklearn.preprocessing.MinMaxScaler", "regressor": regressor}}


def _definition(base, **kw):
    return {DET: {"base_estimator": _ttr(base), **kw}}


def _same_bits(a, b, name=""):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (name, a.shape, b.shape, a.dtype, b.dtype)
    assert np.array_equal(a, b, equal_nan=True), name


def _host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)


# ------------------------------------------------------------------------------------------------ 1. fit replay, slot by slot
@pytest.mark.parametrize("form", ["bare", "piped", "piped-own-targets"])
def test_every_feed_forward_fit_slot_replays(torch, form):
    from gordo_components_b200 import engine, fleet
    from gordo_components_b200.machine.model.factories.feedforward_autoencoder import feedforward_hourglass

    M, N, E, B = 3, 211, 4, 32
    spec = feedforward_hourglass(n_features=T, compression_factor=0.5, encoding_layers=1, func="tanh", out_func="linear")
    eng = engine.ff_engine_for(spec)
    dev = eng.device
    X = np.ascontiguousarray(np.concatenate([_frame(N, m).values for m in range(M)]))  # frame values are column-major
    Y = np.ascontiguousarray(X * 3.0 - 7.0) if form == "piped-own-targets" else X
    xd = torch.from_numpy(X).to(dev)
    yd = xd if Y is X else torch.from_numpy(Y).to(dev)
    piped = form != "bare"
    fb = fleet.build_fleet(eng, xd, yd, N, epochs=E, batch_size=B, n_splits=K, seed=5, adam=spec.adam, shuffle=False, input_scaler=piped,
                           target_scaler=True, keep_init_params=True)
    _, starts = fleet.tss_layout([N] * M, K)
    for m in range(M):
        Xm, Ym = X[m * N:(m + 1) * N], Y[m * N:(m + 1) * N]
        for j, n_rows in enumerate([N] + list(starts[m])):
            slot = m if j == 0 else M + (j - 1) * M + m
            xs = MinMaxScaler().fit(Xm[:n_rows]).transform(Xm[:n_rows]) if piped else Xm[:n_rows]
            ys = MinMaxScaler().fit(Ym[:n_rows]).transform(Ym[:n_rows])  # what TransformedTargetRegressor.fit hands its regressor
            p = fb.init_params[slot:slot + 1].clone()
            jobs = engine.jobs_to_device(engine.make_jobs([0], [n_rows], [0]), dev)
            loss, *_ = eng.fit_split(p, jobs, 1, n_rows, torch.from_numpy(xs.astype(np.float32)).to(dev), torch.from_numpy(ys.astype(np.float32)).to(dev),
                                     epochs=E, batch_size=B, shuffle=False, adam=spec.adam, seed=5)
            got = fb.params[m] if j == 0 else fb.fold_params[m, j - 1]
            got_loss = fb.loss[m] if j == 0 else fb.fold_loss[m, j - 1]
            assert torch.equal(got, p[0]), (m, j, "weights")
            assert torch.equal(got_loss, loss[0]), (m, j, "loss")
            if j:
                _same_bits(fb.fold_y_min[m, j - 1], Ym[:n_rows].min(0), "fold y_min")
                _same_bits(fb.fold_y_max[m, j - 1], Ym[:n_rows].max(0), "fold y_max")


@pytest.mark.parametrize("cls_name,piped", [("KerasLSTMAutoEncoder", False), ("KerasLSTMAutoEncoder", True), ("KerasLSTMForecast", False),
                                            ("KerasLSTMForecast", True)])
def test_every_lstm_fit_slot_replays(torch, cls_name, piped):
    from gordo_components_b200 import engine, fleet
    from oracle import keras_math as km

    M, N, L, E, B = 3, 130, 5, 2, 16
    la = 1 if cls_name == "KerasLSTMForecast" else 0
    spec = km.lstm_hourglass_spec(T, lookback_window=L)
    eng = engine.LSTMEngine(spec.n_features, spec.units, spec.acts, spec.n_features_out, spec.out_func, spec.lookback_window)
    dev = eng.device
    X = np.ascontiguousarray(np.concatenate([_frame(N, 10 + m).values for m in range(M)]))
    xd = torch.from_numpy(X).to(dev)
    fb = fleet.build_lstm_fleet(eng, xd, xd, N, lookahead=la, epochs=E, batch_size=B, n_splits=K, seed=7, input_scaler=piped, target_scaler=True,
                                keep_init_params=True)
    for m in range(M):
        Xm = X[m * N:(m + 1) * N]
        for j, n_rows in enumerate([N] + list(fb.machine_starts[m])):
            slot = m if j == 0 else M + (j - 1) * M + m
            sc = MinMaxScaler().fit(Xm[:n_rows])  # the transformer, and the Pipeline's input scaler: both see the slot's rows
            xs = sc.transform(Xm[:n_rows]) if piped else Xm[:n_rows]
            ys = sc.transform(Xm[:n_rows])
            p = fb.init_params[slot:slot + 1].clone()
            windows = n_rows - L + 1 - la
            jobs = engine.jobs_to_device(engine.make_jobs([0], [windows], [0]), dev)
            loss, *_ = eng.fit_for_batch(B)(p, jobs, 1, windows, torch.from_numpy(xs.astype(np.float32)).to(dev),
                                            torch.from_numpy(ys.astype(np.float32)).to(dev), epochs=E, batch_size=B, lookahead=la, primer=True)
            got = fb.params[m] if j == 0 else fb.fold_params[m, j - 1]
            assert torch.equal(got, p[0]), (m, j, "weights")
            _same_bits(fb.loss[m] if j == 0 else fb.fold_loss[m, j - 1], loss[0].cpu().numpy(), "loss")


# ------------------------------------------------------------------------------------------------ 2. thresholds against the per-machine path
def _fold_detector(definition, eng, fold_params, prefix, lstm: bool):
    """Fold k's detector as sklearn's cross_validate leaves it, around the batched fold model: scalers fitted by sklearn on the prefix."""
    from gordo_components_b200 import serializer
    from gordo_components_b200.machine.model.models import FittedNet

    det = serializer.from_definition(definition)
    ttr = det.base_estimator
    reg = clone(ttr.regressor)
    net = reg.steps[-1][1] if isinstance(reg, Pipeline) else reg
    if isinstance(reg, Pipeline):
        reg.steps[0][1].fit(prefix)
    net.kwargs.update({"n_features": T, "n_features_out": T})
    weights = eng.unpack_params(fold_params)[0]
    if lstm:
        net.model = FittedNet(net._build_spec(), weights)
    else:
        net._prepare_model()
        net.model.weights = weights
    ttr.transformer_, ttr.regressor_, ttr._training_dim = MinMaxScaler().fit(prefix.values), reg, 2
    det.scaler = MinMaxScaler().fit(prefix)  # cross_validate's clone gives every fold its own; the definition's default is shared
    return det


def _per_machine_thresholds(monkeypatch, definition, frame, folds):
    from gordo_components_b200 import serializer
    from gordo_components_b200.machine.model.anomaly import diff

    monkeypatch.setattr(diff, "sk_cross_validate", lambda est, X, y, **kw: {"estimator": folds})
    det = serializer.from_definition(definition)
    det.cross_validate(X=frame, y=frame, cv=TimeSeriesSplit(n_splits=K))
    return det


def _check_thresholds(ref, fold_feat, fold_agg, fold_sfeat, fold_sagg, window):
    _same_bits(ref.feature_thresholds_per_fold_.to_numpy(), fold_feat, "fold feature thresholds")
    _same_bits(np.asarray(list(ref.aggregate_thresholds_per_fold_.values())), fold_agg, "fold aggregate thresholds")
    if window is not None:
        _same_bits(ref.smooth_feature_thresholds_per_fold_.to_numpy(), fold_sfeat, "smooth fold feature thresholds")
        _same_bits(np.asarray(list(ref.smooth_aggregate_thresholds_per_fold_.values())), fold_sagg, "smooth fold aggregate thresholds")


def _check_scalers(det, frame, piped):
    sk = MinMaxScaler().fit(frame)
    for name in ATTRS:
        _same_bits(getattr(det.scaler, name), getattr(sk, name), f"detector scaler {name}")
    assert list(det.scaler.feature_names_in_) == list(frame.columns)
    target = MinMaxScaler().fit(frame.values)  # TransformedTargetRegressor.fit validates y into an array first
    for name in ATTRS:
        _same_bits(getattr(det.base_estimator.transformer_, name), getattr(target, name), f"transformer {name}")
    assert not hasattr(det.base_estimator.transformer_, "feature_names_in_")
    if piped:
        for name in ("scale_", "min_"):
            _same_bits(getattr(det.base_estimator.regressor_.steps[0][1], name), getattr(sk, name), f"input scaler {name}")


@pytest.mark.parametrize("piped", [False, True], ids=["bare", "piped"])
@pytest.mark.parametrize("window", [None, 12])
def test_feed_forward_thresholds_equal_the_per_machine_path(torch, monkeypatch, piped, window):
    from gordo_components_b200 import engine, fleet, serializer

    M, N = 3, 240
    base = _piped(AE) if piped else AE
    definition = _definition(base, **({} if window is None else {"window": window}))
    frames = [_frame(N, 20 + m) for m in range(M)]
    template = serializer.from_definition(definition)
    ae = template.base_estimator.regressor
    ae = ae.steps[-1][1] if piped else ae
    ae.kwargs.update({"n_features": T, "n_features_out": T})
    spec = ae._build_spec()
    eng = engine.ff_engine_for(spec)
    xd = torch.from_numpy(np.ascontiguousarray(np.concatenate([f.values for f in frames]))).to(eng.device)
    fb = fleet.build_fleet(eng, xd, xd, N, epochs=3, batch_size=32, n_splits=K, seed=1, adam=spec.adam, input_scaler=piped, target_scaler=True,
                           window=window)
    tags = list(frames[0].columns)
    for m, frame in enumerate(frames):
        folds = [_fold_detector(definition, eng, fb.fold_params[m, k:k + 1], frame.iloc[:int(fb.starts[m, k])], lstm=False) for k in range(K)]
        ref = _per_machine_thresholds(monkeypatch, definition, frame, folds)
        _check_thresholds(ref, _host(fb.fold_feat_thr[m]), _host(fb.fold_agg_thr[m]),
                          None if window is None else _host(fb.fold_smooth_feat_thr[m]), None if window is None else _host(fb.fold_smooth_agg_thr[m]), window)
        assert np.isfinite(_host(fb.fold_feat_thr[m])).all()
        det = fb.detector(m, tags=tags, template=serializer.from_definition(definition), input_tags=tags)
        _check_scalers(det, frame, piped)
        _same_bits(det.feature_thresholds_.to_numpy(), ref.feature_thresholds_.to_numpy(), "feature_thresholds_")
        assert det.aggregate_threshold_ == ref.aggregate_threshold_
        assert type(det.base_estimator.regressor) is type(det.base_estimator.regressor_)
        assert det.base_estimator.regressor_ is not det.base_estimator.regressor  # a fitted clone, as sklearn leaves it


@pytest.mark.parametrize("cls_name,piped,window", [("KerasLSTMAutoEncoder", False, None), ("KerasLSTMAutoEncoder", True, 12),
                                                   ("KerasLSTMForecast", False, 12), ("KerasLSTMForecast", True, None)])
def test_lstm_thresholds_equal_the_per_machine_path(torch, monkeypatch, cls_name, piped, window):
    from gordo_components_b200 import engine, fleet, serializer
    from oracle import keras_math as km

    M, N, L = 3, 160, 5
    la = 1 if cls_name == "KerasLSTMForecast" else 0
    net = _lstm(cls_name)
    definition = _definition(_piped(net) if piped else net, **({} if window is None else {"window": window}))
    spec = km.lstm_hourglass_spec(T, lookback_window=L)
    eng = engine.LSTMEngine(spec.n_features, spec.units, spec.acts, spec.n_features_out, spec.out_func, spec.lookback_window)
    frames = [_frame(N, 40 + m) for m in range(M)]
    xd = torch.from_numpy(np.ascontiguousarray(np.concatenate([f.values for f in frames]))).to(eng.device)
    fb = fleet.build_lstm_fleet(eng, xd, xd, N, lookahead=la, epochs=2, batch_size=16, n_splits=K, seed=3, input_scaler=piped, target_scaler=True,
                                window=window)
    tags = list(frames[0].columns)
    for m, frame in enumerate(frames):
        folds = [_fold_detector(definition, eng, fb.fold_params[m, k:k + 1], frame.iloc[:int(fb.machine_starts[m, k])], lstm=True) for k in range(K)]
        ref = _per_machine_thresholds(monkeypatch, definition, frame, folds)
        _check_thresholds(ref, fb.fold_feat_thr[m], fb.fold_agg_thr[m], None if window is None else fb.fold_smooth_feat_thr[m],
                          None if window is None else fb.fold_smooth_agg_thr[m], window)
        for k in range(K):  # the fold predictions are in target units: what the fold TransformedTargetRegressor predicts
            test = frame.iloc[int(fb.machine_starts[m, k]):int(fb.machine_starts[m, k]) + N // (K + 1)]
            _same_bits(fb.fold_predictions[m, k].cpu().numpy(), folds[k].predict(test), "fold predictions")
        det = fb.detector(m, tags=tags, template=serializer.from_definition(definition), input_tags=tags)
        _check_scalers(det, frame, piped)
        lstm = det.base_estimator.regressor_.steps[-1][1] if piped else det.base_estimator.regressor_
        assert type(lstm).__name__ == cls_name and lstm.lookahead == la
        assert type(det.base_estimator.regressor) is type(det.base_estimator.regressor_)


# ------------------------------------------------------------------------------------------------ 3. FleetModelBuilder end to end
def _keys(d):
    return {k: _keys(v) for k, v in d.items()} if isinstance(d, dict) else None


def _same_shape(batched, single):
    a, b = _keys(batched), _keys(single)
    for tree in (a, b):
        tree["metadata"]["build_metadata"]["dataset"] = None  # whatever the data source reports
    assert a == b


def test_fleet_builder_builds_ttr_machines_in_one_bucket_per_family(torch, tmp_path, caplog):
    from gordo_components_b200 import builder, serializer, server

    stop = [{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "val_loss", "patience": 1, "min_delta": 0.5, "restore_best_weights": True}}]
    ff_net = {"gordo.machine.model.models.KerasAutoEncoder": {**AE["gordo.machine.model.models.KerasAutoEncoder"], "epochs": 5,
                                                              "validation_split": 0.1, "callbacks": stop}}
    ff = _definition(_piped(ff_net))
    lstm = _definition(_lstm("KerasLSTMForecast"), window=12, smoothing_method="sma")
    frames = {f"ff-{i}": _frame(400, 60 + i) for i in range(3)} | {f"lstm-{i}": _frame(200, 70 + i) for i in range(3)}
    machines = [{"name": name, "model": ff if name.startswith("ff") else lstm, "dataset": {"X": frame, "y": frame}} for name, frame in frames.items()]
    calls = []
    orig = builder.FleetModelBuilder._build_bucket
    builder.FleetModelBuilder._build_bucket = staticmethod(lambda members: calls.append((type(members[0]).__name__, len(members))) or orig(members))
    try:
        with caplog.at_level(logging.INFO, logger="gordo_components_b200.builder"):
            out = builder.FleetModelBuilder(machines, target_scaler=True, early_stopping=True, smoothing=True).build(str(tmp_path))
    finally:
        builder.FleetModelBuilder._build_bucket = staticmethod(orig)
    assert sorted(calls) == [("_Canonical", 3), ("_CanonicalLSTM", 3)]
    messages = [r.getMessage() for r in caplog.records]
    assert not any("per-machine path" in s or "one at a time" in s for s in messages), messages
    results = {meta["name"]: (model, meta) for model, meta in out}
    for name in ("ff-0", "lstm-0"):
        machine = next(m for m in machines if m["name"] == name)
        single_model, single_meta = builder.ModelBuilder(dict(machine)).build()
        model, meta = results[name]
        _same_shape(meta, single_meta)
        assert sorted(vars(model)) == sorted(vars(single_model))
        assert sorted(vars(model.base_estimator)) == sorted(vars(single_model.base_estimator))
        assert sorted(vars(model.base_estimator.transformer_)) == sorted(vars(single_model.base_estimator.transformer_))
        assert sorted(vars(model.scaler)) == sorted(vars(single_model.scaler))
        mm, sm = (m["metadata"]["build_metadata"]["model"] for m in (meta, single_meta))
        assert mm["model_offset"] == sm["model_offset"]
        assert mm["cross_validation"]["splits"] == sm["cross_validation"]["splits"]
        assert set(mm["model_meta"]) == set(sm["model_meta"])
    for model, meta in out:
        cvm = meta["metadata"]["build_metadata"]["model"]["cross_validation"]
        assert cvm["scores"] and all(np.isfinite(list(v.values())).all() for v in cvm["scores"].values()), meta["name"]
        if meta["name"].startswith("ff"):
            hist = meta["metadata"]["build_metadata"]["model"]["model_meta"]["history"]
            assert list(hist) == ["loss", "accuracy", "val_loss", "val_accuracy", "params"] and 1 <= len(hist["loss"]) <= hist["params"]["epochs"] == 5
        else:
            assert model.window == 12 and model.smoothing_method == "sma" and np.isfinite(model.smooth_aggregate_threshold_)
        # every detector has its own scaler, fitted on its own targets (the definitions leave the detector's default scaler)
        sk = MinMaxScaler().fit(frames[meta["name"]])
        for name in ATTRS:
            _same_bits(getattr(model.scaler, name), getattr(sk, name), f"{meta['name']} scaler {name}")
    assert len({id(model.scaler) for model, _ in out}) == len(out)

    # the dumped feed-forward models answer through a resident bucket exactly as through the per-request route
    served = tmp_path / "served"
    names = [f"ff-{i}" for i in range(3)]
    for name in names:
        det = serializer.load(str(tmp_path / name))
        assert type(det.base_estimator).__name__ == "TransformedTargetRegressor"
        serializer.dump(det, str(served / name), metadata={"dataset": {"tag_list": list(frames[name].columns), "resolution": "10min"}})
    store = server.ModelStore(str(served))
    bucket = server.ResidentBucket(store, names=names, target_scaler=True, input_scalers=True, max_wait_ms=20)
    try:
        assert sorted(bucket.names) == names
        for k in range(6):
            X = _frame(80 + 30 * k, 500 + k)
            payload = {"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(X)}
            want = server.anomaly_prediction(store, names[k % 3], json=payload, all_columns=k % 2 == 0)
            got = server.anomaly_prediction(store, names[k % 3], json=payload, all_columns=k % 2 == 0, bucket=[bucket])
            assert want.status == got.status == 200
            assert json.dumps(got.body["data"]) == json.dumps(want.body["data"])
        assert bucket.coalescer.requests > 0
    finally:
        bucket.close()
