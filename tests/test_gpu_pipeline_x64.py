"""
Input scalers applied inside the fused predict+score launch (gb_ffae_infer_score_x64) against the two-launch route it replaces
(gb_affine_f64, then gb_ffae_infer_score on the float32 result): bit for bit, at the kernel, at the detector and through the
served request coalescer.
"""
import json
import threading

import numpy as np
import pandas as pd
import pytest

from test_gpu_builder import DETECTOR, LSTM, _series

pytestmark = pytest.mark.gpu

OUTS = ("model-output", "tag-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-scaled", "total-anomaly-unscaled",
        "anomaly-confidence", "total-anomaly-confidence")


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


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int32) if a.dtype == np.float32 else a.view(np.int64)


# (tags, variants the kernels cover there): 2 = tensor cores (64 tags: two warpgroups with float64 x, 24: three), 3 = row per thread
CASES = [(4, (0, 1, 3)), (13, (0, 1, 3)), (24, (0, 1, 2)), (64, (0, 1, 2)), (100, (0, 1))]


@pytest.mark.parametrize("T,variants", CASES, ids=[f"t{c[0]}" for c in CASES])
def test_kernel_bits_equal_the_two_launch_route(engine, torch, T, variants):
    from oracle import keras_math as km

    S = 3
    spec = km.ff_hourglass_spec(T)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    rng = np.random.default_rng(T)
    params = eng.pack_params([km.init_ff_weights(spec, np.random.default_rng(10 + s)) for s in range(S)])
    # ragged jobs off the 64-row tile, x rows with gaps between them, outputs from row 3 on
    rows = [150, 64, 1, 200, 77, 129]
    slots = [0, 1, 2, 1, 0, 2]
    x_rows = np.cumsum([5] + [r + 7 for r in rows[:-1]])
    out_rows = 3 + np.concatenate([[0], np.cumsum(rows[:-1])])
    n_x, n_out = int(x_rows[-1] + rows[-1] + 11), int(out_rows[-1] + rows[-1] + 2)
    # offset-dominated tags (values near 1e4, scale near 1e-4): the float64 rounding of x * a + b decides x'
    a = 1e-4 * rng.uniform(0.5, 2.0, (S, T))
    b = -rng.uniform(0.5, 1.5, (S, T))
    x = 1e4 * (1.0 + 0.01 * rng.standard_normal((n_x, T)))
    y = (x * 1e-4).astype(np.float32)
    x[x_rows[0] + 3, 1] = np.nan
    x[x_rows[3] + 70, :] = np.nan
    x[x_rows[1] + 5, T - 1] = 1e40 / a[1, T - 1]  # x' overflows float32: +inf
    x[x_rows[4] + 9, 0] = -1e41 / a[0, 0]
    y[x_rows[5] + 2, 2] = np.nan
    jobs_h = engine.make_jobs(slots, rows, x_rows, out_rows)
    jobs = engine.jobs_to_device(jobs_h, dev)
    td = lambda v: torch.from_numpy(np.ascontiguousarray(v)).to(dev)  # noqa: E731
    xd, ad, bd, yd = td(x), td(a), td(b), td(y)
    scale, feat, agg = td(rng.uniform(0.5, 2, (S, T)).astype(np.float32)), td(rng.uniform(0.5, 2, (S, T)).astype(np.float32)), td(rng.uniform(0.5, 2, S).astype(np.float32))
    # x' where every job reads it (the affine pass writes each job's rows at its x rows)
    x32 = torch.full((n_x, T), float("nan"), dtype=torch.float32, device=dev)
    aff_jobs = engine.jobs_to_device(engine.make_jobs(slots, rows, x_rows, x_rows), dev)
    x32.copy_(engine.affine_f64(aff_jobs, len(rows), max(rows), xd, ad, bd, out_rows=n_x))
    for v in variants:
        def outs():
            return {k: torch.full((n_out, T) if k.startswith(("model", "tag", "anomaly")) else (n_out,), -7.0, device=dev) for k in OUTS}
        old = eng.infer_score(params, jobs, len(rows), max(rows), x32, yd, scale, feat, agg, out_rows=n_out, variant=v, out=outs())
        new = eng.infer_score(params, jobs, len(rows), max(rows), xd, yd, scale, feat, agg, out_rows=n_out, variant=v, out=outs(),
                              x_affine=(ad, bd))
        torch.cuda.synchronize()
        for k in OUTS:
            np.testing.assert_array_equal(_bits(new[k].cpu().numpy()), _bits(old[k].cpu().numpy()), err_msg=f"{k} variant {v} T {T}")
        o = new["model-output"].cpu().numpy()
        assert np.isnan(o[out_rows[0] + 3]).all() and np.isfinite(o[out_rows[2]]).all()
    kernel, nwg = eng.infer_plan_x64(0)
    assert kernel == (2 if T in (24, 64) else 3 if T <= 16 else 1) and nwg == {24: 3, 64: 2}.get(T, 0)


def _frame(rows, tags, seed):
    rng = np.random.default_rng(seed)
    idx = pd.date_range("2020-01-01", periods=rows, freq="10min")
    return pd.DataFrame(1e4 + rng.standard_normal((rows, tags)) * rng.uniform(0.1, 5.0, tags), index=idx, columns=[f"tag-{i}" for i in range(tags)])


def _scalers():
    from sklearn.preprocessing import MaxAbsScaler, MinMaxScaler, RobustScaler, StandardScaler

    return {"minmax": [MinMaxScaler()], "standard": [StandardScaler()], "robust": [RobustScaler()], "maxabs": [MaxAbsScaler()],
            "minmax+standard": [MinMaxScaler(), StandardScaler()]}


@pytest.mark.parametrize("T", [8, 64])
@pytest.mark.parametrize("name", list(_scalers()))
def test_detector_frame_bytes_equal_the_two_launch_route(engine, torch, monkeypatch, T, name):
    from sklearn.pipeline import Pipeline

    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    X = _frame(400, T, T)
    steps = [(f"s{i}", s) for i, s in enumerate(_scalers()[name])] + [("ae", KerasAutoEncoder(kind="feedforward_hourglass", epochs=1))]
    det = DiffBasedAnomalyDetector(base_estimator=Pipeline(steps)).fit(X, X)
    det.feature_thresholds_, det.aggregate_threshold_ = pd.Series(np.full(T, 0.3), index=X.columns), 0.2
    req = X.iloc[37:300].copy()
    req.iloc[5, 1] = np.nan

    def fail(*a, **k):
        raise AssertionError("the Pipeline's scalers went through the separate affine pass")

    monkeypatch.setattr(engine, "affine_f64", fail)
    new = det.anomaly(req, req)
    monkeypatch.undo()
    monkeypatch.setattr(engine.FFEngine, "infer_plan_x64", lambda self, variant=0: None)  # the two-launch route
    old = det.anomaly(req, req)
    pd.testing.assert_frame_equal(new, old, check_exact=True)
    for col in new.columns:
        n, o = new[col].to_numpy(), old[col].to_numpy()
        if n.dtype.kind == "f":
            np.testing.assert_array_equal(_bits(n), _bits(o), err_msg=str(col))


REFERENCE_DEFINITION = {  # the reference's examples/config.yaml model (DiffBasedAnomalyDetector around MinMaxScaler + KerasAutoEncoder)
    "gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": {"sklearn.pipeline.Pipeline": {"steps": [
        "sklearn.preprocessing.MinMaxScaler", {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass"}}]}}}}


def test_served_pipeline_models_answer_through_the_coalescer(engine, torch, tmp_path):
    from gordo_components_b200 import builder, server

    N, T = 300, 24
    names = ["p-1", "p-2", "p-3", "bare", "lstm"]
    frames = {n: _series(N, T, seed).astype(np.float64) * 300.0 + 1e4 for seed, n in enumerate(names)}
    models = {"p-1": REFERENCE_DEFINITION, "p-2": REFERENCE_DEFINITION, "p-3": REFERENCE_DEFINITION, "bare": DETECTOR, "lstm": LSTM}
    builder.FleetModelBuilder([{"name": n, "model": models[n], "dataset": (frames[n], frames[n])} for n in names]).build(str(tmp_path))
    store = server.ModelStore(str(tmp_path))

    default = server.ResidentBucket(store)
    assert default.names == ["bare"] and not default.input_scalers  # what the default bucket held before input scalers existed
    default.close()
    bucket = server.ResidentBucket(store, input_scalers=True, max_wait_ms=20.0)
    assert bucket.names == ["p-1", "p-2", "p-3"] and bucket.input_scalers

    reqs = []
    for i in range(48):
        n = names[i % 3]
        X = frames[n].iloc[10 + i: 10 + i + 60 + i % 7]
        if i % 2:
            reqs.append((n, {"json": json.loads(json.dumps({"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(X)}))}, None))
        else:
            reqs.append((n, {"files": {"X": server.dataframe_into_parquet_bytes(X), "y": server.dataframe_into_parquet_bytes(X)}}, "parquet"))
    want = [server.anomaly_prediction(store, n, fmt=fmt, **kw) for n, kw, fmt in reqs]
    got = [None] * len(reqs)

    def worker(k):
        for i in range(k, len(reqs), 8):
            n, kw, fmt = reqs[i]
            got[i] = server.anomaly_prediction(store, n, fmt=fmt, bucket=bucket, **kw)

    threads = [threading.Thread(target=worker, args=(k,)) for k in range(8)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    for (n, _, fmt), w, g in zip(reqs, want, got):
        assert g.status == w.status == 200
        if fmt == "parquet":
            assert g.body == w.body
        else:
            assert json.dumps(g.body["data"]) == json.dumps(w.body["data"])
    co = bucket.coalescer
    assert co.requests == len(reqs) and co.batches < co.requests

    X = frames["p-2"].iloc[:40].copy()
    X.iloc[3, 2] = np.inf
    payload = {"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(frames["p-2"].iloc[:40])}
    with pytest.raises(ValueError) as per_request:
        server.anomaly_prediction(store, "p-2", json=payload)
    with pytest.raises(ValueError) as served:
        server.anomaly_prediction(store, "p-2", json=payload, bucket=bucket)
    assert str(served.value) == str(per_request.value)
    assert co.requests == len(reqs)  # refused before any launch
    bucket.close()
