"""
Anomaly requests to smoothing-window K-fold detectors (the reference's production definition, DiffBasedKFCVAnomalyDetector with
window=144, smm) through ``server.anomaly_prediction``: one request at a time (the per-request route: one fused launch, plus four
gb_smooth round trips when the reply carries the smoothed columns) against ``ResidentBucket(store, smoothing=True)`` (the waiting
requests of all threads as one fused launch, plus one gb_smooth_scores launch over those that asked).

1 000 device-resident 64-tag feedforward_hourglass detectors, 244-row JSON requests (100 rows plus the 144 rows of history the
reference's docs tell clients to fetch, so the first reported row has a full window), 8 client threads (gunicorn threads per worker
in the reference).  Four arms: each route with ``all_columns`` off (the default reply) and on.  The arms' replies must be the same
bytes.  A separate pass times, with CUDA events, the fused launch and the gb_smooth_scores launch of a batch of the size the bucket
formed in its all-columns arm.

``--ttr`` serves the reference's real production definition instead: the estimator is ``TransformedTargetRegressor(transformer=
MinMaxScaler, regressor=Pipeline([MinMaxScaler, KerasAutoEncoder]))``, through ``ResidentBucket(store, input_scalers=True,
smoothing=True, target_scaler=True)`` (prediction-only fused launch, then gb_minmax_inverse_score_f64 and float64 smoothing input).
Its kernel pass times, with CUDA events, gb_minmax_inverse_score_f64 against gb_minmax_inverse_f32 + gb_anomaly_score_f64 at the
fold-scoring shape of ``bench_fleet_builder.py --kfcv`` (125 machines x 10 000 rows x 64 tags, 5 folds), for the two outputs the
builder asks for; algorithmic bytes per 64-tag row are 2 568 for the pair and 1 544 for the single pass.

    python benchmarks/bench_smoothed_server.py [--machines 1000] [--requests 400] [--ttr]

Prints one JSON line (progress goes to stderr).
"""
import argparse, json, os, subprocess, sys, tempfile, threading, time
import numpy as np
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

TAGS, WINDOW = 64, 144


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def _production_estimator(ae, rng):
    """The production definition's fitted TransformedTargetRegressor around ``ae``, without the training."""
    from sklearn.compose import TransformedTargetRegressor
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import MinMaxScaler

    reg = Pipeline([("s", MinMaxScaler().fit(rng.random((50, TAGS)) * 10)), ("m", ae)])
    ttr = TransformedTargetRegressor(transformer=MinMaxScaler(), regressor=reg)
    ttr._training_dim, ttr.transformer_, ttr.regressor_ = 2, MinMaxScaler().fit(rng.random((50, TAGS)) * 10), reg
    return ttr


def make_store(root, machines, ttr=False):
    import pandas as pd

    from gordo_components_b200 import serializer, server
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedKFCVAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    rng = np.random.default_rng(0)
    tags = [f"TAG {i}" for i in range(TAGS)]
    meta = {"dataset": {"tag_list": tags, "resolution": "10min"}}
    for m in range(machines):
        ae = KerasAutoEncoder(kind="feedforward_hourglass")
        ae.kwargs.update({"n_features": TAGS, "n_features_out": TAGS})
        ae._prepare_model()  # Glorot-initialised weights: the arithmetic of a trained model, without the training
        det = DiffBasedKFCVAnomalyDetector(base_estimator=_production_estimator(ae, rng) if ttr else ae, window=WINDOW, smoothing_method="smm")
        det.scaler.fit(rng.random((50, TAGS)) * 10)
        det.feature_thresholds_ = pd.Series(rng.random(TAGS) + 0.5, index=tags)
        det.aggregate_threshold_ = float(rng.random() + 0.5)
        serializer.dump(det, os.path.join(root, f"kfold-{m:04d}"), metadata=meta)
    return server.ModelStore(root)


def payloads(store, n, rows, seed):
    import pandas as pd

    from gordo_components_b200 import server

    rng = np.random.default_rng(seed)
    names = store.names()
    idx = pd.date_range("2020-01-01", periods=rows, freq="10min", tz="UTC")
    out = []
    for k in range(n):
        X = pd.DataFrame(rng.random((rows, TAGS)) * 10, index=idx, columns=store.tags(names[0]))
        y = X + rng.normal(0, 0.1, X.shape)
        out.append((names[int(rng.integers(len(names)))], {"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(y)}))
    return out


def drive(store, reqs, threads, all_columns, bucket):
    from gordo_components_b200 import server

    idx = iter(range(len(reqs)))
    lock = threading.Lock()
    out = [None] * len(reqs)

    def worker():
        while True:
            with lock:
                i = next(idx, None)
            if i is None:
                return
            name, payload = reqs[i]
            r = server.anomaly_prediction(store, name, json=payload, all_columns=all_columns, bucket=bucket)
            assert r.status == 200, r.body
            out[i] = json.dumps(r.body["data"])

    ts = [threading.Thread(target=worker) for _ in range(threads)]
    t0 = time.perf_counter()
    [t.start() for t in ts]
    [t.join() for t in ts]
    return time.perf_counter() - t0, out


def launch_times(torch, bucket, k, rows, reps):
    """Median CUDA-event times (ms) of the fused launch and of gb_smooth_scores for one batch of k requests of ``rows`` rows."""
    from gordo_components_b200 import _cabi, engine

    co = bucket.coalescer
    dev = co.eng.device
    n = k * rows
    rng = np.random.default_rng(1)
    jobs_h = engine.make_jobs(rng.integers(0, co.params.shape[0], k), rows, np.arange(k) * rows)
    jobs = engine.jobs_to_device(jobs_h, dev)
    x = torch.rand((n, TAGS), device=dev) * 10
    y = x + 0.1
    out = {key: torch.empty((n, TAGS) if key.startswith("tag") or key in ("model-output", "anomaly-confidence") else (n,), device=dev) for key in co.want}
    sm = {key: torch.empty_like(out[key]) for key in engine.SMOOTH_SCORE_KEYS}
    lib, p = _cabi.load_library(), _cabi.ptr

    def fused():
        co.eng.infer_score(co.params, jobs, k, rows, x, y, co.scale, co.feat_thr, co.agg_thr, out_rows=n, want=co.want, out=out)

    def smooth():
        _cabi.check(lib.gb_smooth_scores(p(jobs), k, rows, *(p(out[key]) for key in engine.SMOOTH_SCORE_KEYS), 0, TAGS, WINDOW,
                                         engine.SMOOTH_METHODS["smm"], *(p(sm[key]) for key in engine.SMOOTH_SCORE_KEYS), engine._stream_ptr()))

    res = {}
    for name, fn in (("fused", fused), ("smooth_scores", smooth)):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        res[name] = {"ms_median": float(np.median(ms)), "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms))}
    res["smooth_over_fused"] = res["smooth_scores"]["ms_median"] / res["fused"]["ms_median"]
    return res


def ttr_kernel_times(torch, reps, machines=125, rows=10_000, folds=5):
    """Median CUDA-event times (ms) of the K-fold fold scoring of TTR buckets: gb_minmax_inverse_f32 + gb_anomaly_score_f64 against
    gb_minmax_inverse_score_f64, both asked for tag-anomaly-unscaled and total-anomaly-scaled (what build_kfold_fleet asks for).
    Outputs are checked bit for bit before timing."""
    from gordo_components_b200 import engine

    dev = engine.cuda_device()
    rng = np.random.default_rng(3)
    n_test = rows // folds
    km, total = machines * folds, machines * rows
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(km), n_test, np.arange(km) * n_test), dev)
    pred = torch.rand((total, TAGS), device=dev)
    y = torch.rand((total, TAGS), device=dev, dtype=torch.float64) * 100
    y_scale = torch.rand((km, TAGS), device=dev, dtype=torch.float64) * 0.1 + 0.01
    y_min = -torch.rand((km, TAGS), device=dev, dtype=torch.float64)
    mult = torch.rand((km, TAGS), device=dev, dtype=torch.float64)
    want = ("tag-anomaly-unscaled", "total-anomaly-scaled")

    def pair():
        back = engine.minmax_inverse_f32(jobs, km, n_test, pred, y_scale, y_min)
        res = engine.anomaly_score(jobs, km, n_test, back["f64"], y, TAGS, scale=mult, want=want)
        res["model-output"] = back["f32"]
        return res

    def fused():
        return engine.minmax_inverse_score_f64(jobs, km, n_test, pred, y, y_scale, y_min, scale=mult, want=want)

    a, b = pair(), fused()
    identical = all(torch.equal(a[k].view(torch.uint8) if a[k].dtype == torch.float32 else a[k].view(torch.int64),
                                b[k].view(torch.uint8) if b[k].dtype == torch.float32 else b[k].view(torch.int64)) for k in a)
    del a, b
    res = {"shape": {"machines": machines, "rows": rows, "folds": folds, "tags": TAGS}, "bit_identical": bool(identical),
           "bytes_per_row": {"inverse_f32_plus_score_f64": 2568, "inverse_score_f64": 1544}}
    for name, fn in (("inverse_f32_plus_score_f64", pair), ("inverse_score_f64", fused)):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        med = float(np.median(ms))
        res[name] = {"ms_median": med, "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms)),
                     "GB_per_s": res["bytes_per_row"][name] * total / (med * 1e-3) / 1e9}
    res["speedup"] = res["inverse_f32_plus_score_f64"]["ms_median"] / res["inverse_score_f64"]["ms_median"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--machines", type=int, default=1000)
    ap.add_argument("--requests", type=int, default=400)
    ap.add_argument("--rows", type=int, default=100 + WINDOW)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--ttr", action="store_true", help="the production definition's TransformedTargetRegressor estimator")
    a = ap.parse_args()
    import torch
    import __graft_entry__ as ge

    ge.build()
    from gordo_components_b200 import server

    with tempfile.TemporaryDirectory() as root:
        t0 = time.perf_counter()
        store = make_store(root, a.machines, a.ttr)
        for n in store.names():
            est = store.model(n).base_estimator
            (est.regressor_.steps[-1][1] if a.ttr else est)._device_params()  # every model's weights on the device before any arm, for both routes
        setup_s = time.perf_counter() - t0
        print(f"{a.machines} models resident in {setup_s:.1f} s", file=sys.stderr, flush=True)
        bucket = (server.ResidentBucket(store, input_scalers=True, smoothing=True, target_scaler=True) if a.ttr
                  else server.ResidentBucket(store, smoothing=True))
        assert len(bucket.names) == a.machines and bucket.smoothing == (WINDOW, "smm")
        warm = payloads(store, 3 * a.threads, a.rows, 1)
        reqs = payloads(store, a.requests, a.rows, 2)
        arms = {}
        replies = {}
        for all_columns in (False, True):
            for route, b in (("per_request", None), ("bucket", bucket)):
                drive(store, warm, a.threads, all_columns, b)
                b0, r0 = bucket.coalescer.batches, bucket.coalescer.requests
                secs, out = drive(store, reqs, a.threads, all_columns, b)
                key = f"{route}_{'all_columns' if all_columns else 'default'}"
                arms[key] = {"req_per_s": len(reqs) / secs, "seconds": secs}
                if b is not None:
                    arms[key].update(batches=bucket.coalescer.batches - b0, requests=bucket.coalescer.requests - r0)
                replies[key] = out
                print(f"{key}: {arms[key]}", file=sys.stderr, flush=True)
        same = {c: replies[f"per_request_{c}"] == replies[f"bucket_{c}"] for c in ("default", "all_columns")}
        on = arms["bucket_all_columns"]
        k = max(1, round(on["requests"] / max(on["batches"], 1)))
        launches = ttr_kernel_times(torch, min(a.reps, 50)) if a.ttr else launch_times(torch, bucket, k, a.rows, a.reps)
        bucket.close()
    print(json.dumps({"card": card(), "estimator": "ttr" if a.ttr else "autoencoder", "machines": a.machines, "tags": TAGS, "window": WINDOW, "method": "smm", "rows_per_request": a.rows,
                      "requests": a.requests, "threads": a.threads, "setup_s": setup_s, "arms": arms, "replies_identical": same,
                      "per_batch_launches": {"requests_per_batch": k, **launches}}))


if __name__ == "__main__":
    main()
