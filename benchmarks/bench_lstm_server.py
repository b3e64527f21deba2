"""
LSTM anomaly requests through ``server.anomaly_prediction``: one request at a time (the per-request route, one tensor-core launch
sequence of lookback x n_layers step launches each) against ``ResidentBucket(store, lstm=True)`` (the waiting requests of all
threads as one ragged launch sequence).  BASELINE configs[3] architecture (128 tags, lstm_symmetric 256/128/64, lookback 144),
32 models, 8 client threads (gunicorn threads per worker in the reference), parquet in and out.  Three workloads:

  (a) uniform: every request 100 windows;
  (b) mixed:   one request in 64 has 10 000 windows (the uniform layout would give every job of its batch 79 tiles);
  (c) overlap: every request 100 windows from ``--overlap-threads`` threads (32), served by a bucket that waits
      ``--overlap-wait-ms`` (5 ms) for a batch to fill, so that requests actually share launches.  At 8 threads and the default
      1 ms the host work around each request leaves few requests waiting at once.

``--ttr`` wraps every model as the production base estimator in LSTM form, ``TransformedTargetRegressor(MinMaxScaler(),
Pipeline([MinMaxScaler(), KerasLSTMAutoEncoder]))``, served through ``ResidentBucket(lstm=True, target_scaler=True)``; the per-request
route then adds sklearn's host inverse and a copy back to the device per request.

The two arms run alternately in one process.  The result records the card (name, power limit and max SM clock from
nvidia-smi, read in the same run), batches per request and whether the two arms' replies were the same bytes; the run exits
non-zero when they were not.

    python benchmarks/bench_lstm_server.py [--requests 256] [--reps 2] [--ttr]
"""
import argparse, json, os, subprocess, sys, tempfile, threading, time
import numpy as np
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

TAGS, LOOKBACK, MODELS = 128, 144, 32


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def make_store(root, ttr=False):
    import pandas as pd
    from sklearn.compose import TransformedTargetRegressor
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200 import serializer, server
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasLSTMAutoEncoder

    rng = np.random.default_rng(0)
    tags = [f"TAG {i}" for i in range(TAGS)]
    for m in range(MODELS):
        net = KerasLSTMAutoEncoder(kind="lstm_symmetric", lookback_window=LOOKBACK).initialize(TAGS, TAGS)
        if ttr:  # the state TransformedTargetRegressor.fit leaves, with statistics of the payloads' range
            est = TransformedTargetRegressor(transformer=MinMaxScaler(), regressor=Pipeline([("s", MinMaxScaler()), ("m", net)]))
            est._training_dim = 2
            est.transformer_ = MinMaxScaler().fit(rng.random((50, TAGS)) * 10)
            est.regressor_ = Pipeline([("s", MinMaxScaler().fit(rng.random((50, TAGS)) * 10)), ("m", net)])
            net = est
        det = DiffBasedAnomalyDetector(base_estimator=net, scaler=MinMaxScaler().fit(rng.random((50, TAGS)) * 10))
        det.feature_thresholds_ = pd.Series(rng.random(TAGS) + 0.5, index=tags)
        det.aggregate_threshold_ = float(rng.random() + 0.5)
        serializer.dump(det, os.path.join(root, f"m-{m:02d}"), metadata={"dataset": {"tag_list": [{"name": t} for t in tags]}})
    return server.ModelStore(root)


def payloads(n_req, mixed, seed):
    import pandas as pd

    from gordo_components_b200 import server

    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_req):
        windows = 10000 if mixed and k % 64 == 0 else 100
        rows = windows + LOOKBACK - 1
        frame = pd.DataFrame(rng.random((rows, TAGS)) * 10, index=pd.date_range("2020-01-01", periods=rows, freq="10min", tz="UTC"),
                             columns=[f"TAG {i}" for i in range(TAGS)])
        raw = server.dataframe_into_parquet_bytes(frame)
        out.append((f"m-{int(rng.integers(MODELS)):02d}", {"X": raw, "y": raw}, windows))
    rng.shuffle(out)
    return out


def drive(store, reqs, bucket, threads):
    from gordo_components_b200 import server

    it = iter(range(len(reqs)))
    lock = threading.Lock()
    lat, bodies = [0.0] * len(reqs), [None] * len(reqs)

    def worker():
        while True:
            with lock:
                i = next(it, None)
            if i is None:
                return
            name, files, _ = reqs[i]
            t0 = time.perf_counter()
            r = server.anomaly_prediction(store, name, files=files, fmt="parquet", bucket=bucket)
            lat[i] = time.perf_counter() - t0
            assert r.status == 200, r.body
            bodies[i] = r.body

    ts = [threading.Thread(target=worker) for _ in range(threads)]
    t0 = time.perf_counter()
    [t.start() for t in ts]
    [t.join() for t in ts]
    return time.perf_counter() - t0, np.asarray(lat), bodies


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--overlap-threads", type=int, default=32)
    ap.add_argument("--overlap-wait-ms", type=float, default=5.0)
    ap.add_argument("--ttr", action="store_true", help="serve TransformedTargetRegressor models (ResidentBucket(target_scaler=True))")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import __graft_entry__ as ge

    ge.build()
    from gordo_components_b200 import server

    info = card()
    with tempfile.TemporaryDirectory() as root:
        store = make_store(root, a.ttr)
        bucket = server.ResidentBucket(store, lstm=True, target_scaler=a.ttr)
        overlap_bucket = server.ResidentBucket(store, lstm=True, target_scaler=a.ttr, max_wait_ms=a.overlap_wait_ms)
        assert bucket.target_scaler == a.ttr and len(bucket.names) == MODELS
        co = bucket.coalescer
        formed = []  # (windows per request) of every batch either coalescer launched

        def record(c):
            launch = c._launch

            def recording_launch(torch_, batch, cost):
                formed.append([len(item[2]) for item in batch])
                return launch(torch_, batch, cost)

            c._launch = recording_launch

        record(co)
        record(overlap_bucket.coalescer)
        results = {"card": info, "models": MODELS, "threads": a.threads, "lookback": LOOKBACK, "tags": TAGS,
                   "base_estimator": "TTR(MinMaxScaler, Pipeline([MinMaxScaler, KerasLSTMAutoEncoder]))" if a.ttr else "KerasLSTMAutoEncoder"}
        identical = True
        try:
            for wl, mixed, b_wl, threads in (("uniform", False, bucket, a.threads), ("mixed", True, bucket, a.threads),
                                              ("overlap", False, overlap_bucket, a.overlap_threads)):
                reqs = payloads(a.requests, mixed, 1 if mixed else 0)
                windows = sum(w for _, _, w in reqs)
                drive(store, reqs[:16], None, threads)  # warm-up: modules, allocator pools, the models' device copies
                drive(store, reqs[:16], b_wl, threads)
                arms = {"per_request": [], "coalesced": []}
                replies = {}
                batches0, requests0, formed0 = b_wl.coalescer.batches, b_wl.coalescer.requests, len(formed)
                for _ in range(a.reps):
                    for arm, b in (("per_request", None), ("coalesced", b_wl)):
                        wall, lat, bodies = drive(store, reqs, b, threads)
                        arms[arm].append({"requests_per_s": len(reqs) / wall, "windows_per_s": windows / wall,
                                          "p50_ms": float(np.percentile(lat, 50) * 1e3), "p99_ms": float(np.percentile(lat, 99) * 1e3)})
                        if arm in replies:
                            assert replies[arm] == bodies, f"{arm}: replies changed between repetitions"
                        replies[arm] = bodies
                same = replies["per_request"] == replies["coalesced"]
                identical &= same
                batches = formed[formed0:]
                n_batches, n_requests = b_wl.coalescer.batches - batches0, b_wl.coalescer.requests - requests0
                res = {"requests": len(reqs), "windows": windows, "threads": threads, "max_wait_ms": b_wl.coalescer.max_wait * 1e3,
                       "arms": arms, "replies_identical": same, "batches_formed": n_batches,
                       "requests_per_batch": float(np.mean([len(b) for b in batches])), "batches_per_request": n_batches / max(1, n_requests)}
                if mixed:
                    eng = co.eng
                    ws_u = [eng.tc_workspace_bytes(min(len(b), MODELS), len(b), max(b)) for b in batches]
                    ws_r = [eng.tc_workspace_bytes(min(len(b), MODELS), len(b), max(b), int(eng.tile_base(b)[-1])) for b in batches]
                    big = [i for i, b in enumerate(batches) if max(b) >= 10000]
                    res["workspace_bytes"] = {"uniform_max": max(ws_u), "ragged_max": max(ws_r),
                                              "uniform_of_batches_with_a_long_request": [ws_u[i] for i in big][:4],
                                              "ragged_of_batches_with_a_long_request": [ws_r[i] for i in big][:4]}
                results[wl] = res
            # step launches per batch, in a run of its own (the profiler slows the host)
            reqs = payloads(32, False, 2)
            before = co.batches
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                drive(store, reqs, bucket, a.threads)
                torch.cuda.synchronize()
            steps = sum(e.count for e in prof.key_averages() if "lstm_tc_step_kernel" in e.key)
            results["profile"] = {"batches": co.batches - before, "step_launches": steps,
                                  "step_launches_per_batch": steps / max(1, co.batches - before), "lookback_x_layers": LOOKBACK * 6}
        finally:
            bucket.close()
            overlap_bucket.close()
    results["replies_identical"] = identical
    print(json.dumps(results))
    if not identical:
        sys.exit("the coalesced replies differ from the per-request ones")


if __name__ == "__main__":
    main()
