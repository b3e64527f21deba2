"""
The request path end to end on one GPU: JSON body -> frames -> detector.anomaly_blocks (fused predict + score launch) -> JSON reply,
through server.anomaly_prediction, for models built by builder.FleetModelBuilder -- the shape of gordo's load test
(benchmarks/test_ml_server.py: many small POSTs).  Reports per-request latency (single thread) and requests/s with client threads.

    python benchmarks/bench_requests.py [--machines 20] [--tags 8] [--rows 100] [--requests 500] [--threads 8]

Not measured on the H100.
"""
import argparse, json, os, sys, tempfile, time
from concurrent.futures import ThreadPoolExecutor
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--machines", type=int, default=20)
    ap.add_argument("--tags", type=int, default=8)
    ap.add_argument("--rows", type=int, default=100)
    ap.add_argument("--requests", type=int, default=500)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--bucket", action="store_true", help="serve through server.ResidentBucket (one coalescer for all models)")
    a = ap.parse_args()
    import numpy as np
    import pandas as pd
    import torch
    import __graft_entry__ as ge
    ge.build()
    from gordo_components_b200 import builder, server

    class Dataset:
        def __init__(self, frame):
            self.frame = frame

        def get_data(self):
            return self.frame, self.frame

        def to_dict(self):
            return {"tag_list": list(self.frame.columns), "resolution": "10min"}

    rng = np.random.default_rng(0)
    idx = pd.date_range("2019-01-01", periods=2000, freq="10min", tz="UTC")
    model = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": {
        "gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": 2}}}}
    machines = []
    for m in range(a.machines):
        frame = pd.DataFrame(rng.random((len(idx), a.tags)).astype(np.float32), index=idx, columns=[f"tag-{i}" for i in range(a.tags)])
        machines.append({"name": f"machine-{m}", "model": model, "dataset": Dataset(frame)})
    with tempfile.TemporaryDirectory() as out:
        builder.FleetModelBuilder(machines).build(out)
        store = server.ModelStore(out)
        bucket = server.ResidentBucket(store) if a.bucket else None
        bodies = []
        for m in range(a.machines):
            X = machines[m]["dataset"].frame.iloc[: a.rows].astype(np.float64)
            d = server.dataframe_to_dict(X)
            bodies.append((f"machine-{m}", json.dumps({"X": d, "y": d})))

        def one(i):
            name, body = bodies[i % len(bodies)]
            t0 = time.perf_counter()
            reply = server.anomaly_prediction(store, name, json=json.loads(body), bucket=bucket)
            text = json.dumps(reply.body)
            return time.perf_counter() - t0, reply.status, len(text)

        for i in range(len(bodies)):
            one(i)  # every model loaded, weights on the device
        torch.cuda.synchronize()
        lat = np.array([one(i)[0] for i in range(a.requests)])
        t0 = time.perf_counter()
        with ThreadPoolExecutor(a.threads) as ex:
            res = list(ex.map(one, range(a.requests)))
        wall = time.perf_counter() - t0
        launches = (bucket.coalescer.batches, bucket.coalescer.requests) if bucket else None
        if bucket:
            bucket.close()
    assert all(r[1] == 200 for r in res)
    print(json.dumps({
        "workload": f"{a.requests} JSON anomaly requests x {a.rows} rows x {a.tags} tags over {a.machines} resident models",
        "single_thread_ms": {"p50": float(np.percentile(lat, 50) * 1e3), "p95": float(np.percentile(lat, 95) * 1e3), "mean": float(lat.mean() * 1e3)},
        "threads": a.threads, "requests_per_s": a.requests / wall, "windows_per_s": a.requests * a.rows / wall, "reply_bytes": res[0][2],
        "coalescer_batches_requests": launches,
    }))


if __name__ == "__main__":
    main()
