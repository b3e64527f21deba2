"""
`gordo build` for a project from CONFIGURATION: machines as `Machine.to_dict()`-style dicts (model definition + dataset +
evaluation) through builder.FleetModelBuilder -- definitions resolved, machines bucketed, every bucket built in five
launches, detectors materialised, `model.pkl` + `metadata.json` written -- against builder.ModelBuilder (the same machines
one at a time, gordo/builder/build_model.py:192-339 on the GPU estimators).  Wall clock, host work included: this is the
number a `gordo build` user sees.

    python benchmarks/bench_fleet_builder.py [--machines 125] [--rows 10000] [--tags 64] [--epochs 10] [--scaled] [--single 3]

Not measured on the H100; the code paths it times are covered by tests/test_gpu_builder.py.
"""
import argparse, json, os, sys, tempfile, time
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--machines", type=int, default=125)
    ap.add_argument("--rows", type=int, default=10000)
    ap.add_argument("--tags", type=int, default=64)
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--scaled", action="store_true", help="Pipeline([MinMaxScaler, AE]) as in gordo's example config")
    ap.add_argument("--single", type=int, default=3, help="machines to also build one at a time for comparison")
    a = ap.parse_args()
    import numpy as np
    import pandas as pd
    import torch
    import __graft_entry__ as ge
    ge.build()
    from gordo_components_b200 import builder

    ae = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": a.epochs}}
    base = {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", ae]}} if a.scaled else ae
    model = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": base}}
    rng = np.random.default_rng(0)
    idx = pd.date_range("2019-01-01", periods=a.rows, freq="10min", tz="UTC")
    t = np.linspace(0, 60, a.rows)[:, None]
    machines = []
    for m in range(a.machines):
        values = 0.5 + 0.4 * np.sin(t * rng.uniform(0.5, 2, a.tags) + rng.uniform(0, 6, a.tags)) + rng.normal(0, 0.02, (a.rows, a.tags))
        frame = pd.DataFrame(values.astype(np.float32), index=idx, columns=[f"tag-{i}" for i in range(a.tags)])
        machines.append({"name": f"machine-{m}", "model": model, "dataset": {"X": frame, "y": frame}})

    builder.FleetModelBuilder(machines[:2]).build()  # warm-up: library load, first launches
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as out:
        t0 = time.perf_counter()
        results = builder.FleetModelBuilder(machines).build(out)
        torch.cuda.synchronize()
        fleet_s = time.perf_counter() - t0
        size = sum(os.path.getsize(os.path.join(out, m["name"], f)) for _, m in results for f in ("model.pkl", "metadata.json"))
    single_s = None
    if a.single:
        t0 = time.perf_counter()
        for m in machines[: a.single]:
            builder.ModelBuilder(m).build()
        torch.cuda.synchronize()
        single_s = (time.perf_counter() - t0) / a.single
    scores = results[0][1]["metadata"]["build_metadata"]["model"]["cross_validation"]["scores"]
    print(json.dumps({
        "workload": f"{a.machines} machines x {a.tags}-tag hourglass{' behind MinMaxScaler' if a.scaled else ''}, {a.rows} rows, {a.epochs} epochs: "
                    "definition -> 3-fold CV + fit + thresholds + scores metadata -> model.pkl/metadata.json",
        "fleet_builder_s": fleet_s, "machines_per_s": a.machines / fleet_s, "bytes_written": size,
        "model_builder_s_per_machine": single_s, "speedup_per_machine": None if single_s is None else single_s / (fleet_s / a.machines),
        "r2_fold_mean_machine_0": scores["r2-score"]["fold-mean"],
    }))


if __name__ == "__main__":
    main()
