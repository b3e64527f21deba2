"""
`gordo build` for a project from CONFIGURATION: machines as `Machine.to_dict()`-style dicts (model definition + dataset +
evaluation) through builder.FleetModelBuilder -- definitions resolved, machines bucketed, every bucket built in five
launches, detectors materialised, `model.pkl` + `metadata.json` written -- against builder.ModelBuilder (the same machines
one at a time, gordo/builder/build_model.py:192-339 on the GPU estimators).  Wall clock, host work included: this is the
number a `gordo build` user sees.

    python benchmarks/bench_fleet_builder.py [--machines 125] [--rows 10000] [--tags 64] [--epochs 10] [--scaled] [--single 3]
    python benchmarks/bench_fleet_builder.py --lstm [--lookback 24] --machines 16 --rows 2000 --tags 16 --epochs 1 --single 16
    python benchmarks/bench_fleet_builder.py --example-config --machines 125 --rows 10000 --tags 64 --epochs 10 --single 3

``--lstm`` builds DiffBasedAnomalyDetector(KerasLSTMAutoEncoder(lstm_hourglass)) machines instead (batched by
fleet.build_lstm_fleet).  ``--example-config`` builds the model of gordo's examples/model-configuration.yaml:
DiffBasedAnomalyDetector(shuffle=True) around Pipeline([MinMaxScaler, KerasAutoEncoder(feedforward_hourglass, compression_factor
0.6, 1 encoding layer, batch 128, validation_split 0.1)]) under TimeSeriesSplit(5).  Measured numbers and the card they were measured on are in DESIGN.md §7.
"""
import argparse, json, os, sys, tempfile, time
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))


def _power_limit():
    """The card's power limit in watts, read-only query (None when nvidia-smi is not available)."""
    import subprocess

    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--machines", type=int, default=125)
    ap.add_argument("--rows", type=int, default=10000)
    ap.add_argument("--tags", type=int, default=64)
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--scaled", action="store_true", help="Pipeline([MinMaxScaler, AE]) as in gordo's example config")
    ap.add_argument("--single", type=int, default=3, help="machines to also build one at a time for comparison")
    ap.add_argument("--lstm", action="store_true", help="LSTM autoencoder machines (lstm_hourglass) instead of the feed-forward hourglass")
    ap.add_argument("--lookback", type=int, default=24, help="lookback_window of the LSTM machines")
    ap.add_argument("--example-config", action="store_true", help="the model and evaluation of gordo's examples/model-configuration.yaml")
    a = ap.parse_args()
    import numpy as np
    import pandas as pd
    import torch
    import __graft_entry__ as ge
    ge.build()
    from gordo_components_b200 import builder

    if a.lstm:
        ae = {"gordo.machine.model.models.KerasLSTMAutoEncoder": {"kind": "lstm_hourglass", "lookback_window": a.lookback, "epochs": a.epochs}}
    else:
        ae = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "epochs": a.epochs}}
    base = {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", ae]}} if a.scaled else ae
    model = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": base}}
    evaluation, n_splits = {}, 3
    if a.example_config:
        ae = {"gordo.machine.model.models.KerasAutoEncoder": {
            "batch_size": 128, "compression_factor": 0.6, "encoding_layers": 1, "epochs": a.epochs, "func": "tanh", "kind": "feedforward_hourglass",
            "loss": "mse", "optimizer": "Adam", "out_func": "linear", "validation_split": 0.1}}
        model = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {
            "base_estimator": {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", ae]}},
            "scaler": "sklearn.preprocessing.MinMaxScaler", "shuffle": True, "smoothing_method": "smm"}}
        evaluation, n_splits = {"cv": {"sklearn.model_selection.TimeSeriesSplit": {"n_splits": 5}}}, 5
    rng = np.random.default_rng(0)
    idx = pd.date_range("2019-01-01", periods=a.rows, freq="10min", tz="UTC")
    t = np.linspace(0, 60, a.rows)[:, None]
    machines = []
    for m in range(a.machines):
        values = 0.5 + 0.4 * np.sin(t * rng.uniform(0.5, 2, a.tags) + rng.uniform(0, 6, a.tags)) + rng.normal(0, 0.02, (a.rows, a.tags))
        frame = pd.DataFrame(values.astype(np.float32), index=idx, columns=[f"tag-{i}" for i in range(a.tags)])
        machines.append({"name": f"machine-{m}", "model": model, "dataset": {"X": frame, "y": frame}, "evaluation": evaluation})

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
    net = f"LSTM hourglass (lookback {a.lookback})" if a.lstm else "hourglass"
    if a.example_config:
        net = "hourglass (compression 0.6, 1 encoding layer, batch 128, validation_split 0.1) in a shuffling detector"
    print(json.dumps({
        "gpu": torch.cuda.get_device_name(0), "power_limit_w": _power_limit(),
        "workload": f"{a.machines} machines x {a.tags}-tag {net}{' behind MinMaxScaler' if a.scaled or a.example_config else ''}, {a.rows} rows, {a.epochs} epochs: "
                    f"definition -> {n_splits}-fold CV + fit + thresholds + scores metadata -> model.pkl/metadata.json",
        "fleet_builder_s": fleet_s, "machines_per_s": a.machines / fleet_s, "bytes_written": size,
        "model_builder_s_per_machine": single_s, "speedup_per_machine": None if single_s is None else single_s / (fleet_s / a.machines),
        "r2_fold_mean_machine_0": scores["r2-score"]["fold-mean"],
    }))


if __name__ == "__main__":
    main()
