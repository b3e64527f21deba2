"""
`gordo build` for a project from CONFIGURATION: machines as `Machine.to_dict()`-style dicts (model definition + dataset +
evaluation) through builder.FleetModelBuilder -- definitions resolved, machines bucketed, every bucket built in five
launches, detectors materialised, `model.pkl` + `metadata.json` written -- against builder.ModelBuilder (the same machines
one at a time, gordo/builder/build_model.py:192-339 on the GPU estimators).  Wall clock, host work included: this is the
number a `gordo build` user sees.

    python benchmarks/bench_fleet_builder.py [--machines 125] [--rows 10000] [--tags 64] [--epochs 10] [--scaled] [--single 3]
    python benchmarks/bench_fleet_builder.py --lstm [--lookback 24] --machines 16 --rows 2000 --tags 16 --epochs 1 --single 16
    python benchmarks/bench_fleet_builder.py --example-config --machines 125 --rows 10000 --tags 64 --epochs 10 --single 3
    python benchmarks/bench_fleet_builder.py --early-stopping --machines 125 --rows 10000 --tags 64 --epochs 100 --single 1
    python benchmarks/bench_fleet_builder.py --kfcv --machines 125 --rows 10000 --tags 64 --epochs 20 --single 1
    python benchmarks/bench_fleet_builder.py --ragged 5000:15000 --machines 125 --tags 64 --epochs 10 --single 1 [--kfcv | --lstm | --example-config]
    python benchmarks/bench_fleet_builder.py --ttr --scaled --machines 125 --rows 10000 --tags 64 --epochs 10 --single 1 [--lstm]
    python benchmarks/bench_fleet_builder.py --tags 8:96 --machines 125 --rows 10000 --epochs 10 --runs 3 --single 0 [--kfcv]

``--lstm`` builds DiffBasedAnomalyDetector(KerasLSTMAutoEncoder(lstm_hourglass)) machines instead (batched by
fleet.build_lstm_fleet).  ``--example-config`` builds the model of gordo's examples/model-configuration.yaml:
DiffBasedAnomalyDetector(shuffle=True) around Pipeline([MinMaxScaler, KerasAutoEncoder(feedforward_hourglass, compression_factor
0.6, 1 encoding layer, batch 128, validation_split 0.1)]) under TimeSeriesSplit(5).  ``--early-stopping`` adds the callback of
the reference's production definition to that model, EarlyStopping(monitor=val_loss, patience=10, restore_best_weights=True), and
also reports the epochs each fit ran (min / median / max over all final and CV-fold fits) and the time of the bucket's fit
launch with the rule against the same launch with patience = epochs (never stops), alternating, CUDA events around the launch
after a warm-up.  ``--kfcv`` builds the reference's production definition: DiffBasedKFCVAnomalyDetector(window 144, shuffle,
threshold_percentile 0.975) around TransformedTargetRegressor(MinMaxScaler, Pipeline([MinMaxScaler, KerasAutoEncoder(feedforward_hourglass,
compression_factor 0.5, 1 encoding layer, batch 128, validation_split 0.1, EarlyStopping(val_loss, patience 10, restore_best_weights))]))
under KFold(5, shuffle=True, random_state=0), with FleetModelBuilder(early_stopping=True, kfcv=True); it also reports the device
time of the K-fold threshold stage (errors back to time order, smoothing, percentile, metric moments: the launches
fleet.build_kfold_fleet makes after the fold scoring, on arrays of the bucket's shape), CUDA events, after a warm-up.
``--ragged LO:HI`` draws every machine's length uniformly from [LO, HI] (seeded) and builds the project with
FleetModelBuilder(ragged=True) and with the default, alternating, ``--runs`` times each: wall time, the number of buckets and of
fit launches, and the device time of the fit launches (CUDA events around each, summed per build).  Without the flag every
length is its own bucket.
``--tags LO:HI`` draws every machine's tag count uniformly from [LO, HI] (seeded) and builds the project with
FleetModelBuilder(mixed_widths=True) and with the default, alternating, ``--runs`` times each, reporting as ``--ragged`` does
(grouped fit launches counted and timed as one launch each).  Without the flag every tag count is its own bucket and its own fit
launch; with it, the buckets whose nets share a memory plan train in one gb_ffae_fit_group launch.
``--window W`` gives the plain detectors a smoothing window W (smm) and builds them with FleetModelBuilder(smoothing=True), whose
fold thresholds at 6 rows and at W come from one gb_thresholds_pair launch.
``--ttr`` wraps the plain detector's estimator (feed-forward, ``--scaled`` or ``--lstm``) in TransformedTargetRegressor(transformer=
MinMaxScaler()), the reference's production base estimator under the default TimeSeriesSplit(3), and builds it with
FleetModelBuilder(target_scaler=True).
Measured numbers and the card they were measured on are in DESIGN.md §5b and §7.
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
    ap.add_argument("--tags", default="64", metavar="T|LO:HI", help="tags per machine, or LO:HI: per-machine tag counts drawn uniformly "
                    "from [LO, HI]; FleetModelBuilder(mixed_widths=True) against the default")
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--scaled", action="store_true", help="Pipeline([MinMaxScaler, AE]) as in gordo's example config")
    ap.add_argument("--single", type=int, default=3, help="machines to also build one at a time for comparison")
    ap.add_argument("--lstm", action="store_true", help="LSTM autoencoder machines (lstm_hourglass) instead of the feed-forward hourglass")
    ap.add_argument("--lookback", type=int, default=24, help="lookback_window of the LSTM machines")
    ap.add_argument("--example-config", action="store_true", help="the model and evaluation of gordo's examples/model-configuration.yaml")
    ap.add_argument("--early-stopping", action="store_true", help="--example-config with EarlyStopping(val_loss, patience=10, restore_best_weights)")
    ap.add_argument("--launch-runs", type=int, default=3, help="--early-stopping: timed fit launches of each kind")
    ap.add_argument("--min-delta", type=float, default=0.0, help="--early-stopping: the callback's min_delta (the reference's definition has none)")
    ap.add_argument("--kfcv", action="store_true", help="the reference's production definition: a K-fold detector under KFold(5, shuffle, random_state=0)")
    ap.add_argument("--ragged", default=None, metavar="LO:HI", help="per-machine lengths drawn uniformly from [LO, HI]; ragged=True against the default")
    ap.add_argument("--runs", type=int, default=2, help="--ragged / --tags LO:HI: builds of each kind, alternating")
    ap.add_argument("--window", type=int, default=None, help="plain detectors with this smoothing window (smm), batched by FleetModelBuilder(smoothing=True)")
    ap.add_argument("--ttr", action="store_true", help="the plain detector's estimator inside TransformedTargetRegressor(MinMaxScaler), "
                                                        "batched by FleetModelBuilder(target_scaler=True)")
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
    stopping = {"monitor": "val_loss", "patience": 10, "restore_best_weights": True, "min_delta": a.min_delta}
    if a.example_config or a.early_stopping:
        ae = {"gordo.machine.model.models.KerasAutoEncoder": {
            "batch_size": 128, "compression_factor": 0.6, "encoding_layers": 1, "epochs": a.epochs, "func": "tanh", "kind": "feedforward_hourglass",
            "loss": "mse", "optimizer": "Adam", "out_func": "linear", "validation_split": 0.1}}
        if a.early_stopping:
            ae["gordo.machine.model.models.KerasAutoEncoder"]["callbacks"] = [{"tensorflow.keras.callbacks.EarlyStopping": stopping}]
        model = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {
            "base_estimator": {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", ae]}},
            "scaler": "sklearn.preprocessing.MinMaxScaler", "shuffle": True, "smoothing_method": "smm"}}
        evaluation, n_splits = {"cv": {"sklearn.model_selection.TimeSeriesSplit": {"n_splits": 5}}}, 5
    if a.kfcv:
        ae = {"gordo.machine.model.models.KerasAutoEncoder": {
            "kind": "feedforward_hourglass", "batch_size": 128, "compression_factor": 0.5, "encoding_layers": 1, "func": "tanh", "out_func": "linear",
            "epochs": a.epochs, "validation_split": 0.1, "callbacks": [{"tensorflow.keras.callbacks.EarlyStopping": stopping}]}}
        model = {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {
            "base_estimator": {"sklearn.compose.TransformedTargetRegressor": {
                "transformer": "sklearn.preprocessing.MinMaxScaler",
                "regressor": {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", ae]}}}},
            "scaler": "sklearn.preprocessing.MinMaxScaler", "window": 144, "shuffle": True, "threshold_percentile": 0.975}}
        evaluation, n_splits = {"cv": {"sklearn.model_selection.KFold": {"n_splits": 5, "shuffle": True, "random_state": 0}}}, 5
    flags = dict(early_stopping=a.early_stopping or a.kfcv, kfcv=a.kfcv)
    if a.window is not None and not a.kfcv:
        next(iter(model.values())).update({"window": a.window, "smoothing_method": "smm"})
        flags["smoothing"] = True
    if a.ttr and not a.kfcv:
        detector = next(iter(model.values()))
        detector["base_estimator"] = {"sklearn.compose.TransformedTargetRegressor": {
            "transformer": "sklearn.preprocessing.MinMaxScaler", "regressor": detector["base_estimator"]}}
        flags["target_scaler"] = True
    rng = np.random.default_rng(0)
    lo, _, hi = a.tags.partition(":")
    tag_counts = np.random.default_rng(2).integers(int(lo), int(hi) + 1, size=a.machines) if hi else np.full(a.machines, int(lo))
    if a.ragged:
        lo, hi = (int(v) for v in a.ragged.split(":"))
        lengths = np.random.default_rng(1).integers(lo, hi + 1, size=a.machines)
    else:
        lengths = np.full(a.machines, a.rows)
    machines = []
    for m in range(a.machines):
        rows, tags = int(lengths[m]), int(tag_counts[m])
        idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
        t = np.linspace(0, 60 * rows / a.rows, rows)[:, None]
        values = 0.5 + 0.4 * np.sin(t * rng.uniform(0.5, 2, tags) + rng.uniform(0, 6, tags)) + rng.normal(0, 0.02, (rows, tags))
        frame = pd.DataFrame(values.astype(np.float32), index=idx, columns=[f"tag-{i}" for i in range(tags)])
        machines.append({"name": f"machine-{m}", "model": model, "dataset": {"X": frame, "y": frame}, "evaluation": evaluation})
    if hi:
        if a.ragged:
            flags["ragged"] = True
        print(json.dumps(_alternating_builds(a, machines, flags, n_splits, lengths, "mixed_widths", tag_counts)))
        return
    if a.ragged:
        print(json.dumps(_alternating_builds(a, machines, flags, n_splits, lengths, "ragged")))
        return

    builder.FleetModelBuilder(machines[:2], **flags).build()  # warm-up: library load, first launches
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as out:
        t0 = time.perf_counter()
        results = builder.FleetModelBuilder(machines, **flags).build(out)
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
    if a.example_config or a.early_stopping:
        net = "hourglass (compression 0.6, 1 encoding layer, batch 128, validation_split 0.1) in a shuffling detector"
    if a.kfcv:
        net = ("K-fold detector (window 144, percentile 0.975) around TransformedTargetRegressor(MinMaxScaler) of a hourglass (compression 0.5, "
               "1 encoding layer, batch 128, validation_split 0.1), KFold(5, shuffle, random_state=0)")
    if a.window is not None and not a.kfcv:
        net += f", smoothing window {a.window}"
    if a.ttr and not a.kfcv:
        net = f"TransformedTargetRegressor(MinMaxScaler) of a {net}"
    if a.early_stopping or a.kfcv:
        net += f", EarlyStopping(val_loss, patience 10, min_delta {a.min_delta:g}, restore_best_weights)"
    out = {
        "gpu": torch.cuda.get_device_name(0), "power_limit_w": _power_limit(),
        "workload": f"{a.machines} machines x {a.tags}-tag {net}{' behind MinMaxScaler' if a.scaled or a.example_config or a.early_stopping else ''}, "
                    f"{a.rows} rows, {a.epochs} epochs: definition -> {n_splits}-fold CV + fit + thresholds + scores metadata -> model.pkl/metadata.json",
        "fleet_builder_s": fleet_s, "machines_per_s": a.machines / fleet_s, "bytes_written": size,
        "model_builder_s_per_machine": single_s, "speedup_per_machine": None if single_s is None else single_s / (fleet_s / a.machines),
        "r2_fold_mean_machine_0": scores["r2-score"]["fold-mean"],
    }
    if a.early_stopping:
        out.update(_stop_launches(a, machines, stopping))
    if a.kfcv:
        ran = np.asarray([len(r.base_estimator.regressor_.steps[-1][1]._history.epoch) for r, _ in results])
        out.update({"final_fit_epochs_run_min": int(ran.min()), "final_fit_epochs_run_median": float(np.median(ran)), "final_fit_epochs_run_max": int(ran.max())})
        out.update(_kfold_threshold_stage(a))
    print(json.dumps(out))


def _alternating_builds(a, machines, flags, n_splits, lengths, option, tag_counts=None):
    """
    The project built with FleetModelBuilder(**{option: True}) (``ragged`` or ``mixed_widths``) and with the default, alternating:
    wall time of each build (host work and the written files included), buckets, and the fit launches' device time (CUDA events
    around every fit launch of the build, per-net and grouped, read after the build's final synchronise).  One warm-up of each kind
    first.
    """
    import numpy as np
    import torch

    from gordo_components_b200 import builder, engine

    launches, buckets = [], []

    def timed(fn):
        def run(*args, **kw):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            res = fn(*args, **kw)
            ev[1].record()
            launches.append(ev)
            return res
        return run

    def counted(fn, joined=False):
        def run(members):
            buckets.extend(members if joined else [members])
            return fn(members)
        return run

    engine.FFEngine._fit_launch = timed(engine.FFEngine._fit_launch)
    engine.LSTMEngine._fit_launch = timed(engine.LSTMEngine._fit_launch)
    engine.fit_group = timed(engine.fit_group)
    builder.FleetModelBuilder._build_bucket = staticmethod(counted(builder.FleetModelBuilder._build_bucket))
    builder.FleetModelBuilder._build_buckets_joined = staticmethod(counted(builder.FleetModelBuilder._build_buckets_joined, joined=True))

    def build(flagged, project):
        launches.clear()
        buckets.clear()
        with tempfile.TemporaryDirectory() as out:
            t0 = time.perf_counter()
            builder.FleetModelBuilder(project, **{option: flagged}, **flags).build(out)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
        return {"wall_s": wall, "buckets": len(buckets), "fit_launches": len(launches),
                "fit_launch_ms": sum(e[0].elapsed_time(e[1]) for e in launches)}

    name = "ragged" if option == "ragged" else "mixed"
    build(True, machines[:2]), build(False, machines[:2])  # warm-up
    runs = {name: [], "default": []}
    for _ in range(a.runs):
        runs[name].append(build(True, machines))
        runs["default"].append(build(False, machines))
    single_s = None
    if a.single:
        t0 = time.perf_counter()
        for m in machines[: a.single]:
            builder.ModelBuilder(m).build()
        torch.cuda.synchronize()
        single_s = (time.perf_counter() - t0) / a.single
    kind = "K-fold detector (--kfcv)" if a.kfcv else ("LSTM hourglass" if a.lstm else ("example-config hourglass" if a.example_config else "hourglass"))
    tags = f"{a.tags}-tag" if tag_counts is None else f"[{a.tags}]-tag (uniform, seed 2; {len(set(tag_counts.tolist()))} distinct)"
    rows = f"lengths uniform in [{a.ragged}] (seed 1; total {int(lengths.sum())} rows)" if a.ragged else f"{a.rows} rows"
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": _power_limit(),
           "workload": f"{a.machines} machines x {tags} {kind}, {rows}, {a.epochs} epochs, {n_splits}-fold CV, written to disk",
           "model_builder_s_per_machine": single_s}
    for kind, rs in runs.items():
        out[kind] = {key: [r[key] for r in rs] for key in rs[0]}
    out["wall_speedup_median"] = float(np.median(out["default"]["wall_s"]) / np.median(out[name]["wall_s"]))
    out["fit_launch_speedup_median"] = float(np.median(out["default"]["fit_launch_ms"]) / np.median(out[name]["fit_launch_ms"]))
    return out


def _kfold_threshold_stage(a, runs: int = 5):
    """
    Device time of the K-fold threshold stage of fleet.build_kfold_fleet for this bucket's shape, the same launches in the same
    order: the float64 fold errors (per tag and aggregate) back to time order as float32, rolling median over 144 rows, the 0.975
    quantile, and the metric moments of the K*M test blocks.  CUDA events around the stage, after one warm-up.
    """
    import numpy as np
    import torch
    from sklearn.model_selection import KFold

    from gordo_components_b200 import engine, fleet

    dev = engine.cuda_device()
    M, N, T = a.machines, a.rows, int(a.tags)
    tests, _, _, inverse = fleet.kfold_layout(KFold(5, shuffle=True, random_state=0), N)
    K = len(tests)
    n_test = np.asarray([len(t) for t in tests])
    o = np.concatenate([[0], np.cumsum(n_test)[:-1]])
    g = torch.Generator(device=dev).manual_seed(0)
    tag_err = torch.rand((M * N, T), dtype=torch.float64, device=dev, generator=g)
    tot_err = torch.rand((M * N,), dtype=torch.float64, device=dev, generator=g)
    pred = torch.rand((M * N, T), dtype=torch.float32, device=dev, generator=g)
    y32 = torch.rand((M * N, T), dtype=torch.float32, device=dev, generator=g)
    whole = engine.jobs_to_device(engine.make_jobs(np.arange(M), N, np.arange(M) * N), dev)
    fk, fm = np.repeat(np.arange(K), M), np.tile(np.arange(M), K)
    blocks = engine.jobs_to_device(engine.make_jobs(M + np.arange(K * M), n_test[fk], fm * N + o[fk]), dev)
    to_time = torch.from_numpy(inverse.astype(np.int32)).to(dev)

    def stage():
        tag_t = engine.gather_rows(whole, M, N, to_time, tag_err, M * N, to_f32=True)
        tot_t = engine.gather_rows(whole, M, N, to_time, tot_err, M * N, to_f32=True)
        tag_t = engine.smooth(whole, M, tag_t, 144, "smm", max_rows=N)
        tot_t = engine.smooth(whole, M, tot_t, 144, "smm", max_rows=N)
        engine.quantile(whole, M, N, tag_t, 0.975)
        engine.quantile(whole, M, N, tot_t, 0.975)
        engine.cv_moments(blocks, K * M, pred, y32, T)

    stage()
    ms = []
    for _ in range(runs):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        stage()
        ev[1].record()
        torch.cuda.synchronize()
        ms.append(ev[0].elapsed_time(ev[1]))
    return {"threshold_stage_ms": ms}


def _stop_launches(a, machines, stopping):
    """
    The bucket's fit launch (build_fleet as FleetModelBuilder calls it) with the EarlyStopping rule, against the same launch with
    patience = epochs, which never stops: CUDA events around the fit launch alone, alternating, after one warm-up of each.
    """
    import numpy as np
    import torch

    from gordo_components_b200 import engine, fleet
    from gordo_components_b200.machine.model.models import EarlyStopping
    from gordo_components_b200.machine.model.factories.feedforward_autoencoder import feedforward_hourglass

    class TimedEngine:  # the engine, with CUDA events around its fit launch
        def __init__(self, eng):
            self.eng, self.ms = eng, None

        def __getattr__(self, name):
            return getattr(self.eng, name)

        def fit_split(self, *args, **kw):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            res = self.eng.fit_split(*args, **kw)
            ev[1].record()
            torch.cuda.synchronize()
            self.ms = ev[0].elapsed_time(ev[1])
            return res

    spec = feedforward_hourglass(n_features=int(a.tags), compression_factor=0.6, encoding_layers=1, func="tanh", out_func="linear")
    eng = TimedEngine(engine.ff_engine_for(spec))
    x = engine.to_device_f32(np.concatenate([m["dataset"]["X"].values for m in machines]), eng.device)
    never = dict(stopping, patience=a.epochs)

    def launch(rule):
        fb = fleet.build_fleet(eng, x, x, a.rows, epochs=a.epochs, batch_size=128, n_splits=5, adam=spec.adam, input_scaler=True,
                               detector_shuffle=True, validation_split=0.1, early_stopping=EarlyStopping(**rule))
        return eng.ms, fb

    launch(stopping), launch(never)  # warm-up
    rule_ms, never_ms = [], []
    for _ in range(a.launch_runs):
        ms, fb = launch(stopping)
        rule_ms.append(ms)
        never_ms.append(launch(never)[0])
    ran = torch.cat([fb.epochs_run.flatten(), fb.fold_epochs_run.flatten()]).cpu().numpy()
    return {"epochs_run_min": int(ran.min()), "epochs_run_median": float(np.median(ran)), "epochs_run_max": int(ran.max()),
            "fit_slots": int(ran.size), "fit_launch_ms_with_rule": rule_ms, "fit_launch_ms_never_stopping": never_ms}


if __name__ == "__main__":
    main()
