"""
EarlyStopping inside the LSTM fit launches (gb_lstm_fit_stop / gb_lstm_fit_tc_stop), three measurements in one run:

    python benchmarks/bench_lstm_fit_stop.py [--runs 3] [--builder-machines 16]

(a) what the stop path costs when nothing stops: ms per optimizer step of the _opt entry against the _stop entry with a rule that
    never fires, alternated, at batch 32 (fp32 family) and 128 (tensor-core family);
(b) what a step costs once every job has stopped: every job stops after epoch 1 (patience 1, a min_delta only the first epoch
    beats); a launch of 20 epochs against a plain launch of 2, the difference over the skipped steps, against a live step;
(c) the builder end to end: LSTM machines with EarlyStopping(loss, patience=2) on the ``bench_fleet_builder.py --lstm`` shape,
    FleetModelBuilder(lstm_early_stopping=True) per machine against ModelBuilder.
(a) and (b) use the configs[3] share: 8 machines x 128 tags, lstm_symmetric (256, 128, 64), lookback 144, 257 windows.  Prints one
JSON line with the card's name and power limit.
"""
import argparse, json, math, os, sys, time
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

from bench_fleet_builder import _power_limit  # noqa: E402

MACHINES, TAGS, UNITS, LOOKBACK, WINDOWS = 8, 128, [256, 128, 64, 64, 128, 256], 144, 257


def _share(torch, engine):
    eng = engine.LSTMEngine(TAGS, UNITS, ["tanh"] * len(UNITS), TAGS, "linear", LOOKBACK)
    rows = WINDOWS + LOOKBACK - 1
    g = torch.Generator(device=eng.device).manual_seed(0)
    x = torch.rand((MACHINES * rows, TAGS), generator=g, device=eng.device)
    jobs = engine.jobs_to_device(engine.make_jobs(range(MACHINES), [WINDOWS] * MACHINES, [m * rows for m in range(MACHINES)]), eng.device)
    return eng, eng.initial_params(MACHINES, g), jobs, x


def _timed(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def _launches(torch, engine, runs):
    eng, params, jobs, x = _share(torch, engine)
    never = engine.make_stop([{"monitor": "loss", "patience": 10 ** 6}] * MACHINES)
    # every job stops after epoch 1: only epoch 0 (against +inf) beats a min_delta of 1e9
    stops = engine.make_stop([{"monitor": "loss", "patience": 1, "min_delta": 1e9}] * MACHINES)

    def plain(B, epochs):
        return lambda: eng.fit_for_batch(B)(params.clone(), jobs, MACHINES, WINDOWS, x, x, epochs=epochs, batch_size=B)

    def stop(B, epochs, rule):
        return lambda: eng.fit_stop(params.clone(), jobs, MACHINES, WINDOWS, x, x, rule, epochs=epochs, batch_size=B)

    out = {}
    for B in (32, 128):
        steps = 1 + math.ceil(WINDOWS / B)  # primer + one epoch
        plain(B, 1)(), stop(B, 1, never)()  # warm-up
        a = {"opt": [], "stop": []}
        for _ in range(runs):
            a["opt"].append(1e3 * _timed(torch, plain(B, 1)) / steps)
            a["stop"].append(1e3 * _timed(torch, stop(B, 1, never)) / steps)
        out[f"a_b{B}_ms_per_step_opt"] = a["opt"]
        out[f"a_b{B}_ms_per_step_stop_never_fires"] = a["stop"]
    B = 32
    per_epoch = math.ceil(WINDOWS / B)
    skipped = (20 - 2) * per_epoch
    t_plain = [_timed(torch, plain(B, 2)) for _ in range(2)]
    t_stop = [_timed(torch, stop(B, 20, stops)) for _ in range(2)]
    live = min(t_plain) / (1 + 2 * per_epoch)
    per_skipped = (min(t_stop) - min(t_plain)) / skipped
    out.update({"b_b32_plain_2_epochs_s": t_plain, "b_b32_stop_20_epochs_all_stop_after_1_s": t_stop, "b_skipped_steps": skipped,
                "b_us_per_skipped_step": 1e6 * per_skipped, "b_live_step_ms": 1e3 * live, "b_skipped_over_live": per_skipped / live})
    return out


def _builder(torch, machines, rows, tags, epochs, single):
    import numpy as np
    import pandas as pd

    from gordo_components_b200 import builder

    ae = {"gordo.machine.model.models.KerasLSTMAutoEncoder": {
        "kind": "lstm_hourglass", "lookback_window": 24, "epochs": epochs,
        "callbacks": [{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "loss", "patience": 2}}]}}
    model = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": ae}}
    rng = np.random.default_rng(0)
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    t = np.linspace(0, 60, rows)[:, None]
    ms = []
    for m in range(machines):
        values = 0.5 + 0.4 * np.sin(t * rng.uniform(0.5, 2, tags) + rng.uniform(0, 6, tags)) + rng.normal(0, 0.02, (rows, tags))
        frame = pd.DataFrame(values.astype(np.float32), index=idx, columns=[f"tag-{i}" for i in range(tags)])
        ms.append({"name": f"machine-{m}", "model": model, "dataset": {"X": frame, "y": frame}})
    builder.FleetModelBuilder(ms[:2], lstm_early_stopping=True).build()  # warm-up
    fleet_s = _timed(torch, lambda: builder.FleetModelBuilder(ms, lstm_early_stopping=True).build())
    results = builder.FleetModelBuilder(ms[:single], lstm_early_stopping=True).build()
    ran = [len(r.base_estimator._history.epoch) for r, _ in results]
    single_s = _timed(torch, lambda: [builder.ModelBuilder(m).build() for m in ms[:single]]) / single
    return {"c_workload": f"{machines} machines x {tags}-tag LSTM hourglass (lookback 24), {rows} rows, {epochs} epochs, "
                          "EarlyStopping(loss, patience=2): 3-fold CV + fit + thresholds + scores",
            "c_fleet_builder_s_per_machine": fleet_s / machines, "c_model_builder_s_per_machine": single_s,
            "c_speedup_per_machine": single_s / (fleet_s / machines), "c_final_fit_epochs_run": ran}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3, help="(a): alternated timed launches of each entry point")
    ap.add_argument("--builder-machines", type=int, default=16)
    ap.add_argument("--builder-rows", type=int, default=2000)
    ap.add_argument("--builder-tags", type=int, default=16)
    ap.add_argument("--builder-epochs", type=int, default=20)
    ap.add_argument("--builder-single", type=int, default=4)
    a = ap.parse_args()
    import torch

    import __graft_entry__ as ge
    ge.build()
    from gordo_components_b200 import engine

    out = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": _power_limit(),
           "share": f"{MACHINES} machines x {TAGS} tags, lstm_symmetric (256, 128, 64), lookback {LOOKBACK}, {WINDOWS} windows"}
    out.update(_launches(torch, engine, a.runs))
    out.update(_builder(torch, a.builder_machines, a.builder_rows, a.builder_tags, a.builder_epochs, a.builder_single))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
