"""
BASELINE configs[2] (scaled): batched training of 64-tag feedforward_hourglass autoencoders, one persistent CTA per machine.
Reports row-epochs/s, microseconds per optimizer step and the CPU oracle (NumPy Keras-style loop) on a small sample.

    python benchmarks/bench_fit.py [--machines 296] [--rows 10000] [--epochs 3] [--batch 32] [--loss mse] [--optimizer Nadam]
                                   [--dropout 0.2 [--repeats 3]]

With --dropout RATE, Keras Dropout(RATE) on every hidden boundary but the output of the encoder's activity-regularized first
layer (dropout after an activity L1 is not supported): the same fit is
timed with and without dropout, alternating the two --repeats times in the one process, and the result carries both timings
(the GPU's name and power limit beside them).
"""
import argparse, json, os, sys, time
import numpy as np
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--machines", type=int, default=296)
    ap.add_argument("--rows", type=int, default=10000)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--tags", type=int, default=64)
    ap.add_argument("--cpu", type=int, default=1)
    ap.add_argument("--loss", default="mse", help="training loss (a canonical name: mse, mae, mape, msle, huber, log_cosh)")
    ap.add_argument("--optimizer", default=None, help="a Keras optimizer name (RMSprop, Adagrad, Adadelta, Adamax, Nadam, AdamW, Adam) "
                    "with its default hyperparameters; without it, Adam through the Adam kernels")
    ap.add_argument("--dropout", type=float, default=None, help="time the fit with Dropout(RATE) on the hidden boundaries against the same "
                    "fit without it, alternating")
    ap.add_argument("--repeats", type=int, default=3, help="with --dropout: timed rounds of each variant")
    a = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    from gordo_components_b200 import engine, fleet
    from oracle import keras_math as km

    from gordo_components_b200.machine.model.factories.specs import resolve_optimizer

    opt = None if a.optimizer is None else resolve_optimizer(a.optimizer, {})
    spec = km.ff_hourglass_spec(a.tags)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    M, N, E, B = a.machines, a.rows, a.epochs, a.batch
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.rand((M * N, a.tags), generator=g, device=dev)
    params = fleet.random_glorot_params(eng, M, g)
    jobs = engine.jobs_to_device(engine.uniform_jobs(M, N), dev)
    p0 = params.clone()
    eng.fit(p0, jobs, M, N, x, x, epochs=1, batch_size=B, loss=a.loss, optimizer=opt)  # warm-up
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    loss, acc, _ = eng.fit(params, jobs, M, N, x, x, epochs=E, batch_size=B, loss=a.loss, optimizer=opt)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1)
    steps = E * ((N + B - 1) // B)
    sms = 132
    waves = (M + sms - 1) // sms
    out = {
        "workload": f"{M} machines x {a.tags}-tag hourglass, {N} rows, {E} epochs, batch {B}, loss {a.loss}"
                    + (f", optimizer {a.optimizer}" if a.optimizer else ""),
        "ms": ms, "row_epochs_per_s": M * N * E / (ms * 1e-3), "us_per_step_per_cta": ms * 1e3 / (steps * waves),
        "steps_per_fit": steps, "waves": waves, "loss_first_last": [float(loss[:, 0].mean()), float(loss[:, -1].mean())],
        "algorithmic_tflops": M * N * E * 90708 / (ms * 1e-3) / 1e12,
        "extrapolated_s_1000_machines_100_epochs": ms * 1e-3 * (100 / E) * (((1000 + sms - 1) // sms) / waves) if N == 10000 else None,
    }
    if a.dropout is not None:
        rates = [0.0] + [0.0 if spec.l1[l - 1] else a.dropout for l in range(1, spec.n_layers)]  # not after an activity L1 (refused)
        eng.fit(p0.clone(), jobs, M, N, x, x, epochs=1, batch_size=B, loss=a.loss, optimizer=opt, dropout=rates)  # warm-up
        times = {"without": [], "with": []}
        for _ in range(a.repeats):
            for name, d in (("without", None), ("with", rates)):
                p = p0.clone()
                torch.cuda.synchronize()
                ev0.record()
                eng.fit(p, jobs, M, N, x, x, epochs=E, batch_size=B, loss=a.loss, optimizer=opt, dropout=d)
                ev1.record()
                torch.cuda.synchronize()
                times[name].append(ev0.elapsed_time(ev1))
        per_step = {k: [t * 1e3 / (steps * waves) for t in v] for k, v in times.items()}
        out["dropout"] = {
            "rates": rates, "repeats": a.repeats, "ms": times, "us_per_step_per_cta": per_step,
            "median_cost": float(np.median(per_step["with"]) / np.median(per_step["without"]) - 1.0),
            "gpu": torch.cuda.get_device_name(dev), "power_limit": _power_limit(),
        }
    if a.cpu:
        w0 = km.init_ff_weights(spec, np.random.default_rng(0))
        Xc = np.random.default_rng(1).random((2000, a.tags)).astype(np.float32)
        t0 = time.perf_counter()
        km.ff_fit(spec, w0, Xc, Xc, epochs=1, batch_size=B)
        dt = time.perf_counter() - t0
        out["cpu_oracle_row_epochs_per_s_1core"] = 2000 / dt
        out["cpu_oracle_us_per_step"] = dt * 1e6 / ((2000 + B - 1) // B)
    print(json.dumps(out))


def _power_limit():
    """The card's power limit and maximum SM clock, as nvidia-smi reports them (None where it cannot be read)."""
    import subprocess

    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else None
    except (OSError, subprocess.SubprocessError):
        return None


if __name__ == "__main__":
    main()
