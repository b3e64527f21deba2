"""
BASELINE configs[2] (scaled): batched training of 64-tag feedforward_hourglass autoencoders, one persistent CTA per machine.
Reports row-epochs/s, microseconds per optimizer step and the CPU oracle (NumPy Keras-style loop) on a small sample.

    python benchmarks/bench_fit.py [--machines 296] [--rows 10000] [--epochs 3] [--batch 32] [--loss mse] [--optimizer Nadam]
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
    if a.cpu:
        w0 = km.init_ff_weights(spec, np.random.default_rng(0))
        Xc = np.random.default_rng(1).random((2000, a.tags)).astype(np.float32)
        t0 = time.perf_counter()
        km.ff_fit(spec, w0, Xc, Xc, epochs=1, batch_size=B)
        dt = time.perf_counter() - t0
        out["cpu_oracle_row_epochs_per_s_1core"] = 2000 / dt
        out["cpu_oracle_us_per_step"] = dt * 1e6 / ((2000 + B - 1) // B)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
