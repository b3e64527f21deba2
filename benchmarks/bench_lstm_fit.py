"""
LSTM training throughput (gb_lstm_fit): machines x windows trained per second for the BASELINE configs[3] architecture
(128 tags, lstm_symmetric dims (256,128,64), lookback 144) and a smaller one, with the CPU oracle's BPTT timed beside it.

    python benchmarks/bench_lstm_fit.py [--machines 8] [--rows 400] [--tags 128] [--lookback 144] [--batch 32] [--cpu 1]
                                        [--variant auto|fp32|tc[,...]] [--rounds 1]

Batches above 32 windows run the tensor-core family (gb_lstm_fit_tc); ``--variant`` forces a family, and a comma list times
several alternately, ``--rounds`` times each, in one process (e.g. ``--batch 32 --variant fp32,tc --rounds 3``).  With
``--variant`` or a batch above 32, every run prints its own line naming the family, the card and its power limit (read-only
``nvidia-smi`` query), and the algorithmic TF32 rate against the H100 SXM data sheet's 495 TFLOP/s dense: the tc family issues
3 MMAs per product (hi*hi + hi*lo + lo*hi), so its tensor cores do three times the algorithmic work.
"""
import argparse, json, os, subprocess, sys, time
import numpy as np
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--machines", type=int, default=8)
    ap.add_argument("--rows", type=int, default=400)
    ap.add_argument("--tags", type=int, default=128)
    ap.add_argument("--lookback", type=int, default=144)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--cpu", type=int, default=1)
    ap.add_argument("--variant", default=None, help="auto, fp32, tc or a comma list of them, timed alternately")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--optimizer", default=None, help="a Keras optimizer name with its default hyperparameters; without it, Adam")
    a = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    from gordo_components_b200 import engine
    from oracle import keras_math as km

    from gordo_components_b200.machine.model.factories.specs import resolve_optimizer

    opt = None if a.optimizer is None else resolve_optimizer(a.optimizer, {})
    spec = km.lstm_symmetric_spec(a.tags, lookback_window=a.lookback)
    eng = engine.LSTMEngine(spec.n_features, spec.units, spec.acts, spec.n_features_out, spec.out_func, spec.lookback_window)
    dev = eng.device
    M, N = a.machines, a.rows
    nwin = N - a.lookback + 1
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.rand((M * N, a.tags), generator=g, device=dev)
    w0 = km.init_lstm_weights(spec, np.random.default_rng(0))
    params = eng.pack_params([w0] * M)
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(M), nwin, np.arange(M, dtype=np.int64) * N), dev)
    workload = f"{M} machines x {a.tags}-tag lstm_symmetric(256,128,64), lookback {a.lookback}, {nwin} windows, batch {a.batch}, 1 epoch"
    if opt is not None:
        workload += f", optimizer {a.optimizer}"
    steps = 1 + (nwin + a.batch - 1) // a.batch

    def timed(fit):
        p = params.clone()
        fit(p.clone(), jobs, M, min(nwin, a.batch), x, x, epochs=1, batch_size=a.batch, primer=False, optimizer=opt)  # warm-up: one step
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        loss, acc, _ = fit(p, jobs, M, nwin, x, x, epochs=1, batch_size=a.batch, primer=True, optimizer=opt)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), loss

    def result(ms, loss):
        return {"workload": workload, "ms": ms, "steps": steps, "ms_per_step": ms / steps, "window_epochs_per_s": M * nwin / (ms * 1e-3),
                "algorithmic_tflops": 3 * spec.flop_per_window * M * nwin / (ms * 1e-3) / 1e12, "loss": float(loss.mean())}

    if a.variant is not None or a.batch > eng.FP32_MAX_BATCH:
        card = _card()
        variants = (a.variant or "auto").split(",")
        for _ in range(a.rounds):
            for v in variants:
                fit = {"auto": eng.fit_for_batch(a.batch), "fp32": eng.fit, "tc": eng.fit_tc}[v]
                out = result(*timed(fit))
                out.update({"variant": v, "path": "tc (gb_lstm_fit_tc, split TF32 wgmma)" if fit == eng.fit_tc else "fp32 (gb_lstm_fit, CUDA cores)",
                            "pct_of_495_tf32_tflops": 100 * out["algorithmic_tflops"] / 495.0,
                            "mma_per_product": 3 if fit == eng.fit_tc else 0, **card})
                print(json.dumps(out), flush=True)
        return
    out = result(*timed(eng.fit))
    if a.cpu:
        X = np.random.default_rng(1).random((a.lookback + 3, a.tags)).astype(np.float32)
        t0 = time.perf_counter()
        km.lstm_fit(spec, w0, X, X, epochs=1, batch_size=4)
        dt = time.perf_counter() - t0
        out["cpu_oracle_windows_per_s_1core"] = 5 / dt  # primer (1 window) + one batch of 4
    print(json.dumps(out))


def _card():
    """Name and power limit of the GPU, as nvidia-smi reports them (a read-only query)."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = (v.strip() for v in r.stdout.strip().splitlines()[0].split(",", 1))
        return {"gpu": name, "power_limit": power}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return {"gpu": "unknown", "power_limit": "unknown"}


if __name__ == "__main__":
    main()
