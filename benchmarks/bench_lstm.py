"""
BASELINE configs[3] (scaled): 128-tag KerasLSTMAutoEncoder (lstm_symmetric 256-128-64, lookback 144) inference.
Reports windows/s and achieved TFLOP/s (335 085 568 FLOP per window) plus the CPU oracle on a small sample.

    python benchmarks/bench_lstm.py [--machines 8] [--rows 1400]
"""
import argparse, json, os, sys, time
import numpy as np
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--machines", type=int, default=8)
    ap.add_argument("--rows", type=int, default=1400)
    ap.add_argument("--lookback", type=int, default=144)
    ap.add_argument("--cpu", type=int, default=1)
    ap.add_argument("--variant", type=int, default=0, help="0 auto (tensor cores when supported), 1 fp32 CUDA cores, 2 tensor cores (wgmma)")
    a = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    from gordo_components_b200 import engine
    from oracle import keras_math as km

    spec = km.lstm_symmetric_spec(128, lookback_window=a.lookback)
    eng = engine.LSTMEngine(128, spec.units, spec.acts, 128, "linear", a.lookback)
    dev = eng.device
    M, N = a.machines, a.rows
    nwin = N - a.lookback + 1
    ws = [km.init_lstm_weights(spec, np.random.default_rng(m)) for m in range(min(M, 2))]
    params = eng.pack_params([ws[m % len(ws)] for m in range(M)])
    x = torch.rand((M * N, 128), device=dev)
    jobs_h = engine.make_jobs(np.arange(M), nwin, np.arange(M) * N, np.arange(M) * nwin)
    jobs = engine.jobs_to_device(jobs_h, dev)
    eng.infer(params, jobs, M, nwin, x, M * nwin, variant=a.variant)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    eng.infer(params, jobs, M, nwin, x, M * nwin, variant=a.variant)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1)
    out = {"workload": f"{M} machines x 128-tag lstm_symmetric(256,128,64), lookback {a.lookback}, {nwin} windows each",
           "kernel": "wgmma" if (a.variant == 2 or (a.variant == 0 and eng.tc_supported)) else "fp32 CUDA cores",
           "ms": ms, "windows_per_s": M * nwin / (ms * 1e-3), "tflops": M * nwin * spec.flop_per_window / (ms * 1e-3) / 1e12}
    if a.cpu:
        Xc = np.random.default_rng(0).random((a.lookback + 31, 128)).astype(np.float32)
        t0 = time.perf_counter()
        km.lstm_predict(spec, ws[0], Xc)
        dt = time.perf_counter() - t0
        out["cpu_oracle_windows_per_s"] = 32 / dt
    print(json.dumps(out))


if __name__ == "__main__":
    main()
