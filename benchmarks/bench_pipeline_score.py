"""
Scoring behind a Pipeline's input scaler (DiffBasedAnomalyDetector(Pipeline([MinMaxScaler, KerasAutoEncoder])), the definition of
every reference example): the float64 affine pass + fused launch (gb_affine_f64, gb_ffae_infer_score) against the fused launch
that applies the scaler as it reads x (gb_ffae_infer_score_x64).

  (a) kernel: BASELINE configs[1] (1 000 machines x 10 000 rows x 64 tags, feedforward_hourglass(64)) with a per-machine
      MinMaxScaler, the two routes alternated step by step, timed with CUDA events; their outputs are compared bit for bit.
  (b) served: BASELINE configs[4] (benchmarks/bench_server.py: 100-row requests from 8 threads) with Pipeline models, one
      launch per request against the request coalescer with per-slot input scalers.

    python benchmarks/bench_pipeline_score.py [--machines 1000] [--rows 10000] [--steps 10] [--warmup 2] [--requests 2000]

Prints one JSON line.
"""
import argparse, json, os, subprocess, sys, threading, time
import numpy as np
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def window_bytes(T, x64_fused: bool) -> int:
    """Algorithmic HBM bytes per window with every output (model output, three per-tag anomaly arrays, three totals)."""
    outs = 4 * 4 * T + 3 * 4
    fused = 4 * T + outs  # y, outputs
    if x64_fused:
        return 8 * T + fused  # float64 x read once
    return 8 * T + 4 * T + 4 * T + fused  # affine pass: float64 x in, float32 x' out; fused launch reads x' back


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "power_limit_and_max_sm_clock": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


def kernel_arm(a, torch, engine, fleet, eng):
    dev = eng.device
    M, R, T = a.machines, a.rows, eng.n_in
    g = torch.Generator(device=dev).manual_seed(0)
    params = fleet.random_glorot_params(eng, M, g)
    x = torch.randn((M * R, T), generator=g, device=dev, dtype=torch.float64) * 50.0 + 1e4
    lo, hi = x.view(M, R, T).amin(1), x.view(M, R, T).amax(1)
    xa = 1.0 / (hi - lo)  # MinMaxScaler per machine
    xb = -lo * xa
    y = torch.rand((M * R, T), generator=g, device=dev)
    scale = torch.rand((M, T), generator=g, device=dev) + 0.5
    feat = torch.rand((M, T), generator=g, device=dev) + 0.5
    agg = torch.rand((M,), generator=g, device=dev) + 0.5
    jobs = engine.jobs_to_device(engine.uniform_jobs(M, R), dev)
    outs = [{}, {}]

    def two_launch():  # x' from the caching allocator, as the detector's route gets it
        return eng.infer_score(params, jobs, M, R, engine.affine_f64(jobs, M, R, x, xa, xb), y, scale, feat, agg, out=outs[0])

    def fused():
        return eng.infer_score(params, jobs, M, R, x, y, scale, feat, agg, out=outs[1], x_affine=(xa, xb))

    routes = {"two_launch": two_launch, "fused_x64": fused}
    for _ in range(a.warmup):
        for fn in routes.values():
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in routes}
    for _ in range(a.steps):  # alternated in the same run
        for k, fn in routes.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    same = all(torch.equal(outs[0][k].view(torch.int32), outs[1][k].view(torch.int32)) for k in outs[0])
    res = {}
    for k, v in ms.items():
        med = float(np.median(v))
        b = window_bytes(T, k == "fused_x64")
        res[k] = {"ms_per_step_median": med, "ms_min": float(np.min(v)), "ms_max": float(np.max(v)),
                  "windows_per_s": M * R / (med * 1e-3), "bytes_per_window": b,
                  "achieved_GB_per_s": b * M * R / (med * 1e-3) / 1e9, "fraction_of_3.35TB_per_s": b * M * R / (med * 1e-3) / HBM_BYTES_PER_S}
    res["speedup_fused_over_two_launch"] = res["two_launch"]["ms_per_step_median"] / res["fused_x64"]["ms_per_step_median"]
    res["outputs_bit_identical"] = bool(same)
    res["tc_plan_x64"] = eng.infer_plan_x64(0)
    return res


def served_arm(a, torch, engine, fleet, serving, eng):
    dev = eng.device
    M, T = a.machines, eng.n_in
    g = torch.Generator(device=dev).manual_seed(1)
    params = fleet.random_glorot_params(eng, M, g)
    scale = torch.rand((M, T), generator=g, device=dev) + 0.5
    feat = torch.rand((M, T), generator=g, device=dev) + 0.5
    agg = torch.rand((M,), generator=g, device=dev) + 0.5
    rng = np.random.default_rng(0)
    lo = 1e4 + rng.random((M, T)) * 10
    xa = torch.from_numpy(1.0 / (rng.random((M, T)) * 100 + 1)).to(dev)
    xb = torch.from_numpy(-lo).to(dev) * xa
    reqs = [(int(s), 1e4 + rng.random((a.req_rows, T)) * 50) for s in rng.integers(0, M, a.requests)]
    ys = [rng.random((a.req_rows, T)).astype(np.float32) for _ in range(a.requests)]
    pairs = [(s, X, yv) for (s, X), yv in zip(reqs, ys)]

    def per_request(slot, X, yv):  # what DiffBasedAnomalyDetector._score launches for one Pipeline request
        n = len(X)
        jobs = engine.jobs_to_device(engine.make_jobs([0], [n], [0]), dev)
        res = eng.infer_score(params[slot:slot + 1], jobs, 1, n, torch.from_numpy(X).to(dev), torch.from_numpy(yv).to(dev), scale[slot:slot + 1],
                              feat[slot:slot + 1], agg[slot:slot + 1], x_affine=(xa[slot:slot + 1], xb[slot:slot + 1]))
        return {k: v.cpu().numpy() for k, v in res.items()}

    def drive(fn):
        idx = iter(range(len(pairs)))
        lock = threading.Lock()
        out = [None] * len(pairs)

        def worker():
            while True:
                with lock:
                    i = next(idx, None)
                if i is None:
                    return
                out[i] = fn(*pairs[i])

        ts = [threading.Thread(target=worker) for _ in range(a.threads)]
        t0 = time.perf_counter()
        [t.start() for t in ts]
        [t.join() for t in ts]
        return time.perf_counter() - t0, out

    co = serving.AnomalyCoalescer(eng, params, scale, feat, agg, x_scale=xa, x_offset=xb)
    drive(per_request)
    drive(co.anomaly)  # warm-up of both
    t_req, r_req = drive(per_request)
    b0 = co.batches
    t_co, r_co = drive(co.anomaly)
    batches = co.batches - b0
    co.close()
    same = all(np.array_equal(p[k].view(np.int32), c[k].view(np.int32)) for p, c in zip(r_req, r_co) for k in c)
    return {"requests": len(pairs), "rows_per_request": a.req_rows, "threads": a.threads,
            "per_request_req_per_s": len(pairs) / t_req, "coalescer_req_per_s": len(pairs) / t_co,
            "coalescer_batches": batches, "replies_bit_identical": bool(same)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--machines", type=int, default=1000)
    ap.add_argument("--rows", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--requests", type=int, default=2000)
    ap.add_argument("--req-rows", type=int, default=100)
    ap.add_argument("--threads", type=int, default=8)  # gunicorn threads per worker in the reference (gordo/cli/cli.py:288-296)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    from gordo_components_b200 import engine, fleet, serving
    from gordo_components_b200.machine.model.factories.feedforward_autoencoder import feedforward_hourglass

    eng = engine.ff_engine_for(feedforward_hourglass(64))
    out = {"card": card(), "kernel": kernel_arm(a, torch, engine, fleet, eng)}
    torch.cuda.empty_cache()
    out["served"] = served_arm(a, torch, engine, fleet, serving, eng)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
