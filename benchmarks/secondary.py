"""
The other BASELINE.json configurations as one GPU's share each, timed after bench.py's main region (its `secondary` block) so that
every configuration has a driver-run number beside the headline:

* configs[3]  256 machines x 128-tag KerasLSTMAutoEncoder (lstm_symmetric, lookback 144) on 8 GPUs -> 32 machines per GPU
* configs[2]  1 000 machines x 64-tag hourglass AE, 100 epochs, on 8 GPUs                          -> 125 machines per GPU
* configs[4]  gordo.server batch-predict load test shape (benchmarks/test_ml_server.py:21-42: 100-row POSTs), concurrent requests
              against device-resident models through the request coalescer

Each function returns a dict; all inputs are synthetic and live on the device, timing is CUDA events (wall clock for the threaded
request test).  Architectures come from this package's own factories.
"""
from __future__ import annotations

import threading
import time

import numpy as np

LSTM_FLOP_PER_WINDOW = 335_085_568   # SURVEY 8a11: 2 * 1 163 264 MAC * 144 steps + Dense 2*256*128
FIT_FLOP_PER_ROW_EPOCH = 90_708      # SURVEY 8d: 3 x 30 236


def lstm_share(torch, engine, machines: int = 32, rows: int = 10_000, lookback: int = 144, peaks=None):
    """configs[3], one GPU's share: windows/s, algorithmic TFLOP/s, fraction of the sustained bf16 GEMM peak."""
    from gordo_components_b200.machine.model.factories.lstm_autoencoder import lstm_symmetric

    spec = lstm_symmetric(128, lookback_window=lookback)
    eng = engine.lstm_engine_for(spec)
    dev = eng.device
    nwin = rows - lookback + 1
    g = torch.Generator(device=dev).manual_seed(3)
    params = (torch.rand((machines, eng.param_stride), generator=g, device=dev) - 0.5) * 0.2
    x = torch.rand((machines * rows, 128), generator=g, device=dev)
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(machines), nwin, np.arange(machines) * rows, np.arange(machines) * nwin), dev)
    eng.infer(params, jobs, machines, nwin, x, machines * nwin)  # warm-up (tensor maps, workspace)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    eng.infer(params, jobs, machines, nwin, x, machines * nwin)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1)
    wps = machines * nwin / (ms * 1e-3)
    tflops = wps * LSTM_FLOP_PER_WINDOW / 1e12
    out = {"workload": f"configs[3] share: {machines} machines x 128-tag lstm_symmetric(256,128,64), lookback {lookback}, {nwin} windows each",
           "kernel": "wgmma" if eng.tc_supported else "fp32", "ms": ms, "windows_per_s": wps, "algorithmic_tflops": tflops}
    if peaks:
        sustained = peaks.get("bf16_tflops_sustained", peaks.get("bf16_tflops"))
        out["frac_of_bf16_sustained_peak"] = tflops / sustained
        out["tensor_pipe_frac"] = 3 * tflops / sustained  # FP16-pair split: three MMAs per product
    return out


def fit_share(torch, engine, fleet, machines: int = 125, rows: int = 10_000, epochs: int = 100, batch: int = 32):
    """configs[2], one GPU's share: row-epochs/s and microseconds per optimizer step of the persistent-CTA training kernel."""
    from gordo_components_b200.machine.model.factories.feedforward_autoencoder import feedforward_hourglass

    eng = engine.ff_engine_for(feedforward_hourglass(64))
    dev = eng.device
    g = torch.Generator(device=dev).manual_seed(4)
    x = torch.rand((machines * rows, 64), generator=g, device=dev)
    params = fleet.random_glorot_params(eng, machines, g)
    jobs = engine.jobs_to_device(engine.uniform_jobs(machines, rows), dev)
    eng.fit(params.clone(), jobs, machines, rows, x, x, epochs=1, batch_size=batch)  # warm-up
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    loss, _, _ = eng.fit(params, jobs, machines, rows, x, x, epochs=epochs, batch_size=batch)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1)
    steps = epochs * ((rows + batch - 1) // batch)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    waves = (machines + sms - 1) // sms
    return {"workload": f"configs[2] share: {machines} machines x 64-tag hourglass, {rows} rows, {epochs} epochs, batch {batch} (fits only; a build adds 3 CV folds)",
            "ms": ms, "row_epochs_per_s": machines * rows * epochs / (ms * 1e-3), "us_per_optimizer_step": ms * 1e3 / (steps * waves), "steps_per_fit": steps,
            "ctas": machines, "sms": sms, "waves": waves, "algorithmic_tflops": machines * rows * epochs * FIT_FLOP_PER_ROW_EPOCH / (ms * 1e-3) / 1e12,
            "loss_first_last": [float(loss[:, 0].mean()), float(loss[:, -1].mean())]}


def server_shape(torch, engine, fleet, machines: int = 1000, requests: int = 2000, rows: int = 100, threads: int = 8):
    """configs[4] shape: concurrent 100-row anomaly requests over resident models, coalesced into shared launches."""
    from gordo_components_b200 import serving
    from gordo_components_b200.machine.model.factories.feedforward_autoencoder import feedforward_hourglass

    eng = engine.ff_engine_for(feedforward_hourglass(64))
    dev = eng.device
    g = torch.Generator(device=dev).manual_seed(5)
    params = fleet.random_glorot_params(eng, machines, g)
    scale = torch.rand((machines, 64), generator=g, device=dev) + 0.5
    feat = torch.rand((machines, 64), generator=g, device=dev) + 0.5
    agg = torch.rand((machines,), generator=g, device=dev) + 0.5
    rng = np.random.default_rng(0)
    reqs = [(int(rng.integers(0, machines)), rng.random((rows, 64)).astype(np.float32)) for _ in range(requests)]
    co = serving.AnomalyCoalescer(eng, params, scale, feat, agg, max_wait_ms=0.2)
    try:
        co.anomaly(*reqs[0], reqs[0][1])
        idx, lock, lat = iter(range(len(reqs))), threading.Lock(), []

        def worker():
            while True:
                with lock:
                    i = next(idx, None)
                if i is None:
                    return
                t0 = time.perf_counter()
                co.anomaly(reqs[i][0], reqs[i][1], reqs[i][1])
                lat.append(time.perf_counter() - t0)

        ts = [threading.Thread(target=worker) for _ in range(threads)]
        b0 = co.batches
        t0 = time.perf_counter()
        [t.start() for t in ts]
        [t.join() for t in ts]
        dt = time.perf_counter() - t0
        out = {"workload": f"configs[4] shape: {requests} anomaly requests x {rows} rows x 64 tags over {machines} resident machines, {threads} client threads, request coalescer",
               "requests_per_s": requests / dt, "windows_per_s": requests * rows / dt, "p50_ms": 1e3 * float(np.median(lat)), "p99_ms": 1e3 * float(np.quantile(lat, 0.99)),
               "launches": co.batches - b0}
        # the load-test shape proper: all requests in flight at once
        b0 = co.batches
        t0 = time.perf_counter()
        futs = [co.submit(s, X, X) for s, X in reqs]
        [f.result() for f in futs]
        dt = time.perf_counter() - t0
        out["all_in_flight"] = {"windows_in_flight": requests * rows, "windows_per_s": requests * rows / dt, "launches": co.batches - b0}
        return out
    finally:
        co.close()
