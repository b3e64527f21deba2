"""
The batched form of `gordo build` for one bucket of machines: 3-fold TimeSeriesSplit cross-validation + final fit + thresholds +
scalers (what ModelBuilder._build does per machine, gordo/builder/build_model.py:192-339) for ALL machines in four launches.

    python benchmarks/bench_build.py [--machines 132] [--rows 10000] [--epochs 5] [--batch 32]
"""
import argparse, json, os, sys
sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--machines", type=int, default=132)
    ap.add_argument("--rows", type=int, default=10000)
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--tags", type=int, default=64)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as ge
    ge.build()
    from gordo_components_b200 import engine, fleet
    from gordo_components_b200.machine.model.factories.feedforward_autoencoder import feedforward_hourglass

    spec = feedforward_hourglass(a.tags)
    eng = engine.ff_engine_for(spec)
    dev = eng.device
    M, N = a.machines, a.rows
    g = torch.Generator(device=dev).manual_seed(0)
    t = torch.arange(N, device=dev, dtype=torch.float32)[None, :, None] * 0.01
    x = (0.5 + 0.4 * torch.sin(t * (0.5 + torch.rand((M, 1, a.tags), generator=g, device=dev)) + 6 * torch.rand((M, 1, a.tags), generator=g, device=dev))
         + 0.02 * torch.randn((M, N, a.tags), generator=g, device=dev)).reshape(M * N, a.tags).contiguous()
    fleet.build_fleet(eng, x[: 2 * N], x[: 2 * N], rows=N, epochs=1, batch_size=a.batch)  # warm-up
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    fb = fleet.build_fleet(eng, x, x, rows=N, epochs=a.epochs, batch_size=a.batch)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1)
    fits = 4 * M
    print(json.dumps({
        "workload": f"{M} machines x {a.tags}-tag hourglass, {N} rows, {a.epochs} epochs, batch {a.batch}, 3-fold CV + final fit + thresholds",
        "ms": ms, "fits": fits, "machines_per_s": M / (ms * 1e-3),
        "row_epochs_per_s": M * a.epochs * N * (1 + 0.25 + 0.5 + 0.75) / (ms * 1e-3),
        "loss_first_last": [float(fb.loss[:, 0].mean()), float(fb.loss[:, -1].mean())],
        "agg_threshold_median": float(fb.agg_thr.median()),
    }))


if __name__ == "__main__":
    main()
