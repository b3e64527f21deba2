"""
Fold thresholds of detectors with a smoothing window, at the batched builder's fold-scoring shape: one gb_thresholds_pair launch
(the 6-row and the window-W thresholds from one pass over the scores) against the two gb_thresholds launches it replaces, at
W = 144 and W = 6, float32 (the feed-forward path) and float64 (the LSTM path).  Device time per call from CUDA events over
``--reps`` back-to-back calls after a warm-up, the median of ``--trials`` such windows; the outputs of both forms are compared
bit for bit in the same run.  Prints one JSON line with the card's name and power limit.

    python benchmarks/bench_smooth_thresholds.py [--machines 200] [--folds 3] [--rows 4380] [--tags 64]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _power_limit():
    """The card's power limit in watts, read-only query (None when nvidia-smi is not available)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--machines", type=int, default=200)
    ap.add_argument("--folds", type=int, default=3)
    ap.add_argument("--rows", type=int, default=4380, help="rows of every fold's test block")
    ap.add_argument("--tags", type=int, default=64)
    ap.add_argument("--windows", default="144,6")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--trials", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    import torch

    import __graft_entry__ as ge

    ge.build()
    from gordo_components_b200 import engine

    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    dev = torch.device("cuda:0")
    n_jobs, R, T = a.machines * a.folds, a.rows, a.tags
    S = n_jobs + a.machines  # the builder's slot layout: final fits first, then the folds
    jobs = engine.jobs_to_device(engine.make_jobs(a.machines + np.arange(n_jobs), np.full(n_jobs, R), np.zeros(n_jobs, np.int64),
                                                  np.arange(n_jobs, dtype=np.int64) * R), dev)
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": _power_limit(),
           "shape": f"{a.machines} machines x {a.folds} folds x {R}-row test blocks x {T} tags", "results": []}
    g = torch.Generator(device=dev).manual_seed(0)
    for dtype in (torch.float32, torch.float64):
        tag = torch.rand((n_jobs * R, T), generator=g, device=dev, dtype=dtype) ** 2
        tot = tag.mean(1)
        tag[torch.rand(tag.shape, generator=g, device=dev) < 1e-4] = float("nan")
        for w in (int(v) for v in a.windows.split(",")):
            def pair():
                return engine.thresholds_pair(jobs, n_jobs, R, tag, tot, T, S, 6, w, dev)

            def two():
                return engine.thresholds(jobs, n_jobs, R, tag, tot, T, S, 6, dev) + engine.thresholds(jobs, n_jobs, R, tag, tot, T, S, w, dev)

            got, want = pair(), two()
            torch.cuda.synchronize()
            ints = torch.int32 if dtype == torch.float32 else torch.int64
            identical = all(torch.equal(x.view(ints), y.view(ints)) for x, y in zip(got, want))

            def timed(fn):
                for _ in range(2):
                    fn()
                ms = []
                for _ in range(a.trials):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(a.reps):
                        fn()
                    e1.record()
                    torch.cuda.synchronize()
                    ms.append(e0.elapsed_time(e1) / a.reps)
                return float(np.median(ms)), float(min(ms)), float(max(ms))

            t_two, t_pair = [], []
            for _ in range(2):  # alternate the two forms
                t_two.append(timed(two))
                t_pair.append(timed(pair))
            two_ms, pair_ms = min(v[0] for v in t_two), min(v[0] for v in t_pair)
            score_bytes = (tag.numel() + tot.numel()) * tag.element_size()
            out["results"].append({"dtype": str(dtype).replace("torch.", ""), "w0": 6, "w1": w, "identical": bool(identical),
                                   "two_gb_thresholds_ms": two_ms, "gb_thresholds_pair_ms": pair_ms, "speedup": two_ms / pair_ms,
                                   "pair_score_bytes_per_s": score_bytes / (pair_ms * 1e-3), "spread_ms": {"two": t_two, "pair": t_pair}})
        del tag, tot
    print(json.dumps(out))


if __name__ == "__main__":
    main()
