"""
Streaming ceilings of the fused predict+score kernel's data path, next to the kernel itself.

    python benchmarks/bench_tc_stream.py [--windows N] [--rows R] [--passes P] [--warmup W] [--kernel] [--build-dir DIR]

Compiles benchmarks/tc_stream.cu with the flags of gordo_components_b200/csrc/build.py (into DIR, by default
benchmarks/build/, which git ignores) and times, with CUDA events, three kernels that move the headline workload's bytes
(x and y in; model output, three per-tag anomaly arrays and three row totals out: 1 548 B per window of 64 tags) without any
model arithmetic: `half_row` (the fused kernel's tiles, staging boxes and TMA stores of 16 rows x 32 columns), `whole_row`
(the same with 8-row boxes of whole rows) and `plain` (float4 loads and stores at full occupancy).  None of them is the
fused kernel's result.  `--kernel` also times `FFEngine.infer_score` at the same fleet shape for feedforward_hourglass(64) and
for a six-layer 64-wide stack.  Prints one JSON line, with the card's name, power limit and the median SM clock sampled by
`nvidia-smi --query-gpu` while the GPU was busy.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..")))

BYTES_PER_WINDOW = 1548


def smi(fields):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    return [v.strip() for v in r.stdout.strip().split(",")] if r.returncode == 0 else None


class ClockSampler(threading.Thread):
    def __init__(self):
        super().__init__(daemon=True)
        self.samples, self.stop = [], threading.Event()

    def run(self):  # only samples taken while the GPU is busy: the timed passes are a small part of the run
        while not self.stop.wait(0.05):
            v = smi("clocks.sm,utilization.gpu")
            if v and len(v) == 2 and v[0].isdigit() and v[1].isdigit() and int(v[1]) >= 50:
                self.samples.append(int(v[0]))

    def median(self):
        self.stop.set()
        self.join()
        return statistics.median(self.samples) if self.samples else None


def build_probe(build_dir):
    from gordo_components_b200.csrc import build as gb_build

    os.makedirs(build_dir, exist_ok=True)
    exe = os.path.join(build_dir, "tc_stream")
    cmd = [gb_build._nvcc(), *gb_build.NVCC_FLAGS, os.path.join(HERE, "tc_stream.cu"), "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed on tc_stream.cu:\n{r.stdout}\n{r.stderr}")
    return exe


def time_kernel(dims, windows, rows, passes, warmup):
    import torch

    from gordo_components_b200 import engine, fleet

    acts = ["tanh"] * (len(dims) - 2) + ["linear"]
    eng = engine.FFEngine(dims, acts)
    dev = eng.device
    M, T = windows // rows, dims[0]
    g = torch.Generator(device=dev).manual_seed(1000)
    x = torch.rand((M * rows, T), generator=g, device=dev)
    y = x + 0.02 * torch.randn((M * rows, T), generator=g, device=dev)
    params = fleet.random_glorot_params(eng, M, g)
    jobs = engine.jobs_to_device(engine.uniform_jobs(M, rows), dev)
    scale, _ = eng.minmax_fit(jobs, M, rows, y, M)
    feat = torch.rand((M, T), generator=g, device=dev) * 0.2 + 0.05
    agg = torch.rand((M,), generator=g, device=dev) * 0.1 + 0.01
    out = {}
    step = lambda: eng.infer_score(params, jobs, M, rows, x, y, scale, feat, agg, out=out, variant=2)  # noqa: E731
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    ms = []
    for _ in range(passes):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    del out, x, y
    torch.cuda.empty_cache()
    mean = sum(ms) / len(ms)
    return {"dims": dims, "ms": round(mean, 4), "ms_min": round(min(ms), 4), "ms_max": round(max(ms), 4),
            "G_windows_per_s": round(windows / mean / 1e6, 4), "GBps": round(BYTES_PER_WINDOW * windows / (mean * 1e6), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=10_000_000)
    ap.add_argument("--rows", type=int, default=10_000, help="rows per job (a multiple of 16 dividing --windows)")
    ap.add_argument("--passes", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernel", action="store_true", help="also time the fused kernel for the hourglass and the six-layer stack")
    ap.add_argument("--build-dir", default=os.path.join(HERE, "build"))
    args = ap.parse_args()
    if args.passes < 20:
        ap.error("--passes must be at least 20")

    try:
        exe = build_probe(args.build_dir)
    except PermissionError:
        exe = build_probe(tempfile.mkdtemp(prefix="tc_stream_"))
    card = smi("name,power.limit,clocks.max.sm")
    sampler = ClockSampler()
    sampler.start()
    r = subprocess.run([exe, str(args.windows), str(args.rows), str(args.passes), str(args.warmup)], capture_output=True, text=True)
    if r.returncode != 0:
        sampler.median()
        raise RuntimeError(f"tc_stream failed ({r.returncode}):\n{r.stdout}\n{r.stderr}")
    res = json.loads(r.stdout.strip().splitlines()[-1])
    if args.kernel:
        import __graft_entry__ as ge

        ge.build()
        from gordo_components_b200.machine.model.factories.feedforward_autoencoder import feedforward_hourglass

        res["kernel"] = {
            "hourglass64": time_kernel(feedforward_hourglass(64).dims, args.windows, args.rows, args.passes, args.warmup),
            "six_layer_64": time_kernel([64] * 7, args.windows, args.rows, args.passes, args.warmup),
        }
    res["sm_clock_median_mhz"] = sampler.median()
    if card:
        res["gpu"], res["power_limit_w"], res["max_sm_clock_mhz"] = card[0], card[1], card[2]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
