"""
The tensor-core kernel writes its per-tag outputs as 16-row boxes: whole boxes by TMA store, and the live rows of a box that
crosses the end of a job by the warp itself.  These tests put the jobs' output ranges apart, with gaps between them, in
outputs pre-filled with NaN: every row of every job must be written, with the values of the fp32 kernel (variant 1), and
nothing else may be touched.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ALL_KEYS = ["model-output", "tag-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-scaled", "total-anomaly-unscaled",
            "anomaly-confidence", "total-anomaly-confidence"]
N_ROWS = [1, 15, 16, 17, 63, 64, 65, 129]  # around the 16-row warp box and the 64-row warpgroup tile
X_ROWS = [3, 0, 40, 101, 130, 250, 311, 400]
GAP = 5  # output rows between two jobs (and before the first)


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("needs an H100")
    import __graft_entry__ as ge

    ge.build()
    return t


def close(got, want, mag, name):
    err = np.abs(got.astype(np.float64) - want.astype(np.float64))
    tol = 1e-4 * np.abs(want) + 2e-5 * mag  # the tolerance of the parity tests (test_gpu_parity.py)
    assert (err <= tol).all(), f"{name}: {(~(err <= tol)).sum()} values outside tolerance, max err {err.max():.3e}"


def run(torch, eng, params, jobs, X, y, sc, feat, agg, total, want, variant):
    from gordo_components_b200 import engine

    dev = eng.device
    T = X.shape[1]
    out = {k: torch.full((total, T) if k in ("model-output", "tag-anomaly-scaled", "tag-anomaly-unscaled", "anomaly-confidence") else (total,),
                         float("nan"), dtype=torch.float32, device=dev) for k in ALL_KEYS}
    eng.infer_score(params, engine.jobs_to_device(jobs, dev), len(jobs), int(jobs["n_rows"].max()), X, y, sc, feat, agg, out_rows=total,
                    want=want, variant=variant, out=out)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("mode", ["score", "predict-only", "subset"])
@pytest.mark.parametrize("T", [24, 36, 48, 64])
def test_tc_outputs_stay_inside_their_jobs(torch, T, mode):
    from gordo_components_b200 import engine
    from oracle import keras_math as km

    rng = np.random.default_rng(T)
    spec = km.ff_hourglass_spec(T)
    weights = []
    for s in range(2):
        w = km.init_ff_weights(spec, np.random.default_rng(100 * T + s))
        weights.append([(W, rng.uniform(-0.2, 0.2, b.shape).astype(np.float32)) for W, b in w])
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    params = eng.pack_params(weights)
    Xh = (rng.random((600, T)) * 2 - 0.5).astype(np.float32)
    yh = (Xh + rng.normal(0, 0.05, Xh.shape)).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)  # noqa: E731
    X, y = t(Xh), (None if mode == "predict-only" else t(yh))
    sc = t(rng.random((2, T)) + 0.5)
    feat = t(rng.random((2, T)) * 0.2 + 0.05)
    agg = t(rng.random(2) * 0.1 + 0.01)
    out_rows = GAP + np.cumsum([0] + [n + GAP for n in N_ROWS[:-1]])
    total = int(out_rows[-1] + N_ROWS[-1] + GAP)
    jobs = engine.make_jobs([j % 2 for j in range(len(N_ROWS))], N_ROWS, X_ROWS, out_rows)
    want = ["tag-anomaly-scaled", "total-anomaly-unscaled"] if mode == "subset" else ALL_KEYS

    got = run(torch, eng, params, jobs, X, y, sc, feat, agg, total, want, variant=2)
    ref = run(torch, eng, params, jobs, X, y, sc, feat, agg, total, want, variant=1)

    written = np.zeros(total, bool)
    for o, n in zip(out_rows, N_ROWS):
        written[o:o + n] = True
    expected = {"model-output"} | (set() if mode == "predict-only" else set(want))
    smax, fmax = float(sc.max()), float((1 / feat).max())
    mags = {"model-output": 1.0, "tag-anomaly-unscaled": 1.0, "tag-anomaly-scaled": smax, "anomaly-confidence": fmax,
            "total-anomaly-unscaled": 1.0, "total-anomaly-scaled": smax * smax, "total-anomaly-confidence": smax * smax / float(agg.min())}
    for k in ALL_KEYS:
        if k not in expected:
            assert np.isnan(got[k]).all(), f"{k} was not asked for but was written"
            continue
        assert np.isnan(got[k][~written]).all(), f"{k}: rows outside every job were written"
        assert not np.isnan(got[k][written]).any(), f"{k}: rows of a job were not written"
        close(got[k][written], ref[k][written], mags[k], k)
