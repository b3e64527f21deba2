"""
The output stage of the tensor-core kernel (variant 2) scores each element in one pass per array and sums the row totals in
the passes over the unscaled and scaled arrays, whether or not those arrays are asked for.  These tests hold it to: every
subset of the score outputs equal, bit for bit, to the same arrays of a full request; the live rows of 16-row boxes that end
inside a job written at every row residue; and the totals equal to the mean of squares of the per-tag arrays of the same launch.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PER_TAG = ["model-output", "tag-anomaly-scaled", "tag-anomaly-unscaled", "anomaly-confidence"]
TOTALS = ["total-anomaly-scaled", "total-anomaly-unscaled", "total-anomaly-confidence"]
ALL_KEYS = PER_TAG + TOTALS
GAP = 3  # output rows between two jobs (and before the first)


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("needs an H100")
    import __graft_entry__ as ge

    ge.build()
    return t


def fleet(torch, T, n_rows, seed, gap=GAP):
    """Two slots of feedforward_hourglass(T) weights and jobs with the given row counts, their outputs `gap` rows apart."""
    from gordo_components_b200 import engine
    from oracle import keras_math as km

    rng = np.random.default_rng(seed)
    spec = km.ff_hourglass_spec(T)
    weights = []
    for s in range(2):
        w = km.init_ff_weights(spec, np.random.default_rng(1000 * T + seed + s))
        weights.append([(W, rng.uniform(-0.2, 0.2, b.shape).astype(np.float32)) for W, b in w])
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    n_x = int(sum(n_rows)) + 37
    Xh = (rng.random((n_x, T)) * 2 - 0.5).astype(np.float32)
    yh = (Xh + rng.normal(0, 0.05, Xh.shape)).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)  # noqa: E731
    x_rows = np.concatenate([[0], np.cumsum(n_rows[:-1])]) + 5
    out_rows = gap + np.cumsum([0] + [n + gap for n in n_rows[:-1]])
    total = int(out_rows[-1] + n_rows[-1] + gap)
    jobs = engine.make_jobs([j % 2 for j in range(len(n_rows))], n_rows, x_rows, out_rows)
    data = dict(params=eng.pack_params(weights), X=t(Xh), y=t(yh), sc=t(rng.random((2, T)) + 0.5), feat=t(rng.random((2, T)) * 0.2 + 0.05),
                agg=t(rng.random(2) * 0.1 + 0.01))
    written = np.zeros(total, bool)
    for o, n in zip(out_rows, n_rows):
        written[o:o + n] = True
    return eng, jobs, data, total, written


def run(torch, eng, jobs, d, total, want, variant, with_y=True):
    from gordo_components_b200 import engine

    T = d["X"].shape[1]
    out = {k: torch.full((total, T) if k in PER_TAG else (total,), float("nan"), dtype=torch.float32, device=eng.device) for k in ALL_KEYS}
    eng.infer_score(d["params"], engine.jobs_to_device(jobs, eng.device), len(jobs), int(jobs["n_rows"].max()), d["X"],
                    d["y"] if with_y else None, d["sc"], d["feat"], d["agg"], out_rows=total, want=want, variant=variant, out=out)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


SUBSETS = [[k] for k in ALL_KEYS[1:]] + [TOTALS, []]


@pytest.mark.parametrize("want", SUBSETS, ids=["+".join(w) or "prediction-only" for w in SUBSETS])
def test_tc_output_subset_is_bit_identical_to_full_request(torch, want):
    eng, jobs, d, total, written = fleet(torch, 64, [200, 64, 33, 130], seed=7)
    full = run(torch, eng, jobs, d, total, ALL_KEYS[1:], variant=2)
    got = run(torch, eng, jobs, d, total, want, variant=2)
    for k in ALL_KEYS:
        if k == "model-output" or k in want:
            assert not np.isnan(got[k][written]).any(), f"{k}: rows of a job were not written"
            np.testing.assert_array_equal(got[k], full[k], err_msg=f"{k} differs from the full request")
        else:
            assert np.isnan(got[k]).all(), f"{k} was not asked for but was written"


def test_tc_prediction_without_y_is_bit_identical(torch):
    eng, jobs, d, total, written = fleet(torch, 64, [200, 64, 33, 130], seed=8)
    full = run(torch, eng, jobs, d, total, ALL_KEYS[1:], variant=2)
    got = run(torch, eng, jobs, d, total, ALL_KEYS[1:], variant=2, with_y=False)
    np.testing.assert_array_equal(got["model-output"], full["model-output"])
    for k in ALL_KEYS[1:]:
        assert np.isnan(got[k]).all(), f"{k} was written without y"


def close(got, want, mag, name):
    err = np.abs(got.astype(np.float64) - want.astype(np.float64))
    tol = 1e-4 * np.abs(want) + 2e-5 * mag  # the tolerance of the parity tests (test_gpu_parity.py)
    assert (err <= tol).all(), f"{name}: {(~(err <= tol)).sum()} values outside tolerance, max err {err.max():.3e}"


@pytest.mark.parametrize("T", [24, 28, 32, 36, 60, 64])
def test_tc_job_ends_at_every_box_residue(torch, T):
    """Jobs of 64 + r rows, r = 0..15: the last 16-row box of each job holds r live rows (every residue mod 16 and mod 8)."""
    n_rows = [64 + r for r in range(16)]
    eng, jobs, d, total, written = fleet(torch, T, n_rows, seed=T)
    got = run(torch, eng, jobs, d, total, ALL_KEYS[1:], variant=2)
    ref = run(torch, eng, jobs, d, total, ALL_KEYS[1:], variant=1)
    smax, fmax = float(d["sc"].max()), float((1 / d["feat"]).max())
    mags = {"model-output": 1.0, "tag-anomaly-unscaled": 1.0, "tag-anomaly-scaled": smax, "anomaly-confidence": fmax,
            "total-anomaly-unscaled": 1.0, "total-anomaly-scaled": smax * smax, "total-anomaly-confidence": smax * smax / float(d["agg"].min())}
    for k in ALL_KEYS:
        assert np.isnan(got[k][~written]).all(), f"{k}: rows outside every job were written"
        assert not np.isnan(got[k][written]).any(), f"{k}: rows of a job were not written"
        close(got[k][written], ref[k][written], mags[k], k)


@pytest.mark.parametrize("T", [32, 36, 64])
def test_tc_totals_are_the_mean_of_squares_of_the_per_tag_outputs(torch, T):
    eng, jobs, d, total, written = fleet(torch, T, [200, 64, 33, 130, 71], seed=11 + T)
    got = run(torch, eng, jobs, d, total, ALL_KEYS[1:], variant=2)
    for tot, tag in (("total-anomaly-unscaled", "tag-anomaly-unscaled"), ("total-anomaly-scaled", "tag-anomaly-scaled")):
        want = (got[tag][written].astype(np.float64) ** 2).mean(axis=1)
        np.testing.assert_allclose(got[tot][written], want, rtol=1e-5, atol=0, err_msg=tot)
