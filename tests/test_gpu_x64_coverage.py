"""
The float64-x inference path (gb_ffae_infer_score_x64: a Pipeline's per-feature input scalers applied as x is read) on every kernel
instantiation and plan it admits -- the generic kernel's four row-tile plans, the row-per-thread kernel's three widths and the
tensor-core kernel with three and with two warpgroups (tests/test_infer_plan_x64.py pins which shape runs on which) -- against the
float64 oracle (oracle/keras_math, oracle/anomaly_math) at the tolerances of parity_helpers.close, and bit for bit against the
two-launch route (gb_affine_f64, then the float32 launch on the same variant).  Then whole detectors, whose composed scalers are
checked against sklearn's own Pipeline transform, and a bucket of Pipeline detectors served through the request coalescer.
"""
import json
import threading

import numpy as np
import pandas as pd
import pytest
from oracle import keras_math as km
from parity_helpers import close
from test_gpu_infer_coverage import LAYOUT_SPECS, PER_ROW, SCORE, check_dense, dense_net, layout_jobs, run_dense, score_inputs
from test_infer_plan import COLUMN_BLOCKED, PLAN_SHAPES
from test_infer_plan_x64 import instantiation, plan_x64

pytestmark = pytest.mark.gpu

OUTS = ("model-output",) + SCORE


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("needs an H100")
    import __graft_entry__ as ge

    ge.build()
    return t


@pytest.fixture(scope="module")
def engine(torch):
    from gordo_components_b200 import engine as e

    return e


@pytest.fixture(scope="module")
def lib(torch):
    from gordo_components_b200 import _cabi

    return _cabi.load_library()


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int32) if a.dtype == np.float32 else a.view(np.int64)


def x64_inputs(rng, n_rows, n_in, n_slots):
    """Offset-dominated float64 x (values near 1e4) and a scaler per slot (a near 1e-4, b near -1): the float64 rounding of
    x * a + b decides x'."""
    x = 1e4 * (1.0 + 0.01 * rng.standard_normal((n_rows, n_in)))
    a = 1e-4 * rng.uniform(0.5, 2.0, (n_slots, n_in))
    b = -rng.uniform(0.5, 1.5, (n_slots, n_in))
    return x, a, b


def scaled(x, a, b):
    """x' as the kernels specify it: a float64 multiply, then a float64 add (two roundings, no FMA), then one rounding to float32."""
    return (np.multiply(x, a) + b).astype(np.float32)


def two_launch_route(engine, torch, spec, weights, X, a, b, y, jobs_h, scale, feat, agg, out_rows, variant, want=SCORE):
    """gb_affine_f64 writes each job's x' (its slot's scaler) to rows of its own, then the float32 launch reads them there: the same
    outputs, NaN-filled where no job writes, as the fused launch."""
    dev = torch.device("cuda")
    n = jobs_h["n_rows"].astype(np.int64)
    own = np.concatenate([[0], np.cumsum(n)[:-1]])
    total = max(1, int(n.sum()))
    t64 = lambda v: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(dev)  # noqa: E731
    aff = engine.make_jobs(jobs_h["slot"], n, jobs_h["x_row"], own)
    x32 = engine.affine_f64(engine.jobs_to_device(aff, dev), len(aff), max(1, int(n.max())), t64(X), t64(a), t64(b), out_rows=total)
    torch.cuda.synchronize()
    x32 = x32.cpu().numpy()
    y32 = None
    if y is not None:
        y32 = np.zeros((total, y.shape[1]), np.float32)
    for s, k, xr, o in zip(jobs_h["slot"], n, jobs_h["x_row"], own):
        if k:
            np.testing.assert_array_equal(_bits(x32[o:o + k]), _bits(scaled(X[xr:xr + k], a[s], b[s])), err_msg="gb_affine_f64")
            if y is not None:
                y32[o:o + k] = y[xr:xr + k]
    jobs = engine.make_jobs(jobs_h["slot"], n, own, jobs_h["out_row"])
    return run_dense(engine, torch, spec, weights, x32, y32, jobs, scale, feat, agg, out_rows, variant, want=want, nan_fill=True)


def x64_case(engine, torch, spec, weights, X, a, b, y, jobs_h, scale, feat, agg, out_rows, variant, name, want=SCORE):
    """The fused float64-x launch over the jobs `jobs_h` (outputs NaN-filled first): every job's rows against the oracle (all seven
    outputs when all are requested), bit for bit against the two-launch route, and NaN wherever no job writes."""
    got = run_dense(engine, torch, spec, weights, X, y, jobs_h, scale, feat, agg, out_rows, variant, want=want, nan_fill=True, x_affine=(a, b))
    written = np.zeros(out_rows, bool)
    for j, job in enumerate(jobs_h):
        s, n, xr, orow = (int(job[k]) for k in ("slot", "n_rows", "x_row", "out_row"))
        if n == 0:
            continue
        rows = slice(orow, orow + n)
        written[rows] = True
        want_out = km.ff_forward(spec, weights[s], scaled(X[xr:xr + n], a[s], b[s]), np.float64)
        if y is not None and tuple(want) == SCORE:
            check_dense(got, rows, want_out, y[xr:xr + n], scale[s], feat[s], agg[s], f"{name} job {j}")
        else:
            close(got["model-output"][rows], want_out, max(1.0, float(np.abs(want_out).max())), name=f"{name} job {j}: model-output")
    old = two_launch_route(engine, torch, spec, weights, X, a, b, y, jobs_h, scale, feat, agg, out_rows, variant, want=want)
    for k in OUTS:
        assert np.isnan(got[k][~written]).all(), f"{name}: {k} written outside the jobs' output rows"
        np.testing.assert_array_equal(_bits(got[k]), _bits(old[k]), err_msg=f"{name}: {k} against the two-launch route")
    return got


def machines_case(engine, torch, dims, variant, R=200, M=2, seed=0, acts=None):
    """M machines of R rows each over their own float64 rows, each slot with its own scaler."""
    acts = acts or ["tanh"] * (len(dims) - 2) + ["linear"]
    nets = [dense_net(km, dims, acts, seed + 10 + s) for s in range(M)]
    spec = nets[0][0]
    rng = np.random.default_rng(seed)
    X, a, b = x64_inputs(rng, M * R, dims[0], M)
    y = (rng.random((M * R, dims[-1])) * 2 - 0.5).astype(np.float32)
    scale, feat, agg = score_inputs(rng, M, dims[-1])
    x64_case(engine, torch, spec, [w for _, w in nets], X, a, b, y, engine.uniform_jobs(M, R), scale, feat, agg, M * R, variant,
             f"{dims} variant {variant}")


# ------------------------------------------------------------------------------------------------ generic kernel (variant 1)
GENERIC = {**{f"rows{r}_resident{res}": PLAN_SHAPES[(r, res)] for r, res in PLAN_SHAPES}, "column_blocked_0": COLUMN_BLOCKED[0],
           "column_blocked_1": COLUMN_BLOCKED[1], "symmetric170": None, "n_in_30": [30, 40, 30]}


@pytest.mark.parametrize("case", list(GENERIC))
def test_generic_kernel_every_plan(engine, torch, lib, case):
    """Every row-tile plan of the generic kernel with float64 x, the 170-tag feedforward_symmetric default, and an n_in that is not
    a multiple of 4 (x' is loaded element by element and zero padded to the layer's padded width)."""
    dims = km.ff_symmetric_spec(170).dims if case == "symmetric170" else GENERIC[case]
    if case.startswith("rows") or case.startswith("column"):
        assert instantiation(lib, dims, 1).startswith("generic")
    machines_case(engine, torch, dims, 1, R=300 if dims[0] <= 64 else 150, seed=len(dims) + dims[0])


# ------------------------------------------------------------------------------------------------ row per thread (variant 3)
@pytest.mark.parametrize("T,width", [(1, 4), (4, 4), (5, 8), (8, 8), (16, 16)])
def test_row_per_thread_every_width(engine, torch, lib, T, width):
    dims = km.ff_hourglass_spec(T).dims
    assert instantiation(lib, dims, 3) == f"small-w{width}"
    machines_case(engine, torch, dims, 3, R=300, seed=T)


# ------------------------------------------------------------------------------------------------ tensor cores (variant 2)
TC_STACKS = {**{f"hourglass{T}": None for T in range(24, 65, 4)},
             **{"-".join(map(str, d)): d for d in ([48, 12, 48], [48, 16, 48], [48, 32, 48], [48, 48, 48], [48, 64, 48],
                                                   [40, 64, 48, 12, 16, 32, 40], [64, 16, 32, 48, 64, 64, 64], [64] * 7)}}


@pytest.mark.parametrize("case", list(TC_STACKS))
def test_tensor_core_stacks(engine, torch, lib, case):
    """Every hourglass of 24..64 tags (28, 36, 44, 52, 60 end inside a 16-column float64 box; 56 | 60 is the warpgroup boundary),
    hidden layers wider than T and deep stacks, and [64] * 7 (two warpgroups restaging 64 x 64 layers, the largest batch)."""
    dims = km.ff_hourglass_spec(int(case[9:])).dims if case.startswith("hourglass") else TC_STACKS[case]
    nwg = 2 if (dims[0] > 56 and case.startswith("hourglass")) or dims == [64] * 7 else 3
    assert plan_x64(lib, dims, variant=2) == (0, 2, nwg)
    machines_case(engine, torch, dims, 2, R=200, seed=len(dims) * 100 + dims[0])


# ------------------------------------------------------------------------------------------------ job layouts
LAYOUTS = {"generic": (1, LAYOUT_SPECS[1]), "row_per_thread": (3, LAYOUT_SPECS[3]), "tc_nwg3": (2, LAYOUT_SPECS[2]),
           "tc_nwg2": (2, km.ff_hourglass_spec(64).dims)}


@pytest.mark.parametrize("case", list(LAYOUTS))
def test_job_layouts(engine, torch, lib, case):
    """Jobs of different slots over the same x rows in slot order 2, 0, 2, 1, 0, 1 (a persistent tensor-core CTA restages the slot's
    scaler whenever the slot changes), an empty job, x_row off any tile boundary, outputs anywhere in a longer NaN-filled array."""
    variant, dims = LAYOUTS[case]
    if variant == 2:
            assert plan_x64(lib, dims, variant=2)[2] == int(case[-1])
    acts = ["tanh"] * (len(dims) - 2) + ["linear"]
    nets = [dense_net(km, dims, acts, 40 + s) for s in range(3)]
    rng = np.random.default_rng(11)
    X, a, b = x64_inputs(rng, 500, dims[0], 3)
    y = rng.random((500, dims[-1])).astype(np.float32)
    scale, feat, agg = score_inputs(rng, 3, dims[-1])
    x64_case(engine, torch, nets[0][0], [w for _, w in nets], X, a, b, y, layout_jobs(engine), scale, feat, agg, 1400, variant, case)


@pytest.mark.parametrize("nwg", [3, 2])
def test_tensor_core_jobs_at_the_end_of_x(engine, torch, nwg):
    """The last job ends on the last row of an x of 333 rows (not a multiple of the 128-row tile pair), and an x of 5 rows, less
    than one tile: the rows TMA zero-fills past the end of x are never stored."""
    dims = km.ff_hourglass_spec(32 if nwg == 3 else 64).dims
    acts = ["tanh"] * (len(dims) - 2) + ["linear"]
    nets = [dense_net(km, dims, acts, 60 + s) for s in range(2)]
    rng = np.random.default_rng(12)
    for n_x, jobs in ((333, engine.make_jobs([0, 1, 0], [130, 200, 1], [0, 133, 332], [0, 131, 331])),
                      (5, engine.make_jobs([1, 0], [5, 3], [0, 2], [3, 9]))):
        X, a, b = x64_inputs(rng, n_x, dims[0], 2)
        y = rng.random((n_x, dims[-1])).astype(np.float32)
        scale, feat, agg = score_inputs(rng, 2, dims[-1])
        out_rows = int((jobs["out_row"] + jobs["n_rows"]).max()) + 2
        x64_case(engine, torch, nets[0][0], [w for _, w in nets], X, a, b, y, jobs, scale, feat, agg, out_rows, 2, f"nwg {nwg}, {n_x} rows of x")


@pytest.mark.parametrize("nwg", [3, 2])
def test_tensor_core_output_subsets(engine, torch, nwg):
    """Each score output alone, and the prediction alone without y: the outputs nobody asked for stay NaN."""
    dims = km.ff_hourglass_spec(32 if nwg == 3 else 64).dims
    acts = ["tanh"] * (len(dims) - 2) + ["linear"]
    nets = [dense_net(km, dims, acts, 70 + s) for s in range(2)]
    rng = np.random.default_rng(13)
    X, a, b = x64_inputs(rng, 330, dims[0], 2)
    y = rng.random((330, dims[-1])).astype(np.float32)
    scale, feat, agg = score_inputs(rng, 2, dims[-1])
    jobs = engine.make_jobs([1, 0], [170, 160], [0, 170], [0, 170])
    w = [w for _, w in nets]
    full = x64_case(engine, torch, nets[0][0], w, X, a, b, y, jobs, scale, feat, agg, 330, 2, f"nwg {nwg}")
    for want in [(k,) for k in SCORE] + [()]:
        got = x64_case(engine, torch, nets[0][0], w, X, a, b, y if want else None, jobs, scale, feat, agg, 330, 2, f"nwg {nwg} {want}",
                       want=want)
        np.testing.assert_array_equal(_bits(got["model-output"]), _bits(full["model-output"]))
        for k in SCORE:
            if k in want:
                close(got[k], full[k], mag=0.0, rtol=1e-6, name=f"nwg {nwg}: {k}")
            else:
                assert np.isnan(got[k]).all(), f"nwg {nwg}: {k} written although only {want or 'the prediction'} was requested"


@pytest.mark.parametrize("variant", [1, 3])
def test_more_jobs_than_a_grid_dimension(engine, torch, variant):
    """65 540 one-row jobs of two slots, each with its own scaler: the launches that carry the job index on gridDim.y go out in
    several parts, and every part reads its jobs' scalers."""
    J = 65_540
    dims = [8, 6, 8]
    nets = [dense_net(km, dims, ["tanh", "linear"], 80 + s) for s in range(2)]
    spec = nets[0][0]
    rng = np.random.default_rng(14)
    X, a, b = x64_inputs(rng, J, 8, 2)
    y = rng.random((J, 8)).astype(np.float32)
    scale, feat, agg = score_inputs(rng, 2, 8)
    idx = np.arange(J, dtype=np.int64)
    jobs = engine.make_jobs(idx % 2, 1, idx, idx)
    got = run_dense(engine, torch, spec, [w for _, w in nets], X, y, jobs, scale, feat, agg, J, variant, x_affine=(a, b))
    torch.cuda.empty_cache()
    for j in (0, 65_534, 65_535, 65_536, J - 1):
        s = j % 2
        want_out = km.ff_forward(spec, nets[s][1], scaled(X[j:j + 1], a[s], b[s]), np.float64)
        check_dense(got, slice(j, j + 1), want_out, y[j:j + 1], scale[s], feat[s], agg[s], f"variant {variant} job {j}")


# ------------------------------------------------------------------------------------------------ detectors: sklearn's transform
def _scaler_chains():
    from sklearn.preprocessing import MaxAbsScaler, MinMaxScaler, RobustScaler, StandardScaler

    return {
        "minmax": ([MinMaxScaler()], None),
        "minmax_range": ([MinMaxScaler(feature_range=(-1, 2))], None),
        "standard_no_mean": ([StandardScaler(with_mean=False)], None),
        "standard_no_std": ([StandardScaler(with_std=False)], None),
        "standard_constant_column": ([StandardScaler()], "constant"),
        "robust_no_centering": ([RobustScaler(with_centering=False)], None),
        "robust_no_scaling": ([RobustScaler(with_scaling=False, quantile_range=(10, 90))], None),
        "maxabs_zero_column": ([MaxAbsScaler()], "zero"),
        "standard_minmax_maxabs": ([StandardScaler(), MinMaxScaler(feature_range=(-1, 1)), MaxAbsScaler()], None),
    }


# (kind, tags, kernel the detector scores on)
DETECTOR_KINDS = {"tc": ("feedforward_hourglass", 32, 2), "row_per_thread": ("feedforward_hourglass", 8, 3),
                  "generic": ("feedforward_symmetric", 24, 1)}


def _frame(rows, tags, seed, column=None):
    rng = np.random.default_rng(seed)
    idx = pd.date_range("2020-01-01", periods=rows, freq="10min")
    v = 1e4 + rng.standard_normal((rows, tags)) * rng.uniform(0.1, 5.0, tags)
    if column == "constant":
        v[:, 2] = 1e4 + 3.0
    elif column == "zero":
        v[:, 2] = 0.0
    return pd.DataFrame(v, index=idx, columns=[f"tag-{i}" for i in range(tags)])


@pytest.mark.parametrize("kind", list(DETECTOR_KINDS))
@pytest.mark.parametrize("chain", list(_scaler_chains()))
def test_detector_scores_sklearns_own_pipeline_transform(engine, torch, monkeypatch, chain, kind):
    """DiffBasedAnomalyDetector(Pipeline([*scalers, KerasAutoEncoder])) on float64 frames near 1e4: the anomaly frame against the
    float64 oracle fed with ``Pipeline[:-1].transform(X)`` -- sklearn's scalers, not the composed (a, b) the kernels use."""
    from sklearn.pipeline import Pipeline

    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector, _scaler_multiplier
    from gordo_components_b200.machine.model.models import KerasAutoEncoder
    scalers, column = _scaler_chains()[chain]
    model, T, kernel = DETECTOR_KINDS[kind]
    X = _frame(300, T, T, column)
    steps = [(f"s{i}", s) for i, s in enumerate(scalers)] + [("ae", KerasAutoEncoder(kind=model, epochs=1))]
    det = DiffBasedAnomalyDetector(base_estimator=Pipeline(steps)).fit(X, X)
    rng = np.random.default_rng(T)
    feat = rng.uniform(0.5, 2.0, T)
    det.feature_thresholds_, det.aggregate_threshold_ = pd.Series(feat, index=X.columns), 0.3
    ae = det.base_estimator.steps[-1][1]
    assert ae._engine().infer_plan_x64(0)[0] == kernel

    def fail(*a, **k):
        raise AssertionError("the Pipeline's scalers went through the separate affine pass")

    monkeypatch.setattr(engine, "affine_f64", fail)
    req = X.iloc[17:290]
    frame = det.anomaly(req, req)
    got = {k: frame[k].to_numpy() for k in OUTS}
    got = {k: v.ravel() if k in PER_ROW else v for k, v in got.items()}

    xt = np.asarray(det.base_estimator[:-1].transform(req), dtype=np.float64)
    spec = ae.model.spec
    want_out = km.ff_forward(km.FFSpec(list(spec.dims), list(spec.acts), list(spec.l1)), ae.model.weights, xt.astype(np.float32), np.float64)
    mult = _scaler_multiplier(det.scaler, T)
    check_dense(got, slice(None), want_out, req.to_numpy(), mult, feat, 0.3, f"{chain} {kind}")


# ------------------------------------------------------------------------------------------------ served
def test_served_symmetric_pipeline_bucket_answers_through_the_coalescer(engine, torch, tmp_path):
    """Four feedforward_symmetric Pipeline detectors with different scalers in one ResidentBucket(input_scalers=True): the generic
    kernel with float64 x under the coalescer, many slots and jobs a launch.  Replies from 8 threads, JSON and parquet, carry the
    bytes of the per-request route."""
    from gordo_components_b200 import builder, server
    from test_gpu_builder import _series

    N, T = 300, 24
    names = ["minmax", "standard", "robust", "maxabs"]
    scalers = {"minmax": "sklearn.preprocessing.MinMaxScaler", "standard": "sklearn.preprocessing.StandardScaler",
               "robust": "sklearn.preprocessing.RobustScaler", "maxabs": "sklearn.preprocessing.MaxAbsScaler"}

    def definition(scaler):
        return {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": {"sklearn.pipeline.Pipeline": {"steps": [
            scaler, {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_symmetric", "epochs": 1}}]}}}}

    frames = {n: _series(N, T, 20 + seed).astype(np.float64) * 300.0 + 1e4 for seed, n in enumerate(names)}
    builder.FleetModelBuilder([{"name": n, "model": definition(scalers[n]), "dataset": (frames[n], frames[n])} for n in names]).build(str(tmp_path))
    store = server.ModelStore(str(tmp_path))
    bucket = server.ResidentBucket(store, input_scalers=True, max_wait_ms=20.0)
    assert sorted(bucket.names) == sorted(names) and bucket.input_scalers
    spec = store.model("minmax").base_estimator.steps[-1][1].model.spec
    assert engine.FFEngine(spec.dims, spec.acts).infer_plan_x64(0) == (1, 0)

    reqs = []
    for i in range(48):
        n = names[i % 4]
        X = frames[n].iloc[5 + i: 5 + i + 50 + i % 9]
        if i % 3:
            reqs.append((n, {"json": json.loads(json.dumps({"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(X)}))}, None))
        else:
            reqs.append((n, {"files": {"X": server.dataframe_into_parquet_bytes(X), "y": server.dataframe_into_parquet_bytes(X)}}, "parquet"))
    want = [server.anomaly_prediction(store, n, fmt=fmt, **kw) for n, kw, fmt in reqs]
    got = [None] * len(reqs)

    def worker(k):
        for i in range(k, len(reqs), 8):
            n, kw, fmt = reqs[i]
            got[i] = server.anomaly_prediction(store, n, fmt=fmt, bucket=bucket, **kw)

    threads = [threading.Thread(target=worker, args=(k,)) for k in range(8)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    try:
        for (n, _, fmt), w, g in zip(reqs, want, got):
            assert g.status == w.status == 200
            if fmt == "parquet":
                assert g.body == w.body
            else:
                assert json.dumps(g.body["data"]) == json.dumps(w.body["data"])
        co = bucket.coalescer
        assert co.requests == len(reqs) and co.batches < co.requests
    finally:
        bucket.close()
