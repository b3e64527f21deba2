"""
Parity of the CUDA path (through the C ABI) against the CPU oracle and the reference-generated golden fixtures.

Tolerance (north_star: "within 1e-4 relative"): model output |got - want| <= 1e-4*|want| + 2e-5*magnitude, where the
second term covers outputs near zero (the split-precision tensor-core path measures ~2e-6 of the magnitude, so a
regression of its operand scheme shows); quantities formed by subtracting the target (abs diffs, their squares,
confidences) carry the same *absolute* uncertainty as the model output, so they are compared with
atol = 2e-5 * (magnitude of y) -- a relative bound on a difference of nearly equal numbers is not meaningful in
any float32 implementation, the reference's included.  The float64 kernels (foreign base estimators) are held to 1e-9.
"""
import os

import numpy as np
import pandas as pd
import pytest
from parity_helpers import close, random_net

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


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


def run_infer(engine, torch, spec, weights_per_slot, X, y, jobs_h, scale=None, feat=None, agg=None, out_rows=None, variant=0):
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)  # noqa: E731
    res = eng.infer_score(eng.pack_params(weights_per_slot), engine.jobs_to_device(jobs_h, dev), len(jobs_h), int(jobs_h["n_rows"].max()),
                          t(X), t(y), t(scale), t(feat), t(agg), out_rows=out_rows, variant=variant)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in res.items()}


# ------------------------------------------------------------------------------------------------ K1 + K4
@pytest.mark.parametrize("T,variant", [(4, 1), (8, 1), (10, 1), (64, 1), (64, 2), (128, 1), (4, 3), (8, 3), (10, 3), (16, 3), (8, 0), (48, 2), (36, 2), (24, 2), (60, 0)])  # 3: row-per-thread kernel; 2 with T < 64: zero-padded columns
def test_ffae_infer_score_matches_oracle(engine, torch, T, variant):
    """variant 1 = fp32 CUDA-core kernel (any architecture), variant 2 = tensor-core (wgmma) split-precision kernel (64-tag nets)."""
    from oracle import anomaly_math as am
    from oracle import keras_math as km

    M, R = 5, 333  # ragged against the 128-row tile
    rng = np.random.default_rng(T)
    nets = [random_net(km, T, 10 * T + m) for m in range(M)]
    spec = nets[0][0]
    X = (rng.random((M * R, T)) * 2 - 0.5).astype(np.float32)
    y = (X + rng.normal(0, 0.05, X.shape)).astype(np.float32)
    jobs = engine.uniform_jobs(M, R)
    scales = np.stack([am.minmax_fit(y[m * R:(m + 1) * R])[0] for m in range(M)]).astype(np.float32)
    feat = (rng.random((M, T)) * 0.2 + 0.05).astype(np.float32)
    agg = (rng.random(M) * 0.1 + 0.01).astype(np.float32)
    got = run_infer(engine, torch, spec, [w for _, w in nets], X, y, jobs, scales, feat, agg, variant=variant)
    for m in range(M):
        sl = slice(m * R, (m + 1) * R)
        want_out = km.ff_forward(spec, nets[m][1], X[sl], dtype=np.float64)
        sc, mn = am.minmax_fit(y[sl])
        want = am.anomaly_arrays(want_out, y[sl], scales[m].astype(np.float64), mn, feat[m], float(agg[m]))
        close(got["model-output"][sl], want_out, 1.0, name="model-output")
        close(got["tag-anomaly-unscaled"][sl], want["tag-anomaly-unscaled"], 1.0, name="tag-anomaly-unscaled")
        close(got["tag-anomaly-scaled"][sl], want["tag-anomaly-scaled"], float(scales[m].max()), name="tag-anomaly-scaled")
        close(got["total-anomaly-unscaled"][sl], want["total-anomaly-unscaled"], 1.0 * np.sqrt(want["total-anomaly-unscaled"].max()), name="total-unscaled")
        close(got["total-anomaly-scaled"][sl], want["total-anomaly-scaled"], float(scales[m].max()) * np.sqrt(want["total-anomaly-scaled"].max()), name="total-scaled")
        close(got["anomaly-confidence"][sl], want["anomaly-confidence"], float((1 / feat[m]).max()), name="confidence")
        close(got["total-anomaly-confidence"][sl], want["total-anomaly-confidence"], float(scales[m].max()) * np.sqrt(want["total-anomaly-scaled"].max()) / float(agg[m]), name="total-confidence")


@pytest.mark.parametrize("T", [10, 64])
def test_wide_symmetric_stack_defaults(engine, torch, T):
    """feedforward_symmetric / feedforward_model default to 256-128-64 encoders (feedforward_autoencoder.py:19,111): wider than the
    resident-weight budget, so inference stages layer by layer with a smaller row tile and fit keeps the weight image in L2."""
    from gordo_components_b200.machine.model.models import KerasAutoEncoder
    from oracle import keras_math as km

    spec = km.ff_symmetric_spec(T)
    assert max(spec.dims) == 256
    rng = np.random.default_rng(T)
    w = km.init_ff_weights(spec, rng)
    w = [(W, rng.uniform(-0.1, 0.1, b.shape).astype(np.float32)) for W, b in w]
    R = 300
    X = rng.random((R, T)).astype(np.float32)
    got = run_infer(engine, torch, spec, [w], X, X, engine.uniform_jobs(1, R), np.ones((1, T), np.float32), np.ones((1, T), np.float32), np.ones(1, np.float32))
    close(got["model-output"], km.ff_forward(spec, w, X, np.float64), 1.0, name="256-wide model output")
    # fit: same weights + visiting order => same trained weights as the oracle
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    perm = np.stack([[np.random.default_rng(e).permutation(R) for e in range(2)]]).astype(np.int32)
    params = eng.pack_params([w])
    xd = torch.from_numpy(X).to(dev)
    loss, acc, _ = eng.fit(params, engine.jobs_to_device(engine.uniform_jobs(1, R), dev), 1, R, xd, xd.clone(), epochs=2, batch_size=32, perm=torch.from_numpy(perm).to(dev))
    w_ref, hist, _ = km.ff_fit(spec, w, X, X, epochs=2, batch_size=32, perms=list(perm[0]))
    for (Wg, bg), (Wr, br) in zip(eng.unpack_params(params)[0], w_ref):
        close(Wg, Wr, mag=float(np.abs(Wr).max()), name="256-wide trained weights")
    close(loss[0].cpu().numpy(), np.array(hist["loss"]), mag=0.0, rtol=5e-4, name="loss history")
    # and through the estimator with the factory's defaults
    np.random.seed(0)
    m = KerasAutoEncoder(kind="feedforward_symmetric", epochs=2).fit(X, X)
    assert m.predict(X).shape == (R, T) and m.get_metadata()["history"]["loss"][1] < m.get_metadata()["history"]["loss"][0]


@pytest.mark.parametrize("cls_name,kind,kw", [
    ("KerasAutoEncoder", "feedforward_model", {}), ("KerasAutoEncoder", "feedforward_symmetric", {}), ("KerasAutoEncoder", "feedforward_hourglass", {}),
    ("KerasLSTMAutoEncoder", "lstm_model", {"lookback_window": 3}), ("KerasLSTMAutoEncoder", "lstm_symmetric", {"lookback_window": 3}),
    ("KerasLSTMForecast", "lstm_hourglass", {"lookback_window": 3}), ("KerasLSTMAutoEncoder", "lstm_symmetric", {})])
def test_every_registered_factory_with_its_defaults(engine, torch, cls_name, kind, kw):
    """Every `kind` the reference registers (register.py:10-75; factories' default dims are 256-128-64) builds, trains and
    predicts with its default arguments; the trained weights reproduce the prediction in the oracle."""
    from gordo_components_b200.machine.model import models
    from oracle import keras_math as km

    np.random.seed(2)
    X = np.random.random((60, 5)).astype(np.float32)
    m = getattr(models, cls_name)(kind=kind, epochs=1, **kw).fit(X, X)
    out = m.predict(X)
    L = kw.get("lookback_window", 1)
    assert out.shape == (60 - (L - 1 + m.lookahead if cls_name != "KerasAutoEncoder" else 0), 5) and np.isfinite(out).all()
    spec = m.model.spec
    if cls_name == "KerasAutoEncoder":
        want = km.ff_forward(km.FFSpec(list(spec.dims), list(spec.acts), list(spec.l1)), m.model.weights, X, np.float64)
    else:
        ospec = km.LSTMSpec(spec.n_features, list(spec.lstm_units), list(spec.acts), spec.n_features_out, spec.out_func, spec.lookback_window)
        want = km.lstm_predict(ospec, m.model.weights, X, lookahead=m.lookahead, dtype=np.float64)
    close(out, want, 1.0, rtol=2e-4, name=f"{kind} defaults")
    assert "loss" in m.get_metadata()["history"]


def test_tc_work_split_many_ragged_jobs(engine, torch):
    """More jobs than SMs with ragged lengths (whole-job waves + a split tail, empty tiles, jobs shorter than a tile): the tensor-core
    kernel against the generic fp32 kernel (itself checked against the oracle above) on every output."""
    from gordo_components_b200 import fleet
    from oracle import keras_math as km

    spec = km.ff_hourglass_spec(64)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    rng = np.random.default_rng(11)
    M = 333
    n_rows = rng.integers(1, 700, size=M)
    n_rows[[5, 77, 200]] = [1, 128, 129]
    x_rows = np.concatenate([[0], np.cumsum(n_rows)[:-1]])
    slots = rng.permutation(M)
    jobs = engine.jobs_to_device(engine.make_jobs(slots, n_rows, x_rows), dev)
    g = torch.Generator(device=dev).manual_seed(4)
    total = int(n_rows.sum())
    x = torch.rand((total, 64), generator=g, device=dev)
    y = x + 0.05 * torch.randn((total, 64), generator=g, device=dev)
    params = fleet.random_glorot_params(eng, M, g)
    scale = torch.rand((M, 64), generator=g, device=dev) + 0.5
    feat = torch.rand((M, 64), generator=g, device=dev) + 0.5
    agg = torch.rand((M,), generator=g, device=dev) + 0.5
    a = eng.infer_score(params, jobs, M, int(n_rows.max()), x, y, scale, feat, agg, variant=2)
    b = eng.infer_score(params, jobs, M, int(n_rows.max()), x, y, scale, feat, agg, variant=1)
    for k in b:
        close(a[k].cpu().numpy(), b[k].cpu().numpy(), mag=float(b[k].abs().max()), name=f"tensor cores vs fp32: {k}")


def test_more_jobs_than_a_grid_dimension(engine, torch):
    """70 000 four-row jobs (a 16 384-machine bucket with 3 CV folds is 65 536): the kernels that carry the job index on gridDim.y
    go out as several launches; every job still gets its own slot's answer."""
    from oracle import keras_math as km

    J, R, T = 70_000, 4, 8
    spec, w0 = random_net(km, T, 1)
    _, w1 = random_net(km, T, 2)
    rng = np.random.default_rng(0)
    X = rng.random((J * R, T)).astype(np.float32)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    params = eng.pack_params([w0, w1])
    slots = (np.arange(J) % 2).astype(np.int32)
    jobs = engine.jobs_to_device(engine.make_jobs(slots, R, np.arange(J, dtype=np.int64) * R), dev)
    xd = torch.from_numpy(X).to(dev)
    scale = torch.ones((2, T), device=dev)
    for variant in (1, 3):  # generic fp32 kernel, row-per-thread kernel
        res = eng.infer_score(params, jobs, J, R, xd, xd, scale, variant=variant)
        out = res["model-output"].cpu().numpy().reshape(J, R, T)
        for j in (0, 1, 65534, 65535, 65536, J - 1):
            close(out[j], km.ff_forward(spec, (w0, w1)[j % 2], X[j * R:(j + 1) * R], dtype=np.float64), 1.0, name=f"variant {variant} job {j}")
    feat, agg = engine.thresholds(jobs, J, R, res["tag-anomaly-unscaled"], res["total-anomaly-scaled"], T, 2, 2, dev)
    # rolling(2).min().max() of every job, merged per slot over the jobs on both sides of the launch split
    roll = lambda a: np.minimum(a[:, 1:], a[:, :-1]).max(axis=1)  # noqa: E731
    tu = res["tag-anomaly-unscaled"].cpu().numpy().reshape(J, R, T)
    ts = res["total-anomaly-scaled"].cpu().numpy().reshape(J, R, 1)
    np.testing.assert_array_equal(feat.cpu().numpy(), np.stack([roll(tu[s::2]).max(axis=0) for s in (0, 1)]))
    np.testing.assert_array_equal(agg.cpu().numpy(), np.stack([roll(ts[s::2]).max(axis=0) for s in (0, 1)]).ravel())
    lo_hi = engine.minmax_fit(jobs, J, R, xd, T, 2, dev, return_minmax=True)
    np.testing.assert_array_equal(lo_hi[2][0].cpu().numpy(), X.reshape(J, R, T)[0::2].min(axis=(0, 1)))


def test_ffae_jobs_slots_and_row_offsets(engine, torch):
    """Jobs may share a slot, read any row range and write anywhere; empty jobs are no-ops; predict-only mode."""
    from oracle import keras_math as km

    T = 8
    nets = [random_net(km, T, s) for s in (1, 2)]
    spec = nets[0][0]
    X = np.random.default_rng(0).random((1000, T)).astype(np.float32)
    jobs = engine.make_jobs([1, 0, 1, 0], [130, 1, 0, 257], [700, 5, 0, 100], [0, 130, 131, 131])
    got = run_infer(engine, torch, spec, [w for _, w in nets], X, None, jobs, out_rows=131 + 257)
    out = got["model-output"]
    close(out[:130], km.ff_forward(spec, nets[1][1], X[700:830], np.float64), name="job0")
    close(out[130:131], km.ff_forward(spec, nets[0][1], X[5:6], np.float64), name="job1")
    close(out[131:388], km.ff_forward(spec, nets[0][1], X[100:357], np.float64), name="job3")
    assert set(got) == {"model-output"}


@pytest.mark.parametrize("dims,acts", [([6, 5, 3, 7], ["relu", "sigmoid", "linear"]), ([33, 17, 33], ["tanh", "tanh"]), ([5, 9, 2], ["sigmoid", "relu"])])
def test_ffae_generic_architectures(engine, torch, dims, acts):
    """feedforward_model / feedforward_symmetric with arbitrary widths, activations and n_features_out != n_features."""
    from oracle import keras_math as km

    spec, w = random_net(km, dims, 3, acts)
    rng = np.random.default_rng(1)
    X = rng.random((200, dims[0])).astype(np.float32)
    y = rng.random((200, dims[-1])).astype(np.float32)
    sc = np.ones((1, dims[-1]), np.float32)
    got = run_infer(engine, torch, spec, [w], X, y, engine.uniform_jobs(1, 200), sc)
    want = km.ff_forward(spec, w, X, np.float64)
    close(got["model-output"], want, name="out")
    close(got["tag-anomaly-unscaled"], np.abs(want - y), name="tu")
    close(got["total-anomaly-scaled"], ((want - y) ** 2).mean(axis=1), name="tot")


@pytest.mark.parametrize("case", ["ffnet_anomaly", "ffnet_anomaly_t64"])
def test_ffae_against_reference_generated_fixture(engine, torch, case):
    """Fixture columns were produced by the reference's own diff.py (tests/golden/make_golden.py)."""
    from oracle import keras_math as km

    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    dims = [int(d) for d in g["net_dims"]]
    spec = km.ff_hourglass_spec(dims[0])
    w = [(g[f"W{l}"], g[f"b{l}"]) for l in range(spec.n_layers)]
    X, y = g["X"], g["y"]
    got = run_infer(engine, torch, spec, [w], X, y, engine.uniform_jobs(1, len(X)), g["scale"][None], g["feature_thresholds"][None],
                    np.array([float(g["aggregate_threshold"])]))
    smax = float(g["scale"].max())
    close(got["model-output"], g["frame_model-output"], name="model-output")
    close(got["tag-anomaly-unscaled"], g["frame_tag-anomaly-unscaled"], name="tag-anomaly-unscaled")
    close(got["tag-anomaly-scaled"], g["frame_tag-anomaly-scaled"], smax, name="tag-anomaly-scaled")
    close(got["total-anomaly-scaled"], g["frame_total-anomaly-scaled"].ravel(), smax * np.sqrt(g["frame_total-anomaly-scaled"].max()), name="total-scaled")
    close(got["total-anomaly-unscaled"], g["frame_total-anomaly-unscaled"].ravel(), np.sqrt(g["frame_total-anomaly-unscaled"].max()), name="total-unscaled")
    close(got["anomaly-confidence"], g["frame_anomaly-confidence"], float((1 / g["feature_thresholds"]).max()), name="confidence")
    close(got["total-anomaly-confidence"], g["frame_total-anomaly-confidence"].ravel(),
          smax * np.sqrt(g["frame_total-anomaly-scaled"].max()) / float(g["aggregate_threshold"]), name="total-confidence")


# ------------------------------------------------------------------------------------------------ K7, K5, K4-alone
def test_minmax_and_thresholds_against_reference_fixture(engine, torch):
    dev = engine.cuda_device()
    for case in ("anomaly_plain", "anomaly_smm", "ffnet_anomaly"):
        g = np.load(os.path.join(GOLDEN, case + ".npz"))
        y = np.ascontiguousarray(g["y"], dtype=np.float32)  # DataFrame.values saved by the generator is F-ordered
        n, T = y.shape
        yd = torch.from_numpy(y).to(dev)
        # per-fold scalers are fitted on the fold's training rows [0, test_start)
        starts = [int(g[f"fold{i}_test_start"]) for i in range(3)]
        jobs_h = engine.make_jobs([0, 1, 2, 3], starts + [n], [0, 0, 0, 0])
        scale, offset = engine.minmax_fit(engine.jobs_to_device(jobs_h, dev), 4, n, yd, T, 4, dev)
        scale, offset = scale.cpu().numpy(), offset.cpu().numpy()
        for i in range(3):
            close(scale[i], g[f"fold{i}_scale"], rtol=1e-5, mag=0, name="fold scale")
            close(offset[i], g[f"fold{i}_min"], rtol=1e-5, mag=1e-2, name="fold min_")
        close(scale[3], g["scale"], rtol=1e-5, mag=0, name="scale_")
        # thresholds of every fold from the fixture's fold predictions
        tlen = int(g["fold0_test_len"])
        pred = np.ascontiguousarray(np.concatenate([g[f"fold{i}_pred"] for i in range(3)]), dtype=np.float32)
        ytest = np.ascontiguousarray(np.concatenate([y[starts[i]: starts[i] + tlen] for i in range(3)]))
        jobs_h = engine.make_jobs([0, 1, 2], [tlen] * 3, [0, tlen, 2 * tlen])
        jd = engine.jobs_to_device(jobs_h, dev)
        res = engine.anomaly_score(jd, 3, tlen, torch.from_numpy(pred).to(dev), torch.from_numpy(ytest).to(dev), T,
                                   torch.from_numpy(scale[:3].copy()).to(dev), want=("tag-anomaly-unscaled", "total-anomaly-scaled"))
        for window, fkey, akey in ((6, "feature_thresholds_per_fold", "aggregate_thresholds_per_fold"),):
            feat, agg = engine.thresholds(jd, 3, tlen, res["tag-anomaly-unscaled"], res["total-anomaly-scaled"], T, 3, window, dev)
            close(feat.cpu().numpy(), g[fkey], rtol=2e-5, mag=1e-3, name=f"{case} feature thresholds")
            close(agg.cpu().numpy(), g[akey], rtol=1e-4, mag=1e-4, name=f"{case} aggregate thresholds")
        if int(g["window"]) > 0:
            feat, agg = engine.thresholds(jd, 3, tlen, res["tag-anomaly-unscaled"], res["total-anomaly-scaled"], T, 3, int(g["window"]), dev)
            close(feat.cpu().numpy()[2], g["smooth_feature_thresholds"], rtol=2e-5, mag=1e-3, name="smooth feature thresholds")
            close(agg.cpu().numpy()[2], g["smooth_aggregate_threshold"], rtol=1e-4, mag=1e-4, name="smooth aggregate threshold")


def test_thresholds_edge_cases(engine, torch):
    from oracle import anomaly_math as am

    dev = engine.cuda_device()
    rng = np.random.default_rng(5)
    T = 7
    # three jobs: long (crosses the 1024-row chunk), exactly the window, shorter than the window (-> NaN)
    lens = [2300, 6, 4]
    tu = rng.random((sum(lens), T)).astype(np.float32)
    ts = rng.random(sum(lens)).astype(np.float32)
    starts = np.cumsum([0] + lens[:-1])
    jobs = engine.make_jobs([0, 1, 2], lens, starts)
    feat, agg = engine.thresholds(engine.jobs_to_device(jobs, dev), 3, max(lens), torch.from_numpy(tu).to(dev), torch.from_numpy(ts).to(dev), T, 3, 6, dev)
    feat, agg = feat.cpu().numpy(), agg.cpu().numpy()
    for i, (s, n) in enumerate(zip(starts, lens)):
        want_f = am.rolling_min_then_max(tu[s:s + n], 6)
        want_a = am.rolling_min_then_max(ts[s:s + n], 6)
        np.testing.assert_array_equal(feat[i], want_f.astype(np.float32))  # min/max of float32 values is exact
        np.testing.assert_array_equal(agg[i], np.float32(want_a))
    assert np.isnan(feat[2]).all() and np.isnan(agg[2])


def test_float64_score_thresholds_and_extrema(engine, torch):
    """
    gb_anomaly_score_f64 / gb_thresholds_f64 / gb_minmax_f64 against NumPy float64 at data magnitude ~100 with residuals of ~1e-3,
    where a float32 |yhat - y| is off by percents (diff.py:268-300, 350-385 are float64 in the reference).  Two ragged jobs.
    """
    from oracle import anomaly_math as am

    dev = engine.cuda_device()
    rng = np.random.default_rng(11)
    T, lens = 9, [1500, 37]
    n = sum(lens)
    y = 100.0 + rng.random((n, T))
    y[5, 2] = np.nan
    yhat = y + rng.normal(0, 1e-3, (n, T))
    starts = np.cumsum([0] + lens[:-1])
    jobs = engine.jobs_to_device(engine.make_jobs([0, 1], lens, starts), dev)
    lo, hi = engine.minmax_f64(jobs, 2, max(lens), torch.from_numpy(y).to(dev), 2)
    for i, (s, m) in enumerate(zip(starts, lens)):
        np.testing.assert_array_equal(lo[i].cpu().numpy(), np.nanmin(y[s:s + m], axis=0))
        np.testing.assert_array_equal(hi[i].cpu().numpy(), np.nanmax(y[s:s + m], axis=0))
    scale = 1.0 / (hi - lo)
    feat = torch.from_numpy(rng.random((2, T)) * 1e-3 + 1e-4).to(dev)
    agg = torch.from_numpy(rng.random(2) * 1e-6 + 1e-7).to(dev)
    res = engine.anomaly_score(jobs, 2, max(lens), torch.from_numpy(yhat).to(dev), torch.from_numpy(y).to(dev), T, scale, feat, agg)
    assert all(v.dtype == torch.float64 for v in res.values())
    f_thr, a_thr = engine.thresholds(jobs, 2, max(lens), res["tag-anomaly-unscaled"], res["total-anomaly-scaled"], T, 2, 6, dev)
    res = {k: v.cpu().numpy() for k, v in res.items()}
    sc, ft, at = scale.cpu().numpy(), feat.cpu().numpy(), agg.cpu().numpy()
    for i, (s, m) in enumerate(zip(starts, lens)):
        sl = slice(s, s + m)
        d = np.abs(yhat[sl] - y[sl])
        np.testing.assert_array_equal(res["tag-anomaly-unscaled"][sl], d)
        np.testing.assert_array_equal(res["tag-anomaly-scaled"][sl], d * sc[i])
        np.testing.assert_allclose(res["total-anomaly-unscaled"][sl], (d ** 2).mean(axis=1), rtol=1e-13)
        np.testing.assert_allclose(res["total-anomaly-scaled"][sl], ((d * sc[i]) ** 2).mean(axis=1), rtol=1e-13)
        np.testing.assert_array_equal(res["anomaly-confidence"][sl], d / ft[i])
        np.testing.assert_allclose(res["total-anomaly-confidence"][sl], ((d * sc[i]) ** 2).mean(axis=1) / at[i], rtol=1e-13)
        np.testing.assert_array_equal(f_thr[i].cpu().numpy(), am.rolling_min_then_max(res["tag-anomaly-unscaled"][sl], 6))
        np.testing.assert_array_equal(float(a_thr[i]), am.rolling_min_then_max(res["total-anomaly-scaled"][sl], 6))
    # the float32 route on the same data shows why the float64 one exists
    r32 = engine.anomaly_score(jobs, 2, max(lens), torch.from_numpy(yhat.astype(np.float32)).to(dev), torch.from_numpy(y.astype(np.float32)).to(dev), T,
                               want=("tag-anomaly-unscaled",))["tag-anomaly-unscaled"].cpu().numpy()
    rel = np.abs(r32[:lens[0]] - res["tag-anomaly-unscaled"][:lens[0]]) / np.maximum(res["tag-anomaly-unscaled"][:lens[0]], 1e-12)
    assert np.nanmax(rel) > 1e-3


@pytest.mark.parametrize("case", ["anomaly_smm", "anomaly_sma", "anomaly_ewma"])
def test_smoothing_against_reference_fixture(engine, torch, case):
    """smooth-* columns of the reference frame (pandas rolling median / mean / ewm) from its own unsmoothed columns."""
    g = np.load(os.path.join(GOLDEN, case + ".npz"))
    dev = engine.cuda_device()
    window, method = int(g["window"]), str(g["method"])
    for top in ("tag-anomaly-scaled", "total-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-unscaled"):
        src = np.ascontiguousarray(g[f"frame_{top}"], dtype=np.float32)
        if src.ndim == 2 and src.shape[1] == 1:
            src = src.reshape(-1)
        a = torch.from_numpy(src).to(dev)
        jobs = engine.jobs_to_device(engine.make_jobs([0], [len(src)], [0]), dev)
        got = engine.smooth(jobs, 1, a, window, method).cpu().numpy()
        want = g[f"frame_smooth-{top}"].reshape(got.shape)
        assert np.array_equal(np.isnan(got), np.isnan(want)), top
        close(got, want, float(np.nanmax(np.abs(want))), rtol=1e-5, name=f"{case} smooth-{top}")


@pytest.mark.parametrize("method", ["smm", "sma", "ewma"])
def test_smoothing_with_interior_nans_matches_pandas(engine, torch, method):
    """
    Missing sensor values reach the smoothing kernels through requests (the reference tolerates them): pandas' semantics are a NaN
    window for rolling median / mean while the NaN is inside, and for ewm (adjust=True, ignore_na=False) no observation, aged weights
    and the previous average carried forward.  Two ragged jobs crossing the 128-row chunk boundary, even and odd windows, a window
    longer than a job, a wide window (fewer columns per CTA).
    """
    dev = engine.cuda_device()
    rng = np.random.default_rng(17)
    lens = [700, 45]
    n, cols = sum(lens), 5
    a = rng.random((n, cols)).astype(np.float32)
    a[[3, 130, 131, 400, 699, 710], 1] = np.nan      # interior NaNs, one at a job's last row
    a[:7, 2] = np.nan                                # leading NaNs
    a[100:260, 3] = np.nan                           # a gap longer than the window
    a[:, 4] = np.nan                                 # nothing but NaNs
    starts = np.cumsum([0] + lens[:-1])
    jobs = engine.jobs_to_device(engine.make_jobs([0, 1], lens, starts), dev)
    for window in ((6, 13, 144, 1000) if method != "smm" else (6, 13, 144, 900)):
        got = engine.smooth(jobs, 2, torch.from_numpy(a).to(dev), window, method, max_rows=max(lens)).cpu().numpy()
        for s0, m in zip(starts, lens):
            frame = pd.DataFrame(a[s0:s0 + m].astype(np.float64))
            want = {"smm": lambda: frame.rolling(window).median(), "sma": lambda: frame.rolling(window).mean(), "ewma": lambda: frame.ewm(span=window).mean()}[method]().values
            assert np.array_equal(np.isnan(got[s0:s0 + m]), np.isnan(want)), (method, window)
            np.testing.assert_allclose(got[s0:s0 + m], want, rtol=2e-6, atol=1e-7, err_msg=f"{method} window {window}")


def test_detector_with_window_like_reference_tests(engine, torch):
    """test_anomaly_detectors.py:123-371: window/smoothing_method add four smooth-* blocks with window-1 leading NaNs."""
    from sklearn.linear_model import LinearRegression
    from sklearn.multioutput import MultiOutputRegressor

    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector

    g = np.load(os.path.join(GOLDEN, "anomaly_sma.npz"))
    X, y = pd.DataFrame(np.ascontiguousarray(g["X"])), pd.DataFrame(np.ascontiguousarray(g["y"]))
    model = DiffBasedAnomalyDetector(base_estimator=MultiOutputRegressor(LinearRegression()), window=12, smoothing_method="sma")
    model.cross_validate(X=X, y=y)
    model.fit(X, y)
    frame = model.anomaly(X, y)
    level0 = list(dict.fromkeys(frame.columns.get_level_values(0)))
    assert level0 == [str(c) for c in g["columns_level0"]]
    for top in level0[2:]:
        want = g[f"frame_{top}"]
        got = frame[top].values.reshape(want.shape)
        close(got, want, float(np.nanmax(np.abs(want))), name=top)
    assert frame["smooth-total-anomaly-scaled"].isna().sum() == 11
    close(model.smooth_feature_thresholds_.values, g["smooth_feature_thresholds"], rtol=1e-4, mag=1e-4, name="smooth thresholds")
    md = model.get_metadata()
    assert md["window"] == 12 and md["smoothing-method"] == "sma" and "smooth-feature-thresholds" in md


# ------------------------------------------------------------------------------------------------ K2
@pytest.mark.parametrize("T,batch", [(8, 32), (64, 32), (10, 7), (64, 128), (8, 50), (64, 33), (128, 32), (128, 48)])  # batch > 32: gradient sums over 32-row chunks; 128 tags: weight image in L2
def test_ffae_fit_matches_oracle_adam(engine, torch, T, batch):
    """Same initial weights + same visiting order => same weights/loss as the oracle's Keras-style Adam loop."""
    from oracle import keras_math as km

    M, N, E = 3, 150, 2
    spec = km.ff_hourglass_spec(T)
    rng = np.random.default_rng(T)
    t = np.linspace(0, 12, N)[:, None]
    datas = [(0.5 + 0.35 * np.sin(t * rng.uniform(0.5, 2, T) + rng.uniform(0, 3, T)) + rng.normal(0, 0.02, (N, T))).astype(np.float32) for _ in range(M)]
    X = np.concatenate(datas)
    w0 = [km.init_ff_weights(spec, np.random.default_rng(50 + m)) for m in range(M)]
    perm = np.stack([[np.random.default_rng(1000 * m + e).permutation(N) for e in range(E)] for m in range(M)]).astype(np.int32)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    params = eng.pack_params(w0)
    xd = torch.from_numpy(X).to(dev)
    jobs = engine.jobs_to_device(engine.uniform_jobs(M, N), dev)
    loss, acc, _ = eng.fit(params, jobs, M, N, xd, xd.clone(), epochs=E, batch_size=batch, perm=torch.from_numpy(perm).to(dev))
    torch.cuda.synchronize()
    got = eng.unpack_params(params)
    loss, acc = loss.cpu().numpy(), acc.cpu().numpy()
    for m in range(M):
        w_ref, hist, _ = km.ff_fit(spec, w0[m], datas[m], datas[m], epochs=E, batch_size=batch, perms=list(perm[m]))
        for l, ((Wg, bg), (Wr, br)) in enumerate(zip(got[m], w_ref)):
            # weights moved by ~lr*steps = 1e-2; agreement to 1e-4 of the weight scale after 2 epochs of fp32 Adam
            close(Wg, Wr, mag=float(np.abs(Wr).max()), name=f"W{l}")
            close(bg, br, mag=max(float(np.abs(br).max()), 1e-2), name=f"b{l}")
        close(loss[m], np.array(hist["loss"]), mag=0.0, rtol=5e-4, name="loss history")
        close(acc[m], np.array(hist["accuracy"]), mag=0, rtol=0, atol=2.0 / N, name="accuracy history")
    assert (loss[:, -1] < loss[:, 0]).all()


def test_ffae_fit_shuffle_modes_and_reproducibility(engine, torch):
    from oracle import keras_math as km

    T, N = 8, 200
    spec = km.ff_hourglass_spec(T)
    X = np.random.default_rng(0).random((N, T)).astype(np.float32)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    xd = torch.from_numpy(X).to(dev)
    jobs = engine.jobs_to_device(engine.uniform_jobs(1, N), dev)
    w0 = km.init_ff_weights(spec, np.random.default_rng(1))

    def run(shuffle, seed):
        p = eng.pack_params([w0])
        loss, _, _ = eng.fit(p, jobs, 1, N, xd, xd, epochs=3, batch_size=32, shuffle=shuffle, seed=seed)
        torch.cuda.synchronize()
        return p.cpu().numpy(), loss.cpu().numpy()

    a, la = run(True, 7)
    b, lb = run(True, 7)
    c, _ = run(True, 8)
    np.testing.assert_array_equal(a, b)  # same seed -> bit-identical fit
    assert np.abs(a - c).max() > 0  # different visiting order
    # shuffle=False equals the oracle with the identity order
    d, ld = run(False, 0)
    w_ref, hist, _ = km.ff_fit(spec, w0, X, X, epochs=3, batch_size=32, shuffle=False)
    close(ld[0], np.array(hist["loss"]), mag=0, rtol=5e-4, name="loss")
    assert np.isfinite(la).all() and la[0, -1] < la[0, 0]


# ------------------------------------------------------------------------------------------------ K3
@pytest.mark.parametrize("F,units,lookback", [(3, [4, 3, 3, 4], 3), (10, [8, 7, 5, 5, 7, 8], 12), (128, [256, 128, 64, 64, 128, 256], 20)])
def test_lstm_infer_matches_oracle(engine, torch, F, units, lookback):
    from oracle import keras_math as km

    spec = km.LSTMSpec(F, units, ["tanh"] * len(units), F, "linear", lookback)
    M, N = 2, lookback + 37
    ws = [km.init_lstm_weights(spec, np.random.default_rng(20 + m)) for m in range(M)]
    X = np.random.default_rng(3).random((M * N, F)).astype(np.float32)
    eng = engine.LSTMEngine(F, units, spec.acts, F, "linear", lookback)
    dev = eng.device
    nwin = N - lookback + 1
    jobs_h = engine.make_jobs([0, 1], [nwin, nwin], [0, N], [0, nwin])
    out = eng.infer(eng.pack_params(ws), engine.jobs_to_device(jobs_h, dev), 2, nwin, torch.from_numpy(X).to(dev), 2 * nwin)
    torch.cuda.synchronize()
    out = out.cpu().numpy()
    for m in range(M):
        want = km.lstm_predict(spec, ws[m], X[m * N:(m + 1) * N], dtype=np.float64)
        assert want.shape == (nwin, F)
        close(out[m * nwin:(m + 1) * nwin], want, 1.0, name="lstm output")


@pytest.mark.parametrize("F,units,lookback,rows,scale", [(16, [64, 64], 5, [140, 300], 1.0), (128, [256, 128, 64, 64, 128, 256], 20, [57, 190], 1.0),
                                                          (7, [128], 9, [400], 1000.0), (5, [7, 9, 3], 4, [50, 133], 1.0),
                                                          (128, [107, 85, 64, 64, 85, 107], 12, [150], 1.0),  # widths padded to 64 internally
                                                          (128, [256, 128, 64, 64, 128, 256], 144, [144 + 39, 144 + 130], 1.0),  # BASELINE configs[3]: error growth over 144 steps
                                                          (4, [64, 64], 3, [19100, 18950], 1.0)])  # 150 + 149 tiles on 132 SMs: every CTA walks several items (the TMA ring wraps across items)
def test_lstm_infer_tcgen05_matches_oracle(engine, torch, F, units, lookback, rows, scale):
    """gb_lstm_infer_tc: FP16-pair split operands on the tensor cores, state in HBM, one launch per (layer, timestep).
    Jobs of different lengths (tiles with padding rows), machines sharing the launch, raw inputs of large magnitude (the
    input projection stays fp32), and the CUDA-core kernel as a second witness."""
    from oracle import keras_math as km

    spec = km.LSTMSpec(F, units, ["tanh"] * len(units), F, "linear", lookback)
    M = len(rows)
    rng = np.random.default_rng(9)
    ws = [km.init_lstm_weights(spec, np.random.default_rng(40 + m)) for m in range(M)]
    if scale != 1.0:  # keep the pre-activations sane for huge inputs: shrink the input kernel instead of the data
        ws = [([(K / scale if i == 0 else K, U, b) for i, (K, U, b) in enumerate(layers)], dense) for layers, dense in ws]
    Xs = [(rng.random((n, F)) * scale).astype(np.float32) for n in rows]
    eng = engine.LSTMEngine(F, units, spec.acts, F, "linear", lookback)
    assert eng.tc_supported
    dev = eng.device
    nwin = [n - lookback + 1 for n in rows]
    starts = np.concatenate([[0], np.cumsum(rows)[:-1]])
    outs = np.concatenate([[0], np.cumsum(nwin)[:-1]])
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(M), nwin, starts, outs), dev)
    x = torch.from_numpy(np.concatenate(Xs)).to(dev)
    params = eng.pack_params(ws)
    got_tc = eng.infer(params, jobs, M, max(nwin), x, sum(nwin), variant=2).cpu().numpy()
    got_fma = eng.infer(params, jobs, M, max(nwin), x, sum(nwin), variant=1).cpu().numpy()
    for m in range(M):
        want = km.lstm_predict(spec, ws[m], Xs[m], dtype=np.float64)
        close(got_tc[outs[m]:outs[m] + nwin[m]], want, 1.0, name="tensor-core lstm output")
        close(got_fma[outs[m]:outs[m] + nwin[m]], want, 1.0, name="fp32 lstm output")


# ------------------------------------------------------------------------------------------------ estimator API end to end
def test_detector_end_to_end_like_reference_tests(engine, torch):
    """tests/gordo/machine/model/anomaly/test_anomaly_detectors.py:28-120 with our KerasAutoEncoder as base estimator."""
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasAutoEncoder
    from oracle import anomaly_math as am
    from oracle import keras_math as km

    np.random.seed(0)
    n, T = 400, 8
    idx = pd.date_range("2019-01-01", periods=n, freq="10min", tz="UTC")
    t = np.linspace(0, 30, n)[:, None]
    Xv = 0.5 + 0.4 * np.sin(t * np.linspace(0.5, 2, T)) + np.random.normal(0, 0.02, (n, T))
    cols = [f"tag-{i}" for i in range(T)]
    X = pd.DataFrame(Xv, columns=cols, index=idx)
    y = X.copy()
    model = DiffBasedAnomalyDetector(base_estimator=KerasAutoEncoder(kind="feedforward_hourglass", epochs=3, batch_size=32))
    with pytest.raises(AttributeError):
        model.fit(X, y).anomaly(X, y)
    cvo = model.cross_validate(X=X, y=y)
    assert {"fit_time", "score_time", "estimator", "test_score"} <= set(cvo)
    assert len(model.feature_thresholds_) == T and model.feature_thresholds_per_fold_.shape == (3, T)
    assert list(model.aggregate_thresholds_per_fold_) == ["fold-0", "fold-1", "fold-2"]
    model.fit(X, y)
    frame = model.anomaly(X, y, frequency=pd.Timedelta("10min"))
    level0 = list(dict.fromkeys(frame.columns.get_level_values(0)))
    assert level0 == ["start", "end", "model-input", "model-output", "tag-anomaly-scaled", "total-anomaly-scaled", "tag-anomaly-unscaled",
                      "total-anomaly-unscaled", "anomaly-confidence", "total-anomaly-confidence"]
    # the frame equals the oracle's arithmetic applied to the oracle's forward of the trained weights
    ae = model.base_estimator
    spec = km.ff_hourglass_spec(T)
    pred = km.ff_forward(spec, ae.model.weights, Xv, np.float64)
    close(model.predict(X), pred, name="predict")
    sc, mn = am.minmax_fit(Xv)
    close(model.scaler.scale_, sc, rtol=1e-5, mag=0, name="scaler")
    want = am.anomaly_arrays(pred, Xv, sc, mn, model.feature_thresholds_.values, model.aggregate_threshold_)
    close(frame["model-output"].values, pred, name="model-output")
    close(frame["tag-anomaly-unscaled"].values, want["tag-anomaly-unscaled"], name="tag-anomaly-unscaled")
    close(frame["tag-anomaly-scaled"].values, want["tag-anomaly-scaled"], float(sc.max()), name="tag-anomaly-scaled")
    close(frame["anomaly-confidence"].values, want["anomaly-confidence"], float((1 / model.feature_thresholds_.values).max()), name="confidence")
    # thresholds re-derived by the oracle from the fold models the detector trained
    for i, ((tr, te), fold) in enumerate(zip(am.time_series_split(n, 3), cvo["estimator"])):
        fpred = km.ff_forward(spec, fold.base_estimator.model.weights, Xv[te], np.float64)
        fs, fm = am.minmax_fit(Xv[tr])
        ft, at = am.fold_thresholds(Xv[te], fpred, fs, fm, 6)
        close(model.feature_thresholds_per_fold_.values[i], ft, rtol=1e-3, mag=1e-4, name="fold feature thresholds")
        close(model.aggregate_thresholds_per_fold_[f"fold-{i}"], at, rtol=1e-3, mag=1e-5, name="fold aggregate threshold")
    md = model.get_metadata()
    assert {"feature-thresholds", "aggregate-threshold", "feature-thresholds-per-fold", "aggregate-thresholds-per-fold", "history"} <= set(md)
    assert {"loss", "accuracy", "params"} <= set(md["history"]) and len(md["history"]["loss"]) == 3
    # pickle round trip: identical predictions, history preserved (test_model.py:112-158)
    import pickle

    clone_ = pickle.loads(pickle.dumps(model))
    np.testing.assert_array_equal(clone_.predict(X), model.predict(X))
    assert clone_.base_estimator._history.history["loss"] == ae._history.history["loss"]


def test_detector_with_foreign_base_estimator(engine, torch):
    """The reference's detector tests drive it with sklearn regressors; the anomaly arithmetic still runs on the GPU."""
    from sklearn.linear_model import LinearRegression
    from sklearn.multioutput import MultiOutputRegressor
    from sklearn.preprocessing import RobustScaler

    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector

    g = np.load(os.path.join(GOLDEN, "anomaly_plain.npz"))
    X, y = pd.DataFrame(g["X"]), pd.DataFrame(g["y"])
    model = DiffBasedAnomalyDetector(base_estimator=MultiOutputRegressor(LinearRegression()))
    model.cross_validate(X=X, y=y)
    model.fit(X, y)
    frame = model.anomaly(X, y)
    # a foreign estimator's predictions are scored in float64 like the reference (gb_anomaly_score_f64 / gb_thresholds_f64)
    np.testing.assert_allclose(model.feature_thresholds_.values, g["feature_thresholds"], rtol=1e-9, atol=1e-13)
    np.testing.assert_allclose(model.aggregate_threshold_, g["aggregate_threshold"], rtol=1e-9, atol=1e-13)
    for top in ("model-output", "tag-anomaly-scaled", "total-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-unscaled",
                "anomaly-confidence", "total-anomaly-confidence"):
        want = g[f"frame_{top}"]
        got = frame[top].values
        np.testing.assert_allclose(got.reshape(want.shape), want, rtol=1e-9, atol=1e-13, err_msg=top)
    # RobustScaler (reference test parametrisation): slope = 1/scale_
    m2 = DiffBasedAnomalyDetector(base_estimator=MultiOutputRegressor(LinearRegression()), scaler=RobustScaler(), require_thresholds=False)
    f2 = m2.fit(X, y).anomaly(X, y)
    want = np.abs(m2.scaler.transform(m2.predict(X)) - m2.scaler.transform(y))
    np.testing.assert_allclose(f2["tag-anomaly-scaled"].values, want, rtol=1e-9, atol=1e-12, err_msg="robust scaled")
    assert "anomaly-confidence" not in f2.columns


def test_estimator_validation_split_and_score(engine, torch):
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    np.random.seed(1)
    X = np.random.random((300, 4))
    m = KerasAutoEncoder(kind="feedforward_hourglass", epochs=2, validation_split=0.2)
    m.fit(X, X)
    h = m.get_metadata()["history"]
    assert len(h["loss"]) == 2 and len(h["val_loss"]) == 2 and h["params"]["steps"] == 8
    assert m.predict(X).shape == (300, 4) and m.predict(X).dtype == np.float32
    assert isinstance(m.score(X, X), float)
    # seeded numpy => reproducible build (tests/gordo/builder/test_builder.py:658-707)
    np.random.seed(3)
    a = KerasAutoEncoder(kind="feedforward_hourglass", epochs=1).fit(X, X).predict(X)
    np.random.seed(3)
    b = KerasAutoEncoder(kind="feedforward_hourglass", epochs=1).fit(X, X).predict(X)
    np.testing.assert_array_equal(a, b)


def test_estimator_early_stopping_like_the_example_config(engine, torch):
    """test_anomaly_detectors.py:520-534 / test_model.py:341-361: epochs=1000 with EarlyStopping(val_loss, patience, restore_best_weights)
    stops long before, val_loss is the total loss (MSE + activity L1) on the held-out tail, and the best weights come back."""
    from gordo_components_b200.machine.model.models import KerasAutoEncoder
    from oracle import keras_math as km

    np.random.seed(5)
    t = np.linspace(0, 20, 400)[:, None]
    X = (0.5 + 0.4 * np.sin(t * np.linspace(0.5, 2, 6)) + np.random.normal(0, 0.05, (400, 6))).astype(np.float32)
    m = KerasAutoEncoder(kind="feedforward_hourglass", batch_size=128, epochs=1000, validation_split=0.1, compression_factor=0.5, encoding_layers=1,
                         callbacks=[{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "val_loss", "patience": 3, "restore_best_weights": True}}])
    m.fit(X, X)
    h = m.get_metadata()["history"]
    n = len(h["loss"])
    assert 4 <= n < 1000 and len(h["val_loss"]) == n and h["params"]["epochs"] == 1000
    best = int(np.argmin(h["val_loss"]))
    assert n - 1 - best == 3  # stopped `patience` epochs after the best one
    # the restored weights reproduce the best epoch's validation loss (oracle: total loss on the tail, one batch of 40 rows)
    spec = km.ff_hourglass_spec(6, encoding_layers=1)
    total, _mse, _g, _yh = km.ff_loss_and_grads(spec, m.model.weights, X[360:], X[360:], np.float64)
    close(float(total), h["val_loss"][best], rtol=2e-4, mag=0.0, name="restored best weights / val_loss semantics")


def test_lstm_estimator_predict_shapes(engine, torch):
    """tests/gordo/machine/model/test_model.py:324-338 and tests/gordo/builder/test_builder.py:99-115 (offsets)."""
    from gordo_components_b200.machine.model.models import KerasLSTMAutoEncoder, KerasLSTMForecast

    np.random.seed(0)
    m = KerasLSTMAutoEncoder(kind="lstm_model", lookback_window=3).initialize(3)
    assert m.predict(np.random.random((4, 3))).shape == (2, 3)
    f = KerasLSTMForecast(kind="lstm_hourglass", lookback_window=10).initialize(5)
    X = np.random.random((40, 5))
    assert len(X) - len(f.predict(X)) == 10
    a = KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=10).initialize(5)
    assert len(X) - len(a.predict(X)) == 9
    with pytest.raises(ValueError):
        a.predict(np.random.random((10, 5)))
    a.fit(X, X, epochs=2)
    assert a.get_metadata()["history"]["loss"][1] < a.get_metadata()["history"]["loss"][0]
    es = KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=10, epochs=50,
                              callbacks=[{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "loss", "patience": 1, "min_delta": 10.0}}])
    es.fit(X, X)  # no epoch can improve by 10: the first non-improving epoch after epoch 0 stops the training
    assert len(es.get_metadata()["history"]["loss"]) == 2 and es.get_metadata()["history"]["params"]["epochs"] == 50
    assert a.get_metadata()["forecast_steps"] == 0 and len(X) - len(a.predict(X)) == 9


@pytest.mark.parametrize("cls_name,offset", [("KerasLSTMAutoEncoder", 5), ("KerasLSTMForecast", 6)])
def test_detector_with_lstm_base_estimator(engine, torch, cls_name, offset):
    """tests/gordo/builder/test_builder.py:99-115 (model offsets) + test_anomaly_detectors.py with an LSTM base estimator:
    cross_validate / fit / anomaly run end to end on the GPU; the frame is tail-aligned to the shorter model output."""
    from gordo_components_b200.machine.model import models
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from oracle import anomaly_math as am
    from oracle import keras_math as km

    np.random.seed(1)
    n, T, L = 120, 4, 6
    t = np.linspace(0, 20, n)[:, None]
    Xv = 0.5 + 0.4 * np.sin(t * np.linspace(0.5, 2, T)) + np.random.normal(0, 0.02, (n, T))
    cols = [f"tag-{i}" for i in range(T)]
    X = pd.DataFrame(Xv, columns=cols, index=pd.date_range("2019-01-01", periods=n, freq="10min", tz="UTC"))
    det = DiffBasedAnomalyDetector(base_estimator=getattr(models, cls_name)(kind="lstm_hourglass", lookback_window=L, epochs=1, batch_size=16))
    det.cross_validate(X=X, y=X)
    assert len(det.feature_thresholds_) == T and np.isfinite(det.aggregate_threshold_)
    det.fit(X, X)
    frame = det.anomaly(X, X)
    assert len(X) - len(frame) == offset
    ae = det.base_estimator
    spec = km.lstm_hourglass_spec(T, lookback_window=L)
    pred = km.lstm_predict(spec, ae.model.weights, Xv.astype(np.float32), lookahead=ae.lookahead)
    close(frame["model-output"].values, pred, rtol=2e-4, name="lstm detector model-output")
    sc, mn = am.minmax_fit(Xv)
    want = am.anomaly_arrays(pred, Xv, sc, mn, det.feature_thresholds_.values, det.aggregate_threshold_)
    close(frame["tag-anomaly-unscaled"].values, want["tag-anomaly-unscaled"], rtol=2e-4, name="tag-anomaly-unscaled")
    close(frame["total-anomaly-confidence"].values.ravel(), want["total-anomaly-confidence"], float(want["total-anomaly-confidence"].max()), rtol=2e-4, name="confidence")


@pytest.mark.parametrize("case", ["tiny", "tiled", "forecast", "gradients"])
def test_lstm_fit_matches_oracle(engine, torch, case):
    """gb_lstm_fit (BPTT, primer step + ordered batches, Adam) against the oracle's restatement of models.py:557-616 on
    injected weights: the oracle's gradients are themselves pinned by finite differences in test_oracle_golden."""
    from oracle import keras_math as km

    if case == "tiny":
        spec = km.lstm_model_spec(3, 3, lookback_window=4, encoding_dim=(5,), encoding_func=("tanh",), decoding_dim=(4,), decoding_func=("tanh",))
        rows, epochs, B, la = [40], 2, 8, 0
    elif case == "tiled":  # widths that cross the 16-unit / 32-row / 64-column tiles, two machines of different length, partial batches
        spec = km.lstm_model_spec(20, 20, lookback_window=6, encoding_dim=(40, 24), encoding_func=("tanh", "tanh"), decoding_dim=(24, 40), decoding_func=("tanh", "tanh"))
        rows, epochs, B, la = [107, 75], 2, 32, 0
    elif case == "gradients":
        # Adam's update is (nearly) invariant to the gradient's scale; with beta1 = beta2 = 0 and eps = 1 a step is
        # -lr * g / (|g| + 1), so the trained weights expose the raw BPTT gradients
        spec = km.lstm_model_spec(20, 20, lookback_window=6, encoding_dim=(40, 24), encoding_func=("tanh", "tanh"), decoding_dim=(24, 40), decoding_func=("tanh", "tanh"))
        rows, epochs, B, la = [70], 1, 32, 0
        adam = {"lr": 1.0, "beta1": 0.0, "beta2": 0.0, "eps": 1.0}
    else:
        spec = km.lstm_model_spec(4, 2, lookback_window=5, encoding_dim=(9,), encoding_func=("tanh",), decoding_dim=(7,), decoding_func=("sigmoid",), out_func="tanh")
        rows, epochs, B, la = [60], 1, 16, 1
    if case != "gradients":
        adam = {"lr": 1e-3, "beta1": 0.9, "beta2": 0.999, "eps": 1e-7}
    rng = np.random.default_rng(5)
    eng = engine.LSTMEngine(spec.n_features, spec.units, spec.acts, spec.n_features_out, spec.out_func, spec.lookback_window)
    Xs = [rng.random((n, spec.n_features)).astype(np.float32) for n in rows]
    Ys = [rng.random((n, spec.n_features_out)).astype(np.float32) for n in rows]
    ws = [km.init_lstm_weights(spec, np.random.default_rng(10 + i)) for i in range(len(rows))]
    T = max(spec.n_features, spec.n_features_out)  # x and y share the row space; pad the narrower one
    dev = eng.device
    x = torch.from_numpy(np.concatenate(Xs)).to(dev)
    y = torch.from_numpy(np.concatenate(Ys)).to(dev)
    nwin = [n - spec.lookback_window + 1 - la for n in rows]
    starts = np.concatenate([[0], np.cumsum(rows)[:-1]])
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(len(rows)), nwin, starts), dev)
    params = eng.pack_params(ws)
    loss, acc, _ = eng.fit(params, jobs, len(rows), max(nwin), x, y, epochs=epochs, batch_size=B, lookahead=la, primer=True, adam=adam)
    torch.cuda.synchronize()
    got = eng.unpack_params(params)
    for i in range(len(rows)):
        want_w, hist = km.lstm_fit(spec, ws[i], Xs[i], Ys[i], epochs=epochs, batch_size=B, lookahead=la, lr=adam["lr"], b1=adam["beta1"],
                                   b2=adam["beta2"], eps=adam["eps"])
        close(loss[i].cpu().numpy(), np.array(hist["loss"]), rtol=5e-4, name=f"{case} loss history")
        assert np.allclose(acc[i].cpu().numpy(), hist["accuracy"], atol=1.5 / nwin[i])
        steps = 1 + epochs * int(np.ceil(nwin[i] / B))
        for w0, gl, wl in zip(km._lstm_flat(ws[i]), km._lstm_flat(got[i]), km._lstm_flat(want_w)):
            if case == "gradients":
                close(gl - w0, wl - w0, mag=float(np.abs(wl - w0).max()), rtol=1e-3, name="accumulated raw gradients")
            else:  # Adam moves a weight by ~lr per step whatever the gradient's size: compare the distance travelled
                close(gl - w0, wl - w0, mag=adam["lr"] * steps, rtol=2e-2, name=f"{case} trained weights")


@pytest.mark.parametrize("chain", ["minmax", "standard+minmax", "function"])
def test_detector_with_scaler_pipeline(engine, torch, chain):
    """Pipeline([scaler(s), KerasAutoEncoder]) as base estimator (the shape of gordo's example configs): raw, offset-dominated
    tags; per-feature scalers run as one f64 pass on the device and must equal sklearn's float64 transform cast to float32."""
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import FunctionTransformer, MinMaxScaler, StandardScaler

    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasAutoEncoder
    from oracle import anomaly_math as am
    from oracle import keras_math as km

    rng = np.random.default_rng(3)
    n, T = 300, 8
    t = np.linspace(0, 20, n)[:, None]
    Xv = (1000.0 * np.arange(1, T + 1)) + np.sin(t * np.linspace(0.5, 2, T)) + rng.normal(0, 0.05, (n, T))  # range ~2 on offsets up to 8000
    cols = [f"tag-{i}" for i in range(T)]
    X = pd.DataFrame(Xv, columns=cols, index=pd.date_range("2019-01-01", periods=n, freq="10min", tz="UTC"))
    steps = {"minmax": [MinMaxScaler()], "standard+minmax": [StandardScaler(), MinMaxScaler()],
             "function": [MinMaxScaler(), FunctionTransformer(lambda v: v * 1.0)]}[chain]
    pipe = Pipeline([(f"s{i}", s) for i, s in enumerate(steps)] + [("ae", KerasAutoEncoder(kind="feedforward_hourglass", epochs=2, batch_size=32))])
    det = DiffBasedAnomalyDetector(base_estimator=pipe, require_thresholds=False)
    det.fit(X, X)
    frame = det.anomaly(X, X)
    Xt = Xv
    for s in steps:
        Xt = s.transform(Xt)
    spec = km.ff_hourglass_spec(T)
    pred = km.ff_forward(spec, pipe.steps[-1][1].model.weights, np.asarray(Xt, dtype=np.float32), np.float64)
    close(frame["model-output"].values, pred, name=f"pipeline[{chain}] model-output")
    sc, mn = am.minmax_fit(Xv)
    want = am.anomaly_arrays(pred, Xv, sc, mn)
    close(frame["tag-anomaly-unscaled"].values, want["tag-anomaly-unscaled"], name="tag-anomaly-unscaled")


@pytest.mark.parametrize("n_rows,window,method,q", [(300, 12, "smm", 0.99), (300, 144, "sma", 0.9), (1000, 6, "ewma", 0.5)])
def test_kfcv_detector_thresholds(engine, torch, n_rows, window, method, q):
    """DiffBasedKFCVAnomalyDetector (diff.py:461-635; reference test test_anomaly_detectors.py:374-487): percentile of the
    smoothed K-fold validation errors.  Thresholds are re-derived with pandas from the fold models the detector trained."""
    from sklearn.model_selection import KFold

    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedKFCVAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasAutoEncoder
    from oracle import anomaly_math as am
    from oracle import keras_math as km

    np.random.seed(3)
    T = 6
    t = np.linspace(0, 30, n_rows)[:, None]
    Xv = 0.5 + 0.4 * np.sin(t * np.linspace(0.5, 2, T)) + np.random.normal(0, 0.03, (n_rows, T))
    cols = [f"tag-{i}" for i in range(T)]
    X = pd.DataFrame(Xv, columns=cols, index=pd.date_range("2019-01-01", periods=n_rows, freq="10min", tz="UTC"))
    det = DiffBasedKFCVAnomalyDetector(base_estimator=KerasAutoEncoder(kind="feedforward_hourglass", epochs=2), window=window,
                                       smoothing_method=method, threshold_percentile=q)
    assert det.get_params() == dict(base_estimator=det.base_estimator, scaler=det.scaler, window=window, smoothing_method=method, shuffle=True,
                                    threshold_percentile=q)
    with pytest.raises(AttributeError):
        det.fit(X, X).anomaly(X, X)
    cvo = det.cross_validate(X=X, y=X)
    spec = km.ff_hourglass_spec(T)
    abs_err = np.zeros((n_rows, T))
    mse = np.zeros(n_rows)
    for (tr, te), fold in zip(KFold(n_splits=5, shuffle=True, random_state=0).split(X, X), cvo["estimator"]):
        pred = km.ff_forward(spec, fold.base_estimator.model.weights, Xv[te], np.float64)
        abs_err[te] = np.abs(pred - Xv[te])
        mse[te] = (((pred - Xv[te]) * fold.scaler.scale_) ** 2).mean(axis=1)
    want_feat = pd.DataFrame(am.smoothing(abs_err, window, method)).quantile(q).values
    want_agg = pd.Series(am.smoothing(mse, window, method)).quantile(q)
    close(det.feature_thresholds_.values, want_feat, rtol=2e-3, mag=1e-4, name="KFCV feature thresholds")
    close(det.aggregate_threshold_, want_agg, rtol=2e-3, mag=1e-6, name="KFCV aggregate threshold")
    md = det.get_metadata()
    assert not np.isnan(md["feature-thresholds"]).any() and not np.isnan(md["aggregate-threshold"])
    det.fit(X, X)
    frame = det.anomaly(X, X)
    assert "smooth-total-anomaly-scaled" in frame.columns.get_level_values(0) and "total-anomaly-confidence" in frame.columns.get_level_values(0)


@pytest.mark.parametrize("case", ["kfcv_smm", "kfcv_ewma"])
def test_kfcv_detector_against_reference_generated_fixture(engine, torch, case):
    """Thresholds and frame columns of the reference's own DiffBasedKFCVAnomalyDetector (tests/golden/make_golden.py ran it
    from the reference with a LinearRegression base estimator) against ours with the same base estimator."""
    from sklearn.linear_model import LinearRegression
    from sklearn.multioutput import MultiOutputRegressor
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedKFCVAnomalyDetector

    g = np.load(os.path.join(GOLDEN, f"{case}.npz"), allow_pickle=False)
    Xv, yv = np.ascontiguousarray(g["X"]), np.ascontiguousarray(g["y"])
    cols = [f"tag-{i}" for i in range(Xv.shape[1])]
    idx = pd.date_range("2019-01-01", periods=len(Xv), freq="10min", tz="UTC")
    X, y = pd.DataFrame(Xv, columns=cols, index=idx), pd.DataFrame(yv, columns=cols, index=idx)
    det = DiffBasedKFCVAnomalyDetector(base_estimator=MultiOutputRegressor(LinearRegression()), scaler=MinMaxScaler(), window=int(g["window"]),
                                       smoothing_method=str(g["method"]), threshold_percentile=float(g["q"]))
    det.cross_validate(X=X, y=y)
    close(det.feature_thresholds_.values, g["feature_thresholds"], rtol=1e-5, mag=float(np.abs(g["feature_thresholds"]).max()), name="feature thresholds")
    close(det.aggregate_threshold_, float(g["aggregate_threshold"]), rtol=1e-5, mag=float(g["aggregate_threshold"]), name="aggregate threshold")
    det.fit(X, y)
    frame = det.anomaly(X, y, frequency=pd.Timedelta("10min"))
    assert list(dict.fromkeys(frame.columns.get_level_values(0))) == [str(c) for c in g["columns_level0"]]
    for top in ("total-anomaly-confidence", "anomaly-confidence", "smooth-total-anomaly-scaled", "smooth-tag-anomaly-unscaled"):
        want = g[f"frame_{top}"]
        got = np.asarray(frame[top], dtype=np.float64).reshape(want.shape)
        close(got, want, rtol=2e-5, mag=float(np.nanmax(np.abs(want))), name=top)


def test_quantile_kernel_matches_pandas(engine, torch):
    rng = np.random.default_rng(0)
    dev = engine.cuda_device()
    # up to 32768 rows: bitonic sort in shared memory; beyond (a year of 10-minute data is ~52k rows): radix selection over L2
    for n, cols in [(1, 3), (2, 1), (777, 5), (4096, 2), (10000, 3), (32768, 2), (32769, 2), (52560, 3)]:
        a = rng.normal(size=(n, cols)).astype(np.float32)
        if n > 30000:
            a[:, -1] = np.round(a[:, -1], 1)  # heavy ties: both order statistics inside one run of equal values
        a[rng.random(a.shape) < 0.1] = np.nan
        if n > 100:
            a[:, 0] = np.nan  # an all-NaN column stays NaN
        jobs = engine.jobs_to_device(engine.make_jobs([0], [n], [0]), dev)
        for q in (0.0, 0.37, 0.99, 1.0):
            got = engine.quantile(jobs, 1, n, torch.from_numpy(a).to(dev), q)[0].cpu().numpy()
            want = pd.DataFrame(a.astype(np.float64)).quantile(q).values
            assert np.allclose(got, want, rtol=1e-6, atol=1e-7, equal_nan=True), (n, q, got, want)


def test_error_paths_raise_like_the_reference(engine, torch):
    """Status codes surface as the exceptions the reference raises in the same situations (ValueError for bad shapes /
    arguments), never as a silent fallback."""
    from gordo_components_b200 import _cabi
    from oracle import keras_math as km

    dev = engine.cuda_device()
    spec = km.lstm_model_spec(5, 5, lookback_window=3, encoding_dim=(7,), encoding_func=("tanh",), decoding_dim=(7,), decoding_func=("tanh",))
    eng = engine.LSTMEngine(5, spec.units, spec.acts, 5, "linear", 3)
    params = eng.pack_params([km.init_lstm_weights(spec, np.random.default_rng(0))])
    x = torch.rand((20, 5), device=dev)
    jobs = engine.jobs_to_device(engine.make_jobs([0], [18], [0]), dev)
    assert eng.infer(params, jobs, 1, 18, x, 18).shape == (18, 5)
    with pytest.raises(ValueError):  # an unknown kernel variant is an argument error, not a fallback
        eng.lib.gb_lstm_tc_supported(None) == 0 or _cabi.check(eng.lib.gb_lstm_tc_supported(None))
    with pytest.raises(ValueError):  # batches above 32 windows are not supported by gb_lstm_fit
        eng.fit(params, jobs, 1, 18, x, x, epochs=1, batch_size=64)
    with pytest.raises(ValueError):  # pandas: "percentiles should all be in the interval [0, 1]"
        engine.quantile(engine.jobs_to_device(engine.make_jobs([0], [10], [0]), dev), 1, 10, torch.zeros((10, 1), device=dev), 1.5)
    # fused kernel: the tensor-core variant refuses architectures it does not cover
    ff = km.ff_hourglass_spec(10)
    e2 = engine.FFEngine(ff.dims, ff.acts, ff.l1)
    p2 = e2.pack_params([km.init_ff_weights(ff, np.random.default_rng(0))])
    x2 = torch.rand((64, 10), device=dev)
    j2 = engine.jobs_to_device(engine.make_jobs([0], [64], [0]), dev)
    with pytest.raises(ValueError):
        e2.infer_score(p2, j2, 1, 64, x2, x2, variant=2)
    with pytest.raises(ValueError):  # confidence requested without thresholds
        _cabi.check(e2.lib.gb_ffae_infer_score(_cabi.C.byref(e2.net), _cabi.ptr(p2), _cabi.ptr(j2), 1, 64, 64, 64, _cabi.ptr(x2), _cabi.ptr(x2), None,
                                               None, None, _cabi.ptr(torch.empty((64, 10), device=dev)), None, None, None, None,
                                               _cabi.ptr(torch.empty((64, 10), device=dev)), None, 0, None))


def test_request_coalescer_equals_per_request_launches(engine, torch):
    """serving.AnomalyCoalescer: 120 concurrent requests of 1..150 rows for random machines come back bit-identical to one
    launch per request (rows are independent in the kernel), in far fewer launches."""
    import threading

    from gordo_components_b200 import fleet, serving
    from oracle import keras_math as km

    spec = km.ff_hourglass_spec(64)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    M = 40
    g = torch.Generator(device=dev).manual_seed(3)
    params = fleet.random_glorot_params(eng, M, g)
    scale = torch.rand((M, 64), generator=g, device=dev) + 0.5
    feat = torch.rand((M, 64), generator=g, device=dev) + 0.5
    agg = torch.rand((M,), generator=g, device=dev) + 0.5
    rng = np.random.default_rng(0)
    reqs = [(int(rng.integers(0, M)), rng.random((int(rng.integers(1, 151)), 64)).astype(np.float32)) for _ in range(120)]
    co = serving.AnomalyCoalescer(eng, params, scale, feat, agg, max_wait_ms=20.0)
    futs = [None] * len(reqs)

    def client(i):
        futs[i] = co.submit(reqs[i][0], reqs[i][1], reqs[i][1] * 0.9)

    threads = [threading.Thread(target=client, args=(i,)) for i in range(len(reqs))]
    [t.start() for t in threads]
    [t.join() for t in threads]
    results = [f.result(timeout=60) for f in futs]
    assert co.batches < len(reqs) / 4 and co.requests == len(reqs)
    with pytest.raises(ValueError):
        co.submit(0, np.zeros((3, 5), np.float32), np.zeros((3, 5), np.float32))
    co.close()
    for (slot, X), got in zip(reqs, results):
        n = len(X)
        jobs = engine.jobs_to_device(engine.make_jobs([slot], [n], [0]), dev)
        xd = torch.from_numpy(X).to(dev)
        want = eng.infer_score(params, jobs, 1, n, xd, xd * 0.9 if False else torch.from_numpy(X * 0.9).to(dev), scale, feat, agg)
        for k, v in got.items():
            assert np.array_equal(v, want[k].cpu().numpy()), k


def test_fleet_build_matches_per_machine_oracle(engine, torch):
    """build_fleet = CV folds + final fit + thresholds for all machines in one launch each; checked machine by machine against
    the oracle's fold geometry / scaler / threshold arithmetic applied to the weights the fleet trained."""
    from gordo_components_b200 import fleet
    from oracle import anomaly_math as am
    from oracle import keras_math as km

    M, N, T = 5, 480, 8
    spec = km.ff_hourglass_spec(T)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    rng = np.random.default_rng(0)
    t = np.linspace(0, 25, N)[:, None]
    Xs = [(0.5 + 0.4 * np.sin(t * rng.uniform(0.5, 2, T) + rng.uniform(0, 3, T)) + rng.normal(0, 0.02, (N, T))).astype(np.float32) for _ in range(M)]
    x = torch.from_numpy(np.concatenate(Xs)).to(dev)
    fb = fleet.build_fleet(eng, x, x, rows=N, epochs=3, batch_size=32, n_splits=3, seed=1)
    torch.cuda.synchronize()
    assert fb.params.shape[0] == M and fb.fold_feat_thr.shape == (M, 3, T) and fb.loss.shape == (M, 3)
    assert bool((fb.loss[:, -1] < fb.loss[:, 0]).all())
    splits = am.time_series_split(N, 3)
    for m in range(M):
        sc, mn = am.minmax_fit(Xs[m])
        close(fb.scale[m].cpu().numpy(), sc, rtol=1e-5, mag=0, name="scale_")
    # thresholds of the final detector equal the oracle's arithmetic on the last fold model's predictions
    det = fb.detector(2, tags=[f"tag-{i}" for i in range(T)])
    assert list(det.aggregate_thresholds_per_fold_) == ["fold-0", "fold-1", "fold-2"]
    assert det.get_metadata()["feature-thresholds"] == det.feature_thresholds_.tolist()
    idx = pd.date_range("2019-01-01", periods=N, freq="10min", tz="UTC")
    frame_x = pd.DataFrame(Xs[2].astype(np.float64), columns=[f"tag-{i}" for i in range(T)], index=idx)
    frame = det.anomaly(frame_x, frame_x, frequency=pd.Timedelta("10min"))
    pred = km.ff_forward(spec, det.base_estimator.model.weights, Xs[2], np.float64)
    close(frame["model-output"].values, pred, name="fleet detector output")
    sc, mn = am.minmax_fit(Xs[2])
    want = am.anomaly_arrays(pred, Xs[2], sc, mn, det.feature_thresholds_.values, det.aggregate_threshold_)
    close(frame["total-anomaly-confidence"].values.ravel(), want["total-anomaly-confidence"], float(sc.max()) * np.sqrt(want["total-anomaly-scaled"].max()) / det.aggregate_threshold_, name="confidence")
    import json
    import pickle
    import tempfile

    pickle.loads(pickle.dumps(det)).anomaly(frame_x, frame_x)
    # gordo.serializer layout: <root>/<machine>/model.pkl + metadata.json (+ info.json), loadable with plain pickle
    with tempfile.TemporaryDirectory() as root:
        names = [f"machine-{m}" for m in range(M)]
        dirs = fleet.dump_fleet(fb, root, names, tags=[[f"tag-{i}" for i in range(T)]] * M, info={"checksum": "abc"})
        assert [os.path.basename(d) for d in dirs] == names
        with open(os.path.join(dirs[2], "model.pkl"), "rb") as f:
            loaded = pickle.load(f)
        np.testing.assert_array_equal(loaded.anomaly(frame_x, frame_x)["model-output"].values, frame["model-output"].values)
        meta = json.load(open(os.path.join(dirs[2], "metadata.json")))
        assert meta["name"] == "machine-2" and "feature-thresholds" in meta["metadata"]["build_metadata"]["model"]["model_meta"]
        assert json.load(open(os.path.join(dirs[2], "info.json"))) == {"checksum": "abc"}


# ------------------------------------------------------------------------------------------------ BASELINE-size properties
def test_full_size_properties(engine, torch):
    """
    configs[1] size (1000 machines x 64 tags x 10000 rows): too big for the oracle, so check size-independent
    properties -- internal consistency of the fused outputs, idempotence, job-order invariance -- plus oracle
    parity on a random sample of (machine, row-block) pairs.
    """
    from oracle import keras_math as km

    M, R, T = 1000, 10000, 64
    spec = km.ff_hourglass_spec(T)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    dev = eng.device
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.rand((M * R, T), generator=g, device=dev)
    y = x + 0.05 * torch.randn((M * R, T), generator=g, device=dev)
    lim = [np.sqrt(6.0 / (i + o)) for i, o in zip(spec.dims[:-1], spec.dims[1:])]
    params = torch.zeros((M, eng.param_stride), device=dev)
    ofs = 0
    for (i, o), l in zip(zip(spec.dims[:-1], spec.dims[1:]), lim):
        params[:, ofs:ofs + i * o] = (torch.rand((M, i * o), generator=g, device=dev) * 2 - 1) * l
        ofs += i * o
        params[:, ofs:ofs + o] = (torch.rand((M, o), generator=g, device=dev) * 2 - 1) * 0.1
        ofs += o
    jobs_h = engine.uniform_jobs(M, R)
    jobs = engine.jobs_to_device(jobs_h, dev)
    scale, _ = eng.minmax_fit(jobs, M, R, y, M)
    feat = torch.rand((M, T), generator=g, device=dev) * 0.2 + 0.05
    agg = torch.rand((M,), generator=g, device=dev) * 0.1 + 0.01
    res = eng.infer_score(params, jobs, M, R, x, y, scale, feat, agg)
    torch.cuda.synchronize()
    out, tu, ts = res["model-output"], res["tag-anomaly-unscaled"], res["tag-anomaly-scaled"]
    sc_rows = scale.repeat_interleave(R, dim=0)
    assert torch.equal(tu, (out - y).abs())
    assert torch.equal(ts, tu * sc_rows)
    assert torch.allclose(res["total-anomaly-unscaled"], (tu * tu).mean(dim=1), rtol=1e-5, atol=1e-9)
    assert torch.allclose(res["total-anomaly-scaled"], (ts * ts).mean(dim=1), rtol=1e-5, atol=1e-9)
    assert torch.allclose(res["anomaly-confidence"], tu / feat.repeat_interleave(R, dim=0), rtol=1e-6)
    assert torch.allclose(res["total-anomaly-confidence"], res["total-anomaly-scaled"] / agg.repeat_interleave(R), rtol=1e-6)
    assert bool(torch.isfinite(out).all())
    checksum = out.double().sum().item()
    del sc_rows
    # idempotent + independent of job order
    perm = np.random.default_rng(0).permutation(M)
    res2 = eng.infer_score(params, engine.jobs_to_device(jobs_h[perm], dev), M, R, x, y, scale, feat, agg, want=())
    torch.cuda.synchronize()
    assert torch.equal(res2["model-output"], out)
    assert res2["model-output"].double().sum().item() == checksum
    # oracle parity on sampled blocks
    rng = np.random.default_rng(1)
    host_params = params.cpu().numpy()
    for m in rng.choice(M, 6, replace=False):
        r0 = int(rng.integers(0, R - 200))
        w, o = [], 0
        for i, oo in zip(spec.dims[:-1], spec.dims[1:]):
            W = host_params[m, o:o + i * oo].reshape(i, oo); o += i * oo
            b = host_params[m, o:o + oo]; o += oo
            w.append((W, b))
        rows = slice(m * R + r0, m * R + r0 + 200)
        want = km.ff_forward(spec, w, x[rows].cpu().numpy(), np.float64)
        close(out[rows].cpu().numpy(), want, name="sampled block")
    # min-max scaler statistics at full size: exact reductions
    ymin = y.view(M, R, T).amin(dim=1)
    ymax = y.view(M, R, T).amax(dim=1)
    assert torch.allclose(scale, 1.0 / (ymax - ymin), rtol=1e-6)
