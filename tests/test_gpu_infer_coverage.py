"""
The Dense and LSTM inference kernels across the architectures and job layouts their dispatch admits, against the float64 oracle
(oracle/keras_math, oracle/anomaly_math) at the tolerances of parity_helpers.close.

Dense: the generic fp32 kernel (variant 1), the row-per-thread kernel (3, every width <= 16) and the tensor-core kernel (2), each on
every architecture of the grid it admits, every launch plan of the generic kernel (tests/test_infer_plan.py pins them), the widest
default stacks, job layouts and output subsets.  LSTM: the fp32 kernel (1) and the tensor-core kernel (2, tanh and sigmoid cells)
over cells, heads, widths and job layouts, hidden states beyond the FP16 range, and more slots or jobs than a grid dimension holds.
"""
import ctypes as C

import numpy as np
import pytest
from parity_helpers import close
from test_infer_plan import COLUMN_BLOCKED, PLAN_SHAPES

pytestmark = pytest.mark.gpu

SCORE = ("tag-anomaly-scaled", "tag-anomaly-unscaled", "total-anomaly-scaled", "total-anomaly-unscaled", "anomaly-confidence",
         "total-anomaly-confidence")
PER_ROW = ("total-anomaly-scaled", "total-anomaly-unscaled", "total-anomaly-confidence")


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


# ------------------------------------------------------------------------------------------------ Dense helpers
def dense_net(km, dims, acts, seed, scale0=1.0):
    spec = km.FFSpec(list(dims), list(acts))
    rng = np.random.default_rng(seed)
    w = km.init_ff_weights(spec, rng)
    w = [((W * scale0 if i == 0 else W).astype(np.float32), rng.uniform(-0.2, 0.2, b.shape).astype(np.float32)) for i, (W, b) in enumerate(w)]
    return spec, w


def variants_for(lib, spec):
    net = _net(spec)
    return [1] + ([3] if lib.gb_ffae_small_supported(C.byref(net)) == 0 else []) + ([2] if lib.gb_ffae_tc_supported(C.byref(net)) == 0 else [])


def _net(spec):
    from gordo_components_b200 import _cabi

    return _cabi.make_ffnet(spec.dims, spec.acts)


def score_inputs(rng, n_slots, n_out):
    scale = (rng.random((n_slots, n_out)) * 1.5 + 0.5).astype(np.float32)
    feat = (rng.random((n_slots, n_out)) * 0.2 + 0.05).astype(np.float32)
    agg = (rng.random(n_slots) * 0.1 + 0.01).astype(np.float32)
    return scale, feat, agg


def run_dense(engine, torch, spec, weights, X, y, jobs_h, scale, feat, agg, out_rows, variant, want=SCORE, nan_fill=False, x_affine=None):
    """x_affine: None, or the per-slot input scaler (a, b) [n_slots, n_in]; X is then float64 and scaled inside the launch."""
    eng = engine.FFEngine(spec.dims, spec.acts)
    dev = eng.device
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)  # noqa: E731
    t64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(dev)  # noqa: E731
    out = None
    if nan_fill:
        n = eng.n_out
        shapes = {"model-output": (out_rows, n), **{k: (out_rows,) if k in PER_ROW else (out_rows, n) for k in SCORE}}
        out = {k: torch.full(s, float("nan"), device=dev) for k, s in shapes.items()}
    x = t(X) if x_affine is None else t64(X)
    ab = None if x_affine is None else tuple(t64(v) for v in x_affine)
    res = eng.infer_score(eng.pack_params(weights), engine.jobs_to_device(jobs_h, dev), len(jobs_h), max(1, int(jobs_h["n_rows"].max())),
                          x, t(y), t(scale), t(feat), t(agg), out_rows=out_rows, want=want, variant=variant, out=out, x_affine=ab)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in res.items()}


def check_dense(got, rows, want_out, y, scale, feat, agg, name):
    """All seven outputs of the rows `rows` of `got` against the oracle's model output `want_out` for targets `y`."""
    from oracle import anomaly_math as am

    m = max(1.0, float(np.abs(want_out).max()))
    want = am.anomaly_arrays(want_out, y, scale.astype(np.float64), np.zeros(scale.shape), feat, float(agg))
    d = float(want["tag-anomaly-unscaled"].max())
    close(got["model-output"][rows], want_out, m, name=f"{name}: model-output")
    close(got["tag-anomaly-unscaled"][rows], want["tag-anomaly-unscaled"], m, name=f"{name}: tag-unscaled")
    close(got["tag-anomaly-scaled"][rows], want["tag-anomaly-scaled"], m * float(scale.max()), name=f"{name}: tag-scaled")
    close(got["anomaly-confidence"][rows], want["anomaly-confidence"], m / float(feat.min()), name=f"{name}: confidence")
    tot_mag = 2 * m * max(d, 1.0) * float(scale.max()) ** 2
    close(got["total-anomaly-unscaled"][rows], want["total-anomaly-unscaled"], 2 * m * max(d, 1.0), name=f"{name}: total-unscaled")
    close(got["total-anomaly-scaled"][rows], want["total-anomaly-scaled"], tot_mag, name=f"{name}: total-scaled")
    close(got["total-anomaly-confidence"][rows], want["total-anomaly-confidence"], tot_mag / float(agg), name=f"{name}: total-confidence")


def dense_oracle_case(engine, torch, spec, nets, variant, R=333, x_scale=1.0, seed=0):
    """M = len(nets) machines of R rows each (ragged against every row tile), all seven outputs against the oracle."""
    from oracle import keras_math as km

    rng = np.random.default_rng(seed)
    M, n_in, n_out = len(nets), spec.dims[0], spec.dims[-1]
    X = ((rng.random((M * R, n_in)) * 2 - 0.5) * x_scale).astype(np.float32)
    y = rng.random((M * R, n_out)).astype(np.float32)
    scale, feat, agg = score_inputs(rng, M, n_out)
    got = run_dense(engine, torch, spec, nets, X, y, engine.uniform_jobs(M, R), scale, feat, agg, M * R, variant)
    for m in range(M):
        sl = slice(m * R, (m + 1) * R)
        check_dense(got, sl, km.ff_forward(spec, nets[m], X[sl], np.float64), y[sl], scale[m], feat[m], agg[m], f"variant {variant} machine {m}")


# ------------------------------------------------------------------------------------------------ Dense: architecture grid
DENSE_GRID = {
    "one_linear_layer_width1": ([1, 1], ["linear"]),
    "relu_sigmoid_width3_5": ([3, 5, 3], ["relu", "sigmoid"]),
    "out_below_in_not_mult4": ([16, 17, 5], ["sigmoid", "relu"]),
    "out_above_in_pow2_groups": ([5, 3, 16], ["tanh", "linear"]),
    "width12_out_3_groups": ([12, 8, 12], ["sigmoid", "linear"]),
    "depth16_small_mixed": ([8] * 17, ["relu", "sigmoid", "tanh", "linear"] * 3 + ["relu", "sigmoid", "tanh", "tanh"]),
    "relu_width20_24": ([20, 24, 20], ["relu", "tanh"]),
    "sigmoid_width36_48": ([36, 48, 36], ["sigmoid", "sigmoid"]),
    "linear_hidden_width65": ([48, 65, 48], ["linear", "relu"]),
    "out132_over_32_groups": ([24, 132, 132], ["tanh", "linear"]),
    "one_layer_out256": ([17, 256], ["relu"]),
    "out128_32_groups": ([20, 36, 128], ["relu", "linear"]),
    "depth16_tanh": ([24] + [16] * 15 + [24], ["tanh"] * 15 + ["linear"]),
    "tc_pow2_groups": ([64, 32, 64], ["tanh", "linear"]),
    "tc_hourglass48": ([48, 36, 29, 24, 24, 29, 36, 48], ["tanh"] * 6 + ["linear"]),
    "tc_sigmoid_out": ([24, 16, 24], ["tanh", "sigmoid"]),
}


@pytest.mark.parametrize("case", list(DENSE_GRID))
def test_dense_architecture_grid_on_every_admitting_variant(engine, torch, case):
    from gordo_components_b200 import _cabi
    from oracle import keras_math as km

    dims, acts = DENSE_GRID[case]
    nets = [dense_net(km, dims, acts, 100 + s) for s in range(3)]
    spec = nets[0][0]
    variants = variants_for(_cabi.load_library(), spec)
    if case.startswith("tc_") and case != "tc_sigmoid_out":
        assert 2 in variants
    for v in variants:
        dense_oracle_case(engine, torch, spec, [w for _, w in nets], v)


@pytest.mark.parametrize("plan", list(PLAN_SHAPES) + ["column_blocked_0", "column_blocked_1"])
def test_dense_every_generic_plan(engine, torch, plan):
    """One architecture per launch plan of the generic kernel (row tile, resident or staged weights, column-blocked staging)."""
    from oracle import keras_math as km

    dims = PLAN_SHAPES[plan] if plan in PLAN_SHAPES else COLUMN_BLOCKED[int(plan[-1])]
    acts = ["tanh"] * (len(dims) - 2) + ["linear"]
    nets = [dense_net(km, dims, acts, 7 + s) for s in range(2)]
    dense_oracle_case(engine, torch, nets[0][0], [w for _, w in nets], 1, R=300)


def test_widest_default_stacks_predict(engine, torch):
    """symmetric(172) -- the widest feedforward_symmetric default the fit accepts -- and a stack with a 256 x 256 layer, through the
    automatic dispatch; and the estimator that trains a 170-tag symmetric model predicts with it."""
    from gordo_components_b200.machine.model.models import KerasAutoEncoder
    from oracle import keras_math as km

    for dims in COLUMN_BLOCKED:
        acts = ["tanh"] * (len(dims) - 2) + ["linear"]
        nets = [dense_net(km, dims, acts, 3)]
        dense_oracle_case(engine, torch, nets[0][0], [w for _, w in nets], 0, R=200)
    np.random.seed(0)
    X = np.random.random((64, 170)).astype(np.float32)
    m = KerasAutoEncoder(kind="feedforward_symmetric", epochs=1).fit(X, X)
    spec = m.model.spec
    want = km.ff_forward(km.FFSpec(list(spec.dims), list(spec.acts), list(spec.l1)), m.model.weights, X, np.float64)
    close(m.predict(X), want, 1.0, name="feedforward_symmetric, 170 tags")


@pytest.mark.parametrize("T", list(range(24, 65, 4)))
def test_dense_tensor_core_tag_range(engine, torch, T):
    from oracle import keras_math as km

    spec = km.ff_hourglass_spec(T)
    nets = [dense_net(km, spec.dims, spec.acts, T + s) for s in range(2)]
    dense_oracle_case(engine, torch, spec, [w for _, w in nets], 2, R=200)


@pytest.mark.parametrize("dims", [[48, 12, 48], [48, 16, 48], [48, 32, 48], [48, 48, 48], [48, 64, 48], [40, 64, 48, 12, 16, 32, 40],
                                  [64, 16, 32, 48, 64, 64, 64]])
def test_dense_tensor_core_hidden_widths_and_depth(engine, torch, dims):
    from oracle import keras_math as km

    acts = ["tanh"] * (len(dims) - 2) + ["linear"]
    nets = [dense_net(km, dims, acts, len(dims) + s) for s in range(2)]
    dense_oracle_case(engine, torch, nets[0][0], [w for _, w in nets], 2, R=200)


@pytest.mark.parametrize("variant", [1, 2])
def test_dense_raw_magnitude_inputs(engine, torch, variant):
    """x around 1e4 with the first layer's kernel scaled down so that the pre-activations stay O(1)."""
    from oracle import keras_math as km

    spec = km.ff_hourglass_spec(32)
    nets = [dense_net(km, spec.dims, spec.acts, 5 + s, scale0=1e-4) for s in range(2)]
    dense_oracle_case(engine, torch, spec, [w for _, w in nets], variant, R=200, x_scale=1e4)


# ------------------------------------------------------------------------------------------------ Dense: job layouts
LAYOUT_SPECS = {1: [8, 6, 8], 3: [8, 6, 8], 2: [32, 24, 32]}


def layout_jobs(engine):
    # slot, n_rows, x_row, out_row: jobs of different slots over overlapping rows (0 and 1), several jobs of one slot (0, 2, 5), slots
    # out of job order, an empty job, x_row off any tile boundary, outputs anywhere in an array longer than x
    return engine.make_jobs([2, 0, 2, 1, 0, 1], [300, 200, 70, 0, 129, 1], [100, 150, 5, 0, 1, 333], [1000, 3, 700, 0, 300, 299])


@pytest.mark.parametrize("variant", [1, 2, 3])
def test_dense_job_layouts(engine, torch, variant):
    from oracle import keras_math as km

    dims = LAYOUT_SPECS[variant]
    acts = ["tanh"] * (len(dims) - 2) + ["linear"]
    nets = [dense_net(km, dims, acts, 30 + s) for s in range(3)]
    spec = nets[0][0]
    rng = np.random.default_rng(1)
    X = rng.random((500, dims[0])).astype(np.float32)
    y = rng.random((500, dims[-1])).astype(np.float32)
    scale, feat, agg = score_inputs(rng, 3, dims[-1])
    jobs = layout_jobs(engine)
    out_rows = 1400
    got = run_dense(engine, torch, spec, [w for _, w in nets], X, y, jobs, scale, feat, agg, out_rows, variant, nan_fill=True)
    written = np.zeros(out_rows, bool)
    for j, job in enumerate(jobs):
        s, n, xr, orow = (int(job[k]) for k in ("slot", "n_rows", "x_row", "out_row"))
        if n == 0:
            continue
        rows = slice(orow, orow + n)
        written[rows] = True
        check_dense(got, rows, km.ff_forward(spec, nets[s][1], X[xr:xr + n], np.float64), y[xr:xr + n], scale[s], feat[s], agg[s],
                    f"variant {variant} job {j}")
    for k, v in got.items():
        assert np.isnan(v[~written]).all(), f"variant {variant}: {k} written outside the jobs' output rows"


@pytest.mark.parametrize("variant", [1, 2, 3])
def test_dense_rows_are_independent_of_the_job_split(engine, torch, variant):
    """The same 322 rows as one job and as jobs of 1, 63, 64, 65 and 129 rows: every output, the per-row totals included, is
    bit-identical (a row's squares are summed in column order wherever the row lands in a tile)."""
    from oracle import keras_math as km

    dims = [24, 20, 24] if variant == 1 else LAYOUT_SPECS[variant]  # 24 tags: the generic kernel's column-order row sums
    acts = ["tanh"] * (len(dims) - 2) + ["linear"]
    spec, w = dense_net(km, dims, acts, 11)
    rng = np.random.default_rng(2)
    X = rng.random((400, dims[0])).astype(np.float32)
    y = rng.random((400, dims[-1])).astype(np.float32)
    scale, feat, agg = score_inputs(rng, 1, dims[-1])
    sizes = [1, 63, 64, 65, 129]
    starts = 7 + np.concatenate([[0], np.cumsum(sizes)[:-1]])
    whole = run_dense(engine, torch, spec, [w], X, y, engine.make_jobs([0], [sum(sizes)], [7], [0]), scale, feat, agg, 400, variant)
    split = run_dense(engine, torch, spec, [w], X, y, engine.make_jobs([0] * 5, sizes, starts, starts - 7), scale, feat, agg, 400, variant)
    n = sum(sizes)
    for k in whole:
        np.testing.assert_array_equal(split[k][:n], whole[k][:n], err_msg=k)


@pytest.mark.parametrize("variant", [1, 3])
@pytest.mark.parametrize("want", [(k,) for k in SCORE] + [()])
def test_dense_output_subsets(engine, torch, variant, want):
    """Each score output alone, and prediction only (no y): the outputs nobody asked for stay untouched."""
    from oracle import keras_math as km

    dims = [12, 7, 12]
    spec, w = dense_net(km, dims, ["sigmoid", "linear"], 12)
    rng = np.random.default_rng(3)
    X = rng.random((260, 12)).astype(np.float32)
    y = rng.random((260, 12)).astype(np.float32)
    scale, feat, agg = score_inputs(rng, 1, 12)
    jobs = engine.uniform_jobs(1, 260)
    full = run_dense(engine, torch, spec, [w], X, y, jobs, scale, feat, agg, 260, variant)
    check_dense(full, slice(0, 260), km.ff_forward(spec, w, X, np.float64), y, scale[0], feat[0], agg[0], f"variant {variant}")
    got = run_dense(engine, torch, spec, [w], X, y if want else None, jobs, scale, feat, agg, 260, variant, want=want, nan_fill=True)
    np.testing.assert_array_equal(got["model-output"], full["model-output"])
    for k in SCORE:
        if k in want:
            close(got[k], full[k], mag=0.0, rtol=1e-6, name=k)
        else:
            assert np.isnan(got[k]).all(), f"{k} written although only {want or 'the prediction'} was requested"


# ------------------------------------------------------------------------------------------------ LSTM helpers
def lstm_net(km, F, units, acts, F_out, out_func, L, seed, shrink=1.0):
    spec = km.LSTMSpec(F, list(units), list(acts), F_out, out_func, L)
    layers, (Wd, bd) = km.init_lstm_weights(spec, np.random.default_rng(seed))
    rng = np.random.default_rng(seed + 1)
    layers = [((K * shrink).astype(np.float32), (U * shrink).astype(np.float32), rng.uniform(-0.2, 0.2, b.shape).astype(np.float32) + b)
              for K, U, b in layers]
    return spec, (layers, (Wd, rng.uniform(-0.2, 0.2, bd.shape).astype(np.float32)))


def lstm_engine(engine, spec):
    return engine.LSTMEngine(spec.n_features, spec.units, spec.acts, spec.n_features_out, spec.out_func, spec.lookback_window)


def run_lstm(engine, torch, spec, weights, X, jobs_h, out_rows, variant, params=None):
    eng = lstm_engine(engine, spec)
    dev = eng.device
    params = eng.pack_params(weights) if params is None else params
    out = eng.infer(params, engine.jobs_to_device(jobs_h, dev), len(jobs_h), max(1, int(jobs_h["n_rows"].max())),
                    torch.from_numpy(np.ascontiguousarray(X, np.float32)).to(dev), out_rows, variant=variant)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def lstm_oracle(km, spec, weights, X, x_row, n):
    """The float64 oracle on windows [x_row + j, x_row + j + lookback), j < n."""
    L = spec.lookback_window
    win = np.lib.stride_tricks.sliding_window_view(np.asarray(X[x_row:x_row + n + L - 1], np.float64), (L, X.shape[1]))[:, 0]
    return km.lstm_forward_windows(spec, weights, win, np.float64)


def lstm_variants(engine, spec):
    return [0, 1] + ([2] if lstm_engine(engine, spec).tc_supported else [])


# F, units, cell activations, n_features_out, head, lookback, lookahead
LSTM_GRID = {
    "sigmoid_cells_tanh_head_fewer_out": (5, [7, 9], ["sigmoid", "sigmoid"], 3, "tanh", 4, 0),
    "tanh_sigmoid_relu_head_more_out": (33, [63, 65], ["tanh", "sigmoid"], 40, "relu", 3, 0),
    "relu_cells_sigmoid_head": (4, [8, 6], ["relu", "relu"], 4, "sigmoid", 5, 0),
    "linear_cells": (3, [5], ["linear"], 6, "linear", 3, 0),
    "mixed_cells": (6, [10, 8, 6, 4], ["tanh", "relu", "sigmoid", "linear"], 6, "tanh", 4, 0),
    "lookback1": (8, [16], ["tanh"], 8, "linear", 1, 0),
    "width1_features1": (1, [1], ["tanh"], 1, "sigmoid", 6, 0),
    "widths64_129": (33, [64, 129], ["tanh", "tanh"], 33, "linear", 3, 0),
    "width512_features512": (512, [512], ["tanh"], 512, "linear", 2, 0),
    "forecast": (5, [16, 8], ["tanh", "sigmoid"], 5, "linear", 4, 1),
}


@pytest.mark.parametrize("case", list(LSTM_GRID))
def test_lstm_architecture_grid(engine, torch, case):
    from oracle import keras_math as km

    F, units, acts, F_out, head, L, ahead = LSTM_GRID[case]
    shrink = 0.5 if {"relu", "linear"} & set(acts) else 1.0
    nets = [lstm_net(km, F, units, acts, F_out, head, L, 50 + s, shrink) for s in range(2)]
    spec = nets[0][0]
    rows = [L + ahead + 40, L + ahead + 150]
    rng = np.random.default_rng(4)
    Xs = [rng.random((n, F)).astype(np.float32) for n in rows]
    nwin = [n - L + 1 - ahead for n in rows]
    starts = np.concatenate([[0], np.cumsum(rows)[:-1]])
    outs = np.concatenate([[0], np.cumsum(nwin)[:-1]])
    jobs = engine.make_jobs([1, 0], nwin, starts, outs)
    wants = [km.lstm_predict(spec, nets[1 - m][1], Xs[m], lookahead=ahead, dtype=np.float64) for m in range(2)]
    variants = lstm_variants(engine, spec)
    assert (2 in variants) == (set(acts) <= {"tanh", "sigmoid"})
    for v in variants:
        got = run_lstm(engine, torch, spec, [w for _, w in nets], np.concatenate(Xs), jobs, sum(nwin), v)
        for m in range(2):
            want = wants[m]
            close(got[outs[m]:outs[m] + nwin[m]], want, max(1.0, float(np.abs(want).max())), name=f"{case} variant {v} job {m}")
    if 2 not in variants:
        with pytest.raises(ValueError):
            run_lstm(engine, torch, spec, [w for _, w in nets], np.concatenate(Xs), jobs, sum(nwin), 2)


@pytest.mark.parametrize("variant", [1, 2])
def test_lstm_job_layouts(engine, torch, variant):
    """Jobs of different slots over the same x rows, several jobs of one slot, slots out of job order, an empty job, x_row off any
    tile boundary, outputs anywhere in an array longer than x."""
    from oracle import keras_math as km

    L = 4
    nets = [lstm_net(km, 6, [16, 12], ["tanh", "tanh"], 6, "linear", L, 70 + s) for s in range(3)]
    spec = nets[0][0]
    X = np.random.default_rng(5).random((600, 6)).astype(np.float32)
    # slot, windows, x_row, out_row
    jobs = engine.make_jobs([2, 0, 2, 1, 0, 1], [300, 300, 70, 0, 129, 1], [0, 0, 37, 0, 201, 596], [1000, 3, 700, 0, 303, 2])
    out_rows = 1300
    got = run_lstm(engine, torch, spec, [w for _, w in nets], X, jobs, out_rows, variant)
    for j, job in enumerate(jobs):
        s, n, xr, orow = (int(job[k]) for k in ("slot", "n_rows", "x_row", "out_row"))
        if n == 0:
            continue
        close(got[orow:orow + n], lstm_oracle(km, spec, nets[s][1], X, xr, n), 1.0, name=f"variant {variant} job {j}")


def test_lstm_hidden_state_beyond_fp16(engine, torch):
    """relu and linear cells whose float64 hidden state exceeds the FP16 range: the automatic dispatch still matches the oracle, and
    the tensor-core kernel (h carried as an FP16 pair) refuses the architecture."""
    from oracle import keras_math as km

    F, units, acts, L = 2, [4, 3], ["relu", "linear"], 5
    spec, (layers, dense) = lstm_net(km, F, units, acts, 2, "linear", L, 90)
    K0, U0, b0 = layers[0]
    b0 = b0.copy()
    b0[:4] += 8.0                       # input gates open
    b0[4:8] += 8.0                      # forget gates open: c accumulates over the lookback
    b0[12:16] += 8.0                    # output gates open
    K0 = K0.copy()
    K0[:, 8:12] = np.abs(K0[:, 8:12]) * 4e4  # candidate relu(z_g) of order 1e4 per step for x in [0.5, 1]
    layers = [(K0, U0 * 0.0, b0), (layers[1][0] * 0.5, layers[1][1] * 0.5, layers[1][2])]
    weights = (layers, dense)
    X = (np.random.default_rng(6).random((120, F)) * 0.5 + 0.5).astype(np.float32)
    # the oracle's hidden states: each layer's final h, read through an identity head
    h_max = 0.0
    for depth in (1, 2):
        u = units[depth - 1]
        sub = km.LSTMSpec(F, units[:depth], acts[:depth], u, "linear", L)
        h = km.lstm_predict(sub, (layers[:depth], (np.eye(u, dtype=np.float32), np.zeros(u, np.float32))), X, dtype=np.float64)
        h_max = max(h_max, float(np.abs(h).max()))
    assert h_max > 65504.0, h_max
    want = km.lstm_predict(spec, weights, X, dtype=np.float64)
    nwin = len(want)
    jobs = engine.make_jobs([0], [nwin], [0], [0])
    for v in (0, 1):
        got = run_lstm(engine, torch, spec, [weights], X, jobs, nwin, v)
        assert np.isfinite(got).all()
        close(got, want, float(np.abs(want).max()), name=f"variant {v}")
    with pytest.raises(ValueError):
        run_lstm(engine, torch, spec, [weights], X, jobs, nwin, 2)


@pytest.mark.parametrize("variant", [1, 2])
def test_lstm_more_slots_than_a_grid_dimension(engine, torch, variant):
    """65 536 slots (a 16 384-machine bucket with 3 CV folds): the per-slot weight preparation covers every slot."""
    from oracle import keras_math as km

    S, L = 65_536, 2
    spec = km.LSTMSpec(2, [2], ["tanh"], 2, "linear", L)
    eng = lstm_engine(engine, spec)
    g = torch.Generator(device=eng.device).manual_seed(8)
    params = (torch.rand((S, eng.param_stride), generator=g, device=eng.device) - 0.5) * 2
    X = np.random.default_rng(7).random((40, 2)).astype(np.float32)
    slots = [0, 1, 65_534, 65_535]
    jobs = engine.make_jobs(slots, [10] * 4, [0, 5, 20, 29], [0, 10, 20, 30])
    got = run_lstm(engine, torch, spec, None, X, jobs, 40, variant, params=params)
    host = eng.unpack_params(params[slots])
    del params
    torch.cuda.empty_cache()
    for j, s in enumerate(slots):
        xr = int(jobs["x_row"][j])
        close(got[10 * j:10 * j + 10], lstm_oracle(km, spec, host[j], X, xr, 10), 1.0, name=f"slot {s}")


@pytest.mark.parametrize("variant", [1, 2])
def test_lstm_more_jobs_than_a_grid_dimension(engine, torch, variant):
    """65 540 one-window jobs of two slots: the launches that carry the job index on a grid dimension go out in several parts."""
    from oracle import keras_math as km

    J, L = 65_540, 2
    nets = [lstm_net(km, 2, [2], ["tanh"], 2, "linear", L, 95 + s) for s in range(2)]
    spec = nets[0][0]
    X = np.random.default_rng(8).random((J + L, 2)).astype(np.float32)
    jobs = engine.make_jobs(np.arange(J) % 2, 1, np.arange(J, dtype=np.int64), np.arange(J, dtype=np.int64))
    got = run_lstm(engine, torch, spec, [w for _, w in nets], X, jobs, J, variant)
    torch.cuda.empty_cache()
    for j in (0, 1, 65_534, 65_535, 65_536, J - 1):
        close(got[j:j + 1], lstm_oracle(km, spec, nets[j % 2][1], X, j, 1), 1.0, name=f"job {j}")
