"""
The two LSTM fit families (gb_lstm_fit_stop on fp32 CUDA cores up to 32 windows a batch, gb_lstm_fit_tc_stop on the tensor cores up
to 256) at the sizes gb_lstm_fit admits and the fleet builder trains: the production lstm_symmetric stack (128 tags, 256-128-64-64-
128-256 units, lookback 144), 512 units with 512 features, 16 layers.  Every fit is compared with the oracle's float64 fit loop
(oracle/keras_math.py lstm_fit, dtype=np.float64), so the error measured is the kernels' own.

Where these sizes reach code the narrow tests do not:
  - the tensor-core GEMMs reduce over the in + u + 1 rows of [x | h | 1]; when in + u is a multiple of 64 the last weight-gradient
    row tile holds the bias row alone, and when it is a multiple of 32 the forward's last 32-row chunk does;
  - the fp32 head's dynamic shared memory (32 u_last + 64 T_out) floats is 196 608 bytes at u_last = T_out = 512, its largest;
  - the unit, column and row-tile block counts at width 512, and a 16-layer step graph with its 16-entry layer table;
  - gb_orthonormal_rows, which draws every recurrent kernel of the fleet builder, at u = 256 and 512.

Tolerances are those of tests/test_gpu_fit_coverage.py, with two terms added for the float64 reference (check_f64):
  - raw-gradient mode (lr 1, beta 0, eps 1: a step is -g / (|g| + 1)): the weight change within rtol 1e-3 plus 2e-5 of the array's
    largest change;  Keras Adam: loss history rtol 5e-4, accuracy 1.5 / n_windows, weight change within rtol 2e-2 plus a floor
    in units of lr * steps;
  - float32 storage: a float32 fit rounds every weight to float32 at every step, up to half an ulp of the weight, which a float64
    fit does not.  A float32 reference rounds the same way, so the fp32-oracle tests never see it; against float64 it is the
    largest error of a weight whose change is small beside its size (a forget-gate bias near 1 moves ~1e-3 per step in Keras
    Adam and carries up to 1.2e-7 of rounding per step, 6x the old floor of 2e-5 lr).  Every comparison allows one ulp of the
    weight per step, element by element;
  - the Adam floor (ADAM_FLOOR) is 1e-4 of lr * steps for the fp32 family and 5e-3 for the tensor cores instead of 2e-5.  A step
    is lr * m / sqrt(v), so its error is lr times the *relative* error of the weight's gradient sum: (error per product) *
    sqrt(B * L) / r, where r = |sum| / sum of |terms| says how far the sum cancels.  Over B * L ~ 100 terms that is
    ~6e-7 / r for fp32 (2^-24 per product) and ~5e-6 / r for the split-TF32 products of the tensor cores (~2^-21 each,
    lstm_fit_tc.cu).  Among a million weights some cancel to r ~ 1e-3, so the largest error is a tail, not a bound: the float32
    oracle against the float64 one reaches 4.5e-5 lr per step on this file's cases, the tensor-core family 2.4e-3 on an H100
    (10 of the 1 048 576 kernel weights at 512 features and 512 units, whose raw gradients agree in test_tile_edges_raw_gradients
    [in_u_1024]).  The floors are those tails with a margin of 2.  They only decide for weights whose change nearly cancelled:
    any other moves ~lr per step, where rtol 2e-2 is the larger term.  The raw-gradient mode, which shows the gradient sums
    themselves, keeps its tolerance.
"""
import ctypes as C
import math

import numpy as np
import pytest
from parity_helpers import close
from test_gpu_fit_coverage import GRAD_ADAM, KERAS_ADAM

pytestmark = pytest.mark.gpu


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
def km(torch):
    from oracle import keras_math

    return keras_math


SIXTEEN_ACTS = ["sigmoid" if l % 3 == 1 else "tanh" for l in range(16)]

#   name: (n_features, n_features_out, units, cell acts, head act, lookback, lookahead, windows per job, targets)
#   targets: "x" (the autoencoder / forecast of its own input), "random" (other columns in [0, 1)), "binary" (0 / 1)
NETS = {
    "production_stack": (128, 128, [256, 128, 64, 64, 128, 256], ["tanh"] * 6, "linear", 144, 0, [131, 41], "x"),
    "width512_features512": (512, 512, [512], ["tanh"], "linear", 3, 0, [70, 37], "random"),
    "two_layers_512": (512, 512, [512, 512], ["tanh"] * 2, "linear", 2, 0, [70, 37], "random"),
    "sixteen_layers": (6, 5, [8, 16] * 8, SIXTEEN_ACTS, "linear", 3, 0, [70, 37], "random"),
    "forecast_256_128": (128, 128, [256, 128], ["tanh"] * 2, "linear", 4, 1, [70, 37], "x"),
    "binary_head_512": (40, 1, [512], ["tanh"], "sigmoid", 3, 0, [70, 37], "binary"),
}

#   in + u on both sides of 32, 64, 128 and 512, with u itself on 15 / 16 / 17, 63 / 64 / 65 and 255 / 256 / 257: (n_features, units)
TILE_EDGES = {
    "in_u_31": (16, [15]),
    "in_u_32": (16, [16]),
    "in_u_33": (16, [17]),
    "in_u_63": (47, [16]),
    "in_u_64_u_63": (1, [63]),
    "in_u_65_u_64": (1, [64]),
    "in_u_127": (64, [63]),
    "in_u_128": (64, [64]),
    "in_u_129": (64, [65]),
    "in_u_511": (256, [255]),
    "in_u_512": (256, [256]),
    "in_u_513": (256, [257]),
    "in_u_1024": (512, [512]),  # the widest layer: 32 unit blocks; the tensor cores' bias row alone in the 17th weight-gradient tile
    "two_layers_in_u_60_64": (20, [40, 24]),  # layer 1: in + u = 64, its bias row alone in the last weight-gradient tile
}
TILE_EDGE_OUT, TILE_EDGE_LOOKBACK, TILE_EDGE_WINDOWS = 5, 3, [70]

FAMILIES = {"fp32": (False, 32), "tc_b64": (True, 64), "tc_b256": (True, 256)}
ADAM_FLOOR = {False: 1e-4, True: 5e-3}  # by tensor cores or not: the Keras Adam floor in units of lr * steps (module docstring)


def all_nets():
    """Every architecture this file trains: (n_features, n_features_out, units, acts, head act, lookback).  The CPU companion
    (test_lstm_fit_widths_host.py) checks that the C ABI admits each of them."""
    out = {k: v[:6] for k, v in NETS.items()}
    for k, (F, units) in TILE_EDGES.items():
        out[k] = (F, TILE_EDGE_OUT, units, ["tanh"] * len(units), "sigmoid", TILE_EDGE_LOOKBACK)
    out["footprint"] = FOOTPRINT_NET
    return out


def perturbed(km, spec, seed, rng):
    """Keras' initialisers with nonzero biases everywhere, so every bias gradient path carries a signal."""
    layers, (Wd, bd) = km.init_lstm_weights(spec, np.random.default_rng(seed))
    layers = [(K, U, b + rng.uniform(-0.1, 0.1, b.shape).astype(np.float32)) for K, U, b in layers]
    return layers, (Wd, rng.uniform(-0.1, 0.1, bd.shape).astype(np.float32))


def setup(engine, torch, km, net, nwin, lookahead, targets, seed):
    """Jobs of nwin[i] windows each, back to back in x / y, on slots 0.. of a fresh engine."""
    F, F_out, units, acts, head, L = net
    spec = km.LSTMSpec(F, list(units), list(acts), F_out, head, L)
    rng = np.random.default_rng(seed)
    ws = [perturbed(km, spec, seed + 10 + i, rng) for i in range(len(nwin))]
    rows = [n + L - 1 + lookahead for n in nwin]
    Xs = [rng.random((n, F)).astype(np.float32) for n in rows]
    if targets == "x":
        Ys = Xs
    elif targets == "binary":
        Ys = [(rng.random((n, F_out)) > 0.5).astype(np.float32) for n in rows]
    else:
        Ys = [rng.random((n, F_out)).astype(np.float32) for n in rows]
    eng = engine.LSTMEngine(F, spec.units, spec.acts, F_out, head, L)
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(len(rows)), nwin, np.concatenate([[0], np.cumsum(rows)[:-1]])), eng.device)
    x = torch.from_numpy(np.concatenate(Xs)).to(eng.device)
    y = torch.from_numpy(np.concatenate(Ys)).to(eng.device)
    return spec, eng, ws, Xs, Ys, jobs, x, y


def run_fit(eng, tc, params, jobs, nwin, x, y, B, epochs, adam, lookahead=0, state=None):
    fit = eng.fit_tc if tc else eng.fit
    return fit(params, jobs, len(nwin), max(nwin), x, y, epochs=epochs, batch_size=B, lookahead=lookahead, primer=True, adam=adam, state=state)


def float32_storage(w0, w, steps):
    """What storing the weights in float32 alone puts between a float32 fit and a float64 one after `steps` steps: each step
    rounds a weight to float32, half an ulp of it at most (a whole ulp here, for a weight crossing a power of two)."""
    return steps * np.spacing(np.maximum(np.abs(w0), np.abs(w)).astype(np.float32)).astype(np.float64)


def check_f64(km, spec, ws, Xs, Ys, got, loss, acc, nwin, epochs, B, adam, gradients, lookahead=0, floor=ADAM_FLOOR[False]):
    """Job i (slot i) against the oracle's float64 fit of the same weights, windows and batches (tolerances: module docstring)."""
    for i in range(len(Xs)):
        want_w, hist = km.lstm_fit(spec, ws[i], Xs[i], Ys[i], epochs=epochs, batch_size=B, lookahead=lookahead, lr=adam["lr"], b1=adam["beta1"],
                                   b2=adam["beta2"], eps=adam["eps"], dtype=np.float64)
        if epochs:
            close(loss[i], np.array(hist["loss"]), rtol=5e-4, name=f"job {i} loss history")
            assert np.allclose(acc[i], hist["accuracy"], atol=1.5 / nwin[i]), (i, acc[i], hist["accuracy"])
        steps = 1 + epochs * math.ceil(nwin[i] / B)
        for k, (w0, gl, wl) in enumerate(zip(km._lstm_flat(ws[i]), km._lstm_flat(got[i]), km._lstm_flat(want_w))):
            w0 = w0.astype(np.float64)
            storage = float32_storage(w0, wl, steps)
            if gradients:
                close(gl - w0, wl - w0, mag=float(np.abs(wl - w0).max()), rtol=1e-3, atol=storage, name=f"job {i} array {k}: accumulated raw gradients")
            else:  # Adam moves a weight by ~lr per step whatever the gradient's size: compare the distance travelled
                close(gl - w0, wl - w0, mag=adam["lr"] * steps, rtol=2e-2, floor=floor, atol=storage, name=f"job {i} array {k}: trained weights")


# ------------------------------------------------------------------------------------------------ 1: architectures at width
@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("case", list(NETS))
def test_fit_at_width_matches_the_float64_oracle(engine, torch, km, case, family):
    *net, lookahead, nwin, targets = NETS[case]
    tc, B = FAMILIES[family]
    if case == "production_stack":
        F, F_out, units, acts, head, L = net
        assert km.lstm_symmetric_spec(128, lookback_window=144) == km.LSTMSpec(F, units, acts, F_out, head, L)
    spec, eng, ws, Xs, Ys, jobs, x, y = setup(engine, torch, km, net, nwin, lookahead, targets, seed=41)
    params = eng.pack_params(ws)
    loss, acc, (_, _, t) = run_fit(eng, tc, params, jobs, nwin, x, y, B, 1, KERAS_ADAM, lookahead)
    torch.cuda.synchronize()
    assert [int(v) for v in t.cpu()] == [1 + math.ceil(n / B) for n in nwin]
    check_f64(km, spec, ws, Xs, Ys, eng.unpack_params(params), loss.cpu().numpy(), acc.cpu().numpy(), nwin, 1, B, KERAS_ADAM, False, lookahead,
              floor=ADAM_FLOOR[tc])


# ------------------------------------------------------------------------------------------------ 2: tile edges, raw gradients
@pytest.mark.parametrize("epochs", [0, 1])
@pytest.mark.parametrize("family", ["fp32", "tc_b64"])
@pytest.mark.parametrize("case", list(TILE_EDGES))
def test_tile_edges_raw_gradients(engine, torch, km, case, family, epochs):
    """beta1 = beta2 = 0, eps = lr = 1 with a sigmoid head: the weight change is the raw gradient sum; epochs = 0 is the primer alone."""
    tc, B = FAMILIES[family]
    net = all_nets()[case]
    spec, eng, ws, Xs, Ys, jobs, x, y = setup(engine, torch, km, net, TILE_EDGE_WINDOWS, 0, "random", seed=43)
    params = eng.pack_params(ws)
    loss, acc, (_, _, t) = run_fit(eng, tc, params, jobs, TILE_EDGE_WINDOWS, x, y, B, epochs, GRAD_ADAM)
    torch.cuda.synchronize()
    assert int(t[0]) == 1 + epochs * math.ceil(TILE_EDGE_WINDOWS[0] / B)
    check_f64(km, spec, ws, Xs, Ys, eng.unpack_params(params), loss.cpu().numpy(), acc.cpu().numpy(), TILE_EDGE_WINDOWS, epochs, B, GRAD_ADAM, True)


# ------------------------------------------------------------------------------------------------ 3: the families agree at width
@pytest.mark.parametrize("B", [1, 32])
@pytest.mark.parametrize("case", ["width512_features512", "production_stack"])
def test_families_agree_at_width(engine, torch, km, case, B):
    *net, lookahead, nwin, targets = NETS[case]
    _, eng, ws, _, _, jobs, x, y = setup(engine, torch, km, net, nwin, lookahead, targets, seed=45)
    p32, ptc = eng.pack_params(ws), eng.pack_params(ws)
    l32, a32, (_, _, t32) = run_fit(eng, False, p32, jobs, nwin, x, y, B, 1, KERAS_ADAM, lookahead)
    ltc, atc, (_, _, ttc) = run_fit(eng, True, ptc, jobs, nwin, x, y, B, 1, KERAS_ADAM, lookahead)
    torch.cuda.synchronize()
    assert torch.equal(t32, ttc)
    close(ltc.cpu().numpy(), l32.cpu().numpy(), rtol=5e-4, name="loss history")
    got32, gottc = eng.unpack_params(p32), eng.unpack_params(ptc)
    for i in range(len(nwin)):
        assert np.allclose(atc[i].cpu().numpy(), a32[i].cpu().numpy(), atol=1.5 / nwin[i])
        steps = 1 + math.ceil(nwin[i] / B)
        for k, (w0, gt, gf) in enumerate(zip(km._lstm_flat(ws[i]), km._lstm_flat(gottc[i]), km._lstm_flat(got32[i]))):
            w0 = w0.astype(np.float64)
            close(gt - w0, gf - w0, mag=KERAS_ADAM["lr"] * steps, rtol=2e-2, floor=ADAM_FLOOR[True], atol=float32_storage(w0, gf, steps),
                  name=f"job {i} array {k}: trained weights")


# ------------------------------------------------------------------------------------------------ 4: replay
@pytest.mark.parametrize("family", ["fp32", "tc_b256"])
def test_widest_fit_replays_bit_for_bit(engine, torch, km, family):
    """Two identical launches on 512 features and two 512-unit layers: the same bytes in params, m, v, t, loss and accuracy."""
    tc, B = FAMILIES[family]
    *net, lookahead, nwin, targets = NETS["two_layers_512"]
    _, eng, ws, _, _, jobs, x, y = setup(engine, torch, km, net, nwin, lookahead, targets, seed=47)
    runs = []
    for _ in range(2):
        params = eng.pack_params(ws)
        loss, acc, (m, v, t) = run_fit(eng, tc, params, jobs, nwin, x, y, B, 2, KERAS_ADAM)
        runs.append((params, m, v, t, loss, acc))
    torch.cuda.synchronize()
    for name, a, b in zip(("params", "m", "v", "t", "loss", "accuracy"), *runs):
        assert torch.equal(a, b), name
    assert bool(torch.isfinite(runs[0][0]).all())


# ------------------------------------------------------------------------------------------------ 5: what a fit reads and writes
FOOTPRINT_NET = (33, 33, [40, 24], ["tanh", "tanh"], "linear", 4)  # layer 1: in + u = 64


@pytest.mark.parametrize("lookahead", [0, 1])
@pytest.mark.parametrize("family", list(FAMILIES))
def test_fit_reads_only_its_windows_and_targets_and_writes_only_its_slots(engine, torch, km, family, lookahead):
    """
    Three jobs with gaps between them, on slots 3, 0 and 4 of five.  Every x row outside the jobs' windows and every y row that is
    not a target is NaN: the trained slots, their Adam state and the history must be finite and equal, bit for bit, those of the
    same fit on finite rows everywhere.  Slots 1 and 2, and the padding of every slot past the parameters, are left as they were.
    """
    tc, B = FAMILIES[family]
    F, F_out, units, acts, head, L = FOOTPRINT_NET
    spec = km.LSTMSpec(F, units, acts, F_out, head, L)
    eng = engine.LSTMEngine(F, units, acts, F_out, head, L)
    rng = np.random.default_rng(49 + lookahead)
    nwin = np.array([70, 33, 5])
    span = nwin + L - 1 + lookahead                 # rows from a job's first x row to its last target
    gaps = np.array([2, 3, 3])
    x_row = np.cumsum(gaps) + np.concatenate([[0], np.cumsum(span)[:-1]])
    n_rows = int(x_row[-1] + span[-1] + 2)
    X = rng.random((n_rows, F)).astype(np.float32)
    Y = rng.random((n_rows, F_out)).astype(np.float32)
    x_used = np.zeros(n_rows, bool)
    y_used = np.zeros(n_rows, bool)
    for r, n in zip(x_row, nwin):
        x_used[r:r + n + L - 1] = True
        y_used[r + L - 1 + lookahead:r + L - 1 + lookahead + n] = True
    Xn, Yn = X.copy(), Y.copy()
    Xn[~x_used] = np.nan
    Yn[~y_used] = np.nan
    slots = np.array([3, 0, 4])
    S = 5
    host = np.zeros((S, eng.param_stride), np.float32)
    host[:] = rng.uniform(-0.5, 0.5, host.shape)   # padding past n_params included
    for s in slots:
        layers, dense = perturbed(km, spec, 100 + s, rng)
        host[s, :eng.n_params] = np.concatenate([a.ravel() for a in km._lstm_flat((layers, dense))])
    m0 = rng.uniform(-1e-3, 1e-3, host.shape).astype(np.float32)
    v0 = rng.uniform(0, 1e-6, host.shape).astype(np.float32)
    t0 = np.array([0, 7, 9, 0, 0], np.int32)
    jobs = engine.jobs_to_device(engine.make_jobs(slots, nwin, x_row), eng.device)
    runs = []
    for Xa, Ya in ((X, Y), (Xn, Yn)):
        params = torch.from_numpy(host.copy()).to(eng.device)
        state = tuple(torch.from_numpy(a.copy()).to(eng.device) for a in (m0, v0, t0))
        x, y = torch.from_numpy(Xa).to(eng.device), torch.from_numpy(Ya).to(eng.device)
        loss, acc, (m, v, t) = run_fit(eng, tc, params, jobs, list(nwin), x, y, B, 2, KERAS_ADAM, lookahead, state)
        torch.cuda.synchronize()
        runs.append([a.cpu().numpy() for a in (params, m, v, t, loss, acc)])
    for name, clean, dirty in zip(("params", "m", "v", "t", "loss", "accuracy"), *runs):
        assert np.array_equal(clean, dirty, equal_nan=False), f"{name}: the NaN rows changed the fit"
    params, m, v, t, loss, acc = runs[1]
    assert np.isfinite(loss).all() and np.isfinite(acc).all()
    assert np.isfinite(params[slots, :eng.n_params]).all() and np.isfinite(m[slots]).all() and np.isfinite(v[slots]).all()
    assert not np.array_equal(params[slots, :eng.n_params], host[slots, :eng.n_params]), "nothing was trained"
    for s in (1, 2):
        assert np.array_equal(params[s], host[s]) and np.array_equal(m[s], m0[s]) and np.array_equal(v[s], v0[s]) and t[s] == t0[s], f"slot {s}"
    pad = slice(eng.n_params, eng.param_stride)
    assert np.array_equal(params[:, pad], host[:, pad]) and np.array_equal(m[:, pad], m0[:, pad]) and np.array_equal(v[:, pad], v0[:, pad])
    assert [int(t[s]) for s in slots] == [1 + 2 * math.ceil(n / B) for n in nwin]


SENTINEL = np.float32(-3.0e33)


@pytest.mark.parametrize("family", ["fp32", "tc_b256"])
@pytest.mark.parametrize("case", ["production_stack", "sixteen_layers"])
def test_fit_stays_inside_its_reported_workspace(engine, torch, km, case, family):
    """
    One call of gb_lstm_fit_stop / gb_lstm_fit_tc_stop through ctypes, as LSTMEngine._fit_launch makes it, on a workspace of the
    size gb_lstm_fit(_tc)_workspace_bytes reports filled with NaN and followed by 1 MB of a sentinel.  The sentinel is intact
    afterwards, and the fit equals the engine's own launch on a fresh workspace bit for bit (no workspace word is read before
    the fit has written it).
    """
    from gordo_components_b200 import _cabi

    tc, B = FAMILIES[family]
    *net, lookahead, nwin, targets = NETS[case]
    _, eng, ws, _, _, jobs, x, y = setup(engine, torch, km, net, nwin, lookahead, targets, seed=51)
    ws_bytes = eng.fit_tc_workspace_bytes(len(nwin), B) if tc else eng.fit_workspace_bytes(len(nwin))
    assert ws_bytes > 0 and ws_bytes % 4 == 0
    tail = (1 << 20) // 4
    work = torch.full((ws_bytes // 4 + tail,), float("nan"), dtype=torch.float32, device=eng.device)
    work[ws_bytes // 4:] = float(SENTINEL)
    params = eng.pack_params(ws)
    m, v = torch.zeros_like(params), torch.zeros_like(params)
    t = torch.zeros((params.shape[0],), dtype=torch.int32, device=eng.device)
    hist = torch.zeros((len(nwin), 1), dtype=torch.float32, device=eng.device)
    acc = torch.zeros_like(hist)
    hp = _cabi.GbLstmFitHParams()
    hp.epochs, hp.batch_size, hp.lookahead, hp.primer = 1, B, lookahead, 1
    hp.lr, hp.beta1, hp.beta2, hp.eps = KERAS_ADAM["lr"], KERAS_ADAM["beta1"], KERAS_ADAM["beta2"], KERAS_ADAM["eps"]
    entry = eng.lib.gb_lstm_fit_tc_stop if tc else eng.lib.gb_lstm_fit_stop
    p = _cabi.ptr
    _cabi.check(entry(C.byref(eng.net), p(params), p(m), p(v), p(t), p(jobs), len(nwin), max(nwin), p(x), p(y), C.byref(hp), p(work), p(hist),
                      p(acc), _cabi.loss_code("mse"), None, None, None, None, None, engine._stream_ptr()))
    ref = eng.pack_params(ws)
    rloss, racc, (rm, rv, rt) = run_fit(eng, tc, ref, jobs, nwin, x, y, B, 1, KERAS_ADAM, lookahead)
    torch.cuda.synchronize()
    rest = work[ws_bytes // 4:].cpu().numpy()
    assert (rest == SENTINEL).all(), f"{int((rest != SENTINEL).sum())} words past the reported workspace were written"
    assert bool(torch.isfinite(params).all()) and bool(torch.isfinite(hist).all())
    for name, a, b in (("params", params, ref), ("m", m, rm), ("v", v, rv), ("t", t, rt), ("loss", hist, rloss), ("accuracy", acc, racc)):
        assert torch.equal(a, b), name


# ------------------------------------------------------------------------------------------------ 6: orthogonal initialiser at width
@pytest.mark.parametrize("u", [1, 2, 64, 256, 512])
def test_orthonormal_rows_at_width(engine, torch, u):
    """Three [u, 4u] draws written at an offset of 7 words with a stride of one matrix plus 13: each is numpy's QR made
    sign-positive (Keras' Orthogonal), its float32 rows are orthonormal, and no word outside the three matrices is written."""
    dev = engine.cuda_device()
    n, ofs, extra = 3, 7, 13
    size = u * 4 * u
    g = torch.randn((n, u, 4 * u), dtype=torch.float64, device=dev, generator=torch.Generator(device=dev).manual_seed(u))
    draw = g.cpu().numpy()
    out = torch.full((ofs + n * (size + extra) + 5,), float(SENTINEL), dtype=torch.float32, device=dev)
    engine.orthonormal_rows(g, out, ofs, size + extra)
    got = out.cpu().numpy()
    written = np.zeros(got.size, bool)
    for i in range(n):
        s = ofs + i * (size + extra)
        written[s:s + size] = True
        q, r = np.linalg.qr(draw[i].T)
        want = (q * np.sign(np.diag(r))).T
        mat = got[s:s + size].reshape(u, 4 * u)
        np.testing.assert_allclose(mat, want, atol=2e-6, rtol=0, err_msg=f"matrix {i}")
        m64 = mat.astype(np.float64)
        np.testing.assert_allclose(m64 @ m64.T, np.eye(u), atol=1e-5, rtol=0, err_msg=f"matrix {i}: U U^T")
    assert (got[~written] == SENTINEL).all(), "words outside the matrices were written"
