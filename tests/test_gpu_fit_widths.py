"""
The Dense fit kernels (csrc/ffae_fit.cu, ffae_fit_body.cuh) at the widths, depths and memory plans they admit: the widest symmetric
(172 tags) and hourglass (196 tags) stacks, 16 layers, one layer, a 1-wide input and a 1-wide head at width 256, and every width of
a layer pair on both sides of the 4-float padding and the 16-float tile.  Every fit is compared with the oracle's float64 fit loop
(oracle/keras_math.py ff_fit, dtype=np.float64) from the same injected weights and visiting order, so the error measured is the
kernel's own.  hourglass(197), whose activations leave less shared memory than the kernels' own static arrays need, is refused
before any launch.

Where these shapes reach code the narrow tests do not:
  - input_grad sums a layer's Np / 4 column blocks a quarter per lane group: the last round is ragged when Np % 16 != 0, and its
    task loop wraps past the 16 warps once K > 64;
  - weight_step grid-strides over the (Kp / 4) * (Np / 2) blocks of a layer once there are more than 512 of them;
  - the gather of the next chunk goes to the warps without a tile in the narrowest layers, to all of them once that layer is 64
    wide, and to both halves of the chunk in the same layer when the stack has one layer;
  - the bias and weight gradients sum all 32 rows of a chunk, so every dz row past a partial chunk's rows must be written as 0,
    also in the dz buffers the (1, 1) .. (1, 3) plans keep in the slot's Adam-v area (L2), next to the gradient scratch of
    multi-chunk mini-batches and the weight image in the Adam-m area.

Tolerances (the terms of parity_helpers.close: rtol * |want| + floor * mag + atol):
  - raw-gradient mode (beta1 = beta2 = 0, lr = eps = a power of two at least 1e3 x the largest gradient of the oracle's first step:
    a step is -g eps / (|g| + eps), within 1e-3 of -g): the weight change within rtol 1e-3 plus 2e-5 of the array's largest change,
    as in tests/test_gpu_fit_coverage.py;
  - Keras Adam: the trained weights within rtol 1e-4 plus 2e-5 of the layer's largest weight (biases: of max(largest bias, 1e-2)),
    as in test_gpu_fit_coverage.py; loss history rtol 5e-4; accuracy history 2 rows of the job;
  - float32 storage (atol): a float32 fit rounds every weight to float32 at every step, half an ulp of it at most (a whole ulp
    for a weight crossing a power of two), which the float64 reference does not.  A float32 reference rounds the same way, so the
    float32-oracle tests never see it.  Every weight comparison allows one ulp of the weight per optimizer step, element by
    element (float32_storage);
  - the Keras Adam floor (atol, ADAM_FLOOR * lr * steps).  An Adam step is lr * m / sqrt(v), so its error is lr times the
    relative error of the weight's gradient sums, (error per product) * sqrt(terms) / r, where r = |sum| / sum of |terms| says
    how far the sum cancels.  Summed over B rows in float32 (2^-24 per product) that is ~1e-6 / r, and among the 10^5 weights of a
    wide stack some cancel to r ~ 1e-3: the largest error is a tail, not a bound.  Beyond the rtol and storage terms, the float32
    oracle against the float64 one reaches 1.4e-6 lr per step on this file's Keras Adam cases (symmetric(172)), and the kernel
    8.4e-7 (the 16-layer 64-wide stack) on an H100 80GB HBM3 at its 700 W power limit.  ADAM_FLOOR is the larger with a margin of
    2, rounded up: 3e-6.  It only decides for weights whose gradient nearly cancelled: any other weight is held to the rtol term.
"""
import ctypes as C
import math

import numpy as np
import pytest
from parity_helpers import close
from test_gpu_fit_coverage import KERAS_ADAM, uniform_perm, waves

from oracle import keras_math as km

pytestmark = pytest.mark.gpu

ADAM_FLOOR = 3e-6  # Keras Adam floor in units of lr * steps (module docstring)


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


def mixed(L):
    """L layers cycling tanh, relu, sigmoid, with a linear output."""
    return [("tanh", "relu", "sigmoid")[l % 3] for l in range(L - 1)] + ["linear"]


def stack(dims, acts=None, l1=None):
    return km.FFSpec(list(dims), list(acts) if acts else ["tanh"] * (len(dims) - 2) + ["linear"], list(l1) if l1 else [])


# ------------------------------------------------------------------------------------------------ the stacks this file trains
# raw gradients, one layer pair [w_in, w_hidden, w_out] -> memory plan: widths 1 .. 256 on both sides of the padding (4) and the
# tile (16), n_in != n_out, and output widths whose Np % 16 is 4 (17, 65, 129), 8 (40) and 12 (44, 236) past the first quarter
# round; the pairs wide enough for the L2 plans cover (1, 0) .. (1, 3) too
TILE_EDGES = {
    "1_3_1": ([1, 3, 1], (0, 0)),
    "4_5_15": ([4, 5, 15], (0, 0)),
    "16_17_31": ([16, 17, 31], (0, 0)),
    "32_33_63": ([32, 33, 63], (0, 0)),
    "33_32_17": ([33, 32, 17], (0, 0)),
    "63_64_65": ([63, 64, 65], (0, 0)),
    "64_65_127": ([64, 65, 127], (0, 0)),
    "65_63_40": ([65, 63, 40], (0, 0)),
    "15_31_44": ([15, 31, 44], (0, 0)),
    "127_128_129": ([127, 128, 129], (1, 0)),
    "128_129_255": ([128, 129, 255], (1, 1)),
    "255_256_236": ([255, 256, 236], (1, 2)),
    "256_255_256": ([256, 255, 256], (1, 3)),
}
#   name: (batch, rows per job): one or two mini-batches; 33 and 80 are multi-chunk with a ragged last chunk, as is the batch of
#   100 over a 70-row job (one mini-batch of 32 + 32 + 6 rows)
GRAD_BATCHES = {"b1": (1, 2), "b31": (31, 50), "b32": (32, 50), "b33": (33, 50), "b80": (80, 130), "b100_job70": (100, 70)}

# one stack in each memory plan (weights in L2, dz buffers in L2), raw gradients at batch 33 and 80
PLAN_STACKS = {
    "hourglass_64": ((0, 0), km.ff_hourglass_spec(64)),
    "symmetric_10": ((1, 0), km.ff_symmetric_spec(10)),
    "w129_129_129": ((1, 0), stack([129, 129, 129])),
    "symmetric_64": ((1, 1), km.ff_symmetric_spec(64)),
    "symmetric_96": ((1, 2), km.ff_symmetric_spec(96)),
    "w256_128_256": ((1, 2), stack([256, 128, 256])),
    "symmetric_172": ((1, 3), km.ff_symmetric_spec(172)),
    "hourglass_196": ((1, 3), km.ff_hourglass_spec(196)),
}

#   Keras Adam, several epochs.  name: (spec, plan, l1_div_batch, targets, rows per job, batch, epochs)
#   targets: "x" (autoencoder), "waves" (other columns), "binary" (0 / 1)
EVERY_LAYER_L1 = [1e-4] * 16
NETS = {
    "symmetric_172": (km.ff_symmetric_spec(172), (1, 3), False, "x", [150, 97], 32, 3),
    "model_172": (km.ff_model_spec(172), (1, 3), False, "x", [150, 97], 80, 3),
    "hourglass_196": (km.ff_hourglass_spec(196), (1, 3), False, "x", [150, 97], 32, 3),
    "hourglass_80": (km.ff_hourglass_spec(80), (0, 0), False, "x", [150, 97], 50, 3),
    "sixteen_layers_32": (stack([32] * 17, mixed(16), EVERY_LAYER_L1), (0, 0), False, "x", [150, 97], 32, 3),
    "sixteen_layers_64_l1_div_batch": (stack([64] * 17, mixed(16), EVERY_LAYER_L1), (1, 0), True, "x", [150, 97], 32, 3),
    "one_layer_64": (stack([64, 64], ["linear"]), (0, 0), False, "waves", [150, 97], 32, 3),
    "one_layer_256": (stack([256, 256], ["linear"]), (1, 2), False, "waves", [150, 97], 80, 3),
    "n_in_1": (stack([1, 64, 256]), (1, 0), False, "waves", [150, 97], 32, 3),
    "binary_head_256": (stack([256, 128, 1], ["tanh", "sigmoid"]), (1, 0), False, "binary", [150, 97], 32, 3),
}

FOOTPRINT_STACKS = {"hourglass_64": ((0, 0), km.ff_hourglass_spec(64)), "w129_129_129": ((1, 0), stack([129, 129, 129])),
                    "symmetric_172": ((1, 3), km.ff_symmetric_spec(172))}


def all_stacks():
    """Every stack this file trains and the memory plan it is pinned to: name -> (spec, (weights in L2, dz buffers in L2)).  The
    CPU companion (test_fit_widths_host.py) checks each plan without a GPU."""
    out = {f"tile_edge_{k}": (stack(d), p) for k, (d, p) in TILE_EDGES.items()}
    out.update({f"plan_{k}": (s, p) for k, (p, s) in PLAN_STACKS.items()})
    out.update({f"net_{k}": (v[0], v[1]) for k, v in NETS.items()})
    out.update({f"footprint_{k}": (s, p) for k, (p, s) in FOOTPRINT_STACKS.items()})
    return out


# ------------------------------------------------------------------------------------------------ helpers
def ff_plan(spec):
    from gordo_components_b200 import _cabi

    net = _cabi.make_ffnet(spec.dims, spec.acts, spec.l1)
    w, d = C.c_int32(-1), C.c_int32(-1)
    rc = _cabi.load_library().gb_ffae_fit_plan(C.byref(net), C.byref(w), C.byref(d))
    return rc, w.value, d.value


def start_weights(spec, seed):
    """Glorot kernels and biases in +-0.2, so that every bias gradient path carries a signal."""
    rng = np.random.default_rng(seed)
    return [(W, rng.uniform(-0.2, 0.2, b.shape).astype(np.float32)) for W, b in km.init_ff_weights(spec, rng)]


def case_data(spec, rows, targets, seed):
    rng = np.random.default_rng(seed)
    Xs = [waves(rng, n, spec.dims[0]) for n in rows]
    if targets == "x":
        Ys = Xs
    elif targets == "binary":
        Ys = [(rng.random((n, 1)) > 0.5).astype(np.float32) for n in rows]
    else:
        Ys = [waves(rng, n, spec.dims[-1]) for n in rows]
    return Xs, Ys, [start_weights(spec, seed + 7 * j) for j in range(len(rows))]


def job_perms(rows, E, seed):
    """[jobs, E, max rows]: job j's visiting order of epoch e in its first rows[j] entries."""
    perm = np.zeros((len(rows), E, max(rows)), np.int32)
    for j, n in enumerate(rows):
        perm[j, :, :n] = uniform_perm(1, E, n, seed + 31 * j)[0]
    return perm


def gpu_fit(engine, torch, spec, w0s, Xs, Ys, perm, E, B, adam, l1_div_batch=False):
    """One gb_ffae_fit launch over back-to-back jobs on slots 0..: (trained weights per slot, loss, accuracy) on the host."""
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    rows = [len(x) for x in Xs]
    params = eng.pack_params(w0s)
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(len(rows)), rows, np.concatenate([[0], np.cumsum(rows)[:-1]])), eng.device)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)  # noqa: E731
    loss, acc, _ = eng.fit(params, jobs, len(rows), max(rows), dev(np.concatenate(Xs)), dev(np.concatenate(Ys)), epochs=E, batch_size=B,
                           perm=dev(perm), adam=adam, l1_div_batch=l1_div_batch)
    torch.cuda.synchronize()
    return eng.unpack_params(params), loss.cpu().numpy(), acc.cpu().numpy()


def float32_storage(w0, w, steps):
    """What storing the weights in float32 alone puts between a float32 fit and a float64 one after `steps` steps: each step
    rounds a weight to float32, half an ulp of it at most (a whole ulp here, for a weight crossing a power of two)."""
    return steps * np.spacing(np.maximum(np.abs(w0), np.abs(w)).astype(np.float32)).astype(np.float64)


def grad_adam(spec, w0s, Xs, Ys, perm, B, l1_div_batch=False):
    """beta1 = beta2 = 0 and lr = eps = the first power of two at or above 1e3 x the largest gradient of any job's first step."""
    g = 0.0
    for j, (X, Y) in enumerate(zip(Xs, Ys)):
        idx = perm[j, 0, :len(X)][:B]
        _, _, grads, _ = km.ff_loss_and_grads(spec, w0s[j], X[idx], Y[idx], np.float64, l1_div_batch)
        g = max(g, max(float(np.abs(a).max()) for pair in grads for a in pair))
    eps = 2.0 ** math.ceil(math.log2(1e3 * max(g, 1e-30)))
    return {"lr": eps, "beta1": 0.0, "beta2": 0.0, "eps": eps}


def check_f64(spec, w0s, Xs, Ys, perm, got, loss, acc, E, B, adam, l1_div_batch=False, gradients=False):
    """Job j (slot j) against the oracle's float64 fit of the same weights over the same visiting order (module docstring)."""
    for j in range(len(Xs)):
        n = len(Xs[j])
        w_ref, hist, _ = km.ff_fit(spec, w0s[j], Xs[j], Ys[j], epochs=E, batch_size=B, perms=[perm[j, e, :n] for e in range(E)], lr=adam["lr"],
                                   b1=adam["beta1"], b2=adam["beta2"], eps=adam["eps"], l1_div_batch=l1_div_batch, dtype=np.float64)
        steps = E * math.ceil(n / B)
        for l, ((Wg, bg), (Wr, br), (W0, b0)) in enumerate(zip(got[j], w_ref, w0s[j])):
            for g_, r_, z_, what in ((Wg, Wr, W0, "W"), (bg, br, b0, "b")):
                z_ = z_.astype(np.float64)
                storage = float32_storage(z_, r_, steps)
                if gradients:  # the weight change is (nearly) minus the summed gradient of every step
                    close(g_ - z_, r_ - z_, mag=float(np.abs(r_ - z_).max()), rtol=1e-3, atol=storage, name=f"job {j} raw gradients {what}{l}")
                else:
                    mag = float(np.abs(r_).max()) if what == "W" else max(float(np.abs(r_).max()), 1e-2)
                    close(g_, r_, mag=mag, atol=storage + ADAM_FLOOR * adam["lr"] * steps, name=f"job {j} {what}{l}")
        close(loss[j], np.array(hist["loss"]), mag=0.0, rtol=5e-4, name=f"job {j} loss history")
        close(acc[j], np.array(hist["accuracy"]), mag=0, rtol=0, atol=2.0 / n, name=f"job {j} accuracy history")


def run_raw_gradients(engine, torch, spec, B, N, seed):
    rows = [N, N - N // 3] if N > 2 else [N, N]
    Xs, Ys, w0s = case_data(spec, rows, "waves", seed)
    perm = job_perms(rows, 1, seed)
    adam = grad_adam(spec, w0s, Xs, Ys, perm, B)
    got, loss, acc = gpu_fit(engine, torch, spec, w0s, Xs, Ys, perm, 1, B, adam)
    check_f64(spec, w0s, Xs, Ys, perm, got, loss, acc, 1, B, adam, gradients=True)


# ------------------------------------------------------------------------------------------------ a: raw gradients
@pytest.mark.parametrize("batch", list(GRAD_BATCHES))
@pytest.mark.parametrize("case", list(TILE_EDGES))
def test_tile_edges_raw_gradients(engine, torch, case, batch):
    dims, want = TILE_EDGES[case]
    spec = stack(dims)
    assert ff_plan(spec) == (0, *want)
    B, N = GRAD_BATCHES[batch]
    run_raw_gradients(engine, torch, spec, B, N, seed=3)


@pytest.mark.parametrize("batch", ["b33", "b80"])
@pytest.mark.parametrize("case", list(PLAN_STACKS))
def test_every_memory_plan_raw_gradients(engine, torch, case, batch):
    """Batch 80 in the (1, 2) and (1, 3) plans uses the gradient scratch and the dz buffers in L2 in the same step."""
    want, spec = PLAN_STACKS[case]
    assert ff_plan(spec) == (0, *want)
    B, N = GRAD_BATCHES[batch]
    run_raw_gradients(engine, torch, spec, B, N, seed=5)


# ------------------------------------------------------------------------------------------------ b: Keras Adam at the limits
@pytest.mark.parametrize("case", list(NETS))
def test_fit_at_the_limits_matches_the_float64_oracle(engine, torch, case):
    spec, want, div, targets, rows, B, E = NETS[case]
    assert ff_plan(spec) == (0, *want)
    Xs, Ys, w0s = case_data(spec, rows, targets, seed=11)
    perm = job_perms(rows, E, seed=13)
    got, loss, acc = gpu_fit(engine, torch, spec, w0s, Xs, Ys, perm, E, B, KERAS_ADAM, l1_div_batch=div)
    check_f64(spec, w0s, Xs, Ys, perm, got, loss, acc, E, B, KERAS_ADAM, l1_div_batch=div)


@pytest.mark.parametrize("kind,T", [("symmetric", 173), ("hourglass", 197)])
def test_first_stacks_past_the_plans_are_refused_before_any_launch(engine, torch, kind, T):
    """symmetric(173) and hourglass(197) need more shared memory than a block has beside the kernels' static arrays: gb_ffae_fit
    returns GB_E_SMEM, a ValueError naming shared memory, and leaves the slot and its state as they were."""
    spec = km.ff_symmetric_spec(T) if kind == "symmetric" else km.ff_hourglass_spec(T)
    assert ff_plan(spec)[0] == -4
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    params = torch.full((1, eng.param_stride), 0.25, device=eng.device)
    m = torch.zeros((1, eng.state_stride), device=eng.device)
    v = torch.zeros_like(m)
    x = torch.rand((40, T), device=eng.device)
    with pytest.raises(ValueError, match="shared memory"):
        eng.fit(params, engine.jobs_to_device(engine.uniform_jobs(1, 40), eng.device), 1, 40, x, x, epochs=1, state=(m, v))
    torch.cuda.synchronize()
    assert bool((params == 0.25).all()) and not bool(m.any()) and not bool(v.any())


# ------------------------------------------------------------------------------------------------ c: weight regularizers at width
def test_regularized_fit_at_the_widest_symmetric_stack(engine, torch):
    """L1L2 kernel and bias terms on every layer of symmetric(172), the (1, 3) plan, against the float64 restatement of
    tests/test_gpu_raw_regressor.py (its loss and optimizer oracles plus the penalty)."""
    from test_gpu_raw_regressor import check, gpu_fit as reg_fit, oracle_fit, perms_for, reg_record

    spec = km.ff_symmetric_spec(172)
    assert ff_plan(spec) == (0, 1, 3)
    M, N, E, B = 2, 120, 2, 80
    Xs, Ys, w0s = case_data(spec, [N] * M, "x", seed=17)
    reg = reg_record(spec.n_layers, kernel_l1=1e-4, kernel_l2=5e-4, bias_l1=1e-3, bias_l2=1e-2)
    perm = perms_for(M, E, N, 19)
    got, loss, _ = reg_fit(engine, torch, spec, w0s, Xs, Ys, reg, E, B, perm)
    for j in range(M):
        want, hist = oracle_fit(spec, w0s[j], Xs[j], Ys[j], reg, epochs=E, batch_size=B, perms=perm[j])
        check(got[j], want, loss[j], hist, f"symmetric(172) job {j}")


def test_zero_regularizer_record_is_the_optimizer_kernel_at_width(engine, torch):
    """gb_ffae_fit_reg with a record of zeros runs exactly gb_ffae_fit_opt on symmetric(172): the same bytes everywhere."""
    from gordo_components_b200 import _cabi

    spec = km.ff_symmetric_spec(172)
    M, N, E, B = 2, 100, 2, 80
    Xs, Ys, w0s = case_data(spec, [N] * M, "x", seed=23)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    lib = _cabi.load_library()
    p = _cabi.ptr
    x = torch.from_numpy(np.concatenate(Xs)).to(eng.device)
    jobs = engine.jobs_to_device(engine.uniform_jobs(M, N), eng.device)
    hp = engine._fit_hparams(E, B, True, None, None, 5, False, 0, "mse")
    results = []
    for rec in ("opt", _cabi.make_dense_reg(kernel_l1=[0.0] * spec.n_layers, bias_l2=[0.0] * spec.n_layers)):
        params = eng.pack_params(w0s)
        m, v = eng._fit_state(params, None)
        out = [torch.full((M, E), float("nan"), device=eng.device) for _ in range(4)]
        args = (C.byref(eng.net), p(params), p(m), p(v), p(jobs), None, M, N, p(x), p(x), None, None, C.byref(hp), B,
                *(p(t) for t in out), None, None, None, None, None)
        if rec == "opt":
            _cabi.check(lib.gb_ffae_fit_opt(*args, None))
        else:
            _cabi.check(lib.gb_ffae_fit_reg(*args, C.byref(rec), None))
        torch.cuda.synchronize()
        results.append([params.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy()] + [t.cpu().numpy() for t in out])
    for a, b in zip(*results):
        assert np.array_equal(a, b, equal_nan=True)
    assert np.isfinite(results[0][3]).all()


# ------------------------------------------------------------------------------------------------ d: what a fit reads and writes
SENTINEL = np.float32(-3.0e33)


@pytest.mark.parametrize("case", list(FOOTPRINT_STACKS))
def test_fit_reads_only_its_rows_and_writes_only_its_slots(engine, torch, case):
    """
    Three ragged jobs on slots 3, 0 and 4 of five, the first two over overlapping x rows, at row offsets that are not multiples of
    4.  Every x and y row outside the jobs is NaN, and so are the gradient scratch and dz thirds of the trained slots' state (a
    fit writes them before it reads them): the trained slots, their moments and the history must be finite and equal, bit for
    bit, those of the same fit on finite rows and zero scratch.  Slots 1 and 2 (parameters, padding and state) keep their
    sentinel values, and the 1 MB past the last slot's parameter and state strides is intact.
    """
    want, spec = FOOTPRINT_STACKS[case]
    assert ff_plan(spec) == (0, *want)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    n_in, n_out = spec.dims[0], spec.dims[-1]
    rng = np.random.default_rng(29)
    slots, lens, x_row = np.array([3, 0, 4]), np.array([70, 33, 5]), np.array([3, 41, 119])  # jobs 0 and 1 share rows 41 .. 72
    n_rows = int(x_row[-1] + lens[-1] + 6)
    X = waves(rng, n_rows, n_in)
    Y = waves(rng, n_rows, n_out)
    used = np.zeros(n_rows, bool)
    for r, n in zip(x_row, lens):
        used[r:r + n] = True
    Xn, Yn = X.copy(), Y.copy()
    Xn[~used] = np.nan
    Yn[~used] = np.nan
    S, ps, ss, wf = 5, eng.param_stride, eng.state_stride, eng.state_stride // 3
    tail = (1 << 20) // 4
    host = np.full(S * ps + tail, SENTINEL, np.float32)
    m0 = np.full(S * ss + tail, SENTINEL, np.float32)
    v0 = m0.copy()
    for s in slots:
        w = start_weights(spec, 100 + int(s))
        host[s * ps:s * ps + eng.n_params] = np.concatenate([a.ravel() for pair in w for a in pair])
        m0[s * ss:s * ss + wf] = rng.uniform(-1e-3, 1e-3, wf)
        v0[s * ss:s * ss + wf] = rng.uniform(0, 1e-6, wf)
    E, B = 2, 32
    perm = job_perms(list(lens), E, seed=31)
    jobs = engine.jobs_to_device(engine.make_jobs(slots, lens, x_row), eng.device)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)  # noqa: E731
    runs = []
    for Xa, Ya, scratch in ((X, Y, 0.0), (Xn, Yn, np.nan)):
        m, v = m0.copy(), v0.copy()
        for s in slots:
            m[s * ss + wf:(s + 1) * ss] = scratch
            v[s * ss + wf:(s + 1) * ss] = scratch
        pt, mt, vt = dev(host), dev(m), dev(v)
        loss, acc, _ = eng.fit(pt[:S * ps].view(S, ps), jobs, len(slots), int(lens.max()), dev(Xa), dev(Ya), epochs=E, batch_size=B,
                               perm=dev(perm), state=(mt[:S * ss].view(S, ss), vt[:S * ss].view(S, ss)))
        torch.cuda.synchronize()
        runs.append([a.cpu().numpy() for a in (pt, mt, vt, loss, acc)])
    (pc, mc, vc, lc, ac), (pd, md, vd, ld, ad) = runs
    moments = np.zeros(S * ss + tail, bool)
    for s in slots:
        moments[s * ss:s * ss + wf] = True
    assert np.array_equal(pc, pd) and np.array_equal(lc, ld) and np.array_equal(ac, ad), "the NaN rows or scratch changed the fit"
    assert np.array_equal(mc[moments], md[moments]) and np.array_equal(vc[moments], vd[moments]), "the NaN rows or scratch changed the moments"
    assert np.isfinite(ld).all() and np.isfinite(ad).all() and np.isfinite(md[moments]).all() and np.isfinite(vd[moments]).all()
    trained = np.zeros(S * ps + tail, bool)
    for s in slots:
        trained[s * ps:s * ps + eng.n_params] = True
    assert np.isfinite(pd[trained]).all() and not np.array_equal(pd[trained], host[trained]), "nothing was trained"
    assert np.array_equal(pd[~trained], host[~trained]), "parameters of another slot, the padding or the tail were written"
    untouched = np.ones(S * ss + tail, bool)
    for s in slots:
        untouched[s * ss:(s + 1) * ss] = False
    for name, got, start in (("m", md, m0), ("v", vd, v0)):
        assert np.array_equal(got[untouched], start[untouched]), f"adam_{name} of another slot or past the last state stride was written"


@pytest.mark.parametrize("case", ["symmetric_172", "hourglass_196"])
def test_widest_fit_replays_bit_for_bit(engine, torch, case):
    """Two identical launches at batch 80 (scratch and dz buffers in L2): the same bytes in params, m, v, loss and accuracy."""
    spec = NETS[case][0]
    rows, E, B = [150, 97], 2, 80
    Xs, _, w0s = case_data(spec, rows, "x", seed=37)
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    x = torch.from_numpy(np.concatenate(Xs)).to(eng.device)
    jobs = engine.jobs_to_device(engine.make_jobs([0, 1], rows, [0, rows[0]]), eng.device)
    runs = []
    for _ in range(2):
        params = eng.pack_params(w0s)
        loss, acc, (m, v) = eng.fit(params, jobs, 2, max(rows), x, x, epochs=E, batch_size=B, seed=41)
        runs.append((params, m, v, loss, acc))
    torch.cuda.synchronize()
    for name, a, b in zip(("params", "m", "v", "loss", "accuracy"), *runs):
        assert torch.equal(a, b), name
    assert bool(torch.isfinite(runs[0][0]).all())
