"""
Comparison helpers shared by the GPU parity tests.

Tolerance (north_star: "within 1e-4 relative"): model output |got - want| <= 1e-4*|want| + 2e-5*magnitude, where the
second term covers outputs near zero (the split-precision tensor-core path measures ~2e-6 of the magnitude, so a
regression of its operand scheme shows).
"""
import numpy as np

RTOL = 1e-4
FLOOR = 2e-5  # absolute part of the tolerance, in units of the data magnitude: the tensor-core split-precision path measures ~2e-6


def close(got, want, mag=1.0, rtol=RTOL, name="", atol=0.0, floor=FLOOR):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (name, got.shape, want.shape)
    err = np.abs(got - want)
    tol = rtol * np.abs(want) + floor * mag + atol
    bad = ~(err <= tol) & ~(np.isnan(got) & np.isnan(want))
    assert not bad.any(), f"{name}: {bad.sum()} of {bad.size} outside tolerance; max err {err[bad].max():.3e} (tol {tol[bad].min():.3e})"


def _opt(name, **kw):
    from gordo_components_b200.machine.model.factories.specs import resolve_optimizer

    return resolve_optimizer(name, kw)


# The three kernel families of the Dense fit (csrc/ffae_fit.cu launch_fit), as keyword arguments of FFEngine.fit / fit_split: MSE with
# Adam; another loss (the LOSS kernels); another optimizer (the LOSS + OPT kernels).  Plain Adam through gb_ffae_fit_opt runs the Adam
# kernels, so every optimizer here is another rule.  Centered RMSprop keeps its mean gradient in state slot 1, the area whose two spare
# thirds hold the dz buffers that the L2 memory plans move out of shared memory.
FIT_KW = {
    "mse-adam": {},
    "huber-adam": {"loss": "huber"},
    "mae-nadam": {"loss": "mae", "optimizer": _opt("nadam", learning_rate=0.01, clipvalue=0.02, weight_decay=0.05)},
    "mse-rmsprop-centered": {"optimizer": _opt("rmsprop", learning_rate=0.01, centered=True)},
}


# How the memory-plan tests launch a fit, as (split, batch): gb_ffae_fit at batch 32 (a chunk a step) and at batch 80 (two 32-row chunks
# and a partial one, their gradients summed in the L2 scratch image), and gb_ffae_fit_split at batch 80 over a row map with a held-out
# tail (ff_split_run), evaluated in batches of 80 too.
ENTRIES = {"fit": (False, 32), "fit-b80": (False, 80), "split-b80": (True, 80)}


def crossed(values, options):
    """pytest params (value, option) of every value with every option of the dict ``options``.  The first option, the default, keeps
    the value's own id; the others append their name."""
    import pytest

    first = next(iter(options))
    return [pytest.param(v, o, id=str(v) if k == first else f"{v}-{k}") for k, o in options.items() for v in values]


def ff_split_run(engine, torch, spec, w0s, Xs, Ys, maps, n_val, E, B, perm, **fit):
    """FFEngine.fit_split of job j over the positions of maps[j]: position p reads row maps[j][p] of Xs[j] / Ys[j], and the last n_val
    positions are held out (val_batch = B).  perm [jobs, E, n_train] orders the training positions.  Returns (engine, trained weights,
    loss, accuracy, state slot 0, state slot 1, val_loss, val_accuracy), on the host."""
    eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
    J = len(w0s)
    lens = np.array([len(x) for x in Xs])
    x_row = np.concatenate([[0], np.cumsum(lens)[:-1]])
    n_train = lens - n_val

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(eng.device)

    params = eng.pack_params(w0s)
    jobs = engine.jobs_to_device(engine.make_jobs(np.arange(J), n_train, x_row), eng.device)
    split = engine.make_split(np.full(J, n_val), x_row)
    hist, acc, vl, va, (m, v) = eng.fit_split(params, jobs, J, int(n_train.max()), dev(np.concatenate(Xs)), dev(np.concatenate(Ys)), split=split,
                                              row_map=dev(np.concatenate(maps).astype(np.int32)), epochs=E, batch_size=B, perm=dev(perm), **fit)
    torch.cuda.synchronize()
    return (eng, eng.unpack_params(params), *(t.cpu().numpy() for t in (hist, acc, m, v, vl, va)))


def random_net(km, dims_or_T, seed, acts=None):
    """An hourglass of T tags (int) or a Dense stack of the given widths (tanh hidden layers and a linear output unless `acts`
    says otherwise): Glorot kernels and nonzero biases, so that every bias gradient path is exercised."""
    rng = np.random.default_rng(seed)
    spec = km.ff_hourglass_spec(dims_or_T) if isinstance(dims_or_T, int) else km.FFSpec(list(dims_or_T), acts or ["tanh"] * (len(dims_or_T) - 2) + ["linear"])
    w = km.init_ff_weights(spec, rng)
    w = [(W, rng.uniform(-0.2, 0.2, b.shape).astype(np.float32)) for W, b in w]
    return spec, w
