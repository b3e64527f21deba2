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


def random_net(km, dims_or_T, seed, acts=None):
    """An hourglass of T tags (int) or a Dense stack of the given widths (tanh hidden layers and a linear output unless `acts`
    says otherwise): Glorot kernels and nonzero biases, so that every bias gradient path is exercised."""
    rng = np.random.default_rng(seed)
    spec = km.ff_hourglass_spec(dims_or_T) if isinstance(dims_or_T, int) else km.FFSpec(list(dims_or_T), acts or ["tanh"] * (len(dims_or_T) - 2) + ["linear"])
    w = km.init_ff_weights(spec, rng)
    w = [(W, rng.uniform(-0.2, 0.2, b.shape).astype(np.float32)) for W, b in w]
    return spec, w
