"""Which Dense inference kernel takes an architecture, and the launch plan of the generic (variant 1) kernel: the dispatch checks and
the planner are host code and need no GPU.  Every plan pinned here runs on the GPU in tests/test_gpu_infer_coverage.py."""
import ctypes as C

import pytest

from gordo_components_b200 import _cabi
from oracle import keras_math as km


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def ffnet(dims, acts=None):
    return _cabi.make_ffnet(dims, acts or ["tanh"] * (len(dims) - 2) + ["linear"])


def infer_plan(lib, dims, acts=None):
    net = ffnet(dims, acts)
    rows, resident = C.c_int32(-1), C.c_int32(-1)
    rc = lib.gb_ffae_infer_plan(C.byref(net), C.byref(rows), C.byref(resident))
    return rc, rows.value, resident.value


def fit_accepts(lib, spec):
    net = _cabi.make_ffnet(spec.dims, spec.acts, spec.l1)
    return lib.gb_ffae_fit_plan(C.byref(net), None, None) == 0


# (rows per tile, weights resident) -> the architecture the GPU coverage tests run in that plan on variant 1
PLAN_SHAPES = {
    (128, 1): km.ff_hourglass_spec(64).dims,
    (128, 0): km.ff_hourglass_spec(128).dims,
    (64, 1): [64, 200, 64],
    (64, 0): km.ff_hourglass_spec(160).dims,
    (32, 1): [16, 256, 128, 16],
    (32, 0): km.ff_symmetric_spec(64).dims,
}
# 32-row tiles with staged layers too large to stage whole next to the activations: staged in blocks of output columns
COLUMN_BLOCKED = [km.ff_symmetric_spec(172).dims, [64, 256, 256, 64]]


@pytest.mark.parametrize("want", list(PLAN_SHAPES))
def test_each_plan_has_a_gpu_tested_shape(lib, want):
    assert infer_plan(lib, PLAN_SHAPES[want]) == (0, *want)


@pytest.mark.parametrize("dims", COLUMN_BLOCKED)
def test_layers_too_large_to_stage_whole_are_planned(lib, dims):
    assert infer_plan(lib, dims) == (0, 32, 0)


def test_outputs_may_be_null_and_bad_nets_are_refused(lib):
    assert lib.gb_ffae_infer_plan(C.byref(ffnet([8, 4, 8])), None, None) == 0
    bad = ffnet([8, 4, 8])
    bad.dims[1] = 4096
    assert lib.gb_ffae_infer_plan(C.byref(bad), None, None) == -2  # GB_E_SHAPE


@pytest.mark.parametrize("factory", ["ff_symmetric_spec", "ff_model_spec", "ff_hourglass_spec"])
def test_every_trainable_default_stack_can_predict(lib, factory):
    """A model that trains must predict: the generic kernel (every dispatch falls back to it) accepts every factory default the fit
    accepts, 1..256 tags."""
    make = getattr(km, factory)
    trainable = [T for T in range(1, 257) if fit_accepts(lib, make(T))]
    assert len(trainable) >= 172
    refused = [T for T in trainable if infer_plan(lib, make(T).dims, make(T).acts)[0] != 0]
    assert not refused, f"{factory}: fit accepts but inference refuses {refused}"


@pytest.mark.parametrize("dims", [[64, 256, 256, 64], [256, 256], [256] * 17, [3, 256, 256, 256, 3], [256, 256, 5]])
def test_stacks_with_256_by_256_layers_can_predict(lib, dims):
    spec = km.FFSpec(dims, ["relu"] * (len(dims) - 2) + ["linear"])
    assert infer_plan(lib, dims, spec.acts)[0] == 0
    if fit_accepts(lib, spec):
        assert infer_plan(lib, dims, spec.acts)[1] == 32


@pytest.mark.parametrize("dims,acts,ok", [
    (km.ff_hourglass_spec(20).dims, None, False),   # fewer than 24 tags
    (km.ff_hourglass_spec(24).dims, None, True),
    (km.ff_hourglass_spec(64).dims, None, True),
    (km.ff_hourglass_spec(68).dims, None, False),   # wider than 64 tags
    (km.ff_hourglass_spec(30).dims, None, False),   # not a multiple of 4
    (km.ff_hourglass_spec(63).dims, None, False),
    ([64, 65, 64], None, False),                     # a 65-wide hidden layer
    ([64, 64, 64], None, True),
    ([48, 32, 48], ["relu", "linear"], False),       # non-tanh hidden layer
    ([48, 32, 48], ["tanh", "tanh"], False),         # non-linear output layer
    ([48, 48], ["linear"], False),                   # n_layers = 1
    ([48, 24, 40], None, False),                     # n_out != n_in
])
def test_tensor_core_dispatch_boundaries(lib, dims, acts, ok):
    assert (lib.gb_ffae_tc_supported(C.byref(ffnet(dims, acts))) == 0) == ok


@pytest.mark.parametrize("dims,ok", [([16, 16, 16], True), ([16, 8, 16], True), ([17, 8, 17], False), ([8, 17, 8], False), ([1, 1], True),
                                     ([4, 16, 16, 16], True), ([16, 4, 17], False)])
def test_row_per_thread_dispatch_boundary(lib, dims, ok):
    assert (lib.gb_ffae_small_supported(C.byref(ffnet(dims))) == 0) == ok
