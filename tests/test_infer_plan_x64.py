"""The kernel and tensor-core warpgroup count a Dense stack scores on when a Pipeline's input scalers are applied inside the fused
launch (gb_ffae_infer_plan_x64, float64 x): host code, no GPU.  X64_SHAPES names one architecture per float64-x kernel
instantiation; tests/test_gpu_x64_coverage.py runs each of them against the float64 oracle."""
import ctypes as C
import itertools

import pytest

from gordo_components_b200 import _cabi
from oracle import keras_math as km
from test_infer_plan import COLUMN_BLOCKED, PLAN_SHAPES, ffnet, infer_plan


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def plan_x64(lib, dims, acts=None, variant=0, net=None):
    """(return code, kernel, warpgroups) of gb_ffae_infer_plan_x64."""
    net = ffnet(dims, acts) if net is None else net
    kernel, nwg = C.c_int32(-1), C.c_int32(-1)
    rc = lib.gb_ffae_infer_plan_x64(C.byref(net), int(variant), C.byref(kernel), C.byref(nwg))
    return rc, kernel.value, nwg.value


def hourglass(T):
    return km.ff_hourglass_spec(T).dims


# float64-x instantiation -> the architecture the GPU coverage tests run it on (kernel 1: generic, 3: row per thread, 2: tensor cores)
X64_SHAPES = {
    "generic-rt4": PLAN_SHAPES[(128, 1)],
    "generic-rt2": PLAN_SHAPES[(64, 1)],
    "generic-rt1": PLAN_SHAPES[(32, 0)],
    "generic-rt1-blocked": COLUMN_BLOCKED[0],
    "small-w4": hourglass(4),
    "small-w8": hourglass(8),
    "small-w16": hourglass(16),
    "tc-nwg3": hourglass(32),
    "tc-nwg2": hourglass(64),
}
# the generic kernel's instantiation of each (rows per tile, column-blocked) plan
GENERIC_ROWS = {"generic-rt4": 128, "generic-rt2": 64, "generic-rt1": 32, "generic-rt1-blocked": 32}


def instantiation(lib, dims, variant):
    """The name of the float64-x kernel instantiation `variant` runs `dims` on (as in X64_SHAPES)."""
    rc, kernel, nwg = plan_x64(lib, dims, variant=variant)
    assert rc == 0, (dims, variant, rc)
    if kernel == 2:
        return f"tc-nwg{nwg}"
    if kernel == 3:
        w = max(dims)
        return "small-w4" if w <= 4 else "small-w8" if w <= 8 else "small-w16"
    rows = infer_plan(lib, dims)[1]
    if rows == 32 and list(dims) in [list(d) for d in COLUMN_BLOCKED]:
        return "generic-rt1-blocked"
    return {128: "generic-rt4", 64: "generic-rt2", 32: "generic-rt1"}[rows]


@pytest.mark.parametrize("name", list(X64_SHAPES))
def test_each_x64_instantiation_has_a_gpu_tested_shape(lib, name):
    dims = X64_SHAPES[name]
    variant = 1 if name.startswith("generic") else 3 if name.startswith("small") else 2
    assert instantiation(lib, dims, variant) == name
    if name.startswith("generic"):
        assert infer_plan(lib, dims)[:2] == (0, GENERIC_ROWS[name])


@pytest.mark.parametrize("T", list(range(24, 57, 4)))
def test_hourglass_up_to_56_tags_runs_three_warpgroups(lib, T):
    assert plan_x64(lib, hourglass(T)) == (0, 2, 3)


@pytest.mark.parametrize("T", [60, 64])
def test_hourglass_of_60_and_64_tags_runs_two_warpgroups(lib, T):
    """The layer-0 weight images of a 64-column stack leave room for two warpgroups' float64 x tiles, not three."""
    assert plan_x64(lib, hourglass(T)) == (0, 2, 2)


@pytest.mark.parametrize("dims,nwg", [([64] * 5, 2), ([64] * 7, 2), ([64, 64, 64], 3), ([48, 64, 48], 3),
                                      ([64, 16, 32, 48, 64, 64, 64], 3)])
def test_tensor_core_warpgroups_of_other_stacks(lib, dims, nwg):
    assert plan_x64(lib, dims) == (0, 2, nwg)


@pytest.mark.parametrize("factory", ["ff_symmetric_spec", "ff_model_spec"])
@pytest.mark.parametrize("T", [24, 32, 48, 64])
def test_wide_factory_defaults_score_on_the_generic_kernel(lib, factory, T):
    """feedforward_symmetric / feedforward_model defaults (256-wide layers): 32-row tiles with staged weights."""
    spec = getattr(km, factory)(T)
    assert plan_x64(lib, spec.dims, spec.acts) == (0, 1, 0)
    assert infer_plan(lib, spec.dims, spec.acts) == (0, 32, 0)


@pytest.mark.parametrize("T", list(range(1, 17)))
def test_narrow_hourglass_scores_row_per_thread(lib, T):
    assert plan_x64(lib, hourglass(T)) == (0, 3, 0)


def test_variants_outside_their_range_are_refused(lib):
    assert plan_x64(lib, hourglass(20), variant=2)[0] == -2  # GB_E_SHAPE: under 24 tags
    assert plan_x64(lib, hourglass(32), variant=3)[0] == -2  # wider than 16
    assert plan_x64(lib, hourglass(32), variant=4)[0] == -1  # GB_E_ARG
    assert plan_x64(lib, hourglass(32), variant=1)[:2] == (0, 1)


def test_no_admitted_tensor_core_stack_is_refused_for_shared_memory(lib):
    """gb_ffae_tc_warpgroups_x64 refuses a stack whose weights leave no room for two warpgroups' float64 x tiles (GB_E_SMEM); then
    the detector falls back to two launches.  Shared memory depends on the widths rounded up to 16 only, so every T in 24..64 with
    2..8 layers of hidden widths 16, 32, 48, 64 covers every stack the tensor-core variant admits (it refuses, in float32 mode
    already, the deepest stacks of 64-wide layers): each admitted one plans 2 or 3 warpgroups."""
    net = ffnet([24, 24])
    counts, refused, admitted = {2: 0, 3: 0}, [], 0
    for L in range(2, 9):
        net.n_layers = L
        for l in range(L):
            net.act[l] = _cabi.ACT_CODES["tanh" if l + 1 < L else "linear"]
        for hidden in itertools.product((16, 32, 48, 64), repeat=L - 1):
            for i, h in enumerate(hidden):
                net.dims[i + 1] = h
            for T in range(24, 65, 4):
                net.dims[0] = net.dims[L] = T
                if lib.gb_ffae_tc_supported(C.byref(net)) != 0:
                    continue
                admitted += 1
                rc, kernel, nwg = plan_x64(lib, None, net=net)
                if rc != 0 or kernel != 2 or nwg not in counts:
                    refused.append((T, hidden, rc, kernel, nwg))
                    continue
                counts[nwg] += 1
    assert not refused, f"{len(refused)} admitted stacks without a float64-x tensor-core plan, e.g. {refused[:5]}"
    # nearly all of the 11 * (4 + 16 + ... + 4^7) stacks are admitted, and both warpgroup counts occur
    assert admitted > 0.99 * 11 * sum(4 ** (L - 1) for L in range(2, 9)), admitted
    assert counts[2] > 0 and counts[3] > 0 and sum(counts.values()) == admitted, counts
