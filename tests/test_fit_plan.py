"""The memory plan gb_ffae_fit picks for each architecture the GPU fit tests train, and the widest stack it accepts: the planner
is host code and needs no GPU."""
import ctypes as C

import pytest

from gordo_components_b200 import _cabi
from oracle import keras_math as km


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def plan(lib, spec):
    net = _cabi.make_ffnet(spec.dims, spec.acts, spec.l1)
    w, d = C.c_int32(-1), C.c_int32(-1)
    rc = lib.gb_ffae_fit_plan(C.byref(net), C.byref(w), C.byref(d))
    return rc, w.value, d.value


# (weights in L2, dz buffers in L2) of the five plans, each with the shape tests/test_gpu_fit_coverage.py trains in it
PLAN_SHAPES = {
    (0, 0): km.ff_hourglass_spec(64),      # everything in shared memory
    (1, 0): km.ff_symmetric_spec(10),      # the weight image in L2
    (1, 1): km.ff_symmetric_spec(64),      # ... and one dz buffer
    (1, 2): km.ff_symmetric_spec(96),      # ... two
    (1, 3): km.ff_symmetric_spec(128),     # ... all three
}


@pytest.mark.parametrize("want", list(PLAN_SHAPES))
def test_each_plan_has_a_gpu_tested_shape(lib, want):
    assert plan(lib, PLAN_SHAPES[want]) == (0, *want)


def test_hourglass_128_keeps_its_weights_in_l2(lib):
    assert plan(lib, km.ff_hourglass_spec(128)) == (0, 1, 0)


def test_widest_symmetric_default_stack(lib):
    """The 256-128-64 default of feedforward_symmetric / feedforward_model trains up to 172 tags; 173 needs more shared memory
    than an SM has for one 32-row chunk's activations even with the weights and every dz buffer in L2."""
    assert plan(lib, km.ff_symmetric_spec(172)) == (0, 1, 3)
    assert plan(lib, km.ff_model_spec(172)) == (0, 1, 3)
    rc, _, _ = plan(lib, km.ff_symmetric_spec(173))
    assert rc == -4  # GB_E_SMEM
    assert b"shared memory" in lib.gb_last_error()
    with pytest.raises(ValueError):
        _cabi.check(rc)


def test_widest_trainable_hourglass_default_stack(lib):
    """The hourglass default trains up to 196 tags: 197 needs 231 936 bytes of shared memory for one chunk's activations, within
    227 KB but not beside the fit kernels' own static arrays, so cudaFuncSetAttribute refuses every launch of it.  The planner
    refuses it instead, with GB_E_SMEM before any device work."""
    assert plan(lib, km.ff_hourglass_spec(80)) == (0, 0, 0)
    assert plan(lib, km.ff_hourglass_spec(196)) == (0, 1, 3)
    assert plan(lib, km.ff_hourglass_spec(197))[0] == -4
    assert plan(lib, km.ff_hourglass_spec(198))[0] == -4


def test_outputs_may_be_null(lib):
    net = _cabi.make_ffnet([8, 4, 8], ["tanh", "linear"])
    assert lib.gb_ffae_fit_plan(C.byref(net), None, None) == 0
