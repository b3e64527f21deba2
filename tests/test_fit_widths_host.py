"""
The memory plan gb_ffae_fit_plan picks for every Dense stack tests/test_gpu_fit_widths.py trains, so that the GPU file's grid cannot
drift into other plans or into refusals, and the refusal of the first stacks past the limits: symmetric(173), hourglass(197) and four
256-wide layers need more shared memory than a block has beside the kernels' static arrays (GB_E_SMEM, before any launch); 17
layers or a width of 257 are outside what the kernels take at all (GB_E_SHAPE).  Host logic, no GPU.
"""
import ctypes as C
import os
import re
import subprocess

import pytest
from test_gpu_fit_widths import all_stacks

from gordo_components_b200 import _cabi
from oracle import keras_math as km

GB_E_SHAPE, GB_E_SMEM = -2, -4


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def net_of(spec):
    return _cabi.make_ffnet(spec.dims, spec.acts, spec.l1)


def plan(lib, net):
    w, d = C.c_int32(-1), C.c_int32(-1)
    rc = lib.gb_ffae_fit_plan(C.byref(net), C.byref(w), C.byref(d))
    return rc, w.value, d.value


@pytest.mark.parametrize("case", list(all_stacks()))
def test_every_trained_stack_has_its_plan(lib, case):
    spec, want = all_stacks()[case]
    assert plan(lib, net_of(spec)) == (0, *want)


def test_one_layer_stacks_and_the_sixteen_layer_limit_are_admitted(lib):
    """[64, 64] and [256, 256] are one-layer stacks (the gather's both-halves path); 16 layers is GB_MAX_LAYERS."""
    assert plan(lib, _cabi.make_ffnet([64, 64], ["linear"])) == (0, 0, 0)
    assert plan(lib, _cabi.make_ffnet([256, 256], ["linear"])) == (0, 1, 2)
    assert plan(lib, _cabi.make_ffnet([32] * 17, ["tanh"] * 16)) == (0, 0, 0)
    assert plan(lib, _cabi.make_ffnet([64] * 17, ["tanh"] * 16)) == (0, 1, 0)


def fit(lib, net):
    """gb_ffae_fit on placeholder device addresses: a refusal returns before anything is enqueued or dereferenced."""
    hp = _cabi.GbFitHParams()
    hp.epochs, hp.batch_size, hp.shuffle = 1, 32, 1
    hp.lr, hp.beta1, hp.beta2, hp.eps = 1e-3, 0.9, 0.999, 1e-7
    p = C.c_void_p(256)
    return lib.gb_ffae_fit(C.byref(net), p, p, p, p, 1, 40, p, p, None, C.byref(hp), p, p, None)


PAST_SHARED_MEMORY = {
    "symmetric_173": km.ff_symmetric_spec(173),
    "hourglass_197": km.ff_hourglass_spec(197),
    "four_layers_256": km.FFSpec([256] * 5, ["tanh"] * 3 + ["linear"]),
}


@pytest.mark.parametrize("case", list(PAST_SHARED_MEMORY))
def test_first_stacks_past_shared_memory_are_refused(lib, case):
    net = net_of(PAST_SHARED_MEMORY[case])
    rc, w, d = plan(lib, net)
    assert (rc, w, d) == (GB_E_SMEM, -1, -1)
    assert b"shared memory" in lib.gb_last_error()
    assert fit(lib, net) == GB_E_SMEM
    assert b"shared memory" in lib.gb_last_error()
    with pytest.raises(ValueError, match="shared memory"):
        _cabi.check(GB_E_SMEM)


def _past_the_shape_limits():
    wide = _cabi.make_ffnet([64, 64, 64], ["tanh", "linear"])
    wide.dims[1] = 257
    wide_in = _cabi.make_ffnet([64, 64], ["linear"])
    wide_in.dims[0] = 257
    deep = _cabi.make_ffnet([8] * 17, ["tanh"] * 16)
    deep.n_layers = 17
    return {"width_257": wide, "n_in_257": wide_in, "layers_17": deep}


@pytest.mark.parametrize("case", list(_past_the_shape_limits()))
def test_stacks_past_the_shape_limits_are_refused(lib, case):
    net = _past_the_shape_limits()[case]
    assert plan(lib, net) == (GB_E_SHAPE, -1, -1)
    assert b"outside" in lib.gb_last_error()
    assert fit(lib, net) == GB_E_SHAPE
    assert lib.gb_ffae_fit_state_stride(C.byref(net)) == 0
    with pytest.raises(ValueError):
        _cabi.make_ffnet([8] * 18, ["tanh"] * 17)


def test_fit_kernels_static_shared_memory_fits_the_reserve(lib):
    """The plans leave 2 KB of the 227 KB a block may opt into for the fit kernels' static shared memory (FIT_STATIC_SMEM in
    csrc/ffae_fit.cu); a launch whose static and dynamic shared memory exceed 227 KB is refused by cudaFuncSetAttribute.  Every
    compiled fit kernel must stay within the reserve."""
    from gordo_components_b200.csrc import build

    obj = os.path.join(build.OBJ, "ffae_fit.o")
    tool = os.path.join(os.path.dirname(build._nvcc()), "cuobjdump")
    out = subprocess.run([tool, "-res-usage", obj], capture_output=True, text=True, check=True).stdout
    sizes = [int(v) for v in re.findall(r"SHARED:(\d+)", out)]
    assert len(sizes) == 36, "one entry per fit kernel instantiation"
    assert max(sizes) <= 2048, sorted(set(sizes))
