"""The depth limit of the tensor-core inference kernel's dispatch, at the boundary: the check needs no GPU."""
import ctypes as C

import pytest

from gordo_components_b200 import _cabi


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def test_six_layer_64_wide_stack_takes_the_tensor_core_kernel(lib):
    """Six 64-wide layers still fit beside the x / y tiles (they stage their outputs through the y tile alone)."""
    net = _cabi.make_ffnet([64] * 7, ["tanh"] * 5 + ["linear"])
    assert lib.gb_ffae_tc_supported(C.byref(net)) == 0


def test_seven_layer_64_wide_stack_is_refused(lib):
    net = _cabi.make_ffnet([64] * 8, ["tanh"] * 6 + ["linear"])
    assert lib.gb_ffae_tc_supported(C.byref(net)) != 0
    assert b"shared memory" in lib.gb_last_error()
