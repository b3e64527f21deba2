"""Which feed-forward stacks the tensor-core inference kernel takes: the check needs no GPU."""
import ctypes as C

import pytest

from gordo_components_b200 import _cabi


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def test_hourglass_takes_the_tensor_core_kernel(lib):
    net = _cabi.make_ffnet([64, 53, 43, 32, 32, 43, 53, 64], ["tanh"] * 6 + ["linear"])
    assert lib.gb_ffae_tc_supported(C.byref(net)) == 0


def test_stack_beyond_shared_memory_is_refused(lib):
    """Eight 64-wide layers: their weight images and the x / y tiles together exceed an SM's shared memory, so the stack goes
    to the generic kernel under automatic dispatch."""
    net = _cabi.make_ffnet([64] * 9, ["tanh"] * 7 + ["linear"])
    assert lib.gb_ffae_tc_supported(C.byref(net)) != 0
    assert b"shared memory" in lib.gb_last_error()
