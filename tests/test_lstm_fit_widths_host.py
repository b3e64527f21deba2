"""
The C ABI admits every LSTM stack tests/test_gpu_lstm_fit_widths.py trains, so that grid cannot turn into a set of refusals, and
refuses the first stacks past the limits (513 units, 513 features in or out, 17 layers) with GB_E_SHAPE before it launches
anything.  Host logic, no GPU.
"""
import ctypes as C

import pytest
from test_gpu_lstm_fit_widths import FAMILIES, all_nets

from gordo_components_b200 import _cabi

GB_E_SHAPE = -2


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def _net(F, F_out, units, acts, head, L):
    return _cabi.make_lstmnet(F, units, acts, F_out, head, L)


@pytest.mark.parametrize("case", list(all_nets()))
def test_every_trained_stack_is_admitted(lib, case):
    F, F_out, units, acts, head, L = all_nets()[case]
    net = _net(F, F_out, units, acts, head, L)
    n_params = 0
    i = F
    for u in units:
        n_params += 4 * u * (i + u + 1)
        i = u
    assert lib.gb_lstm_param_count(C.byref(net)) == n_params + i * F_out + F_out
    assert lib.gb_lstm_fit_workspace_bytes(C.byref(net), 3) > 0
    for _, B in FAMILIES.values():
        assert lib.gb_lstm_fit_tc_workspace_bytes(C.byref(net), 3, B) > 0


def test_the_largest_stacks_are_admitted(lib):
    """512 units, 512 features in and out, 16 layers: the limits themselves."""
    net = _net(512, 512, [512] * 16, ["tanh"] * 16, "linear", 2)
    assert lib.gb_lstm_param_count(C.byref(net)) > 0
    assert lib.gb_lstm_fit_workspace_bytes(C.byref(net), 1) > 0
    assert lib.gb_lstm_fit_tc_workspace_bytes(C.byref(net), 1, 256) > 0


def _past_the_limits():
    """The first inadmissible neighbour of each limit, as a gb_lstmnet (17 layers cannot go through make_lstmnet)."""
    out = {
        "units_513": _net(16, 16, [513], ["tanh"], "linear", 3),
        "units_513_in_layer_16": _net(16, 16, [8] * 15 + [513], ["tanh"] * 16, "linear", 3),
        "features_513": _net(513, 16, [16], ["tanh"], "linear", 3),
        "features_out_513": _net(16, 513, [16], ["tanh"], "linear", 3),
    }
    deep = _net(16, 16, [8] * 16, ["tanh"] * 16, "linear", 3)
    deep.n_layers = 17
    out["layers_17"] = deep
    return out


@pytest.mark.parametrize("case", list(_past_the_limits()))
def test_stacks_past_the_limits_get_no_workspace(lib, case):
    net = _past_the_limits()[case]
    assert lib.gb_lstm_param_count(C.byref(net)) == 0
    assert lib.gb_lstm_fit_workspace_bytes(C.byref(net), 1) == 0
    for B in (1, 64, 256):
        assert lib.gb_lstm_fit_tc_workspace_bytes(C.byref(net), 1, B) == 0


@pytest.mark.parametrize("entry", ["gb_lstm_fit_stop", "gb_lstm_fit_tc_stop"])
@pytest.mark.parametrize("case", list(_past_the_limits()))
def test_fit_entries_refuse_stacks_past_the_limits(lib, case, entry):
    net = _past_the_limits()[case]
    hp = _cabi.GbLstmFitHParams()
    hp.epochs, hp.batch_size, hp.lookahead, hp.primer = 1, 32, 0, 1
    hp.lr, hp.beta1, hp.beta2, hp.eps = 1e-3, 0.9, 0.999, 1e-7
    p = C.c_void_p(256)  # never dereferenced: the refusal comes before anything is enqueued
    rc = getattr(lib, entry)(C.byref(net), p, p, p, p, p, 1, 10, p, p, C.byref(hp), p, p, p, 0, None, None, None, None, None, None)
    assert rc == GB_E_SHAPE, lib.gb_last_error()
    assert b"outside" in lib.gb_last_error()
