"""The LSTM fit families share one host driver (csrc/lstm_fit_common.cuh): their workspace queries and the argument refusals of
every legacy C entry point of both families.  No GPU needed: every refusal happens before anything is enqueued."""
import ctypes as C

import pytest

from gordo_components_b200 import _cabi, engine


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


# ------------------------------------------------------------------------------------------------ workspace queries
BATCHES = [1, 31, 32, 33, 64, 200, 256]
# (n_features, units, lookback, n_features_out), gb_lstm_fit_workspace_bytes at 1 and 3 jobs,
# gb_lstm_fit_tc_workspace_bytes at 3 jobs for each of BATCHES
WORKSPACE = [
    ((3, [5], 1, 3), [6584, 19720], [39400, 39400, 39400, 39400, 39400, 150280, 150280]),
    ((7, [9, 5], 13, 7), [162824, 488440], [970840, 970840, 970840, 970840, 970840, 3848824, 3848824]),
    ((20, [33, 17, 33], 144, 20), [10198264, 30594760], [60988840, 60988840, 60988840, 60988840, 60988840, 243306952, 243306952]),
    ((1, [1, 1, 1], 2, 1), [6200, 18568], [37480, 37480, 37480, 37480, 37480, 148360, 148360]),
    ((11, [127, 63], 37, 5), [6533496, 19600456], [37776040, 37776040, 37776040, 37776040, 37776040, 146817736, 146817736]),
    ((64, [511], 144, 64), [61549208, 184647592], [354823048, 354823048, 354823048, 354823048, 354823048, 1375728040, 1375728040]),
    ((512, [3, 512], 1, 512), [5895768, 17687272], [19860424, 19860424, 19860424, 19860424, 19860424, 31719400, 31719400]),
]


@pytest.mark.parametrize("shape,fp32,tc", WORKSPACE, ids=[str(w[0]) for w in WORKSPACE])
def test_workspace_bytes_are_pinned(lib, shape, fp32, tc):
    F, units, L, T = shape
    net = _cabi.make_lstmnet(F, units, ["tanh"] * len(units), T, "linear", L)
    assert [lib.gb_lstm_fit_workspace_bytes(C.byref(net), n) for n in (1, 3)] == fp32
    assert [lib.gb_lstm_fit_tc_workspace_bytes(C.byref(net), 3, b) for b in BATCHES] == tc
    for batch in (0, 257):
        assert lib.gb_lstm_fit_tc_workspace_bytes(C.byref(net), 3, batch) == 0
    assert lib.gb_lstm_fit_workspace_bytes(C.byref(net), -1) == 0


# ------------------------------------------------------------------------------------------------ refusals
# entry: (largest batch of its family, takes a loss, takes an optimizer, takes a stop rule)
ENTRIES = {
    "gb_lstm_fit": (32, False, False, False),
    "gb_lstm_fit_loss": (32, True, False, False),
    "gb_lstm_fit_opt": (32, True, True, False),
    "gb_lstm_fit_stop": (32, True, True, True),
    "gb_lstm_fit_tc": (256, True, False, False),
    "gb_lstm_fit_tc_opt": (256, True, True, False),
    "gb_lstm_fit_tc_stop": (256, True, True, True),
}
CAP_TEXT = {32: b"this kernel family handles batches of at most 32 windows",
            256: b"the tensor-core LSTM fit handles batches of at most 256 windows"}


def _call(lib, entry, batch=16, lookahead=0, loss=0, opt=None, stop=None, null_x=False):
    _, has_loss, has_opt, has_stop = ENTRIES[entry]
    net = _cabi.make_lstmnet(4, [8, 3, 8], ["tanh"] * 3, 4, "linear", 6)
    hp = _cabi.GbLstmFitHParams()
    hp.epochs, hp.batch_size, hp.lookahead, hp.primer = 3, batch, lookahead, 1
    hp.lr, hp.beta1, hp.beta2, hp.eps = 1e-3, 0.9, 0.999, 1e-7
    p = C.c_void_p(256)  # never dereferenced
    args = [C.byref(net), p, p, p, p, p, 2, 10, None if null_x else p, p, C.byref(hp), p, p, p]
    if has_loss:
        args.append(loss)
    if has_opt:
        args.append(None if opt is None else C.byref(opt))
    if has_stop:
        rules = stop if stop is not None else engine.make_stop([{"monitor": "loss", "patience": 2}] * 2)
        args += [rules.ctypes.data_as(C.c_void_p), p, p, p]
    return getattr(lib, entry)(*args, None)


def _bad_optimizer():
    opt = _cabi.GbOptimizer()
    opt.kind = 42
    return opt


def _bad_stop():
    rules = engine.make_stop([{"monitor": "loss"}] * 2)
    rules[1]["monitor"] = 4
    return rules


REFUSALS = {  # name: (applies to the entry, call keywords, status, text in gb_last_error)
    "loss": (lambda e: ENTRIES[e][1], dict(loss=6), -1, b"loss=6 unknown"),
    "optimizer": (lambda e: ENTRIES[e][2], dict(opt=_bad_optimizer()), -1, b"optimizer kind=42 unknown"),
    "null": (lambda e: True, dict(null_x=True), -1, b"NULL argument"),
    "lookahead": (lambda e: True, dict(lookahead=-1), -1, b"`lookahead` can not be negative"),
    "batch": (lambda e: True, None, -2, None),
    "stop": (lambda e: ENTRIES[e][3], dict(stop=_bad_stop()), -1, b"stop[1].monitor=4 unknown"),
}


@pytest.mark.parametrize("entry,refusal", [(e, r) for e in ENTRIES for r in REFUSALS if REFUSALS[r][0](e)])
def test_every_entry_refuses_with_one_status(lib, entry, refusal):
    _, kw, status, text = REFUSALS[refusal]
    if refusal == "batch":
        cap = ENTRIES[entry][0]
        kw, text = dict(batch=cap + 1), CAP_TEXT[cap]
    assert _call(lib, entry, **kw) == status
    assert text in lib.gb_last_error()
