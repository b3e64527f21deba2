"""LSTM training above 32 windows per batch: the tensor-core fit family's C ABI checks, its workspace size and the batched
builder's opt-in (``FleetModelBuilder(lstm_wide_batches=True)``).  Host logic, no GPU."""
import ctypes as C

import numpy as np
import pandas as pd
import pytest

from gordo_components_b200 import _cabi, builder
from gordo_components_b200.engine import LSTMEngine


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def _frame(rows=200, tags=4):
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(np.random.default_rng(0).random((rows, tags)), index=idx, columns=[f"tag-{i}" for i in range(tags)])


def _machine(name="m", batch_size=64, cls_name="KerasLSTMAutoEncoder", **kwargs):
    est = {f"gordo.machine.model.models.{cls_name}": {"kind": "lstm_hourglass", "lookback_window": 6, "epochs": 2, "batch_size": batch_size,
                                                      **kwargs}}
    model = {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": est}}
    return {"name": name, "model": model, "dataset": {"X": _frame()}}


def test_cap_constants():
    assert LSTMEngine.FP32_MAX_BATCH == 32
    assert LSTMEngine.TC_MAX_BATCH == 256


@pytest.mark.parametrize("batch", [33, 64, 100, 128, 256])
@pytest.mark.parametrize("cls_name", ["KerasLSTMAutoEncoder", "KerasLSTMForecast"])
def test_wide_batches_are_accepted_with_the_flag(batch, cls_name):
    m = _machine(batch_size=batch, cls_name=cls_name)
    assert builder._canonical_lstm(0, m) is None  # the default keeps refusing batches above 32
    c = builder._canonical_lstm(0, m, wide_batches=True)
    assert isinstance(c, builder._CanonicalLSTM)
    assert c.fit == {"epochs": 2, "batch_size": batch, "shuffle": False}


@pytest.mark.parametrize("batch", [1, 16, 32])
def test_narrow_batches_are_accepted_either_way(batch):
    a = builder._canonical_lstm(0, _machine(batch_size=batch))
    b = builder._canonical_lstm(0, _machine(batch_size=batch), wide_batches=True)
    assert a.bucket() == b.bucket() and a.fit == b.fit


@pytest.mark.parametrize("batch", [257, 512, 0])
def test_batches_outside_the_cap_are_refused_with_the_flag(batch):
    assert builder._canonical_lstm(0, _machine(batch_size=batch), wide_batches=True) is None


def test_batch_size_is_part_of_the_bucket_key():
    keys = {builder._canonical_lstm(i, _machine(name=f"m{i}", batch_size=b), wide_batches=True).bucket() for i, b in enumerate([32, 64, 128, 256])}
    assert len(keys) == 4
    same = [builder._canonical_lstm(i, _machine(name=f"n{i}", batch_size=128), wide_batches=True).bucket() for i in range(2)]
    assert same[0] == same[1]


def test_flag_survives_shard():
    machines = [_machine(name=f"lstm-{i}", batch_size=64 * (1 + i % 4)) for i in range(7)]
    fleet = builder.FleetModelBuilder(machines, lstm_wide_batches=True)
    assert fleet.lstm_wide_batches
    seen = []
    for rank in range(3):
        part = fleet.shard(rank, 3)
        assert part.lstm_wide_batches and not part.early_stopping and not part.kfcv
        seen += [m["name"] for m in part.machines]
    assert sorted(seen) == sorted(m["name"] for m in machines)
    assert not builder.FleetModelBuilder(machines).shard(0, 2).lstm_wide_batches


def _net():
    return _cabi.make_lstmnet(4, [8, 3, 8], ["tanh"] * 3, 4, "linear", 6)


def test_tc_workspace_grows_with_the_padded_batch(lib):
    net = _net()
    ws = lambda n, b: lib.gb_lstm_fit_tc_workspace_bytes(C.byref(net), n, b)  # noqa: E731
    assert ws(1, 1) == ws(1, 64) > 0
    assert ws(1, 65) == ws(1, 128) > ws(1, 64)
    assert ws(1, 256) > ws(1, 128)
    assert ws(3, 100) > 2 * ws(1, 100)
    assert ws(1, 0) == 0 and ws(1, 257) == 0 and ws(-1, 64) == 0
    bad = _net()
    bad.units[1] = 4096
    assert ws(1, 64) > 0 and lib.gb_lstm_fit_tc_workspace_bytes(C.byref(bad), 1, 64) == 0


def _call(lib, net, batch, loss=0, null=False):
    hp = _cabi.GbLstmFitHParams()
    hp.epochs, hp.batch_size, hp.lookahead, hp.primer = 1, batch, 0, 1
    hp.lr, hp.beta1, hp.beta2, hp.eps = 1e-3, 0.9, 0.999, 1e-7
    p = None if null else C.c_void_p(256)  # never dereferenced: every refusal below happens before anything is enqueued
    return lib.gb_lstm_fit_tc(C.byref(net), p, p, p, p, p, 1, 10, p, p, C.byref(hp), p, p, p, loss, None)


def test_tc_entry_refuses_before_any_work(lib):
    net = _net()
    assert _call(lib, net, 257) == -2 and b"at most 256" in lib.gb_last_error()
    with pytest.raises(ValueError):
        _cabi.check(_call(lib, net, 1000))
    assert _call(lib, net, 0) == -1
    assert _call(lib, net, 64, loss=6) == -1 and b"loss" in lib.gb_last_error()
    assert _call(lib, net, 64, null=True) == -1 and b"NULL" in lib.gb_last_error()
    bad = _net()
    bad.units[0] = 0
    assert _call(lib, bad, 64) == -2


def test_fp32_entry_still_refuses_wide_batches(lib):
    hp = _cabi.GbLstmFitHParams()
    hp.epochs, hp.batch_size, hp.primer = 1, 64, 1
    p = C.c_void_p(256)
    assert lib.gb_lstm_fit_loss(C.byref(_net()), p, p, p, p, p, 1, 10, p, p, C.byref(hp), p, p, p, 0, None) == -2
