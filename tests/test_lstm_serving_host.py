"""
LSTM serving without a GPU: the argument checks of the ragged tensor-core LSTM entry, its workspace query against the uniform
one, which LSTM detectors ResidentBucket(lstm=True) admits and how it groups them, and the tile cap of the LSTM coalescer's batches.
"""
import ctypes as C
import queue
import threading
import time

import numpy as np
import pandas as pd
import pytest

from gordo_components_b200 import _cabi

CONFIG3 = dict(n_features=128, units=[256, 128, 64, 64, 128, 256], acts=["tanh"] * 6, n_features_out=128, out_func="linear", lookback=144)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def _net(**kw):
    c = dict(CONFIG3, **kw)
    return _cabi.make_lstmnet(c["n_features"], c["units"], c["acts"], c["n_features_out"], c["out_func"], c["lookback"])


def _tiles(windows):
    return int(sum((w + 127) // 128 for w in windows))


def test_ragged_workspace_equals_uniform_for_uniform_jobs(lib):
    net = _net()
    for n_slots, n_jobs, windows in ((1, 1, 1), (3, 5, 128), (32, 64, 100), (2, 7, 300), (4, 3, 10000)):
        uniform = lib.gb_lstm_tc_workspace_bytes(C.byref(net), n_slots, n_jobs, windows, 1)
        ragged = lib.gb_lstm_tc_ragged_workspace_bytes(C.byref(net), n_slots, n_jobs, _tiles([windows] * n_jobs), windows)
        assert uniform > 0 and ragged == uniform


def test_ragged_workspace_follows_the_jobs_own_windows(lib):
    """One 10 000-window request with 63 of 100 windows: 142 tiles instead of 64 x 79."""
    net = _net()
    windows = [10000] + [100] * 63
    n_tiles = _tiles(windows)
    assert n_tiles == 142
    uniform = lib.gb_lstm_tc_workspace_bytes(C.byref(net), 32, 64, 10000, 1)
    ragged = lib.gb_lstm_tc_ragged_workspace_bytes(C.byref(net), 32, 64, n_tiles, 10000)
    state_per_tile = 128 * sum(CONFIG3["units"]) * 12  # h as two FP16 pairs (double-buffered) and c in fp32
    assert uniform > 64 * 79 * state_per_tile > 6.9e9
    assert 142 * state_per_tile < ragged < 0.5e9
    # the engine's helper gives the same prefix sums
    from gordo_components_b200.engine import LSTMEngine

    tb = LSTMEngine.tile_base(windows)
    assert tb.dtype == np.int32 and tb[0] == 0 and tb[-1] == n_tiles and tb[1] == 79 and np.all(np.diff(tb)[1:] == 1)
    assert list(LSTMEngine.tile_base([0, 1, 128, 129, 0])) == [0, 0, 1, 2, 4, 4]


def test_ragged_workspace_query_refuses_what_the_entry_refuses(lib):
    net = _net()
    assert lib.gb_lstm_tc_ragged_workspace_bytes(C.byref(net), 1, 2, 3, 128) == 0  # 3 tiles > 2 jobs x 1 tile
    assert lib.gb_lstm_tc_ragged_workspace_bytes(C.byref(net), 1, 2, -1, 128) == 0
    assert lib.gb_lstm_tc_ragged_workspace_bytes(C.byref(net), 1, -1, 0, 128) == 0
    assert lib.gb_lstm_tc_ragged_workspace_bytes(C.byref(_net(acts=["relu"] * 6)), 1, 2, 2, 128) == 0
    assert lib.gb_lstm_tc_ragged_workspace_bytes(C.byref(net), 1, 0, 0, 0) > 0  # nothing to run: the weight images only


def test_ragged_entry_checks_arguments_before_any_launch(lib):
    net = _net()
    fake = C.c_void_p(256)  # never dereferenced: every call below is refused on the host
    ws_misaligned = C.c_void_p(258)

    def call(params=fake, n_slots=1, jobs=fake, n_jobs=2, tile_base=fake, n_tiles=2, max_windows=128, x=fake, x_rows=200, out=fake, ws=fake, net=net):
        return lib.gb_lstm_infer_tc_ragged(C.byref(net), params, n_slots, jobs, n_jobs, tile_base, n_tiles, max_windows, x, x_rows, out, ws, None)

    for kw in ({"params": None}, {"jobs": None}, {"tile_base": None}, {"x": None}, {"out": None}, {"ws": None}):
        assert call(**kw) == -1 and b"non-NULL" in lib.gb_last_error(), kw
    assert call(n_tiles=3) == -2 and b"n_tiles" in lib.gb_last_error()  # more tiles than n_jobs x ceil(max_windows / 128)
    assert call(n_tiles=300, max_windows=128 * 100, n_jobs=2) == -2
    assert call(n_tiles=-1) == -1
    assert call(n_jobs=-1) == -1
    assert call(max_windows=-1) == -1
    assert call(n_slots=0) == -1
    assert call(x_rows=0) == -1
    assert call(ws=ws_misaligned) == -3
    assert call(net=_net(acts=["relu"] * 6)) == -2  # relu cells: the fp32 kernel only
    with pytest.raises(ValueError):
        _cabi.check(call(tile_base=None))
    # the uniform entry keeps its checks, and refuses a layout too large to count
    assert lib.gb_lstm_infer_tc(C.byref(net), fake, 1, fake, 1 << 30, 1 << 30, fake, 1, fake, fake, None) == -2


# ------------------------------------------------------------------------------------------------ eligibility and grouping
def _detector(est, thresholds=True, window=None, scaler=None, require_thresholds=True, n=4):
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector

    det = DiffBasedAnomalyDetector(base_estimator=est, scaler=scaler if scaler is not None else MinMaxScaler(), window=window,
                                   require_thresholds=require_thresholds)
    det.scaler.fit(np.random.default_rng(0).random((10, n)))
    if thresholds:
        det.feature_thresholds_ = pd.Series(np.ones(n))
        det.aggregate_threshold_ = 1.0
    return det


def _lstm(cls="KerasLSTMAutoEncoder", lookback=3, n=4, **kw):
    from gordo_components_b200.machine.model import models

    return getattr(models, cls)(kind="lstm_hourglass", lookback_window=lookback, encoding_layers=1, **kw).initialize(n, n)


def test_lstm_eligibility():
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import MinMaxScaler, QuantileTransformer, StandardScaler

    from gordo_components_b200.machine.model.models import KerasAutoEncoder
    from gordo_components_b200.server import ResidentBucket

    ok = [
        _detector(_lstm()),
        _detector(_lstm("KerasLSTMForecast")),
        _detector(Pipeline([("s", MinMaxScaler()), ("m", _lstm())])),
        _detector(Pipeline([("s", StandardScaler()), ("m", _lstm("KerasLSTMForecast"))])),
        _detector(_lstm(), thresholds=False, require_thresholds=False),
    ]
    for det in ok:
        assert ResidentBucket.eligible_lstm(det)
        assert not ResidentBucket.eligible(det, input_scalers=True)  # never in a feed-forward bucket
    ff = KerasAutoEncoder(kind="feedforward_hourglass")
    ff.kwargs.update(n_features=4, n_features_out=4)
    ff._prepare_model()
    refused = [
        _detector(_lstm(), window=6),                                     # smoothing window
        _detector(_lstm(), thresholds=False),                             # thresholds required but missing
        _detector(_lstm(), scaler=QuantileTransformer(n_quantiles=5)),    # the error scaler is not affine
        _detector(_lstm(func="relu")),                                    # relu cells: the fp32 kernel only
        _detector(ff),                                                    # a feed-forward network
        _detector(_lstm_unfitted()),
    ]
    for det in refused:
        assert not ResidentBucket.eligible_lstm(det)


def _lstm_unfitted():
    from gordo_components_b200.machine.model.models import KerasLSTMAutoEncoder

    return KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=3)


def test_lstm_grouping_by_architecture_and_thresholds():
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import MinMaxScaler

    from gordo_components_b200.server import ResidentBucket

    models = {
        "ae": _detector(_lstm()),
        "fc": _detector(_lstm("KerasLSTMForecast")),                                 # forecast and autoencoder share a group
        "pipe": _detector(Pipeline([("s", MinMaxScaler()), ("m", _lstm())])),       # so does a Pipeline of the same stack
        "no-thr": _detector(_lstm(), thresholds=False, require_thresholds=False),   # thresholds absent: a group of its own
        "lb5": _detector(_lstm(lookback=5)),                                         # another lookback: another architecture
        "window": _detector(_lstm(), window=6),                                      # not eligible at all
    }
    groups = ResidentBucket.lstm_groups(models)
    assert sorted(map(sorted, groups.values())) == [["ae", "fc", "pipe"], ["lb5"], ["no-thr"]]
    assert max(groups.values(), key=len) == ["ae", "fc", "pipe"]


# ------------------------------------------------------------------------------------------------ the batching rule
class _Eng:
    TILE, lookback, n_features, n_out = 128, 3, 2, 2


def _coalescer(max_tiles):
    from gordo_components_b200.serving import LSTMAnomalyCoalescer

    co = LSTMAnomalyCoalescer.__new__(LSTMAnomalyCoalescer)
    co.eng, co.params, co.max_cost, co.max_wait = _Eng(), np.zeros((4, 1)), max_tiles, 0.2
    co.launched = []
    co.gate = threading.Event()

    def launch(torch, batch, cost):
        co.gate.wait(5)
        co.launched.append(([len(item[2]) for item in batch], cost))
        for item in batch:
            item[-1].set_result(None)

    co._launch = launch
    return co


def test_lstm_batches_close_at_the_tile_cap():
    co = _coalescer(max_tiles=4)
    co._start()
    try:
        first = co.submit(0, np.zeros((130, 2)), np.zeros((128, 2)))  # 1 tile
        time.sleep(0.05)  # inside the first batch's 0.2 s wait
        futs = [co.submit(1, np.zeros((n + 2, 2)), np.zeros((n, 2))) for n in (129, 100, 1, 256, 384)]  # 2, 1, 1, 2, 3 tiles
        co.gate.set()
        for f in [first, *futs]:
            f.result(5)
    finally:
        co.close()
    batches = co.launched
    assert [w for b, _ in batches for w in b] == [128, 129, 100, 1, 256, 384]
    assert all(cost <= 4 for _, cost in batches)
    assert [cost for _, cost in batches] == [sum(-(-w // 128) for w in b) for b, _ in batches]
    assert batches == [([128, 129, 100], 4), ([1, 256], 3), ([384], 3)]
    assert co.batches == 0  # counted by the real _launch only


def test_lstm_requests_are_checked_on_submit():
    co = _coalescer(max_tiles=2)
    co._q, co._closed = queue.Queue(), False
    with pytest.raises(ValueError, match="max_batch_tiles"):
        co.submit(0, np.zeros((259, 2)), np.zeros((257, 2)))  # 3 tiles
    with pytest.raises(ValueError, match="windows"):
        co.submit(0, np.zeros((10, 2)), np.zeros((9, 2)))  # a lookback of 3 gives at most 8 windows
    with pytest.raises(ValueError, match="does not fit"):
        co.submit(0, np.zeros((10, 3)), np.zeros((8, 2)))
    with pytest.raises(ValueError, match="slot"):
        co.submit(4, np.zeros((10, 2)), np.zeros((8, 2)))
    co.submit(3, np.zeros((10, 2)), np.zeros((8, 2)))
    assert co._q.qsize() == 1
