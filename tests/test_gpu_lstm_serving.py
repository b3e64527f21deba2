"""
LSTM detectors served through the request coalescer (server.ResidentBucket(lstm=True), serving.LSTMAnomalyCoalescer) and the
ragged tile layout of the tensor-core LSTM launch under it (gb_lstm_infer_tc_ragged): every window is the same bits as in the
uniform entry, every reply the same bytes as the per-request route.
"""
import json
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("needs an H100")
    import __graft_entry__ as ge

    ge.build()
    return t


# ------------------------------------------------------------------------------------------------ kernel
RAGGED_CASES = {
    "padded-widths-tanh-L1": dict(F=5, units=[65, 130], acts=["tanh", "tanh"], F_out=3, L=1),
    "sigmoid-L144": dict(F=4, units=[64, 32], acts=["sigmoid", "tanh"], F_out=6, L=144),
    "sigmoid-cells-L7": dict(F=9, units=[130], acts=["sigmoid"], F_out=9, L=7),
}


@pytest.mark.parametrize("case", sorted(RAGGED_CASES))
def test_ragged_launch_equals_uniform_per_job(torch, case):
    from gordo_components_b200 import engine

    c = RAGGED_CASES[case]
    eng = engine.LSTMEngine(c["F"], c["units"], c["acts"], c["F_out"], "linear", c["L"])
    params = eng.initial_params(3, torch.Generator(device=eng.device).manual_seed(7))
    windows = np.array([1, 127, 128, 129, 300, 0, 64])
    slots = np.array([0, 1, 2, 0, 1, 2, 2])
    x_rows = np.array([0, 5, 40, 5, 100, 0, 90])  # jobs of different slots read overlapping x rows
    n_x = int(max(x_rows + windows + c["L"] - 1))
    x = torch.randn((n_x, c["F"]), generator=torch.Generator().manual_seed(1)).to(eng.device) * 3
    out_rows = np.concatenate([[0], np.cumsum(windows)])
    jobs = engine.make_jobs(slots, windows, x_rows, out_rows[:-1])
    tb = eng.tile_base(windows)
    got = eng.infer(params, engine.jobs_to_device(jobs, eng.device), len(jobs), int(windows.max()), x, int(out_rows[-1]),
                    tile_base=torch.from_numpy(tb).to(eng.device), n_tiles=int(tb[-1]))
    uniform = eng.infer(params, engine.jobs_to_device(jobs, eng.device), len(jobs), int(windows.max()), x, int(out_rows[-1]), variant=2)
    assert torch.equal(got, uniform)
    for j, n in enumerate(windows):
        if n == 0:
            continue
        one = engine.make_jobs([slots[j]], [n], [x_rows[j]], [0])
        want = eng.infer(params, engine.jobs_to_device(one, eng.device), 1, int(n), x, int(n), variant=2)
        assert torch.equal(got[out_rows[j]:out_rows[j + 1]], want), (case, j)
    assert torch.isfinite(got).all()


# ------------------------------------------------------------------------------------------------ coalescer and server
T, L = 4, 6


def _series(rows, seed):
    rng = np.random.default_rng(seed)
    t = np.linspace(0, 25, rows)[:, None]
    values = (0.5 + 0.4 * np.sin(t * rng.uniform(0.5, 2, T) + rng.uniform(0, 3, T)) + rng.normal(0, 0.02, (rows, T))) * rng.uniform(1, 50, T)
    idx = pd.date_range("2019-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(values, index=idx, columns=[f"TAG {i}" for i in range(T)])


def _lstm_detector(kind, pre, thresholds, frame):
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import MinMaxScaler, StandardScaler

    from gordo_components_b200.machine.model import models
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector

    net = getattr(models, kind)(kind="lstm_hourglass", lookback_window=L, epochs=1, encoding_layers=2)
    est = net if pre is None else Pipeline([("scale", {"minmax": MinMaxScaler, "standard": StandardScaler}[pre]()), ("net", net)])
    det = DiffBasedAnomalyDetector(base_estimator=est, require_thresholds=thresholds)
    if thresholds:
        det.cross_validate(X=frame, y=frame)
    return det.fit(frame, frame)


@pytest.fixture(scope="module")
def store(torch, tmp_path_factory):
    from gordo_components_b200 import serializer, server
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    root = tmp_path_factory.mktemp("lstm-store")
    names = []
    i = 0
    for thresholds in (True, False):
        for kind in ("KerasLSTMAutoEncoder", "KerasLSTMForecast"):
            for pre in (None, "minmax", "standard"):
                name = f"lstm-{i}"
                det = _lstm_detector(kind, pre, thresholds, _series(300, i))
                serializer.dump(det, str(root / name), metadata={"dataset": {"tag_list": [f"TAG {t}" for t in range(T)]}})
                names.append(name)
                i += 1
    ff = DiffBasedAnomalyDetector(base_estimator=KerasAutoEncoder(kind="feedforward_hourglass", epochs=1))
    frame = _series(300, 99)
    ff.cross_validate(X=frame, y=frame)
    ff.fit(frame, frame)
    serializer.dump(ff, str(root / "ff-0"), metadata={"dataset": {"tag_list": [f"TAG {t}" for t in range(T)]}})
    return server.ModelStore(str(root))


def _requests(n_req, seed):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_req):
        rows = int(rng.integers(L + 2, 180))
        X = _series(rows, 1000 + seed * 100 + k)
        y = X.copy()
        if k % 3 == 0:
            X.iloc[int(rng.integers(rows)), int(rng.integers(T))] = np.nan
        if k % 4 == 1:
            y.iloc[int(rng.integers(rows)), int(rng.integers(T))] = np.nan
        out.append((X, y))
    return out


def _assert_blocks_equal(got, want):
    (gi, gb, gc), (wi, wb, wc) = got, want
    assert list(gc) == list(wc)
    assert (gi == wi).all()
    assert len(gb) == len(wb)
    for g, w in zip(gb, wb):
        g = g.to_numpy() if isinstance(g, pd.DataFrame) else np.asarray(g)
        w = w.to_numpy() if isinstance(w, pd.DataFrame) else np.asarray(w)
        assert g.dtype == w.dtype and g.shape == w.shape
        if g.dtype == object:  # the start / end timestamp strings
            assert g.tolist() == w.tolist()
        else:
            assert g.tobytes() == w.tobytes()  # bit for bit, NaN included


def test_coalesced_lstm_blocks_equal_the_models_own(store, torch):
    from torch.profiler import ProfilerActivity, profile

    from gordo_components_b200 import server

    lstm_names = [n for n in store.names() if n.startswith("lstm-")]
    with_thr = [n for n in lstm_names if store.model(n).require_thresholds]
    without = [n for n in lstm_names if n not in with_thr]
    buckets = [server.ResidentBucket(store, names=with_thr, lstm=True, max_wait_ms=20),
               server.ResidentBucket(store, names=without, lstm=True, max_wait_ms=20)]
    try:
        assert sorted(buckets[0].names) == sorted(with_thr) and sorted(buckets[1].names) == sorted(without)
        work = [(name, X, y) for k, (X, y) in enumerate(_requests(48, 3)) for name in [lstm_names[k % len(lstm_names)]]]
        want = [store.model(n).anomaly_blocks(X, y) for n, X, y in work]

        def ask(job):
            n, X, y = job
            return next(b for b in buckets if n in b.slot).anomaly_blocks(store, n, X, y)

        with ThreadPoolExecutor(8) as ex:
            got = list(ex.map(ask, work))
        for g, w in zip(got, want):
            _assert_blocks_equal(g, w)
        requests = sum(b.coalescer.requests for b in buckets)
        assert requests == len(work) and sum(b.coalescer.batches for b in buckets) < requests

        # one batch runs lookback x n_layers step kernels, whatever number of requests it holds
        co = buckets[0].coalescer
        n_layers = len(co.eng.units)
        before = co.batches
        reqs = _requests(6, 4)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            # the profiler can lose device records at the edges of its capture window: keep the batch well inside it
            time.sleep(0.2)
            futs = []
            for k, (X, y) in enumerate(reqs):
                Xv = np.asarray(X.values, dtype=np.float32)
                futs.append(co.submit(k % len(co.params), Xv, y.values[-(len(Xv) - L + 1):]))
            for f in futs:
                f.result()
            torch.cuda.synchronize()
            time.sleep(0.2)
        steps = sum(e.count for e in prof.key_averages() if "lstm_tc_step_kernel" in e.key)
        if steps == 0:
            pytest.skip("the profiler lists no kernels here")
        assert steps == (co.batches - before) * L * n_layers
    finally:
        for b in buckets:
            b.close()


def test_server_replies_through_both_buckets_equal_the_per_request_route(store, torch):
    from gordo_components_b200 import server

    ff_bucket = server.ResidentBucket(store)
    lstm_bucket = server.ResidentBucket(store, lstm=True)
    try:
        assert ff_bucket.names == ["ff-0"]  # the LSTM models do not change what a feed-forward bucket holds
        assert all(n.startswith("lstm-") for n in lstm_bucket.names) and len(lstm_bucket.names) == 6
        both = [ff_bucket, lstm_bucket]
        names = ["ff-0", *lstm_bucket.names]
        X, y = _requests(1, 9)[0]
        for name in names:
            payload = {"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(y)}
            want = server.anomaly_prediction(store, name, json=payload)
            got = server.anomaly_prediction(store, name, json=payload, bucket=both)
            assert got.status == want.status == 200
            assert json.dumps(got.body["data"]) == json.dumps(want.body["data"])
            files = {"X": server.dataframe_into_parquet_bytes(X), "y": server.dataframe_into_parquet_bytes(y)}
            assert server.anomaly_prediction(store, name, files=files, fmt="parquet", bucket=both).body == \
                server.anomaly_prediction(store, name, files=files, fmt="parquet").body

        bare = next(n for n in lstm_bucket.names if type(store.model(n).base_estimator).__name__.startswith("KerasLSTM"))
        piped = next(n for n in lstm_bucket.names if n != bare and not type(store.model(n).base_estimator).__name__.startswith("KerasLSTM"))

        def outcome(name, X, y, bucket):
            try:
                r = server.anomaly_prediction(store, name, json={"X": server.dataframe_to_dict(X), "y": server.dataframe_to_dict(y)}, bucket=bucket)
                return r.status, json.dumps(r.body.get("data", r.body))
            except ValueError as e:
                return "ValueError", str(e)

        Xi = X.copy()
        Xi.iloc[3, 1] = np.inf
        yi = y.copy()
        yi.iloc[5, 0] = -np.inf
        short = X.iloc[:L]
        before = lstm_bucket.coalescer.requests
        for name, Xr, yr in ((bare, X, yi), (piped, X, yi), (bare, Xi, y), (piped, Xi, y), (bare, short, short), (piped, short, short)):
            assert outcome(name, Xr, yr, both) == outcome(name, Xr, yr, None), name
        assert outcome(bare, Xi, y, None)[0] == 200  # ±inf in a bare model's X is answered, on the fp32 kernel
        assert lstm_bucket.coalescer.requests == before  # none of these went through the coalescer
    finally:
        ff_bucket.close()
        lstm_bucket.close()
