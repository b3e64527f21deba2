"""
The ragged tile layout of the tensor-core LSTM launch (gb_lstm_infer_tc_ragged, through ``LSTMEngine.infer(tile_base=)``) and the
LSTM request coalescer built on it (``serving.LSTMAnomalyCoalescer``), against the float64 oracle (oracle/keras_math,
oracle/anomaly_math) at the tolerances of parity_helpers.close.

Kernel: lookbacks that take each job's extra input-projection blocks (xk_pad = ceil((lookback - 1) / 128)) through 0, 1 and 2 and
past the 128-row blocks of the projection, widths on both sides of the 64-unit blocks, feature counts up to 512 with more and fewer
outputs than inputs, a sigmoid cell between tanh cells and raw-magnitude inputs.  Each runs in one launch over jobs of 1 to 300
windows (both sides of every 128-window tile edge), empty jobs first, last and in a row, jobs of different slots over the same x
rows, outputs scattered through a longer array whose other rows must keep what they held; and 3000 jobs of 1 to 3 windows.

Coalescer: every block of every reply against the oracle's prediction scored in float64, for batches that gather a subset of the
slots out of order, close at the tile cap or at ``max_jobs`` requests, invert a MinMax target scaler, smooth some of their
requests, hold a forecast-shaped request, or carry no thresholds.
"""
import ctypes as C
import types
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
from parity_helpers import close
from test_gpu_infer_coverage import lstm_engine, lstm_net, lstm_oracle

from oracle import anomaly_math as am
from oracle import keras_math as km

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch as t

    if not t.cuda.is_available():
        pytest.skip("needs an H100")
    import __graft_entry__ as ge

    ge.build()
    return t


@pytest.fixture(scope="module")
def engine(torch):
    from gordo_components_b200 import engine as e

    return e


# ------------------------------------------------------------------------------------------------ the ragged launch
# F, units, cell activations, n_features_out, head, lookback, x magnitude (the input kernel is shrunk by as much)
KERNEL_CASES = {
    "L1_F512_width512": (512, [512], ["tanh"], 300, "linear", 1, 1.0),
    "L2_F300_widths200_65": (300, [200, 65], ["sigmoid", "tanh"], 512, "tanh", 2, 1.0),
    "L127_F1_width1": (1, [1], ["tanh"], 5, "sigmoid", 127, 1.0),
    "L128_width63": (5, [63], ["sigmoid"], 1, "linear", 128, 1.0),
    "L129_width64": (5, [64], ["tanh"], 3, "linear", 129, 1.0),
    "L130_F1_width65": (1, [65], ["tanh"], 4, "linear", 130, 1.0),
    "L144_sigmoid_between_tanh": (5, [32, 16, 32], ["tanh", "sigmoid", "tanh"], 5, "linear", 144, 1.0),
    "L257_width8": (5, [8], ["tanh"], 2, "tanh", 257, 1.0),
    "raw_magnitude_x": (7, [128, 64], ["tanh", "tanh"], 7, "linear", 9, 1e4),
}

# slot, windows, x_row of each job: every window count on both sides of a tile edge; empty jobs first, last and two in a row; jobs
# of different slots over the same x rows (x_row 77, and 0 / 1 / 5); several jobs of each slot, slots out of job order; x rows off
# any 128 boundary
LAYOUT = ([1, 2, 0, 2, 1, 0, 0, 2, 1, 0, 1, 2, 0],
          [0, 1, 127, 128, 0, 0, 129, 255, 256, 257, 300, 3, 0],
          [3, 0, 5, 77, 301, 5, 130, 41, 200, 1, 77, 9, 11])


def scattered_out_rows(windows, seed=0, gap=3):
    """Each job's out_row, in a shuffled job order with `gap` rows before each job and after the last; the output's length."""
    out_row = np.zeros(len(windows), np.int64)
    pos = gap
    for j in np.random.default_rng(seed).permutation(len(windows)):
        out_row[j] = pos
        pos += int(windows[j]) + gap
    return out_row, pos


def infer_into(engine, torch, eng, out, params, jobs_d, n_jobs, max_windows, x, tb_d, n_tiles):
    """The gb_lstm_infer_tc_ragged call of ``LSTMEngine.infer(tile_base=)``, writing into a given ``out``: the engine allocates its
    own, whose rows outside every job hold whatever the allocator left there."""
    from gordo_components_b200 import _cabi

    p = _cabi.ptr
    ws = torch.empty((eng.tc_workspace_bytes(params.shape[0], n_jobs, max_windows, n_tiles) + 255,), dtype=torch.uint8, device=eng.device)
    _cabi.check(eng.lib.gb_lstm_infer_tc_ragged(C.byref(eng.net), p(params), int(params.shape[0]), p(jobs_d), int(n_jobs), p(tb_d), int(n_tiles),
                                                int(max_windows), p(x), int(x.shape[0]), p(out), p(ws), engine._stream_ptr()))


def run_ragged(engine, torch, spec, nets, X, jobs_h, out_rows):
    """One ragged launch of the jobs through ``LSTMEngine.infer``, and the same launch into an output filled with NaN; both on the host."""
    eng = lstm_engine(engine, spec)
    assert eng.tc_supported
    dev = eng.device
    params = eng.pack_params([w for _, w in nets])
    jobs_d = engine.jobs_to_device(jobs_h, dev)
    windows = jobs_h["n_rows"]
    tb = eng.tile_base(windows)
    tb_d = torch.from_numpy(tb).to(dev)
    x = torch.from_numpy(np.ascontiguousarray(X, np.float32)).to(dev)
    max_windows = int(windows.max())
    got = eng.infer(params, jobs_d, len(jobs_h), max_windows, x, out_rows, tile_base=tb_d, n_tiles=int(tb[-1]))
    filled = torch.full((out_rows, spec.n_features_out), float("nan"), device=dev)
    infer_into(engine, torch, eng, filled, params, jobs_d, len(jobs_h), max_windows, x, tb_d, int(tb[-1]))
    torch.cuda.synchronize()
    return got.cpu().numpy(), filled.cpu().numpy()


@pytest.mark.parametrize("case", list(KERNEL_CASES))
def test_ragged_launch_matches_the_oracle(engine, torch, case):
    F, units, acts, F_out, head, L, x_mag = KERNEL_CASES[case]
    nets = [lstm_net(km, F, units, acts, F_out, head, L, 20 + 2 * s) for s in range(3)]
    if x_mag != 1.0:  # pre-activations of order 1 for x of order x_mag: the input kernel is shrunk, not the data
        nets = [(spec, ([((K / np.float32(x_mag)).astype(np.float32) if i == 0 else K, U, b) for i, (K, U, b) in enumerate(layers)], dense))
                for spec, (layers, dense) in nets]
    spec = nets[0][0]
    slots, windows, x_row = (np.array(v, np.int64) for v in LAYOUT)
    out_row, out_rows = scattered_out_rows(windows)
    n_x = int((x_row + windows + L - 1).max())
    X = (np.random.default_rng(L).random((n_x, F)) * x_mag).astype(np.float32)
    jobs = engine.make_jobs(slots, windows, x_row, out_row)
    got, filled = run_ragged(engine, torch, spec, nets, X, jobs, out_rows)
    written = np.zeros(out_rows, bool)
    for j in range(len(jobs)):
        s, n, xr, orow = int(slots[j]), int(windows[j]), int(x_row[j]), int(out_row[j])
        if n == 0:
            continue
        rows = slice(orow, orow + n)
        written[rows] = True
        want = lstm_oracle(km, spec, nets[s][1], X, xr, n)
        close(got[rows], want, max(1.0, float(np.abs(want).max())), name=f"{case}: job {j} ({n} windows of slot {s} from x row {xr})")
    assert written.sum() == windows.sum()
    np.testing.assert_array_equal(filled[written], got[written])
    assert np.isnan(filled[~written]).all(), f"{case}: rows outside every job's output written"


def test_ragged_launch_of_3000_short_jobs(engine, torch):
    """3000 jobs of 1 to 3 windows over two slots, a tile each, at x rows anywhere: every window against the oracle."""
    J, L, F = 3000, 5, 3
    nets = [lstm_net(km, F, [20], ["tanh"], F, "linear", L, 60 + s) for s in range(2)]
    spec = nets[0][0]
    rng = np.random.default_rng(12)
    n_x = 2000
    windows = rng.integers(1, 4, J)
    slots = rng.integers(0, 2, J)
    x_row = rng.integers(0, n_x - L - 1, J)  # the last window of a 3-window job ends at row n_x - 1 at most
    out_row = np.concatenate([[0], np.cumsum(windows)[:-1]])
    X = rng.random((n_x, F)).astype(np.float32)
    got, filled = run_ragged(engine, torch, spec, nets, X, engine.make_jobs(slots, windows, x_row, out_row), int(windows.sum()))
    every = np.stack([km.lstm_predict(spec, w, X, dtype=np.float64) for _, w in nets])  # [slot, window starting at x row, out]
    job = np.repeat(np.arange(J), windows)
    src = x_row[job] + np.arange(len(job)) - out_row[job]
    want = every[slots[job], src]
    close(got, want, max(1.0, float(np.abs(want).max())), name="3000 short jobs")
    np.testing.assert_array_equal(filled, got)


# ------------------------------------------------------------------------------------------------ the LSTM request coalescer
CO_F, CO_L, N_SLOTS = 5, 6, 6
WAIT_MS = 2000.0  # requests submitted together always meet in one batch; a batch not closed by a cap waits this long


@pytest.fixture(scope="module")
def fleet(engine, torch):
    """Six detectors of one architecture (the first layer two unit blocks wide), each slot with its own scale, feature thresholds,
    aggregate threshold and MinMax target scaler."""
    from sklearn.preprocessing import MinMaxScaler

    nets = [lstm_net(km, CO_F, [70, 20], ["tanh", "sigmoid"], CO_F, "linear", CO_L, 80 + s) for s in range(N_SLOTS)]
    spec = nets[0][0]
    eng = lstm_engine(engine, spec)
    rng = np.random.default_rng(13)
    lo, width = rng.uniform(-20, 20, (N_SLOTS, CO_F)), rng.uniform(1, 60, (N_SLOTS, CO_F))
    targets = [MinMaxScaler().fit(lo[s] + width[s] * rng.random((50, CO_F))) for s in range(N_SLOTS)]
    return types.SimpleNamespace(spec=spec, weights=[w for _, w in nets], eng=eng, params=eng.pack_params([w for _, w in nets]),
                                 scale=rng.uniform(0.5, 2.0, (N_SLOTS, CO_F)), feat=rng.uniform(0.05, 0.25, (N_SLOTS, CO_F)),
                                 agg=rng.uniform(0.01, 0.11, N_SLOTS), targets=targets, lo=lo, width=width)


def make_coalescer(torch, fleet, feat=True, agg=True, ttr=False, **kw):
    from gordo_components_b200 import serving

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(fleet.eng.device)

    y_inverse = (dev([t.scale_ for t in fleet.targets]), dev([t.min_ for t in fleet.targets])) if ttr else None
    return serving.LSTMAnomalyCoalescer(fleet.eng, fleet.params, dev(fleet.scale), dev(fleet.feat) if feat else None,
                                        dev(fleet.agg) if agg else None, max_wait_ms=WAIT_MS, y_inverse=y_inverse, **kw)


def make_request(fleet, slot, n_windows, seed, forecast=False, ttr=False, smooth=False):
    """(slot, X, y, smooth): X of n_windows + lookback - 1 rows (one more for a forecast, whose last row is not read), float64 y of
    the windows' targets, in the targets' own units when the detectors invert a target scaler."""
    rng = np.random.default_rng(seed)
    X = rng.random((n_windows + CO_L - 1 + int(forecast), CO_F)).astype(np.float32)
    y = rng.random((n_windows, CO_F))
    if ttr:
        y = fleet.lo[slot] + fleet.width[slot] * y
    return slot, X, y, smooth


def submit_all(co, reqs, threads=8):
    """Every request submitted from a thread pool; the replies in request order."""
    with ThreadPoolExecutor(threads) as ex:
        futs = list(ex.map(lambda r: co.submit(*r), reqs))
    return [f.result(timeout=300) for f in futs]


def oracle_reply(fleet, slot, X, y, smooth, feat=True, agg=True, ttr=False, smoothing=None):
    """What the reply must hold: the float64 oracle's prediction (through sklearn's float32 inverse of the slot's target scaler when
    ``ttr``) scored in float64; and the magnitude of the prediction, in the reply's units."""
    pred = lstm_oracle(km, fleet.spec, fleet.weights[slot], X, 0, len(y))  # the windows from X's first row: a forecast's last row unread
    mag = max(1.0, float(np.abs(pred).max()))
    if ttr:
        t = fleet.targets[slot]
        pred = t.inverse_transform(pred.astype(np.float32))
        assert pred.dtype == np.float32
        mag = max(float(np.abs(pred).max()), mag / float(t.scale_.min()))
    window, method = smoothing if smooth else (None, None)
    want = am.anomaly_arrays(pred, y, fleet.scale[slot], np.zeros(CO_F), fleet.feat[slot] if feat else None,
                             float(fleet.agg[slot]) if agg else None, window, method)
    return want, mag


def check_reply(got, want, mag, scale, feat, agg, name):
    """Every block of a reply against the oracle's, at tolerances scaled as test_gpu_infer_coverage.check_dense scales them."""
    assert sorted(got) == sorted(want), name
    d = max(1.0, float(np.nanmax(want["tag-anomaly-unscaled"])))
    tot = 2 * mag * d * float(scale.max()) ** 2
    mags = {"model-output": mag, "tag-anomaly-unscaled": mag, "tag-anomaly-scaled": mag * float(scale.max()),
            "anomaly-confidence": mag / float(feat.min()), "total-anomaly-unscaled": 2 * mag * d, "total-anomaly-scaled": tot,
            "total-anomaly-confidence": tot / float(np.min(agg))}
    for k, w in want.items():
        dtype = np.float32 if k == "model-output" or k.startswith("smooth-") else np.float64
        assert got[k].dtype == dtype and got[k].shape == w.shape, (name, k, got[k].dtype, got[k].shape)
        close(got[k], w, mags[k.removeprefix("smooth-")], name=f"{name}: {k}")


def check_replies(fleet, reqs, replies, feat=True, agg=True, ttr=False, smoothing=None):
    for i, ((slot, X, y, smooth), got) in enumerate(zip(reqs, replies)):
        want, mag = oracle_reply(fleet, slot, X, y, smooth, feat, agg, ttr, smoothing)
        check_reply(got, want, mag, fleet.scale[slot], fleet.feat[slot], fleet.agg[slot], f"request {i} ({len(y)} windows of slot {slot})")


def test_coalesced_replies_match_the_oracle(torch, fleet):
    """A batch of slots {5, 0, 5, 2} (slot 1 never asked for: the compact map is no identity) with 1, 128 and 129 windows and a
    forecast-shaped request; then 24 requests of every slot and 1 to 300 windows."""
    co = make_coalescer(torch, fleet)
    try:
        reqs = [make_request(fleet, s, n, 100 + i, forecast=i == 3) for i, (s, n) in enumerate(zip([5, 0, 5, 2], [1, 128, 129, 40]))]
        check_replies(fleet, reqs, submit_all(co, reqs))
        assert (co.batches, co.requests) == (1, 4)
        rng = np.random.default_rng(14)
        reqs = [make_request(fleet, int(rng.integers(N_SLOTS)), int(rng.integers(1, 301)), 200 + i, forecast=i % 5 == 0) for i in range(24)]
        check_replies(fleet, reqs, submit_all(co, reqs))
        assert co.requests == 28 and co.batches < co.requests
    finally:
        co.close()


def test_batch_closes_at_the_tile_cap(torch, fleet):
    """max_batch_tiles=4: requests of 1, 2 and 1 tiles close a batch at exactly 4 tiles; the next request is a batch of its own."""
    co = make_coalescer(torch, fleet, max_batch_tiles=4)
    try:
        reqs = [make_request(fleet, s, n, 300 + i) for i, (s, n) in enumerate(zip([3, 1, 3, 0], [128, 129, 1, 7]))]
        futs = [co.submit(*r) for r in reqs]  # in order, from one thread: the first three fill the cap
        check_replies(fleet, reqs, [f.result(timeout=300) for f in futs])
        assert (co.batches, co.requests) == (2, 4)
    finally:
        co.close()


def test_batch_of_max_jobs_requests(torch, fleet):
    """max_jobs one-window requests of every slot in one batch (a tile each), and one more request in the next."""
    co = make_coalescer(torch, fleet, max_batch_tiles=8192)
    J = co.max_jobs + 1
    try:
        slots = np.arange(J) % N_SLOTS
        reqs = [make_request(fleet, int(s), 1, 400 + i) for i, s in enumerate(slots)]
        replies = submit_all(co, reqs)
        assert (co.batches, co.requests) == (2, J)
    finally:
        co.close()
    # every request at once: per slot, the oracle on all of its windows; the scores on every row with its own slot's scale and thresholds
    pred = np.empty((J, CO_F))
    for s in range(N_SLOTS):
        sel = np.flatnonzero(slots == s)
        pred[sel] = km.lstm_forward_windows(fleet.spec, fleet.weights[s], np.stack([reqs[i][1] for i in sel]), np.float64)
    y = np.concatenate([r[2] for r in reqs])
    want = am.anomaly_arrays(pred, y, fleet.scale[slots], np.zeros(CO_F), fleet.feat[slots], fleet.agg[slots])
    got = {k: np.concatenate([r[k] for r in replies]) for k in replies[0]}
    check_reply(got, want, max(1.0, float(np.abs(pred).max())), fleet.scale, fleet.feat, fleet.agg, f"{J} one-window requests")


def test_target_inverse_replies(torch, fleet):
    """``y_inverse``: the prediction through each slot's float32 MinMax inverse, then scored in float64 against y in the targets' units."""
    co = make_coalescer(torch, fleet, ttr=True)
    try:
        reqs = [make_request(fleet, s, n, 500 + i, forecast=i == 4, ttr=True)
                for i, (s, n) in enumerate(zip([5, 0, 5, 2, 4, 1], [1, 128, 129, 300, 40, 17]))]
        check_replies(fleet, reqs, submit_all(co, reqs), ttr=True)
        assert (co.batches, co.requests) == (1, 6)
    finally:
        co.close()


@pytest.mark.parametrize("method,window", [("smm", 5), ("sma", 12), ("ewma", 30)])
def test_smoothed_replies(torch, fleet, method, window):
    """``smoothing=(window, method)``: the requests that ask for it get the four smoothed score arrays of their own rows (shorter
    ones than the window included), the others none."""
    co = make_coalescer(torch, fleet, smoothing=(window, method))
    try:
        reqs = [make_request(fleet, s, n, 600 + i, forecast=i == 2, smooth=sm)
                for i, (s, n, sm) in enumerate(zip([5, 0, 5, 2, 1, 3], [1, 4, 12, 128, 129, 300], [True, False, True, True, False, True]))]
        check_replies(fleet, reqs, submit_all(co, reqs), smoothing=(window, method))
        assert (co.batches, co.requests) == (1, 6)
    finally:
        co.close()


@pytest.mark.parametrize("feat,agg", [(False, False), (True, False), (False, True)], ids=["neither", "feature-only", "aggregate-only"])
def test_replies_without_thresholds(torch, fleet, feat, agg):
    """A coalescer without feature or aggregate thresholds answers no confidence block for the missing ones."""
    co = make_coalescer(torch, fleet, feat=feat, agg=agg)
    try:
        reqs = [make_request(fleet, s, n, 700 + i) for i, (s, n) in enumerate(zip([5, 0, 5, 2], [1, 128, 129, 64]))]
        replies = submit_all(co, reqs)
        assert all(("anomaly-confidence" in r) == feat and ("total-anomaly-confidence" in r) == agg for r in replies)
        check_replies(fleet, reqs, replies, feat=feat, agg=agg)
    finally:
        co.close()
