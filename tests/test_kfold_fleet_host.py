"""
The batched K-fold build without a device: which DiffBasedKFCVAnomalyDetector machines FleetModelBuilder(kfcv=True) batches and
how it buckets them, the fold layout and row maps against sklearn's KFold + shuffle, the per-slot scaler extrema combined from
test blocks, and the CV metrics from moments on folds of unequal size.
"""
import numpy as np
import pandas as pd
import pytest
from sklearn import metrics as skm
from sklearn.model_selection import KFold
from sklearn.preprocessing import MinMaxScaler
from sklearn.utils import shuffle as sk_shuffle

from gordo_components_b200 import builder, fleet

AE = {"gordo.machine.model.models.KerasAutoEncoder": {"kind": "feedforward_hourglass", "batch_size": 128, "compression_factor": 0.5,
                                                      "encoding_layers": 1, "func": "tanh", "out_func": "linear", "epochs": 3}}
PIPE = {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", AE]}}
KFOLD = {"sklearn.model_selection.KFold": {"n_splits": 5, "shuffle": True, "random_state": 0}}


def ttr(regressor, **kw):
    return {"sklearn.compose.TransformedTargetRegressor": {"transformer": "sklearn.preprocessing.MinMaxScaler", "regressor": regressor, **kw}}


def machine(base=PIPE, cv=KFOLD, name="m", rows=300, tags=6, **det):
    frame = pd.DataFrame(np.random.default_rng(0).random((rows, tags)), columns=[f"t{i}" for i in range(tags)])
    model = {"gordo.machine.model.anomaly.diff.DiffBasedKFCVAnomalyDetector": {
        "base_estimator": base, "scaler": "sklearn.preprocessing.MinMaxScaler", "window": 144, "shuffle": True, "threshold_percentile": 0.975, **det}}
    evaluation = {} if cv is None else {"cv": cv}
    return {"name": name, "model": model, "dataset": {"X": frame, "y": frame}, "evaluation": evaluation}


@pytest.mark.parametrize("base", [AE, PIPE, ttr(AE), ttr(PIPE)], ids=["bare", "pipeline", "ttr-bare", "ttr-pipeline"])
def test_canonical_forms_are_batched_only_with_the_flag(base):
    m = machine(base)
    assert builder._is_kfcv_definition(m)
    c = builder._canonical_kfcv(0, m)
    assert c is not None and c.n_splits == 5
    assert c.target_scaler == ("TransformedTargetRegressor" in str(base))
    assert c.input_scaler == ("Pipeline" in str(base))
    assert builder._canonical(0, m) is None  # the flag off: the TimeSeriesSplit path refuses it, so ModelBuilder builds it


def test_window_none_and_smoothing_methods_are_batched():
    for det in ({"window": None}, {"smoothing_method": "sma"}, {"smoothing_method": "ewma"}, {"shuffle": False}):
        assert builder._canonical_kfcv(0, machine(**det)) is not None, det
    assert builder._canonical_kfcv(0, machine(cv={"sklearn.model_selection.KFold": {"n_splits": 3}})) is not None


@pytest.mark.parametrize("case", ["timeseries", "default-cv", "unseeded", "randomstate", "transformer", "func", "callbacks", "other-scaler"])
def test_refusals(case, monkeypatch):
    if case == "randomstate":  # a definition cannot name a RandomState object: hand the builder one as if it had
        build = builder.serializer.from_definition
        monkeypatch.setattr(builder.serializer, "from_definition",
                            lambda d: KFold(5, shuffle=True, random_state=np.random.RandomState(0)) if d == "kfold-randomstate" else build(d))
    m = {
        "timeseries": lambda: machine(cv={"sklearn.model_selection.TimeSeriesSplit": {"n_splits": 3}}),
        "default-cv": lambda: machine(cv=None),
        "unseeded": lambda: machine(cv={"sklearn.model_selection.KFold": {"n_splits": 5, "shuffle": True}}),
        "randomstate": lambda: machine(cv="kfold-randomstate"),
        "transformer": lambda: machine(ttr(AE, transformer="sklearn.preprocessing.StandardScaler")),
        "func": lambda: machine({"sklearn.compose.TransformedTargetRegressor": {"regressor": AE, "func": "numpy.log1p", "inverse_func": "numpy.expm1"}}),
        "callbacks": lambda: machine({"gordo.machine.model.models.KerasAutoEncoder": {
            **AE["gordo.machine.model.models.KerasAutoEncoder"], "validation_split": 0.1,
            "callbacks": [{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "val_loss", "patience": 2}}]}}),
        "other-scaler": lambda: machine({"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.StandardScaler", AE]}}),
    }[case]()
    assert builder._canonical_kfcv(0, m) is None


def test_early_stopping_is_batched_with_its_flag():
    m = machine({"gordo.machine.model.models.KerasAutoEncoder": {
        **AE["gordo.machine.model.models.KerasAutoEncoder"], "validation_split": 0.1,
        "callbacks": [{"tensorflow.keras.callbacks.EarlyStopping": {"monitor": "val_loss", "patience": 10, "restore_best_weights": True}}]}})
    assert builder._canonical_kfcv(0, m) is None
    c = builder._canonical_kfcv(0, m, early_stopping=True)
    assert c is not None and c.early_stopping.patience == 10 and c.split[1] == 0.1


def test_an_lstm_kfold_detector_stays_refused():
    lstm = {"gordo.machine.model.models.KerasLSTMAutoEncoder": {"kind": "lstm_hourglass", "lookback_window": 8, "epochs": 1}}
    m = machine(lstm)
    assert builder._is_lstm_definition(m)  # FleetModelBuilder asks the LSTM classifier first, which refuses a K-fold detector
    assert builder._canonical_lstm(0, m) is None
    assert builder._canonical_kfcv(0, m) is None


def test_bucket_keys_separate_on_every_new_field():
    ref = builder._canonical_kfcv(0, machine()).bucket()
    variants = [
        machine(cv={"sklearn.model_selection.KFold": {"n_splits": 4, "shuffle": True, "random_state": 0}}),
        machine(cv={"sklearn.model_selection.KFold": {"n_splits": 5}}),
        machine(cv={"sklearn.model_selection.KFold": {"n_splits": 5, "shuffle": True, "random_state": 1}}),
        machine(window=12), machine(window=None), machine(smoothing_method="ewma"), machine(threshold_percentile=0.99),
        machine(shuffle=False), machine(ttr(PIPE)),
    ]
    keys = [builder._canonical_kfcv(0, v).bucket() for v in variants]
    assert all(k != ref for k in keys)
    assert len(set(keys)) == len(keys)
    assert builder._canonical_kfcv(1, machine(name="other")).bucket() == ref


@pytest.mark.parametrize("rows,k,detector_shuffle", [(103, 5, True), (103, 5, False), (60, 3, True), (11, 2, True)])
def test_row_maps_give_every_estimator_its_sklearn_rows(rows, k, detector_shuffle):
    cv = KFold(k, shuffle=True, random_state=0)
    tests, trains, order, inverse = fleet.kfold_layout(cv, rows)
    data = np.random.default_rng(1).random((rows, 3))
    folded = data[order]  # the fold-order copy gb_gather_rows lays out
    ofs = 0
    for j, (tr, te) in enumerate(cv.split(data)):
        assert np.array_equal(folded[ofs:ofs + len(te)], data[te])  # fold k's test rows are one contiguous block
        ofs += len(te)
    maps = fleet.kfold_row_maps(trains, inverse, rows, detector_shuffle)
    assert len(maps) == k + 1
    want_final = sk_shuffle(data, random_state=0) if detector_shuffle else data
    assert np.array_equal(folded[maps[0]], want_final)
    for j, (tr, _) in enumerate(cv.split(data)):
        want = sk_shuffle(data[tr], random_state=0) if detector_shuffle else data[tr]  # what the fold clone's fit hands its estimator
        assert np.array_equal(folded[maps[j + 1]], want)


def test_a_cv_that_does_not_test_every_row_is_refused():
    from sklearn.model_selection import TimeSeriesSplit

    with pytest.raises(ValueError, match="exactly once"):
        fleet.kfold_layout(TimeSeriesSplit(3), 40)


def test_fold_extrema_from_block_extrema_equal_sklearn_to_the_last_bit():
    rows, K, M = 257, 5, 3
    rng = np.random.default_rng(4)
    data = [rng.normal(100.0, 3.0, (rows, 7)) * rng.uniform(0.01, 10, 7) for _ in range(M)]
    data[1][:, 2] = 5.0  # a constant column: _handle_zeros_in_scale
    cv = KFold(K, shuffle=True, random_state=0)
    tests, trains, order, inverse = fleet.kfold_layout(cv, rows)
    lo = np.stack([[d[t].min(axis=0) for d in data] for t in tests])  # what gb_minmax_f64 gives per test block: [K, M, T]
    hi = np.stack([[d[t].max(axis=0) for d in data] for t in tests])
    s_lo, s_hi = fleet.combine_fold_extrema(lo, hi)
    for m in range(M):
        for slot, rows_of in [(m, np.arange(rows))] + [(M + k * M + m, trains[k]) for k in range(K)]:
            ref = MinMaxScaler().fit(data[m][rows_of])
            sc = fleet._fill_minmax_from_extrema(MinMaxScaler(), s_lo[slot], s_hi[slot], len(rows_of), None)
            for name in ("data_min_", "data_max_", "data_range_", "scale_", "min_"):
                assert np.array_equal(getattr(sc, name), getattr(ref, name)), (m, slot, name)


def test_scores_from_moments_with_per_fold_counts_equal_sklearn_on_unequal_folds():
    rows, K, T = 103, 5, 4  # KFold(5) over 103 rows: folds of 21, 21, 21, 20, 20 rows
    rng = np.random.default_rng(7)
    y = rng.normal(size=(rows, T)) * [1.0, 10.0, 0.1, 3.0] + [0.0, 50.0, -2.0, 7.0]
    pred = y + rng.normal(scale=0.2, size=(rows, T))
    pred[:, 3] = y[:, 3]  # exact predictions of one tag
    folds = [te for _, te in KFold(K, shuffle=True, random_state=0).split(y)]
    counts = np.asarray([len(te) for te in folds])
    assert len(set(counts)) == 2
    moments = []
    for te in folds:  # the five sums gb_cv_moments computes per fold and tag
        e, c = pred[te] - y[te], y[te] - y[te][0]
        moments.append(np.stack([e.sum(0), (e * e).sum(0), np.abs(e).sum(0), c.sum(0), (c * c).sum(0)]))
    scale = MinMaxScaler().fit(y).scale_
    got = builder.scores_from_moments(np.stack(moments), counts, scale)
    sy, sp = MinMaxScaler().fit(y).transform(y), None
    sp = MinMaxScaler().fit(y).transform(pred)
    for name, func, scaled in [("explained_variance_score", skm.explained_variance_score, False), ("r2_score", skm.r2_score, False),
                               ("mean_squared_error", skm.mean_squared_error, True), ("mean_absolute_error", skm.mean_absolute_error, True)]:
        per_tag, averaged = got[name]
        for k, te in enumerate(folds):
            yt, yp = (sy[te], sp[te]) if scaled else (y[te], pred[te])
            want = [func(yt[:, j], yp[:, j]) for j in range(T)]
            np.testing.assert_allclose(per_tag[k], want, rtol=1e-9, atol=1e-12, err_msg=f"{name} fold {k}")
            np.testing.assert_allclose(averaged[k], func(yt, yp), rtol=1e-9, atol=1e-12, err_msg=f"{name} fold {k}")
    # the int form is unchanged
    same = builder.scores_from_moments(np.stack(moments), 21, scale)
    np.testing.assert_array_equal(same["r2_score"][0][:3], builder.scores_from_moments(np.stack(moments), counts, scale)["r2_score"][0][:3])
