"""
TransformedTargetRegressor detectors on the serving side, without a GPU: the argument checks of gb_minmax_inverse_score_f64, which
detectors a ``ResidentBucket(target_scaler=True)`` admits and how it groups them, and that the other buckets still refuse them.
"""
import ctypes as C

import numpy as np
import pandas as pd
import pytest

from gordo_components_b200 import _cabi, server

T = 4
TAGS = [f"tag-{i}" for i in range(T)]


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


# ------------------------------------------------------------------------------------------------ gb_minmax_inverse_score_f64 arguments
FAKE = C.c_void_p(256)  # never dereferenced: every call below is refused, or has no job, before any launch
OUTS = ("o_ts", "o_tu", "o_tots", "o_totu", "o_conf", "o_totc")


def _call(lib, **kw):
    a = dict(jobs=FAKE, n_jobs=2, max_rows=10, p=FAKE, y=FAKE, n_out=T, y_scale=FAKE, y_min=FAKE, scale=FAKE, feat_thr=FAKE,
             agg_thr=FAKE, o_model=FAKE, **{k: FAKE for k in OUTS})
    a.update(kw)
    return lib.gb_minmax_inverse_score_f64(a["jobs"], a["n_jobs"], a["max_rows"], a["p"], a["y"], a["n_out"], a["y_scale"], a["y_min"],
                                           a["scale"], a["feat_thr"], a["agg_thr"], a["o_model"], *(a[k] for k in OUTS), None)


@pytest.mark.parametrize("arg", ["jobs", "p", "y", "y_scale", "y_min", "o_model"])
def test_refuses_null_pointers(lib, arg):
    assert _call(lib, **{arg: None}) == -1
    assert lib.gb_last_error() == b"jobs/p/y/y_scale/y_min/out_model must be non-NULL"


@pytest.mark.parametrize("kw, code, msg", [
    ({"n_out": 0}, -2, b"n_out=0 must be >= 1"),
    ({"n_out": -3}, -2, b"n_out=-3 must be >= 1"),
    ({"scale": None}, -1, b"scaled outputs requested without scale"),
    ({"scale": None, "o_ts": None, "o_tots": None}, -1, b"scaled outputs requested without scale"),  # the total confidence is scaled too
    ({"scale": None, "o_ts": None, "o_totc": None}, -1, b"scaled outputs requested without scale"),
    ({"feat_thr": None}, -1, b"out_conf requested without feat_thr"),
    ({"agg_thr": None}, -1, b"out_total_conf requested without agg_thr"),
    ({"n_jobs": -1}, -1, b"bad n_jobs"),
    ({"n_out": 0, "n_jobs": 0}, -2, b"n_out=0 must be >= 1"),  # checked even when there is nothing to launch
    ({"p": None, "n_jobs": 0}, -1, b"non-NULL"),
])
def test_refuses_bad_arguments(lib, kw, code, msg):
    assert _call(lib, **kw) == code and msg in lib.gb_last_error()
    with pytest.raises(ValueError):
        _cabi.check(code)


@pytest.mark.parametrize("kw", [{"n_jobs": 0}, {"max_rows": 0}, {"max_rows": -1},
                                {"n_jobs": 0, "scale": None, "feat_thr": None, "agg_thr": None, **{k: None for k in OUTS}},
                                {"n_jobs": 0, "feat_thr": None, "o_conf": None}, {"n_jobs": 0, "agg_thr": None, "o_totc": None}])
def test_accepts_empty_batches_and_absent_outputs_without_a_launch(lib, kw):
    assert _call(lib, **kw) == 0


def test_engine_wrapper_checks_dtypes(lib):
    import torch

    from gordo_components_b200 import engine

    f64 = torch.zeros(5, T, dtype=torch.float64)
    with pytest.raises(ValueError, match="float32 prediction"):
        engine.minmax_inverse_score_f64(None, 1, 5, f64, f64, f64[:1], f64[:1])
    with pytest.raises(ValueError, match="y is torch.float32"):
        engine.minmax_inverse_score_f64(None, 1, 5, f64.float(), f64.float(), f64[:1], f64[:1])
    with pytest.raises(ValueError, match="feat_thr is torch.float32"):
        engine.minmax_inverse_score_f64(None, 1, 5, f64.float(), f64, f64[:1], f64[:1], feat_thr=f64[:1].float())


def test_exported_and_declared(lib):
    import os

    assert "gb_minmax_inverse_score_f64" in _cabi.EXPORTS
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "gordo_b200.h")).read()
    assert "int gb_minmax_inverse_score_f64(" in header


# ------------------------------------------------------------------------------------------------ eligibility and grouping
def _ae(n=T):
    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    ae = KerasAutoEncoder(kind="feedforward_hourglass")
    ae.kwargs.update({"n_features": n, "n_features_out": n})
    ae._prepare_model()
    return ae


def _lstm(n=T):
    from gordo_components_b200.machine.model.models import KerasLSTMAutoEncoder

    return KerasLSTMAutoEncoder(kind="lstm_hourglass", lookback_window=3, encoding_layers=1).initialize(n, n)


def _ttr(reg, transformer=None, fitted=True, **kw):
    """A TransformedTargetRegressor around ``reg`` in the state its fit leaves (what the fleet builder assembles)."""
    from sklearn.base import clone
    from sklearn.compose import TransformedTargetRegressor
    from sklearn.preprocessing import MinMaxScaler

    ttr = TransformedTargetRegressor(regressor=reg, transformer=transformer if transformer is not None else MinMaxScaler(), **kw)
    if fitted:
        rng = np.random.default_rng(1)
        ttr._training_dim = 2
        ttr.transformer_ = clone(ttr.transformer).fit(rng.random((8, T)) * 50)
        ttr.regressor_ = reg
    return ttr


def _piped(est, *steps):
    from sklearn.pipeline import Pipeline
    from sklearn.preprocessing import MinMaxScaler

    steps = steps or (MinMaxScaler(),)
    rng = np.random.default_rng(2)
    for s in steps:
        s.fit(rng.random((8, T)) * 100)
    return Pipeline([(f"s{i}", s) for i, s in enumerate(steps)] + [("m", est)])


def _det(est, kfcv=False, window=None, method=None):
    from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector, DiffBasedKFCVAnomalyDetector

    det = DiffBasedKFCVAnomalyDetector(base_estimator=est) if kfcv else DiffBasedAnomalyDetector(base_estimator=est, window=window,
                                                                                                 smoothing_method=method)
    det.scaler.fit(np.random.default_rng(0).random((8, T)))
    det.feature_thresholds_, det.aggregate_threshold_ = pd.Series(np.ones(T), index=TAGS), 0.5
    return det


ALL_FLAGS = dict(input_scalers=True, smoothing=True, target_scaler=True)


def test_admitted_forms(lib):
    for kfcv in (False, True):
        bare = _det(_ttr(_ae()), kfcv)
        piped = _det(_ttr(_piped(_ae())), kfcv)
        for det in (bare, piped):
            assert server.ResidentBucket.eligible(det, **ALL_FLAGS)
            assert not server.ResidentBucket.eligible(det)  # the default bucket refuses a TTR, as before
            assert not server.ResidentBucket.eligible(det, input_scalers=True, smoothing=True)  # and so do the existing flags
            assert not server.ResidentBucket.eligible_lstm(det, smoothing=True)
        window = {"smoothing": True} if kfcv else {}
        assert server.ResidentBucket.eligible(bare, target_scaler=True, **window)
        assert not server.ResidentBucket.eligible(piped, target_scaler=True, **window)  # a Pipeline needs input_scalers=True, as before
        assert server.ResidentBucket.eligible(piped, input_scalers=True, target_scaler=True, **window)
    assert not server.ResidentBucket.eligible(_det(_ttr(_ae()), True), target_scaler=True)  # a window needs smoothing=True, as before


def test_refused_forms(lib):
    from sklearn.preprocessing import MaxAbsScaler, MinMaxScaler, RobustScaler, StandardScaler

    from gordo_components_b200.machine.model.models import KerasAutoEncoder

    refused = {
        "LSTM regressor": _ttr(_lstm()),
        "LSTM Pipeline": _ttr(_piped(_lstm())),
        "StandardScaler transformer": _ttr(_ae(), StandardScaler()),
        "RobustScaler transformer": _ttr(_ae(), RobustScaler()),
        "StandardScaler input": _ttr(_piped(_ae(), StandardScaler())),
        "RobustScaler input": _ttr(_piped(_ae(), RobustScaler())),
        "MaxAbsScaler input": _ttr(_piped(_ae(), MaxAbsScaler())),
        "clipping input": _ttr(_piped(_ae(), MinMaxScaler(clip=True))),
        "two input scalers": _ttr(_piped(_ae(), MinMaxScaler(), MinMaxScaler())),
        "func": _ttr(_ae(), transformer=None, func=np.log1p, inverse_func=np.expm1),
        "not fitted": _ttr(_ae(), fitted=False),
        "AE without weights": _ttr(KerasAutoEncoder(kind="feedforward_hourglass")),
    }
    for why, est in refused.items():
        for kfcv in (False, True):
            assert not server.ResidentBucket.eligible(_det(est, kfcv), **ALL_FLAGS), why
    # a TTR fitted on a 1-D target predicts 1-D: its reply shape is the per-request route's business
    one_d = _ttr(_ae())
    one_d._training_dim = 1
    assert not server.ResidentBucket.eligible(_det(one_d), **ALL_FLAGS)
    # a transformer fitted on another number of targets than the network predicts
    wide = _ttr(_ae())
    wide.transformer_ = MinMaxScaler().fit(np.random.default_rng(0).random((8, T + 1)))
    assert not server.ResidentBucket.eligible(_det(wide), **ALL_FLAGS)


def test_func_without_transformer_is_refused(lib):
    from sklearn.compose import TransformedTargetRegressor

    ttr = TransformedTargetRegressor(regressor=_ae(), func=np.log1p, inverse_func=np.expm1)
    ttr._training_dim, ttr.regressor_ = 2, ttr.regressor
    from sklearn.preprocessing import FunctionTransformer

    ttr.transformer_ = FunctionTransformer(func=np.log1p, inverse_func=np.expm1)
    assert not server.ResidentBucket.eligible(_det(ttr), **ALL_FLAGS)


def test_target_minmax_attributes(lib):
    ttr = _ttr(_piped(_ae()))
    scale, mn = server._target_minmax(_det(ttr))
    assert scale.dtype == mn.dtype == np.float64
    assert np.array_equal(scale, ttr.transformer_.scale_) and np.array_equal(mn, ttr.transformer_.min_)
    assert server._target_minmax(_det(_ae())) is None
    assert server._target_minmax(_det(_piped(_ae()))) is None


def test_target_scaler_models_get_a_group_of_their_own(lib):
    models = {
        "plain": _det(_ae()), "piped": _det(_piped(_ae())),
        "ttr": _det(_ttr(_ae())), "ttr-b": _det(_ttr(_ae())),
        "ttr-piped": _det(_ttr(_piped(_ae()))),
        "ttr-kfcv": _det(_ttr(_piped(_ae())), kfcv=True), "ttr-kfcv-b": _det(_ttr(_piped(_ae())), kfcv=True),
        "kfcv": _det(_piped(_ae()), kfcv=True),
        "ttr-lstm": _det(_ttr(_lstm())),
    }
    groups = server.ResidentBucket.ff_groups(models, **ALL_FLAGS)
    assert sorted(map(sorted, groups.values())) == [["kfcv"], ["piped"], ["plain"], ["ttr", "ttr-b"], ["ttr-kfcv", "ttr-kfcv-b"], ["ttr-piped"]]
    by_name = {n: k for k, names in groups.items() for n in names}
    assert by_name["ttr-kfcv"][5] is True and by_name["kfcv"][5] is False  # the flag; everything else of the key is the same
    assert by_name["ttr-kfcv"][:5] == by_name["kfcv"][:5] and by_name["ttr-kfcv"][6:] == by_name["kfcv"][6:]
    assert by_name["ttr-kfcv"][-1] == (144, "smm")
    # without the flag the groups are what they were
    assert sorted(map(sorted, server.ResidentBucket.ff_groups(models, input_scalers=True, smoothing=True).values())) == [["kfcv"], ["piped"], ["plain"]]
    assert list(server.ResidentBucket.ff_groups(models).values()) == [["plain"]]
    assert server.ResidentBucket.lstm_groups(models, smoothing=True) == {}
