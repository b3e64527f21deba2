"""
Host side of the input-scaler mode of the fused predict+score launch: the plan query and argument checks of
gb_ffae_infer_score_x64, and which models ``server.ResidentBucket(input_scalers=...)`` serves and how it groups them.  No GPU.
"""
import ctypes as C

import numpy as np
import pandas as pd
import pytest

from gordo_components_b200 import _cabi, serializer, server
from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
from gordo_components_b200.machine.model.models import KerasAutoEncoder

GB_E_ARG, GB_E_SHAPE = -1, -2


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def _hourglass(T):
    from gordo_components_b200.machine.model.factories.feedforward_autoencoder import feedforward_hourglass

    spec = feedforward_hourglass(T)
    return _cabi.make_ffnet(spec.dims, spec.acts, spec.l1)


def _plan(lib, net, variant):
    kernel, nwg = C.c_int32(-1), C.c_int32(-1)
    rc = lib.gb_ffae_infer_plan_x64(C.byref(net), variant, C.byref(kernel), C.byref(nwg))
    return rc, kernel.value, nwg.value


def test_plan_query(lib):
    # feedforward_hourglass(64): 90 KB of weights leave room for two warpgroups' float64 x tiles, not three
    assert _plan(lib, _hourglass(64), 0) == (0, 2, 2)
    assert _plan(lib, _hourglass(64), 2) == (0, 2, 2)
    assert _plan(lib, _hourglass(24), 0) == (0, 2, 3)
    assert _plan(lib, _hourglass(64), 1)[:2] == (0, 1)
    assert _plan(lib, _hourglass(8), 0)[:2] == (0, 3)
    assert _plan(lib, _hourglass(100), 0)[:2] == (0, 1)
    assert _plan(lib, _hourglass(100), 2)[0] == GB_E_SHAPE
    assert _plan(lib, _hourglass(100), 3)[0] == GB_E_SHAPE
    assert _plan(lib, _hourglass(64), 4)[0] == GB_E_ARG
    assert _plan(lib, _hourglass(64), 0x100)[0] == GB_E_ARG
    assert lib.gb_ffae_infer_plan_x64(C.byref(_hourglass(64)), 0, None, None) == 0


def test_entry_point_argument_checks(lib):
    net = _hourglass(64)
    fake = C.c_void_p(1 << 20)  # aligned and never dereferenced: every call below is refused before it touches the device

    def call(x_scale, x_offset, variant):
        return lib.gb_ffae_infer_score_x64(C.byref(net), fake, fake, 1, 10, 10, 10, fake, x_scale, x_offset, None, None, None, None, fake,
                                           None, None, None, None, None, None, variant, None)

    assert call(None, fake, 0) == GB_E_ARG and b"x_scale/x_offset" in lib.gb_last_error()
    assert call(fake, None, 0) == GB_E_ARG and b"x_scale/x_offset" in lib.gb_last_error()
    assert call(fake, fake, 4) == GB_E_ARG and b"variant" in lib.gb_last_error()
    assert call(fake, fake, 2 | 0x100) == GB_E_ARG and b"low byte" in lib.gb_last_error()
    assert call(fake, fake, 3) == GB_E_SHAPE


T = 4
TAGS = [f"tag-{i}" for i in range(T)]


def _detector(pre=(), thresholds=True):
    from sklearn.pipeline import Pipeline

    ae = KerasAutoEncoder(kind="feedforward_hourglass")
    ae.kwargs.update({"n_features": T, "n_features_out": T})
    ae._prepare_model()
    base = Pipeline([(f"s{i}", s) for i, s in enumerate(pre)] + [("ae", ae)]) if pre else ae
    det = DiffBasedAnomalyDetector(base_estimator=base, require_thresholds=thresholds)
    rng = np.random.default_rng(len(pre))
    for s in pre:
        s.fit(rng.random((8, T)) * 100)
    det.scaler.fit(rng.random((8, T)))
    if thresholds:
        det.feature_thresholds_, det.aggregate_threshold_ = pd.Series(np.ones(T), index=TAGS), 0.5
    return det


def test_eligibility():
    from sklearn.decomposition import PCA
    from sklearn.preprocessing import MaxAbsScaler, MinMaxScaler, RobustScaler, StandardScaler

    bare = _detector()
    assert server.ResidentBucket.eligible(bare) and server.ResidentBucket.eligible(bare, input_scalers=True)
    for pre in ([MinMaxScaler()], [StandardScaler()], [RobustScaler()], [MaxAbsScaler()], [MinMaxScaler(), StandardScaler()]):
        det = _detector(pre)
        assert not server.ResidentBucket.eligible(det)  # the default: bare auto-encoders only
        assert server.ResidentBucket.eligible(det, input_scalers=True)
    assert not server.ResidentBucket.eligible(_detector([MinMaxScaler(clip=True)]), input_scalers=True)  # not affine
    assert not server.ResidentBucket.eligible(_detector([PCA(n_components=T)]), input_scalers=True)
    det = _detector([MinMaxScaler()])
    det.window = 6
    assert not server.ResidentBucket.eligible(det, input_scalers=True)  # smoothing stays on the per-request route
    det = _detector([MinMaxScaler()], thresholds=True)
    del det.feature_thresholds_, det.aggregate_threshold_
    assert not server.ResidentBucket.eligible(det, input_scalers=True)  # thresholds the model requires are missing
    det = _detector([MinMaxScaler()])
    det.base_estimator.steps[-1][1].model = None
    assert not server.ResidentBucket.eligible(det, input_scalers=True)


class _FakeEngine:
    def __init__(self, spec):
        self.n_in, self.n_out, self.device = spec.dims[0], spec.dims[-1], "cpu"

    def pack_params(self, weights):
        import torch

        return torch.zeros((len(weights), 4))


@pytest.fixture()
def mixed_store(tmp_path, monkeypatch):
    """Two bare detectors and three behind input scalers; the bucket's device side replaced by stand-ins that record what they get."""
    from sklearn.preprocessing import MinMaxScaler, StandardScaler

    from gordo_components_b200 import engine, serving

    dets = {"bare-1": _detector(), "bare-2": _detector(), "pipe-1": _detector([MinMaxScaler()]), "pipe-2": _detector([StandardScaler()]),
            "pipe-3": _detector([MinMaxScaler(), StandardScaler()])}
    for name, det in dets.items():
        serializer.dump(det, str(tmp_path / name), metadata={"name": name, "dataset": {"tag_list": TAGS}})
    made = []

    class FakeCoalescer:
        def __init__(self, eng, params, scale, feat_thr, agg_thr, **kwargs):
            self.params, self.kwargs = params, kwargs
            made.append(self)

    monkeypatch.setattr(engine, "ff_engine_for", _FakeEngine)
    monkeypatch.setattr(serving, "AnomalyCoalescer", FakeCoalescer)
    return server.ModelStore(str(tmp_path)), made


def test_grouping(mixed_store):
    from gordo_components_b200.machine.model.anomaly.diff import _compose_affine

    store, made = mixed_store
    default = server.ResidentBucket(store)
    assert default.names == ["bare-1", "bare-2"] and not default.input_scalers  # exactly what it held before
    assert "x_scale" not in made[-1].kwargs and "x_offset" not in made[-1].kwargs
    pipes = server.ResidentBucket(store, input_scalers=True, max_wait_ms=5.0)
    assert pipes.names == ["pipe-1", "pipe-2", "pipe-3"] and pipes.input_scalers and pipes.slot["pipe-3"] == 2
    kw = made[-1].kwargs
    assert kw["max_wait_ms"] == 5.0 and kw["x_scale"].dtype == kw["x_offset"].dtype == __import__("torch").float64
    for i, name in enumerate(pipes.names):
        pre = [s for _, s in store.model(name).base_estimator.steps[:-1]]
        a, b = _compose_affine(pre, T)
        np.testing.assert_array_equal(kw["x_scale"][i].numpy(), a)
        np.testing.assert_array_equal(kw["x_offset"][i].numpy(), b)
    # the bare group wins a store where it is the larger one, input scalers or not: bare and Pipeline models never share a bucket
    assert server.ResidentBucket(store, names=["bare-1", "bare-2", "pipe-1"], input_scalers=True).names == ["bare-1", "bare-2"]
    with pytest.raises(ValueError, match="no model"):
        server.ResidentBucket(store, names=["pipe-1", "pipe-2"])


def test_inf_in_x_is_refused_before_any_launch(mixed_store):
    store, _ = mixed_store
    bucket = server.ResidentBucket(store, input_scalers=True)

    class NoLaunch:
        def anomaly(self, *a):
            raise AssertionError("launched")

    bucket.coalescer = NoLaunch()
    X = pd.DataFrame(np.ones((3, T)), columns=TAGS)
    X.iloc[1, 2] = -np.inf
    with pytest.raises(ValueError, match="infinity"):
        bucket.anomaly_blocks(store, "pipe-1", X, X.abs().clip(upper=1.0))
