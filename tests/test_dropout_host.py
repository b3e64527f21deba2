"""
Dropout layers of KerasRawModelRegressor specs without a GPU: the translation of every placement and spelling into
``FFNetSpec.dropout``, every refusal and its message, the serializer, clone and pickle round trips, the bucket keys, the fleet
builder's and the serving bucket's classification, the argument checks of gb_ffae_fit_drop, and the statistics of the mask
generator the header documents (restated in tests/dropout_oracle.py).
"""
import ctypes as C
import pickle

import numpy as np
import pandas as pd
import pytest
from sklearn.base import clone

import dropout_oracle as do
from gordo_components_b200 import _cabi, builder, serializer, server
from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
from gordo_components_b200.machine.model.factories.raw import raw_spec
from gordo_components_b200.machine.model.factories.specs import FFNetSpec, dropout_key, fit_dropout
from gordo_components_b200.machine.model.models import KerasRawModelRegressor

TF = "tensorflow.keras."


def dense(units, prefix=TF, **kw):
    return {prefix + "layers.Dense": {"units": units, **kw}}


def drop(rate, prefix=TF, **kw):
    return {prefix + "layers.Dropout": {"rate": rate, **kw}}


def kind(*layers, prefix=TF):
    return {"spec": {prefix + "models.Sequential": {"layers": list(layers)}}, "compile": {"loss": "mse", "optimizer": "adam"}}


# ------------------------------------------------------------------------------------------------ translation
def test_hidden_and_input_dropout_become_the_rates_of_the_next_layer():
    s = raw_spec(kind(dense(6, activation="tanh"), drop(0.3), dense(3, activation="tanh"), drop(0.5, seed=7, name="d2"), dense(4)), 4, 4)
    assert s.dims == [4, 6, 3, 4] and s.dropout == [0.0, 0.3, 0.5]
    assert fit_dropout(s) == [0.0, 0.3, 0.5]
    s = raw_spec(kind({TF + "layers.Input": {"shape": [4]}}, drop(0.2), dense(3), dense(4)), None)
    assert s.dims == [4, 3, 4] and s.dropout == [0.2, 0.0]
    s = raw_spec(kind(drop(0.25, input_shape=[5]), dense(3), drop(0.1), dense(5)), None)
    assert s.dims == [5, 3, 5] and s.dropout == [0.25, 0.1]
    s = raw_spec(kind(drop(0.25), dense(3, input_shape=[5]), dense(5)), None)  # the first Dense layer still takes the input shape
    assert s.dims == [5, 3, 5] and s.dropout == [0.25, 0.0]


@pytest.mark.parametrize("prefix", [TF, "keras.", "", "layers-only"])
def test_every_spelling_of_dropout_is_taken(prefix):
    if prefix == "layers-only":
        layers = [{"Dense": {"units": 3}}, {"Dropout": {"rate": 0.4}}, {"Dense": {"units": 4}}]
        k = {"spec": {"Sequential": {"layers": layers}}, "compile": {}}
    else:
        k = kind(dense(3, prefix=prefix), drop(0.4, prefix=prefix), dense(4, prefix=prefix), prefix=prefix)
    assert raw_spec(k, 4).dropout == [0.0, 0.4]


def test_a_rate_of_zero_is_the_identity():
    s = raw_spec(kind(drop(0.0), dense(3), drop(0), dense(4)), 4)
    assert s.dropout is None and fit_dropout(s) is None and dropout_key(s) == ()
    assert s == raw_spec(kind(dense(3), dense(4)), 4)


@pytest.mark.parametrize("layers, message", [
    ([dense(4), drop(0.1)], r"layer 1 'tensorflow.keras.layers.Dropout' after the last Dense layer is not supported"),
    ([dense(4), drop(0.0)], r"layer 1 .*Dropout.* after the last Dense layer is not supported"),
    ([dense(3), drop(0.1), drop(0.2), dense(4)], r"layer 2 .*Dropout.* two Dropout layers in a row"),
    ([drop(0.1), drop(0.2), dense(4)], r"two Dropout layers in a row"),
    ([dense(3, activity_regularizer="l1"), drop(0.2), dense(4)], r"layer 1 .*Dropout.* after a Dense layer with an activity_regularizer"),
    ([dense(3), drop(1.0), dense(4)], r"rate=1.0 must be a finite float in \[0, 1\)"),
    ([dense(3), drop(-0.1), dense(4)], r"rate=-0.1 must be"),
    ([dense(3), drop(float("nan")), dense(4)], r"rate=nan must be"),
    ([dense(3), drop("0.1"), dense(4)], r"rate='0.1' must be"),
    ([dense(3), drop(True), dense(4)], r"rate=True must be"),
    ([dense(3), {TF + "layers.Dropout": {}}, dense(4)], r"rate=None must be"),
    ([dense(3), drop(0.1, noise_shape=[None, 1]), dense(4)], r"noise_shape is not supported"),
    ([dense(3), drop(0.1, training=True), dense(4)], r"unsupported arguments \['training'\]"),
    ([dense(3), drop(0.1, input_shape=[4]), dense(4)], r"input_shape is only taken on the first layer"),
    ([dense(3), drop(0.1, seed="x"), dense(4)], r"seed='x' must be an int"),
])
def test_what_the_fit_kernel_does_not_run_is_refused(layers, message):
    with pytest.raises(ValueError, match=message) as e:
        raw_spec(kind(*layers), 4)
    if "after the last" in message or "in a row" in message or "activity" in message:
        assert "layers.Dropout (rate, seed, name" in str(e.value)  # the message names what is supported


def test_an_activity_regularizer_before_a_rate_of_zero_is_taken():
    s = raw_spec(kind(dense(3, activity_regularizer="l1"), drop(0.0), dense(4)), 4)
    assert s.l1 == [0.01, 0.0] and s.dropout is None


# ------------------------------------------------------------------------------------------------ round trips and keys
DEFINITION = kind(dense(4, activation="tanh", input_shape=[4]), drop(0.3, seed=3), dense(1))


def _constructed(k, n_in=4, n_out=1):
    m = KerasRawModelRegressor(k)
    m.kwargs.update({"n_features": n_in, "n_features_out": n_out})
    m._prepare_model()
    return m


def test_serializer_clone_and_pickle_round_trips():
    definition = {"gordo.machine.model.models.KerasRawModelRegressor": {"kind": DEFINITION, "epochs": 2}}
    model = serializer.from_definition(definition)
    assert type(model) is KerasRawModelRegressor and model.kind == DEFINITION
    again = serializer.from_definition(serializer.into_definition(model))
    assert again.kind == DEFINITION and again.kwargs == {"epochs": 2}
    c = clone(model)
    assert c.kind == DEFINITION and c.kind is not model.kind
    built = _constructed(DEFINITION)
    assert built.model.spec.dropout == [0.0, 0.3]
    p = pickle.loads(pickle.dumps(built))
    assert p.model.spec == built.model.spec and p.model.spec.dropout == [0.0, 0.3]


def test_specs_pickled_before_the_dropout_field_load_without_it():
    s = FFNetSpec([4, 3, 4], ["tanh", "linear"], [0.0, 0.0])
    state = dict(s.__dict__)
    state.pop("dropout")
    old = FFNetSpec.__new__(FFNetSpec)
    old.__dict__.update(state)
    assert old.dropout is None and fit_dropout(old) is None and dropout_key(old) == ()
    old = pickle.loads(pickle.dumps(old))
    assert fit_dropout(old) is None


def test_bucket_keys_are_unchanged_without_dropout_and_separated_by_rate():
    assert dropout_key(FFNetSpec([4, 3, 4], ["tanh", "linear"], [0.0, 0.0], dropout=[0.0, 0.0])) == ()
    assert dropout_key(FFNetSpec([4, 3, 4], ["tanh", "linear"], [0.0, 0.0], dropout=[0.0, 0.5])) == (("dropout", (0.0, 0.5)),)
    plain = kind(dense(3, activation="tanh"), dense(4))
    a = builder._canonical(0, _raw_machine("a", plain))
    b = builder._canonical(1, _raw_machine("b", kind(dense(3, activation="tanh"), drop(0.2), dense(4))))
    b2 = builder._canonical(2, _raw_machine("b2", kind(dense(3, activation="tanh"), drop(0.2), dense(4))))
    c = builder._canonical(3, _raw_machine("c", kind(dense(3, activation="tanh"), drop(0.4), dense(4))))
    d = builder._canonical(4, _raw_machine("d", kind(drop(0.2), dense(3, activation="tanh"), dense(4))))
    assert None not in (a, b, b2, c, d)
    assert b.bucket() == b2.bucket()
    assert len({a.bucket(), b.bucket(), c.bucket(), d.bucket()}) == 4
    assert b.bucket()[:-1] == a.bucket() and b.bucket()[-1] == ("dropout", (0.0, 0.2))
    assert d.bucket()[-1] == ("dropout", (0.2, 0.0))


# ------------------------------------------------------------------------------------------------ fleet builder and serving
def _frame(rows=200, tags=4, seed=0):
    rng = np.random.default_rng(seed)
    idx = pd.date_range("2020-01-01", periods=rows, freq="10min", tz="UTC")
    return pd.DataFrame(rng.random((rows, tags)).astype(np.float32), index=idx, columns=[f"TAG {i}" for i in range(tags)])


def _raw_machine(name, k, scaled=False, epochs=2):
    est = {"gordo.machine.model.models.KerasRawModelRegressor": {"kind": k, "epochs": epochs}}
    if scaled:
        est = {"sklearn.pipeline.Pipeline": {"steps": ["sklearn.preprocessing.MinMaxScaler", est]}}
    X = _frame()
    return {"name": name, "model": {"gordo.machine.model.anomaly.diff.DiffBasedAnomalyDetector": {"base_estimator": est}},
            "dataset": {"X": X, "y": X}}


def test_the_fleet_builder_takes_dropout_detectors_bare_and_scaled():
    k = kind(dense(3, activation="tanh", kernel_regularizer="l2"), drop(0.3), dense(4))
    a, s = builder._canonical(0, _raw_machine("a", k)), builder._canonical(1, _raw_machine("s", k, scaled=True))
    assert a is not None and s is not None and s.input_scaler and not a.input_scaler
    assert a.spec.dropout == [0.0, 0.3] and a.bucket() != s.bucket()
    assert a.bucket()[-2:] == (("reg", (0.0, 0.0), (0.01, 0.0), (0.0, 0.0), (0.0, 0.0)), ("dropout", (0.0, 0.3)))


def test_a_dropout_detector_is_served_as_any_raw_detector():
    k = kind(dense(5, activation="tanh"), drop(0.5), dense(4))
    det = DiffBasedAnomalyDetector(base_estimator=KerasRawModelRegressor(k))
    det.base_estimator.kwargs.update({"n_features": 4, "n_features_out": 4})
    det.base_estimator._prepare_model()
    det.feature_thresholds_, det.aggregate_threshold_ = pd.Series(np.ones(4)), 0.5
    det.scaler.fit(np.random.default_rng(0).random((8, 4)))
    assert server.ResidentBucket.eligible(det)
    assert server._served_parts(det) == ([], det.base_estimator)


# ------------------------------------------------------------------------------------------------ the C entry point
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def test_the_entry_point_is_exported(lib):
    assert "gb_ffae_fit_drop" in _cabi.EXPORTS and hasattr(lib, "gb_ffae_fit_drop")
    assert C.sizeof(_cabi.GbDenseDropout) == 4 * _cabi.GB_MAX_LAYERS
    r = _cabi.make_dense_dropout([0.0, 0.25])
    assert list(r.rate[:3]) == [0.0, 0.25, 0.0]
    with pytest.raises(ValueError):
        _cabi.make_dense_dropout([0.1] * (_cabi.GB_MAX_LAYERS + 1))


def _call(lib, rates, dims=(4, 3, 4), l1=None):
    net = _cabi.make_ffnet(list(dims), ["tanh"] * (len(dims) - 2) + ["linear"], l1)
    hp = _cabi.GbFitHParams(epochs=1, batch_size=8, shuffle=0, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7)
    rec = _cabi.make_dense_dropout(rates)
    fake = C.c_void_p(16)  # never dereferenced: validation refuses first
    return lib.gb_ffae_fit_drop(C.byref(net), fake, fake, fake, fake, None, 1, 8, fake, fake, None, None, C.byref(hp), 8, fake, fake,
                                None, None, None, None, None, None, None, None, C.byref(rec), None)


@pytest.mark.parametrize("rates, where", [
    ([0.0, -0.1], b"dropout rate[1]"), ([0.0, 1.0], b"dropout rate[1]"), ([float("nan")], b"dropout rate[0]"),
    ([0.0, float("inf")], b"dropout rate[1]"), ([0.0, 0.0, 0.2], b"dropout rate[2]"), ([0.0] * 15 + [0.5], b"dropout rate[15]"),
])
def test_a_bad_rate_is_refused_without_a_gpu(lib, rates, where):
    """The record is checked before anything touches a device: GB_E_ARG on a GPU-less host, the message naming the layer."""
    rc = _call(lib, rates)
    assert rc == -1 and where in lib.gb_last_error()
    with pytest.raises(ValueError):
        _cabi.check(rc)


def test_dropout_after_an_activity_l1_is_refused_without_a_gpu(lib):
    assert _call(lib, [0.0, 0.3], l1=[0.01, 0.0]) == -1 and b"activity L1" in lib.gb_last_error()


def test_the_memory_plan_does_not_depend_on_a_record(lib):
    """gb_ffae_fit_plan takes no record: the DROP kernels run in the plans the others do (masks are recomputed, never stored)."""
    assert lib.gb_ffae_fit_plan.argtypes == [C.POINTER(_cabi.GbFFNet), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    for dims in ([64, 32, 16, 32, 64], [10, 256, 128, 64, 128, 256, 10], [128, 256, 128, 64, 128, 256, 128]):
        net = _cabi.make_ffnet(dims, ["tanh"] * (len(dims) - 2) + ["linear"])
        w, d = C.c_int32(-1), C.c_int32(-1)
        assert lib.gb_ffae_fit_plan(C.byref(net), C.byref(w), C.byref(d)) == 0


def test_dropout_kernels_static_shared_memory_fits_the_reserve(lib):
    """The nine dropout kernels live in an object of their own (ffae_fit_drop.o) and, as every fit kernel, must leave the plans'
    dynamic shared memory its 227 KB: their static arrays stay within the 2 KB reserve (FIT_STATIC_SMEM in csrc/ffae_fit.cu)."""
    import os
    import re
    import subprocess

    from gordo_components_b200.csrc import build

    obj = os.path.join(build.OBJ, "ffae_fit_drop.o")
    tool = os.path.join(os.path.dirname(build._nvcc()), "cuobjdump")
    out = subprocess.run([tool, "-res-usage", obj], capture_output=True, text=True, check=True).stdout
    sizes = [int(v) for v in re.findall(r"SHARED:(\d+)", out)]
    assert len(sizes) == 9 and out.count("ffae_fit_drop_kernel") >= 9, "one entry per dropout kernel instantiation"
    assert max(sizes) <= 2048, sorted(set(sizes))


# ------------------------------------------------------------------------------------------------ the mask generator
@pytest.mark.parametrize("rate", [0.05, 0.1, 0.25, 0.5, 0.9])
def test_the_keep_fraction_is_one_minus_the_rate(rate):
    """10^6 draws (1000 steps x 20 positions x 50 units): the kept share within 5 sigma of 1 - rate."""
    n = 0
    kept = 0
    for t in range(1, 1001):
        m = do.keep_mask(seed=12345, slot=3, t=t, n_rows=20, layer=1, units=50, rate=rate)
        kept += int(m.sum())
        n += m.size
    assert n == 10**6
    p = 1.0 - rate
    assert abs(kept / n - p) <= 5 * np.sqrt(p * (1 - p) / n)


def test_masks_differ_across_step_position_layer_unit_and_job():
    base = do.words(7, 0, 5, np.arange(32), 1, 64)
    for other in (do.words(7, 0, 6, np.arange(32), 1, 64), do.words(7, 0, 5, np.arange(32), 2, 64), do.words(7, 1, 5, np.arange(32), 1, 64),
                  do.words(8, 0, 5, np.arange(32), 1, 64)):
        assert (other != base).mean() > 0.99
    assert len(np.unique(base)) > 0.99 * base.size  # positions and units: distinct words within one step and layer
    m = base >= do.threshold(0.5)
    assert 0.4 < m.mean() < 0.6 and len({tuple(r) for r in m}) == 32 and len({tuple(c) for c in m.T}) == 64


def test_threshold_and_scale_follow_the_header():
    assert do.threshold(0.5) == 2**31 and do.threshold(0.0) == 0
    assert do.threshold(0.1) == int(np.floor(float(np.float32(0.1)) * 2**32))
    assert do.scale(0.5) == 2.0 and np.float32(do.scale(0.1)) == np.float32(1 / (1 - float(np.float32(0.1))))
    # mix32 is the lowbias32 finalizer the fit kernels share
    assert int(do.mix32(0)) == 0 and int(do.mix32(1)) != 1
