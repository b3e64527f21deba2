"""
KerasRawModelRegressor without a GPU: a raw ``Sequential`` definition into the Dense spec (widths, activations, activity L1 and
weight regularizer coefficients), every refusal and its message, the regularizer names and defaults, the serializer and pickle
round trips, the fleet builder's and the serving bucket's classification, and the argument checks of gb_ffae_fit_reg.
"""
import ctypes as C
import math
import pickle

import numpy as np
import pandas as pd
import pytest
import yaml
from sklearn.base import clone

from gordo_components_b200 import _cabi, builder, serializer, server
from gordo_components_b200.machine.model.anomaly.diff import DiffBasedAnomalyDetector
from gordo_components_b200.machine.model.factories.raw import raw_spec, resolve_regularizer
from gordo_components_b200.machine.model.factories.specs import FFNetSpec, fit_reg, reg_key
from gordo_components_b200.machine.model.models import KerasAutoEncoder, KerasRawModelRegressor

TF = "tensorflow.keras."


def dense(units, **kw):
    return {TF + "layers.Dense": {"units": units, **kw}}


def kind(*layers, compile=None, container=TF + "models.Sequential"):
    return {"spec": {container: {"layers": list(layers)}}, "compile": {"loss": "mse", "optimizer": "adam"} if compile is None else compile}


def spec_of(k, n_features=4, n_features_out=None):
    return raw_spec(k, n_features, n_features_out)


# ------------------------------------------------------------------------------------------------ translation
def test_a_dense_stack_becomes_its_spec():
    k = kind(dense(6, activation="tanh", input_shape=[5], kernel_regularizer={TF + "regularizers.L1L2": {"l1": 0.2, "l2": 0.05}},
                   activity_regularizer={TF + "regularizers.L1": {"l1": 1e-4}}),
             dense(3, activation="relu", bias_regularizer="l2", name="middle"),
             dense(5, activation=None, kernel_regularizer={"keras.regularizers.L2": {"l2": 0.3}}))
    s = spec_of(k, 5, 5)
    assert isinstance(s, FFNetSpec)
    assert s.dims == [5, 6, 3, 5] and s.acts == ["tanh", "relu", "linear"] and s.l1 == [1e-4, 0.0, 0.0]
    assert s.kernel_l1 == [0.2, 0.0, 0.0] and s.kernel_l2 == [0.05, 0.0, 0.3]
    assert s.bias_l1 == [0.0, 0.0, 0.0] and s.bias_l2 == [0.0, 0.01, 0.0]
    assert s.loss == "mse" and s.metrics == [] and s.optimizer_config is None
    assert fit_reg(s) == {"kernel_l1": [0.2, 0.0, 0.0], "kernel_l2": [0.05, 0.0, 0.3], "bias_l1": [0.0] * 3, "bias_l2": [0.0, 0.01, 0.0]}


def test_every_spelling_of_the_container_and_layers_is_taken():
    for container, layer, inp in (("tensorflow.keras.models.Sequential", "tensorflow.keras.layers.Dense", "tensorflow.keras.layers.Input"),
                                  ("keras.models.Sequential", "keras.layers.Dense", "keras.layers.InputLayer"),
                                  ("models.Sequential", "layers.Dense", "layers.Input"), ("Sequential", "Dense", "Input")):
        shape = {"shape": [3]}
        k = {"spec": {container: {"layers": [{inp: shape}, {layer: {"units": 2}}, {layer: {"units": 3}}]}}, "compile": {}}
        s = spec_of(k, 3, 3)
        assert s.dims == [3, 2, 3] and s.acts == ["linear", "linear"]
    assert spec_of(kind({TF + "layers.InputLayer": {"batch_shape": [None, 4]}}, dense(4)), 4).dims == [4, 4]
    assert spec_of(kind(dense(2, input_dim=4), dense(4)), 4).dims == [4, 2, 4]


def test_the_input_width_comes_from_the_data_when_the_spec_has_none():
    assert spec_of(kind(dense(10), dense(32), dense(1)), 7, 1).dims == [7, 10, 32, 1]
    with pytest.raises(ValueError, match="no input shape"):
        spec_of(kind(dense(3)), None)


def test_compile_arguments():
    s = spec_of(kind(dense(4), compile={"loss": "mean_absolute_error", "optimizer": {TF + "optimizers.RMSprop": {"learning_rate": 0.01}},
                                        "metrics": ["accuracy"], "run_eagerly": True, "jit_compile": False, "steps_per_execution": 4}))
    assert s.loss == "mae" and s.metrics == ["accuracy"] and s.optimizer == "rmsprop" and s.optimizer_config["lr"] == 0.01
    assert spec_of(kind(dense(4), compile={"optimizer": "Adam"})).optimizer_config is None  # plain Adam keeps the Adam kernels
    assert spec_of(kind(dense(4), compile={"loss": "mse"})).optimizer == "rmsprop"  # Model.compile's default optimizer
    nadam = spec_of(kind(dense(4), compile={"optimizer": {"keras.optimizers.Nadam": {"clipvalue": 0.5}}}))
    assert nadam.optimizer == "nadam" and nadam.optimizer_config["clipvalue"] == 0.5


def test_regularizer_names_and_defaults():
    assert resolve_regularizer(None) == (0.0, 0.0)
    assert resolve_regularizer("l1") == (0.01, 0.0) and resolve_regularizer("L1") == (0.01, 0.0)
    assert resolve_regularizer("l2") == (0.0, 0.01) and resolve_regularizer("L2") == (0.0, 0.01)
    assert resolve_regularizer("l1_l2") == (0.0, 0.0) and resolve_regularizer("L1L2") == (0.0, 0.0)
    assert resolve_regularizer({TF + "regularizers.L1": None}) == (0.01, 0.0)
    assert resolve_regularizer({TF + "regularizers.L2": {}}) == (0.0, 0.01)
    assert resolve_regularizer({TF + "regularizers.L1L2": {"l2": 0.5}}) == (0.0, 0.5)
    assert resolve_regularizer({"keras.regularizers.l1_l2": {"l1": 0.1, "l2": 0.2}}) == (0.1, 0.2)
    assert resolve_regularizer({"regularizers.L1": {"l1": 3}}) == (3.0, 0.0)
    assert resolve_regularizer(TF + "regularizers.L2") == (0.0, 0.01)


@pytest.mark.parametrize("bad, message", [
    ({TF + "regularizers.OrthogonalRegularizer": {}}, "implements the regularizers L1, L2 and L1L2"),
    ("l3", "implements the regularizers L1, L2 and L1L2"),
    ({TF + "regularizers.L1": {"l2": 0.1}}, r"unsupported arguments \['l2'\]"),
    ({TF + "regularizers.L1": {"l1": -0.1}}, "must be a finite float >= 0"),
    ({TF + "regularizers.L2": {"l2": float("nan")}}, "must be a finite float >= 0"),
    ({TF + "regularizers.L1L2": {"l1": "big"}}, "must be a finite float >= 0"),
])
def test_bad_regularizers_are_refused(bad, message):
    with pytest.raises(ValueError, match=message):
        resolve_regularizer(bad)
    with pytest.raises(ValueError, match=message):
        spec_of(kind(dense(4, kernel_regularizer=bad)))


@pytest.mark.parametrize("k, message", [
    (kind({TF + "layers.Input": {"shape": [9]}}, {TF + "layers.Reshape": {"target_shape": [3, 3]}}, {TF + "layers.LSTM": {"units": 12}},
          TF + "layers.Flatten", dense(1)), "layer 1 'tensorflow.keras.layers.Reshape' is not supported"),
    (kind(dense(4), {TF + "layers.Dropout": {"rate": 0.1}}), "layer 1 .*Dropout.* is not supported"),
    (kind(dense(4), TF + "layers.BatchNormalization"), "BatchNormalization.* is not supported"),
    (kind(TF + "layers.Flatten", dense(4)), "Flatten.* is not supported"),
    (kind(dense(4, use_bias=False)), "use_bias=False is not supported"),
    (kind(dense(4, kernel_initializer="he_normal")), "kernel_initializer 'he_normal' is not supported"),
    (kind(dense(4, bias_initializer="ones")), "bias_initializer 'ones' is not supported"),
    (kind(dense(4, kernel_constraint="non_neg")), "kernel_constraint is not supported"),
    (kind(dense(4, activity_regularizer="l2")), "L2 activity_regularizer is not supported"),
    (kind(dense(4, activity_regularizer={TF + "regularizers.L1L2": {"l1": 0.1, "l2": 0.1}})), "L2 activity_regularizer"),
    (kind(dense(4, activation="softmax")), "activation 'softmax' is not supported"),
    (kind(dense(4, dtype="float64")), r"unsupported arguments \['dtype'\]"),
    (kind(dense(0)), r"units=0 must be an int in \[1, 256\]"),
    (kind(dense(300)), r"units=300 must be an int in \[1, 256\]"),
    (kind(dense(4), dense(4, input_shape=[4])), "only taken on the first layer"),
    (kind(dense(4), {TF + "layers.Input": {"shape": [4]}}), "must come first"),
    (kind({TF + "layers.Input": {"shape": [2, 2]}}, dense(4)), "one-dimensional rows"),
    (kind(), "has no Dense layer"),
    (kind(dense(4), container=TF + "models.Model"), "spec 'tensorflow.keras.models.Model' is not supported"),
    ({"spec": {TF + "models.Sequential": {"layers": [dense(4)], "trainable": False}}, "compile": {}}, r"unsupported arguments \['trainable'\]"),
    (kind(dense(4), compile={"optimizer": "sgd"}), "optimizer 'sgd'"),
    (kind(dense(4), compile={"optimizer": {TF + "optimizers.SGD": {"learning_rate": 0.001}}}), "optimizer 'SGD'"),
    (kind(dense(4), compile={"loss": "binary_crossentropy"}), "loss 'binary_crossentropy'"),
    (kind(dense(4), compile={"metrics": ["mae"]}), "metrics: none or \\['accuracy'\\]"),
    (kind(dense(4), compile={"loss_weights": [1.0]}), r"compile: unsupported arguments \['loss_weights'\]"),
])
def test_what_the_dense_kernels_do_not_run_is_refused(k, message):
    with pytest.raises(ValueError, match=message):
        spec_of(k)


def test_shapes_must_match_the_data():
    with pytest.raises(ValueError, match=r"input shape \[5\] does not match the 4 features"):
        spec_of(kind(dense(4, input_shape=[5])), 4)
    with pytest.raises(ValueError, match="last Dense layer has 4 units, but y has 1 columns"):
        spec_of(kind(dense(4)), 4, 1)
    model = KerasRawModelRegressor(kind(dense(3, input_shape=[5]), dense(1)))
    with pytest.raises(ValueError, match="does not match the 4 features"):
        model.fit(np.random.rand(10, 4), np.random.rand(10, 1))  # refused while building, before anything reaches a device


# ------------------------------------------------------------------------------------------------ the estimator
REFERENCE_STYLE = """
compile:
  loss: mse
  optimizer: adam
spec:
  tensorflow.keras.models.Sequential:
    layers:
      - tensorflow.keras.layers.Dense:
          units: 4
          input_shape: [4]
      - tensorflow.keras.layers.Dense:
          units: 1
          kernel_regularizer:
            tensorflow.keras.regularizers.L1L2:
              l1: 0.2
"""


def test_the_estimator_surface():
    k = yaml.safe_load(REFERENCE_STYLE)
    model = KerasRawModelRegressor(kind=k)
    assert model.kind is k and model.load_kind(k) is k
    assert repr(model).startswith("KerasRawModelRegressor(kind: {'compile': {'loss': 'mse', 'optimizer': 'adam'},")
    assert model.get_params() == {"kind": k}
    assert isinstance(model, KerasAutoEncoder) and hasattr(model, "score")
    for missing in ({"spec": k["spec"]}, {"compile": k["compile"]}):
        with pytest.raises(ValueError, match=r"Expected spec to have keys: \('spec', 'compile'\)"):
            KerasRawModelRegressor(missing).fit(np.random.rand(10, 4), np.random.rand(10, 1))


def test_definition_pickle_and_clone_round_trips():
    k = yaml.safe_load(REFERENCE_STYLE)
    definition = {"sklearn.pipeline.Pipeline": {"steps": [{"sklearn.decomposition.PCA": {"n_components": 4}},
                                                           {"gordo.machine.model.models.KerasRawModelRegressor": {"kind": k, "epochs": 3}}]}}
    pipe = serializer.from_definition(definition)
    model = pipe.steps[-1][1]
    assert type(model) is KerasRawModelRegressor and model.kind == k and model.kwargs == {"epochs": 3}
    again = serializer.from_definition(serializer.into_definition(pipe)).steps[-1][1]
    assert type(again) is KerasRawModelRegressor and again.kind == k and again.kwargs == {"epochs": 3}
    c = clone(model)
    assert type(c) is KerasRawModelRegressor and c.kind == k and c.kind is not k and c.kwargs == {"epochs": 3}
    for est in (model, _constructed(k)):
        p = pickle.loads(pickle.dumps(est))
        assert type(p) is KerasRawModelRegressor and p.kind == est.kind and p.kwargs == est.kwargs
        if est.model is not None:
            assert p.model.spec == est.model.spec
            for (W0, b0), (W1, b1) in zip(est.model.weights, p.model.weights):
                assert np.array_equal(W0, W1) and np.array_equal(b0, b1)


def _constructed(k, n_in=4, n_out=1):
    """A raw estimator with its network built (Dense initialisers), no fit."""
    m = KerasRawModelRegressor(k)
    m.kwargs.update({"n_features": n_in, "n_features_out": n_out})
    m._prepare_model()
    return m


def test_the_network_is_initialised_as_dense_layers_are():
    m = _constructed(yaml.safe_load(REFERENCE_STYLE))
    (W0, b0), (W1, b1) = m.model.weights
    assert W0.shape == (4, 4) and W1.shape == (4, 1) and not b0.any() and not b1.any()
    assert np.abs(W0).max() <= math.sqrt(6 / 8) and np.abs(W1).max() <= math.sqrt(6 / 5)


def test_specs_pickled_before_the_regularizer_fields_load_without_them():
    s = FFNetSpec([4, 3, 4], ["tanh", "linear"], [0.0, 0.0])
    state = dict(s.__dict__)
    for k in ("kernel_l1", "kernel_l2", "bias_l1", "bias_l2"):
        state.pop(k)
    old = FFNetSpec.__new__(FFNetSpec)
    old.__dict__.update(state)
    assert fit_reg(old) is None and reg_key(old) == ()
    assert reg_key(FFNetSpec([4, 3, 4], ["tanh", "linear"], [0.0, 0.0], kernel_l2=[0.0, 0.0])) == ()
    assert reg_key(FFNetSpec([4, 3, 4], ["tanh", "linear"], [0.0, 0.0], bias_l1=[0.0, 0.1])) == (("reg", (0.0, 0.0), (0.0, 0.0), (0.0, 0.1), (0.0, 0.0)),)


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


def test_the_fleet_builder_batches_raw_detectors_by_their_regularizers():
    plain = kind(dense(3, activation="tanh"), dense(4))
    l2 = kind(dense(3, activation="tanh", kernel_regularizer="l2"), dense(4))
    l1 = kind(dense(3, activation="tanh", kernel_regularizer="l1"), dense(4))
    a, b = builder._canonical(0, _raw_machine("a", plain)), builder._canonical(1, _raw_machine("b", plain))
    c, d = builder._canonical(2, _raw_machine("c", l2)), builder._canonical(3, _raw_machine("d", l1))
    s = builder._canonical(4, _raw_machine("s", l2, scaled=True))
    assert None not in (a, b, c, d, s)
    assert a.spec.dims == [4, 3, 4] and s.input_scaler and not c.input_scaler
    assert a.bucket() == b.bucket()
    assert len({a.bucket(), c.bucket(), d.bucket(), s.bucket()}) == 4
    assert c.bucket()[:-1] == a.bucket() and c.bucket()[-1] == ("reg", (0.0, 0.0), (0.01, 0.0), (0.0, 0.0), (0.0, 0.0))
    assert a.bucket()[:2] == ((4, 3, 4), ("tanh", "linear"))


def test_a_raw_detector_is_served_from_a_resident_bucket():
    for n_out in (4, 1):
        k = kind(dense(5, activation="tanh", kernel_regularizer="l2"), dense(n_out))
        det = DiffBasedAnomalyDetector(base_estimator=KerasRawModelRegressor(k))
        assert not server.ResidentBucket.eligible(det)  # no network yet
        det.base_estimator.kwargs.update({"n_features": 4, "n_features_out": n_out})
        det.base_estimator._prepare_model()
        det.feature_thresholds_, det.aggregate_threshold_ = pd.Series(np.ones(n_out)), 0.5
        det.scaler.fit(np.random.default_rng(0).random((8, n_out)))
        assert server.ResidentBucket.eligible(det)
        assert server._served_parts(det) == ([], det.base_estimator)


# ------------------------------------------------------------------------------------------------ the C entry point
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge

    ge.build()
    return _cabi.load_library()


def test_the_entry_point_is_exported(lib):
    assert "gb_ffae_fit_reg" in _cabi.EXPORTS and hasattr(lib, "gb_ffae_fit_reg")
    assert C.sizeof(_cabi.GbDenseReg) == 4 * 4 * _cabi.GB_MAX_LAYERS
    r = _cabi.make_dense_reg(kernel_l1=[0.1, 0.2], bias_l2=[0.0, 0.5])
    assert list(r.kernel_l1[:3]) == pytest.approx([0.1, 0.2, 0.0]) and list(r.bias_l2[:2]) == [0.0, 0.5] and not any(r.kernel_l2)


@pytest.mark.parametrize("field, value", [("kernel_l1", -0.1), ("kernel_l2", float("nan")), ("bias_l1", float("inf")), ("bias_l2", -1e-9)])
def test_a_bad_coefficient_is_refused_without_a_gpu(lib, field, value):
    """The record is checked before anything touches a device: GB_E_ARG on a GPU-less host, the message naming the field."""
    net = _cabi.make_ffnet([4, 3, 4], ["tanh", "linear"])
    hp = _cabi.GbFitHParams(epochs=1, batch_size=8, shuffle=0, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-7)
    reg = _cabi.make_dense_reg(**{field: [0.0, value]})
    fake = C.c_void_p(16)  # never dereferenced: validation refuses first
    rc = lib.gb_ffae_fit_reg(C.byref(net), fake, fake, fake, fake, None, 1, 8, fake, fake, None, None, C.byref(hp), 8, fake, fake, None, None,
                             None, None, None, None, None, C.byref(reg), None)
    assert rc == -1 and f"reg {field}[1]".encode() in lib.gb_last_error()
    with pytest.raises(ValueError):
        _cabi.check(rc)


def test_the_memory_plan_does_not_depend_on_a_record(lib):
    """gb_ffae_fit_plan takes no record: the REG kernels run in the plans the others do (the penalty lives in registers)."""
    for dims in ([64, 32, 16, 32, 64], [10, 256, 128, 64, 128, 256, 10], [128, 256, 128, 64, 128, 256, 128]):
        net = _cabi.make_ffnet(dims, ["tanh"] * (len(dims) - 2) + ["linear"])
        w, d = C.c_int32(-1), C.c_int32(-1)
        assert lib.gb_ffae_fit_plan(C.byref(net), C.byref(w), C.byref(d)) == 0
    assert lib.gb_ffae_fit_plan.argtypes == [C.POINTER(_cabi.GbFFNet), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
