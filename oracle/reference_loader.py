"""
TEST INFRASTRUCTURE ONLY -- never imported by the product package.

Loads the parts of the *unmodified* reference that can execute without its heavy dependencies
straight from a checkout of equinor/gordo-components named by ``GORDO_REFERENCE_ROOT`` (read-only), so that golden vectors under
``tests/golden/`` are produced by the reference's own code, not by our restatement:

* ``gordo/machine/model/anomaly/diff.py``  (DiffBasedAnomalyDetector, KFCV variant)
* ``gordo/machine/model/utils.py``         (make_base_dataframe, metric_wrapper)
* ``gordo/machine/model/factories/utils.py`` (hourglass_calc_dims, check_dim_func_len)

TensorFlow / Keras / scikeras / xarray / gordo_core are not installed here, so the
modules they would provide are replaced by inert stubs *before* import; none of the
stubbed symbols take part in the anomaly arithmetic.  Only tests/golden/make_golden.py loads
the reference; the test suite reads the fixtures it stored.

Nothing is copied: the reference files are executed where they lie.
"""
from __future__ import annotations

import importlib
import importlib.machinery
import importlib.util
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("GORDO_REFERENCE_ROOT", "")


def reference_available() -> bool:
    """True when GORDO_REFERENCE_ROOT names a reference checkout (never a path relative to the working directory)."""
    return bool(REFERENCE_ROOT) and os.path.isfile(
        os.path.join(REFERENCE_ROOT, "gordo", "machine", "model", "anomaly", "diff.py")
    )


def _ns_module(name: str, path: str | None = None) -> types.ModuleType:
    mod = types.ModuleType(name)
    mod.__spec__ = importlib.machinery.ModuleSpec(name, loader=None)  # importlib.util.find_spec() on a stub must not raise (torch probes for tensorflow)
    if path is not None:
        mod.__path__ = [path]  # namespace-style package; its __init__.py is skipped
    sys.modules[name] = mod
    return mod


def _install_stubs() -> None:
    """Inert stand-ins for third-party packages the reference imports at module scope."""
    if "tensorflow" not in sys.modules:
        tf = _ns_module("tensorflow", path="<stub>")
        keras = _ns_module("tensorflow.keras", path="<stub>")
        tf.keras = keras
        for sub in ("models", "layers", "optimizers", "callbacks", "regularizers"):
            m = _ns_module(f"tensorflow.keras.{sub}")
            setattr(keras, sub, m)
        keras.models.Model = type("Model", (), {})
        keras.models.Sequential = type("Sequential", (), {})
        keras.models.load_model = lambda *a, **k: None
        keras.models.save_model = lambda *a, **k: None
        keras.optimizers.Optimizer = type("Optimizer", (), {})
        keras.layers.Dense = type("Dense", (), {})
        keras.layers.LSTM = type("LSTM", (), {})
        pre = _ns_module("tensorflow.keras.preprocessing", path="<stub>")
        seq = _ns_module("tensorflow.keras.preprocessing.sequence")
        seq.pad_sequences = lambda *a, **k: None
        seq.TimeseriesGenerator = type("TimeseriesGenerator", (), {})
        pre.sequence = seq
        keras.preprocessing = pre
    if "keras" not in sys.modules:
        k = _ns_module("keras", path="<stub>")
        ks = _ns_module("keras.src", path="<stub>")
        kc = _ns_module("keras.src.callbacks")
        kc.Callback = type("Callback", (), {})
        k.src = ks
        ks.callbacks = kc
    if "scikeras" not in sys.modules:
        sk = _ns_module("scikeras", path="<stub>")
        w = _ns_module("scikeras.wrappers")

        class KerasRegressor:  # noqa: D401 - stub
            _fit_kwargs: set = set()
            _predict_kwargs: set = set()
            _compile_kwargs: set = set()
            model = None

            def __init__(self, **kwargs):
                pass

            def get_params(self, **kw):
                return {}

        w.KerasRegressor = KerasRegressor
        sk.wrappers = w
    if "xarray" not in sys.modules:
        xr = _ns_module("xarray")
        xr.DataArray = type("DataArray", (), {})
        xr.Dataset = type("Dataset", (), {})
    if "simplejson" not in sys.modules:
        import json

        sj = _ns_module("simplejson")
        sj.dumps, sj.loads, sj.dump, sj.load = json.dumps, json.loads, json.dump, json.load
    if "gordo_core" not in sys.modules:
        gc = _ns_module("gordo_core", path="<stub>")
        st = _ns_module("gordo_core.sensor_tag")

        class SensorTag:  # minimal value object; only `.name` is read by model/utils.py
            def __init__(self, name, **kw):
                self.name = name

        st.SensorTag = SensorTag
        iu = _ns_module("gordo_core.import_utils")
        iu.import_location = lambda loc: importlib.import_module(loc)
        gc.sensor_tag, gc.import_utils = st, iu


def _install_pandas_append_shim() -> None:
    """
    The reference pins pandas 1.5.3 and calls ``DataFrame.append`` (diff.py:235-237,
    :250-253); pandas >= 2 removed it.  Same semantics, expressed with concat.
    """
    import pandas as pd

    if not hasattr(pd.DataFrame, "append"):

        def _append(self, other, ignore_index=False):
            if isinstance(other, pd.Series):
                other = other.to_frame().T
            if self.empty and len(self.columns) == 0:
                return other.copy()
            return pd.concat([self, other], ignore_index=ignore_index)

        pd.DataFrame.append = _append  # type: ignore[attr-defined]


_loaded: dict = {}


def load_reference():
    """
    Returns a namespace with the reference's own objects:
    ``DiffBasedAnomalyDetector, DiffBasedKFCVAnomalyDetector, make_base_dataframe,
    metric_wrapper, hourglass_calc_dims, check_dim_func_len``.
    """
    if _loaded:
        return types.SimpleNamespace(**_loaded)
    if not reference_available():
        raise FileNotFoundError(
            f"no reference checkout at GORDO_REFERENCE_ROOT={REFERENCE_ROOT!r}; set it to a gordo-components checkout (the tests use tests/golden fixtures)"
        )
    _install_stubs()
    _install_pandas_append_shim()
    g = os.path.join(REFERENCE_ROOT, "gordo")
    # package skeleton whose __init__ chains (gordo_core, dataclasses_json ...) are skipped
    for name, sub in (
        ("gordo", ""),
        ("gordo.machine", "machine"),
        ("gordo.machine.model", "machine/model"),
        ("gordo.machine.model.anomaly", "machine/model/anomaly"),
        ("gordo.machine.model.factories", "machine/model/factories"),
    ):
        if name not in sys.modules:
            _ns_module(name, os.path.join(g, sub))
    # `from gordo import serializer` in models.py -- only attribute access at call time
    if "gordo.serializer" not in sys.modules:
        ser = _ns_module("gordo.serializer")
        sys.modules["gordo"].serializer = ser
    # the real models.py cannot import (it needs TF); diff.py only needs the class
    # object for its default argument, which our goldens never use.
    if "gordo.machine.model.models" not in sys.modules:
        mm = _ns_module("gordo.machine.model.models")

        class KerasAutoEncoder:  # placeholder for diff.py's default base_estimator
            def __init__(self, kind=None, **kw):
                self.kind = kind

        mm.KerasAutoEncoder = KerasAutoEncoder

    def _exec(modname: str, relpath: str):
        spec = importlib.util.spec_from_file_location(modname, os.path.join(g, relpath))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[modname] = mod
        spec.loader.exec_module(mod)
        return mod

    base = _exec("gordo.machine.model.base", "machine/model/base.py")
    mutils = _exec("gordo.machine.model.utils", "machine/model/utils.py")
    sys.modules["gordo.machine.model"].utils = mutils
    sys.modules["gordo.machine.model"].base = base
    _exec("gordo.machine.model.anomaly.base", "machine/model/anomaly/base.py")
    diff = _exec("gordo.machine.model.anomaly.diff", "machine/model/anomaly/diff.py")
    futils = _exec("gordo.machine.model.factories.utils", "machine/model/factories/utils.py")
    _loaded.update(
        DiffBasedAnomalyDetector=diff.DiffBasedAnomalyDetector,
        DiffBasedKFCVAnomalyDetector=diff.DiffBasedKFCVAnomalyDetector,
        make_base_dataframe=mutils.make_base_dataframe,
        metric_wrapper=mutils.metric_wrapper,
        hourglass_calc_dims=futils.hourglass_calc_dims,
        check_dim_func_len=futils.check_dim_func_len,
        GordoBase=base.GordoBase,
    )
    return types.SimpleNamespace(**_loaded)


# ------------------------------------------------------------------------------------------------ the path's callers
_loaded_callers: dict = {}


def _locate(location: str):
    """What gordo_core.import_utils.import_location [3P, absent here] does for ``pkg.mod.attr`` strings."""
    module, _, name = location.rpartition(".")
    if not module:
        raise ValueError(f"not a dotted path: {location!r}")
    return getattr(importlib.import_module(module), name)


def _default_config_globals(gordo_dir: str) -> dict:
    import ast

    with open(os.path.join(gordo_dir, "workflow", "config_elements", "normalized_config.py")) as f:
        tree = ast.parse(f.read())
    for cls in (n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "NormalizedConfig"):
        for node in cls.body:
            target = node.target if isinstance(node, ast.AnnAssign) else (node.targets[0] if isinstance(node, ast.Assign) else None)
            if getattr(target, "id", None) == "DEFAULT_CONFIG_GLOBALS":
                return ast.literal_eval(node.value)
    raise LookupError("NormalizedConfig.DEFAULT_CONFIG_GLOBALS not found in the reference")


class _Record:
    """Stand-in for gordo's metadata dataclasses: keeps the keyword arguments it was built with."""

    def __init__(self, **kwargs):
        self.__dict__.update(kwargs)

    def to_dict(self):
        return {k: (v.to_dict() if isinstance(v, _Record) else v) for k, v in self.__dict__.items()}


def load_reference_callers():
    """
    The reference's own code either side of the hot path, executed from the reference checkout for the golden fixtures of
    tests/golden/make_golden.py (callers_* files):

    * ``gordo/serializer/{from_definition,into_definition,serializer,utils}.py`` -> ``from_definition, into_definition, dump, load ...``
    * ``gordo/machine/model/transformers/imputer.py`` -> ``InfImputer``; ``transformer_funcs/general.py`` -> ``multiply_by``
    * ``gordo/server/utils.py`` -> ``dataframe_to_dict, dataframe_from_dict, dataframe_into_parquet_bytes,
      dataframe_from_parquet_bytes, verify_dataframe`` (flask is absent: ``make_response`` / ``jsonify`` are stubs that hand back
      ``(payload, status)``)
    * ``gordo/builder/build_model.py`` -> ``ModelBuilder`` (its ``_build`` runs against stand-ins for ``Machine`` and the metadata
      dataclasses that merely record what they are given: the cross-validation, scoring, offset and metadata logic is the reference's)
    """
    if _loaded_callers:
        return types.SimpleNamespace(**_loaded_callers)
    ref = load_reference()
    g = os.path.join(REFERENCE_ROOT, "gordo")
    sys.modules["gordo_core.import_utils"].import_location = _locate
    sys.modules["gordo_core.import_utils"].BackCompatibleLocations = type("BackCompatibleLocations", (), {})
    tfk = sys.modules["tensorflow.keras"]
    tfk.Sequential = sys.modules["tensorflow.keras.models"].Sequential
    tf = sys.modules["tensorflow"]
    if not hasattr(tf, "random"):
        tf.random = types.SimpleNamespace(set_seed=lambda seed: None)

    def _exec(modname: str, relpath: str):
        spec = importlib.util.spec_from_file_location(modname, os.path.join(g, relpath))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[modname] = mod
        spec.loader.exec_module(mod)
        return mod

    # the real serializer package replaces the inert stand-in load_reference() registered
    ser = _ns_module("gordo.serializer", os.path.join(g, "serializer"))
    sys.modules["gordo"].serializer = ser
    _exec("gordo.serializer.utils", "serializer/utils.py")
    fd = _exec("gordo.serializer.from_definition", "serializer/from_definition.py")
    idf = _exec("gordo.serializer.into_definition", "serializer/into_definition.py")
    sz = _exec("gordo.serializer.serializer", "serializer/serializer.py")
    for mod, names in ((fd, ("from_definition", "load_params_from_definition", "build_callbacks")), (idf, ("into_definition", "load_definition_from_params")),
                       (sz, ("dump", "dumps", "load", "loads", "load_metadata", "metadata_path", "load_info"))):
        for n in names:
            setattr(ser, n, getattr(mod, n))

    for name, sub in (("gordo.machine.model.transformers", "machine/model/transformers"), ("gordo.machine.model.transformer_funcs", "machine/model/transformer_funcs")):
        if name not in sys.modules:
            _ns_module(name, os.path.join(g, sub))
    imputer = _exec("gordo.machine.model.transformers.imputer", "machine/model/transformers/imputer.py")
    general = _exec("gordo.machine.model.transformer_funcs.general", "machine/model/transformer_funcs/general.py")

    # ---- gordo/server/utils.py: flask is not installed; the two helpers it calls hand back (payload, status)
    if "flask" not in sys.modules:
        fl = _ns_module("flask")
        fl.request, fl.g = types.SimpleNamespace(), types.SimpleNamespace()
        fl.jsonify = lambda payload=None, **kw: payload if payload is not None else kw
        fl.Response = type("Response", (tuple,), {})

        def make_response(*args):
            args = args[0] if len(args) == 1 and isinstance(args[0], tuple) else args
            return fl.Response(args)

        fl.make_response = make_response
    if "gordo.server" not in sys.modules:
        _ns_module("gordo.server", os.path.join(g, "server"))
        props = _ns_module("gordo.server.properties")
        props.get_tags = props.get_target_tags = lambda: []
    server_utils = _exec("gordo.server.utils", "server/utils.py")

    # ---- gordo/builder/build_model.py
    root = sys.modules["gordo"]
    root.__version__ = "0.0.0"
    root.parse_version = lambda v: (0, 0, False)
    if "gordo.util" not in sys.modules:
        util = _ns_module("gordo.util", os.path.join(g, "util"))
        util.disk_registry = _ns_module("gordo.util.disk_registry")
    base_mod = _ns_module("gordo_core.base")

    class GordoBaseDataset:
        registry: dict = {}

        @classmethod
        def from_dict(cls, config):
            return cls.registry[config["key"]]

    base_mod.GordoBaseDataset = GordoBaseDataset
    wf = _ns_module("gordo.workflow", os.path.join(g, "workflow"))
    ce = _ns_module("gordo.workflow.config_elements", os.path.join(g, "workflow", "config_elements"))
    nc = _ns_module("gordo.workflow.config_elements.normalized_config")
    # normalized_config.py itself cannot import here (pydantic schemas, gordo.machine ...); the one thing build_model.py reads from it,
    # the DEFAULT_CONFIG_GLOBALS literal, is evaluated from the reference's source where it lies
    nc.NormalizedConfig = type("NormalizedConfig", (), {"DEFAULT_CONFIG_GLOBALS": _default_config_globals(g)})
    wf.config_elements, ce.normalized_config = ce, nc
    machine_mod = sys.modules["gordo.machine"]

    class Machine(_Record):
        @classmethod
        def from_dict(cls, config, **kwargs):
            config = dict(config)
            config["metadata"] = _Record(**(config.get("metadata") or {}))
            return cls(**config)

    machine_mod.Machine = Machine
    machine_mod.load_model_config = lambda *a, **k: None
    md = _ns_module("gordo.machine.metadata")
    for n in ("BuildMetadata", "ModelBuildMetadata", "DatasetBuildMetadata", "CrossValidationMetaData"):
        setattr(md, n, type(n, (_Record,), {}))
    if "gordo.builder" not in sys.modules:
        _ns_module("gordo.builder", os.path.join(g, "builder"))
    build_model = _exec("gordo.builder.build_model", "builder/build_model.py")

    _loaded_callers.update(
        from_definition=fd.from_definition, into_definition=idf.into_definition, serializer=ser,
        InfImputer=imputer.InfImputer, multiply_by=general.multiply_by,
        dataframe_to_dict=server_utils.dataframe_to_dict, dataframe_from_dict=server_utils.dataframe_from_dict,
        dataframe_into_parquet_bytes=server_utils.dataframe_into_parquet_bytes, dataframe_from_parquet_bytes=server_utils.dataframe_from_parquet_bytes,
        verify_dataframe=server_utils._verify_dataframe,
        ModelBuilder=build_model.ModelBuilder, GordoBaseDataset=GordoBaseDataset, Record=_Record,
        default_evaluation=nc.NormalizedConfig.DEFAULT_CONFIG_GLOBALS["evaluation"],
        DiffBasedAnomalyDetector=ref.DiffBasedAnomalyDetector,
    )
    return types.SimpleNamespace(**_loaded_callers)
