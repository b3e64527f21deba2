"""
ctypes binding of the C-ABI library (include/gordo_b200.h, built by csrc/build.py).

There is no CPU fallback: if the shared library is missing, or no sm_90 (H100) device is
visible, every compute entry point raises.  PyTorch is used only as the owner of device
memory and streams; the pointers handed to the library are raw device addresses.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libgordo_b200.so")

GB_MAX_LAYERS = 16
GB_MAX_WIDTH = 256
ACT_CODES = {"linear": 0, None: 0, "tanh": 1, "relu": 2, "sigmoid": 3}
GB_LOSS_MSE, GB_LOSS_MAE, GB_LOSS_MAPE, GB_LOSS_MSLE, GB_LOSS_HUBER, GB_LOSS_LOG_COSH = range(6)  # gb_loss
LOSS_CODES = {"mse": GB_LOSS_MSE, "mae": GB_LOSS_MAE, "mape": GB_LOSS_MAPE, "msle": GB_LOSS_MSLE, "huber": GB_LOSS_HUBER,
              "log_cosh": GB_LOSS_LOG_COSH}


def loss_code(loss: str) -> int:
    """gb_loss id of a canonical loss name (``factories.specs.resolve_loss`` maps the Keras spellings to these)."""
    if loss not in LOSS_CODES:
        raise ValueError(f"loss {loss!r} is not one the CUDA fit kernels implement {sorted(LOSS_CODES)}")
    return LOSS_CODES[loss]

GB_OPT_ADAM, GB_OPT_ADAMW, GB_OPT_RMSPROP, GB_OPT_ADAGRAD, GB_OPT_ADADELTA, GB_OPT_ADAMAX, GB_OPT_NADAM = range(7)  # gb_opt
GB_OPT_CENTERED = 1
OPT_CODES = {"adam": GB_OPT_ADAM, "adamw": GB_OPT_ADAMW, "rmsprop": GB_OPT_RMSPROP, "adagrad": GB_OPT_ADAGRAD, "adadelta": GB_OPT_ADADELTA,
             "adamax": GB_OPT_ADAMAX, "nadam": GB_OPT_NADAM}


class GbOptimizer(C.Structure):
    _fields_ = [("kind", C.c_int32), ("flags", C.c_int32), ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float),
                ("eps", C.c_float), ("momentum", C.c_float), ("initial_accumulator", C.c_float), ("weight_decay", C.c_float),
                ("clipvalue", C.c_float)]


def make_optimizer(name: str, cfg) -> GbOptimizer:
    """gb_optimizer of a canonical optimizer name and its complete record (``factories.specs.resolve_optimizer``)."""
    if name not in OPT_CODES:
        raise ValueError(f"optimizer {name!r} is not one the CUDA fit kernels implement {sorted(OPT_CODES)}")
    o = GbOptimizer()
    o.kind = OPT_CODES[name]
    o.flags = GB_OPT_CENTERED if cfg.get("centered") else 0
    o.lr, o.eps = float(cfg["lr"]), float(cfg["eps"])
    o.beta1 = float(cfg.get("beta1", cfg.get("rho", 0.0)))
    o.beta2 = float(cfg.get("beta2", 0.0))
    o.momentum = float(cfg.get("momentum", 0.0))
    o.initial_accumulator = float(cfg.get("initial_accumulator_value", 0.0))
    o.weight_decay = float(cfg.get("weight_decay") or 0.0)
    o.clipvalue = float(cfg.get("clipvalue") or 0.0)
    return o


class GbDenseReg(C.Structure):
    _fields_ = [("kernel_l1", C.c_float * GB_MAX_LAYERS), ("kernel_l2", C.c_float * GB_MAX_LAYERS), ("bias_l1", C.c_float * GB_MAX_LAYERS),
                ("bias_l2", C.c_float * GB_MAX_LAYERS)]


REG_FIELDS = ("kernel_l1", "kernel_l2", "bias_l1", "bias_l2")


def make_dense_reg(kernel_l1=None, kernel_l2=None, bias_l1=None, bias_l2=None) -> GbDenseReg:
    """gb_dense_reg of per-layer Keras kernel / bias regularizer coefficients (None or a list per field, zeros where absent)."""
    r = GbDenseReg()
    for name, vals in zip(REG_FIELDS, (kernel_l1, kernel_l2, bias_l1, bias_l2)):
        vals = list(vals or ())
        if len(vals) > GB_MAX_LAYERS:
            raise ValueError(f"{name}: {len(vals)} layers is more than {GB_MAX_LAYERS}")
        for i, v in enumerate(vals):
            getattr(r, name)[i] = float(v)
    return r


class GbDenseDropout(C.Structure):
    _fields_ = [("rate", C.c_float * GB_MAX_LAYERS)]


def make_dense_dropout(rate=None) -> GbDenseDropout:
    """gb_dense_dropout of per-layer Keras Dropout rates (``rate[l]`` on the input of Dense layer l; zeros where absent)."""
    r = GbDenseDropout()
    vals = list(rate or ())
    if len(vals) > GB_MAX_LAYERS:
        raise ValueError(f"dropout: {len(vals)} layers is more than {GB_MAX_LAYERS}")
    for i, v in enumerate(vals):
        r.rate[i] = float(v)
    return r


EXPORTS = (
    "gb_abi_version", "gb_last_error", "gb_device_check", "gb_ffnet_param_count", "gb_ffnet_param_stride",
    "gb_ffae_infer_score", "gb_ffae_tc_supported", "gb_ffae_infer_plan", "gb_ffae_infer_score_x64", "gb_ffae_infer_plan_x64", "gb_anomaly_score", "gb_anomaly_score_f64", "gb_minmax_fit", "gb_minmax_f64", "gb_thresholds", "gb_thresholds_f64", "gb_thresholds_pair", "gb_thresholds_pair_f64", "gb_cv_moments", "gb_smooth", "gb_smooth_scores", "gb_quantile", "gb_affine_f64", "gb_gather_rows", "gb_gather_rows_ragged", "gb_minmax_inverse_f32", "gb_minmax_inverse_score_f64", "gb_ffae_fit_state_stride", "gb_ffae_fit", "gb_ffae_fit_split", "gb_ffae_fit_stop", "gb_ffae_fit_plan", "gb_ffae_fit_opt", "gb_ffae_fit_reg", "gb_ffae_fit_drop", "gb_ffae_fit_group", "gb_ffae_fit_group_workspace_bytes",
    "gb_lstm_param_count", "gb_lstm_param_stride", "gb_lstm_workspace_bytes", "gb_lstm_infer", "gb_lstm_tc_supported", "gb_lstm_tc_workspace_bytes", "gb_lstm_infer_tc", "gb_lstm_tc_ragged_workspace_bytes", "gb_lstm_infer_tc_ragged", "gb_lstm_fit_workspace_bytes", "gb_lstm_fit", "gb_lstm_fit_loss", "gb_lstm_fit_tc_workspace_bytes", "gb_lstm_fit_tc", "gb_lstm_fit_opt", "gb_lstm_fit_tc_opt",
    "gb_lstm_fit_stop_state_bytes", "gb_lstm_fit_stop", "gb_lstm_fit_tc_stop",
    "gb_orthonormal_rows",
)


class GbFFNet(C.Structure):
    _fields_ = [("n_layers", C.c_int32), ("dims", C.c_int32 * (GB_MAX_LAYERS + 1)), ("act", C.c_int32 * GB_MAX_LAYERS),
                ("l1", C.c_float * GB_MAX_LAYERS)]


class GbFitGroup(C.Structure):
    _fields_ = [("net", GbFFNet), ("params", C.c_void_p), ("adam_m", C.c_void_p), ("adam_v", C.c_void_p), ("best_params", C.c_void_p),
                ("x", C.c_void_p), ("y", C.c_void_p)]


class GbJob(C.Structure):
    _fields_ = [("slot", C.c_int32), ("n_rows", C.c_int32), ("x_row", C.c_int64), ("out_row", C.c_int64)]


JOB_DTYPE = np.dtype([("slot", "<i4"), ("n_rows", "<i4"), ("x_row", "<i8"), ("out_row", "<i8")])
assert JOB_DTYPE.itemsize == C.sizeof(GbJob) == 24


class GbFitHParams(C.Structure):
    _fields_ = [("epochs", C.c_int32), ("batch_size", C.c_int32), ("shuffle", C.c_int32), ("l1_div_batch", C.c_int32),
                ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
                ("seed", C.c_uint64), ("step0", C.c_int32), ("loss", C.c_int32)]


class GbFitSplit(C.Structure):
    _fields_ = [("n_val", C.c_int32), ("reserved", C.c_int32), ("map_ofs", C.c_int64)]


SPLIT_DTYPE = np.dtype([("n_val", "<i4"), ("reserved", "<i4"), ("map_ofs", "<i8")])
assert SPLIT_DTYPE.itemsize == C.sizeof(GbFitSplit) == 16


class GbFitStop(C.Structure):
    _fields_ = [("monitor", C.c_int32), ("mode", C.c_int32), ("patience", C.c_int32), ("start_from_epoch", C.c_int32),
                ("restore_best", C.c_int32), ("has_baseline", C.c_int32), ("min_delta", C.c_double), ("baseline", C.c_double)]


STOP_DTYPE = np.dtype([("monitor", "<i4"), ("mode", "<i4"), ("patience", "<i4"), ("start_from_epoch", "<i4"), ("restore_best", "<i4"),
                       ("has_baseline", "<i4"), ("min_delta", "<f8"), ("baseline", "<f8")])
assert STOP_DTYPE.itemsize == C.sizeof(GbFitStop) == 40
STOP_MONITORS = {"loss": 0, "accuracy": 1, "val_loss": 2, "val_accuracy": 3}


class GbLstmNet(C.Structure):
    _fields_ = [("n_layers", C.c_int32), ("n_features", C.c_int32), ("n_features_out", C.c_int32),
                ("units", C.c_int32 * GB_MAX_LAYERS), ("act", C.c_int32 * GB_MAX_LAYERS), ("out_act", C.c_int32),
                ("lookback", C.c_int32)]


class GbLstmFitHParams(C.Structure):
    _fields_ = [("epochs", C.c_int32), ("batch_size", C.c_int32), ("lookahead", C.c_int32), ("primer", C.c_int32),
                ("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float)]


class GordoB200Error(RuntimeError):
    pass


_lib = None
_lock = threading.Lock()
_P = C.c_void_p


def _declare(lib):
    lib.gb_abi_version.restype = C.c_int
    lib.gb_last_error.restype = C.c_char_p
    lib.gb_device_check.argtypes = [C.c_int, C.POINTER(C.c_int)]
    for name in ("gb_ffnet_param_count", "gb_ffnet_param_stride", "gb_ffae_fit_state_stride"):
        getattr(lib, name).restype = C.c_size_t
        getattr(lib, name).argtypes = [C.POINTER(GbFFNet)]
    for name in ("gb_lstm_param_count", "gb_lstm_param_stride"):
        getattr(lib, name).restype = C.c_size_t
        getattr(lib, name).argtypes = [C.POINTER(GbLstmNet)]
    lib.gb_lstm_workspace_bytes.restype = C.c_size_t
    lib.gb_lstm_workspace_bytes.argtypes = [C.POINTER(GbLstmNet), C.c_int32, C.c_int32]
    lib.gb_ffae_infer_score.argtypes = [C.POINTER(GbFFNet), _P, _P, C.c_int32, C.c_int32, C.c_int64, C.c_int64] + [_P] * 12 + [C.c_int32, _P]
    lib.gb_ffae_infer_score_x64.argtypes = [C.POINTER(GbFFNet), _P, _P, C.c_int32, C.c_int32, C.c_int64, C.c_int64] + [_P] * 14 + [C.c_int32, _P]
    lib.gb_ffae_infer_score_x64.restype = C.c_int
    lib.gb_ffae_infer_plan_x64.argtypes = [C.POINTER(GbFFNet), C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    lib.gb_ffae_infer_plan_x64.restype = C.c_int
    lib.gb_ffae_tc_supported.argtypes = [C.POINTER(GbFFNet)]
    lib.gb_ffae_tc_supported.restype = C.c_int
    lib.gb_anomaly_score.argtypes = [_P, C.c_int32, C.c_int32, _P, _P, C.c_int32] + [_P] * 9 + [_P]
    lib.gb_anomaly_score.restype = C.c_int
    lib.gb_anomaly_score_f64.argtypes = lib.gb_anomaly_score.argtypes
    lib.gb_anomaly_score_f64.restype = C.c_int
    lib.gb_minmax_fit.argtypes = [_P, C.c_int32, C.c_int32, _P, C.c_int32, _P, _P, _P, C.c_int32, _P]
    lib.gb_minmax_f64.argtypes = [_P, C.c_int32, C.c_int32, _P, C.c_int32, _P, C.c_int32, _P]
    lib.gb_minmax_f64.restype = C.c_int
    lib.gb_thresholds.argtypes = [_P, C.c_int32, C.c_int32, _P, _P, C.c_int32, C.c_int32, _P, _P, C.c_int32, _P]
    lib.gb_thresholds_f64.argtypes = lib.gb_thresholds.argtypes
    lib.gb_thresholds_f64.restype = C.c_int
    lib.gb_thresholds_pair.argtypes = [_P, C.c_int32, C.c_int32, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P, C.c_int32, _P]
    lib.gb_thresholds_pair.restype = C.c_int
    lib.gb_thresholds_pair_f64.argtypes = lib.gb_thresholds_pair.argtypes
    lib.gb_thresholds_pair_f64.restype = C.c_int
    lib.gb_cv_moments.argtypes = [_P, C.c_int32, _P, _P, C.c_int32, _P, _P]
    lib.gb_cv_moments.restype = C.c_int
    lib.gb_smooth.argtypes = [_P, C.c_int32, C.c_int32, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P]
    lib.gb_smooth.restype = C.c_int
    lib.gb_smooth_scores.argtypes = [_P, C.c_int32, C.c_int32, _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P, _P]
    lib.gb_smooth_scores.restype = C.c_int
    lib.gb_quantile.argtypes = [_P, C.c_int32, C.c_int32, _P, C.c_int32, C.c_float, _P, _P]
    lib.gb_quantile.restype = C.c_int
    lib.gb_affine_f64.argtypes = [_P, C.c_int32, C.c_int32, _P, C.c_int32, _P, _P, _P, _P]
    lib.gb_affine_f64.restype = C.c_int
    lib.gb_gather_rows.argtypes = [_P, C.c_int32, C.c_int32, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P]
    lib.gb_gather_rows.restype = C.c_int
    lib.gb_gather_rows_ragged.argtypes = [_P, C.c_int32, C.c_int32, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P]
    lib.gb_gather_rows_ragged.restype = C.c_int
    lib.gb_minmax_inverse_f32.argtypes = [_P, C.c_int32, C.c_int32, _P, C.c_int32, _P, _P, _P, _P, _P]
    lib.gb_minmax_inverse_f32.restype = C.c_int
    lib.gb_minmax_inverse_score_f64.argtypes = [_P, C.c_int32, C.c_int32, _P, _P, C.c_int32] + [_P] * 12 + [_P]
    lib.gb_minmax_inverse_score_f64.restype = C.c_int
    lib.gb_ffae_fit.argtypes = [C.POINTER(GbFFNet), _P, _P, _P, _P, C.c_int32, C.c_int32, _P, _P, _P,
                                C.POINTER(GbFitHParams), _P, _P, _P]
    lib.gb_ffae_fit_split.argtypes = [C.POINTER(GbFFNet), _P, _P, _P, _P, _P, C.c_int32, C.c_int32, _P, _P, _P, _P,
                                      C.POINTER(GbFitHParams), C.c_int32, _P, _P, _P, _P, _P]
    lib.gb_ffae_fit_stop.argtypes = lib.gb_ffae_fit_split.argtypes[:-1] + [_P] * 5
    lib.gb_ffae_fit_plan.argtypes = [C.POINTER(GbFFNet), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    lib.gb_ffae_fit_plan.restype = C.c_int
    lib.gb_ffae_infer_plan.argtypes = [C.POINTER(GbFFNet), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    lib.gb_ffae_infer_plan.restype = C.c_int
    lib.gb_lstm_infer.argtypes = [C.POINTER(GbLstmNet), _P, _P, C.c_int32, C.c_int32, _P, _P, _P, _P]
    lib.gb_lstm_tc_supported.argtypes = [C.POINTER(GbLstmNet)]
    lib.gb_lstm_tc_supported.restype = C.c_int
    lib.gb_lstm_tc_workspace_bytes.argtypes = [C.POINTER(GbLstmNet), C.c_int32, C.c_int32, C.c_int32, C.c_int64]
    lib.gb_lstm_tc_workspace_bytes.restype = C.c_size_t
    lib.gb_lstm_infer_tc.argtypes = [C.POINTER(GbLstmNet), _P, C.c_int32, _P, C.c_int32, C.c_int32, _P, C.c_int64, _P, _P, _P]
    lib.gb_lstm_infer_tc.restype = C.c_int
    lib.gb_lstm_tc_ragged_workspace_bytes.argtypes = [C.POINTER(GbLstmNet), C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    lib.gb_lstm_tc_ragged_workspace_bytes.restype = C.c_size_t
    lib.gb_lstm_infer_tc_ragged.argtypes = [C.POINTER(GbLstmNet), _P, C.c_int32, _P, C.c_int32, _P, C.c_int32, C.c_int32, _P, C.c_int64, _P, _P, _P]
    lib.gb_lstm_infer_tc_ragged.restype = C.c_int
    lib.gb_lstm_fit_workspace_bytes.restype = C.c_size_t
    lib.gb_lstm_fit_workspace_bytes.argtypes = [C.POINTER(GbLstmNet), C.c_int32]
    lib.gb_lstm_fit.argtypes = [C.POINTER(GbLstmNet), _P, _P, _P, _P, _P, C.c_int32, C.c_int32, _P, _P, C.POINTER(GbLstmFitHParams), _P, _P, _P, _P]
    lib.gb_lstm_fit.restype = C.c_int
    lib.gb_lstm_fit_loss.argtypes = lib.gb_lstm_fit.argtypes[:-1] + [C.c_int32, _P]
    lib.gb_lstm_fit_loss.restype = C.c_int
    lib.gb_lstm_fit_tc_workspace_bytes.restype = C.c_size_t
    lib.gb_lstm_fit_tc_workspace_bytes.argtypes = [C.POINTER(GbLstmNet), C.c_int32, C.c_int32]
    lib.gb_lstm_fit_tc.argtypes = lib.gb_lstm_fit_loss.argtypes
    lib.gb_lstm_fit_tc.restype = C.c_int
    lib.gb_ffae_fit_opt.argtypes = lib.gb_ffae_fit_stop.argtypes[:-1] + [C.POINTER(GbOptimizer), _P]
    lib.gb_ffae_fit_opt.restype = C.c_int
    lib.gb_ffae_fit_reg.argtypes = lib.gb_ffae_fit_opt.argtypes[:-1] + [C.POINTER(GbDenseReg), _P]
    lib.gb_ffae_fit_reg.restype = C.c_int
    lib.gb_ffae_fit_drop.argtypes = lib.gb_ffae_fit_reg.argtypes[:-1] + [C.POINTER(GbDenseDropout), _P]
    lib.gb_ffae_fit_drop.restype = C.c_int
    lib.gb_ffae_fit_group.argtypes = [C.POINTER(GbFitGroup), C.c_int32, C.POINTER(C.c_int32), _P, _P, C.c_int32, C.c_int32, _P, _P,
                                      C.POINTER(GbFitHParams), C.c_int32] + [_P] * 7 + [C.POINTER(GbOptimizer), C.POINTER(GbDenseReg),
                                                                                       C.POINTER(GbDenseDropout), _P, _P]
    lib.gb_ffae_fit_group.restype = C.c_int
    lib.gb_ffae_fit_group_workspace_bytes.argtypes = [C.c_int32, C.c_int32]
    lib.gb_ffae_fit_group_workspace_bytes.restype = C.c_size_t
    for name in ("gb_lstm_fit_opt", "gb_lstm_fit_tc_opt"):
        getattr(lib, name).argtypes = lib.gb_lstm_fit_loss.argtypes[:-1] + [C.POINTER(GbOptimizer), _P]
        getattr(lib, name).restype = C.c_int
    lib.gb_lstm_fit_stop_state_bytes.restype = C.c_size_t
    lib.gb_lstm_fit_stop_state_bytes.argtypes = [C.c_int32]
    for name in ("gb_lstm_fit_stop", "gb_lstm_fit_tc_stop"):
        getattr(lib, name).argtypes = lib.gb_lstm_fit_opt.argtypes[:-1] + [_P] * 5
        getattr(lib, name).restype = C.c_int
    lib.gb_orthonormal_rows.argtypes = [_P, C.c_int32, C.c_int32, C.c_int32, _P, C.c_int64, C.c_int64, _P]
    lib.gb_orthonormal_rows.restype = C.c_int
    for name in ("gb_device_check", "gb_ffae_infer_score", "gb_ffae_tc_supported", "gb_ffae_infer_plan", "gb_anomaly_score", "gb_minmax_fit", "gb_thresholds", "gb_smooth", "gb_ffae_fit", "gb_ffae_fit_split", "gb_ffae_fit_stop", "gb_lstm_infer"):
        getattr(lib, name).restype = C.c_int


def load_library():
    """dlopen the C-ABI library (no GPU needed for this step).  Raises if it has not been built."""
    global _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise GordoB200Error(
                    f"{LIB_PATH} is missing: build it with `python gordo_components_b200/csrc/build.py` "
                    "(or __graft_entry__.build()).  gordo_components_b200 has no CPU fallback."
                )
            lib = C.CDLL(LIB_PATH)
            _declare(lib)
            if lib.gb_abi_version() != 2:
                raise GordoB200Error(f"ABI version mismatch: library {lib.gb_abi_version()}, binding 2")
            _lib = lib
    return _lib


_STATUS_EXC = {-1: ValueError, -2: ValueError, -3: ValueError, -4: ValueError, -5: GordoB200Error, -6: GordoB200Error}


def check(rc: int):
    if rc != 0:
        msg = load_library().gb_last_error().decode("utf-8", "replace")
        raise _STATUS_EXC.get(rc, GordoB200Error)(f"gordo_b200 [{rc}]: {msg}")


_device_ok = {}


def require_device(device_index: int = 0) -> int:
    """Fail loudly unless `device_index` is an sm_90 (H100) GPU.  Returns its SM count."""
    if device_index in _device_ok:
        return _device_ok[device_index]
    lib = load_library()
    sms = C.c_int(0)
    check(lib.gb_device_check(int(device_index), C.byref(sms)))
    _device_ok[device_index] = sms.value
    return sms.value


def make_ffnet(dims, acts, l1=None) -> GbFFNet:
    n_layers = len(dims) - 1
    if not (1 <= n_layers <= GB_MAX_LAYERS):
        raise ValueError(f"a Dense stack of {n_layers} layers is outside [1, {GB_MAX_LAYERS}]")
    if len(acts) != n_layers:
        raise ValueError("one activation per layer is required")
    net = GbFFNet()
    net.n_layers = n_layers
    for i, d in enumerate(dims):
        net.dims[i] = int(d)
    for i, a in enumerate(acts):
        if a not in ACT_CODES:
            raise ValueError(f"activation {a!r} is not supported by the CUDA kernels (supported: tanh, relu, sigmoid, linear)")
        net.act[i] = ACT_CODES[a]
        net.l1[i] = float(l1[i]) if l1 is not None else 0.0
    return net


def make_lstmnet(n_features, units, acts, n_features_out, out_act, lookback) -> GbLstmNet:
    if not (1 <= len(units) <= GB_MAX_LAYERS):
        raise ValueError(f"an LSTM stack of {len(units)} layers is outside [1, {GB_MAX_LAYERS}]")
    net = GbLstmNet()
    net.n_layers = len(units)
    net.n_features, net.n_features_out = int(n_features), int(n_features_out)
    for i, (u, a) in enumerate(zip(units, acts)):
        if a not in ACT_CODES:
            raise ValueError(f"activation {a!r} is not supported by the CUDA kernels")
        net.units[i], net.act[i] = int(u), ACT_CODES[a]
    if out_act not in ACT_CODES:
        raise ValueError(f"activation {out_act!r} is not supported by the CUDA kernels")
    net.out_act = ACT_CODES[out_act]
    net.lookback = int(lookback)
    return net


def ptr(t):
    """Raw device address of a torch tensor (None -> NULL).  The kernels index dense row-major memory: anything else is refused."""
    if t is None:
        return None
    if not t.is_contiguous():
        raise ValueError(f"tensor of shape {tuple(t.shape)} with strides {tuple(t.stride())} is not C-contiguous; the gordo_b200 "
                         "kernels take dense row-major arrays (call .contiguous() / np.ascontiguousarray first)")
    return C.c_void_p(t.data_ptr())
