"""
The path's callers against the reference's own code (no GPU needed): tests/golden/callers.{json,npz} were produced by
tests/golden/make_golden.py running the reference's serializer, ModelBuilder._build, server wire helpers and InfImputer
(through oracle/reference_loader.load_reference_callers); here the same inputs go through this package.
"""
import json
import os

import numpy as np
import pandas as pd
import pytest
from sklearn.base import clone

from gordo_components_b200 import builder, serializer, server
from gordo_components_b200.machine.model.transformers.imputer import InfImputer

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(GOLDEN, "callers.json")) as f:
        return json.load(f), np.load(os.path.join(GOLDEN, "callers.npz"))


def _plain(obj):
    """JSON normal form: what the definitions look like after json.dumps (tuples are lists there)."""
    return json.loads(json.dumps(obj))


def test_definition_expansions_equal_the_reference(golden):
    """into_definition(from_definition(d)): the expansion `gordo build` hashes for its cache key (gordo/cli/cli.py:142-144)."""
    meta, _ = golden
    assert len(meta["expansions"]) >= 9
    for case in meta["expansions"]:
        ours = _plain(serializer.into_definition(serializer.from_definition(case["definition"])))
        assert ours == case["expanded"], case["definition"]
        # and the expansion is a fixed point, as it is for the reference
        assert _plain(serializer.into_definition(serializer.from_definition(case["expanded"]))) == case["expanded"]


def _build_frame(meta, arrays):
    info = meta["build_frame"]
    idx = pd.date_range(info["start"], periods=info["rows"], freq=info["freq"])
    return pd.DataFrame(arrays["build_frame"], index=idx, columns=info["columns"])


class _Dataset:
    def __init__(self, frame):
        self.frame = frame

    def get_data(self):
        return self.frame, self.frame

    def get_metadata(self):
        return {"rows": len(self.frame)}


def _assert_scores(ours: dict, theirs: dict, rtol=1e-9):
    assert list(ours) == list(theirs)  # same keys in the same order: '<metric>-<tag>' per tag, then '<metric>'
    for key in theirs:
        assert list(ours[key]) == list(theirs[key]), key
        for stat in theirs[key]:
            np.testing.assert_allclose(ours[key][stat], theirs[key][stat], rtol=rtol, atol=1e-12, err_msg=f"{key} {stat}")


@pytest.mark.parametrize("case", ["default", "five_folds_unscaled", "cv_only"])
def test_model_builder_equals_the_reference_build(golden, case):
    """ModelBuilder._build (build_model.py:192-339) on a scikit-learn model: scores, splits, offset, metadata layout."""
    meta, arrays = golden
    frame = _build_frame(meta, arrays)
    want = meta["build"][case]["build_metadata"]
    machine = {"name": "fixture-machine", "project_name": "p", "model": meta["build_model"], "dataset": _Dataset(frame),
               "evaluation": meta["build"][case]["evaluation"], "metadata": {"user_defined": {"k": 1}}}
    model, built = builder.ModelBuilder(machine).build()
    got = built["metadata"]["build_metadata"]
    assert built["metadata"]["user_defined"] == {"k": 1} and built["name"] == "fixture-machine"
    assert got["dataset"]["dataset_meta"] == want["dataset"]["dataset_meta"]
    timing = {"model_creation_date", "model_training_duration_sec"}
    assert set(got["model"]) - timing == set(want["model"])
    _assert_scores(got["model"]["cross_validation"]["scores"], want["model"]["cross_validation"]["scores"])
    assert {k: str(v) if "start" in k or "end" in k else v for k, v in got["model"]["cross_validation"]["splits"].items()} == want["model"]["cross_validation"]["splits"]
    if case != "cv_only":
        assert got["model"]["model_offset"] == want["model"]["model_offset"] == 0
        assert got["model"]["model_meta"] == want["model"]["model_meta"]
        np.testing.assert_allclose(model.predict(frame), arrays[f"build_{case}_prediction"], rtol=1e-12)
    else:
        assert not hasattr(model.steps[-1][1], "coef_")  # cross_val_only leaves the model itself unfitted


def test_default_evaluation_is_the_reference_default(golden):
    meta, _ = golden
    assert builder.DEFAULT_EVALUATION == meta["default_evaluation"]
    assert [f.__name__ for f in builder.metrics_from_list(None)] == meta["default_evaluation"]["metrics"]


@pytest.mark.parametrize("case", ["default", "five_folds_unscaled", "cv_only"])
def test_moment_scores_equal_the_reference_scorers(golden, case):
    """
    The batched builder's route -- five column sums per fold, then `scores_from_moments` -- gives what the reference's sklearn
    scorers gave for the same fold predictions, under a MinMaxScaler, no scaler and a RobustScaler as scoring scaler.
    """
    meta, arrays = golden
    frame = _build_frame(meta, arrays)
    evaluation = meta["build"][case]["evaluation"]
    want = meta["build"][case]["build_metadata"]["model"]["cross_validation"]["scores"]
    split = serializer.from_definition(evaluation.get("cv", builder.DEFAULT_CV))
    scale = None
    if evaluation.get("scoring_scaler"):
        fitted = serializer.from_definition(evaluation["scoring_scaler"]).fit(frame)
        probe = fitted.transform(np.vstack([np.zeros(frame.shape[1]), np.ones(frame.shape[1])]))
        scale = probe[1] - probe[0]  # the per-tag slope of any affine scaler
    moments, rows = [], set()
    for train, test in split.split(frame):
        fold = clone(serializer.from_definition(meta["build_model"])).fit(frame.iloc[train], frame.iloc[train])
        pred, y = np.asarray(fold.predict(frame.iloc[test]), dtype=np.float64), frame.values[test]
        e, c = pred - y, y - y[0]
        moments.append(np.stack([e.sum(0), (e * e).sum(0), np.abs(e).sum(0), c.sum(0), (c * c).sum(0)]))
        rows.add(len(test))
    assert len(rows) == 1
    names = [m.rpartition(".")[2] for m in evaluation["metrics"]]
    ours = builder.scores_block(builder.scores_from_moments(np.stack(moments), rows.pop(), scale, names), list(frame.columns))
    _assert_scores(ours, want, rtol=1e-8)


# ---------------------------------------------------------------- server wire formats (gordo/server/utils.py:47-247)
def _wire_frames():
    idx = pd.date_range("2016-01-01", periods=4, freq="10min", tz="UTC")
    cols = pd.MultiIndex.from_tuples([("start", ""), ("model-output", "tag 0"), ("model-output", "tag 1"), ("total-anomaly-scaled", "")])
    multi = pd.DataFrame(np.arange(16.0).reshape(4, 4) / 7.0, columns=cols, index=idx)
    multi[("start", "")] = [t.isoformat() for t in idx]
    plain = pd.DataFrame(np.arange(8.0).reshape(4, 2) / 3.0, columns=["a", "b"], index=idx)
    numbered = pd.DataFrame({"a": [1.5, 2.5, 3.5]}, index=[2, 0, 1])
    return multi, plain, numbered


def test_wire_formats_equal_the_reference(golden):
    meta, _ = golden
    wire = meta["wire"]
    multi, plain, numbered = _wire_frames()
    assert _plain(server.dataframe_to_dict(multi)) == wire["multi"]
    assert _plain(server.dataframe_to_dict(plain)) == wire["plain"]
    assert _plain(server.dataframe_to_dict(numbered)) == wire["numbered"]
    back = server.dataframe_from_dict(wire["multi"])
    assert [list(c) for c in back.columns] == wire["multi_back"]["columns"]
    assert [str(t) for t in back.index] == wire["multi_back"]["index"]
    np.testing.assert_array_equal(back["model-output"].values, np.asarray(wire["multi_back"]["model_output"]))
    nb = server.dataframe_from_dict(wire["numbered"])
    assert [int(i) for i in nb.index] == wire["numbered_back"]["index"] and nb["a"].tolist() == wire["numbered_back"]["a"]

    expected = ["tag-0", "tag-1", "tag-2"]
    cases = {"unlabelled": pd.DataFrame(np.zeros((2, 3))), "shuffled_superset": pd.DataFrame(np.zeros((2, 4)), columns=["tag-2", "x", "tag-0", "tag-1"]),
             "too_wide": pd.DataFrame(np.zeros((2, 4))), "multi_level": multi}
    for name, df in cases.items():
        res, want = server.verify_dataframe(df, expected), wire["verify"][name]
        if "columns" in want:
            assert [str(c) for c in res.columns] == want["columns"], name
        else:
            assert isinstance(res, server.Reply) and res.status == want["status"] and res.body["message"] == want["message"], name


# ---------------------------------------------------------------- InfImputer (transformers/imputer.py:12-127)
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_infimputer_equals_the_reference(golden, dtype):
    _, arrays = golden
    base = arrays[f"imputer_{dtype}_input"]
    assert str(base.dtype) == dtype and np.isinf(base).sum() > 20
    runs = {"minmax": InfImputer(strategy="minmax", delta=2.0), "extremes": InfImputer(strategy="extremes"),
            "filled": InfImputer(inf_fill_value=99.0, neg_inf_fill_value=-99.0, strategy=None), "half": InfImputer(inf_fill_value=99.0, delta=0.5)}
    for name, imputer in runs.items():
        got = imputer.fit_transform(base.copy())
        assert got.dtype == arrays[f"imputer_{dtype}_{name}"].dtype
        np.testing.assert_array_equal(got, arrays[f"imputer_{dtype}_{name}"], err_msg=name)
