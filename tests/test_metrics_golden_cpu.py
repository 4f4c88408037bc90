"""CPU: the AUC of metrics.py and of the drop-in's compute_auc_sklearn against the reference's own compute_auc_sklearn
(tests/golden/metrics_golden.npz, tools/make_golden_metrics.py), and the host side of examples/eval_bop_results.py:
the walk over a result file, skipped frames and the choice of symmetric objects."""
import os
import sys

import numpy as np
import pytest
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "metrics_golden.npz"))
AUC_CASES = sorted({k.split("/")[1] for k in GOLDEN.files if k.startswith("auc/")})
sys.path[:0] = [os.path.join(ROOT, "examples"), os.path.join(ROOT, "foundationpose_b200", "dropin"), ROOT]


@pytest.mark.parametrize("case", AUC_CASES)
def test_auc_matches_reference(case):
    import Utils

    from foundationpose_b200 import metrics

    errs, (max_val, step), want = GOLDEN[f"auc/{case}/errs"], GOLDEN[f"auc/{case}/params"], float(GOLDEN[f"auc/{case}/auc"])
    assert abs(metrics.auc(errs, max_val=max_val, step=step) - want) <= 1e-12
    assert abs(Utils.compute_auc_sklearn(errs, max_val=max_val, step=step) - want) <= 1e-12
    assert abs(metrics.auc(list(errs[::-1]), max_val=max_val, step=step) - want) <= 1e-12  # order does not matter


def test_auc_closed_form():
    """One error e on a step: the curve is 0 below e, 1 from e on, with one trapezoid of width `step` between."""
    from foundationpose_b200 import metrics

    assert metrics.auc([0.0]) == 1.0
    assert metrics.auc([0.05]) == pytest.approx(1.0 - 0.05 / 0.1 + 0.5 * 0.001 / 0.1, abs=1e-12)
    assert metrics.auc([np.inf]) == 0.0


def test_recall():
    from foundationpose_b200 import metrics

    assert metrics.recall([0.0, 0.01, 0.02, np.inf], 0.02) == 0.5
    assert metrics.recall([0.01, 0.01], [0.02, 0.005]) == 0.5


def _result_file(tmp_path):
    res = {1: {"000000": {2: np.eye(4).tolist(), 5: (np.eye(4) + 0.1).tolist()}, "000001": {2: np.diag([1.0, 1, 1, 1]).tolist()}},
           0: {"000003": {2: (2 * np.eye(4)).tolist()}}}
    path = tmp_path / "linemod_res.yml"
    path.write_text(yaml.safe_dump(res))
    return str(path)


def test_result_walk_groups_by_object_and_flags_skipped_frames(tmp_path):
    import eval_bop_results as ev

    groups = ev.group_by_object(ev.load_results(_result_file(tmp_path)))
    assert list(groups) == [2, 5]
    assert [(v, s, skip) for v, s, _, skip in groups[2]] == [(0, "000003", False), (1, "000000", True), (1, "000001", True)]
    assert [(v, s, skip) for v, s, _, skip in groups[5]] == [(1, "000000", False)]
    np.testing.assert_array_equal(groups[2][0][2], 2 * np.eye(4))


def test_rows_count_skipped_frames_as_failures():
    import eval_bop_results as ev

    add = np.array([0.001, np.inf, 0.05])
    adds = np.array([0.001, np.inf, 0.002])
    row = ev.summarize(add, adds, symmetric=False, diameter=0.2)
    assert row["poses"] == 3
    assert row["add_s_recall"] == pytest.approx(1 / 3)
    assert ev.summarize(add, adds, symmetric=True, diameter=0.2)["add_s_recall"] == pytest.approx(2 / 3)
    assert row["add_auc"] < ev.summarize(add[:1], adds[:1], False, 0.2)["add_auc"]
    overall = ev.summarize_all({1: row, 2: ev.summarize(adds, add, True, 0.01)}, {1: (add, adds), 2: (adds, add)})
    # object 1 by ADD under 0.02 m: 1 of 3; object 2 by ADD-S (= `add` here) under 0.001 m: 0 of 3
    assert overall["poses"] == 6 and overall["add_s_recall"] == pytest.approx(1 / 6)


def test_symmetric_objects_of_a_synthetic_dataset(tmp_path):
    import eval_bop_results as ev

    from foundationpose_b200 import synth

    synth.write_bop_dataset(str(tmp_path / "LM"), "lm", n_frames=1, symmetric=(6,))
    reader = ev.make_reader_factory("lm", str(tmp_path / "LM"))(2)
    sym = [ob_id for ob_id in reader.ob_ids if ev.is_symmetric(reader.symmetry_tfs[ob_id])]
    assert sym == [6]
    assert not ev.is_symmetric(np.eye(4)[None])
