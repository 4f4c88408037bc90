"""CPU: BOP's symmetry sets (metrics.bop_symmetries) from models_info.json entries, the average recall of MSSD / MSPD,
and the host side of `examples/eval_bop_results.py --bop`: per-object thresholds, skipped frames as failures and the
unchanged table without --bop."""
import math
import os
import sys

import numpy as np
import pytest
from scipy.spatial import cKDTree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "examples"), os.path.join(ROOT, "foundationpose_b200", "dropin"), ROOT]

N_STEPS = 315  # ceil(pi / 0.01)


def _rotation(axis, angle):
    from scipy.spatial.transform import Rotation

    a = np.asarray(axis, dtype=np.float64)
    return Rotation.from_rotvec(a / np.linalg.norm(a) * angle).as_matrix()


def _rigid_mm(R, offset_mm):
    """The 4x4 rotation R about an axis through `offset_mm`, translation in millimetres (models_info.json units)."""
    m = np.eye(4)
    m[:3, :3] = R
    m[:3, 3] = np.asarray(offset_mm) - R @ np.asarray(offset_mm)
    return m


def _cylinder(axis, offset_m, n_ring=N_STEPS, radii=(0.02, 0.035), heights=(-0.03, -0.01, 0.01, 0.03)):
    """Points on rings about `axis` through `offset_m`, one point every 2 pi / n_ring: invariant (as a set) under every
    continuous step and under a half turn about the first frame vector u (heights are symmetric about 0)."""
    a = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    u = np.cross(a, [1.0, 0.0, 0.0] if abs(a[0]) < 0.9 else [0.0, 1.0, 0.0])
    u /= np.linalg.norm(u)
    v = np.cross(a, u)
    th = np.arange(n_ring) * 2.0 * np.pi / n_ring
    pts = [np.asarray(offset_m) + r * (np.cos(t) * u + np.sin(t) * v) + h * a for r in radii for h in heights for t in th]
    return np.array(pts), u


def test_counts_identity_first_and_millimetres():
    from foundationpose_b200 import metrics

    flip = _rigid_mm(_rotation([1, 0, 0], np.pi), [0.0, 12.0, -4.0])
    quarter = _rigid_mm(_rotation([0, 0, 1], np.pi / 2), [3.0, 0.0, 0.0])
    assert metrics.bop_symmetries({}).shape == (1, 4, 4)
    for k, disc in enumerate([[], [flip], [flip, quarter]]):
        info = {"diameter": 100.0, "symmetries_discrete": [d.reshape(-1).tolist() for d in disc]}
        syms = metrics.bop_symmetries(info)
        assert syms.shape == (1 + k, 4, 4) and syms.dtype == np.float64
        np.testing.assert_array_equal(syms[0], np.eye(4))
        for d, s in zip(disc, syms[1:]):
            np.testing.assert_array_equal(s[:3, :3], d[:3, :3])
            np.testing.assert_allclose(s[:3, 3], d[:3, 3] * 1e-3, rtol=0, atol=1e-15)  # mm -> m
        info["symmetries_continuous"] = [{"axis": [0, 0, 1], "offset": [0, 0, 0]}]
        syms = metrics.bop_symmetries(info)
        assert syms.shape == (N_STEPS * (1 + k), 4, 4)
        np.testing.assert_array_equal(syms[0], np.eye(4))
    # a coarser step: n = ceil(pi / step)
    assert len(metrics.bop_symmetries({"symmetries_continuous": [{"axis": [0, 1, 0], "offset": [0, 0, 0]}]}, 0.5)) == 7


@pytest.mark.parametrize("axis, offset_mm", [([0, 0, 1], [0.0, 0.0, 0.0]), ([1, 2, 2], [10.0, -20.0, 5.0])])
def test_every_transform_maps_a_symmetric_model_onto_itself(axis, offset_mm):
    from foundationpose_b200 import metrics

    offset_m = np.asarray(offset_mm) * 1e-3
    pts, u = _cylinder(axis, offset_m)
    flip = _rigid_mm(_rotation(u, np.pi), offset_mm)  # half turn about u through the offset
    info = {"symmetries_continuous": [{"axis": list(axis), "offset": list(offset_mm)}],
            "symmetries_discrete": [flip.reshape(-1).tolist()]}
    syms = metrics.bop_symmetries(info)
    assert syms.shape == (2 * N_STEPS, 4, 4)
    tree = cKDTree(pts)
    worst = max(tree.query(pts @ s[:3, :3].T + s[:3, 3], k=1)[0].max() for s in syms)
    assert worst < 1e-12, worst
    # and they are N_STEPS * 2 distinct transforms
    assert len({tuple(np.round(s, 9).reshape(-1)) for s in syms}) == len(syms)
    # rotation steps of exactly 2 pi / 315 about the axis: trace = 1 + 2 cos(i 2 pi / 315)
    ang = np.arccos(np.clip((np.trace(syms[:N_STEPS, :3, :3], axis1=1, axis2=2) - 1) / 2, -1, 1))
    want = np.minimum(np.arange(N_STEPS), N_STEPS - np.arange(N_STEPS)) * 2 * math.pi / N_STEPS
    np.testing.assert_allclose(ang, want, atol=1e-7)


def test_average_recall_by_hand():
    from foundationpose_b200 import metrics

    errs = [0.01, 0.03, np.inf, 0.2]
    # shares below 0.02, 0.05, 0.5: 1/4, 2/4, 3/4
    assert metrics.average_recall(errs, [0.02, 0.05, 0.5]) == pytest.approx(0.5, abs=1e-15)
    # one column of thresholds per error: error j against thresholds[:, j]; rows pass 0.01, then 0.01 and 0.2
    thr = np.array([[0.02, 0.02, 1.0, 0.1], [0.04, 0.02, 1.0, 0.3]])
    assert metrics.average_recall(errs, thr) == pytest.approx((1 / 4 + 2 / 4) / 2, abs=1e-15)
    assert metrics.average_recall([0.0], [0.0]) == 0.0  # strictly below
    np.testing.assert_allclose(metrics.mssd_thresholds(0.2), 0.2 * np.arange(1, 11) * 0.05, rtol=0, atol=1e-15)
    np.testing.assert_allclose(metrics.mspd_thresholds(640), np.arange(5, 55, 5), rtol=0, atol=1e-12)
    np.testing.assert_allclose(metrics.mspd_thresholds(1280), np.arange(5, 55, 5) / 2, rtol=0, atol=1e-12)


def test_evaluator_thresholds_per_object_and_skipped_frames():
    import eval_bop_results as ev

    from foundationpose_b200 import metrics

    mssd_thr, mspd_thr = ev.bop_thresholds(0.1, [640, 1280, 640])
    assert mssd_thr.shape == (10, 3) and mspd_thr.shape == (10, 3)
    np.testing.assert_array_equal(mssd_thr[:, 1], metrics.mssd_thresholds(0.1))
    np.testing.assert_array_equal(mspd_thr[:, 1], metrics.mspd_thresholds(1280))
    # object 1 (d = 0.1 m): MSSD 4 mm passes 0.05 d on, 12 mm from 0.15 d on, the skipped frame never
    e1 = (None, None, np.array([0.004, 0.012, np.inf]), np.array([1.0, 12.0, np.inf]))
    row = ev.summarize_bop(e1[2], e1[3], (mssd_thr, mspd_thr))
    assert row["mssd_ar"] == pytest.approx((10 + 8) / 30)
    # MSPD 1 px < every threshold; 12 px at width 1280 (2.5 .. 25 px) passes 12.5 px on: 6 of 10
    assert row["mspd_ar"] == pytest.approx((10 + 6) / 30)
    # object 2 (d = 0.01 m): 4 mm passes 0.45 d and 0.5 d only
    e2 = (None, None, np.array([0.004]), np.array([100.0]))
    thr2 = ev.bop_thresholds(0.01, [640])
    overall = ev.summarize_bop_all({1: e1, 2: e2}, {1: (mssd_thr, mspd_thr), 2: thr2})
    assert overall["mssd_ar"] == pytest.approx((10 + 8 + 2) / 40)
    assert overall["mspd_ar"] == pytest.approx((10 + 6 + 0) / 40)


def test_table_without_bop_is_unchanged(capsys):
    import eval_bop_results as ev

    rows = {2: {"poses": 3, "add_auc": 0.5, "adds_auc": 0.75, "add_s_recall": 1 / 3, "symmetric": False, "diameter": 0.1},
            6: {"poses": 1, "add_auc": 0.0, "adds_auc": 1.0, "add_s_recall": 1.0, "symmetric": True, "diameter": 0.1}}
    overall = {"poses": 4, "add_auc": 0.375, "adds_auc": 0.8125, "add_s_recall": 0.5}
    ev.print_table(rows, overall)
    assert capsys.readouterr().out.splitlines() == [
        "  object  poses  ADD AUC  ADD-S AUC  ADD(-S)<0.1d",
        "       2      3    50.00      75.00         33.33",
        "      6*      1     0.00     100.00        100.00",
        "     all      4    37.50      81.25         50.00",
        "(percent; * = symmetric object, scored by ADD-S in the last column)"]
    for r in list(rows.values()) + [overall]:
        r.update(mssd_ar=0.25, mspd_ar=0.5)
    ev.print_table(rows, overall, bop=True)
    out = capsys.readouterr().out.splitlines()
    assert out[0].split()[-4:] == ["AR", "MSSD", "AR", "MSPD"]
    assert out[3].split() == ["all", "4", "37.50", "81.25", "50.00", "25.00", "50.00"]
    assert "without VSD" in out[-1]
