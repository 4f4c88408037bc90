"""GPU: ADD / ADD-S of fp_pose_errors (metrics.pose_errors, the drop-in's add_err / adds_err) against the reference's own
add_err / adds_err (tests/golden/metrics_golden.npz) and against float64 numpy + cKDTree; exactness on identical
poses, symmetry, determinism and batch invariance, argument checks, and examples/eval_bop_results.py end to end."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch
import yaml
from scipy.spatial import cKDTree

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "examples"), os.path.join(ROOT, "foundationpose_b200", "dropin"), ROOT]
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "metrics_golden.npz"))
SETS = sorted({k.split("/")[1] for k in GOLDEN.files if k.startswith("pose/")})
ATOL, RTOL = 1e-6, 1e-5


def _close(got, want):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert np.all(np.abs(got - want) <= ATOL + RTOL * np.abs(want)), np.abs(got - want).max()


def _random_poses(rng, n, t=(0.0, 0.0, 0.6), rot_deg=180.0, trans=0.05):
    from scipy.spatial.transform import Rotation

    out = np.repeat(np.eye(4)[None], n, axis=0)
    rv = rng.normal(size=(n, 3))
    rv *= (np.deg2rad(rot_deg) * rng.uniform(0, 1, size=(n, 1))) / np.linalg.norm(rv, axis=1, keepdims=True)
    out[:, :3, :3] = Rotation.from_rotvec(rv).as_matrix()
    out[:, :3, 3] = np.asarray(t) + rng.uniform(-trans, trans, size=(n, 3))
    return out.astype(np.float32)


def _reference(pts, pred, gt):
    """float64 numpy + cKDTree, the reference's formulas."""
    pts = pts.astype(np.float64)
    add, adds = [], []
    for p, g in zip(pred.astype(np.float64), np.broadcast_to(gt.astype(np.float64), pred.shape)):
        a, b = pts @ p[:3, :3].T + p[:3, 3], pts @ g[:3, :3].T + g[:3, 3]
        add.append(np.linalg.norm(a - b, axis=1).mean())
        adds.append(cKDTree(a).query(b, k=1)[0].mean())
    return np.array(add), np.array(adds)


@pytest.mark.parametrize("name", SETS)
def test_golden_from_reference(name):
    import Utils

    from foundationpose_b200 import metrics

    pts, pred, gt = (GOLDEN[f"pose/{name}/{k}"] for k in ("pts", "pred", "gt"))
    add, adds = metrics.pose_errors(pts, pred, gt)
    _close(add.cpu().numpy(), GOLDEN[f"pose/{name}/add"])
    _close(adds.cpu().numpy(), GOLDEN[f"pose/{name}/adds"])
    # ADD alone / ADD-S alone give the same bits as both together
    assert torch.equal(metrics.pose_errors(pts, pred, gt[0], adds=False)[0], add)
    assert torch.equal(metrics.pose_errors(pts, pred, gt[0], add=False)[1], adds)
    for i in range(len(pred)):
        assert Utils.add_err(pred[i], gt[i], pts) == pytest.approx(GOLDEN[f"pose/{name}/add"][i], rel=RTOL, abs=ATOL)
        assert Utils.adds_err(pred[i], gt[i], pts) == pytest.approx(GOLDEN[f"pose/{name}/adds"][i], rel=RTOL, abs=ATOL)
    assert add[0].item() == 0.0 and adds[0].item() == 0.0  # the first estimate is the ground truth itself


@pytest.mark.parametrize("n_gt", [1, 252])
def test_252_hypotheses_against_float64(n_gt):
    from foundationpose_b200 import metrics

    rng = np.random.default_rng(7)
    pts = (rng.normal(size=(4099, 3)) * [0.05, 0.03, 0.09]).astype(np.float32)
    gt = _random_poses(rng, n_gt)
    # small perturbations of the ground truth, then arbitrary poses
    near = _random_poses(rng, 126, t=(0, 0, 0), rot_deg=10.0, trans=0.01) @ np.broadcast_to(gt, (252, 4, 4))[:126]
    pred = np.concatenate([near.astype(np.float32), _random_poses(rng, 126)])
    add, adds = metrics.pose_errors(pts, pred, gt)
    want_add, want_adds = _reference(pts, pred, gt)
    _close(add.cpu().numpy(), want_add)
    _close(adds.cpu().numpy(), want_adds)


def test_identity_and_symmetry():
    from foundationpose_b200 import metrics, synth

    pts = synth.make_mesh(4, tex_size=8).vertices.astype(np.float32)  # ellipsoid: invariant under a half turn about z
    gt = _random_poses(np.random.default_rng(3), 5)
    add, adds = metrics.pose_errors(pts, gt, gt)
    assert torch.count_nonzero(add).item() == 0 and torch.count_nonzero(adds).item() == 0
    flipped = (gt.astype(np.float64) @ np.diag([-1.0, -1.0, 1.0, 1.0])).astype(np.float32)
    add, adds = metrics.pose_errors(pts, flipped, gt)
    assert adds.max().item() < 1e-6
    assert add.min().item() > 0.03


def test_deterministic_and_batch_invariant():
    from foundationpose_b200 import metrics

    rng = np.random.default_rng(11)
    pts = (rng.normal(size=(2620, 3)) * [0.05, 0.03, 0.09]).astype(np.float32)
    gt = _random_poses(rng, 1)
    pred = _random_poses(rng, 252)
    a1, s1 = metrics.pose_errors(pts, pred, gt)
    a2, s2 = metrics.pose_errors(pts, pred, gt)
    assert torch.equal(a1, a2) and torch.equal(s1, s2)
    for i in (0, 97, 251):
        a, s = metrics.pose_errors(pts, pred[i], gt)
        assert torch.equal(a, a1[i:i + 1]) and torch.equal(s, s1[i:i + 1])
    a, s = metrics.pose_errors(pts, pred, np.repeat(gt, 252, axis=0))  # one ground truth per pose: same bits
    assert torch.equal(a, a1) and torch.equal(s, s1)
    a, s = metrics.pose_errors(pts, pred[:0], gt)
    assert a.shape == (0,) and s.shape == (0,)


def test_bad_arguments_raise_and_leave_the_device_usable():
    from foundationpose_b200 import _lib, metrics

    lib = _lib.lib
    dev = torch.device("cuda")
    pts = torch.zeros(10, 3, device=dev)
    pred = torch.eye(4, device=dev).reshape(1, 16).repeat(3, 1)
    out = torch.empty(3, device=dev)
    host_pts = np.zeros((10, 3), dtype=np.float32)
    host_out = np.zeros(3, dtype=np.float32)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    h = lambda a: C.c_void_p(a.ctypes.data)  # noqa: E731
    bad = {
        "null pts": (None, 10, p(pred), 3, p(pred), 1, p(out), p(out)),
        "null pred": (p(pts), 10, None, 3, p(pred), 1, p(out), p(out)),
        "null gt": (p(pts), 10, p(pred), 3, None, 1, p(out), None),
        "P = 0": (p(pts), 0, p(pred), 3, p(pred), 1, p(out), p(out)),
        "P too large": (p(pts), 131073, p(pred), 3, p(pred), 1, p(out), p(out)),
        "N < 0": (p(pts), 10, p(pred), -1, p(pred), 1, p(out), p(out)),
        "n_gt not 1 or N": (p(pts), 10, p(pred), 3, p(pred), 2, p(out), p(out)),
        "host pts": (h(host_pts), 10, p(pred), 3, p(pred), 1, p(out), p(out)),
        "host add_out": (p(pts), 10, p(pred), 3, p(pred), 1, h(host_out), None),
        "host adds_out": (p(pts), 10, p(pred), 3, p(pred), 1, None, h(host_out)),
    }
    for what, args in bad.items():
        rc = lib.fp_pose_errors(*args, st)
        assert rc != 0, what
        with pytest.raises(_lib.FposeError, match="fp_pose_errors"):
            _lib.check(rc, "fp_pose_errors")
    with pytest.raises(_lib.FposeError, match="n_gt"):
        metrics.pose_errors(pts, pred, pred[:2])
    torch.cuda.synchronize()
    add, adds = metrics.pose_errors(pts + 1, pred, pred[0])
    assert add.sum().item() == 0.0 and adds.sum().item() == 0.0


def test_eval_bop_results_on_a_synthetic_dataset(tmp_path):
    """Ground truth shifted by k mm in frame k: every ADD is k mm; AUC and recall as computed here."""
    import eval_bop_results as ev

    from foundationpose_b200 import metrics, synth

    root = str(tmp_path / "LINEMOD")
    gts = synth.write_bop_dataset(root, "lm", n_frames=4, symmetric=(6,))
    res = {}
    for (vid, id_str, ob_id), pose in gts.items():
        k = int(id_str)
        p = np.array(pose, dtype=np.float64)
        p[:3, 3] += np.array([0.6, 0.0, 0.8]) * 0.001 * k
        res.setdefault(vid, {}).setdefault(id_str, {})[ob_id] = p.tolist()
    res[1]["000003"][1] = np.eye(4).tolist()  # a frame the driver skipped
    path = tmp_path / "linemod_res.yml"
    path.write_text(yaml.safe_dump(res))
    rows, overall = ev.main(["--res", str(path), "--dataset_dir", root, "--json", str(tmp_path / "t.json")])
    _, _, errors = ev.evaluate(ev.load_results(str(path)), "lm", root)
    reader = ev.make_reader_factory("lm", root)(2)
    assert [o for o in rows if rows[o]["symmetric"]] == [6]
    all_crit, all_thr = [], []
    for ob_id, row in rows.items():
        add, adds = errors[ob_id]
        want = np.array([0.0, 0.001, 0.002, 0.003])
        if ob_id == 1:
            assert add[3] == np.inf and adds[3] == np.inf
            add, adds, want = add[:3], adds[:3], want[:3]
        assert np.all(np.abs(add - want) <= 1e-6), (ob_id, add)
        assert np.all(adds <= add + 1e-6)
        assert row["poses"] == 4
        full_add, full_adds = errors[ob_id]
        assert row["add_auc"] == metrics.auc(full_add) and row["adds_auc"] == metrics.auc(full_adds)
        d = reader.get_model_diameter(ob_id)
        crit = full_adds if ob_id == 6 else full_add
        assert row["add_s_recall"] == np.mean(crit < 0.1 * d)
        all_crit.append(crit)
        all_thr.append(np.full(4, 0.1 * d))
    assert overall["poses"] == 4 * len(rows)
    assert overall["add_s_recall"] == pytest.approx(np.mean(np.concatenate(all_crit) < np.concatenate(all_thr)))
    assert overall["add_auc"] == pytest.approx(metrics.auc(np.concatenate([errors[o][0] for o in rows])))
    assert os.path.exists(tmp_path / "t.json")
