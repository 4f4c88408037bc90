"""CPU: estimater.register_objects' host logic through an engine double (slots shared with track_objects, reload after
reset_object, per-object ranking, the model_center shift, the early exit, refusals), and the grids of the
register_objects golden."""
import os

import numpy as np
import pytest
import torch

from foundationpose_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W = 6, 8


class _Refiner:
    last_trans_update = last_rot_update = "stale"


class _Engine:
    """Stands in for engine.Engine: records mesh uploads and calls.  register_objects gives hypothesis j of object i the
    pose "grid row j moved to x = i" and the score `scores[i][j]`; info = (i, 0, 0.5, n_valid[i])."""

    def __init__(self, scores=None, n_valid=None):
        self.uploads, self.calls = [], []
        self.scores, self.n_valid = scores, n_valid

    def set_mesh(self, pos, normals, faces, diameter, uv=None, tex=None, vertex_colors=None, slot=0):
        self.uploads.append((slot, len(pos), float(diameter)))

    def register_objects(self, rgb, depth, K, masks, rot_grids, slots, iterations):
        self.calls.append(("register", list(slots), [len(g) for g in rot_grids], iterations, masks.shape))
        poses = torch.cat([g.clone() for g in rot_grids])
        scores, o = [], 0
        for i, g in enumerate(rot_grids):
            poses[o:o + len(g), 0, 3] = float(i)
            scores.append(torch.as_tensor(self.scores[i], dtype=torch.float32) if self.scores else torch.zeros(len(g)))
            o += len(g)
        n_valid = self.n_valid or [100] * len(slots)
        info = torch.tensor([[float(i), 0.0, 0.5, float(n_valid[i])] for i in range(len(slots))])
        return poses, torch.cat(scores), torch.zeros(len(slots), dtype=torch.int32), info

    def track_objects(self, rgb, depth, K, poses_in, slots, iterations):
        self.calls.append(("track", list(slots)))
        return poses_in.clone(), poses_in.numpy().copy()


def _est(engine, n_verts, n_hyp, center=(0.0, 0.0, 0.0)):
    from foundationpose_b200.estimater import FoundationPose

    est = FoundationPose.__new__(FoundationPose)
    est.engine = engine
    est.refiner = _Refiner()
    est.mesh_tensors = dict(pos=np.zeros((n_verts, 3), np.float32), normals=np.zeros((n_verts, 3), np.float32),
                            faces=np.zeros((1, 3), np.int32), vcolor=np.zeros((n_verts, 3), np.float32))
    est.diameter = 0.1 * n_verts
    est.model_center = np.asarray(center, dtype=np.float64)
    est.strict_early_out = False
    grid = torch.eye(4).repeat(n_hyp, 1, 1)
    for j in range(n_hyp):
        grid[j, :3, :3] = torch.from_numpy(synth.random_rotation(j)).float()
    est.rot_grid = grid
    tf = torch.eye(4)
    tf[:3, 3] = -torch.as_tensor(est.model_center, dtype=torch.float32)
    est.get_tf_to_centered_mesh = lambda: tf  # the real one builds it on the GPU
    est.pose_last = None
    return est


def _frame():
    masks = [np.zeros((H, W), bool) for _ in range(3)]
    return np.zeros((H, W, 3), np.uint8), np.zeros((H, W), np.float32), masks


def test_slots_shared_with_track_objects_and_reloaded_after_reset():
    from foundationpose_b200.estimater import register_objects, track_objects

    e = _Engine()
    a, b = _est(e, 3, 4), _est(e, 4, 2)
    rgb, depth, masks = _frame()
    register_objects([a, b], synth.DEFAULT_K, rgb, depth, masks[:2], iteration=3)
    assert e.uploads == [(1, 3, pytest.approx(0.3)), (2, 4, pytest.approx(0.4))]
    assert e.calls == [("register", [1, 2], [4, 2], 3, (2, H, W))]
    track_objects([b, a], rgb, depth, synth.DEFAULT_K)
    assert e.calls[-1] == ("track", [2, 1]) and len(e.uploads) == 2, "tracking after registering uploads no mesh"
    b.mesh_tensors = dict(b.mesh_tensors, pos=np.zeros((5, 3), np.float32))  # what reset_object does: new mesh tensors
    register_objects([a, b], synth.DEFAULT_K, rgb, depth, masks[:2])
    assert e.uploads[-1][:2] == (2, 5) and len(e.uploads) == 3
    assert e.calls[-1][3] == 5, "iteration defaults to register()'s 5"


def test_ranking_per_object_and_model_center_shift():
    from foundationpose_b200.estimater import register_objects

    scores = [[0.1, 0.9, 0.5], [2.0, -1.0], [0.3, 0.7, 0.2, 0.6]]
    e = _Engine(scores=scores)
    c = (0.01, -0.02, 0.03)
    ests = [_est(e, 3, 3, center=c), _est(e, 4, 2), _est(e, 5, 4)]
    rgb, depth, masks = _frame()
    out = register_objects(ests, synth.DEFAULT_K, rgb, depth, masks, ob_ids=[7, 8, 9])
    for i, est in enumerate(ests):
        order = np.argsort(-np.asarray(scores[i]), kind="stable")
        assert int(est.best_id) == order[0]
        assert torch.equal(est.scores, torch.tensor(scores[i], dtype=torch.float32)[order])
        want_poses = est.rot_grid[order].clone()
        want_poses[:, 0, 3] = float(i)
        assert torch.equal(est.poses, want_poses) and torch.equal(est.pose_last, want_poses[0])
        want = (want_poses[0] @ est.get_tf_to_centered_mesh()).numpy()
        assert np.array_equal(out[i], want) and out[i].dtype == np.float32
        assert (est.H, est.W, est.ob_id) == (H, W, 7 + i) and est.ob_mask is masks[i] and est.K is synth.DEFAULT_K
        assert est.refiner.last_trans_update is None and est.refiner.last_rot_update is None
    best0 = ests[0].rot_grid[int(np.argmax(scores[0]))].numpy().astype(np.float64)
    best0[0, 3] = 0.0
    assert np.allclose(out[0][:3, 3], best0[:3, 3] - best0[:3, :3] @ np.asarray(c), atol=1e-7), "pose of the un-centred mesh"


def test_early_exit_leaves_state_untouched():
    from foundationpose_b200.estimater import register_objects

    e = _Engine(scores=[[0.0, 1.0], [1.0, 0.0]], n_valid=[3, 50])
    a, b = _est(e, 3, 2), _est(e, 4, 2)
    a.pose_last, a.best_id, a.poses, a.scores = "last", "id", "poses", "scores"
    rgb, depth, masks = _frame()
    out = register_objects([a, b], synth.DEFAULT_K, rgb, depth, masks[:2])
    want = np.eye(4)
    want[:3, 3] = [0.0, 0.0, 0.5]
    assert np.array_equal(out[0], want) and out[0].dtype == np.float64
    assert (a.pose_last, a.best_id, a.poses, a.scores) == ("last", "id", "poses", "scores")
    assert a.H == H and a.ob_mask is masks[0], "the sync-free register() records the frame before its early exit"
    assert int(b.best_id) == 0 and out[1][0, 3] == 1.0
    strict = _est(_Engine(n_valid=[0]), 3, 2)
    strict.strict_early_out = True
    register_objects([strict], synth.DEFAULT_K, rgb, depth, masks[:1])
    assert not hasattr(strict, "H") and strict.pose_last is None, "the strict register() returns before recording the frame"


def test_refusals():
    from foundationpose_b200.estimater import MAX_MESHES, register_objects

    e = _Engine()
    rgb, depth, masks = _frame()
    K = synth.DEFAULT_K
    assert register_objects([], K, rgb, depth, []) == []
    a = _est(e, 3, 2)
    with pytest.raises(ValueError):
        register_objects([a, _est(_Engine(), 3, 2)], K, rgb, depth, masks[:2])
    with pytest.raises(ValueError):
        register_objects([a, a], K, rgb, depth, masks[:2])
    with pytest.raises(ValueError):
        register_objects([_est(e, 3, 2) for _ in range(MAX_MESHES)], K, rgb, depth, masks * MAX_MESHES)
    with pytest.raises(TypeError):
        register_objects([a], K, torch.zeros(H, W, 3, dtype=torch.uint8), torch.zeros(H, W), masks[:1])
    with pytest.raises(ValueError):
        register_objects([a], K, rgb, depth, masks[:2])
    with pytest.raises(ValueError):
        register_objects([a], K, rgb, depth, [np.zeros((H, W + 1), bool)])
    with pytest.raises(ValueError):
        register_objects([a], K, rgb, depth, masks[:1], ob_ids=[1, 2])
    assert e.calls == [] and e.uploads == [], "every error is raised before anything reaches the engine"


def test_golden_grids_are_the_symmetry_reduced_grids():
    import sys

    from foundationpose_b200 import hypotheses

    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_golden_register_objects as gen

    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "register_objects.npz")))
    tfs = np.split(g["symmetry_tfs"], np.cumsum(g["symmetry_counts"])[:-1])
    assert list(g["n_hyp"]) == [126, 63, 20]
    o = 0
    for k, name in enumerate(g["symmetries"]):
        assert np.array_equal(tfs[k], gen.symmetry_tfs(str(name)))
        grid = hypotheses.make_rotation_grid(40, 60, tfs[k])
        assert len(grid) == g["n_hyp"][k]
        assert np.abs(g["start"][o:o + len(grid), :3, :3] - grid[:, :3, :3]).max() == 0
        o += len(grid)
    assert len(g["scores"]) == o and (g["top2_margin"] >= gen.MIN_MARGIN_SPREAD * g["spread"]).all()
