"""CPU: estimater.register_cameras' host logic through an engine double (grouping by camera, slots shared with
register_objects / track_cameras, per-camera result shape, per-camera frame state, the early exit, refusals), and the rig
of the register_cameras golden."""
import os

import numpy as np
import pytest
import torch

from foundationpose_b200 import synth
from test_register_objects_cpu import _Engine as _ObjectsEngine
from test_register_objects_cpu import _est

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Engine(_ObjectsEngine):
    """register_cameras gives hypothesis j of object i the pose "grid row j moved to x = i" and the score scores[i][j],
    info = (i, 0, 0.5, n_valid[i]), as register_objects of the double does for one camera."""

    def register_cameras(self, frames, masks, rot_grids, camera_of, slots, iterations):
        self.calls.append(("cameras", [np.shape(d) for _, d, _ in frames], list(camera_of), list(slots), [len(g) for g in rot_grids],
                           iterations, [m.shape for m in masks]))
        out = _ObjectsEngine.register_objects(self, None, None, None, np.zeros(0), rot_grids, slots, iterations)
        del self.calls[-1]  # the call the one-camera double recorded
        return out

    def track_cameras(self, frames, poses_in, camera_of, slots, iterations):
        self.calls.append(("track", list(slots)))
        return poses_in.clone(), poses_in.numpy().copy()


def _view(ests, H, W, K=synth.DEFAULT_K):
    return (ests, np.zeros((H, W, 3), np.uint8), np.zeros((H, W), np.float32), K, [np.zeros((H, W), bool) for _ in ests])


def test_grouping_slots_and_result_shape():
    from foundationpose_b200.estimater import register_cameras, track_cameras

    e = _Engine()
    a, b, c = _est(e, 3, 4), _est(e, 4, 2), _est(e, 5, 3)
    K1 = np.array([[300.0, 0, 100.0], [0, 300.0, 80.0], [0, 0, 1]])
    views = [_view([a, b], 6, 8), _view([], 3, 3), _view([c], 5, 7, K1)]
    out = register_cameras(views, ob_ids=[[7, 8], None, [9]], iteration=3)
    assert [len(v) for v in out] == [2, 0, 1]
    assert e.uploads == [(1, 3, pytest.approx(0.3)), (2, 4, pytest.approx(0.4)), (3, 5, pytest.approx(0.5))]
    # the camera without estimators is not uploaded: camera ids count the cameras with objects only
    assert e.calls == [("cameras", [(6, 8), (5, 7)], [0, 0, 1], [1, 2, 3], [4, 2, 3], 3, [(6, 8), (6, 8), (5, 7)])]
    assert (a.H, a.W, a.ob_id, b.ob_id, c.H, c.W, c.ob_id) == (6, 8, 7, 8, 5, 7, 9)
    assert a.K is synth.DEFAULT_K and c.K is K1 and c.ob_mask is views[2][4][0]
    for i, est in enumerate((a, b, c)):  # every object ranked on its own rows
        assert torch.equal(est.pose_last[0, 3], torch.tensor(float(i)))
    track_cameras([(ests, rgb, depth, K) for ests, rgb, depth, K, _ in views])
    assert len(e.uploads) == 3, "tracking after registering uploads no mesh"
    assert register_cameras([_view([], 2, 2)]) == [[]] and register_cameras([]) == []
    assert register_cameras(views[:1], iteration=5)[0][0].shape == (4, 4) and e.calls[-1][5] == 5


def test_equals_register_objects_per_view():
    from foundationpose_b200.estimater import register_cameras, register_objects

    scores = [[0.1, 0.9, 0.5], [2.0, -1.0], [0.3, 0.7, 0.2, 0.6]]

    def run(per_view):
        e = _Engine(scores=scores)
        ests = [_est(e, 3, 3, center=(0.01, -0.02, 0.03)), _est(e, 4, 2), _est(e, 5, 4)]
        views = [_view(ests[:2], 6, 8), _view(ests[2:], 4, 5)]
        if per_view:
            e.scores = scores[:2]
            got = [register_objects(views[0][0], views[0][3], views[0][1], views[0][2], views[0][4])]
            e.scores = scores[2:]
            got.append(register_objects(views[1][0], views[1][3], views[1][1], views[1][2], views[1][4]))
        else:
            got = register_cameras(views)
        return got, [(est.pose_last, int(est.best_id), est.poses, est.scores, est.H, est.W) for est in ests]

    (a, sa), (b, sb) = run(False), run(True)
    for x, y in zip(sum(a, []), sum(b, [])):
        assert np.array_equal(x[:3, :3], y[:3, :3]) and x.dtype == y.dtype
    for x, y in zip(sa, sb):
        assert torch.equal(x[0][:3, :3], y[0][:3, :3]) and x[1] == y[1] and torch.equal(x[3], y[3]) and x[4:] == y[4:]


def test_early_exit_leaves_state_untouched():
    from foundationpose_b200.estimater import register_cameras

    e = _Engine(scores=[[0.0, 1.0], [1.0, 0.0]], n_valid=[50, 3])
    a, b = _est(e, 3, 2), _est(e, 4, 2)
    b.pose_last, b.best_id, b.poses, b.scores = "last", "id", "poses", "scores"
    out = register_cameras([_view([a], 6, 8), _view([b], 4, 5)])
    want = np.eye(4)
    want[:3, 3] = [1.0, 0.0, 0.5]
    assert np.array_equal(out[1][0], want) and out[1][0].dtype == np.float64
    assert (b.pose_last, b.best_id, b.poses, b.scores) == ("last", "id", "poses", "scores")
    assert (b.H, b.W) == (4, 5), "the sync-free register() records the frame before its early exit"
    assert int(a.best_id) == 1
    strict = _est(_Engine(n_valid=[0]), 3, 2)
    strict.strict_early_out = True
    register_cameras([_view([strict], 6, 8)])
    assert not hasattr(strict, "H") and strict.pose_last is None, "the strict register() returns before recording the frame"


def test_refusals():
    from foundationpose_b200.estimater import MAX_CAMERAS, MAX_MESHES, register_cameras

    e = _Engine()
    a, b = _est(e, 3, 2), _est(e, 4, 2)
    with pytest.raises(ValueError):  # mixed engines
        register_cameras([_view([a], 6, 8), _view([_est(_Engine(), 3, 2)], 4, 5)])
    with pytest.raises(ValueError):  # one estimator in two cameras
        register_cameras([_view([a], 6, 8), _view([a], 4, 5)])
    with pytest.raises(ValueError):  # one estimator twice in one camera
        register_cameras([_view([a, a], 6, 8)])
    with pytest.raises(ValueError):
        register_cameras([_view([_est(e, 3, 2) for _ in range(MAX_MESHES)], 2, 2)])
    with pytest.raises(ValueError):
        register_cameras([_view([_est(e, 3, 2)], 2, 2) for _ in range(MAX_CAMERAS + 1)])
    bad = _view([a, b], 6, 8)
    with pytest.raises(ValueError):  # a mask of another size than its camera's frame
        register_cameras([bad[:4] + ([bad[4][0], np.zeros((6, 9), bool)],)])
    with pytest.raises(ValueError):
        register_cameras([bad[:4] + (bad[4][:1],)])
    with pytest.raises(ValueError):
        register_cameras([bad], ob_ids=[[1]])
    with pytest.raises(ValueError):
        register_cameras([bad], ob_ids=[None, None])
    with pytest.raises(TypeError):
        register_cameras([(bad[0], torch.zeros(6, 8, 3, dtype=torch.uint8), torch.zeros(6, 8), bad[3], bad[4])])
    assert e.calls == [] and e.uploads == [], "every error is raised before anything reaches the engine"


def test_golden_rig():
    import sys

    from foundationpose_b200 import hypotheses

    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_golden_register_cameras as gen

    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "register_cameras.npz")))
    assert list(g["H"]) == [480, 300] and list(g["W"]) == [640, 400] and g["W"][1] % 32 and g["H"][1] % 8 == 4
    assert np.array_equal(g["K"][0], synth.DEFAULT_K) and not np.array_equal(g["K"][1], g["K"][0])
    assert list(g["camera_of"]) == [0, 0, 1], "two objects in one camera, one in the other"
    tfs = np.split(g["symmetry_tfs"], np.cumsum(g["symmetry_counts"])[:-1])
    assert list(g["n_hyp"]) == [126, 20, 63]
    o = 0
    for k, name in enumerate(g["symmetries"]):
        assert np.array_equal(tfs[k], gen.symmetry_tfs(str(name)))
        grid = hypotheses.make_rotation_grid(40, 60, tfs[k])
        assert len(grid) == g["n_hyp"][k]
        assert np.abs(g["start"][o:o + len(grid), :3, :3] - grid[:, :3, :3]).max() == 0
        o += len(grid)
    assert len(g["scores"]) == o and (g["top2_margin"] >= gen.MIN_MARGIN_SPREAD * g["spread"]).sum() >= 2
