"""CPU: PoseFit's arithmetic, and the host reference of the tracking fit counts (tests/fit_reference.py) on synthetic
scenes: a pose on the object agrees with the depth, a pose in front of the surface, beside the object or in a frame
without it sees past its surface (behind), a pose behind the surface is hidden (occluded)."""
import numpy as np
import pytest

import crop_reference as cr
import fit_reference as fr

DELTA = 0.01


def test_pose_fit_ratios():
    from foundationpose_b200.estimater import PoseFit

    f = PoseFit.from_counts(np.array([200, 160, 120, 30, 10], dtype=np.int32))
    assert (f.covered, f.valid, f.inlier, f.occluded, f.behind) == (200, 160, 120, 30, 10)
    assert all(type(v) is int for v in (f.covered, f.valid, f.inlier, f.occluded, f.behind))
    assert f.inlier_ratio == 0.75 and f.behind_ratio == 0.0625 and f.visible_ratio == 0.8
    gone = PoseFit.from_counts([0, 0, 0, 0, 0])  # the object left the view: every ratio fires a `< threshold` test
    assert (gone.inlier_ratio, gone.behind_ratio, gone.visible_ratio) == (0.0, 0.0, 0.0)
    dark = PoseFit(covered=50, valid=0, inlier=0, occluded=0, behind=0)  # covered, no valid depth
    assert (dark.inlier_ratio, dark.behind_ratio, dark.visible_ratio) == (0.0, 0.0, 0.0)
    with pytest.raises(Exception):
        f.inlier = 3  # a measurement, not a mutable record


def _scene(pose, with_object=True):
    from foundationpose_b200 import synth
    from oracle import geometry, pipeline

    mesh = synth.make_mesh(3)
    K = synth.DEFAULT_K
    objs = [(mesh.visual.image, pose, 1.0)] if with_object else []
    rgb, depth, _ = synth.make_multi_scene(objs, K, seed=5, depth_noise=0.001)
    return cr.Scene(pipeline.mesh_tensors(mesh), K, rgb, depth, geometry.depth2xyzmap(depth, K), synth.mesh_diameter(mesh.vertices))


def _gt():
    from foundationpose_b200 import synth

    p = np.eye(4)
    p[:3, :3] = synth.random_rotation(4)
    p[:3, 3] = [0.02, -0.01, 0.6]
    return p


def _moved(p, dx=0.0, dz=0.0):
    q = p.copy()
    q[0, 3] += dx
    q[2, 3] += dz
    return q.astype(np.float32)[None]


def test_counts_add_up_and_agree_at_the_true_pose():
    gt = _gt()
    c = fr.counts(_scene(gt), gt.astype(np.float32)[None], DELTA)[0]
    covered, valid, inlier, occluded, behind = c
    assert inlier + occluded + behind == valid <= covered
    assert covered > 5000 and valid == covered
    assert inlier / valid > 0.95, dict(zip(fr.NAMES, c))


@pytest.mark.parametrize("case", ["toward the camera", "one diameter aside", "object absent"])
def test_behind_dominates_when_the_track_is_lost(case):
    gt = _gt()
    if case == "toward the camera":
        sc, pose = _scene(gt), _moved(gt, dz=-0.03)
    elif case == "one diameter aside":
        sc, pose = _scene(gt), _moved(gt, dx=0.19)
    else:
        sc, pose = _scene(gt, with_object=False), _moved(gt)
    c = dict(zip(fr.NAMES, fr.counts(sc, pose, DELTA)[0]))
    assert c["valid"] > 1000
    assert c["behind"] > 0.8 * c["valid"] and c["behind"] > max(c["inlier"], c["occluded"]), (case, c)


def test_occluded_dominates_behind_the_surface():
    gt = _gt()
    c = dict(zip(fr.NAMES, fr.counts(_scene(gt), _moved(gt, dz=0.03), DELTA)[0]))
    assert c["occluded"] > 0.8 * c["valid"] and c["occluded"] > max(c["inlier"], c["behind"]), c


def test_near_delta_counts_pixels_at_the_threshold():
    gt = _gt()
    sc = _scene(gt)
    covered, zr, zo = fr.depths(sc, gt.astype(np.float32)[None])
    d = (zo - zr)[covered & (zo >= 0.001)]
    delta = float(d.abs().median())  # half the valid pixels lie within it: the threshold sits among them
    assert fr.near_delta(covered, zr, zo, delta, tol=1e-12)[0] >= 1
    assert fr.near_delta(covered, zr, zo, 10.0)[0] == 0
