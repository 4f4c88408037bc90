"""CPU: estimater.track_cameras' host logic (flattening order and camera ids, slots shared with track_objects /
register_objects, un-centring, empty cameras, refusals) through an engine double, and the scene of
tests/golden/track_cameras.npz."""
import os

import numpy as np
import pytest
import torch

from foundationpose_b200 import synth

GOLD = os.path.join(os.path.dirname(__file__), "golden", "track_cameras.npz")


class _Refiner:
    last_trans_update = last_rot_update = "stale"


class _Engine:
    """Stands in for engine.Engine: records mesh uploads and calls, returns poses shifted by +1 cm in x."""

    def __init__(self):
        self.uploads = []
        self.calls = []

    def set_mesh(self, pos, normals, faces, diameter, uv=None, tex=None, vertex_colors=None, slot=0):
        self.uploads.append((slot, len(pos), float(diameter)))

    def _shifted(self, poses_in):
        out = poses_in.clone()
        out[:, 0, 3] += 0.01
        return out, out.numpy().copy()

    def track_objects(self, rgb, depth, K, poses_in, slots, iterations):
        self.calls.append(("track_objects", list(slots), iterations))
        return self._shifted(poses_in)

    def track_cameras(self, frames, poses_in, camera_of, slots, iterations):
        self.calls.append(("track_cameras", [f[0] for f in frames], list(camera_of), list(slots), iterations))
        return self._shifted(poses_in)


def _est(engine, n_verts, center=(0.0, 0.0, 0.0), x=0.0):
    from foundationpose_b200.estimater import FoundationPose

    est = FoundationPose.__new__(FoundationPose)
    est.engine = engine
    est.refiner = _Refiner()
    est.mesh_tensors = dict(pos=np.zeros((n_verts, 3), np.float32), normals=np.zeros((n_verts, 3), np.float32),
                            faces=np.zeros((1, 3), np.int32), vcolor=np.zeros((n_verts, 3), np.float32))
    est.diameter = 0.1 * n_verts
    est.model_center = np.asarray(center, dtype=np.float64)
    est.pose_last = torch.eye(4).reshape(1, 4, 4)
    est.pose_last[0, 0, 3] = x
    return est


def test_flattening_order_camera_ids_and_empty_cameras():
    from foundationpose_b200.estimater import track_cameras

    e = _Engine()
    a, b, c = _est(e, 3, x=1.0), _est(e, 4, x=2.0), _est(e, 5, x=3.0)
    out = track_cameras([([a, b], "rgb0", None, None), ([], "rgb1", None, None), ([c], "rgb2", None, None), ([], "rgb3", None, None)])
    # the empty cameras are not passed on: the engine sees two cameras, objects camera-major
    assert e.calls == [("track_cameras", ["rgb0", "rgb2"], [0, 0, 1], [1, 2, 3], 2)]
    assert [len(v) for v in out] == [2, 0, 1, 0]
    assert [float(p[0, 3]) for p in out[0] + out[2]] == pytest.approx([1.01, 2.01, 3.01])
    assert track_cameras([]) == []
    assert track_cameras([([], "rgb0", None, None)]) == [[]]
    assert len(e.calls) == 1, "nothing to track: the engine is not called"


def test_slots_are_shared_with_track_objects():
    from foundationpose_b200.estimater import track_cameras, track_objects

    e = _Engine()
    a, b, c = _est(e, 3), _est(e, 4), _est(e, 5)
    track_objects([a, b], None, None, synth.DEFAULT_K)
    track_cameras([([b], "rgb0", None, None), ([c, a], "rgb1", None, None)], iteration=3)
    assert e.calls[-1] == ("track_cameras", ["rgb0", "rgb1"], [0, 1, 1], [2, 3, 1], 3)
    assert [u[0] for u in e.uploads] == [1, 2, 3], "a and b keep the slots track_objects gave them; only c is uploaded"
    b.mesh_tensors = dict(b.mesh_tensors, pos=np.zeros((6, 3), np.float32))  # what reset_object does: new mesh tensors
    track_cameras([([b], "rgb0", None, None)])
    assert e.uploads[-1][:2] == (2, 6) and len(e.uploads) == 4


def test_poses_uncentred_and_pose_last_updated():
    from foundationpose_b200.estimater import track_cameras

    e = _Engine()
    ca, cb = (0.01, -0.02, 0.03), (-0.03, 0.0, 0.02)
    a, b = _est(e, 3, center=ca), _est(e, 4, center=cb)
    a.pose_last[0, :3, :3] = torch.from_numpy(synth.random_rotation(2)).float()
    b.pose_last[0, :3, :3] = torch.from_numpy(synth.random_rotation(3)).float()
    out = track_cameras([([a], "rgb0", None, None), ([b], "rgb1", None, None)])
    for est, c, got in ((a, ca, out[0][0]), (b, cb, out[1][0])):
        want = est.pose_last.reshape(4, 4).numpy().astype(np.float64)
        want[:3, 3] -= want[:3, :3] @ np.asarray(c)
        assert np.array_equal(got, want.astype(np.float32))
        assert float(est.pose_last[0, 0, 3]) == pytest.approx(0.01)
        assert est.refiner.last_trans_update is None and est.refiner.last_rot_update is None


def test_refusals():
    from foundationpose_b200.estimater import MAX_CAMERAS, MAX_MESHES, track_cameras

    e = _Engine()
    a, b = _est(e, 3), _est(e, 4)
    with pytest.raises(ValueError):
        track_cameras([([a], "rgb0", None, None), ([_est(_Engine(), 3)], "rgb1", None, None)])  # mixed engines
    with pytest.raises(ValueError):
        track_cameras([([a], "rgb0", None, None), ([b, a], "rgb1", None, None)])  # a in two cameras
    with pytest.raises(ValueError):
        track_cameras([([a, a], "rgb0", None, None)])
    with pytest.raises(TypeError):
        track_cameras([([a], torch.zeros(4, 4, 3, dtype=torch.uint8), torch.zeros(4, 4), synth.DEFAULT_K)])
    with pytest.raises(TypeError):  # refused even on a camera without objects
        track_cameras([([a], "rgb0", None, None), ([], torch.zeros(4, 4, 3, dtype=torch.uint8), torch.zeros(4, 4), None)])
    b.pose_last = None
    with pytest.raises(RuntimeError):
        track_cameras([([a], "rgb0", None, None), ([b], "rgb1", None, None)])
    with pytest.raises(ValueError):
        track_cameras([([_est(e, 3)], f"rgb{c}", None, None) for c in range(MAX_CAMERAS + 1)])
    with pytest.raises(ValueError):
        track_cameras([([_est(e, 3) for _ in range(MAX_MESHES)], "rgb0", None, None)])
    assert e.calls == [] and e.uploads == [], "every refusal comes before anything reaches the engine"
    # an empty camera does not count towards the limit
    views = [([_est(e, 3)], f"rgb{c}", None, None) for c in range(MAX_CAMERAS)] + [([], "rgb_empty", None, None)]
    assert len(track_cameras(views)) == MAX_CAMERAS + 1


def test_golden_scene():
    """The rig of tests/golden/track_cameras.npz: two cameras of different size and intrinsics, objects 0 and 2 seen by
    both, object 1 by camera 0 only, and the recorded pairs are exactly those."""
    g = dict(np.load(GOLD))
    assert [tuple(x) for x in zip(g["H"], g["W"])] == [(480, 640), (720, 1280)]
    assert np.array_equal(g["K"][0], synth.DEFAULT_K) and not np.array_equal(g["K"][1], g["K"][0])
    assert [tuple(p) for p in g["pairs"]] == [(0, 0), (0, 1), (0, 2), (1, 0), (1, 2)]
    assert g["pose_in"].shape == g["pose_out"].shape == (5, 5, 4, 4)
    meshes = [synth.make_mesh(int(g["subdivisions"][k]), tex_seed=int(g["tex_seeds"][k]), tex_size=int(g["tex_size"]),
                              scale=float(g["scales"][k])) for k in range(len(g["scales"]))]
    for k, m in enumerate(meshes):
        assert abs(synth.mesh_diameter(m.vertices) - g["diameters"][k]) < 1e-12
    T = g["extrinsic"]
    assert np.allclose(T[:3, :3] @ T[:3, :3].T, np.eye(3)) and np.linalg.norm(T[:3, 3]) > 0.2
    for c in range(2):
        objs = [(m.visual.image, (T if c else np.eye(4)) @ g["gt"][k, 1], float(g["scales"][k])) for k, m in enumerate(meshes)]
        _, _, owner = synth.make_multi_scene(objs, g["K"][c], int(g["H"][c]), int(g["W"][c]), seed=2 + 100 * c)
        seen = [k for k in range(len(meshes)) if (owner == k).any()]
        assert seen == [k for cc, k in g["pairs"] if cc == c], f"camera {c} sees {seen}"
