"""CPU: the multi-object synthetic scene, and estimater.track_objects' host logic (slot assignment, reload after
reset_object, errors, the model_center shift) through an engine double."""
import numpy as np
import pytest
import torch

from foundationpose_b200 import synth


def _pose(seed, t):
    p = np.eye(4)
    p[:3, :3] = synth.random_rotation(seed)
    p[:3, 3] = t
    return p


def test_one_object_at_scale_one_is_make_scene():
    tex = synth.make_texture(3, 256)
    p = _pose(1, [0.01, -0.02, 0.6])
    rgb, depth, mask = synth.make_scene(tex, p, seed=4)
    rgb2, depth2, owner = synth.make_multi_scene([(tex, p, 1.0)], seed=4)
    assert np.array_equal(rgb, rgb2) and np.array_equal(depth, depth2) and np.array_equal(mask, owner == 0)


def test_nearest_object_wins():
    a, b = synth.make_texture(1, 256), synth.make_texture(2, 256)
    far, near = _pose(0, [0.0, 0.0, 0.7]), _pose(1, [0.02, 0.0, 0.5])
    _, depth, owner = synth.make_multi_scene([(a, far, 1.0), (b, near, 0.6)], depth_noise=0.0)
    _, _, alone_far = synth.make_multi_scene([(a, far, 1.0)], depth_noise=0.0)
    _, depth_near, alone_near = synth.make_multi_scene([(b, near, 0.6)], depth_noise=0.0)
    both = (alone_far == 0) & (alone_near == 0)
    assert both.any() and (owner[both] == 1).all(), "the nearer object must cover the farther one"
    assert np.array_equal(owner == 0, (alone_far == 0) & ~both)
    assert np.array_equal(depth[owner == 1], depth_near[owner == 1])


class _Refiner:
    last_trans_update = last_rot_update = "stale"


class _Engine:
    """Stands in for engine.Engine: records mesh uploads and returns poses shifted by +1 cm in x per call."""

    def __init__(self):
        self.uploads = []
        self.calls = []

    def set_mesh(self, pos, normals, faces, diameter, uv=None, tex=None, vertex_colors=None, slot=0):
        self.uploads.append((slot, len(pos), float(diameter)))

    def track_objects(self, rgb, depth, K, poses_in, slots, iterations):
        self.calls.append((list(slots), iterations))
        out = poses_in.clone()
        out[:, 0, 3] += 0.01
        return out, out.numpy().copy()


def _est(engine, n_verts, center=(0.0, 0.0, 0.0)):
    from foundationpose_b200.estimater import FoundationPose

    est = FoundationPose.__new__(FoundationPose)
    est.engine = engine
    est.refiner = _Refiner()
    est.mesh_tensors = dict(pos=np.zeros((n_verts, 3), np.float32), normals=np.zeros((n_verts, 3), np.float32),
                            faces=np.zeros((1, 3), np.int32), vcolor=np.zeros((n_verts, 3), np.float32))
    est.diameter = 0.1 * n_verts
    est.model_center = np.asarray(center, dtype=np.float64)
    est.pose_last = torch.eye(4).reshape(1, 4, 4)
    return est


def test_slots_assigned_once_and_reloaded_after_reset():
    from foundationpose_b200.estimater import track_objects

    e = _Engine()
    a, b = _est(e, 3), _est(e, 4)
    track_objects([a, b], None, None, synth.DEFAULT_K, iteration=2)
    assert e.uploads == [(1, 3, pytest.approx(0.3)), (2, 4, pytest.approx(0.4))]
    assert e.calls == [([1, 2], 2)]
    track_objects([b, a], None, None, synth.DEFAULT_K)
    assert len(e.uploads) == 2 and e.calls[-1] == ([2, 1], 2), "known meshes are not uploaded again; order follows the list"
    b.mesh_tensors = dict(b.mesh_tensors, pos=np.zeros((5, 3), np.float32))  # what reset_object does: new mesh tensors
    track_objects([a, b], None, None, synth.DEFAULT_K)
    assert e.uploads[-1][:2] == (2, 5) and len(e.uploads) == 3
    assert all(slot != 0 for slot, _, _ in e.uploads), "slot 0 belongs to the single-object calls"


def test_slots_of_collected_estimators_are_reused():
    import gc

    from foundationpose_b200.estimater import track_objects

    e = _Engine()
    keep = _est(e, 3)
    track_objects([keep, _est(e, 4)], None, None, synth.DEFAULT_K)
    gc.collect()
    track_objects([_est(e, 6)], None, None, synth.DEFAULT_K)
    assert e.calls[-1][0] == [2]


def test_poses_uncentred_and_pose_last_updated():
    from foundationpose_b200.estimater import track_objects

    e = _Engine()
    c = (0.01, -0.02, 0.03)
    a = _est(e, 3, center=c)
    R = torch.from_numpy(synth.random_rotation(2)).float()
    a.pose_last[0, :3, :3] = R
    out = track_objects([a], None, None, synth.DEFAULT_K)
    want = a.pose_last.reshape(4, 4).numpy().astype(np.float64)
    want[:3, 3] -= want[:3, :3] @ np.asarray(c)
    assert np.array_equal(out[0], want.astype(np.float32))
    assert float(a.pose_last[0, 0, 3]) == pytest.approx(0.01)
    assert a.refiner.last_trans_update is None and a.refiner.last_rot_update is None


def test_errors():
    from foundationpose_b200.estimater import MAX_MESHES, track_objects

    e = _Engine()
    assert track_objects([], None, None, synth.DEFAULT_K) == []
    a = _est(e, 3)
    with pytest.raises(ValueError):
        track_objects([a, _est(_Engine(), 3)], None, None, synth.DEFAULT_K)
    with pytest.raises(ValueError):
        track_objects([a, a], None, None, synth.DEFAULT_K)
    with pytest.raises(TypeError):
        track_objects([a], torch.zeros(4, 4, 3, dtype=torch.uint8), torch.zeros(4, 4), synth.DEFAULT_K)
    b = _est(e, 3)
    b.pose_last = None
    with pytest.raises(RuntimeError):
        track_objects([a, b], None, None, synth.DEFAULT_K)
    with pytest.raises(ValueError):
        track_objects([_est(e, 3) for _ in range(MAX_MESHES)], None, None, synth.DEFAULT_K)
    assert e.calls == [] and e.uploads == [], "every error is raised before anything reaches the engine"
    many = [_est(e, 3) for _ in range(MAX_MESHES - 1)]
    track_objects(many, None, None, synth.DEFAULT_K)
    with pytest.raises(ValueError):
        track_objects([a], None, None, synth.DEFAULT_K)  # all 63 object slots are owned by live estimators
