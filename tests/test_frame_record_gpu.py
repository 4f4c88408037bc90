"""The calls that take the context's frame (camera 0) by value keep their CUDA graphs until the frame's size or intrinsics
change: with warm graphs, a frame with new fx fy cx cy at the same size, then a frame of another size, captures each
graph the call replays exactly once, and every result equals the same call on a fresh context bit for bit.  fp_track
takes the frame from the camera table: the same two frames capture no graph."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# H, W, K: the frame the graphs are warmed on, new intrinsics at the same size, a smaller frame
FRAMES = [(480, 640, [[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1]]),
          (480, 640, [[600.0, 0, 316.0], [0, 606.0, 244.0], [0, 0, 1]]),
          (360, 480, [[460.0, 0, 240.0], [0, 462.0, 180.0], [0, 0, 1]])]
N_HYP = 24


@pytest.fixture(scope="module")
def scene():
    from foundationpose_b200 import hypotheses, synth

    mesh = synth.make_mesh(3, tex_seed=0, tex_size=256)
    pose = np.eye(4)
    pose[:3, :3] = synth.random_rotation(3)
    pose[:3, 3] = [0.01, -0.01, 0.7]
    start = pose.copy()
    start[:3, 3] += [0.003, -0.002, 0.004]
    frames = []
    for i, (H, W, K) in enumerate(FRAMES):
        K = np.asarray(K, dtype=np.float64)
        rgb, depth, mask = synth.make_scene(mesh.visual.image, pose, K, H, W, seed=11 + i)
        assert mask.sum() >= 100
        frames.append(dict(rgb=rgb, depth=depth, K=K, mask=mask))
    grid = torch.from_numpy(hypotheses.make_rotation_grid(40, 60, None)[:N_HYP]).cuda()
    return dict(mesh=mesh, frames=frames, start=torch.from_numpy(start.astype(np.float32)).cuda(), grid=grid)


def _engine(mesh):
    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.estimater import make_mesh_tensors
    from foundationpose_b200.weights import random_state_dict

    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    e.set_config("refine")
    e.set_config("score")
    mt = make_mesh_tensors(mesh)
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(mesh.vertices), uv=mt.get("uv"), tex=mt.get("tex"))
    return e


def _track(e, f, scene):
    return [torch.from_numpy(e.track(f["rgb"], f["depth"], f["K"], scene["start"], 2)[1])]


def _register_objects(e, f, scene):
    return [t.cpu() for t in e.register_objects(f["rgb"], f["depth"], f["K"], f["mask"][None], [scene["grid"]], [0], 2)]


def _register(e, f, scene):
    """FoundationPose.register's engine calls: the filtered frame, start poses, refinement, scores."""
    e.set_frame(f["rgb"], f["depth"], f["K"], filter_depth=True, zfar=float("inf"))
    poses, info = e.start_poses(f["mask"], scene["grid"])
    refined, _, _ = e.refine(poses, 2)
    scores, best = e.score(refined)
    return [t.cpu() for t in (poses, info, refined, scores, best)]


# each call and the number of by-value graphs it replays: one register pass's refinement and scorer features; refine's
# and score_features'
CALLS = [(_register_objects, 2), (_register, 2)]


@pytest.mark.parametrize("call,graphs", CALLS, ids=[c.__name__.lstrip("_") for c, _ in CALLS])
def test_by_value_graphs_follow_the_frame(scene, call, graphs):
    _follow_the_frames(scene, call, graphs)


def test_track_replays_its_graph_on_a_new_frame(scene):
    """fp_track is fp_track_cameras with one camera and one object: new intrinsics or a smaller frame replay its graph."""
    _follow_the_frames(scene, _track, 0)


def _follow_the_frames(scene, call, graphs):
    """Warms every graph of `call` on the first frame, then asserts that new intrinsics, then another frame size, capture
    `graphs` graphs each and give what a fresh context gives."""
    e = _engine(scene["mesh"])
    first = scene["frames"][0]
    for _ in range(3):  # first sight of every graph runs eagerly, the second captures, the third replays
        call(e, first, scene)
    captures = e.graph_captures()
    assert _equal(call(e, first, scene), call(e, first, scene)) and e.graph_captures() == captures, "a warm call captured"
    for which, f in (("new intrinsics", scene["frames"][1]), ("another frame size", scene["frames"][2])):
        got = call(e, f, scene)
        assert e.graph_captures() == captures + graphs, f"{which}: {e.graph_captures() - captures} captures"
        captures = e.graph_captures()
        fresh = _engine(scene["mesh"])
        want = call(fresh, f, scene)
        fresh.close()
        assert _equal(got, want), f"{which}: differs from a fresh context"
    e.close()


def _equal(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))
