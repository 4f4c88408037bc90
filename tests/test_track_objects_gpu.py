"""fp_track_objects (several objects of one frame, ONE graph launch) against fp_track and the by-value fp_set_frame +
fp_refine per object, against the CPU oracle (tests/golden/track_objects.npz, tools/make_golden_track_objects.py), and
through estimater.track_objects."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden", "track_objects.npz")
# subdivisions, texture seed, scale, vertex-coloured, open
SPECS = [(3, 0, 1.0, False, False), (2, 5, 0.7, True, False), (3, 9, 1.3, False, True), (2, 2, 0.85, True, True),
         (4, 4, 1.1, False, False), (2, 7, 0.9, False, True)]


def _object(sub, seed, scale, vc, open_):
    from foundationpose_b200 import synth

    m = synth.make_mesh(sub, tex_seed=seed, tex_size=256, scale=scale)
    tex = m.visual.image
    if open_:
        z = m.vertices[:, 2]
        m.faces = m.faces[~(z[m.faces] > 0.6 * z.max()).all(1)]  # cut off one cap: a mesh with a hole
    if vc:
        m = synth.vertex_coloured(m)
    return m, tex, scale


def _load(e, mesh, slot):
    from foundationpose_b200 import synth
    from foundationpose_b200.estimater import make_mesh_tensors

    mt = make_mesh_tensors(mesh)
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(mesh.vertices), uv=mt.get("uv"), tex=mt.get("tex"),
               vertex_colors=mt.get("vcolor"), slot=slot)


def _engine():
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.weights import random_state_dict

    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.set_config("refine")
    return e


@pytest.fixture(scope="module")
def rig():
    from foundationpose_b200 import synth

    objs = [_object(*s) for s in SPECS]
    gt, start = [], []
    rng = np.random.default_rng(5)
    for k in range(len(objs)):
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(30 + k)
        p[:3, 3] = [-0.15 + 0.06 * k, 0.05 * (-1) ** k, 0.55 + 0.05 * k]
        gt.append(p)
        q = p.copy()
        q[:3, 3] += rng.normal(0, 0.004, 3)
        start.append(q.astype(np.float32))
    rgb, depth, owner = synth.make_multi_scene([(tex, p, sc) for (_, tex, sc), p in zip(objs, gt)], seed=3)
    assert all((owner == k).any() for k in range(len(objs)))
    e = _engine()
    for k, (m, _, _) in enumerate(objs):
        _load(e, m, k + 1)
    return dict(e=e, objs=objs, rgb=rgb, depth=depth, start=np.stack(start))


def _single(r, k):
    """Object k alone, its mesh in slot 0: {path: pose} for fp_track (the camera-table path) and for the by-value path
    fp_set_frame (filtered, zfar = inf) + fp_refine."""
    from foundationpose_b200 import synth

    e = r["e"]
    _load(e, r["objs"][k][0], 0)
    start = torch.from_numpy(r["start"][k]).cuda()
    _, tracked = e.track(r["rgb"], r["depth"], synth.DEFAULT_K, start, 2)
    e.set_frame(r["rgb"], r["depth"], synth.DEFAULT_K, filter_depth=True, zfar=float("inf"))
    refined = e.refine(start, 2)[0][0].cpu().numpy()
    return {"track": tracked, "set_frame + refine": refined}


@pytest.mark.parametrize("M", [1, 2, 3, 5])
def test_equals_tracking_each_object_alone(rig, M):
    from foundationpose_b200 import synth

    e = rig["e"]
    dev, host = e.track_objects(rig["rgb"], rig["depth"], synth.DEFAULT_K, torch.from_numpy(rig["start"][:M]).cuda(),
                                list(range(1, M + 1)), 2)
    assert np.array_equal(dev.cpu().numpy(), host), "device and host copies of the poses differ"
    for k in range(M):
        for path, single in _single(rig, k).items():
            assert np.array_equal(host[k], single), f"M={M}, object {k}: off {path} by {np.abs(host[k] - single).max():.2e}"


def test_against_the_oracle():
    from foundationpose_b200 import synth

    g = dict(np.load(GOLD))
    e = _engine()
    objs = []
    for k in range(len(g["scales"])):
        m = synth.make_mesh(int(g["subdivisions"][k]), tex_seed=int(g["tex_seeds"][k]), tex_size=int(g["tex_size"]),
                            scale=float(g["scales"][k]))
        objs.append((m.visual.image, float(g["scales"][k])))
        _load(e, synth.vertex_coloured(m) if g["vertex_coloured"][k] else m, k + 1)
        assert abs(synth.mesh_diameter(m.vertices) - g["diameters"][k]) < 1e-12
    slots = list(range(1, len(objs) + 1))
    worst = 0.0
    for i in range(len(g["pose_in"])):
        rgb, depth, _ = synth.make_multi_scene([(tex, g["gt"][k, i + 1], sc) for k, (tex, sc) in enumerate(objs)], seed=2 + i)
        _, host = e.track_objects(rgb, depth, synth.DEFAULT_K, torch.from_numpy(g["pose_in"][i]).cuda(), slots, 2)
        err = np.abs(host - g["pose_out"][i])
        worst = max(worst, err.max())
        assert err.max() <= 1e-3, f"frame {i + 1}: pose off by {err.max():.2e} (per object {err.reshape(len(objs), -1).max(1)})"
    print(f"track_objects over {len(g['pose_in'])} frames x {len(objs)} objects: worst error {worst:.2e}")
    e.close()


def test_object_order_and_slot_reuse(rig):
    from foundationpose_b200 import synth

    e, K = rig["e"], synth.DEFAULT_K
    start = torch.from_numpy(rig["start"][:3]).cuda()
    for _ in range(3):  # first sight runs eagerly, the second call captures, later calls replay
        _, base = e.track_objects(rig["rgb"], rig["depth"], K, start, [1, 2, 3], 2)
    captures = e.graph_captures()
    perm = [2, 0, 1]
    _, permuted = e.track_objects(rig["rgb"], rig["depth"], K, start[perm], [p + 1 for p in perm], 2)
    assert np.array_equal(permuted, base[perm])
    assert e.graph_captures() == captures, "a different order of the same objects captured a new graph"
    # other intrinsics, then also a smaller frame whose right edge cuts through object 2 (at u ~ 290 px): the graph reads
    # the frame from the camera table and replays, each result differs from the one before (the new intrinsics and the
    # new size are read) and is the same as a fresh context's
    K2 = K.copy()
    K2[0, 2] += 3.0
    K2[1, 1] *= 1.01
    before = base
    for rgb, depth in ((rig["rgb"], rig["depth"]), (rig["rgb"][:400, :300], rig["depth"][:400, :300])):
        _, got = e.track_objects(rgb, depth, K2, start, [1, 2, 3], 2)
        assert e.graph_captures() == captures, f"a {depth.shape} frame with other intrinsics captured a new graph"
        assert not np.array_equal(got, before), f"a {depth.shape} frame with other intrinsics changed no pose"
        fresh = _engine()
        for k in range(3):
            _load(fresh, rig["objs"][k][0], k + 1)
        _, want = fresh.track_objects(rgb, depth, K2, start, [1, 2, 3], 2)
        fresh.close()
        assert np.array_equal(got, want), f"{depth.shape} frame: off a fresh context by {np.abs(got - want).max():.2e}"
        before = got
    # reload slot 2 with object 3's mesh between replays: same as a fresh context holding that set of meshes
    _load(e, rig["objs"][3][0], 2)
    _, swapped = e.track_objects(rig["rgb"], rig["depth"], K, start, [1, 2, 3], 2)
    fresh = _engine()
    for slot, k in ((1, 0), (2, 3), (3, 2)):
        _load(fresh, rig["objs"][k][0], slot)
    _, ref = fresh.track_objects(rig["rgb"], rig["depth"], K, start, [1, 2, 3], 2)
    fresh.close()
    _load(e, rig["objs"][1][0], 2)
    assert np.array_equal(swapped, ref)
    assert not np.array_equal(swapped[1], base[1])


def test_one_launch_sequence_per_frame(rig):
    from foundationpose_b200 import _lib, synth

    e, K = rig["e"], synth.DEFAULT_K
    per_frame = {}
    for M in (1, 6):
        start = torch.from_numpy(rig["start"][:M]).cuda()
        for _ in range(3):
            e.track_objects(rig["rgb"], rig["depth"], K, start, list(range(1, M + 1)), 2)
        n0 = _lib.launch_count()
        e.track_objects(rig["rgb"], rig["depth"], K, start, list(range(1, M + 1)), 2)
        per_frame[M] = _lib.launch_count() - n0
    assert per_frame[1] == per_frame[6], per_frame


def test_bad_slots_are_refused_before_any_launch(rig):
    from foundationpose_b200 import _lib, synth

    e, K = rig["e"], synth.DEFAULT_K
    start = torch.from_numpy(rig["start"][:2]).cuda()
    n0 = _lib.launch_count()
    for slots in ([1, 64], [-1, 2], [1, 40]):  # out of range, out of range, never loaded
        with pytest.raises(_lib.FposeError):
            e.track_objects(rig["rgb"], rig["depth"], K, start, slots, 2)
    with pytest.raises(_lib.FposeError):
        _load(e, rig["objs"][0][0], 64)
    assert _lib.launch_count() == n0


def test_public_api_equals_track_one_in_turn(rig):
    from foundationpose_b200 import synth
    from foundationpose_b200.estimater import FoundationPose, PoseRefinePredictor, ScorePredictor, track_objects
    from foundationpose_b200.weights import random_state_dict

    e = _engine()
    refiner = PoseRefinePredictor(engine=e, state_dict=random_state_dict("refine", 0))
    scorer = ScorePredictor(engine=e, state_dict=random_state_dict("score", 0))
    ests = []
    for k, (m, _, _) in enumerate(rig["objs"][:3]):
        m = m.copy()
        m.vertices = m.vertices + np.array([0.01, -0.02, 0.005]) * (k + 1)  # off-centre: exercises the un-centring shift
        ests.append(FoundationPose(model_pts=m.vertices, model_normals=m.vertex_normals, mesh=m, scorer=scorer, refiner=refiner))
        assert np.abs(ests[-1].model_center).max() > 1e-3

    def reset():
        for k, est in enumerate(ests):
            # the centred mesh is the rig's mesh, so the rig's start pose is its pose_last
            est.pose_last = torch.from_numpy(rig["start"][k]).cuda().reshape(1, 4, 4)

    K = synth.DEFAULT_K
    reset()
    got = track_objects(ests, rig["rgb"], rig["depth"], K, iteration=2)
    got_last = [est.pose_last.cpu() for est in ests]
    reset()
    want = [est.track_one(rig["rgb"], rig["depth"], K, 2) for est in ests]
    for k in range(3):
        assert np.array_equal(got[k], want[k]), f"object {k}"
        assert torch.equal(got_last[k], ests[k].pose_last.cpu())
    other = _engine()
    ests_other = FoundationPose(model_pts=rig["objs"][0][0].vertices, model_normals=rig["objs"][0][0].vertex_normals,
                                mesh=rig["objs"][0][0], refiner=PoseRefinePredictor(engine=other, state_dict=random_state_dict("refine", 0)),
                                scorer=ScorePredictor(engine=other, state_dict=random_state_dict("score", 0)))
    ests_other.pose_last = ests[0].pose_last.clone()
    with pytest.raises(ValueError):
        track_objects([ests[0], ests_other], rig["rgb"], rig["depth"], K)
    with pytest.raises(TypeError):
        track_objects(ests, torch.from_numpy(rig["rgb"]).cuda(), torch.from_numpy(rig["depth"]).cuda(), K)
    assert track_objects([], rig["rgb"], rig["depth"], K) == []
    other.close()
    e.close()
