"""fp_register_objects (several objects of one frame registered in one call) against FoundationPose.register per object in
turn, against the CPU oracle (tests/golden/register_objects.npz, tools/make_golden_register_objects.py), and followed by
track_objects."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "register_objects.npz")
# subdivisions, texture seed, scale, vertex-coloured, open, symmetry group (252 / 126 / 63 / 20 hypotheses), translation
SPECS = [(3, 0, 1.0, False, False, None, (-0.05, 0.0, 0.6)), (2, 5, 0.7, True, False, "half_z", (0.0, 0.02, 0.5)),
         (3, 9, 1.3, False, True, "box", (0.03, -0.13, 0.8)), (2, 2, 0.85, True, True, "cont_z", (0.15, 0.08, 0.65))]


def _symmetry(name):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from make_golden_register_objects import symmetry_tfs

    return None if name is None else symmetry_tfs(name)


def _mesh(sub, seed, scale, vc, open_):
    from foundationpose_b200 import synth

    m = synth.make_mesh(sub, tex_seed=seed, tex_size=256, scale=scale)
    tex = m.visual.image
    if open_:
        z = m.vertices[:, 2]
        m.faces = m.faces[~(z[m.faces] > 0.6 * z.max()).all(1)]  # cut off one cap: a mesh with a hole
    if vc:
        m = synth.vertex_coloured(m)
    return m, tex


@pytest.fixture(scope="module")
def rig():
    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.estimater import FoundationPose, PoseRefinePredictor, ScorePredictor
    from foundationpose_b200.weights import random_state_dict

    e = Engine()
    refiner = PoseRefinePredictor(engine=e, state_dict=random_state_dict("refine", 0))
    scorer = ScorePredictor(engine=e, state_dict=random_state_dict("score", 0))
    objs, placed = [], []
    for k, (sub, seed, scale, vc, open_, sym, t) in enumerate(SPECS):
        m, tex = _mesh(sub, seed, scale, vc, open_)
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(60 + k)
        p[:3, 3] = t
        placed.append((tex, p, scale))
        objs.append((m, sym))
    rgb, depth, owner = synth.make_multi_scene(placed, seed=7)
    alone = [synth.make_multi_scene([o])[2] == 0 for o in placed[:2]]
    assert all((owner == k).any() for k in range(len(objs)))
    assert (alone[0] & alone[1]).any() and (alone[0] & (owner == 1)).any(), "object 1 must partly cover object 0"

    def make(k, sym="spec"):
        m, s = objs[k]
        m = m.copy()
        m.vertices = m.vertices + np.array([0.004, -0.003, 0.002]) * (k + 1)  # off-centre: exercises the model_center shift
        return FoundationPose(model_pts=m.vertices, model_normals=m.vertex_normals, mesh=m, symmetry_tfs=_symmetry(s if sym == "spec" else sym),
                              scorer=scorer, refiner=refiner)

    ests = [make(k) for k in range(len(objs))]
    assert [len(est.rot_grid) for est in ests] == [252, 126, 63, 20]
    masks = [owner == k for k in range(len(objs))]
    yield dict(e=e, ests=ests, make=make, rgb=rgb, depth=depth, masks=masks, K=synth.DEFAULT_K)
    e.close()


def _state(est):
    return (est.pose_last.clone(), int(est.best_id), est.poses.clone(), est.scores.clone())


def _register_both(r, ests, masks, depth=None, iteration=5):
    """register_objects, then est.register per object in turn; returns both (poses, states)."""
    from foundationpose_b200.estimater import register_objects

    depth = r["depth"] if depth is None else depth
    got = register_objects(ests, r["K"], r["rgb"], depth, masks, iteration=iteration)
    got_state = [_state(est) for est in ests]
    want, want_state = [], []
    for est, m in zip(ests, masks):
        want.append(est.register(K=r["K"], rgb=r["rgb"], depth=depth, ob_mask=m, iteration=iteration))
        want_state.append(_state(est))
    return got, got_state, want, want_state


def _assert_equal(got, got_state, want, want_state):
    for k in range(len(got)):
        assert np.array_equal(got[k], want[k]), f"object {k}: pose off by {np.abs(got[k] - want[k]).max():.2e}"
        g, w = got_state[k], want_state[k]
        assert g[1] == w[1], f"object {k}: best_id {g[1]} != {w[1]}"
        for name, a, b in (("pose_last", g[0], w[0]), ("poses", g[2], w[2]), ("scores", g[3], w[3])):
            assert torch.equal(a, b), f"object {k}: ranked {name} differ"


@pytest.mark.parametrize("objects", [[0], [2, 3], [0, 1, 2, 3], [3, 1, 0, 2]])
def test_equals_register_each_object_in_turn(rig, objects):
    ests = [rig["ests"][k] for k in objects]
    masks = [rig["masks"][k] for k in objects]
    _assert_equal(*_register_both(rig, ests, masks))


@pytest.mark.parametrize("syms", [[None] * 4, [None, None, None, "cont_z"]])
def test_several_passes_equal_register_each_object(rig, syms):
    """4 x 252 hypotheses run as passes of 504 + 504, 3 x 252 + 20 as 504 + 272: the first batches above 252."""
    ests = [rig["make"](k, s) for k, s in enumerate(syms)]
    _assert_equal(*_register_both(rig, ests, rig["masks"]))


def test_early_exit_object(rig):
    """A mask without valid depth: identity rotation with the guessed translation, the estimator's state untouched, and
    the other objects' results the same as without it."""
    from foundationpose_b200.estimater import register_objects

    depth = rig["depth"].copy()
    hole = np.zeros_like(rig["masks"][0])
    hole[15:35, 15:55] = True
    assert not any(m[5:45, 5:65].any() for m in rig["masks"])
    depth[5:45, 5:65] = 0.0  # 10 px beyond the mask: the bilateral filter fills holes from up to 2 px away
    a, bad, b = rig["ests"][1], rig["make"](0), rig["ests"][3]
    bad.pose_last = sentinel = torch.full((4, 4), 7.0, device="cuda")
    with_bad = register_objects([a, bad, b], rig["K"], rig["rgb"], depth, [rig["masks"][1], hole, rig["masks"][3]])
    with_bad_state = [_state(a), _state(b)]
    assert bad.pose_last is sentinel and getattr(bad, "poses", None) is None
    want = bad.register(K=rig["K"], rgb=rig["rgb"], depth=depth, ob_mask=hole)
    assert np.array_equal(with_bad[1], want) and np.array_equal(with_bad[1][:3, :3], np.eye(3))
    assert bad.pose_last is sentinel
    without = register_objects([a, b], rig["K"], rig["rgb"], depth, [rig["masks"][1], rig["masks"][3]])
    assert np.array_equal(with_bad[0], without[0]) and np.array_equal(with_bad[2], without[1])
    for g, w in zip(with_bad_state, [_state(a), _state(b)]):
        assert all(torch.equal(x, y) if torch.is_tensor(x) else x == y for x, y in zip(g, w))


def test_against_the_oracle():
    from foundationpose_b200 import hypotheses, synth
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.estimater import make_mesh_tensors
    from foundationpose_b200.weights import random_state_dict

    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_golden_register_objects as gen

    g = dict(np.load(GOLD))
    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    e.set_config("refine")
    e.set_config("score")
    meshes, _, rgb, depth, owner = gen.scene(int(g["seed"]))
    grids = []
    for k, m in enumerate(meshes):
        mesh = synth.vertex_coloured(m) if g["vertex_coloured"][k] else m.copy()
        mesh.vertices = mesh.vertices - g["model_centers"][k].reshape(1, 3)
        mt = make_mesh_tensors(mesh)
        e.set_mesh(mt["pos"], mt["normals"], mt["faces"], float(g["diameters"][k]), uv=mt.get("uv"), tex=mt.get("tex"),
                   vertex_colors=mt.get("vcolor"), slot=k + 1)
        grids.append(torch.from_numpy(hypotheses.make_rotation_grid(40, 60, gen.symmetry_tfs(str(g["symmetries"][k])))).cuda())
    assert [len(x) for x in grids] == list(g["n_hyp"])
    masks = np.stack([owner == k for k in range(len(meshes))])
    slots = list(range(1, len(meshes) + 1))
    start, _, _, info = e.register_objects(rgb, depth, synth.DEFAULT_K, masks, grids, slots, 0)
    np.testing.assert_allclose(start.cpu().numpy(), g["start"], atol=2e-6, rtol=0)
    np.testing.assert_allclose(info.cpu().numpy()[:, :3], g["centers"], atol=2e-6, rtol=0)
    poses, scores, best, _ = e.register_objects(rgb, depth, synth.DEFAULT_K, masks, grids, slots, int(g["iterations"]))
    perr = np.abs(poses.cpu().numpy() - g["refined"]).max()
    print(f"refined poses: max error {perr:.2e}")
    assert perr <= 2e-3
    # the scores are of the free-running refined poses, so their error carries the pose differences too; the selected
    # index is held to the oracle's wherever the oracle's top-2 margin dominates that error
    s_all, best = scores.cpu().numpy(), best.cpu().numpy()
    o = checked = 0
    for k, n in enumerate(g["n_hyp"]):
        s, gs = s_all[o:o + n], g["scores"][o:o + n]
        err = s - gs
        rank_err = np.abs(err - err.mean()).max()  # a common offset cannot change the ranking
        margin, spread = float(g["top2_margin"][k]), float(g["spread"][k])
        print(f"object {k}: rank-relevant score error {rank_err:.2e}, oracle spread {spread:.3f}, top-2 margin {margin:.3f}")
        assert int(best[k]) == int(np.argmax(s))
        if margin >= 5 * rank_err:  # the rule of test_register_golden_gpu.py::test_scores_and_index
            assert int(best[k]) == int(g["ids"][o]), f"object {k}: selected {best[k]}, oracle {g['ids'][o]}"
            checked += 1
        o += n
    assert checked >= 1, "no object's golden margin dominates its score error"
    e.close()


def test_repeated_call_captures_no_graph(rig):
    from foundationpose_b200.estimater import register_objects

    e, ests = rig["e"], rig["ests"]
    for _ in range(2):  # first sight of a pass size runs eagerly, the second captures
        first = register_objects(ests, rig["K"], rig["rgb"], rig["depth"], rig["masks"])
    captures = e.graph_captures()
    again = register_objects(ests, rig["K"], rig["rgb"], rig["depth"], rig["masks"])
    assert e.graph_captures() == captures
    assert all(np.array_equal(a, b) for a, b in zip(first, again))


def test_refusals_launch_nothing(rig):
    from foundationpose_b200 import _lib
    from foundationpose_b200.estimater import register_objects

    e, K = rig["e"], rig["K"]
    masks = np.stack(rig["masks"][:2])
    grids = [rig["ests"][0].rot_grid, rig["ests"][1].rot_grid]
    n0 = _lib.launch_count()
    for slots in ([1, 64], [-1, 2], [1, 40]):  # out of range, out of range, never loaded
        with pytest.raises(_lib.FposeError):
            e.register_objects(rig["rgb"], rig["depth"], K, masks, grids, slots, 5)
    with pytest.raises(_lib.FposeError):  # an object without hypotheses
        e.register_objects(rig["rgb"], rig["depth"], K, masks, [grids[0], grids[1][:0]], [0, 0], 5)
    with pytest.raises(ValueError):
        e.register_objects(rig["rgb"], rig["depth"], K, masks[:, :-1], grids, [0, 0], 5)
    with pytest.raises(ValueError):
        register_objects(rig["ests"][:2], K, rig["rgb"], rig["depth"], rig["masks"][:1])
    with pytest.raises(ValueError):
        register_objects(rig["ests"][:2], K, rig["rgb"], rig["depth"], [rig["masks"][0], rig["masks"][1][:-1]])
    with pytest.raises(TypeError):
        register_objects(rig["ests"][:1], K, torch.from_numpy(rig["rgb"]).cuda(), torch.from_numpy(rig["depth"]).cuda(), rig["masks"][:1])
    assert _lib.launch_count() == n0


def test_then_track_objects(rig):
    """register_objects then track_objects: equal to track_one per object, and no mesh is uploaded again."""
    from foundationpose_b200.estimater import register_objects, track_objects

    e, ests = rig["e"], rig["ests"][:3]
    register_objects(ests, rig["K"], rig["rgb"], rig["depth"], rig["masks"][:3])
    start = [est.pose_last.clone() for est in ests]
    uploads = []
    set_mesh = e.set_mesh
    e.set_mesh = lambda *a, **k: uploads.append(k.get("slot", 0)) or set_mesh(*a, **k)
    try:
        got = track_objects(ests, rig["rgb"], rig["depth"], rig["K"], iteration=2)
    finally:
        del e.set_mesh
    assert uploads == [], "track_objects after register_objects re-uploaded meshes"
    for est, p in zip(ests, start):
        est.pose_last = p.clone()
    want = [est.track_one(rig["rgb"], rig["depth"], rig["K"], 2) for est in ests]
    for k in range(len(ests)):
        assert np.array_equal(got[k], want[k]), f"object {k}"
