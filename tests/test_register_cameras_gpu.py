"""fp_register_cameras (objects of several camera streams registered in one call) against fp_register_objects per camera
and FoundationPose.register per object, against the CPU oracle (tests/golden/register_cameras.npz,
tools/make_golden_register_cameras.py), its graph caching, its refusals, its teardown, and followed by track_cameras."""
import ctypes as C
import gc
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "register_cameras.npz")
MiB = 1 << 20
# subdivisions, texture seed, scale, vertex-coloured, open, symmetry group (252 / 126 / 63 / 20 hypotheses)
SPECS = [(3, 0, 1.0, False, False, None), (2, 5, 0.7, True, False, "half_z"), (3, 9, 1.3, False, True, "box"),
         (2, 2, 0.85, True, True, "cont_z")]
# per camera: H, W, K, objects it sees (indices into SPECS).  333 x 257 is not a multiple of the frame filter's tile.
CAMERAS = [(480, 640, [[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1]], [0, 1]),
           (240, 320, [[300.0, 0, 158.0], [0, 305.0, 121.0], [0, 0, 1]], [2]),
           (720, 1280, [[920.0, 0, 640.0], [0, 915.0, 360.0], [0, 0, 1]], [3, 1]),
           (257, 333, [[330.0, 0, 165.5], [0, 328.0, 130.0], [0, 0, 1]], [2, 3])]


def _symmetry(name):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from make_golden_register_objects import symmetry_tfs

    return None if name is None else symmetry_tfs(name)


def _object(sub, seed, scale, vc, open_, sym):
    from foundationpose_b200 import synth

    m = synth.make_mesh(sub, tex_seed=seed, tex_size=256, scale=scale)
    tex = m.visual.image
    if open_:
        z = m.vertices[:, 2]
        m.faces = m.faces[~(z[m.faces] > 0.6 * z.max()).all(1)]  # cut off one cap: a mesh with a hole
    if vc:
        m = synth.vertex_coloured(m)
    return m, tex, scale, sym


def _load(e, mesh, slot):
    from foundationpose_b200 import synth
    from foundationpose_b200.estimater import make_mesh_tensors

    mt = make_mesh_tensors(mesh)
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(mesh.vertices), uv=mt.get("uv"), tex=mt.get("tex"),
               vertex_colors=mt.get("vcolor"), slot=slot)


def _engine(objs=()):
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.weights import random_state_dict

    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    e.set_config("refine")
    e.set_config("score")
    for k, (m, _, _, _) in enumerate(objs):
        _load(e, m, k + 1)
    return e


def _camera(objs, H, W, K, seen, seed):
    """A frame of camera (H, W, K) showing objects `seen` side by side, and each one's mask."""
    from foundationpose_b200 import synth

    K = np.asarray(K, dtype=np.float64)
    placed = []
    for j, k in enumerate(seen):
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(50 + 7 * seed + k)
        z = 0.65 + 0.05 * j
        p[:3, 3] = [((W * (j + 1) / (len(seen) + 1)) - K[0, 2]) * z / K[0, 0], 0.02 * (-1) ** j, z]
        placed.append((objs[k][1], p, objs[k][2]))
    rgb, depth, owner = synth.make_multi_scene(placed, K, H, W, seed=seed)
    masks = [owner == j for j in range(len(seen))]
    assert all(m.sum() >= 4 for m in masks)
    return dict(rgb=rgb, depth=depth, K=K, seen=list(seen), masks=masks)


def _grid(sym):
    from foundationpose_b200 import hypotheses

    return torch.from_numpy(hypotheses.make_rotation_grid(40, 60, _symmetry(sym))).cuda()


@pytest.fixture(scope="module")
def rig():
    objs = [_object(*s) for s in SPECS]
    cams = [_camera(objs, H, W, K, seen, seed=3 + c) for c, (H, W, K, seen) in enumerate(CAMERAS)]
    grids = {sym: _grid(sym) for sym in (None, "half_z", "box", "cont_z")}
    assert [len(grids[s[5]]) for s in SPECS] == [252, 126, 63, 20]
    e = _engine(objs)
    yield dict(e=e, objs=objs, cams=cams, grids=grids)
    e.close()


def _objects(rig, cams, order=None, full=False):
    """(frames, masks, grids, camera ids, slots, pairs) of every (camera, object) pair, camera-major or in `order`."""
    pairs = [(c, j) for c, cam in enumerate(cams) for j in range(len(cam["seen"]))]
    if order is not None:
        pairs = [pairs[i] for i in order]
    sym = lambda k: None if full else rig["objs"][k][3]
    frames = [(cam["rgb"], cam["depth"], cam["K"]) for cam in cams]
    masks = [cams[c]["masks"][j] for c, j in pairs]
    grids = [rig["grids"][sym(cams[c]["seen"][j])] for c, j in pairs]
    return frames, masks, grids, [c for c, _ in pairs], [cams[c]["seen"][j] + 1 for c, j in pairs], pairs


def _split(out, n_hyp):
    """Object-major outputs -> per object (poses, scores, best, info)."""
    poses, scores, best, info = (t.cpu() for t in out)
    o, res = 0, []
    for i, n in enumerate(n_hyp):
        res.append((poses[o:o + n], scores[o:o + n], int(best[i]), info[i]))
        o += n
    return res


def _assert_alone(rig, cams, iterations=2, order=None, full=False):
    """register_cameras of `cams` equals register_objects of each camera alone, object by object, bit for bit."""
    e = rig["e"]
    frames, masks, grids, cam_of, slots, pairs = _objects(rig, cams, order, full)
    got = _split(e.register_cameras(frames, masks, grids, cam_of, slots, iterations), [len(g) for g in grids])
    for c, cam in enumerate(cams):
        idx = [i for i, (cc, _) in enumerate(pairs) if cc == c]
        alone = _split(e.register_objects(cam["rgb"], cam["depth"], cam["K"], np.stack([masks[i] for i in idx]),
                                          [grids[i] for i in idx], [slots[i] for i in idx], iterations), [len(grids[i]) for i in idx])
        for i, a in zip(idx, alone):
            g = got[i]
            assert torch.equal(g[0], a[0]), f"camera {c}, object {pairs[i][1]}: poses off by {(g[0] - a[0]).abs().max():.2e}"
            assert torch.equal(g[1], a[1]), f"camera {c}, object {pairs[i][1]}: scores differ"
            assert g[2] == a[2] and torch.equal(g[3], a[3]), f"camera {c}, object {pairs[i][1]}: best / info differ"
    return got


@pytest.mark.parametrize("n_cam", [1, 2, 4])
def test_equals_register_objects_of_each_camera(rig, n_cam):
    cams = rig["cams"][:n_cam]
    pairs = _objects(rig, cams)[5]
    interleaved = sorted(range(len(pairs)), key=lambda i: pairs[i][::-1])  # the first object of every camera, then the second
    _assert_alone(rig, cams, order=interleaved)


def test_full_grids(rig):
    """252 hypotheses per object: 2 + 1 + 2 objects over three cameras run as passes of 504 + 504 + 252, the second
    one holding objects of cameras 1 and 2."""
    _assert_alone(rig, rig["cams"][:3], full=True)


def test_several_passes_mixing_cameras(rig):
    """Four 252-pose objects over two cameras: passes of 504 + 504, each holding one object of each camera."""
    cams = [rig["cams"][0], rig["cams"][2]]
    _assert_alone(rig, cams, order=[0, 2, 1, 3], full=True)


def test_the_largest_number_of_cameras(rig):
    from foundationpose_b200.engine import MAX_CAMERAS

    objs = rig["objs"]
    cams = []
    for c in range(MAX_CAMERAS):
        H, W = (96, 128) if c % 2 else (121, 177)
        f = 1.1 * W
        K = [[f, 0, W / 2 - 1.5 * (c % 3)], [0, f * (1 + 0.01 * c), H / 2 + (c % 4)], [0, 0, 1]]
        cams.append(_camera(objs, H, W, K, [1 + c % 3], seed=40 + c))
    _assert_alone(rig, cams, order=list(range(MAX_CAMERAS))[::-1])


def test_against_the_oracle():
    from foundationpose_b200 import hypotheses, synth
    from foundationpose_b200.estimater import make_mesh_tensors

    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_golden_register_cameras as gen

    g = dict(np.load(GOLD))
    e = _engine()
    meshes, _, frames = gen.scene(int(g["seed"]))
    grids = []
    for k, m in enumerate(meshes):
        mesh = synth.vertex_coloured(m) if g["vertex_coloured"][k] else m.copy()
        mesh.vertices = mesh.vertices - g["model_centers"][k].reshape(1, 3)
        mt = make_mesh_tensors(mesh)
        e.set_mesh(mt["pos"], mt["normals"], mt["faces"], float(g["diameters"][k]), uv=mt.get("uv"), tex=mt.get("tex"),
                   vertex_colors=mt.get("vcolor"), slot=k + 1)
        grids.append(torch.from_numpy(hypotheses.make_rotation_grid(40, 60, gen.symmetry_tfs(str(g["symmetries"][k])))).cuda())
    assert [len(x) for x in grids] == list(g["n_hyp"])
    views = [(rgb, depth, g["K"][c]) for c, (rgb, depth, _) in enumerate(frames)]
    masks = gen.masks_of(frames)
    slots = list(range(1, len(meshes) + 1))
    start, _, _, info = e.register_cameras(views, masks, grids, g["camera_of"], slots, 0)
    np.testing.assert_allclose(start.cpu().numpy(), g["start"], atol=2e-6, rtol=0)
    np.testing.assert_allclose(info.cpu().numpy()[:, :3], g["centers"], atol=2e-6, rtol=0)
    poses, scores, best, _ = e.register_cameras(views, masks, grids, g["camera_of"], slots, int(g["iterations"]))
    perr = np.abs(poses.cpu().numpy() - g["refined"]).max()
    print(f"refined poses: max error {perr:.2e}")
    assert perr <= 2e-3
    # the selected index is held to the oracle's wherever the oracle's top-2 margin dominates the score error (the rule of
    # test_register_objects_gpu.py::test_against_the_oracle).  On this golden no object's margin does (measured on an
    # H100: score errors of 0.007-0.03 against margins of 0.014-0.044), so the rule is kept for a regenerated golden.
    s_all, best = scores.cpu().numpy(), best.cpu().numpy()
    o = 0
    for k, n in enumerate(g["n_hyp"]):
        s, gs = s_all[o:o + n], g["scores"][o:o + n]
        err = s - gs
        rank_err = np.abs(err - err.mean()).max()
        margin, spread = float(g["top2_margin"][k]), float(g["spread"][k])
        print(f"object {k}: rank-relevant score error {rank_err:.2e}, oracle spread {spread:.3f}, top-2 margin {margin:.3f}")
        assert int(best[k]) == int(np.argmax(s))
        # under the oracle's scores the selected hypothesis is within the score error of the oracle's best one
        assert gs[int(best[k])] >= gs.max() - 2 * rank_err, f"object {k}: selected {best[k]} scores far below the oracle's best"
        if margin >= 5 * rank_err:
            assert int(best[k]) == int(g["ids"][o]), f"object {k}: selected {best[k]}, oracle {g['ids'][o]}"
        o += n
    e.close()


def test_early_exit_object(rig):
    """An object without valid depth in its camera: its n_valid is below 4 and every other object's results are the
    same as without it."""
    e, cams = rig["e"], [dict(c) for c in rig["cams"][:2]]
    depth = cams[1]["depth"].copy()
    assert not any(m[5:45, 5:65].any() for m in cams[1]["masks"])
    depth[5:45, 5:65] = 0.0  # 10 px beyond the hole: the bilateral filter fills holes from up to 2 px away
    hole = np.zeros(depth.shape, bool)
    hole[15:35, 15:55] = True
    cams[1]["depth"] = depth
    frames, masks, grids, cam_of, slots, _ = _objects(rig, cams)
    with_bad = _split(e.register_cameras(frames, masks[:2] + [hole] + masks[2:], grids[:2] + [grids[2]] + grids[2:],
                                         cam_of[:2] + [1] + cam_of[2:], slots[:2] + [slots[2]] + slots[2:], 2),
                      [len(g) for g in grids[:2] + [grids[2]] + grids[2:]])
    without = _split(e.register_cameras(frames, masks, grids, cam_of, slots, 2), [len(g) for g in grids])
    assert float(with_bad[2][3][3]) < 4
    for a, b in zip(with_bad[:2] + with_bad[3:], without):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2] and torch.equal(a[3], b[3])


def test_graphs_are_reused(rig):
    """Passes of 461 + 209 hypotheses, in camera-major and in permuted object order alike."""
    e, cams = rig["e"], rig["cams"]
    frames, masks, grids, cam_of, slots, _ = _objects(rig, cams)
    n_hyp = [len(g) for g in grids]
    for _ in range(2):  # first sight of a pass size runs eagerly, the second captures
        base = _split(e.register_cameras(frames, masks, grids, cam_of, slots, 2), n_hyp)
    captures = e.graph_captures()
    again = _split(e.register_cameras(frames, masks, grids, cam_of, slots, 2), n_hyp)
    perm = [4, 0, 6, 2, 5, 1, 3]
    permuted = _split(e.register_cameras(frames, [masks[i] for i in perm], [grids[i] for i in perm], [cam_of[i] for i in perm],
                                         [slots[i] for i in perm], 2), [n_hyp[i] for i in perm])
    cam_perm = [2, 0, 3, 1]  # new camera i is old camera cam_perm[i]
    cams_permuted = _split(e.register_cameras([frames[i] for i in cam_perm], masks, grids, [cam_perm.index(c) for c in cam_of],
                                              slots, 2), n_hyp)
    assert e.graph_captures() == captures, "repeating the call or reordering objects or cameras captured a new graph"
    for i in range(len(base)):
        for a, b, c in zip(base[i], again[i], cams_permuted[i]):
            assert (torch.equal(a, b) and torch.equal(a, c)) if torch.is_tensor(a) else a == b == c
        j = perm.index(i)
        assert torch.equal(base[i][0], permuted[j][0]) and torch.equal(base[i][1], permuted[j][1])
    # other intrinsics for camera 1: no capture, and the same as a fresh context registering that rig
    moved = list(frames)
    K1 = frames[1][2].copy()
    K1[0, 2] += 3.0
    K1[1, 1] *= 1.01
    moved[1] = (frames[1][0], frames[1][1], K1)
    got = e.register_cameras(moved, masks, grids, cam_of, slots, 2)
    assert e.graph_captures() == captures, "new intrinsics captured a new graph"
    fresh = _engine(rig["objs"])
    want = fresh.register_cameras(moved, masks, grids, cam_of, slots, 2)
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    fresh.close()


def test_refusals_launch_nothing(rig):
    from foundationpose_b200 import _lib
    from foundationpose_b200._lib import lib
    from foundationpose_b200.engine import MAX_CAMERAS, _p, _stream

    e, cams = rig["e"], rig["cams"][:2]
    frames, masks, grids, cam_of, slots, _ = _objects(rig, cams)
    g = torch.cat(grids).contiguous()
    out = [torch.empty(len(g), 16, device="cuda"), torch.empty(len(g), device="cuda"),
           torch.empty(len(slots), dtype=torch.int32, device="cuda"), torch.empty(len(slots), 4, device="cuda")]
    m8 = [np.ascontiguousarray(m, dtype=np.uint8) for m in masks]

    def call(n_cam=2, cam_of=cam_of, slots=slots, n_hyp=None, null=None, H=None):
        idx = [c % 2 for c in range(n_cam)]
        rgbs = (C.c_void_p * max(n_cam, 1))(*[None if null == ("rgb", c) else cams[i]["rgb"].ctypes.data for c, i in enumerate(idx)])
        depths = (C.c_void_p * max(n_cam, 1))(*[cams[i]["depth"].ctypes.data for i in idx])
        Ks = (C.c_float * (9 * max(n_cam, 1)))(*[float(x) for i in idx for x in cams[i]["K"].reshape(-1)])
        Hs = (C.c_int * max(n_cam, 1))(*(H or [cams[i]["depth"].shape[0] for i in idx]))
        Ws = (C.c_int * max(n_cam, 1))(*[cams[i]["depth"].shape[1] for i in idx])
        M = len(slots)
        nh = n_hyp or [len(x) for x in grids]
        ms = (C.c_void_p * M)(*[None if null == ("mask", i) else m8[i].ctypes.data for i in range(M)])
        return lib.fp_register_cameras(e._h, n_cam, rgbs, depths, Ks, Hs, Ws, M, (C.c_int * M)(*cam_of), (C.c_int * M)(*slots),
                                       (C.c_int * M)(*nh), ms, _p(g), 2, *[_p(t) for t in out], _stream())

    assert call() == 0
    n0 = _lib.launch_count()
    bad = [dict(n_cam=0), dict(n_cam=MAX_CAMERAS + 1), dict(cam_of=[-1] + cam_of[1:]), dict(cam_of=cam_of[:-1] + [2]),
           dict(cam_of=[0] * len(cam_of)),  # camera 1 owns no object
           dict(slots=[64] + slots[1:]), dict(slots=slots[:-1] + [-1]), dict(slots=[40] + slots[1:]),  # 40: never loaded
           dict(n_hyp=[0, 126, 63]), dict(n_hyp=[4097, 126, 63]), dict(null=("rgb", 1)), dict(null=("mask", 2)), dict(H=[480, 0])]
    for kw in bad:
        assert call(**kw) != 0, kw
    with pytest.raises(ValueError):  # a mask of another camera's size
        e.register_cameras(frames, [masks[2]] + masks[1:], grids, cam_of, slots, 2)
    assert _lib.launch_count() == n0


def _estimators(e, rig, ks):
    from foundationpose_b200.estimater import FoundationPose, PoseRefinePredictor, ScorePredictor
    from foundationpose_b200.weights import random_state_dict

    refiner = PoseRefinePredictor(engine=e, state_dict=random_state_dict("refine", 0))
    scorer = ScorePredictor(engine=e, state_dict=random_state_dict("score", 0))
    out = []
    for n, k in enumerate(ks):
        m = rig["objs"][k][0].copy()
        m.vertices = m.vertices + np.array([0.004, -0.003, 0.002]) * (n + 1)  # off-centre: exercises the model_center shift
        out.append(FoundationPose(model_pts=m.vertices, model_normals=m.vertex_normals, mesh=m,
                                  symmetry_tfs=_symmetry(rig["objs"][k][3]), scorer=scorer, refiner=refiner))
    return out


def _state(est):
    return (est.pose_last.clone(), int(est.best_id), est.poses.clone(), est.scores.clone(), est.H, est.W, id(est.K), est.ob_id,
            id(est.ob_mask))


def test_public_api_equals_register_objects_per_view(rig):
    """estimater.register_cameras equals register_objects per view and register per object, in the returned poses and
    the estimators' state; a camera without estimators gives []; refusals reach no engine call."""
    from foundationpose_b200.estimater import register_cameras, register_objects

    e = _engine()
    cams = rig["cams"]
    ests = _estimators(e, rig, [0, 1, 2, 3, 1])  # camera 0 sees objects 0, 1; camera 1 object 2; camera 2 objects 3, 1
    views = [(ests[0:2], cams[0]["rgb"], cams[0]["depth"], cams[0]["K"], cams[0]["masks"]),
             ([], cams[3]["rgb"], cams[3]["depth"], cams[3]["K"], []),
             (ests[2:3], cams[1]["rgb"], cams[1]["depth"], cams[1]["K"], cams[1]["masks"]),
             (ests[3:5], cams[2]["rgb"], cams[2]["depth"], cams[2]["K"], cams[2]["masks"])]
    ob_ids = [[1, 2], None, [3], [4, 5]]
    got = register_cameras(views, ob_ids=ob_ids, iteration=3)
    got_state = [_state(est) for est in ests]
    want = [register_objects(v[0], v[3], v[1], v[2], v[4], ob_ids=i, iteration=3) for v, i in zip(views, ob_ids)]
    assert [len(v) for v in got] == [2, 0, 1, 2]
    for a, b in zip(got, want):
        assert all(np.array_equal(x, y) and x.dtype == y.dtype for x, y in zip(a, b))
    for g, est in zip(got_state, ests):
        w = _state(est)
        assert all(torch.equal(x, y) if torch.is_tensor(x) else x == y for x, y in zip(g, w))
    # and register() of each object alone
    for v, gv in zip(views, got):
        for est, m, pose in zip(v[0], v[4], gv):
            assert np.array_equal(est.register(K=v[3], rgb=v[1], depth=v[2], ob_mask=m, iteration=3), pose)
    other = _engine()
    stranger = _estimators(other, rig, [0])[0]
    n0 = e.graph_captures()
    with pytest.raises(ValueError):
        register_cameras([views[0], ([stranger],) + views[2][1:]])
    with pytest.raises(ValueError):
        register_cameras([views[0], ([ests[0]],) + views[2][1:]])
    with pytest.raises(ValueError):
        register_cameras([views[0], (views[2][0],) + views[2][1:4] + ([cams[0]["masks"][0]],)])
    with pytest.raises(TypeError):
        register_cameras([(views[0][0], torch.from_numpy(cams[0]["rgb"]).cuda(), cams[0]["depth"], cams[0]["K"], cams[0]["masks"])])
    assert register_cameras([]) == [] and register_cameras([views[1]]) == [[]]
    assert e.graph_captures() == n0
    other.close()
    e.close()


def test_then_track_cameras_equals_register_then_track_one(rig):
    from foundationpose_b200.estimater import register_cameras, track_cameras

    cams = rig["cams"][:3]
    e = _engine()
    ests = _estimators(e, rig, [0, 1, 2, 3, 1])
    groups = [ests[0:2], ests[2:3], ests[3:5]]
    views = [(g, c["rgb"], c["depth"], c["K"], c["masks"]) for g, c in zip(groups, cams)]
    register_cameras(views)
    uploads = []
    set_mesh = e.set_mesh
    e.set_mesh = lambda *a, **k: uploads.append(k.get("slot", 0)) or set_mesh(*a, **k)
    try:
        got = track_cameras([(g, c["rgb"], c["depth"], c["K"]) for g, c in zip(groups, cams)], iteration=2)
    finally:
        del e.set_mesh
    assert uploads == [], "track_cameras after register_cameras re-uploaded meshes"
    for g, c in zip(groups, cams):
        for est, m in zip(g, c["masks"]):
            est.register(K=c["K"], rgb=c["rgb"], depth=c["depth"], ob_mask=m)
    want = [[est.track_one(c["rgb"], c["depth"], c["K"], 2) for est in g] for g, c in zip(groups, cams)]
    for a, b in zip(got, want):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    e.close()


def _cycle(rig):
    e = _engine(rig["objs"])
    frames, masks, grids, cam_of, slots, _ = _objects(rig, rig["cams"][:2])
    for _ in range(3):
        e.register_cameras(frames, masks, grids, cam_of, slots, 2)
    e.close()
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def test_closing_returns_device_memory(rig):
    first = _cycle(rig)
    second = _cycle(rig)
    assert abs(second - first) <= 4 * MiB, f"free device memory moved by {(first - second) / MiB:.1f} MiB from one cycle to the next"
