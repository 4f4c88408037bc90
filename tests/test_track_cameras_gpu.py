"""fp_track_cameras (objects of several camera streams, ONE graph launch) against fp_track_objects per camera, fp_track
and the by-value fp_set_frame + fp_refine per object, against the CPU oracle (tests/golden/track_cameras.npz,
tools/make_golden_track_cameras.py), its graph caching, its refusals, and estimater.track_cameras against track_one."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden", "track_cameras.npz")
# subdivisions, texture seed, scale, vertex-coloured, open
SPECS = [(3, 0, 1.0, False, False), (2, 5, 0.7, True, False), (3, 9, 1.3, False, True), (2, 2, 0.85, True, True),
         (4, 4, 1.1, False, False), (2, 7, 0.9, False, True)]
# per camera: H, W, K, objects it sees (indices into SPECS)
CAMERAS = [(480, 640, [[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1]], [0, 1, 2]),
           (720, 1280, [[920.0, 0, 640.0], [0, 915.0, 360.0], [0, 0, 1]], [3, 4]),
           (360, 480, [[450.0, 0, 236.0], [0, 455.0, 182.0], [0, 0, 1]], [5]),
           (600, 800, [[700.0, 0, 410.0], [0, 690.0, 290.0], [0, 0, 1]], [1, 3])]


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


def _engine(objs=()):
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.weights import random_state_dict

    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.set_config("refine")
    for k, (m, _, _) in enumerate(objs):
        _load(e, m, k + 1)
    return e


def _camera(objs, H, W, K, seen, seed, scale_xy=1.0):
    """A frame of camera (H, W, K) showing objects `seen`; the start pose of each is its pose plus a little noise."""
    from foundationpose_b200 import synth

    K = np.asarray(K, dtype=np.float64)
    rng = np.random.default_rng(seed)
    gt, start = [], []
    for j, k in enumerate(seen):
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(30 + 7 * seed + k)
        z = 0.6 + 0.05 * j
        p[:3, 3] = [((W * (j + 1) / (len(seen) + 1)) - K[0, 2]) * z / K[0, 0] * scale_xy, 0.03 * (-1) ** j, z]
        gt.append(p)
        q = p.copy()
        q[:3, 3] += rng.normal(0, 0.004, 3)
        start.append(q.astype(np.float32))
    rgb, depth, owner = synth.make_multi_scene([(objs[k][1], p, objs[k][2]) for k, p in zip(seen, gt)], K, H, W, seed=seed)
    assert all((owner == j).any() for j in range(len(seen)))
    return dict(rgb=rgb, depth=depth, K=K, seen=list(seen), start=np.stack(start))


@pytest.fixture(scope="module")
def rig():
    objs = [_object(*s) for s in SPECS]
    cams = [_camera(objs, H, W, K, seen, seed=3 + c) for c, (H, W, K, seen) in enumerate(CAMERAS)]
    return dict(e=_engine(objs), objs=objs, cams=cams)


def _pairs(cams, order=None):
    """(frames, start poses, camera ids, slots) of every (camera, object) pair, in `order` (default camera-major)."""
    pairs = [(c, j) for c, cam in enumerate(cams) for j in range(len(cam["seen"]))]
    if order is not None:
        pairs = [pairs[i] for i in order]
    frames = [(cam["rgb"], cam["depth"], cam["K"]) for cam in cams]
    start = torch.from_numpy(np.stack([cams[c]["start"][j] for c, j in pairs])).cuda()
    return frames, start, [c for c, _ in pairs], [cams[c]["seen"][j] + 1 for c, j in pairs], pairs


def _alone(e, cam):
    """fp_track_objects of one camera's objects (fp_track_cameras' one-camera case, with that camera as camera 0)."""
    _, host = e.track_objects(cam["rgb"], cam["depth"], cam["K"], torch.from_numpy(cam["start"]).cuda(),
                              [k + 1 for k in cam["seen"]], 2)
    return host


def _single(e, objs, cam, j):
    """Object j of a camera alone, its mesh in slot 0: {path: pose} for fp_track (the camera-table path) and for the
    by-value path fp_set_frame (filtered, zfar = inf) + fp_refine."""
    _load(e, objs[cam["seen"][j]][0], 0)
    start = torch.from_numpy(cam["start"][j]).cuda()
    tracked = e.track(cam["rgb"], cam["depth"], cam["K"], start, 2)[1]
    e.set_frame(cam["rgb"], cam["depth"], cam["K"], filter_depth=True, zfar=float("inf"))
    return {"track": tracked, "set_frame + refine": e.refine(start, 2)[0][0].cpu().numpy()}


@pytest.mark.parametrize("C", [1, 2, 4])
def test_equals_tracking_each_camera_alone(rig, C):
    e, cams = rig["e"], rig["cams"][:C]
    # interleaved: the first object of every camera, then the second, ...
    camera_major = _pairs(cams)[4]
    order = sorted(range(len(camera_major)), key=lambda i: camera_major[i][::-1])
    frames, start, cam_of, slots, pairs = _pairs(cams, order)
    dev, host = e.track_cameras(frames, start, cam_of, slots, 2)
    assert np.array_equal(dev.cpu().numpy(), host), "device and host copies of the poses differ"
    alone = [_alone(e, cam) for cam in cams]
    for i, (c, j) in enumerate(pairs):
        assert np.array_equal(host[i], alone[c][j]), f"C={C}, camera {c}, object {j}: off by {np.abs(host[i] - alone[c][j]).max():.2e}"
        for path, single in _single(e, rig["objs"], cams[c], j).items():
            assert np.array_equal(host[i], single), f"C={C}, camera {c}, object {j}: off {path} by {np.abs(host[i] - single).max():.2e}"


def test_the_largest_number_of_cameras(rig):
    from foundationpose_b200.engine import MAX_CAMERAS

    objs = rig["objs"]
    cams = []
    for c in range(MAX_CAMERAS):
        H, W = (96, 128) if c % 2 else (120, 176)
        f = 1.1 * W
        K = [[f, 0, W / 2 - 1.5 * (c % 3)], [0, f * (1 + 0.01 * c), H / 2 + (c % 4)], [0, 0, 1]]
        cams.append(_camera(objs, H, W, K, [c % len(objs)], seed=40 + c))
    e = rig["e"]
    frames, start, cam_of, slots, pairs = _pairs(cams, list(range(MAX_CAMERAS))[::-1])
    _, host = e.track_cameras(frames, start, cam_of, slots, 2)
    for i, (c, j) in enumerate(pairs):
        assert np.array_equal(host[i], _alone(e, cams[c])[j]), f"camera {c}"
        for path, single in _single(e, objs, cams[c], j).items():
            assert np.array_equal(host[i], single), f"camera {c}: {path}"


def test_against_the_oracle():
    from foundationpose_b200 import synth

    g = dict(np.load(GOLD))
    meshes = [synth.make_mesh(int(g["subdivisions"][k]), tex_seed=int(g["tex_seeds"][k]), tex_size=int(g["tex_size"]),
                              scale=float(g["scales"][k])) for k in range(len(g["scales"]))]
    e = _engine()
    for k, m in enumerate(meshes):
        _load(e, synth.vertex_coloured(m) if g["vertex_coloured"][k] else m, k + 1)
        assert abs(synth.mesh_diameter(m.vertices) - g["diameters"][k]) < 1e-12
    T = g["extrinsic"]
    pairs = g["pairs"]
    order = np.array([0, 3, 1, 4, 2])  # the pairs in interleaved camera order
    worst = 0.0
    for i in range(len(g["pose_in"])):
        frames = []
        for c in range(len(g["K"])):
            objs = [(m.visual.image, (T if c else np.eye(4)) @ g["gt"][k, i + 1], float(g["scales"][k])) for k, m in enumerate(meshes)]
            rgb, depth, _ = synth.make_multi_scene(objs, g["K"][c], int(g["H"][c]), int(g["W"][c]), seed=2 + i + 100 * c)
            frames.append((rgb, depth, g["K"][c]))
        _, host = e.track_cameras(frames, torch.from_numpy(g["pose_in"][i][order]).cuda(), pairs[order, 0], pairs[order, 1] + 1, 2)
        err = np.abs(host - g["pose_out"][i][order])
        worst = max(worst, err.max())
        assert err.max() <= 1e-3, f"frame {i + 1}: pose off by {err.max():.2e} (per pair {err.reshape(len(pairs), -1).max(1)})"
    print(f"track_cameras over {len(g['pose_in'])} frames x {len(pairs)} (object, camera) pairs: worst error {worst:.2e}")
    e.close()


def test_graphs_are_reused(rig):
    from foundationpose_b200 import _lib

    e, cams, objs = rig["e"], rig["cams"], rig["objs"]
    frames, start, cam_of, slots, _ = _pairs(cams)
    for _ in range(3):  # first sight runs eagerly, the second call captures, later calls replay
        _, base = e.track_cameras(frames, start, cam_of, slots, 2)
    captures = e.graph_captures()
    _, again = e.track_cameras(frames, start, cam_of, slots, 2)
    assert np.array_equal(again, base)
    perm = [5, 0, 7, 2, 4, 1, 6, 3]
    _, permuted = e.track_cameras(frames, start[perm], [cam_of[i] for i in perm], [slots[i] for i in perm], 2)
    assert np.array_equal(permuted, base[perm])
    cam_perm = [2, 0, 3, 1]  # new camera i is old camera cam_perm[i]
    _, cams_permuted = e.track_cameras([frames[i] for i in cam_perm], start, [cam_perm.index(c) for c in cam_of], slots, 2)
    assert np.array_equal(cams_permuted, base)
    assert e.graph_captures() == captures, "reordering objects or cameras captured a new graph"
    # other intrinsics for camera 1: the same as a fresh context tracking that rig
    moved = list(frames)
    K1 = frames[1][2].copy()
    K1[0, 2] += 3.0
    K1[1, 1] *= 1.01
    moved[1] = (frames[1][0], frames[1][1], K1)
    _, got = e.track_cameras(moved, start, cam_of, slots, 2)
    assert e.graph_captures() == captures, "new intrinsics captured a new graph"
    fresh = _engine(objs)
    _, want = fresh.track_cameras(moved, start, cam_of, slots, 2)
    fresh.close()
    assert np.array_equal(got, want)
    assert not np.array_equal(got[3:5], base[3:5]) and np.array_equal(got[:3], base[:3])
    # one launch sequence per call, whatever the number of cameras and objects
    per_call = {}
    for n_cam, M in ((1, 1), (4, 8)):
        f, st, co, sl = frames[:n_cam], start[:M], cam_of[:M], slots[:M]
        for _ in range(3):
            e.track_cameras(f, st, co, sl, 2)
        n0 = _lib.launch_count()
        e.track_cameras(f, st, co, sl, 2)
        per_call[(n_cam, M)] = _lib.launch_count() - n0
    assert per_call[(1, 1)] == per_call[(4, 8)], per_call


def test_other_paths_keep_their_graphs(rig):
    """Interleaving the rig (camera 0 640x480, a 1280x720 camera) with track_objects and track on another camera's frame
    captures nothing once every path is warm: each graph keeps the frame it was captured with."""
    e, cams, objs = rig["e"], rig["cams"], rig["objs"]
    frames, start, cam_of, slots, _ = _pairs(cams)
    _load(e, objs[cams[2]["seen"][0]][0], 0)

    def round_():
        out = [e.track_cameras(frames, start, cam_of, slots, 2)[1], _alone(e, cams[1]), _alone(e, cams[2])]
        out.append(e.track(cams[2]["rgb"], cams[2]["depth"], cams[2]["K"], torch.from_numpy(cams[2]["start"][0]).cuda(), 2)[1])
        return out

    for _ in range(3):
        first = round_()
    captures = e.graph_captures()
    again = round_()
    assert e.graph_captures() == captures, "a frame of another size or other intrinsics recaptured another path's graph"
    assert all(np.array_equal(a, b) for a, b in zip(first, again))


def test_context_frame_stays_consistent(rig):
    """After a multi-camera call the context holds camera 0's frame; track / track_objects on it equal a fresh context."""
    e, cams, objs = rig["e"], rig["cams"], rig["objs"]
    frames, start, cam_of, slots, _ = _pairs(cams)
    fresh = _engine(objs)
    for first in (1, 0):  # camera 0 with another frame size, then the same one as the calls below
        order = [first] + [c for c in range(len(cams)) if c != first]
        e.track_cameras([frames[c] for c in order], start, [order.index(c) for c in cam_of], slots, 2)
        for c in (0, 1):
            assert np.array_equal(_alone(e, cams[c]), _alone(fresh, cams[c])), f"track_objects, camera {c}"
        for eng in (e, fresh):
            _load(eng, objs[cams[1]["seen"][0]][0], 0)
        got = e.track(cams[1]["rgb"], cams[1]["depth"], cams[1]["K"], torch.from_numpy(cams[1]["start"][0]).cuda(), 2)[1]
        want = fresh.track(cams[1]["rgb"], cams[1]["depth"], cams[1]["K"], torch.from_numpy(cams[1]["start"][0]).cuda(), 2)[1]
        assert np.array_equal(got, want), "track"
        # and the multi-camera call after those single-camera ones
        _, a = e.track_cameras(frames, start, cam_of, slots, 2)
        _, b = fresh.track_cameras(frames, start, cam_of, slots, 2)
        assert np.array_equal(a, b)
    fresh.close()


def test_bad_arguments_are_refused_before_any_launch(rig):
    from foundationpose_b200 import _lib
    from foundationpose_b200.engine import MAX_CAMERAS, _p, _stream
    from foundationpose_b200._lib import lib

    e, cams = rig["e"], rig["cams"][:2]
    frames, start, cam_of, slots, _ = _pairs(cams)

    def call(n_cam=2, cam_of=cam_of, slots=slots, null=None, H=None, W=None):
        idx = [c % 2 for c in range(n_cam)]
        rgbs = (C.c_void_p * n_cam)(*[None if null == ("rgb", c) else cams[i]["rgb"].ctypes.data for c, i in enumerate(idx)])
        depths = (C.c_void_p * n_cam)(*[None if null == ("depth", c) else cams[i]["depth"].ctypes.data for c, i in enumerate(idx)])
        Ks = (C.c_float * (9 * n_cam))(*[float(x) for i in idx for x in cams[i]["K"].reshape(-1)])
        Hs = (C.c_int * n_cam)(*(H or [cams[i]["depth"].shape[0] for i in idx]))
        Ws = (C.c_int * n_cam)(*(W or [cams[i]["depth"].shape[1] for i in idx]))
        M = len(slots)
        out = torch.empty(M, 4, 4, device="cuda")
        return lib.fp_track_cameras(e._h, n_cam, rgbs, depths, Ks, Hs, Ws, M, (C.c_int * M)(*cam_of), (C.c_int * M)(*slots),
                                    _p(start[:M].contiguous()), 2, _p(out), None, _stream())

    assert call() == 0
    n0 = _lib.launch_count()
    bad = [dict(n_cam=0), dict(n_cam=MAX_CAMERAS + 1), dict(cam_of=[-1] + cam_of[1:]), dict(cam_of=cam_of[:-1] + [2]),
           dict(cam_of=[0] * len(cam_of)),  # camera 1 owns no object
           dict(slots=[64] + slots[1:]), dict(slots=slots[:-1] + [-1]), dict(slots=[40] + slots[1:]),  # 40: never loaded
           dict(null=("rgb", 1)), dict(null=("depth", 0)), dict(H=[480, 0]), dict(W=[-640, 1280])]
    for kw in bad:
        assert call(**kw) != 0, kw
    assert _lib.launch_count() == n0


def test_public_api_equals_track_one_in_turn(rig):
    from foundationpose_b200.estimater import FoundationPose, PoseRefinePredictor, ScorePredictor, track_cameras
    from foundationpose_b200.weights import random_state_dict

    def estimators(e):
        refiner = PoseRefinePredictor(engine=e, state_dict=random_state_dict("refine", 0))
        scorer = ScorePredictor(engine=e, state_dict=random_state_dict("score", 0))
        out = {}
        for k in (0, 1, 2, 3, 4):
            m = rig["objs"][k][0].copy()
            m.vertices = m.vertices + np.array([0.01, -0.02, 0.005]) * (k + 1)  # off-centre: exercises the un-centring shift
            out[k] = FoundationPose(model_pts=m.vertices, model_normals=m.vertex_normals, mesh=m, scorer=scorer, refiner=refiner)
        return out

    e = _engine()
    cams = rig["cams"]
    ests = estimators(e)
    # camera 0 sees objects 0, 1, 2; camera 1 objects 3, 4; a third camera sees none.  Each estimator is one object of one
    # camera: object 1 of camera 3 would be a second estimator for the same object, which track_one could not compare.
    views = [([ests[k] for k in cams[0]["seen"]], cams[0]["rgb"], cams[0]["depth"], cams[0]["K"]),
             ([], cams[2]["rgb"], cams[2]["depth"], cams[2]["K"]),
             ([ests[k] for k in cams[1]["seen"]], cams[1]["rgb"], cams[1]["depth"], cams[1]["K"])]

    def reset():
        for c in (0, 1):
            for j, k in enumerate(cams[c]["seen"]):
                ests[k].pose_last = torch.from_numpy(cams[c]["start"][j]).cuda().reshape(1, 4, 4)

    reset()
    got = track_cameras(views, iteration=2)
    got_last = {k: est.pose_last.cpu() for k, est in ests.items()}
    reset()
    want = [[est.track_one(rgb, depth, K, 2) for est in v] for v, rgb, depth, K in views]
    assert [len(v) for v in got] == [3, 0, 2]
    for a, b in zip(got, want):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
    for k, est in ests.items():
        assert torch.equal(got_last[k], est.pose_last.cpu())
    other = _engine()
    stranger = estimators(other)[0]
    stranger.pose_last = ests[0].pose_last.clone()
    with pytest.raises(ValueError):
        track_cameras([views[0], ([stranger], cams[1]["rgb"], cams[1]["depth"], cams[1]["K"])])
    with pytest.raises(ValueError):
        track_cameras([views[0], ([ests[0]], cams[1]["rgb"], cams[1]["depth"], cams[1]["K"])])
    with pytest.raises(TypeError):
        track_cameras([(views[0][0], torch.from_numpy(cams[0]["rgb"]).cuda(), torch.from_numpy(cams[0]["depth"]).cuda(), cams[0]["K"])])
    assert track_cameras([]) == []
    other.close()
    e.close()
