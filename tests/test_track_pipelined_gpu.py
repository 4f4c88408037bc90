"""Non-blocking tracking (fp_track_*_submit + fp_track_wait, wait=False in Python) against the blocking calls on the same
seeded inputs: a sequence tracked with one call always in flight, collection order, a third submit, other entry points
and another stream between a submit and its wait, bad tickets, refused submits, close with calls pending, the golden of
track_cameras through the pipelined path, and examples/track_sequence_pipelined.py against a blocking track_one loop."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(os.path.dirname(__file__), "golden", "track_cameras.npz")
N_FRAMES = 30
# subdivisions, texture seed, scale
SPECS = [(3, 0, 1.0), (2, 5, 0.8), (3, 9, 1.2)]
# per camera: H, W, K, objects it sees (indices into SPECS); camera 0 sees two objects
CAMERAS = [(480, 640, [[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1]], [0, 1]),
           (360, 480, [[450.0, 0, 236.0], [0, 455.0, 182.0], [0, 0, 1]], [2]),
           (300, 400, [[380.0, 0, 204.0], [0, 385.0, 148.0], [0, 0, 1]], [1])]


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
    for k, m in enumerate(objs):
        _load(e, m, k + 1)
    if objs:
        _load(e, objs[0], 0)
    return e


@pytest.fixture(scope="module")
def rig():
    """N_FRAMES frames of every camera, each object moving along its own smooth random walk, and the (camera, object)
    pairs' start poses: the first frame's poses plus a few millimetres."""
    from foundationpose_b200 import synth

    objs = [synth.make_mesh(s, tex_seed=t, tex_size=256, scale=sc) for s, t, sc in SPECS]
    rng = np.random.default_rng(7)
    cams = []
    for c, (H, W, K, seen) in enumerate(CAMERAS):
        K = np.asarray(K, dtype=np.float64)
        walks = []
        for j, k in enumerate(seen):
            p = np.eye(4)
            p[:3, :3] = synth.random_rotation(11 + 5 * c + k)
            z = 0.6 + 0.05 * j
            p[:3, 3] = [((W * (j + 1) / (len(seen) + 1)) - K[0, 2]) * z / K[0, 0], 0.02 * (-1) ** j, z]
            walks.append(synth.track_sequence(N_FRAMES, p, seed=20 + 3 * c + j))
        frames, owners = [], []
        for t in range(N_FRAMES):
            rgb, depth, owner = synth.make_multi_scene([(objs[k].visual.image, walks[j][t], SPECS[k][2]) for j, k in enumerate(seen)],
                                                       K, H, W, seed=100 * c + t)
            frames.append((rgb, depth, K))
            owners.append(owner)
        start = []
        for w in walks:
            q = w[0].copy()
            q[:3, 3] += rng.normal(0, 0.003, 3)
            start.append(q.astype(np.float32))
        cams.append(dict(frames=frames, owners=owners, seen=list(seen), start=start))
    pairs = [(c, j) for c, cam in enumerate(cams) for j in range(len(cam["seen"]))]
    return dict(e=_engine(objs), objs=objs, cams=cams, pairs=pairs,
                cam_of=[c for c, _ in pairs], slots=[cams[c]["seen"][j] + 1 for c, j in pairs],
                start=torch.from_numpy(np.stack([cams[c]["start"][j] for c, j in pairs])).cuda())


def _views(rig, t):
    return [cam["frames"][t] for cam in rig["cams"]]


def _call(rig, kind, e, t, poses_in, wait):
    """One tracking call of frame t: `cameras` tracks every pair of every camera, `objects` camera 0's objects."""
    if kind == "cameras":
        return e.track_cameras(_views(rig, t), poses_in, rig["cam_of"], rig["slots"], 2, wait=wait)
    rgb, depth, K = rig["cams"][0]["frames"][t]
    return e.track_objects(rgb, depth, K, poses_in, [k + 1 for k in rig["cams"][0]["seen"]], 2, wait=wait)


def _start(rig, kind):
    return rig["start"] if kind == "cameras" else rig["start"][:len(rig["cams"][0]["seen"])]


def _blocking(rig, kind, e, frames=range(N_FRAMES)):
    """The sequence tracked with blocking calls, each frame starting from the previous one's device poses."""
    pose, dev, host = _start(rig, kind), [], []
    for t in frames:
        pose, h = _call(rig, kind, e, t, pose, True)
        dev.append(pose.clone())
        host.append(h)
    return dev, host


def _assert_same(dev, host, want_dev, want_host, what):
    torch.cuda.synchronize()
    for t, (a, b, x, y) in enumerate(zip(dev, want_dev, host, want_host)):
        assert torch.equal(a, b), f"{what}: frame {t}: device poses differ"
        assert np.array_equal(x, y), f"{what}: frame {t}: host poses off by {np.abs(x - y).max():.2e}"


@pytest.fixture(scope="module")
def reference(rig):
    return {kind: _blocking(rig, kind, rig["e"]) for kind in ("cameras", "objects")}


@pytest.mark.parametrize("kind", ["cameras", "objects"])
def test_sequence_with_one_call_in_flight(rig, reference, kind):
    e = rig["e"]
    pose, dev, host, prev = _start(rig, kind), [], [], None
    for t in range(N_FRAMES):
        pose, pending = _call(rig, kind, e, t, pose, False)  # submit t ...
        dev.append(pose)
        if prev is not None:
            host.append(prev.result())  # ... then collect t - 1
        prev = pending
    host.append(prev.result())
    _assert_same(dev, host, *reference[kind], f"track_{kind}")


@pytest.mark.parametrize("kind", ["cameras", "objects"])
def test_public_api_sequence(rig, kind):
    """estimater.track_cameras / track_objects with wait=False: pose_last is set at submit, result() is the blocking list."""
    from foundationpose_b200 import estimater
    from foundationpose_b200.weights import random_state_dict

    e = _engine()
    refiner = estimater.PoseRefinePredictor(engine=e, state_dict=random_state_dict("refine", 0))
    scorer = estimater.ScorePredictor(engine=e, state_dict=random_state_dict("score", 0))
    ests = {}
    for c, j in rig["pairs"]:
        m = rig["objs"][rig["cams"][c]["seen"][j]].copy()
        m.vertices = m.vertices + np.array([0.01, -0.02, 0.005]) * (len(ests) + 1)  # off-centre: the un-centring shift
        ests[(c, j)] = estimater.FoundationPose(model_pts=m.vertices, model_normals=m.vertex_normals, mesh=m, scorer=scorer,
                                                refiner=refiner)
    cams = rig["cams"] if kind == "cameras" else rig["cams"][:1]

    def reset():
        for (c, j), est in ests.items():
            est.pose_last = torch.from_numpy(rig["cams"][c]["start"][j]).cuda().reshape(1, 4, 4)

    def call(t, wait):
        if kind == "cameras":
            views = [([ests[(c, j)] for j in range(len(cam["seen"]))], *cam["frames"][t]) for c, cam in enumerate(cams)]
            return estimater.track_cameras(views, iteration=2, wait=wait)
        return estimater.track_objects([ests[(0, j)] for j in range(len(cams[0]["seen"]))], *cams[0]["frames"][t], iteration=2,
                                       wait=wait)

    reset()
    want, want_last = [], []
    for t in range(N_FRAMES):
        want.append(call(t, True))
        want_last.append({k: est.pose_last.clone() for k, est in ests.items()})
    reset()
    got, last, prev = [], [], None
    for t in range(N_FRAMES):
        pending = call(t, False)
        last.append({k: est.pose_last for k, est in ests.items()})
        if prev is not None:
            got.append(prev.result())
        prev = pending
    got.append(prev.result())
    assert got[-1] is prev.result(), "result() returns the same list on every call"
    torch.cuda.synchronize()
    for t in range(N_FRAMES):
        assert all(torch.equal(last[t][k], want_last[t][k]) for k in ests), f"frame {t}: pose_last differs"
        flat = lambda r: [p for v in r for p in v] if kind == "cameras" else r
        assert len(flat(got[t])) == len(flat(want[t]))
        assert all(np.array_equal(a, b) for a, b in zip(flat(got[t]), flat(want[t]))), f"frame {t}"
    e.close()


def test_golden_through_the_pipelined_path():
    """tests/golden/track_cameras.npz at test_track_cameras_gpu.py's bar, every frame submitted before the previous one
    is collected."""
    from foundationpose_b200 import synth

    g = dict(np.load(GOLD))
    meshes = [synth.make_mesh(int(g["subdivisions"][k]), tex_seed=int(g["tex_seeds"][k]), tex_size=int(g["tex_size"]),
                              scale=float(g["scales"][k])) for k in range(len(g["scales"]))]
    e = _engine()
    for k, m in enumerate(meshes):
        _load(e, synth.vertex_coloured(m) if g["vertex_coloured"][k] else m, k + 1)
    T = g["extrinsic"]
    pairs = g["pairs"]
    order = np.array([0, 3, 1, 4, 2])
    got, prev = [], None
    for i in range(len(g["pose_in"])):
        frames = []
        for c in range(len(g["K"])):
            objs = [(m.visual.image, (T if c else np.eye(4)) @ g["gt"][k, i + 1], float(g["scales"][k])) for k, m in enumerate(meshes)]
            rgb, depth, _ = synth.make_multi_scene(objs, g["K"][c], int(g["H"][c]), int(g["W"][c]), seed=2 + i + 100 * c)
            frames.append((rgb, depth, g["K"][c]))
        _, pending = e.track_cameras(frames, torch.from_numpy(g["pose_in"][i][order]).cuda(), pairs[order, 0], pairs[order, 1] + 1,
                                     2, wait=False)
        if prev is not None:
            got.append(prev.result())
        prev = pending
    got.append(prev.result())
    for i, host in enumerate(got):
        err = np.abs(host - g["pose_out"][i][order])
        assert err.max() <= 1e-3, f"frame {i + 1}: pose off by {err.max():.2e}"
    e.close()


def test_no_new_captures_when_alternating(rig, reference):
    e = rig["e"]
    for _ in range(3):
        _call(rig, "cameras", e, 0, rig["start"], True)
    captures = e.graph_captures()
    pose, prev = rig["start"], None
    for t in range(6):
        pose, res = _call(rig, "cameras", e, t, pose, t % 2 == 0)
        if t % 2 == 0:
            assert np.array_equal(res, reference["cameras"][1][t])
        else:
            prev = res
    assert np.array_equal(prev.result(), reference["cameras"][1][5])
    assert e.graph_captures() == captures, "a non-blocking call captured a new graph"


def test_host_frames_are_free_after_submit(rig, reference):
    e = rig["e"]
    frames = [(rgb.copy(), depth.copy(), K) for rgb, depth, K in _views(rig, 0)]
    dev, pending = e.track_cameras(frames, rig["start"], rig["cam_of"], rig["slots"], 2, wait=False)
    for rgb, depth, _ in frames:
        rgb[...] = 255 - rgb
        depth[...] = 0.0
    dev2, pending2 = e.track_cameras(frames, dev, rig["cam_of"], rig["slots"], 2, wait=False)  # the overwritten frames
    assert np.array_equal(pending.result(), reference["cameras"][1][0])
    torch.cuda.synchronize()
    assert torch.equal(dev, reference["cameras"][0][0])
    pending2.result()


def test_third_submit_and_collection_order(rig, reference):
    """Three submits with nothing collected (the third waits for the first call's uploads), then collected newest first."""
    e = rig["e"]
    pose, pend, dev = rig["start"], [], []
    for t in range(3):
        pose, p = _call(rig, "cameras", e, t, pose, False)
        pend.append(p)
        dev.append(pose)
    host = [p.result() for p in pend[::-1]][::-1]
    _assert_same(dev, host, reference["cameras"][0][:3], reference["cameras"][1][:3], "third submit")


def _interleaved_calls(rig):
    """Other entry points, each a function of the engine returning host arrays, independent of the tracking state."""
    from foundationpose_b200 import synth

    cam = rig["cams"][1]
    rgb, depth, K = cam["frames"][3]
    start = torch.from_numpy(np.stack(cam["start"])).cuda()
    masks = np.stack([cam["owners"][3] == j for j in range(len(cam["seen"]))])
    grid = np.tile(np.eye(4, dtype=np.float32), (8, 1, 1))
    for s in range(8):
        grid[s, :3, :3] = synth.random_rotation(s)
    grids = [torch.from_numpy(grid).cuda()]
    slots = [k + 1 for k in cam["seen"]]

    def register(e):
        poses, scores, best, info = e.register_objects(rgb, depth, K, masks, grids, slots, 2)
        return [poses.cpu().numpy(), scores.cpu().numpy(), best.cpu().numpy(), info.cpu().numpy()]

    def refine(e):
        e.set_frame(rgb, depth, K, filter_depth=True, zfar=float("inf"))
        return [x.cpu().numpy() for x in e.refine(start, 2)]

    def vis(e):
        e.set_frame(rgb, depth, K, filter_depth=False)
        return [e.vis("refine", start, start + 0.001).cpu().numpy()]

    return dict(register_objects=register, set_frame_refine=refine, vis=vis)


@pytest.mark.parametrize("other", ["register_objects", "set_frame_refine", "vis"])
def test_other_entry_points_between_submit_and_wait(rig, reference, other):
    e = rig["e"]
    fn = _interleaved_calls(rig)[other]
    _call(rig, "cameras", e, 0, rig["start"], True)
    want = fn(e)
    dev, pending = _call(rig, "cameras", e, 0, rig["start"], False)
    got = fn(e)
    assert np.array_equal(pending.result(), reference["cameras"][1][0]), other
    torch.cuda.synchronize()
    assert torch.equal(dev, reference["cameras"][0][0]), other
    assert all(np.array_equal(a, b) for a, b in zip(got, want)), f"{other} changed with a tracking call in flight"


def test_submits_from_two_streams(rig, reference):
    e = rig["e"]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    pose, dev, host, prev = rig["start"], [], [], None
    for t in range(8):
        with torch.cuda.stream(streams[t % 2]):
            pose, pending = _call(rig, "cameras", e, t, pose, False)
        dev.append(pose)
        if prev is not None:
            host.append(prev.result())
        prev = pending
    host.append(prev.result())
    torch.cuda.synchronize()
    _assert_same(dev, host, reference["cameras"][0][:8], reference["cameras"][1][:8], "two streams")


def test_bad_tickets_are_refused(rig, reference):
    from foundationpose_b200 import _lib
    from foundationpose_b200._lib import lib

    e = rig["e"]
    _, pending = _call(rig, "cameras", e, 0, rig["start"], False)
    out = np.empty((len(rig["slots"]), 4, 4), dtype=np.float32)
    assert lib.fp_track_wait(e._h, pending.ticket, C.c_void_p(out.ctypes.data)) == 0
    assert np.array_equal(out, reference["cameras"][1][0])
    with pytest.raises(_lib.FposeError):
        pending.result()  # the second wait on that ticket
    for t in (0, pending.ticket + 1000):
        with pytest.raises(_lib.FposeError):
            e._wait(t, out)
    _, host = _call(rig, "cameras", e, 1, reference["cameras"][0][0], True)
    assert np.array_equal(host, reference["cameras"][1][1])


def test_refused_submits_enqueue_nothing(rig, reference):
    from foundationpose_b200 import _lib

    e = rig["e"]
    views = _views(rig, 0)
    dev, pending = _call(rig, "cameras", e, 0, rig["start"], False)
    n0 = _lib.launch_count()
    bad = [dict(cam_of=[3] + rig["cam_of"][1:]), dict(cam_of=[0] * len(rig["cam_of"])), dict(slots=[64] + rig["slots"][1:]),
           dict(slots=[40] + rig["slots"][1:])]
    for kw in bad:
        args = {**dict(cam_of=rig["cam_of"], slots=rig["slots"]), **kw}
        with pytest.raises(_lib.FposeError):
            e.track_cameras(views, rig["start"], args["cam_of"], args["slots"], 2, wait=False)
    with pytest.raises(_lib.FposeError):
        e.track_objects(*views[0], rig["start"][:2], [1, 40], 2, wait=False)
    assert _lib.launch_count() == n0, "a refused submit enqueued work"
    assert np.array_equal(pending.result(), reference["cameras"][1][0])
    torch.cuda.synchronize()
    assert torch.equal(dev, reference["cameras"][0][0])


def test_close_with_calls_pending(rig):
    import gc

    from foundationpose_b200 import _lib

    e = _engine(rig["objs"])
    pose, kept = rig["start"], None
    for t in range(4):
        pose, pending = _call(rig, "cameras", e, t, pose, False)
        if t == 1:
            kept = pending
    del pending
    gc.collect()  # the last handle is dropped without result(): the engine collects its ticket
    e.close()
    with pytest.raises(_lib.FposeError):
        kept.result()


def test_example_equals_blocking_track_one(tmp_path):
    import sys

    from foundationpose_b200 import synth

    scene = str(tmp_path / "scene")
    synth.write_demo_scene(scene, n_frames=8, subdivisions=3)
    spec = importlib.util.spec_from_file_location("track_sequence_pipelined", os.path.join(ROOT, "examples", "track_sequence_pipelined.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    out = str(tmp_path / "pipelined")
    ex.run(scene + "/mesh/textured_simple.obj", scene, out, est_refine_iter=5, track_refine_iter=2)
    # the same flow with the blocking drop-in call, run_demo.py's loop
    dropin = os.path.join(ROOT, "foundationpose_b200", "dropin")
    if dropin not in sys.path:
        sys.path.insert(0, dropin)
    from datareader import YcbineoatReader
    from Utils import trimesh

    from foundationpose_b200.estimater import FoundationPose, PoseRefinePredictor, ScorePredictor

    mesh = trimesh.load(scene + "/mesh/textured_simple.obj")
    est = FoundationPose(model_pts=mesh.vertices, model_normals=mesh.vertex_normals, mesh=mesh, scorer=ScorePredictor(),
                         refiner=PoseRefinePredictor())
    reader = YcbineoatReader(video_dir=scene, shorter_side=None, zfar=np.inf)
    for i in range(len(reader.color_files)):
        color, depth = reader.get_color(i), reader.get_depth(i)
        if i == 0:
            pose = est.register(K=reader.K, rgb=color, depth=depth, ob_mask=reader.get_mask(0).astype(bool), iteration=5)
        else:
            pose = est.track_one(rgb=color, depth=depth, K=reader.K, iteration=2)
        got = np.loadtxt(os.path.join(out, "ob_in_cam", f"{reader.id_strs[i]}.txt"))
        assert np.array_equal(got, _saved(pose, tmp_path)), f"frame {i}"


def _saved(pose, tmp_path):
    """`pose` as np.savetxt writes it and np.loadtxt reads it back (the example's file format)."""
    f = str(tmp_path / "blocking.txt")
    np.savetxt(f, pose.reshape(4, 4))
    return np.loadtxt(f)
