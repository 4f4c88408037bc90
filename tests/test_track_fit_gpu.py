"""The tracking calls with a fit (fp_track_cameras_fit_submit / fp_track_fit_wait, Engine.track_cameras(fit_delta=),
the estimator's fit_delta): the poses are those of the same call without a fit, bit for bit; the counts equal, integer
for integer, an independent path (the scorer-window vis record of the same poses) and the host reference
(tests/fit_reference.py); they do not depend on the number or order of objects and cameras, the crop tile, blocking,
host or device frames, or graphs; the graphs are reused; bad arguments are refused before anything is enqueued."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import crop_reference as cr
import fit_reference as fr

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "track_seq.npz")
DELTA = 0.01
# subdivisions, texture seed, scale, vertex-coloured, open
SPECS = [(3, 0, 1.0, False, False), (2, 5, 0.7, True, False), (3, 9, 1.3, False, True), (2, 2, 0.85, True, True)]
# per camera: H, W, K, objects it sees (indices into SPECS); cameras of different sizes and intrinsics
CAMERAS = [(480, 640, [[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1]], [0, 1, 2]),
           (720, 1280, [[920.0, 0, 640.0], [0, 915.0, 360.0], [0, 0, 1]], [3, 0]),
           (360, 480, [[450.0, 0, 236.0], [0, 455.0, 182.0], [0, 0, 1]], [2]),
           (600, 800, [[700.0, 0, 410.0], [0, 690.0, 290.0], [0, 0, 1]], [1, 3])]


def _object(sub, seed, scale, vc, open_):
    from foundationpose_b200 import synth

    m = synth.make_mesh(sub, tex_seed=seed, tex_size=256, scale=scale)
    tex = m.visual.image
    if open_:
        z = m.vertices[:, 2]
        m.faces = m.faces[~(z[m.faces] > 0.6 * z.max()).all(1)]  # one cap cut off: a mesh with a hole
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
    e.set_config("refine", crop_ratio=1.2)
    e.set_config("score", crop_ratio=1.2)  # the scorer's window coincides with the refiner's: vis_crops(mode=1) sees it
    for k, (m, _, _) in enumerate(objs):
        _load(e, m, k + 1)
    return e


def _camera(objs, H, W, K, seen, seed):
    """A frame of camera (H, W, K) showing objects `seen`; start poses = true poses plus a little noise."""
    from foundationpose_b200 import synth

    K = np.asarray(K, dtype=np.float64)
    rng = np.random.default_rng(seed)
    gt, start = [], []
    for j, k in enumerate(seen):
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(30 + 7 * seed + k)
        z = 0.6 + 0.05 * j
        p[:3, 3] = [((W * (j + 1) / (len(seen) + 1)) - K[0, 2]) * z / K[0, 0], 0.03 * (-1) ** j, z]
        gt.append(p)
        q = p.copy()
        q[:3, 3] += rng.normal(0, 0.004, 3)
        start.append(q.astype(np.float32))
    rgb, depth, _ = synth.make_multi_scene([(objs[k][1], p, objs[k][2]) for k, p in zip(seen, gt)], K, H, W, seed=seed)
    return dict(rgb=rgb, depth=depth, K=K, seen=list(seen), start=np.stack(start))


def _make_rig():
    objs = [_object(*s) for s in SPECS]
    cams = [_camera(objs, H, W, K, seen, seed=3 + c) for c, (H, W, K, seen) in enumerate(CAMERAS)]
    return objs, cams


@pytest.fixture(scope="module")
def rig():
    objs, cams = _make_rig()
    e = _engine(objs)
    yield dict(e=e, objs=objs, cams=cams)
    e.close()


def _pairs(cams, M=None, order=None):
    """(frames, start poses, camera ids, slots, pairs) of the first M (camera, object) pairs, camera-major, over the
    cameras that own one of them (renumbered), in `order`."""
    pairs = [(c, j) for c, cam in enumerate(cams) for j in range(len(cam["seen"]))][:M]
    used = sorted({c for c, _ in pairs})
    if order is not None:
        pairs = [pairs[i] for i in order]
    frames = [(cams[c]["rgb"], cams[c]["depth"], cams[c]["K"]) for c in used]
    start = torch.from_numpy(np.stack([cams[c]["start"][j] for c, j in pairs])).cuda()
    return frames, start, [used.index(c) for c, _ in pairs], [cams[c]["seen"][j] + 1 for c, j in pairs], pairs


def _on_device(frames):
    return [(torch.from_numpy(rgb).cuda(), torch.from_numpy(depth).cuda(), K) for rgb, depth, K in frames]


def _fit(e, frames, start, cam_of, slots, it, delta=DELTA, wait=True):
    if wait:
        return e.track_cameras(frames, start, cam_of, slots, it, fit_delta=delta)
    dev, pending = e.track_cameras(frames, start, cam_of, slots, it, wait=False, fit_delta=delta)
    host, fit = pending.result()
    return dev, host, fit


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("it", [1, 2])
@pytest.mark.parametrize("wait", [True, False])
@pytest.mark.parametrize("where", ["host", "device"])
def test_poses_unchanged_by_the_fit(rig, it, wait, where):
    e, cams = rig["e"], rig["cams"]
    for M in range(1, 9):
        frames, start, cam_of, slots, _ = _pairs(cams, M)
        if where == "device":
            frames = _on_device(frames)
        if wait:
            dev0, host0 = e.track_cameras(frames, start, cam_of, slots, it)
        else:
            dev0, pending = e.track_cameras(frames, start, cam_of, slots, it, wait=False)
            host0 = pending.result()
        dev1, host1, fit = _fit(e, frames, start, cam_of, slots, it, wait=wait)
        what = f"M={M} C={len(frames)} it={it} wait={wait} {where}"
        assert torch.equal(dev0, dev1) and np.array_equal(host0, host1), what
        assert np.array_equal(dev1.cpu().numpy(), host1), what
        assert fit.shape == (M, 5) and fit.dtype == np.int32
        assert (fit[:, 2] + fit[:, 3] + fit[:, 4] == fit[:, 1]).all() and (fit[:, 1] <= fit[:, 0]).all(), (what, fit)
        assert (fit[:, 0] > 0).all(), (what, fit)


def test_track_one_with_and_without_fit(rig):
    from foundationpose_b200.estimater import FoundationPose, PoseRefinePredictor, ScorePredictor
    from foundationpose_b200.weights import random_state_dict

    e = _engine()
    refiner = PoseRefinePredictor(engine=e, state_dict=random_state_dict("refine", 0))
    scorer = ScorePredictor(engine=e, state_dict=random_state_dict("score", 0))
    m = rig["objs"][0][0].copy()
    m.vertices = m.vertices + np.array([0.01, -0.02, 0.005])  # off-centre: the un-centring shift is exercised
    est = FoundationPose(model_pts=m.vertices, model_normals=m.vertex_normals, mesh=m, scorer=scorer, refiner=refiner)
    cam = rig["cams"][0]
    start = torch.from_numpy(cam["start"][0]).cuda().reshape(1, 4, 4)
    frames = {"host": (cam["rgb"], cam["depth"]),
              "device": (torch.from_numpy(cam["rgb"]).cuda(), torch.from_numpy(cam["depth"]).cuda())}
    out = {}
    for where, (rgb, depth) in frames.items():
        for fit in (None, DELTA):
            est.pose_last = start.clone()
            est.fit_last = None
            out[(where, fit)] = (est.track_one(rgb, depth, cam["K"], 2, fit_delta=fit), est.pose_last.clone(), est.fit_last)
    # fp_track on the same centred mesh in slot 0 (FoundationPose loaded it there)
    _, want = e.track(cam["rgb"], cam["depth"], cam["K"], start.reshape(4, 4), 2)
    for key, (pose, last, fit) in out.items():
        assert torch.equal(last.reshape(4, 4).cpu(), torch.from_numpy(want)), key
        assert np.array_equal(pose, out[("host", None)][0]), key
        assert (fit is None) == (key[1] is None), key
    f = out[("host", DELTA)][2]
    assert f == out[("device", DELTA)][2]
    assert f.valid > 1000 and f.inlier + f.occluded + f.behind == f.valid
    e.close()


# ---------------------------------------------------------------------------------------------------------------------
def _vis_counts(e, poses, delta):
    """The counts from the by-value single-camera vis record of the scorer's window (equal to the refiner's here):
    the rendered camera z and the nearest filtered depth in metres at every crop pixel."""
    rec = e.vis_crops(poses, mode=1)
    za, zb = rec[:, 0, ..., 3], rec[:, 1, ..., 3]
    covered = za > 0
    valid = covered & (zb >= 0.001)
    d = zb - za
    c = [covered, valid, valid & (d.abs() <= delta), valid & (d < -delta), valid & (d > delta)]
    return torch.stack([x.flatten(1).sum(1) for x in c], 1).cpu().numpy()


def _cases():
    """name -> (mesh, frame rgb, depth, K, start pose (4,4), iterations)"""
    from foundationpose_b200 import synth

    g = dict(np.load(GOLD))
    gold_mesh = synth.make_mesh(3)
    rgb, depth, _ = synth.make_scene(gold_mesh.visual.image, g["gt"][1], seed=2)
    out = {"golden scene": (gold_mesh, rgb, depth, synth.DEFAULT_K, g["pose_in"][0], 2)}
    for name, spec in (("open mesh", SPECS[2]), ("vertex-coloured mesh", SPECS[1])):
        m, tex, scale = _object(*spec)
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(17)
        p[:3, 3] = [0.01, -0.02, 0.55]
        rgb, depth, _ = synth.make_multi_scene([(tex, p, scale)], synth.DEFAULT_K, seed=8)
        q = p.copy()
        q[:3, 3] += [0.003, -0.002, 0.004]
        out[name] = (m, rgb, depth, synth.DEFAULT_K, q, 0)
    near = synth.make_mesh(2)
    p = np.eye(4)
    p[:3, 3] = [0.0, 0.0, 0.3]
    rgb, depth, _ = synth.make_scene(near.visual.image, p, seed=9)
    q = np.eye(4)
    q[:3, 3] = [0.0, 0.0, 0.0955]  # the surface 0.5 mm in front of the camera: it crosses the near plane
    out["near plane"] = (near, rgb, depth, synth.DEFAULT_K, q, 0)
    return out


def _one(e, mesh, rgb, depth, K, pose, it, delta=DELTA):
    _load(e, mesh, 0)
    start = torch.from_numpy(np.asarray(pose, dtype=np.float32)).cuda().reshape(1, 4, 4)
    return e.track_cameras([(rgb, depth, K)], start, [0], [0], it, fit_delta=delta)


@pytest.mark.parametrize("name", ["golden scene", "open mesh", "vertex-coloured mesh", "near plane"])
def test_counts_equal_the_vis_record(name):
    mesh, rgb, depth, K, pose, it = _cases()[name]
    e = _engine()
    for delta in (DELTA, 0.002):
        dev, _, fit = _one(e, mesh, rgb, depth, K, pose, it, delta)
        want = _vis_counts(e, dev, delta)
        assert np.array_equal(fit, want), (name, delta, fit, want)
    assert fit[0, 1] > 100, fit
    e.close()


@pytest.mark.parametrize("name", ["golden scene", "open mesh", "vertex-coloured mesh", "near plane"])
def test_counts_against_the_host_reference(name):
    from oracle import pipeline

    mesh, rgb, depth, K, pose, it = _cases()[name]
    e = _engine()
    dev, _, fit = _one(e, mesh, rgb, depth, K, pose, it)
    mt = pipeline.mesh_tensors(mesh)
    d = float(e.diameter)
    p = np.asarray(mt["pos"], dtype=np.float64)
    c = (p.min(0) + p.max(0)) / 2
    sphere = np.float32(c).tolist() + [float(np.float32(np.sqrt(((p - c) ** 2).sum(1)).max() * 1.0001 + 1e-9))]
    fdepth, xyz = e.get_depth()
    sc = cr.Scene(mt, K, rgb, fdepth, xyz, d, front_sign=e.mesh_info()["front_sign"], sphere=sphere, device="cuda")
    covered, zr, zo = fr.depths(sc, dev.cpu().numpy())
    want = fr.counts_of(covered, zr, zo, DELTA)
    near = int(fr.near_delta(covered, zr, zo, DELTA)[0])
    diff = np.abs(fit.astype(np.int64) - want)
    print(f"{name}: counts {fit[0].tolist()}, reference {want[0].tolist()}, pixels within 1e-6 m of delta: {near}")
    assert diff[0, 0] == 0 and diff[0, 1] == 0, (name, fit, want)
    assert diff[0, 2:].sum() <= 2 * near, (name, fit, want, near)
    e.close()


# ---------------------------------------------------------------------------------------------------------------------
def _per_pair(fit, pairs):
    return {p: tuple(fit[i]) for i, p in enumerate(pairs)}


def test_counts_do_not_depend_on_the_batch(rig):
    e, cams = rig["e"], rig["cams"]
    frames, start, cam_of, slots, pairs = _pairs(cams)
    _, _, fit = _fit(e, frames, start, cam_of, slots, 2)
    base = _per_pair(fit, pairs)
    # object order, camera order, fewer objects
    perm = [5, 0, 7, 2, 4, 1, 6, 3]
    f2 = _pairs(cams, order=perm)
    assert _per_pair(_fit(e, *f2[:4], 2)[2], f2[4]) == base
    cam_perm = [2, 0, 3, 1]
    _, _, fit3 = _fit(e, [frames[i] for i in cam_perm], start, [cam_perm.index(c) for c in cam_of], slots, 2)
    assert _per_pair(fit3, pairs) == base
    for M in (1, 3, 5):
        f4 = _pairs(cams, M)
        got = _per_pair(_fit(e, *f4[:4], 2)[2], f4[4])
        assert got == {p: base[p] for p in f4[4]}, M
    # each object alone, its camera as camera 0
    for (c, j), want in base.items():
        cam = cams[c]
        _, _, alone = _fit(e, [(cam["rgb"], cam["depth"], cam["K"])], torch.from_numpy(cam["start"][j:j + 1]).cuda(), [0],
                           [cam["seen"][j] + 1], 2)
        assert tuple(alone[0]) == want, (c, j)
    # the crop tile, non-blocking calls, device frames
    for tile in (16, 32, 80):
        e.set_crop_tile(tile)
        try:
            assert _per_pair(_fit(e, frames, start, cam_of, slots, 2)[2], pairs) == base, tile
        finally:
            e.set_crop_tile(0)
    assert _per_pair(_fit(e, frames, start, cam_of, slots, 2, wait=False)[2], pairs) == base
    assert _per_pair(_fit(e, _on_device(frames), start, cam_of, slots, 2)[2], pairs) == base


def eager_counts():
    """The rig's counts in a fresh process (run with FPOSE_NO_GRAPH=1): JSON list of lists."""
    objs, cams = _make_rig()
    e = _engine(objs)
    frames, start, cam_of, slots, _ = _pairs(cams)
    out = [_fit(e, frames, start, cam_of, slots, 2)[2].tolist() for _ in range(3)]
    e.close()
    return out


def test_eager_launches_give_the_same_counts(rig):
    e, cams = rig["e"], rig["cams"]
    frames, start, cam_of, slots, _ = _pairs(cams)
    want = _fit(e, frames, start, cam_of, slots, 2)[2].tolist()
    env = dict(os.environ, FPOSE_NO_GRAPH="1")
    code = f"import json, sys; sys.path.insert(0, {ROOT!r}); import test_track_fit_gpu as t; print('COUNTS', json.dumps(t.eager_counts()))"
    r = subprocess.run([sys.executable, "-c", code], cwd=os.path.join(ROOT, "tests"), env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("COUNTS ")][-1][len("COUNTS "):])
    assert all(g == want for g in got), (got, want)


def test_graphs_are_reused(rig):
    e, cams = rig["e"], rig["cams"]
    frames, start, cam_of, slots, _ = _pairs(cams)
    for _ in range(3):
        e.track_cameras(frames, start, cam_of, slots, 2)
        _fit(e, frames, start, cam_of, slots, 2)
    captures = e.graph_captures()
    fits = {}
    for delta in (DELTA, 0.002, 0.05, 0.0, DELTA):
        e.track_cameras(frames, start, cam_of, slots, 2)
        fits[delta] = _fit(e, frames, start, cam_of, slots, 2, delta)[2]
    assert e.graph_captures() == captures, "a fit call, a plain call or a new delta captured a graph"
    assert (fits[0.002][:, 2] <= fits[DELTA][:, 2]).all() and (fits[DELTA][:, 2] <= fits[0.05][:, 2]).all()
    assert not np.array_equal(fits[0.002], fits[0.05])


def test_refusals(rig):
    from foundationpose_b200 import _lib
    from foundationpose_b200.engine import _camera_args, _p, _stream
    from foundationpose_b200._lib import lib

    e, cams = rig["e"], rig["cams"]
    frames, start, cam_of, slots, _ = _pairs(cams, 3)
    rgbs, depths, Ks, Hs, Ws = _camera_args(frames)
    M = len(slots)
    out = torch.empty(M, 4, 4, device="cuda")

    def submit(delta, fn=lib.fp_track_cameras_fit_submit):
        t = C.c_ulonglong()
        extra = (float(delta), _p(out), None) if fn is lib.fp_track_cameras_fit_submit else (_p(out),)
        rc = fn(e._h, len(frames), rgbs, depths, Ks, Hs, Ws, M, (C.c_int * M)(*cam_of), (C.c_int * M)(*slots), _p(start), 2,
                *extra, _stream(), C.byref(t))
        return rc, t.value

    rc, t = submit(DELTA)
    assert rc == 0 and lib.fp_track_fit_wait(e._h, t, None, None) == 0
    n0 = _lib.launch_count()
    for bad in (-1e-3, float("nan"), float("inf"), -float("inf")):
        assert submit(bad)[0] != 0, bad
    assert _lib.launch_count() == n0, "a refused call enqueued work"
    # a plain ticket: refused by fp_track_fit_wait, left for fp_track_wait
    rc, t = submit(None, lib.fp_track_cameras_submit)
    assert rc == 0
    counts = np.full((M, 5), -7, dtype=np.int32)
    assert lib.fp_track_fit_wait(e._h, t, None, C.c_void_p(counts.ctypes.data)) != 0
    assert (counts == -7).all()
    host = np.empty((M, 4, 4), dtype=np.float32)
    assert lib.fp_track_wait(e._h, t, C.c_void_p(host.ctypes.data)) == 0
    assert lib.fp_track_wait(e._h, t, None) != 0, "collected twice"
    # unknown tickets
    assert lib.fp_track_fit_wait(e._h, t + 1000, None, None) != 0
    assert lib.fp_track_fit_wait(e._h, 0, None, None) != 0
    # fp_track_wait accepts a fit ticket and drops its counts; the context stays usable
    rc, t = submit(DELTA)
    assert rc == 0 and lib.fp_track_wait(e._h, t, C.c_void_p(host.ctypes.data)) == 0
    _, again, fit = _fit(e, frames, start, cam_of, slots, 2)
    assert np.array_equal(again, host) and (fit[:, 0] > 0).all()


def test_estimator_surfaces_set_fit_last(rig):
    from foundationpose_b200.estimater import FoundationPose, PoseFit, PoseRefinePredictor, ScorePredictor, track_cameras, track_objects
    from foundationpose_b200.weights import random_state_dict

    e = _engine()
    refiner = PoseRefinePredictor(engine=e, state_dict=random_state_dict("refine", 0))
    scorer = ScorePredictor(engine=e, state_dict=random_state_dict("score", 0))
    cams = rig["cams"]
    ests = {}
    for k in range(4):
        m = rig["objs"][k][0]
        ests[k] = FoundationPose(model_pts=m.vertices, model_normals=m.vertex_normals, mesh=m, scorer=scorer, refiner=refiner)
    views = [([ests[k] for k in cams[0]["seen"]], cams[0]["rgb"], cams[0]["depth"], cams[0]["K"]),
             ([ests[3]], cams[1]["rgb"], cams[1]["depth"], cams[1]["K"])]

    def reset():
        for j, k in enumerate(cams[0]["seen"]):
            ests[k].pose_last = torch.from_numpy(cams[0]["start"][j]).cuda().reshape(1, 4, 4)
            ests[k].fit_last = None
        ests[3].pose_last = torch.from_numpy(cams[1]["start"][0]).cuda().reshape(1, 4, 4)
        ests[3].fit_last = None

    reset()
    plain = track_cameras(views, iteration=2)
    reset()
    got = track_cameras(views, iteration=2, fit_delta=DELTA)
    assert all(np.array_equal(a, b) for v, w in zip(plain, got) for a, b in zip(v, w))
    fits = {k: est.fit_last for k, est in ests.items()}
    assert all(isinstance(f, PoseFit) and f.valid > 0 for f in fits.values())
    reset()
    pending = track_cameras(views, iteration=2, wait=False, fit_delta=DELTA)
    assert all(est.fit_last is None for est in ests.values()), "fit_last is set when result() collects the call"
    assert all(np.array_equal(a, b) for v, w in zip(plain, pending.result()) for a, b in zip(v, w))
    assert {k: est.fit_last for k, est in ests.items()} == fits
    # track_objects: one camera, same poses and counts as the object's row of the camera call
    objs0 = [ests[k] for k in cams[0]["seen"]]
    reset()
    want = track_objects(objs0, cams[0]["rgb"], cams[0]["depth"], cams[0]["K"], iteration=2)
    reset()
    got = track_objects(objs0, cams[0]["rgb"], cams[0]["depth"], cams[0]["K"], iteration=2, fit_delta=DELTA)
    assert all(np.array_equal(a, b) for a, b in zip(want, got))
    assert [est.fit_last for est in objs0] == [fits[k] for k in cams[0]["seen"]]
    reset()
    pending = track_objects(objs0, cams[0]["rgb"], cams[0]["depth"], cams[0]["K"], iteration=2, wait=False, fit_delta=DELTA)
    assert all(np.array_equal(a, b) for a, b in zip(want, pending.result()))
    assert [est.fit_last for est in objs0] == [fits[k] for k in cams[0]["seen"]]
    e.close()


def test_recovery_example_fires_at_the_jump():
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    try:
        import track_with_recovery as ex
    finally:
        sys.path.pop(0)
    log = ex.run()  # the example's own defaults: 8 frames, the jump at frame 5
    fired = [r["frame"] for r in log if r["recovered"]]
    assert fired and fired[0] == 5, log
    assert all(r["fit"].inlier_ratio >= ex.THRESHOLD for r in log if r["frame"] < 5), log
