"""Frames as sensors deliver them, on the GPU: every call on Color / Depth frames (BGR / BGRA / RGBA colour, uint16 depth
with a scale, pitched rows and region-of-interest views, host pageable, host page-locked and device buffers) against the
same call on the frame converted on the host to packed RGB8 and float32 metres, bit for bit.  Also: formats alternating
call by call with calls in flight, graph reuse when only formats change, and refusals that enqueue nothing."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# per camera: H, W, K.  333 x 257 is not a multiple of the frame filter's 32 x 8 tile.
CAMERAS = [(480, 640, [[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1]]),
           (257, 333, [[330.0, 0, 165.5], [0, 328.0, 130.0], [0, 0, 1]]),
           (720, 1280, [[920.0, 0, 640.0], [0, 915.0, 360.0], [0, 0, 1]])]
SCALES = (0.001, 0.0001, 0.00025)


def _load(e, mesh, slot):
    from foundationpose_b200 import synth
    from foundationpose_b200.estimater import make_mesh_tensors

    mt = make_mesh_tensors(mesh)
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(mesh.vertices), uv=mt.get("uv"), tex=mt.get("tex"),
               vertex_colors=mt.get("vcolor"), slot=slot)


@pytest.fixture(scope="module")
def rig():
    """One engine, one object per camera (slot c + 1, and object 0 in slot 0), each camera's frame as packed RGB8 and
    float32 metres in whole millimetres (so uint16 at every scale of SCALES holds it), and each object's start pose."""
    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.weights import random_state_dict

    objs = [synth.make_mesh(3, tex_seed=s, tex_size=256, scale=sc) for s, sc in ((0, 1.0), (5, 0.8), (9, 1.2))]
    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    e.set_config("refine")
    e.set_config("score")
    for k, m in enumerate(objs):
        _load(e, m, k + 1)
    _load(e, objs[0], 0)
    cams, start = [], []
    for c, (H, W, K) in enumerate(CAMERAS):
        K = np.asarray(K, dtype=np.float64)
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(31 + c)
        p[:3, 3] = [0.01, -0.01, 0.6]
        rgb, depth, owner = synth.make_multi_scene([(objs[c].visual.image, p, (1.0, 0.8, 1.2)[c])], K, H, W, seed=7 + c)
        # whole millimetres: no uint16 value of SCALES overflows or clips
        depth = (np.round(depth.astype(np.float64) * 1000.0) / 1000.0).astype(np.float32)
        depth[::17, ::13] = 0.0  # invalid pixels stay invalid
        q = p.copy()
        q[:3, 3] += [0.002, -0.003, 0.004]
        cams.append(dict(rgb=rgb, depth=depth, K=K, mask=owner == 0))
        start.append(q.astype(np.float32))
    return dict(e=e, objs=objs, cams=cams, start=torch.from_numpy(np.stack(start)).cuda())


def _place(a, where):
    """`a` (numpy) as the caller holds it: packed numpy, a region-of-interest view of a larger numpy frame, a view of a
    larger page-locked CPU tensor, or a CUDA tensor (packed or a view of a larger one)."""
    if where == "packed":
        return np.ascontiguousarray(a)
    big = np.zeros((a.shape[0] + 3, a.shape[1] + 11) + a.shape[2:], a.dtype)
    big[2:2 + a.shape[0], 5:5 + a.shape[1]] = a
    roi = (slice(2, 2 + a.shape[0]), slice(5, 5 + a.shape[1]))
    if where == "roi":
        return big[roi]
    if where == "pinned":
        return torch.from_numpy(big).pin_memory()[roi]
    if where == "device":
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()
    assert where == "device_roi"
    return torch.from_numpy(big).cuda()[roi]


def sensor(cam, order, scale, where, alpha_seed=0):
    """Camera frame `cam` as a sensor delivers it: (Color, Depth), and the host conversion the results must equal:
    (packed RGB8, float32 metres), converted by the documented expressions."""
    from foundationpose_b200.frames import Color, Depth

    rgb, depth = cam["rgb"], cam["depth"]
    img = rgb[..., ::-1] if order.startswith("b") else rgb
    if order.endswith("a"):
        alpha = np.random.default_rng(alpha_seed).integers(0, 256, rgb.shape[:2] + (1,), dtype=np.uint8)
        img = np.concatenate([img, alpha], -1)
    if scale is None:
        raw, ref_depth = depth, depth
    else:
        raw = np.round(depth.astype(np.float64) / np.float32(scale)).astype(np.uint16)
        ref_depth = raw.astype(np.float32) * np.float32(scale)
    conv = np.ascontiguousarray((img[..., 2::-1] if order.startswith("b") else img[..., :3]))
    np.testing.assert_array_equal(conv, rgb)
    return (Color(_place(img, where), order), Depth(_place(raw, where), scale)), (rgb, ref_depth)


def _eq(a, b):
    a = a.cpu() if torch.is_tensor(a) else torch.from_numpy(np.asarray(a))
    b = b.cpu() if torch.is_tensor(b) else torch.from_numpy(np.asarray(b))
    return a.shape == b.shape and torch.equal(a, b)


# colour order, uint16 scale (None: float32), placement: every order, every scale, every placement
SET_FRAME_CASES = [("rgb", None, "roi"), ("bgr", 0.001, "packed"), ("rgba", 0.0001, "pinned"), ("bgra", 0.00025, "device_roi"),
                   ("bgr", None, "device"), ("rgba", 0.001, "roi"), ("bgra", 0.0001, "packed"), ("rgb", 0.00025, "device")]


@pytest.mark.parametrize("filter_depth", [True, False])
def test_set_frame_depth_xyz_and_crops(rig, filter_depth):
    e, cam = rig["e"], rig["cams"][1]
    pose = rig["start"][1:2]
    e.set_frame(cam["rgb"], cam["depth"], cam["K"], filter_depth=filter_depth)
    ref = [t.clone() for t in e.get_depth()] + [e.vis_crops(pose, 0), e.vis_crops(pose, 1)]
    for order, scale, where in SET_FRAME_CASES:
        (rgb, depth), conv = sensor(cam, order, scale, where)
        e.set_frame(conv[0], conv[1], cam["K"], filter_depth=filter_depth)
        want = [t.clone() for t in e.get_depth()] + [e.vis_crops(pose, 0), e.vis_crops(pose, 1)]
        e.set_frame(rgb, depth, cam["K"], filter_depth=filter_depth)
        got = list(e.get_depth()) + [e.vis_crops(pose, 0), e.vis_crops(pose, 1)]
        for k, (g, w) in enumerate(zip(got, want)):
            assert torch.equal(g, w), (order, scale, where, k)
        if scale is None:
            for g, r in zip(got, ref):  # the converted frame is the original one
                assert torch.equal(g, r), (order, scale, where)


# per camera of track_cameras: (order, scale, placement); mixed formats across cameras
MIXES = [[("bgr", 0.001, "roi"), ("bgra", 0.00025, "device_roi"), ("rgba", None, "pinned")],
         [("rgba", 0.0001, "device"), ("rgb", None, "packed"), ("bgr", 0.001, "roi")],
         [("bgra", 0.00025, "pinned"), ("bgr", 0.0001, "roi"), ("rgb", 0.001, "device")]]


def _mix(rig, mix):
    got, conv = [], []
    for cam, (order, scale, where) in zip(rig["cams"], mix):
        (rgb, depth), (r, d) = sensor(cam, order, scale, where)
        got.append((rgb, depth, cam["K"]))
        conv.append((r, d, cam["K"]))
    return got, conv


def test_track_cameras_objects_and_track(rig):
    e, start = rig["e"], rig["start"]
    cam_of, slots = [0, 1, 2], [1, 2, 3]
    for mix in MIXES:
        got, conv = _mix(rig, mix)
        _, want = e.track_cameras(conv, start, cam_of, slots, 2)
        _, host = e.track_cameras(got, start, cam_of, slots, 2)
        assert _eq(host, want), mix
        _, want_p, want_fit = e.track_cameras(conv, start, cam_of, slots, 2, fit_delta=0.01)
        _, host_p, fit = e.track_cameras(got, start, cam_of, slots, 2, fit_delta=0.01)
        assert _eq(host_p, want_p) and _eq(fit, want_fit), mix
        for c in range(3):
            _, want = e.track_objects(conv[c][0], conv[c][1], conv[c][2], start[c:c + 1], [slots[c]], 2)
            _, host = e.track_objects(got[c][0], got[c][1], got[c][2], start[c:c + 1], [slots[c]], 2)
            assert _eq(host, want), (mix, c)
        _, want = e.track(conv[0][0], conv[0][1], conv[0][2], start[0], 2)
        _, host = e.track(got[0][0], got[0][1], got[0][2], start[0], 2)
        assert _eq(host, want), mix


def test_graph_reuse_when_only_formats_change(rig):
    """After each format has been seen once (the raw buffers reach their widest), a new scale, order, pitch or buffer
    address replays the cached graphs, and so do default-format calls afterwards."""
    e, start = rig["e"], rig["start"]
    cam_of, slots = [0, 1, 2], [1, 2, 3]
    plain = [(c["rgb"], c["depth"], c["K"]) for c in rig["cams"]]
    for mix in MIXES + MIXES:
        e.track_cameras(_mix(rig, mix)[0], start, cam_of, slots, 2)
    e.track_cameras(plain, start, cam_of, slots, 2)
    n = e.graph_captures()
    other = [[("rgb", 0.00025, "roi"), ("rgba", 0.001, "device"), ("bgra", 0.0001, "device_roi")],
             [("bgr", None, "pinned"), ("bgr", 0.0001, "device_roi"), ("rgb", 0.00025, "roi")]]
    for mix in other + MIXES:
        e.track_cameras(_mix(rig, mix)[0], start, cam_of, slots, 2)
    e.track_cameras(plain, start, cam_of, slots, 2)
    assert e.graph_captures() == n


def test_wait_false_with_formats_alternating(rig):
    """Host frames, formats alternating call by call on every camera while the previous call is in flight: the staging
    sets are reused at other byte sizes.  Every result equals the blocking call's on the converted frames."""
    e, start = rig["e"], rig["start"]
    cam_of, slots = [0, 1, 2], [1, 2, 3]
    host_mixes = [[("bgr", 0.001, "roi"), ("bgra", 0.00025, "packed"), ("rgba", None, "pinned")],
                  [("rgb", None, "packed"), ("rgb", None, "packed"), ("rgb", None, "packed")],
                  [("bgra", 0.0001, "pinned"), ("bgr", 0.0001, "roi"), ("rgba", 0.001, "packed")]]
    want = [e.track_cameras(_mix(rig, m)[1], start, cam_of, slots, 2)[1] for m in host_mixes]
    pending = []
    for k in range(9):
        got, _ = _mix(rig, host_mixes[k % 3])
        pending.append(e.track_cameras(got, start, cam_of, slots, 2, wait=False)[1])
        del got  # the host frames may go as soon as the call is submitted
    for k, p in enumerate(pending):
        assert _eq(p.result(), want[k % 3]), k


def _grids(n, seed):
    from foundationpose_b200 import synth

    g = np.tile(np.eye(4, dtype=np.float32), (n, 1, 1))
    for i in range(n):
        g[i, :3, :3] = synth.random_rotation(seed + i)
    return torch.from_numpy(g).cuda()


def test_register_objects_and_cameras(rig):
    e = rig["e"]
    for order, scale, where in [("bgr", 0.001, "roi"), ("bgra", 0.0001, "device_roi"), ("rgba", 0.00025, "pinned")]:
        cam = rig["cams"][0]
        (rgb, depth), (r, d) = sensor(cam, order, scale, where)
        masks = cam["mask"][None]
        want = e.register_objects(r, d, cam["K"], masks, [_grids(12, 3)], [1], 2)
        got = e.register_objects(rgb, depth, cam["K"], masks, [_grids(12, 3)], [1], 2)
        assert all(_eq(g, w) for g, w in zip(got, want)), (order, scale, where)
    for mix in MIXES:
        got, conv = _mix(rig, mix)
        masks = [c["mask"] for c in rig["cams"]]
        grids = [_grids(10, 5 + c) for c in range(3)]
        want = e.register_cameras(conv, masks, grids, [0, 1, 2], [1, 2, 3], 2)
        res = e.register_cameras(got, masks, grids, [0, 1, 2], [1, 2, 3], 2)
        assert all(_eq(g, w) for g, w in zip(res, want)), mix


def test_refusals_enqueue_nothing(rig):
    from foundationpose_b200 import _lib
    from foundationpose_b200.engine import _FpFrameFormat, lib
    from foundationpose_b200.frames import Color, Depth

    e, start = rig["e"], rig["start"]
    cam = rig["cams"][0]
    H, W = cam["depth"].shape
    for _ in range(2):  # seen, then captured
        _, want = e.track(cam["rgb"], cam["depth"], cam["K"], start[0], 2)
    n = e.graph_captures()

    def refused(fmt, camera, match):
        f = None if fmt is None else C.byref(_FpFrameFormat(*fmt))
        with pytest.raises(_lib.FposeError, match=match):
            _lib.check(lib.fp_set_camera_format(e._h, camera, f), "fp_set_camera_format")

    refused((0, 0, 0.0, 0, 0), 16, "camera 16 out of range")
    refused((0, 0, 0.0, 0, 0), -1, "camera -1 out of range")
    refused((4, 0, 0.0, 0, 0), 1, "camera 1: unknown colour format 4")
    refused((0, 2, 0.0, 0, 0), 2, "camera 2: unknown depth format 2")
    for bad in (0.0, -0.001, float("nan"), float("inf")):
        refused((0, 1, bad, 0, 0), 3, "camera 3: uint16 depth scale")
    # at call time, before anything is enqueued: pitches below a row, a misaligned depth pitch or pointer
    Kf = (C.c_float * 9)(*cam["K"].reshape(-1))
    rgb = np.ascontiguousarray(cam["rgb"])
    dep = np.ascontiguousarray(cam["depth"])
    for fmt, match in (((0, 0, 0.0, 3 * W - 1, 0), "camera 0: rgb pitch"), ((0, 0, 0.0, 0, 4 * W - 4), "camera 0: depth pitch"),
                       ((0, 1, 0.001, 0, 2 * W + 1), "camera 0: depth pitch .* not a multiple")):
        e._set_formats([fmt])
        with pytest.raises(_lib.FposeError, match=match):
            _lib.check(lib.fp_set_frame(e._h, C.c_void_p(rgb.ctypes.data), C.c_void_p(dep.ctypes.data), Kf, H, W, 2,
                                        float("inf"), None), "fp_set_frame")
        ticket = C.c_ulonglong()
        with pytest.raises(_lib.FposeError, match=match):
            _lib.check(lib.fp_track_submit(e._h, C.c_void_p(rgb.ctypes.data), C.c_void_p(dep.ctypes.data), Kf, H, W,
                                           C.c_void_p(start[0].data_ptr()), 2, None, None, C.byref(ticket)), "fp_track")
    raw = np.round(cam["depth"].astype(np.float64) * 1000).astype(np.uint16)
    buf = np.zeros(H * W * 2 + 2, np.uint8)
    odd = np.frombuffer(buf.data, np.uint16, H * W, offset=1).reshape(H, W)
    odd[...] = raw
    with pytest.raises(_lib.FposeError, match="camera 0: depth buffer .* not aligned"):
        e.track(Color(rgb, "rgb"), Depth(odd, 0.001), cam["K"], start[0], 2)
    with pytest.raises(_lib.FposeError, match="camera 1: depth buffer .* not aligned"):
        e.track_cameras([(cam["rgb"], cam["depth"], cam["K"]), (Color(rgb, "rgb"), Depth(odd, 0.001), cam["K"])], start[:2],
                        [0, 1], [1, 1], 2)
    # the context is as it was: nothing ran, nothing was captured, the next call gives the same pose
    assert e.graph_captures() == n
    _, again = e.track(cam["rgb"], cam["depth"], cam["K"], start[0], 2)
    assert _eq(again, want)
    _, want = e.track(rgb, raw.astype(np.float32) * np.float32(0.001), cam["K"], start[0], 2)
    _, again = e.track(Color(rgb, "rgb"), Depth(raw, 0.001), cam["K"], start[0], 2)
    assert _eq(again, want)
    assert e.graph_captures() == n


def test_estimator_calls_with_wrappers(rig):
    from foundationpose_b200 import estimater
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.estimater import FoundationPose, PoseRefinePredictor, ScorePredictor
    from foundationpose_b200.weights import random_state_dict

    e = Engine()
    refiner = PoseRefinePredictor(engine=e, state_dict=random_state_dict("refine", 0))
    scorer = ScorePredictor(engine=e, state_dict=random_state_dict("score", 0))
    m = rig["objs"][0]
    mk = lambda: FoundationPose(model_pts=m.vertices, model_normals=m.vertex_normals, mesh=m, scorer=scorer, refiner=refiner)
    plain, wrapped = mk(), mk()
    cam = rig["cams"][0]
    (rgb, depth), (r, d) = sensor(cam, "bgra", 0.0001, "roi")
    assert np.array_equal(plain.register(cam["K"], r, d, cam["mask"], iteration=2),
                          wrapped.register(cam["K"], rgb, depth, cam["mask"], iteration=2))
    for order, scale, where in [("bgr", 0.001, "packed"), ("rgba", 0.00025, "device_roi"), ("bgra", None, "pinned")]:
        (rgb, depth), (r, d) = sensor(cam, order, scale, where)
        # the plain frame of the same kind: a host array takes fp_track, a tensor fp_set_frame + fp_refine
        if where.startswith("device"):
            r, d = torch.from_numpy(r).cuda(), torch.from_numpy(d).cuda()
        elif where == "pinned":
            r, d = torch.from_numpy(r), torch.from_numpy(d)
        assert np.array_equal(plain.track_one(r, d, cam["K"], 2), wrapped.track_one(rgb, depth, cam["K"], 2)), order
    (rgb, depth), (r, d) = sensor(cam, "bgr", 0.0001, "roi")
    assert np.array_equal(estimater.track_objects([plain], r, d, cam["K"]), estimater.track_objects([wrapped], rgb, depth, cam["K"]))
    assert np.array_equal(estimater.register_objects([plain], cam["K"], r, d, [cam["mask"]], iteration=2),
                          estimater.register_objects([wrapped], cam["K"], rgb, depth, [cam["mask"]], iteration=2))
    (dev_rgb, dev_depth), _ = sensor(cam, "bgr", 0.001, "device")
    with pytest.raises(TypeError, match="takes host frames"):
        estimater.track_objects([wrapped], dev_rgb, depth, cam["K"])
    with pytest.raises(TypeError, match="takes host frames"):
        estimater.register_objects([wrapped], cam["K"], rgb, dev_depth, [cam["mask"]])
    # two cameras with formats of their own: register_cameras, then track_cameras
    m1 = rig["objs"][1]
    mk1 = lambda: FoundationPose(model_pts=m1.vertices, model_normals=m1.vertex_normals, mesh=m1, scorer=scorer, refiner=refiner)
    ests = dict(plain=[plain, mk1()], wrapped=[wrapped, mk1()])
    cams = rig["cams"][:2]
    for k, mix in enumerate([[("bgr", 0.001, "roi"), ("rgba", 0.00025, "pinned")], [("bgra", 0.0001, "packed"), ("rgb", None, "roi")]]):
        frames = [sensor(c, *f) for c, f in zip(cams, mix)]
        views = {kind: [([ests[kind][i]], *frames[i][0 if kind == "wrapped" else 1], cams[i]["K"]) for i in range(2)]
                 for kind in ("plain", "wrapped")}
        if k == 0:
            got = {kind: estimater.register_cameras([(*v, [c["mask"]]) for v, c in zip(views[kind], cams)], iteration=2)
                   for kind in views}
        else:
            got = {kind: estimater.track_cameras(views[kind]) for kind in views}
        for a_, b_ in zip(got["plain"], got["wrapped"]):
            assert np.array_equal(np.stack(a_), np.stack(b_)), (k, mix)
    dev_views = [([ests["wrapped"][0]], dev_rgb, depth, cam["K"])]
    with pytest.raises(TypeError, match="takes host frames"):
        estimater.track_cameras(dev_views)
    with pytest.raises(TypeError, match="takes host frames"):
        estimater.register_cameras([(*dev_views[0], [cam["mask"]])])
    e.close()
