"""Depth from its own sensor, on the GPU: fp_align_depth bit for bit against the numpy float32 reference
(tests/align_reference.py), and every frame-taking call on sensor-native depth with a DepthSensor against the same call
on depth aligned on the host by that reference and passed as float32 metres, bit for bit in every output.  Also: graph
reuse when only the sensor changes, launch counts with and without a sensor, and refusals that enqueue nothing."""
import ctypes as C

import numpy as np
import pytest
import torch

import align_reference as ar

pytestmark = pytest.mark.gpu

SCALES = (0.001, 0.0001, 0.00025)


def _sensor_frame(rng_seed, Kd, Hd, Wd, T):
    """A synthetic depth image seen by the depth imager: a slanted background, boxes in front of it, holes; whole
    millimetres below 1.7 m, so uint16 holds it at every scale of SCALES."""
    rng = np.random.default_rng(rng_seed)
    yy, xx = np.mgrid[0:Hd, 0:Wd]
    d = 1.2 + 0.4 * xx / Wd + 0.2 * yy / Hd
    d[Hd // 4:Hd // 2, Wd // 5:Wd // 2] = 0.55
    d[Hd // 2:3 * Hd // 4, Wd // 2:3 * Wd // 4] = 0.33
    d += rng.normal(0, 0.002, d.shape)
    d = np.round(d * 1000) / 1000
    d[rng.random(d.shape) < 0.02] = 0
    return d.astype(np.float32)


def _scene_depth(obj, pose_c, T, Kd, Hd, Wd, seed):
    """The synthetic scene's depth as the depth imager sees it: the object at pose_c in the colour camera is at
    inv(T) @ pose_c in the depth camera.  Whole millimetres, with holes."""
    from foundationpose_b200 import synth

    pose_d = np.linalg.inv(T) @ pose_c
    _, depth, _ = synth.make_multi_scene([(obj.visual.image, pose_d, 1.0)], Kd, Hd, Wd, seed=seed)
    depth = (np.round(depth.astype(np.float64) * 1000.0) / 1000.0).astype(np.float32)
    depth[::19, ::11] = 0.0
    return depth


def _place(a, where):
    """`a` (numpy) as the caller holds it (see test_frame_formats_gpu._place)."""
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


def _raw(depth_m, scale):
    """Sensor-native depth of float32 metres `depth_m` (whole millimetres) at `scale` (None: float32), and its metres as
    the library reads them with the valid mask."""
    if scale is None:
        return depth_m, depth_m, depth_m != 0
    raw = np.round(depth_m.astype(np.float64) / np.float32(scale)).astype(np.uint16)
    m, valid = ar.depth_metres(raw, scale)
    return raw, m, valid


def _eq(a, b):
    a = a.cpu() if torch.is_tensor(a) else torch.from_numpy(np.asarray(a))
    b = b.cpu() if torch.is_tensor(b) else torch.from_numpy(np.asarray(b))
    return a.shape == b.shape and torch.equal(a, b)


RIGS = {"d435": (ar.D435_DEPTH_K, (480, 848), ar.D435_COLOR_K, (720, 1280)),
        "vga": (ar.VGA_DEPTH_K, (480, 640), ar.VGA_COLOR_K, (480, 640))}


@pytest.mark.parametrize("rig_name", sorted(RIGS))
@pytest.mark.parametrize("scale", SCALES + (None,))
@pytest.mark.parametrize("where", ["device", "device_roi"])
def test_align_op_is_bit_identical_to_the_reference(rig_name, scale, where):
    from foundationpose_b200 import ops
    from foundationpose_b200.frames import Depth, DepthSensor

    Kd, (Hd, Wd), Kc, (H, W) = RIGS[rig_name]
    T = ar.rig_T()
    raw, m, valid = _raw(_sensor_frame(3, Kd, Hd, Wd, T), scale)
    want = ar.align(m, valid, Kd, T, Kc, H, W)
    s = DepthSensor(Kd, T)
    got = ops.align_depth(Depth(_place(raw, where), scale, sensor=s), None, Kc, H, W)
    again = ops.align_depth(Depth(_place(raw, where), scale, sensor=s), None, Kc, H, W)
    torch.cuda.synchronize()
    assert _eq(got, want) and _eq(again, got)
    assert (want > 0).mean() > 0.5  # the rig covers most of the colour frame


def test_align_op_near_pixel_covers_a_large_area():
    from foundationpose_b200 import ops
    from foundationpose_b200.frames import DepthSensor

    Kd, (Hd, Wd), Kc, (H, W) = RIGS["d435"]
    T = ar.rig_T(angle_deg=0.0, t=(0.0, 0.0, -0.05))  # the colour camera 5 cm in front of the depth camera
    d = _sensor_frame(5, Kd, Hd, Wd, T)
    d[240, 423] = 0.0505  # half a millimetre in front of the colour camera: its corners land ~200 px apart
    d[100, 100] = 0.02  # behind the colour camera: dropped
    valid = d != 0
    want = ar.align(d, valid, Kd, T, Kc, H, W)
    x0, x1, y0, y1, _, _ = ar.rectangles(d, valid, Kd, T, Kc, H, W)
    assert ((x1 - x0 + 1) * (y1 - y0 + 1)).max() > 10000
    assert (want == np.float32(0.0505)).sum() > 10000
    got = ops.align_depth(torch.from_numpy(d).cuda(), DepthSensor(Kd, T), Kc, H, W)
    assert _eq(got, want)


def _load(e, mesh, slot):
    from foundationpose_b200 import synth
    from foundationpose_b200.estimater import make_mesh_tensors

    mt = make_mesh_tensors(mesh)
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(mesh.vertices), uv=mt.get("uv"), tex=mt.get("tex"),
               vertex_colors=mt.get("vcolor"), slot=slot)


# per camera: colour (H, W, K), and its depth imager ((Hd, Wd), Kd) or None.  333 x 257 is not a multiple of the frame
# filter's tile; camera 1 has no sensor.
CAMERAS = [((480, 640, ar.VGA_COLOR_K), ((480, 640), ar.VGA_DEPTH_K)),
           ((257, 333, np.array([[330.0, 0, 165.5], [0, 328.0, 130.0], [0, 0, 1]])), None),
           ((720, 1280, ar.D435_COLOR_K), ((480, 848), ar.D435_DEPTH_K))]


@pytest.fixture(scope="module")
def rig():
    """One engine, one object per camera (slot c + 1, object 0 also in slot 0).  Each camera's colour frame, its
    sensor-native depth (the depth imager's own image, or the colour frame's for camera 1), the host-aligned float32
    depth the sensor-native calls must equal, the object's mask and start pose."""
    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.frames import DepthSensor
    from foundationpose_b200.weights import random_state_dict

    objs = [synth.make_mesh(3, tex_seed=s, tex_size=256, scale=1.0) for s in (0, 5, 9)]
    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    e.set_config("refine")
    e.set_config("score")
    for k, m in enumerate(objs):
        _load(e, m, k + 1)
    _load(e, objs[0], 0)
    cams, start = [], []
    for c, ((H, W, K), sens) in enumerate(CAMERAS):
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(31 + c)
        p[:3, 3] = [0.01, -0.01, 0.6]
        rgb, depth, owner = synth.make_multi_scene([(objs[c].visual.image, p, 1.0)], K, H, W, seed=7 + c)
        cam = dict(rgb=rgb, K=K, mask=owner == 0, H=H, W=W)
        if sens is None:
            depth = (np.round(depth.astype(np.float64) * 1000.0) / 1000.0).astype(np.float32)
            cam.update(native=depth, aligned=depth, sensor=None)
        else:
            (Hd, Wd), Kd = sens
            T = ar.rig_T(t=(0.015 + 0.01 * c, 0.0002, -0.0004))
            native = _scene_depth(objs[c], p, T, Kd, Hd, Wd, 7 + c)
            cam.update(native=native, aligned=ar.align(native, native != 0, Kd, T, K, H, W), sensor=DepthSensor(Kd, T),
                       Kd=Kd, T=T)
            assert cam["mask"][cam["aligned"] > 0].any()  # the object is in the aligned depth
        q = p.copy()
        q[:3, 3] += [0.002, -0.003, 0.004]
        cams.append(cam)
        start.append(q.astype(np.float32))
    return dict(e=e, objs=objs, cams=cams, start=torch.from_numpy(np.stack(start)).cuda())


_ALIGNED = {}


def native(cam, scale, where):
    """Camera `cam`'s depth as its sensor delivers it: a Depth (with the sensor, if the camera has one) and the plain
    float32 metres aligned on the host that the call must equal."""
    from foundationpose_b200.frames import Depth

    raw, m, valid = _raw(cam["native"], scale)
    if cam["sensor"] is None:
        return Depth(_place(raw, where), scale), m
    key = (id(cam), scale)
    if key not in _ALIGNED:
        _ALIGNED[key] = ar.align(m, valid, cam["Kd"], cam["T"], cam["K"], cam["H"], cam["W"])
    return Depth(_place(raw, where), scale, sensor=cam["sensor"]), _ALIGNED[key]


def _rgb(cam, where):
    return _place(cam["rgb"], where)


@pytest.mark.parametrize("filter_depth", [True, False])
def test_set_frame(rig, filter_depth):
    e = rig["e"]
    for c in (0, 2):
        cam = rig["cams"][c]
        pose = rig["start"][c:c + 1]
        for scale, where in [(0.001, "packed"), (0.0001, "roi"), (None, "pinned"), (0.00025, "device_roi"), (None, "device")]:
            depth, plain = native(cam, scale, where)
            dev = where.startswith("device")
            rgb_p = torch.from_numpy(cam["rgb"]).cuda() if dev else cam["rgb"]
            e.set_frame(rgb_p, torch.from_numpy(plain).cuda() if dev else plain, cam["K"], filter_depth=filter_depth)
            want = [t.clone() for t in e.get_depth()] + [e.vis_crops(pose, 0), e.vis_crops(pose, 1)]
            e.set_frame(_rgb(cam, where), depth, cam["K"], filter_depth=filter_depth)
            got = list(e.get_depth()) + [e.vis_crops(pose, 0), e.vis_crops(pose, 1)]
            for k, (g, w) in enumerate(zip(got, want)):
                assert torch.equal(g, w), (c, scale, where, k)
            if not filter_depth:  # the unfiltered depth is the aligned depth itself
                assert _eq(got[0], plain), (c, scale, where)


# per camera of track_cameras: (uint16 scale or None, placement)
MIXES = [[(0.001, "roi"), (None, "device"), (0.00025, "pinned")],
         [(None, "device_roi"), (0.001, "packed"), (0.0001, "device")],
         [(0.0001, "pinned"), (None, "roi"), (None, "packed")]]


def _mix(rig, mix, cams=(0, 1, 2)):
    got, conv = [], []
    for c, (scale, where) in zip(cams, mix):
        cam = rig["cams"][c]
        depth, plain = native(cam, scale, where)
        got.append((_rgb(cam, where), depth, cam["K"]))
        conv.append((cam["rgb"], plain, cam["K"]))
    return got, conv


def test_track_cameras_objects_and_track(rig):
    e, start = rig["e"], rig["start"]
    cam_of, slots = [0, 1, 2], [1, 2, 3]
    for mix in MIXES:
        got, conv = _mix(rig, mix)
        _, want = e.track_cameras(conv, start, cam_of, slots, 2)
        want_depth = [e.get_depth(c)[0].clone() for c in range(3)]
        _, host = e.track_cameras(got, start, cam_of, slots, 2)
        assert _eq(host, want), mix
        for c in range(3):  # the filtered depth of every camera
            assert torch.equal(e.get_depth(c)[0], want_depth[c]), (mix, c)
        _, want_p, want_fit = e.track_cameras(conv, start, cam_of, slots, 2, fit_delta=0.01)
        _, host_p, fit = e.track_cameras(got, start, cam_of, slots, 2, fit_delta=0.01)
        assert _eq(host_p, want_p) and _eq(fit, want_fit), mix
        for c in range(3):
            _, want = e.track_objects(conv[c][0], conv[c][1], conv[c][2], start[c:c + 1], [slots[c]], 2)
            _, host = e.track_objects(got[c][0], got[c][1], got[c][2], start[c:c + 1], [slots[c]], 2)
            assert _eq(host, want), (mix, c)
        for c in (0, 2):  # track is camera 0: each sensor in turn
            _, want = e.track(conv[c][0], conv[c][1], conv[c][2], start[c], 2)
            _, host = e.track(got[c][0], got[c][1], got[c][2], start[c], 2)
            assert _eq(host, want), (mix, c)


def test_one_table_launch_equals_each_camera_alone(rig):
    """The aligned depth of every camera of one call (the filtered depth the table launch prepares) against the same
    camera in a call of its own, in another camera order."""
    e, start = rig["e"], rig["start"]
    got, _ = _mix(rig, MIXES[0])
    e.track_cameras(got, start, [0, 1, 2], [1, 2, 3], 1)
    together = [e.get_depth(c)[0].clone() for c in range(3)]
    for c in range(3):
        e.track_cameras([got[c]], start[c:c + 1], [0], [c + 1], 1)
        assert torch.equal(e.get_depth(0)[0], together[c]), c
    order = [2, 0, 1]
    e.track_cameras([got[c] for c in order], start[order], [0, 1, 2], [3, 1, 2], 1)
    for k, c in enumerate(order):
        assert torch.equal(e.get_depth(k)[0], together[c]), c


def test_wait_false_with_sensors_toggled(rig):
    """Host frames, camera 0's and 2's sensors on and off call by call while the previous call is in flight: every result
    equals the blocking call's on the host-aligned frames."""
    e, start = rig["e"], rig["start"]
    cam_of, slots = [0, 1, 2], [1, 2, 3]
    plain = [(c["rgb"], c["aligned"], c["K"]) for c in rig["cams"]]
    host_mixes = [[(0.001, "roi"), (None, "packed"), (0.00025, "pinned")], None, [(None, "pinned"), (0.0001, "roi"), (0.001, "packed")]]
    calls = [plain if m is None else _mix(rig, m)[0] for m in host_mixes]
    want = [e.track_cameras(plain if m is None else _mix(rig, m)[1], start, cam_of, slots, 2)[1] for m in host_mixes]
    pending = []
    for k in range(9):
        pending.append(e.track_cameras(calls[k % 3], start, cam_of, slots, 2, wait=False)[1])
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
    for c, scale, where in [(0, 0.001, "roi"), (2, 0.0001, "device_roi"), (2, None, "pinned")]:
        cam = rig["cams"][c]
        depth, plain = native(cam, scale, where)
        masks = cam["mask"][None]
        want = e.register_objects(cam["rgb"], plain, cam["K"], masks, [_grids(12, 3)], [c + 1], 2)
        got = e.register_objects(_rgb(cam, where), depth, cam["K"], masks, [_grids(12, 3)], [c + 1], 2)
        assert all(_eq(g, w) for g, w in zip(got, want)), (c, scale, where)
    for mix in MIXES:
        got, conv = _mix(rig, mix)
        masks = [c["mask"] for c in rig["cams"]]
        grids = [_grids(10, 5 + c) for c in range(3)]
        want = e.register_cameras(conv, masks, grids, [0, 1, 2], [1, 2, 3], 2)
        res = e.register_cameras(got, masks, grids, [0, 1, 2], [1, 2, 3], 2)
        assert all(_eq(g, w) for g, w in zip(res, want)), mix


def test_graphs_replay_and_launch_counts(rig):
    """After warm-up, new extrinsics, new depth intrinsics, a smaller depth image or a new depth address capture nothing.
    A call with no sensor launches what it launched before any sensor was set; an aligned call adds one launch."""
    from foundationpose_b200 import _lib
    from foundationpose_b200.frames import Depth, DepthSensor

    e, start = rig["e"], rig["start"]
    cam_of, slots = [0, 1, 2], [1, 2, 3]
    plain = [(c["rgb"], c["aligned"], c["K"]) for c in rig["cams"]]

    def launches(frames):
        n0 = _lib.launch_count()
        e.track_cameras(frames, start, cam_of, slots, 2)
        return _lib.launch_count() - n0

    for _ in range(3):
        base = launches(plain)
    for _ in range(3):
        aligned = launches(_mix(rig, MIXES[0])[0])
    assert aligned == base + 1
    assert launches(plain) == base
    n = e.graph_captures()
    c0, c2 = rig["cams"][0], rig["cams"][2]
    raw0 = np.round(c0["native"].astype(np.float64) * 1000).astype(np.uint16)
    raw2 = torch.from_numpy(np.round(c2["native"].astype(np.float64) * 1000).astype(np.uint16)).cuda()
    variants = [DepthSensor(c2["Kd"], ar.rig_T(angle_deg=1.0, t=(0.02, 0.001, 0.0))),  # new extrinsics
                DepthSensor(c2["Kd"] * np.array([[1.01, 1, 1], [1, 1.01, 1], [1, 1, 1]]), c2["T"])]  # new intrinsics
    for s2 in variants:
        assert launches([(c0["rgb"], Depth(raw0, 0.001, sensor=c0["sensor"]), c0["K"]), plain[1],
                         (c2["rgb"], Depth(raw2, 0.001, sensor=s2), c2["K"])]) == aligned
    small = raw2[::2, ::2].contiguous()  # a smaller depth image, at a new address
    Ks = c2["Kd"] * np.array([[0.5, 1, 0.5], [1, 0.5, 0.5], [1, 1, 1]])
    assert launches([plain[0], plain[1], (c2["rgb"], Depth(small, 0.001, sensor=DepthSensor(Ks, c2["T"])), c2["K"])]) == aligned
    assert launches([plain[0], plain[1], (c2["rgb"], Depth(raw2[1:, 1:], 0.001, sensor=c2["sensor"]), c2["K"])]) == aligned
    assert e.graph_captures() == n
    assert launches(plain) == base and e.graph_captures() == n


def test_refusals_enqueue_nothing(rig):
    from foundationpose_b200 import _lib, ops
    from foundationpose_b200.engine import lib
    from foundationpose_b200.frames import Depth, DepthSensor

    e, start = rig["e"], rig["start"]
    cam = rig["cams"][2]  # colour 1280 wide, depth 848: the depth pitch is checked against 848
    for _ in range(2):  # seen, then captured
        _, want = e.track(cam["rgb"], cam["aligned"], cam["K"], start[2], 2)
    n = e.graph_captures()
    Kd = cam["Kd"]

    def rec(H=480, W=640, K=Kd, T=np.eye(4)):
        return _lib.DepthSensor.of(H, W, np.asarray(K, np.float32).reshape(-1), np.asarray(T, np.float32).reshape(-1))

    def refused(camera, r, match):
        with pytest.raises(_lib.FposeError, match=match):
            _lib.check(lib.fp_set_camera_depth_sensor(e._h, camera, C.byref(r)), "fp_set_camera_depth_sensor")

    refused(16, rec(), "camera 16 out of range")
    refused(-1, rec(), "camera -1 out of range")
    for H, W in ((0, 640), (480, 0), (4097, 640), (480, 4097)):
        refused(1, rec(H, W), "depth image .* outside")
    for k, v in ((0, 0.0), (4, -1.0)):
        K = Kd.copy()
        K.reshape(-1)[k] = v
        refused(1, rec(K=K), "focal lengths")
    for k in (2, 8):
        K = Kd.copy()
        K.reshape(-1)[k] = np.inf
        refused(1, rec(K=K), f"K\\[{k}\\] = inf is not finite")
    T = np.eye(4)
    T[1, 3] = np.nan
    refused(1, rec(T=T), r"T_color_from_depth\[7\] = nan is not finite")
    # at call time: a depth pitch short of the sensor's width, a misaligned depth pointer
    raw = np.round(cam["native"].astype(np.float64) * 1000).astype(np.uint16)
    Hd, Wd = raw.shape
    e._set_formats([(0, 1, 0.001, 0, 2 * Wd - 2)], [(Hd, Wd, tuple(Kd.reshape(-1)), tuple(cam["T"].reshape(-1)))])
    Kf = (C.c_float * 9)(*cam["K"].reshape(-1))
    rgb = np.ascontiguousarray(cam["rgb"])
    ticket = C.c_ulonglong()
    with pytest.raises(_lib.FposeError, match="camera 0: depth pitch"):
        _lib.check(lib.fp_track_submit(e._h, C.c_void_p(rgb.ctypes.data), C.c_void_p(raw.ctypes.data), Kf, cam["H"], cam["W"],
                                       C.c_void_p(start[2].data_ptr()), 2, None, None, C.byref(ticket)), "fp_track")
    with pytest.raises(_lib.FposeError, match="camera 0: depth pitch"):
        _lib.check(lib.fp_set_frame(e._h, C.c_void_p(rgb.ctypes.data), C.c_void_p(raw.ctypes.data), Kf, cam["H"], cam["W"], 2,
                                    float("inf"), None), "fp_set_frame")
    buf = np.zeros(Hd * Wd * 2 + 2, np.uint8)
    odd = np.frombuffer(buf.data, np.uint16, Hd * Wd, offset=1).reshape(Hd, Wd)
    odd[...] = raw
    with pytest.raises(_lib.FposeError, match="camera 0: depth buffer .* not aligned"):
        e.track(rgb, Depth(odd, 0.001, sensor=cam["sensor"]), cam["K"], start[2], 2)
    with pytest.raises(_lib.FposeError, match="camera 2: depth buffer .* not aligned"):
        e.track_cameras([(rgb, cam["aligned"], cam["K"])] * 2 + [(rgb, Depth(odd, 0.001, sensor=cam["sensor"]), cam["K"])],
                        start, [0, 1, 2], [1, 1, 1], 2)
    # fp_align_depth: host memory, bad arguments
    s = DepthSensor(Kd, cam["T"])
    with pytest.raises(_lib.FposeError, match="must be a CUDA tensor"):
        ops.align_depth(Depth(raw, 0.001, sensor=s), None, cam["K"], cam["H"], cam["W"])
    r = rec(Hd, Wd)
    pinned = torch.from_numpy(raw).pin_memory()
    out = torch.empty(cam["H"], cam["W"], device="cuda")
    dev_raw = torch.from_numpy(raw).cuda()
    Kc = (C.c_float * 9)(*cam["K"].reshape(-1))
    host_out = np.empty((cam["H"], cam["W"]), np.float32)
    for args, match in [((pinned.data_ptr(), 1, 0.001, 0, C.byref(r), Kc, cam["H"], cam["W"], out.data_ptr()), "depth is not device"),
                        ((dev_raw.data_ptr(), 1, 0.001, 0, C.byref(r), Kc, cam["H"], cam["W"], host_out.ctypes.data), "out is not device"),
                        ((dev_raw.data_ptr(), 1, 0.001, 2 * Wd - 2, C.byref(r), Kc, cam["H"], cam["W"], out.data_ptr()), "depth pitch"),
                        ((dev_raw.data_ptr() + 1, 1, 0.001, 0, C.byref(r), Kc, cam["H"], cam["W"], out.data_ptr()), "not aligned"),
                        ((dev_raw.data_ptr(), 1, 0.0, 0, C.byref(r), Kc, cam["H"], cam["W"], out.data_ptr()), "depth scale"),
                        ((dev_raw.data_ptr(), 2, 0.001, 0, C.byref(r), Kc, cam["H"], cam["W"], out.data_ptr()), "unknown depth format"),
                        ((dev_raw.data_ptr(), 1, 0.001, 0, C.byref(rec(0, Wd)), Kc, cam["H"], cam["W"], out.data_ptr()), "outside"),
                        ((dev_raw.data_ptr(), 1, 0.001, 0, C.byref(r), Kc, 0, cam["W"], out.data_ptr()), "empty"),
                        ((dev_raw.data_ptr(), 1, 0.001, 0, C.byref(r), C.cast(out.data_ptr(), C.POINTER(C.c_float)), cam["H"],
                          cam["W"], out.data_ptr()), "K_color is device memory")]:
        with pytest.raises(_lib.FposeError, match=match):
            _lib.check(lib.fp_align_depth(*args, None), "fp_align_depth")
    if torch.cuda.device_count() > 1:
        other = torch.from_numpy(raw).to("cuda:1")
        with pytest.raises(_lib.FposeError, match="lives on device 1"):
            _lib.check(lib.fp_align_depth(other.data_ptr(), 1, 0.001, 0, C.byref(r), Kc, cam["H"], cam["W"], out.data_ptr(), None),
                       "fp_align_depth")
        with pytest.raises(_lib.FposeError, match="device memory of another device"):
            e.track(_place(cam["rgb"], "device"), Depth(other, 0.001, sensor=s), cam["K"], start[2], 2)
    # the context is as it was: nothing was captured, the next calls give the same pose
    e._set_formats([(0, 0, 0.0, 0, 0)], [None])
    assert e.graph_captures() == n
    _, again = e.track(cam["rgb"], cam["aligned"], cam["K"], start[2], 2)
    assert _eq(again, want)
    assert e.graph_captures() == n


def test_estimator_calls_with_sensors(rig):
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
    depth, d = native(cam, 0.001, "roi")
    assert np.array_equal(plain.register(cam["K"], cam["rgb"], d, cam["mask"], iteration=2),
                          wrapped.register(cam["K"], cam["rgb"], depth, cam["mask"], iteration=2))
    for scale, where in [(0.0001, "packed"), (0.00025, "device_roi"), (None, "pinned")]:
        depth, d = native(cam, scale, where)
        r = cam["rgb"]
        if where.startswith("device"):
            r, d = torch.from_numpy(r).cuda(), torch.from_numpy(d).cuda()
        elif where == "pinned":
            r, d = torch.from_numpy(r), torch.from_numpy(d)
        rw = torch.from_numpy(cam["rgb"]).cuda() if where.startswith("device") else cam["rgb"]
        assert np.array_equal(plain.track_one(r, d, cam["K"], 2), wrapped.track_one(rw, depth, cam["K"], 2)), where
    depth, d = native(cam, 0.001, "roi")
    assert np.array_equal(estimater.track_objects([plain], cam["rgb"], d, cam["K"]),
                          estimater.track_objects([wrapped], cam["rgb"], depth, cam["K"]))
    assert np.array_equal(estimater.register_objects([plain], cam["K"], cam["rgb"], d, [cam["mask"]], iteration=2),
                          estimater.register_objects([wrapped], cam["K"], cam["rgb"], depth, [cam["mask"]], iteration=2))
    # cameras 0 (with a sensor) and 1 (without): register_cameras, then track_cameras
    m1 = rig["objs"][1]
    mk1 = lambda: FoundationPose(model_pts=m1.vertices, model_normals=m1.vertex_normals, mesh=m1, scorer=scorer, refiner=refiner)
    ests = dict(plain=[plain, mk1()], wrapped=[wrapped, mk1()])
    cams = rig["cams"][:2]
    for k, mix in enumerate([[(0.001, "roi"), (None, "packed")], [(0.0001, "packed"), (0.001, "roi")]]):  # host numpy only
        got, conv = _mix(rig, mix, cams=(0, 1))
        views = {kind: [([ests[kind][i]], *fr[i]) for i in range(2)] for kind, fr in (("plain", conv), ("wrapped", got))}
        if k == 0:
            res = {kind: estimater.register_cameras([(*v, [c["mask"]]) for v, c in zip(views[kind], cams)], iteration=2)
                   for kind in views}
        else:
            res = {kind: estimater.track_cameras(views[kind]) for kind in views}
        for a_, b_ in zip(res["plain"], res["wrapped"]):
            assert np.array_equal(np.stack(a_), np.stack(b_)), (k, mix)
    e.close()


def test_debug_canvas_of_one_register(rig, tmp_path):
    """The debug >= 2 register: poses and the refiner's vis canvas equal those of the host-aligned frame."""
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.estimater import FoundationPose, PoseRefinePredictor, ScorePredictor
    from foundationpose_b200.weights import random_state_dict

    cam = rig["cams"][2]
    depth, d = native(cam, 0.001, "packed")
    m = rig["objs"][2]
    out = []
    for kind, dep in (("plain", d), ("wrapped", depth)):
        e = Engine()
        refiner = PoseRefinePredictor(engine=e, state_dict=random_state_dict("refine", 0))
        scorer = ScorePredictor(engine=e, state_dict=random_state_dict("score", 0))
        est = FoundationPose(model_pts=m.vertices, model_normals=m.vertex_normals, mesh=m, scorer=scorer, refiner=refiner)
        pose = est.register(cam["K"], cam["rgb"], dep, cam["mask"], iteration=2)
        poses = rig["start"][2:3].repeat(4, 1, 1)
        poses[1:, :3, 3] += torch.tensor([0.003, -0.002, 0.005], device="cuda")
        canvases = [e.vis("refine", rig["start"][2:3].repeat(4, 1, 1), poses).cpu(), e.vis("score", poses, order=[2, 0, 3, 1]).cpu()]
        out.append((pose, canvases))
        e.close()
    assert np.array_equal(out[0][0], out[1][0])
    assert all(torch.equal(a, b) for a, b in zip(out[0][1], out[1][1]))
