"""Frames and masks already on the GPU: Engine.track, track_objects, track_cameras, register_objects and register_cameras
with CUDA tensors as frames and masks, read in place by the library, against the same calls with host arrays on the same
seeded scenes, bit for bit.  Also: a camera mix of host and device buffers, non-blocking calls whose device buffers are
rewritten or released while the call is in flight, a call on a side stream right after the kernel that produced its
frame, graph captures and launch counts, refusals, and memory of the allocator's expandable segments."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N_FRAMES = 4
# subdivisions, texture seed, scale
SPECS = [(3, 0, 1.0), (2, 5, 0.8), (3, 9, 1.2)]
# per camera: H, W, K, objects it sees (indices into SPECS).  333 x 257 is not a multiple of the frame filter's tile.
CAMERAS = [(480, 640, [[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1]], [0, 1]),
           (720, 1280, [[920.0, 0, 640.0], [0, 915.0, 360.0], [0, 0, 1]], [2]),
           (257, 333, [[330.0, 0, 165.5], [0, 328.0, 130.0], [0, 0, 1]], [1])]


def _load(e, mesh, slot):
    from foundationpose_b200 import synth
    from foundationpose_b200.estimater import make_mesh_tensors

    mt = make_mesh_tensors(mesh)
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(mesh.vertices), uv=mt.get("uv"), tex=mt.get("tex"),
               vertex_colors=mt.get("vcolor"), slot=slot)


def _engine(objs):
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.weights import random_state_dict

    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    e.set_config("refine")
    e.set_config("score")
    for k, m in enumerate(objs):
        _load(e, m, k + 1)
    _load(e, objs[0], 0)
    return e


def make_rig():
    """N_FRAMES frames of every camera (each object on its own random walk), every object's mask in every frame, and the
    (camera, object) pairs' start poses: the first frame's poses plus a few millimetres."""
    from foundationpose_b200 import synth

    objs = [synth.make_mesh(s, tex_seed=t, tex_size=256, scale=sc) for s, t, sc in SPECS]
    rng = np.random.default_rng(3)
    cams = []
    for c, (H, W, K, seen) in enumerate(CAMERAS):
        K = np.asarray(K, dtype=np.float64)
        walks = []
        for j, k in enumerate(seen):
            p = np.eye(4)
            p[:3, :3] = synth.random_rotation(31 + 5 * c + k)
            z = 0.6 + 0.05 * j
            p[:3, 3] = [((W * (j + 1) / (len(seen) + 1)) - K[0, 2]) * z / K[0, 0], 0.01 * (-1) ** j, z]
            walks.append(synth.track_sequence(N_FRAMES, p, seed=40 + 3 * c + j))
        frames, masks = [], []
        for t in range(N_FRAMES):
            rgb, depth, owner = synth.make_multi_scene([(objs[k].visual.image, walks[j][t], SPECS[k][2]) for j, k in enumerate(seen)],
                                                       K, H, W, seed=200 * c + t)
            frames.append((rgb, depth.astype(np.float32), K))
            masks.append([owner == j for j in range(len(seen))])
        start = []
        for w in walks:
            q = w[0].copy()
            q[:3, 3] += rng.normal(0, 0.003, 3)
            start.append(q.astype(np.float32))
        cams.append(dict(frames=frames, masks=masks, seen=list(seen), start=start))
    pairs = [(c, j) for c, cam in enumerate(cams) for j in range(len(cam["seen"]))]
    return dict(objs=objs, cams=cams, pairs=pairs, cam_of=[c for c, _ in pairs], slots=[cams[c]["seen"][j] + 1 for c, j in pairs],
                start=torch.from_numpy(np.stack([cams[c]["start"][j] for c, j in pairs])).cuda())


@pytest.fixture(scope="module")
def rig():
    r = make_rig()
    r["e"] = _engine(r["objs"])
    yield r
    r["e"].close()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _views(rig, t, on_device):
    """Frame t of every camera; camera c's rgb / depth are CUDA tensors where on_device[c] says so ("rgb" / "depth": only
    that buffer)."""
    out = []
    for c, cam in enumerate(rig["cams"]):
        rgb, depth, K = cam["frames"][t]
        where = on_device[c]
        out.append((_dev(rgb) if where in (True, "rgb") else rgb, _dev(depth) if where in (True, "depth") else depth, K))
    return out


def _track_cameras(rig, views, poses_in, wait=True):
    return rig["e"].track_cameras(views, poses_in, rig["cam_of"], rig["slots"], 2, wait=wait)


def _grids(n_obj, n_rot=12, seed=0):
    from foundationpose_b200 import synth

    out = []
    for i in range(n_obj):
        g = np.tile(np.eye(4, dtype=np.float32), (n_rot, 1, 1))
        for s in range(n_rot):
            g[s, :3, :3] = synth.random_rotation(seed + 100 * i + s)
        out.append(torch.from_numpy(g).cuda())
    return out


def _same(a, b, what):
    if torch.is_tensor(a):
        assert torch.equal(a, b), what
    else:
        assert np.array_equal(a, b), what


def test_track_sequence_with_continuation(rig):
    """Engine.track over N_FRAMES frames of camera 0 (the first with pose_in, then continuing from the context's pose)."""
    e, cam = rig["e"], rig["cams"][0]
    got = {}
    for on_dev in (False, True):
        outs = []
        for t in range(N_FRAMES):
            rgb, depth, K = cam["frames"][t]
            if on_dev:
                rgb, depth = _dev(rgb), _dev(depth)
            dev, host = e.track(rgb, depth, K, rig["start"][0] if t == 0 else None, 2)
            outs.append((dev.clone(), host))
        got[on_dev] = outs
    for t, ((a, x), (b, y)) in enumerate(zip(got[False], got[True])):
        _same(a, b, f"frame {t}: device poses differ")
        _same(x, y, f"frame {t}: host poses differ")


def test_track_objects(rig):
    """track_objects with M = 3 objects of one frame (camera 0's two objects and one of them again)."""
    e, cam = rig["e"], rig["cams"][0]
    rgb, depth, K = cam["frames"][1]
    poses_in = torch.stack([rig["start"][0], rig["start"][1], rig["start"][0] + 0.002])
    slots = [cam["seen"][0] + 1, cam["seen"][1] + 1, cam["seen"][0] + 1]
    want = e.track_objects(rgb, depth, K, poses_in, slots, 2)
    got = e.track_objects(_dev(rgb), _dev(depth), K, poses_in, slots, 2)
    _same(got[0], want[0], "device poses differ")
    _same(got[1], want[1], "host poses differ")


@pytest.mark.parametrize("on_device", [(True, False, True), (True, True, True), (False, "rgb", "depth")],
                         ids=["mixed", "all_device", "per_buffer"])
def test_track_cameras(rig, on_device):
    """C = 3 cameras of 640x480, 1280x720 and 333x257: cameras 0 and 2 on the device and camera 1 on the host, all on the
    device, or one buffer of a camera on the device and the other on the host."""
    pose_h = pose_d = rig["start"]
    for t in range(N_FRAMES):
        pose_h, want = _track_cameras(rig, _views(rig, t, (False,) * 3), pose_h)
        pose_d, got = _track_cameras(rig, _views(rig, t, on_device), pose_d)
        _same(pose_d, pose_h, f"frame {t}: device poses differ")
        _same(got, want, f"frame {t}: host poses differ")


def _register_objects_args(rig, t=0):
    cam = rig["cams"][0]
    rgb, depth, K = cam["frames"][t]
    masks = np.stack(cam["masks"][t])
    return rgb, depth, K, masks, [k + 1 for k in cam["seen"]]


@pytest.mark.parametrize("mask_dtype", [torch.bool, torch.uint8, torch.float32])
def test_register_objects(rig, mask_dtype):
    e = rig["e"]
    rgb, depth, K, masks, slots = _register_objects_args(rig)
    grids = _grids(len(slots))
    want = e.register_objects(rgb, depth, K, masks, grids, slots, 2)
    dmask = _dev(masks).to(mask_dtype)
    if mask_dtype == torch.float32:
        dmask = dmask * 0.5  # fractional: only `> 0` counts
    got = e.register_objects(_dev(rgb), _dev(depth), K, dmask, grids, slots, 2)
    for name, a, b in zip(("poses", "scores", "best", "info"), got, want):
        _same(a, b, f"{name} differ")
    # a sequence of per-object CUDA masks, one of them a non-contiguous view
    wide = torch.zeros(masks.shape[1], 2 * masks.shape[2], dtype=torch.uint8, device="cuda")
    wide[:, ::2] = _dev(masks[1]).to(torch.uint8)
    got = e.register_objects(_dev(rgb), depth, K, [_dev(masks[0]).to(torch.uint8), wide[:, ::2]], grids, slots, 2)
    for name, a, b in zip(("poses", "scores", "best", "info"), got, want):
        _same(a, b, f"{name} differ (a list of masks)")


def _register_cameras_args(rig, t=0):
    views = [cam["frames"][t] for cam in rig["cams"]]
    masks = [rig["cams"][c]["masks"][t][j] for c, j in rig["pairs"]]
    return views, masks


def test_register_cameras_mixed(rig):
    """Cameras 0 and 2 on the device, camera 1 on the host; the masks alternate between host and device."""
    e = rig["e"]
    views, masks = _register_cameras_args(rig)
    grids = _grids(len(masks), seed=7)
    want = e.register_cameras(views, masks, grids, rig["cam_of"], rig["slots"], 2)
    dviews = [(_dev(rgb), _dev(depth), K) if c != 1 else (rgb, depth, K) for c, (rgb, depth, K) in enumerate(views)]
    dmasks = [_dev(m) if i % 2 == 0 else m for i, m in enumerate(masks)]
    got = e.register_cameras(dviews, dmasks, grids, rig["cam_of"], rig["slots"], 2)
    for name, a, b in zip(("poses", "scores", "best", "info"), got, want):
        _same(a, b, f"{name} differ")
    got = e.register_cameras([(_dev(rgb), _dev(depth), K) for rgb, depth, K in views], [_dev(m).float() for m in masks], grids,
                             rig["cam_of"], rig["slots"], 2)
    for name, a, b in zip(("poses", "scores", "best", "info"), got, want):
        _same(a, b, f"{name} differ (all on the device)")


@pytest.fixture(scope="module")
def blocking(rig):
    """The host-frame blocking sequence of track_cameras: device and host poses of every frame."""
    pose, dev, host = rig["start"], [], []
    for t in range(N_FRAMES):
        pose, h = _track_cameras(rig, _views(rig, t, (False,) * 3), pose)
        dev.append(pose.clone())
        host.append(h)
    return dev, host


def _garbage_like(views):
    return [(torch.full_like(rgb, 7), torch.full_like(depth, -1.0)) for rgb, depth, _ in views]


def test_in_flight_buffers_rewritten_on_the_stream(rig, blocking):
    """wait=False, two calls in flight, every camera's frame in one device buffer that the caller rewrites on the same
    stream with the next frame right after each submit."""
    src = [_views(rig, t, (True,) * 3) for t in range(N_FRAMES)]
    bufs = [(torch.empty_like(rgb), torch.empty_like(depth), K) for rgb, depth, K in src[0]]
    pose, dev, host, prev = rig["start"], [], [], None
    for (rgb, depth, _), (r, d, _) in zip(bufs, src[0]):
        rgb.copy_(r)
        depth.copy_(d)
    for t in range(N_FRAMES):
        pose, pending = _track_cameras(rig, bufs, pose, wait=False)
        dev.append(pose)
        if t + 1 < N_FRAMES:
            for (rgb, depth, _), (r, d, _) in zip(bufs, src[t + 1]):  # ordered after the call on the stream
                rgb.copy_(r)
                depth.copy_(d)
        if prev is not None:
            host.append(prev.result())
        prev = pending
    del bufs
    junk = _garbage_like(src[0])
    host.append(prev.result())
    torch.cuda.synchronize()
    for t in range(N_FRAMES):
        _same(dev[t], blocking[0][t], f"frame {t}: device poses differ")
        _same(host[t], blocking[1][t], f"frame {t}: host poses differ")
    del junk


def test_in_flight_buffers_released(rig, blocking):
    """wait=False, two calls in flight, each call's frames made on a producer stream; the caller drops them right after
    the submit and the producer stream at once allocates and fills buffers of the same sizes before the result is
    collected.  The engine holds the frames and records them on the call's stream, so nothing overwrites them."""
    src = [_views(rig, t, (True,) * 3) for t in range(N_FRAMES)]
    producer = torch.cuda.Stream()
    pose, dev, host, prev, junk = rig["start"], [], [], None, []
    for t in range(N_FRAMES):
        with torch.cuda.stream(producer):
            views = [(rgb.clone(), depth.clone(), K) for rgb, depth, K in src[t]]
        torch.cuda.current_stream().wait_stream(producer)
        pose, pending = _track_cameras(rig, views, pose, wait=False)
        dev.append(pose)
        del views
        with torch.cuda.stream(producer):
            junk.append(_garbage_like(src[t]))  # the sizes of the frames just dropped
        if prev is not None:
            host.append(prev.result())
        prev = pending
    host.append(prev.result())
    torch.cuda.synchronize()
    for t in range(N_FRAMES):
        _same(dev[t], blocking[0][t], f"frame {t}: device poses differ")
        _same(host[t], blocking[1][t], f"frame {t}: host poses differ")


def test_side_stream_frame_made_just_before(rig, blocking):
    """The call runs under torch.cuda.stream(s), its frames produced by kernels on s just before it."""
    src = _views(rig, 0, (True,) * 3)
    inverted = [(255 - rgb, depth * 0.5, K) for rgb, depth, K in src]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        views = [(255 - rgb, depth * 2.0, K) for rgb, depth, K in inverted]
        dev, host = _track_cameras(rig, views, rig["start"])
    s.synchronize()
    _same(dev, blocking[0][0], "device poses differ")
    _same(host, blocking[1][0], "host poses differ")


def test_no_captures_and_same_launches(rig):
    """After warm-up, device frames at new addresses and host <-> device alternation capture no graph, and a call launches
    the same kernels whichever way its frames arrive."""
    from foundationpose_b200 import _lib

    e = rig["e"]
    for on_dev in ((False,) * 3, (True,) * 3, (True, False, True)):
        for _ in range(2):
            _track_cameras(rig, _views(rig, 0, on_dev), rig["start"])
    rgb, depth, K, masks, slots = _register_objects_args(rig)
    grids = _grids(len(slots))
    for _ in range(2):
        e.register_objects(rgb, depth, K, masks, grids, slots, 2)
        e.register_objects(_dev(rgb), _dev(depth), K, _dev(masks), grids, slots, 2)
    captures = e.graph_captures()
    launches = {}
    for t in range(N_FRAMES):
        for on_dev in ((False,) * 3, (True,) * 3, (True, False, True)):
            n0 = _lib.launch_count()
            _track_cameras(rig, _views(rig, t, on_dev), rig["start"])  # fresh tensors: new addresses every call
            launches.setdefault(on_dev, set()).add(_lib.launch_count() - n0)
    for on_dev in (False, True):
        n0 = _lib.launch_count()
        if on_dev:
            e.register_objects(_dev(rgb), _dev(depth), K, _dev(masks), grids, slots, 2)
        else:
            e.register_objects(rgb, depth, K, masks, grids, slots, 2)
        launches.setdefault(("register", on_dev), set()).add(_lib.launch_count() - n0)
    assert e.graph_captures() == captures, "where a frame lives made a graph capture"
    assert launches[(False,) * 3] == launches[(True,) * 3] == launches[(True, False, True)], launches
    assert len(launches[(False,) * 3]) == 1, launches
    assert launches[("register", False)] == launches[("register", True)], launches


def test_refusals_enqueue_nothing(rig, blocking):
    from foundationpose_b200 import _lib

    e = rig["e"]
    views = _views(rig, 0, (True,) * 3)
    rgb0, depth0, K0 = views[0]
    rgb, depth, K, masks, slots = _register_objects_args(rig)
    grids = _grids(len(slots))
    bad = [
        lambda: e.track_cameras([(rgb0.float(), depth0, K0)] + views[1:], rig["start"], rig["cam_of"], rig["slots"], 2),
        lambda: e.track_cameras([(rgb0[:-1], depth0, K0)] + views[1:], rig["start"], rig["cam_of"], rig["slots"], 2),
        lambda: e.track(rgb0, depth0[:, :-1], K0, rig["start"][0], 2),
        lambda: e.track_objects(rgb0.to(torch.int32), depth0, K0, rig["start"][:2], slots, 2, wait=False),
        lambda: e.register_objects(_dev(rgb), _dev(depth), K, _dev(masks)[:, :-1], grids, slots, 2),
        lambda: e.register_cameras([(_dev(r), _dev(d), k) for r, d, k in _register_cameras_args(rig)[0]],
                                   [_dev(m)[1:] for m in _register_cameras_args(rig)[1]], _grids(len(rig["pairs"])),
                                   rig["cam_of"], rig["slots"], 2),
    ]
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    for i, call in enumerate(bad):
        with pytest.raises(ValueError):
            call()
        assert _lib.launch_count() == n0, f"refusal {i} enqueued work"
    if torch.cuda.device_count() >= 2:
        with torch.cuda.device(1):
            other = [(rgb0.to("cuda:1"), depth0, K0)] + views[1:]
        with pytest.raises(_lib.FposeError, match="another device"):
            e.track_cameras(other, rig["start"], rig["cam_of"], rig["slots"], 2)
        with pytest.raises(_lib.FposeError, match="another device"):
            e.register_objects(_dev(rgb), _dev(depth), K, _dev(masks).to("cuda:1"), grids, slots, 2)
        assert _lib.launch_count() == n0, "a frame of another device enqueued work"
    dev, host = _track_cameras(rig, views, rig["start"])
    _same(dev, blocking[0][0], "the engine after the refusals: device poses differ")
    _same(host, blocking[1][0], "the engine after the refusals: host poses differ")


def mixed_cameras_check():
    """The mixed track_cameras case on a fresh engine, against the same calls with host frames."""
    r = make_rig()
    r["e"] = _engine(r["objs"])
    pose_h = pose_d = r["start"]
    for t in range(N_FRAMES):
        pose_h, want = _track_cameras(r, _views(r, t, (False,) * 3), pose_h)
        pose_d, got = _track_cameras(r, _views(r, t, (True, False, True)), pose_d)
        _same(pose_d, pose_h, f"frame {t}: device poses differ")
        _same(got, want, f"frame {t}: host poses differ")
    segments = torch.cuda.memory_snapshot()
    if segments and "is_expandable" in segments[0]:
        assert any(s["is_expandable"] for s in segments), "the allocator made no expandable segment"
    r["e"].close()


def test_expandable_segments_subprocess():
    """Tensors of the caching allocator's expandable segments (virtual memory mapped in pieces) are device memory too."""
    env = dict(os.environ, PYTORCH_CUDA_ALLOC_CONF="expandable_segments:True")
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path.insert(0, {os.path.dirname(here)!r}); sys.path.insert(0, {here!r}); "
            "import test_device_frames_gpu as t; t.mixed_cameras_check(); print('ok')")
    res = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and res.stdout.strip().endswith("ok"), res.stdout[-2000:] + res.stderr[-4000:]
