"""Host inputs of fp_set_frame, fp_start_poses and fp_register: pageable memory is staged by the library through the
context's staging sets, page-locked memory is read in place.  Every path gives the same results bit for bit, pageable
buffers may be overwritten as soon as the call returns, set_frame / start_poses / refine on pageable input do not wait
on the host for earlier work on the stream, and set_frame shares the staging sets with non-blocking tracking calls without changing their results."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N_HYP = 16
ITERS = 2


@pytest.fixture(scope="module")
def scene():
    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.estimater import make_mesh_tensors
    from foundationpose_b200.weights import random_state_dict

    mesh = synth.make_mesh(3)
    pose = np.eye(4)
    pose[:3, :3] = synth.random_rotation(2)
    pose[:3, 3] = [0.01, 0.015, 0.62]
    rgb, depth, mask = synth.make_scene(mesh.visual.image, pose)
    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    mt = make_mesh_tensors(mesh)
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(mesh.vertices), uv=mt.get("uv"), tex=mt.get("tex"),
               vertex_colors=mt.get("vcolor"))
    grid = np.tile(np.eye(4, dtype=np.float32), (N_HYP, 1, 1))
    for i in range(N_HYP):
        grid[i, :3, :3] = synth.random_rotation(30 + i)
    seq = synth.track_sequence(6, pose, seed=4)
    frames = [synth.make_scene(mesh.visual.image, p, seed=10 + t)[:2] for t, p in enumerate(seq)]
    return dict(e=e, rgb=rgb, depth=depth, mask=(mask > 0).astype(np.uint8), K=synth.DEFAULT_K, pose=pose,
                grid=torch.from_numpy(grid).cuda(), frames=frames)


def _start_poses_pinned(e, mask, grid):
    """fp_start_poses on a page-locked host mask (Engine.start_poses always hands the library a fresh pageable copy)."""
    from foundationpose_b200 import _lib
    from foundationpose_b200.engine import _p, _stream, lib

    m = torch.from_numpy(mask).pin_memory()
    poses = torch.empty(len(grid), 4, 4, dtype=torch.float32, device="cuda")
    info = torch.empty(4, dtype=torch.float32, device="cuda")
    _lib.check(lib.fp_start_poses(e._h, C.c_void_p(m.data_ptr()), 0, _p(grid), len(grid), _p(poses), _p(info), _stream()),
               "fp_start_poses")
    torch.cuda.synchronize()  # the library reads the pinned mask in place
    return poses, info


def _frame_and_start(s, kind):
    e = s["e"]
    if kind == "pageable":
        e.set_frame(s["rgb"], s["depth"], s["K"])
        poses, info = e.start_poses(s["mask"], s["grid"])
    elif kind == "pinned":
        rgb, depth = torch.from_numpy(s["rgb"]).pin_memory(), torch.from_numpy(s["depth"]).pin_memory()
        e.set_frame(rgb, depth, s["K"])
        poses, info = _start_poses_pinned(e, s["mask"], s["grid"])
    else:
        e.set_frame(torch.from_numpy(s["rgb"]).cuda(), torch.from_numpy(s["depth"]).cuda(), s["K"])
        poses, info = e.start_poses(torch.from_numpy(s["mask"]).cuda(), s["grid"])
    depth, xyz = e.get_depth()
    return [t.clone() for t in (depth, xyz, poses, info)]


def test_pageable_pinned_and_device_inputs_agree(scene):
    ref = _frame_and_start(scene, "device")
    assert float(ref[3][3]) >= 4, "the scene's mask must hold valid depth"
    for kind in ("pageable", "pinned"):
        got = _frame_and_start(scene, kind)
        for name, a, b in zip(("depth", "xyz", "start poses", "info"), got, ref):
            assert torch.equal(a, b), f"{kind} input: {name} differs from device input"
    # fp_register's start poses: staged from pageable memory or read in place from page-locked memory
    start = ref[2].cpu().numpy()
    p1, s1, b1 = scene["e"].register_host(start, ITERS)
    p2, s2, b2 = scene["e"].register_host(torch.from_numpy(start).pin_memory(), ITERS)
    assert torch.equal(p1, p2) and torch.equal(s1, s2) and b1 == b2


def _queue_sleep():
    """Queues ~0.1-0.3 s of device work on the current stream, with nothing of the library's in flight, and returns an
    event recorded after it."""
    torch.cuda.synchronize()
    torch.cuda._sleep(500_000_000)
    after_sleep = torch.cuda.Event()
    after_sleep.record()
    return after_sleep


def test_pageable_inputs_may_be_overwritten_on_return(scene):
    s, e = scene, scene["e"]
    ref = _frame_and_start(s, "pageable")
    ref_out, _, _ = e.refine(ref[2], ITERS)
    rgb, depth, mask = s["rgb"].copy(), s["depth"].copy(), s["mask"].copy()
    after_sleep = _queue_sleep()
    e.set_frame(rgb, depth, s["K"])
    rgb[:] = 0
    depth[:] = 0
    poses, info = e.start_poses(mask, s["grid"])
    mask[:] = 0
    # the uploads queue behind the sleep: the host overwrote every array before any of them ran
    assert not after_sleep.query(), "the sleep ended before the arrays were overwritten"
    out, _, _ = e.refine(poses, ITERS)
    assert torch.equal(poses, ref[2]) and torch.equal(info, ref[3])
    assert torch.equal(out, ref_out)


def test_pageable_inputs_do_not_wait_on_the_stream(scene):
    s, e = scene, scene["e"]
    ref = _frame_and_start(s, "pageable")
    ref_out, _, _ = e.refine(ref[2], ITERS)  # the refine graph is cached: the timed calls capture nothing
    after_sleep = _queue_sleep()
    e.set_frame(s["rgb"], s["depth"], s["K"])
    poses, info = e.start_poses(s["mask"], s["grid"])
    out, _, _ = e.refine(poses, ITERS)
    returned_early = not after_sleep.query()
    torch.cuda.synchronize()
    assert returned_early, "set_frame, start_poses or refine waited on the host for work queued before them"
    assert torch.equal(poses, ref[2]) and torch.equal(info, ref[3]) and torch.equal(out, ref_out)


def test_set_frame_between_pipelined_tracking_calls(scene):
    s, e = scene, scene["e"]
    pose0 = torch.from_numpy(s["pose"].astype(np.float32)).cuda()
    blocking = [e.track(rgb, depth, s["K"], pose0 if t == 0 else None, ITERS)[1] for t, (rgb, depth) in enumerate(s["frames"])]
    ref_depth = _frame_and_start(s, "pageable")[0]
    pending = []
    for t, (rgb, depth) in enumerate(s["frames"]):
        pending.append(e.track(rgb, depth, s["K"], pose0 if t == 0 else None, ITERS, wait=False)[1])
        e.set_frame(s["rgb"], s["depth"], s["K"])  # stages through the set after the submit's, in turn
    got = [p.result() for p in pending]
    for t, (a, b) in enumerate(zip(got, blocking)):
        assert np.array_equal(a, b), f"frame {t}: the pipelined pose differs from the blocking one"
    assert torch.equal(e.get_depth()[0], ref_depth)
