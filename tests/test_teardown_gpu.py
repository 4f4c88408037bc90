"""Closing an engine and an fp_group returns the device memory they held: two identical create / warm / close cycles in
one process leave the same free device memory.  The first cycle also pays one-time costs (modules loaded on first
launch), so the cycles are compared with each other, not with the memory before them."""
import gc

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MiB = 1 << 20


@pytest.fixture(scope="module")
def scene():
    from foundationpose_b200 import hypotheses, synth
    from foundationpose_b200.estimater import make_mesh_tensors
    from foundationpose_b200.weights import random_state_dict

    mesh = synth.make_mesh(3)
    mt = make_mesh_tensors(mesh)
    poses = []
    for k, t in enumerate(([-0.05, 0.0, 0.6], [0.06, 0.02, 0.65])):
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(k)
        p[:3, 3] = t
        poses.append(p)
    tex = mesh.visual.image
    rgb, depth, owner = synth.make_multi_scene([(tex, p, 1.0) for p in poses])
    K1 = np.array([[460.0, 0, 242.0], [0, 455.0, 178.0], [0, 0, 1]])
    rgb1, depth1, _ = synth.make_multi_scene([(tex, poses[1], 1.0)], K1, 360, 480, seed=2)
    return dict(mesh=(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(mesh.vertices)), uv=mt["uv"], tex=mt["tex"],
                sd_r=random_state_dict("refine", 0), sd_s=random_state_dict("score", 0), poses=np.stack(poses).astype(np.float32),
                rgb=rgb, depth=depth, masks=np.stack([owner == 0, owner == 1]), cam1=(rgb1, depth1, K1),
                grid=hypotheses.make_rotation_grid()[:40].astype(np.float32))


def _cycle(s):
    """Every entry point that owns buffers, warmed (eager, capture, replay), then everything closed; the free device
    memory after."""
    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.group import EngineGroup

    K = synth.DEFAULT_K
    e = Engine()
    e.load_network("refine", s["sd_r"])
    e.load_network("score", s["sd_s"])
    for slot in (0, 1):
        e.set_mesh(*s["mesh"], uv=s["uv"], tex=s["tex"], slot=slot)
    poses = torch.from_numpy(s["poses"]).cuda()
    grid = torch.from_numpy(s["grid"]).cuda()
    for _ in range(3):
        e.track(s["rgb"], s["depth"], K, poses[0], 2)
        e.track_objects(s["rgb"], s["depth"], K, poses, [0, 1], 2)
        e.track_cameras([(s["rgb"], s["depth"], K), s["cam1"]], poses, [0, 1], [0, 1], 2)
        e.register_objects(s["rgb"], s["depth"], K, s["masks"], [grid, grid], [0, 1], 2)
    g = EngineGroup([0])
    g.load_network("refine", s["sd_r"])
    g.load_network("score", s["sd_s"])
    g.set_mesh(*s["mesh"], uv=s["uv"], tex=s["tex"])
    for _ in range(3):
        g.register(s["rgb"], s["depth"], K, s["masks"][0], s["grid"], iterations=2)
    e.close()
    g.close()
    del poses, grid
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def test_closing_returns_device_memory(scene):
    first = _cycle(scene)
    second = _cycle(scene)
    assert abs(second - first) <= 4 * MiB, f"free device memory moved by {(first - second) / MiB:.1f} MiB from one cycle to the next"
