"""The four multi-object paths (track_objects, track_cameras, register_objects, register_cameras) and track interleaved
on one context: they share the context's frame (camera 0), the other cameras' buffers and one argument block, so each
call's output must not depend on what the others did before it."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# subdivisions, texture seed, scale
SPECS = [(3, 0, 1.0), (2, 5, 0.7), (3, 9, 1.3)]
# per camera: H, W, K, objects it sees (indices into SPECS); two frame sizes
CAMERAS = [(480, 640, [[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1]], [0, 1]),
           (720, 1280, [[920.0, 0, 640.0], [0, 915.0, 360.0], [0, 0, 1]], [2]),
           (480, 640, [[600.0, 0, 316.0], [0, 604.0, 244.0], [0, 0, 1]], [1, 2])]


def _load(e, mesh, slot):
    from foundationpose_b200 import synth
    from foundationpose_b200.estimater import make_mesh_tensors

    mt = make_mesh_tensors(mesh)
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(mesh.vertices), uv=mt.get("uv"), tex=mt.get("tex"),
               vertex_colors=mt.get("vcolor"), slot=slot)


def _engine(meshes):
    """Refiner and scorer, object k in slot k + 1, and in slot 0 the object `track` follows (camera 2's first)."""
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.weights import random_state_dict

    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    e.set_config("refine")
    e.set_config("score")
    for k, m in enumerate(meshes):
        _load(e, m, k + 1)
    _load(e, meshes[CAMERAS[2][3][0]], 0)
    return e


def _camera(textures, H, W, K, seen, seed):
    """A frame of camera (H, W, K) showing objects `seen`, each one's mask and a start pose near its pose."""
    from foundationpose_b200 import synth

    K = np.asarray(K, dtype=np.float64)
    rng = np.random.default_rng(seed)
    placed, start = [], []
    for j, k in enumerate(seen):
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(20 + 7 * seed + k)
        z = 0.65 + 0.05 * j
        p[:3, 3] = [((W * (j + 1) / (len(seen) + 1)) - K[0, 2]) * z / K[0, 0], 0.02 * (-1) ** j, z]
        placed.append((textures[k][0], p, textures[k][1]))
        q = p.copy()
        q[:3, 3] += rng.normal(0, 0.004, 3)
        start.append(q.astype(np.float32))
    rgb, depth, owner = synth.make_multi_scene(placed, K, H, W, seed=seed)
    masks = [owner == j for j in range(len(seen))]
    assert all(m.sum() >= 4 for m in masks)
    return dict(rgb=rgb, depth=depth, K=K, seen=list(seen), masks=masks, start=np.stack(start))


@pytest.fixture(scope="module")
def scene():
    from foundationpose_b200 import hypotheses, synth

    meshes, textures = [], []
    for sub, seed, scale in SPECS:
        m = synth.make_mesh(sub, tex_seed=seed, tex_size=256, scale=scale)
        meshes.append(m)
        textures.append((m.visual.image, scale))
    cams = [_camera(textures, H, W, K, seen, seed=5 + c) for c, (H, W, K, seen) in enumerate(CAMERAS)]
    grid = torch.from_numpy(hypotheses.make_rotation_grid(40, 60, None)).cuda()
    return dict(meshes=meshes, cams=cams, grid=grid)


def _calls(scene):
    """Every call of a round by name: each one's arguments as an engine method and its inputs."""
    cams, grid = scene["cams"], scene["grid"]
    pairs = [(c, j) for c in range(3) for j in range(len(cams[c]["seen"]))]
    frames = [(cam["rgb"], cam["depth"], cam["K"]) for cam in cams]
    start = torch.from_numpy(np.stack([cams[c]["start"][j] for c, j in pairs])).cuda()
    cam_of = [c for c, _ in pairs]
    slots = [cams[c]["seen"][j] + 1 for c, j in pairs]
    reg = [(c, j) for c, j in pairs if c < 2]  # register_cameras on cameras 0 and 1
    a, b = cams[0], cams[1]
    return {
        "track_cameras": lambda e: e.track_cameras(frames, start, cam_of, slots, 2)[1],
        "register_cameras": lambda e: e.register_cameras(frames[:2], [cams[c]["masks"][j] for c, j in reg],
                                                         [grid[:24 - 4 * i] for i in range(len(reg))], [c for c, _ in reg],
                                                         [cams[c]["seen"][j] + 1 for c, j in reg], 2),
        "register_objects": lambda e: e.register_objects(b["rgb"], b["depth"], b["K"], np.stack(b["masks"]), [grid[:28]],
                                                         [k + 1 for k in b["seen"]], 2),
        "track_objects": lambda e: e.track_objects(a["rgb"], a["depth"], a["K"], torch.from_numpy(a["start"]).cuda(),
                                                   [k + 1 for k in a["seen"]], 2)[1],
        "track": lambda e: e.track(cams[2]["rgb"], cams[2]["depth"], cams[2]["K"], torch.from_numpy(cams[2]["start"][0]).cuda(),
                                   2)[1],
    }


# one round: track_objects on camera 0 after every multi-object call, then track on a third frame
ROUND = ["track_cameras", "track_objects", "register_cameras", "track_objects", "register_objects", "track_objects", "track"]


def _host(out):
    return [t.cpu() for t in out] if isinstance(out, tuple) else torch.from_numpy(out)


def _equal(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b)) if isinstance(a, list) else torch.equal(a, b)


def test_interleaved_paths_equal_each_call_alone(scene):
    calls = _calls(scene)
    e = _engine(scene["meshes"])
    for _ in range(3):  # first sight of every graph runs eagerly, the second captures
        warm = [_host(calls[name](e)) for name in ROUND]
    captures = e.graph_captures()
    again = [_host(calls[name](e)) for name in ROUND]
    assert e.graph_captures() == captures, "a warm round captured a graph"
    for name, a, b in zip(ROUND, warm, again):
        assert _equal(a, b), f"{name}: a repeated round differs"
    # each call on a context of its own
    alone = {}
    for name, call in calls.items():
        fresh = _engine(scene["meshes"])
        alone[name] = _host(call(fresh))
        fresh.close()
    for i, (name, got) in enumerate(zip(ROUND, again)):
        assert _equal(got, alone[name]), f"call {i} ({name}) differs from the same call on a fresh context"
    # a register pass larger than any before grows the argument block between two track_cameras replays
    first = _host(calls["track_cameras"](e))
    cams = scene["cams"]
    reg = [(0, 0), (0, 1), (1, 0)]
    e.register_cameras([(c["rgb"], c["depth"], c["K"]) for c in cams[:2]], [cams[c]["masks"][j] for c, j in reg],
                       [scene["grid"][:120]] * 3, [c for c, _ in reg], [cams[c]["seen"][j] + 1 for c, j in reg], 2)
    second = _host(calls["track_cameras"](e))
    assert _equal(first, second), "track_cameras after a larger register pass differs"
    assert _equal(_host(calls["track_objects"](e)), alone["track_objects"]), "track_objects after the larger pass differs"
    e.close()
