"""Generate tests/golden/register_cameras.npz: the CPU oracle's FoundationPose.register (oracle.pipeline.register,
estimater.py:159-240) applied to each of three objects seen by a two-camera rig, each camera with its own frame drawn by
foundationpose_b200.synth.make_multi_scene, its own size and its own intrinsics.

Camera 0 is 640x480 with synth.DEFAULT_K and sees objects 0 and 1, which partly overlap (1 is in front).  Camera 1 is
400x300, a size that is not a multiple of the frame filter's 32 x 8 tile, with other intrinsics, and sees object 2.
Every object has its own mask (from its camera's owner map), mesh, diameter and symmetry-reduced rotation grid: a
half-turn about z (126 hypotheses), continuous about z (20) and the box group (63), which keeps the generator to
minutes.  The objects are those of tools/make_golden_register_objects.py (object 1 is vertex-coloured).  Recorded per
object: its camera, the start poses, the refined poses and scores in grid order, the ranking ids, the top-2 margin and
the score spread.

SEED picks the object rotations and the depth noise.  With the seeded stand-in scorer (weights.random_state_dict) the
selected index is only a meaningful check where the oracle's top-2 margin is a sizeable fraction of the score spread;
the generator refuses a seed where fewer than two objects have a margin of MIN_MARGIN_SPREAD spreads.  Seed 3 (the seed
of tools/make_golden_register_objects.py) gives object 0 only 0.09 spreads here; seed 4 gives objects 0 and 2 margins of
0.74 and 0.25 spreads and object 1 (20 hypotheses) 0.06.  The GPU's score error on the free-running refined poses is
larger than those margins, so tests/test_register_cameras_gpu.py holds the poses to the oracle and the selected index
only where a margin dominates that error.

    python tools/make_golden_register_cameras.py [SEED]
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from make_golden_register_objects import symmetry_tfs  # noqa: E402

SEED = 4
ITERATIONS = 5
MIN_MARGIN_SPREAD = 0.2
TEX_SIZE = 256
# per camera: intrinsics and frame size
KS = np.array([[[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1.0]], [[380.0, 0, 205.0], [0, 375.0, 148.0], [0, 0, 1.0]]])
HS = np.array([480, 300])
WS = np.array([640, 400])
# per object: its camera, subdivisions, texture seed, scale, vertex-coloured, translation in its camera, symmetry group
CAMERA_OF = np.array([0, 0, 1])
SUBDIVISIONS = np.array([3, 2, 3])
TEX_SEEDS = np.array([0, 5, 9])
SCALES = np.array([1.0, 0.7, 1.3])
VERTEX_COLOURED = np.array([False, True, False])
TRANSLATIONS = np.array([[-0.05, 0.0, 0.6], [0.0, 0.02, 0.5], [0.02, -0.03, 0.75]])
SYMMETRIES = ("half_z", "cont_z", "box")


def scene(seed=SEED):
    """(meshes, poses, frames) of the golden rig, frames[c] = (rgb, depth, masks of camera c's objects in object order);
    shared with tests/test_register_cameras_gpu.py."""
    from foundationpose_b200 import synth

    meshes, poses = [], []
    for k in range(len(SCALES)):
        meshes.append(synth.make_mesh(int(SUBDIVISIONS[k]), tex_seed=int(TEX_SEEDS[k]), tex_size=TEX_SIZE, scale=float(SCALES[k])))
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(10 * seed + k)
        p[:3, 3] = TRANSLATIONS[k]
        poses.append(p)
    frames = []
    for c in range(len(KS)):
        seen = [k for k in range(len(meshes)) if CAMERA_OF[k] == c]
        rgb, depth, owner = synth.make_multi_scene([(meshes[k].visual.image, poses[k], float(SCALES[k])) for k in seen], KS[c],
                                                   int(HS[c]), int(WS[c]), seed=seed + 100 * c)
        frames.append((rgb, depth, [owner == j for j in range(len(seen))]))
    return meshes, poses, frames


def masks_of(frames):
    """Every object's mask, in object order."""
    it = [iter(f[2]) for f in frames]
    return [next(it[c]) for c in CAMERA_OF]


def main():
    from foundationpose_b200 import hypotheses, synth
    from foundationpose_b200.weights import random_state_dict
    from oracle import geometry, pipeline

    seed = int(sys.argv[1]) if len(sys.argv) > 1 else SEED
    torch.set_num_threads(os.cpu_count())
    sd_r, sd_s = random_state_dict("refine", 0), random_state_dict("score", 0)
    meshes, poses, frames = scene(seed)
    masks = masks_of(frames)
    assert all(m.any() for m in masks), "every object must be visible"
    alone = synth.make_multi_scene([(meshes[0].visual.image, poses[0], float(SCALES[0]))], KS[0], int(HS[0]), int(WS[0]))[2] == 0
    assert (alone & masks[1]).any(), "object 1 must partly cover object 0"
    out = {k: [] for k in ("start", "refined", "scores", "ids", "top2_margin", "spread", "centers", "diameters", "model_centers")}
    t0 = time.time()
    for k, m in enumerate(meshes):
        c = int(CAMERA_OF[k])
        rgb, depth, _ = frames[c]
        # FoundationPose.reset_object: the mesh is centred on its bounding box; the diameter is the centred mesh's
        mc = (m.vertices.max(axis=0) + m.vertices.min(axis=0)) / 2
        mesh = synth.vertex_coloured(m) if VERTEX_COLOURED[k] else m.copy()
        mesh.vertices = mesh.vertices - mc.reshape(1, 3)
        d = synth.mesh_diameter(mesh.vertices)
        grid = hypotheses.make_rotation_grid(40, 60, symmetry_tfs(SYMMETRIES[k]))
        r = pipeline.register(sd_r, sd_s, grid, pipeline.mesh_tensors(mesh), rgb, depth, masks[k], KS[c], d, mc, iterations=ITERATIONS)
        assert not r["early"]
        ids = r["ids"].numpy()
        refined = np.empty((len(grid), 4, 4), np.float32)
        refined[ids] = r["poses"].numpy()
        scores = np.empty(len(grid), np.float32)
        scores[ids] = r["scores"].numpy()
        # the start poses: the rotation grid with guess_translation of the camera's filtered depth (estimater.py:203-209)
        center = geometry.guess_translation(geometry.bilateral_filter_depth(geometry.erode_depth(depth)), masks[k], KS[c])
        start = grid.copy()
        start[:, :3, 3] = center.astype(np.float32)
        ss = np.sort(scores)
        out["start"].append(start)
        out["refined"].append(refined)
        out["scores"].append(scores)
        out["ids"].append(ids)
        out["top2_margin"].append(float(ss[-1] - ss[-2]))
        out["spread"].append(float(scores.std()))
        out["centers"].append(center)
        out["diameters"].append(d)
        out["model_centers"].append(mc)
        print(f"object {k} (camera {c}): {len(grid)} hypotheses, best {ids[0]}, top-2 margin {ss[-1] - ss[-2]:.4f} = "
              f"{(ss[-1] - ss[-2]) / scores.std():.2f} spreads ({time.time() - t0:.0f} s)", flush=True)
    margins = np.array(out["top2_margin"]) / np.array(out["spread"])
    assert (margins >= MIN_MARGIN_SPREAD).sum() >= 2, f"seed {seed}: top-2 margins {margins} spreads; pick another seed"
    n_hyp = np.array([len(s) for s in out["start"]])
    cat = lambda k: np.concatenate(out[k])
    path = os.path.join(ROOT, "tests", "golden", "register_cameras.npz")
    np.savez_compressed(path, seed=seed, iterations=ITERATIONS, K=KS, H=HS, W=WS, camera_of=CAMERA_OF, n_hyp=n_hyp,
                        start=cat("start"), refined=cat("refined"), scores=cat("scores"), ids=cat("ids"),
                        top2_margin=np.array(out["top2_margin"]), spread=np.array(out["spread"]), centers=np.stack(out["centers"]),
                        diameters=np.array(out["diameters"]), model_centers=np.stack(out["model_centers"]),
                        symmetries=np.array(SYMMETRIES), symmetry_tfs=np.concatenate([symmetry_tfs(s) for s in SYMMETRIES]),
                        symmetry_counts=np.array([len(symmetry_tfs(s)) for s in SYMMETRIES]), subdivisions=SUBDIVISIONS,
                        tex_seeds=TEX_SEEDS, scales=SCALES, vertex_coloured=VERTEX_COLOURED, translations=TRANSLATIONS, tex_size=TEX_SIZE)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
