"""Generate tests/golden/register_objects.npz: the CPU oracle's FoundationPose.register (oracle.pipeline.register,
estimater.py:159-240) applied to each of three objects of ONE frame drawn by foundationpose_b200.synth.make_multi_scene,
every object with its own mask (from the scene's owner map), mesh, diameter and symmetry-reduced rotation grid.

The objects differ in texture, scale (so their diameters differ) and colour source (object 1 is vertex-coloured), and
objects 0 and 1 partly overlap in the image (1 is in front).  Their symmetries reduce the 252-pose grid to 126 (a
half-turn about z), 63 (the box group) and 20 (continuous about z) hypotheses, which keeps the generator to minutes.
Recorded per object: the start poses, the refined poses and scores in grid order, the ranking ids, the top-2 margin and
the score spread.

SEED picks the object rotations and the depth noise.  With the seeded stand-in scorer (weights.random_state_dict) the
selected index is only a meaningful check where the oracle's top-2 margin is a sizeable fraction of the score spread;
SEED = 3 gives the three objects margins of 0.30, 0.25 and 0.70 spreads (the generator refuses a seed below
MIN_MARGIN_SPREAD).

    python tools/make_golden_register_objects.py
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEED = 3
ITERATIONS = 5
MIN_MARGIN_SPREAD = 0.2
TEX_SIZE = 256
# per object: subdivisions, texture seed, scale, vertex-coloured, translation, symmetry group
SUBDIVISIONS = np.array([3, 2, 3])
TEX_SEEDS = np.array([0, 5, 9])
SCALES = np.array([1.0, 0.7, 1.3])
VERTEX_COLOURED = np.array([False, True, False])
TRANSLATIONS = np.array([[-0.05, 0.0, 0.6], [0.0, 0.02, 0.5], [0.02, -0.13, 0.8]])
SYMMETRIES = ("half_z", "box", "cont_z")


def _euler(rx, ry, rz):
    from scipy.spatial.transform import Rotation

    m = np.eye(4)
    m[:3, :3] = Rotation.from_euler("xyz", [rx, ry, rz]).as_matrix()
    return m


def symmetry_tfs(name):
    """The symmetry groups of tools/make_golden_cluster.py, as (S,4,4) float32."""
    if name == "half_z":
        tfs = np.stack([np.eye(4), np.diag([-1.0, -1.0, 1.0, 1.0])])
    elif name == "box":
        tfs = np.stack([_euler(rx, ry, rz) for rz in (0, np.pi) for rx in (0, np.pi) for ry in (0, np.pi)])
    elif name == "cont_z":
        tfs = np.stack([_euler(0, 0, a) for a in np.arange(0, 360, 5) / 180 * np.pi])
    else:
        raise ValueError(name)
    return tfs.astype(np.float32)


def scene(seed=SEED):
    """(meshes, poses, rgb, depth, owner) of the golden frame; shared with tests/test_register_objects_gpu.py."""
    from foundationpose_b200 import synth

    meshes, poses = [], []
    for k in range(len(SCALES)):
        meshes.append(synth.make_mesh(int(SUBDIVISIONS[k]), tex_seed=int(TEX_SEEDS[k]), tex_size=TEX_SIZE, scale=float(SCALES[k])))
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(10 * seed + k)
        p[:3, 3] = TRANSLATIONS[k]
        poses.append(p)
    rgb, depth, owner = synth.make_multi_scene([(m.visual.image, p, float(sc)) for m, p, sc in zip(meshes, poses, SCALES)], seed=seed)
    return meshes, poses, rgb, depth, owner


def main():
    from foundationpose_b200 import hypotheses, synth
    from foundationpose_b200.weights import random_state_dict
    from oracle import pipeline

    torch.set_num_threads(os.cpu_count())
    K = synth.DEFAULT_K
    sd_r, sd_s = random_state_dict("refine", 0), random_state_dict("score", 0)
    meshes, poses, rgb, depth, owner = scene()
    alone = [synth.make_multi_scene([(m.visual.image, p, float(sc))])[2] == 0 for m, p, sc in zip(meshes, poses, SCALES)]
    assert all((owner == k).any() for k in range(len(meshes))), "every object must be visible"
    assert (alone[0] & alone[1]).any() and (alone[0] & (owner == 1)).any(), "object 1 must partly cover object 0"
    out = {k: [] for k in ("start", "refined", "scores", "ids", "top2_margin", "spread", "centers", "diameters", "model_centers")}
    t0 = time.time()
    for k, m in enumerate(meshes):
        # FoundationPose.reset_object: the mesh is centred on its bounding box; the diameter is the centred mesh's
        mc = (m.vertices.max(axis=0) + m.vertices.min(axis=0)) / 2
        mesh = synth.vertex_coloured(m) if VERTEX_COLOURED[k] else m.copy()
        mesh.vertices = mesh.vertices - mc.reshape(1, 3)
        d = synth.mesh_diameter(mesh.vertices)
        grid = hypotheses.make_rotation_grid(40, 60, symmetry_tfs(SYMMETRIES[k]))
        mask = owner == k
        r = pipeline.register(sd_r, sd_s, grid, pipeline.mesh_tensors(mesh), rgb, depth, mask, K, d, mc, iterations=ITERATIONS)
        assert not r["early"]
        ids = r["ids"].numpy()
        refined = np.empty((len(grid), 4, 4), np.float32)
        refined[ids] = r["poses"].numpy()
        scores = np.empty(len(grid), np.float32)
        scores[ids] = r["scores"].numpy()
        # the start poses: the rotation grid with guess_translation of the filtered depth (estimater.py:203-209)
        from oracle import geometry

        center = geometry.guess_translation(geometry.bilateral_filter_depth(geometry.erode_depth(depth)), mask, K)
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
        print(f"object {k}: {len(grid)} hypotheses, best {ids[0]}, top-2 margin {ss[-1] - ss[-2]:.4f} = "
              f"{(ss[-1] - ss[-2]) / scores.std():.2f} spreads ({time.time() - t0:.0f} s)", flush=True)
    margins = np.array(out["top2_margin"]) / np.array(out["spread"])
    assert (margins >= MIN_MARGIN_SPREAD).all(), f"SEED {SEED}: top-2 margins {margins} spreads; pick another seed"
    n_hyp = np.array([len(s) for s in out["start"]])
    cat = lambda k: np.concatenate(out[k])
    path = os.path.join(ROOT, "tests", "golden", "register_objects.npz")
    np.savez_compressed(path, seed=SEED, iterations=ITERATIONS, n_hyp=n_hyp, start=cat("start"), refined=cat("refined"),
                        scores=cat("scores"), ids=cat("ids"), top2_margin=np.array(out["top2_margin"]), spread=np.array(out["spread"]),
                        centers=np.stack(out["centers"]), diameters=np.array(out["diameters"]), model_centers=np.stack(out["model_centers"]),
                        symmetries=np.array(SYMMETRIES), symmetry_tfs=np.concatenate([symmetry_tfs(s) for s in SYMMETRIES]),
                        symmetry_counts=np.array([len(symmetry_tfs(s)) for s in SYMMETRIES]), subdivisions=SUBDIVISIONS,
                        tex_seeds=TEX_SEEDS, scales=SCALES, vertex_coloured=VERTEX_COLOURED, translations=TRANSLATIONS, tex_size=TEX_SIZE)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
