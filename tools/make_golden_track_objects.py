"""Generate tests/golden/track_objects.npz: the CPU oracle over track_one (estimater.py:250-268) applied to each of three
objects of the same frames (one erode + bilateral filtered depth, depth2xyzmap(zfar=inf), then per object ONE pose
through `iteration` = 2 refiner passes with its own mesh and diameter), on a 10-frame synthetic sequence drawn by
foundationpose_b200.synth.make_multi_scene.

The objects differ in subdivisions, texture, scale (so their diameters differ) and colour source (object 1 is
vertex-coloured), and objects 0 and 1 partly overlap in the image (1 is in front).  As in tools/make_golden_track.py the
stand-in weights are random-init and do not converge, so every frame is anchored: each object is tracked from its
previous ground-truth pose plus a small seeded perturbation.

    python tools/make_golden_track_objects.py
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_FRAMES = 11  # 10 tracked frames
K_ITERS = 2
# per object: subdivisions, texture seed, scale, vertex-coloured, start translation
SUBDIVISIONS = np.array([3, 2, 4])
TEX_SEEDS = np.array([0, 5, 9])
SCALES = np.array([1.0, 0.7, 1.3])
VERTEX_COLOURED = np.array([False, True, False])
START_T = np.array([[-0.05, 0.0, 0.6], [0.0, 0.02, 0.5], [0.0, -0.13, 0.8]])
TEX_SIZE = 256


def main():
    from foundationpose_b200 import synth
    from foundationpose_b200.weights import random_state_dict
    from oracle import geometry, pipeline

    torch.set_num_threads(os.cpu_count())
    K = synth.DEFAULT_K
    sd_r = random_state_dict("refine", 0)
    meshes, gts = [], []
    for k in range(len(SCALES)):
        m = synth.make_mesh(int(SUBDIVISIONS[k]), tex_seed=int(TEX_SEEDS[k]), tex_size=TEX_SIZE, scale=float(SCALES[k]))
        meshes.append(m)
        pose0 = np.eye(4)
        pose0[:3, :3] = synth.random_rotation(10 + k)
        pose0[:3, 3] = START_T[k]
        gts.append(synth.track_sequence(N_FRAMES, pose0, seed=20 + k))
    gt = np.stack(gts)  # [object][frame][4][4]
    mts = [pipeline.mesh_tensors(synth.vertex_coloured(m) if VERTEX_COLOURED[k] else m) for k, m in enumerate(meshes)]
    diam = [synth.mesh_diameter(m.vertices) for m in meshes]
    rng = np.random.default_rng(13)
    pose_in, pose_out = [], []
    t0 = time.time()
    for i in range(1, N_FRAMES):
        rgb, depth, owner = synth.make_multi_scene([(m.visual.image, gt[k, i], float(SCALES[k])) for k, m in enumerate(meshes)], seed=1 + i)
        if i == 1:
            alone = [synth.make_multi_scene([(m.visual.image, gt[k, i], float(SCALES[k]))])[2] == 0 for k, m in enumerate(meshes)]
            assert all((owner == k).any() for k in range(len(meshes))), "every object must be visible"
            assert (alone[0] & alone[1]).any() and (alone[0] & (owner == 1)).any(), "object 1 must partly cover object 0"
        depth_f = geometry.bilateral_filter_depth(geometry.erode_depth(depth))
        xyz_map = geometry.depth2xyzmap(depth_f, K, zfar=np.inf)
        pin, pout = [], []
        for k in range(len(meshes)):
            p = gt[k, i - 1].copy()
            ax = rng.normal(size=3)
            ax /= np.linalg.norm(ax)
            ang = np.deg2rad(1.0)
            Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
            p[:3, :3] = (np.eye(3) + np.sin(ang) * Kx + (1 - np.cos(ang)) * (Kx @ Kx)) @ p[:3, :3]
            p[:3, 3] += rng.normal(0, 0.003, 3)
            p = p.astype(np.float32)
            out, _, _ = pipeline.refine(sd_r, p[None], mts[k], rgb, depth_f, K, diam[k], K_ITERS, xyz_map=xyz_map)
            pin.append(p)
            pout.append(out[0].numpy())
        pose_in.append(np.stack(pin))
        pose_out.append(np.stack(pout))
        print(f"frame {i}: {time.time() - t0:.0f} s", flush=True)
    path = os.path.join(ROOT, "tests", "golden", "track_objects.npz")
    np.savez_compressed(path, gt=gt, pose_in=np.stack(pose_in), pose_out=np.stack(pose_out), subdivisions=SUBDIVISIONS,
                        tex_seeds=TEX_SEEDS, scales=SCALES, vertex_coloured=VERTEX_COLOURED, tex_size=TEX_SIZE,
                        diameters=np.array(diam))
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
