"""Generate tests/golden/track_cameras.npz: the CPU oracle over track_one (estimater.py:250-268) applied to every (object,
camera) pair of a two-camera rig: per camera one erode + bilateral filtered depth and depth2xyzmap(zfar=inf) of that
camera's frame, then per pair ONE pose through `iteration` = 2 refiner passes with the object's mesh and the camera's
intrinsics, on a 5-frame synthetic sequence drawn by foundationpose_b200.synth.make_multi_scene.

Camera 0 is 640x480 with synth.DEFAULT_K; camera 1 is 1280x720 with other intrinsics, 0.3 m to the side and turned by
10 degrees (extrinsic() maps camera 0 coordinates to camera 1's).  Each camera sees its own background plane.  Objects 0
and 2 are seen by both cameras, object 1 by camera 0 only.  The objects differ in subdivisions, texture, scale and colour
source (object 1 is vertex-coloured).  As in tools/make_golden_track_objects.py the stand-in weights are random-init and
do not converge, so every frame is anchored: each pair is tracked from its previous ground-truth pose plus a small
seeded perturbation.

    python tools/make_golden_track_cameras.py
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_FRAMES = 6  # 5 tracked frames
K_ITERS = 2
# per object: subdivisions, texture seed, scale, vertex-coloured, start translation (camera 0)
SUBDIVISIONS = np.array([3, 2, 3])
TEX_SEEDS = np.array([0, 5, 9])
SCALES = np.array([1.0, 0.8, 1.2])
VERTEX_COLOURED = np.array([False, True, False])
START_T = np.array([[0.12, 0.0, 0.62], [-0.2, 0.04, 0.55], [0.0, -0.12, 0.8]])
TEX_SIZE = 256
# per camera: intrinsics and frame size
KS = np.array([[[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1.0]], [[920.0, 0, 640.0], [0, 915.0, 360.0], [0, 0, 1.0]]])
HS = np.array([480, 720])
WS = np.array([640, 1280])
# (camera, object) pairs, camera-major
PAIRS = np.array([[0, 0], [0, 1], [0, 2], [1, 0], [1, 2]])


def extrinsic():
    """Camera 0 -> camera 1 coordinates."""
    a = np.deg2rad(-10.0)
    T = np.eye(4)
    T[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    T[:3, 3] = [-0.3, 0.02, 0.05]
    return T


def gt_in_camera(gt, cam, T):
    """[object][frame] poses in camera 0 -> in camera `cam`."""
    return gt if cam == 0 else np.stack([[T @ p for p in seq] for seq in gt])


def main():
    from foundationpose_b200 import synth
    from foundationpose_b200.weights import random_state_dict
    from oracle import geometry, pipeline

    torch.set_num_threads(os.cpu_count())
    sd_r = random_state_dict("refine", 0)
    T = extrinsic()
    meshes, gts = [], []
    for k in range(len(SCALES)):
        m = synth.make_mesh(int(SUBDIVISIONS[k]), tex_seed=int(TEX_SEEDS[k]), tex_size=TEX_SIZE, scale=float(SCALES[k]))
        meshes.append(m)
        pose0 = np.eye(4)
        pose0[:3, :3] = synth.random_rotation(10 + k)
        pose0[:3, 3] = START_T[k]
        gts.append(synth.track_sequence(N_FRAMES, pose0, seed=20 + k))
    gt = np.stack(gts)  # [object][frame][4][4], camera 0
    gt_cam = [gt_in_camera(gt, c, T) for c in range(len(KS))]
    mts = [pipeline.mesh_tensors(synth.vertex_coloured(m) if VERTEX_COLOURED[k] else m) for k, m in enumerate(meshes)]
    diam = [synth.mesh_diameter(m.vertices) for m in meshes]
    rng = np.random.default_rng(17)
    pose_in, pose_out = [], []
    t0 = time.time()
    for i in range(1, N_FRAMES):
        frames = []
        for c in range(len(KS)):
            objs = [(m.visual.image, gt_cam[c][k, i], float(SCALES[k])) for k, m in enumerate(meshes)]
            rgb, depth, owner = synth.make_multi_scene(objs, KS[c], int(HS[c]), int(WS[c]), seed=1 + i + 100 * c)
            for k in range(len(meshes)):
                seen = bool((owner == k).any())
                assert seen == any((PAIRS == [c, k]).all(1)), f"frame {i}: object {k} {'is' if seen else 'is not'} seen by camera {c}"
            depth_f = geometry.bilateral_filter_depth(geometry.erode_depth(depth))
            frames.append((rgb, depth_f, geometry.depth2xyzmap(depth_f, KS[c], zfar=np.inf)))
        pin, pout = [], []
        for c, k in PAIRS:
            p = gt_cam[c][k, i - 1].copy()
            ax = rng.normal(size=3)
            ax /= np.linalg.norm(ax)
            ang = np.deg2rad(1.0)
            Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
            p[:3, :3] = (np.eye(3) + np.sin(ang) * Kx + (1 - np.cos(ang)) * (Kx @ Kx)) @ p[:3, :3]
            p[:3, 3] += rng.normal(0, 0.003, 3)
            p = p.astype(np.float32)
            rgb, depth_f, xyz_map = frames[c]
            out, _, _ = pipeline.refine(sd_r, p[None], mts[k], rgb, depth_f, KS[c], diam[k], K_ITERS, xyz_map=xyz_map)
            pin.append(p)
            pout.append(out[0].numpy())
        pose_in.append(np.stack(pin))
        pose_out.append(np.stack(pout))
        print(f"frame {i}: {time.time() - t0:.0f} s", flush=True)
    path = os.path.join(ROOT, "tests", "golden", "track_cameras.npz")
    np.savez_compressed(path, gt=gt, extrinsic=T, K=KS, H=HS, W=WS, pairs=PAIRS, pose_in=np.stack(pose_in),
                        pose_out=np.stack(pose_out), subdivisions=SUBDIVISIONS, tex_seeds=TEX_SEEDS, scales=SCALES,
                        vertex_coloured=VERTEX_COLOURED, tex_size=TEX_SIZE, diameters=np.array(diam))
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
