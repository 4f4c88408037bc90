"""Several objects tracked in one camera stream: `estimater.track_objects` (one CUDA-graph launch per frame for all M
objects) against the best path that existed before it, M estimators each with its own Engine calling `track_one` in turn.

    python tools/bench_track_objects.py [n_frames]

Prints one JSON line: p50 / p99 wall-clock ms per frame of both paths for M = 1, 2, 4, 8 (host numpy frames, two
refiner passes), with the name and power limit of the GPU they were measured on."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True


def track_objects_leg(n_frames=400, m_values=(1, 2, 4, 8)):
    """M objects tracked in one camera stream: estimater.track_objects (one graph launch per frame for all M) against the
    best existing path, M estimators each with its own Engine calling track_one in turn.  Both paths compute the same
    poses, run on the same frames and alternate frame by frame, so they see the same clocks.  Wall clock per frame."""
    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.estimater import FoundationPose, PoseRefinePredictor, ScorePredictor, track_objects
    from foundationpose_b200.weights import random_state_dict

    K = synth.DEFAULT_K
    sd_r, sd_s = random_state_dict("refine", 0), random_state_dict("score", 0)
    n_obj = max(m_values)
    meshes, seqs = [], []
    for k in range(n_obj):  # a 4 x 2 grid of ellipsoids of four sizes, each on its own random walk
        scale = 0.6 + 0.1 * (k % 4)
        meshes.append((synth.make_mesh(3, tex_seed=k, tex_size=256, scale=scale), scale))
        p0 = np.eye(4)
        p0[:3, :3] = synth.random_rotation(40 + k)
        p0[:3, 3] = [-0.21 + 0.14 * (k % 4), -0.08 + 0.16 * (k // 4 % 2), 0.75]
        seqs.append(synth.track_sequence(20, p0, seed=50 + k))
    frames = [synth.make_multi_scene([(m.visual.image, seqs[k][i], sc) for k, (m, sc) in enumerate(meshes)], seed=1 + i)[:2]
              for i in range(20)]

    def estimators(shared):
        out, engines = [], []
        for k, (m, _) in enumerate(meshes):
            if shared is None or not engines:
                engines.append(shared or Engine())
                refiner = PoseRefinePredictor(engine=engines[-1], state_dict=sd_r)
                scorer = ScorePredictor(engine=engines[-1], state_dict=sd_s)
            out.append(FoundationPose(model_pts=m.vertices, model_normals=m.vertex_normals, mesh=m, scorer=scorer, refiner=refiner))
        return out, engines

    multi, multi_engines = estimators(Engine())
    alone, alone_engines = estimators(None)
    pct = lambda a, q: float(a[min(int(len(a) * q), len(a) - 1)])
    per_m = {}
    for M in m_values:
        for k in range(M):
            for est in (multi[k], alone[k]):
                est.pose_last = torch.as_tensor(seqs[k][0], dtype=torch.float32, device="cuda").reshape(1, 4, 4)
        t_multi, t_alone = [], []
        for i in range(20 + n_frames):
            k40 = i % 40
            f_rgb, f_depth = frames[k40 if k40 < 20 else 39 - k40]  # forwards, then backwards: no jumps
            t0 = time.perf_counter()
            track_objects(multi[:M], f_rgb, f_depth, K, iteration=2)
            t1 = time.perf_counter()
            for est in alone[:M]:
                est.track_one(rgb=f_rgb, depth=f_depth, K=K, iteration=2)
            t2 = time.perf_counter()
            if i >= 20:  # the first 20 frames warm up both paths (graphs captured)
                t_multi.append((t1 - t0) * 1e3)
                t_alone.append((t2 - t1) * 1e3)
        t_multi, t_alone = np.sort(t_multi), np.sort(t_alone)
        per_m[str(M)] = {"track_objects": {"ms_p50": pct(t_multi, 0.5), "ms_p99": pct(t_multi, 0.99)},
                         "per_object_engines": {"ms_p50": pct(t_alone, 0.5), "ms_p99": pct(t_alone, 0.99)},
                         "speedup_p50": pct(t_alone, 0.5) / pct(t_multi, 0.5)}
    for e in multi_engines + alone_engines:
        e.close()
    return {"per_objects": per_m, "frames": n_frames, "refine_iters": 2,
            "api": "estimater.track_objects(estimators, rgb, depth, K, iteration=2) with host numpy frames: one CUDA-graph launch per "
                   "frame for all M objects (upload, depth filters, xyz map, 2 refiner passes at N = M, read-back); wall clock per frame",
            "baseline": "per_object_engines: M FoundationPose estimators, each with its own Engine, track_one(...) called in turn",
            "sequence": "8 textured ellipsoids (icosphere-3, four sizes) each on its own walk (<= 5 mm / 2 deg per frame); 20 distinct "
                        "640x480 frames played forwards and backwards; the first M objects are tracked"}


def main():
    from bench import device_info

    n_frames = int(sys.argv[1]) if len(sys.argv) > 1 else 400
    out = track_objects_leg(n_frames)
    out["device"] = device_info(torch.cuda.current_device())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
