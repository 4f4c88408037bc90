"""Several objects registered in one frame: `estimater.register_objects` (one call for all M objects) against the path
that existed before it, M estimators calling `register` in turn.

    python tools/bench_register_objects.py [n_frames]

The per-object baseline runs twice: with every estimator on one shared engine (what a user writes today; each register
re-uploads its mesh into slot 0) and, for M <= 4, with one engine per estimator.  Workloads: M = 1, 2, 4, 8 objects with
full 252-pose grids, and with a symmetric mix whose grids hold 20 / 63 / 126 / 252 poses (object k takes the k % 4-th).
After a warm-up the paths alternate frame by frame, so they see the same clocks.  Prints one JSON line: p50 / p99
wall-clock ms per frame of each path, with the name and power limit of the GPU they were measured on."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.dont_write_bytecode = True

MIX = ("cont_z", "box", "half_z", None)  # 20 / 63 / 126 / 252 hypotheses


def register_objects_leg(n_frames=30, m_values=(1, 2, 4, 8), warmup=3):
    from make_golden_register_objects import symmetry_tfs

    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.estimater import FoundationPose, PoseRefinePredictor, ScorePredictor, register_objects
    from foundationpose_b200.weights import random_state_dict

    K = synth.DEFAULT_K
    sd_r, sd_s = random_state_dict("refine", 0), random_state_dict("score", 0)
    n_obj = max(m_values)
    meshes, poses = [], []
    for k in range(n_obj):  # a 4 x 2 grid of ellipsoids of four sizes
        scale = 0.6 + 0.1 * (k % 4)
        meshes.append((synth.make_mesh(3, tex_seed=k, tex_size=256, scale=scale), scale))
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(40 + k)
        p[:3, 3] = [-0.21 + 0.14 * (k % 4), -0.08 + 0.16 * (k // 4 % 2), 0.75]
        poses.append(p)
    rgb, depth, owner = synth.make_multi_scene([(m.visual.image, p, sc) for (m, sc), p in zip(meshes, poses)], seed=1)
    masks = [owner == k for k in range(n_obj)]
    assert all(m.any() for m in masks)

    def estimators(grids, shared, n=n_obj):
        out, engines = [], []
        for k, (m, _) in enumerate(meshes[:n]):
            if shared is None or not engines:
                engines.append(shared or Engine())
                refiner = PoseRefinePredictor(engine=engines[-1], state_dict=sd_r)
                scorer = ScorePredictor(engine=engines[-1], state_dict=sd_s)
            sym = None if grids == "full" else MIX[k % 4]
            out.append(FoundationPose(model_pts=m.vertices, model_normals=m.vertex_normals, mesh=m, scorer=scorer, refiner=refiner,
                                      symmetry_tfs=None if sym is None else symmetry_tfs(sym)))
        return out, engines

    pct = lambda a, q: float(a[min(int(len(a) * q), len(a) - 1)])
    stats = lambda a: {"ms_p50": pct(np.sort(a), 0.5), "ms_p99": pct(np.sort(a), 0.99)}
    result = {}
    for grids in ("full", "mix"):
        multi, e_multi = estimators(grids, Engine())
        shared, e_shared = estimators(grids, Engine())
        own, e_own = estimators(grids, None, n=4)
        per_m = {}
        for M in m_values:
            paths = {"register_objects": lambda: register_objects(multi[:M], K, rgb, depth, masks[:M]),
                     "register_shared_engine": lambda: [est.register(K=K, rgb=rgb, depth=depth, ob_mask=masks[k])
                                                        for k, est in enumerate(shared[:M])]}
            if M <= 4:
                paths["register_own_engines"] = lambda: [est.register(K=K, rgb=rgb, depth=depth, ob_mask=masks[k])
                                                         for k, est in enumerate(own[:M])]
            times = {name: [] for name in paths}
            for i in range(warmup + n_frames):
                for name, run in paths.items():
                    t0 = time.perf_counter()
                    run()
                    torch.cuda.synchronize()
                    if i >= warmup:
                        times[name].append((time.perf_counter() - t0) * 1e3)
            per_m[str(M)] = {name: stats(t) for name, t in times.items()}
            per_m[str(M)]["hypotheses"] = sum(len(est.rot_grid) for est in multi[:M])
            per_m[str(M)]["speedup_p50_vs_shared"] = per_m[str(M)]["register_shared_engine"]["ms_p50"] / per_m[str(M)]["register_objects"]["ms_p50"]
        result[grids] = per_m
        for e in e_multi + e_shared + e_own:
            e.close()
        torch.cuda.empty_cache()
    return {"per_objects": result, "frames": n_frames, "warmup_frames": warmup, "iterations": 5,
            "api": "estimater.register_objects(estimators, K, rgb, depth, masks) with host numpy frames; wall clock per frame",
            "baselines": "register_shared_engine: the estimators share one Engine and call register in turn (each call uploads its "
                         "mesh to slot 0); register_own_engines (M <= 4): one Engine per estimator",
            "workloads": "full: every object with the 252-pose grid; mix: object k's grid reduced by symmetry to 20 / 63 / 126 / 252 "
                         "poses for k % 4 = 0..3",
            "scene": "8 textured ellipsoids (icosphere-3, four sizes) in one 640x480 frame; the first M objects are registered"}


def main():
    from bench import device_info

    n_frames = int(sys.argv[1]) if len(sys.argv) > 1 else 30
    out = register_objects_leg(n_frames)
    out["device"] = device_info(torch.cuda.current_device())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
