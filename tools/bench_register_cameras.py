"""Objects of several cameras registered in one call: `estimater.register_cameras` against one shared engine calling
`register_objects` once per camera (the path that existed before it).

    python tools/bench_register_cameras.py [n_calls]

Workloads: C = 1, 2, 4, 8 cameras at 640x480 with one and two objects per camera, each with full 252-pose grids and with
symmetry-reduced grids (object k of a camera's pair takes 20 / 63 / 126 poses in turn).  Each camera has its own frame
and slightly different intrinsics.  After a warm-up the two paths alternate call by call, so they see the same clocks.
Prints one JSON line: p50 / p99 wall-clock ms per call of each path, with the name and power limit of the GPU they were
measured on."""
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

REDUCED = ("cont_z", "box", "half_z")  # 20 / 63 / 126 hypotheses


def register_cameras_leg(n_calls=10, c_values=(1, 2, 4, 8), per_camera=(1, 2), warmup=2):
    from make_golden_register_objects import symmetry_tfs

    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.estimater import FoundationPose, PoseRefinePredictor, ScorePredictor, register_cameras, register_objects
    from foundationpose_b200.weights import random_state_dict

    sd_r, sd_s = random_state_dict("refine", 0), random_state_dict("score", 0)
    n_cam, n_per = max(c_values), max(per_camera)
    meshes = [(synth.make_mesh(3, tex_seed=k, tex_size=256, scale=0.7 + 0.1 * (k % 4)), 0.7 + 0.1 * (k % 4)) for k in range(n_cam * n_per)]
    cams = []
    for c in range(n_cam):  # camera c sees objects n_per * c ..., side by side
        K = synth.DEFAULT_K.copy()
        K[0, 2] += 2.0 * c
        K[1, 1] *= 1.0 + 0.005 * c
        placed = []
        for j in range(n_per):
            m, sc = meshes[n_per * c + j]
            p = np.eye(4)
            p[:3, :3] = synth.random_rotation(60 + 7 * c + j)
            p[:3, 3] = [-0.08 + 0.16 * j, 0.01 * (c % 3), 0.7]
            placed.append((m.visual.image, p, sc))
        rgb, depth, owner = synth.make_multi_scene(placed, K, 480, 640, seed=1 + c)
        masks = [owner == j for j in range(n_per)]
        assert all(m.any() for m in masks)
        cams.append((rgb, depth, K, masks))

    def estimators(grids):
        e = Engine()
        refiner = PoseRefinePredictor(engine=e, state_dict=sd_r)
        scorer = ScorePredictor(engine=e, state_dict=sd_s)
        out = []
        for k, (m, _) in enumerate(meshes):
            sym = None if grids == "full" else REDUCED[k % len(REDUCED)]
            out.append(FoundationPose(model_pts=m.vertices, model_normals=m.vertex_normals, mesh=m, scorer=scorer, refiner=refiner,
                                      symmetry_tfs=None if sym is None else symmetry_tfs(sym)))
        return out, e

    pct = lambda a, q: float(a[min(int(len(a) * q), len(a) - 1)])
    stats = lambda a: {"ms_p50": pct(np.sort(a), 0.5), "ms_p99": pct(np.sort(a), 0.99)}
    result = {}
    for grids in ("full", "reduced"):
        multi, e_multi = estimators(grids)
        single, e_single = estimators(grids)
        for P in per_camera:
            for C in c_values:
                views = lambda ests: [(ests[n_per * c:n_per * c + P], cams[c][0], cams[c][1], cams[c][2], cams[c][3][:P]) for c in range(C)]
                paths = {"register_cameras": lambda: register_cameras(views(multi)),
                         "register_objects_per_camera": lambda: [register_objects(ests, K, rgb, depth, masks)
                                                                 for ests, rgb, depth, K, masks in views(single)]}
                times = {name: [] for name in paths}
                for i in range(warmup + n_calls):
                    for name, run in paths.items():
                        t0 = time.perf_counter()
                        run()
                        torch.cuda.synchronize()
                        if i >= warmup:
                            times[name].append((time.perf_counter() - t0) * 1e3)
                r = {name: stats(t) for name, t in times.items()}
                r["hypotheses"] = sum(len(est.rot_grid) for ests, *_ in views(multi) for est in ests)
                r["speedup_p50"] = r["register_objects_per_camera"]["ms_p50"] / r["register_cameras"]["ms_p50"]
                result[f"{grids}/{P}_per_camera/C={C}"] = r
        e_multi.close()
        e_single.close()
        torch.cuda.empty_cache()
    return {"register_cameras": result, "calls": n_calls, "warmup_calls": warmup, "iterations": 5,
            "api": "estimater.register_cameras(views) against register_objects(...) per view on one shared engine, host numpy "
                   "frames; wall clock per call",
            "workloads": "full: 252-pose grids; reduced: the objects' grids reduced by symmetry to 20 / 63 / 126 poses in turn",
            "scene": "C cameras at 640x480, each with its own frame and intrinsics, showing 1 or 2 textured ellipsoids (icosphere-3)"}


def main():
    from bench import device_info

    n_calls = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    out = register_cameras_leg(n_calls)
    out["device"] = device_info(torch.cuda.current_device())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
