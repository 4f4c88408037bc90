"""Cost of get_vis at N = 252 on the register scene of bench.py, split into its stages: the two refiner crop passes and
the scorer crop pass (fp_vis_crops), the canvas composition on the device (fp_vis minus its crop passes), the D2H copy,
the labels and the PNG encode; and, for comparison, the host composition of the same crop records
(tests/vis_compose.py, the reference's recipe).  CUDA events for device stages, wall clock for host stages.

    python tools/bench_vis.py [--reps 5]       # prints one JSON line; GPU model and power limit included
"""
import argparse
import json
import os
import subprocess
import sys
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def dev_ms(fn, reps):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def wall_ms(fn, reps):
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import vis_compose
    from foundationpose_b200 import hypotheses, synth, vis
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.estimater import make_mesh_tensors
    from foundationpose_b200.weights import random_state_dict

    mesh = synth.make_mesh(5)
    pose = np.eye(4)
    pose[:3, :3] = synth.random_rotation(0)
    pose[:3, 3] = [0.02, -0.01, 0.6]
    rgb, depth, mask = synth.make_scene(mesh.visual.image, pose)
    mt = make_mesh_tensors(mesh)
    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(mesh.vertices), uv=mt.get("uv"), tex=mt.get("tex"))
    e.set_frame(rgb, depth, synth.DEFAULT_K, filter_depth=True)
    grid = torch.as_tensor(hypotheses.make_rotation_grid(40, 60, np.eye(4, dtype=np.float32)[None]), device="cuda", dtype=torch.float32)
    start, _ = e.start_poses(mask, grid)
    refined, _, _ = e.refine(start, 5)
    scores, _ = e.score(refined)
    order = scores.argsort(descending=True).to(torch.int32)
    N, r = len(start), args.reps
    out = dict(N=N, reps=r)
    for kind in ("refine", "score"):
        crops = (lambda: (e.vis_crops(start, 0), e.vis_crops(refined, 0))) if kind == "refine" else (lambda: e.vis_crops(refined, 1))
        full = (lambda: e.vis("refine", start, refined)) if kind == "refine" else (lambda: e.vis("score", refined, order=order))
        t_crops, t_full = dev_ms(crops, r), dev_ms(full, r)
        canvas = full()
        torch.cuda.synchronize()
        t_d2h = wall_ms(lambda: canvas.cpu(), r)
        host = canvas.cpu().numpy()
        t_label = wall_ms(lambda: (vis.refine_canvas if kind == "refine" else vis.score_canvas)(e, start if kind == "refine" else refined,
                                                                                            refined if kind == "refine" else scores), r) - t_d2h - t_full
        t_png = wall_ms(lambda: cv2.imencode(".png", host[..., ::-1]), r)
        if kind == "refine":
            ra, rb = e.vis_crops(start, 0).cpu().numpy(), e.vis_crops(refined, 0).cpu().numpy()
            t_host = wall_ms(lambda: vis_compose.refine_canvas(ra, rb), 1)
        else:
            rs = e.vis_crops(refined, 1).cpu().numpy()
            o = order.cpu().numpy()
            t_host = wall_ms(lambda: vis_compose.score_canvas(rs, o), 1)
        out[kind] = dict(shape=list(host.shape), crop_passes_ms=t_crops, canvas_kernels_ms=t_full - t_crops, d2h_ms=t_d2h,
                         labels_ms=max(t_label, 0.0), png_encode_ms=t_png, host_composition_ms=t_host)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out["device"] = q.stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
