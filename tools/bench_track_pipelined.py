"""Blocking against non-blocking tracking calls: per-frame time (p50 / p99) and frames/s of Engine.track_cameras at
C = 1, 2, 4, 8 cameras of 640x480 with one and two objects per camera, 2 refine iterations.

  blocking      each call returns the host poses: the host copies frame t into pinned staging only after frame t - 1
                has been tracked.
  non-blocking  wait=False: frame t is submitted (staged, uploaded, launched) before frame t - 1 is collected, so the
                host's copies of frame t run while the device tracks frame t - 1.

A frame's time is the interval between two successive collected results (the call time for the blocking mode); every
frame chains its start poses from the previous frame's device poses.  Every shape is warmed up in both modes first, then
the two modes alternate run by run.  The card's name and power limit are printed with the results.

    python tools/bench_track_pipelined.py [--frames 200] [--runs 5] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from foundationpose_b200 import synth  # noqa: E402
from foundationpose_b200.engine import Engine  # noqa: E402
from foundationpose_b200.estimater import make_mesh_tensors  # noqa: E402
from foundationpose_b200.weights import random_state_dict  # noqa: E402

H, W = 480, 640
N_UNIQUE = 4  # distinct frames per camera, cycled


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def scenes(meshes, n_cam):
    """N_UNIQUE frames of each of n_cam cameras (intrinsics differ slightly per camera), both objects in view."""
    out = []
    for c in range(n_cam):
        K = synth.DEFAULT_K.copy()
        K[0, 2] += 2.0 * c
        K[1, 1] *= 1.0 + 0.005 * c
        poses = []
        for k in range(len(meshes)):
            p = np.eye(4)
            p[:3, :3] = synth.random_rotation(10 * c + k)
            p[:3, 3] = [-0.08 + 0.16 * k, 0.0, 0.6 + 0.05 * k]
            poses.append(p)
        frames = []
        for t in range(N_UNIQUE):
            rgb, depth, _ = synth.make_multi_scene([(m.visual.image, p, 1.0) for m, p in zip(meshes, poses)], K, H, W, seed=c * 10 + t)
            frames.append((rgb, depth, K))
        out.append((frames, [p.astype(np.float32) for p in poses]))
    return out


def run(e, cams, n_obj, frames, wait):
    """Per-frame times (ms) and the total time of `frames` calls."""
    views = lambda t: [fr[t % N_UNIQUE] for fr, _ in cams]
    cam_of = [c for c in range(len(cams)) for _ in range(n_obj)]
    slots = [k + 1 for _ in cams for k in range(n_obj)]
    pose = torch.from_numpy(np.stack([p for _, poses in cams for p in poses[:n_obj]])).cuda()
    torch.cuda.synchronize()
    stamps = [time.perf_counter()]
    prev = None
    for t in range(frames):
        if wait:
            pose, _ = e.track_cameras(views(t), pose, cam_of, slots, 2)
            stamps.append(time.perf_counter())
        else:
            pose, pending = e.track_cameras(views(t), pose, cam_of, slots, 2, wait=False)
            if prev is not None:
                prev.result()
                stamps.append(time.perf_counter())
            prev = pending
    if prev is not None:
        prev.result()
        stamps.append(time.perf_counter())
    dt = np.diff(stamps) * 1e3
    return dt, stamps[-1] - stamps[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_track_pipelined needs a CUDA device")
    meshes = [synth.make_mesh(4, tex_seed=k, tex_size=512) for k in range(2)]
    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.set_config("refine")
    for k, m in enumerate(meshes):
        mt = make_mesh_tensors(m)
        e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(m.vertices), uv=mt["uv"], tex=mt["tex"], slot=k + 1)
    all_cams = scenes(meshes, 8)
    shapes = [(C, n_obj) for C in (1, 2, 4, 8) for n_obj in (1, 2)]
    for C, n_obj in shapes:  # warm-up: first sight runs eagerly, the second call captures, later calls replay
        for wait in (True, False):
            run(e, all_cams[:C], n_obj, 20, wait)
    rows = []
    for C, n_obj in shapes:
        res = {True: ([], 0.0, 0), False: ([], 0.0, 0)}
        for r in range(args.runs):
            for wait in ((True, False) if r % 2 == 0 else (False, True)):
                dt, total = run(e, all_cams[:C], n_obj, args.frames, wait)
                a, tt, n = res[wait]
                res[wait] = (a + list(dt), tt + total, n + args.frames)
        row = dict(cameras=C, objects_per_camera=n_obj)
        for wait, name in ((True, "blocking"), (False, "non_blocking")):
            a, tt, n = res[wait]
            a = np.asarray(a)
            row[name] = dict(ms_p50=round(float(np.percentile(a, 50)), 3), ms_p99=round(float(np.percentile(a, 99)), 3),
                             fps=round(n / tt, 1))
        row["speedup_fps"] = round(row["non_blocking"]["fps"] / row["blocking"]["fps"], 3)
        rows.append(row)
        print(json.dumps(row), flush=True)
    out = dict(card=card(), frame=f"{W}x{H}", iterations=2, frames_per_run=args.frames, runs=args.runs, results=rows)
    print(json.dumps(dict(card=out["card"])))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)
    e.close()


if __name__ == "__main__":
    main()
