"""Frames already on the GPU against host frames: per-frame time (p50 / p99) of Engine.track_cameras at C = 1, 2, 4, 8
cameras of 640x480, one object per camera, two refiner passes, blocking and non-blocking (wait=False); and the call time
of Engine.register_objects with M = 1 and 4 objects and full 252-pose grids, host against device frames and masks.

  host    numpy frames: the library copies each into pinned staging on the calling thread and uploads it.
  device  CUDA tensors, read in place: a ring of distinct pre-filled device frames per camera, so the addresses change
          every call.

A tracking frame's time is the interval between two successive collected results (the call time for the blocking mode);
every frame chains its start poses from the previous frame's device poses.  Every shape is warmed up in every mode
first, then the modes take turns run by run, each run starting with the next mode in turn.  Register calls alternate
host and device call by call.  Prints the card's name and power limit, one JSON line per tracking shape, and one JSON line
with every result.

    python tools/bench_track_device.py [--frames 200] [--runs 4] [--register-calls 8] [--out FILE.json]
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
from foundationpose_b200.hypotheses import make_rotation_grid  # noqa: E402
from foundationpose_b200.weights import random_state_dict  # noqa: E402

H, W = 480, 640
N_UNIQUE = 4  # distinct host frames per camera, cycled
RING = 8  # distinct device frames per camera, cycled: the library sees a new address every call
MODES = [("host", True), ("host", False), ("device", True), ("device", False)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def cameras(mesh, n_cam):
    """N_UNIQUE host frames and RING device frames of each of n_cam cameras (intrinsics differ slightly per camera), and
    each camera's object pose."""
    out = []
    for c in range(n_cam):
        K = synth.DEFAULT_K.copy()
        K[0, 2] += 2.0 * c
        K[1, 1] *= 1.0 + 0.005 * c
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(10 * c)
        p[:3, 3] = [0.0, 0.0, 0.6]
        host = []
        for t in range(N_UNIQUE):
            rgb, depth, _ = synth.make_multi_scene([(mesh.visual.image, p, 1.0)], K, H, W, seed=c * 10 + t)
            host.append((rgb, depth.astype(np.float32), K))
        dev = [(torch.from_numpy(host[t % N_UNIQUE][0]).cuda(), torch.from_numpy(host[t % N_UNIQUE][1]).cuda(), K)
               for t in range(RING)]
        out.append(dict(host=host, device=dev, pose=p.astype(np.float32)))
    return out


def run(e, cams, frames, where, wait):
    """Per-frame times (ms) of `frames` tracking calls."""
    ring = N_UNIQUE if where == "host" else RING
    views = lambda t: [cam[where][t % ring] for cam in cams]
    cam_of = list(range(len(cams)))
    slots = [1] * len(cams)
    pose = torch.from_numpy(np.stack([cam["pose"] for cam in cams])).cuda()
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
    return np.diff(stamps) * 1e3


def stats(a):
    a = np.asarray(a)
    return dict(ms_p50=round(float(np.percentile(a, 50)), 3), ms_p99=round(float(np.percentile(a, 99)), 3))


def register_leg(e, meshes, n_calls):
    """register_objects with M = 1 and 4 objects, full 252-pose grids, host against device frames and masks."""
    grid = torch.from_numpy(make_rotation_grid().astype(np.float32)).cuda()
    poses = []
    for k in range(4):
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(40 + k)
        p[:3, 3] = [-0.21 + 0.14 * k, 0.0, 0.75]
        poses.append(p)
    rgb, depth, owner = synth.make_multi_scene([(meshes[k].visual.image, poses[k], 1.0) for k in range(4)], seed=1)
    depth = depth.astype(np.float32)
    K = synth.DEFAULT_K
    rows = []
    for M in (1, 4):
        masks = np.stack([owner == k for k in range(M)])
        args = dict(host=(rgb, depth, masks), device=(torch.from_numpy(rgb).cuda(), torch.from_numpy(depth).cuda(),
                                                      torch.from_numpy(masks).cuda()))
        slots = [k + 1 for k in range(M)]
        times = dict(host=[], device=[])
        for i in range(2 + n_calls):  # two warm-up calls of each: the first runs eagerly, the second captures
            for where in (("host", "device") if i % 2 == 0 else ("device", "host")):
                r, d, m = args[where]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e.register_objects(r, d, K, m, [grid] * M, slots, 5)
                dt = (time.perf_counter() - t0) * 1e3  # the call synchronises its stream
                if i >= 2:
                    times[where].append(dt)
        row = dict(objects=M, hypotheses=int(M * len(grid)), iterations=5, calls=n_calls)
        for where in ("host", "device"):
            row[where] = stats(times[where])
        rows.append(row)
        print(json.dumps(dict(register_objects=row)), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--runs", type=int, default=4)
    ap.add_argument("--register-calls", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_track_device needs a CUDA device")
    print(json.dumps(dict(card=card())), flush=True)
    meshes = [synth.make_mesh(4, tex_seed=k, tex_size=512) for k in range(4)]
    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    e.set_config("refine")
    e.set_config("score")
    for k, m in enumerate(meshes):
        mt = make_mesh_tensors(m)
        e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(m.vertices), uv=mt["uv"], tex=mt["tex"], slot=k + 1)
    all_cams = cameras(meshes[0], 8)
    counts = (1, 2, 4, 8)
    for C in counts:  # warm-up: first sight runs eagerly, the second call captures, later calls replay
        for where, wait in MODES:
            run(e, all_cams[:C], 20, where, wait)
    rows = []
    for C in counts:
        res = {m: [] for m in MODES}
        for r in range(args.runs):
            for k in range(len(MODES)):
                mode = MODES[(r + k) % len(MODES)]
                res[mode] += list(run(e, all_cams[:C], args.frames, *mode))
        row = dict(cameras=C)
        for where, wait in MODES:
            row[f"{where}_{'blocking' if wait else 'non_blocking'}"] = stats(res[(where, wait)])
        rows.append(row)
        print(json.dumps(row), flush=True)
    reg = register_leg(e, meshes, args.register_calls)
    out = dict(card=card(), frame=f"{W}x{H}", objects_per_camera=1, iterations=2, frames_per_run=args.frames, runs=args.runs,
               track_cameras=rows, register_objects=reg)
    print(json.dumps(out), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)
    e.close()


if __name__ == "__main__":
    main()
