"""The cost of the tracking fit counts: `Engine.track_cameras` with and without `fit_delta` (the fit pass at the returned
poses, one more crop-producer launch in the same graph plus a 20-byte-per-object read-back).

    python tools/bench_track_fit.py [n_calls]

Prints one JSON line: p50 / p99 wall-clock ms per call with the fit off and on, alternated call by call, at C cameras x
objects per camera = 1 x 1, 1 x 8 and 4 x 1, 640x480 host frames, two refiner passes, blocking and non-blocking (one call
always in flight, wait=False); the GPU time of the fit pass's crop_tile_kernel launch from torch.profiler over eager
launches (FPOSE_NO_GRAPH=1) in a separate process; and the name and power limit of the GPU."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

CONFIGS = [(1, 1), (1, 8), (4, 1)]  # (cameras, objects per camera)
DELTA = 0.015


def _setup():
    """An engine with 8 meshes in slots 1..8 and, per camera, 20 frames of its objects on their walks."""
    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.estimater import make_mesh_tensors
    from foundationpose_b200.weights import random_state_dict

    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.set_config("refine")
    n_cam, n_obj = 4, 8
    meshes = []
    for k in range(n_obj):
        scale = 0.5 + 0.05 * k
        m = synth.make_mesh(3, tex_seed=k, tex_size=256, scale=scale)
        mt = make_mesh_tensors(m)
        e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(m.vertices), uv=mt["uv"], tex=mt["tex"], slot=k + 1)
        meshes.append((m, scale))
    scenes = []
    for c in range(n_cam):
        objs = range(n_obj) if c == 0 else [c]
        walks = {}
        for j, k in enumerate(objs):
            p0 = np.eye(4)
            p0[:3, :3] = synth.random_rotation(100 + 10 * c + k)
            p0[:3, 3] = [-0.24 + 0.16 * (j % 4), -0.08 + 0.16 * (j // 4), 0.8]
            walks[k] = synth.track_sequence(20, p0, seed=200 + 10 * c + k)
        frames = [synth.make_multi_scene([(meshes[k][0].visual.image, walks[k][i], meshes[k][1]) for k in objs],
                                         seed=1 + i + 50 * c)[:2] for i in range(20)]
        scenes.append((list(objs), walks, frames))
    return e, scenes


def _args(scenes, C, per_cam, f):
    frames, start, cam_of, slots = [], [], [], []
    for c in range(C):
        objs, walks, fr = scenes[c]
        frames.append((fr[f][0], fr[f][1], np.array([[615.0, 0, 320.0], [0, 615.0, 240.0], [0, 0, 1]])))
        for k in objs[:per_cam]:
            start.append(walks[k][f])
            cam_of.append(c)
            slots.append(k + 1)
    return frames, torch.as_tensor(np.stack(start), dtype=torch.float32, device="cuda"), cam_of, slots


def wall_clock(n_calls):
    e, scenes = _setup()
    pct = lambda a, q: float(np.sort(a)[min(int(len(a) * q), len(a) - 1)])
    out = {}
    for C, per_cam in CONFIGS:
        for blocking in (True, False):
            t = {"fit_off": [], "fit_on": []}
            pending = None
            for i in range(40 + 2 * n_calls):
                k40 = i % 40
                f = k40 if k40 < 20 else 39 - k40  # forwards, then backwards
                frames, start, cam_of, slots = _args(scenes, C, per_cam, f)
                mode = "fit_on" if i % 2 else "fit_off"
                delta = DELTA if mode == "fit_on" else None
                t0 = time.perf_counter()
                if blocking:
                    e.track_cameras(frames, start, cam_of, slots, 2, fit_delta=delta)
                else:
                    _, nxt = e.track_cameras(frames, start, cam_of, slots, 2, wait=False, fit_delta=delta)
                    if pending is not None:
                        pending.result()
                    pending = nxt
                t1 = time.perf_counter()
                if i >= 40:  # every shape warmed up, graphs captured
                    t[mode].append((t1 - t0) * 1e3)
            if pending is not None:
                pending.result()
            r = {m: {"ms_p50": pct(v, 0.5), "ms_p99": pct(v, 0.99)} for m, v in t.items()}
            r["p50_added_ms"] = r["fit_on"]["ms_p50"] - r["fit_off"]["ms_p50"]
            out[f"C={C},objects_per_camera={per_cam},{'blocking' if blocking else 'wait=False'}"] = r
    e.close()
    return out


def kernel_time(n_calls=50):
    """GPU time of the fit pass (the crop_tile_kernel instantiation with kFit) per launch, eager launches under
    torch.profiler; run with FPOSE_NO_GRAPH=1."""
    from torch.profiler import ProfilerActivity, profile

    e, scenes = _setup()
    out = {}
    for C, per_cam in CONFIGS:
        frames, start, cam_of, slots = _args(scenes, C, per_cam, 0)
        for _ in range(3):
            e.track_cameras(frames, start, cam_of, slots, 2, fit_delta=DELTA)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n_calls):
                e.track_cameras(frames, start, cam_of, slots, 2, fit_delta=DELTA)
            torch.cuda.synchronize()
        fit_us, n, crop_us, all_us = 0.0, 0, 0.0, 0.0
        for ev in prof.key_averages():
            dt = getattr(ev, "device_time_total", None)
            dt = ev.cuda_time_total if dt is None else dt
            if ev.key.startswith("void fp::crop_tile_kernel<") and ev.key.split(">")[0].endswith("true"):
                fit_us += dt
                n += ev.count
            elif ev.key.startswith("void fp::crop_tile_kernel<"):
                crop_us += dt
            if not ev.key.startswith("Memcpy") and not ev.key.startswith("Memset"):
                all_us += dt
        out[f"C={C},objects_per_camera={per_cam}"] = {
            "fit_kernel_us_per_launch": fit_us / max(n, 1), "fit_launches": n,
            "refiner_crop_kernels_us_per_call": crop_us / n_calls, "all_kernels_us_per_call": all_us / n_calls}
    e.close()
    return out


def main():
    from bench import device_info

    if "--kernel-time" in sys.argv:
        print("KERNEL " + json.dumps(kernel_time()))
        return
    n_calls = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    out = {"wall_clock": wall_clock(n_calls), "calls_per_mode": n_calls, "refine_iters": 2, "delta_m": DELTA,
           "api": "Engine.track_cameras(frames, poses, camera_of, slots, 2[, fit_delta]) with 640x480 host numpy frames; "
                  "wait=False: one call in flight, time from one submit to the next after collecting the previous call"}
    env = dict(os.environ, FPOSE_NO_GRAPH="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--kernel-time"], env=env, capture_output=True, text=True)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("KERNEL ")]
    out["fit_kernel"] = json.loads(lines[-1][len("KERNEL "):]) if lines else {"error": r.stderr[-2000:]}
    out["fit_kernel_note"] = "torch.profiler over 50 eager calls (FPOSE_NO_GRAPH=1) per config, in its own process"
    out["device"] = device_info(torch.cuda.current_device())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
