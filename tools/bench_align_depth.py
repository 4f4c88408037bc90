"""Depth from its own sensor: what aligning on the GPU costs and saves.

  * In a process of its own, under torch.profiler: the GPU time of align_depth_kernel (camera-table launch, inside
    track_cameras) at 848x480 -> 1280x720 (a D435-like rig) and 640x480 -> 640x480, for C = 1 and 4 cameras, device
    uint16 frames (so only the launches run).
  * Engine.track_cameras per call (p50 / p99), one object per camera, two refiner passes, C = 1 and 4, both rigs:
    sensor-native uint16 depth with a DepthSensor (aligned by the library) against the same depth pre-aligned to the
    colour frame as float32 metres (aligned once beforehand, not timed), for host frames and device frames, blocking and
    wait=False; the modes alternate call by call.
  * The bytes staged per call for host frames in each mode (colour + depth uploads, computed from the shapes).
  * The host cost of aligning one frame with the numpy float32 restatement of the rule (tests/align_reference.py) --
    the numpy restatement, not librealsense's rs2::align, which is not measured here.

Prints the card's name and power limit, read in the same run, and one JSON line with every result.

    python tools/bench_align_depth.py [--calls 100] [--out FILE.json]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import align_reference as ar  # noqa: E402
from foundationpose_b200 import ops, synth  # noqa: E402
from foundationpose_b200.engine import Engine  # noqa: E402
from foundationpose_b200.estimater import make_mesh_tensors  # noqa: E402
from foundationpose_b200.frames import Depth, DepthSensor  # noqa: E402
from foundationpose_b200.weights import random_state_dict  # noqa: E402

SCALE = 0.001
RIGS = {"848x480->1280x720": (ar.D435_DEPTH_K, (480, 848), ar.D435_COLOR_K, (720, 1280)),
        "640x480->640x480": (ar.VGA_DEPTH_K, (480, 640), ar.VGA_COLOR_K, (480, 640))}
COUNTS = (1, 4)
MODES = [(kind, where, wait) for kind in ("native", "prealigned") for where in ("host", "device") for wait in (True, False)]
N_UNIQUE = 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def stats(a):
    a = np.asarray(a)
    return dict(ms_p50=round(float(np.percentile(a, 50)), 3), ms_p99=round(float(np.percentile(a, 99)), 3))


def engine(mesh):
    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    e.set_config("refine")
    e.set_config("score")
    mt = make_mesh_tensors(mesh)
    e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(mesh.vertices), uv=mt["uv"], tex=mt["tex"], slot=0)
    return e


def cameras(mesh, rig, n_cam):
    """Per camera: its sensor, colour K, N_UNIQUE (rgb, uint16 depth of the depth imager, the same depth pre-aligned to
    the colour frame by fp_align_depth) and its object's pose in the colour camera."""
    Kd, (Hd, Wd), Kc, (H, W) = RIGS[rig]
    out = []
    for c in range(n_cam):
        T = ar.rig_T(t=(0.015 + 0.002 * c, 0.0002, -0.0004))
        s = DepthSensor(Kd, T)
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(10 * c)
        p[:3, 3] = [0.0, 0.0, 0.6]
        frames = []
        for t in range(N_UNIQUE):
            rgb, _, _ = synth.make_multi_scene([(mesh.visual.image, p, 1.0)], Kc, H, W, seed=c * 10 + t)
            _, depth, _ = synth.make_multi_scene([(mesh.visual.image, np.linalg.inv(T) @ p, 1.0)], Kd, Hd, Wd, seed=c * 10 + t)
            u16 = np.round(depth.astype(np.float64) / SCALE).astype(np.uint16)
            aligned = ops.align_depth(Depth(torch.from_numpy(u16).cuda(), SCALE, sensor=s), None, Kc, H, W).cpu().numpy()
            frames.append(dict(rgb=rgb, u16=u16, aligned=aligned, rgb_d=torch.from_numpy(rgb).cuda(),
                               u16_d=torch.from_numpy(u16).cuda(), aligned_d=torch.from_numpy(aligned).cuda()))
        out.append(dict(sensor=s, K=Kc, frames=frames, pose=p.astype(np.float32)))
    return out


def views(cams, t, kind, where):
    out = []
    for cam in cams:
        f = cam["frames"][t % N_UNIQUE]
        d = "_d" if where == "device" else ""
        depth = Depth(f["u16" + d], SCALE, sensor=cam["sensor"]) if kind == "native" else f["aligned" + d]
        out.append((f["rgb" + d], depth, cam["K"]))
    return out


def staged_bytes(rig, n, kind):
    """Host bytes uploaded per call for the frames: colour RGB8, then uint16 depth of the depth imager or float32 depth of
    the colour frame."""
    _, (Hd, Wd), _, (H, W) = RIGS[rig]
    return n * (H * W * 3 + (Hd * Wd * 2 if kind == "native" else H * W * 4))


def track_leg(e, mesh, n_calls):
    rows = []
    for rig in RIGS:
        all_cams = cameras(mesh, rig, max(COUNTS))
        for n in COUNTS:
            cams = all_cams[:n]
            pose0 = torch.from_numpy(np.stack([c["pose"] for c in cams])).cuda()
            a = e.track_cameras(views(cams, 0, "prealigned", "host"), pose0, list(range(n)), [0] * n, 2)[1]
            b = e.track_cameras(views(cams, 0, "native", "host"), pose0, list(range(n)), [0] * n, 2)[1]
            assert np.array_equal(a, b), "sensor-native and pre-aligned depth must give the same poses"
            pose = {m: pose0.clone() for m in MODES}
            pending = {m: None for m in MODES}
            times = {m: [] for m in MODES}
            for t in range(4 + n_calls):
                for k in range(len(MODES)):
                    m = MODES[(t + k) % len(MODES)]
                    kind, where, wait = m
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    pose[m], res = e.track_cameras(views(cams, t, kind, where), pose[m], list(range(n)), [0] * n, 2, wait=wait)
                    if not wait:
                        if pending[m] is not None:
                            pending[m].result()
                        pending[m] = res
                    if t >= 4:
                        times[m].append((time.perf_counter() - t0) * 1e3)
            for m in MODES:
                if pending[m] is not None:
                    pending[m].result()
            row = dict(rig=rig, cameras=n, host_bytes_staged=dict(native=staged_bytes(rig, n, "native"),
                                                                  prealigned=staged_bytes(rig, n, "prealigned")))
            for kind, where, wait in MODES:
                row[f"{kind}_{where}_{'blocking' if wait else 'non_blocking'}"] = stats(times[(kind, where, wait)])
            rows.append(row)
            print(json.dumps(row), flush=True)
    return rows


def numpy_leg(mesh, reps=5):
    """Host ms per frame of the numpy float32 restatement of the rule (not librealsense)."""
    out = {}
    for rig in RIGS:
        Kd, (Hd, Wd), Kc, (H, W) = RIGS[rig]
        cam = cameras(mesh, rig, 1)[0]
        m, valid = ar.depth_metres(cam["frames"][0]["u16"], SCALE)
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            ar.align(m, valid, Kd, cam["sensor"].T, Kc, H, W)
            ts.append((time.perf_counter() - t0) * 1e3)
        out[rig] = dict(ms_p50=round(float(np.median(ts)), 1))
    return out


def profile_leg(calls=50):
    """Run in a process of its own: align_depth_kernel's GPU time per launch inside track_cameras (a graph replay), device
    uint16 frames, both rigs, C = 1 and 4."""
    from torch.profiler import ProfilerActivity, profile

    mesh = synth.make_mesh(3, tex_seed=0, tex_size=256)
    e = engine(mesh)
    out = {}
    for rig in RIGS:
        all_cams = cameras(mesh, rig, max(COUNTS))
        for n in COUNTS:
            cams = all_cams[:n]
            pose = torch.from_numpy(np.stack([c["pose"] for c in cams])).cuda()
            v = views(cams, 0, "native", "device")
            fn = lambda: e.track_cameras(v, pose, list(range(n)), [0] * n, 2)
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(calls):
                    fn()
                torch.cuda.synchronize()
            ts = [ev.device_time for ev in prof.events() if "align_depth_kernel" in ev.name]
            fp = [ev.device_time for ev in prof.events() if "frame_prep_kernel" in ev.name]
            out[f"{rig} C={n}"] = dict(align_us_p50=round(float(np.median(ts)), 2) if ts else None, n=len(ts),
                                       frame_prep_us_p50=round(float(np.median(fp)), 2) if fp else None)
    e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile-only", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_align_depth needs a CUDA device")
    if args.profile_only:
        print(json.dumps(dict(profile=profile_leg())), flush=True)
        return
    print(json.dumps(dict(card=card())), flush=True)
    mesh = synth.make_mesh(4, tex_seed=0, tex_size=512)
    e = engine(mesh)
    rows = track_leg(e, mesh, args.calls)
    e.close()
    host = numpy_leg(mesh)
    q = subprocess.run([sys.executable, os.path.abspath(__file__), "--profile-only"], capture_output=True, text=True)
    prof = None
    for line in q.stdout.splitlines():
        if line.startswith('{"profile"'):
            prof = json.loads(line)["profile"]
    if prof is None:
        sys.stderr.write(q.stdout[-2000:] + q.stderr[-4000:])
    out = dict(card=card(), objects_per_camera=1, iterations=2, depth_scale=SCALE, calls=args.calls, track_cameras=rows,
               numpy_restatement_ms_per_frame=host, align_kernel_gpu_us=prof)
    print(json.dumps(out), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
