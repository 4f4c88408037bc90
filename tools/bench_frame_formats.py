"""Sensor-native frames against converting on the host: per-call time (p50 / p99) of Engine.track_cameras at C = 1, 2, 4,
8 cameras of 640x480 and of 1280x720, one object per camera, two refiner passes, host frames, blocking and non-blocking
(wait=False), for two recipes on the same BGR8 colour and uint16 depth (scale 1 mm) as a RealSense or OpenCV delivers:

  convert  today's recipe: per camera cv2.cvtColor(BGR -> RGB) and depth.astype(np.float32) * scale on the host, then
           the plain packed RGB8 / float32 frames (staged at 3 + 4 bytes per pixel)
  native   Color(bgr, "bgr") and Depth(u16, scale): no host conversion, staged at 3 + 2 bytes per pixel, unpacked by the
           frame filter

Both recipes compute the same poses (checked on the first frame of every shape).  A call's time is the interval between
two successive collected results (the call time for the blocking mode), host conversion included.  Every shape is warmed
up in every mode first, then the four modes take turns call by call.  Also: register_objects p50 at M = 1 with a full
252-pose grid, plain and native, alternated call by call; and, in a separate process under torch.profiler, the GPU time
of the frame-preparation launch per format at both sizes, by value (fp_set_frame) and from the camera table
(track_cameras), and with --parent-lib (a build of the parent commit's sources) both launches on default frames against
that library's (fp_set_frame and fp_track), alternated call by call.  And device frames (CUDA tensors) at C = 1 and 4,
640x480, blocking: converted on the device with torch before each call, against the same tensors wrapped.  Prints the card's name and power limit, read in the same run, and one JSON line with every result.

    python tools/bench_frame_formats.py [--calls 100] [--out FILE.json] [--parent-lib PATH]
"""
import argparse
import ctypes as C
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
from foundationpose_b200.frames import Color, Depth  # noqa: E402
from foundationpose_b200.hypotheses import make_rotation_grid  # noqa: E402
from foundationpose_b200.weights import random_state_dict  # noqa: E402

SCALE = 0.001
SIZES = [(480, 640), (720, 1280)]
COUNTS = (1, 2, 4, 8)
MODES = [("convert", True), ("native", True), ("convert", False), ("native", False)]
N_UNIQUE = 3  # distinct frames per camera, cycled


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def stats(a):
    a = np.asarray(a)
    return dict(ms_p50=round(float(np.percentile(a, 50)), 3), ms_p99=round(float(np.percentile(a, 99)), 3))


def engine(meshes):
    e = Engine()
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", random_state_dict("score", 0))
    e.set_config("refine")
    e.set_config("score")
    for k, m in enumerate(meshes):
        mt = make_mesh_tensors(m)
        e.set_mesh(mt["pos"], mt["normals"], mt["faces"], synth.mesh_diameter(m.vertices), uv=mt["uv"], tex=mt["tex"], slot=k)
    return e


def sensor_frames(mesh, H, W, n_cam):
    """N_UNIQUE sensor frames (BGR8, uint16 mm) of each camera, its intrinsics and its object's pose."""
    out = []
    for c in range(n_cam):
        K = np.array([[615.0 * W / 640, 0, W / 2 + 2.0 * c], [0, 615.0 * W / 640, H / 2], [0, 0, 1]])
        p = np.eye(4)
        p[:3, :3] = synth.random_rotation(10 * c)
        p[:3, 3] = [0.0, 0.0, 0.6]
        frames = []
        for t in range(N_UNIQUE):
            rgb, depth, _ = synth.make_multi_scene([(mesh.visual.image, p, 1.0)], K, H, W, seed=c * 10 + t)
            u16 = np.round(depth.astype(np.float64) / SCALE).astype(np.uint16)
            frames.append((np.ascontiguousarray(rgb[..., ::-1]), u16))
        out.append(dict(K=K, frames=frames, pose=p.astype(np.float32)))
    return out


def views(cams, t, recipe):
    import cv2

    out = []
    for cam in cams:
        bgr, u16 = cam["frames"][t % N_UNIQUE]
        if recipe == "convert":
            out.append((cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB), u16.astype(np.float32) * np.float32(SCALE), cam["K"]))
        else:
            out.append((Color(bgr, "bgr"), Depth(u16, SCALE), cam["K"]))
    return out


def call(e, cams, t, recipe, wait, pose):
    """One call of `recipe`, conversion included; returns (new device poses, host poses or a PendingPoses)."""
    n = len(cams)
    return e.track_cameras(views(cams, t, recipe), pose, list(range(n)), [0] * n, 2, wait=wait)


def track_leg(e, mesh, n_calls):
    rows = []
    for H, W in SIZES:
        all_cams = sensor_frames(mesh, H, W, max(COUNTS))
        for n in COUNTS:
            cams = all_cams[:n]
            pose0 = torch.from_numpy(np.stack([c["pose"] for c in cams])).cuda()
            a = call(e, cams, 0, "convert", True, pose0)[1]
            b = call(e, cams, 0, "native", True, pose0)[1]
            assert np.array_equal(a, b), "the two recipes must give the same poses"
            pose = {m: pose0.clone() for m in MODES}
            pending = {m: None for m in MODES}
            times = {m: [] for m in MODES}
            for t in range(4 + n_calls):  # warm-up: first sight runs eagerly, the second call captures, later replay
                for k in range(len(MODES)):
                    m = MODES[(t + k) % len(MODES)]
                    recipe, wait = m
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    pose[m], res = call(e, cams, t, recipe, wait, pose[m])
                    if not wait:
                        # one call of this mode in flight: collect the previous one after submitting this one
                        if pending[m] is not None:
                            pending[m].result()
                        pending[m] = res
                    dt = (time.perf_counter() - t0) * 1e3
                    if t >= 4:
                        times[m].append(dt)
            for m in MODES:
                if pending[m] is not None:
                    pending[m].result()
            row = dict(frame=f"{W}x{H}", cameras=n)
            for recipe, wait in MODES:
                row[f"{recipe}_{'blocking' if wait else 'non_blocking'}"] = stats(times[(recipe, wait)])
            rows.append(row)
            print(json.dumps(row), flush=True)
    return rows


def register_leg(e, mesh, n_calls):
    grid = torch.from_numpy(make_rotation_grid().astype(np.float32)).cuda()
    cam = sensor_frames(mesh, 480, 640, 1)[0]
    p = cam["pose"]
    rgb, depth, owner = synth.make_multi_scene([(mesh.visual.image, p, 1.0)], cam["K"], 480, 640, seed=1)
    bgr = np.ascontiguousarray(rgb[..., ::-1])
    u16 = np.round(depth.astype(np.float64) / SCALE).astype(np.uint16)
    masks = (owner == 0)[None]
    times = dict(convert=[], native=[])
    for i in range(2 + n_calls):
        for recipe in (("convert", "native") if i % 2 == 0 else ("native", "convert")):
            import cv2

            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if recipe == "convert":
                args = (cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB), u16.astype(np.float32) * np.float32(SCALE))
            else:
                args = (Color(bgr, "bgr"), Depth(u16, SCALE))
            e.register_objects(*args, cam["K"], masks, [grid], [0], 5)
            dt = (time.perf_counter() - t0) * 1e3  # the call synchronises its stream
            if i >= 2:
                times[recipe].append(dt)
    row = dict(objects=1, hypotheses=len(grid), iterations=5, calls=n_calls,
               convert=stats(times["convert"]), native=stats(times["native"]))
    print(json.dumps(dict(register_objects=row)), flush=True)
    return row


# formats of the profiled frame-preparation launches: (name, colour order, uint16?, pitched?)
PROFILE_FORMATS = [("rgb8_f32_packed", "rgb", False, False), ("bgr8_u16_packed", "bgr", True, False),
                   ("bgra8_u16_pitched", "bgra", True, True)]


def _parent_ctx(parent_lib, mesh):
    """A context of the library at `parent_lib` (a build of other sources with the same C ABI for these calls), with the
    same seeded networks and mesh in slot 0 as engine([mesh])."""
    from foundationpose_b200.engine import _mesh_args, _tensor_array, pack_network

    par = C.CDLL(parent_lib)
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    par.fp_create.argtypes = [C.POINTER(vp)]
    par.fp_destroy.argtypes = [vp]
    par.fp_load_network.argtypes = [vp, i, vp, i]
    par.fp_set_mesh.argtypes = [vp, i, i, vp, vp, vp, vp, vp, vp, i, i, f]
    par.fp_set_frame.argtypes = [vp, vp, vp, C.POINTER(f), i, i, i, f, vp]
    par.fp_track.argtypes = [vp, vp, vp, C.POINTER(f), i, i, vp, i, vp, vp, vp]
    ctx = vp()
    assert par.fp_create(C.byref(ctx)) == 0
    for which, kind in enumerate(("refine", "score")):
        arr, keep = _tensor_array(pack_network(random_state_dict(kind, 0), kind))
        assert par.fp_load_network(ctx, which, C.cast(arr, vp), len(arr)) == 0
    mt = make_mesh_tensors(mesh)
    args, keep = _mesh_args(mt["pos"], mt["normals"], mt["faces"], mt["uv"], mt["tex"])
    assert par.fp_set_mesh(ctx, *args, float(synth.mesh_diameter(mesh.vertices))) == 0
    return par, ctx


def _alternated(fns, n, matches):
    """GPU time (us, p50 and mean) of the kernels picked by each of `matches`, over n rounds that call every fn of `fns`
    in turn, under torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    for _ in range(5):
        for fn in fns:
            fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            for fn in fns:
                fn()
        torch.cuda.synchronize()
    out = []
    for match in matches:
        ts = [ev.device_time for ev in prof.events() if match(ev.name)]
        out.append(dict(p50=round(float(np.median(ts)), 2), mean=round(float(np.mean(ts)), 2), n=len(ts)) if ts else None)
    return out


def profile_leg(parent_lib, n=200):
    """Run in a process of its own: GPU time of the frame-preparation launch per format at 640x480 and 1280x720, by value
    (set_frame) and from the camera table (track_cameras, a graph replay); with parent_lib, both launches on default
    device frames against the other library's, alternated call by call."""
    mesh = synth.make_mesh(3, tex_seed=0, tex_size=256)
    e = engine([mesh])
    par = _parent_ctx(parent_lib, mesh) if parent_lib else None
    by_value = lambda s: "frame_prep_kernel<false" in s and "FrameFmtDev" in s
    table = lambda s: "frame_prep_kernel<true" in s and "FrameFmtDev" in s
    out = {}
    for H, W in SIZES:
        cam = sensor_frames(mesh, H, W, 1)[0]
        bgr, u16 = cam["frames"][0]
        rgb = np.ascontiguousarray(bgr[..., ::-1])
        row = dict(by_value={}, camera_table={})
        pose = torch.from_numpy(cam["pose"][None]).cuda()
        for name, order, is_u16, pitched in PROFILE_FORMATS:
            img = rgb if order == "rgb" else bgr
            if order == "bgra":
                img = np.concatenate([bgr, np.full((H, W, 1), 255, np.uint8)], -1)
            d = u16 if is_u16 else u16.astype(np.float32) * np.float32(SCALE)
            pad = 64 if pitched else 0
            big_c = np.zeros((H, W + pad, img.shape[2]), np.uint8)
            big_c[:, :W] = img
            big_d = np.zeros((H, W + pad), d.dtype)
            big_d[:, :W] = d
            # device frames: the launch, not the upload
            c_arg = Color(torch.from_numpy(big_c).cuda()[:, :W], order)
            d_arg = Depth(torch.from_numpy(big_d).cuda()[:, :W], SCALE if is_u16 else None)
            row["by_value"][name] = _alternated([lambda: e.set_frame(c_arg, d_arg, cam["K"])], n, [by_value])[0]
            row["camera_table"][name] = _alternated([lambda: e.track_cameras([(c_arg, d_arg, cam["K"])], pose, [0], [0], 2)],
                                                    n, [table])[0]
        if par:
            lib, ctx = par
            r_dev = torch.from_numpy(rgb).cuda()
            d_dev = torch.from_numpy(u16.astype(np.float32) * np.float32(SCALE)).cuda()
            Kf = (C.c_float * 9)(*cam["K"].reshape(-1))
            st = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
            p_in = pose[0].contiguous()
            p_out = torch.empty(4, 4, device="cuda")

            def par_set_frame():
                assert lib.fp_set_frame(ctx, C.c_void_p(r_dev.data_ptr()), C.c_void_p(d_dev.data_ptr()), Kf, H, W, 3,
                                        float("inf"), st()) == 0

            def par_track():
                assert lib.fp_track(ctx, C.c_void_p(r_dev.data_ptr()), C.c_void_p(d_dev.data_ptr()), Kf, H, W,
                                    C.c_void_p(p_in.data_ptr()), 2, C.c_void_p(p_out.data_ptr()), None, st()) == 0

            old_bv = lambda s: "frame_prep_kernel<false>" in s and "FrameFmtDev" not in s
            old_tb = lambda s: "frame_prep_kernel<true>" in s and "FrameFmtDev" not in s
            parent, this = _alternated([par_set_frame, lambda: e.set_frame(r_dev, d_dev, cam["K"])], n, [old_bv, by_value])
            row["default_by_value_vs_parent"] = dict(parent_us=parent, this_us=this)
            parent, this = _alternated([par_track, lambda: e.track(r_dev, d_dev, cam["K"], pose[0], 2)], n, [old_tb, table])
            row["default_camera_table_vs_parent"] = dict(parent_us=parent, this_us=this)
        out[f"{W}x{H}"] = row
    if par:
        par[0].fp_destroy(par[1])
    e.close()
    return out


def device_leg(e, mesh, n_calls):
    """Device frames (CUDA tensors read in place), one object per camera at 640x480, blocking: BGR8 + uint16 converted on
    the device with torch (channel flip, float multiply) before each call, against the same tensors wrapped."""
    rows = []
    all_cams = sensor_frames(mesh, 480, 640, 4)
    for cam in all_cams:
        cam["dev"] = [(torch.from_numpy(b).cuda(), torch.from_numpy(u).cuda()) for b, u in cam["frames"]]
    for n in (1, 4):
        cams = all_cams[:n]
        pose = {r: torch.from_numpy(np.stack([c["pose"] for c in cams])).cuda() for r in ("convert", "native")}
        times = dict(convert=[], native=[])
        for t in range(4 + n_calls):
            for recipe in (("convert", "native") if t % 2 == 0 else ("native", "convert")):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                views = []
                for cam in cams:
                    bgr, u16 = cam["dev"][t % N_UNIQUE]
                    if recipe == "convert":
                        views.append((bgr.flip(-1).contiguous(), u16.float() * SCALE, cam["K"]))
                    else:
                        views.append((Color(bgr, "bgr"), Depth(u16, SCALE), cam["K"]))
                pose[recipe], _ = e.track_cameras(views, pose[recipe], list(range(n)), [0] * n, 2)
                dt = (time.perf_counter() - t0) * 1e3
                if t >= 4:
                    times[recipe].append(dt)
        row = dict(frame="640x480", cameras=n, convert_blocking=stats(times["convert"]), native_blocking=stats(times["native"]))
        rows.append(row)
        print(json.dumps(dict(device=row)), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--register-calls", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--profile-only", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frame_formats needs a CUDA device")
    if args.profile_only:
        print(json.dumps(dict(profile=profile_leg(args.parent_lib))), flush=True)
        return
    print(json.dumps(dict(card=card())), flush=True)
    mesh = synth.make_mesh(4, tex_seed=0, tex_size=512)
    e = engine([mesh])
    rows = track_leg(e, mesh, args.calls)
    dev = device_leg(e, mesh, args.calls)
    reg = register_leg(e, mesh, args.register_calls)
    e.close()
    cmd = [sys.executable, os.path.abspath(__file__), "--profile-only"] + (["--parent-lib", args.parent_lib] if args.parent_lib else [])
    q = subprocess.run(cmd, capture_output=True, text=True)
    prof = None
    for line in q.stdout.splitlines():
        if line.startswith('{"profile"'):
            prof = json.loads(line)["profile"]
    if prof is None:
        sys.stderr.write(q.stdout[-2000:] + q.stderr[-4000:])
    out = dict(card=card(), objects_per_camera=1, iterations=2, depth_scale=SCALE, calls=args.calls, track_cameras=rows,
               track_cameras_device=dev, register_objects=reg, frame_prep_gpu_us=prof)
    print(json.dumps(out), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
