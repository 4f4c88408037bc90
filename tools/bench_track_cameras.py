"""Objects of several camera streams tracked on one GPU: `estimater.track_cameras` (one CUDA-graph launch per call for every
camera) against the best path that existed before it, one Engine per camera calling `track_objects` in turn, and against
one shared Engine calling `track_objects` per camera.

    python tools/bench_track_cameras.py [n_frames]

Prints one JSON line: p50 / p99 wall-clock ms per frame (one frame of every camera) of the three paths for C = 1, 2, 4, 8
cameras at 640x480 with 1 and 2 objects per camera (host numpy frames, two refiner passes), the host time of the same
copies into pinned buffers that the call makes for its staging, timed on their own, and the name and power limit of the
GPU they were measured on."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True


def track_cameras_leg(n_frames=400, c_values=(1, 2, 4, 8), per_camera=(1, 2)):
    """Each camera is its own recording: its objects on their own walks in front of its own background.  The three paths
    compute the same poses, run on the same frames and alternate frame by frame, so they see the same clocks."""
    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.estimater import FoundationPose, PoseRefinePredictor, ScorePredictor, track_cameras, track_objects
    from foundationpose_b200.weights import random_state_dict

    K = synth.DEFAULT_K
    sd_r, sd_s = random_state_dict("refine", 0), random_state_dict("score", 0)
    n_cam, n_obj = max(c_values), max(per_camera)
    scenes = []  # per camera: meshes, walks, 20 frames
    for c in range(n_cam):
        meshes, seqs = [], []
        for k in range(n_obj):
            scale = 0.6 + 0.1 * ((c + k) % 4)
            meshes.append((synth.make_mesh(3, tex_seed=10 * c + k, tex_size=256, scale=scale), scale))
            p0 = np.eye(4)
            p0[:3, :3] = synth.random_rotation(100 + 10 * c + k)
            p0[:3, 3] = [-0.1 + 0.2 * k, 0.02 * (c % 3 - 1), 0.7]
            seqs.append(synth.track_sequence(20, p0, seed=200 + 10 * c + k))
        frames = [synth.make_multi_scene([(m.visual.image, seqs[k][i], sc) for k, (m, sc) in enumerate(meshes)],
                                         seed=1 + i + 50 * c)[:2] for i in range(20)]
        scenes.append((meshes, seqs, frames))

    def make_estimators(engine_of_camera):
        out, engines = [], {}
        for c, (meshes, _, _) in enumerate(scenes):
            e = engine_of_camera(c)
            if id(e) not in engines:
                engines[id(e)] = (e, PoseRefinePredictor(engine=e, state_dict=sd_r), ScorePredictor(engine=e, state_dict=sd_s))
            _, refiner, scorer = engines[id(e)]
            out.append([FoundationPose(model_pts=m.vertices, model_normals=m.vertex_normals, mesh=m, scorer=scorer, refiner=refiner)
                        for m, _ in meshes])
        return out, [e for e, _, _ in engines.values()]

    shared = Engine()
    multi, e1 = make_estimators(lambda c: shared)
    per_cam_engines = [Engine() for _ in range(n_cam)]
    alone, e2 = make_estimators(lambda c: per_cam_engines[c])
    shared2 = Engine()
    turn, e3 = make_estimators(lambda c: shared2)
    pct = lambda a, q: float(a[min(int(len(a) * q), len(a) - 1)])
    stats = lambda a: {"ms_p50": pct(np.sort(a), 0.5), "ms_p99": pct(np.sort(a), 0.99)}
    # the copies fp_track_cameras makes into its pinned staging, repeated on their own: the same bytes into pinned buffers
    stage = [(torch.empty(480, 640, 3, dtype=torch.uint8).pin_memory().numpy(),
              torch.empty(480, 640, dtype=torch.float32).pin_memory().numpy()) for _ in range(n_cam)]
    results = {}
    for n_o in per_camera:
        for C in c_values:
            for ests in (multi, alone, turn):
                for c in range(C):
                    for k in range(n_o):
                        ests[c][k].pose_last = torch.as_tensor(scenes[c][1][k][0], dtype=torch.float32, device="cuda").reshape(1, 4, 4)
            t = {"track_cameras": [], "engine_per_camera": [], "shared_engine_in_turn": [], "host_staging_copies": []}
            for i in range(20 + n_frames):
                k40 = i % 40
                f = k40 if k40 < 20 else 39 - k40  # forwards, then backwards: no jumps
                views = [(multi[c][:n_o], scenes[c][2][f][0], scenes[c][2][f][1], K) for c in range(C)]
                t0 = time.perf_counter()
                track_cameras(views, iteration=2)
                t1 = time.perf_counter()
                for c in range(C):
                    track_objects(alone[c][:n_o], scenes[c][2][f][0], scenes[c][2][f][1], K, iteration=2)
                t2 = time.perf_counter()
                for c in range(C):
                    track_objects(turn[c][:n_o], scenes[c][2][f][0], scenes[c][2][f][1], K, iteration=2)
                t3 = time.perf_counter()
                for c in range(C):
                    rgb, depth = scenes[c][2][f]
                    np.copyto(stage[c][1], depth)
                    np.copyto(stage[c][0], rgb)
                t4 = time.perf_counter()
                if i >= 20:  # the first 20 frames warm up every path (graphs captured)
                    for name, dt in zip(t, (t1 - t0, t2 - t1, t3 - t2, t4 - t3)):
                        t[name].append(dt * 1e3)
            r = {name: stats(v) for name, v in t.items()}
            r["speedup_p50_vs_engine_per_camera"] = r["engine_per_camera"]["ms_p50"] / r["track_cameras"]["ms_p50"]
            r["speedup_p50_vs_shared_engine_in_turn"] = r["shared_engine_in_turn"]["ms_p50"] / r["track_cameras"]["ms_p50"]
            results[f"C={C},objects_per_camera={n_o}"] = r
    for e in e1 + e2 + e3:
        e.close()
    return {"per_config": results, "frames": n_frames, "refine_iters": 2,
            "api": "estimater.track_cameras(views, iteration=2) with host numpy frames: one CUDA-graph launch per call for every "
                   "camera (C uploads, one frame-preparation launch, 2 refiner passes at N = sum of objects, read-back); wall clock "
                   "per call",
            "baselines": {"engine_per_camera": "one Engine per camera, track_objects(...) of each camera in turn",
                          "shared_engine_in_turn": "one Engine, track_objects(...) of each camera in turn"},
            "host_staging_copies": "np.copyto of every camera's depth and rgb into pinned host buffers of its own, timed apart "
                                   "from the call: the same copies fp_track_cameras makes into its pinned staging before the "
                                   "graph launch, measured outside it (a stand-in, not a timer inside the call)",
            "sequence": "per camera: its own 640x480 recording of 1-2 textured ellipsoids on their own walks (<= 5 mm / 2 deg per "
                        "frame); 20 distinct frames played forwards and backwards"}


def main():
    from bench import device_info

    n_frames = int(sys.argv[1]) if len(sys.argv) > 1 else 400
    out = track_cameras_leg(n_frames)
    out["device"] = device_info(torch.cuda.current_device())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
