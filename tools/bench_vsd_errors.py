"""Device time of fp_vsd_errors (BOP's VSD, 10 taus) on the synthetic ellipsoid at subdivision 5 (20 480 faces), beside
the float64 numpy restatement over the oracle's full-frame renders (tests/vsd_reference.py) timed per pose on the host.

    python tools/bench_vsd_errors.py [--seconds 0.5] [--host-poses 2]

Workloads, both 640 x 480:
  register   the 252 hypotheses of one register call (poses within 30 degrees and 2 cm of the ground truth) against one
             test depth frame, one ground truth and one K (broadcast);
  dataset    1 024 poses, each with its own ground truth, K and 640 x 480 test depth frame (a dataset-evaluation batch;
             the 1 024 frames, 1.26 GB, are on the device before the timing).
Per workload: mean ms per call from CUDA events around back-to-back calls (after two warm-up calls), poses per second,
and the host restatement's seconds per pose.  A call includes the host meshlet build and the upload of the mesh.
Prints one JSON line, with the name and power limit of the GPU read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
sys.dont_write_bytecode = True

K = np.array([[615.0, 0.0, 320.0], [0.0, 615.0, 240.0], [0.0, 0.0, 1.0]], dtype=np.float32)
H, W = 480, 640


def _poses(rng, n, t, rot_deg, trans):
    from scipy.spatial.transform import Rotation

    out = np.repeat(np.eye(4)[None], n, axis=0)
    rv = rng.normal(size=(n, 3))
    rv *= (np.deg2rad(rot_deg) * rng.uniform(0, 1, size=(n, 1))) / np.linalg.norm(rv, axis=1, keepdims=True)
    out[:, :3, :3] = Rotation.from_rotvec(rv).as_matrix()
    out[:, :3, 3] = np.asarray(t) + rng.uniform(-trans, trans, size=(n, 3))
    return out.astype(np.float32)


def _device_ms(fn, seconds):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    reps = max(3, min(500, int(seconds / max(time.perf_counter() - t0, 1e-6))))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps, reps


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--host-poses", type=int, default=2)
    opt = ap.parse_args()
    import vsd_reference as ref

    from foundationpose_b200 import metrics, synth

    rng = np.random.default_rng(0)
    mesh = synth.make_mesh(5)
    v, f = mesh.vertices.astype(np.float32), mesh.faces.astype(np.int32)
    diameter = float(synth.mesh_diameter(mesh.vertices))
    gt = _poses(rng, 1, (0.0, 0.0, 0.6), 180.0, 0.0)[0]
    _, D, _ = synth.make_multi_scene([(mesh.visual.image, gt.astype(np.float64), 1.0)], K)
    hyps = _poses(rng, 252, gt[:3, 3], 30.0, 0.02) @ np.eye(4, dtype=np.float32)
    hyps[:, :3, :3] = hyps[:, :3, :3] @ gt[:3, :3]
    dev = torch.device("cuda", 0)
    out = {}
    # register: 252 hypotheses, one frame
    Dd, Kd = torch.as_tensor(D, device=dev), torch.as_tensor(K, device=dev)
    hd, gd = torch.as_tensor(hyps, device=dev), torch.as_tensor(gt, device=dev)
    ms, reps = _device_ms(lambda: metrics.vsd_errors(v, f, hd, gd, Dd, Kd, diameter), opt.seconds)
    out["register_252"] = {"ms_per_call": round(ms, 4), "poses_per_s": round(252 / ms * 1e3, 1), "reps": reps}
    # dataset: 1 024 poses with their own frames
    n = 1024
    gts = _poses(rng, n, (0.0, 0.0, 0.6), 180.0, 0.05)
    preds = gts.copy()
    preds[:, :3, 3] += rng.uniform(-0.01, 0.01, size=(n, 3)).astype(np.float32)
    Dn = torch.empty(n, H, W, device=dev)
    noise = torch.randn(H, W, device=dev) * 0.002
    for i in range(0, n, 64):  # 16 distinct synthetic frames shifted per pose: 1 024 distinct depth images
        _, d_i, _ = synth.make_multi_scene([(mesh.visual.image, gts[i].astype(np.float64), 1.0)], K, seed=i)
        base = torch.as_tensor(d_i, device=dev)
        for j in range(i, min(n, i + 64)):
            Dn[j] = base + noise.roll(j, 1)
    Kn = torch.as_tensor(np.repeat(K[None], n, 0), device=dev)
    pd, gdn = torch.as_tensor(preds, device=dev), torch.as_tensor(gts, device=dev)
    ms, reps = _device_ms(lambda: metrics.vsd_errors(v, f, pd, gdn, Dn, Kn, diameter), opt.seconds)
    out["dataset_1024"] = {"ms_per_call": round(ms, 4), "poses_per_s": round(n / ms * 1e3, 1), "reps": reps}
    # host: float64 restatement over the oracle renders, per pose
    taus = (metrics.VSD_TAUS * diameter).astype(np.float32)
    t0 = time.perf_counter()
    for i in range(opt.host_poses):
        ref.vsd_errors(v, f, hyps[i], gt, D, K, 0.015, taus)
    host = (time.perf_counter() - t0) / opt.host_poses
    out["host_s_per_pose"] = round(host, 3)
    name, power = _gpu_info()
    print(json.dumps({"gpu": name, "power_limit": power, "mesh_faces": int(len(f)), "frame": [W, H], **out}))


if __name__ == "__main__":
    main()
