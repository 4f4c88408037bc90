"""Device time of fp_pose_errors (ADD + ADD-S, and ADD alone) over N in {1, 252, 4096} poses x P in {2620, 10000} model
points, beside the reference's host method (one scipy cKDTree per pose, `query(workers=-1)`) over the same inputs.

    python tools/bench_pose_errors.py [--seconds 0.5]

Per cell: mean ms per call from CUDA events around back-to-back launches (after two warm-up calls, enough launches
for about --seconds of device time), point-pair distances per second (N P^2), and the share of the data sheet's
67 TFLOP/s FP32 of the H100 SXM, counting 8 flops per pair (3 subtractions, 1 multiply, 2 fused multiply-adds).  The
nearest-neighbour search is FP32-issue bound: it reads each tile from shared memory once per four queries and touches
no other memory.  The host column times cKDTree build + query on up to 16 poses and reports ms per pose.  Prints one
JSON line, with the name and power limit of the GPU."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
from scipy.spatial import cKDTree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

PEAK_FP32 = 67e12  # H100 SXM data sheet, dense FP32, at up to 700 W
FLOPS_PER_PAIR = 8


def _inputs(N, P, seed=0):
    from scipy.spatial.transform import Rotation

    rng = np.random.default_rng(seed)
    pts = (rng.normal(size=(P, 3)) * [0.05, 0.03, 0.09]).astype(np.float32)
    pred = np.repeat(np.eye(4)[None], N, axis=0)
    pred[:, :3, :3] = Rotation.random(N, random_state=seed).as_matrix()
    pred[:, :3, 3] = [0.0, 0.0, 0.6] + rng.uniform(-0.02, 0.02, size=(N, 3))
    gt = np.eye(4)
    gt[:3, 3] = [0.0, 0.0, 0.6]
    return pts, pred.astype(np.float32), gt.astype(np.float32)


def _device_ms(fn, seconds):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    reps = max(3, min(2000, int(seconds / max(time.perf_counter() - t0, 1e-6))))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps, reps


def _host_ms_per_pose(pts, pred, gt, n_max=16):
    p64, g = pts.astype(np.float64), gt.astype(np.float64)
    gt_pts = p64 @ g[:3, :3].T + g[:3, 3]
    n = min(n_max, len(pred))
    t0 = time.perf_counter()
    for p in pred[:n].astype(np.float64):
        cKDTree(p64 @ p[:3, :3].T + p[:3, 3]).query(gt_pts, k=1, workers=-1)
    return (time.perf_counter() - t0) * 1e3 / n


def main():
    from bench import device_info

    from foundationpose_b200 import _lib
    from foundationpose_b200._lib import lib

    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5, help="device time per cell")
    opt = ap.parse_args()
    assert torch.cuda.is_available(), "bench_pose_errors.py measures the GPU: it needs a CUDA device"
    dev = torch.device("cuda", torch.cuda.current_device())
    cells = []
    for P in (2620, 10000):
        for N in (1, 252, 4096):
            pts, pred, gt = _inputs(N, P)
            d_pts = torch.as_tensor(pts, device=dev)
            d_pred = torch.as_tensor(pred, device=dev).reshape(N, 16)
            d_gt = torch.as_tensor(gt, device=dev).reshape(1, 16)
            add, adds = torch.empty(N, device=dev), torch.empty(N, device=dev)
            st = torch.cuda.current_stream(dev).cuda_stream

            def call(with_adds):
                return lambda: _lib.check(lib.fp_pose_errors(d_pts.data_ptr(), P, d_pred.data_ptr(), N, d_gt.data_ptr(), 1,
                                                             add.data_ptr(), adds.data_ptr() if with_adds else None, st))

            ms, reps = _device_ms(call(True), opt.seconds)
            ms_add, reps_add = _device_ms(call(False), opt.seconds)
            pairs = float(N) * P * P
            cell = {"N": N, "P": P, "add_adds_ms": ms, "launches": reps, "pairs_per_s": pairs / (ms * 1e-3),
                    "fp32_share_of_67_tflops": pairs * FLOPS_PER_PAIR / (ms * 1e-3) / PEAK_FP32,
                    "add_only_ms": ms_add, "add_only_launches": reps_add,
                    "host_ckdtree_ms_per_pose": _host_ms_per_pose(pts, pred, gt)}
            cell["host_ckdtree_ms_all_poses"] = cell["host_ckdtree_ms_per_pose"] * N
            cells.append(cell)
            print(f"N={N:5d} P={P:6d}  ADD+ADD-S {ms:9.3f} ms  {cell['pairs_per_s'] / 1e12:6.2f} Tpairs/s  "
                  f"{100 * cell['fp32_share_of_67_tflops']:5.1f}% of 67 TFLOP/s  | ADD alone {ms_add:7.4f} ms  | "
                  f"cKDTree {cell['host_ckdtree_ms_per_pose']:.2f} ms/pose", file=sys.stderr)
    print(json.dumps({"cells": cells, "device": device_info(dev.index), "host_cpus": os.cpu_count(),
                      "flops_per_pair": FLOPS_PER_PAIR, "peak_fp32_flops": PEAK_FP32,
                      "bound": "FP32 issue (nearest-neighbour search); ADD alone: launch / memory"}))


if __name__ == "__main__":
    main()
