"""Device time of fp_sym_pose_errors (MSSD + MSPD together) over N in {252, 4096} poses x S in {1, 315, 1260}
symmetries x P in {2620, 10000} model points, beside a float64 numpy restatement of the definitions on the host.

    python tools/bench_sym_pose_errors.py [--seconds 0.3]

Per cell: mean ms per call from CUDA events around back-to-back launches (after two warm-up calls, enough launches
for about --seconds of device time), point pairs per second (N S P) and the share of the data sheet's 67 TFLOP/s FP32
of the H100 SXM, counting 45 flops per pair: the transform by G s (9 fused multiply-adds), the MSSD distance (3
subtractions, 1 multiply, 2 fused multiply-adds) and the MSPD distance (6 fused multiply-adds for the numerators, 2
multiplies by the reciprocal depth, 2 subtractions, 1 multiply, 1 fused multiply-add); the reciprocal and the maxima
are not counted.  The host column runs the numpy restatement (symmetries in chunks of 64) on 16 poses and reports ms
per pose.  Prints one JSON line, with the name and power limit of the GPU."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

PEAK_FP32 = 67e12  # H100 SXM data sheet, dense FP32, at up to 700 W
FLOPS_PER_PAIR = 45
K = np.array([[615.0, 0.0, 320.0], [0.0, 615.0, 240.0], [0.0, 0.0, 1.0]], dtype=np.float32)
CONT = {"axis": [0.0, 0.0, 1.0], "offset": [0.0, 0.0, 0.0]}
DISC = [np.diag(d).reshape(-1).tolist() for d in ([1.0, -1.0, -1.0, 1.0], [-1.0, 1.0, -1.0, 1.0], [-1.0, -1.0, 1.0, 1.0])]


def _symmetries(S):
    from foundationpose_b200 import metrics

    info = {1: {}, 315: {"symmetries_continuous": [CONT]}, 1260: {"symmetries_continuous": [CONT], "symmetries_discrete": DISC}}
    syms = metrics.bop_symmetries(info[S])
    assert len(syms) == S
    return syms.astype(np.float32)


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


def host_errors(pts, pred, gt, syms, k):
    """float64 numpy: (MSSD, MSPD) of every pose in `pred`."""
    pts, syms, g, k = pts.astype(np.float64), syms.astype(np.float64), gt.astype(np.float64), k.astype(np.float64)
    out = []
    for e in pred.astype(np.float64):
        ep = pts @ e[:3, :3].T + e[:3, 3]
        eu = (ep @ k.T)[:, :2] / ep[:, 2:3]
        w3, w2 = np.inf, np.inf
        for c in range(0, len(syms), 64):
            gs = g[None] @ syms[c:c + 64]
            q = np.einsum("sij,pj->spi", gs[:, :3, :3], pts) + gs[:, None, :3, 3]
            qu = (q @ k.T)[..., :2] / q[..., 2:3]
            w3 = min(w3, np.linalg.norm(ep[None] - q, axis=-1).max(1).min())
            w2 = min(w2, np.linalg.norm(eu[None] - qu, axis=-1).max(1).min())
        out.append((w3, w2))
    return out


def main():
    from bench import device_info

    from foundationpose_b200 import _lib
    from foundationpose_b200._lib import lib

    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.3, help="device time per cell")
    ap.add_argument("--host_poses", type=int, default=16, help="poses of the host restatement per (S, P)")
    opt = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sym_pose_errors.py measures the GPU: it needs a CUDA device"
    dev = torch.device("cuda", torch.cuda.current_device())
    st = torch.cuda.current_stream(dev).cuda_stream
    cells, host = [], {}
    for P in (2620, 10000):
        for S in (1, 315, 1260):
            syms = _symmetries(S)
            pts, pred, gt = _inputs(opt.host_poses, P)
            t0 = time.perf_counter()
            want = host_errors(pts, pred, gt, syms, K)
            host[(S, P)] = (time.perf_counter() - t0) * 1e3 / opt.host_poses
            d_sym = torch.as_tensor(syms, device=dev).reshape(S, 16)
            d_k = torch.as_tensor(K, device=dev).reshape(1, 9)
            for N in (252, 4096):
                pts, pred, gt = _inputs(N, P)
                d_pts = torch.as_tensor(pts, device=dev)
                d_pred = torch.as_tensor(pred, device=dev).reshape(N, 16)
                d_gt = torch.as_tensor(gt, device=dev).reshape(1, 16)
                mssd, mspd = torch.empty(N, device=dev), torch.empty(N, device=dev)

                def call():
                    _lib.check(lib.fp_sym_pose_errors(d_pts.data_ptr(), P, d_pred.data_ptr(), N, d_gt.data_ptr(), 1,
                                                      d_sym.data_ptr(), S, d_k.data_ptr(), 1, mssd.data_ptr(),
                                                      mspd.data_ptr(), st))

                ms, reps = _device_ms(call, opt.seconds)
                # the first host poses are the first device poses: the two agree
                n = opt.host_poses
                got3, got2 = mssd[:n].double().cpu().numpy(), mspd[:n].double().cpu().numpy()
                w3, w2 = np.array([w[0] for w in want]), np.array([w[1] for w in want])
                pairs = float(N) * S * P
                cell = {"N": N, "S": S, "P": P, "mssd_mspd_ms": ms, "launches": reps, "pairs_per_s": pairs / (ms * 1e-3),
                        "fp32_share_of_67_tflops": pairs * FLOPS_PER_PAIR / (ms * 1e-3) / PEAK_FP32,
                        "host_numpy_ms_per_pose": host[(S, P)], "host_numpy_ms_all_poses": host[(S, P)] * N,
                        "max_abs_diff_mssd_m": float(np.abs(got3 - w3).max()),
                        "max_abs_diff_mspd_px": float(np.abs(got2 - w2).max())}
                cells.append(cell)
                print(f"N={N:5d} S={S:5d} P={P:6d}  MSSD+MSPD {ms:9.3f} ms  {cell['pairs_per_s'] / 1e12:6.3f} Tpairs/s  "
                      f"{100 * cell['fp32_share_of_67_tflops']:5.1f}% of 67 TFLOP/s  | numpy "
                      f"{host[(S, P)]:9.2f} ms/pose  | |diff| {cell['max_abs_diff_mssd_m']:.1e} m "
                      f"{cell['max_abs_diff_mspd_px']:.1e} px", file=sys.stderr)
    print(json.dumps({"cells": cells, "device": device_info(dev.index), "host_cpus": os.cpu_count(),
                      "flops_per_pair": FLOPS_PER_PAIR, "peak_fp32_flops": PEAK_FP32,
                      "bound": "FP32 issue (one transform and two distances per point pair)"}))


if __name__ == "__main__":
    main()
