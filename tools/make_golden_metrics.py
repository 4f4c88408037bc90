"""Golden vectors for the pose-accuracy metrics, produced by the REFERENCE's own `add_err`, `adds_err` and
`compute_auc_sklearn` (Utils.py:232-266).

Utils.py cannot be imported (pytorch3d, nvdiffrast, open3d, ... are absent), so — as tools/make_golden_shim.py does —
the unmodified source of each function, and of `transform_pts` that the first two call, is extracted with `ast` and
executed on the CPU in a namespace holding what it really uses: numpy, scipy's `cKDTree`, sklearn (imported by the
function itself).

    python tools/make_golden_metrics.py      # needs the reference tree; writes tests/golden/metrics_golden.npz

Model points and poses are float32 values (stored as float32, evaluated in float64 by the reference), so the only
difference left to the GPU's fp32 kernel is its arithmetic.  Cases:
  pose/<set>/{pts, pred, gt, add, adds}  a textured-ellipsoid model of `synth`, random point sets of P = 1, 7, 257,
      2 620, 4 099, a set symmetric under a half turn about z and one with duplicated points; each against one
      ground-truth pose with the estimates: identical, a 3 mm translation, a 120 degree rotation, a small rotation +
      8 mm, and (symmetric sets) the half turn about z.
  auc/<case>/{errs, params (max_val, step), auc}  curves that reach 1 early, never reach it (inf included), have
      errors exactly on a step, other max_val / step, one error.
tests/test_metrics_golden_cpu.py (AUC) and tests/test_metrics_gpu.py (ADD / ADD-S) hold the project to these vectors.
"""
import os
import sys

import numpy as np
from scipy.spatial import cKDTree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
REF = os.environ.get("FPOSE_REFERENCE", "/root/reference")


def reference_namespace():
    from make_golden_geometry import extract

    ns = {"np": np, "cKDTree": cKDTree}
    for name in ("transform_pts", "add_err", "adds_err", "compute_auc_sklearn"):
        exec(extract(os.path.join(REF, "Utils.py"), name), ns)
    return ns


def _rot(axis, deg):
    from scipy.spatial.transform import Rotation

    axis = np.asarray(axis, dtype=np.float64)
    return Rotation.from_rotvec(axis / np.linalg.norm(axis) * np.deg2rad(deg)).as_matrix()


def point_sets():
    from foundationpose_b200 import synth

    rng = np.random.default_rng(20)
    scale = np.array([0.05, 0.03, 0.09])
    sets = {"ellipsoid": (synth.make_mesh(3, tex_size=8).vertices, True)}
    for P in (1, 7, 257, 2620, 4099):
        sets[f"random{P}"] = (rng.normal(size=(P, 3)) * scale, False)
    half = rng.normal(size=(1310, 3)) * scale
    sets["halfturn2620"] = (np.concatenate([half, half * np.array([-1.0, -1.0, 1.0])]), True)
    dup = rng.normal(size=(257, 3)) * scale
    dup[128:] = dup[:129]
    sets["duplicated257"] = (dup, False)
    return {k: (np.asarray(v, dtype=np.float32), sym) for k, (v, sym) in sets.items()}


def pose_pairs(symmetric, seed):
    rng = np.random.default_rng(seed)
    gt = np.eye(4)
    gt[:3, :3] = _rot(rng.normal(size=3), rng.uniform(20, 170))
    gt[:3, 3] = [0.02, -0.03, 0.55]
    preds = [gt.copy()]
    p = gt.copy()
    p[:3, 3] += [0.002, -0.001, 0.002]
    preds.append(p)
    p = gt.copy()
    p[:3, :3] = gt[:3, :3] @ _rot(rng.normal(size=3), 120.0)
    preds.append(p)
    p = gt.copy()
    p[:3, :3] = gt[:3, :3] @ _rot(rng.normal(size=3), 5.0)
    p[:3, 3] += [0.008, 0.0, 0.0]
    preds.append(p)
    if symmetric:
        preds.append(gt @ np.diag([-1.0, -1.0, 1.0, 1.0]))
    preds = np.asarray(preds, dtype=np.float32)
    return preds, np.repeat(gt.astype(np.float32)[None], len(preds), axis=0)


def auc_cases(step_grid):
    rng = np.random.default_rng(21)
    return {
        "early": (rng.uniform(0.0, 0.03, 50), 0.1, 0.001),
        "never": (np.concatenate([rng.uniform(0.0, 0.2, 40), [np.inf]]), 0.1, 0.001),
        "on_step": (step_grid[[0, 3, 3, 17, 50, 99]], 0.1, 0.001),
        "other_grid": (rng.uniform(0.0, 0.06, 30), 0.05, 0.0005),
        "single": (np.array([0.0]), 0.1, 0.001),
    }


def main():
    ns = reference_namespace()
    out = {}
    for i, (name, (pts, sym)) in enumerate(point_sets().items()):
        pred, gt = pose_pairs(sym, seed=100 + i)
        p64 = pts.astype(np.float64)
        out[f"pose/{name}/pts"] = pts
        out[f"pose/{name}/pred"] = pred
        out[f"pose/{name}/gt"] = gt
        out[f"pose/{name}/add"] = np.array([ns["add_err"](a.astype(np.float64), b.astype(np.float64), p64) for a, b in zip(pred, gt)])
        out[f"pose/{name}/adds"] = np.array([ns["adds_err"](a.astype(np.float64), b.astype(np.float64), p64) for a, b in zip(pred, gt)])
        if sym:
            assert out[f"pose/{name}/adds"][-1] < 1e-6, f"{name} is not symmetric under the half turn"
        print(f"{name:14s} P={len(pts):5d}  ADD {np.array2string(out[f'pose/{name}/add'], precision=5)}  "
              f"ADD-S {np.array2string(out[f'pose/{name}/adds'], precision=5)}")
    for name, (errs, max_val, step) in auc_cases(np.arange(0, 0.1 + 0.001, 0.001)).items():
        out[f"auc/{name}/errs"] = np.asarray(errs, dtype=np.float64)
        out[f"auc/{name}/params"] = np.array([max_val, step])
        out[f"auc/{name}/auc"] = np.float64(ns["compute_auc_sklearn"](errs, max_val=max_val, step=step))
        print(f"auc {name:10s} {out[f'auc/{name}/auc']:.12f}")
    dst = os.path.join(ROOT, "tests", "golden", "metrics_golden.npz")
    np.savez_compressed(dst, **out)
    print(f"wrote {dst}: {len(out)} entries, {os.path.getsize(dst) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
