"""CPU references of fp_vsd_errors: a full-frame depth render with the oracle's coverage rule (oracle/raster.py's
projection, edge test and homogeneous path, the same per-face loop on an H x W raster with umin = vmin = 0 and scale 1)
and a float64 restatement of BOP's VSD (visib_mode 'bop19', cost 'step') from depth images."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.raster import _edge_ok, _hom_cover, _project  # noqa: E402

f32 = np.float32


def render_depth(pose, verts, faces, K, H, W, znear=0.001, zfar=100.0):
    """Camera-Z depth (H, W) float32 of the mesh at `pose`, 0 where nothing is covered: 1 / the interpolated 1/Z of
    the winning fragment, as the GPU reads it from its depth key."""
    X, Y, Z, iz, xi, yi = _project(np.asarray(pose, dtype=f32), np.asarray(verts), K, f32(0), f32(0), f32(1), f32(1))
    best = np.zeros((H, W), dtype=f32)
    iz_far = f32(1.0) / f32(zfar)
    ray_x = ((((np.arange(W, dtype=f32) + f32(0.5)) / f32(1)).astype(f32) - f32(K[0, 2])) / f32(K[0, 0])).astype(f32)
    ray_y = ((((np.arange(H, dtype=f32) + f32(0.5)) / f32(1)).astype(f32) - f32(K[1, 2])) / f32(K[1, 1])).astype(f32)
    for i0, i1, i2 in np.asarray(faces):
        nfront = int(Z[i0] > znear) + int(Z[i1] > znear) + int(Z[i2] > znear)
        if nfront == 0:
            continue
        if nfront < 3:
            dy, dx = np.meshgrid(ray_y, ray_x, indexing="ij")
            inside, _, izp = _hom_cover((X[i0], Y[i0], Z[i0]), (X[i1], Y[i1], Z[i1]), (X[i2], Y[i2], Z[i2]), dx, dy, znear, zfar)
            if inside is None or not inside.any():
                continue
            win = inside & (izp.view(np.uint32) > best.view(np.uint32))
            best[win] = izp[win]
            continue
        x0, y0, x1, y1, x2, y2 = int(xi[i0]), int(yi[i0]), int(xi[i1]), int(yi[i1]), int(xi[i2]), int(yi[i2])
        area2 = (x1 - x0) * (y2 - y0) - (y1 - y0) * (x2 - x0)
        if area2 == 0:
            continue
        swapped = area2 < 0
        if swapped:
            x1, y1, x2, y2 = x2, y2, x1, y1
            area2 = -area2
        j0 = max((min(x0, x1, x2) + 127) >> 8, 0)
        j1 = min((max(x0, x1, x2) - 128) >> 8, W - 1)
        r0 = max((min(y0, y1, y2) + 127) >> 8, 0)
        r1 = min((max(y0, y1, y2) - 128) >> 8, H - 1)
        if j0 > j1 or r0 > r1:
            continue
        py, px = np.meshgrid(np.arange(r0, r1 + 1) * 256 + 128, np.arange(j0, j1 + 1) * 256 + 128, indexing="ij")
        e0 = (x2 - x1) * (py - y1) - (y2 - y1) * (px - x1)
        e1 = (x0 - x2) * (py - y2) - (y0 - y2) * (px - x2)
        e2 = area2 - e0 - e1
        inside = _edge_ok(e0, x2 - x1, y2 - y1) & _edge_ok(e1, x0 - x2, y0 - y2) & _edge_ok(e2, x1 - x0, y1 - y0)
        if not inside.any():
            continue
        fa = f32(area2)
        b0 = (e0.astype(f32) / fa).astype(f32)
        w1 = (e1.astype(f32) / fa).astype(f32)
        w2 = (e2.astype(f32) / fa).astype(f32)
        b1, b2 = (w2, w1) if swapped else (w1, w2)
        izp = ((b0 * iz[i0] + b1 * iz[i1]) + b2 * iz[i2]).astype(f32)
        sub = best[r0:r1 + 1, j0:j1 + 1]
        win = inside & (izp > iz_far) & (izp.view(np.uint32) > sub.view(np.uint32))
        sub[win] = izp[win]
    with np.errstate(divide="ignore"):
        return np.where(best > 0, f32(1) / best, f32(0)).astype(f32)


def dist_scale(K, H, W):
    """sqrt(((u - cx) / fx)^2 + ((v - cy) / fy)^2 + 1) at integer u, v, float64 from the float32 intrinsics."""
    k = np.asarray(K, dtype=f32).astype(np.float64)
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    a = (u - k[0, 2]) / k[0, 0]
    b = (v - k[1, 2]) / k[1, 1]
    return np.sqrt((a * a + b * b) + 1.0)


def vsd_counts(dE, dG, D, K, delta, taus, margin=1e-6):
    """float64 VSD from depth images: (counts [T + 2] int64 = union, intersection, c_0 .. c_{T-1}; errors [T];
    number of pixels within `margin` metres of a delta or tau decision)."""
    H, W = D.shape
    s = dist_scale(K, H, W)
    dE, dG, D = (np.asarray(x, dtype=f32).astype(np.float64) for x in (dE, dG, D))
    tT, tE, tG = D * s, dE * s, dG * s
    delta = float(np.float32(delta))
    taus = np.asarray(taus, dtype=f32).astype(np.float64).reshape(-1)
    vG = ((tG - tT <= delta) | (D == 0)) & (dG > 0)
    vE = (((tE - tT <= delta) | (D == 0)) & (dE > 0)) | (vG & (dE > 0))
    both = vG & vE
    union, inter = int((vG | vE).sum()), int(both.sum())
    diff = np.abs(tG - tE)[both]
    c = np.array([(diff >= t).sum() for t in taus], dtype=np.int64)
    near = (np.abs(tG - tT - delta) < margin) & (dG > 0) & (D > 0)
    near |= (np.abs(tE - tT - delta) < margin) & (dE > 0) & (D > 0)
    n_near = int(near.sum()) + int(sum((np.abs(diff - t) < margin).sum() for t in taus))
    errs = np.ones(len(taus)) if union == 0 else (c + (union - inter)) / union
    return np.concatenate([[union, inter], c]).astype(np.int64), errs, n_near


def vsd_errors(verts, faces, pred, gt, D, K, delta, taus):
    """Per pose: the float64 VSD of the oracle's renders, (counts, errors, near-boundary pixels)."""
    H, W = D.shape
    dE = render_depth(pred, verts, faces, K, H, W)
    dG = render_depth(gt, verts, faces, K, H, W)
    return vsd_counts(dE, dG, D, K, delta, taus)
