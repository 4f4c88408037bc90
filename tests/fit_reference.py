"""Host reference of the tracking calls' fit counts (FP_FIT_COUNTS, include/fpose.h), built on the exact crop reference
(tests/crop_reference.py): at each pose, over the refiner's 160 x 160 crop window, the winning face of every crop pixel
(exact coverage), its rendered camera z in float64 and the observed z the refiner's B side reads at the same pixel (the
z of the nearest xyz-map sample, 0 outside the frame), then the five counts.

The kernel computes z_r and d = z_o - z_r in fp32; here both are float64, so a pixel may be counted differently only
where |d| lies within a few ulps of delta.  near_delta() counts those pixels."""
import numpy as np
import torch

import crop_reference as cr

NAMES = ("covered", "valid", "inlier", "occluded", "behind")


def depths(scene, poses):
    """(covered (N,S,S) bool, z_r (N,S,S) float64 rendered camera z (0 where uncovered), z_o (N,S,S) float64)."""
    res = scene.run(poses, mode=0)
    face, bary = res["face"], res["bary"]
    P = torch.as_tensor(np.asarray(poses, dtype=np.float32), device=scene.dev)
    win = scene._win_t(res["win"])
    _, _, Z, iz, _, _ = scene.project(P, win)
    n = len(P)
    covered = face >= 0
    zr = torch.zeros(n, cr.S, cr.S, dtype=torch.float64, device=scene.dev)
    pi, r, j = torch.nonzero(covered, as_tuple=True)
    if len(pi):
        vid = scene.faces[face[pi, r, j]]
        Zv, izv = Z[pi[:, None], vid].double(), iz[pi[:, None], vid].double()
        b = bary[pi, r, j].double()
        planar = (Zv > cr.ZNEAR).all(1)
        # planar: screen-space barycentrics, z = 1 / interpolated 1/Z; near-plane path: perspective-correct weights
        zr[pi, r, j] = torch.where(planar, 1.0 / (b * izv).sum(1), (b * Zv).sum(1))
    tb = scene.taps(win)
    cn, rn = tb["col"]["n"], tb["row"]["n"]
    inside = (cn[:, None, :] >= 0) & (rn[:, :, None] >= 0)
    zmap = scene.xyz[..., 2]
    zo = torch.where(inside, zmap[rn.clamp(min=0)[:, :, None], cn.clamp(min=0)[:, None, :]], 0.0).double()
    return covered, zr, zo


def counts_of(covered, zr, zo, delta):
    """The five counts (N,5) int64 from depths()."""
    d = zo - zr
    valid = covered & (zo >= float(np.float32(0.001)))
    c = [covered, valid, valid & (d.abs() <= delta), valid & (d < -delta), valid & (d > delta)]
    return torch.stack([x.flatten(1).sum(1) for x in c], 1).cpu().numpy()


def near_delta(covered, zr, zo, delta, tol=1e-6):
    """Per pose: valid pixels whose |d| lies within tol of delta (where fp32 and float64 may classify differently)."""
    d = zo - zr
    valid = covered & (zo >= float(np.float32(0.001)))
    return (valid & ((d.abs() - delta).abs() <= tol)).flatten(1).sum(1).cpu().numpy()


def counts(scene, poses, delta):
    return counts_of(*depths(scene, poses), delta)

