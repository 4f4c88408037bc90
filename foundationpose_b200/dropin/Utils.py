"""`from Utils import *` for the reference's unmodified drivers (SURVEY.md Appendix C): the module-level names
run_demo.py / run_ycb_video.py / run_linemod.py use unqualified, on top of libfpose.so.

Only the surface the drivers touch is provided (the reference's Utils.py is 1000 lines of training / NeRF helpers):
  imports        os, sys, time, np, torch, nn, F, cv2, glob, logging, copy, math, itertools, uuid, json, trimesh,
                 imageio, dr (nvdiffrast.torch stand-in)                                        (Utils.py:10-37)
  logging / rng  set_logging_format (Utils.py:94-99), set_seed (Utils.py:222-229)
  geometry       depth2xyzmap (:399-417), depth2xyzmap_batch (:420-438), to_homo (:511-517), transform_pts (:529-537),
                 glcam_in_cvcam (:66), compute_mesh_diameter (:559-574, exact instead of sampled), sample_views_icosphere
                 (:483-507), make_mesh_tensors (:104-130), erode_depth / bilateral_filter_depth (:304-395, on the GPU)
  drawing        project_3d_to_2d (:667-672), draw_xyz_axis (:675-710), draw_posed_3d_box (:713-750)
  clouds         toOpen3dCloud (:280-289) — needs open3d, which only debug >= 2 / 3 paths call
  dataset runs   argparse, NestDict (:60-61), make_yaml_dumpable (:996-1020), symmetry_tfs_from_info (:806-834),
                 euler_matrix (the `transformations` package's static-xyz convention), wp (warp stand-in: force_load)
                 — what run_linemod.py / run_ycb_video.py and the BOP readers use unqualified
  pose accuracy  add_err (:232-240), adds_err (:243-253) — on the GPU (fp_pose_errors), fp32 —, compute_auc_sklearn
                 (:256-266, without sklearn)
trimesh and imageio are the real packages when installed, else the minimal stand-ins under _fallback/.
"""
import argparse  # noqa: F401
import copy  # noqa: F401
import glob  # noqa: F401
import importlib
import itertools  # noqa: F401
import json  # noqa: F401
import logging
import math  # noqa: F401
import os
import sys
import time  # noqa: F401
import uuid  # noqa: F401
from collections import OrderedDict, defaultdict  # noqa: F401

import cv2
import numpy as np
import torch
import torch.nn as nn  # noqa: F401
import torch.nn.functional as F  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
if _ROOT not in sys.path:
    sys.path.append(_ROOT)


def _import_or_fallback(name):
    try:
        return importlib.import_module(name)
    except ImportError:
        fb = os.path.join(_HERE, "_fallback")
        if fb not in sys.path:
            sys.path.append(fb)
        return importlib.import_module(name)


trimesh = _import_or_fallback("trimesh")
imageio = _import_or_fallback("imageio")
import nvdiffrast.torch as dr  # noqa: E402,F401  (dropin/nvdiffrast unless the real one is installed)

try:  # only the debug >= 2 / 3 point-cloud dumps need it
    import open3d as o3d  # noqa: F401
except ImportError:
    o3d = None

from foundationpose_b200 import hypotheses as _hyp  # noqa: E402
from foundationpose_b200 import meshprep as _meshprep  # noqa: E402
from foundationpose_b200 import metrics as _metrics  # noqa: E402
from foundationpose_b200.estimater import make_mesh_tensors  # noqa: E402,F401



class _WarpStandIn:
    """`wp.force_load(device='cuda')` (run_linemod.py:89, run_ycb_video.py:84) pre-compiles the reference's Warp depth
    filters; here they are CUDA kernels inside libfpose.so, so there is nothing to load."""

    @staticmethod
    def init():
        return None

    @staticmethod
    def force_load(device=None):
        return None


wp = _WarpStandIn()

code_dir = _HERE
BAD_DEPTH = 99
BAD_COLOR = 0
glcam_in_cvcam = np.array([[1, 0, 0, 0], [0, -1, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]]).astype(float)


def set_logging_format(level=logging.INFO):
    importlib.reload(logging)
    logging.basicConfig(level=level, format="[%(funcName)s()] %(message)s")


def set_seed(random_seed):
    import random

    np.random.seed(random_seed)
    random.seed(random_seed)
    torch.manual_seed(random_seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(random_seed)
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False


def NestDict():
    return defaultdict(NestDict)


def make_yaml_dumpable(D):
    """Nested dicts / arrays / numpy scalars -> plain Python containers that yaml.safe_dump accepts (in place for dicts,
    like the reference's helper: the drivers pass their NestDict of 4x4 poses)."""
    if isinstance(D, np.ndarray):
        return D.tolist()
    if isinstance(D, np.generic):  # numpy scalars, np.str_ included (a str subclass that yaml.safe_dump rejects)
        return D.item()
    if isinstance(D, dict):
        for k in list(D.keys()):
            D[k] = make_yaml_dumpable(dict(D[k]) if isinstance(D[k], dict) else D[k])
        return dict(D)
    if isinstance(D, (list, tuple)):
        return [make_yaml_dumpable(x) for x in D]
    return D


def euler_matrix(ai, aj, ak, axes="sxyz"):
    """Homogeneous rotation from Euler angles, `transformations.euler_matrix` for its default static-xyz axes
    (R = Rz(ak) Ry(aj) Rx(ai)); the reference only calls it with the default."""
    if axes != "sxyz":
        raise NotImplementedError("euler_matrix: only the default 'sxyz' convention is provided")
    ci, si, cj, sj, ck, sk = math.cos(ai), math.sin(ai), math.cos(aj), math.sin(aj), math.cos(ak), math.sin(ak)
    M = np.eye(4)
    M[:3, :3] = [[cj * ck, sj * si * ck - ci * sk, sj * ci * ck + si * sk],
                 [cj * sk, sj * si * sk + ci * ck, sj * ci * sk - si * ck],
                 [-sj, cj * si, cj * ci]]
    return M


def symmetry_tfs_from_info(info, rot_angle_discrete=5):
    """BOP `models_info.json` entry -> (n,4,4) symmetry transforms: identity, the listed discrete symmetries
    (translations mm -> m) and the first continuous axis sampled every `rot_angle_discrete` degrees."""
    tfs = [np.eye(4)]
    if "symmetries_discrete" in info:
        d = np.array(info["symmetries_discrete"], dtype=float).reshape(-1, 4, 4)
        d[..., :3, 3] *= 0.001
        tfs += list(d)
    if "symmetries_continuous" in info:
        axis = np.array(info["symmetries_continuous"][0]["axis"]).reshape(3)
        offset = info["symmetries_continuous"][0]["offset"]
        angles = np.arange(0, 360, rot_angle_discrete) / 180.0 * np.pi
        which = 0 if axis[0] > 0 else (1 if axis[1] > 0 else (2 if axis[2] > 0 else -1))
        for a in (angles if which >= 0 else [0.0]):
            e = [0.0, 0.0, 0.0]
            if which >= 0:
                e[which] = float(a)
            tf = euler_matrix(*e)
            tf[:3, 3] = offset
            tfs.append(tf)
    return np.array(tfs)


def to_homo(pts):
    assert len(pts.shape) == 2, f"pts.shape: {pts.shape}"
    return np.concatenate((pts, np.ones((pts.shape[0], 1))), axis=-1)


def transform_pts(pts, tf):
    """(..., N, d) points through a (..., d+1, d+1) homogeneous transform, d = 3 or 2 (numpy or torch): the
    predictors also push 2-D window corners through 3x3 crop transforms (predict_pose_refine.py:44-45)."""
    if len(tf.shape) >= 3 and tf.shape[-3] != pts.shape[-2]:
        tf = tf[..., None, :, :]
    return (tf[..., :-1, :-1] @ pts[..., None] + tf[..., :-1, -1:])[..., 0]


def depth2xyzmap(depth, K, uvs=None):
    depth = np.asarray(depth)
    H, W = depth.shape[:2]
    if uvs is None:
        vs, us = np.meshgrid(np.arange(0, H), np.arange(0, W), sparse=False, indexing="ij")
        vs, us = vs.reshape(-1), us.reshape(-1)
    else:
        uvs = np.asarray(uvs).round().astype(int)
        us, vs = uvs[:, 0], uvs[:, 1]
    zs = depth[vs, us]
    xyz_map = np.zeros((H, W, 3), dtype=np.float32)
    xyz_map[vs, us] = np.stack(((us - K[0, 2]) * zs / K[0, 0], (vs - K[1, 2]) * zs / K[1, 1], zs), 1)
    xyz_map[depth < 0.001] = 0
    return xyz_map


def depth2xyzmap_batch(depths, Ks, zfar):
    """depths (B,H,W) torch, Ks (B,3,3) torch -> (B,H,W,3); invalid (z < 0.001 or z > zfar) -> 0."""
    B, H, W = depths.shape
    vs, us = torch.meshgrid(torch.arange(0, H, device=depths.device), torch.arange(0, W, device=depths.device), indexing="ij")
    us, vs = us.float()[None], vs.float()[None]
    Ks = Ks.to(depths.device).float()
    xs = (us - Ks[:, 0, 2].reshape(B, 1, 1)) * depths / Ks[:, 0, 0].reshape(B, 1, 1)
    ys = (vs - Ks[:, 1, 2].reshape(B, 1, 1)) * depths / Ks[:, 1, 1].reshape(B, 1, 1)
    out = torch.stack([xs, ys, depths], dim=-1)
    out[(depths < 0.001) | (depths > zfar)] = 0
    return out


def compute_mesh_diameter(model_pts=None, mesh=None, n_sample=1000):
    """Largest pairwise vertex distance.  The reference samples `n_sample` points (random, so its value varies from run
    to run above 10 000 vertices); this one is exact."""
    pts = np.asarray(mesh.vertices if mesh is not None else model_pts)
    return float(_meshprep.mesh_diameter(pts))


def add_err(pred, gt, model_pts, symetry_tfs=np.eye(4)[None]):
    """ADD: mean distance between the model points under `pred` and under `gt` (4x4 poses, model_pts (P,3)).
    `symetry_tfs` is accepted and ignored, as in the reference."""
    add, _ = _metrics.pose_errors(model_pts, pred, gt, add=True, adds=False)
    return float(add[0])


def adds_err(pred, gt, model_pts):
    """ADD-S: mean over the model points under `gt` of the distance to the nearest model point under `pred`."""
    _, adds = _metrics.pose_errors(model_pts, pred, gt, add=False, adds=True)
    return float(adds[0])


def compute_auc_sklearn(errs, max_val=0.1, step=0.001):
    return _metrics.auc(errs, max_val=max_val, step=step)


def sample_views_icosphere(n_views, subdivisions=None, radius=1):
    return _hyp.sample_views_icosphere(n_views, subdivisions, radius)


def _depth_filter(depth, which):
    from foundationpose_b200.engine import op_depth_filter

    is_np = isinstance(depth, np.ndarray)
    d = torch.as_tensor(depth, dtype=torch.float, device="cuda")
    out = op_depth_filter(d, which)
    return out.data.cpu().numpy() if is_np else out


def erode_depth(depth, radius=2, depth_diff_thres=0.001, ratio_thres=0.8, zfar=100, device="cuda"):
    if (radius, depth_diff_thres, ratio_thres, zfar) != (2, 0.001, 0.8, 100):
        raise NotImplementedError("erode_depth: libfpose implements the parameters the estimator uses (estimater.py:173)")
    return _depth_filter(depth, 0)


def bilateral_filter_depth(depth, radius=2, zfar=100, sigmaD=2, sigmaR=100000, device="cuda"):
    if (radius, zfar, sigmaD, sigmaR) != (2, 100, 2, 100000):
        raise NotImplementedError("bilateral_filter_depth: libfpose implements the parameters the estimator uses (estimater.py:174)")
    return _depth_filter(depth, 1)


def toOpen3dCloud(points, colors=None, normals=None):
    if o3d is None:
        raise ImportError("toOpen3dCloud needs open3d (only the reference's debug >= 2 dumps call it)")
    cloud = o3d.geometry.PointCloud()
    cloud.points = o3d.utility.Vector3dVector(np.asarray(points).astype(np.float64))
    if colors is not None:
        colors = np.asarray(colors)
        if colors.max() > 1:
            colors = colors / 255.0
        cloud.colors = o3d.utility.Vector3dVector(colors.astype(np.float64))
    if normals is not None:
        cloud.normals = o3d.utility.Vector3dVector(np.asarray(normals).astype(np.float64))
    return cloud


# ---------------------------------------------------------------------------------------------
# visualisation of a pose (run_demo.py:71-74)
# ---------------------------------------------------------------------------------------------
def project_3d_to_2d(pt, K, ob_in_cam):
    p = np.asarray(K) @ (np.asarray(ob_in_cam) @ np.asarray(pt, dtype=float).reshape(4, 1))[:3]
    p = p.reshape(-1)
    return (p[:2] / p[2]).round().astype(int)


def draw_xyz_axis(color, ob_in_cam, scale=0.1, K=np.eye(3), thickness=3, transparency=0, is_input_rgb=False):
    """Draws the object frame's x / y / z axes (red / green / blue) of length `scale` into the image."""
    img = cv2.cvtColor(color, cv2.COLOR_RGB2BGR) if is_input_rgb else color.copy()
    origin = tuple(int(v) for v in project_3d_to_2d([0, 0, 0, 1], K, ob_in_cam))
    for axis, bgr in ((0, (0, 0, 255)), (1, (0, 255, 0)), (2, (255, 0, 0))):
        tip = np.array([0, 0, 0, 1], dtype=float)
        tip[axis] = scale
        end = tuple(int(v) for v in project_3d_to_2d(tip, K, ob_in_cam))
        layer = cv2.arrowedLine(img.copy(), origin, end, color=bgr, thickness=thickness, line_type=cv2.LINE_AA, tipLength=0)
        changed = np.linalg.norm(layer.astype(float) - img.astype(float), axis=-1) > 0
        img[changed] = (img[changed] * transparency + layer[changed] * (1 - transparency)).astype(img.dtype)
    img = img.astype(np.uint8)
    return cv2.cvtColor(img, cv2.COLOR_BGR2RGB) if is_input_rgb else img


def draw_posed_3d_box(K, img, ob_in_cam, bbox, line_color=(0, 255, 0), linewidth=2):
    """Draws the 12 edges of the box `bbox` ((2,3) min / max corners in the object frame) posed by `ob_in_cam`.
    Edge order as in the reference (Utils.py:713-749: the four x-edges, then y, then z; each from the low to the high
    corner): the anti-aliased lines overlap at the corners, so the order shows in the pixels."""
    K, ob_in_cam = np.asarray(K), np.asarray(ob_in_cam)
    lo, hi = np.asarray(bbox).min(axis=0), np.asarray(bbox).max(axis=0)
    for axis in range(3):
        u_ax, v_ax = [a for a in range(3) if a != axis]
        for u in (lo[u_ax], hi[u_ax]):
            for v in (lo[v_ax], hi[v_ax]):
                ends = np.empty((2, 3))
                ends[:, u_ax], ends[:, v_ax] = u, v
                ends[0, axis], ends[1, axis] = lo[axis], lo[axis] + (hi[axis] - lo[axis])
                cam = (ob_in_cam @ to_homo(ends).T).T[:, :3]
                proj = (K @ cam.T).T
                uv = np.round(proj[:, :2] / proj[:, 2:3]).astype(int)
                img = cv2.line(img, uv[0].tolist(), uv[1].tolist(), color=line_color, thickness=linewidth, lineType=cv2.LINE_AA)
    return img
