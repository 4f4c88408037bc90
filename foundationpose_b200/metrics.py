"""Pose accuracy: ADD / ADD-S on the GPU (`fp_pose_errors`) and the area-under-curve / recall summaries of
FoundationPose's evaluation (Utils.py:232-266).

    add, adds = pose_errors(model_pts, pred, gt)   # [N] float32 CUDA tensors, metres
    auc(adds.cpu().numpy())                          # AUC of the accuracy-threshold curve up to 0.1 m
    recall(add.cpu().numpy(), 0.1 * diameter)        # share of poses with ADD < 0.1 d
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import lib


def _device_f32(x, dev, cols):
    return torch.as_tensor(x).to(device=dev, dtype=torch.float32).reshape(-1, cols).contiguous()


def pose_errors(model_pts, pred, gt, add=True, adds=True):
    """ADD and ADD-S of every pose in `pred` against `gt` over `model_pts`, computed by libfpose.so.

    model_pts: [P, 3]; pred: [N, 4, 4] or one [4, 4]; gt: one [4, 4] pose for every prediction or [N, 4, 4].
    numpy arrays or torch tensors (any device, any float dtype).  Returns (add, adds): float32 tensors [N] on the
    current CUDA device, None for a metric that was not requested.  ADD alone skips the O(N P^2) nearest-neighbour
    search of ADD-S.  There is no CPU path: without a CUDA device this raises.
    """
    if not torch.cuda.is_available():
        raise _lib.FposeError("pose_errors needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", torch.cuda.current_device())
    pts = _device_f32(model_pts, dev, 3)
    pred = _device_f32(pred, dev, 16)
    gt = _device_f32(gt, dev, 16)
    n = pred.shape[0]
    add_out = torch.empty(n, dtype=torch.float32, device=dev) if add else None
    adds_out = torch.empty(n, dtype=torch.float32, device=dev) if adds else None

    def ptr(t):
        return None if t is None or t.numel() == 0 else C.c_void_p(t.data_ptr())

    rc = lib.fp_pose_errors(ptr(pts), pts.shape[0], ptr(pred), n, ptr(gt), gt.shape[0], ptr(add_out), ptr(adds_out),
                            C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    _lib.check(rc, "fp_pose_errors")
    return add_out, adds_out


def _host(errs):
    if isinstance(errs, torch.Tensor):
        errs = errs.detach().cpu().numpy()
    return np.asarray(errs, dtype=np.float64).reshape(-1)


def auc(errs, max_val=0.1, step=0.001):
    """compute_auc_sklearn (Utils.py:256-266) without sklearn: the trapezoidal area under the share of errors <= x for
    x = 0, step, ... max_val, divided by max_val.  As in the reference, the curve is evaluated only until it reaches 1;
    the thresholds after that keep their initial value, 1."""
    errs = np.sort(_host(errs))
    X = np.arange(0, max_val + step, step)
    Y = np.ones(len(X))
    for i, x in enumerate(X):
        y = (errs <= x).sum() / len(errs)
        Y[i] = y
        if y >= 1:
            break
    # sklearn.metrics.auc = numpy's trapezoidal rule over increasing X, summed in the same order
    return float(np.add.reduce(np.diff(X) * (Y[1:] + Y[:-1]) / 2.0) / max_val)


def recall(errs, threshold):
    """Share of the errors strictly below `threshold` (a scalar, or one threshold per error)."""
    errs = _host(errs)
    return float(np.mean(errs < np.asarray(threshold, dtype=np.float64)))
