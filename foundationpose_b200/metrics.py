"""Pose accuracy: ADD / ADD-S on the GPU (`fp_pose_errors`) and the area-under-curve / recall summaries of
FoundationPose's evaluation (Utils.py:232-266); BOP's symmetry-aware MSSD / MSPD on the GPU (`fp_sym_pose_errors`) and
their average recalls; BOP's visible surface discrepancy on the GPU (`fp_vsd_errors`), its average recall and the
combined BOP AR.

    add, adds = pose_errors(model_pts, pred, gt)   # [N] float32 CUDA tensors, metres
    auc(adds.cpu().numpy())                          # AUC of the accuracy-threshold curve up to 0.1 m
    recall(add.cpu().numpy(), 0.1 * diameter)        # share of poses with ADD < 0.1 d

    syms = bop_symmetries(models_info[str(ob_id)])   # (S, 4, 4) float64, metres, identity first
    mssd, mspd = sym_pose_errors(model_pts, pred, gt, syms, K)   # [N] float32 CUDA tensors, metres / pixels
    average_recall(mssd, mssd_thresholds(diameter))  # BOP's AR_MSSD
    average_recall(mspd, mspd_thresholds(width))     # BOP's AR_MSPD

    vsd = vsd_errors(vertices, faces, pred, gt, depth, K, diameter)   # [N, 10] float32 CUDA tensor
    ar_vsd = vsd_average_recall(vsd)                                  # BOP's AR_VSD
    bop_ar(ar_vsd, ar_mssd, ar_mspd)                                  # (AR_VSD + AR_MSSD + AR_MSPD) / 3
"""
import math
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


def sym_pose_errors(model_pts, pred, gt, symmetries, K=None, mssd=True, mspd=True):
    """BOP's MSSD (metres) and MSPD (pixels) of every pose in `pred` against `gt`, computed by libfpose.so:

        MSSD = min_s max_i |E x_i - (G s) x_i|,   MSPD = min_s max_i |pi(K, E x_i) - pi(K, (G s) x_i)|

    with pi(K, x) = (K x)[:2] / x_z.  model_pts: [P, 3]; pred: [N, 4, 4] or one [4, 4]; gt: one [4, 4] pose for every
    prediction or [N, 4, 4]; symmetries: [S, 4, 4] in metres with the identity among them (`bop_symmetries`); K: one
    [3, 3] or [N, 3, 3], needed for MSPD only.  numpy arrays or torch tensors (any device, any float dtype).  Returns
    (mssd, mspd): float32 tensors [N] on the current CUDA device, None for a metric that was not requested.  A point
    projected from z = 0 makes its symmetry's MSPD infinite.  There is no CPU path: without a CUDA device this raises.
    """
    if not torch.cuda.is_available():
        raise _lib.FposeError("sym_pose_errors needs a CUDA device (there is no CPU path)")
    if mspd and K is None:
        raise _lib.FposeError("sym_pose_errors: MSPD needs the intrinsics K")
    dev = torch.device("cuda", torch.cuda.current_device())
    pts = _device_f32(model_pts, dev, 3)
    pred = _device_f32(pred, dev, 16)
    gt = _device_f32(gt, dev, 16)
    sym = _device_f32(symmetries, dev, 16)
    k = _device_f32(K, dev, 9) if mspd else None
    n = pred.shape[0]
    mssd_out = torch.empty(n, dtype=torch.float32, device=dev) if mssd else None
    mspd_out = torch.empty(n, dtype=torch.float32, device=dev) if mspd else None

    def ptr(t):
        return None if t is None or t.numel() == 0 else C.c_void_p(t.data_ptr())

    rc = lib.fp_sym_pose_errors(ptr(pts), pts.shape[0], ptr(pred), n, ptr(gt), gt.shape[0], ptr(sym), sym.shape[0],
                                ptr(k), 0 if k is None else k.shape[0], ptr(mssd_out), ptr(mspd_out),
                                C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    _lib.check(rc, "fp_sym_pose_errors")
    return mssd_out, mspd_out


def _axis_rotation(axis, angle):
    """Rodrigues: the rotation by `angle` about the unit vector along `axis`."""
    a = np.asarray(axis, dtype=np.float64).reshape(3)
    a = a / np.linalg.norm(a)
    c, s = math.cos(angle), math.sin(angle)
    cross = np.array([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]])
    return c * np.eye(3) + s * cross + (1.0 - c) * np.outer(a, a)


def bop_symmetries(model_info, max_sym_disc_step=0.01):
    """The symmetry transforms of a BOP `models_info.json` entry, (S, 4, 4) float64 in metres, identity first.

    Discrete: the identity and every `symmetries_discrete` entry (translations mm -> m).  Each continuous symmetry
    (axis a, offset o in mm) is sampled as n = ceil(pi / max_sym_disc_step) rotations R_i by i 2 pi / n about a,
    i = 0 .. n-1, with t_i = o - R_i o, so that no model point moves by more than `max_sym_disc_step` diameters between
    steps.  The set is every continuous step composed with every discrete symmetry, R = R_c R_d, t = R_c t_d + t_c
    (discrete outer, continuous inner); without continuous symmetries it is the discrete set.  This follows the
    description of bop_toolkit's misc.get_symmetry_transformations, with step i = 0 included so that the identity is
    always a member (a pose is never penalised against itself)."""
    disc = [np.eye(4)]
    for d in model_info.get("symmetries_discrete", []):
        d = np.array(d, dtype=np.float64).reshape(4, 4)
        d[:3, 3] *= 1e-3
        disc.append(d)
    cont = []
    for sym in model_info.get("symmetries_continuous", []):
        offset = np.asarray(sym["offset"], dtype=np.float64).reshape(3) * 1e-3
        n = int(math.ceil(math.pi / max_sym_disc_step))
        for i in range(n):
            c = np.eye(4)
            c[:3, :3] = _axis_rotation(sym["axis"], i * 2.0 * math.pi / n)
            c[:3, 3] = offset - c[:3, :3] @ offset
            cont.append(c)
    if not cont:
        return np.stack(disc)
    out = []
    for d in disc:
        for c in cont:
            m = np.eye(4)
            m[:3, :3] = c[:3, :3] @ d[:3, :3]
            m[:3, 3] = c[:3, :3] @ d[:3, 3] + c[:3, 3]
            out.append(m)
    return np.stack(out)


MSSD_STEPS = np.arange(1, 11) * 0.05  # x the object diameter: 0.05 d .. 0.50 d
MSPD_STEPS = np.arange(1, 11) * 5.0   # pixels at an image width of 640: 5 .. 50 px


def mssd_thresholds(diameter):
    """BOP's MSSD thresholds for an object of `diameter` metres."""
    return MSSD_STEPS * float(diameter)


def mspd_thresholds(image_width):
    """BOP's MSPD thresholds in pixels, scaled from 640-pixel-wide images to `image_width`."""
    return MSPD_STEPS * (640.0 / float(image_width))


def average_recall(errs, thresholds):
    """Mean over the thresholds of the share of errors strictly below each.  thresholds: [T] (the same for every
    error) or [T, n] (column j for error j, e.g. each pose with its own object's thresholds)."""
    errs = _host(errs)
    thr = np.asarray(thresholds, dtype=np.float64)
    thr = thr[:, None] if thr.ndim == 1 else thr
    return float(np.mean(errs[None, :] < thr))


VSD_TAUS = np.arange(1, 11) * 0.05        # misalignment tolerances x the object diameter: 0.05 d .. 0.50 d
VSD_THRESHOLDS = np.arange(1, 11) * 0.05  # correctness thresholds on the VSD error: 0.05 .. 0.50
VSD_DELTA = 0.015                         # visibility tolerance, metres (BOP 2019 for LM / YCB-V)


def vsd_errors(vertices, faces, pred, gt, depth, K, diameter, delta=VSD_DELTA, taus=VSD_TAUS, return_counts=False):
    """BOP's VSD (visib_mode 'bop19', cost 'step') of every pose in `pred` against `gt`, computed by libfpose.so: the
    mesh is rendered at both poses with the crop producer's coverage rule on the full frame, and

        e_t = (|{visG and visE, |distG - distE| >= tau_t d}| + |visG xor visE|) / |visG or visE|   (1 if nothing is visible)

    vertices: [V, 3] metres, faces: [F, 3] (host data; numpy or torch); pred: [N, 4, 4] or one [4, 4]; gt, depth [H, W]
    (metres, 0 = no measurement) and K [3, 3]: one for every prediction or one per prediction; diameter in metres,
    `taus` in diameters, `delta` in metres.  Returns float32 [N, T] on the current CUDA device; with `return_counts`
    also the int32 [N, T + 2] counts (union, intersection, c_0 .. c_{T-1}).  There is no CPU path: without a CUDA
    device this raises."""
    if not torch.cuda.is_available():
        raise _lib.FposeError("vsd_errors needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", torch.cuda.current_device())
    pos = np.ascontiguousarray(_host_array(vertices), dtype=np.float32).reshape(-1, 3)
    fcs = np.ascontiguousarray(_host_array(faces), dtype=np.int32).reshape(-1, 3)
    pred = _device_f32(pred, dev, 16)
    gt = _device_f32(gt, dev, 16)
    depth = torch.as_tensor(depth).to(device=dev, dtype=torch.float32)
    if depth.dim() == 2:
        depth = depth[None]
    depth = depth.contiguous()
    k = _device_f32(K, dev, 9)
    tau = torch.as_tensor(np.asarray(taus, dtype=np.float64).reshape(-1) * float(diameter), dtype=torch.float32).to(dev)
    n, T = pred.shape[0], tau.numel()
    errs = torch.empty(n, T, dtype=torch.float32, device=dev)
    counts = torch.empty(n, T + 2, dtype=torch.int32, device=dev) if return_counts else None

    def ptr(t):
        return None if t is None or t.numel() == 0 else C.c_void_p(t.data_ptr())

    rc = lib.fp_vsd_errors(C.c_void_p(pos.ctypes.data), pos.shape[0], C.c_void_p(fcs.ctypes.data), fcs.shape[0],
                           ptr(pred), n, ptr(gt), gt.shape[0], ptr(depth), depth.shape[0], depth.shape[1], depth.shape[2],
                           ptr(k), k.shape[0], float(delta), ptr(tau), T, ptr(errs), ptr(counts),
                           C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    _lib.check(rc, "fp_vsd_errors")
    return (errs, counts) if return_counts else errs


def _host_array(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def vsd_average_recall(errs, thresholds=VSD_THRESHOLDS):
    """BOP's AR_VSD: the mean over every (tau, threshold) pair of the share of poses with e_tau < threshold.
    errs: [N, T] (one row per pose, one column per tau)."""
    if isinstance(errs, torch.Tensor):
        errs = errs.detach().cpu().numpy()
    errs = np.asarray(errs, dtype=np.float64)
    errs = errs.reshape(errs.shape[0], -1) if errs.ndim else errs.reshape(1, 1)
    thr = np.asarray(thresholds, dtype=np.float64).reshape(-1)
    return float(np.mean(errs[:, :, None] < thr[None, None, :]))


def bop_ar(ar_vsd, ar_mssd, ar_mspd):
    """The BOP Challenge score of one method: (AR_VSD + AR_MSSD + AR_MSPD) / 3."""
    return (float(ar_vsd) + float(ar_mssd) + float(ar_mspd)) / 3.0
