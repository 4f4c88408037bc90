"""Host references of depth alignment (fp_set_camera_depth_sensor / fp_align_depth, include/fpose.h): librealsense's
rs2::align rule for depth -> colour, restated in numpy float32 with every operation rounded on its own, in the order the
kernel computes it, and the same rule in float64 for comparison.

Also the rigs the tests use: a D435-like one (848x480 depth next to 1280x720 colour, 15 mm baseline, about 0.5 degrees
of rotation) and a same-size one (640x480 -> 640x480)."""
import numpy as np

D435_DEPTH_K = np.array([[421.4, 0.0, 422.9], [0.0, 421.4, 239.7], [0.0, 0.0, 1.0]])
D435_COLOR_K = np.array([[912.3, 0.0, 641.8], [0.0, 911.7, 365.2], [0.0, 0.0, 1.0]])
VGA_DEPTH_K = np.array([[383.2, 0.0, 319.1], [0.0, 383.2, 241.6], [0.0, 0.0, 1.0]])
VGA_COLOR_K = np.array([[615.0, 0.0, 320.0], [0.0, 615.0, 240.0], [0.0, 0.0, 1.0]])


def rig_T(angle_deg=0.5, t=(0.015, 0.0002, -0.0004), axis=(0.3, 1.0, 0.2)):
    """T_color_from_depth: a rotation of angle_deg about `axis`, then the translation t (metres)."""
    a = np.asarray(axis, dtype=np.float64)
    a /= np.linalg.norm(a)
    th = np.deg2rad(angle_deg)
    k = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + np.sin(th) * k + (1 - np.cos(th)) * k @ k
    T[:3, 3] = t
    return T


def _corners(z, xs, ys, Kd, T, Kc, dt):
    """Per corner (x - 0.5, y - 0.5), (x + 0.5, y + 0.5): (xi, yi, Z') in dtype dt, the operation order of the rule."""
    c = lambda v: dt(v)
    fxd, fyd, cxd, cyd = c(Kd[0][0]), c(Kd[1][1]), c(Kd[0][2]), c(Kd[1][2])
    fxc, fyc, cxc, cyc = c(Kc[0][0]), c(Kc[1][1]), c(Kc[0][2]), c(Kc[1][2])
    R = np.asarray(T, dtype=np.float64)
    out = []
    for off in (-0.5, 0.5):
        px = xs.astype(dt) + c(off)
        py = ys.astype(dt) + c(off)
        X = ((px - cxd) / fxd) * z
        Y = ((py - cyd) / fyd) * z
        P = [((c(R[r, 0]) * X + c(R[r, 1]) * Y) + c(R[r, 2]) * z) + c(R[r, 3]) for r in range(3)]
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            u = (P[0] / P[2]) * fxc + cxc
            v = (P[1] / P[2]) * fyc + cyc
            out.append((np.trunc(u + c(0.5)), np.trunc(v + c(0.5)), P[2], u, v))
    return out


def rectangles(depth_m, valid, Kd, T, Kc, H, W, dt=np.float32):
    """The rectangle of every depth pixel the rule keeps: (x0, x1, y0, y1, z) int64 / dt arrays over the kept pixels, in
    row-major depth order, and the kept mask over the pixels where `valid` (raw value != 0)."""
    ys, xs = np.nonzero(valid)
    z = depth_m[ys, xs].astype(dt)
    (x0, y0, z0, _, _), (x1, y1, z1, _, _) = _corners(z, xs, ys, Kd, T, Kc, dt)
    with np.errstate(invalid="ignore"):
        keep = (z0 > 0) & (z1 > 0) & (x0 >= 0) & (x0 <= x1) & (x1 <= dt(W - 1)) & (y0 >= 0) & (y0 <= y1) & (y1 <= dt(H - 1))
    k = lambda a: a[keep].astype(np.int64)
    return k(x0), k(x1), k(y0), k(y1), z[keep], keep


def near_boundary(depth_m, valid, Kd, T, Kc, tol=1e-4):
    """Over the valid pixels: whether any corner coordinate u + 0.5 or v + 0.5 (float64) lies within tol of an integer,
    where the float32 and float64 rules may round to different pixels."""
    ys, xs = np.nonzero(valid)
    z = depth_m[ys, xs].astype(np.float64)
    near = np.zeros(len(z), bool)
    for (_, _, _, u, v) in _corners(z, xs, ys, Kd, T, Kc, np.float64):
        for a in (u + 0.5, v + 0.5):
            with np.errstate(invalid="ignore"):
                near |= np.abs(a - np.round(a)) < tol
    return near


def align(depth_m, valid, Kd, T, Kc, H, W, dt=np.float32):
    """The aligned (H, W) depth of dtype dt: each colour pixel the smallest z of the rectangles that cover it, 0 where
    none does.  depth_m: (Hd, Wd) metres (float32 for the float32 rule); valid: raw value != 0."""
    x0, x1, y0, y1, z, _ = rectangles(depth_m, valid, Kd, T, Kc, H, W, dt)
    out = np.full((H, W), np.inf, dtype=dt)
    w, h = x1 - x0 + 1, y1 - y0 + 1
    big = w * h > 64
    for i in np.nonzero(big)[0]:  # the few large rectangles (near pixels) by slices
        blk = out[y0[i]:y1[i] + 1, x0[i]:x1[i] + 1]
        np.minimum(blk, z[i], out=blk)
    small = ~big
    for dy in range(int(h[small].max(initial=0))):
        for dx in range(int(w[small].max(initial=0))):
            s = small & (h > dy) & (w > dx)
            np.minimum.at(out, (y0[s] + dy, x0[s] + dx), z[s])
    out[np.isinf(out) & (out > 0)] = 0
    return out


def depth_metres(raw, scale):
    """A sensor's raw depth in metres and its valid mask (raw != 0): float32 as stored, or uint16 * scale in float32."""
    if scale is None:
        raw = np.asarray(raw, dtype=np.float32)
        return raw, raw != 0
    return raw.astype(np.float32) * np.float32(scale), raw != 0
