"""Host composition of the get_vis canvases from per-pixel crop records, step for step as the reference builds them
(predict_pose_refine.py:241-293, predict_score.py:27-52) with the reference's helpers (foundationpose_b200/vis.py,
held to the reference's own functions by tests/test_vis_cpu.py), torchvision-style grids and cv2.resize.  No labels.

A record is (N, 2, 160, 160, 4) float32: per hypothesis the rendered (A) and observed (B) crop, channels r, g, b (0..1)
and one depth value (refiner: normalised z; scorer: raw depth in metres) — the layout fp_vis's crop pass writes."""
import cv2
import numpy as np

from foundationpose_b200.vis import depth_to_vis, make_grid_image


def oracle_records(poses, mt, rgb, depth, xyz_map, K, mesh_diameter, mode):
    """The crop records of the CPU oracle (oracle/pipeline.py, held to the reference's crop code by
    tests/test_flow_golden_cpu.py): refiner (mode 0) normalised z; scorer (mode 1) rendered camera z for A and the
    nearest-warped depth for B (predict_score.py:90), both raw metres."""
    import torch

    from oracle import geometry, pipeline, raster

    A, B, _ = pipeline.make_crops(poses, mt, rgb, depth, xyz_map, K, mesh_diameter, mode)
    rec = np.zeros((len(poses), 2, 160, 160, 4), np.float32)
    rec[:, 0, ..., :3] = A[:, :3].permute(0, 2, 3, 1).numpy()
    rec[:, 1, ..., :3] = B[:, :3].permute(0, 2, 3, 1).numpy()
    if mode == 0:
        rec[:, 0, ..., 3], rec[:, 1, ..., 3] = A[:, 5].numpy(), B[:, 5].numpy()
        return rec
    win, tf = geometry.crop_window(np.asarray(poses, np.float32), K, mesh_diameter, 1.2, 160)
    umin, vmin, umax, vmax = geometry.render_window(win, 160)
    for n in range(len(poses)):
        rec[n, 0, ..., 3] = raster.render_crop(np.asarray(poses[n], np.float32), mt, K, (umin[n], vmin[n], umax[n], vmax[n]))[1][..., 2]
    d_t = torch.as_tensor(depth, dtype=torch.float32)[None, None].expand(len(poses), -1, -1, -1)
    rec[:, 1, ..., 3] = geometry.warp_perspective(d_t, torch.from_numpy(tf), (160, 160), "nearest")[:, 0].numpy()
    return rec


def refine_rows(rec):
    rows = []
    for n in range(len(rec)):
        dA, dB = rec[n, 0, ..., 3], rec[n, 1, ..., 3]
        zmin, zmax = min(dA.min(), dB.min()), max(dA.max(), dB.max())
        imgs = [rec[n, 0, ..., :3] * np.float32(255), rec[n, 1, ..., :3] * np.float32(255),
                depth_to_vis(dA, zmin=zmin, zmax=zmax, inverse=False), depth_to_vis(dB, zmin=zmin, zmax=zmax, inverse=False)]
        rows.append(make_grid_image(imgs, nrow=4, padding=2, pad_value=255))
    return rows


def refine_canvas(rec_start, rec_refined):
    blocks = [make_grid_image(refine_rows(r), nrow=1, padding=2, pad_value=255) for r in (rec_start, rec_refined)]
    return make_grid_image(blocks, nrow=2, padding=2, pad_value=255)


def score_row(rec, i):
    dA, dB = rec[i, 0, ..., 3], rec[i, 1, ..., 3]
    zmin, zmax = dA.min(), dA.max()
    pad = np.ones((160, 5, 3)) * 255
    row = np.concatenate([rec[i, 0, ..., :3] * np.float32(255), pad, depth_to_vis(dA, zmin=zmin, zmax=zmax, inverse=False), pad,
                          rec[i, 1, ..., :3] * np.float32(255), pad, depth_to_vis(dB, zmin=zmin, zmax=zmax, inverse=False)], axis=1)
    s = 100 / row.shape[0]
    return cv2.resize(row, fx=s, fy=s, dsize=None)


def score_canvas(rec, order):
    out = []
    for i in order:
        out += [score_row(rec, int(i)), np.ones((5, 409, 3)) * 255]
    return np.concatenate(out, axis=0).astype(np.uint8)


def resize_rule(row):
    """The resample fp_vis's scorer kernel implements, restated: cv2's INTER_LINEAR source coordinate
    (d + 0.5) * 1.6 - 0.5, weights (1 - f, f), all in float64, horizontal pass first."""
    def taps(n):
        x = (np.arange(n) + 0.5) * (1.0 / 0.625) - 0.5
        s = np.floor(x).astype(np.int64)
        f = x - s
        return s, 1.0 - f, f
    sy, b0, b1 = taps(100)
    sx, a0, a1 = taps(409)
    h = row[:, sx] * a0[None, :, None] + row[:, sx + 1] * a1[None, :, None]
    return h[sy] * b0[:, None, None] + h[sy + 1] * b1[:, None, None]
