"""Host side of the debug canvases: the text labels the reference draws on the canvases fp_vis composes on the device,
and the reference's three drawing helpers (Utils.py:293-300 make_grid_image, :456-479 depth_to_vis, :630-655
cv_draw_text), which the drop-in Utils re-exports.

    refine_canvas(engine, poses_in, poses_out)  predict_pose_refine.py:241-293  (N*166+6, 1314, 3); (168, 1306, 3) for N = 1
    score_canvas(engine, poses, scores)         predict_score.py:27-52, :219-224  (N*105, 409, 3)

Both return numpy uint8 arrays; the pixels come back from the device in one copy and only the labels are drawn here.
"""
import cv2
import numpy as np
import torch

PAD = 2          # make_grid_image(padding=2)
ROW_H, ROW_W = 164, 650
SCORE_PITCH = 105  # 100-pixel scorer row + 5 rows of 255


def depth_to_vis(depth, zmin=None, zmax=None, mode="rgb", inverse=True):
    """Utils.py:456-479: a depth image as a colour (mode 'rgb': JET, RGB order) or gray uint8 image."""
    zmin = depth.min() if zmin is None else zmin
    zmax = depth.max() if zmax is None else zmax
    if inverse:
        vis = zmin / (depth + 1e-8)
        vis[depth < 0.001] = 0
    else:
        d = depth.clip(zmin, zmax)
        with np.errstate(divide="ignore", invalid="ignore"):
            vis = (d - zmin) / (zmax - zmin)
        vis[(d == zmin) | (d == zmax)] = 1
    if mode == "gray":
        return (vis * 255).clip(0, 255).astype(np.uint8)
    if mode == "rgb":
        return cv2.applyColorMap((vis * 255).astype(np.uint8), cv2.COLORMAP_JET)[..., ::-1]
    raise RuntimeError


def make_grid_image(imgs, nrow, padding=5, pad_value=255):
    """Utils.py:293-300 (torchvision.utils.make_grid on (B,H,W,C) images, then uint8 by truncation): images in rows of
    `nrow`, `padding` pixels of `pad_value` around each; a single image comes back as it is."""
    a = np.asarray(imgs)
    if a.ndim == 3:
        a = a[None]
    if a.shape[-1] == 1:
        a = np.repeat(a, 3, axis=-1)
    if len(a) == 1:
        return a[0].astype(np.uint8)
    B, H, W, C = a.shape
    cols = min(nrow, B)
    rows = -(-B // cols)
    h, w = H + padding, W + padding
    grid = np.full((rows * h + padding, cols * w + padding, C), pad_value, dtype=a.dtype)
    for k in range(B):
        y, x = divmod(k, cols)
        grid[y * h + padding:y * h + padding + H, x * w + padding:x * w + padding + W] = a[k]
    return grid.astype(np.uint8)


def cv_draw_text(img, text, uv_top_left, color=(255, 255, 255), fontScale=0.5, thickness=1, fontFace=cv2.FONT_HERSHEY_SIMPLEX,
                 outline_color=None, line_spacing=1.5):
    """Utils.py:630-655: anti-aliased text, one line at a time, each line moved back inside the image if it would
    cross an edge.  Draws into `img` and returns it."""
    H, W = img.shape[:2]
    top_left = np.array(uv_top_left, dtype=float)
    assert top_left.shape == (2,)
    for line in text.splitlines():
        (w, h), _ = cv2.getTextSize(text=line, fontFace=fontFace, fontScale=fontScale, thickness=thickness)
        x, y = top_left[0], top_left[1] + h
        while x < 0:
            x += 1
        while x + w >= W:
            x -= 1
        while y >= H:
            y -= 1
        while y - h < 0:
            y += 1
        org = (int(x), int(y))
        for c in ([outline_color] if outline_color is not None else []) + [color]:
            cv2.putText(img, text=line, org=org, fontFace=fontFace, fontScale=fontScale, color=c, thickness=thickness,
                        lineType=cv2.LINE_AA)
        top_left[1] = y - h + h * line_spacing
    return img


def _label(canvas, y, x, h, w, text, as_float):
    """cv_draw_text on the (h, w) block at (y, x) of `canvas`, as the reference draws it on that block alone: on uint8
    (refiner rows, anti-aliased) or on float64 (scorer rows, where OpenCV draws without anti-aliasing)."""
    block = canvas[y:y + h, x:x + w]
    block = block.astype(np.float64) if as_float else block.copy()
    canvas[y:y + h, x:x + w] = cv_draw_text(block, text=text, uv_top_left=(10, 10), color=(0, 255, 0), fontScale=0.5).astype(np.uint8)


def label_refine_canvas(canvas, N):
    """Draws the refiner canvas's labels ('id:<i>' on the start-pose rows) into the (H, W, 3) uint8 `canvas`."""
    bp = 0 if N == 1 else PAD
    for i in range(N):
        _label(canvas, PAD + bp + i * (ROW_H + PAD), PAD + bp, ROW_H, ROW_W, f"id:{i}", as_float=False)
    return canvas


def label_score_canvas(canvas, ids, scores):
    """Draws the scorer canvas's labels ('id:<i>, score:<s>' on row s = hypothesis ids[s]) into `canvas`."""
    for s, i in enumerate(np.asarray(ids)):
        _label(canvas, s * SCORE_PITCH, 0, SCORE_PITCH - 5, canvas.shape[1], f"id:{i}, score:{float(scores[i]):.3f}", as_float=True)
    return canvas


def refine_canvas(engine, poses_in, poses_out):
    """PoseRefinePredictor.predict(get_vis=True)'s canvas: every hypothesis's crops at its start pose (left, labelled
    'id:<i>') and at its refined pose (right)."""
    canvas = engine.vis("refine", poses_in, poses_out).cpu().numpy()
    return label_refine_canvas(canvas, len(engine._poses(poses_in)))


def score_canvas(engine, poses, scores):
    """ScorePredictor.predict(get_vis=True)'s canvas: one row per hypothesis by descending score, labelled
    'id:<i>, score:<s>'."""
    scores = torch.as_tensor(scores)
    ids = scores.argsort(descending=True)
    canvas = engine.vis("score", poses, order=ids).cpu().numpy()
    return label_score_canvas(canvas, ids.cpu().numpy(), scores.float().cpu().numpy())
