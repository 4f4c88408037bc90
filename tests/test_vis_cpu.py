"""CPU: the debug-canvas helpers against the reference's own functions (tests/golden/vis_golden.npz,
tools/make_golden_vis.py), the canvas sizes and colour map libfpose.so reports against cv2 / torchvision, and the
resample rule of the scorer canvas kernel against cv2.resize."""
import os

import cv2
import numpy as np
import pytest
import torch
import torchvision

from foundationpose_b200.engine import vis_colormap, vis_size
from foundationpose_b200.vis import cv_draw_text, depth_to_vis, make_grid_image

from vis_compose import resize_rule, score_row

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vis_golden.npz")


@pytest.fixture(scope="module")
def g():
    return dict(np.load(GOLDEN))


def test_depth_to_vis_matches_reference(g):
    assert np.array_equal(depth_to_vis(g["depth"]), g["d2v_inverse"])
    assert np.array_equal(depth_to_vis(g["depth"], zmin=np.float32(0.3), zmax=np.float32(0.7), inverse=False), g["d2v_range"])
    assert np.array_equal(depth_to_vis(g["norm"], zmin=g["norm"].min(), zmax=g["norm"].max(), inverse=False), g["d2v_norm"])
    assert np.array_equal(depth_to_vis(np.zeros((8, 8), np.float32), zmin=np.float32(0), zmax=np.float32(0), inverse=False), g["d2v_flat"])
    assert np.array_equal(depth_to_vis(g["depth"], mode="gray"), g["d2v_gray"])


def test_make_grid_image_matches_reference(g):
    f, u = g["rgb_f"], g["rgb_u"]
    assert np.array_equal(make_grid_image([f[0], f[1], u[0], u[1]], nrow=4, padding=2, pad_value=255), g["grid_mixed"])
    assert np.array_equal(make_grid_image(list(u), nrow=2, padding=5, pad_value=255), g["grid_rows"])
    assert np.array_equal(make_grid_image([f[2]], nrow=1, padding=2, pad_value=255), g["grid_one"])
    assert np.array_equal(make_grid_image(list(f), nrow=1, padding=2, pad_value=0), g["grid_col"])


def test_cv_draw_text_matches_reference(g):
    base = g["rgb_u"][0].repeat(4, axis=0).repeat(8, axis=1)
    assert np.array_equal(cv_draw_text(base.copy(), text="id:7", uv_top_left=(10, 10), color=(0, 255, 0), fontScale=0.5), g["text_u8"])
    assert np.array_equal(cv_draw_text(base.copy(), text="id:123, score:101.234\nline two", uv_top_left=(150, 120),
                                       color=(255, 0, 0), fontScale=0.5, outline_color=(0, 0, 0)), g["text_edge"])
    assert np.array_equal(cv_draw_text(base.astype(np.float64), text="id:3, score:100.500", uv_top_left=(10, 10),
                                       color=(0, 255, 0), fontScale=0.5), g["text_f64"])


def test_colormap_is_cv2_jet():
    jet = cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(-1, 1), cv2.COLORMAP_JET)[:, 0, ::-1]
    assert np.array_equal(vis_colormap(), jet)


def _tv_grid(imgs, nrow):
    t = torch.as_tensor(np.asarray(imgs)).permute(0, 3, 1, 2)
    return torchvision.utils.make_grid(t, nrow=nrow, padding=2, pad_value=255).permute(1, 2, 0).numpy()


@pytest.mark.parametrize("N", [1, 2, 5, 252])
def test_canvas_sizes(N):
    row = _tv_grid([np.zeros((160, 160, 3), np.float32)] * 2 + [np.zeros((160, 160, 3), np.uint8)] * 2, 4).astype(np.uint8)
    assert row.shape == (164, 650, 3)
    block = _tv_grid([row] * N, 1)
    assert vis_size("refine", N) == _tv_grid([block, block], 2).shape[:2]
    if N > 1:
        assert vis_size("refine", N) == (N * 166 + 6, 1314)
    rec = np.zeros((1, 2, 160, 160, 4), np.float32)
    assert score_row(rec, 0).shape == (100, 409, 3)
    assert vis_size("score", N) == (N * 105, 409)


def test_scorer_resample_rule_is_cv2_resize():
    """The kernel's arithmetic, restated in numpy, is within 1e-9 of cv2.resize on float64 rows built like the scorer's
    (float32 rgb * 255, 255 gaps, uint8 colour-mapped depth).  cv2 rounds its float64 weights and sums differently in
    the last bits, so after the reference's truncation to uint8 a pixel whose exact value is an integer (constant
    regions: gaps, flat colour-mapped depth) may come out one lower on either side: at most 1, on about 1 % of them."""
    rng = np.random.default_rng(3)
    rec = rng.uniform(0, 1, (4, 2, 160, 160, 4)).astype(np.float32)
    rec[..., 3] = rng.uniform(0.4, 0.8, (4, 2, 160, 160)).astype(np.float32)
    rec[1, 0, :40, :, 3] = 0.0
    for i in range(len(rec)):
        dA, dB = rec[i, 0, ..., 3], rec[i, 1, ..., 3]
        pad = np.ones((160, 5, 3)) * 255
        vA = depth_to_vis(dA, zmin=dA.min(), zmax=dA.max(), inverse=False)
        vB = depth_to_vis(dB, zmin=dA.min(), zmax=dA.max(), inverse=False)
        row = np.concatenate([rec[i, 0, ..., :3] * np.float32(255), pad, vA, pad, rec[i, 1, ..., :3] * np.float32(255), pad, vB], axis=1)
        ours, ref = resize_rule(row), cv2.resize(row, fx=0.625, fy=0.625, dsize=None)
        assert np.abs(ours - ref).max() < 1e-9
        d = np.abs(ours.astype(np.uint8).astype(int) - ref.astype(np.uint8).astype(int))
        assert d.max() <= 1 and (d > 0).mean() < 0.03


# rows of the flow scene whose crops the CPU oracle reproduces bit for bit (tests/test_flow_golden_cpu.py: the reference's
# render window comes out of a fp32 LU inverse, which moves a few rendered silhouette pixels of some poses)
EXACT_START_ROWS = (1, 2, 3, 4)     # start pose 0 is the axis-aligned one of DESIGN.md §4
EXACT_REFINED_ROWS = (0, 1, 3)
EXACT_SCORE_IDS = (0, 1, 3)         # the scorer crops the refined poses


@pytest.fixture(scope="module")
def flow(g):
    import sys

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import make_golden_flow as gen  # scene() only: nothing of the reference is read

    import vis_compose
    from oracle import geometry

    mesh, mt, _, rgb, depth, mask, K, d, _ = gen.scene()
    depth_f = geometry.bilateral_filter_depth(geometry.erode_depth(depth))
    xyz = geometry.depth2xyzmap(depth_f, K)
    a = vis_compose.oracle_records(g["canvas_start"], mt, rgb, depth_f, xyz, K, d, 0)
    b = vis_compose.oracle_records(g["canvas_refined"], mt, rgb, depth_f, xyz, K, d, 0)
    s = vis_compose.oracle_records(g["canvas_refined"], mt, rgb, depth_f, None, K, d, 1)
    return a, b, s


def test_oracle_refiner_canvas_matches_the_reference(g, flow):
    """The host composer on the oracle's crops draws the reference's refiner canvas: same size, labels and layout, rows
    bit-identical wherever the crops are; the other rows differ only in the rendered crop (image 0 / its depth, image
    2) on < 0.1 % of their pixels, by at most 16 grey levels."""
    import vis_compose
    from foundationpose_b200.vis import label_refine_canvas

    a, b, _ = flow
    got = label_refine_canvas(vis_compose.refine_canvas(a, b), len(a))
    want = g["canvas_refine"]
    assert got.shape == want.shape
    for blk, (x0, exact) in enumerate(((4, EXACT_START_ROWS), (660, EXACT_REFINED_ROWS))):
        for i in range(len(a)):
            y0 = 4 + 166 * i
            d = np.abs(got[y0:y0 + 164, x0:x0 + 650].astype(int) - want[y0:y0 + 164, x0:x0 + 650].astype(int)).max(-1)
            if i in exact:
                assert not d.any(), (blk, i)
                continue
            ys, xs = np.nonzero(d)
            assert set(((xs - 2) // 162).tolist()) <= {0, 2}, (blk, i)
            assert (d > 0).mean() < 1e-3 and d.max() <= 16, (blk, i, (d > 0).mean(), d.max())
    rows = np.zeros(want.shape[:2], bool)
    rows[4:4 + 166 * len(a)] = True
    assert np.array_equal(got[~rows], want[~rows])  # borders


def test_oracle_scorer_canvas_matches_the_reference(g, flow):
    """The host composer on the oracle's crops draws the reference's scorer canvas: rows in the same (descending
    score) order with the same labels, bit-identical for the hypotheses whose crops are; the others within 2 grey
    levels on < 0.1 % of their pixels."""
    import vis_compose
    from foundationpose_b200.vis import label_score_canvas

    _, _, s = flow
    scores = g["canvas_scores"]
    ids = torch.as_tensor(scores).argsort(descending=True).numpy()
    got = label_score_canvas(vis_compose.score_canvas(s, ids), ids, scores)
    want = g["canvas_score"]
    assert got.shape == want.shape
    for slot, i in enumerate(ids):
        d = np.abs(got[105 * slot:105 * slot + 105].astype(int) - want[105 * slot:105 * slot + 105].astype(int))
        if i in EXACT_SCORE_IDS:
            assert not d.any(), i
        else:
            assert (d.max(-1) > 0).mean() < 1e-3 and d.max() <= 2, (i, d.max())
