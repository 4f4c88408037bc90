"""CPU: the full-frame depth render of the VSD reference against the analytic ellipsoid and the oracle's crop
rasteriser, the float64 VSD restatement on hand-computable cases, the AR_VSD / BOP AR arithmetic and the host side of
`examples/eval_bop_results.py --vsd`."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "examples"), os.path.join(ROOT, "foundationpose_b200", "dropin"), ROOT,
                os.path.dirname(os.path.abspath(__file__))]

import vsd_reference as ref  # noqa: E402

K0 = np.array([[615.0, 0.0, 320.0], [0.0, 615.0, 240.0], [0.0, 0.0, 1.0]])
TAUS = np.arange(1, 11) * 0.05 * 0.2  # diameter 0.2 m


def _pose(R=np.eye(3), t=(0.0, 0.0, 0.6)):
    p = np.eye(4)
    p[:3, :3] = R
    p[:3, 3] = t
    return p


def _quad(half=0.05):
    """Two triangles of a square in the object's z = 0 plane (fronto-parallel under a pose without rotation)."""
    v = np.array([[-half, -half, 0.0], [half, -half, 0.0], [half, half, 0.0], [-half, half, 0.0]])
    return v, np.array([[0, 1, 2], [0, 2, 3]])


def test_full_frame_depth_matches_the_analytic_ellipsoid():
    from scipy.ndimage import binary_erosion

    from foundationpose_b200 import synth

    mesh = synth.make_mesh(4)
    pose = _pose(synth.random_rotation(3), (0.02, -0.01, 0.55))
    # make_multi_scene casts its rays through integer pixel coordinates, the render through pixel centres
    Ka = K0.copy()
    Ka[:2, 2] -= 0.5
    _, depth, owner = synth.make_multi_scene([(mesh.visual.image, pose, 1.0)], Ka, depth_noise=0.0)
    d = ref.render_depth(pose, mesh.vertices, mesh.faces, K0, 480, 640)
    inner = binary_erosion(owner == 0, iterations=3)
    assert inner.sum() > 5000
    assert (d[inner] > 0).all()
    # the tessellation sits inside the ellipsoid: rendered depth >= analytic, by less than the largest chord sag
    err = d[inner].astype(np.float64) - depth[inner]
    assert err.min() > -1e-5 and err.max() < 1.5e-3, (err.min(), err.max())
    assert np.median(err) < 3e-4
    # nothing rendered where the analytic ray misses the ellipsoid (away from the silhouette)
    outer = binary_erosion(owner != 0, iterations=3)
    assert (d[outer] == 0).all()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_full_frame_render_and_rasterize_agree_on_coverage(seed):
    from oracle import raster

    from foundationpose_b200 import synth

    mesh = synth.make_mesh(2)
    rng = np.random.default_rng(seed)
    K = np.array([[300.0, 0.0, 80.0], [0.0, 310.0, 78.0], [0.0, 0.0, 1.0]])
    pose = _pose(synth.random_rotation(seed), (rng.uniform(-0.03, 0.03), rng.uniform(-0.03, 0.03), 0.45))
    d = ref.render_depth(pose, mesh.vertices, mesh.faces, K, 160, 160)
    tri_id = raster.rasterize(pose, mesh.vertices, mesh.faces, K, (0.0, 0.0, 160.0, 160.0))[0]
    np.testing.assert_array_equal(d > 0, tri_id >= 0)
    assert (tri_id >= 0).sum() > 1000


def test_near_plane_crossing_triangles_cover_the_frame():
    """A floor quad 5 cm below the camera that reaches behind it takes the homogeneous path: the rows below the
    horizon see it at depth 0.05 / ray_y."""
    v, f = _quad(0.5)
    pose = _pose(np.array([[1.0, 0, 0], [0, 0.0, -1.0], [0, 1.0, 0.0]]), (0.0, 0.05, 0.2))  # z from -0.3 to 0.7 m
    K = np.array([[60.0, 0.0, 32.0], [0.0, 60.0, 24.0], [0.0, 0.0, 1.0]])
    d = ref.render_depth(pose, v, f, K, 48, 64)
    ray_y = (np.arange(48) + 0.5 - 24.0) / 60.0
    want = np.where(ray_y > 0.05 / 0.7, 0.05 / np.maximum(ray_y, 1e-9), 0.0)
    cov = (d > 0).any(axis=1)
    rows = np.flatnonzero(cov)
    assert len(rows) > 10
    np.testing.assert_allclose(d[rows, 32], want[rows], rtol=1e-5)


def test_pose_against_itself_is_zero_and_invisible_is_one():
    v, f = _quad()
    g = _pose()
    dG = ref.render_depth(g, v, f, K0, 480, 640)
    D = dG.copy()
    D[::7, ::5] = 0  # holes
    counts, errs, _ = ref.vsd_counts(dG, dG, D, K0, 0.015, TAUS)
    assert counts[0] == counts[1] == (dG > 0).sum() and (counts[2:] == 0).all()
    assert (errs == 0).all()
    # estimate off-screen: nothing of E is visible, everything of G is -> 1 for every tau
    off = ref.render_depth(_pose(t=(5.0, 0.0, 0.6)), v, f, K0, 480, 640)
    assert (off == 0).all()
    counts, errs, _ = ref.vsd_counts(off, dG, D, K0, 0.015, TAUS)
    assert counts[1] == 0 and (errs == 1).all()
    # nothing visible under either pose: union 0 -> 1
    counts, errs, _ = ref.vsd_counts(off, off, D, K0, 0.015, TAUS)
    assert counts[0] == 0 and (errs == 1).all()


@pytest.mark.parametrize("k_mm", [3, 7, 12])
def test_shift_along_the_axis_steps_at_the_right_tau(k_mm):
    """G: a fronto-parallel quad at 0.6 m over the principal point; E: the same quad k mm farther.  Over the quad
    |distG - distE| = k mm * s with 1 <= s <= 1.0002, so e_tau = 1 for tau <= k mm and 0 for tau > 1.0002 k mm."""
    v, f = _quad(0.004)  # about 8 x 8 px
    g, e = _pose(), _pose(t=(0.0, 0.0, 0.6 + k_mm * 1e-3))
    dG = ref.render_depth(g, v, f, K0, 480, 640)
    dE = ref.render_depth(e, v, f, K0, 480, 640)
    taus = np.array([0.5, 0.99, 1.01, 2.0]) * k_mm * 1e-3
    counts, errs, _ = ref.vsd_counts(dE, dG, dG, K0, 0.015, taus)
    # the farther quad covers fewer pixels: those of G outside it count as misaligned (visG and not visE)
    comp = counts[0] - counts[1]
    assert counts[1] > 30
    np.testing.assert_array_equal(counts[2:], [counts[1], counts[1], 0, 0])
    np.testing.assert_allclose(errs, [1, 1, comp / counts[0], comp / counts[0]], rtol=0, atol=1e-15)


def test_vsd_average_recall_and_bop_ar_by_hand():
    from foundationpose_b200 import metrics

    np.testing.assert_allclose(metrics.VSD_TAUS, np.arange(1, 11) * 0.05, rtol=0, atol=1e-15)
    np.testing.assert_allclose(metrics.VSD_THRESHOLDS, np.arange(1, 11) * 0.05, rtol=0, atol=1e-15)
    assert metrics.VSD_DELTA == 0.015
    # two poses x two taus against thresholds 0.1, 0.3: pose 0 (0.05, 0.2) passes 1 + 2, pose 1 (0.25, inf) passes 1
    errs = np.array([[0.05, 0.2], [0.25, np.inf]])
    assert metrics.vsd_average_recall(errs, [0.1, 0.3]) == pytest.approx(4 / 8, abs=1e-15)
    assert metrics.vsd_average_recall(np.zeros((3, 10))) == 1.0
    assert metrics.vsd_average_recall(np.full((3, 10), 0.05)) == pytest.approx(0.9, abs=1e-15)  # strictly below
    assert metrics.bop_ar(0.3, 0.6, 0.9) == pytest.approx(0.6, abs=1e-15)


def test_evaluator_vsd_implies_bop_and_chunks():
    import eval_bop_results as ev

    opt = ev.parse_args(["--res", "r.yml", "--dataset_dir", "d", "--vsd"])
    assert opt.vsd and opt.bop
    opt = ev.parse_args(["--res", "r.yml", "--dataset_dir", "d", "--bop"])
    assert opt.bop and not opt.vsd
    opt = ev.parse_args(["--res", "r.yml", "--dataset_dir", "d"])
    assert not opt.bop and not opt.vsd
    # chunks: same frame size, at most VSD_CHUNK poses, skipped frames (None) in runs of their own
    shapes = [(480, 640)] * 3 + [None] + [(480, 640)] * (ev.VSD_CHUNK + 1) + [(720, 1280)]
    chunks = ev.vsd_chunks(shapes, shapes)
    assert chunks == [(0, 3), (3, 4), (4, 4 + ev.VSD_CHUNK), (4 + ev.VSD_CHUNK, 5 + ev.VSD_CHUNK),
                      (5 + ev.VSD_CHUNK, 6 + ev.VSD_CHUNK)]


def test_evaluator_vsd_rows_and_skipped_frames():
    import eval_bop_results as ev

    err = np.array([[0.0] * 10, [0.2] * 10, [np.inf] * 10])  # a perfect pose, one at 0.2, a skipped frame
    row = ev.summarize_vsd(err, 0.5, 0.25)
    # thresholds 0.05 .. 0.5: pose 0 passes all 10, pose 1 passes 0.25 .. 0.5 (6), pose 2 none
    assert row["vsd_ar"] == pytest.approx(16 / 30, abs=1e-15)
    assert row["bop_ar"] == pytest.approx((16 / 30 + 0.5 + 0.25) / 3, abs=1e-15)


def test_table_with_vsd_and_unchanged_bop_table(capsys):
    import eval_bop_results as ev

    rows = {2: {"poses": 3, "add_auc": 0.5, "adds_auc": 0.75, "add_s_recall": 1 / 3, "symmetric": False, "diameter": 0.1,
                "mssd_ar": 0.25, "mspd_ar": 0.5}}
    overall = {"poses": 3, "add_auc": 0.5, "adds_auc": 0.75, "add_s_recall": 1 / 3, "mssd_ar": 0.25, "mspd_ar": 0.5}
    ev.print_table(rows, overall, bop=True)
    bop_out = capsys.readouterr().out.splitlines()
    assert "without VSD" in bop_out[-1] and bop_out[0].split()[-2:] == ["AR", "MSPD"]
    for r in (rows[2], overall):
        r.update(vsd_ar=0.75, bop_ar=0.5)
    ev.print_table(rows, overall, bop=True, vsd=True)
    out = capsys.readouterr().out.splitlines()
    assert out[0].split()[-4:] == ["AR", "VSD", "BOP", "AR"]
    assert out[2].split() == ["all", "3", "50.00", "75.00", "33.33", "25.00", "50.00", "75.00", "50.00"]
    assert "BOP AR" in out[-1]
    # the --bop table does not change when the rows carry VSD columns
    ev.print_table(rows, overall, bop=True)
    assert capsys.readouterr().out.splitlines() == bop_out
