"""GPU: BOP's VSD of fp_vsd_errors (metrics.vsd_errors) against the full-frame oracle render and the float64
restatement (tests/vsd_reference.py): exact counts on a closed mesh, an open mesh that shows its back faces and
triangles that cross the near plane, errors from the counts bit for bit, bit-identical results across batches,
broadcasting and frame sizes, argument checks, and `examples/eval_bop_results.py --vsd` end to end."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch
import yaml

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "examples"), os.path.join(ROOT, "foundationpose_b200", "dropin"), ROOT,
                os.path.dirname(os.path.abspath(__file__))]

import vsd_reference as ref  # noqa: E402

K0 = np.array([[615.0, 0.0, 320.0], [0.0, 612.0, 240.0], [0.0, 0.0, 1.0]], dtype=np.float32)
DIAM = 0.1
TAUS = np.arange(1, 11) * 0.05


def _poses(rng, n, t=(0.0, 0.0, 0.5), rot_deg=20.0, trans=0.01):
    from scipy.spatial.transform import Rotation

    out = np.repeat(np.eye(4)[None], n, axis=0)
    rv = rng.normal(size=(n, 3))
    rv *= (np.deg2rad(rot_deg) * rng.uniform(0, 1, size=(n, 1))) / np.linalg.norm(rv, axis=1, keepdims=True)
    out[:, :3, :3] = Rotation.from_rotvec(rv).as_matrix()
    out[:, :3, 3] = np.asarray(t) + rng.uniform(-trans, trans, size=(n, 3))
    return out.astype(np.float32)


def _sphere(subdiv=2, r=0.05):
    from foundationpose_b200 import synth

    v, f = synth.icosphere(subdiv)
    return (v * r).astype(np.float32), f.astype(np.int32)


def _open_cup(subdiv=3, r=0.05):
    """The icosphere's faces with z < 0.3 r: an open shell whose inside shows through the opening."""
    v, f = _sphere(subdiv, r)
    keep = v[f].mean(1)[:, 2] < 0.3 * r
    return v, f[keep]


def _test_depth(verts, faces, gt, K, H, W, seed):
    """The ground truth's render with 2 mm noise, holes (D = 0) and an occluder 3 cm in front of part of the object."""
    rng = np.random.default_rng(seed)
    d = ref.render_depth(gt, verts, faces, K, H, W)
    D = np.where(d > 0, d + rng.normal(0, 0.002, size=d.shape), 1.0).astype(np.float32)
    D[rng.uniform(size=D.shape) < 0.05] = 0.0
    ys, xs = np.nonzero(d > 0)
    if len(ys):
        y0, x0 = int(ys.mean()), int(xs.mean())
        D[y0:y0 + 25, x0 - 40:x0] = np.where(d[y0:y0 + 25, x0 - 40:x0] > 0, d[y0:y0 + 25, x0 - 40:x0] - 0.03, 0.7)
    return D


def _check_counts(verts, faces, pred, gt, D, K, delta=0.015):
    from foundationpose_b200 import metrics

    errs, counts = metrics.vsd_errors(verts, faces, pred, gt, D, K, DIAM, delta=delta, taus=TAUS, return_counts=True)
    errs, counts = errs.cpu().numpy(), counts.cpu().numpy()
    taus32 = (TAUS * DIAM).astype(np.float32)
    near_total = 0
    for i, p in enumerate(pred):
        want, _, n_near = ref.vsd_errors(verts, faces, p, gt, D, K, delta, taus32)
        near_total += n_near
        assert np.abs(counts[i].astype(np.int64) - want).max() <= n_near, (i, counts[i], want, n_near)
        # the errors are the counts' fp64 quotient rounded to fp32, bit for bit
        u, inter, c = counts[i, 0], counts[i, 1], counts[i, 2:].astype(np.float64)
        e = np.ones(len(TAUS), dtype=np.float32) if u == 0 else ((c + (u - inter)) / u).astype(np.float32)
        np.testing.assert_array_equal(errs[i], e)
    print(f"pixels within 1e-6 m of a delta or tau decision: {near_total}")
    return errs, counts


def test_exact_counts_closed_mesh():
    rng = np.random.default_rng(1)
    v, f = _sphere(2)
    gt = _poses(rng, 1, rot_deg=180)[0]
    pred = np.concatenate([gt[None], _poses(rng, 5, t=gt[:3, 3], rot_deg=30, trans=0.012)])
    D = _test_depth(v, f, gt, K0, 480, 640, 2)
    errs, counts = _check_counts(v, f, pred, gt, D, K0)
    assert counts[0, 0] > 2000 and (errs[0] == 0).all()  # the ground truth against itself
    assert (errs[1:] > 0).any()


def test_exact_counts_open_mesh_shows_back_faces():
    from foundationpose_b200 import synth

    rng = np.random.default_rng(3)
    v, f = _open_cup(3)
    gt = np.eye(4, dtype=np.float32)
    gt[:3, :3] = synth.random_rotation(4)[:3, :3] @ np.diag([1.0, -1.0, -1.0])  # opening roughly towards the camera
    gt[:3, 3] = [0.01, 0.0, 0.45]
    pred = np.concatenate([gt[None], _poses(rng, 4, t=gt[:3, 3], rot_deg=25, trans=0.01)])
    D = _test_depth(v, f, gt, K0, 480, 640, 5)
    _check_counts(v, f, pred, gt, D, K0)


def test_exact_counts_near_plane_crossing():
    """A floor 6 cm below the camera that reaches behind it: every triangle crosses the near plane."""
    v = np.array([[-0.6, -0.6, 0.0], [0.6, -0.6, 0.0], [0.6, 0.6, 0.0], [-0.6, 0.6, 0.0]], dtype=np.float32)
    f = np.array([[0, 1, 2], [0, 2, 3]], dtype=np.int32)
    gt = np.eye(4, dtype=np.float32)
    gt[:3, :3] = [[1, 0, 0], [0, 0, -1], [0, 1, 0]]
    gt[:3, 3] = [0.0, 0.06, 0.3]
    pred = np.repeat(gt[None], 4, axis=0)
    pred[1, 1, 3] += 0.004
    pred[2, 2, 3] += 0.05
    pred[3, 0, 3] += 0.3
    D = _test_depth(v, f, gt, K0, 480, 640, 7)
    _, counts = _check_counts(v, f, pred, gt, D, K0)
    assert counts[0, 0] > 50000


def test_identity_is_zero_and_invisible_is_one():
    from foundationpose_b200 import metrics

    rng = np.random.default_rng(11)
    v, f = _sphere(3)
    gt = _poses(rng, 64, rot_deg=180, trans=0.05)
    D = np.zeros((480, 640), dtype=np.float32)  # no measurement anywhere: everything rendered is visible
    e = metrics.vsd_errors(v, f, gt, gt, D, K0, DIAM)
    assert torch.count_nonzero(e).item() == 0
    away = gt.copy()
    away[:, 0, 3] += 3.0  # off-screen
    e = metrics.vsd_errors(v, f, away, gt, D, K0, DIAM)
    assert (e == 1).all()
    e, c = metrics.vsd_errors(v, f, away, away, D, K0, DIAM, return_counts=True)
    assert (e == 1).all() and (c == 0).all()


@pytest.mark.parametrize("H, W", [(480, 640), (720, 1280)])
def test_bit_identical_across_batches_and_broadcasting(H, W):
    from foundationpose_b200 import metrics, synth

    rng = np.random.default_rng(H)
    mesh = synth.make_mesh(3)
    v, f = mesh.vertices.astype(np.float32), mesh.faces.astype(np.int32)
    K = K0.copy()
    K[0, 2], K[1, 2] = W / 2, H / 2
    gt = _poses(rng, 1, t=(0.0, 0.0, 0.55), rot_deg=180)[0]
    pred = _poses(rng, 1024, t=gt[:3, 3], rot_deg=40, trans=0.03)
    D = _test_depth(v, f, gt, K, H, W, 3)
    e, c = metrics.vsd_errors(v, f, pred, gt, D, K, 0.2, return_counts=True)
    e2, c2 = metrics.vsd_errors(v, f, pred, gt, D, K, 0.2, return_counts=True)
    assert torch.equal(e, e2) and torch.equal(c, c2)
    assert (c[:, 0] > 0).all() and len(torch.unique(e[:, 4])) > 50
    a, b = metrics.vsd_errors(v, f, pred[:252], gt, D, K, 0.2, return_counts=True)
    assert torch.equal(a, e[:252]) and torch.equal(b, c[:252])
    for i in (0, 251, 777, 1023):
        a, b = metrics.vsd_errors(v, f, pred[i], gt, D, K, 0.2, return_counts=True)
        assert torch.equal(a, e[i:i + 1]) and torch.equal(b, c[i:i + 1])
    # per-pose ground truth, depth and K: the same bits
    n = 252
    a, b = metrics.vsd_errors(v, f, pred[:n], np.repeat(gt[None], n, 0), np.repeat(D[None], n, 0), np.repeat(K[None], n, 0),
                              0.2, return_counts=True)
    assert torch.equal(a, e[:n]) and torch.equal(b, c[:n])
    # errors without counts: the same bits
    assert torch.equal(metrics.vsd_errors(v, f, pred, gt, D, K, 0.2), e)
    assert metrics.vsd_errors(v, f, pred[:0], gt, D, K, 0.2).shape == (0, 10)


def test_bad_arguments_raise_and_leave_the_device_usable():
    from foundationpose_b200 import _lib, metrics

    lib = _lib.lib
    dev = torch.device("cuda")
    v, f = _sphere(1)
    pose = torch.eye(4, device=dev).reshape(1, 16).repeat(3, 1)
    pose[:, 11] = 0.5
    depth = torch.zeros(3, 48, 64, device=dev)
    K = torch.tensor(K0, device=dev).reshape(1, 9)
    taus = torch.full((65,), 0.01, device=dev)
    out = torch.empty(3, 65, device=dev)
    cnt = torch.empty(3, 67, dtype=torch.int32, device=dev)
    host = np.zeros(3 * 48 * 64 * 16, dtype=np.float32)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    h = C.c_void_p(host.ctypes.data)
    dev_pos = torch.as_tensor(v, device=dev)
    bad_faces = f.copy()
    bad_faces[3, 1] = len(v)
    ok = dict(pos=C.c_void_p(v.ctypes.data), V=len(v), faces=C.c_void_p(f.ctypes.data), F=len(f), pred=p(pose), N=3,
              gt=p(pose), n_gt=1, depth=p(depth), n_depth=3, H=48, W=64, K=p(K), n_K=1, delta=0.015, taus=p(taus), T=10,
              errs=p(out), counts=p(cnt))
    bad = {"null pos": dict(pos=None), "null faces": dict(faces=None), "device pos": dict(pos=p(dev_pos)),
           "face index out of range": dict(faces=C.c_void_p(bad_faces.ctypes.data)), "V < 3": dict(V=2), "F = 0": dict(F=0),
           "N < 0": dict(N=-1), "null pred": dict(pred=None), "null gt": dict(gt=None), "null depth": dict(depth=None),
           "null K": dict(K=None), "null taus": dict(taus=None), "null errs_out": dict(errs=None),
           "host pred": dict(pred=h), "host gt": dict(gt=h), "host depth": dict(depth=h), "host K": dict(K=h),
           "host taus": dict(taus=h), "host errs_out": dict(errs=h), "host counts_out": dict(counts=h),
           "n_gt not 1 or N": dict(n_gt=2), "n_depth not 1 or N": dict(n_depth=2), "n_K not 1 or N": dict(n_K=2),
           "H = 0": dict(H=0), "W too large": dict(W=4097), "T = 0": dict(T=0), "T too large": dict(T=65),
           "delta < 0": dict(delta=-0.001), "delta inf": dict(delta=float("inf")), "delta nan": dict(delta=float("nan"))}
    torch.cuda.synchronize()
    launches = lib.fp_launch_count()
    for what, change in bad.items():
        a = {**ok, **change}
        rc = lib.fp_vsd_errors(*a.values(), st)
        assert rc != 0, what
        with pytest.raises(_lib.FposeError, match="fp_vsd_errors"):
            _lib.check(rc, "fp_vsd_errors")
    assert lib.fp_launch_count() == launches
    assert lib.fp_vsd_errors(*{**ok, "counts": None}.values(), st) == 0
    assert lib.fp_launch_count() == launches + 2
    with pytest.raises(_lib.FposeError, match="n_depth"):
        metrics.vsd_errors(v, f, pose, pose[0], depth[:2], K0, DIAM)
    torch.cuda.synchronize()
    K_small = np.array([[60.0, 0.0, 32.0], [0.0, 60.0, 24.0], [0.0, 0.0, 1.0]])  # the sphere in the middle of 64 x 48
    e, c = metrics.vsd_errors(v, f, pose, pose, depth[0], K_small, DIAM, return_counts=True)
    assert e.shape == (3, 10) and torch.count_nonzero(e).item() == 0 and (c[:, 0] > 100).all()


def test_eval_bop_results_with_vsd(tmp_path):
    """Ground truth in frame 0, shifted by k mm along x and 4 k mm along z in frame k, one skipped frame: AR_VSD and
    BOP AR as computed here from the oracle renders and the float64 restatement; the --bop output unchanged."""
    import eval_bop_results as ev

    from foundationpose_b200 import metrics, synth

    root = str(tmp_path / "LINEMOD")
    gts = synth.write_bop_dataset(root, "lm", n_frames=3, symmetric=(6,))
    res = {}
    for (vid, id_str, ob_id), pose in gts.items():
        p = np.array(pose, dtype=np.float64)
        p[:3, 3] += np.array([1.0, 0.0, 4.0]) * 0.001 * int(id_str) * (1 + ob_id % 3)
        res.setdefault(vid, {}).setdefault(id_str, {})[ob_id] = p.tolist()
    res[1]["000002"][1] = np.eye(4).tolist()  # a frame the driver skipped
    path = tmp_path / "linemod_res.yml"
    path.write_text(yaml.safe_dump(res))
    bop_rows, bop_overall = ev.main(["--res", str(path), "--dataset_dir", root, "--bop"])
    rows, overall = ev.main(["--res", str(path), "--dataset_dir", root, "--vsd", "--json", str(tmp_path / "t.json")])
    for ob_id, r in rows.items():
        assert {k: v for k, v in r.items() if k not in ("vsd_ar", "bop_ar")} == bop_rows[ob_id]
    assert {k: v for k, v in overall.items() if k not in ("vsd_ar", "bop_ar")} == bop_overall
    factory = ev.make_reader_factory("lm", root)
    all_err, near = [], 0
    for ob_id, row in rows.items():
        reader = factory(ob_id)  # one scene per object, scene id = object id
        mesh = reader.get_gt_mesh(ob_id)
        d = reader.get_model_diameter(ob_id)
        taus32 = (metrics.VSD_TAUS * d).astype(np.float32)
        errs = []
        for i in range(3):
            if ob_id == 1 and i == 2:
                errs.append(np.full(10, np.inf))
                continue
            pred = np.asarray(res[ob_id][f"{i:06d}"][ob_id], dtype=np.float32)
            gt = reader.get_gt_pose(i, ob_id).astype(np.float32)
            D = reader.get_depth(i).astype(np.float32)
            _, e, n_near = ref.vsd_errors(mesh.vertices.astype(np.float32), mesh.faces, pred, gt, D, reader.get_K(i), 0.015,
                                          taus32)
            near += n_near
            errs.append(e.astype(np.float32).astype(np.float64))
        errs = np.stack(errs)
        assert row["vsd_ar"] == pytest.approx(metrics.vsd_average_recall(errs), abs=1e-12)
        assert row["bop_ar"] == pytest.approx((row["vsd_ar"] + row["mssd_ar"] + row["mspd_ar"]) / 3, abs=1e-12)
        all_err.append(errs)
    assert overall["vsd_ar"] == pytest.approx(metrics.vsd_average_recall(np.concatenate(all_err)), abs=1e-12)
    assert overall["bop_ar"] == pytest.approx((overall["vsd_ar"] + overall["mssd_ar"] + overall["mspd_ar"]) / 3, abs=1e-12)
    assert 0.0 < overall["vsd_ar"] < 1.0
    print(f"pixels within 1e-6 m of a delta or tau decision: {near}")
    assert os.path.exists(tmp_path / "t.json")
