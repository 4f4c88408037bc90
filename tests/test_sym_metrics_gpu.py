"""GPU: BOP's MSSD / MSPD of fp_sym_pose_errors (metrics.sym_pose_errors) against a float64 numpy restatement of the
definitions, exact zeros, continuous-symmetry steps, bit-identical results across launch shapes and symmetry order,
projections from z = 0, argument checks, and `examples/eval_bop_results.py --bop` end to end."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch
import yaml

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "examples"), os.path.join(ROOT, "foundationpose_b200", "dropin"), ROOT]
K0 = np.array([[615.0, 0.0, 320.0], [0.0, 612.0, 240.0], [0.0, 0.0, 1.0]])


def _random_poses(rng, n, t=(0.0, 0.0, 0.6), rot_deg=180.0, trans=0.05):
    from scipy.spatial.transform import Rotation

    out = np.repeat(np.eye(4)[None], n, axis=0)
    rv = rng.normal(size=(n, 3))
    rv *= (np.deg2rad(rot_deg) * rng.uniform(0, 1, size=(n, 1))) / np.linalg.norm(rv, axis=1, keepdims=True)
    out[:, :3, :3] = Rotation.from_rotvec(rv).as_matrix()
    out[:, :3, 3] = np.asarray(t) + rng.uniform(-trans, trans, size=(n, 3))
    return out.astype(np.float32)


def _half_turn_mm(axis, offset_mm=(0.0, 0.0, 0.0)):
    from scipy.spatial.transform import Rotation

    a = np.asarray(axis, dtype=np.float64)
    m = np.eye(4)
    m[:3, :3] = Rotation.from_rotvec(a / np.linalg.norm(a) * np.pi).as_matrix()
    m[:3, 3] = np.asarray(offset_mm) - m[:3, :3] @ np.asarray(offset_mm)
    return m.reshape(-1).tolist()


CONT = {"axis": [0.0, 0.6, 0.8], "offset": [4.0, -3.0, 2.0]}


def _symmetries(S):
    """1: identity; 4: three discrete half turns; 315: one continuous axis; 1260: the axis and the half turns."""
    from foundationpose_b200 import metrics

    disc = [_half_turn_mm(a, (4.0, -3.0, 2.0)) for a in ([1, 0, 0], [0, 0.8, -0.6], [1, 0.6, 0.8])]
    info = {1: {}, 4: {"symmetries_discrete": disc}, 315: {"symmetries_continuous": [CONT]},
            1260: {"symmetries_discrete": disc, "symmetries_continuous": [CONT]}}[S]
    syms = metrics.bop_symmetries(info)
    assert len(syms) == S
    return syms


def _numpy_errors(pts, pred, gt, syms, K):
    """float64 restatement: per pose, (MSSD, MSPD, per-symmetry MSSD [S], per-symmetry MSPD [S])."""
    with np.errstate(divide="ignore", invalid="ignore"):  # a skipped frame's identity pose may put points at z = 0
        return _numpy_errors_64(pts.astype(np.float64), pred, gt, syms.astype(np.float64), K)


def _numpy_errors_64(pts, pred, gt, syms, K):
    out = []
    for e, g, k in zip(pred.astype(np.float64), np.broadcast_to(gt.astype(np.float64), pred.shape),
                       np.broadcast_to(K.astype(np.float64), (len(pred), 3, 3))):
        ep = pts @ e[:3, :3].T + e[:3, 3]
        eu = (ep @ k.T)[:, :2] / ep[:, 2:3]
        w3, w2 = [], []
        for c in range(0, len(syms), 64):
            gs = g[None] @ syms[c:c + 64]
            q = np.einsum("sij,pj->spi", gs[:, :3, :3], pts) + gs[:, None, :3, 3]
            qu = (q @ k.T)[..., :2] / q[..., 2:3]
            w3.append(np.linalg.norm(ep[None] - q, axis=-1).max(1))
            w2.append(np.linalg.norm(eu[None] - qu, axis=-1).max(1))
        w3, w2 = np.concatenate(w3), np.concatenate(w2)
        out.append((w3.min(), w2.min(), w3, w2))
    return out


def _margin_ok(per_sym, tol):
    """argmin of per_sym and whether the runner-up is more than `tol` above it."""
    order = np.argsort(per_sym, kind="stable")
    return order[0], len(per_sym) == 1 or per_sym[order[1]] - per_sym[order[0]] > 2 * tol


@pytest.mark.parametrize("S", [1, 4, 315, 1260])
@pytest.mark.parametrize("P", [1, 97, 10000])
def test_against_float64(S, P):
    from foundationpose_b200 import metrics

    rng = np.random.default_rng(S * 7 + P)
    pts = (rng.normal(size=(P, 3)) * [0.05, 0.03, 0.09]).astype(np.float32)
    n = 6 if S * P > 1e6 else 24
    gt = _random_poses(rng, 1)
    syms = _symmetries(S)
    # half near a symmetric image of the ground truth, half anywhere
    pick = syms[rng.integers(0, S, size=n // 2)]
    near = _random_poses(rng, n // 2, t=(0, 0, 0), rot_deg=8.0, trans=0.005).astype(np.float64) @ (gt[0] @ pick)
    pred = np.concatenate([near.astype(np.float32), _random_poses(rng, n - n // 2)])
    K = np.repeat(K0[None], n, axis=0).astype(np.float32)
    K[:, 0, 1] = rng.uniform(-2, 2, size=n)  # a skewed K exercises the full 3x3 product
    mssd, mspd = metrics.sym_pose_errors(pts, pred, gt, syms, K)
    mssd, mspd = mssd.cpu().numpy().astype(np.float64), mspd.cpu().numpy().astype(np.float64)
    syms32 = syms.astype(np.float32)
    want = _numpy_errors(pts, pred, gt, syms32, K)
    tol3 = lambda x: 1e-6 + 1e-6 * abs(x)  # noqa: E731
    for i, (w3, w2, per3, per2) in enumerate(want):
        assert abs(mssd[i] - w3) <= tol3(w3), (i, mssd[i], w3)
        assert abs(mspd[i] - w2) <= 1e-3, (i, mspd[i], w2)
        # the minimiser: scored against its symmetry alone, the pose gets the very same bits
        for per, tol, j in ((per3, tol3(w3), 0), (per2, 1e-3, 1)):
            s, clear = _margin_ok(per, tol)
            if clear:
                one = metrics.sym_pose_errors(pts, pred[i], gt, syms32[s:s + 1], K[i])[j].item()
                assert one == (mssd if j == 0 else mspd)[i], (i, j, s)


def test_pose_against_itself_is_exactly_zero():
    from foundationpose_b200 import metrics

    rng = np.random.default_rng(5)
    pts = (rng.normal(size=(3001, 3)) * [0.05, 0.03, 0.09]).astype(np.float32)
    gt = _random_poses(rng, 40)
    mssd, mspd = metrics.sym_pose_errors(pts, gt, gt, _symmetries(1260), K0)
    assert torch.count_nonzero(mssd).item() == 0 and torch.count_nonzero(mspd).item() == 0


def test_continuous_steps_and_half_steps():
    """A ground truth turned about the continuous axis by k 2 pi / 315 scores ~0; by half a step, at most the chord
    2 r sin(pi / 630) of the point farthest from the axis."""
    from scipy.spatial.transform import Rotation

    from foundationpose_b200 import metrics

    rng = np.random.default_rng(9)
    pts = (rng.normal(size=(5000, 3)) * [0.06, 0.05, 0.1]).astype(np.float32)
    syms = _symmetries(315)
    gt = _random_poses(rng, 1, t=(0.02, -0.01, 0.35), trans=0.01)[0].astype(np.float64)
    axis = np.asarray(CONT["axis"]) / np.linalg.norm(CONT["axis"])
    o = np.asarray(CONT["offset"]) * 1e-3

    def turn(angle):
        m = np.eye(4)
        m[:3, :3] = Rotation.from_rotvec(axis * angle).as_matrix()
        m[:3, 3] = o - m[:3, :3] @ o
        return m

    step = 2 * math.pi / 315
    ks = [0, 1, 17, 158, 314]
    exact = np.stack([gt @ turn(k * step) for k in ks]).astype(np.float32)
    half = np.stack([gt @ turn((k + 0.5) * step) for k in ks]).astype(np.float32)
    p64 = pts.astype(np.float64) - o
    r = np.linalg.norm(p64 - np.outer(p64 @ axis, axis), axis=1).max()
    diameter = np.linalg.norm(pts[:, None].astype(np.float64) - pts[None, :500], axis=-1).max()
    mssd, _ = metrics.sym_pose_errors(pts, exact, gt, syms, mspd=False)
    assert mssd.max().item() <= 1e-6 * diameter, mssd
    mssd, _ = metrics.sym_pose_errors(pts, half, gt, syms, mspd=False)
    chord = 2 * r * math.sin(math.pi / 630)
    assert mssd.max().item() <= chord + 1e-6 and mssd.min().item() >= 0.99 * chord, (mssd, chord)


def test_bit_identical_across_launch_shapes_and_symmetry_order():
    from foundationpose_b200 import metrics

    rng = np.random.default_rng(13)
    pts = (rng.normal(size=(2620, 3)) * [0.05, 0.03, 0.09]).astype(np.float32)
    syms = _symmetries(1260)
    gt = _random_poses(rng, 1)
    pred = _random_poses(rng, 100)
    m3, m2 = metrics.sym_pose_errors(pts, pred, gt, syms, K0)
    a3, a2 = metrics.sym_pose_errors(pts, pred, gt, syms, K0)
    assert torch.equal(a3, m3) and torch.equal(a2, m2)
    for lo, hi in ((0, 1), (1, 37), (37, 100)):
        a3, a2 = metrics.sym_pose_errors(pts, pred[lo:hi], gt, syms, K0)
        assert torch.equal(a3, m3[lo:hi]) and torch.equal(a2, m2[lo:hi])
    a3, a2 = metrics.sym_pose_errors(pts, pred, np.repeat(gt, 100, axis=0), syms, np.repeat(K0[None], 100, axis=0))
    assert torch.equal(a3, m3) and torch.equal(a2, m2)
    a3, a2 = metrics.sym_pose_errors(pts, pred, gt, syms[rng.permutation(len(syms))], K0)
    assert torch.equal(a3, m3) and torch.equal(a2, m2)
    assert torch.equal(metrics.sym_pose_errors(pts, pred, gt, syms, mspd=False)[0], m3)
    assert torch.equal(metrics.sym_pose_errors(pts, pred, gt, syms, K0, mssd=False)[1], m2)
    # few symmetries split the tiles over more warps: still the same bits as one pose at a time
    b3, b2 = metrics.sym_pose_errors(pts, pred, gt, syms[:3], K0)
    for i in (0, 50, 99):
        a3, a2 = metrics.sym_pose_errors(pts, pred[i], gt, syms[:3], K0)
        assert torch.equal(a3, b3[i:i + 1]) and torch.equal(a2, b2[i:i + 1])
    a3, a2 = metrics.sym_pose_errors(pts, pred[:0], gt, syms, K0)
    assert a3.shape == (0,) and a2.shape == (0,)


def test_projection_from_depth_zero_is_inf_not_nan():
    from foundationpose_b200 import metrics

    pts = np.array([[0.01, 0.02, 0.0], [0.0, 0.01, 0.05], [0.0, 0.0, 0.0]], dtype=np.float32)
    pred = np.repeat(np.eye(4, dtype=np.float32)[None], 2, axis=0)  # depth 0 at the first and last point
    gt = np.eye(4, dtype=np.float32)
    gt[:3, 3] = [0.0, 0.0, 0.5]
    mssd, mspd = metrics.sym_pose_errors(pts, pred, gt, _symmetries(4), K0)
    assert torch.isfinite(mssd).all()
    assert torch.isinf(mspd).all() and not torch.isnan(mspd).any(), mspd
    # only the origin (0 / 0): still inf
    mssd, mspd = metrics.sym_pose_errors(pts[2:], pred, gt, _symmetries(1), K0)
    assert torch.isinf(mspd).all() and not torch.isnan(mspd).any(), mspd


def test_bad_arguments_raise_and_leave_the_device_usable():
    from foundationpose_b200 import _lib, metrics

    lib = _lib.lib
    dev = torch.device("cuda")
    pts = torch.zeros(10, 3, device=dev)
    pred = torch.eye(4, device=dev).reshape(1, 16).repeat(3, 1)
    sym = torch.eye(4, device=dev).reshape(1, 16).repeat(4097, 1)
    K = torch.tensor(K0, dtype=torch.float32, device=dev).reshape(1, 9).repeat(3, 1)
    out = torch.empty(3, device=dev)
    host = np.zeros((4097, 16), dtype=np.float32)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    h = C.c_void_p(host.ctypes.data)
    ok = dict(pts=p(pts), P=10, pred=p(pred), N=3, gt=p(pred), n_gt=1, sym=p(sym), S=4, K=p(K), n_K=1, mssd=p(out),
              mspd=p(out))
    bad = {"null pts": dict(pts=None), "null pred": dict(pred=None), "null gt": dict(gt=None), "null sym": dict(sym=None),
           "host pts": dict(pts=h), "host gt": dict(gt=h), "host sym": dict(sym=h), "host K": dict(K=h),
           "host mssd_out": dict(mssd=h), "host mspd_out": dict(mspd=h), "S = 0": dict(S=0), "S too large": dict(S=4097),
           "P = 0": dict(P=0), "N < 0": dict(N=-1), "n_gt not 1 or N": dict(n_gt=2), "n_K not 1 or N": dict(n_K=2),
           "K missing with mspd_out": dict(K=None)}
    torch.cuda.synchronize()
    launches = lib.fp_launch_count()
    for what, change in bad.items():
        a = {**ok, **change}
        rc = lib.fp_sym_pose_errors(*a.values(), st)
        assert rc != 0, what
        with pytest.raises(_lib.FposeError, match="fp_sym_pose_errors"):
            _lib.check(rc, "fp_sym_pose_errors")
    assert lib.fp_launch_count() == launches
    # K is not needed (and not checked) without mspd_out
    assert lib.fp_sym_pose_errors(*{**ok, "K": None, "n_K": 7, "mspd": None}.values(), st) == 0
    with pytest.raises(_lib.FposeError, match="n_gt"):
        metrics.sym_pose_errors(pts, pred, pred[:2], sym[:4], K0)
    with pytest.raises(_lib.FposeError, match="K"):
        metrics.sym_pose_errors(pts, pred, pred[0], sym[:4])
    torch.cuda.synchronize()
    pts[:, 2] = 1.0
    mssd, mspd = metrics.sym_pose_errors(pts, pred, pred[0], sym[:4], K0)
    assert mssd.sum().item() == 0.0 and mspd.sum().item() == 0.0


def test_eval_bop_results_with_bop(tmp_path):
    """Object 6 (half-turn symmetric) predicted at its ground truth turned by the half turn: MSSD ~ 0, ADD large.
    The other objects shifted by k mm in frame k.  AR columns as computed here from the numpy restatement."""
    import eval_bop_results as ev

    from foundationpose_b200 import metrics, synth

    root = str(tmp_path / "LINEMOD")
    gts = synth.write_bop_dataset(root, "lm", n_frames=4, symmetric=(6,))
    res = {}
    for (vid, id_str, ob_id), pose in gts.items():
        p = np.array(pose, dtype=np.float64)
        if ob_id == 6:
            p = p @ np.diag([-1.0, -1.0, 1.0, 1.0])
        else:
            p[:3, 3] += np.array([0.6, 0.0, 0.8]) * 0.001 * int(id_str)
        res.setdefault(vid, {}).setdefault(id_str, {})[ob_id] = p.tolist()
    res[1]["000003"][1] = np.eye(4).tolist()  # a frame the driver skipped
    path = tmp_path / "linemod_res.yml"
    path.write_text(yaml.safe_dump(res))
    plain_rows, plain_overall = ev.main(["--res", str(path), "--dataset_dir", root])
    rows, overall = ev.main(["--res", str(path), "--dataset_dir", root, "--bop", "--json", str(tmp_path / "t.json")])
    _, _, errors = ev.evaluate(ev.load_results(str(path)), "lm", root, bop=True)
    # without --bop: nothing new
    assert all(set(r) == {"poses", "add_auc", "adds_auc", "add_s_recall", "symmetric", "diameter"} for r in plain_rows.values())
    assert set(plain_overall) == {"poses", "add_auc", "adds_auc", "add_s_recall"}
    assert all(len(e) == 2 for e in ev.evaluate(ev.load_results(str(path)), "lm", root)[2].values())
    for ob_id, r in rows.items():
        assert {k: v for k, v in r.items() if k not in ("mssd_ar", "mspd_ar")} == plain_rows[ob_id]
    add, _, mssd, mspd = errors[6]
    assert mssd.max() < 1e-6 and add.min() > 0.01
    factory = ev.make_reader_factory("lm", root)
    all3, all2, thr3, thr2 = [], [], [], []
    for ob_id, row in rows.items():
        reader = factory(ob_id)  # one scene per object, scene id = object id
        width = reader.get_color(0).shape[1]
        pts = reader.get_gt_mesh(ob_id).vertices.astype(np.float32)
        pred = np.stack([np.asarray(res[ob_id][f"{i:06d}"][ob_id], dtype=np.float32) for i in range(4)])
        gt = np.stack([reader.get_gt_pose(i, ob_id) for i in range(4)]).astype(np.float32)
        K = np.stack([reader.get_K(i) for i in range(4)]).astype(np.float32)
        syms = metrics.bop_symmetries(reader.symmetry_info_table[ob_id]).astype(np.float32)
        want = _numpy_errors(pts, pred, gt, syms, K)
        w3, w2 = np.array([w[0] for w in want]), np.array([w[1] for w in want])
        if ob_id == 1:
            w3[3] = w2[3] = np.inf
        np.testing.assert_allclose(errors[ob_id][2], w3, rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(errors[ob_id][3], w2, rtol=0, atol=1e-3)
        d = reader.get_model_diameter(ob_id)
        t3 = (np.arange(1, 11) * 0.05 * d)[:, None]
        t2 = (np.arange(1, 11) * 5.0 * 640.0 / width)[:, None]
        assert row["mssd_ar"] == pytest.approx(np.mean(w3[None] < t3), abs=1e-12)
        assert row["mspd_ar"] == pytest.approx(np.mean(w2[None] < t2), abs=1e-12)
        all3.append(w3)
        all2.append(w2)
        thr3.append(np.repeat(t3, 4, axis=1))
        thr2.append(np.repeat(t2, 4, axis=1))
    assert overall["mssd_ar"] == pytest.approx(np.mean(np.concatenate(all3)[None] < np.concatenate(thr3, axis=1)), abs=1e-12)
    assert overall["mspd_ar"] == pytest.approx(np.mean(np.concatenate(all2)[None] < np.concatenate(thr2, axis=1)), abs=1e-12)
    assert overall["mssd_ar"] < 1.0  # the skipped frame is a failure
    assert os.path.exists(tmp_path / "t.json")
