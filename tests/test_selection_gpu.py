"""The kernels that make the register calls' final decisions, against float64 references (tests/tail_reference.py):

  * the segmented scorer tail (cross_attn_score_kernel with seg / n_seg / seg_max, through fp_op_score_tail_segments, which
    sets its launch up with the same helper as fp_register_objects / _cameras): scores within derived bars, each
    segment's first arg-max, bit-equality with one-segment launches, the per-segment tickets between launches;
  * pose_update_kernel through the mesh table (fp_op_pose_update launches it as the refine loop does);
  * frame_prep_kernel's camera-table instantiation (fp_get_depth per camera) and the start poses of fp_register_cameras.

Each check prints its worst error / bar ratio."""
import numpy as np
import pytest
import torch

import tail_reference as tr

pytestmark = pytest.mark.gpu

DIAMETERS = (0.05, 0.31, 0.74, 1.2)  # mesh slots 0..3
LAYOUTS = {
    "252": [252],
    "objects": [252, 126, 63, 20],
    "64 x 1": [1] * 64,
    "strides": [31, 32, 33, 127, 128, 129],
    "4096": [4096],
    "1 4096 2": [1, 4096, 2],
    "252 252 20": [252, 252, 20],
    "20 252 252": [20, 252, 252],
    "252 20 252": [252, 20, 252],
}


def _offsets(sizes):
    return [0] + np.cumsum(sizes).tolist()


@pytest.fixture(scope="module")
def rig():
    from foundationpose_b200 import synth
    from foundationpose_b200.engine import Engine
    from foundationpose_b200.weights import random_state_dict
    from oracle import pipeline

    e = Engine()
    sd_s = random_state_dict("score", 0)
    e.load_network("refine", random_state_dict("refine", 0))
    e.load_network("score", sd_s)
    mesh = synth.make_mesh(2)
    mt = pipeline.mesh_tensors(mesh)
    for slot, d in enumerate(DIAMETERS):
        e.set_mesh(mt["pos"], mt["normals"], mt["faces"], d, uv=mt["uv"], tex=mt["tex"], slot=slot)
    return dict(e=e, sd=sd_s, sd64=tr.state_dict64(sd_s, "cuda"), mesh=mesh)


def _features(sizes, seed, sd64, peaked):
    """Random rows at the scale of test_score_tail_252 (x 2), or scaled so the largest logit is ~60 (one key dominates
    each softmax); every segment of >= 129 rows has an exact tie of
    its best row at index 5 and at an index >= 128 that a lower-numbered thread of the 128-thread arg-max visits; with
    two or more segments of >= 2 rows, the shortest of them has identical rows."""
    g = torch.Generator().manual_seed(seed)
    seg = _offsets(sizes)
    x = (torch.randn(seg[-1], 512, generator=g) * 2).cuda().double()
    if peaked:
        s_max = 0.0
        for a, b in tr.spans(seg):
            qkv = x[a:b] @ sd64["att_cross.in_proj_weight"].t()
            s_max = max(s_max, float((qkv[:, :512] @ qkv[:, 512:1024].t()).abs().max()) / 128 ** 0.5 / 4)
        x = x * (60.0 / s_max) ** 0.5
    x = x.float().double()  # fp32 features
    multi = [i for i, n in enumerate(sizes) if n >= 2]
    same = min(multi, key=lambda i: sizes[i]) if len(multi) >= 2 else None
    ties = []
    if same is not None:
        a, b = seg[same], seg[same + 1]
        x[a:b] = x[a]
    for gi, n in enumerate(sizes):
        if n < 129 or gi == same:
            continue
        a = seg[gi]
        j = 128 + min(2, n - 129)  # visited by thread j - 128 < 5
        for _ in range(6):  # copy the best row to rows 5 and j until the pair is the segment's maximum
            ref = tr.tail_ref(sd64, x, seg)[a:a + n]
            r = tr.first_argmax(ref)
            if r in (5, j):
                break
            x[a + 5] = x[a + r]
            x[a + j] = x[a + r]
        ties.append((gi, 5, j))
    return x, seg, same, ties


def _run(e, x, seg, scores=None, best=None):
    scores = torch.full((seg[-1],), float("nan"), device="cuda") if scores is None else scores.fill_(float("nan"))
    best = torch.full((len(seg) - 1,), -7, dtype=torch.int32, device="cuda") if best is None else best.fill_(-7)
    e.score_tail_segments(x.float(), seg, scores, best)
    torch.cuda.synchronize()
    return scores, best


@pytest.mark.parametrize("peaked", [False, True], ids=["random", "peaked"])
@pytest.mark.parametrize("name", list(LAYOUTS))
def test_segmented_tail_against_float64(rig, name, peaked):
    """Scores within the derived bar of tail_reference.tail_bar; best[g] = the first arg-max of the kernel's own scores
    of segment g, and the float64 arg-max wherever the float64 top-2 margin exceeds twice the bar; identical rows give
    bit-equal scores and best 0; an exact tie goes to the lower index; every segment is bit-equal to a one-segment launch
    over its rows alone (fp_score_tail, no segment table); the outputs are filled with NaN / -7 first, so a score or
    an arg-max the kernel never wrote (a ticket left non-zero by an earlier launch) fails."""
    e, sd64 = rig["e"], rig["sd64"]
    sizes = LAYOUTS[name]
    x, seg, same, ties = _features(sizes, 100 + len(sizes) + sizes[0], sd64, peaked)
    scores, best = _run(e, x, seg)
    got = scores.double()
    ref = tr.tail_ref(sd64, x, seg)
    bar = tr.tail_bar(sd64, x, seg)
    assert torch.isfinite(got).all()
    ratio = float(((got - ref).abs() / bar).max())
    print(f"\n[{name} {'peaked' if peaked else 'random'}] worst |score - float64| / bar = {ratio:.3g}, "
          f"bar {float(bar.min()):.3g} .. {float(bar.max()):.3g}")
    assert ratio <= 1.0
    best = best.cpu().tolist()
    checked = 0
    for gi, (a, b) in enumerate(tr.spans(seg)):
        mine = scores[a:b].cpu()
        assert best[gi] == tr.first_argmax(mine), f"segment {gi}: best {best[gi]}"
        r = ref[a:b].cpu()
        top = torch.topk(r, min(2, b - a)).values
        if b - a == 1 or float(top[0] - top[1]) > 2 * float(bar[a:b].max()):
            assert best[gi] == tr.first_argmax(r), f"segment {gi}: best {best[gi]}, float64 {tr.first_argmax(r)}"
            checked += 1
        alone, best1 = e.score_tail(x[a:b].float())
        assert torch.equal(alone, scores[a:b]) and int(best1.item()) == best[gi], f"segment {gi} differs from its own launch"
    print(f"[{name}] best checked against float64 in {checked} of {len(sizes)} segments")
    if same is not None:
        a, b = seg[same], seg[same + 1]
        assert (scores[a:b] == scores[a]).all() and best[same] == 0
    for gi, i, j in ties:
        a = seg[gi]
        assert scores[a + i] == scores[a + j]
        if tr.first_argmax(scores[a:seg[gi + 1]].cpu()) in (i, j):
            assert best[gi] == i, f"segment {gi}: tie at {i} and {j} went to {best[gi]}"


def test_one_segment_is_the_unsegmented_tail(rig):
    e, sd64 = rig["e"], rig["sd64"]
    for L in (252, 4096, 129):
        x, seg, _, _ = _features([L], 7 + L, sd64, False)
        s1, b1 = _run(e, x, seg)
        s0, b0 = e.score_tail(x.float())
        assert torch.equal(s1, s0) and torch.equal(b1, b0.to(b1.dtype))


def test_tickets_between_launches(rig):
    """64 one-row segments, then [252], then the 64 segments again: identical results (each segment's last CTA resets
    its ticket word, and the one-segment launch shares word 0)."""
    e, sd64 = rig["e"], rig["sd64"]
    x64, seg64, _, _ = _features([1] * 64, 3, sd64, False)
    x252, seg252, _, _ = _features([252], 4, sd64, False)
    s_a, b_a = _run(e, x64, seg64)
    s_m, b_m = _run(e, x252, seg252)
    s_b, b_b = _run(e, x64, seg64)
    assert torch.equal(s_a.clone(), s_b) and torch.equal(b_a.clone(), b_b)
    s_m2, b_m2 = e.score_tail(x252.float())
    assert torch.equal(s_m, s_m2) and torch.equal(b_m, b_m2)


def test_probes_are_rejected(rig):
    """The comparison sees slightly wrong references: a segment whose keys include its neighbour's first row, the
    softmax scale 1/sqrt(512) (q halved), the out_proj bias dropped.  Prints the fraction of scores each one fails."""
    e, sd64 = rig["e"], rig["sd64"]
    sd_scale = dict(sd64)
    sd_scale["att_cross.in_proj_weight"] = sd64["att_cross.in_proj_weight"].clone()
    sd_scale["att_cross.in_proj_bias"] = sd64["att_cross.in_proj_bias"].clone()
    sd_scale["att_cross.in_proj_weight"][:512] *= 0.5
    sd_scale["att_cross.in_proj_bias"][:512] *= 0.5
    sd_nob = dict(sd64)
    sd_nob["att_cross.out_proj.bias"] = torch.zeros_like(sd64["att_cross.out_proj.bias"])
    for name in ("objects", "strides"):
        x, seg, _, _ = _features(LAYOUTS[name], 11, sd64, False)
        got = _run(e, x, seg)[0].double()
        bar = tr.tail_bar(sd64, x, seg)
        n0 = seg[1]
        probes = {"neighbour's first row": (tr.tail_ref(sd64, x, seg, extra_key=0), slice(0, n0)),
                  "1/sqrt(512)": (tr.tail_ref(sd_scale, x, seg), slice(None)),
                  "no out_proj bias": (tr.tail_ref(sd_nob, x, seg), slice(None))}
        for what, (p, sl) in probes.items():
            frac = float(((got - p).abs() > bar)[sl].double().mean())
            print(f"\n[{name}] probe {what}: fails on {frac * 100:.1f}% of the scores it changes")
            assert frac > 0, what


def test_refusals_launch_nothing(rig):
    from foundationpose_b200 import _lib

    e = rig["e"]
    x = torch.randn(300, 512, device="cuda")
    n0 = _lib.launch_count()
    for seg in ([1, 300], [0, 100, 100, 300], [0, 200, 150, 300], [0, 299], [0, 301], [0]):
        with pytest.raises(_lib.FposeError):
            e.score_tail_segments(x, seg)
    xl = torch.randn(4097, 512, device="cuda")
    with pytest.raises(_lib.FposeError):
        e.score_tail_segments(xl, [0, 4097])
    assert _lib.launch_count() == n0


def test_register_objects_unchanged_by_the_hook(rig):
    from foundationpose_b200 import hypotheses, synth

    e = rig["e"]
    pose = np.eye(4)
    pose[:3, :3] = synth.random_rotation(3)
    pose[:3, 3] = [0.01, -0.02, 0.6]
    rgb, depth, mask = synth.make_scene(rig["mesh"].visual.image, pose)
    grid = torch.from_numpy(hypotheses.make_rotation_grid()).float().cuda()
    args = (rgb, depth, synth.DEFAULT_K, np.stack([mask, mask]), [grid[:40], grid[40:60]], [1, 2], 1)
    before = [t.clone() for t in e.register_objects(*args)]
    x, seg, _, _ = _features([1, 4096, 2], 5, rig["sd64"], False)
    _run(e, x, seg)
    x, seg, _, _ = _features([1] * 64, 6, rig["sd64"], False)
    _run(e, x, seg)
    after = e.register_objects(*args)
    for u, v in zip(before, after):
        assert torch.equal(u, v)


# ------------------------------------------------------------------------------------------------------------------
# pose update through the mesh table
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 127, 128, 129, 252, 504])
def test_pose_update_through_the_mesh_table(rig, N):
    """Poses, trans_delta and rot_delta of fp_op_pose_update against tail_reference.pose_update_ref at the bars of
    tail_reference.pose_update_bars.  rot rows cycle through 0, |tanh(rot) rn| = 0.01 (1 - 1e-3) and 0.01 (1 + 1e-3)
    (either side of so3_exp_map's clamp of the squared norm at 1e-4), |rot| = 10 (tanh saturated) and random; each
    hypothesis takes one of four mesh slots (diameters 0.05 .. 1.2 m)."""
    from oracle import geometry

    e = rig["e"]
    rn = np.float32(0.3490658503988659)
    g = torch.Generator().manual_seed(N)
    poses = torch.eye(4).repeat(N, 1, 1)
    poses[:, :3, :3] = geometry.so3_exp_map(torch.randn(N, 3, generator=g) * 2)
    poses[:, :3, 3] = torch.randn(N, 3, generator=g) * 0.2 + torch.tensor([0.0, 0.0, 0.8])
    trans = torch.randn(N, 3, generator=g)
    rot = torch.randn(N, 3, generator=g)
    dirs = torch.nn.functional.normalize(torch.randn(N, 3, generator=g, dtype=torch.float64), dim=1)
    for i in range(N):
        kind = i % 5
        if kind == 0:
            rot[i] = 0
        elif kind in (1, 2):
            r = 0.01 * (1 - 1e-3 if kind == 1 else 1 + 1e-3)
            rot[i] = torch.atanh(dirs[i] * r / float(rn)).float()
        elif kind == 3:
            rot[i] = torch.sign(rot[i]) * 10
    mesh_of = torch.randint(0, 4, (N,), generator=g)
    out, td, rd = e.op_pose_update(poses.cuda(), trans.cuda(), rot.cuda(), mesh_of.tolist())
    half = torch.tensor([np.float32(DIAMETERS[m]) / np.float32(2) for m in mesh_of.tolist()], dtype=torch.float64)
    ref, td_ref, rd_ref = tr.pose_update_ref(poses, trans, rot, half, rn)
    nrm = ((torch.tanh(rot.double()) * float(rn)) ** 2).sum(1)
    assert ((nrm[1::5] < 1e-4).all() and (nrm[2::5] > 1e-4).all())
    bar_R, bar_td, bar_t = tr.pose_update_bars(poses, rd_ref, td_ref)
    out, td, rd = out.cpu().double(), td.cpu().double(), rd.cpu().double()
    ratios = {"rot_delta": float(((rd - rd_ref).abs() / tr.ROT_DELTA_BAR).max()),
              "R": float(((out[:, :3, :3] - ref[:, :3, :3]).abs() / bar_R).max()),
              "trans_delta": float(((td - td_ref).abs() / bar_td.clamp_min(1e-300)).max()),
              "t": float(((out[:, :3, 3] - ref[:, :3, 3]).abs() / bar_t).max())}
    print(f"\n[N = {N}] worst error / bar: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()))
    assert all(v <= 1.0 for v in ratios.values()), ratios
    assert torch.equal(out[:, 3], torch.tensor([0.0, 0.0, 0.0, 1.0], dtype=torch.float64).repeat(N, 1))
    # no slot ids = slot 0 for every hypothesis; a slot without a mesh is refused before any launch
    out0, _, _ = e.op_pose_update(poses.cuda(), trans.cuda(), rot.cuda())
    out0s, _, _ = e.op_pose_update(poses.cuda(), trans.cuda(), rot.cuda(), [0] * N)
    assert torch.equal(out0, out0s)
    from foundationpose_b200 import _lib

    n0 = _lib.launch_count()
    with pytest.raises(_lib.FposeError):
        e.op_pose_update(poses.cuda(), trans.cuda(), rot.cuda(), [5] * N)
    assert _lib.launch_count() == n0


# ------------------------------------------------------------------------------------------------------------------
# frame preparation and start poses through the camera table
# ------------------------------------------------------------------------------------------------------------------
SIZES = [(121, 177), (97, 131), (33, 40), (480, 640)]


def _frame(H, W, seed):
    """A depth plane with noise, holes, steps, values just under 0.001 and near zfar = 100 within 2 px of every border
    and on the 32 x 8 tile seams."""
    rng = np.random.default_rng(seed)
    d = (0.6 + 0.3 * np.linspace(0, 1, W)[None, :] + 0.001 * rng.standard_normal((H, W))).astype(np.float32)
    d = np.repeat(d, 1, 0)
    d[: H // 2] += 0.05  # a step
    special = np.array([0.0, 0.00099, 0.0009999, 99.99, 100.0, 100.01, 0.7], dtype=np.float32)
    rows = sorted({0, 1, H - 2, H - 1} | {r for r in range(7, H, 8)} | {r for r in range(8, H, 8)})
    cols = sorted({0, 1, W - 2, W - 1} | {c for c in range(31, W, 32)} | {c for c in range(32, W, 32)})
    for r in rows:
        pick = rng.random(W) < 0.25
        d[r, pick] = rng.choice(special, pick.sum())
    for c in cols:
        pick = rng.random(H) < 0.25
        d[pick, c] = rng.choice(special, pick.sum())
    d[rng.random((H, W)) < 0.02] = 0  # holes
    rgb = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    K = np.array([[W * 0.9, 0, W / 2 - 0.5], [0, W * 0.9, H / 2 + 0.25], [0, 0, 1]], dtype=np.float32).astype(np.float64)
    return rgb, d, K


def test_frames_and_start_poses_through_the_camera_table(rig):
    """fp_register_cameras(iterations = 0) over four cameras of different sizes: every camera's filtered depth and xyz
    map (frame_prep_kernel<true>, one grid over the largest frame) against oracle erode_depth -> bilateral_filter_depth
    -> depth2xyzmap at 2e-6 / 1e-6 and bit-equal to fp_set_frame of that frame alone (the by-value instantiation); the
    start poses' translation against hypotheses.guess_translation on the reference-filtered depth within 1 ulp of the
    fp32 median (scaled to each component), n_valid exact, rotation blocks bit-equal to the grid."""
    from foundationpose_b200 import _lib, hypotheses
    from oracle import geometry

    e = rig["e"]
    frames = [_frame(H, W, 20 + i) for i, (H, W) in enumerate(SIZES)]
    rgb3, d3, K3 = frames[3]
    d3 = d3.copy()
    d3[200:260, 300:400] = np.float32(0.8125)  # a region of equal depths
    d3[::7, ::5] *= np.float32(2.0) ** np.random.default_rng(9).integers(-3, 4, d3[::7, ::5].shape).astype(np.float32)
    frames[3] = (rgb3, d3, K3)
    ref_depth = [geometry.bilateral_filter_depth(geometry.erode_depth(d)) for _, d, _ in frames]
    masks, camera_of = [], []
    for cam, (H, W) in enumerate(SIZES):
        f = ref_depth[cam]
        m = np.zeros((H, W), np.uint8)
        m[0, 0] = 1
        masks.append(m), camera_of.append(cam)
        m = np.zeros((H, W), np.uint8)
        m[H - 1, W - 1] = 1
        masks.append(m), camera_of.append(cam)
    H, W = SIZES[3]
    f = ref_depth[3]
    masks.append(np.ones((H, W), np.uint8)), camera_of.append(3)  # the full frame
    m = np.zeros((H, W), np.uint8)
    m[210:250, 310:390] = 1  # inside the region of equal depths
    masks.append(m), camera_of.append(3)
    m = np.zeros((H, W), np.uint8)
    valid = np.argwhere(f >= 0.001)
    m[tuple(valid[5])] = 1
    m[tuple(valid[-9])] = 1  # exactly two valid pixels
    masks.append(m), camera_of.append(3)
    m = np.zeros((H, W), np.uint8)
    m[::7, ::5] = 1  # depths scaled by 2^-3 .. 2^3
    masks.append(m), camera_of.append(3)
    frames3 = frames
    grid = torch.from_numpy(hypotheses.make_rotation_grid()).float().cuda()
    grids = [grid[3 * i:3 * i + 3] for i in range(len(masks))]
    poses, _, _, info = e.register_cameras(frames3, masks, grids, camera_of, [0] * len(masks), 0)
    torch.cuda.synchronize()
    table = [tuple(t.cpu().numpy() for t in e.get_depth(cam)) for cam in range(4)]
    with pytest.raises(_lib.FposeError):
        e.get_depth(4)
    worst_d = worst_x = 0.0
    for cam, (rgb, d, K) in enumerate(frames3):
        dd, xx = table[cam]
        assert dd.shape == SIZES[cam] and xx.shape == (*SIZES[cam], 3)
        ref_x = geometry.depth2xyzmap(ref_depth[cam], K)
        worst_d = max(worst_d, float(np.abs(dd - ref_depth[cam]).max()) / 2e-6)
        worst_x = max(worst_x, float(np.abs(xx - ref_x).max()) / 1e-6)
        np.testing.assert_allclose(dd, ref_depth[cam], atol=2e-6, rtol=0)
        np.testing.assert_allclose(xx, ref_x, atol=1e-6, rtol=0)
        e.set_frame(rgb, d, K, filter_depth=True)
        d1, x1 = (t.cpu().numpy() for t in e.get_depth())
        np.testing.assert_array_equal(d1, dd)
        np.testing.assert_array_equal(x1, xx)
        with pytest.raises(_lib.FposeError):
            e.get_depth(1)
    print(f"\nframes: worst depth error / 2e-6 = {worst_d:.3g}, xyz / 1e-6 = {worst_x:.3g}")
    info = info.cpu().numpy()
    p = poses.cpu().numpy().reshape(len(masks), 3, 4, 4)
    worst_t = 0.0
    for i, (m, cam) in enumerate(zip(masks, camera_of)):
        f, K = ref_depth[cam], frames3[cam][2]
        ref_t = hypotheses.guess_translation(f, m, K)
        valid = (m > 0) & (f >= 0.001)
        assert int(info[i, 3]) == int(valid.sum()), f"object {i}"
        zc = float(np.median(f[valid])) if valid.any() else 0.0
        bar = np.spacing(np.float32(zc)) * np.maximum(1.0, np.abs(ref_t) / max(zc, 1e-30)) + 4 * tr.U * np.abs(ref_t) + 1e-30
        worst_t = max(worst_t, float((np.abs(info[i, :3] - ref_t) / bar).max()))
        assert (np.abs(info[i, :3] - ref_t) <= bar).all(), f"object {i}: {info[i, :3]} vs {ref_t}"
        np.testing.assert_array_equal(p[i, :, :3, :3], grids[i].cpu().numpy()[:, :3, :3])
    print(f"start poses: worst translation error / bar = {worst_t:.3g}")

