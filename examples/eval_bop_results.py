"""ADD / ADD-S tables for the result files of the dataset drivers (run_linemod.py -> linemod_res.yml, run_ycb_video.py ->
ycbv_res.yml, examples/run_linemod_replicas.py), scored on the GPU.

    python examples/eval_bop_results.py --res debug/linemod_res.yml --dataset_dir <LINEMOD root> [--json table.json]
    python examples/eval_bop_results.py --res debug/ycbv_res.yml --dataset_dir <YCB_Video root> [--kind ycbv]
    python examples/eval_bop_results.py --res debug/linemod_res.yml --dataset_dir <LINEMOD root> --vsd

A result file maps video id -> frame id string -> object id -> 4x4 estimated pose.  The ground truth comes from the
drop-in readers (`get_gt_pose`), the model points from `get_gt_mesh(ob_id).vertices`; all poses of one object go to
one `fp_pose_errors` call.  A frame the driver skipped (it writes the identity) counts as a failure: its errors are
infinite.  An object is symmetric when the reader's `symmetry_tfs[ob_id]` holds more than the identity.  Printed per
object and overall: the number of poses, ADD and ADD-S AUC (up to 0.1 m in 1 mm steps) and ADD(-S) < 0.1 d (ADD-S for
symmetric objects, d = `get_model_diameter`).

--bop adds BOP's symmetry-aware average recalls, scored by `fp_sym_pose_errors`: AR_MSSD over the thresholds
0.05 d .. 0.50 d and AR_MSPD over 5 .. 50 px scaled by 640 / image width, both as the mean over the thresholds of the
share of errors below each.  The symmetries are those of `models_info.json` (`reader.symmetry_info_table`) sampled by
`metrics.bop_symmetries`, K is `reader.get_K(frame)` and the image width that of the video's frames.  The overall row
scores every pose with its own object's thresholds.  The errors are taken over the same model vertices as the ADD
columns, not over BOP's resampled `models_eval` points, so they are not comparable with the BOP leaderboard; and
without --vsd no combined BOP AR is printed.

--vsd (implies --bop) adds BOP's visible surface discrepancy, scored by `fp_vsd_errors`: the model (`get_gt_mesh`,
vertices and faces) is rendered at the estimated and at the ground-truth pose against the test depth
(`reader.get_depth(frame)`) with delta = 15 mm and the step cost at tau = 0.05 d .. 0.50 d.  AR_VSD is the mean over
every (tau, threshold 0.05 .. 0.50) pair of the share of poses with an error below the threshold, and BOP AR =
(AR_VSD + AR_MSSD + AR_MSPD) / 3, per object and overall.  A skipped frame counts as a failure for every tau.  The
renderer follows the crop producer's coverage rule, not bop_toolkit's OpenGL renderer: the two may differ on silhouette
pixels.  The models_eval caveat of MSSD / MSPD applies to BOP AR as well.
"""
import argparse
import json
import os
import sys
from collections import defaultdict

import numpy as np
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "foundationpose_b200", "dropin"), ROOT]

from foundationpose_b200 import metrics  # noqa: E402


def load_results(path):
    with open(path) as fh:
        return yaml.safe_load(fh) or {}


def group_by_object(res):
    """{ob_id: [(video_id, id_str, pose 4x4 float64, skipped)]} in video, frame order."""
    groups = defaultdict(list)
    for video_id in sorted(res, key=int):
        for id_str in sorted(res[video_id], key=str):
            for ob_id, pose in res[video_id][id_str].items():
                pose = np.asarray(pose, dtype=np.float64).reshape(4, 4)
                groups[int(ob_id)].append((int(video_id), str(id_str), pose, bool(np.array_equal(pose, np.eye(4)))))
    return dict(sorted(groups.items()))


def is_symmetric(symmetry_tfs):
    tfs = np.asarray(symmetry_tfs, dtype=np.float64).reshape(-1, 4, 4)
    return any(not np.allclose(tf, np.eye(4)) for tf in tfs)


def summarize(add, adds, symmetric, diameter):
    """One table row from per-pose errors (inf for failures)."""
    add, adds = np.asarray(add, dtype=np.float64), np.asarray(adds, dtype=np.float64)
    return {"poses": int(len(add)), "add_auc": metrics.auc(add), "adds_auc": metrics.auc(adds),
            "add_s_recall": metrics.recall(adds if symmetric else add, 0.1 * diameter), "symmetric": bool(symmetric),
            "diameter": float(diameter)}


def summarize_all(rows, errors):
    """Overall row: AUCs over every pose, ADD(-S) < 0.1 d with each pose's own metric and diameter."""
    add = np.concatenate([errors[o][0] for o in rows])
    adds = np.concatenate([errors[o][1] for o in rows])
    crit = np.concatenate([errors[o][1] if rows[o]["symmetric"] else errors[o][0] for o in rows])
    thr = np.concatenate([np.full(rows[o]["poses"], 0.1 * rows[o]["diameter"]) for o in rows])
    return {"poses": int(len(add)), "add_auc": metrics.auc(add), "adds_auc": metrics.auc(adds),
            "add_s_recall": metrics.recall(crit, thr)}


def bop_thresholds(diameter, widths):
    """([T, n] MSSD, [T, n] MSPD) thresholds of n poses of one object, `widths` the image width of each pose's frame."""
    widths = np.asarray(widths, dtype=np.float64).reshape(-1)
    mssd = np.repeat(metrics.mssd_thresholds(diameter)[:, None], len(widths), axis=1)
    mspd = np.stack([metrics.mspd_thresholds(w) for w in widths], axis=1).reshape(len(metrics.MSPD_STEPS), -1)
    return mssd, mspd


def summarize_bop(mssd, mspd, thresholds):
    """AR_MSSD and AR_MSPD of one row from per-pose errors (inf for failures) and their [T, n] thresholds."""
    return {"mssd_ar": metrics.average_recall(mssd, thresholds[0]), "mspd_ar": metrics.average_recall(mspd, thresholds[1])}


def summarize_bop_all(errors, thresholds):
    """Overall AR_MSSD / AR_MSPD: every pose, each with its own object's thresholds."""
    cat = lambda lists: np.concatenate(lists, axis=-1)  # noqa: E731
    return summarize_bop(cat([errors[o][2] for o in errors]), cat([errors[o][3] for o in errors]),
                         (cat([thresholds[o][0] for o in errors]), cat([thresholds[o][1] for o in errors])))


VSD_CHUNK = 64  # poses per fp_vsd_errors call: their test depths are on the device together


def vsd_chunks(entries, shapes):
    """Index ranges [lo, hi) of consecutive entries with the same frame size, at most VSD_CHUNK long."""
    out, lo = [], 0
    for i in range(1, len(entries) + 1):
        if i == len(entries) or i - lo == VSD_CHUNK or shapes[i] != shapes[lo]:
            out.append((lo, i))
            lo = i
    return out


def summarize_vsd(vsd, mssd_ar, mspd_ar):
    """AR_VSD of one row from its per-pose errors [n, T] (inf for failures), and the BOP AR with the row's AR_MSSD and
    AR_MSPD."""
    ar = metrics.vsd_average_recall(vsd)
    return {"vsd_ar": ar, "bop_ar": metrics.bop_ar(ar, mssd_ar, mspd_ar)}


def make_reader_factory(kind, dataset_dir):
    from datareader import LinemodReader, YcbVideoReader

    cache = {}

    def reader(video_id):
        if video_id not in cache:
            if kind == "lm":
                cache[video_id] = LinemodReader(os.path.join(dataset_dir, "lm_test_all", "test", f"{video_id:06d}"), split=None)
            else:
                os.environ.setdefault("YCB_VIDEO_DIR", dataset_dir)
                cache[video_id] = YcbVideoReader(os.path.join(dataset_dir, "test", f"{video_id:06d}"))
        return cache[video_id]

    return reader


def evaluate(res, kind, dataset_dir, bop=False, vsd=False):
    """-> (rows {ob_id: row}, overall row, errors {ob_id: (add [n], adds [n])}).  With `bop`, every row also holds
    `mssd_ar` and `mspd_ar`, and errors[ob_id] is (add, adds, mssd [n], mspd [n]).  `vsd` implies `bop`: every row
    also holds `vsd_ar` and `bop_ar`, and errors[ob_id] gains vsd [n, T]."""
    bop = bop or vsd
    reader = make_reader_factory(kind, dataset_dir)
    rows, errors, thresholds, widths = {}, {}, {}, {}
    for ob_id, entries in group_by_object(res).items():
        r0 = reader(entries[0][0])
        frame = {vid: {s: i for i, s in enumerate(reader(vid).id_strs)} for vid in {e[0] for e in entries}}
        gt = np.stack([reader(vid).get_gt_pose(frame[vid][id_str], ob_id) for vid, id_str, _, _ in entries])
        pred = np.stack([e[2] for e in entries])
        skipped = np.array([e[3] for e in entries])
        pts = r0.get_gt_mesh(ob_id).vertices
        add, adds = metrics.pose_errors(pts, pred, gt)
        add, adds = add.double().cpu().numpy(), adds.double().cpu().numpy()
        add[skipped], adds[skipped] = np.inf, np.inf
        errors[ob_id] = (add, adds)
        rows[ob_id] = summarize(add, adds, is_symmetric(r0.symmetry_tfs[ob_id]), r0.get_model_diameter(ob_id))
        if bop:
            K = np.stack([reader(vid).get_K(frame[vid][id_str]) for vid, id_str, _, _ in entries])
            for vid in frame:
                if vid not in widths:
                    widths[vid] = reader(vid).get_color(0).shape[1]
            syms = metrics.bop_symmetries(r0.symmetry_info_table[ob_id])
            mssd, mspd = metrics.sym_pose_errors(pts, pred, gt, syms, K)
            mssd, mspd = mssd.double().cpu().numpy(), mspd.double().cpu().numpy()
            mssd[skipped], mspd[skipped] = np.inf, np.inf
            errors[ob_id] = (add, adds, mssd, mspd)
            thresholds[ob_id] = bop_thresholds(r0.get_model_diameter(ob_id), [widths[e[0]] for e in entries])
            rows[ob_id].update(summarize_bop(mssd, mspd, thresholds[ob_id]))
        if vsd:
            mesh = r0.get_gt_mesh(ob_id)
            diameter = r0.get_model_diameter(ob_id)
            depths = [None if e[3] else reader(e[0]).get_depth(frame[e[0]][e[1]]) for e in entries]
            shapes = [None if d is None else d.shape for d in depths]
            err = np.full((len(entries), len(metrics.VSD_TAUS)), np.inf)
            for lo, hi in vsd_chunks(entries, shapes):
                if shapes[lo] is None:
                    continue  # skipped frames: failures for every tau
                err[lo:hi] = metrics.vsd_errors(mesh.vertices, mesh.faces, pred[lo:hi], gt[lo:hi], np.stack(depths[lo:hi]),
                                                K[lo:hi], diameter).double().cpu().numpy()
            errors[ob_id] = errors[ob_id] + (err,)
            rows[ob_id].update(summarize_vsd(err, rows[ob_id]["mssd_ar"], rows[ob_id]["mspd_ar"]))
    overall = summarize_all(rows, errors) if rows else None
    if bop and rows:
        overall.update(summarize_bop_all(errors, thresholds))
    if vsd and rows:
        overall.update(summarize_vsd(np.concatenate([errors[o][4] for o in rows]), overall["mssd_ar"], overall["mspd_ar"]))
    return rows, overall, errors


def print_table(rows, overall, bop=False, vsd=False):
    if vsd:
        print(f"{'object':>8} {'poses':>6} {'ADD AUC':>8} {'ADD-S AUC':>10} {'ADD(-S)<0.1d':>13} {'AR MSSD':>8} {'AR MSPD':>8} "
              f"{'AR VSD':>7} {'BOP AR':>7}")
        for tag, r in [(f"{o}{'*' if r['symmetric'] else ''}", r) for o, r in rows.items()] + ([("all", overall)] if overall else []):
            print(f"{tag:>8} {r['poses']:6d} {100 * r['add_auc']:8.2f} {100 * r['adds_auc']:10.2f} {100 * r['add_s_recall']:13.2f} "
                  f"{100 * r['mssd_ar']:8.2f} {100 * r['mspd_ar']:8.2f} {100 * r['vsd_ar']:7.2f} {100 * r['bop_ar']:7.2f}")
        print("(percent; * = symmetric object, scored by ADD-S in the fifth column; MSSD / MSPD over the model vertices, "
              "not BOP's models_eval points; VSD with delta = 15 mm and the step cost, rendered with the crop producer's "
              "coverage rule; BOP AR = mean of the three ARs)")
        return
    if not bop:
        print(f"{'object':>8} {'poses':>6} {'ADD AUC':>8} {'ADD-S AUC':>10} {'ADD(-S)<0.1d':>13}")
        for ob_id, r in rows.items():
            tag = f"{ob_id}{'*' if r['symmetric'] else ''}"
            print(f"{tag:>8} {r['poses']:6d} {100 * r['add_auc']:8.2f} {100 * r['adds_auc']:10.2f} {100 * r['add_s_recall']:13.2f}")
        if overall:
            print(f"{'all':>8} {overall['poses']:6d} {100 * overall['add_auc']:8.2f} {100 * overall['adds_auc']:10.2f} "
                  f"{100 * overall['add_s_recall']:13.2f}")
        print("(percent; * = symmetric object, scored by ADD-S in the last column)")
        return
    print(f"{'object':>8} {'poses':>6} {'ADD AUC':>8} {'ADD-S AUC':>10} {'ADD(-S)<0.1d':>13} {'AR MSSD':>8} {'AR MSPD':>8}")
    for tag, r in [(f"{o}{'*' if r['symmetric'] else ''}", r) for o, r in rows.items()] + ([("all", overall)] if overall else []):
        print(f"{tag:>8} {r['poses']:6d} {100 * r['add_auc']:8.2f} {100 * r['adds_auc']:10.2f} {100 * r['add_s_recall']:13.2f} "
              f"{100 * r['mssd_ar']:8.2f} {100 * r['mspd_ar']:8.2f}")
    print("(percent; * = symmetric object, scored by ADD-S in the fifth column; MSSD / MSPD over the model vertices, "
          "not BOP's models_eval points, and without VSD, so there is no BOP AR)")


def make_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", required=True, help="linemod_res.yml / ycbv_res.yml written by a dataset driver")
    ap.add_argument("--dataset_dir", required=True, help="the --linemod_dir / --ycbv_dir the driver ran on")
    ap.add_argument("--kind", choices=("lm", "ycbv"), default=None, help="default: ycbv if the file name says so, else lm")
    ap.add_argument("--json", default=None, help="also write the table as JSON here")
    ap.add_argument("--bop", action="store_true", help="also BOP's symmetry-aware AR_MSSD and AR_MSPD")
    ap.add_argument("--vsd", action="store_true", help="also BOP's AR_VSD and the combined BOP AR (implies --bop)")
    return ap


def parse_args(argv=None):
    opt = make_parser().parse_args(argv)
    opt.bop = opt.bop or opt.vsd
    return opt


def main(argv=None):
    opt = parse_args(argv)
    kind = opt.kind or ("ycbv" if "ycbv" in os.path.basename(opt.res) else "lm")
    rows, overall, _ = evaluate(load_results(opt.res), kind, opt.dataset_dir, bop=opt.bop, vsd=opt.vsd)
    print_table(rows, overall, bop=opt.bop, vsd=opt.vsd)
    if opt.json:
        with open(opt.json, "w") as fh:
            json.dump({"objects": {str(k): v for k, v in rows.items()}, "overall": overall}, fh, indent=1)
    return rows, overall


if __name__ == "__main__":
    main()
