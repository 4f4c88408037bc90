"""CPU: the host side of non-blocking tracking.  estimater.track_cameras / track_objects with wait=False through an engine
double (pose_last set at submit, the pending result shaped as the blocking call's, every refusal raised before the engine
is called), PendingPoses' dropped-handle bookkeeping, and the C ABI declaring and exporting the submit / wait pair."""
import ctypes
import gc
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Refiner:
    last_trans_update = last_rot_update = "stale"


class _Pending:
    def __init__(self, host):
        self.host, self.waits = host, 0

    def result(self):
        self.waits += 1
        return self.host


class _Engine:
    """Stands in for engine.Engine: records calls, returns poses shifted by +1 cm in x, blocking or pending."""

    def __init__(self):
        self.calls = []
        self.pending = []

    def set_mesh(self, pos, normals, faces, diameter, uv=None, tex=None, vertex_colors=None, slot=0):
        pass

    def _shifted(self, poses_in, wait):
        out = poses_in.clone()
        out[:, 0, 3] += 0.01
        if wait:
            return out, out.numpy().copy()
        self.pending.append(_Pending(out.numpy().copy()))
        return out, self.pending[-1]

    def track_objects(self, rgb, depth, K, poses_in, slots, iterations, wait=True):
        self.calls.append(("track_objects", list(slots), iterations, wait))
        return self._shifted(poses_in, wait)

    def track_cameras(self, frames, poses_in, camera_of, slots, iterations, wait=True):
        self.calls.append(("track_cameras", [f[0] for f in frames], list(camera_of), list(slots), iterations, wait))
        return self._shifted(poses_in, wait)


def _est(engine, n_verts, center=(0.0, 0.0, 0.0), x=0.0):
    from foundationpose_b200.estimater import FoundationPose

    est = FoundationPose.__new__(FoundationPose)
    est.engine = engine
    est.refiner = _Refiner()
    est.mesh_tensors = dict(pos=np.zeros((n_verts, 3), np.float32), normals=np.zeros((n_verts, 3), np.float32),
                            faces=np.zeros((1, 3), np.int32), vcolor=np.zeros((n_verts, 3), np.float32))
    est.diameter = 0.1 * n_verts
    est.model_center = np.asarray(center, dtype=np.float64)
    est.pose_last = torch.eye(4).reshape(1, 4, 4)
    est.pose_last[0, 0, 3] = x
    return est


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if isinstance(x, list):
            _same(x, y)
        else:
            assert x.shape == y.shape == (4, 4) and np.array_equal(x, y)


def test_track_cameras_pending_state_and_result():
    from foundationpose_b200.estimater import PendingTrack, track_cameras

    views = lambda ests: [(ests[:2], "rgb0", None, None), ([], "rgb1", None, None), (ests[2:], "rgb2", None, None)]
    e = _Engine()
    ests = [_est(e, 3, center=(0.0, 0.0, 0.1), x=1.0), _est(e, 4, x=2.0), _est(e, 5, center=(0.02, 0.0, 0.0), x=3.0)]
    want = track_cameras(views(ests), iteration=3)
    for est in ests:
        est.pose_last[0, 0, 3] -= 0.01
    got = track_cameras(views(ests), iteration=3, wait=False)
    assert isinstance(got, PendingTrack)
    assert e.calls[-1] == ("track_cameras", ["rgb0", "rgb2"], [0, 0, 1], [1, 2, 3], 3, False)
    # pose_last is the pending device pose at once, before anything is collected
    assert e.pending[-1].waits == 0
    assert [float(est.pose_last[0, 0, 3]) for est in ests] == pytest.approx([1.01, 2.01, 3.01])
    assert all(est.refiner.last_trans_update is None for est in ests)
    out = got.result()
    _same(out, want)
    assert [len(v) for v in out] == [2, 0, 1]
    assert got.result() is out and e.pending[-1].waits == 1
    assert track_cameras([([], "rgb0", None, None)], wait=False).result() == [[]]


def test_track_objects_pending_state_and_result():
    from foundationpose_b200.estimater import PendingTrack, track_objects

    e = _Engine()
    ests = [_est(e, 3, center=(0.0, 0.05, 0.0), x=1.0), _est(e, 4, x=2.0)]
    want = track_objects(ests, "rgb", None, None, iteration=2)
    for est in ests:
        est.pose_last[0, 0, 3] -= 0.01
    got = track_objects(ests, "rgb", None, None, iteration=2, wait=False)
    assert isinstance(got, PendingTrack) and e.calls[-1] == ("track_objects", [1, 2], 2, False)
    assert [float(est.pose_last[0, 0, 3]) for est in ests] == pytest.approx([1.01, 2.01])
    _same(got.result(), want)
    assert track_objects([], "rgb", None, None, wait=False).result() == []


def test_refusals_reach_no_engine():
    from foundationpose_b200.estimater import track_cameras, track_objects

    e, other = _Engine(), _Engine()
    a, b, stranger = _est(e, 3), _est(e, 4), _est(other, 5)
    dev = torch.zeros(4, 4, 3, dtype=torch.uint8)
    bad = [(TypeError, lambda: track_objects([a], dev, dev, None, wait=False)),
           (TypeError, lambda: track_cameras([([a], dev, dev, None)], wait=False)),
           (ValueError, lambda: track_objects([a, a], "rgb", None, None, wait=False)),
           (ValueError, lambda: track_cameras([([a], "rgb0", None, None), ([stranger], "rgb1", None, None)], wait=False)),
           (ValueError, lambda: track_cameras([([a], "rgb0", None, None), ([a, b], "rgb1", None, None)], wait=False))]
    for exc, fn in bad:
        with pytest.raises(exc):
            fn()
    b.pose_last = None
    with pytest.raises(RuntimeError):
        track_objects([a, b], "rgb", None, None, wait=False)
    with pytest.raises(RuntimeError):
        track_cameras([([a], "rgb0", None, None), ([b], "rgb1", None, None)], wait=False)
    assert e.calls == [] and other.calls == []
    assert float(a.pose_last[0, 0, 3]) == 0.0, "a refused call touched pose_last"


def test_dropped_handles_are_handed_back_to_their_engine():
    from foundationpose_b200.engine import PendingPoses

    class Owner:
        def __init__(self):
            self._dropped, self.waited = [], []

        def _wait(self, ticket, host):
            self.waited.append(ticket)
            host[...] = ticket

    o = Owner()
    kept, dropped = PendingPoses(o, 7, (2, 4, 4)), PendingPoses(o, 8, (4, 4))
    del dropped
    gc.collect()
    assert o._dropped == [8]
    r = kept.result()
    assert r.shape == (2, 4, 4) and (r == 7).all() and kept.result() is r and o.waited == [7]
    del kept
    gc.collect()
    assert o._dropped == [8], "a collected handle is not handed back"


def _declared():
    src = open(os.path.join(ROOT, "include", "fpose.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b(fp_[a-z0-9_]+)\s*\(", src)), src


def test_header_declares_and_library_exports_submit_and_wait():
    from foundationpose_b200 import _lib
    from foundationpose_b200.engine import MAX_IN_FLIGHT

    names, src = _declared()
    new = {"fp_track_cameras_submit", "fp_track_objects_submit", "fp_track_submit", "fp_track_wait"}
    assert new <= names
    assert re.search(r"#define FP_TRACK_MAX_IN_FLIGHT (\d+)", src).group(1) == str(MAX_IN_FLIGHT) == "2"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    assert all(hasattr(lib, n) for n in new)
    assert _lib.lib.fp_track_wait(None, 1, None) != 0, "a null context is refused"
