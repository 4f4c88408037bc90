"""Depth from its own sensor, without a GPU: the float32 reference of the alignment rule (tests/align_reference.py)
against a float64 restatement and on hand-made cases whose answer is known, DepthSensor / Depth(sensor=) validation, and
the new entry points in the C ABI."""
import os
import re

import numpy as np
import pytest
import torch

import align_reference as ar

ROOT = os.path.join(os.path.dirname(__file__), "..")


def _scene(Hd, Wd, seed):
    """A depth image with discontinuities: a slanted background, two boxes in front of it, holes."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:Hd, 0:Wd]
    d = 1.5 + 0.3 * xx / Wd + 0.2 * yy / Hd
    d[Hd // 4:Hd // 2, Wd // 5:Wd // 2] = 0.6
    d[Hd // 2:3 * Hd // 4, Wd // 2:3 * Wd // 4] = 0.35
    d += rng.normal(0, 0.002, d.shape)
    raw = np.round(d * 1000).astype(np.uint16)
    raw[rng.random(d.shape) < 0.03] = 0
    return raw


@pytest.mark.parametrize("rig", ["d435", "vga"])
def test_float32_rule_agrees_with_float64_away_from_rounding_boundaries(rig):
    Kd, Kc, (Hd, Wd), (H, W) = ((ar.D435_DEPTH_K, ar.D435_COLOR_K, (480, 848), (720, 1280)) if rig == "d435" else
                                (ar.VGA_DEPTH_K, ar.VGA_COLOR_K, (480, 640), (480, 640)))
    T = ar.rig_T()
    d, valid = ar.depth_metres(_scene(Hd, Wd, 3), 0.001)
    r32 = ar.rectangles(d, valid, Kd, T, Kc, H, W, np.float32)
    r64 = ar.rectangles(d.astype(np.float64), valid, Kd, T, Kc, H, W, np.float64)
    near = ar.near_boundary(d, valid, Kd, T, Kc)
    # the kept pixels, and each kept pixel's rectangle, agree except where a corner lies within 1e-4 px of a boundary
    differ = r32[5] != r64[5]
    both = r32[5] & r64[5]
    i32, i64 = np.cumsum(r32[5]) - 1, np.cumsum(r64[5]) - 1
    for a, b in zip(r32[:4], r64[:4]):
        differ[both] |= a[i32[both]] != b[i64[both]]
    assert not (differ & ~near).any()
    n = int(differ.sum())
    print(f"{rig}: {n} of {int(valid.sum())} depth pixels round differently in float32 and float64, "
          f"all within 1e-4 px of a rounding boundary ({int(near.sum())} pixels lie that close)")
    assert r32[5].sum() > 0.3 * valid.sum()  # the D435 depth imager sees wider than its colour camera


def _exact_rig(H=6, W=7):
    """Focal lengths, centres and depths that make every step of the rule exact in float32."""
    K = np.array([[512.0, 0, 3.5], [0, 256.0, 2.5], [0, 0, 1]])
    return K, H, W


def test_identity_rig_fills_2x2_blocks_and_drops_last_row_and_column():
    K, H, W = _exact_rig()
    rng = np.random.default_rng(0)
    d = rng.choice(np.array([0.5, 1.0, 2.0, 4.0], np.float32), (H, W))
    out = ar.align(d, d != 0, K, np.eye(4), K, H, W)
    want = np.full((H, W), np.inf, np.float32)
    for y in range(H - 1):
        for x in range(W - 1):
            want[y:y + 2, x:x + 2] = np.minimum(want[y:y + 2, x:x + 2], d[y, x])
    want[np.isinf(want)] = 0
    np.testing.assert_array_equal(out, want)
    assert (out[0, :] > 0).all() and (out[:, 0] > 0).all()  # row and column 0 covered by one rectangle each


def test_integer_pixel_translation():
    K, H, W = _exact_rig(8, 10)
    T = np.eye(4)
    T[0, 3] = 3.0 / 512.0  # 3 px at z = 1
    T[1, 3] = -1.0 / 256.0  # -1 px
    d = np.ones((H, W), np.float32)
    out = ar.align(d, d != 0, K, T, K, H, W)
    want = np.zeros((H, W), np.float32)
    for y in range(H):
        for x in range(W):
            x0, y0 = x + 3, y - 1
            if x0 >= 0 and y0 >= 0 and x0 + 1 <= W - 1 and y0 + 1 <= H - 1:
                want[y0:y0 + 2, x0:x0 + 2] = 1.0
    np.testing.assert_array_equal(out, want)


def test_behind_the_colour_camera_and_nan_are_dropped():
    K, H, W = _exact_rig()
    T = np.eye(4)
    T[2, 3] = -2.0
    d = np.full((H, W), 1.0, np.float32)  # Z' = -1
    d[2, 3] = 2.0  # Z' = 0: dropped too
    d[3, 3] = 4.0  # Z' = 2: kept
    out = ar.align(d, d != 0, K, T, K, H, W)
    assert (out[out > 0] == 4.0).all() and (out > 0).sum() > 0
    d = np.full((H, W), np.nan, np.float32)
    assert (ar.align(d, d != 0, K, np.eye(4), K, H, W) == 0).all()


def test_raw_zero_is_skipped_and_65535_kept():
    K, H, W = _exact_rig()
    raw = np.zeros((H, W), np.uint16)
    raw[1, 1] = 65535
    d, valid = ar.depth_metres(raw, 1.0 / 65536.0)
    out = ar.align(d, valid, K, np.eye(4), K, H, W)
    want = np.zeros((H, W), np.float32)
    want[1:3, 1:3] = np.float32(65535) * np.float32(1.0 / 65536.0)
    np.testing.assert_array_equal(out, want)


def test_overlapping_rectangles_take_the_minimum():
    K, H, W = _exact_rig(8, 10)
    d = np.zeros((H, W), np.float32)
    d[3, 4] = 2.0
    d[3, 5] = 1.0  # shares column 5 with (3, 4)'s rectangle
    d[4, 4] = 4.0  # shares row 4
    out = ar.align(d, d != 0, K, np.eye(4), K, H, W)
    assert out[3, 4] == 2.0 and out[3, 5] == 1.0 and out[4, 5] == 1.0 and out[4, 4] == 2.0 and out[5, 4] == 4.0
    # a near pixel whose corners spread far covers many colour pixels and wins where it is nearest
    T = np.eye(4)
    d2 = np.full((H, W), 2.0, np.float32)
    out = ar.align(d2, d2 != 0, K, T, np.array([[512.0 * 4, 0, 3.5], [0, 256.0 * 4, 2.5], [0, 0, 1]]), H, W)
    assert (out[out > 0] == 2.0).all()


def test_colour_frame_smaller_than_the_depth_image():
    K, H, W = _exact_rig(12, 14)
    d = np.ones((H, W), np.float32)
    out = ar.align(d, d != 0, K, np.eye(4), K, 5, 6)
    assert out.shape == (5, 6) and (out == 1.0).all()
    x0, x1, y0, y1, _, keep = ar.rectangles(d, d != 0, K, np.eye(4), K, 5, 6)
    assert (x1 <= 5).all() and (y1 <= 4).all() and keep.sum() == 4 * 5


def test_depth_sensor_and_wrapper_validation():
    from foundationpose_b200.frames import Depth, DepthSensor, depth_sensor, frame_hw

    K = ar.D435_DEPTH_K
    s = DepthSensor(K, ar.rig_T())
    assert s.K.dtype == np.float32 and s.T.shape == (4, 4)
    bad_K = K.copy()
    bad_K[0, 0] = 0
    with pytest.raises(ValueError, match="focal lengths must be > 0"):
        DepthSensor(bad_K, np.eye(4))
    bad_T = np.eye(4)
    bad_T[0, 3] = np.nan
    with pytest.raises(ValueError, match="must be finite"):
        DepthSensor(K, bad_T)
    with pytest.raises(ValueError, match="must be finite"):
        DepthSensor(K * 1e39, np.eye(4))  # overflows float32
    with pytest.raises(ValueError, match=r"\(3, 3\).*\(4, 4\)"):
        DepthSensor(np.eye(4), np.eye(4))
    with pytest.raises(TypeError, match="sensor must be a DepthSensor"):
        Depth(np.zeros((4, 5), np.float32), sensor=K)
    with pytest.raises(ValueError, match="at most 4096 pixels"):
        Depth(np.zeros((2, 4097), np.float32), sensor=s)
    d = Depth(np.zeros((480, 848), np.uint16), 0.001, sensor=s)
    H, W, Kr, Tr = depth_sensor(d)
    assert (H, W) == (480, 848) and len(Kr) == 9 and len(Tr) == 16
    assert depth_sensor(Depth(np.zeros((4, 5), np.float32))) is None and depth_sensor(np.zeros((4, 5))) is None
    rgb = np.zeros((720, 1280, 3), np.uint8)
    assert frame_hw(rgb, d) == (720, 1280)
    assert frame_hw(rgb, np.zeros((720, 1280), np.float32)) == (720, 1280)
    assert frame_hw(torch.zeros(7, 9, 3, dtype=torch.uint8), Depth(torch.zeros(3, 4), sensor=s)) == (7, 9)


def test_frame_takes_colour_size_with_a_sensor():
    from foundationpose_b200.engine import _frame
    from foundationpose_b200.frames import Color, Depth, DepthSensor

    s = DepthSensor(ar.D435_DEPTH_K, np.eye(4))
    rgb = np.zeros((720, 1280, 3), np.uint8)
    raw = np.zeros((480, 848), np.uint16)
    r, d, hw, fmt, sensor = _frame(rgb, Depth(raw, 0.001, sensor=s), "t")
    assert hw == (720, 1280) and d is raw and sensor[:2] == (480, 848) and fmt[1] == 1
    r, d, hw, fmt, sensor = _frame(Color(rgb[..., ::-1].copy(), "bgr"), Depth(raw, 0.001, sensor=s), "t")
    assert hw == (720, 1280)
    _, _, hw, _, sensor = _frame(rgb, np.zeros((720, 1280), np.float32), "t")
    assert hw == (720, 1280) and sensor is None


def test_c_abi_declares_and_guards_the_new_entry_points():
    with open(os.path.join(ROOT, "include", "fpose.h")) as fh:
        h = fh.read()
    assert "#define FP_DEPTH_SENSOR_MAX_DIM 4096" in h
    assert re.search(r"typedef struct fp_depth_sensor \{\s*int H, W;\s*float K\[9\];\s*float T_color_from_depth\[16\];\s*\}", h)
    for name in ("fp_set_camera_depth_sensor", "fp_align_depth"):
        assert re.search(rf"\bint {name}\(", h), name
    src = ""
    for f in ("fp_api.cu", "fp_api_ops.cu"):
        with open(os.path.join(ROOT, "foundationpose_b200", "csrc", f)) as fh:
            src += fh.read()
    for name in ("fp_set_camera_depth_sensor", "fp_align_depth"):
        m = re.search(rf"\nint {name}\([^{{]*\{{\s*(\w+)", src)
        assert m and m.group(1) == "FP_API_BEGIN", name
