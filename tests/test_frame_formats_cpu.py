"""Frames as sensors deliver them, without a GPU: the Color / Depth wrappers' validation and refusal messages, the format
each pair of frame arguments asks the library for, the uint16 depth rule against numpy (and its float64 identity), and
fp_set_camera_format's place in the C ABI."""
import os
import re

import numpy as np
import pytest
import torch

from foundationpose_b200 import frames
from foundationpose_b200.frames import Color, Depth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, "include", "fpose.h")) as fh:
        return fh.read()


def test_format_constants_match_the_header():
    h = _header()
    for name, value in (("FP_COLOR_RGB8", frames.COLOR_RGB8), ("FP_COLOR_BGR8", frames.COLOR_BGR8),
                        ("FP_COLOR_RGBA8", frames.COLOR_RGBA8), ("FP_COLOR_BGRA8", frames.COLOR_BGRA8),
                        ("FP_DEPTH_F32", frames.DEPTH_F32), ("FP_DEPTH_U16", frames.DEPTH_U16)):
        assert re.search(rf"#define {name} {value}\b", h), name
    fields = re.search(r"typedef struct fp_frame_format \{(.*?)\} fp_frame_format_t;", h, re.S).group(1)
    assert re.findall(r"(\w+);", fields) == ["color", "depth", "depth_scale", "rgb_pitch", "depth_pitch"]


def test_set_camera_format_is_a_guarded_entry_point():
    with open(os.path.join(ROOT, "foundationpose_b200", "csrc", "fp_api.cu")) as fh:
        src = fh.read()
    m = re.search(r"^int fp_set_camera_format\([^)]*\)\s*\{\s*(\S+)", src, re.M)
    assert m and m.group(1) == "FP_API_BEGIN"
    body = src[m.end():src.index("FP_API_END", m.end())]
    # host state only: nothing is enqueued, nothing waits
    assert not re.search(r"cuda\w*\(|order_after_track|take_set", body)


@pytest.mark.parametrize("order,ch,code", [("rgb", 3, 0), ("bgr", 3, 1), ("rgba", 4, 2), ("bgra", 4, 3)])
def test_color_orders_and_packed_pitch(order, ch, code):
    img = np.zeros((5, 7, ch), np.uint8)
    c = Color(img, order)
    assert (c.code, c.H, c.W, c.pitch, c.shape) == (code, 5, 7, 0, (5, 7, ch))
    t = Color(torch.from_numpy(img), order)
    assert (t.code, t.H, t.W, t.pitch) == (code, 5, 7, 0)


def test_region_of_interest_views_pass_their_row_pitch():
    big = np.zeros((20, 30, 4), np.uint8)
    assert Color(big[2:12, 3:13], "bgra").pitch == 30 * 4
    assert Color(torch.from_numpy(big)[2:12, 3:13], "rgba").pitch == 30 * 4
    d = np.zeros((20, 30), np.uint16)
    assert Depth(d[1:5, 2:9], 0.001).pitch == 60
    f = np.zeros((20, 30), np.float32)
    assert Depth(torch.from_numpy(f)[1:5, :7]).pitch == 120
    # one row: any stride is packed
    assert Depth(f[3:4, :5]).pitch == 0


def test_wrapper_refusals():
    with pytest.raises(ValueError, match="order must be one of"):
        Color(np.zeros((2, 2, 3), np.uint8), "yuv")
    with pytest.raises(ValueError, match=r"non-empty \(H, W, 4\)"):
        Color(np.zeros((2, 2, 3), np.uint8), "rgba")
    with pytest.raises(ValueError, match=r"non-empty \(H, W, 3\)"):
        Color(np.zeros((2, 2, 4), np.uint8), "bgr")
    with pytest.raises(TypeError, match="needs uint8"):
        Color(np.zeros((2, 2, 3), np.float32), "rgb")
    with pytest.raises(TypeError, match="needs uint16"):
        Depth(np.zeros((2, 2), np.float32), 0.001)
    with pytest.raises(TypeError, match="needs float32"):
        Depth(np.zeros((2, 2), np.uint16))
    with pytest.raises(TypeError, match="needs torch.uint16"):
        Depth(torch.zeros(2, 2, dtype=torch.int16), 0.001)
    with pytest.raises(TypeError, match="numpy array or a torch tensor"):
        Depth([[0.0, 1.0]])
    for bad in (0.0, -0.001, float("nan"), float("inf"), 1e-50, 1e40):
        with pytest.raises(ValueError, match="scale must be finite and > 0"):
            Depth(np.zeros((2, 2), np.uint16), bad)
    with pytest.raises(ValueError, match=r"non-empty \(H, W\)"):
        Depth(np.zeros((0, 3), np.float32))
    with pytest.raises(ValueError, match="pixels must be packed"):
        Color(np.zeros((4, 6, 3), np.uint8)[:, ::2], "rgb")
    with pytest.raises(ValueError, match="pixels must be packed"):
        Color(np.zeros((4, 6, 3), np.uint8).transpose(1, 0, 2), "rgb")
    with pytest.raises(ValueError, match="pixels must be packed"):
        Color(np.zeros((4, 6, 5), np.uint8)[..., :3], "rgb")
    with pytest.raises(ValueError, match="rows must be at least"):
        Depth(np.zeros((4, 6), np.float32)[::-1])


def test_frame_format_of_plain_and_wrapped_arguments():
    rgb, depth = np.zeros((4, 6, 3), np.uint8), np.zeros((4, 6), np.float32)
    assert frames.frame_format(rgb, depth) == frames.DEFAULT_FORMAT
    # a packed wrapper of the default layout is the default format
    assert frames.frame_format(Color(rgb, "rgb"), Depth(depth)) == frames.DEFAULT_FORMAT
    big = np.zeros((8, 10, 4), np.uint8)
    d16 = np.zeros((8, 10), np.uint16)
    f = frames.frame_format(Color(big[:4, :6], "bgra"), Depth(d16[:4, :6], 0.00025))
    assert f == (frames.COLOR_BGRA8, frames.DEPTH_U16, float(np.float32(0.00025)), 40, 20)


def test_host_rgb_is_rgb():
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (5, 4, 3), dtype=np.uint8)
    bgra = np.concatenate([img[..., ::-1], np.full((5, 4, 1), 7, np.uint8)], -1)
    np.testing.assert_array_equal(frames.host_rgb(Color(bgra, "bgra")), img)
    np.testing.assert_array_equal(frames.host_rgb(Color(np.ascontiguousarray(img[..., ::-1]), "bgr")), img)
    np.testing.assert_array_equal(frames.host_rgb(Color(torch.from_numpy(img), "rgb")), img)
    np.testing.assert_array_equal(frames.host_rgb(img), img)


@pytest.mark.parametrize("scale", [0.001, 0.0001, 0.00025, 1.0 / 3.0, 0.0010000001])
def test_depth_rule_matches_numpy_and_float64(scale):
    """The kernels' rule, __fmul_rn((float)v, s): one fp32 multiply rounded to nearest.  numpy's float32 product is that
    multiply; the float64 product of two floats is exact (24 + 16 significant bits), so rounding it once to float32
    gives the same value."""
    v = np.arange(65536, dtype=np.uint16)
    s32 = np.float32(scale)
    rule = v.astype(np.float32) * s32
    assert rule.dtype == np.float32
    via64 = (v.astype(np.float64) * np.float64(s32)).astype(np.float32)
    np.testing.assert_array_equal(rule.view(np.uint32), via64.view(np.uint32))
    assert rule[0] == 0.0  # invalid stays invalid
    # what the Depth wrapper hands the library
    assert np.float32(Depth(np.zeros((1, 1), np.uint16), scale).scale) == s32
