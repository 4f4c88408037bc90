"""Frames as sensors deliver them: `Color` and `Depth` describe a camera's buffers in their own layout, and the library
unpacks them on the GPU in the frame filter (fp_set_camera_format, include/fpose.h), so no caller converts on the host.

    Color(img, order)   uint8 (H,W,3) for order "rgb" / "bgr", (H,W,4) for "rgba" / "bgra" (alpha ignored)
    Depth(img)          float32 (H,W) metres
    Depth(img, scale)   uint16 (H,W) units of `scale` metres (RealSense z16: 0.001, a D405: 0.0001)

Each takes a numpy array, a CPU tensor or a CUDA tensor on the engine's device.  Pixels must be packed; rows may be any
positive number of bytes apart (a region-of-interest view of a larger frame, a pitched GPU mat), and are read where they
are.  A uint16 depth becomes `np.float32(v) * np.float32(scale)` in metres, one fp32 multiply rounded to nearest, bit for
bit what the same call gives on that host-converted frame; 0 stays invalid.

A plain uint16 array passed where depth is expected (no `Depth`) is cast to float32 as it always was: its values are
then taken as metres.  Wrap it in `Depth(img, scale)` instead.

    Depth(img, scale, sensor=DepthSensor(K, T_color_from_depth))

is depth from a depth imager of its own (fp_set_camera_depth_sensor, include/fpose.h): `img` is the depth sensor's
(Hd, Wd) image, K its intrinsics and T_color_from_depth the rigid transform from the depth camera to the colour camera
(4x4, metres).  The library aligns it to the colour frame on the GPU by librealsense's rs2::align rule, so the call's
frame size, K and masks are the colour camera's."""
import math

import numpy as np
import torch

COLOR_RGB8, COLOR_BGR8, COLOR_RGBA8, COLOR_BGRA8 = 0, 1, 2, 3  # FP_COLOR_* (include/fpose.h)
DEPTH_F32, DEPTH_U16 = 0, 1  # FP_DEPTH_*
DEPTH_SENSOR_MAX_DIM = 4096  # FP_DEPTH_SENSOR_MAX_DIM
DEFAULT_FORMAT = (COLOR_RGB8, DEPTH_F32, 0.0, 0, 0)  # (color, depth, depth_scale, rgb_pitch, depth_pitch): packed RGB8 + float32

_ORDERS = {"rgb": (COLOR_RGB8, 3), "bgr": (COLOR_BGR8, 3), "rgba": (COLOR_RGBA8, 4), "bgra": (COLOR_BGRA8, 4)}


def _layout(img, what, channels, np_dtype, torch_dtype):
    """(H, W) and the row pitch in bytes of an image whose pixels are packed: (H,W) for channels = 0, else
    (H,W,channels).  The pitch is 0 when the rows are packed too."""
    if torch.is_tensor(img):
        if img.dtype != torch_dtype:
            raise TypeError(f"{what}: needs {torch_dtype}, got {img.dtype}")
        item = img.element_size()
        shape, strides = tuple(img.shape), [s * item for s in img.stride()]
    elif isinstance(img, np.ndarray):
        if img.dtype != np_dtype:
            raise TypeError(f"{what}: needs {np.dtype(np_dtype).name}, got {img.dtype}")
        item = img.itemsize
        shape, strides = img.shape, list(img.strides)
    else:
        raise TypeError(f"{what}: needs a numpy array or a torch tensor, got {type(img).__name__}")
    want = (-1, -1, channels) if channels else (-1, -1)
    if len(shape) != len(want) or any(w > 0 and s != w for s, w in zip(shape, want)) or 0 in shape:
        dims = f"(H, W, {channels})" if channels else "(H, W)"
        raise ValueError(f"{what}: needs a non-empty {dims} image, got {tuple(shape)}")
    H, W = int(shape[0]), int(shape[1])
    px = item * (channels or 1)
    # a dimension of size 1 has no meaningful stride
    if (channels and strides[2] != item) or (W > 1 and strides[1] != px):
        raise ValueError(f"{what}: pixels must be packed ({px} bytes each, channels adjacent), got strides {tuple(strides)} bytes")
    row = W * px
    pitch = strides[0] if H > 1 else row
    if pitch < row:
        raise ValueError(f"{what}: rows must be at least {row} bytes apart and in order, got a row stride of {pitch} bytes")
    return (H, W), (0 if pitch == row else int(pitch))


class Color:
    """A camera's colour frame as the sensor delivers it (see the module docstring): `img` uint8 (H,W,3) for order "rgb"
    or "bgr", (H,W,4) for "rgba" or "bgra"."""

    def __init__(self, img, order="rgb"):
        if order not in _ORDERS:
            raise ValueError(f"Color: order must be one of {sorted(_ORDERS)}, got {order!r}")
        self.code, channels = _ORDERS[order]
        self.order, self.img = order, img
        (self.H, self.W), self.pitch = _layout(img, f"Color(order={order!r})", channels, np.uint8, torch.uint8)

    @property
    def shape(self):
        return tuple(self.img.shape)


class DepthSensor:
    """A depth imager of its own (see the module docstring): K (3,3) its intrinsics (fx, fy > 0) and T_color_from_depth
    (4,4) the rigid transform from the depth camera to the colour camera, in metres, both finite in float32.  From
    pyrealsense2: T[:3, :3] = np.reshape(extr.rotation, (3, 3)).T, T[:3, 3] = extr.translation, with extr the depth
    stream profile's get_extrinsics_to(colour profile)."""

    def __init__(self, K, T_color_from_depth):
        with np.errstate(over="ignore", invalid="ignore"):
            K = np.asarray(K, dtype=np.float64).astype(np.float32)
            T = np.asarray(T_color_from_depth, dtype=np.float64).astype(np.float32)
        if K.shape != (3, 3) or T.shape != (4, 4):
            raise ValueError(f"DepthSensor: K must be (3, 3) and T_color_from_depth (4, 4), got {K.shape} and {T.shape}")
        if not (np.isfinite(K).all() and np.isfinite(T).all()):
            raise ValueError("DepthSensor: K and T_color_from_depth must be finite in float32")
        if not (K[0, 0] > 0 and K[1, 1] > 0):
            raise ValueError(f"DepthSensor: focal lengths must be > 0, got fx = {K[0, 0]}, fy = {K[1, 1]}")
        self.K, self.T = K, T


class Depth:
    """A camera's depth frame as the sensor delivers it (see the module docstring): `img` float32 (H,W) metres with
    scale=None, or uint16 (H,W) with `scale` metres per unit (finite and > 0 in float32).  sensor: a DepthSensor when
    the image is a depth imager's own (H,W), aligned to the colour frame by the library."""

    def __init__(self, img, scale=None, sensor=None):
        if sensor is not None and not isinstance(sensor, DepthSensor):
            raise TypeError(f"Depth: sensor must be a DepthSensor or None, got {type(sensor).__name__}")
        self.sensor = sensor
        if scale is None:
            self.code, self.scale = DEPTH_F32, 0.0
            what, np_dtype, torch_dtype = "Depth(scale=None)", np.float32, torch.float32
        else:
            with np.errstate(over="ignore"):
                s = float(np.float32(scale))
            if not (math.isfinite(s) and s > 0.0):
                raise ValueError(f"Depth: scale must be finite and > 0 metres per unit in float32, got {scale!r}")
            self.code, self.scale = DEPTH_U16, s
            what, np_dtype, torch_dtype = f"Depth(scale={scale!r})", np.uint16, torch.uint16
        self.img = img
        (self.H, self.W), self.pitch = _layout(img, what, 0, np_dtype, torch_dtype)
        if sensor is not None and max(self.H, self.W) > DEPTH_SENSOR_MAX_DIM:
            raise ValueError(f"Depth: a depth sensor's image is at most {DEPTH_SENSOR_MAX_DIM} pixels a side, got {self.H} x {self.W}")

    @property
    def shape(self):
        return tuple(self.img.shape)


def image(x):
    """The array or tensor behind a frame argument: a wrapper's image, or the argument itself."""
    return x.img if isinstance(x, (Color, Depth)) else x


def frame_hw(rgb, depth):
    """The (H, W) of a camera's frame arguments: the depth's, or the colour's when the depth comes from a sensor of its
    own (Depth(sensor=))."""
    x = rgb if isinstance(depth, Depth) and depth.sensor is not None else depth
    return tuple(int(n) for n in (x.shape if isinstance(x, (Color, Depth)) or torch.is_tensor(x) else np.shape(x))[:2])


def on_cuda(x):
    """Whether a frame argument, plain or wrapped, is a CUDA tensor."""
    x = image(x)
    return torch.is_tensor(x) and x.is_cuda


def host_rgb(rgb):
    """A colour frame argument as a packed uint8 (H,W,3) RGB numpy array on the host (debug dumps)."""
    if not isinstance(rgb, Color):
        return rgb.cpu().numpy() if torch.is_tensor(rgb) else np.asarray(rgb)
    img = rgb.img.cpu().numpy() if torch.is_tensor(rgb.img) else np.asarray(rgb.img)
    img = img[..., :3]
    return np.ascontiguousarray(img[..., ::-1] if rgb.order in ("bgr", "bgra") else img)


def frame_format(rgb, depth):
    """The (color, depth, depth_scale, rgb_pitch, depth_pitch) format of a camera's frame arguments, for
    fp_set_camera_format: plain arrays are packed RGB8 and float32, as the library always took them."""
    c = (rgb.code, rgb.pitch) if isinstance(rgb, Color) else (COLOR_RGB8, 0)
    d = (depth.code, depth.scale, depth.pitch) if isinstance(depth, Depth) else (DEPTH_F32, 0.0, 0)
    return (c[0], d[0], d[1], c[1], d[2])


def depth_sensor(depth):
    """The (H, W, K, T) depth sensor of a depth frame argument for fp_set_camera_depth_sensor (K 9 and T 16 floats,
    row-major), or None: plain arrays and a Depth without a sensor are in the colour frame's geometry."""
    if not isinstance(depth, Depth) or depth.sensor is None:
        return None
    return (depth.H, depth.W, tuple(float(x) for x in depth.sensor.K.reshape(-1)),
            tuple(float(x) for x in depth.sensor.T.reshape(-1)))
