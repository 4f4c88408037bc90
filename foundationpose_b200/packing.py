"""Host-side weight preparation: fold eval-mode BatchNorm into the convolutions and repack the
reference `state_dict` tensors into the K-major fp16 layouts the wgmma kernels consume.

Reference layouts: learning/models/network_modules.py:37-50 (ConvBNReLU: net.0 = Conv2d, net.1 = BN),
:73-111 (ResnetBasicBlock: conv1/bn1/conv2/bn2).  BatchNorm2d in eval mode is the per-channel affine
y = (x - mean) / sqrt(var + eps) * gamma + beta, folded here in fp32 before the fp16 cast.
"""
import torch


def fold_bn(w, b, bn):
    """w (Co,Ci,kh,kw), b (Co) or None, bn = dict(weight,bias,running_mean,running_var,eps) or None."""
    w = w.detach().float()
    b = torch.zeros(w.shape[0]) if b is None else b.detach().float()
    if bn is None:
        return w, b
    scale = bn["weight"].float() / torch.sqrt(bn["running_var"].float() + bn["eps"])
    w = w * scale.reshape(-1, 1, 1, 1)
    b = (b - bn["running_mean"].float()) * scale + bn["bias"].float()
    return w, b


def pack_conv3(w):
    """(Co,Ci,3,3) fp32 -> (Co, 9*Ci) fp16, K ordered (r, s, c)."""
    co, ci = w.shape[:2]
    return w.permute(0, 2, 3, 1).reshape(co, 9 * ci).contiguous().half()


def pack_conv7(w):
    """(Co,Ci<=8,7,7) fp32 -> (7, 4, 2, Co, 8) fp16 = [filter row r][tap pair s][tap 2s + e][Co][8 ch]: one
    un-swizzled K-major wgmma B tile (N = Co, K = 16) per (r, s); tap 7 and channels >= Ci are zero
    (csrc/fp_stem.cu)."""
    co, ci = w.shape[:2]
    out = torch.zeros(7, 8, co, 8, dtype=torch.float32)  # (r, tap padded to 8, co, c padded to 8)
    out[:, :7, :, :ci] = w.detach().float().permute(2, 3, 0, 1)
    return out.reshape(7, 4, 2, co, 8).contiguous().half()


def pack_linear(w):
    """(Co, K) -> fp16 contiguous."""
    return w.detach().float().contiguous().half()


def pad_image_c8(x):
    """(N,C<=8,H,W) float -> stem input layout [N][H+6][2][(W+8)/2][8] fp16: the image sits at (3,3) of a
    zero-bordered (H+6, W+8) canvas whose rows are stored as even columns then odd columns ("EO" layout,
    csrc/fp_stem.cu)."""
    n, c, h, w = x.shape
    canvas = torch.zeros(n, h + 6, w + 8, 8, dtype=torch.float16, device=x.device)
    canvas[:, 3 : 3 + h, 3 : 3 + w, :c] = x.permute(0, 2, 3, 1).half()
    return canvas.reshape(n, h + 6, (w + 8) // 2, 2, 8).permute(0, 1, 3, 2, 4).contiguous()


def unpad_image_c8(buf):
    """Inverse view of pad_image_c8: [N][H+6][2][(W+8)/2][8] -> the padded NHWC canvas (N, H+6, W+8, 8)."""
    n, hp, two, wh, c = buf.shape
    return buf.permute(0, 1, 3, 2, 4).reshape(n, hp, 2 * wh, c)
