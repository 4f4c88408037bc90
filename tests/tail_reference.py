"""Float64 references and derived error bars for the scorer tail's segmented launch (cross_attn_score_kernel) and for the
refine loop's pose update (pose_update_kernel), shared by tests/test_selection_gpu.py and its CPU self-check
(tests/test_selection_cpu.py).  Device-agnostic torch: the GPU test evaluates them in float64 on the device.

Notation: u = 2^-24 is the fp32 unit roundoff and gamma(n) = n u / (1 - n u) the standard bound on the relative error
of an n-term fp32 sum or dot product (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., sec. 3.1)."""
import math

import torch

from oracle import geometry, nets

U = 2.0 ** -24
OFFSET = 100.0  # predict_score.py:207


def gamma(n):
    return n * U / (1.0 - n * U)


def spans(seg):
    return list(zip(seg[:-1], seg[1:]))


def state_dict64(sd, device):
    """The scorer tail's tensors of a reference-layout state dict, in float64 on `device`."""
    keys = ("att_cross.in_proj_weight", "att_cross.in_proj_bias", "att_cross.out_proj.weight", "att_cross.out_proj.bias",
            "linear.weight", "linear.bias")
    return {k: sd[k].to(device=device, dtype=torch.float64) for k in keys}


@torch.no_grad()
def tail_ref(sd64, x, seg, extra_key=None):
    """score_network.py:84-88 per segment, in the dtype of `x`: oracle.nets.mha over the segment's rows, then
    Linear(512, 1), plus the +100 of predict_score.py:207.  out_proj and linear are applied one after the other (not the
    kernel's folded vector), so the comparison also checks the fold of fp_load_network.  extra_key = g: segment g's
    keys (and values) also include the next row, the first of its neighbour (a probe: a wrong key range)."""
    out = []
    for g, (a, b) in enumerate(spans(seg)):
        rows = x[a:b + 1] if g == extra_key else x[a:b]
        y = nets.mha(rows[None], sd64, "att_cross")[0][: b - a]
        out.append((y @ sd64["linear.weight"].t() + sd64["linear.bias"]).reshape(-1))
    return torch.cat(out) + OFFSET


@torch.no_grad()
def tail_bar(sd64, x, seg):
    """Per-score bound on |kernel - tail_ref| for fp32 features `x` (held in float64), from the operation order of
    fp_attn.cu (rowwise_linear_kernel, cross_attn_score_kernel).  A sum evaluated as a tree of depth d is within
    gamma(d) sum |terms| of the exact sum; each fused multiply-add is one rounding.

    1. in-projection: per lane 16 FMAs, a 5-level butterfly, + bias (depth 22):
         |dqkv_j| <= E_j = gamma(22) (sum_i |W_ji x_i| + |b_j|)
    2. logit = fl(fl(q . k) * fl(1/sqrt(128))): 4 products per lane, the butterfly, the rounded scale (depth 11):
         |ds_k| <= scale (1 + gamma(11)) (|q| . E_k + E_q . |k| + E_q . E_k) + gamma(11) scale |q| . |k|
       expf (within 2 ulp < 5u relatively) of the rounded argument fl(s_k - max) (|s_k - max| u) perturbs e_k as a
       logit error would, so every weight's logit is off by at most eps = max_k |ds_k| + 5u + D u, D = max |s_k - max|
       (+ 2 max |ds_k|).
    3. softmax: logits off by <= eps give p'_k = p_k e^(d_k) / sum_j p_j e^(d_j), within (e^(2 eps) - 1) p_k of p_k, and
       sum_k p'_k = sum_k p_k = 1.  With z_k = v_k . w (key k's value read out through w = out_proj.weight^T
       linear.weight, per head) and zbar = sum_k p_k z_k the head's exact read-out:
         |sum_k (p'_k - p_k) z_k| = |sum_k (p'_k - p_k)(z_k - zbar)| <= (e^(2 eps) - 1) sum_k p_k |z_k - zbar|   (T1)
       value errors: e^(2 eps) sum_k p_k sum_d E_v,kd |w_d|                                                   (T2)
       the n-term sequential value sum per lane (depth n): gamma(n) e^(2 eps) sum_k p_k sum_d (|v_kd| + E_v,kd) |w_d|  (T3)
       the exponentials' sum (ceil(n / 32) per lane + the butterfly), 1 / sum and o * inv scale the head by one factor
       within gamma(ceil(n / 32) + 7):  head error <= T1 + T2 + T3 + gamma(ceil(n / 32) + 7) (|zbar| + T1 + T2 + T3)
    4. read-out: fold_v rounded to fp32, 4 products per lane, the butterfly, three head sums, + fold_c (rounded), + 100
       (depth 15):  |dscore| <= (1 + gamma(15)) sum_h (head error) + gamma(15) (sum_hd |a_hd w_hd| + |fold_c| + 100)
    Every step is a worst-case bound for this operation order, so the bar holds on any IEEE fp32 device; nothing in it
    is fitted to a run."""
    Win, bin_ = sd64["att_cross.in_proj_weight"], sd64["att_cross.in_proj_bias"]
    qkv = x @ Win.t() + bin_
    E = gamma(22) * (x.abs() @ Win.abs().t() + bin_.abs())
    wv = (sd64["linear.weight"].reshape(-1) @ sd64["att_cross.out_proj.weight"]).reshape(4, 128, 1)  # per head [128][1]
    c = float((sd64["linear.weight"].reshape(-1) @ sd64["att_cross.out_proj.bias"] + sd64["linear.bias"]).abs())
    scale = 1.0 / math.sqrt(128.0)
    g11, g15 = gamma(11), gamma(15)
    out = []
    for a, b in spans(seg):
        n = b - a

        def heads(t, part):
            return t[a:b, 512 * part:512 * (part + 1)].reshape(n, 4, 128).transpose(0, 1)  # (4, n, 128)

        q, k, v = heads(qkv, 0), heads(qkv, 1), heads(qkv, 2)
        Eq, Ek, Ev = heads(E, 0), heads(E, 1), heads(E, 2)
        s = scale * (q @ k.transpose(1, 2))
        ds = scale * (1 + g11) * (q.abs() @ Ek.transpose(1, 2) + Eq @ k.abs().transpose(1, 2) + Eq @ Ek.transpose(1, 2))
        ds = (ds + g11 * scale * (q.abs() @ k.abs().transpose(1, 2))).amax(-1)  # (4, n)
        D = (s.amax(-1, keepdim=True) - s).amax(-1) + 2 * ds
        eps = ds + 5 * U + D * U
        grow = torch.exp(2 * eps)
        P = torch.softmax(s, dim=-1)  # (4, n, n)
        z = (v @ wv).squeeze(-1)  # (4, n): each key's value read out
        zbar = P @ z[..., None]  # (4, n, 1)
        T1 = (grow - 1) * (P * (z[:, None, :] - zbar).abs()).sum(-1)
        zeta = (Ev @ wv.abs()).squeeze(-1)  # (4, n)
        T2 = grow * (P @ zeta[..., None]).squeeze(-1)
        T3 = gamma(n) * grow * (P @ ((v.abs() + Ev) @ wv.abs())).squeeze(-1)
        head = T1 + T2 + T3
        head = head + gamma(-(-n // 32) + 7) * (zbar.squeeze(-1).abs() + head)
        att = P @ v  # (4, n, 128)
        readout = (att.abs() @ wv.abs()).squeeze(-1).sum(0)
        out.append((1 + g15) * head.sum(0) + g15 * (readout + c + OFFSET))
    return torch.cat(out)


def first_argmax(v):
    """First index of the maximum (estimater.py:226 takes ids[0] of a stable descending sort)."""
    v = torch.as_tensor(v)
    return int(torch.nonzero(v == v.max())[0, 0])


@torch.no_grad()
def pose_update_ref(poses, trans, rot, half_diam, rot_normalizer):
    """predict_pose_refine.py:195-231 + Utils.py:848-855 in float64 on the fp32 inputs: trans_delta = trans * half
    diameter (per hypothesis), rot_delta = so3_exp_map(tanh(rot) * rot_normalizer)^T (pytorch3d, squared norm clamped at
    1e-4: oracle.geometry.so3_exp_map is dtype-generic), R' = rot_delta R, t' = t + trans_delta."""
    poses, trans, rot = poses.double(), trans.double(), rot.double()
    td = trans * half_diam.double()[:, None]
    rd = geometry.so3_exp_map(torch.tanh(rot) * float(rot_normalizer)).transpose(1, 2)
    out = torch.zeros_like(poses)
    out[:, 3, 3] = 1.0
    out[:, :3, :3] = rd @ poses[:, :3, :3]
    out[:, :3, 3] = poses[:, :3, 3] + td
    return out, td, rd


# bound on |rot_delta entry - reference| of pose_update_kernel (see pose_update_bars)
ROT_DELTA_BAR = 24 * U


def pose_update_bars(poses, rd_ref, td_ref):
    """Per-element bars of pose_update_kernel's outputs against pose_update_ref, for |tanh(rot) * rot_normalizer| <=
    theta_max = 0.35 sqrt(3) = 0.61 (rot_normalizer = 20 degrees):
      v = fl(tanhf(r) * rn): tanhf within 2 ulp, one product: |dv| <= 5u |v|, so theta = |v| is off by 7.5u relatively
      (the 3-term squared norm gamma(3) + 2 * 5u, halved by the square root, + its rounding).  rot_delta = f1 K + f2 K^2 + I:
      f1 = sinf(th) / th within 10u relatively (sinf 2 ulp, the reciprocal and product, th's own error scaled by
      th^2 / 3); f2 = (1 - cosf(th)) / th^2: cosf's 2 ulp = 2^-23 absolute on 1 - cos (the subtraction is exact) is
      2^-23 / (th^2 / 2) relatively, and f2 |K^2| <= th^2 / 2, so the f2 term is off by <= 2^-23 + 20u th^2 / 2; the f1
      term by <= th (5u + 10u + u); the two sums with I round at <= 2u (1 + th + th^2).  With th <= 0.61:
      9.8u + 2u + 3.8u + 2u * 1.98 < 24u per rot_delta entry (ROT_DELTA_BAR).
      R' = rot_delta R (3 products, 2 sums): sum_k ROT_DELTA_BAR |R_kj| + gamma(3) sum_k |rot_delta_ik R_kj|.
      trans_delta = fl(trans * half): u |trans_delta|;  t' = fl(t + trans_delta): 2u (|t| + |trans_delta|)."""
    R = poses[:, :3, :3].double().abs()
    bar_R = ROT_DELTA_BAR * R.sum(1, keepdim=True).expand(-1, 3, -1) + gamma(3) * (rd_ref.abs() @ R)
    bar_td = U * td_ref.abs()
    bar_t = 2 * U * (poses[:, :3, 3].double().abs() + td_ref.abs())
    return bar_R, bar_td, bar_t
