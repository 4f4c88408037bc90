"""Vectorised exact reference of the crop producer (csrc/fp_crop.cu, crop_tile_kernel), for the pixel tests.

Everything the kernel computes with explicit round-to-nearest intrinsics and no contraction is restated here in fp32
with one elementwise torch op per rounding (a separate kernel per op, so nothing is fused), and is therefore
bit-exact: the crop window (oracle/geometry.crop_window), the vertex transform and its 1/256 px snap (xform_vertex),
the integer edge functions with the top-left tie rule (tri_cover), the screen-space barycentrics and the interpolated
1/Z (inv_depth), the 64-bit depth key (iz bits << 32 | 0xFFFFFFFF - face), the homogeneous path of triangles crossing
the near plane (hom_setup / hom_cover), and the per-axis tap tables of the observed-crop resampling.  Division is
`a / b` and reciprocals `1.0 / x` (IEEE round to nearest, like __fdiv_rn / __frcp_rn); torch.compile is not used.

Coverage is enumerated from (triangle, pixel) candidate pairs: each triangle's pixel-centre bounding box, clipped to
the crop.  At 160 px most triangles of a large mesh cover 0 to 2 centres, so the pairs are few and the same code runs
on the CPU (cross-checked against oracle/raster.py) and on the GPU at 252 hypotheses.  The depth test is a
scatter_reduce(amax) of the keys per pixel.

Culling is the kernel's rule, stated: with `front_sign != 0` and the mesh's bounding sphere entirely beyond the near
plane, a triangle whose snapped area2 is zero or has the other sign is skipped (raster_tri); every other triangle is
rasterised.  The kernel's meshlet binning (bounding spheres, normal cones) has no counterpart here: it is an
optimisation, and where it is correct the kernel's coverage equals this one exactly.

The shading lines of the kernel are plain fp32 expressions the compiler may contract, so the values (rendered rgb and
xyz, observed rgb and xyz) are computed in float64 from the exact fp32 barycentrics, weights and taps, and compared
within a bar.
"""
import numpy as np
import torch

from oracle import geometry

S = 160
f32 = torch.float32
TAU = (float(np.float32(0.001)), float(np.float32(0.1)))  # normalise_xyz's cut, fp32: refiner, scorer
ZNEAR, ZFAR = float(np.float32(0.001)), 100.0  # CropParams::znear / zfar (fp32)


def _c(x, dev):
    return torch.tensor(x, dtype=f32, device=dev)


def windows(poses, K, diameter, crop_ratio=1.2):
    """Crop window (left, top, sx, sy) and render window (umin, vmin, rsx, rsy) of each pose, fp32 numpy, as
    crop_window_warp computes them.  The radius is the context's r3: the fp32 diameter times the fp32 crop ratio / 2,
    in double, rounded to fp32."""
    win, _ = geometry.crop_window(np.asarray(poses, dtype=np.float32), K, float(np.float32(diameter)),
                                  float(np.float32(crop_ratio)), S)
    umin, vmin, umax, vmax = geometry.render_window(win, S)
    rsx = (np.float32(S) / (umax - umin).astype(np.float32)).astype(np.float32)
    rsy = (np.float32(S) / (vmax - vmin).astype(np.float32)).astype(np.float32)
    return dict(left=win["left"], top=win["top"], sx=win["sx"], sy=win["sy"], umin=umin, vmin=vmin, rsx=rsx, rsy=rsy)


class Scene:
    """One mesh and one frame on a device.  mesh: dict(pos, faces, normals, and uv + tex | vcolor) as
    oracle.pipeline.mesh_tensors returns it; frame: rgb uint8 (H,W,3), depth (H,W) and xyz_map (H,W,3) float32 as the
    kernel reads them; K the intrinsics; front_sign / bounding sphere as fp_set_mesh derives them (0 = no culling)."""

    def __init__(self, mesh, K, rgb, depth, xyz_map, diameter, front_sign=0, sphere=None, device="cpu"):
        dev = torch.device(device)
        self.dev = dev
        t = lambda a, dt=f32: (a if torch.is_tensor(a) else torch.as_tensor(np.asarray(a))).to(dev, dt)
        self.pos = t(mesh["pos"])
        self.faces = t(mesh["faces"], torch.int64)
        self.nrm = t(mesh["normals"])
        self.tex = None if mesh.get("tex") is None else t(mesh["tex"][..., :3], torch.uint8)
        self.uv = t(mesh["uv"]) if self.tex is not None else None
        self.vcol = t(mesh["vcolor"]) if self.tex is None else None
        K = np.asarray(K, dtype=np.float32)
        self.fx, self.fy, self.cx, self.cy = (float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]))
        self.K = K
        self.rgb = t(rgb, torch.uint8)
        self.depth = t(depth)
        self.xyz = t(xyz_map)
        self.H, self.W = self.depth.shape
        self.diameter = diameter
        self.inv_radius = float(np.float32(1.0) / (np.float32(diameter) / np.float32(2.0)))
        self.front_sign = int(front_sign)
        self.sphere = sphere  # (x, y, z, r) float32, only read when front_sign != 0

    # ---------------------------------------------------------------------------------------------------------------
    def cull_sign(self, P):
        """Per pose: the front_sign raster_tri uses, 0 when the bounding sphere reaches the near plane (a front face
        clipped by it would uncover the back faces behind it)."""
        if self.front_sign == 0:
            return torch.zeros(len(P), dtype=torch.int64, device=self.dev)
        Pd = P.double()
        c = torch.tensor(self.sphere[:3], dtype=torch.float64, device=self.dev)
        zc = Pd[:, 2, :3] @ c + Pd[:, 2, 3]
        return torch.where(zc - float(self.sphere[3]) <= ZNEAR, 0, self.front_sign).to(torch.int64)

    def project(self, P, win):
        """xform_vertex for every vertex of every pose: X, Y, Z, iz (n,V) fp32 and the snapped xi, yi (n,V) int64."""
        dev = self.dev
        x, y, z = self.pos[:, 0][None], self.pos[:, 1][None], self.pos[:, 2][None]
        e = lambda i, j: P[:, i, j][:, None]
        X = ((e(0, 0) * x + e(0, 1) * y) + e(0, 2) * z) + e(0, 3)
        Y = ((e(1, 0) * x + e(1, 1) * y) + e(1, 2) * z) + e(1, 3)
        Z = ((e(2, 0) * x + e(2, 1) * y) + e(2, 2) * z) + e(2, 3)
        iz = 1.0 / Z
        u = (_c(self.fx, dev) * X) * iz + _c(self.cx, dev)
        v = (_c(self.fy, dev) * Y) * iz + _c(self.cy, dev)
        px = ((u - win["umin"][:, None]) * win["rsx"][:, None]).clamp(-30000.0, 30000.0)
        py = ((v - win["vmin"][:, None]) * win["rsy"][:, None]).clamp(-30000.0, 30000.0)
        xi = torch.round(px * _c(256.0, dev)).to(torch.int64)
        yi = torch.round(py * _c(256.0, dev)).to(torch.int64)
        return X, Y, Z, iz, xi, yi

    def rays(self, win):
        """pixel_ray of every crop column / row: (n,S) fp32 each."""
        dev = self.dev
        c = torch.arange(S, dtype=f32, device=dev)[None] + _c(0.5, dev)
        dx = ((win["umin"][:, None] + c / win["rsx"][:, None]) - _c(self.cx, dev)) / _c(self.fx, dev)
        dy = ((win["vmin"][:, None] + c / win["rsy"][:, None]) - _c(self.cy, dev)) / _c(self.fy, dev)
        return dx, dy

    # ---------------------------------------------------------------------------------------------------------------
    def _win_t(self, win):
        return {k: torch.as_tensor(np.asarray(v), dtype=f32, device=self.dev) for k, v in win.items()}

    def run(self, poses, mode, cull=True, drop_faces=None, tie_flip=False, border=False, second=False, chunk=16):
        """Everything the kernel's dbg record and window output hold, for poses (N,4,4).  Returns a dict:
          win      the window dict (numpy fp32)
          face     (N,S,S) int64 winning face, -1 = empty
          bary     (N,S,S,3) fp32 weights of its vertices: screen-space barycentrics, or the perspective-correct
                   weights of the homogeneous path when a vertex is behind the near plane
          A, B     (N,S,S,6) float64 rendered / observed values (dbg layout: rgb, normalised xyz)
          barA, barB   per-element bars (see the test file), near  (N,S,S,6) bool: within its bar of a discontinuity
          face2, A2    with second=True: the second-nearest covering face and the rendered values it would give
        Options that state a deliberately wrong rule (defect probes): cull=False (reference culling off), drop_faces
        (bool mask over faces never rasterised), tie_flip (top-left rule mirrored), border (border padding of the
        bilinear taps instead of zeros)."""
        P_all = torch.as_tensor(np.asarray(poses, dtype=np.float32), device=self.dev)
        win_np = windows(poses, self.K, self.diameter)
        win_all = self._win_t(win_np)
        out = {k: [] for k in ("face", "bary", "A", "barA", "nearA", "B", "barB", "nearB", "face2", "A2", "bar2")}
        for s in range(0, len(P_all), chunk):
            P = P_all[s:s + chunk]
            win = {k: v[s:s + chunk] for k, v in win_all.items()}
            key, key2 = self._cover(P, win, mode, cull, drop_faces, tie_flip, second)
            face, bary, A, barA, nearA = self._shade(P, win, key, mode)
            B, barB, nearB = self._observed(P, win, mode, border)
            for k, v in (("face", face), ("bary", bary), ("A", A), ("barA", barA), ("nearA", nearA), ("B", B), ("barB", barB), ("nearB", nearB)):
                out[k].append(v)
            if second:
                f2, _, A2, bar2, _ = self._shade(P, win, key2, mode)
                out["face2"].append(f2)
                out["A2"].append(A2)
                out["bar2"].append(bar2)
        res = {k: torch.cat(v) for k, v in out.items() if v}
        res["win"] = win_np
        return res

    # ---------------------------------------------------------------------------------------------------------------
    def _cover(self, P, win, mode, cull, drop_faces, tie_flip, second):
        """Depth keys (n, S*S) int64 (0 = empty) of the nearest and, with `second`, the second-nearest covering face."""
        dev = self.dev
        n = len(P)
        X, Y, Z, iz, xi, yi = self.project(P, win)
        fa, fb, fc = self.faces[:, 0], self.faces[:, 1], self.faces[:, 2]
        zn = _c(ZNEAR, dev)
        nfront = (Z[:, fa] > zn).long() + (Z[:, fb] > zn).long() + (Z[:, fc] > zn).long()
        x0, y0, x1, y1, x2, y2 = xi[:, fa], yi[:, fa], xi[:, fb], yi[:, fb], xi[:, fc], yi[:, fc]
        area2 = (x1 - x0) * (y2 - y0) - (y1 - y0) * (x2 - x0)
        planar = (nfront == 3) & (area2 != 0)
        mixed = (nfront > 0) & (nfront < 3)
        if cull:
            cs = self.cull_sign(P)[:, None]
            planar &= (cs == 0) | (torch.sign(area2) == cs)
        if drop_faces is not None:
            keep = ~torch.as_tensor(drop_faces, device=dev)[None]
            planar &= keep
            mixed &= keep
        j0 = ((torch.minimum(torch.minimum(x0, x1), x2) + 127) >> 8).clamp(min=0)
        j1 = ((torch.maximum(torch.maximum(x0, x1), x2) - 128) >> 8).clamp(max=S - 1)
        r0 = ((torch.minimum(torch.minimum(y0, y1), y2) + 127) >> 8).clamp(min=0)
        r1 = ((torch.maximum(torch.maximum(y0, y1), y2) - 128) >> 8).clamp(max=S - 1)
        w, h = j1 - j0 + 1, r1 - r0 + 1
        cnt = torch.where(planar & (w > 0) & (h > 0), w * h, 0)
        pi, fi = torch.nonzero(cnt, as_tuple=True)
        c = cnt[pi, fi]
        rep = torch.repeat_interleave(torch.arange(len(c), device=dev), c)
        local = torch.arange(int(c.sum()), device=dev) - (torch.cumsum(c, 0) - c)[rep]
        pi, fi = pi[rep], fi[rep]
        ww = w[pi, fi]
        j = j0[pi, fi] + local % ww
        r = r0[pi, fi] + local // ww
        ok, b0, b1, b2 = planar_bary(x0[pi, fi], y0[pi, fi], x1[pi, fi], y1[pi, fi], x2[pi, fi], y2[pi, fi],
                                     j * 256 + 128, r * 256 + 128, tie_flip)
        izp = inv_depth(b0, b1, b2, iz[pi, fa[fi]], iz[pi, fb[fi]], iz[pi, fc[fi]])
        ok &= izp > 1.0 / _c(ZFAR, dev)
        keys = [_key(izp[ok], fi[ok])]
        pix = [pi[ok] * S * S + r[ok] * S + j[ok]]
        # triangles crossing the near plane: the homogeneous path over the whole crop
        mp, mf = torch.nonzero(mixed, as_tuple=True)
        if len(mp):
            dx, dy = self.rays(win)
            Pc = [torch.stack([X[mp, v[mf]], Y[mp, v[mf]], Z[mp, v[mf]]], -1) for v in (fa, fb, fc)]
            for s in range(0, len(mp), 64):
                sl = slice(s, s + 64)
                ok, _, izh = hom_cover([p[sl] for p in Pc], dx[mp[sl]][:, None, :], dy[mp[sl]][:, :, None])
                t_, rr, jj = torch.nonzero(ok, as_tuple=True)
                keys.append(_key(izh[t_, rr, jj], mf[sl][t_]))
                pix.append(mp[sl][t_] * S * S + rr * S + jj)
        keys, pix = torch.cat(keys), torch.cat(pix)
        key = torch.zeros(n * S * S, dtype=torch.int64, device=dev).scatter_reduce(0, pix, keys, "amax")
        key2 = None
        if second:
            lower = keys < key[pix]
            key2 = torch.zeros_like(key).scatter_reduce(0, pix[lower], keys[lower], "amax")
        return key.view(n, S, S), None if key2 is None else key2.view(n, S, S)

    # ---------------------------------------------------------------------------------------------------------------
    def _shade(self, P, win, key, mode):
        """Rendered crop of the faces the keys name: (face, bary, A, bar, near) as in run()."""
        dev = self.dev
        n = len(P)
        face = torch.where(key != 0, 0xFFFFFFFF - (key & 0xFFFFFFFF), -1)
        A = torch.zeros(n, S, S, 6, dtype=torch.float64, device=dev)
        bar = torch.zeros_like(A)
        near = torch.zeros(n, S, S, 6, dtype=torch.bool, device=dev)
        bary = torch.zeros(n, S, S, 3, dtype=f32, device=dev)
        pi, r, j = torch.nonzero(face >= 0, as_tuple=True)
        if len(pi) == 0:
            return face, bary, A, bar, near
        b32 = torch.zeros(len(pi), 3, dtype=f32, device=dev)
        f = face[pi, r, j]
        vid = self.faces[f]  # (M,3)
        X, Y, Z, iz, xi, yi = self.project(P, win)
        g = lambda a: a[pi[:, None], vid]  # (M,3)
        Xv, Yv, Zv, izv, xv, yv = g(X), g(Y), g(Z), g(iz), g(xi), g(yi)
        planar = (Zv > _c(ZNEAR, dev)).all(1)
        w = torch.zeros(len(pi), 3, dtype=torch.float64, device=dev)
        wrel = torch.zeros(len(pi), dtype=torch.float64, device=dev)  # relative error of the kernel's weights, in u
        if planar.any():
            q = planar
            _, b0, b1, b2 = planar_bary(xv[q, 0], yv[q, 0], xv[q, 1], yv[q, 1], xv[q, 2], yv[q, 2],
                                        j[q] * 256 + 128, r[q] * 256 + 128)
            izp = inv_depth(b0, b1, b2, izv[q, 0], izv[q, 1], izv[q, 2]).double()
            b32[q] = torch.stack([b0, b1, b2], 1)
            w[q] = b32[q].double() * izv[q].double() / izp[:, None]
            wrel[q] = 3.0  # z = 1 / iz, b * iz, (b * iz) * z: three roundings
        if (~planar).any():
            q = ~planar
            dx, dy = self.rays(win)
            _, lam, _ = hom_cover([torch.stack([Xv[q, k], Yv[q, k], Zv[q, k]], -1) for k in range(3)],
                                  dx[pi[q], j[q]], dy[pi[q], r[q]])
            b32[q] = lam
            w[q] = lam.double()  # bit-exact in the kernel (hom_cover is all _rn intrinsics)
        cam = torch.stack([Xv, Yv, Zv], -1).double()  # (M,3 vertices,3 coords)
        xyz = (w[..., None] * cam).sum(1)
        mag = (w.abs()[..., None] * cam.abs()).sum(1)  # sum_i |w_i| |X_i|
        # per-vertex Lambert term: clip(normalize(R n) . (0,0,-1), 0, 1)
        R = P[:, :3, :3].double()[pi]
        nc = (R[:, None] @ self.nrm[vid].double()[..., None])[..., 0]  # (M,3,3)
        dif = (-nc[..., 2] / nc.norm(dim=-1).clamp(min=1e-12)).clamp(0, 1)
        diffuse = (w * dif).sum(1)
        U = 2.0 ** -24
        if self.tex is not None:
            Ht, Wt = self.tex.shape[:2]
            uv = self.uv[vid].double()
            tu, tv = (w[..., None] * uv).sum(1).unbind(-1)
            muv = (w.abs()[..., None] * uv.abs()).sum(1)
            col, slope = _bilinear_wrap(self.tex, tu * Wt - 0.5, tv * Ht - 0.5)
            # tu, tv: the weights' roundings + 2 of the sum; x = tu * Wt - 0.5: 2 more (or one fused); the fraction: 1
            dxx = (wrel + 2) * U * muv[:, 0] * Wt + 2 * U * (tu.abs() * Wt + 0.5) + U
            dyy = (wrel + 2) * U * muv[:, 1] * Ht + 2 * U * (tv.abs() * Ht + 0.5) + U
            dcol = slope * (dxx + dyy)[:, None] + 12 * U * col
        else:
            col = (w[..., None] * self.vcol[vid].double()).sum(1)
            dcol = (wrel + 2)[:, None] * U * (w.abs()[..., None] * self.vcol[vid].double()).sum(1)
        shaded = col * 0.8 + diffuse[:, None] * col * 0.5
        rgb = shaded.clamp(0, 1)
        # diffuse: each vertex term ~10 roundings (transform, norm, division), then the weights and a 3-term sum
        ddif = (10 + wrel + 2) * U * (w.abs() * dif).sum(1) + 10 * U
        drgb = (0.8 + 0.5 * diffuse)[:, None] * dcol + 0.5 * col * ddif[:, None] + 4 * U * shaded.abs()
        t = P[:, :3, 3].double()[pi]
        o, dxyz, nr = _normalise(xyz, t, self.inv_radius, TAU[mode],
                                 (wrel[:, None] + 2) * U * mag)
        A[pi, r, j] = torch.cat([rgb, o], 1)
        bar[pi, r, j] = 2 * torch.cat([drgb, dxyz], 1) + 1e-12
        near_rgb = ((shaded - 0).abs() <= 2 * drgb) | ((shaded - 1).abs() <= 2 * drgb)
        near[pi, r, j] = torch.cat([near_rgb, nr], 1)
        bary[pi, r, j] = b32
        return face, bary, A, bar, near

    # ---------------------------------------------------------------------------------------------------------------
    def taps(self, win, tie_tol=0.0):
        """The per-axis tables of crop_tile_kernel for every crop column (size W) and row (size H), fp32 exact:
        dict(col=..., row=...) of dict(n nearest (-1 outside), z depth round trip (-1 none), i0 first bilinear tap
        (clamped to [-2, size]), frac weight of the second tap, tie: a nearest index rounded a coordinate within tie_tol of x.5), each (n,S)."""
        dev = self.dev
        d = torch.arange(S, dtype=f32, device=dev)[None]
        out = {}
        for name, sc, org, size in (("col", win["sx"], win["left"], self.W), ("row", win["sy"], win["top"], self.H)):
            sc, org = sc[:, None], org[:, None]
            ix = kornia_src_coord(d / sc + org, size)
            un = torch.round(ix).long()
            un = torch.where((un < 0) | (un >= size), -1, un)
            xc = sc * un.to(f32) + (-org) * sc
            kc = kornia_src_coord(xc, S)
            jc = torch.round(kc).long()
            k2 = kornia_src_coord(jc.to(f32) / sc + org, size)
            u2 = torch.round(k2).long()
            half = lambda x: ((x - torch.floor(x)) - 0.5).abs() <= tie_tol
            tie = half(ix) | half(kc) | half(k2)
            uz = torch.where((un >= 0) & (jc >= 0) & (jc < S) & (u2 >= 0) & (u2 < size), u2, -1)
            f0 = torch.floor(ix)
            i0 = f0.clamp(-2.0, float(size)).long()
            out[name] = dict(n=un, z=uz, i0=i0, frac=ix - f0, size=size, tie=tie)
        return out

    def _observed(self, P, win, mode, border):
        dev = self.dev
        n = len(P)
        U = 2.0 ** -24
        tb = self.taps(win)
        ax = []
        for a in (tb["col"], tb["row"]):
            size, i0, fr = a["size"], a["i0"], a["frac"].double()
            if border:  # the wrong padding: taps clamped into the image, weights never zeroed
                k0, k1 = i0.clamp(0, size - 1), (i0 + 1).clamp(0, size - 1)
                w0, w1 = 1 - fr, fr
            else:
                k0, k1 = i0.clamp(0, size - 1), (i0 + 1).clamp(0, size - 1)
                w0 = torch.where((i0 < 0) | (i0 >= size), 0.0, 1 - fr)
                w1 = torch.where((i0 + 1 < 0) | (i0 + 1 >= size), 0.0, fr)
            ax.append((k0, k1, w0, w1))
        (c0, c1, wc0, wc1), (r0, r1, wr0, wr1) = ax
        img = self.rgb.double()
        bidx = lambda rr, cc: img[rr[:, :, None], cc[:, None, :]]  # (n,S,S,3)
        rgb = (wr0[:, :, None, None] * wc0[:, None, :, None] * bidx(r0, c0) + wr0[:, :, None, None] * wc1[:, None, :, None] * bidx(r0, c1)
               + wr1[:, :, None, None] * wc0[:, None, :, None] * bidx(r1, c0) + wr1[:, :, None, None] * wc1[:, None, :, None] * bidx(r1, c1)) / 255.0
        cn, rn = tb["col"]["n"], tb["row"]["n"]
        valid = (cn[:, None, :] >= 0) & (rn[:, :, None] >= 0)
        rc, cc = rn.clamp(min=0)[:, :, None], cn.clamp(min=0)[:, None, :]
        if mode == 0:
            xyz = torch.where(valid[..., None], self.xyz[rc, cc], 0.0).double()
        else:
            cz, rz = tb["col"]["z"], tb["row"]["z"]
            vz = valid & (cz[:, None, :] >= 0) & (rz[:, :, None] >= 0)
            zz = torch.where(vz, self.depth[rz.clamp(min=0)[:, :, None], cz.clamp(min=0)[:, None, :]], 0.0)
            okz = zz >= _c(0.001, dev)
            Xs = ((cc.expand(n, S, S).to(f32) - _c(self.cx, dev)) * zz) / _c(self.fx, dev)
            Ys = ((rc.expand(n, S, S).to(f32) - _c(self.cy, dev)) * zz) / _c(self.fy, dev)
            xyz = torch.where(okz[..., None], torch.stack([Xs, Ys, zz], -1), 0.0).double()
        t = P[:, :3, 3].double()
        o, dxyz, nr = _normalise(xyz.reshape(-1, 3), t[:, None, None].expand(n, S, S, 3).reshape(-1, 3), self.inv_radius,
                                 TAU[mode], torch.zeros(n * S * S, 3, dtype=torch.float64, device=dev))
        B = torch.cat([rgb, o.view(n, S, S, 3)], -1)
        # rgb: 4 weight products (2 roundings each), a 4-term sum, the 1/255 scale and its constant
        bar = 2 * torch.cat([10 * U * rgb.abs() + U * 1e-3, dxyz.view(n, S, S, 3)], -1) + 1e-12
        near = torch.cat([torch.zeros_like(rgb, dtype=torch.bool), nr.view(n, S, S, 3)], -1)
        return B, bar, near


# ---------------------------------------------------------------------------------------------------------------------
def planar_bary(x0, y0, x1, y1, x2, y2, px, py, tie_flip=False):
    """tri_setup + tri_cover (64-bit edge functions, top-left rule) at pixel centres (px, py) in 1/256 px, elementwise.
    Returns (inside, b0, b1, b2): fp32 screen-space weights of the vertices in their original order."""
    area2 = (x1 - x0) * (y2 - y0) - (y1 - y0) * (x2 - x0)
    sw = area2 < 0
    x1, y1, x2, y2 = torch.where(sw, x2, x1), torch.where(sw, y2, y1), torch.where(sw, x1, x2), torch.where(sw, y1, y2)
    area2 = area2.abs()
    e0 = (x2 - x1) * (py - y1) - (y2 - y1) * (px - x1)
    e1 = (x0 - x2) * (py - y2) - (y0 - y2) * (px - x2)
    e2 = area2 - e0 - e1
    ok = (area2 != 0) & _edge_ok(e0, x2 - x1, y2 - y1, tie_flip) & _edge_ok(e1, x0 - x2, y0 - y2, tie_flip) \
        & _edge_ok(e2, x1 - x0, y1 - y0, tie_flip)
    fa = area2.to(f32)
    b0, w1, w2 = e0.to(f32) / fa, e1.to(f32) / fa, e2.to(f32) / fa
    return ok, b0, torch.where(sw, w2, w1), torch.where(sw, w1, w2)


def _edge_ok(e, dx, dy, flip=False):
    if flip:
        dx, dy = -dx, -dy
    return (e > 0) | ((e == 0) & ((dy > 0) | ((dy == 0) & (dx > 0))))


def inv_depth(b0, b1, b2, iz0, iz1, iz2):
    return (b0 * iz0 + b1 * iz1) + b2 * iz2


def _key(iz, face):
    return (iz.view(torch.int32).to(torch.int64) << 32) | (0xFFFFFFFF - face)


def hom_cover(Pv, dx, dy):
    """hom_setup + hom_cover: Pv = three (..., 3) fp32 camera-space vertices, broadcast against the ray components
    dx, dy.  Returns (inside, lam (..., 3) fp32 perspective-correct weights, iz)."""
    A, B, C = [p.unbind(-1) for p in Pv]
    ex = lambda t: t.reshape(t.shape + (1,) * max(0, dx.dim() - 1))

    def cross(a, b):
        return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])

    ns = [cross(B, C), cross(C, A), cross(A, B)]
    det = (A[0] * ns[0][0] + A[1] * ns[0][1]) + A[2] * ns[0][2]
    w = [((ex(nv[0]) * dx + ex(nv[1]) * dy) + ex(nv[2])) / ex(det) for nv in ns]
    iz = (w[0] + w[1]) + w[2]
    z = 1.0 / iz
    ok = (ex(det) != 0) & (w[0] >= 0) & (w[1] >= 0) & (w[2] >= 0) & (iz > 0) & (z > _c(ZNEAR, z.device)) \
        & (z < _c(ZFAR, z.device))
    return ok, torch.stack([w[0] * z, w[1] * z, w[2] * z], -1), iz


def kornia_src_coord(x, size):
    # a division by a Python number is a multiplication by its reciprocal on CUDA: divide by a device scalar
    xn = (2.0 * x) / _c(size - 1, x.device) - 1.0
    return (((xn + 1.0) * float(size)) - 1.0) * 0.5


def _bilinear_wrap(tex, x, y):
    """dr.texture linear filtering with wrap, float64 at continuous texel coordinates x, y (texel centres at
    integers).  Returns the colour (M,3) in 0..1 and the largest colour step between the four taps (the slope bound
    per texel unit)."""
    Ht, Wt = tex.shape[:2]
    xf, yf = torch.floor(x), torch.floor(y)
    ax, ay = (x - xf)[:, None], (y - yf)[:, None]
    x0, y0 = torch.remainder(xf.long(), Wt), torch.remainder(yf.long(), Ht)
    x1, y1 = torch.remainder(x0 + 1, Wt), torch.remainder(y0 + 1, Ht)
    t = [tex[a, b].double() / 255.0 for a, b in ((y0, x0), (y0, x1), (y1, x0), (y1, x1))]
    col = (1 - ax) * (1 - ay) * t[0] + ax * (1 - ay) * t[1] + (1 - ax) * ay * t[2] + ax * ay * t[3]
    tt = torch.stack(t, 0)
    slope = tt.amax(0) - tt.amin(0)
    return col, slope


def _normalise(xyz, t, inv_radius, tau, dxyz_in):
    """normalise_xyz in float64, its bar and the elements within their bar of the cuts (z < tau, |o| >= 2).
    The kernel rounds x - t and (x - t) * inv_radius once each, on top of the error dxyz_in of x."""
    U = 2.0 ** -24
    d = xyz - t
    o = d * inv_radius
    bar = (dxyz_in + U * d.abs()) * inv_radius + U * o.abs()
    z, dz = xyz[:, 2:3], dxyz_in[:, 2:3]
    inv = z < tau
    cut = inv | (o.abs() >= 2)
    out = torch.where(cut, 0.0, o)
    near = ((z - tau).abs() <= 2 * dz + 1e-300) | ((o.abs() - 2).abs() <= 2 * bar)
    return out, bar, near


def tie_grid(step=8, lo=20, hi=140):
    """A flat, camera-facing grid of quads whose vertices all snap exactly to pixel centres of the crop of its pose,
    so that every grid line and every quad diagonal passes through pixel centres and the tie rule decides them.
    Returns (mesh dict as pipeline.mesh_tensors gives it, pose (1,4,4) fp32, diameter)."""
    from foundationpose_b200 import synth

    K = synth.DEFAULT_K
    diameter = 0.19
    pose = np.eye(4, dtype=np.float32)[None].copy()
    pose[0, :3, 3] = [0.0, 0.0, 0.5]
    w = windows(pose, K, diameter)
    idx = np.arange(lo, hi + 1, step)
    g = len(idx)
    # invert the projection in double: the snap tolerates 1/512 px, far above the fp32 error of the forward chain
    u = w["umin"][0] + (idx + 0.5) / np.float64(w["rsx"][0])
    v = w["vmin"][0] + (idx + 0.5) / np.float64(w["rsy"][0])
    X = (u - K[0, 2]) * 0.5 / K[0, 0]
    Y = (v - K[1, 2]) * 0.5 / K[1, 1]
    yy, xx = np.meshgrid(Y, X, indexing="ij")
    pos = np.stack([xx, yy, np.zeros_like(xx)], -1).reshape(-1, 3).astype(np.float32)
    faces = []
    for r in range(g - 1):
        for c in range(g - 1):
            a, b, d, e = r * g + c, r * g + c + 1, (r + 1) * g + c, (r + 1) * g + c + 1
            faces += [[a, b, e], [a, e, d]]
    rng = np.random.default_rng(11)
    mesh = dict(pos=pos, faces=np.asarray(faces, dtype=np.int64), normals=np.tile(np.float32([0, 0, -1]), (len(pos), 1)),
                tex=None, vcolor=rng.integers(1, 256, size=(len(pos), 3)).astype(np.float32) / 255.0)
    return mesh, pose, diameter


def meshlet_of_face(verts, faces):
    """Meshlet index of every face, in the order the crop producer bins the meshlets (fp_op_build_meshlets lists the
    faces meshlet by meshlet, fp_op_meshlet_sizes gives how many each has)."""
    import ctypes as C

    from foundationpose_b200 import _lib

    lib = _lib.lib
    pos = np.ascontiguousarray(verts, dtype=np.float32)
    fc = np.ascontiguousarray(faces, dtype=np.int32)
    info = (C.c_int * 6)()
    face_of = np.full(len(fc), -1, dtype=np.int32)
    tris = np.zeros(len(fc), dtype=np.int32)
    lib.fp_op_build_meshlets.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_void_p, C.c_void_p]
    lib.fp_op_build_meshlets.restype = C.c_int
    lib.fp_op_meshlet_sizes.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.fp_op_meshlet_sizes.restype = C.c_int
    rc = lib.fp_op_build_meshlets(len(pos), len(fc), pos.ctypes.data, fc.ctypes.data, info, face_of.ctypes.data, None)
    assert rc == 0, lib.fp_last_error()
    m = lib.fp_op_meshlet_sizes(len(pos), len(fc), pos.ctypes.data, fc.ctypes.data, tris.ctypes.data)
    assert m == info[0], lib.fp_last_error()
    tris = tris[:m]
    assert tris.min() >= 1 and tris.max() <= 64 and tris.sum() == len(fc)
    out = np.empty(len(fc), dtype=np.int64)
    out[face_of] = np.repeat(np.arange(m), tris)
    return out
