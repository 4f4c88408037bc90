// fp_raster.cuh — the coverage rule of the mesh rasteriser, shared by the crop producer (fp_crop.cu) and the visible
// surface discrepancy (fp_vsd.cu): vertex transform into a raster window, exact integer coverage (64- and 32-bit edge
// functions, top-left tie rule), the depth key (interpolated 1/Z | ~face id), the homogeneous path of triangles that
// cross the near plane, the per-triangle raster loop into a TILE x TILE shared-memory z-tile, and the binning test of a
// meshlet against such a tile.  oracle/raster.py restates the same rule on the CPU.
//
// A raster window maps image coordinates (u, v) to raster pixels ((u - umin) rsx, (v - vmin) rsy); raster pixel (j, r)
// samples (j + 0.5, r + 0.5).  The crop producer's window is the crop's; a full frame is umin = vmin = 0, rsx = rsy = 1.
#pragma once
#include <cuda_runtime.h>

#include "fp_crop.cuh"

namespace fp {

struct Window {  // crop: the crop window and its render window; full frame: 0, 0, 1, 1, 0, 0, 1, 1
  float left, top, sx, sy;     // tf_to_crop = [[sx,0,-left*sx],[0,sy,-top*sy],[0,0,1]]
  float umin, vmin, rsx, rsy;  // render window origin and raster scale (pixels of crop per image pixel)
};

struct VtxScreen {
  int xi, yi;     // 1/256-pixel fixed point, crop raster space (y down)
  float iz;       // 1 / camera Z
  float X, Y, Z;  // camera-space position
};

__device__ __forceinline__ void xform_vertex(const float* __restrict__ P /*pose 4x4 row-major, smem*/, float x, float y,
                                             float z, const Window& w, float fx, float fy, float cx, float cy,
                                             VtxScreen& o) {
  o.X = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[0], x), __fmul_rn(P[1], y)), __fmul_rn(P[2], z)), P[3]);
  o.Y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[4], x), __fmul_rn(P[5], y)), __fmul_rn(P[6], z)), P[7]);
  o.Z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[8], x), __fmul_rn(P[9], y)), __fmul_rn(P[10], z)), P[11]);
  o.iz = __frcp_rn(o.Z);
  const float u = __fadd_rn(__fmul_rn(__fmul_rn(fx, o.X), o.iz), cx);
  const float v = __fadd_rn(__fmul_rn(__fmul_rn(fy, o.Y), o.iz), cy);
  float px = __fmul_rn(__fsub_rn(u, w.umin), w.rsx);
  float py = __fmul_rn(__fsub_rn(v, w.vmin), w.rsy);
  px = fminf(fmaxf(px, -30000.f), 30000.f);
  py = fminf(fmaxf(py, -30000.f), 30000.f);
  o.xi = __float2int_rn(__fmul_rn(px, 256.f));
  o.yi = __float2int_rn(__fmul_rn(py, 256.f));
}

// what the raster phase keeps per vertex in shared memory
struct __align__(16) VtxS {
  int xi, yi;
  float iz, Z;
};

// ---- exact coverage: 64-bit edge functions (any triangle) ------------------------------------------------------
struct TriSetup {
  long long area2;
  int x0, y0, x1, y1, x2, y2;  // after orientation fix (area2 > 0)
  int swapped;                 // vertices 1 and 2 were exchanged
};
__device__ __forceinline__ bool tri_setup(int ax, int ay, int bx, int by, int cx, int cy, TriSetup& t) {
  t.x0 = ax; t.y0 = ay; t.x1 = bx; t.y1 = by; t.x2 = cx; t.y2 = cy;
  t.swapped = 0;
  long long area2 = (long long)(t.x1 - t.x0) * (t.y2 - t.y0) - (long long)(t.y1 - t.y0) * (t.x2 - t.x0);
  if (area2 == 0) return false;
  if (area2 < 0) {
    int tx = t.x1, ty = t.y1;
    t.x1 = t.x2; t.y1 = t.y2; t.x2 = tx; t.y2 = ty;
    t.swapped = 1;
    area2 = -area2;
  }
  t.area2 = area2;
  return true;
}
__device__ __forceinline__ long long edge_fn(int xa, int ya, int xb, int yb, int px, int py) {
  return (long long)(xb - xa) * (py - ya) - (long long)(yb - ya) * (px - xa);
}
// tie rule: a pixel centre exactly on an edge belongs to the triangle for which the (oriented) edge
// direction satisfies dy > 0 || (dy == 0 && dx > 0): exactly one of the two triangles sharing it.
__device__ __forceinline__ bool edge_ok(long long e, int dx, int dy) {
  return e > 0 || (e == 0 && (dy > 0 || (dy == 0 && dx > 0)));
}
// barycentric weights (screen space) of the *original* vertex order a, b, c; false if outside
__device__ __forceinline__ bool tri_cover(const TriSetup& t, int px, int py, float& b0, float& b1, float& b2) {
  const long long e0 = edge_fn(t.x1, t.y1, t.x2, t.y2, px, py);  // weight of vertex 0
  const long long e1 = edge_fn(t.x2, t.y2, t.x0, t.y0, px, py);  // weight of (oriented) vertex 1
  const long long e2 = t.area2 - e0 - e1;
  if (!edge_ok(e0, t.x2 - t.x1, t.y2 - t.y1) || !edge_ok(e1, t.x0 - t.x2, t.y0 - t.y2) ||
      !edge_ok(e2, t.x1 - t.x0, t.y1 - t.y0))
    return false;
  const float fa = __ll2float_rn(t.area2);
  b0 = __fdiv_rn(__ll2float_rn(e0), fa);
  const float w1 = __fdiv_rn(__ll2float_rn(e1), fa);
  const float w2 = __fdiv_rn(__ll2float_rn(e2), fa);
  b1 = t.swapped ? w2 : w1;
  b2 = t.swapped ? w1 : w2;
  return true;
}

// ---- the same integers in 32 bits when the triangle is small enough (all deltas < 2^15, i.e. < 128 px: products
// < 2^30), relative to vertex 0: coverage is unchanged ------------------------------------------------------------
struct TriSetup32 {
  int area2;
  int x0, y0;          // vertex 0 (absolute, 1/256 px)
  int ax, ay, bx, by;  // oriented vertices 1 and 2 relative to vertex 0
  int swapped;
};
__device__ __forceinline__ bool tri_small(int x0, int y0, int x1, int y1, int x2, int y2) {
  const int m = max(max(abs(x1 - x0), abs(y1 - y0)), max(abs(x2 - x0), abs(y2 - y0)));
  return m < 16384;
}
__device__ __forceinline__ bool tri_setup32(int x0, int y0, int x1, int y1, int x2, int y2, TriSetup32& t) {
  t.x0 = x0; t.y0 = y0;
  t.ax = x1 - x0; t.ay = y1 - y0; t.bx = x2 - x0; t.by = y2 - y0;
  t.swapped = 0;
  int area2 = t.ax * t.by - t.ay * t.bx;
  if (area2 == 0) return false;
  if (area2 < 0) {
    int tx = t.ax, ty = t.ay;
    t.ax = t.bx; t.ay = t.by; t.bx = tx; t.by = ty;
    t.swapped = 1;
    area2 = -area2;
  }
  t.area2 = area2;
  return true;
}
__device__ __forceinline__ bool edge_ok32(int e, int dx, int dy) {
  return e > 0 || (e == 0 && (dy > 0 || (dy == 0 && dx > 0)));
}
// pixel centre (px, py) absolute; must lie inside the triangle's bounding box (deltas < 2^15)
__device__ __forceinline__ bool tri_cover32(const TriSetup32& t, int px, int py, float& b0, float& b1, float& b2) {
  const int qx = px - t.x0, qy = py - t.y0;
  // e0: edge v1->v2 (weight of v0); e1: edge v2->v0 (weight of v1); e2 = area2 - e0 - e1
  const int e0 = (t.bx - t.ax) * (qy - t.ay) - (t.by - t.ay) * (qx - t.ax);
  const int e1 = (-t.bx) * (qy - t.by) - (-t.by) * (qx - t.bx);
  const int e2 = t.area2 - e0 - e1;
  if (!edge_ok32(e0, t.bx - t.ax, t.by - t.ay) || !edge_ok32(e1, -t.bx, -t.by) || !edge_ok32(e2, t.ax, t.ay)) return false;
  const float fa = __int2float_rn(t.area2);
  b0 = __fdiv_rn(__int2float_rn(e0), fa);
  const float w1 = __fdiv_rn(__int2float_rn(e1), fa);
  const float w2 = __fdiv_rn(__int2float_rn(e2), fa);
  b1 = t.swapped ? w2 : w1;
  b2 = t.swapped ? w1 : w2;
  return true;
}

__device__ __forceinline__ float inv_depth(float b0, float b1, float b2, float iz0, float iz1, float iz2) {
  return __fadd_rn(__fadd_rn(__fmul_rn(b0, iz0), __fmul_rn(b1, iz1)), __fmul_rn(b2, iz2));
}
__device__ __forceinline__ unsigned long long depth_key(float iz, unsigned face) {
  return ((unsigned long long)__float_as_uint(iz) << 32) | (unsigned long long)(0xFFFFFFFFu - face);
}

// ---- homogeneous path for triangles that cross the near plane: solve [P0 P1 P2] w = d for the pixel ray d; w / sum(w)
// are the perspective-correct barycentrics, sum(w) = 1 / Z.  fp32, same order in oracle/raster.py. -------------------
struct HomTri {
  float n0x, n0y, n0z, n1x, n1y, n1z, n2x, n2y, n2z;  // P1 x P2, P2 x P0, P0 x P1
  float det;
};
__device__ __forceinline__ void hom_setup(const float* A, const float* B, const float* C, HomTri& h) {
  h.n0x = __fsub_rn(__fmul_rn(B[1], C[2]), __fmul_rn(B[2], C[1]));
  h.n0y = __fsub_rn(__fmul_rn(B[2], C[0]), __fmul_rn(B[0], C[2]));
  h.n0z = __fsub_rn(__fmul_rn(B[0], C[1]), __fmul_rn(B[1], C[0]));
  h.n1x = __fsub_rn(__fmul_rn(C[1], A[2]), __fmul_rn(C[2], A[1]));
  h.n1y = __fsub_rn(__fmul_rn(C[2], A[0]), __fmul_rn(C[0], A[2]));
  h.n1z = __fsub_rn(__fmul_rn(C[0], A[1]), __fmul_rn(C[1], A[0]));
  h.n2x = __fsub_rn(__fmul_rn(A[1], B[2]), __fmul_rn(A[2], B[1]));
  h.n2y = __fsub_rn(__fmul_rn(A[2], B[0]), __fmul_rn(A[0], B[2]));
  h.n2z = __fsub_rn(__fmul_rn(A[0], B[1]), __fmul_rn(A[1], B[0]));
  h.det = __fadd_rn(__fadd_rn(__fmul_rn(A[0], h.n0x), __fmul_rn(A[1], h.n0y)), __fmul_rn(A[2], h.n0z));
}
// pixel ray d = (dx, dy, 1); returns false outside / outside the depth range; l* = perspective-correct weights
__device__ __forceinline__ bool hom_cover(const HomTri& h, float dx, float dy, float znear, float zfar, float& l0,
                                          float& l1, float& l2, float& iz) {
  if (h.det == 0.f) return false;
  const float w0 = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(h.n0x, dx), __fmul_rn(h.n0y, dy)), h.n0z), h.det);
  const float w1 = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(h.n1x, dx), __fmul_rn(h.n1y, dy)), h.n1z), h.det);
  const float w2 = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(h.n2x, dx), __fmul_rn(h.n2y, dy)), h.n2z), h.det);
  if (!(w0 >= 0.f && w1 >= 0.f && w2 >= 0.f)) return false;
  iz = __fadd_rn(__fadd_rn(w0, w1), w2);
  if (!(iz > 0.f)) return false;
  const float z = __frcp_rn(iz);
  if (!(z > znear && z < zfar)) return false;
  l0 = __fmul_rn(w0, z);
  l1 = __fmul_rn(w1, z);
  l2 = __fmul_rn(w2, z);
  return true;
}

// one triangle of a meshlet, all three vertices in front of the near plane: coverage inside the tile + depth test
template <int TILE>
__device__ __forceinline__ void raster_tri(const VtxS& a, const VtxS& b, const VtxS& c, unsigned face, int front_sign,
                                           int tx0, int ty0, float iz_far, unsigned long long* zt, int& n_frag) {
  if (front_sign != 0) {
    // closed mesh: a back-facing triangle is always behind a front-facing one that covers the same pixel centre.
    // Same integer as the setup's area2 (the exact sign decides), computed first so that back faces leave early.
    const long long area2 = (long long)(b.xi - a.xi) * (c.yi - a.yi) - (long long)(b.yi - a.yi) * (c.xi - a.xi);
    if (area2 == 0 || (area2 > 0 ? 1 : -1) != front_sign) return;
  }
  const int minx = min(a.xi, min(b.xi, c.xi)), maxx = max(a.xi, max(b.xi, c.xi));
  const int miny = min(a.yi, min(b.yi, c.yi)), maxy = max(a.yi, max(b.yi, c.yi));
  const int j0 = max((minx + 127) >> 8, tx0), j1 = min((maxx - 128) >> 8, tx0 + TILE - 1);
  const int r0 = max((miny + 127) >> 8, ty0), r1 = min((maxy - 128) >> 8, ty0 + TILE - 1);
  if (j0 > j1 || r0 > r1) return;
  if (tri_small(a.xi, a.yi, b.xi, b.yi, c.xi, c.yi)) {
    TriSetup32 t;
    if (!tri_setup32(a.xi, a.yi, b.xi, b.yi, c.xi, c.yi, t)) return;
    // Incremental form of tri_cover32: the three edge functions, each biased by its tie flag (an integer e passes
    // the top-left rule iff e + tie > 0), stepped by one pixel = 256 sub-pixel units.  Same integers, same coverage;
    // ~10 instructions per tested pixel centre instead of ~35.
    const int dx0 = t.bx - t.ax, dy0 = t.by - t.ay;
    const int tie0 = (dy0 > 0 || (dy0 == 0 && dx0 > 0)) ? 1 : 0;
    const int tie1 = (-t.by > 0 || (t.by == 0 && -t.bx > 0)) ? 1 : 0;
    const int tie2 = (t.ay > 0 || (t.ay == 0 && t.ax > 0)) ? 1 : 0;
    const int qx0 = j0 * 256 + 128 - t.x0, qy0 = r0 * 256 + 128 - t.y0;
    int E0r = dx0 * (qy0 - t.ay) - dy0 * (qx0 - t.ax) + tie0;
    int E1r = (-t.bx) * (qy0 - t.by) + t.by * (qx0 - t.bx) + tie1;
    const int sum = t.area2 + tie0 + tie1 + tie2;
    const int sx0 = -dy0 * 256, sy0 = dx0 * 256, sx1 = t.by * 256, sy1 = -t.bx * 256;
    const float fa = __int2float_rn(t.area2);
    for (int r = r0; r <= r1; ++r, E0r += sy0, E1r += sy1) {
      int E0 = E0r, E1 = E1r;
      for (int j = j0; j <= j1; ++j, E0 += sx0, E1 += sx1) {
        if (min(min(E0, E1), sum - E0 - E1) <= 0) continue;
        const int e0 = E0 - tie0, e1 = E1 - tie1, e2 = t.area2 - e0 - e1;
        const float b0 = __fdiv_rn(__int2float_rn(e0), fa);
        const float w1 = __fdiv_rn(__int2float_rn(e1), fa);
        const float w2 = __fdiv_rn(__int2float_rn(e2), fa);
        const float iz = inv_depth(b0, t.swapped ? w2 : w1, t.swapped ? w1 : w2, a.iz, b.iz, c.iz);
        if (!(iz > iz_far)) continue;
        atomicMax(&zt[(r - ty0) * TILE + (j - tx0)], depth_key(iz, face));
        ++n_frag;
      }
    }
  } else {
    TriSetup t;
    if (!tri_setup(a.xi, a.yi, b.xi, b.yi, c.xi, c.yi, t)) return;
    for (int r = r0; r <= r1; ++r)
      for (int j = j0; j <= j1; ++j) {
        float b0, b1, b2;
        if (!tri_cover(t, j * 256 + 128, r * 256 + 128, b0, b1, b2)) continue;
        const float iz = inv_depth(b0, b1, b2, a.iz, b.iz, c.iz);
        if (!(iz > iz_far)) continue;
        atomicMax(&zt[(r - ty0) * TILE + (j - tx0)], depth_key(iz, face));
        ++n_frag;
      }
  }
}

__device__ __forceinline__ float pixel_ray(float idx_plus_half, float origin, float rscale, float c, float f) {
  // raster pixel centre -> image coordinate -> normalised camera ray component
  const float u = __fadd_rn(origin, __fdiv_rn(idx_plus_half, rscale));
  return __fdiv_rn(__fsub_rn(u, c), f);
}

}  // namespace fp
