// fp_crop.cu — tiled "pose -> 160x160 network inputs" producer.  ONE kernel; one CTA per (pose hypothesis, TILE x TILE
// pixel tile of the crop; TILE = 80 / 32 / 16 by batch size); nothing full-frame, nothing fp32 and no intermediate of
// any kind is materialised in HBM.  Each hypothesis renders the mesh of its own slot of the context's mesh table
// (CropParams::mesh_of), and optionally takes its frame from its own entry of a camera table (CropParams::cams,
// camera_of), so one launch can crop several objects seen by several cameras:
//   1. crop window from the pose                         (Utils.py:577-621 compute_crop_window_tf_batch, 'box_3d')
//   2. binning: every MESHLET of the mesh (<= 64 triangles, fp_meshlet.cu) is tested against the tile with its
//      bounding sphere and — closed meshes — its normal cone; survivors go to a shared-memory list
//   3. raster: each warp takes meshlets off the list, transforms their <= 64 vertices into shared memory, sets up
//      their triangles from there (two per lane) and depth-tests the covered pixels into a SHARED-MEMORY z-tile
//      (TILE x TILE 64-bit keys: interpolated 1/Z | ~face id, one atomicMax per fragment)
//                                                          (Utils.py:133-219 nvdiffrast_render with bbox2d: dr.rasterize)
//   4. shade: warps resolve 8 x 4-pixel blocks of the tile: perspective-correct attributes of the winning triangle,
//      bilinear wrap texture, Lambert term (dr.interpolate / dr.texture, Utils.py:183-215), the observed frame resampled
//      into the same window (predict_pose_refine.py:63,72 / predict_score.py:89-90 kornia warp_perspective;
//      h5_dataset.py:158-161 depth round trip for the scorer), normalisation of both (h5_dataset.py:79-127, :137-179)
//   5. one coalesced 16-byte store per crop pixel: the fp16 8-channel images with the 3-pixel zero border and the
//      even/odd column split the 7x7 stem convolution reads (fp_stem.cu, LK_CONV7_S2).
//
// Integer / fp32 load-store work (no tensor cores).  Coverage rule: vertices snapped to 1/256 pixel, exact integer edge
// functions with a top-left tie rule (watertight), depth test on the interpolated 1/Z (largest wins, ties -> lowest
// original face id).  Triangles crossing the near plane (Utils.py:161 znear = 0.001) are not dropped: they take a
// homogeneous (clip-space) path — nvdiffrast computes its barycentrics in clip space — with the depth range test
// znear < Z < zfar per pixel.
#include "fp_crop.cuh"

#include <stdlib.h>

#include "fp_common.cuh"
#include "fp_gemm.cuh"
#include "fp_raster.cuh"

namespace fp {

constexpr int S = 160;    // crop size (cfg.input_resize)
// Tile edge in pixels = template parameter TILE of the kernel: 80 (4 CTAs per hypothesis) for large batches — every
// meshlet is set up by ~1.35 tiles instead of ~2 and the per-CTA prologue (window, tables, binning) is paid 4x, not 25x —
// 32 for mid-size batches and 16 (100 CTAs per hypothesis) for track_one's single pose, where latency is what counts.
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kListCap = 1024;  // meshlet list entries per binning round
#ifndef FP_CROP_MIN_CTAS
#define FP_CROP_MIN_CTAS 3  // resident CTAs per SM the register allocation aims for (85 registers / thread)
#endif

// Utils.py:602-621 + :584-598, fp32 with the reference's operation order (no FMA contraction so the rounded window
// edges are reproducible bit-for-bit by the oracle).  Called by lanes 0..4 of one warp: lane k projects point k.
__device__ __forceinline__ void crop_window_warp(const float* __restrict__ pose, float fx, float fy, float cx, float cy,
                                                 float r3, int lane, Window& w) {
  const float tx = pose[3], ty = pose[7], tz = pose[11];
  const int k = lane < 5 ? lane : 0;
  const float ox = (k == 1) ? r3 : (k == 2 ? -r3 : 0.f);
  const float oy = (k == 3) ? r3 : (k == 4 ? -r3 : 0.f);
  const float px = __fadd_rn(tx, ox), py = __fadd_rn(ty, oy), pz = tz;
  const float x = __fadd_rn(__fmul_rn(fx, px), __fmul_rn(cx, pz));
  const float y = __fadd_rn(__fmul_rn(fy, py), __fmul_rn(cy, pz));
  const float u = __fdiv_rn(x, pz), v = __fdiv_rn(y, pz);
  const float u0 = __shfl_sync(0xffffffffu, u, 0), v0 = __shfl_sync(0xffffffffu, v, 0);
  float radius = fmaxf(fabsf(__fsub_rn(u, u0)), fabsf(__fsub_rn(v, v0)));
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) radius = fmaxf(radius, __shfl_xor_sync(0xffffffffu, radius, o));
  radius = __shfl_sync(0xffffffffu, radius, 0);  // lanes 0..7 hold max over lanes 0..7 (lanes 5..7 duplicate point 0)
  const float left = rintf(__fsub_rn(u0, radius)), right = rintf(__fadd_rn(u0, radius));
  const float top = rintf(__fsub_rn(v0, radius)), bottom = rintf(__fadd_rn(v0, radius));
  w.left = left;
  w.top = top;
  // Utils.py:594-595 `out_size[0] / (right - left)` is int / Tensor = Tensor.__rtruediv__ = reciprocal() * 160 in
  // torch: two roundings, not one division (tests/golden/geometry_golden.npz pins the bits)
  w.sx = __fmul_rn(__frcp_rn(__fsub_rn(right, left)), (float)S);
  w.sy = __fmul_rn(__frcp_rn(__fsub_rn(bottom, top)), (float)S);
  // predict_pose_refine.py:44-45: render window = crop corners (0,0)-(159,159) mapped back to the image
  w.umin = left;
  w.vmin = top;
  const float umax = __fadd_rn(left, __fdiv_rn(159.f, w.sx));
  const float vmax = __fadd_rn(top, __fdiv_rn(159.f, w.sy));
  w.rsx = __fdiv_rn((float)S, __fsub_rn(umax, w.umin));
  w.rsy = __fdiv_rn((float)S, __fsub_rn(vmax, w.vmin));
}

// kornia.warp_perspective(..., align_corners=False) coordinate chain (SURVEY.md §8c K1): destination
// pixel index d, affine map x = d * inv_scale + offset into a source of `size` pixels, then the
// (size-1)-normalisation followed by grid_sample's align_corners=False un-normalisation.
__device__ __forceinline__ float kornia_src_coord(float x_src, int size) {
  const float xn = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, x_src), (float)(size - 1)), 1.f);
  return __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(xn, 1.f), (float)size), 1.f), 0.5f);
}

__device__ __forceinline__ void normalise_xyz(float x, float y, float z, const float* t, float inv_radius, float tau,
                                              float& ox, float& oy, float& oz) {
  // h5_dataset.py:93-99 / :151-156
  const bool inv = z < tau;
  ox = (x - t[0]) * inv_radius;
  oy = (y - t[1]) * inv_radius;
  oz = (z - t[2]) * inv_radius;
  if (inv || fabsf(ox) >= 2.f) ox = 0.f;
  if (inv || fabsf(oy) >= 2.f) oy = 0.f;
  if (inv || fabsf(oz) >= 2.f) oz = 0.f;
}

template <int TILE>
struct TileSmem {
  unsigned long long zt[TILE * TILE];  // depth keys of the tile (0 = empty)
  VtxS sv[kWarps][kMeshletVerts];      // per-warp transformed vertices of the meshlet in flight
  float P[16];
  Window win;
  float colf[TILE], rowf[TILE];  // bilinear weight of the right / lower tap of the observed-crop resampling (separable)
  int colx[TILE], rowy[TILE];    // right / lower tap index; bit 30 / 31 set when the left (upper) / right (lower) tap is outside
  int coln[TILE], rown[TILE];    // nearest source column / row (-1 = outside)
  int colz[TILE], rowz[TILE];    // scorer depth round trip: source column / row of the depth sample
  int list[kListCap];
  int n_list, next;
  int stat[4];
  MeshSlotDev slot;  // mesh table entry of this CTA's hypothesis
  CameraDev cam;     // camera table entry of this CTA's hypothesis (kCams)
  int fit[kFitCounts];  // kFit: this CTA's counts (after every member the other instantiations read)
};
static_assert(sizeof(MeshSlotDev) % 16 == 0 && sizeof(MeshSlotDev) / 16 <= 32, "table entry copied as uint4s by warp 0");

// kCams: the frame comes from the camera table entry of the hypothesis (p.cams[p.camera_of[n]], copied to shared memory
// next to the mesh entry) instead of the by-value p.frame.  A template flag rather than a branch, so that the
// single-camera instantiations carry no camera-table code.
// FRAME(f): field f of the frame this hypothesis is cropped from, read where it is used
#define FRAME(f) (kCams ? sm.cam.f : p.frame.f)
// kVis: also write the fp32 record of every crop pixel to p.vis (fp_vis, the debug canvases).  A template flag for the
// same reason: the instantiations without it compile to the same code as before the record existed.
// kFit (with kCams only, mode 0): the tracking calls' fit pass at the returned poses.  Binning and raster as always;
// the shade loop takes only the rendered camera z of the winning triangle (the Z the A side normalises) and the z of
// the nearest xyz_map sample (what the B side reads at the same crop pixel), and counts, per pixel p with d = z_o - z_r:
// covered, valid (covered and z_o >= 0.001), inlier (valid, |d| <= delta), occluded (valid, d < -delta) and behind
// (valid, d > delta).  Per lane, per warp (__reduce_add_sync), per CTA in shared memory, one atomicAdd per counter per
// CTA: integer counts, independent of the tile size and of the order of CTAs, hypotheses and cameras.  Nothing is
// stored but the counts.  The A and B windows differ by the 159/160 scale of SURVEY F5; like the refiner, the counts
// compare the same crop pixel on both sides.
template <int TILE, bool kStats, bool kCams, bool kVis, bool kFit>
__global__ void __launch_bounds__(kThreads, FP_CROP_MIN_CTAS) crop_tile_kernel(const CropParams p) {
  constexpr int TPR = S / TILE;
  extern __shared__ __align__(16) unsigned char crop_smem_raw[];
  TileSmem<TILE>& sm = *reinterpret_cast<TileSmem<TILE>*>(crop_smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n = blockIdx.y;
  const int tile = blockIdx.x;
  const int ty0 = (tile / TPR) * TILE, tx0 = (tile % TPR) * TILE;
  const MeshDev& M = sm.slot.mesh;

  for (int i = tid; i < TILE * TILE; i += kThreads) sm.zt[i] = 0ull;
  if (tid == 0) {
    sm.n_list = 0;
    sm.next = 0;
    sm.stat[0] = sm.stat[1] = sm.stat[2] = sm.stat[3] = 0;
  }
  if (kFit && tid < kFitCounts) sm.fit[tid] = 0;
  // The mesh table, the camera table and the slot and camera ids are written by copies that precede the whole launch
  // sequence, never by a kernel of it: they may be read before the programmatic-dependency wait.  The pixels the camera
  // entry points to come from frame_prep_kernel of the same sequence and are only read after it.
  if (tid < (int)(sizeof(MeshSlotDev) / 16)) {
    const int s = p.mesh_of ? __ldg(p.mesh_of + n) : 0;
    reinterpret_cast<uint4*>(&sm.slot)[tid] = __ldg(reinterpret_cast<const uint4*>(p.slots + s) + tid);
  }
  if (kCams && tid >= 32 && tid < 32 + (int)(sizeof(CameraDev) / 16)) {
    const int cam = __ldg(p.camera_of + n);
    reinterpret_cast<uint4*>(&sm.cam)[tid - 32] = __ldg(reinterpret_cast<const uint4*>(p.cams + cam) + tid - 32);
  }
  pdl_trigger();
  pdl_wait();  // the poses come from the previous iteration's pose update; the crop buffer is read by its stem conv
  if (tid < 16) sm.P[tid] = p.poses[(size_t)n * 16 + tid];
  __syncthreads();
  if (warp == 0) {
    Window w;
    crop_window_warp(sm.P, FRAME(fx), FRAME(fy), FRAME(cx), FRAME(cy), sm.slot.r3[p.mode ? 1 : 0], lane, w);
    if (lane == 0) {
      sm.win = w;
      if (p.win_out && tile == 0) {
        p.win_out[n * 4 + 0] = w.left;
        p.win_out[n * 4 + 1] = w.top;
        p.win_out[n * 4 + 2] = w.sx;
        p.win_out[n * 4 + 3] = w.sy;
      }
    }
  }
  __syncthreads();
  const Window W = sm.win;

  // ---- per-axis tables of the observed-crop resampling for this tile's 32 columns and 32 rows
  static_assert(2 * TILE <= kThreads, "one thread per table entry");
  if (tid < 2 * TILE) {
    const bool is_row = tid >= TILE;
    const int k = is_row ? tid - TILE : tid;
    const int d = (is_row ? ty0 : tx0) + k;
    const float sc = is_row ? W.sy : W.sx, org = is_row ? W.top : W.left;
    const int size = is_row ? FRAME(H) : FRAME(W);
    const float xs = __fadd_rn(__fdiv_rn((float)d, sc), org);
    const float ix = kornia_src_coord(xs, size);
    int un = (int)rintf(ix);
    if (un < 0 || un >= size) un = -1;
    int uz = -1;
    if (un >= 0) {
      // scorer: depth crop -> full-res (nearest) -> back-project -> crop (nearest), h5_dataset.py:158-161
      const float xc = __fadd_rn(__fmul_rn(sc, (float)un), __fmul_rn(-org, sc));
      const int jc = (int)rintf(kornia_src_coord(xc, S));
      if (jc >= 0 && jc < S) {
        const float xs2 = __fadd_rn(__fdiv_rn((float)jc, sc), org);
        const int u2 = (int)rintf(kornia_src_coord(xs2, size));
        if (u2 >= 0 && u2 < size) uz = u2;
      }
    }
    {
      // bilinear taps (zeros padding): index of the first tap, weight of the second, out-of-range flags
      const float f0 = floorf(ix);
      const int i0 = (int)fminf(fmaxf(f0, -2.f), (float)size);
      const unsigned out0 = (i0 < 0 || i0 >= size) ? 0x40000000u : 0u;
      const unsigned out1 = (i0 + 1 < 0 || i0 + 1 >= size) ? 0x80000000u : 0u;
      (is_row ? sm.rowf : sm.colf)[k] = ix - f0;
      // stored index = the SECOND tap, clamped into the image; the first tap is one before it (or the same pixel
      // when the second one fell off the far edge)
      (is_row ? sm.rowy : sm.colx)[k] = (int)((unsigned)(max(min(i0 + 1, size - 1), 0)) | out0 | out1);
    }
    (is_row ? sm.rown : sm.coln)[k] = un;
    (is_row ? sm.rowz : sm.colz)[k] = uz;
  }

  // camera position in object space (for the normal cones): o = -R^T t
  const float ox = -(sm.P[0] * sm.P[3] + sm.P[4] * sm.P[7] + sm.P[8] * sm.P[11]);
  const float oy = -(sm.P[1] * sm.P[3] + sm.P[5] * sm.P[7] + sm.P[9] * sm.P[11]);
  const float oz = -(sm.P[2] * sm.P[3] + sm.P[6] * sm.P[7] + sm.P[10] * sm.P[11]);
  const float iz_far = 1.f / p.zfar;
  int n_vis = 0, n_tri = 0, n_frag = 0, n_mixed = 0;
  // back faces may only be skipped when the near plane clips nothing of the solid: a front face cut away by it uncovers
  // the back faces behind it.  Bounding sphere, conservative; it also rules out a camera centre inside the solid.
  int front_sign = M.front_sign;
  if (sm.P[8] * M.bs_x + sm.P[9] * M.bs_y + sm.P[10] * M.bs_z + sm.P[11] - M.bs_r <= p.znear) front_sign = 0;

  for (int base = 0; base < M.n_meshlets; base += kListCap) {
    // ---- binning: meshlet bounding sphere vs this tile, normal cone vs the camera
    const int lim = min(M.n_meshlets, base + kListCap);
    for (int m = base + tid; m < lim; m += kThreads) {
      const float4 sph = __ldg(reinterpret_cast<const float4*>(M.meshlets + m));
      const float X = sm.P[0] * sph.x + sm.P[1] * sph.y + sm.P[2] * sph.z + sm.P[3];
      const float Y = sm.P[4] * sph.x + sm.P[5] * sph.y + sm.P[6] * sph.z + sm.P[7];
      const float Z = sm.P[8] * sph.x + sm.P[9] * sph.y + sm.P[10] * sph.z + sm.P[11];
      const float r = sph.w;
      bool keep = true;
      if (Z + r <= p.znear) {
        keep = false;  // entirely behind the near plane
      } else if (Z - r > p.znear) {
        // |delta u| <= fx r (1 + |X| / Z) / (Z - r) for any point of the sphere; crop raster pixels; 1 px of slack
        const float izc = 1.f / Z, izn = 1.f / (Z - r);
        const float pu = (FRAME(fx) * X * izc + FRAME(cx) - W.umin) * W.rsx;
        const float pv = (FRAME(fy) * Y * izc + FRAME(cy) - W.vmin) * W.rsy;
        const float ru = FRAME(fx) * W.rsx * r * (1.f + fabsf(X) * izc) * izn + 1.f;
        const float rv = FRAME(fy) * W.rsy * r * (1.f + fabsf(Y) * izc) * izn + 1.f;
        keep = pu + ru >= (float)tx0 && pu - ru <= (float)(tx0 + TILE) && pv + rv >= (float)ty0 &&
               pv - rv <= (float)(ty0 + TILE);
      }
      if (keep && front_sign != 0) {
        const float4 cone = __ldg(reinterpret_cast<const float4*>(M.meshlets + m) + 1);
        if (cone.w >= 0.f) {
          // every face normal n_f has dot(axis, n_f) >= cutoff; the meshlet is entirely back-facing if
          // max over the cone and the sphere of dot(n, cam - p) < 0:  d cos(theta - alpha) + r < 0
          const float vx = ox - sph.x, vy = oy - sph.y, vz = oz - sph.z;
          const float d = sqrtf(vx * vx + vy * vy + vz * vz);
          if (d > r) {
            // cone of the OUTWARD normals: for an inside-out mesh (front_sign = +1) the stored face normals point inwards
            const float ct = fminf(fmaxf((float)(-front_sign) * (cone.x * vx + cone.y * vy + cone.z * vz) / d, -1.f), 1.f);
            const float st = sqrtf(fmaxf(1.f - ct * ct, 0.f));
            const float ca = fminf(cone.w, 1.f), sa = sqrtf(fmaxf(1.f - ca * ca, 0.f));
            // 0.03 of slack on the cosine: snapping to 1/256 px may flip triangles within ~1 degree of edge-on
            if (ct * ca + st * sa < -r / d - 0.03f) keep = false;
          }
        }
      }
      if (keep) sm.list[atomicAdd(&sm.n_list, 1)] = m;
    }
    __syncthreads();
    const int n_list = sm.n_list;

    // ---- raster: warps pull meshlets off the list
    VtxS* sv = sm.sv[warp];
    for (;;) {
      int li = 0;
      if (lane == 0) li = atomicAdd(&sm.next, 1);
      li = __shfl_sync(0xffffffffu, li, 0);
      if (li >= n_list) break;
      const int m = sm.list[li];
      const int4 hdr = __ldg(reinterpret_cast<const int4*>(M.meshlets + m) + 2);  // vert_off, n_verts, tri_off, n_tris
      ++n_vis;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int s = lane + 32 * h;
        if (s < hdr.y) {
          const int gid = __ldg(M.ml_verts + hdr.x + s);
          const float4 q = __ldg(M.vpos + gid);
          VtxScreen o;
          xform_vertex(sm.P, q.x, q.y, q.z, W, FRAME(fx), FRAME(fy), FRAME(cx), FRAME(cy), o);
          VtxS v;
          v.xi = o.xi; v.yi = o.yi; v.iz = o.iz; v.Z = o.Z;
          sv[s] = v;
        }
      }
      __syncwarp();
      unsigned mixed_mask[2] = {0u, 0u};
      uint2 trec[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int t = lane + 32 * h;
        bool mixed = false;
        if (t < hdr.w) {
          trec[h] = __ldg(M.ml_tris + hdr.z + t);
          const VtxS a = sv[trec[h].x & 255], b = sv[(trec[h].x >> 8) & 255], c = sv[(trec[h].x >> 16) & 255];
          const int nfront = (a.Z > p.znear) + (b.Z > p.znear) + (c.Z > p.znear);
          if (nfront == 3) {
            ++n_tri;
            raster_tri<TILE>(a, b, c, trec[h].y, front_sign, tx0, ty0, iz_far, sm.zt, n_frag);
          } else if (nfront > 0) {
            mixed = true;
          }
        }
        mixed_mask[h] = __ballot_sync(0xffffffffu, mixed);
      }
      // triangles crossing the near plane (rare): the whole warp scans the tile for one such triangle at a time
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        unsigned mm = mixed_mask[h];
        while (mm) {
          const int src = __ffs(mm) - 1;
          mm &= mm - 1;
          ++n_mixed;
          const unsigned packed = __shfl_sync(0xffffffffu, trec[h].x, src);
          const unsigned face = __shfl_sync(0xffffffffu, trec[h].y, src);
          float Pc[3][3];
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const int gid = __ldg(M.ml_verts + hdr.x + ((packed >> (8 * k)) & 255));
            const float4 q = __ldg(M.vpos + gid);
            VtxScreen o;
            xform_vertex(sm.P, q.x, q.y, q.z, W, FRAME(fx), FRAME(fy), FRAME(cx), FRAME(cy), o);
            Pc[k][0] = o.X; Pc[k][1] = o.Y; Pc[k][2] = o.Z;
          }
          HomTri ht;
          hom_setup(Pc[0], Pc[1], Pc[2], ht);
          for (int px = lane; px < TILE * TILE; px += 32) {
            const int r = px / TILE, jl = px - r * TILE;
            const float dx = pixel_ray((float)(tx0 + jl) + 0.5f, W.umin, W.rsx, FRAME(cx), FRAME(fx));
            const float dy = pixel_ray((float)(ty0 + r) + 0.5f, W.vmin, W.rsy, FRAME(cy), FRAME(fy));
            float l0, l1, l2, iz;
            if (hom_cover(ht, dx, dy, p.znear, p.zfar, l0, l1, l2, iz)) {
              atomicMax(&sm.zt[px], depth_key(iz, face));
              ++n_frag;
            }
          }
        }
      }
      __syncwarp();
    }
    __syncthreads();
    if (tid == 0) {
      sm.n_list = 0;
      sm.next = 0;
    }
    __syncthreads();
  }
  if (kStats && p.stats) {
    atomicAdd(&sm.stat[0], lane == 0 ? n_vis : 0);
    atomicAdd(&sm.stat[1], n_tri);
    atomicAdd(&sm.stat[2], n_frag);
    atomicAdd(&sm.stat[3], lane == 0 ? n_mixed : 0);
    __syncthreads();
    if (tid < 4) atomicAdd(p.stats + tid, sm.stat[tid]);
  }

  // ---- shade: a warp resolves 8 x 4-pixel blocks (coverage is coherent in 2-D: fewer warps straddle the silhouette
  // than with 32 x 1 rows, and those are the ones that pay for both the covered and the background path)
  const float inv_radius = sm.slot.inv_radius;
  const float tvec[3] = {sm.P[3], sm.P[7], sm.P[11]};
  const float tau = p.mode == 0 ? 0.001f : 0.1f;
  const size_t img_stride = (size_t)(S + 6) * (S + 8) * 8;
  __half* outA = p.crops + (size_t)n * img_stride;
  __half* outB = p.crops + (size_t)(p.b_img0 + n) * img_stride;
  constexpr int kBlocksX = TILE / 8, kBlocks = kBlocksX * (TILE / 4);
  float delta = 0.f;  // kFit: the threshold, written with the slot and camera ids (readable before the wait)
  int fit_n[kFitCounts] = {0, 0, 0, 0, 0};  // kFit: this lane's counts
  if constexpr (kFit) delta = __ldg(p.fit_delta);
#pragma unroll 1
  for (int blk = warp; blk < kBlocks; blk += kWarps) {
    const int jl = (blk % kBlocksX) * 8 + (lane & 7), rl = (blk / kBlocksX) * 4 + (lane >> 3);
    const int j = tx0 + jl, r = ty0 + rl;
    const float wx1 = sm.colf[jl];
    const int cxi = sm.colx[jl];
    const int unc = sm.coln[jl], uzc = sm.colz[jl];
    // ---- A: rendered crop
    float ar = 0.f, ag = 0.f, ab = 0.f, ax = 0.f, ay = 0.f, az = 0.f;
    float za = 0.f;  // kVis, kFit: rendered camera z
    const unsigned long long key = sm.zt[rl * TILE + jl];
    if (key != 0ull) {
      const int f = (int)(0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFull));
      const int4 fi = __ldg(M.faces + f);
      const int vid[3] = {fi.x, fi.y, fi.z};
      VtxScreen vs[3];
      float dif[3];
      float4 att[3];
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const float4 pp = __ldg(M.vpos + vid[q]);
        if constexpr (kFit) {
          xform_vertex(sm.P, pp.x, pp.y, pp.z, W, FRAME(fx), FRAME(fy), FRAME(cx), FRAME(cy), vs[q]);
        } else {
          const float4 nn = __ldg(M.vnrm + vid[q]);
          att[q] = __ldg(M.vatt + vid[q]);
          xform_vertex(sm.P, pp.x, pp.y, pp.z, W, FRAME(fx), FRAME(fy), FRAME(cx), FRAME(cy), vs[q]);
          // diffuse = clip(normalize(R n) . (0,0,-1), 0, 1)   (Utils.py:203-207)
          const float cxn = sm.P[0] * nn.x + sm.P[1] * nn.y + sm.P[2] * nn.z;
          const float cyn = sm.P[4] * nn.x + sm.P[5] * nn.y + sm.P[6] * nn.z;
          const float czn = sm.P[8] * nn.x + sm.P[9] * nn.y + sm.P[10] * nn.z;
          const float len = fmaxf(sqrtf(cxn * cxn + cyn * cyn + czn * czn), 1e-12f);
          dif[q] = fminf(fmaxf(-czn / len, 0.f), 1.f);
        }
      }
      float w0, w1, w2;  // perspective-correct weights (nvdiffrast: barycentrics computed in clip space)
      if (vs[0].Z > p.znear && vs[1].Z > p.znear && vs[2].Z > p.znear) {
        float b0 = 0.f, b1 = 0.f, b2 = 0.f;
        if (tri_small(vs[0].xi, vs[0].yi, vs[1].xi, vs[1].yi, vs[2].xi, vs[2].yi)) {
          TriSetup32 t;
          tri_setup32(vs[0].xi, vs[0].yi, vs[1].xi, vs[1].yi, vs[2].xi, vs[2].yi, t);
          tri_cover32(t, j * 256 + 128, r * 256 + 128, b0, b1, b2);
        } else {
          TriSetup t;
          tri_setup(vs[0].xi, vs[0].yi, vs[1].xi, vs[1].yi, vs[2].xi, vs[2].yi, t);
          tri_cover(t, j * 256 + 128, r * 256 + 128, b0, b1, b2);
        }
        const float iz = inv_depth(b0, b1, b2, vs[0].iz, vs[1].iz, vs[2].iz);
        const float z = 1.f / iz;
        w0 = b0 * vs[0].iz * z;
        w1 = b1 * vs[1].iz * z;
        w2 = b2 * vs[2].iz * z;
      } else {
        const float A3[3] = {vs[0].X, vs[0].Y, vs[0].Z}, B3[3] = {vs[1].X, vs[1].Y, vs[1].Z}, C3[3] = {vs[2].X, vs[2].Y, vs[2].Z};
        HomTri ht;
        hom_setup(A3, B3, C3, ht);
        const float dx = pixel_ray((float)j + 0.5f, W.umin, W.rsx, FRAME(cx), FRAME(fx));
        const float dy = pixel_ray((float)r + 0.5f, W.vmin, W.rsy, FRAME(cy), FRAME(fy));
        float iz;
        w0 = w1 = w2 = 0.f;
        hom_cover(ht, dx, dy, p.znear, p.zfar, w0, w1, w2, iz);
      }
      const float X = w0 * vs[0].X + w1 * vs[1].X + w2 * vs[2].X;
      const float Y = w0 * vs[0].Y + w1 * vs[1].Y + w2 * vs[2].Y;
      const float Z = w0 * vs[0].Z + w1 * vs[1].Z + w2 * vs[2].Z;
      if constexpr (kFit) {
        za = Z;
      } else {
        const float diffuse = w0 * dif[0] + w1 * dif[1] + w2 * dif[2];
        float cr, cg, cb;
        if (sm.slot.has_tex) {
          const int Ht = sm.slot.Ht, Wt = sm.slot.Wt;
          const uchar4* tex = sm.slot.tex;
          const float tu = w0 * att[0].x + w1 * att[1].x + w2 * att[2].x;
          const float tv = w0 * att[0].y + w1 * att[1].y + w2 * att[2].y;
          // dr.texture(filter_mode='linear', boundary 'wrap'): texel centres at +0.5.  Interpolated uv of a mesh lie in
          // (-1, 2): the wrap is two conditional adds; anything further out takes the general modulo.
          const float xx = tu * Wt - 0.5f, yy = tv * Ht - 0.5f;
          const float xf = floorf(xx), yf = floorf(yy);
          const float ax1 = xx - xf, ay1 = yy - yf;
          int x0 = (int)xf, y0 = (int)yf;
          if ((unsigned)(x0 + Wt) >= (unsigned)(3 * Wt)) x0 %= Wt;
          if ((unsigned)(y0 + Ht) >= (unsigned)(3 * Ht)) y0 %= Ht;
          if (x0 < 0) x0 += Wt;
          if (y0 < 0) y0 += Ht;
          if (x0 >= Wt) x0 -= Wt;
          if (y0 >= Ht) y0 -= Ht;
          const int x1 = (x0 + 1 == Wt) ? 0 : x0 + 1, y1 = (y0 + 1 == Ht) ? 0 : y0 + 1;
          const uchar4 t00 = __ldg(tex + (size_t)y0 * Wt + x0), t01 = __ldg(tex + (size_t)y0 * Wt + x1);
          const uchar4 t10 = __ldg(tex + (size_t)y1 * Wt + x0), t11 = __ldg(tex + (size_t)y1 * Wt + x1);
          const float w00 = (1.f - ax1) * (1.f - ay1), w01 = ax1 * (1.f - ay1), w10 = (1.f - ax1) * ay1, w11 = ax1 * ay1;
          const float k255 = 1.f / 255.f;
          cr = (w00 * t00.x + w01 * t01.x + w10 * t10.x + w11 * t11.x) * k255;
          cg = (w00 * t00.y + w01 * t01.y + w10 * t10.y + w11 * t11.y) * k255;
          cb = (w00 * t00.z + w01 * t01.z + w10 * t10.z + w11 * t11.z) * k255;
        } else {
          cr = w0 * att[0].x + w1 * att[1].x + w2 * att[2].x;
          cg = w0 * att[0].y + w1 * att[1].y + w2 * att[2].y;
          cb = w0 * att[0].z + w1 * att[1].z + w2 * att[2].z;
        }
        // color*w_ambient + diffuse*color*w_diffuse, clip(0,1)   (Utils.py:211-213)
        ar = fminf(fmaxf(cr * 0.8f + diffuse * cr * 0.5f, 0.f), 1.f);
        ag = fminf(fmaxf(cg * 0.8f + diffuse * cg * 0.5f, 0.f), 1.f);
        ab = fminf(fmaxf(cb * 0.8f + diffuse * cb * 0.5f, 0.f), 1.f);
        normalise_xyz(X, Y, Z, tvec, inv_radius, tau, ax, ay, az);
        if (kVis) za = Z;
      }
    }
    if constexpr (kFit) {
      const int vn = sm.rown[rl];
      float zo = 0.f;  // z of the nearest xyz_map sample: 0 outside the frame and where the filtered depth is invalid
      if (unc >= 0 && vn >= 0) zo = __ldg(reinterpret_cast<const float*>(FRAME(xyz_map) + (size_t)vn * FRAME(W) + unc) + 2);
      const float d = zo - za;
      const bool covered = key != 0ull, valid = covered && zo >= 0.001f;
      fit_n[0] += covered;
      fit_n[1] += valid;
      fit_n[2] += valid && fabsf(d) <= delta;
      fit_n[3] += valid && d < -delta;
      fit_n[4] += valid && d > delta;
      continue;
    }
    // ---- B: observed crop
    float br = 0.f, bg = 0.f, bb = 0.f, bx = 0.f, by = 0.f, bz = 0.f;
    float zb = 0.f;  // kVis: nearest sample of the filtered depth
    {
      // bilinear rgb, zeros padding: tap indices / weights / validity come from the per-axis tables
      const float wy1 = sm.rowf[rl];
      const int ryi = sm.rowy[rl];
      const int x1 = cxi & 0x3fffffff, y1 = ryi & 0x3fffffff;
      const int x0 = (cxi & 0x80000000) ? x1 : max(x1 - 1, 0), y0 = (ryi & 0x80000000) ? y1 : max(y1 - 1, 0);
      const float wx[2] = {(cxi & 0x40000000) ? 0.f : 1.f - wx1, (cxi & 0x80000000) ? 0.f : wx1};
      const float wy[2] = {(ryi & 0x40000000) ? 0.f : 1.f - wy1, (ryi & 0x80000000) ? 0.f : wy1};
      const uchar4* row0 = FRAME(rgb) + (size_t)y0 * FRAME(W);
      const uchar4* row1 = FRAME(rgb) + (size_t)y1 * FRAME(W);
      const uchar4 t00 = __ldg(row0 + x0), t01 = __ldg(row0 + x1), t10 = __ldg(row1 + x0), t11 = __ldg(row1 + x1);
      const float w00 = wx[0] * wy[0], w01 = wx[1] * wy[0], w10 = wx[0] * wy[1], w11 = wx[1] * wy[1];
      br = w00 * t00.x + w01 * t01.x + w10 * t10.x + w11 * t11.x;
      bg = w00 * t00.y + w01 * t01.y + w10 * t10.y + w11 * t11.y;
      bb = w00 * t00.z + w01 * t01.z + w10 * t10.z + w11 * t11.z;
      br *= (1.f / 255.f);
      bg *= (1.f / 255.f);
      bb *= (1.f / 255.f);
      // nearest geometry
      const int vn = sm.rown[rl];
      if (kVis && p.mode == 1 && unc >= 0 && vn >= 0) zb = __ldg(FRAME(depth) + (size_t)vn * FRAME(W) + unc);
      float X = 0.f, Y = 0.f, Z = 0.f;
      if (unc >= 0 && vn >= 0) {
        if (p.mode == 0) {
          // refiner: xyz_map (depth2xyzmap, Utils.py:399-438) sampled nearest
          const float4 q = __ldg(FRAME(xyz_map) + (size_t)vn * FRAME(W) + unc);
          X = q.x;
          Y = q.y;
          Z = q.z;
        } else {
          const int v2 = sm.rowz[rl];
          float zz = 0.f;
          if (uzc >= 0 && v2 >= 0) zz = __ldg(FRAME(depth) + (size_t)v2 * FRAME(W) + uzc);
          if (zz >= 0.001f) {  // depth2xyzmap_batch(zfar=inf): invalid z<0.001 -> 0
            X = ((float)unc - FRAME(cx)) * zz / FRAME(fx);
            Y = ((float)vn - FRAME(cy)) * zz / FRAME(fy);
            Z = zz;
          }
        }
      }
      normalise_xyz(X, Y, Z, tvec, inv_radius, tau, bx, by, bz);
    }
    // even / odd padded columns live in separate half-rows ("EO" layout, fp_stem.cu): pixel (row, col) ->
    // [row][col & 1][col >> 1][8]; a warp (8 columns x 4 rows) writes two 64-byte runs per row and image
    const int pc = j + 3;
    const size_t off = (((size_t)(r + 3) * 2 + (pc & 1)) * ((S + 8) / 2) + (pc >> 1)) * 8;
    *reinterpret_cast<uint4*>(outA + off) = make_uint4(pack_half2(ar, ag), pack_half2(ab, ax), pack_half2(ay, az), 0u);
    *reinterpret_cast<uint4*>(outB + off) = make_uint4(pack_half2(br, bg), pack_half2(bb, bx), pack_half2(by, bz), 0u);
    if (p.dbg) {
      const int pix = r * S + j;
      float* d = p.dbg + (((size_t)n * 2 + 0) * S * S + pix) * 6;
      d[0] = ar; d[1] = ag; d[2] = ab; d[3] = ax; d[4] = ay; d[5] = az;
      d = p.dbg + (((size_t)n * 2 + 1) * S * S + pix) * 6;
      d[0] = br; d[1] = bg; d[2] = bb; d[3] = bx; d[4] = by; d[5] = bz;
    }
    if (kVis) {
      float4* v = p.vis + (size_t)n * 2 * S * S + r * S + j;
      v[0] = make_float4(ar, ag, ab, p.mode == 0 ? az : za);
      v[S * S] = make_float4(br, bg, bb, p.mode == 0 ? bz : zb);
    }
  }
  if constexpr (kFit) {
#pragma unroll
    for (int k = 0; k < kFitCounts; ++k) {
      const int w = __reduce_add_sync(0xffffffffu, fit_n[k]);
      if (lane == 0 && w) atomicAdd(&sm.fit[k], w);
    }
    __syncthreads();
    if (tid < kFitCounts && sm.fit[tid]) atomicAdd(p.fit + (size_t)n * kFitCounts + tid, sm.fit[tid]);
  }
}

#undef FRAME

static int g_crop_tile_override = [] {
  const char* e = getenv("FPOSE_CROP_TILE");  // 16 / 32 / 80: force one tile size (A/B measurements)
  const int v = e ? atoi(e) : 0;
  return (v == 16 || v == 32 || v == 80) ? v : 0;
}();

template <int TILE>
static int launch_tile(const CropParams& p, cudaStream_t stream) {
  constexpr int TPR = S / TILE;
  const size_t smem = sizeof(TileSmem<TILE>);
  static std::atomic<unsigned long long> attr_mask{0};  // per device
  if (!device_bit_test(attr_mask)) {
    FP_CUDA_OK(cudaFuncSetAttribute(crop_tile_kernel<TILE, false, false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    FP_CUDA_OK(cudaFuncSetAttribute(crop_tile_kernel<TILE, true, false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    FP_CUDA_OK(cudaFuncSetAttribute(crop_tile_kernel<TILE, false, true, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    FP_CUDA_OK(cudaFuncSetAttribute(crop_tile_kernel<TILE, false, false, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    FP_CUDA_OK(cudaFuncSetAttribute(crop_tile_kernel<TILE, false, true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    device_bit_set(attr_mask);
  }
  const dim3 grid(TPR * TPR, p.N);
  if (p.fit) {
    FP_CUDA_OK(launch_pdl(crop_tile_kernel<TILE, false, true, false, true>, grid, dim3(kThreads), smem, stream, 1, p));
  } else if (p.cams) {
    FP_CUDA_OK(launch_pdl(crop_tile_kernel<TILE, false, true, false, false>, grid, dim3(kThreads), smem, stream, 1, p));
  } else if (p.stats) {
    FP_CUDA_OK(launch_pdl(crop_tile_kernel<TILE, true, false, false, false>, grid, dim3(kThreads), smem, stream, 1, p));
  } else if (p.vis) {
    FP_CUDA_OK(launch_pdl(crop_tile_kernel<TILE, false, false, true, false>, grid, dim3(kThreads), smem, stream, 1, p));
  } else {
    FP_CUDA_OK(launch_pdl(crop_tile_kernel<TILE, false, false, false, false>, grid, dim3(kThreads), smem, stream, 1, p));
  }
  return 0;
}

int crop_launch(const CropParams& p, cudaStream_t stream) {
  if (p.N == 0) return 0;
  FP_REQUIRE(!p.cams == !p.camera_of, "crop_launch: the camera table and the camera ids go together");
  FP_REQUIRE(!(p.cams && p.stats), "crop_launch: work counters are collected on the single-camera path only");
  FP_REQUIRE(!(p.vis && (p.cams || p.stats)), "crop_launch: the vis record is written on the single-camera path only");
  FP_REQUIRE(!p.fit == !p.fit_delta, "crop_launch: the fit counts and their threshold go together");
  FP_REQUIRE(!p.fit || (p.cams && p.mode == 0 && !p.dbg && !p.win_out),
             "crop_launch: the fit pass runs on the camera-table path, in the refiner's window, and writes only its counts");
  // algorithmic bytes: the two 6-channel fp16 crops each hypothesis produces (SURVEY.md §8d); the fit pass stores none
  prof_mark_begin(1, p.fit ? 0.0 : (double)p.N * 2.0 * 6.0 * S * S * 2.0, stream);
  int tile = p.N >= 64 ? 80 : (p.N >= 4 ? 32 : 16);
  if (g_crop_tile_override) tile = g_crop_tile_override;
  if (p.tile_override == 16 || p.tile_override == 32 || p.tile_override == 80) tile = p.tile_override;
  FP_TRY(tile == 80 ? launch_tile<80>(p, stream) : (tile == 32 ? launch_tile<32>(p, stream) : launch_tile<16>(p, stream)));
  prof_mark_end(stream);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// frame preparation: the raw frame (camera format) -> uchar4 and float32 metres, depth -> xyz map (Utils.py:399-438)
// ------------------------------------------------------------------------------------------------
template <bool kDepth>
__global__ void raw_frame_kernel(const CameraDev one, const FrameFmtDev f) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= one.H * one.W) return;
  const int v = i / one.W, u = i - v * one.W;
  one.rgb[i] = raw_rgba_at(one.rgb_raw, f, v, u);
  if (kDepth) one.depth[i] = raw_depth_at(one.depth_raw, f, v, u);
}

__global__ void depth_to_xyz_kernel(const CameraDev one, float zfar) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= one.H * one.W) return;
  const int v = i / one.W, u = i - v * one.W;
  const float z = __ldg(one.depth + i);
  float X = 0.f, Y = 0.f, Z = 0.f;
  if (!(z < 0.001f) && !(z > zfar)) {
    X = ((float)u - one.cx) * z / one.fx;
    Y = ((float)v - one.cy) * z / one.fy;
    Z = z;
  }
  one.xyz_map[i] = make_float4(X, Y, Z, 0.f);
}

int raw_frame_launch(const CameraDev& one, const FrameFmtDev& f, bool depth, cudaStream_t stream) {
  const int npix = one.H * one.W;
  (depth ? raw_frame_kernel<true> : raw_frame_kernel<false>)<<<(npix + 255) / 256, 256, 0, stream>>>(one, f);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

int depth_to_xyz_launch(const CameraDev& one, float zfar, cudaStream_t stream) {
  depth_to_xyz_kernel<<<(one.H * one.W + 255) / 256, 256, 0, stream>>>(one, zfar);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace fp
