// fp_vsd.cu — BOP's visible surface discrepancy (Hodan et al., "On Evaluation of 6D Object Pose Estimation", ECCV
// Workshops 2016; bop_toolkit's pose_error.vsd with visib_mode 'bop19' and cost_type 'step') of N estimated poses E
// against their ground truth G, over a test depth image D.
//
//   vsd_count_kernel   one CTA per (pose, kVsdTile x kVsdTile screen tile of the full frame).  A tile that the projected
//                      bounding sphere of the mesh meets neither under E nor under G leaves at once, so the work scales
//                      with the object's footprint, not with H x W.  A surviving CTA renders E and G into two
//                      shared-memory z-tiles with the crop producer's coverage rule (fp_raster.cuh) on a full-frame
//                      window (umin = vmin = 0, scale 1: pixel (j, r) samples (j + 0.5, r + 0.5)), then every pixel of
//                      the tile reads D, forms the three distances, the two visibility bits and the T step costs, and
//                      the CTA adds union, intersection and c_0 .. c_{T-1} — integers: warp reductions, one shared atomic
//                      per warp, one global atomicAdd per counter per CTA — to the pose's counter row.
//   vsd_finish_kernel  e_t = (c_t + union - intersection) / union in fp64, rounded to fp32; 1 when union = 0.
//
// Depth of a covered pixel = 1 / (interpolated 1/Z of the winning fragment), fp32 (__frcp_rn).  Distances are fp64
// with BOP's integer pixel indices: dist(u, v) = d sqrt(((u - cx) / fx)^2 + ((v - cy) / fy)^2 + 1), with rounded (never
// fused) operations so that a host restatement in float64 gets the same bits.  Integer counts make a pose's errors
// independent of the batch, of n_gt / n_K / n_depth broadcasting and of the order in which CTAs run.  Nothing
// full-frame is written to device memory.
#include <math.h>

#include <vector>

#include "../../include/fpose.h"
#include "fp_common.cuh"
#include "fp_crop.cuh"
#include "fp_raster.cuh"

namespace fp {

constexpr int kVsdTile = 32;
constexpr int kVsdThreads = 256;
constexpr int kVsdWarps = kVsdThreads / 32;
constexpr int kVsdPix = kVsdTile * kVsdTile / kVsdThreads;  // pixels per thread in the evaluation
constexpr int kVsdListCap = 1024;                           // meshlet list entries per binning round
constexpr float kVsdZnear = 0.001f, kVsdZfar = 100.f;       // the crop producer's (Utils.py:161)

struct VsdParams {
  // mesh (device copies of build_mesh_host's records)
  const float4* vpos;
  const Meshlet* meshlets;
  const int* ml_verts;
  const uint2* ml_tris;
  int n_meshlets;
  float4 bs;  // bounding sphere of the whole mesh
  int front_sign;
  // poses and frames
  const float* pred;  // [N][16]
  const float* gt;    // [n_gt][16]
  int gt_stride;      // 0 or 16
  const float* depth;  // [n_depth][H][W]
  size_t depth_stride;  // 0 or H W
  const float* K;      // [n_K][9]
  int k_stride;        // 0 or 9
  int H, W, tiles_x;
  double delta;
  const float* taus;  // [T]
  int T;
  int* counts;  // [N][T + 2]
};

struct VsdSmem {
  unsigned long long zt[2][kVsdTile * kVsdTile];  // depth keys under E and G (0 = not covered)
  VtxS sv[kVsdWarps][kMeshletVerts];
  float P[2][16];
  double tau[FP_VSD_MAX_TAUS];
  int list[kVsdListCap];
  int n_list, next;
  int render[2];
  int cnt[2 + FP_VSD_MAX_TAUS];  // union, intersection, c_0 .. c_{T-1}
};

// May a sphere (object space, centre + radius) under pose P cover a pixel centre of the tile at (tx0, ty0) of the full
// frame?  The crop producer's binning bound on a full-frame window: |delta u| <= fx r (1 + |X| / Z) / (Z - r) for any
// point of the sphere, 1 px of slack; a sphere that reaches the near plane is kept, one behind it is not.
__device__ __forceinline__ bool sphere_meets_tile(const float* P, float4 s, float fx, float fy, float cx, float cy,
                                                  int tx0, int ty0) {
  const float X = P[0] * s.x + P[1] * s.y + P[2] * s.z + P[3];
  const float Y = P[4] * s.x + P[5] * s.y + P[6] * s.z + P[7];
  const float Z = P[8] * s.x + P[9] * s.y + P[10] * s.z + P[11];
  if (Z + s.w <= kVsdZnear) return false;
  if (!(Z - s.w > kVsdZnear)) return true;
  const float izc = 1.f / Z, izn = 1.f / (Z - s.w);
  const float pu = fx * X * izc + cx, pv = fy * Y * izc + cy;
  const float ru = fx * s.w * (1.f + fabsf(X) * izc) * izn + 1.f;
  const float rv = fy * s.w * (1.f + fabsf(Y) * izc) * izn + 1.f;
  return pu + ru >= (float)tx0 && pu - ru <= (float)(tx0 + kVsdTile) && pv + rv >= (float)ty0 &&
         pv - rv <= (float)(ty0 + kVsdTile);
}

// The crop producer's normal-cone test: is every face of the meshlet turned away from the camera centre o?
__device__ __forceinline__ bool cone_back_facing(const Meshlet* __restrict__ ml, float4 sph, int front_sign, float ox,
                                                 float oy, float oz) {
  const float4 cone = __ldg(reinterpret_cast<const float4*>(ml) + 1);
  if (!(cone.w >= 0.f)) return false;
  const float vx = ox - sph.x, vy = oy - sph.y, vz = oz - sph.z;
  const float d = sqrtf(vx * vx + vy * vy + vz * vz);
  if (!(d > sph.w)) return false;
  const float ct = fminf(fmaxf((float)(-front_sign) * (cone.x * vx + cone.y * vy + cone.z * vz) / d, -1.f), 1.f);
  const float st = sqrtf(fmaxf(1.f - ct * ct, 0.f));
  const float ca = fminf(cone.w, 1.f), sa = sqrtf(fmaxf(1.f - ca * ca, 0.f));
  return ct * ca + st * sa < -sph.w / d - 0.03f;
}

// Renders the mesh at pose P into the z-tile zt (zeroed by the caller): the crop producer's binning and raster loops on
// a full-frame window.  Called by the whole CTA.
__device__ __forceinline__ void render_ztile(const VsdParams& p, VsdSmem& sm, const float* P, unsigned long long* zt,
                                             float fx, float fy, float cx, float cy, int tx0, int ty0) {
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  Window win;
  win.left = win.top = win.umin = win.vmin = 0.f;
  win.sx = win.sy = win.rsx = win.rsy = 1.f;
  const float ox = -(P[0] * P[3] + P[4] * P[7] + P[8] * P[11]);
  const float oy = -(P[1] * P[3] + P[5] * P[7] + P[9] * P[11]);
  const float oz = -(P[2] * P[3] + P[6] * P[7] + P[10] * P[11]);
  const float iz_far = 1.f / kVsdZfar;
  int front_sign = p.front_sign;
  {
    // back faces may only be skipped when the camera centre is outside the solid (bounding sphere: conservative)
    const float bx = ox - p.bs.x, by = oy - p.bs.y, bz = oz - p.bs.z;
    if (bx * bx + by * by + bz * bz <= p.bs.w * p.bs.w) front_sign = 0;
  }
  int n_frag = 0;  // raster_tri's fragment counter (unused here)
  for (int base = 0; base < p.n_meshlets; base += kVsdListCap) {
    const int lim = min(p.n_meshlets, base + kVsdListCap);
    for (int m = base + tid; m < lim; m += kVsdThreads) {
      const float4 sph = __ldg(reinterpret_cast<const float4*>(p.meshlets + m));
      bool keep = sphere_meets_tile(P, sph, fx, fy, cx, cy, tx0, ty0);
      if (keep && front_sign != 0 && cone_back_facing(p.meshlets + m, sph, front_sign, ox, oy, oz)) keep = false;
      if (keep) sm.list[atomicAdd(&sm.n_list, 1)] = m;
    }
    __syncthreads();
    const int n_list = sm.n_list;
    VtxS* sv = sm.sv[warp];
    for (;;) {
      int li = 0;
      if (lane == 0) li = atomicAdd(&sm.next, 1);
      li = __shfl_sync(0xffffffffu, li, 0);
      if (li >= n_list) break;
      const int m = sm.list[li];
      const int4 hdr = __ldg(reinterpret_cast<const int4*>(p.meshlets + m) + 2);  // vert_off, n_verts, tri_off, n_tris
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int s = lane + 32 * h;
        if (s < hdr.y) {
          const float4 q = __ldg(p.vpos + __ldg(p.ml_verts + hdr.x + s));
          VtxScreen o;
          xform_vertex(P, q.x, q.y, q.z, win, fx, fy, cx, cy, o);
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
          trec[h] = __ldg(p.ml_tris + hdr.z + t);
          const VtxS a = sv[trec[h].x & 255], b = sv[(trec[h].x >> 8) & 255], c = sv[(trec[h].x >> 16) & 255];
          const int nfront = (a.Z > kVsdZnear) + (b.Z > kVsdZnear) + (c.Z > kVsdZnear);
          if (nfront == 3)
            raster_tri<kVsdTile>(a, b, c, trec[h].y, front_sign, tx0, ty0, iz_far, zt, n_frag);
          else if (nfront > 0)
            mixed = true;
        }
        mixed_mask[h] = __ballot_sync(0xffffffffu, mixed);
      }
      // triangles crossing the near plane: the whole warp scans the tile for one such triangle at a time
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        unsigned mm = mixed_mask[h];
        while (mm) {
          const int src = __ffs(mm) - 1;
          mm &= mm - 1;
          const unsigned packed = __shfl_sync(0xffffffffu, trec[h].x, src);
          const unsigned face = __shfl_sync(0xffffffffu, trec[h].y, src);
          float Pc[3][3];
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            const float4 q = __ldg(p.vpos + __ldg(p.ml_verts + hdr.x + ((packed >> (8 * k)) & 255)));
            VtxScreen o;
            xform_vertex(P, q.x, q.y, q.z, win, fx, fy, cx, cy, o);
            Pc[k][0] = o.X; Pc[k][1] = o.Y; Pc[k][2] = o.Z;
          }
          HomTri ht;
          hom_setup(Pc[0], Pc[1], Pc[2], ht);
          for (int px = lane; px < kVsdTile * kVsdTile; px += 32) {
            const int r = px / kVsdTile, jl = px - r * kVsdTile;
            const float dx = pixel_ray((float)(tx0 + jl) + 0.5f, 0.f, 1.f, cx, fx);
            const float dy = pixel_ray((float)(ty0 + r) + 0.5f, 0.f, 1.f, cy, fy);
            float l0, l1, l2, iz;
            if (hom_cover(ht, dx, dy, kVsdZnear, kVsdZfar, l0, l1, l2, iz)) atomicMax(&zt[px], depth_key(iz, face));
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
}

// rounded (never contracted) fp64: the same bits as numpy's float64
__device__ __forceinline__ double ray_scale(int u, int v, double fx, double fy, double cx, double cy) {
  const double a = __ddiv_rn(__dsub_rn((double)u, cx), fx), b = __ddiv_rn(__dsub_rn((double)v, cy), fy);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)), 1.0));
}

__device__ __forceinline__ float key_depth(unsigned long long key) {
  return key ? __frcp_rn(__uint_as_float((unsigned)(key >> 32))) : 0.f;
}

// grid = (N, tiles_x * tiles_y), kVsdThreads threads
__global__ void __launch_bounds__(kVsdThreads, 2) vsd_count_kernel(const VsdParams p) {
  __shared__ VsdSmem sm;
  const int tid = threadIdx.x, lane = tid & 31;
  const int n = blockIdx.x;
  const int tile = blockIdx.y;
  const int ty0 = (tile / p.tiles_x) * kVsdTile, tx0 = (tile % p.tiles_x) * kVsdTile;
  pdl_wait();  // the counters are zeroed, and the inputs may be written, by earlier work of the stream
  pdl_trigger();
  if (tid < 16) sm.P[0][tid] = __ldg(p.pred + (size_t)n * 16 + tid);
  else if (tid < 32) sm.P[1][tid - 16] = __ldg(p.gt + (size_t)n * p.gt_stride + tid - 16);
  const float* Kn = p.K + (size_t)n * p.k_stride;
  const float fx = __ldg(Kn + 0), cx = __ldg(Kn + 2), fy = __ldg(Kn + 4), cy = __ldg(Kn + 5);
  __syncthreads();
  if (tid < 2) sm.render[tid] = sphere_meets_tile(sm.P[tid], p.bs, fx, fy, cx, cy, tx0, ty0);
  if (tid == 0) sm.n_list = sm.next = 0;
  for (int i = tid; i < 2 + p.T; i += kVsdThreads) sm.cnt[i] = 0;
  for (int i = tid; i < p.T; i += kVsdThreads) sm.tau[i] = (double)__ldg(p.taus + i);
  __syncthreads();
  const bool rE = sm.render[0], rG = sm.render[1];
  if (!rE && !rG) return;  // uniform over the CTA: the mesh is seen in this tile under neither pose
  for (int i = tid; i < 2 * kVsdTile * kVsdTile; i += kVsdThreads) (&sm.zt[0][0])[i] = 0ull;
  __syncthreads();
  if (rE) render_ztile(p, sm, sm.P[0], sm.zt[0], fx, fy, cx, cy, tx0, ty0);
  if (rG) render_ztile(p, sm, sm.P[1], sm.zt[1], fx, fy, cx, cy, tx0, ty0);
  __syncthreads();

  const double fxd = fx, fyd = fy, cxd = cx, cyd = cy, delta = p.delta;
  const float* D = p.depth + (size_t)n * p.depth_stride;
  int n_union = 0, n_inter = 0;
  double diff[kVsdPix];  // |dist_G - dist_E| of pixels in both visibility masks, NaN elsewhere (fails every >=)
#pragma unroll
  for (int k = 0; k < kVsdPix; ++k) {
    diff[k] = __longlong_as_double(0x7ff8000000000000ll);
    const int px = tid + k * kVsdThreads;
    const int u = tx0 + (px % kVsdTile), v = ty0 + px / kVsdTile;
    if (u >= p.W || v >= p.H) continue;
    const float dE = key_depth(sm.zt[0][px]), dG = key_depth(sm.zt[1][px]);
    if (!(dE > 0.f) && !(dG > 0.f)) continue;
    const double d = (double)__ldg(D + (size_t)v * p.W + u);
    const double s = ray_scale(u, v, fxd, fyd, cxd, cyd);
    const double tT = __dmul_rn(d, s), tE = __dmul_rn((double)dE, s), tG = __dmul_rn((double)dG, s);
    const bool vG = (__dsub_rn(tG, tT) <= delta || d == 0.0) && dG > 0.f;
    const bool vE = ((__dsub_rn(tE, tT) <= delta || d == 0.0) && dE > 0.f) || (vG && dE > 0.f);
    n_union += (vG || vE) ? 1 : 0;
    if (vG && vE) {
      ++n_inter;
      diff[k] = fabs(__dsub_rn(tG, tE));
    }
  }
  n_union = __reduce_add_sync(0xffffffffu, n_union);
  n_inter = __reduce_add_sync(0xffffffffu, n_inter);
  if (lane == 0 && n_union) {
    atomicAdd(&sm.cnt[0], n_union);
    atomicAdd(&sm.cnt[1], n_inter);
  }
  if (__any_sync(0xffffffffu, n_inter != 0)) {  // n_inter is warp-uniform after the reduction
    for (int t = 0; t < p.T; ++t) {
      const double tau = sm.tau[t];
      int c = 0;
#pragma unroll
      for (int k = 0; k < kVsdPix; ++k) c += diff[k] >= tau ? 1 : 0;
      c = __reduce_add_sync(0xffffffffu, c);
      if (lane == 0 && c) atomicAdd(&sm.cnt[2 + t], c);
    }
  }
  __syncthreads();
  int* row = p.counts + (size_t)n * (p.T + 2);
  for (int i = tid; i < 2 + p.T; i += kVsdThreads)
    if (sm.cnt[i]) atomicAdd(row + i, sm.cnt[i]);
}

__global__ void __launch_bounds__(256) vsd_finish_kernel(const int* __restrict__ counts, long long N, int T,
                                                        float* __restrict__ errs) {
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * T) return;
  const long long n = i / T;
  const int t = (int)(i - n * T);
  const int* c = counts + n * (T + 2);
  const int u = c[0], inter = c[1];
  errs[i] = u == 0 ? 1.f : (float)((double)(c[2 + t] + (u - inter)) / (double)u);
}

// Arguments are checked by fp_vsd_errors (fp_api_ops.cu).  Builds the meshlets on the host, uploads them with
// stream-ordered allocation, counts, finishes and frees the upload stream-ordered.
int vsd_errors_launch(const float* pos, int V, const int* faces, int F, const float* pred, int N, const float* gt,
                      int n_gt, const float* depth, int n_depth, int H, int W, const float* K, int n_K, float delta,
                      const float* taus, int T, float* errs_out, int* counts_out, cudaStream_t stream) {
  if (N == 0) return 0;
  MeshHost mh;
  const int rc = build_mesh_host(V, F, pos, nullptr, nullptr, 3, faces, mh);
  if (rc) return rc;
  // one stream-ordered allocation: vertex positions, meshlets, meshlet vertex ids, meshlet triangles and (without
  // counts_out) the counter rows, each 256-byte aligned
  auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
  const size_t b_pos = up(mh.vpos.size() * sizeof(float4)), b_ml = up(mh.meshlets.size() * sizeof(Meshlet));
  const size_t b_mv = up(mh.ml_verts.size() * sizeof(int)), b_mt = up(mh.ml_tris.size() * sizeof(uint2));
  const size_t b_cnt = counts_out ? 0 : up((size_t)N * (T + 2) * sizeof(int));
  char* buf = nullptr;
  FP_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&buf), b_pos + b_ml + b_mv + b_mt + b_cnt, stream));
  VsdParams p;
  p.vpos = reinterpret_cast<const float4*>(buf);
  p.meshlets = reinterpret_cast<const Meshlet*>(buf + b_pos);
  p.ml_verts = reinterpret_cast<const int*>(buf + b_pos + b_ml);
  p.ml_tris = reinterpret_cast<const uint2*>(buf + b_pos + b_ml + b_mv);
  p.counts = counts_out ? counts_out : reinterpret_cast<int*>(buf + b_pos + b_ml + b_mv + b_mt);
  int status = 0;
  // pageable sources: each copy has read its source when it returns, so mh may go out of scope after the launches
  cudaError_t e = cudaMemcpyAsync(buf, mh.vpos.data(), mh.vpos.size() * sizeof(float4), cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(buf + b_pos, mh.meshlets.data(), mh.meshlets.size() * sizeof(Meshlet), cudaMemcpyHostToDevice,
                        stream);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(buf + b_pos + b_ml, mh.ml_verts.data(), mh.ml_verts.size() * sizeof(int),
                        cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(buf + b_pos + b_ml + b_mv, mh.ml_tris.data(), mh.ml_tris.size() * sizeof(uint2),
                        cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(p.counts, 0, (size_t)N * (T + 2) * sizeof(int), stream);
  if (e == cudaSuccess) {
    p.n_meshlets = (int)mh.meshlets.size();
    p.bs = make_float4(mh.bs[0], mh.bs[1], mh.bs[2], mh.bs[3]);
    p.front_sign = mh.front_sign;
    p.pred = pred;
    p.gt = gt;
    p.gt_stride = n_gt == 1 ? 0 : 16;
    p.depth = depth;
    p.depth_stride = n_depth == 1 ? 0 : (size_t)H * W;
    p.K = K;
    p.k_stride = n_K == 1 ? 0 : 9;
    p.H = H;
    p.W = W;
    p.tiles_x = (W + kVsdTile - 1) / kVsdTile;
    p.delta = (double)delta;
    p.taus = taus;
    p.T = T;
    const dim3 grid((unsigned)N, (unsigned)(p.tiles_x * ((H + kVsdTile - 1) / kVsdTile)));
    e = launch_pdl(vsd_count_kernel, grid, dim3(kVsdThreads), 0, stream, 1, p);
    if (e == cudaSuccess) {
      note_launches(1);
      const long long total = (long long)N * T;
      e = launch_pdl(vsd_finish_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, stream, 1,
                     (const int*)p.counts, (long long)N, T, errs_out);
      if (e == cudaSuccess) note_launches(1);
    }
  }
  if (e != cudaSuccess) {
    set_last_error("fp_vsd_errors: %s", cudaGetErrorString(e));
    status = -2;
  }
  const cudaError_t ef = cudaFreeAsync(buf, stream);
  if (status) return status;
  FP_CUDA_OK(ef);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace fp
