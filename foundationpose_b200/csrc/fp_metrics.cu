// fp_metrics.cu — pose accuracy: ADD and ADD-S (Utils.py:232-253) of N estimated poses against their ground truth.
//
//   pose_errors_kernel  one cluster of eight CTAs per pose.  Each CTA owns a contiguous eighth of the model points as
//                       queries, transformed by the ground-truth pose and held in registers (kMetQ per thread).  ADD
//                       pairs each query with the same point under the estimated pose (O(P) per pose).  ADD-S streams
//                       every model point through shared memory in tiles of kMetTile, transformed by the estimated
//                       pose as the tile is loaded, and keeps each query's smallest squared distance (O(P^2) per pose).
//                       Squared distances are dx^2 + dy^2 + dz^2 of the two transformed points in fp32: the expansion
//                       |a|^2 + |b|^2 - 2 a.b cancels catastrophically at 0.5 m coordinates and millimetre distances.
//                       Per-query distances are summed in fp64 in a fixed order (slots, warp tree, warps, then the
//                       eight CTAs in rank order over distributed shared memory), and the launch shape depends on P
//                       only: a pose's errors are bit-identical across calls and batch sizes.
//
//   sym_pose_errors_kernel  BOP's MSSD / MSPD: one CTA per pose.  The model points are staged through shared memory
//                       in tiles of kSymTile, each with its image under the estimated pose E (and that image's
//                       projection).  A work item is one symmetry s over one chunk of the tile: the warp composes G s
//                       in registers, every lane takes a point of the chunk at a time and keeps the largest squared
//                       distance, and the warp's maximum is merged into s's slot in shared memory by an integer
//                       atomicMax (squared distances are >= +0, so their bit patterns order as the floats do).  The
//                       minimum over the slots is taken once at the end.  Max and min are exact and every distance is
//                       one expression of (point, E, G, s, K), so the results do not depend on the launch shape, on
//                       the batch or on the order of the symmetries.
#include "../../include/fpose.h"
#include "fp_common.cuh"

namespace fp {

constexpr int kMetCluster = 8;       // CTAs per pose
constexpr int kMetQ = 4;             // queries per thread and batch
constexpr int kMetTile = 512;        // estimated points per shared-memory tile
constexpr int kMetMaxThreads = 256;  // threads per CTA (the launch uses fewer for small slices)

// rows of [R | t] of a row-major 4x4 pose
__device__ __forceinline__ void load_rt(const float* __restrict__ m, float (&r)[12]) {
#pragma unroll
  for (int i = 0; i < 12; ++i) r[i] = __ldg(m + i);
}
// one rounding order for both poses: a pose compared with itself gives bit-identical points
__device__ __forceinline__ float3 xform(const float (&m)[12], float x, float y, float z) {
  return make_float3(fmaf(m[0], x, fmaf(m[1], y, fmaf(m[2], z, m[3]))), fmaf(m[4], x, fmaf(m[5], y, fmaf(m[6], z, m[7]))),
                     fmaf(m[8], x, fmaf(m[9], y, fmaf(m[10], z, m[11]))));
}
__device__ __forceinline__ double warp_sum_f64(double x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

// grid = N clusters of kMetCluster CTAs; blockDim.x a multiple of 32, at most kMetMaxThreads.  Each CTA walks its
// slice in `batches` batches of `per_batch` queries, query slot s of thread t being base + s * blockDim.x + t.
template <bool kAdd, bool kAdds>
__global__ void __launch_bounds__(kMetMaxThreads) pose_errors_kernel(const float* __restrict__ pts, int P,
                                                                     const float* __restrict__ pred,
                                                                     const float* __restrict__ gt, int gt_stride,
                                                                     float* __restrict__ add_out, float* __restrict__ adds_out,
                                                                     int batches, int per_batch) {
  __shared__ float4 tile[kMetTile];
  __shared__ double warp_part[2][kMetMaxThreads / 32];
  __shared__ double cta_part[2];  // read by rank 0 over DSMEM
  const int rank = (int)cluster_ctarank();
  const int pose = blockIdx.x / kMetCluster;
  const int nthr = blockDim.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_wait();
  float mp[12], mg[12];
  load_rt(pred + (size_t)pose * 16, mp);
  load_rt(gt + (size_t)pose * gt_stride, mg);
  const int per_cta = (P + kMetCluster - 1) / kMetCluster;
  const int q_begin = min(P, rank * per_cta), q_end = min(P, q_begin + per_cta);
  double add_sum = 0.0, adds_sum = 0.0;
  for (int b = 0; b < batches; ++b) {
    const int base = q_begin + b * per_batch, lim = min(q_end, base + per_batch);
    float qx[kMetQ], qy[kMetQ], qz[kMetQ], best[kMetQ];
#pragma unroll
    for (int s = 0; s < kMetQ; ++s) {
      const int q = base + s * nthr + threadIdx.x;
      const int qi = q < lim ? q : 0;  // idle slots compute on point 0 and are not summed
      const float x = __ldg(pts + 3 * qi), y = __ldg(pts + 3 * qi + 1), z = __ldg(pts + 3 * qi + 2);
      const float3 g = xform(mg, x, y, z);
      qx[s] = g.x;
      qy[s] = g.y;
      qz[s] = g.z;
      best[s] = __int_as_float(0x7f800000);
      if (kAdd && q < lim) {
        const float3 p = xform(mp, x, y, z);
        const float dx = p.x - g.x, dy = p.y - g.y, dz = p.z - g.z;
        add_sum += (double)sqrtf(fmaf(dx, dx, fmaf(dy, dy, dz * dz)));
      }
    }
    if (kAdds && base < lim) {  // uniform over the CTA
      for (int t0 = 0; t0 < P; t0 += kMetTile) {
        __syncthreads();  // the previous tile has been consumed
        for (int j = threadIdx.x; j < kMetTile; j += nthr) {
          float4 v = make_float4(__int_as_float(0x7f800000), __int_as_float(0x7f800000), __int_as_float(0x7f800000), 0.f);
          if (t0 + j < P) {
            const float* e = pts + 3 * (t0 + j);
            const float3 p = xform(mp, __ldg(e), __ldg(e + 1), __ldg(e + 2));
            v = make_float4(p.x, p.y, p.z, 0.f);
          }
          tile[j] = v;
        }
        __syncthreads();
#pragma unroll 8
        for (int j = 0; j < kMetTile; ++j) {
          const float4 e = tile[j];
#pragma unroll
          for (int s = 0; s < kMetQ; ++s) {
            const float dx = qx[s] - e.x, dy = qy[s] - e.y, dz = qz[s] - e.z;
            best[s] = fminf(best[s], fmaf(dx, dx, fmaf(dy, dy, dz * dz)));
          }
        }
      }
#pragma unroll
      for (int s = 0; s < kMetQ; ++s)
        if (base + s * nthr + (int)threadIdx.x < lim) adds_sum += (double)sqrtf(best[s]);
    }
  }
  add_sum = warp_sum_f64(add_sum);
  adds_sum = warp_sum_f64(adds_sum);
  if (lane == 0) {
    warp_part[0][warp] = add_sum;
    warp_part[1][warp] = adds_sum;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, s = 0.0;
    for (int w = 0; w < nthr / 32; ++w) {
      a += warp_part[0][w];
      s += warp_part[1][w];
    }
    cta_part[0] = a;
    cta_part[1] = s;
  }
  cluster_sync_all();  // every CTA's partial sums are visible cluster-wide
  if (rank == 0 && threadIdx.x < 2) {
    const uint32_t mine = smem_u32(&cta_part[threadIdx.x]);
    double sum = 0.0;
#pragma unroll
    for (int r = 0; r < kMetCluster; ++r) {
      uint32_t remote;
      double v;
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(mine), "r"((unsigned)r));
      asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(remote));
      sum += v;
    }
    const float mean = (float)(sum / (double)P);
    if (threadIdx.x == 0 && kAdd) add_out[pose] = mean;
    if (threadIdx.x == 1 && kAdds) adds_out[pose] = mean;
  }
  cluster_sync_all();  // peers keep their shared memory alive until rank 0 has read it
}

// Arguments are checked by fp_pose_errors (fp_api_ops.cu).  The launch shape is a function of P alone.
int pose_errors_launch(const float* pts, int P, const float* pred, int N, const float* gt, int n_gt, float* add_out,
                       float* adds_out, cudaStream_t stream) {
  if (N == 0 || (!add_out && !adds_out)) return 0;
  const int per_cta = (P + kMetCluster - 1) / kMetCluster;
  const int batches = (per_cta + kMetMaxThreads * kMetQ - 1) / (kMetMaxThreads * kMetQ);
  const int per_batch = (per_cta + batches - 1) / batches;
  const int threads = ((per_batch + kMetQ - 1) / kMetQ + 31) / 32 * 32;
  const int gt_stride = n_gt == 1 ? 0 : 16;
  const dim3 grid((unsigned)N * kMetCluster), block((unsigned)threads);
  cudaError_t e;
  if (add_out && adds_out)
    e = launch_pdl(pose_errors_kernel<true, true>, grid, block, 0, stream, kMetCluster, pts, P, pred, gt, gt_stride, add_out,
                   adds_out, batches, per_batch);
  else if (add_out)
    e = launch_pdl(pose_errors_kernel<true, false>, grid, block, 0, stream, kMetCluster, pts, P, pred, gt, gt_stride, add_out,
                   adds_out, batches, per_batch);
  else
    e = launch_pdl(pose_errors_kernel<false, true>, grid, block, 0, stream, kMetCluster, pts, P, pred, gt, gt_stride, add_out,
                   adds_out, batches, per_batch);
  FP_CUDA_OK(e);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// MSSD / MSPD
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kSymTile = 1024;    // model points per shared-memory tile
constexpr int kSymThreads = 256;  // threads per CTA
constexpr int kSymWarps = kSymThreads / 32;

// NaN-propagating maximum: a NaN distance must win over every number (fmaxf would drop it)
__device__ __forceinline__ float max_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
// the squared maximum of a work item as an ordered bit pattern: NaN counts as +inf
__device__ __forceinline__ unsigned worst_bits(float w) { return w == w ? __float_as_uint(w) : 0x7f800000u; }

// [R | t] rows of G s for a row-major 4x4 symmetry s, in fp32.  For s = I every sum is x * 1 + 0 terms: G s = G exactly.
__device__ __forceinline__ void compose_sym(const float (&g)[12], const float* __restrict__ s, float (&m)[12]) {
  float a[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) a[i] = __ldg(s + i);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c)
      m[4 * r + c] = fmaf(g[4 * r], a[c], fmaf(g[4 * r + 1], a[4 + c], g[4 * r + 2] * a[8 + c]));
    m[4 * r + 3] = fmaf(g[4 * r], a[3], fmaf(g[4 * r + 1], a[7], fmaf(g[4 * r + 2], a[11], g[4 * r + 3])));
  }
}
// rows 0 and 1 of K [R | t]: the numerators of the projection
__device__ __forceinline__ void compose_k(const float (&k)[9], const float (&m)[12], float (&km)[8]) {
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) km[4 * r + c] = fmaf(k[3 * r], m[c], fmaf(k[3 * r + 1], m[4 + c], k[3 * r + 2] * m[8 + c]));
}
// pi(K, M p) = (K M p)[:2] / (M p)_z, for both poses by the same expression.  z = 0 gives +-inf or NaN, never a number.
// __fmul_rn keeps the product rounded: contracted into the caller's subtraction it would differ from the staged one.
__device__ __forceinline__ float2 project(const float (&km)[8], float depth, float x, float y, float z) {
  const float r = __fdividef(1.f, depth);
  return make_float2(__fmul_rn(fmaf(km[0], x, fmaf(km[1], y, fmaf(km[2], z, km[3]))), r),
                     __fmul_rn(fmaf(km[4], x, fmaf(km[5], y, fmaf(km[6], z, km[7]))), r));
}

// grid = N CTAs of kSymThreads.  Dynamic shared memory: two float4 per tile point, (x y z u_E) and (E p, v_E), then
// one slot per symmetry and metric.  `chunks` (1, 2, 4 or 8) splits every tile so that small S still fills the warps.
template <bool kMssd, bool kMspd>
__global__ void __launch_bounds__(kSymThreads) sym_pose_errors_kernel(const float* __restrict__ pts, int P,
                                                                      const float* __restrict__ pred,
                                                                      const float* __restrict__ gt, int gt_stride,
                                                                      const float* __restrict__ sym, int S,
                                                                      const float* __restrict__ Kmat, int k_stride,
                                                                      float* __restrict__ mssd_out,
                                                                      float* __restrict__ mspd_out, int chunks) {
  extern __shared__ float4 sym_smem[];
  float4* tile_a = sym_smem;
  float4* tile_b = sym_smem + kSymTile;
  unsigned* worst3 = reinterpret_cast<unsigned*>(sym_smem + 2 * kSymTile);  // [S] squared MSSD candidates
  unsigned* worst2 = worst3 + (kMssd ? S : 0);                                // [S] squared MSPD candidates
  __shared__ unsigned warp_best[2][kSymWarps];
  const int pose = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_wait();
  float me[12], mg[12], k[9], ke[8];
  load_rt(pred + (size_t)pose * 16, me);
  load_rt(gt + (size_t)pose * gt_stride, mg);
  if (kMspd) {
#pragma unroll
    for (int i = 0; i < 9; ++i) k[i] = __ldg(Kmat + (size_t)pose * k_stride + i);
    compose_k(k, me, ke);
  }
  for (int s = threadIdx.x; s < S * (int(kMssd) + int(kMspd)); s += kSymThreads) worst3[s] = 0u;
  const int chunk = kSymTile / chunks, items = S * chunks;
  for (int t0 = 0; t0 < P; t0 += kSymTile) {
    const int n = min(kSymTile, P - t0);
    __syncthreads();  // the previous tile has been consumed (and, first time round, the slots are zeroed)
    for (int j = threadIdx.x; j < kSymTile; j += kSymThreads) {
      // slots past the end repeat the tile's first point: a repeated pair cannot change a maximum
      const float* p = pts + 3 * (size_t)(t0 + (j < n ? j : 0));
      const float x = __ldg(p), y = __ldg(p + 1), z = __ldg(p + 2);
      const float3 e = xform(me, x, y, z);
      float2 uv = make_float2(0.f, 0.f);
      if (kMspd) uv = project(ke, e.z, x, y, z);
      tile_a[j] = make_float4(x, y, z, uv.x);
      tile_b[j] = make_float4(e.x, e.y, e.z, uv.y);
    }
    __syncthreads();
    for (int it = warp; it < items; it += kSymWarps) {
      const int s = it / chunks, j0 = (it - s * chunks) * chunk;
      if (j0 >= n) continue;  // uniform over the warp
      float m[12], km[8];
      compose_sym(mg, sym + (size_t)s * 16, m);
      if (kMspd) compose_k(k, m, km);
      float w3 = 0.f, w2 = 0.f;
      const int j_end = min(j0 + chunk, (n + 31) & ~31);
#pragma unroll 4
      for (int j = j0 + lane; j < j_end; j += 32) {
        const float4 a = tile_a[j], b = tile_b[j];
        const float3 q = xform(m, a.x, a.y, a.z);
        if (kMssd) {
          const float dx = b.x - q.x, dy = b.y - q.y, dz = b.z - q.z;
          w3 = max_nan(w3, fmaf(dx, dx, fmaf(dy, dy, dz * dz)));
        }
        if (kMspd) {
          const float2 uv = project(km, q.z, a.x, a.y, a.z);
          const float du = a.w - uv.x, dv = b.w - uv.y;
          w2 = max_nan(w2, fmaf(du, du, dv * dv));
        }
      }
      if (kMssd) {
        const unsigned w = __reduce_max_sync(0xffffffffu, worst_bits(w3));
        if (lane == 0) atomicMax(worst3 + s, w);
      }
      if (kMspd) {
        const unsigned w = __reduce_max_sync(0xffffffffu, worst_bits(w2));
        if (lane == 0) atomicMax(worst2 + s, w);
      }
    }
  }
  __syncthreads();
  unsigned b3 = 0x7f800000u, b2 = 0x7f800000u;
  for (int s = threadIdx.x; s < S; s += kSymThreads) {
    if (kMssd) b3 = min(b3, worst3[s]);
    if (kMspd) b2 = min(b2, worst2[s]);
  }
  b3 = __reduce_min_sync(0xffffffffu, b3);
  b2 = __reduce_min_sync(0xffffffffu, b2);
  if (lane == 0) {
    warp_best[0][warp] = b3;
    warp_best[1][warp] = b2;
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    unsigned b = 0x7f800000u;
#pragma unroll
    for (int w = 0; w < kSymWarps; ++w) b = min(b, warp_best[threadIdx.x][w]);
    if (threadIdx.x == 0 && kMssd) mssd_out[pose] = sqrtf(__uint_as_float(b));
    if (threadIdx.x == 1 && kMspd) mspd_out[pose] = sqrtf(__uint_as_float(b));
  }
}

// Arguments are checked by fp_sym_pose_errors (fp_api_ops.cu).  The launch shape is a function of S alone.
int sym_pose_errors_launch(const float* pts, int P, const float* pred, int N, const float* gt, int n_gt, const float* sym,
                           int S, const float* K, int n_K, float* mssd_out, float* mspd_out, cudaStream_t stream) {
  if (N == 0 || (!mssd_out && !mspd_out)) return 0;
  const int chunks = S >= kSymWarps ? 1 : S >= kSymWarps / 2 ? 2 : S >= kSymWarps / 4 ? 4 : 8;
  const size_t smem = 2 * kSymTile * sizeof(float4) + (size_t)S * ((mssd_out ? 1 : 0) + (mspd_out ? 1 : 0)) * sizeof(unsigned);
  const int gt_stride = n_gt == 1 ? 0 : 16, k_stride = n_K == 1 ? 0 : 9;
  const dim3 grid((unsigned)N), block(kSymThreads);
  static std::atomic<unsigned long long> attr_mask{0};  // per device: the attribute is device state
  if (!device_bit_test(attr_mask)) {
    const int most = 2 * kSymTile * (int)sizeof(float4) + 2 * FP_METRICS_MAX_SYMMETRIES * (int)sizeof(unsigned);
    FP_CUDA_OK(cudaFuncSetAttribute(sym_pose_errors_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
    FP_CUDA_OK(cudaFuncSetAttribute(sym_pose_errors_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
    FP_CUDA_OK(cudaFuncSetAttribute(sym_pose_errors_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
    device_bit_set(attr_mask);
  }
  cudaError_t e;
  if (mssd_out && mspd_out)
    e = launch_pdl(sym_pose_errors_kernel<true, true>, grid, block, smem, stream, 1, pts, P, pred, gt, gt_stride, sym, S, K,
                   k_stride, mssd_out, mspd_out, chunks);
  else if (mssd_out)
    e = launch_pdl(sym_pose_errors_kernel<true, false>, grid, block, smem, stream, 1, pts, P, pred, gt, gt_stride, sym, S, K,
                   k_stride, mssd_out, mspd_out, chunks);
  else
    e = launch_pdl(sym_pose_errors_kernel<false, true>, grid, block, smem, stream, 1, pts, P, pred, gt, gt_stride, sym, S, K,
                   k_stride, mssd_out, mspd_out, chunks);
  FP_CUDA_OK(e);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace fp
