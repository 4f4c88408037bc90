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

}  // namespace fp
