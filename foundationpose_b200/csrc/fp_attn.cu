// fp_attn.cu — the non-GEMM parts of the transformer heads and the scorer tail.
//
//   layernorm_kernel     row LayerNorm over 512 channels (norm1 of the encoder layer; the residual add is
//                        fused in the producing GEMM's epilogue).
//   token_reduce_kernel  a cluster of eight CTAs per sequence (or one CTA walking the same eight ranges): norm2 -> mean over the 400 tokens -> Linear(512, 3)
//                        (refine_network.py:89-90; the mean commutes with the final linear layer), or the plain token
//                        mean of the scorer's attention output (score_network.py:72-74; out_proj then runs over all
//                        hypotheses at once).
//   cross_attn_score_kernel  scorer: attention across the L pose hypotheses (score_network.py:85-86), out_proj and
//                        Linear(512,1) folded into one 512-vector, first-max argmax by the last CTA (score_network.py:87-88,
//                        predict_score.py:196, estimater.py:226); several objects' hypotheses as independent segments.
//   pose_update_kernel   predict_pose_refine.py:195-231 + Utils.py:848-855 + pytorch3d so3_exp_map.
#include "fp_attn.cuh"

#include <stdlib.h>

#include "fp_common.cuh"
#include "fp_crop.cuh"
#include "fp_gemm.cuh"

namespace fp {

// attention itself lives in fp_attn_tc.cu (wgmma); this file keeps the SIMT pieces around it
int attn_core_launch(const AttnParams& p, cudaStream_t stream) { return attn_tc_launch(p, stream); }

// ------------------------------------------------------------------------------------------------
// LayerNorm helpers: one warp per 512-channel row, 16 channels per lane
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void load_row16(const __half* row, int lane, float (&v)[16]) {
  const uint4 a = __ldg(reinterpret_cast<const uint4*>(row + lane * 16));
  const uint4 b = __ldg(reinterpret_cast<const uint4*>(row + lane * 16) + 1);
  const __half2* ha = reinterpret_cast<const __half2*>(&a);
  const __half2* hb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __half22float2(ha[i]);
    v[2 * i] = f.x;
    v[2 * i + 1] = f.y;
    const float2 g = __half22float2(hb[i]);
    v[8 + 2 * i] = g.x;
    v[8 + 2 * i + 1] = g.y;
  }
}
__device__ __forceinline__ void load_row16(const float* row, int lane, float (&v)[16]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(row + lane * 16) + q);
    v[4 * q] = a.x;
    v[4 * q + 1] = a.y;
    v[4 * q + 2] = a.z;
    v[4 * q + 3] = a.w;
  }
}
__device__ __forceinline__ float warp_sum(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}
// gamma/beta slices of this lane (16 channels), loaded once per warp with vector loads
struct LnAffine {
  float g[16], b[16];
};
__device__ __forceinline__ void ln_load_affine(LnAffine& a, const float* gamma, const float* beta, int lane) {
  load_row16(gamma, lane, a.g);
  load_row16(beta, lane, a.b);
}
__device__ __forceinline__ void ln_row16(float (&v)[16], const LnAffine& a, float eps) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) s += v[i];
  const float mean = warp_sum(s) * (1.f / 512.f);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float d = v[i] - mean;
    q += d * d;
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.f / 512.f) + eps);
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = (v[i] - mean) * rstd * a.g[i] + a.b[i];
}

// persistent: each warp walks rows with a grid stride, keeping gamma/beta in registers
__global__ void __launch_bounds__(256) layernorm_kernel(const __half* __restrict__ x, __half* __restrict__ y,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        int rows, float eps) {
  const int lane = threadIdx.x & 31;
  const int warps_total = gridDim.x * (blockDim.x >> 5);
  LnAffine af;
  ln_load_affine(af, gamma, beta, lane);
  pdl_trigger();
  pdl_wait();
  for (int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += warps_total) {
    float v[16];
    load_row16(x + (size_t)row * 512, lane, v);
    ln_row16(v, af, eps);
    uint32_t o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = pack_half2(v[2 * i], v[2 * i + 1]);
    uint4* dst = reinterpret_cast<uint4*>(y + (size_t)row * 512 + lane * 16);
    dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
    dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
  }
}

int layernorm_launch(const __half* x, __half* y, const float* gamma, const float* beta, int rows, cudaStream_t stream) {
  if (rows == 0) return 0;
  const int blocks = min((rows + 7) / 8, num_sms() * 8);
  FP_CUDA_OK(launch_pdl(layernorm_kernel, dim3(blocks), dim3(256), 0, stream, 1, x, y, gamma, beta, rows, 1e-5f));
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

// Token reduction of one sequence (400 tokens x 512 channels), always as EIGHT token ranges of 50:
//   kLN = true : norm2 -> token mean -> Linear(512, out_dim <= 8)   (refiner heads, refine_network.py:89-90; the mean
//                commutes with the final linear layer)
//   kLN = false: token mean of the attention output -> [512] fp32   (scorer, score_network.py:72-74; the out_proj that
//                follows is a [N,512] x [512,512] product done by rowwise_linear_kernel for all hypotheses at once)
// The launch decides who owns the ranges: a CLUSTER of eight CTAs (one range each) at small batches — one CTA per
// sequence left 32 hypotheses per GPU (8-GPU shards) on 32 of 132 SMs and a single tracked pose on one — or ONE CTA
// walking the eight ranges at large batches, where 8x the CTAs only add fixed cost.
// Either way each range's partial sum is built in the same fixed order and the eight partials are added in range
// order (rank 0 reads its peers' over distributed shared memory): the result is bit-identical for both launches and
// does not depend on N or the shard.
constexpr int kHeadWarps = 8;
constexpr int kTokSplit = 8;
template <bool kLN>
__global__ void __launch_bounds__(kHeadWarps * 32) token_reduce_kernel(const __half* __restrict__ x,
                                                                       const float* __restrict__ gamma,
                                                                       const float* __restrict__ beta,
                                                                       const float* __restrict__ w,
                                                                       const float* __restrict__ bias, float* __restrict__ out,
                                                                       int T, int out_dim, float eps) {
  __shared__ float acc[kHeadWarps][512];
  __shared__ float part[kTokSplit][512];  // [range owned by this CTA][channel]
  __shared__ float meanv[512];
  const unsigned csize = cluster_nctarank();  // kTokSplit (one range per CTA) or 1 (this CTA walks all of them)
  const unsigned rank = cluster_ctarank();
  const int per_cta = kTokSplit / (int)csize;  // launches use a cluster of kTokSplit or of 1
  const int b = blockIdx.x / (int)csize, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  LnAffine af;
  if (kLN) ln_load_affine(af, gamma, beta, lane);
  pdl_trigger();
  pdl_wait();
  const int per = (T + kTokSplit - 1) / kTokSplit;
  const __half* xb = x + (size_t)b * T * 512;
  for (int ql = 0; ql < per_cta; ++ql) {
    const int q = (int)rank * per_cta + ql;
    float a[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = 0.f;
    const int t_end = min(T, (q + 1) * per);
    int t = q * per + warp;
    // two rows in flight per warp: the second row's loads overlap the first row's reductions
    for (; t + kHeadWarps < t_end; t += 2 * kHeadWarps) {
      float v0[16], v1[16];
      load_row16(xb + (size_t)t * 512, lane, v0);
      load_row16(xb + (size_t)(t + kHeadWarps) * 512, lane, v1);
      if (kLN) {
        ln_row16(v0, af, eps);
        ln_row16(v1, af, eps);
      }
#pragma unroll
      for (int i = 0; i < 16; ++i) a[i] += v0[i];
#pragma unroll
      for (int i = 0; i < 16; ++i) a[i] += v1[i];
    }
    if (t < t_end) {
      float v[16];
      load_row16(xb + (size_t)t * 512, lane, v);
      if (kLN) ln_row16(v, af, eps);
#pragma unroll
      for (int i = 0; i < 16; ++i) a[i] += v[i];
    }
    if (ql > 0) __syncthreads();  // the previous range's cross-warp sums have been read
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[warp][lane * 16 + i] = a[i];
    __syncthreads();
    for (int c = threadIdx.x; c < 512; c += kHeadWarps * 32) {
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < kHeadWarps; ++k) s += acc[k][c];
      part[ql][c] = s;
    }
  }
  if (csize > 1) cluster_sync_all();  // every CTA's `part` is complete and visible cluster-wide
  else __syncthreads();
  if (rank == 0) {
    const uint32_t mine = smem_u32(&part[0][0]);
    for (int c = threadIdx.x; c < 512; c += kHeadWarps * 32) {
      float s = 0.f;
#pragma unroll
      for (int q = 0; q < kTokSplit; ++q) {
        float v;
        if (csize == 1) {
          v = part[q][c];
        } else {
          uint32_t remote;
          asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(mine + 4u * (uint32_t)c), "r"((unsigned)q));
          asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(remote));
        }
        s += v;
      }
      meanv[c] = s / (float)T;
    }
  }
  if (csize > 1) cluster_sync_all();  // peers keep their shared memory alive until rank 0 has read it
  if (rank != 0) return;
  __syncthreads();
  if (kLN) {
    if (warp < out_dim) {
      float s = 0.f;
      for (int c = lane; c < 512; c += 32) s += meanv[c] * __ldg(w + warp * 512 + c);
      s = warp_sum(s);
      if (lane == 0) out[b * out_dim + warp] = s + bias[warp];
    }
  } else {
    for (int c = threadIdx.x; c < 512; c += kHeadWarps * 32) out[(size_t)b * 512 + c] = meanv[c];
  }
}

// cluster of eight (the portable maximum) while the eight CTAs per sequence fit four per SM, one CTA per sequence above
static inline int token_split_for(int B) { return B * kTokSplit <= 4 * num_sms() ? kTokSplit : 1; }

int head_final_launch(const __half* x, const float* gamma, const float* beta, const float* w, const float* bias,
                      float* out, int B, int T, int out_dim, cudaStream_t stream) {
  FP_REQUIRE(out_dim <= kHeadWarps, "head_final: out_dim %d > %d", out_dim, kHeadWarps);
  if (B == 0) return 0;
  const int split = token_split_for(B);
  FP_CUDA_OK(launch_pdl(token_reduce_kernel<true>, dim3(B * split), dim3(kHeadWarps * 32), 0, stream, split, x, gamma, beta,
                        w, bias, out, T, out_dim, 1e-5f));
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

// scorer: feat[b] = out_proj(mean_t attn[b, t, :])   (mean commutes with the linear projection): token means of all
// hypotheses, then one [N,512] x [512,512]^T product in fp32
int rowwise_linear_launch(const float* x, const float* w, const float* bias, float* y, int L, int n_out, cudaStream_t stream);
int token_mean_proj_launch(const __half* x, const float* w_f32, const float* bias, float* mean_ws, float* out, int B, int T,
                           cudaStream_t stream) {
  if (B == 0) return 0;
  const int split = token_split_for(B);
  FP_CUDA_OK(launch_pdl(token_reduce_kernel<false>, dim3(B * split), dim3(kHeadWarps * 32), 0, stream, split, x,
                        (const float*)nullptr, (const float*)nullptr, (const float*)nullptr, (const float*)nullptr, mean_ws, T, 0,
                        0.f));
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return rowwise_linear_launch(mean_ws, w_f32, bias, out, B, 512, stream);
}

// ------------------------------------------------------------------------------------------------
// scorer tail: attention across the L hypotheses (fp32 SIMT; 0.3 GFLOP total)
// ------------------------------------------------------------------------------------------------
// y[l, :] = W x[l, :] + b : [L][512] fp32 -> [L][n_out] fp32.  One CTA per (8 rows, n_out / gridDim.y outputs): a
// weight row is fetched once per 8 hypotheses.  Per output the summation order (16 in-lane FMAs, then the butterfly)
// does not depend on L or on the blocking.
constexpr int kRowBlock = 8;
__global__ void __launch_bounds__(256) rowwise_linear_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                             const float* __restrict__ bias, float* __restrict__ y,
                                                             int L, int n_out) {
  // x rows staged per lane: xs4[r][q][lane] = elements [16 lane + 4 q, +4) of row r (conflict-free 128-bit reads)
  __shared__ float4 xs4[kRowBlock][4][32];
  const int l0 = blockIdx.x * kRowBlock, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rows = min(kRowBlock, L - l0);
  for (int c = threadIdx.x; c < kRowBlock * 128; c += 256) {
    const int r = c >> 7, c4 = c & 127;  // c4 = float4 index inside the row
    float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < rows) q = *reinterpret_cast<const float4*>(x + (size_t)(l0 + r) * 512 + c4 * 4);
    xs4[r][c4 & 3][c4 >> 2] = q;
  }
  __syncthreads();
  const int per_cta = n_out / gridDim.y;
  const int o_end = (blockIdx.y + 1) * per_cta;
  for (int o = blockIdx.y * per_cta + warp; o < o_end; o += 8) {
    float v[16];
    load_row16(w + (size_t)o * 512, lane, v);
    float s[kRowBlock];
#pragma unroll
    for (int r = 0; r < kRowBlock; ++r) {
      float acc = 0.f;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 xv = xs4[r][q][lane];
        acc += v[4 * q] * xv.x;
        acc += v[4 * q + 1] * xv.y;
        acc += v[4 * q + 2] * xv.z;
        acc += v[4 * q + 3] * xv.w;
      }
      s[r] = warp_sum(acc);
    }
    if (lane == 0) {
      const float bo = bias[o];
      for (int r = 0; r < rows; ++r) y[(size_t)(l0 + r) * n_out + o] = s[r] + bo;
    }
  }
}

// One CTA per query hypothesis, one warp per head: attention across the hypotheses of the query's segment
// (score_network.py:85-86: one register() call's hypotheses), then out_proj and Linear(512, 1) (score_network.py:87-88)
// folded into ONE 512-vector: score = v . attn + c with v = W_out^T w_lin and c = w_lin . b_out + b_lin (both prepared
// in fp64 by fp_load_network).  The last CTA of each segment to finish takes that segment's arg-max (first index of the
// maximum, relative to the segment = ids[0] of estimater.py:226) — two launches for the whole tail.
// Segment g is rows [seg[g], seg[g + 1]) (seg = null: one segment of all L rows).  Every loop runs over
// segment-relative indices (shared scores, the lanes' stride through the exponentials, the key / value order), so a
// segment's scores are bit-identical to a launch over that segment's rows alone.
__global__ void __launch_bounds__(128) cross_attn_score_kernel(const float* __restrict__ qkv, const float* __restrict__ fold_v,
                                                               float fold_c, float offset, float* __restrict__ scores,
                                                               int* __restrict__ best, unsigned int* __restrict__ counter,
                                                               const int* __restrict__ seg, int n_seg, int seg_max, int L,
                                                               float scale) {
  extern __shared__ float sc[];  // [4][seg_max]
  __shared__ float part[4];
  __shared__ unsigned int ticket;
  const int q = blockIdx.x, h = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int g = 0, k0 = 0, n = L;
  if (seg) {  // the segment holding q: seg[g] <= q < seg[g + 1]
    int lo = 0, hi = n_seg - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (seg[mid] <= q) lo = mid;
      else hi = mid - 1;
    }
    g = lo;
    k0 = seg[g];
    n = seg[g + 1] - k0;
  }
  const float* keys = qkv + (size_t)k0 * 1536;
  float* s = sc + h * seg_max;
  const float* qv = qkv + (size_t)q * 1536 + h * 128;
  float qr[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) qr[i] = qv[lane * 4 + i];
  float mx = -INFINITY;
#pragma unroll 6  // independent key rows: keep several L2 loads in flight (the loop is latency-bound)
  for (int k = 0; k < n; ++k) {
    const float4 kv = __ldg(reinterpret_cast<const float4*>(keys + (size_t)k * 1536 + 512 + h * 128 + lane * 4));
    float d = qr[0] * kv.x + qr[1] * kv.y + qr[2] * kv.z + qr[3] * kv.w;
    d = warp_sum(d) * scale;
    if (lane == 0) s[k] = d;
    mx = fmaxf(mx, d);
  }
  __syncwarp();
  float sum = 0.f;
  for (int k = lane; k < n; k += 32) {
    const float e = expf(s[k] - mx);
    s[k] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  __syncwarp();
  float o[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 6
  for (int k = 0; k < n; ++k) {
    const float pk = s[k];
    const float4 vv = __ldg(reinterpret_cast<const float4*>(keys + (size_t)k * 1536 + 1024 + h * 128 + lane * 4));
    o[0] += pk * vv.x;
    o[1] += pk * vv.y;
    o[2] += pk * vv.z;
    o[3] += pk * vv.w;
  }
  const float inv = 1.f / sum;
  const float4 fv = __ldg(reinterpret_cast<const float4*>(fold_v + h * 128 + lane * 4));
  float p = (o[0] * inv) * fv.x + (o[1] * inv) * fv.y + (o[2] * inv) * fv.z + (o[3] * inv) * fv.w;
  p = warp_sum(p);
  if (lane == 0) part[h] = p;
  __syncthreads();
  if (threadIdx.x == 0) {
    scores[q] = (((part[0] + part[1]) + part[2]) + part[3]) + fold_c + offset;
    __threadfence();
    ticket = atomicAdd(counter + g, 1u);
  }
  __syncthreads();
  if (ticket != (unsigned)(n - 1)) return;
  // last CTA of the segment: every score of it is visible; first index of the maximum
  __threadfence();
  __shared__ float sv[128];
  __shared__ int si[128];
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int l = threadIdx.x; l < n; l += 128) {
    const float v = __ldcg(scores + k0 + l);
    if (v > bv || (v == bv && l < bi)) {
      bv = v;
      bi = l;
    }
  }
  sv[threadIdx.x] = bv;
  si[threadIdx.x] = bi;
  __syncthreads();
  for (int st = 64; st > 0; st >>= 1) {
    if (threadIdx.x < st) {
      const float ov = sv[threadIdx.x + st];
      const int oi = si[threadIdx.x + st];
      if (ov > sv[threadIdx.x] || (ov == sv[threadIdx.x] && oi < si[threadIdx.x])) {
        sv[threadIdx.x] = ov;
        si[threadIdx.x] = oi;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (best) best[g] = si[0];
    counter[g] = 0u;  // ready for the next launch (graph replays included)
  }
}

int rowwise_linear_launch(const float* x, const float* w, const float* bias, float* y, int L, int n_out, cudaStream_t stream) {
  rowwise_linear_kernel<<<dim3((L + kRowBlock - 1) / kRowBlock, 8), 256, 0, stream>>>(x, w, bias, y, L, n_out);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

int score_tail_launch(const ScoreTailParams& p, cudaStream_t stream) {
  if (p.L == 0) return 0;
  const int seg_max = p.seg ? p.seg_max : p.L;
  FP_REQUIRE(seg_max <= 4096, "score tail: %d hypotheses in one segment, at most 4096", seg_max);
  FP_REQUIRE(!p.seg || (p.n_seg >= 1 && seg_max >= 1), "score tail: bad segments");
  const size_t smem = 4 * (size_t)seg_max * sizeof(float);
  static std::atomic<unsigned long long> attr_mask{0};  // per device: the attribute is device state
  if (!device_bit_test(attr_mask)) {
    FP_CUDA_OK(cudaFuncSetAttribute(cross_attn_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 4096 * 4));
    device_bit_set(attr_mask);
  }
  FP_TRY(rowwise_linear_launch(p.feats, p.w_in, p.b_in, p.qkv, p.L, 1536, stream));
  cross_attn_score_kernel<<<p.L, 128, smem, stream>>>(p.qkv, p.fold_v, p.fold_c, p.offset, p.scores, p.best, p.counter, p.seg,
                                                      p.n_seg, seg_max, p.L, 0.08838834764831845f);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// pose update
// ------------------------------------------------------------------------------------------------
__global__ void pose_update_kernel(const float* __restrict__ pose_in, const float* __restrict__ trans,
                                   const float* __restrict__ rot, float* __restrict__ pose_out,
                                   float* __restrict__ trans_delta_out, float* __restrict__ rot_delta_out, int N,
                                   const MeshSlotDev* __restrict__ slots, const int* __restrict__ mesh_of,
                                   float trans_scale, float rot_normalizer) {
  pdl_trigger();
  pdl_wait();
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  // the half-diameter of the hypothesis's own mesh when a mesh table is given (slot 0 without slot ids)
  if (slots) trans_scale = slots[mesh_of ? mesh_of[n] : 0].half_diameter;
  const float* A = pose_in + (size_t)n * 16;
  // trans_delta = output['trans'] * (mesh_diameter / 2)   (normalize_xyz, predict_pose_refine.py:199,228-229)
  const float td[3] = {trans[n * 3] * trans_scale, trans[n * 3 + 1] * trans_scale, trans[n * 3 + 2] * trans_scale};
  // rot: so3_exp_map(tanh(rot) * rot_normalizer).T   (predict_pose_refine.py:220-222; pytorch3d eps = 1e-4)
  const float vx = tanhf(rot[n * 3]) * rot_normalizer, vy = tanhf(rot[n * 3 + 1]) * rot_normalizer,
              vz = tanhf(rot[n * 3 + 2]) * rot_normalizer;
  const float nrm = vx * vx + vy * vy + vz * vz;
  const float th = sqrtf(fmaxf(nrm, 1e-4f));
  const float ith = 1.f / th;
  const float f1 = ith * sinf(th);
  const float f2 = ith * ith * (1.f - cosf(th));
  // K = hat(v), K2 = K*K
  const float K[9] = {0.f, -vz, vy, vz, 0.f, -vx, -vy, vx, 0.f};
  float K2[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) K2[i * 3 + j] = K[i * 3] * K[j] + K[i * 3 + 1] * K[3 + j] + K[i * 3 + 2] * K[6 + j];
  float Rd[9];  // transposed exponential
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) Rd[j * 3 + i] = f1 * K[i * 3 + j] + f2 * K2[i * 3 + j] + (i == j ? 1.f : 0.f);
  float* B = pose_out + (size_t)n * 16;
  float Rn[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) Rn[i * 3 + j] = Rd[i * 3] * A[j] + Rd[i * 3 + 1] * A[4 + j] + Rd[i * 3 + 2] * A[8 + j];
  const float t0 = A[3] + td[0], t1 = A[7] + td[1], t2 = A[11] + td[2];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    B[i * 4 + 0] = Rn[i * 3 + 0];
    B[i * 4 + 1] = Rn[i * 3 + 1];
    B[i * 4 + 2] = Rn[i * 3 + 2];
  }
  B[3] = t0;
  B[7] = t1;
  B[11] = t2;
  B[12] = 0.f;
  B[13] = 0.f;
  B[14] = 0.f;
  B[15] = 1.f;
  if (trans_delta_out) {
    trans_delta_out[n * 3] = td[0];
    trans_delta_out[n * 3 + 1] = td[1];
    trans_delta_out[n * 3 + 2] = td[2];
  }
  if (rot_delta_out) {
#pragma unroll
    for (int i = 0; i < 9; ++i) rot_delta_out[n * 9 + i] = Rd[i];
  }
}

int pose_update_launch(const float* pose_in, const float* trans, const float* rot, float* pose_out,
                       float* trans_delta_out, float* rot_delta_out, int N, const MeshSlotDev* slots, const int* mesh_of,
                       float trans_scale, float rot_normalizer, cudaStream_t stream) {
  if (N == 0) return 0;
  FP_CUDA_OK(launch_pdl(pose_update_kernel, dim3((N + 127) / 128), dim3(128), 0, stream, 1, pose_in, trans, rot, pose_out,
                        trans_delta_out, rot_delta_out, N, slots, mesh_of, trans_scale, rot_normalizer));
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

// fp32 [rows][cols] -> fp16
__global__ void f32_to_f16_kernel(const float* __restrict__ x, __half* __restrict__ y, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = __float2half_rn(x[i]);
}
int f32_to_f16_launch(const float* x, __half* y, size_t n, cudaStream_t stream) {
  if (n == 0) return 0;
  f32_to_f16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(x, y, n);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace fp
