// fp_vis.cu — the debug canvases of get_vis (predict_pose_refine.py:241-293, predict_score.py:27-52), composed on the
// device from the crop producer's fp32 vis record (CropParams::vis, [N][2][160][160] (r, g, b, depth)) and written as
// the uint8 RGB image the reference returns, less its text labels (drawn on the host).
//
//   vis_range_kernel   one CTA per canvas row: min and max of the row's depth values (refiner: both images, scorer:
//                      the rendered one).  Min and max are exact, and the reduction order is fixed anyway: the range of
//                      a hypothesis does not depend on the batch it is in.
//   vis_refine_kernel  one thread per canvas pixel of one half (start poses left, refined poses right) of the refiner
//                      canvas: make_grid_image's padding (torchvision make_grid, pad 255; a single image is returned
//                      unpadded), rgb*255 and depth_to_vis (Utils.py:456-479, inverse=False) truncated to uint8.
//   vis_score_kernel   one thread per canvas pixel of the scorer canvas: the 160 x 655 row [rgbA | 5 | depthA | 5 | rgbB
//                      | 5 | depthB] resampled to 100 x 409 with cv2.resize(fx=fy=0.625, INTER_LINEAR)'s rule in fp64
//                      (source coordinate (d + 0.5) * 1.6 - 0.5, weights 1 - f and f, horizontal pass first; within
//                      1e-9 of cv2's float64 result, tests/test_vis_cpu.py), rows in the order of a device index
//                      array, each followed by 5 rows of 255, truncated to uint8.
#include "fp_common.cuh"
#include "fp_vis.cuh"

namespace fp {

namespace {

constexpr int S = 160;
constexpr int kPix = S * S;

// cv2.COLORMAP_JET, index -> 0xRRGGBB (applyColorMap(...)[..., ::-1]: the reference reverses BGR to RGB)
#define FP_JET_TABLE \
    0x000080u, 0x000084u, 0x000088u, 0x00008cu, 0x000090u, 0x000094u, 0x000098u, 0x00009cu, \
    0x0000a0u, 0x0000a4u, 0x0000a8u, 0x0000acu, 0x0000b0u, 0x0000b4u, 0x0000b8u, 0x0000bcu, \
    0x0000c0u, 0x0000c4u, 0x0000c8u, 0x0000ccu, 0x0000d0u, 0x0000d4u, 0x0000d8u, 0x0000dcu, \
    0x0000e0u, 0x0000e4u, 0x0000e8u, 0x0000ecu, 0x0000f0u, 0x0000f4u, 0x0000f8u, 0x0000fcu, \
    0x0000ffu, 0x0004ffu, 0x0008ffu, 0x000cffu, 0x0010ffu, 0x0014ffu, 0x0018ffu, 0x001cffu, \
    0x0020ffu, 0x0024ffu, 0x0028ffu, 0x002cffu, 0x0030ffu, 0x0034ffu, 0x0038ffu, 0x003cffu, \
    0x0040ffu, 0x0044ffu, 0x0048ffu, 0x004cffu, 0x0050ffu, 0x0054ffu, 0x0058ffu, 0x005cffu, \
    0x0060ffu, 0x0064ffu, 0x0068ffu, 0x006cffu, 0x0070ffu, 0x0074ffu, 0x0078ffu, 0x007cffu, \
    0x0080ffu, 0x0084ffu, 0x0088ffu, 0x008cffu, 0x0090ffu, 0x0094ffu, 0x0098ffu, 0x009cffu, \
    0x00a0ffu, 0x00a4ffu, 0x00a8ffu, 0x00acffu, 0x00b0ffu, 0x00b4ffu, 0x00b8ffu, 0x00bcffu, \
    0x00c0ffu, 0x00c4ffu, 0x00c8ffu, 0x00ccffu, 0x00d0ffu, 0x00d4ffu, 0x00d8ffu, 0x00dcffu, \
    0x00e0ffu, 0x00e4ffu, 0x00e8ffu, 0x00ecffu, 0x00f0ffu, 0x00f4ffu, 0x00f8ffu, 0x00fcffu, \
    0x02fffeu, 0x06fffau, 0x0afff6u, 0x0efff2u, 0x12ffeeu, 0x16ffeau, 0x1affe6u, 0x1effe2u, \
    0x22ffdeu, 0x26ffdau, 0x2affd6u, 0x2effd2u, 0x32ffceu, 0x36ffcau, 0x3affc6u, 0x3effc2u, \
    0x42ffbeu, 0x46ffbau, 0x4affb6u, 0x4effb2u, 0x52ffaeu, 0x56ffaau, 0x5affa6u, 0x5effa2u, \
    0x62ff9eu, 0x66ff9au, 0x6aff96u, 0x6eff92u, 0x72ff8eu, 0x76ff8au, 0x7aff86u, 0x7eff82u, \
    0x82ff7eu, 0x86ff7au, 0x8aff76u, 0x8eff72u, 0x92ff6eu, 0x96ff6au, 0x9aff66u, 0x9eff62u, \
    0xa2ff5eu, 0xa6ff5au, 0xaaff56u, 0xaeff52u, 0xb2ff4eu, 0xb6ff4au, 0xbaff46u, 0xbeff42u, \
    0xc2ff3eu, 0xc6ff3au, 0xcaff36u, 0xceff32u, 0xd2ff2eu, 0xd6ff2au, 0xdaff26u, 0xdeff22u, \
    0xe2ff1eu, 0xe6ff1au, 0xeaff16u, 0xeeff12u, 0xf2ff0eu, 0xf6ff0au, 0xfaff06u, 0xfeff01u, \
    0xfffc00u, 0xfff800u, 0xfff400u, 0xfff000u, 0xffec00u, 0xffe800u, 0xffe400u, 0xffe000u, \
    0xffdc00u, 0xffd800u, 0xffd400u, 0xffd000u, 0xffcc00u, 0xffc800u, 0xffc400u, 0xffc000u, \
    0xffbc00u, 0xffb800u, 0xffb400u, 0xffb000u, 0xffac00u, 0xffa800u, 0xffa400u, 0xffa000u, \
    0xff9c00u, 0xff9800u, 0xff9400u, 0xff9000u, 0xff8c00u, 0xff8800u, 0xff8400u, 0xff8000u, \
    0xff7c00u, 0xff7800u, 0xff7400u, 0xff7000u, 0xff6c00u, 0xff6800u, 0xff6400u, 0xff6000u, \
    0xff5c00u, 0xff5800u, 0xff5400u, 0xff5000u, 0xff4c00u, 0xff4800u, 0xff4400u, 0xff4000u, \
    0xff3c00u, 0xff3800u, 0xff3400u, 0xff3000u, 0xff2c00u, 0xff2800u, 0xff2400u, 0xff2000u, \
    0xff1c00u, 0xff1800u, 0xff1400u, 0xff1000u, 0xff0c00u, 0xff0800u, 0xff0400u, 0xff0000u, \
    0xfc0000u, 0xf80000u, 0xf40000u, 0xf00000u, 0xec0000u, 0xe80000u, 0xe40000u, 0xe00000u, \
    0xdc0000u, 0xd80000u, 0xd40000u, 0xd00000u, 0xcc0000u, 0xc80000u, 0xc40000u, 0xc00000u, \
    0xbc0000u, 0xb80000u, 0xb40000u, 0xb00000u, 0xac0000u, 0xa80000u, 0xa40000u, 0xa00000u, \
    0x9c0000u, 0x980000u, 0x940000u, 0x900000u, 0x8c0000u, 0x880000u, 0x840000u, 0x800000u \

__constant__ unsigned c_jet[256] = {FP_JET_TABLE};
const unsigned h_jet[256] = {FP_JET_TABLE};

// Utils.py:467-475 depth_to_vis(inverse=False, mode='rgb') of one float32 value: clip, the two ends map to 1,
// (vis * 255).astype(uint8) truncates, then the colour map
__device__ __forceinline__ unsigned depth_vis(float z, float zmin, float zmax) {
  const float d = fminf(fmaxf(z, zmin), zmax);
  const float v = (d == zmin || d == zmax) ? 1.f : __fdiv_rn(__fsub_rn(d, zmin), __fsub_rn(zmax, zmin));
  return c_jet[(int)__fmul_rn(v, 255.f)];
}
__device__ __forceinline__ unsigned char chan(unsigned rgb, int c) { return (unsigned char)(rgb >> (16 - 8 * c)); }
// (rgb * 255) in float32, as the reference's `rgbAs[id] * 255`
__device__ __forceinline__ float rgb255(const float4& q, int c) { return __fmul_rn(c == 0 ? q.x : (c == 1 ? q.y : q.z), 255.f); }

__global__ void vis_range_kernel(const float4* __restrict__ rec, int n_img, float2* __restrict__ range) {
  const float4* r = rec + (size_t)blockIdx.x * 2 * kPix;
  float lo = INFINITY, hi = -INFINITY;
  for (int i = threadIdx.x; i < n_img * kPix; i += blockDim.x) {
    const float z = __ldg(&r[i].w);
    lo = fminf(lo, z);
    hi = fmaxf(hi, z);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  __shared__ float2 part[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) part[warp] = make_float2(lo, hi);
  __syncthreads();
  if (threadIdx.x == 0) {
    float2 a = part[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) a = make_float2(fminf(a.x, part[w].x), fmaxf(a.y, part[w].y));
    range[blockIdx.x] = a;
  }
}

// refiner canvas: half `blk` (0 = start poses, 1 = refined poses) = columns [blk * W / 2, (blk + 1) * W / 2)
__global__ void vis_refine_kernel(const float4* __restrict__ rec, const float2* __restrict__ range, int N, int blk,
                                  unsigned char* __restrict__ canvas, int H, int W) {
  const int half = W / 2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)H * half) return;
  const int y = (int)(i / half), x = blk * half + (int)(i - (long long)(i / half) * half);
  unsigned char* out = canvas + ((size_t)y * W + x) * 3;
  // make_grid([start, refined], nrow=2, padding=2) of two blocks of bw x bh; each block is make_grid(rows, nrow=1,
  // padding=2) — or the row itself when N == 1 — of 650 x 164 rows; each row make_grid of four 160 x 160 images
  const int bp = N == 1 ? 0 : kVisPad;
  const int bw = kVisRowW + 2 * bp;
  const int lx = x - kVisPad - blk * (bw + kVisPad) - bp, ly = y - kVisPad - bp;
  const int row = ly >= 0 ? ly / (kVisRowH + kVisPad) : -1;
  const int ry = ly - row * (kVisRowH + kVisPad) - kVisPad, rx = lx - kVisPad;
  const int k = rx >= 0 ? rx / (S + kVisPad) : -1;
  const int px = rx - k * (S + kVisPad);
  if (row < 0 || row >= N || lx < 0 || lx >= kVisRowW || ry < 0 || ry >= S || k < 0 || k >= 4 || px >= S) {
    out[0] = out[1] = out[2] = 255;
    return;
  }
  const float4* r = rec + (size_t)row * 2 * kPix + (size_t)(k & 1) * kPix + ry * S + px;
  const float4 q = __ldg(r);
  if (k < 2) {
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = (unsigned char)(int)rgb255(q, c);
  } else {
    const float2 zr = __ldg(range + row);
    const unsigned v = depth_vis(q.w, zr.x, zr.y);
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = chan(v, c);
  }
}

// one pixel of the scorer's 160 x 655 row of hypothesis `id`, channel c, as a double (it is float64 in the reference)
__device__ __forceinline__ double score_row_px(const float4* __restrict__ rec, float2 zr, int vy, int vx, int c) {
  constexpr int kSeg = S + kVisScorePad;
  const int seg = vx / kSeg, px = vx - seg * kSeg;
  if (px >= S) return 255.0;
  const float4 q = __ldg(rec + (size_t)(seg >= 2) * kPix + vy * S + px);
  if ((seg & 1) == 0) return (double)rgb255(q, c);
  return (double)chan(depth_vis(q.w, zr.x, zr.y), c);
}

// cv2 resize's INTER_LINEAR source coordinate for destination index d at scale 1 / 0.625: (d + 0.5) * 1.6 - 0.5, its
// floor and the weights (1 - f, f).  The scale never reaches an edge of the 160 x 655 row.
__device__ __forceinline__ int cv_linear_tap(int d, double& w0, double& w1) {
  const double x = __dsub_rn(__dmul_rn((double)d + 0.5, 1.0 / 0.625), 0.5);
  const int s = (int)floor(x);
  w1 = __dsub_rn(x, (double)s);
  w0 = __dsub_rn(1.0, w1);
  return s;
}

__global__ void vis_score_kernel(const float4* __restrict__ rec, const float2* __restrict__ range, const int* __restrict__ order,
                                 int N, unsigned char* __restrict__ canvas) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int W = kVisScoreW;
  if (i >= (long long)N * kVisScorePitch * W) return;
  const int y = (int)(i / W), x = (int)(i - (long long)y * W);
  unsigned char* out = canvas + (size_t)i * 3;
  const int slot = y / kVisScorePitch, dy = y - slot * kVisScorePitch;
  const int id = __ldg(order + slot);
  if (dy >= kVisScoreRowH || (unsigned)id >= (unsigned)N) {
    out[0] = out[1] = out[2] = 255;
    return;
  }
  const float4* r = rec + (size_t)id * 2 * kPix;
  const float2 zr = __ldg(range + id);
  double a0, a1, b0, b1;
  const int sx = cv_linear_tap(x, a0, a1), sy = cv_linear_tap(dy, b0, b1);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    // horizontal, then vertical (no contraction: tests/vis_compose.py restates this order in numpy)
    const double h0 = __dadd_rn(__dmul_rn(score_row_px(r, zr, sy, sx, c), a0), __dmul_rn(score_row_px(r, zr, sy, sx + 1, c), a1));
    const double h1 = __dadd_rn(__dmul_rn(score_row_px(r, zr, sy + 1, sx, c), a0), __dmul_rn(score_row_px(r, zr, sy + 1, sx + 1, c), a1));
    const double v = __dadd_rn(__dmul_rn(h0, b0), __dmul_rn(h1, b1));
    out[c] = (unsigned char)(int)v;  // astype(np.uint8) truncates
  }
}

}  // namespace

int vis_canvas_size(int kind, int N, int* H, int* W) {
  FP_REQUIRE(N > 0 && (kind == 0 || kind == 1), "vis: kind must be 0 (refiner) or 1 (scorer) and N positive");
  if (kind == 1) {
    *H = N * kVisScorePitch;
    *W = kVisScoreW;
    return 0;
  }
  const int bp = N == 1 ? 0 : kVisPad;
  const int bh = N == 1 ? kVisRowH : N * (kVisRowH + kVisPad) + kVisPad;
  const int bw = kVisRowW + 2 * bp;
  *H = bh + 2 * kVisPad;
  *W = 2 * (bw + kVisPad) + kVisPad;
  return 0;
}

const unsigned* vis_colormap() { return h_jet; }

int vis_range_launch(const float4* rec, int N, int n_img, float2* range, cudaStream_t stream) {
  vis_range_kernel<<<N, 256, 0, stream>>>(rec, n_img, range);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

int vis_refine_launch(const float4* rec, const float2* range, int N, int blk, unsigned char* canvas, cudaStream_t stream) {
  int H = 0, W = 0;
  if (int rc = vis_canvas_size(0, N, &H, &W)) return rc;
  const long long n = (long long)H * (W / 2);
  vis_refine_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(rec, range, N, blk, canvas, H, W);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

int vis_score_launch(const float4* rec, const float2* range, const int* order, int N, unsigned char* canvas,
                     cudaStream_t stream) {
  const long long n = (long long)N * kVisScorePitch * kVisScoreW;
  vis_score_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(rec, range, order, N, canvas);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace fp
