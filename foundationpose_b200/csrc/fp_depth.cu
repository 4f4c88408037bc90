// fp_depth.cu — per-frame depth pre-processing (once per register()/track_one() call).
//   erode_depth_kernel      restates Utils.py:359-384 (Warp kernel `erode_depth_kernel`)
//   bilateral_depth_kernel  restates Utils.py:304-343 (Warp kernel `bilateral_filter_depth_kernel`)
//   frame_prep_kernel       the two filters + depth2xyzmap + the rgb repack fused into one launch per frame
// 5x5 stencils over a 480x640 fp32 image: one thread per pixel; the stand-alone kernels (operator hooks, parity tests)
// read through L1, the fused kernel from a shared-memory tile.
#include "fp_depth.cuh"

#include "fp_common.cuh"
#include "fp_gemm.cuh"

namespace fp {

// Per-pixel bodies, shared by the stand-alone kernels (global-memory source) and the fused frame kernel (shared-memory
// tile source): the loops run column-outer / row-inner like the Warp kernels, so the float sums are formed in the
// reference's order whichever source is used.
struct GlobalSrc {
  const float* p;
  int W;
  __device__ __forceinline__ float operator()(int v, int u) const { return p[v * W + u]; }
};
struct TileSrc {  // rows [v0, ...), columns [u0, ...) of the image, `pitch` floats per row
  const float* s;
  int v0, u0, pitch;
  __device__ __forceinline__ float operator()(int v, int u) const { return s[(v - v0) * pitch + (u - u0)]; }
};

template <class Src>
__device__ __forceinline__ float erode_px(const Src& src, int w, int h, int H, int W, int radius, float diff_thres,
                                          float ratio_thres, float zfar) {
  const float d_ori = src(h, w);
  // NB: the reference writes 0 for an invalid centre and then *falls through* (Utils.py:366-384);
  // the final select below decides the value, exactly as there.
  float bad = 0.f, total = 0.f;
  for (int u = w - radius; u <= w + radius; ++u) {
    if (u < 0 || u >= W) continue;
    for (int v = h - radius; v <= h + radius; ++v) {
      if (v < 0 || v >= H) continue;
      const float cur = src(v, u);
      total += 1.f;
      if (cur < 0.001f || cur >= zfar || fabsf(cur - d_ori) > diff_thres) bad += 1.f;
    }
  }
  return (bad / total > ratio_thres) ? 0.f : d_ori;
}

template <class Src>
__device__ __forceinline__ float bilateral_px(const Src& src, int w, int h, int H, int W, int radius, float zfar,
                                              float sigmaD, float sigmaR) {
  float mean_depth = 0.f;
  int num_valid = 0;
  for (int u = w - radius; u <= w + radius; ++u) {
    if (u < 0 || u >= W) continue;
    for (int v = h - radius; v <= h + radius; ++v) {
      if (v < 0 || v >= H) continue;
      const float cur = src(v, u);
      if (cur >= 0.001f && cur < zfar) {
        ++num_valid;
        mean_depth += cur;
      }
    }
  }
  float result = 0.f;
  if (num_valid > 0) {
    mean_depth /= (float)num_valid;
    const float dc = src(h, w);
    float sum_w = 0.f, sum = 0.f;
    for (int u = w - radius; u <= w + radius; ++u) {
      if (u < 0 || u >= W) continue;
      for (int v = h - radius; v <= h + radius; ++v) {
        if (v < 0 || v >= H) continue;
        const float cur = src(v, u);
        if (cur >= 0.001f && cur < zfar && fabsf(cur - mean_depth) < 0.01f) {
          const float wgt = expf(-(float)((u - w) * (u - w) + (h - v) * (h - v)) / (2.f * sigmaD * sigmaD) -
                                 (dc - cur) * (dc - cur) / (2.f * sigmaR * sigmaR));
          sum_w += wgt;
          sum += wgt * cur;
        }
      }
    }
    if (sum_w > 0.f) result = sum / sum_w;
  }
  return result;
}

__global__ void erode_depth_kernel(const float* __restrict__ depth, float* __restrict__ out, int H, int W, int radius,
                                   float diff_thres, float ratio_thres, float zfar) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  const int h = blockIdx.y * blockDim.y + threadIdx.y;
  if (w >= W || h >= H) return;
  out[h * W + w] = erode_px(GlobalSrc{depth, W}, w, h, H, W, radius, diff_thres, ratio_thres, zfar);
}

__global__ void bilateral_depth_kernel(const float* __restrict__ depth, float* __restrict__ out, int H, int W,
                                       int radius, float zfar, float sigmaD, float sigmaR) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  const int h = blockIdx.y * blockDim.y + threadIdx.y;
  if (w >= W || h >= H) return;
  out[h * W + w] = bilateral_px(GlobalSrc{depth, W}, w, h, H, W, radius, zfar, sigmaD, sigmaR);
}

// The whole per-frame preparation of register() / track_one() in ONE launch (estimater.py:173-174, :214 / :258-262):
// erode (radius 2) -> bilateral (radius 2) -> back-projection, plus the rgb -> rgba repack, per 32 x 8-pixel block.
// The block stages its raw depth tile with a 4-pixel halo in shared memory, erodes the tile with a 2-pixel halo into
// a second shared tile (halo pixels are recomputed by the neighbouring blocks, identically) and filters from there:
// one read of the depth image instead of ~50 per pixel from L1 / L2, three launches fewer per frame (47 -> ~12 us of
// a 0.97 ms tracked frame).  Same per-pixel code as the stand-alone kernels above: bit-identical.
// kTable: one launch for several cameras (fp_track_objects / _cameras, fp_register_cameras).  blockIdx.z selects the
// camera's entry of the device table `cams` and of the format table `fmts`; the grid covers the largest frame and the
// blocks outside a smaller one leave at once.  Otherwise the one frame is `one` in format `fone`, passed by value.  The
// raw frame is read in its camera's format (FrameFmtDev): depth converted to float32 metres as the tile is loaded,
// colour repacked to RGBA8.  A frame in the default layout (FrameFmtDev::packed: packed RGB8 + float32) is read by the
// body the kernel had before formats existed (kFmt = false), which never looks at the format: on default frames the
// format-reading body measured 7.8 % slower by value (109.5 against 101.6 us per 1280x720 frame, H100 80GB HBM3 at
// 700 W, torch.profiler, alternated).  By value the launch selects the body; from the table each block branches on its
// camera's flag (block-uniform), so the tracking graphs replay whatever the formats and their key does not change.
constexpr int kFpW = 32, kFpH = 8, kFpR = 2;
constexpr int kFpRW = kFpW + 4 * kFpR, kFpRH = kFpH + 4 * kFpR;  // raw tile 40 x 16
constexpr int kFpEW = kFpW + 2 * kFpR, kFpEH = kFpH + 2 * kFpR;  // eroded tile 36 x 12

template <bool kTable, bool kFmt>
__device__ __forceinline__ void frame_prep_body(const CameraDev& cam, const FrameFmtDev& fmt, float zfar_xyz, float* raw,
                                                float* er) {
  constexpr int RW = kFpRW, RH = kFpRH, EW = kFpEW, EH = kFpEH;
  const int H = cam.H, W = cam.W;
  const float fx = cam.fx, fy = cam.fy, cx = cam.cx, cy = cam.cy;
  const int w0 = blockIdx.x * kFpW, h0 = blockIdx.y * kFpH;
  if (kTable && (w0 >= W || h0 >= H)) return;  // the whole block lies outside this camera's (smaller) frame
  const int tid = threadIdx.y * kFpW + threadIdx.x;
  for (int i = tid; i < RH * RW; i += kFpW * kFpH) {
    const int v = h0 - 2 * kFpR + i / RW, u = w0 - 2 * kFpR + i % RW;
    const bool in = v >= 0 && v < H && u >= 0 && u < W;  // out-of-image cells are never read
    raw[i] = !in ? 0.f : kFmt ? raw_depth_at(cam.depth_raw, fmt, v, u) : __ldg(cam.depth_raw + v * W + u);
  }
  __syncthreads();
  const TileSrc rsrc{raw, h0 - 2 * kFpR, w0 - 2 * kFpR, RW};
  for (int i = tid; i < EH * EW; i += kFpW * kFpH) {
    const int v = h0 - kFpR + i / EW, u = w0 - kFpR + i % EW;
    er[i] = (v >= 0 && v < H && u >= 0 && u < W) ? erode_px(rsrc, u, v, H, W, kFpR, 0.001f, 0.8f, 100.f) : 0.f;
  }
  __syncthreads();
  const int w = w0 + threadIdx.x, h = h0 + threadIdx.y;
  if (w >= W || h >= H) return;
  const float z = bilateral_px(TileSrc{er, h0 - kFpR, w0 - kFpR, EW}, w, h, H, W, kFpR, 100.f, 2.f, 100000.f);
  const int i = h * W + w;
  cam.depth[i] = z;
  float X = 0.f, Y = 0.f, Z = 0.f;
  if (!(z < 0.001f) && !(z > zfar_xyz)) {  // depth2xyzmap(_batch): Utils.py:399-438
    X = ((float)w - cx) * z / fx;
    Y = ((float)h - cy) * z / fy;
    Z = z;
  }
  cam.xyz_map[i] = make_float4(X, Y, Z, 0.f);
  cam.rgb[i] = kFmt ? raw_rgba_at(cam.rgb_raw, fmt, h, w)
                   : make_uchar4(__ldg(cam.rgb_raw + 3 * i), __ldg(cam.rgb_raw + 3 * i + 1), __ldg(cam.rgb_raw + 3 * i + 2), 255);
}

// kFmt: the by-value body (ignored with kTable, where each block branches on its camera's FrameFmtDev::packed).  The
// table kernel holds both bodies; six blocks per SM keep it at the occupancy it had with one (39 registers, no spills).
template <bool kTable, bool kFmt>
__global__ void __launch_bounds__(kFpW* kFpH, kTable ? 6 : 1)
    frame_prep_kernel(const CameraDev one, const FrameFmtDev fone, const CameraDev* __restrict__ cams,
                      const FrameFmtDev* __restrict__ fmts, float zfar_xyz) {
  __shared__ float raw[kFpRH * kFpRW];
  __shared__ float er[kFpEH * kFpEW];
  if (!kTable) {
    frame_prep_body<false, kFmt>(one, fone, zfar_xyz, raw, er);
    return;
  }
  const CameraDev cam = cams[blockIdx.z];
  const FrameFmtDev fmt = fmts[blockIdx.z];
  if (fmt.packed)
    frame_prep_body<true, false>(cam, fmt, zfar_xyz, raw, er);
  else
    frame_prep_body<true, true>(cam, fmt, zfar_xyz, raw, er);
}

int frame_prep_launch(const CameraDev& one, const FrameFmtDev& fmt, float zfar_xyz, cudaStream_t stream) {
  dim3 block(kFpW, kFpH), grid((one.W + kFpW - 1) / kFpW, (one.H + kFpH - 1) / kFpH);
  (fmt.packed ? frame_prep_kernel<false, false> : frame_prep_kernel<false, true>)<<<grid, block, 0, stream>>>(
      one, fmt, nullptr, nullptr, zfar_xyz);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

int frame_prep_cameras_launch(const CameraDev* cams, const FrameFmtDev* fmts, int C, int max_H, int max_W, float zfar_xyz,
                              cudaStream_t stream) {
  dim3 block(kFpW, kFpH), grid((max_W + kFpW - 1) / kFpW, (max_H + kFpH - 1) / kFpH, C);
  frame_prep_kernel<true, true><<<grid, block, 0, stream>>>(CameraDev{}, FrameFmtDev{}, cams, fmts, zfar_xyz);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

// Depth from its own sensor aligned to the colour camera, librealsense's rs2::align rule for depth -> colour (the rule
// is restated in include/fpose.h, fp_set_camera_depth_sensor): one thread per depth pixel deprojects the two corners of
// its pixel at its depth, moves them into the colour camera, projects them and writes the slot of its z
// (aligned_slot_of) into every colour pixel of the rectangle they span with an atomicMax, so each colour pixel keeps
// the smallest z that covers it whatever the order of the threads.  Every operation is rounded on its own (no FMA
// contraction), as numpy float32 computes it.  The caller zeroes the aligned buffer first.
// kTable: blockIdx.z selects the camera's entries of the sensor table `sensors` and the camera table `cams` (colour
// intrinsics and size); the grid covers the largest depth image, and a camera without a sensor or a block outside its
// depth image leaves at once.  Otherwise the sensor `one` aligns to the colour frame `colour`, both by value.
constexpr int kAlW = 32, kAlH = 8;

template <bool kTable>
__global__ void __launch_bounds__(kAlW* kAlH) align_depth_kernel(const SensorDev one, const CameraDev colour,
                                                                 const SensorDev* __restrict__ sensors,
                                                                 const CameraDev* __restrict__ cams) {
  const SensorDev& s = kTable ? sensors[blockIdx.z] : one;
  if (kTable && !s.aligned) return;
  const int x = blockIdx.x * kAlW + threadIdx.x, y = blockIdx.y * kAlH + threadIdx.y;
  if (x >= s.W || y >= s.H) return;
  const char* row = static_cast<const char*>(s.depth) + (size_t)y * s.pitch;
  float z;
  if (s.u16) {
    const unsigned short r = __ldg(reinterpret_cast<const unsigned short*>(row) + x);
    if (r == 0) return;
    z = __fmul_rn((float)r, s.scale);
  } else {
    z = __ldg(reinterpret_cast<const float*>(row) + x);
    if (z == 0.f) return;
  }
  const CameraDev& c = kTable ? cams[blockIdx.z] : colour;
  float xi[2], yi[2], zc[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const float px = __fadd_rn((float)x, k ? 0.5f : -0.5f), py = __fadd_rn((float)y, k ? 0.5f : -0.5f);
    const float X = __fmul_rn(__fdiv_rn(__fsub_rn(px, s.cx), s.fx), z);
    const float Y = __fmul_rn(__fdiv_rn(__fsub_rn(py, s.cy), s.fy), z);
    float P[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
      P[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(s.T[4 * r], X), __fmul_rn(s.T[4 * r + 1], Y)), __fmul_rn(s.T[4 * r + 2], z)),
                       s.T[4 * r + 3]);
    const float u = __fadd_rn(__fmul_rn(__fdiv_rn(P[0], P[2]), c.fx), c.cx);
    const float v = __fadd_rn(__fmul_rn(__fdiv_rn(P[1], P[2]), c.fy), c.cy);
    xi[k] = truncf(__fadd_rn(u, 0.5f));
    yi[k] = truncf(__fadd_rn(v, 0.5f));
    zc[k] = P[2];
  }
  // on the float values, so that NaN and values beyond int fail here
  if (!(zc[0] > 0.f && zc[1] > 0.f)) return;
  if (!(xi[0] >= 0.f && xi[0] <= xi[1] && xi[1] <= (float)(c.W - 1))) return;
  if (!(yi[0] >= 0.f && yi[0] <= yi[1] && yi[1] <= (float)(c.H - 1))) return;
  const unsigned int slot = aligned_slot_of(z);
  const int x0 = (int)xi[0], x1 = (int)xi[1], y0 = (int)yi[0], y1 = (int)yi[1];
  for (int yy = y0; yy <= y1; ++yy)
    for (int xx = x0; xx <= x1; ++xx) atomicMax(s.aligned + (size_t)yy * c.W + xx, slot);
}

int align_depth_launch(const SensorDev& s, const CameraDev& colour, cudaStream_t stream) {
  dim3 block(kAlW, kAlH), grid((s.W + kAlW - 1) / kAlW, (s.H + kAlH - 1) / kAlH);
  align_depth_kernel<false><<<grid, block, 0, stream>>>(s, colour, nullptr, nullptr);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

int align_depth_cameras_launch(const SensorDev* sensors, const CameraDev* cams, int C, int max_H, int max_W,
                               cudaStream_t stream) {
  dim3 block(kAlW, kAlH), grid((max_W + kAlW - 1) / kAlW, (max_H + kAlH - 1) / kAlH, C);
  align_depth_kernel<true><<<grid, block, 0, stream>>>(SensorDev{}, CameraDev{}, sensors, cams);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

// An aligned buffer of n slots to float32 metres in place (fp_align_depth)
__global__ void aligned_to_depth_kernel(unsigned int* __restrict__ buf, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) reinterpret_cast<float*>(buf)[i] = aligned_depth_of(buf[i]);
}

int aligned_to_depth_launch(unsigned int* buf, size_t n, cudaStream_t stream) {
  aligned_to_depth_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(buf, n);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

int erode_depth_launch(const float* depth, float* out, int H, int W, int radius, float diff_thres, float ratio_thres,
                       float zfar, cudaStream_t stream) {
  dim3 block(32, 8), grid((W + 31) / 32, (H + 7) / 8);
  erode_depth_kernel<<<grid, block, 0, stream>>>(depth, out, H, W, radius, diff_thres, ratio_thres, zfar);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

int bilateral_depth_launch(const float* depth, float* out, int H, int W, int radius, float zfar, float sigmaD,
                           float sigmaR, cudaStream_t stream) {
  dim3 block(32, 8), grid((W + 31) / 32, (H + 7) / 8);
  bilateral_depth_kernel<<<grid, block, 0, stream>>>(depth, out, H, W, radius, zfar, sigmaD, sigmaR);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace fp

// ------------------------------------------------------------------------------------------------
// start poses on the device: guess_translation (estimater.py:137-156) + rot_grid with that translation
// (estimater.py:127-134, :203-209).  The median of the masked valid depths is an exact radix
// select over the float bit patterns (depths are positive, so the patterns are ordered), np.median's
// mean of the two middle elements for an even count included.
// ------------------------------------------------------------------------------------------------
namespace fp {

__device__ unsigned int radix_select(const float* __restrict__ depth, const unsigned char* __restrict__ mask, int W,
                                     int u0, int v0, int bw, int bh, unsigned int k, unsigned int* hist /*smem[256]*/,
                                     unsigned int* sh /*smem[2]*/) {
  // returns the bit pattern of the k-th smallest (0-based) valid masked depth; only the mask's bounding box
  // (u0, v0, bw x bh) is scanned
  unsigned int prefix = 0, prefix_mask = 0;
  const int nbox = bw * bh;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int q = threadIdx.x; q < nbox; q += blockDim.x) {
      const int i = (v0 + q / bw) * W + u0 + q % bw;
      const float d = depth[i];
      if (mask[i] && d >= 0.001f) {
        const unsigned int b = __float_as_uint(d);
        if ((b & prefix_mask) == prefix) atomicAdd(&hist[(b >> shift) & 255u], 1u);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned int acc = 0, bin = 0;
      for (; bin < 256; ++bin) {
        if (acc + hist[bin] > k) break;
        acc += hist[bin];
      }
      sh[0] = bin;
      sh[1] = k - acc;
    }
    __syncthreads();
    prefix |= sh[0] << shift;
    prefix_mask |= 255u << shift;
    k = sh[1];
    __syncthreads();
  }
  return prefix;
}

// pass 1 (grid-wide, one grid row per object): mask bounding box and pixel counts.  All six statistics are max / sum
// reductions over values that start at 0 (the box minima are stored mirrored), so one memset of 6 words per object
// initialises them.  Object m reads masks[m] ([H][W]) and writes stats[6 m, 6 m + 6).
// The filtered depth and H x W come from `one` (by value), or with kTable (fp_register_cameras) from entry camera_of[m]
// of the device table `cams`; object m's mask ([H][W] of its camera) then starts at byte mask_off[m] of `masks`.
template <bool kTable>
__global__ void __launch_bounds__(256) mask_stats_kernel(const CameraDev one, const unsigned char* __restrict__ masks,
                                                         unsigned int* __restrict__ stats,
                                                         const CameraDev* __restrict__ cams,
                                                         const int* __restrict__ camera_of,
                                                         const size_t* __restrict__ mask_off) {
  const CameraDev cam = kTable ? cams[camera_of[blockIdx.y]] : one;
  const float* depth = cam.depth;
  const int H = cam.H, W = cam.W;
  const int npix = H * W;
  const unsigned char* mask = masks + (kTable ? mask_off[blockIdx.y] : (size_t)blockIdx.y * npix);
  stats += 6 * blockIdx.y;
  unsigned int mu0 = 0, u1 = 0, mv0 = 0, v1 = 0, n_mask = 0, n_valid = 0;  // mu0 = W - 1 - umin, mv0 = H - 1 - vmin
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += gridDim.x * blockDim.x) {
    if (mask[i]) {
      const int v = i / W, u = i - v * W;
      mu0 = max(mu0, (unsigned)(W - 1 - u) + 1u);  // +1: 0 stays "no pixel"
      u1 = max(u1, (unsigned)u + 1u);
      mv0 = max(mv0, (unsigned)(H - 1 - v) + 1u);
      v1 = max(v1, (unsigned)v + 1u);
      ++n_mask;
      if (depth[i] >= 0.001f) ++n_valid;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mu0 = max(mu0, __shfl_xor_sync(0xffffffffu, mu0, o));
    u1 = max(u1, __shfl_xor_sync(0xffffffffu, u1, o));
    mv0 = max(mv0, __shfl_xor_sync(0xffffffffu, mv0, o));
    v1 = max(v1, __shfl_xor_sync(0xffffffffu, v1, o));
    n_mask += __shfl_xor_sync(0xffffffffu, n_mask, o);
    n_valid += __shfl_xor_sync(0xffffffffu, n_valid, o);
  }
  if ((threadIdx.x & 31) == 0 && n_mask) {
    atomicMax(&stats[0], mu0);
    atomicMax(&stats[1], u1);
    atomicMax(&stats[2], mv0);
    atomicMax(&stats[3], v1);
    atomicAdd(&stats[4], n_mask);
    atomicAdd(&stats[5], n_valid);
  }
}

// pass 2 (one CTA per object): exact median over the object's bounding box, translation, start poses.  Object m owns
// rows [off[m], off[m + 1]) of the concatenated rotation grids and start poses (off = null: one object, rows [0, N)),
// and writes info[4 m, 4 m + 4).  The object's frame (depth, H x W, fx fy cx cy) and mask as in mask_stats_kernel.
template <bool kTable>
__global__ void __launch_bounds__(1024) start_poses_kernel(const CameraDev one, const unsigned char* __restrict__ masks,
                                                           const float* __restrict__ rot_grid, int N,
                                                           const int* __restrict__ off,
                                                           const unsigned int* __restrict__ stats,
                                                           float* __restrict__ poses_out, float* __restrict__ info,
                                                           const CameraDev* __restrict__ cams,
                                                           const int* __restrict__ camera_of,
                                                           const size_t* __restrict__ mask_off) {
  __shared__ unsigned int hist[256];
  __shared__ unsigned int sh[2];
  __shared__ float tvec[3];
  const int m = blockIdx.x;
  const CameraDev cam = kTable ? cams[camera_of[m]] : one;
  const float* depth = cam.depth;
  const int H = cam.H, W = cam.W;
  const float fx = cam.fx, fy = cam.fy, cx = cam.cx, cy = cam.cy;
  const unsigned char* mask = masks + (kTable ? mask_off[m] : (size_t)m * H * W);
  stats += 6 * m;
  info += 4 * m;
  const int row0 = off ? off[m] : 0;
  const int n = off ? off[m + 1] - row0 : N;
  rot_grid += (size_t)row0 * 16;
  poses_out += (size_t)row0 * 16;
  const unsigned int nm = stats[4], nv = stats[5];
  // umin, umax, vmin, vmax
  const int bb[4] = {W - (int)stats[0], (int)stats[1] - 1, H - (int)stats[2], (int)stats[3] - 1};
  float zc = 0.f;
  if (nm > 0 && nv > 0) {  // uniform branch
    const int u0 = bb[0], v0 = bb[2], bw = bb[1] - bb[0] + 1, bh = bb[3] - bb[2] + 1;
    const unsigned int lo = radix_select(depth, mask, W, u0, v0, bw, bh, (nv - 1) / 2, hist, sh);
    const unsigned int hi = (nv & 1u) ? lo : radix_select(depth, mask, W, u0, v0, bw, bh, nv / 2, hist, sh);
    zc = (nv & 1u) ? __uint_as_float(lo) : (__uint_as_float(lo) + __uint_as_float(hi)) * 0.5f;
  }
  if (threadIdx.x == 0) {
    double t[3] = {0.0, 0.0, 0.0};
    if (nm > 0 && nv > 0) {
      const double uc = (bb[0] + bb[1]) / 2.0, vc = (bb[2] + bb[3]) / 2.0;
      // np.linalg.inv(K) @ [uc, vc, 1] * zc  for K = [[fx,0,cx],[0,fy,cy],[0,0,1]]
      t[0] = (uc - (double)cx) / (double)fx * (double)zc;
      t[1] = (vc - (double)cy) / (double)fy * (double)zc;
      t[2] = (double)zc;
    }
    tvec[0] = (float)t[0]; tvec[1] = (float)t[1]; tvec[2] = (float)t[2];
    info[0] = tvec[0]; info[1] = tvec[1]; info[2] = tvec[2]; info[3] = (float)nv;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n * 16; i += blockDim.x) {
    const int e = i & 15;
    float v = rot_grid[i];
    if (e == 3) v = tvec[0];
    else if (e == 7) v = tvec[1];
    else if (e == 11) v = tvec[2];
    poses_out[i] = v;
  }
}

int start_poses_launch(const CameraDev& one, const CameraDev* cams, const int* camera_of, const unsigned char* masks,
                       const size_t* mask_off, const float* rot_grid, int N, int M, const int* off, unsigned int* stats,
                       float* poses_out, float* info, cudaStream_t stream) {
  FP_REQUIRE(M >= 1 && M <= 65535 && (off || (M == 1 && !cams)), "start_poses: bad object count %d", M);
  FP_CUDA_OK(cudaMemsetAsync(stats, 0, (size_t)M * 6 * sizeof(unsigned int), stream));
  const auto stats_kernel = cams ? mask_stats_kernel<true> : mask_stats_kernel<false>;
  const auto poses_kernel = cams ? start_poses_kernel<true> : start_poses_kernel<false>;
  stats_kernel<<<dim3(num_sms(), M), 256, 0, stream>>>(one, masks, stats, cams, camera_of, mask_off);
  poses_kernel<<<M, 1024, 0, stream>>>(one, masks, rot_grid, N, off, stats, poses_out, info, cams, camera_of, mask_off);
  note_launches(2);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace fp
