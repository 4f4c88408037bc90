// fp_api_ops.cu — C-ABI entry points that expose single operators (used by the parity tests to
// bisect the pipeline layer by layer; the product entry points live in fp_api.cu).
#include "../../include/fpose.h"
#include "fp_common.cuh"
#include "fp_attn.cuh"
#include "fp_crop.cuh"
#include "fp_ctx.cuh"
#include "fp_depth.cuh"
#include "fp_gemm.cuh"

#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

namespace fp {
const char* get_last_error();
int prof_collect(int kind, double* total_ms, double* total_work, int* launches);
int pose_errors_launch(const float* pts, int P, const float* pred, int N, const float* gt, int n_gt, float* add_out,
                       float* adds_out, cudaStream_t stream);
int sym_pose_errors_launch(const float* pts, int P, const float* pred, int N, const float* gt, int n_gt, const float* sym,
                           int S, const float* K, int n_K, float* mssd_out, float* mspd_out, cudaStream_t stream);

int vsd_errors_launch(const float* pos, int V, const int* faces, int F, const float* pred, int N, const float* gt,
                      int n_gt, const float* depth, int n_depth, int H, int W, const float* K, int n_K, float delta,
                      const float* taus, int T, float* errs_out, int* counts_out, cudaStream_t stream);

int check_device_ptr(const void* p, const char* what, const char* fn) {
  int dev = 0;
  FP_CUDA_OK(cudaGetDevice(&dev));
  cudaPointerAttributes a;
  const cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) {
    cudaGetLastError();  // not sticky; keep it out of the next caller's error check
    fp::set_last_error("%s: %s: cudaPointerGetAttributes failed (%s)", fn, what, cudaGetErrorString(e));
    return -1;
  }
  if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) {
    fp::set_last_error("%s: %s is not device memory", fn, what);
    return -1;
  }
  if (a.type == cudaMemoryTypeDevice && a.device != dev) {
    fp::set_last_error("%s: %s lives on device %d, the current device is %d", fn, what, a.device, dev);
    return -1;
  }
  return 0;
}
}  // namespace fp

using namespace fp;

extern "C" {

const char* fp_last_error(void) { return fp::get_last_error(); }

unsigned long long fp_launch_count(void) { return fp::launch_count(); }

int fp_prof_enable(int on) {
  fp::g_prof_on = on != 0;
  return 0;
}

int fp_prof_collect(int kind, double* total_ms, double* total_work, int* launches) {
  FP_API_BEGIN
  if (!total_ms || !total_work || !launches) {
    fp::set_last_error("fp_prof_collect: null output");
    return -1;
  }
  return fp::prof_collect(kind, total_ms, total_work, launches);
  FP_API_END
}

int fp_op_build_meshlets(int V, int F, const float* pos, const int* faces, int* info, int* face_of_tri_out,
                         float* meshlets_out) {
  FP_API_BEGIN
  if (!pos || !faces || !info || V <= 0 || F <= 0) {
    fp::set_last_error("fp_op_build_meshlets: bad argument");
    return -1;
  }
  for (int i = 0; i < 3 * F; ++i)
    if (faces[i] < 0 || faces[i] >= V) {
      fp::set_last_error("fp_op_build_meshlets: face index out of range");
      return -1;
    }
  std::vector<float> nrm((size_t)V * 3, 0.f), att((size_t)V * 3, 0.f);
  fp::MeshHost mh;
  int rc = fp::build_mesh_host(V, F, pos, nrm.data(), att.data(), 3, faces, mh);
  if (rc) return rc;
  int max_t = 0, max_v = 0, total = 0;
  for (const fp::Meshlet& m : mh.meshlets) {
    max_t = m.n_tris > max_t ? m.n_tris : max_t;
    max_v = m.n_verts > max_v ? m.n_verts : max_v;
    total += m.n_tris;
    for (int t = 0; t < m.n_tris; ++t) {
      const uint2 tr = mh.ml_tris[m.tri_off + t];
      for (int k = 0; k < 3; ++k) {
        const int slot = (tr.x >> (8 * k)) & 255;
        if (slot >= m.n_verts || mh.ml_verts[m.vert_off + slot] != faces[3 * tr.y + k]) {
          fp::set_last_error("fp_op_build_meshlets: meshlet triangle does not map back to its face");
          return -4;
        }
        // every vertex of the meshlet lies inside its bounding sphere
        const float* q = pos + 3 * faces[3 * tr.y + k];
        const float dx = q[0] - m.cx, dy = q[1] - m.cy, dz = q[2] - m.cz;
        if (dx * dx + dy * dy + dz * dz > m.r * m.r * 1.0001f + 1e-12f) {
          fp::set_last_error("fp_op_build_meshlets: vertex outside the meshlet's bounding sphere");
          return -4;
        }
      }
      if (face_of_tri_out) face_of_tri_out[m.tri_off + t] = (int)tr.y;
    }
  }
  if (meshlets_out)
    for (size_t i = 0; i < mh.meshlets.size(); ++i) {
      const fp::Meshlet& m = mh.meshlets[i];
      const float rec[8] = {m.cx, m.cy, m.cz, m.r, m.ax, m.ay, m.az, m.cutoff};
      for (int k = 0; k < 8; ++k) meshlets_out[8 * i + k] = rec[k];
    }
  info[0] = (int)mh.meshlets.size();
  info[1] = mh.closed;
  info[2] = mh.front_sign;
  info[3] = max_t;
  info[4] = max_v;
  info[5] = total;
  return 0;
  FP_API_END
}

int fp_op_meshlet_sizes(int V, int F, const float* pos, const int* faces, int* tris_of_meshlet_out) {
  FP_API_BEGIN
  if (!pos || !faces || !tris_of_meshlet_out || V <= 0 || F <= 0) {
    fp::set_last_error("fp_op_meshlet_sizes: bad argument");
    return -1;
  }
  for (int i = 0; i < 3 * F; ++i)
    if (faces[i] < 0 || faces[i] >= V) {
      fp::set_last_error("fp_op_meshlet_sizes: face index out of range");
      return -1;
    }
  std::vector<float> nrm((size_t)V * 3, 0.f), att((size_t)V * 3, 0.f);
  fp::MeshHost mh;
  int rc = fp::build_mesh_host(V, F, pos, nrm.data(), att.data(), 3, faces, mh);
  if (rc) return rc;
  for (size_t i = 0; i < mh.meshlets.size(); ++i) tris_of_meshlet_out[i] = mh.meshlets[i].n_tris;
  return (int)mh.meshlets.size();
  FP_API_END
}

int fp_op_attention(const void* qkv, void* out, int B, int impl, void* stream) {
  FP_API_BEGIN
  if (!qkv || !out) {
    fp::set_last_error("fp_op_attention: null argument");
    return -1;
  }
  (void)impl;  // one implementation: the wgmma kernel
  return fp::attn_tc_launch(
      fp::head_attn_params(reinterpret_cast<const __half*>(qkv), 1536, 1, reinterpret_cast<__half*>(out), B),
      reinterpret_cast<cudaStream_t>(stream));
  FP_API_END
}

// 0 when `p` is device memory of the current device aligned to the 16 bytes of the kernels' uint4 / float4 loads
static int check_dev16(const void* p, const char* what, const char* fn) {
  FP_REQUIRE(p, "%s: %s is null", fn, what);
  FP_REQUIRE(reinterpret_cast<uintptr_t>(p) % 16 == 0, "%s: %s is not 16-byte aligned", fn, what);
  return check_device_ptr(p, what, fn);
}

int fp_op_attention_groups(const void* qkv, int ld, int n_groups, void* out, int B, void* stream) {
  FP_API_BEGIN
  const char* fn = "fp_op_attention_groups";
  FP_REQUIRE(n_groups == 1 || n_groups == 2, "%s: n_groups = %d, must be 1 or 2", fn, n_groups);
  FP_REQUIRE(ld >= 1536 * n_groups && ld % 8 == 0, "%s: ld = %d, must be a multiple of 8 and >= %d", fn, ld, 1536 * n_groups);
  FP_REQUIRE(B >= 0 && B <= FP_OP_MAX_SEQUENCES, "%s: B = %d outside [0, %d]", fn, B, FP_OP_MAX_SEQUENCES);
  if (check_dev16(qkv, "qkv", fn) || check_dev16(out, "out", fn)) return -1;
  return fp::attn_core_launch(
      fp::head_attn_params(reinterpret_cast<const __half*>(qkv), ld, n_groups, reinterpret_cast<__half*>(out), B),
      reinterpret_cast<cudaStream_t>(stream));
  FP_API_END
}

int fp_op_layernorm(const void* x, void* y, const float* gamma, const float* beta, int rows, void* stream) {
  FP_API_BEGIN
  const char* fn = "fp_op_layernorm";
  FP_REQUIRE(rows >= 0 && rows <= FP_OP_MAX_SEQUENCES * 400, "%s: rows = %d outside [0, %d]", fn, rows,
             FP_OP_MAX_SEQUENCES * 400);
  if (check_dev16(x, "x", fn) || check_dev16(y, "y", fn) || check_dev16(gamma, "gamma", fn) || check_dev16(beta, "beta", fn))
    return -1;
  return fp::layernorm_launch(reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), gamma, beta, rows,
                              reinterpret_cast<cudaStream_t>(stream));
  FP_API_END
}

int fp_op_head_final(const void* x, const float* gamma, const float* beta, const float* w, const float* bias, float* out,
                     int B, int out_dim, void* stream) {
  FP_API_BEGIN
  const char* fn = "fp_op_head_final";
  FP_REQUIRE(B >= 0 && B <= FP_OP_MAX_SEQUENCES, "%s: B = %d outside [0, %d]", fn, B, FP_OP_MAX_SEQUENCES);
  FP_REQUIRE(out_dim >= 1 && out_dim <= 8, "%s: out_dim = %d outside [1, 8]", fn, out_dim);
  if (check_dev16(x, "x", fn) || check_dev16(gamma, "gamma", fn) || check_dev16(beta, "beta", fn)) return -1;
  FP_REQUIRE(w && bias && out, "%s: null w, bias or out", fn);
  if (check_device_ptr(w, "w", fn) || check_device_ptr(bias, "bias", fn) || check_device_ptr(out, "out", fn)) return -1;
  return fp::head_final_launch(reinterpret_cast<const __half*>(x), gamma, beta, w, bias, out, B, 400, out_dim,
                               reinterpret_cast<cudaStream_t>(stream));
  FP_API_END
}

int fp_op_token_mean_proj(const void* x, const float* w_f32, const float* bias, float* mean_ws, float* out, int B,
                          void* stream) {
  FP_API_BEGIN
  const char* fn = "fp_op_token_mean_proj";
  FP_REQUIRE(B >= 0 && B <= FP_OP_MAX_SEQUENCES, "%s: B = %d outside [0, %d]", fn, B, FP_OP_MAX_SEQUENCES);
  if (check_dev16(x, "x", fn) || check_dev16(w_f32, "w_f32", fn) || check_dev16(mean_ws, "mean_ws", fn)) return -1;
  FP_REQUIRE(bias && out, "%s: null bias or out", fn);
  if (check_device_ptr(bias, "bias", fn) || check_device_ptr(out, "out", fn)) return -1;
  return fp::token_mean_proj_launch(reinterpret_cast<const __half*>(x), w_f32, bias, mean_ws, out, B, 400,
                                    reinterpret_cast<cudaStream_t>(stream));
  FP_API_END
}

static fp::GemmLayer to_gemm_layer(const fp_gemm_layer_t* l) {
  fp::GemmLayer L;
  L.kind = l->kind;
  L.n_img = l->n_img;
  L.Hin = l->Hin;
  L.Win = l->Win;
  L.Cin = l->Cin;
  L.Cout = l->Cout;
  L.in = l->in;
  L.w = l->w;
  L.bias = l->bias;
  L.res = l->res;
  L.res_ld = l->res_ld;
  L.out = l->out;
  L.out_ld = l->out_ld;
  L.out_split = l->out_split;
  L.post_add = l->post_add;
  L.relu = l->relu;
  return L;
}

int fp_op_gemm_layer(const fp_gemm_layer_t* l, void* stream) {
  FP_API_BEGIN
  if (!l) {
    fp::set_last_error("fp_op_gemm_layer: null layer");
    return -1;
  }
  return fp::gemm_layer_launch(to_gemm_layer(l), reinterpret_cast<cudaStream_t>(stream));
  FP_API_END
}

int fp_op_gemm_tile_n(const fp_gemm_layer_t* l, int* tile_n) {
  FP_API_BEGIN
  if (!l || !tile_n) {
    fp::set_last_error("fp_op_gemm_tile_n: null argument");
    return -1;
  }
  return fp::gemm_layer_tile_n(to_gemm_layer(l), tile_n);
  FP_API_END
}

int fp_op_gemm_tile_m(const fp_gemm_layer_t* l, int* tile_m) {
  FP_API_BEGIN
  if (!l || !tile_m) {
    fp::set_last_error("fp_op_gemm_tile_m: null argument");
    return -1;
  }
  return fp::gemm_layer_tile_m(to_gemm_layer(l), tile_m);
  FP_API_END
}

int fp_pose_errors(const float* pts, int P, const float* pred, int N, const float* gt, int n_gt, float* add_out,
                   float* adds_out, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(P >= 1 && P <= FP_METRICS_MAX_POINTS, "fp_pose_errors: P = %d outside [1, %d]", P, FP_METRICS_MAX_POINTS);
  FP_REQUIRE(N >= 0 && N <= FP_METRICS_MAX_POSES, "fp_pose_errors: N = %d outside [0, %d]", N, FP_METRICS_MAX_POSES);
  FP_REQUIRE(n_gt == 1 || n_gt == N, "fp_pose_errors: n_gt = %d, must be 1 or N = %d", n_gt, N);
  if (N == 0) return 0;
  FP_REQUIRE(pts && pred && gt, "fp_pose_errors: null input pointer");
  const void* ptrs[5] = {pts, pred, gt, add_out, adds_out};
  const char* names[5] = {"pts", "pred", "gt", "add_out", "adds_out"};
  for (int i = 0; i < 5; ++i)
    if (ptrs[i] && check_device_ptr(ptrs[i], names[i])) return -1;
  return fp::pose_errors_launch(pts, P, pred, N, gt, n_gt, add_out, adds_out, reinterpret_cast<cudaStream_t>(stream));
  FP_API_END
}

int fp_align_depth(const void* depth, int depth_format, float depth_scale, long long depth_pitch, const fp_depth_sensor_t* s,
                   const float* K_color, int H, int W, float* out, void* stream) {
  FP_API_BEGIN
  const char* fn = "fp_align_depth";
  FP_REQUIRE(depth && s && K_color && out, "%s: null argument", fn);
  FP_TRY(check_depth_sensor(s, fn));
  FP_REQUIRE(depth_format == FP_DEPTH_F32 || depth_format == FP_DEPTH_U16, "%s: unknown depth format %d", fn, depth_format);
  FP_REQUIRE(depth_format != FP_DEPTH_U16 || (isfinite(depth_scale) && depth_scale > 0.f),
             "%s: uint16 depth scale %g must be finite and > 0 (metres per unit)", fn, (double)depth_scale);
  FP_REQUIRE(H >= 1 && W >= 1 && (long long)H * W <= 0x7fffffffLL, "%s: colour frame %d x %d is empty or too large", fn, H,
             W);
  {
    // K_color is read on the host
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, K_color) != cudaSuccess)
      cudaGetLastError();
    else
      FP_REQUIRE(a.type != cudaMemoryTypeDevice, "%s: K_color is device memory; it is read on the host", fn);
  }
  for (int k = 0; k < 9; ++k) FP_REQUIRE(isfinite(K_color[k]), "%s: K_color[%d] = %g is not finite", fn, k, (double)K_color[k]);
  const int bpp = depth_format == FP_DEPTH_U16 ? 2 : 4;
  const long long row = (long long)s->W * bpp, pitch = depth_pitch ? depth_pitch : row;
  FP_REQUIRE(pitch >= row && pitch <= 0x7fffffffLL, "%s: depth pitch %lld bytes is below the %lld bytes of a row or too large", fn,
             pitch, row);
  FP_REQUIRE(pitch % bpp == 0, "%s: depth pitch %lld bytes is not a multiple of the %d-byte depth value", fn, pitch, bpp);
  FP_REQUIRE(reinterpret_cast<uintptr_t>(depth) % bpp == 0, "%s: depth buffer %p is not aligned to its %d-byte depth value", fn,
             depth, bpp);
  FP_REQUIRE(reinterpret_cast<uintptr_t>(out) % 4 == 0, "%s: out %p is not aligned to 4 bytes", fn, (const void*)out);
  if (check_device_ptr(depth, "depth", fn) || check_device_ptr(out, "out", fn)) return -1;
  SensorDev d;
  memset(&d, 0, sizeof d);
  d.depth = depth;
  d.aligned = reinterpret_cast<unsigned int*>(out);
  d.pitch = (int)pitch;
  d.u16 = depth_format == FP_DEPTH_U16 ? 1 : 0;
  d.scale = d.u16 ? depth_scale : 0.f;
  d.H = s->H;
  d.W = s->W;
  d.fx = s->K[0];
  d.fy = s->K[4];
  d.cx = s->K[2];
  d.cy = s->K[5];
  for (int k = 0; k < 12; ++k) d.T[k] = s->T_color_from_depth[k];
  CameraDev colour;  // the colour frame's size and intrinsics, as a call's K gives them
  memset(&colour, 0, sizeof colour);
  colour.fx = K_color[0];
  colour.fy = K_color[4];
  colour.cx = K_color[2];
  colour.cy = K_color[5];
  colour.H = H;
  colour.W = W;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t npix = (size_t)H * W;
  FP_CUDA_OK(cudaMemsetAsync(out, 0, npix * 4, st));
  FP_TRY(align_depth_launch(d, colour, st));
  return aligned_to_depth_launch(d.aligned, npix, st);
  FP_API_END
}

int fp_sym_pose_errors(const float* pts, int P, const float* pred, int N, const float* gt, int n_gt, const float* sym,
                       int S, const float* K, int n_K, float* mssd_out, float* mspd_out, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(P >= 1 && P <= FP_METRICS_MAX_POINTS, "fp_sym_pose_errors: P = %d outside [1, %d]", P, FP_METRICS_MAX_POINTS);
  FP_REQUIRE(N >= 0 && N <= FP_METRICS_MAX_POSES, "fp_sym_pose_errors: N = %d outside [0, %d]", N, FP_METRICS_MAX_POSES);
  FP_REQUIRE(S >= 1 && S <= FP_METRICS_MAX_SYMMETRIES, "fp_sym_pose_errors: S = %d outside [1, %d]", S,
             FP_METRICS_MAX_SYMMETRIES);
  FP_REQUIRE(n_gt == 1 || n_gt == N, "fp_sym_pose_errors: n_gt = %d, must be 1 or N = %d", n_gt, N);
  if (mspd_out) FP_REQUIRE(n_K == 1 || n_K == N, "fp_sym_pose_errors: n_K = %d, must be 1 or N = %d", n_K, N);
  if (N == 0) return 0;
  FP_REQUIRE(pts && pred && gt && sym, "fp_sym_pose_errors: null input pointer");
  FP_REQUIRE(K || !mspd_out, "fp_sym_pose_errors: mspd_out needs K");
  const void* ptrs[7] = {pts, pred, gt, sym, mspd_out ? K : nullptr, mssd_out, mspd_out};
  const char* names[7] = {"pts", "pred", "gt", "sym", "K", "mssd_out", "mspd_out"};
  for (int i = 0; i < 7; ++i)
    if (ptrs[i] && check_device_ptr(ptrs[i], names[i], "fp_sym_pose_errors")) return -1;
  return fp::sym_pose_errors_launch(pts, P, pred, N, gt, n_gt, sym, S, K, n_K, mssd_out, mspd_out,
                                    reinterpret_cast<cudaStream_t>(stream));
  FP_API_END
}

int fp_vsd_errors(const float* pos, int V, const int* faces, int F, const float* pred, int N, const float* gt, int n_gt,
                  const float* depth, int n_depth, int H, int W, const float* K, int n_K, float delta, const float* taus,
                  int T, float* errs_out, int* counts_out, void* stream) {
  FP_API_BEGIN
  const char* fn = "fp_vsd_errors";
  FP_REQUIRE(V >= 3 && V <= FP_VSD_MAX_VERTICES, "%s: V = %d outside [3, %d]", fn, V, FP_VSD_MAX_VERTICES);
  FP_REQUIRE(F >= 1 && F <= FP_VSD_MAX_FACES, "%s: F = %d outside [1, %d]", fn, F, FP_VSD_MAX_FACES);
  FP_REQUIRE(N >= 0 && N <= FP_METRICS_MAX_POSES, "%s: N = %d outside [0, %d]", fn, N, FP_METRICS_MAX_POSES);
  FP_REQUIRE(n_gt == 1 || n_gt == N, "%s: n_gt = %d, must be 1 or N = %d", fn, n_gt, N);
  FP_REQUIRE(n_depth == 1 || n_depth == N, "%s: n_depth = %d, must be 1 or N = %d", fn, n_depth, N);
  FP_REQUIRE(n_K == 1 || n_K == N, "%s: n_K = %d, must be 1 or N = %d", fn, n_K, N);
  FP_REQUIRE(H >= 1 && H <= FP_VSD_MAX_DIM && W >= 1 && W <= FP_VSD_MAX_DIM, "%s: H x W = %d x %d outside [1, %d]", fn, H,
             W, FP_VSD_MAX_DIM);
  FP_REQUIRE(T >= 1 && T <= FP_VSD_MAX_TAUS, "%s: T = %d outside [1, %d]", fn, T, FP_VSD_MAX_TAUS);
  FP_REQUIRE(delta >= 0.f && delta < INFINITY, "%s: delta = %g must be finite and >= 0", fn, (double)delta);
  FP_REQUIRE(pos && faces, "%s: null mesh pointer", fn);
  {
    // the mesh comes as host arrays: a device pointer here would be read by the host
    const void* hp[2] = {pos, faces};
    const char* hn[2] = {"pos", "faces"};
    for (int i = 0; i < 2; ++i) {
      cudaPointerAttributes a;
      if (cudaPointerGetAttributes(&a, hp[i]) != cudaSuccess) {
        cudaGetLastError();
        continue;
      }
      FP_REQUIRE(a.type != cudaMemoryTypeDevice, "%s: %s is device memory; the mesh is read on the host", fn, hn[i]);
    }
  }
  for (long long i = 0; i < 3LL * F; ++i)
    FP_REQUIRE(faces[i] >= 0 && faces[i] < V, "%s: faces[%lld] = %d outside [0, %d)", fn, i / 3, faces[i], V);
  if (N == 0) return 0;
  FP_REQUIRE(pred && gt && depth && K && taus && errs_out, "%s: null input or output pointer", fn);
  const void* ptrs[7] = {pred, gt, depth, K, taus, errs_out, counts_out};
  const char* names[7] = {"pred", "gt", "depth", "K", "taus", "errs_out", "counts_out"};
  for (int i = 0; i < 7; ++i)
    if (ptrs[i] && check_device_ptr(ptrs[i], names[i], fn)) return -1;
  return fp::vsd_errors_launch(pos, V, faces, F, pred, N, gt, n_gt, depth, n_depth, H, W, K, n_K, delta, taus, T,
                               errs_out, counts_out, reinterpret_cast<cudaStream_t>(stream));
  FP_API_END
}

int fp_op_refine_net(fp_ctx* c, const void* crops, int N, float* trans_out, float* rot_out, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && crops && trans_out && rot_out, "fp_op_refine_net: null argument");
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  if (N == 0) return 0;
  FP_TRY(ensure_capacity(c, N));
  FP_TRY(crops_import(c, crops, N, st));
  FP_TRY(run_encoder(c, c->net[0], reinterpret_cast<const __half*>(c->crops.p), N, st));
  FP_TRY(run_refine_heads(c, c->net[0], N, st));
  const float* ho = reinterpret_cast<const float*>(c->head_out.p);
  FP_CUDA_OK(cudaMemcpyAsync(trans_out, ho, (size_t)N * 12, cudaMemcpyDeviceToDevice, st));
  FP_CUDA_OK(cudaMemcpyAsync(rot_out, ho + (size_t)N * 3, (size_t)N * 12, cudaMemcpyDeviceToDevice, st));
  return 0;
  FP_API_END
}

int fp_op_score_feats(fp_ctx* c, const void* crops, int N, float* feats_out, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && crops && feats_out, "fp_op_score_feats: null argument");
  FP_REQUIRE(c->net[1].loaded, "scorer weights not loaded");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  if (N == 0) return 0;
  FP_TRY(ensure_capacity(c, N));
  FP_TRY(crops_import(c, crops, N, st));
  FP_TRY(run_encoder(c, c->net[1], reinterpret_cast<const __half*>(c->crops.p), N, st));
  FP_TRY(run_score_feats(c, c->net[1], N, feats_out, st));
  return 0;
  FP_API_END
}

int fp_op_encoder_layer(int layer, int N, int* info) {
  FP_API_BEGIN
  FP_REQUIRE(info, "fp_op_encoder_layer: null info");
  FP_REQUIRE(layer >= 0 && layer < kEncLayers, "fp_op_encoder_layer: layer = %d outside [0, %d]", layer, kEncLayers - 1);
  FP_REQUIRE(N >= 0 && N <= kRegisterPassCap, "fp_op_encoder_layer: N = %d outside [0, %d]", N, kRegisterPassCap);
  const EncLayer& l = kEncoder[layer];
  const int Np = b_img0_of(N);
  info[0] = l.kind;
  info[1] = l.ab_batch ? Np + N : N;
  info[2] = l.H;
  info[3] = l.Cin;
  info[4] = l.Cout;
  info[5] = enc_source(layer, l.in);
  info[6] = l.res == EB_NONE ? -1 : enc_source(layer, l.res);
  info[7] = l.split ? Np : 0;
  info[8] = l.pe ? 1 : 0;
  enc_out_shape(layer, N, info + 9);
  return 0;
  FP_API_END
}

long long fp_op_encoder(fp_ctx* c, int which, const void* crops, int N, int last, void* out, void* stream) {
  FP_API_BEGIN
  const char* fn = "fp_op_encoder";
  FP_REQUIRE(c, "%s: null context", fn);
  FP_REQUIRE(which == 0 || which == 1, "%s: which = %d, must be 0 (refiner) or 1 (scorer)", fn, which);
  FP_REQUIRE(last >= 0 && last < kEncLayers, "%s: last = %d outside [0, %d]", fn, last, kEncLayers - 1);
  FP_REQUIRE(N >= 0 && N <= kRegisterPassCap, "%s: N = %d outside [0, %d]", fn, N, kRegisterPassCap);
  FP_REQUIRE(crops && out, "%s: null crops or out", fn);
  FP_REQUIRE(c->net[which].loaded, "%s: %s weights not loaded", fn, which == 0 ? "refiner" : "scorer");
  DeviceGuard dg(c->device);
  if (check_device_ptr(crops, "crops", fn) || check_device_ptr(out, "out", fn)) return -1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  if (N == 0) return 0;
  int shape[4];
  enc_out_shape(last, N, shape);
  const size_t bytes = (size_t)shape[0] * shape[1] * shape[2] * shape[3] * 2;
  FP_TRY(ensure_capacity(c, N));
  FP_TRY(crops_import(c, crops, N, st));
  FP_TRY(run_encoder(c, c->net[which], reinterpret_cast<const __half*>(c->crops.p), N, st, last));
  FP_CUDA_OK(cudaMemcpyAsync(out, enc_buf(c, nullptr, kEncoder[last].out), bytes, cudaMemcpyDeviceToDevice, st));
  return (long long)bytes;
  FP_API_END
}

long long fp_op_heads(fp_ctx* c, int which, const void* tok, int N, int stage, void* out, void* stream) {
  FP_API_BEGIN
  const char* fn = "fp_op_heads";
  FP_REQUIRE(c, "%s: null context", fn);
  FP_REQUIRE(which == 0 || which == 1, "%s: which = %d, must be 0 (refiner) or 1 (scorer)", fn, which);
  const int stages = which == 0 ? 7 : 4;
  FP_REQUIRE(stage >= 0 && stage < stages, "%s: stage = %d outside [0, %d]", fn, stage, stages - 1);
  FP_REQUIRE(N >= 1 && N <= kRegisterPassCap, "%s: N = %d outside [1, %d]", fn, N, kRegisterPassCap);
  FP_REQUIRE(tok && out, "%s: null tok or out", fn);
  FP_REQUIRE(c->net[which].loaded, "%s: %s weights not loaded", fn, which == 0 ? "refiner" : "scorer");
  DeviceGuard dg(c->device);
  if (check_device_ptr(tok, "tok", fn) || check_device_ptr(out, "out", fn)) return -1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  FP_TRY(ensure_capacity(c, N));  // may reallocate: the buffers are looked up after it
  const size_t M = (size_t)N * T;
  FP_CUDA_OK(cudaMemcpyAsync(c->tok.p, tok, M * 512 * 2, cudaMemcpyDeviceToDevice, st));
  const void* src;
  size_t bytes;
  if (which == 0) {
    FP_TRY(run_refine_heads(c, c->net[0], N, st));
    const size_t act = 2 * M * 512 * 2;  // [2][M][512] fp16
    const void* bufs[7] = {c->qkv.p, c->att.p, c->x1pre.p, c->x1.p, c->ff.p, c->x2pre.p, c->head_out.p};
    const size_t sizes[7] = {M * 3072 * 2, act, act, act, act, act, (size_t)2 * N * 3 * 4};
    src = bufs[stage], bytes = sizes[stage];
  } else {
    FP_TRY(run_score_feats(c, c->net[1], N, reinterpret_cast<float*>(c->feats.p), st));
    const void* bufs[4] = {c->qkv.p, c->att.p, c->tok_mean.p, c->feats.p};
    const size_t sizes[4] = {M * 1536 * 2, M * 512 * 2, (size_t)N * 512 * 4, (size_t)N * 512 * 4};
    src = bufs[stage], bytes = sizes[stage];
  }
  FP_CUDA_OK(cudaMemcpyAsync(out, src, bytes, cudaMemcpyDeviceToDevice, st));
  return (long long)bytes;
  FP_API_END
}

int fp_op_score_tail_segments(fp_ctx* c, const float* feats, int L, const int* seg_host, int n_seg, float* scores_out,
                              int* best_out, void* stream) {
  FP_API_BEGIN
  const char* fn = "fp_op_score_tail_segments";
  FP_REQUIRE(c && feats && seg_host && scores_out && best_out, "%s: null argument", fn);
  FP_REQUIRE(c->net[1].loaded, "scorer weights not loaded");
  FP_REQUIRE(n_seg >= 1, "%s: %d segments, need at least 1", fn, n_seg);
  FP_REQUIRE(seg_host[n_seg] == L, "%s: the last segment ends at row %d, not at L = %d", fn, seg_host[n_seg], L);
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  ScoreTailParams p;
  FP_TRY(segmented_tail_params(c, feats, seg_host, n_seg, /*trailing=*/0, scores_out, best_out, st, fn, p));
  return score_tail_launch(p, st);
  FP_API_END
}

int fp_op_depth_filter(const float* depth_dev, float* out_dev, int H, int W, int which, void* stream) {
  FP_API_BEGIN
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_REQUIRE(depth_dev && out_dev && H > 0 && W > 0, "fp_op_depth_filter: bad argument");
  if (which == 0) return erode_depth_launch(depth_dev, out_dev, H, W, 2, 0.001f, 0.8f, 100.f, st);
  return bilateral_depth_launch(depth_dev, out_dev, H, W, 2, 100.f, 2.f, 100000.f, st);
  FP_API_END
}

int fp_op_pose_update(fp_ctx* c, const float* poses_in, const float* trans, const float* rot, const int* mesh_of_host, int N,
                      float* poses_out, float* trans_delta_out, float* rot_delta_out, void* stream) {
  FP_API_BEGIN
  const char* fn = "fp_op_pose_update";
  FP_REQUIRE(c && poses_in && trans && rot && poses_out && N >= 0, "%s: bad argument", fn);
  const int slot0 = 0;
  FP_TRY(check_slots(c, mesh_of_host ? N : 1, mesh_of_host ? mesh_of_host : &slot0, fn));
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  if (N == 0) return 0;
  const int* mesh_of = nullptr;
  if (mesh_of_host) {
    FP_TRY(dev_alloc(&c->epoch, c->op_mesh_of, (size_t)N * sizeof(int)));
    FP_CUDA_OK(cudaMemcpyAsync(c->op_mesh_of.p, mesh_of_host, (size_t)N * sizeof(int), cudaMemcpyHostToDevice, st));
    mesh_of = reinterpret_cast<const int*>(c->op_mesh_of.p);
  }
  // as refine_body launches it: each hypothesis's half-diameter from the mesh table, the context's rot_normalizer
  return pose_update_launch(poses_in, trans, rot, poses_out, trans_delta_out, rot_delta_out, N,
                            reinterpret_cast<const MeshSlotDev*>(c->mesh_table.p), mesh_of, 0.f, c->rot_normalizer, st);
  FP_API_END
}

}  // extern "C"
