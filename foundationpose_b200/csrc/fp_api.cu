// fp_api.cu — the product C ABI (include/fpose.h): context, meshes, frames, and the per-frame hot loop (crops ->
// encoder -> heads -> pose update, K times; then scoring) enqueued on one stream with no host synchronisation.  The
// network plan the loop launches is in fp_net.cu, the operator hooks in fp_api_ops.cu, fp_group in fp_group.cu.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <tuple>
#include <vector>

#include "../../include/fpose.h"
#include "fp_attn.cuh"
#include "fp_common.cuh"
#include "fp_crop.cuh"
#include "fp_ctx.cuh"
#include "fp_depth.cuh"
#include "fp_gemm.cuh"
#include "fp_vis.cuh"

namespace fp {

// Entry `s` of the device mesh table, with the expressions the crop producer and the pose update always used.
static MeshSlotDev mesh_entry(const fp_ctx* c, int s) {
  const MeshSlot& m = c->mesh[s];
  MeshSlotDev e;
  memset(&e, 0, sizeof e);
  e.mesh.vpos = reinterpret_cast<const float4*>(m.vpos.p);
  e.mesh.vnrm = reinterpret_cast<const float4*>(m.vnrm.p);
  e.mesh.vatt = reinterpret_cast<const float4*>(m.vatt.p);
  e.mesh.faces = reinterpret_cast<const int4*>(m.faces.p);
  e.mesh.meshlets = reinterpret_cast<const Meshlet*>(m.meshlets.p);
  e.mesh.ml_verts = reinterpret_cast<const int*>(m.ml_verts.p);
  e.mesh.ml_tris = reinterpret_cast<const uint2*>(m.ml_tris.p);
  e.mesh.n_meshlets = m.n_meshlets;
  e.mesh.V = m.V;
  e.mesh.F = m.F;
  e.mesh.front_sign = c->cull_backfaces ? m.front_sign : 0;
  e.mesh.bs_x = m.bs[0];
  e.mesh.bs_y = m.bs[1];
  e.mesh.bs_z = m.bs[2];
  e.mesh.bs_r = m.bs[3];
  e.has_tex = m.has_tex ? 1 : 0;
  e.tex = m.has_tex ? reinterpret_cast<const uchar4*>(m.tex.p) : nullptr;
  e.Ht = m.Ht;
  e.Wt = m.Wt;
  for (int mode = 0; mode < 2; ++mode) e.r3[mode] = (float)((double)m.diameter * (double)c->crop_ratio[mode] / 2.0);
  e.inv_radius = 1.0f / (m.diameter / 2.0f);
  e.half_diameter = m.diameter / 2.0f;
  return e;
}

// Rewrites the table entries of every loaded slot.  Synchronises: kernels enqueued earlier may be reading the table.
static int write_mesh_table(fp_ctx* c) {
  FP_CUDA_OK(cudaDeviceSynchronize());
  FP_TRY(dev_alloc(&c->epoch, c->mesh_table, sizeof(MeshSlotDev) * kMaxMeshes, /*zero=*/true));
  std::vector<MeshSlotDev> table(kMaxMeshes);
  memset(table.data(), 0, sizeof(MeshSlotDev) * kMaxMeshes);
  for (int s = 0; s < kMaxMeshes; ++s)
    if (c->mesh[s].loaded) table[s] = mesh_entry(c, s);
  FP_CUDA_OK(cudaMemcpy(c->mesh_table.p, table.data(), sizeof(MeshSlotDev) * kMaxMeshes, cudaMemcpyHostToDevice));
  FP_CUDA_OK(cudaDeviceSynchronize());
  return 0;
}

// Camera i's frame as the kernels read it: the by-value frame (camera 0) or camera i's entry of the camera table
static CameraDev camera_dev(const fp_ctx* c, int i) {
  const CameraBufs& b = c->cam[i];
  CameraDev e;
  e.rgb_raw = static_cast<const unsigned char*>(b.rgb_raw.p);
  e.depth_raw = static_cast<const float*>(b.depth_raw.p);
  e.rgb = static_cast<uchar4*>(b.rgba.p);
  e.depth = static_cast<float*>(b.depth.p);
  e.xyz_map = static_cast<float4*>(b.xyz.p);
  e.fx = b.fx;
  e.fy = b.fy;
  e.cx = b.cx;
  e.cy = b.cy;
  e.H = b.H;
  e.W = b.W;
  return e;
}

// mesh_of: [N] device slot ids (validated by the caller), or null = every hypothesis renders slot 0.  cams / camera_of:
// device camera table and [N] camera ids (the tracking calls, fp_register_cameras), or null = the context's frame
// (camera 0), by value.  fit / fit_delta: the fit pass of the tracking calls (CropParams::fit), no crops
static int make_crops(fp_ctx* c, const float* poses, int N, int mode, float* dbg, float* win, int* stats,
                      cudaStream_t st, const int* mesh_of = nullptr, const CameraDev* cams = nullptr,
                      const int* camera_of = nullptr, float4* vis = nullptr, int* fit = nullptr,
                      const float* fit_delta = nullptr) {
  FP_REQUIRE(mesh_of || c->mesh[0].loaded, "no mesh: call fp_set_mesh first");
  FP_REQUIRE(c->has_frame, "no frame: call fp_set_frame first");
  // only launches below: this body is also what run_graphed captures (no allocation, no synchronisation)
  CropParams p;
  p.poses = poses;
  p.N = N;
  p.frame = camera_dev(c, 0);
  p.znear = 0.001f;  // Utils.py:161
  p.zfar = 100.f;
  p.slots = reinterpret_cast<const MeshSlotDev*>(c->mesh_table.p);
  p.mesh_of = mesh_of;
  p.mode = mode;
  p.crops = reinterpret_cast<__half*>(c->crops.p);
  p.b_img0 = b_img0_of(N);
  p.dbg = dbg;
  p.win_out = win;
  p.stats = stats;
  p.tile_override = c->crop_tile;
  p.cams = cams;
  p.camera_of = camera_of;
  p.vis = vis;
  p.fit = fit;
  p.fit_delta = fit_delta;
  return crop_launch(p, st);
}

// The launch sequence a cached graph holds: the first element of its key
enum class GraphKind {
  Refine = 0,            // fp_refine
  ScoreFeatures = 1,     // fp_score_features
  TrackObjects = 2,      // fp_track, fp_track_objects, fp_track_cameras
  RegisterRefine = 3,    // fp_register_objects / _cameras: one pass's refinement
  RegisterFeatures = 4,  // fp_register_objects / _cameras: one pass's scorer features
  TrackObjectsFit = 5,   // fp_track_cameras_fit_submit: TrackObjects, then the fit pass at the returned poses
  TrackObjectsAligned = 6,     // TrackObjects with a camera's depth from its sensor: memset + align ahead of the filter
  TrackObjectsFitAligned = 7,  // TrackObjectsFit likewise
};

// Runs `body(stream)` — a fixed sequence of kernel launches (and fixed-address copies) on ctx-owned buffers —
// through a cached CUDA graph: first sight of a key runs eagerly (sets function attributes), the second
// captures + instantiates, later calls replay.  Replay removes ~170 launch + 60 tensor-map-encode host
// calls per register(), which is what bounds track_one() and small per-GPU shards.  The body never allocates:
// callers size every workspace first, so a capture after an epoch bump (new mesh, new N) is safe.
// frame: where the body's kernels take their frame from, the last element of the key.  -1 (fp_refine, fp_score_features,
// fp_register_objects): camera 0's record (CameraDev) by value; such a graph is captured again when the record differs
// from its capture's, and only that graph: a frame of another size or other intrinsics does not invalidate the others.
// The record holds fx fy cx cy, the only entries of K a kernel reads, so a K that differs only in its skew or bottom
// row replays the graph.  Its buffer addresses change only with the epoch.  0 or
// more (the tracking calls, fp_register_cameras): the camera table, which holds every camera's size and intrinsics, so
// new intrinsics or a smaller frame replay the graph; the tracking calls pass their number of cameras C, which their
// frame-preparation launch covers, fp_register_cameras' passes 0 (their frames are prepared before the passes).
template <class Body>
static int run_graphed(fp_ctx* c, GraphKind kind, int N, int iters, cudaStream_t st, Body body, int frame = -1) {
  if (!c->use_graphs || g_prof_on) return body(st);
  const auto key = std::make_tuple(static_cast<int>(kind), N, iters, frame);
  auto it = c->graphs.find(key);
  if (it == c->graphs.end()) {
    c->graphs[key] = fp_ctx::GraphEntry();  // seen once: next call captures
    return body(st);
  }
  fp_ctx::GraphEntry& g = it->second;
  const CameraDev frame0 = camera_dev(c, 0);
  const bool frame_moved = frame < 0 && memcmp(&g.frame, &frame0, sizeof frame0) != 0;
  if (g.exec == nullptr || g.epoch != c->epoch || frame_moved) {
    if (g.exec) {
      cudaGraphExecDestroy(g.exec);
      g.exec = nullptr;
    }
    if (!c->cap_stream) FP_CUDA_OK(cudaStreamCreateWithFlags(&c->cap_stream, cudaStreamNonBlocking));
    FP_CUDA_OK(cudaStreamBeginCapture(c->cap_stream, cudaStreamCaptureModeThreadLocal));
    set_capturing(true);  // nothing runs during capture: launches are counted per replay
    int rc = 0;
    try {
      rc = body(c->cap_stream);
    } catch (...) {
      rc = -3;
      set_last_error("exception while capturing the launch sequence");
    }
    set_capturing(false);
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(c->cap_stream, &graph);
    if (rc != 0) {
      if (graph) cudaGraphDestroy(graph);
      return rc;
    }
    FP_CUDA_OK(ce);
    size_t n_nodes = 0;
    cudaGraphGetNodes(graph, nullptr, &n_nodes);
    size_t n_kernels = 0;
    {
      std::vector<cudaGraphNode_t> nodes(n_nodes);
      if (n_nodes && cudaGraphGetNodes(graph, nodes.data(), &n_nodes) == cudaSuccess)
        for (auto nd : nodes) {
          cudaGraphNodeType ty;
          if (cudaGraphNodeGetType(nd, &ty) == cudaSuccess && ty == cudaGraphNodeTypeKernel) ++n_kernels;
        }
    }
    const cudaError_t ie = cudaGraphInstantiate(&g.exec, graph, 0);
    cudaGraphDestroy(graph);
    FP_CUDA_OK(ie);
    g.epoch = c->epoch;
    g.frame = frame0;
    c->graph_nodes[key] = (int)n_kernels;
    ++c->graph_captures;
  }
  FP_CUDA_OK(cudaGraphLaunch(g.exec, st));
  note_launches(c->graph_nodes[key]);
  return 0;
}

// camera 0's filtered frame from rgb_dev / depth_dev in format fmt, with camera 0's record by value (fp_set_frame,
// fp_register_objects).  sensor (non-null: camera 0 has a depth sensor, and depth_dev / fmt are then its aligned buffer
// and aligned_fmt): the aligned buffer is zeroed and the sensor's depth aligned into it first.
static int set_frame_launches(fp_ctx* c, const unsigned char* rgb_dev, const float* depth_dev, const FrameFmtDev& fmt,
                              int flags, float zfar, cudaStream_t st, const SensorDev* sensor = nullptr) {
  CameraDev one = camera_dev(c, 0);
  if (sensor) {
    FP_CUDA_OK(cudaMemsetAsync(sensor->aligned, 0, (size_t)one.H * one.W * 4, st));
    FP_TRY(align_depth_launch(*sensor, one, st));
  }
  one.rgb_raw = rgb_dev;  // camera 0's upload buffers, or the caller's device frame (FP_FRAME_ON_DEVICE)
  one.depth_raw = depth_dev;
  if (flags & FP_FRAME_FILTER_DEPTH) {
    // estimater.py:173-174 erode_depth(radius=2), bilateral_filter_depth(radius=2); :214 depth2xyzmap: one launch
    return frame_prep_launch(one, fmt, zfar, st);
  }
  const size_t npix = (size_t)one.H * one.W;
  // packed float32 depth is copied as it is; any other depth is converted by the colour kernel
  const bool depth_as_is = fmt.depth_kind == kDepthF32 && (size_t)fmt.depth_pitch == (size_t)one.W * 4;
  FP_TRY(raw_frame_launch(one, fmt, !depth_as_is, st));
  if (depth_as_is) FP_CUDA_OK(cudaMemcpyAsync(one.depth, depth_dev, npix * 4, cudaMemcpyDeviceToDevice, st));
  return depth_to_xyz_launch(one, zfar, st);
}

// A camera's raw frame of width W in format f: the one place that knows its bytes per pixel, row bytes and pitches.
// Wd: the width of its depth image, W's unless the camera has a depth sensor.
struct FrameLayout {
  int rgb_bpp, depth_bpp;          // bytes per pixel
  size_t rgb_row, depth_row;       // bytes per packed row
  long long rgb_pitch, depth_pitch;  // bytes from one row of the caller's buffer to the next
};
static FrameLayout frame_layout(const fp_frame_format_t& f, int W, int Wd) {
  FrameLayout L;
  L.rgb_bpp = (f.color == FP_COLOR_RGBA8 || f.color == FP_COLOR_BGRA8) ? 4 : 3;
  L.depth_bpp = f.depth == FP_DEPTH_U16 ? 2 : 4;
  L.rgb_row = (size_t)W * L.rgb_bpp;
  L.depth_row = (size_t)Wd * L.depth_bpp;
  L.rgb_pitch = f.rgb_pitch ? f.rgb_pitch : (long long)L.rgb_row;
  L.depth_pitch = f.depth_pitch ? f.depth_pitch : (long long)L.depth_row;
  return L;
}

// The kernels' record of a raw frame in format f: read in place with the caller's pitches, or from the context's upload
// buffers, where it was staged packed
static FrameFmtDev fmt_dev(const fp_frame_format_t& f, const FrameLayout& L, bool rgb_in_place, bool depth_in_place) {
  FrameFmtDev d;
  memset(&d, 0, sizeof d);
  d.rgb_pitch = (int)(rgb_in_place ? L.rgb_pitch : (long long)L.rgb_row);
  d.depth_pitch = (int)(depth_in_place ? L.depth_pitch : (long long)L.depth_row);
  d.depth_scale = f.depth == FP_DEPTH_U16 ? f.depth_scale : 0.f;
  d.bpp = (unsigned char)L.rgb_bpp;
  d.bgr = (f.color == FP_COLOR_BGR8 || f.color == FP_COLOR_BGRA8) ? 1 : 0;
  d.depth_kind = f.depth == FP_DEPTH_U16 ? kDepthU16 : kDepthF32;
  d.packed = (d.bpp == 3 && !d.bgr && d.depth_kind == kDepthF32 && (size_t)d.rgb_pitch == L.rgb_row &&
              (size_t)d.depth_pitch == L.depth_row) ? 1 : 0;
  return d;
}

// The size of camera i's depth image for a colour frame of H x W: its depth sensor's, or the colour frame's
static void depth_size(const fp_ctx* c, int i, int H, int W, int& Hd, int& Wd) {
  Hd = c->has_sensor[i] ? c->sensor[i].H : H;
  Wd = c->has_sensor[i] ? c->sensor[i].W : W;
}

// Camera i's aligned buffer (fp_ctx::aligned)
static unsigned int* aligned_buf(const fp_ctx* c, int i) {
  return static_cast<unsigned int*>(c->aligned.p) + (size_t)i * c->aligned_stride;
}

// Sizes the aligned buffers of C cameras for frames of up to npix pixels.  A graph holds the block's address and its
// memset's size, so growing either moves the epoch.
static int ensure_aligned(fp_ctx* c, int C, size_t npix) {
  if (npix > c->aligned_stride) {
    ++c->epoch;
    c->aligned_stride = npix;
  }
  return dev_alloc(&c->epoch, c->aligned, (size_t)C * c->aligned_stride * 4);
}

// Camera i's sensor record for the kernels, its raw depth read at `depth` with layout L (in place: the caller's pitch,
// else the packed rows of the upload buffer); zero (aligned = null) when the camera has no sensor
static SensorDev sensor_dev(const fp_ctx* c, int i, const void* depth, const FrameLayout& L, bool in_place) {
  SensorDev d;
  memset(&d, 0, sizeof d);
  if (!c->has_sensor[i]) return d;
  const fp_depth_sensor_t& s = c->sensor[i];
  d.depth = depth;
  d.aligned = aligned_buf(c, i);
  d.pitch = (int)(in_place ? L.depth_pitch : (long long)L.depth_row);
  d.u16 = c->fmt[i].depth == FP_DEPTH_U16 ? 1 : 0;
  d.scale = d.u16 ? c->fmt[i].depth_scale : 0.f;
  d.H = s.H;
  d.W = s.W;
  d.fx = s.K[0];
  d.fy = s.K[4];
  d.cx = s.K[2];
  d.cy = s.K[5];
  for (int k = 0; k < 12; ++k) d.T[k] = s.T_color_from_depth[k];
  return d;
}

// The format record of a camera's aligned buffer (colour width W), which the frame filter reads in place of the raw
// depth: the colour part of f stays, the depth becomes kDepthAligned rows of W slots
static FrameFmtDev aligned_fmt(FrameFmtDev f, int W) {
  f.depth_pitch = W * 4;
  f.depth_scale = 0.f;
  f.depth_kind = kDepthAligned;
  f.packed = 0;
  return f;
}

// Camera i's frame (depth buffer `depth`, colour width W) against camera i's format: pitches no shorter than a packed
// row (of the depth sensor's width for the depth of a camera with one), the depth pitch and pointer aligned to the
// depth element.  Checked before anything is enqueued.
static int check_frame_format(const fp_ctx* c, int i, const void* depth, int W, const char* caller) {
  const fp_frame_format_t& f = c->fmt[i];
  int Hd, Wd;
  depth_size(c, i, 1, W, Hd, Wd);
  const FrameLayout L = frame_layout(f, W, Wd);
  FP_REQUIRE(L.rgb_pitch >= (long long)L.rgb_row, "%s: camera %d: rgb pitch %lld bytes is below the %zu bytes of a row", caller,
             i, L.rgb_pitch, L.rgb_row);
  FP_REQUIRE(L.depth_pitch >= (long long)L.depth_row, "%s: camera %d: depth pitch %lld bytes is below the %zu bytes of a row",
             caller, i, L.depth_pitch, L.depth_row);
  FP_REQUIRE(L.depth_pitch % L.depth_bpp == 0, "%s: camera %d: depth pitch %lld bytes is not a multiple of the %d-byte depth value",
             caller, i, L.depth_pitch, L.depth_bpp);
  FP_REQUIRE(reinterpret_cast<uintptr_t>(depth) % L.depth_bpp == 0,
             "%s: camera %d: depth buffer %p is not aligned to its %d-byte depth value", caller, i, depth, L.depth_bpp);
  return 0;
}
static int check_frame_formats(const fp_ctx* c, int C, const float* const* depth, const int* W, const char* caller) {
  for (int i = 0; i < C; ++i) FP_TRY(check_frame_format(c, i, depth[i], W[i], caller));
  return 0;
}

// Copies `rows` host rows of `row` bytes, `pitch` bytes apart at `src`, into `dst` (device) on `st`: one copy when the
// rows are packed, a 2D copy otherwise
static int copy_rows(void* dst, const void* src, size_t row, long long pitch, int rows, cudaStream_t st) {
  if (pitch == (long long)row) {
    FP_CUDA_OK(cudaMemcpyAsync(dst, src, row * rows, cudaMemcpyHostToDevice, st));
  } else {
    FP_CUDA_OK(cudaMemcpy2DAsync(dst, row, src, (size_t)pitch, row, rows, cudaMemcpyHostToDevice, st));
  }
  return 0;
}

// Sizes camera i's buffers for npix pixels: the filtered frame always, the raw upload if `raw`.  Camera 0's addresses
// are held by the graphs that take the frame by value, so growing its buffers bumps the graph epoch.  Cameras 1.. are
// reached only through the camera table, which every call rewrites: growing them invalidates no graph.
// The raw upload holds rgb_bpp / depth_bpp bytes per pixel (the frame format's), the depth one for depth_npix pixels
// (0: npix; a depth sensor's image); buffers only grow, so a camera that alternates between formats of a size it has
// seen allocates nothing after the first time.
static int alloc_camera(fp_ctx* c, int i, size_t npix, bool raw, int rgb_bpp = 3, int depth_bpp = 4, size_t depth_npix = 0) {
  CameraBufs& b = c->cam[i];
  unsigned long long* epoch = i == 0 ? &c->epoch : nullptr;
  FP_TRY(dev_alloc(epoch, b.rgba, npix * 4));
  FP_TRY(dev_alloc(epoch, b.depth, npix * 4));
  FP_TRY(dev_alloc(epoch, b.xyz, npix * 16));
  if (raw) {
    FP_TRY(dev_alloc(epoch, b.rgb_raw, npix * rgb_bpp));
    FP_TRY(dev_alloc(epoch, b.depth_raw, (depth_npix ? depth_npix : npix) * depth_bpp));
  }
  return 0;
}

// records camera i's frame size and intrinsics (K: [3][3] row-major).  Camera 0's are the context's frame geometry: a
// graph that holds them by value is captured again when they change, see run_graphed
static void set_frame_geometry(fp_ctx* c, int i, const float* K, int H, int W) {
  CameraBufs& b = c->cam[i];
  b.fx = K[0];
  b.fy = K[4];
  b.cx = K[2];
  b.cy = K[5];
  b.H = H;
  b.W = W;
}

// mesh_of: [N] device slot ids, or null = slot 0 for every hypothesis; cams / camera_of as make_crops
static int refine_body(fp_ctx* c, int N, int iterations, cudaStream_t s2, const int* mesh_of = nullptr,
                       const CameraDev* cams = nullptr, const int* camera_of = nullptr) {
  float* cur = reinterpret_cast<float*>(c->poses_a.p);
  float* nxt = reinterpret_cast<float*>(c->poses_b.p);
  const float* ho = reinterpret_cast<const float*>(c->head_out.p);
  const MeshSlotDev* table = reinterpret_cast<const MeshSlotDev*>(c->mesh_table.p);
  for (int it = 0; it < iterations; ++it) {
    FP_TRY(make_crops(c, cur, N, 0, nullptr, nullptr, nullptr, s2, mesh_of, cams, camera_of));
    FP_TRY(run_encoder(c, c->net[0], reinterpret_cast<const __half*>(c->crops.p), N, s2));
    FP_TRY(run_refine_heads(c, c->net[0], N, s2));
    const bool last = it == iterations - 1;
    FP_TRY(pose_update_launch(cur, ho, ho + (size_t)N * 3, nxt, last ? reinterpret_cast<float*>(c->lt_buf.p) : nullptr,
                              last ? reinterpret_cast<float*>(c->lr_buf.p) : nullptr, N, table, mesh_of, 0.f,
                              c->rot_normalizer, s2));
    float* t = cur;
    cur = nxt;
    nxt = t;
  }
  return 0;
}

// Copies `bytes` of host memory `src` into the pinned `stage` (grown as needed) and enqueues its upload to `dst`: the
// caller's memory is free again once this returns.
// The same for `rows` rows of `row` bytes, `pitch` bytes apart at `src`: staged packed, in one copy when they are packed.
static int stage_rows(void* dst, PinnedBuf& stage, const void* src, size_t row, long long pitch, int rows, cudaStream_t st) {
  const size_t bytes = row * rows;
  FP_TRY(pinned_alloc(nullptr, stage, bytes));
  if (pitch == (long long)row) {
    memcpy(stage.p, src, bytes);
  } else {
    for (int r = 0; r < rows; ++r)
      memcpy(static_cast<char*>(stage.p) + r * row, static_cast<const char*>(src) + r * pitch, row);
  }
  FP_CUDA_OK(cudaMemcpyAsync(dst, stage.p, bytes, cudaMemcpyHostToDevice, st));
  return 0;
}
static int stage_copy(void* dst, PinnedBuf& stage, const void* src, size_t bytes, cudaStream_t st) {
  return stage_rows(dst, stage, src, bytes, (long long)bytes, 1, st);
}

// Uploads one camera's frame (H rows of rgb and Hd rows of depth of layout L) through its staging (free: the set is not
// busy).  The two uploads are issued as soon as their staging copy is done — the depth DMA runs under the host's rgb
// copy, the rgb DMA under the next camera's copies or the graph launch — instead of being nodes of the graph (measured:
// -40 us per frame)
static int upload_staged_frame(CameraBufs& b, PinnedBuf& stage_rgb, PinnedBuf& stage_depth, const unsigned char* rgb_host,
                               const void* depth_host, const FrameLayout& L, int H, int Hd, cudaStream_t st) {
  FP_TRY(stage_rows(b.depth_raw.p, stage_depth, depth_host, L.depth_row, L.depth_pitch, Hd, st));
  return stage_rows(b.rgb_raw.p, stage_rgb, rgb_host, L.rgb_row, L.rgb_pitch, H, st);
}

// The one place that decides which staging set a call uses: the next one in turn, waited for first, if it is still
// busy, until the uploads of the call that used it have left it.
static int take_set(fp_ctx* c, StagingSet*& set) {
  set = &c->sets[c->next_set];
  if (set->busy) {
    FP_CUDA_OK(cudaEventSynchronize(set->uploaded.e));
    set->busy = false;
  }
  c->next_set = (c->next_set + 1) % kMaxInFlight;
  return 0;
}

// After a call's last copy out of `set`: the set stays busy until `st` has passed that copy.
static int set_busy(StagingSet& set, cudaStream_t st) {
  FP_CUDA_OK(set.uploaded.record(st));
  set.busy = true;
  return 0;
}

// Where one of the caller's input buffers lives, as cudaPointerGetAttributes sees it
enum class Residence {
  Pageable,     // host memory the device cannot read in place: a copy from it may wait on the stream
  HostLocked,   // page-locked or managed memory: host memory the device can also read
  Device,       // device memory of the context's device: the kernels can read it in place
  OtherDevice,  // device memory of another device: refused where a call would read it in place
};
static Residence residence(const fp_ctx* c, const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();  // not sticky; keep it out of the next caller's error check
    return Residence::Pageable;
  }
  if (a.type == cudaMemoryTypeUnregistered) return Residence::Pageable;
  if (a.type == cudaMemoryTypeDevice) return a.device == c->device ? Residence::Device : Residence::OtherDevice;
  return Residence::HostLocked;  // cudaMemoryTypeHost, cudaMemoryTypeManaged
}

// Whether the caller's frame or mask buffer `p` of a tracking or register call is read in place (device memory of the
// context's device) or staged (host memory).  Device memory of another device is refused.  what / i name the buffer.
static int read_in_place(const fp_ctx* c, const void* p, bool& in_place, const char* caller, const char* what, int i) {
  const Residence r = residence(c, p);
  FP_REQUIRE(r != Residence::OtherDevice, "%s: %s %d is device memory of another device than the context's (device %d)",
             caller, what, i, c->device);
  in_place = r == Residence::Device;
  return 0;
}

// Which frame buffers of a call's C cameras are read in place (see read_in_place), each camera's rgb and depth on
// their own.  Classified before anything is enqueued.
struct FrameSources {
  bool rgb[kMaxCameras] = {}, depth[kMaxCameras] = {};
};
static int frame_sources(const fp_ctx* c, int C, const unsigned char* const* rgb, const float* const* depth, FrameSources& on_dev,
                         const char* caller) {
  for (int i = 0; i < C; ++i) {
    FP_TRY(read_in_place(c, rgb[i], on_dev.rgb[i], caller, "the rgb frame of camera", i));
    FP_TRY(read_in_place(c, depth[i], on_dev.depth[i], caller, "the depth frame of camera", i));
  }
  return 0;
}

// Uploads `bytes` of the caller's host memory `src` to `dst` on `st`.  Page-locked memory is copied straight from the
// caller's buffer, which must stay untouched until `st` has passed the copy; pageable memory goes through `stage` of the
// next staging set, so the caller may reuse it once this returns and the host does not wait on the stream for it.
static int upload_host(fp_ctx* c, void* dst, const void* src, size_t bytes, PinnedBuf StagingSet::*stage, cudaStream_t st) {
  if (residence(c, src) != Residence::Pageable) {
    FP_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st));
    return 0;
  }
  StagingSet* set;
  FP_TRY(take_set(c, set));
  const int staged = stage_copy(dst, set->*stage, src, bytes, st);
  FP_TRY(set_busy(*set, st));  // after a failure too: a copy may have been enqueued
  return staged;
}

// Orders `st` after the last tracking call submitted: its device buffers and the context's frames are then free on `st`
// (a call on the same stream is ordered already).  Every entry point that uses the context's frames or workspaces
// calls this first.  It never waits on the host: a staging set is waited for only by the call that takes it again
// (take_set), and results are collected separately (fp_track_wait).
int order_after_track(fp_ctx* c, cudaStream_t st) {
  if (c->last_done && st != c->last_stream) FP_CUDA_OK(cudaStreamWaitEvent(st, c->last_done, 0));
  return 0;
}

constexpr size_t kTableBytes = sizeof(CameraDev) * kMaxCameras;  // the camera table at the head of fp_ctx::args
constexpr size_t kSensorsAt = kTableBytes + sizeof(FrameFmtDev) * kMaxCameras;  // then the cameras' frame formats
constexpr size_t kHeadBytes = kSensorsAt + sizeof(SensorDev) * kMaxCameras;  // then the cameras' depth sensors
// fp_ctx::args (and its staging) for `rows` slot and camera ids: the three tables, the ids, and a tracking call's fit
// threshold
static size_t args_bytes(int rows) { return kHeadBytes + (size_t)2 * rows * sizeof(int) + sizeof(float); }

// The cameras of fp_track_cameras / _objects and fp_register_cameras / _objects, before anything reads a frame.  Every
// camera's buffers are sized for the largest frame of the call (kept at the largest size seen, so a permutation of the
// same cameras allocates nothing), the argument block is sized for `rows` slot and camera ids and its staging for
// `staged_rows`, every camera records its size and intrinsics (K: [C][9]; camera 0's become the context's frame
// geometry), the staging receives the camera table (every camera's record; entries C.. zeroed), and every host frame is
// uploaded through its camera's staging (camera i's DMA runs while camera i + 1 is copied on the host).  A frame buffer
// on the device (on_dev) is read in place: its table entry points at the caller's buffer, and nothing is staged or
// uploaded for it.  Every camera still gets its raw upload buffers, so where a frame lives never changes an allocation
// or the graph epoch.  Each camera's frame is read in its format (fp_ctx::fmt, copied into the format table beside the
// camera table here): host frames are staged packed, at the format's bytes per pixel, device frames are read with their
// pitch; the raw buffers are sized for the largest frame and the widest pixels of the call.  A camera with a depth
// sensor (fp_ctx::sensor, copied into the sensor table here) has its raw depth staged or read at the sensor's size, its
// table entry reads its aligned buffer as depth (aligned_fmt), and the call's aligned buffers are sized.
// `set`: the staging set the call uploads through (not busy).
struct CallFrames {
  int H_max = 0, W_max = 0;    // the largest frame height and width of the call
  bool aligned = false;        // some camera of the call has a depth sensor
  int Hd_max = 0, Wd_max = 0;  // the largest depth image of those cameras
};
static int setup_cameras(fp_ctx* c, StagingSet& set, int C, const unsigned char* const* rgb, const float* const* depth,
                         const FrameSources& on_dev, const float* K, const int* H, const int* W, int rows, int staged_rows,
                         cudaStream_t st, CallFrames& g) {
  size_t npix_max = 0, depth_npix_max = 0;
  int rgb_bpp = 0, depth_bpp = 0;
  g = CallFrames{};
  for (int i = 0; i < C; ++i) {
    npix_max = std::max(npix_max, (size_t)H[i] * W[i]);
    g.H_max = std::max(g.H_max, H[i]);
    g.W_max = std::max(g.W_max, W[i]);
    int Hd, Wd;
    depth_size(c, i, H[i], W[i], Hd, Wd);
    depth_npix_max = std::max(depth_npix_max, (size_t)Hd * Wd);
    if (c->has_sensor[i]) {
      g.aligned = true;
      g.Hd_max = std::max(g.Hd_max, Hd);
      g.Wd_max = std::max(g.Wd_max, Wd);
    }
    const FrameLayout L = frame_layout(c->fmt[i], W[i], Wd);
    rgb_bpp = std::max(rgb_bpp, L.rgb_bpp);
    depth_bpp = std::max(depth_bpp, L.depth_bpp);
  }
  for (int i = 0; i < C; ++i) {
    FP_TRY(alloc_camera(c, i, npix_max, /*raw=*/true, rgb_bpp, depth_bpp, depth_npix_max));
    if (!on_dev.rgb[i]) FP_TRY(pinned_alloc(nullptr, set.rgb[i], npix_max * rgb_bpp));
    if (!on_dev.depth[i]) FP_TRY(pinned_alloc(nullptr, set.depth[i], depth_npix_max * depth_bpp));
  }
  if (g.aligned) FP_TRY(ensure_aligned(c, C, npix_max));
  c->n_frames = C;
  FP_TRY(dev_alloc(&c->epoch, c->args, args_bytes(rows)));
  FP_TRY(pinned_alloc(nullptr, set.args, args_bytes(staged_rows)));
  CameraDev* table = reinterpret_cast<CameraDev*>(set.args.p);
  FrameFmtDev* fmts = reinterpret_cast<FrameFmtDev*>(static_cast<char*>(set.args.p) + kTableBytes);
  SensorDev* sensors = reinterpret_cast<SensorDev*>(static_cast<char*>(set.args.p) + kSensorsAt);
  memset(table, 0, kHeadBytes);
  for (int i = 0; i < C; ++i) {
    set_frame_geometry(c, i, K + 9 * i, H[i], W[i]);
    table[i] = camera_dev(c, i);
    if (on_dev.rgb[i]) table[i].rgb_raw = rgb[i];
    if (on_dev.depth[i]) table[i].depth_raw = depth[i];
    int Hd, Wd;
    depth_size(c, i, H[i], W[i], Hd, Wd);
    const FrameLayout L = frame_layout(c->fmt[i], W[i], Wd);
    fmts[i] = fmt_dev(c->fmt[i], L, on_dev.rgb[i], on_dev.depth[i]);
    if (c->has_sensor[i]) {
      sensors[i] = sensor_dev(c, i, table[i].depth_raw, L, on_dev.depth[i]);
      table[i].depth_raw = reinterpret_cast<const float*>(sensors[i].aligned);
      fmts[i] = aligned_fmt(fmts[i], W[i]);
    }
    // the order of upload_staged_frame: depth, then rgb
    if (!on_dev.depth[i]) FP_TRY(stage_rows(c->cam[i].depth_raw.p, set.depth[i], depth[i], L.depth_row, L.depth_pitch, Hd, st));
    if (!on_dev.rgb[i]) FP_TRY(stage_rows(c->cam[i].rgb_raw.p, set.rgb[i], rgb[i], L.rgb_row, L.rgb_pitch, H[i], st));
  }
  return 0;
}

// The staging uploads of one tracking call: the frames, then the camera table, the slot ids, the camera ids and, with a
// fit (delta non-null), its threshold in one copy to the argument block.  g as setup_cameras.
static int stage_track_call(fp_ctx* c, StagingSet& set, int C, const unsigned char* const* rgb, const float* const* depth,
                            const FrameSources& on_dev, const float* K, const int* H, const int* W, int M,
                            const int* camera_of, const int* slots_host, const float* delta, cudaStream_t st, CallFrames& g) {
  FP_TRY(setup_cameras(c, set, C, rgb, depth, on_dev, K, H, W, M, M, st, g));
  int* ids = reinterpret_cast<int*>(static_cast<char*>(set.args.p) + kHeadBytes);
  memcpy(ids, slots_host, (size_t)M * sizeof(int));
  memcpy(ids + M, camera_of, (size_t)M * sizeof(int));
  if (delta) memcpy(ids + 2 * M, delta, sizeof(float));
  const size_t bytes = kHeadBytes + (size_t)2 * M * sizeof(int) + (delta ? sizeof(float) : 0);
  FP_CUDA_OK(cudaMemcpyAsync(c->args.p, set.args.p, bytes, cudaMemcpyHostToDevice, st));
  return 0;
}

// fp_track_cameras_submit, fp_track_objects_submit (C = 1) and fp_track_submit (C = M = 1) after validation, and so
// every blocking tracking call, which is a submit and its fp_track_wait.  The call stages through the next staging set,
// waiting first, if that set is still busy, until the uploads of the call that used it have left it.  The camera
// table, the slot ids and the camera ids go to the argument block in one copy ahead of the launch.  The graph holds the
// block's address, not the frames' sizes, intrinsics or buffers, and is keyed on (M, iterations, C): reordering objects
// or cameras, new intrinsics or a smaller frame replay it.  One frame_prep_kernel launch filters every camera and the
// crops take their frame from the table.  The pose read-back follows the launch outside the graph, into the call's own
// Readback, so one graph serves every staging set.  Frames on the device are read in place through the camera table
// (setup_cameras), so where a frame lives changes neither the graph nor its key.  poses_out_dev and poses_keep_dev
// (fp_track's continuation pose) are optional and complete in stream order; *ticket receives the call's ticket.
// delta (host, validated) makes it a call with a fit: the TrackObjectsFit graph zeroes the fit counts first and ends
// with the fit pass at the returned poses; delta travels in the argument block, so a new delta replays the graph.  The
// counts go to fit_out_dev (optional, stream order) and to the Readback right after the poses.
static int track_cameras_submit(fp_ctx* c, const char* caller, int C, const unsigned char* const* rgb,
                                const float* const* depth, const float* K, const int* H, const int* W, int M,
                                const int* camera_of, const int* slots_host, const float* poses_in_dev, int iterations,
                                float* poses_out_dev, cudaStream_t st, unsigned long long* ticket,
                                float* poses_keep_dev = nullptr, const float* delta = nullptr, int* fit_out_dev = nullptr) {
  FrameSources on_dev;
  FP_TRY(frame_sources(c, C, rgb, depth, on_dev, caller));  // refused before anything is enqueued
  FP_TRY(check_frame_formats(c, C, depth, W, caller));
  StagingSet* set;
  FP_TRY(take_set(c, set));
  FP_TRY(order_after_track(c, st));  // the context's device buffers are never used by two streams at once
  Readback* rb = nullptr;
  for (auto& r : c->readbacks)
    if (r->ticket == 0) rb = r.get();
  if (!rb) {
    c->readbacks.push_back(std::make_unique<Readback>());
    rb = c->readbacks.back().get();
  }
  FP_TRY(ensure_capacity(c, M));
  FP_TRY(pinned_alloc(nullptr, rb->poses, (size_t)M * 64));
  const size_t fit_bytes = (size_t)M * kFitCounts * sizeof(int);
  if (delta) {
    FP_TRY(dev_alloc(&c->epoch, c->fit, fit_bytes));
    FP_TRY(pinned_alloc(nullptr, rb->fit, fit_bytes));
  }
  c->has_frame = false;
  CallFrames g;
  const int staged = stage_track_call(c, *set, C, rgb, depth, on_dev, K, H, W, M, camera_of, slots_host, delta, st, g);
  // whatever was staged before a failure is still on its way out: the set stays busy until then
  FP_TRY(set_busy(*set, st));
  FP_TRY(staged);
  if (g.H_max > c->cam_grid_h || g.W_max > c->cam_grid_w) {
    // the frame-preparation grid is a by-value launch parameter: it covers the largest frame seen, the blocks outside
    // a smaller frame return at once
    ++c->epoch;
    c->cam_grid_h = std::max(c->cam_grid_h, g.H_max);
    c->cam_grid_w = std::max(c->cam_grid_w, g.W_max);
  }
  if (g.aligned && (g.Hd_max > c->sensor_grid_h || g.Wd_max > c->sensor_grid_w)) {
    // the alignment grid likewise covers the largest depth image seen
    ++c->epoch;
    c->sensor_grid_h = std::max(c->sensor_grid_h, g.Hd_max);
    c->sensor_grid_w = std::max(c->sensor_grid_w, g.Wd_max);
  }
  const CameraDev* cams_dev = reinterpret_cast<const CameraDev*>(c->args.p);
  const FrameFmtDev* fmts_dev = reinterpret_cast<const FrameFmtDev*>(static_cast<const char*>(c->args.p) + kTableBytes);
  const SensorDev* sensors_dev = reinterpret_cast<const SensorDev*>(static_cast<const char*>(c->args.p) + kSensorsAt);
  const size_t aligned_bytes = (size_t)C * c->aligned_stride * 4;
  const int* mesh_of = reinterpret_cast<const int*>(static_cast<const char*>(c->args.p) + kHeadBytes);
  const int* cam_of = mesh_of + M;
  const float* delta_dev = reinterpret_cast<const float*>(cam_of + M);
  int* fit = reinterpret_cast<int*>(c->fit.p);
  float* pa = reinterpret_cast<float*>(c->poses_a.p);
  float* pb = reinterpret_cast<float*>(c->poses_b.p);
  FP_CUDA_OK(cudaMemcpyAsync(pa, poses_in_dev, (size_t)M * 64, cudaMemcpyDeviceToDevice, st));
  const float* fin = (iterations % 2 == 0) ? pa : pb;
  const int grid_h = c->cam_grid_h, grid_w = c->cam_grid_w;
  const int sgrid_h = c->sensor_grid_h, sgrid_w = c->sensor_grid_w;
  auto body = [&](cudaStream_t s2) -> int {
    // the counts are zeroed at the head of the sequence, so the fit pass follows the last pose update by programmatic
    // dependent launch like every other link of the chain
    if (delta) FP_CUDA_OK(cudaMemsetAsync(fit, 0, fit_bytes, s2));
    if (g.aligned) {
      // the depth of the cameras with a sensor aligned into their zeroed aligned buffers, which the frame filter (an
      // ordinary launch, after this one in stream order) reads as their depth
      FP_CUDA_OK(cudaMemsetAsync(c->aligned.p, 0, aligned_bytes, s2));
      FP_TRY(align_depth_cameras_launch(sensors_dev, cams_dev, C, sgrid_h, sgrid_w, s2));
    }
    // estimater.py:250-268 for every object of every camera at once: each camera's frame filtered once (erode +
    // bilateral, depth2xyzmap_batch(zfar = inf)), M hypotheses each rendering its own mesh and cropping its own
    // camera's frame
    FP_TRY(frame_prep_cameras_launch(cams_dev, fmts_dev, C, grid_h, grid_w, INFINITY, s2));
    c->has_frame = true;
    FP_TRY(refine_body(c, M, iterations, s2, mesh_of, cams_dev, cam_of));
    if (delta) FP_TRY(make_crops(c, fin, M, 0, nullptr, nullptr, nullptr, s2, mesh_of, cams_dev, cam_of, nullptr, fit, delta_dev));
    return 0;
  };
  const GraphKind kind = g.aligned ? (delta ? GraphKind::TrackObjectsFitAligned : GraphKind::TrackObjectsAligned)
                                   : (delta ? GraphKind::TrackObjectsFit : GraphKind::TrackObjects);
  FP_TRY(run_graphed(c, kind, M, iterations, st, body, C));
  c->has_frame = true;
  if (poses_out_dev) FP_CUDA_OK(cudaMemcpyAsync(poses_out_dev, fin, (size_t)M * 64, cudaMemcpyDeviceToDevice, st));
  if (fit_out_dev) FP_CUDA_OK(cudaMemcpyAsync(fit_out_dev, fit, fit_bytes, cudaMemcpyDeviceToDevice, st));
  if (poses_keep_dev) FP_CUDA_OK(cudaMemcpyAsync(poses_keep_dev, fin, (size_t)M * 64, cudaMemcpyDeviceToDevice, st));
  FP_CUDA_OK(cudaMemcpyAsync(rb->poses.p, fin, (size_t)M * 64, cudaMemcpyDeviceToHost, st));
  if (delta) FP_CUDA_OK(cudaMemcpyAsync(rb->fit.p, fit, fit_bytes, cudaMemcpyDeviceToHost, st));
  FP_CUDA_OK(rb->done.record(st));
  c->last_done = rb->done.e;
  c->last_stream = st;
  rb->M = M;
  rb->has_fit = delta != nullptr;
  rb->ticket = ++c->last_ticket;
  *ticket = rb->ticket;
  return 0;
}

// fp_track_wait / fp_track_fit_wait (fit): waits for ticket's read-back and copies its poses out, and its fit counts for
// fp_track_fit_wait (either output may be null: that result is dropped).  fp_track_fit_wait refuses a ticket submitted
// without a fit and leaves it uncollected.  Otherwise the ticket is collected whatever the outcome, so an asynchronous
// error is reported once.
static int track_wait(fp_ctx* c, unsigned long long ticket, float* poses_out_host, bool fit = false,
                      int* fit_out_host = nullptr) {
  const char* caller = fit ? "fp_track_fit_wait" : "fp_track_wait";
  Readback* rb = nullptr;
  for (auto& r : c->readbacks)
    if (ticket != 0 && r->ticket == ticket) rb = r.get();
  FP_REQUIRE(rb, "%s: ticket %llu is unknown or already collected", caller, ticket);
  FP_REQUIRE(!fit || rb->has_fit, "%s: ticket %llu was submitted without a fit: collect it with fp_track_wait", caller, ticket);
  rb->ticket = 0;
  FP_CUDA_OK(cudaEventSynchronize(rb->done.e));
  if (poses_out_host) memcpy(poses_out_host, rb->poses.p, (size_t)rb->M * 64);
  if (fit_out_host) memcpy(fit_out_host, rb->fit.p, (size_t)rb->M * kFitCounts * sizeof(int));
  return 0;
}

// The mesh slot of each of `M` objects.  The kernels index the mesh table with these ids unchecked, so an empty or
// out-of-range slot must be refused before anything is enqueued.
int check_slots(const fp_ctx* c, int M, const int* slots, const char* caller) {
  for (int i = 0; i < M; ++i) {
    FP_REQUIRE(slots[i] >= 0 && slots[i] < kMaxMeshes, "%s: object %d: slot %d out of range [0, %d)", caller, i, slots[i],
               kMaxMeshes);
    FP_REQUIRE(c->mesh[slots[i]].loaded, "%s: object %d: slot %d holds no mesh", caller, i, slots[i]);
  }
  return 0;
}

// A depth sensor's values (fp_set_camera_depth_sensor, fp_align_depth): a size the kernels index in int, finite
// intrinsics and transform, and focal lengths > 0
int check_depth_sensor(const fp_depth_sensor_t* s, const char* caller) {
  FP_REQUIRE(s->H >= 1 && s->H <= FP_DEPTH_SENSOR_MAX_DIM && s->W >= 1 && s->W <= FP_DEPTH_SENSOR_MAX_DIM,
             "%s: depth image %d x %d outside [1, %d]", caller, s->H, s->W, FP_DEPTH_SENSOR_MAX_DIM);
  for (int k = 0; k < 9; ++k) FP_REQUIRE(isfinite(s->K[k]), "%s: K[%d] = %g is not finite", caller, k, (double)s->K[k]);
  for (int k = 0; k < 16; ++k)
    FP_REQUIRE(isfinite(s->T_color_from_depth[k]), "%s: T_color_from_depth[%d] = %g is not finite", caller, k,
               (double)s->T_color_from_depth[k]);
  FP_REQUIRE(s->K[0] > 0.f && s->K[4] > 0.f, "%s: focal lengths fx = %g, fy = %g must be > 0", caller, (double)s->K[0],
             (double)s->K[4]);
  return 0;
}

// The frames of C cameras and the camera of each of M objects: non-null frames of positive size, every camera id in
// [0, C) and every camera owning at least one object.  The kernels index the camera table with these ids unchecked.
static int check_cameras(int C, const unsigned char* const* rgb, const float* const* depth, const int* H, const int* W,
                         int M, const int* camera_of, const char* caller) {
  FP_REQUIRE(C >= 1 && C <= kMaxCameras, "%s: %d cameras, need 1..%d", caller, C, kMaxCameras);
  for (int i = 0; i < C; ++i) {
    FP_REQUIRE(rgb[i] && depth[i], "%s: camera %d: null frame", caller, i);
    FP_REQUIRE(H[i] > 0 && W[i] > 0, "%s: camera %d: empty frame (%d x %d)", caller, i, H[i], W[i]);
  }
  std::vector<int> owns(C, 0);
  for (int i = 0; i < M; ++i) {
    FP_REQUIRE(camera_of[i] >= 0 && camera_of[i] < C, "%s: object %d: camera %d out of range [0, %d)", caller, i, camera_of[i], C);
    owns[camera_of[i]] = 1;
  }
  for (int i = 0; i < C; ++i) FP_REQUIRE(owns[i], "%s: camera %d owns no object", caller, i);
  return 0;
}

// fp_register_cameras and fp_register_objects after validation (n_hyp_host is checked here, before anything is
// enqueued).  Object i is seen by camera camera_of[i]; its mask is masks[i], of its camera's size.  Frames and masks on
// the context's device are read in place (frames through the camera table or camera 0's record, masks by device copies
// into mask_buf), host ones are staged; fp_register_objects' masks are one block, classified once.  Each pass copies
// its slot ids and per-hypothesis camera ids to the argument block, so the refine / feature graphs hold no per-pass
// address and are keyed on (kind, pass size, iterations, frame source).
//   by_value = false (fp_register_cameras): the camera table goes to the argument block once per call.  One
//     frame_prep_kernel launch filters every camera, the start-pose kernels read each object's depth, size and
//     intrinsics from the table, and the crops take their frame from it: the graphs hold no frame, so reordering
//     cameras or objects or changing intrinsics replays them.
//   by_value = true (fp_register_objects, C = 1): the frame filter, the start-pose kernels and the crop producer take
//     camera 0's record by value (the single-camera kernel instantiations), as fp_register does, and its graphs are
//     captured again when that record changes (run_graphed).  Kept for speed: at 252 hypotheses the crop producer's
//     camera-table instantiation runs 3.6 % longer (2.76 against 2.67 ms of crops per one-object call, H100 80GB HBM3
//     at 700 W), the one camera-table kernel whose cost shows.  Tracking's few hypotheses show none, so
//     fp_track_objects shares fp_track_cameras' table path.
// Both: whole objects in the given order in passes of up to kRegisterPassCap hypotheses (an object above the cap alone),
// then one segmented scorer tail over all objects.  Synchronises.
static int register_cameras_body(fp_ctx* c, int C, const unsigned char* const* rgb, const float* const* depth,
                                 const float* K, const int* H, const int* W, int M, const int* camera_of, const int* slots_host,
                                 const int* n_hyp_host, const unsigned char* const* masks, const float* rot_grids_dev,
                                 int iterations, float* poses_out_dev, float* scores_out_dev, int* best_out_dev,
                                 float* info_out_dev, cudaStream_t st, bool by_value) {
  const char* caller = by_value ? "fp_register_objects" : "fp_register_cameras";
  std::vector<int> off(M + 1, 0);
  for (int i = 0; i < M; ++i) {
    FP_REQUIRE(n_hyp_host[i] >= 1 && n_hyp_host[i] <= 4096, "%s: object %d: %d hypotheses, need 1..4096", caller, i,
               n_hyp_host[i]);
    off[i + 1] = off[i] + n_hyp_host[i];
  }
  FrameSources on_dev;
  FP_TRY(frame_sources(c, C, rgb, depth, on_dev, caller));
  FP_TRY(check_frame_formats(c, C, depth, W, caller));
  std::vector<char> mask_on_dev(M, 0);
  for (int i = 0; i < M; ++i) {
    bool d = false;
    if (by_value && i > 0)
      d = mask_on_dev[0];
    else
      FP_TRY(read_in_place(c, masks[i], d, caller, by_value ? "the mask block starting at object" : "the mask of object", i));
    mask_on_dev[i] = d;
  }
  const bool staged_masks = std::find(mask_on_dev.begin(), mask_on_dev.end(), 0) != mask_on_dev.end();
  FP_TRY(order_after_track(c, st));
  const int total = off[M];
  // passes: whole objects in the given order, up to kRegisterPassCap hypotheses; an object above the cap alone
  std::vector<int> pass_obj(1, 0);  // first object of every pass, then M
  for (int i = 1; i < M; ++i)
    if (off[i + 1] - off[pass_obj.back()] > kRegisterPassCap) pass_obj.push_back(i);
  pass_obj.push_back(M);
  int max_pass = 0;
  for (size_t p = 0; p + 1 < pass_obj.size(); ++p) max_pass = std::max(max_pass, off[pass_obj[p + 1]] - off[pass_obj[p]]);
  // each object's mask at its byte offset of one block
  std::vector<size_t> mask_at(M + 1, 0);
  for (int i = 0; i < M; ++i) mask_at[i + 1] = mask_at[i] + (size_t)H[camera_of[i]] * W[camera_of[i]];
  const size_t mask_bytes = mask_at[M];
  // every workspace is sized for the largest pass here, so no pass bumps the graph epoch
  FP_TRY(ensure_capacity(c, max_pass));
  FP_TRY(ensure_tail(c, total));
  FP_TRY(dev_alloc(&c->epoch, c->reg_feats, (size_t)total * 512 * sizeof(float)));
  FP_TRY(dev_alloc(&c->epoch, c->mask_buf, mask_bytes));
  FP_TRY(dev_alloc(&c->epoch, c->mask_stats, (size_t)M * 6 * sizeof(unsigned int)));
  if (!by_value) FP_TRY(dev_alloc(&c->epoch, c->mask_off, (size_t)M * sizeof(size_t)));
  // pinned staging (never read by a captured graph): the copies below leave as soon as they are enqueued
  StagingSet* set;
  FP_TRY(take_set(c, set));
  // every return from here on, a failure's included, leaves the set busy until the copies enqueued from it have left it
  struct MarkBusy {
    StagingSet& set;
    cudaStream_t st;
    ~MarkBusy() { set_busy(set, st); }
  } mark_busy{*set, st};
  if (staged_masks) FP_TRY(pinned_alloc(nullptr, set->masks, mask_bytes));
  FP_TRY(pinned_alloc(nullptr, set->ints, (size_t)(2 * M + 2) * sizeof(int) + (size_t)M * sizeof(size_t)));
  c->has_frame = false;
  CallFrames g;
  FP_TRY(setup_cameras(c, *set, C, rgb, depth, on_dev, K, H, W, max_pass, total, st, g));
  int* ints = reinterpret_cast<int*>(set->ints.p);
  size_t* stage_mask_off = reinterpret_cast<size_t*>(ints + 2 * M + 2);
  memcpy(ints, off.data(), (size_t)(M + 1) * sizeof(int));
  memcpy(ints + M + 1, camera_of, (size_t)M * sizeof(int));
  memcpy(stage_mask_off, mask_at.data(), (size_t)M * sizeof(size_t));
  for (int i = 0; i < M; ++i)
    if (!mask_on_dev[i])
      memcpy(static_cast<unsigned char*>(set->masks.p) + mask_at[i], masks[i], mask_at[i + 1] - mask_at[i]);
  // the ids of the pass starting at row r0 are staged at 2 * r0 after the table: its slot ids, then its camera ids
  int* ids = reinterpret_cast<int*>(static_cast<char*>(set->args.p) + kHeadBytes);
  for (size_t p = 0; p + 1 < pass_obj.size(); ++p) {
    const int row0 = off[pass_obj[p]], n = off[pass_obj[p + 1]] - row0;
    for (int i = pass_obj[p]; i < pass_obj[p + 1]; ++i) {
      std::fill(ids + row0 + off[i], ids + row0 + off[i + 1], slots_host[i]);
      std::fill(ids + row0 + n + off[i], ids + row0 + n + off[i + 1], camera_of[i]);
    }
  }
  // seg_off: the offsets [M + 1], then the camera ids [M]; the scorer tail at the end runs over these segments
  ScoreTailParams tp;
  FP_TRY(segmented_tail_params(c, reinterpret_cast<const float*>(c->reg_feats.p), ints, M, /*trailing=*/M, scores_out_dev,
                               best_out_dev, st, caller, tp));
  // the masks into mask_buf: every run of staged masks in one copy (all of them in one when every mask is on the host),
  // every run of device masks that follow each other in the caller's memory in one device-to-device copy
  for (int i = 0, j; i < M; i = j) {
    for (j = i + 1; j < M && mask_on_dev[j] == mask_on_dev[i]; ++j)
      if (mask_on_dev[j] && masks[j] != masks[j - 1] + (mask_at[j] - mask_at[j - 1])) break;
    unsigned char* dst = static_cast<unsigned char*>(c->mask_buf.p) + mask_at[i];
    const size_t bytes = mask_at[j] - mask_at[i];
    if (mask_on_dev[i])
      FP_CUDA_OK(cudaMemcpyAsync(dst, masks[i], bytes, cudaMemcpyDeviceToDevice, st));
    else
      FP_CUDA_OK(cudaMemcpyAsync(dst, static_cast<unsigned char*>(set->masks.p) + mask_at[i], bytes, cudaMemcpyHostToDevice, st));
  }
  const CameraDev* cams_dev = by_value ? nullptr : reinterpret_cast<const CameraDev*>(c->args.p);
  // estimater.py:173-174, :214 once per camera for every object: erode + bilateral, depth2xyzmap(zfar = inf)
  if (by_value) {
    const unsigned char* rgb0 = on_dev.rgb[0] ? rgb[0] : static_cast<const unsigned char*>(c->cam[0].rgb_raw.p);
    const float* depth0 = on_dev.depth[0] ? depth[0] : static_cast<const float*>(c->cam[0].depth_raw.p);
    const FrameFmtDev fmt0 = *reinterpret_cast<const FrameFmtDev*>(static_cast<const char*>(set->args.p) + kTableBytes);
    const SensorDev s0 = *reinterpret_cast<const SensorDev*>(static_cast<const char*>(set->args.p) + kSensorsAt);
    if (s0.aligned) depth0 = reinterpret_cast<const float*>(s0.aligned);  // fmt0 is then aligned_fmt
    FP_TRY(set_frame_launches(c, rgb0, depth0, fmt0, FP_FRAME_FILTER_DEPTH, INFINITY, st, s0.aligned ? &s0 : nullptr));
  } else {
    const FrameFmtDev* fmts_dev = reinterpret_cast<const FrameFmtDev*>(static_cast<const char*>(c->args.p) + kTableBytes);
    FP_CUDA_OK(cudaMemcpyAsync(c->args.p, set->args.p, kHeadBytes, cudaMemcpyHostToDevice, st));
    FP_CUDA_OK(cudaMemcpyAsync(c->mask_off.p, stage_mask_off, (size_t)M * sizeof(size_t), cudaMemcpyHostToDevice, st));
    if (g.aligned) {
      const SensorDev* sensors_dev = reinterpret_cast<const SensorDev*>(static_cast<const char*>(c->args.p) + kSensorsAt);
      FP_CUDA_OK(cudaMemsetAsync(c->aligned.p, 0, (size_t)C * c->aligned_stride * 4, st));
      FP_TRY(align_depth_cameras_launch(sensors_dev, cams_dev, C, g.Hd_max, g.Wd_max, st));
    }
    FP_TRY(frame_prep_cameras_launch(cams_dev, fmts_dev, C, g.H_max, g.W_max, INFINITY, st));
  }
  c->has_frame = true;
  // estimater.py:137-156, :203-209 for every object in one launch pair; the start poses go to poses_out_dev and are
  // replaced pass by pass with the refined ones
  const int* seg = reinterpret_cast<const int*>(c->seg_off.p);
  const unsigned char* masks_dev = reinterpret_cast<const unsigned char*>(c->mask_buf.p);
  unsigned int* stats = reinterpret_cast<unsigned int*>(c->mask_stats.p);
  const size_t* mask_off = reinterpret_cast<const size_t*>(c->mask_off.p);
  FP_TRY(start_poses_launch(camera_dev(c, 0), cams_dev, seg + M + 1, masks_dev, mask_off, rot_grids_dev, total, M, seg, stats,
                            poses_out_dev, info_out_dev, st));
  float* pa = reinterpret_cast<float*>(c->poses_a.p);
  float* pb = reinterpret_cast<float*>(c->poses_b.p);
  float* ps = reinterpret_cast<float*>(c->pose_stage.p);
  float* fb = reinterpret_cast<float*>(c->feat_buf.p);
  const int* mesh_of = reinterpret_cast<const int*>(static_cast<const char*>(c->args.p) + kHeadBytes);
  const float* fin = (iterations % 2 == 0) ? pa : pb;
  const int frame = by_value ? -1 : 0;  // from the table: prepared above, outside the graphs
  for (size_t p = 0; p + 1 < pass_obj.size(); ++p) {
    const int row0 = off[pass_obj[p]], n = off[pass_obj[p + 1]] - row0;
    const int* hyp_cam = by_value ? nullptr : mesh_of + n;
    // the pass's slot and camera ids and its start poses go to fixed context buffers and its outputs are copied out
    // after the replays: the graphs hold no per-pass address
    FP_CUDA_OK(cudaMemcpyAsync(static_cast<char*>(c->args.p) + kHeadBytes, ids + 2 * row0, (size_t)2 * n * sizeof(int),
                               cudaMemcpyHostToDevice, st));
    FP_CUDA_OK(cudaMemcpyAsync(pa, poses_out_dev + (size_t)row0 * 16, (size_t)n * 64, cudaMemcpyDeviceToDevice, st));
    FP_TRY(run_graphed(
        c, GraphKind::RegisterRefine, n, iterations, st,
        [&](cudaStream_t s2) -> int { return refine_body(c, n, iterations, s2, mesh_of, cams_dev, hyp_cam); }, frame));
    FP_CUDA_OK(cudaMemcpyAsync(poses_out_dev + (size_t)row0 * 16, fin, (size_t)n * 64, cudaMemcpyDeviceToDevice, st));
    FP_CUDA_OK(cudaMemcpyAsync(ps, fin, (size_t)n * 64, cudaMemcpyDeviceToDevice, st));
    FP_TRY(run_graphed(
        c, GraphKind::RegisterFeatures, n, 0, st,
        [&](cudaStream_t s2) -> int {
          FP_TRY(make_crops(c, ps, n, 1, nullptr, nullptr, nullptr, s2, mesh_of, cams_dev, hyp_cam));
          FP_TRY(run_encoder(c, c->net[1], reinterpret_cast<const __half*>(c->crops.p), n, s2));
          return run_score_feats(c, c->net[1], n, fb, s2);
        },
        frame));
    FP_CUDA_OK(cudaMemcpyAsync(reinterpret_cast<float*>(c->reg_feats.p) + (size_t)row0 * 512, fb, (size_t)n * 2048,
                               cudaMemcpyDeviceToDevice, st));
  }
  // score_network.py:84-88 per object: one tail launch, each object's hypotheses attending only to each other
  FP_TRY(score_tail_launch(tp, st));
  FP_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace fp

using namespace fp;

extern "C" {

int fp_create(fp_ctx** out) {
  FP_API_BEGIN
  if (!out) {
    set_last_error("fp_create: null output");
    return -1;
  }
  int dev = 0;
  FP_CUDA_OK(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  FP_CUDA_OK(cudaGetDeviceProperties(&prop, dev));
  FP_REQUIRE(prop.major == 9 && prop.minor == 0, "libfpose targets sm_90a (H100); device %d is sm_%d%d", dev, prop.major,
             prop.minor);
  fp_ctx* c = new fp_ctx();
  c->device = dev;
  const char* ng = getenv("FPOSE_NO_GRAPH");
  c->use_graphs = !(ng && ng[0] == '1');
  const char* nc = getenv("FPOSE_NO_CULL");
  c->cull_backfaces = !(nc && nc[0] == '1');
  if (const char* fk = getenv("FPOSE_FORK_MAX_N")) c->fork_max_n = atoi(fk);
  *out = c;
  return 0;
  FP_API_END
}

int fp_destroy(fp_ctx* c) {
  FP_API_BEGIN
  if (!c) return 0;
  DeviceGuard dg(c->device);
  cudaDeviceSynchronize();  // calls still in flight finish; their uncollected read-backs are freed with the context
  for (auto& kv : c->graphs)
    if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
  if (c->cap_stream) cudaStreamDestroy(c->cap_stream);
  if (c->side_stream) cudaStreamDestroy(c->side_stream);
  if (c->ev_fork) cudaEventDestroy(c->ev_fork);
  if (c->ev_join) cudaEventDestroy(c->ev_join);
  delete c;  // the buffers free themselves, with the context's device current
  return 0;
  FP_API_END
}

int fp_set_config(fp_ctx* c, int which, float crop_ratio, float rot_normalizer) {
  FP_API_BEGIN
  FP_REQUIRE(c, "null ctx");
  FP_REQUIRE(which == 0 || which == 1, "fp_set_config: which must be 0 (refiner) or 1 (scorer)");
  FP_REQUIRE(crop_ratio > 0.f, "fp_set_config: crop_ratio must be positive");
  DeviceGuard dg(c->device);
  c->crop_ratio[which] = crop_ratio;
  if (which == 0) c->rot_normalizer = rot_normalizer;
  ++c->epoch;
  if (c->mesh_table.p) FP_TRY(write_mesh_table(c));  // the table holds r3 = diameter * crop_ratio / 2
  return 0;
  FP_API_END
}

int fp_set_mesh_slot(fp_ctx* c, int slot, int V, int F, const float* pos, const float* nrm, const float* uv,
                     const float* vcol, const int* faces, const unsigned char* tex_rgb, int Ht, int Wt, float diameter) {
  FP_API_BEGIN
  FP_REQUIRE(c && pos && nrm && faces, "fp_set_mesh: null argument");
  FP_REQUIRE(slot >= 0 && slot < kMaxMeshes, "fp_set_mesh_slot: slot %d out of range [0, %d)", slot, kMaxMeshes);
  FP_REQUIRE(V > 0 && F > 0 && diameter > 0.f, "fp_set_mesh: empty mesh");
  FP_REQUIRE((uv && tex_rgb && Ht > 0 && Wt > 0) || vcol, "fp_set_mesh: need (uv + texture) or vertex colours");
  for (int i = 0; i < 3 * F; ++i) FP_REQUIRE(faces[i] >= 0 && faces[i] < V, "fp_set_mesh: face index out of range");
  DeviceGuard dg(c->device);
  // graphs rendering the previous mesh of this slot may still be running on the caller's stream
  FP_CUDA_OK(cudaDeviceSynchronize());
  MeshSlot& m = c->mesh[slot];
  m.loaded = false;
  const bool has_tex = (uv && tex_rgb);
  MeshHost mh;
  FP_TRY(build_mesh_host(V, F, pos, nrm, has_tex ? uv : vcol, has_tex ? 2 : 3, faces, mh));
  FP_TRY(upload(&c->epoch, m.vpos, mh.vpos));
  FP_TRY(upload(&c->epoch, m.vnrm, mh.vnrm));
  FP_TRY(upload(&c->epoch, m.vatt, mh.vatt));
  FP_TRY(upload(&c->epoch, m.faces, mh.faces));
  FP_TRY(upload(&c->epoch, m.meshlets, mh.meshlets));
  FP_TRY(upload(&c->epoch, m.ml_verts, mh.ml_verts));
  FP_TRY(upload(&c->epoch, m.ml_tris, mh.ml_tris));
  m.has_tex = has_tex;
  if (has_tex) {
    std::vector<unsigned char> rgba((size_t)Ht * Wt * 4);
    for (size_t i = 0; i < (size_t)Ht * Wt; ++i) {
      rgba[4 * i] = tex_rgb[3 * i];
      rgba[4 * i + 1] = tex_rgb[3 * i + 1];
      rgba[4 * i + 2] = tex_rgb[3 * i + 2];
      rgba[4 * i + 3] = 255;
    }
    FP_TRY(upload(&c->epoch, m.tex, rgba));
    m.Ht = Ht;
    m.Wt = Wt;
  }
  m.V = V;
  m.F = F;
  m.n_meshlets = (int)mh.meshlets.size();
  m.front_sign = mh.front_sign;
  m.closed = mh.closed;
  for (int i = 0; i < 4; ++i) m.bs[i] = mh.bs[i];
  m.diameter = diameter;
  m.loaded = true;
  FP_TRY(write_mesh_table(c));
  return 0;
  FP_API_END
}

int fp_set_mesh(fp_ctx* c, int V, int F, const float* pos, const float* nrm, const float* uv, const float* vcol,
                const int* faces, const unsigned char* tex_rgb, int Ht, int Wt, float diameter) {
  return fp_set_mesh_slot(c, 0, V, F, pos, nrm, uv, vcol, faces, tex_rgb, Ht, Wt, diameter);
}

int fp_set_crop_tile(fp_ctx* c, int tile) {
  FP_API_BEGIN
  FP_REQUIRE(c && (tile == 0 || tile == 16 || tile == 32 || tile == 80), "fp_set_crop_tile: tile must be 0 (automatic), 16, 32 or 80");
  c->crop_tile = tile;
  ++c->epoch;
  return 0;
  FP_API_END
}

int fp_set_camera_format(fp_ctx* c, int camera, const fp_frame_format_t* fmt) {
  FP_API_BEGIN
  FP_REQUIRE(c, "fp_set_camera_format: null ctx");
  FP_REQUIRE(camera >= 0 && camera < kMaxCameras, "fp_set_camera_format: camera %d out of range [0, %d)", camera, kMaxCameras);
  if (!fmt) {
    c->fmt[camera] = fp_frame_format_t{};
    return 0;
  }
  FP_REQUIRE(fmt->color >= FP_COLOR_RGB8 && fmt->color <= FP_COLOR_BGRA8, "fp_set_camera_format: camera %d: unknown colour format %d",
             camera, fmt->color);
  FP_REQUIRE(fmt->depth == FP_DEPTH_F32 || fmt->depth == FP_DEPTH_U16, "fp_set_camera_format: camera %d: unknown depth format %d",
             camera, fmt->depth);
  FP_REQUIRE(fmt->depth != FP_DEPTH_U16 || (isfinite(fmt->depth_scale) && fmt->depth_scale > 0.f),
             "fp_set_camera_format: camera %d: uint16 depth scale %g must be finite and > 0 (metres per unit)", camera,
             (double)fmt->depth_scale);
  c->fmt[camera] = *fmt;
  return 0;
  FP_API_END
}

int fp_set_camera_depth_sensor(fp_ctx* c, int camera, const fp_depth_sensor_t* s) {
  FP_API_BEGIN
  FP_REQUIRE(c, "fp_set_camera_depth_sensor: null ctx");
  FP_REQUIRE(camera >= 0 && camera < kMaxCameras, "fp_set_camera_depth_sensor: camera %d out of range [0, %d)", camera,
             kMaxCameras);
  if (!s) {
    c->has_sensor[camera] = false;
    c->sensor[camera] = fp_depth_sensor_t{};
    return 0;
  }
  FP_TRY(check_depth_sensor(s, "fp_set_camera_depth_sensor"));
  c->sensor[camera] = *s;
  c->has_sensor[camera] = true;
  return 0;
  FP_API_END
}

int fp_mesh_info(fp_ctx* c, int* info) {
  FP_API_BEGIN
  FP_REQUIRE(c && info && c->mesh[0].loaded, "fp_mesh_info: no mesh");
  const MeshSlot& m = c->mesh[0];
  info[0] = m.n_meshlets;
  info[1] = m.closed;
  info[2] = c->cull_backfaces ? m.front_sign : 0;
  info[3] = m.V;
  info[4] = m.F;
  return 0;
  FP_API_END
}

int fp_set_frame(fp_ctx* c, const unsigned char* rgb, const float* depth, const float* K, int H, int W, int flags,
                 float zfar, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && rgb && depth && K, "fp_set_frame: null argument");
  FP_REQUIRE(H > 0 && W > 0, "fp_set_frame: empty frame");
  FP_TRY(check_frame_format(c, 0, depth, W, "fp_set_frame"));
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  const size_t npix = (size_t)H * W;
  c->has_frame = false;
  const bool on_dev = (flags & FP_FRAME_ON_DEVICE) != 0;
  int Hd, Wd;  // the depth image: the colour frame's size, or its depth sensor's
  depth_size(c, 0, H, W, Hd, Wd);
  const FrameLayout L = frame_layout(c->fmt[0], W, Wd);
  FP_TRY(alloc_camera(c, 0, npix, /*raw=*/!on_dev, L.rgb_bpp, L.depth_bpp, (size_t)Hd * Wd));
  if (c->has_sensor[0]) FP_TRY(ensure_aligned(c, 1, npix));
  set_frame_geometry(c, 0, K, H, W);
  c->n_frames = 1;
  const unsigned char* rgb_dev = rgb;
  const float* depth_dev = depth;
  if (!on_dev) {
    CameraBufs& f = c->cam[0];
    if (residence(c, rgb) == Residence::Pageable || residence(c, depth) == Residence::Pageable) {
      StagingSet* set;
      FP_TRY(take_set(c, set));
      const int staged = upload_staged_frame(f, set->rgb[0], set->depth[0], rgb, depth, L, H, Hd, st);
      FP_TRY(set_busy(*set, st));
      FP_TRY(staged);
    } else {
      // page-locked frames, fp_group_register's among them, are read in place: one host copy fewer
      FP_TRY(copy_rows(f.rgb_raw.p, rgb, L.rgb_row, L.rgb_pitch, H, st));
      FP_TRY(copy_rows(f.depth_raw.p, depth, L.depth_row, L.depth_pitch, Hd, st));
    }
    rgb_dev = reinterpret_cast<const unsigned char*>(f.rgb_raw.p);
    depth_dev = reinterpret_cast<const float*>(f.depth_raw.p);
  }
  FrameFmtDev fmt = fmt_dev(c->fmt[0], L, on_dev, on_dev);
  if (c->has_sensor[0]) {
    const SensorDev s = sensor_dev(c, 0, depth_dev, L, on_dev);
    FP_TRY(set_frame_launches(c, rgb_dev, reinterpret_cast<const float*>(s.aligned), aligned_fmt(fmt, W), flags, zfar, st, &s));
  } else {
    FP_TRY(set_frame_launches(c, rgb_dev, depth_dev, fmt, flags, zfar, st));
  }
  c->has_frame = true;
  return 0;
  FP_API_END
}

int fp_set_xyz_map(fp_ctx* c, const float* xyz, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && xyz, "fp_set_xyz_map: null argument");
  FP_REQUIRE(c->has_frame, "fp_set_xyz_map: no frame (call fp_set_frame first)");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  // [H][W][3] (host or device) -> the float4-per-pixel layout the crop kernel samples
  const CameraBufs& f = c->cam[0];
  FP_CUDA_OK(cudaMemcpy2DAsync(f.xyz.p, 16, xyz, 12, 12, (size_t)f.H * f.W, cudaMemcpyDefault, st));
  return 0;
  FP_API_END
}

int fp_get_depth(fp_ctx* c, int camera, float* depth_out_dev, float* xyz_out_dev, int* hw_out, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && c->has_frame, "fp_get_depth: no frame");
  FP_REQUIRE(camera >= 0 && camera < c->n_frames, "fp_get_depth: camera %d: the last call prepared cameras 0..%d", camera,
             c->n_frames - 1);
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  const CameraBufs& b = c->cam[camera];
  if (hw_out) {
    hw_out[0] = b.H;
    hw_out[1] = b.W;
  }
  const size_t npix = (size_t)b.H * b.W;
  if (depth_out_dev) FP_CUDA_OK(cudaMemcpyAsync(depth_out_dev, b.depth.p, npix * 4, cudaMemcpyDeviceToDevice, st));
  // internal layout is float4 per pixel; the hook returns the reference's [H][W][3]
  if (xyz_out_dev) FP_CUDA_OK(cudaMemcpy2DAsync(xyz_out_dev, 12, b.xyz.p, 16, 12, npix, cudaMemcpyDeviceToDevice, st));
  return 0;
  FP_API_END
}

int fp_start_poses(fp_ctx* c, const unsigned char* mask, int mask_on_device, const float* rot_grid, int N, float* poses_out,
                   float* info_out, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && mask && rot_grid && poses_out && info_out && N >= 0, "fp_start_poses: bad argument");
  FP_REQUIRE(c->has_frame, "fp_start_poses: no frame (call fp_set_frame first)");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  const CameraDev frame = camera_dev(c, 0);
  const size_t npix = (size_t)frame.H * frame.W;
  const unsigned char* mdev = mask;
  if (!mask_on_device) {
    FP_TRY(dev_alloc(&c->epoch, c->mask_buf, npix));
    FP_TRY(upload_host(c, c->mask_buf.p, mask, npix, &StagingSet::masks, st));
    mdev = reinterpret_cast<const unsigned char*>(c->mask_buf.p);
  }
  FP_TRY(dev_alloc(&c->epoch, c->mask_stats, 64));
  return start_poses_launch(frame, nullptr, nullptr, mdev, nullptr, rot_grid, N, 1, nullptr,
                            reinterpret_cast<unsigned int*>(c->mask_stats.p), poses_out, info_out, st);
  FP_API_END
}

int fp_make_crops(fp_ctx* c, const float* poses, int N, int mode, void* crops_out, float* dbg_out, float* win_out,
                  void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && poses && N >= 0, "fp_make_crops: bad argument");
  FP_REQUIRE(mode == 0 || mode == 1, "fp_make_crops: mode must be 0 (refiner) or 1 (scorer)");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  if (N == 0) return 0;
  FP_TRY(ensure_capacity(c, N));
  FP_TRY(make_crops(c, poses, N, mode, dbg_out, win_out, nullptr, st));
  if (crops_out) FP_TRY(crops_export(c, crops_out, N, st));
  return 0;
  FP_API_END
}

int fp_crop_stats(fp_ctx* c, const float* poses, int N, int mode, int* stats_out_host, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && poses && stats_out_host && N > 0, "fp_crop_stats: bad argument");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  FP_TRY(ensure_capacity(c, N));
  FP_TRY(dev_alloc(&c->epoch, c->crop_stats, 16));
  FP_CUDA_OK(cudaMemsetAsync(c->crop_stats.p, 0, 16, st));
  FP_TRY(make_crops(c, poses, N, mode, nullptr, nullptr, reinterpret_cast<int*>(c->crop_stats.p), st));
  FP_CUDA_OK(cudaMemcpyAsync(stats_out_host, c->crop_stats.p, 16, cudaMemcpyDeviceToHost, st));
  FP_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
  FP_API_END
}

int fp_refine(fp_ctx* c, const float* poses_in, int N, int iterations, float* poses_out, float* last_trans,
              float* last_rot, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && poses_in && poses_out && N >= 0 && iterations >= 0, "fp_refine: bad argument");
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  FP_REQUIRE(c->mesh[0].loaded && c->has_frame, "fp_refine: needs fp_set_mesh and fp_set_frame first");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  if (N == 0) return 0;
  FP_TRY(ensure_capacity(c, N));
  float* pa = reinterpret_cast<float*>(c->poses_a.p);
  float* pb = reinterpret_cast<float*>(c->poses_b.p);
  FP_CUDA_OK(cudaMemcpyAsync(pa, poses_in, (size_t)N * 64, cudaMemcpyDeviceToDevice, st));
  FP_TRY(run_graphed(c, GraphKind::Refine, N, iterations, st,
                     [&](cudaStream_t s2) -> int { return refine_body(c, N, iterations, s2); }));
  const float* fin = (iterations % 2 == 0) ? pa : pb;
  FP_CUDA_OK(cudaMemcpyAsync(poses_out, fin, (size_t)N * 64, cudaMemcpyDeviceToDevice, st));
  if (iterations > 0) {
    if (last_trans) FP_CUDA_OK(cudaMemcpyAsync(last_trans, c->lt_buf.p, (size_t)N * 12, cudaMemcpyDeviceToDevice, st));
    if (last_rot) FP_CUDA_OK(cudaMemcpyAsync(last_rot, c->lr_buf.p, (size_t)N * 36, cudaMemcpyDeviceToDevice, st));
  }
  return 0;
  FP_API_END
}

int fp_score_features(fp_ctx* c, const float* poses, int N, float* feats_out, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && poses && feats_out && N >= 0, "fp_score_features: bad argument");
  FP_REQUIRE(c->net[1].loaded, "scorer weights not loaded");
  FP_REQUIRE(c->mesh[0].loaded && c->has_frame, "fp_score_features: needs fp_set_mesh and fp_set_frame first");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  if (N == 0) return 0;
  FP_TRY(ensure_capacity(c, N));
  float* ps = reinterpret_cast<float*>(c->pose_stage.p);
  float* fb = reinterpret_cast<float*>(c->feat_buf.p);
  FP_CUDA_OK(cudaMemcpyAsync(ps, poses, (size_t)N * 64, cudaMemcpyDeviceToDevice, st));
  auto body = [&](cudaStream_t s2) -> int {
    FP_TRY(make_crops(c, ps, N, 1, nullptr, nullptr, nullptr, s2));
    FP_TRY(run_encoder(c, c->net[1], reinterpret_cast<const __half*>(c->crops.p), N, s2));
    FP_TRY(run_score_feats(c, c->net[1], N, fb, s2));
    return 0;
  };
  FP_TRY(run_graphed(c, GraphKind::ScoreFeatures, N, 0, st, body));
  // feats_out may live on another GPU of the same process (peer access enabled by fp_group_create): the gather of
  // the sharded register is this copy, device to device over NVLink
  FP_CUDA_OK(cudaMemcpyAsync(feats_out, fb, (size_t)N * 2048, cudaMemcpyDefault, st));
  return 0;
  FP_API_END
}

int fp_score_tail(fp_ctx* c, const float* feats, int L, float* scores_out, int* best_out, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && feats && scores_out && L >= 0, "fp_score_tail: bad argument");
  FP_REQUIRE(c->net[1].loaded, "scorer weights not loaded");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  if (L == 0) return 0;
  FP_TRY(ensure_tail(c, L));
  return score_tail_launch(score_tail_params(c, feats, L, scores_out, best_out), st);
  FP_API_END
}

int fp_score(fp_ctx* c, const float* poses, int N, float* scores_out, int* best_out, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && poses && scores_out && N >= 0, "fp_score: bad argument");
  if (N == 0) return 0;
  DeviceGuard dg(c->device);
  FP_TRY(ensure_capacity(c, N));
  FP_TRY(fp_score_features(c, poses, N, reinterpret_cast<float*>(c->feats.p), stream));
  return fp_score_tail(c, reinterpret_cast<const float*>(c->feats.p), N, scores_out, best_out, stream);
  FP_API_END
}

int fp_register(fp_ctx* c, const float* poses_host, int N, int iterations, float* poses_out_host, float* scores_out_host,
                int* best_out_host, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && poses_host && poses_out_host && scores_out_host && best_out_host && N > 0, "fp_register: bad argument");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  FP_TRY(ensure_capacity(c, N));
  FP_TRY(ensure_tail(c, N));
  // the start poses go up to pose_stage, which fp_refine reads before its loop and takes its result back into; the
  // refined poses then move to poses_b (idle after the loop), since fp_score stages its input in pose_stage
  float* ps = reinterpret_cast<float*>(c->pose_stage.p);
  FP_TRY(upload_host(c, ps, poses_host, (size_t)N * 64, &StagingSet::poses, st));
  FP_TRY(fp_refine(c, ps, N, iterations, ps, nullptr, nullptr, stream));
  float* refined = reinterpret_cast<float*>(c->poses_b.p);
  FP_CUDA_OK(cudaMemcpyAsync(refined, ps, (size_t)N * 64, cudaMemcpyDeviceToDevice, st));
  FP_TRY(fp_score(c, refined, N, reinterpret_cast<float*>(c->scores.p), reinterpret_cast<int*>(c->best.p), stream));
  FP_CUDA_OK(cudaMemcpyAsync(poses_out_host, refined, (size_t)N * 64, cudaMemcpyDeviceToHost, st));
  FP_CUDA_OK(cudaMemcpyAsync(scores_out_host, c->scores.p, (size_t)N * 4, cudaMemcpyDeviceToHost, st));
  FP_CUDA_OK(cudaMemcpyAsync(best_out_host, c->best.p, 4, cudaMemcpyDeviceToHost, st));
  FP_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
  FP_API_END
}

int fp_track_submit(fp_ctx* c, const unsigned char* rgb, const float* depth, const float* K, int H, int W,
                    const float* pose_in_dev, int iterations, float* pose_out_dev, void* stream, unsigned long long* ticket) {
  FP_API_BEGIN
  FP_REQUIRE(c && rgb && depth && K && H > 0 && W > 0 && iterations >= 0 && ticket, "fp_track: bad argument");
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  FP_REQUIRE(c->mesh[0].loaded, "fp_track: no mesh");
  FP_REQUIRE(pose_in_dev || c->track_valid, "fp_track: no previous pose in this context: pass pose_in");
  DeviceGuard dg(c->device);
  FP_TRY(dev_alloc(nullptr, c->track_pose, 64));  // the continuation pose is copied outside the graph
  float* keep = reinterpret_cast<float*>(c->track_pose.p);
  // fp_track_cameras' one-object, one-camera case: object 0 renders slot 0 in camera 0
  const int zero = 0;
  FP_TRY(track_cameras_submit(c, "fp_track", 1, &rgb, &depth, K, &H, &W, 1, &zero, &zero, pose_in_dev ? pose_in_dev : keep,
                              iterations, pose_out_dev, reinterpret_cast<cudaStream_t>(stream), ticket, keep));
  c->track_valid = true;
  return 0;
  FP_API_END
}

int fp_track(fp_ctx* c, const unsigned char* rgb, const float* depth, const float* K, int H, int W,
             const float* pose_in_dev, int iterations, float* pose_out_dev, float* pose_out_host, void* stream) {
  unsigned long long ticket = 0;
  const int rc = fp_track_submit(c, rgb, depth, K, H, W, pose_in_dev, iterations, pose_out_dev, stream, &ticket);
  return rc ? rc : fp_track_wait(c, ticket, pose_out_host);
}

int fp_track_wait(fp_ctx* c, unsigned long long ticket, float* poses_out_host) {
  FP_API_BEGIN
  FP_REQUIRE(c, "fp_track_wait: null ctx");
  DeviceGuard dg(c->device);
  return track_wait(c, ticket, poses_out_host);
  FP_API_END
}

int fp_track_fit_wait(fp_ctx* c, unsigned long long ticket, float* poses_out_host, int* fit_out_host) {
  FP_API_BEGIN
  FP_REQUIRE(c, "fp_track_fit_wait: null ctx");
  DeviceGuard dg(c->device);
  return track_wait(c, ticket, poses_out_host, /*fit=*/true, fit_out_host);
  FP_API_END
}

int fp_vis_size(int kind, int N, int* hw_out) {
  FP_API_BEGIN
  FP_REQUIRE(hw_out, "fp_vis_size: null output");
  return vis_canvas_size(kind, N, hw_out, hw_out + 1);
  FP_API_END
}

int fp_vis_colormap(unsigned char* rgb_out) {
  FP_API_BEGIN
  FP_REQUIRE(rgb_out, "fp_vis_colormap: null output");
  const unsigned* t = vis_colormap();
  for (int i = 0; i < 256; ++i)
    for (int ch = 0; ch < 3; ++ch) rgb_out[3 * i + ch] = (unsigned char)(t[i] >> (16 - 8 * ch));
  return 0;
  FP_API_END
}

int fp_vis_crops(fp_ctx* c, const float* poses, int N, int mode, float* rec_out, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && poses && rec_out && N > 0 && (mode == 0 || mode == 1), "fp_vis_crops: bad argument");
  DeviceGuard dg(c->device);
  FP_TRY(order_after_track(c, reinterpret_cast<cudaStream_t>(stream)));
  FP_TRY(ensure_capacity(c, N));
  return make_crops(c, poses, N, mode, nullptr, nullptr, nullptr, reinterpret_cast<cudaStream_t>(stream), nullptr, nullptr,
                    nullptr, reinterpret_cast<float4*>(rec_out));
  FP_API_END
}

unsigned long long fp_vis_workspace_bytes(fp_ctx* c) { return c ? (unsigned long long)(c->vis_rec.bytes + c->vis_range.bytes) : 0ull; }

int fp_vis(fp_ctx* c, int kind, const float* poses_a, const float* poses_b, int N, const int* order, unsigned char* canvas_out,
           int* hw_out, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && poses_a && canvas_out && N > 0 && (kind == 0 || kind == 1), "fp_vis: bad argument");
  FP_REQUIRE(kind == 1 || poses_b, "fp_vis: the refiner canvas needs the refined poses (poses_b)");
  FP_REQUIRE(kind == 0 || order, "fp_vis: the scorer canvas needs the row order");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(order_after_track(c, st));
  int hw[2];
  FP_TRY(vis_canvas_size(kind, N, hw, hw + 1));
  if (hw_out) {
    hw_out[0] = hw[0];
    hw_out[1] = hw[1];
  }
  FP_TRY(ensure_capacity(c, N));
  // no captured graph holds the vis buffers (fp_vis runs eagerly): growing them must not invalidate the cached graphs
  FP_TRY(dev_alloc(nullptr, c->vis_rec, (size_t)N * 2 * S * S * sizeof(float4)));
  FP_TRY(dev_alloc(nullptr, c->vis_range, (size_t)N * sizeof(float2)));
  float4* rec = reinterpret_cast<float4*>(c->vis_rec.p);
  float2* range = reinterpret_cast<float2*>(c->vis_range.p);
  if (kind == 0) {
    // predict_pose_refine.py:241-293: one crop pass at the start poses (left half), one at the refined poses (right)
    for (int blk = 0; blk < 2; ++blk) {
      FP_TRY(make_crops(c, blk ? poses_b : poses_a, N, 0, nullptr, nullptr, nullptr, st, nullptr, nullptr, nullptr, rec));
      FP_TRY(vis_range_launch(rec, N, 2, range, st));
      FP_TRY(vis_refine_launch(rec, range, N, blk, canvas_out, st));
    }
  } else {
    // predict_score.py:219-224 + :27-52: the scorer's crops, depth range of the rendered image, rows in `order`
    FP_TRY(make_crops(c, poses_a, N, 1, nullptr, nullptr, nullptr, st, nullptr, nullptr, nullptr, rec));
    FP_TRY(vis_range_launch(rec, N, 1, range, st));
    FP_TRY(vis_score_launch(rec, range, order, N, canvas_out, st));
  }
  return 0;
  FP_API_END
}

int fp_track_objects_submit(fp_ctx* c, const unsigned char* rgb, const float* depth, const float* K, int H, int W,
                            int M, const int* slots_host, const float* poses_in_dev, int iterations, float* poses_out_dev,
                            void* stream, unsigned long long* ticket) {
  FP_API_BEGIN
  FP_REQUIRE(c && rgb && depth && K && H > 0 && W > 0 && M > 0 && slots_host && poses_in_dev && iterations >= 0 &&
                 ticket,
             "fp_track_objects: bad argument");
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  FP_TRY(check_slots(c, M, slots_host, "fp_track_objects"));
  DeviceGuard dg(c->device);
  const std::vector<int> camera_of(M, 0);
  return track_cameras_submit(c, "fp_track_objects", 1, &rgb, &depth, K, &H, &W, M, camera_of.data(), slots_host, poses_in_dev,
                              iterations, poses_out_dev, reinterpret_cast<cudaStream_t>(stream), ticket);
  FP_API_END
}

int fp_track_objects(fp_ctx* c, const unsigned char* rgb, const float* depth, const float* K, int H, int W, int M,
                     const int* slots_host, const float* poses_in_dev, int iterations, float* poses_out_dev,
                     float* poses_out_host, void* stream) {
  unsigned long long ticket = 0;
  const int rc = fp_track_objects_submit(c, rgb, depth, K, H, W, M, slots_host, poses_in_dev, iterations,
                                         poses_out_dev, stream, &ticket);
  return rc ? rc : fp_track_wait(c, ticket, poses_out_host);
}

int fp_track_cameras_submit(fp_ctx* c, int C, const unsigned char* const* rgb, const float* const* depth,
                            const float* K, const int* H, const int* W, int M, const int* camera_of, const int* slots_host,
                            const float* poses_in_dev, int iterations, float* poses_out_dev, void* stream,
                            unsigned long long* ticket) {
  FP_API_BEGIN
  FP_REQUIRE(c && rgb && depth && K && H && W && M > 0 && camera_of && slots_host && poses_in_dev && iterations >= 0 &&
                 ticket,
             "fp_track_cameras: bad argument");
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  // everything is checked before anything is enqueued: the kernels index the mesh and camera tables unchecked
  FP_TRY(check_cameras(C, rgb, depth, H, W, M, camera_of, "fp_track_cameras"));
  FP_TRY(check_slots(c, M, slots_host, "fp_track_cameras"));
  DeviceGuard dg(c->device);
  return track_cameras_submit(c, "fp_track_cameras", C, rgb, depth, K, H, W, M, camera_of, slots_host, poses_in_dev, iterations,
                              poses_out_dev, reinterpret_cast<cudaStream_t>(stream), ticket);
  FP_API_END
}

int fp_track_cameras_fit_submit(fp_ctx* c, int C, const unsigned char* const* rgb, const float* const* depth,
                                const float* K, const int* H, const int* W, int M, const int* camera_of,
                                const int* slots_host, const float* poses_in_dev, int iterations, float delta,
                                float* poses_out_dev, int* fit_out_dev, void* stream, unsigned long long* ticket) {
  FP_API_BEGIN
  FP_REQUIRE(c && rgb && depth && K && H && W && M > 0 && camera_of && slots_host && poses_in_dev && iterations >= 0 &&
                 ticket,
             "fp_track_cameras_fit: bad argument");
  FP_REQUIRE(isfinite(delta) && delta >= 0.f, "fp_track_cameras_fit: delta %g must be finite and >= 0 (metres)", (double)delta);
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  FP_TRY(check_cameras(C, rgb, depth, H, W, M, camera_of, "fp_track_cameras_fit"));
  FP_TRY(check_slots(c, M, slots_host, "fp_track_cameras_fit"));
  DeviceGuard dg(c->device);
  return track_cameras_submit(c, "fp_track_cameras_fit", C, rgb, depth, K, H, W, M, camera_of, slots_host, poses_in_dev,
                              iterations, poses_out_dev, reinterpret_cast<cudaStream_t>(stream), ticket, nullptr, &delta,
                              fit_out_dev);
  FP_API_END
}

int fp_track_cameras(fp_ctx* c, int C, const unsigned char* const* rgb, const float* const* depth, const float* K,
                     const int* H, const int* W, int M, const int* camera_of, const int* slots_host, const float* poses_in_dev,
                     int iterations, float* poses_out_dev, float* poses_out_host, void* stream) {
  unsigned long long ticket = 0;
  const int rc = fp_track_cameras_submit(c, C, rgb, depth, K, H, W, M, camera_of, slots_host, poses_in_dev,
                                         iterations, poses_out_dev, stream, &ticket);
  return rc ? rc : fp_track_wait(c, ticket, poses_out_host);
}

int fp_register_objects(fp_ctx* c, const unsigned char* rgb, const float* depth, const float* K, int H, int W,
                        int M, const int* slots_host, const int* n_hyp_host, const unsigned char* masks,
                        const float* rot_grids_dev, int iterations, float* poses_out_dev, float* scores_out_dev,
                        int* best_out_dev, float* info_out_dev, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && rgb && depth && K && H > 0 && W > 0 && M > 0 && M <= 65535 && slots_host && n_hyp_host &&
                 masks && rot_grids_dev && iterations >= 0 && poses_out_dev && scores_out_dev && best_out_dev &&
                 info_out_dev,
             "fp_register_objects: bad argument");
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  FP_REQUIRE(c->net[1].loaded, "scorer weights not loaded");
  // everything is checked before anything is enqueued
  FP_TRY(check_slots(c, M, slots_host, "fp_register_objects"));
  DeviceGuard dg(c->device);
  const size_t npix = (size_t)H * W;
  std::vector<const unsigned char*> mask_of(M);
  for (int i = 0; i < M; ++i) mask_of[i] = masks + (size_t)i * npix;
  const std::vector<int> camera_of(M, 0);
  return register_cameras_body(c, 1, &rgb, &depth, K, &H, &W, M, camera_of.data(), slots_host, n_hyp_host,
                               mask_of.data(), rot_grids_dev, iterations, poses_out_dev, scores_out_dev, best_out_dev,
                               info_out_dev, reinterpret_cast<cudaStream_t>(stream), /*by_value=*/true);
  FP_API_END
}

int fp_register_cameras(fp_ctx* c, int C, const unsigned char* const* rgb, const float* const* depth, const float* K,
                        const int* H, const int* W, int M, const int* camera_of, const int* slots_host, const int* n_hyp_host,
                        const unsigned char* const* masks, const float* rot_grids_dev, int iterations,
                        float* poses_out_dev, float* scores_out_dev, int* best_out_dev, float* info_out_dev, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && rgb && depth && K && H && W && M > 0 && M <= 65535 && camera_of && slots_host && n_hyp_host &&
                 masks && rot_grids_dev && iterations >= 0 && poses_out_dev && scores_out_dev && best_out_dev &&
                 info_out_dev,
             "fp_register_cameras: bad argument");
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  FP_REQUIRE(c->net[1].loaded, "scorer weights not loaded");
  // everything is checked before anything is enqueued: the kernels index the mesh and camera tables unchecked
  FP_TRY(check_cameras(C, rgb, depth, H, W, M, camera_of, "fp_register_cameras"));
  for (int i = 0; i < M; ++i) FP_REQUIRE(masks[i], "fp_register_cameras: object %d: null mask", i);
  FP_TRY(check_slots(c, M, slots_host, "fp_register_cameras"));
  DeviceGuard dg(c->device);
  return register_cameras_body(c, C, rgb, depth, K, H, W, M, camera_of, slots_host, n_hyp_host, masks,
                               rot_grids_dev, iterations, poses_out_dev, scores_out_dev, best_out_dev, info_out_dev,
                               reinterpret_cast<cudaStream_t>(stream), /*by_value=*/false);
  FP_API_END
}

unsigned long long fp_graph_captures(fp_ctx* c) { return c ? c->graph_captures : 0ull; }

}  // extern "C"
