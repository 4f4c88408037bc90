// fp_ctx.cuh — internal to libfpose: the context behind the C ABI (include/fpose.h), its owning buffer types and
// allocation helpers, and the host functions that more than one translation unit of the ABI calls.
#pragma once
#include <algorithm>
#include <exception>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "../../include/fpose.h"
#include "fp_attn.cuh"
#include "fp_common.cuh"
#include "fp_crop.cuh"

namespace fp {

// An allocation that `Free` releases when its owner goes away or grows it.  Move-only: every allocation has one owner,
// so destroying a context, a mesh slot or a replaced weight tensor frees exactly what it held.  Device memory must be
// released with its device current.
template <cudaError_t (*Free)(void*)>
struct OwnedBuf {
  void* p = nullptr;
  size_t bytes = 0;
  OwnedBuf() = default;
  OwnedBuf(OwnedBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), bytes(std::exchange(o.bytes, 0)) {}
  OwnedBuf& operator=(OwnedBuf&& o) noexcept {
    if (this != &o) {
      reset();
      p = std::exchange(o.p, nullptr);
      bytes = std::exchange(o.bytes, 0);
    }
    return *this;
  }
  ~OwnedBuf() { reset(); }
  void reset() {
    if (p) Free(p);
    p = nullptr;
    bytes = 0;
  }
};
using DevBuf = OwnedBuf<cudaFree>;         // device memory
using PinnedBuf = OwnedBuf<cudaFreeHost>;  // page-locked host memory

// A CUDA event (timing disabled), created on first use and destroyed with its owner.  Move-only, as OwnedBuf.
struct OwnedEvent {
  cudaEvent_t e = nullptr;
  OwnedEvent() = default;
  OwnedEvent(OwnedEvent&& o) noexcept : e(std::exchange(o.e, nullptr)) {}
  OwnedEvent& operator=(OwnedEvent&& o) noexcept {
    if (this != &o) {
      if (e) cudaEventDestroy(e);
      e = std::exchange(o.e, nullptr);
    }
    return *this;
  }
  ~OwnedEvent() {
    if (e) cudaEventDestroy(e);
  }
  cudaError_t record(cudaStream_t st) {
    if (!e) {
      const cudaError_t ce = cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
      if (ce != cudaSuccess) return ce;
    }
    return cudaEventRecord(e, st);
  }
};

// (Re)allocates `b` to at least `bytes`.  `epoch` is the owning context's graph epoch, or null where no captured graph
// holds b's address: it is bumped whenever a device pointer or by-value kernel parameter that a captured CUDA graph may
// hold changes (re-allocation, new weights / intrinsics), and cached graphs older than it are rebuilt.  Never called
// while a stream is capturing:
// every workspace is sized by ensure_capacity / fp_set_mesh_slot / fp_set_frame BEFORE run_graphed.  A tracking call
// still in flight may be reading the buffer being replaced, so growing one waits for the device first.
inline int dev_alloc(unsigned long long* epoch, DevBuf& b, size_t bytes, bool zero = false) {
  if (b.bytes >= bytes && b.p) return 0;
  if (epoch) ++*epoch;
  if (b.p) FP_CUDA_OK(cudaDeviceSynchronize());
  b.reset();
  FP_CUDA_OK(cudaMalloc(&b.p, bytes));
  b.bytes = bytes;
  if (zero) {
    // legacy-stream memset + full synchronisation: the consumers run on the caller's (possibly non-blocking) stream
    FP_CUDA_OK(cudaMemset(b.p, 0, bytes));
    FP_CUDA_OK(cudaDeviceSynchronize());
  }
  return 0;
}
template <class T>
int upload(unsigned long long* epoch, DevBuf& b, const std::vector<T>& v) {
  const size_t bytes = std::max<size_t>(v.size() * sizeof(T), 16);
  if (dev_alloc(epoch, b, bytes)) return -2;
  if (!v.empty()) FP_CUDA_OK(cudaMemcpy(b.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  return 0;
}

// (Re)allocates pinned `b` to at least `bytes` (cudaHostAlloc `flags`).  `epoch`: the graph epoch of the context whose
// captured graph holds b's address (a read-back node), bumped when the address changes; null where no graph holds it.
inline int pinned_alloc(unsigned long long* epoch, PinnedBuf& b, size_t bytes, unsigned flags = cudaHostAllocDefault) {
  if (b.bytes >= bytes && b.p) return 0;
  if (epoch) ++*epoch;
  b.reset();
  FP_CUDA_OK(cudaHostAlloc(&b.p, bytes, flags));
  b.bytes = bytes;
  return 0;
}

struct Tensor {
  DevBuf buf;
  int dtype = 0;  // 0 = f32, 1 = f16
  long long numel = 0;
};

struct Net {
  std::map<std::string, Tensor> t;
  bool loaded = false;
  // fp_load_network verified that every name the execution plan uses is present; a miss is a programming error
  // and surfaces as an exception that the extern "C" wrappers turn into an error code
  const __half* h(const char* name) const { return reinterpret_cast<const __half*>(t.at(name).buf.p); }
  const float* f(const char* name) const { return reinterpret_cast<const float*>(t.at(name).buf.p); }
};

constexpr int S = 160;
constexpr int T = 400;
// fp_register_objects refines and featurises whole objects in passes of at most this many hypotheses (an object above
// it gets a pass of its own).  ensure_capacity costs ~15.6 MB per hypothesis, so the context keeps ~8 GB of workspace
// after such a call; the largest buffer (refiner qkv, N * 400 * 3072 fp16) is 1.26 GB, and every element and byte
// offset inside a buffer stays below 2^31.
constexpr int kRegisterPassCap = 512;
constexpr size_t kCropImg = (size_t)(S + 6) * (S + 8) * 8;  // fp16 elements per padded crop image
// The encoder's first stage runs on the A (rendered) and B (observed) crops as one batch.  The 40x40
// 128-channel layers tile four images per MMA (gemm_swap_patch_kernel), and the layer that fuses
// torch.cat((a, b), 1) stores A and B tiles to different channel halves, so the A/B boundary must fall on a tile
// boundary: B starts at N rounded up to 4 (up to three never-read pad images).
inline int b_img0_of(int N) { return (N + 3) & ~3; }

static_assert(kMaxMeshes == FP_MAX_MESHES, "fp_crop.cuh and fpose.h disagree on the number of mesh slots");
static_assert(kMaxCameras == FP_MAX_CAMERAS, "fp_crop.cuh and fpose.h disagree on the number of cameras");
static_assert(kFitCounts == FP_FIT_COUNTS, "fp_crop.cuh and fpose.h disagree on the number of fit counts");

// One mesh of the context (fp_meshlet.cu layout).  Slot 0 is the mesh of every single-object entry point.
struct MeshSlot {
  DevBuf vpos, vnrm, vatt, faces, meshlets, ml_verts, ml_tris, tex;
  int V = 0, F = 0, Ht = 0, Wt = 0, n_meshlets = 0, front_sign = 0, closed = 0;
  float bs[4] = {0.f, 0.f, 0.f, 0.f};
  bool has_tex = false, loaded = false;
  float diameter = 0.f;
};

// One camera's frame: the raw upload and the filtered frame (rgba, depth, xyz), and the size and intrinsics of the frame
// the last call prepared in this camera.  Camera 0 is the context's frame, the one every single-frame entry point reads
// (see alloc_camera).  camera_dev() makes the kernels' record of it.
struct CameraBufs {
  DevBuf rgb_raw, depth_raw, rgba, depth, xyz;
  int H = 0, W = 0;
  float fx = 0.f, fy = 0.f, cx = 0.f, cy = 0.f;
};

// All pinned staging of host inputs.  The tracking calls keep up to FP_TRACK_MAX_IN_FLIGHT calls in flight, each
// uploading through a staging set of its own: the host copies the next call's frames while the device still tracks the
// previous call.  Only the host side is doubled: the device buffers the uploads land in are ordered by the stream.
// Every call that stages pageable host memory takes the next set in turn (take_set) and marks it busy after its last
// copy out of it (set_busy): a set is busy until `uploaded`, recorded after that copy, has passed.
constexpr int kMaxInFlight = FP_TRACK_MAX_IN_FLIGHT;
struct StagingSet {
  PinnedBuf rgb[kMaxCameras], depth[kMaxCameras];
  PinnedBuf args;  // the camera table, then the slot ids and camera ids (layout of fp_ctx::args)
  // the register calls' masks of every object at its byte offset, and their (offsets [M + 1], camera ids [M], one int of
  // padding, each object's mask byte offset size_t [M]); fp_start_poses' mask; fp_register's start poses
  PinnedBuf masks, ints, poses;
  OwnedEvent uploaded;
  bool busy = false;
};

// The pose read-back of one submitted tracking call: pinned [M][16] poses, and with a fit (fp_track_cameras_fit_submit)
// its [M][FP_FIT_COUNTS] counts, complete once `done` has passed.  Owned by the call's ticket until fp_track_wait or
// fp_track_fit_wait collects it (ticket 0: free for the next submit).  A call's read-back outlives its staging set, which
// the call after next may reuse before this result is collected.
struct Readback {
  PinnedBuf poses, fit;
  OwnedEvent done;
  unsigned long long ticket = 0;
  int M = 0;
  bool has_fit = false;
};

}  // namespace fp

struct fp_ctx {
  int device = 0;
  fp::Net net[2];  // 0 = refiner, 1 = scorer
  unsigned long long epoch = 1;  // graph epoch (see dev_alloc)
  unsigned long long graph_captures = 0;
  // meshes, and their device table (MeshSlotDev [FP_MAX_MESHES]) that kernels index by slot.  Captured graphs hold only
  // the table's address: loading a slot rewrites its entry in place and needs no new capture.
  fp::MeshSlot mesh[fp::kMaxMeshes];
  fp::DevBuf mesh_table;
  float rot_normalizer = 0.3490658503988659f;
  float crop_ratio[2] = {1.2f, 1.2f};  // per predictor: each reads its own config.yml (predict_pose_refine.py:117, predict_score.py:137)
  // frames: cam[0] is the context's frame, cameras 1.. those of the multi-camera calls
  fp::CameraBufs cam[fp::kMaxCameras];
  int n_frames = 0;  // the last call prepared the frames of cameras 0 .. n_frames - 1
  // every camera's frame format (fp_set_camera_format; all zero = packed RGB8 + float32), read when a call is staged
  fp_frame_format_t fmt[fp::kMaxCameras] = {};
  // every camera's depth sensor (fp_set_camera_depth_sensor), read when a call is staged; has_sensor false: the depth
  // is in the colour frame's geometry
  fp_depth_sensor_t sensor[fp::kMaxCameras] = {};
  bool has_sensor[fp::kMaxCameras] = {};
  // the aligned buffers of a call's cameras: camera i's [H][W] uint32 slots at slot i * aligned_stride, zeroed by one
  // memset per call and scattered into by align_depth_kernel; aligned_stride only grows (and moves the graph epoch)
  fp::DevBuf aligned;
  size_t aligned_stride = 0;
  bool has_frame = false;
  // workspaces (sized for cap_n hypotheses)
  int cap_n = 0;
  fp::DevBuf crops, act0, a1, a2, a3, ab0, ab1, ab2, c0, c1, c2, tok, qkv, att, x1pre, x1, ff, x2pre;
  fp::DevBuf head_out, poses_a, poses_b, feats, tail_qkv, tail_attn, scores, best;
  int tail_cap = 0;
  float fold_c = 0.f;      // linear.weight . out_proj.bias + linear.bias (by-value kernel parameter)
  fp::DevBuf fold_v, tail_counter;  // out_proj^T linear.weight [512]; arg-max ticket
  // CUDA graphs of the launch-bound inner loops, keyed by (kind, N, iterations, frame source: see run_graphed).
  // frame: camera 0's record when the graph was captured (read by a graph that takes the frame by value)
  struct GraphEntry {
    cudaGraphExec_t exec = nullptr;
    unsigned long long epoch = 0;
    fp::CameraDev frame{};
  };
  std::map<std::tuple<int, int, int, int>, GraphEntry> graphs;
  std::map<std::tuple<int, int, int, int>, int> graph_nodes;
  cudaStream_t cap_stream = nullptr;
  // the refiner's two decoder heads are independent after the shared attention core: at small batches
  // (one linear layer = 1-2 waves of tiles) the second head runs on `side_stream` so that its kernels fill
  // the SMs the first head's tail wave leaves idle.  Fork / join are events, captured into the graph.
  cudaStream_t side_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  int fork_max_n = 128;  // FPOSE_FORK_MAX_N; 0 disables.  Measured (profiles/r02_fork_probe.log): -5 % at 32, -1 % at 126, +1 % at 252 hypotheses
  bool use_graphs = true;
  bool cull_backfaces = true;  // FPOSE_NO_CULL=1: render both sides even for closed meshes (A/B checks)
  bool track_valid = false;
  int crop_tile = 0;
  fp::DevBuf lt_buf, lr_buf, feat_buf, pose_stage, tok_mean;
  fp::DevBuf mask_buf, mask_stats, crop_stats;
  fp::DevBuf op_mesh_of;  // fp_op_pose_update: the uploaded slot id of every hypothesis
  fp::DevBuf track_pose;      // fp_track: the pose it produced last, where pose_in = NULL continues from
  // the tracking calls in flight: their staging sets (used in turn), their read-backs by ticket, the last ticket issued,
  // and the stream and completion event (after the read-back) of the last call submitted
  fp::StagingSet sets[fp::kMaxInFlight];
  int next_set = 0;
  std::vector<std::unique_ptr<fp::Readback>> readbacks;
  unsigned long long last_ticket = 0;
  cudaStream_t last_stream = nullptr;
  cudaEvent_t last_done = nullptr;  // the last call's Readback::done (a Readback is reused only by a later call)
  // the arguments of a multi-object call or register pass, one device block at a fixed address (a graph holds it),
  // staged through a StagingSet: the camera table (CameraDev [FP_MAX_CAMERAS]), the slot ids [n], the camera ids [n],
  // and for a tracking call with a fit its threshold (one float)
  fp::DevBuf args;
  fp::DevBuf fit;  // the fit counts of the last tracking call with a fit, [M][FP_FIT_COUNTS] int32 (a graph holds it)
  int cam_grid_h = 0, cam_grid_w = 0;  // the tracking calls' frame-preparation grid: the largest frame seen
  int sensor_grid_h = 0, sensor_grid_w = 0;  // the tracking calls' alignment grid: the largest depth image seen
  // fp_register_objects / _cameras: row offsets of the objects' hypotheses [M + 1] and the objects' camera ids [M], the
  // objects' feature rows [sum N][512], each object's byte offset into mask_buf
  fp::DevBuf seg_off, reg_feats, mask_off;
  // fp_vis: the crop producer's vis record [N][2][160][160] float4 and the per-row depth ranges [N] float2, sized at the
  // first call for the largest N seen; never allocated by the other entry points
  fp::DevBuf vis_rec, vis_range;
};

namespace fp {

// RAII: make the context's device current for the duration of an entry point
struct DeviceGuard {
  int prev = -1;
  bool switched = false;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) switched = cudaSetDevice(dev) == cudaSuccess;
  }
  ~DeviceGuard() {
    if (switched) cudaSetDevice(prev);
  }
};

// The encoder's activation buffers, as the layer table names them
enum EncBuf : int { EB_NONE = -1, EB_CROPS, EB_ACT0, EB_A1, EB_A2, EB_A3, EB_AB0, EB_AB1, EB_AB2, EB_C0, EB_C1, EB_C2, EB_TOK };

// One layer of the encoder (encodeA + encodeAB of refine_network.py:34-50, encoderA + encoderAB of
// score_network.py:37-51), BatchNorm folded, ReLU after every layer.  Weights "enc.<layer>.w" / "enc.<layer>.b".
struct EncLayer {
  int kind;
  bool ab_batch;    // runs on the M = Np + N images of the A and B crops (Np = b_img0_of(N)), else on the N pairs
  int H;            // input height = width
  int Cin, Cout;
  EncBuf in, out, res;
  int out_ld;       // 0: Cout
  bool split;       // out_split = Np: image n < Np -> image n, channels [0, Cout); n >= Np -> image n - Np, [Cout, 2 Cout)
  bool pe;          // adds the positional embedding "pe" after the ReLU
};

// The encoder, in launch order: run_encoder, fp_op_encoder and fp_op_encoder_layer all read this table.  Every
// residual block's second layer adds the block's input, which the buffer rotation keeps until then.
constexpr int kEncLayers = 15;
extern const EncLayer kEncoder[kEncLayers];  // fp_net.cu

// fp_net.cu: the network execution plan on the context's workspaces
int ensure_capacity(fp_ctx* c, int N);
int ensure_tail(fp_ctx* c, int L);
void* enc_buf(fp_ctx* c, const __half* crops, EncBuf b);
void enc_out_shape(int k, int N, int shape[4]);
int enc_source(int k, EncBuf b);
int run_encoder(fp_ctx* c, const Net& net, const __half* crops, int N, cudaStream_t st, int last = kEncLayers - 1);
int run_refine_heads(fp_ctx* c, const Net& net, int N, cudaStream_t st);
int run_score_feats(fp_ctx* c, const Net& net, int N, float* feats, cudaStream_t st);
int crops_import(fp_ctx* c, const void* ext, int N, cudaStream_t st);
int crops_export(fp_ctx* c, void* ext, int N, cudaStream_t st);
ScoreTailParams score_tail_params(const fp_ctx* c, const float* feats, int L, float* scores, int* best);
int segmented_tail_params(fp_ctx* c, const float* feats, const int* off_host, int n_seg, int trailing, float* scores,
                          int* best, cudaStream_t st, const char* caller, ScoreTailParams& p);

// fp_api.cu
int order_after_track(fp_ctx* c, cudaStream_t st);
int check_slots(const fp_ctx* c, int M, const int* slots, const char* caller);
int check_depth_sensor(const fp_depth_sensor_t* s, const char* caller);

}  // namespace fp

// every entry point: exceptions never cross the C boundary, the context's device is current inside
#define FP_API_BEGIN try {
#define FP_API_END                                                        \
  }                                                                       \
  catch (const std::exception& e) {                                       \
    fp::set_last_error("%s: exception: %s", __func__, e.what());          \
    return -3;                                                            \
  }                                                                       \
  catch (...) {                                                           \
    fp::set_last_error("%s: unknown exception", __func__);                \
    return -3;                                                            \
  }
