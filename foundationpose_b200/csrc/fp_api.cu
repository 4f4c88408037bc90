// fp_api.cu — the product C ABI (include/fpose.h): context, weights, mesh, frame, and the per-frame
// hot loop (crops -> encoder -> heads -> pose update, K times; then scoring) enqueued on one stream
// with no host synchronisation.
#include <math.h>
#include <stdlib.h>
#include <string.h>

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
#include "fp_depth.cuh"
#include "fp_gemm.cuh"
#include "fp_vis.cuh"

namespace fp {
const char* get_last_error();

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

// (Re)allocates `b` to at least `bytes`.  `epoch` is the owning context's graph epoch: it is bumped whenever a device
// pointer or by-value kernel parameter that a captured CUDA graph may hold changes (re-allocation, new weights /
// intrinsics), and cached graphs older than it are rebuilt.  Never called while a stream is capturing:
// every workspace is sized by ensure_capacity / fp_set_mesh_slot / fp_set_frame BEFORE run_graphed.
static int dev_alloc(unsigned long long& epoch, DevBuf& b, size_t bytes, bool zero = false) {
  if (b.bytes >= bytes && b.p) return 0;
  ++epoch;
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
static int upload(unsigned long long& epoch, DevBuf& b, const std::vector<T>& v) {
  const size_t bytes = std::max<size_t>(v.size() * sizeof(T), 16);
  if (dev_alloc(epoch, b, bytes)) return -2;
  if (!v.empty()) FP_CUDA_OK(cudaMemcpy(b.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
  return 0;
}

// (Re)allocates pinned `b` to at least `bytes` (cudaHostAlloc `flags`).  `epoch`: the graph epoch of the context whose
// captured graph holds b's address (a read-back node), bumped when the address changes; null where no graph holds it.
static int pinned_alloc(unsigned long long* epoch, PinnedBuf& b, size_t bytes, unsigned flags = cudaHostAllocDefault) {
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
static inline int b_img0_of(int N) { return (N + 3) & ~3; }

static_assert(kMaxMeshes == FP_MAX_MESHES, "fp_crop.cuh and fpose.h disagree on the number of mesh slots");
static_assert(kMaxCameras == FP_MAX_CAMERAS, "fp_crop.cuh and fpose.h disagree on the number of cameras");

// One mesh of the context (fp_meshlet.cu layout).  Slot 0 is the mesh of every single-object entry point.
struct MeshSlot {
  DevBuf vpos, vnrm, vatt, faces, meshlets, ml_verts, ml_tris, tex;
  int V = 0, F = 0, Ht = 0, Wt = 0, n_meshlets = 0, front_sign = 0, closed = 0;
  float bs[4] = {0.f, 0.f, 0.f, 0.f};
  bool has_tex = false, loaded = false;
  float diameter = 0.f;
};

// Frame buffers of cameras 1.. of fp_track_cameras (camera 0 is the context's frame), sized for the largest frame seen,
// and the pinned staging of their uploads.
struct CameraBufs {
  DevBuf rgb_raw, depth_raw, rgba, depth, xyz;
  PinnedBuf stage_rgb, stage_depth;
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
  fp::DevBuf mesh_table, mesh_of;  // mesh_of: slot id of every hypothesis of an fp_register_objects pass
  float rot_normalizer = 0.3490658503988659f;
  float crop_ratio[2] = {1.2f, 1.2f};  // per predictor: each reads its own config.yml (predict_pose_refine.py:117, predict_score.py:137)
  // frame
  fp::DevBuf rgb_raw, rgba, depth_raw, depth_a, depth_b, xyz;
  const float* depth_cur = nullptr;
  float K[9] = {0};
  int H = 0, W = 0;
  bool has_frame = false;
  // workspaces (sized for cap_n hypotheses)
  int cap_n = 0;
  fp::DevBuf crops, act0, a1, a2, a3, ab0, ab1, ab2, c0, c1, c2, tok, qkv, att, x1pre, x1, ff, x2pre;
  fp::DevBuf head_out, poses_a, poses_b, feats, tail_qkv, tail_attn, tail_proj, scores, best;
  int tail_cap = 0;
  float fold_c = 0.f;      // linear.weight . out_proj.bias + linear.bias (by-value kernel parameter)
  fp::DevBuf fold_v, tail_counter;  // out_proj^T linear.weight [512]; arg-max ticket
  // CUDA graphs of the launch-bound inner loops, keyed by (kind, N, iterations, cameras).  K / H / W: the frame
  // geometry a graph that passes it by value was captured with
  struct GraphEntry {
    cudaGraphExec_t exec = nullptr;
    unsigned long long epoch = 0;
    float K[9] = {0};
    int H = 0, W = 0;
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
  // fp_track: pinned host staging (frame in, pose out) so that the whole frame is ONE graph launch
  fp::PinnedBuf stage_rgb, stage_depth, stage_pose;
  fp::DevBuf track_pose;
  fp::PinnedBuf stage_poses;  // fp_track_objects: pinned [M][16] pose read-back
  // fp_register_objects: row offsets of the objects' hypotheses [M + 1], their feature rows [sum N][512]; pinned staging
  // of the masks and of (offsets, per-hypothesis slot ids)
  fp::DevBuf seg_off, reg_feats;
  fp::PinnedBuf stage_masks, stage_ints;
  // fp_register_cameras: the camera table [FP_MAX_CAMERAS] (fixed size, so its address never changes), the camera id of
  // every hypothesis of a pass, each object's byte offset into mask_buf, and the pinned staging of the table and offsets
  fp::DevBuf reg_cams, reg_cam_of, mask_off;
  fp::PinnedBuf stage_cams;
  // fp_track_cameras: buffers of cameras 1..; the per-call arguments (camera table [FP_MAX_CAMERAS], slot ids [M],
  // camera ids [M]) as one device block and its pinned staging; the frame size its frame-preparation grid covers (the
  // largest seen)
  fp::CameraBufs cams[fp::kMaxCameras];
  fp::DevBuf cam_args;
  fp::PinnedBuf stage_args;
  int cam_grid_h = 0, cam_grid_w = 0;
  // fp_vis: the crop producer's vis record [N][2][160][160] float4 and the per-row depth ranges [N] float2, sized at the
  // first call for the largest N seen; never allocated by the other entry points
  fp::DevBuf vis_rec, vis_range;
};

namespace fp {

static int ensure_capacity(fp_ctx* c, int N) {
  if (N <= c->cap_n) return 0;
  const size_t n = (size_t)N;
  int rc = 0;
  // the crop buffer is zeroed once: the 3-pixel border is never written afterwards
  const size_t m = 2 * n + 3;  // A + pad + B images
  rc |= dev_alloc(c->epoch, c->crops, m * kCropImg * 2, true);
  rc |= dev_alloc(c->epoch, c->act0, m * 80 * 80 * 64 * 2);
  rc |= dev_alloc(c->epoch, c->a1, m * 1600 * 128 * 2);
  rc |= dev_alloc(c->epoch, c->a2, m * 1600 * 128 * 2);
  rc |= dev_alloc(c->epoch, c->a3, m * 1600 * 128 * 2);
  rc |= dev_alloc(c->epoch, c->ab0, n * 1600 * 256 * 2);
  rc |= dev_alloc(c->epoch, c->ab1, n * 1600 * 256 * 2);
  rc |= dev_alloc(c->epoch, c->ab2, n * 1600 * 256 * 2);
  rc |= dev_alloc(c->epoch, c->c0, n * T * 512 * 2);
  rc |= dev_alloc(c->epoch, c->c1, n * T * 512 * 2);
  rc |= dev_alloc(c->epoch, c->c2, n * T * 512 * 2);
  rc |= dev_alloc(c->epoch, c->tok, n * T * 512 * 2);
  rc |= dev_alloc(c->epoch, c->qkv, n * T * 3072 * 2);
  rc |= dev_alloc(c->epoch, c->att, 2 * n * T * 512 * 2);
  // x 2: one set per decoder head (they may run concurrently, see run_refine_heads)
  rc |= dev_alloc(c->epoch, c->x1pre, 2 * n * T * 512 * 2);
  rc |= dev_alloc(c->epoch, c->x1, 2 * n * T * 512 * 2);
  rc |= dev_alloc(c->epoch, c->ff, 2 * n * T * 512 * 2);
  rc |= dev_alloc(c->epoch, c->x2pre, 2 * n * T * 512 * 2);
  rc |= dev_alloc(c->epoch, c->head_out, 2 * n * 3 * 4);
  rc |= dev_alloc(c->epoch, c->poses_a, n * 16 * 4);
  rc |= dev_alloc(c->epoch, c->poses_b, n * 16 * 4);
  rc |= dev_alloc(c->epoch, c->feats, n * 512 * 4);
  rc |= dev_alloc(c->epoch, c->lt_buf, n * 3 * 4);
  rc |= dev_alloc(c->epoch, c->lr_buf, n * 9 * 4);
  rc |= dev_alloc(c->epoch, c->feat_buf, n * 512 * 4);
  rc |= dev_alloc(c->epoch, c->pose_stage, n * 16 * 4);
  rc |= dev_alloc(c->epoch, c->tok_mean, n * 512 * 4);
  if (rc) return -2;
  c->cap_n = N;
  return 0;
}

static int ensure_tail(fp_ctx* c, int L) {
  if (L <= c->tail_cap) return 0;
  int rc = 0;
  rc |= dev_alloc(c->epoch, c->tail_qkv, (size_t)L * 1536 * 4);
  rc |= dev_alloc(c->epoch, c->tail_attn, (size_t)L * 512 * 4);
  rc |= dev_alloc(c->epoch, c->tail_proj, (size_t)L * 512 * 4);
  rc |= dev_alloc(c->epoch, c->scores, (size_t)L * 4);
  rc |= dev_alloc(c->epoch, c->best, 16);
  if (rc) return -2;
  c->tail_cap = L;
  return 0;
}

static GemmLayer mk(int kind, int n_img, int H, int W, int Cin, int Cout, const void* in, const __half* w,
                    const float* b, void* out, int relu, const void* res = nullptr, int out_ld = 0, int out_split = 0,
                    const float* post_add = nullptr) {
  GemmLayer L;
  L.kind = kind;
  L.n_img = n_img;
  L.Hin = H;
  L.Win = W;
  L.Cin = Cin;
  L.Cout = Cout;
  L.in = in;
  L.w = w;
  L.bias = b;
  L.res = res;
  L.res_ld = Cout;
  L.out = out;
  L.out_ld = out_ld ? out_ld : Cout;
  L.out_split = out_split;
  L.post_add = post_add;
  L.relu = relu;
  return L;
}

#define FP_TRY(expr)         \
  do {                       \
    int _rc = (expr);        \
    if (_rc) return _rc;     \
  } while (0)

// crops [2N][166][168][8] -> tokens [N][400][512] (+ positional embedding)
static int run_encoder(fp_ctx* c, const Net& net, const __half* crops, int N, cudaStream_t st) {
  char wn[32], bn[32];
  auto W = [&](int i) { snprintf(wn, sizeof wn, "enc.%d.w", i); return net.h(wn); };
  auto B = [&](int i) { snprintf(bn, sizeof bn, "enc.%d.b", i); return net.f(bn); };
  const int Np = b_img0_of(N);
  const int M = Np + N;
  FP_TRY(gemm_layer_launch(mk(LK_CONV7_S2, M, S, S, 8, 64, crops, W(0), B(0), c->act0.p, 1), st));
  FP_TRY(gemm_layer_launch(mk(LK_CONV3_S2, M, 80, 80, 64, 128, c->act0.p, W(1), B(1), c->a1.p, 1), st));
  FP_TRY(gemm_layer_launch(mk(LK_CONV3_S1, M, 40, 40, 128, 128, c->a1.p, W(2), B(2), c->a2.p, 1), st));
  FP_TRY(gemm_layer_launch(mk(LK_CONV3_S1, M, 40, 40, 128, 128, c->a2.p, W(3), B(3), c->a3.p, 1, c->a1.p), st));
  FP_TRY(gemm_layer_launch(mk(LK_CONV3_S1, M, 40, 40, 128, 128, c->a3.p, W(4), B(4), c->a2.p, 1), st));
  // last encodeA layer writes straight into the 256-channel concat buffer (refine_network.py:85)
  FP_TRY(gemm_layer_launch(mk(LK_CONV3_S1, M, 40, 40, 128, 128, c->a2.p, W(5), B(5), c->ab0.p, 1, c->a3.p, 256, Np), st));
  FP_TRY(gemm_layer_launch(mk(LK_CONV3_S1, N, 40, 40, 256, 256, c->ab0.p, W(6), B(6), c->ab1.p, 1), st));
  FP_TRY(gemm_layer_launch(mk(LK_CONV3_S1, N, 40, 40, 256, 256, c->ab1.p, W(7), B(7), c->ab2.p, 1, c->ab0.p), st));
  FP_TRY(gemm_layer_launch(mk(LK_CONV3_S1, N, 40, 40, 256, 256, c->ab2.p, W(8), B(8), c->ab1.p, 1), st));
  FP_TRY(gemm_layer_launch(mk(LK_CONV3_S1, N, 40, 40, 256, 256, c->ab1.p, W(9), B(9), c->ab0.p, 1, c->ab2.p), st));
  FP_TRY(gemm_layer_launch(mk(LK_CONV3_S2, N, 40, 40, 256, 512, c->ab0.p, W(10), B(10), c->c0.p, 1), st));
  FP_TRY(gemm_layer_launch(mk(LK_CONV3_S1, N, 20, 20, 512, 512, c->c0.p, W(11), B(11), c->c1.p, 1), st));
  FP_TRY(gemm_layer_launch(mk(LK_CONV3_S1, N, 20, 20, 512, 512, c->c1.p, W(12), B(12), c->c2.p, 1, c->c0.p), st));
  FP_TRY(gemm_layer_launch(mk(LK_CONV3_S1, N, 20, 20, 512, 512, c->c2.p, W(13), B(13), c->c1.p, 1), st));
  FP_TRY(gemm_layer_launch(
      mk(LK_CONV3_S1, N, 20, 20, 512, 512, c->c1.p, W(14), B(14), c->tok.p, 1, c->c2.p, 0, 0, net.f("pe")), st));
  return 0;
}

// tokens -> (trans, rot) raw network outputs, [2][N][3] fp32 in head_out
static int run_refine_heads(fp_ctx* c, const Net& net, int N, cudaStream_t st) {
  const int M = N * T;
  // both heads' in_proj as one GEMM: [M,512] x [3072,512]^T
  FP_TRY(gemm_layer_launch(mk(LK_LINEAR, 1, 1, M, 512, 3072, c->tok.p, net.h("heads.in_w"), net.f("heads.in_b"), c->qkv.p, 0), st));
  AttnParams ap;
  ap.qkv = reinterpret_cast<const __half*>(c->qkv.p);
  ap.ld = 3072;
  ap.q_off = 0;
  ap.k_off = 512;
  ap.v_off = 1024;
  ap.group_col_stride = 1536;
  ap.n_groups = 2;
  ap.out = reinterpret_cast<__half*>(c->att.p);
  ap.ld_out = 512;
  ap.out_group_stride = (size_t)M * 512;
  ap.B = N;
  ap.T = T;
  ap.n_heads = 4;
  ap.scale = 0.08838834764831845f;
  FP_TRY(attn_core_launch(ap, st));
  const bool fork = N <= c->fork_max_n;
  if (fork) {
    if (!c->side_stream) {
      FP_CUDA_OK(cudaStreamCreateWithFlags(&c->side_stream, cudaStreamNonBlocking));
      FP_CUDA_OK(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
      FP_CUDA_OK(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
    }
    FP_CUDA_OK(cudaEventRecord(c->ev_fork, st));
    FP_CUDA_OK(cudaStreamWaitEvent(c->side_stream, c->ev_fork, 0));
  }
  for (int g = 0; g < 2; ++g) {
    cudaStream_t sg = (fork && g == 1) ? c->side_stream : st;
    char nm[48];
    auto H = [&](const char* s) { snprintf(nm, sizeof nm, "head%d.%s", g, s); return net.h(nm); };
    auto Fp = [&](const char* s) { snprintf(nm, sizeof nm, "head%d.%s", g, s); return net.f(nm); };
    const size_t off = (size_t)g * M * 512;
    const __half* att_g = reinterpret_cast<const __half*>(c->att.p) + off;
    __half* x1pre = reinterpret_cast<__half*>(c->x1pre.p) + off;
    __half* x1 = reinterpret_cast<__half*>(c->x1.p) + off;
    __half* ff = reinterpret_cast<__half*>(c->ff.p) + off;
    __half* x2pre = reinterpret_cast<__half*>(c->x2pre.p) + off;
    const __half* w;
    const float* b;
    w = H("out_w"); b = Fp("out_b");
    // the first kernel behind an event wait has a full (not programmatic) dependency
    if (fork && g == 1) pdl_skip_next();
    FP_TRY(gemm_layer_launch(mk(LK_LINEAR, 1, 1, M, 512, 512, att_g, w, b, x1pre, 0, c->tok.p), sg));
    const float* g1 = Fp("ln1_g");
    const float* b1 = Fp("ln1_b");
    FP_TRY(layernorm_launch(x1pre, x1, g1, b1, M, sg));
    w = H("ff1_w"); b = Fp("ff1_b");
    FP_TRY(gemm_layer_launch(mk(LK_LINEAR, 1, 1, M, 512, 512, x1, w, b, ff, 1), sg));
    w = H("ff2_w"); b = Fp("ff2_b");
    FP_TRY(gemm_layer_launch(mk(LK_LINEAR, 1, 1, M, 512, 512, ff, w, b, x2pre, 0, x1), sg));
    const float* g2 = Fp("ln2_g");
    const float* b2 = Fp("ln2_b");
    const float* fw = Fp("fin_w");
    const float* fb = Fp("fin_b");
    FP_TRY(head_final_launch(x2pre, g2, b2, fw, fb, reinterpret_cast<float*>(c->head_out.p) + (size_t)g * N * 3, N, T, 3, sg));
  }
  if (fork) {
    FP_CUDA_OK(cudaEventRecord(c->ev_join, c->side_stream));
    FP_CUDA_OK(cudaStreamWaitEvent(st, c->ev_join, 0));
    pdl_skip_next();  // the consumer of head_out joins two streams
  }
  return 0;
}

// tokens -> per-hypothesis 512-d features (score_network.py:72-74)
static int run_score_feats(fp_ctx* c, const Net& net, int N, float* feats, cudaStream_t st) {
  const int M = N * T;
  FP_TRY(gemm_layer_launch(mk(LK_LINEAR, 1, 1, M, 512, 1536, c->tok.p, net.h("att.in_w"), net.f("att.in_b"), c->qkv.p, 0), st));
  AttnParams ap;
  ap.qkv = reinterpret_cast<const __half*>(c->qkv.p);
  ap.ld = 1536;
  ap.q_off = 0;
  ap.k_off = 512;
  ap.v_off = 1024;
  ap.group_col_stride = 0;
  ap.n_groups = 1;
  ap.out = reinterpret_cast<__half*>(c->att.p);
  ap.ld_out = 512;
  ap.out_group_stride = 0;
  ap.B = N;
  ap.T = T;
  ap.n_heads = 4;
  ap.scale = 0.08838834764831845f;
  FP_TRY(attn_core_launch(ap, st));
  FP_TRY(token_mean_proj_launch(reinterpret_cast<const __half*>(c->att.p), net.f("att.out_w32"), net.f("att.out_b"),
                                reinterpret_cast<float*>(c->tok_mean.p), feats, N, T, st));
  return 0;
}

// external crop layout of the test hooks: [2N] images, A then B, contiguous
static int crops_import(fp_ctx* c, const void* ext, int N, cudaStream_t st) {
  const size_t img = kCropImg * 2;
  __half* dst = reinterpret_cast<__half*>(c->crops.p);
  const char* src = reinterpret_cast<const char*>(ext);
  FP_CUDA_OK(cudaMemcpyAsync(dst, src, (size_t)N * img, cudaMemcpyDeviceToDevice, st));
  FP_CUDA_OK(cudaMemcpyAsync(dst + (size_t)b_img0_of(N) * kCropImg, src + (size_t)N * img, (size_t)N * img,
                             cudaMemcpyDeviceToDevice, st));
  return 0;
}
static int crops_export(fp_ctx* c, void* ext, int N, cudaStream_t st) {
  const size_t img = kCropImg * 2;
  const __half* src = reinterpret_cast<const __half*>(c->crops.p);
  char* dst = reinterpret_cast<char*>(ext);
  FP_CUDA_OK(cudaMemcpyAsync(dst, src, (size_t)N * img, cudaMemcpyDeviceToDevice, st));
  FP_CUDA_OK(cudaMemcpyAsync(dst + (size_t)N * img, src + (size_t)b_img0_of(N) * kCropImg, (size_t)N * img,
                             cudaMemcpyDeviceToDevice, st));
  return 0;
}

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
  FP_TRY(dev_alloc(c->epoch, c->mesh_table, sizeof(MeshSlotDev) * kMaxMeshes, /*zero=*/true));
  std::vector<MeshSlotDev> table(kMaxMeshes);
  memset(table.data(), 0, sizeof(MeshSlotDev) * kMaxMeshes);
  for (int s = 0; s < kMaxMeshes; ++s)
    if (c->mesh[s].loaded) table[s] = mesh_entry(c, s);
  FP_CUDA_OK(cudaMemcpy(c->mesh_table.p, table.data(), sizeof(MeshSlotDev) * kMaxMeshes, cudaMemcpyHostToDevice));
  FP_CUDA_OK(cudaDeviceSynchronize());
  return 0;
}

// mesh_of: [N] device slot ids (validated by the caller), or null = every hypothesis renders slot 0.  cams / camera_of:
// device camera table and [N] camera ids (fp_track_cameras), or null = the context's frame
static int make_crops(fp_ctx* c, const float* poses, int N, int mode, float* dbg, float* win, int* stats,
                      cudaStream_t st, const int* mesh_of = nullptr, const CameraDev* cams = nullptr,
                      const int* camera_of = nullptr, float4* vis = nullptr) {
  FP_REQUIRE(mesh_of || c->mesh[0].loaded, "no mesh: call fp_set_mesh first");
  FP_REQUIRE(c->has_frame, "no frame: call fp_set_frame first");
  // only launches below: this body is also what run_graphed captures (no allocation, no synchronisation)
  CropParams p;
  p.poses = poses;
  p.N = N;
  p.fx = c->K[0];
  p.fy = c->K[4];
  p.cx = c->K[2];
  p.cy = c->K[5];
  p.H = c->H;
  p.W = c->W;
  p.znear = 0.001f;  // Utils.py:161
  p.zfar = 100.f;
  p.slots = reinterpret_cast<const MeshSlotDev*>(c->mesh_table.p);
  p.mesh_of = mesh_of;
  p.rgb = reinterpret_cast<const uchar4*>(c->rgba.p);
  p.xyz_map = reinterpret_cast<const float4*>(c->xyz.p);
  p.depth = c->depth_cur;
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
  return crop_launch(p, st);
}

// The launch sequence a cached graph holds: the first element of its key
enum class GraphKind {
  Refine = 0,            // fp_refine
  ScoreFeatures = 1,     // fp_score_features
  Track = 2,             // fp_track
  TrackObjects = 3,      // fp_track_objects
  RegisterRefine = 4,    // fp_register_objects: one pass's refinement
  RegisterFeatures = 5,  // fp_register_objects: one pass's scorer features
  TrackCameras = 6,      // fp_track_cameras
  RegisterCamerasRefine = 7,    // fp_register_cameras: one pass's refinement, frames from the camera table
  RegisterCamerasFeatures = 8,  // fp_register_cameras: one pass's scorer features, frames from the camera table
};

// Runs `body(stream)` — a fixed sequence of kernel launches (and fixed-address copies) on ctx-owned buffers —
// through a cached CUDA graph: first sight of a key runs eagerly (sets function attributes), the second
// captures + instantiates, later calls replay.  Replay removes ~170 launch + 60 tensor-map-encode host
// calls per register(), which is what bounds track_one() and small per-GPU shards.  The body never allocates:
// callers size every workspace first, so a capture after an epoch bump (new mesh, new N) is safe.
// frame_by_value: the body passes the context's K / H / W to its kernels by value (every body except fp_track_cameras',
// which reads them from the camera table); such a graph is captured again when they differ from its capture's.  Only
// that graph: a frame of another size or other intrinsics does not invalidate the others.
template <class Body>
static int run_graphed(fp_ctx* c, GraphKind kind, int N, int iters, cudaStream_t st, Body body, int cameras = 0,
                       bool frame_by_value = true) {
  if (!c->use_graphs || g_prof_on) return body(st);
  const auto key = std::make_tuple(static_cast<int>(kind), N, iters, cameras);
  auto it = c->graphs.find(key);
  if (it == c->graphs.end()) {
    c->graphs[key] = fp_ctx::GraphEntry();  // seen once: next call captures
    return body(st);
  }
  fp_ctx::GraphEntry& g = it->second;
  const bool frame_moved =
      frame_by_value && (g.H != c->H || g.W != c->W || memcmp(g.K, c->K, sizeof g.K) != 0);
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
    memcpy(g.K, c->K, sizeof g.K);
    g.H = c->H;
    g.W = c->W;
    c->graph_nodes[key] = (int)n_kernels;
    ++c->graph_captures;
  }
  FP_CUDA_OK(cudaGraphLaunch(g.exec, st));
  note_launches(c->graph_nodes[key]);
  return 0;
}

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

// FPOSE_FUSED_PREP=0: the frame filters as four separate launches instead of frame_prep_kernel (A/B)
static bool fused_prep() {
  static const bool fused = [] {
    const char* e = getenv("FPOSE_FUSED_PREP");
    return !(e && e[0] == '0');
  }();
  return fused;
}

static int set_frame_launches(fp_ctx* c, const unsigned char* rgb_dev, const float* depth_dev, int flags, float zfar,
                              cudaStream_t st) {
  const int H = c->H, W = c->W;
  const size_t npix = (size_t)H * W;
  if ((flags & FP_FRAME_FILTER_DEPTH) && !fused_prep()) {
    FP_TRY(rgb_to_rgba_launch(rgb_dev, reinterpret_cast<uchar4*>(c->rgba.p), (int)npix, st));
    FP_TRY(erode_depth_launch(depth_dev, reinterpret_cast<float*>(c->depth_a.p), H, W, 2, 0.001f, 0.8f, 100.f, st));
    FP_TRY(bilateral_depth_launch(reinterpret_cast<const float*>(c->depth_a.p), reinterpret_cast<float*>(c->depth_b.p), H,
                                  W, 2, 100.f, 2.f, 100000.f, st));
    c->depth_cur = reinterpret_cast<const float*>(c->depth_b.p);
    return depth_to_xyz_launch(c->depth_cur, reinterpret_cast<float4*>(c->xyz.p), H, W, c->K[0], c->K[4], c->K[2], c->K[5], zfar, st);
  }
  if (flags & FP_FRAME_FILTER_DEPTH) {
    // estimater.py:173-174 erode_depth(radius=2), bilateral_filter_depth(radius=2); :214 depth2xyzmap: one launch
    c->depth_cur = reinterpret_cast<const float*>(c->depth_b.p);
    return frame_prep_launch(rgb_dev, depth_dev, reinterpret_cast<uchar4*>(c->rgba.p), reinterpret_cast<float*>(c->depth_b.p),
                             reinterpret_cast<float4*>(c->xyz.p), H, W, c->K[0], c->K[4], c->K[2], c->K[5], zfar, st);
  }
  FP_TRY(rgb_to_rgba_launch(rgb_dev, reinterpret_cast<uchar4*>(c->rgba.p), (int)npix, st));
  FP_CUDA_OK(cudaMemcpyAsync(c->depth_b.p, depth_dev, npix * 4, cudaMemcpyDeviceToDevice, st));
  c->depth_cur = reinterpret_cast<const float*>(c->depth_b.p);
  FP_TRY(depth_to_xyz_launch(c->depth_cur, reinterpret_cast<float4*>(c->xyz.p), H, W, c->K[0], c->K[4], c->K[2], c->K[5],
                             zfar, st));
  return 0;
}

static int alloc_frame_buffers(fp_ctx* c, size_t npix, bool need_raw) {
  FP_TRY(dev_alloc(c->epoch, c->rgba, npix * 4));
  FP_TRY(dev_alloc(c->epoch, c->depth_a, npix * 4));
  FP_TRY(dev_alloc(c->epoch, c->depth_b, npix * 4));
  FP_TRY(dev_alloc(c->epoch, c->xyz, npix * 16));
  if (need_raw) {
    FP_TRY(dev_alloc(c->epoch, c->rgb_raw, npix * 3));
    FP_TRY(dev_alloc(c->epoch, c->depth_raw, npix * 4));
  }
  return 0;
}

// records K / H / W as the context's frame geometry
static void set_frame_geometry(fp_ctx* c, const float* K, int H, int W) {
  for (int i = 0; i < 9; ++i) c->K[i] = K[i];
  c->H = H;
  c->W = W;
}

// frame buffers + intrinsics (a graph that holds them by value is captured again when they change, see run_graphed)
static int prepare_frame(fp_ctx* c, const float* K, int H, int W, bool need_raw) {
  FP_TRY(alloc_frame_buffers(c, (size_t)H * W, need_raw));
  set_frame_geometry(c, K, H, W);
  return 0;
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

// pinned host staging of the context's frame (fp_track, fp_track_objects, fp_track_cameras' camera 0,
// fp_register_objects).  No graph holds these addresses: upload_staged_frame copies out of them ahead of the launch.
static int alloc_frame_staging(fp_ctx* c, size_t npix) {
  FP_TRY(pinned_alloc(nullptr, c->stage_rgb, npix * 3));
  return pinned_alloc(nullptr, c->stage_depth, npix * 4);
}

// The previous frame's graph has finished (every caller synchronises), so the staging buffers are free.  The two
// uploads are issued as soon as their staging copy is done — the depth DMA runs under the host's rgb copy, the
// rgb DMA under the next camera's copies or the graph launch — instead of being nodes of the graph (measured: -40 us
// per frame)
static int upload_staged_frame(void* stage_rgb, void* stage_depth, void* rgb_dev, void* depth_dev,
                               const unsigned char* rgb_host, const float* depth_host, size_t npix, cudaStream_t st) {
  memcpy(stage_depth, depth_host, npix * 4);
  FP_CUDA_OK(cudaMemcpyAsync(depth_dev, stage_depth, npix * 4, cudaMemcpyHostToDevice, st));
  memcpy(stage_rgb, rgb_host, npix * 3);
  FP_CUDA_OK(cudaMemcpyAsync(rgb_dev, stage_rgb, npix * 3, cudaMemcpyHostToDevice, st));
  return 0;
}
static int upload_staged_frame(fp_ctx* c, const unsigned char* rgb_host, const float* depth_host, size_t npix,
                               cudaStream_t st) {
  return upload_staged_frame(c->stage_rgb.p, c->stage_depth.p, c->rgb_raw.p, c->depth_raw.p, rgb_host, depth_host, npix, st);
}

// Frame buffers and pinned staging of cameras 1.. of a multi-camera call, at npix_max pixels each (camera 0 is the
// context's frame, sized by the caller).  Only the camera table holds these addresses: no graph is affected.
static int alloc_camera_bufs(fp_ctx* c, int C, size_t npix_max) {
  for (int i = 1; i < C; ++i) {
    CameraBufs& b = c->cams[i];
    unsigned long long table_only = 0;
    FP_TRY(dev_alloc(table_only, b.rgb_raw, npix_max * 3));
    FP_TRY(dev_alloc(table_only, b.depth_raw, npix_max * 4));
    FP_TRY(dev_alloc(table_only, b.rgba, npix_max * 4));
    FP_TRY(dev_alloc(table_only, b.depth, npix_max * 4));
    FP_TRY(dev_alloc(table_only, b.xyz, npix_max * 16));
    FP_TRY(pinned_alloc(nullptr, b.stage_rgb, npix_max * 3));
    FP_TRY(pinned_alloc(nullptr, b.stage_depth, npix_max * 4));
  }
  return 0;
}

// The camera table of C cameras (entries C.. zeroed): buffers, size and intrinsics (K: [C][9]) of every camera
static void fill_camera_table(const fp_ctx* c, int C, const float* K, const int* H, const int* W, CameraDev* table) {
  memset(table, 0, sizeof(CameraDev) * kMaxCameras);
  for (int i = 0; i < C; ++i) {
    CameraDev& e = table[i];
    e.rgb_raw = reinterpret_cast<const unsigned char*>(i ? c->cams[i].rgb_raw.p : c->rgb_raw.p);
    e.depth_raw = reinterpret_cast<const float*>(i ? c->cams[i].depth_raw.p : c->depth_raw.p);
    e.rgb = reinterpret_cast<uchar4*>(i ? c->cams[i].rgba.p : c->rgba.p);
    e.depth = reinterpret_cast<float*>(i ? c->cams[i].depth.p : c->depth_b.p);
    e.xyz_map = reinterpret_cast<float4*>(i ? c->cams[i].xyz.p : c->xyz.p);
    e.fx = K[9 * i + 0];
    e.fy = K[9 * i + 4];
    e.cx = K[9 * i + 2];
    e.cy = K[9 * i + 5];
    e.H = H[i];
    e.W = W[i];
  }
}

// Every camera's frame through its own pinned staging; camera i's DMA runs while camera i + 1 is copied on the host
static int upload_camera_frames(fp_ctx* c, int C, const unsigned char* const* rgb_host, const float* const* depth_host,
                                const int* H, const int* W, cudaStream_t st) {
  for (int i = 0; i < C; ++i) {
    const size_t npix = (size_t)H[i] * W[i];
    if (i == 0) {
      FP_TRY(upload_staged_frame(c, rgb_host[0], depth_host[0], npix, st));
    } else {
      CameraBufs& b = c->cams[i];
      FP_TRY(upload_staged_frame(b.stage_rgb.p, b.stage_depth.p, b.rgb_raw.p, b.depth_raw.p, rgb_host[i], depth_host[i], npix, st));
    }
  }
  return 0;
}

// fp_track_cameras and fp_track_objects after validation.  Camera 0 is the context's frame (buffers, staging, K / H / W),
// cameras 1.. have buffers of their own.
//   by_value = false (fp_track_cameras): every camera's buffers are sized for the largest frame of the call, so a
//     permutation of the same cameras reallocates nothing.  The camera table, the slot ids and the camera ids go to one
//     fixed device block in one copy ahead of the launch: the graph holds that block's address, not the frames' sizes,
//     intrinsics or buffers, and is keyed on (C, M, iterations).  One frame_prep_kernel launch filters every camera
//     (FPOSE_FUSED_PREP=0 does not apply) and the crops take their frame from the table.
//   by_value = true (fp_track_objects, C = 1): the context's frame as fp_track sees it; the frame filters and the crop
//     producer take it by value (the single-camera kernel instantiations), so the graph is captured again when the
//     frame's size or intrinsics change.  Only the slot ids are copied.
static int track_cameras_body(fp_ctx* c, int C, const unsigned char* const* rgb_host, const float* const* depth_host,
                              const float* K, const int* H, const int* W, int M, const int* camera_of, const int* slots_host,
                              const float* poses_in_dev, int iterations, float* poses_out_dev, float* poses_out_host,
                              cudaStream_t st, bool by_value) {
  size_t npix_max = 0;
  int H_max = 0, W_max = 0;
  for (int i = 0; i < C; ++i) {
    npix_max = std::max(npix_max, (size_t)H[i] * W[i]);
    H_max = std::max(H_max, H[i]);
    W_max = std::max(W_max, W[i]);
  }
  FP_TRY(ensure_capacity(c, M));
  FP_TRY(alloc_frame_buffers(c, npix_max, true));
  FP_TRY(alloc_frame_staging(c, npix_max));
  set_frame_geometry(c, K, H[0], W[0]);
  if (!by_value && (H_max > c->cam_grid_h || W_max > c->cam_grid_w)) {
    // the frame-preparation grid is a by-value launch parameter: it covers the largest frame seen, the blocks outside
    // a smaller frame return at once
    ++c->epoch;
    c->cam_grid_h = std::max(c->cam_grid_h, H_max);
    c->cam_grid_w = std::max(c->cam_grid_w, W_max);
  }
  FP_TRY(alloc_camera_bufs(c, C, npix_max));
  const size_t table_bytes = sizeof(CameraDev) * kMaxCameras;
  const size_t args_bytes = table_bytes + (size_t)2 * M * sizeof(int);
  FP_TRY(dev_alloc(c->epoch, c->cam_args, args_bytes));
  FP_TRY(pinned_alloc(nullptr, c->stage_args, args_bytes));
  FP_TRY(pinned_alloc(&c->epoch, c->stage_poses, (size_t)M * 64));  // the graph's read-back node holds this address
  // the per-call arguments: one staged block, one copy
  int* ints = reinterpret_cast<int*>(reinterpret_cast<char*>(c->stage_args.p) + table_bytes);
  memcpy(ints, slots_host, (size_t)M * sizeof(int));
  if (by_value) {
    FP_CUDA_OK(cudaMemcpyAsync(reinterpret_cast<char*>(c->cam_args.p) + table_bytes, ints, (size_t)M * sizeof(int),
                               cudaMemcpyHostToDevice, st));
  } else {
    fill_camera_table(c, C, K, H, W, reinterpret_cast<CameraDev*>(c->stage_args.p));
    memcpy(ints + M, camera_of, (size_t)M * sizeof(int));
    FP_CUDA_OK(cudaMemcpyAsync(c->cam_args.p, c->stage_args.p, args_bytes, cudaMemcpyHostToDevice, st));
  }
  const CameraDev* cams_dev = by_value ? nullptr : reinterpret_cast<const CameraDev*>(c->cam_args.p);
  const int* mesh_of = reinterpret_cast<const int*>(reinterpret_cast<const char*>(c->cam_args.p) + table_bytes);
  const int* cam_of = by_value ? nullptr : mesh_of + M;
  float* pa = reinterpret_cast<float*>(c->poses_a.p);
  float* pb = reinterpret_cast<float*>(c->poses_b.p);
  FP_CUDA_OK(cudaMemcpyAsync(pa, poses_in_dev, (size_t)M * 64, cudaMemcpyDeviceToDevice, st));
  FP_TRY(upload_camera_frames(c, C, rgb_host, depth_host, H, W, st));
  c->has_frame = false;
  const float* fin = (iterations % 2 == 0) ? pa : pb;
  const int grid_h = c->cam_grid_h, grid_w = c->cam_grid_w;
  auto body = [&](cudaStream_t s2) -> int {
    // estimater.py:250-268 for every object of every camera at once: each camera's frame filtered once, M hypotheses
    // each rendering its own mesh and cropping its own camera's frame
    if (by_value) {
      FP_TRY(set_frame_launches(c, reinterpret_cast<const unsigned char*>(c->rgb_raw.p),
                                reinterpret_cast<const float*>(c->depth_raw.p), FP_FRAME_FILTER_DEPTH, INFINITY, s2));
    } else {
      c->depth_cur = reinterpret_cast<const float*>(c->depth_b.p);
      FP_TRY(frame_prep_cameras_launch(cams_dev, C, grid_h, grid_w, INFINITY, s2));
    }
    c->has_frame = true;
    FP_TRY(refine_body(c, M, iterations, s2, mesh_of, cams_dev, cam_of));
    FP_CUDA_OK(cudaMemcpyAsync(c->stage_poses.p, fin, (size_t)M * 64, cudaMemcpyDeviceToHost, s2));
    return 0;
  };
  if (by_value) {
    FP_TRY(run_graphed(c, GraphKind::TrackObjects, M, iterations, st, body));
  } else {
    FP_TRY(run_graphed(c, GraphKind::TrackCameras, M, iterations, st, body, C, /*frame_by_value=*/false));
  }
  c->has_frame = true;
  if (poses_out_dev) FP_CUDA_OK(cudaMemcpyAsync(poses_out_dev, fin, (size_t)M * 64, cudaMemcpyDeviceToDevice, st));
  FP_CUDA_OK(cudaStreamSynchronize(st));
  if (poses_out_host) memcpy(poses_out_host, c->stage_poses.p, (size_t)M * 64);
  return 0;
}

// The mesh slot of each of `M` objects.  The kernels index the mesh table with these ids unchecked, so an empty or
// out-of-range slot must be refused before anything is enqueued.
static int check_slots(const fp_ctx* c, int M, const int* slots, const char* caller) {
  for (int i = 0; i < M; ++i) {
    FP_REQUIRE(slots[i] >= 0 && slots[i] < kMaxMeshes, "%s: object %d: slot %d out of range [0, %d)", caller, i, slots[i],
               kMaxMeshes);
    FP_REQUIRE(c->mesh[slots[i]].loaded, "%s: object %d: slot %d holds no mesh", caller, i, slots[i]);
  }
  return 0;
}

// The frames of C cameras and the camera of each of M objects: non-null frames of positive size, every camera id in
// [0, C) and every camera owning at least one object.  The kernels index the camera table with these ids unchecked.
static int check_cameras(int C, const unsigned char* const* rgb_host, const float* const* depth_host, const int* H, const int* W,
                         int M, const int* camera_of, const char* caller) {
  FP_REQUIRE(C >= 1 && C <= kMaxCameras, "%s: %d cameras, need 1..%d", caller, C, kMaxCameras);
  for (int i = 0; i < C; ++i) {
    FP_REQUIRE(rgb_host[i] && depth_host[i], "%s: camera %d: null frame", caller, i);
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

// The scorer tail over `L` feature rows as one segment; a segmented launch sets seg / n_seg / seg_max on top.
static ScoreTailParams score_tail_params(const fp_ctx* c, const float* feats, int L, float* scores, int* best) {
  const Net& net = c->net[1];
  ScoreTailParams p;
  p.feats = feats;
  p.L = L;
  p.w_in = net.f("cross.in_w");
  p.b_in = net.f("cross.in_b");
  p.fold_v = reinterpret_cast<const float*>(c->fold_v.p);
  p.fold_c = c->fold_c;
  p.offset = 100.f;
  p.qkv = reinterpret_cast<float*>(c->tail_qkv.p);
  p.scores = scores;
  p.best = best;
  p.counter = reinterpret_cast<unsigned int*>(c->tail_counter.p);
  return p;
}

// fp_register_cameras and fp_register_objects after validation (n_hyp_host is checked here, before anything is
// enqueued).  Object i is seen by camera camera_of[i]; its mask is masks_host[i], of its camera's size.  Camera 0 is the
// context's frame, cameras 1.. have buffers of their own (as track_cameras_body).
//   by_value = false (fp_register_cameras): every camera's buffers are sized for the largest frame of the call.  One
//     frame_prep_kernel launch filters every camera and the start-pose kernels read each object's depth, size and
//     intrinsics from the camera table.  Each pass copies its slot ids and per-hypothesis camera ids into fixed context
//     buffers and the crops take their frame from the table at its fixed address, so the refine / feature graphs hold
//     no frame and are keyed on (kind, pass size, iterations) alone: reordering cameras or objects or changing
//     intrinsics replays them.
//   by_value = true (fp_register_objects, C = 1): the frame filters, the start-pose kernels and the crop producer take
//     the context's frame by value (the single-camera kernel instantiations), as fp_register does.
// Both: whole objects in the given order in passes of up to kRegisterPassCap hypotheses (an object above the cap alone),
// then one segmented scorer tail over all objects.  Synchronises.
static int register_cameras_body(fp_ctx* c, int C, const unsigned char* const* rgb_host, const float* const* depth_host,
                                 const float* K, const int* H, const int* W, int M, const int* camera_of, const int* slots_host,
                                 const int* n_hyp_host, const unsigned char* const* masks_host, const float* rot_grids_dev,
                                 int iterations, float* poses_out_dev, float* scores_out_dev, int* best_out_dev,
                                 float* info_out_dev, cudaStream_t st, bool by_value) {
  const char* caller = by_value ? "fp_register_objects" : "fp_register_cameras";
  std::vector<int> off(M + 1, 0);
  int seg_max = 0;
  for (int i = 0; i < M; ++i) {
    FP_REQUIRE(n_hyp_host[i] >= 1 && n_hyp_host[i] <= 4096, "%s: object %d: %d hypotheses, need 1..4096", caller, i,
               n_hyp_host[i]);
    off[i + 1] = off[i] + n_hyp_host[i];
    seg_max = std::max(seg_max, n_hyp_host[i]);
  }
  const int total = off[M];
  // passes: whole objects in the given order, up to kRegisterPassCap hypotheses; an object above the cap alone
  std::vector<int> pass_obj(1, 0);  // first object of every pass, then M
  for (int i = 1; i < M; ++i)
    if (off[i + 1] - off[pass_obj.back()] > kRegisterPassCap) pass_obj.push_back(i);
  pass_obj.push_back(M);
  int max_pass = 0;
  for (size_t p = 0; p + 1 < pass_obj.size(); ++p) max_pass = std::max(max_pass, off[pass_obj[p + 1]] - off[pass_obj[p]]);
  // each object's mask at its byte offset of one block
  size_t npix_max = 0;
  int H_max = 0, W_max = 0;
  for (int i = 0; i < C; ++i) {
    npix_max = std::max(npix_max, (size_t)H[i] * W[i]);
    H_max = std::max(H_max, H[i]);
    W_max = std::max(W_max, W[i]);
  }
  std::vector<size_t> mask_at(M + 1, 0);
  for (int i = 0; i < M; ++i) mask_at[i + 1] = mask_at[i] + (size_t)H[camera_of[i]] * W[camera_of[i]];
  const size_t mask_bytes = mask_at[M];
  // every workspace is sized for the largest pass here, so no pass bumps the graph epoch
  FP_TRY(ensure_capacity(c, max_pass));
  FP_TRY(ensure_tail(c, total));
  FP_TRY(alloc_frame_buffers(c, npix_max, true));
  set_frame_geometry(c, K, H[0], W[0]);
  FP_TRY(alloc_frame_staging(c, npix_max));
  FP_TRY(alloc_camera_bufs(c, C, npix_max));
  FP_TRY(dev_alloc(c->epoch, c->mesh_of, (size_t)max_pass * sizeof(int)));
  FP_TRY(dev_alloc(c->epoch, c->seg_off, (size_t)(2 * M + 1) * sizeof(int)));  // offsets [M + 1], camera ids [M]
  FP_TRY(dev_alloc(c->epoch, c->reg_feats, (size_t)total * 512 * sizeof(float)));
  FP_TRY(dev_alloc(c->epoch, c->mask_buf, mask_bytes));
  FP_TRY(dev_alloc(c->epoch, c->mask_stats, (size_t)M * 6 * sizeof(unsigned int)));
  FP_TRY(dev_alloc(c->epoch, c->tail_counter, std::max<size_t>(16, (size_t)M * sizeof(unsigned int)), /*zero=*/true));
  const size_t table_bytes = sizeof(CameraDev) * kMaxCameras;
  if (!by_value) {
    FP_TRY(dev_alloc(c->epoch, c->reg_cams, table_bytes));
    FP_TRY(dev_alloc(c->epoch, c->reg_cam_of, (size_t)max_pass * sizeof(int)));
    FP_TRY(dev_alloc(c->epoch, c->mask_off, (size_t)M * sizeof(size_t)));
    FP_TRY(pinned_alloc(nullptr, c->stage_cams, table_bytes + (size_t)M * sizeof(size_t)));
  }
  // pinned staging (never read by a captured graph): the copies below leave as soon as they are enqueued
  FP_TRY(pinned_alloc(nullptr, c->stage_masks, mask_bytes));
  FP_TRY(pinned_alloc(nullptr, c->stage_ints, (size_t)(2 * M + 1 + 2 * total) * sizeof(int)));
  // offsets [M + 1], camera of every object [M], slot of every hypothesis [total], camera of every hypothesis [total]
  int* ints = reinterpret_cast<int*>(c->stage_ints.p);
  int* slot_of = ints + 2 * M + 1;
  int* cam_of = slot_of + total;
  memcpy(ints, off.data(), (size_t)(M + 1) * sizeof(int));
  memcpy(ints + M + 1, camera_of, (size_t)M * sizeof(int));
  for (int i = 0; i < M; ++i) {
    std::fill(slot_of + off[i], slot_of + off[i + 1], slots_host[i]);
    std::fill(cam_of + off[i], cam_of + off[i + 1], camera_of[i]);
    memcpy(reinterpret_cast<unsigned char*>(c->stage_masks.p) + mask_at[i], masks_host[i], mask_at[i + 1] - mask_at[i]);
  }
  FP_CUDA_OK(cudaMemcpyAsync(c->seg_off.p, ints, (size_t)(2 * M + 1) * sizeof(int), cudaMemcpyHostToDevice, st));
  FP_CUDA_OK(cudaMemcpyAsync(c->mask_buf.p, c->stage_masks.p, mask_bytes, cudaMemcpyHostToDevice, st));
  const CameraDev* cams_dev = by_value ? nullptr : reinterpret_cast<const CameraDev*>(c->reg_cams.p);
  if (!by_value) {
    char* stage = reinterpret_cast<char*>(c->stage_cams.p);
    fill_camera_table(c, C, K, H, W, reinterpret_cast<CameraDev*>(stage));
    memcpy(stage + table_bytes, mask_at.data(), (size_t)M * sizeof(size_t));
    FP_CUDA_OK(cudaMemcpyAsync(c->reg_cams.p, stage, table_bytes, cudaMemcpyHostToDevice, st));
    FP_CUDA_OK(cudaMemcpyAsync(c->mask_off.p, stage + table_bytes, (size_t)M * sizeof(size_t), cudaMemcpyHostToDevice, st));
  }
  FP_TRY(upload_camera_frames(c, C, rgb_host, depth_host, H, W, st));
  // estimater.py:173-174, :214 once per camera for every object: erode + bilateral, depth2xyzmap(zfar = inf)
  c->has_frame = false;
  if (by_value) {
    FP_TRY(set_frame_launches(c, reinterpret_cast<const unsigned char*>(c->rgb_raw.p),
                              reinterpret_cast<const float*>(c->depth_raw.p), FP_FRAME_FILTER_DEPTH, INFINITY, st));
  } else {
    c->depth_cur = reinterpret_cast<const float*>(c->depth_b.p);
    FP_TRY(frame_prep_cameras_launch(cams_dev, C, H_max, W_max, INFINITY, st));
  }
  c->has_frame = true;
  // estimater.py:137-156, :203-209 for every object in one launch pair; the start poses go to poses_out_dev and are
  // replaced pass by pass with the refined ones
  const int* seg = reinterpret_cast<const int*>(c->seg_off.p);
  const unsigned char* masks_dev = reinterpret_cast<const unsigned char*>(c->mask_buf.p);
  unsigned int* stats = reinterpret_cast<unsigned int*>(c->mask_stats.p);
  if (by_value) {
    FP_TRY(start_poses_launch(c->depth_cur, masks_dev, H[0], W[0], c->K[0], c->K[4], c->K[2], c->K[5], rot_grids_dev, total, M,
                              seg, stats, poses_out_dev, info_out_dev, st));
  } else {
    FP_TRY(start_poses_cameras_launch(cams_dev, seg + M + 1, masks_dev, reinterpret_cast<const size_t*>(c->mask_off.p),
                                      rot_grids_dev, M, seg, stats, poses_out_dev, info_out_dev, st));
  }
  float* pa = reinterpret_cast<float*>(c->poses_a.p);
  float* pb = reinterpret_cast<float*>(c->poses_b.p);
  float* ps = reinterpret_cast<float*>(c->pose_stage.p);
  float* fb = reinterpret_cast<float*>(c->feat_buf.p);
  const int* mesh_of = reinterpret_cast<const int*>(c->mesh_of.p);
  const int* hyp_cam = by_value ? nullptr : reinterpret_cast<const int*>(c->reg_cam_of.p);
  const float* fin = (iterations % 2 == 0) ? pa : pb;
  const GraphKind refine_kind = by_value ? GraphKind::RegisterRefine : GraphKind::RegisterCamerasRefine;
  const GraphKind feature_kind = by_value ? GraphKind::RegisterFeatures : GraphKind::RegisterCamerasFeatures;
  for (size_t p = 0; p + 1 < pass_obj.size(); ++p) {
    const int row0 = off[pass_obj[p]], n = off[pass_obj[p + 1]] - row0;
    // the pass's slot ids, camera ids and start poses go to fixed context buffers and its outputs are copied out after
    // the replays: the graphs hold no per-pass address and are keyed on (kind, n, iterations) alone
    FP_CUDA_OK(cudaMemcpyAsync(c->mesh_of.p, slot_of + row0, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
    if (!by_value)
      FP_CUDA_OK(cudaMemcpyAsync(c->reg_cam_of.p, cam_of + row0, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
    FP_CUDA_OK(cudaMemcpyAsync(pa, poses_out_dev + (size_t)row0 * 16, (size_t)n * 64, cudaMemcpyDeviceToDevice, st));
    FP_TRY(run_graphed(
        c, refine_kind, n, iterations, st,
        [&](cudaStream_t s2) -> int { return refine_body(c, n, iterations, s2, mesh_of, cams_dev, hyp_cam); }, 0, by_value));
    FP_CUDA_OK(cudaMemcpyAsync(poses_out_dev + (size_t)row0 * 16, fin, (size_t)n * 64, cudaMemcpyDeviceToDevice, st));
    FP_CUDA_OK(cudaMemcpyAsync(ps, fin, (size_t)n * 64, cudaMemcpyDeviceToDevice, st));
    FP_TRY(run_graphed(
        c, feature_kind, n, 0, st,
        [&](cudaStream_t s2) -> int {
          FP_TRY(make_crops(c, ps, n, 1, nullptr, nullptr, nullptr, s2, mesh_of, cams_dev, hyp_cam));
          FP_TRY(run_encoder(c, c->net[1], reinterpret_cast<const __half*>(c->crops.p), n, s2));
          return run_score_feats(c, c->net[1], n, fb, s2);
        },
        0, by_value));
    FP_CUDA_OK(cudaMemcpyAsync(reinterpret_cast<float*>(c->reg_feats.p) + (size_t)row0 * 512, fb, (size_t)n * 2048,
                               cudaMemcpyDeviceToDevice, st));
  }
  // score_network.py:84-88 per object: one tail launch, each object's hypotheses attending only to each other
  ScoreTailParams tp = score_tail_params(c, reinterpret_cast<const float*>(c->reg_feats.p), total, scores_out_dev, best_out_dev);
  tp.seg = seg;
  tp.n_seg = M;
  tp.seg_max = seg_max;
  FP_TRY(score_tail_launch(tp, st));
  FP_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace fp

using namespace fp;

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
  cudaDeviceSynchronize();
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

int fp_load_network(fp_ctx* c, int which, const fp_tensor_t* tensors, int n) {
  FP_API_BEGIN
  FP_REQUIRE(c && tensors, "fp_load_network: null argument");
  FP_REQUIRE(which == 0 || which == 1, "fp_load_network: which must be 0 (refiner) or 1 (scorer)");
  DeviceGuard dg(c->device);
  Net& net = c->net[which];
  ++c->epoch;
  FP_CUDA_OK(cudaDeviceSynchronize());
  net.t.clear();
  net.loaded = false;
  for (int i = 0; i < n; ++i) {
    const fp_tensor_t& t = tensors[i];
    FP_REQUIRE(t.name && t.data && t.numel > 0, "fp_load_network: bad tensor #%d", i);
    Tensor d;
    d.dtype = t.dtype;
    d.numel = t.numel;
    const size_t bytes = (size_t)t.numel * (t.dtype == 1 ? 2 : 4);
    FP_TRY(dev_alloc(c->epoch, d.buf, bytes));
    FP_CUDA_OK(cudaMemcpy(d.buf.p, t.data, bytes, cudaMemcpyHostToDevice));
    net.t[t.name] = std::move(d);  // a repeated name frees the earlier tensor
  }
  // verify that everything the execution plan needs is present, with the right size
  std::vector<std::pair<std::string, long long>> need;
  const int cin[15] = {0, 64, 128, 128, 128, 128, 256, 256, 256, 256, 256, 512, 512, 512, 512};
  const int cout[15] = {64, 128, 128, 128, 128, 128, 256, 256, 256, 256, 512, 512, 512, 512, 512};
  for (int i = 0; i < 15; ++i) {
    const long long k = i == 0 ? 7 * 64 : 9LL * cin[i];
    need.push_back({"enc." + std::to_string(i) + ".w", k * cout[i]});
    need.push_back({"enc." + std::to_string(i) + ".b", cout[i]});
  }
  need.push_back({"pe", 400LL * 512});
  if (which == 0) {
    need.push_back({"heads.in_w", 3072LL * 512});
    need.push_back({"heads.in_b", 3072});
    for (int g = 0; g < 2; ++g) {
      const std::string h = "head" + std::to_string(g) + ".";
      for (const char* s : {"out_w", "ff1_w", "ff2_w"}) need.push_back({h + s, 512LL * 512});
      for (const char* s : {"out_b", "ff1_b", "ff2_b", "ln1_g", "ln1_b", "ln2_g", "ln2_b"}) need.push_back({h + s, 512});
      need.push_back({h + "fin_w", 3LL * 512});
      need.push_back({h + "fin_b", 3});
    }
  } else {
    need.push_back({"att.in_w", 1536LL * 512});
    need.push_back({"att.in_b", 1536});
    need.push_back({"att.out_w32", 512LL * 512});
    need.push_back({"att.out_b", 512});
    need.push_back({"cross.in_w", 1536LL * 512});
    need.push_back({"cross.in_b", 1536});
    need.push_back({"cross.out_w", 512LL * 512});
    need.push_back({"cross.out_b", 512});
    need.push_back({"lin.w", 512});
    need.push_back({"lin.b", 1});
  }
  for (auto& nd : need) {
    auto it = net.t.find(nd.first);
    FP_REQUIRE(it != net.t.end(), "fp_load_network: tensor '%s' missing", nd.first.c_str());
    FP_REQUIRE(it->second.numel == nd.second, "fp_load_network: tensor '%s' has %lld elements, expected %lld",
               nd.first.c_str(), it->second.numel, nd.second);
  }
  if (which == 1) {
    // score = linear(out_proj(a)) = (W_out^T w_lin) . a + (w_lin . b_out + b_lin): fold once, in fp64
    const float *wo = nullptr, *bo = nullptr, *wl = nullptr, *bl = nullptr;
    for (int i = 0; i < n; ++i) {
      const std::string nm = tensors[i].name;
      const float* d = reinterpret_cast<const float*>(tensors[i].data);
      if (tensors[i].dtype != 0) continue;
      if (nm == "cross.out_w") wo = d;
      else if (nm == "cross.out_b") bo = d;
      else if (nm == "lin.w") wl = d;
      else if (nm == "lin.b") bl = d;
    }
    FP_REQUIRE(wo && bo && wl && bl, "fp_load_network: the scorer tail tensors must be float32");
    std::vector<float> v(512);
    for (int i = 0; i < 512; ++i) {
      double acc = 0.0;
      for (int o = 0; o < 512; ++o) acc += (double)wl[o] * (double)wo[(size_t)o * 512 + i];
      v[i] = (float)acc;
    }
    double cc = (double)bl[0];
    for (int o = 0; o < 512; ++o) cc += (double)wl[o] * (double)bo[o];
    c->fold_c = (float)cc;
    FP_TRY(upload(c->epoch, c->fold_v, v));
    FP_TRY(dev_alloc(c->epoch, c->tail_counter, 16, /*zero=*/true));
  }
  net.loaded = true;
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
  FP_TRY(upload(c->epoch, m.vpos, mh.vpos));
  FP_TRY(upload(c->epoch, m.vnrm, mh.vnrm));
  FP_TRY(upload(c->epoch, m.vatt, mh.vatt));
  FP_TRY(upload(c->epoch, m.faces, mh.faces));
  FP_TRY(upload(c->epoch, m.meshlets, mh.meshlets));
  FP_TRY(upload(c->epoch, m.ml_verts, mh.ml_verts));
  FP_TRY(upload(c->epoch, m.ml_tris, mh.ml_tris));
  m.has_tex = has_tex;
  if (has_tex) {
    std::vector<unsigned char> rgba((size_t)Ht * Wt * 4);
    for (size_t i = 0; i < (size_t)Ht * Wt; ++i) {
      rgba[4 * i] = tex_rgb[3 * i];
      rgba[4 * i + 1] = tex_rgb[3 * i + 1];
      rgba[4 * i + 2] = tex_rgb[3 * i + 2];
      rgba[4 * i + 3] = 255;
    }
    FP_TRY(upload(c->epoch, m.tex, rgba));
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
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t npix = (size_t)H * W;
  c->has_frame = false;
  const bool on_dev = (flags & FP_FRAME_ON_DEVICE) != 0;
  FP_TRY(prepare_frame(c, K, H, W, !on_dev));
  const unsigned char* rgb_dev = rgb;
  const float* depth_dev = depth;
  if (!on_dev) {
    FP_CUDA_OK(cudaMemcpyAsync(c->rgb_raw.p, rgb, npix * 3, cudaMemcpyHostToDevice, st));
    FP_CUDA_OK(cudaMemcpyAsync(c->depth_raw.p, depth, npix * 4, cudaMemcpyHostToDevice, st));
    rgb_dev = reinterpret_cast<const unsigned char*>(c->rgb_raw.p);
    depth_dev = reinterpret_cast<const float*>(c->depth_raw.p);
  }
  FP_TRY(set_frame_launches(c, rgb_dev, depth_dev, flags, zfar, st));
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
  // [H][W][3] (host or device) -> the float4-per-pixel layout the crop kernel samples
  FP_CUDA_OK(cudaMemcpy2DAsync(c->xyz.p, 16, xyz, 12, 12, (size_t)c->H * c->W, cudaMemcpyDefault, st));
  return 0;
  FP_API_END
}

int fp_get_depth(fp_ctx* c, float* depth_out_dev, float* xyz_out_dev, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && c->has_frame, "fp_get_depth: no frame");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t npix = (size_t)c->H * c->W;
  if (depth_out_dev) FP_CUDA_OK(cudaMemcpyAsync(depth_out_dev, c->depth_cur, npix * 4, cudaMemcpyDeviceToDevice, st));
  // internal layout is float4 per pixel; the hook returns the reference's [H][W][3]
  if (xyz_out_dev)
    FP_CUDA_OK(cudaMemcpy2DAsync(xyz_out_dev, 12, c->xyz.p, 16, 12, npix, cudaMemcpyDeviceToDevice, st));
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
  const size_t npix = (size_t)c->H * c->W;
  const unsigned char* mdev = mask;
  if (!mask_on_device) {
    FP_TRY(dev_alloc(c->epoch, c->mask_buf, npix));
    FP_CUDA_OK(cudaMemcpyAsync(c->mask_buf.p, mask, npix, cudaMemcpyHostToDevice, st));
    mdev = reinterpret_cast<const unsigned char*>(c->mask_buf.p);
  }
  FP_TRY(dev_alloc(c->epoch, c->mask_stats, 64));
  return start_poses_launch(c->depth_cur, mdev, c->H, c->W, c->K[0], c->K[4], c->K[2], c->K[5], rot_grid, N, 1, nullptr,
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
  FP_TRY(ensure_capacity(c, N));
  FP_TRY(dev_alloc(c->epoch, c->crop_stats, 16));
  FP_CUDA_OK(cudaMemsetAsync(c->crop_stats.p, 0, 16, st));
  FP_TRY(make_crops(c, poses, N, mode, nullptr, nullptr, reinterpret_cast<int*>(c->crop_stats.p), st));
  FP_CUDA_OK(cudaMemcpyAsync(stats_out_host, c->crop_stats.p, 16, cudaMemcpyDeviceToHost, st));
  FP_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
  FP_API_END
}

int fp_op_refine_net(fp_ctx* c, const void* crops, int N, float* trans_out, float* rot_out, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && crops && trans_out && rot_out, "fp_op_refine_net: null argument");
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
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
  if (N == 0) return 0;
  FP_TRY(ensure_capacity(c, N));
  FP_TRY(crops_import(c, crops, N, st));
  FP_TRY(run_encoder(c, c->net[1], reinterpret_cast<const __half*>(c->crops.p), N, st));
  FP_TRY(run_score_feats(c, c->net[1], N, feats_out, st));
  return 0;
  FP_API_END
}

int fp_op_tokens(fp_ctx* c, int which, const void* crops, int N, void* tokens_out, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && crops && tokens_out && (which == 0 || which == 1), "fp_op_tokens: bad argument");
  FP_REQUIRE(c->net[which].loaded, "weights not loaded");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (N == 0) return 0;
  FP_TRY(ensure_capacity(c, N));
  FP_TRY(crops_import(c, crops, N, st));
  FP_TRY(run_encoder(c, c->net[which], reinterpret_cast<const __half*>(c->crops.p), N, st));
  FP_CUDA_OK(cudaMemcpyAsync(tokens_out, c->tok.p, (size_t)N * T * 512 * 2, cudaMemcpyDeviceToDevice, st));
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
  FP_TRY(ensure_capacity(c, N));
  FP_TRY(ensure_tail(c, N));
  // poses_b is the loop's ping-pong partner; stage the input in `feats`' neighbour: use tail_proj as scratch
  float* pin = reinterpret_cast<float*>(c->tail_proj.p);  // >= N*512 floats
  float* pout = pin + (size_t)N * 16;
  FP_CUDA_OK(cudaMemcpyAsync(pin, poses_host, (size_t)N * 64, cudaMemcpyHostToDevice, st));
  FP_TRY(fp_refine(c, pin, N, iterations, pout, nullptr, nullptr, stream));
  // keep the refined poses out of the tail's scratch: copy to poses_b's idle half (poses_a/b are free now)
  float* refined = reinterpret_cast<float*>(c->poses_b.p);
  FP_CUDA_OK(cudaMemcpyAsync(refined, pout, (size_t)N * 64, cudaMemcpyDeviceToDevice, st));
  FP_TRY(fp_score(c, refined, N, reinterpret_cast<float*>(c->scores.p), reinterpret_cast<int*>(c->best.p), stream));
  FP_CUDA_OK(cudaMemcpyAsync(poses_out_host, refined, (size_t)N * 64, cudaMemcpyDeviceToHost, st));
  FP_CUDA_OK(cudaMemcpyAsync(scores_out_host, c->scores.p, (size_t)N * 4, cudaMemcpyDeviceToHost, st));
  FP_CUDA_OK(cudaMemcpyAsync(best_out_host, c->best.p, 4, cudaMemcpyDeviceToHost, st));
  FP_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
  FP_API_END
}

int fp_track(fp_ctx* c, const unsigned char* rgb_host, const float* depth_host, const float* K, int H, int W,
             const float* pose_in_dev, int iterations, float* pose_out_dev, float* pose_out_host, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && rgb_host && depth_host && K && H > 0 && W > 0 && iterations >= 0, "fp_track: bad argument");
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  FP_REQUIRE(c->mesh[0].loaded, "fp_track: no mesh");
  DeviceGuard dg(c->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_TRY(ensure_capacity(c, 1));
  FP_TRY(prepare_frame(c, K, H, W, true));
  FP_TRY(dev_alloc(c->epoch, c->track_pose, 64));
  FP_TRY(alloc_frame_staging(c, (size_t)H * W));
  FP_TRY(pinned_alloc(&c->epoch, c->stage_pose, 64));  // the graph's read-back node holds this address
  if (pose_in_dev) {
    FP_CUDA_OK(cudaMemcpyAsync(c->track_pose.p, pose_in_dev, 64, cudaMemcpyDeviceToDevice, st));
  } else {
    FP_REQUIRE(c->track_valid, "fp_track: no previous pose in this context: pass pose_in");
  }
  FP_TRY(upload_staged_frame(c, rgb_host, depth_host, (size_t)H * W, st));
  c->has_frame = false;
  float* pa = reinterpret_cast<float*>(c->poses_a.p);
  float* pb = reinterpret_cast<float*>(c->poses_b.p);
  auto body = [&](cudaStream_t s2) -> int {
    // estimater.py:250-268 in one launch sequence: erode + bilateral, depth2xyzmap_batch(zfar=inf), K refiner passes
    FP_TRY(set_frame_launches(c, reinterpret_cast<const unsigned char*>(c->rgb_raw.p),
                              reinterpret_cast<const float*>(c->depth_raw.p), FP_FRAME_FILTER_DEPTH, INFINITY, s2));
    FP_CUDA_OK(cudaMemcpyAsync(pa, c->track_pose.p, 64, cudaMemcpyDeviceToDevice, s2));
    c->has_frame = true;
    FP_TRY(refine_body(c, 1, iterations, s2));
    const float* fin = (iterations % 2 == 0) ? pa : pb;
    FP_CUDA_OK(cudaMemcpyAsync(c->track_pose.p, fin, 64, cudaMemcpyDeviceToDevice, s2));
    FP_CUDA_OK(cudaMemcpyAsync(c->stage_pose.p, fin, 64, cudaMemcpyDeviceToHost, s2));
    return 0;
  };
  FP_TRY(run_graphed(c, GraphKind::Track, 1, iterations, st, body));
  c->has_frame = true;
  c->track_valid = true;
  if (pose_out_dev) FP_CUDA_OK(cudaMemcpyAsync(pose_out_dev, c->track_pose.p, 64, cudaMemcpyDeviceToDevice, st));
  FP_CUDA_OK(cudaStreamSynchronize(st));
  if (pose_out_host) memcpy(pose_out_host, c->stage_pose.p, 64);
  return 0;
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
  int hw[2];
  FP_TRY(vis_canvas_size(kind, N, hw, hw + 1));
  if (hw_out) {
    hw_out[0] = hw[0];
    hw_out[1] = hw[1];
  }
  FP_TRY(ensure_capacity(c, N));
  // no captured graph holds the vis buffers (fp_vis runs eagerly): growing them must not invalidate the cached graphs
  unsigned long long no_graph = 0;
  FP_TRY(dev_alloc(no_graph, c->vis_rec, (size_t)N * 2 * S * S * sizeof(float4)));
  FP_TRY(dev_alloc(no_graph, c->vis_range, (size_t)N * sizeof(float2)));
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

int fp_track_objects(fp_ctx* c, const unsigned char* rgb_host, const float* depth_host, const float* K, int H, int W, int M,
                     const int* slots_host, const float* poses_in_dev, int iterations, float* poses_out_dev,
                     float* poses_out_host, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && rgb_host && depth_host && K && H > 0 && W > 0 && M > 0 && slots_host && poses_in_dev && iterations >= 0,
             "fp_track_objects: bad argument");
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  FP_TRY(check_slots(c, M, slots_host, "fp_track_objects"));
  DeviceGuard dg(c->device);
  const std::vector<int> camera_of(M, 0);
  return track_cameras_body(c, 1, &rgb_host, &depth_host, K, &H, &W, M, camera_of.data(), slots_host, poses_in_dev, iterations,
                            poses_out_dev, poses_out_host, reinterpret_cast<cudaStream_t>(stream), /*by_value=*/true);
  FP_API_END
}

int fp_track_cameras(fp_ctx* c, int C, const unsigned char* const* rgb_host, const float* const* depth_host, const float* K,
                     const int* H, const int* W, int M, const int* camera_of, const int* slots_host, const float* poses_in_dev,
                     int iterations, float* poses_out_dev, float* poses_out_host, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && rgb_host && depth_host && K && H && W && M > 0 && camera_of && slots_host && poses_in_dev && iterations >= 0,
             "fp_track_cameras: bad argument");
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  // everything is checked before anything is enqueued: the kernels index the mesh and camera tables unchecked
  FP_TRY(check_cameras(C, rgb_host, depth_host, H, W, M, camera_of, "fp_track_cameras"));
  FP_TRY(check_slots(c, M, slots_host, "fp_track_cameras"));
  DeviceGuard dg(c->device);
  return track_cameras_body(c, C, rgb_host, depth_host, K, H, W, M, camera_of, slots_host, poses_in_dev, iterations,
                            poses_out_dev, poses_out_host, reinterpret_cast<cudaStream_t>(stream), /*by_value=*/false);
  FP_API_END
}

int fp_register_objects(fp_ctx* c, const unsigned char* rgb_host, const float* depth_host, const float* K, int H, int W,
                        int M, const int* slots_host, const int* n_hyp_host, const unsigned char* masks_host,
                        const float* rot_grids_dev, int iterations, float* poses_out_dev, float* scores_out_dev,
                        int* best_out_dev, float* info_out_dev, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && rgb_host && depth_host && K && H > 0 && W > 0 && M > 0 && M <= 65535 && slots_host && n_hyp_host &&
                 masks_host && rot_grids_dev && iterations >= 0 && poses_out_dev && scores_out_dev && best_out_dev &&
                 info_out_dev,
             "fp_register_objects: bad argument");
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  FP_REQUIRE(c->net[1].loaded, "scorer weights not loaded");
  // everything is checked before anything is enqueued
  FP_TRY(check_slots(c, M, slots_host, "fp_register_objects"));
  DeviceGuard dg(c->device);
  const size_t npix = (size_t)H * W;
  std::vector<const unsigned char*> masks(M);
  for (int i = 0; i < M; ++i) masks[i] = masks_host + (size_t)i * npix;
  const std::vector<int> camera_of(M, 0);
  return register_cameras_body(c, 1, &rgb_host, &depth_host, K, &H, &W, M, camera_of.data(), slots_host, n_hyp_host,
                               masks.data(), rot_grids_dev, iterations, poses_out_dev, scores_out_dev, best_out_dev,
                               info_out_dev, reinterpret_cast<cudaStream_t>(stream), /*by_value=*/true);
  FP_API_END
}

int fp_register_cameras(fp_ctx* c, int C, const unsigned char* const* rgb_host, const float* const* depth_host, const float* K,
                        const int* H, const int* W, int M, const int* camera_of, const int* slots_host, const int* n_hyp_host,
                        const unsigned char* const* masks_host, const float* rot_grids_dev, int iterations,
                        float* poses_out_dev, float* scores_out_dev, int* best_out_dev, float* info_out_dev, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(c && rgb_host && depth_host && K && H && W && M > 0 && M <= 65535 && camera_of && slots_host && n_hyp_host &&
                 masks_host && rot_grids_dev && iterations >= 0 && poses_out_dev && scores_out_dev && best_out_dev &&
                 info_out_dev,
             "fp_register_cameras: bad argument");
  FP_REQUIRE(c->net[0].loaded, "refiner weights not loaded");
  FP_REQUIRE(c->net[1].loaded, "scorer weights not loaded");
  // everything is checked before anything is enqueued: the kernels index the mesh and camera tables unchecked
  FP_TRY(check_cameras(C, rgb_host, depth_host, H, W, M, camera_of, "fp_register_cameras"));
  for (int i = 0; i < M; ++i) FP_REQUIRE(masks_host[i], "fp_register_cameras: object %d: null mask", i);
  FP_TRY(check_slots(c, M, slots_host, "fp_register_cameras"));
  DeviceGuard dg(c->device);
  return register_cameras_body(c, C, rgb_host, depth_host, K, H, W, M, camera_of, slots_host, n_hyp_host, masks_host,
                               rot_grids_dev, iterations, poses_out_dev, scores_out_dev, best_out_dev, info_out_dev,
                               reinterpret_cast<cudaStream_t>(stream), /*by_value=*/false);
  FP_API_END
}

unsigned long long fp_graph_captures(fp_ctx* c) { return c ? c->graph_captures : 0ull; }

int fp_op_depth_filter(const float* depth_dev, float* out_dev, int H, int W, int which, void* stream) {
  FP_API_BEGIN
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  FP_REQUIRE(depth_dev && out_dev && H > 0 && W > 0, "fp_op_depth_filter: bad argument");
  if (which == 0) return erode_depth_launch(depth_dev, out_dev, H, W, 2, 0.001f, 0.8f, 100.f, st);
  return bilateral_depth_launch(depth_dev, out_dev, H, W, 2, 100.f, 2.f, 100000.f, st);
  FP_API_END
}

int fp_op_pose_update(const float* poses_in, const float* trans, const float* rot, float* poses_out, int N,
                      float mesh_diameter, float rot_normalizer, void* stream) {
  FP_API_BEGIN
  FP_REQUIRE(poses_in && trans && rot && poses_out, "fp_op_pose_update: null argument");
  return pose_update_launch(poses_in, trans, rot, poses_out, nullptr, nullptr, N, nullptr, nullptr, mesh_diameter / 2.0f,
                            rot_normalizer, reinterpret_cast<cudaStream_t>(stream));
  FP_API_END
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// fp_group: ONE process (one host thread) driving several GPUs — the reference's process model (run_demo.py is one
// script).  One fp_ctx per device, each with its own stream; register() shards the hypothesis list contiguously,
// every device filters the frame, derives the start poses and refines / featurises its slice; the only exchange is
// the per-hypothesis feature rows (+ refined poses), written by each device DIRECTLY into device 0's gather buffer
// over NVLink peer memory (cudaMemcpyAsync device-to-device on the producing device's stream: no host staging, no
// collective library); device 0 waits on one event per peer and runs the cross-hypothesis tail once.
// ------------------------------------------------------------------------------------------------
struct fp_group {
  // One device's share: its context, stream and completion event, and register()'s buffers there (rot grid [N][16],
  // start poses, info[4], refined slice).  Destroyed with its device current.
  struct Device {
    fp_ctx* ctx = nullptr;
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr;
    fp::DevBuf grid, start, info, refined;
    ~Device() {
      if (stream) cudaStreamDestroy(stream);
      if (done) cudaEventDestroy(done);
      fp_destroy(ctx);
    }
  };
  std::vector<std::unique_ptr<Device>> dev;
  struct Gather {
    fp::DevBuf feats_all, poses_all, scores, best;
  } gather;  // on device 0
  fp::PinnedBuf pin_rgb, pin_depth, pin_mask, pin_grid;  // portable: every device reads them
  unsigned long long epoch = 0;
};

extern "C" {

int fp_group_destroy(fp_group* g) {
  FP_API_BEGIN
  if (!g) return 0;
  for (size_t i = 0; i < g->dev.size(); ++i) {
    DeviceGuard dg(g->dev[i]->ctx->device);
    cudaDeviceSynchronize();
    if (i == 0) g->gather = fp_group::Gather();
    g->dev[i].reset();
  }
  delete g;
  return 0;
  FP_API_END
}

int fp_group_create(int ndev, const int* dev_ids, fp_group** out) {
  FP_API_BEGIN
  FP_REQUIRE(out && ndev > 0, "fp_group_create: bad argument");
  int visible = 0;
  FP_CUDA_OK(cudaGetDeviceCount(&visible));
  fp_group* g = new fp_group();
  int prev = 0;
  cudaGetDevice(&prev);
  for (int i = 0; i < ndev; ++i) {
    const int dev = dev_ids ? dev_ids[i] : i;
    if (dev < 0 || dev >= visible) {
      fp_group_destroy(g);
      set_last_error("fp_group_create: device %d not visible (%d devices)", dev, visible);
      cudaSetDevice(prev);
      return -1;
    }
    cudaSetDevice(dev);
    fp_ctx* c = nullptr;
    const int rc = fp_create(&c);
    if (rc) {
      fp_group_destroy(g);
      cudaSetDevice(prev);
      return rc;
    }
    auto d = std::make_unique<fp_group::Device>();
    d->ctx = c;
    cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking);
    cudaEventCreateWithFlags(&d->done, cudaEventDisableTiming);
    g->dev.push_back(std::move(d));
    if (i > 0) {
      // peers write their feature rows into device 0's buffer: map device 0's memory into this device
      const int dev0 = g->dev[0]->ctx->device;
      int can = 0;
      cudaDeviceCanAccessPeer(&can, dev, dev0);
      if (can) {
        const cudaError_t pe = cudaDeviceEnablePeerAccess(dev0, 0);
        if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) {
          set_last_error("fp_group_create: cudaDeviceEnablePeerAccess(%d -> %d): %s", dev, dev0, cudaGetErrorString(pe));
          fp_group_destroy(g);
          cudaSetDevice(prev);
          return -2;
        }
        cudaGetLastError();
      }
    }
  }
  cudaSetDevice(prev);
  *out = g;
  return 0;
  FP_API_END
}

int fp_group_size(fp_group* g) { return g ? (int)g->dev.size() : 0; }

fp_ctx* fp_group_ctx(fp_group* g, int i) { return (g && i >= 0 && i < (int)g->dev.size()) ? g->dev[i]->ctx : nullptr; }

int fp_group_load_network(fp_group* g, int which, const fp_tensor_t* tensors, int n) {
  FP_API_BEGIN
  FP_REQUIRE(g, "fp_group_load_network: null group");
  for (auto& d : g->dev) FP_TRY(fp_load_network(d->ctx, which, tensors, n));
  return 0;
  FP_API_END
}

int fp_group_set_config(fp_group* g, int which, float crop_ratio, float rot_normalizer) {
  FP_API_BEGIN
  FP_REQUIRE(g, "fp_group_set_config: null group");
  for (auto& d : g->dev) FP_TRY(fp_set_config(d->ctx, which, crop_ratio, rot_normalizer));
  return 0;
  FP_API_END
}

int fp_group_set_mesh(fp_group* g, int V, int F, const float* pos, const float* nrm, const float* uv, const float* vcol,
                      const int* faces, const unsigned char* tex_rgb, int Ht, int Wt, float diameter) {
  FP_API_BEGIN
  FP_REQUIRE(g, "fp_group_set_mesh: null group");
  for (auto& d : g->dev) FP_TRY(fp_set_mesh(d->ctx, V, F, pos, nrm, uv, vcol, faces, tex_rgb, Ht, Wt, diameter));
  return 0;
  FP_API_END
}

int fp_group_register(fp_group* g, const unsigned char* rgb_host, const float* depth_host, const float* K, int H, int W,
                      const unsigned char* mask_host, const float* rot_grid_host, int N, int iterations,
                      float* poses_out_host, float* scores_out_host, int* best_out_host, float* info_out_host) {
  FP_API_BEGIN
  FP_REQUIRE(g && rgb_host && depth_host && K && mask_host && rot_grid_host && poses_out_host && scores_out_host &&
                 best_out_host && N > 0 && H > 0 && W > 0,
             "fp_group_register: bad argument");
  const int G = (int)g->dev.size();
  const size_t npix = (size_t)H * W;
  // pinned staging, filled once, read by every device
  FP_TRY(pinned_alloc(nullptr, g->pin_rgb, npix * 3, cudaHostAllocPortable));
  FP_TRY(pinned_alloc(nullptr, g->pin_depth, npix * 4, cudaHostAllocPortable));
  FP_TRY(pinned_alloc(nullptr, g->pin_mask, npix, cudaHostAllocPortable));
  FP_TRY(pinned_alloc(nullptr, g->pin_grid, (size_t)N * 64, cudaHostAllocPortable));
  memcpy(g->pin_rgb.p, rgb_host, npix * 3);
  memcpy(g->pin_depth.p, depth_host, npix * 4);
  memcpy(g->pin_mask.p, mask_host, npix);
  memcpy(g->pin_grid.p, rot_grid_host, (size_t)N * 64);
  fp_ctx* c0 = g->dev[0]->ctx;
  fp_group::Gather& ga = g->gather;
  {
    DeviceGuard dg(c0->device);
    FP_TRY(dev_alloc(g->epoch, ga.feats_all, (size_t)N * 2048));
    FP_TRY(dev_alloc(g->epoch, ga.poses_all, (size_t)N * 64));
    FP_TRY(dev_alloc(g->epoch, ga.scores, (size_t)N * 4));
    FP_TRY(dev_alloc(g->epoch, ga.best, 16));
  }
  const int base = N / G, rem = N % G;
  for (int i = 0; i < G; ++i) {
    fp_group::Device& d = *g->dev[i];
    fp_ctx* c = d.ctx;
    DeviceGuard dg(c->device);
    cudaStream_t st = d.stream;
    const int lo = i * base + (i < rem ? i : rem), n = base + (i < rem ? 1 : 0);
    FP_TRY(dev_alloc(g->epoch, d.grid, (size_t)N * 64));
    FP_TRY(dev_alloc(g->epoch, d.start, (size_t)N * 64));
    FP_TRY(dev_alloc(g->epoch, d.info, 16));
    FP_TRY(dev_alloc(g->epoch, d.refined, (size_t)(n > 0 ? n : 1) * 64));
    FP_TRY(fp_set_frame(c, reinterpret_cast<const unsigned char*>(g->pin_rgb.p), reinterpret_cast<const float*>(g->pin_depth.p),
                        K, H, W, FP_FRAME_FILTER_DEPTH, INFINITY, st));
    FP_CUDA_OK(cudaMemcpyAsync(d.grid.p, g->pin_grid.p, (size_t)N * 64, cudaMemcpyHostToDevice, st));
    FP_TRY(fp_start_poses(c, reinterpret_cast<const unsigned char*>(g->pin_mask.p), 0, reinterpret_cast<const float*>(d.grid.p),
                          N, reinterpret_cast<float*>(d.start.p), reinterpret_cast<float*>(d.info.p), st));
    if (n > 0) {
      float* refined = reinterpret_cast<float*>(d.refined.p);
      FP_TRY(fp_refine(c, reinterpret_cast<const float*>(d.start.p) + (size_t)lo * 16, n, iterations, refined, nullptr,
                       nullptr, st));
      // the gather: feature rows and refined poses land in device 0's buffers, straight over peer memory
      FP_TRY(fp_score_features(c, refined, n, reinterpret_cast<float*>(ga.feats_all.p) + (size_t)lo * 512, st));
      FP_CUDA_OK(cudaMemcpyAsync(reinterpret_cast<float*>(ga.poses_all.p) + (size_t)lo * 16, refined, (size_t)n * 64,
                                 cudaMemcpyDefault, st));
    }
    FP_CUDA_OK(cudaEventRecord(d.done, st));
  }
  {
    DeviceGuard dg(c0->device);
    cudaStream_t s0 = g->dev[0]->stream;
    for (int i = 1; i < G; ++i) FP_CUDA_OK(cudaStreamWaitEvent(s0, g->dev[i]->done, 0));
    FP_TRY(fp_score_tail(c0, reinterpret_cast<const float*>(ga.feats_all.p), N, reinterpret_cast<float*>(ga.scores.p),
                         reinterpret_cast<int*>(ga.best.p), s0));
    FP_CUDA_OK(cudaMemcpyAsync(poses_out_host, ga.poses_all.p, (size_t)N * 64, cudaMemcpyDeviceToHost, s0));
    FP_CUDA_OK(cudaMemcpyAsync(scores_out_host, ga.scores.p, (size_t)N * 4, cudaMemcpyDeviceToHost, s0));
    FP_CUDA_OK(cudaMemcpyAsync(best_out_host, ga.best.p, 4, cudaMemcpyDeviceToHost, s0));
    if (info_out_host) FP_CUDA_OK(cudaMemcpyAsync(info_out_host, g->dev[0]->info.p, 16, cudaMemcpyDeviceToHost, s0));
    FP_CUDA_OK(cudaStreamSynchronize(s0));
  }
  return 0;
  FP_API_END
}

}  // extern "C"
