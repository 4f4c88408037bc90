/* fpose.h — C ABI of libfpose.so, the H100-native (sm_90a) render-and-compare hot path behind
 * NVlabs/FoundationPose's Python surfaces.
 *
 * Every entry point is `extern "C"`, takes plain pointers and sizes, returns 0 on success or a
 * negative error code (fp_last_error() returns a thread-local message); nothing throws or aborts.
 * All `void* stream` arguments are a cudaStream_t (pass torch.cuda.current_stream().cuda_stream);
 * all work is enqueued on that stream and is asynchronous unless stated otherwise.
 * Device pointers are owned by the caller; the library owns only what it allocates inside an
 * fp_ctx (packed weights, mesh copy, frame copy, workspaces).
 *
 * Each declaration cites the reference interface it replaces (paths relative to the
 * FoundationPose repository root).
 */
#ifndef FPOSE_H_
#define FPOSE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------ */
/* errors / counters                                                                          */
/* ------------------------------------------------------------------------------------------ */
const char* fp_last_error(void);
/* Number of CUDA kernels this library has launched so far in this process (bench.py's
 * `gpu_launches`). */
unsigned long long fp_launch_count(void);

/* Per-launch device timing of the two roofline kernels (CUDA events on the launching stream):
 * kind 0 = wgmma implicit-GEMM kernel (work = algorithmic FLOPs), kind 1 = crop producer
 * (work = algorithmic output bytes).  fp_prof_collect synchronises the device, returns and clears
 * the sums accumulated since fp_prof_enable(1). */
int fp_prof_enable(int on);
int fp_prof_collect(int kind, double* total_ms, double* total_work, int* launches);

/* ------------------------------------------------------------------------------------------ */
/* single operators (parity-test hooks; the product path below calls the same code)           */
/* ------------------------------------------------------------------------------------------ */

/* kinds of dense layer the wgmma implicit-GEMM kernel executes */
#define FP_LAYER_LINEAR 0   /* torch.nn.Linear / in_proj / out_proj (refine_network.py:56-70)      */
#define FP_LAYER_CONV3_S1 1 /* 3x3 s1 p1 conv of ResnetBasicBlock (network_modules.py:73-111)       */
#define FP_LAYER_CONV3_S2 2 /* 3x3 s2 p1 ConvBNReLU (refine_network.py:37, :45)                      */
#define FP_LAYER_CONV7_S2 3 /* 7x7 s2 p3 stem ConvBNReLU (refine_network.py:36)                      */

typedef struct fp_gemm_layer {
  int kind;
  int n_img;          /* images in the batch (LINEAR: 1)                                          */
  int Hin, Win;       /* un-padded input size (LINEAR: Hin = 1, Win = number of rows M)           */
  int Cin;            /* input channels (LINEAR: K; CONV7_S2: 8 = 6 real + 2 zero)                */
  int Cout;           /* output channels, multiple of 64                                          */
  const void* in;     /* fp16; NHWC.  CONV7_S2: [n][Hin+6][2][(Win+8)/2][8] = a zero-bordered
                         (Hin+6) x (Win+8) canvas, image at (3,3), every row stored as its even
                         columns then its odd columns (packing.pad_image_c8)                      */
  const void* w;      /* fp16 [Cout][taps*Cin] (tap-major, channel-minor); CONV7_S2:
                         [7 rows][4 tap pairs][2][64][8] (packing.pack_conv7)                     */
  const float* bias;  /* fp32 [Cout] (BatchNorm folded in)                                        */
  const void* res;    /* optional fp16 residual, same indexing as the output, leading dim res_ld  */
  int res_ld;
  void* out;          /* fp16 NHWC output                                                         */
  int out_ld;         /* elements between consecutive output pixels                               */
  int out_split;      /* >0: image n goes to image n % out_split at channel (n / out_split)*Cout;
                         must be a multiple of the tile's image count (2 for >= 8x8 outputs, else 8)  */
  const float* post_add; /* optional fp32 [Ho*Wo][Cout], added after the activation               */
  int relu;
} fp_gemm_layer_t;

/* Runs one layer: out = act(in (*) w + bias [+ res]) [+ post_add]. */
int fp_op_gemm_layer(const fp_gemm_layer_t* layer, void* stream);
/* Output channels per tile (64, 128 or 256) fp_op_gemm_layer would use for `layer`, which depends on the layer's
 * shape and the current device's SM count only.  Launches nothing and dereferences no pointer of the layer. */
int fp_op_gemm_tile_n(const fp_gemm_layer_t* layer, int* tile_n);
/* Output pixels (or linear rows) per tile that fp_op_gemm_layer would use for `layer`: 256 where a 128-channel 3x3
 * convolution runs with the weights as the wgmma M operand (FPOSE_SWAP_TILE=0 turns that tile off), 64 where a K = 512
 * linear layer runs on the weight-stationary kernel (FPOSE_LINEAR_WS=0 turns it off), else 128.  Same rules as
 * fp_op_gemm_tile_n. */
int fp_op_gemm_tile_m(const fp_gemm_layer_t* layer, int* tile_m);

/* softmax(Q K^T / sqrt(128)) V of nn.MultiheadAttention (refine_network.py:56-70, score_network.py:53):
 * qkv fp16 [B*400][1536] (q | k | v, 4 heads of 128 each), out fp16 [B*400][512].
 * `impl` is ignored (kept for ABI stability): there is one implementation, the wgmma kernel. */
int fp_op_attention(const void* qkv, void* out, int B, int impl, void* stream);

/* Transformer-head operators on the launch shapes of the product, for testing each kernel alone.  B sequences of 400
 * tokens x 512 channels.  Every pointer must be device memory of the current device; fp16 activations, gamma / beta,
 * w_f32 and mean_ws must be 16-byte aligned.  All arguments are checked before anything is enqueued on `stream`. */
#define FP_OP_MAX_SEQUENCES 65536
/* Attention of n_groups (1 or 2) column blocks of 1536 (q | k | v) per row of `ld` columns: qkv fp16 [B*400][ld],
 * out fp16 [n_groups][B*400][512].  The refiner's heads run ld 3072 with two groups, the scorer ld 1536 with one. */
int fp_op_attention_groups(const void* qkv, int ld, int n_groups, void* out, int B, void* stream);
/* LayerNorm over 512 channels (eps 1e-5): x, y fp16 [rows][512], gamma, beta fp32 [512]. */
int fp_op_layernorm(const void* x, void* y, const float* gamma, const float* beta, int rows, void* stream);
/* Refiner head read-out: out[b] = w . mean_t LayerNorm(x[b, t]) + bias.  x fp16 [B][400][512], gamma, beta fp32
 * [512], w fp32 [out_dim][512], bias fp32 [out_dim], out fp32 [B][out_dim], 1 <= out_dim <= 8. */
int fp_op_head_final(const void* x, const float* gamma, const float* beta, const float* w, const float* bias, float* out,
                     int B, int out_dim, void* stream);
/* Scorer features: out[b] = w_f32 mean_t x[b, t] + bias.  x fp16 [B][400][512], w_f32 fp32 [512][512], bias fp32
 * [512], mean_ws fp32 [B][512] workspace (receives the token means), out fp32 [B][512]. */
int fp_op_token_mean_proj(const void* x, const float* w_f32, const float* bias, float* mean_ws, float* out, int B,
                          void* stream);


/* ------------------------------------------------------------------------------------------ */
/* pose accuracy                                                                              */
/* ------------------------------------------------------------------------------------------ */

/* Largest model and batch fp_pose_errors accepts: every point coordinate index (3 P) and pose element index (16 N)
 * stays in `int`, and the grid (8 N CTAs) within the launch limits. */
#define FP_METRICS_MAX_POINTS 131072
#define FP_METRICS_MAX_POSES (1 << 24)
/* ADD / ADD-S (Utils.py:232-253) of N poses against n_gt (1 or N) ground-truth poses over P model points, on the
 * current device.  pts [P][3], pred [N][16], gt [n_gt][16] row-major, outputs [N]: DEVICE float32.  add_out or
 * adds_out may be NULL (not computed).  1 <= P <= FP_METRICS_MAX_POINTS, 0 <= N <= FP_METRICS_MAX_POSES.
 *   ADD   = mean_i |(R_p x_i + t_p) - (R_g x_i + t_g)|      (the reference's unused symetry_tfs is not an argument)
 *   ADD-S = mean_i min_j |(R_g x_i + t_g) - (R_p x_j + t_p)|   (ground-truth points query the estimated points)
 * fp32 distances of the transformed points, fp64 means.  Deterministic: a pose's errors do not depend on N, on n_gt
 * or on the call.  ADD alone costs O(N P); ADD-S O(N P^2).  Every pointer must be device memory of the current device
 * (cudaPointerGetAttributes); all arguments are checked before anything is enqueued.  Enqueued on `stream`; no sync. */
int fp_pose_errors(const float* pts, int P, const float* pred, int N, const float* gt, int n_gt,
                   float* add_out, float* adds_out, void* stream);

/* Largest symmetry set fp_sym_pose_errors accepts: four discrete symmetries times 315 steps of a continuous one fit
 * three times over. */
#define FP_METRICS_MAX_SYMMETRIES 4096
/* MSSD / MSPD of the BOP Challenge (Hodan et al., "BOP Challenge 2020 on 6D Object Localization", ECCV Workshops
 * 2020; bop_toolkit's pose_error.mssd / pose_error.mspd) of N poses against n_gt (1 or N) ground-truth poses over P model points and S symmetries, on the current device.
 * pts [P][3] metres, pred [N][16], gt [n_gt][16], sym [S][16] row-major (metres, the identity included by the caller),
 * K [n_K][9] row-major intrinsics (n_K 1 or N; needed only for mspd_out), outputs [N]: DEVICE float32.  mssd_out or
 * mspd_out may be NULL (not computed).  1 <= P <= FP_METRICS_MAX_POINTS, 0 <= N <= FP_METRICS_MAX_POSES,
 * 1 <= S <= FP_METRICS_MAX_SYMMETRIES.
 *   MSSD = min_s max_i |E x_i - (G s) x_i|                    metres
 *   MSPD = min_s max_i |pi(K, E x_i) - pi(K, (G s) x_i)|       pixels, pi(K, x) = (K x)[:2] / x_z
 * G s is composed in fp32 on the device (for s = I it is G exactly, so a pose scored against itself gives 0); distances
 * are fp32 differences of the transformed points.  A projection with x_z = 0 gives an infinite MSPD for that symmetry,
 * never a NaN.  Deterministic: a pose's errors do not depend on N, on n_gt, on n_K or on the order of `sym`.  Costs
 * O(N S P).  Every pointer must be device memory of the current device (cudaPointerGetAttributes); all arguments are
 * checked before anything is enqueued.  Enqueued on `stream`; no sync. */
int fp_sym_pose_errors(const float* pts, int P, const float* pred, int N, const float* gt, int n_gt, const float* sym,
                       int S, const float* K, int n_K, float* mssd_out, float* mspd_out, void* stream);

/* Limits of fp_vsd_errors.  FP_VSD_MAX_TAUS: misalignment tolerances per call (BOP uses 10); the per-CTA counters
 * live in shared memory.  FP_VSD_MAX_DIM: largest H and W — BOP's largest test frames (T-LESS Canon, 2560 x 1920) fit,
 * and 1/256-pixel vertex coordinates stay far inside int.  FP_VSD_MAX_VERTICES / FP_VSD_MAX_FACES: mesh size. */
#define FP_VSD_MAX_TAUS 64
#define FP_VSD_MAX_DIM 4096
#define FP_VSD_MAX_VERTICES (1 << 22)
#define FP_VSD_MAX_FACES (1 << 22)
/* VSD of the BOP Challenge (Hodan et al., ECCV Workshops 2016; bop_toolkit's pose_error.vsd with visib_mode 'bop19',
 * cost_type 'step') of N poses against n_gt (1 or N) ground-truth poses, on the current device.
 * Mesh: HOST arrays pos [V][3] metres and faces [F][3] int32 (meshlets are built and uploaded per call, stream-ordered).
 * DEVICE arrays: pred [N][16], gt [n_gt][16] row-major, depth [n_depth][H][W] float32 metres (0 = no measurement),
 * K [n_K][9] row-major, taus [T] metres, errs_out [N][T] float32, and the optional counts_out [N][T + 2] int32 =
 * (union, intersection, c_0 .. c_{T-1}); n_gt, n_depth, n_K are 1 or N.  1 <= T <= FP_VSD_MAX_TAUS,
 * 1 <= H, W <= FP_VSD_MAX_DIM, delta >= 0 and finite (metres).
 *   dE, dG  depth of the mesh rendered at E and at G (0 where not covered): the crop producer's coverage rule on a full
 *           frame (pixel (u, v) samples (u + 0.5, v + 0.5); 1/256-px snapping, top-left ties, depth test on 1/Z,
 *           znear 0.001, zfar 100); an OpenGL renderer may differ on silhouette pixels
 *   dist    d sqrt(((u - cx) / fx)^2 + ((v - cy) / fy)^2 + 1), integer u, v (BOP's depth_im_to_dist_im_fast), fp64
 *   visG  = (distG - distT <= delta or D = 0) and dG > 0
 *   visE  = ((distE - distT <= delta or D = 0) and dE > 0) or (visG and dE > 0)
 *   c_t   = |{visG and visE, |distG - distE| >= taus[t]}|;  e_t = (c_t + |visG or visE| - |visG and visE|) / |visG or visE|,
 *           1 when nothing is visible.
 * Counts are integers: a pose's errors and counts do not depend on N, on broadcasting or on the call.  Every device
 * pointer must be device memory of the current device; all arguments are checked before anything is enqueued.
 * Enqueued on `stream`; no sync. */
int fp_vsd_errors(const float* pos, int V, const int* faces, int F, const float* pred, int N, const float* gt, int n_gt,
                  const float* depth, int n_depth, int H, int W, const float* K, int n_K, float delta, const float* taus,
                  int T, float* errs_out, int* counts_out, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* product path                                                                               */
/* ------------------------------------------------------------------------------------------ */
typedef struct fp_ctx fp_ctx;

/* Creates a context on the current CUDA device (must be sm_90).  Replaces the implicit global
 * state of the reference predictors (`.cuda()` modules, nvdiffrast `RasterizeCudaContext`,
 * estimater.py:29-41, :166-171). */
int fp_create(fp_ctx** ctx);
int fp_destroy(fp_ctx* ctx);

/* Per-predictor configuration, as each reference predictor reads its own config.yml: which = 0 the refiner's
 * crop_ratio (predict_pose_refine.py:117-118) and rot_normalizer (cfg['rot_normalizer'], :221); which = 1 the
 * scorer's crop_ratio (predict_score.py:137-138; rot_normalizer ignored). */
int fp_set_config(fp_ctx* ctx, int which, float crop_ratio, float rot_normalizer);

/* One named host tensor of a packed network (see foundationpose_b200/engine.py for the packing:
 * BatchNorm folded, conv weights K-major fp16).  dtype: 0 = float32, 1 = float16. */
typedef struct fp_tensor {
  const char* name;
  const void* data; /* HOST pointer */
  int dtype;
  long long numel;
} fp_tensor_t;

/* which: 0 = RefineNet (predict_pose_refine.py:133-143 `load_state_dict`), 1 = ScoreNetMultiPair
 * (predict_score.py:146-156).  Copies to device memory owned by the context; validates names/sizes. */
int fp_load_network(fp_ctx* ctx, int which, const fp_tensor_t* tensors, int n);

/* Replaces Utils.py:104-130 `make_mesh_tensors` (HOST pointers; uv already v-flipped as in :117;
 * texture uint8 RGB [Ht][Wt][3]; pass uv = tex = NULL and vcol (float 0..1, [V][3]) for
 * vertex-coloured meshes).  diameter = estimater.py:54. */
int fp_set_mesh(fp_ctx* ctx, int V, int F, const float* pos, const float* nrm, const float* uv, const float* vcol,
                const int* faces, const unsigned char* tex_rgb, int Ht, int Wt, float diameter);
/* A context holds up to FP_MAX_MESHES meshes, one per slot.  fp_set_mesh is fp_set_mesh_slot(ctx, 0, ...); every
 * single-object entry point renders slot 0, fp_track_objects renders the slots it is given.  Same arguments and
 * validation as fp_set_mesh, plus the slot (0 <= slot < FP_MAX_MESHES).  Synchronises the device. */
#define FP_MAX_MESHES 64
int fp_set_mesh_slot(fp_ctx* ctx, int slot, int V, int F, const float* pos, const float* nrm, const float* uv,
                     const float* vcol, const int* faces, const unsigned char* tex_rgb, int Ht, int Wt, float diameter);
/* What fp_set_mesh derived for slot 0 (test hook): info[5] = {meshlets, mesh is closed and consistently oriented (0/1),
 * front-face winding sign used for back-face culling (0 = both sides are rendered, as nvdiffrast does), V, F}. */
int fp_mesh_info(fp_ctx* ctx, int* info);

/* Host inputs of fp_set_frame, fp_start_poses and fp_register.  Pageable host memory is copied into the context's
 * pinned staging before the call returns: the caller may reuse it at once, and the call does not wait on `stream` for
 * it.  Page-locked memory (cudaHostAlloc, cudaHostRegister) is copied straight from the caller's buffer on `stream`:
 * the caller keeps it unchanged until `stream` has passed the call.
 * Frames and masks of the tracking calls (fp_track, fp_track_objects, fp_track_cameras and their _submit variants),
 * fp_register_objects and fp_register_cameras: each buffer (each camera's rgb, each camera's depth, each mask;
 * fp_register_objects' mask block as one buffer) may be host or device memory, classified on its own with
 * cudaPointerGetAttributes, and one call may mix them.  Host memory, pageable, page-locked or managed, is copied into the
 * context's pinned staging before the call returns: the caller may reuse it at once.  Device memory of the context's
 * device is read in place: nothing is staged or uploaded for it (a device mask is copied into the context on the
 * device), and the kernels read it in stream order on `stream`.  The caller keeps it allocated and unchanged until
 * `stream` has passed the call; for a submit, until its ticket's work is done, so a producer that writes the next frame
 * into the same buffer on the same stream after the submit is safe.  Device memory of another device is refused before
 * anything is enqueued. */
#define FP_FRAME_ON_DEVICE 1    /* rgb/depth are device pointers (default: host, copied on `stream`) */
#define FP_FRAME_FILTER_DEPTH 2 /* erode_depth + bilateral_filter_depth (estimater.py:173-174, :257-258) */
/* Uploads one RGB-D frame (rgb uint8 [H][W][3], depth float32 [H][W] metres, K row-major 3x3), runs
 * the depth filters (Utils.py:304-395) and depth2xyzmap (Utils.py:399-438; zfar as in :426, use
 * INFINITY for register()).  Asynchronous on `stream`. */
int fp_set_frame(fp_ctx* ctx, const unsigned char* rgb, const float* depth, const float* K, int H, int W, int flags,
                 float zfar, void* stream);
/* Frames as sensors deliver them.  Each camera of a context has a frame format, the layout in which every later
 * frame-taking call reads that camera's rgb and depth buffers: fp_set_frame, fp_track*, fp_track_objects* and
 * fp_register_objects read camera 0; fp_track_cameras* and fp_register_cameras read camera i in camera i's format.
 *   color:       FP_COLOR_RGB8 / BGR8 (3 bytes per pixel) or RGBA8 / BGRA8 (4 bytes per pixel, alpha ignored)
 *   depth:       FP_DEPTH_F32 (float32 metres) or FP_DEPTH_U16 (uint16 units of depth_scale metres: the depth is
 *                (float)v * depth_scale rounded to nearest in fp32, numpy's v.astype(np.float32) * np.float32(s));
 *                0 stays invalid depth
 *   depth_scale: metres per unit (FP_DEPTH_U16 only; finite and > 0)
 *   rgb_pitch, depth_pitch: bytes from one row to the next (0 = packed rows); pixels within a row are packed
 * The result of any call is bit-identical to the same call on the frame converted on the host to packed RGB8 and
 * float32 metres by those expressions.  The default (all zero) is packed RGB8 + float32.  Host frames are staged
 * packed in their own format (2 bytes per depth pixel for FP_DEPTH_U16); device frames are read in place with their
 * pitch.  A call copies its cameras' formats when it is staged, so a call already submitted keeps the formats it was
 * submitted with; this call only records the format (host state: it never waits and enqueues nothing) and refuses an
 * unknown enum, a FP_DEPTH_U16 scale that is not finite and > 0, or a camera outside [0, FP_MAX_CAMERAS).  fmt = NULL
 * restores the default.  A frame-taking call refuses, before anything is enqueued, a pitch below the packed row bytes
 * and a depth pitch or depth pointer not aligned to the depth element size.  The cached graphs read the formats from
 * the argument block (tracking calls, fp_register_cameras) or take them eagerly: a new format replays them. */
#define FP_COLOR_RGB8 0
#define FP_COLOR_BGR8 1
#define FP_COLOR_RGBA8 2
#define FP_COLOR_BGRA8 3
#define FP_DEPTH_F32 0
#define FP_DEPTH_U16 1
typedef struct fp_frame_format {
  int color;
  int depth;
  float depth_scale;
  int rgb_pitch;
  int depth_pitch;
} fp_frame_format_t;
int fp_set_camera_format(fp_ctx* ctx, int camera, const fp_frame_format_t* fmt);
/* Depth from its own sensor.  A camera may be given a depth sensor: the depth image's size H x W, its intrinsics K
 * (row-major 3x3; only fx = K[0], fy = K[4], cx = K[2], cy = K[5] are read) and the rigid transform from the depth
 * camera to the colour camera T_color_from_depth (row-major 4x4, metres; only its top three rows are read).  Every
 * later frame-taking call then reads that camera's depth buffer as the depth sensor's H x W image, in the camera's
 * depth format and pitch (fp_set_camera_format), and aligns it to the colour frame on the device before the frame
 * filter, by librealsense's rs2::align rule for depth to colour, in fp32 with every operation rounded on its own: for
 * every depth pixel (x, y) whose raw value is not 0, with z its depth in metres, the corners (x - 0.5, y - 0.5) and
 * (x + 0.5, y + 0.5) are deprojected with the depth intrinsics at z, moved by T and projected with the colour
 * intrinsics (the call's K) to (u, v), rounded as (int)(u + 0.5), (int)(v + 0.5).  Unless Z > 0 at both corners and
 * 0 <= x0 <= x1 <= W - 1, 0 <= y0 <= y1 <= H - 1 (colour W x H), the pixel is dropped; otherwise every colour pixel
 * of [x0, x1] x [y0, y1] takes the smallest z of all depth pixels that cover it, and a pixel nothing covers is 0.
 * The stored value is the depth sensor's z, as rs2::align stores it.  The call's H, W, K and masks stay the colour
 * frame's.  Like fp_set_camera_format this is host state that a call copies when it is staged; it refuses a camera
 * outside [0, FP_MAX_CAMERAS), H or W outside [1, FP_DEPTH_SENSOR_MAX_DIM], a K or T that is not finite, and fx <= 0 or
 * fy <= 0.  s = NULL removes the camera's sensor.  Honoured by fp_set_frame, fp_track*, fp_register_objects (camera
 * 0) and fp_register_cameras; a frame-taking call checks the depth pitch against the sensor's W.  A new sensor, depth
 * size or depth address replays the cached graphs. */
#define FP_DEPTH_SENSOR_MAX_DIM 4096
typedef struct fp_depth_sensor {
  int H, W;
  float K[9];
  float T_color_from_depth[16];
} fp_depth_sensor_t;
int fp_set_camera_depth_sensor(fp_ctx* ctx, int camera, const fp_depth_sensor_t* s);
/* The alignment above as an operator, with no context: depth (device memory, s->H rows depth_pitch bytes apart, 0 =
 * packed) in depth_format FP_DEPTH_F32 or FP_DEPTH_U16 (times depth_scale) is aligned to a colour frame of H x W with
 * intrinsics K_color (host, row-major 3x3) into out (device, float32 [H][W] metres, 0 where nothing lands), on `stream`
 * of the current device.  Every pointer is checked before anything is enqueued. */
int fp_align_depth(const void* depth, int depth_format, float depth_scale, long long depth_pitch, const fp_depth_sensor_t* s,
                   const float* K_color, int H, int W, float* out, void* stream);
/* Replaces the xyz map derived by fp_set_frame with the caller's own (PoseRefinePredictor.predict's `xyz_map`
 * argument, predict_pose_refine.py:150,177): float32 [H][W][3], host or device pointer. */
int fp_set_xyz_map(fp_ctx* ctx, const float* xyz, void* stream);
/* Copies camera `camera`'s filtered depth [H][W] and/or xyz map [H][W][3], as the last frame-taking call prepared
 * them, to device buffers; hw_out[2] (optional) receives that camera's H and W (test hook).  Refuses a camera the last
 * call did not prepare (fp_set_frame, fp_track, fp_register_objects: camera 0 only). */
int fp_get_depth(fp_ctx* ctx, int camera, float* depth_out_dev, float* xyz_out_dev, int* hw_out, void* stream);

/* FoundationPose.guess_translation (estimater.py:137-156: centre of the mask's bounding box, median of the
 * masked valid depths of the CURRENT FILTERED frame) and generate_random_pose_hypo (estimater.py:127-134,
 * :203-209) on the device: mask uint8/bool [H][W] (host, or device if mask_on_device), rot_grid [N][16]
 * device -> poses_out [N][16] device (grid rotations, guessed translation) and info_out[4] device =
 * {tx, ty, tz, number of valid masked pixels (the `valid.sum() < 4` test of estimater.py:183)}. */
int fp_start_poses(fp_ctx* ctx, const unsigned char* mask, int mask_on_device, const float* rot_grid, int N,
                   float* poses_out, float* info_out, void* stream);

/* make_crop_data_batch (predict_pose_refine.py:25-89 for mode 0, predict_score.py:56-114 for mode 1):
 * poses [N][16] device.  Fills the context's crop buffer; optionally copies it to crops_out
 * (fp16 [2N][166][2][84][8]: images 0..N-1 rendered, N..2N-1 observed), an fp32 copy of the
 * normalised crops to dbg_out ([N][2][160][160][6]) and the crop windows to win_out
 * ([N][4] = left, top, sx, sy of tf_to_crop). */
int fp_make_crops(fp_ctx* ctx, const float* poses, int N, int mode, void* crops_out, float* dbg_out, float* win_out,
                  void* stream);
/* Tile edge of the crop producer: 0 = chosen from the batch size (80 px for >= 64 hypotheses, 32 px, 16 px for < 4),
 * or force 16 / 32 / 80 (A/B measurements and the tile-size invariance test: the crops do not depend on it). */
int fp_set_crop_tile(fp_ctx* ctx, int tile);
/* Work counters of one crop pass (profiling hook; synchronises): stats_out_host[4] = {meshlet visits, triangles set
 * up, fragments depth-tested, triangles that took the near-plane path}. */
int fp_crop_stats(fp_ctx* ctx, const float* poses, int N, int mode, int* stats_out_host, void* stream);

/* PoseRefinePredictor.predict (predict_pose_refine.py:149-239) without the host round trips: poses
 * in/out are DEVICE [N][16]; last_trans [N][3] / last_rot [N][9] (optional) receive
 * `last_trans_update` / `last_rot_update` (:238-239). */
int fp_refine(fp_ctx* ctx, const float* poses_in, int N, int iterations, float* poses_out, float* last_trans,
              float* last_rot, void* stream);

/* ScorePredictor.predict (predict_score.py:160-214): scores_out DEVICE [N] (= logits + 100),
 * best_out DEVICE int (first index of the maximum = ids[0] of estimater.py:226). */
int fp_score(fp_ctx* ctx, const float* poses, int N, float* scores_out, int* best_out, void* stream);
/* The two halves of fp_score, split where the hypothesis batch shards across GPUs: per-hypothesis
 * features (score_network.py:60-74), then — after an all-gather of the [N][512] features — the
 * cross-hypothesis attention + linear + argmax (score_network.py:84-88). */
int fp_score_features(fp_ctx* ctx, const float* poses, int N, float* feats_out, void* stream);
int fp_score_tail(fp_ctx* ctx, const float* feats, int L, float* scores_out, int* best_out, void* stream);
/* The segmented tail of the register calls (test hook): segment g is feature rows [seg_host[g], seg_host[g + 1]) and
 * its hypotheses attend only to each other.  seg_host: HOST [n_seg + 1] with seg_host[0] = 0, strictly increasing,
 * seg_host[n_seg] = L and at most 4096 rows per segment (refused, with nothing enqueued, otherwise).  scores_out DEVICE
 * [L] (= logits + 100), best_out DEVICE [n_seg]: each segment's first arg-max, relative to its first row. */
int fp_op_score_tail_segments(fp_ctx* ctx, const float* feats, int L, const int* seg_host, int n_seg, float* scores_out,
                              int* best_out, void* stream);

/* Hot loop of FoundationPose.register (estimater.py:203-235) with HOST buffers: uploads the N
 * start poses, refines `iterations` times, scores, and returns refined poses [N][16], scores [N]
 * and the best index.  Synchronises `stream` before returning. */
int fp_register(fp_ctx* ctx, const float* poses_host, int N, int iterations, float* poses_out_host,
                float* scores_out_host, int* best_out_host, void* stream);

/* FoundationPose.track_one (estimater.py:250-268) as ONE CUDA-graph launch per frame: the frame (rgb uint8 [H][W][3],
 * depth float32 [H][W], host or device: a host frame is staged through pinned memory owned by the context and uploaded,
 * a device frame is read in place, see above), erode_depth +
 * bilateral_filter_depth, depth2xyzmap_batch(zfar = inf), `iterations` refiner passes on ONE pose, pose read-back.
 * pose_in_dev: DEVICE [16] ob_in_cam of the centred mesh (pose_last), or NULL = continue from the pose this context's
 * previous fp_track produced.  pose_out_dev (DEVICE [16]) / pose_out_host (HOST [16]) are optional.  This is the
 * one-object case of fp_track_cameras (one camera, the mesh in slot 0) and shares its cached graph with
 * fp_track_objects of one object: the graph takes the frame from the camera table, so new intrinsics or a frame no
 * larger than one tracked before replay it.  The first tracking call, or one with a larger frame than any tracked
 * before, captures every cached graph of the context once more (the tracking calls' frame-preparation grid grows).
 * Synchronises. */
int fp_track(fp_ctx* ctx, const unsigned char* rgb, const float* depth, const float* K, int H, int W,
             const float* pose_in_dev, int iterations, float* pose_out_dev, float* pose_out_host, void* stream);
/* FoundationPose.track_one (estimater.py:250-268) applied to M objects of the same frame, as ONE CUDA-graph launch:
 * the frame (host or device, as fp_track), one erode_depth + bilateral_filter_depth + depth2xyzmap_batch(zfar = inf),
 * `iterations` refiner passes over a batch of M hypotheses where hypothesis i renders the mesh in slot slots_host[i],
 * read-back of the M poses.  slots_host: HOST [M] slot ids, each loaded (checked before anything is enqueued);
 * poses_in_dev: DEVICE [M][16] ob_in_cam of each centred mesh; poses_out_dev (DEVICE [M][16]) / poses_out_host
 * (HOST [M][16]) are optional.  Each pose equals what fp_track gives for that object alone, and what fp_set_frame
 * (FP_FRAME_FILTER_DEPTH, zfar = inf) + fp_refine give for it with its mesh in slot 0.  This is fp_track_cameras
 * with one camera (C = 1, every object seen by camera 0), and shares its cached graph: new intrinsics or a frame no
 * larger than one seen before replay it.  Leaves fp_track's continuation pose untouched.  Synchronises. */
int fp_track_objects(fp_ctx* ctx, const unsigned char* rgb, const float* depth, const float* K, int H, int W,
                     int M, const int* slots_host, const float* poses_in_dev, int iterations, float* poses_out_dev,
                     float* poses_out_host, void* stream);
/* fp_track_objects for M objects spread over C camera streams (1 <= C <= FP_MAX_CAMERAS), each camera with its own
 * frame size and intrinsics, as ONE CUDA-graph launch: object i is seen by camera camera_of[i] and tracked exactly as
 * fp_track_objects tracks it in that camera's frame alone, bit for bit; fp_track_objects is its one-camera case.
 *   rgb[c] / depth[c]: host or device uint8 [H[c]][W[c]][3] / float32 [H[c]][W[c]] frame of camera c, each host buffer
 *   uploaded through its camera's pinned staging, each device buffer read in place through the camera table (see above);
 *   K: [C][9] row-major intrinsics; camera_of, slots_host: HOST [M] camera and mesh
 *   slot of every object; poses_in_dev: DEVICE [M][16]; poses_out_dev (DEVICE [M][16]) / poses_out_host (HOST [M][16])
 *   are optional.
 * Everything is checked before anything is enqueued: every camera id in [0, C), every camera owning at least one
 * object, every slot loaded, non-null frames of positive size.  One frame-preparation launch filters every camera's
 * depth, then `iterations` refiner passes run over all M objects.  The camera table (buffers, sizes, intrinsics), the
 * slot ids and the camera ids are copied into the context first, so the cached graph depends on (C, M, iterations)
 * only: reordering objects or cameras, changing intrinsics, a frame no larger than one seen before, or frames at other
 * addresses, on the host or on the device, replay it.
 * Camera 0 is the context's frame: afterwards the context holds camera 0's filtered frame, as fp_track on that frame
 * leaves it.  Cameras 1.. get buffers of their own, kept at the largest frame size seen.  Leaves fp_track's
 * continuation pose untouched.  Synchronises. */
#define FP_MAX_CAMERAS 16
int fp_track_cameras(fp_ctx* ctx, int C, const unsigned char* const* rgb, const float* const* depth,
                     const float* K, const int* H, const int* W, int M, const int* camera_of, const int* slots_host,
                     const float* poses_in_dev, int iterations, float* poses_out_dev, float* poses_out_host, void* stream);

/* Non-blocking tracking: the host stages and submits the next call while the device still tracks the previous one.
 * Each blocking tracking call is its submit followed by fp_track_wait on its ticket.
 *   fp_track_cameras_submit / fp_track_objects_submit / fp_track_submit take the arguments of fp_track_cameras /
 *   fp_track_objects / fp_track except poses_out_host / pose_out_host, and check them the same way: a refused call
 *   enqueues nothing.  Each copies the host frames into pinned staging on the calling thread and enqueues the uploads,
 *   the graph launch and the pose read-back on `stream`, then writes the call's ticket to *ticket.  Once it returns the
 *   caller may reuse its host frame buffers (device frames: once the ticket's work is done); poses_out_dev (and
 *   fp_track's continuation pose) are complete in stream order, so the next call may read them as its poses_in_dev
 *   without any host synchronisation.
 *   The context has FP_TRACK_MAX_IN_FLIGHT staging sets, used in turn.  A submit that finds its set still in use
 *   blocks only until the uploads of the call that used it have left it, not until that call's result is ready.
 *   A submit on a stream other than the previous submit's makes its stream wait for the previous call first: the
 *   context's device buffers are never used by two streams at once.
 * fp_track_wait waits for the call's read-back and copies its poses (HOST [M][16], or [16] for fp_track) to
 * poses_out_host (NULL: the result is dropped).  Tickets may be collected in any order, each once: an unknown or
 * already collected ticket is refused and the context stays usable.  Asynchronous CUDA errors of the call are reported
 * here.  Every other entry point that uses the context's frames or workspaces first orders its stream after the last
 * submitted call, on the device: it does not wait on the host.  A staging set is waited for only by the call that
 * takes it again.  Results stay pending until collected.  fp_destroy waits for calls in flight and frees uncollected results. */
#define FP_TRACK_MAX_IN_FLIGHT 2
int fp_track_cameras_submit(fp_ctx* ctx, int C, const unsigned char* const* rgb, const float* const* depth,
                            const float* K, const int* H, const int* W, int M, const int* camera_of, const int* slots_host,
                            const float* poses_in_dev, int iterations, float* poses_out_dev, void* stream,
                            unsigned long long* ticket);
int fp_track_objects_submit(fp_ctx* ctx, const unsigned char* rgb, const float* depth, const float* K, int H,
                            int W, int M, const int* slots_host, const float* poses_in_dev, int iterations,
                            float* poses_out_dev, void* stream, unsigned long long* ticket);
int fp_track_submit(fp_ctx* ctx, const unsigned char* rgb, const float* depth, const float* K, int H, int W,
                    const float* pose_in_dev, int iterations, float* pose_out_dev, void* stream, unsigned long long* ticket);
int fp_track_wait(fp_ctx* ctx, unsigned long long ticket, float* poses_out_host);
/* Tracking health: how well each returned pose's rendered depth agrees with the observed depth, counted in the same
 * graph launch and read back with the poses.  For object i, at its OUTPUT pose, over the 160 x 160 pixels p of the
 * refiner's crop window (the refiner's crop_ratio, the object's camera and mesh slot): z_r(p) is the camera-space Z of
 * the mesh's nearest triangle at p (what the refiner's rendered crop normalises), z_o(p) the z of the nearest xyz-map
 * sample of the filtered depth the refiner's observed crop reads at p (0 outside the frame or where the depth is
 * invalid), d = z_o - z_r in fp32.  The counts, int32 [M][FP_FIT_COUNTS]:
 *   [0] covered   the mesh covers p
 *   [1] valid     covered and z_o >= 0.001
 *   [2] inlier    valid and |d| <= delta
 *   [3] occluded  valid and d < -delta: something is in front of the model (occlusion, not failure)
 *   [4] behind    valid and d > delta: the camera sees past the model's surface (free space violated: a lost track)
 * so inlier + occluded + behind = valid.  The rendered and observed windows differ by the refiner's 159/160 scale; the
 * counts compare the same crop pixel on both sides, as the refiner does.  Integer counts: they do not depend on the
 * number or order of objects and cameras, nor on the crop tile.  The poses are exactly those of the call without a fit. */
#define FP_FIT_COUNTS 5
/* fp_track_cameras_submit plus the counts above at every output pose.  delta: metres, finite and >= 0 (checked with the
 * other arguments: a refused call enqueues nothing).  fit_out_dev: optional DEVICE int32 [M][5], complete in stream
 * order.  delta travels with the slot and camera ids, so a new delta replays the cached graph.  A fit ticket may be
 * collected with fp_track_wait, which drops its counts. */
int fp_track_cameras_fit_submit(fp_ctx* ctx, int C, const unsigned char* const* rgb, const float* const* depth,
                                const float* K, const int* H, const int* W, int M, const int* camera_of,
                                const int* slots_host, const float* poses_in_dev, int iterations, float delta,
                                float* poses_out_dev, int* fit_out_dev, void* stream, unsigned long long* ticket);
/* fp_track_wait for a ticket of fp_track_cameras_fit_submit, also copying its counts to fit_out_host (HOST int32
 * [M][5], may be NULL).  A ticket submitted without a fit is refused and left uncollected: fp_track_wait still collects
 * it. */
int fp_track_fit_wait(fp_ctx* ctx, unsigned long long ticket, float* poses_out_host, int* fit_out_host);
/* FoundationPose.register (estimater.py:159-240) applied to M objects of the same frame in one call; object i gives
 * exactly what fp_set_frame + fp_start_poses + fp_refine + fp_score give for that object alone, bit for bit.
 *   1. Checks every argument before anything is enqueued: slots_host HOST [M] loaded slot ids (one slot may appear
 *      more than once: two instances of one object), n_hyp_host HOST [M] hypotheses per object (1..4096), both
 *      networks loaded.
 *   2. The frame (rgb uint8 [H][W][3], depth float32 [H][W]) and masks (uint8 [M][H][W], nonzero = object), each host
 *      or device as the tracking calls' frames (host buffers pinned-staged and uploaded, device ones read in place, the
 *      masks by one device copy), one erode_depth + bilateral_filter_depth + depth2xyzmap(zfar = inf).
 *   3. guess_translation + start poses of every object in one launch pair: rot_grids_dev DEVICE [sum N][16], object i's
 *      n_hyp_host[i] rotations after object i - 1's.
 *   4. Refines (`iterations` passes) and featurises whole objects in passes of at most 512 hypotheses (an object above
 *      that alone); hypothesis rows render their own object's slot.
 *   5. One cross-hypothesis scorer tail in which every object's hypotheses attend only to each other.
 * Outputs (DEVICE): poses_out_dev [sum N][16] refined poses, object-major, in grid order (not ranked; with iterations = 0
 * the start poses); scores_out_dev [sum N]; best_out_dev [M] first index of each object's maximum, relative to the
 * object; info_out_dev [M][4] = {tx, ty, tz, n_valid} as fp_start_poses.  An object with fewer than 4 valid masked
 * pixels still runs; the caller discards its results (estimater.py:183-189).  The frame filter, the start poses and
 * the crops take the frame by value, as fp_register does, so the cached graphs are captured again when the frame's
 * size or intrinsics change (not when it moves between host and device: the graphs hold the context's filtered frame,
 * prepared outside them).  Synchronises. */
int fp_register_objects(fp_ctx* ctx, const unsigned char* rgb, const float* depth, const float* K, int H, int W,
                        int M, const int* slots_host, const int* n_hyp_host, const unsigned char* masks,
                        const float* rot_grids_dev, int iterations, float* poses_out_dev, float* scores_out_dev,
                        int* best_out_dev, float* info_out_dev, void* stream);
/* fp_register_objects for M objects spread over C camera streams (1 <= C <= FP_MAX_CAMERAS), each camera with its own
 * frame size and intrinsics: object i is seen by camera camera_of[i] and gives exactly what fp_register_objects gives
 * for it with that camera's frame alone, bit for bit.
 *   rgb[c] / depth[c]: host or device uint8 [H[c]][W[c]][3] / float32 [H[c]][W[c]] frame of camera c, as
 *   fp_track_cameras; K: [C][9] row-major intrinsics; camera_of, slots_host, n_hyp_host: HOST [M] camera, mesh slot and
 *   hypothesis count (1..4096) of every object; masks[i]: host or device uint8 [H[camera_of[i]]][W[...]] (nonzero =
 *   object); rot_grids_dev as fp_register_objects.
 * Everything is checked before anything is enqueued: every camera id in [0, C), every camera owning at least one
 * object, non-null frames of positive size and non-null masks, every slot loaded, both networks loaded.  The host masks
 * go to the device in one copy per run of consecutive host masks (one copy when all are on the host), the device masks
 * by device copies; one frame-preparation launch filters every camera's depth and one launch pair computes
 * every object's start poses, each from its own camera's filtered depth and intrinsics.  Passes and the scorer tail as
 * fp_register_objects; a pass may mix cameras.  The camera table and each pass's slot and camera ids are copied into
 * the context first, so the cached graphs depend on the pass sizes and iterations only: reordering objects or cameras
 * or changing intrinsics replays them.  Camera 0 is the context's frame, as after fp_track_cameras.  Outputs: exactly
 * fp_register_objects' (object-major, unranked, best relative to the object, info [M][4]).  Synchronises. */
int fp_register_cameras(fp_ctx* ctx, int C, const unsigned char* const* rgb, const float* const* depth,
                        const float* K, const int* H, const int* W, int M, const int* camera_of, const int* slots_host,
                        const int* n_hyp_host, const unsigned char* const* masks, const float* rot_grids_dev,
                        int iterations, float* poses_out_dev, float* scores_out_dev, int* best_out_dev, float* info_out_dev,
                        void* stream);
/* Number of CUDA graphs this context has captured so far (test hook: a replay captures nothing). */
unsigned long long fp_graph_captures(fp_ctx* ctx);

/* The debug canvases of get_vis, composed on the device from the context's CURRENT frame and mesh slot 0, without the
 * text labels (the caller draws them: cv_draw_text).  canvas_out: DEVICE uint8 [H][W][3] of the size fp_vis_size
 * gives; hw_out (HOST [2], optional) receives (H, W).  Asynchronous on `stream`.
 *   kind 0 replaces predict_pose_refine.py:241-293: N rows of [rgbA | rgbB | depthA | depthB] (make_grid_image,
 *          padding 2, depth_to_vis of the normalised z over the row's range), crops at poses_a (DEVICE [N][16], the
 *          poses predict() received) on the left, at poses_b (the refined poses) on the right.
 *   kind 1 replaces predict_score.py:27-52, :219-224: row s = hypothesis order[s] (DEVICE int [N], e.g. the scores'
 *          descending argsort) of poses_a: [rgbA | depthA | rgbB | depthB] with 5-pixel gaps, raw depths over the
 *          rendered depth's range, resized to 100 x 409 by cv2's INTER_LINEAR rule, then 5 rows of 255.
 * The first call allocates the crop record (819 200 B per hypothesis, 206 MB at N = 252) as the context's high-water
 * mark; no other entry point does, and no cached graph is invalidated by it. */
int fp_vis(fp_ctx* ctx, int kind, const float* poses_a, const float* poses_b, int N, const int* order,
           unsigned char* canvas_out, int* hw_out, void* stream);
/* Canvas size of fp_vis (no GPU needed): hw_out[2] = (H, W).  Refiner: (166 N + 6, 1314), (168, 1306) for N = 1 (a
 * one-row grid is not padded); scorer: (105 N, 409). */
int fp_vis_size(int kind, int N, int* hw_out);
/* The canvases' 256-entry colour map (cv2.COLORMAP_JET as RGB) into rgb_out [256][3] (no GPU needed). */
int fp_vis_colormap(unsigned char* rgb_out);
/* The crop pass of fp_vis alone (test hook): rec_out DEVICE [N][2][160][160][4] fp32 = (r, g, b, depth) of the rendered
 * and the observed crop at poses (DEVICE [N][16]); depth is the normalised z for mode 0 (refiner), raw metres for mode 1
 * (scorer: rendered camera z, 0 where nothing is covered; nearest sample of the filtered depth). */
int fp_vis_crops(fp_ctx* ctx, const float* poses, int N, int mode, float* rec_out, void* stream);
/* Bytes of device memory fp_vis holds in this context (0 until the first fp_vis call). */
unsigned long long fp_vis_workspace_bytes(fp_ctx* ctx);

/* ------------------------------------------------------------------------------------------ */
/* one process, several GPUs (the reference's process model: run_demo.py is a single script)  */
/* ------------------------------------------------------------------------------------------ */
typedef struct fp_group fp_group;
/* One fp_ctx per device (dev_ids = NULL: devices 0..ndev-1), each with its own stream; devices 1.. get peer access to
 * device 0, where the gathered features live.  Call from one thread. */
int fp_group_create(int ndev, const int* dev_ids, fp_group** out);
int fp_group_destroy(fp_group* g);
int fp_group_size(fp_group* g);
fp_ctx* fp_group_ctx(fp_group* g, int i); /* for per-device calls of the single-context API */
/* fp_load_network / fp_set_config / fp_set_mesh on every context of the group */
int fp_group_load_network(fp_group* g, int which, const fp_tensor_t* tensors, int n);
int fp_group_set_config(fp_group* g, int which, float crop_ratio, float rot_normalizer);
int fp_group_set_mesh(fp_group* g, int V, int F, const float* pos, const float* nrm, const float* uv, const float* vcol,
                      const int* faces, const unsigned char* tex_rgb, int Ht, int Wt, float diameter);
/* FoundationPose.register (estimater.py:159-240) with the N hypotheses sharded contiguously over the group's devices
 * (BASELINE.json configs[3]): HOST frame, mask (uint8 [H][W]) and rotation grid [N][16]; every device filters the frame,
 * derives the start poses and refines / featurises its slice, writing its feature rows and refined poses straight into
 * device 0's buffers over NVLink peer memory; device 0 runs the cross-hypothesis tail once.  Outputs (HOST): refined
 * poses [N][16], scores [N], best index, optional info[4] = {tx, ty, tz, n_valid} of guess_translation.  Synchronises. */
int fp_group_register(fp_group* g, const unsigned char* rgb_host, const float* depth_host, const float* K, int H, int W,
                      const unsigned char* mask_host, const float* rot_grid_host, int N, int iterations,
                      float* poses_out_host, float* scores_out_host, int* best_out_host, float* info_out_host);

/* parity-test hooks on pre-built crops (fp16 [2N][166][2][84][8], device) */
int fp_op_refine_net(fp_ctx* ctx, const void* crops, int N, float* trans_out, float* rot_out, void* stream);
int fp_op_score_feats(fp_ctx* ctx, const void* crops, int N, float* feats_out, void* stream);
/* The encoder's 15 convolutions, one layer table for the product and these hooks.  N hypotheses, 0 <= N <= 512; the
 * A and B crops run as one batch of M = Np + N images, B from image Np = N rounded up to 4 (images N .. Np - 1 are
 * pads, never read by layer 6 on).
 * fp_op_encoder_layer (no GPU needed): layer `layer` (0 .. 14) at N into info[13] = {kind (fp_gemm_layer_t), launch
 * images, input height = width, Cin, Cout, the layer whose output is its input (-1: the crops), the layer whose output
 * is its residual (-1: none), out_split, adds the positional embedding (0 / 1), then the shape of its output buffer
 * (images, height, width, channels)}.  Layers 0-4 keep all M images; layer 5 writes N images of [A_i | B_{Np+i}]
 * (256 channels); layer 14's output is the tokens [N][20 x 20][512]. */
int fp_op_encoder_layer(int layer, int N, int* info);
/* Runs layers 0 .. last (0 .. 14) of network `which` (0 = refiner, 1 = scorer) on the crops (device, [2N] images as
 * fp_op_refine_net) and copies layer last's whole output buffer, fp16 NHWC of the shape fp_op_encoder_layer gives,
 * to `out` (device).  Returns the bytes copied, or a negative error code; every argument is checked before anything
 * is enqueued on `stream`. */
long long fp_op_encoder(fp_ctx* ctx, int which, const void* crops, int N, int last, void* out, void* stream);
/* Runs the heads of network `which` (0 = refiner: run_refine_heads, 1 = scorer: run_score_feats) on given tokens `tok`
 * (device, fp16 [N][400][512], 1 <= N <= 512) and copies one of the workspace buffers they leave to `out` (device).
 * M = 400 N rows; fp16 unless marked fp32; [2] = the two refiner heads (0 trans, 1 rot):
 *   refiner  0 qkv [M][3072], 1 att [2][M][512], 2 x1pre = out_proj(att) + tok, 3 x1 = LayerNorm1(x1pre),
 *            4 ff = relu(linear1(x1)), 5 x2pre = linear2(ff) + x1 (2-5 each [2][M][512]), 6 head_out fp32 [2][N][3]
 *   scorer   0 qkv [M][1536], 1 att [M][512], 2 token mean of att fp32 [N][512], 3 features fp32 [N][512]
 * Returns the bytes copied, or a negative error code; every argument is checked before anything is enqueued. */
long long fp_op_heads(fp_ctx* ctx, int which, const void* tok, int N, int stage, void* out, void* stream);
/* Host-only hook (no GPU needed) on the mesh preparation fp_set_mesh performs: meshlets of <= 64 triangles / <= 64
 * vertices + closedness / orientation analysis.  info[6] = {meshlets, closed (0/1), front-face winding sign (0 = none),
 * max triangles per meshlet, max vertices per meshlet, total triangles}; face_of_tri_out (optional, [F]) receives the
 * original face id of every meshlet triangle.  Verifies internally that every meshlet triangle maps back to its face. */
int fp_op_build_meshlets(int V, int F, const float* pos, const int* faces, int* info, int* face_of_tri_out,
                         float* meshlets_out /* optional [ceil(F/1)][8]: sphere xyz r, cone axis xyz cutoff */);
/* Host-only hook on the same mesh preparation: writes the number of triangles of each meshlet, in the order the crop
 * producer bins them (and fp_op_build_meshlets' face_of_tri_out lists their faces), to tris_of_meshlet_out ([F]
 * suffices).  Returns the number of meshlets, or a negative error code. */
int fp_op_meshlet_sizes(int V, int F, const float* pos, const int* faces, int* tris_of_meshlet_out);
/* which: 0 = erode_depth (Utils.py:359-395), 1 = bilateral_filter_depth (Utils.py:304-356) */
int fp_op_depth_filter(const float* depth_dev, float* out_dev, int H, int W, int which, void* stream);
/* egocentric_delta_pose_to_pose with the refiner's output decoding (predict_pose_refine.py:195-231), launched as the
 * refine loop launches it: hypothesis n moves by trans[n] times the half-diameter of the mesh in slot mesh_of_host[n]
 * (host [N]; null = slot 0; every slot must hold a mesh), rotations use the context's rot_normalizer (fp_set_config).
 * Device [N][16] poses; trans_delta_out [N][3] / rot_delta_out [N][9] (optional) receive the decoded deltas. */
int fp_op_pose_update(fp_ctx* ctx, const float* poses_in, const float* trans, const float* rot, const int* mesh_of_host,
                      int N, float* poses_out, float* trans_delta_out, float* rot_delta_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FPOSE_H_ */
