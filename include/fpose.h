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

/* softmax(Q K^T / sqrt(128)) V of nn.MultiheadAttention (refine_network.py:56-70, score_network.py:53):
 * qkv fp16 [B*400][1536] (q | k | v, 4 heads of 128 each), out fp16 [B*400][512].
 * `impl` is ignored (kept for ABI stability): there is one implementation, the wgmma kernel. */
int fp_op_attention(const void* qkv, void* out, int B, int impl, void* stream);


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

#define FP_FRAME_ON_DEVICE 1    /* rgb/depth are device pointers (default: host, copied on `stream`) */
#define FP_FRAME_FILTER_DEPTH 2 /* erode_depth + bilateral_filter_depth (estimater.py:173-174, :257-258) */
/* Uploads one RGB-D frame (rgb uint8 [H][W][3], depth float32 [H][W] metres, K row-major 3x3), runs
 * the depth filters (Utils.py:304-395) and depth2xyzmap (Utils.py:399-438; zfar as in :426, use
 * INFINITY for register()).  Asynchronous on `stream`. */
int fp_set_frame(fp_ctx* ctx, const unsigned char* rgb, const float* depth, const float* K, int H, int W, int flags,
                 float zfar, void* stream);
/* Replaces the xyz map derived by fp_set_frame with the caller's own (PoseRefinePredictor.predict's `xyz_map`
 * argument, predict_pose_refine.py:150,177): float32 [H][W][3], host or device pointer. */
int fp_set_xyz_map(fp_ctx* ctx, const float* xyz, void* stream);
/* Copies the filtered depth [H][W] and/or the xyz map [H][W][3] to device buffers (test hook). */
int fp_get_depth(fp_ctx* ctx, float* depth_out_dev, float* xyz_out_dev, void* stream);

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

/* Hot loop of FoundationPose.register (estimater.py:203-235) with HOST buffers: uploads the N
 * start poses, refines `iterations` times, scores, and returns refined poses [N][16], scores [N]
 * and the best index.  Synchronises `stream` before returning. */
int fp_register(fp_ctx* ctx, const float* poses_host, int N, int iterations, float* poses_out_host,
                float* scores_out_host, int* best_out_host, void* stream);

/* FoundationPose.track_one (estimater.py:250-268) as ONE CUDA-graph launch per frame: upload of the frame (HOST rgb
 * uint8 [H][W][3], depth float32 [H][W]; staged through pinned memory owned by the context), erode_depth +
 * bilateral_filter_depth, depth2xyzmap_batch(zfar = inf), `iterations` refiner passes on ONE pose, pose read-back.
 * pose_in_dev: DEVICE [16] ob_in_cam of the centred mesh (pose_last), or NULL = continue from the pose this context's
 * previous fp_track produced.  pose_out_dev (DEVICE [16]) / pose_out_host (HOST [16]) are optional.  Synchronises. */
int fp_track(fp_ctx* ctx, const unsigned char* rgb_host, const float* depth_host, const float* K, int H, int W,
             const float* pose_in_dev, int iterations, float* pose_out_dev, float* pose_out_host, void* stream);
/* FoundationPose.track_one (estimater.py:250-268) applied to M objects of the same frame, as ONE CUDA-graph launch:
 * one pinned-staged upload of the frame, one erode_depth + bilateral_filter_depth + depth2xyzmap_batch(zfar = inf),
 * `iterations` refiner passes over a batch of M hypotheses where hypothesis i renders the mesh in slot slots_host[i],
 * read-back of the M poses.  slots_host: HOST [M] slot ids, each loaded (checked before anything is enqueued);
 * poses_in_dev: DEVICE [M][16] ob_in_cam of each centred mesh; poses_out_dev (DEVICE [M][16]) / poses_out_host
 * (HOST [M][16]) are optional.  Each pose equals what fp_track gives for that object alone.  The slot ids and poses
 * are copied into the context first, so the cached graph depends on (M, iterations) only.  Leaves fp_track's
 * continuation pose untouched.  Synchronises. */
int fp_track_objects(fp_ctx* ctx, const unsigned char* rgb_host, const float* depth_host, const float* K, int H, int W,
                     int M, const int* slots_host, const float* poses_in_dev, int iterations, float* poses_out_dev,
                     float* poses_out_host, void* stream);
/* fp_track_objects for M objects spread over C camera streams (1 <= C <= FP_MAX_CAMERAS), each camera with its own
 * frame size and intrinsics, as ONE CUDA-graph launch: object i is seen by camera camera_of[i] and tracked exactly as
 * fp_track_objects tracks it in that camera's frame alone, bit for bit.
 *   rgb_host[c] / depth_host[c]: HOST uint8 [H[c]][W[c]][3] / float32 [H[c]][W[c]] frame of camera c, each uploaded
 *   through its own pinned staging; K: [C][9] row-major intrinsics; camera_of, slots_host: HOST [M] camera and mesh
 *   slot of every object; poses_in_dev: DEVICE [M][16]; poses_out_dev (DEVICE [M][16]) / poses_out_host (HOST [M][16])
 *   are optional.
 * Everything is checked before anything is enqueued: every camera id in [0, C), every camera owning at least one
 * object, every slot loaded, non-null frames of positive size.  One frame-preparation launch filters every camera's
 * depth, then `iterations` refiner passes run over all M objects.  The camera table (buffers, sizes, intrinsics), the
 * slot ids and the camera ids are copied into the context first, so the cached graph depends on (C, M, iterations)
 * only: reordering objects or cameras or changing intrinsics replays it.  Camera 0 is the context's frame: afterwards
 * the context holds camera 0's frame as fp_track_objects leaves it.  Cameras 1.. get buffers of their own, kept at the
 * largest frame size seen.  Leaves fp_track's continuation pose untouched.  Synchronises. */
#define FP_MAX_CAMERAS 16
int fp_track_cameras(fp_ctx* ctx, int C, const unsigned char* const* rgb_host, const float* const* depth_host,
                     const float* K, const int* H, const int* W, int M, const int* camera_of, const int* slots_host,
                     const float* poses_in_dev, int iterations, float* poses_out_dev, float* poses_out_host, void* stream);
/* FoundationPose.register (estimater.py:159-240) applied to M objects of the same frame in one call; object i gives
 * exactly what fp_set_frame + fp_start_poses + fp_refine + fp_score give for that object alone, bit for bit.
 *   1. Checks every argument before anything is enqueued: slots_host HOST [M] loaded slot ids (one slot may appear
 *      more than once: two instances of one object), n_hyp_host HOST [M] hypotheses per object (1..4096), both
 *      networks loaded.
 *   2. One pinned-staged upload of the frame (HOST rgb uint8 [H][W][3], depth float32 [H][W]) and of masks_host
 *      (HOST uint8 [M][H][W], nonzero = object), one erode_depth + bilateral_filter_depth + depth2xyzmap(zfar = inf).
 *   3. guess_translation + start poses of every object in one launch pair: rot_grids_dev DEVICE [sum N][16], object i's
 *      n_hyp_host[i] rotations after object i - 1's.
 *   4. Refines (`iterations` passes) and featurises whole objects in passes of at most 512 hypotheses (an object above
 *      that alone); hypothesis rows render their own object's slot.
 *   5. One cross-hypothesis scorer tail in which every object's hypotheses attend only to each other.
 * Outputs (DEVICE): poses_out_dev [sum N][16] refined poses, object-major, in grid order (not ranked; with iterations = 0
 * the start poses); scores_out_dev [sum N]; best_out_dev [M] first index of each object's maximum, relative to the
 * object; info_out_dev [M][4] = {tx, ty, tz, n_valid} as fp_start_poses.  An object with fewer than 4 valid masked
 * pixels still runs; the caller discards its results (estimater.py:183-189).  Synchronises. */
int fp_register_objects(fp_ctx* ctx, const unsigned char* rgb_host, const float* depth_host, const float* K, int H, int W,
                        int M, const int* slots_host, const int* n_hyp_host, const unsigned char* masks_host,
                        const float* rot_grids_dev, int iterations, float* poses_out_dev, float* scores_out_dev,
                        int* best_out_dev, float* info_out_dev, void* stream);
/* fp_register_objects for M objects spread over C camera streams (1 <= C <= FP_MAX_CAMERAS), each camera with its own
 * frame size and intrinsics: object i is seen by camera camera_of[i] and gives exactly what fp_register_objects gives
 * for it with that camera's frame alone, bit for bit.
 *   rgb_host[c] / depth_host[c]: HOST uint8 [H[c]][W[c]][3] / float32 [H[c]][W[c]] frame of camera c, each uploaded
 *   through its own pinned staging; K: [C][9] row-major intrinsics; camera_of, slots_host, n_hyp_host: HOST [M] camera,
 *   mesh slot and hypothesis count (1..4096) of every object; masks_host[i]: HOST uint8 [H[camera_of[i]]][W[...]]
 *   (nonzero = object); rot_grids_dev as fp_register_objects.
 * Everything is checked before anything is enqueued: every camera id in [0, C), every camera owning at least one
 * object, non-null frames of positive size and non-null masks, every slot loaded, both networks loaded.  All masks go
 * to the device in one copy; one frame-preparation launch filters every camera's depth and one launch pair computes
 * every object's start poses, each from its own camera's filtered depth and intrinsics.  Passes and the scorer tail as
 * fp_register_objects; a pass may mix cameras.  The camera table and each pass's slot and camera ids are copied into
 * the context first, so the cached graphs depend on the pass sizes and iterations only: reordering objects or cameras
 * or changing intrinsics replays them.  Camera 0 is the context's frame, as after fp_track_cameras.  Outputs: exactly
 * fp_register_objects' (object-major, unranked, best relative to the object, info [M][4]).  Synchronises. */
int fp_register_cameras(fp_ctx* ctx, int C, const unsigned char* const* rgb_host, const float* const* depth_host,
                        const float* K, const int* H, const int* W, int M, const int* camera_of, const int* slots_host,
                        const int* n_hyp_host, const unsigned char* const* masks_host, const float* rot_grids_dev,
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
int fp_op_tokens(fp_ctx* ctx, int which, const void* crops, int N, void* tokens_out, void* stream);
/* Host-only hook (no GPU needed) on the mesh preparation fp_set_mesh performs: meshlets of <= 64 triangles / <= 64
 * vertices + closedness / orientation analysis.  info[6] = {meshlets, closed (0/1), front-face winding sign (0 = none),
 * max triangles per meshlet, max vertices per meshlet, total triangles}; face_of_tri_out (optional, [F]) receives the
 * original face id of every meshlet triangle.  Verifies internally that every meshlet triangle maps back to its face. */
int fp_op_build_meshlets(int V, int F, const float* pos, const int* faces, int* info, int* face_of_tri_out,
                         float* meshlets_out /* optional [ceil(F/1)][8]: sphere xyz r, cone axis xyz cutoff */);
/* which: 0 = erode_depth (Utils.py:359-395), 1 = bilateral_filter_depth (Utils.py:304-356) */
int fp_op_depth_filter(const float* depth_dev, float* out_dev, int H, int W, int which, void* stream);
/* egocentric_delta_pose_to_pose with the refiner's output decoding (predict_pose_refine.py:195-231) */
int fp_op_pose_update(const float* poses_in, const float* trans, const float* rot, float* poses_out, int N,
                      float mesh_diameter, float rot_normalizer, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FPOSE_H_ */
