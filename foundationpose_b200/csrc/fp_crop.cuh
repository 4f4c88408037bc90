// fp_crop.cuh — parameters of the tiled crop producer (fp_crop.cu) and the device mesh it reads (fp_meshlet.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <vector>

namespace fp {

constexpr int kMeshletTris = 64;   // triangles per meshlet (one warp: two per lane)
constexpr int kMeshletVerts = 64;  // unique vertices per meshlet (one warp: two per lane)

// A meshlet = up to 64 spatially coherent triangles with their (up to 64) unique vertices, a bounding sphere
// and a normal cone in object space.  The crop kernel bins MESHLETS (not single triangles) to its 32x32-pixel
// tiles: one sphere / cone test per (tile, meshlet) instead of a per-triangle list.
struct __align__(16) Meshlet {
  float cx, cy, cz, r;       // bounding sphere
  float ax, ay, az, cutoff;  // normal cone: unit axis and min over faces of dot(axis, unit face normal); cutoff < -1: no cone
  int vert_off, n_verts, tri_off, n_tris;
};

struct MeshDev {
  const float4* vpos;  // [V] (x, y, z, 0)
  const float4* vnrm;  // [V] (nx, ny, nz, 0)
  const float4* vatt;  // [V] (u, v, 0, 0) [v already flipped, Utils.py:117] or (r, g, b, 0) in 0..1
  const int4* faces;   // [F] (i0, i1, i2, 0), ORIGINAL face order: the depth test breaks ties by the original id
  const Meshlet* meshlets;
  const int* ml_verts;   // global vertex id of every meshlet vertex slot
  const uint2* ml_tris;  // x = local vertex slots i0 | i1 << 8 | i2 << 16, y = original face id
  int n_meshlets;
  int V, F;
  float bs_x, bs_y, bs_z, bs_r;  // bounding sphere of the whole mesh (object space)
  int front_sign;  // 0: render both sides (open or inconsistently oriented mesh); +-1: sign of the snapped signed area
                   // of a FRONT-facing triangle (closed, consistently oriented mesh): back faces can never win the
                   // depth test and are culled per triangle and, through the normal cone, per meshlet — for hypotheses
                   // whose camera centre lies OUTSIDE the bounding sphere (from inside the solid the nearest surface
                   // is a back face, which nvdiffrast shows)
};

constexpr int kMaxMeshes = 64;  // FP_MAX_MESHES (include/fpose.h)

// One entry of the context's device-side mesh table: everything the crop producer and the pose update read about
// the mesh a hypothesis renders, filled by the host from the slot's buffers and the context's crop ratios.
struct __align__(16) MeshSlotDev {
  MeshDev mesh;       // front_sign already 0 when back-face culling is disabled (FPOSE_NO_CULL)
  const uchar4* tex;  // [Ht][Wt] RGBA8 or null
  int has_tex;
  int Ht, Wt;
  float r3[2];          // mesh_diameter * crop_ratio / 2 (Utils.py:603), [0] refiner, [1] scorer crop ratio
  float inv_radius;     // 1 / (mesh_diameter / 2)       (h5_dataset.py:96)
  float half_diameter;  // mesh_diameter / 2             (predict_pose_refine.py:199, pose update)
};

constexpr int kMaxCameras = 16;  // FP_MAX_CAMERAS (include/fpose.h)

// One camera's frame: its buffers (device), size and intrinsics.  Kernels take it by value (camera 0, the context's
// frame) or read it from the camera table of the tracking calls and fp_register_cameras.  frame_prep_kernel reads the
// raw frame and writes the filtered one; the crop producer and the start poses read the filtered one.
struct __align__(16) CameraDev {
  const unsigned char* rgb_raw;  // [H][W] uploaded frame, in the camera's format (FrameFmtDev)
  const float* depth_raw;        // [H][W], in the camera's format
  uchar4* rgb;                   // [H][W] RGBA8
  float* depth;                  // [H][W] eroded + bilateral-filtered depth
  float4* xyz_map;               // [H][W] (x, y, z, 0) back-projected filtered depth
  float fx, fy, cx, cy;
  int H, W;
};
static_assert(sizeof(CameraDev) == 64, "camera table entry: four uint4s");

// How a camera's raw frame (CameraDev::rgb_raw / depth_raw) is laid out (fp_frame_format_t, resolved by the host for
// where the frame is read: the caller's pitch in place, the packed row bytes once staged).  Only the frame preparation
// reads it, by value or from the format table beside the camera table.
// FrameFmtDev::depth_kind: how a raw depth frame stores its values
constexpr unsigned char kDepthF32 = 0;      // float32 metres
constexpr unsigned char kDepthU16 = 1;      // uint16 * depth_scale
constexpr unsigned char kDepthAligned = 2;  // a camera's aligned buffer (align_depth_kernel): uint32 slots, 0 = no depth
struct __align__(16) FrameFmtDev {
  int rgb_pitch;      // bytes per rgb row
  int depth_pitch;    // bytes per depth row
  float depth_scale;  // metres per unit (kDepthU16)
  unsigned char bpp;  // rgb bytes per pixel: 3 or 4
  unsigned char bgr;  // 1: channel order B, G, R
  unsigned char depth_kind;  // kDepthF32, kDepthU16 or kDepthAligned
  unsigned char packed;  // 1: packed RGB8 + float32, the layout frames had before formats (read without the fields above)
};
static_assert(sizeof(FrameFmtDev) == 16, "format table entry: one uint4");

// A camera's depth sensor (fp_set_camera_depth_sensor) as align_depth_kernel reads it: the raw depth image of the
// sensor, H x W, `pitch` bytes per row, float32 metres or uint16 * scale; its intrinsics; the top three rows of
// T_color_from_depth; and the camera's aligned buffer ([H][W] of the colour frame, uint32 slots, zeroed before the
// launch).  aligned = null: the camera has no sensor.  By value (camera 0) or from the sensor table beside the format
// table.
struct __align__(16) SensorDev {
  const void* depth;
  unsigned int* aligned;
  int pitch, u16;
  float scale;
  int H, W;
  float fx, fy, cx, cy;
  float T[12];
};
static_assert(sizeof(SensorDev) == 112, "sensor table entry: seven uint4s");

#ifdef __CUDACC__
// An aligned buffer's slot for depth z: the complement of an order key (unsigned order of the keys = float order of the
// values, negative ones included), so an atomicMax over a zeroed buffer keeps the smallest z whatever the order of the
// writes, and 0 (the key of a NaN, which is never stored) means no depth.
__device__ __forceinline__ unsigned int aligned_slot_of(float z) {
  const unsigned int b = __float_as_uint(z);
  return ~((b & 0x80000000u) ? ~b : (b | 0x80000000u));
}
__device__ __forceinline__ float aligned_depth_of(unsigned int s) {
  if (s == 0u) return 0.f;
  const unsigned int key = ~s;
  return __uint_as_float((key & 0x80000000u) ? (key & 0x7fffffffu) : ~key);
}
// Pixel (v, u) of a raw depth frame in metres: float32 as stored, uint16 * scale in one fp32 multiply rounded to
// nearest (no contraction), numpy's v.astype(np.float32) * np.float32(scale), or an aligned buffer's slot
__device__ __forceinline__ float raw_depth_at(const float* base, const FrameFmtDev& f, int v, int u) {
  const char* row = reinterpret_cast<const char*>(base) + (size_t)v * f.depth_pitch;
  if (f.depth_kind == kDepthU16) return __fmul_rn((float)__ldg(reinterpret_cast<const unsigned short*>(row) + u), f.depth_scale);
  if (f.depth_kind == kDepthAligned) return aligned_depth_of(__ldg(reinterpret_cast<const unsigned int*>(row) + u));
  return __ldg(reinterpret_cast<const float*>(row) + u);
}
// Pixel (v, u) of a raw colour frame as the context's RGBA8
__device__ __forceinline__ uchar4 raw_rgba_at(const unsigned char* base, const FrameFmtDev& f, int v, int u) {
  const unsigned char* p = base + (size_t)v * f.rgb_pitch + (size_t)u * f.bpp;
  const unsigned char c0 = __ldg(p), c1 = __ldg(p + 1), c2 = __ldg(p + 2);
  return f.bgr ? make_uchar4(c2, c1, c0, 255) : make_uchar4(c0, c1, c2, 255);
}
#endif

struct CropParams {
  const float* poses;  // [N][16] row-major ob_in_cam
  int N;
  float znear, zfar; // Utils.py:161 projection_matrix_from_intrinsics(znear=0.001, zfar=100)
  const MeshSlotDev* slots;  // [kMaxMeshes] device mesh table
  const int* mesh_of;        // [N] slot of every hypothesis, device; null = every hypothesis renders slot 0
  int mode;                  // 0 = refiner crops, 1 = scorer crops
  // outputs
  __half* crops;   // [b_img0 + N][166][2][84][8] fp16 (rows x {even, odd columns} x column pairs x 8 channels, the
                   // "EO" layout of fp_stem.cu): images 0..N-1 = rendered (A), b_img0..b_img0+N-1 = observed (B)
  int b_img0;      // first B image (N rounded up to the conv tile's image count, see b_img0_of in fp_ctx.cuh)
  float* dbg;      // optional [N][2][160][160][6] fp32 copy of the normalised crops
  float* win_out;  // optional [N][4] = (left, top, sx, sy)
  int tile_override;  // 0 = pick by batch size; 16 / 32 / 80 = force (fp_set_crop_tile, A/B tests)
  int* stats;      // optional [4]: meshlet visits, triangles set up, fragments, mixed (near-plane) triangles
  // optional, device: hypothesis n takes its frame from cams[camera_of[n]] instead of `frame` (the tracking calls,
  // fp_register_cameras); both null or both set
  const CameraDev* cams;
  const int* camera_of;
  // without `cams`, the frame of every hypothesis: rgb, xyz_map (mode 0), depth (mode 1), fx fy cx cy, H W
  CameraDev frame;
  // optional, single-camera (fp_vis): [N][2][160][160] fp32 record of every crop pixel, A then B: the r, g, b the
  // crops hold (0..1) and one depth value — mode 0 the normalised z of the xyz channels, mode 1 the raw depth in metres
  // (A: rendered camera z, 0 where nothing is covered; B: the nearest sample of the filtered depth, predict_score.py:90)
  float4* vis;
  // optional, camera-table path only (the tracking calls' fit pass, mode 0): no crop, dbg or vis record is written;
  // instead every hypothesis adds its kFitCounts agreement counts of rendered and observed depth at threshold
  // *fit_delta (device, metres) to fit[n][kFitCounts], which the caller zeroes first.  Both null or both set.
  int* fit;
  const float* fit_delta;
};
constexpr int kFitCounts = 5;  // FP_FIT_COUNTS (include/fpose.h): covered, valid, inlier, occluded, behind

int crop_launch(const CropParams& p, cudaStream_t stream);
// the unfiltered frame of fp_set_frame: one.rgb from one.rgb_raw, and with `depth` one.depth from one.depth_raw (a
// frame that is not packed float32), both read in format f
int raw_frame_launch(const CameraDev& one, const FrameFmtDev& f, bool depth, cudaStream_t stream);
// one.xyz_map from one.depth (invalid: z < 0.001 or z > zfar)
int depth_to_xyz_launch(const CameraDev& one, float zfar, cudaStream_t stream);

// Host-side mesh preparation (fp_meshlet.cu): meshlets + closedness / orientation analysis.
struct MeshHost {
  std::vector<float4> vpos, vnrm, vatt;
  std::vector<int4> faces;
  std::vector<Meshlet> meshlets;
  std::vector<int> ml_verts;
  std::vector<uint2> ml_tris;
  int front_sign = 0;
  int closed = 0;
  float bs[4] = {0.f, 0.f, 0.f, 0.f};  // bounding sphere of the mesh
};
// att: [V][2] uv (n_att = 2) or [V][3] colours (n_att = 3).  nrm or att may be null (zeros: geometry only, fp_vsd.cu).
// Returns 0 or a negative error (fp_last_error()).
int build_mesh_host(int V, int F, const float* pos, const float* nrm, const float* att, int n_att, const int* faces,
                    MeshHost& out);

}  // namespace fp
