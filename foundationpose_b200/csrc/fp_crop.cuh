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
// the mesh a hypothesis renders.  The host fills it with the expressions fp_api.cu used for its by-value kernel
// parameters, so slot 0 reproduces those values bit for bit.
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

// One entry of the camera table of fp_track_cameras: one camera stream's frame buffers (device), size and intrinsics.
// frame_prep_kernel reads the raw frame and writes the filtered one; the crop producer reads the filtered one.
struct __align__(16) CameraDev {
  const unsigned char* rgb_raw;  // [H][W][3] uploaded frame
  const float* depth_raw;        // [H][W]
  uchar4* rgb;                   // [H][W] RGBA8
  float* depth;                  // [H][W] eroded + bilateral-filtered depth
  float4* xyz_map;               // [H][W] (x, y, z, 0) back-projected filtered depth
  float fx, fy, cx, cy;
  int H, W;
};
static_assert(sizeof(CameraDev) == 64, "camera table entry: four uint4s");

struct CropParams {
  const float* poses;  // [N][16] row-major ob_in_cam
  int N;
  float fx, fy, cx, cy;
  int H, W;
  float znear, zfar; // Utils.py:161 projection_matrix_from_intrinsics(znear=0.001, zfar=100)
  const MeshSlotDev* slots;  // [kMaxMeshes] device mesh table
  const int* mesh_of;        // [N] slot of every hypothesis, device; null = every hypothesis renders slot 0
  // frame (device)
  const uchar4* rgb;      // [H][W] RGBA8
  const float4* xyz_map;  // [H][W] (x, y, z, 0)   (mode 0)
  const float* depth;     // [H][W]                (mode 1)
  int mode;               // 0 = refiner crops, 1 = scorer crops
  // outputs
  __half* crops;   // [b_img0 + N][166][2][84][8] fp16 (rows x {even, odd columns} x column pairs x 8 channels, the
                   // "EO" layout of fp_stem.cu): images 0..N-1 = rendered (A), b_img0..b_img0+N-1 = observed (B)
  int b_img0;      // first B image (N rounded up to the conv tile's image count, see fp_api.cu)
  float* dbg;      // optional [N][2][160][160][6] fp32 copy of the normalised crops
  float* win_out;  // optional [N][4] = (left, top, sx, sy)
  int tile_override;  // 0 = pick by batch size; 16 / 32 / 80 = force (fp_set_crop_tile, A/B tests)
  int* stats;      // optional [4]: meshlet visits, triangles set up, fragments, mixed (near-plane) triangles
  // optional, device: hypothesis n takes its frame (rgba, xyz, filtered depth, fx fy cx cy, H W) from
  // cams[camera_of[n]] instead of the by-value frame fields above (fp_track_cameras); both null or both set
  const CameraDev* cams;
  const int* camera_of;
  // optional, single-camera (fp_vis): [N][2][160][160] fp32 record of every crop pixel, A then B: the r, g, b the
  // crops hold (0..1) and one depth value — mode 0 the normalised z of the xyz channels, mode 1 the raw depth in metres
  // (A: rendered camera z, 0 where nothing is covered; B: the nearest sample of the filtered depth, predict_score.py:90)
  float4* vis;
};

int crop_launch(const CropParams& p, cudaStream_t stream);
int rgb_to_rgba_launch(const unsigned char* rgb, uchar4* out, int npix, cudaStream_t stream);
int depth_to_xyz_launch(const float* depth, float4* xyz, int H, int W, float fx, float fy, float cx, float cy,
                        float zfar, cudaStream_t stream);

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
// att: [V][2] uv (n_att = 2) or [V][3] colours (n_att = 3).  Returns 0 or a negative error (fp_last_error()).
int build_mesh_host(int V, int F, const float* pos, const float* nrm, const float* att, int n_att, const int* faces,
                    MeshHost& out);

}  // namespace fp
