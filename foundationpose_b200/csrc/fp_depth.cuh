// fp_depth.cuh — launchers of the depth pre-processing kernels (fp_depth.cu).
#pragma once
#include <cuda_runtime.h>

#include "fp_crop.cuh"  // CameraDev

namespace fp {
int erode_depth_launch(const float* depth, float* out, int H, int W, int radius, float diff_thres, float ratio_thres,
                       float zfar, cudaStream_t stream);
int bilateral_depth_launch(const float* depth, float* out, int H, int W, int radius, float zfar, float sigmaD,
                           float sigmaR, cudaStream_t stream);
// erode(2) -> bilateral(2) -> back-projection (invalid: z < 0.001 or z > zfar_xyz) + rgb -> rgba of one frame, one
// launch (raw frame in format fmt in, filtered frame out)
int frame_prep_launch(const CameraDev& one, const FrameFmtDev& fmt, float zfar_xyz, cudaStream_t stream);
// the same for C cameras in one launch: cams, fmts DEVICE [C]; max_H x max_W covers the largest of the frames
int frame_prep_cameras_launch(const CameraDev* cams, const FrameFmtDev* fmts, int C, int max_H, int max_W, float zfar_xyz,
                              cudaStream_t stream);
// depth from its own sensor aligned to the colour frame (align_depth_kernel): sensor `s` to colour frame `colour` (size
// and intrinsics) by value, or for C cameras in one launch from the DEVICE sensor and camera tables [C], max_H x max_W
// covering the largest depth image.  The aligned buffers must be zero.
int align_depth_launch(const SensorDev& s, const CameraDev& colour, cudaStream_t stream);
int align_depth_cameras_launch(const SensorDev* sensors, const CameraDev* cams, int C, int max_H, int max_W,
                               cudaStream_t stream);
// n aligned slots to float32 metres in place
int aligned_to_depth_launch(unsigned int* buf, size_t n, cudaStream_t stream);
// guess_translation + start poses of M objects in two launches; off [M + 1] device row offsets of each object in
// rot_grid / poses_out ([off[M]][16]; null when M = 1 by value: rows [0, N)); stats: 6 M words of device scratch;
// info [M][4] = {tx, ty, tz, n_valid}.  cams null: every object is seen in frame `one` (filtered depth, H x W,
// intrinsics) and its mask is masks[m] ([M][H][W]).  Otherwise (fp_register_cameras) object m is seen in
// cams[camera_of[m]] (DEVICE table and [M] camera ids) and its mask ([H][W] of that camera) starts at byte mask_off[m]
// (DEVICE [M]) of `masks`; off is then never null
int start_poses_launch(const CameraDev& one, const CameraDev* cams, const int* camera_of, const unsigned char* masks,
                       const size_t* mask_off, const float* rot_grid, int N, int M, const int* off, unsigned int* stats,
                       float* poses_out, float* info, cudaStream_t stream);
}  // namespace fp
