// fp_vis.cuh — the debug canvases of get_vis (fp_vis.cu), composed from the crop producer's vis record.
#pragma once
#include <cuda_runtime.h>

namespace fp {

constexpr int kVisPad = 2;          // make_grid_image(padding=2)
constexpr int kVisRowH = 164;       // refiner row: make_grid of [rgbA, rgbB, depthA, depthB], nrow=4
constexpr int kVisRowW = 650;
constexpr int kVisScorePad = 5;     // scorer row: 5-pixel columns of 255 between the four images, 5 rows of 255 below
constexpr int kVisScoreRowH = 100;  // 160 x 655 resized by 0.625
constexpr int kVisScoreW = 409;
constexpr int kVisScorePitch = kVisScoreRowH + kVisScorePad;

// canvas height / width: kind 0 = refiner (N rows of start and refined poses side by side), 1 = scorer (N rows)
int vis_canvas_size(int kind, int N, int* H, int* W);
// the 256-entry colour map of the canvases, 0xRRGGBB
const unsigned* vis_colormap();
// rec: [N][2][160][160] vis record (CropParams::vis).  range[n] = (min, max) of hypothesis n's depth values over its
// first n_img images
int vis_range_launch(const float4* rec, int N, int n_img, float2* range, cudaStream_t stream);
// half blk (0 = start poses, 1 = refined poses) of the refiner canvas [H][W][3]
int vis_refine_launch(const float4* rec, const float2* range, int N, int blk, unsigned char* canvas, cudaStream_t stream);
// scorer canvas [N * 105][409][3]: row s shows hypothesis order[s]
int vis_score_launch(const float4* rec, const float2* range, const int* order, int N, unsigned char* canvas,
                     cudaStream_t stream);

}  // namespace fp
