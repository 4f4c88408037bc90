// fp_gemm.cuh — host-side description of one implicit-GEMM layer (conv / linear) for the
// wgmma tile kernel in fp_gemm.cu.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

namespace fp {

enum LayerKind : int {
  LK_LINEAR = 0,    // out[m, :] = in[m, :] @ W^T            (in: [M, K] fp16 row-major)
  LK_CONV3_S1 = 1,  // 3x3 stride 1 pad 1                      (in: NHWC fp16)
  LK_CONV3_S2 = 2,  // 3x3 stride 2 pad 1                      (in: NHWC fp16, H, W even)
  LK_CONV7_S2 = 3,  // 7x7 stride 2 pad 3, Cin padded to 8     (in: [n][Hin+6][2][(Win+8)/2][8] fp16,
                    //   3-pixel zero border already in memory, even/odd column split: fp_stem.cu)
};

// Geometry + pointers of one layer launch.  All pointers are device pointers.
struct GemmLayer {
  int kind;
  int n_img;        // images (LINEAR: 1)
  int Hin, Win;     // input spatial size, un-padded (LINEAR: Hin = 1, Win = M)
  int Cin;          // input channels (LINEAR: K).  CONV7: 8 (6 real + 2 zero)
  int Cout;         // output channels; multiple of the N tile (64 / 128 / 256)
  const void* in;   // fp16 activations
  const void* w;    // fp16 packed weights [Cout][Ktot], Ktot = taps * Cin (CONV7: [7][4][2][64][8], fp_stem.cu)
  const float* bias;      // [Cout] fp32 (BN folded)
  const void* res;        // optional residual, fp16, indexed like the output with ld = res_ld
  int res_ld;
  void* out;              // fp16 output
  int out_ld;             // elements between consecutive output pixels (>= Cout)
  int out_split;          // if > 0: image n writes to image (n % out_split) at channel offset
                          //         (n / out_split) * Cout   (fuses torch.cat((a, b), 1))
  const float* post_add;  // optional fp32 table [Ho*Wo][Cout] added after the activation (pos. emb.)
  int relu;
};

// Enqueue one layer on `stream`.  Returns 0 or a negative error code (fp_last_error() has text).
int gemm_layer_launch(const GemmLayer& L, cudaStream_t stream);
// The output channels per tile (64, 128 or 256) gemm_layer_launch would use for L; launches nothing.
int gemm_layer_tile_n(const GemmLayer& L, int* tile_n);
// The output pixels per tile (256 for the swapped 128-channel tile, 64 for the weight-stationary linear kernel, else
// 128); launches nothing.
int gemm_layer_tile_m(const GemmLayer& L, int* tile_m);


// Optional per-launch device timing (CUDA events on the launching stream) of the two kernels the
// roofline is reported for: kind 0 = gemm_tile_kernel (work = algorithmic FLOPs), kind 1 = crop_kernel
// (work = algorithmic output bytes).  Off by default; bench.py turns it on for a dedicated pass.
void prof_mark_begin(int kind, double work, cudaStream_t stream);
void prof_mark_end(cudaStream_t stream);
extern std::atomic<bool> g_prof_on;

}  // namespace fp
