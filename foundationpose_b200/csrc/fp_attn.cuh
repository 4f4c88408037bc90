// fp_attn.cuh — launchers of the non-GEMM transformer / scorer-tail / pose-update kernels.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stddef.h>

namespace fp {

struct AttnParams {
  const __half* qkv;  // [B*T][ld]; q at q_off + h*128, k at k_off + h*128, v at v_off + h*128
  int ld;
  int q_off, k_off, v_off;
  int group_col_stride;  // groups (e.g. trans / rot head) are further column blocks of the same rows
  int n_groups;
  __half* out;  // [group][B*T][ld_out], head h at column h*128
  int ld_out;
  size_t out_group_stride;
  int B, T, n_heads;
  float scale;  // 1/sqrt(head_dim)
};
// The heads' attention layout: T = 400 tokens, 4 heads of 128, q / k / v at columns 0 / 512 / 1024 of each group's
// 1536-column block.  Group g reads columns [1536 g, 1536 g + 1536) of rows of `ld` columns and writes
// out + g * B * 400 * 512.  Refiner: ld 3072, two groups (trans / rot head); scorer: ld 1536, one group.
inline AttnParams head_attn_params(const __half* qkv, int ld, int n_groups, __half* out, int B) {
  AttnParams ap;
  ap.qkv = qkv;
  ap.ld = ld;
  ap.q_off = 0;
  ap.k_off = 512;
  ap.v_off = 1024;
  ap.group_col_stride = 1536;
  ap.n_groups = n_groups;
  ap.out = out;
  ap.ld_out = 512;
  ap.out_group_stride = (size_t)B * 400 * 512;
  ap.B = B;
  ap.T = 400;
  ap.n_heads = 4;
  ap.scale = 0.08838834764831845f;
  return ap;
}
// the wgmma kernel (fp_attn_tc.cu)
int attn_core_launch(const AttnParams& p, cudaStream_t stream);
int attn_tc_launch(const AttnParams& p, cudaStream_t stream);

int layernorm_launch(const __half* x, __half* y, const float* gamma, const float* beta, int rows, cudaStream_t stream);
int head_final_launch(const __half* x, const float* gamma, const float* beta, const float* w, const float* bias,
                      float* out, int B, int T, int out_dim, cudaStream_t stream);
// w_f32: att.out_proj.weight as fp32 [512][512]; mean_ws: [B][512] fp32 workspace
int token_mean_proj_launch(const __half* x, const float* w_f32, const float* bias, float* mean_ws, float* out, int B, int T,
                           cudaStream_t stream);

struct ScoreTailParams {
  const float* feats;  // [L][512]
  int L;
  const float* w_in;    // att_cross.in_proj_weight  [1536][512] (fp32: the tail decides the argmax)
  const float* b_in;    // [1536]
  const float* fold_v;  // [512] = out_proj.weight^T linear.weight: out_proj followed by Linear(512, 1) is one dot product
  float fold_c;         // linear.weight . out_proj.bias + linear.bias
  float offset;         // +100 of predict_score.py:207
  float* qkv;           // workspace [L][1536]
  float* scores;        // out [L]
  int* best;            // out, optional: [n_seg] (one segment: [1]) arg-max of each segment, relative to its start
  unsigned int* counter;  // device words [n_seg], zero between launches (each segment's last CTA takes its arg-max and
                          // resets its word)
  // segments: hypotheses of different objects attend only within their own object's rows.  seg: DEVICE [n_seg + 1]
  // row offsets (seg[0] = 0, seg[n_seg] = L, no empty segment), seg_max: the longest segment (<= 4096).
  // seg = null: one segment of all L rows.
  const int* seg = nullptr;
  int n_seg = 1;
  int seg_max = 0;
};
int score_tail_launch(const ScoreTailParams& p, cudaStream_t stream);

struct MeshSlotDev;  // fp_crop.cuh
// trans_scale = mesh_diameter / 2 of every hypothesis; with a mesh table (`slots`, device) each hypothesis takes the
// half-diameter of its slot mesh_of[n] instead (slot 0 when mesh_of is null)
int pose_update_launch(const float* pose_in, const float* trans, const float* rot, float* pose_out,
                       float* trans_delta_out, float* rot_delta_out, int N, const MeshSlotDev* slots, const int* mesh_of,
                       float trans_scale, float rot_normalizer, cudaStream_t stream);
int f32_to_f16_launch(const float* x, __half* y, size_t n, cudaStream_t stream);

}  // namespace fp
