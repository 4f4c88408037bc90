// fp_net.cu — the network execution plan: the encoder's layer table, the refiner heads and the scorer features as
// kernel launches on the context's workspaces, workspace sizing, the scorer tail's parameters, and fp_load_network,
// which checks the weights against that plan.
#include <stdio.h>

#include <algorithm>
#include <string>
#include <utility>
#include <vector>

#include "../../include/fpose.h"
#include "fp_attn.cuh"
#include "fp_common.cuh"
#include "fp_ctx.cuh"
#include "fp_gemm.cuh"

namespace fp {

int ensure_capacity(fp_ctx* c, int N) {
  if (N <= c->cap_n) return 0;
  const size_t n = (size_t)N;
  int rc = 0;
  // the crop buffer is zeroed once: the 3-pixel border is never written afterwards
  const size_t m = 2 * n + 3;  // A + pad + B images
  rc |= dev_alloc(&c->epoch, c->crops, m * kCropImg * 2, true);
  rc |= dev_alloc(&c->epoch, c->act0, m * 80 * 80 * 64 * 2);
  rc |= dev_alloc(&c->epoch, c->a1, m * 1600 * 128 * 2);
  rc |= dev_alloc(&c->epoch, c->a2, m * 1600 * 128 * 2);
  rc |= dev_alloc(&c->epoch, c->a3, m * 1600 * 128 * 2);
  rc |= dev_alloc(&c->epoch, c->ab0, n * 1600 * 256 * 2);
  rc |= dev_alloc(&c->epoch, c->ab1, n * 1600 * 256 * 2);
  rc |= dev_alloc(&c->epoch, c->ab2, n * 1600 * 256 * 2);
  rc |= dev_alloc(&c->epoch, c->c0, n * T * 512 * 2);
  rc |= dev_alloc(&c->epoch, c->c1, n * T * 512 * 2);
  rc |= dev_alloc(&c->epoch, c->c2, n * T * 512 * 2);
  rc |= dev_alloc(&c->epoch, c->tok, n * T * 512 * 2);
  rc |= dev_alloc(&c->epoch, c->qkv, n * T * 3072 * 2);
  rc |= dev_alloc(&c->epoch, c->att, 2 * n * T * 512 * 2);
  // x 2: one set per decoder head (they may run concurrently, see run_refine_heads)
  rc |= dev_alloc(&c->epoch, c->x1pre, 2 * n * T * 512 * 2);
  rc |= dev_alloc(&c->epoch, c->x1, 2 * n * T * 512 * 2);
  rc |= dev_alloc(&c->epoch, c->ff, 2 * n * T * 512 * 2);
  rc |= dev_alloc(&c->epoch, c->x2pre, 2 * n * T * 512 * 2);
  rc |= dev_alloc(&c->epoch, c->head_out, 2 * n * 3 * 4);
  rc |= dev_alloc(&c->epoch, c->poses_a, n * 16 * 4);
  rc |= dev_alloc(&c->epoch, c->poses_b, n * 16 * 4);
  rc |= dev_alloc(&c->epoch, c->feats, n * 512 * 4);
  rc |= dev_alloc(&c->epoch, c->lt_buf, n * 3 * 4);
  rc |= dev_alloc(&c->epoch, c->lr_buf, n * 9 * 4);
  rc |= dev_alloc(&c->epoch, c->feat_buf, n * 512 * 4);
  rc |= dev_alloc(&c->epoch, c->pose_stage, n * 16 * 4);
  rc |= dev_alloc(&c->epoch, c->tok_mean, n * 512 * 4);
  if (rc) return -2;
  c->cap_n = N;
  return 0;
}

int ensure_tail(fp_ctx* c, int L) {
  if (L <= c->tail_cap) return 0;
  int rc = 0;
  rc |= dev_alloc(&c->epoch, c->tail_qkv, (size_t)L * 1536 * 4);
  rc |= dev_alloc(&c->epoch, c->tail_attn, (size_t)L * 512 * 4);
  rc |= dev_alloc(&c->epoch, c->scores, (size_t)L * 4);
  rc |= dev_alloc(&c->epoch, c->best, 16);
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

const EncLayer kEncoder[kEncLayers] = {
    {LK_CONV7_S2, true, S, 8, 64, EB_CROPS, EB_ACT0, EB_NONE, 0, false, false},
    {LK_CONV3_S2, true, 80, 64, 128, EB_ACT0, EB_A1, EB_NONE, 0, false, false},
    {LK_CONV3_S1, true, 40, 128, 128, EB_A1, EB_A2, EB_NONE, 0, false, false},
    {LK_CONV3_S1, true, 40, 128, 128, EB_A2, EB_A3, EB_A1, 0, false, false},
    {LK_CONV3_S1, true, 40, 128, 128, EB_A3, EB_A2, EB_NONE, 0, false, false},
    // the last encodeA layer writes straight into the 256-channel concat buffer (refine_network.py:85)
    {LK_CONV3_S1, true, 40, 128, 128, EB_A2, EB_AB0, EB_A3, 256, true, false},
    {LK_CONV3_S1, false, 40, 256, 256, EB_AB0, EB_AB1, EB_NONE, 0, false, false},
    {LK_CONV3_S1, false, 40, 256, 256, EB_AB1, EB_AB2, EB_AB0, 0, false, false},
    {LK_CONV3_S1, false, 40, 256, 256, EB_AB2, EB_AB1, EB_NONE, 0, false, false},
    {LK_CONV3_S1, false, 40, 256, 256, EB_AB1, EB_AB0, EB_AB2, 0, false, false},
    {LK_CONV3_S2, false, 40, 256, 512, EB_AB0, EB_C0, EB_NONE, 0, false, false},
    {LK_CONV3_S1, false, 20, 512, 512, EB_C0, EB_C1, EB_NONE, 0, false, false},
    {LK_CONV3_S1, false, 20, 512, 512, EB_C1, EB_C2, EB_C0, 0, false, false},
    {LK_CONV3_S1, false, 20, 512, 512, EB_C2, EB_C1, EB_NONE, 0, false, false},
    {LK_CONV3_S1, false, 20, 512, 512, EB_C1, EB_TOK, EB_C2, 0, false, true},
};

void* enc_buf(fp_ctx* c, const __half* crops, EncBuf b) {
  switch (b) {
    case EB_CROPS: return const_cast<__half*>(crops);
    case EB_ACT0: return c->act0.p;
    case EB_A1: return c->a1.p;
    case EB_A2: return c->a2.p;
    case EB_A3: return c->a3.p;
    case EB_AB0: return c->ab0.p;
    case EB_AB1: return c->ab1.p;
    case EB_AB2: return c->ab2.p;
    case EB_C0: return c->c0.p;
    case EB_C1: return c->c1.p;
    case EB_C2: return c->c2.p;
    case EB_TOK: return c->tok.p;
    default: return nullptr;
  }
}

// Layer k's output buffer as the next layers read it, NHWC: {images, height, width, channels}.  The concat layer's
// buffer holds N images of [A_i | B_i] (2 Cout channels); the A / B layers' buffers hold all M images, pads included.
void enc_out_shape(int k, int N, int shape[4]) {
  const EncLayer& l = kEncoder[k];
  shape[0] = (l.ab_batch && !l.split) ? b_img0_of(N) + N : N;
  shape[1] = shape[2] = l.kind == LK_CONV3_S1 ? l.H : l.H / 2;
  shape[3] = l.out_ld ? l.out_ld : l.Cout;
}

// The layer whose output is still in buffer `b` when layer k runs: the last writer before k (-1: the crops)
int enc_source(int k, EncBuf b) {
  for (int j = k - 1; j >= 0; --j)
    if (kEncoder[j].out == b) return j;
  return -1;
}

// crops [2N][166][168][8] -> tokens [N][400][512] (+ positional embedding), or layers 0 .. last only
int run_encoder(fp_ctx* c, const Net& net, const __half* crops, int N, cudaStream_t st, int last) {
  char wn[32], bn[32];
  const int Np = b_img0_of(N);
  for (int k = 0; k <= last; ++k) {
    const EncLayer& l = kEncoder[k];
    snprintf(wn, sizeof wn, "enc.%d.w", k);
    snprintf(bn, sizeof bn, "enc.%d.b", k);
    FP_TRY(gemm_layer_launch(mk(l.kind, l.ab_batch ? Np + N : N, l.H, l.H, l.Cin, l.Cout, enc_buf(c, crops, l.in),
                                net.h(wn), net.f(bn), enc_buf(c, crops, l.out), 1, enc_buf(c, crops, l.res), l.out_ld,
                                l.split ? Np : 0, l.pe ? net.f("pe") : nullptr),
                             st));
  }
  return 0;
}

// tokens -> (trans, rot) raw network outputs, [2][N][3] fp32 in head_out
int run_refine_heads(fp_ctx* c, const Net& net, int N, cudaStream_t st) {
  const int M = N * T;
  // both heads' in_proj as one GEMM: [M,512] x [3072,512]^T
  FP_TRY(gemm_layer_launch(mk(LK_LINEAR, 1, 1, M, 512, 3072, c->tok.p, net.h("heads.in_w"), net.f("heads.in_b"), c->qkv.p, 0), st));
  FP_TRY(attn_core_launch(
      head_attn_params(reinterpret_cast<const __half*>(c->qkv.p), 3072, 2, reinterpret_cast<__half*>(c->att.p), N), st));
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
int run_score_feats(fp_ctx* c, const Net& net, int N, float* feats, cudaStream_t st) {
  const int M = N * T;
  FP_TRY(gemm_layer_launch(mk(LK_LINEAR, 1, 1, M, 512, 1536, c->tok.p, net.h("att.in_w"), net.f("att.in_b"), c->qkv.p, 0), st));
  FP_TRY(attn_core_launch(
      head_attn_params(reinterpret_cast<const __half*>(c->qkv.p), 1536, 1, reinterpret_cast<__half*>(c->att.p), N), st));
  FP_TRY(token_mean_proj_launch(reinterpret_cast<const __half*>(c->att.p), net.f("att.out_w32"), net.f("att.out_b"),
                                reinterpret_cast<float*>(c->tok_mean.p), feats, N, T, st));
  return 0;
}

// external crop layout of the test hooks: [2N] images, A then B, contiguous
int crops_import(fp_ctx* c, const void* ext, int N, cudaStream_t st) {
  const size_t img = kCropImg * 2;
  __half* dst = reinterpret_cast<__half*>(c->crops.p);
  const char* src = reinterpret_cast<const char*>(ext);
  FP_CUDA_OK(cudaMemcpyAsync(dst, src, (size_t)N * img, cudaMemcpyDeviceToDevice, st));
  FP_CUDA_OK(cudaMemcpyAsync(dst + (size_t)b_img0_of(N) * kCropImg, src + (size_t)N * img, (size_t)N * img,
                             cudaMemcpyDeviceToDevice, st));
  return 0;
}
int crops_export(fp_ctx* c, void* ext, int N, cudaStream_t st) {
  const size_t img = kCropImg * 2;
  const __half* src = reinterpret_cast<const __half*>(c->crops.p);
  char* dst = reinterpret_cast<char*>(ext);
  FP_CUDA_OK(cudaMemcpyAsync(dst, src, (size_t)N * img, cudaMemcpyDeviceToDevice, st));
  FP_CUDA_OK(cudaMemcpyAsync(dst + (size_t)N * img, src + (size_t)b_img0_of(N) * kCropImg, (size_t)N * img,
                             cudaMemcpyDeviceToDevice, st));
  return 0;
}

// The scorer tail over `L` feature rows as one segment; a segmented launch sets seg / n_seg / seg_max on top.
ScoreTailParams score_tail_params(const fp_ctx* c, const float* feats, int L, float* scores, int* best) {
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

// The scorer tail over n_seg segments of `feats`, segment g being rows [off_host[g], off_host[g + 1]).  Checks the
// offsets before anything is enqueued (off_host[0] = 0, every segment 1..4096 rows: the kernel's shared memory holds
// one segment's logits per head), sizes the tail's workspace and its per-segment arg-max tickets, uploads the offsets to
// seg_off and sets seg / n_seg / seg_max.  `trailing` more ints the caller keeps after the offsets go up in the same copy (the register
// calls' camera ids).  The register calls and fp_op_score_tail_segments both set their launch up here.
int segmented_tail_params(fp_ctx* c, const float* feats, const int* off_host, int n_seg, int trailing, float* scores,
                                 int* best, cudaStream_t st, const char* caller, ScoreTailParams& p) {
  FP_REQUIRE(n_seg >= 1, "%s: %d segments, need at least 1", caller, n_seg);
  FP_REQUIRE(off_host[0] == 0, "%s: the first segment starts at row %d, not 0", caller, off_host[0]);
  int seg_max = 0;
  for (int g = 0; g < n_seg; ++g) {
    const long long n = (long long)off_host[g + 1] - off_host[g];
    FP_REQUIRE(n >= 1 && n <= 4096, "%s: segment %d has %lld rows, need 1..4096", caller, g, n);
    seg_max = std::max(seg_max, (int)n);
  }
  const size_t ints = (size_t)(n_seg + 1 + trailing);
  FP_TRY(ensure_tail(c, off_host[n_seg]));
  FP_TRY(dev_alloc(&c->epoch, c->seg_off, ints * sizeof(int)));
  FP_TRY(dev_alloc(&c->epoch, c->tail_counter, std::max<size_t>(16, (size_t)n_seg * sizeof(unsigned int)), /*zero=*/true));
  FP_CUDA_OK(cudaMemcpyAsync(c->seg_off.p, off_host, ints * sizeof(int), cudaMemcpyHostToDevice, st));
  p = score_tail_params(c, feats, off_host[n_seg], scores, best);
  p.seg = reinterpret_cast<const int*>(c->seg_off.p);
  p.n_seg = n_seg;
  p.seg_max = seg_max;
  return 0;
}

}  // namespace fp

using namespace fp;

extern "C" {

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
    FP_TRY(dev_alloc(&c->epoch, d.buf, bytes));
    FP_CUDA_OK(cudaMemcpy(d.buf.p, t.data, bytes, cudaMemcpyHostToDevice));
    net.t[t.name] = std::move(d);  // a repeated name frees the earlier tensor
  }
  // verify that everything the execution plan needs is present, with the right size
  std::vector<std::pair<std::string, long long>> need;
  for (int i = 0; i < kEncLayers; ++i) {
    const EncLayer& l = kEncoder[i];
    // weights per output channel as packing.py lays them out: 7 filter rows x 8 taps x 8 channels (both zero-padded) for
    // the stem, 3 x 3 taps x Cin otherwise
    const long long k = l.kind == LK_CONV7_S2 ? 7 * 64 : 9LL * l.Cin;
    need.push_back({"enc." + std::to_string(i) + ".w", k * l.Cout});
    need.push_back({"enc." + std::to_string(i) + ".b", l.Cout});
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
    FP_TRY(upload(&c->epoch, c->fold_v, v));
    FP_TRY(dev_alloc(&c->epoch, c->tail_counter, 16, /*zero=*/true));
  }
  net.loaded = true;
  return 0;
  FP_API_END
}

}  // extern "C"
