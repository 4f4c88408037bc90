// fp_group.cu — the fp_group_* entry points of the C ABI (include/fpose.h).
#include <math.h>
#include <string.h>

#include <memory>
#include <vector>

#include "../../include/fpose.h"
#include "fp_common.cuh"
#include "fp_ctx.cuh"

using namespace fp;

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
    FP_TRY(dev_alloc(nullptr, ga.feats_all, (size_t)N * 2048));
    FP_TRY(dev_alloc(nullptr, ga.poses_all, (size_t)N * 64));
    FP_TRY(dev_alloc(nullptr, ga.scores, (size_t)N * 4));
    FP_TRY(dev_alloc(nullptr, ga.best, 16));
  }
  const int base = N / G, rem = N % G;
  for (int i = 0; i < G; ++i) {
    fp_group::Device& d = *g->dev[i];
    fp_ctx* c = d.ctx;
    DeviceGuard dg(c->device);
    cudaStream_t st = d.stream;
    const int lo = i * base + (i < rem ? i : rem), n = base + (i < rem ? 1 : 0);
    FP_TRY(dev_alloc(nullptr, d.grid, (size_t)N * 64));
    FP_TRY(dev_alloc(nullptr, d.start, (size_t)N * 64));
    FP_TRY(dev_alloc(nullptr, d.info, 16));
    FP_TRY(dev_alloc(nullptr, d.refined, (size_t)(n > 0 ? n : 1) * 64));
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
