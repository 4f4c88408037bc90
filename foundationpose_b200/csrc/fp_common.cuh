// fp_common.cuh — shared device helpers for the sm_90a kernels of libfpose.
//
// Raw PTX wrappers for mbarrier / TMA / wgmma (no CUTLASS dependency).
// Everything here targets sm_90a only; there is no fallback path.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <atomic>

namespace fp {

// ----------------------------------------------------------------------------------------------
// process-wide state that several fp_ctx (one per thread / GPU) may touch concurrently
// ----------------------------------------------------------------------------------------------
// kernels launched by this library (bench.py's gpu_launches); launches recorded into a CUDA graph are
// counted when the graph is replayed, not while it is captured
void note_launches(int n);
unsigned long long launch_count();
void set_capturing(bool on);  // thread-local
// cudaFuncSetAttribute is per-device state: a bit per device ordinal
inline bool device_bit_test(const std::atomic<unsigned long long>& m) {
  int d = 0;
  cudaGetDevice(&d);
  return (m.load(std::memory_order_acquire) >> (d & 63)) & 1ull;
}
inline void device_bit_set(std::atomic<unsigned long long>& m) {
  int d = 0;
  cudaGetDevice(&d);
  m.fetch_or(1ull << (d & 63), std::memory_order_release);
}
int num_sms();  // of the current device

// ----------------------------------------------------------------------------------------------
// error plumbing (host)
// ----------------------------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);
// 0 when `p` is memory a kernel on the current device may read and write, else -1 with the reason (prefixed by `fn`)
// in fp_last_error()
int check_device_ptr(const void* p, const char* what, const char* fn = "fp_pose_errors");
#define FP_CUDA_OK(expr)                                                                   \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      fp::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return -2;                                                                           \
    }                                                                                      \
  } while (0)
#define FP_REQUIRE(cond, ...)                                                              \
  do {                                                                                     \
    if (!(cond)) {                                                                         \
      fp::set_last_error(__VA_ARGS__);                                                     \
      return -1;                                                                           \
    }                                                                                      \
  } while (0)
// returns the status of a call that failed (nonzero)
#define FP_TRY(expr)     \
  do {                   \
    int _rc = (expr);    \
    if (_rc) return _rc; \
  } while (0)

// ----------------------------------------------------------------------------------------------
// programmatic dependent launch (PDL).  Every kernel of a network pass is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization: its CTAs may be scheduled (on SMs the previous kernel has
// already left) and run their prologue — barrier init, tensor-map prefetch, loads of constant
// weights — while the previous kernel's last wave is still draining.  Contract inside a kernel: pdl_trigger()
// early (lets the NEXT kernel be scheduled once every CTA of this one has started), and pdl_wait() before the
// first access to global memory that an earlier kernel writes or reads (it returns when all earlier kernels of
// the stream have completed and flushed).  FPOSE_PDL=0 falls back to plain stream order.
// ----------------------------------------------------------------------------------------------
bool pdl_enabled();
void pdl_skip_next();  // the next launch_pdl on this thread omits the programmatic-serialisation attribute

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              int cluster_x, Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (cluster_x > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = cluster_x;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// ----------------------------------------------------------------------------------------------
// device PTX helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n\t"
      "@P1 bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity), "r"(0x989680)
      : "memory");
}

// TMA: 5-D tiled load, global -> shared, completes on an mbarrier.
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* map, uint64_t* bar, void* dst,
                                            int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// TMA: 5-D tiled store, shared -> global (bulk async group)
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3,
                                             int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// ---- clusters
__device__ __forceinline__ uint32_t cluster_nctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---- register reallocation between warpgroups (setmaxnreg).  Every warp of a warpgroup executes the same call; the
// kernel must be allocated the register count the releases and requests are balanced against (its launch bound).
template <uint32_t N>
__device__ __forceinline__ void regs_release() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <uint32_t N>
__device__ __forceinline__ void regs_acquire() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// wgmma (warpgroup MMA) ------------------------------------------------------------------------
// fence before the first wgmma of a batch (orders earlier register / shared-memory accesses before it)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed groups of this warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// read-out of fragment registers only after the wgmma that writes them has been waited for
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// wgmma shared-memory descriptors (sm_90): start address, leading / stride byte offsets (16 B units), layout type in
// bits [62, 64): 0 = no swizzle, 1 = 128-byte swizzle.
//
// K-major operand, 128-byte swizzle: rows of 64 fp16 (128 B), 8-row groups `sbo` bytes apart (1024 for a dense tile),
// LBO unused.  Advancing 16 fp16 along K inside the swizzle atom is +32 B = +2 on the descriptor.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr, uint32_t sbo = 1024) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(sbo >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// MN-major operand, 128-byte swizzle: slab [k rows][64 mn-elements]; 8-row k groups 1024 B apart (SBO), consecutive
// 64-element mn atoms `lbo` bytes apart (LBO).
__device__ __forceinline__ uint64_t gmma_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// K-major operand without swizzle: core matrices of 8 rows x 16 B; the two 8-element K halves of a k-step `lbo` bytes
// apart, consecutive 8-row groups `sbo` bytes apart.
__device__ __forceinline__ uint64_t gmma_desc_linear(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)(lbo >> 4) << 16;
  d |= (uint64_t)(sbo >> 4) << 32;
  return d;
}

// Four 8 x 8 fp16 matrices between shared memory and registers, transposed.  Lane 8 i + r gives the address of row r
// (16 bytes) of matrix i; register i of lane l holds that matrix's elements (row 2 (l % 4) + e, column l / 4), e = 0, 1.
// So a memory row of eight consecutive channels of one pixel meets the wgmma accumulator fragment of a tile whose rows
// are channels and whose columns are pixels.
__device__ __forceinline__ void ldsm_x4_trans(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
__device__ __forceinline__ void stsm_x4_trans(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]),
               "r"(r[1]), "r"(r[2]), "r"(r[3])
               : "memory");
}

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

}  // namespace fp
