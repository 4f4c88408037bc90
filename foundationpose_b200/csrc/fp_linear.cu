// fp_linear.cu — weight-stationary wgmma kernel for the K = 512 linear layers of the attention heads (in-projections,
// out-projections, FF1 / FF2) on tall row counts.
//
// At K = 512 the k-loop of a 128 x 128 tile of gemm_tile_kernel is only eight k-blocks, and its epilogue (bias,
// residual, ReLU, fp16 conversion, slab writes, TMA store) does not overlap the next tile's wgmmas, so a large share of
// every tile is fixed cost.  Here a CTA keeps one 128-column weight panel (128 output channels x 512 K, 128 KB)
// resident in shared memory and streams only 64-row activation tiles past it.  The two consumer warpgroups take
// alternate tiles, and two named barriers order their k-loops so that one warpgroup's k-loop runs while the other
// runs its epilogue.
//
//   * Work items are (panel, 64-row tile) pairs in panel-major order; each persistent CTA takes one contiguous range,
//     which crosses at most one panel boundary (the host keeps ranges no longer than a panel).  CTAs running at the
//     same moment on different panels read the same activation rows, so those come from L2.
//   * The weights are constant during a pass, so the first panel is loaded before the programmatic-dependency wait.
//   * The A ring holds exactly one tile: stage kb holds k-block kb, and the fill of the CTA's j-th tile is phase j of
//     its barriers.  Each stage is released by the one warpgroup that reads it (128 arrivals).
//   * Each output element goes through the same m64n128k16 wgmmas in the same k order (k-blocks 0..7, four k16 steps
//     each) and the same fp32 epilogue (+bias, +residual, ReLU, one fp16 rounding) as in gemm_tile_kernel<128>, so the
//     output is bit-identical to it.
#include <stdlib.h>
#include <string.h>

#include "fp_common.cuh"
#include "fp_gemm.cuh"
#include "fp_wgmma.cuh"

namespace fp {

int encode_map_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box);  // fp_gemm.cu

constexpr int kLwsK = 512;
constexpr int kLwsKBlocks = kLwsK / 64;                     // 8 k-blocks of 64
constexpr int kLwsRows = 64;                                // rows per tile: one warpgroup's wgmma M
constexpr int kLwsCols = 128;                               // output channels per panel: the wgmma N
constexpr int kLwsThreads = 384;                            // warpgroup 0: TMA producer; warpgroups 1, 2: tiles
constexpr int kLwsBoxBytes = kLwsCols * 64 * 2;             // 16 KB: one k-block of the panel
constexpr int kLwsPanelBytes = kLwsKBlocks * kLwsBoxBytes;  // 128 KB
constexpr int kLwsStages = kLwsKBlocks;                     // the ring holds one tile
constexpr int kLwsStageBytes = kLwsRows * 64 * 2;           // 8 KB: 64 rows x 64 K
constexpr int kLwsSlabBytes = kLwsRows * 64 * 2;            // 8 KB: 64 rows x 64 channels, 128B-swizzled
constexpr int kLwsSlabs = 4;                                // two per consumer warpgroup
constexpr int kLwsSmemBytes =
    kLwsPanelBytes + kLwsStages * kLwsStageBytes + kLwsSlabs * kLwsSlabBytes + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert(kLwsSmemBytes <= 232448, "the weight-stationary linear kernel exceeds the 227 KB opt-in shared memory");
static_assert((2 * kLwsStages + 4) * 8 <= 256, "the mbarriers must fit their 256 bytes");

// Named barriers (0 is __syncthreads): kOrderBar + w lets warpgroup w start its next k-loop, kWgBar + w spans warpgroup
// w's own 128 threads
constexpr uint32_t kOrderBar = 2;
constexpr uint32_t kWgBar = 4;

struct LinearWsParams {
  int row_tiles;  // ceil(M / 64)
  int total;      // work items: (Cout / 128) * row_tiles
  const float* bias;
  int has_res;
  int relu;
};

__device__ __forceinline__ void named_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_arrive(uint32_t id, uint32_t count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

__global__ void __launch_bounds__(kLwsThreads, 1)
    linear_ws_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w,
                     const __grid_constant__ CUtensorMap map_out, const __grid_constant__ CUtensorMap map_res,
                     const __grid_constant__ LinearWsParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* panel = smem;                                   // [8 k-blocks][128 rows][128 B]
  uint8_t* ring = panel + kLwsPanelBytes;                  // [8 stages][64 rows][128 B]
  uint8_t* staging = ring + kLwsStages * kLwsStageBytes;   // [2 warpgroups][2 slabs]
  uint64_t* bars = reinterpret_cast<uint64_t*>(staging + kLwsSlabs * kLwsSlabBytes);
  uint64_t* full = bars;                        // [8]
  uint64_t* empty = bars + kLwsStages;          // [8]
  uint64_t* panel_full = bars + 2 * kLwsStages;
  uint64_t* panel_empty = panel_full + 1;       // both warpgroups are done with the first panel
  uint64_t* res_full = panel_full + 2;          // [2], one per warpgroup

  // this CTA's items [i0, i0 + n); local tile jb is the first on the next panel (n: the range stays on one panel)
  const int i0 = (int)((long long)blockIdx.x * p.total / gridDim.x);
  const int n = (int)((long long)(blockIdx.x + 1) * p.total / gridDim.x) - i0;
  const int panel0 = i0 / p.row_tiles;
  const int jb = min(n, (panel0 + 1) * p.row_tiles - i0);
  const bool reload = jb < n;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_w);
    tma_prefetch_desc(&map_out);
    if (p.has_res) tma_prefetch_desc(&map_res);
    for (int s = 0; s < kLwsStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 128);
    }
    mbar_init(panel_full, 1);
    mbar_init(panel_empty, 256);
    mbar_init(&res_full[0], 1);
    mbar_init(&res_full[1], 1);
    mbar_fence_init();
    // Only the network loader writes the weights, never a kernel of the pass: the first panel loads under the
    // previous kernel's tail
    mbar_expect_tx(panel_full, kLwsPanelBytes);
    for (int kb = 0; kb < kLwsKBlocks; ++kb)
      tma_load_2d(&map_w, panel_full, panel + kb * kLwsBoxBytes, kb * 64, panel0 * kLwsCols);
  }
  __syncthreads();
  pdl_trigger();
  pdl_wait();  // activations and the residual are touched only from here on

  if (threadIdx.x < 128) {
    // ------------------------------------------------------------------ TMA producer
    if (threadIdx.x == 0) {
      for (int j = 0; j < n; ++j) {
        if (j == jb) {
          // the second panel replaces the first once both warpgroups' last wgmmas on it have completed
          mbar_wait(panel_empty, 0);
          mbar_expect_tx(panel_full, kLwsPanelBytes);
          for (int kb = 0; kb < kLwsKBlocks; ++kb)
            tma_load_2d(&map_w, panel_full, panel + kb * kLwsBoxBytes, kb * 64, (panel0 + 1) * kLwsCols);
        }
        const int row0 = ((i0 + j) % p.row_tiles) * kLwsRows;
        for (int kb = 0; kb < kLwsKBlocks; ++kb) {
          mbar_wait(&empty[kb], (uint32_t)((j & 1) ^ 1));
          mbar_expect_tx(&full[kb], kLwsStageBytes);
          tma_load_2d(&map_a, &full[kb], ring + kb * kLwsStageBytes, kb * 64, row0);
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: warpgroup w takes tiles w, w + 2, ...
  const int ct = threadIdx.x - 128;
  const int w = ct >> 7;
  const int lane = threadIdx.x & 31;
  const int r0 = 16 * ((ct >> 5) & 3) + (lane >> 2);  // this thread's rows of the tile: r0 and r0 + 8
  const int cq = 2 * (lane & 3);                       // and columns 8 j + cq, 8 j + cq + 1
  const bool leader = (ct & 127) == 0;
  uint8_t* slabs = staging + w * 2 * kLwsSlabBytes;
  // warpgroup 1 never reads the first panel when the boundary follows the range's first tile
  if (reload && w >= jb) mbar_arrive(panel_empty);
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  for (int j = w, it = 0; j < n; j += 2, ++it) {
    const int item = i0 + j;
    const int pn = item / p.row_tiles;
    const int row0 = (item - pn * p.row_tiles) * kLwsRows;
    // k-loops run in tile order: tile j's starts once tile j - 1's wgmmas are issued, and so also after all of that
    // tile's stages were filled (a fill is awaited by parity, which cannot tell fill j from fill j - 2)
    if (j > 0) named_sync(kOrderBar + w, 256);
    mbar_wait(panel_full, j >= jb ? 1u : 0u);
    for (int kb = 0; kb < kLwsKBlocks; ++kb) {
      mbar_wait(&full[kb], (uint32_t)(j & 1));
      const uint64_t da = gmma_desc_sw128(smem_u32(ring + kb * kLwsStageBytes));
      const uint64_t db = gmma_desc_sw128(smem_u32(panel + kb * kLwsBoxBytes));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        Wgmma<128>::ss(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      if (kb == 0 && leader) {
        // this warpgroup's previous stores leave its slabs while the first wgmmas run; then the tile's residual goes
        // into them and arrives during the k-loop
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        if (p.has_res) {
          mbar_expect_tx(&res_full[w], 2 * kLwsSlabBytes);
          for (int s = 0; s < 2; ++s)
            tma_load_5d(&map_res, &res_full[w], slabs + s * kLwsSlabBytes, pn * kLwsCols + 64 * s, row0, 0, 0, 0);
        }
      }
      if (kb > 0) {
        wgmma_wait<1>();
        mbar_arrive(&empty[kb - 1]);
      }
    }
    if (j + 1 < n) named_arrive(kOrderBar + (w ^ 1), 256);
    wgmma_wait<0>();
    fence_regs(acc);
    mbar_arrive(&empty[kLwsKBlocks - 1]);
    if (reload && j < jb && j + 2 >= jb) mbar_arrive(panel_empty);  // this warpgroup's last tile on the first panel

    // ---- epilogue: channels [64 b, 64 b + 64) of the tile into slab b, the arithmetic of gemm_tile_kernel<128>
    const float* bias = p.bias + pn * kLwsCols;
    if (p.has_res) mbar_wait(&res_full[w], (uint32_t)(it & 1));
    else named_sync(kWgBar + w, 128);  // the leader saw the previous stores leave the slabs
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      uint8_t* slab = slabs + b * kLwsSlabBytes;
#pragma unroll
      for (int jh = 0; jh < 8; jh += 4) {  // four 8-column groups at a time: their loads first, then the arithmetic
        float2 bb[4];
        __half2 rv[4][2];
#pragma unroll
        for (int jl = 0; jl < 4; ++jl) {
          bb[jl] = __ldg(reinterpret_cast<const float2*>(bias + 64 * b + 8 * (jh + jl) + cq));
          if (p.has_res) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = r0 + 8 * h;
              rv[jl][h] = *reinterpret_cast<const __half2*>(slab + row * 128 + (((uint32_t)(jh + jl) ^ (uint32_t)(row & 7)) << 4) + cq * 2);
            }
          }
        }
#pragma unroll
        for (int jl = 0; jl < 4; ++jl) {
          const int jc = 8 * b + jh + jl;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = r0 + 8 * h;
            uint32_t* cell = reinterpret_cast<uint32_t*>(slab + row * 128 + (((uint32_t)(jh + jl) ^ (uint32_t)(row & 7)) << 4) + cq * 2);
            float a0 = acc[4 * jc + 2 * h] + bb[jl].x, a1 = acc[4 * jc + 2 * h + 1] + bb[jl].y;
            if (p.has_res) {
              const float2 r = __half22float2(rv[jl][h]);
              a0 += r.x;
              a1 += r.y;
            }
            if (p.relu) {
              a0 = fmaxf(a0, 0.f);
              a1 = fmaxf(a1, 0.f);
            }
            *cell = pack_half2(a0, a1);
          }
        }
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> async proxy
    named_sync(kWgBar + w, 128);
    if (leader) {
      for (int s = 0; s < 2; ++s)
        tma_store_5d(&map_out, slabs + s * kLwsSlabBytes, pn * kLwsCols + 64 * s, row0, 0, 0, 0);
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
  }
  if (leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // smem must outlive the stores
}

// FPOSE_LINEAR_WS=0 keeps every linear layer on gemm_tile_kernel's 128 x 128 tile.  Read at every plan, so that one
// process can time and compare both kernels; a captured graph keeps the kernels of its capture.
static bool linear_ws_enabled() {
  const char* e = getenv("FPOSE_LINEAR_WS");
  return !(e && e[0] == '0');
}

// Items per CTA below which a layer keeps the 128 x 128 tile: every CTA loads a 128 KB panel before its first tile,
// which a short range does not amortise (track_one's 400 rows are 28 items on 132 SMs).
constexpr int kLinearWsMinItemsPerCta = 8;

bool linear_ws_takes(const GemmLayer& L) {
  if (L.kind != LK_LINEAR || L.Cin != kLwsK || L.Cout % kLwsCols != 0 || L.out_split != 0 || L.post_add ||
      !linear_ws_enabled())
    return false;
  const int sms = num_sms();
  const int panels = L.Cout / kLwsCols;
  const long long items = (long long)panels * ((L.Win + kLwsRows - 1) / kLwsRows);
  // panels <= CTAs keeps every CTA's range within two panels
  return sms > 0 && panels <= sms && items >= (long long)kLinearWsMinItemsPerCta * sms;
}

int linear_ws_launch(const GemmLayer& L, cudaStream_t stream) {
  const uint64_t E = 2;
  const int M = L.Win;
  LinearWsParams p;
  memset(&p, 0, sizeof(p));
  p.row_tiles = (M + kLwsRows - 1) / kLwsRows;
  p.total = (L.Cout / kLwsCols) * p.row_tiles;
  p.bias = L.bias;
  p.has_res = L.res != nullptr;
  p.relu = L.relu;
  CUtensorMap ma, mw, mo, mr;
  {
    const uint64_t d[2] = {(uint64_t)kLwsK, (uint64_t)M}, s[1] = {(uint64_t)kLwsK * E};
    const uint32_t b[2] = {64, kLwsRows};
    if (int rc = encode_map_f16(&ma, L.in, 2, d, s, b)) return rc;
  }
  {
    const uint64_t d[2] = {(uint64_t)kLwsK, (uint64_t)L.Cout}, s[1] = {(uint64_t)kLwsK * E};
    const uint32_t b[2] = {64, kLwsCols};
    if (int rc = encode_map_f16(&mw, L.w, 2, d, s, b)) return rc;
  }
  // output / residual: [M][ld], one box = 64 rows x 64 channels (5-D, like gemm_tile_kernel's maps)
  auto rows_map = [&](CUtensorMap* m, const void* base, int ld) {
    const uint64_t row = (uint64_t)ld * E;
    const uint64_t d[5] = {(uint64_t)ld, (uint64_t)M, 1, 1, 1}, s[4] = {row, row * M, row * M, row * M};
    const uint32_t b[5] = {64, kLwsRows, 1, 1, 1};
    return encode_map_f16(m, base, 5, d, s, b);
  };
  if (int rc = rows_map(&mo, L.out, L.out_ld)) return rc;
  mr = mo;
  if (L.res) {
    if (int rc = rows_map(&mr, L.res, L.res_ld)) return rc;
  }

  static std::atomic<unsigned long long> attr_mask{0};  // per device: the attribute is device state
  if (!device_bit_test(attr_mask)) {
    FP_CUDA_OK(cudaFuncSetAttribute(linear_ws_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kLwsSmemBytes));
    device_bit_set(attr_mask);
  }
  const int sms = num_sms();
  FP_REQUIRE(sms > 0, "no CUDA device");
  const int grid = p.total < sms ? p.total : sms;
  prof_mark_begin(0, 2.0 * (double)M * L.Cout * kLwsK, stream);
  FP_CUDA_OK(launch_pdl(linear_ws_kernel, dim3(grid), dim3(kLwsThreads), kLwsSmemBytes, stream, 1, ma, mw, mo, mr, p));
  prof_mark_end(stream);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace fp
