// fp_gemm.cu — wgmma / TMA implicit-GEMM tile kernel for every dense contraction on the hot path: the 15
// convolutions of RefineNet / ScoreNetMultiPair's encoders and the linear layers of their attention heads.
//
// Replaces (reference, via torch -> cuDNN / cuBLAS under fp16 autocast):
//   learning/models/network_modules.py:37-50   ConvBNReLU          (conv + folded BN + ReLU)
//   learning/models/network_modules.py:73-111  ResnetBasicBlock    (conv,BN,ReLU,conv,BN,+id,ReLU)
//   learning/models/refine_network.py:80-92    encodeA / encodeAB / pos_embed / linear layers
//   learning/models/score_network.py:60-74     encoderA / encoderAB / att projections
//
// Design (sm_90a, no library GEMM):
//   * D[128 x BN] tiles (BN = 128; 256 for long 3x3 convolutions on tall grids; 64 for 64-channel layers; for the
//     128-channel 3x3 convolutions on tall grids the swapped D^T[128 x 256 pixels] with the weights as M), fp16
//     operands, fp32 accumulators in registers: two
//     consumer warpgroups issue m64nBNk16 wgmmas on 64 rows each; one producer thread feeds a ring of TMA stages
//     (A 16 KB + B BN x 128 B, 128-byte swizzle) through full / empty mbarriers.  Persistent CTAs, one per SM.
//   * The convolution is an *implicit* GEMM: the A tile for k-block (tap, 64-channel chunk) is one 5-D TMA box over
//     the NHWC activation tensor, displaced by the tap offset; out-of-bounds coordinates are zero-filled by the TMA
//     unit, which implements the zero padding.  Stride-2 convolutions use a (2C, W/2, 2, H/2, N) view of the same
//     memory so that every tap is again a dense box; the 7x7/s2 stem has its own kernel (fp_stem.cu).  No im2col
//     buffer is ever materialised.
//   * Epilogue: registers -> +bias/+residual/ReLU/+PE -> fp16 -> 128B-swizzled smem slabs -> TMA tensor store, in
//     64-channel batches; the residual arrives by TMA into the same slabs, as much of it as the slabs hold while the
//     tile's main loop runs.
#include "fp_gemm.cuh"

#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <vector>

#include "fp_common.cuh"
#include "fp_wgmma.cuh"

namespace fp {

static std::atomic<unsigned long long> g_launch_count{0};
static thread_local bool t_capturing = false;
void note_launches(int n) {
  if (!t_capturing) g_launch_count.fetch_add((unsigned long long)n, std::memory_order_relaxed);
}
unsigned long long launch_count() { return g_launch_count.load(std::memory_order_relaxed); }
void set_capturing(bool on) { t_capturing = on; }

std::atomic<bool> g_prof_on{false};
static std::mutex g_prof_mu;

struct ProfRec {
  cudaEvent_t e0, e1;
  double work;
  int kind;
};
static std::vector<ProfRec> g_prof_recs;

void prof_mark_begin(int kind, double work, cudaStream_t stream) {
  if (!g_prof_on) return;
  ProfRec r;
  r.kind = kind;
  r.work = work;
  cudaEventCreate(&r.e0);
  cudaEventCreate(&r.e1);
  cudaEventRecord(r.e0, stream);
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof_recs.push_back(r);
}
void prof_mark_end(cudaStream_t stream) {
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (g_prof_recs.empty()) return;
  cudaEventRecord(g_prof_recs.back().e1, stream);
}
// sums and clears the records of `kind`; synchronises the device
int prof_collect(int kind, double* total_ms, double* total_work, int* launches) {
  FP_CUDA_OK(cudaDeviceSynchronize());
  std::lock_guard<std::mutex> lk(g_prof_mu);
  double ms = 0, work = 0;
  int n = 0;
  std::vector<ProfRec> keep;
  for (auto& r : g_prof_recs) {
    if (r.kind != kind) {
      keep.push_back(r);
      continue;
    }
    float t = 0.f;
    cudaEventElapsedTime(&t, r.e0, r.e1);
    ms += t;
    work += r.work;
    ++n;
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  g_prof_recs.swap(keep);
  *total_ms = ms;
  *total_work = work;
  *launches = n;
  return 0;
}

static thread_local char t_last_error[1024] = "";
void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(t_last_error, sizeof(t_last_error), fmt, ap);
  va_end(ap);
}
const char* get_last_error() { return t_last_error; }

static thread_local int t_pdl_skip = 0;
void pdl_skip_next() { t_pdl_skip = 1; }

bool pdl_enabled() {
  if (t_pdl_skip) {  // consumed by exactly one launch_pdl
    t_pdl_skip = 0;
    return false;
  }
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("FPOSE_PDL");
    on = (e && e[0] == '0') ? 0 : 1;
  }
  return on != 0;
}

struct GemmParams {
  int lg_bw, lg_bh;  // tile rows m -> (nn, ii, jj): jj = m & (bw-1), ii = (m >> lg_bw) & (bh-1)
  int bw, bh, bn;
  int tiles_w, tiles_h, tiles_n, n_tiles_n, total_tiles;
  // Packing of the last, partial image group (conv3, non-swapped tiles): tiles_n counts the full groups only, and
  // every m-tile after them holds up to `pack` spatial blocks of the last group's n_img % bn images, block q at tile
  // rows [q pack_rows, (q + 1) pack_rows).  pack = 0: no packing, the last group is one zero-filled box per block.
  int pack, pack_rows;
  int num_kb, chunks_per_tap;
  int dim_w, dim_h, dim_n;
  short tap_off[9][5];
  int Ho, Wo, n_img, Cout;
  const float* bias;
  int has_res;
  int odim_h, odim_n;  // which coordinate of the output / residual maps receives the tile's row / image
  int out_split;
  const float* post_add;
  int relu;
  double alg_flops;  // 2 * M * Cout * K_real of this launch (host-side bookkeeping only)
};

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kABytes = kBlockM * kBlockK * 2;  // 16 KB
constexpr int kTileThreads = 384;               // warpgroup 0: TMA producer; warpgroups 1, 2: wgmma + epilogue
constexpr int kSlabBytes = kBlockM * 64 * 2;    // 16 KB: one output slab (128 pixels x 64 channels, 128B-swizzled)
constexpr int kSmemOptIn = 232448;              // 227 KB opt-in shared memory per block

// BN = output channels per tile (64, 128 or 256).  Each consumer warpgroup owns 64 of the tile's 128 pixel rows and
// keeps its 64 x BN fp32 accumulator in registers (BN / 2 per thread).
//
// The epilogue converts the tile in 64-channel batches, one staging slab each.  The 64- and 128-wide tiles have a
// slab per batch and store them all at the end.  The 256-wide tile has two slabs (a stage is 48 KB there, and with
// two slabs four stages fit where four slabs leave three) and stores each batch as its own pass, alternating between
// the slabs, so that one slab's store and the next batch's residual load run while the other slab is converted.
//
// kSwap (BN = 128): the operands trade places, D^T[128 channels x 256 pixels] = W[128 x K] * X^T[K x 256].  The
// 16 KB M slot of a stage holds the tile's 128 weight rows and the N slot 256 pixels (a 5-D box of four images), so
// each consumer warpgroup owns 64 channels over all 256 pixels and issues the m64n256k16 wgmmas of the 256-wide tile.
// Its epilogue moves the transposed fragment through the slabs with ldmatrix / stmatrix .trans: four slabs, one per
// (128-pixel half, 64-channel half), stored together at the end of the tile like the 64- and 128-wide tiles.
constexpr int kWideSlabs = 2;
constexpr int kWideProducerRegs = 40;   // setmaxnreg of the 256-wide tiles: producer warpgroup ...
constexpr int kWideConsumerRegs = 232;  // ... and the two consumer warpgroups; 128 x 40 + 256 x 232 <= 384 x 168
template <int BN, bool kSwap = false>
struct TileCfg {
  static constexpr int kRows = kSwap ? 2 * kBlockM : kBlockM;  // output pixels (or linear rows) per tile
  static constexpr int kN = kSwap ? kRows : BN;                 // wgmma N: pixels with kSwap, else channels
  static constexpr int kBBytes = kN * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBatches = (kRows / kBlockM) * (BN / 64);  // 128-pixel x 64-channel epilogue batches
  static constexpr bool kAlternate = !kSwap && BN > 128;           // one pass per batch, through alternating slabs
  static constexpr int kSlabs = kAlternate ? kWideSlabs : kBatches;  // staging slabs
  static constexpr int kStagingBytes = kSlabs * kSlabBytes;
  static constexpr int kRing = kSmemOptIn - kStagingBytes - 1024 /*align slack*/ - 256 /*barriers*/;
  static constexpr int kStages = (kRing / kStageBytes) > 8 ? 8 : (kRing / kStageBytes);
  static constexpr int kSmemBytes = kStages * kStageBytes + kStagingBytes + 1024 + 256;
  static_assert(kSmemBytes <= kSmemOptIn, "tile configuration exceeds the 227 KB opt-in shared memory");
  static_assert((2 * kStages + kSlabs) * 8 <= 256, "the mbarriers must fit their 256 bytes");
  static_assert(kBatches % kSlabs == 0, "every slab must take the same number of batches per tile");
};

// Persistent, warp-specialised: thread 0 streams (A, B) k-blocks through a ring of TMA stages; the two consumer
// warpgroups issue m64nBNk16 wgmmas from it, then run the epilogue (+bias, +residual, ReLU, +pos.emb. -> fp16 ->
// 128B-swizzled slabs -> one TMA tensor store per 64-channel slab).  The producer runs ahead into the next tile while
// the consumers drain this one.  The 256-wide tile moves registers from the producer warpgroup to the consumers
// (128 accumulators per thread do not fit the 168 a 384-thread CTA gets), and so does the swapped tile.
//
// Packed tiles (p.pack > 0) read, store and take the residual of each spatial block as its own box of the last
// group's images (the *_pk maps, whose image box is n_img % bn), at the block's rows of the A slot and of every
// slab; tile rows that no block fills are computed but never stored.
template <int BN, bool kSwap = false>
__global__ void __launch_bounds__(kTileThreads, 1)
    gemm_tile_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                     const __grid_constant__ CUtensorMap map_out, const __grid_constant__ CUtensorMap map_res,
                     const __grid_constant__ CUtensorMap map_a_pk, const __grid_constant__ CUtensorMap map_out_pk,
                     const __grid_constant__ CUtensorMap map_res_pk, const __grid_constant__ GemmParams p) {
  using Cfg = TileCfg<BN, kSwap>;
  constexpr int S = Cfg::kStages;
  constexpr int NSLAB = Cfg::kSlabs;
  constexpr int NB = Cfg::kBatches;
  constexpr bool kAlt = Cfg::kAlternate;
  extern __shared__ uint8_t smem_raw[];
  // offset from the __shared__ array itself, so that the compiler sees every access below as shared memory
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* staging = smem + S * Cfg::kStageBytes;  // [NSLAB][kSlabBytes], 1024-aligned
  uint64_t* bars = reinterpret_cast<uint64_t*>(staging + Cfg::kStagingBytes);
  uint64_t* full = bars;          // [S]
  uint64_t* empty = bars + S;     // [S]
  uint64_t* res_full = bars + 2 * S;  // [NSLAB] with kAlt (one per slab), else [1] (all slabs)

  const int full_m_tiles = p.tiles_w * p.tiles_h * p.tiles_n;
  const int total = p.total_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
    tma_prefetch_desc(&map_out);
    if (p.has_res) tma_prefetch_desc(&map_res);
    if (p.pack) {
      tma_prefetch_desc(&map_a_pk);
      tma_prefetch_desc(&map_out_pk);
      if (p.has_res) tma_prefetch_desc(&map_res_pk);
    }
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 256);
    }
    for (int s = 0; s < (kAlt ? NSLAB : 1); ++s) mbar_init(&res_full[s], 1);
    mbar_fence_init();
  }
  __syncthreads();
  pdl_trigger();
  pdl_wait();  // everything above overlapped the previous kernel's tail; activations are touched only from here on

  // nsub = 0: a full tile at block (tw, th) of image group tn.  Otherwise a packed tile (m-tiles past the full
  // groups): nsub blocks of the last group tn, from (tw, th) on in row-major block order.
  auto decode = [&](int t, int& n_tile, int& tw, int& th, int& tn, int& nsub) {
    n_tile = t % p.n_tiles_n;
    const int m_tile = t / p.n_tiles_n;
    if (!kSwap && m_tile >= full_m_tiles) {
      const int blk = (m_tile - full_m_tiles) * p.pack;
      nsub = min(p.pack, p.tiles_w * p.tiles_h - blk);
      tw = blk % p.tiles_w;
      th = blk / p.tiles_w;
      tn = p.tiles_n;
      return;
    }
    nsub = 0;
    tw = m_tile % p.tiles_w;
    th = (m_tile / p.tiles_w) % p.tiles_h;
    tn = m_tile / (p.tiles_w * p.tiles_h);
  };

  if (threadIdx.x < 128) {
    // ------------------------------------------------------------------ TMA producer
    if constexpr (Cfg::kN > 128) regs_release<kWideProducerRegs>();  // all four warps, before three of them leave
    if (threadIdx.x == 0) {
      int stage = 0, phase = 0;
      for (int t = blockIdx.x; t < total; t += gridDim.x) {
        int n_tile, tw, th, tn, nsub;
        decode(t, n_tile, tw, th, tn, nsub);
        int base[5] = {0, 0, 0, 0, 0};
        base[p.dim_w] += tw * p.bw;
        if (p.dim_h >= 0) base[p.dim_h] += th * p.bh;
        if (p.dim_n >= 0) base[p.dim_n] += tn * p.bn;
        int tap = 0, chunk = 0;
        for (int kb = 0; kb < p.num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          if (kSwap || nsub == 0) {
            mbar_expect_tx(&full[stage], Cfg::kStageBytes);
            // kSwap: the pixels are the N operand and the weights the M operand
            tma_load_5d(&map_a, &full[stage], kSwap ? sa + kABytes : sa, base[0] + p.tap_off[tap][0] + chunk * kBlockK,
                        base[1] + p.tap_off[tap][1], base[2] + p.tap_off[tap][2], base[3] + p.tap_off[tap][3],
                        base[4] + p.tap_off[tap][4]);
          } else {
            // one box of the last group's images per block, into the block's rows of the A slot
            mbar_expect_tx(&full[stage], Cfg::kBBytes + nsub * p.pack_rows * 128);
            for (int q = 0, x = tw, y = th; q < nsub; ++q) {
              // block q's displacement from the tile's first block, along w (dimension 1 of both conv3 views) and h
              const int dw = (x - tw) * p.bw, dh = (y - th) * p.bh;
              tma_load_5d(&map_a_pk, &full[stage], sa + q * p.pack_rows * 128,
                          base[0] + p.tap_off[tap][0] + chunk * kBlockK, base[1] + p.tap_off[tap][1] + dw,
                          base[2] + p.tap_off[tap][2] + (p.dim_h == 2 ? dh : 0),
                          base[3] + p.tap_off[tap][3] + (p.dim_h == 3 ? dh : 0), base[4] + p.tap_off[tap][4]);
              if (++x == p.tiles_w) {
                x = 0;
                ++y;
              }
            }
          }
          tma_load_2d(&map_b, &full[stage], kSwap ? sa : sa + kABytes, kb * kBlockK, n_tile * BN);
          if (++chunk == p.chunks_per_tap) {
            chunk = 0;
            ++tap;
          }
          if (++stage == S) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers (warpgroups 1, 2)
  if constexpr (Cfg::kN > 128) regs_acquire<kWideConsumerRegs>();
  const int ct = threadIdx.x - 128;
  const int cw = ct >> 7;  // rows [64 cw, 64 cw + 64) of the tile (kSwap: channels, else pixels)
  const int lane = threadIdx.x & 31;
  const int r0 = 64 * cw + 16 * ((ct >> 5) & 3) + (lane >> 2);  // this thread's rows: r0 and r0 + 8
  const int cq = 2 * (lane & 3);                                  // and columns 8 j + cq, 8 j + cq + 1
  const bool leader = (ct == 0);
  // slab q of the tile: kSwap: pixel half q >> 1 (images 2 (q >> 1) and 2 (q >> 1) + 1 of the four), channel half q & 1;
  // otherwise channels [64 q, 64 q + 64).  kSwap runs 3x3 convolutions only, whose image coordinate is 3.
  auto slab_ch = [](int q) { return kSwap ? 64 * (q & 1) : 64 * q; };
  auto slab_img = [](int q) { return kSwap ? 2 * (q >> 1) : 0; };
  float acc[Cfg::kN / 2];
#pragma unroll
  for (int i = 0; i < Cfg::kN / 2; ++i) acc[i] = 0.f;
  int stage = 0, phase = 0, it = 0;
  for (int t = blockIdx.x; t < total; t += gridDim.x, ++it) {
    int n_tile, tw, th, tn, nsub;
    decode(t, n_tile, tw, th, tn, nsub);
    const int n0 = tn * p.bn;
    int n_o0 = n0, coff = 0;
    if (p.out_split > 0) {
      n_o0 = n0 % p.out_split;
      coff = (n0 / p.out_split) * p.Cout;
    }
    // output / residual box coordinates (dim 0 = channel is added per slab)
    int oc[5] = {0, 0, 0, 0, 0}, rc[5] = {0, 0, 0, 0, 0};
    oc[1] = rc[1] = tw * p.bw;
    if (p.odim_h >= 0) oc[p.odim_h] = rc[p.odim_h] = th * p.bh;
    if (p.odim_n >= 0) {
      oc[p.odim_n] = n_o0;
      rc[p.odim_n] = n0;
    }
    // A packed tile's output / residual boxes: f(row byte offset in a slab, x, y) for each of its blocks, whose
    // images are those of the last group (the *_pk maps; conv3 only, so the coordinates are (c, w, h, n)).
    auto for_blocks = [&](auto&& f) {
      for (int q = 0, x = tw, y = th; q < nsub; ++q) {
        f((uint32_t)(q * p.pack_rows * 128), x * p.bw, y * p.bh);
        if (++x == p.tiles_w) {
          x = 0;
          ++y;
        }
      }
    };
    // the residual of 64 channels from `ch` (kSwap: and images from `img` on) into slab `dst`, on barrier rb
    auto load_res = [&](uint64_t* rb, uint8_t* dst, int ch, int img) {
      if (nsub == 0)
        tma_load_5d(&map_res, rb, dst, ch, rc[1], rc[2], rc[3] + img, rc[4]);
      else
        for_blocks([&](uint32_t off, int x, int y) { tma_load_5d(&map_res_pk, rb, dst + off, ch, x, y, n0, 0); });
    };
    auto slab_bytes = [&]() -> uint32_t { return nsub ? nsub * p.pack_rows * 128 : kSlabBytes; };  // a slab's boxes
    // ---- main loop: one wgmma batch (4 x K = 16) per k-block; a stage is released once the NEXT batch is issued
    int prev = -1;
    for (int kb = 0; kb < p.num_kb; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * Cfg::kStageBytes);
      const uint64_t da = gmma_desc_sw128(sa + (uint32_t)cw * 8192u);
      const uint64_t db = gmma_desc_sw128(sa + kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / 16; ++k)
        Wgmma<Cfg::kN>::ss(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      if (kb == 0 && leader) {
        // The previous tile's stores leave the staging slabs while the first wgmmas run; only the leader waits for
        // that, and the epilogue's barrier (or its residual wait) tells the other threads.  Then the residual of the
        // tile's first NSLAB batches goes into the slabs and arrives while the main loop runs (kAlt: one barrier per
        // slab, else one for all).
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        if (p.has_res) {
          for (int s = 0; s < NSLAB; ++s) {
            uint64_t* rb = &res_full[kAlt ? s : 0];
            if (kAlt || s == 0) mbar_expect_tx(rb, (kAlt ? 1 : NSLAB) * slab_bytes());
            load_res(rb, staging + s * kSlabBytes, n_tile * BN + slab_ch(s), slab_img(s));
          }
        }
      }
      if (prev >= 0) {
        wgmma_wait<1>();
        mbar_arrive(&empty[prev]);
      }
      prev = stage;
      if (++stage == S) {
        stage = 0;
        phase ^= 1;
      }
    }
    if constexpr (kSwap) {
      // ---- epilogue of the swapped tile: this thread holds channels r0 and r0 + 8 for pixels 8 j + cq (+1), j < 32.
      // The same fp32 arithmetic as below (bias, residual, ReLU, one fp16 rounding) on each element.  An 8 x 8 block
      // (column group j, channel half h) is one ldmatrix / stmatrix .trans matrix, whose memory rows are the block's
      // eight pixels, each 16 bytes of eight consecutive channels: the slabs' swizzle unit.
      const float bc[2] = {__ldg(p.bias + n_tile * BN + r0), __ldg(p.bias + n_tile * BN + r0 + 8)};
      wgmma_wait<0>();
      fence_regs(acc);
      if (prev >= 0) mbar_arrive(&empty[prev]);
      // the slabs are free: the residual arrived after the leader saw the previous stores read out, or the barrier
      // tells every thread that the leader did
      if (p.has_res) mbar_wait(&res_full[0], (uint32_t)(it & 1));
      else asm volatile("bar.sync 1, 256;" ::: "memory");
      // lane 8 i + r addresses row r of matrix i = (column group jl = i >> 1 of a pair, channel half h = i & 1): the
      // pair's pixel 8 jl + r, 16-byte chunk 2 w + h of the warpgroup's 64 channels, swizzled by the pixel's row & 7
      const int mi = lane >> 3, mr = lane & 7;
      const uint32_t lane_off =
          (uint32_t)(8 * (mi >> 1) + mr) * 128u + ((uint32_t)((2 * ((ct >> 5) & 3) + (mi & 1)) ^ mr) << 4);
#pragma unroll
      for (int ph = 0; ph < 2; ++ph) {
        const uint32_t slab = smem_u32(staging + (2 * ph + cw) * kSlabBytes) + lane_off;
        uint32_t rv[8][4];
        if (p.has_res) {
#pragma unroll
          for (int g = 0; g < 8; ++g) ldsm_x4_trans(slab + g * 2048u, rv[g]);
        }
#pragma unroll
        for (int g = 0; g < 8; ++g) {  // column groups j = 16 ph + 2 g, 16 ph + 2 g + 1: pixels 16 g .. 16 g + 15
          uint32_t o[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int j = 16 * ph + 2 * g + (i >> 1), h = i & 1;
            float a0 = acc[4 * j + 2 * h] + bc[h], a1 = acc[4 * j + 2 * h + 1] + bc[h];
            if (p.has_res) {
              const float2 r = __half22float2(*reinterpret_cast<const __half2*>(&rv[g][i]));
              a0 += r.x;
              a1 += r.y;
            }
            if (p.relu) {
              a0 = fmaxf(a0, 0.f);
              a1 = fmaxf(a1, 0.f);
            }
            o[i] = pack_half2(a0, a1);
          }
          stsm_x4_trans(slab + g * 2048u, o);
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> async proxy
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (leader) {
        for (int q = 0; q < NSLAB; ++q)
          tma_store_5d(&map_out, staging + q * kSlabBytes, coff + n_tile * BN + slab_ch(q), oc[1], oc[2],
                       oc[3] + slab_img(q), oc[4]);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
      continue;
    }
    // ---- epilogue: 64-channel batches b, channels [64 b, 64 b + 64) of the tile, each converted into one slab.
    // Every load of a batch (bias, residual, positional embedding) is issued before the batch's first conversion,
    // so their latencies overlap instead of adding up element by element.
    const float* bias = p.bias + n_tile * BN;
    const float* pap[2] = {nullptr, nullptr};  // positional-embedding rows of this thread's two pixels
    if (p.post_add) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        const int jj = row & (p.bw - 1), ii = (row >> p.lg_bw) & (p.bh - 1);
        int bx = tw, by = th;  // the row's spatial block; in a packed tile, that of its block q (rows no block fills
        if (nsub) {            // take the last block's)
          const int blk = th * p.tiles_w + tw + min(row / p.pack_rows, nsub - 1);
          bx = blk % p.tiles_w;
          by = blk / p.tiles_w;
        }
        const int i = by * p.bh + ii, j = min(bx * p.bw + jj, p.Wo - 1);
        pap[h] = p.post_add + (size_t)(i * p.Wo + j) * p.Cout + n_tile * BN;
      }
    }
    // positional embedding of one batch in registers: batch 0's issued while the last wgmma batch drains, batch
    // b + 1's as soon as batch b is converted (for the 256-wide tile, ahead of that pass's barrier and store)
    float2 pe[8][2];
    auto load_pe = [&](int b) {
#pragma unroll
      for (int jl = 0; jl < 8; ++jl)
#pragma unroll
        for (int h = 0; h < 2; ++h) pe[jl][h] = __ldg(reinterpret_cast<const float2*>(pap[h] + 64 * b + 8 * jl + cq));
    };
    if (p.post_add) load_pe(0);
    wgmma_wait<0>();
    fence_regs(acc);
    if (prev >= 0) mbar_arrive(&empty[prev]);
    // Without a residual nothing else tells the threads that the leader saw the previous stores leave the slabs
    // (with one, batch 0's residual wait does: it arrived after that).
    if (!p.has_res) asm volatile("bar.sync 1, 256;" ::: "memory");

#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const int s = kAlt ? (b & 1) : b;
      uint8_t* slab = staging + s * kSlabBytes;
      if (kAlt && p.has_res && b > 0 && b + 1 < NB) {
        // The other slab's last store (batch b - 1's) has been read out: batch b + 1's residual goes into it now,
        // and arrives while this batch is converted.  Batches 0 and 1 were fetched during the main loop.
        if (leader) {
          asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
          uint64_t* rb = &res_full[(b + 1) & 1];
          mbar_expect_tx(rb, slab_bytes());
          load_res(rb, staging + ((b + 1) & 1) * kSlabBytes, n_tile * BN + (b + 1) * 64, 0);
        }
      }
      // Phase of the barrier that batch b waits on, in the CTA's it-th tile: it completes NB / NSLAB times per tile
      // (kAlt: res_full[b & 1] twice, for batches b & 1 and (b & 1) + 2; otherwise res_full[0] once, for all slabs),
      // so this is its completion it * (NB / NSLAB) + b / NSLAB.  Every thread waits each completion before the
      // leader can start the next fill of the same barrier.
      if (p.has_res && (kAlt || b == 0))
        mbar_wait(&res_full[kAlt ? s : 0], (uint32_t)((it * (NB / NSLAB) + b / NSLAB) & 1));
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
          const int j = 8 * b + jh + jl;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = r0 + 8 * h;
            uint32_t* cell = reinterpret_cast<uint32_t*>(slab + row * 128 + (((uint32_t)(jh + jl) ^ (uint32_t)(row & 7)) << 4) + cq * 2);
            float a0 = acc[4 * j + 2 * h] + bb[jl].x, a1 = acc[4 * j + 2 * h + 1] + bb[jl].y;
            if (p.has_res) {
              const float2 r = __half22float2(rv[jl][h]);
              a0 += r.x;
              a1 += r.y;
            }
            if (p.relu) {
              a0 = fmaxf(a0, 0.f);
              a1 = fmaxf(a1, 0.f);
            }
            if (p.post_add) {
              a0 += pe[jh + jl][h].x;
              a1 += pe[jh + jl][h].y;
            }
            *cell = pack_half2(a0, a1);
          }
        }
      }
      if (p.post_add && b + 1 < NB) load_pe(b + 1);
      if (kAlt || b == NB - 1) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> async proxy
        // kAlt: the other slab's last store has been read out, so the next batch may convert into it
        if (kAlt && leader) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (leader) {
          for (int q = kAlt ? s : 0; q < (kAlt ? s + 1 : NSLAB); ++q) {
            const int ch = coff + n_tile * BN + (kAlt ? 64 * b : 64 * q);
            if (nsub == 0)
              tma_store_5d(&map_out, staging + q * kSlabBytes, ch, oc[1], oc[2], oc[3], oc[4]);
            else
              for_blocks([&](uint32_t off, int x, int y) {
                tma_store_5d(&map_out_pk, staging + q * kSlabBytes + off, ch, x, y, n_o0, 0);
              });
          }
          asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
      }
    }
  }
  if (leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // smem must outlive the stores
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static int g_num_sms = 0;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static int encode_map(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                      const uint64_t* strides_bytes /*rank-1*/, const uint32_t* box, bool swizzle128 = true) {
  EncodeTiledFn fn = get_encode_fn();
  FP_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
  }
  for (int i = 0; i < rank - 1; ++i) gstr[i] = strides_bytes[i];
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr,
                  bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  FP_REQUIRE(r == CUDA_SUCCESS,
             "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu %llu] box [%u %u %u %u %u]",
             (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
             (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
             (unsigned long long)(rank > 4 ? dims[4] : 0), box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0,
             rank > 3 ? box[3] : 0, rank > 4 ? box[4] : 0);
  return 0;
}

int encode_map_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box) {
  return encode_map(map, base, rank, dims, strides_bytes, box);
}
int encode_map_f16_linear(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                          const uint64_t* strides_bytes, const uint32_t* box) {
  return encode_map(map, base, rank, dims, strides_bytes, box, false);
}
int num_sms() {
  if (g_num_sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
  }
  return g_num_sms;
}

static int ilog2(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}

template <int BN, bool kSwap = false>
static int launch_bn(const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mo, const CUtensorMap& mr,
                     const CUtensorMap& ma_pk, const CUtensorMap& mo_pk, const CUtensorMap& mr_pk, const GemmParams& p,
                     cudaStream_t stream) {
  using Cfg = TileCfg<BN, kSwap>;
  static std::atomic<unsigned long long> attr_mask{0};  // per device: the attribute is device state
  if (!device_bit_test(attr_mask)) {
    FP_CUDA_OK(cudaFuncSetAttribute(gemm_tile_kernel<BN, kSwap>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    Cfg::kSmemBytes));
    device_bit_set(attr_mask);
  }
  const int sms = num_sms();
  FP_REQUIRE(sms > 0, "no CUDA device");
  const int grid = p.total_tiles < sms ? p.total_tiles : sms;
  prof_mark_begin(0, p.alg_flops, stream);
  FP_CUDA_OK(launch_pdl(gemm_tile_kernel<BN, kSwap>, dim3(grid), dim3(kTileThreads), Cfg::kSmemBytes, stream, 1, ma, mb,
                        mo, mr, ma_pk, mo_pk, mr_pk, p));
  prof_mark_end(stream);
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

int stem_conv_launch(const GemmLayer& L, cudaStream_t stream);  // fp_stem.cu
bool linear_ws_takes(const GemmLayer& L);                        // fp_linear.cu
int linear_ws_launch(const GemmLayer& L, cudaStream_t stream);

// FPOSE_SWAP_TILE=0 keeps the 128-channel convolutions on the 128 x 128 tile.  Read at every plan, so that one process
// can time and compare both tiles; a captured graph keeps the tiles of its capture.
static bool swap_tile_enabled() {
  const char* e = getenv("FPOSE_SWAP_TILE");
  return !(e && e[0] == '0');
}

// Plans the layer and launches it, or, with `tile_n` or `tile_m`, only reports the tile the launch would use: its
// output channels and its output pixels (linear rows).
static int gemm_layer_plan(const GemmLayer& L, cudaStream_t stream, int* tile_n, int* tile_m) {
  if (L.kind == LK_CONV7_S2) {
    if (tile_n || tile_m) {
      if (tile_n) *tile_n = 64;  // the stem kernel's 128-pixel x 64-channel tile
      if (tile_m) *tile_m = 128;
      return 0;
    }
    return stem_conv_launch(L, stream);
  }
  GemmParams p;
  memset(&p, 0, sizeof(p));
  CUtensorMap ma, mb;
  const uint64_t E = 2;  // bytes per fp16
  int Ho, Wo, taps, ktot;
  int BN;
  uint64_t dims[5], str[4];
  uint32_t box[5];

  switch (L.kind) {
    case LK_LINEAR: {
      FP_REQUIRE(L.Cin % 64 == 0, "LINEAR: K=%d not a multiple of 64", L.Cin);
      Ho = 1;
      Wo = L.Win;
      taps = 1;
      p.chunks_per_tap = L.Cin / 64;
      p.bw = 128; p.bh = 1; p.bn = 1;
      p.dim_w = 1; p.dim_h = -1; p.dim_n = -1;
      dims[0] = L.Cin; dims[1] = L.Win; dims[2] = 1; dims[3] = 1; dims[4] = 1;
      str[0] = L.Cin * E; str[1] = str[0] * L.Win; str[2] = str[1]; str[3] = str[1];
      box[0] = 64; box[1] = 128; box[2] = 1; box[3] = 1; box[4] = 1;
      p.tiles_w = (L.Win + 127) / 128; p.tiles_h = 1; p.tiles_n = 1;
      break;
    }
    case LK_CONV3_S1: {
      FP_REQUIRE(L.Cin % 64 == 0, "CONV3_S1: Cin=%d not a multiple of 64", L.Cin);
      Ho = L.Hin; Wo = L.Win;
      taps = 9;
      p.chunks_per_tap = L.Cin / 64;
      if (Wo % 8 == 0 && Ho % 8 == 0) { p.bw = 8; p.bh = 8; p.bn = 2; }
      else if (Wo % 4 == 0 && Ho % 4 == 0) { p.bw = 4; p.bh = 4; p.bn = 8; }
      else FP_REQUIRE(false, "CONV3_S1: unsupported spatial size %dx%d", Ho, Wo);
      // one TMA box (64 ch, bw, bh, bn images) per (tap, 64-channel chunk), displaced by the tap offset; the zero
      // padding is the TMA unit's out-of-bounds fill
      const uint64_t sw_ = (uint64_t)L.Cin * E, sh_ = sw_ * L.Win, sn_ = sh_ * L.Hin;
      p.dim_w = 1; p.dim_h = 2; p.dim_n = 3;
      dims[0] = L.Cin; dims[1] = L.Win; dims[2] = L.Hin; dims[3] = L.n_img; dims[4] = 1;
      str[0] = sw_; str[1] = sh_; str[2] = sn_; str[3] = sn_ * L.n_img;
      box[0] = 64; box[1] = p.bw; box[2] = p.bh; box[3] = p.bn; box[4] = 1;
      for (int r = 0; r < 3; ++r)
        for (int s = 0; s < 3; ++s) {
          p.tap_off[r * 3 + s][1] = (short)(s - 1);
          p.tap_off[r * 3 + s][2] = (short)(r - 1);
        }
      p.tiles_w = Wo / p.bw; p.tiles_h = Ho / p.bh; p.tiles_n = (L.n_img + p.bn - 1) / p.bn;
      break;
    }
    case LK_CONV3_S2: {
      FP_REQUIRE(L.Cin % 64 == 0, "CONV3_S2: Cin=%d not a multiple of 64", L.Cin);
      FP_REQUIRE(L.Hin % 2 == 0 && L.Win % 2 == 0, "CONV3_S2: odd input size");
      Ho = L.Hin / 2; Wo = L.Win / 2;
      taps = 9;
      p.chunks_per_tap = L.Cin / 64;
      if (Wo % 8 == 0 && Ho % 8 == 0) { p.bw = 8; p.bh = 8; p.bn = 2; }
      else if (Wo % 4 == 0 && Ho % 4 == 0) { p.bw = 4; p.bh = 4; p.bn = 8; }
      else FP_REQUIRE(false, "CONV3_S2: unsupported output size %dx%d", Ho, Wo);
      p.dim_w = 1; p.dim_h = 3; p.dim_n = 4;
      // view (N, H, W, C) as (N, H/2, 2, W/2, [2, C]): every (tap, chunk) is a dense box
      dims[0] = 2 * L.Cin; dims[1] = Wo; dims[2] = 2; dims[3] = Ho; dims[4] = L.n_img;
      str[0] = 2 * L.Cin * E; str[1] = (uint64_t)L.Win * L.Cin * E; str[2] = 2 * str[1];
      str[3] = (uint64_t)L.Hin * L.Win * L.Cin * E;
      box[0] = 64; box[1] = p.bw; box[2] = 1; box[3] = p.bh; box[4] = p.bn;
      for (int r = 0; r < 3; ++r)
        for (int s = 0; s < 3; ++s) {
          const int t = r * 3 + s;
          // input row 2i + r - 1: r=0 -> (i-1, phase 1), r=1 -> (i, 0), r=2 -> (i, 1)
          p.tap_off[t][0] = (short)((s == 1 ? 0 : 1) * L.Cin);
          p.tap_off[t][1] = (short)(s == 0 ? -1 : 0);
          p.tap_off[t][2] = (short)(r == 1 ? 0 : 1);
          p.tap_off[t][3] = (short)(r == 0 ? -1 : 0);
        }
      p.tiles_w = Wo / p.bw; p.tiles_h = Ho / p.bh; p.tiles_n = (L.n_img + p.bn - 1) / p.bn;
      break;
    }
    default:
      FP_REQUIRE(false, "unknown layer kind %d", L.kind);
  }
  ktot = taps * L.Cin;
  p.num_kb = ktot / 64;
  p.lg_bw = ilog2(p.bw);
  p.lg_bh = ilog2(p.bh);

  // 128 channels per tile: two 64 x 128 register accumulators per CTA (64 fp32 registers per thread).  256 channels
  // when the 256-wide grid still fills kWideMinWaves waves of persistent CTAs and the k-loop is long: the wide tile
  // reads half the weight bytes per FLOP, but it halves the CTA count, its last, partial wave costs relatively more
  // on a short grid, and its two-pass epilogue is not hidden behind a short k-loop.  Measured per layer on an H100
  // SXM at 700 W against the 128-wide tile, the 3x3 convolutions (K = 2304 / 4608) are +7 to +13 % at 9 wide waves,
  // +16 to +24 % at 12 to 24 (252 hypotheses), even at 6 and about 10 % slower at 3 (a 32-hypothesis shard;
  // track_one's single image is under one wave); the K = 512 linear layers (8 k-blocks) were no faster at any height.
  //
  // A 3x3 convolution with Cout = 128 cannot take the wide tile; it takes the swapped tile (256 pixels of four 8 x 8
  // blocks, the weights as the M operand) under the same rule on its 256-pixel grid.  Measured at 504 images (H100 SXM,
  // 700 W) against the 128 x 128 tile: 128 @ 40 (18 k-blocks) +7 to +10 % without a residual and -2 to +3 % with one;
  // the stride-2 64 -> 128 layer (9 k-blocks) no faster.
  constexpr int kWideMinWaves = 8;
  constexpr int kWideMinKBlocks = 16;
  bool swap = false;
  if (L.Cout == 128 && L.kind != LK_LINEAR && p.bw == 8 && p.num_kb >= kWideMinKBlocks && !L.post_add &&
      L.out_split % 4 == 0 && swap_tile_enabled()) {
    const int sms = num_sms();
    FP_REQUIRE(sms > 0, "no CUDA device");
    swap = (long long)p.tiles_w * p.tiles_h * ((L.n_img + 3) / 4) >= (long long)kWideMinWaves * sms;
  }
  if (swap) {
    p.bn = 4;
    box[p.dim_n] = 4;
    p.tiles_n = (L.n_img + 3) / 4;
  }
  // The last image group holds r = n_img % bn images.  As one box per spatial block it would leave bn - r of the
  // tile's bn images to the TMA unit's zero fill; instead, k = bn / r >= 2 of its blocks share a tile, each as a box
  // of r images at rows q * bw * bh * r (a multiple of the 1024-byte swizzle atom).  Every output element keeps its
  // k-order and epilogue arithmetic.  At 252 hypotheses the 20 x 20 layers' 4 x 4 x 8 tiles go from 25 x 32 to
  // 25 x 31 + 13 m-tiles: 1576 instead of 1600 tiles of 256 channels, 12 rounds of 132 persistent CTAs instead of 13.
  // A grid of one round or less gains nothing (its time is one tile's): there, packing would only put the same work
  // on fewer SMs (packing track_one's layers, one to five images, took its p50 from 1.2-1.3 ms to 1.5 ms on an H100
  // SXM at 700 W).  The tile width is chosen from the packed count; packing itself is decided below, against the SM
  // count, after the tile queries have returned.
  const int last_n = L.n_img % p.bn;
  const int pack = (!swap && last_n > 0) ? p.bn / last_n : 0;
  const int blocks = p.tiles_w * p.tiles_h;
  int m_tiles = pack >= 2 ? blocks * (L.n_img / p.bn) + (blocks + pack - 1) / pack : blocks * p.tiles_n;
  if (swap) BN = 128;
  else if (L.Cout % 256 == 0 && p.num_kb >= kWideMinKBlocks) {
    const int sms = num_sms();
    FP_REQUIRE(sms > 0, "no CUDA device");
    BN = (long long)m_tiles * (L.Cout / 256) >= (long long)kWideMinWaves * sms ? 256 : 128;
  } else if (L.Cout % 128 == 0) BN = 128;
  else if (L.Cout % 64 == 0) BN = 64;
  else FP_REQUIRE(false, "Cout=%d must be a multiple of 64", L.Cout);
  p.n_tiles_n = L.Cout / BN;
  p.Ho = Ho; p.Wo = Wo; p.n_img = L.n_img; p.Cout = L.Cout;
  p.bias = L.bias;
  p.has_res = L.res != nullptr;
  p.out_split = L.out_split;
  p.post_add = L.post_add;
  p.relu = L.relu;
  {
    const double k_real = (double)taps * L.Cin;
    p.alg_flops = 2.0 * (double)L.n_img * Ho * Wo * L.Cout * k_real;
  }
  FP_REQUIRE(L.out_ld % 8 == 0 && (!L.res || L.res_ld % 8 == 0), "out_ld / res_ld must be multiples of 8");
  FP_REQUIRE(L.out_split == 0 || L.out_split % p.bn == 0,
             "out_split=%d must be a multiple of the tile's image count %d (pad the A/B batch boundary)", L.out_split,
             p.bn);
  // the K = 512 linear layers on tall row counts: 64-row x 128-channel tiles of the weight-stationary kernel
  const bool linear_ws = linear_ws_takes(L);
  if (tile_n || tile_m) {
    if (tile_n) *tile_n = BN;
    if (tile_m) *tile_m = swap ? 256 : linear_ws ? 64 : 128;
    return 0;
  }
  if (pack >= 2) {
    const int sms = num_sms();
    FP_REQUIRE(sms > 0, "no CUDA device");
    if ((long long)blocks * p.tiles_n * p.n_tiles_n > sms) {
      p.pack = pack;
      p.pack_rows = p.bw * p.bh * last_n;
      p.tiles_n = L.n_img / p.bn;
    } else {
      m_tiles = blocks * p.tiles_n;
    }
  }
  p.total_tiles = m_tiles * p.n_tiles_n;
  if (p.total_tiles == 0) return 0;
  if (linear_ws) return linear_ws_launch(L, stream);

  int rc = encode_map(&ma, L.in, 5, dims, str, box);
  if (rc) return rc;
  // packed tiles: the same maps with a box of the last group's images (unused copies without packing)
  CUtensorMap ma_pk = ma, mo_pk, mr_pk;
  if (p.pack) {
    box[p.dim_n] = (uint32_t)last_n;
    rc = encode_map(&ma_pk, L.in, 5, dims, str, box);
    if (rc) return rc;
  }
  uint64_t wd[2] = {(uint64_t)ktot, (uint64_t)L.Cout};
  uint64_t ws[1] = {(uint64_t)ktot * E};
  uint32_t wb[2] = {64, (uint32_t)BN};
  rc = encode_map(&mb, L.w, 2, wd, ws, wb);
  if (rc) return rc;
  // output / residual maps: NHWC (conv) or [M][ld] (linear), one box = 128 pixels x 64 channels
  CUtensorMap mo, mr;
  {
    uint64_t od[5], os[4];
    uint32_t ob[5];
    const bool lin = (L.kind == LK_LINEAR);
    const int n_out = L.out_split > 0 ? (L.n_img - L.out_split) : L.n_img;
    FP_REQUIRE(n_out > 0, "out_split=%d leaves no output images (n_img=%d)", L.out_split, L.n_img);
    auto fill = [&](int ld, int nimg) {
      const uint64_t sw_ = (uint64_t)ld * E, sh_ = sw_ * Wo, sn_ = sh_ * Ho;
      od[0] = (uint64_t)ld;
      ob[0] = 64;
      od[4] = 1;
      ob[4] = 1;
      if (lin) {
        od[1] = (uint64_t)Wo; od[2] = 1; od[3] = 1;
        os[0] = sw_; os[1] = sh_; os[2] = sh_; os[3] = sh_;
        ob[1] = (uint32_t)p.bw; ob[2] = 1; ob[3] = 1;
      } else {  // (n, h, w)
        od[1] = (uint64_t)Wo; od[2] = (uint64_t)Ho; od[3] = (uint64_t)nimg;
        os[0] = sw_; os[1] = sh_; os[2] = sn_; os[3] = sn_ * nimg;
        ob[1] = (uint32_t)p.bw; ob[2] = (uint32_t)p.bh; ob[3] = (uint32_t)(swap ? p.bn / 2 : p.bn);  // 128 pixels
      }
    };
    p.odim_h = lin ? -1 : 2;
    p.odim_n = lin ? -1 : 3;
    // the map of 128-pixel boxes and its packed-tile twin, whose box holds the last group's images
    auto encode_out = [&](CUtensorMap* m, CUtensorMap* m_pk, const void* base) {
      int e = encode_map(m, base, 5, od, os, ob);
      if (e || !p.pack) {
        *m_pk = *m;
        return e;
      }
      ob[3] = (uint32_t)last_n;
      return encode_map(m_pk, base, 5, od, os, ob);
    };
    fill(L.out_ld, n_out);
    rc = encode_out(&mo, &mo_pk, L.out);
    if (rc) return rc;
    if (L.res) {
      fill(L.res_ld, L.n_img);
      rc = encode_out(&mr, &mr_pk, L.res);
      if (rc) return rc;
    } else {
      mr = mo;
      mr_pk = mo_pk;
    }
  }
  if (swap) return launch_bn<128, true>(ma, mb, mo, mr, ma_pk, mo_pk, mr_pk, p, stream);
  if (BN == 256) return launch_bn<256>(ma, mb, mo, mr, ma_pk, mo_pk, mr_pk, p, stream);
  return BN == 128 ? launch_bn<128>(ma, mb, mo, mr, ma_pk, mo_pk, mr_pk, p, stream)
                   : launch_bn<64>(ma, mb, mo, mr, ma_pk, mo_pk, mr_pk, p, stream);
}

int gemm_layer_launch(const GemmLayer& L, cudaStream_t stream) { return gemm_layer_plan(L, stream, nullptr, nullptr); }

int gemm_layer_tile_n(const GemmLayer& L, int* tile_n) { return gemm_layer_plan(L, nullptr, tile_n, nullptr); }

int gemm_layer_tile_m(const GemmLayer& L, int* tile_m) { return gemm_layer_plan(L, nullptr, nullptr, tile_m); }

}  // namespace fp
