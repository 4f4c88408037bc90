// fp_attn_tc.cu — softmax(Q K^T / sqrt(128)) V on the Hopper tensor cores (wgmma).
//
// Replaces the SDPA inside nn.MultiheadAttention (refine_network.py:56-70 `trans_head` / `rot_head`,
// score_network.py:53 `att`) for T = 400 tokens and 4 heads of 128.  Persistent CTAs walk the work units
// (sequence, head[, group], 128-row query tile); per unit:
//
//   smem   Q tile, 128 query rows: 2 slabs [128][64 dims] (K-major, 128B swizzle), 2 stages        64 KB
//          K and V of 80 keys:     2 + 2 slabs [80 keys][64 dims], 3 stages                         120 KB
//   warps  thread 0 = TMA producer; warpgroups 1, 2 = query rows [0, 64) and [64, 128) of the tile
//
// A consumer warpgroup walks the five 80-key chunks with an online softmax: S = Q K^T (m64n80k16, accumulators in
// registers), running row maximum, P = exp2(S c - m c) packed to fp16 A fragments in registers, O = O alpha + P V
// (m64n128k16, V the MN-major B operand straight from the TMA tile), row sum in fp32.  O / l goes to fp16 into the
// warpgroup's own rows of the Q stage and leaves by TMA store.  Rows >= 400 of the last tile are zero-filled on load
// and clipped on store by the TMA unit.
#include "fp_attn.cuh"
#include "fp_common.cuh"
#include "fp_gemm.cuh"
#include "fp_wgmma.cuh"

namespace fp {

int encode_map_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box);
int num_sms();

namespace {

constexpr int T = 400;
constexpr int DH = 128;
constexpr int kQTiles = (T + 127) / 128;    // 4
constexpr int kKeys = 80;                   // keys per chunk
constexpr int kChunks = T / kKeys;          // 5
constexpr int kKVSlab = kKeys * 128;        // 10 KB: [80 keys][64 dims]
constexpr int kKVStage = 4 * kKVSlab;       // K dims [0,64), [64,128); V dims [0,64), [64,128)
constexpr int kKVStages = 3;
constexpr int kQSlab = 128 * 128;           // 16 KB: [128 rows][64 dims]
constexpr int kQStage = 2 * kQSlab;
constexpr int kQStages = 2;
constexpr int kOffKV = 0;
constexpr int kOffQ = kOffKV + kKVStages * kKVStage;  // 122880
constexpr int kOffBar = kOffQ + kQStages * kQStage;   // 188416
constexpr int kSmem = kOffBar + 256 + 1024;
constexpr int kThreadsTc = 384;

__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}

struct TcParams {
  int q_col, k_col, v_col;  // column of head 0 inside a qkv row (group offset added per work item)
  int group_col_stride;
  float scale_log2e;        // softmax scale * log2(e)
  int B, H, G;              // work items: (sequence, head, group)
};

__global__ void __launch_bounds__(kThreadsTc, 1)
    attn_tc_kernel(const __grid_constant__ CUtensorMap map_kv,  // (cols, T, B), box (64, 80, 1): K and V chunks
                   const __grid_constant__ CUtensorMap map_q,   // (cols, T, B), box (64, 128, 1)
                   const __grid_constant__ CUtensorMap map_o,   // (512, T, B, G), box (64, 64, 1, 1)
                   const TcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* q_full = bars;                           // [kQStages]
  uint64_t* q_empty = bars + kQStages;               // [kQStages]
  uint64_t* kv_full = bars + 2 * kQStages;           // [kKVStages]
  uint64_t* kv_empty = bars + 2 * kQStages + kKVStages;

  const int total = p.B * p.H * p.G * kQTiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_kv);
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_o);
    for (int i = 0; i < kQStages; ++i) {
      mbar_init(&q_full[i], 1);
      mbar_init(&q_empty[i], 2);  // one arrival per consumer warpgroup, after its O stores have left the stage
    }
    for (int i = 0; i < kKVStages; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 256);
    }
    mbar_fence_init();
  }
  __syncthreads();
  pdl_trigger();
  pdl_wait();

  auto unit = [&](int u, int& b, int& h, int& g, int& gcol, int& qt) {
    qt = u % kQTiles;
    const int w = u / kQTiles;
    b = w % p.B;
    h = (w / p.B) % p.H;
    g = w / (p.B * p.H);
    gcol = g * p.group_col_stride + h * DH;
  };

  if (threadIdx.x < 128) {
    if (threadIdx.x == 0) {
      int qs = 0, qph = 0, ks = 0, kph = 0;
      for (int u = blockIdx.x; u < total; u += gridDim.x) {
        int b, h, g, gcol, qt;
        unit(u, b, h, g, gcol, qt);
        mbar_wait(&q_empty[qs], qph ^ 1);
        mbar_expect_tx(&q_full[qs], kQStage);
        for (int s = 0; s < 2; ++s)
          tma_load_3d(&map_q, &q_full[qs], smem + kOffQ + qs * kQStage + s * kQSlab, gcol + p.q_col + s * 64, qt * 128, b);
        if (++qs == kQStages) {
          qs = 0;
          qph ^= 1;
        }
        for (int c = 0; c < kChunks; ++c) {
          mbar_wait(&kv_empty[ks], kph ^ 1);
          mbar_expect_tx(&kv_full[ks], kKVStage);
          uint8_t* st = smem + kOffKV + ks * kKVStage;
          for (int s = 0; s < 2; ++s) {
            tma_load_3d(&map_kv, &kv_full[ks], st + s * kKVSlab, gcol + p.k_col + s * 64, c * kKeys, b);
            tma_load_3d(&map_kv, &kv_full[ks], st + (2 + s) * kKVSlab, gcol + p.v_col + s * 64, c * kKeys, b);
          }
          if (++ks == kKVStages) {
            ks = 0;
            kph ^= 1;
          }
        }
      }
    }
    return;
  }

  const int ct = threadIdx.x - 128;
  const int cw = ct >> 7;  // query rows [64 cw, 64 cw + 64) of the tile
  const int lane = threadIdx.x & 31;
  const int r0 = 64 * cw + 16 * ((ct >> 5) & 3) + (lane >> 2);  // this thread's rows: r0, r0 + 8
  const int cq = 2 * (lane & 3);
  const bool leader = ((ct & 127) == 0);
  const float c = p.scale_log2e;
  float s_acc[kKeys / 2], o[DH / 2];
#pragma unroll
  for (int i = 0; i < kKeys / 2; ++i) s_acc[i] = 0.f;
  int qs = 0, qph = 0, ks = 0, kph = 0;
  for (int u = blockIdx.x; u < total; u += gridDim.x) {
    int b, h, g, gcol, qt;
    unit(u, b, h, g, gcol, qt);
#pragma unroll
    for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};  // l: this thread's partial row sums
    mbar_wait(&q_full[qs], qph);
    const uint32_t qbase = smem_u32(smem + kOffQ + qs * kQStage) + (uint32_t)cw * 8192u;
    for (int ch = 0; ch < kChunks; ++ch) {
      mbar_wait(&kv_full[ks], kph);
      const uint32_t kvbase = smem_u32(smem + kOffKV + ks * kKVStage);
      // S = Q K^T over the 80 keys of this chunk; K = 128 dims = 2 slabs x 4 k-steps
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const int s = kk >> 2, k = kk & 3;
        Wgmma<kKeys>::ss(s_acc, gmma_desc_sw128(qbase + s * kQSlab) + (uint64_t)(2 * k),
                         gmma_desc_sw128(kvbase + s * kKVSlab) + (uint64_t)(2 * k), kk > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s_acc);
      // running row maximum (a row's 80 values live in the 4 lanes of a quad)
      float mx[2] = {m[0], m[1]};
#pragma unroll
      for (int j = 0; j < kKeys / 8; ++j) {
        mx[0] = fmaxf(mx[0], fmaxf(s_acc[4 * j], s_acc[4 * j + 1]));
        mx[1] = fmaxf(mx[1], fmaxf(s_acc[4 * j + 2], s_acc[4 * j + 3]));
      }
      float mc[2], alpha[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
        mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
        alpha[hh] = exp2f((m[hh] - mx[hh]) * c);  // 0 on the first chunk (m = -inf)
        m[hh] = mx[hh];
        mc[hh] = mx[hh] * c;
        l[hh] *= alpha[hh];
      }
#pragma unroll
      for (int j = 0; j < DH / 8; ++j) {
        o[4 * j] *= alpha[0];
        o[4 * j + 1] *= alpha[0];
        o[4 * j + 2] *= alpha[1];
        o[4 * j + 3] *= alpha[1];
      }
      // P = exp2(s c - m c) in fp32 (row sums), packed to the fp16 A fragments of the PV wgmma
      uint32_t pa[kKeys / 16][4];
#pragma unroll
      for (int j = 0; j < kKeys / 8; ++j) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const float p0 = exp2f(fmaf(s_acc[4 * j + 2 * hh], c, -mc[hh]));
          const float p1 = exp2f(fmaf(s_acc[4 * j + 2 * hh + 1], c, -mc[hh]));
          l[hh] += p0 + p1;
          pa[j >> 1][(j & 1) * 2 + hh] = pack_half2(p0, p1);
        }
      }
      // O += P V: V chunk [80 keys][128 dims] is the MN-major B operand (dims = N, two 64-dim slabs)
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kKeys / 16; ++kk)
        Wgmma<DH>::rs_mn(o, pa[kk], gmma_desc_mn_sw128(kvbase + 2 * kKVSlab + kk * 16 * 128, kKVSlab), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(o);
      mbar_arrive(&kv_empty[ks]);
      if (++ks == kKVStages) {
        ks = 0;
        kph ^= 1;
      }
    }
    float inv[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
      l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
      inv[hh] = 1.f / l[hh];
    }
    // O tile -> fp16 -> this warpgroup's own rows of the Q stage (its Q reads have all retired) -> TMA store
    uint8_t* qst = smem + kOffQ + qs * kQStage;
#pragma unroll
    for (int j = 0; j < DH / 8; ++j) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = r0 + 8 * hh;
        *reinterpret_cast<uint32_t*>(qst + (j >> 3) * kQSlab + row * 128 + ((((uint32_t)j & 7u) ^ (uint32_t)(row & 7)) << 4) +
                                     cq * 2) = pack_half2(o[4 * j + 2 * hh] * inv[hh], o[4 * j + 2 * hh + 1] * inv[hh]);
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
    if (leader) {
      for (int s = 0; s < 2; ++s)
        tma_store_4d(&map_o, qst + s * kQSlab + cw * 8192, h * DH + s * 64, qt * 128 + 64 * cw, b, g);
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // the stage may be refilled once read out
      mbar_arrive(&q_empty[qs]);
    }
    if (++qs == kQStages) {
      qs = 0;
      qph ^= 1;
    }
  }
  if (leader) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

}  // namespace

int attn_tc_launch(const AttnParams& p, cudaStream_t stream) {
  FP_REQUIRE(p.T == T && p.n_heads == 4, "wgmma attention is specialised for T=400, 4 heads of 128");
  FP_REQUIRE(p.ld_out == 512, "wgmma attention writes [*, 512] rows");
  static std::atomic<unsigned long long> attr_mask{0};  // per device: the attribute is device state
  if (!device_bit_test(attr_mask)) {
    FP_CUDA_OK(cudaFuncSetAttribute(attn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    device_bit_set(attr_mask);
  }
  if (p.B == 0) return 0;
  CUtensorMap mkv, mq, mo;
  const uint64_t E = 2;
  uint64_t d3[3] = {(uint64_t)p.ld, (uint64_t)T, (uint64_t)p.B};
  uint64_t s3[2] = {(uint64_t)p.ld * E, (uint64_t)p.ld * E * T};
  uint32_t bkv[3] = {64, (uint32_t)kKeys, 1}, bq[3] = {64, 128, 1};
  int rc = encode_map_f16(&mkv, p.qkv, 3, d3, s3, bkv);
  if (rc) return rc;
  rc = encode_map_f16(&mq, p.qkv, 3, d3, s3, bq);
  if (rc) return rc;
  uint64_t d4[4] = {512, (uint64_t)T, (uint64_t)p.B, (uint64_t)p.n_groups};
  uint64_t s4[3] = {512 * E, 512 * E * T, (uint64_t)p.out_group_stride * E};
  if (p.n_groups == 1) s4[2] = 512 * E * T * p.B;
  uint32_t bo[4] = {64, 64, 1, 1};
  rc = encode_map_f16(&mo, p.out, 4, d4, s4, bo);
  if (rc) return rc;
  TcParams tp;
  tp.q_col = p.q_off;
  tp.k_col = p.k_off;
  tp.v_col = p.v_off;
  tp.group_col_stride = p.group_col_stride;
  tp.scale_log2e = p.scale * 1.4426950408889634f;
  tp.B = p.B;
  tp.H = p.n_heads;
  tp.G = p.n_groups;
  const int total = p.B * p.n_heads * p.n_groups * kQTiles;
  const int sms = num_sms();
  FP_REQUIRE(sms > 0, "no CUDA device");
  dim3 grid(total < sms ? total : sms);
  FP_CUDA_OK(launch_pdl(attn_tc_kernel, grid, dim3(kThreadsTc), kSmem, stream, 1, mkv, mq, mo, tp));
  note_launches(1);
  FP_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace fp
