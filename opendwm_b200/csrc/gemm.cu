// Persistent warp-specialised wgmma GEMM with fused epilogues (sm_90a).
//
//   D[M,N] = A[M,K] · W[N,K]^T     A, W 16-bit (bf16/fp16), fp32 accumulation in registers
//   FP8:   D[M,N] = a_scale[M] w_scale[N] (A8[M,K] · W8[N,K]^T)  with E4M3 operands (opt-in)
//
// Roles (384 threads, one CTA per SM, persistent over 128 x NT output tiles):
//   warpgroup 0    TMA producer (one elected thread): 128x64 A tile + NTx64 W tile per k-block
//                  into a 4-stage 128B-swizzled shared-memory ring (mbarrier tx-count completion);
//                  runs ahead into the next tile while the consumers drain the current one
//   warpgroups 1-2 consumers: each issues wgmma m64nNTk16 (k32 for E4M3) for its 64 rows of
//                  the tile and then applies the fused epilogue straight from its register
//                  fragment (E4M3: after scaling it by the row and channel scales); 16-bit
//                  outputs go to shared memory and leave by TMA store (TmaOut), so the
//                  warpgroup returns to the next tile's MMAs while the stores drain, except
//                  when they are also scattered to peer GPUs, which is done from registers
// A stage is 128 bytes of K per row in either case: 64 16-bit or 128 E4M3 elements.
// NT = 256 (the widest wgmma; 128 accumulator registers per thread) unless the 256-wide tiles
// leave most SMs idle (pick_tile_n).
//
// Replaces the cuBLASLt GEMM + ~10 elementwise launches per sub-layer that the
// reference runs (SURVEY.md §2.3 K5-K8).
#include <stdlib.h>
#include <string.h>

#include "gemm_epilogue.cuh"

namespace dwm {

constexpr int STAGES = 4;
constexpr int A_STAGE_BYTES = BM * BK * 2;

// The epilogue region holds either the TMA store boxes or the fp32 transpose buffers of the
// register path: one launch uses one of them.
static_assert(EPI_BOXES_BYTES >= EPI_STAGE_BYTES, "epilogue region");
template <int NT>
struct GemmCfg {
  static constexpr int kBStageBytes = NT * BK * 2;
  static constexpr int kSmemBytes =
      STAGES * (A_STAGE_BYTES + kBStageBytes) + EPI_BOXES_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

// CL = 2: a cluster of two CTAs computes two vertically adjacent output tiles that share one
// W tile; each CTA loads its own A tile and HALF of the W tile, multicast into both CTAs, so
// every CTA reads half as much weight data from L2.  A stage of a CTA is refilled only after
// the consumers of BOTH CTAs have released it (the peer writes into it too).  An odd number
// of M tiles gives the last pair a dummy tile: its A loads are out of bounds (zero fill) and
// its rows are never stored.  Both variants accumulate in the same order: same bits.
// TA: operand type (bf16 / fp16 / E4M3); T: type of the 16-bit outputs (TA unless E4M3).
template <typename TA, typename T, int EPI, int NT, int CL>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a,
                      const __grid_constant__ CUtensorMap tmap_b,
                      const __grid_constant__ CUtensorMap tmap_out, int M, int N, int K,
                      EpiParams p) {
  constexpr int B_STAGE_BYTES = GemmCfg<NT>::kBStageBytes;
  constexpr int BKE = BK * 2 / static_cast<int>(sizeof(TA));   // K elements per stage
  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzled TMA / wgmma tiles need 1024-byte alignment.
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
  uint8_t* epi_region = smem + STAGES * (A_STAGE_BYTES + B_STAGE_BYTES);   // 1024-byte aligned
  float* epi_stage = reinterpret_cast<float*>(epi_region);
  uint64_t* bars = reinterpret_cast<uint64_t*>(epi_region + EPI_BOXES_BYTES);
  uint64_t* full_bar = bars;                 // [STAGES]  TMA -> consumers
  uint64_t* empty_bar = bars + STAGES;       // [STAGES]  consumers (of both CTAs when CL = 2) -> TMA

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const uint32_t rank = CL == 2 ? cluster_ctarank() : 0u;

  const int m_blocks = (M + BM - 1) / BM;
  const int n_blocks = (N + NT - 1) / NT;
  const int k_blocks = (K + BKE - 1) / BKE;
  const int num_tiles = ((m_blocks + CL - 1) / CL) * n_blocks;   // CL vertically adjacent tiles each
  const int first = static_cast<int>(blockIdx.x) / CL, step = static_cast<int>(gridDim.x) / CL;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], CL * EPI_WARPS);
    }
    fence_barrier_init();
  }
  if constexpr (CL == 2) cluster_sync_all(); else __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = first; tile < num_tiles; tile += step) {
        const int m_blk = (tile / n_blocks) * CL + static_cast<int>(rank);
        const int n_blk = tile % n_blocks;
        for (int kb = 0; kb < k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], A_STAGE_BYTES + B_STAGE_BYTES);
          tma_load_2d(&tmap_a, &full_bar[stage], smem_a + stage * A_STAGE_BYTES, kb * BKE,
                      m_blk * BM, kEvictNormal);
          if constexpr (CL == 2) {
            tma_load_2d_mc(&tmap_b, &full_bar[stage], smem_b + stage * B_STAGE_BYTES + rank * (B_STAGE_BYTES / 2),
                           kb * BKE, n_blk * NT + static_cast<int>(rank) * (NT / 2), 0x3, kEvictLast);
          } else {
            tma_load_2d(&tmap_b, &full_bar[stage], smem_b + stage * B_STAGE_BYTES, kb * BKE,
                        n_blk * NT, kEvictLast);
          }
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== consumers (warpgroups 1, 2) =====================
    setmaxnreg_inc<CONSUMER_REGS>();
    const int cw = wg - 1;                       // 64-row half of the tile
    const int wrow = cw * 64 + (warp & 3) * 16;  // first tile row of this warp
    float* stg = epi_stage + (warp - 4) * 512;
    TmaOut tout{epi_out16(EPI) && p.tma_out, &tmap_out, epi_region + cw * 2 * EPI_BOX_BYTES, 1 + cw,
                (threadIdx.x & 127) == 0, 0};
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = first; tile < num_tiles; tile += step) {
      const int m_blk = (tile / n_blocks) * CL + static_cast<int>(rank);
      const int n_blk = tile % n_blocks;
      const int t = threadIdx.x & 127;
      prefetch_resid_tile<EPI, NT>(p, m_blk * BM + cw * 64 + (t >> 1), M, n_blk * NT, N, t & 1);
      float acc[NT / 2];
      wg_mainloop<TA, NT, CL>(acc, smem_a, A_STAGE_BYTES, cw * 64 * 128, smem_b, B_STAGE_BYTES, full_bar,
                              empty_bar, STAGES, k_blocks, stage, phase, lane, rank ^ 1u);
      if constexpr (sizeof(TA) == 1)
        dequant_frag<NT>(acc, p.a_scale, p.w_scale, m_blk * BM + wrow, M, n_blk * NT, N, lane);
      drain_tile<T, EPI, NT>(acc, stg, m_blk * BM, wrow, M, n_blk * NT, N, p, lane, TileGeom{0, 0, 0, 0, 0}, &tout);
    }
    if (tout.on && tout.leader) bulk_wait_all();   // no CTA exits with its stores in flight
  }
  // a CTA of a pair must not exit while its peer may still multicast into it or arrive on it
  if constexpr (CL == 2) cluster_sync_all();
}

int g_resid_tma = 1;   // option "resid_tma": L2 prefetch of the RESID operands by the TMA unit

template <typename TA, typename T, int EPI, int NT, int CL>
static int launch_gemm(const dwm_linear_args* a, cudaStream_t stream) {
  constexpr int eb = static_cast<int>(sizeof(TA));
  CUtensorMap ta, tb;
  int rc = make_tmap_2d(&ta, a->A, a->M, a->K, a->lda, BM, BK * 2 / eb, eb);
  if (rc) return rc;
  rc = make_tmap_2d(&tb, a->W, a->N, a->K, a->ldw, NT / CL, BK * 2 / eb, eb);
  if (rc) return rc;

  EpiParams p;
  fill_epi_params(p, a);
  p.resid_prefetch = g_resid_tma;
  // 16-bit outputs by TMA store: the whole items [items, rows per item, N] at the remapped rows
  // (a layout without items is one item of M rows); the rows of a partial last item are copied
  // by the consumer threads
  CUtensorMap to = {};
  if (epi_out16(EPI) && a->n_peer_out == 0) {
    const long long rpi = a->rows_per_item > 0 ? a->rows_per_item : a->M;
    const long long items = a->M / rpi;
    const long long item_ld = (a->rows_per_item > 0 ? a->out_item_stride : a->M) * a->ldo;
    const long long n_out = (EPI == DWM_EPI_GEGLU || EPI == DWM_EPI_GEGLU_TANH) ? a->N / 2 : a->N;
    if (items > 0) {
      rc = make_tmap_3d(&to, reinterpret_cast<const T*>(a->out) + a->out_row_offset * a->ldo, items, rpi, n_out,
                        a->ldo, item_ld, 64, 64, 2);
      if (rc) return rc;
    }
    p.tma_out = 1;
    p.out_rpi = static_cast<int>(rpi);
    p.out_items = static_cast<int>(items);
  }

  constexpr int smem_bytes = GemmCfg<NT>::kSmemBytes;
  auto kern = gemm_wgmma_kernel<TA, T, EPI, NT, CL>;
  static bool attr_set = false;  // per instantiation
  if (!attr_set) {
    DWM_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    attr_set = true;
  }
  const long long m_blocks = (a->M + BM - 1) / BM;
  const long long n_blocks = (a->N + NT - 1) / NT;
  const long long tiles = ((m_blocks + CL - 1) / CL) * n_blocks;
  const long long slots = sm_count() / CL;
  const int grid = CL * static_cast<int>(tiles < slots ? tiles : slots);
  const int Mi = static_cast<int>(a->M), Ni = static_cast<int>(a->N), Ki = static_cast<int>(a->K);
  if constexpr (CL == 1) {
    kern<<<grid, GEMM_THREADS, smem_bytes, stream>>>(ta, tb, to, Mi, Ni, Ki, p);
  } else {
    DWM_CHECK_CUDA(launch_cluster2(kern, grid, GEMM_THREADS, smem_bytes, stream,
                                   ta, tb, to, Mi, Ni, Ki, p));
  }
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int g_gemm_bn = 0;   // 0: tile width by wave efficiency; 128 / 256 force it (option "gemm_bn")
int g_gemm_2cta = -1;   // -1: from env DWM_GEMM_2CTA (default 1), 0 / 1: forced (option "gemm_2cta")

// Time of a persistent launch ~ waves x tile width / rate.  A 128-wide tile streams 1.5x the
// A + W bytes from L2 per FLOP of a 256-wide one, and with every SM busy it runs at about 0.9 of
// its rate (tools/gemm_bench.py on an H100 80GB HBM3 at 400 W, the step's 86016- and 29568-row
// shapes, fp16 and bf16: median 0.92-0.94, range 0.82-1.12).  So the 128-wide tile wins when
// it saves a tenth of the waves x width, not for a smaller fraction of a wave that the tile
// count rounds off: 4096 x 1536 x 1536 RESID picks 128 (1.1-1.3x), 2048 x 1536 keeps 256.
static int pick_tile_n(const dwm_linear_args* a, int cl) {
  if (a->epilogue == DWM_EPI_GEGLU || a->epilogue == DWM_EPI_GEGLU_TANH) return 256;
  if (g_gemm_bn == 128 || g_gemm_bn == 256) return g_gemm_bn;
  const long long slots = sm_count() / cl;
  const long long m_groups = ((a->M + BM - 1) / BM + cl - 1) / cl;
  const long long t256 = m_groups * ((a->N + 255) / 256), t128 = m_groups * ((a->N + 127) / 128);
  const long long waves256 = (t256 + slots - 1) / slots, waves128 = (t128 + slots - 1) / slots;
  return waves128 * 128 * 10 < waves256 * 256 * 9 ? 128 : 256;   // 128-wide cost / 0.9
}

template <typename TA, typename T, int EPI, int CL>
static int launch_pick_n(const dwm_linear_args* a, cudaStream_t s) {
  if (pick_tile_n(a, CL) == 128) return launch_gemm<TA, T, EPI, 128, CL>(a, s);
  return launch_gemm<TA, T, EPI, 256, CL>(a, s);
}

// TF: the 16-bit type named in the kernel of the fp32-output epilogues, which never use it.
// 16-bit operands keep TF = T; E4M3 operands share one instantiation between both out_dtypes.
template <typename TA, typename T, int CL, typename TF = T>
static int dispatch_epi(const dwm_linear_args* a, cudaStream_t s) {
  if constexpr (sizeof(TA) == 2) {   // text-encoder epilogues: 16-bit operands only
    if (a->epilogue == DWM_EPI_STORE && a->act == DWM_ACT_QUICK_GELU)
      return launch_pick_n<TA, T, EPI_STORE_QUICK_GELU, CL>(a, s);
    if (a->epilogue == DWM_EPI_GEGLU_TANH) return launch_gemm<TA, T, DWM_EPI_GEGLU_TANH, 256, CL>(a, s);
  }
  switch (a->epilogue) {
    case DWM_EPI_STORE: return launch_pick_n<TA, T, DWM_EPI_STORE, CL>(a, s);
    case DWM_EPI_GEGLU: return launch_gemm<TA, T, DWM_EPI_GEGLU, 256, CL>(a, s);
    case DWM_EPI_QKNORM: return launch_pick_n<TA, T, DWM_EPI_QKNORM, CL>(a, s);
    case DWM_EPI_RESID: return launch_pick_n<TA, TF, DWM_EPI_RESID, CL>(a, s);
    case DWM_EPI_F32: return launch_pick_n<TA, TF, DWM_EPI_F32, CL>(a, s);
    default: set_last_error("dwm_b200_linear: unknown epilogue %d", a->epilogue); return -1;
  }
}

template <int CL>
static int dispatch_e4m3(const dwm_linear_args* a, cudaStream_t s) {
  if (a->out_dtype == DWM_BF16) return dispatch_epi<__nv_fp8_e4m3, __nv_bfloat16, CL>(a, s);
  return dispatch_epi<__nv_fp8_e4m3, __half, CL, __nv_bfloat16>(a, s);
}

}  // namespace dwm

namespace dwm { int g_attn_tc = -1; extern int g_ln_staged; extern int g_conv_2cta; extern int g_conv_halo; }

extern "C" int dwm_b200_set_option(const char* name, int value) {
  using namespace dwm;
  DWM_REQUIRE(name != nullptr, "dwm_b200_set_option: null name");
  if (strcmp(name, "attn_tc") == 0) { g_attn_tc = value; return 0; }
  if (strcmp(name, "ln_staged") == 0) { g_ln_staged = value; return 0; }
  if (strcmp(name, "gemm_bn") == 0) { g_gemm_bn = value; return 0; }
  if (strcmp(name, "gemm_2cta") == 0) { g_gemm_2cta = value; return 0; }
  if (strcmp(name, "resid_tma") == 0) { g_resid_tma = value; return 0; }
  if (strcmp(name, "conv_2cta") == 0) { g_conv_2cta = value; return 0; }
  if (strcmp(name, "conv_halo") == 0) { g_conv_halo = value; return 0; }
  set_last_error("dwm_b200_set_option: unknown option %s", name);
  return -1;
}

extern "C" int dwm_b200_linear(const dwm_linear_args* a, dwm_stream_t stream) {
  using namespace dwm;
  DWM_REQUIRE(a != nullptr, "dwm_b200_linear: null args");
  DWM_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, "dwm_b200_linear: empty problem %lld x %lld x %lld",
              (long long)a->M, (long long)a->N, (long long)a->K);
  DWM_REQUIRE(a->M < (1ll << 31) && a->N < (1ll << 31) && a->K < (1ll << 31),
              "dwm_b200_linear: dimension exceeds int32");
  DWM_REQUIRE(a->A && a->W && a->out, "dwm_b200_linear: null A/W/out");
  DWM_REQUIRE(a->K % 8 == 0 && a->lda % 8 == 0 && a->ldw % 8 == 0,
              "dwm_b200_linear: K, lda, ldw must be multiples of 8 (16-byte TMA pitch); got %lld %lld %lld",
              (long long)a->K, (long long)a->lda, (long long)a->ldw);
  if (a->dtype == DWM_E4M3) {
    DWM_REQUIRE(a->K % 16 == 0 && a->lda % 16 == 0 && a->ldw % 16 == 0,
                "dwm_b200_linear: E4M3 needs K, lda, ldw multiples of 16 (16-byte TMA pitch); got %lld %lld %lld",
                (long long)a->K, (long long)a->lda, (long long)a->ldw);
    DWM_REQUIRE(a->a_scale && a->w_scale, "dwm_b200_linear: E4M3 operands need a_scale and w_scale");
    DWM_REQUIRE(a->out_dtype == DWM_BF16 || a->out_dtype == DWM_F16,
                "dwm_b200_linear: E4M3 operands need out_dtype DWM_BF16 or DWM_F16, got %d", a->out_dtype);
    DWM_REQUIRE((reinterpret_cast<uintptr_t>(a->w_scale) & 7) == 0,
                "dwm_b200_linear: w_scale must be 8-byte aligned");
  }
  DWM_REQUIRE((reinterpret_cast<uintptr_t>(a->A) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(a->W) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(a->out) & 15) == 0,
              "dwm_b200_linear: A, W, out must be 16-byte aligned");
  DWM_REQUIRE(a->N % 32 == 0, "dwm_b200_linear: N must be a multiple of 32, got %lld", (long long)a->N);
  DWM_REQUIRE(a->ldo % 8 == 0, "dwm_b200_linear: ldo must be a multiple of 8");
  if (a->epilogue == DWM_EPI_GEGLU || a->epilogue == DWM_EPI_GEGLU_TANH)
    DWM_REQUIRE(a->N % 256 == 0, "dwm_b200_linear: GEGLU needs N %% 256 == 0 (packed weight)");
  if (a->epilogue == DWM_EPI_GEGLU_TANH || a->act == DWM_ACT_QUICK_GELU) {
    DWM_REQUIRE(a->dtype == DWM_BF16 || a->dtype == DWM_F16,
                "dwm_b200_linear: DWM_EPI_GEGLU_TANH and DWM_ACT_QUICK_GELU need 16-bit operands");
    DWM_REQUIRE(a->act != DWM_ACT_QUICK_GELU || a->epilogue == DWM_EPI_STORE,
                "dwm_b200_linear: DWM_ACT_QUICK_GELU needs the DWM_EPI_STORE epilogue");
  }
  if (a->epilogue == DWM_EPI_QKNORM) {
    DWM_REQUIRE(a->N % 64 == 0 && a->qk_region > 0 && a->qk_region % 64 == 0 && a->q_norm_weight &&
                    (a->k_norm_weight || a->qk_norm_regions == 1),
                "dwm_b200_linear: QKNORM needs head_dim 64 regions and both norm weights");
  }
  DWM_REQUIRE(a->n_peer_out >= 0 && a->n_peer_out <= 8, "dwm_b200_linear: n_peer_out out of range");
  if (a->n_peer_out > 0)
    DWM_REQUIRE(a->epilogue == DWM_EPI_STORE || a->epilogue == DWM_EPI_QKNORM || a->epilogue == DWM_EPI_GEGLU ||
                    a->epilogue == DWM_EPI_GEGLU_TANH,
                "dwm_b200_linear: peer_out needs a 16-bit epilogue");
  if (a->epilogue == DWM_EPI_RESID && a->blend_x)
    DWM_REQUIRE(a->alpha != nullptr, "dwm_b200_linear: blend_x without alpha");
  // the epilogue reads bias / resid / gate / blend_x rows as float2 / float4, stores to the peers
  // as 8-byte words at the offsets of `out`, and prefetches the RESID rows with cp.async.bulk
  for (const void* p : {static_cast<const void*>(a->bias), static_cast<const void*>(a->resid),
                        static_cast<const void*>(a->gate), static_cast<const void*>(a->blend_x)})
    DWM_REQUIRE((reinterpret_cast<uintptr_t>(p) & 15) == 0,
                "dwm_b200_linear: bias, resid, gate, blend_x must be 16-byte aligned");
  for (int i = 0; i < a->n_peer_out; ++i)
    DWM_REQUIRE(a->peer_out[i] && (reinterpret_cast<uintptr_t>(a->peer_out[i]) & 15) == 0,
                "dwm_b200_linear: peer_out[%d] must be a 16-byte aligned pointer", i);
  DWM_REQUIRE((!a->resid || a->ldr % 4 == 0) && (!a->gate || a->gate_ld % 4 == 0) &&
                  (!a->blend_x || a->ldx % 4 == 0),
              "dwm_b200_linear: ldr, gate_ld, ldx must be multiples of 4 (16-byte rows); got %lld %lld %lld",
              (long long)a->ldr, (long long)a->gate_ld, (long long)a->ldx);
  if (a->rows_per_item > 0 && a->epilogue != DWM_EPI_RESID && a->epilogue != DWM_EPI_F32)
    DWM_REQUIRE(a->out_item_stride >= a->rows_per_item,
                "dwm_b200_linear: out_item_stride %lld < rows_per_item %lld would write several items "
                "to the same output rows", (long long)a->out_item_stride, (long long)a->rows_per_item);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (g_gemm_2cta < 0) {
    const char* e = getenv("DWM_GEMM_2CTA");
    g_gemm_2cta = (e && e[0] == '0') ? 0 : 1;
  }
  // Pairs halve the W traffic from L2, which pays at large K (8192^3: 1.25-1.4x, K = 6144: up
  // to 1.15x); at K = 1536 and 8192 rows or more the two kernels are even (gemm_bench, H100
  // 80GB HBM3 at 400 W).  From 512 to 4096 rows the 1-CTA kernel is ahead by a median 1.06x,
  // about the spread between two runs of the same shape, and 5376 x 640 x 640 is even, so
  // pairs start once there are enough 128-row tiles to give both CTAs of a cluster work.
  const bool pair = g_gemm_2cta == 1 && a->M >= 512;
  if (a->dtype == DWM_BF16)
    return pair ? dispatch_epi<__nv_bfloat16, __nv_bfloat16, 2>(a, s) : dispatch_epi<__nv_bfloat16, __nv_bfloat16, 1>(a, s);
  if (a->dtype == DWM_F16) return pair ? dispatch_epi<__half, __half, 2>(a, s) : dispatch_epi<__half, __half, 1>(a, s);
  if (a->dtype == DWM_E4M3) return pair ? dispatch_e4m3<2>(a, s) : dispatch_e4m3<1>(a, s);
  set_last_error("dwm_b200_linear: dtype must be DWM_BF16, DWM_F16 or DWM_E4M3, got %d", a->dtype);
  return -1;
}
