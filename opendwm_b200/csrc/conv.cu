// im2col-free convolution on wgmma (sm_90a): implicit GEMM over channels-last
// activations.  For every filter tap (dt, dh, dw) the producer TMA-loads the SHIFTED
// bw x bh pixel patch (5-D tensor map over [NB, TP, H, W, C]; spatial zero padding is the
// TMA out-of-bounds fill) plus that tap's [C_out, C_in] weight slice, and the two consumer
// warpgroups accumulate all taps x channel blocks into one register accumulator (64 pixel
// rows each).  No column matrix is ever materialised.  Temporal padding is NOT implicit: the
// caller provides TP = T_out + KT - 1 frames (causal convolutions keep their cache /
// replicated frames in front).
//
// Used by: CogVideoX causal conv3d (3x3x3), its per-frame upsampler conv2d (1x3x3), the
// T2I-adapter 3x3 convs and the UNet ResBlock convs.  Epilogues are the GEMM ones (bias/act
// store, fp32 residual).
//
// FP8 (opt-in; RESID epilogue, and F32 at C_out tiles of 128 / 256 for the VAE ResNet conv1):
// E4M3 activations with ONE fp32 scale per volume nb and
// E4M3 weights with one scale per output channel (over all taps and input channels).  A
// per-pixel scale could not be factored out of a sum over taps that read different pixels;
// a volume scale can, because tiles never cross volumes and the padding is zero.  A stage is
// still 128 bytes of K per pixel row (128 E4M3 channels, four k32 MMAs), so the patch, halo
// and weight-slice layouts and every descriptor step are the 16-bit ones.
#include "gemm_epilogue.cuh"

namespace dwm {

constexpr int CV_STAGES = 4;
constexpr int CV_ROW_BYTES = BK * 2;           // bytes of K per pixel row and stage (either precision)
constexpr int CV_A_BYTES = 128 * CV_ROW_BYTES;

struct ConvGeom {
  int nb, t_out, h, w;
  int kt, kh, kw;
  int bw, bh;          // pixel patch of one M tile
  int tiles_w, tiles_h;
  int c_in, c_out;
};

// Variants of one kernel (same pipeline, same epilogues):
//   CL = 2    cluster of two CTAs on two pixel tiles that share the weight slice: each CTA loads
//             its own shifted patch and HALF of the slice, multicast into both (protocol of the
//             paired GEMM, gemm.cu); same accumulation order as CL = 1, so the same bits
//   HALO      kw = 3 and rows of >= 128 pixels: an M tile is ONE image-row segment of 128
//             pixels.  Per (dt, dh, C_in block) the producer loads the segment with a one-pixel
//             halo on both sides ONCE (130 rows x 128 B; TMA zero fill = the spatial padding)
//             plus the three weight slices of dw = 0, 1, 2, and the consumers issue the three
//             taps against ROW-SHIFTED views of that tile (descriptor start dw rows in, base
//             offset 0: the swizzle follows the absolute address).  A traffic drops 3x
//             (27 -> 9 loads per C_in block for 3x3x3).
constexpr int CVH_A_ROWS = 130;
constexpr int CVH_A_BYTES = 17 * 1024;        // 130 rows x 128 B, rounded up to the swizzle pattern

template <int CBN, bool HALO>
struct ConvCfg {
  static constexpr int kTaps = HALO ? 3 : 1;                   // weight slices per stage
  static constexpr int kABytes = HALO ? CVH_A_BYTES : CV_A_BYTES;
  static constexpr int kBBytes = kTaps * CBN * BK * 2;
  static constexpr int kStages = (kABytes + kBBytes) > 48 * 1024 ? 3 : CV_STAGES;
  static constexpr int kSmemBytes = kStages * (kABytes + kBBytes) + EPI_STAGE_BYTES + 1024 + 256;
};

// TA: operand type (bf16 / fp16 / E4M3); T: type of the 16-bit outputs (TA unless E4M3)
template <typename TA, typename T, int EPI, int CBN, int CL, bool HALO>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    conv_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                      const ConvGeom g, EpiParams p) {
  using Cfg = ConvCfg<CBN, HALO>;
  constexpr int A_BYTES = Cfg::kABytes, B_BYTES = Cfg::kBBytes, STAGES = Cfg::kStages;
  constexpr int BKE = CV_ROW_BYTES / static_cast<int>(sizeof(TA));   // channels per stage
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_BYTES;
  float* epi_stage = reinterpret_cast<float*>(smem + STAGES * (A_BYTES + B_BYTES));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * (A_BYTES + B_BYTES) + EPI_STAGE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const uint32_t rank = CL == 2 ? cluster_ctarank() : 0u;
  const int n_blocks = (g.c_out + CBN - 1) / CBN;
  const int c_blocks = (g.c_in + BKE - 1) / BKE;   // a ragged last block is TMA zero fill
  const int outer_taps = HALO ? g.kt * g.kh : g.kt * g.kh * g.kw;   // HALO: dw runs inside the stage
  const int k_iters = outer_taps * c_blocks;
  const int w_tiles = HALO ? (g.w + 127) / 128 : g.tiles_w;
  const long long m_tiles = static_cast<long long>(g.nb) * g.t_out * (HALO ? g.h * w_tiles : g.tiles_w * g.tiles_h);
  const long long num_tiles = ((m_tiles + CL - 1) / CL) * n_blocks;
  const long long first = static_cast<long long>(blockIdx.x) / CL, step = static_cast<long long>(gridDim.x) / CL;
  const uint32_t stage_tx = HALO ? static_cast<uint32_t>(CVH_A_ROWS * CV_ROW_BYTES + B_BYTES)
                                 : static_cast<uint32_t>(g.bw * g.bh * CV_ROW_BYTES + B_BYTES);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_w);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], CL * EPI_WARPS); }
    fence_barrier_init();
  }
  if constexpr (CL == 2) cluster_sync_all(); else __syncthreads();

  // tile -> (n_blk fastest, then the group of CL pixel tiles); this CTA's pixel tile: its
  // (w0, h0) origin, frame and volume.  HALO tiles are row segments (bh = 1, bw = 128).  The
  // dummy tile of an odd pair has nb == g.nb: out of bounds, zero fill, never stored.
  auto decode = [&](long long tile, int& n_blk, int& w0, int& h0, int& t, int& nb) -> bool {
    n_blk = static_cast<int>(tile % n_blocks);
    long long r = (tile / n_blocks) * CL + rank;
    const bool valid = r < m_tiles;
    if (HALO) {
      w0 = static_cast<int>(r % w_tiles) * 128; r /= w_tiles;
      h0 = static_cast<int>(r % g.h); r /= g.h;
    } else {
      w0 = static_cast<int>(r % g.tiles_w) * g.bw; r /= g.tiles_w;
      h0 = static_cast<int>(r % g.tiles_h) * g.bh; r /= g.tiles_h;
    }
    t = static_cast<int>(r % g.t_out);
    nb = static_cast<int>(r / g.t_out);
    return valid;
  };

  if (wg == 0) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (long long tile = first; tile < num_tiles; tile += step) {
        int n_blk, w0, h0, t, nb;
        decode(tile, n_blk, w0, h0, t, nb);
        for (int ot = 0; ot < outer_taps; ++ot) {
          const int kw_in = HALO ? 1 : g.kw;
          const int dw = ot % kw_in, dh = (ot / kw_in) % g.kh, dt = ot / (kw_in * g.kh);
          for (int cb = 0; cb < c_blocks; ++cb) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_expect_tx(&full_bar[stage], stage_tx);
            uint8_t* sb = smem_b + stage * B_BYTES;
            if constexpr (HALO) {
              tma_load_5d(&tmap_x, &full_bar[stage], smem_a + stage * A_BYTES, cb * BKE, w0 - 1,
                          h0 + dh - g.kh / 2, t + dt, nb, kEvictNormal);
#pragma unroll
              for (int d = 0; d < 3; ++d)
                tma_load_2d(&tmap_w, &full_bar[stage], sb + d * CBN * CV_ROW_BYTES, cb * BKE,
                            (ot * 3 + d) * g.c_out + n_blk * CBN, kEvictLast);
            } else {
              tma_load_5d(&tmap_x, &full_bar[stage], smem_a + stage * A_BYTES, cb * BKE,
                          w0 + dw - g.kw / 2, h0 + dh - g.kh / 2, t + dt, nb, kEvictNormal);
              if constexpr (CL == 2)
                tma_load_2d_mc(&tmap_w, &full_bar[stage], sb + rank * (B_BYTES / 2), cb * BKE,
                               ot * g.c_out + n_blk * CBN + static_cast<int>(rank) * (CBN / 2), 0x3, kEvictLast);
              else
                tma_load_2d(&tmap_w, &full_bar[stage], sb, cb * BKE, ot * g.c_out + n_blk * CBN, kEvictLast);
            }
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    __syncwarp();
  } else {
    setmaxnreg_inc<CONSUMER_REGS>();
    const int cw = wg - 1;
    const int wrow = cw * 64 + (warp & 3) * 16;
    float* stg = epi_stage + (warp - 4) * 512;
    int stage = 0;
    uint32_t phase = 0;
    for (long long tile = first; tile < num_tiles; tile += step) {
      int n_blk, w0, h0, t, nb;
      const bool valid = decode(tile, n_blk, w0, h0, t, nb);
      float acc[CBN / 2];
      wg_mainloop<TA, CBN, CL, Cfg::kTaps>(acc, smem_a, A_BYTES, cw * 64 * 128, smem_b, B_BYTES, full_bar, empty_bar,
                                          STAGES, k_iters, stage, phase, lane, rank ^ 1u);
      if (!valid) continue;   // (the dummy tile's nb == g.nb has no scale)
      if constexpr (sizeof(TA) == 1) dequant_frag_vol<CBN>(acc, __ldg(p.a_scale + nb), p.w_scale, n_blk * CBN, g.c_out, lane);
      TileGeom tg;
      tg.bw = HALO ? 128 : g.bw; tg.rows = HALO ? 128 : g.bw * g.bh;
      tg.w_lim = g.w - w0; tg.h_lim = HALO ? 1 : g.h - h0; tg.img_w = g.w;
      const int m_base = ((nb * g.t_out + t) * g.h + h0) * g.w + w0;
      drain_tile<T, EPI, CBN>(acc, stg, m_base, wrow, 0, n_blk * CBN, g.c_out, p, lane, tg);
    }
  }
  if constexpr (CL == 2) cluster_sync_all();
}

int make_tmap_nd(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, int elem_bytes);   // host.cu

extern int g_conv_2cta, g_conv_halo;

template <typename TA, typename T, int EPI, int CBN>
static int launch_conv(const dwm_conv_args* a, cudaStream_t stream) {
  constexpr int eb = static_cast<int>(sizeof(TA));
  constexpr uint32_t BKE = CV_ROW_BYTES / eb;
  ConvGeom g;
  g.nb = static_cast<int>(a->nb);
  g.kt = a->kt; g.kh = a->kh; g.kw = a->kw;
  g.t_out = static_cast<int>(a->tp) - a->kt + 1;
  g.h = static_cast<int>(a->h); g.w = static_cast<int>(a->w);
  g.c_in = static_cast<int>(a->c_in); g.c_out = static_cast<int>(a->c_out);
  g.bw = g.w < 128 ? g.w : 128;
  g.bh = 128 / g.bw;
  if (g.bh > g.h) g.bh = g.h;
  if (g.bh < 1) g.bh = 1;
  g.tiles_w = (g.w + g.bw - 1) / g.bw;
  g.tiles_h = (g.h + g.bh - 1) / g.bh;

  CUtensorMap tx, tw;
  const uint64_t dims[5] = {static_cast<uint64_t>(a->c_in), static_cast<uint64_t>(a->w), static_cast<uint64_t>(a->h),
                            static_cast<uint64_t>(a->tp), static_cast<uint64_t>(a->nb)};
  const uint64_t st[4] = {static_cast<uint64_t>(a->c_in) * eb, static_cast<uint64_t>(a->c_in) * a->w * eb,
                          static_cast<uint64_t>(a->c_in) * a->w * a->h * eb,
                          static_cast<uint64_t>(a->c_in) * a->w * a->h * a->tp * eb};
  const uint32_t box[5] = {BKE, static_cast<uint32_t>(g.bw), static_cast<uint32_t>(g.bh), 1, 1};
  int rc = make_tmap_nd(&tx, a->x, 5, dims, st, box, eb);
  if (rc) return rc;
  const int taps = a->kt * a->kh * a->kw;
  rc = make_tmap_2d(&tw, a->weight, static_cast<uint64_t>(taps) * a->c_out, a->c_in, a->c_in, CBN, BKE, eb);
  if (rc) return rc;

  EpiParams p = {};
  p.out = a->out; p.ldo = a->ldo; p.bias = a->bias; p.act = a->act;
  p.resid = a->resid; p.ldr = a->ldr;
  p.resid_row_mod = a->resid_per_item ? -1 : 0;
  // rows_per_item only picks the residual row; the 16-bit store must not remap its rows by it
  p.rows_per_item = EPI == DWM_EPI_RESID ? a->rows_per_item : 0;
  p.blend_x = a->blend_x; p.ldx = a->ldx; p.alpha = a->alpha; p.rows_per_batch = a->rows_per_batch;
  p.norm_regions = 2;
  p.n_peers = 0;
  p.a_scale = a->a_scale;
  p.w_scale = a->w_scale;

  const long long n_blocks = (g.c_out + CBN - 1) / CBN;
  const long long m_tiles = static_cast<long long>(g.nb) * g.t_out * g.tiles_w * g.tiles_h;
  const long long seg_tiles = static_cast<long long>(g.nb) * g.t_out * g.h * ((g.w + 127) / 128);
  const int sms = sm_count();
  if (g_conv_2cta < 0) {
    const char* e = getenv("DWM_CONV_2CTA");
    g_conv_2cta = (e && e[0] == '0') ? 0 : 1;
  }
  if (g_conv_halo < 0) {
    const char* e = getenv("DWM_CONV_HALO");
    g_conv_halo = (e && e[0] == '0') ? 0 : 1;
  }
  // shared-memory opt-in once per kernel instantiation (one flag per variant)
  static bool attr_halo = false, attr_pair = false, attr_one = false;
  auto go = [&](auto kern, bool& attr_set, int smem_bytes, int cl, long long mt, const CUtensorMap& x,
                const CUtensorMap& w) -> int {
    if (!attr_set) {
      DWM_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
      attr_set = true;
    }
    const long long tiles = ((mt + cl - 1) / cl) * n_blocks;
    const long long slots = sms / cl;
    const int grid = cl * static_cast<int>(tiles < slots ? tiles : slots);
    if (cl == 1) kern<<<grid, GEMM_THREADS, smem_bytes, stream>>>(x, w, g, p);
    else DWM_CHECK_CUDA(launch_cluster2(kern, grid, GEMM_THREADS, smem_bytes, stream, x, w, g, p));
    DWM_CHECK_CUDA(cudaGetLastError());
    return 0;
  };
  if constexpr (CBN <= 128) {
    // halo-row kernel: kw = 3, rows of at least 128 pixels, enough row segments for the SMs
    // (C_out tiles of 256 columns: three weight slices per stage would not fit)
    if (g_conv_halo == 1 && a->kw == 3 && g.w >= 128 && seg_tiles * n_blocks >= sms) {
      CUtensorMap txh;
      const uint32_t boxh[5] = {BKE, static_cast<uint32_t>(CVH_A_ROWS), 1, 1, 1};
      rc = make_tmap_nd(&txh, a->x, 5, dims, st, boxh, eb);
      if (rc) return rc;
      return go(conv_wgmma_kernel<TA, T, EPI, CBN, 1, true>, attr_halo, ConvCfg<CBN, true>::kSmemBytes, 1, seg_tiles, txh, tw);
    }
  }
  if constexpr (CBN >= 64) {
    // pairs once there are enough pixel tiles for both CTAs of every cluster (the weight half
    // of a CTA must be whole 8-row swizzle atoms)
    if (g_conv_2cta == 1 && m_tiles * n_blocks >= 2 * sms) {
      rc = make_tmap_2d(&tw, a->weight, static_cast<uint64_t>(taps) * a->c_out, a->c_in, a->c_in, CBN / 2, BKE, eb);
      if (rc) return rc;
      return go(conv_wgmma_kernel<TA, T, EPI, CBN, 2, false>, attr_pair, ConvCfg<CBN, false>::kSmemBytes, 2, m_tiles, tx, tw);
    }
  }
  return go(conv_wgmma_kernel<TA, T, EPI, CBN, 1, false>, attr_one, ConvCfg<CBN, false>::kSmemBytes, 1, m_tiles, tx, tw);
}

int g_conv_2cta = -1;   // -1: env DWM_CONV_2CTA (default 1); option "conv_2cta"
int g_conv_halo = -1;   // -1: env DWM_CONV_HALO (default 1); option "conv_halo"

template <typename TA, typename T, int EPI>
static int conv_pick_bn(const dwm_conv_args* a, cudaStream_t s) {
  if (a->c_out % 256 == 0) return launch_conv<TA, T, EPI, 256>(a, s);
  if (a->c_out % 128 == 0) return launch_conv<TA, T, EPI, 128>(a, s);
  if (a->c_out % 64 == 0) return launch_conv<TA, T, EPI, 64>(a, s);
  if (a->c_out % 32 == 0) return launch_conv<TA, T, EPI, 32>(a, s);
  set_last_error("dwm_b200_conv: C_out must be a multiple of 32 (pad the weight rows); got %lld", (long long)a->c_out);
  return -1;
}

// E4M3 with the fp32 store (the VAE ResNet conv1): only the C_out tiles the VAE widths
// (128 / 256 / 512) select are instantiated
static int conv_pick_bn_e4m3_f32(const dwm_conv_args* a, cudaStream_t s) {
  if (a->c_out % 256 == 0) return launch_conv<__nv_fp8_e4m3, __nv_bfloat16, DWM_EPI_F32, 256>(a, s);
  if (a->c_out % 128 == 0) return launch_conv<__nv_fp8_e4m3, __nv_bfloat16, DWM_EPI_F32, 128>(a, s);
  set_last_error("dwm_b200_conv: E4M3 with DWM_EPI_F32 needs C_out %% 128 == 0; got %lld", (long long)a->c_out);
  return -1;
}

template <typename T>
static int conv_pick_epi(const dwm_conv_args* a, cudaStream_t s) {
  switch (a->epilogue) {
    case DWM_EPI_STORE: return conv_pick_bn<T, T, DWM_EPI_STORE>(a, s);
    case DWM_EPI_RESID: return conv_pick_bn<T, T, DWM_EPI_RESID>(a, s);
    case DWM_EPI_F32: return conv_pick_bn<T, T, DWM_EPI_F32>(a, s);
    default: set_last_error("dwm_b200_conv: epilogue must be STORE, RESID or F32"); return -1;
  }
}

}  // namespace dwm

extern "C" int dwm_b200_conv(const dwm_conv_args* a, dwm_stream_t stream) {
  using namespace dwm;
  DWM_REQUIRE(a != nullptr && a->x && a->weight && a->out, "dwm_b200_conv: null pointer");
  DWM_REQUIRE(a->nb > 0 && a->tp >= a->kt && a->h > 0 && a->w > 0 && a->c_in > 0 && a->c_out > 0,
              "dwm_b200_conv: bad shape");
  DWM_REQUIRE(a->kt >= 1 && a->kh >= 1 && a->kw >= 1 && a->kh % 2 == 1 && a->kw % 2 == 1,
              "dwm_b200_conv: odd spatial kernel sizes required");
  DWM_REQUIRE(a->c_in % 8 == 0, "dwm_b200_conv: C_in must be a multiple of 8 (pad the channels)");
  DWM_REQUIRE(a->ldo % 8 == 0 && (reinterpret_cast<uintptr_t>(a->x) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(a->weight) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->out) & 15) == 0,
              "dwm_b200_conv: alignment");
  const long long rows = a->nb * (a->tp - a->kt + 1) * a->h * a->w;
  DWM_REQUIRE(rows < (1ll << 31), "dwm_b200_conv: too many output pixels");
  if (a->epilogue != DWM_EPI_RESID)
    DWM_REQUIRE(!a->resid && !a->blend_x && !a->resid_per_item,
                "dwm_b200_conv: resid, blend_x and resid_per_item need epilogue DWM_EPI_RESID");
  if (a->blend_x) DWM_REQUIRE(a->alpha != nullptr, "dwm_b200_conv: blend_x without alpha");
  if (a->resid_per_item)
    DWM_REQUIRE(a->rows_per_item > 0, "dwm_b200_conv: resid_per_item needs rows_per_item > 0");
  // the epilogue reads bias / resid / blend_x rows as float2 / float4
  for (const void* p : {static_cast<const void*>(a->bias), static_cast<const void*>(a->resid),
                        static_cast<const void*>(a->blend_x)})
    DWM_REQUIRE((reinterpret_cast<uintptr_t>(p) & 15) == 0,
                "dwm_b200_conv: bias, resid, blend_x must be 16-byte aligned");
  DWM_REQUIRE((!a->resid || a->ldr % 4 == 0) && (!a->blend_x || a->ldx % 4 == 0),
              "dwm_b200_conv: ldr, ldx must be multiples of 4 (16-byte rows); got %lld %lld",
              (long long)a->ldr, (long long)a->ldx);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (a->dtype == DWM_BF16) return conv_pick_epi<__nv_bfloat16>(a, s);
  if (a->dtype == DWM_F16) return conv_pick_epi<__half>(a, s);
  if (a->dtype == DWM_E4M3) {
    DWM_REQUIRE(a->epilogue == DWM_EPI_RESID || a->epilogue == DWM_EPI_F32,
                "dwm_b200_conv: E4M3 operands need epilogue DWM_EPI_RESID or DWM_EPI_F32, got %d", a->epilogue);
    DWM_REQUIRE(a->a_scale && a->w_scale, "dwm_b200_conv: E4M3 operands need a_scale [nb] and w_scale [c_out]");
    DWM_REQUIRE(a->c_in % 16 == 0, "dwm_b200_conv: E4M3 needs C_in %% 16 == 0 (16-byte TMA pitch); got %lld",
                (long long)a->c_in);
    DWM_REQUIRE((reinterpret_cast<uintptr_t>(a->w_scale) & 7) == 0, "dwm_b200_conv: w_scale must be 8-byte aligned");
    // the fp32-output epilogues never name their 16-bit type
    if (a->epilogue == DWM_EPI_F32) return conv_pick_bn_e4m3_f32(a, s);
    return conv_pick_bn<__nv_fp8_e4m3, __nv_bfloat16, DWM_EPI_RESID>(a, s);
  }
  set_last_error("dwm_b200_conv: dtype must be DWM_BF16, DWM_F16 or DWM_E4M3");
  return -1;
}
