// wgmma flash attention (sm_90a) for head_dim-64 sequences: S = Q.K^T and O += P.V on the
// warpgroup MMA with S, P and O held in registers.
//
//   warpgroup 0     TMA producer (one elected thread): Q tile of 128 rows (single buffer) and
//                   K / V blocks of 128 keys through a 3-stage ring
//   warpgroups 1-2  consumers, 64 query rows each: S = Q.K_blk^T (wgmma m64n128k16, both
//                   operands from shared memory), online softmax on the accumulator fragment
//                   (a row lives in the 4 lanes of a quad), P packed to 16 bit in registers
//                   and used directly as the A operand of O += P.V_blk (wgmma m64n64k16, V
//                   MN-major in shared memory)
//
// Gathered sequences (template flag G): cross-view row-wise attention
// "(bt v) (h w) c -> (bt h) (v w) c" with its [B,V,V] view mask, and temporal row-wise
// attention "(b t v) (h w) c -> (b v h) (t w) c" run on the same pipeline.  A sequence is
// n_out "outer" units (views / frames) of `inner` contiguous tokens (one latent row); a 5-D
// tensor map (col, w, outer, g1, g0) lets ONE bulk tensor load fetch a tile of `upt` whole
// units (upt * inner <= 128 rows) straight from the un-permuted q|k|v buffer — the
// reference's two 264 MB permutes and its [512,168,168] mask never exist.  The view mask is
// a per-row bit set over key units, expanded once per key block to a 128-bit column mask.
//
// Separate K,V (template flag SKV, gathered sequences only): queries are the local views of a
// view shard, keys / values the gathered views of every rank in a second buffer with its own
// 5-D tensor map.  Key blocks, their unit count `upt` and the mask columns are those of the
// unsharded launch, and query unit u reads mask row mask_q0 + u, so each local query row sees
// the same key blocks in the same order with the same arithmetic as its row of the unsharded
// launch: its output is bit-identical.
//
// Text encoders (template flags CAUSAL, BIAS; contiguous sequences only): CLIP's causal mask
// drops key j > query i; T5's relative-position bias [heads, seq, seq] (fp32, shared by every
// group) is added to the scaled scores, which are then kept in log2 units, s*scale*log2(e) +
// bias*log2(e), so the softmax below runs with a unit scale.
#include <string.h>

#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/dwm_b200.h"

namespace dwm {

namespace fa {
constexpr int BQ = 128, BK = 128, HD = 64;
constexpr int KV_STAGES = 3;
constexpr int TILE = 128 * 64 * 2;            // one 128-row x 64-col 16-bit tile
constexpr int THREADS = 384;                  // warpgroup 0: TMA; warpgroups 1, 2: consumers
constexpr int CONSUMER_WARPS = 8;
constexpr int TILES_BYTES = TILE /*Q*/ + KV_STAGES * 2 * TILE /*K,V*/;
constexpr int SMEM_BYTES = 1024 + TILES_BYTES + 256 /*barriers*/;
}  // namespace fa

struct FaParams {
  int groups, heads, seq, q_tiles, n_kb;
  long long group_stride;
  int D;
  void* out; long long ldo; long long out_group_stride;
  int split; void* out2; long long ldo2;
  float scale_log2;
  // gathered sequences (G): group g = g0 * g1n + i1
  int inner, n_out, upt, g1n;
  long long out_gs1, out_so;
  const unsigned char* mask; int mask_div, mask_n;
  // key / value columns of head 0 (in the qkv map, or in the K,V map with SKV), key units
  // (n_out without SKV) and the mask row of query unit 0
  int kcol, vcol, n_out_k, mask_q0;
  const float* bias;   // BIAS: [heads, seq, seq]
};

// Descriptor of an MN-major operand (V: keys x head_dim, head_dim contiguous) written by TMA
// with 128-byte swizzle.  head_dim 64 is exactly one swizzle atom wide, so only the stride
// between 8-key groups matters; it is given in both offset fields.
__device__ __forceinline__ uint64_t gmma_desc_sw128_mn(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1024 >> 4) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <typename T, bool G, bool SKV, bool CAUSAL, bool BIAS>
__global__ void __launch_bounds__(fa::THREADS, 1)
    attn_wgmma_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap_kv,
                      const FaParams p) {
  using namespace fa;
  static_assert(G || !SKV, "separate K,V needs gathered sequences");
  static_assert(!G || (!CAUSAL && !BIAS), "causal / bias attention needs contiguous sequences");
  const CUtensorMap* kvmap = SKV ? &tmap_kv : &tmap;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sq = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // Q  [16 KB]
  uint8_t* skv = sq + TILE;                                                     // [stages][K | V]
  uint64_t* bars = reinterpret_cast<uint64_t*>(skv + KV_STAGES * 2 * TILE);
  uint64_t* q_full = bars;                    // [1]
  uint64_t* q_empty = bars + 1;               // [1]
  uint64_t* kv_full = bars + 2;               // [KV_STAGES]
  uint64_t* kv_empty = bars + 2 + KV_STAGES;  // [KV_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int n_items = p.groups * p.heads * p.q_tiles;
  // G: a tile holds upt * inner <= 128 rows; the rows behind them are never written by TMA and
  // must be finite (P = 0 times a stale NaN in V would poison O): zero all tiles once
  const uint32_t tile_tx = G ? static_cast<uint32_t>(p.upt * p.inner * 128) : static_cast<uint32_t>(TILE);
  if constexpr (G) {
    uint4* z = reinterpret_cast<uint4*>(sq);
    for (int i = threadIdx.x; i < TILES_BYTES / 16; i += THREADS) z[i] = make_uint4(0u, 0u, 0u, 0u);
    fence_proxy_async();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap);
    if constexpr (SKV) tma_prefetch_desc(&tmap_kv);
    mbar_init(q_full, 1);
    mbar_init(q_empty, CONSUMER_WARPS);
    for (int i = 0; i < KV_STAGES; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();

  auto decode = [&](int w, int& g, int& h, int& qt) {
    h = w % p.heads;
    const int r = w / p.heads;
    qt = r % p.q_tiles;
    g = r / p.q_tiles;
  };

  if (wg == 0) {
    setmaxnreg_dec<24>();
    // ================= TMA producer =================
    if (warp == 0 && elect_one()) {
      int it = 0, kvs = 0;
      uint32_t kvph = 0;
      for (int w = blockIdx.x; w < n_items; w += gridDim.x, ++it) {
        int g, h, qt;
        decode(w, g, h, qt);
        const int row0 = static_cast<int>(g * p.group_stride);
        const int g0 = G ? g / p.g1n : 0, i1 = G ? g - g0 * p.g1n : 0;
        // the NEXT item's Q / K / V boxes start their trip from HBM to L2 now: its loads can
        // only be issued once this item's P.V has released the K,V stages
        if (w + static_cast<int>(gridDim.x) < n_items) {
          int g2, h2, qt2;
          decode(w + gridDim.x, g2, h2, qt2);
          if constexpr (G) {
            const int g02 = g2 / p.g1n, i12 = g2 - g02 * p.g1n;
            tma_prefetch_5d(&tmap, h2 * HD, 0, qt2 * p.upt, i12, g02);
            for (int kb = 0; kb < p.n_kb; ++kb) {
              tma_prefetch_5d(kvmap, p.kcol + h2 * HD, 0, kb * p.upt, i12, g02);
              tma_prefetch_5d(kvmap, p.vcol + h2 * HD, 0, kb * p.upt, i12, g02);
            }
          } else {
            const int r2 = static_cast<int>(g2 * p.group_stride);
            tma_prefetch_2d(&tmap, h2 * HD, r2 + qt2 * BQ);
            for (int kb = 0; kb < p.n_kb; ++kb) {
              tma_prefetch_2d(&tmap, p.kcol + h2 * HD, r2 + kb * BK);
              tma_prefetch_2d(&tmap, p.vcol + h2 * HD, r2 + kb * BK);
            }
          }
        }
        mbar_wait(q_empty, (it & 1) ^ 1);
        mbar_expect_tx(q_full, tile_tx);
        if constexpr (G) tma_load_5d(&tmap, q_full, sq, h * HD, 0, qt * p.upt, i1, g0, kEvictFirst);
        else tma_load_2d(&tmap, q_full, sq, h * HD, row0 + qt * BQ, kEvictFirst);
        for (int kb = 0; kb < p.n_kb; ++kb) {
          mbar_wait(&kv_empty[kvs], kvph ^ 1);
          mbar_expect_tx(&kv_full[kvs], 2 * tile_tx);
          uint8_t* st = skv + kvs * 2 * TILE;
          if constexpr (G) {
            tma_load_5d(kvmap, &kv_full[kvs], st, p.kcol + h * HD, 0, kb * p.upt, i1, g0, kEvictLast);
            tma_load_5d(kvmap, &kv_full[kvs], st + TILE, p.vcol + h * HD, 0, kb * p.upt, i1, g0, kEvictLast);
          } else {
            tma_load_2d(&tmap, &kv_full[kvs], st, p.kcol + h * HD, row0 + kb * BK, kEvictLast);
            tma_load_2d(&tmap, &kv_full[kvs], st + TILE, p.vcol + h * HD, row0 + kb * BK, kEvictLast);
          }
          if (++kvs == KV_STAGES) { kvs = 0; kvph ^= 1; }
        }
      }
    }
  } else {
    setmaxnreg_inc<240>();
    // ================= consumers: 64 query rows per warpgroup =================
    const int cw = wg - 1;
    const int quad_col = 2 * (lane & 3);                       // first fragment column of this lane
    const int rows[2] = {cw * 64 + (warp & 3) * 16 + (lane >> 2), cw * 64 + (warp & 3) * 16 + (lane >> 2) + 8};
    const float sc = p.scale_log2;
    const float sc_s = BIAS ? 1.0f : sc;   // scale still to apply to the (biased) scores
    const uint64_t dq = gmma_desc_sw128(smem_u32(sq + cw * 64 * 128));
    int kvs = 0, it = 0;
    uint32_t kvph = 0;
    for (int w = blockIdx.x; w < n_items; w += gridDim.x, ++it) {
      int g, h, qt;
      decode(w, g, h, qt);
      // G: a row's query token = (outer unit qo, token wi of the unit); `allowed` = key units it
      // may attend to (the [B,V,V] mask row; everything for padding rows)
      int qo[2] = {0, 0}, wi[2] = {0, 0};
      bool row_ok[2] = {true, true};
      uint32_t allowed[2] = {0xffffffffu, 0xffffffffu};
      if constexpr (G) {
#pragma unroll
        for (int hi = 0; hi < 2; ++hi) {
          const int u = rows[hi] / p.inner;
          wi[hi] = rows[hi] - u * p.inner;
          qo[hi] = qt * p.upt + u;
          row_ok[hi] = u < p.upt && qo[hi] < p.n_out;
          if (p.mask && row_ok[hi]) {
            const int g0 = g / p.g1n;
            const unsigned char* mr =
                p.mask + (static_cast<long long>(g0 / p.mask_div) * p.mask_n + p.mask_q0 + qo[hi]) * p.mask_n;
            uint32_t al = 0u;
            for (int ko = 0; ko < p.n_out_k; ++ko) al |= (__ldg(mr + ko) != 0 ? 1u : 0u) << ko;
            allowed[hi] = al;
          }
        }
      }
      // CAUSAL / BIAS: sequence position of each row; a padding row (>= seq) reads the bias row
      // of the last query, its output is never stored
      int qpos[2] = {0, 0};
      const float* brow[2] = {nullptr, nullptr};
      if constexpr (CAUSAL || BIAS) {
#pragma unroll
        for (int hi = 0; hi < 2; ++hi) {
          qpos[hi] = qt * BQ + rows[hi];
          if constexpr (BIAS)
            brow[hi] = p.bias + (static_cast<long long>(h) * p.seq + min(qpos[hi], p.seq - 1)) * p.seq;
        }
      }
      float o[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] = 0.f;
      float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
      mbar_wait(q_full, it & 1);
      for (int kb = 0; kb < p.n_kb; ++kb) {
        const int kvalid = p.seq - kb * BK;   // keys < kvalid are real (contiguous sequences)
        uint32_t cmw[2][4];
        if constexpr (G) {
          // 128-bit column mask of this key block per row: unit u2 covers columns [u2*inner, (u2+1)*inner)
          const unsigned __int128 ones = p.inner >= 128 ? ~static_cast<unsigned __int128>(0)
                                                        : ((static_cast<unsigned __int128>(1) << p.inner) - 1);
#pragma unroll
          for (int hi = 0; hi < 2; ++hi) {
            unsigned __int128 cm = 0;
            for (int u2 = 0; u2 < p.upt; ++u2) {
              const int ko = kb * p.upt + u2;
              if (ko < p.n_out_k && ((allowed[hi] >> ko) & 1u)) cm |= ones << (u2 * p.inner);
            }
            cmw[hi][0] = static_cast<uint32_t>(cm);
            cmw[hi][1] = static_cast<uint32_t>(cm >> 32);
            cmw[hi][2] = static_cast<uint32_t>(cm >> 64);
            cmw[hi][3] = static_cast<uint32_t>(cm >> 96);
          }
        }
        mbar_wait(&kv_full[kvs], kvph);
        const uint32_t sk = smem_u32(skv + kvs * 2 * TILE);
        // ---- S = Q K^T ----
        float s[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) s[i] = 0.f;
        fence_operands(s);
        wgmma_fence();
        const uint64_t dk = gmma_desc_sw128(sk);
#pragma unroll
        for (int k = 0; k < HD / 16; ++k) Wgmma<128, T>::ss(s, dq + 2 * k, dk + 2 * k, 1u);
        wgmma_commit();
        wgmma_wait<0>();
        fence_operands(s);
        if (kb == p.n_kb - 1) {   // Q tile fully consumed
          __syncwarp();
          if (lane == 0) mbar_arrive(q_empty);
        }
        // ---- online softmax on the fragment: s[4j + e] = row rows[e >> 1], column 8j + quad_col + (e & 1)
        const bool full = !G && !CAUSAL && !BIAS && kvalid >= BK;   // only the last block of a contiguous sequence is ragged
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int col = 8 * j + quad_col + (e & 1);
            const int hi = e >> 1;
            if (!full) {
              bool ok = G ? ((cmw[hi][col >> 5] >> (col & 31)) & 1u) != 0u : col < kvalid;
              if constexpr (CAUSAL) ok = ok && kb * BK + col <= qpos[hi];
              if (!ok) s[4 * j + e] = -INFINITY;
              else if constexpr (BIAS)
                s[4 * j + e] = fmaf(s[4 * j + e], sc, __ldg(brow[hi] + kb * BK + col) * 1.4426950408889634f);
            }
            mx[hi] = fmaxf(mx[hi], s[4 * j + e]);
          }
        float mref[2], corr[2];
#pragma unroll
        for (int hi = 0; hi < 2; ++hi) {
          mx[hi] = fmaxf(mx[hi], __shfl_xor_sync(0xffffffffu, mx[hi], 1));
          mx[hi] = fmaxf(mx[hi], __shfl_xor_sync(0xffffffffu, mx[hi], 2));
          const float m_new = fmaxf(m[hi], mx[hi] * sc_s);
          // a row whose keys were all masked so far (m_new = -inf, G only) keeps l = 0 / O = 0
          corr[hi] = m_new == -INFINITY ? 1.0f : ex2_approx(m[hi] - m_new);
          m[hi] = m_new;
          mref[hi] = m_new == -INFINITY ? 0.f : m_new;
          l[hi] *= corr[hi];
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) o[i] *= corr[(i >> 1) & 1];
        // p = exp2(s*scale - m), packed to 16 bit in the A-operand layout of m64n64k16:
        // k step kk covers key columns [16kk, 16kk + 16) = n8 blocks 2kk, 2kk + 1
        uint32_t pa[8][4];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          float pv[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            pv[e] = ex2_approx(fmaf(s[4 * j + e], sc_s, -mref[e >> 1]));
            l[e >> 1] += pv[e];
          }
          pa[j >> 1][(j & 1) * 2] = Cvt<T>::pack2(pv[0], pv[1]);
          pa[j >> 1][(j & 1) * 2 + 1] = Cvt<T>::pack2(pv[2], pv[3]);
        }
        // ---- O += P V ----
        fence_operands(o);
        wgmma_fence();
        const uint32_t sv = sk + TILE;
#pragma unroll
        for (int kk = 0; kk < BK / 16; ++kk) Wgmma<64, T>::rs(o, pa[kk], gmma_desc_sw128_mn(sv + kk * 2048), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        fence_operands(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(&kv_empty[kvs]);
        if (++kvs == KV_STAGES) { kvs = 0; kvph ^= 1; }
      }
      // ---- out = O / l ----
#pragma unroll
      for (int hi = 0; hi < 2; ++hi) {
        l[hi] += __shfl_xor_sync(0xffffffffu, l[hi], 1);
        l[hi] += __shfl_xor_sync(0xffffffffu, l[hi], 2);
        const int row = rows[hi];
        const int j = qt * BQ + row;
        if (!(G ? row_ok[hi] : (j < p.seq))) continue;
        // a query whose every key is masked (G only) has l = 0 and O = 0: write 0, not 0 * inf
        const float inv = l[hi] > 0.f ? 1.0f / l[hi] : 0.f;
        T* dst;
        if constexpr (G) {
          const int g0 = g / p.g1n, i1 = g - g0 * p.g1n;
          dst = reinterpret_cast<T*>(p.out) +
                (static_cast<long long>(g0) * p.out_group_stride + static_cast<long long>(i1) * p.out_gs1 +
                 static_cast<long long>(qo[hi]) * p.out_so + wi[hi]) * p.ldo;
        } else if (p.split > 0 && j >= p.split) {
          dst = reinterpret_cast<T*>(p.out2) + (static_cast<long long>(g) * (p.seq - p.split) + (j - p.split)) * p.ldo2;
        } else {
          dst = reinterpret_cast<T*>(p.out) + (static_cast<long long>(g) * p.out_group_stride + j) * p.ldo;
        }
        dst += h * HD + quad_col;
#pragma unroll
        for (int jn = 0; jn < 8; ++jn)
          *reinterpret_cast<uint32_t*>(dst + 8 * jn) = Cvt<T>::pack2(o[4 * jn + 2 * hi] * inv, o[4 * jn + 2 * hi + 1] * inv);
      }
    }
  }
}

template <typename T, bool G, bool SKV, bool CAUSAL = false, bool BIAS = false>
static int launch_attn_wgmma(const dwm_attention_args* a, cudaStream_t s, const float* bias = nullptr) {
  using namespace fa;
  FaParams p;
  memset(&p, 0, sizeof(p));
  CUtensorMap tm, tm_kv;
  long long groups;
  p.kcol = static_cast<int>(SKV ? a->k_col : a->D);
  p.vcol = static_cast<int>(SKV ? a->v_col : 2 * a->D);
  if (G) {
    // merge the (optional) third group dim into the second: row offset i1*gs1 + i2*gs2 with
    // gs1 == gd2*gs2 is (i1*gd2 + i2)*gs2 (checked by attn_tcg_eligible)
    const long long gd1 = a->group_dims[1] * a->group_dims[2];
    const long long gs1 = a->group_dims[2] > 1 ? a->group_strides[2] : a->group_strides[1];
    const long long ogs1 = a->group_dims[2] > 1 ? a->out_group_strides[2] : a->out_group_strides[1];
    p.inner = a->inner;
    p.n_out = a->seq / a->inner;
    p.n_out_k = SKV ? a->seq_kv / a->inner_kv : p.n_out;
    // key blocks of `upt` units, as many as the unsharded launch over all n_out_k units takes
    p.upt = 128 / a->inner;
    if (p.upt > p.n_out_k) p.upt = p.n_out_k;
    p.g1n = static_cast<int>(gd1);
    p.out_gs1 = ogs1;
    p.out_so = a->out_stride_outer;
    p.mask = a->mask; p.mask_div = a->mask_div; p.mask_n = a->n_outer; p.mask_q0 = a->mask_q_offset;
    groups = a->group_dims[0] * gd1;
    const uint64_t eb = 2;
    const uint32_t box[5] = {64u, static_cast<uint32_t>(a->inner), static_cast<uint32_t>(p.upt), 1u, 1u};
    if (SKV) {
      const long long kgs1 = a->group_dims[2] > 1 ? a->kv_group_strides[2] : a->kv_group_strides[1];
      const long long kcols = (a->k_col > a->v_col ? a->k_col : a->v_col) + a->D;
      const uint64_t kdims[5] = {static_cast<uint64_t>(kcols), static_cast<uint64_t>(a->inner_kv),
                                 static_cast<uint64_t>(p.n_out_k), static_cast<uint64_t>(gd1),
                                 static_cast<uint64_t>(a->group_dims[0])};
      const uint64_t kst[4] = {static_cast<uint64_t>(a->ld_kv) * eb,
                               static_cast<uint64_t>(a->kv_stride_outer * a->ld_kv) * eb,
                               static_cast<uint64_t>(kgs1 * a->ld_kv) * eb,
                               static_cast<uint64_t>(a->kv_group_strides[0] * a->ld_kv) * eb};
      int rc = make_tmap_nd(&tm_kv, a->kv, 5, kdims, kst, box, 2);
      if (rc) return rc;
    }
    const uint64_t dims[5] = {static_cast<uint64_t>(SKV ? a->D : 3 * a->D), static_cast<uint64_t>(a->inner),
                              static_cast<uint64_t>(p.n_out), static_cast<uint64_t>(gd1),
                              static_cast<uint64_t>(a->group_dims[0])};
    const uint64_t st[4] = {static_cast<uint64_t>(a->ld) * eb, static_cast<uint64_t>(a->stride_outer * a->ld) * eb,
                            static_cast<uint64_t>(gs1 * a->ld) * eb,
                            static_cast<uint64_t>(a->group_strides[0] * a->ld) * eb};
    int rc = make_tmap_nd(&tm, a->qkv, 5, dims, st, box, 2);
    if (rc) return rc;
    p.q_tiles = (p.n_out + p.upt - 1) / p.upt;
    p.n_kb = (p.n_out_k + p.upt - 1) / p.upt;
  } else {
    groups = a->group_dims[0];
    const long long rows_total = groups * a->group_strides[0];
    int rc = make_tmap_2d(&tm, a->qkv, rows_total, 3 * a->D, a->ld, 128, 64, 2);
    if (rc) return rc;
    p.q_tiles = (a->seq + BQ - 1) / BQ;
    p.n_kb = (a->seq + BK - 1) / BK;
  }
  p.groups = static_cast<int>(groups);
  p.heads = a->heads;
  p.seq = a->seq;
  p.group_stride = a->group_strides[0];
  p.D = static_cast<int>(a->D);
  p.out = a->out; p.ldo = a->ldo; p.out_group_stride = a->out_group_strides[0];
  p.split = a->split; p.out2 = a->out2; p.ldo2 = a->ldo2;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.bias = bias;
  if (!SKV) tm_kv = tm;
  auto kern = attn_wgmma_kernel<T, G, SKV, CAUSAL, BIAS>;
  static bool attr_set = false;
  if (!attr_set) {
    DWM_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    attr_set = true;
  }
  const long long items = groups * a->heads * p.q_tiles;
  const long long slots = sm_count();
  const int grid = static_cast<int>(items < slots ? items : slots);
  kern<<<grid, THREADS, SMEM_BYTES, s>>>(tm, tm_kv, p);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// contiguous, unmasked head_dim-64 sequences (joint / dual attention, UNet spatial attention)
// packed back to back: the 2-D tensor map loads whole 128-row K / V blocks, so the rows after a
// sequence must be the next sequence or the map's zero fill.  Padding rows between sequences
// could hold anything, and P = 0 times a NaN / Inf there would still reach O; such layouts go to
// the mma.sync kernel, which zero-fills out-of-sequence rows.
bool attn_tc_eligible(const dwm_attention_args* a) {
  return a->kv == nullptr && a->mask == nullptr && a->group_dims[1] == 1 && a->group_dims[2] == 1 &&
         a->inner == a->seq && a->stride_inner == 1 && a->out_stride_inner == 1 && a->seq > 64 &&
         a->group_strides[0] == a->seq && a->group_dims[0] * a->group_strides[0] < (1ll << 31);
}

// causal or biased attention (text encoders): the contiguous layout of attn_tc_eligible at any
// seq >= 1 (a short sequence's 128-row tiles hold the next sequences' rows, which the key
// mask drops and whose query rows are not stored), no split
bool attn_text_eligible(const dwm_attention_args* a) {
  return a->kv == nullptr && a->mask == nullptr &&
         a->split == 0 && a->group_dims[1] == 1 && a->group_dims[2] == 1 && a->inner == a->seq &&
         a->stride_inner == 1 && a->out_stride_inner == 1 && a->group_strides[0] == a->seq &&
         a->group_dims[0] * a->group_strides[0] < (1ll << 31) &&
         static_cast<long long>(a->heads) * a->seq * a->seq < (1ll << 31);
}

// gathered sequences of whole units of `inner` contiguous tokens (cross-view / temporal
// row-wise), optional [B, n_outer, n_outer] unit mask
bool attn_tcg_eligible(const dwm_attention_args* a) {
  if (a->kv != nullptr || a->split > 0 || a->seq <= 64 || a->inner <= 0 || a->inner > 128) return false;
  if (a->inner == a->seq && a->mask == nullptr) return false;      // contiguous: the 2-D path
  if (a->seq % a->inner || a->stride_inner != 1 || a->out_stride_inner != 1) return false;
  const long long n_out = a->seq / a->inner;
  if (n_out > 32) return false;      // unit masks are 32-bit sets
  if (a->mask && a->n_outer != n_out) return false;
  if (a->group_dims[2] > 1 &&
      (a->group_strides[1] != a->group_dims[2] * a->group_strides[2] ||
       a->out_group_strides[1] != a->group_dims[2] * a->out_group_strides[2]))
    return false;
  if (a->stride_outer <= 0 || a->group_strides[0] <= 0) return false;
  const long long groups = a->group_dims[0] * a->group_dims[1] * a->group_dims[2];
  return groups * a->heads * 8 < (1ll << 31);
}

// local query units of a view shard against the gathered units of every view in a separate K,V
// buffer, with the [B, n_outer, n_outer] unit mask (cross-view row-wise attention under a view
// plan).  The key side must be a sequence the unsharded launch runs here (attn_tcg_eligible with
// the key geometry), so the key blocks are the same.  Separate K,V without a mask (frame-sharded
// temporal attention, text cross-attention) stays on the mma.sync kernel.
bool attn_tcg_kv_eligible(const dwm_attention_args* a) {
  if (a->kv == nullptr || a->mask == nullptr || a->split > 0) return false;
  if (a->inner <= 0 || a->inner > 128 || a->inner_kv != a->inner || a->seq_kv <= 64) return false;
  if (a->seq % a->inner || a->seq_kv % a->inner_kv || a->stride_inner != 1 || a->out_stride_inner != 1 ||
      a->kv_stride_inner != 1)
    return false;
  const long long n_out_k = a->seq_kv / a->inner_kv;
  if (n_out_k > 32 || a->n_outer != n_out_k) return false;
  if (a->k_col + a->D > a->ld_kv || a->v_col + a->D > a->ld_kv || a->D > a->ld) return false;
  if (a->group_dims[2] > 1 &&
      (a->group_strides[1] != a->group_dims[2] * a->group_strides[2] ||
       a->out_group_strides[1] != a->group_dims[2] * a->out_group_strides[2] ||
       a->kv_group_strides[1] != a->group_dims[2] * a->kv_group_strides[2]))
    return false;
  if (a->stride_outer <= 0 || a->group_strides[0] <= 0 || a->kv_stride_outer <= 0 || a->kv_group_strides[0] <= 0)
    return false;
  const long long groups = a->group_dims[0] * a->group_dims[1] * a->group_dims[2];
  return groups * a->heads * 8 < (1ll << 31);
}

int attn_wgmma_launch(const dwm_attention_args* a, cudaStream_t s) {
  if (a->dtype == DWM_BF16) return launch_attn_wgmma<__nv_bfloat16, false, false>(a, s);
  if (a->dtype == DWM_F16) return launch_attn_wgmma<__half, false, false>(a, s);
  set_last_error("dwm_b200_attention: dtype must be DWM_BF16 or DWM_F16, got %d", a->dtype);
  return -1;
}

int attn_text_launch(const dwm_attention_args* a, bool causal, const float* bias, cudaStream_t s) {
  const bool bf = a->dtype == DWM_BF16;
  if (a->dtype != DWM_BF16 && a->dtype != DWM_F16) {
    set_last_error("dwm_b200_attention: dtype must be DWM_BF16 or DWM_F16, got %d", a->dtype);
    return -1;
  }
  if (causal) return bf ? launch_attn_wgmma<__nv_bfloat16, false, false, true, false>(a, s)
                        : launch_attn_wgmma<__half, false, false, true, false>(a, s);
  return bf ? launch_attn_wgmma<__nv_bfloat16, false, false, false, true>(a, s, bias)
            : launch_attn_wgmma<__half, false, false, false, true>(a, s, bias);
}

int attn_tcg_launch(const dwm_attention_args* a, cudaStream_t s) {
  if (a->dtype == DWM_BF16) return launch_attn_wgmma<__nv_bfloat16, true, false>(a, s);
  if (a->dtype == DWM_F16) return launch_attn_wgmma<__half, true, false>(a, s);
  set_last_error("dwm_b200_attention: dtype must be DWM_BF16 or DWM_F16, got %d", a->dtype);
  return -1;
}

int attn_tcg_kv_launch(const dwm_attention_args* a, cudaStream_t s) {
  if (a->dtype == DWM_BF16) return launch_attn_wgmma<__nv_bfloat16, true, true>(a, s);
  if (a->dtype == DWM_F16) return launch_attn_wgmma<__half, true, true>(a, s);
  set_last_error("dwm_b200_attention: dtype must be DWM_BF16 or DWM_F16, got %d", a->dtype);
  return -1;
}

}  // namespace dwm
