// Gathered multi-head self-attention for the regrouped CTSD attentions (head_dim 64).
//
// One kernel covers every token regrouping of the reference without materialising a
// permuted copy (the reference does two einops permutes of the whole activation per
// block, crossview_temporal_dit.py:306-315,353-361):
//   * joint text+latent attention of JointTransformerBlock (seq 602, [sample ; context])
//   * dual attn2 (seq 448)
//   * cross-view "rowwise"  (bt h) x (v w)   with the [B,V,V] view mask
//   * temporal  "pointwise" (b v hw) x t ,  "rowwise" (b v h) x (t w),  "full" (b v) x (t hw)
// Sequence position j of group g lives at row
//     row = g0*gs[0] + g1*gs[1] + g2*gs[2] + (j / inner)*so + (j % inner)*si
// of the fused [rows, 3*D] q|k|v buffer written by the QKNORM GEMM epilogue.
//
// Flash-style streaming softmax, fp32 statistics; QK^T and PV run on mma.sync
// m16n8k16.  The long contiguous and gathered-unit sequences go to the wgmma kernel of
// attention_wgmma.cu; this kernel takes the rest (pointwise temporal, separate K,V, short
// sequences).
#include <stdlib.h>

#include "common.cuh"
#include "../../include/dwm_b200.h"

namespace dwm {
extern int g_attn_tc;   // -1: from env, 0: mma.sync kernel only, >= 1: attention_wgmma.cu when eligible (gemm.cu)

constexpr int HD = 64;

struct AttnParams {
  const void* q;      // queries: row pitch ldq, head h at column h*64
  long long ldq;
  const void* kv;     // keys at column kcol0 + h*64, values at vcol0 + h*64
  long long ldkv;
  int kcol0, vcol0;
  int heads;
  int groups, G1, G2;
  long long gs0, gs1, gs2;     // query group strides
  long long kgs0, kgs1, kgs2;  // key/value group strides
  int seq, inner;              // queries
  long long so, si;
  int seq_k, inner_k;          // keys / values
  long long kso, ksi;
  void* out;
  long long ldo;
  long long ogs0, ogs1, ogs2, oso, osi;
  int split;       // tokens j >= split go to out2 (row g*(seq-split) + j-split); 0 = off
  void* out2;
  long long ldo2;
  const unsigned char* mask;  // [mask_batches, n_outer, n_outer] (1 = attend) or null
  int mask_div;               // mask batch = g0 / mask_div
  int n_outer;
  int mask_q0;                // mask row of query unit 0 (the view offset of a view shard)
  float scale_log2;           // softmax scale * log2(e)
};

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const uint32_t s = smem_u32(smem);
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(sz)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2,
                                        uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2,
                                          uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
template <typename T>
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0,
                                         uint32_t b1);
template <>
__device__ __forceinline__ void mma16816<__nv_bfloat16>(float (&c)[4], const uint32_t (&a)[4],
                                                        uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <>
__device__ __forceinline__ void mma16816<__half>(float (&c)[4], const uint32_t (&a)[4],
                                                 uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// smem tile: rows of 64 elements (128 B) = 8 chunks of 16 B, chunk index XOR (row & 7)
__device__ __forceinline__ uint32_t tile_off(int row, int chunk) {
  return static_cast<uint32_t>(row * 128 + ((chunk ^ (row & 7)) << 4));
}

__device__ __forceinline__ long long tok_row(const AttnParams& p, long long base, int j) {
  return base + static_cast<long long>(j / p.inner) * p.so + static_cast<long long>(j % p.inner) * p.si;
}
__device__ __forceinline__ long long key_row(const AttnParams& p, long long base, int j) {
  return base + static_cast<long long>(j / p.inner_k) * p.kso + static_cast<long long>(j % p.inner_k) * p.ksi;
}

// NW warps per CTA, 16 query rows per warp, KVT keys per streamed tile.
template <typename T, int NW, int KVT>
__global__ void __launch_bounds__(NW * 32, NW == 4 ? 4 : 1) attn_kernel(const AttnParams p) {
  constexpr int QROWS = NW * 16;
  constexpr int NT = NW * 32;
  __shared__ __align__(128) uint8_t sq[QROWS * 128];
  __shared__ __align__(128) uint8_t sk[2][KVT * 128];
  __shared__ __align__(128) uint8_t sv[2][KVT * 128];

  const int q_tiles = (p.seq + QROWS - 1) / QROWS;
  int bid = blockIdx.x;
  const int head = bid % p.heads;
  bid /= p.heads;
  const int qt = bid % q_tiles;
  const int g = bid / q_tiles;
  const int g2 = g % p.G2;
  const int g1 = (g / p.G2) % p.G1;
  const int g0 = g / (p.G2 * p.G1);
  const long long base = g0 * p.gs0 + g1 * p.gs1 + g2 * p.gs2;
  const long long kbase = g0 * p.kgs0 + g1 * p.kgs1 + g2 * p.kgs2;

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const T* qptr = reinterpret_cast<const T*>(p.q);
  const T* kvptr = reinterpret_cast<const T*>(p.kv);
  const int q0 = qt * QROWS;

  // ---- stage Q (gathered rows) ----
  for (int i = tid; i < QROWS * 8; i += NT) {
    const int r = i >> 3, c = i & 7;
    const int j = q0 + r;
    const bool ok = j < p.seq;
    const T* src = qptr + (ok ? tok_row(p, base, j) : 0) * p.ldq + head * HD + c * 8;
    cp_async16(sq + tile_off(r, c), src, ok);
  }
  auto load_kv = [&](int buf, int k0) {
    for (int i = tid; i < KVT * 8; i += NT) {
      const int r = i >> 3, c = i & 7;
      const int j = k0 + r;
      const bool ok = j < p.seq_k;
      const T* src = kvptr + (ok ? key_row(p, kbase, j) : 0) * p.ldkv + head * HD + c * 8;
      cp_async16(sk[buf] + tile_off(r, c), src + p.kcol0, ok);
      cp_async16(sv[buf] + tile_off(r, c), src + p.vcol0, ok);
    }
  };
  load_kv(0, 0);
  cp_async_commit();

  const int n_kv = (p.seq_k + KVT - 1) / KVT;
  const int gq = lane >> 2;  // fragment row within 8
  const int tq = lane & 3;

  // my two query rows (sequence positions) and their mask rows
  const int jq0 = q0 + warp * 16 + gq;
  const int jq1 = jq0 + 8;
  const unsigned char* mrow0 = nullptr;
  const unsigned char* mrow1 = nullptr;
  if (p.mask) {
    const unsigned char* mb = p.mask + static_cast<long long>(g0 / p.mask_div) * p.n_outer * p.n_outer;
    mrow0 = mb + (p.mask_q0 + (jq0 < p.seq ? jq0 / p.inner : 0)) * p.n_outer;
    mrow1 = mb + (p.mask_q0 + (jq1 < p.seq ? jq1 / p.inner : 0)) * p.n_outer;
  }

  uint32_t qf[4][4];
  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float mx0 = -INFINITY, mx1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  for (int kt = 0; kt < n_kv; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < n_kv) load_kv(buf ^ 1, (kt + 1) * KVT);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    if (kt == 0) {
      // Q fragments (A operand, 4 k-steps of 16)
      const uint32_t sqa = smem_u32(sq);
      const int mi = lane >> 3, r8 = lane & 7;
      const int row = warp * 16 + r8 + (mi & 1) * 8;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
        ldsm_x4(sqa + tile_off(row, ks * 2 + (mi >> 1)), qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
    }
    // ---- S = Q K^T ----
    float s[KVT / 8][4];
#pragma unroll
    for (int i = 0; i < KVT / 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
    const uint32_t ska = smem_u32(sk[buf]);
    {
      const int mi = lane >> 3, r8 = lane & 7;
#pragma unroll
      for (int np = 0; np < KVT / 16; ++np) {
        const int krow = np * 16 + (mi >> 1) * 8 + r8;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          uint32_t b0, b1, b2, b3;
          ldsm_x4(ska + tile_off(krow, ks * 2 + (mi & 1)), b0, b1, b2, b3);
          mma16816<T>(s[np * 2], qf[ks], b0, b1);
          mma16816<T>(s[np * 2 + 1], qf[ks], b2, b3);
        }
      }
    }
    // ---- mask + online softmax (rows gq and gq+8) ----
    const int k0 = kt * KVT;
    float tmax0 = -INFINITY, tmax1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < KVT / 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int jk = k0 + nt * 8 + tq * 2 + e;
        bool ok0 = jk < p.seq_k, ok1 = ok0;
        if (p.mask && ok0) {
          const int vo = jk / p.inner_k;
          ok0 = mrow0[vo] != 0;
          ok1 = mrow1[vo] != 0;
        }
        s[nt][e] = ok0 ? s[nt][e] * p.scale_log2 : -INFINITY;
        s[nt][2 + e] = ok1 ? s[nt][2 + e] * p.scale_log2 : -INFINITY;
        tmax0 = fmaxf(tmax0, s[nt][e]);
        tmax1 = fmaxf(tmax1, s[nt][2 + e]);
      }
    }
    tmax0 = fmaxf(tmax0, __shfl_xor_sync(0xffffffffu, tmax0, 1));
    tmax0 = fmaxf(tmax0, __shfl_xor_sync(0xffffffffu, tmax0, 2));
    tmax1 = fmaxf(tmax1, __shfl_xor_sync(0xffffffffu, tmax1, 1));
    tmax1 = fmaxf(tmax1, __shfl_xor_sync(0xffffffffu, tmax1, 2));
    const float nm0 = fmaxf(mx0, tmax0), nm1 = fmaxf(mx1, tmax1);
    // guard fully-masked prefixes: keep exponent arguments finite
    const float ref0 = nm0 == -INFINITY ? 0.f : nm0;
    const float ref1 = nm1 == -INFINITY ? 0.f : nm1;
    const float corr0 = exp2f(mx0 - ref0), corr1 = exp2f(mx1 - ref1);
    mx0 = nm0;
    mx1 = nm1;
    float rs0 = 0.f, rs1 = 0.f;
    uint32_t pf[KVT / 8][2];
#pragma unroll
    for (int nt = 0; nt < KVT / 8; ++nt) {
      const float p00 = exp2f(s[nt][0] - ref0), p01 = exp2f(s[nt][1] - ref0);
      const float p10 = exp2f(s[nt][2] - ref1), p11 = exp2f(s[nt][3] - ref1);
      rs0 += p00 + p01;
      rs1 += p10 + p11;
      pf[nt][0] = Cvt<T>::pack2(p00, p01);
      pf[nt][1] = Cvt<T>::pack2(p10, p11);
    }
    l0 = l0 * corr0 + rs0;
    l1 = l1 * corr1 + rs1;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[i][0] *= corr0; o[i][1] *= corr0;
      o[i][2] *= corr1; o[i][3] *= corr1;
    }
    // ---- O += P V ----
    const uint32_t sva = smem_u32(sv[buf]);
    {
      const int mi = lane >> 3, r8 = lane & 7;
#pragma unroll
      for (int kk = 0; kk < KVT / 16; ++kk) {
        const uint32_t a[4] = {pf[kk * 2][0], pf[kk * 2][1], pf[kk * 2 + 1][0], pf[kk * 2 + 1][1]};
        const int vrow = kk * 16 + (mi & 1) * 8 + r8;
#pragma unroll
        for (int dp = 0; dp < 4; ++dp) {
          uint32_t b0, b1, b2, b3;
          ldsm_x4_t(sva + tile_off(vrow, dp * 2 + (mi >> 1)), b0, b1, b2, b3);
          mma16816<T>(o[dp * 2], a, b0, b1);
          mma16816<T>(o[dp * 2 + 1], a, b2, b3);
        }
      }
    }
    __syncthreads();  // everyone done with buf before it is refilled
  }
  cp_async_wait<0>();

  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = l0 > 0.f ? 1.0f / l0 : 0.f;
  const float inv1 = l1 > 0.f ? 1.0f / l1 : 0.f;

  // ---- write O: stage through sq (each warp its own 16 rows) for 16-byte row stores ----
  __syncwarp();
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    const int r0 = warp * 16 + gq, r1 = r0 + 8;
    const int chunk = nt;  // 8 columns = one 16-byte chunk
    *reinterpret_cast<uint32_t*>(sq + tile_off(r0, chunk) + tq * 4) = Cvt<T>::pack2(o[nt][0] * inv0, o[nt][1] * inv0);
    *reinterpret_cast<uint32_t*>(sq + tile_off(r1, chunk) + tq * 4) = Cvt<T>::pack2(o[nt][2] * inv1, o[nt][3] * inv1);
  }
  __syncwarp();
  for (int i = lane; i < 16 * 8; i += 32) {
    const int r = i >> 3, c = i & 7;
    const int j = q0 + warp * 16 + r;
    if (j < p.seq) {
      const uint4 v = *reinterpret_cast<const uint4*>(sq + tile_off(warp * 16 + r, c));
      T* dst;
      if (p.split > 0 && j >= p.split) {
        dst = reinterpret_cast<T*>(p.out2) + (static_cast<long long>(g) * (p.seq - p.split) + (j - p.split)) * p.ldo2;
      } else {
        const long long orow = g0 * p.ogs0 + g1 * p.ogs1 + g2 * p.ogs2 +
                               static_cast<long long>(j / p.inner) * p.oso + static_cast<long long>(j % p.inner) * p.osi;
        dst = reinterpret_cast<T*>(p.out) + orow * p.ldo;
      }
      *reinterpret_cast<uint4*>(dst + head * HD + c * 8) = v;
    }
  }
}

template <typename T>
static int launch_attn(const AttnParams& p, cudaStream_t s) {
  const int smax = p.seq > p.seq_k ? p.seq : p.seq_k;
  if (smax <= 16) {
    const long long blocks = static_cast<long long>(p.groups) * p.heads;
    attn_kernel<T, 1, 16><<<static_cast<unsigned>(blocks), 32, 0, s>>>(p);
  } else if (smax <= 32) {
    const long long blocks = static_cast<long long>(p.groups) * p.heads;
    attn_kernel<T, 2, 32><<<static_cast<unsigned>(blocks), 64, 0, s>>>(p);
  } else {
    const int q_tiles = (p.seq + 63) / 64;
    const long long blocks = static_cast<long long>(p.groups) * p.heads * q_tiles;
    attn_kernel<T, 4, 64><<<static_cast<unsigned>(blocks), 128, 0, s>>>(p);
  }
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// attention_wgmma.cu: contiguous sequences and gathered unit sequences (cross-view /
// temporal row-wise, optional unit mask; local query views against separate gathered K,V)
bool attn_tc_eligible(const dwm_attention_args* a);
bool attn_tcg_eligible(const dwm_attention_args* a);
bool attn_tcg_kv_eligible(const dwm_attention_args* a);
int attn_wgmma_launch(const dwm_attention_args* a, cudaStream_t s);
int attn_tcg_launch(const dwm_attention_args* a, cudaStream_t s);
int attn_tcg_kv_launch(const dwm_attention_args* a, cudaStream_t s);
bool attn_text_eligible(const dwm_attention_args* a);
int attn_text_launch(const dwm_attention_args* a, bool causal, const float* bias, cudaStream_t s);

}  // namespace dwm

namespace dwm {
// text == true: dwm_b200_attention_text (causal / bias given, checked by the caller)
static int attention_entry(const dwm_attention_args* a, bool text, bool causal, const float* bias,
                           dwm_stream_t stream) {
  DWM_REQUIRE(a != nullptr, "dwm_b200_attention: null args");
  DWM_REQUIRE(a->head_dim == 64, "dwm_b200_attention: head_dim must be 64, got %d", a->head_dim);
  DWM_REQUIRE(a->qkv && a->out, "dwm_b200_attention: null qkv/out");
  DWM_REQUIRE(a->heads > 0 && a->seq > 0 && a->inner > 0, "dwm_b200_attention: bad heads/seq/inner");
  DWM_REQUIRE(a->group_dims[0] > 0 && a->group_dims[1] > 0 && a->group_dims[2] > 0,
              "dwm_b200_attention: group dims must be positive");
  DWM_REQUIRE(a->ld % 8 == 0 && a->ldo % 8 == 0 && a->D % 8 == 0 &&
                  (reinterpret_cast<uintptr_t>(a->qkv) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(a->out) & 15) == 0,
              "dwm_b200_attention: 16-byte alignment of qkv/out rows required");
  if (a->split > 0)
    DWM_REQUIRE(a->out2 && a->ldo2 % 8 == 0 && a->split < a->seq, "dwm_b200_attention: bad split/out2");
  if (a->mask) DWM_REQUIRE(a->mask_div > 0 && a->n_outer > 0, "dwm_b200_attention: mask needs mask_div, n_outer");
  DWM_REQUIRE(a->mask_q_offset >= 0, "dwm_b200_attention: mask_q_offset must be >= 0, got %d", a->mask_q_offset);
  if (a->mask && a->mask_q_offset > 0)
    DWM_REQUIRE(static_cast<long long>(a->mask_q_offset) + (a->seq - 1) / a->inner < a->n_outer,
                "dwm_b200_attention: query units [%d, %d) lie outside the %d mask rows", a->mask_q_offset,
                a->mask_q_offset + (a->seq - 1) / a->inner + 1, a->n_outer);
  if (a->kv)
    DWM_REQUIRE(a->ld_kv % 8 == 0 && a->k_col % 8 == 0 && a->v_col % 8 == 0 && a->seq_kv > 0 && a->inner_kv > 0 &&
                    (reinterpret_cast<uintptr_t>(a->kv) & 15) == 0,
                "dwm_b200_attention: bad separate kv description");
  if (text) {
    // only the wgmma kernel has the causal mask and the additive bias
    DWM_REQUIRE(causal != (bias != nullptr),
                "dwm_b200_attention_text: give one of causal and bias (causal=%d, bias=%p)", int(causal),
                static_cast<const void*>(bias));
    DWM_REQUIRE(attn_text_eligible(a),
                "dwm_b200_attention_text: needs contiguous sequences (group_strides[0] = inner = seq, unit "
                "strides, one group dim) without mask, kv or split");
    DWM_REQUIRE((reinterpret_cast<uintptr_t>(bias) & 3) == 0, "dwm_b200_attention_text: bias must be 4-byte aligned");
    return attn_text_launch(a, causal, bias, reinterpret_cast<cudaStream_t>(stream));
  }
  {
    // contiguous sequences (joint / dual attention) and gathered unit sequences (cross-view /
    // temporal row-wise) run on the wgmma kernel; the rest (pointwise temporal, separate K,V,
    // short sequences) on the mma.sync kernel below
    if (g_attn_tc < 0) {   // env DWM_ATTN_TC = 0 | 1 (DWM_ATTN_LEGACY: same as 0); default 1
      const char* e = getenv("DWM_ATTN_TC");
      g_attn_tc = getenv("DWM_ATTN_LEGACY") != nullptr ? 0 : (e && e[0] >= '0' && e[0] <= '1') ? e[0] - '0' : 1;
    }
    if (g_attn_tc >= 1 && attn_tc_eligible(a)) return attn_wgmma_launch(a, reinterpret_cast<cudaStream_t>(stream));
    if (g_attn_tc >= 1 && attn_tcg_eligible(a)) return attn_tcg_launch(a, reinterpret_cast<cudaStream_t>(stream));
    if (g_attn_tc >= 1 && attn_tcg_kv_eligible(a)) return attn_tcg_kv_launch(a, reinterpret_cast<cudaStream_t>(stream));
  }
  const long long groups = static_cast<long long>(a->group_dims[0]) * a->group_dims[1] * a->group_dims[2];
  const int seq_max = (a->kv && a->seq_kv > a->seq) ? a->seq_kv : a->seq;
  const long long q_tiles = seq_max <= 32 ? 1 : (a->seq + 63) / 64;
  DWM_REQUIRE(groups * a->heads * q_tiles < (1ll << 31), "dwm_b200_attention: grid too large");
  AttnParams p;
  p.q = a->qkv; p.ldq = a->ld; p.heads = a->heads;
  if (a->kv) {
    p.kv = a->kv; p.ldkv = a->ld_kv; p.kcol0 = static_cast<int>(a->k_col); p.vcol0 = static_cast<int>(a->v_col);
    p.kgs0 = a->kv_group_strides[0]; p.kgs1 = a->kv_group_strides[1]; p.kgs2 = a->kv_group_strides[2];
    p.seq_k = a->seq_kv; p.inner_k = a->inner_kv; p.kso = a->kv_stride_outer; p.ksi = a->kv_stride_inner;
  } else {
    p.kv = a->qkv; p.ldkv = a->ld; p.kcol0 = static_cast<int>(a->D); p.vcol0 = static_cast<int>(2 * a->D);
    p.kgs0 = a->group_strides[0]; p.kgs1 = a->group_strides[1]; p.kgs2 = a->group_strides[2];
    p.seq_k = a->seq; p.inner_k = a->inner; p.kso = a->stride_outer; p.ksi = a->stride_inner;
  }
  p.groups = static_cast<int>(groups); p.G1 = static_cast<int>(a->group_dims[1]); p.G2 = static_cast<int>(a->group_dims[2]);
  p.gs0 = a->group_strides[0]; p.gs1 = a->group_strides[1]; p.gs2 = a->group_strides[2];
  p.seq = a->seq; p.inner = a->inner; p.so = a->stride_outer; p.si = a->stride_inner;
  p.out = a->out; p.ldo = a->ldo;
  p.ogs0 = a->out_group_strides[0]; p.ogs1 = a->out_group_strides[1]; p.ogs2 = a->out_group_strides[2];
  p.oso = a->out_stride_outer; p.osi = a->out_stride_inner;
  p.split = a->split; p.out2 = a->out2; p.ldo2 = a->ldo2;
  p.mask = a->mask; p.mask_div = a->mask_div; p.n_outer = a->n_outer; p.mask_q0 = a->mask_q_offset;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (a->dtype == DWM_BF16) return launch_attn<__nv_bfloat16>(p, s);
  if (a->dtype == DWM_F16) return launch_attn<__half>(p, s);
  set_last_error("dwm_b200_attention: dtype must be DWM_BF16 or DWM_F16, got %d", a->dtype);
  return -1;
}
}  // namespace dwm

extern "C" int dwm_b200_attention(const dwm_attention_args* a, dwm_stream_t stream) {
  return dwm::attention_entry(a, false, false, nullptr, stream);
}

extern "C" int dwm_b200_attention_text(const dwm_attention_args* a, int causal, const float* bias,
                                       dwm_stream_t stream) {
  return dwm::attention_entry(a, true, causal != 0, bias, stream);
}
