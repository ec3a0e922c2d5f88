// Fused-epilogue machinery and the warpgroup main loop shared by the wgmma GEMM and
// convolution kernels (sm_90a).
#pragma once
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/dwm_b200.h"

namespace dwm {

constexpr int BM = 128;   // accumulator rows per CTA: two consumer warpgroups x 64 rows
constexpr int BK = 64;    // one 128-byte swizzle atom of 16-bit K per stage (128 E4M3 elements)
constexpr int WG_K = 16;
constexpr int CONSUMER_WGS = 2;
constexpr int GEMM_THREADS = 128 * (1 + CONSUMER_WGS);   // warpgroup 0: TMA producer
constexpr int EPI_WARPS = 4 * CONSUMER_WGS;
constexpr int EPI_STAGE_BYTES = EPI_WARPS * 16 * 32 * 4;  // per consumer warp: 16x32 fp32
// TMA-stored 16-bit outputs: a 64 x 64 box (128B-swizzled, 128 bytes per row), two per warpgroup
constexpr int EPI_BOX_BYTES = 64 * 64 * 2;
constexpr int EPI_BOXES_BYTES = CONSUMER_WGS * 2 * EPI_BOX_BYTES;
// register split (65536 per SM, one CTA): producer warpgroup 40, consumers 232 each
constexpr int PRODUCER_REGS = 40;
constexpr int CONSUMER_REGS = 232;
// DWM_EPI_STORE with act = DWM_ACT_QUICK_GELU, compiled as an epilogue of its own so that the
// run-time activation switch of DWM_EPI_STORE keeps its instructions
constexpr int EPI_STORE_QUICK_GELU = 16;

// epilogues whose output is the 16-bit tile (the others read-modify-write fp32)
__host__ __device__ constexpr bool epi_out16(int epi) {
  return epi == DWM_EPI_STORE || epi == DWM_EPI_GEGLU || epi == DWM_EPI_QKNORM || epi == EPI_STORE_QUICK_GELU ||
         epi == DWM_EPI_GEGLU_TANH;
}

__device__ __forceinline__ float quick_gelu(float x) { return x / (1.0f + __expf(-1.702f * x)); }

struct EpiParams {
  void* out;
  long long ldo;
  const float* bias;
  int act;
  long long rows_per_item, out_item_stride, out_row_offset;
  const float* qw;
  const float* kw;
  long long qk_region;
  float eps;
  int norm_regions;
  const float* resid;
  long long ldr, resid_row_mod;   // resid_row_mod < 0: one residual row per ITEM (m / rows_per_item)
  const float* gate;
  long long gate_ld;
  const float* blend_x;
  long long ldx;
  const float* alpha;
  long long rows_per_batch;
  void* peer_out[8];
  int n_peers;
  int resid_prefetch;   // RESID: L2 prefetch of the tile's residual / blend rows by the TMA unit
  const float* a_scale;  // FP8 operands: row scales of A [M] and of W [N]
  const float* w_scale;
  // 16-bit outputs stored by TMA (see TmaOut): the M rows are out_items whole items of out_rpi
  // rows (a layout without items: one item of M rows), then the rows of a partial last item
  int tma_out;
  int out_rpi, out_items;
};

// A consumer warpgroup's TMA store of its 16-bit tile rows, box by box.  The warps write a
// 64 x 64 box into one of two swizzled shared-memory buffers with stmatrix; one leader thread
// stores it through `map`, the whole items [out_items, out_rpi, N] (row pitch ldo, item pitch
// out_item_stride * ldo, based at the output's first row), and commits it as a bulk
// async-group.  The store starts at the box's first row, so its coordinates are never negative,
// and TMA clips it to that row's item and to N.  The rows of the box in later items, or in a
// partial last item, are copied from the box by the warpgroup's threads.
struct TmaOut {
  bool on;          // false: the register path stores the rows
  const CUtensorMap* map;
  uint8_t* bufs;    // this warpgroup's two boxes
  int bar;          // named barrier of this warpgroup
  bool leader;      // the thread that stores (and owns the bulk async-groups)
  uint32_t boxes;   // boxes stored so far: the parity picks the buffer
};

__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case DWM_ACT_GELU_TANH: return gelu_tanh(v);
    case DWM_ACT_GELU_ERF: return gelu_erf(v);
    case DWM_ACT_SILU: return silu(v);
    case DWM_ACT_RELU: return fmaxf(v, 0.f);
    default: return v;
  }
}

// RESID arithmetic, spelled with explicit roundings so that every kernel variant (1-CTA /
// 2-CTA, register / TMA-staged epilogue, convolution) produces the same bits whatever the
// compiler would contract: v = fma(acc + bias, gate, resid); blend: fma(alpha, x, (1-alpha) v).
// Absent bias / gate are 0 / 1, which leaves the value exact.
__device__ __forceinline__ float resid_elem(float acc, float b, float g, float r) {
  return __fmaf_rn(__fadd_rn(acc, b), g, r);
}
__device__ __forceinline__ float blend_elem(float a, float a1, float x, float v) {
  return __fmaf_rn(a, x, __fmul_rn(a1, v));
}

__device__ __forceinline__ void st_global_v4(void* p, uint32_t a, uint32_t b, uint32_t c,
                                             uint32_t d) {
  asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d)
               : "memory");
}

// ---- tile drain (consumer warps) -----------------------------------------------
// Each consumer warp owns 16 accumulator rows of its warpgroup's 64 (wgmma fragment: lane l
// holds rows l/4 and l/4 + 8, two adjacent columns per n8 block).  Per 32-column chunk the
// warp applies the column-local math on the fragment, then transposes the 16x32 fp32 chunk
// through a 2 KB XOR-swizzled shared-memory buffer (phase 1) so that the global traffic,
// including the fp32 residual read-modify-write, is coalesced: 8 lanes per row, a float4
// per lane, 4 rows per instruction (phase 2).

// chunk c of the fragment: v[4jj + e] = acc[4(4c + jj) + e]
template <int NA>
__device__ __forceinline__ void frag_chunk(const float (&acc)[NA], int c, float (&v)[16]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = acc[16 * c + i];
}

__device__ __forceinline__ void stage_dump(float* stg, int lane, const float (&v)[16]) {
  __syncwarp();  // phase-2 readers of the previous chunk are done
  const int r0 = lane >> 2, q0 = (lane & 3) >> 1, h = (lane & 1) * 2;
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int q = (2 * jj + q0) ^ r0;       // float4 slot, swizzled by row (r0 + 8 has the same r & 7)
    *reinterpret_cast<float2*>(stg + r0 * 32 + q * 4 + h) = make_float2(v[4 * jj], v[4 * jj + 1]);
    *reinterpret_cast<float2*>(stg + (r0 + 8) * 32 + q * 4 + h) = make_float2(v[4 * jj + 2], v[4 * jj + 3]);
  }
  __syncwarp();
}

// column of fragment value v[4jj + e] inside its 32-column chunk
__device__ __forceinline__ int frag_col(int lane, int jj, int e) { return 8 * jj + 2 * (lane & 3) + (e & 1); }

// Row mapping of an accumulator tile.  Linear (GEMM): tile row r is global row m_base + r,
// valid while < M.  Pixel tile (implicit-GEMM convolution): the 128 accumulator rows are a
// bw x bh patch of an image of width img_w; row r = (r / bw, r % bw) maps to global row
// m_base + (r / bw) * img_w + r % bw and is valid inside the patch / image limits.
struct TileGeom {
  int bw;      // 0 => linear
  int rows;    // bw * bh
  int w_lim;   // img_w - w0
  int h_lim;   // img_h - h0
  int img_w;
};

// acc: the NT-column fragment of this warp's warpgroup; row0: tile row of the warp's first row.
// tma (linear tiles with 16-bit outputs only): store the rows by TMA instead of from registers.
template <typename T, int EPI, int NT>
__device__ __forceinline__ void drain_tile(const float (&acc)[NT / 2], float* stg, int m_base, int row0, int M,
                                           int n_tile0, int N, const EpiParams& p, int lane,
                                           const TileGeom geom = TileGeom{0, 0, 0, 0, 0}, TmaOut* tma = nullptr) {
  constexpr bool kOut16 = epi_out16(EPI);
  const bool use_tma = kOut16 && tma != nullptr && tma->on;
  const int rs = lane >> 3;  // phase-2: row within a group of 4
  const int c4 = lane & 7;   // phase-2: float4 column within the 32-col chunk

  // phase-2 per-row metadata for the 4 rows this lane stores (it*4 + rs)
  int orow[4];
  int rrow[4];
  int item[4];
  float alpha[4];
  const int rpi = static_cast<int>(p.rows_per_item);
#pragma unroll
  for (int it = 0; it < 4 && !use_tma; ++it) {
    int m;
    bool valid;
    if (geom.bw > 0) {
      const int r = row0 + it * 4 + rs;
      const int ph = r / geom.bw, pw = r - ph * geom.bw;
      valid = r < geom.rows && pw < geom.w_lim && ph < geom.h_lim;
      m = m_base + ph * geom.img_w + pw;
    } else {
      m = m_base + row0 + it * 4 + rs;
      valid = m < M;
    }
    if (valid) {
      int o = m;
      if (kOut16) {
        if (rpi > 0) o = (m / rpi) * static_cast<int>(p.out_item_stride) + (m % rpi);
        o += static_cast<int>(p.out_row_offset);
      }
      orow[it] = o;
      if (EPI == DWM_EPI_RESID) {
        item[it] = rpi > 0 ? m / rpi : 0;
        rrow[it] = p.resid_row_mod > 0 ? m % static_cast<int>(p.resid_row_mod)
                   : (p.resid_row_mod < 0 ? item[it] : m);
        alpha[it] = p.blend_x ? __ldg(p.alpha + (p.rows_per_batch > 0 ? m / static_cast<int>(p.rows_per_batch) : 0)) : 0.f;
      }
    } else {
      orow[it] = -1;
    }
  }

  auto stg4 = [&](int r) { return *reinterpret_cast<const float4*>(stg + r * 32 + ((c4 ^ (r & 7)) << 2)); };
  // phase 2 for 16-bit outputs: `ocol` = first output column of the staged chunk
  auto flush16 = [&](int ocol) {
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const float4 v = stg4(it * 4 + rs);
      if (orow[it] >= 0) {
        T* dst = reinterpret_cast<T*>(p.out) + static_cast<long long>(orow[it]) * p.ldo + ocol + c4 * 4;
        uint2 pk;
        pk.x = Cvt<T>::pack2(v.x, v.y);
        pk.y = Cvt<T>::pack2(v.z, v.w);
        *reinterpret_cast<uint2*>(dst) = pk;
        // fused scatter to the peers' buffers over NVLink (same element offset)
        const long long eoff = static_cast<long long>(orow[it]) * p.ldo + ocol + c4 * 4;
        for (int q = 0; q < p.n_peers; ++q)
          *reinterpret_cast<uint2*>(reinterpret_cast<T*>(p.peer_out[q]) + eoff) = pk;
      }
    }
  };
  // TMA path: the 32-column chunk at output column `ocol` goes to its half of the current box
  // (boxes start at multiples of 64 columns); box_store(ocol) then stores that box
  auto box_put = [&](const float (&v)[16], int ocol) {
    const uint32_t buf = smem_u32(tma->bufs + (tma->boxes & 1) * EPI_BOX_BYTES);
    const int i = lane >> 3;                               // the 8x8 matrix this lane addresses
    const int r = (row0 & 63) + (i & 1) * 8 + (lane & 7);  // its box row
#pragma unroll
    for (int q = 0; q < 2; ++q) {   // n8 blocks 2q and 2q + 1 of the chunk, rows 0-7 and 8-15 each
      const int c16 = ((ocol >> 5) & 1) * 4 + 2 * q + (i >> 1);   // 16-byte column in the box row
      stmatrix_x4(buf + r * 128 + ((c16 ^ (r & 7)) << 4), Cvt<T>::pack2(v[8 * q], v[8 * q + 1]),
                  Cvt<T>::pack2(v[8 * q + 2], v[8 * q + 3]), Cvt<T>::pack2(v[8 * q + 4], v[8 * q + 5]),
                  Cvt<T>::pack2(v[8 * q + 6], v[8 * q + 7]));
    }
  };
  auto box_store = [&](int ocol) {
    fence_proxy_async();                       // this thread's stmatrix writes -> the TMA unit
    if (tma->leader) bulk_wait_read_all();     // the previous box's store has read the other buffer
    named_bar_sync(tma->bar, 128);
    const uint8_t* buf = tma->bufs + (tma->boxes & 1) * EPI_BOX_BYTES;
    const int m0 = m_base + (row0 & ~63), col = ocol & ~63;
    const int item = m0 / p.out_rpi, r = m0 - item * p.out_rpi;
    if (tma->leader) {
      if (item < p.out_items) tma_store_3d(tma->map, buf, col, r, item);
      bulk_commit();
    }
    // rows [j0, j1) of the box are past the end of the stored item (or in a partial last item):
    // 8 threads per row, 16 bytes each, un-swizzled from the box.  The buffer is rewritten only
    // after the next box's barrier, which every thread reaches after its copies.
    const int j0 = item < p.out_items ? p.out_rpi - r : 0;
    const int j1 = M - m0 < 64 ? M - m0 : 64;
    if (j0 < j1) {
      const int t = ((row0 & 63) << 1) + lane;   // thread of the warpgroup
      const int c = t & 7;
      const int n_out = (EPI == DWM_EPI_GEGLU || EPI == DWM_EPI_GEGLU_TANH) ? N / 2 : N;
#pragma unroll 1
      for (int j = j0 + (t >> 3); j < j1; j += 16) {
        const int m = m0 + j;
        if (col + 8 * c < n_out) {
          const long long o = static_cast<long long>(m / p.out_rpi) * p.out_item_stride + m % p.out_rpi + p.out_row_offset;
          *reinterpret_cast<uint4*>(reinterpret_cast<T*>(p.out) + o * p.ldo + col + 8 * c) =
              *reinterpret_cast<const uint4*>(buf + j * 128 + ((c ^ (j & 7)) << 4));
        }
      }
    }
    ++tma->boxes;
  };
  // 16-bit chunk at output column `ocol`; box_done: the last chunk of its box
  auto put16 = [&](const float (&v)[16], int ocol, bool box_done) {
    if (use_tma) {
      box_put(v, ocol);
      if (box_done) box_store(ocol);
    } else {
      stage_dump(stg, lane, v);
      flush16(ocol);
    }
  };
  // phase 2 for fp32 outputs (optionally gated / residual / blended).  The residual
  // (and blend) operands are prefetched into registers at the top of each chunk so
  // their HBM latency overlaps the transpose; in-place update is safe because each
  // lane reads exactly the elements it later writes.
  float4 rq[4], bq[4];
  auto prefetch32 = [&](int ocol) {
    if constexpr (EPI == DWM_EPI_RESID) {
      const int col = ocol + c4 * 4;
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        rq[it] = make_float4(0.f, 0.f, 0.f, 0.f);
        bq[it] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (orow[it] >= 0) {
          if (p.resid) rq[it] = *reinterpret_cast<const float4*>(p.resid + static_cast<long long>(rrow[it]) * p.ldr + col);
          if (p.blend_x) bq[it] = *reinterpret_cast<const float4*>(p.blend_x + static_cast<long long>(orow[it]) * p.ldx + col);
        }
      }
    }
  };
  auto flush32 = [&](int ocol) {
    const int col = ocol + c4 * 4;
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (EPI == DWM_EPI_RESID && p.bias) b = __ldg(reinterpret_cast<const float4*>(p.bias + col));
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      float4 v = stg4(it * 4 + rs);
      if (orow[it] >= 0) {
        if (EPI == DWM_EPI_RESID) {
          float4 g = make_float4(1.f, 1.f, 1.f, 1.f);
          if (p.gate)
            g = __ldg(reinterpret_cast<const float4*>(p.gate + static_cast<long long>(item[it]) * p.gate_ld + col));
          v.x = resid_elem(v.x, b.x, g.x, rq[it].x); v.y = resid_elem(v.y, b.y, g.y, rq[it].y);
          v.z = resid_elem(v.z, b.z, g.z, rq[it].z); v.w = resid_elem(v.w, b.w, g.w, rq[it].w);
          if (p.blend_x) {
            const float a = alpha[it], a1 = 1.0f - alpha[it];
            v.x = blend_elem(a, a1, bq[it].x, v.x); v.y = blend_elem(a, a1, bq[it].y, v.y);
            v.z = blend_elem(a, a1, bq[it].z, v.z); v.w = blend_elem(a, a1, bq[it].w, v.w);
          }
        }
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + static_cast<long long>(orow[it]) * p.ldo + col) = v;
      }
    }
  };

  if constexpr (EPI == DWM_EPI_STORE || EPI == DWM_EPI_F32 || EPI == DWM_EPI_RESID || EPI == EPI_STORE_QUICK_GELU) {
    // fully unrolled: the fragment is indexed with compile-time offsets only
#pragma unroll
    for (int c = 0; c < NT / 32; ++c) {
      const int n0 = n_tile0 + c * 32;
      if (n0 >= N) break;
      prefetch32(n0);
      float v[16];
      frag_chunk(acc, c, v);
      if (EPI != DWM_EPI_RESID) {
        if (p.bias) {
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + frag_col(lane, jj, 0)));
            v[4 * jj] += b.x; v[4 * jj + 1] += b.y; v[4 * jj + 2] += b.x; v[4 * jj + 3] += b.y;
          }
        }
        // activation selected once per chunk (warp-uniform), loops fully unrolled
        if constexpr (EPI == EPI_STORE_QUICK_GELU) {
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] = quick_gelu(v[j]);
        } else if (p.act == DWM_ACT_GELU_TANH) {
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] = gelu_tanh(v[j]);
        } else if (p.act == DWM_ACT_SILU) {
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] = silu(v[j]);
        } else if (p.act == DWM_ACT_GELU_ERF) {
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] = gelu_erf(v[j]);
        } else if (p.act == DWM_ACT_RELU) {
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.f);
        }
      }
      if constexpr (kOut16) {
        put16(v, n0, c & 1);
      } else {
        stage_dump(stg, lane, v);
        flush32(n0);
      }
    }
    // N % 64 = 32: the last box of the row holds one chunk (one store site, not one per chunk)
    if (use_tma && N - n_tile0 < NT && ((N - n_tile0) & 32)) box_store(N - 32);
  } else if constexpr (EPI == DWM_EPI_GEGLU || EPI == DWM_EPI_GEGLU_TANH) {
    static_assert(NT == 256, "GEGLU packs value / gate halves per 256-column tile");
    // tile columns [0,128) hold the value half, [128,256) the gate half of output
    // columns [n_tile0/2, n_tile0/2 + 128).
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float a[16], g[16], v[16];
      frag_chunk(acc, c, a);
      frag_chunk(acc, c + 4, g);
      const float* bv = p.bias ? p.bias + n_tile0 + c * 32 : nullptr;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float x = a[j], y = g[j];
        if (bv) {
          const int col = frag_col(lane, j >> 2, j);
          x += __ldg(bv + col);
          y += __ldg(bv + 128 + col);
        }
        v[j] = x * (EPI == DWM_EPI_GEGLU ? gelu_erf(y) : gelu_tanh(y));
      }
      put16(v, n_tile0 / 2 + c * 32, c & 1);
    }
  } else {  // DWM_EPI_QKNORM: 64-column heads
#pragma unroll
    for (int g = 0; g < NT / 64; ++g) {
      const int n0 = n_tile0 + g * 64;
      if (n0 >= N) break;
      float v0[16], v1[16];
      frag_chunk(acc, 2 * g, v0);
      frag_chunk(acc, 2 * g + 1, v1);
      if (p.bias) {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = frag_col(lane, j >> 2, j);
          v0[j] += __ldg(p.bias + n0 + col);
          v1[j] += __ldg(p.bias + n0 + 32 + col);
        }
      }
      const int region = n0 / static_cast<int>(p.qk_region);
      if (region < p.norm_regions) {
        const float* w = region == 0 ? p.qw : p.kw;
        // a row's 64 values sit in the 4 lanes of a quad: e < 2 row l/4, e >= 2 row l/4 + 8
        float ss_lo = 0.f, ss_hi = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          if ((j & 3) < 2) ss_lo += v0[j] * v0[j] + v1[j] * v1[j];
          else ss_hi += v0[j] * v0[j] + v1[j] * v1[j];
        }
        ss_lo += __shfl_xor_sync(0xffffffffu, ss_lo, 1);
        ss_lo += __shfl_xor_sync(0xffffffffu, ss_lo, 2);
        ss_hi += __shfl_xor_sync(0xffffffffu, ss_hi, 1);
        ss_hi += __shfl_xor_sync(0xffffffffu, ss_hi, 2);
        const float inv_lo = rsqrtf(ss_lo * (1.0f / 64.0f) + p.eps);
        const float inv_hi = rsqrtf(ss_hi * (1.0f / 64.0f) + p.eps);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = frag_col(lane, j >> 2, j);
          const float inv = (j & 3) < 2 ? inv_lo : inv_hi;
          v0[j] = v0[j] * inv * __ldg(w + col);
          v1[j] = v1[j] * inv * __ldg(w + 32 + col);
        }
      }
      put16(v0, n0, false);
      put16(v1, n0 + 32, true);
    }
  }
}

// FP8 operands: acc[r, n] *= a_scale[m] * w_scale[n] over the fragment of this warp's 16 rows
// (first global row m0), before the epilogue adds the bias.  Rows >= M (tile padding) and
// columns >= N are scaled by 0 so that no scale is read out of bounds.  The product of the two
// scales is rounded once and applied with one rounded multiply, whatever the tile shape.
template <int NT>
__device__ __forceinline__ void dequant_frag(float (&acc)[NT / 2], const float* a_scale, const float* w_scale,
                                             int m0, int M, int n_tile0, int N, int lane) {
  const int r = m0 + (lane >> 2);
  const float s_lo = r < M ? __ldg(a_scale + r) : 0.f;
  const float s_hi = r + 8 < M ? __ldg(a_scale + r + 8) : 0.f;
  // groups of 8 column pairs: the compiler barrier keeps the next group's scale loads from
  // being hoisted next to the 128 live accumulators (which would spill)
#pragma unroll
  for (int g = 0; g < NT / 64; ++g) {
    float2 w[8];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int col = n_tile0 + 8 * (8 * g + jj) + 2 * (lane & 3);
      w[jj] = col < N ? __ldg(reinterpret_cast<const float2*>(w_scale + col)) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int j = 8 * g + jj;
      acc[4 * j + 0] = __fmul_rn(acc[4 * j + 0], __fmul_rn(s_lo, w[jj].x));
      acc[4 * j + 1] = __fmul_rn(acc[4 * j + 1], __fmul_rn(s_lo, w[jj].y));
      acc[4 * j + 2] = __fmul_rn(acc[4 * j + 2], __fmul_rn(s_hi, w[jj].x));
      acc[4 * j + 3] = __fmul_rn(acc[4 * j + 3], __fmul_rn(s_hi, w[jj].y));
    }
    asm volatile("" ::: "memory");
  }
}

// FP8 convolution: acc[r, n] *= s * w_scale[n], where s is the activation scale of the tile's
// volume (every tap of an output pixel reads its own volume, so one scalar covers the tile).
// Same rounding as dequant_frag: the scale product is rounded once, then one rounded multiply.
template <int NT>
__device__ __forceinline__ void dequant_frag_vol(float (&acc)[NT / 2], float s, const float* w_scale,
                                                 int n_tile0, int N, int lane) {
#pragma unroll
  for (int g = 0; g < NT / 32; ++g) {
    constexpr int G = 4;   // n8 blocks per group (a 32-column chunk)
    float2 w[G];
#pragma unroll
    for (int jj = 0; jj < G; ++jj) {
      const int col = n_tile0 + 8 * (G * g + jj) + 2 * (lane & 3);
      w[jj] = col < N ? __ldg(reinterpret_cast<const float2*>(w_scale + col)) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int jj = 0; jj < G; ++jj) {
      const int j = G * g + jj;
      const float sx = __fmul_rn(s, w[jj].x), sy = __fmul_rn(s, w[jj].y);
      acc[4 * j + 0] = __fmul_rn(acc[4 * j + 0], sx);
      acc[4 * j + 1] = __fmul_rn(acc[4 * j + 1], sy);
      acc[4 * j + 2] = __fmul_rn(acc[4 * j + 2], sx);
      acc[4 * j + 3] = __fmul_rn(acc[4 * j + 3], sy);
    }
    asm volatile("" ::: "memory");
  }
}

// One output tile of one consumer warpgroup: acc[64 x NT] = sum over k_iters stages and TAPS
// taps of A[64 rows at a_row_off (+ t rows for tap t)] . B[NT rows of tap t]^T.  TAPS = 3 is
// the halo-row convolution: the three dw taps read row-shifted views of one A tile.  Every stage
// is released (one arrive per consumer warp, on this CTA's barrier and, in a cluster of two
// that shares the B tile by multicast, on the peer's) as soon as the wgmma that read it has
// completed; one wgmma group stays in flight.  T is the operand type: a 128-byte K row of a
// stage is four k16 MMAs of 16-bit or four k32 MMAs of E4M3 elements, with the same descriptor
// steps.
template <typename T, int NT, int CL = 1, int TAPS = 1>
__device__ __forceinline__ void wg_mainloop(float (&acc)[NT / 2], const uint8_t* smem_a, int a_stage_bytes,
                                            int a_row_off_bytes, const uint8_t* smem_b, int b_stage_bytes,
                                            uint64_t* full_bar, uint64_t* empty_bar, int stages, int k_iters,
                                            int& stage, uint32_t& phase, int lane, uint32_t peer = 0) {
#pragma unroll
  for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
  fence_operands(acc);
  auto release = [&](int s) {
    mbar_arrive(&empty_bar[s]);
    if constexpr (CL == 2) mbar_arrive_remote(mapa_u32(smem_u32(&empty_bar[s]), peer));
  };
  int prev = -1;
  for (int ki = 0; ki < k_iters; ++ki) {
    mbar_wait(&full_bar[stage], phase);
    wgmma_fence();
#pragma unroll
    for (int t = 0; t < TAPS; ++t) {
      const uint64_t da = gmma_desc_sw128(smem_u32(smem_a + stage * a_stage_bytes + a_row_off_bytes + t * 128));
      const uint64_t db = gmma_desc_sw128(smem_u32(smem_b + stage * b_stage_bytes + t * NT * BK * 2));
#pragma unroll
      for (int k = 0; k < BK / WG_K; ++k) Wgmma<NT, T>::ss(acc, da + 2 * k, db + 2 * k, 1u);
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && lane == 0) release(prev);
    prev = stage;
    if (++stage == stages) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  fence_operands(acc);
  if (prev >= 0 && lane == 0) release(prev);
}

// RESID epilogues read-modify-write an fp32 tile of up to 128 KB whose HBM latency the 8 consumer
// warps cannot cover with register prefetch alone.  While the MMAs of the tile are still
// running, each epilogue thread asks the L2 to fetch its row segment (512 B) of the
// residual (and blend) operand, so the later loads hit L2.
template <int EPI, int NT>
__device__ __forceinline__ void prefetch_resid_tile(const EpiParams& p, int m, int M, int n_tile0,
                                                    int N, int half) {
  constexpr int half_cols = NT / 2;
  if constexpr (EPI == DWM_EPI_RESID) {
    if (!p.resid_prefetch) return;
    const int n0 = n_tile0 + half * half_cols;
    if (m < M && n0 < N) {
      const int cols = (N - n0) < half_cols ? (N - n0) : half_cols;
      const uint32_t bytes = static_cast<uint32_t>(cols) * 4u;
      if (p.resid) {
        if (p.resid_row_mod >= 0) {
          const long long rr = p.resid_row_mod > 0 ? m % static_cast<int>(p.resid_row_mod) : m;
          const float* src = p.resid + rr * p.ldr + n0;
          asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
        }
      }
      if (p.blend_x) {
        const float* src = p.blend_x + static_cast<long long>(m) * p.ldx + n0;
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
      }
    }
  }
}

// host side: launches a kernel in clusters of two CTAs along x (grid must be even)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_cluster2(void (*kern)(KArgs...), int grid, int threads, int smem, cudaStream_t s,
                                   Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, args...);
}

// host side: fills EpiParams from the C-ABI struct
inline void fill_epi_params(EpiParams& p, const dwm_linear_args* a) {
  p.out = a->out;
  p.ldo = a->ldo;
  p.bias = a->bias;
  p.act = a->act;
  p.rows_per_item = a->rows_per_item;
  p.out_item_stride = a->out_item_stride;
  p.out_row_offset = a->out_row_offset;
  p.qw = a->q_norm_weight;
  p.kw = a->k_norm_weight;
  p.qk_region = a->qk_region;
  p.eps = a->eps;
  p.norm_regions = a->qk_norm_regions > 0 ? a->qk_norm_regions : 2;
  p.resid = a->resid;
  p.ldr = a->ldr;
  p.resid_row_mod = a->resid_row_mod;
  p.gate = a->gate;
  p.gate_ld = a->gate_ld;
  p.blend_x = a->blend_x;
  p.ldx = a->ldx;
  p.alpha = a->alpha;
  p.rows_per_batch = a->rows_per_batch;
  p.n_peers = a->n_peer_out;
  p.resid_prefetch = 1;
  for (int i = 0; i < 8; ++i) p.peer_out[i] = i < a->n_peer_out ? a->peer_out[i] : nullptr;
  p.a_scale = a->a_scale;
  p.w_scale = a->w_scale;
  p.tma_out = 0;
  p.out_rpi = p.out_items = 0;
}

}  // namespace dwm
