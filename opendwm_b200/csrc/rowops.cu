// Memory-bound row / elementwise kernels of the CTSD step (sm_90a): LayerNorm with
// AdaLN modulation (emits the 16-bit or row-scaled E4M3 GEMM operand), E4M3 row quantization,
// activation casts, sinusoidal embeddings, patchify, and the fused CFG + un-patchify +
// per-frame Euler update; the RMSNorm and the embedding gather of the text encoders.
// All are single-pass over HBM with 128-bit accesses.
#include "common.cuh"
#include "../../include/dwm_b200.h"

namespace dwm {

// ------------------------------------------------------------------ LayerNorm
struct LnParams {
  int M, D;
  const float* x; long long ldx;
  const float* add_item; long long add_item_ld;
  const float* add_full; long long add_full_ld;
  int rows_per_item;
  float* sum_out; long long ld_sum;
  const float* weight; const float* bias; float eps;
  const float* shift; const float* scale; const float* shift2; const float* scale2; long long mod_ld;
  void* out; long long ldo; void* out2; long long ldo2;
  float* out_scale; float* out2_scale;   // E4M3 outputs: row scales
};

constexpr int LN_WARPS = 4;   // rows per block (one warp per row)

// Everything after the x row sits in registers: optional adds, statistics, write-back of the
// summed row, affine / AdaLN modulation (optionally two modulations), 16-bit stores, or
// (T = E4M3) the row's amax and the E4M3 quantization of the fp32 values.
// EXACT: D / 4 == 32 * VPL, so the per-vector bounds checks fold away.
template <typename T, int VPL, bool DUAL, bool EXACT>
__device__ __forceinline__ void ln_finish(const LnParams& p, const int m, const int lane, float4 (&v)[VPL]) {
  const int nvec = EXACT ? 32 * VPL : (p.D >> 2);
  const int item = p.rows_per_item > 0 ? m / p.rows_per_item : 0;
  const float4* ai = p.add_item ? reinterpret_cast<const float4*>(p.add_item + static_cast<long long>(item) * p.add_item_ld) : nullptr;
  const float4* af = p.add_full ? reinterpret_cast<const float4*>(p.add_full + static_cast<long long>(m) * p.add_full_ld) : nullptr;
  if (ai) {
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int idx = lane + 32 * i;
      if (idx < nvec) { const float4 a = __ldg(ai + idx); v[i].x += a.x; v[i].y += a.y; v[i].z += a.z; v[i].w += a.w; }
    }
  }
  if (af) {
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int idx = lane + 32 * i;
      if (idx < nvec) { const float4 a = af[idx]; v[i].x += a.x; v[i].y += a.y; v[i].z += a.z; v[i].w += a.w; }
    }
  }
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) sum += v[i].x + v[i].y + v[i].z + v[i].w;
  if (p.sum_out) {
    float4* so = reinterpret_cast<float4*>(p.sum_out + static_cast<long long>(m) * p.ld_sum);
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int idx = lane + 32 * i;
      if (idx < nvec) so[idx] = v[i];
    }
  }
  const float mean = warp_sum(sum) / static_cast<float>(p.D);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int idx = lane + 32 * i;
    if (idx < nvec) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      sq += a * a + b * b + c * c + d * d;
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / static_cast<float>(p.D) + p.eps);
  const float4* w4 = reinterpret_cast<const float4*>(p.weight);
  const float4* b4 = reinterpret_cast<const float4*>(p.bias);
  const float4* sh = p.shift ? reinterpret_cast<const float4*>(p.shift + static_cast<long long>(item) * p.mod_ld) : nullptr;
  const float4* sc = p.scale ? reinterpret_cast<const float4*>(p.scale + static_cast<long long>(item) * p.mod_ld) : nullptr;
  const float4* sh2 = p.shift2 ? reinterpret_cast<const float4*>(p.shift2 + static_cast<long long>(item) * p.mod_ld) : nullptr;
  const float4* sc2 = p.scale2 ? reinterpret_cast<const float4*>(p.scale2 + static_cast<long long>(item) * p.mod_ld) : nullptr;
  T* o1 = reinterpret_cast<T*>(p.out) + static_cast<long long>(m) * p.ldo;
  T* o2 = DUAL ? reinterpret_cast<T*>(p.out2) + static_cast<long long>(m) * p.ldo2 : nullptr;
  // Each optional vector is applied in its own fully unrolled loop so that its VPL loads
  // are issued back to back (one exposed latency per vector instead of one per element).
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    v[i].x = (v[i].x - mean) * rstd; v[i].y = (v[i].y - mean) * rstd;
    v[i].z = (v[i].z - mean) * rstd; v[i].w = (v[i].w - mean) * rstd;
  }
  auto mul_vec = [&](float4 (&d)[VPL], const float4* src, float add_one) {
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int idx = lane + 32 * i;
      if (idx < nvec) {
        const float4 s = __ldg(src + idx);
        d[i].x *= add_one + s.x; d[i].y *= add_one + s.y; d[i].z *= add_one + s.z; d[i].w *= add_one + s.w;
      }
    }
  };
  auto add_vec = [&](float4 (&d)[VPL], const float4* src) {
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const int idx = lane + 32 * i;
      if (idx < nvec) {
        const float4 s = __ldg(src + idx);
        d[i].x += s.x; d[i].y += s.y; d[i].z += s.z; d[i].w += s.w;
      }
    }
  };
  auto store_vec = [&](const float4 (&d)[VPL], T* dst, float* row_scale) {
    if constexpr (sizeof(T) == 1) {
      float amax = 0.f;
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        const int idx = lane + 32 * i;
        if (idx < nvec)
          amax = fmaxf(amax, fmaxf(fmaxf(fabsf(d[i].x), fabsf(d[i].y)), fmaxf(fabsf(d[i].z), fabsf(d[i].w))));
      }
      amax = warp_max(amax);
      const float inv = e4m3_inv(amax);
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        const int idx = lane + 32 * i;
        if (idx < nvec) reinterpret_cast<uint32_t*>(dst)[idx] = e4m3x4(d[i].x, d[i].y, d[i].z, d[i].w, inv);
      }
      if (lane == 0) row_scale[m] = e4m3_scale(amax);
    } else {
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        const int idx = lane + 32 * i;
        if (idx < nvec) {
          uint2 pk; pk.x = Cvt<T>::pack2(d[i].x, d[i].y); pk.y = Cvt<T>::pack2(d[i].z, d[i].w);
          reinterpret_cast<uint2*>(dst)[idx] = pk;
        }
      }
    }
  };
  if (w4) mul_vec(v, w4, 0.f);
  if (b4) add_vec(v, b4);
  if constexpr (DUAL) {   // second modulation of the same normalised row (SD35AdaLayerNormZeroX)
    float4 z[VPL];
#pragma unroll
    for (int i = 0; i < VPL; ++i) z[i] = v[i];
    if (sc2) mul_vec(z, sc2, 1.f);
    if (sh2) add_vec(z, sh2);
    store_vec(z, o2, p.out2_scale);
  }
  if (sc) mul_vec(v, sc, 1.f);
  if (sh) add_vec(v, sh);
  store_vec(v, o1, p.out_scale);
}

template <typename T, int VPL, bool DUAL>
__global__ void __launch_bounds__(LN_WARPS * 32) layernorm_kernel(const LnParams p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * LN_WARPS + warp;
  if (m >= p.M) return;
  const int nvec = p.D >> 2;
  const float4* xr = reinterpret_cast<const float4*>(p.x + static_cast<long long>(m) * p.ldx);
  float4 v[VPL];
  // all loads of the row are issued back to back (no control flow in between) so that
  // VPL 16-byte requests per lane are in flight; the optional adds follow.
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int idx = lane + 32 * i;
    v[i] = idx < nvec ? xr[idx] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  ln_finish<T, VPL, DUAL, false>(p, m, lane, v);
}

// Staged variant: a producer thread streams groups of 16 rows into a 2-stage shared-memory ring
// with 1-D bulk copies (cp.async.bulk + mbarrier transaction counts); 16 compute warps take
// one row each.  Memory-level parallelism (96-192 KB in flight per SM) no longer depends on
// occupancy — the register-resident kernel above stalls on long_scoreboard at 31 % occupancy.
constexpr int LNS_ROWS = 16, LNS_STAGES = 2, LNS_THREADS = (LNS_ROWS + 1) * 32;

__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst_smem)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

template <typename T, int VPL, bool DUAL, bool EXACT>
__global__ void __launch_bounds__(LNS_THREADS, 1) layernorm_staged_kernel(const LnParams p, const int n_groups) {
  extern __shared__ __align__(128) uint8_t ln_smem[];
  const int row_bytes = p.D * 4;
  float* stages = reinterpret_cast<float*>(ln_smem);
  uint64_t* full = reinterpret_cast<uint64_t*>(ln_smem + static_cast<size_t>(LNS_STAGES) * LNS_ROWS * row_bytes);
  uint64_t* empty = full + LNS_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < LNS_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], LNS_ROWS); }
    fence_barrier_init();
  }
  __syncthreads();
  int st = 0;
  uint32_t ph = 0;
  // every CTA streams a CONTIGUOUS range of row groups: consecutive groups belong to the same
  // view-frame item (448 rows = 28 groups), so its modulation vectors (2-4 x 6 KB) stay in L1;
  // with a grid-strided assignment every stage met a new item and each warp paid two L2 round
  // trips per row (ncu r02: 64 % of the stall samples on long_scoreboard, 51 % of DRAM peak)
  const int per_cta = (n_groups + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
  const int g_begin = static_cast<int>(blockIdx.x) * per_cta;
  const int g_end = g_begin + per_cta < n_groups ? g_begin + per_cta : n_groups;
  if (warp == LNS_ROWS) {
    if (lane == 0) {
      for (int g = g_begin; g < g_end; ++g) {
        mbar_wait(&empty[st], ph ^ 1);
        const int m0 = g * LNS_ROWS;
        const int rows = p.M - m0 < LNS_ROWS ? p.M - m0 : LNS_ROWS;
        mbar_expect_tx(&full[st], static_cast<uint32_t>(rows) * row_bytes);
        for (int r = 0; r < rows; ++r)
          bulk_g2s(stages + static_cast<size_t>(st * LNS_ROWS + r) * p.D,
                   p.x + static_cast<long long>(m0 + r) * p.ldx, row_bytes, &full[st]);
        if (++st == LNS_STAGES) { st = 0; ph ^= 1; }
      }
    }
    return;
  }
  const int nvec = EXACT ? 32 * VPL : (p.D >> 2);
  for (int g = g_begin; g < g_end; ++g) {
    mbar_wait(&full[st], ph);
    const int m = g * LNS_ROWS + warp;
    float4 v[VPL];
    if (m < p.M) {
      const float4* row = reinterpret_cast<const float4*>(stages + static_cast<size_t>(st * LNS_ROWS + warp) * p.D);
#pragma unroll
      for (int i = 0; i < VPL; ++i) {
        const int idx = lane + 32 * i;
        v[i] = (EXACT || idx < nvec) ? row[idx] : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[st]);      // the row sits in registers: release the stage
    if (m < p.M) ln_finish<T, VPL, DUAL, EXACT>(p, m, lane, v);
    if (++st == LNS_STAGES) { st = 0; ph ^= 1; }
  }
}

int g_ln_staged = 1;   // dwm_b200_set_option("ln_staged", 0 | 1)

template <typename T, int VPL, bool DUAL>
static int launch_ln_staged(const LnParams& p, cudaStream_t s) {
  const int n_groups = (p.M + LNS_ROWS - 1) / LNS_ROWS;
  const int smem = LNS_STAGES * LNS_ROWS * p.D * 4 + 2 * LNS_STAGES * 8;
  const int grid = n_groups < sm_count() ? n_groups : sm_count();
  const bool exact = (p.D >> 2) == 32 * VPL;
  auto go = [&](auto kern) -> int {
    DWM_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<grid, LNS_THREADS, smem, s>>>(p, n_groups);
    DWM_CHECK_CUDA(cudaGetLastError());
    return 0;
  };
  return exact ? go(layernorm_staged_kernel<T, VPL, DUAL, true>) : go(layernorm_staged_kernel<T, VPL, DUAL, false>);
}

template <typename T, bool DUAL>
static int launch_ln2(const LnParams& p, cudaStream_t s) {
  const int need = (p.D / 4 + 31) / 32;
  // staged path: no per-row residual input, ring <= 220 KB, enough rows (x and ldx are
  // 16-byte aligned: dwm_b200_layernorm checks them)
  const bool staged = g_ln_staged && !p.add_full && LNS_STAGES * LNS_ROWS * p.D * 4 <= 220 * 1024 && p.M >= 4096;
  if (staged) {
    if (need <= 3) return launch_ln_staged<T, 3, DUAL>(p, s);
    if (need <= 6) return launch_ln_staged<T, 6, DUAL>(p, s);
    if (need <= 12) return launch_ln_staged<T, 12, DUAL>(p, s);
    return launch_ln_staged<T, 16, DUAL>(p, s);
  }
  const unsigned grid = static_cast<unsigned>((p.M + LN_WARPS - 1) / LN_WARPS);
  const int threads = LN_WARPS * 32;
  if (need <= 3) layernorm_kernel<T, 3, DUAL><<<grid, threads, 0, s>>>(p);
  else if (need <= 6) layernorm_kernel<T, 6, DUAL><<<grid, threads, 0, s>>>(p);
  else if (need <= 12) layernorm_kernel<T, 12, DUAL><<<grid, threads, 0, s>>>(p);
  else layernorm_kernel<T, 16, DUAL><<<grid, threads, 0, s>>>(p);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

template <typename T>
static int launch_ln(const LnParams& p, cudaStream_t s) {
  return p.out2 ? launch_ln2<T, true>(p, s) : launch_ln2<T, false>(p, s);
}

// ------------------------------------------------------------------ E4M3 row quantization
// One warp per row, 8 elements per lane and step: pass 1 finds the row's amax, pass 2 re-reads
// the row (from L1 / L2) and writes 8 E4M3 bytes per step.
constexpr int QR_WARPS = 4;

template <typename T>
__device__ __forceinline__ void load8(const T* src, float (&v)[8]) {
  if constexpr (sizeof(T) == 4) {
    const float4 a = reinterpret_cast<const float4*>(src)[0], b = reinterpret_cast<const float4*>(src)[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
    const uint4 u = *reinterpret_cast<const uint4*>(src);
    const float2 a = Cvt<T>::unpack2(u.x), b = Cvt<T>::unpack2(u.y), c = Cvt<T>::unpack2(u.z),
                 d = Cvt<T>::unpack2(u.w);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
  }
}

template <typename T>
__global__ void __launch_bounds__(QR_WARPS * 32) quantize_rows_kernel(const T* __restrict__ x, int M, int K,
                                                                      long long ld, uint8_t* __restrict__ out,
                                                                      long long ldo, float* __restrict__ scale) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * QR_WARPS + warp;
  if (m >= M) return;
  const T* row = x + static_cast<long long>(m) * ld;
  const int n8 = K >> 3;
  float amax = 0.f;
  for (int c = lane; c < n8; c += 32) {
    float v[8];
    load8(row + 8 * c, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(v[j]));
  }
  amax = warp_max(amax);
  const float inv = e4m3_inv(amax);
  uint2* orow = reinterpret_cast<uint2*>(out + static_cast<long long>(m) * ldo);
  for (int c = lane; c < n8; c += 32) {
    float v[8];
    load8(row + 8 * c, v);
    orow[c] = make_uint2(e4m3x4(v[0], v[1], v[2], v[3], inv), e4m3x4(v[4], v[5], v[6], v[7], inv));
  }
  if (lane == 0) scale[m] = e4m3_scale(amax);
}

// ------------------------------------------------------------------ act + cast
template <typename T>
__global__ void act_cast_kernel(const float* __restrict__ in, T* __restrict__ out, long long n, int act) {
  const long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i + 3 < n) {
    float4 v = *reinterpret_cast<const float4*>(in + i);
    if (act == DWM_ACT_SILU) { v.x = silu(v.x); v.y = silu(v.y); v.z = silu(v.z); v.w = silu(v.w); }
    else if (act == DWM_ACT_GELU_TANH) { v.x = gelu_tanh(v.x); v.y = gelu_tanh(v.y); v.z = gelu_tanh(v.z); v.w = gelu_tanh(v.w); }
    else if (act == DWM_ACT_GELU_ERF) { v.x = gelu_erf(v.x); v.y = gelu_erf(v.y); v.z = gelu_erf(v.z); v.w = gelu_erf(v.w); }
    uint2 pk; pk.x = Cvt<T>::pack2(v.x, v.y); pk.y = Cvt<T>::pack2(v.z, v.w);
    *reinterpret_cast<uint2*>(out + i) = pk;
  } else {
    for (long long k = i; k < n; ++k) {
      float v = in[k];
      if (act == DWM_ACT_SILU) v = silu(v);
      else if (act == DWM_ACT_GELU_TANH) v = gelu_tanh(v);
      else if (act == DWM_ACT_GELU_ERF) v = gelu_erf(v);
      out[k] = Cvt<T>::from_f(v);
    }
  }
}

// ------------------------------------------------------------------ sinusoid
template <typename T>
__global__ void sinusoid_kernel(const float* __restrict__ t, long long n, int channels, int flip,
                                float shift, T* __restrict__ out, long long ldo) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int half = channels / 2;
  if (i >= n * half) return;
  const long long r = i / half;
  const int k = static_cast<int>(i % half);
  const float freq = expf(-9.210340371976184f * static_cast<float>(k) / (static_cast<float>(half) - shift));
  const float arg = t[r] * freq;
  const float sn = sinf(arg), cs = cosf(arg);
  T* o = out + r * ldo;
  if (flip) { o[k] = Cvt<T>::from_f(cs); o[half + k] = Cvt<T>::from_f(sn); }
  else { o[k] = Cvt<T>::from_f(sn); o[half + k] = Cvt<T>::from_f(cs); }
}

// ------------------------------------------------------------------ patchify
template <typename T>
__global__ void patchify_kernel(const float* __restrict__ x, long long items, int C, int H, int W,
                                int P, T* __restrict__ out, long long ldo) {
  const int Hp = H / P, Wp = W / P;
  const long long total = items * C * H * W;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  // iterate in OUTPUT order so writes are contiguous: (item, hy, wx, c, py, px)
  long long r = i;
  const int px = r % P; r /= P;
  const int py = r % P; r /= P;
  const int c = r % C; r /= C;
  const int wx = r % Wp; r /= Wp;
  const int hy = r % Hp; r /= Hp;
  const long long n = r;
  const float v = x[((n * C + c) * H + hy * P + py) * W + wx * P + px];
  out[((n * Hp + hy) * Wp + wx) * ldo + (c * P + py) * P + px] = Cvt<T>::from_f(v);
}

// ------------------------------------------------------------------ CFG + Euler
__global__ void cfg_euler_kernel(const float* __restrict__ tok, long long ld_tok, int cfg, float gs,
                                 long long B, long long T, long long V, int C, int H, int W, int P,
                                 const int* __restrict__ idx, const float* __restrict__ sigmas, int n_sigmas,
                                 const unsigned char* __restrict__ in_range,
                                 float* __restrict__ lat, float* __restrict__ npred, int round_dtype) {
  const long long total = B * T * V * C * H * W;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  long long r = i;
  const int xw = r % W; r /= W;
  const int yh = r % H; r /= H;
  const int c = r % C; r /= C;
  const long long btv = r;  // (b*T + t)*V + v
  const long long t = (btv / V) % T;
  const int Hp = H / P, Wp = W / P;
  const long long S = static_cast<long long>(Hp) * Wp;
  const long long row = btv * S + (yh / P) * Wp + xw / P;
  const int col = ((yh % P) * P + xw % P) * C + c;
  float v = tok[row * ld_tok + col];
  if (cfg == 2) {
    const float vc = tok[(row + B * T * V * S) * ld_tok + col];
    v = v + gs * (vc - v);  // uncond + scale * (cond - uncond)
  }
  if (npred) npred[i] = v;
  const int k = idx[btv];
  if (k < 0 || k + 1 >= n_sigmas) __trap();   // index outside the scheduler table: fail loudly
  const float dsig = sigmas[k + 1] - sigmas[k];
  const float old = lat[i];
  float nv = old + dsig * v;
  if (round_dtype == DWM_BF16) nv = __bfloat162float(__float2bfloat16_rn(nv));
  else if (round_dtype == DWM_F16) nv = __half2float(__float2half_rn(nv));
  lat[i] = (in_range == nullptr || in_range[t]) ? nv : old;
}

// Per-element Euler update with per-(leading index) sigma indices:
//   x[e] = round(x[e] + (sigma[idx[e / inner] + 1] - sigma[idx[e / inner]]) * v[e])
__global__ void euler_idx_kernel(const float* __restrict__ v, float* __restrict__ x, long long n,
                                 long long inner, const int* __restrict__ idx,
                                 const float* __restrict__ sigmas, int n_sigmas, int round_dtype) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k = idx[i / inner];
  if (k < 0 || k + 1 >= n_sigmas) __trap();
  float nv = x[i] + (sigmas[k + 1] - sigmas[k]) * v[i];
  if (round_dtype == DWM_BF16) nv = __bfloat162float(__float2bfloat16_rn(nv));
  else if (round_dtype == DWM_F16) nv = __half2float(__float2half_rn(nv));
  x[i] = nv;
}

// y[i] += a * x[i]
__global__ void axpy_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float a) {
  const long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i + 3 < n) {
    const float4 xv = *reinterpret_cast<const float4*>(x + i);
    float4 yv = *reinterpret_cast<float4*>(y + i);
    yv.x += a * xv.x; yv.y += a * xv.y; yv.z += a * xv.z; yv.w += a * xv.w;
    *reinterpret_cast<float4*>(y + i) = yv;
  } else {
    for (long long k = i; k < n; ++k) y[k] += a * x[k];
  }
}

// Row softmax of fp32 scores: out[r, c] = softmax_c(scale * x[r, c]) in 16 bits.  One CTA per
// row; the row (<= 64 KB of fp32) is re-read from L2.  Used by the single-head, head_dim 512
// mid-block attention of the 2-D AutoencoderKL decoder, where S = Q K^T and P V run as GEMMs.
template <typename T>
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ x, long long ld, int cols,
                                                           float scale_log2e, T* __restrict__ out, long long ldo) {
  __shared__ float red[8];
  const float* row = x + static_cast<long long>(blockIdx.x) * ld;
  T* orow = out + static_cast<long long>(blockIdx.x) * ldo;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float m = -INFINITY;
  for (int c = tid; c < cols; c += 256) m = fmaxf(m, row[c]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red[warp] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
  __syncthreads();
  float sum = 0.f;
  for (int c = tid; c < cols; c += 256) sum += exp2f((row[c] - m) * scale_log2e);
  sum = warp_sum(sum);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) sum += red[w];
  const float inv = 1.f / sum;
  for (int c = tid; c < cols; c += 256) orow[c] = Cvt<T>::from_f(exp2f((row[c] - m) * scale_log2e) * inv);
}

// Fused CFG combine + DDIM update (eta = 0) with per-(b,t,v) timesteps:
//   pred: fp32 [cfg*B, T, V, C, H, W] (uncond half first);  lat (in/out): fp32 [B, T, V, C, H, W]
//   ts: int32 [B, T, V] current timesteps; prev = ts - step_ratio; alphas: fp32 [num_train]
__global__ void cfg_ddim_kernel(const float* __restrict__ pred, int cfg, float gs, long long per_b,
                                long long inner, long long total, const int* __restrict__ ts, int step_ratio,
                                const float* __restrict__ alphas, int n_alphas, float final_alpha, int pred_type,
                                float* __restrict__ lat, int round_dtype) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  float v = pred[i];
  if (cfg == 2) {
    const float vc = pred[i + total];
    v = v + gs * (vc - v);
  }
  const int t = ts[i / inner];
  const int tp = t - step_ratio;
  if (t < 0 || t >= n_alphas || tp >= n_alphas) __trap();   // timestep outside alphas_cumprod
  const float a_t = alphas[t];
  const float a_p = tp >= 0 ? alphas[tp] : final_alpha;
  const float b_t = 1.0f - a_t;
  const float x = lat[i];
  float x0, eps;
  if (pred_type == 0) {          // epsilon
    x0 = (x - sqrtf(b_t) * v) / sqrtf(a_t);
    eps = v;
  } else if (pred_type == 1) {   // sample
    x0 = v;
    eps = (x - sqrtf(a_t) * x0) / sqrtf(b_t);
  } else {                       // v_prediction
    x0 = sqrtf(a_t) * x - sqrtf(b_t) * v;
    eps = sqrtf(a_t) * v + sqrtf(b_t) * x;
  }
  float nv = sqrtf(a_p) * x0 + sqrtf(1.0f - a_p) * eps;
  if (round_dtype == DWM_BF16) nv = __bfloat162float(__float2bfloat16_rn(nv));
  else if (round_dtype == DWM_F16) nv = __half2float(__float2half_rn(nv));
  lat[i] = nv;
  (void)per_b;
}

// RMSNorm (T5LayerNorm) of one fp32 row per CTA: the sum of squares in fp32 (per-thread float4
// partials, then a fixed-order warp / CTA reduction, so a row's result does not depend on the
// batch), then out = weight * (x * rsqrt(mean + eps)) in the output type.
constexpr int RMS_THREADS = 256;

template <typename T>
__device__ __forceinline__ void store4(T* dst, float a, float b, float c, float d) {
  uint2 pk;
  pk.x = Cvt<T>::pack2(a, b);
  pk.y = Cvt<T>::pack2(c, d);
  *reinterpret_cast<uint2*>(dst) = pk;
}
template <>
__device__ __forceinline__ void store4<float>(float* dst, float a, float b, float c, float d) {
  *reinterpret_cast<float4*>(dst) = make_float4(a, b, c, d);
}

template <typename T>
__global__ void __launch_bounds__(RMS_THREADS) rmsnorm_kernel(const float* __restrict__ x, long long ldx, int D,
                                                              const float* __restrict__ w, float eps,
                                                              T* __restrict__ out, long long ldo) {
  __shared__ float red[RMS_THREADS / 32];
  const float4* row = reinterpret_cast<const float4*>(x + static_cast<long long>(blockIdx.x) * ldx);
  T* orow = out + static_cast<long long>(blockIdx.x) * ldo;
  const int tid = threadIdx.x, nvec = D >> 2;
  float ss = 0.f;
  for (int i = tid; i < nvec; i += RMS_THREADS) {
    const float4 v = row[i];
    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  ss = warp_sum(ss);
  if ((tid & 31) == 0) red[tid >> 5] = ss;
  __syncthreads();
  ss = 0.f;
#pragma unroll
  for (int i = 0; i < RMS_THREADS / 32; ++i) ss += red[i];
  const float r = rsqrtf(ss / static_cast<float>(D) + eps);
  for (int i = tid; i < nvec; i += RMS_THREADS) {
    const float4 v = row[i];
    const float4 g = __ldg(reinterpret_cast<const float4*>(w) + i);
    store4<T>(orow + 4 * i, g.x * (v.x * r), g.y * (v.y * r), g.z * (v.z * r), g.w * (v.w * r));
  }
}

// out[m, :] = tok[ids[m], :] (+ pos[m % seq, :]): one fp32 add per element, as torch does it
__global__ void embed_kernel(const long long* __restrict__ ids, long long M, long long seq,
                             const float* __restrict__ tok, long long vocab, const float* __restrict__ pos,
                             int D, float* __restrict__ out, long long ldo) {
  const long long m = blockIdx.x;
  const long long id = ids[m];
  if (id < 0 || id >= vocab) __trap();   // token id outside the embedding table
  const float4* t = reinterpret_cast<const float4*>(tok + id * D);
  const float4* q = pos ? reinterpret_cast<const float4*>(pos + (m % seq) * D) : nullptr;
  float4* o = reinterpret_cast<float4*>(out + m * ldo);
  for (int i = threadIdx.x; i < (D >> 2); i += blockDim.x) {
    float4 v = __ldg(t + i);
    if (q) {
      const float4 a = __ldg(q + i);
      v.x = __fadd_rn(v.x, a.x); v.y = __fadd_rn(v.y, a.y); v.z = __fadd_rn(v.z, a.z); v.w = __fadd_rn(v.w, a.w);
    }
    o[i] = v;
  }
  (void)M;
}

// out[i] = s0[i / inner] * x[i] + s1[i / inner] * y[i]
__global__ void lincomb2_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                const float* __restrict__ s0, const float* __restrict__ s1, long long n,
                                long long inner, float* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long it = i / inner;
  out[i] = s0[it] * x[i] + s1[it] * y[i];
}

// s0 * x + s1 * y rounded as nvcc contracts lincomb2_kernel's expression: fma(s0, x, s1 * y).
// Spelled out so that a literal s0 = 1 cannot be folded into a different contraction.
__device__ __forceinline__ float lincomb2_rn(float s0, float x, float s1, float y) {
  return __fmaf_rn(s0, x, __fmul_rn(s1, y));
}

// Fused CFG combine + DPM-Solver++ (midpoint, order <= 2) step, in place; the same roundings as
// the chain of lincomb2 launches it replaces.  row = (c_x, c_m, k_s, k_0, k_1, order) is read
// from device memory, so a replayed CUDA graph takes the step its caller loaded.  A first-order
// step never reads x0_prev.
__global__ void cfg_dpmpp_kernel(const float* __restrict__ pred, int cfg, float w_u, float w_c, long long n,
                                 const float* __restrict__ row, float* __restrict__ lat,
                                 float* __restrict__ x0_prev) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float m = pred[i];
  if (cfg == 2) m = lincomb2_rn(w_u, m, w_c, pred[i + n]);
  const float x = lat[i];
  const float x0 = lincomb2_rn(__ldg(row), x, __ldg(row + 1), m);
  float p = lincomb2_rn(__ldg(row + 2), x, __ldg(row + 3), x0);
  if (__ldg(row + 5) == 2.f) p = lincomb2_rn(1.f, p, __ldg(row + 4), x0_prev[i]);
  x0_prev[i] = x0;
  lat[i] = p;
}

}  // namespace dwm

using namespace dwm;

extern "C" int dwm_b200_rmsnorm(const float* x, int64_t M, int64_t D, int64_t ldx, const float* weight, float eps,
                                void* out, int64_t ldo, int dtype, dwm_stream_t stream) {
  DWM_REQUIRE(x && weight && out, "dwm_b200_rmsnorm: null x/weight/out");
  DWM_REQUIRE(M > 0 && M < (1ll << 31) && D > 0 && D % 4 == 0 && D < (1ll << 31) && ldx >= D && ldo >= D &&
                  ldx % 4 == 0 && ldo % 4 == 0,
              "dwm_b200_rmsnorm: need M > 0, D a multiple of 4, ldx / ldo >= D and multiples of 4; got M=%lld "
              "D=%lld ldx=%lld ldo=%lld", (long long)M, (long long)D, (long long)ldx, (long long)ldo);
  DWM_REQUIRE(is_aligned(x, 16) && is_aligned(weight, 16) && is_aligned(out, dtype == DWM_F32 ? 16 : 8),
              "dwm_b200_rmsnorm: x, weight must be 16-byte and out 8-byte (fp32: 16-byte) aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const unsigned grid = static_cast<unsigned>(M);
  const int Di = static_cast<int>(D);
  if (dtype == DWM_BF16)
    rmsnorm_kernel<<<grid, RMS_THREADS, 0, s>>>(x, ldx, Di, weight, eps, static_cast<__nv_bfloat16*>(out), ldo);
  else if (dtype == DWM_F16)
    rmsnorm_kernel<<<grid, RMS_THREADS, 0, s>>>(x, ldx, Di, weight, eps, static_cast<__half*>(out), ldo);
  else if (dtype == DWM_F32)
    rmsnorm_kernel<<<grid, RMS_THREADS, 0, s>>>(x, ldx, Di, weight, eps, static_cast<float*>(out), ldo);
  else
    DWM_REQUIRE(false, "dwm_b200_rmsnorm: dtype must be DWM_BF16, DWM_F16 or DWM_F32, got %d", dtype);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_embed(const int64_t* ids, int64_t M, int64_t seq, const float* tok, int64_t vocab,
                              const float* pos, int64_t D, float* out, int64_t ldo, dwm_stream_t stream) {
  DWM_REQUIRE(ids && tok && out, "dwm_b200_embed: null ids/tok/out");
  DWM_REQUIRE(M > 0 && M < (1ll << 31) && seq > 0 && vocab > 0 && D > 0 && D % 4 == 0 && D < (1ll << 31) &&
                  ldo >= D && ldo % 4 == 0,
              "dwm_b200_embed: need M, seq, vocab > 0, D a multiple of 4, ldo >= D a multiple of 4");
  DWM_REQUIRE(is_aligned(tok, 16) && is_aligned(pos, 16) && is_aligned(out, 16) && is_aligned(ids, 8),
              "dwm_b200_embed: tok, pos, out must be 16-byte and ids 8-byte aligned");
  const int threads = D >= 1024 ? 256 : 128;
  embed_kernel<<<static_cast<unsigned>(M), threads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(ids), M, seq, tok, vocab, pos, static_cast<int>(D), out, ldo);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_lincomb2(const float* x, const float* y, const float* s0, const float* s1,
                                 int64_t n, int64_t inner, float* out, dwm_stream_t stream) {
  DWM_REQUIRE(x && y && s0 && s1 && out && n > 0 && inner > 0 && n % inner == 0, "dwm_b200_lincomb2: bad arguments");
  const unsigned grid = static_cast<unsigned>((n + 255) / 256);
  lincomb2_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, y, s0, s1, n, inner, out);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static bool disjoint(const float* a, int64_t na, const float* b, int64_t nb) {
  return a + na <= b || b + nb <= a;
}

extern "C" int dwm_b200_cfg_dpmpp_step(const float* pred, int cfg, float w_uncond, float w_cond, int64_t n,
                                       const float* row, float* latents, float* x0_prev, dwm_stream_t stream) {
  DWM_REQUIRE(pred && row && latents && x0_prev, "dwm_b200_cfg_dpmpp_step: null pred/row/latents/x0_prev");
  DWM_REQUIRE(cfg == 1 || cfg == 2, "dwm_b200_cfg_dpmpp_step: cfg must be 1 or 2, got %d", cfg);
  DWM_REQUIRE(n > 0 && (n + 255) / 256 <= INT32_MAX, "dwm_b200_cfg_dpmpp_step: bad n %lld", (long long)n);
  DWM_REQUIRE(is_aligned(pred, 4) && is_aligned(row, 4) && is_aligned(latents, 4) && is_aligned(x0_prev, 4),
              "dwm_b200_cfg_dpmpp_step: pred, row, latents, x0_prev must be 4-byte aligned");
  DWM_REQUIRE(disjoint(latents, n, x0_prev, n) && disjoint(latents, n, pred, cfg * n) &&
                  disjoint(x0_prev, n, pred, cfg * n) && disjoint(row, 6, latents, n) && disjoint(row, 6, x0_prev, n),
              "dwm_b200_cfg_dpmpp_step: latents and x0_prev must not overlap each other, pred or row");
  const unsigned grid = static_cast<unsigned>((n + 255) / 256);
  cfg_dpmpp_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(pred, cfg, w_uncond, w_cond, n, row,
                                                                             latents, x0_prev);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_axpy(const float* x, float* y, int64_t n, float a, dwm_stream_t stream) {
  DWM_REQUIRE(x && y && n > 0, "dwm_b200_axpy: bad arguments");
  DWM_REQUIRE(is_aligned(x, 16) && is_aligned(y, 16), "dwm_b200_axpy: x and y must be 16-byte aligned");
  const unsigned grid = static_cast<unsigned>((n / 4 + 1 + 255) / 256);
  axpy_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, y, n, a);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_softmax_rows(const float* x, int64_t rows, int64_t cols, int64_t ld, float scale, void* out,
                                     int64_t ldo, int dtype, dwm_stream_t stream) {
  DWM_REQUIRE(x && out && rows > 0 && cols > 0 && ld >= cols && ldo >= cols && rows < (1ll << 31) &&
                  cols < (1ll << 31),
              "dwm_b200_softmax_rows: bad arguments");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const float sl = scale * 1.4426950408889634f;
  const unsigned grid = static_cast<unsigned>(rows);
  if (dtype == DWM_BF16)
    softmax_rows_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(x, ld, (int)cols, sl, static_cast<__nv_bfloat16*>(out), ldo);
  else if (dtype == DWM_F16)
    softmax_rows_kernel<__half><<<grid, 256, 0, s>>>(x, ld, (int)cols, sl, static_cast<__half*>(out), ldo);
  else { set_last_error("dwm_b200_softmax_rows: bad dtype %d", dtype); return -1; }
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_cfg_ddim_step(const float* pred, int cfg, float guidance_scale, int64_t n_items,
                                      int64_t inner, const int32_t* timesteps, int step_ratio,
                                      const float* alphas_cumprod, int n_alphas, float final_alpha_cumprod,
                                      int prediction_type, float* latents, int round_dtype, dwm_stream_t stream) {
  DWM_REQUIRE(pred && timesteps && alphas_cumprod && latents, "dwm_b200_cfg_ddim_step: null pointer");
  DWM_REQUIRE((cfg == 1 || cfg == 2) && n_items > 0 && inner > 0 && n_alphas > 0 && prediction_type >= 0 &&
                  prediction_type <= 2,
              "dwm_b200_cfg_ddim_step: bad arguments");
  const long long total = n_items * inner;
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  cfg_ddim_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      pred, cfg, guidance_scale, 0, inner, total, timesteps, step_ratio, alphas_cumprod, n_alphas, final_alpha_cumprod,
      prediction_type, latents, round_dtype);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_euler_step_by_indices(const float* model_output, float* sample, int64_t n,
                                              int64_t inner, const int32_t* idx, const float* sigmas,
                                              int n_sigmas, int round_dtype, dwm_stream_t stream) {
  DWM_REQUIRE(model_output && sample && idx && sigmas && n > 0 && inner > 0 && n % inner == 0 && n_sigmas > 1,
              "dwm_b200_euler_step_by_indices: bad arguments");
  const unsigned grid = static_cast<unsigned>((n + 255) / 256);
  euler_idx_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(model_output, sample, n, inner, idx,
                                                                            sigmas, n_sigmas, round_dtype);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_layernorm(const dwm_layernorm_args* a, dwm_stream_t stream) {
  DWM_REQUIRE(a != nullptr, "dwm_b200_layernorm: null args");
  DWM_REQUIRE(a->M > 0 && a->D > 0 && a->M < (1ll << 31), "dwm_b200_layernorm: bad M/D");
  DWM_REQUIRE(a->D % 4 == 0 && a->D <= 2048, "dwm_b200_layernorm: D must be a multiple of 4 and <= 2048, got %lld", (long long)a->D);
  DWM_REQUIRE(a->x && a->out, "dwm_b200_layernorm: null x/out");
  DWM_REQUIRE(a->ldx % 4 == 0 && a->ldo % 4 == 0, "dwm_b200_layernorm: ldx/ldo must be multiples of 4");
  if (a->shift || a->scale || a->shift2 || a->scale2)
    DWM_REQUIRE(a->mod_ld % 4 == 0, "dwm_b200_layernorm: mod_ld must be a multiple of 4");
  // every fp32 operand is read (sum_out written) as float4
  const float* f32s[] = {a->x, a->add_item, a->add_full, a->sum_out, a->weight, a->bias,
                         a->shift, a->scale, a->shift2, a->scale2};
  for (const float* q : f32s)
    DWM_REQUIRE(is_aligned(q, 16),
                "dwm_b200_layernorm: x, add_item, add_full, sum_out, weight, bias, shift, scale, shift2, scale2 "
                "must be 16-byte aligned");
  DWM_REQUIRE((!a->add_item || a->add_item_ld % 4 == 0) && (!a->add_full || a->add_full_ld % 4 == 0) &&
                  (!a->sum_out || a->ld_sum % 4 == 0) && (!a->out2 || a->ldo2 % 4 == 0),
              "dwm_b200_layernorm: add_item_ld, add_full_ld, ld_sum, ldo2 must be multiples of 4");
  // four outputs per store: 8 bytes of 16-bit values, 4 bytes of E4M3
  const uintptr_t out_align = a->dtype == DWM_E4M3 ? 4 : 8;
  DWM_REQUIRE(is_aligned(a->out, out_align) && is_aligned(a->out2, out_align),
              "dwm_b200_layernorm: out and out2 must be %d-byte aligned", (int)out_align);
  LnParams p;
  p.M = static_cast<int>(a->M); p.D = static_cast<int>(a->D);
  p.x = a->x; p.ldx = a->ldx;
  p.add_item = a->add_item; p.add_item_ld = a->add_item_ld;
  p.add_full = a->add_full; p.add_full_ld = a->add_full_ld;
  p.rows_per_item = static_cast<int>(a->rows_per_item);
  p.sum_out = a->sum_out; p.ld_sum = a->ld_sum;
  p.weight = a->weight; p.bias = a->bias; p.eps = a->eps;
  p.shift = a->shift; p.scale = a->scale; p.shift2 = a->shift2; p.scale2 = a->scale2; p.mod_ld = a->mod_ld;
  p.out = a->out; p.ldo = a->ldo; p.out2 = a->out2; p.ldo2 = a->ldo2;
  p.out_scale = a->out_scale; p.out2_scale = a->out2_scale;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (a->dtype == DWM_BF16) return launch_ln<__nv_bfloat16>(p, s);
  if (a->dtype == DWM_F16) return launch_ln<__half>(p, s);
  if (a->dtype == DWM_E4M3) {
    DWM_REQUIRE(a->out_scale && (!a->out2 || a->out2_scale),
                "dwm_b200_layernorm: E4M3 output needs out_scale (and out2_scale with out2)");
    return launch_ln<__nv_fp8_e4m3>(p, s);
  }
  set_last_error("dwm_b200_layernorm: dtype must be DWM_BF16, DWM_F16 or DWM_E4M3");
  return -1;
}

extern "C" int dwm_b200_quantize_rows(const void* x, int64_t M, int64_t K, int64_t ld, int dtype, void* out,
                                      int64_t ldo, float* scale, dwm_stream_t stream) {
  DWM_REQUIRE(x && out && scale, "dwm_b200_quantize_rows: null x/out/scale");
  DWM_REQUIRE(M > 0 && K > 0 && M < (1ll << 31) && K < (1ll << 31), "dwm_b200_quantize_rows: bad M/K");
  DWM_REQUIRE(K % 16 == 0 && ld % 8 == 0 && ldo % 16 == 0 && ld >= K && ldo >= K,
              "dwm_b200_quantize_rows: K and ldo must be multiples of 16 and ld of 8 (ld, ldo >= K); "
              "got K=%lld ld=%lld ldo=%lld", (long long)K, (long long)ld, (long long)ldo);
  DWM_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
              "dwm_b200_quantize_rows: x and out must be 16-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const unsigned grid = static_cast<unsigned>((M + QR_WARPS - 1) / QR_WARPS);
  const int Mi = static_cast<int>(M), Ki = static_cast<int>(K);
  uint8_t* o = reinterpret_cast<uint8_t*>(out);
  if (dtype == DWM_BF16)
    quantize_rows_kernel<<<grid, QR_WARPS * 32, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x), Mi, Ki, ld, o, ldo, scale);
  else if (dtype == DWM_F16)
    quantize_rows_kernel<<<grid, QR_WARPS * 32, 0, s>>>(reinterpret_cast<const __half*>(x), Mi, Ki, ld, o, ldo, scale);
  else if (dtype == DWM_F32)
    quantize_rows_kernel<<<grid, QR_WARPS * 32, 0, s>>>(reinterpret_cast<const float*>(x), Mi, Ki, ld, o, ldo, scale);
  else
    DWM_REQUIRE(false, "dwm_b200_quantize_rows: dtype must be DWM_BF16, DWM_F16 or DWM_F32, got %d", dtype);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_act_cast(const float* in, void* out, int64_t n, int act, int dtype, dwm_stream_t stream) {
  DWM_REQUIRE(in && out && n > 0, "dwm_b200_act_cast: bad arguments");
  DWM_REQUIRE(act == DWM_ACT_NONE || act == DWM_ACT_SILU || act == DWM_ACT_GELU_TANH || act == DWM_ACT_GELU_ERF,
              "dwm_b200_act_cast: activation %d is not implemented (NONE, SILU, GELU_TANH, GELU_ERF)", act);
  DWM_REQUIRE(is_aligned(in, 16) && is_aligned(out, 8),
              "dwm_b200_act_cast: in must be 16-byte and out 8-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const unsigned grid = static_cast<unsigned>((n / 4 + 1 + 255) / 256);
  if (dtype == DWM_BF16) act_cast_kernel<<<grid, 256, 0, s>>>(in, reinterpret_cast<__nv_bfloat16*>(out), n, act);
  else if (dtype == DWM_F16) act_cast_kernel<<<grid, 256, 0, s>>>(in, reinterpret_cast<__half*>(out), n, act);
  else { set_last_error("dwm_b200_act_cast: bad dtype"); return -1; }
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_sinusoid(const float* t, int64_t n, int channels, int flip, float shift,
                                 void* out, int64_t ldo, int dtype, dwm_stream_t stream) {
  DWM_REQUIRE(t && out && n > 0 && channels > 0 && channels % 2 == 0, "dwm_b200_sinusoid: bad arguments");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = n * (channels / 2);
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  if (dtype == DWM_BF16) sinusoid_kernel<<<grid, 256, 0, s>>>(t, n, channels, flip, shift, reinterpret_cast<__nv_bfloat16*>(out), ldo);
  else if (dtype == DWM_F16) sinusoid_kernel<<<grid, 256, 0, s>>>(t, n, channels, flip, shift, reinterpret_cast<__half*>(out), ldo);
  else { set_last_error("dwm_b200_sinusoid: bad dtype"); return -1; }
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_patchify(const float* x, int64_t items, int C, int H, int W, int patch,
                                 void* out, int64_t ldo, int dtype, dwm_stream_t stream) {
  DWM_REQUIRE(x && out && items > 0 && patch > 0 && H % patch == 0 && W % patch == 0, "dwm_b200_patchify: bad arguments");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = items * C * H * W;
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  if (dtype == DWM_BF16) patchify_kernel<<<grid, 256, 0, s>>>(x, items, C, H, W, patch, reinterpret_cast<__nv_bfloat16*>(out), ldo);
  else if (dtype == DWM_F16) patchify_kernel<<<grid, 256, 0, s>>>(x, items, C, H, W, patch, reinterpret_cast<__half*>(out), ldo);
  else { set_last_error("dwm_b200_patchify: bad dtype"); return -1; }
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_cfg_euler_step(const float* tokens, int64_t ld_tok, int cfg, float guidance_scale,
                                       int64_t B, int64_t T, int64_t V, int C, int H, int W, int patch,
                                       const int32_t* idx, const float* sigmas, int n_sigmas,
                                       const unsigned char* in_range, float* latents, float* noise_pred,
                                       int round_dtype, dwm_stream_t stream) {
  DWM_REQUIRE(tokens && idx && sigmas && latents, "dwm_b200_cfg_euler_step: null pointer");
  DWM_REQUIRE(cfg == 1 || cfg == 2, "dwm_b200_cfg_euler_step: cfg must be 1 or 2");
  DWM_REQUIRE(B > 0 && T > 0 && V > 0 && C > 0 && patch > 0 && H % patch == 0 && W % patch == 0 && n_sigmas > 1,
              "dwm_b200_cfg_euler_step: bad shape");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = B * T * V * C * H * W;
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  cfg_euler_kernel<<<grid, 256, 0, s>>>(tokens, ld_tok, cfg, guidance_scale, B, T, V, C, H, W, patch, idx,
                                        sigmas, n_sigmas, in_range, latents, noise_pred, round_dtype);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}
