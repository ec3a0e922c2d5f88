// HBM-bound kernels of the CogVideoX temporal-VAE decoder (channels-last activations):
// GroupNorm statistics, the fused SpatialNorm3D (GroupNorm * conv_y(zq) + conv_b(zq)) +
// SiLU that writes the 16-bit, causally time-padded input of the next convolution (or, for
// the FP8 UNet ResBlock and VAE ResNet convs, its E4M3 version with one scale per volume), and the
// nearest-neighbour (space / space-time) upsampler.
#include <algorithm>

#include "common.cuh"
#include "../../include/dwm_b200.h"

namespace dwm {

// ---- GroupNorm statistics: sums[n][g] = (sum x, sum x^2) over (C/G channels, all pixels) ----
// Every loaded float is widened to double before it is added or squared, and the per-thread
// partials, the per-block shared-memory reduction and the cross-block atomics all stay in
// double.  The apply kernel forms the variance as sum x^2 / n - mean^2, which cancels when
// |mean| >> std: an fp32 accumulation lost every significant bit of the variance of groups
// with |mean| / std ~ 1e3 and made it negative (NaN output) for constant groups.  The
// kernels remain HBM-bound; the (sum, sum sq) format is what ShardPlan.reduce_group_sums
// all-reduces across frame shards.
__device__ __forceinline__ void gn_acc(double& s, double& q, float v) {
  const double d = static_cast<double>(v);
  s += d;
  q = fma(d, d, q);
}

// block = 256 threads; thread handles float4 channel vector c4 = tid % (C/4) of pixels
// tid / (C/4), +stride...  Partial sums are combined per group in shared memory, then one
// double atomicAdd per (block, group).
__global__ void __launch_bounds__(256) gn_stats_kernel(const float* __restrict__ x, long long pixels, int C, int G,
                                                       long long pixels_per_block, double* __restrict__ sums) {
  __shared__ double s_sum[64], s_sq[64];
  const int n = blockIdx.y;
  const int vec = C >> 2;
  const int tid = threadIdx.x;
  if (tid < 64) { s_sum[tid] = 0.0; s_sq[tid] = 0.0; }
  __syncthreads();
  const int c4 = tid % vec;
  const int prow = tid / vec;
  const int rows_per_iter = 256 / vec;
  const long long p0 = static_cast<long long>(blockIdx.x) * pixels_per_block;
  long long p1 = p0 + pixels_per_block;
  if (p1 > pixels) p1 = pixels;
  double a = 0.0, b = 0.0;
  if (prow < rows_per_iter) {
    const float4* base = reinterpret_cast<const float4*>(x + static_cast<long long>(n) * pixels * C);
    for (long long p = p0 + prow; p < p1; p += rows_per_iter) {
      const float4 v = base[p * vec + c4];
      gn_acc(a, b, v.x); gn_acc(a, b, v.y); gn_acc(a, b, v.z); gn_acc(a, b, v.w);
    }
  }
  const int g = (c4 * 4) / (C / G);
  atomicAdd(&s_sum[g], a);
  atomicAdd(&s_sq[g], b);
  __syncthreads();
  if (tid < G) {
    atomicAdd(&sums[(static_cast<long long>(n) * G + tid) * 2], s_sum[tid]);
    atomicAdd(&sums[(static_cast<long long>(n) * G + tid) * 2 + 1], s_sq[tid]);
  }
}

// wide variant: any C % 4 == 0 with C / 4 <= 1024 and any group size (UNet widths 320 ... 2560,
// 10 / 20 / 40 ... channels per group).  blockDim = (C/4) * k so that every thread keeps ONE
// channel quad for all its pixels: per-element register sums, then at most 4 shared atomics
// per thread and one double atomic per (block, group).
__global__ void __launch_bounds__(1024) gn_stats_wide_kernel(const float* __restrict__ x, long long pixels, int C, int G,
                                                             long long pixels_per_block, double* __restrict__ sums) {
  __shared__ double s_sum[64], s_sq[64];
  const int n = blockIdx.y, tid = threadIdx.x;
  const int vec = C >> 2;
  if (tid < 64) { s_sum[tid] = 0.0; s_sq[tid] = 0.0; }
  __syncthreads();
  const int c4 = tid % vec, prow = tid / vec, k = blockDim.x / vec;
  const long long p0 = static_cast<long long>(blockIdx.x) * pixels_per_block;
  long long p1 = p0 + pixels_per_block;
  if (p1 > pixels) p1 = pixels;
  double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0, q0 = 0.0, q1 = 0.0, q2 = 0.0, q3 = 0.0;
  const float4* base = reinterpret_cast<const float4*>(x + static_cast<long long>(n) * pixels * C);
  for (long long p = p0 + prow; p < p1; p += k) {
    const float4 v = base[p * vec + c4];
    gn_acc(s0, q0, v.x); gn_acc(s1, q1, v.y); gn_acc(s2, q2, v.z); gn_acc(s3, q3, v.w);
  }
  const int cg = C / G;
  const double ss[4] = {s0, s1, s2, s3}, qq[4] = {q0, q1, q2, q3};
  int cur = (c4 * 4) / cg;
  double a = 0.0, b = 0.0;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int g = (c4 * 4 + e) / cg;
    if (g != cur) {
      atomicAdd(&s_sum[cur], a); atomicAdd(&s_sq[cur], b);
      cur = g; a = 0.0; b = 0.0;
    }
    a += ss[e]; b += qq[e];
  }
  atomicAdd(&s_sum[cur], a); atomicAdd(&s_sq[cur], b);
  __syncthreads();
  if (tid < G) {
    atomicAdd(&sums[(static_cast<long long>(n) * G + tid) * 2], s_sum[tid]);
    atomicAdd(&sums[(static_cast<long long>(n) * G + tid) * 2 + 1], s_sq[tid]);
  }
}

// last-resort variant (C / 4 > 1024): any C, any group size (scalar loads; UNet widths 320 / 960 / 1920 ...)
__global__ void __launch_bounds__(256) gn_stats_generic_kernel(const float* __restrict__ x, long long pixels, int C,
                                                               int G, long long pixels_per_block,
                                                               double* __restrict__ sums) {
  __shared__ double s_sum[64], s_sq[64];
  const int n = blockIdx.y, tid = threadIdx.x;
  if (tid < 64) { s_sum[tid] = 0.0; s_sq[tid] = 0.0; }
  __syncthreads();
  const int cg = C / G;
  const long long e0 = static_cast<long long>(blockIdx.x) * pixels_per_block * C;
  long long e1 = e0 + pixels_per_block * C;
  if (e1 > pixels * C) e1 = pixels * C;
  const float* base = x + static_cast<long long>(n) * pixels * C;
  // consecutive threads read consecutive elements; accumulate runs of equal group locally
  int cur_g = -1;
  double a = 0.0, b = 0.0;
  for (long long e = e0 + tid; e < e1; e += 256) {
    const int g = static_cast<int>(e % C) / cg;
    if (g != cur_g) {
      if (cur_g >= 0) { atomicAdd(&s_sum[cur_g], a); atomicAdd(&s_sq[cur_g], b); }
      cur_g = g; a = 0.0; b = 0.0;
    }
    gn_acc(a, b, base[e]);
  }
  if (cur_g >= 0) { atomicAdd(&s_sum[cur_g], a); atomicAdd(&s_sq[cur_g], b); }
  __syncthreads();
  if (tid < G) {
    atomicAdd(&sums[(static_cast<long long>(n) * G + tid) * 2], s_sum[tid]);
    atomicAdd(&sums[(static_cast<long long>(n) * G + tid) * 2 + 1], s_sq[tid]);
  }
}

// ---- SpatialNorm3D / GroupNorm apply (+SiLU) -> 16-bit, written at a frame offset ----
struct SnParams {
  const float* x; int nb, T, H, W, C, G;
  const double* sums; float eps;
  const float* gamma; const float* beta;
  const float* zy; const float* zb; int Tz, hz, wz;
  int silu;
  void* out; int out_T, out_t0;
  float* scale;   // E4M3 output: [nb] amax bits (SN_AMAX pass), then the volume scale
  int stat_T;     // frames the GroupNorm sums cover (T, or the whole window of a frame shard)
  // HALO: frame-shard operand [nb, T + 2, H, W, C]; local frame 0 is also stored at frame
  // prev_T - 1 of prev_out, the last local frame at frame 0 of next_out (both [nb, *_T, H, W, C]);
  // without a neighbour the own halo frame is stored as zero.
  // SN_E4M3_TAIL (no HALO): next_out is the 16-bit [nb, 2, H, W, C] causal-conv cache of the
  // next chunk, the operand's last two frames; prev_out the cache this call's operand starts with
  // (NULL: a first chunk, whose leading frames replicate frame out_t0)
  void* prev_out = nullptr; int prev_T = 0;
  void* next_out = nullptr; int next_T = 0;
};

// What a spatialnorm_kernel pass does with each normalised float4: store it as 16 bit, only
// fold it into the volume's amax, or store it as E4M3 with the volume's inverse scale
// (SN_E4M3_TAIL: and the operand's last two frames once more as T into next_out).
enum { SN_STORE16 = 0, SN_AMAX = 1, SN_E4M3 = 2, SN_E4M3_TAIL = 3 };

// grid = (chunks, nb): a block works on one chunk (16 float4 per thread) of ONE image, so the (mean, rstd) of its
// G groups are finalised once per block from the fp64 sums (first G threads, shared memory)
// instead of per thread — the fp64 divisions made the per-thread version XU-pipe bound.

// Per-thread state is set up ONCE: with blockDim a multiple of C/4 a thread keeps the same
// channel quad for all its elements, so gamma / beta / (mean, rstd) are registers, the pixel
// position (t, h, w) advances by a constant number of pixels per iteration and is tracked with
// carries instead of 64-bit divisions, the latent-grid coordinates are shifts when the sizes
// are powers of two apart (always in the VAEs) and the frame map is a 64-entry shared table.
// A version that spent ~10 integer divisions per float4 was far from DRAM-bound; this one is
// a plain stream.
template <typename T, int MODE = SN_STORE16, bool HALO = false>
__global__ void __launch_bounds__(1024) spatialnorm_kernel(const SnParams p, const int chunk) {
  // blockDim.x is a multiple of C/4 whenever C/4 <= 1024 (host side), `chunk` = blockDim.x * 16
  __shared__ float2 s_stat[64];
  __shared__ int s_tz[64];
  __shared__ unsigned int s_amax;
  const int NT = static_cast<int>(blockDim.x);
  const int vec = p.C >> 2;
  const int n = blockIdx.y;
  const int cg = p.C / p.G;
  const long long per_img = static_cast<long long>(p.T) * p.H * p.W * vec;
  if (threadIdx.x < p.G) {
    const double cnt = static_cast<double>(cg) * p.stat_T * p.H * p.W;
    const double s = p.sums[(static_cast<long long>(n) * p.G + threadIdx.x) * 2];
    const double ss = p.sums[(static_cast<long long>(n) * p.G + threadIdx.x) * 2 + 1];
    const double mean_d = s / cnt;
    // rounding of the sums can leave a (near-)constant group a variance slightly below 0
    const double var_d = fmax(ss / cnt - mean_d * mean_d, 0.0);
    s_stat[threadIdx.x] = make_float2(static_cast<float>(mean_d), rsqrtf(static_cast<float>(var_d) + p.eps));
  }
  if (MODE == SN_AMAX && threadIdx.x == 0) s_amax = 0u;
  if (p.zy && threadIdx.x < 64 && threadIdx.x < p.T) {
    // nearest-neighbour frame of the latent grid; odd T > 1 treats the first frame apart
    const int t = threadIdx.x;
    s_tz[t] = (p.T > 1 && (p.T & 1)) ? (t == 0 ? 0 : 1 + ((t - 1) * (p.Tz - 1)) / (p.T - 1))
                                     : (t * p.Tz) / p.T;
  }
  __syncthreads();
  // SN_AMAX: max |v| of this thread, reduced per block in shared memory, then one atomicMax
  // per block on the bits of the non-negative fp32 value (their integer order is the float
  // order, so the result does not depend on the order of the atomics).  Blocks need not be
  // whole warps (C/4 = 80 gives 240 threads), hence no warp shuffles.
  float amax = 0.f;
  float inv = 0.f;
  if constexpr (MODE == SN_E4M3 || MODE == SN_E4M3_TAIL) inv = e4m3_inv(__uint_as_float(reinterpret_cast<const uint32_t*>(p.scale)[n]));
  auto store = [&](void* base, long long o, const float4& v) {
    if constexpr (MODE == SN_STORE16) {
      uint2 pk; pk.x = Cvt<T>::pack2(v.x, v.y); pk.y = Cvt<T>::pack2(v.z, v.w);
      reinterpret_cast<uint2*>(base)[o] = pk;
    } else {
      reinterpret_cast<uint32_t*>(base)[o] = e4m3x4(v.x, v.y, v.z, v.w, inv);
    }
  };
  // the zero time padding, stored as bits (E4M3 through e4m3x4 left non-zero upper bytes)
  auto store_zero = [&](long long o) {
    if constexpr (MODE == SN_STORE16) reinterpret_cast<uint2*>(p.out)[o] = make_uint2(0u, 0u);
    else reinterpret_cast<uint32_t*>(p.out)[o] = 0u;
  };
  // frame-to-frame distance of the output in float4 units (HALO offsets are whole frames)
  const long long frame4 = static_cast<long long>(p.H) * p.W * vec;
  auto emit = [&](long long o, const float4& v, int t) {
    if constexpr (MODE == SN_AMAX) {
      amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    } else {
      store(p.out, o, v);
      if constexpr (MODE == SN_E4M3_TAIL) {
        // operand frame out_t0 + t is tail frame tt; with T = 1 and no previous tail, tail frame
        // 0 is its replica
        const int tt = t + 2 - p.T;
        if (tt >= 0) {
          uint2 pk; pk.x = Cvt<T>::pack2(v.x, v.y); pk.y = Cvt<T>::pack2(v.z, v.w);
          const long long ot = o + (static_cast<long long>(n) * (2 - p.out_T) - p.out_t0 - t + tt) * frame4;
          reinterpret_cast<uint2*>(p.next_out)[ot] = pk;
          if (p.T == 1 && !p.prev_out) reinterpret_cast<uint2*>(p.next_out)[ot - frame4] = pk;
        }
      }
      if constexpr (HALO) {
        // o = ((n * out_T + out_t0 + t) * H*W + pixel) * vec + c4; re-based onto a neighbour's
        // frame by whole frames
        if (t == 0) {
          if (p.prev_out)
            store(p.prev_out, o + (static_cast<long long>(n) * (p.prev_T - p.out_T) + p.prev_T - 1 - p.out_t0) * frame4, v);
          else
            store_zero(o - frame4);
        }
        if (t == p.T - 1) {
          if (p.next_out)
            store(p.next_out, o + (static_cast<long long>(n) * (p.next_T - p.out_T) - p.out_t0 - t) * frame4, v);
          else
            store_zero(o + frame4);
        }
      }
    }
  };
  auto finish = [&]() {
    if constexpr (MODE == SN_AMAX) {
      atomicMax(&s_amax, __float_as_uint(amax));
      __syncthreads();
      if (threadIdx.x == 0) atomicMax(reinterpret_cast<unsigned int*>(p.scale) + n, s_amax);
    }
  };
  const long long i0 = static_cast<long long>(blockIdx.x) * chunk;
  long long i1 = i0 + chunk;
  if (i1 > per_img) i1 = per_img;
  const float4* xin = reinterpret_cast<const float4*>(p.x) + static_cast<long long>(n) * per_img;
  const float4* g4 = reinterpret_cast<const float4*>(p.gamma);
  const float4* b4 = reinterpret_cast<const float4*>(p.beta);
  const bool fast = (NT % vec) == 0 && (chunk % vec) == 0 && p.T <= 64;
  if (fast) {
    const int c4 = threadIdx.x % vec;
    const int pstep = NT / vec;                                   // pixels per iteration
    long long pix = i0 / vec + threadIdx.x / vec;                 // i0 % vec == 0
    int w = static_cast<int>(pix % p.W);
    long long r = pix / p.W;
    int h = static_cast<int>(r % p.H);
    int t = static_cast<int>(r / p.H);
    const float4 ga = __ldg(g4 + c4), be = __ldg(b4 + c4);
    // the four channels of the quad may sit in different groups (UNet: 10 / 20 / 40 channels
    // per group): one (mean, rstd) per element, all in registers
    const float2 st0 = s_stat[(c4 * 4) / cg], st1 = s_stat[(c4 * 4 + 1) / cg];
    const float2 st2 = s_stat[(c4 * 4 + 2) / cg], st3 = s_stat[(c4 * 4 + 3) / cg];
    // (x - mean) * (rstd * gamma) + beta: the subtraction stays first (no cancellation in a
    // pre-folded offset when |mean| >> std)
    const float4 aa = make_float4(st0.y * ga.x, st1.y * ga.y, st2.y * ga.z, st3.y * ga.w);
    const float4 mu = make_float4(st0.x, st1.x, st2.x, st3.x);
    // latent-grid coordinates: shifts when H = hz << k (else a division per element)
    int hs = -1, ws = -1;
    if (p.zy) {
      for (int k = 0; k < 8; ++k) {
        if ((p.hz << k) == p.H) hs = k;
        if ((p.wz << k) == p.W) ws = k;
      }
    }
    const long long zn = static_cast<long long>(n) * p.Tz;
    const long long on = static_cast<long long>(n) * p.out_T + p.out_t0;
    for (long long i = i0 + threadIdx.x; i < i1; i += NT) {
      float4 v = xin[i];
      v.x = fmaf(v.x - mu.x, aa.x, be.x); v.y = fmaf(v.y - mu.y, aa.y, be.y);
      v.z = fmaf(v.z - mu.z, aa.z, be.z); v.w = fmaf(v.w - mu.w, aa.w, be.w);
      if (p.zy) {
        const int hq = hs >= 0 ? (h >> hs) : (h * p.hz) / p.H;
        const int wq = ws >= 0 ? (w >> ws) : (w * p.wz) / p.W;
        const long long zi = (((zn + s_tz[t]) * p.hz + hq) * p.wz + wq) * vec + c4;
        const float4 y = __ldg(reinterpret_cast<const float4*>(p.zy) + zi);
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.zb) + zi);
        v.x = fmaf(v.x, y.x, b.x); v.y = fmaf(v.y, y.y, b.y);
        v.z = fmaf(v.z, y.z, b.z); v.w = fmaf(v.w, y.w, b.w);
      }
      if (p.silu) { v.x = silu(v.x); v.y = silu(v.y); v.z = silu(v.z); v.w = silu(v.w); }
      const long long o = (((on + t) * p.H + h) * p.W + w) * vec + c4;
      emit(o, v, t);
      w += pstep;
      while (w >= p.W) { w -= p.W; if (++h == p.H) { h = 0; ++t; } }
    }
    finish();
    return;
  }
  // general path (C / 4 > 1024 or more than 64 frames)
  for (long long i = i0 + threadIdx.x; i < i1; i += NT) {
    const int c4 = static_cast<int>(i % vec);
    long long r = i / vec;
    const int w = static_cast<int>(r % p.W); r /= p.W;
    const int h = static_cast<int>(r % p.H);
    const int t = static_cast<int>(r / p.H);
    float4 v = xin[i];
    const float4 ga = __ldg(g4 + c4);
    const float4 be = __ldg(b4 + c4);
    if ((cg & 3) == 0) {
      const float2 st = s_stat[(c4 * 4) / cg];
      v.x = (v.x - st.x) * st.y * ga.x + be.x;
      v.y = (v.y - st.x) * st.y * ga.y + be.y;
      v.z = (v.z - st.x) * st.y * ga.z + be.z;
      v.w = (v.w - st.x) * st.y * ga.w + be.w;
    } else {   // a float4 may straddle groups (e.g. 10 or 2 channels per group)
      float* ve = reinterpret_cast<float*>(&v);
      const float* gae = reinterpret_cast<const float*>(&ga);
      const float* bee = reinterpret_cast<const float*>(&be);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 st = s_stat[(c4 * 4 + e) / cg];
        ve[e] = (ve[e] - st.x) * st.y * gae[e] + bee[e];
      }
    }
    if (p.zy) {
      int tz;
      if (p.T > 1 && (p.T & 1)) tz = t == 0 ? 0 : 1 + ((t - 1) * (p.Tz - 1)) / (p.T - 1);
      else tz = (t * p.Tz) / p.T;
      const int hq = (h * p.hz) / p.H, wq = (w * p.wz) / p.W;
      const long long zi = (((static_cast<long long>(n) * p.Tz + tz) * p.hz + hq) * p.wz + wq) * vec + c4;
      const float4 y = __ldg(reinterpret_cast<const float4*>(p.zy) + zi);
      const float4 b = __ldg(reinterpret_cast<const float4*>(p.zb) + zi);
      v.x = v.x * y.x + b.x; v.y = v.y * y.y + b.y; v.z = v.z * y.z + b.z; v.w = v.w * y.w + b.w;
    }
    if (p.silu) { v.x = silu(v.x); v.y = silu(v.y); v.z = silu(v.z); v.w = silu(v.w); }
    const long long o = (((static_cast<long long>(n) * p.out_T + p.out_t0 + t) * p.H + h) * p.W + w) * vec + c4;
    emit(o, v, t);
  }
  finish();
}

// amax (bits, left by the SN_AMAX pass; may alias scale) -> E4M3 volume scale
__global__ void e4m3_amax_to_scale_kernel(const float* amax, float* scale, int nb) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n < nb) scale[n] = e4m3_scale(__uint_as_float(reinterpret_cast<const uint32_t*>(amax)[n]));
}

// The previous chunk's 16-bit causal-conv cache tail [nb, 2, H, W, C] (frame4 float4 groups per
// frame) as frames out_t0 - 2, out_t0 - 1 of this chunk's E4M3 operand, under the chunk's volume
// scale.  AMAX: folds max |tail| into the amax bits of each volume.  Else: quantizes the tail
// with that amax and, when next_tail is given (T = 1: the new tail is tail frame 1 and the new
// frame), stores tail frame 1 as next_tail's frame 0; tail and next_tail may be one buffer.
template <typename T, bool AMAX>
__global__ void __launch_bounds__(256) sn_tail_kernel(const void* tail, long long frame4, float* amax, void* out,
                                                      int out_T, int out_t0, void* next_tail) {
  const int n = blockIdx.y;
  const uint2* src = reinterpret_cast<const uint2*>(tail) + static_cast<long long>(n) * 2 * frame4;
  float inv = 0.f, a = 0.f;
  if constexpr (!AMAX) inv = e4m3_inv(__uint_as_float(reinterpret_cast<const uint32_t*>(amax)[n]));
  uint32_t* dst = reinterpret_cast<uint32_t*>(out) + (static_cast<long long>(n) * out_T + out_t0 - 2) * frame4;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < frame4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint2 u[2] = {src[i], src[frame4 + i]};
#pragma unroll
    for (int f = 0; f < 2; ++f) {
      const float2 lo = Cvt<T>::unpack2(u[f].x), hi = Cvt<T>::unpack2(u[f].y);
      if constexpr (AMAX) a = fmaxf(a, fmaxf(fmaxf(fabsf(lo.x), fabsf(lo.y)), fmaxf(fabsf(hi.x), fabsf(hi.y))));
      else dst[f * frame4 + i] = e4m3x4(lo.x, lo.y, hi.x, hi.y, inv);
    }
    if constexpr (!AMAX) {
      if (next_tail) reinterpret_cast<uint2*>(next_tail)[static_cast<long long>(n) * 2 * frame4 + i] = u[1];
    }
  }
  if constexpr (AMAX) {
    // non-negative floats: the integer order of the bits is the float order
    const unsigned int m = __reduce_max_sync(0xffffffffu, __float_as_uint(a));
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned int*>(amax) + n, m);
  }
}

// ---- nearest upsample x2 in space, optionally in time (CogVideoXUpsample3D rules) ----
template <typename T>
__global__ void __launch_bounds__(256) upsample_kernel(const float* __restrict__ x, int nb, int Ti, int H, int W, int C,
                                                       int To, int mode, T* __restrict__ out) {
  // mode 0: space only; 1: space+time all frames; 2: first frame space only, rest space+time
  const int vec = C >> 2;
  const long long total = static_cast<long long>(nb) * To * (2 * H) * (2 * W) * vec;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c4 = static_cast<int>(i % vec);
  long long r = i / vec;
  const int w = static_cast<int>(r % (2 * W)); r /= 2 * W;
  const int h = static_cast<int>(r % (2 * H)); r /= 2 * H;
  const int t = static_cast<int>(r % To);
  const int n = static_cast<int>(r / To);
  int ti;
  if (mode == 0) ti = t;
  else if (mode == 1) ti = t >> 1;
  else ti = t == 0 ? 0 : 1 + ((t - 1) >> 1);
  const float4 v = reinterpret_cast<const float4*>(x)[(((static_cast<long long>(n) * Ti + ti) * H + (h >> 1)) * W + (w >> 1)) * vec + c4];
  uint2 pk; pk.x = Cvt<T>::pack2(v.x, v.y); pk.y = Cvt<T>::pack2(v.z, v.w);
  reinterpret_cast<uint2*>(out)[i] = pk;
}

}  // namespace dwm

using namespace dwm;

namespace {
// float4 operands of the GroupNorm apply kernels; nullptr if all are aligned (null zy / zb too)
const char* gn_align_check(const float* x, const double* sums, const float* gamma, const float* beta,
                           const float* zy, const float* zb) {
  if (!is_aligned(x, 16) || !is_aligned(gamma, 16) || !is_aligned(beta, 16) || !is_aligned(zy, 16) ||
      !is_aligned(zb, 16))
    return "x, gamma, beta (zy, zb) must be 16-byte aligned";
  if (!is_aligned(sums, 8)) return "sums must be 8-byte aligned";
  return nullptr;
}
}  // namespace

extern "C" int dwm_b200_groupnorm_stats(const float* x, int64_t nb, int64_t pixels, int C, int groups,
                                        double* sums, dwm_stream_t stream) {
  DWM_REQUIRE(x && sums && nb > 0 && pixels > 0, "dwm_b200_groupnorm_stats: bad arguments");
  DWM_REQUIRE(C % 4 == 0 && groups > 0 && groups <= 64 && C % groups == 0,
              "dwm_b200_groupnorm_stats: need C %% 4 == 0, C %% groups == 0, groups <= 64 (got C=%d, groups=%d)", C, groups);
  DWM_REQUIRE(is_aligned(x, 16) && is_aligned(sums, 8),
              "dwm_b200_groupnorm_stats: x must be 16-byte and sums 8-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  DWM_CHECK_CUDA(cudaMemsetAsync(sums, 0, sizeof(double) * 2 * nb * groups, s));
  const int vec = C / 4;
  const bool fast = (C / groups) % 4 == 0 && vec <= 256 && 256 % vec == 0;
  // pixels per block: about 4 blocks per SM over the whole launch, whole thread-rows per block
  auto pick = [&](long long rows_per_iter) {
    const long long target = std::max<long long>(1, 592 / nb);
    const long long chunks = std::min((pixels + rows_per_iter - 1) / rows_per_iter, target);
    const long long ppb = (pixels + chunks - 1) / chunks;
    return (ppb + rows_per_iter - 1) / rows_per_iter * rows_per_iter;
  };
  if (fast) {
    const long long ppb = pick(256 / vec);
    dim3 grid(static_cast<unsigned>((pixels + ppb - 1) / ppb), static_cast<unsigned>(nb));
    gn_stats_kernel<<<grid, 256, 0, s>>>(x, pixels, C, groups, ppb, sums);
  } else if (vec <= 1024) {
    const int k = std::max(1, 256 / vec);
    const long long ppb = pick(k);
    dim3 grid(static_cast<unsigned>((pixels + ppb - 1) / ppb), static_cast<unsigned>(nb));
    gn_stats_wide_kernel<<<grid, vec * k, 0, s>>>(x, pixels, C, groups, ppb, sums);
  } else {
    const long long ppb = 64;
    dim3 grid(static_cast<unsigned>((pixels + ppb - 1) / ppb), static_cast<unsigned>(nb));
    gn_stats_generic_kernel<<<grid, 256, 0, s>>>(x, pixels, C, groups, ppb, sums);
  }
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_spatialnorm_silu(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W, int C,
                                         int groups, const double* sums, float eps, const float* gamma,
                                         const float* beta, const float* zy, const float* zb, int Tz, int hz,
                                         int wz, int apply_silu, void* out, int64_t out_T, int64_t out_t0,
                                         int dtype, dwm_stream_t stream) {
  DWM_REQUIRE(x && sums && gamma && beta && out, "dwm_b200_spatialnorm_silu: null pointer");
  DWM_REQUIRE(C % 4 == 0 && groups > 0 && C % groups == 0, "dwm_b200_spatialnorm_silu: bad C/groups");
  DWM_REQUIRE((zy == nullptr) == (zb == nullptr), "dwm_b200_spatialnorm_silu: zy and zb go together");
  DWM_REQUIRE(out_t0 >= 0 && out_t0 + T <= out_T, "dwm_b200_spatialnorm_silu: frame window outside out buffer");
  DWM_REQUIRE(!gn_align_check(x, sums, gamma, beta, zy, zb) && is_aligned(out, 8),
              "dwm_b200_spatialnorm_silu: x, gamma, beta, zy, zb must be 16-byte, sums and out 8-byte aligned");
  SnParams p;
  p.x = x; p.nb = (int)nb; p.T = (int)T; p.H = (int)H; p.W = (int)W; p.C = C; p.G = groups;
  p.sums = sums; p.eps = eps; p.gamma = gamma; p.beta = beta; p.zy = zy; p.zb = zb;
  p.Tz = Tz; p.hz = hz; p.wz = wz; p.silu = apply_silu; p.out = out; p.out_T = (int)out_T; p.out_t0 = (int)out_t0;
  p.scale = nullptr; p.stat_T = (int)T;
  DWM_REQUIRE(groups <= 64 && nb <= 65535, "dwm_b200_spatialnorm_silu: groups <= 64 and nb <= 65535 required");
  const long long per_img = T * H * W * (C / 4);
  // block = the largest multiple of C/4 that fits 256 threads (or C/4 itself up to 1024), so a
  // thread keeps one channel quad; 16 float4 per thread
  const int vec = C / 4;
  int threads = 256;
  if (vec <= 1024) threads = vec <= 256 ? (256 / vec) * vec : vec;
  const int chunk = threads * 16;
  dim3 grid(static_cast<unsigned>((per_img + chunk - 1) / chunk), static_cast<unsigned>(nb));
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == DWM_BF16) spatialnorm_kernel<__nv_bfloat16><<<grid, threads, 0, s>>>(p, chunk);
  else if (dtype == DWM_F16) spatialnorm_kernel<__half><<<grid, threads, 0, s>>>(p, chunk);
  else { set_last_error("dwm_b200_spatialnorm_silu: bad dtype"); return -1; }
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_groupnorm_silu_e4m3(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W, int C,
                                            int groups, const double* sums, float eps, const float* gamma,
                                            const float* beta, int apply_silu, void* out, int64_t out_T,
                                            int64_t out_t0, float* out_scale, dwm_stream_t stream) {
  DWM_REQUIRE(x && sums && gamma && beta && out && out_scale, "dwm_b200_groupnorm_silu_e4m3: null pointer");
  DWM_REQUIRE(nb > 0 && T > 0 && H > 0 && W > 0, "dwm_b200_groupnorm_silu_e4m3: bad shape");
  DWM_REQUIRE(C % 16 == 0 && groups > 0 && C % groups == 0 && groups <= 64,
              "dwm_b200_groupnorm_silu_e4m3: need C %% 16 == 0, C %% groups == 0, groups <= 64 (got C=%d, groups=%d)",
              C, groups);
  DWM_REQUIRE(out_t0 >= 0 && out_t0 + T <= out_T, "dwm_b200_groupnorm_silu_e4m3: frame window outside out buffer");
  DWM_REQUIRE(nb <= 65535, "dwm_b200_groupnorm_silu_e4m3: nb <= 65535 required");
  DWM_REQUIRE(!gn_align_check(x, sums, gamma, beta, nullptr, nullptr) && is_aligned(out, 4),
              "dwm_b200_groupnorm_silu_e4m3: x, gamma, beta must be 16-byte, sums 8-byte, out 4-byte aligned");
  SnParams p;
  p.x = x; p.nb = (int)nb; p.T = (int)T; p.H = (int)H; p.W = (int)W; p.C = C; p.G = groups;
  p.sums = sums; p.eps = eps; p.gamma = gamma; p.beta = beta; p.zy = nullptr; p.zb = nullptr;
  p.Tz = p.hz = p.wz = 0; p.silu = apply_silu; p.out = out; p.out_T = (int)out_T; p.out_t0 = (int)out_t0;
  p.scale = out_scale; p.stat_T = (int)T;
  const long long per_img = T * H * W * (C / 4);
  const int vec = C / 4;
  int threads = 256;
  if (vec <= 1024) threads = vec <= 256 ? (256 / vec) * vec : vec;
  const int chunk = threads * 16;
  dim3 grid(static_cast<unsigned>((per_img + chunk - 1) / chunk), static_cast<unsigned>(nb));
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  DWM_CHECK_CUDA(cudaMemsetAsync(out_scale, 0, sizeof(float) * nb, s));
  spatialnorm_kernel<__nv_fp8_e4m3, SN_AMAX><<<grid, threads, 0, s>>>(p, chunk);
  spatialnorm_kernel<__nv_fp8_e4m3, SN_E4M3><<<grid, threads, 0, s>>>(p, chunk);
  e4m3_amax_to_scale_kernel<<<static_cast<unsigned>((nb + 127) / 128), 128, 0, s>>>(out_scale, out_scale, (int)nb);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_spatialnorm_silu_e4m3(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W, int C,
                                              int groups, const double* sums, float eps, const float* gamma,
                                              const float* beta, const float* zy, const float* zb, int Tz, int hz,
                                              int wz, int apply_silu, void* out, int64_t out_T, int64_t out_t0,
                                              float* out_scale, const void* tail_in, void* tail_out, int tail_dtype,
                                              dwm_stream_t stream) {
  DWM_REQUIRE(x && sums && gamma && beta && out && out_scale, "dwm_b200_spatialnorm_silu_e4m3: null pointer");
  DWM_REQUIRE(nb > 0 && T > 0 && H > 0 && W > 0 && nb <= 65535, "dwm_b200_spatialnorm_silu_e4m3: bad shape");
  DWM_REQUIRE(C % 16 == 0 && groups > 0 && C % groups == 0 && groups <= 64,
              "dwm_b200_spatialnorm_silu_e4m3: need C %% 16 == 0, C %% groups == 0, groups <= 64 (got C=%d, groups=%d)",
              C, groups);
  DWM_REQUIRE((zy == nullptr) == (zb == nullptr), "dwm_b200_spatialnorm_silu_e4m3: zy and zb go together");
  DWM_REQUIRE(out_t0 >= 0 && out_t0 + T <= out_T, "dwm_b200_spatialnorm_silu_e4m3: frame window outside out buffer");
  DWM_REQUIRE(!tail_in || out_t0 >= 2, "dwm_b200_spatialnorm_silu_e4m3: tail_in needs out_t0 >= 2");
  DWM_REQUIRE(!(tail_in || tail_out) || tail_dtype == DWM_BF16 || tail_dtype == DWM_F16,
              "dwm_b200_spatialnorm_silu_e4m3: tail_dtype must be DWM_BF16 or DWM_F16");
  DWM_REQUIRE(!gn_align_check(x, sums, gamma, beta, zy, zb) && is_aligned(out, 4) && is_aligned(tail_in, 8) &&
                  is_aligned(tail_out, 8),
              "dwm_b200_spatialnorm_silu_e4m3: x, gamma, beta, zy, zb must be 16-byte, sums, tail_in, tail_out "
              "8-byte and out 4-byte aligned");
  SnParams p;
  p.x = x; p.nb = (int)nb; p.T = (int)T; p.H = (int)H; p.W = (int)W; p.C = C; p.G = groups;
  p.sums = sums; p.eps = eps; p.gamma = gamma; p.beta = beta; p.zy = zy; p.zb = zb;
  p.Tz = Tz; p.hz = hz; p.wz = wz; p.silu = apply_silu; p.out = out; p.out_T = (int)out_T; p.out_t0 = (int)out_t0;
  p.scale = out_scale; p.stat_T = (int)T;
  p.prev_out = const_cast<void*>(tail_in); p.next_out = tail_out;
  const long long per_img = T * H * W * (C / 4);
  const int vec = C / 4;
  int threads = 256;
  if (vec <= 1024) threads = vec <= 256 ? (256 / vec) * vec : vec;
  const int chunk = threads * 16;
  dim3 grid(static_cast<unsigned>((per_img + chunk - 1) / chunk), static_cast<unsigned>(nb));
  const long long frame4 = H * W * (C / 4);
  dim3 tgrid(static_cast<unsigned>(std::min<long long>((frame4 + 1023) / 1024, 2048)), static_cast<unsigned>(nb));
  const bool bf = tail_dtype == DWM_BF16;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  DWM_CHECK_CUDA(cudaMemsetAsync(out_scale, 0, sizeof(float) * nb, s));
  // amax over the cached tail and the new frames, then both quantized with the one volume scale
  if (tail_in) {
    if (bf) sn_tail_kernel<__nv_bfloat16, true><<<tgrid, 256, 0, s>>>(tail_in, frame4, out_scale, out, p.out_T, p.out_t0, nullptr);
    else sn_tail_kernel<__half, true><<<tgrid, 256, 0, s>>>(tail_in, frame4, out_scale, out, p.out_T, p.out_t0, nullptr);
  }
  spatialnorm_kernel<__nv_fp8_e4m3, SN_AMAX><<<grid, threads, 0, s>>>(p, chunk);
  if (tail_in) {
    void* shift = T == 1 ? tail_out : nullptr;
    if (bf) sn_tail_kernel<__nv_bfloat16, false><<<tgrid, 256, 0, s>>>(tail_in, frame4, out_scale, out, p.out_T, p.out_t0, shift);
    else sn_tail_kernel<__half, false><<<tgrid, 256, 0, s>>>(tail_in, frame4, out_scale, out, p.out_T, p.out_t0, shift);
  }
  if (!tail_out) spatialnorm_kernel<__nv_fp8_e4m3, SN_E4M3><<<grid, threads, 0, s>>>(p, chunk);
  else if (bf) spatialnorm_kernel<__nv_bfloat16, SN_E4M3_TAIL><<<grid, threads, 0, s>>>(p, chunk);
  else spatialnorm_kernel<__half, SN_E4M3_TAIL><<<grid, threads, 0, s>>>(p, chunk);
  e4m3_amax_to_scale_kernel<<<static_cast<unsigned>((nb + 127) / 128), 128, 0, s>>>(out_scale, out_scale, (int)nb);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ---- frame-shard variants: statistics of the whole window, halo frames into the neighbours ----
namespace {

const char* gn_shard_check(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W, int C, int groups,
                           const double* sums, int64_t stat_frames, const float* gamma, const float* beta,
                           int c_align) {
  if (!x || !sums || !gamma || !beta) return "null pointer";
  if (nb <= 0 || T <= 0 || H <= 0 || W <= 0 || nb > 65535) return "bad shape (need nb <= 65535)";
  if (C % c_align || groups <= 0 || groups > 64 || C % groups) return "bad C / groups";
  if (stat_frames < T) return "stat_frames < T";
  return gn_align_check(x, sums, gamma, beta, nullptr, nullptr);
}

SnParams gn_shard_params(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W, int C, int groups,
                         const double* sums, int64_t stat_frames, float eps, const float* gamma,
                         const float* beta, int apply_silu) {
  SnParams p;
  p.x = x; p.nb = (int)nb; p.T = (int)T; p.H = (int)H; p.W = (int)W; p.C = C; p.G = groups;
  p.sums = sums; p.eps = eps; p.gamma = gamma; p.beta = beta; p.zy = nullptr; p.zb = nullptr;
  p.Tz = p.hz = p.wz = 0; p.silu = apply_silu; p.out = nullptr; p.out_T = (int)T + 2; p.out_t0 = 1;
  p.scale = nullptr; p.stat_T = (int)stat_frames;
  return p;
}

// the launch shape of dwm_b200_spatialnorm_silu
void gn_launch_shape(const SnParams& p, int* threads, int* chunk, dim3* grid) {
  const int vec = p.C / 4;
  *threads = 256;
  if (vec <= 1024) *threads = vec <= 256 ? (256 / vec) * vec : vec;
  *chunk = *threads * 16;
  const long long per_img = static_cast<long long>(p.T) * p.H * p.W * vec;
  *grid = dim3(static_cast<unsigned>((per_img + *chunk - 1) / *chunk), static_cast<unsigned>(p.nb));
}

// `bytes`: the store width of four outputs (8 for 16-bit, 4 for E4M3)
const char* gn_halo_check(void* out, void* prev_out, int64_t prev_out_T, void* next_out, int64_t next_out_T,
                          uintptr_t bytes) {
  if (!out) return "null out";
  if ((prev_out && prev_out_T < 3) || (next_out && next_out_T < 3)) return "neighbour buffers hold >= 3 frames";
  if (!is_aligned(out, bytes) || !is_aligned(prev_out, bytes) || !is_aligned(next_out, bytes))
    return bytes == 8 ? "out, prev_out, next_out must be 8-byte aligned" : "out, prev_out, next_out must be 4-byte aligned";
  return nullptr;
}

}  // namespace

extern "C" int dwm_b200_groupnorm_silu_halo(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W, int C,
                                            int groups, const double* sums, int64_t stat_frames, float eps,
                                            const float* gamma, const float* beta, int apply_silu, void* out,
                                            void* prev_out, int64_t prev_out_T, void* next_out,
                                            int64_t next_out_T, int dtype, dwm_stream_t stream) {
  const char* bad = gn_shard_check(x, nb, T, H, W, C, groups, sums, stat_frames, gamma, beta, 4);
  if (!bad) bad = gn_halo_check(out, prev_out, prev_out_T, next_out, next_out_T, 8);
  DWM_REQUIRE(!bad, "dwm_b200_groupnorm_silu_halo: %s", bad);
  SnParams p = gn_shard_params(x, nb, T, H, W, C, groups, sums, stat_frames, eps, gamma, beta, apply_silu);
  p.out = out; p.prev_out = prev_out; p.prev_T = (int)prev_out_T; p.next_out = next_out; p.next_T = (int)next_out_T;
  int threads, chunk;
  dim3 grid;
  gn_launch_shape(p, &threads, &chunk, &grid);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == DWM_BF16) spatialnorm_kernel<__nv_bfloat16, SN_STORE16, true><<<grid, threads, 0, s>>>(p, chunk);
  else if (dtype == DWM_F16) spatialnorm_kernel<__half, SN_STORE16, true><<<grid, threads, 0, s>>>(p, chunk);
  else { set_last_error("dwm_b200_groupnorm_silu_halo: bad dtype"); return -1; }
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_groupnorm_silu_e4m3_amax(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W,
                                                 int C, int groups, const double* sums, int64_t stat_frames,
                                                 float eps, const float* gamma, const float* beta, int apply_silu,
                                                 float* amax, dwm_stream_t stream) {
  const char* bad = gn_shard_check(x, nb, T, H, W, C, groups, sums, stat_frames, gamma, beta, 16);
  if (!bad && !amax) bad = "null amax";
  DWM_REQUIRE(!bad, "dwm_b200_groupnorm_silu_e4m3_amax: %s", bad);
  SnParams p = gn_shard_params(x, nb, T, H, W, C, groups, sums, stat_frames, eps, gamma, beta, apply_silu);
  p.scale = amax;
  int threads, chunk;
  dim3 grid;
  gn_launch_shape(p, &threads, &chunk, &grid);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  DWM_CHECK_CUDA(cudaMemsetAsync(amax, 0, sizeof(float) * nb, s));
  spatialnorm_kernel<__nv_fp8_e4m3, SN_AMAX><<<grid, threads, 0, s>>>(p, chunk);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_groupnorm_silu_e4m3_halo(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W,
                                                 int C, int groups, const double* sums, int64_t stat_frames,
                                                 float eps, const float* gamma, const float* beta, int apply_silu,
                                                 const float* amax, void* out, void* prev_out, int64_t prev_out_T,
                                                 void* next_out, int64_t next_out_T, float* out_scale,
                                                 dwm_stream_t stream) {
  const char* bad = gn_shard_check(x, nb, T, H, W, C, groups, sums, stat_frames, gamma, beta, 16);
  if (!bad) bad = gn_halo_check(out, prev_out, prev_out_T, next_out, next_out_T, 4);
  if (!bad && (!amax || !out_scale)) bad = "null amax / out_scale";
  DWM_REQUIRE(!bad, "dwm_b200_groupnorm_silu_e4m3_halo: %s", bad);
  SnParams p = gn_shard_params(x, nb, T, H, W, C, groups, sums, stat_frames, eps, gamma, beta, apply_silu);
  p.out = out; p.prev_out = prev_out; p.prev_T = (int)prev_out_T; p.next_out = next_out; p.next_T = (int)next_out_T;
  p.scale = const_cast<float*>(amax);     // SN_E4M3 only reads it
  int threads, chunk;
  dim3 grid;
  gn_launch_shape(p, &threads, &chunk, &grid);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  spatialnorm_kernel<__nv_fp8_e4m3, SN_E4M3, true><<<grid, threads, 0, s>>>(p, chunk);
  e4m3_amax_to_scale_kernel<<<static_cast<unsigned>((nb + 127) / 128), 128, 0, s>>>(amax, out_scale, (int)nb);
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dwm_b200_upsample_nearest(const float* x, int64_t nb, int64_t T, int64_t H, int64_t W, int C,
                                         int compress_time, void* out, int dtype, dwm_stream_t stream) {
  DWM_REQUIRE(x && out && C % 4 == 0, "dwm_b200_upsample_nearest: bad arguments");
  DWM_REQUIRE(is_aligned(x, 16) && is_aligned(out, 8), "dwm_b200_upsample_nearest: x must be 16-byte and out 8-byte aligned");
  int mode = 0;
  long long To = T;
  if (compress_time && T > 1) {
    if (T % 2 == 1) { mode = 2; To = 1 + 2 * (T - 1); }
    else { mode = 1; To = 2 * T; }
  }
  const long long total = nb * To * 2 * H * 2 * W * (C / 4);
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == DWM_BF16)
    upsample_kernel<<<grid, 256, 0, s>>>(x, (int)nb, (int)T, (int)H, (int)W, C, (int)To, mode, reinterpret_cast<__nv_bfloat16*>(out));
  else if (dtype == DWM_F16)
    upsample_kernel<<<grid, 256, 0, s>>>(x, (int)nb, (int)T, (int)H, (int)W, C, (int)To, mode, reinterpret_cast<__half*>(out));
  else { set_last_error("dwm_b200_upsample_nearest: bad dtype"); return -1; }
  DWM_CHECK_CUDA(cudaGetLastError());
  return 0;
}
