// Path D — the HBM-bound glue of the DiT forward, each fused to one pass over its operands.
// Reference arithmetic (cosmos_predict1/diffusion):
//   adaLN   : blocks.py:339-341 (LN eps 1e-6 no affine, *(1+scale)+shift), :547-548 (abs-pos add)
//   RMSNorm : attention.py:131 (te RMSNorm eps 1e-6 over head_dim 128, "RRI" -> q,k only)
//   RoPE    : attention.py:278-279 rotate-half, angles position_embedding.py:106-187
//   patchify: blocks.py:153-159 "b c (t r)(h m)(w n) -> b t h w (c r m n)"
//   unpatch : general_dit.py:348-357 "(p1 p2 t C)"
//   t-embed : blocks.py:38-51,68-80 ; abs-pos normalise: position_embedding.py:220-233
//   sampler : model/model_v2w.py:130-149,201-259 ; EDM Euler (diffusers 0.32.2, restated)
#include <cuda_fp8.h>

#include <type_traits>

#include "kernels.h"

namespace g3c {

__device__ __forceinline__ float bf16_round(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  int nw = (blockDim.x + 31) >> 5;
  float t = lane < nw ? red[lane] : 0.0f;
  t = warp_sum(t);
  return t;  // every thread of every warp holds the block total
}

__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  int nw = (blockDim.x + 31) >> 5;
  float t = lane < nw ? red[lane] : 0.0f;
  return warp_max(t);
}

// ------------------------------------------------------------------------------------------------
// e4m3 row quantisation (the fp8 Linear mode; DESIGN.md §3.1): for a row with amax = max |x|,
//   inv = 448 / amax (IEEE division), code = e4m3_rn_satfinite(x * inv), scale = amax / 448;
//   a zero row gets codes 0 and scale 1.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float e4m3_inv_scale(float amax) { return amax > 0.0f ? __fdiv_rn(448.0f, amax) : 0.0f; }
__device__ __forceinline__ float e4m3_row_scale(float amax) { return amax > 0.0f ? __fdiv_rn(amax, 448.0f) : 1.0f; }
// four codes, the first in the lowest byte
__device__ __forceinline__ uint32_t e4m3x4(float a, float b, float c, float d, float inv) {
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(__fmul_rn(a, inv), __fmul_rn(b, inv)), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(__fmul_rn(c, inv), __fmul_rn(d, inv)), __NV_SATFINITE, __NV_E4M3);
  return lo | (hi << 16);
}

// bf16 x [R, C] (ld) -> codes [R, C] (ldq) + scales [R]; one CTA per row, 8 elements per thread and step
__global__ void __launch_bounds__(256)
    k_quant_rows_e4m3(const __nv_bfloat16* __restrict__ x, int ld, int C, uint8_t* __restrict__ codes, int ldq,
                      float* __restrict__ scales) {
  __shared__ float red[32];
  const __nv_bfloat16* xr = x + (size_t)blockIdx.x * ld;
  float amax = 0.0f;
  for (int i = threadIdx.x * 8; i < C; i += blockDim.x * 8) {
    uint4 q = *reinterpret_cast<const uint4*>(xr + i);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
    for (int j = 0; j < 4; ++j) amax = fmaxf(amax, fmaxf(fabsf(__low2float(h[j])), fabsf(__high2float(h[j]))));
  }
  amax = block_max(amax, red);
  const float inv = e4m3_inv_scale(amax);
  uint8_t* cr = codes + (size_t)blockIdx.x * ldq;
  for (int i = threadIdx.x * 8; i < C; i += blockDim.x * 8) {
    uint4 q = *reinterpret_cast<const uint4*>(xr + i);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&q);
    uint2 o;
    o.x = e4m3x4(__low2float(h[0]), __high2float(h[0]), __low2float(h[1]), __high2float(h[1]), inv);
    o.y = e4m3x4(__low2float(h[2]), __high2float(h[2]), __low2float(h[3]), __high2float(h[3]), inv);
    *reinterpret_cast<uint2*>(cr + i) = o;
  }
  if (threadIdx.x == 0) scales[blockIdx.x] = e4m3_row_scale(amax);
}

// ------------------------------------------------------------------------------------------------
// x (fp32 residual stream) [+= pos] ; y = LN(x) * (1 + scale) + shift   -> bf16
// one CTA per token row, the row cached in shared memory between the two statistics passes
// TOut = uint8_t: y is quantised to e4m3 codes from the fp32 row (never rounded to bf16) with the row scale in y_scale
// ------------------------------------------------------------------------------------------------
template <typename TOut>
__global__ void __launch_bounds__(256)
    k_ln_modulate(float* __restrict__ x, const __nv_bfloat16* __restrict__ pos,
                  const float* __restrict__ shift, const float* __restrict__ scale,
                  TOut* __restrict__ y, int D, float eps, float* __restrict__ y_scale) {
  extern __shared__ float row[];
  __shared__ float red[32];
  const size_t base = (size_t)blockIdx.x * D;
  float sum = 0.0f;
  for (int i = threadIdx.x * 4; i < D; i += blockDim.x * 4) {
    float4 v = *reinterpret_cast<const float4*>(x + base + i);
    if (pos) {
      uint2 pr = *reinterpret_cast<const uint2*>(pos + base + i);
      __nv_bfloat162 p0 = *reinterpret_cast<__nv_bfloat162*>(&pr.x);
      __nv_bfloat162 p1 = *reinterpret_cast<__nv_bfloat162*>(&pr.y);
      v.x += __low2float(p0);
      v.y += __high2float(p0);
      v.z += __low2float(p1);
      v.w += __high2float(p1);
      *reinterpret_cast<float4*>(x + base + i) = v;
    }
    *reinterpret_cast<float4*>(row + i) = v;
    sum += (v.x + v.y) + (v.z + v.w);
  }
  const float mean = block_sum(sum, red) / (float)D;
  float sq = 0.0f;
  for (int i = threadIdx.x * 4; i < D; i += blockDim.x * 4) {
    float4 v = *reinterpret_cast<const float4*>(row + i);
    float a = v.x - mean, b = v.y - mean, c = v.z - mean, d = v.w - mean;
    sq += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = rsqrtf(block_sum(sq, red) / (float)D + eps);
  if constexpr (std::is_same<TOut, __nv_bfloat16>::value) {
    for (int i = threadIdx.x * 4; i < D; i += blockDim.x * 4) {
      float4 v = *reinterpret_cast<const float4*>(row + i);
      float4 sc = *reinterpret_cast<const float4*>(scale + i);
      float4 sh = *reinterpret_cast<const float4*>(shift + i);
      uint2 o;
      o.x = pack_bf16x2(fmaf((v.x - mean) * rstd, 1.0f + sc.x, sh.x),
                        fmaf((v.y - mean) * rstd, 1.0f + sc.y, sh.y));
      o.y = pack_bf16x2(fmaf((v.z - mean) * rstd, 1.0f + sc.z, sh.z),
                        fmaf((v.w - mean) * rstd, 1.0f + sc.w, sh.w));
      *reinterpret_cast<uint2*>(y + base + i) = o;
    }
  } else {
    // the modulated row replaces x in shared memory (each thread rewrites and rereads its own elements)
    float amax = 0.0f;
    for (int i = threadIdx.x * 4; i < D; i += blockDim.x * 4) {
      float4 v = *reinterpret_cast<const float4*>(row + i);
      float4 sc = *reinterpret_cast<const float4*>(scale + i);
      float4 sh = *reinterpret_cast<const float4*>(shift + i);
      v = make_float4(fmaf((v.x - mean) * rstd, 1.0f + sc.x, sh.x), fmaf((v.y - mean) * rstd, 1.0f + sc.y, sh.y),
                      fmaf((v.z - mean) * rstd, 1.0f + sc.z, sh.z), fmaf((v.w - mean) * rstd, 1.0f + sc.w, sh.w));
      *reinterpret_cast<float4*>(row + i) = v;
      amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    }
    amax = block_max(amax, red);
    const float inv = e4m3_inv_scale(amax);
    for (int i = threadIdx.x * 4; i < D; i += blockDim.x * 4) {
      float4 v = *reinterpret_cast<const float4*>(row + i);
      *reinterpret_cast<uint32_t*>(y + base + i) = e4m3x4(v.x, v.y, v.z, v.w, inv);
    }
    if (threadIdx.x == 0) y_scale[blockIdx.x] = e4m3_row_scale(amax);
  }
}

// ------------------------------------------------------------------------------------------------
// per-head RMSNorm (+ rotate-half RoPE) in place on bf16 [L, heads*128]; one warp per (token, head)
// lane owns elements {2l, 2l+1} and {64+2l, 64+2l+1}: the rotate-half partners live in one thread
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    k_rmsnorm_rope(__nv_bfloat16* __restrict__ qk, int ld, int L, int heads,
                   const float* __restrict__ gamma, const float* __restrict__ cs, float eps) {
  const int lane = threadIdx.x & 31;
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= (long long)L * heads) return;
  const int tok = (int)(wid / heads), head = (int)(wid % heads);
  __nv_bfloat16* p = qk + (size_t)tok * ld + head * 128;
  __nv_bfloat162 lo = *reinterpret_cast<__nv_bfloat162*>(p + 2 * lane);
  __nv_bfloat162 hi = *reinterpret_cast<__nv_bfloat162*>(p + 64 + 2 * lane);
  float a0 = __low2float(lo), a1 = __high2float(lo), b0 = __low2float(hi), b1 = __high2float(hi);
  float ss = warp_sum((a0 * a0 + a1 * a1) + (b0 * b0 + b1 * b1));
  float r = rsqrtf(ss * (1.0f / 128.0f) + eps);
  float2 g0 = *reinterpret_cast<const float2*>(gamma + 2 * lane);
  float2 g1 = *reinterpret_cast<const float2*>(gamma + 64 + 2 * lane);
  a0 *= r * g0.x;
  a1 *= r * g0.y;
  b0 *= r * g1.x;
  b1 *= r * g1.y;
  if (cs) {
    // cs: [L][2][64] = cos(angle[0:64]) | sin(angle[0:64]); angles repeat over both halves
    const float* c = cs + (size_t)tok * 128;
    float2 co = *reinterpret_cast<const float2*>(c + 2 * lane);
    float2 si = *reinterpret_cast<const float2*>(c + 64 + 2 * lane);
    float n0 = a0 * co.x - b0 * si.x, n1 = a1 * co.y - b1 * si.y;
    float m0 = b0 * co.x + a0 * si.x, m1 = b1 * co.y + a1 * si.y;
    a0 = n0; a1 = n1; b0 = m0; b1 = m1;
  }
  *reinterpret_cast<__nv_bfloat162*>(p + 2 * lane) = __floats2bfloat162_rn(a0, a1);
  *reinterpret_cast<__nv_bfloat162*>(p + 64 + 2 * lane) = __floats2bfloat162_rn(b0, b1);
}

// ------------------------------------------------------------------------------------------------
// patchify: channel groups (x | cond mask | pose | padding mask) -> tokens [L, Kpad] bf16
// column = c*4 + m*2 + n ; token = (t*Hp + h)*Wp + w.  Zero pad columns >= 4*Ctot.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    k_patchify(PatchSrc src, int T, int Hp, int Wp, int Kpad, __nv_bfloat16* __restrict__ out) {
  const int H2 = Hp * 2, W2 = Wp * 2;
  const long long tok = blockIdx.x;
  const int w = (int)(tok % Wp), h = (int)((tok / Wp) % Hp), t = (int)(tok / ((long long)Wp * Hp));
  for (int col = threadIdx.x; col < Kpad; col += blockDim.x) {
    int c = col >> 2, m = (col >> 1) & 1, n = col & 1;
    float v = 0.0f;
    int g = 0;
    while (g < 4 && c >= src.nch[g]) {
      c -= src.nch[g];
      ++g;
    }
    if (g < 4 && src.ptr[g]) {
      size_t plane = (size_t)H2 * W2;
      size_t off = src.per_frame[g] ? ((size_t)c * T + t) * plane : (size_t)c * plane;
      v = __bfloat162float(src.ptr[g][off + (size_t)(2 * h + m) * W2 + (2 * w + n)]);
    }
    out[(size_t)tok * Kpad + col] = __float2bfloat16_rn(v);
  }
}

// final projection output [L, p*p*C] fp32 (column = (p1*2 + p2)*C + c) -> [C, T, H2, W2] bf16
__global__ void __launch_bounds__(256)
    k_unpatchify(const float* __restrict__ y, int ldy, int T, int Hp, int Wp, int C,
                 __nv_bfloat16* __restrict__ out) {
  const int H2 = Hp * 2, W2 = Wp * 2;
  size_t total = (size_t)C * T * H2 * W2;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    int x = (int)(i % W2), yy = (int)((i / W2) % H2), t = (int)((i / ((size_t)W2 * H2)) % T);
    int c = (int)(i / ((size_t)W2 * H2 * T));
    int w = x >> 1, p2 = x & 1, h = yy >> 1, p1 = yy & 1;
    size_t tok = ((size_t)t * Hp + h) * Wp + w;
    out[i] = __float2bfloat16_rn(y[tok * ldy + (p1 * 2 + p2) * C + c]);
  }
}

// ------------------------------------------------------------------------------------------------
// small dense vector ops for the timestep / adaLN-LoRA path (B = 1)
// ------------------------------------------------------------------------------------------------
// y[n] = post( sum_k W[n,k] * pre(x[k]) ) (+ add[n]);  W bf16 [N,K]; one warp per output row.
// pre: 0 none, 1 SiLU(x).  These B=1 vectors stay in fp32 end to end (the reference rounds them to
// bf16 after every Linear: blocks.py:68-75, :442-445); round_out != 0 reproduces that rounding.
__global__ void __launch_bounds__(256)
    k_gemv(const __nv_bfloat16* __restrict__ W, const float* __restrict__ x,
           const float* __restrict__ add, float* __restrict__ y, int N, int K, int pre,
           int round_out) {
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  const __nv_bfloat16* w = W + (size_t)n * K;
  float acc = 0.0f;
  for (int k = lane * 8; k < K; k += 32 * 8) {
    uint4 q = *reinterpret_cast<const uint4*>(w + k);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float x0 = x[k + 2 * i], x1 = x[k + 2 * i + 1];
      if (pre == 1) {
        x0 = x0 / (1.0f + expf(-x0));
        x1 = x1 / (1.0f + expf(-x1));
      }
      acc = fmaf(__low2float(h[i]), x0, acc);
      acc = fmaf(__high2float(h[i]), x1, acc);
    }
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    if (round_out) acc = bf16_round(acc);
    if (add) acc = round_out ? bf16_round(acc + add[n]) : acc + add[n];
    y[n] = acc;
  }
}

// s = [cos(t*e_i) | sin(t*e_i)], e_i = exp(-ln(1e4) * i / half) (blocks.py:38-51) ;
// emb = RMSNorm(s) * gamma (general_dit.py:405).  fp32 throughout.
__global__ void __launch_bounds__(256)
    k_timestep_embed(float t_in, int D, const __nv_bfloat16* __restrict__ gamma, float eps,
                     float* __restrict__ s_out, float* __restrict__ emb_out) {
  __shared__ float red[32];
  const int half = D / 2;
  const float t = t_in;
  float ss = 0.0f;
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    int j = i < half ? i : i - half;
    float e = expf(-9.210340371976184f * (float)j / (float)half);
    float a = t * e;
    float v = i < half ? cosf(a) : sinf(a);
    s_out[i] = v;
    ss += v * v;
  }
  float tot = block_sum(ss, red);
  float r = rsqrtf(tot / (float)D + eps);
  for (int i = threadIdx.x; i < D; i += blockDim.x)
    emb_out[i] = s_out[i] * r * __bfloat162float(gamma[i]);
}

// abs-pos: v = pt + ph + pw ; out = bf16(v / (1e-6 + ||v|| / sqrt(D)))   (fp32 math, bf16 storage)
__global__ void __launch_bounds__(256)
    k_abs_pos(const __nv_bfloat16* __restrict__ pos_t, const __nv_bfloat16* __restrict__ pos_h,
              const __nv_bfloat16* __restrict__ pos_w, int t0, int Hp, int Wp, int D,
              __nv_bfloat16* __restrict__ out) {
  extern __shared__ float row[];
  __shared__ float red[32];
  const long long tok = blockIdx.x;
  const int w = (int)(tok % Wp), h = (int)((tok / Wp) % Hp), t = t0 + (int)(tok / ((long long)Wp * Hp));
  float ss = 0.0f;
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    float v = __bfloat162float(pos_t[(size_t)t * D + i]) + __bfloat162float(pos_h[(size_t)h * D + i]) +
              __bfloat162float(pos_w[(size_t)w * D + i]);
    row[i] = v;
    ss += v * v;
  }
  float tot = block_sum(ss, red);
  float nrm = 1e-6f + sqrtf(tot) / sqrtf((float)D);
  for (int i = threadIdx.x; i < D; i += blockDim.x)
    out[(size_t)tok * D + i] = __float2bfloat16_rn(row[i] / nrm);
}

// RoPE cos|sin table [L][128] from per-axis frequencies (22 | 21 | 21 for head_dim 128)
__global__ void __launch_bounds__(128)
    k_rope_table(const float* __restrict__ freqs, int nt, int nh, int nw, int t0, float t_scale,
                 int Hp, int Wp, float* __restrict__ cs) {
  const long long tok = blockIdx.x;
  const int w = (int)(tok % Wp), h = (int)((tok / Wp) % Hp), t = t0 + (int)(tok / ((long long)Wp * Hp));
  const int j = threadIdx.x;
  if (j >= 64) return;
  float pos, f;
  if (j < nt) {
    pos = (float)t * t_scale;
    f = freqs[j];
  } else if (j < nt + nh) {
    pos = (float)h;
    f = freqs[j];
  } else {
    pos = (float)w;
    f = freqs[j];
  }
  float a = pos * f, s, c;
  sincosf(a, &s, &c);
  cs[(size_t)tok * 128 + j] = c;
  cs[(size_t)tok * 128 + 64 + j] = s;
}

__global__ void k_bf16_to_f32(const __nv_bfloat16* __restrict__ in, float* __restrict__ out, size_t n, float scale) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x)
    out[i] = __bfloat162float(in[i]) * scale;
}

// ------------------------------------------------------------------------------------------------
// sampler glue (per latent element; fp32 math, bf16 only where the reference stores a bf16 tensor
// that crosses a kernel boundary: x~, x_in, the net outputs and x_next)
// ------------------------------------------------------------------------------------------------
// pre : x~ = ind*aug + (1-ind)*x ; x_in = x~ * 1/sqrt(sigma^2 + sd^2)
//       aug = (gt + s_aug*noise) / sqrt(s_aug^2 + sd^2) * sqrt(sigma^2 + sd^2)
__global__ void __launch_bounds__(256)
    k_sampler_pre(const __nv_bfloat16* __restrict__ xt, const __nv_bfloat16* __restrict__ gt,
                  const float* __restrict__ noise, const float* __restrict__ ind_t, int T, size_t plane,
                  size_t n, float sigma, float sigma_aug, float sd, __nv_bfloat16* __restrict__ xtilde,
                  __nv_bfloat16* __restrict__ xin) {
  const float c_in_aug = 1.0f / sqrtf(sigma_aug * sigma_aug + sd * sd);
  const float inv_c_in = sqrtf(sigma * sigma + sd * sd);
  const float c_in = 1.0f / inv_c_in;
  const bool aug_on = !(sigma_aug >= sigma);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x) {
    int t = (int)((i / plane) % T);
    float ind = aug_on ? ind_t[t] : 0.0f;
    float g = __bfloat162float(gt[i]);
    float a = (g + noise[i] * sigma_aug) * c_in_aug;  // fp32 (noise is fp32 in the reference)
    a = a * inv_c_in;
    float x = __bfloat162float(xt[i]);
    float v = bf16_round(ind * a + (1.0f - ind) * x);  // new_xt is a bf16 tensor (model_v2w.py:137)
    xtilde[i] = __float2bfloat16_rn(v);
    xin[i] = __float2bfloat16_rn(v * c_in);
  }
}

// post: o = oc + g*(oc-ou) ; o = ind*(gt - c_skip*x~)/c_out + (1-ind)*o ;
//       x0 = c_skip*x~ + c_out*o ; x <- x~ + (x~ - x0)/sigma * (sigma_next - sigma)
__global__ void __launch_bounds__(256)
    k_sampler_post(const __nv_bfloat16* __restrict__ xtilde, const __nv_bfloat16* __restrict__ oc,
                   const __nv_bfloat16* __restrict__ ou, const __nv_bfloat16* __restrict__ gt,
                   const float* __restrict__ ind_t, int T, size_t plane, size_t n, float guidance,
                   float sigma, float sigma_next, float sigma_aug, float sd,
                   __nv_bfloat16* __restrict__ xnext, __nv_bfloat16* __restrict__ net_out) {
  const float c_skip = sd * sd / (sigma * sigma + sd * sd);
  const float c_out = sigma * sd / sqrtf(sigma * sigma + sd * sd);
  const bool aug_on = !(sigma_aug >= sigma);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x) {
    int t = (int)((i / plane) % T);
    float ind = aug_on ? ind_t[t] : 0.0f;
    float c = __bfloat162float(oc[i]), u = __bfloat162float(ou[i]);
    float o = c + guidance * (c - u);
    if (net_out) net_out[i] = __float2bfloat16_rn(o);  // net_output of model_v2w.py:143 (test / inspection hook)
    float xs = __bfloat162float(xtilde[i]);
    float lat = (__bfloat162float(gt[i]) - c_skip * xs) / c_out;
    o = ind * lat + (1.0f - ind) * o;
    // scheduler.step in fp32 (diffusers upcasts the sample), result cast back to bf16
    float x0 = c_skip * xs + c_out * o;
    float d = (xs - x0) / sigma;
    xnext[i] = __float2bfloat16_rn(xs + d * (sigma_next - sigma));
  }
}

// ------------------------------------------------------------------------------------------------
// host launchers (used by dit_engine.cu and the C ABI test hooks)
// ------------------------------------------------------------------------------------------------
int ln_modulate(float* x, const __nv_bfloat16* pos, const float* shift, const float* scale,
                __nv_bfloat16* y, int L, int D, float eps, cudaStream_t st) {
  G3C_REQUIRE(D % 4 == 0 && D * 4 <= 96 * 1024, "ln_modulate: D=%d unsupported", D);
  static bool configured = false;
  if (!configured) {
    G3C_CUDA(cudaFuncSetAttribute(k_ln_modulate<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    configured = true;
  }
  k_ln_modulate<__nv_bfloat16><<<L, 256, D * sizeof(float), st>>>(x, pos, shift, scale, y, D, eps, nullptr);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int ln_modulate_e4m3(float* x, const __nv_bfloat16* pos, const float* shift, const float* scale, uint8_t* y8,
                     float* y_scale, int L, int D, float eps, cudaStream_t st) {
  G3C_REQUIRE(D % 16 == 0 && D * 4 <= 96 * 1024, "ln_modulate_e4m3: D=%d unsupported", D);
  static bool configured = false;
  if (!configured) {
    G3C_CUDA(cudaFuncSetAttribute(k_ln_modulate<uint8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    configured = true;
  }
  k_ln_modulate<uint8_t><<<L, 256, D * sizeof(float), st>>>(x, pos, shift, scale, y8, D, eps, y_scale);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int quant_rows_e4m3(const __nv_bfloat16* x, int ld, int R, int C, uint8_t* codes, int ldq, float* scales,
                    cudaStream_t st) {
  G3C_REQUIRE(x && codes && scales, "quantize_rows_fp8: null argument");
  G3C_REQUIRE(R > 0 && C > 0 && C % 16 == 0, "quantize_rows_fp8: C=%d must be a positive multiple of 16 (R=%d)", C, R);
  G3C_REQUIRE(ld >= C && ld % 8 == 0 && ldq >= C && ldq % 16 == 0,
              "quantize_rows_fp8: leading dimensions ld=%d (multiple of 8) and ldq=%d (multiple of 16) must be >= C=%d",
              ld, ldq, C);
  G3C_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(codes) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(scales) & 15) == 0,
              "quantize_rows_fp8: x, codes and scales must be 16-byte aligned");
  k_quant_rows_e4m3<<<R, 256, 0, st>>>(x, ld, C, codes, ldq, scales);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int rmsnorm_rope(__nv_bfloat16* qk, int ld, int L, int heads, const float* gamma, const float* cs,
                 float eps, cudaStream_t st) {
  long long warps = (long long)L * heads;
  int blocks = (int)((warps + 7) / 8);
  k_rmsnorm_rope<<<blocks, 256, 0, st>>>(qk, ld, L, heads, gamma, cs, eps);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int gemv(const __nv_bfloat16* W, const float* x, const float* add, float* y, int N, int K, int pre,
         int round_out, cudaStream_t st) {
  G3C_REQUIRE(K % 8 == 0, "gemv: K=%d must be a multiple of 8", K);
  k_gemv<<<(N + 7) / 8, 256, 0, st>>>(W, x, add, y, N, K, pre, round_out);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int patchify(const PatchSrc& src, int T, int Hp, int Wp, int Kpad, __nv_bfloat16* out, cudaStream_t st) {
  k_patchify<<<T * Hp * Wp, 128, 0, st>>>(src, T, Hp, Wp, Kpad, out);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int unpatchify(const float* y, int ldy, int T, int Hp, int Wp, int C, __nv_bfloat16* out, cudaStream_t st) {
  k_unpatchify<<<4 * sm_count(), 256, 0, st>>>(y, ldy, T, Hp, Wp, C, out);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int timestep_embed(float t, int D, const __nv_bfloat16* gamma, float eps, float* s, float* emb,
                   cudaStream_t st) {
  k_timestep_embed<<<1, 256, 0, st>>>(t, D, gamma, eps, s, emb);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int abs_pos(const __nv_bfloat16* pt, const __nv_bfloat16* ph, const __nv_bfloat16* pw, int t0, int T,
            int Hp, int Wp, int D, __nv_bfloat16* out, cudaStream_t st) {
  k_abs_pos<<<T * Hp * Wp, 256, D * sizeof(float), st>>>(pt, ph, pw, t0, Hp, Wp, D, out);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int rope_table(const float* freqs, int nt, int nh, int nw, int t0, float t_scale, int T, int Hp, int Wp,
               float* cs, cudaStream_t st) {
  k_rope_table<<<T * Hp * Wp, 128, 0, st>>>(freqs, nt, nh, nw, t0, t_scale, Hp, Wp, cs);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int bf16_to_f32(const __nv_bfloat16* in, float* out, size_t n, cudaStream_t st, float scale) {
  k_bf16_to_f32<<<(int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024), 256, 0, st>>>(in, out, n, scale);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int sampler_pre(const __nv_bfloat16* xt, const __nv_bfloat16* gt, const float* noise, const float* ind_t,
                int C, int T, size_t plane, float sigma, float sigma_aug, float sd,
                __nv_bfloat16* xtilde, __nv_bfloat16* xin, cudaStream_t st) {
  size_t n = (size_t)C * T * plane;
  k_sampler_pre<<<4 * sm_count(), 256, 0, st>>>(xt, gt, noise, ind_t, T, plane, n, sigma, sigma_aug, sd,
                                                xtilde, xin);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int sampler_post(const __nv_bfloat16* xtilde, const __nv_bfloat16* oc, const __nv_bfloat16* ou,
                 const __nv_bfloat16* gt, const float* ind_t, int C, int T, size_t plane, float guidance,
                 float sigma, float sigma_next, float sigma_aug, float sd, __nv_bfloat16* xnext,
                 __nv_bfloat16* net_out, cudaStream_t st) {
  size_t n = (size_t)C * T * plane;
  k_sampler_post<<<4 * sm_count(), 256, 0, st>>>(xtilde, oc, ou, gt, ind_t, T, plane, n, guidance, sigma,
                                                 sigma_next, sigma_aug, sd, xnext, net_out);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

}  // namespace g3c

// ---- C ABI test hooks for the elementwise kernels ----------------------------------------------
extern "C" {

int g3c_ln_modulate(float* x, const void* pos_bf16, const float* shift, const float* scale, void* y_bf16,
                    int L, int D, float eps, void* stream) {
  G3C_REQUIRE(x && shift && scale && y_bf16 && L > 0, "ln_modulate: bad arguments");
  return g3c::ln_modulate(x, (const __nv_bfloat16*)pos_bf16, shift, scale, (__nv_bfloat16*)y_bf16, L, D,
                          eps, (cudaStream_t)stream);
}

int g3c_quantize_rows_fp8(const void* x_bf16, int ld, int R, int C, void* codes, int ldq, float* scales,
                          void* stream) {
  return g3c::quant_rows_e4m3((const __nv_bfloat16*)x_bf16, ld, R, C, (uint8_t*)codes, ldq, scales,
                              (cudaStream_t)stream);
}

int g3c_ln_modulate_fp8(float* x, const void* pos_bf16, const float* shift, const float* scale, void* y_codes,
                        float* y_scales, int L, int D, float eps, void* stream) {
  G3C_REQUIRE(x && shift && scale && y_codes && y_scales && L > 0, "ln_modulate_fp8: bad arguments");
  G3C_REQUIRE((reinterpret_cast<uintptr_t>(y_codes) & 15) == 0 && (reinterpret_cast<uintptr_t>(y_scales) & 15) == 0,
              "ln_modulate_fp8: codes and scales must be 16-byte aligned");
  return g3c::ln_modulate_e4m3(x, (const __nv_bfloat16*)pos_bf16, shift, scale, (uint8_t*)y_codes, y_scales, L, D, eps,
                               (cudaStream_t)stream);
}

int g3c_rmsnorm_rope(void* qk_bf16, int ld, int L, int heads, const float* gamma, const float* cos_sin,
                     float eps, void* stream) {
  G3C_REQUIRE(qk_bf16 && gamma && L > 0 && heads > 0 && ld >= heads * 128 && ld % 2 == 0,
              "rmsnorm_rope: bad arguments");
  return g3c::rmsnorm_rope((__nv_bfloat16*)qk_bf16, ld, L, heads, gamma, cos_sin, eps,
                           (cudaStream_t)stream);
}

}  // extern "C"
