// Path D — dense bf16 GEMM on the Hopper tensor cores:  D[M,N] = A[M,K] · B[N,K]^T  (fp32 accum)
//
// Every Linear of the DiT (reference: cosmos_predict1/diffusion/module/attention.py:263-266,289,
// 91-102; blocks.py:153-163,222-242) is `y = x · W^T` with x [tokens, in] and W [out, in], i.e.
// both operands K-major — exactly the layout wgmma consumes from 128-byte-swizzled shared memory.
// V^T for the attention kernel is produced by the same kernel with the operands swapped
// (A = W_v, B = x), so no transpose pass exists anywhere.
//
// Structure (one persistent CTA per SM, 384 threads = three warpgroups):
//   warpgroup 0   TMA producer : one thread, cp.async.bulk.tensor A/B tiles -> smem ring (kStages), mbarrier tx
//   warpgroups 1-2 consumers   : wgmma 64 x BN x 16 each (rows 0-63 / 64-127 of the 128-row tile), accumulators in
//                                registers, fused epilogue straight from the registers to global memory
// The producer runs ahead into the next tile while the consumers run the epilogue of the current one.
//
// FP8 (e4m3) instantiation (kFp8): the operands are row-quantized codes, D[m,n] = (sum_k A8[m,k] B8[n,k]) *
// scale_a[m] * scale_b[n].  A k-block is then 128 codes instead of 64 bf16: still 128 bytes, one swizzle span, so the
// TMA boxes, the stage ring, the barriers and the 32-byte descriptor advance per wgmma (k16 bf16 / k32 e4m3) are the
// same bytes.  Only the instruction, the tensor-map element type and the scaling ahead of the epilogue change.
#include <cstdlib>
#include <cstring>

#include "kernels.h"

namespace g3c {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle span
constexpr int WG_K = 16;
template <bool kFp8>
constexpr int kBlockK = kFp8 ? 2 * BK : BK;  // elements of K per stage: 128 bytes either way
constexpr int GEMM_THREADS = 384;

struct GemmParams {
  int M, N, K;
  int ldd;             // leading dimension of D in elements
  void* D;             // bf16 or f32
  const float* gate;   // [N] for EPI_GATED_RESIDUAL
  int num_m_blk, num_n_blk, num_k_blk;
  int super_n;         // n-blocks per super-column (L2 reuse of the B operand)
  // EPI_NORM_ROPE_BF16: per-head (128 columns) RMSNorm gain [128], cos|sin table [M][128] (or NULL: no rotation), eps
  const float* nr_gamma;
  const float* nr_cs;
  float nr_eps;
  // fp8 operands: row scales of A [M] and of B [N] (dequantisation factors)
  const float* scale_a;
  const float* scale_b;
};

// internal epilogue (not part of the C ABI enum; reached through gemm_bf16(..., norm_rope)):
// D (bf16) = RoPE(RMSNorm_head(acc) * gamma) — the to_q / to_k Sequential(Linear, RMSNorm) of the reference followed by
// the rotate-half RoPE, applied to the fp32 accumulators of one head while they are still in registers.
constexpr int EPI_NORM_ROPE_BF16 = 4;

template <int BN>
struct GemmSmem {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (192 * 1024) / kStageBytes;  // 4 / 6 / 8 stages for BN = 256 / 128 / 64
  static constexpr int kBarBytes = 256;
  static constexpr int kTotal = kStages * kStageBytes + kBarBytes + 1024;  // + alignment slack
};

__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}

__device__ __forceinline__ void tile_coords(const GemmParams& p, int tile, int& m_blk, int& n_blk) {
  // super-columns of `super_n` n-blocks; inside one, n fastest so that concurrently running CTAs
  // share A row-blocks and the B super-column stays L2 resident.
  int per_super = p.num_m_blk * p.super_n;
  int sc = tile / per_super;
  int rem = tile - sc * per_super;
  int n0 = sc * p.super_n;
  int width = p.num_n_blk - n0 < p.super_n ? p.num_n_blk - n0 : p.super_n;
  // the last super-column may be narrower
  m_blk = rem / width;
  n_blk = n0 + rem - m_blk * width;
}

// Accumulator layout of wgmma m64nNk16 (f32): thread t of the warpgroup holds, for i in [0, N/8),
//   acc[4i + 0], acc[4i + 1] -> row 16 * (t / 32) + (t % 32) / 4,     columns 8i + 2 (t % 4) + {0, 1}
//   acc[4i + 2], acc[4i + 3] -> the same columns eight rows further down.
// Fused Linear -> per-head RMSNorm -> rotate-half RoPE for the heads of a tile: the 128 columns of one head and row
// are spread over the four threads of a quad (reduced with two shuffles), and the rotate-half partners c and c + 64
// (accumulator indices i and i + 8) sit in the same thread.  reference: module/attention.py:263-266 (to_q/to_k =
// Linear + RMSNorm) and :268-283 (apply_rotary_pos_emb); same arithmetic as k_rmsnorm_rope (dit_elementwise.cu).
template <int BN>
__device__ __forceinline__ void epilogue_norm_rope(const float (&acc)[BN / 2], const GemmParams& p, int row_a, int col_q,
                                                   int n_base) {
#pragma unroll
  for (int hd = 0; hd < BN / 128; ++hd) {
    if (n_base + hd * 128 >= p.N) break;
    float ss[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 16 * hd; i < 16 * hd + 16; ++i) {
      ss[0] = fmaf(acc[4 * i], acc[4 * i], fmaf(acc[4 * i + 1], acc[4 * i + 1], ss[0]));
      ss[1] = fmaf(acc[4 * i + 2], acc[4 * i + 2], fmaf(acc[4 * i + 3], acc[4 * i + 3], ss[1]));
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      ss[h] += __shfl_xor_sync(0xffffffffu, ss[h], 1);
      ss[h] += __shfl_xor_sync(0xffffffffu, ss[h], 2);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row_a + 8 * h;
      if (row >= p.M) continue;
      const float rstd = rsqrtf(ss[h] * (1.0f / 128.0f) + p.nr_eps);
      const float* cs = p.nr_cs ? p.nr_cs + (size_t)row * 128 : nullptr;
      __nv_bfloat16* dptr = reinterpret_cast<__nv_bfloat16*>(p.D) + (size_t)row * p.ldd + n_base + hd * 128;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = 8 * i + col_q;  // column inside the head, < 64; the partner is c + 64
        const float2 ga = *reinterpret_cast<const float2*>(p.nr_gamma + c);
        const float2 gb = *reinterpret_cast<const float2*>(p.nr_gamma + 64 + c);
        const int ia = 4 * (16 * hd + i) + 2 * h, ib = 4 * (16 * hd + i + 8) + 2 * h;
        float a[2] = {acc[ia] * (rstd * ga.x), acc[ia + 1] * (rstd * ga.y)};
        float b[2] = {acc[ib] * (rstd * gb.x), acc[ib + 1] * (rstd * gb.y)};
        if (cs) {
          const float2 co = *reinterpret_cast<const float2*>(cs + c);
          const float2 si = *reinterpret_cast<const float2*>(cs + 64 + c);
          const float cv[2] = {co.x, co.y}, sv[2] = {si.x, si.y};
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float n = a[e] * cv[e] - b[e] * sv[e], m = b[e] * cv[e] + a[e] * sv[e];
            a[e] = n;
            b[e] = m;
          }
        }
        *reinterpret_cast<uint32_t*>(dptr + c) = pack_bf16x2(a[0], a[1]);
        *reinterpret_cast<uint32_t*>(dptr + 64 + c) = pack_bf16x2(b[0], b[1]);
      }
    }
  }
}

// fp8: dequantise the accumulators in place, acc * scale_a[row] * scale_b[col], before any epilogue arithmetic (the
// RMSNorm of the fused to_q / to_k epilogue must see the dequantised values).  Rows / columns past M / N keep their
// zero accumulators (scale 0): the epilogue does not store them.
template <int BN>
__device__ __forceinline__ void dequantise(float (&acc)[BN / 2], const GemmParams& p, int row_a, int col_q, int n_base) {
  float sa[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) sa[h] = row_a + 8 * h < p.M ? p.scale_a[row_a + 8 * h] : 0.f;
#pragma unroll
  for (int i = 0; i < BN / 8; ++i) {
    const int col = n_base + 8 * i + col_q;
    float2 sb = make_float2(0.f, 0.f);
    if (col + 1 < p.N) sb = *reinterpret_cast<const float2*>(p.scale_b + col);
    else if (col < p.N) sb.x = p.scale_b[col];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      acc[4 * i + 2 * h] = acc[4 * i + 2 * h] * sa[h] * sb.x;
      acc[4 * i + 2 * h + 1] = acc[4 * i + 2 * h + 1] * sa[h] * sb.y;
    }
  }
}

template <int BN, int EPI>
__device__ __forceinline__ void epilogue(const float (&acc)[BN / 2], const GemmParams& p, int row_a, int col_q,
                                         int n_base) {
  if constexpr (EPI == EPI_NORM_ROPE_BF16) {
    epilogue_norm_rope<BN>(acc, p, row_a, col_q, n_base);
  } else {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row_a + 8 * h;
      if (row >= p.M) continue;
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int col = n_base + 8 * i + col_q;
        if (col >= p.N) continue;
        const bool pair = col + 1 < p.N;
        float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
        if constexpr (EPI == G3C_EPI_BF16 || EPI == G3C_EPI_GELU_BF16) {
          if constexpr (EPI == G3C_EPI_GELU_BF16) {
            v0 = gelu_erf(v0);
            v1 = gelu_erf(v1);
          }
          __nv_bfloat16* dptr = reinterpret_cast<__nv_bfloat16*>(p.D) + (size_t)row * p.ldd + col;
          if (pair) *reinterpret_cast<uint32_t*>(dptr) = pack_bf16x2(v0, v1);
          else dptr[0] = __float2bfloat16_rn(v0);
        } else {
          float* dptr = reinterpret_cast<float*>(p.D) + (size_t)row * p.ldd + col;
          if constexpr (EPI == G3C_EPI_GATED_RESIDUAL_F32) {
            // x += gate * acc on the fp32 residual stream; every element has exactly one owner
            if (pair) {
              const float2 g = *reinterpret_cast<const float2*>(p.gate + col);
              float2 x = *reinterpret_cast<float2*>(dptr);
              x.x = fmaf(g.x, v0, x.x);
              x.y = fmaf(g.y, v1, x.y);
              *reinterpret_cast<float2*>(dptr) = x;
            } else {
              dptr[0] = fmaf(p.gate[col], v0, dptr[0]);
            }
          } else {
            if (pair) *reinterpret_cast<float2*>(dptr) = make_float2(v0, v1);
            else dptr[0] = v0;
          }
        }
      }
    }
  }
}

template <int BN, int EPI, bool kFp8>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    k_gemm(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  using S = GemmSmem<BN>;
  constexpr int kStages = S::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * S::kABytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * S::kStageBytes);
  uint64_t* full = bars;              // [kStages]
  uint64_t* empty = bars + kStages;   // [kStages]

  const uint32_t wg = threadIdx.x / 128;
  const uint32_t tid = threadIdx.x % 128;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int num_tiles = p.num_m_blk * p.num_n_blk;

  if (wg == 0) {
    // ===== TMA producer =====
    setmaxnreg_dec<40>();
    if (tid == 0) {
      uint32_t stage = 0, phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        tile_coords(p, tile, m_blk, n_blk);
        for (int kb = 0; kb < p.num_k_blk; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], S::kStageBytes);
          tma_load_2d(smem_a + stage * S::kABytes, &tmA, &full[stage], kb * kBlockK<kFp8>, m_blk * BM);
          tma_load_2d(smem_b + stage * S::kBBytes, &tmB, &full[stage], kb * kBlockK<kFp8>, n_blk * BN);
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===== consumers: warpgroup c owns rows [64c, 64c + 64) of every tile =====
    setmaxnreg_inc<232>();
    const uint32_t c = wg - 1;
    const uint32_t warp = tid / 32, lane = tid % 32;
    uint32_t stage = 0, phase = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int m_blk, n_blk;
      tile_coords(p, tile, m_blk, n_blk);
      if constexpr (kFp8) {
        // The e4m3 wgmma does not keep a full fp32 sum internally (measured on an H100: rel-L2 1.3e-3 against an exact
        // product at K = 4096).  Each k-block's 128-code partial sum is therefore formed by the tensor cores from
        // zero and added to the fp32 accumulators here, so the error does not grow with K.  The partial sums double
        // the accumulator registers: fp8 tiles are at most 128 columns wide.
        static_assert(BN <= 128, "fp8 tiles hold two accumulator sets");
        float part[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        for (int kb = 0; kb < p.num_k_blk; ++kb) {
          mbar_wait(&full[stage], phase);
          const uint64_t da = make_sdesc_sw128(smem_u32(smem_a + stage * S::kABytes + c * 64 * 128));
          const uint64_t db = make_sdesc_sw128(smem_u32(smem_b + stage * S::kBBytes));
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / WG_K; ++k) {
            const uint64_t a = sdesc_advance(da, k * WG_K * 2), b = sdesc_advance(db, k * WG_K * 2);
            if constexpr (BN == 128) wgmma_ss_n128_e4m3(part, a, b, k != 0 ? 1u : 0u);
            else wgmma_ss_n64_e4m3(part, a, b, k != 0 ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          fence_regs(part);
          if (tid == 0) mbar_arrive(&empty[stage]);
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      } else {
        uint32_t prev_stage = 0;
        for (int kb = 0; kb < p.num_k_blk; ++kb) {
          mbar_wait(&full[stage], phase);
          const uint64_t da = make_sdesc_sw128(smem_u32(smem_a + stage * S::kABytes + c * 64 * 128));
          const uint64_t db = make_sdesc_sw128(smem_u32(smem_b + stage * S::kBBytes));
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / WG_K; ++k) {
            const uint64_t a = sdesc_advance(da, k * WG_K * 2), b = sdesc_advance(db, k * WG_K * 2);
            const uint32_t accumulate = (kb | k) != 0 ? 1u : 0u;
            if constexpr (BN == 256) wgmma_ss_n256(acc, a, b, accumulate);
            else if constexpr (BN == 128) wgmma_ss_n128(acc, a, b, accumulate);
            else wgmma_ss_n64(acc, a, b, accumulate);
          }
          wgmma_commit();
          // one group stays in flight: the stage of the previous k-block is free once its group has completed
          wgmma_wait<1>();
          fence_regs(acc);
          if (kb > 0 && tid == 0) mbar_arrive(&empty[prev_stage]);
          prev_stage = stage;
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
        wgmma_wait<0>();
        fence_regs(acc);
        if (tid == 0) mbar_arrive(&empty[prev_stage]);
      }
      const int row_a = m_blk * BM + (int)(c * 64 + warp * 16 + lane / 4), col_q = (int)(2 * (lane % 4));
      if constexpr (kFp8) dequantise<BN>(acc, p, row_a, col_q, n_blk * BN);
      epilogue<BN, EPI>(acc, p, row_a, col_q, n_blk * BN);
    }
  }
}

template <int BN, int EPI, bool kFp8>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, cudaStream_t st) {
  using S = GemmSmem<BN>;
  static bool configured = false;
  if (!configured) {
    G3C_CUDA(cudaFuncSetAttribute(k_gemm<BN, EPI, kFp8>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal));
    configured = true;
  }
  int tiles = p.num_m_blk * p.num_n_blk;
  int grid = tiles < sm_count() ? tiles : sm_count();
  k_gemm<BN, EPI, kFp8><<<grid, GEMM_THREADS, S::kTotal, st>>>(tmA, tmB, p);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

template <int BN, bool kFp8>
static int dispatch_epi(int epi, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, cudaStream_t st) {
  switch (epi) {
    case G3C_EPI_BF16: return launch_gemm<BN, G3C_EPI_BF16, kFp8>(tmA, tmB, p, st);
    case G3C_EPI_GELU_BF16: return launch_gemm<BN, G3C_EPI_GELU_BF16, kFp8>(tmA, tmB, p, st);
    case G3C_EPI_GATED_RESIDUAL_F32: return launch_gemm<BN, G3C_EPI_GATED_RESIDUAL_F32, kFp8>(tmA, tmB, p, st);
    case G3C_EPI_F32: return launch_gemm<BN, G3C_EPI_F32, kFp8>(tmA, tmB, p, st);
    case EPI_NORM_ROPE_BF16:
      if constexpr (BN >= 128) return launch_gemm<BN, EPI_NORM_ROPE_BF16, kFp8>(tmA, tmB, p, st);
      break;
  }
  set_error("gemm: unknown epilogue %d", epi);
  return G3C_EINVAL;
}

// Shared host path of gemm_bf16 / gemm_fp8: scale_a / scale_b non-null selects the e4m3 kernels.
static int gemm_any(const void* A, const void* B, const float* scale_a, const float* scale_b, void* D, int M, int N,
                    int K, int lda, int ldb, int ldd, int epilogue, const float* gate, int block_n, cudaStream_t st,
                    const NormRope* norm_rope) {
  const bool fp8 = scale_a != nullptr;
  G3C_REQUIRE(A && B && D, "gemm: null operand");
  // only the C ABI's four epilogues are accepted here: EPI_NORM_ROPE_BF16 is selected by `norm_rope` alone (passed as
  // an epilogue code it would launch the fused norm without a gain vector)
  G3C_REQUIRE(epilogue >= G3C_EPI_BF16 && epilogue <= G3C_EPI_F32, "gemm: unknown epilogue %d", epilogue);
  if (norm_rope) {
    G3C_REQUIRE(epilogue == G3C_EPI_BF16 && N % 128 == 0 && norm_rope->gamma,
                "gemm: the RMSNorm/RoPE epilogue needs the bf16 epilogue, N %% 128 == 0 and a gain vector");
    G3C_REQUIRE((reinterpret_cast<uintptr_t>(norm_rope->gamma) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(norm_rope->cs) & 15) == 0,
                "gemm: RMSNorm gain / RoPE table must be 16-byte aligned");
    epilogue = EPI_NORM_ROPE_BF16;
  }
  G3C_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: bad shape %dx%dx%d", M, N, K);
  if (fp8)  // 16-byte TMA strides
    G3C_REQUIRE(K % 16 == 0 && lda % 16 == 0 && ldb % 16 == 0, "gemm_fp8: K/lda/ldb must be multiples of 16");
  else
    G3C_REQUIRE(K % 8 == 0 && lda % 8 == 0 && ldb % 8 == 0, "gemm: K/lda/ldb must be multiples of 8");
  G3C_REQUIRE(lda >= K && ldb >= K && ldd >= N, "gemm: leading dimension smaller than extent");
  if (epilogue == G3C_EPI_BF16 || epilogue == G3C_EPI_GELU_BF16 || epilogue == EPI_NORM_ROPE_BF16)
    G3C_REQUIRE(ldd % 8 == 0 && (reinterpret_cast<uintptr_t>(D) & 15) == 0,
                "gemm: bf16 output needs ldd %% 8 == 0 and 16-byte aligned base");
  else
    G3C_REQUIRE(ldd % 4 == 0 && (reinterpret_cast<uintptr_t>(D) & 15) == 0,
                "gemm: f32 output needs ldd %% 4 == 0 and 16-byte aligned base");
  G3C_REQUIRE(epilogue != G3C_EPI_GATED_RESIDUAL_F32 ||
                  (gate && (reinterpret_cast<uintptr_t>(gate) & 15) == 0),
              "gemm: gated-residual epilogue needs a 16-byte aligned gate vector");
  int bn = block_n;
  G3C_REQUIRE(bn == 0 || bn == 64 || bn == 128 || bn == 256 || bn == 512, "gemm: block_n %d unsupported", bn);
  // block_n 512 (the C ABI's request for the widest tile) runs the 256-column tile
  if (bn == 512) {
    G3C_REQUIRE(N % 256 == 0, "gemm: block_n 512 needs N %% 256 == 0 (N=%d)", N);
    bn = 256;
  }
  if (bn == 0) bn = (N >= 256 && N % 256 == 0) ? 256 : (N > 64 ? 128 : 64);
  if (fp8 && bn == 256) bn = 128;  // fp8 tiles hold a second (partial-sum) accumulator set: at most 128 columns
  G3C_REQUIRE(epilogue != EPI_NORM_ROPE_BF16 || bn >= 128, "gemm: the RMSNorm/RoPE epilogue needs tiles of whole heads");

  CUtensorMap tmA, tmB;
  const int esize = fp8 ? 1 : 2, bk = fp8 ? kBlockK<true> : kBlockK<false>;
  const CUtensorMapDataType dt = fp8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  uint64_t dimsA[2] = {(uint64_t)K, (uint64_t)M}, strA[1] = {(uint64_t)lda * esize};
  uint32_t boxA[2] = {(uint32_t)bk, BM};
  int rc = make_tmap_bf16_sw128(&tmA, A, 2, dimsA, strA, boxA, dt);
  if (rc) return rc;
  uint64_t dimsB[2] = {(uint64_t)K, (uint64_t)N}, strB[1] = {(uint64_t)ldb * esize};
  uint32_t boxB[2] = {(uint32_t)bk, (uint32_t)bn};
  rc = make_tmap_bf16_sw128(&tmB, B, 2, dimsB, strB, boxB, dt);
  if (rc) return rc;

  GemmParams p;
  p.M = M;
  p.N = N;
  p.K = K;
  p.ldd = ldd;
  p.D = D;
  p.gate = gate;
  p.nr_gamma = norm_rope ? norm_rope->gamma : nullptr;
  p.nr_cs = norm_rope ? norm_rope->cs : nullptr;
  p.nr_eps = norm_rope ? norm_rope->eps : 0.0f;
  p.scale_a = scale_a;
  p.scale_b = scale_b;
  p.num_m_blk = (M + BM - 1) / BM;
  p.num_n_blk = (N + bn - 1) / bn;
  p.num_k_blk = (K + bk - 1) / bk;
  // keep one super-column of B (super_n * bn * K * esize bytes) well inside the 50 MB L2
  long long col_bytes = (long long)bn * K * esize;
  int sn = (int)((16ll << 20) / (col_bytes > 0 ? col_bytes : 1));
  if (sn < 1) sn = 1;
  if (sn > p.num_n_blk) sn = p.num_n_blk;
  p.super_n = sn;
  if (fp8) return bn == 64 ? dispatch_epi<64, true>(epilogue, tmA, tmB, p, st)
                           : dispatch_epi<128, true>(epilogue, tmA, tmB, p, st);
  switch (bn) {
    case 64: return dispatch_epi<64, false>(epilogue, tmA, tmB, p, st);
    case 128: return dispatch_epi<128, false>(epilogue, tmA, tmB, p, st);
    default: return dispatch_epi<256, false>(epilogue, tmA, tmB, p, st);
  }
}

// Host entries used by the engine and by the C ABI.
int gemm_bf16(const void* A, const void* B, void* D, int M, int N, int K, int lda, int ldb, int ldd,
              int epilogue, const float* gate, int block_n, cudaStream_t st, const NormRope* norm_rope) {
  return gemm_any(A, B, nullptr, nullptr, D, M, N, K, lda, ldb, ldd, epilogue, gate, block_n, st, norm_rope);
}

int gemm_fp8(const void* A8, const float* scale_a, const void* B8, const float* scale_b, void* D, int M, int N, int K,
             int lda, int ldb, int ldd, int epilogue, const float* gate, int block_n, cudaStream_t st,
             const NormRope* norm_rope) {
  G3C_REQUIRE(scale_a && scale_b, "gemm_fp8: null scale vector");
  G3C_REQUIRE((reinterpret_cast<uintptr_t>(scale_a) & 15) == 0 && (reinterpret_cast<uintptr_t>(scale_b) & 15) == 0,
              "gemm_fp8: scale vectors must be 16-byte aligned");
  return gemm_any(A8, B8, scale_a, scale_b, D, M, N, K, lda, ldb, ldd, epilogue, gate, block_n, st, norm_rope);
}

}  // namespace g3c

extern "C" int g3c_gemm_bf16(const void* A, const void* B, void* D, int M, int N, int K, int lda,
                             int ldb, int ldd, int epilogue, const float* gate, int block_n,
                             void* stream) {
  return g3c::gemm_bf16(A, B, D, M, N, K, lda, ldb, ldd, epilogue, gate, block_n,
                        (cudaStream_t)stream);
}

extern "C" int g3c_gemm_fp8(const void* A8, const float* scale_A, const void* B8, const float* scale_B, void* D, int M,
                            int N, int K, int lda, int ldb, int ldd, int epilogue, const float* gate, int block_n,
                            void* stream) {
  return g3c::gemm_fp8(A8, scale_A, B8, scale_B, D, M, N, K, lda, ldb, ldd, epilogue, gate, block_n,
                       (cudaStream_t)stream);
}

extern "C" int g3c_gemm_norm_rope_fp8(const void* A8, const float* scale_A, const void* B8, const float* scale_B, void* D,
                                      int M, int N, int K, int lda, int ldb, int ldd, const float* gamma,
                                      const float* cos_sin, float eps, void* stream) {
  g3c::NormRope nr;
  nr.gamma = gamma;
  nr.cs = cos_sin;
  nr.eps = eps;
  return g3c::gemm_fp8(A8, scale_A, B8, scale_B, D, M, N, K, lda, ldb, ldd, G3C_EPI_BF16, nullptr, 0,
                       (cudaStream_t)stream, &nr);
}

extern "C" int g3c_gemm_norm_rope_bf16(const void* A, const void* B, void* D, int M, int N, int K, int lda, int ldb,
                                       int ldd, const float* gamma, const float* cos_sin, float eps, void* stream) {
  g3c::NormRope nr;
  nr.gamma = gamma;
  nr.cs = cos_sin;
  nr.eps = eps;
  return g3c::gemm_bf16(A, B, D, M, N, K, lda, ldb, ldd, G3C_EPI_BF16, nullptr, 0, (cudaStream_t)stream, &nr);
}
