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
//                                registers, fused epilogue from the registers into a shared-memory staging buffer
//                                that TMA stores to global memory (or, for the gated residual, reduce-adds into it)
// The producer runs ahead into the next tile while the consumers run the epilogue of the current one, and the last
// TMA store of a tile drains while the consumers already run the next tile's MMAs.
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
  int n_tma;           // columns [0, n_tma) leave through the TMA map of D: N rounded down to 16 bytes (TMA writes
                       // whole 16-byte pieces of a row); the rest of the row is stored by the threads
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

// Output boxes: 64 rows (one consumer warpgroup) x 128 bytes (64 bf16 / 32 f32 columns, one swizzle span).
constexpr int OUT_BOX_ROWS = 64;
constexpr int OUT_BOX_BYTES = OUT_BOX_ROWS * 128;

template <int BN>
struct GemmSmem {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (192 * 1024) / kStageBytes;  // 4 / 6 / 8 stages for BN = 256 / 128 / 64
  static constexpr int kRingBytes = kStages * kStageBytes;
  static constexpr int kStagingBytes = 2 * OUT_BOX_BYTES;      // per consumer warpgroup: two output boxes per round
  static constexpr int kBarBytes = 256;
  static constexpr int kTotal = kRingBytes + 2 * kStagingBytes + kBarBytes + 1024;  // + alignment slack
  static_assert(kRingBytes % 1024 == 0, "the staging buffers need the 1024-byte alignment of the 128-byte swizzle");
  static_assert(kTotal <= 227 * 1024, "shared memory per CTA");
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

// Output staging of one consumer warpgroup.  Its 64 rows of a tile leave in rounds of at most two output boxes: the
// warpgroup writes a round into its staging half in the layout of the TMA box with the 128-byte swizzle (16-byte chunk
// j of box row r at chunk j ^ (r % 8)), and one thread stores the boxes to D, or for the gated residual reduce-adds them
// into x in L2 (every element of x still has exactly one owning tile, so the sum stays deterministic).  TMA clips rows
// >= M and columns >= n_tma.  A round only waits until the previous round's boxes have been read out of shared memory, so
// the last round of a tile drains while the warpgroup already runs the next tile's MMAs.
struct OutStage {
  uint8_t* base;    // this warpgroup's staging half (1024-byte aligned)
  uint32_t buf;     // its shared-window address
  uint32_t bar_id;  // named barrier of the warpgroup's 128 threads
  bool leader;      // the one thread that issues, commits and waits for the TMA stores
  uint32_t row;     // byte offset of the thread's first accumulator row r = 16 warp + lane / 4 inside a box
  uint32_t sw;      // lane / 4 = r % 8, the same for both of the thread's rows (r, r + 8): the swizzle of its chunks
  uint32_t col_q;   // 2 (lane % 4): the thread's first column inside an 8-column accumulator group
};

// The thread's staging addresses for elements of kEsize bytes: `thr` is its first value pair in row r of box 0 before
// the swizzle, `sw16` = (r % 8) << 4 the XOR on the chunk bits [4, 7) of a box row.  Both are produced after the
// mainloop (an empty asm the compiler cannot look through), so that the addresses are not hoisted into it and kept
// live beside the accumulators.
struct StageAddr {
  uint32_t thr, sw16;
};
template <int kEsize>
__device__ __forceinline__ StageAddr stage_addr_base(const OutStage& o) {
  StageAddr a{o.buf + o.row + o.col_q * kEsize, o.sw << 4};
  asm volatile("" : "+r"(a.thr), "+r"(a.sw16));
  return a;
}
// Shared address of the thread's value pair for accumulator group i (columns 8i + col_q + {0, 1} of the tile; only
// i modulo the groups of one round matters) and row half h (rows r + 8h).  The chunk bits of `thr` + the column byte
// offset are those of the unswizzled row (the buffer is 1024-byte aligned and rows are 128 bytes), so the swizzle is
// one XOR.
template <int kEsize>
__device__ __forceinline__ uint32_t stage_addr(const StageAddr& a, int i, int h) {
  constexpr int kGroupsPerBox = 128 / (8 * kEsize);  // 8 (bf16) or 4 (f32)
  const uint32_t col_byte = (uint32_t)(i % kGroupsPerBox) * 8 * kEsize;
  const uint32_t box = (uint32_t)(i / kGroupsPerBox) % 2;
  return ((a.thr + h * 8 * 128 + col_byte) ^ a.sw16) + box * OUT_BOX_BYTES;
}
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;\n" ::"r"(addr), "r"(v));
}
__device__ __forceinline__ void st_shared_f32x2(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};\n" ::"r"(addr), "f"(a), "f"(b));
}
// Before the warpgroup writes a round: the previous round's boxes have been read out of the staging half.
__device__ __forceinline__ void stage_acquire(const OutStage& o) {
  if (o.leader) tma_store_wait_read<0>();
  named_bar_sync(o.bar_id, 128);
}
// After it: make the writes visible to the async proxy, then one thread stores `nbox` boxes (columns col0 + b * 128
// bytes, rows row0 ..) and commits them as one bulk group.  Columns [n_tma, N) (less than 16 bytes of a row, only when
// N is not a multiple of 16 bytes) are copied from the staging buffer by the warpgroup's threads.
template <bool kReduce, int kEsize>
__device__ __forceinline__ void stage_issue(const OutStage& o, const CUtensorMap* tmD, int nbox, int box_cols, int col0,
                                            int row0, const GemmParams& p) {
  fence_proxy_async();
  named_bar_sync(o.bar_id, 128);
  if (p.n_tma < p.N && p.n_tma >= col0 && p.n_tma < col0 + nbox * box_cols) {
    const int ntail = p.N - p.n_tma, tid = (int)(threadIdx.x % 128);
#pragma unroll 1
    for (int e = tid; e < OUT_BOX_ROWS * ntail; e += 128) {
      const int r = e / ntail, col = p.n_tma + e % ntail;
      if (row0 + r >= p.M) break;
      const uint32_t byte = (uint32_t)((col - col0) % box_cols) * kEsize;
      const uint32_t off = (uint32_t)((col - col0) / box_cols) * OUT_BOX_BYTES + r * 128 +
                           ((((byte >> 4) ^ (uint32_t)(r % 8))) << 4) + (byte & 15);
      const size_t g = (size_t)(row0 + r) * p.ldd + col;
      uint32_t v;
      if constexpr (kEsize == 2) {
        asm volatile("ld.shared.u16 %0, [%1];\n" : "=r"(v) : "r"(o.buf + off));
        reinterpret_cast<uint16_t*>(p.D)[g] = (uint16_t)v;
      } else {
        asm volatile("ld.shared.b32 %0, [%1];\n" : "=r"(v) : "r"(o.buf + off));
        float* d = reinterpret_cast<float*>(p.D) + g;
        *d = kReduce ? *d + __uint_as_float(v) : __uint_as_float(v);  // RN(x + RN(gate * acc)), as the TMA reduction
      }
    }
  }
  if (o.leader && row0 < p.M) {
    for (int b = 0; b < nbox; ++b) {
      if (col0 + b * box_cols >= p.n_tma) break;
      if constexpr (kReduce) tma_reduce_add_2d(tmD, o.base + b * OUT_BOX_BYTES, col0 + b * box_cols, row0);
      else tma_store_2d(tmD, o.base + b * OUT_BOX_BYTES, col0 + b * box_cols, row0);
    }
    tma_store_commit();
  }
}

// Accumulator layout of wgmma m64nNk16 (f32): thread t of the warpgroup holds, for i in [0, N/8),
//   acc[4i + 0], acc[4i + 1] -> row 16 * (t / 32) + (t % 32) / 4,     columns 8i + 2 (t % 4) + {0, 1}
//   acc[4i + 2], acc[4i + 3] -> the same columns eight rows further down.
// Fused Linear -> per-head RMSNorm -> rotate-half RoPE for the heads of a tile: the 128 columns of one head and row
// are spread over the four threads of a quad (reduced with two shuffles), and the rotate-half partners c and c + 64
// (accumulator indices i and i + 8) sit in the same thread.  reference: module/attention.py:263-266 (to_q/to_k =
// Linear + RMSNorm) and :268-283 (apply_rotary_pos_emb); same arithmetic as k_rmsnorm_rope (dit_elementwise.cu).
// One head is one round of two bf16 boxes (columns c and c + 64).
template <int BN>
__device__ __forceinline__ void epilogue_norm_rope(const float (&acc)[BN / 2], const GemmParams& p,
                                                   const CUtensorMap* tmD, const OutStage& o, int row_a, int row0,
                                                   int n_base) {
  const float* __restrict__ gamma = p.nr_gamma;
  const float* __restrict__ cs_tab = p.nr_cs;
  const int col_q = (int)o.col_q;
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
    stage_acquire(o);
    const StageAddr sa = stage_addr_base<2>(o);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row_a + 8 * h;
      if (row >= p.M) continue;
      const float rstd = rsqrtf(ss[h] * (1.0f / 128.0f) + p.nr_eps);
      const float* cs = cs_tab ? cs_tab + (size_t)row * 128 : nullptr;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = 8 * i + col_q;  // column inside the head, < 64; the partner is c + 64
        const float2 ga = __ldg(reinterpret_cast<const float2*>(gamma + c));
        const float2 gb = __ldg(reinterpret_cast<const float2*>(gamma + 64 + c));
        const int ia = 4 * (16 * hd + i) + 2 * h, ib = 4 * (16 * hd + i + 8) + 2 * h;
        float a[2] = {acc[ia] * (rstd * ga.x), acc[ia + 1] * (rstd * ga.y)};
        float b[2] = {acc[ib] * (rstd * gb.x), acc[ib + 1] * (rstd * gb.y)};
        if (cs) {
          const float2 co = __ldg(reinterpret_cast<const float2*>(cs + c));
          const float2 si = __ldg(reinterpret_cast<const float2*>(cs + 64 + c));
          const float cv[2] = {co.x, co.y}, sv[2] = {si.x, si.y};
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float n = a[e] * cv[e] - b[e] * sv[e], m = b[e] * cv[e] + a[e] * sv[e];
            a[e] = n;
            b[e] = m;
          }
        }
        st_shared_b32(stage_addr<2>(sa, i, h), pack_bf16x2(a[0], a[1]));
        st_shared_b32(stage_addr<2>(sa, i + 8, h), pack_bf16x2(b[0], b[1]));
      }
    }
    stage_issue<false, 2>(o, tmD, 2, 64, n_base + hd * 128, row0, p);
  }
}

// fp8: dequantise the accumulators in place, acc * scale_a[row] * scale_b[col], before any epilogue arithmetic (the
// RMSNorm of the fused to_q / to_k epilogue must see the dequantised values).  Rows / columns past M / N get zero
// accumulators (scale 0): TMA does not store them.
template <int BN>
__device__ __forceinline__ void dequantise(float (&acc)[BN / 2], const GemmParams& p, int row_a, int col_q, int n_base) {
  const float* __restrict__ scale_a = p.scale_a;
  const float* __restrict__ scale_b = p.scale_b;
  float sa[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) sa[h] = row_a + 8 * h < p.M ? __ldg(scale_a + row_a + 8 * h) : 0.f;
#pragma unroll
  for (int i = 0; i < BN / 8; ++i) {
    const int col = n_base + 8 * i + col_q;
    float2 sb = make_float2(0.f, 0.f);
    if (col + 1 < p.N) sb = __ldg(reinterpret_cast<const float2*>(scale_b + col));
    else if (col < p.N) sb.x = __ldg(scale_b + col);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      acc[4 * i + 2 * h] = acc[4 * i + 2 * h] * sa[h] * sb.x;
      acc[4 * i + 2 * h + 1] = acc[4 * i + 2 * h + 1] * sa[h] * sb.y;
    }
  }
}

// bf16 / GELU / f32 outputs, and the gated residual: x += RN(gate * acc), reduce-added by TMA.  A round is two boxes
// (128 bf16 or 64 f32 columns) or the whole tile when it is narrower.
template <int BN, int EPI>
__device__ __forceinline__ void epilogue(const float (&acc)[BN / 2], const GemmParams& p, const CUtensorMap* tmD,
                                         const OutStage& o, int row0, int n_base) {
  constexpr bool kGated = EPI == G3C_EPI_GATED_RESIDUAL_F32;
  constexpr int kEsize = (kGated || EPI == G3C_EPI_F32) ? 4 : 2;
  constexpr int kBoxCols = 128 / kEsize;
  constexpr int kRoundGroups = 2 * kBoxCols / 8 < BN / 8 ? 2 * kBoxCols / 8 : BN / 8;
  constexpr int kRoundBoxes = (8 * kRoundGroups + kBoxCols - 1) / kBoxCols;
  const float* __restrict__ gate = p.gate;
#pragma unroll
  for (int rd = 0; rd < BN / 8 / kRoundGroups; ++rd) {
    float2 g[kGated ? kRoundGroups : 1];
    if constexpr (kGated) {
      // the round's gate pairs, loaded ahead of the staging wait and the arithmetic
#pragma unroll
      for (int j = 0; j < kRoundGroups; ++j) {
        const int col = n_base + 8 * (rd * kRoundGroups + j) + (int)o.col_q;
        g[j] = make_float2(0.f, 0.f);
        if (col + 1 < p.N) g[j] = __ldg(reinterpret_cast<const float2*>(gate + col));
        else if (col < p.N) g[j].x = __ldg(gate + col);
      }
    }
    stage_acquire(o);
    const StageAddr sa = stage_addr_base<kEsize>(o);
#pragma unroll
    for (int j = 0; j < kRoundGroups; ++j) {
      const int i = rd * kRoundGroups + j;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
        if constexpr (EPI == G3C_EPI_GELU_BF16) {
          v0 = gelu_erf(v0);
          v1 = gelu_erf(v1);
        }
        if constexpr (kGated) {
          v0 = g[j].x * v0;
          v1 = g[j].y * v1;
        }
        if constexpr (kEsize == 2) st_shared_b32(stage_addr<2>(sa, i, h), pack_bf16x2(v0, v1));
        else st_shared_f32x2(stage_addr<4>(sa, i, h), v0, v1);
      }
    }
    stage_issue<kGated, kEsize>(o, tmD, kRoundBoxes, kBoxCols, n_base + rd * 8 * kRoundGroups, row0, p);
  }
}

template <int BN, int EPI, bool kFp8>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    k_gemm(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
           const __grid_constant__ CUtensorMap tmD, const GemmParams p) {
  using S = GemmSmem<BN>;
  constexpr int kStages = S::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * S::kABytes;
  uint8_t* staging = smem + S::kRingBytes;  // [2][kStagingBytes], one half per consumer warpgroup
  uint64_t* bars = reinterpret_cast<uint64_t*>(staging + 2 * S::kStagingBytes);
  uint64_t* full = bars;              // [kStages]
  uint64_t* empty = bars + kStages;   // [kStages]

  const uint32_t wg = threadIdx.x / 128;
  const uint32_t tid = threadIdx.x % 128;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmD);
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
    OutStage out;
    out.base = staging + c * S::kStagingBytes;
    out.buf = smem_u32(out.base);
    out.bar_id = 1 + c;
    out.leader = tid == 0;
    out.row = (16 * warp + lane / 4) * 128;
    out.sw = lane / 4;
    out.col_q = 2 * (lane % 4);
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
      const int row0 = m_blk * BM + (int)c * 64, row_a = row0 + (int)(warp * 16 + lane / 4);
      if constexpr (kFp8) dequantise<BN>(acc, p, row_a, (int)out.col_q, n_blk * BN);
      if constexpr (EPI == EPI_NORM_ROPE_BF16) epilogue_norm_rope<BN>(acc, p, &tmD, out, row_a, row0, n_blk * BN);
      else epilogue<BN, EPI>(acc, p, &tmD, out, row0, n_blk * BN);
    }
    // the staging buffer must outlive the reads of the last boxes, and the stores complete before the CTA retires
    if (out.leader) tma_store_wait_all<0>();
  }
}

template <int BN, int EPI, bool kFp8>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD, const GemmParams& p,
                       cudaStream_t st) {
  using S = GemmSmem<BN>;
  static bool configured = false;
  if (!configured) {
    G3C_CUDA(cudaFuncSetAttribute(k_gemm<BN, EPI, kFp8>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal));
    configured = true;
  }
  int tiles = p.num_m_blk * p.num_n_blk;
  int grid = tiles < sm_count() ? tiles : sm_count();
  k_gemm<BN, EPI, kFp8><<<grid, GEMM_THREADS, S::kTotal, st>>>(tmA, tmB, tmD, p);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

template <int BN, bool kFp8>
static int dispatch_epi(int epi, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmD,
                        const GemmParams& p, cudaStream_t st) {
  switch (epi) {
    case G3C_EPI_BF16: return launch_gemm<BN, G3C_EPI_BF16, kFp8>(tmA, tmB, tmD, p, st);
    case G3C_EPI_GELU_BF16: return launch_gemm<BN, G3C_EPI_GELU_BF16, kFp8>(tmA, tmB, tmD, p, st);
    case G3C_EPI_GATED_RESIDUAL_F32: return launch_gemm<BN, G3C_EPI_GATED_RESIDUAL_F32, kFp8>(tmA, tmB, tmD, p, st);
    case G3C_EPI_F32: return launch_gemm<BN, G3C_EPI_F32, kFp8>(tmA, tmB, tmD, p, st);
    case EPI_NORM_ROPE_BF16:
      if constexpr (BN >= 128) return launch_gemm<BN, EPI_NORM_ROPE_BF16, kFp8>(tmA, tmB, tmD, p, st);
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

  CUtensorMap tmA, tmB, tmD;
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
  // D in boxes of 64 rows x 128 bytes (the epilogue's staging layout); TMA clips rows >= M and columns >= n_tma
  const bool f32_out = epilogue == G3C_EPI_GATED_RESIDUAL_F32 || epilogue == G3C_EPI_F32;
  const int dsize = f32_out ? 4 : 2;
  const int n_tma = N / (16 / dsize) * (16 / dsize);
  // with n_tma = 0 the map is never used (the dimension must not be empty)
  uint64_t dimsD[2] = {(uint64_t)(n_tma > 0 ? n_tma : 16 / dsize), (uint64_t)M}, strD[1] = {(uint64_t)ldd * dsize};
  uint32_t boxD[2] = {(uint32_t)(128 / dsize), (uint32_t)OUT_BOX_ROWS};
  rc = make_tmap_bf16_sw128(&tmD, D, 2, dimsD, strD, boxD,
                            f32_out ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
  if (rc) return rc;

  GemmParams p;
  p.M = M;
  p.N = N;
  p.K = K;
  p.ldd = ldd;
  p.n_tma = n_tma;
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
  if (fp8) return bn == 64 ? dispatch_epi<64, true>(epilogue, tmA, tmB, tmD, p, st)
                           : dispatch_epi<128, true>(epilogue, tmA, tmB, tmD, p, st);
  switch (bn) {
    case 64: return dispatch_epi<64, false>(epilogue, tmA, tmB, tmD, p, st);
    case 128: return dispatch_epi<128, false>(epilogue, tmA, tmB, tmD, p, st);
    default: return dispatch_epi<256, false>(epilogue, tmA, tmB, tmD, p, st);
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
