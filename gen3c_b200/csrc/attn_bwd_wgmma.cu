// Backward of the drop-in attention operator (g3c_attn_fwd_sbhd_lse), head_dim 128, no mask, on wgmma.
//   P = 2^(s sl2 - lse)  (s = q . k, lse from the forward in log2 units),  Delta_i = sum_d dO_id O_id,
//   dS = P o (dP - Delta),  dP = dO V^T,  dV = P^T dO,  dQ = scale dS K,  dK = scale dS^T Q
// in three launches, every gradient element with exactly one writer (no atomics: bitwise reproducible):
//   k_attn_bwd_delta  Delta [heads][Lq] from the bf16 O and dO, one warp per (token, head).
//   k_attn_bwd_dkdv   one CTA = 128 keys of one head.  Warpgroup 0 is the TMA producer: K and V once, then Q_i and dO_i
//                     tiles of 64 queries (with that tile's lse and Delta) through a ring of ABKV_STAGES stages.
//                     Warpgroups 1-2 own 64 keys each and keep dK, dV (64 x 128 fp32 each) in registers; per query tile
//                       S^T = K Q_i^T and dP^T = V dO_i^T     (A: K, V rows in shared memory, K-major in d;
//                                                              B: Q_i, dO_i, K-major in d)
//                       P^T, dS^T in registers                 (lse +inf and Delta 0 past Lq: those columns are 0)
//                       dV += bf16(P^T) dO_i, dK += bf16(dS^T) Q_i   (A: registers, the accumulator-as-A layout;
//                                                              B: dO_i, Q_i token-major, MN-major with imm-trans-b)
//   k_attn_bwd_dq     one CTA = 128 queries of one head, Q and dO resident, K_j and V_j streamed through K and V rings
//                     as in the forward; warpgroups 1-2 own 64 queries each and keep dQ in registers:
//                       S = Q K_j^T, dP = dO V_j^T             (A: Q, dO rows K-major; B: K_j, V_j K-major)
//                       P (keys past Lk masked to 0), dS
//                       dQ += bf16(dS) K_j                     (B: K_j token-major, MN-major as V in the forward's P.V)
// S and dP are computed in both kernels (7 tile products per (query, key) tile instead of FlashAttention's 5): the price
// of a dQ without atomics.  Waits are bounded as in the forward (G3C_MBAR_TIMEOUT_NS).
#include <cmath>

#include "kernels.h"

namespace g3c {

constexpr int AB_THREADS = 384;
constexpr int AB_TILE = 128;               // keys per dK/dV CTA, queries per dQ CTA, keys per dQ step, head dim
constexpr int AB_QT = 64;                  // queries per dK/dV step
constexpr int AB_HALF = 128 * 128;         // one 64-dim half of a 128-token tile (bytes)
constexpr int AB_TILE_BYTES = 2 * AB_HALF;
constexpr int AB_QT_HALF = AB_QT * 128;    // one 64-dim half of a 64-token tile
constexpr int AB_QT_BYTES = 2 * AB_QT_HALF;
constexpr int ABKV_STAGES = 4;
// K, V; the Q_i and dO_i stages; lse and Delta of each stage; barriers
constexpr int ABKV_SMEM = 2 * AB_TILE_BYTES + ABKV_STAGES * 2 * AB_QT_BYTES + ABKV_STAGES * 2 * AB_QT * 4 + 256 + 1024;
static_assert(ABKV_SMEM <= 227 * 1024, "attention backward: dK/dV shared memory exceeds 227 KB");
static_assert(1 + 2 * ABKV_STAGES + 1 <= 256 / 8, "attention backward: dK/dV barriers exceed their 256-byte area");
constexpr int ABQ_STAGES = 2;
// Q, dO; the K and V rings; barriers
constexpr int ABQ_SMEM = 2 * AB_TILE_BYTES + ABQ_STAGES * 2 * AB_TILE_BYTES + 256 + 1024;
static_assert(ABQ_SMEM <= 227 * 1024, "attention backward: dQ shared memory exceeds 227 KB");

struct AttnBwdParams {
  int Lq, Lk;
  float sl2;            // attn_scale_log2(scale), as in the forward
  float scale;          // the natural-log softmax scale: dQ and dK carry it
  const float* lse;     // [heads][Lq]
  const float* delta;   // [heads][Lq]
  __nv_bfloat16* dq;
  __nv_bfloat16* dk;
  __nv_bfloat16* dv;
  int lddq, lddk, lddv;
};

// m64nN fp32 accumulator -> the bf16 A fragments of the next wgmma (k-step kk = a[4kk .. 4kk + 3]): a[2i] = row r,
// a[2i + 1] = row r + 8, columns 8i + 2 (lane % 4) + {0, 1} (pack_p of the forward, for any N)
template <int N>
__device__ __forceinline__ void pack_a(uint32_t (&a)[N / 2], const float (&s)[N]) {
#pragma unroll
  for (int i = 0; i < N / 4; ++i) {
    a[2 * i] = pack_bf16x2(s[4 * i], s[4 * i + 1]);
    a[2 * i + 1] = pack_bf16x2(s[4 * i + 2], s[4 * i + 3]);
  }
}

// rows row0 + 16 warp + lane / 4 + {0, 8} of a 64 x 128 accumulator, times f, to bf16 at dst (ld), rows < limit
__device__ __forceinline__ void store_acc(__nv_bfloat16* dst, int ld, int row0, int limit, const float (&acc)[64],
                                          float f, uint32_t warp, uint32_t lane) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + (int)(warp * 16 + lane / 4) + 8 * h;
    if (row >= limit) continue;
    __nv_bfloat16* d = dst + (size_t)row * ld + 2 * (lane % 4);
#pragma unroll
    for (int i = 0; i < 16; ++i)
      *reinterpret_cast<uint32_t*>(d + 8 * i) = pack_bf16x2(acc[4 * i + 2 * h] * f, acc[4 * i + 2 * h + 1] * f);
  }
}

// Delta[h][q] = sum_d dO[q, h, d] O[q, h, d] in fp32 (products of the bf16 values, a fixed summation order)
__global__ void k_attn_bwd_delta(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ dout,
                                 float* __restrict__ delta, int Lq, int heads, int ldo, int lddo) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const uint32_t lane = threadIdx.x % 32;
  if (w >= (long long)Lq * heads) return;
  const int q = (int)(w / heads), h = (int)(w % heads);  // consecutive warps: the heads of one token row
  const uint2 a = *reinterpret_cast<const uint2*>(o + (size_t)q * ldo + h * 128 + 4 * lane);
  const uint2 b = *reinterpret_cast<const uint2*>(dout + (size_t)q * lddo + h * 128 + 4 * lane);
  const float2 a0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&a.x));
  const float2 a1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&a.y));
  const float2 b0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&b.x));
  const float2 b1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&b.y));
  float s = a0.x * b0.x;
  s = fmaf(a0.y, b0.y, s);
  s = fmaf(a1.x, b1.x, s);
  s = fmaf(a1.y, b1.y, s);
  s = warp_sum(s);
  if (lane == 0) delta[(size_t)h * Lq + q] = s;
}

__global__ void __launch_bounds__(AB_THREADS, 1)
    k_attn_bwd_dkdv(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmDO,
                    const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                    const AttnBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_k = smem;
  uint8_t* smem_v = smem_k + AB_TILE_BYTES;
  uint8_t* smem_q = smem_v + AB_TILE_BYTES;              // [ABKV_STAGES] Q_i tiles
  uint8_t* smem_do = smem_q + ABKV_STAGES * AB_QT_BYTES;  // [ABKV_STAGES] dO_i tiles
  float* stat = reinterpret_cast<float*>(smem_do + ABKV_STAGES * AB_QT_BYTES);  // [ABKV_STAGES][lse 64 | Delta 64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(stat + ABKV_STAGES * 2 * AB_QT);
  uint64_t* kv_full = bars;              // [1]
  uint64_t* full = bars + 1;             // [ABKV_STAGES]
  uint64_t* empty = full + ABKV_STAGES;  // [ABKV_STAGES]
  uint64_t* done = empty + ABKV_STAGES;  // [1]: both consumer warpgroups finished

  const uint32_t wg = threadIdx.x / 128;
  const uint32_t tid = threadIdx.x % 128;
  const int head = blockIdx.y;
  const int k0 = blockIdx.x * AB_TILE;
  const int n_q = (p.Lq + AB_QT - 1) / AB_QT;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmDO);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(kv_full, 1);
    for (int i = 0; i < ABKV_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);  // one arrive per consumer warpgroup
    }
    mbar_init(done, 2);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===== producer: warp 0 (lane 0 issues the TMA, the warp copies lse and Delta) =====
    setmaxnreg_dec<24>();
    if (tid < 32) {
      const uint32_t lane = tid;
      if (lane == 0) {
        mbar_expect_tx(kv_full, 2 * AB_TILE_BYTES);
        for (int h = 0; h < 2; ++h) {
          tma_load_2d(smem_k + h * AB_HALF, &tmK, kv_full, head * 128 + h * 64, k0);
          tma_load_2d(smem_v + h * AB_HALF, &tmV, kv_full, head * 128 + h * 64, k0);
        }
      }
      uint32_t stage = 0, phase = 0;
      for (int i = 0; i < n_q; ++i) {
        if (lane == 0) mbar_wait_ns(&empty[stage], phase ^ 1, G3C_MBAR_TIMEOUT_NS);
        __syncwarp();
        // queries past Lq: lse = +inf and Delta = 0, so their P^T and dS^T columns are exactly 0 (Q and dO are
        // zero-filled there by the TMA, and 2^(0 - lse) would not be)
        float* st = stat + stage * 2 * AB_QT;
        for (int r = (int)lane; r < AB_QT; r += 32) {
          const int q = i * AB_QT + r;
          const bool in = q < p.Lq;
          st[r] = in ? p.lse[(size_t)head * p.Lq + q] : INFINITY;
          st[AB_QT + r] = in ? p.delta[(size_t)head * p.Lq + q] : 0.f;
        }
        __syncwarp();  // the warp's stores happen before lane 0's arrive, which releases them to the consumers
        if (lane == 0) {
          mbar_expect_tx(&full[stage], 2 * AB_QT_BYTES);
          for (int h = 0; h < 2; ++h) {
            tma_load_2d(smem_q + stage * AB_QT_BYTES + h * AB_QT_HALF, &tmQ, &full[stage], head * 128 + h * 64,
                        i * AB_QT);
            tma_load_2d(smem_do + stage * AB_QT_BYTES + h * AB_QT_HALF, &tmDO, &full[stage], head * 128 + h * 64,
                        i * AB_QT);
          }
        }
        if (++stage == ABKV_STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      // a consumer whose barrier wait timed out has exited without arriving: trap here, within the bound
      if (lane == 0) mbar_wait_ns(done, 0, G3C_MBAR_TIMEOUT_NS);
    }
  } else {
    // ===== consumers: warpgroup c owns keys [k0 + 64c, k0 + 64c + 64) =====
    setmaxnreg_inc<240>();
    const uint32_t c = __shfl_sync(0xffffffffu, wg - 1, 0);
    const uint32_t warp = tid / 32, lane = tid % 32;
    const unsigned long long tmo = G3C_MBAR_TIMEOUT_NS;
    // accumulator layouts: m64n128 (dK, dV) as in the forward; m64n64 (S^T, dP^T), i in [0, 8): s[4i + {0,1}] = key
    // 16 warp + lane/4, queries 8i + 2 (lane%4) + {0,1} of the tile; s[4i + {2,3}] = the key eight rows further down
    float dk[64], dv[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) dk[i] = dv[i] = 0.f;
    float s[32], dp[32];
    uint32_t pa[16], pd[16];  // bf16 P^T and dS^T: the A operands of the dV and dK MMAs
    const float sl2 = p.sl2;
    const uint64_t dka = make_sdesc_sw128(smem_u32(smem_k + c * 64 * 128));
    const uint64_t dva = make_sdesc_sw128(smem_u32(smem_v + c * 64 * 128));
    mbar_wait_ns_or_exit(kv_full, 0, tmo);
    uint32_t stage = 0, phase = 0;
    for (int i = 0; i < n_q; ++i) {
      mbar_wait_ns_or_exit(&full[stage], phase, tmo);
      const uint32_t qa = smem_u32(smem_q + stage * AB_QT_BYTES), oa = smem_u32(smem_do + stage * AB_QT_BYTES);
      const uint64_t dqk = make_sdesc_sw128(qa), dok = make_sdesc_sw128(oa);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {  // head dimensions 16 kk .. 16 kk + 15
        const uint32_t half = kk >> 2, off = (kk & 3) * 32;
        wgmma_ss_n64(s, sdesc_advance(dka, half * AB_HALF + off), sdesc_advance(dqk, half * AB_QT_HALF + off),
                     kk > 0 ? 1u : 0u);
      }
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const uint32_t half = kk >> 2, off = (kk & 3) * 32;
        wgmma_ss_n64(dp, sdesc_advance(dva, half * AB_HALF + off), sdesc_advance(dok, half * AB_QT_HALF + off),
                     kk > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
      fence_regs(dp);
      const float* st = stat + stage * 2 * AB_QT;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * j + 2 * (int)(lane % 4) + e;
          const float nl = -st[col], dl = st[AB_QT + col];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int x = 4 * j + 2 * h + e;
            const float pv = ex2_approx(fmaf(s[x], sl2, nl));
            s[x] = pv;
            dp[x] = pv * (dp[x] - dl);
          }
        }
      }
      pack_a<32>(pa, s);
      pack_a<32>(pd, dp);
      const uint64_t dqm = make_sdesc_sw128_mn(qa, AB_QT_HALF), dom = make_sdesc_sw128_mn(oa, AB_QT_HALF);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {  // queries 16 kk .. 16 kk + 15 of the tile
        const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
        wgmma_rs_n128_tb(dv, a, sdesc_advance(dom, kk * 16 * 128));
      }
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t a[4] = {pd[4 * kk], pd[4 * kk + 1], pd[4 * kk + 2], pd[4 * kk + 3]};
        wgmma_rs_n128_tb(dk, a, sdesc_advance(dqm, kk * 16 * 128));
      }
      wgmma_commit();
      wgmma_wait<0>();  // nothing stays in flight across a barrier wait (that would serialise every wgmma)
      fence_regs(dk);
      fence_regs(dv);
      fence_regs(pa);
      fence_regs(pd);
      if (tid == 0) mbar_arrive(&empty[stage]);  // Q_i, dO_i and their lse, Delta read for the last time
      if (++stage == ABKV_STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    const int row0 = k0 + (int)c * 64;
    store_acc(p.dv + head * 128, p.lddv, row0, p.Lk, dv, 1.0f, warp, lane);
    store_acc(p.dk + head * 128, p.lddk, row0, p.Lk, dk, p.scale, warp, lane);
    if (tid == 0) mbar_arrive(done);
  }
}

__global__ void __launch_bounds__(AB_THREADS, 1)
    k_attn_bwd_dq(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmDO,
                  const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                  const AttnBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_do = smem_q + AB_TILE_BYTES;
  uint8_t* smem_k = smem_do + AB_TILE_BYTES;             // [ABQ_STAGES] K tiles
  uint8_t* smem_v = smem_k + ABQ_STAGES * AB_TILE_BYTES;  // [ABQ_STAGES] V tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_v + ABQ_STAGES * AB_TILE_BYTES);
  uint64_t* q_full = bars;                   // [1]
  uint64_t* k_full = bars + 1;               // [ABQ_STAGES]
  uint64_t* v_full = k_full + ABQ_STAGES;    // [ABQ_STAGES]
  uint64_t* k_empty = v_full + ABQ_STAGES;   // [ABQ_STAGES]
  uint64_t* v_empty = k_empty + ABQ_STAGES;  // [ABQ_STAGES]
  uint64_t* done = v_empty + ABQ_STAGES;     // [1]

  const uint32_t wg = threadIdx.x / 128;
  const uint32_t tid = threadIdx.x % 128;
  const int head = blockIdx.y;
  const int q0 = blockIdx.x * AB_TILE;
  const int n_kv = (p.Lk + AB_TILE - 1) / AB_TILE;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmDO);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < ABQ_STAGES; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&k_empty[i], 2);
      mbar_init(&v_empty[i], 2);
    }
    mbar_init(done, 2);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===== TMA producer =====
    setmaxnreg_dec<24>();
    if (tid == 0) {
      mbar_expect_tx(q_full, 2 * AB_TILE_BYTES);
      for (int h = 0; h < 2; ++h) {
        tma_load_2d(smem_q + h * AB_HALF, &tmQ, q_full, head * 128 + h * 64, q0);
        tma_load_2d(smem_do + h * AB_HALF, &tmDO, q_full, head * 128 + h * 64, q0);
      }
      uint32_t stage = 0, phase = 0;
      for (int j = 0; j < n_kv; ++j) {
        mbar_wait_ns(&k_empty[stage], phase ^ 1, G3C_MBAR_TIMEOUT_NS);
        mbar_expect_tx(&k_full[stage], AB_TILE_BYTES);
        for (int h = 0; h < 2; ++h)
          tma_load_2d(smem_k + stage * AB_TILE_BYTES + h * AB_HALF, &tmK, &k_full[stage], head * 128 + h * 64,
                      j * AB_TILE);
        mbar_wait_ns(&v_empty[stage], phase ^ 1, G3C_MBAR_TIMEOUT_NS);
        mbar_expect_tx(&v_full[stage], AB_TILE_BYTES);
        for (int h = 0; h < 2; ++h)
          tma_load_2d(smem_v + stage * AB_TILE_BYTES + h * AB_HALF, &tmV, &v_full[stage], head * 128 + h * 64,
                      j * AB_TILE);
        if (++stage == ABQ_STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      mbar_wait_ns(done, 0, G3C_MBAR_TIMEOUT_NS);
    }
  } else {
    // ===== consumers: warpgroup c owns query rows [q0 + 64c, q0 + 64c + 64) =====
    setmaxnreg_inc<240>();
    const uint32_t c = __shfl_sync(0xffffffffu, wg - 1, 0);
    const uint32_t warp = tid / 32, lane = tid % 32;
    const unsigned long long tmo = G3C_MBAR_TIMEOUT_NS;
    // this thread's rows (row_a and row_a + 8): rows past Lq get lse = +inf and Delta = 0 (P = dS = 0; not stored)
    const int row_a = q0 + (int)(c * 64 + warp * 16 + lane / 4);
    float nl[2], dl[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row_a + 8 * h;
      nl[h] = row < p.Lq ? -p.lse[(size_t)head * p.Lq + row] : -INFINITY;
      dl[h] = row < p.Lq ? p.delta[(size_t)head * p.Lq + row] : 0.f;
    }
    float dq[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) dq[i] = 0.f;
    float s[64], dp[64];
    uint32_t pd[32];  // bf16 dS: the A operand of the dQ MMA
    const float sl2 = p.sl2;
    const uint64_t dqa = make_sdesc_sw128(smem_u32(smem_q + c * 64 * 128));
    const uint64_t doa = make_sdesc_sw128(smem_u32(smem_do + c * 64 * 128));
    mbar_wait_ns_or_exit(q_full, 0, tmo);
    for (int j = 0; j < n_kv; ++j) {
      const int st = j & 1;
      const uint32_t par = ((uint32_t)j >> 1) & 1u;
      mbar_wait_ns_or_exit(&k_full[st], par, tmo);
      mbar_wait_ns_or_exit(&v_full[st], par, tmo);
      const uint32_t ka = smem_u32(smem_k + st * AB_TILE_BYTES), va = smem_u32(smem_v + st * AB_TILE_BYTES);
      const uint64_t dkk = make_sdesc_sw128(ka), dvk = make_sdesc_sw128(va);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {  // head dimensions 16 kk .. 16 kk + 15
        const uint32_t off = (kk >> 2) * AB_HALF + (kk & 3) * 32;
        wgmma_ss_n128(s, sdesc_advance(dqa, off), sdesc_advance(dkk, off), kk > 0 ? 1u : 0u);
      }
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const uint32_t off = (kk >> 2) * AB_HALF + (kk & 3) * 32;
        wgmma_ss_n128(dp, sdesc_advance(doa, off), sdesc_advance(dvk, off), kk > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
      fence_regs(dp);
      if (tid == 0) mbar_arrive(&v_empty[st]);  // V_j read for the last time
      const int valid = p.Lk - j * AB_TILE;  // keys of this tile below Lk (>= 128 except in a ragged last tile)
#pragma unroll
      for (int i = 0; i < 16; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const bool in = 8 * i + 2 * (int)(lane % 4) + e < valid;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int x = 4 * i + 2 * h + e;
            const float pv = in ? ex2_approx(fmaf(s[x], sl2, nl[h])) : 0.f;
            dp[x] = pv * (dp[x] - dl[h]);
          }
        }
      }
      pack_a<64>(pd, dp);
      const uint64_t dkm = make_sdesc_sw128_mn(ka, AB_HALF);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {  // keys 16 kk .. 16 kk + 15 of the tile
        const uint32_t a[4] = {pd[4 * kk], pd[4 * kk + 1], pd[4 * kk + 2], pd[4 * kk + 3]};
        wgmma_rs_n128_tb(dq, a, sdesc_advance(dkm, kk * 16 * 128));
      }
      wgmma_commit();
      wgmma_wait<0>();  // nothing stays in flight across a barrier wait (that would serialise every wgmma)
      fence_regs(dq);
      fence_regs(pd);
      if (tid == 0) mbar_arrive(&k_empty[st]);  // K_j read for the last time
    }
    store_acc(p.dq + head * 128, p.lddq, q0 + (int)c * 64, p.Lq, dq, p.scale, warp, lane);
    if (tid == 0) mbar_arrive(done);
  }
}

// TMA map of a token-major bf16 operand [rows, heads*128] (leading dimension ld): boxes of 64 head dims x box_rows
static int make_tmap_rows(CUtensorMap* m, const void* base, int rows, int heads, int ld, int box_rows) {
  uint64_t dims[2] = {(uint64_t)heads * 128, (uint64_t)rows}, str[1] = {(uint64_t)ld * 2};
  uint32_t box[2] = {64, (uint32_t)box_rows};
  return make_tmap_bf16_sw128(m, base, 2, dims, str, box);
}

int attn_bwd_sbhd(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                  float* delta_ws, void* dq, void* dk, void* dv, int Lq, int Lk, int batch, int heads, int ldq, int ldk,
                  int ldv, int ldo, int lddo, int lddq, int lddk, int lddv, float scale, cudaStream_t st) {
  G3C_REQUIRE(q && k && v && o && dout && lse && delta_ws && dq && dk && dv, "attn_bwd_sbhd: null operand");
  G3C_REQUIRE(Lq > 0 && Lk > 0, "attn_bwd_sbhd: Lq=%d and Lk=%d must be >= 1", Lq, Lk);
  G3C_REQUIRE(batch > 0 && heads > 0 && (long long)batch * heads <= 65535,
              "attn_bwd_sbhd: batch=%d x heads=%d must be in [1, 65535]", batch, heads);
  const int bh = batch * heads;
  const int lds[8] = {ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv};
  bool ld_ok = true;
  for (int ld : lds) ld_ok = ld_ok && ld % 8 == 0 && ld >= bh * 128;
  G3C_REQUIRE(ld_ok,
              "attn_bwd_sbhd: leading dimensions (%d, %d, %d, %d, %d, %d, %d, %d) must be >= batch*heads*128 = %d and "
              "multiples of 8",
              ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv, bh * 128);
  G3C_REQUIRE(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
                reinterpret_cast<uintptr_t>(o) | reinterpret_cast<uintptr_t>(dout) | reinterpret_cast<uintptr_t>(dq) |
                reinterpret_cast<uintptr_t>(dk) | reinterpret_cast<uintptr_t>(dv)) & 15) == 0,
              "attn_bwd_sbhd: q, k, v, o, dout, dq, dk and dv must be 16-byte aligned");
  G3C_REQUIRE(((reinterpret_cast<uintptr_t>(lse) | reinterpret_cast<uintptr_t>(delta_ws)) & 3) == 0,
              "attn_bwd_sbhd: lse and delta_ws must be 4-byte aligned");
  CUtensorMap tmQ64, tmDO64, tmQ, tmDO, tmK, tmV;
  int rc = make_tmap_rows(&tmQ64, q, Lq, bh, ldq, AB_QT);
  if (!rc) rc = make_tmap_rows(&tmDO64, dout, Lq, bh, lddo, AB_QT);
  if (!rc) rc = make_tmap_rows(&tmQ, q, Lq, bh, ldq, AB_TILE);
  if (!rc) rc = make_tmap_rows(&tmDO, dout, Lq, bh, lddo, AB_TILE);
  if (!rc) rc = make_tmap_rows(&tmK, k, Lk, bh, ldk, AB_TILE);
  if (!rc) rc = make_tmap_rows(&tmV, v, Lk, bh, ldv, AB_TILE);
  if (rc) return rc;
  static bool configured = false;
  if (!configured) {
    G3C_CUDA(cudaFuncSetAttribute(k_attn_bwd_dkdv, cudaFuncAttributeMaxDynamicSharedMemorySize, ABKV_SMEM));
    G3C_CUDA(cudaFuncSetAttribute(k_attn_bwd_dq, cudaFuncAttributeMaxDynamicSharedMemorySize, ABQ_SMEM));
    configured = true;
  }
  AttnBwdParams p = {};
  p.Lq = Lq;
  p.Lk = Lk;
  p.sl2 = attn_scale_log2(scale);
  p.scale = scale;
  p.lse = lse;
  p.delta = delta_ws;
  p.dq = reinterpret_cast<__nv_bfloat16*>(dq);
  p.dk = reinterpret_cast<__nv_bfloat16*>(dk);
  p.dv = reinterpret_cast<__nv_bfloat16*>(dv);
  p.lddq = lddq;
  p.lddk = lddk;
  p.lddv = lddv;
  const long long warps = (long long)Lq * bh;
  k_attn_bwd_delta<<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(o),
                                                                reinterpret_cast<const __nv_bfloat16*>(dout), delta_ws,
                                                                Lq, bh, ldo, lddo);
  G3C_CUDA(cudaGetLastError());
  k_attn_bwd_dkdv<<<dim3((Lk + AB_TILE - 1) / AB_TILE, bh), AB_THREADS, ABKV_SMEM, st>>>(tmQ64, tmDO64, tmK, tmV, p);
  G3C_CUDA(cudaGetLastError());
  k_attn_bwd_dq<<<dim3((Lq + AB_TILE - 1) / AB_TILE, bh), AB_THREADS, ABQ_SMEM, st>>>(tmQ, tmDO, tmK, tmV, p);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

}  // namespace g3c

extern "C" int g3c_attn_bwd_sbhd(const void* q, const void* k, const void* v, const void* o, const void* dout,
                                 const float* lse, float* delta_ws, void* dq, void* dk, void* dv, int Lq, int Lk,
                                 int batch, int heads, int ldq, int ldk, int ldv, int ldo, int lddo, int lddq, int lddk,
                                 int lddv, float scale, void* stream) {
  return g3c::attn_bwd_sbhd(q, k, v, o, dout, lse, delta_ws, dq, dk, dv, Lq, Lk, batch, heads, ldq, ldk, ldv, ldo, lddo,
                            lddq, lddk, lddv, scale, (cudaStream_t)stream);
}
