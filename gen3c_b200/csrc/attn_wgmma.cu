// Path D — non-causal multi-head attention forward, head_dim 128, on the Hopper tensor cores (wgmma).
//   O = softmax(Q K^T * scale) V        (reference: cosmos_predict1/diffusion/module/attention.py
//   :282-297 `cal_attn` -> transformer_engine DotProductAttention(sbhd, no_mask, dropout 0);
//   self-attention Lq = Lk = 56 320, cross-attention Lk = 512; SURVEY.md §8a row D9)
//
// Layouts (all bf16, produced by the projection GEMMs of gemm_wgmma.cu):
//   Q  [Lq, heads*128]  token-major          K [Lk, heads*128] token-major
//   Vt [chunks][heads*128][chunk_len]        (V transposed, keys contiguous -> K-major B operand;
//                                             `chunks` = context-parallel ranks after the KV
//                                             all-gather, 1 otherwise)
//   O  [Lq, heads*128]
//   kVTokenMajor (g3c_attn_fwd_sbhd): V [Lk, heads*128] token-major like K, any Lk >= 1, heads = batch x heads of sbhd
//   kLse (g3c_attn_fwd_sbhd_lse, with kVTokenMajor): also lse [heads][Lq] f32 for the backward (attn_bwd_wgmma.cu)
//
// One CTA = ATT_ROWS_PER_CTA (128) query rows of one head, 384 threads (three warpgroups):
//   warpgroup 0     TMA producer: Q once, then K_j and V^T_j through two rings of ATT_STAGES 32 KB stages each (a K
//                   ring and a V ring with their own full / empty barriers: step j of a consumer reads K_j and V_{j-1})
//   warpgroups 1-2  consumers, 64 query rows each, software-pipelined with one S tile of lookahead:
//                     prologue  S_0 = Q K_0^T, softmax, pack P_0
//                     step j    [turn] issue S_j = Q K_j^T and O += P_{j-1} V_{j-1} [pass turn]; wait<1> (S_j done);
//                               2^(s - m) of S_j in place against the current m, no row max (exp_tile); warpgroup
//                               vote on the sum guard; in the rare case it fails, S_j again from K_j, wait<0> and the
//                               exact softmax_tile (row max, m moves); release K_j; wait<0> (P.V done, release
//                               V_{j-1}); rescale O if m moved; pack P_j (bf16 A fragments of the next P.V, from
//                               registers)
//                     epilogue  [turn] O += P_{n-1} V_{n-1} [pass turn]; wait<0>; normalise and store
//                   so the softmax of step j runs under this warpgroup's own P.V(j-1).  Between the two warpgroups a turn
//                   token (two mbarriers) alternates the MMA issue, so one warpgroup's softmax sits under the other's
//                   MMAs instead of both drifting into the softmax together.  Both warpgroups take n_kv + 1 turns,
//                   including one whose rows are all past Lq (it masks at the store).  The fallback's second S wgmma is
//                   issued outside the turn: it only costs overlap, no barrier waits on it.
// K_j is released after the guard decision (after the fallback's S on that path), not right after wait<1>: the fallback
// reads K_j again.  That does not delay the producer: its next load into K_j's stage comes after its load of
// V_{j+ATT_STAGES-1}, which waits for both consumers' release of V_{j-1}, and each consumer releases V_{j-1} after the
// softmax of step j, with or without the guard.  The same order is why the fallback's read of K_j could not be overwritten
// even by an early release; the release still comes after it, as the barrier's contract says.
// The protocol (rings, wgmma group waits, turn token) is modelled in tests/test_attn_pingpong_model_cpu.py, with the sum
// guard's fallback and K release in tests/test_attn_sum_guard_cpu.py.
#include <cmath>
#include <cstdlib>

#include "kernels.h"

namespace g3c {

constexpr int ATT_THREADS = 384;
constexpr int ATT_TILE = ATT_ROWS_PER_CTA;  // query rows per CTA, keys per KV tile, head dim
constexpr int ATT_HALF_BYTES = 128 * 128;   // one 64-column half of a 128x128 bf16 tile
constexpr int ATT_TILE_BYTES = 2 * ATT_HALF_BYTES;
// Depth of each of the K and V rings.  3 stages (224 KB with Q) also fit, but measured slower on an H100 SXM at 700 W
// (sustained 56 320 x 56 320 x 32 heads: 604 TFLOP/s against 613 with 2 stages).
constexpr int ATT_STAGES = 2;
constexpr int ATT_SMEM = ATT_TILE_BYTES + ATT_STAGES * 2 * ATT_TILE_BYTES + 256 + 1024;
static_assert(ATT_SMEM <= 227 * 1024, "attention: Q + K/V rings exceed the 227 KB of shared memory per block");
static_assert(1 + 4 * ATT_STAGES + 3 <= 256 / 8, "attention: barriers exceed their 256-byte area");
// The consumers' steady-state loop is unrolled by the ring depth, so every stage index and parity in it is a constant.
static_assert(ATT_STAGES == 2, "attention: the consumer loop is unrolled for a ring depth of 2");
// Lazy rescale (softmax_tile): the reference row max moves only when a row's tile max exceeds it by more than this many
// powers of two, so P <= 2^8 between moves.
constexpr float ATT_RESCALE_LOG2 = 8.0f;
// Sum guard of the steady-state tiles (exp_tile), G = 24: a tile exponentiated against the current reference is accepted
// when each thread's partial row sums over its 32 columns stay below 2^G.  Every accepted P is then < 2^24, a row's tile
// sum < 4 * 2^24 (four threads share a row) and l < n_kv * 2^26 (< 2^35 at the 440 tiles of Lk = 56 320; fp32 reaches
// 2^128), and |O| <= l max|v| stays finite for max|v| < 2^128 / (n_kv 2^26), 2^93 at 440 tiles (2^104 with the lazy
// rule alone).  A failing tile holds some P >= 2^G / 32 = 2^19, beyond ATT_RESCALE_LOG2, so its exact redo
// (softmax_tile) moves m; that needs G >= 14.  G also bounds how far m trails the row max (< 24 instead of <= 8): the
// fma argument of an exponential grows by that much, 2^-24 (|x - max x| + 24) of relative rounding, three orders of
// magnitude below bf16 P's 2^-8; scaling P by a power of two leaves its bf16 rounding as it was, so only the fractional
// part of m moves the roundings.  A fallback that moves m over a jump of more than 126 flushes earlier P of up to 2^G
// (not 2^8) to 0 with alpha: each such key then held less than 2^-100 of its row's weight, all of them less than 2^-85.
constexpr float ATT_GUARD = 16777216.0f;  // 2^G

struct AttnParams {
  int Lq, Lk, heads;
  int ldo;
  int vt_chunk_len;
  __nv_bfloat16* O;
  float scale_log2;             // softmax scale * log2(e)
  const uint32_t* chunk_flags;  // context-parallel gate (or NULL): chunk c readable once chunk_flags[c] >= flag_seq
  uint32_t flag_seq;
  int first_chunk;
  unsigned long long peer_timeout_ns;  // bound of the wait for a peer's chunk flag (and of this CTA's barrier waits
                                       // while such a wait may be pending): an inter-process dependency, not a protocol bug
  unsigned long long* wait_ns;         // optional profiling counter: ns spent polling chunk flags, summed over CTAs
  unsigned long long* trace;           // kTrace only: [3 roles][64 steps][8 slots] clock64 stamps of CTA (0,0), see
                                       // g3c_attn_set_trace in include/gen3c_b200.h
  float* lse;                          // kLse only: [heads][Lq] log-sum-exp of each query row, log2 units of s sl2
};

static unsigned long long* g_attn_trace = nullptr;

#define ATT_TR(role, slot)                                                                                  \
  do {                                                                                                      \
    if constexpr (kTrace) {                                                                                 \
      if (blockIdx.x == 0 && blockIdx.y == 0 && j < 64 && (threadIdx.x % 128) == 0)                         \
        p.trace[((role) * 64 + j) * 8 + (slot)] = clock64();                                                \
    }                                                                                                       \
  } while (0)

// S <- P = 2^(S sl2 - m) in place against the reference m of this thread's two rows; acc[h] += this thread's sum of
// its 32 P of row h.
__device__ __forceinline__ void exp_tile(float (&s)[64], const float (&m_ref)[2], float (&acc)[2], float sl2) {
  const float nm0 = -m_ref[0], nm1 = -m_ref[1];
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    s[4 * i] = ex2_approx(fmaf(s[4 * i], sl2, nm0));
    s[4 * i + 1] = ex2_approx(fmaf(s[4 * i + 1], sl2, nm0));
    s[4 * i + 2] = ex2_approx(fmaf(s[4 * i + 2], sl2, nm1));
    s[4 * i + 3] = ex2_approx(fmaf(s[4 * i + 3], sl2, nm1));
    acc[0] += s[4 * i] + s[4 * i + 1];
    acc[1] += s[4 * i + 2] + s[4 * i + 3];
  }
}

// Online softmax of one S tile (this thread's two rows), with a lazy reference.  The row max of the tile is exact; the
// reference m the exponentials are taken against only moves when some row of the warp's 16 exceeds its m by more than
// ATT_RESCALE_LOG2 (log2 units).  Then m <- max(m, row max), alpha = 2^(m_old - m_new), l <- l alpha, and the function
// returns true: the caller rescales O by alpha.  Otherwise (most tiles once the first few have set m) it returns false,
// and P = 2^(S sl2 - m) <= 2^ATT_RESCALE_LOG2 against the stale m, which bf16 P and the fp32 row sums hold with room to
// spare.  The first tile always moves m (m = -inf).  The decision is a warp vote, so the branch on it stays uniform.
// S <- P in place, l <- l + row sums of P.
__device__ __forceinline__ bool softmax_tile(float (&s)[64], float (&m_ref)[2], float (&l_run)[2], float (&alpha)[2],
                                             float sl2) {
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    mx[0] = fmaxf(mx[0], fmaxf(s[4 * i], s[4 * i + 1]));
    mx[1] = fmaxf(mx[1], fmaxf(s[4 * i + 2], s[4 * i + 3]));
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    mx[h] *= sl2;
  }
  const bool keep = __all_sync(0xffffffffu, mx[0] - m_ref[0] <= ATT_RESCALE_LOG2 && mx[1] - m_ref[1] <= ATT_RESCALE_LOG2);
  if (!keep) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float nm = fmaxf(m_ref[h], mx[h]);
      alpha[h] = ex2_approx(m_ref[h] - nm);  // 0 on the first tile (m = -inf)
      m_ref[h] = nm;
      l_run[h] *= alpha[h];
    }
  }
  exp_tile(s, m_ref, l_run, sl2);
  return !keep;
}

// The wgmma shared-memory descriptors of this kernel, split in two 32-bit words: the low word carries the start address
// (and the LBO of the MN-major V tile), the high word is the same for all of them (SBO 1024 B, SWIZZLE_128B; see
// make_sdesc_sw128).  A k-step offset is added to the low word alone: the 14-bit address field of a shared-memory
// address plus an offset inside its tile never carries out.  The loop-invariant low words are computed once per CTA.
constexpr uint32_t ATT_SDESC_HI = (1024u >> 4) | (1u << 30);
__device__ __forceinline__ uint64_t sdesc_at(uint32_t lo, uint32_t bytes) {
  return (static_cast<uint64_t>(ATT_SDESC_HI) << 32) | (lo + (bytes >> 4));
}

// S = Q K^T of one KV tile: 8 k-steps over the head dimension, A (Q rows of this warpgroup) and B (K tile) in shared memory
__device__ __forceinline__ void issue_s(float (&s)[64], uint32_t dq, uint32_t dk) {
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {  // head dimensions 16 kk .. 16 kk + 15
    const uint32_t off = (kk >> 2) * ATT_HALF_BYTES + (kk & 3) * 32;
    wgmma_ss_n128(s, sdesc_at(dq, off), sdesc_at(dk, off), kk > 0 ? 1u : 0u);
  }
}

// O += P V of one KV tile: P from registers (bf16 A fragments), V in shared memory.  V^T tile (keys contiguous): K-major
// B.  Token-major V tile (kVTokenMajor; head dims contiguous, loaded like K): MN-major B whose two 64-dim halves are
// ATT_HALF_BYTES apart (LBO, in `dv`), and k-step kk starts 16 keys of 128-byte rows into each half.
template <bool kVTokenMajor>
__device__ __forceinline__ void issue_pv(float (&o)[64], const uint32_t (&pa)[32], uint32_t dv) {
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {  // keys 16 kk .. 16 kk + 15 = accumulator columns of S
    const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
    if constexpr (kVTokenMajor)
      wgmma_rs_n128_tb(o, a, sdesc_at(dv, kk * 16 * 128));
    else
      wgmma_rs_n128(o, a, sdesc_at(dv, (kk >> 2) * ATT_HALF_BYTES + (kk & 3) * 32));
  }
}

// Last KV tile when Lk % 128 != 0: the TMA zero-filled the K rows past Lk, whose scores (0) would still enter the
// softmax.  Columns >= `valid` (keys of this tile below Lk, 1..128) are set to -inf before the softmax, so their
// exponentials are 0.
__device__ __forceinline__ void mask_key_tail(float (&s)[64], int valid, uint32_t lane) {
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int col = 8 * i + 2 * (int)(lane % 4);
    if (col >= valid) s[4 * i] = s[4 * i + 2] = -INFINITY;
    if (col + 1 >= valid) s[4 * i + 1] = s[4 * i + 3] = -INFINITY;
  }
}

// P as bf16 pairs from the exponentiated S: pa[2i] = row a, pa[2i + 1] = row a + 8, keys 8i + 2 (lane % 4) + {0, 1}
__device__ __forceinline__ void pack_p(uint32_t (&pa)[32], const float (&s)[64]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    pa[2 * i] = pack_bf16x2(s[4 * i], s[4 * i + 1]);
    pa[2 * i + 1] = pack_bf16x2(s[4 * i + 2], s[4 * i + 3]);
  }
}

// kVTokenMajor: V is [Lk, heads*128] like K (instead of the chunked V^T), any Lk >= 1 (the last KV tile is partial and
// masked), no context-parallel gate.  kLse (with kVTokenMajor, for the backward of attn_bwd_wgmma.cu): also store
// lse = m + log2(l) of each query row, from the final reference m and the quad-reduced l of the normalisation, so
// 2^(s sl2 - lse) is the row's softmax whatever m the lazy rescale or the sum guard left.
template <bool kTrace, bool kVTokenMajor = false, bool kLse = false>
__global__ void __launch_bounds__(ATT_THREADS, 1)
    k_attn_fwd(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
               const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_q = smem;
  uint8_t* smem_k = smem + ATT_TILE_BYTES;                          // [ATT_STAGES] K tiles
  uint8_t* smem_v = smem_k + ATT_STAGES * ATT_TILE_BYTES;            // [ATT_STAGES] V^T tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_v + ATT_STAGES * ATT_TILE_BYTES);
  uint64_t* q_full = bars;                   // [1]
  uint64_t* k_full = bars + 1;               // [ATT_STAGES]
  uint64_t* v_full = k_full + ATT_STAGES;    // [ATT_STAGES]
  uint64_t* k_empty = v_full + ATT_STAGES;   // [ATT_STAGES]
  uint64_t* v_empty = k_empty + ATT_STAGES;  // [ATT_STAGES]
  uint64_t* turn = v_empty + ATT_STAGES;     // [2]: phase t of turn[c] completes when consumer c may take its turn t
  uint64_t* done = turn + 2;                 // [1]: both consumer warpgroups finished (their waits exit, not trap)

  const uint32_t wg = threadIdx.x / 128;
  const uint32_t tid = threadIdx.x % 128;
  const int head = blockIdx.y;
  const int q0 = blockIdx.x * ATT_TILE;
  const int n_kv = kVTokenMajor ? (p.Lk + ATT_TILE - 1) / ATT_TILE : p.Lk / ATT_TILE;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < ATT_STAGES; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&k_empty[i], 2);  // one arrive per consumer warpgroup
      mbar_init(&v_empty[i], 2);
    }
    for (int c = 0; c < 2; ++c) mbar_init(&turn[c], 4);  // one arrive per warp of the other consumer warpgroup
    for (int w = 0; w < 4; ++w) mbar_arrive(&turn[0]);   // consumer 0 holds the first turn
    mbar_init(done, 2);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===== TMA producer =====
    setmaxnreg_dec<24>();
    if (tid == 0) {
      mbar_expect_tx(q_full, ATT_TILE_BYTES);
      for (int h = 0; h < 2; ++h) tma_load_2d(smem_q + h * ATT_HALF_BYTES, &tmQ, q_full, head * 128 + h * 64, q0);
      const int tiles_per_chunk = p.vt_chunk_len / ATT_TILE;
      const int n_chunks = p.Lk / p.vt_chunk_len;
      uint32_t stage = 0, phase = 0;
      for (int j = 0; j < n_kv; ++j) {
        int chunk = 0, within = j;  // token-major V: one chunk of all Lk keys
        if constexpr (!kVTokenMajor) {
          // KV tiles are visited chunk by chunk starting with `first_chunk` (the local one under context
          // parallelism); a remote chunk is only touched after its producer rank has published it.
          chunk = p.first_chunk + j / tiles_per_chunk;
          if (chunk >= n_chunks) chunk -= n_chunks;
          within = j % tiles_per_chunk;
          if (p.chunk_flags && within == 0 && chunk != p.first_chunk) {  // the local chunk is ordered by the stream
            uint32_t v, spins = 0;
            uint64_t t0 = 0;
            for (;;) {
              asm volatile("ld.acquire.sys.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p.chunk_flags + chunk) : "memory");
              if ((int)(v - p.flag_seq) >= 0) break;
              if (t0 == 0) t0 = global_timer_ns();
              if ((++spins & 0x3FFu) == 0 && global_timer_ns() - t0 > p.peer_timeout_ns) asm volatile("trap;\n");
            }
            if (t0 != 0 && p.wait_ns) atomicAdd(p.wait_ns, (unsigned long long)(global_timer_ns() - t0));
            asm volatile("fence.proxy.async.global;\n" ::: "memory");  // peer-written data is read by the TMA next
          }
        }
        const int kv0 = chunk * p.vt_chunk_len + within * ATT_TILE;
        mbar_wait_ns(&k_empty[stage], phase ^ 1, p.peer_timeout_ns);
        mbar_expect_tx(&k_full[stage], ATT_TILE_BYTES);
        for (int h = 0; h < 2; ++h)  // the two 64-dim halves of 128 keys
          tma_load_2d(smem_k + stage * ATT_TILE_BYTES + h * ATT_HALF_BYTES, &tmK, &k_full[stage], head * 128 + h * 64,
                      kv0);
        mbar_wait_ns(&v_empty[stage], phase ^ 1, p.peer_timeout_ns);
        mbar_expect_tx(&v_full[stage], ATT_TILE_BYTES);
        for (int h = 0; h < 2; ++h) {
          if constexpr (kVTokenMajor)  // as K: the two 64-dim halves of 128 keys
            tma_load_2d(smem_v + stage * ATT_TILE_BYTES + h * ATT_HALF_BYTES, &tmV, &v_full[stage],
                        head * 128 + h * 64, kv0);
          else  // the two 64-key halves of 128 head dimensions
            tma_load_3d(smem_v + stage * ATT_TILE_BYTES + h * ATT_HALF_BYTES, &tmV, &v_full[stage],
                        within * ATT_TILE + h * 64, head * 128, chunk);
        }
        if (++stage == ATT_STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      // a consumer whose barrier wait timed out has exited without arriving: trap here, within the bound
      mbar_wait_ns(done, 0, p.peer_timeout_ns);
    }
  } else {
    // ===== consumers: warpgroup c owns query rows [64c, 64c + 64) of the tile =====
    setmaxnreg_inc<240>();
    const uint32_t c = __shfl_sync(0xffffffffu, wg - 1, 0);  // warp-uniform for the compiler: descriptors and barrier
                                                               // addresses derived from it stay in uniform registers
    const uint32_t warp = tid / 32, lane = tid % 32;
    const unsigned long long tmo = p.peer_timeout_ns;
    // accumulator layout (wgmma m64n128k16, f32), i in [0, 16): acc[4i + {0,1}] = row 16 warp + lane/4, columns 8i + 2 (lane%4) + {0,1};
    // acc[4i + {2,3}] = the same columns eight rows further down
    float o[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.f;
    float s[64];      // S_j, then 2^(S_j - m) in place
    uint32_t pa[32];  // P_{j-1}: the A operand of the P.V in flight during the softmax of step j
    float m_ref[2] = {-INFINITY, -INFINITY};  // reference row max (log2 units) of the two rows of this thread
    float l_run[2] = {0.f, 0.f};              // this thread's partial row sums (quad-reduced at the end)
    float alpha[2];
    const float sl2 = p.scale_log2;
    // descriptor low words (sdesc_at): this warpgroup's Q rows, and the K and V tile of each ring stage
    const uint32_t dq = (uint32_t)make_sdesc_sw128(smem_u32(smem_q + c * 64 * 128));
    uint32_t dk[ATT_STAGES], dv[ATT_STAGES];
#pragma unroll
    for (int st = 0; st < ATT_STAGES; ++st) {
      dk[st] = (uint32_t)make_sdesc_sw128(smem_u32(smem_k + st * ATT_TILE_BYTES));
      dv[st] = (uint32_t)(kVTokenMajor ? make_sdesc_sw128_mn(smem_u32(smem_v + st * ATT_TILE_BYTES), ATT_HALF_BYTES)
                                       : make_sdesc_sw128(smem_u32(smem_v + st * ATT_TILE_BYTES)));
    }
    // Ring positions as functions of the KV tile: K_j sits in stage j % 2 at parity (j / 2) % 2, V_{j-1} in stage
    // (j - 1) % 2 at parity ((j - 1) / 2) % 2, and this warpgroup's turn t waits for parity t % 2 of turn[c] (turn j is
    // taken at step j).
    int j = 0;
    // ---- prologue: S_0, softmax, P_0 ----
    mbar_wait_ns_or_exit(q_full, 0, tmo);
    mbar_wait_ns_or_exit(&k_full[0], 0, tmo);
    mbar_wait_ns_or_exit(&turn[c], 0, tmo);
    ATT_TR(1 + c, 0);
    wgmma_fence();
    issue_s(s, dq, dk[0]);
    wgmma_commit();
    if (lane == 0) mbar_arrive(&turn[c ^ 1]);
    ATT_TR(1 + c, 1);
    wgmma_wait<0>();
    fence_regs(s);
    if (tid == 0) mbar_arrive(&k_empty[0]);
    ATT_TR(1 + c, 2);
    if constexpr (kVTokenMajor) {
      if (n_kv == 1) mask_key_tail(s, p.Lk, lane);
    }
    softmax_tile(s, m_ref, l_run, alpha, sl2);  // sets m: O and l are still 0
    pack_p(pa, s);
    ATT_TR(1 + c, 3);
    // ---- step j: S_j is computed while P.V(j-1) runs; the softmax of S_j runs under P.V(j-1).  K_j in stage kst at
    // parity kpar, V_{j-1} in stage vst at parity vpar, turn parity j % 2; keys of the tile from `valid` on are masked
    // (valid < ATT_TILE only in the last tile of a ragged token-major Lk) ----
    auto step = [&](int kst, int vst, uint32_t kpar, uint32_t vpar, int valid) {
      mbar_wait_ns_or_exit(&k_full[kst], kpar, tmo);
      mbar_wait_ns_or_exit(&v_full[vst], vpar, tmo);
      mbar_wait_ns_or_exit(&turn[c], (uint32_t)j & 1u, tmo);
      ATT_TR(1 + c, 0);
      wgmma_fence();
      issue_s(s, dq, kst ? dk[1] : dk[0]);
      wgmma_commit();
      issue_pv<kVTokenMajor>(o, pa, vst ? dv[1] : dv[0]);
      wgmma_commit();
      if (lane == 0) mbar_arrive(&turn[c ^ 1]);
      ATT_TR(1 + c, 1);
      wgmma_wait<1>();  // S_j complete; P.V(j-1) may still run
      fence_regs(s);
      ATT_TR(1 + c, 2);
      if (valid < ATT_TILE) mask_key_tail(s, valid, lane);
      // P_{j-1} (pa) and O are still read / written by the P.V in flight
      // sum guard: this thread's partial row sums t against the current m, accepted when every thread of the
      // warpgroup has both below ATT_GUARD (a NaN or inf fails the comparison); otherwise redone with softmax_tile
      float t[2] = {0.f, 0.f};
      exp_tile(s, m_ref, t, sl2);
      const bool redo = bar_red_or(1 + c, 128, !(t[0] < ATT_GUARD && t[1] < ATT_GUARD));
      if (redo) {  // warpgroup-uniform: S_j again from K_j, still held, then the exact softmax
        wgmma_fence();
        issue_s(s, dq, kst ? dk[1] : dk[0]);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s);
      }
      if (tid == 0) mbar_arrive(&k_empty[kst]);
      bool rescale = false;
      if (redo) {
        if (valid < ATT_TILE) mask_key_tail(s, valid, lane);
        rescale = softmax_tile(s, m_ref, l_run, alpha, sl2);
      } else {
        l_run[0] += t[0];
        l_run[1] += t[1];
      }
      ATT_TR(1 + c, 3);
      wgmma_wait<0>();
      fence_regs(o);
      fence_regs(pa);  // pa stays allocated (not reused for the exponentials above) until the P.V has read it
      if (tid == 0) mbar_arrive(&v_empty[vst]);
      ATT_TR(1 + c, 4);
      if (rescale) {  // warp-uniform
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          o[4 * i] *= alpha[0];
          o[4 * i + 1] *= alpha[0];
          o[4 * i + 2] *= alpha[1];
          o[4 * i + 3] *= alpha[1];
        }
      }
      pack_p(pa, s);
    };
    // ---- steady state, two steps per iteration: j = 2u + 1 (K stage 1, V stage 0) and j = 2u + 2 (K stage 0, V
    // stage 1); `ph` = u % 2 ----
    const int j_end = kVTokenMajor ? n_kv - 1 : n_kv;  // the token-major build peels the last tile off (masked)
    uint32_t ph = 0;
    for (j = 1; j < j_end; ++j) {
      step(1, 0, ph, ph, ATT_TILE);
      if (++j == j_end) break;
      step(0, 1, ph ^ 1u, ph, ATT_TILE);
      ph ^= 1u;
    }
    if constexpr (kVTokenMajor) {
      // ---- the last KV tile: the same step with the keys past Lk masked before the softmax ----
      if (n_kv > 1) {
        j = n_kv - 1;
        step(j & 1, (j - 1) & 1, ((uint32_t)j >> 1) & 1u, ((uint32_t)(j - 1) >> 1) & 1u, p.Lk - j * ATT_TILE);
      }
      j = n_kv;
    }
    // ---- epilogue: O += P_{n-1} V_{n-1} (the last turn: both warpgroups take n_kv + 1 turns) ----
    const int vst = (n_kv - 1) & 1;
    mbar_wait_ns_or_exit(&v_full[vst], ((uint32_t)(n_kv - 1) >> 1) & 1u, tmo);
    mbar_wait_ns_or_exit(&turn[c], (uint32_t)n_kv & 1u, tmo);
    ATT_TR(1 + c, 0);
    wgmma_fence();
    issue_pv<kVTokenMajor>(o, pa, vst ? dv[1] : dv[0]);
    wgmma_commit();
    if (lane == 0) mbar_arrive(&turn[c ^ 1]);
    ATT_TR(1 + c, 1);
    wgmma_wait<0>();
    fence_regs(o);
    fence_regs(pa);
    if (tid == 0) mbar_arrive(&v_empty[vst]);
    ATT_TR(1 + c, 4);
    // ---- normalise and store ----
    float inv[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float l = l_run[h];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      inv[h] = 1.0f / l;
      if constexpr (kLse) {
        const int row = q0 + (int)(c * 64 + warp * 16 + lane / 4) + 8 * h;
        if (lane % 4 == 0 && row < p.Lq) p.lse[(size_t)head * p.Lq + row] = m_ref[h] + log2f(l);
      }
    }
    const int row_a = q0 + (int)(c * 64 + warp * 16 + lane / 4);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row_a + 8 * h;
      if (row >= p.Lq) continue;
      __nv_bfloat16* dst = p.O + (size_t)row * p.ldo + head * 128 + 2 * (lane % 4);
#pragma unroll
      for (int i = 0; i < 16; ++i)
        *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_bf16x2(o[4 * i + 2 * h] * inv[h], o[4 * i + 2 * h + 1] * inv[h]);
    }
    if (tid == 0) mbar_arrive(done);
  }
}

// TMA map of a token-major operand [rows, heads*128] (leading dimension ld): boxes of 64 head dims x 128 tokens
static int make_tmap_tokens(CUtensorMap* m, const void* base, int rows, int heads, int ld) {
  uint64_t dims[2] = {(uint64_t)heads * 128, (uint64_t)rows}, str[1] = {(uint64_t)ld * 2};
  uint32_t box[2] = {64, 128};
  return make_tmap_bf16_sw128(m, base, 2, dims, str, box);
}

// scale = ln 2 declares that Q already carries softmax scale * log2(e): S is then in log2 units
float attn_scale_log2(float scale) {
  const float s = scale * 1.4426950408889634f;
  return fabsf(s - 1.0f) < 1e-6f ? 1.0f : s;
}

int attn_fwd(const void* q, const void* k, const void* vt, void* o, int Lq, int Lk, int heads,
             int ldq, int ldk, int ldo, int vt_chunk_len, float scale, cudaStream_t st, const ChunkGate* gate) {
  G3C_REQUIRE(q && k && vt && o, "attn: null operand");
  G3C_REQUIRE(Lq > 0 && Lk > 0 && heads > 0, "attn: bad sizes");
  G3C_REQUIRE(Lk % ATT_TILE == 0, "attn: Lk=%d must be a multiple of 128", Lk);
  if (vt_chunk_len <= 0) vt_chunk_len = Lk;
  G3C_REQUIRE(Lk % vt_chunk_len == 0 && vt_chunk_len % ATT_TILE == 0,
              "attn: vt_chunk_len=%d must divide Lk=%d and be a multiple of 128", vt_chunk_len, Lk);
  G3C_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldo % 8 == 0 && ldq >= heads * 128 &&
                  ldk >= heads * 128 && ldo >= heads * 128,
              "attn: leading dimensions must be >= heads*128 and multiples of 8");
  G3C_REQUIRE((reinterpret_cast<uintptr_t>(o) & 15) == 0, "attn: O must be 16-byte aligned");
  CUtensorMap tmQ, tmK, tmV;
  int rc = make_tmap_tokens(&tmQ, q, Lq, heads, ldq);
  if (rc) return rc;
  rc = make_tmap_tokens(&tmK, k, Lk, heads, ldk);
  if (rc) return rc;
  {
    const int chunks = Lk / vt_chunk_len;
    uint64_t dims[3] = {(uint64_t)vt_chunk_len, (uint64_t)heads * 128, (uint64_t)chunks};
    uint64_t str[2] = {(uint64_t)vt_chunk_len * 2, (uint64_t)vt_chunk_len * 2 * heads * 128};
    uint32_t box[3] = {64, 128, 1};
    rc = make_tmap_bf16_sw128(&tmV, vt, 3, dims, str, box);
    if (rc) return rc;
  }
  static bool configured = false;
  if (!configured) {
    G3C_CUDA(cudaFuncSetAttribute(k_attn_fwd<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM));
    G3C_CUDA(cudaFuncSetAttribute(k_attn_fwd<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM));
    configured = true;
  }
  AttnParams p;
  p.Lq = Lq;
  p.Lk = Lk;
  p.heads = heads;
  p.ldo = ldo;
  p.vt_chunk_len = vt_chunk_len;
  p.O = reinterpret_cast<__nv_bfloat16*>(o);
  p.scale_log2 = attn_scale_log2(scale);
  p.chunk_flags = gate ? gate->flags : nullptr;
  p.peer_timeout_ns = gate ? peer_timeout_ns() : G3C_MBAR_TIMEOUT_NS;
  p.wait_ns = gate ? gate->wait_ns : nullptr;
  p.flag_seq = gate ? gate->seq : 0;
  p.first_chunk = gate ? gate->first : 0;
  p.trace = g_attn_trace;
  G3C_REQUIRE(p.first_chunk >= 0 && p.first_chunk < Lk / vt_chunk_len, "attn: first chunk %d out of range", p.first_chunk);
  dim3 grid((Lq + ATT_TILE - 1) / ATT_TILE, heads);
  if (g_attn_trace) k_attn_fwd<true><<<grid, ATT_THREADS, ATT_SMEM, st>>>(tmQ, tmK, tmV, p);
  else k_attn_fwd<false><<<grid, ATT_THREADS, ATT_SMEM, st>>>(tmQ, tmK, tmV, p);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

// q, k, v, o: `batch` x `heads` heads of 128 per token (the rows of contiguous sbhd [s, b, h, 128] tensors viewed as
// [s, b*h*128]), so the batch is b*h heads of one launch.  V token-major like K; any Lq, Lk >= 1.  lse (or NULL):
// f32 [batch*heads][Lq], written by the kLse build of the same kernel.
int attn_fwd_sbhd(const void* q, const void* k, const void* v, void* o, float* lse, int Lq, int Lk, int batch,
                  int heads, int ldq, int ldk, int ldv, int ldo, float scale, cudaStream_t st) {
  G3C_REQUIRE(q && k && v && o, "attn_sbhd: null operand");
  G3C_REQUIRE(Lq > 0 && Lk > 0, "attn_sbhd: Lq=%d and Lk=%d must be >= 1", Lq, Lk);
  G3C_REQUIRE(batch > 0 && heads > 0 && (long long)batch * heads <= 65535,
              "attn_sbhd: batch=%d x heads=%d must be in [1, 65535]", batch, heads);
  const int bh = batch * heads;
  G3C_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && ldq >= bh * 128 && ldk >= bh * 128 &&
                  ldv >= bh * 128 && ldo >= bh * 128,
              "attn_sbhd: leading dimensions (%d, %d, %d, %d) must be >= batch*heads*128 = %d and multiples of 8", ldq,
              ldk, ldv, ldo, bh * 128);
  G3C_REQUIRE(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
                reinterpret_cast<uintptr_t>(o)) & 15) == 0,
              "attn_sbhd: q, k, v and o must be 16-byte aligned");
  G3C_REQUIRE((reinterpret_cast<uintptr_t>(lse) & 3) == 0, "attn_sbhd: lse must be 4-byte aligned");
  CUtensorMap tmQ, tmK, tmV;
  int rc = make_tmap_tokens(&tmQ, q, Lq, bh, ldq);
  if (rc) return rc;
  rc = make_tmap_tokens(&tmK, k, Lk, bh, ldk);
  if (rc) return rc;
  rc = make_tmap_tokens(&tmV, v, Lk, bh, ldv);
  if (rc) return rc;
  static bool configured = false;
  if (!configured) {
    G3C_CUDA(cudaFuncSetAttribute(k_attn_fwd<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM));
    G3C_CUDA(cudaFuncSetAttribute(k_attn_fwd<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  ATT_SMEM));
    configured = true;
  }
  AttnParams p = {};
  p.Lq = Lq;
  p.Lk = Lk;
  p.heads = bh;
  p.ldo = ldo;
  p.vt_chunk_len = Lk;
  p.O = reinterpret_cast<__nv_bfloat16*>(o);
  p.scale_log2 = attn_scale_log2(scale);
  p.peer_timeout_ns = G3C_MBAR_TIMEOUT_NS;
  p.lse = lse;
  dim3 grid((Lq + ATT_TILE - 1) / ATT_TILE, bh);
  if (lse) k_attn_fwd<false, true, true><<<grid, ATT_THREADS, ATT_SMEM, st>>>(tmQ, tmK, tmV, p);
  else k_attn_fwd<false, true><<<grid, ATT_THREADS, ATT_SMEM, st>>>(tmQ, tmK, tmV, p);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

}  // namespace g3c

extern "C" int g3c_attn_set_trace(unsigned long long* device_buffer) {
  g3c::g_attn_trace = device_buffer;
  return G3C_OK;
}

extern "C" int g3c_attn_fwd(const void* q, const void* k, const void* vt, void* o, int Lq, int Lk,
                            int heads, int ldq, int ldk, int ldo, int vt_chunk_len, float scale,
                            void* stream) {
  return g3c::attn_fwd(q, k, vt, o, Lq, Lk, heads, ldq, ldk, ldo, vt_chunk_len, scale,
                       (cudaStream_t)stream, nullptr);
}

extern "C" int g3c_attn_fwd_gated(const void* q, const void* k, const void* vt, void* o, int Lq, int Lk, int heads,
                                  int ldq, int ldk, int ldo, int vt_chunk_len, float scale, const uint32_t* flags,
                                  uint32_t seq, int first, unsigned long long* wait_ns, void* stream) {
  g3c::ChunkGate gate;
  gate.flags = flags;
  gate.seq = seq;
  gate.first = first;
  gate.wait_ns = wait_ns;
  return g3c::attn_fwd(q, k, vt, o, Lq, Lk, heads, ldq, ldk, ldo, vt_chunk_len, scale, (cudaStream_t)stream, &gate);
}

extern "C" int g3c_attn_fwd_sbhd(const void* q, const void* k, const void* v, void* o, int Lq, int Lk, int batch,
                                 int heads, int ldq, int ldk, int ldv, int ldo, float scale, void* stream) {
  return g3c::attn_fwd_sbhd(q, k, v, o, nullptr, Lq, Lk, batch, heads, ldq, ldk, ldv, ldo, scale,
                            (cudaStream_t)stream);
}

extern "C" int g3c_attn_fwd_sbhd_lse(const void* q, const void* k, const void* v, void* o, float* lse, int Lq, int Lk,
                                     int batch, int heads, int ldq, int ldk, int ldv, int ldo, float scale,
                                     void* stream) {
  if (!lse) {
    g3c::set_error("attn_sbhd_lse: null lse");
    return G3C_EINVAL;
  }
  return g3c::attn_fwd_sbhd(q, k, v, o, lse, Lq, Lk, batch, heads, ldq, ldk, ldv, ldo, scale, (cudaStream_t)stream);
}
