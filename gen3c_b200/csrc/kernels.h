// Internal host-side launchers shared between translation units of libgen3c_b200.so.
#pragma once
#include "common.cuh"

namespace g3c {

// Optional fused tail of a projection: per-head (128 columns) RMSNorm with gain `gamma` [128] and, when `cs` is given,
// rotate-half RoPE with the cos|sin table `cs` [M][128] — applied to the fp32 accumulators in the GEMM epilogue.
struct NormRope {
  const float* gamma = nullptr;
  const float* cs = nullptr;
  float eps = 1e-6f;
};

int gemm_bf16(const void* A, const void* B, void* D, int M, int N, int K, int lda, int ldb, int ldd,
              int epilogue, const float* gate, int block_n, cudaStream_t st, const NormRope* norm_rope = nullptr);
// Same GEMM on e4m3 row-quantised operands: D = (A8 . B8^T) * scale_a[m] * scale_b[n], then the epilogue.
int gemm_fp8(const void* A8, const float* scale_a, const void* B8, const float* scale_b, void* D, int M, int N, int K,
             int lda, int ldb, int ldd, int epilogue, const float* gate, int block_n, cudaStream_t st,
             const NormRope* norm_rope = nullptr);
// Row quantiser: bf16 x [R, C] (ld) -> e4m3 codes [R, C] (ldq) + fp32 row scales [R] (amax / 448; 1 for a zero row).
int quant_rows_e4m3(const __nv_bfloat16* x, int ld, int R, int C, uint8_t* codes, int ldq, float* scales,
                    cudaStream_t st);
// Chunk-ordered attention for context parallelism: KV chunk c (= source rank) may only be read once
// flags[c] >= seq (written with system scope by rank c after its K / V^T slices have landed here); chunks are
// visited starting at `first` so that the local chunk overlaps the arrival of the remote ones.
struct ChunkGate {
  const uint32_t* flags = nullptr;
  uint32_t seq = 0;
  int first = 0;
  unsigned long long* wait_ns = nullptr;  // optional: += ns each CTA's loader spent polling flags (profiling)
};
unsigned long long peer_timeout_ns();  // bound of inter-process waits (G3C_PEER_TIMEOUT_S, default 600 s)
// attn_fwd launches one CTA per ATT_ROWS_PER_CTA query rows of one head (also its KV tile width: Lk % 128 == 0)
constexpr int ATT_ROWS_PER_CTA = 128;
int attn_fwd(const void* q, const void* k, const void* vt, void* o, int Lq, int Lk, int heads,
             int ldq, int ldk, int ldo, int vt_chunk_len, float scale, cudaStream_t st,
             const ChunkGate* gate = nullptr);
// log2-unit score scale of the attention kernels: fp32(scale * log2(e)), exactly 1 within 1e-6 of it (scale = ln 2
// declares that Q already carries softmax scale * log2(e))
float attn_scale_log2(float scale);

struct PatchSrc {
  const __nv_bfloat16* ptr[4];
  int nch[4];
  int per_frame[4];  // 1: [C,T,H2,W2], 0: [C,H2,W2] broadcast over T (padding mask)
};

int ln_modulate(float* x, const __nv_bfloat16* pos, const float* shift, const float* scale,
                __nv_bfloat16* y, int L, int D, float eps, cudaStream_t st);
// Same, the modulated row quantised straight from fp32: e4m3 codes y8 [L, D] + row scales y_scale [L].
int ln_modulate_e4m3(float* x, const __nv_bfloat16* pos, const float* shift, const float* scale, uint8_t* y8,
                     float* y_scale, int L, int D, float eps, cudaStream_t st);
int rmsnorm_rope(__nv_bfloat16* qk, int ld, int L, int heads, const float* gamma, const float* cs,
                 float eps, cudaStream_t st);
int gemv(const __nv_bfloat16* W, const float* x, const float* add, float* y, int N, int K, int pre,
         int round_out, cudaStream_t st);
int patchify(const PatchSrc& src, int T, int Hp, int Wp, int Kpad, __nv_bfloat16* out, cudaStream_t st);
int unpatchify(const float* y, int ldy, int T, int Hp, int Wp, int C, __nv_bfloat16* out, cudaStream_t st);
int timestep_embed(float t, int D, const __nv_bfloat16* gamma, float eps, float* s, float* emb,
                   cudaStream_t st);
int abs_pos(const __nv_bfloat16* pt, const __nv_bfloat16* ph, const __nv_bfloat16* pw, int t0, int T,
            int Hp, int Wp, int D, __nv_bfloat16* out, cudaStream_t st);
int rope_table(const float* freqs, int nt, int nh, int nw, int t0, float t_scale, int T, int Hp, int Wp,
               float* cs, cudaStream_t st);
int bf16_to_f32(const __nv_bfloat16* in, float* out, size_t n, cudaStream_t st, float scale = 1.0f);
int sampler_pre(const __nv_bfloat16* xt, const __nv_bfloat16* gt, const float* noise, const float* ind_t,
                int C, int T, size_t plane, float sigma, float sigma_aug, float sd,
                __nv_bfloat16* xtilde, __nv_bfloat16* xin, cudaStream_t st);
int sampler_post(const __nv_bfloat16* xtilde, const __nv_bfloat16* oc, const __nv_bfloat16* ou,
                 const __nv_bfloat16* gt, const float* ind_t, int C, int T, size_t plane, float guidance,
                 float sigma, float sigma_next, float sigma_aug, float sd, __nv_bfloat16* xnext,
                 __nv_bfloat16* net_out, cudaStream_t st);

}  // namespace g3c
