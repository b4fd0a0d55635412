// Path D — the DiT forward and the denoise-step loop body as a native engine.
//
// Mirrors VideoExtendGeneralDIT.forward (reference: cosmos_predict1/diffusion/networks/
// general_dit_video_conditioned.py:58-217, general_dit.py:272-358,439-522, module/blocks.py:419-475,
// 537-558) for B = 1 and the FA-CA-MLP block layout, and the loop body of
// DiffusionV2WModel.generate_samples_from_batch (model/model_v2w.py:130-149).
//
// Data layout in HBM (L = T_local*Hp*Wp tokens of this rank, D = model_channels):
//   x      f32  [L, D]        residual stream (kept fp32; the reference keeps bf16)
//   xn     bf16 [L, D]        LN-modulated activations = GEMM A operand
//   q      bf16 [L, D]        k_all bf16 [cp*L, D]      vt_all bf16 [cp][D][L]  (V transposed)
//   att    bf16 [L, D]        hid  bf16 [L, ffn]
//   pos    bf16 [L, D]        per-block absolute position embedding (precomputed per shape)
//   rope   f32  [L, 128]      cos|sin table (precomputed per shape)
// Context parallelism: tokens are split contiguously along latent T (module/parallel.py:44-53), and every
// self-attention layer gathers the K and V^T of all ranks (same result as the reference's TE ring:
// general_dit.py:524-543).  Default (p2p): each rank projects its K / V^T slice into its slot of a peer-mapped region,
// the copy engines push the slice to every peer and raise an arrival flag there, and attention reads each remote chunk
// once its flag is up.  NCCL mode (G3C_CP_MODE=nccl): one in-place ncclAllGather of K and one of V^T per layer.
#include <dlfcn.h>

#include <array>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "kernels.h"

namespace g3c {

// ---- NCCL, loaded at run time (the process normally already holds torch's libnccl.so.2) --------
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
struct NcclApi {
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool ok = false;
};
static NcclApi& nccl() {
  static NcclApi api;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (h) {
      api.GetUniqueId = (int (*)(ncclUniqueId*))dlsym(h, "ncclGetUniqueId");
      api.CommInitRank = (int (*)(ncclComm_t*, int, ncclUniqueId, int))dlsym(h, "ncclCommInitRank");
      api.CommDestroy = (int (*)(ncclComm_t))dlsym(h, "ncclCommDestroy");
      api.AllGather = (int (*)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t))dlsym(h, "ncclAllGather");
      api.GroupStart = (int (*)())dlsym(h, "ncclGroupStart");
      api.GroupEnd = (int (*)())dlsym(h, "ncclGroupEnd");
      api.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
      api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather &&
               api.GroupStart && api.GroupEnd;
    }
  }
  return api;
}
constexpr int kNcclBfloat16 = 9;
#define G3C_NCCL(x)                                                                      \
  do {                                                                                   \
    int _r = (x);                                                                        \
    if (_r != 0) {                                                                       \
      set_error("NCCL error %d (%s) in `%s`", _r,                                        \
                nccl().GetErrorString ? nccl().GetErrorString(_r) : "?", #x);            \
      return G3C_ENCCL;                                                                  \
    }                                                                                    \
  } while (0)

struct WTensor {
  const void* ptr = nullptr;
  std::vector<int64_t> shape;
  int dtype = 0;
};

// One Linear weight [N, K]: the registered bf16 tensor and, in the fp8 Linear mode, the engine's e4m3 copy of it
// (codes + per-output-channel scales [N]).  A Linear without codes runs in bf16.
struct Linear {
  const __nv_bfloat16* w = nullptr;
  uint8_t* codes = nullptr;
  float* scale = nullptr;
};

// The activation rows [M, K] a Linear reads: bf16 rows, and in the fp8 Linear mode their e4m3 codes + row scales [M]
struct Act {
  const __nv_bfloat16* rows = nullptr;
  uint8_t* codes = nullptr;
  float* scale = nullptr;
};

struct SubBlock {
  Linear q, k, v, o;                                    // attention to_q / to_k / to_v / to_out
  const float *gq = nullptr, *gk = nullptr;             // RMSNorm gamma (f32 copy)
  Linear l1, l2;                                        // MLP layer1 / layer2
  const __nv_bfloat16 *ada1 = nullptr, *ada2 = nullptr;  // adaLN-LoRA
};

// The Linears of a block that run in e4m3 in the fp8 Linear mode, in their order inside h->w8: FA to_q / to_k / to_v /
// to_out, CA to_q / to_out, MLP layer1 [F, D] and layer2 [D, F]; the others are [D, D].
struct Fp8Linear {
  int sub;  // 0 FA, 1 CA, 2 MLP
  Linear SubBlock::*lin;
  bool n_ffn, k_ffn;  // N, K is ffn_dim (else model_channels)
  size_t n(const g3c_dit_config& c) const { return n_ffn ? c.ffn_dim : c.model_channels; }
  size_t k(const g3c_dit_config& c) const { return k_ffn ? c.ffn_dim : c.model_channels; }
};
constexpr Fp8Linear kFp8Linears[] = {
    {0, &SubBlock::q, false, false}, {0, &SubBlock::k, false, false}, {0, &SubBlock::v, false, false},
    {0, &SubBlock::o, false, false}, {1, &SubBlock::q, false, false}, {1, &SubBlock::o, false, false},
    {2, &SubBlock::l1, true, false}, {2, &SubBlock::l2, false, true}};

}  // namespace g3c

using namespace g3c;

struct g3c_dit {
  g3c_dit_config cfg;
  std::unordered_map<std::string, WTensor> w;
  bool resolved = false;
  std::vector<std::array<SubBlock, 3>> blk;
  const __nv_bfloat16 *w_t1 = nullptr, *w_t2 = nullptr, *w_final = nullptr, *f_ada1 = nullptr,
                      *f_ada2 = nullptr, *affine_gamma = nullptr, *pos_t = nullptr, *pos_h = nullptr,
                      *pos_w = nullptr;
  __nv_bfloat16* w_patch_pad = nullptr;  // [D, Kpad] owned
  float* gammas = nullptr;               // owned f32 copies of the RMSNorm weights
  int Kpatch = 0, Kpad = 0;
  // fp8 Linear mode (g3c_dit_set_linear_fp8): e4m3 copies of the eight large Linears of every block, quantised by
  // resolve() from the registered bf16 weights, in one allocation of w8_bytes
  bool fp8 = false;
  void* w8 = nullptr;
  size_t w8_bytes = 0;

  // shape
  int T = 0, Hl = 0, Wl = 0, Hp = 0, Wp = 0, L = 0, ctx_len = 0;
  float fps = 24.f;
  // cp
  int cp_rank = 0, cp_size = 1;
  ncclComm_t comm = nullptr;  // only in the NCCL all-gather mode (G3C_CP_MODE=nccl)
  cudaStream_t comm_stream = nullptr;
  cudaEvent_t ev_kv = nullptr, ev_gathered = nullptr;
  // default CP mode: fused projection -> all-gather through NVLink peer memory.  One cudaMalloc'd region per
  // rank, IPC-mapped by every peer: K / V^T of all ranks, double buffered by layer parity, plus arrival flags.
  bool cp_p2p = true;
  void* cp_region = nullptr;
  size_t cp_region_bytes = 0, off_k[2] = {0, 0}, off_vt[2] = {0, 0}, off_flags = 0;
  void* peer_base[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool peers_open = false;
  // peer_base holds device pointers of this process (g3c_dit_cp_attach), not IPC mappings: never close them
  bool peers_attached = false;
  uint32_t kv_seq = 0;
  // pinned ring of sequence numbers: the copy engine writes flags[rank] = seq on every peer by copying 4 bytes from
  // here after the K / V^T copies (no kernel on the side stream: a flag kernel queued behind a grid whose CTAs spin
  // on exactly that flag would never be dispatched)
  uint32_t* seq_ring = nullptr;
  static constexpr uint32_t kSeqRing = 8192;
  // workspace
  void* ws = nullptr;
  size_t ws_bytes = 0;
  float* x = nullptr;
  __nv_bfloat16 *xn = nullptr, *q = nullptr, *k_all = nullptr, *vt_all = nullptr, *att = nullptr,
                *hid = nullptr, *tok = nullptr, *pos = nullptr, *kc = nullptr, *vtc = nullptr;
  float *rope = nullptr, *yfin = nullptr, *mods = nullptr, *modf = nullptr, *vec_s = nullptr,
        *vec_emb = nullptr, *vec_h1 = nullptr, *vec_lora = nullptr, *vec_a = nullptr, *freqs = nullptr;
  __nv_bfloat16 *lat_xtilde = nullptr, *lat_xin = nullptr, *lat_oc = nullptr, *lat_ou = nullptr;
  // the cond / uncond outputs the last denoise step's sampler_post read (lat_oc / lat_ou, or the CFG exchange region);
  // NULL until a step completes after g3c_dit_set_shape or g3c_dit_set_linear_fp8 (g3c_dit_read_step)
  const __nv_bfloat16 *step_oc = nullptr, *step_ou = nullptr;
  // fp8 Linear mode: e4m3 codes + row scales of the GEMM A operands (xn, att, hid)
  uint8_t *xn8 = nullptr, *att8 = nullptr, *hid8 = nullptr;
  float *xn8_s = nullptr, *att8_s = nullptr, *hid8_s = nullptr;
  bool tables_ready = false;
  // the B=1 modulation vectors depend on the timestep only: the second forward of a denoise step reuses them
  bool mods_valid = false;
  float mods_timestep = 0.f;
  // classifier-free-guidance parallelism: this rank evaluates one branch (0 cond / 1 uncond); the partner holds the
  // other.  Exchange region (IPC-mapped by the partner): 2 slots of one latent + 2 arrival flags.
  int cfg_role = -1;
  void* cfg_region = nullptr;
  void* cfg_peer = nullptr;
  bool cfg_attached = false;  // cfg_peer is a device pointer of this process (g3c_dit_cfg_attach), not an IPC mapping
  size_t cfg_slot_bytes = 0;
  uint32_t cfg_seq = 0;
  // attention kernel: ns spent polling peer flags (summed over CTAs), CTA count of those launches
  unsigned long long* wait_ns = nullptr;
  double wait_cta_launches = 0.0;
  int launches = 0;
  // optional per-category device timing (bench.py roofline): events around every launch
  bool prof = false;
  std::vector<cudaEvent_t> ev_pool;
  std::vector<int> ev_cat;  // category of pair i (events 2i, 2i+1)
  size_t ev_used = 0;
};

namespace g3c {

// softmax scale 1/sqrt(head_dim) times log2(e), folded into the query RMSNorm gain (see resolve())
constexpr float kQScale = 0.08838834764831845f * 1.4426950408889634f;

static const WTensor* find(const g3c_dit* h, const std::string& name) {
  auto it = h->w.find(name);
  return it == h->w.end() ? nullptr : &it->second;
}

static int need_bf16(const g3c_dit* h, const std::string& name, std::initializer_list<int64_t> shape,
                     const __nv_bfloat16** out) {
  const WTensor* t = find(h, name);
  if (!t) {
    set_error("dit: weight `%s` was never loaded", name.c_str());
    return G3C_ESTATE;
  }
  if (t->dtype != G3C_DTYPE_BF16) {
    set_error("dit: weight `%s` must be bf16", name.c_str());
    return G3C_EINVAL;
  }
  std::vector<int64_t> want(shape);
  if (t->shape != want) {
    std::string got, exp;
    for (auto v : t->shape) got += std::to_string(v) + ",";
    for (auto v : want) exp += std::to_string(v) + ",";
    set_error("dit: weight `%s` has shape [%s] expected [%s]", name.c_str(), got.c_str(), exp.c_str());
    return G3C_EINVAL;
  }
  *out = reinterpret_cast<const __nv_bfloat16*>(t->ptr);
  return G3C_OK;
}

#define TRY(x)            \
  do {                    \
    int _rc = (x);        \
    if (_rc) return _rc;  \
  } while (0)

enum { CAT_GEMM = 0, CAT_ATTN_SELF = 1, CAT_ATTN_CROSS = 2, CAT_ELTWISE = 3, CAT_COMM = 4, CAT_VECTOR = 5, CAT_N = 6 };

static int prof_mark(g3c_dit* h, int cat, bool begin, cudaStream_t st) {
  if (!h->prof) return G3C_OK;
  if (h->ev_used >= h->ev_pool.size()) {
    cudaEvent_t e;
    G3C_CUDA(cudaEventCreate(&e));
    h->ev_pool.push_back(e);
  }
  G3C_CUDA(cudaEventRecord(h->ev_pool[h->ev_used++], st));
  if (begin) h->ev_cat.push_back(cat);
  return G3C_OK;
}
// K(category, launch): count the launch and, in profiling mode, bracket it with events
#define K(cat, call)                    \
  do {                                  \
    TRY(prof_mark(h, cat, true, st));   \
    TRY(call);                          \
    TRY(prof_mark(h, cat, false, st));  \
    ++n;                                \
  } while (0)

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Bytes of one e4m3 copy inside h->w8: codes [N, K], then scales [N] from offset align_up(N * K, 1024)
static size_t fp8_copy_bytes(size_t n, size_t k) { return align_up(n * k, 1024) + align_up(n * 4, 1024); }

static int resolve(g3c_dit* h, cudaStream_t st) {
  if (h->resolved) return G3C_OK;
  const g3c_dit_config& c = h->cfg;
  const int64_t D = c.model_channels, R = c.adaln_lora_dim, F = c.ffn_dim, C = c.context_dim;
  h->Kpatch = (c.in_channels + (c.concat_padding_mask ? 1 : 0)) * 4;
  h->Kpad = (h->Kpatch + 63) / 64 * 64;
  const __nv_bfloat16* wpe = nullptr;
  TRY(need_bf16(h, "x_embedder.proj.1.weight", {D, h->Kpatch}, &wpe));
  if (!h->w_patch_pad) G3C_CUDA(cudaMalloc(&h->w_patch_pad, (size_t)D * h->Kpad * 2));
  G3C_CUDA(cudaMemsetAsync(h->w_patch_pad, 0, (size_t)D * h->Kpad * 2, st));
  G3C_CUDA(cudaMemcpy2DAsync(h->w_patch_pad, (size_t)h->Kpad * 2, wpe, (size_t)h->Kpatch * 2,
                             (size_t)h->Kpatch * 2, D, cudaMemcpyDeviceToDevice, st));
  TRY(need_bf16(h, "extra_pos_embedder.pos_emb_t", {c.max_frames, D}, &h->pos_t));
  TRY(need_bf16(h, "extra_pos_embedder.pos_emb_h", {c.max_h, D}, &h->pos_h));
  TRY(need_bf16(h, "extra_pos_embedder.pos_emb_w", {c.max_w, D}, &h->pos_w));
  TRY(need_bf16(h, "t_embedder.1.linear_1.weight", {D, D}, &h->w_t1));
  TRY(need_bf16(h, "t_embedder.1.linear_2.weight", {3 * D, D}, &h->w_t2));
  TRY(need_bf16(h, "affline_norm.weight", {D}, &h->affine_gamma));
  TRY(need_bf16(h, "final_layer.linear.weight", {(int64_t)c.out_channels * 4, D}, &h->w_final));
  TRY(need_bf16(h, "final_layer.adaLN_modulation.1.weight", {R, D}, &h->f_ada1));
  TRY(need_bf16(h, "final_layer.adaLN_modulation.2.weight", {2 * D, R}, &h->f_ada2));
  h->blk.assign(c.num_blocks, std::array<SubBlock, 3>{});  // no e4m3 copies until the fp8 pass below
  if (!h->gammas) G3C_CUDA(cudaMalloc(&h->gammas, sizeof(float) * 128 * 4 * c.num_blocks));
  for (int i = 0; i < c.num_blocks; ++i) {
    for (int j = 0; j < 3; ++j) {
      SubBlock& s = h->blk[i][j];
      std::string p = "blocks.block" + std::to_string(i) + ".blocks." + std::to_string(j) + ".";
      TRY(need_bf16(h, p + "adaLN_modulation.1.weight", {R, D}, &s.ada1));
      TRY(need_bf16(h, p + "adaLN_modulation.2.weight", {3 * D, R}, &s.ada2));
      if (j < 2) {
        const int64_t kin = j == 0 ? D : C;
        TRY(need_bf16(h, p + "block.attn.to_q.0.weight", {D, D}, &s.q.w));
        TRY(need_bf16(h, p + "block.attn.to_k.0.weight", {D, kin}, &s.k.w));
        TRY(need_bf16(h, p + "block.attn.to_v.0.weight", {D, kin}, &s.v.w));
        TRY(need_bf16(h, p + "block.attn.to_out.0.weight", {D, D}, &s.o.w));
        const __nv_bfloat16 *gq = nullptr, *gk = nullptr;
        TRY(need_bf16(h, p + "block.attn.to_q.1.weight", {128}, &gq));
        TRY(need_bf16(h, p + "block.attn.to_k.1.weight", {128}, &gk));
        float* dst = h->gammas + (size_t)(i * 4 + j * 2) * 128;
        // the query gain also carries the softmax scale and log2(e): the attention kernel then receives its scores
        // in log2 units (scale = ln 2 below) and its fast tiles need no multiply-subtract per score.  RoPE is a
        // rotation, so the factor commutes with it.
        TRY(bf16_to_f32(gq, dst, 128, st, kQScale));
        TRY(bf16_to_f32(gk, dst + 128, 128, st));
        s.gq = dst;
        s.gk = dst + 128;
      } else {
        TRY(need_bf16(h, p + "block.layer1.weight", {F, D}, &s.l1.w));
        TRY(need_bf16(h, p + "block.layer2.weight", {D, F}, &s.l2.w));
      }
    }
  }
  // fp8 Linear mode: (re)quantise every fp8 Linear from the registered weights into its slot of h->w8 (block after
  // block, in the order of kFp8Linears).  Reached after g3c_dit_load and after enabling the mode.
  if (h->fp8) {
    char* w8 = (char*)h->w8;
    for (auto& b : h->blk)
      for (const Fp8Linear& l : kFp8Linears) {
        Linear& lin = b[l.sub].*l.lin;
        const size_t n = l.n(c), k = l.k(c);
        lin.codes = (uint8_t*)w8;
        lin.scale = (float*)(w8 + align_up(n * k, 1024));
        w8 += fp8_copy_bytes(n, k);
        TRY(quant_rows_e4m3(lin.w, (int)k, (int)n, (int)k, lin.codes, (int)k, lin.scale, st));
      }
  }
  h->resolved = true;
  return G3C_OK;
}

// Publish "my output of step `seq` has landed" in the CFG partner's flag.  Launched after the copy into the partner's
// memory on the same stream (complete when this kernel starts); release at system scope.
__global__ void k_cp_signal(uint32_t* flag, uint32_t seq) {
  __threadfence_system();
  asm volatile("st.release.sys.global.u32 [%0], %1;\n" ::"l"(flag), "r"(seq) : "memory");
}

// Stream-ordered wait for a peer's flag (CFG-parallel output exchange): one warp polls with system-scope acquire loads.
// The data the flag covers was written by the peer's copy engine into this GPU's memory, no SM of this GPU is needed for
// it to arrive, so a resident spinning warp cannot block its own producer.
__global__ void k_wait_flag(const uint32_t* flag, uint32_t seq, unsigned long long timeout_ns) {
  if (threadIdx.x != 0) return;
  uint32_t v, spins = 0;
  uint64_t t0 = 0;
  for (;;) {
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];\n" : "=r"(v) : "l"(flag) : "memory");
    if ((int)(v - seq) >= 0) break;
    __nanosleep(200);
    if ((++spins & 0xFFu) == 0) {
      const uint64_t now = global_timer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > timeout_ns) asm volatile("trap;\n");
    }
  }
}

// Inter-process waits (peer K/V flags, CFG partner) may legitimately take as long as the slowest rank's first-step
// set-up: their bound is separate from the 4 s intra-CTA protocol timeout and configurable (G3C_PEER_TIMEOUT_S, 600 s).
unsigned long long peer_timeout_ns() {
  static unsigned long long v = 0;
  if (!v) {
    const char* e = getenv("G3C_PEER_TIMEOUT_S");
    double sec = e ? atof(e) : 600.0;
    if (!(sec > 0)) sec = 600.0;
    v = (unsigned long long)(sec * 1e9);
  }
  return v;
}

// RoPE cos|sin table [L,128] f32 and abs-pos table [L,D] bf16 of the current shape, for a rank whose first latent frame
// is t0 (the forward's tables: t0 = cp_rank * T)
static int write_tables(g3c_dit* h, int t0, float* rope, __nv_bfloat16* pos, cudaStream_t st) {
  const g3c_dit_config& c = h->cfg;
  // RoPE frequencies — reference: position_embedding.py:106-160 (head_dim 128 -> 44 | 42 | 42)
  const int dim = 128, dim_h = dim / 6 * 2, dim_w = dim_h, dim_t = dim - 2 * dim_h;
  const int nt = dim_t / 2, nh = dim_h / 2, nw = dim_w / 2;
  std::vector<float> fr(64);
  auto ntk = [](float ratio, int d) { return powf(ratio, (float)d / (float)(d - 2)); };
  const float th_h = 10000.0f * ntk(c.rope_h_ratio, dim_h), th_w = 10000.0f * ntk(c.rope_w_ratio, dim_w),
              th_t = 10000.0f * ntk(c.rope_t_ratio, dim_t);
  for (int j = 0; j < nt; ++j) fr[j] = 1.0f / powf(th_t, (float)(2 * j) / (float)dim_t);
  for (int j = 0; j < nh; ++j) fr[nt + j] = 1.0f / powf(th_h, (float)(2 * j) / (float)dim_h);
  for (int j = 0; j < nw; ++j) fr[nt + nh + j] = 1.0f / powf(th_w, (float)(2 * j) / (float)dim_w);
  G3C_CUDA(cudaMemcpyAsync(h->freqs, fr.data(), 64 * sizeof(float), cudaMemcpyHostToDevice, st));
  G3C_CUDA(cudaStreamSynchronize(st));  // fr is a stack-lifetime host buffer
  // seq[:T] / fps * base_fps  (position_embedding.py:163)
  const float t_scale = (1.0f / h->fps) * (float)c.base_fps;
  TRY(rope_table(h->freqs, nt, nh, nw, t0, t_scale, h->T, h->Hp, h->Wp, rope, st));
  TRY(abs_pos(h->pos_t, h->pos_h, h->pos_w, t0, h->T, h->Hp, h->Wp, c.model_channels, pos, st));
  return G3C_OK;
}

static int build_tables(g3c_dit* h, cudaStream_t st) {
  if (h->tables_ready) return G3C_OK;
  TRY(write_tables(h, h->cp_rank * h->T, h->rope, h->pos, st));
  h->tables_ready = true;
  return G3C_OK;
}

// timestep embedding + all adaLN-LoRA modulation vectors (blocks.py:38-80, :442-445; general_dit.py:405) into h->mods /
// h->modf.  They depend on t only: the cond and uncond forwards of one denoise step share t (model_v2w.py:140-142), so
// they are computed once per timestep.  n counts the launches.
static int modulation(g3c_dit* h, float timestep, int& n, cudaStream_t st) {
  if (h->mods_valid && h->mods_timestep == timestep) return G3C_OK;
  const g3c_dit_config& c = h->cfg;
  const int D = c.model_channels, R = c.adaln_lora_dim;
  K(CAT_VECTOR, timestep_embed(timestep, D, h->affine_gamma, 1e-6f, h->vec_s, h->vec_emb, st));
  K(CAT_VECTOR, gemv(h->w_t1, h->vec_s, nullptr, h->vec_h1, D, D, 0, 0, st));
  K(CAT_VECTOR, gemv(h->w_t2, h->vec_h1, nullptr, h->vec_lora, 3 * D, D, 1, 0, st));
  for (int i = 0; i < c.num_blocks; ++i)
    for (int j = 0; j < 3; ++j) {
      const SubBlock& s = h->blk[i][j];
      K(CAT_VECTOR, gemv(s.ada1, h->vec_emb, nullptr, h->vec_a, R, D, 1, 0, st));
      K(CAT_VECTOR, gemv(s.ada2, h->vec_a, h->vec_lora, h->mods + (size_t)(i * 3 + j) * 3 * D, 3 * D, R, 0, 0, st));
    }
  K(CAT_VECTOR, gemv(h->f_ada1, h->vec_emb, nullptr, h->vec_a, R, D, 1, 0, st));
  K(CAT_VECTOR, gemv(h->f_ada2, h->vec_a, h->vec_lora, h->modf, 2 * D, R, 0, 0, st));
  h->mods_valid = true;
  h->mods_timestep = timestep;
  return G3C_OK;
}

// Every Linear of a block: out = epi(a . W^T) [M, N], or with vt = true its transpose W . a^T [N, M] (V^T).  It runs on
// the e4m3 copy when the Linear has one, dequantising with both row scales before the epilogue, and on the bf16 weight
// otherwise; `a` must carry codes exactly when the weight does.
static int linear(const Linear& w, const Act& a, bool vt, int M, int N, int Kin, void* out, int epi, const float* gate,
                  const NormRope* nr, cudaStream_t st) {
  const bool f8 = w.codes != nullptr;
  if (f8 != (a.codes != nullptr)) {
    set_error("dit_forward: a Linear with%s e4m3 weights got activations with%s codes", f8 ? "" : "out", f8 ? "out" : "");
    return G3C_ESTATE;
  }
  const void *A = f8 ? (const void*)a.codes : a.rows, *B = f8 ? (const void*)w.codes : w.w;
  const float *sa = a.scale, *sb = w.scale;
  if (vt) {
    std::swap(A, B);
    std::swap(sa, sb);
    std::swap(M, N);
  }
  if (f8) return gemm_fp8(A, sa, B, sb, out, M, N, Kin, Kin, Kin, N, epi, gate, 0, st, nr);
  return gemm_bf16(A, B, out, M, N, Kin, Kin, Kin, N, epi, gate, 0, st, nr);
}

static int forward(g3c_dit* h, const void* x_in, const void* cond_mask, const void* cond_pose,
                   const void* padding_mask, float timestep, const void* ctx, void* out,
                   cudaStream_t st) {
  static_assert(sizeof(float) == 4, "");
  G3C_REQUIRE(h && x_in && cond_mask && ctx && out, "dit_forward: null argument");
  G3C_REQUIRE(h->L > 0, "dit_forward: g3c_dit_set_shape was not called");
  TRY(resolve(h, st));
  TRY(build_tables(h, st));
  const g3c_dit_config& c = h->cfg;
  const int D = c.model_channels, F = c.ffn_dim, L = h->L, heads = c.num_heads;
  const int Lk_all = L * h->cp_size;
  const float attn_scale = 0.6931471805599453f;  // ln 2: 1/sqrt(128) * log2(e) is folded into the query RMSNorm gain
  int n = 0;
  // fp8 Linear mode (h->fp8): the Linears of kFp8Linears read e4m3 codes of their activation rows, xn from the fused
  // LN-modulate (which then writes no bf16 xn), att and hid from a quantisation pass of their own.  K and V^T stay bf16,
  // so the context-parallel exchange is the same in both modes.
  Act xn{h->xn}, att{h->att}, hid{h->hid};
  if (h->fp8) {
    xn = {nullptr, h->xn8, h->xn8_s};
    att = {h->att, h->att8, h->att8_s};
    hid = {h->hid, h->hid8, h->hid8_s};
  }
  const Act ctx_rows{(const __nv_bfloat16*)ctx};
  auto ln_mod = [&](const __nv_bfloat16* pos, const float* m) {
    return xn.codes ? ln_modulate_e4m3(h->x, pos, m, m + D, xn.codes, xn.scale, L, D, 1e-6f, st)
                    : ln_modulate(h->x, pos, m, m + D, h->xn, L, D, 1e-6f, st);
  };
  // to_q / to_k: Linear + per-head RMSNorm (+ RoPE), fused into the GEMM epilogue: the norm and the rotation act on the
  // fp32 accumulators in registers, so the projection never round-trips [tokens, D] bf16 through a separate pass.
  auto proj_norm_rope = [&](const Linear& w, const Act& a, int M, int Kin, __nv_bfloat16* out, const float* gamma,
                            const float* cs) {
    NormRope nr;
    nr.gamma = gamma;
    nr.cs = cs;
    nr.eps = 1e-6f;
    return linear(w, a, false, M, D, Kin, out, G3C_EPI_BF16, nullptr, &nr, st);
  };
  // x += gate * (a . W^T): the gated-residual output projection, after the pass that quantises a when it feeds codes
  auto out_proj = [&](const Linear& w, const Act& a, int Kin, const float* gate) -> int {
    if (a.codes) K(CAT_ELTWISE, quant_rows_e4m3(a.rows, Kin, L, Kin, a.codes, Kin, a.scale, st));
    K(CAT_GEMM, linear(w, a, false, L, D, Kin, h->x, G3C_EPI_GATED_RESIDUAL_F32, gate, nullptr, st));
    return G3C_OK;
  };

  // ---- input assembly + patch embedding (general_dit_video_conditioned.py:112-118,
  //      general_dit.py:304-311, blocks.py:153-163)
  PatchSrc src;
  src.ptr[0] = (const __nv_bfloat16*)x_in;        src.nch[0] = 16;                      src.per_frame[0] = 1;
  src.ptr[1] = (const __nv_bfloat16*)cond_mask;   src.nch[1] = 1;                       src.per_frame[1] = 1;
  src.ptr[2] = (const __nv_bfloat16*)cond_pose;   src.nch[2] = c.in_channels - 17;      src.per_frame[2] = 1;
  src.ptr[3] = (const __nv_bfloat16*)padding_mask; src.nch[3] = c.concat_padding_mask ? 1 : 0; src.per_frame[3] = 0;
  K(CAT_ELTWISE, patchify(src, h->T, h->Hp, h->Wp, h->Kpad, h->tok, st));
  K(CAT_GEMM, gemm_bf16(h->tok, h->w_patch_pad, h->x, L, D, h->Kpad, h->Kpad, h->Kpad, D, G3C_EPI_F32, nullptr, 0, st));

  // ---- timestep embedding + adaLN-LoRA modulation vectors (cached per timestep)
  TRY(modulation(h, timestep, n, st));

  const bool p2p = h->cp_size > 1 && h->cp_p2p;
  for (int i = 0; i < c.num_blocks; ++i) {
    // ---------------- FA: full self-attention (blocks.py:455-463, attention.py:247-289)
    {
      const SubBlock& s = h->blk[i][0];
      const float* m = h->mods + (size_t)(i * 3 + 0) * 3 * D;
      K(CAT_ELTWISE, ln_mod(h->pos, m));   // + abs-pos add
      // K and V^T of every rank, [cp][L, D] and [cp][D][L]: in p2p mode one of the two layer-parity sets of the
      // peer-mapped region, else k_all / vt_all.  This rank projects its slice straight into it.
      if (p2p) G3C_REQUIRE(h->peers_open, "dit_forward: context-parallel peers not imported (g3c_dit_cp_import)");
      const uint32_t seq = p2p ? ++h->kv_seq : 0;
      const int set = seq & 1, me = h->cp_rank;
      char* reg = (char*)h->cp_region;
      __nv_bfloat16* kb = p2p ? (__nv_bfloat16*)(reg + h->off_k[set]) : h->k_all;
      __nv_bfloat16* vb = p2p ? (__nv_bfloat16*)(reg + h->off_vt[set]) : h->vt_all;
      __nv_bfloat16* kl = kb + (size_t)me * L * D;
      __nv_bfloat16* vl = vb + (size_t)me * L * D;
      K(CAT_GEMM, proj_norm_rope(s.k, xn, L, D, kl, s.gk, h->rope));
      K(CAT_GEMM, linear(s.v, xn, true, L, D, D, vl, G3C_EPI_BF16, nullptr, nullptr, st));  // V^T
      if (p2p) {
        // all-gather through peer memory: every rank produces its K / V^T slice locally, then the copy engines push
        // it into every peer's buffer on a side stream and raise a flag there, while this stream already runs the Q
        // projection and attention over the local chunk; attention picks up the remote chunks as their flags arrive.
        // Peer (me-1) is served first, then (me-2), ...: rank c consumes chunk c+1 first, so its k-th remote chunk is
        // the k-th push of its producer.  The flag that opens the chunk on a peer follows that peer's two copies on the
        // same stream (a 4-byte copy from a pinned ring: no kernel, see seq_ring).
        const size_t slice = (size_t)L * D * 2;
        G3C_CUDA(cudaEventRecord(h->ev_kv, st));
        G3C_CUDA(cudaStreamWaitEvent(h->comm_stream, h->ev_kv, 0));
        uint32_t* slot = h->seq_ring + (seq % g3c_dit::kSeqRing);
        *slot = seq;  // read by the copy engine when the copies queued before it have completed
        for (int i2 = 1; i2 < h->cp_size; ++i2) {
          const int r = (me - i2 + h->cp_size) % h->cp_size;
          char* pb = (char*)h->peer_base[r];
          G3C_CUDA(cudaMemcpyAsync(pb + h->off_k[set] + (size_t)me * slice, kl, slice, cudaMemcpyDeviceToDevice,
                                   h->comm_stream));
          G3C_CUDA(cudaMemcpyAsync(pb + h->off_vt[set] + (size_t)me * slice, vl, slice, cudaMemcpyDeviceToDevice,
                                   h->comm_stream));
          G3C_CUDA(cudaMemcpyAsync(pb + h->off_flags + (size_t)(set * 8 + me) * 4, slot, 4, cudaMemcpyHostToDevice,
                                   h->comm_stream));
        }
      } else if (h->cp_size > 1) {
        // baseline mode (G3C_CP_MODE=nccl): one in-place all-gather of K and of V^T per layer on a side stream
        G3C_CUDA(cudaEventRecord(h->ev_kv, st));
        G3C_CUDA(cudaStreamWaitEvent(h->comm_stream, h->ev_kv, 0));
        G3C_NCCL(nccl().GroupStart());
        G3C_NCCL(nccl().AllGather(kl, h->k_all, (size_t)L * D, kNcclBfloat16, h->comm, h->comm_stream));
        G3C_NCCL(nccl().AllGather(vl, h->vt_all, (size_t)L * D, kNcclBfloat16, h->comm, h->comm_stream));
        G3C_NCCL(nccl().GroupEnd());
        G3C_CUDA(cudaEventRecord(h->ev_gathered, h->comm_stream));
        n += 2;
      }
      K(CAT_GEMM, proj_norm_rope(s.q, xn, L, D, h->q, s.gq, h->rope));
      ChunkGate gate;
      if (p2p) {
        gate.flags = (const uint32_t*)(reg + h->off_flags) + set * 8;
        gate.seq = seq;
        gate.first = me;
        gate.wait_ns = h->prof ? h->wait_ns : nullptr;
        h->wait_cta_launches = (double)((L + ATT_ROWS_PER_CTA - 1) / ATT_ROWS_PER_CTA) * heads;  // CTAs of one gated launch
      } else if (h->cp_size > 1) {
        G3C_CUDA(cudaStreamWaitEvent(st, h->ev_gathered, 0));
      }
      K(CAT_ATTN_SELF,
        attn_fwd(h->q, kb, vb, h->att, L, Lk_all, heads, D, D, D, L, attn_scale, st, p2p ? &gate : nullptr));
      TRY(out_proj(s.o, att, D, m + 2 * D));
    }
    // ---------------- CA: cross-attention to the T5 context (blocks.py:464-471)
    {
      const SubBlock& s = h->blk[i][1];
      const float* m = h->mods + (size_t)(i * 3 + 1) * 3 * D;
      const int C = c.context_dim, M = h->ctx_len;
      K(CAT_ELTWISE, ln_mod(nullptr, m));
      K(CAT_GEMM, proj_norm_rope(s.k, ctx_rows, M, C, h->kc, s.gk, nullptr));
      K(CAT_GEMM, linear(s.v, ctx_rows, true, M, D, C, h->vtc, G3C_EPI_BF16, nullptr, nullptr, st));  // V^T
      K(CAT_GEMM, proj_norm_rope(s.q, xn, L, D, h->q, s.gq, nullptr));
      K(CAT_ATTN_CROSS, attn_fwd(h->q, h->kc, h->vtc, h->att, L, M, heads, D, D, D, M, attn_scale, st));
      TRY(out_proj(s.o, att, D, m + 2 * D));
    }
    // ---------------- MLP (attention.py:91-102)
    {
      const SubBlock& s = h->blk[i][2];
      const float* m = h->mods + (size_t)(i * 3 + 2) * 3 * D;
      K(CAT_ELTWISE, ln_mod(nullptr, m));
      K(CAT_GEMM, linear(s.l1, xn, false, L, F, D, h->hid, G3C_EPI_GELU_BF16, nullptr, nullptr, st));
      TRY(out_proj(s.l2, hid, F, m + 2 * D));
    }
  }
  // ---- final layer + unpatchify (blocks.py:222-242, general_dit.py:328-358)
  const int No = c.out_channels * 4;
  K(CAT_ELTWISE, ln_modulate(h->x, nullptr, h->modf, h->modf + D, h->xn, L, D, 1e-6f, st));
  K(CAT_GEMM, gemm_bf16(h->xn, h->w_final, h->yfin, L, No, D, D, D, No, G3C_EPI_F32, nullptr, 64, st));
  K(CAT_ELTWISE, unpatchify(h->yfin, No, h->T, h->Hp, h->Wp, c.out_channels, (__nv_bfloat16*)out, st));
  h->launches = n;
  return G3C_OK;
}

}  // namespace g3c

extern "C" {

int g3c_dit_create(const g3c_dit_config* cfg, g3c_dit_t** out) {
  G3C_REQUIRE(cfg && out, "dit_create: null argument");
  G3C_REQUIRE(cfg->model_channels % 128 == 0 && cfg->num_heads * 128 == cfg->model_channels,
              "dit_create: head_dim must be 128 (model_channels=%d heads=%d)", cfg->model_channels,
              cfg->num_heads);
  G3C_REQUIRE(cfg->adaln_lora_dim % 8 == 0 && cfg->context_dim % 8 == 0 && cfg->ffn_dim % 8 == 0,
              "dit_create: adaln_lora_dim/context_dim/ffn_dim must be multiples of 8");
  G3C_REQUIRE(cfg->in_channels >= 17 && cfg->out_channels > 0 && cfg->num_blocks > 0, "dit_create: bad config");
  g3c_dit* h = new g3c_dit();
  h->cfg = *cfg;
  *out = h;
  return G3C_OK;
}

static void free_cp_region(g3c_dit* h) {
  // queued peer copies / flag writes may still target these mappings (denoise_step is asynchronous): drain this device
  // before unmapping.  The cross-rank half of the hazard (peers still pushing into OUR region) is closed by the caller's
  // barrier on the cp group (gen3c_b200/dit.py::_teardown_barrier).
  if (h->cp_region || h->cfg_region) cudaDeviceSynchronize();
  if (h->cfg_peer && !h->cfg_attached) cudaIpcCloseMemHandle(h->cfg_peer);
  h->cfg_peer = nullptr;
  h->cfg_attached = false;
  if (h->cfg_region) cudaFree(h->cfg_region);
  h->cfg_region = nullptr;
  for (int r = 0; r < 8; ++r) {
    if (h->peer_base[r] && h->peer_base[r] != h->cp_region && !h->peers_attached)
      cudaIpcCloseMemHandle(h->peer_base[r]);
    h->peer_base[r] = nullptr;
  }
  h->peers_open = false;
  h->peers_attached = false;
  if (h->cp_region) cudaFree(h->cp_region);
  h->cp_region = nullptr;
  h->cp_region_bytes = 0;
}

static void free_ws(g3c_dit* h) {
  free_cp_region(h);
  if (h->ws) cudaFree(h->ws);
  h->ws = nullptr;
  h->ws_bytes = 0;
  h->L = 0;
  h->tables_ready = false;
  h->mods_valid = false;
  h->step_oc = h->step_ou = nullptr;
}

int g3c_dit_destroy(g3c_dit_t* h) {
  if (!h) return G3C_OK;
  free_ws(h);
  if (h->w_patch_pad) cudaFree(h->w_patch_pad);
  if (h->gammas) cudaFree(h->gammas);
  if (h->w8) cudaFree(h->w8);
  if (h->comm && nccl().ok) nccl().CommDestroy(h->comm);
  if (h->comm_stream) cudaStreamDestroy(h->comm_stream);
  if (h->seq_ring) cudaFreeHost(h->seq_ring);
  if (h->wait_ns) cudaFree(h->wait_ns);
  if (h->ev_kv) cudaEventDestroy(h->ev_kv);
  if (h->ev_gathered) cudaEventDestroy(h->ev_gathered);
  for (cudaEvent_t e : h->ev_pool) cudaEventDestroy(e);
  delete h;
  return G3C_OK;
}

int g3c_dit_load(g3c_dit_t* h, const char* name, const void* ptr, const int64_t* shape, int ndim, int dtype) {
  G3C_REQUIRE(h && name && ptr && shape && ndim >= 1 && ndim <= 4, "dit_load: bad arguments");
  WTensor t;
  t.ptr = ptr;
  t.shape.assign(shape, shape + ndim);
  t.dtype = dtype;
  h->w[name] = t;
  h->resolved = false;
  h->tables_ready = false;
  h->mods_valid = false;
  return G3C_OK;
}

int g3c_nccl_unique_id(void* out128) {
  G3C_REQUIRE(out128, "nccl_unique_id: null argument");
  if (!nccl().ok) {
    set_error("libnccl.so.2 could not be loaded");
    return G3C_ENCCL;
  }
  ncclUniqueId id;
  G3C_NCCL(nccl().GetUniqueId(&id));
  memcpy(out128, &id, 128);
  return G3C_OK;
}

int g3c_dit_enable_cp(g3c_dit_t* h, const void* nccl_unique_id, int cp_rank, int cp_size) {
  G3C_REQUIRE(h && cp_size >= 1 && cp_size <= 8 && cp_rank >= 0 && cp_rank < cp_size, "enable_cp: bad arguments");
  if (h->comm && nccl().ok) {
    nccl().CommDestroy(h->comm);
    h->comm = nullptr;
  }
  h->cp_p2p = nccl_unique_id == nullptr;  // NULL id: fused peer-memory mode (default); else NCCL all-gather mode
  if (!h->cp_p2p) {
    if (!nccl().ok) {
      set_error("libnccl.so.2 could not be loaded");
      return G3C_ENCCL;
    }
    ncclUniqueId id;
    memcpy(&id, nccl_unique_id, 128);
    G3C_NCCL(nccl().CommInitRank(&h->comm, cp_size, id, cp_rank));
  }
  if (!h->comm_stream) {
    int lo = 0, hi = 0;
    G3C_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    G3C_CUDA(cudaStreamCreateWithPriority(&h->comm_stream, cudaStreamNonBlocking, hi));
  }
  if (!h->seq_ring) G3C_CUDA(cudaHostAlloc(&h->seq_ring, g3c_dit::kSeqRing * sizeof(uint32_t), cudaHostAllocPortable));
  if (!h->ev_kv) G3C_CUDA(cudaEventCreateWithFlags(&h->ev_kv, cudaEventDisableTiming));
  if (!h->ev_gathered) G3C_CUDA(cudaEventCreateWithFlags(&h->ev_gathered, cudaEventDisableTiming));
  h->cp_rank = cp_rank;
  h->cp_size = cp_size;
  free_ws(h);  // shape-dependent buffers change with cp_size
  return G3C_OK;
}

int g3c_dit_cp_export(g3c_dit_t* h, void* out_handle64) {
  G3C_REQUIRE(h && out_handle64, "cp_export: null argument");
  G3C_REQUIRE(h->cp_region, "cp_export: no context-parallel region (enable_cp without NCCL id, then set_shape)");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t hd;
  G3C_CUDA(cudaIpcGetMemHandle(&hd, h->cp_region));
  memcpy(out_handle64, &hd, 64);
  return G3C_OK;
}

int g3c_dit_cp_import(g3c_dit_t* h, const void* handles, int n) {
  G3C_REQUIRE(h && handles && n == h->cp_size, "cp_import: need one 64-byte handle per rank (%d)", h ? h->cp_size : 0);
  G3C_REQUIRE(h->cp_region, "cp_import: no context-parallel region");
  for (int r = 0; r < n; ++r) {
    if (r == h->cp_rank) {
      h->peer_base[r] = h->cp_region;
      continue;
    }
    if (h->peer_base[r]) continue;
    cudaIpcMemHandle_t hd;
    memcpy(&hd, (const char*)handles + 64 * r, 64);
    G3C_CUDA(cudaIpcOpenMemHandle(&h->peer_base[r], hd, cudaIpcMemLazyEnablePeerAccess));
  }
  h->peers_open = true;
  return G3C_OK;
}

int g3c_dit_cp_mode(const g3c_dit_t* h) { return (h && h->cp_size > 1) ? (h->cp_p2p ? 1 : 2) : 0; }

int g3c_dit_disable_cp(g3c_dit_t* h) {
  G3C_REQUIRE(h, "disable_cp: null handle");
  if (h->comm && nccl().ok) nccl().CommDestroy(h->comm);
  h->comm = nullptr;
  h->cp_rank = 0;
  h->cp_size = 1;
  free_ws(h);
  return G3C_OK;
}

int g3c_dit_set_shape(g3c_dit_t* h, int T_local, int H_latent, int W_latent, int ctx_len, float fps) {
  G3C_REQUIRE(h, "set_shape: null handle");
  h->step_oc = h->step_ou = nullptr;
  const g3c_dit_config& c = h->cfg;
  G3C_REQUIRE(T_local > 0 && H_latent > 0 && W_latent > 0 && H_latent % 2 == 0 && W_latent % 2 == 0,
              "set_shape: latent H, W must be positive and even (patch 2)");
  const int Hp = H_latent / 2, Wp = W_latent / 2;
  G3C_REQUIRE(Hp <= c.max_h && Wp <= c.max_w && T_local * h->cp_size <= c.max_frames,
              "set_shape: token grid %dx%dx%d exceeds the position tables", T_local * h->cp_size, Hp, Wp);
  const long long L = (long long)T_local * Hp * Wp;
  G3C_REQUIRE((L * h->cp_size) % 128 == 0 && L % 128 == 0,
              "set_shape: tokens per rank (%lld) must be a multiple of 128", L);
  G3C_REQUIRE(ctx_len > 0 && ctx_len % 128 == 0, "set_shape: ctx_len=%d must be a multiple of 128", ctx_len);
  G3C_REQUIRE(fps > 0, "set_shape: fps must be positive");
  if (h->ws && h->T == T_local && h->Hl == H_latent && h->Wl == W_latent && h->ctx_len == ctx_len &&
      h->fps == fps)
    return G3C_OK;
  free_ws(h);
  const size_t D = c.model_channels, F = c.ffn_dim, cp = h->cp_size;
  const size_t Kpad = ((size_t)(c.in_channels + (c.concat_padding_mask ? 1 : 0)) * 4 + 63) / 64 * 64;
  const size_t lat = (size_t)16 * T_local * H_latent * W_latent;
  struct Item { void** p; size_t bytes; };
  std::vector<Item> items = {
      {(void**)&h->x, (size_t)L * D * 4},        {(void**)&h->xn, (size_t)L * D * 2},
      {(void**)&h->q, (size_t)L * D * 2},        {(void**)&h->k_all, (size_t)L * D * 2 * cp},
      {(void**)&h->vt_all, (size_t)L * D * 2 * cp}, {(void**)&h->att, (size_t)L * D * 2},
      {(void**)&h->hid, (size_t)L * F * 2},      {(void**)&h->tok, (size_t)L * Kpad * 2},
      {(void**)&h->pos, (size_t)L * D * 2},      {(void**)&h->kc, (size_t)ctx_len * D * 2},
      {(void**)&h->vtc, (size_t)ctx_len * D * 2}, {(void**)&h->rope, (size_t)L * 128 * 4},
      {(void**)&h->yfin, (size_t)L * c.out_channels * 4 * 4},
      {(void**)&h->mods, (size_t)c.num_blocks * 3 * 3 * D * 4}, {(void**)&h->modf, 2 * D * 4},
      {(void**)&h->vec_s, D * 4},                {(void**)&h->vec_emb, D * 4},
      {(void**)&h->vec_h1, D * 4},               {(void**)&h->vec_lora, 3 * D * 4},
      {(void**)&h->vec_a, (size_t)c.adaln_lora_dim * 4}, {(void**)&h->freqs, 64 * 4},
      {(void**)&h->lat_xtilde, lat * 2},         {(void**)&h->lat_xin, lat * 2},
      {(void**)&h->lat_oc, lat * 2},             {(void**)&h->lat_ou, lat * 2},
  };
  if (h->fp8) {
    items.push_back({(void**)&h->xn8, (size_t)L * D});
    items.push_back({(void**)&h->att8, (size_t)L * D});
    items.push_back({(void**)&h->hid8, (size_t)L * F});
    items.push_back({(void**)&h->xn8_s, (size_t)L * 4});
    items.push_back({(void**)&h->att8_s, (size_t)L * 4});
    items.push_back({(void**)&h->hid8_s, (size_t)L * 4});
  }
  size_t total = 0;
  for (auto& it : items) total += align_up(it.bytes, 1024);
  cudaError_t e = cudaMalloc(&h->ws, total);
  if (e != cudaSuccess) {
    h->ws = nullptr;
    set_error("dit_set_shape: cudaMalloc of %zu bytes failed: %s", total, cudaGetErrorString(e));
    return G3C_ENOMEM;
  }
  size_t off = 0;
  for (auto& it : items) {
    *it.p = (char*)h->ws + off;
    off += align_up(it.bytes, 1024);
  }
  h->ws_bytes = total;
  if (h->cp_size > 1 && h->cp_p2p) {
    const size_t set_bytes = align_up((size_t)L * D * 2 * cp, 1024);
    h->off_k[0] = 0;
    h->off_k[1] = set_bytes;
    h->off_vt[0] = 2 * set_bytes;
    h->off_vt[1] = 3 * set_bytes;
    h->off_flags = 4 * set_bytes;
    h->cp_region_bytes = 4 * set_bytes + 1024;
    e = cudaMalloc(&h->cp_region, h->cp_region_bytes);
    if (e != cudaSuccess) {
      h->cp_region = nullptr;
      set_error("dit_set_shape: cudaMalloc of the %zu-byte context-parallel region failed: %s", h->cp_region_bytes,
                cudaGetErrorString(e));
      return G3C_ENOMEM;
    }
    G3C_CUDA(cudaMemset(h->cp_region, 0, h->cp_region_bytes));
    h->peer_base[h->cp_rank] = h->cp_region;
    h->ws_bytes += h->cp_region_bytes;
  }
  if (h->cfg_role >= 0) {
    h->cfg_slot_bytes = align_up(lat * 2, 1024);
    e = cudaMalloc(&h->cfg_region, 2 * h->cfg_slot_bytes + 1024);
    if (e != cudaSuccess) {
      h->cfg_region = nullptr;
      set_error("dit_set_shape: cudaMalloc of the CFG exchange region failed: %s", cudaGetErrorString(e));
      return G3C_ENOMEM;
    }
    G3C_CUDA(cudaMemset(h->cfg_region, 0, 2 * h->cfg_slot_bytes + 1024));
    h->ws_bytes += 2 * h->cfg_slot_bytes + 1024;
    h->cfg_seq = 0;
  }
  if (!h->wait_ns) {
    G3C_CUDA(cudaMalloc(&h->wait_ns, sizeof(unsigned long long)));
    G3C_CUDA(cudaMemset(h->wait_ns, 0, sizeof(unsigned long long)));
  }
  h->T = T_local;
  h->Hl = H_latent;
  h->Wl = W_latent;
  h->Hp = Hp;
  h->Wp = Wp;
  h->L = (int)L;
  h->ctx_len = ctx_len;
  h->fps = fps;
  h->tables_ready = false;
  return G3C_OK;
}

int g3c_dit_forward(g3c_dit_t* h, const void* x, const void* cond_mask, const void* cond_pose,
                    const void* padding_mask, float timestep, const void* ctx, void* out, void* stream) {
  return g3c::forward(h, x, cond_mask, cond_pose, padding_mask, timestep, ctx, out, (cudaStream_t)stream);
}

int g3c_denoise_step(g3c_dit_t* h, const g3c_step_args* a, void* stream) {
  G3C_REQUIRE(h && a && a->xt && a->gt_latent && a->aug_noise && a->indicator && a->cond_mask &&
                  a->ctx_cond && a->ctx_uncond && a->xt_next,
              "denoise_step: null argument");
  G3C_REQUIRE(h->L > 0, "denoise_step: g3c_dit_set_shape was not called");
  G3C_REQUIRE(a->sigma > 0, "denoise_step: sigma must be positive");
  h->step_oc = h->step_ou = nullptr;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t plane = (size_t)h->Hl * h->Wl;
  // t = 0.25 * ln(sigma)  (EDMEulerScheduler timesteps; model_v2w.py:131-140)
  // ... fed to the net as a bf16 tensor (model_v2w.py:140 `t.to(**self.tensor_kwargs)`)
  const float timestep = __bfloat162float(__float2bfloat16_rn(0.25f * logf(a->sigma)));
  const void* mask_u = a->cond_mask_uncond ? a->cond_mask_uncond : a->cond_mask;
  TRY(sampler_pre((const __nv_bfloat16*)a->xt, (const __nv_bfloat16*)a->gt_latent, a->aug_noise,
                  a->indicator, 16, h->T, plane, a->sigma, a->sigma_aug, a->sigma_data, h->lat_xtilde,
                  h->lat_xin, st));
  const __nv_bfloat16 *oc = h->lat_oc, *ou = h->lat_ou;
  int n_launch = 2;
  if (h->cfg_role < 0) {
    TRY(g3c::forward(h, h->lat_xin, a->cond_mask, a->pose_cond, a->padding_mask, timestep, a->ctx_cond,
                     h->lat_oc, st));
    n_launch += h->launches;
    TRY(g3c::forward(h, h->lat_xin, mask_u, nullptr, a->padding_mask, timestep, a->ctx_uncond, h->lat_ou, st));
    n_launch += h->launches;
  } else {
    // CFG-parallel: this rank evaluates one branch, the partner the other; the two outputs are swapped through peer
    // memory (copy engine push + system-scope flag), then both ranks apply the same sampler update.
    G3C_REQUIRE(h->cfg_region && h->cfg_peer, "denoise_step: CFG partner not imported (g3c_dit_cfg_import)");
    __nv_bfloat16* mine = h->cfg_role == 0 ? h->lat_oc : h->lat_ou;
    if (h->cfg_role == 0)
      TRY(g3c::forward(h, h->lat_xin, a->cond_mask, a->pose_cond, a->padding_mask, timestep, a->ctx_cond, mine, st));
    else
      TRY(g3c::forward(h, h->lat_xin, mask_u, nullptr, a->padding_mask, timestep, a->ctx_uncond, mine, st));
    n_launch += h->launches;
    const uint32_t seq = ++h->cfg_seq;
    const int slot = seq & 1;
    const size_t bytes = (size_t)16 * h->T * plane * 2;
    char* peer = (char*)h->cfg_peer;
    char* own = (char*)h->cfg_region;
    TRY(prof_mark(h, CAT_COMM, true, st));
    G3C_CUDA(cudaMemcpyAsync(peer + (size_t)slot * h->cfg_slot_bytes, mine, bytes, cudaMemcpyDeviceToDevice, st));
    k_cp_signal<<<1, 1, 0, st>>>((uint32_t*)(peer + 2 * h->cfg_slot_bytes) + slot, seq);
    k_wait_flag<<<1, 32, 0, st>>>((const uint32_t*)(own + 2 * h->cfg_slot_bytes) + slot, seq, peer_timeout_ns());
    G3C_CUDA(cudaGetLastError());
    TRY(prof_mark(h, CAT_COMM, false, st));
    n_launch += 2;
    const __nv_bfloat16* theirs = (const __nv_bfloat16*)(own + (size_t)slot * h->cfg_slot_bytes);
    oc = h->cfg_role == 0 ? mine : theirs;
    ou = h->cfg_role == 0 ? theirs : mine;
  }
  TRY(sampler_post(h->lat_xtilde, oc, ou, (const __nv_bfloat16*)a->gt_latent, a->indicator, 16, h->T, plane,
                   a->guidance, a->sigma, a->sigma_next, a->sigma_aug, a->sigma_data, (__nv_bfloat16*)a->xt_next,
                   (__nv_bfloat16*)a->net_output, st));
  h->launches = n_launch;
  h->step_oc = oc;
  h->step_ou = ou;
  return G3C_OK;
}

int g3c_dit_set_linear_fp8(g3c_dit_t* h, int on) {
  G3C_REQUIRE(h, "set_linear_fp8: null handle");
  G3C_REQUIRE(h->cfg.ffn_dim % 16 == 0, "set_linear_fp8: ffn_dim=%d must be a multiple of 16", h->cfg.ffn_dim);
  h->step_oc = h->step_ou = nullptr;
  if ((on != 0) == h->fp8) return G3C_OK;
  free_ws(h);  // the fp8 activation buffers come and go with the shape's workspace
  if (on) {
    size_t bytes = 0;
    for (const Fp8Linear& l : kFp8Linears) bytes += h->cfg.num_blocks * fp8_copy_bytes(l.n(h->cfg), l.k(h->cfg));
    cudaError_t e = cudaMalloc(&h->w8, bytes);
    if (e != cudaSuccess) {
      h->w8 = nullptr;
      set_error("set_linear_fp8: cudaMalloc of %zu bytes of e4m3 weights failed: %s", bytes, cudaGetErrorString(e));
      return G3C_ENOMEM;
    }
    h->w8_bytes = bytes;
  } else {
    G3C_CUDA(cudaDeviceSynchronize());  // forwards still queued may read the copies
    G3C_CUDA(cudaFree(h->w8));
    h->w8 = nullptr;
    h->w8_bytes = 0;
  }
  h->fp8 = on != 0;
  h->resolved = false;  // resolve() points the Linears at the new copies and quantises into them, or drops the old ones
  return G3C_OK;
}

int g3c_dit_enable_cfg_parallel(g3c_dit_t* h, int role) {
  G3C_REQUIRE(h && role <= 1, "enable_cfg_parallel: role must be 0 (cond), 1 (uncond) or negative (off)");
  h->cfg_role = role < 0 ? -1 : role;
  free_ws(h);  // the exchange region is allocated with the shape
  return G3C_OK;
}

int g3c_dit_cfg_export(g3c_dit_t* h, void* out_handle64) {
  G3C_REQUIRE(h && out_handle64, "cfg_export: null argument");
  G3C_REQUIRE(h->cfg_region, "cfg_export: no exchange region (enable_cfg_parallel, then set_shape)");
  cudaIpcMemHandle_t hd;
  G3C_CUDA(cudaIpcGetMemHandle(&hd, h->cfg_region));
  memcpy(out_handle64, &hd, 64);
  return G3C_OK;
}

int g3c_dit_cfg_import(g3c_dit_t* h, const void* partner_handle64) {
  G3C_REQUIRE(h && partner_handle64, "cfg_import: null argument");
  G3C_REQUIRE(h->cfg_region, "cfg_import: no exchange region");
  if (h->cfg_peer) return G3C_OK;
  cudaIpcMemHandle_t hd;
  memcpy(&hd, partner_handle64, 64);
  G3C_CUDA(cudaIpcOpenMemHandle(&h->cfg_peer, hd, cudaIpcMemLazyEnablePeerAccess));
  return G3C_OK;
}

int g3c_dit_profile_wait_ms(g3c_dit_t* h, float* ms) {
  G3C_REQUIRE(h && ms, "dit_profile_wait_ms: null argument");
  *ms = 0.f;
  if (!h->wait_ns) return G3C_OK;
  unsigned long long v = 0;
  G3C_CUDA(cudaDeviceSynchronize());
  G3C_CUDA(cudaMemcpy(&v, h->wait_ns, sizeof(v), cudaMemcpyDeviceToHost));
  G3C_CUDA(cudaMemset(h->wait_ns, 0, sizeof(v)));
  // total ns over all CTAs and launches / CTAs per launch = sum over launches of the mean wait per CTA
  if (h->wait_cta_launches > 0) *ms = (float)((double)v * 1e-6 / h->wait_cta_launches);
  return G3C_OK;
}

int g3c_dit_profile(g3c_dit_t* h, int enable) {
  G3C_REQUIRE(h, "dit_profile: null handle");
  h->prof = enable != 0;
  h->ev_used = 0;
  h->ev_cat.clear();
  if (h->wait_ns) G3C_CUDA(cudaMemset(h->wait_ns, 0, sizeof(unsigned long long)));
  return G3C_OK;
}

int g3c_dit_profile_read(g3c_dit_t* h, float* ms_by_category, int* launches_by_category, int ncat) {
  G3C_REQUIRE(h && ms_by_category && launches_by_category && ncat >= CAT_N, "dit_profile_read: need %d categories", CAT_N);
  for (int i = 0; i < ncat; ++i) {
    ms_by_category[i] = 0.f;
    launches_by_category[i] = 0;
  }
  G3C_CUDA(cudaDeviceSynchronize());
  for (size_t i = 0; i < h->ev_cat.size() && 2 * i + 1 < h->ev_used; ++i) {
    float ms = 0.f;
    G3C_CUDA(cudaEventElapsedTime(&ms, h->ev_pool[2 * i], h->ev_pool[2 * i + 1]));
    ms_by_category[h->ev_cat[i]] += ms;
    launches_by_category[h->ev_cat[i]] += 1;
  }
  h->ev_used = 0;
  h->ev_cat.clear();
  return G3C_OK;
}

int64_t g3c_dit_workspace_bytes(const g3c_dit_t* h) { return h ? (int64_t)(h->ws_bytes + h->w8_bytes) : 0; }
int g3c_dit_last_launch_count(const g3c_dit_t* h) { return h ? h->launches : 0; }

// ---- C ABI test hooks for the engine's derived tables and vectors --------------------------------
int g3c_dit_read_tables(g3c_dit_t* h, int t0, float* rope, void* pos, void* stream) {
  G3C_REQUIRE(h && rope && pos, "dit_read_tables: null argument");
  G3C_REQUIRE(h->L > 0, "dit_read_tables: g3c_dit_set_shape was not called");
  G3C_REQUIRE(t0 >= 0 && t0 + h->T <= h->cfg.max_frames, "dit_read_tables: frames [%d, %d) exceed max_frames=%d", t0,
              t0 + h->T, h->cfg.max_frames);
  cudaStream_t st = (cudaStream_t)stream;
  TRY(resolve(h, st));
  return write_tables(h, t0, rope, (__nv_bfloat16*)pos, st);
}

int g3c_dit_read_modulation(g3c_dit_t* h, float timestep, float* mods, float* modf, void* stream) {
  G3C_REQUIRE(h && mods && modf, "dit_read_modulation: null argument");
  G3C_REQUIRE(h->L > 0, "dit_read_modulation: g3c_dit_set_shape was not called");
  cudaStream_t st = (cudaStream_t)stream;
  TRY(resolve(h, st));
  int n = 0;
  TRY(modulation(h, timestep, n, st));
  const size_t D = h->cfg.model_channels;
  G3C_CUDA(cudaMemcpyAsync(mods, h->mods, (size_t)h->cfg.num_blocks * 3 * 3 * D * sizeof(float),
                           cudaMemcpyDeviceToDevice, st));
  G3C_CUDA(cudaMemcpyAsync(modf, h->modf, 2 * D * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return G3C_OK;
}

int g3c_dit_read_step(g3c_dit_t* h, void* xtilde, void* xin, void* oc, void* ou, void* stream) {
  G3C_REQUIRE(h && xtilde && xin && oc && ou, "dit_read_step: null argument");
  if (!h->step_oc) {
    set_error("dit_read_step: no g3c_denoise_step since the last g3c_dit_set_shape or g3c_dit_set_linear_fp8");
    return G3C_ESTATE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t bytes = (size_t)16 * h->T * h->Hl * h->Wl * sizeof(__nv_bfloat16);
  G3C_CUDA(cudaMemcpyAsync(xtilde, h->lat_xtilde, bytes, cudaMemcpyDeviceToDevice, st));
  G3C_CUDA(cudaMemcpyAsync(xin, h->lat_xin, bytes, cudaMemcpyDeviceToDevice, st));
  G3C_CUDA(cudaMemcpyAsync(oc, h->step_oc, bytes, cudaMemcpyDeviceToDevice, st));
  G3C_CUDA(cudaMemcpyAsync(ou, h->step_ou, bytes, cudaMemcpyDeviceToDevice, st));
  return G3C_OK;
}

int g3c_dit_cp_region(g3c_dit_t* h, void** base, int64_t* off_k2, int64_t* off_vt2, int64_t* off_flags) {
  G3C_REQUIRE(h && base && off_k2 && off_vt2 && off_flags, "dit_cp_region: null argument");
  if (!h->cp_region) {
    set_error("dit_cp_region: no context-parallel region (enable_cp without NCCL id, then set_shape)");
    return G3C_ESTATE;
  }
  *base = h->cp_region;
  for (int s = 0; s < 2; ++s) {
    off_k2[s] = (int64_t)h->off_k[s];
    off_vt2[s] = (int64_t)h->off_vt[s];
  }
  *off_flags = (int64_t)h->off_flags;
  return G3C_OK;
}

int g3c_dit_cp_attach(g3c_dit_t* h, const void* const* bases, int n) {
  G3C_REQUIRE(h && bases, "dit_cp_attach: null argument");
  if (!h->cp_region) {
    set_error("dit_cp_attach: no context-parallel region (enable_cp without NCCL id, then set_shape)");
    return G3C_ESTATE;
  }
  if (h->peers_open && !h->peers_attached) {
    set_error("dit_cp_attach: the peers' regions are already imported (g3c_dit_cp_import)");
    return G3C_ESTATE;
  }
  G3C_REQUIRE(n == h->cp_size, "dit_cp_attach: need one region per rank (%d), got %d", h->cp_size, n);
  for (int r = 0; r < n; ++r) G3C_REQUIRE(bases[r], "dit_cp_attach: null region of rank %d", r);
  G3C_REQUIRE(bases[h->cp_rank] == h->cp_region, "dit_cp_attach: entry %d must be this handle's own region",
              h->cp_rank);
  for (int r = 0; r < n; ++r) h->peer_base[r] = const_cast<void*>(bases[r]);
  h->peers_attached = true;
  h->peers_open = true;
  return G3C_OK;
}

int g3c_dit_cfg_region(g3c_dit_t* h, void** base, int64_t* slot_bytes) {
  G3C_REQUIRE(h && base && slot_bytes, "dit_cfg_region: null argument");
  if (!h->cfg_region) {
    set_error("dit_cfg_region: no exchange region (enable_cfg_parallel, then set_shape)");
    return G3C_ESTATE;
  }
  *base = h->cfg_region;
  *slot_bytes = (int64_t)h->cfg_slot_bytes;
  return G3C_OK;
}

int g3c_dit_cfg_attach(g3c_dit_t* h, const void* partner_base) {
  G3C_REQUIRE(h && partner_base, "dit_cfg_attach: null argument");
  if (!h->cfg_region) {
    set_error("dit_cfg_attach: no exchange region (enable_cfg_parallel, then set_shape)");
    return G3C_ESTATE;
  }
  if (h->cfg_peer && !h->cfg_attached) {
    set_error("dit_cfg_attach: the partner's region is already imported (g3c_dit_cfg_import)");
    return G3C_ESTATE;
  }
  h->cfg_peer = const_cast<void*>(partner_base);
  h->cfg_attached = true;
  return G3C_OK;
}

}  // extern "C"
