// Path R — 3D-cache render: project cached world points into the target camera, depth-weighted
// bilinear (4-corner) splat with fp32 vector atomics into a padded accumulation buffer, normalise.
//
// Re-designed from the arithmetic of the reference (cited per function), not from its op graph:
//   reference: cosmos_predict1/diffusion/inference/forward_warp_utils_pytorch.py
//     project_points      :462-486     forward_warp (depth1=None branch) :219-250,281-284
//     bilinear_splatting  :576-695     create_grid :697-703     unproject_points :410-460
//     reliable_depth_mask_range_batch :338-353
//   reference: cosmos_predict1/diffusion/inference/cache_3d.py  render_cache :151-236
//
// Three passes over a batch of items that stays L2-resident:
//   pass 1  k_project_max : z = (K·(w2c·[p;1])).z ; per-group max of log1p(max(z,0))  (warp
//                           shuffle + block reduce + one atomicMax per block)
//   pass 2  k_splat       : recompute the projection (cheaper than a round trip through HBM),
//                           4 x red.global.add.v4.f32 {r*w, g*w, b*w, w} per source pixel
//   pass 3  k_normalise   : crop the 1-px ring, acc/w, fill, clamp, write planar outputs
// HBM-bound by design: algorithmic traffic 44 B/px (SURVEY.md §8d).
#include "common.cuh"

namespace g3c {

struct Cam {
  float w[12];  // first three rows of w2c
  float k[9];
};

__device__ __forceinline__ Cam load_cam(const float* __restrict__ w2c, const float* __restrict__ K) {
  Cam c;
#pragma unroll
  for (int i = 0; i < 12; ++i) c.w[i] = __ldg(w2c + i);
#pragma unroll
  for (int i = 0; i < 9; ++i) c.k[i] = __ldg(K + i);
  return c;
}

// q = K · (w2c · [p;1])[:3]   — explicit rounding order so that pass 1 and pass 2 agree bit for bit
// (reference: project_points :469-479)
__device__ __forceinline__ void project(const Cam& c, float px, float py, float pz, float& qx,
                                        float& qy, float& qz) {
  float cx = __fadd_rn(__fmaf_rn(c.w[2], pz, __fmaf_rn(c.w[1], py, __fmul_rn(c.w[0], px))), c.w[3]);
  float cy = __fadd_rn(__fmaf_rn(c.w[6], pz, __fmaf_rn(c.w[5], py, __fmul_rn(c.w[4], px))), c.w[7]);
  float cz = __fadd_rn(__fmaf_rn(c.w[10], pz, __fmaf_rn(c.w[9], py, __fmul_rn(c.w[8], px))), c.w[11]);
  qx = __fmaf_rn(c.k[2], cz, __fmaf_rn(c.k[1], cy, __fmul_rn(c.k[0], cx)));
  qy = __fmaf_rn(c.k[5], cz, __fmaf_rn(c.k[4], cy, __fmul_rn(c.k[3], cx)));
  qz = __fmaf_rn(c.k[8], cz, __fmaf_rn(c.k[7], cy, __fmul_rn(c.k[6], cx)));
}

// Destination indices and clamped position of one source pixel.
// reference: bilinear_splatting :605-621 — floor/ceil are taken BEFORE clamping the position;
// all three are clamped to x in [0, W+1], y in [0, H+1].
struct SplatIdx {
  int fx, fy, cx, cy;
  float px, py;  // clamped positions
};
__device__ __forceinline__ SplatIdx splat_indices(float flow_x, float flow_y, int x, int y, int W,
                                                  int H) {
  SplatIdx s;
  float pos_x = __fadd_rn(__fadd_rn(flow_x, (float)x), 1.0f);
  float pos_y = __fadd_rn(__fadd_rn(flow_y, (float)y), 1.0f);
  float wmax = (float)(W + 1), hmax = (float)(H + 1);
  // fmaxf(NaN, 0) = 0: NaN coordinates land on the cropped border, as torch's GPU float->long does
  s.fx = (int)fminf(fmaxf(floorf(pos_x), 0.0f), wmax);
  s.cx = (int)fminf(fmaxf(ceilf(pos_x), 0.0f), wmax);
  s.fy = (int)fminf(fmaxf(floorf(pos_y), 0.0f), hmax);
  s.cy = (int)fminf(fmaxf(ceilf(pos_y), 0.0f), hmax);
  s.px = fminf(fmaxf(pos_x, 0.0f), wmax);
  s.py = fminf(fmaxf(pos_y, 0.0f), hmax);
  return s;
}

// fmaxf(NaN, 0) = 0: a NaN depth contributes log-depth 0, so it never reaches the group max.  Such a source also fails
// q_z > 0 and splats with weight 0: a NaN point is dropped, like a point behind the camera.  (The reference's
// torch.clamp / torch.max would propagate it and turn every weight of the chunk into NaN.)  +Inf gives +Inf.
__device__ __forceinline__ float log_depth(float z) { return log1pf(fmaxf(z, 0.0f)); }

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"l"(addr), "f"(a), "f"(b),
               "f"(c), "f"(d)
               : "memory");
}

// lz >= 0 (log_depth never returns NaN), so the int ordering of the bit pattern equals the float ordering.
__device__ __forceinline__ void block_atomic_max(float v, float* dst) {
  __shared__ float red[32];
  v = warp_max(v);
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    int nw = (blockDim.x + 31) >> 5;
    float m = lane < nw ? red[lane] : 0.0f;
    m = warp_max(m);
    if (lane == 0) atomicMax(reinterpret_cast<int*>(dst), __float_as_int(m));
  }
}

// ------------------------------------------------------------------------------------------------
// pass 1: per-group max of log1p(max(z,0))
// item i: camera index cam_of(i) = i / N ; source index = src_bcast ? (i/(N*F))*N + i%N : i
// ------------------------------------------------------------------------------------------------
struct ItemMap {
  int N;          // buffers per camera
  int F;          // cameras (target frames) per batch element
  int src_bcast;  // 1: cache has a single frame broadcast over F targets
  int item0;      // first item of the current pass (foreground pass: blockIdx.y counts from here)
  __host__ __device__ __forceinline__ int cam(int i) const { return (i + item0) / N; }
  __host__ __device__ __forceinline__ int src(int i) const {
    const int j = i + item0;
    return src_bcast ? (j / (N * F)) * N + (j % N) : j;
  }
};

__global__ void __launch_bounds__(256) k_project_max(const float* __restrict__ points,
                                                    const float* __restrict__ w2c,
                                                    const float* __restrict__ K, ItemMap map,
                                                    int item0, int HW, int group, float* gmax) {
  int item = item0 + blockIdx.y;
  Cam c = load_cam(w2c + 16 * map.cam(item), K + 9 * map.cam(item));
  const float* p = points + (size_t)map.src(item) * HW * 3;
  float m = 0.0f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
    float qx, qy, qz;
    project(c, p[3 * i], p[3 * i + 1], p[3 * i + 2], qx, qy, qz);
    float lz = log_depth(qz);
    m = (lz > m || lz != lz) ? lz : m;  // lz is never NaN (log_depth drops NaN depths)
  }
  block_atomic_max(m, gmax + item / group);
}

// Broadcast cache frame (src_frames == 1: every target camera of a batch element renders the same N source frames): all
// F cameras in ONE pass over the points.  A thread keeps 4 points in registers and evaluates the projected depth for
// camera after camera (uniform loads of the 21 camera floats); per camera: warp max -> shared-memory atomicMax, at the
// end one global atomicMax per camera and block.  The separate per-item pass above re-read the 10.8 MB point cloud once
// per target frame (121 x): 372 us -> ~20 us for the 121-frame render.
constexpr int PM_MAX_CAM = 512;
__global__ void __launch_bounds__(256)
    k_project_max_bcast(const float* __restrict__ points, const float* __restrict__ w2c, const float* __restrict__ K,
                        int N, int F, int HW, int group, float* gmax) {
  __shared__ float smax[PM_MAX_CAM];
  const int srcidx = blockIdx.y;           // (b, n)
  const int b = srcidx / N, n = srcidx - b * N;
  for (int f = threadIdx.x; f < F; f += blockDim.x) smax[f] = 0.0f;
  __syncthreads();
  const float* p = points + (size_t)srcidx * HW * 3;
  float px[4], py[4], pz[4];
  int cnt = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW && cnt < 4; i += gridDim.x * blockDim.x, ++cnt) {
    px[cnt] = p[3 * i]; py[cnt] = p[3 * i + 1]; pz[cnt] = p[3 * i + 2];
  }
  for (int f = 0; f < F; ++f) {
    const int cam = b * F + f;
    const Cam c = load_cam(w2c + 16 * cam, K + 9 * cam);
    float m = 0.0f;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (j < cnt) {
        float qx, qy, qz;
        project(c, px[j], py[j], pz[j], qx, qy, qz);
        const float lz = log_depth(qz);
        m = (lz > m || lz != lz) ? lz : m;  // lz is never NaN (log_depth drops NaN depths)
      }
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(&smax[f]), __float_as_int(m));
  }
  __syncthreads();
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    const int item = (b * F + f) * N + n;
    atomicMax(reinterpret_cast<int*>(gmax + item / group), __float_as_int(smax[f]));
  }
}

__global__ void __launch_bounds__(256) k_depth_max(const float* __restrict__ depth, size_t n,
                                                  float* gmax) {
  float m = 0.0f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x) {
    float lz = log_depth(depth[i]);
    m = (lz > m || lz != lz) ? lz : m;
  }
  block_atomic_max(m, gmax);
}

// ------------------------------------------------------------------------------------------------
// pass 2: splat.  acc: [items_in_pass][H+2][W+2][4] = {c0*w, c1*w, c2*w, w};  accz: [..][H+2][W+2]
// ------------------------------------------------------------------------------------------------
// The reference's splat weights of the nw, sw, ne, se corners (:623-646), IEEE divisions, expf and log1pf.
__device__ __forceinline__ void corner_weights(const SplatIdx& s, float z, float lz_max, float mask, float& w_nw,
                                               float& w_sw, float& w_ne, float& w_se) {
  // reference :623-634
  float dyf = __fsub_rn(1.0f, __fsub_rn(s.py, (float)s.fy));
  float dyc = __fsub_rn(1.0f, __fsub_rn((float)s.cy, s.py));
  float dxf = __fsub_rn(1.0f, __fsub_rn(s.px, (float)s.fx));
  float dxc = __fsub_rn(1.0f, __fsub_rn((float)s.cx, s.px));
  // reference :638-646
  float lz = log_depth(z);
  float e = __fmul_rn(__fdiv_rn(lz, __fadd_rn(lz_max, 1e-7f)), 50.0f);
  e = fminf(e, 80.0f);
  float dw = __fadd_rn(expf(e), 1e-7f);
  w_nw = __fdiv_rn(__fmul_rn(__fmul_rn(dyf, dxf), mask), dw);
  w_sw = __fdiv_rn(__fmul_rn(__fmul_rn(dyc, dxf), mask), dw);
  w_ne = __fdiv_rn(__fmul_rn(__fmul_rn(dyf, dxc), mask), dw);
  w_se = __fdiv_rn(__fmul_rn(__fmul_rn(dyc, dxc), mask), dw);
}

__device__ __forceinline__ void splat_pixel(float* __restrict__ acc, float* __restrict__ accz,
                                            const SplatIdx& s, float z, float lz_max, float mask,
                                            float v0, float v1, float v2, int W) {
  float w_nw, w_sw, w_ne, w_se;
  corner_weights(s, z, lz_max, mask, w_nw, w_sw, w_ne, w_se);
  const int Wp = W + 2;
  size_t i_nw = (size_t)s.fy * Wp + s.fx, i_sw = (size_t)s.cy * Wp + s.fx;
  size_t i_ne = (size_t)s.fy * Wp + s.cx, i_se = (size_t)s.cy * Wp + s.cx;
  // a zero weight adds +0 to every slot: skip the atomics (identical result for finite inputs)
  if (w_nw != 0.0f) red_add_v4(acc + 4 * i_nw, v0 * w_nw, v1 * w_nw, v2 * w_nw, w_nw);
  if (w_sw != 0.0f) red_add_v4(acc + 4 * i_sw, v0 * w_sw, v1 * w_sw, v2 * w_sw, w_sw);
  if (w_ne != 0.0f) red_add_v4(acc + 4 * i_ne, v0 * w_ne, v1 * w_ne, v2 * w_ne, w_ne);
  if (w_se != 0.0f) red_add_v4(acc + 4 * i_se, v0 * w_se, v1 * w_se, v2 * w_se, w_se);
  if (accz) {
    if (w_nw != 0.0f) atomicAdd(accz + i_nw, z * w_nw);
    if (w_sw != 0.0f) atomicAdd(accz + i_sw, z * w_sw);
    if (w_ne != 0.0f) atomicAdd(accz + i_ne, z * w_ne);
    if (w_se != 0.0f) atomicAdd(accz + i_se, z * w_se);
  }
}

__global__ void __launch_bounds__(256)
    k_splat_points(const float* __restrict__ points, const float* __restrict__ image,
                   const float* __restrict__ mask, const float* __restrict__ w2c,
                   const float* __restrict__ K, ItemMap map, int item0, int C, int H, int W,
                   int group, const float* __restrict__ gmax, float* __restrict__ acc,
                   float* __restrict__ accz, float* __restrict__ flow_out) {
  const int HW = H * W;
  int item = item0 + blockIdx.y;
  int src = map.src(item);
  Cam c = load_cam(w2c + 16 * map.cam(item), K + 9 * map.cam(item));
  const float* p = points + (size_t)src * HW * 3;
  const float* img = image + (size_t)src * C * HW;
  const float* msk = mask ? mask + (size_t)src * HW : nullptr;
  float lz_max = gmax[item / group];
  float* a = acc + (size_t)blockIdx.y * (H + 2) * (W + 2) * 4;
  float* az = accz ? accz + (size_t)blockIdx.y * (H + 2) * (W + 2) : nullptr;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
    int y = i / W, x = i - y * W;
    float qx, qy, qz;
    project(c, p[3 * i], p[3 * i + 1], p[3 * i + 2], qx, qy, qz);
    // reference forward_warp :244-250
    float m = (msk ? msk[i] : 1.0f) * (qz > 0.0f ? 1.0f : 0.0f);
    float den = __fadd_rn(qz, 1e-7f);
    float fx = __fsub_rn(__fdiv_rn(qx, den), (float)x);
    float fy = __fsub_rn(__fdiv_rn(qy, den), (float)y);
    if (flow_out) {
      flow_out[((size_t)item * 2) * HW + i] = fx;
      flow_out[((size_t)item * 2 + 1) * HW + i] = fy;
    }
    SplatIdx s = splat_indices(fx, fy, x, y, W, H);
    float v0 = img[i], v1 = C > 1 ? img[HW + i] : 0.0f, v2 = C > 2 ? img[2 * HW + i] : 0.0f;
    splat_pixel(a, az, s, qz, lz_max, m, v0, v1, v2, W);
  }
}

// ---- fast variant (default): 4 consecutive source pixels per thread, merged destinations, cheaper weight arithmetic ----
// The round-1 kernel was issue / atomic bound (ncu: XU 42 %, L2 47 %, DRAM 17 %): 7 IEEE divisions + expf + log1pf per
// pixel and 4 vector reds.  Here:
//  * per pixel 2 IEEE divisions (the projected coordinates: their floor / ceil pick the destination, kept exact), one
//    LG2, one EX2, one RCP: dw = exp(50 lz / lzmax) is inverted once (rcp.approx, 1 ulp) and multiplies the four
//    bilinear weights; 50 / (lzmax + 1e-7) is a per-item constant; log1p(z) = lg2(1 + z) ln 2 — its absolute error is
//    multiplied by 50 / lzmax, so a weight's relative error grows as the depth range shrinks (1.2e-4 derived at depths
//    of 0.02, DESIGN.md §3.4); tests/test_render_edges_gpu.py holds every pixel to the bound that follows;
//  * a thread walks 4 neighbouring source pixels of one row and keeps one pending destination per output row in
//    registers: under a smooth warp the north-east corner of pixel j is the north-west corner of pixel j+1, so a thread
//    issues ~10 vector reds for 4 pixels instead of 16 (contributions to the same texel are added in registers first).
struct Pending {
  long long idx;  // texel index in the padded accumulator, -1 = empty
  float a, b, c, w, z;
};
__device__ __forceinline__ void pend_flush(const Pending& p, float* __restrict__ acc, float* __restrict__ accz) {
  if (p.idx >= 0) {
    red_add_v4(acc + 4 * p.idx, p.a, p.b, p.c, p.w);
    if (accz) atomicAdd(accz + p.idx, p.z);
  }
}
__device__ __forceinline__ void pend_add(Pending& p, long long idx, float wt, float v0, float v1, float v2, float z,
                                         float* __restrict__ acc, float* __restrict__ accz) {
  if (wt == 0.0f) return;  // a zero weight adds +0 to every slot (identical result for finite inputs)
  if (idx == p.idx) {
    p.a += v0 * wt; p.b += v1 * wt; p.c += v2 * wt; p.w += wt; p.z += z * wt;
  } else {
    pend_flush(p, acc, accz);
    p.idx = idx; p.a = v0 * wt; p.b = v1 * wt; p.c = v2 * wt; p.w = wt; p.z = z * wt;
  }
}
__device__ __forceinline__ float ex2_fast(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(256)
    k_splat_points4(const float* __restrict__ points, const float* __restrict__ image,
                    const float* __restrict__ mask, const float* __restrict__ w2c,
                    const float* __restrict__ K, ItemMap map, int item0, int C, int H, int W,
                    int group, const float* __restrict__ gmax, float* __restrict__ acc,
                    float* __restrict__ accz, float* __restrict__ flow_out) {
  const int HW = H * W, Wq = W >> 2, nq = H * Wq;
  const int item = item0 + blockIdx.y;
  const int src = map.src(item);
  const Cam c = load_cam(w2c + 16 * map.cam(item), K + 9 * map.cam(item));
  const float4* p4 = reinterpret_cast<const float4*>(points + (size_t)src * HW * 3);
  const float* img = image + (size_t)src * C * HW;
  const float* msk = mask ? mask + (size_t)src * HW : nullptr;
  const float escale = __fdiv_rn(50.0f, __fadd_rn(gmax[item / group], 1e-7f));
  float* a = acc + (size_t)blockIdx.y * (H + 2) * (W + 2) * 4;
  float* az = accz ? accz + (size_t)blockIdx.y * (H + 2) * (W + 2) : nullptr;
  const int Wp = W + 2;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x) {
    const int y = q / Wq, x0 = (q - y * Wq) * 4;
    const int i0 = y * W + x0;
    // 4 points = 12 floats = 3 aligned float4 (i0 is a multiple of 4)
    const float4 pa = p4[(i0 * 3) / 4], pb = p4[(i0 * 3) / 4 + 1], pc = p4[(i0 * 3) / 4 + 2];
    const float px[4] = {pa.x, pa.w, pb.z, pc.y}, py[4] = {pa.y, pb.x, pb.w, pc.z}, pz[4] = {pa.z, pb.y, pc.x, pc.w};
    const float4 r4 = *reinterpret_cast<const float4*>(img + i0);
    const float4 g4 = C > 1 ? *reinterpret_cast<const float4*>(img + HW + i0) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 b4 = C > 2 ? *reinterpret_cast<const float4*>(img + 2 * HW + i0) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 m4 = msk ? *reinterpret_cast<const float4*>(msk + i0) : make_float4(1.f, 1.f, 1.f, 1.f);
    const float v0[4] = {r4.x, r4.y, r4.z, r4.w}, v1[4] = {g4.x, g4.y, g4.z, g4.w}, v2[4] = {b4.x, b4.y, b4.z, b4.w};
    const float mk[4] = {m4.x, m4.y, m4.z, m4.w};
    Pending top{-1, 0.f, 0.f, 0.f, 0.f, 0.f}, bot{-1, 0.f, 0.f, 0.f, 0.f, 0.f};
    float fxs[4], fys[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int x = x0 + j;
      float qx, qy, qz;
      project(c, px[j], py[j], pz[j], qx, qy, qz);
      const float m = mk[j] * (qz > 0.0f ? 1.0f : 0.0f);
      const float den = __fadd_rn(qz, 1e-7f);
      const float fx = __fsub_rn(__fdiv_rn(qx, den), (float)x);
      const float fy = __fsub_rn(__fdiv_rn(qy, den), (float)y);
      fxs[j] = fx;
      fys[j] = fy;
      const SplatIdx s = splat_indices(fx, fy, x, y, W, H);
      const float dyf = __fsub_rn(1.0f, __fsub_rn(s.py, (float)s.fy));
      const float dyc = __fsub_rn(1.0f, __fsub_rn((float)s.cy, s.py));
      const float dxf = __fsub_rn(1.0f, __fsub_rn(s.px, (float)s.fx));
      const float dxc = __fsub_rn(1.0f, __fsub_rn((float)s.cx, s.px));
      const float zc = fmaxf(qz, 0.0f);
      const float lz = __log2f(1.0f + zc) * 0.6931471805599453f;
      const float e = fminf(lz * escale, 80.0f);
      // m / (exp(e) + 1e-7); a NaN depth has m = 0 and zc = 0, so its weights are 0 (dropped, as in log_depth)
      const float rdw = m * rcp_approx(__fadd_rn(ex2_fast(e * 1.4426950408889634f), 1e-7f));
      const long long rt = (long long)s.fy * Wp, rb = (long long)s.cy * Wp;
      pend_add(top, rt + s.fx, dyf * dxf * rdw, v0[j], v1[j], v2[j], qz, a, az);
      pend_add(top, rt + s.cx, dyf * dxc * rdw, v0[j], v1[j], v2[j], qz, a, az);
      pend_add(bot, rb + s.fx, dyc * dxf * rdw, v0[j], v1[j], v2[j], qz, a, az);
      pend_add(bot, rb + s.cx, dyc * dxc * rdw, v0[j], v1[j], v2[j], qz, a, az);
    }
    pend_flush(top, a, az);
    pend_flush(bot, a, az);
    if (flow_out) {
      *reinterpret_cast<float4*>(flow_out + ((size_t)item * 2) * HW + i0) = make_float4(fxs[0], fxs[1], fxs[2], fxs[3]);
      *reinterpret_cast<float4*>(flow_out + ((size_t)item * 2 + 1) * HW + i0) = make_float4(fys[0], fys[1], fys[2], fys[3]);
    }
  }
}

__global__ void __launch_bounds__(256)
    k_splat_flow(const float* __restrict__ frame, const float* __restrict__ mask,
                 const float* __restrict__ depth, const float* __restrict__ flow, int item0, int C,
                 int H, int W, const float* __restrict__ gmax, float* __restrict__ acc) {
  const int HW = H * W;
  int item = item0 + blockIdx.y;
  const float* img = frame + (size_t)item * C * HW;
  float lz_max = gmax[0];
  float* a = acc + (size_t)blockIdx.y * (H + 2) * (W + 2) * 4;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
    int y = i / W, x = i - y * W;
    float fx = flow[((size_t)item * 2) * HW + i], fy = flow[((size_t)item * 2 + 1) * HW + i];
    float m = mask ? mask[(size_t)item * HW + i] : 1.0f;
    SplatIdx s = splat_indices(fx, fy, x, y, W, H);
    float v0 = img[i], v1 = C > 1 ? img[HW + i] : 0.0f, v2 = C > 2 ? img[2 * HW + i] : 0.0f;
    splat_pixel(a, nullptr, s, depth[(size_t)item * HW + i], lz_max, m, v0, v1, v2, W);
  }
}

__global__ void __launch_bounds__(256)
    k_splat_indices(const float* __restrict__ flow, int H, int W, int32_t* __restrict__ idx) {
  const int HW = H * W;
  int item = blockIdx.y;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
    int y = i / W, x = i - y * W;
    SplatIdx s = splat_indices(flow[((size_t)item * 2) * HW + i],
                               flow[((size_t)item * 2 + 1) * HW + i], x, y, W, H);
    int32_t* o = idx + (size_t)item * 4 * HW;
    o[i] = s.fx;
    o[HW + i] = s.fy;
    o[2 * HW + i] = s.cx;
    o[3 * HW + i] = s.cy;
  }
}

// ------------------------------------------------------------------------------------------------
// pass 2, ordered (torch.use_deterministic_algorithms): the splat of ONE item without float atomics, bitwise
// reproducible.  Every (source pixel, corner) pair is a record with id = corner * HW + source (corners nw, sw, ne, se
// = 0..3) and key = its interior destination texel.  A stable LSD radix sort of (key, id) lists each texel's records
// in ascending id, i.e. corner-major, then source row-major: the order of the reference's index_put_(accumulate=True)
// under the deterministic flag (and of a sequential np.add.at).  One thread per texel then recomputes its records'
// contributions and sums them sequentially in fp32 from 0.  Records with weight 0 or a destination in the cropped
// 1-px ring change no output for finite inputs and are dropped by the key pass.  Integer shared-memory atomics only
// count; every rank that decides an order comes from __match_any_sync / popc in warp, lane and block order.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t RS_NONE = 0xFFFFFFFFu;  // dropped record
constexpr int RS_BITS = 10, RS_DIGITS = 1 << RS_BITS;
constexpr int RS_THREADS = 256, RS_WARPS = RS_THREADS / 32, RS_PER_THREAD = 16;
constexpr int RS_TILE = RS_THREADS * RS_PER_THREAD;  // a warp ranks 32 * RS_PER_THREAD consecutive records
constexpr int DET_BATCH = 8;                         // records whose contributions one thread computes at once

// One item's splat inputs: projected points (forward_warp, render_cache) or a given flow (bilinear_splatting).
struct DetItem {
  const float* points;  // [HW][3], or NULL: flow / depth given
  const float* w2c;     // [4][4] and [3][3] target camera (points only)
  const float* K;
  const float* flow;    // [2][HW] (flow only)
  const float* depth;   // [HW] (flow only)
  const float* image;   // [C][HW]
  const float* mask;    // [HW] or NULL
  const float* lz_max;  // the item's log-depth max
  int C, H, W;
};

struct DetSrc {
  float fx, fy, z, m, v0, v1, v2;
};

// the per-source arithmetic of k_splat_points (reference forward_warp :244-250) / k_splat_flow
__device__ __forceinline__ DetSrc det_load(const DetItem& a, const Cam& c, int i) {
  const int HW = a.H * a.W, y = i / a.W, x = i - y * a.W;
  DetSrc s;
  if (a.points) {
    float qx, qy, qz;
    project(c, a.points[3 * i], a.points[3 * i + 1], a.points[3 * i + 2], qx, qy, qz);
    s.m = (a.mask ? a.mask[i] : 1.0f) * (qz > 0.0f ? 1.0f : 0.0f);
    const float den = __fadd_rn(qz, 1e-7f);
    s.fx = __fsub_rn(__fdiv_rn(qx, den), (float)x);
    s.fy = __fsub_rn(__fdiv_rn(qy, den), (float)y);
    s.z = qz;
  } else {
    s.fx = a.flow[i];
    s.fy = a.flow[HW + i];
    s.z = a.depth[i];
    s.m = a.mask ? a.mask[i] : 1.0f;
  }
  s.v0 = a.image[i];
  s.v1 = a.C > 1 ? a.image[HW + i] : 0.0f;
  s.v2 = a.C > 2 ? a.image[2 * HW + i] : 0.0f;
  return s;
}

__device__ __forceinline__ Cam det_cam(const DetItem& a) {
  Cam c{};
  if (a.points) c = load_cam(a.w2c, a.K);
  return c;
}

// keys[corner * HW + i] = interior texel (y - 1) * W + (x - 1), or RS_NONE; optionally the flow of each source
__global__ void __launch_bounds__(256) k_det_keys(DetItem a, uint32_t* __restrict__ keys, float* __restrict__ flow_out) {
  const int H = a.H, W = a.W, HW = H * W;
  const Cam c = det_cam(a);
  const float lz_max = *a.lz_max;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
    const int y = i / W, x = i - y * W;
    const DetSrc s = det_load(a, c, i);
    if (flow_out) {
      flow_out[i] = s.fx;
      flow_out[HW + i] = s.fy;
    }
    const SplatIdx si = splat_indices(s.fx, s.fy, x, y, W, H);
    float w[4];
    corner_weights(si, s.z, lz_max, s.m, w[0], w[1], w[2], w[3]);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int ty = (k & 1) ? si.cy : si.fy, tx = (k & 2) ? si.cx : si.fx;
      const bool keep = w[k] != 0.0f && ty >= 1 && ty <= H && tx >= 1 && tx <= W;
      keys[(size_t)k * HW + i] = keep ? (uint32_t)((ty - 1) * W + (tx - 1)) : RS_NONE;
    }
  }
}

__device__ __forceinline__ uint32_t rs_digit(uint32_t key, int shift) {
  return key == RS_NONE ? RS_NONE : (key >> shift) & (RS_DIGITS - 1);
}

// n: the record count, from the host (first pass) or from the device (later passes, after dropping)
__device__ __forceinline__ int rs_count(int n_host, const int* n_dev) { return n_dev ? *n_dev : n_host; }

// hist[digit][block]: records of each digit in each block's tile
__global__ void __launch_bounds__(RS_THREADS)
    k_rs_hist(const uint32_t* __restrict__ keys, int n_host, const int* __restrict__ n_dev, int shift, int nblocks,
              uint32_t* __restrict__ hist) {
  __shared__ uint32_t h[RS_DIGITS];
  for (int d = threadIdx.x; d < RS_DIGITS; d += RS_THREADS) h[d] = 0;
  __syncthreads();
  const int n = rs_count(n_host, n_dev);
  const int lane = threadIdx.x & 31;
  for (int j = threadIdx.x; j < RS_TILE; j += RS_THREADS) {
    const int e = blockIdx.x * RS_TILE + j;
    const uint32_t d = rs_digit(e < n ? keys[e] : RS_NONE, shift);
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    if (d != RS_NONE && lane == __ffs(peers) - 1) atomicAdd(&h[d], (uint32_t)__popc(peers));
  }
  __syncthreads();
  for (int d = threadIdx.x; d < RS_DIGITS; d += RS_THREADS) hist[(size_t)d * nblocks + blockIdx.x] = h[d];
}

// exclusive scan over a block of RS_THREADS threads; *total = the sum of all v
__device__ __forceinline__ uint32_t rs_block_scan(uint32_t v, uint32_t* total) {
  __shared__ uint32_t ws[RS_WARPS];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) ws[w] = x;
  __syncthreads();
  uint32_t before = 0, all = 0;
#pragma unroll
  for (int k = 0; k < RS_WARPS; ++k) {
    before += k < w ? ws[k] : 0u;
    all += ws[k];
  }
  __syncthreads();
  *total = all;
  return before + x - v;
}

// one block per digit: hist[d][*] := exclusive scan over the blocks (block order); dtot[d] = the digit's total
__global__ void __launch_bounds__(RS_THREADS)
    k_rs_rowscan(uint32_t* __restrict__ hist, int nblocks, uint32_t* __restrict__ dtot) {
  uint32_t* row = hist + (size_t)blockIdx.x * nblocks;
  const int per = (nblocks + RS_THREADS - 1) / RS_THREADS;
  const int b0 = min(threadIdx.x * per, nblocks), b1 = min(b0 + per, nblocks);
  uint32_t s = 0;
  for (int b = b0; b < b1; ++b) s += row[b];
  uint32_t total;
  uint32_t run = rs_block_scan(s, &total);
  for (int b = b0; b < b1; ++b) {
    const uint32_t t = row[b];
    row[b] = run;
    run += t;
  }
  if (threadIdx.x == 0) dtot[blockIdx.x] = total;
}

// Stable scatter of one radix pass.  Position = (records of smaller digits) + (records of this digit in earlier
// blocks) + (in earlier warps of this block) + (in earlier 32-record chunks of this warp) + (in lower lanes).
// ids_in == NULL: the first pass, id = position in keys_in.  Block 0 stores the number of records kept in *n_out.
__global__ void __launch_bounds__(RS_THREADS)
    k_rs_scatter(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ ids_in, int n_host,
                 const int* __restrict__ n_dev, int shift, int nblocks, const uint32_t* __restrict__ hist,
                 const uint32_t* __restrict__ dtot, uint32_t* __restrict__ keys_out, uint32_t* __restrict__ ids_out,
                 int* __restrict__ n_out) {
  __shared__ uint32_t wcnt[RS_WARPS][RS_DIGITS];
  __shared__ uint32_t dbase[RS_DIGITS];
  constexpr int DPT = RS_DIGITS / RS_THREADS;
  uint32_t t[DPT], s = 0;
#pragma unroll
  for (int k = 0; k < DPT; ++k) s += (t[k] = dtot[DPT * threadIdx.x + k]);
  uint32_t total;
  uint32_t run = rs_block_scan(s, &total);
#pragma unroll
  for (int k = 0; k < DPT; ++k) {
    dbase[DPT * threadIdx.x + k] = run;
    run += t[k];
  }
  if (n_out && blockIdx.x == 0 && threadIdx.x == 0) *n_out = (int)total;
  for (int d = threadIdx.x; d < RS_WARPS * RS_DIGITS; d += RS_THREADS) (&wcnt[0][0])[d] = 0;
  __syncthreads();
  const int n = rs_count(n_host, n_dev);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const uint32_t lower = (1u << lane) - 1u;
  const int base = blockIdx.x * RS_TILE + w * 32 * RS_PER_THREAD + lane;
  uint32_t key[RS_PER_THREAD], rank[RS_PER_THREAD];
#pragma unroll
  for (int c = 0; c < RS_PER_THREAD; ++c) {
    const int e = base + 32 * c;
    key[c] = e < n ? keys_in[e] : RS_NONE;
    const uint32_t d = rs_digit(key[c], shift);
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    rank[c] = d != RS_NONE ? wcnt[w][d] + __popc(peers & lower) : 0u;
    __syncwarp();
    if (d != RS_NONE && lane == __ffs(peers) - 1) wcnt[w][d] += __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  for (int d = threadIdx.x; d < RS_DIGITS; d += RS_THREADS) {
    uint32_t r = dbase[d] + hist[(size_t)d * nblocks + blockIdx.x];
#pragma unroll
    for (int k = 0; k < RS_WARPS; ++k) {
      const uint32_t c = wcnt[k][d];
      wcnt[k][d] = r;
      r += c;
    }
  }
  __syncthreads();
#pragma unroll
  for (int c = 0; c < RS_PER_THREAD; ++c) {
    const uint32_t d = rs_digit(key[c], shift);
    if (d == RS_NONE) continue;
    const int e = base + 32 * c;
    const uint32_t pos = wcnt[w][d] + rank[c];
    keys_out[pos] = key[c];
    ids_out[pos] = ids_in ? ids_in[e] : (uint32_t)e;
  }
}

// seg[texel] = [first, last + 1) of its records in the sorted keys (seg zeroed beforehand: empty texels stay [0, 0))
__global__ void __launch_bounds__(256)
    k_det_bounds(const uint32_t* __restrict__ keys, const int* __restrict__ n_dev, uint2* __restrict__ seg) {
  const int n = *n_dev;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
    const uint32_t k = keys[p];
    if (p == 0 || keys[p - 1] != k) seg[k].x = p;
    if (p == n - 1 || keys[p + 1] != k) seg[k].y = p + 1;
  }
}

// One thread per interior texel: its records' contributions summed in sorted order, written to the padded acc / accz
// layout k_normalise reads (every interior texel is written, so the planes need no clearing).
__global__ void __launch_bounds__(256)
    k_det_accum(DetItem a, const uint32_t* __restrict__ ids, const uint2* __restrict__ seg, float* __restrict__ acc,
                float* __restrict__ accz) {
  const int H = a.H, W = a.W, HW = H * W;
  const Cam c = det_cam(a);
  const float lz_max = *a.lz_max;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < HW; t += gridDim.x * blockDim.x) {
    const uint2 sg = seg[t];
    float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, sw = 0.0f, sz = 0.0f;
    for (uint32_t p0 = sg.x; p0 < sg.y; p0 += DET_BATCH) {
      // the contributions of a batch are independent: compute them together, add them in order
      float c0[DET_BATCH], c1[DET_BATCH], c2[DET_BATCH], cw[DET_BATCH], cz[DET_BATCH];
#pragma unroll
      for (int j = 0; j < DET_BATCH; ++j) {
        c0[j] = c1[j] = c2[j] = cw[j] = cz[j] = 0.0f;
        if (p0 + j < sg.y) {
          const uint32_t id = ids[p0 + j];
          const int corner = (int)(id / (uint32_t)HW), i = (int)(id - (uint32_t)corner * HW);
          const int y = i / W, x = i - y * W;
          const DetSrc s = det_load(a, c, i);
          const SplatIdx si = splat_indices(s.fx, s.fy, x, y, W, H);
          float w[4];
          corner_weights(si, s.z, lz_max, s.m, w[0], w[1], w[2], w[3]);
          const float wt = corner == 0 ? w[0] : corner == 1 ? w[1] : corner == 2 ? w[2] : w[3];
          c0[j] = __fmul_rn(s.v0, wt);
          c1[j] = __fmul_rn(s.v1, wt);
          c2[j] = __fmul_rn(s.v2, wt);
          cw[j] = wt;
          cz[j] = __fmul_rn(s.z, wt);
        }
      }
#pragma unroll
      for (int j = 0; j < DET_BATCH; ++j)
        if (p0 + j < sg.y) {
          s0 = __fadd_rn(s0, c0[j]);
          s1 = __fadd_rn(s1, c1[j]);
          s2 = __fadd_rn(s2, c2[j]);
          sw = __fadd_rn(sw, cw[j]);
          sz = __fadd_rn(sz, cz[j]);
        }
    }
    const int ty = t / W, tx = t - ty * W;
    const size_t j = (size_t)(ty + 1) * (W + 2) + (tx + 1);
    reinterpret_cast<float4*>(acc)[j] = make_float4(s0, s1, s2, sw);
    if (accz) accz[j] = sz;
  }
}

// ------------------------------------------------------------------------------------------------
// pass 3: crop + normalise (reference :680-695)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    k_normalise(const float* __restrict__ acc, const float* __restrict__ accz, int item0, int C,
                int H, int W, int is_image, float* __restrict__ out, float* __restrict__ mask_out,
                float* __restrict__ depth_out) {
  const int HW = H * W;
  int item = item0 + blockIdx.y;
  const float4* a = reinterpret_cast<const float4*>(acc) + (size_t)blockIdx.y * (H + 2) * (W + 2);
  const float* az = accz ? accz + (size_t)blockIdx.y * (H + 2) * (W + 2) : nullptr;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
    int y = i / W, x = i - y * W;
    size_t j = (size_t)(y + 1) * (W + 2) + (x + 1);
    float4 v = a[j];
    float w = v.w;
    if (w != w) w = 1000.0f;                  // nan_to_num(nan=1000)
    else if (isinf(w)) w = w > 0 ? 3.4028234663852886e38f : -3.4028234663852886e38f;
    bool hit = w > 0.0f;
    float zero = is_image ? -1.0f : 0.0f;
    float o0 = hit ? __fdiv_rn(v.x, w) : zero;
    float o1 = hit ? __fdiv_rn(v.y, w) : zero;
    float o2 = hit ? __fdiv_rn(v.z, w) : zero;
    if (is_image) {
      o0 = fminf(fmaxf(o0, -1.0f), 1.0f);
      o1 = fminf(fmaxf(o1, -1.0f), 1.0f);
      o2 = fminf(fmaxf(o2, -1.0f), 1.0f);
    }
    float* o = out + (size_t)item * C * HW;
    o[i] = o0;
    if (C > 1) o[HW + i] = o1;
    if (C > 2) o[2 * HW + i] = o2;
    if (mask_out) mask_out[(size_t)item * HW + i] = hit ? 1.0f : 0.0f;
    if (depth_out) depth_out[(size_t)item * HW + i] = hit ? __fdiv_rn(az[j], w) : 0.0f;
  }
}

// ------------------------------------------------------------------------------------------------
// unproject (reference :410-460) and the 5x5 reliability mask (:338-353)
// ------------------------------------------------------------------------------------------------
// Inverses in double (Gauss-Jordan with partial pivoting), rounded to fp32 — reference uses
// torch.linalg.inv in fp32 (:147-148); agreement is at fp32 round-off, stated in the tests.
__device__ void invert_small(const float* __restrict__ m, int n, float* __restrict__ out) {
  double a[4][8];
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) {
      a[i][j] = m[i * n + j];
      a[i][n + j] = (i == j) ? 1.0 : 0.0;
    }
  for (int c = 0; c < n; ++c) {
    int piv = c;
    for (int r = c + 1; r < n; ++r)
      if (fabs(a[r][c]) > fabs(a[piv][c])) piv = r;
    if (piv != c)
      for (int j = 0; j < 2 * n; ++j) {
        double t = a[c][j];
        a[c][j] = a[piv][j];
        a[piv][j] = t;
      }
    double d = 1.0 / a[c][c];
    for (int j = 0; j < 2 * n; ++j) a[c][j] *= d;
    for (int r = 0; r < n; ++r)
      if (r != c) {
        double f = a[r][c];
        for (int j = 0; j < 2 * n; ++j) a[r][j] -= f * a[c][j];
      }
  }
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) out[i * n + j] = (float)a[i][n + j];
}

__global__ void __launch_bounds__(256)
    k_unproject(const float* __restrict__ depth, const float* __restrict__ w2c,
                const float* __restrict__ K, const uint8_t* __restrict__ mask, int H, int W,
                int is_depth, float* __restrict__ points) {
  __shared__ float kinv[9];
  __shared__ float c2w[16];
  int item = blockIdx.y;
  if (threadIdx.x == 0) invert_small(K + 9 * item, 3, kinv);
  if (threadIdx.x == 32) invert_small(w2c + 16 * item, 4, c2w);
  __syncthreads();
  const int HW = H * W;
  const float* d = depth + (size_t)item * HW;
  float* out = points + (size_t)item * HW * 3;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
    int y = i / W, x = i - y * W;
    float z = d[i];
    bool valid = mask ? mask[(size_t)item * HW + i] != 0 : z > 0.0f;
    float ox = 0.f, oy = 0.f, oz = 0.f;
    if (valid) {
      float fx = (float)x, fy = (float)y;
      float rx = __fadd_rn(__fmaf_rn(kinv[1], fy, __fmul_rn(kinv[0], fx)), kinv[2]);
      float ry = __fadd_rn(__fmaf_rn(kinv[4], fy, __fmul_rn(kinv[3], fx)), kinv[5]);
      float rz = __fadd_rn(__fmaf_rn(kinv[7], fy, __fmul_rn(kinv[6], fx)), kinv[8]);
      if (!is_depth) {
        float nrm = __fadd_rn(sqrtf(rx * rx + ry * ry + rz * rz), 1e-8f);
        rx = __fdiv_rn(rx, nrm);
        ry = __fdiv_rn(ry, nrm);
        rz = __fdiv_rn(rz, nrm);
      }
      float cx = z * rx, cy = z * ry, cz = z * rz;
      ox = __fadd_rn(__fmaf_rn(c2w[2], cz, __fmaf_rn(c2w[1], cy, __fmul_rn(c2w[0], cx))), c2w[3]);
      oy = __fadd_rn(__fmaf_rn(c2w[6], cz, __fmaf_rn(c2w[5], cy, __fmul_rn(c2w[4], cx))), c2w[7]);
      oz = __fadd_rn(__fmaf_rn(c2w[10], cz, __fmaf_rn(c2w[9], cy, __fmul_rn(c2w[8], cx))), c2w[11]);
    }
    out[3 * i] = ox;
    out[3 * i + 1] = oy;
    out[3 * i + 2] = oz;
  }
}

// max/min pool pad with -inf/+inf (ignored), avg pool pads with zeros and divides by window^2
// (torch defaults: count_include_pad=True).
__global__ void __launch_bounds__(256)
    k_reliable_mask(const float* __restrict__ depth, int H, int W, int win, float thresh, float eps,
                    uint8_t* __restrict__ out) {
  const int HW = H * W;
  int item = blockIdx.y;
  const float* d = depth + (size_t)item * HW;
  int r = win / 2;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
    int y = i / W, x = i - y * W;
    float mx = -INFINITY, mn = INFINITY, sum = 0.0f;
    for (int dy = -r; dy <= r; ++dy) {
      int yy = y + dy;
      if (yy < 0 || yy >= H) continue;
      for (int dx = -r; dx <= r; ++dx) {
        int xx = x + dx;
        if (xx < 0 || xx >= W) continue;
        float v = d[yy * W + xx];
        mx = fmaxf(mx, v);
        mn = fminf(mn, v);
        sum += v;
      }
    }
    float mean = sum / (float)(win * win);
    float ratio = __fdiv_rn(mx - mn, mean + eps);
    out[(size_t)item * HW + i] = (ratio < thresh && d[i] > 0.0f) ? 1 : 0;
  }
}

}  // namespace g3c

// =================================================================================================
// C ABI
// =================================================================================================
using namespace g3c;

struct g3c_render {
  int H, W, max_items;
  float* acc;   // [max_items][H+2][W+2][4]
  float* accz;  // [max_items][H+2][W+2]
  float* gmax;  // per-group maxima
  int gmax_cap;
  // ordered splat (g3c_render_set_deterministic); the workspace is allocated when it is first enabled
  int det;
  uint32_t* rs;         // the one allocation below
  uint32_t* keys[2];    // [4 H W] each: radix sort ping-pong
  uint32_t* ids[2];
  uint32_t* hist;       // [RS_DIGITS][rs_blocks]
  uint32_t* dtot;       // [RS_DIGITS]
  uint2* seg;           // [H W] record range of each texel
  int* count;           // records kept
  int rs_blocks;
};


// ------------------------------------------------------------------------------------------------
// Foreground-masking occlusion pass (SURVEY.md §8f rank 1; reference forward_warp :285-335, points_to_mesh :49-132,
// get_camera_rays :151-168, NVIDIA-Warp kernel ray_triangle_intersection_warp.py:23-105).
// The reference ray-traces every target pixel against every triangle of a 1/4-resolution mesh built around the
// depth-discontinuity pixels.  Here every mesh patch rasterises its own two triangles: the Moeller-Trumbore test is
// only evaluated for the pixels inside the triangle's (conservative) screen bounding box and the nearest hit is an
// atomicMin on the float bits (t > 0, so the unsigned order is the float order) — the same set of (ray, triangle)
// hits, order independent and therefore deterministic.
// ------------------------------------------------------------------------------------------------
struct AxisTap {
  int i0, i1;
  float lam;
};
// F.interpolate(mode="bilinear", align_corners=False) along one axis
__device__ __forceinline__ AxisTap bilinear_tap(int dst, int n_in, int n_out) {
  const float scale = (float)n_in / (float)n_out;
  float src = fmaxf(((float)dst + 0.5f) * scale - 0.5f, 0.0f);
  AxisTap t;
  t.i0 = min((int)floorf(src), n_in - 1);
  t.i1 = min(t.i0 + 1, n_in - 1);
  t.lam = src - (float)t.i0;
  return t;
}

// vertices of the 1/4-resolution mesh: bilinear resample of the camera-space points (w2c . [p;1]) of one item, plus
// the nearest-resampled boundary mask.  verts [item][nh][nw][3], vmask [item][nh][nw]
__global__ void __launch_bounds__(256)
    k_fg_mesh_points(const float* __restrict__ points, const uint8_t* __restrict__ boundary,
                     const float* __restrict__ w2c, ItemMap map, int H, int W, int nh, int nw, float* __restrict__ verts,
                     uint8_t* __restrict__ vmask) {
  const int item = blockIdx.y;
  const float* m = w2c + 16 * map.cam(item);
  const float* p = points + (size_t)map.src(item) * H * W * 3;
  const uint8_t* bm = boundary + (size_t)map.src(item) * H * W;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nh * nw; i += gridDim.x * blockDim.x) {
    const int vy = i / nw, vx = i - vy * nw;
    const AxisTap ty = bilinear_tap(vy, H, nh), tx = bilinear_tap(vx, W, nw);
    float acc[3] = {0.f, 0.f, 0.f};
    const int ys[2] = {ty.i0, ty.i1}, xs[2] = {tx.i0, tx.i1};
    const float wy[2] = {1.0f - ty.lam, ty.lam}, wx[2] = {1.0f - tx.lam, tx.lam};
    float row[2][3];
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      float c[2][3];
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const float* q = p + ((size_t)ys[a] * W + xs[b]) * 3;
        const float px = q[0], py = q[1], pz = q[2];
#pragma unroll
        for (int r = 0; r < 3; ++r)
          c[b][r] = __fadd_rn(__fmaf_rn(m[4 * r + 2], pz, __fmaf_rn(m[4 * r + 1], py, __fmul_rn(m[4 * r], px))), m[4 * r + 3]);
      }
#pragma unroll
      for (int r = 0; r < 3; ++r) row[a][r] = c[0][r] * wx[0] + c[1][r] * wx[1];
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) acc[r] = row[0][r] * wy[0] + row[1][r] * wy[1];
    float* o = verts + ((size_t)item * nh * nw + i) * 3;
    o[0] = acc[0]; o[1] = acc[1]; o[2] = acc[2];
    // mode="nearest": source index floor(dst * in / out)
    const int sy = min((int)floorf((float)vy * ((float)H / (float)nh)), H - 1);
    const int sx = min((int)floorf((float)vx * ((float)W / (float)nw)), W - 1);
    vmask[(size_t)item * nh * nw + i] = bm[(size_t)sy * W + sx] ? 1 : 0;
  }
}

struct Ray {
  float x, y, z;
};
// get_camera_rays :151-168: normalised K^-1 (x, y, 1)
__device__ __forceinline__ Ray camera_ray(const float* __restrict__ kinv, int x, int y) {
  const float fx = (float)x, fy = (float)y;
  float ux = __fadd_rn(__fmaf_rn(kinv[1], fy, __fmul_rn(kinv[0], fx)), kinv[2]);
  float uy = __fadd_rn(__fmaf_rn(kinv[4], fy, __fmul_rn(kinv[3], fx)), kinv[5]);
  float uz = __fadd_rn(__fmaf_rn(kinv[7], fy, __fmul_rn(kinv[6], fx)), kinv[8]);
  float n = sqrtf(ux * ux + uy * uy + uz * uz);
  if (n == 0.0f) n = 1.0f;
  Ray r;
  r.x = ux / n; r.y = uy / n; r.z = uz / n;
  return r;
}

// Moeller-Trumbore for a ray from the origin (the target camera centre); returns t or 0 (ray_triangle_intersection_warp.py:56-105)
__device__ __forceinline__ float ray_tri(const Ray& d, const float* v0, const float* v1, const float* v2, float eps) {
  const float e1x = v1[0] - v0[0], e1y = v1[1] - v0[1], e1z = v1[2] - v0[2];
  const float e2x = v2[0] - v0[0], e2y = v2[1] - v0[1], e2z = v2[2] - v0[2];
  const float hx = d.y * e2z - d.z * e2y, hy = d.z * e2x - d.x * e2z, hz = d.x * e2y - d.y * e2x;
  const float a = e1x * hx + e1y * hy + e1z * hz;
  if (fabsf(a) < eps) return 0.0f;
  const float f = 1.0f / a;
  const float sx = -v0[0], sy = -v0[1], sz = -v0[2];
  const float u = f * (sx * hx + sy * hy + sz * hz);
  if (u < 0.0f || u > 1.0f) return 0.0f;
  const float qx = sy * e1z - sz * e1y, qy = sz * e1x - sx * e1z, qz = sx * e1y - sy * e1x;
  const float v = f * (d.x * qx + d.y * qy + d.z * qz);
  if (v < 0.0f || (u + v) > 1.0f) return 0.0f;
  const float t = f * (e2x * qx + e2y * qy + e2z * qz);
  return t > eps ? t : 0.0f;
}

// one thread per mesh patch (u, v): its two triangles (tl, tr, bl) and (tr, br, bl) when any corner is on the boundary
__global__ void __launch_bounds__(256)
    k_fg_raster(const float* __restrict__ verts, const uint8_t* __restrict__ vmask, const float* __restrict__ K,
                const float* __restrict__ Kinv, ItemMap map, int H, int W, int nh, int nw, uint32_t* __restrict__ tbuf) {
  const int item = blockIdx.y;
  const float* k = K + 9 * map.cam(item);
  const float* kinv = Kinv + 9 * map.cam(item);
  const float* vb = verts + (size_t)item * nh * nw * 3;
  const uint8_t* mb = vmask + (size_t)item * nh * nw;
  uint32_t* tb = tbuf + (size_t)item * H * W;
  const int np = (nh - 1) * (nw - 1);
  for (int pidx = blockIdx.x * blockDim.x + threadIdx.x; pidx < np; pidx += gridDim.x * blockDim.x) {
    const int u = pidx / (nw - 1), v = pidx - u * (nw - 1);
    const int itl = u * nw + v, itr = itl + 1, ibl = itl + nw, ibr = ibl + 1;
    if (!(mb[itl] | mb[itr] | mb[ibl] | mb[ibr])) continue;
    const int tri[2][3] = {{itl, itr, ibl}, {itr, ibr, ibl}};
#pragma unroll 1
    for (int t = 0; t < 2; ++t) {
      const float* v0 = vb + 3 * tri[t][0];
      const float* v1 = vb + 3 * tri[t][1];
      const float* v2 = vb + 3 * tri[t][2];
      // conservative screen bounding box; a vertex at or behind the camera plane makes the whole frame the box
      int x0 = 0, x1 = W - 1, y0 = 0, y1 = H - 1;
      const float zmin = fminf(v0[2], fminf(v1[2], v2[2]));
      if (zmin > 1e-4f) {
        float xmin = 3.0e38f, xmax = -3.0e38f, ymin = 3.0e38f, ymax = -3.0e38f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float* vv = c == 0 ? v0 : (c == 1 ? v1 : v2);
          const float px = (k[0] * vv[0] + k[1] * vv[1] + k[2] * vv[2]) / (k[6] * vv[0] + k[7] * vv[1] + k[8] * vv[2]);
          const float py = (k[3] * vv[0] + k[4] * vv[1] + k[5] * vv[2]) / (k[6] * vv[0] + k[7] * vv[1] + k[8] * vv[2]);
          xmin = fminf(xmin, px); xmax = fmaxf(xmax, px);
          ymin = fminf(ymin, py); ymax = fmaxf(ymax, py);
        }
        if (!(xmax >= -2.0f && ymax >= -2.0f && xmin <= (float)W + 1.0f && ymin <= (float)H + 1.0f)) continue;  // off screen (or NaN)
        x0 = max(0, (int)floorf(xmin) - 1); x1 = min(W - 1, (int)ceilf(xmax) + 1);
        y0 = max(0, (int)floorf(ymin) - 1); y1 = min(H - 1, (int)ceilf(ymax) + 1);
      }
      for (int y = y0; y <= y1; ++y)
        for (int x = x0; x <= x1; ++x) {
          const Ray d = camera_ray(kinv, x, y);
          const float tt = ray_tri(d, v0, v1, v2, 1e-8f);
          if (tt > 0.0f) atomicMin(tb + (size_t)y * W + x, __float_as_uint(tt));
        }
    }
  }
}

// :317-334: mesh z-depth = t * ray_z (the bilinear resample to the same size is the identity), pixels whose mesh depth
// is more than 0.02 in front of the splatted depth are removed from mask / image (fill -1) / depth
__global__ void __launch_bounds__(256)
    k_fg_apply(const uint32_t* __restrict__ tbuf, const float* __restrict__ Kinv, ItemMap map, int C, int H, int W,
               float* __restrict__ warped, float* __restrict__ mask, float* __restrict__ depth) {
  const int item = blockIdx.y;
  const int HW = H * W;
  const float* kinv = Kinv + 9 * map.cam(item);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
    const uint32_t bits = tbuf[(size_t)item * HW + i];
    if (bits >= 0x7F800000u) continue;  // no hit (initialised to 0xFFFFFFFF)
    const int y = i / W, x = i - y * W;
    const float mesh_z = __uint_as_float(bits) * camera_ray(kinv, x, y).z;
    float* dz = depth + (size_t)item * HW + i;
    if (mesh_z > 0.0f && (mesh_z + 0.02f) < *dz) {
      *dz = 0.0f;
      mask[(size_t)item * HW + i] = 0.0f;
      // (warped + 1) * 0 - 1 (:333): -1 whatever the frame holds
      for (int c = 0; c < C; ++c) warped[((size_t)item * C + c) * HW + i] = -1.0f;
    }
  }
}

__global__ void k_fg_invert_k(const float* __restrict__ K, int n, float* __restrict__ Kinv) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) invert_small(K + 9 * i, 3, Kinv + 9 * i);
}

// ------------------------------------------------------------------------------------------------
// Non-rigid depth alignment of Cache3D_Buffer.update_cache (SURVEY.md §8a row R7; reference camera_utils.py:292-345):
// a per-pixel scale map sc, num_iters Adam steps on
//     mean_{p in mask, c} | (R (d_p sc_p r_p) + t)_c - (R (t_p r_p) + t)_c |  +  lambda * mean_p | box3(sc)_p - sc_p |
// The reference runs 100 x (unproject_points twice + autograd + torch.optim.Adam) = ~4 000 ATen launches; the gradient
// is closed form (sign(d_p sc_p - t_p) d_p |R r_p|_1 / 3n  +  lambda (box3(g) - g)/HW, g = sign(box3(sc) - sc)), so one
// stencil kernel per iteration does loss gradient + Adam update.  HBM/L2-resident: 28 B/px per iteration.
// ------------------------------------------------------------------------------------------------
__global__ void k_align_setup(const float* __restrict__ K, const float* __restrict__ c2w, float* __restrict__ mats) {
  // mats[0..8] = K^-1, mats[9..17] = rotation of inverse(c2w) (unproject_points inverts the matrix it is given)
  if (threadIdx.x == 0) {
    float kinv[9], w2c[16];
    invert_small(K, 3, kinv);
    invert_small(c2w, 4, w2c);
    for (int i = 0; i < 9; ++i) mats[i] = kinv[i];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) mats[9 + 3 * r + c] = w2c[4 * r + c];
  }
}

__global__ void __launch_bounds__(256)
    k_align_count(const uint8_t* __restrict__ mask, int HW, unsigned int* __restrict__ count) {
  unsigned int n = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) n += mask[i] ? 1u : 0u;
  n = __reduce_add_sync(0xffffffffu, n);
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(count, n);
}

// coef_p = mask_p ? d_p |R K^-1 (x,y,1)|_1 / (3 n) : 0 ; sc = 1 ; Adam moments = 0
__global__ void __launch_bounds__(256)
    k_align_init(const float* __restrict__ depth, const uint8_t* __restrict__ mask, const float* __restrict__ mats,
                 const unsigned int* __restrict__ count, int H, int W, float* __restrict__ coef, float* __restrict__ sc,
                 float* __restrict__ m1, float* __restrict__ m2) {
  const float inv3n = 1.0f / (3.0f * (float)max(*count, 1u));
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < H * W; i += gridDim.x * blockDim.x) {
    const int y = i / W, x = i - y * W;
    const float fx = (float)x, fy = (float)y;
    const float rx = __fadd_rn(__fmaf_rn(mats[1], fy, __fmul_rn(mats[0], fx)), mats[2]);
    const float ry = __fadd_rn(__fmaf_rn(mats[4], fy, __fmul_rn(mats[3], fx)), mats[5]);
    const float rz = __fadd_rn(__fmaf_rn(mats[7], fy, __fmul_rn(mats[6], fx)), mats[8]);
    float l1 = 0.0f;
#pragma unroll
    for (int r = 0; r < 3; ++r) l1 += fabsf(mats[9 + 3 * r] * rx + mats[10 + 3 * r] * ry + mats[11 + 3 * r] * rz);
    coef[i] = mask[i] ? depth[i] * l1 * inv3n : 0.0f;
    sc[i] = 1.0f;
    m1[i] = 0.0f;
    m2[i] = 0.0f;
  }
}

__device__ __forceinline__ float sign_f(float v) { return v > 0.0f ? 1.0f : (v < 0.0f ? -1.0f : 0.0f); }

constexpr int AL_TX = 32, AL_TY = 8;
__global__ void __launch_bounds__(AL_TX * AL_TY)
    k_align_step(const float* __restrict__ depth, const float* __restrict__ target, const float* __restrict__ coef,
                 const float* __restrict__ sc_in, float* __restrict__ sc_out, float* __restrict__ m1,
                 float* __restrict__ m2, int H, int W, float arap_w, float step_size, float bc2_sqrt) {
  __shared__ float s_sc[AL_TY + 4][AL_TX + 4];
  __shared__ float s_g[AL_TY + 2][AL_TX + 2];
  const int x0 = blockIdx.x * AL_TX, y0 = blockIdx.y * AL_TY;
  const int tid = threadIdx.y * AL_TX + threadIdx.x;
  for (int i = tid; i < (AL_TY + 4) * (AL_TX + 4); i += AL_TX * AL_TY) {
    const int ly = i / (AL_TX + 4), lx = i - ly * (AL_TX + 4);
    const int y = y0 + ly - 2, x = x0 + lx - 2;
    s_sc[ly][lx] = (y >= 0 && y < H && x >= 0 && x < W) ? sc_in[(size_t)y * W + x] : 0.0f;  // conv2d zero padding
  }
  __syncthreads();
  const float ninth = 1.0f / 9.0f;
  for (int i = tid; i < (AL_TY + 2) * (AL_TX + 2); i += AL_TX * AL_TY) {
    const int ly = i / (AL_TX + 2), lx = i - ly * (AL_TX + 2);
    const int y = y0 + ly - 1, x = x0 + lx - 1;
    float g = 0.0f;
    if (y >= 0 && y < H && x >= 0 && x < W) {
      float sm = 0.0f;
#pragma unroll
      for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) sm = __fmaf_rn(s_sc[ly + dy][lx + dx], ninth, sm);
      g = sign_f(sm - s_sc[ly + 1][lx + 1]);
    }
    s_g[ly][lx] = g;
  }
  __syncthreads();
  const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
  if (x >= W || y >= H) return;
  const size_t p = (size_t)y * W + x;
  float bg = 0.0f;
#pragma unroll
  for (int dy = 0; dy < 3; ++dy)
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) bg = __fmaf_rn(s_g[threadIdx.y + dy][threadIdx.x + dx], ninth, bg);
  const float sc = s_sc[threadIdx.y + 2][threadIdx.x + 2];
  const float e = depth[p] * sc - target[p];
  const float grad = coef[p] * sign_f(e) + arap_w * (bg - s_g[threadIdx.y + 1][threadIdx.x + 1]);
  // torch.optim.Adam (betas .9/.999, eps 1e-8, no weight decay)
  const float a = 0.9f * m1[p] + 0.1f * grad;
  const float b = 0.999f * m2[p] + 0.001f * grad * grad;
  m1[p] = a;
  m2[p] = b;
  sc_out[p] = sc - step_size * a / (sqrtf(b) / bc2_sqrt + 1e-8f);
}

__global__ void __launch_bounds__(256)
    k_align_finish(const float* __restrict__ depth, const float* __restrict__ sc, int HW, float* __restrict__ out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) out[i] = depth[i] * sc[i];
}

static inline dim3 px_grid(int HW, int items) {
  int bx = (HW + 255) / 256;
  int cap = 4 * sm_count();
  if (bx > cap) bx = cap;
  return dim3(bx, items);
}

extern "C" {

int g3c_render_create(int H, int W, int max_items_per_pass, g3c_render_t** out) {
  G3C_REQUIRE(H > 0 && W > 0 && max_items_per_pass > 0 && out, "render_create: bad arguments");
  g3c_render* r = new g3c_render();
  r->H = H;
  r->W = W;
  r->max_items = max_items_per_pass;
  r->gmax_cap = 4096;
  size_t plane = (size_t)(H + 2) * (W + 2);
  cudaError_t e = cudaMalloc(&r->acc, plane * 4 * sizeof(float) * max_items_per_pass);
  if (e == cudaSuccess) e = cudaMalloc(&r->accz, plane * sizeof(float) * max_items_per_pass);
  if (e == cudaSuccess) e = cudaMalloc(&r->gmax, sizeof(float) * r->gmax_cap);
  if (e != cudaSuccess) {
    delete r;
    return cuda_fail(e, "cudaMalloc(render workspace)", __FILE__, __LINE__);
  }
  *out = r;
  return G3C_OK;
}

int g3c_render_destroy(g3c_render_t* r) {
  if (!r) return G3C_OK;
  cudaFree(r->acc);
  cudaFree(r->accz);
  cudaFree(r->gmax);
  cudaFree(r->rs);
  delete r;
  return G3C_OK;
}

int g3c_render_set_deterministic(g3c_render_t* r, int on) {
  G3C_REQUIRE(r, "render_set_deterministic: null handle");
  if (on && !r->rs) {
    const size_t HW = (size_t)r->H * r->W, n4 = 4 * HW;
    G3C_REQUIRE(n4 <= (size_t)INT32_MAX, "render_set_deterministic: %d x %d frames are too large", r->H, r->W);
    const int blocks = (int)((n4 + RS_TILE - 1) / RS_TILE);
    // keys x2 | ids x2 | hist | dtot | seg | count (every part starts at an even word: seg is 8-byte aligned)
    const size_t words = 4 * n4 + (size_t)RS_DIGITS * blocks + RS_DIGITS + 2 * HW + 2;
    uint32_t* buf = nullptr;
    G3C_CUDA(cudaMalloc(&buf, words * sizeof(uint32_t)));
    r->rs = buf;
    r->rs_blocks = blocks;
    r->keys[0] = buf;
    r->keys[1] = buf + n4;
    r->ids[0] = buf + 2 * n4;
    r->ids[1] = buf + 3 * n4;
    r->hist = buf + 4 * n4;
    r->dtot = r->hist + (size_t)RS_DIGITS * blocks;
    r->seg = reinterpret_cast<uint2*>(r->dtot + RS_DIGITS);
    r->count = reinterpret_cast<int*>(r->seg + HW);
  }
  r->det = on ? 1 : 0;
  return G3C_OK;
}

// The ordered splat of one item (k_det_keys .. k_det_accum) into one acc / accz plane.
static int det_splat_item(g3c_render* r, const DetItem& a, float* acc, float* accz, float* flow_out, cudaStream_t st) {
  const int HW = r->H * r->W, n4 = 4 * HW;
  int bits = 1;
  while ((1LL << bits) < HW) ++bits;
  const int passes = (bits + RS_BITS - 1) / RS_BITS;
  // pass p reads buffer (p + 1) & 1 and writes p & 1; the keys pass writes buffer 1, the ids of pass 0 are implicit
  k_det_keys<<<px_grid(HW, 1), 256, 0, st>>>(a, r->keys[1], flow_out);
  for (int p = 0; p < passes; ++p) {
    const int in = (p + 1) & 1, out = p & 1;
    const int* n_dev = p ? r->count : nullptr;
    k_rs_hist<<<r->rs_blocks, RS_THREADS, 0, st>>>(r->keys[in], n4, n_dev, RS_BITS * p, r->rs_blocks, r->hist);
    k_rs_rowscan<<<RS_DIGITS, RS_THREADS, 0, st>>>(r->hist, r->rs_blocks, r->dtot);
    k_rs_scatter<<<r->rs_blocks, RS_THREADS, 0, st>>>(r->keys[in], p ? r->ids[in] : nullptr, n4, n_dev, RS_BITS * p,
                                                      r->rs_blocks, r->hist, r->dtot, r->keys[out], r->ids[out],
                                                      p ? nullptr : r->count);
  }
  const int last = (passes - 1) & 1;
  G3C_CUDA(cudaMemsetAsync(r->seg, 0, sizeof(uint2) * HW, st));
  k_det_bounds<<<px_grid(n4, 1), 256, 0, st>>>(r->keys[last], r->count, r->seg);
  k_det_accum<<<px_grid(HW, 1), 256, 0, st>>>(a, r->ids[last], r->seg, acc, accz);
  return G3C_OK;
}

// Shared driver: items = n_cam * N flattened with N fastest; groups of `group` consecutive items
// share one max (reference chunking: cache_3d.py:175,183 -> group = 2; forward_warp -> group = b).
static int render_items(g3c_render* r, const float* points, const float* image, const float* mask,
                        const float* w2c, const float* K, ItemMap map, int n_items, int C,
                        int group, int is_image, int want_depth, float* out, float* mask_out,
                        float* depth_out, float* flow_out, cudaStream_t st) {
  const int H = r->H, W = r->W, HW = H * W;
  int n_groups = (n_items + group - 1) / group;
  G3C_REQUIRE(n_groups <= r->gmax_cap, "render: %d groups exceed workspace (%d)", n_groups,
              r->gmax_cap);
  G3C_REQUIRE(C >= 1 && C <= 3, "render: C=%d unsupported (1..3)", C);
  G3C_CUDA(cudaMemsetAsync(r->gmax, 0, sizeof(float) * n_groups, st));
  if (map.src_bcast && map.F <= PM_MAX_CAM && n_items / map.F <= 65535) {
    // every pixel exactly once: 4 pixels per thread, no grid-stride remainder beyond that
    const int bx = (HW + 4 * 256 - 1) / (4 * 256);
    k_project_max_bcast<<<dim3(bx, n_items / map.F), 256, 0, st>>>(points, w2c, K, map.N, map.F, HW, group, r->gmax);
  } else {
    for (int i0 = 0; i0 < n_items; i0 += 65535) {
      int n = n_items - i0 < 65535 ? n_items - i0 : 65535;
      k_project_max<<<px_grid(HW, n), 256, 0, st>>>(points, w2c, K, map, i0, HW, group, r->gmax);
    }
  }
  size_t plane = (size_t)(H + 2) * (W + 2);
  for (int i0 = 0; i0 < n_items; i0 += r->max_items) {
    int n = n_items - i0 < r->max_items ? n_items - i0 : r->max_items;
    if (r->det) {
      for (int j = 0; j < n; ++j) {
        const int item = i0 + j, src = map.src(item), cam = map.cam(item);
        const DetItem a{points + (size_t)src * HW * 3, w2c + 16 * cam, K + 9 * cam, nullptr, nullptr,
                        image + (size_t)src * C * HW, mask ? mask + (size_t)src * HW : nullptr, r->gmax + item / group,
                        C, H, W};
        const int rc = det_splat_item(r, a, r->acc + plane * 4 * j, want_depth ? r->accz + plane * j : nullptr,
                                      flow_out ? flow_out + (size_t)item * 2 * HW : nullptr, st);
        if (rc != G3C_OK) return rc;
      }
    } else {
      G3C_CUDA(cudaMemsetAsync(r->acc, 0, plane * 4 * sizeof(float) * n, st));
      if (want_depth) G3C_CUDA(cudaMemsetAsync(r->accz, 0, plane * sizeof(float) * n, st));
      // 4 pixels per thread with 16-byte loads; frames with W % 4 != 0 or unaligned inputs take one pixel per thread
      const bool aligned = (W % 4 == 0) && ((reinterpret_cast<uintptr_t>(points) | reinterpret_cast<uintptr_t>(image) |
                                             reinterpret_cast<uintptr_t>(mask) | reinterpret_cast<uintptr_t>(flow_out)) % 16 == 0);
      if (aligned)
        k_splat_points4<<<px_grid(HW / 4, n), 256, 0, st>>>(points, image, mask, w2c, K, map, i0, C, H, W, group, r->gmax,
                                                            r->acc, want_depth ? r->accz : nullptr, flow_out);
      else
        k_splat_points<<<px_grid(HW, n), 256, 0, st>>>(points, image, mask, w2c, K, map, i0, C, H, W,
                                                       group, r->gmax, r->acc,
                                                       want_depth ? r->accz : nullptr, flow_out);
    }
    k_normalise<<<px_grid(HW, n), 256, 0, st>>>(r->acc, want_depth ? r->accz : nullptr, i0, C, H,
                                                W, is_image, out, mask_out,
                                                want_depth ? depth_out : nullptr);
  }
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int g3c_forward_warp(g3c_render_t* r, const float* points, const float* image, const float* mask,
                     const float* w2c, const float* K, int b, int C, int flags, float* warped,
                     float* mask_out, float* depth_out, float* flow_out, void* stream) {
  G3C_REQUIRE(r && points && image && w2c && K && warped && mask_out && b > 0,
              "forward_warp: null argument");
  int want_depth = (flags & G3C_WARP_RENDER_DEPTH) != 0;
  G3C_REQUIRE(!want_depth || depth_out, "forward_warp: render_depth set but depth_out is NULL");
  ItemMap map{1, b, 0, 0};
  return render_items(r, points, image, mask, w2c, K, map, b, C, /*group=*/b,
                      (flags & G3C_WARP_NOT_IMAGE) ? 0 : 1, want_depth, warped, mask_out, depth_out,
                      flow_out, (cudaStream_t)stream);
}

int g3c_render_cache(g3c_render_t* r, const float* points, const float* images, const float* masks,
                     const float* w2cs, const float* Ks, int B, int F_target, int N, int src_frames,
                     int render_depth, float* pixels, float* masks_out, float* depth_out,
                     void* stream) {
  G3C_REQUIRE(r && points && images && w2cs && Ks && pixels && masks_out, "render_cache: null argument");
  G3C_REQUIRE(B > 0 && F_target > 0 && N > 0, "render_cache: bad sizes");
  G3C_REQUIRE(src_frames == 1 || src_frames == F_target,
              "render_cache: cache has %d frames, targets %d (must be 1 or equal)", src_frames,
              F_target);
  G3C_REQUIRE(!render_depth || depth_out, "render_cache: render_depth set but depth_out is NULL");
  ItemMap map{N, F_target, src_frames == 1 ? 1 : 0, 0};
  return render_items(r, points, images, masks, w2cs, Ks, map, B * F_target * N, 3,
                      /*group=*/2, 1, render_depth, pixels, masks_out, depth_out, nullptr,
                      (cudaStream_t)stream);
}

int g3c_bilinear_splatting(g3c_render_t* r, const float* frame, const float* mask,
                           const float* depth, const float* flow, int b, int C, int is_image,
                           float* out, float* mask_out, void* stream) {
  G3C_REQUIRE(r && frame && depth && flow && out && mask_out && b > 0,
              "bilinear_splatting: null argument");
  G3C_REQUIRE(C >= 1 && C <= 3, "bilinear_splatting: C=%d unsupported (1..3)", C);
  cudaStream_t st = (cudaStream_t)stream;
  const int H = r->H, W = r->W, HW = H * W;
  G3C_CUDA(cudaMemsetAsync(r->gmax, 0, sizeof(float), st));
  k_depth_max<<<4 * sm_count(), 256, 0, st>>>(depth, (size_t)b * HW, r->gmax);
  size_t plane = (size_t)(H + 2) * (W + 2);
  for (int i0 = 0; i0 < b; i0 += r->max_items) {
    int n = b - i0 < r->max_items ? b - i0 : r->max_items;
    if (r->det) {
      for (int j = 0; j < n; ++j) {
        const size_t item = i0 + j;
        const DetItem a{nullptr, nullptr, nullptr, flow + item * 2 * HW, depth + item * HW, frame + item * C * HW,
                        mask ? mask + item * HW : nullptr, r->gmax, C, H, W};
        const int rc = det_splat_item(r, a, r->acc + plane * 4 * j, nullptr, nullptr, st);
        if (rc != G3C_OK) return rc;
      }
    } else {
      G3C_CUDA(cudaMemsetAsync(r->acc, 0, plane * 4 * sizeof(float) * n, st));
      k_splat_flow<<<px_grid(HW, n), 256, 0, st>>>(frame, mask, depth, flow, i0, C, H, W, r->gmax,
                                                   r->acc);
    }
    k_normalise<<<px_grid(HW, n), 256, 0, st>>>(r->acc, nullptr, i0, C, H, W, is_image, out,
                                                mask_out, nullptr);
  }
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int g3c_splat_indices(const float* flow, int b, int H, int W, int32_t* idx, void* stream) {
  G3C_REQUIRE(flow && idx && b > 0 && H > 0 && W > 0, "splat_indices: bad arguments");
  k_splat_indices<<<px_grid(H * W, b), 256, 0, (cudaStream_t)stream>>>(flow, H, W, idx);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int g3c_unproject_points(const float* depth, const float* w2c, const float* K, const uint8_t* mask,
                         int b, int H, int W, int is_depth, float* points, void* stream) {
  G3C_REQUIRE(depth && w2c && K && points && b > 0 && H > 0 && W > 0, "unproject: bad arguments");
  k_unproject<<<px_grid(H * W, b), 256, 0, (cudaStream_t)stream>>>(depth, w2c, K, mask, H, W,
                                                                   is_depth, points);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int g3c_reliable_depth_mask(const float* depth, int b, int H, int W, int window, float ratio_thresh,
                            float eps, uint8_t* out, void* stream) {
  G3C_REQUIRE(depth && out && b > 0 && H > 0 && W > 0, "reliable_depth_mask: bad arguments");
  G3C_REQUIRE(window % 2 == 1, "Window size must be odd.");
  k_reliable_mask<<<px_grid(H * W, b), 256, 0, (cudaStream_t)stream>>>(depth, H, W, window,
                                                                       ratio_thresh, eps, out);
  G3C_CUDA(cudaGetLastError());
  return G3C_OK;
}

int g3c_align_depth_nonrigid(const float* depth, const float* target_depth, const uint8_t* target_mask, const float* K,
                             const float* c2w, int H, int W, int num_iters, float lambda_arap, float lr, float* out_depth,
                             void* stream) {
  G3C_REQUIRE(depth && target_depth && target_mask && K && c2w && out_depth, "align_depth_nonrigid: null argument");
  G3C_REQUIRE(H > 0 && W > 0 && num_iters >= 0 && lr > 0, "align_depth_nonrigid: bad sizes");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t HW = (size_t)H * W;
  float* buf = nullptr;  // coef | sc0 | sc1 | m1 | m2 | mats(18) | count
  G3C_CUDA(cudaMallocAsync(&buf, (5 * HW + 32) * sizeof(float), st));
  float *coef = buf, *sc0 = buf + HW, *sc1 = buf + 2 * HW, *m1 = buf + 3 * HW, *m2 = buf + 4 * HW, *mats = buf + 5 * HW;
  unsigned int* count = reinterpret_cast<unsigned int*>(mats + 24);
  G3C_CUDA(cudaMemsetAsync(count, 0, sizeof(unsigned int), st));
  k_align_setup<<<1, 32, 0, st>>>(K, c2w, mats);
  k_align_count<<<px_grid((int)HW, 1), 256, 0, st>>>(target_mask, (int)HW, count);
  k_align_init<<<px_grid((int)HW, 1), 256, 0, st>>>(depth, target_mask, mats, count, H, W, coef, sc0, m1, m2);
  const dim3 grid((W + AL_TX - 1) / AL_TX, (H + AL_TY - 1) / AL_TY), block(AL_TX, AL_TY);
  float *cur = sc0, *nxt = sc1;
  for (int it = 1; it <= num_iters; ++it) {
    const float step = (float)((double)lr / (1.0 - pow(0.9, (double)it)));
    const float bc2 = (float)sqrt(1.0 - pow(0.999, (double)it));
    k_align_step<<<grid, block, 0, st>>>(depth, target_depth, coef, cur, nxt, m1, m2, H, W,
                                         lambda_arap / (float)HW, step, bc2);
    float* t = cur;
    cur = nxt;
    nxt = t;
  }
  k_align_finish<<<px_grid((int)HW, 1), 256, 0, st>>>(depth, cur, (int)HW, out_depth);
  G3C_CUDA(cudaGetLastError());
  G3C_CUDA(cudaFreeAsync(buf, st));
  return G3C_OK;
}

static int foreground_items(const float* points, const uint8_t* boundary, const float* w2c, const float* K, ItemMap map,
                            int n_cam, int n_items, int C, int H, int W, float* warped, float* mask, float* depth,
                            cudaStream_t st) {
  const int nh = H / 4, nw = W / 4;  // mesh_downsample_factor = 4 (:289)
  float *verts = nullptr, *kinv = nullptr;
  uint8_t* vmask = nullptr;
  uint32_t* tbuf = nullptr;
  G3C_CUDA(cudaMallocAsync(&kinv, (size_t)n_cam * 9 * sizeof(float), st));
  k_fg_invert_k<<<(n_cam + 63) / 64, 64, 0, st>>>(K, n_cam, kinv);
  // items in passes of <= 64 frames: bounds the scratch (verts, t-buffer) at full resolution
  const int pass = n_items < 64 ? n_items : 64;
  G3C_CUDA(cudaMallocAsync(&verts, (size_t)pass * nh * nw * 3 * sizeof(float), st));
  G3C_CUDA(cudaMallocAsync(&vmask, (size_t)pass * nh * nw, st));
  G3C_CUDA(cudaMallocAsync(&tbuf, (size_t)pass * H * W * sizeof(uint32_t), st));
  for (int i0 = 0; i0 < n_items; i0 += pass) {
    const int n = n_items - i0 < pass ? n_items - i0 : pass;
    ItemMap m = map;
    m.item0 = i0;
    G3C_CUDA(cudaMemsetAsync(tbuf, 0xFF, (size_t)n * H * W * sizeof(uint32_t), st));
    k_fg_mesh_points<<<px_grid(nh * nw, n), 256, 0, st>>>(points, boundary, w2c, m, H, W, nh, nw, verts, vmask);
    k_fg_raster<<<px_grid((nh - 1) * (nw - 1), n), 256, 0, st>>>(verts, vmask, K, kinv, m, H, W, nh, nw, tbuf);
    k_fg_apply<<<px_grid(H * W, n), 256, 0, st>>>(tbuf, kinv, m, C, H, W, warped + (size_t)i0 * C * H * W,
                                                  mask + (size_t)i0 * H * W, depth + (size_t)i0 * H * W);
  }
  G3C_CUDA(cudaGetLastError());
  G3C_CUDA(cudaFreeAsync(verts, st));
  G3C_CUDA(cudaFreeAsync(vmask, st));
  G3C_CUDA(cudaFreeAsync(kinv, st));
  G3C_CUDA(cudaFreeAsync(tbuf, st));
  return G3C_OK;
}

int g3c_foreground_occlusion(const float* points, const uint8_t* boundary, const float* w2c, const float* K, int b, int C,
                             int H, int W, float* warped, float* mask, float* depth, void* stream) {
  G3C_REQUIRE(points && boundary && w2c && K && warped && mask && depth, "foreground_occlusion: null argument");
  G3C_REQUIRE(b > 0 && C >= 1 && C <= 3 && H >= 8 && W >= 8, "foreground_occlusion: bad sizes");
  return foreground_items(points, boundary, w2c, K, ItemMap{1, b, 0, 0}, b, b, C, H, W, warped, mask, depth,
                          (cudaStream_t)stream);
}

int g3c_render_cache_occlusion(const float* points, const uint8_t* boundary, const float* w2cs, const float* Ks, int B,
                               int F_target, int N, int src_frames, float* pixels, float* masks, float* depth,
                               int H, int W, void* stream) {
  G3C_REQUIRE(points && boundary && w2cs && Ks && pixels && masks && depth, "render_cache_occlusion: null argument");
  G3C_REQUIRE(B > 0 && F_target > 0 && N > 0 && (src_frames == 1 || src_frames == F_target) && H >= 8 && W >= 8,
              "render_cache_occlusion: bad sizes");
  return foreground_items(points, boundary, w2cs, Ks, ItemMap{N, F_target, src_frames == 1 ? 1 : 0, 0}, B * F_target,
                          B * F_target * N, 3, H, W, pixels, masks, depth, (cudaStream_t)stream);
}

}  // extern "C"
