// Fused soft-argmax (softmax + 3-D integral) forward / backward and the fused
// joint-location losses.  Reference arithmetic: lib/core/integral_loss.py:7-86.
//
// HBM-bound: the forward reads every logit exactly once (online softmax with
// running max), the backward reads every logit once and writes one gradient.
// No tensor cores: there is no contraction here, only a 5-term reduction.
//
// Partials per CTA are (m, s, sx, sy, sz): running max m and
//   s  = sum e^{v-m},  sx = sum e^{v-m} x,  sy = sum e^{v-m} y,  sz = sum e^{v-m} z
// merged exactly like flash-style online softmax.
#include "common.cuh"
#include <math_constants.h>

namespace {

struct Part {
  float m, s, sx, sy, sz;
};

__device__ __forceinline__ void part_init(Part& p) {
  p.m = -CUDART_INF_F;
  p.s = p.sx = p.sy = p.sz = 0.f;
}

__device__ __forceinline__ void part_merge(Part& a, const Part& b) {
  float m = fmaxf(a.m, b.m);
  if (m == -CUDART_INF_F) return;
  float fa = __expf(a.m - m), fb = __expf(b.m - m);
  a.s = a.s * fa + b.s * fb;
  a.sx = a.sx * fa + b.sx * fb;
  a.sy = a.sy * fa + b.sy * fb;
  a.sz = a.sz * fa + b.sz * fb;
  a.m = m;
}

// accumulate 4 logits that share (y, z) and have x = x0..x0+3  (NCHW layout)
__device__ __forceinline__ void acc4_x(Part& p, const float4 v, float x0, float y, float z) {
  float mx = fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w));
  if (mx > p.m) {
    float f = __expf(p.m - mx);
    p.s *= f; p.sx *= f; p.sy *= f; p.sz *= f;
    p.m = mx;
  }
  float e0 = __expf(v.x - p.m), e1 = __expf(v.y - p.m), e2 = __expf(v.z - p.m), e3 = __expf(v.w - p.m);
  float es = (e0 + e1) + (e2 + e3);
  p.s += es;
  p.sx += x0 * es + (e1 + 2.f * e2 + 3.f * e3);
  p.sy += y * es;
  p.sz += z * es;
}

// accumulate 4 logits that share (x, y) and have z = z0..z0+3  (NHWC layout)
__device__ __forceinline__ void acc4_z(Part& p, const float4 v, float x, float y, float z0) {
  float mx = fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w));
  if (mx > p.m) {
    float f = __expf(p.m - mx);
    p.s *= f; p.sx *= f; p.sy *= f; p.sz *= f;
    p.m = mx;
  }
  float e0 = __expf(v.x - p.m), e1 = __expf(v.y - p.m), e2 = __expf(v.z - p.m), e3 = __expf(v.w - p.m);
  float es = (e0 + e1) + (e2 + e3);
  p.s += es;
  p.sx += x * es;
  p.sy += y * es;
  p.sz += z0 * es + (e1 + 2.f * e2 + 3.f * e3);
}

__device__ __forceinline__ Part warp_merge(Part p) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Part q;
    q.m = __shfl_xor_sync(0xffffffffu, p.m, o);
    q.s = __shfl_xor_sync(0xffffffffu, p.s, o);
    q.sx = __shfl_xor_sync(0xffffffffu, p.sx, o);
    q.sy = __shfl_xor_sync(0xffffffffu, p.sy, o);
    q.sz = __shfl_xor_sync(0xffffffffu, p.sz, o);
    part_merge(p, q);
  }
  return p;
}

// ---------------------------------------------------------------- NCHW fwd
// grid (S, N*J); CTA streams a contiguous chunk of the (n,j) volume.
// Requires W % 4 == 0.  rows = D*H rows of W floats.
constexpr int kFwdThreads = 512;

__global__ void __launch_bounds__(kFwdThreads)
softargmax_fwd_nchw(const float* __restrict__ logits, int D, int H, int W, int S,
                    Part* __restrict__ parts) {
  const int nj = blockIdx.y, sp = blockIdx.x;
  const int W4 = W >> 2;
  const int64_t vol4 = (int64_t)D * H * W4;
  const int64_t per = (vol4 + S - 1) / S;
  const int64_t beg = (int64_t)sp * per;
  const int64_t end = min(vol4, beg + per);
  const float4* base = reinterpret_cast<const float4*>(logits) + (int64_t)nj * vol4;

  Part p;
  part_init(p);
  int64_t f = beg + threadIdx.x;
  // decompose f once, then advance incrementally (no divisions in the loop)
  int64_t row = f / W4;
  int x4 = (int)(f - row * W4);
  int z = (int)(row / H);
  int y = (int)(row - (int64_t)z * H);
  const int step_rows = kFwdThreads / W4, step_x4 = kFwdThreads % W4;
  for (; f < end; f += kFwdThreads) {
    float4 v = ldg_stream(base + f);
    acc4_x(p, v, (float)(x4 << 2), (float)y, (float)z);
    x4 += step_x4;
    y += step_rows;
    if (x4 >= W4) { x4 -= W4; ++y; }
    while (y >= H) { y -= H; ++z; }
  }
  p = warp_merge(p);
  __shared__ Part sh[kFwdThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) sh[wid] = p;
  __syncthreads();
  if (wid == 0) {
    Part q;
    part_init(q);
    if (lane < kFwdThreads / 32) q = sh[lane];
    q = warp_merge(q);
    if (lane == 0) parts[(int64_t)nj * S + sp] = q;
  }
}

// Scalar variant for W % 4 != 0 (any volume shape; the reference accepts every J/D/H/W,
// integral_loss.py:71-86).  Same partition, one logit per thread and iteration.
__global__ void __launch_bounds__(kFwdThreads)
softargmax_fwd_nchw_scalar(const float* __restrict__ logits, int D, int H, int W, int S,
                           Part* __restrict__ parts) {
  const int nj = blockIdx.y, sp = blockIdx.x;
  const int64_t vol = (int64_t)D * H * W;
  const int64_t per = (vol + S - 1) / S;
  const int64_t beg = (int64_t)sp * per;
  const int64_t end = min(vol, beg + per);
  const float* base = logits + (int64_t)nj * vol;
  Part p;
  part_init(p);
  for (int64_t f = beg + threadIdx.x; f < end; f += kFwdThreads) {
    const int64_t row = f / W;
    const int x = (int)(f - row * W);
    const int z = (int)(row / H);
    const int y = (int)(row - (int64_t)z * H);
    const float v = __ldg(base + f);
    if (v > p.m) {
      const float g = __expf(p.m - v);
      p.s *= g; p.sx *= g; p.sy *= g; p.sz *= g;
      p.m = v;
    }
    const float e = __expf(v - p.m);
    p.s += e;
    p.sx += e * (float)x;
    p.sy += e * (float)y;
    p.sz += e * (float)z;
  }
  p = warp_merge(p);
  __shared__ Part sh[kFwdThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) sh[wid] = p;
  __syncthreads();
  if (wid == 0) {
    Part q;
    part_init(q);
    if (lane < kFwdThreads / 32) q = sh[lane];
    q = warp_merge(q);
    if (lane == 0) parts[(int64_t)nj * S + sp] = q;
  }
}

// ---------------------------------------------------------------- NHWC fwd
// grid (S, N); CTA handles a pixel range of one image for ALL joints, reading
// fully contiguous memory.  C = J*D channels, C4 = C/4 threads per pixel,
// ppi pixels per iteration, blockDim = C4*ppi.  Requires D % 4 == 0.
__global__ void softargmax_fwd_nhwc(const float* __restrict__ logits, int J, int D, int H,
                                    int W, int S, int ppi, Part* __restrict__ parts) {
  extern __shared__ Part shp[];  // [blockDim]
  const int n = blockIdx.y, sp = blockIdx.x;
  const int C4 = (J * D) >> 2;
  const int HW = H * W;
  const int per = (HW + S - 1) / S;
  const int pbeg = sp * per, pend = min(HW, pbeg + per);
  const int c4 = threadIdx.x % C4, sub = threadIdx.x / C4;
  const int D4 = D >> 2;
  const float z0 = (float)((c4 % D4) << 2);
  const float4* base = reinterpret_cast<const float4*>(logits) + (int64_t)n * HW * C4 + c4;

  Part p;
  part_init(p);
  int pix = pbeg + sub;
  int y = pix / W, x = pix - y * W;
  for (; pix < pend; pix += ppi) {
    float4 v = ldg_stream(base + (int64_t)pix * C4);
    acc4_z(p, v, (float)x, (float)y, z0);
    x += ppi;
    while (x >= W) { x -= W; ++y; }
  }
  shp[threadIdx.x] = p;
  __syncthreads();
  // one thread per joint merges its D4*ppi partials (tiny, once per CTA)
  if ((int)threadIdx.x < J) {
    const int j = threadIdx.x;
    Part q;
    part_init(q);
    for (int s2 = 0; s2 < ppi; ++s2)
      for (int k = 0; k < D4; ++k) part_merge(q, shp[s2 * C4 + j * D4 + k]);
    parts[((int64_t)n * J + j) * S + sp] = q;
  }
}

// ---------------------------------------------------------------- NHWC fwd, flip test
// Same partition as softargmax_fwd_nhwc over the first N images of a [x; flip(x)] batch of 2N:
// every thread averages its quad of image n with the mirrored pixel of image n+N in the paired
// joint's channels (the flip-back of lib/utils/transforms.py:5-19, optionally shifted one column),
// so the merged volume is never written.  pi: joint involution, J entries.
constexpr int kFlipMaxJ = 1024;          // J*D/4 <= 1024 threads per pixel and D >= 4

struct FlipPerm {
  unsigned short p[kFlipMaxJ];
};

__global__ void softargmax_fwd_nhwc_flip(const float* __restrict__ logits, int N, int J, int D, int H,
                                         int W, int S, int ppi, int shift, const FlipPerm pi,
                                         Part* __restrict__ parts) {
  extern __shared__ Part shp[];  // [blockDim]
  __shared__ unsigned short sperm[kFlipMaxJ];
  for (int j = threadIdx.x; j < J; j += blockDim.x) sperm[j] = pi.p[j];
  __syncthreads();
  const int n = blockIdx.y, sp = blockIdx.x;
  const int C4 = (J * D) >> 2;
  const int HW = H * W;
  const int per = (HW + S - 1) / S;
  const int pbeg = sp * per, pend = min(HW, pbeg + per);
  const int c4 = threadIdx.x % C4, sub = threadIdx.x / C4;
  const int D4 = D >> 2;
  const int k4 = c4 % D4;
  const int c4f = (int)sperm[c4 / D4] * D4 + k4;      // quad of the paired joint, same depth bins
  const float z0 = (float)(k4 << 2);
  const float4* base = reinterpret_cast<const float4*>(logits) + (int64_t)n * HW * C4 + c4;
  const float4* fbase = reinterpret_cast<const float4*>(logits) + (int64_t)(n + N) * HW * C4 + c4f;

  Part p;
  part_init(p);
  int pix = pbeg + sub;
  int y = pix / W, x = pix - y * W;
  for (; pix < pend; pix += ppi) {
    // w' = W-1-w; with the shift column w reads the flip-back's column w-1 (column 0 keeps its own)
    const int xf = shift ? (x == 0 ? W - 1 : W - x) : W - 1 - x;
    const float4 a = ldg_stream(base + (int64_t)pix * C4);
    const float4 b = ldg_stream(fbase + (int64_t)(y * W + xf) * C4);
    const float4 v = make_float4(0.5f * (a.x + b.x), 0.5f * (a.y + b.y), 0.5f * (a.z + b.z),
                                 0.5f * (a.w + b.w));
    acc4_z(p, v, (float)x, (float)y, z0);
    x += ppi;
    while (x >= W) { x -= W; ++y; }
  }
  shp[threadIdx.x] = p;
  __syncthreads();
  if ((int)threadIdx.x < J) {
    const int j = threadIdx.x;
    Part q;
    part_init(q);
    for (int s2 = 0; s2 < ppi; ++s2)
      for (int k = 0; k < D4; ++k) part_merge(q, shp[s2 * C4 + j * D4 + k]);
    parts[((int64_t)n * J + j) * S + sp] = q;
  }
}

// ---------------------------------------------------------------- finalize
// lse may be null (the flip-test forward has no backward)
__global__ void softargmax_finalize(const Part* __restrict__ parts, int NJ, int S, float invW,
                                    float invH, float invD, float* __restrict__ coords,
                                    float* __restrict__ lse) {
  const int nj = blockIdx.x * blockDim.x + threadIdx.x;
  if (nj >= NJ) return;
  Part q;
  part_init(q);
  for (int s = 0; s < S; ++s) part_merge(q, parts[(int64_t)nj * S + s]);
  const float inv = 1.f / q.s;
  // integral_loss.py:81-83: coord/dim - 0.5
  coords[nj * 3 + 0] = q.sx * inv * invW - 0.5f;
  coords[nj * 3 + 1] = q.sy * inv * invH - 0.5f;
  coords[nj * 3 + 2] = q.sz * inv * invD - 0.5f;
  if (lse) {
    lse[nj * 2 + 0] = q.m;
    lse[nj * 2 + 1] = inv;
  }
}

// ---------------------------------------------------------------- backward
// dlogit = p * (s - sbar),  s = gx*x/W + gy*y/H + gz*z/D,
// sbar = sum p s = gx*(cx+.5) + gy*(cy+.5) + gz*(cz+.5)  (from the forward outputs)
__global__ void __launch_bounds__(kFwdThreads)
softargmax_bwd_nchw(const float* __restrict__ logits, int D, int H, int W, int S,
                    const float* __restrict__ coords, const float* __restrict__ lse,
                    const float* __restrict__ dcoords, float* __restrict__ dlogits) {
  const int nj = blockIdx.y, sp = blockIdx.x;
  const int W4 = W >> 2;
  const int64_t vol4 = (int64_t)D * H * W4;
  const int64_t per = (vol4 + S - 1) / S;
  const int64_t beg = (int64_t)sp * per;
  const int64_t end = min(vol4, beg + per);
  const float4* base = reinterpret_cast<const float4*>(logits) + (int64_t)nj * vol4;
  float4* obase = reinterpret_cast<float4*>(dlogits) + (int64_t)nj * vol4;
  const float m = lse[nj * 2], inv = lse[nj * 2 + 1];
  const float gx = dcoords[nj * 3] / W, gy = dcoords[nj * 3 + 1] / H, gz = dcoords[nj * 3 + 2] / D;
  const float sbar = gx * (coords[nj * 3] + 0.5f) * W + gy * (coords[nj * 3 + 1] + 0.5f) * H +
                     gz * (coords[nj * 3 + 2] + 0.5f) * D;
  int64_t f = beg + threadIdx.x;
  int64_t row = f / W4;
  int x4 = (int)(f - row * W4);
  int z = (int)(row / H);
  int y = (int)(row - (int64_t)z * H);
  const int step_rows = kFwdThreads / W4, step_x4 = kFwdThreads % W4;
  for (; f < end; f += kFwdThreads) {
    float4 v = ldg_stream(base + f);
    const float s0 = gy * y + gz * z + gx * (float)(x4 << 2) - sbar;
    float4 o;
    o.x = __expf(v.x - m) * inv * (s0);
    o.y = __expf(v.y - m) * inv * (s0 + gx);
    o.z = __expf(v.z - m) * inv * (s0 + 2.f * gx);
    o.w = __expf(v.w - m) * inv * (s0 + 3.f * gx);
    obase[f] = o;
    x4 += step_x4;
    y += step_rows;
    if (x4 >= W4) { x4 -= W4; ++y; }
    while (y >= H) { y -= H; ++z; }
  }
}

__global__ void __launch_bounds__(kFwdThreads)
softargmax_bwd_nchw_scalar(const float* __restrict__ logits, int D, int H, int W, int S,
                           const float* __restrict__ coords, const float* __restrict__ lse,
                           const float* __restrict__ dcoords, float* __restrict__ dlogits) {
  const int nj = blockIdx.y, sp = blockIdx.x;
  const int64_t vol = (int64_t)D * H * W;
  const int64_t per = (vol + S - 1) / S;
  const int64_t beg = (int64_t)sp * per;
  const int64_t end = min(vol, beg + per);
  const float* base = logits + (int64_t)nj * vol;
  float* obase = dlogits + (int64_t)nj * vol;
  const float m = lse[nj * 2], inv = lse[nj * 2 + 1];
  const float gx = dcoords[nj * 3] / W, gy = dcoords[nj * 3 + 1] / H, gz = dcoords[nj * 3 + 2] / D;
  const float sbar = gx * (coords[nj * 3] + 0.5f) * W + gy * (coords[nj * 3 + 1] + 0.5f) * H +
                     gz * (coords[nj * 3 + 2] + 0.5f) * D;
  for (int64_t f = beg + threadIdx.x; f < end; f += kFwdThreads) {
    const int64_t row = f / W;
    const int x = (int)(f - row * W);
    const int z = (int)(row / H);
    const int y = (int)(row - (int64_t)z * H);
    obase[f] = __expf(__ldg(base + f) - m) * inv * (gy * y + gz * z + gx * (float)x - sbar);
  }
}

__global__ void softargmax_bwd_nhwc(const float* __restrict__ logits, int J, int D, int H, int W,
                                    int S, int ppi, const float* __restrict__ coords,
                                    const float* __restrict__ lse,
                                    const float* __restrict__ dcoords,
                                    float* __restrict__ dlogits) {
  const int n = blockIdx.y, sp = blockIdx.x;
  const int C4 = (J * D) >> 2;
  const int HW = H * W;
  const int per = (HW + S - 1) / S;
  const int pbeg = sp * per, pend = min(HW, pbeg + per);
  const int c4 = threadIdx.x % C4, sub = threadIdx.x / C4;
  const int D4 = D >> 2;
  const int j = c4 / D4;
  const float z0 = (float)((c4 % D4) << 2);
  const int nj = n * J + j;
  const float m = lse[nj * 2], inv = lse[nj * 2 + 1];
  const float gx = dcoords[nj * 3] / W, gy = dcoords[nj * 3 + 1] / H, gz = dcoords[nj * 3 + 2] / D;
  const float sbar = gx * (coords[nj * 3] + 0.5f) * W + gy * (coords[nj * 3 + 1] + 0.5f) * H +
                     gz * (coords[nj * 3 + 2] + 0.5f) * D;
  const float4* base = reinterpret_cast<const float4*>(logits) + (int64_t)n * HW * C4 + c4;
  float4* obase = reinterpret_cast<float4*>(dlogits) + (int64_t)n * HW * C4 + c4;
  int pix = pbeg + sub;
  int y = pix / W, x = pix - y * W;
  for (; pix < pend; pix += ppi) {
    float4 v = ldg_stream(base + (int64_t)pix * C4);
    const float s0 = gx * x + gy * y + gz * z0 - sbar;
    float4 o;
    o.x = __expf(v.x - m) * inv * (s0);
    o.y = __expf(v.y - m) * inv * (s0 + gz);
    o.z = __expf(v.z - m) * inv * (s0 + 2.f * gz);
    o.w = __expf(v.w - m) * inv * (s0 + 3.f * gz);
    obase[(int64_t)pix * C4] = o;
    x += ppi;
    while (x >= W) { x -= W; ++y; }
  }
}

// ---------------------------------------------------------------- losses
// integral_loss.py:7-47.  Single CTA: n = N*J*3 is a few thousand at most.
constexpr int kLossThreads = 1024;

__device__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) sh[wid] = v;
  __syncthreads();
  float r = (threadIdx.x < kLossThreads / 32) ? sh[threadIdx.x] : 0.f;
  if (wid == 0) r = warp_sum(r);
  if (threadIdx.x == 0) sh[32] = r;
  __syncthreads();
  return sh[32];
}

__global__ void __launch_bounds__(kLossThreads)
jointloss_kernel(const float* __restrict__ x, const float* __restrict__ t,
                 const float* __restrict__ w, int n, int kind, int norm, float div,
                 float* __restrict__ loss, float* __restrict__ dx) {
  __shared__ float sh[33];
  float sx = 1.f, st = 1.f;
  if (norm) {  // integral_loss.py:9-11  torch.norm(.,1) over the whole tensor
    float ax = 0.f, at = 0.f;
    for (int i = threadIdx.x; i < n; i += kLossThreads) { ax += fabsf(x[i]); at += fabsf(t[i]); }
    sx = block_sum(ax, sh);
    st = block_sum(at, sh);
  }
  const float isx = 1.f / sx, ist = 1.f / st, idiv = 1.f / div;
  float acc = 0.f, gdot = 0.f;
  for (int i = threadIdx.x; i < n; i += kLossThreads) {
    const float xi = x[i];
    const float d = xi * isx - t[i] * ist;
    const float a = fabsf(d);
    float l, g;
    if (kind == 0) { l = d * d; g = 2.f * d; }
    else if (kind == 1) { l = a; g = (d > 0.f) - (d < 0.f); }
    else { l = a < 1.f ? 0.5f * d * d : a - 0.5f; g = a < 1.f ? d : (float)((d > 0.f) - (d < 0.f)); }
    const float wi = w[i];
    acc += l * wi;
    g *= wi * idiv;
    if (norm) gdot += g * xi;
    if (dx) dx[i] = g * isx;  // completed below when norm
  }
  const float total = block_sum(acc, sh);
  if (threadIdx.x == 0 && loss) *loss = total * idiv;
  if (norm && dx) {
    const float gd = block_sum(gdot, sh);
    const float c = gd * isx * isx;
    for (int i = threadIdx.x; i < n; i += kLossThreads) {
      const float xi = x[i];
      dx[i] -= (float)((xi > 0.f) - (xi < 0.f)) * c;
    }
  }
}

// ---------------------------------------------------------------- heat-map MSE + joint loss
// One launch for the VOLUME=False training objective: mean squared error of the 2-D heat-maps
// against their (Gaussian) targets, fused with the weighted L1 / SmoothL1 / MSE joint-location
// loss of the 3-D branch.  HBM-bound: reads hm and target once, writes dhm once (12 B per
// heat-map element); per-CTA partial sums are combined by the LAST CTA to finish (ticket
// counter) in a fixed order, so the loss is deterministic; that CTA also evaluates the tiny
// joint part (n <= a few thousand elements) and writes the three loss values.
constexpr int kHmThreads = 256;
constexpr int kHmMaxBlocks = 8 * kNumSMs;

__global__ void __launch_bounds__(kHmThreads)
heatmap_joint_loss_kernel(const float* __restrict__ hm, const float* __restrict__ target,
                          const float* __restrict__ wh, int R, int HW, float hm_scale,
                          const float* __restrict__ x, const float* __restrict__ t,
                          const float* __restrict__ w, int n, int kind, float div, float jt_scale,
                          float* __restrict__ loss, float* __restrict__ dhm,
                          float* __restrict__ dx, double* __restrict__ parts,
                          unsigned* __restrict__ ticket) {
  __shared__ double shd[kHmThreads / 32];
  __shared__ bool last;
  const int64_t total = (int64_t)R * HW;
  const float inv = 1.f / (float)total;
  const float gs = 2.f * hm_scale * inv;
  double acc = 0.0;
  if ((HW & 3) == 0) {
    const int64_t total4 = total >> 2;
    const int hw4 = HW >> 2;
    const int64_t stride = (int64_t)gridDim.x * kHmThreads;
    float facc = 0.f;
    const bool small = total4 < (1LL << 31);       // 32-bit row index: the 64-bit division costs ~100 instructions
    auto one = [&](int64_t i, const float4 h, const float4 g) {
      const float wr = wh ? wh[small ? (int64_t)((uint32_t)i / (uint32_t)hw4) : i / hw4] : 1.f;
      const float4 d = make_float4(wr * (h.x - g.x), wr * (h.y - g.y), wr * (h.z - g.z),
                                   wr * (h.w - g.w));
      facc += (d.x * d.x + d.y * d.y) + (d.z * d.z + d.w * d.w);      // <= a few hundred terms per thread in fp32
      if (dhm) {
        const float c = gs * wr;
        __stcs(reinterpret_cast<float4*>(dhm) + i, make_float4(c * d.x, c * d.y, c * d.z, c * d.w));
      }
    };
    int64_t i = (int64_t)blockIdx.x * kHmThreads + threadIdx.x;
    for (; i + 3 * stride < total4; i += 4 * stride) {        // four element quads per trip: 8 loads in flight
      float4 h[4], g[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        h[u] = ldg_stream(reinterpret_cast<const float4*>(hm) + i + u * stride);
        g[u] = ldg_stream(reinterpret_cast<const float4*>(target) + i + u * stride);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) one(i + u * stride, h[u], g[u]);
    }
    for (; i < total4; i += stride)
      one(i, ldg_stream(reinterpret_cast<const float4*>(hm) + i),
          ldg_stream(reinterpret_cast<const float4*>(target) + i));
    acc = (double)facc;
  } else {
    for (int64_t i = (int64_t)blockIdx.x * kHmThreads + threadIdx.x; i < total;
         i += (int64_t)gridDim.x * kHmThreads) {
      const float wr = wh ? wh[i / HW] : 1.f;
      const float d = wr * (hm[i] - target[i]);
      acc += (double)(d * d);
      if (dhm) dhm[i] = gs * wr * d;
    }
  }
  acc = warp_sum(acc);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) shd[wid] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double b = 0.0;
    for (int k = 0; k < kHmThreads / 32; ++k) b += shd[k];
    parts[blockIdx.x] = b;
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();                            // partials of every CTA are visible
  // joint-location part (integral_loss.py:7-47 without `norm`)
  const float idiv = n > 0 ? 1.f / div : 0.f;
  double jacc = 0.0;
  for (int i = threadIdx.x; i < n; i += kHmThreads) {
    const float d = x[i] - t[i];
    const float a = fabsf(d);
    float l, g;
    if (kind == 0) { l = d * d; g = 2.f * d; }
    else if (kind == 1) { l = a; g = (float)((d > 0.f) - (d < 0.f)); }
    else { l = a < 1.f ? 0.5f * d * d : a - 0.5f; g = a < 1.f ? d : (float)((d > 0.f) - (d < 0.f)); }
    jacc += (double)(l * w[i]);
    if (dx) dx[i] = g * w[i] * idiv * jt_scale;
  }
  jacc = warp_sum(jacc);
  __syncthreads();
  if (lane == 0) shd[wid] = jacc;
  __syncthreads();
  // heat-map partials of all CTAs: lane l of warp 0 adds parts[l], parts[l+32], ... then a shuffle tree
  // (a fixed order: run-to-run identical)
  double lhp = 0.0;
  if (wid == 0) {
    for (unsigned k = lane; k < gridDim.x; k += 32) lhp += parts[k];
    lhp = warp_sum(lhp);
  }
  if (threadIdx.x == 0) {
    double lj = 0.0;
    const double lh = lhp;
    for (int k = 0; k < kHmThreads / 32; ++k) lj += shd[k];
    const float loss_hm = (float)(lh / (double)total);
    const float loss_jt = (float)(lj * (double)idiv);
    loss[0] = loss_hm;
    loss[1] = loss_jt;
    loss[2] = hm_scale * loss_hm + jt_scale * loss_jt;
    *ticket = 0u;                             // ready for the next launch (stream ordered)
  }
}

int pick_splits(int rows, int64_t work_per_row, int max_splits) {
  // aim for >= 4 CTAs per SM without making chunks smaller than ~16 KB
  int s = 1;
  while (rows * s < 4 * kNumSMs && s * 2 <= max_splits && work_per_row / (s * 2) >= 4096) s *= 2;
  return s;
}

}  // namespace

extern "C" __attribute__((visibility("default"))) int epb_softargmax_fwd(const float* logits, int layout, int N, int J, int D, int H,
                                  int W, float* coords, float* lse_ws, epb_stream_t stream) {
  EPB_CHECK_ARG(logits && coords && lse_ws);
  EPB_CHECK_ARG(N > 0 && J > 0 && D > 0 && H > 0 && W > 0);
  cudaStream_t st = as_stream(stream);
  const int NJ = N * J;
  int S;
  Part* parts = nullptr;        // per-CTA partials: scratch of this (device, stream)
  if (layout == 0) {
    const int64_t vol = (int64_t)D * H * W;
    S = pick_splits(NJ, vol, 64);
    int rc = epb_workspace(EPB_WS_SOFTARGMAX, (size_t)NJ * S * sizeof(Part), st, (void**)&parts);
    if (rc) return rc;
    if (W % 4 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0)
      softargmax_fwd_nchw<<<dim3(S, NJ), kFwdThreads, 0, st>>>(logits, D, H, W, S, parts);
    else
      softargmax_fwd_nchw_scalar<<<dim3(S, NJ), kFwdThreads, 0, st>>>(logits, D, H, W, S, parts);
  } else if (layout == 1) {
    EPB_CHECK_ARG(D % 4 == 0);
    const int C4 = J * D / 4;
    EPB_CHECK_ARG(C4 <= 1024);
    const int ppi = (512 / C4) > 0 ? (512 / C4) : 1;
    S = 1;
    while (N * S < 8 * kNumSMs && (H * W) / (S * 2) >= 16 * ppi) S *= 2;
    int rc = epb_workspace(EPB_WS_SOFTARGMAX, (size_t)NJ * S * sizeof(Part), st, (void**)&parts);
    if (rc) return rc;
    const int threads = C4 * ppi;
    softargmax_fwd_nhwc<<<dim3(S, N), threads, threads * sizeof(Part), st>>>(
        logits, J, D, H, W, S, ppi, parts);
  } else {
    EPB_CHECK_ARG(layout == 0 || layout == 1);
    return EPB_EINVAL;
  }
  EPB_LAUNCH_CHECK();
  softargmax_finalize<<<(NJ + 127) / 128, 128, 0, st>>>(parts, NJ, S, 1.f / W, 1.f / H, 1.f / D,
                                                      coords, lse_ws);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

// shared by the two flip-test entries; lse_ws may be null
static int softargmax_flip_run(const float* logits2N, int N, int J, int D, int H, int W,
                               const int* perm_host, int shift, float* coords, float* lse_ws,
                               epb_stream_t stream) {
  EPB_CHECK_ARG(logits2N && perm_host && coords);
  EPB_CHECK_ARG(N > 0 && J > 0 && D > 0 && H > 0 && W > 0);
  EPB_CHECK_ARG(shift == 0 || shift == 1);
  EPB_CHECK_ARG(D % 4 == 0);
  EPB_CHECK_ARG((int64_t)J * D / 4 <= 1024);
  EPB_CHECK_ARG((reinterpret_cast<uintptr_t>(logits2N) & 15) == 0);
  FlipPerm pi;
  for (int j = 0; j < J; ++j) {
    const int q = perm_host[j];
    if (q < 0 || q >= J) {
      epb_set_error("epb_softargmax_flip_fwd: perm[%d] = %d is outside [0, %d)", j, q, J);
      return EPB_EINVAL;
    }
    if (perm_host[q] != j) {
      epb_set_error("epb_softargmax_flip_fwd: perm is not an involution (perm[%d] = %d, perm[%d] = %d)",
                    j, q, q, perm_host[q]);
      return EPB_EINVAL;
    }
    pi.p[j] = (unsigned short)q;
  }
  cudaStream_t st = as_stream(stream);
  const int NJ = N * J;
  const int C4 = J * D / 4;
  const int ppi = (512 / C4) > 0 ? (512 / C4) : 1;
  int S = 1;
  while (N * S < 8 * kNumSMs && (H * W) / (S * 2) >= 16 * ppi) S *= 2;
  Part* parts = nullptr;
  int rc = epb_workspace(EPB_WS_SOFTARGMAX, (size_t)NJ * S * sizeof(Part), st, (void**)&parts);
  if (rc) return rc;
  const int threads = C4 * ppi;
  softargmax_fwd_nhwc_flip<<<dim3(S, N), threads, threads * sizeof(Part), st>>>(
      logits2N, N, J, D, H, W, S, ppi, shift, pi, parts);
  EPB_LAUNCH_CHECK();
  softargmax_finalize<<<(NJ + 127) / 128, 128, 0, st>>>(parts, NJ, S, 1.f / W, 1.f / H, 1.f / D,
                                                      coords, lse_ws);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_softargmax_flip_fwd(
    const float* logits2N, int N, int J, int D, int H, int W, const int* perm_host, int shift,
    float* coords, epb_stream_t stream) {
  return softargmax_flip_run(logits2N, N, J, D, H, W, perm_host, shift, coords, nullptr, stream);
}

extern "C" __attribute__((visibility("default"))) int epb_softargmax_flip_lse_fwd(
    const float* logits2N, int N, int J, int D, int H, int W, const int* perm_host, int shift,
    float* coords, float* lse_ws, epb_stream_t stream) {
  EPB_CHECK_ARG(lse_ws);
  return softargmax_flip_run(logits2N, N, J, D, H, W, perm_host, shift, coords, lse_ws, stream);
}

extern "C" __attribute__((visibility("default"))) int epb_softargmax_bwd(const float* logits, int layout, int N, int J, int D, int H,
                                  int W, const float* coords, const float* lse_ws,
                                  const float* dcoords, float* dlogits, epb_stream_t stream) {
  EPB_CHECK_ARG(logits && coords && lse_ws && dcoords && dlogits);
  EPB_CHECK_ARG(N > 0 && J > 0 && D > 0 && H > 0 && W > 0);
  cudaStream_t st = as_stream(stream);
  const int NJ = N * J;
  if (layout == 0) {
    const int S = pick_splits(NJ, (int64_t)D * H * W, 64);
    if (W % 4 == 0 && ((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(dlogits)) & 15) == 0)
      softargmax_bwd_nchw<<<dim3(S, NJ), kFwdThreads, 0, st>>>(logits, D, H, W, S, coords, lse_ws,
                                                                dcoords, dlogits);
    else
      softargmax_bwd_nchw_scalar<<<dim3(S, NJ), kFwdThreads, 0, st>>>(logits, D, H, W, S, coords,
                                                                       lse_ws, dcoords, dlogits);
  } else if (layout == 1) {
    EPB_CHECK_ARG(D % 4 == 0);
    const int C4 = J * D / 4;
    EPB_CHECK_ARG(C4 <= 1024);
    const int ppi = (512 / C4) > 0 ? (512 / C4) : 1;
    int S = 1;
    while (N * S < 8 * kNumSMs && (H * W) / (S * 2) >= 16 * ppi) S *= 2;
    softargmax_bwd_nhwc<<<dim3(S, N), C4 * ppi, 0, st>>>(logits, J, D, H, W, S, ppi, coords,
                                                         lse_ws, dcoords, dlogits);
  } else {
    EPB_CHECK_ARG(layout == 0 || layout == 1);
    return EPB_EINVAL;
  }
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_jointloss_fwd_bwd(const float* x, const float* t, const float* w, int n,
                                     int kind, int norm, float div, float* loss, float* dx,
                                     epb_stream_t stream) {
  EPB_CHECK_ARG(x && t && w && n > 0);
  EPB_CHECK_ARG(kind >= 0 && kind <= 2);
  EPB_CHECK_ARG(div != 0.f);
  jointloss_kernel<<<1, kLossThreads, 0, as_stream(stream)>>>(x, t, w, n, kind, norm, div, loss, dx);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_heatmap_joint_loss(
    const float* hm, const float* target, const float* hm_weight, int R, int HW, float hm_scale,
    const float* x, const float* t, const float* w, int n, int kind, float div, float jt_scale,
    float* loss, float* dhm, float* dx, epb_stream_t stream) {
  EPB_CHECK_ARG(hm && target && loss);
  EPB_CHECK_ARG(R > 0 && HW > 0);
  EPB_CHECK_ARG(n >= 0 && (n == 0 || (x && t && w)));
  EPB_CHECK_ARG(kind >= 0 && kind <= 2);
  EPB_CHECK_ARG(n == 0 || div != 0.f);
  double* hm_parts = nullptr;   // [kHmMaxBlocks] partials + ticket counter (zero-filled when created)
  int rc = epb_workspace(EPB_WS_HMLOSS, (kHmMaxBlocks + 1) * sizeof(double), as_stream(stream),
                         (void**)&hm_parts);
  if (rc) return rc;
  const int64_t work = ((int64_t)R * HW + 3) / 4;
  int64_t blocks = (work + kHmThreads - 1) / kHmThreads;
  if (blocks > kHmMaxBlocks) blocks = kHmMaxBlocks;
  heatmap_joint_loss_kernel<<<(int)blocks, kHmThreads, 0, as_stream(stream)>>>(
      hm, target, hm_weight, R, HW, hm_scale, x, t, w, n, kind, div, jt_scale, loss, dhm, dx,
      hm_parts, reinterpret_cast<unsigned*>(hm_parts + kHmMaxBlocks));
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}
