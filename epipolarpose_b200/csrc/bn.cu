// BatchNorm2d (training semantics, momentum 0.1) statistics / finalize / apply,
// fused residual-add + ReLU, fused stem BN+ReLU+MaxPool, and their backward
// passes.  Reference call sites: lib/models/pose3d_resnet.py:24,31-47,56-88,
// 101-103,134,179,187-189 (nn.BatchNorm2d / ReLU / MaxPool2d / `out += residual`).
//
// All kernels are HBM-bound elementwise / per-channel reductions over NHWC
// float32 rows x[M][C]: threads map to channel quads (float4) so every warp
// reads full 128-byte lines; per-channel sums are accumulated per thread in
// fp32 over a bounded row span, then combined in float64 (atomicAdd double).
// var = E[x^2]-E[x]^2 inherits the sums' relative error times 1 + (mean/std)^2:
// ~1e-7 relative for centred channels, growing as (mean/std)^2 (~1e-5 at 10,
// ~1e-3 at 100; tests/test_gpu_bn_chain.py measures the conv16 epilogue's sums).
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kRowsPerThread = 64;   // fp32 accumulation span per thread

struct RowMap {
  int C4;      // float4 per row
  int tpr;     // threads per row (<= kThreads)
  int rpi;     // rows per iteration per CTA
  int chunks;  // channel chunks (gridDim.y)
};

inline RowMap make_rowmap(int C) {
  RowMap r;
  r.C4 = C / 4;
  r.tpr = r.C4 < kThreads ? r.C4 : kThreads;
  // largest power of two <= tpr so that rows align to whole warps when possible
  r.rpi = kThreads / r.tpr;
  if (r.rpi < 1) r.rpi = 1;
  r.chunks = (r.C4 + r.tpr - 1) / r.tpr;
  return r;
}

// reduce `NV` float4 accumulators across the rpi row-slots of a CTA and add to
// double outputs: out[v*C + c]
template <int NV>
__device__ void cta_reduce_to_global(float4 (&acc)[NV], int c4, bool active, int tpr, int rpi,
                                     int C, double* out) {
  __shared__ float4 sh[NV][kThreads];
  const int slot = threadIdx.x / tpr, tin = threadIdx.x % tpr;
#pragma unroll
  for (int v = 0; v < NV; ++v) sh[v][threadIdx.x] = acc[v];
  __syncthreads();
  if (slot == 0 && active && threadIdx.x < tpr * rpi) {
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      double a0 = 0, a1 = 0, a2 = 0, a3 = 0;
      for (int s = 0; s < rpi; ++s) {
        const float4 t = sh[v][s * tpr + tin];
        a0 += t.x; a1 += t.y; a2 += t.z; a3 += t.w;
      }
      double* o = out + (int64_t)v * C + c4 * 4;
      atomicAdd(o + 0, a0); atomicAdd(o + 1, a1); atomicAdd(o + 2, a2); atomicAdd(o + 3, a3);
    }
  }
}

__global__ void __launch_bounds__(kThreads)
channel_stats_kernel(const float4* __restrict__ x, int64_t M, int C, RowMap rm,
                     double* __restrict__ stats) {
  const int slot = threadIdx.x / rm.tpr, tin = threadIdx.x % rm.tpr;
  const int c4 = blockIdx.y * rm.tpr + tin;
  const bool active = (c4 < rm.C4) && (slot < rm.rpi);
  const int64_t rows_per_cta = (int64_t)rm.rpi * kRowsPerThread;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta;
  float4 acc[2] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
  if (active) {
    for (int k = 0; k < kRowsPerThread; ++k) {
      const int64_t r = r0 + (int64_t)k * rm.rpi + slot;
      if (r >= M) break;
      const float4 v = ldg_stream(x + r * rm.C4 + c4);
      acc[0].x += v.x; acc[0].y += v.y; acc[0].z += v.z; acc[0].w += v.w;
      acc[1].x += v.x * v.x; acc[1].y += v.y * v.y; acc[1].z += v.z * v.z; acc[1].w += v.w * v.w;
    }
  }
  cta_reduce_to_global<2>(acc, c4, active, rm.tpr, rm.rpi, C, stats);
}

__global__ void bn_finalize_kernel(const double* __restrict__ stats, double M, int C,
                                   const float* __restrict__ gamma, const float* __restrict__ beta,
                                   float eps, float momentum, float* __restrict__ running_mean,
                                   float* __restrict__ running_var, float* __restrict__ scale,
                                   float* __restrict__ shift, float* __restrict__ mean_out,
                                   float* __restrict__ invstd_out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double mean = stats[c] / M;
  double var = stats[C + c] / M - mean * mean;   // biased (normalisation)
  if (var < 0) var = 0;
  const double invstd = 1.0 / sqrt(var + (double)eps);
  const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
  scale[c] = (float)(g * invstd);
  shift[c] = (float)(b - mean * g * invstd);
  if (mean_out) mean_out[c] = (float)mean;
  if (invstd_out) invstd_out[c] = (float)invstd;
  if (running_mean) {
    const double unbiased = var * (M / (M > 1.0 ? (M - 1.0) : 1.0));
    running_mean[c] = (float)((1.0 - momentum) * running_mean[c] + momentum * mean);
    running_var[c] = (float)((1.0 - momentum) * running_var[c] + momentum * unbiased);
  }
}

__global__ void bn_eval_affine_kernel(int C, const float* __restrict__ gamma,
                                      const float* __restrict__ beta,
                                      const float* __restrict__ rm, const float* __restrict__ rv,
                                      float eps, float* __restrict__ scale,
                                      float* __restrict__ shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  // in double, rounded once: shift = beta - mean * scale cancels when the two are close, and fp32
  // arithmetic there left shift many of its own ulps off
  const double s = (gamma ? (double)gamma[c] : 1.0) / sqrt((double)rv[c] + (double)eps);
  scale[c] = (float)s;
  shift[c] = (float)((beta ? (double)beta[c] : 0.0) - (double)rm[c] * s);
}

__device__ __forceinline__ float4 fma4(float4 x, float4 s, float4 b) {
  return make_float4(fmaf(x.x, s.x, b.x), fmaf(x.y, s.y, b.y), fmaf(x.z, s.z, b.z),
                     fmaf(x.w, s.w, b.w));
}
__device__ __forceinline__ float4 relu4(float4 v) {
  return make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
}

__global__ void __launch_bounds__(kThreads)
bn_act_kernel(const float4* __restrict__ x, const float4* __restrict__ scale,
              const float4* __restrict__ shift, const float4* __restrict__ r,
              const float4* __restrict__ rscale, const float4* __restrict__ rshift, int relu,
              float4* __restrict__ y, int64_t total4, int C4) {
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < total4;
       i += (int64_t)gridDim.x * kThreads) {
    const int c4 = (int)(i % C4);
    float4 v = ldg_stream(x + i);
    if (scale) v = fma4(v, scale[c4], shift[c4]);
    if (r) {
      float4 q = ldg_stream(r + i);
      if (rscale) q = fma4(q, rscale[c4], rshift[c4]);
      v.x += q.x; v.y += q.y; v.z += q.z; v.w += q.w;
    }
    if (relu) v = relu4(v);
    y[i] = v;
  }
}

// stem: y = maxpool3x3 s2 p1 ( relu(x*scale+shift) ), argidx = window slot 0..8
__global__ void __launch_bounds__(kThreads)
bn_relu_maxpool_kernel(const float4* __restrict__ x, const float4* __restrict__ scale,
                       const float4* __restrict__ shift, float4* __restrict__ y,
                       uchar4* __restrict__ argidx, int N, int H, int W, int C4) {
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const int64_t total = (int64_t)N * Ho * Wo * C4;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * kThreads) {
    const int c4 = (int)(i % C4);
    int64_t p = i / C4;
    const int ow = (int)(p % Wo); p /= Wo;
    const int oh = (int)(p % Ho);
    const int n = (int)(p / Ho);
    const float4 s = scale[c4], b = shift[c4];
    float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    uchar4 bi = make_uchar4(0, 0, 0, 0);
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int ih = oh * 2 - 1 + kh;
      if (ih < 0 || ih >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int iw = ow * 2 - 1 + kw;
        if (iw < 0 || iw >= W) continue;
        const float4 v = relu4(fma4(x[((int64_t)(n * H + ih) * W + iw) * C4 + c4], s, b));
        const unsigned char k = (unsigned char)(kh * 3 + kw);
        if (v.x > best.x) { best.x = v.x; bi.x = k; }
        if (v.y > best.y) { best.y = v.y; bi.y = k; }
        if (v.z > best.z) { best.z = v.z; bi.z = k; }
        if (v.w > best.w) { best.w = v.w; bi.w = k; }
      }
    }
    y[i] = best;
    if (argidx) argidx[i] = bi;
  }
}

// dx[n,h,w,c] = sum of dy over the (<= 4) pooling windows whose argmax is (h,w)
__global__ void __launch_bounds__(kThreads)
maxpool_bwd_kernel(const float4* __restrict__ dy, const uchar4* __restrict__ argidx,
                   float4* __restrict__ dx, int N, int H, int W, int C4) {
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const int64_t total = (int64_t)N * H * W * C4;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * kThreads) {
    const int c4 = (int)(i % C4);
    int64_t p = i / C4;
    const int w = (int)(p % W); p /= W;
    const int h = (int)(p % H);
    const int n = (int)(p / H);
    float4 acc = make_float4(0, 0, 0, 0);
    // windows oh with oh*2-1+kh == h, kh in 0..2
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int t = h + 1 - kh;
      if (t < 0 || (t & 1)) continue;
      const int oh = t >> 1;
      if (oh >= Ho) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int u = w + 1 - kw;
        if (u < 0 || (u & 1)) continue;
        const int ow = u >> 1;
        if (ow >= Wo) continue;
        const int64_t o = ((int64_t)(n * Ho + oh) * Wo + ow) * C4 + c4;
        const uchar4 k = argidx[o];
        const float4 g = dy[o];
        const unsigned char me = (unsigned char)(kh * 3 + kw);
        if (k.x == me) acc.x += g.x;
        if (k.y == me) acc.y += g.y;
        if (k.z == me) acc.z += g.z;
        if (k.w == me) acc.w += g.w;
      }
    }
    dx[i] = acc;
  }
}

// g = dy * mask ; mask from y_out>0, or (x*scale+shift)>0 when relu, else 1
__device__ __forceinline__ float4 masked_grad(float4 dy, float4 xv, const float4* y_out, int64_t i,
                                              float4 s, float4 b, int relu) {
  if (y_out) {
    const float4 yo = y_out[i];
    return make_float4(yo.x > 0.f ? dy.x : 0.f, yo.y > 0.f ? dy.y : 0.f, yo.z > 0.f ? dy.z : 0.f,
                       yo.w > 0.f ? dy.w : 0.f);
  }
  if (relu) {
    const float4 a = fma4(xv, s, b);
    return make_float4(a.x > 0.f ? dy.x : 0.f, a.y > 0.f ? dy.y : 0.f, a.z > 0.f ? dy.z : 0.f,
                       a.w > 0.f ? dy.w : 0.f);
  }
  return dy;
}

__global__ void __launch_bounds__(kThreads)
bn_bwd_reduce_kernel(const float4* __restrict__ dy, const float4* __restrict__ x,
                     const float4* __restrict__ y_out, const float4* __restrict__ scale,
                     const float4* __restrict__ shift, const float4* __restrict__ mean,
                     const float4* __restrict__ invstd, int relu, int64_t M, int C, RowMap rm,
                     double* __restrict__ sums) {
  const int slot = threadIdx.x / rm.tpr, tin = threadIdx.x % rm.tpr;
  const int c4 = blockIdx.y * rm.tpr + tin;
  const bool active = (c4 < rm.C4) && (slot < rm.rpi);
  const int64_t rows_per_cta = (int64_t)rm.rpi * kRowsPerThread;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta;
  float4 acc[2] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
  if (active) {
    const float4 s = scale[c4], b = shift[c4], mu = mean[c4], is = invstd[c4];
    auto fold = [&](float4 dv, float4 xv, int64_t i) {
      const float4 g = masked_grad(dv, xv, y_out, i, s, b, relu);
      acc[0].x += g.x; acc[0].y += g.y; acc[0].z += g.z; acc[0].w += g.w;
      acc[1].x += g.x * (xv.x - mu.x) * is.x;
      acc[1].y += g.y * (xv.y - mu.y) * is.y;
      acc[1].z += g.z * (xv.z - mu.z) * is.z;
      acc[1].w += g.w * (xv.w - mu.w) * is.w;
    };
    // four rows per trip: the eight streaming loads are issued before the first use
    int k = 0;
    for (; k + 4 <= kRowsPerThread; k += 4) {
      const int64_t rl = r0 + (int64_t)(k + 3) * rm.rpi + slot;
      if (rl >= M) break;
      float4 xv[4], dv[4];
      int64_t idx[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        idx[u] = (r0 + (int64_t)(k + u) * rm.rpi + slot) * rm.C4 + c4;
        xv[u] = ldg_stream(x + idx[u]);
        dv[u] = ldg_stream(dy + idx[u]);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) fold(dv[u], xv[u], idx[u]);
    }
    for (; k < kRowsPerThread; ++k) {
      const int64_t r = r0 + (int64_t)k * rm.rpi + slot;
      if (r >= M) break;
      const int64_t i = r * rm.C4 + c4;
      const float4 xv = ldg_stream(x + i);
      fold(ldg_stream(dy + i), xv, i);
    }
  }
  cta_reduce_to_global<2>(acc, c4, active, rm.tpr, rm.rpi, C, sums);
}

__global__ void bn_bwd_coef_kernel(const double* __restrict__ sums, double M, int C,
                                   const float* __restrict__ gamma,
                                   const float* __restrict__ invstd, float* __restrict__ k0,
                                   float* __restrict__ k1, float* __restrict__ k2,
                                   float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double sg = sums[c], sgx = sums[C + c];
  const double gi = (double)(gamma ? gamma[c] : 1.f) * invstd[c];
  // dx = gi * (g - sg/M - xhat * sgx/M)
  k0[c] = (float)gi;
  k1[c] = (float)(sg / M);
  k2[c] = (float)(sgx / M);
  if (dgamma) dgamma[c] = (float)sgx;
  if (dbeta) dbeta[c] = (float)sg;
}

__global__ void __launch_bounds__(kThreads)
bn_bwd_apply_kernel(const float4* __restrict__ dy, const float4* __restrict__ x,
                    const float4* __restrict__ y_out, const float4* __restrict__ scale,
                    const float4* __restrict__ shift, const float4* __restrict__ mean,
                    const float4* __restrict__ invstd, int relu, const float4* __restrict__ k0,
                    const float4* __restrict__ k1, const float4* __restrict__ k2,
                    float4* __restrict__ dx, int64_t total4, int C4) {
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < total4;
       i += (int64_t)gridDim.x * kThreads) {
    const int c4 = (int)(i % C4);
    const float4 xv = ldg_stream(x + i);
    const float4 g = masked_grad(ldg_stream(dy + i), xv, y_out, i, scale[c4], shift[c4], relu);
    const float4 mu = mean[c4], is = invstd[c4], a = k0[c4], b = k1[c4], c = k2[c4];
    float4 o;
    o.x = a.x * (g.x - b.x - (xv.x - mu.x) * is.x * c.x);
    o.y = a.y * (g.y - b.y - (xv.y - mu.y) * is.y * c.y);
    o.z = a.z * (g.z - b.z - (xv.z - mu.z) * is.z * c.z);
    o.w = a.w * (g.w - b.w - (xv.w - mu.w) * is.w * c.w);
    dx[i] = o;
  }
}

__global__ void __launch_bounds__(kThreads)
add_masked_kernel(const float4* __restrict__ a, const float4* __restrict__ b,
                  const float4* __restrict__ mask_src, float4* __restrict__ dx, int64_t total4) {
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < total4;
       i += (int64_t)gridDim.x * kThreads) {
    float4 v = a[i];
    float4 q = b[i];
    if (mask_src) {
      const float4 m = mask_src[i];
      q.x = m.x > 0.f ? q.x : 0.f; q.y = m.y > 0.f ? q.y : 0.f;
      q.z = m.z > 0.f ? q.z : 0.f; q.w = m.w > 0.f ? q.w : 0.f;
    }
    v.x += q.x; v.y += q.y; v.z += q.z; v.w += q.w;
    dx[i] = v;
  }
}

__global__ void avgpool_kernel(const float* __restrict__ x, float* __restrict__ y, int HW, int C) {
  const int n = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float acc = 0.f;
  for (int p = 0; p < HW; ++p) acc += x[((int64_t)n * HW + p) * C + c];
  y[(int64_t)n * C + c] = acc / (float)HW;
}

__global__ void avgpool_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int HW,
                                   int C, int accumulate) {
  const int n = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float g = dy[(int64_t)n * C + c] / (float)HW;
  for (int p = 0; p < HW; ++p) {
    float* o = dx + ((int64_t)n * HW + p) * C + c;
    *o = accumulate ? (*o + g) : g;
  }
}

__global__ void __launch_bounds__(kThreads)
colsum_kernel(const float4* __restrict__ x, int64_t M, int C, RowMap rm, double* __restrict__ ws) {
  const int slot = threadIdx.x / rm.tpr, tin = threadIdx.x % rm.tpr;
  const int c4 = blockIdx.y * rm.tpr + tin;
  const bool active = (c4 < rm.C4) && (slot < rm.rpi);
  const int64_t rows_per_cta = (int64_t)rm.rpi * kRowsPerThread;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta;
  float4 acc[1] = {{0, 0, 0, 0}};
  if (active) {
    for (int k = 0; k < kRowsPerThread; ++k) {
      const int64_t r = r0 + (int64_t)k * rm.rpi + slot;
      if (r >= M) break;
      const float4 v = ldg_stream(x + r * rm.C4 + c4);
      acc[0].x += v.x; acc[0].y += v.y; acc[0].z += v.z; acc[0].w += v.w;
    }
  }
  cta_reduce_to_global<1>(acc, c4, active, rm.tpr, rm.rpi, C, ws);
}

__global__ void d2f_kernel(const double* __restrict__ in, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (float)in[i];
}

inline int ew_blocks(int64_t total4) {
  int64_t b = (total4 + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)kNumSMs * 16;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

}  // namespace

extern "C" __attribute__((visibility("default"))) int epb_channel_stats(const float* x, int64_t M, int C, double* stats,
                                 epb_stream_t stream) {
  EPB_CHECK_ARG(x && stats && M > 0 && C > 0 && C % 4 == 0);
  const RowMap rm = make_rowmap(C);
  const int64_t rows_per_cta = (int64_t)rm.rpi * kRowsPerThread;
  dim3 grid((unsigned)((M + rows_per_cta - 1) / rows_per_cta), rm.chunks);
  channel_stats_kernel<<<grid, kThreads, 0, as_stream(stream)>>>(
      reinterpret_cast<const float4*>(x), M, C, rm, stats);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_bn_finalize(const double* stats, int64_t M, int C, const float* gamma,
                               const float* beta, float eps, float momentum, float* running_mean,
                               float* running_var, float* scale, float* shift, float* mean,
                               float* invstd, epb_stream_t stream) {
  EPB_CHECK_ARG(stats && scale && shift && M > 0 && C > 0);
  EPB_CHECK_ARG((running_mean == nullptr) == (running_var == nullptr));
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, as_stream(stream)>>>(
      stats, (double)M, C, gamma, beta, eps, momentum, running_mean, running_var, scale, shift,
      mean, invstd);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_bn_eval_affine(int C, const float* gamma, const float* beta,
                                  const float* running_mean, const float* running_var, float eps,
                                  float* scale, float* shift, epb_stream_t stream) {
  EPB_CHECK_ARG(C > 0 && running_mean && running_var && scale && shift);
  bn_eval_affine_kernel<<<(C + 127) / 128, 128, 0, as_stream(stream)>>>(
      C, gamma, beta, running_mean, running_var, eps, scale, shift);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_bn_act(const float* x, const float* scale, const float* shift, const float* r,
                          const float* rscale, const float* rshift, int relu, float* y, int64_t M,
                          int C, epb_stream_t stream) {
  EPB_CHECK_ARG(x && y && M > 0 && C > 0 && C % 4 == 0);
  EPB_CHECK_ARG((scale == nullptr) == (shift == nullptr));
  EPB_CHECK_ARG((rscale == nullptr) == (rshift == nullptr));
  const int64_t total4 = M * (C / 4);
  bn_act_kernel<<<ew_blocks(total4), kThreads, 0, as_stream(stream)>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(scale),
      reinterpret_cast<const float4*>(shift), reinterpret_cast<const float4*>(r),
      reinterpret_cast<const float4*>(rscale), reinterpret_cast<const float4*>(rshift), relu,
      reinterpret_cast<float4*>(y), total4, C / 4);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_bn_relu_maxpool(const float* x, const float* scale, const float* shift,
                                   float* y, uint8_t* argidx, int N, int H, int W, int C,
                                   epb_stream_t stream) {
  EPB_CHECK_ARG(x && scale && shift && y && N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0);
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const int64_t total = (int64_t)N * Ho * Wo * (C / 4);
  bn_relu_maxpool_kernel<<<ew_blocks(total), kThreads, 0, as_stream(stream)>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(scale),
      reinterpret_cast<const float4*>(shift), reinterpret_cast<float4*>(y),
      reinterpret_cast<uchar4*>(argidx), N, H, W, C / 4);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_maxpool_bwd(const float* dy, const uint8_t* argidx, float* dx, int N, int H,
                               int W, int C, epb_stream_t stream) {
  EPB_CHECK_ARG(dy && argidx && dx && N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0);
  const int64_t total = (int64_t)N * H * W * (C / 4);
  maxpool_bwd_kernel<<<ew_blocks(total), kThreads, 0, as_stream(stream)>>>(
      reinterpret_cast<const float4*>(dy), reinterpret_cast<const uchar4*>(argidx),
      reinterpret_cast<float4*>(dx), N, H, W, C / 4);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_bn_bwd_reduce(const float* dy, const float* x, const float* y_out,
                                 const float* scale, const float* shift, const float* mean,
                                 const float* invstd, int relu, int64_t M, int C, double* sums,
                                 epb_stream_t stream) {
  EPB_CHECK_ARG(dy && x && scale && shift && mean && invstd && sums);
  EPB_CHECK_ARG(M > 0 && C > 0 && C % 4 == 0);
  const RowMap rm = make_rowmap(C);
  const int64_t rows_per_cta = (int64_t)rm.rpi * kRowsPerThread;
  dim3 grid((unsigned)((M + rows_per_cta - 1) / rows_per_cta), rm.chunks);
  bn_bwd_reduce_kernel<<<grid, kThreads, 0, as_stream(stream)>>>(
      reinterpret_cast<const float4*>(dy), reinterpret_cast<const float4*>(x),
      reinterpret_cast<const float4*>(y_out), reinterpret_cast<const float4*>(scale),
      reinterpret_cast<const float4*>(shift), reinterpret_cast<const float4*>(mean),
      reinterpret_cast<const float4*>(invstd), relu, M, C, rm, sums);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_bn_bwd_apply(const float* dy, const float* x, const float* y_out,
                                const float* scale, const float* shift, const float* mean,
                                const float* invstd, const float* gamma, int relu,
                                const double* sums, int64_t M, int C, float* dx, float* dgamma,
                                float* dbeta, epb_stream_t stream) {
  EPB_CHECK_ARG(dy && x && scale && shift && mean && invstd && sums && dx);
  EPB_CHECK_ARG(M > 0 && C > 0 && C % 4 == 0);
  EPB_CHECK_ARG(C <= 8192);
  cudaStream_t st = as_stream(stream);
  float* coef = nullptr;
  int rc = epb_workspace(EPB_WS_BNCOEF, 3 * (size_t)8192 * sizeof(float), st, (void**)&coef);
  if (rc) return rc;
  float* k0 = coef;
  float* k1 = coef + 8192;
  float* k2 = coef + 2 * 8192;
  bn_bwd_coef_kernel<<<(C + 127) / 128, 128, 0, st>>>(sums, (double)M, C, gamma, invstd, k0, k1, k2,
                                                      dgamma, dbeta);
  EPB_LAUNCH_CHECK();
  const int64_t total4 = M * (C / 4);
  bn_bwd_apply_kernel<<<ew_blocks(total4), kThreads, 0, st>>>(
      reinterpret_cast<const float4*>(dy), reinterpret_cast<const float4*>(x),
      reinterpret_cast<const float4*>(y_out), reinterpret_cast<const float4*>(scale),
      reinterpret_cast<const float4*>(shift), reinterpret_cast<const float4*>(mean),
      reinterpret_cast<const float4*>(invstd), relu, reinterpret_cast<const float4*>(k0),
      reinterpret_cast<const float4*>(k1), reinterpret_cast<const float4*>(k2),
      reinterpret_cast<float4*>(dx), total4, C / 4);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_add_masked(const float* a, const float* b, const float* mask_src, float* dx,
                              int64_t n, epb_stream_t stream) {
  EPB_CHECK_ARG(a && b && dx && n > 0 && n % 4 == 0);
  add_masked_kernel<<<ew_blocks(n / 4), kThreads, 0, as_stream(stream)>>>(
      reinterpret_cast<const float4*>(a), reinterpret_cast<const float4*>(b),
      reinterpret_cast<const float4*>(mask_src), reinterpret_cast<float4*>(dx), n / 4);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_avgpool(const float* x, float* y, int N, int HW, int C, epb_stream_t stream) {
  EPB_CHECK_ARG(x && y && N > 0 && HW > 0 && C > 0);
  avgpool_kernel<<<dim3((C + 127) / 128, N), 128, 0, as_stream(stream)>>>(x, y, HW, C);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_avgpool_bwd(const float* dy, float* dx, int N, int HW, int C, int accumulate,
                               epb_stream_t stream) {
  EPB_CHECK_ARG(dy && dx && N > 0 && HW > 0 && C > 0);
  avgpool_bwd_kernel<<<dim3((C + 127) / 128, N), 128, 0, as_stream(stream)>>>(dy, dx, HW, C,
                                                                              accumulate);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_colsum(const float* x, int64_t M, int C, float* out, epb_stream_t stream) {
  EPB_CHECK_ARG(x && out && M > 0 && C > 0 && C % 4 == 0 && C <= 8192);
  cudaStream_t st = as_stream(stream);
  float* coef = nullptr;
  int rc = epb_workspace(EPB_WS_BNCOEF, 3 * (size_t)8192 * sizeof(float), st, (void**)&coef);
  if (rc) return rc;
  double* ws = reinterpret_cast<double*>(coef);  // 8192 doubles fit in 3*8192 floats
  EPB_CUDA(cudaMemsetAsync(ws, 0, sizeof(double) * C, st));
  const RowMap rm = make_rowmap(C);
  const int64_t rows_per_cta = (int64_t)rm.rpi * kRowsPerThread;
  dim3 grid((unsigned)((M + rows_per_cta - 1) / rows_per_cta), rm.chunks);
  colsum_kernel<<<grid, kThreads, 0, st>>>(reinterpret_cast<const float4*>(x), M, C, rm, ws);
  EPB_LAUNCH_CHECK();
  d2f_kernel<<<(C + 127) / 128, 128, 0, st>>>(ws, out, C);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}
