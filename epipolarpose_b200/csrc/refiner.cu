// Eval-mode refiner MLP (LinearModelPG.forward, refiner/model.py:117-143 of the reference) in one
// C-ABI call: one launch per linear layer, each
//     Y = [relu]((X W^T + b) * scale + shift) [+ R1] [+ R2]
// with eval BatchNorm folded into (scale, shift), dropout the identity, the residual joins of the
// graph in the epilogue, and optionally the input normalisation at the first layer's load and
// the label denormalisation in the last layer's epilogue.
//
// Arithmetic: fp32 CUDA-core FMAs; every output is accumulated by ONE thread, fmaf in k order
// 0..K-1 from +0, then the epilogue with explicitly rounded adds / multiplies (no contraction).
// So a row's result does not depend on N, on the row's position or on which kernel ran it
// (batch invariance): the column-slab GEMV form (small N) and the 2-D tiled form (large N) give
// the same bits.  Tensor cores are not used: at inference sizes a layer is bound by its weight
// reads, and the exact-fp32 batch-invariant result is what the callers rely on.
#include "common.cuh"

namespace {

constexpr int kNumLayers = 12;
constexpr int kNumBN = 10;
constexpr int kGemvRows = 4;        // rows per GEMV block (one accumulator each per thread)
constexpr int kGemvCols = 32;       // columns per GEMV block (one warp, one column per lane)
constexpr int kGemvMaxN = 128;      // N at or below which the GEMV form runs
constexpr int kTile = 64, kTK = 16; // tiled form: 64x64 outputs per 256-thread block, 4x4 per thread

inline int pad4(int x) { return (x + 3) / 4 * 4; }

// Layer table of LinearModelPG (num_stage = 2).  Activations live in workspace slots:
//   slot 0 = p1 [N][out_p]; slots 1..4 = [N][L] (1: inp, the pre-processing output, alive to the end).
// Source -1 = the caller's input x; destination -1 = the caller's output.
struct LayerDesc { int kin, kout, bn, relu, src, dst, r1, r2; };  // kin/kout: 0 = in, 1 = L, 2 = out
constexpr LayerDesc kLayers[kNumLayers] = {
    {0, 1, 1, 1, -1, 1, -1, -1},  // w1, batch_norm1, relu                      -> inp
    {1, 1, 1, 1, 1, 2, -1, -1},   // stage0 w1
    {1, 1, 1, 1, 2, 3, 1, -1},    // stage0 w2, + x                             -> out
    {1, 1, 1, 1, 3, 2, -1, -1},   // stage0 w3
    {1, 1, 1, 1, 2, 4, 3, -1},    // stage0 w4, + out                           -> s1
    {1, 2, 0, 0, 4, 0, -1, -1},   // w2                                         -> p1
    {2, 1, 1, 1, 0, 2, 4, 1},     // w3, batch_norm3, relu, (+ s1) + inp        -> y
    {1, 1, 1, 1, 2, 3, -1, -1},   // stage1 w1
    {1, 1, 1, 1, 3, 4, 2, -1},    // stage1 w2, + y                             -> out
    {1, 1, 1, 1, 4, 3, -1, -1},   // stage1 w3
    {1, 1, 1, 1, 3, 2, 4, 1},     // stage1 w4, (+ out) + inp                   -> y
    {1, 2, 0, 0, 2, -1, -1, -1},  // w4                                         -> p2
};

struct Dims {
  int in, L, out;
  int kdim(int code) const { return code == 0 ? in : (code == 1 ? L : out); }
};

// Offsets (floats) of the flat parameter buffer: per layer W [O_p][K_p], b [O_p], and for BN
// layers scale [O_p], shift [O_p]; then data_mean, data_std [in_p], labels_mean, labels_std [out_p].
struct Layout {
  int64_t w[kNumLayers], b[kNumLayers], scale[kNumLayers], shift[kNumLayers];
  int64_t dmean, dstd, lmean, lstd, total;
  Layout(const Dims& d) {
    int64_t o = 0;
    for (int l = 0; l < kNumLayers; ++l) {
      const int K = pad4(d.kdim(kLayers[l].kin)), O = pad4(d.kdim(kLayers[l].kout));
      w[l] = o; o += (int64_t)O * K;
      b[l] = o; o += O;
      scale[l] = shift[l] = -1;
      if (kLayers[l].bn) { scale[l] = o; o += O; shift[l] = o; o += O; }
    }
    dmean = o; o += pad4(d.in);
    dstd = o; o += pad4(d.in);
    lmean = o; o += pad4(d.out);
    lstd = o; o += pad4(d.out);
    total = o;
  }
};

// ------------------------------------------------------------------------------ prepare
struct PrepJob {
  const float* src[4];   // copy: src[0] [rows][cols]; bn: gamma, beta, running_mean, running_var
  int kind;              // 0 copy with zero padding, 1 BatchNorm fold
  int rows, cols, cols_p, rows_p;
  int64_t dst, dst2;     // float offsets into params (bn: scale, shift)
};
constexpr int kMaxJobs = 2 * kNumLayers + kNumBN + 4;
struct PrepJobs { PrepJob j[kMaxJobs]; };

__global__ void refiner_prepare_kernel(PrepJobs jobs, float* __restrict__ params, float eps) {
  const PrepJob& jb = jobs.j[blockIdx.y];
  const int64_t n = (int64_t)jb.rows_p * jb.cols_p;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / jb.cols_p), c = (int)(i % jb.cols_p);
    if (jb.kind == 0) {
      params[jb.dst + i] = (r < jb.rows && c < jb.cols) ? jb.src[0][(int64_t)r * jb.cols + c] : 0.f;
    } else {
      float scale = 1.f, shift = 0.f;
      if (c < jb.cols) {   // torch BatchNorm1d eval: (z - mean) / sqrt(var + eps) * gamma + beta
        const double s = (double)jb.src[0][c] / sqrt((double)jb.src[3][c] + (double)eps);
        scale = (float)s;
        shift = (float)((double)jb.src[1][c] - (double)jb.src[2][c] * s);
      }
      params[jb.dst + c] = scale;
      params[jb.dst2 + c] = shift;
    }
  }
}

// ------------------------------------------------------------------------------ forward
struct LayerArgs {
  const float* x; int ldx, K, Kp;          // input rows (row stride ldx), K real, Kp = pad4(K)
  const float* w; const float* b;          // W [Op][Kp], b [Op]
  const float* scale; const float* shift;  // or null (no BatchNorm)
  const float* nmean; const float* nstd;   // input normalisation (first layer) or null
  const float* dmean; const float* dstd;   // output denormalisation (last layer) or null
  const float* r1; const float* r2; int ldr;
  float* y; int ldy, Op, Ostore;           // Ostore: columns written (Op, or the real width)
  int relu, N;
};

__device__ __forceinline__ float load_x(const LayerArgs& a, int n, int k) {
  if (n >= a.N || k >= a.K) return 0.f;
  const float v = a.x[(int64_t)n * a.ldx + k];
  return a.nmean ? __fdiv_rn(__fsub_rn(v, a.nmean[k]), a.nstd[k]) : v;
}

__device__ __forceinline__ void epilogue(const LayerArgs& a, int n, int o, float acc) {
  if (n >= a.N || o >= a.Ostore) return;
  float y = __fadd_rn(acc, a.b[o]);
  if (a.scale) y = __fadd_rn(__fmul_rn(y, a.scale[o]), a.shift[o]);
  if (a.relu) y = y < 0.f ? 0.f : y;
  const int64_t ri = (int64_t)n * a.ldr + o;
  if (a.r1) y = __fadd_rn(y, a.r1[ri]);
  if (a.r2) y = __fadd_rn(y, a.r2[ri]);
  if (a.dmean) y = __fadd_rn(__fmul_rn(y, a.dstd[o]), a.dmean[o]);
  a.y[(int64_t)n * a.ldy + o] = y;
}

// Small N: one warp per 32 output columns and kGemvRows rows; lane = column.  The rows are staged
// in shared memory (zero-padded to whole k chunks).  The warp's 32 weight rows go through shared
// memory in chunks of kGemvK columns, loaded coalesced (four 128-byte row pieces per instruction),
// the next chunk in flight while the current one is consumed.
constexpr int kGemvK = 32;
__global__ void __launch_bounds__(kGemvCols) refiner_gemv_kernel(LayerArgs a) {
  extern __shared__ __align__(16) float xs[];          // [kGemvRows][Kc]
  __shared__ float ws[kGemvCols][kGemvK + 1];
  const int lane = threadIdx.x;
  const int o0 = blockIdx.x * kGemvCols, n0 = blockIdx.y * kGemvRows;
  const int Kc = (a.Kp + kGemvK - 1) / kGemvK * kGemvK;
  for (int r = 0; r < kGemvRows; ++r) {     // independent loads, unrolled so that many are in flight
#pragma unroll 8
    for (int k = lane; k < Kc; k += kGemvCols) xs[r * Kc + k] = load_x(a, n0 + r, k);
  }
  constexpr int kLoads = kGemvCols * kGemvK / 4 / 32;   // float4 per lane per chunk
  float4 buf[kLoads];
  auto fetch = [&](int k0) {
#pragma unroll
    for (int i = 0; i < kLoads; ++i) {
      const int f = i * 32 + lane, row = f / (kGemvK / 4), k = k0 + (f % (kGemvK / 4)) * 4;
      buf[i] = (o0 + row < a.Op && k < a.Kp)
                   ? __ldg(reinterpret_cast<const float4*>(a.w + (int64_t)(o0 + row) * a.Kp + k))
                   : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  float acc[kGemvRows];
#pragma unroll
  for (int r = 0; r < kGemvRows; ++r) acc[r] = 0.f;
  fetch(0);
  for (int k0 = 0; k0 < Kc; k0 += kGemvK) {
    __syncwarp();
#pragma unroll
    for (int i = 0; i < kLoads; ++i) {
      const int f = i * 32 + lane, row = f / (kGemvK / 4), k = (f % (kGemvK / 4)) * 4;
      ws[row][k] = buf[i].x; ws[row][k + 1] = buf[i].y; ws[row][k + 2] = buf[i].z; ws[row][k + 3] = buf[i].w;
    }
    if (k0 + kGemvK < Kc) fetch(k0 + kGemvK);
    __syncwarp();
#pragma unroll 16
    for (int k = 0; k < kGemvK; ++k) {
      const float w = ws[lane][k];
#pragma unroll
      for (int r = 0; r < kGemvRows; ++r) acc[r] = __fmaf_rn(xs[r * Kc + k0 + k], w, acc[r]);
    }
  }
#pragma unroll
  for (int r = 0; r < kGemvRows; ++r) epilogue(a, n0 + r, o0 + lane, acc[r]);
}

// Large N: 64x64 output tile per 256-thread block, 4x4 outputs per thread, k in steps of 16
// through shared memory (zero beyond Kp; fmaf(0, 0, acc) leaves acc unchanged, and acc is never
// -0 since it starts at +0).
__global__ void __launch_bounds__(256) refiner_tiled_kernel(LayerArgs a) {
  __shared__ __align__(16) float As[kTK][kTile + 4];   // X^T tile
  __shared__ __align__(16) float Bs[kTK][kTile + 4];   // W^T tile
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int n0 = blockIdx.y * kTile, o0 = blockIdx.x * kTile;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < a.Kp; k0 += kTK) {
    const int kk = tid % kTK, k = k0 + kk;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = tid / kTK + 16 * i;
      As[kk][r] = load_x(a, n0 + r, k);
      const int o = o0 + r;
      Bs[kk][r] = (o < a.Op && k < a.Kp) ? __ldg(a.w + (int64_t)o * a.Kp + k) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kTK; ++q) {
      const float4 x = *reinterpret_cast<const float4*>(&As[q][ty * 4]);
      const float4 w = *reinterpret_cast<const float4*>(&Bs[q][tx * 4]);
      const float xv[4] = {x.x, x.y, x.z, x.w}, wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = __fmaf_rn(xv[i], wv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) epilogue(a, n0 + ty * 4 + i, o0 + tx * 4 + j, acc[i][j]);
}

constexpr int kNumSources = 2 * kNumLayers + 4 * kNumBN + 4;
constexpr int kMaxWidth = 2048;     // GEMV shared memory: kGemvRows rows of K floats (32 KB) + the 4.2 KB weight tile

bool dims_ok(const Dims& d) {
  return d.in > 0 && d.in <= kMaxWidth && d.L > 0 && d.L <= kMaxWidth && d.L % 4 == 0 && d.out > 0 &&
         d.out <= kMaxWidth;
}

}  // namespace

extern "C" __attribute__((visibility("default"))) int epb_refiner_sizes(int in, int L, int out, int N,
                                                                       int64_t* param_floats,
                                                                       int64_t* ws_floats) {
  const Dims d{in, L, out};
  EPB_CHECK_ARG(dims_ok(d) && N >= 0);
  if (param_floats) *param_floats = Layout(d).total;
  if (ws_floats) *ws_floats = (int64_t)N * (pad4(out) + 4LL * L);
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_refiner_prepare(int in, int L, int out,
                                                                         const float* const* src,
                                                                         float eps, float* params,
                                                                         epb_stream_t stream) {
  const Dims d{in, L, out};
  EPB_CHECK_ARG(dims_ok(d) && src && params);
  const Layout lay(d);
  PrepJobs jobs;
  int nj = 0, s = 0;
  for (int l = 0; l < kNumLayers; ++l) {
    const int K = d.kdim(kLayers[l].kin), O = d.kdim(kLayers[l].kout);
    jobs.j[nj++] = PrepJob{{src[s], nullptr, nullptr, nullptr}, 0, O, K, pad4(K), pad4(O), lay.w[l], 0};
    jobs.j[nj++] = PrepJob{{src[s + 1], nullptr, nullptr, nullptr}, 0, 1, O, pad4(O), 1, lay.b[l], 0};
    s += 2;
  }
  for (int l = 0; l < kNumLayers; ++l) {
    if (!kLayers[l].bn) continue;
    const int O = d.kdim(kLayers[l].kout);
    jobs.j[nj++] = PrepJob{{src[s], src[s + 1], src[s + 2], src[s + 3]}, 1, 1, O, pad4(O), 1,
                           lay.scale[l], lay.shift[l]};
    s += 4;
  }
  const int64_t norm_dst[4] = {lay.dmean, lay.dstd, lay.lmean, lay.lstd};
  for (int i = 0; i < 4; ++i) {
    const int C = i < 2 ? in : out;
    jobs.j[nj++] = PrepJob{{src[s + i], nullptr, nullptr, nullptr}, 0, 1, C, pad4(C), 1, norm_dst[i], 0};
  }
  for (int i = 0; i < kNumSources; ++i) EPB_CHECK_ARG(src[i] != nullptr);
  refiner_prepare_kernel<<<dim3(64, nj), 256, 0, as_stream(stream)>>>(jobs, params, eps);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_refiner_forward(int in, int L, int out,
                                                                         const float* params, const float* x,
                                                                         int N, int normalize_in,
                                                                         int denormalize_out, float* y,
                                                                         float* ws, int64_t ws_floats,
                                                                         int force_form, epb_stream_t stream) {
  const Dims d{in, L, out};
  EPB_CHECK_ARG(dims_ok(d) && params && x && y && N >= 0 && force_form >= 0 && force_form <= 2);
  const int64_t need = (int64_t)N * (pad4(out) + 4LL * L);
  EPB_CHECK_ARG(N == 0 || (ws && ws_floats >= need));
  EPB_CHECK_ARG(((uintptr_t)params & 15) == 0 && ((uintptr_t)ws & 15) == 0);
  if (N == 0) return EPB_OK;
  const Layout lay(d);
  const int outp = pad4(out);
  float* slot[5] = {ws, ws + (int64_t)N * outp, nullptr, nullptr, nullptr};
  for (int i = 2; i < 5; ++i) slot[i] = slot[i - 1] + (int64_t)N * L;
  const bool gemv = force_form == 1 || (force_form == 0 && N <= kGemvMaxN);
  // grid.y limit: N <= 262140 rows per call for the GEMV form, 4194240 for the tiled form
  EPB_CHECK_ARG((gemv ? (N + kGemvRows - 1) / kGemvRows : (N + kTile - 1) / kTile) <= 65535);
  for (int l = 0; l < kNumLayers; ++l) {
    const LayerDesc& ld = kLayers[l];
    LayerArgs a;
    a.K = d.kdim(ld.kin);
    a.Kp = pad4(a.K);
    a.Op = pad4(d.kdim(ld.kout));
    a.x = ld.src < 0 ? x : slot[ld.src];
    a.ldx = ld.src < 0 ? in : (ld.src == 0 ? outp : L);
    a.w = params + lay.w[l];
    a.b = params + lay.b[l];
    a.scale = ld.bn ? params + lay.scale[l] : nullptr;
    a.shift = ld.bn ? params + lay.shift[l] : nullptr;
    a.nmean = (ld.src < 0 && normalize_in) ? params + lay.dmean : nullptr;
    a.nstd = (ld.src < 0 && normalize_in) ? params + lay.dstd : nullptr;
    a.dmean = (ld.dst < 0 && denormalize_out) ? params + lay.lmean : nullptr;
    a.dstd = (ld.dst < 0 && denormalize_out) ? params + lay.lstd : nullptr;
    a.r1 = ld.r1 < 0 ? nullptr : slot[ld.r1];
    a.r2 = ld.r2 < 0 ? nullptr : slot[ld.r2];
    a.ldr = L;
    a.y = ld.dst < 0 ? y : slot[ld.dst];
    a.ldy = ld.dst < 0 ? out : (ld.dst == 0 ? outp : L);
    a.Ostore = ld.dst < 0 ? out : a.Op;
    a.relu = ld.relu;
    a.N = N;
    if (gemv) {
      const dim3 grid((a.Op + kGemvCols - 1) / kGemvCols, (N + kGemvRows - 1) / kGemvRows);
      const int Kc = (a.Kp + kGemvK - 1) / kGemvK * kGemvK;
      refiner_gemv_kernel<<<grid, kGemvCols, kGemvRows * Kc * sizeof(float), as_stream(stream)>>>(a);
    } else {
      const dim3 grid((a.Op + kTile - 1) / kTile, (N + kTile - 1) / kTile);
      refiner_tiled_kernel<<<grid, 256, 0, as_stream(stream)>>>(a);
    }
    EPB_LAUNCH_CHECK();
  }
  return EPB_OK;
}
