// Split-fp16 ("f16x3") tensor-core path of the tap-list implicit GEMM (include/epb.h,
// epb_conv16_fprop): forward convs, transposed convs (one call per output phase) and both of
// their data gradients, i.e. the cuDNN call sites behind nn.Conv2d / nn.ConvTranspose2d of
// lib/models/pose3d_resnet.py:12-15,55-60,99,116-122,132,171-178 and their autograd.
//
//   out[m, co] = (1 / (s_in * s_w)) * sum_k A[m, k] * W[co, k],   m = phase-grid pixel,
//   k = (tap, ci),  A = hi + lo, W = hi + lo  (fp16 planes),
//   A*W ~= A_lo*W_hi + A_hi*W_lo + A_hi*W_hi   (three wgmma passes, FP32 accumulate).
//
// Both operands are TMA-fed: the activation planes are post-BatchNorm/ReLU (written once by
// split16.cu), so an M tile of 128 pixels is ONE 5-D box load per plane and tap -- (64 channels,
// tw, th, tn) of the (C, W, H, N, plane) tensor, shifted by the tap offset; the zero padding
// of the convolution is the TMA out-of-bounds fill, strided convs use the four parity views of
// the tensor.  Weight planes are 3-D (k, co, plane) box loads.
//
// One persistent CTA per SM on the pipeline of tc_common.cuh: warpgroup 0 is the TMA
// producer (one lane: A hi/lo + B hi/lo boxes per k-block), warpgroups 1-2 the consumers
// (4 k-steps x 3 wgmma m64nBNk16 per k-block).  The epilogue scales, adds the bias, stores
// or adds, and keeps the BatchNorm statistics of a run of tiles of one N tile in the
// per-warp slices, flushed once per run.
#include "split16_common.cuh"

namespace {

constexpr int BM = 128;
constexpr int kThreads16 = 384;
constexpr int kConsumers = 256;
constexpr int kStageBudget = 200 * 1024;

struct Plan16 {
  epb_phase_grid grid;           // pixel tiles of the phase grid (M side), tap views
  int Ho, Wo, Cout, os, ph, pw;  // output tensor / phase
  int Wv, Hv;                    // extent of the output phase view (rows beyond it are not stored)
  int T, CB;                     // taps, channel blocks of 64 per tap
  int n_tiles;
  int accumulate;
  int m_fastest;                 // tile order: consecutive tiles walk M (statistics runs) or N
  int koff[EPB_MAX_TAPS];        // wt[t] * Cin: k offset of the tap inside a packed weight row
};

struct Maps16 {
  CUtensorMap a[4];
  CUtensorMap w;
};

template <int BN>
struct Cfg16 {
  static constexpr int A_PLANE = BM * 128;
  static constexpr int B_PLANE = BN * 128;
  static constexpr int A_BYTES = 2 * A_PLANE;
  static constexpr int B_BYTES = 2 * B_PLANE;
  static constexpr int STAGE = A_BYTES + B_BYTES;
  static constexpr int S_ = kStageBudget / STAGE;
  static constexpr int S = S_ > 6 ? 6 : S_;
  static constexpr int STAT_BYTES = (kConsumers / 32) * 2 * BN * 4;   // per warp [sum | sum of squares][BN]
  static constexpr int SMEM = S * STAGE + 1024 /*align*/ + 256 /*barriers*/ + STAT_BYTES;
  static_assert(SMEM <= 227 * 1024, "shared memory budget");
  static_assert(S >= 2, "ring too shallow");
};

template <int BN>
__global__ void __launch_bounds__(kThreads16, 1)
conv16_kernel(const __grid_constant__ Plan16 P, const __grid_constant__ Maps16 maps,
              const float* __restrict__ in_sc, const float* __restrict__ w_sc,
              const float* __restrict__ bias, float* __restrict__ out,
              double* __restrict__ stats) {
  using C = Cfg16<BN>;
  const epb_phase_grid& G = P.grid;
  constexpr int CTRL = C::S * C::STAGE;
  extern __shared__ uint8_t smem_raw[];
  tc::Ring<C::S, C::STAGE> ring(smem_raw, 0, CTRL, CTRL + 64);     // full[8], empty[8]
  float* sstat = reinterpret_cast<float*>(ring.sm + CTRL + 256);   // [8 warps][2][BN]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int KB = P.T * P.CB;
  const int total_tiles = G.tiles * P.n_tiles;
  auto nt_of = [&](int tile) { return P.m_fastest ? tile / G.tiles : tile % P.n_tiles; };
  auto mt_of = [&](int tile) { return P.m_fastest ? tile % G.tiles : tile / P.n_tiles; };

  if (threadIdx.x == 0) ring.init(1, kConsumers / 32);   // producer's arrive.expect_tx; consumer warps
  __syncthreads();

  if (warp < 4) {
    // =================================================== TMA producer
    if (warp == 0 && lane == 0) {
      for (int v = 0; v < 4; ++v) tc::tma_prefetch_desc(&maps.a[v]);
      tc::tma_prefetch_desc(&maps.w);
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int nt = nt_of(tile);
        int w0, h0, n0;
        G.tile_origin(mt_of(tile), w0, h0, n0);
        int t = 0, cb = 0;
        for (int kb = 0; kb < KB; ++kb) {
          tc::mbar_wait(ring.empty(ring.stage), ring.phase ^ 1);
          const uint32_t fb = ring.full(ring.stage);
          tc::mbar_arrive_expect_tx(fb, C::STAGE);
          const uint32_t a_dst = ring.stage_addr(ring.stage);
          const CUtensorMap* am = &maps.a[G.map[t]];
          const int cx = cb * 64, wx = w0 + G.dwq[t], hx = h0 + G.dhq[t];
          tc::tma_load_5d(a_dst, am, fb, cx, wx, hx, n0, 0);
          tc::tma_load_5d(a_dst + C::A_PLANE, am, fb, cx, wx, hx, n0, 1);
          const uint32_t b_dst = a_dst + C::A_BYTES;
          const int kx = P.koff[t] + cx, rx = nt * BN;
          tc::tma_load_3d(b_dst, &maps.w, fb, kx, rx, 0);
          tc::tma_load_3d(b_dst + C::B_PLANE, &maps.w, fb, kx, rx, 1);
          if (++cb == P.CB) { cb = 0; ++t; }
          ring.advance();
        }
      }
    }
    return;
  }

  // =================================================== consumers (2 warpgroups)
  const int wgc = (warp >> 2) - 1;             // rows 64 * wgc .. + 63 of the tile
  const int ct = threadIdx.x - 128;            // 0..255
  float* wstat = sstat + (ct >> 5) * 2 * BN;   // this warp's statistics slice
  const int lc = (lane & 3) * 2;
  const int ra = wgc * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows ra, ra + 8
  const float alpha = in_sc[1] * w_sc[1];
  const int twh = G.tw * G.th;
  if (stats) {
    for (int c = ct; c < (kConsumers / 32) * 2 * BN; c += kConsumers) sstat[c] = 0.f;
    tc::named_sync(1, kConsumers);
  }

  float acc[BN / 2];
  int nt_prev = -1;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int nt = nt_of(tile);
    // statistics: one flush per run of tiles of the same N tile
    if (stats && nt_prev >= 0 && nt != nt_prev)
      tc::stats_flush<BN, kConsumers / 32>(sstat, ct, nt_prev, P.Cout, stats);
    nt_prev = nt;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < KB; ++kb)
      ring.consume(acc, [&](uint32_t st) {
        const uint32_t a_hi = st + wgc * 64 * 128, b_hi = st + C::A_BYTES;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)               // 4 x K = 16 fp16 (32 bytes)
          tc::mma3_f16<0, 0>(acc, tc::desc_kmajor_sw128(a_hi + kk * 32),
                             tc::desc_kmajor_sw128(a_hi + C::A_PLANE + kk * 32),
                             tc::desc_kmajor_sw128(b_hi + kk * 32),
                             tc::desc_kmajor_sw128(b_hi + C::B_PLANE + kk * 32));
      });
    ring.drain(acc);

    // ---- epilogue straight from the fragment: rows ra (h = 0) and ra + 8 (h = 1)
    int w0, h0, n0;
    G.tile_origin(mt_of(tile), w0, h0, n0);
    float* orow[2];
    bool srow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = ra + 8 * h;
      const int w = w0 + r % G.tw, hh = h0 + (r / G.tw) % G.th, n = n0 + r / twh;
      orow[h] = (w < P.Wv && hh < P.Hv && n < G.N)
                    ? out + (((int64_t)n * P.Ho + (int64_t)hh * P.os + P.ph) * P.Wo +
                             (int64_t)w * P.os + P.pw) * P.Cout
                    : nullptr;
      srow[h] = w < G.Wp && hh < G.Hp && n < G.N;
    }
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int cl = 8 * j + lc, col = nt * BN + cl;
      float v[2][2];
      float2 b = make_float2(0.f, 0.f);
      if (bias && col < P.Cout) b = *reinterpret_cast<const float2*>(bias + col);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        v[h][0] = acc[4 * j + 2 * h] * alpha + b.x;
        v[h][1] = acc[4 * j + 2 * h + 1] * alpha + b.y;
        if (orow[h] && col < P.Cout) {
          float2* o = reinterpret_cast<float2*>(orow[h] + col);
          float2 x = make_float2(v[h][0], v[h][1]);
          if (P.accumulate) {
            const float2 pv = *o;
            x.x += pv.x; x.y += pv.y;
          }
          *o = x;
        }
      }
      if (stats) tc::stats_add<BN>(wstat, cl, v, srow);
    }
  }
  if (stats && nt_prev >= 0) tc::stats_flush<BN, kConsumers / 32>(sstat, ct, nt_prev, P.Cout, stats);
}

}  // namespace

extern "C" __attribute__((visibility("default"))) int epb_conv16_fprop(
    const epb_conv_geom* g, const epb_half* in, const float* in_sc, const epb_half* w,
    const float* w_sc, const float* bias, float* out, double* stats, epb_stream_t stream) {
  int rc = epb_conv_geom_check(g);
  if (rc) return rc;
  EPB_CHECK_ARG(in && in_sc && w && w_sc && out);
  EPB_CHECK_ARG(g->Cin % 64 == 0 && g->Cout % 4 == 0 && g->Cout >= 4);
  EPB_CHECK_ARG(g->is == 1 || g->is == 2);
  EPB_CHECK_ARG(!(stats && g->accumulate));
  EPB_CHECK_ARG((reinterpret_cast<uintptr_t>(in) & 127) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0);
  EPB_CHECK_ARG((reinterpret_cast<uintptr_t>(out) & 7) == 0 && (reinterpret_cast<uintptr_t>(bias) & 7) == 0);
  Plan16 P;
  Maps16 maps;
  memset(&maps, 0, sizeof(maps));
  bool dense;
  rc = epb_plan_phase_grid(g, in, BM, P.grid, maps.a, dense);
  if (rc) return rc;
  // a dense layer's output is the same [M][Cout] matrix as its phase grid
  P.Ho = dense ? 1 : g->Ho; P.Wo = dense ? P.grid.Wp : g->Wo; P.Cout = g->Cout; P.os = g->os;
  P.ph = dense ? 0 : g->ph; P.pw = dense ? 0 : g->pw;
  P.Wv = dense ? P.grid.Wp : (g->Wo - g->pw + g->os - 1) / g->os;
  P.Hv = dense ? 1 : (g->Ho - g->ph + g->os - 1) / g->os;
  P.T = g->T; P.CB = g->Cin / 64; P.accumulate = g->accumulate;
  for (int t = 0; t < g->T; ++t) P.koff[t] = g->wt[t] * g->Cin;
  // tile order: statistics want runs of tiles with the same N tile (one flush per run); without
  // statistics, N-fastest lets the concurrently running tiles of one M tile share its A rows in L2
  P.m_fastest = stats != nullptr;
  // N tile: the 128-column accumulator of a consumer warpgroup (64 fp32 registers per thread),
  // 64 columns for narrow layers
  const int bn = g->Cout <= 64 ? 64 : 128;
  P.n_tiles = (g->Cout + bn - 1) / bn;
  const int64_t K = (int64_t)g->Tw * g->Cin;
  const cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)g->Cout, 2};
  const cuuint64_t strides[2] = {(cuuint64_t)K * 2, (cuuint64_t)K * 2 * g->Cout};
  const cuuint32_t box[3] = {64, (cuuint32_t)bn, 1};
  rc = epb_encode_map(&maps.w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, w, dims, strides, box,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "weights");
  if (rc) return rc;
  const int64_t tiles = (int64_t)P.grid.tiles * P.n_tiles;
  const unsigned grid = (unsigned)(tiles < kNumSMs ? tiles : kNumSMs);
  cudaStream_t st = as_stream(stream);
  if (bn == 64)
    return tc::launch<conv16_kernel<64>>(grid, kThreads16, Cfg16<64>::SMEM, st, P, maps, in_sc,
                                         w_sc, bias, out, stats);
  return tc::launch<conv16_kernel<128>>(grid, kThreads16, Cfg16<128>::SMEM, st, P, maps, in_sc,
                                        w_sc, bias, out, stats);
}
