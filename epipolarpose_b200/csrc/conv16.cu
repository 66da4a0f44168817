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
// (4 k-steps x 3 wgmma m64nBNk16 per k-block).  The epilogue scales and adds the bias; each
// consumer warp writes its 16 tile rows 32 columns at a time into its own 2 KB staging box and
// one lane hands the box to a TMA store (a TMA reduce-add with `accumulate`), so the output
// write runs in the background while the warp goes on to the next chunk and the next tile's
// MMAs.  The store map has the extents of the output view: TMA drops the rows and columns
// beyond it.  The BatchNorm statistics of a run of tiles of one N tile are kept in the
// per-warp slices from the register values, flushed once per run.
//
// Split-K (epb_conv16_fprop_splitk): a layer with few tiles leaves most SMs idle while each CTA
// walks the whole K loop.  The work items are then (tile, split) pairs, split s covering the
// contiguous k-blocks [s KB / S, (s + 1) KB / S); the same kernel (SPLIT = true) stores each
// item's scaled accumulator into a dense fp32 workspace [S][tiles * 128][Cout] through the same
// staging boxes, and conv16_splitk_reduce sums the splits in the order 0..S-1, adds the bias,
// writes the output view and adds the statistics of its valid rows.
#include "split16_common.cuh"

namespace {

constexpr int BM = 128;
constexpr int kThreads16 = 384;
constexpr int kConsumers = 256;
constexpr int kStageBudget = 200 * 1024;
constexpr int kBoxBytes = 16 * 128;   // staging box of a consumer warp: 16 rows x 32 fp32, SWIZZLE_128B

struct Plan16 {
  epb_phase_grid grid;           // pixel tiles of the phase grid (M side), tap views
  int Cout;
  int Wv, Hv;                    // extent of the output phase view (rows beyond it are not stored)
  int T, CB;                     // taps, channel blocks of 64 per tap
  int n_tiles;
  int accumulate;
  int m_fastest;                 // tile order: consecutive tiles walk M (statistics runs) or N
  int splits;                    // K splits per tile (SPLIT kernel only)
  int koff[EPB_MAX_TAPS];        // wt[t] * Cin: k offset of the tap inside a packed weight row
};

struct Maps16 {
  CUtensorMap a[4];
  CUtensorMap w;
  CUtensorMap out;               // fp32 (Cout, Wv, Hv, N) output view, box 32 x one warp's 16 rows;
                                 // SPLIT: the (Cout, 16, tiles * 8, S) workspace, box 32 x 16 x 1 x 1
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
  static constexpr int BOX_BYTES = (kConsumers / 32) * kBoxBytes;
  static constexpr int STAT_BYTES = (kConsumers / 32) * 2 * BN * 4;   // per warp [sum | sum of squares][BN]
  static constexpr int SMEM =
      S * STAGE + BOX_BYTES + 1024 /*align*/ + 256 /*barriers*/ + STAT_BYTES;
  static_assert(SMEM <= 227 * 1024, "shared memory budget");
  static_assert(S >= 2, "ring too shallow");
};

template <int BN, bool SPLIT>
__global__ void __launch_bounds__(kThreads16, 1)
conv16_kernel(const __grid_constant__ Plan16 P, const __grid_constant__ Maps16 maps,
              const float* __restrict__ in_sc, const float* __restrict__ w_sc,
              const float* __restrict__ bias, double* __restrict__ stats) {
  using C = Cfg16<BN>;
  const epb_phase_grid& G = P.grid;
  constexpr int BOXES = C::S * C::STAGE;          // staging boxes follow the slots (1024-aligned)
  constexpr int CTRL = BOXES + C::BOX_BYTES;
  extern __shared__ uint8_t smem_raw[];
  tc::Ring<C::S, C::STAGE> ring(smem_raw, 0, CTRL, CTRL + 64);     // full[8], empty[8]
  float* sstat = reinterpret_cast<float*>(ring.sm + CTRL + 256);   // [8 warps][2][BN]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int KB = P.T * P.CB;
  const int total_tiles = G.tiles * P.n_tiles;
  const int items = SPLIT ? total_tiles * P.splits : total_tiles;
  // work item -> (tile, split); split s runs k-blocks [kb_lo(s), kb_lo(s + 1))
  auto tile_of = [&](int item) { return SPLIT ? item % total_tiles : item; };
  auto kb_lo = [&](int s) { return SPLIT ? (int)((int64_t)s * KB / P.splits) : (s ? KB : 0); };
  auto nt_of = [&](int tile) { return P.m_fastest ? tile / G.tiles : tile % P.n_tiles; };
  auto mt_of = [&](int tile) { return P.m_fastest ? tile % G.tiles : tile / P.n_tiles; };

  if (threadIdx.x == 0) ring.init(1, kConsumers / 32);   // producer's arrive.expect_tx; consumer warps
  __syncthreads();

  if (warp < 4) {
    // =================================================== TMA producer
    if (warp == 0 && lane == 0) {
      for (int v = 0; v < 4; ++v) tc::tma_prefetch_desc(&maps.a[v]);
      tc::tma_prefetch_desc(&maps.w);
      tc::tma_prefetch_desc(&maps.out);
      for (int item = blockIdx.x; item < items; item += gridDim.x) {
        const int tile = tile_of(item), s = SPLIT ? item / total_tiles : 0;
        const int nt = nt_of(tile);
        int w0, h0, n0;
        G.tile_origin(mt_of(tile), w0, h0, n0);
        const int kb0 = kb_lo(s), kb1 = kb_lo(s + 1);
        int t = kb0 / P.CB, cb = kb0 % P.CB;
        for (int kb = kb0; kb < kb1; ++kb) {
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
  const int rb = wgc * 64 + (warp & 3) * 16;   // this warp's 16 tile rows rb .. rb + 15
  const int ra = rb + (lane >> 2);             // fragment rows ra, ra + 8
  // staging box: row i at 128 * i, its 16-byte chunk c at chunk c ^ (i % 8) (SWIZZLE_128B);
  // this lane's float2 of fragment column group jj (columns 8 jj + lc, + 1 of the 32) in row
  // lane / 4 (+ 8) lies at box + 128 * (lane / 4) (+ 1024) + chunk(jj)
  uint8_t* box = ring.sm + BOXES + (ct >> 5) * kBoxBytes;
  const uint32_t box_addr = tc::smem_u32(box);
  auto chunk = [&](int jj) { return ((2 * jj + ((lane & 3) >> 1)) ^ (lane >> 2)) * 16 + (lane & 1) * 8; };
  const float alpha = in_sc[1] * w_sc[1];
  const int twh = G.tw * G.th;
  if (stats) {
    for (int c = ct; c < (kConsumers / 32) * 2 * BN; c += kConsumers) sstat[c] = 0.f;
    tc::named_sync(1, kConsumers);
  }

  float acc[BN / 2];
  int nt_prev = -1;
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int tile = tile_of(item), s = SPLIT ? item / total_tiles : 0;
    const int nt = nt_of(tile);
    // statistics: one flush per run of tiles of the same N tile
    if (stats && nt_prev >= 0 && nt != nt_prev)
      tc::stats_flush<BN, kConsumers / 32>(sstat, ct, nt_prev, P.Cout, stats);
    nt_prev = nt;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int kb = kb_lo(s), kb1 = kb_lo(s + 1); kb < kb1; ++kb)
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

    // ---- epilogue: rows ra (h = 0) and ra + 8 (h = 1) of the fragment
    int w0, h0, n0;
    G.tile_origin(mt_of(tile), w0, h0, n0);
    bool srow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = ra + 8 * h;
      const int w = w0 + r % G.tw, hh = h0 + (r / G.tw) % G.th, n = n0 + r / twh;
      srow[h] = w < G.Wp && hh < G.Hp && n < G.N;
    }
    // the warp's rows are the (bw, bh, bn) sub-box of the tile box at (bx, by, bz), bw * bh *
    // bn = 16 (tile extents are powers of two); a band that starts past the view is all past it
    const int bx = w0 + rb % G.tw, by = h0 + (rb / G.tw) % G.th, bz = n0 + rb / twh;
    const bool band = SPLIT || (bx < P.Wv && by < P.Hv && bz < G.N);
#pragma unroll
    for (int q = 0; q < BN / 32; ++q) {
      // the previous store has finished reading the box
      if (lane == 0) tc::tma_store_wait_read<0>();
      __syncwarp();
#pragma unroll
      float v[4][2][2];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int col = nt * BN + 32 * q + 8 * jj + lc;
        float2 b = make_float2(0.f, 0.f);
        if (bias && col < P.Cout) b = *reinterpret_cast<const float2*>(bias + col);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          v[jj][h][0] = acc[16 * q + 4 * jj + 2 * h] * alpha + b.x;
          v[jj][h][1] = acc[16 * q + 4 * jj + 2 * h + 1] * alpha + b.y;
          *reinterpret_cast<float2*>(box + 128 * ((lane >> 2) + 8 * h) + chunk(jj)) =
              make_float2(v[jj][h][0], v[jj][h][1]);
        }
      }
      tc::fence_proxy_async();
      __syncwarp();
      const int c0 = nt * BN + 32 * q;
      if (lane == 0 && band && c0 < P.Cout) {
        // With `accumulate` the add of the old value happens in the L2: one fp32 add, round to
        // nearest even, as old + new in registers.  A subnormal old value is kept, not flushed
        // (tests/test_gpu_conv16_store.py checks both against numpy's fp32 sum).
        if constexpr (SPLIT) tc::tma_store_4d(&maps.out, box_addr, c0, 0, (mt_of(tile) * BM + rb) / 16, s);
        else if (P.accumulate) tc::tma_reduce_add_4d(&maps.out, box_addr, c0, bx, by, bz);
        else tc::tma_store_4d(&maps.out, box_addr, c0, bx, by, bz);
        tc::tma_store_commit();
      }
      // the statistics (same columns, same order) while the store reads the box
      if (stats) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) tc::stats_add<BN>(wstat, 32 * q + 8 * jj + lc, v[jj], srow);
      }
    }
  }
  if (stats && nt_prev >= 0) tc::stats_flush<BN, kConsumers / 32>(sstat, ct, nt_prev, P.Cout, stats);
  if (lane == 0) tc::tma_store_wait<0>();   // the output is written before the CTA retires
}

// Split-K second pass: out = bias + sum over s = 0..S-1 (in that order) of the workspace
// partials, for the pixels of the phase grid that lie in the output view, and the per-channel
// sum / sum of squares of every pixel of the phase grid (the rows the fused epilogue counts)
// added to `stats`.  Threads: 32 column quads x 8 rows; the rows of a column block are summed
// in double per thread, then over the 8 row lanes in a fixed order, one atomic per channel.
struct Reduce16 {
  epb_phase_grid grid;
  int Cout, Wv, Hv, splits;
  int64_t sw, sh, sn;            // element strides of w, h, n in the output phase view
};

__global__ void __launch_bounds__(256)
conv16_splitk_reduce(const __grid_constant__ Reduce16 R, const float* __restrict__ ws,
                     const float* __restrict__ bias, float* __restrict__ out,
                     double* __restrict__ stats) {
  __shared__ double red[2][8][128];
  const epb_phase_grid& G = R.grid;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c = (blockIdx.x * 32 + tx) * 4;
  const bool cok = c < R.Cout;
  const int64_t M = (int64_t)G.N * G.Hp * G.Wp;
  const int64_t split_stride = (int64_t)G.tiles * BM * R.Cout;
  float b[4] = {0.f, 0.f, 0.f, 0.f};
  if (bias && cok)
    for (int e = 0; e < 4; ++e) b[e] = bias[c + e];
  double s1[4] = {0.0, 0.0, 0.0, 0.0}, s2[4] = {0.0, 0.0, 0.0, 0.0};
  if (cok) {
    for (int64_t m = (int64_t)blockIdx.y * 8 + ty; m < M; m += (int64_t)gridDim.y * 8) {
      const int w = (int)(m % G.Wp);
      const int64_t q = m / G.Wp;
      const int h = (int)(q % G.Hp), n = (int)(q / G.Hp);
      // tile and tile row of pixel (w, h, n): the inverse of tile_origin and the epilogue's rows
      const int mt = w / G.tw + G.tiles_w * (h / G.th + G.tiles_h * (n / G.tn));
      const int r = w % G.tw + G.tw * (h % G.th + G.th * (n % G.tn));
      const float* src = ws + ((int64_t)mt * BM + r) * R.Cout + c;
      float4 v = *reinterpret_cast<const float4*>(src);
      for (int s = 1; s < R.splits; ++s) {
        const float4 u = *reinterpret_cast<const float4*>(src + s * split_stride);
        v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w;
      }
      v.x += b[0]; v.y += b[1]; v.z += b[2]; v.w += b[3];
      if (w < R.Wv && h < R.Hv)
        *reinterpret_cast<float4*>(out + n * R.sn + h * R.sh + w * R.sw + c) = v;
      const float a[4] = {v.x, v.y, v.z, v.w};
      for (int e = 0; e < 4; ++e) {
        s1[e] += a[e];
        s2[e] += (double)a[e] * a[e];
      }
    }
  }
  if (!stats) return;
  for (int e = 0; e < 4; ++e) {
    red[0][ty][tx * 4 + e] = s1[e];
    red[1][ty][tx * 4 + e] = s2[e];
  }
  __syncthreads();
  if (ty == 0 && cok)
    for (int e = 0; e < 4; ++e) {
      double t1 = 0.0, t2 = 0.0;
      for (int y = 0; y < 8; ++y) {
        t1 += red[0][y][tx * 4 + e];
        t2 += red[1][y][tx * 4 + e];
      }
      atomicAdd(stats + c + e, t1);
      atomicAdd(stats + R.Cout + c + e, t2);
    }
}

// N tile: the 128-column accumulator of a consumer warpgroup (64 fp32 registers per thread),
// 64 columns for narrow layers
inline int conv16_bn(int Cout) { return Cout <= 64 ? 64 : 128; }

// Shortest K range of a split (k-blocks of 64): a work item also pays the pipeline fill, the
// epilogue and the partial's round trip through the workspace.  Two or three splits save at most
// two thirds of the K loop, which pays for the partials and the reduce only when every split is
// still kSplitLongKB k-blocks long (H100 per-layer table, tools/bench_infer.py, DESIGN.md 5).
constexpr int kSplitMinKB = 4;
constexpr int kSplitLongKB = 16;

// One conv16 call: splits == 1 is the fused kernel writing `out`; splits > 1 the SPLIT kernel
// into `ws` (checked by the caller) followed by conv16_splitk_reduce.
int conv16_run(const epb_conv_geom* g, const epb_half* in, const float* in_sc, const epb_half* w,
               const float* w_sc, const float* bias, float* out, double* stats, int splits,
               float* ws, epb_stream_t stream) {
  int rc = epb_conv_geom_check(g);
  if (rc) return rc;
  EPB_CHECK_ARG(in && in_sc && w && w_sc && out);
  EPB_CHECK_ARG(g->Cin % 64 == 0 && g->Cout % 4 == 0 && g->Cout >= 4);
  EPB_CHECK_ARG(g->is == 1 || g->is == 2);
  EPB_CHECK_ARG(!(stats && g->accumulate));
  EPB_CHECK_ARG((reinterpret_cast<uintptr_t>(in) & 127) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0);
  EPB_CHECK_ARG((reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(bias) & 7) == 0);
  Plan16 P;
  Maps16 maps;
  memset(&maps, 0, sizeof(maps));
  bool dense;
  rc = epb_plan_phase_grid(g, in, BM, P.grid, maps.a, dense);
  if (rc) return rc;
  // a dense layer's output is the same [M][Cout] matrix as its phase grid
  const int64_t Ho = dense ? 1 : g->Ho, Wo = dense ? P.grid.Wp : g->Wo, os = dense ? 1 : g->os;
  const int64_t ph = dense ? 0 : g->ph, pw = dense ? 0 : g->pw;
  P.Cout = g->Cout;
  P.Wv = dense ? P.grid.Wp : (g->Wo - g->pw + g->os - 1) / g->os;
  P.Hv = dense ? 1 : (g->Ho - g->ph + g->os - 1) / g->os;
  P.T = g->T; P.CB = g->Cin / 64; P.accumulate = g->accumulate;
  P.splits = splits;
  float* const view = out + (ph * Wo + pw) * g->Cout;
  if (splits == 1) {
    // (Cout, Wv, Hv, N) view of output phase (ph, pw); Cout % 4 == 0 keeps base and strides
    // 16-byte aligned.  Box: 32 columns x the 16 tile rows of one consumer warp.
    const int bw = P.grid.tw < 16 ? P.grid.tw : 16;
    const int bh = P.grid.th < 16 / bw ? P.grid.th : 16 / bw;
    const int64_t C4 = (int64_t)g->Cout * 4;
    const cuuint64_t dims[4] = {(cuuint64_t)g->Cout, (cuuint64_t)P.Wv, (cuuint64_t)P.Hv,
                                (cuuint64_t)P.grid.N};
    const cuuint64_t strides[3] = {(cuuint64_t)(os * C4), (cuuint64_t)(os * Wo * C4),
                                   (cuuint64_t)(Ho * Wo * C4)};
    const cuuint32_t box[4] = {32, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)(16 / (bw * bh))};
    rc = epb_encode_map(&maps.out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, view, dims, strides, box,
                        CU_TENSOR_MAP_L2_PROMOTION_NONE, "output");
    if (rc) return rc;
  } else {
    // dense workspace [S][tiles * 128][Cout] as (Cout, 16, tiles * 8, S): one warp's 16 rows per box
    const int64_t C4 = (int64_t)g->Cout * 4;
    const cuuint64_t dims[4] = {(cuuint64_t)g->Cout, 16, (cuuint64_t)P.grid.tiles * (BM / 16),
                                (cuuint64_t)splits};
    const cuuint64_t strides[3] = {(cuuint64_t)C4, (cuuint64_t)(16 * C4),
                                   (cuuint64_t)((int64_t)P.grid.tiles * BM * C4)};
    const cuuint32_t box[4] = {32, 16, 1, 1};
    rc = epb_encode_map(&maps.out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, ws, dims, strides, box,
                        CU_TENSOR_MAP_L2_PROMOTION_NONE, "split-K workspace");
    if (rc) return rc;
  }
  for (int t = 0; t < g->T; ++t) P.koff[t] = g->wt[t] * g->Cin;
  // tile order: statistics want runs of tiles with the same N tile (one flush per run); without
  // statistics, N-fastest lets the concurrently running tiles of one M tile share its A rows in L2
  P.m_fastest = stats != nullptr;
  const int bn = conv16_bn(g->Cout);
  P.n_tiles = (g->Cout + bn - 1) / bn;
  const int64_t K = (int64_t)g->Tw * g->Cin;
  const cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)g->Cout, 2};
  const cuuint64_t strides[2] = {(cuuint64_t)K * 2, (cuuint64_t)K * 2 * g->Cout};
  const cuuint32_t box[3] = {64, (cuuint32_t)bn, 1};
  rc = epb_encode_map(&maps.w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, w, dims, strides, box,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "weights");
  if (rc) return rc;
  const int64_t tiles = (int64_t)P.grid.tiles * P.n_tiles;
  cudaStream_t st = as_stream(stream);
  if (splits == 1) {
    const unsigned grid = (unsigned)(tiles < kNumSMs ? tiles : kNumSMs);
    if (bn == 64)
      return tc::launch<conv16_kernel<64, false>>(grid, kThreads16, Cfg16<64>::SMEM, st, P, maps,
                                                  in_sc, w_sc, bias, stats);
    return tc::launch<conv16_kernel<128, false>>(grid, kThreads16, Cfg16<128>::SMEM, st, P, maps,
                                                 in_sc, w_sc, bias, stats);
  }
  P.m_fastest = 0;
  const int64_t items = tiles * splits;
  const unsigned grid = (unsigned)(items < kNumSMs ? items : kNumSMs);
  const float* no_bias = nullptr;
  double* no_stats = nullptr;
  rc = bn == 64 ? tc::launch<conv16_kernel<64, true>>(grid, kThreads16, Cfg16<64>::SMEM, st, P, maps,
                                                      in_sc, w_sc, no_bias, no_stats)
                : tc::launch<conv16_kernel<128, true>>(grid, kThreads16, Cfg16<128>::SMEM, st, P,
                                                       maps, in_sc, w_sc, no_bias, no_stats);
  if (rc) return rc;
  Reduce16 R;
  R.grid = P.grid;
  R.Cout = g->Cout; R.Wv = P.Wv; R.Hv = P.Hv; R.splits = splits;
  R.sw = os * g->Cout; R.sh = os * Wo * g->Cout; R.sn = Ho * Wo * g->Cout;
  const int64_t M = (int64_t)P.grid.N * P.grid.Hp * P.grid.Wp;
  const unsigned gx = (unsigned)((g->Cout + 127) / 128);
  int64_t gy = (M + 7) / 8, cap = 4 * kNumSMs / gx + 1;
  if (gy > cap) gy = cap;
  conv16_splitk_reduce<<<dim3(gx, (unsigned)gy), dim3(32, 8), 0, st>>>(R, ws, bias, view, stats);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

}  // namespace

extern "C" __attribute__((visibility("default"))) int epb_conv16_fprop(
    const epb_conv_geom* g, const epb_half* in, const float* in_sc, const epb_half* w,
    const float* w_sc, const float* bias, float* out, double* stats, epb_stream_t stream) {
  return conv16_run(g, in, in_sc, w, w_sc, bias, out, stats, 1, nullptr, stream);
}

extern "C" __attribute__((visibility("default"))) int epb_conv16_splits(const epb_conv_geom* g,
                                                                          int* splits,
                                                                          long long* ws_floats) {
  int rc = epb_conv_geom_check(g);
  if (rc) return rc;
  EPB_CHECK_ARG(splits && ws_floats && g->Cin % 64 == 0 && g->Cout >= 4);
  epb_phase_grid G;
  bool dense;
  rc = epb_tile_phase_grid(g, BM, G, dense);
  if (rc) return rc;
  const int bn = conv16_bn(g->Cout);
  const int64_t tiles = (int64_t)G.tiles * ((g->Cout + bn - 1) / bn);
  const int64_t kb = (int64_t)g->T * (g->Cin / 64);
  // as many splits as keep every SM busy with one work item, none when the tiles already fill
  // more than half of the SMs (a second split would start a second wave)
  int64_t s = kNumSMs / tiles;
  if (s > kb / kSplitMinKB) s = kb / kSplitMinKB;
  if (s < 4 && kb < kSplitLongKB * s) s = 1;
  if (s < 1) s = 1;
  *splits = (int)s;
  *ws_floats = s > 1 ? s * G.tiles * BM * g->Cout : 0;
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_conv16_fprop_splitk(
    const epb_conv_geom* g, const epb_half* in, const float* in_sc, const epb_half* w,
    const float* w_sc, const float* bias, float* out, double* stats, int splits, float* ws,
    long long ws_floats, epb_stream_t stream) {
  int rc = epb_conv_geom_check(g);
  if (rc) return rc;
  EPB_CHECK_ARG(!g->accumulate);            // an inference forward: no data-gradient accumulate
  EPB_CHECK_ARG(g->Cin % 64 == 0 && splits >= 1 && splits <= g->T * (g->Cin / 64));
  if (splits > 1) {
    epb_phase_grid G;
    bool dense;
    rc = epb_tile_phase_grid(g, BM, G, dense);
    if (rc) return rc;
    EPB_CHECK_ARG(ws && (reinterpret_cast<uintptr_t>(ws) & 15) == 0);
    EPB_CHECK_ARG(ws_floats >= (long long)splits * G.tiles * BM * g->Cout);
  }
  return conv16_run(g, in, in_sc, w, w_sc, bias, out, stats, splits, ws, stream);
}
