// Split-fp16 ("f16x3") weight-gradient kernel of the tap-list implicit GEMM (include/epb.h,
// epb_conv16_wgrad; cuDNN wgrad behind the autograd of lib/models/pose3d_resnet.py:12-15,
// 55-60,99,116-122,171-178):
//
//   dw[co][wt[t]][ci] += (1 / (s_in * s_dout)) * sum_m in[pix_in(m, t)][ci] * dout[pix_out(m)][co]
//
// GEMM view: D[(t, ci), co] with the reduction over phase-grid pixels m.  Both operands are
// MN-major for the tensor core (channels contiguous in NHWC memory, the reduction index
// strides over pixel rows) and come straight from the fp16 planes by TMA: a tile of 64 pixels
// x 64 channels is one 5-D box load -- 64 rows of 128 bytes, exactly the SWIZZLE_128B MN-major
// atom sequence wgmma reads (8-row atoms 1024 B apart, 64-channel chunks LBO apart).
// The M side is a list of CHUNKS (tap, 64-channel block): 2 chunks per CTA (M = 128, one per
// consumer warpgroup, wgmma m64nBNk16 with transposed operands), each chunk its own
// tap-shifted box, so every tap of a 64-channel layer still fills the M rows; the N side is
// min(Cout, 128) output channels.  The pixel range is split across CTAs; partial tiles go to
// `ws` and are summed in split order by a second kernel (deterministic; no atomics).
#include "split16_common.cuh"

namespace {

constexpr int KT = 64;                 // pixels per stage (4 MMAs of K = 16)
constexpr int kThreadsW16 = 384;       // warpgroup 0: TMA producer; warpgroups 1-2: consumers
constexpr int kChunk = KT * 128;       // bytes of one (64 pixels x 64 channels) box

struct PlanW16 {
  epb_phase_grid grid;           // pixel tiles of the phase grid (the reduction), tap views
  int Cin, Cout, Tw;
  int T, CB, CH;                 // taps, 64-channel blocks per tap, chunks = T * CB
  int groups, n_tiles, splits, tiles_per_split;
  int swap;                      // 1: M side = 64-channel blocks of dout, N side = input channels
  int Nn;                        // channels on the N side (Cout, or Cin when swapped)
  int bdw, bdh;                  // box offset of the N-side operand (the tap, when swapped)
  int wt[EPB_MAX_TAPS];
};

struct MapsW16 {
  CUtensorMap a[4];
  CUtensorMap d;
};

template <int BN>
struct CfgW16 {
  static constexpr int BCH = BN / 64;                    // 64-channel chunks of the N side
  static constexpr int A_PLANE = 2 * kChunk;
  static constexpr int B_PLANE = BCH * kChunk;
  static constexpr int STAGE = 2 * A_PLANE + 2 * B_PLANE;
  static constexpr int S_ = (200 * 1024) / STAGE;
  static constexpr int S = S_ > 6 ? 6 : S_;
  static constexpr int SMEM = S * STAGE + 1024 + 256;
};

template <int BN>
__global__ void __launch_bounds__(kThreadsW16, 1)
wgrad16_kernel(const __grid_constant__ PlanW16 P, const __grid_constant__ MapsW16 maps,
               const float* __restrict__ in_sc, const float* __restrict__ dout_sc,
               float* __restrict__ dw, float* __restrict__ ws) {
  using C = CfgW16<BN>;
  constexpr int CTRL = C::S * C::STAGE;
  const epb_phase_grid& G = P.grid;
  extern __shared__ uint8_t smem_raw[];
  tc::Ring<C::S, C::STAGE> ring(smem_raw, 0, CTRL, CTRL + 64);     // full[8], empty[8]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // work item: blockIdx.x = ((split * n_tiles + nt) * groups + grp)
  int wi = (int)blockIdx.x;
  const int grp = wi % P.groups; wi /= P.groups;
  const int nt = wi % P.n_tiles;
  const int split = wi / P.n_tiles;
  const int pt0 = split * P.tiles_per_split;
  const int pt1 = min(G.tiles, pt0 + P.tiles_per_split);
  const int nst = pt1 - pt0;                                   // stages of this CTA (>= 1)

  if (threadIdx.x == 0) ring.init(1, 8);                       // one arrive per consumer warp
  __syncthreads();

  if (warp < 4) {
    // =================================================== TMA producer
    if (warp == 0 && lane == 0) {
      for (int v = 0; v < 4; ++v) tc::tma_prefetch_desc(&maps.a[v]);
      tc::tma_prefetch_desc(&maps.d);
      // this CTA's two chunks (clamped: rows of a chunk past the end are computed, never stored)
      int ct[2], cc[2];
      for (int j = 0; j < 2; ++j) {
        const int c = min(grp * 2 + j, P.CH - 1);
        ct[j] = c / P.CB;
        cc[j] = (c % P.CB) * 64;
      }
      for (int pt = pt0; pt < pt1; ++pt) {
        int w0, h0, n0;
        G.tile_origin(pt, w0, h0, n0);
        tc::mbar_wait(ring.empty(ring.stage), ring.phase ^ 1);
        const uint32_t fb = ring.full(ring.stage);
        tc::mbar_arrive_expect_tx(fb, C::STAGE);
        const uint32_t a_dst = ring.stage_addr(ring.stage);
        const uint32_t b_dst = a_dst + 2 * C::A_PLANE;
#pragma unroll
        for (int pl = 0; pl < 2; ++pl) {
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int t = ct[j];
            tc::tma_load_5d(a_dst + pl * C::A_PLANE + j * kChunk, &maps.a[G.map[t]], fb,
                            cc[j], w0 + G.dwq[t], h0 + G.dhq[t], n0, pl);
          }
#pragma unroll
          for (int jb = 0; jb < C::BCH; ++jb)
            tc::tma_load_5d(b_dst + pl * C::B_PLANE + jb * kChunk, &maps.d, fb,
                            nt * BN + jb * 64, w0 + P.bdw, h0 + P.bdh, n0, pl);
        }
        ring.advance();
      }
    }
    return;
  }

  // =================================================== consumers: warpgroup wgc owns chunk wgc
  const int wgc = (warp >> 2) - 1;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int k = 0; k < nst; ++k)
    ring.consume(acc, [&](uint32_t st) {
      const uint32_t a_hi = st + wgc * kChunk, b_hi = st + 2 * C::A_PLANE;
#pragma unroll
      for (int ks = 0; ks < KT / 16; ++ks)
        tc::mma3_f16<1, 1>(acc, tc::desc_mnmajor16_sw128(a_hi + ks * 2048, kChunk, 1024),
                           tc::desc_mnmajor16_sw128(a_hi + C::A_PLANE + ks * 2048, kChunk, 1024),
                           tc::desc_mnmajor16_sw128(b_hi + ks * 2048, kChunk, 1024),
                           tc::desc_mnmajor16_sw128(b_hi + C::B_PLANE + ks * 2048, kChunk, 1024));
    });
  ring.drain(acc);

  const int c = grp * 2 + wgc;                                // chunk of this warpgroup's 64 rows
  if (c >= P.CH) return;
  const int64_t K = (int64_t)P.Tw * P.Cin;
  const float alpha = in_sc[1] * dout_sc[1];
  float* dst = P.splits > 1 ? ws + (int64_t)split * P.Cout * K : dw;
  // normal : row = input channel ci of tap t,  column = output channel co
  // swapped: row = output channel co,          column = input channel ci (T == 1)
  const int t = P.swap ? 0 : c / P.CB;
  const int64_t col_stride = P.swap ? 1 : K;
  const int lc = (lane & 3) * 2;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int rowc = (warp & 3) * 16 + (lane >> 2) + 8 * h;  // this thread's row inside the chunk
    const int64_t row_off = P.swap ? (int64_t)(c * 64 + rowc) * K + (int64_t)P.wt[0] * P.Cin
                                   : (int64_t)P.wt[t] * P.Cin + (c % P.CB) * 64 + rowc;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = nt * BN + 8 * j + lc + e;
        if (col < P.Nn) {
          float* o = dst + row_off + (int64_t)col * col_stride;
          const float v = acc[4 * j + 2 * h + e];
          if (P.splits > 1) *o = v;
          else *o += alpha * v;
        }
      }
    }
  }
}

// dw[co][wt[t]][ci] += alpha * sum_s ws[s][co][wt[t]][ci]   (fixed order)
__global__ void __launch_bounds__(256)
wgrad16_reduce_kernel(const __grid_constant__ PlanW16 P, const float* __restrict__ in_sc,
                      const float* __restrict__ dout_sc, const float* __restrict__ ws,
                      float* __restrict__ dw) {
  const int C4 = P.Cin / 4;
  const int64_t K = (int64_t)P.Tw * P.Cin;
  const int64_t total = (int64_t)P.Cout * P.T * C4;
  const int64_t plane4 = (int64_t)P.Cout * K / 4;
  const float alpha = in_sc[1] * dout_sc[1];
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * 256) {
    const int c4 = (int)(i % C4);
    const int t = (int)((i / C4) % P.T);
    const int64_t co = i / ((int64_t)C4 * P.T);
    const int64_t o4 = (co * K + (int64_t)P.wt[t] * P.Cin) / 4 + c4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < P.splits; ++s) {
      const float4 v = reinterpret_cast<const float4*>(ws)[s * plane4 + o4];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    float4* o = reinterpret_cast<float4*>(dw) + o4;
    float4 d = *o;
    d.x += alpha * acc.x; d.y += alpha * acc.y; d.z += alpha * acc.z; d.w += alpha * acc.w;
    *o = d;
  }
}

template <int BN>
int launch_w16(const PlanW16& P, const MapsW16& maps, const float* in_sc, const float* dout_sc,
               float* dw, float* ws, cudaStream_t st) {
  const int64_t ctas = (int64_t)P.groups * P.n_tiles * P.splits;
  EPB_CHECK_ARG(ctas < (1LL << 31));
  int rc = tc::launch<wgrad16_kernel<BN>>((unsigned)ctas, kThreadsW16, CfgW16<BN>::SMEM, st, P,
                                          maps, in_sc, dout_sc, dw, ws);
  if (rc || P.splits == 1) return rc;
  const int64_t total = (int64_t)P.Cout * P.T * (P.Cin / 4);
  int64_t blocks = (total + 255) / 256;
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  wgrad16_reduce_kernel<<<(unsigned)blocks, 256, 0, st>>>(P, in_sc, dout_sc, ws, dw);
  EPB_LAUNCH_CHECK();
  return EPB_OK;
}

}  // namespace

extern "C" __attribute__((visibility("default"))) int epb_conv16_wgrad(
    const epb_conv_geom* g, const epb_half* in, const float* in_sc, const epb_half* dout,
    const float* dout_sc, float* dw, float* ws, long long ws_floats, epb_stream_t stream) {
  int rc = epb_conv_geom_check(g);
  if (rc) return rc;
  EPB_CHECK_ARG(in && in_sc && dout && dout_sc && dw);
  EPB_CHECK_ARG(g->Cin % 64 == 0 && g->Cout % 64 == 0);
  EPB_CHECK_ARG((g->is == 1 || g->is == 2) && (g->os == 1 || g->os == 2));
  PlanW16 P;
  MapsW16 maps;
  memset(&maps, 0, sizeof(maps));
  P.Cin = g->Cin; P.Cout = g->Cout; P.Tw = g->Tw; P.T = g->T; P.CB = g->Cin / 64;
  P.CH = P.T * P.CB;
  // A 1x1 layer with 64 input channels leaves one of the 2 M-side chunks of a CTA empty: put
  // the output channels on the M side instead (D^T; same products, same sums)
  P.swap = (g->T == 1 && P.CH < 2 && g->Cout / 64 > P.CH) ? 1 : 0;
  P.bdw = P.bdh = 0;
  for (int t = 0; t < g->T; ++t) P.wt[t] = g->wt[t];
  bool dense;
  CUtensorMap in_maps[4];
  memset(in_maps, 0, sizeof(in_maps));
  rc = epb_plan_phase_grid(g, in, KT, P.grid, in_maps, dense);
  if (rc) return rc;
  // dout on the phase grid: a dense layer's output is the same [M][Cout] matrix
  CUtensorMap d_map;
  rc = epb_make_act_map(&d_map, dout, P.grid.N, dense ? 1 : g->Ho, dense ? P.grid.Wp : g->Wo,
                        g->Cout, g->os, g->ph, g->pw, P.grid.tw, P.grid.th, P.grid.tn);
  if (rc) return rc;
  if (!P.swap) {
    for (int v = 0; v < 4; ++v) maps.a[v] = in_maps[v];
    maps.d = d_map;
    P.Nn = g->Cout;
  } else {
    // M side: the CH' = Cout / 64 blocks of dout (no tap shift); N side: the input, shifted by the tap
    for (int v = 0; v < 4; ++v) maps.a[v] = d_map;
    maps.d = in_maps[P.grid.map[0]];
    P.bdw = P.grid.dwq[0]; P.bdh = P.grid.dhq[0];
    P.grid.map[0] = 0; P.grid.dwq[0] = 0; P.grid.dhq[0] = 0;
    P.CB = g->Cout / 64;
    P.CH = P.CB;
    P.Nn = g->Cin;
  }
  const int bn = P.Nn <= 64 ? 64 : 128;
  P.n_tiles = (P.Nn + bn - 1) / bn;
  P.groups = (P.CH + 1) / 2;
  // pixel-range splits: fill two waves of CTAs (which also keeps the fp32 accumulation runs
  // short), keep >= 8 stages per CTA, and stay inside the scratch the caller gave
  const int64_t basec = (int64_t)P.groups * P.n_tiles;
  int64_t splits = 2 * kNumSMs / basec;
  if (splits > P.grid.tiles / 8) splits = P.grid.tiles / 8;
  const int64_t per_split = (int64_t)g->Cout * g->Tw * g->Cin;
  if (!ws || splits * per_split > ws_floats) splits = ws ? ws_floats / per_split : 1;
  if (splits < 1) splits = 1;
  P.tiles_per_split = (int)((P.grid.tiles + splits - 1) / splits);
  P.splits = (P.grid.tiles + P.tiles_per_split - 1) / P.tiles_per_split;
  cudaStream_t st = as_stream(stream);
  if (bn == 64) return launch_w16<64>(P, maps, in_sc, dout_sc, dw, ws, st);
  return launch_w16<128>(P, maps, in_sc, dout_sc, dw, ws, st);
}
