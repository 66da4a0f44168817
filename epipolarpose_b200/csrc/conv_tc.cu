// wgmma tensor-core path of the tap-list implicit GEMM (include/epb.h).
//
//   out[m, co] = sum_k A[m, k] * W[co, k],  m = (n, i, j) phase-grid pixel,
//   k = (tap, ci);  A gathered from the NHWC input with the producing layer's
//   BatchNorm+ReLU applied on the fly.
//
// One persistent CTA per SM on the pipeline of tc_common.cuh:
//   warps 0-7  consumers: wgmma m64nBNk8 tf32 per k-step; the epilogue adds the bias,
//              stores or accumulates, and flushes the BatchNorm statistics every tile;
//   warps 8-15 producers: gather 128 pixel rows x 32 channels (128-byte rows), fused
//              BN+ReLU, split into TF32 hi (+ lo for the 3xTF32 mode) and store into the
//              SWIZZLE_128B K-major smem layout wgmma reads; the k-blocks of all tiles of
//              the CTA form ONE stream that the two producer groups take round-robin
//              (warp-private row tables, no CTA barrier).  The first lane of each group
//              also issues the TMA loads of the packed weight tile (hi / lo planes) of the
//              slot it fills.
//
// precision 1: TF32 single pass.  precision 3: 3xTF32 error-compensated
// (a_hi*b_hi + a_lo*b_hi + a_hi*b_lo, FP32 accumulate): fp32-grade results on
// the tensor pipe, which is what the 1e-3 end-to-end parity bar needs.
#include <cstdlib>
#include "split16_common.cuh"

namespace {

constexpr int BM = 128;          // pixel rows per tile (two wgmma M = 64 halves)
constexpr int BKE = 32;          // tf32 elements per k-block (128 bytes)
constexpr int kConsumerWarps = 8;
constexpr int kProducerWarps = 8;       // G groups of W = 4 warps take k-blocks round-robin
constexpr int kThreads = 32 * (kConsumerWarps + kProducerWarps);       // 512
constexpr int kSmemBudget = 200 * 1024;
constexpr int kRowTab = kProducerWarps * 32;   // one private table of <= 32 rows per producer warp

template <int BN, int NS>
struct Cfg {
  static constexpr int PL = (NS == 3) ? 2 : 1;                 // operand planes (hi, lo)
  static constexpr int A_BYTES = BM * 128 * PL;
  static constexpr int B_BYTES = BN * 128 * PL;
  static constexpr int STAGE = A_BYTES + B_BYTES;
  static constexpr int S_ = kSmemBudget / STAGE;
  static constexpr int S = S_ > 8 ? 8 : S_;
  // Producer groups.  A group waits on a slot's empty barrier by PARITY, which is only
  // sound while it is less than two phases ahead of the barrier: G <= S.  2 groups of 4
  // warps with a register double buffer: the loads of four k-blocks are in flight and every
  // SM sub-partition has 2 producer warps.
  static constexpr int G = kProducerWarps / 4;
  static constexpr int D = 2;                                  // register buffers per group
  static constexpr int W = kProducerWarps / G;                 // warps per group
  static constexpr int NQ = 32 / W;                            // float4 per thread per k-block
  static constexpr int STAT_BYTES = kConsumerWarps * 2 * BN * 4;   // per warp [sum | sum of squares][BN]
  static constexpr int SMEM = S * STAGE + 1024 /*align*/ + 1024 /*barriers*/ + kRowTab * 12 /*rowinfo*/ +
                              STAT_BYTES;
  static_assert(SMEM <= 227 * 1024, "shared memory budget");
  static_assert(G <= S, "producer groups must stay within two ring phases");
};

struct RowInfo {
  int off0[kRowTab];                  // ((n*Hi + i*is)*Wi + j*is)*Cin : element offset of the un-shifted pixel
  unsigned long long vmask[kRowTab];  // bit t set <=> tap t reads inside the image (0 for rows past M)
};

template <int BN, int NS>
__global__ void __launch_bounds__(kThreads, 1)
conv_fprop_tc_kernel(const __grid_constant__ epb_conv_geom g,
                     const __grid_constant__ CUtensorMap tmap_w, const float* __restrict__ in,
                     const float* __restrict__ in_scale, const float* __restrict__ in_shift,
                     const float* __restrict__ bias, float* __restrict__ out,
                     double* __restrict__ stats, int npad, int m_tiles, int n_tiles) {
  using C = Cfg<BN, NS>;
  const int tile0 = (int)blockIdx.x;
  const int tstep = (int)gridDim.x;
  auto m_tile_of = [&](int tile) { return tile / n_tiles; };
  constexpr int CTRL = C::S * C::STAGE;
  extern __shared__ uint8_t smem_raw[];
  tc::Ring<C::S, C::STAGE> ring(smem_raw, 0, CTRL, CTRL + 64);     // full[8], empty[8]
  uint8_t* ctrl = ring.sm + CTRL;
  RowInfo* rows = reinterpret_cast<RowInfo*>(ctrl + 1024);
  float* sstat = reinterpret_cast<float*>(ctrl + 1024 + sizeof(RowInfo));   // [8 warps][2][BN]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t M = (int64_t)g.N * g.Hp * g.Wp;
  const int CB = g.Cin / BKE;              // channel blocks per tap
  const int KB = g.T * CB;                 // k-blocks per tile
  const int total_tiles = m_tiles * n_tiles;

  if (threadIdx.x == 0) ring.init(C::W + 1, kConsumerWarps);   // the group's A warps + its weight TMA
  if (stats)
    for (int c = threadIdx.x; c < kConsumerWarps * 2 * BN; c += kThreads) sstat[c] = 0.f;
  __syncthreads();

  if (warp >= kConsumerWarps) {
    // =================================================== producers (256 threads), flat stream
    // The k-blocks of ALL tiles of this CTA form one stream n = 0, 1, 2, ...; group g takes
    // n = g, g + G, ... (ring slot n % S).  A warp only ever touches its own RPW pixel rows,
    // so the row geometry lives in a WARP-PRIVATE table that the warp rebuilds when its issue
    // cursor enters a new tile: no CTA-wide barrier between tiles, and the loads of the next
    // tile's first k-blocks are in flight while the current tile is still being converted.
    //
    // L2 prefetch policy of the A stream:
    //  * dense 1x1 layers (phase-grid pixel == input pixel): ROLLING prefetch kPfDist k-blocks
    //    ahead of the loads, crossing into this CTA's next tiles -- bounded footprint;
    //  * otherwise the whole NEXT tile while the current one is processed, but only for rows
    //    of <= 1 KB: with wider rows one CTA per SM x 2 tiles overflow L2.
    // Single-use loads of 1x1 layers with one N tile are marked evict-first.
    constexpr int kPfDist = 6;
    constexpr int G = C::G, D = C::D, NQ = C::NQ, RPW = BM / C::W;
    const int pwarp = warp - kConsumerWarps;
    const bool roll = g.T == 1 && g.is == 1 && g.Hp == g.Hi && g.Wp == g.Wi;
    const bool pf_tile = !roll && g.Cin <= 256;
    const int dmt = (n_tiles == 1 && tile0 + tstep < total_tiles)
                        ? m_tile_of(tile0 + tstep) - m_tile_of(tile0) : 0;   // M-tile stride of this CTA
    const bool once = g.T == 1 && n_tiles == 1;
    const float lb = g.in_relu ? 0.f : -INFINITY;
    uint64_t pol_first;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_first));
    const int c4 = lane & 7;                   // 16-byte chunk within the 128-byte row
    const int rsub = lane >> 3;                // 0..3
    const int grp = pwarp / C::W, wg = pwarp % C::W;
    int* w_off = rows->off0 + pwarp * 32;                  // this warp's rows wg*RPW .. +RPW-1
    unsigned long long* w_vm = rows->vmask + pwarp * 32;
    const int my_tiles = tile0 < total_tiles ? (total_tiles - tile0 + tstep - 1) / tstep : 0;
    const long long total_kb = (long long)my_tiles * KB;
    const int mine = (int)((total_kb - grp + G - 1) / G);  // k-blocks of this group (>= 0)
    int i_tile = tile0, i_kb = grp, it = 0, icb = 0, i_mt = 0;
    int p_kb = grp, pcb = 0, p_tile = tile0;
    bool i_new = true;                         // the issue cursor stands on a tile whose rows are not tabled yet
    while (i_kb >= KB) { i_kb -= KB; i_tile += tstep; }
    it = i_kb / CB; icb = i_kb - it * CB;
    while (p_kb >= KB) { p_kb -= KB; p_tile += tstep; }
    pcb = p_kb % CB;
    if (grp == 0 && wg == 0 && lane == 0) tc::tma_prefetch_desc(&tmap_w);
    int st = grp;                              // G <= S: ring slot / phase of this group's next k-block
    uint32_t ph = 0;
    auto table_rows = [&]() {
      i_mt = m_tile_of(i_tile);
      __syncwarp();
      if (lane < RPW) {
        const int64_t m = (int64_t)i_mt * BM + wg * RPW + lane;
        unsigned long long vm = 0;
        int off = 0;
        if (m < M) {
          const unsigned um = (unsigned)m;
          const unsigned j = um % (unsigned)g.Wp, qq = um / (unsigned)g.Wp;
          const unsigned i = qq % (unsigned)g.Hp, n = qq / (unsigned)g.Hp;
          const int ih0 = (int)i * g.is, iw0 = (int)j * g.is;
          off = (((int)n * g.Hi + ih0) * g.Wi + iw0) * g.Cin;
          for (int t = 0; t < g.T; ++t) {
            const int ih = ih0 + g.dh[t], iw = iw0 + g.dw[t];
            if (ih >= 0 && ih < g.Hi && iw >= 0 && iw < g.Wi) vm |= 1ull << t;
          }
        }
        w_off[lane] = off;
        w_vm[lane] = vm;
        const int ntile = i_tile + tstep;
        if (pf_tile && grp == 0 && ntile < total_tiles && m_tile_of(ntile) != i_mt) {
          const int64_t mn = (int64_t)m_tile_of(ntile) * BM + wg * RPW + lane;
          if (mn < M) {
            const unsigned um = (unsigned)mn;
            const unsigned j = um % (unsigned)g.Wp, qq = um / (unsigned)g.Wp;
            const unsigned i = qq % (unsigned)g.Hp, n = qq / (unsigned)g.Hp;
            int ih = (int)i * g.is, iw = (int)j * g.is;
            ih = ih < g.Hi ? ih : g.Hi - 1;
            iw = iw < g.Wi ? iw : g.Wi - 1;
            const float* rowp = in + (((int64_t)n * g.Hi + ih) * g.Wi + iw) * g.Cin;
            for (int c = 0; c < g.Cin; c += 32)
              asm volatile("prefetch.global.L2 [%0];" ::"l"(rowp + c));
          }
        }
      }
      __syncwarp();
      i_new = false;
    };
    float4 buf[D][NQ];
    unsigned okm[D];
    auto issue = [&](float4 (&dst)[NQ], unsigned& mask) {
      if (i_new) table_rows();
      const int delta = (g.dh[it] * g.Wi + g.dw[it]) * g.Cin + icb * BKE + c4 * 4;
      const int tap = it;
      if (roll) {
        int pb = icb + kPfDist, ta = 0;          // channel block / tiles ahead of this CTA
        while (pb >= CB) { pb -= CB; ++ta; }
        if ((ta == 0 || dmt > 0) && lane < RPW) {
          if ((int64_t)(i_mt + ta * dmt) * BM + wg * RPW + lane < M)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(
                in + ((int64_t)w_off[lane] + (int64_t)ta * dmt * BM * g.Cin + pb * BKE)));
        }
      }
      mask = 0;
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int lr = q * 4 + rsub;
        dst[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        if ((w_vm[lr] >> tap) & 1ull) {
          const float* ap = in + ((int64_t)w_off[lr] + delta);
          if (once) {
            asm volatile("ld.global.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
                         : "=f"(dst[q].x), "=f"(dst[q].y), "=f"(dst[q].z), "=f"(dst[q].w)
                         : "l"(ap), "l"(pol_first));
          } else {
            dst[q] = *reinterpret_cast<const float4*>(ap);
          }
          mask |= 1u << q;
        }
      }
      i_kb += G;
      icb += G;
      while (icb >= CB) { icb -= CB; ++it; }
      if (i_kb >= KB) {
        do { i_kb -= KB; i_tile += tstep; } while (i_kb >= KB);
        it = i_kb / CB; icb = i_kb - it * CB;
        i_new = true;
      }
    };
    auto process = [&](const float4 (&v)[NQ], unsigned mask) {
      const int ch = pcb * BKE + c4 * 4;
      const int kx = g.wt[p_kb / CB] * g.Cin + pcb * BKE;     // weight column of this k-block
      const int nt = p_tile % n_tiles;
      p_kb += G;
      pcb += G;
      while (pcb >= CB) pcb -= CB;
      if (p_kb >= KB) {
        do { p_kb -= KB; p_tile += tstep; } while (p_kb >= KB);
        pcb = p_kb % CB;
      }
      float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
      if (in_scale) {
        sc = *reinterpret_cast<const float4*>(in_scale + ch);
        sh = *reinterpret_cast<const float4*>(in_shift + ch);
      }
      tc::mbar_wait(ring.empty(st), ph ^ 1);
      if (wg == 0 && lane == 0) {
        const uint32_t b_dst = ring.stage_addr(st) + C::A_BYTES;
        tc::mbar_arrive_expect_tx(ring.full(st), C::B_BYTES);
#pragma unroll
        for (int pl = 0; pl < C::PL; ++pl)
          tc::tma_load_2d(b_dst + pl * BN * 128, &tmap_w, ring.full(st), kx, pl * npad + nt * BN);
      }
      uint8_t* a_hi = ring.sm + st * C::STAGE;
      float4 xv[NQ];
#pragma unroll
      for (int q = 0; q < NQ; ++q) xv[q] = v[q];
      if (in_scale) {
#pragma unroll
        for (int q = 0; q < NQ; ++q) xv[q] = tc::bn_act4(xv[q], sc, sh, lb);
        if (mask != (1u << NQ) - 1u) {
#pragma unroll
          for (int q = 0; q < NQ; ++q)
            if (!((mask >> q) & 1u)) xv[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int r = wg * RPW + q * 4 + rsub;
        const float4 x = xv[q];
        const uint32_t off = (uint32_t)r * 128u + (uint32_t)((c4 ^ (r & 7)) << 4);
        float4 hi = make_float4(tc::to_tf32(x.x), tc::to_tf32(x.y), tc::to_tf32(x.z),
                                tc::to_tf32(x.w));
        *reinterpret_cast<float4*>(a_hi + off) = hi;
        if (NS == 3) {
          float4 lo = make_float4(x.x - hi.x, x.y - hi.y, x.z - hi.z, x.w - hi.w);
          *reinterpret_cast<float4*>(a_hi + BM * 128 + off) = lo;
        }
      }
      tc::fence_proxy_async();
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(ring.full(st));
      st += G;
      ph ^= (uint32_t)((st / C::S) & 1);
      st %= C::S;
    };
    if (mine > 0) issue(buf[0], okm[0]);
    for (int k0 = 0; k0 < mine; k0 += 2) {
#pragma unroll
      for (int d = 0; d < 2; ++d) {
        const int k = k0 + d;
        if (k < mine) {
          if (k + 1 < mine) issue(buf[d ^ 1], okm[d ^ 1]);
          process(buf[d], okm[d]);
        }
      }
    }
  } else {
    // =================================================== consumers (2 warpgroups)
    const int wgc = warp >> 2;                 // rows 64 * wgc .. + 63 of the tile
    const int lc = (lane & 3) * 2;
    const int ra = wgc * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows ra, ra + 8
    float acc[BN / 2];
    for (int tile = tile0; tile < total_tiles; tile += tstep) {
      const int mt = m_tile_of(tile), nt = tile % n_tiles;
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < KB; ++kb)
        ring.consume(acc, [&](uint32_t st) {
          const uint32_t a_hi = st + wgc * 64 * 128, b_hi = st + C::A_BYTES;
#pragma unroll
          for (int kk = 0; kk < BKE / 8; ++kk) {
            const uint64_t ah = tc::desc_kmajor_sw128(a_hi + kk * 32);
            const uint64_t bh = tc::desc_kmajor_sw128(b_hi + kk * 32);
            if (NS == 3)
              tc::mma3_tf32(acc, ah, tc::desc_kmajor_sw128(a_hi + BM * 128 + kk * 32), bh,
                            tc::desc_kmajor_sw128(b_hi + BN * 128 + kk * 32));
            else
              tc::wgmma_tf32(acc, ah, bh, 1);
          }
        });
      ring.drain(acc);

      // ---- epilogue straight from the fragment: rows ra (h = 0) and ra + 8 (h = 1)
      float* orow[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t m = (int64_t)mt * BM + ra + 8 * h;
        orow[h] = nullptr;
        if (m < M) {
          const int j = (int)(m % g.Wp);
          const int i = (int)((m / g.Wp) % g.Hp);
          const int n = (int)(m / ((int64_t)g.Wp * g.Hp));
          orow[h] = out + (((int64_t)n * g.Ho + (i * g.os + g.ph)) * g.Wo + (j * g.os + g.pw)) * g.Cout;
        }
      }
#pragma unroll
      for (int jj = 0; jj < BN / 8; ++jj) {
        const int cl = 8 * jj + lc, col = nt * BN + cl;
        if (nt * BN + 8 * jj >= g.Cout) break;       // N tail (Cout % 32 == 0)
        float2 b = make_float2(0.f, 0.f);
        if (bias) b = *reinterpret_cast<const float2*>(bias + col);
        float v[2][2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          v[h][0] = acc[4 * jj + 2 * h] + b.x;
          v[h][1] = acc[4 * jj + 2 * h + 1] + b.y;
          if (orow[h]) {
            float2* o = reinterpret_cast<float2*>(orow[h] + col);
            float2 x = make_float2(v[h][0], v[h][1]);
            if (g.accumulate) {
              const float2 pv = *o;
              x.x += pv.x; x.y += pv.y;
            }
            *o = x;
          }
        }
        if (stats)
          tc::stats_add<BN>(sstat + warp * 2 * BN, cl, v, {orow[0] != nullptr, orow[1] != nullptr});
      }
      if (stats) tc::stats_flush<BN, kConsumerWarps>(sstat, threadIdx.x, nt, g.Cout, stats);
    }
  }
}

// ---------------------------------------------------------------- weight prep
// packed [Cout][K] fp32 -> planes [PL][npad][K]: TF32 hi (RN) and fp32 residual lo;
// rows >= Cout are zero so N-tail tiles need no predication.
__global__ void prep_weight_tc(const float* __restrict__ w, float* __restrict__ dst, int Cout,
                               int64_t K, int npad, int planes) {
  const int64_t total = (int64_t)npad * K;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / K;
    const float x = row < Cout ? w[i] : 0.f;
    const float hi = tc::to_tf32(x);
    dst[i] = hi;
    if (planes == 2) dst[total + i] = x - hi;
  }
}

template <int BN, int NS>
int launch_fprop(const epb_conv_geom* g, const CUtensorMap& tmap, const float* in,
                 const float* in_scale, const float* in_shift, const float* bias, float* out,
                 double* stats, int npad, cudaStream_t st) {
  const int64_t M = (int64_t)g->N * g->Hp * g->Wp;
  const int m_tiles = (int)((M + BM - 1) / BM);
  const int n_tiles = npad / BN;
  const int64_t tiles = (int64_t)m_tiles * n_tiles;
  const unsigned grid = (unsigned)(tiles < kNumSMs ? tiles : kNumSMs);
  return tc::launch<conv_fprop_tc_kernel<BN, NS>>(grid, kThreads, Cfg<BN, NS>::SMEM, st, *g, tmap,
                                                  in, in_scale, in_shift, bias, out, stats, npad,
                                                  m_tiles, n_tiles);
}

}  // namespace

bool epb_conv_wgrad_tc_supported(const epb_conv_geom* g);

bool epb_conv_tc_supported(const epb_conv_geom* g, bool wgrad) {
  if (wgrad) return epb_conv_wgrad_tc_supported(g);
  // the producers address the input with 32-bit element offsets
  return g->Cin % 32 == 0 && g->Cout % 32 == 0 && g->Cout >= 32 &&
         (int64_t)g->N * g->Hi * g->Wi * g->Cin < (1LL << 31);
}

int epb_conv_fprop_tc(const epb_conv_geom* g, const float* in, const float* w,
                      const float* in_scale, const float* in_shift, const float* bias, float* out,
                      double* stats, cudaStream_t st) {
  const int ns = g->precision == 3 ? 3 : 1;
  const int planes = ns == 3 ? 2 : 1;
  // N tile: the 128-column accumulator of a consumer warpgroup (64 fp32 registers per thread)
  const int bn = g->Cout >= 128 ? 128 : 64;
  const int npad = (g->Cout + bn - 1) / bn * bn;
  const int64_t K = (int64_t)g->Tw * g->Cin;
  // hi / lo operand planes of this call: scratch of this (device, stream); one slot per
  // stream, so concurrent calls on different streams do not share it
  float* wws = nullptr;
  int rc = epb_workspace(EPB_WS_WPLANES, (size_t)planes * npad * K * sizeof(float), st, (void**)&wws);
  if (rc) return rc;
  {
    int64_t blocks = ((int64_t)npad * K + 255) / 256;
    if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
    prep_weight_tc<<<(int)blocks, 256, 0, st>>>(w, wws, g->Cout, K, npad, planes);
    EPB_LAUNCH_CHECK();
  }
  CUtensorMap tmap;
  const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)((int64_t)planes * npad)};
  const cuuint64_t strides[1] = {(cuuint64_t)(K * sizeof(float))};
  const cuuint32_t box[2] = {(cuuint32_t)BKE, (cuuint32_t)bn};
  rc = epb_encode_map(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, wws, dims, strides, box,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "weight planes");
  if (rc) return rc;
#define EPB_TC_CASE(BN_, NS_)                   \
  if (bn == BN_ && ns == NS_)                   \
    return launch_fprop<BN_, NS_>(g, tmap, in, in_scale, in_shift, bias, out, stats, npad, st);
  EPB_TC_CASE(64, 1) EPB_TC_CASE(128, 1) EPB_TC_CASE(64, 3) EPB_TC_CASE(128, 3)
#undef EPB_TC_CASE
  epb_set_error("no wgmma tile configuration for Cout=%d", g->Cout);
  return EPB_EINVAL;
}
