// wgmma weight-gradient kernel of the tap-list implicit GEMM (include/epb.h):
//
//   dw[co][wt[t]][ci] += sum_m dout[pix_out(m)][co] * f(in[pix_in(m, t)][ci])
//
// GEMM view: D[co, ci] with the reduction over pixels m.  wgmma takes 32-bit operands
// only K-major, so the producer warps transpose while they store: they gather 32 pixel
// rows per tile (dout rows, and the tap-shifted input rows with the fused
// BatchNorm+ReLU of the producing layer), split them into TF32 hi (+ lo for 3xTF32) and
// store them channel-major in the SWIZZLE_128B K-major layout (128-byte rows = the 32
// pixels of one channel; 8 channel rows form a 1024-byte atom).
//
// One CTA = (co tile of 128, a group of NB "slots" = (tap, ci tile) pairs, a
// split of the pixel range).  The dout tile A(p) of pixel block p is produced
// ONCE and multiplied against the NB input tiles B(p, b) (two smem rings), each
// slot accumulating into its own registers (NB * BNW <= 128 fp32 columns), so
// dout is gathered once per NB taps instead of once per tap.  Two groups of four
// producer warps take tiles round-robin, so two tiles' global loads are in flight.
// Two consumer warpgroups (64 co rows each) issue wgmma m64nBNWk8 kind tf32 (K = 8
// pixels); their epilogue adds the partial tiles to dw with red.global.add.v2.f32
// (split-K).
#include "conv_common.cuh"
#include "tc_common.cuh"

namespace {

constexpr int WM = 128;          // co rows per tile (two wgmma M = 64 halves); rows >= Cout are zero
constexpr int KPIX = 32;         // pixels per tile (4 MMAs of K = 8)
constexpr int kConsWarps = 8;    // two consumer warpgroups (warps 0-7)
constexpr int kProdWarps = 8;    // producers (warps 8-15)
constexpr int kGroups = 2;       // producer groups of 4 warps (one tile each, round-robin)
constexpr int kProd = 32 * kProdWarps;
constexpr int kThreadsW = 32 * kConsWarps + kProd;
constexpr int kMaxSlots = 16;
// Longest pixel run one CTA accumulates in registers, in KPIX blocks, for 3xTF32.  wgmma adds
// into its fp32 accumulator rounding toward zero, so a run of K pixels drifts toward zero by up
// to ~0.75 * 2^-24 * passes * K / 8 of the result: 184 blocks (5888 pixels) keep that below
// 1e-4 with three passes; one pass may run three times as long.
constexpr int kMaxRunBlocks3 = 184;

template <int BNW, int NS>
struct WCfg {
  static constexpr int PL = (NS == 3) ? 2 : 1;
  static constexpr int A_TILE = WM * KPIX * 4 * PL;      // dout tile  (hi[,lo])
  static constexpr int B_TILE = BNW * KPIX * 4 * PL;     // input tile (hi[,lo])
  static constexpr int SA = 2;
  static constexpr int SB_ = (196 * 1024 - SA * A_TILE) / B_TILE;
  static constexpr int SB = SB_ > 8 ? 8 : SB_;
  static_assert(SB >= 2, "input ring too small");
  static constexpr int NB_MAX = 128 / BNW;              // accumulator registers: 64 per thread
  static constexpr int SMEM = SA * A_TILE + SB * B_TILE + 1024 + 3072;
};

__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

// Store one float4 (4 consecutive channels `ch4*4..` of pixel r) into the K-major tile:
// channel c is the 128-byte row c (its 32 pixels), 16-byte chunk r / 4 of the row XORed
// with c mod 8 (SWIZZLE_128B), pixel r % 4 inside the chunk.
__device__ __forceinline__ void st_k(uint8_t* tile, int r, int ch4, float4 v) {
  const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int c = ch4 * 4 + e;
    const uint32_t off = (uint32_t)c * 128u + (uint32_t)((((r >> 2) ^ (c & 7)) << 4) | ((r & 3) << 2));
    *reinterpret_cast<float*>(tile + off) = x[e];
  }
}

// Slots are awaited by mbarrier PARITY, which is ambiguous for a waiter two phases ahead of
// the barrier.  With tiles handed round-robin to four groups a group can get that far ahead,
// so every ring slot carries a use counter in smem: use k of a slot may start its parity
// wait only after use k-1 has PASSED its own wait (i.e. the release before last is known to
// have happened), and publishes k+1 once it has passed.
__device__ __forceinline__ void wait_seen(const volatile int* p, int need) {
  if (*p >= need) return;
  const long long t0 = clock64();
  while (*p < need)
    if (clock64() - t0 > 4000000000LL) __trap();
}

template <int BNW, int NS>
__global__ void __launch_bounds__(kThreadsW, 1)
conv_wgrad_tc_kernel(const __grid_constant__ epb_conv_geom g, const float* __restrict__ in,
                     const float* __restrict__ dout, const float* __restrict__ in_scale,
                     const float* __restrict__ in_shift, float* __restrict__ dw, int co_tiles,
                     int ci_tiles, int groups, int nb_per_group, int rows_per_split) {
  using C = WCfg<BNW, NS>;
  constexpr int QA = WM / 4;                 // float4 per dout row (32)
  constexpr int QB = BNW / 4;                // float4 per input row
  constexpr int A0 = 0, B0 = C::SA * C::A_TILE, CTRL = B0 + C::SB * C::B_TILE;
  extern __shared__ uint8_t smem_raw[];
  // barriers: fullA[2] emptyA[2] fullB[8] emptyB[8]
  tc::Ring<C::SA, C::A_TILE> ringA(smem_raw, A0, CTRL, CTRL + 16);
  tc::Ring<C::SB, C::B_TILE> ringB(smem_raw, B0, CTRL + 32, CTRL + 96);
  uint8_t* sm = ringA.sm;
  uint8_t* ctrl = sm + CTRL;
  int* slot_t = reinterpret_cast<int*>(ctrl + 256);          // [kMaxSlots] tap of each slot
  int* slot_cit = slot_t + kMaxSlots;                        // [kMaxSlots] ci tile of each slot
  int* rowtab = slot_cit + kMaxSlots;                        // [kGroups][4][KPIX]
  volatile int* seenA = rowtab + kGroups * 4 * KPIX;         // [SA] uses whose wait has passed
  volatile int* seenB = seenA + C::SA;                       // [SB]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // work item decode: blockIdx.x = ((split * co_tiles + cot) * groups + grp)
  int w = blockIdx.x;
  const int grp = w % groups; w /= groups;
  const int cot = w % co_tiles;
  const int split = w / co_tiles;
  const int total_slots = g.T * ci_tiles;
  const int slot0 = grp * nb_per_group;
  const int NB = min(nb_per_group, total_slots - slot0);
  const int M = g.N * g.Hp * g.Wp;
  const int mbeg = split * rows_per_split;
  const int mend = min(M, mbeg + rows_per_split);
  const int nblk = (mend - mbeg + KPIX - 1) / KPIX;
  const int co0 = cot * WM;

  if (threadIdx.x == 0) {
    ringA.init(kProdWarps / kGroups, kConsWarps);
    ringB.init(kProdWarps / kGroups, kConsWarps);
    for (int s = 0; s < C::SA; ++s) seenA[s] = 0;
    for (int s = 0; s < C::SB; ++s) seenB[s] = 0;
    for (int b = 0; b < NB; ++b) {
      slot_t[b] = (slot0 + b) / ci_tiles;
      slot_cit[b] = (slot0 + b) % ci_tiles;
    }
  }
  __syncthreads();

  if (warp >= kConsWarps) {
    // ======================================================== producers (2 groups of 4 warps)
    // Tiles go round-robin to the groups (group = u % 2): each warp pays the per-tile fixed
    // costs (mbarrier wait, proxy fence, arrive) for every second tile, the loads of two
    // tiles are in flight at once, and each SM sub-partition always has the other group's
    // warp to issue from while one waits for its loads (slot hand-over: wait_seen).
    constexpr int GT = kProd / kGroups;            // threads per group (128)
    constexpr int RAg = GT / QA, PAg = KPIX / RAg; // dout rows per pass / passes (4, 8)
    constexpr int RBg = GT / QB, PBg = KPIX / RBg; // input rows per pass / passes
    constexpr int NREG = PAg > PBg ? PAg : PBg;
    const int grpi = (warp - kConsWarps) >> 2;
    const int tg = threadIdx.x & (GT - 1);
    const int qa = tg % QA, ra0 = tg / QA;
    const int qb = tg % QB, rb0 = tg / QB;
    const int co = co0 + qa * 4;
    const bool co_ok = co < g.Cout;
    // dense: phase-grid pixel m IS the dout / input pixel (1x1 stride-1 layers and the
    // dout side of every stride-1 conv): no row table, no bounds checks
    const bool dense_out = g.os == 1 && g.Hp == g.Ho && g.Wp == g.Wo;
    const bool dense_in = g.is == 1 && g.Hp == g.Hi && g.Wp == g.Wi && g.T == 1 &&
                          g.dh[0] == 0 && g.dw[0] == 0;
    const bool need_tab = !(dense_out && dense_in);
    const float lb = g.in_relu ? 0.f : -INFINITY;
    int* rt = rowtab + grpi * 4 * KPIX;           // [dout pixel | n*Hi*Wi | i*is | j*is][KPIX]
    const int per_blk = NB + 1;
    const int total = nblk * per_blk;
    float4 buf[NREG];
    unsigned msk;
    int ie = grpi, iblk = 0, tab_blk = -1;        // tile cursor of this group
    while (ie >= per_blk) { ie -= per_blk; ++iblk; }
    auto split_store = [&](uint8_t* tile, int tile_plane_bytes, int r, int ch4, float4 x) {
      const float4 hi = make_float4(tc::to_tf32(x.x), tc::to_tf32(x.y), tc::to_tf32(x.z),
                                    tc::to_tf32(x.w));
      st_k(tile, r, ch4, hi);
      if (NS == 3)
        st_k(tile + tile_plane_bytes, r, ch4,
              make_float4(x.x - hi.x, x.y - hi.y, x.z - hi.z, x.w - hi.w));
    };
    const int mine = (total - grpi + kGroups - 1) / kGroups;
    for (int k0 = 0; k0 < mine; ++k0) {
      // ---------------------------------------------------------------- loads of this tile
      if (tab_blk != iblk) {                      // the cursor entered a new pixel block
        if (need_tab) {
          asm volatile("bar.sync %0, 128;" ::"r"(2 + grpi) : "memory");
          if (tg < KPIX) {
            const int m = mbeg + iblk * KPIX + tg;
            if (m < mend) {
              const unsigned um = (unsigned)m;
              const unsigned j = um % (unsigned)g.Wp, qq = um / (unsigned)g.Wp;
              const unsigned i = qq % (unsigned)g.Hp, n = qq / (unsigned)g.Hp;
              rt[tg] = ((int)n * g.Ho + ((int)i * g.os + g.ph)) * g.Wo + ((int)j * g.os + g.pw);
              rt[KPIX + tg] = (int)n * g.Hi * g.Wi;
              rt[2 * KPIX + tg] = (int)i * g.is;
              rt[3 * KPIX + tg] = (int)j * g.is;
            } else {
              rt[tg] = -1;
            }
          }
          asm volatile("bar.sync %0, 128;" ::"r"(2 + grpi) : "memory");
        }
        tab_blk = iblk;
      }
      const int m0 = mbeg + iblk * KPIX;
      msk = 0;
      if (ie == 0) {
        // warm L2 eight pixel blocks ahead (rows of a block are contiguous when the phase
        // grid is dense): the register buffers alone keep too few bytes in flight for HBM
        const int pfm = m0 + 8 * KPIX;
        if (pfm < mend) {
          if (g.os == 1) {
            const int lines = (KPIX * WM * 4) / 128;
            for (int l = tg; l < lines; l += GT) {
              const int r = l >> 2, c = (l & 3) * 32;
              if (co0 + c < g.Cout)
                asm volatile("prefetch.global.L2 [%0];" ::"l"(dout + (int64_t)(pfm + r) * g.Cout + co0 + c));
            }
          }
          if (g.is == 1 && g.Hp == g.Hi && g.Wp == g.Wi) {
            const int lpr = g.Cin >> 5;
            for (int l = tg; l < KPIX * lpr; l += GT) {
              const int r = l / lpr, c = (l - r * lpr) * 32;
              asm volatile("prefetch.global.L2 [%0];" ::"l"(in + (int64_t)(pfm + r) * g.Cin + c));
            }
          }
        }
#pragma unroll
        for (int k = 0; k < PAg; ++k) {
          buf[k] = make_float4(0.f, 0.f, 0.f, 0.f);
          const int r = ra0 + k * RAg;
          const int dp = dense_out ? (m0 + r < mend ? m0 + r : -1) : rt[r];
          if (co_ok && dp >= 0)
            buf[k] = *reinterpret_cast<const float4*>(dout + (int64_t)dp * g.Cout + co);
        }
      } else {
        const int sl = ie - 1;
        const int ci = slot_cit[sl] * BNW + qb * 4;
        if (dense_in) {
#pragma unroll
          for (int k = 0; k < PBg; ++k) {
            buf[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            const int mr = m0 + rb0 + k * RBg;
            if (ci < g.Cin && mr < mend) {
              buf[k] = *reinterpret_cast<const float4*>(in + (int64_t)mr * g.Cin + ci);
              msk |= 1u << k;
            }
          }
        } else {
          const int dh = g.dh[slot_t[sl]], dwv = g.dw[slot_t[sl]];
#pragma unroll
          for (int k = 0; k < PBg; ++k) {
            buf[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            const int r = rb0 + k * RBg;
            const int ih = rt[2 * KPIX + r] + dh, iw = rt[3 * KPIX + r] + dwv;
            if (ci < g.Cin && rt[r] >= 0 && ih >= 0 && ih < g.Hi && iw >= 0 && iw < g.Wi) {
              buf[k] = *reinterpret_cast<const float4*>(
                  in + ((int64_t)rt[KPIX + r] + (int64_t)ih * g.Wi + iw) * g.Cin + ci);
              msk |= 1u << k;
            }
          }
        }
      }
      // ---------------------------------------------------------------- convert + store
      if (ie == 0) {
        const int s = iblk % C::SA, use = iblk / C::SA;
        wait_seen(seenA + s, use);
        tc::mbar_wait(ringA.empty(s), (use & 1) ^ 1);
        if (lane == 0) seenA[s] = use + 1;
        uint8_t* tile = sm + A0 + s * C::A_TILE;
#pragma unroll
        for (int k = 0; k < PAg; ++k) split_store(tile, WM * KPIX * 4, ra0 + k * RAg, qa, buf[k]);
        tc::fence_proxy_async();
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(ringA.full(s));
      } else {
        const int qn = iblk * NB + (ie - 1);
        const int s = qn % C::SB;
        const int ci = slot_cit[ie - 1] * BNW + qb * 4;
        float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
        if (in_scale && ci < g.Cin) {
          sc = *reinterpret_cast<const float4*>(in_scale + ci);
          sh = *reinterpret_cast<const float4*>(in_shift + ci);
        }
        const int use = qn / C::SB;
        wait_seen(seenB + s, use);
        tc::mbar_wait(ringB.empty(s), (use & 1) ^ 1);
        if (lane == 0) seenB[s] = use + 1;
        uint8_t* tile = sm + B0 + s * C::B_TILE;
        if (in_scale) {
          // branch-free affine (+ReLU) on every row; rows that were not loaded (image border,
          // end of the pixel range) are post-activation zeros and are patched afterwards
#pragma unroll
          for (int k = 0; k < PBg; ++k) buf[k] = tc::bn_act4(buf[k], sc, sh, lb);
          if (msk != (1u << PBg) - 1u) {
#pragma unroll
            for (int k = 0; k < PBg; ++k)
              if (!((msk >> k) & 1u)) buf[k] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
#pragma unroll
        for (int k = 0; k < PBg; ++k) split_store(tile, BNW * KPIX * 4, rb0 + k * RBg, qb, buf[k]);
        tc::fence_proxy_async();
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(ringB.full(s));
      }
      ie += kGroups;
      while (ie >= per_blk) { ie -= per_blk; ++iblk; }
    }
  } else {
    // ======================================================== consumers (2 warpgroups)
    constexpr int NBM = C::NB_MAX;
    const int wgc = warp >> 2;                  // co rows 64 * wgc .. + 63 of the tile
    float acc[NBM][BNW / 2];
#pragma unroll
    for (int b = 0; b < NBM; ++b)
#pragma unroll
      for (int i = 0; i < BNW / 2; ++i) acc[b][i] = 0.f;
    for (int blk = 0; blk < nblk; ++blk) {
      tc::mbar_wait(ringA.full(ringA.stage), ringA.phase);
      const uint32_t a_hi = ringA.stage_addr(ringA.stage) + wgc * 64 * 128;
#pragma unroll
      for (int b = 0; b < NBM; ++b) {
        if (b < NB) {
          tc::mbar_wait(ringB.full(ringB.stage), ringB.phase);
          const uint32_t b_hi = ringB.stage_addr(ringB.stage);
          tc::fence_acc(acc[b]);
          tc::wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < KPIX / 8; ++ks) {
            const uint64_t ah = tc::desc_kmajor_sw128(a_hi + ks * 32);
            const uint64_t bh = tc::desc_kmajor_sw128(b_hi + ks * 32);
            if (NS == 3)
              tc::mma3_tf32(acc[b], ah, tc::desc_kmajor_sw128(a_hi + WM * KPIX * 4 + ks * 32), bh,
                            tc::desc_kmajor_sw128(b_hi + BNW * KPIX * 4 + ks * 32));
            else
              tc::wgmma_tf32(acc[b], ah, bh, 1);
          }
          tc::wgmma_commit();
          tc::wgmma_wait<0>();
          tc::fence_acc(acc[b]);
          if (lane == 0) tc::mbar_arrive(ringB.empty(ringB.stage));
          ringB.advance();
        }
      }
      if (lane == 0) tc::mbar_arrive(ringA.empty(ringA.stage));
      ringA.advance();
    }
    // ---- epilogue: add the partial tiles to dw (rows co, columns ci of the slot's tap)
    const int64_t wrow = (int64_t)g.Tw * g.Cin;
    const int lc = (lane & 3) * 2;
#pragma unroll
    for (int b = 0; b < NBM; ++b) {
      if (b < NB && nblk > 0) {
        const int t = slot_t[b], cit = slot_cit[b];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int co = co0 + wgc * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
          if (co < g.Cout) {
            float* dst = dw + (int64_t)co * wrow + (int64_t)g.wt[t] * g.Cin;
#pragma unroll
            for (int j = 0; j < BNW / 8; ++j) {
              const int ci = cit * BNW + 8 * j + lc;
              if (ci < g.Cin) red_add_v2(dst + ci, acc[b][4 * j + 2 * h], acc[b][4 * j + 2 * h + 1]);
            }
          }
        }
      }
    }
  }
}

template <int BNW, int NS>
int launch_wgrad(const epb_conv_geom* g, const float* in, const float* dout, const float* in_scale,
                 const float* in_shift, float* dw, cudaStream_t st) {
  using C = WCfg<BNW, NS>;
  const int64_t M = (int64_t)g->N * g->Hp * g->Wp;
  EPB_CHECK_ARG(M < (1LL << 31));
  const int co_tiles = (g->Cout + WM - 1) / WM;
  const int ci_tiles = (g->Cin + BNW - 1) / BNW;
  const int total_slots = g->T * ci_tiles;
  const int groups = (total_slots + C::NB_MAX - 1) / C::NB_MAX;
  const int nb = (total_slots + groups - 1) / groups;          // balanced group size
  const int groups2 = (total_slots + nb - 1) / nb;
  const int64_t tiles = (int64_t)co_tiles * groups2;
  // Split the pixel range so that no CTA's run exceeds the accumulation cap (kMaxRunBlocks3)
  // and the grid fills whole waves of one CTA per SM (a 2.16-wave grid idles most SMs in its
  // last round).  Cost model per split count: rounds x (pixel blocks per CTA + fixed
  // prologue/epilogue cost worth ~6 blocks), over up to three waves past the fewest splits.
  const int64_t max_splits = (M + 8 * KPIX - 1) / (8 * KPIX);   // >= 8 pixel blocks per CTA
  const int64_t run_cap = (int64_t)kMaxRunBlocks3 * 3 / NS * KPIX;
  const int64_t min_splits = (M + run_cap - 1) / run_cap;
  int64_t splits = min_splits;
  int64_t best = -1;
  for (int64_t sp = min_splits; sp <= max_splits && (sp - min_splits) * tiles <= 3 * kNumSMs; ++sp) {
    const int64_t rounds = (sp * tiles + kNumSMs - 1) / kNumSMs;
    const int64_t blocks = ((M + sp - 1) / sp + KPIX - 1) / KPIX;
    const int64_t cost = rounds * (blocks + 6);
    if (best < 0 || cost < best) { best = cost; splits = sp; }
  }
  int64_t rows = (M + splits - 1) / splits;
  rows = (rows + KPIX - 1) / KPIX * KPIX;
  splits = (M + rows - 1) / rows;
  const int64_t grid = tiles * splits;
  EPB_CHECK_ARG(grid < (1LL << 31));
  return tc::launch<conv_wgrad_tc_kernel<BNW, NS>>((unsigned)grid, kThreadsW, C::SMEM, st, *g, in,
                                                   dout, in_scale, in_shift, dw, co_tiles,
                                                   ci_tiles, groups2, nb, (int)rows);
}

}  // namespace

bool epb_conv_wgrad_tc_supported(const epb_conv_geom* g) {
  // 32-bit element offsets into the input / pixel indices into dout
  return g->Cin % 32 == 0 && g->Cout % 4 == 0 && g->Cout >= 32 &&
         (int64_t)g->N * g->Hi * g->Wi * g->Cin < (1LL << 31) &&
         (int64_t)g->N * g->Ho * g->Wo < (1LL << 31);
}

int epb_conv_wgrad_tc(const epb_conv_geom* g, const float* in, const float* dout,
                      const float* in_scale, const float* in_shift, float* dw, cudaStream_t st) {
  const int ns = g->precision == 3 ? 3 : 1;
  const int bn = g->Cin >= 128 ? 128 : (g->Cin >= 64 ? 64 : 32);
#define EPB_WG_CASE(BN_, NS_) \
  if (bn == BN_ && ns == NS_) return launch_wgrad<BN_, NS_>(g, in, dout, in_scale, in_shift, dw, st);
  EPB_WG_CASE(32, 1) EPB_WG_CASE(64, 1) EPB_WG_CASE(128, 1)
  EPB_WG_CASE(32, 3) EPB_WG_CASE(64, 3) EPB_WG_CASE(128, 3)
#undef EPB_WG_CASE
  epb_set_error("no wgmma wgrad configuration for Cin=%d", g->Cin);
  return EPB_EINVAL;
}
