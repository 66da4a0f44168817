// Host-side helpers of the tensor-core kernels: TMA tensor-map encoding (all four GEMM
// kernels), and the phase-grid tiling and activation maps of the split-fp16 kernels
// (conv16.cu, wgrad16.cu).
#pragma once
#include "conv_common.cuh"
#include "tc_common.cuh"

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency
// on libcuda)
typedef CUresult (*epb_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                        const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                        const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                        CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline epb_encode_tiled_fn epb_get_encode_tiled() {
  static epb_encode_tiled_fn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) ==
            cudaSuccess && qr == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<epb_encode_tiled_fn>(p);
  }
  return fn;
}

// SWIZZLE_128B tiled map of a `rank`-D tensor (dims[0] contiguous, strides in bytes of
// dims 1..rank-1), dense boxes, out-of-range elements read as zero.  `what` names the
// tensor in the error message.
inline int epb_encode_map(CUtensorMap* m, CUtensorMapDataType type, int rank, const void* base,
                          const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box,
                          CUtensorMapL2promotion l2, const char* what) {
  epb_encode_tiled_fn enc = epb_get_encode_tiled();
  if (!enc) {
    epb_set_error("cuTensorMapEncodeTiled entry point unavailable");
    return EPB_ECUDA;
  }
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  const CUresult cr = enc(m, type, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box,
                          estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, l2,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    epb_set_error("cuTensorMapEncodeTiled(%s: dims %llu x %llu, box %u x %u) failed (%d)", what,
                  (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1], (int)cr);
    return EPB_ECUDA;
  }
  return EPB_OK;
}

// A tile of `rows` phase-grid pixels is the box (tw, th, tn) of the (Wp, Hp, N) grid, all
// powers of two with tw*th*tn == rows, so that ONE TMA box load brings the tile (rows in
// w-fastest order).  Chosen to minimise the covered-but-invalid pixels.
inline void epb_choose_tile(int N, int Hp, int Wp, int rows, int& tw, int& th, int& tn) {
  long long best = -1;
  tw = rows; th = 1; tn = 1;
  for (int a = rows; a >= 1; a >>= 1) {
    for (int b = rows / a; b >= 1; b >>= 1) {
      const int c = rows / (a * b);
      const long long cov = (long long)((Wp + a - 1) / a) * ((Hp + b - 1) / b) * ((N + c - 1) / c);
      if (best < 0 || cov < best) { best = cov; tw = a; th = b; tn = c; }
    }
  }
}

// 5-D map over the planes of a split NHWC tensor [2][N][H][W][C] fp16, viewed with spatial
// stride `stride` starting at pixel (qh, qw): coordinates (c, w', h', n, plane) address pixel
// (h'*stride + qh, w'*stride + qw).  Out-of-range coordinates (negative included) read 0.
inline int epb_make_act_map(CUtensorMap* m, const epb_half* base, int N, int H, int W, int C,
                            int stride, int qh, int qw, int tw, int th, int tn) {
  const int Wv = (W - qw + stride - 1) / stride, Hv = (H - qh + stride - 1) / stride;
  if (Wv <= 0 || Hv <= 0) {
    epb_set_error("empty strided view");
    return EPB_EINVAL;
  }
  const cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)Wv, (cuuint64_t)Hv, (cuuint64_t)N, 2};
  const cuuint64_t strides[4] = {(cuuint64_t)stride * C * 2, (cuuint64_t)stride * W * C * 2,
                                 (cuuint64_t)H * W * C * 2, (cuuint64_t)N * H * W * C * 2};
  const cuuint32_t box[5] = {64, (cuuint32_t)tw, (cuuint32_t)th, (cuuint32_t)tn, 1};
  return epb_encode_map(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, base + ((int64_t)qh * W + qw) * C,
                        dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, "activation");
}

// Pixel tiles of the phase grid and the parity view of every tap (kernel parameter)
struct epb_phase_grid {
  int N, Hp, Wp;                               // phase grid
  int tw, th, tn, tiles_w, tiles_h, tiles;     // tile box, tile counts
  short dwq[EPB_MAX_TAPS], dhq[EPB_MAX_TAPS];  // tap offset on its parity view
  unsigned char map[EPB_MAX_TAPS];             // parity view of the tap

  // first pixel (w0, h0, n0) of tile `it`
  __host__ __device__ __forceinline__ void tile_origin(int it, int& w0, int& h0, int& n0) const {
    w0 = (it % tiles_w) * tw; it /= tiles_w;
    h0 = (it % tiles_h) * th;
    n0 = (it / tiles_h) * tn;
  }
};

// Tiles the phase grid of `g` into boxes of `rows` pixels (G's tap fields are left unset).
// A 1x1 stride-1 layer whose phase grid IS the input and the output grid is a plain [M][C]
// matrix: it is collapsed to one row of M pixels (no waste whatever H and W are) and `dense`
// is set.
inline int epb_tile_phase_grid(const epb_conv_geom* g, int rows, epb_phase_grid& G, bool& dense) {
  dense = g->T == 1 && g->is == 1 && g->os == 1 && g->dh[0] == 0 && g->dw[0] == 0 &&
          g->Hp == g->Hi && g->Wp == g->Wi && g->Hp == g->Ho && g->Wp == g->Wo;
  G.N = g->N; G.Hp = g->Hp; G.Wp = g->Wp;
  if (dense) {
    const int64_t M = (int64_t)g->N * g->Hp * g->Wp;
    EPB_CHECK_ARG(M < (1LL << 31));
    G.N = 1; G.Hp = 1; G.Wp = (int)M;
  }
  epb_choose_tile(G.N, G.Hp, G.Wp, rows, G.tw, G.th, G.tn);
  G.tiles_w = (G.Wp + G.tw - 1) / G.tw;
  G.tiles_h = (G.Hp + G.th - 1) / G.th;
  const int64_t tiles = (int64_t)G.tiles_w * G.tiles_h * ((G.N + G.tn - 1) / G.tn);
  EPB_CHECK_ARG(tiles < (1LL << 30));
  G.tiles = (int)tiles;
  return EPB_OK;
}

// epb_tile_phase_grid, then encodes the parity views of the split input `in` that the taps
// read (a tap offset d on a stride-s view has parity q = d mod s and quotient (d - q) / s).
// Slots no tap uses repeat a used view, since the kernels prefetch all four.
inline int epb_plan_phase_grid(const epb_conv_geom* g, const epb_half* in, int rows,
                               epb_phase_grid& G, CUtensorMap (&maps)[4], bool& dense) {
  const int rc = epb_tile_phase_grid(g, rows, G, dense);
  if (rc) return rc;
  bool need[4] = {false, false, false, false};
  for (int t = 0; t < g->T; ++t) {
    const int qh = ((g->dh[t] % g->is) + g->is) % g->is;
    const int qw = ((g->dw[t] % g->is) + g->is) % g->is;
    G.map[t] = (unsigned char)(qh * 2 + qw);
    G.dhq[t] = (short)((g->dh[t] - qh) / g->is);
    G.dwq[t] = (short)((g->dw[t] - qw) / g->is);
    need[qh * 2 + qw] = true;
  }
  const int Hi = dense ? 1 : g->Hi, Wi = dense ? G.Wp : g->Wi;
  for (int v = 0; v < 4; ++v) {
    if (!need[v]) continue;
    const int rv = epb_make_act_map(&maps[v], in, G.N, Hi, Wi, g->Cin, g->is, v >> 1, v & 1,
                                    G.tw, G.th, G.tn);
    if (rv) return rv;
  }
  for (int v = 0; v < 4; ++v)
    if (!need[v]) {
      for (int u = 0; u < 4; ++u)
        if (need[u]) { maps[v] = maps[u]; break; }
    }
  return EPB_OK;
}
