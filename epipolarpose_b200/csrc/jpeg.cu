// JPEG decode on the device, bit-exact against cv2.imread(IMREAD_COLOR | IMREAD_IGNORE_ORIENTATION)
// (libjpeg-turbo): the first stage of the reference's get_single_patch_sample
// (lib/utils/img_utils.py:251-252).  Baseline / extended-sequential Huffman, 8-bit, one interleaved
// scan; 1 component or YCbCr with luma 1x1, 2x1, 1x2, 2x2 and chroma 1x1; restart intervals.
//
// Stages (one call, one stream, no host round trip):
//   1. header parse on the host (epb_jpeg_parse): one fixed-size JpegDesc per image;
//   2. unstuff: drop the 0x00 after each 0xFF, cut at RSTn (one segment per restart interval),
//      stop at the first other marker -- one block per image, block scans over 2 KB chunks;
//   3. Huffman decode by self-synchronisation (Weissenberger & Schmidt, ICPP 2018): every segment
//      is cut into subsequences of kJpegSubBits bits, one thread each.  The decoder state
//      (bit position, block slot in the MCU, zig-zag index) fixes the next table, so decoding is
//      a deterministic map.  Phase A: each thread decodes its subsequence from an assumed start
//      (slot 0, index 0) and records the exit state; then rounds in which each thread carries
//      the exit state into the next subsequence and walks on until it meets the recorded state,
//      overwriting what differs.  A round without a write proves every state exact (by induction
//      from the segment start, which is exact).  Phase B: count the blocks and DC differences
//      each subsequence holds from its exact start, and scan them per segment.  Phase C: decode again from the exact states and
//      write int16 coefficients (natural order, absolute DC);
//   4. dequantise + ISLOW IDCT (jidctint.c) into per-component planes at MCU-padded size;
//   5. fancy upsampling (jdsample.c) + YCbCr->BGR (jdcolor.c) into the frame layout that
//      epb_patch_sample reads.
// Integer arithmetic throughout: the decode is bitwise deterministic.
#include "common.cuh"
#include <string.h>

namespace {

constexpr int kJpegSubBits = 1024;     // subsequence length of the device decode
constexpr int kJpegRounds = 6;         // phase-A rounds before the per-segment sequential walk
constexpr int kUnstuffThreads = 512;
constexpr int kUnstuffItems = 4;

enum { JPEG_OK = 0, JPEG_UNSUPPORTED = 1, JPEG_MALFORMED = 2 };

struct JpegHuff {
  uint16_t look[512];      // 9-bit prefix -> (length << 8) | symbol, 0 when the code is longer
  int32_t maxcode[18];     // largest code of each length, -1 if none
  int32_t valoff[18];      // index into val of code c of length l: c + valoff[l]
  uint8_t val[256];
};

struct JpegDesc {
  int32_t status, H, W, ncomp;
  int32_t hmax, vmax, mcux, mcuy, bpm, ri, nseg, nsub_max;
  int32_t ch[3], cv[3], cdc[3], cac[3];          // sampling; Huffman table slot (dc 0..1, ac 2..3)
  int32_t pw[3], ph[3], dw[3], dh[3];            // padded plane / downsampled (real) extent
  int32_t slot_comp[10], slot_bx[10], slot_by[10];
  int32_t pad0;
  int64_t ent_off, ent_len, nblocks;
  int64_t ws_stream, ws_seg, ws_ent, ws_pb, ws_coef, ws_plane[3];
  uint16_t qt[3][64];                            // per component, zig-zag order
  JpegHuff huff[4];
};
static_assert(sizeof(JpegDesc) <= EPB_JPEG_DESC_BYTES, "descriptor size");

// per-image info block at the start of ws_seg: [0] bytes, [1] segments found, [2] bad,
// then seg[nseg + 1] (byte starts; seg[nseg] = end), then sub[nseg + 1] (first subsequence)
constexpr int kSegHdr = 4;

// one phase-A/C record per subsequence: exit state and what the subsequence holds
struct JpegEntry {
  uint64_t st;             // p:32 | c:4 | k:7 | dead:1 | n:20 (blocks completed)
  int32_t dc[3];           // sum of DC differences per component
  int32_t pad;
};
struct JpegPrefix {
  int32_t first;           // blocks completed in the segment before this subsequence
  int32_t dc[3];           // DC predictor per component at its start
};

__host__ __device__ inline uint64_t st_make(uint32_t p, int c, int k, int dead, int n) {
  return (uint64_t)p | ((uint64_t)c << 32) | ((uint64_t)k << 36) | ((uint64_t)dead << 43) |
         ((uint64_t)n << 44);
}
__host__ __device__ inline uint32_t st_p(uint64_t s) { return (uint32_t)s; }
__host__ __device__ inline int st_c(uint64_t s) { return (int)((s >> 32) & 15); }
__host__ __device__ inline int st_k(uint64_t s) { return (int)((s >> 36) & 127); }
__host__ __device__ inline int st_dead(uint64_t s) { return (int)((s >> 43) & 1); }
__host__ __device__ inline int st_n(uint64_t s) { return (int)(s >> 44); }
__host__ __device__ inline uint64_t st_clear_n(uint64_t s) { return s & ((1ull << 44) - 1); }

#define JPEG_ZIGZAG {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  \
                     12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, \
                     35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, \
                     58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63}
__constant__ uint8_t kZigzagDev[64] = JPEG_ZIGZAG;
const uint8_t kZigzagHost[64] = JPEG_ZIGZAG;

__host__ __device__ inline int zigzag_natural(int k) {
#ifdef __CUDA_ARCH__
  return kZigzagDev[k];
#else
  return kZigzagHost[k];
#endif
}

// ------------------------------------------------------------------ 1. header parse (host)
inline int rd16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// jdhuff.c jpeg_make_d_derived_tbl: canonical codes; an over-full code is malformed
inline int huff_build(const uint8_t* bits, const uint8_t* val, int nsym, bool dc, JpegHuff* t) {
  memset(t, 0, sizeof(*t));
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    t->valoff[l] = k - code;
    k += bits[l];
    code += bits[l];
    if (code > (1 << l)) return JPEG_MALFORMED;
    t->maxcode[l] = bits[l] ? code - 1 : -1;
    code <<= 1;
  }
  t->maxcode[17] = 0x7fffffff;
  for (int i = 0; i < nsym; ++i) {
    if (dc && val[i] > 15) return JPEG_MALFORMED;
    t->val[i] = val[i];
  }
  code = 0;
  k = 0;
  for (int l = 1; l <= 9; ++l) {
    for (int i = 0; i < bits[l]; ++i, ++code, ++k)
      for (int f = 0; f < (1 << (9 - l)); ++f) t->look[(code << (9 - l)) | f] = (uint16_t)((l << 8) | val[k]);
    code <<= 1;
  }
  return JPEG_OK;
}

struct ParseTables {
  uint16_t q[4][64];
  bool qdef[4];
  uint8_t hbits[8][17], hval[8][256];
  int hn[8];
  bool hdef[8];            // 0..3 DC, 4..7 AC
};

// Reads a blob up to SOS and fills d (geometry, tables, entropy range).  Returns the status.
inline int jpeg_parse_one(const uint8_t* b, int64_t n, int sub_bits, JpegDesc* d) {
  memset(d, 0, sizeof(*d));
  ParseTables* T = new ParseTables();
  memset(T, 0, sizeof(*T));
  int rc = JPEG_MALFORMED;
  int64_t i = 2;
  bool sof = false, jfif = false, adobe = false;
  int adobe_transform = -1, cid[3] = {0, 0, 0}, cq[3] = {0, 0, 0};
  if (n < 4 || b[0] != 0xFF || b[1] != 0xD8) goto done;
  for (;;) {
    if (i + 4 > n) goto done;
    if (b[i] != 0xFF) goto done;
    while (i < n && b[i] == 0xFF) ++i;
    if (i + 3 > n) goto done;
    const int m = b[i++];
    if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) goto done;
    const int len = rd16(b + i);
    if (len < 2 || i + len > n) goto done;
    const uint8_t* s = b + i + 2;
    const int sl = len - 2;
    i += len;
    if (m == 0xC0 || m == 0xC1) {
      if (sof || sl < 6) goto done;
      sof = true;
      if (s[0] != 8) { rc = JPEG_UNSUPPORTED; goto done; }
      d->H = rd16(s + 1);
      d->W = rd16(s + 3);
      d->ncomp = s[5];
      if (d->W == 0) goto done;
      if (d->H == 0) { rc = JPEG_UNSUPPORTED; goto done; }              // DNL
      if (d->ncomp != 1 && d->ncomp != 3) { rc = d->ncomp == 0 ? JPEG_MALFORMED : JPEG_UNSUPPORTED; goto done; }
      if (sl < 6 + 3 * d->ncomp) goto done;
      for (int c = 0; c < d->ncomp; ++c) {
        cid[c] = s[6 + 3 * c];
        d->ch[c] = s[7 + 3 * c] >> 4;
        d->cv[c] = s[7 + 3 * c] & 15;
        cq[c] = s[8 + 3 * c];
        if (d->ch[c] < 1 || d->ch[c] > 4 || d->cv[c] < 1 || d->cv[c] > 4 || cq[c] > 3) goto done;
      }
    } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4) {
      rc = JPEG_UNSUPPORTED;                    // progressive, lossless, hierarchical, arithmetic
      goto done;
    } else if (m == 0xC4) {
      int o = 0;
      while (o < sl) {
        if (o + 17 > sl) goto done;
        const int tc = s[o] >> 4, th = s[o] & 15;
        if (tc > 1 || th > 3) goto done;
        int cnt = 0;
        for (int l = 1; l <= 16; ++l) cnt += s[o + l];
        if (cnt > 256 || o + 17 + cnt > sl) goto done;
        const int slot = tc * 4 + th;
        T->hbits[slot][0] = 0;
        for (int l = 1; l <= 16; ++l) T->hbits[slot][l] = s[o + l];
        memcpy(T->hval[slot], s + o + 17, cnt);
        T->hn[slot] = cnt;
        T->hdef[slot] = true;
        JpegHuff tmp;
        if (huff_build(T->hbits[slot], T->hval[slot], cnt, tc == 0, &tmp) != JPEG_OK) goto done;
        o += 17 + cnt;
      }
    } else if (m == 0xDB) {
      int o = 0;
      while (o < sl) {
        const int pq = s[o] >> 4, tq = s[o] & 15;
        if (pq > 1 || tq > 3) goto done;
        const int need = 1 + 64 * (pq + 1);
        if (o + need > sl) goto done;
        for (int k = 0; k < 64; ++k) T->q[tq][k] = pq ? (uint16_t)rd16(s + o + 1 + 2 * k) : s[o + 1 + k];
        T->qdef[tq] = true;
        o += need;
      }
    } else if (m == 0xDD) {
      if (sl != 2) goto done;
      d->ri = rd16(s);
    } else if (m == 0xE0) {
      if (sl >= 5 && !memcmp(s, "JFIF\0", 5)) jfif = true;
    } else if (m == 0xEE) {
      if (sl >= 12 && !memcmp(s, "Adobe", 5)) { adobe = true; adobe_transform = s[11]; }
    } else if ((m >= 0xE1 && m <= 0xEF) || m == 0xFE) {
      // APPn / COM: skipped (EXIF orientation is ignored, as IMREAD_IGNORE_ORIENTATION does)
    } else if (m == 0xDA) {
      if (!sof || sl < 1) goto done;
      const int ns = s[0];
      if (sl != 4 + 2 * ns || ns < 1) goto done;
      if (ns != d->ncomp) { rc = JPEG_UNSUPPORTED; goto done; }       // non-interleaved scans
      const int ss = s[1 + 2 * ns], se = s[2 + 2 * ns], a = s[3 + 2 * ns];
      if (ss != 0 || se != 63 || a != 0) { rc = JPEG_UNSUPPORTED; goto done; }
      if (d->ncomp == 3) {
        const bool rgb = jfif ? false : adobe ? adobe_transform != 1
                                              : (cid[0] == 'R' && cid[1] == 'G' && cid[2] == 'B');
        if (rgb) { rc = JPEG_UNSUPPORTED; goto done; }
        for (int c = 1; c < 3; ++c)
          if (d->ch[c] != 1 || d->cv[c] != 1) { rc = JPEG_UNSUPPORTED; goto done; }
        if (d->ch[0] > 2 || d->cv[0] > 2) { rc = JPEG_UNSUPPORTED; goto done; }   // 4:1:1 and wider
        d->hmax = d->ch[0];
        d->vmax = d->cv[0];
      } else {
        d->ch[0] = d->cv[0] = d->hmax = d->vmax = 1;                  // one block per MCU
      }
      int used_dc[2] = {-1, -1}, used_ac[2] = {-1, -1}, order[3];
      for (int q = 0; q < ns; ++q) {
        const int id = s[1 + 2 * q], td = s[2 + 2 * q] >> 4, ta = s[2 + 2 * q] & 15;
        int c = -1;
        for (int k = 0; k < d->ncomp; ++k)
          if (cid[k] == id) c = k;
        if (c < 0 || td > 3 || ta > 3) goto done;
        for (int k = 0; k < q; ++k)
          if (order[k] == c) goto done;
        order[q] = c;
        if (!T->hdef[td] || !T->hdef[4 + ta] || !T->qdef[cq[c]]) goto done;
        int sd = used_dc[0] == td ? 0 : used_dc[1] == td ? 1 : used_dc[0] < 0 ? 0 : used_dc[1] < 0 ? 1 : -1;
        int sa = used_ac[0] == ta ? 0 : used_ac[1] == ta ? 1 : used_ac[0] < 0 ? 0 : used_ac[1] < 0 ? 1 : -1;
        if (sd < 0 || sa < 0) { rc = JPEG_UNSUPPORTED; goto done; }
        used_dc[sd] = td;
        used_ac[sa] = ta;
        d->cdc[c] = sd;
        d->cac[c] = 2 + sa;
        memcpy(d->qt[c], T->q[cq[c]], sizeof(d->qt[c]));
      }
      for (int k = 0; k < 2; ++k) {
        if (used_dc[k] >= 0) huff_build(T->hbits[used_dc[k]], T->hval[used_dc[k]], T->hn[used_dc[k]], true, &d->huff[k]);
        if (used_ac[k] >= 0)
          huff_build(T->hbits[4 + used_ac[k]], T->hval[4 + used_ac[k]], T->hn[4 + used_ac[k]], false, &d->huff[2 + k]);
      }
      d->mcux = (d->W + 8 * d->hmax - 1) / (8 * d->hmax);
      d->mcuy = (d->H + 8 * d->vmax - 1) / (8 * d->vmax);
      int slot = 0;
      for (int q = 0; q < ns; ++q) {
        const int c = order[q];
        for (int y = 0; y < d->cv[c]; ++y)
          for (int x = 0; x < d->ch[c]; ++x) {
            d->slot_comp[slot] = c;
            d->slot_bx[slot] = x;
            d->slot_by[slot] = y;
            ++slot;
          }
      }
      d->bpm = slot;
      for (int c = 0; c < d->ncomp; ++c) {
        d->pw[c] = d->mcux * d->ch[c] * 8;
        d->ph[c] = d->mcuy * d->cv[c] * 8;
        d->dw[c] = (int)(((int64_t)d->W * d->ch[c] + d->hmax - 1) / d->hmax);
        d->dh[c] = (int)(((int64_t)d->H * d->cv[c] + d->vmax - 1) / d->vmax);
      }
      const int64_t mcus = (int64_t)d->mcux * d->mcuy;
      d->nblocks = mcus * d->bpm;
      d->nseg = d->ri ? (int32_t)((mcus + d->ri - 1) / d->ri) : 1;
      d->ent_off = i;
      d->ent_len = n - i;
      if (d->ent_len >= (int64_t)1 << 28) { rc = JPEG_UNSUPPORTED; goto done; }   // 32-bit bit positions
      d->nsub_max = (int32_t)((d->ent_len * 8 + sub_bits - 1) / sub_bits) + d->nseg;
      rc = JPEG_OK;
      goto done;
    } else if (m == 0xDC) {
      rc = JPEG_UNSUPPORTED;
      goto done;
    }
  }
done:
  delete T;
  d->status = rc;
  return rc;
}

__host__ __device__ inline int64_t align16(int64_t v) { return (v + 15) & ~(int64_t)15; }

// workspace layout: every region of every image, 16-byte aligned; returns the total bytes and
// the byte range [coef[0], coef[1]) that holds every image's coefficients
inline int64_t jpeg_layout(JpegDesc* d, int B, int64_t* coef) {
  int64_t o = 64 + 16 * kJpegRounds;         // header: phase-A round flags
  for (int b = 0; b < B; ++b) {
    if (d[b].status != JPEG_OK) continue;
    d[b].ws_stream = o; o = align16(o + d[b].ent_len + 16);
    d[b].ws_seg = o;    o = align16(o + 4 * ((int64_t)kSegHdr + 2 * (d[b].nseg + 1)));
    d[b].ws_ent = o;    o = align16(o + (int64_t)sizeof(JpegEntry) * d[b].nsub_max);
    d[b].ws_pb = o;     o = align16(o + (int64_t)sizeof(JpegPrefix) * d[b].nsub_max);
  }
  coef[0] = o;
  for (int b = 0; b < B; ++b) {               // coefficients together: one memset
    if (d[b].status != JPEG_OK) continue;
    d[b].ws_coef = o; o = align16(o + d[b].nblocks * 128);
  }
  coef[1] = o;
  for (int b = 0; b < B; ++b) {
    if (d[b].status != JPEG_OK) continue;
    for (int c = 0; c < d[b].ncomp; ++c) {
      d[b].ws_plane[c] = o;
      o = align16(o + (int64_t)d[b].pw[c] * d[b].ph[c]);
    }
  }
  return o;
}

// ------------------------------------------------------------------ 3. Huffman decode
__host__ __device__ inline uint32_t peek32(const uint8_t* s, uint32_t p) {
  const uint8_t* q = s + (p >> 3);
  const uint64_t w = ((uint64_t)q[0] << 32) | ((uint64_t)q[1] << 24) | ((uint64_t)q[2] << 16) |
                     ((uint64_t)q[3] << 8) | (uint64_t)q[4];
  return (uint32_t)(w >> (8 - (p & 7)));
}

__host__ __device__ inline int huff_extend(uint32_t v, int s) {
  return v < (1u << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v;
}

// Decodes from `st` while the bit position is below end_bit.  A codeword that is not in the
// table, a coefficient index past 63, or a codeword that runs past the segment end makes the
// state dead (absorbing).  The exit state's n counts the blocks completed in this run.
// sink.dc(comp, diff, nblk) / sink.ac(k, value, nblk) receive the coefficients.
template <class Sink>
__host__ __device__ inline uint64_t jpeg_run(const JpegDesc& d, const uint8_t* bits, uint64_t st,
                                             uint32_t end_bit, uint32_t seg_end_bit, Sink& sink) {
  uint32_t p = st_p(st);
  int c = st_c(st), k = st_k(st), n = 0;
  if (st_dead(st)) return st_make(p < end_bit ? end_bit : p, c, k, 1, 0);
  while (p < end_bit) {
    const int comp = d.slot_comp[c];
    const JpegHuff& t = d.huff[k == 0 ? d.cdc[comp] : d.cac[comp]];
    const uint32_t w = peek32(bits, p);
    int len, sym;
    const uint32_t look = t.look[w >> 23];
    if (look) {
      len = (int)(look >> 8);
      sym = (int)(look & 255);
    } else {
      len = 0;
      sym = 0;
      for (int l = 10; l <= 16; ++l) {
        const int32_t code = (int32_t)(w >> (32 - l));
        if (code <= t.maxcode[l]) { len = l; sym = t.val[(code + t.valoff[l]) & 255]; break; }
      }
      if (!len) return st_make(end_bit, c, k, 1, n);
    }
    const int s = k == 0 ? sym : (sym & 15);
    const uint32_t v = s ? ((w << len) >> (32 - s)) : 0u;
    p += (uint32_t)(len + s);
    if (p > seg_end_bit) return st_make(p, c, k, 1, n);
    if (k == 0) {
      sink.dc(comp, s ? huff_extend(v, s) : 0, n);
      k = 1;
    } else {
      const int r = sym >> 4;
      if (s) {
        k += r;
        if (k > 63) return st_make(p < end_bit ? end_bit : p, c, k & 63, 1, n);
        sink.ac(k, huff_extend(v, s), n);
        ++k;
      } else if (r == 15) {
        k += 16;
      } else {
        k = 64;
      }
    }
    if (k >= 64) {
      ++n;
      k = 0;
      c = c + 1 == d.bpm ? 0 : c + 1;
    }
  }
  return st_make(p, c, k, 0, n);
}

struct SinkCount {
  int32_t sum[3] = {0, 0, 0};
  __host__ __device__ void dc(int comp, int v, int) { sum[comp] += v; }
  __host__ __device__ void ac(int, int, int) {}
};

struct SinkWrite {
  int16_t* coef;           // first block of this run
  int32_t pred[3];
  int32_t limit;           // blocks of the segment left from the run's first block
  __host__ __device__ void dc(int comp, int v, int blk) {
    pred[comp] += v;
    if (blk < limit) coef[(int64_t)blk * 64] = (int16_t)pred[comp];
  }
  __host__ __device__ void ac(int k, int v, int blk) {
    if (blk < limit) coef[(int64_t)blk * 64 + zigzag_natural(k)] = (int16_t)v;
  }
};

// geometry of subsequence j of an image whose unstuffing is done
struct SubGeom {
  int seg, first, last;            // segment, its first and one-past-last subsequence
  uint32_t start, end, seg_end;    // bits
};

__host__ __device__ inline SubGeom sub_geom(const int32_t* seg, const int32_t* sub, int nseg, int j,
                                            int sub_bits) {
  int lo = 0, hi = nseg;             // largest s with sub[s] <= j
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (sub[mid] <= j) lo = mid; else hi = mid;
  }
  SubGeom g;
  g.seg = lo;
  g.first = sub[lo];
  g.last = sub[lo + 1];
  const uint32_t s0 = (uint32_t)seg[lo] * 8u;
  g.seg_end = (uint32_t)seg[lo + 1] * 8u;
  g.start = s0 + (uint32_t)(j - g.first) * (uint32_t)sub_bits;
  g.end = g.start + (uint32_t)sub_bits < g.seg_end ? g.start + (uint32_t)sub_bits : g.seg_end;
  return g;
}

__host__ __device__ inline int nsub_of(int32_t bytes, int sub_bits) {
  const int64_t n = ((int64_t)bytes * 8 + sub_bits - 1) / sub_bits;
  return n < 1 ? 1 : (int)n;
}

// decode subsequence j (geometry g) from start state st: its entry
__host__ __device__ inline JpegEntry jpeg_sub_entry(const JpegDesc& d, const uint8_t* bits, const SubGeom& g,
                                                    uint64_t st) {
  SinkCount sk;
  JpegEntry e;
  e.st = jpeg_run(d, bits, st, g.end, g.seg_end, sk);
  e.dc[0] = sk.sum[0];
  e.dc[1] = sk.sum[1];
  e.dc[2] = sk.sum[2];
  e.pad = 0;
  return e;
}

// phase A, first pass: subsequence j from the assumed start (the exact one at a segment start)
__host__ __device__ inline JpegEntry jpeg_sub_phase_a(const JpegDesc& d, const uint8_t* bits, const SubGeom& g) {
  return jpeg_sub_entry(d, bits, g, st_make(g.start, 0, 0, 0, 0));
}

// synchronised: the same decoder state (bit position, slot, zig-zag index, dead); what the
// subsequence holds (blocks, DC sums) depends on where it started and is counted afterwards
__host__ __device__ inline bool state_eq(uint64_t a, uint64_t b) { return st_clear_n(a) == st_clear_n(b); }

// after synchronisation: blocks and DC sums of subsequence j from its exact start
__host__ __device__ inline JpegPrefix jpeg_sub_count(const JpegDesc& d, const uint8_t* bits, const SubGeom& g,
                                                     uint64_t start) {
  const JpegEntry e = jpeg_sub_entry(d, bits, g, start);
  JpegPrefix c;
  c.first = st_n(e.st);
  c.dc[0] = e.dc[0];
  c.dc[1] = e.dc[1];
  c.dc[2] = e.dc[2];
  return c;
}

// phase C: decode subsequence j from its exact start and write its coefficients
__host__ __device__ inline void jpeg_sub_phase_c(const JpegDesc& d, const uint8_t* bits, const SubGeom& g,
                                                 uint64_t start, const JpegPrefix& pf, int16_t* coef_img,
                                                 int64_t seg_first_block, int32_t seg_blocks) {
  SinkWrite w;
  w.coef = coef_img + (seg_first_block + pf.first) * 64;
  w.pred[0] = pf.dc[0];
  w.pred[1] = pf.dc[1];
  w.pred[2] = pf.dc[2];
  w.limit = seg_blocks - pf.first;
  // a block that began in the previous subsequence is block 0 of this run
  jpeg_run(d, bits, start, g.end, g.seg_end, w);
}

__host__ __device__ inline int64_t seg_first_block(const JpegDesc& d, int s) {
  return d.ri ? (int64_t)s * d.ri * d.bpm : 0;
}
__host__ __device__ inline int32_t seg_blocks(const JpegDesc& d, int s) {
  const int64_t mcus = (int64_t)d.mcux * d.mcuy;
  if (!d.ri) return (int32_t)(mcus * d.bpm);
  const int64_t m0 = (int64_t)s * d.ri, m1 = m0 + d.ri < mcus ? m0 + d.ri : mcus;
  return (int32_t)((m1 - m0) * d.bpm);
}

// ------------------------------------------------------------------ 4. ISLOW IDCT (jidctint.c)
__host__ __device__ inline uint8_t idct_limit(int v) {
  const int x = v & 1023;                      // range_limit[x & RANGE_MASK] of IDCT_range_limit
  return (uint8_t)(x < 128 ? x + 128 : x < 512 ? 255 : x < 896 ? 0 : x - 896);
}

__host__ __device__ inline void jpeg_idct_block(const int16_t* coef, const uint16_t* qt_zz, uint8_t* out,
                                                int64_t pitch) {
  const int CB = 13, P1 = 2;
  int q[64];
  for (int k = 0; k < 64; ++k) q[zigzag_natural(k)] = (int)(int16_t)qt_zz[k];
  int ws[64];
  for (int col = 0; col < 8; ++col) {
    int64_t in[8];
    for (int r = 0; r < 8; ++r) in[r] = (int64_t)coef[r * 8 + col] * q[r * 8 + col];
    int64_t z2 = in[2], z3 = in[6];
    int64_t z1 = (z2 + z3) * 4433;
    int64_t tmp2 = z1 + z3 * -15137, tmp3 = z1 + z2 * 6270;
    z2 = in[0];
    z3 = in[4];
    int64_t tmp0 = (z2 + z3) * (1 << CB), tmp1 = (z2 - z3) * (1 << CB);
    const int64_t t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
    tmp0 = in[7]; tmp1 = in[5]; tmp2 = in[3]; tmp3 = in[1];
    z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
    int64_t z4 = tmp1 + tmp3;
    const int64_t z5 = (z3 + z4) * 9633;
    tmp0 *= 2446; tmp1 *= 16819; tmp2 *= 25172; tmp3 *= 12299;
    z1 *= -7373; z2 *= -20995; z3 *= -16069; z4 *= -3196;
    z3 += z5; z4 += z5;
    tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
    const int sh = CB - P1;
    const int64_t rnd = (int64_t)1 << (sh - 1);
    ws[0 * 8 + col] = (int)((t10 + tmp3 + rnd) >> sh);
    ws[7 * 8 + col] = (int)((t10 - tmp3 + rnd) >> sh);
    ws[1 * 8 + col] = (int)((t11 + tmp2 + rnd) >> sh);
    ws[6 * 8 + col] = (int)((t11 - tmp2 + rnd) >> sh);
    ws[2 * 8 + col] = (int)((t12 + tmp1 + rnd) >> sh);
    ws[5 * 8 + col] = (int)((t12 - tmp1 + rnd) >> sh);
    ws[3 * 8 + col] = (int)((t13 + tmp0 + rnd) >> sh);
    ws[4 * 8 + col] = (int)((t13 - tmp0 + rnd) >> sh);
  }
  for (int row = 0; row < 8; ++row) {
    const int* w = ws + row * 8;
    int64_t z2 = w[2], z3 = w[6];
    int64_t z1 = (z2 + z3) * 4433;
    int64_t tmp2 = z1 + z3 * -15137, tmp3 = z1 + z2 * 6270;
    int64_t tmp0 = ((int64_t)w[0] + w[4]) * (1 << CB), tmp1 = ((int64_t)w[0] - w[4]) * (1 << CB);
    const int64_t t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
    tmp0 = w[7]; tmp1 = w[5]; tmp2 = w[3]; tmp3 = w[1];
    z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
    int64_t z4 = tmp1 + tmp3;
    const int64_t z5 = (z3 + z4) * 9633;
    tmp0 *= 2446; tmp1 *= 16819; tmp2 *= 25172; tmp3 *= 12299;
    z1 *= -7373; z2 *= -20995; z3 *= -16069; z4 *= -3196;
    z3 += z5; z4 += z5;
    tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
    const int sh = CB + P1 + 3;
    const int64_t rnd = (int64_t)1 << (sh - 1);
    uint8_t* o = out + row * pitch;
    o[0] = idct_limit((int)((t10 + tmp3 + rnd) >> sh));
    o[7] = idct_limit((int)((t10 - tmp3 + rnd) >> sh));
    o[1] = idct_limit((int)((t11 + tmp2 + rnd) >> sh));
    o[6] = idct_limit((int)((t11 - tmp2 + rnd) >> sh));
    o[2] = idct_limit((int)((t12 + tmp1 + rnd) >> sh));
    o[5] = idct_limit((int)((t12 - tmp1 + rnd) >> sh));
    o[3] = idct_limit((int)((t13 + tmp0 + rnd) >> sh));
    o[4] = idct_limit((int)((t13 - tmp0 + rnd) >> sh));
  }
}

// block blk (MCU order) of an image -> its plane and the top-left of its 8x8 tile
__host__ __device__ inline void block_place(const JpegDesc& d, int64_t blk, int* comp, int64_t* off) {
  const int64_t mcu = blk / d.bpm;
  const int slot = (int)(blk - mcu * d.bpm);
  const int c = d.slot_comp[slot];
  const int64_t mx = mcu % d.mcux, my = mcu / d.mcux;
  const int64_t bx = mx * d.ch[c] + d.slot_bx[slot], by = my * d.cv[c] + d.slot_by[slot];
  *comp = c;
  *off = by * 8 * d.pw[c] + bx * 8;
}

// ------------------------------------------------------------------ 5. upsample + colour
// jdsample.c: fancy (triangle) upsampling of chroma sample (x, y) of the output grid
__host__ __device__ inline int chroma_at(const JpegDesc& d, const uint8_t* pl, int c, int x, int y) {
  const int hs = d.hmax / d.ch[c], vs = d.vmax / d.cv[c];
  const int64_t pw = d.pw[c];
  const int dw = d.dw[c], dh = d.dh[c];
  auto P = [&](int yy, int xx) -> int { return pl[(int64_t)yy * pw + xx]; };
  if (hs == 1 && vs == 1) return P(y, x);
  if (hs == 2 && vs == 1) {
    const int cx = x >> 1;
    if (dw <= 2) return P(y, cx);
    if (!(x & 1)) return cx == 0 ? P(y, 0) : (P(y, cx) * 3 + P(y, cx - 1) + 1) >> 2;
    return cx == dw - 1 ? P(y, cx) : (P(y, cx) * 3 + P(y, cx + 1) + 2) >> 2;
  }
  if (hs == 1 && vs == 2) {
    const int cy = y >> 1;
    if (!(y & 1)) return (P(cy, x) * 3 + P(cy > 0 ? cy - 1 : 0, x) + 1) >> 2;
    return (P(cy, x) * 3 + P(cy + 1 < dh ? cy + 1 : dh - 1, x) + 2) >> 2;
  }
  // h2v2
  const int cx = x >> 1, cy = y >> 1;
  if (dw <= 2) return P(cy, cx);
  const int ny = (y & 1) ? (cy + 1 < dh ? cy + 1 : dh - 1) : (cy > 0 ? cy - 1 : 0);
  auto colsum = [&](int xx) { return P(cy, xx) * 3 + P(ny, xx); };
  const int t = colsum(cx);
  if (!(x & 1)) return cx == 0 ? (t * 4 + 8) >> 4 : (t * 3 + colsum(cx - 1) + 8) >> 4;
  return cx == dw - 1 ? (t * 4 + 7) >> 4 : (t * 3 + colsum(cx + 1) + 7) >> 4;
}

__host__ __device__ inline uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }

// jdcolor.c ycc_rgb_convert (SCALEBITS 16) for one pixel, stored B, G, R
__host__ __device__ inline void jpeg_color_pixel(const JpegDesc& d, const uint8_t* const* pl, int x, int y,
                                                 uint8_t* bgr) {
  const int Y = pl[0][(int64_t)y * d.pw[0] + x];
  if (d.ncomp == 1) { bgr[0] = bgr[1] = bgr[2] = (uint8_t)Y; return; }
  const int cb = chroma_at(d, pl[1], 1, x, y) - 128, cr = chroma_at(d, pl[2], 2, x, y) - 128;
  const int half = 1 << 15;
  const int cr_r = (91881 * cr + half) >> 16, cb_b = (116130 * cb + half) >> 16;
  const int g = (-46802 * cr + -22554 * cb + half) >> 16;
  bgr[0] = clamp255(Y + cb_b);
  bgr[1] = clamp255(Y + g);
  bgr[2] = clamp255(Y + cr_r);
}

__host__ __device__ inline void jpeg_color_row(const JpegDesc& d, const uint8_t* const* pl, int y, uint8_t* row) {
  for (int x = 0; x < d.W; ++x) jpeg_color_pixel(d, pl, x, y, row + 3 * x);
}

// ------------------------------------------------------------------ kernels
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* total) {
  __shared__ uint32_t warp_tot[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_tot[wid] = x;
  __syncthreads();
  if (wid == 0) {
    uint32_t t = lane < nw ? warp_tot[lane] : 0u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += y;
    }
    warp_tot[lane] = t;
  }
  __syncthreads();
  const uint32_t before = (wid ? warp_tot[wid - 1] : 0u) + x - v;
  *total = warp_tot[nw - 1];
  __syncthreads();
  return before;
}

// kind of entropy byte i: 0 drop, 1 keep, 2 RSTn (its 0xFF), 3 end of the scan
__device__ __forceinline__ int byte_kind(const uint8_t* s, int64_t n, int64_t i, int* rst) {
  if (i >= n) return 3;
  const int x = s[i];
  if (x == 0xFF) {
    if (i + 1 >= n) return 3;
    const int nx = s[i + 1];
    if (nx == 0x00) return 1;
    if (nx == 0xFF) return 0;
    if (nx >= 0xD0 && nx <= 0xD7) { *rst = nx - 0xD0; return 2; }
    return 3;
  }
  if (i > 0 && s[i - 1] == 0xFF) return 0;     // stuffed 0x00 or the RSTn byte
  return 1;
}

__global__ void __launch_bounds__(kUnstuffThreads)
jpeg_unstuff_kernel(const uint8_t* __restrict__ blob_base, const int64_t* __restrict__ blob_off,
                    const JpegDesc* __restrict__ descs, uint8_t* __restrict__ ws, int32_t* __restrict__ status) {
  const int b = blockIdx.x;
  const JpegDesc& d = descs[b];
  if (d.status != JPEG_OK) return;
  const uint8_t* src = blob_base + blob_off[b] + d.ent_off;
  const int64_t n = d.ent_len;
  uint8_t* dst = ws + d.ws_stream;
  int32_t* hdr = reinterpret_cast<int32_t*>(ws + d.ws_seg);
  int32_t* seg = hdr + kSegHdr;
  int32_t* sub = seg + d.nseg + 1;
  __shared__ int64_t s_stop;
  __shared__ int s_bad;
  if (threadIdx.x == 0) { s_bad = 0; status[b] = JPEG_OK; }
  uint32_t kept = 0, rsts = 0;
  constexpr int CH = kUnstuffThreads * kUnstuffItems;
  for (int64_t c0 = 0;; c0 += CH) {
    if (threadIdx.x == 0) s_stop = INT64_MAX;
    __syncthreads();
    int kind[kUnstuffItems], rn[kUnstuffItems];
    const int64_t i0 = c0 + (int64_t)threadIdx.x * kUnstuffItems;
    for (int e = 0; e < kUnstuffItems; ++e) {
      rn[e] = 0;
      kind[e] = byte_kind(src, n, i0 + e, &rn[e]);
      if (kind[e] == 3) atomicMin((unsigned long long*)&s_stop, (unsigned long long)(i0 + e));
    }
    __syncthreads();
    const int64_t stop = s_stop;
    uint32_t cnt = 0;
    for (int e = 0; e < kUnstuffItems; ++e) {
      if (i0 + e >= stop) kind[e] = 0;
      cnt += kind[e] == 1 ? 1u : kind[e] == 2 ? (1u << 16) : 0u;
    }
    uint32_t tot;
    const uint32_t pre = block_excl_scan(cnt, &tot);
    uint32_t ok = kept + (pre & 0xffff), orr = rsts + (pre >> 16);
    for (int e = 0; e < kUnstuffItems; ++e) {
      if (kind[e] == 1) {
        dst[ok++] = src[i0 + e];
      } else if (kind[e] == 2) {
        ++orr;
        if ((int)orr < d.nseg) seg[orr] = (int32_t)ok;
        if (rn[e] != (int)((orr - 1) & 7)) s_bad = 1;
      }
    }
    kept += tot & 0xffff;
    rsts += tot >> 16;
    if (stop != INT64_MAX) break;
  }
  __syncthreads();
  if (threadIdx.x < 16) dst[kept + threadIdx.x] = 0;
  const bool bad = s_bad || rsts + 1 != (uint32_t)d.nseg;
  if (threadIdx.x == 0) {
    hdr[0] = (int32_t)kept;
    hdr[1] = (int32_t)(rsts + 1);
    hdr[2] = bad ? 1 : 0;
    seg[0] = 0;
    seg[d.nseg] = (int32_t)kept;
    if (bad) status[b] = JPEG_MALFORMED;
  }
  if (bad) return;
  __syncthreads();
  // first subsequence of every segment
  uint32_t base = 0;
  for (int s0 = 0; s0 <= d.nseg; s0 += kUnstuffThreads) {
    const int s = s0 + threadIdx.x;
    const uint32_t v = s < d.nseg ? (uint32_t)nsub_of(seg[s + 1] - seg[s], kJpegSubBits) : 0u;
    uint32_t tot;
    const uint32_t pre = block_excl_scan(v, &tot);
    if (s <= d.nseg) sub[s] = (int32_t)(base + pre);
    base += tot;
  }
}

struct ImgView {
  const JpegDesc* d;
  const uint8_t* bits;
  const int32_t *hdr, *seg, *sub;
  JpegEntry* ent;
  JpegPrefix* pb;
};

__device__ __forceinline__ bool img_view(const JpegDesc* descs, uint8_t* ws, int b, ImgView& v) {
  v.d = &descs[b];
  if (v.d->status != JPEG_OK) return false;
  v.hdr = reinterpret_cast<const int32_t*>(ws + v.d->ws_seg);
  if (v.hdr[2]) return false;
  v.seg = v.hdr + kSegHdr;
  v.sub = v.seg + v.d->nseg + 1;
  v.bits = ws + v.d->ws_stream;
  v.ent = reinterpret_cast<JpegEntry*>(ws + v.d->ws_ent);
  v.pb = reinterpret_cast<JpegPrefix*>(ws + v.d->ws_pb);
  return true;
}

__device__ __forceinline__ JpegEntry ld_entry(const JpegEntry* e) {
  const volatile JpegEntry* v = e;
  JpegEntry r;
  r.st = v->st;
  r.dc[0] = v->dc[0];
  r.dc[1] = v->dc[1];
  r.dc[2] = v->dc[2];
  r.pad = 0;
  return r;
}
__device__ __forceinline__ void st_entry(JpegEntry* e, const JpegEntry& r) {
  volatile JpegEntry* v = e;
  v->dc[0] = r.dc[0];
  v->dc[1] = r.dc[1];
  v->dc[2] = r.dc[2];
  v->st = r.st;
}

__global__ void __launch_bounds__(128)
jpeg_phase_a_kernel(const JpegDesc* __restrict__ descs, uint8_t* __restrict__ ws) {
  ImgView v;
  if (!img_view(descs, ws, blockIdx.y, v)) return;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= v.sub[v.d->nseg]) return;
  const SubGeom g = sub_geom(v.seg, v.sub, v.d->nseg, j, kJpegSubBits);
  v.ent[j] = jpeg_sub_phase_a(*v.d, v.bits, g);
}

// round r: thread j carries its exit state into subsequence j+1 and walks on while it differs
__global__ void __launch_bounds__(128)
jpeg_sync_kernel(const JpegDesc* __restrict__ descs, uint8_t* __restrict__ ws, int r) {
  int32_t* flags = reinterpret_cast<int32_t*>(ws + 64);
  if (r > 0 && *(volatile int32_t*)&flags[r - 1] == 0) return;
  ImgView v;
  if (!img_view(descs, ws, blockIdx.y, v)) return;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= v.sub[v.d->nseg]) return;
  const SubGeom g = sub_geom(v.seg, v.sub, v.d->nseg, j, kJpegSubBits);
  JpegEntry cur = ld_entry(&v.ent[j]);
  for (int q = j + 1; q < g.last; ++q) {
    const SubGeom gq = sub_geom(v.seg, v.sub, v.d->nseg, q, kJpegSubBits);
    const JpegEntry e = jpeg_sub_entry(*v.d, v.bits, gq, st_clear_n(cur.st));
    if (state_eq(e.st, ld_entry(&v.ent[q]).st)) break;
    st_entry(&v.ent[q], e);
    *(volatile int32_t*)&flags[r] = 1;
    cur = e;
  }
}

// after kJpegRounds rounds that all changed something: one sequential walk per segment
__global__ void __launch_bounds__(128)
jpeg_sync_walk_kernel(const JpegDesc* __restrict__ descs, uint8_t* __restrict__ ws) {
  int32_t* flags = reinterpret_cast<int32_t*>(ws + 64);
  if (flags[kJpegRounds - 1] == 0) return;
  ImgView v;
  if (!img_view(descs, ws, blockIdx.y, v)) return;
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= v.d->nseg) return;
  if (s == 0) flags[kJpegRounds] = 1;
  uint64_t cur = 0;
  for (int q = v.sub[s]; q < v.sub[s + 1]; ++q) {
    const SubGeom g = sub_geom(v.seg, v.sub, v.d->nseg, q, kJpegSubBits);
    const JpegEntry e = q == v.sub[s] ? jpeg_sub_phase_a(*v.d, v.bits, g)
                                      : jpeg_sub_entry(*v.d, v.bits, g, st_clear_n(cur));
    v.ent[q] = e;
    cur = e.st;
  }
}

// blocks and DC sums of every subsequence from its exact start state, into pb
__global__ void __launch_bounds__(128)
jpeg_count_kernel(const JpegDesc* __restrict__ descs, uint8_t* __restrict__ ws) {
  ImgView v;
  if (!img_view(descs, ws, blockIdx.y, v)) return;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= v.sub[v.d->nseg]) return;
  const SubGeom g = sub_geom(v.seg, v.sub, v.d->nseg, j, kJpegSubBits);
  const uint64_t start = j == g.first ? st_make(g.start, 0, 0, 0, 0) : st_clear_n(v.ent[j - 1].st);
  v.pb[j] = jpeg_sub_count(*v.d, v.bits, g, start);
}

// phase B: one warp per segment; exclusive scan of blocks and DC sums (in place); a segment that holds
// fewer blocks than its MCUs need ended early (malformed)
__global__ void __launch_bounds__(256)
jpeg_phase_b_kernel(const JpegDesc* __restrict__ descs, uint8_t* __restrict__ ws, int32_t* __restrict__ status) {
  ImgView v;
  if (!img_view(descs, ws, blockIdx.y, v)) return;
  const int s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (s >= v.d->nseg) return;
  int32_t acc[4] = {0, 0, 0, 0};
  for (int q0 = v.sub[s]; q0 < v.sub[s + 1]; q0 += 32) {
    const int q = q0 + lane;
    int32_t x[4] = {0, 0, 0, 0};
    if (q < v.sub[s + 1]) {
      const JpegPrefix c = v.pb[q];
      x[0] = c.first;
      x[1] = c.dc[0];
      x[2] = c.dc[1];
      x[3] = c.dc[2];
    }
    int32_t inc[4];
    for (int t = 0; t < 4; ++t) {
      inc[t] = x[t];
      for (int o = 1; o < 32; o <<= 1) {
        const int32_t y = __shfl_up_sync(0xffffffffu, inc[t], o);
        if (lane >= o) inc[t] += y;
      }
    }
    if (q < v.sub[s + 1]) {
      JpegPrefix p;
      p.first = acc[0] + inc[0] - x[0];
      for (int t = 0; t < 3; ++t) p.dc[t] = acc[t + 1] + inc[t + 1] - x[t + 1];
      v.pb[q] = p;
    }
    for (int t = 0; t < 4; ++t) acc[t] += __shfl_sync(0xffffffffu, inc[t], 31);
  }
  if (lane == 0 && acc[0] < seg_blocks(*v.d, s)) status[blockIdx.y] = JPEG_MALFORMED;
}

__global__ void __launch_bounds__(128)
jpeg_phase_c_kernel(const JpegDesc* __restrict__ descs, uint8_t* __restrict__ ws,
                    const int32_t* __restrict__ status) {
  ImgView v;
  if (status[blockIdx.y] != JPEG_OK || !img_view(descs, ws, blockIdx.y, v)) return;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= v.sub[v.d->nseg]) return;
  const SubGeom g = sub_geom(v.seg, v.sub, v.d->nseg, j, kJpegSubBits);
  const uint64_t start = j == g.first ? st_make(g.start, 0, 0, 0, 0) : st_clear_n(v.ent[j - 1].st);
  jpeg_sub_phase_c(*v.d, v.bits, g, start, v.pb[j], reinterpret_cast<int16_t*>(ws + v.d->ws_coef),
                   seg_first_block(*v.d, g.seg), seg_blocks(*v.d, g.seg));
}

__global__ void __launch_bounds__(128)
jpeg_idct_kernel(const JpegDesc* __restrict__ descs, uint8_t* __restrict__ ws, const int32_t* __restrict__ status) {
  const int b = blockIdx.y;
  const JpegDesc& d = descs[b];
  if (d.status != JPEG_OK || status[b] != JPEG_OK) return;
  const int64_t blk = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (blk >= d.nblocks) return;
  int c;
  int64_t off;
  block_place(d, blk, &c, &off);
  jpeg_idct_block(reinterpret_cast<const int16_t*>(ws + d.ws_coef) + blk * 64, d.qt[c], ws + d.ws_plane[c] + off,
                  d.pw[c]);
}

__global__ void __launch_bounds__(128)
jpeg_color_kernel(const JpegDesc* __restrict__ descs, const uint8_t* __restrict__ ws,
                  const int32_t* __restrict__ status, uint8_t* __restrict__ out_base,
                  const int64_t* __restrict__ out_off, const int32_t* __restrict__ out_hwp) {
  const int b = blockIdx.z;
  const JpegDesc& d = descs[b];
  if (d.status != JPEG_OK || status[b] != JPEG_OK) return;
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= d.W || y >= d.H) return;
  const uint8_t* pl[3] = {ws + d.ws_plane[0], ws + d.ws_plane[1], ws + d.ws_plane[2]};
  jpeg_color_pixel(d, pl, x, y, out_base + out_off[b] + (int64_t)y * out_hwp[b * 3 + 2] + 3 * x);
}

// ------------------------------------------------------------------ 6. lossless transcode
// The coefficients of stages 2-3 coded again with a restart interval of R MCUs: every interval
// starts from DC predictors 0 and a byte boundary, so a decoder can start at any RSTn in an exact
// state.  Every Huffman table of the scan is regenerated from the new symbol counts (Annex K.2);
// the coefficients, and so every decoder's pixels, stay exactly those of the source.
constexpr int kTcDcBins = 16;                          // DC categories 0..15
constexpr int kTcBins = 2 * kTcDcBins + 2 * 256;       // one interval: DC slots 0, 1 and AC slots 2, 3
constexpr int kTcDhtMax = 4 + 4 * (17 + 256) + 6;      // new DHT segment + DRI segment, at most

struct TcDesc {                // per image, from epb_jpeg_transcode_plan
  int32_t ri, nint;            // restart interval (MCUs) and number of intervals; 0 when not transcoded
  int64_t ws_hist, ws_len, ws_off, ws_tab;
};
static_assert(sizeof(TcDesc) <= EPB_JPEG_TC_DESC_BYTES, "transcode descriptor size");

struct TcLen {                 // one interval: coded bits (-1: a category no table can code), stuffed bytes
  int32_t bits, bytes;
};

struct TcTable {               // encoder form of one regenerated table; size 0: symbol absent
  uint16_t code[256];
  uint8_t size[256];
};

struct TcInfo {                // per image, read back by the host (layout in include/epb.h)
  int32_t status, ri;
  int64_t bytes, off, hdr_bytes;
  uint8_t bits[4][17];         // DHT lists of slots DC 0, DC 1, AC 0, AC 1
  uint8_t val[4][256];
};
static_assert(sizeof(TcInfo) == EPB_JPEG_TC_INFO_BYTES, "transcode info size");

__host__ __device__ inline int tc_cat(int v) {
  const uint32_t a = (uint32_t)(v < 0 ? -v : v);
#ifdef __CUDA_ARCH__
  return a ? 32 - __clz(a) : 0;
#else
  return a ? 32 - __builtin_clz(a) : 0;
#endif
}
// the extra bits of value v of category s (F.1.2.1: negative values as v - 1, low s bits)
__host__ __device__ inline uint32_t tc_extra(int v, int s) {
  return (uint32_t)(v < 0 ? v + (1 << s) - 1 : v) & ((1u << s) - 1);
}

// Interval i of an image: MCUs [i R, min((i + 1) R, MCUs)) in the decoder's block order
// (slot_comp), DC predictors reset to 0, each symbol handed to sink.sym(table slot, symbol,
// extra-bit count, extra bits): the DC category, then AC run/size with ZRL and EOB.  Returns
// false on a category above 15, which a Huffman table of the scan cannot code.
template <class Sink>
__host__ __device__ inline bool tc_walk(const JpegDesc& d, const int16_t* coef, int ri, int i, Sink& sink) {
  const int64_t mcus = (int64_t)d.mcux * d.mcuy;
  const int64_t m0 = (int64_t)i * ri, m1 = m0 + ri < mcus ? m0 + ri : mcus;
  int pred[3] = {0, 0, 0};
  for (int64_t m = m0; m < m1; ++m) {
    for (int slot = 0; slot < d.bpm; ++slot) {
      const int comp = d.slot_comp[slot];
      const int16_t* blk = coef + (m * d.bpm + slot) * 64;
      const int diff = blk[0] - pred[comp];
      pred[comp] = blk[0];
      const int cat = tc_cat(diff);
      if (cat > 15) return false;
      sink.sym(d.cdc[comp], cat, cat, tc_extra(diff, cat));
      int run = 0;
      for (int k = 1; k < 64; ++k) {
        const int v = blk[zigzag_natural(k)];
        if (!v) { ++run; continue; }
        for (; run >= 16; run -= 16) sink.sym(d.cac[comp], 0xF0, 0, 0u);
        const int s = tc_cat(v);
        if (s > 15) return false;
        sink.sym(d.cac[comp], (run << 4) | s, s, tc_extra(v, s));
        run = 0;
      }
      if (run) sink.sym(d.cac[comp], 0x00, 0, 0u);
    }
  }
  return true;
}

struct TcHist {                // symbol counts of one interval, kTcBins
  int32_t* h;
  __host__ __device__ void sym(int slot, int s, int, uint32_t) {
    ++h[slot < 2 ? slot * kTcDcBins + s : 2 * kTcDcBins + (slot - 2) * 256 + s];
  }
};

// Bit writer of one interval: codes MSB first, then 1-bits to the next byte; every 0xFF is
// followed by a stuffed 0x00.  With out null it only counts; otherwise it stores at most cap
// bytes and sets over when it would store more.
struct TcWriter {
  const TcTable* tab;
  uint8_t* out;
  int64_t cap;
  uint64_t acc = 0;
  int nacc = 0;
  int64_t bits = 0, bytes = 0;
  bool over = false;
  __host__ __device__ void emit(int v) {
    if (out) {
      if (bytes < cap) out[bytes] = (uint8_t)v; else over = true;
    }
    ++bytes;
  }
  __host__ __device__ void put(uint32_t v, int n) {
    acc = (acc << n) | v;
    nacc += n;
    while (nacc >= 8) {
      nacc -= 8;
      const int x = (int)((acc >> nacc) & 255);
      emit(x);
      if (x == 0xFF) emit(0);
    }
  }
  __host__ __device__ void sym(int slot, int s, int n, uint32_t v) {
    put(tab[slot].code[s], tab[slot].size[s]);
    bits += tab[slot].size[s] + n;
    if (n) put(v, n);
  }
  __host__ __device__ void finish() {
    if (nacc) put((1u << (8 - nacc)) - 1, 8 - nacc);
  }
};

struct TcWork {                // scratch of huff_optimal
  int64_t freq[257];
  int16_t sym[257], size[257], next[257];
  int32_t nbits[258];
};

// Optimal table of Annex K.2 (figures K.1 to K.4) for the symbols of count > 0 among count[0..n),
// plus a reserved symbol 256 of count 1 so that no code is all 1-bits.  Tie rule: of equal counts
// the larger symbol value is taken first (the reserved symbol before every real one).  Lengths
// are limited to 16 by K.3, and K.3's last step drops the reserved symbol's code.  Writes
// bits[0..16] (bits[0] = 0) and val (symbols by unlimited code length, then by value); returns
// the number of symbols.
__host__ __device__ inline int huff_optimal(const int64_t* count, int n, TcWork& w, uint8_t* bits, uint8_t* val) {
  int m = 0;
  for (int s = 0; s < n; ++s)
    if (count[s] > 0) { w.sym[m] = (int16_t)s; w.freq[m] = count[s]; ++m; }
  for (int l = 0; l <= 16; ++l) bits[l] = 0;
  if (m == 0) return 0;
  w.sym[m] = 256;
  w.freq[m] = 1;
  ++m;
  for (int i = 0; i < m; ++i) { w.size[i] = 0; w.next[i] = -1; }
  for (;;) {                                   // K.1: merge the two least counts
    int v1 = -1, v2 = -1;
    for (int i = m - 1; i >= 0; --i) {         // descending: the first of equal counts is the larger symbol
      const int64_t f = w.freq[i];
      if (f <= 0) continue;
      if (v1 < 0 || f < w.freq[v1]) { v2 = v1; v1 = i; }
      else if (v2 < 0 || f < w.freq[v2]) v2 = i;
    }
    if (v2 < 0) break;
    w.freq[v1] += w.freq[v2];
    w.freq[v2] = 0;
    ++w.size[v1];
    while (w.next[v1] >= 0) { v1 = w.next[v1]; ++w.size[v1]; }
    w.next[v1] = (int16_t)v2;
    ++w.size[v2];
    while (w.next[v2] >= 0) { v2 = w.next[v2]; ++w.size[v2]; }
  }
  for (int l = 0; l < 258; ++l) w.nbits[l] = 0;          // K.2
  int lmax = 0;
  for (int i = 0; i < m; ++i) {
    ++w.nbits[w.size[i]];
    lmax = w.size[i] > lmax ? w.size[i] : lmax;
  }
  for (int i = lmax; i > 16;) {                           // K.3
    if (w.nbits[i] > 0) {
      int j = i - 2;
      while (w.nbits[j] == 0) --j;
      w.nbits[i] -= 2;
      w.nbits[i - 1] += 1;
      w.nbits[j + 1] += 2;
      w.nbits[j] -= 1;
    } else {
      --i;
    }
  }
  int i = 16;
  while (w.nbits[i] == 0) --i;
  w.nbits[i] -= 1;
  for (int l = 1; l <= 16; ++l) bits[l] = (uint8_t)w.nbits[l];
  int k = 0;                                              // K.4
  for (int l = 1; l <= lmax; ++l)
    for (int q = 0; q < m; ++q)
      if (w.size[q] == l && w.sym[q] != 256) val[k++] = (uint8_t)w.sym[q];
  return k;
}

// encoder codes of a table (C.2 / C.3); every other symbol gets size 0
__host__ __device__ inline void huff_codes(const uint8_t* bits, const uint8_t* val, TcTable& t) {
  for (int s = 0; s < 256; ++s) { t.code[s] = 0; t.size[s] = 0; }
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    for (int q = 0; q < bits[l]; ++q, ++code, ++k) {
      t.code[val[k]] = (uint16_t)code;
      t.size[val[k]] = (uint8_t)l;
    }
    code <<= 1;
  }
}

// length pass of interval i: coded bits and stuffed bytes, the RSTn after it included
__host__ __device__ inline TcLen tc_interval_len(const JpegDesc& d, const int16_t* coef, const TcTable* tab, int ri,
                                                 int nint, int i) {
  TcWriter w{tab, nullptr, 0};
  tc_walk(d, coef, ri, i, w);
  w.finish();
  TcLen r;
  r.bits = (int32_t)w.bits;
  r.bytes = (int32_t)w.bytes + (i + 1 < nint ? 2 : 0);
  return r;
}

// write pass of interval i into out[0, len.bytes): its bytes, then RSTn (n = i mod 8) unless it is
// the last; false when the interval does not come out at len.bytes
__host__ __device__ inline bool tc_interval_write(const JpegDesc& d, const int16_t* coef, const TcTable* tab, int ri,
                                                  int nint, int i, TcLen len, uint8_t* out) {
  const int rst = i + 1 < nint ? 2 : 0;
  TcWriter w{tab, out, (int64_t)len.bytes - rst};
  tc_walk(d, coef, ri, i, w);
  w.finish();
  if (w.over || w.bytes + rst != len.bytes) return false;
  if (rst) {
    out[w.bytes] = 0xFF;
    out[w.bytes + 1] = (uint8_t)(0xD0 + (i & 7));
  }
  return true;
}

// symbol pass: one thread per interval, its histogram
__global__ void __launch_bounds__(128)
jpeg_tc_symbols_kernel(const JpegDesc* __restrict__ descs, const TcDesc* __restrict__ tdesc, uint8_t* __restrict__ ws,
                       const int32_t* __restrict__ status) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const JpegDesc& d = descs[b];
  const TcDesc& t = tdesc[b];
  if (d.status != JPEG_OK || status[b] != JPEG_OK || i >= t.nint) return;
  int32_t* h = reinterpret_cast<int32_t*>(ws + t.ws_hist) + (int64_t)i * kTcBins;
  for (int k = 0; k < kTcBins; ++k) h[k] = 0;
  TcHist sink{h};
  const bool ok = tc_walk(d, reinterpret_cast<const int16_t*>(ws + d.ws_coef), t.ri, i, sink);
  reinterpret_cast<TcLen*>(ws + t.ws_len)[i].bits = ok ? 0 : -1;
}

// one block per image: the interval histograms summed in interval order, one table per slot in use
__global__ void __launch_bounds__(256)
jpeg_tc_tables_kernel(const JpegDesc* __restrict__ descs, const TcDesc* __restrict__ tdesc, uint8_t* __restrict__ ws,
                      int32_t* __restrict__ status, TcInfo* __restrict__ info) {
  const int b = blockIdx.x;
  const JpegDesc& d = descs[b];
  const TcDesc& t = tdesc[b];
  if (d.status != JPEG_OK || status[b] != JPEG_OK) return;
  __shared__ int64_t cnt[kTcBins];
  __shared__ TcWork work[4];
  const TcLen* len = reinterpret_cast<const TcLen*>(ws + t.ws_len);
  int bad = 0;
  for (int q = threadIdx.x; q < t.nint; q += blockDim.x) bad |= len[q].bits < 0;
  if (__syncthreads_or(bad)) {
    if (threadIdx.x == 0) status[b] = JPEG_UNSUPPORTED;
    return;
  }
  const int32_t* h = reinterpret_cast<const int32_t*>(ws + t.ws_hist);
  for (int k = threadIdx.x; k < kTcBins; k += blockDim.x) {
    int64_t s = 0;
    for (int q = 0; q < t.nint; ++q) s += h[(int64_t)q * kTcBins + k];
    cnt[k] = s;
  }
  __syncthreads();
  const int slot = threadIdx.x >> 5;
  TcInfo& o = info[b];
  TcTable* tab = reinterpret_cast<TcTable*>(ws + t.ws_tab);
  if (slot < 4 && (threadIdx.x & 31) == 0) {           // one lane per table: the four run side by side
    const int64_t* c = slot < 2 ? cnt + slot * kTcDcBins : cnt + 2 * kTcDcBins + (slot - 2) * 256;
    huff_optimal(c, slot < 2 ? kTcDcBins : 256, work[slot], o.bits[slot], o.val[slot]);
    huff_codes(o.bits[slot], o.val[slot], tab[slot]);
  }
}

// length pass: one thread per interval
__global__ void __launch_bounds__(128)
jpeg_tc_length_kernel(const JpegDesc* __restrict__ descs, const TcDesc* __restrict__ tdesc, uint8_t* __restrict__ ws,
                      const int32_t* __restrict__ status) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const JpegDesc& d = descs[b];
  const TcDesc& t = tdesc[b];
  if (d.status != JPEG_OK || status[b] != JPEG_OK || i >= t.nint) return;
  reinterpret_cast<TcLen*>(ws + t.ws_len)[i] =
      tc_interval_len(d, reinterpret_cast<const int16_t*>(ws + d.ws_coef), reinterpret_cast<const TcTable*>(ws + t.ws_tab),
                      t.ri, t.nint, i);
}

// one block per image: exclusive scan of the stuffed interval lengths -> byte offsets, and the total
__global__ void __launch_bounds__(512)
jpeg_tc_scan_kernel(const JpegDesc* __restrict__ descs, const TcDesc* __restrict__ tdesc, uint8_t* __restrict__ ws,
                    const int32_t* __restrict__ status, TcInfo* __restrict__ info) {
  const int b = blockIdx.x;
  const JpegDesc& d = descs[b];
  const TcDesc& t = tdesc[b];
  if (d.status != JPEG_OK || status[b] != JPEG_OK) return;
  const TcLen* len = reinterpret_cast<const TcLen*>(ws + t.ws_len);
  int64_t* off = reinterpret_cast<int64_t*>(ws + t.ws_off);
  int64_t base = 0;
  for (int q0 = 0; q0 < t.nint; q0 += blockDim.x) {
    const int q = q0 + threadIdx.x;
    const uint32_t v = q < t.nint ? (uint32_t)len[q].bytes : 0u;
    uint32_t tot;
    const uint32_t pre = block_excl_scan(v, &tot);
    if (q < t.nint) off[q] = base + pre;
    base += tot;
  }
  if (threadIdx.x == 0) info[b].bytes = base;
}

// one block: every image's final status and restart interval, then its output offset, a 64-bit
// running sum over the images in order (one thread: B is at most 65535)
__global__ void __launch_bounds__(512)
jpeg_tc_finish_kernel(const JpegDesc* __restrict__ descs, const TcDesc* __restrict__ tdesc, const int32_t* __restrict__ status,
                      TcInfo* __restrict__ info, int B) {
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const int s = descs[b].status != JPEG_OK ? descs[b].status : status[b];
    info[b].status = s;
    info[b].ri = s == JPEG_OK ? tdesc[b].ri : 0;
    if (s != JPEG_OK) info[b].bytes = 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t base = 0;
    for (int b = 0; b < B; ++b) {
      info[b].off = base;
      base += info[b].bytes;
    }
  }
}

// write pass: one thread per interval, into out_base at info.off + its offset, inside out_bytes.
// An interval whose offsets fail the checks, or that does not come out at its counted length,
// sets *failed (the host reads it back and fails the call).
__global__ void __launch_bounds__(128)
jpeg_tc_write_kernel(const JpegDesc* __restrict__ descs, const TcDesc* __restrict__ tdesc, const uint8_t* __restrict__ ws,
                     const int32_t* __restrict__ status, const TcInfo* __restrict__ info, uint8_t* __restrict__ out_base,
                     int64_t out_bytes, int32_t* __restrict__ failed) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const JpegDesc& d = descs[b];
  const TcDesc& t = tdesc[b];
  if (d.status != JPEG_OK || status[b] != JPEG_OK || i >= t.nint) return;
  const TcLen len = reinterpret_cast<const TcLen*>(ws + t.ws_len)[i];
  const int64_t rel = reinterpret_cast<const int64_t*>(ws + t.ws_off)[i], img = info[b].off;
  if (rel < 0 || len.bytes < 0 || rel + len.bytes > info[b].bytes || img < 0 || img + info[b].bytes > out_bytes ||
      !tc_interval_write(d, reinterpret_cast<const int16_t*>(ws + d.ws_coef),
                         reinterpret_cast<const TcTable*>(ws + t.ws_tab), t.ri, t.nint, i, len, out_base + img + rel))
    *failed = 1;
}

// R = 0 (auto): the largest R whose mean interval, entropy bits / MCUs * R, is at most 3/4 of
// kJpegSubBits.  The entropy bits are those of the bytes from SOS to the end of the blob.
inline int tc_auto_interval(const JpegDesc& d) {
  const int64_t mcus = (int64_t)d.mcux * d.mcuy, bits = d.ent_len * 8 > 0 ? d.ent_len * 8 : 1;
  const int64_t r = (int64_t)kJpegSubBits * 3 / 4 * mcus / bits;
  return (int)(r < 1 ? 1 : r > 65535 ? 65535 : r);
}

// The transcoded file's header: SOI; every segment of the source before SOS except DHT and DRI,
// verbatim and in order; one DHT with the regenerated tables under the source's table ids (the
// SOS selectors are kept); DRI(ri); the source's SOS segment.  b must have parsed OK.
// Returns the bytes written, or -1 when cap is short.
inline int64_t jpeg_tc_header(const uint8_t* b, int ri, const uint8_t (*bits)[17],
                              const uint8_t (*val)[256], uint8_t* out, int64_t cap) {
  int64_t n = 0, i = 2;
  auto put = [&](const uint8_t* p, int64_t k) -> bool {
    if (n + k > cap) return false;
    memcpy(out + n, p, (size_t)k);
    n += k;
    return true;
  };
  const uint8_t soi[2] = {0xFF, 0xD8};
  if (!put(soi, 2)) return -1;
  for (;;) {
    while (b[i] == 0xFF) ++i;
    const int m = b[i++];
    const int len = rd16(b + i);
    const uint8_t mk[2] = {0xFF, (uint8_t)m};
    if (m == 0xDA) {
      const uint8_t* s = b + i + 2;
      int td[2] = {-1, -1}, ta[2] = {-1, -1};           // table id of each slot, first use first (as the parser)
      for (int q = 0; q < s[0]; ++q) {
        const int x = s[2 + 2 * q] >> 4, y = s[2 + 2 * q] & 15;
        if (td[0] != x && td[1] != x) td[td[0] < 0 ? 0 : 1] = x;
        if (ta[0] != y && ta[1] != y) ta[ta[0] < 0 ? 0 : 1] = y;
      }
      uint8_t dht[kTcDhtMax];
      int k = 4;
      for (int slot = 0; slot < 4; ++slot) {
        const int id = slot < 2 ? td[slot] : ta[slot - 2];
        if (id < 0) continue;
        int cnt = 0;
        dht[k++] = (uint8_t)((slot < 2 ? 0x00 : 0x10) | id);
        for (int l = 1; l <= 16; ++l) { dht[k++] = bits[slot][l]; cnt += bits[slot][l]; }
        for (int q = 0; q < cnt; ++q) dht[k++] = val[slot][q];
      }
      dht[0] = 0xFF;
      dht[1] = 0xC4;
      dht[2] = (uint8_t)((k - 2) >> 8);
      dht[3] = (uint8_t)(k - 2);
      const uint8_t dri[6] = {0xFF, 0xDD, 0x00, 0x04, (uint8_t)(ri >> 8), (uint8_t)ri};
      if (!put(dht, k) || !put(dri, 6) || !put(mk, 2) || !put(b + i, len)) return -1;
      return n;
    }
    if (m != 0xC4 && m != 0xDD && (!put(mk, 2) || !put(b + i, len))) return -1;
    i += len;
  }
}

}  // namespace

extern "C" __attribute__((visibility("default"))) int epb_jpeg_parse(
    const uint8_t* const* blobs_host, const int64_t* lens_host, int B, void* desc_host, int32_t* status_host,
    int32_t* hw_host, int64_t* out_off_host, int64_t* plan_host) {
  EPB_CHECK_ARG(B >= 0 && B <= 65535 && (B == 0 || (blobs_host && lens_host && desc_host && status_host && hw_host &&
                                                    out_off_host)) && plan_host);
  JpegDesc* d = static_cast<JpegDesc*>(desc_host);
  int64_t out = 0;
  int64_t mx[6] = {0, 0, 0, 0, 0, 0};
  for (int b = 0; b < B; ++b) {
    EPB_CHECK_ARG(lens_host[b] >= 0 && (blobs_host[b] || lens_host[b] == 0));
    status_host[b] = jpeg_parse_one(blobs_host[b], lens_host[b], kJpegSubBits, &d[b]);
    hw_host[2 * b] = d[b].H;
    hw_host[2 * b + 1] = d[b].W;
    out_off_host[b] = out;
    out = align16(out + (int64_t)d[b].H * d[b].W * 3);
    if (d[b].status != JPEG_OK) continue;
    const int64_t v[6] = {d[b].nsub_max, d[b].nseg, d[b].nblocks, d[b].H, d[b].W, 1};
    for (int k = 0; k < 5; ++k) mx[k] = v[k] > mx[k] ? v[k] : mx[k];
    mx[5] += 1;
  }
  plan_host[0] = jpeg_layout(d, B, plan_host + 8);
  plan_host[1] = out;
  for (int k = 0; k < 6; ++k) plan_host[2 + k] = mx[k];
  return EPB_OK;
}

namespace {

// Stages 2 and 3 of every image whose parse status is OK (event marks 0..3): the quantised
// coefficients, natural order with absolute DC, at ws + ws_coef; status[b] OK or MALFORMED.
// Shared by epb_jpeg_decode and epb_jpeg_transcode.
int jpeg_launch_coefs(const uint8_t* blob_base, const int64_t* blob_off, const JpegDesc* d, int B,
                      const int64_t* plan_host, uint8_t* w, int32_t* status, int32_t* stats,
                      void* const* events_host, cudaStream_t st) {
  auto mark = [&](int i) -> int {
    if (events_host) EPB_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(events_host[i]), st));
    return EPB_OK;
  };
  int rc;
  if ((rc = mark(0))) return rc;
  EPB_CUDA(cudaMemsetAsync(w, 0, 64 + 16 * kJpegRounds, st));
  jpeg_unstuff_kernel<<<B, kUnstuffThreads, 0, st>>>(blob_base, blob_off, d, w, status);
  EPB_LAUNCH_CHECK();
  if ((rc = mark(1))) return rc;
  const dim3 gsub((unsigned)((plan_host[2] + 127) / 128), B);
  const dim3 gseg((unsigned)((plan_host[3] + 127) / 128), B);
  jpeg_phase_a_kernel<<<gsub, 128, 0, st>>>(d, w);
  EPB_LAUNCH_CHECK();
  for (int r = 0; r < kJpegRounds; ++r) {
    jpeg_sync_kernel<<<gsub, 128, 0, st>>>(d, w, r);
    EPB_LAUNCH_CHECK();
  }
  jpeg_sync_walk_kernel<<<gseg, 128, 0, st>>>(d, w);
  EPB_LAUNCH_CHECK();
  if (stats) EPB_CUDA(cudaMemcpyAsync(stats, w + 64, 4 * (kJpegRounds + 1), cudaMemcpyDeviceToDevice, st));
  if ((rc = mark(2))) return rc;
  jpeg_count_kernel<<<gsub, 128, 0, st>>>(d, w);
  EPB_LAUNCH_CHECK();
  const dim3 gwarp((unsigned)((plan_host[3] * 32 + 255) / 256), B);
  jpeg_phase_b_kernel<<<gwarp, 256, 0, st>>>(d, w, status);
  EPB_LAUNCH_CHECK();
  // the coefficients of all images are one region (jpeg_layout): one memset
  if (plan_host[9] > plan_host[8])
    EPB_CUDA(cudaMemsetAsync(w + plan_host[8], 0, (size_t)(plan_host[9] - plan_host[8]), st));
  jpeg_phase_c_kernel<<<gsub, 128, 0, st>>>(d, w, status);
  EPB_LAUNCH_CHECK();
  return mark(3);
}

}  // namespace

extern "C" __attribute__((visibility("default"))) int epb_jpeg_decode(
    const uint8_t* blob_base, const int64_t* blob_off, const void* desc, int B, const int64_t* plan_host, void* ws,
    int64_t ws_bytes, uint8_t* out_base, const int64_t* out_off, const int32_t* out_hwp, int32_t* status,
    int32_t* stats, void* const* events_host, epb_stream_t stream) {
  EPB_CHECK_ARG(B >= 0 && B <= 65535 && plan_host);
  if (B == 0 || plan_host[7] == 0) return EPB_OK;
  EPB_CHECK_ARG(blob_base && blob_off && desc && ws && out_base && out_off && out_hwp && status);
  EPB_CHECK_ARG(ws_bytes >= plan_host[0]);
  EPB_CHECK_ARG(plan_host[2] < (1LL << 31) && plan_host[4] < (1LL << 37) && plan_host[5] <= 65535);
  const JpegDesc* d = static_cast<const JpegDesc*>(desc);
  uint8_t* w = static_cast<uint8_t*>(ws);
  cudaStream_t st = as_stream(stream);
  auto mark = [&](int i) -> int {
    if (events_host) EPB_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(events_host[i]), st));
    return EPB_OK;
  };
  int rc;
  if ((rc = jpeg_launch_coefs(blob_base, blob_off, d, B, plan_host, w, status, stats, events_host, st))) return rc;
  const dim3 gblk((unsigned)((plan_host[4] + 127) / 128), B);
  jpeg_idct_kernel<<<gblk, 128, 0, st>>>(d, w, status);
  EPB_LAUNCH_CHECK();
  if ((rc = mark(4))) return rc;
  const dim3 gpix((unsigned)((plan_host[6] + 127) / 128), (unsigned)plan_host[5], B);
  jpeg_color_kernel<<<gpix, 128, 0, st>>>(d, w, status, out_base, out_off, out_hwp);
  EPB_LAUNCH_CHECK();
  return mark(5);
}

extern "C" __attribute__((visibility("default"))) int epb_jpeg_transcode_plan(
    const void* desc_host, int B, const int32_t* interval_host, const int64_t* plan_host, void* tdesc_host,
    int64_t* tplan_host) {
  EPB_CHECK_ARG(B >= 0 && B <= 65535 && plan_host && tplan_host && (B == 0 || (desc_host && interval_host && tdesc_host)));
  const JpegDesc* d = static_cast<const JpegDesc*>(desc_host);
  TcDesc* t = static_cast<TcDesc*>(tdesc_host);
  int64_t o = align16(plan_host[0]);
  tplan_host[2] = o;
  o = align16(o + (int64_t)sizeof(TcInfo) * B) + 16;      // info records, then the write pass's failure word
  int64_t mx = 0;
  for (int b = 0; b < B; ++b) {
    EPB_CHECK_ARG(interval_host[b] >= 0 && interval_host[b] <= 65535);
    memset(&t[b], 0, sizeof(TcDesc));
    if (d[b].status != JPEG_OK) continue;
    const int64_t mcus = (int64_t)d[b].mcux * d[b].mcuy;
    t[b].ri = interval_host[b] ? interval_host[b] : tc_auto_interval(d[b]);
    const int64_t nint = (mcus + t[b].ri - 1) / t[b].ri;
    // every stuffed byte count, per interval and per image, must fit 32 bits: at most 31 bits per
    // symbol, 64 symbols per block, each byte stuffed, plus an RSTn per interval
    EPB_CHECK_ARG(d[b].nblocks * 64 * 31 / 8 * 2 + 2 * nint + 16 < (1LL << 31));
    t[b].nint = (int32_t)nint;
    t[b].ws_hist = o; o = align16(o + nint * kTcBins * 4);
    t[b].ws_len = o;  o = align16(o + nint * (int64_t)sizeof(TcLen));
    t[b].ws_off = o;  o = align16(o + nint * 8);
    t[b].ws_tab = o;  o = align16(o + 4 * (int64_t)sizeof(TcTable));
    mx = nint > mx ? nint : mx;
  }
  tplan_host[0] = o;
  tplan_host[1] = mx;
  tplan_host[3] = kTcDhtMax;
  return EPB_OK;
}

extern "C" __attribute__((visibility("default"))) int epb_jpeg_transcode(
    const uint8_t* blob_base, const int64_t* blob_off, const void* desc, const void* tdesc, int B,
    const int64_t* plan_host, const int64_t* tplan_host, void* ws, int64_t ws_bytes, int32_t* status,
    const uint8_t* const* blobs_host, void* info_host, uint8_t* hdr_host, const int64_t* hdr_off_host,
    uint8_t* out_base, int64_t out_bytes, epb_stream_t stream) {
  EPB_CHECK_ARG(B >= 0 && B <= 65535 && plan_host && tplan_host);
  if (B == 0) return EPB_OK;
  EPB_CHECK_ARG(blob_base && blob_off && desc && tdesc && ws && status && info_host);
  EPB_CHECK_ARG(ws_bytes >= tplan_host[0] && tplan_host[0] >= plan_host[0]);
  EPB_CHECK_ARG(plan_host[2] < (1LL << 31) && plan_host[5] <= 65535 && tplan_host[1] < (1LL << 31));
  const JpegDesc* d = static_cast<const JpegDesc*>(desc);
  const TcDesc* t = static_cast<const TcDesc*>(tdesc);
  uint8_t* w = static_cast<uint8_t*>(ws);
  TcInfo* info = reinterpret_cast<TcInfo*>(w + tplan_host[2]);
  TcInfo* ih = static_cast<TcInfo*>(info_host);
  cudaStream_t st = as_stream(stream);
  const dim3 gint((unsigned)((tplan_host[1] + 127) / 128), B);
  if (out_base) {                            // second call: the entropy data at the offsets read back
    for (int b = 0; b < B; ++b)
      EPB_CHECK_ARG(ih[b].status != JPEG_OK || (ih[b].off >= 0 && ih[b].bytes >= 0 && ih[b].off + ih[b].bytes <= out_bytes));
    if (tplan_host[1] == 0) return EPB_OK;
    int32_t* failed = reinterpret_cast<int32_t*>(w + align16(tplan_host[2] + (int64_t)sizeof(TcInfo) * B));
    int32_t failed_host = 0;
    EPB_CUDA(cudaMemsetAsync(failed, 0, 4, st));
    jpeg_tc_write_kernel<<<gint, 128, 0, st>>>(d, t, w, status, info, out_base, out_bytes, failed);
    EPB_LAUNCH_CHECK();
    EPB_CUDA(cudaMemcpyAsync(&failed_host, failed, 4, cudaMemcpyDeviceToHost, st));
    EPB_CUDA(cudaStreamSynchronize(st));
    if (failed_host) {
      epb_set_error("epb_jpeg_transcode: an interval's offsets or length disagree with the first call's (was the "
                    "workspace reused by another call, or the output smaller than the sizes read back?)");
      return EPB_EINVAL;
    }
    return EPB_OK;
  }
  EPB_CHECK_ARG(blobs_host && hdr_host && hdr_off_host);
  EPB_CUDA(cudaMemsetAsync(info, 0, sizeof(TcInfo) * B, st));
  int rc;
  if (plan_host[7] &&
      (rc = jpeg_launch_coefs(blob_base, blob_off, d, B, plan_host, w, status, nullptr, nullptr, st)))
    return rc;
  if (tplan_host[1]) {
    jpeg_tc_symbols_kernel<<<gint, 128, 0, st>>>(d, t, w, status);
    EPB_LAUNCH_CHECK();
    jpeg_tc_tables_kernel<<<B, 256, 0, st>>>(d, t, w, status, info);
    EPB_LAUNCH_CHECK();
    jpeg_tc_length_kernel<<<gint, 128, 0, st>>>(d, t, w, status);
    EPB_LAUNCH_CHECK();
    jpeg_tc_scan_kernel<<<B, 512, 0, st>>>(d, t, w, status, info);
    EPB_LAUNCH_CHECK();
  }
  jpeg_tc_finish_kernel<<<1, 512, 0, st>>>(d, t, status, info, B);
  EPB_LAUNCH_CHECK();
  EPB_CUDA(cudaMemcpyAsync(ih, info, sizeof(TcInfo) * B, cudaMemcpyDeviceToHost, st));
  EPB_CUDA(cudaStreamSynchronize(st));
  for (int b = 0; b < B; ++b) {
    if (ih[b].status != JPEG_OK) continue;
    ih[b].hdr_bytes = jpeg_tc_header(blobs_host[b], ih[b].ri, ih[b].bits, ih[b].val, hdr_host + hdr_off_host[b],
                                     hdr_off_host[b + 1] - hdr_off_host[b]);
    EPB_CHECK_ARG(ih[b].hdr_bytes >= 0);
  }
  return EPB_OK;
}
