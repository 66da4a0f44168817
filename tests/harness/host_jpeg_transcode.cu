// TEST INFRASTRUCTURE: runs the lossless transcode of csrc/jpeg.cu on the CPU -- the parser, the
// phase A / B / C bodies of the decoder (subsequences of kJpegSubBits, rounds until none writes),
// then the symbol, table, length and write bodies of the transcode and its header -- and decodes
// the result again with the same bodies.
//   host_jpeg_transcode R        stdin: int32 count, then per blob int64 length + bytes; R = 0: auto
//   -> per blob: int32 status, R, intervals, coefficients of the output equal to the source's (1 / 0),
//      ri and nseg of the output's parse; int64 size; the output file (size bytes; empty when the
//      status is not OK); int32 coded bits of every interval
//   host_jpeg_transcode table    stdin: int32 count, then per histogram int32 n + n int64 counts
//   -> per histogram: bits[17], val[256] of huff_optimal
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
void epb_set_error(const char*, ...) {}
#include "../../epipolarpose_b200/csrc/jpeg.cu"

static void rd(void* p, size_t n) {
  if (fread(p, 1, n, stdin) != n) { fprintf(stderr, "short read\n"); exit(2); }
}

// parse + coefficients of one blob (the decoder's stages 2-3); returns the status
static int coefs(const std::vector<uint8_t>& blob, JpegDesc& d, std::vector<int16_t>& coef) {
  const int L = kJpegSubBits;
  if (jpeg_parse_one(blob.data(), (int64_t)blob.size(), L, &d) != JPEG_OK) return d.status;
  std::vector<uint8_t> bits;
  std::vector<int32_t> seg(1, 0);
  const uint8_t* s = blob.data() + d.ent_off;
  for (int64_t i = 0; i < d.ent_len; ++i) {        // the unstuffing rules of jpeg_unstuff_kernel
    const int x = s[i];
    if (x != 0xFF) { bits.push_back((uint8_t)x); continue; }
    if (i + 1 >= d.ent_len) break;
    const int nx = s[i + 1];
    if (nx == 0x00) { bits.push_back(0xFF); ++i; continue; }
    if (nx == 0xFF) continue;
    if (nx >= 0xD0 && nx <= 0xD7) {
      if (nx - 0xD0 != (int)((seg.size() - 1) & 7)) return JPEG_MALFORMED;
      seg.push_back((int32_t)bits.size());
      ++i;
      continue;
    }
    break;
  }
  if ((int)seg.size() != d.nseg) return JPEG_MALFORMED;
  seg.push_back((int32_t)bits.size());
  bits.resize(bits.size() + 16, 0);
  const int nseg = d.nseg;
  std::vector<int32_t> sub(nseg + 1, 0);
  for (int q = 0; q < nseg; ++q) sub[q + 1] = sub[q] + nsub_of(seg[q + 1] - seg[q], L);
  const int nsub = sub[nseg];
  std::vector<JpegEntry> ent(nsub);
  for (int j = 0; j < nsub; ++j) ent[j] = jpeg_sub_phase_a(d, bits.data(), sub_geom(seg.data(), sub.data(), nseg, j, L));
  for (bool changed = true; changed;) {
    changed = false;
    for (int j = 0; j < nsub; ++j) {
      const SubGeom g = sub_geom(seg.data(), sub.data(), nseg, j, L);
      JpegEntry cur = ent[j];
      for (int q = j + 1; q < g.last; ++q) {
        const JpegEntry e = jpeg_sub_entry(d, bits.data(), sub_geom(seg.data(), sub.data(), nseg, q, L), st_clear_n(cur.st));
        if (state_eq(e.st, ent[q].st)) break;
        ent[q] = e;
        changed = true;
        cur = e;
      }
    }
  }
  std::vector<JpegPrefix> pb(nsub);
  for (int q = 0; q < nseg; ++q) {
    JpegPrefix acc = {0, {0, 0, 0}};
    for (int j = sub[q]; j < sub[q + 1]; ++j) {
      const SubGeom g = sub_geom(seg.data(), sub.data(), nseg, j, L);
      const JpegPrefix n = jpeg_sub_count(d, bits.data(), g, j == g.first ? st_make(g.start, 0, 0, 0, 0) : st_clear_n(ent[j - 1].st));
      pb[j] = acc;
      acc.first += n.first;
      for (int c = 0; c < 3; ++c) acc.dc[c] += n.dc[c];
    }
    if (acc.first < seg_blocks(d, q)) return JPEG_MALFORMED;
  }
  coef.assign((size_t)d.nblocks * 64, 0);
  for (int j = 0; j < nsub; ++j) {
    const SubGeom g = sub_geom(seg.data(), sub.data(), nseg, j, L);
    const uint64_t start = j == g.first ? st_make(g.start, 0, 0, 0, 0) : st_clear_n(ent[j - 1].st);
    jpeg_sub_phase_c(d, bits.data(), g, start, pb[j], coef.data(), seg_first_block(d, g.seg), seg_blocks(d, g.seg));
  }
  return JPEG_OK;
}

static int table_mode() {
  int32_t count;
  rd(&count, 4);
  TcWork* w = new TcWork;
  for (int h = 0; h < count; ++h) {
    int32_t n;
    rd(&n, 4);
    std::vector<int64_t> c(n);
    rd(c.data(), 8 * (size_t)n);
    uint8_t bits[17], val[256] = {0};
    huff_optimal(c.data(), n, *w, bits, val);
    fwrite(bits, 1, 17, stdout);
    fwrite(val, 1, 256, stdout);
  }
  delete w;
  return 0;
}

int main(int argc, char** argv) {
  if (argc < 2) return 1;
  if (!strcmp(argv[1], "table")) return table_mode();
  const int R = atoi(argv[1]);
  int32_t count;
  rd(&count, 4);
  TcWork* work = new TcWork;
  for (int im = 0; im < count; ++im) {
    int64_t len;
    rd(&len, 8);
    std::vector<uint8_t> blob((size_t)len);
    rd(blob.data(), (size_t)len);
    blob.reserve(blob.size() + 16);
    JpegDesc* d = new JpegDesc;
    std::vector<int16_t> coef;
    int32_t hdr[6] = {coefs(blob, *d, coef), 0, 0, 0, 0, 0};
    std::vector<uint8_t> out;
    std::vector<int32_t> ibits;
    if (hdr[0] == JPEG_OK) {
      const int ri = R ? R : tc_auto_interval(*d);
      const int64_t mcus = (int64_t)d->mcux * d->mcuy;
      const int nint = (int)((mcus + ri - 1) / ri);
      hdr[1] = ri;
      hdr[2] = nint;
      std::vector<int32_t> hist((size_t)nint * kTcBins, 0);
      bool ok = true;
      for (int i = 0; i < nint; ++i) {
        TcHist sink{hist.data() + (size_t)i * kTcBins};
        ok = tc_walk(*d, coef.data(), ri, i, sink) && ok;
      }
      if (!ok) hdr[0] = JPEG_UNSUPPORTED;
      if (ok) {
        int64_t cnt[kTcBins] = {0};
        for (int i = 0; i < nint; ++i)
          for (int k = 0; k < kTcBins; ++k) cnt[k] += hist[(size_t)i * kTcBins + k];
        uint8_t bits[4][17], val[4][256] = {{0}};
        TcTable tab[4];
        for (int slot = 0; slot < 4; ++slot) {
          huff_optimal(slot < 2 ? cnt + slot * kTcDcBins : cnt + 2 * kTcDcBins + (slot - 2) * 256,
                       slot < 2 ? kTcDcBins : 256, *work, bits[slot], val[slot]);
          huff_codes(bits[slot], val[slot], tab[slot]);
        }
        out.resize((size_t)d->ent_off + kTcDhtMax + 8);
        const int64_t h = jpeg_tc_header(blob.data(), ri, bits, val, out.data(), (int64_t)out.size());
        if (h < 0) { fprintf(stderr, "header\n"); return 3; }
        out.resize((size_t)h);
        for (int i = 0; i < nint; ++i) {
          const TcLen l = tc_interval_len(*d, coef.data(), tab, ri, nint, i);
          const size_t o = out.size();
          out.resize(o + (size_t)l.bytes);
          if (!tc_interval_write(*d, coef.data(), tab, ri, nint, i, l, out.data() + o)) { fprintf(stderr, "write\n"); return 3; }
          ibits.push_back(l.bits);
        }
        out.push_back(0xFF);
        out.push_back(0xD9);
        JpegDesc* d2 = new JpegDesc;
        std::vector<int16_t> coef2;
        if (coefs(out, *d2, coef2) == JPEG_OK) {
          hdr[3] = coef2 == coef ? 1 : 0;
          hdr[4] = d2->ri;
          hdr[5] = d2->nseg;
        }
        delete d2;
      }
    }
    if (hdr[0] != JPEG_OK) { out.clear(); ibits.clear(); }
    const int64_t size = (int64_t)out.size();
    fwrite(hdr, 4, 6, stdout);
    fwrite(&size, 8, 1, stdout);
    if (!out.empty()) fwrite(out.data(), 1, out.size(), stdout);
    if (!ibits.empty()) fwrite(ibits.data(), 4, ibits.size(), stdout);
    delete d;
  }
  delete work;
  return 0;
}
