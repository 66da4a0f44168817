// TEST INFRASTRUCTURE: runs the JPEG decode of csrc/jpeg.cu on the CPU -- the same parser,
// subsequence bodies of phase A / C, IDCT and upsample / colour -- with the subsequence length
// as a parameter, so that self-synchronisation happens many times even in small images.  The
// unstuffing is a plain serial loop here; the threads of a phase-A round run one after another
// ("fwd") or in reverse order ("rev", so later subsequences read states not yet corrected).
//   host_jpeg SUB_BITS fwd|rev   stdin: int32 count, then per blob int64 length + bytes
//   -> per blob: int32 status, H, W, coefficients equal to a sequential decode (1 / 0), rounds;
//      then H*W*3 BGR bytes when the status is OK
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
void epb_set_error(const char*, ...) {}
#include "../../epipolarpose_b200/csrc/jpeg.cu"

static void rd(void* p, size_t n) {
  if (fread(p, 1, n, stdin) != n) { fprintf(stderr, "short read\n"); exit(2); }
}

// serial unstuffing with the rules of jpeg_unstuff_kernel; false when the scan is malformed
static bool unstuff(const uint8_t* s, int64_t n, const JpegDesc& d, std::vector<uint8_t>& out,
                    std::vector<int32_t>& seg) {
  seg.assign(1, 0);
  for (int64_t i = 0; i < n; ++i) {
    const int x = s[i];
    if (x != 0xFF) { out.push_back((uint8_t)x); continue; }
    if (i + 1 >= n) break;
    const int nx = s[i + 1];
    if (nx == 0x00) { out.push_back(0xFF); ++i; continue; }
    if (nx == 0xFF) continue;
    if (nx >= 0xD0 && nx <= 0xD7) {
      if (nx - 0xD0 != (int)((seg.size() - 1) & 7)) return false;
      seg.push_back((int32_t)out.size());
      ++i;
      continue;
    }
    break;
  }
  if ((int)seg.size() != d.nseg) return false;
  seg.push_back((int32_t)out.size());
  return true;
}

int main(int argc, char** argv) {
  if (argc < 3) return 1;
  const int L = atoi(argv[1]);
  const bool rev = !strcmp(argv[2], "rev");
  int32_t count;
  rd(&count, 4);
  for (int im = 0; im < count; ++im) {
    int64_t len;
    rd(&len, 8);
    std::vector<uint8_t> blob((size_t)len + 1);
    rd(blob.data(), (size_t)len);
    JpegDesc* d = new JpegDesc;
    int32_t hdr[5] = {jpeg_parse_one(blob.data(), len, L, d), d->H, d->W, 0, 0};
    std::vector<uint8_t> bgr;
    std::vector<uint8_t> bits;
    std::vector<int32_t> seg;
    if (hdr[0] == JPEG_OK && !unstuff(blob.data() + d->ent_off, d->ent_len, *d, bits, seg)) hdr[0] = JPEG_MALFORMED;
    if (hdr[0] == JPEG_OK) {
      bits.resize(bits.size() + 16, 0);
      const int nseg = d->nseg;
      std::vector<int32_t> sub(nseg + 1, 0);
      for (int s = 0; s < nseg; ++s) sub[s + 1] = sub[s] + nsub_of(seg[s + 1] - seg[s], L);
      const int nsub = sub[nseg];
      std::vector<JpegEntry> ent(nsub);
      for (int j = 0; j < nsub; ++j) ent[j] = jpeg_sub_phase_a(*d, bits.data(), sub_geom(seg.data(), sub.data(), nseg, j, L));
      for (bool changed = true; changed;) {         // rounds until one writes nothing
        changed = false;
        ++hdr[4];
        for (int t = 0; t < nsub; ++t) {
          const int j = rev ? nsub - 1 - t : t;
          const SubGeom g = sub_geom(seg.data(), sub.data(), nseg, j, L);
          JpegEntry cur = ent[j];
          for (int q = j + 1; q < g.last; ++q) {
            const JpegEntry e = jpeg_sub_entry(*d, bits.data(), sub_geom(seg.data(), sub.data(), nseg, q, L),
                                               st_clear_n(cur.st));
            if (state_eq(e.st, ent[q].st)) break;
            ent[q] = e;
            changed = true;
            cur = e;
          }
        }
      }
      std::vector<JpegPrefix> pb(nsub);
      for (int s = 0; s < nseg && hdr[0] == JPEG_OK; ++s) {
        JpegPrefix acc = {0, {0, 0, 0}};
        for (int q = sub[s]; q < sub[s + 1]; ++q) {
          const SubGeom g = sub_geom(seg.data(), sub.data(), nseg, q, L);
          const JpegPrefix n = jpeg_sub_count(*d, bits.data(), g, q == g.first ? st_make(g.start, 0, 0, 0, 0)
                                                                                : st_clear_n(ent[q - 1].st));
          pb[q] = acc;
          acc.first += n.first;
          for (int c = 0; c < 3; ++c) acc.dc[c] += n.dc[c];
        }
        if (acc.first < seg_blocks(*d, s)) hdr[0] = JPEG_MALFORMED;
      }
      if (hdr[0] == JPEG_OK) {
        std::vector<int16_t> coef((size_t)d->nblocks * 64, 0), ref((size_t)d->nblocks * 64, 0);
        for (int j = 0; j < nsub; ++j) {
          const SubGeom g = sub_geom(seg.data(), sub.data(), nseg, j, L);
          const uint64_t start = j == g.first ? st_make(g.start, 0, 0, 0, 0) : st_clear_n(ent[j - 1].st);
          jpeg_sub_phase_c(*d, bits.data(), g, start, pb[j], coef.data(), seg_first_block(*d, g.seg),
                           seg_blocks(*d, g.seg));
        }
        for (int s = 0; s < nseg; ++s) {           // plain sequential decode of each segment
          SinkWrite w;
          w.coef = ref.data() + seg_first_block(*d, s) * 64;
          w.pred[0] = w.pred[1] = w.pred[2] = 0;
          w.limit = seg_blocks(*d, s);
          jpeg_run(*d, bits.data(), st_make((uint32_t)seg[s] * 8, 0, 0, 0, 0), (uint32_t)seg[s + 1] * 8,
                   (uint32_t)seg[s + 1] * 8, w);
        }
        hdr[3] = coef == ref ? 1 : 0;
        std::vector<std::vector<uint8_t>> planes(d->ncomp);
        for (int c = 0; c < d->ncomp; ++c) planes[c].assign((size_t)d->pw[c] * d->ph[c], 0);
        for (int64_t blk = 0; blk < d->nblocks; ++blk) {
          int c;
          int64_t off;
          block_place(*d, blk, &c, &off);
          jpeg_idct_block(coef.data() + blk * 64, d->qt[c], planes[c].data() + off, d->pw[c]);
        }
        const uint8_t* pl[3] = {planes[0].data(), d->ncomp > 1 ? planes[1].data() : nullptr,
                                d->ncomp > 1 ? planes[2].data() : nullptr};
        bgr.resize((size_t)d->H * d->W * 3);
        for (int y = 0; y < d->H; ++y) jpeg_color_row(*d, pl, y, bgr.data() + (size_t)y * d->W * 3);
      }
    }
    fwrite(hdr, 4, 5, stdout);
    if (hdr[0] == JPEG_OK) fwrite(bgr.data(), 1, bgr.size(), stdout);
    delete d;
  }
  return 0;
}
