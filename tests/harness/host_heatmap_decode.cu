// TEST INFRASTRUCTURE: runs the per-joint bodies of heatmap_decode_kernel (csrc/geometry.cu) on the
// CPU (same source, same --fmad=false arithmetic; the argmax scans each map serially, the depth
// soft-argmax keeps the kernel's 32 lane partials and their order).  Binary protocol on stdin/stdout:
//   "decode" layout C N J H W D patch_w patch_h depth_range post_process flip shift has_box
//   then hm (float32, B*J*H*W for layout 0 or B*H*W*C for layout 1), depth (float32, B*J*D),
//   box (float64, N*6, when has_box), perm (int32, J, when flip); B = 2N with flip, else N
//   ->  kps (float64, N*J*4)
//   "p2i" B patch_w patch_h  then coords (float32, B*3), box (float64, B*6)  ->  kps (float64, B*4):
//   patch_to_image_point, the body of epb_patch_to_image
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
void epb_set_error(const char*, ...) {}
int epb_workspace(int, size_t, struct CUstream_st*, void**) { return -1; }   // entry points are not run here
#include "../../epipolarpose_b200/csrc/geometry.cu"

static void rd(void* p, size_t n) { if (n && fread(p, 1, n, stdin) != n) { fprintf(stderr, "short read\n"); exit(2); } }

int main(int argc, char** argv) {
  if (argc == 5 && !strcmp(argv[1], "p2i")) {
    const int B = atoi(argv[2]);
    const double pw = atof(argv[3]), ph = atof(argv[4]);
    std::vector<float> c((size_t)B * 3);
    std::vector<double> box((size_t)B * 6), kps((size_t)B * 4);
    rd(c.data(), c.size() * 4);
    rd(box.data(), box.size() * 8);
    for (int b = 0; b < B; ++b) patch_to_image_point(&c[b * 3], &box[b * 6], pw, ph, 2000.0, &kps[b * 4]);
    fwrite(kps.data(), 8, kps.size(), stdout);
    return 0;
  }
  if (argc < 16 || strcmp(argv[1], "decode")) return 1;
  HmDec a;
  a.layout = atoi(argv[2]); a.C = atoi(argv[3]); a.N = atoi(argv[4]); a.J = atoi(argv[5]);
  a.H = atoi(argv[6]); a.W = atoi(argv[7]); a.D = atoi(argv[8]);
  a.patch_w = atof(argv[9]); a.patch_h = atof(argv[10]); a.depth_range = atof(argv[11]);
  a.post_process = atoi(argv[12]); a.flip = atoi(argv[13]); a.shift = atoi(argv[14]);
  const int has_box = atoi(argv[15]);
  if (a.N < 1 || a.J < 1 || a.J > kHmDecMaxJ || a.H < 1 || a.W < 1 || a.D < 1) return 1;
  if (a.layout != 0 && !(a.layout == 1 && a.C >= a.J)) return 1;
  a.depth_ld = a.J * a.D;
  const size_t B = a.flip ? 2 * (size_t)a.N : (size_t)a.N, HW = (size_t)a.H * a.W;
  std::vector<float> hm(B * HW * (a.layout == 0 ? a.J : a.C)), depth(B * a.depth_ld);
  std::vector<double> box(has_box ? (size_t)a.N * 6 : 0), kps((size_t)a.N * a.J * 4);
  std::vector<int32_t> perm(a.J);
  rd(hm.data(), hm.size() * 4);
  rd(depth.data(), depth.size() * 4);
  rd(box.data(), box.size() * 8);
  if (a.flip) rd(perm.data(), perm.size() * 4);
  unsigned short p16[kHmDecMaxJ];
  for (int j = 0; j < a.J; ++j) p16[j] = (unsigned short)(a.flip ? perm[j] : j);
  a.hm = hm.data(); a.depth = depth.data(); a.box = has_box ? box.data() : nullptr;
  for (int n = 0; n < a.N; ++n)
    for (int j = 0; j < a.J; ++j) {
      float bv = -INFINITY;
      int bi = 0x7fffffff;
      for (int pix = 0; pix < (int)HW; ++pix) {
        const float v = hm_value(a, p16, n, j, pix / a.W, pix % a.W);
        if (hm_better(v, pix, bv, bi)) { bv = v; bi = pix; }
      }
      double* k = &kps[((size_t)n * a.J + j) * 4];
      hm_finish_joint(a, p16, n, j, bv, bi, k);
      float m = -INFINITY;
      for (int d = 0; d < a.D; ++d) m = fmaxf(m, depth_logit(a, p16, n, j, d));
      double s[32], t[32];
      for (int l = 0; l < 32; ++l) depth_lane(a, p16, n, j, l, m, &s[l], &t[l]);
      k[2] = depth_finish(a, s, t);
    }
  fwrite(kps.data(), 8, kps.size(), stdout);
  return 0;
}
