// TEST INFRASTRUCTURE: runs relpose_pair, the per-pair body of relative_pose_kernel in
// csrc/geometry.cu, on the CPU (same source, same --fmad=false arithmetic, one lane instead of a
// warp).  Binary protocol on stdin/stdout (little-endian doubles):
//   "pairs" N J  then per pair: ua[J*2] ub[J*2] intr_a[4] intr_b[4] box_a[6] box_b[6] rect3d_w[1]
//   ->  per pair: Pa[12] Pb[12] cam_a[16] cam_b[16] inliers[J] status[1] diag[3] scores[256]
//       (scores: the LMedS score of every hypothesis, NaN where it is invalid)
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
void epb_set_error(const char*, ...) {}
int epb_workspace(int, size_t, struct CUstream_st*, void**) { return -1; }   // entry points are not run here
#include "../../epipolarpose_b200/csrc/geometry.cu"

static void rd(void* p, size_t n) { if (fread(p, 1, n, stdin) != n) { fprintf(stderr, "short read\n"); exit(2); } }

int main(int argc, char** argv) {
  if (argc < 4 || strcmp(argv[1], "pairs")) return 1;
  const int N = atoi(argv[2]), J = atoi(argv[3]);
  if (J < 8 || J > RP_MAXJ) return 1;
  const int nin = 4 * J + 4 + 4 + 6 + 6 + 1;
  std::vector<double> in((size_t)nin), out;
  for (int p = 0; p < N; ++p) {
    rd(in.data(), in.size() * 8);
    const double *ua = &in[0], *ub = &in[2 * J], *ia = &in[4 * J], *ib = ia + 4, *ba = ib + 4, *bb = ba + 6;
    const double rect = bb[6];
    double Pa[12], Pb[12], cam[32];
    std::vector<int32_t> inl(J);
    int32_t st, diag[3];
    RpSerial red;
    relpose_pair(red, ua, ub, 2, J, ia, ib, ba, bb, rect, Pa, Pb, cam, cam + 16, inl.data(), &st, diag);
    out.insert(out.end(), Pa, Pa + 12);
    out.insert(out.end(), Pb, Pb + 12);
    out.insert(out.end(), cam, cam + 32);
    for (int j = 0; j < J; ++j) out.push_back(inl[j]);
    out.push_back(st);
    for (int k = 0; k < 3; ++k) out.push_back(diag[k]);
    for (int h = 0; h < RP_HYP; ++h) {
      double F[9];
      out.push_back(relpose_hypothesis(ua, ub, 2, J, h, F) ? relpose_score(F, ua, ub, 2, J) : NAN);
    }
  }
  fwrite(out.data(), 8, out.size(), stdout);
  return 0;
}
