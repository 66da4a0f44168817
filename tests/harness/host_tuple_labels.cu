// TEST INFRASTRUCTURE: runs the bodies of epb_tuple_labels in csrc/geometry.cu on the CPU (same
// source, same --fmad=false arithmetic, one lane instead of a warp).  Binary protocol on
// stdin/stdout (little-endian doubles; float32 inputs travel as doubles and are rounded here):
//   "project" B J: X[B*J*3] cam[B*16] box[B*6]  ->  label[B*J*3] cz[B*J] pelvis_z[B*J]
//       project_label_point, the label body shared by project_labels_kernel and tuple_label_kernel
//   "tuple" T V J threshold_px has_lse: coords[V*T*J*3] box[V*T*6] P[V*T*12] cam[V*T*16]
//       (lse[V*T*J*2] when has_lse)  ->  label[V*T*J*3] weight[V*T*J*3] X[T*J*3] inliers[T*J]
//       resid[T*J] status[T*J]: tuple_point for every (tuple, joint), then tuple_label for every
//       (row, joint); patch 256 x 256, rect3d_w 2000
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
void epb_set_error(const char*, ...) {}
int epb_workspace(int, size_t, struct CUstream_st*, void**) { return -1; }   // entry points are not run here
#include "../../epipolarpose_b200/csrc/geometry.cu"

static std::vector<double> rd(size_t n) {
  std::vector<double> v(n);
  if (n && fread(v.data(), 8, n, stdin) != n) { fprintf(stderr, "short read\n"); exit(2); }
  return v;
}
static std::vector<float> f32(const std::vector<double>& v) { return std::vector<float>(v.begin(), v.end()); }

int main(int argc, char** argv) {
  std::vector<double> out;
  if (argc == 4 && !strcmp(argv[1], "project")) {
    const int B = atoi(argv[2]), J = atoi(argv[3]);
    const auto X = rd((size_t)B * J * 3), cam = rd((size_t)B * 16), box = rd((size_t)B * 6);
    std::vector<double> cz((size_t)B * J), pz((size_t)B * J);
    for (int b = 0; b < B; ++b)
      for (int j = 0; j < J; ++j) {
        float lab[3];
        project_label_point(&X[((size_t)b * J + j) * 3], &X[(size_t)b * J * 3], &cam[(size_t)b * 16],
                            &box[(size_t)b * 6], 256.0, 256.0, 2000.0, lab, cz[(size_t)b * J + j],
                            pz[(size_t)b * J + j]);
        out.insert(out.end(), lab, lab + 3);
      }
    out.insert(out.end(), cz.begin(), cz.end());
    out.insert(out.end(), pz.begin(), pz.end());
  } else if (argc == 7 && !strcmp(argv[1], "tuple")) {
    const int T = atoi(argv[2]), V = atoi(argv[3]), J = atoi(argv[4]);
    const double thr = atof(argv[5]);
    const int has_lse = atoi(argv[6]);
    if (T < 0 || V < 2 || V > RB_MAXV || J < 0) return 1;
    const size_t B = (size_t)V * T;
    const auto coords = f32(rd(B * J * 3));
    const auto box = rd(B * 6), P = rd(B * 12), cam = rd(B * 16);
    const auto lse = f32(rd(has_lse ? B * J * 2 : 0));
    std::vector<double> X((size_t)T * J * 3), resid((size_t)T * J);
    std::vector<int32_t> inl((size_t)T * J), st((size_t)T * J);
    for (int t = 0; t < T; ++t)
      for (int j = 0; j < J; ++j) {
        double u[RB_MAXV * 2], Pv[RB_MAXV * 12], w[RB_MAXV];
        const size_t i = (size_t)t * J + j;
        RbSerial red;
        tuple_point(red, coords.data(), has_lse ? lse.data() : nullptr, box.data(), P.data(), T, V, J, t, j, 256.0,
                    256.0, 2000.0, thr, u, Pv, w, &X[i * 3], &inl[i], &resid[i], &st[i]);
      }
    std::vector<float> label(B * J * 3), weight(B * J * 3);
    for (size_t row = 0; row < B; ++row)
      for (int j = 0; j < J; ++j)
        tuple_label(X.data(), st.data(), cam.data(), box.data(), T, J, (int64_t)row, j, 256.0, 256.0, 2000.0,
                    &label[(row * J + j) * 3], &weight[(row * J + j) * 3]);
    out.insert(out.end(), label.begin(), label.end());
    out.insert(out.end(), weight.begin(), weight.end());
    out.insert(out.end(), X.begin(), X.end());
    out.insert(out.end(), inl.begin(), inl.end());
    out.insert(out.end(), resid.begin(), resid.end());
    out.insert(out.end(), st.begin(), st.end());
  } else {
    return 1;
  }
  fwrite(out.data(), 8, out.size(), stdout);
  return 0;
}
