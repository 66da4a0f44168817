// TEST INFRASTRUCTURE: runs robust_point, the per-(tuple, joint) body of triangulate_robust_kernel
// in csrc/geometry.cu, on the CPU (same source, same --fmad=false arithmetic, one lane instead of
// a warp).  Binary protocol on stdin/stdout (little-endian doubles):
//   "robust" N V J threshold_px has_w  then per tuple: u[V*J*2] P[V*12] (w[V*J] when has_w)
//   ->  per tuple: X[J*3] inliers[J] resid[J] status[J]
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
  if (argc < 7 || strcmp(argv[1], "robust")) return 1;
  const int N = atoi(argv[2]), V = atoi(argv[3]), J = atoi(argv[4]);
  const double thr = atof(argv[5]);
  const int has_w = atoi(argv[6]);
  if (N < 0 || V < 2 || V > RB_MAXV || J < 0) return 1;
  std::vector<double> u((size_t)V * J * 2), P((size_t)V * 12), w((size_t)V * J, 1.0), out;
  for (int t = 0; t < N; ++t) {
    rd(u.data(), u.size() * 8);
    rd(P.data(), P.size() * 8);
    if (has_w) rd(w.data(), w.size() * 8);
    std::vector<double> X((size_t)J * 3), res(J);
    std::vector<int32_t> inl(J), st(J);
    for (int j = 0; j < J; ++j) {
      double uu[RB_MAXV * 2], ww[RB_MAXV];
      for (int v = 0; v < V; ++v) {
        uu[2 * v] = u[((size_t)v * J + j) * 2];
        uu[2 * v + 1] = u[((size_t)v * J + j) * 2 + 1];
        ww[v] = w[(size_t)v * J + j];
      }
      RbSerial red;
      robust_point(red, uu, P.data(), ww, V, thr, &X[(size_t)j * 3], &inl[j], &res[j], &st[j]);
    }
    out.insert(out.end(), X.begin(), X.end());
    for (int j = 0; j < J; ++j) out.push_back(inl[j]);
    out.insert(out.end(), res.begin(), res.end());
    for (int j = 0; j < J; ++j) out.push_back(st[j]);
  }
  fwrite(out.data(), 8, out.size(), stdout);
  return 0;
}
