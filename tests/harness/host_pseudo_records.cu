// TEST INFRASTRUCTURE: runs cam_pseudo_record, the per-(frame, camera) body of
// pseudo_records_kernel in csrc/geometry.cu (csrc/camera.cuh), on the CPU (same source, same
// --fmad=false arithmetic), and the host-side argument checks of epb_pseudo_records.
// Binary protocol on stdin/stdout (little-endian):
//   "records" T S V J root  stdin: X f64[T*S*J*3] status i32[T*S*J] cam f64[T*V*16]
//       ->  f64: joints_3d[T*V*J*3] vis[T*V*J*3] pelvis[T*V*3] ok[T*V]
//   "args" T S V J root     ->  the return code of the size checks (text); where they refuse, or
//       T = 0, epb_pseudo_records itself is called on dummy buffers and must return the same
//       (exit 3 otherwise).  Nothing is ever launched.
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
  if (argc < 7) return 1;
  const int T = atoi(argv[2]), S = atoi(argv[3]), V = atoi(argv[4]), J = atoi(argv[5]), root = atoi(argv[6]);
  if (!strcmp(argv[1], "args")) {
    // the entry is called only where it cannot launch: sizes its checks refuse, or T = 0
    const int rc = pseudo_records_sizes(T, S, V, J, root);
    if (rc == EPB_OK && T != 0) {
      printf("%d\n", rc);
      return 0;
    }
    double d[4];
    int32_t i[4];
    const int rc2 = epb_pseudo_records(d, i, d, T, S, V, J, root, d, d, d, i, nullptr);
    if (rc2 != rc) return 3;
    printf("%d\n", rc2);
    return 0;
  }
  if (strcmp(argv[1], "records") || T < 0 || V < 2 || V > 8 || (S != 1 && S != V) || J < 1 || root < 0 || root >= J)
    return 1;
  std::vector<double> X((size_t)T * S * J * 3), cam((size_t)T * V * 16);
  std::vector<int32_t> st((size_t)T * S * J);
  rd(X.data(), X.size() * 8);
  rd(st.data(), st.size() * 4);
  rd(cam.data(), cam.size() * 8);
  std::vector<double> jt((size_t)T * V * J * 3), vis(jt.size()), pel((size_t)T * V * 3), ok((size_t)T * V);
  for (size_t i = 0; i < (size_t)T * V; ++i) {
    const size_t t = i / V, v = i % V, s = t * S + (S == 1 ? 0 : v);
    ok[i] = cam_pseudo_record(&X[s * J * 3], &st[s * J], &cam[i * 16], J, root, &jt[i * J * 3], &vis[i * J * 3],
                              &pel[i * 3]);
  }
  fwrite(jt.data(), 8, jt.size(), stdout);
  fwrite(vis.data(), 8, vis.size(), stdout);
  fwrite(pel.data(), 8, pel.size(), stdout);
  fwrite(ok.data(), 8, ok.size(), stdout);
  return 0;
}
