// TEST INFRASTRUCTURE: runs pose_errors_sample and pose_to_camera_sample, the per-sample bodies of
// epb_pose_errors / epb_pose_to_camera in csrc/geometry.cu, on the CPU (same source, same
// --fmad=false arithmetic).  Binary protocol on stdin/stdout (little-endian doubles):
//   "errors" S J mask  then pred[S*J*3] gt[S*J*3]  ->  metrics[S*7] per_joint[S*J]
//   "camera" N J root  then joints[N*J*3] cam[N*5]  ->  out[N*J*3]
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
void epb_set_error(const char*, ...) {}
int epb_workspace(int, size_t, struct CUstream_st*, void**) { return -1; }   // entry points are not run here
#include "../../epipolarpose_b200/csrc/geometry.cu"

static void rd(void* p, size_t n) { if (n && fread(p, 1, n, stdin) != n) { fprintf(stderr, "short read\n"); exit(2); } }

int main(int argc, char** argv) {
  if (argc < 5) return 1;
  const int S = atoi(argv[2]), J = atoi(argv[3]);
  if (S < 0 || J < 1 || J > 32) return 1;
  if (!strcmp(argv[1], "errors")) {
    const unsigned mask = (unsigned)strtoul(argv[4], nullptr, 10);
    std::vector<double> pred((size_t)S * J * 3), gt(pred.size()), met((size_t)S * 7), pj((size_t)S * J);
    rd(pred.data(), pred.size() * 8);
    rd(gt.data(), gt.size() * 8);
    for (int s = 0; s < S; ++s)
      pose_errors_sample(&pred[(size_t)s * J * 3], &gt[(size_t)s * J * 3], J, mask, &met[(size_t)s * 7],
                         &pj[(size_t)s * J]);
    fwrite(met.data(), 8, met.size(), stdout);
    fwrite(pj.data(), 8, pj.size(), stdout);
    return 0;
  }
  if (!strcmp(argv[1], "camera")) {
    const int root = atoi(argv[4]);
    if (root < 0 || root >= J) return 1;
    std::vector<double> joints((size_t)S * J * 3), cam((size_t)S * 5), out(joints.size());
    rd(joints.data(), joints.size() * 8);
    rd(cam.data(), cam.size() * 8);
    for (int s = 0; s < S; ++s)
      pose_to_camera_sample(&joints[(size_t)s * J * 3], &cam[(size_t)s * 5], J, root, &out[(size_t)s * J * 3]);
    fwrite(out.data(), 8, out.size(), stdout);
    return 0;
  }
  return 1;
}
