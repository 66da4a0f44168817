// Camera helpers shared by the float64 evaluation kernels (geometry.cu, pss.cu).  Both files
// are compiled with --fmad=false, so every caller rounds a*b+c twice, as numpy does.
#pragma once
#include <math.h>
#include <stdint.h>

// CamBackProj (lib/utils/prep_h36m.py:85-89) of joint j of an image-space pose a [J][3]
// (x px, y px, root-relative depth mm); cam = fx, fy, cx, cy, pelvis depth.  o: camera-frame mm.
__host__ __device__ inline void cam_back_proj(const double* a, int j, const double* cam, double (&o)[3]) {
  const double d = a[j * 3 + 2] + cam[4];
  o[0] = (a[j * 3 + 0] - cam[2]) / cam[0] * d;
  o[1] = (a[j * 3 + 1] - cam[3]) / cam[1] * d;
  o[2] = d;
}

// X_cam = R (X - T) (prep_h36m.py:186) of one world point; c = R(9) T(3) f(2) c(2).
__host__ __device__ inline void cam_from_world(const double* x, const double* c, double (&o)[3]) {
  const double dx = x[0] - c[9], dy = x[1] - c[10], dz = x[2] - c[11];
  o[0] = (c[0] * dx + c[1] * dy) + c[2] * dz;
  o[1] = (c[3] * dx + c[4] * dy) + c[5] * dz;
  o[2] = (c[6] * dx + c[7] * dy) + c[8] * dz;
}

// from_worldjt_to_imagejt (lib/utils/prep_h36m.py:176-204, without the 3-D rectangle) of one
// (frame, camera): world joints X [J][3] with their triangulation status [J] seen by camera c (the
// epb_project_labels layout) -> jt [J][3] = CamProj x, y (px) and camera-frame depth minus the
// root's (mm), vis [J][3], pelvis [3] = the camera-frame root.  Returns ok: the root has status 1
// and lies, finite, in front of the camera.  A joint is visible when ok, its status is 1, its depth
// is > 0 and its row is finite; every row that is not visible is 0, and pelvis is 0 when not ok,
// so nothing non-finite is ever written.
__host__ __device__ inline int32_t cam_pseudo_record(const double* X, const int32_t* status, const double* c, int J,
                                                     int root, double* jt, double* vis, double* pelvis) {
  double r[3];
  cam_from_world(X + root * 3, c, r);
  const int32_t ok = status[root] == 1 && isfinite(r[0]) && isfinite(r[1]) && isfinite(r[2]) && r[2] > 0.0;
  for (int k = 0; k < 3; ++k) pelvis[k] = ok ? r[k] : 0.0;
  for (int j = 0; j < J; ++j) {
    double p[3];
    cam_from_world(X + j * 3, c, p);
    const double u = p[0] / p[2] * c[12] + c[14];     // CamProj :170-175
    const double v = p[1] / p[2] * c[13] + c[15];
    const double z = p[2] - r[2];                      // :199
    const bool on = ok && status[j] == 1 && p[2] > 0.0 && isfinite(u) && isfinite(v) && isfinite(z);
    jt[j * 3 + 0] = on ? u : 0.0;
    jt[j * 3 + 1] = on ? v : 0.0;
    jt[j * 3 + 2] = on ? z : 0.0;
    for (int k = 0; k < 3; ++k) vis[j * 3 + k] = on ? 1.0 : 0.0;
  }
  return ok;
}
