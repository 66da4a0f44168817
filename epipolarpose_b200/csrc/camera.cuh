// Camera helpers shared by the float64 evaluation kernels (geometry.cu, pss.cu).  Both files
// are compiled with --fmad=false, so every caller rounds a*b+c twice, as numpy does.
#pragma once

// CamBackProj (lib/utils/prep_h36m.py:85-89) of joint j of an image-space pose a [J][3]
// (x px, y px, root-relative depth mm); cam = fx, fy, cx, cy, pelvis depth.  o: camera-frame mm.
__host__ __device__ inline void cam_back_proj(const double* a, int j, const double* cam, double (&o)[3]) {
  const double d = a[j * 3 + 2] + cam[4];
  o[0] = (a[j * 3 + 0] - cam[2]) / cam[0] * d;
  o[1] = (a[j * 3 + 1] - cam[3]) / cam[1] * d;
  o[2] = d;
}
