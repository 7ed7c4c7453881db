// Convex-footprint geometry shared by NMS (pg_post.cu) and the KITTI evaluator (pg_eval.cu): one box footprint
// record and one Sutherland-Hodgman clipper, all in fp64.
#pragma once
#include "pg_common.cuh"

namespace pg {

struct BoxGeom {
  double fx[4], fz[4];   // footprint corners (x, z), nms.py:17-20 order
  double ymin, ymax, xmin, xmax, zmin, zmax;
  double area;
};

__device__ inline double shoelace(const double* x, const double* z, int n) {
  double a = 0.0;
  for (int i = 0; i < n; ++i) {
    const int j = (i + 1 == n) ? 0 : i + 1;
    a += x[i] * z[j] - z[i] * x[j];
  }
  return 0.5 * a;
}

// area of (convex subject) clipped by (convex clip), Sutherland-Hodgman
__device__ inline double clipped_area(const BoxGeom& subj, const BoxGeom& clip) {
  double px[12], pz[12], qx[12], qz[12];
  int n = 4;
  for (int i = 0; i < 4; ++i) { px[i] = subj.fx[i]; pz[i] = subj.fz[i]; }
  const bool ccw = shoelace(clip.fx, clip.fz, 4) >= 0.0;
  for (int e = 0; e < 4 && n > 0; ++e) {
    // walk the clip polygon counter-clockwise
    const int ia = ccw ? e : (4 - e) & 3, ib = ccw ? (e + 1) & 3 : (3 - e);
    const double ax = clip.fx[ia], az = clip.fz[ia];
    const double ex = clip.fx[ib] - ax, ez = clip.fz[ib] - az;
    int m = 0;
    for (int j = 0; j < n; ++j) {
      const int k = (j + 1 == n) ? 0 : j + 1;
      const double sp = ex * (pz[j] - az) - ez * (px[j] - ax);
      const double sq = ex * (pz[k] - az) - ez * (px[k] - ax);
      if (sp >= 0.0) { qx[m] = px[j]; qz[m] = pz[j]; ++m; }
      if ((sp >= 0.0) != (sq >= 0.0)) {
        const double t = sp / (sp - sq);
        qx[m] = px[j] + t * (px[k] - px[j]);
        qz[m] = pz[j] + t * (pz[k] - pz[j]);
        ++m;
      }
    }
    n = m;
    for (int j = 0; j < n; ++j) { px[j] = qx[j]; pz[j] = qz[j]; }
  }
  return n >= 3 ? fabs(shoelace(px, pz, n)) : 0.0;
}

}  // namespace pg
