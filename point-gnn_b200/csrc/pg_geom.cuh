// Box geometry shared by NMS and box decoding (pg_post.cu), the KITTI rows (pg_kitti.cu) and the KITTI evaluator
// (pg_eval.cu): NumPy's float32 sin / cos, one box footprint record and one Sutherland-Hodgman clipper in fp64.
#pragma once
#include "pg_common.cuh"

namespace pg {

// NumPy's float32 sin (want_cos = 0) or cos (want_cos = 1) for |x| below its Cody-Waite range.  NumPy's float32
// cos / sin are not the correctly rounded values: they are its SIMD routine (Cody-Waite reduction by pi/2 in three
// FMA steps, then a degree-8 cosine or degree-9 sine polynomial evaluated with FMA), restated here operation for
// operation.  Outside that range NumPy calls the C library's float routine, which the correctly rounded double
// result stands in for.
__device__ inline float np_trig(float x, int want_cos) {
  if (!(fabsf(x) <= (want_cos ? 71476.0625f : 117435.992f))) {
    if (isnan(x) || isinf(x)) return __int_as_float(0x7fc00000);
    return float(want_cos ? cos(double(x)) : sin(double(x)));
  }
  const float magic = 0x1.800000p+23f;
  float q = __fmul_rn(x, 0x1.45f306p-1f);                      // x * 2 / pi, rounded to an integer:
  q = __fsub_rn(__fadd_rn(q, magic), magic);
  float r = __fmaf_rn(q, -0x1.921fb0p+00f, x);                 // x - q * pi / 2 in three parts
  r = __fmaf_rn(q, -0x1.5110b4p-22f, r);
  r = __fmaf_rn(q, -0x1.846988p-48f, r);
  const float r2 = __fmul_rn(r, r);
  float c = __fmaf_rn(0x1.98e616p-16f, r2, -0x1.6c06dcp-10f);
  c = __fmaf_rn(c, r2, 0x1.55553cp-05f);
  c = __fmaf_rn(c, r2, -0x1.000000p-01f);
  c = __fmaf_rn(c, r2, 0x1.000000p+00f);
  float s = __fmaf_rn(0x1.7d3bbcp-19f, r2, -0x1.a06bbap-13f);
  s = __fmaf_rn(s, r2, 0x1.11119ap-07f);
  s = __fmaf_rn(s, r2, -0x1.555556p-03f);
  s = __fmaf_rn(s, r2, 0.0f);
  s = __fmaf_rn(s, r, r);
  const int quadrant = int(q) + want_cos;
  const float v = (quadrant & 1) ? c : s;
  return (quadrant & 2) ? __fsub_rn(0.0f, v) : v;
}

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
