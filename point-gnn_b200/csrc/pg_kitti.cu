// KITTI result rows on the GPU: the per-detection conversion the KITTI writer runs after NMS, for every kept box of
// every frame of a batch in one call.
//
// Replaces
//   run.py:361-408            corners -> image projection -> 2-D box clipped to 1242 x 375 -> truncation filter
//                             (> 0.4 drops the box) -> `assert l > 0` -> occlusion rescoring
//   run.py:88-100             occlusion: the product of the three cover rates of the candidates inside the box
//   nms.py:9-27               boxes_3d_to_corners
//   kitti_dataset.py:85-162   box3d_to_cam_points / box3d_to_normals / sel_xyz_in_box3d (strict in-box test)
//   kitti_dataset.py:1036-1052 cam_points_to_image
//
// Arithmetic: the dtype chain of run.kitti_labels under NumPy 2, value by value.
//   float32  the box (x, y, z, l, h, w, yaw) and the score as NMS returns them; l / 2, w / 2, -h; and np.cos / np.sin
//            of the float32 yaw.  NumPy's float32 cos / sin are not the correctly rounded values: they are its SIMD
//            routine (Cody-Waite reduction by pi/2 in three FMA steps, then a degree-8 cosine or degree-9 sine
//            polynomial evaluated with FMA), which np_trig below restates operation for operation.
//   float64  everything else.  np.array([[l / 2, 0.0, w / 2], ...]) holds a Python float, so the corner matrix and
//            the rotation matrix are float64 (the float32 values widened).  Every matrix product (corners . R^T,
//            [corners | 1] . cam_to_image^T, wx . p, candidates . normals^T) goes through BLAS dgemm / ddot, whose
//            x86 kernels accumulate a row-column product as acc = fma(a_k, b_k, acc) for k = 0, 1, ..., starting
//            from the rounded first product: dot3 / dot4 below, with explicit __fma_rn.  The additions of the box
//            centre, the differences of corners, the divisions by the projective coordinate, the clip bounds, the
//            truncation rate, the cover rates and (1 + occlusion) * score are element-wise float64 operations:
//            explicit __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn, so that no FMA contraction changes them.
//   The candidate coordinates are float32 and widened before the product with the float64 normals.
//   When rescoring finds no candidate inside, occlusion is the Python int 0 and the score stays the float32 value;
//   the caller restores that type from the inside count of the row.
#include "pg_common.cuh"

namespace pg {
namespace {

constexpr int kBoxLen = 7;
constexpr int kWarpsPerBlock = 8;
constexpr double kImageWidth = 1242.0, kImageHeight = 375.0;   // run.py:385-388 hard-codes these, not the image size
constexpr double kMaxTruncation = 0.4;                           // run.py:392

// NumPy's float32 sin (want_cos = 0) or cos (want_cos = 1) for |x| below its Cody-Waite range; outside it NumPy
// calls the C library's float routine, which the correctly rounded double result stands in for.
__device__ float np_trig(float x, int want_cos) {
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

// BLAS's row . column: fma chain over k from the rounded first product
__device__ __forceinline__ double dot3(double a0, double a1, double a2, double b0, double b1, double b2) {
  return __fma_rn(a2, b2, __fma_rn(a1, b1, __dmul_rn(a0, b0)));
}

// nms.py:9-27 corner k of the box (cos c, sin s): corners . R^T + centre, R = [[c, 0, s], [0, 1, 0], [-s, 0, c]]
__device__ __forceinline__ void corner(const float* b, double c, double s, int k, double* p) {
  const double hl = double(__fdiv_rn(b[3], 2.0f)), hw = double(__fdiv_rn(b[5], 2.0f));
  const double lx = (k & 3) < 2 ? hl : -hl;
  const double ly = k < 4 ? 0.0 : double(-b[4]);
  const double lz = ((k & 3) == 0 || (k & 3) == 3) ? hw : -hw;
  p[0] = __dadd_rn(dot3(lx, ly, lz, c, 0.0, s), double(b[0]));
  p[1] = __dadd_rn(dot3(lx, ly, lz, 0.0, 1.0, 0.0), double(b[1]));
  p[2] = __dadd_rn(dot3(lx, ly, lz, -s, 0.0, c), double(b[2]));
}

// np.amin / np.amax: a NaN anywhere wins
__device__ __forceinline__ double nan_min(double a, double b) { return (isnan(a) || a < b) ? a : b; }
__device__ __forceinline__ double nan_max(double a, double b) { return (isnan(a) || a > b) ? a : b; }

__device__ __forceinline__ double warp_nan_min(double v) {
  for (int o = 16; o > 0; o >>= 1) v = nan_min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_nan_max(double v) {
  for (int o = 16; o > 0; o >>= 1) v = nan_max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One warp per detection: lanes on the 8 corners for the 2-D box, then strided over the frame's candidates for
// the in-box test and the cover rates.  Writes the row record (unconditionally) and keep[d].
__global__ void __launch_bounds__(kWarpsPerBlock * 32) kitti_rows_kernel(
    const float* __restrict__ boxes, const int32_t* __restrict__ labels, const float* __restrict__ scores,
    const int32_t* __restrict__ det_frame_ptr, int num_frames, int64_t num_dets, const float* __restrict__ xyz,
    const int32_t* __restrict__ cand_index, const int32_t* __restrict__ cand_frame_ptr, int num_classes,
    const double* __restrict__ cam_to_image, int rescore, int32_t* __restrict__ keep, double* __restrict__ rec,
    int32_t* __restrict__ bad_length) {
  const int lane = threadIdx.x & 31;
  const int64_t d = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (d >= num_dets) return;                                   // warp-uniform
  const int f = find_frame(det_frame_ptr, num_frames, d);
  float b[kBoxLen];
#pragma unroll
  for (int j = 0; j < kBoxLen; ++j) b[j] = boxes[d * kBoxLen + j];
  const double c = double(np_trig(b[6], 1)), s = double(np_trig(b[6], 0));

  // cam_points_to_image of corner lane % 8: [p | 1] . M^T, then / the third coordinate
  double p[3];
  corner(b, c, s, lane & 7, p);
  const double* m = cam_to_image + int64_t(f) * 12;
  double img[3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
    img[r] = __fma_rn(1.0, m[r * 4 + 3], dot3(p[0], p[1], p[2], m[r * 4 + 0], m[r * 4 + 1], m[r * 4 + 2]));
  const double u = __ddiv_rn(img[0], img[2]), v = __ddiv_rn(img[1], img[2]);
  const double xmin = warp_nan_min(u), xmax = warp_nan_max(u), ymin = warp_nan_min(v), ymax = warp_nan_max(v);
  // Python's max(a, 0.0) / min(a, 1242.0): the first argument unless the second compares greater / smaller
  const double cx0 = 0.0 > xmin ? 0.0 : xmin, cy0 = 0.0 > ymin ? 0.0 : ymin;
  const double cx1 = kImageWidth < xmax ? kImageWidth : xmax, cy1 = kImageHeight < ymax ? kImageHeight : ymax;
  const double covered = __ddiv_rn(__dmul_rn(__dsub_rn(cy1, cy0), __dsub_rn(cx1, cx0)),
                                   __dmul_rn(__dsub_rn(ymax, ymin), __dsub_rn(xmax, xmin)));
  const bool kept = !(__dsub_rn(1.0, covered) > kMaxTruncation);

  double score = double(scores[d]);
  int inside = 0;
  if (kept && rescore) {
    // box3d_to_normals: the face normals wx = p0 - p4, wy = p0 - p1, wz = p0 - p3 and the face offsets
    double p0[3], p1[3], p3[3], p4[3];
    corner(b, c, s, 0, p0);
    corner(b, c, s, 1, p1);
    corner(b, c, s, 3, p3);
    corner(b, c, s, 4, p4);
    double n[3][3], lo[3], hi[3];
    const double* other[3] = {p4, p1, p3};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
      for (int j = 0; j < 3; ++j) n[a][j] = __dsub_rn(p0[j], other[a][j]);
      lo[a] = dot3(n[a][0], n[a][1], n[a][2], other[a][0], other[a][1], other[a][2]);
      hi[a] = dot3(n[a][0], n[a][1], n[a][2], p0[0], p0[1], p0[2]);
    }
    double mn[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, mx[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
    const int begin = cand_frame_ptr[f], end = cand_frame_ptr[f + 1];
    for (int j = begin + lane; j < end; j += 32) {
      const float* q = xyz + int64_t(cand_index[j] / num_classes) * 3;
      const double q0 = double(q[0]), q1 = double(q[1]), q2 = double(q[2]);
      double pr[3];
      bool in = true;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        pr[a] = dot3(q0, q1, q2, n[a][0], n[a][1], n[a][2]);
        in = in && pr[a] > lo[a] && pr[a] < hi[a];
      }
      if (in) {
        ++inside;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          mn[a] = fmin(mn[a], pr[a]);
          mx[a] = fmax(mx[a], pr[a]);
        }
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      inside += __shfl_xor_sync(0xffffffffu, inside, o);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        mn[a] = fmin(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
        mx[a] = fmax(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
      }
    }
    if (inside > 0) {   // occlusion = x_cover_rate * y_cover_rate * z_cover_rate, then (1 + occlusion) * score
      double rate[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) rate[a] = __ddiv_rn(__dsub_rn(mx[a], mn[a]), __dsub_rn(hi[a], lo[a]));
      const double occlusion = __dmul_rn(__dmul_rn(rate[0], rate[1]), rate[2]);
      score = __dmul_rn(__dadd_rn(1.0, occlusion), score);
    }
  }
  if (lane != 0) return;
  keep[d] = kept ? 1 : 0;
  if (kept && !(b[3] > 0.0f)) atomicMin(bad_length, int32_t(d));   // run.py:395, on surviving rows only
  double* r = rec + d * PG_KITTI_ROW_FIELDS;
  r[0] = double(d);
  r[1] = double(f);
  r[2] = double(labels[d]);
#pragma unroll
  for (int j = 0; j < kBoxLen; ++j) r[3 + j] = double(b[j]);
  r[10] = cx0;
  r[11] = cy0;
  r[12] = cx1;
  r[13] = cy1;
  r[14] = score;
  r[15] = double(inside);
}

// rows in detection order; row_frame_ptr[f] = kept detections before frame f; status[0] = number of rows
__global__ void kitti_rows_compact_kernel(const int32_t* __restrict__ keep, const int32_t* __restrict__ keep_scan,
                                          const double* __restrict__ rec, int64_t num_dets,
                                          const int32_t* __restrict__ det_frame_ptr, int num_frames,
                                          double* __restrict__ out_rows, int32_t* __restrict__ out_row_frame_ptr,
                                          int32_t* __restrict__ status) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i <= num_frames) out_row_frame_ptr[i] = keep_scan[det_frame_ptr[i]];
  if (i == 0) status[0] = keep_scan[num_dets];
  if (i >= num_dets || !keep[i]) return;
  const int64_t o = keep_scan[i];
#pragma unroll
  for (int j = 0; j < PG_KITTI_ROW_FIELDS; ++j) out_rows[o * PG_KITTI_ROW_FIELDS + j] = rec[i * PG_KITTI_ROW_FIELDS + j];
}

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" int pg_kitti_rows(const float* boxes, const int32_t* labels, const float* scores, const int32_t* det_frame_ptr,
                             int32_t num_frames, int64_t num_dets, const float* xyz, const int32_t* cand_index,
                             const int32_t* cand_frame_ptr, int32_t num_classes, const double* cam_to_image,
                             int32_t flags, double* out_rows, int32_t* out_row_frame_ptr, int64_t* out_num_rows_host,
                             void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool rescore = (flags & PG_KITTI_ROWS_RESCORE) != 0;
  PG_REQUIRE(det_frame_ptr && cam_to_image && out_row_frame_ptr && out_num_rows_host, "pg_kitti_rows: null argument");
  PG_REQUIRE(num_frames >= 1 && num_dets >= 0 && num_dets < (int64_t(1) << 31), "pg_kitti_rows: bad sizes");
  PG_REQUIRE(num_classes >= 1, "pg_kitti_rows: num_classes must be >= 1");
  *out_num_rows_host = 0;
  if (num_dets == 0) {
    PG_CUDA_OK(cudaMemsetAsync(out_row_frame_ptr, 0, sizeof(int32_t) * (num_frames + 1), s));
    return PG_OK;
  }
  PG_REQUIRE(boxes && labels && scores && out_rows, "pg_kitti_rows: null detection argument");
  PG_REQUIRE(!rescore || (xyz && cand_index && cand_frame_ptr), "pg_kitti_rows: rescoring needs the candidates");
  Temp keep, keep_scan, rec, status;
  PG_CUDA_OK(keep.alloc(sizeof(int32_t) * (num_dets + 1), s));
  PG_CUDA_OK(keep_scan.alloc(sizeof(int32_t) * (num_dets + 1), s));
  PG_CUDA_OK(rec.alloc(sizeof(double) * num_dets * PG_KITTI_ROW_FIELDS, s));
  PG_CUDA_OK(status.alloc(sizeof(int32_t) * 2, s));
  PG_CUDA_OK(cudaMemsetAsync(keep.as<int32_t>() + num_dets, 0, sizeof(int32_t), s));
  PG_CUDA_OK(cudaMemsetAsync(status.as<int32_t>() + 1, 0x7f, sizeof(int32_t), s));   // no bad length: 0x7f7f7f7f
  kitti_rows_kernel<<<ceil_div(num_dets, kWarpsPerBlock), kWarpsPerBlock * 32, 0, s>>>(
      boxes, labels, scores, det_frame_ptr, num_frames, num_dets, xyz, cand_index, cand_frame_ptr, num_classes,
      cam_to_image, rescore ? 1 : 0, keep.as<int32_t>(), rec.as<double>(), status.as<int32_t>() + 1);
  PG_LAUNCH_CHECK();
  if (int rc = exclusive_sum(keep.as<int32_t>(), keep_scan.as<int32_t>(), num_dets + 1, s)) return rc;
  kitti_rows_compact_kernel<<<ceil_div(std::max<int64_t>(num_dets, num_frames + 1), 256), 256, 0, s>>>(
      keep.as<int32_t>(), keep_scan.as<int32_t>(), rec.as<double>(), num_dets, det_frame_ptr, num_frames, out_rows,
      out_row_frame_ptr, status.as<int32_t>());
  PG_LAUNCH_CHECK();
  int32_t h_status[2] = {0, 0};
  PG_CUDA_OK(cudaMemcpyAsync(h_status, status.ptr, sizeof(h_status), cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaStreamSynchronize(s));
  if (h_status[1] != 0x7f7f7f7f) {
    set_error("pg_kitti_rows: detection %d survives the truncation filter with length <= 0 (run.py:395 assert l > 0)",
              h_status[1]);
    return PG_ERR_INVALID_ARGUMENT;
  }
  *out_num_rows_host = h_status[0];
  return PG_OK;
}
