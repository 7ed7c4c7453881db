// KITTI object evaluation on the GPU: the twin of kitti_native_evaluation/src/evaluate_object_3d_offline.cpp.
//
// For every metric (image, bird's-eye view, 3D), class (car, pedestrian, cyclist) and difficulty (easy, moderate,
// hard) - 27 "segments" - the reference runs eval_class (:639-739): cleanData + computeStatistics without false
// positives on every frame to collect the TP scores, getThresholds to pick up to 41 score thresholds, then
// computeStatistics with false positives for every (frame, threshold), summed over frames into precision / AOS / AHS.
// All arithmetic is fp64, as there.
//
//   1. overlaps: every (detection, ground-truth row) pair of a frame once, for the three metrics
//      (imageBoxOverlap :224-258, groundBoxOverlap :291-311, box3DOverlap :314-341; DontCare rows with criterion 0)
//   2. cleanData (:378-451): the ignore state of every ground-truth row and detection per (class, difficulty)
//   3. recall pass: one thread per (frame, segment), the greedy sequential matching of the reference, emits TP scores
//   4. thresholds: TP scores sorted descending per segment (full 64-bit order-preserving key, then a stable pass by
//      segment), then getThresholds (:343-376) per segment
//   5. PR pass: one thread per (frame, segment, threshold) -> tp / fp / fn / similarity sums of that frame
//   6. the sums over frames, in frame order (the reference's order, so the double sums are its sums), then precision,
//      AOS / AHS and the suffix max (:703-734) per segment
#include <vector>

#include "pg_common.cuh"
#include "pg_geom.cuh"

namespace pg {
namespace {

constexpr int kMetrics = 3, kClasses = 3, kDiffs = 3;
constexpr int kSegments = kMetrics * kClasses * kDiffs;
constexpr int kPoints = 41;                       // N_SAMPLE_PTS
constexpr int kGtCols = 14, kDetCols = 15;
constexpr double kNoDetection = -10000000;
constexpr uint64_t kEmptyKey = ~0ull;

// class codes of the caller's rows (pg_kitti_eval's header comment)
enum { kCar = 0, kPedestrian = 1, kCyclist = 2, kVan = 3, kPersonSitting = 4, kDontCare = 5 };

__constant__ int kMinHeight[3] = {40, 25, 25};
__constant__ int kMaxOcclusion[3] = {0, 1, 2};
__constant__ double kMaxTruncation[3] = {0.15, 0.3, 0.5};

__device__ __forceinline__ double min_overlap(int cls) { return cls == kCar ? 0.7 : 0.5; }   // MIN_OVERLAP rows

// double <-> order-preserving uint64 (a < b iff ordered(a) < ordered(b), non-NaN values)
__device__ __forceinline__ uint64_t double_to_ordered(double d) {
  const uint64_t b = uint64_t(__double_as_longlong(d));
  return (b >> 63) ? ~b : (b | (1ull << 63));
}
__device__ __forceinline__ double ordered_to_double(uint64_t u) {
  return __longlong_as_double((long long)((u >> 63) ? (u & ~(1ull << 63)) : ~u));
}

// Per-frame layout: rows of frame f are [gt_ptr[f], gt_ptr[f+1]) and [det_ptr[f], det_ptr[f+1]); its pairs
// (detection j, ground truth i) are pair_ptr[f] + j * G_f + i; its assigned-detection bits are word_ptr[f] + j / 32.
struct Frames {
  const int64_t* gt_ptr;
  const int64_t* det_ptr;
  const int64_t* pair_ptr;
  const int64_t* word_ptr;
  int num_frames;
};

__device__ __forceinline__ int frame_of(const int64_t* ptr, int num_frames, int64_t row) {
  int lo = 0, hi = num_frames;   // ptr[lo] <= row < ptr[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (ptr[mid] <= row) lo = mid; else hi = mid;
  }
  return lo;
}

// toPolygon (:265-288): R = [[c, s], [-s, c]] times the (l, w) corner matrix, then + (t1, t3); fp64 as there,
// products and sums rounded separately (no contraction) like the host build
__device__ inline void make_footprint(double l, double w, double t1, double t3, double ry, BoxGeom* g) {
  const double c = cos(ry), s = sin(ry);
  const double lx[4] = {l / 2, l / 2, -l / 2, -l / 2}, lz[4] = {w / 2, -w / 2, -w / 2, w / 2};
  for (int k = 0; k < 4; ++k) {
    g->fx[k] = __dadd_rn(__dadd_rn(__dmul_rn(c, lx[k]), __dmul_rn(s, lz[k])), t1);
    g->fz[k] = __dadd_rn(__dadd_rn(__dmul_rn(-s, lx[k]), __dmul_rn(c, lz[k])), t3);
  }
  g->area = fabs(shoelace(g->fx, g->fz, 4));
}

// ---- 1. overlaps ---------------------------------------------------------------------------------------------------
// ov[m * num_pairs + pair]: criterion -1 (union) against ordinary rows, criterion 0 (detection area) against DontCare
__global__ void overlap_kernel(const double* __restrict__ gt, const int32_t* __restrict__ gt_class,
                               const double* __restrict__ det, Frames fr, int64_t num_pairs, double* __restrict__ ov) {
  const int64_t p = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= num_pairs) return;
  const int f = frame_of(fr.pair_ptr, fr.num_frames, p);
  const int64_t g0 = fr.gt_ptr[f], ng = fr.gt_ptr[f + 1] - g0;
  const int64_t q = p - fr.pair_ptr[f];
  const int64_t j = q / ng, i = q - j * ng;
  const double* g = gt + (g0 + i) * kGtCols;
  const double* d = det + (fr.det_ptr[f] + j) * kDetCols;
  const bool dc = gt_class[g0 + i] == kDontCare;

  // image: imageBoxOverlap(det box a, gt box b)
  double o_img = 0.0;
  {
    const double x1 = fmax(d[3], g[3]), y1 = fmax(d[4], g[4]);
    const double x2 = fmin(d[5], g[5]), y2 = fmin(d[6], g[6]);
    const double w = x2 - x1, h = y2 - y1;
    if (!(w <= 0 || h <= 0)) {
      const double inter = w * h;
      const double a_area = (d[5] - d[3]) * (d[6] - d[4]);
      const double b_area = (g[5] - g[3]) * (g[6] - g[4]);
      o_img = dc ? inter / a_area : inter / (a_area + b_area - inter);
    }
  }
  // ground and 3D: the footprint intersection of the ground-truth polygon clipped by the detection polygon
  BoxGeom gp, dp;
  make_footprint(g[9], g[8], g[10], g[12], g[13], &gp);
  make_footprint(d[9], d[8], d[10], d[12], d[13], &dp);
  const double inter_area = clipped_area(gp, dp);
  const double o_ground = dc ? inter_area / dp.area : inter_area / (gp.area + dp.area - inter_area);
  const double ymax = fmin(d[11], g[11]);
  const double ymin = fmax(d[11] - d[7], g[11] - g[7]);
  const double inter_vol = inter_area * fmax(0.0, ymax - ymin);
  const double det_vol = d[7] * d[9] * d[8];
  const double gt_vol = g[7] * g[9] * g[8];
  const double o_3d = dc ? inter_vol / det_vol : inter_vol / (det_vol + gt_vol - inter_vol);
  ov[p] = o_img;
  ov[num_pairs + p] = o_ground;
  ov[2 * num_pairs + p] = o_3d;
}

// ---- 2. cleanData --------------------------------------------------------------------------------------------------
// gt_state / det_state [(class * 3 + difficulty) * rows + row] = ignored_gt / ignored_det; n_gt[class * 3 + diff]
__global__ void clean_kernel(const double* __restrict__ gt, const int32_t* __restrict__ gt_class, int64_t num_gt,
                             const double* __restrict__ det, const int32_t* __restrict__ det_class, int64_t num_det,
                             int8_t* __restrict__ gt_state, int8_t* __restrict__ det_state, int32_t* __restrict__ n_gt) {
  const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r < num_gt) {
    const double* g = gt + r * kGtCols;
    const int code = gt_class[r];
    const double height = g[6] - g[4];
    for (int c = 0; c < kClasses; ++c) {
      int valid_class = -1;
      if (code == c) valid_class = 1;
      else if (c == kPedestrian && code == kPersonSitting) valid_class = 0;
      else if (c == kCar && code == kVan) valid_class = 0;
      for (int d = 0; d < kDiffs; ++d) {
        const bool ignore = g[1] > kMaxOcclusion[d] || g[0] > kMaxTruncation[d] || height <= kMinHeight[d];
        int8_t s = -1;
        if (valid_class == 1 && !ignore) {
          s = 0;
          atomicAdd(&n_gt[c * kDiffs + d], 1);
        } else if (valid_class == 0 || (ignore && valid_class == 1)) {
          s = 1;
        }
        gt_state[(c * kDiffs + d) * num_gt + r] = s;
      }
    }
  } else if (r < num_gt + num_det) {
    const int64_t j = r - num_gt;
    const double* d = det + j * kDetCols;
    const int code = det_class[j];
    const int32_t height = int32_t(fabs(d[4] - d[6]));
    for (int c = 0; c < kClasses; ++c)
      for (int k = 0; k < kDiffs; ++k)
        det_state[(c * kDiffs + k) * num_det + j] = height < kMinHeight[k] ? 1 : (code == c ? 0 : -1);
  }
}

// ---- 3 / 5. computeStatistics (:453-633) -------------------------------------------------------------------------------
struct Inputs {
  const double* gt;
  const int32_t* gt_class;
  const double* det;
  const int8_t* gt_state;
  const int8_t* det_state;
  const double* ov;
  int64_t num_gt, num_det, num_pairs;
  Frames fr;
};

struct Stat {
  int32_t tp = 0, fp = 0, fn = 0;
  double similarity = 0.0, similarity_ground = 0.0;
};

// segment s = (metric * 3 + class) * 3 + difficulty.  FP = compute_fp.  assigned: zeroed bits, one per detection
// of the frame.  Without FP, each TP's score goes to tp_scores[k] for the k-th TP.
template <bool FP>
__device__ Stat compute_statistics(const Inputs& in, int f, int seg, double thresh, bool compute_aos,
                                   bool compute_aos_ground, uint32_t* __restrict__ assigned, double* tp_scores) {
  const int metric = seg / (kClasses * kDiffs), cls = (seg / kDiffs) % kClasses;
  const int cd = seg % (kClasses * kDiffs);
  const double min_ov = min_overlap(cls);
  const int64_t g0 = in.fr.gt_ptr[f], ng = in.fr.gt_ptr[f + 1] - g0;
  const int64_t d0 = in.fr.det_ptr[f], nd = in.fr.det_ptr[f + 1] - d0;
  const double* ov = in.ov + int64_t(metric) * in.num_pairs + in.fr.pair_ptr[f];
  const int8_t* ig_gt = in.gt_state + cd * in.num_gt + g0;
  const int8_t* ig_det = in.det_state + cd * in.num_det + d0;
  const double* det = in.det + d0 * kDetCols;
  Stat st;
  for (int64_t i = 0; i < ng; ++i) {
    const int ig = ig_gt[i];
    if (ig == -1) continue;
    int64_t det_idx = -1;
    double valid_detection = kNoDetection, max_overlap = 0;
    bool assigned_ignored_det = false;
    for (int64_t j = 0; j < nd; ++j) {
      const int id = ig_det[j];
      if (id == -1) continue;
      if ((assigned[j >> 5] >> (j & 31)) & 1u) continue;
      const double score = det[j * kDetCols + 14];
      if (FP && score < thresh) continue;
      const double overlap = ov[j * ng + i];
      if (!FP) {
        if (overlap > min_ov && score > valid_detection) {
          det_idx = j;
          valid_detection = score;
        }
      } else if (overlap > min_ov && (overlap > max_overlap || assigned_ignored_det) && id == 0) {
        max_overlap = overlap;
        det_idx = j;
        valid_detection = 1;
        assigned_ignored_det = false;
      } else if (overlap > min_ov && valid_detection == kNoDetection && id == 1) {
        det_idx = j;
        valid_detection = 1;
        assigned_ignored_det = true;
      }
    }
    if (valid_detection == kNoDetection && ig == 0) {
      st.fn++;
    } else if (valid_detection != kNoDetection && (ig == 1 || ig_det[det_idx] == 1)) {
      assigned[det_idx >> 5] |= 1u << (det_idx & 31);
    } else if (valid_detection != kNoDetection) {
      const double* g = in.gt + (g0 + i) * kGtCols;
      const double* d = det + det_idx * kDetCols;
      if (!FP) tp_scores[st.tp] = d[14];
      st.tp++;
      if (compute_aos) st.similarity += (1.0 + cos(g[2] - d[2])) / 2.0;
      if (compute_aos_ground) st.similarity_ground += (1.0 + cos(fabs(g[13] - d[13]))) / 2.0;
      assigned[det_idx >> 5] |= 1u << (det_idx & 31);
    }
  }
  if (FP) {
    for (int64_t j = 0; j < nd; ++j) {
      const int id = ig_det[j];
      const bool a = (assigned[j >> 5] >> (j & 31)) & 1u;
      if (!(a || id == -1 || id == 1 || det[j * kDetCols + 14] < thresh)) st.fp++;
    }
    int32_t nstuff = 0;
    for (int64_t i = 0; i < ng; ++i) {
      if (in.gt_class[g0 + i] != kDontCare) continue;
      for (int64_t j = 0; j < nd; ++j) {
        if ((assigned[j >> 5] >> (j & 31)) & 1u) continue;
        const int id = ig_det[j];
        if (id == -1 || id == 1) continue;
        if (det[j * kDetCols + 14] < thresh) continue;
        if (ov[j * ng + i] > min_ov) {
          assigned[j >> 5] |= 1u << (j & 31);
          nstuff++;
        }
      }
    }
    st.fp -= nstuff;
    if (compute_aos && !(st.tp > 0 || st.fp > 0)) st.similarity = -1;
    if (compute_aos_ground && !(st.tp > 0 || st.fp > 0)) st.similarity_ground = -1;
  }
  return st;
}

// ---- 3. recall pass --------------------------------------------------------------------------------------------------
// task = f * 27 + seg.  TP scores -> keys[seg * num_gt + gt_ptr[f] + k] (descending-order key), vals = the slot
__global__ void recall_kernel(Inputs in, uint32_t* __restrict__ bits, int64_t words, uint64_t* __restrict__ keys,
                              int32_t* __restrict__ vals, int32_t* __restrict__ tp_count) {
  const int64_t task = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (task >= int64_t(in.fr.num_frames) * kSegments) return;
  const int f = int(task / kSegments), seg = int(task % kSegments);
  const int64_t slot0 = seg * in.num_gt + in.fr.gt_ptr[f];
  // the scores are staged in the key array, then turned into keys in place
  double* scores = reinterpret_cast<double*>(keys + slot0);
  const Stat st = compute_statistics<false>(in, f, seg, 0.0, false, false, bits + seg * words + in.fr.word_ptr[f], scores);
  for (int k = 0; k < st.tp; ++k) {
    keys[slot0 + k] = ~double_to_ordered(scores[k]);
    vals[slot0 + k] = int32_t(slot0 + k);
  }
  tp_count[seg * in.fr.num_frames + f] = st.tp;
}

// ---- 4. thresholds -------------------------------------------------------------------------------------------------
// second sort key: the segment of each score-sorted entry (empty slots: segment 27, sorted last)
__global__ void segment_key_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals, int64_t n,
                                   int64_t num_gt, uint64_t* __restrict__ seg_keys, int32_t* __restrict__ pos) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  seg_keys[i] = keys[i] == kEmptyKey ? uint64_t(kSegments) : uint64_t(vals[i] / num_gt);
  pos[i] = int32_t(i);
}

// one block per segment: TP scores over all frames (integer sums: any order gives the same result)
__global__ void segment_count_kernel(const int32_t* __restrict__ tp_count, int num_frames, int32_t* __restrict__ n_tp) {
  __shared__ int32_t s;
  if (threadIdx.x == 0) s = 0;
  __syncthreads();
  int32_t part = 0;
  for (int f = threadIdx.x; f < num_frames; f += blockDim.x) part += tp_count[blockIdx.x * num_frames + f];
  atomicAdd(&s, part);
  __syncthreads();
  if (threadIdx.x == 0) n_tp[blockIdx.x] = s;
}

// getThresholds (:343-376) per segment on its TP scores v (descending).  The skip test at i,
// (r_recall - current_recall) < (current_recall - l_recall), turns false as i grows and then stays false (l and r
// grow with i), so the next accepted index is found by bisection.  At most 41 thresholds are kept: the reference
// writes past its 41-entry arrays when there are more (undefined behaviour); here the later ones are dropped.
__global__ void threshold_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ order,
                                 const int32_t* __restrict__ n_tp, const int32_t* __restrict__ n_gt,
                                 double* __restrict__ thr, int32_t* __restrict__ num_thr) {
  const int seg = threadIdx.x;
  if (seg >= kSegments) return;
  int64_t start = 0;
  for (int s = 0; s < seg; ++s) start += n_tp[s];
  const int64_t n = n_tp[seg];
  const double n_groundtruth = double(n_gt[seg % (kClasses * kDiffs)]);
  double current_recall = 0;
  int k = 0;
  for (int64_t i = 0; i < n && k < kPoints;) {
    int64_t lo = i, hi = n - 1;           // index n - 1 is always taken
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      const double l_recall = double(mid + 1) / n_groundtruth, r_recall = double(mid + 2) / n_groundtruth;
      if ((r_recall - current_recall) < (current_recall - l_recall)) lo = mid + 1; else hi = mid;
    }
    thr[seg * kPoints + k++] = ordered_to_double(~keys[order[start + lo]]);
    current_recall += 1.0 / (double(kPoints) - 1.0);
    i = lo + 1;
  }
  num_thr[seg] = k;
}

// ---- 5. PR pass --------------------------------------------------------------------------------------------------
// task = f * 27 * 41 + seg * 41 + t; results at the same index
__global__ void pr_kernel(Inputs in, const double* __restrict__ thr, const int32_t* __restrict__ num_thr,
                          int compute_aos, uint32_t* __restrict__ bits, int64_t words, int32_t* __restrict__ tp,
                          int32_t* __restrict__ fp, int32_t* __restrict__ fn, double* __restrict__ sim,
                          double* __restrict__ sim_ground) {
  const int64_t task = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (task >= int64_t(in.fr.num_frames) * kSegments * kPoints) return;
  const int f = int(task / (kSegments * kPoints));
  const int st_idx = int(task % (kSegments * kPoints));
  const int seg = st_idx / kPoints, t = st_idx % kPoints;
  if (t >= num_thr[seg]) return;
  const bool image = seg < kClasses * kDiffs;
  const Stat st = compute_statistics<true>(in, f, seg, thr[st_idx], image && compute_aos, !image,
                                           bits + st_idx * words + in.fr.word_ptr[f], nullptr);
  tp[task] = st.tp;
  fp[task] = st.fp;
  fn[task] = st.fn;
  sim[task] = st.similarity;
  sim_ground[task] = st.similarity_ground;
}

// ---- 6. sums over frames (frame order), precision / AOS / AHS, suffix max ------------------------------------------
__global__ void frame_sum_kernel(const int32_t* __restrict__ num_thr, int num_frames, const int32_t* __restrict__ tp,
                                 const int32_t* __restrict__ fp, const int32_t* __restrict__ fn,
                                 const double* __restrict__ sim, const double* __restrict__ sim_ground,
                                 int32_t* __restrict__ tp_sum, int32_t* __restrict__ fp_sum, int32_t* __restrict__ fn_sum,
                                 double* __restrict__ sim_sum, double* __restrict__ sim_ground_sum) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= kSegments * kPoints) return;
  int32_t a = 0, b = 0, c = 0;
  double s = 0, sg = 0;
  if (k % kPoints < num_thr[k / kPoints]) {
    for (int f = 0; f < num_frames; ++f) {
      const int64_t i = int64_t(f) * kSegments * kPoints + k;
      a += tp[i];
      b += fp[i];
      c += fn[i];
      if (sim[i] != -1) s += sim[i];
      if (sim_ground[i] != -1) sg += sim_ground[i];
    }
  }
  tp_sum[k] = a;
  fp_sum[k] = b;
  fn_sum[k] = c;
  sim_sum[k] = s;
  sim_ground_sum[k] = sg;
}

// *max_element(v + i, v + n): the first element no later element exceeds under <
__device__ __forceinline__ double max_element(const double* v, int i, int n) {
  int largest = i;
  for (int j = i + 1; j < n; ++j)
    if (v[largest] < v[j]) largest = j;
  return v[largest];
}

__global__ void precision_kernel(const int32_t* __restrict__ num_thr, const int32_t* __restrict__ tp,
                                 const int32_t* __restrict__ fp, const double* __restrict__ sim,
                                 const double* __restrict__ sim_ground, int compute_aos, double* __restrict__ precision,
                                 double* __restrict__ aos, double* __restrict__ ahs) {
  const int seg = threadIdx.x;
  if (seg >= kSegments) return;
  const bool image = seg < kClasses * kDiffs;
  const bool do_aos = image && compute_aos, do_ahs = !image;
  double* p = precision + seg * kPoints;
  double* a = aos + seg * kPoints;
  double* h = ahs + seg * kPoints;
  const int n = num_thr[seg];
  for (int i = 0; i < kPoints; ++i) p[i] = a[i] = h[i] = 0.0;
  for (int i = 0; i < n; ++i) {
    const int k = seg * kPoints + i;
    const double den = double(tp[k] + fp[k]);
    p[i] = tp[k] / den;
    if (do_aos) a[i] = sim[k] / den;
    if (do_ahs) h[i] = sim_ground[k] / den;
  }
  for (int i = 0; i < n; ++i) {
    p[i] = max_element(p, i, kPoints);
    if (do_aos) a[i] = max_element(a, i, kPoints);
    if (do_ahs) h[i] = max_element(h, i, kPoints);
  }
}

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" int pg_kitti_eval(const double* gt, const int32_t* gt_class, const double* det, const int32_t* det_class,
                             const int64_t* gt_frame_ptr_host, const int64_t* det_frame_ptr_host, int32_t num_frames,
                             int32_t flags, double* out_precision_host, double* out_aos_host, double* out_ahs_host,
                             int32_t* out_num_thresholds_host, int32_t* out_tp_host, int32_t* out_fp_host,
                             int32_t* out_fn_host, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(gt_frame_ptr_host && det_frame_ptr_host && out_precision_host && out_aos_host && out_ahs_host &&
                 out_num_thresholds_host && out_tp_host && out_fp_host && out_fn_host,
             "pg_kitti_eval: null argument");
  PG_REQUIRE(num_frames >= 1, "pg_kitti_eval: num_frames must be >= 1");
  const int64_t num_gt = gt_frame_ptr_host[num_frames], num_det = det_frame_ptr_host[num_frames];
  PG_REQUIRE(gt_frame_ptr_host[0] == 0 && det_frame_ptr_host[0] == 0, "pg_kitti_eval: frame pointers must start at 0");
  PG_REQUIRE((gt && gt_class) || num_gt == 0, "pg_kitti_eval: null ground truth");
  PG_REQUIRE((det && det_class) || num_det == 0, "pg_kitti_eval: null detections");
  // the TP-score slots (27 per ground-truth row) are addressed by int32 sort values
  PG_REQUIRE(num_gt * kSegments < (int64_t(1) << 31), "pg_kitti_eval: too many ground-truth rows (%lld)",
             (long long)num_gt);

  // per-frame offsets, computed on the host from the frame pointers
  std::vector<int64_t> host(4 * (int64_t(num_frames) + 1));
  int64_t* h_gt = host.data();
  int64_t* h_det = h_gt + num_frames + 1;
  int64_t* h_pair = h_det + num_frames + 1;
  int64_t* h_word = h_pair + num_frames + 1;
  h_pair[0] = h_word[0] = 0;
  for (int f = 0; f <= num_frames; ++f) {
    h_gt[f] = gt_frame_ptr_host[f];
    h_det[f] = det_frame_ptr_host[f];
    if (f == num_frames) break;
    const int64_t ng = gt_frame_ptr_host[f + 1] - gt_frame_ptr_host[f];
    const int64_t nd = det_frame_ptr_host[f + 1] - det_frame_ptr_host[f];
    PG_REQUIRE(ng >= 0 && nd >= 0, "pg_kitti_eval: frame pointers must not decrease (frame %d)", f);
    h_pair[f + 1] = h_pair[f] + ng * nd;
    h_word[f + 1] = h_word[f] + (nd + 31) / 32;
  }
  const int64_t num_pairs = h_pair[num_frames], words = h_word[num_frames];

  Temp offsets, ov, gt_state, det_state, n_gt, bits, keys, vals, keys_s, vals_s, seg_keys, seg_keys_s, pos, order;
  Temp tp_count, n_tp, thr, num_thr, tp, fp, fn, sim, sim_g, tp_sum, fp_sum, fn_sum, sim_sum, sim_g_sum, prec, aos, ahs;
  PG_CUDA_OK(offsets.alloc(sizeof(int64_t) * host.size(), s));
  PG_CUDA_OK(cudaMemcpyAsync(offsets.ptr, host.data(), sizeof(int64_t) * host.size(), cudaMemcpyHostToDevice, s));
  const int64_t* d_off = offsets.as<int64_t>();
  Frames fr{d_off, d_off + num_frames + 1, d_off + 2 * (num_frames + 1), d_off + 3 * (num_frames + 1), num_frames};

  const int64_t slots = kSegments * num_gt;
  const int64_t pr_tasks = int64_t(num_frames) * kSegments * kPoints;
  const int64_t bit_words = words * kSegments * kPoints;
  PG_CUDA_OK(ov.alloc(sizeof(double) * 3 * num_pairs, s));
  PG_CUDA_OK(gt_state.alloc(kClasses * kDiffs * num_gt, s));
  PG_CUDA_OK(det_state.alloc(kClasses * kDiffs * num_det, s));
  PG_CUDA_OK(n_gt.alloc(sizeof(int32_t) * kClasses * kDiffs, s));
  PG_CUDA_OK(bits.alloc(sizeof(uint32_t) * bit_words, s));
  PG_CUDA_OK(keys.alloc(sizeof(uint64_t) * slots, s));
  PG_CUDA_OK(vals.alloc(sizeof(int32_t) * slots, s));
  PG_CUDA_OK(keys_s.alloc(sizeof(uint64_t) * slots, s));
  PG_CUDA_OK(vals_s.alloc(sizeof(int32_t) * slots, s));
  PG_CUDA_OK(seg_keys.alloc(sizeof(uint64_t) * slots, s));
  PG_CUDA_OK(seg_keys_s.alloc(sizeof(uint64_t) * slots, s));
  PG_CUDA_OK(pos.alloc(sizeof(int32_t) * slots, s));
  PG_CUDA_OK(order.alloc(sizeof(int32_t) * slots, s));
  PG_CUDA_OK(tp_count.alloc(sizeof(int32_t) * kSegments * num_frames, s));
  PG_CUDA_OK(n_tp.alloc(sizeof(int32_t) * kSegments, s));
  PG_CUDA_OK(thr.alloc(sizeof(double) * kSegments * kPoints, s));
  PG_CUDA_OK(num_thr.alloc(sizeof(int32_t) * kSegments, s));
  PG_CUDA_OK(tp.alloc(sizeof(int32_t) * pr_tasks, s));
  PG_CUDA_OK(fp.alloc(sizeof(int32_t) * pr_tasks, s));
  PG_CUDA_OK(fn.alloc(sizeof(int32_t) * pr_tasks, s));
  PG_CUDA_OK(sim.alloc(sizeof(double) * pr_tasks, s));
  PG_CUDA_OK(sim_g.alloc(sizeof(double) * pr_tasks, s));
  PG_CUDA_OK(tp_sum.alloc(sizeof(int32_t) * kSegments * kPoints, s));
  PG_CUDA_OK(fp_sum.alloc(sizeof(int32_t) * kSegments * kPoints, s));
  PG_CUDA_OK(fn_sum.alloc(sizeof(int32_t) * kSegments * kPoints, s));
  PG_CUDA_OK(sim_sum.alloc(sizeof(double) * kSegments * kPoints, s));
  PG_CUDA_OK(sim_g_sum.alloc(sizeof(double) * kSegments * kPoints, s));
  PG_CUDA_OK(prec.alloc(sizeof(double) * kSegments * kPoints, s));
  PG_CUDA_OK(aos.alloc(sizeof(double) * kSegments * kPoints, s));
  PG_CUDA_OK(ahs.alloc(sizeof(double) * kSegments * kPoints, s));
  PG_CUDA_OK(cudaMemsetAsync(n_gt.ptr, 0, sizeof(int32_t) * kClasses * kDiffs, s));
  PG_CUDA_OK(cudaMemsetAsync(keys.ptr, 0xff, sizeof(uint64_t) * slots, s));     // kEmptyKey
  PG_CUDA_OK(cudaMemsetAsync(vals.ptr, 0, sizeof(int32_t) * slots, s));
  PG_CUDA_OK(cudaMemsetAsync(n_tp.ptr, 0, sizeof(int32_t) * kSegments, s));

  const Inputs in{gt, gt_class, det, gt_state.as<int8_t>(), det_state.as<int8_t>(), ov.as<double>(),
                  num_gt, num_det, num_pairs, fr};
  if (num_pairs > 0) {
    overlap_kernel<<<ceil_div(num_pairs, 128), 128, 0, s>>>(gt, gt_class, det, fr, num_pairs, ov.as<double>());
    PG_LAUNCH_CHECK();
  }
  if (num_gt + num_det > 0) {
    clean_kernel<<<ceil_div(num_gt + num_det, 128), 128, 0, s>>>(gt, gt_class, num_gt, det, det_class, num_det,
                                                                 gt_state.as<int8_t>(), det_state.as<int8_t>(),
                                                                 n_gt.as<int32_t>());
    PG_LAUNCH_CHECK();
  }
  // recall pass (its bit region is the first 27 * words words of the PR pass's)
  PG_CUDA_OK(cudaMemsetAsync(bits.ptr, 0, sizeof(uint32_t) * words * kSegments, s));
  recall_kernel<<<ceil_div(int64_t(num_frames) * kSegments, 128), 128, 0, s>>>(
      in, bits.as<uint32_t>(), words, keys.as<uint64_t>(), vals.as<int32_t>(), tp_count.as<int32_t>());
  PG_LAUNCH_CHECK();
  segment_count_kernel<<<kSegments, 256, 0, s>>>(tp_count.as<int32_t>(), num_frames, n_tp.as<int32_t>());
  PG_LAUNCH_CHECK();
  if (slots > 0) {
    // sort (getThresholds :350): score descending by the full 64-bit key, then stably by segment
    if (int rc = sort_pairs(keys.as<uint64_t>(), keys_s.as<uint64_t>(), vals.as<int32_t>(), vals_s.as<int32_t>(), slots,
                            64, s))
      return rc;
    segment_key_kernel<<<ceil_div(slots, 256), 256, 0, s>>>(keys_s.as<uint64_t>(), vals_s.as<int32_t>(), slots, num_gt,
                                                            seg_keys.as<uint64_t>(), pos.as<int32_t>());
    PG_LAUNCH_CHECK();
    if (int rc = sort_pairs(seg_keys.as<uint64_t>(), seg_keys_s.as<uint64_t>(), pos.as<int32_t>(), order.as<int32_t>(),
                            slots, 5, s))
      return rc;
  }
  threshold_kernel<<<1, 32, 0, s>>>(keys_s.as<uint64_t>(), order.as<int32_t>(), n_tp.as<int32_t>(), n_gt.as<int32_t>(),
                                    thr.as<double>(), num_thr.as<int32_t>());
  PG_LAUNCH_CHECK();
  // PR pass
  PG_CUDA_OK(cudaMemsetAsync(bits.ptr, 0, sizeof(uint32_t) * bit_words, s));
  pr_kernel<<<ceil_div(pr_tasks, 128), 128, 0, s>>>(in, thr.as<double>(), num_thr.as<int32_t>(), flags & PG_KITTI_EVAL_AOS,
                                                    bits.as<uint32_t>(), words, tp.as<int32_t>(), fp.as<int32_t>(),
                                                    fn.as<int32_t>(), sim.as<double>(), sim_g.as<double>());
  PG_LAUNCH_CHECK();
  frame_sum_kernel<<<ceil_div(kSegments * kPoints, 64), 64, 0, s>>>(
      num_thr.as<int32_t>(), num_frames, tp.as<int32_t>(), fp.as<int32_t>(), fn.as<int32_t>(), sim.as<double>(),
      sim_g.as<double>(), tp_sum.as<int32_t>(), fp_sum.as<int32_t>(), fn_sum.as<int32_t>(), sim_sum.as<double>(),
      sim_g_sum.as<double>());
  PG_LAUNCH_CHECK();
  precision_kernel<<<1, 32, 0, s>>>(num_thr.as<int32_t>(), tp_sum.as<int32_t>(), fp_sum.as<int32_t>(),
                                    sim_sum.as<double>(), sim_g_sum.as<double>(), flags & PG_KITTI_EVAL_AOS,
                                    prec.as<double>(), aos.as<double>(), ahs.as<double>());
  PG_LAUNCH_CHECK();

  const size_t curve = sizeof(double) * kSegments * kPoints, counts = sizeof(int32_t) * kSegments * kPoints;
  PG_CUDA_OK(cudaMemcpyAsync(out_precision_host, prec.ptr, curve, cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaMemcpyAsync(out_aos_host, aos.ptr, curve, cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaMemcpyAsync(out_ahs_host, ahs.ptr, curve, cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaMemcpyAsync(out_num_thresholds_host, num_thr.ptr, sizeof(int32_t) * kSegments, cudaMemcpyDeviceToHost,
                             s));
  PG_CUDA_OK(cudaMemcpyAsync(out_tp_host, tp_sum.ptr, counts, cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaMemcpyAsync(out_fp_host, fp_sum.ptr, counts, cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaMemcpyAsync(out_fn_host, fn_sum.ptr, counts, cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaStreamSynchronize(s));
  return PG_OK;
}
