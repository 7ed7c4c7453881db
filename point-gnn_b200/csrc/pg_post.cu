// Box decoding + NMS / merge / rescore on the GPU: the step right after the message-passing path.
//
// Replaces (for batches of frames, everything staying on the device until one final read-back)
//   run.py:265-296            candidate selection: class c of vertex v iff 0 < c < C-1 and prob > 1/C,
//                             "vertical" labels folded onto their class (2->1, 4->3, 6->5)
//   box_encoding.py:265-299   classaware_all_class_box_decoding (float32 arithmetic, as NumPy does there)
//   nms.py:9-27               boxes_3d_to_corners
//   nms.py:64-88              overlapped_boxes_3d_fast_poly: 3-D IoU, footprints intersected as convex
//                             polygons (the reference uses shapely; Sutherland-Hodgman in fp64 here)
//   nms.py:90-107, 133-170, 172-240, 256-270
//                             score sort + greedy per-class suppression in which the kept box becomes the
//                             coordinate-wise MEDIAN of itself and the boxes it suppresses (merge) and its
//                             score grows by sum_j score_j * IoU(median box, box_j) (rescore)
//
// The reference's loop is sequential over boxes; here only the cheap part is:
//   1. candidates: pg_postprocess flags, scans, decodes (decode_box, the rule pg_decode_boxes uses) and scatters them
//      in ascending (vertex, class) order per frame; pg_nms_boxes_3d takes the caller's boxes as they are.  Either
//      way the result is one Candidates set that nms_stage runs stages 2-6 on.
//   2. stable radix sort by (frame, score desc)  = bboxes_sort, ties in ascending candidate position
//   3. geometry per candidate (corners, extents) and the pairwise same-class "IoU > threshold" bit matrix,
//      all pairs of a frame in parallel over the whole GPU
//   4. sweep: one warp per frame walks the sorted list with bit operations only (who is kept, whom it removes)
//   5. merge + rescore: one block per kept box (median by rank selection, IoU with the merged box)
//   6. compaction of the kept boxes per frame
#include "pg_common.cuh"
#include "pg_geom.cuh"

namespace pg {
namespace {

constexpr int kMaxClasses = 16;
constexpr int kBoxLen = 7;

struct ClassTable {
  float l[kMaxClasses], h[kMaxClasses], w[kMaxClasses], yaw0[kMaxClasses];
  int decoded[kMaxClasses];
};

__device__ __forceinline__ int fold_label(int c) { return (c == 2 || c == 4 || c == 6) ? c - 1 : c; }

// ---- 1. candidates ---------------------------------------------------------------------------------
__global__ void flag_candidates_kernel(const float* __restrict__ probs, int64_t num_vertices, int num_classes,
                                       int32_t* __restrict__ flags) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= num_vertices * num_classes) return;
  const int c = int(i % num_classes);
  // run.py:281-282; the comparison is made in double like NumPy's float32-array > Python-float (value-based cast)
  flags[i] = (c > 0 && c < num_classes - 1 && double(probs[i]) > 1.0 / double(num_classes)) ? 1 : 0;
}

// classaware_all_class_box_decoding of (vertex, class c): the encoding e [7] at the vertex position p [3] -> b [7]
// (box_encoding.py:276-298, float32 arithmetic in NumPy's order)
__device__ __forceinline__ void decode_box(const float* __restrict__ e, const float* __restrict__ p, const ClassTable& tab,
                                           int c, float* b) {
#pragma unroll
  for (int j = 0; j < kBoxLen; ++j) b[j] = e[j];
  if (tab.decoded[c]) {
    const float pi4 = float(M_PI * 0.25), pi2 = float(0.5 * M_PI);
    b[0] = __fmul_rn(e[0], tab.l[c]);
    b[1] = __fmul_rn(e[1], tab.h[c]);
    b[2] = __fmul_rn(e[2], tab.w[c]);
    b[3] = __fmul_rn(expf(e[3]), tab.l[c]);
    b[4] = __fmul_rn(expf(e[4]), tab.h[c]);
    b[5] = __fmul_rn(expf(e[5]), tab.w[c]);
    b[6] = __fmul_rn(e[6], pi4);
    if (tab.yaw0[c] != 0.0f) b[6] = __fadd_rn(b[6], pi2);
  }
  b[0] = __fadd_rn(b[0], p[0]);
  b[1] = __fadd_rn(b[1], p[1]);
  b[2] = __fadd_rn(b[2], p[2]);
}

// sort key of a candidate: frame, then score descending
__device__ __forceinline__ uint64_t sort_key(int frame, float score) {
  return (uint64_t(uint32_t(frame)) << 32) | uint64_t(~float_to_ordered(score));
}

// decode + scatter in flat (vertex, class) order, with the sort key
__global__ void decode_scatter_kernel(const float* __restrict__ probs, const float* __restrict__ enc,
                                      const float* __restrict__ xyz, const int32_t* __restrict__ frame_ptr,
                                      int num_frames, int64_t num_vertices, int num_classes, ClassTable tab,
                                      const int32_t* __restrict__ flags, const int32_t* __restrict__ slot_of,
                                      float* __restrict__ cand_box, float* __restrict__ cand_score,
                                      int32_t* __restrict__ cand_label, int32_t* __restrict__ cand_index,
                                      uint64_t* __restrict__ keys, int32_t* __restrict__ vals,
                                      int32_t* __restrict__ frame_count) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= num_vertices * num_classes) return;
  if (!flags[i]) return;
  const int64_t v = i / num_classes;
  const int c = int(i - v * num_classes);
  const int s = slot_of[i];
  float b[kBoxLen];
  decode_box(enc + i * kBoxLen, xyz + 3 * v, tab, c, b);
#pragma unroll
  for (int j = 0; j < kBoxLen; ++j) cand_box[int64_t(s) * kBoxLen + j] = b[j];
  const float p = probs[i];
  cand_score[s] = p;
  cand_label[s] = fold_label(c);
  cand_index[s] = int32_t(i);
  const int f = find_frame(frame_ptr, num_frames, v);
  keys[s] = sort_key(f, p);
  vals[s] = s;
  atomicAdd(&frame_count[f], 1);
}

// sort keys of caller-provided candidates (pg_nms_boxes_3d), value = position
__global__ void candidate_keys_kernel(const float* __restrict__ score, const int32_t* __restrict__ frame_ptr, int num_frames,
                                      int64_t n, uint64_t* __restrict__ keys, int32_t* __restrict__ vals,
                                      int32_t* __restrict__ frame_count, int32_t* __restrict__ index) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = find_frame(frame_ptr, num_frames, i);
  keys[i] = sort_key(f, score[i]);
  vals[i] = int32_t(i);
  index[i] = int32_t(i);
  atomicAdd(&frame_count[f], 1);
}

// classaware_all_class_box_decoding for every (vertex, class) pair -> [K, C, 7]
__global__ void decode_all_kernel(const float* __restrict__ enc, const float* __restrict__ xyz, int64_t num_vertices,
                                  int num_classes, ClassTable tab, float* __restrict__ out) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= num_vertices * num_classes) return;
  const int64_t v = i / num_classes;
  const int c = int(i - v * num_classes);
  float b[kBoxLen];
  decode_box(enc + i * kBoxLen, xyz + 3 * v, tab, c, b);
#pragma unroll
  for (int j = 0; j < kBoxLen; ++j) out[i * kBoxLen + j] = b[j];
}

__global__ void fill_tail_keys_kernel(const int32_t* __restrict__ total, int64_t capacity, uint64_t* __restrict__ keys,
                                      int32_t* __restrict__ vals) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= capacity || i < *total) return;
  keys[i] = ~0ull;
  vals[i] = int32_t(i);
}

// ---- 2. sort ---------------------------------------------------------------------------------------
// one thread: ptr = exclusive scan of the per-frame counts (ptr[num_frames] = all candidates), and
// counts[num_frames] = the largest count
__global__ void frame_ptr_kernel(int32_t* __restrict__ counts, int num_frames, int32_t* __restrict__ ptr) {
  int acc = 0, widest = 0;
  for (int f = 0; f < num_frames; ++f) {
    ptr[f] = acc;
    acc += counts[f];
    widest = max(widest, counts[f]);
  }
  ptr[num_frames] = acc;
  counts[num_frames] = widest;
}

// ---- 3. geometry -----------------------------------------------------------------------------------
// nms.py:9-27: trigonometry and the half extents in float32 (the box dtype), the rest in float64
// appr > 0: the corners are converted to integer "pixels" first, np.int32(corners * appr) (bboxes_nms, nms.py:114)
__device__ inline void make_geom(const float* b, BoxGeom* g, double appr = 0.0) {
  const float x = b[0], y = b[1], z = b[2], l = b[3], h = b[4], w = b[5], yaw = b[6];
  const double c = double(cosf(yaw)), s = double(sinf(yaw));
  const double hl = double(l / 2.0f), hw = double(w / 2.0f);
  const double lx[4] = {hl, hl, -hl, -hl}, lz[4] = {hw, -hw, -hw, hw};
  g->xmin = g->zmin = DBL_MAX;
  g->xmax = g->zmax = -DBL_MAX;
  for (int i = 0; i < 4; ++i) {
    g->fx[i] = (lx[i] * c + 0.0) + lz[i] * s + double(x);
    g->fz[i] = (lx[i] * (-s) + 0.0) + lz[i] * c + double(z);
    if (appr > 0.0) {
      g->fx[i] = trunc(g->fx[i] * appr);
      g->fz[i] = trunc(g->fz[i] * appr);
    }
    g->xmin = fmin(g->xmin, g->fx[i]);
    g->xmax = fmax(g->xmax, g->fx[i]);
    g->zmin = fmin(g->zmin, g->fz[i]);
    g->zmax = fmax(g->zmax, g->fz[i]);
  }
  double y_top = 0.0 + double(y), y_bot = double(-h) + double(y);
  if (appr > 0.0) {
    y_top = trunc(y_top * appr);
    y_bot = trunc(y_bot * appr);
  }
  g->ymax = fmax(y_top, y_bot);
  g->ymin = fmin(y_top, y_bot);
  g->area = fabs(shoelace(g->fx, g->fz, 4));
}

// nms.py:64-88: IoU of `a` (single_box) against `b` (an element of box_list)
__device__ inline double iou_3d(const BoxGeom& a, const BoxGeom& b) {
  if (a.xmax < b.xmin || a.xmin > b.xmax || a.ymax < b.ymin || a.ymin > b.ymax || a.zmax < b.zmin || a.zmin > b.zmax)
    return 0.0;
  double shared = 0.0;
  if (a.area != 0.0 && b.area != 0.0) shared = clipped_area(a, b);
  const double shared_y = fmin(b.ymax, a.ymax) - fmax(b.ymin, a.ymin);
  const double inter = shared_y * shared;
  const double uni = (b.ymax - b.ymin) * b.area + (a.ymax - a.ymin) * a.area;
  return double(float(inter)) / (uni - inter);
}

__global__ void sorted_geometry_kernel(const int32_t* __restrict__ order, const int32_t* __restrict__ total,
                                       const float* __restrict__ cand_box, const float* __restrict__ cand_score,
                                       const int32_t* __restrict__ cand_label, const int32_t* __restrict__ cand_index,
                                       float* __restrict__ s_box, float* __restrict__ s_score, int32_t* __restrict__ s_label,
                                       int32_t* __restrict__ s_index, BoxGeom* __restrict__ geom, double appr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *total) return;
  const int s = order[i];
#pragma unroll
  for (int j = 0; j < kBoxLen; ++j) s_box[int64_t(i) * kBoxLen + j] = cand_box[int64_t(s) * kBoxLen + j];
  s_score[i] = cand_score[s];
  s_label[i] = cand_label[s];
  s_index[i] = cand_index[s];
  make_geom(cand_box + int64_t(s) * kBoxLen, &geom[i], appr);
}

// bit j - (i & ~31)... of row i: candidate j (> i, same frame, same class) overlaps candidate i by more than thres.
// Rows are `words` 32-bit words wide and indexed by the position INSIDE the frame.  The two rules differ only for a
// NaN overlap (0 / 0: both unions zero, e.g. two boxes of height 0): nms.py's merge / rescore variants remove a box iff
// `overlap > thres` (NaN: kept), bboxes_nms (the int_corners path) keeps it iff `overlap <= thres` (NaN: removed).
__global__ void adjacency_kernel(const BoxGeom* __restrict__ geom, const int32_t* __restrict__ s_label,
                                 const int32_t* __restrict__ cand_frame_ptr, int num_frames, int words, double thres,
                                 bool keep_if_le, uint32_t* __restrict__ adj) {
  const int f = blockIdx.z;
  const int begin = cand_frame_ptr[f], count = cand_frame_ptr[f + 1] - begin;
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  for (int li = blockIdx.y; li < count; li += gridDim.y) {
    const BoxGeom a = geom[begin + li];
    const int la = s_label[begin + li];
    for (int wj = (li >> 5) + blockIdx.x * warps_per_block + (threadIdx.x >> 5); wj * 32 < count;
         wj += gridDim.x * warps_per_block) {
      const int lj = wj * 32 + lane;
      bool hit = false;
      if (lj > li && lj < count && s_label[begin + lj] == la) {
        const double ov = iou_3d(a, geom[begin + lj]);
        hit = keep_if_le ? !(ov <= thres) : ov > thres;
      }
      const uint32_t m = __ballot_sync(0xffffffffu, hit);
      if (lane == 0) adj[(int64_t(begin) + li) * words + wj] = m;
    }
  }
}

// ---- 4. sweep ----------------------------------------------------------------------------------------
// One warp per frame.  valid = boxes not yet suppressed.  Box i (in score order) is kept iff still valid; it then
// removes R_i = adj[i] & valid.  adj[i] is overwritten with R_i for the merge step.
__global__ void sweep_kernel(const int32_t* __restrict__ cand_frame_ptr, int words, uint32_t* __restrict__ adj,
                             uint32_t* __restrict__ valid_buf, int32_t* __restrict__ kept) {
  const int f = blockIdx.x;
  const int lane = threadIdx.x;
  const int begin = cand_frame_ptr[f], count = cand_frame_ptr[f + 1] - begin;
  uint32_t* valid = valid_buf + int64_t(f) * words;
  for (int w = lane; w < words; w += 32) {
    const int base = w * 32;
    valid[w] = base + 32 <= count ? 0xffffffffu : (base < count ? ((1u << (count - base)) - 1u) : 0u);
  }
  __syncwarp();
  for (int i = 0; i < count; ++i) {
    const bool alive = (valid[i >> 5] >> (i & 31)) & 1u;      // uniform
    if (lane == 0) kept[begin + i] = alive ? 1 : 0;
    if (!alive) continue;
    uint32_t* row = adj + (int64_t(begin) + i) * words;
    for (int w = (i >> 5) + lane; w < words; w += 32) {
      const uint32_t r = row[w] & valid[w];
      row[w] = r;
      valid[w] &= ~r;
    }
    __syncwarp();
  }
}

// ---- 5. merge + rescore --------------------------------------------------------------------------------
constexpr int kMergeThreads = 256;
__global__ void __launch_bounds__(kMergeThreads) merge_rescore_kernel(
    const int32_t* __restrict__ cand_frame_ptr, int num_frames, const int32_t* __restrict__ total, int words,
    const uint32_t* __restrict__ adj, const int32_t* __restrict__ kept, const BoxGeom* __restrict__ geom,
    const float* __restrict__ s_box, const float* __restrict__ s_score, int do_merge, int do_rescore,
    float* __restrict__ out_box, float* __restrict__ out_score, int32_t* __restrict__ scratch_idx) {
  __shared__ int s_n;
  __shared__ float s_med[kBoxLen];
  __shared__ double s_sum[kMergeThreads / 32];
  __shared__ BoxGeom s_geom;
  const int tid = threadIdx.x;
  for (int i = blockIdx.x; i < *total; i += gridDim.x) {
    __syncthreads();
    if (!kept[i]) continue;                                   // uniform
    const int f = find_frame(cand_frame_ptr, num_frames, i);
    const int begin = cand_frame_ptr[f];
    const int li = i - begin;
    const uint32_t* row = adj + int64_t(i) * words;
    int32_t* list = scratch_idx + int64_t(blockIdx.x) * (int64_t(words) * 32 + 1);
    // removed set -> index list (ascending), box i itself appended last (nms.py:153-154 concatenation order)
    if (tid == 0) {
      int n = 0;
      for (int w = li >> 5; w < words; ++w) {
        uint32_t m = row[w];
        while (m) {
          const int b = __ffs(m) - 1;
          m &= m - 1;
          list[n++] = begin + w * 32 + b;
        }
      }
      list[n++] = i;
      s_n = n;
    }
    __syncthreads();
    const int n = s_n;
    // coordinate-wise median (np.median: middle element, or the float32 mean of the two middle ones)
    if (do_merge && n > 1) {
      for (int d = 0; d < kBoxLen; ++d) {
        const int lo_rank = (n - 1) >> 1, hi_rank = n >> 1;
        for (int e = tid; e < n; e += kMergeThreads) {
          const float v = s_box[int64_t(list[e]) * kBoxLen + d];
          int rank = 0;
          for (int q = 0; q < n; ++q) {
            const float u = s_box[int64_t(list[q]) * kBoxLen + d];
            rank += (u < v || (u == v && q < e)) ? 1 : 0;
          }
          if (rank == lo_rank) s_med[d] = v;                  // exactly one element has each rank
        }
        __syncthreads();
        if (hi_rank != lo_rank) {
          const float lo_v = s_med[d];
          __syncthreads();
          for (int e = tid; e < n; e += kMergeThreads) {
            const float v = s_box[int64_t(list[e]) * kBoxLen + d];
            int rank = 0;
            for (int q = 0; q < n; ++q) {
              const float u = s_box[int64_t(list[q]) * kBoxLen + d];
              rank += (u < v || (u == v && q < e)) ? 1 : 0;
            }
            if (rank == hi_rank) s_med[d] = __fmul_rn(__fadd_rn(lo_v, v), 0.5f);
          }
          __syncthreads();
        }
      }
    } else if (tid < kBoxLen) {
      s_med[tid] = s_box[int64_t(i) * kBoxLen + tid];
    }
    __syncthreads();
    if (tid < kBoxLen) out_box[int64_t(i) * kBoxLen + tid] = s_med[tid];
    // rescore: score_i += sum_j score_j * IoU(merged box, ORIGINAL box j)   (nms.py:157-161)
    double part = 0.0;
    if (do_rescore && n > 1) {
      if (tid == 0) make_geom(s_med, &s_geom);
      __syncthreads();
      for (int e = tid; e < n - 1; e += kMergeThreads) {
        const int j = list[e];
        part += double(s_score[j]) * iou_3d(s_geom, geom[j]);
      }
    }
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if ((tid & 31) == 0) s_sum[tid >> 5] = part;
    __syncthreads();
    if (tid == 0) {
      double tot = 0.0;
      for (int w = 0; w < kMergeThreads / 32; ++w) tot += s_sum[w];
      out_score[i] = float(double(s_score[i]) + tot);        // scores[i] += float64 sum, stored as float32
    }
  }
}

// ---- 6. compaction ---------------------------------------------------------------------------------------
__global__ void compact_kernel(const int32_t* __restrict__ total, const int32_t* __restrict__ kept,
                               const int32_t* __restrict__ kept_scan, const float* __restrict__ out_box,
                               const float* __restrict__ out_score, const int32_t* __restrict__ s_label,
                               const int32_t* __restrict__ s_index, int64_t capacity, int32_t* __restrict__ det_label,
                               float* __restrict__ det_box, float* __restrict__ det_score, int32_t* __restrict__ det_index) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *total || !kept[i]) return;
  const int o = kept_scan[i];
  if (o >= capacity) return;
  det_label[o] = s_label[i];
  det_score[o] = out_score[i];
  det_index[o] = s_index[i];
#pragma unroll
  for (int j = 0; j < kBoxLen; ++j) det_box[int64_t(o) * kBoxLen + j] = out_box[int64_t(i) * kBoxLen + j];
}

__global__ void det_frame_ptr_kernel(const int32_t* __restrict__ cand_frame_ptr, int num_frames,
                                     const int32_t* __restrict__ kept_scan, int32_t* __restrict__ det_frame_ptr) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > num_frames) return;
  det_frame_ptr[f] = kept_scan[cand_frame_ptr[f]];     // kept_scan has total + 1 entries (exclusive scan)
}

// The candidate boxes of a batch: the input of stages 2-6.  box / score / label / index are indexed by candidate
// position (frame by frame); the sort runs over sort_n entries, the keys of any entries past the candidates sort last.
struct Candidates {
  const float* box = nullptr;            // [n, 7]
  const float* score = nullptr;          // [n]
  const int32_t* label = nullptr;        // [n]
  Temp index;                            // int32 [n]: flat (vertex, class) index, or the position in the caller's arrays
  Temp keys_a, keys_b, vals_a, vals_b;   // sort input and output: sort_key -> candidate position
  Temp frame_count;                      // int32 [num_frames + 1]: candidates per frame, then the largest count
  Temp frame_ptr;                        // int32 [num_frames + 1]: frame_ptr[num_frames] = number of candidates
  int64_t sort_n = 0;
  int num_frames = 0;

  // n sort entries and index slots; frame_count zeroed
  int alloc(int64_t n, int frames, cudaStream_t s) {
    sort_n = n;
    num_frames = frames;
    PG_CUDA_OK(index.alloc(sizeof(int32_t) * n, s));
    PG_CUDA_OK(keys_a.alloc(sizeof(uint64_t) * n, s));
    PG_CUDA_OK(keys_b.alloc(sizeof(uint64_t) * n, s));
    PG_CUDA_OK(vals_a.alloc(sizeof(int32_t) * n, s));
    PG_CUDA_OK(vals_b.alloc(sizeof(int32_t) * n, s));
    PG_CUDA_OK(frame_count.alloc(sizeof(int32_t) * (frames + 1), s));
    PG_CUDA_OK(frame_ptr.alloc(sizeof(int32_t) * (frames + 1), s));
    PG_CUDA_OK(cudaMemsetAsync(frame_count.ptr, 0, sizeof(int32_t) * (frames + 1), s));
    return PG_OK;
  }
};

// The caller's outputs
struct Detections {
  int32_t* label; float* box; float* score; int32_t* index;   // [capacity] kept boxes
  int64_t capacity;
  int32_t* frame_ptr;                                         // [num_frames + 1] into the kept boxes
  int32_t* cand_index; int32_t* cand_frame_ptr;               // the candidate list, or null when not wanted
  int64_t* sizes_host;                                        // {kept boxes, candidates}
};

}  // namespace
}  // namespace pg

using namespace pg;

// Stages 2-6 on candidates whose sort input (keys_a, vals_a) and per-frame counts are filled.  Two host round trips:
// the widest frame (to size the bit matrix), then the number of kept boxes.
static int nms_stage(Candidates& c, const Detections& out, double overlapped_thres, double appr_factor, int32_t flags,
                     int64_t max_candidates_per_frame, cudaStream_t s) {
  const int num_frames = c.num_frames;
  const int32_t* cfp = c.frame_ptr.as<int32_t>();
  const int32_t* total_dev = cfp + num_frames;     // number of candidates
  frame_ptr_kernel<<<1, 1, 0, s>>>(c.frame_count.as<int32_t>(), num_frames, c.frame_ptr.as<int32_t>());
  PG_LAUNCH_CHECK();
  // bboxes_sort (nms.py:90-107): score descending inside a frame; stable, so ties keep ascending candidate position
  if (int rc = sort_pairs(c.keys_a.as<uint64_t>(), c.keys_b.as<uint64_t>(), c.vals_a.as<int32_t>(), c.vals_b.as<int32_t>(),
                          c.sort_n, 64, s))
    return rc;

  // the widest frame decides the bit-matrix row width; it must be known on the host to size the matrix
  int32_t h_max = 0, h_total = 0;
  PG_CUDA_OK(cudaMemcpyAsync(&h_max, c.frame_count.as<int32_t>() + num_frames, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaMemcpyAsync(&h_total, total_dev, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaStreamSynchronize(s));
  out.sizes_host[0] = 0;
  out.sizes_host[1] = h_total;
  if (out.cand_frame_ptr)
    PG_CUDA_OK(cudaMemcpyAsync(out.cand_frame_ptr, cfp, sizeof(int32_t) * (num_frames + 1), cudaMemcpyDeviceToDevice, s));
  if (h_total == 0) {
    PG_CUDA_OK(cudaMemsetAsync(out.frame_ptr, 0, sizeof(int32_t) * (num_frames + 1), s));
    return PG_OK;
  }
  if (h_max > max_candidates_per_frame) {
    set_error("a frame has %d box candidates, more than max_candidates_per_frame = %lld", h_max,
              (long long)max_candidates_per_frame);
    return PG_ERR_CAPACITY;
  }
  const int words = (h_max + 31) / 32;
  Temp sbox, sscore, slabel, sindex, geom, adj, valid, kept, kept_scan, obox, oscore, scratch;
  PG_CUDA_OK(sbox.alloc(sizeof(float) * h_total * kBoxLen, s));
  PG_CUDA_OK(sscore.alloc(sizeof(float) * h_total, s));
  PG_CUDA_OK(slabel.alloc(sizeof(int32_t) * h_total, s));
  PG_CUDA_OK(sindex.alloc(sizeof(int32_t) * h_total, s));
  PG_CUDA_OK(geom.alloc(sizeof(BoxGeom) * h_total, s));
  PG_CUDA_OK(adj.alloc(sizeof(uint32_t) * int64_t(h_total) * words, s));
  PG_CUDA_OK(cudaMemsetAsync(adj.ptr, 0, sizeof(uint32_t) * int64_t(h_total) * words, s));
  PG_CUDA_OK(valid.alloc(sizeof(uint32_t) * int64_t(num_frames) * words, s));
  PG_CUDA_OK(kept.alloc(sizeof(int32_t) * (h_total + 1), s));
  PG_CUDA_OK(kept_scan.alloc(sizeof(int32_t) * (h_total + 1), s));
  PG_CUDA_OK(obox.alloc(sizeof(float) * h_total * kBoxLen, s));
  PG_CUDA_OK(oscore.alloc(sizeof(float) * h_total, s));
  sorted_geometry_kernel<<<ceil_div(h_total, 128), 128, 0, s>>>(
      c.vals_b.as<int32_t>(), total_dev, c.box, c.score, c.label, c.index.as<int32_t>(), sbox.as<float>(),
      sscore.as<float>(), slabel.as<int32_t>(), sindex.as<int32_t>(), geom.as<BoxGeom>(),
      (flags & PG_NMS_INT_CORNERS) ? appr_factor : 0.0);
  PG_LAUNCH_CHECK();
  {
    dim3 grid(std::max(1, std::min(words / 4 + 1, 16)), std::min(h_max, 4096), num_frames);
    adjacency_kernel<<<grid, 128, 0, s>>>(geom.as<BoxGeom>(), slabel.as<int32_t>(), cfp, num_frames, words,
                                          overlapped_thres, (flags & PG_NMS_INT_CORNERS) != 0, adj.as<uint32_t>());
    PG_LAUNCH_CHECK();
  }
  sweep_kernel<<<num_frames, 32, 0, s>>>(cfp, words, adj.as<uint32_t>(), valid.as<uint32_t>(), kept.as<int32_t>());
  PG_LAUNCH_CHECK();
  const int mblocks = std::min(h_total, num_sms() * 4);
  PG_CUDA_OK(scratch.alloc(sizeof(int32_t) * int64_t(mblocks) * (int64_t(words) * 32 + 1), s));
  merge_rescore_kernel<<<mblocks, kMergeThreads, 0, s>>>(
      cfp, num_frames, total_dev, words, adj.as<uint32_t>(), kept.as<int32_t>(), geom.as<BoxGeom>(), sbox.as<float>(),
      sscore.as<float>(), (flags & PG_NMS_MERGE) ? 1 : 0, (flags & PG_NMS_RESCORE) ? 1 : 0, obox.as<float>(),
      oscore.as<float>(), scratch.as<int32_t>());
  PG_LAUNCH_CHECK();
  PG_CUDA_OK(cudaMemsetAsync(kept.as<int32_t>() + h_total, 0, sizeof(int32_t), s));
  if (int rc = exclusive_sum(kept.as<int32_t>(), kept_scan.as<int32_t>(), h_total + 1, s)) return rc;
  compact_kernel<<<ceil_div(h_total, 256), 256, 0, s>>>(total_dev, kept.as<int32_t>(), kept_scan.as<int32_t>(), obox.as<float>(),
                                                        oscore.as<float>(), slabel.as<int32_t>(), sindex.as<int32_t>(),
                                                        out.capacity, out.label, out.box, out.score, out.index);
  PG_LAUNCH_CHECK();
  det_frame_ptr_kernel<<<ceil_div(num_frames + 1, 64), 64, 0, s>>>(cfp, num_frames, kept_scan.as<int32_t>(), out.frame_ptr);
  PG_LAUNCH_CHECK();
  if (out.cand_index)   // all candidates in ascending (vertex, class) order: run.py:284 box_indices, per frame
    PG_CUDA_OK(cudaMemcpyAsync(out.cand_index, c.index.ptr, sizeof(int32_t) * h_total, cudaMemcpyDeviceToDevice, s));
  int32_t h_det = 0;
  PG_CUDA_OK(cudaMemcpyAsync(&h_det, kept_scan.as<int32_t>() + h_total, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaStreamSynchronize(s));
  out.sizes_host[0] = h_det;
  if (h_det > out.capacity) {
    set_error("detection buffer too small: need %d, capacity %lld", h_det, (long long)out.capacity);
    return PG_ERR_CAPACITY;
  }
  return PG_OK;
}

static void make_class_table(const float* class_table_host, int num_classes, ClassTable* tab) {
  for (int c = 0; c < kMaxClasses; ++c) {
    tab->l[c] = tab->h[c] = tab->w[c] = 1.0f;
    tab->yaw0[c] = 0.0f;
    tab->decoded[c] = 0;
  }
  for (int c = 0; c < num_classes; ++c) {
    const float* t = class_table_host + 4 * c;
    if (t[0] > 0.0f) {
      tab->l[c] = t[0];
      tab->h[c] = t[1];
      tab->w[c] = t[2];
      tab->yaw0[c] = t[3];
      tab->decoded[c] = 1;
    }
  }
}

extern "C" int pg_decode_boxes(const float* box_encodings, const float* xyz, int64_t num_vertices, int32_t num_classes,
                               const float* class_table_host, float* out_boxes, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (num_vertices == 0) return PG_OK;
  PG_REQUIRE(box_encodings && xyz && class_table_host && out_boxes, "pg_decode_boxes: null argument");
  PG_REQUIRE(num_classes >= 1 && num_classes <= kMaxClasses, "pg_decode_boxes: num_classes %d not in [1, %d]", num_classes,
             kMaxClasses);
  ClassTable tab;
  make_class_table(class_table_host, num_classes, &tab);
  decode_all_kernel<<<ceil_div(num_vertices * num_classes, 256), 256, 0, s>>>(box_encodings, xyz, num_vertices, num_classes, tab,
                                                                              out_boxes);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_postprocess(const float* probs, const float* box_encodings, const float* xyz,
                              const int32_t* frame_ptr, int32_t num_frames, int64_t num_vertices, int32_t num_classes,
                              const float* class_table_host, double overlapped_thres, int32_t flags,
                              int64_t max_candidates_per_frame, int32_t* out_label, float* out_box, float* out_score,
                              int32_t* out_index, int64_t capacity, int32_t* out_det_frame_ptr,
                              int32_t* out_cand_index, int32_t* out_cand_frame_ptr, int64_t* out_sizes_host,
                              void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(probs && box_encodings && xyz && frame_ptr && class_table_host && out_sizes_host && out_det_frame_ptr,
             "pg_postprocess: null argument");
  PG_REQUIRE(out_label && out_box && out_score && out_index && capacity >= 1, "pg_postprocess: output buffers are required");
  PG_REQUIRE(num_classes >= 3 && num_classes <= kMaxClasses, "pg_postprocess: num_classes %d not in [3, %d]", num_classes,
             kMaxClasses);
  PG_REQUIRE(num_frames >= 1 && num_frames <= 65535 && num_vertices >= 1, "pg_postprocess: bad sizes");
  PG_REQUIRE(num_vertices * num_classes < (int64_t(1) << 31), "pg_postprocess: too many (vertex, class) pairs");
  PG_REQUIRE(max_candidates_per_frame >= 32, "pg_postprocess: max_candidates_per_frame must be >= 32");
  ClassTable tab;
  make_class_table(class_table_host, num_classes, &tab);
  const int64_t cap = num_vertices * (num_classes - 2);      // at most C - 2 candidate classes per vertex
  const int64_t pairs = num_vertices * num_classes;
  Candidates cand;
  if (int rc = cand.alloc(cap, num_frames, s)) return rc;
  Temp flags_b, slots, cbox, cscore, clabel;
  PG_CUDA_OK(flags_b.alloc(sizeof(int32_t) * (pairs + 1), s));
  PG_CUDA_OK(slots.alloc(sizeof(int32_t) * (pairs + 1), s));
  PG_CUDA_OK(cbox.alloc(sizeof(float) * cap * kBoxLen, s));
  PG_CUDA_OK(cscore.alloc(sizeof(float) * cap, s));
  PG_CUDA_OK(clabel.alloc(sizeof(int32_t) * cap, s));
  PG_CUDA_OK(cudaMemsetAsync(flags_b.as<int32_t>() + pairs, 0, sizeof(int32_t), s));
  cand.box = cbox.as<float>();
  cand.score = cscore.as<float>();
  cand.label = clabel.as<int32_t>();

  flag_candidates_kernel<<<ceil_div(pairs, 256), 256, 0, s>>>(probs, num_vertices, num_classes, flags_b.as<int32_t>());
  PG_LAUNCH_CHECK();
  if (int rc = exclusive_sum(flags_b.as<int32_t>(), slots.as<int32_t>(), pairs + 1, s)) return rc;
  decode_scatter_kernel<<<ceil_div(pairs, 256), 256, 0, s>>>(
      probs, box_encodings, xyz, frame_ptr, num_frames, num_vertices, num_classes, tab, flags_b.as<int32_t>(),
      slots.as<int32_t>(), cbox.as<float>(), cscore.as<float>(), clabel.as<int32_t>(), cand.index.as<int32_t>(),
      cand.keys_a.as<uint64_t>(), cand.vals_a.as<int32_t>(), cand.frame_count.as<int32_t>());
  PG_LAUNCH_CHECK();
  // slots[pairs] = number of candidates
  fill_tail_keys_kernel<<<ceil_div(cap, 256), 256, 0, s>>>(slots.as<int32_t>() + pairs, cap, cand.keys_a.as<uint64_t>(),
                                                          cand.vals_a.as<int32_t>());
  PG_LAUNCH_CHECK();
  const Detections out{out_label, out_box, out_score, out_index, capacity, out_det_frame_ptr, out_cand_index,
                       out_cand_frame_ptr, out_sizes_host};
  return nms_stage(cand, out, overlapped_thres, 0.0, flags, max_candidates_per_frame, s);
}

extern "C" int pg_nms_boxes_3d(const int32_t* class_labels, const float* boxes, const float* scores,
                               const int32_t* frame_ptr, int32_t num_frames, int64_t num_boxes, double overlapped_thres,
                               double appr_factor, int32_t flags, int64_t max_candidates_per_frame, int32_t* out_label, float* out_box,
                               float* out_score, int32_t* out_index, int64_t capacity, int32_t* out_det_frame_ptr,
                               int64_t* out_sizes_host, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(class_labels && boxes && scores && frame_ptr && out_sizes_host && out_det_frame_ptr, "pg_nms_boxes_3d: null argument");
  PG_REQUIRE(out_label && out_box && out_score && out_index && capacity >= 1, "pg_nms_boxes_3d: output buffers are required");
  PG_REQUIRE(num_frames >= 1 && num_frames <= 65535 && num_boxes >= 1 && num_boxes < (int64_t(1) << 31), "pg_nms_boxes_3d: bad sizes");
  PG_REQUIRE(max_candidates_per_frame >= 32, "pg_nms_boxes_3d: max_candidates_per_frame must be >= 32");
  Candidates cand;
  if (int rc = cand.alloc(num_boxes, num_frames, s)) return rc;
  cand.box = boxes;
  cand.score = scores;
  cand.label = class_labels;
  candidate_keys_kernel<<<ceil_div(num_boxes, 256), 256, 0, s>>>(scores, frame_ptr, num_frames, num_boxes,
                                                                  cand.keys_a.as<uint64_t>(), cand.vals_a.as<int32_t>(),
                                                                  cand.frame_count.as<int32_t>(), cand.index.as<int32_t>());
  PG_LAUNCH_CHECK();
  const Detections out{out_label, out_box, out_score, out_index, capacity, out_det_frame_ptr, nullptr, nullptr, out_sizes_host};
  return nms_stage(cand, out, overlapped_thres, appr_factor, flags, max_candidates_per_frame, s);
}
