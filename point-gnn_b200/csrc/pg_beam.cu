// LiDAR beam downsampling on the GPU: the reference's data tool scripts/point_cloud_downsample.py:19-53 for every
// frame of a batch in one call, with its scikit-learn KMeans replaced by the exact 1-D k-means.
//
// Per point (original order), the reference's dtype chain:
//   xyz_norm = sqrt((x*x + y*y) + z*z)            float32 products, sum and square root
//   dot      = (x*0 + y*0) + z*1                  xyz.dot(int64 [[0],[0],[1]]): float64, equal to double(z)
//   cos      = dot / double(xyz_norm)             float64
// A point whose cosine is not finite (a zero norm, or one that underflows to zero in float32) compares false
// against every band limit in the reference, so it is never kept; here it also takes no part in the clustering
// (KMeans rejects NaN and inf).
//
// Clustering (per frame, the frame's n finite cosines sorted ascending as x_0 <= ... <= x_{n-1}):
//   F_1(j) = cost(0, j),  F_l(j) = min over a in [l-1, j-1] of F_{l-1}(a) + cost(a, j),  answer F_k(n),
//   cost(a, b) = sum over [a, b) of (x_i - mean)^2 = S2(a, b) - S1(a, b)^2 / (b - a)
// with S1 / S2 double-double prefix sums of e_i = x_i - x_0 (exact differences) and e_i^2, so the subtraction
// does not cancel a narrow beam's cost away; a group whose first and last values are equal costs exactly 0.
// Each layer is a divide-and-conquer over the monotone optimal split (Gronlund et al. 2017): the split of the
// middle position of a range bounds the splits of both halves.  The top kTopLevels recursion levels run
// kLevelBlocks blocks per frame, parallel across frames, segments and chunks of each segment's split range; each
// segment left after them is one warp's depth-first subtree.  Ties between equal totals go to the smallest split
// index.  The centres are the group means, the inertia the sum of the group costs.
//
// Bands (reference :27-35): centers = [-1] + sorted centres + [1]; for i in range(0, k, rate) the points with
// (c[i] + c[i+1]) / 2 < cos < (c[i+1] + c[i+2]) / 2 are kept, float64, both inequalities strict.  The kept rows
// are copied bit for bit in their original order.
#include <climits>
#include <utility>
#include <algorithm>

#include "pg_common.cuh"

namespace pg {
namespace {

constexpr uint64_t kExcludedKey = ~0ull;    // sort key of a non-finite cosine: last in its frame
constexpr int kTopLevels = 10;              // recursion levels run level by level across blocks
constexpr int kSegThreads = 256;
constexpr int kLevelBlocks = 256;          // blocks per frame on each top level: a segment's split range in chunks
constexpr int kScanThreads = 512;
constexpr int kSubtreeWarps = 8;
constexpr int kStackDepth = 40;             // > log2 of any int32 range + 2

// ---- double-double arithmetic, every operation explicitly rounded (no contraction) ----
struct __align__(16) dd {
  double hi, lo;
};
__device__ __forceinline__ dd two_sum(double a, double b) {
  const double s = __dadd_rn(a, b), bb = __dsub_rn(s, a);
  return {s, __dadd_rn(__dsub_rn(a, __dsub_rn(s, bb)), __dsub_rn(b, bb))};
}
__device__ __forceinline__ dd fast_two_sum(double a, double b) {
  const double s = __dadd_rn(a, b);
  return {s, __dsub_rn(b, __dsub_rn(s, a))};
}
__device__ __forceinline__ dd dd_add(dd x, dd y) {
  dd s = two_sum(x.hi, y.hi);
  const dd t = two_sum(x.lo, y.lo);
  s = fast_two_sum(s.hi, __dadd_rn(s.lo, t.hi));
  return fast_two_sum(s.hi, __dadd_rn(s.lo, t.lo));
}
__device__ __forceinline__ dd dd_sub(dd x, dd y) { return dd_add(x, dd{-y.hi, -y.lo}); }
__device__ __forceinline__ dd dd_mul(dd x, dd y) {
  const double p = __dmul_rn(x.hi, y.hi);
  const double e = __fma_rn(x.hi, y.hi, -p);   // the exact rounding error of p
  return fast_two_sum(p, __dadd_rn(e, __dadd_rn(__dmul_rn(x.hi, y.lo), __dmul_rn(x.lo, y.hi))));
}
__device__ __forceinline__ dd dd_div(dd x, double n) {
  const double q1 = __ddiv_rn(x.hi, n);
  const double p = __dmul_rn(q1, n);
  const dd r = dd_sub(x, dd{p, __fma_rn(q1, n, -p)});
  return fast_two_sum(q1, __ddiv_rn(r.hi, n));
}

// the frame's sorted cosines x [n], prefix sums s1 / s2 [n + 1]: the cost of the group [a, b), a < b
__device__ __forceinline__ double group_cost(const double* __restrict__ x, const dd* __restrict__ s1,
                                             const dd* __restrict__ s2, int a, int b) {
  if (x[a] == x[b - 1]) return 0.0;
  const dd d1 = dd_sub(s1[b], s1[a]);
  const dd c = dd_sub(dd_sub(s2[b], s2[a]), dd_div(dd_mul(d1, d1), double(b - a)));
  return c.hi > 0.0 ? c.hi : 0.0;
}

// (total, split) with the smaller total, the smaller split on equal totals
__device__ __forceinline__ void better(double& v, int& a, double v2, int a2) {
  if (v2 < v || (v2 == v && a2 < a)) {
    v = v2;
    a = a2;
  }
}
__device__ __forceinline__ void warp_best(double& v, int& a) {
  for (int o = 16; o > 0; o >>= 1) better(v, a, __shfl_xor_sync(0xffffffffu, v, o), __shfl_xor_sync(0xffffffffu, a, o));
}

struct FrameView {   // one frame's clustering arrays
  const double* x;
  const dd* s1;
  const dd* s2;
  const double* f_prev;
  double* f_cur;
  int32_t* opt;
  int n;
};

__device__ __forceinline__ bool frame_view(int f, const int32_t* frame_ptr, const int32_t* n_clus, int k, int layer,
                                           const double* x, const dd* s1, const dd* s2, const double* f_prev,
                                           double* f_cur, int32_t* opt, int64_t stride, FrameView& fv) {
  fv.n = n_clus[f];
  if (fv.n < k || fv.n == 0) return false;
  const int64_t b = frame_ptr[f] + int64_t(f);
  fv.x = x + frame_ptr[f];
  fv.s1 = s1 + b;
  fv.s2 = s2 + b;
  fv.f_prev = f_prev + b;
  fv.f_cur = f_cur + b;
  fv.opt = opt + int64_t(layer - 2) * stride + b;
  return true;
}

// the root range of layer l: positions [l, n - k + l] (only n on the last layer), splits [l - 1, J1 - 1]
__device__ __forceinline__ void layer_root(int n, int k, int l, int& jlo, int& jhi, int& alo, int& ahi) {
  jhi = n - k + l;
  jlo = l == k ? n : l;
  alo = l - 1;
  ahi = jhi - 1;
}

// descend `depth` levels along `path` (most significant bit first); false when the segment is empty
__device__ __forceinline__ bool descend(const int32_t* opt, uint32_t path, int depth, int& jlo, int& jhi, int& alo,
                                        int& ahi) {
  for (int s = 0; s < depth; ++s) {
    if (jlo > jhi) return false;
    const int m = (jlo + jhi) >> 1, o = opt[m];
    if ((path >> (depth - 1 - s)) & 1) {
      jlo = m + 1;
      alo = o;
    } else {
      jhi = m - 1;
      ahi = o;
    }
  }
  return jlo <= jhi;
}

// ---- kernels ----

__global__ void beam_cos_kernel(const float* __restrict__ velo, int64_t m, double* __restrict__ cosv,
                                uint64_t* __restrict__ key, int32_t* __restrict__ idx) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const float x = velo[i * 4 + 0], y = velo[i * 4 + 1], z = velo[i * 4 + 2];
  const float norm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
  const double dot = __dadd_rn(__dadd_rn(__dmul_rn(double(x), 0.0), __dmul_rn(double(y), 0.0)), __dmul_rn(double(z), 1.0));
  const double c = __ddiv_rn(dot, double(norm));
  cosv[i] = c;
  if (!key) return;
  if (isfinite(c)) {
    const uint64_t b = uint64_t(__double_as_longlong(__dadd_rn(c, 0.0)));   // -0 sorts with +0
    key[i] = (b >> 63) ? ~b : (b | (1ull << 63));
  } else {
    key[i] = kExcludedKey;
  }
  idx[i] = int32_t(i);
}

__global__ void beam_frame_key_kernel(const int32_t* __restrict__ idx, int64_t m, const int32_t* __restrict__ frame_ptr,
                                      int num_frames, uint64_t* __restrict__ key) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j < m) key[j] = uint64_t(find_frame(frame_ptr, num_frames, idx[j]));
}

__global__ void beam_gather_kernel(const int32_t* __restrict__ idx, int64_t m, const double* __restrict__ cosv,
                                   double* __restrict__ x) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j < m) x[j] = cosv[idx[j]];
}

// one thread per frame: its number of finite cosines (they sort first); flags a frame with 0 < n < k
__global__ void beam_count_kernel(const double* __restrict__ x, const int32_t* __restrict__ frame_ptr, int num_frames,
                                  int k, int32_t* __restrict__ n_clus, unsigned long long* __restrict__ bad) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= num_frames) return;
  int lo = frame_ptr[f], hi = frame_ptr[f + 1];   // first non-finite position in [lo, hi)
  const int begin = lo;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (isfinite(x[mid])) lo = mid + 1; else hi = mid;
  }
  const int n = lo - begin;
  n_clus[f] = n;
  if (n > 0 && n < k) atomicMin(bad, (static_cast<unsigned long long>(f) << 32) | static_cast<unsigned>(n));
}

// one block per frame: s1 / s2 [n + 1], chunk sums per thread, an in-order scan of the chunk totals, then the chunks
__global__ void __launch_bounds__(kScanThreads) beam_prefix_kernel(const double* __restrict__ x,
                                                                   const int32_t* __restrict__ frame_ptr,
                                                                   const int32_t* __restrict__ n_clus, int k,
                                                                   dd* __restrict__ s1, dd* __restrict__ s2) {
  __shared__ dd t1[kScanThreads], t2[kScanThreads];
  const int f = blockIdx.x;
  const int n = n_clus[f];
  if (n < k || n == 0) return;
  const double* xf = x + frame_ptr[f];
  dd* o1 = s1 + frame_ptr[f] + f;
  dd* o2 = s2 + frame_ptr[f] + f;
  const double x0 = xf[0];
  const int chunk = (n + kScanThreads - 1) / kScanThreads;
  const int begin = min(n, int(threadIdx.x) * chunk), end = min(n, begin + chunk);
  dd a1{0.0, 0.0}, a2{0.0, 0.0};
  for (int i = begin; i < end; ++i) {
    const dd e = two_sum(xf[i], -x0);
    a1 = dd_add(a1, e);
    a2 = dd_add(a2, dd_mul(e, e));
  }
  t1[threadIdx.x] = a1;
  t2[threadIdx.x] = a2;
  __syncthreads();
  if (threadIdx.x == 0) {
    dd r1{0.0, 0.0}, r2{0.0, 0.0};
    for (int t = 0; t < kScanThreads; ++t) {
      const dd c1 = t1[t], c2 = t2[t];
      t1[t] = r1;
      t2[t] = r2;
      r1 = dd_add(r1, c1);
      r2 = dd_add(r2, c2);
    }
    o1[0] = dd{0.0, 0.0};
    o2[0] = dd{0.0, 0.0};
  }
  __syncthreads();
  a1 = t1[threadIdx.x];
  a2 = t2[threadIdx.x];
  for (int i = begin; i < end; ++i) {
    const dd e = two_sum(xf[i], -x0);
    a1 = dd_add(a1, e);
    a2 = dd_add(a2, dd_mul(e, e));
    o1[i + 1] = a1;
    o2[i + 1] = a2;
  }
}

// layer 1: F_1(j) = cost(0, j) for j in [1, n - k + 1]; one thread per sorted position
__global__ void beam_layer1_kernel(const double* __restrict__ x, const dd* __restrict__ s1, const dd* __restrict__ s2,
                                   const int32_t* __restrict__ frame_ptr, int num_frames, int64_t m,
                                   const int32_t* __restrict__ n_clus, int k, double* __restrict__ f1) {
  const int64_t p = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= m) return;
  const int f = find_frame(frame_ptr, num_frames, p);
  const int n = n_clus[f];
  const int j = int(p - frame_ptr[f]) + 1;
  if (n < k || j > n - k + 1) return;
  const int64_t b = frame_ptr[f] + int64_t(f);
  f1[b + j] = group_cost(x + frame_ptr[f], s1 + b, s2 + b, 0, j);
}

// one recursion level `depth` of layer l: blocks (segment * chunks + chunk, frame) each search one of `chunks` equal
// parts of the segment's split range for its middle position; with chunks > 1 the last block of a segment to finish
// combines the parts (the minimum with the smaller-index tie rule does not depend on their order)
__global__ void __launch_bounds__(kSegThreads) beam_level_kernel(
    const double* __restrict__ x, const dd* __restrict__ s1, const dd* __restrict__ s2,
    const int32_t* __restrict__ frame_ptr, const int32_t* __restrict__ n_clus, int k, int layer, int depth,
    int chunks, const double* __restrict__ f_prev, double* __restrict__ f_cur, int32_t* __restrict__ opt,
    int64_t stride, double* __restrict__ part_v, int32_t* __restrict__ part_a, int32_t* __restrict__ arrived) {
  __shared__ double sv[kSegThreads / 32];
  __shared__ int sa[kSegThreads / 32];
  FrameView fv;
  if (!frame_view(blockIdx.y, frame_ptr, n_clus, k, layer, x, s1, s2, f_prev, f_cur, opt, stride, fv)) return;
  const int seg = blockIdx.x / chunks, chunk = blockIdx.x % chunks;
  int jlo, jhi, alo, ahi;
  layer_root(fv.n, k, layer, jlo, jhi, alo, ahi);
  if (!descend(fv.opt, seg, depth, jlo, jhi, alo, ahi)) return;   // uniform over the segment's blocks
  const int j = (jlo + jhi) >> 1, last = min(ahi, j - 1);
  const int per = (last - alo + chunks) / chunks;
  const int begin = alo + chunk * per, end = min(last, begin + per - 1);
  double best = DBL_MAX;
  int arg = INT_MAX;
  for (int a = begin + int(threadIdx.x); a <= end; a += kSegThreads)
    better(best, arg, __dadd_rn(fv.f_prev[a], group_cost(fv.x, fv.s1, fv.s2, a, j)), a);
  warp_best(best, arg);
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    sv[w] = best;
    sa[w] = arg;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int i = 1; i < kSegThreads / 32; ++i) better(best, arg, sv[i], sa[i]);
  if (chunks > 1) {
    const int64_t slot = int64_t(blockIdx.y) * kLevelBlocks + blockIdx.x;
    part_v[slot] = best;
    part_a[slot] = arg;
    __threadfence();
    int32_t* counter = arrived + int64_t(blockIdx.y) * kLevelBlocks + seg;
    if (atomicAdd(counter, 1) != chunks - 1) return;
    __threadfence();
    const int64_t first = int64_t(blockIdx.y) * kLevelBlocks + int64_t(seg) * chunks;
    for (int c = 0; c < chunks; ++c) better(best, arg, __ldcg(part_v + first + c), __ldcg(part_a + first + c));
    *counter = 0;   // ready for the next level
  }
  fv.opt[j] = arg;
  fv.f_cur[j] = best;
}

// the levels below kTopLevels of layer l: one warp per remaining segment, depth first with the split bounds
__global__ void __launch_bounds__(kSubtreeWarps * 32) beam_subtree_kernel(
    const double* __restrict__ x, const dd* __restrict__ s1, const dd* __restrict__ s2,
    const int32_t* __restrict__ frame_ptr, int num_frames, const int32_t* __restrict__ n_clus, int k, int layer,
    const double* __restrict__ f_prev, double* __restrict__ f_cur, int32_t* __restrict__ opt, int64_t stride) {
  const int64_t warp = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int f = int(warp >> kTopLevels);
  if (f >= num_frames) return;                               // warp-uniform
  FrameView fv;
  if (!frame_view(f, frame_ptr, n_clus, k, layer, x, s1, s2, f_prev, f_cur, opt, stride, fv)) return;
  int jlo, jhi, alo, ahi;
  layer_root(fv.n, k, layer, jlo, jhi, alo, ahi);
  if (!descend(fv.opt, uint32_t(warp & ((1 << kTopLevels) - 1)), kTopLevels, jlo, jhi, alo, ahi)) return;
  int4 stack[kStackDepth];
  int top = 0;
  stack[top++] = make_int4(jlo, jhi, alo, ahi);
  while (top > 0) {
    const int4 s = stack[--top];
    if (s.x > s.y) continue;
    const int j = (s.x + s.y) >> 1, last = min(s.w, j - 1);
    double best = DBL_MAX;
    int arg = INT_MAX;
    for (int a = s.z + lane; a <= last; a += 32)
      better(best, arg, __dadd_rn(fv.f_prev[a], group_cost(fv.x, fv.s1, fv.s2, a, j)), a);
    warp_best(best, arg);
    if (lane == 0) {
      fv.opt[j] = arg;
      fv.f_cur[j] = best;
    }
    stack[top++] = make_int4(j + 1, s.y, arg, s.w);
    stack[top++] = make_int4(s.x, j - 1, s.z, arg);
  }
}

// one thread per frame: backtrack the splits, then the group means, sizes and the inertia
__global__ void beam_backtrack_kernel(const double* __restrict__ x, const dd* __restrict__ s1,
                                      const dd* __restrict__ s2, const int32_t* __restrict__ frame_ptr,
                                      int num_frames, const int32_t* __restrict__ n_clus, int k,
                                      const int32_t* __restrict__ opt, int64_t stride, double* __restrict__ centers,
                                      double* __restrict__ inertia, int32_t* __restrict__ sizes) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= num_frames) return;
  const int n = n_clus[f];
  double* c = centers + int64_t(f) * k;
  if (n < k || n == 0) {   // no clusterable point (or too few: the call fails): no centre, no group
    for (int g = 0; g < k; ++g) {
      c[g] = __longlong_as_double(0x7ff8000000000000ll);
      if (sizes) sizes[int64_t(f) * k + g] = 0;
    }
    if (inertia) inertia[f] = 0.0;
    return;
  }
  const int64_t b = frame_ptr[f] + int64_t(f);
  const double* xf = x + frame_ptr[f];
  const dd* p1 = s1 + b;
  const dd* p2 = s2 + b;
  double total = 0.0;
  int hi = n;
  for (int g = k - 1; g >= 0; --g) {
    const int lo = g == 0 ? 0 : opt[int64_t(g - 1) * stride + b + hi];   // layer g + 1's split of position hi
    if (xf[lo] == xf[hi - 1]) {
      c[g] = xf[lo];
    } else {
      c[g] = dd_add(dd_div(dd_sub(p1[hi], p1[lo]), double(hi - lo)), dd{xf[0], 0.0}).hi;
    }
    if (sizes) sizes[int64_t(f) * k + g] = hi - lo;
    total = __dadd_rn(total, group_cost(xf, p1, p2, lo, hi));   // summed from the last group down
    hi = lo;
  }
  if (inertia) inertia[f] = total;
}

// one thread per point, original order: inside one of the kept bands of its frame's centres
__global__ void beam_mask_kernel(const double* __restrict__ cosv, int64_t m, const int32_t* __restrict__ frame_ptr,
                                 int num_frames, const double* __restrict__ centers, int k, int rate,
                                 int32_t* __restrict__ keep) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i > m) return;
  if (i == m) {
    keep[m] = 0;
    return;
  }
  const int f = find_frame(frame_ptr, num_frames, i);
  const double* c = centers + int64_t(f) * k;
  const double v = cosv[i];
  bool kept = false;
  for (int b = 0; b < k; b += rate) {   // centers = [-1] + c + [1]; band b is (ext[b] + ext[b+1]) / 2 .. (ext[b+1] + ext[b+2]) / 2
    const double e0 = b == 0 ? -1.0 : c[b - 1], e1 = c[b], e2 = b + 1 == k ? 1.0 : c[b + 1];
    const double lower = __ddiv_rn(__dadd_rn(e0, e1), 2.0), higher = __ddiv_rn(__dadd_rn(e1, e2), 2.0);
    kept = kept || (v > lower && v < higher);
  }
  keep[i] = kept ? 1 : 0;
}

__global__ void beam_compact_kernel(const float4* __restrict__ velo, const int32_t* __restrict__ keep,
                                    const int32_t* __restrict__ scan, int64_t m, const int32_t* __restrict__ frame_ptr,
                                    int num_frames, float4* __restrict__ out, int32_t* __restrict__ out_frame_ptr,
                                    int64_t* __restrict__ count) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i <= num_frames) out_frame_ptr[i] = scan[frame_ptr[i]];
  if (i == 0) count[0] = scan[m];
  if (i < m && keep[i]) out[scan[i]] = velo[i];
}

__global__ void beam_nan_kernel(double* __restrict__ p, int64_t n) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) p[i] = __longlong_as_double(0x7ff8000000000000ll);
}

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" int pg_beam_downsample(const float* velo, const int32_t* frame_ptr, int32_t num_frames, int64_t num_points,
                                  int32_t num_clusters, int32_t downsample_rate, const double* centers_in,
                                  double* centers_out, double* inertia_out, int32_t* group_sizes_out, float* out_velo,
                                  int32_t* out_frame_ptr, int64_t* out_num_points_host, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(frame_ptr && out_frame_ptr && out_num_points_host, "pg_beam_downsample: null argument");
  PG_REQUIRE(num_frames >= 1 && num_points >= 0 && num_points < (int64_t(1) << 31), "pg_beam_downsample: bad sizes");
  PG_REQUIRE(num_clusters >= 1, "pg_beam_downsample: num_clusters must be >= 1, got %d", num_clusters);
  PG_REQUIRE(downsample_rate >= 1, "pg_beam_downsample: downsample_rate must be >= 1, got %d", downsample_rate);
  PG_REQUIRE(centers_in || centers_out, "pg_beam_downsample: needs centers_in or centers_out");
  PG_REQUIRE(num_points == 0 || (velo && out_velo), "pg_beam_downsample: null point buffer");
  const int k = num_clusters;
  const int64_t m = num_points;
  *out_num_points_host = 0;
  if (m == 0) {   // nothing to keep; without caller centres every frame is empty: NaN centres, zero inertia
    PG_CUDA_OK(cudaMemsetAsync(out_frame_ptr, 0, sizeof(int32_t) * (num_frames + 1), s));
    if (!centers_in) {
      beam_nan_kernel<<<ceil_div(int64_t(num_frames) * k, 256), 256, 0, s>>>(centers_out, int64_t(num_frames) * k);
      PG_LAUNCH_CHECK();
      if (inertia_out) PG_CUDA_OK(cudaMemsetAsync(inertia_out, 0, sizeof(double) * num_frames, s));
      if (group_sizes_out) PG_CUDA_OK(cudaMemsetAsync(group_sizes_out, 0, sizeof(int32_t) * num_frames * k, s));
    }
    return PG_OK;
  }
  Temp cosv, status;
  PG_CUDA_OK(cosv.alloc(sizeof(double) * m, s));
  PG_CUDA_OK(status.alloc(sizeof(int64_t) * 2, s));
  PG_CUDA_OK(cudaMemsetAsync(status.as<int64_t>() + 1, 0xff, sizeof(int64_t), s));   // no short frame: ~0
  const double* centers = centers_in;
  if (!centers_in) {
    const int64_t slots = m + num_frames;   // frame f's prefix arrays and layer values start at frame_ptr[f] + f
    Temp key, key2, idx, idx2, x, n_clus, s1, s2, fa, fb, opt;
    PG_CUDA_OK(key.alloc(sizeof(uint64_t) * m, s));
    PG_CUDA_OK(key2.alloc(sizeof(uint64_t) * m, s));
    PG_CUDA_OK(idx.alloc(sizeof(int32_t) * m, s));
    PG_CUDA_OK(idx2.alloc(sizeof(int32_t) * m, s));
    PG_CUDA_OK(x.alloc(sizeof(double) * m, s));
    PG_CUDA_OK(n_clus.alloc(sizeof(int32_t) * num_frames, s));
    PG_CUDA_OK(s1.alloc(sizeof(dd) * slots, s));
    PG_CUDA_OK(s2.alloc(sizeof(dd) * slots, s));
    PG_CUDA_OK(fa.alloc(sizeof(double) * slots, s));
    PG_CUDA_OK(fb.alloc(sizeof(double) * slots, s));
    PG_CUDA_OK(opt.alloc(sizeof(int32_t) * slots * std::max(k - 1, 1), s));
    Temp part_v, part_a, arrived;
    PG_CUDA_OK(part_v.alloc(sizeof(double) * num_frames * kLevelBlocks, s));
    PG_CUDA_OK(part_a.alloc(sizeof(int32_t) * num_frames * kLevelBlocks, s));
    PG_CUDA_OK(arrived.alloc(sizeof(int32_t) * num_frames * kLevelBlocks, s));
    PG_CUDA_OK(cudaMemsetAsync(arrived.ptr, 0, sizeof(int32_t) * num_frames * kLevelBlocks, s));
    const int blocks = int(ceil_div(m, 256));
    beam_cos_kernel<<<blocks, 256, 0, s>>>(velo, m, cosv.as<double>(), key.as<uint64_t>(), idx.as<int32_t>());
    PG_LAUNCH_CHECK();
    // by cosine, then stably by frame: each frame's finite cosines ascending, the excluded points after them
    if (int rc = sort_pairs(key.as<uint64_t>(), key2.as<uint64_t>(), idx.as<int32_t>(), idx2.as<int32_t>(), m, 64, s))
      return rc;
    beam_frame_key_kernel<<<blocks, 256, 0, s>>>(idx2.as<int32_t>(), m, frame_ptr, num_frames, key.as<uint64_t>());
    PG_LAUNCH_CHECK();
    int frame_bits = 1;
    while ((int64_t(1) << frame_bits) < num_frames) ++frame_bits;
    if (int rc = sort_pairs(key.as<uint64_t>(), key2.as<uint64_t>(), idx2.as<int32_t>(), idx.as<int32_t>(), m,
                            frame_bits, s))
      return rc;
    beam_gather_kernel<<<blocks, 256, 0, s>>>(idx.as<int32_t>(), m, cosv.as<double>(), x.as<double>());
    PG_LAUNCH_CHECK();
    beam_count_kernel<<<ceil_div(num_frames, 128), 128, 0, s>>>(
        x.as<double>(), frame_ptr, num_frames, k, n_clus.as<int32_t>(),
        reinterpret_cast<unsigned long long*>(status.as<int64_t>() + 1));
    PG_LAUNCH_CHECK();
    beam_prefix_kernel<<<num_frames, kScanThreads, 0, s>>>(x.as<double>(), frame_ptr, n_clus.as<int32_t>(), k,
                                                           s1.as<dd>(), s2.as<dd>());
    PG_LAUNCH_CHECK();
    double* f_prev = fa.as<double>();
    double* f_cur = fb.as<double>();
    if (k >= 2) {
      beam_layer1_kernel<<<blocks, 256, 0, s>>>(x.as<double>(), s1.as<dd>(), s2.as<dd>(), frame_ptr, num_frames, m,
                                                n_clus.as<int32_t>(), k, f_prev);
      PG_LAUNCH_CHECK();
    }
    const int64_t subtree_warps = int64_t(num_frames) << kTopLevels;
    for (int layer = 2; layer <= k; ++layer) {
      for (int depth = 0; depth < kTopLevels; ++depth) {
        const int chunks = std::max(1, kLevelBlocks >> depth);
        beam_level_kernel<<<dim3((1u << depth) * chunks, num_frames), kSegThreads, 0, s>>>(
            x.as<double>(), s1.as<dd>(), s2.as<dd>(), frame_ptr, n_clus.as<int32_t>(), k, layer, depth, chunks,
            f_prev, f_cur, opt.as<int32_t>(), slots, part_v.as<double>(), part_a.as<int32_t>(), arrived.as<int32_t>());
        PG_LAUNCH_CHECK();
      }
      beam_subtree_kernel<<<ceil_div(subtree_warps, kSubtreeWarps), kSubtreeWarps * 32, 0, s>>>(
          x.as<double>(), s1.as<dd>(), s2.as<dd>(), frame_ptr, num_frames, n_clus.as<int32_t>(), k, layer, f_prev,
          f_cur, opt.as<int32_t>(), slots);
      PG_LAUNCH_CHECK();
      std::swap(f_prev, f_cur);
    }
    beam_backtrack_kernel<<<ceil_div(num_frames, 128), 128, 0, s>>>(
        x.as<double>(), s1.as<dd>(), s2.as<dd>(), frame_ptr, num_frames, n_clus.as<int32_t>(), k, opt.as<int32_t>(),
        slots, centers_out, inertia_out, group_sizes_out);
    PG_LAUNCH_CHECK();
    centers = centers_out;
  } else {
    beam_cos_kernel<<<ceil_div(m, 256), 256, 0, s>>>(velo, m, cosv.as<double>(), nullptr, nullptr);
    PG_LAUNCH_CHECK();
    if (centers_out && centers_out != centers_in)
      PG_CUDA_OK(cudaMemcpyAsync(centers_out, centers_in, sizeof(double) * num_frames * k, cudaMemcpyDeviceToDevice, s));
  }
  Temp keep, scan;
  PG_CUDA_OK(keep.alloc(sizeof(int32_t) * (m + 1), s));
  PG_CUDA_OK(scan.alloc(sizeof(int32_t) * (m + 1), s));
  beam_mask_kernel<<<ceil_div(m + 1, 256), 256, 0, s>>>(cosv.as<double>(), m, frame_ptr, num_frames, centers, k,
                                                        downsample_rate, keep.as<int32_t>());
  PG_LAUNCH_CHECK();
  if (int rc = exclusive_sum(keep.as<int32_t>(), scan.as<int32_t>(), m + 1, s)) return rc;
  beam_compact_kernel<<<ceil_div(std::max<int64_t>(m, num_frames + 1), 256), 256, 0, s>>>(
      reinterpret_cast<const float4*>(velo), keep.as<int32_t>(), scan.as<int32_t>(), m, frame_ptr, num_frames,
      reinterpret_cast<float4*>(out_velo), out_frame_ptr, status.as<int64_t>());
  PG_LAUNCH_CHECK();
  int64_t h_status[2] = {0, 0};
  PG_CUDA_OK(cudaMemcpyAsync(h_status, status.ptr, sizeof(h_status), cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaStreamSynchronize(s));
  if (h_status[1] != -1) {
    const uint64_t bad = uint64_t(h_status[1]);
    set_error("pg_beam_downsample: frame %d has %d points with a finite cosine, fewer than num_clusters = %d",
              int(bad >> 32), int(bad & 0xffffffffu), k);
    return PG_ERR_INVALID_ARGUMENT;
  }
  *out_num_points_host = h_status[0];
  return PG_OK;
}
