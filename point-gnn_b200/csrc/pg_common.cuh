// Shared helpers for libpointgnn_b200 (error plumbing, launch accounting, temp buffers) and the internal functions
// one source file calls in another.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <float.h>

#include "../../include/pointgnn_b200.h"

namespace pg {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define PG_CUDA_OK(expr)                                                              \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess) {                                                          \
      pg::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return PG_ERR_CUDA;                                                             \
    }                                                                                 \
  } while (0)

#define PG_REQUIRE(cond, ...)              \
  do {                                     \
    if (!(cond)) {                         \
      pg::set_error(__VA_ARGS__);          \
      return PG_ERR_INVALID_ARGUMENT;      \
    }                                      \
  } while (0)

#define PG_LAUNCH_CHECK()                     \
  do {                                        \
    pg::count_launch();                       \
    PG_CUDA_OK(cudaGetLastError());           \
  } while (0)

// Stream-ordered temporary buffer; freed (stream-ordered) when it goes out of scope.
struct Temp {
  void* ptr = nullptr;
  cudaStream_t stream = nullptr;
  Temp() {}
  Temp(const Temp&) = delete;
  Temp& operator=(const Temp&) = delete;
  Temp(Temp&& o) noexcept : ptr(o.ptr), stream(o.stream) { o.ptr = nullptr; }
  cudaError_t alloc(size_t bytes, cudaStream_t s) {
    stream = s;
    if (bytes == 0) bytes = 16;
    keep_pool_warm();
    return cudaMallocAsync(&ptr, bytes, s);
  }
  // By default the stream-ordered pool returns freed memory to the OS at every synchronisation,
  // which turns each temporary into a driver allocation (measured: graph build 2.8 -> 26 ms/step).
  static void keep_pool_warm() {
    static bool done = false;
    if (done) return;
    done = true;
    int dev = 0;
    cudaMemPool_t pool;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      unsigned long long threshold = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &threshold);
    }
  }
  template <typename T>
  T* as() const { return reinterpret_cast<T*>(ptr); }
  ~Temp() {
    if (ptr) cudaFreeAsync(ptr, stream);
  }
};

// Device word a kernel sets to nonzero when it meets an out-of-range index: allocated and zeroed on the stream;
// read() returns its value after the stream's work.  trusted (PG_FLAG_TRUSTED_INDICES: the caller guarantees the
// ranges) skips the read-back and the synchronisation and reports 0.
struct ErrorWord {
  Temp word;
  int init(cudaStream_t s) {
    PG_CUDA_OK(word.alloc(sizeof(int), s));
    PG_CUDA_OK(cudaMemsetAsync(word.ptr, 0, sizeof(int), s));
    return PG_OK;
  }
  int* ptr() const { return word.as<int>(); }
  int read(int* value, bool trusted, cudaStream_t s) const {
    *value = 0;
    if (trusted) return PG_OK;
    PG_CUDA_OK(cudaMemcpyAsync(value, word.ptr, sizeof(int), cudaMemcpyDeviceToHost, s));
    PG_CUDA_OK(cudaStreamSynchronize(s));
    return PG_OK;
  }
};

// max(float) through integer atomics: valid for any finite values and any initial value.
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
  v += 0.0f;  // canonicalise -0.0f
  if (v >= 0.0f)
    atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
  else
    atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

// The PG_ACT_* activations, the one definition every kernel calls.  TF 1.15 semantics as recalled (TF's source is
// not at hand to check against): leaky_relu with the alpha 0.01 the reference passes; elu is exp(x) - 1 below zero
// in TF, expm1f here (they differ by < 1e-7).  The accurate CUDA functions, not the __expf intrinsics.  Each one is
// monotone non-decreasing, which the fused segment max relies on: max_e f(a_e + b) = f(max_e a_e + b).
__device__ __forceinline__ float activate(int act, float x) {
  switch (act) {
    case PG_ACT_RELU: return fmaxf(x, 0.0f);
    case PG_ACT_RELU6: return fminf(fmaxf(x, 0.0f), 6.0f);
    case PG_ACT_LEAKY_RELU: return x > 0.0f ? x : 0.01f * x;
    case PG_ACT_ELU: return x > 0.0f ? x : expm1f(x);
    case PG_ACT_SIGMOID: return 1.0f / (1.0f + expf(-x));
    case PG_ACT_TANH: return tanhf(x);
    default: return x;   // PG_ACT_NONE
  }
}

// the activation a precision word's flag bits select (ReLU without PG_FLAG_ACTIVATION); -1 for an unknown code
inline int activation_of(int32_t precision) {
  if (!(precision & PG_FLAG_ACTIVATION)) return PG_ACT_RELU;
  const uint32_t act = uint32_t(precision) >> PG_ACT_SHIFT;   // every bit above the field counts: 256 is not 0
  return act < PG_ACT_COUNT ? int(act) : -1;
}

// the PG_AGG_* aggregation a flag word selects (max without the field); -1 for the unused code 3
inline int aggregation_of(int32_t flags) {
  const int agg = (flags & PG_AGG_MASK) >> PG_AGG_SHIFT;
  return agg <= PG_AGG_MEAN ? agg : -1;
}

// float <-> order-preserving uint: a < b iff float_to_ordered(a) < float_to_ordered(b), for any non-NaN values
__device__ inline uint32_t float_to_ordered(float f) {
  uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ inline float ordered_to_float(uint32_t u) {
  uint32_t b = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
  return __uint_as_float(b);
}

// the frame f with frame_ptr[f] <= row < frame_ptr[f + 1] (rows past the end fall into the last frame)
__device__ inline int find_frame(const int32_t* __restrict__ frame_ptr, int num_frames, int64_t row) {
  int lo = 0, hi = num_frames;  // invariant: frame_ptr[lo] <= row < frame_ptr[hi]
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (frame_ptr[mid] <= row) lo = mid; else hi = mid;
  }
  return lo;
}

// pg_api.cu: CUB device-wide scans and the stable radix sort of (key, value) pairs over bits [0, end_bit), each with
// a stream-ordered temporary; they count their launches (scan 2, sort 4)
int exclusive_sum(const int32_t* in, int32_t* out, int64_t n, cudaStream_t s);
int inclusive_sum(const int32_t* in, int32_t* out, int64_t n, cudaStream_t s);
int sort_pairs(const uint64_t* keys_in, uint64_t* keys_out, const int32_t* vals_in, int32_t* vals_out, int64_t n,
               int end_bit, cudaStream_t s);
// pg_ops.cu
int fill_async(float* p, int64_t n, float v, cudaStream_t s);
// out [m, ldo] = act(x [m, k] @ w [k, n] + bias) (+ residual [m, n]); columns [n, ldo) are written as zeros
int fc_fp32_launch(const float* x, int64_t m, int k, const float* w, const float* bias, int n, int act,
                   const float* residual, float* out, int ldo, cudaStream_t s);
// out [rows, ldo], columns [0, n): v = act(v + bias) (+ residual [rows, ldr]); bias and residual may be null.
// skip_empty leaves -FLT_MAX (an empty segment of a segment max) as it is
int activate_rows(float* out, int64_t rows, int n, int ldo, const float* bias, int act, const float* residual, int ldr,
                  bool skip_empty, cudaStream_t s);
// out [num_dst, n] /= max(number of edges e with dst[e] = row, 1): the segment sum -> unsorted_segment_mean.  Edges
// whose dst is out of range are not counted
int divide_by_segment_count(float* out, int64_t num_dst, int n, const int32_t* dst, int64_t num_edges, cudaStream_t s);
// The ordered segment sum (PG_FLAG_DETERMINISTIC) of the three sum paths (pg_tc.cu, pg_edge_simt.cu, pg_ops.cu), DESIGN
// §4.1.2.  A kernel cuts its rows into units it reduces in a fixed order (a warp's 16 edges, a 64-edge tile).  The
// rows of one destination are adjacent (the edge calls stable-sort their edges by dst first, pg_scatter_* their ids),
// so a run of them that holds neither the first nor the last row of its unit
// is the whole destination: it is stored into out.  The run that holds the unit's first row goes to slot 2 u of a side
// buffer, the run that holds its last row to slot 2 u + 1, each with the destination's id (-1: no run there).
// ordered_fixup then adds each destination's partial rows one after another in ascending slot order, and adds that
// into out (still 0 unless an earlier slice of the same edge list left a partial sum there).
// The launches that write a side buffer take at most kOrderedSlice edges each, which bounds the buffer: 2 rows of n
// floats per unit, for the tensor-core path (16-edge units) 2^15 rows.
constexpr int64_t kOrderedSlice = int64_t(1) << 18;
struct OrderedParts {
  Temp val, id;           // [slots, n] partial rows, [slots] destination ids
  int64_t slots = 0;
  int n = 0;
  int alloc(int64_t units, int cols, cudaStream_t s);   // ids filled with -1
  int reset(cudaStream_t s);                            // ids back to -1 for the next slice
  float* v() const { return val.as<float>(); }
  int32_t* i() const { return id.as<int32_t>(); }
};
int ordered_fixup(const OrderedParts& parts, float* out, int ldo, cudaStream_t s);
// pg_ops.cu: the stable order of ids [n] (ids outside [0, num_ids) last, as num_ids): keys_sorted [n] uint64, order
// [n] int32 (input positions); n < 2^31.  sort_edges_by_dst: src / dst in that order of dst, into src_s / dst_s
int stable_order(const int32_t* ids, int64_t n, int64_t num_ids, Temp& keys_sorted, Temp& order, cudaStream_t s);
int sort_edges_by_dst(const int32_t* src, const int32_t* dst, int64_t n, int64_t num_dst, Temp& src_s, Temp& dst_s,
                      cudaStream_t s);
// pg_tc.cu: count one fix-up launch (pg_tc_launch_count(2))
void count_ordered_launch();
// pg_edge_simt.cu: the fp32 FFMA edge MLP (activation act after every layer) + segment max (agg PG_AGG_MAX) or sum
// (any other) into out (already filled with -FLT_MAX or 0), the sum in a fixed order when ordered; sets *err on an
// out-of-range src / dst
int edge_mlp_max_fp32(int mode, const float* features, int c_in, const float* xyz_src, const float* xyz_dst,
                      const int32_t* dst_index, const int32_t* src, const int32_t* dst, int64_t num_edges,
                      int64_t num_src, int64_t num_dst, const float* const* weights, const float* const* biases,
                      const int32_t* dims, int num_layers, int act, int agg, bool ordered, float* out, int* err,
                      cudaStream_t s);

inline int num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

}  // namespace pg
