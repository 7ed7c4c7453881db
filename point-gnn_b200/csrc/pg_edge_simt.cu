// Fused per-edge MLP + destination-segment max, fp32 FFMA version (precision = 0).
//
// Replaces, without materialising any [E, *] tensor in HBM:
//   PointSetPooling.apply_regular   /root/reference/models/gnn.py:256-277
//   GraphNetAutoCenter.apply_regular /root/reference/models/gnn.py:338-365
// (gather -> concat(feature, relative xyz) -> L x act(x@W+b) -> unsorted_segment_max).
//
// One persistent CTA per SM walks 64-edge tiles.  The tile's activations ping-pong between two
// shared-memory buffers, each layer is a register-tiled FFMA GEMM against weights streamed
// through L1/L2 (they are a few hundred KB and stay cache resident), and the epilogue reduces the
// tile per destination before touching HBM: because edges are grouped by destination, each
// column thread walks the 64 rows keeping a running max and issues one atomic per (segment,
// tile, column).  This is the bit-faithful baseline (same fp32 association order as a CPU loop);
// the wgmma version in pg_tc.cu is the fast path.
#include "pg_common.cuh"

namespace pg {
namespace {

constexpr int kMaxLayers = 8;
constexpr int kTileE = 64;   // edges per tile
constexpr int kThreads = 256;
constexpr int kColBlock = 256;  // output columns per accumulation pass (8 per lane)

struct EdgeMlpParams {
  int mode;
  const float* features;
  int c_in;
  const float* xyz_src;
  const float* xyz_dst;
  const int32_t* dst_index;
  const int32_t* src;
  const int32_t* dst;
  int64_t num_edges;
  int64_t num_src;
  int64_t num_dst;
  const float* w[kMaxLayers];
  const float* b[kMaxLayers];
  int dims[kMaxLayers + 1];
  int num_layers;
  int act;               // PG_ACT_* after every layer
  int stride0, stride1;  // row strides (floats) of the two activation buffers
  float* out;
  int* err;
};

__global__ void __launch_bounds__(kThreads, 1) edge_mlp_max_fp32_kernel(EdgeMlpParams p) {
  extern __shared__ __align__(16) float smem[];
  float* buf0 = smem;
  float* buf1 = smem + size_t(kTileE) * p.stride0;
  __shared__ int s_src[kTileE];
  __shared__ int s_dst[kTileE];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t num_tiles = (p.num_edges + kTileE - 1) / kTileE;

  for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int64_t e0 = tile * kTileE;
    const int64_t remaining = p.num_edges - e0;
    const int rows = remaining < kTileE ? int(remaining) : kTileE;
    __syncthreads();  // previous tile's epilogue done with the buffers / index arrays
    if (threadIdx.x < kTileE) {
      int s = 0, d = -1;
      if (threadIdx.x < rows) {
        s = p.src[e0 + threadIdx.x];
        d = p.dst[e0 + threadIdx.x];
        if (s < 0 || s >= p.num_src || d < 0 || d >= p.num_dst) { *p.err = 1; s = 0; d = -1; }
      }
      s_src[threadIdx.x] = s;
      s_dst[threadIdx.x] = d;
    }
    __syncthreads();
    // ---- layer-0 input: [feature(src) , xyz_src(src) - xyz_dst(dst')] -------------------------
    const int d0 = p.dims[0];
    for (int r = warp; r < kTileE; r += kThreads / 32) {
      float* row = buf0 + size_t(r) * p.stride0;
      const int s = s_src[r], d = s_dst[r];
      if (r < rows && d >= 0) {
        const float* f = p.features + int64_t(s) * p.c_in;
        for (int c = lane; c < p.c_in; c += 32) row[c] = f[c];
        if (lane < 3) {
          const int64_t dd = p.dst_index ? int64_t(p.dst_index[d]) : int64_t(d);
          row[p.c_in + lane] = p.xyz_src[int64_t(s) * 3 + lane] - p.xyz_dst[dd * 3 + lane];
        }
      } else {
        for (int c = lane; c < d0; c += 32) row[c] = 0.0f;
      }
    }
    __syncthreads();
    // ---- L x act(x @ W + b) -------------------------------------------------------------------
    for (int l = 0; l < p.num_layers; ++l) {
      const float* in = (l & 1) ? buf1 : buf0;
      float* outb = (l & 1) ? buf0 : buf1;
      const int in_stride = (l & 1) ? p.stride1 : p.stride0;
      const int out_stride = (l & 1) ? p.stride0 : p.stride1;
      const int kd = p.dims[l], n = p.dims[l + 1];
      const float* __restrict__ w = p.w[l];
      const float* __restrict__ bias = p.b[l];
      const float* a_rows = in + size_t(warp * 8) * in_stride;  // this warp owns 8 tile rows
      for (int cb = 0; cb < n; cb += kColBlock) {
        float acc[8][8];
#pragma unroll
        for (int r = 0; r < 8; ++r)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[r][j] = 0.0f;
        const int ncols = min(kColBlock, n - cb);
        const int jmax = (ncols + 31) / 32;
        for (int k = 0; k < kd; ++k) {
          float wv[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int c = cb + lane + 32 * j;
            wv[j] = (j < jmax && c < n) ? __ldg(w + int64_t(k) * n + c) : 0.0f;
          }
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            const float a = a_rows[size_t(r) * in_stride + k];  // warp-wide broadcast
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[r][j] = fmaf(a, wv[j], acc[r][j]);
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = cb + lane + 32 * j;
          if (j < jmax && c < n) {
            const float bv = bias[c];
#pragma unroll
            for (int r = 0; r < 8; ++r)
              outb[size_t(warp * 8 + r) * out_stride + c] = activate(p.act, acc[r][j] + bv);
          }
        }
      }
      __syncthreads();
    }
    // ---- per-destination max over the tile, then one atomic per (segment, column) -------------
    const float* fin = (p.num_layers & 1) ? buf1 : buf0;
    const int fstride = (p.num_layers & 1) ? p.stride1 : p.stride0;
    const int n_out = p.dims[p.num_layers];
    for (int c = threadIdx.x; c < n_out; c += kThreads) {
      int cur = -1;
      float m = -FLT_MAX;
      for (int r = 0; r < rows; ++r) {
        const int d = s_dst[r];
        if (d != cur) {
          if (cur >= 0) atomic_max_float(p.out + int64_t(cur) * n_out + c, m);
          cur = d;
          m = -FLT_MAX;
        }
        m = fmaxf(m, fin[size_t(r) * fstride + c]);
      }
      if (cur >= 0) atomic_max_float(p.out + int64_t(cur) * n_out + c, m);
    }
  }
}

}  // namespace

int edge_mlp_max_fp32(int mode, const float* features, int c_in, const float* xyz_src, const float* xyz_dst,
                      const int32_t* dst_index, const int32_t* src, const int32_t* dst, int64_t num_edges,
                      int64_t num_src, int64_t num_dst, const float* const* weights, const float* const* biases,
                      const int32_t* dims, int num_layers, int act, float* out, int* err, cudaStream_t s) {
  PG_REQUIRE(num_layers >= 1 && num_layers <= kMaxLayers, "edge MLP depth %d not in [1,%d]", num_layers, kMaxLayers);
  PG_REQUIRE(dims[0] == c_in + 3, "dims[0]=%d must equal feature channels + 3 = %d", dims[0], c_in + 3);
  EdgeMlpParams p{};
  p.mode = mode;
  p.features = features;
  p.c_in = c_in;
  p.xyz_src = xyz_src;
  p.xyz_dst = xyz_dst;
  p.dst_index = dst_index;
  p.src = src;
  p.dst = dst;
  p.num_edges = num_edges;
  p.num_src = num_src;
  p.num_dst = num_dst;
  int w0 = 0, w1 = 0;
  for (int l = 0; l <= num_layers; ++l) {
    PG_REQUIRE(dims[l] >= 1 && dims[l] <= 4096, "layer width %d unsupported", dims[l]);
    p.dims[l] = dims[l];
    if (l & 1) w1 = std::max(w1, dims[l]); else w0 = std::max(w0, dims[l]);
  }
  for (int l = 0; l < num_layers; ++l) {
    PG_REQUIRE(weights[l] && biases[l], "null weight/bias for layer %d", l);
    p.w[l] = weights[l];
    p.b[l] = biases[l];
  }
  p.num_layers = num_layers;
  p.act = act;
  p.stride0 = w0 + 1;
  p.stride1 = w1 + 1;
  p.out = out;
  p.err = err;
  const size_t smem = size_t(kTileE) * (p.stride0 + p.stride1) * sizeof(float);
  PG_REQUIRE(smem <= 227 * 1024 - 1024, "edge MLP widths need %zu B of shared memory (> 226 KB)", smem);
  if (num_edges > 0) {
    PG_CUDA_OK(cudaFuncSetAttribute(edge_mlp_max_fp32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    const int64_t tiles = ceil_div(num_edges, kTileE);
    const int grid = int(std::min<int64_t>(tiles, num_sms()));
    edge_mlp_max_fp32_kernel<<<grid, kThreads, smem, s>>>(p);
    PG_LAUNCH_CHECK();
  }
  return PG_OK;
}

}  // namespace pg
