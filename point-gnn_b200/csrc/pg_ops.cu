// Stand-alone GNN ops: segment max, row gather, fp32 fully-connected layer, row softmax.
//
// Replaces the TF ops behind /root/reference/models/gnn.py:
//   graph_scatter_max_fn  (:106-109, tf.math.unsorted_segment_max)
//   tf.gather             (:256-262, :338-348)
//   slim.fully_connected  (:63-80, :93-103)   normalizer NONE, any PG_ACT_* activation
//   tf.nn.softmax         (models.py:165-168)
#include "pg_common.cuh"

namespace pg {

__global__ void fill_kernel(float* __restrict__ p, int64_t n, float v) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x)
    p[i] = v;
}

int fill_async(float* p, int64_t n, float v, cudaStream_t s) {
  if (n == 0) return PG_OK;
  const int blocks = int(std::min<int64_t>(ceil_div(n, 256), int64_t(num_sms()) * 8));
  fill_kernel<<<blocks, 256, 0, s>>>(p, n, v);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

namespace {

// Each thread owns one channel and walks a chunk of consecutive edges, keeping the running max
// of the current destination in a register; an atomic is issued only when the destination
// changes.  For destination-sorted input (the generator's order) that is ~1 atomic per
// (segment, chunk, channel); for arbitrary order it degrades gracefully to 1 per element.
constexpr int kScatterChunk = 64;
__global__ void __launch_bounds__(256) scatter_max_kernel(const float* __restrict__ feat,
                                                           const int32_t* __restrict__ centers, int64_t num_edges,
                                                           int num_channels, int64_t num_centers,
                                                           float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= num_channels) return;
  for (int64_t chunk = blockIdx.y; chunk * kScatterChunk < num_edges; chunk += gridDim.y) {
    const int64_t e0 = chunk * kScatterChunk;
    const int64_t e1 = min(e0 + kScatterChunk, num_edges);
    int cur = -1;
    float m = -FLT_MAX;
    for (int64_t e = e0; e < e1; ++e) {
      const int d = centers[e];
      if (d != cur) {
        if (cur >= 0 && cur < num_centers) atomic_max_float(out + int64_t(cur) * num_channels + c, m);
        cur = d;
        m = -FLT_MAX;
      }
      m = fmaxf(m, feat[e * num_channels + c]);
    }
    if (cur >= 0 && cur < num_centers) atomic_max_float(out + int64_t(cur) * num_channels + c, m);
  }
}

// Vectorised variant (C % 4 == 0, C / 4 <= 256): a thread owns FOUR channels of one edge stream; a block of
// 256 threads runs 256 / (C/4) streams side by side (C = 300: 3 streams x 75 threads), every stream walks its
// own 64-edge chunks, and the loads of 8 consecutive edges (8 independent LDG.128 per thread, 2 x C*4 bytes of
// fully used lines per edge) are issued before they are consumed.  HBM-bound: E*C*4 bytes are read once.
__global__ void __launch_bounds__(256) scatter_max_vec4_kernel(const float4* __restrict__ feat,
                                                                const int32_t* __restrict__ centers,
                                                                int64_t num_edges, int vecs_per_row, int64_t num_centers,
                                                                float* __restrict__ out) {
  const int streams = 256 / vecs_per_row;
  const int s = threadIdx.x / vecs_per_row, v = threadIdx.x - s * vecs_per_row;
  if (s >= streams) return;
  const int num_channels = vecs_per_row * 4;
  const int64_t num_chunks = (num_edges + kScatterChunk - 1) / kScatterChunk;
  auto flush = [&](int cur, const float4& m) {
    if (cur >= 0 && cur < num_centers) {
      float* o = out + int64_t(cur) * num_channels + 4 * v;
      atomic_max_float(o + 0, m.x);
      atomic_max_float(o + 1, m.y);
      atomic_max_float(o + 2, m.z);
      atomic_max_float(o + 3, m.w);
    }
  };
  for (int64_t chunk = int64_t(blockIdx.x) * streams + s; chunk < num_chunks; chunk += int64_t(gridDim.x) * streams) {
    const int64_t e0 = chunk * kScatterChunk;
    const int64_t e1 = min(e0 + kScatterChunk, num_edges);
    int cur = -1;
    float4 m = make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX);
    for (int64_t e = e0; e < e1; e += 8) {
      float4 val[8];
      int d[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const bool ok = e + i < e1;
        d[i] = ok ? __ldg(centers + e + i) : -1;
        val[i] = ok ? __ldg(feat + (e + i) * vecs_per_row + v) : make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (e + i >= e1) break;
        if (d[i] != cur) {
          flush(cur, m);
          cur = d[i];
          m = make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX);
        }
        m.x = fmaxf(m.x, val[i].x);
        m.y = fmaxf(m.y, val[i].y);
        m.z = fmaxf(m.z, val[i].z);
        m.w = fmaxf(m.w, val[i].w);
      }
    }
    flush(cur, m);
  }
}

// ---- graph_scatter_sum_fn / graph_scatter_mean_fn (gnn.py:111-119): tf.math.unsorted_segment_sum / _mean ----------
// Same streaming structure as the max: a thread walks a chunk of consecutive edges with a running partial sum per
// destination run and flushes it with one atomicAdd per (run, channel); sorted or unsorted ids both work (unsorted ids
// just flush every edge).  fp32 accumulation; the order of the partial sums is not fixed (atomics), as TF's GPU kernel.
__global__ void scatter_sum_kernel(const float* __restrict__ feat, const int32_t* __restrict__ centers, int64_t num_edges,
                                   int num_channels, int64_t num_centers, float* __restrict__ out,
                                   float* __restrict__ count) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= num_channels) return;
  const int64_t num_chunks = (num_edges + kScatterChunk - 1) / kScatterChunk;
  for (int64_t chunk = blockIdx.y; chunk < num_chunks; chunk += gridDim.y) {
    const int64_t e0 = chunk * kScatterChunk, e1 = min(e0 + kScatterChunk, num_edges);
    int cur = -1;
    float acc = 0.0f, n = 0.0f;
    for (int64_t e = e0; e < e1; ++e) {
      const int d = __ldg(centers + e);
      if (d != cur) {
        if (cur >= 0 && cur < num_centers) {
          atomicAdd(out + int64_t(cur) * num_channels + c, acc);
          if (count != nullptr && c == 0) atomicAdd(count + cur, n);
        }
        cur = d;
        acc = 0.0f;
        n = 0.0f;
      }
      acc += __ldg(feat + e * num_channels + c);
      n += 1.0f;
    }
    if (cur >= 0 && cur < num_centers) {
      atomicAdd(out + int64_t(cur) * num_channels + c, acc);
      if (count != nullptr && c == 0) atomicAdd(count + cur, n);
    }
  }
}

// The same with PG_FLAG_DETERMINISTIC, over the edges stable-sorted by id (order [e] = the input position of sorted edge
// e, sorted [e] its id; dropped ids sort last as num_centers): tile t of PG_ORDERED_SCATTER_TILE sorted edges is unit t
// of the ordered sum (pg_common.cuh), summed sequentially from 0 per destination.  The counts of the mean are integers
// added as floats: exact up to 2^24 edges per destination in any order, so they keep their atomics
__global__ void scatter_sum_ordered_kernel(const float* __restrict__ feat, const int32_t* __restrict__ order,
                                           const uint64_t* __restrict__ sorted, int64_t num_edges, int num_channels,
                                           int64_t num_centers, float* __restrict__ out, float* __restrict__ count,
                                           float* __restrict__ part, int32_t* __restrict__ part_id) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= num_channels) return;
  const int64_t num_chunks = (num_edges + PG_ORDERED_SCATTER_TILE - 1) / PG_ORDERED_SCATTER_TILE;
  for (int64_t chunk = blockIdx.y; chunk < num_chunks; chunk += gridDim.y) {
    const int64_t e0 = chunk * PG_ORDERED_SCATTER_TILE, e1 = min(e0 + PG_ORDERED_SCATTER_TILE, num_edges);
    int64_t cur = -1;
    int runs = 0;
    float acc = 0.0f, n = 0.0f;
    auto flush = [&](bool last) {
      if (cur < 0 || cur >= num_centers) return;
      const int slot = runs == 0 ? 0 : last ? 1 : -1;
      if (slot < 0) {
        out[cur * num_channels + c] = acc;
      } else {
        part[(2 * chunk + slot) * num_channels + c] = acc;
        if (c == 0) part_id[2 * chunk + slot] = int32_t(cur);
      }
      if (count != nullptr && c == 0) atomicAdd(count + cur, n);
      ++runs;
    };
    for (int64_t e = e0; e < e1; ++e) {
      const int64_t d = int64_t(__ldg(sorted + e));
      if (d != cur) {
        flush(false);
        cur = d;
        acc = 0.0f;
        n = 0.0f;
      }
      acc += __ldg(feat + int64_t(__ldg(order + e)) * num_channels + c);
      n += 1.0f;
    }
    flush(true);
  }
}

// The fix-up of the ordered segment sum (pg_common.cuh): thread (slot, column).  A destination's chain can only go on
// from one unit into the next through the next unit's slot 0 (its run holds that unit's first row), so an empty slot 0
// ends every chain and the walks stay within one chain.  The first slot of a chain (no slot of the previous unit
// continues into it) adds the chain's partial rows in ascending slot order and adds the total into out; the edges are
// grouped by destination, so no other thread writes that row
__global__ void ordered_fixup_kernel(const float* __restrict__ part, const int32_t* __restrict__ part_id, int64_t slots,
                                     int n, float* __restrict__ out, int ldo) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < slots * n; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t slot = i / n;
    const int c = int(i - slot * n);
    const int32_t d = part_id[slot];
    if (d < 0) continue;
    if ((slot & 1) == 0 && slot > 0) {
      // slot 0 of its unit: a chain goes on into it from the previous unit's last run (slot 1, or slot 0 when that
      // unit had one run)
      const int32_t prev = part_id[slot - 1] >= 0 ? part_id[slot - 1] : part_id[slot - 2];
      if (prev == d) continue;
    } else if (slot & 1) {
      if (part_id[slot - 1] == d) continue;   // cannot happen (two runs of one unit), kept for safety
    }
    float t = part[slot * n + c];
    for (int64_t j = slot + 1; j < slots; ++j) {
      const int32_t dj = part_id[j];
      if (dj < 0) {
        if ((j & 1) == 0) break;   // an empty slot 0: the next unit does not continue the chain
        continue;
      }
      if (dj != d) break;
      t += part[j * n + c];
    }
    float* o = out + int64_t(d) * ldo + c;
    *o = *o + t;
  }
}

__global__ void divide_rows_kernel(float* __restrict__ out, const float* __restrict__ count, int64_t num_centers,
                                   int num_channels) {
  const int64_t total = num_centers * num_channels;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x)
    out[i] = out[i] / fmaxf(count[i / num_channels], 1.0f);      // unsorted_segment_mean: empty segment -> 0
}

__global__ void gather_rows_kernel(const float* __restrict__ params, int64_t num_rows, int num_channels,
                                   const int32_t* __restrict__ indices, int64_t num_indices,
                                   float* __restrict__ out, int* __restrict__ err) {
  const int64_t total = num_indices * num_channels;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t r = i / num_channels;
    const int c = int(i - r * num_channels);
    const int32_t j = indices[r];
    if (j < 0 || j >= num_rows) { *err = 1; continue; }
    out[i] = params[int64_t(j) * num_channels + c];
  }
}

// ---- fp32 fully-connected: out = act(x @ w + b) (+ residual) ---------------------------------
// 64x64 output tile, 16-deep k slices staged in shared memory, 4x4 register micro-tile, FFMA
// accumulation in ascending k (the same association order as a naive CPU loop).
constexpr int kTM = 64, kTN = 64, kTK = 16;
__global__ void __launch_bounds__(256) fc_fp32_kernel(const float* __restrict__ x, int64_t m, int k,
                                                       const float* __restrict__ w, const float* __restrict__ bias,
                                                       int n, int act, const float* __restrict__ residual,
                                                       float* __restrict__ out, int ldo) {
  __shared__ float xs[kTK][kTM + 4];
  __shared__ float ws[kTK][kTN + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t row0 = int64_t(blockIdx.y) * kTM;
  const int col0 = blockIdx.x * kTN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
  for (int k0 = 0; k0 < k; k0 += kTK) {
    // x tile: 64 rows x 16 k  (thread t loads 4 elements)
    for (int t = threadIdx.x; t < kTM * kTK; t += 256) {
      const int r = t / kTK, kk = t % kTK;
      const int64_t gr = row0 + r;
      xs[kk][r] = (gr < m && k0 + kk < k) ? x[gr * k + k0 + kk] : 0.0f;
    }
    for (int t = threadIdx.x; t < kTK * kTN; t += 256) {
      const int kk = t / kTN, cidx = t % kTN;
      ws[kk][cidx] = (k0 + kk < k && col0 + cidx < n) ? w[int64_t(k0 + kk) * n + col0 + cidx] : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kTK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = xs[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = ws[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t gr = row0 + ty * 4 + i;
    if (gr >= m) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gc = col0 + tx * 4 + j;
      if (gc >= ldo) continue;
      if (gc >= n) { out[gr * ldo + gc] = 0.0f; continue; }   // zero padding columns [n, ldo)
      float v = acc[i][j] + bias[gc];
      v = activate(act, v);
      if (residual != nullptr) v += residual[gr * n + gc];
      out[gr * ldo + gc] = v;
    }
  }
}

__global__ void activate_rows_kernel(float* __restrict__ out, int64_t rows, int n, int ldo, const float* __restrict__ bias,
                                     int act, const float* __restrict__ residual, int ldr, bool skip_empty) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < rows * n; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t r = i / n;
    const int c = int(i - r * n);
    float v = out[r * ldo + c];
    if (skip_empty && v == -FLT_MAX) continue;
    v = activate(act, bias ? v + bias[c] : v);
    if (residual) v += residual[r * ldr + c];
    out[r * ldo + c] = v;
  }
}

__global__ void check_edges_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ dst, int64_t n,
                                   int64_t num_src, int64_t num_dst, int* __restrict__ err) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
    const int a = src[i], b = dst[i];
    if (a < 0 || a >= num_src || b < 0 || b >= num_dst) *err = 1;
  }
}

__global__ void softmax_rows_kernel(const float* __restrict__ logits, int64_t num_rows, int num_classes,
                                    float* __restrict__ out) {
  const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= num_rows) return;
  const float* in = logits + r * num_classes;
  float mx = -FLT_MAX;
  for (int c = 0; c < num_classes; ++c) mx = fmaxf(mx, in[c]);
  float sum = 0.0f;
  for (int c = 0; c < num_classes; ++c) sum += expf(in[c] - mx);
  for (int c = 0; c < num_classes; ++c) out[r * num_classes + c] = expf(in[c] - mx) / sum;
}

}  // namespace

// out has row stride ldo >= n; columns [n, ldo) are written as zeros (ldo <= n rounded up to 64)
int fc_fp32_launch(const float* x, int64_t m, int k, const float* w, const float* bias, int n, int act,
                   const float* residual, float* out, int ldo, cudaStream_t s) {
  PG_REQUIRE(ldo >= n && ldo <= (n + kTN - 1) / kTN * kTN, "fc: bad output stride %d for n=%d", ldo, n);
  dim3 grid(ceil_div(n, kTN), ceil_div(m, kTM));
  fc_fp32_kernel<<<grid, 256, 0, s>>>(x, m, k, w, bias, n, act, residual, out, ldo);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

int OrderedParts::alloc(int64_t units, int cols, cudaStream_t s) {
  slots = 2 * units;
  n = cols;
  PG_CUDA_OK(val.alloc(sizeof(float) * size_t(slots) * n, s));
  PG_CUDA_OK(id.alloc(sizeof(int32_t) * size_t(slots), s));
  return reset(s);
}

int OrderedParts::reset(cudaStream_t s) {
  PG_CUDA_OK(cudaMemsetAsync(id.ptr, 0xff, sizeof(int32_t) * size_t(slots), s));
  return PG_OK;
}

int ordered_fixup(const OrderedParts& parts, float* out, int ldo, cudaStream_t s) {
  if (parts.slots == 0) return PG_OK;
  const int blocks = int(std::min<int64_t>(ceil_div(parts.slots * parts.n, 256), int64_t(num_sms()) * 8));
  ordered_fixup_kernel<<<blocks, 256, 0, s>>>(parts.v(), parts.i(), parts.slots, parts.n, out, ldo);
  PG_LAUNCH_CHECK();
  count_ordered_launch();
  return PG_OK;
}

// the in-degree histogram of an edge list: one atomic per edge (the counts are integers, exact in fp32 up to 2^24 in
// any order: the ordered segment sum's mean divides by them as they are)
__global__ void count_segments_kernel(const int32_t* __restrict__ dst, int64_t num_edges, int64_t num_dst,
                                      float* __restrict__ count) {
  for (int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; e < num_edges; e += int64_t(gridDim.x) * blockDim.x) {
    const int d = __ldg(dst + e);
    if (d >= 0 && d < num_dst) atomicAdd(count + d, 1.0f);
  }
}

int divide_by_segment_count(float* out, int64_t num_dst, int n, const int32_t* dst, int64_t num_edges, cudaStream_t s) {
  if (num_dst == 0 || num_edges == 0) return PG_OK;
  Temp count;
  PG_CUDA_OK(count.alloc(sizeof(float) * num_dst, s));
  PG_CUDA_OK(cudaMemsetAsync(count.ptr, 0, sizeof(float) * num_dst, s));
  count_segments_kernel<<<int(std::min<int64_t>(ceil_div(num_edges, 256), int64_t(num_sms()) * 8)), 256, 0, s>>>(
      dst, num_edges, num_dst, count.as<float>());
  PG_LAUNCH_CHECK();
  const int blocks = int(std::min<int64_t>(ceil_div(num_dst * n, 256), int64_t(num_sms()) * 8));
  divide_rows_kernel<<<blocks, 256, 0, s>>>(out, count.as<float>(), num_dst, n);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

int activate_rows(float* out, int64_t rows, int n, int ldo, const float* bias, int act, const float* residual, int ldr,
                  bool skip_empty, cudaStream_t s) {
  if (rows == 0) return PG_OK;
  const int grid = int(std::min<int64_t>(ceil_div(rows * n, 256), int64_t(num_sms()) * 8));
  activate_rows_kernel<<<grid, 256, 0, s>>>(out, rows, n, ldo, bias, act, residual, ldr, skip_empty);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

namespace {

// the keys of the stable order by id: ids outside [0, num_ids) become num_ids and sort after every kept one
__global__ void order_keys_kernel(const int32_t* __restrict__ ids, int64_t n, int64_t num_ids, uint64_t* __restrict__ keys,
                                  int32_t* __restrict__ pos) {
  for (int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; e < n; e += int64_t(gridDim.x) * blockDim.x) {
    const int32_t d = ids[e];
    keys[e] = d >= 0 && d < num_ids ? uint64_t(d) : uint64_t(num_ids);
    pos[e] = int32_t(e);
  }
}

__global__ void gather_i32_kernel(const int32_t* __restrict__ in, const int32_t* __restrict__ order, int64_t n,
                                  int32_t* __restrict__ out) {
  for (int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; e < n; e += int64_t(gridDim.x) * blockDim.x)
    out[e] = in[order[e]];
}

}  // namespace

int stable_order(const int32_t* ids, int64_t n, int64_t num_ids, Temp& keys_sorted, Temp& order, cudaStream_t s) {
  PG_REQUIRE(n < (int64_t(1) << 31), "ordered segment sum: %lld edges (int32 positions)", (long long)n);
  Temp keys, pos;
  PG_CUDA_OK(keys.alloc(sizeof(uint64_t) * n, s));
  PG_CUDA_OK(keys_sorted.alloc(sizeof(uint64_t) * n, s));
  PG_CUDA_OK(pos.alloc(sizeof(int32_t) * n, s));
  PG_CUDA_OK(order.alloc(sizeof(int32_t) * n, s));
  if (n == 0) return PG_OK;
  order_keys_kernel<<<int(std::min<int64_t>(ceil_div(n, 256), int64_t(num_sms()) * 8)), 256, 0, s>>>(
      ids, n, num_ids, keys.as<uint64_t>(), pos.as<int32_t>());
  PG_LAUNCH_CHECK();
  int end_bit = 1;
  while (end_bit < 64 && (uint64_t(num_ids) >> end_bit) != 0) ++end_bit;
  return sort_pairs(keys.as<uint64_t>(), keys_sorted.as<uint64_t>(), pos.as<int32_t>(), order.as<int32_t>(), n, end_bit,
                    s);
}

int sort_edges_by_dst(const int32_t* src, const int32_t* dst, int64_t n, int64_t num_dst, Temp& src_s, Temp& dst_s,
                      cudaStream_t s) {
  Temp keys, order;
  if (int rc = stable_order(dst, n, num_dst, keys, order, s)) return rc;
  PG_CUDA_OK(src_s.alloc(sizeof(int32_t) * n, s));
  PG_CUDA_OK(dst_s.alloc(sizeof(int32_t) * n, s));
  if (n == 0) return PG_OK;
  const int blocks = int(std::min<int64_t>(ceil_div(n, 256), int64_t(num_sms()) * 8));
  gather_i32_kernel<<<blocks, 256, 0, s>>>(src, order.as<int32_t>(), n, src_s.as<int32_t>());
  PG_LAUNCH_CHECK();
  gather_i32_kernel<<<blocks, 256, 0, s>>>(dst, order.as<int32_t>(), n, dst_s.as<int32_t>());
  PG_LAUNCH_CHECK();
  return PG_OK;
}

}  // namespace pg

using namespace pg;

extern "C" int pg_scatter_max(const float* features, const int32_t* centers, int64_t num_edges, int32_t num_channels,
                              int64_t num_centers, float* out, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(out != nullptr || num_centers == 0, "pg_scatter_max: out is null");
  PG_REQUIRE(num_channels >= 1 && num_edges >= 0 && num_centers >= 0, "pg_scatter_max: bad sizes");
  if (int rc = fill_async(out, num_centers * num_channels, -FLT_MAX, s)) return rc;
  if (num_edges == 0) return PG_OK;
  PG_REQUIRE(features && centers, "pg_scatter_max: null input");
  const int64_t chunks = ceil_div(num_edges, kScatterChunk);
  if ((num_channels & 3) == 0 && num_channels / 4 <= 256 && (reinterpret_cast<uintptr_t>(features) & 15) == 0) {
    const int vecs = num_channels / 4, streams = 256 / vecs;
    const int blocks = int(std::min<int64_t>(ceil_div(chunks, streams), int64_t(num_sms()) * 8));
    scatter_max_vec4_kernel<<<blocks, 256, 0, s>>>(reinterpret_cast<const float4*>(features), centers, num_edges, vecs,
                                                   num_centers, out);
    PG_LAUNCH_CHECK();
    return PG_OK;
  }
  const int threads = num_channels >= 256 ? 256 : (num_channels >= 128 ? 128 : (num_channels >= 64 ? 64 : 32));
  dim3 grid(ceil_div(num_channels, threads), int(std::min<int64_t>(chunks, 65535)));
  scatter_max_kernel<<<grid, threads, 0, s>>>(features, centers, num_edges, num_channels, num_centers, out);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

static int scatter_sum_impl(const float* features, const int32_t* centers, int64_t num_edges, int32_t num_channels,
                            int64_t num_centers, float* out, bool mean, int32_t flags, cudaStream_t s) {
  PG_REQUIRE(out != nullptr || num_centers == 0, "pg_scatter_sum: out is null");
  PG_REQUIRE(num_channels >= 1 && num_edges >= 0 && num_centers >= 0, "pg_scatter_sum: bad sizes");
  PG_REQUIRE((flags & ~PG_FLAG_DETERMINISTIC) == 0, "pg_scatter_sum: unknown flags 0x%x", flags);
  const bool ordered = (flags & PG_FLAG_DETERMINISTIC) != 0;
  if (num_centers == 0) return PG_OK;
  PG_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(float) * num_centers * num_channels, s));
  if (num_edges == 0) return PG_OK;
  PG_REQUIRE(features && centers, "pg_scatter_sum: null input");
  Temp count;
  if (mean) {
    PG_CUDA_OK(count.alloc(sizeof(float) * num_centers, s));
    PG_CUDA_OK(cudaMemsetAsync(count.ptr, 0, sizeof(float) * num_centers, s));
  }
  const int threads = num_channels >= 256 ? 256 : (num_channels >= 128 ? 128 : (num_channels >= 64 ? 64 : 32));
  if (ordered) {
    Temp keys_s, order;
    if (int rc = stable_order(centers, num_edges, num_centers, keys_s, order, s)) return rc;
    const int64_t chunks = ceil_div(num_edges, PG_ORDERED_SCATTER_TILE);
    OrderedParts parts;
    if (int rc = parts.alloc(chunks, num_channels, s)) return rc;
    dim3 grid(ceil_div(num_channels, threads), int(std::min<int64_t>(chunks, 65535)));
    scatter_sum_ordered_kernel<<<grid, threads, 0, s>>>(features, order.as<int32_t>(), keys_s.as<uint64_t>(), num_edges,
                                                        num_channels, num_centers, out,
                                                        mean ? count.as<float>() : nullptr, parts.v(), parts.i());
    PG_LAUNCH_CHECK();
    if (int rc = ordered_fixup(parts, out, num_channels, s)) return rc;
  } else {
    const int64_t chunks = ceil_div(num_edges, kScatterChunk);
    dim3 grid(ceil_div(num_channels, threads), int(std::min<int64_t>(chunks, 65535)));
    scatter_sum_kernel<<<grid, threads, 0, s>>>(features, centers, num_edges, num_channels, num_centers, out,
                                                mean ? count.as<float>() : nullptr);
    PG_LAUNCH_CHECK();
  }
  if (mean) {
    const int blocks = int(std::min<int64_t>(ceil_div(num_centers * num_channels, 256), int64_t(num_sms()) * 8));
    divide_rows_kernel<<<blocks, 256, 0, s>>>(out, count.as<float>(), num_centers, num_channels);
    PG_LAUNCH_CHECK();
  }
  return PG_OK;
}

extern "C" int pg_scatter_sum(const float* features, const int32_t* centers, int64_t num_edges, int32_t num_channels,
                              int64_t num_centers, float* out, void* stream) {
  return scatter_sum_impl(features, centers, num_edges, num_channels, num_centers, out, false, 0,
                          static_cast<cudaStream_t>(stream));
}

extern "C" int pg_scatter_mean(const float* features, const int32_t* centers, int64_t num_edges, int32_t num_channels,
                               int64_t num_centers, float* out, void* stream) {
  return scatter_sum_impl(features, centers, num_edges, num_channels, num_centers, out, true, 0,
                          static_cast<cudaStream_t>(stream));
}

extern "C" int pg_scatter_sum_flags(const float* features, const int32_t* centers, int64_t num_edges,
                                    int32_t num_channels, int64_t num_centers, float* out, int32_t flags, void* stream) {
  return scatter_sum_impl(features, centers, num_edges, num_channels, num_centers, out, false, flags,
                          static_cast<cudaStream_t>(stream));
}

extern "C" int pg_scatter_mean_flags(const float* features, const int32_t* centers, int64_t num_edges,
                                     int32_t num_channels, int64_t num_centers, float* out, int32_t flags,
                                     void* stream) {
  return scatter_sum_impl(features, centers, num_edges, num_channels, num_centers, out, true, flags,
                          static_cast<cudaStream_t>(stream));
}

extern "C" int pg_gather_rows(const float* params, int64_t num_rows, int32_t num_channels, const int32_t* indices,
                              int64_t num_indices, float* out, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (num_indices == 0) return PG_OK;
  PG_REQUIRE(params && indices && out && num_channels >= 1, "pg_gather_rows: bad argument");
  ErrorWord err;
  if (int rc = err.init(s)) return rc;
  const int64_t total = num_indices * num_channels;
  const int blocks = int(std::min<int64_t>(ceil_div(total, 256), int64_t(num_sms()) * 16));
  gather_rows_kernel<<<blocks, 256, 0, s>>>(params, num_rows, num_channels, indices, num_indices, out, err.ptr());
  PG_LAUNCH_CHECK();
  int h = 0;
  if (int rc = err.read(&h, false, s)) return rc;
  PG_REQUIRE(h == 0, "pg_gather_rows: index out of range [0,%lld)", (long long)num_rows);  // TF: InvalidArgumentError
  return PG_OK;
}

extern "C" int pg_check_edges(const int32_t* src, const int32_t* dst, int64_t num_edges, int64_t num_src,
                              int64_t num_dst, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (num_edges == 0) return PG_OK;
  PG_REQUIRE(src && dst && num_edges > 0, "pg_check_edges: bad argument");
  ErrorWord err;
  if (int rc = err.init(s)) return rc;
  const int blocks = int(std::min<int64_t>(ceil_div(num_edges, 256), int64_t(num_sms()) * 8));
  check_edges_kernel<<<blocks, 256, 0, s>>>(src, dst, num_edges, num_src, num_dst, err.ptr());
  PG_LAUNCH_CHECK();
  int h = 0;
  if (int rc = err.read(&h, false, s)) return rc;
  PG_REQUIRE(h == 0, "edge index out of range (src in [0,%lld), dst in [0,%lld))", (long long)num_src,
             (long long)num_dst);   // TF: InvalidArgumentError
  return PG_OK;
}

extern "C" int pg_softmax_rows(const float* logits, int64_t num_rows, int32_t num_classes, float* out, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (num_rows == 0) return PG_OK;
  PG_REQUIRE(logits && out && num_classes >= 1, "pg_softmax_rows: bad argument");
  softmax_rows_kernel<<<ceil_div(num_rows, 128), 128, 0, s>>>(logits, num_rows, num_classes, out);
  PG_LAUNCH_CHECK();
  return PG_OK;
}
