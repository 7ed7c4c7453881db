// Voxel averaging of the input cloud on the GPU: the reference's `downsample_by_voxel_size` config key.
//
// Replaces, for a batch of frames,
//   dataset/kitti_dataset.py:16-48   downsample_by_average_voxel: xyz_idx = ((xyz - min) // voxel_size).astype(int32)
//                                    on float32 values, key = ix + iy * dim_x + iz * dim_y * dim_x, one point per
//                                    occupied voxel in ascending key order, xyz and attr = the voxel's means
//   dataset/kitti_dataset.py:624-626 its call from get_cam_points, on the camera-frame cloud, ahead of the image crop
// The voxels are the cells of pg_graph.cu's sorted grid under the NumPy float32 floor_divide rule; its key orders a
// frame's voxels as the linear key does (iz major, ix minor).
//
// Two things the reference's code does are not reproduced, on purpose:
//  * Its sums are float32 np.add.reduceat in np.argsort(keys) order.  That sort is not stable, so the order of addition
//    inside a voxel is unspecified.  Here: fp64 sums in original point order (the radix sort is stable).  Which points
//    share a voxel, the number of voxels and their order are exact; the means agree within 1e-4.
//  * float32 / int64 makes its means float64, and its graph is built from them.  Here the fp64 mean is rounded once to
//    float32, and that array is the cloud for everything downstream.
// Its int32 key wraps when dim_x * dim_y * dim_z exceeds 2^31 - 1 (a tiny voxel size); that is an error here.
#include <vector>

#include "pg_grid.cuh"

namespace pg {
namespace {

constexpr int kMaxAttr = 4;

// One thread per occupied voxel v: the means of its points, written at its rank, and the cell count its frame needs
// per axis (dims [num_frames][3], zero-initialised).
__global__ void voxel_average_kernel(SortedGrid g, const float* __restrict__ attr, int channels, int64_t capacity,
                                     float* __restrict__ out_xyz, float* __restrict__ out_attr, int32_t* __restrict__ dims) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = v < __ldg(g.num_cells);
  int f = -1, ix = 0, iy = 0, iz = 0;
  if (active) {
    const uint64_t key = g.cell_key[v];
    f = int(key >> 48);
    iz = int((key >> 32) & 0xffff) + 1;
    iy = int((key >> 16) & 0xffff) + 1;
    ix = int(key & 0xffff) + 1;
    if (v < capacity) {
      const int s = g.cell_start[v], e = g.cell_start[v + 1];
      double c[3];
      voxel_centroid(g, s, e, c);
      out_xyz[3 * int64_t(v) + 0] = __double2float_rn(c[0]);
      out_xyz[3 * int64_t(v) + 1] = __double2float_rn(c[1]);
      out_xyz[3 * int64_t(v) + 2] = __double2float_rn(c[2]);
      double sum[kMaxAttr] = {0.0, 0.0, 0.0, 0.0};
      for (int i = s; i < e; ++i) {
        const int64_t j = __float_as_int(g.pts[i].w);
#pragma unroll
        for (int ch = 0; ch < kMaxAttr; ++ch)
          if (ch < channels) sum[ch] = __dadd_rn(sum[ch], double(attr[j * channels + ch]));
      }
#pragma unroll
      for (int ch = 0; ch < kMaxAttr; ++ch)
        if (ch < channels) out_attr[int64_t(v) * channels + ch] = __double2float_rn(__ddiv_rn(sum[ch], double(e - s)));
    }
  }
  // a warp's voxels are consecutive keys, so nearly always one frame: one atomic per axis then
  const int f0 = __shfl_sync(0xffffffffu, f, 0);
  if (__all_sync(0xffffffffu, f == f0)) {
    if (f0 < 0) return;
    ix = __reduce_max_sync(0xffffffffu, ix);
    iy = __reduce_max_sync(0xffffffffu, iy);
    iz = __reduce_max_sync(0xffffffffu, iz);
    if ((threadIdx.x & 31) != 0) return;
  } else if (!active) {
    return;
  }
  atomicMax(&dims[3 * f + 0], ix);
  atomicMax(&dims[3 * f + 1], iy);
  atomicMax(&dims[3 * f + 2], iz);
}

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" int pg_voxel_average(const float* xyz, const float* attr, int32_t attr_channels, const int32_t* frame_ptr,
                                int32_t num_frames, int64_t num_points, double voxel_size, float* out_xyz,
                                float* out_attr, int64_t capacity, int32_t* out_frame_ptr, int64_t* out_num_host,
                                void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(frame_ptr && out_frame_ptr && out_num_host, "pg_voxel_average: null argument");
  PG_REQUIRE(attr_channels >= 0 && attr_channels <= kMaxAttr, "pg_voxel_average: attr_channels=%d out of range [0,%d]",
             attr_channels, kMaxAttr);
  // the comparison is false for NaN; the reference divides by the float32 value, which must not be 0 or inf either
  PG_REQUIRE(voxel_size > 0.0 && float(voxel_size) > 0.0f && float(voxel_size) <= FLT_MAX,
             "pg_voxel_average: voxel_size must be positive and finite, got %g", voxel_size);
  PG_REQUIRE(num_frames >= 1 && num_frames <= 65534, "num_frames=%d out of range [1,65534]", num_frames);
  PG_REQUIRE(num_points >= 0, "pg_voxel_average: num_points=%lld", (long long)num_points);
  *out_num_host = 0;
  if (num_points == 0) {
    PG_CUDA_OK(cudaMemsetAsync(out_frame_ptr, 0, sizeof(int32_t) * (num_frames + 1), s));
    return PG_OK;
  }
  PG_REQUIRE(xyz && out_xyz && (attr_channels == 0 || (attr && out_attr)), "pg_voxel_average: null argument");
  const double cell[3] = {voxel_size, voxel_size, voxel_size};
  GridSpec spec;
  if (int rc = voxel_spec(cell, CellRule::kNumpyF32, &spec)) return rc;
  BuiltGrid grid;
  if (int rc = build_grid(xyz, frame_ptr, num_frames, num_points, spec, s, &grid)) return rc;
  Temp dims;
  PG_CUDA_OK(dims.alloc(sizeof(int32_t) * 3 * num_frames, s));
  PG_CUDA_OK(cudaMemsetAsync(dims.ptr, 0, sizeof(int32_t) * 3 * num_frames, s));
  // the number of occupied voxels <= N is only known on the device: launch for N, surplus threads do nothing
  voxel_average_kernel<<<ceil_div(num_points, 128), 128, 0, s>>>(grid.view, attr, attr_channels, capacity, out_xyz,
                                                                  out_attr, dims.as<int32_t>());
  PG_LAUNCH_CHECK();
  if (int rc = frame_ranges(grid.view.cell_key, grid.view.num_cells, num_frames, 48, out_frame_ptr, s)) return rc;
  // the one host round trip: the voxel count, the grid's error word and the cell counts of the frames
  int32_t h[2] = {0, 0};
  std::vector<int32_t> h_dims(3 * size_t(num_frames));
  PG_CUDA_OK(cudaMemcpyAsync(&h[0], grid.view.num_cells, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaMemcpyAsync(&h[1], grid.err.ptr, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaMemcpyAsync(h_dims.data(), dims.ptr, sizeof(int32_t) * h_dims.size(), cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaStreamSynchronize(s));
  if (int rc = graph_error(h[1])) return rc;
  for (int f = 0; f < num_frames; ++f) {
    const int64_t cells = int64_t(h_dims[3 * f]) * h_dims[3 * f + 1] * h_dims[3 * f + 2];   // <= 2^48
    PG_REQUIRE(cells <= INT32_MAX,
               "pg_voxel_average: frame %d has %d x %d x %d voxels of size %g, more than the 2^31 - 1 an int32 voxel key "
               "can number",
               f, h_dims[3 * f], h_dims[3 * f + 1], h_dims[3 * f + 2], voxel_size);
  }
  *out_num_host = h[0];
  if (h[0] > capacity) {
    set_error("voxel buffer too small: need %d, capacity %lld", h[0], (long long)capacity);
    return PG_ERR_CAPACITY;
  }
  return PG_OK;
}
