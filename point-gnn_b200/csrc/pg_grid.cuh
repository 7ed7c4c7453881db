// The sorted-key uniform grid of pg_graph.cu, for the source files that voxelise a cloud with it: the grid
// description, the sorted view the kernels read, and the host functions that build it and close a call on it.
#pragma once
#include "pg_common.cuh"

namespace pg {

// How a point's cell index follows from its coordinates and the bounding-box minimum of its frame.
enum class CellRule : int {
  // open3d.voxel_down_sample (graph_gen.py:41-45): origin = frame_min - cell / 2, floor((p - origin) / cell) in fp64
  kVoxel,
  // radius and nearest-vertex search grids: origin = frame_min, floor((p - origin) / cell) in fp64 on the coordinates
  // divided by `scale` if `scaled`
  kRadius,
  // multi_layer_downsampling_random without add_rnd3d (graph_gen.py:124-126) and downsample_by_average_voxel
  // (kitti_dataset.py:23-28): floor_divide(p - frame_min, cell) in float32
  kNumpyF32,
  // add_rnd3d (graph_gen.py:24-31, 127-130): floor_divide((p - frame_min)[float32] + cell * shift[frame], cell) in
  // float64, shift = the np.random.random((1, 3)) draw of the frame
  kNumpyF64Shift,
};

// Grid description shared by key generation and queries.
struct GridSpec {
  double cell[3];     // cell edge per axis
  CellRule rule;
  // gen_disjointed_rnn_local_graph_v3's `scale` (graph_gen.py:203-206): every coordinate is DIVIDED by scale[axis] in
  // float64 before anything else (points_xyz / np.array(scale) -> float64).  scaled == 0: coordinates as they are.
  int scaled;
  double scale[3];
  const double* shift;   // kNumpyF64Shift: [num_frames][3] on the device
};

// A point's 64-bit key is frame(16) | iz(16) | iy(16) | ix(16): ascending key order is, inside a frame, the order of
// the linear voxel key ix + iy * dim_x + iz * dim_y * dim_x.
struct SortedGrid {
  const uint64_t* cell_key;   // [num_cells]
  const int32_t* cell_start;  // [num_cells+1]
  const float4* pts;          // [n] sorted (x,y,z,orig idx)
  const int32_t* num_cells;   // device scalar (= last element of the head-flag scan): no host round trip
};

struct BuiltGrid {
  Temp bounds, keys_a, keys_b, vals_a, vals_b, sorted_pts, head, head_scan, cell_key, cell_start, err;
  SortedGrid view{};
};

// fp64 centroid of the sorted points [s, e) of one voxel, summed in ascending point order (the sort is stable)
__device__ inline void voxel_centroid(const SortedGrid& g, int s, int e, double c[3]) {
  double sx = 0.0, sy = 0.0, sz = 0.0;
  for (int i = s; i < e; ++i) {
    const float4 p = g.pts[i];
    sx = __dadd_rn(sx, double(p.x));
    sy = __dadd_rn(sy, double(p.y));
    sz = __dadd_rn(sz, double(p.z));
  }
  const double cnt = double(e - s);
  c[0] = __ddiv_rn(sx, cnt);
  c[1] = __ddiv_rn(sy, cnt);
  c[2] = __ddiv_rn(sz, cnt);
}

// pg_graph.cu.  `spec` with one cell edge per axis (all positive, else PG_ERR_INVALID_ARGUMENT) and no scale
int voxel_spec(const double* voxel_size_host, CellRule rule, GridSpec* spec);
// Sorts the n points of the frames into `out` (n >= 1).  No host round trip: the number of occupied cells stays on the
// device (out->view.num_cells) and out->err is the device error word of the call, which graph_error decodes.
int build_grid(const float* xyz, const int32_t* frame_ptr, int num_frames, int64_t n, const GridSpec& spec,
               cudaStream_t s, BuiltGrid* out, const int32_t* n_valid = nullptr);
// out_frame_ptr[f] = first of the *num_keys sorted keys whose frame field (bits from `frame_shift` up) is >= f
int frame_ranges(const uint64_t* keys, const int32_t* num_keys, int num_frames, int frame_shift, int32_t* out_frame_ptr,
                 cudaStream_t s);
// PG_OK, or the error a device error word stands for (with its message set)
int graph_error(int err);

}  // namespace pg
