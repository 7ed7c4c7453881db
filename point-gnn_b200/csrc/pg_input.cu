// Input stage on the GPU: the step right before the message-passing path (SURVEY 8f-2).
//
// Replaces, for a batch of frames and without a host round trip before the graph kernels,
//   dataset/kitti_dataset.py:998-1006  velo_points_to_cam   cam = velo @ R (float32) + t (float32)
//   dataset/kitti_dataset.py:666-689   get_cam_points_in_image_with_rgb: keep points with z > 0.1 whose image
//                                      projection ([x y z 1] @ cam_to_image^T in float64, :1036-1052) lies strictly
//                                      inside the image; optional colour lookup (:990-996)
//   run.py:236-237 / train.py:99-111   the `input_features` selection ('i' = reflectance, 'irgb', ...) is left to
//                                      the caller: attr = [reflectance, r, g, b] (rgb only when an image is given)
// The velodyne .bin read (kitti_dataset.py:587-609) is a host file read; its bytes are copied to the device as they
// are ([M, 4] float32) and everything after that runs here.  Output order = input order (stable compaction).
#include <vector>

#include "pg_common.cuh"

namespace pg {
namespace {

struct FrameCalib {
  float r[9];        // transpose(velo_to_cam)[:3,:3] as float32, row-major: cam = velo @ r
  float t[3];        // transpose(velo_to_cam)[3,:3] as float32
  double p[12];      // cam_to_image [3,4], float64
  int width, height;
};

__device__ inline int frame_of(const int32_t* __restrict__ frame_ptr, int num_frames, int64_t row) {
  int lo = 0, hi = num_frames;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (frame_ptr[mid] <= row) lo = mid; else hi = mid;
  }
  return lo;
}

// float32 product-sum in the order of a plain dot product: (x r0 + y r1) + z r2, each operation rounded
__device__ __forceinline__ float dot3_rn(float x, float y, float z, float a, float b, float c) {
  return __fadd_rn(__fadd_rn(__fmul_rn(x, a), __fmul_rn(y, b)), __fmul_rn(z, c));
}

__global__ void cam_flag_kernel(const float* __restrict__ velo, const int32_t* __restrict__ frame_ptr, int num_frames,
                                int64_t n, const FrameCalib* __restrict__ calib, float* __restrict__ cam_xyz,
                                float* __restrict__ uv, int32_t* __restrict__ flags) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const FrameCalib& c = calib[frame_of(frame_ptr, num_frames, i)];
  const float4 v = reinterpret_cast<const float4*>(velo)[i];
  const float x = __fadd_rn(dot3_rn(v.x, v.y, v.z, c.r[0], c.r[3], c.r[6]), c.t[0]);
  const float y = __fadd_rn(dot3_rn(v.x, v.y, v.z, c.r[1], c.r[4], c.r[7]), c.t[1]);
  const float z = __fadd_rn(dot3_rn(v.x, v.y, v.z, c.r[2], c.r[5], c.r[8]), c.t[2]);
  cam_xyz[3 * i + 0] = x;
  cam_xyz[3 * i + 1] = y;
  cam_xyz[3 * i + 2] = z;
  // cam_points_to_image (kitti_dataset.py:1036-1052) in float64
  const double X = double(x), Y = double(y), Z = double(z);
  const double iu = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(X, c.p[0]), __dmul_rn(Y, c.p[1])), __dmul_rn(Z, c.p[2])), c.p[3]);
  const double iv = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(X, c.p[4]), __dmul_rn(Y, c.p[5])), __dmul_rn(Z, c.p[6])), c.p[7]);
  const double iw = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(X, c.p[8]), __dmul_rn(Y, c.p[9])), __dmul_rn(Z, c.p[10])), c.p[11]);
  const double u = __ddiv_rn(iu, iw), w = __ddiv_rn(iv, iw);
  uv[2 * i + 0] = float(u);
  uv[2 * i + 1] = float(w);
  flags[i] = (double(z) > 0.1 && u > 0.0 && u < double(c.width) && w > 0.0 && w < double(c.height)) ? 1 : 0;
  if (i == 0) flags[n] = 0;
}

__global__ void cam_compact_kernel(const float* __restrict__ velo, const int32_t* __restrict__ frame_ptr, int num_frames,
                                   int64_t n, const FrameCalib* __restrict__ calib, const float* __restrict__ cam_xyz,
                                   const float* __restrict__ uv, const int32_t* __restrict__ flags,
                                   const int32_t* __restrict__ slot, const uint8_t* __restrict__ images,
                                   const int64_t* __restrict__ image_offset, int attr_channels, int64_t capacity,
                                   float* __restrict__ out_xyz, float* __restrict__ out_attr, int32_t* __restrict__ out_frame_ptr) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i <= num_frames) out_frame_ptr[i] = slot[frame_ptr[i]];       // exclusive scan: kept points before the frame
  if (i >= n || !flags[i]) return;
  const int o = slot[i];
  if (o >= capacity) return;
  out_xyz[3 * o + 0] = cam_xyz[3 * i + 0];
  out_xyz[3 * o + 1] = cam_xyz[3 * i + 1];
  out_xyz[3 * o + 2] = cam_xyz[3 * i + 2];
  out_attr[int64_t(o) * attr_channels] = velo[4 * i + 3];
  if (attr_channels == 4) {
    // rgb_to_cam_points (kitti_dataset.py:990-996): image[int32(v), int32(u), ::-1] / 255
    const int f = frame_of(frame_ptr, num_frames, i);
    const FrameCalib& c = calib[f];
    const int px = int(uv[2 * i + 0]), py = int(uv[2 * i + 1]);
    const uint8_t* pix = images + image_offset[f] + (int64_t(py) * c.width + px) * 3;
    out_attr[int64_t(o) * 4 + 1] = float(pix[2]) / 255.0f;
    out_attr[int64_t(o) * 4 + 2] = float(pix[1]) / 255.0f;
    out_attr[int64_t(o) * 4 + 3] = float(pix[0]) / 255.0f;
  }
}

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" int pg_cam_points_in_image(const float* velo_points, const int32_t* frame_ptr, int32_t num_frames,
                                      int64_t num_points, const float* velo_to_cam_host, const double* cam_to_image_host,
                                      const int32_t* image_size_host, const uint8_t* images,
                                      const int64_t* image_offset_host, float* out_xyz, float* out_attr,
                                      int32_t attr_channels, int64_t capacity, int32_t* out_frame_ptr,
                                      int64_t* out_num_points_host, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(velo_points && frame_ptr && velo_to_cam_host && cam_to_image_host && image_size_host && out_xyz && out_attr &&
                 out_frame_ptr && out_num_points_host,
             "pg_cam_points_in_image: null argument");
  PG_REQUIRE(num_frames >= 1 && num_frames <= 65535 && num_points >= 1 && num_points < (int64_t(1) << 31),
             "pg_cam_points_in_image: bad sizes");
  PG_REQUIRE(attr_channels == 1 || (attr_channels == 4 && images && image_offset_host),
             "pg_cam_points_in_image: attr_channels must be 1 (reflectance) or 4 (reflectance + rgb, needs images)");
  PG_REQUIRE((reinterpret_cast<uintptr_t>(velo_points) & 15) == 0, "pg_cam_points_in_image: velo_points must be 16-byte aligned");
  std::vector<FrameCalib> h(num_frames);
  for (int f = 0; f < num_frames; ++f) {
    // velo_to_cam_host: [F][4][4] float32 (the matrix of kitti_dataset.py:510-511); cam = velo @ transpose(M)[:3,:3] + M[:3,3]
    const float* m = velo_to_cam_host + 16 * f;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) h[f].r[3 * i + j] = m[4 * j + i];
    for (int j = 0; j < 3; ++j) h[f].t[j] = m[4 * j + 3];
    for (int i = 0; i < 12; ++i) h[f].p[i] = cam_to_image_host[12 * f + i];
    h[f].width = image_size_host[2 * f];
    h[f].height = image_size_host[2 * f + 1];
    PG_REQUIRE(h[f].width > 0 && h[f].height > 0, "pg_cam_points_in_image: bad image size of frame %d", f);
  }
  Temp calib, cam, uv, flags, slot, offs;
  PG_CUDA_OK(calib.alloc(sizeof(FrameCalib) * num_frames, s));
  PG_CUDA_OK(cudaMemcpyAsync(calib.ptr, h.data(), sizeof(FrameCalib) * num_frames, cudaMemcpyHostToDevice, s));
  if (attr_channels == 4) {
    PG_CUDA_OK(offs.alloc(sizeof(int64_t) * num_frames, s));
    PG_CUDA_OK(cudaMemcpyAsync(offs.ptr, image_offset_host, sizeof(int64_t) * num_frames, cudaMemcpyHostToDevice, s));
  }
  PG_CUDA_OK(cam.alloc(sizeof(float) * 3 * num_points, s));
  PG_CUDA_OK(uv.alloc(sizeof(float) * 2 * num_points, s));
  PG_CUDA_OK(flags.alloc(sizeof(int32_t) * (num_points + 1), s));
  PG_CUDA_OK(slot.alloc(sizeof(int32_t) * (num_points + 1), s));
  cam_flag_kernel<<<ceil_div(num_points, 256), 256, 0, s>>>(velo_points, frame_ptr, num_frames, num_points,
                                                           calib.as<FrameCalib>(), cam.as<float>(), uv.as<float>(),
                                                           flags.as<int32_t>());
  PG_LAUNCH_CHECK();
  if (int rc = exclusive_sum(flags.as<int32_t>(), slot.as<int32_t>(), num_points + 1, s)) return rc;
  cam_compact_kernel<<<ceil_div(std::max<int64_t>(num_points, num_frames + 1), 256), 256, 0, s>>>(
      velo_points, frame_ptr, num_frames, num_points, calib.as<FrameCalib>(), cam.as<float>(), uv.as<float>(),
      flags.as<int32_t>(), slot.as<int32_t>(), images, offs.as<int64_t>(), attr_channels, capacity, out_xyz, out_attr,
      out_frame_ptr);
  PG_LAUNCH_CHECK();
  int32_t h_n = 0;
  PG_CUDA_OK(cudaMemcpyAsync(&h_n, slot.as<int32_t>() + num_points, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaStreamSynchronize(s));     // also keeps the host calibration array alive until it was copied
  *out_num_points_host = h_n;
  if (h_n > capacity) {
    set_error("point buffer too small: need %d, capacity %lld", h_n, (long long)capacity);
    return PG_ERR_CAPACITY;
  }
  return PG_OK;
}
