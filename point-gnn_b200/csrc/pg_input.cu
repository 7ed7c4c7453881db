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

// velo_points_to_cam (kitti_dataset.py:998-1006) for one point
__device__ __forceinline__ void velo_to_cam_point(const FrameCalib& c, float vx, float vy, float vz, float* x, float* y,
                                                  float* z) {
  *x = __fadd_rn(dot3_rn(vx, vy, vz, c.r[0], c.r[3], c.r[6]), c.t[0]);
  *y = __fadd_rn(dot3_rn(vx, vy, vz, c.r[1], c.r[4], c.r[7]), c.t[1]);
  *z = __fadd_rn(dot3_rn(vx, vy, vz, c.r[2], c.r[5], c.r[8]), c.t[2]);
}

// The crop test of one camera-frame point: z > 0.1 and the projection (cam_points_to_image, kitti_dataset.py:1036-1052,
// float64) strictly inside the image.  uv = the projection as float32, which the colour lookup truncates to a pixel.
__device__ __forceinline__ int project_and_test(const FrameCalib& c, float x, float y, float z, float* uv) {
  const double X = double(x), Y = double(y), Z = double(z);
  const double iu = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(X, c.p[0]), __dmul_rn(Y, c.p[1])), __dmul_rn(Z, c.p[2])), c.p[3]);
  const double iv = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(X, c.p[4]), __dmul_rn(Y, c.p[5])), __dmul_rn(Z, c.p[6])), c.p[7]);
  const double iw = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(X, c.p[8]), __dmul_rn(Y, c.p[9])), __dmul_rn(Z, c.p[10])), c.p[11]);
  const double u = __ddiv_rn(iu, iw), w = __ddiv_rn(iv, iw);
  uv[0] = float(u);
  uv[1] = float(w);
  return (double(z) > 0.1 && u > 0.0 && u < double(c.width) && w > 0.0 && w < double(c.height)) ? 1 : 0;
}

__global__ void cam_flag_kernel(const float* __restrict__ velo, const int32_t* __restrict__ frame_ptr, int num_frames,
                                int64_t n, const FrameCalib* __restrict__ calib, float* __restrict__ cam_xyz,
                                float* __restrict__ uv, int32_t* __restrict__ flags) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const FrameCalib& c = calib[frame_of(frame_ptr, num_frames, i)];
  const float4 v = reinterpret_cast<const float4*>(velo)[i];
  float x, y, z;
  velo_to_cam_point(c, v.x, v.y, v.z, &x, &y, &z);
  cam_xyz[3 * i + 0] = x;
  cam_xyz[3 * i + 1] = y;
  cam_xyz[3 * i + 2] = z;
  flags[i] = project_and_test(c, x, y, z, uv + 2 * i);
  if (i == 0) flags[n] = 0;
}

// cam_flag_kernel for points that are in the camera frame already
__global__ void crop_flag_kernel(const float* __restrict__ cam_xyz, const int32_t* __restrict__ frame_ptr, int num_frames,
                                 int64_t n, const FrameCalib* __restrict__ calib, float* __restrict__ uv,
                                 int32_t* __restrict__ flags) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const FrameCalib& c = calib[frame_of(frame_ptr, num_frames, i)];
  flags[i] = project_and_test(c, cam_xyz[3 * i + 0], cam_xyz[3 * i + 1], cam_xyz[3 * i + 2], uv + 2 * i);
  if (i == 0) flags[n] = 0;
}

// the transform alone: every point, with its reflectance as the one attribute
__global__ void velo_to_cam_kernel(const float* __restrict__ velo, const int32_t* __restrict__ frame_ptr, int num_frames,
                                   int64_t n, const FrameCalib* __restrict__ calib, float* __restrict__ out_xyz,
                                   float* __restrict__ out_attr) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const FrameCalib& c = calib[frame_of(frame_ptr, num_frames, i)];
  const float4 v = reinterpret_cast<const float4*>(velo)[i];
  velo_to_cam_point(c, v.x, v.y, v.z, out_xyz + 3 * i, out_xyz + 3 * i + 1, out_xyz + 3 * i + 2);
  out_attr[i] = v.w;
}

// reflectance of point i = refl[i * refl_stride]: column 3 of the velodyne rows, or an [n, 1] attribute array
__global__ void cam_compact_kernel(const float* __restrict__ refl, int refl_stride, const int32_t* __restrict__ frame_ptr,
                                   int num_frames, int64_t n, const FrameCalib* __restrict__ calib,
                                   const float* __restrict__ cam_xyz, const float* __restrict__ uv,
                                   const int32_t* __restrict__ flags, const int32_t* __restrict__ slot,
                                   const uint8_t* __restrict__ images, const int64_t* __restrict__ image_offset,
                                   int attr_channels, int64_t capacity, float* __restrict__ out_xyz,
                                   float* __restrict__ out_attr, int32_t* __restrict__ out_frame_ptr) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i <= num_frames) out_frame_ptr[i] = slot[frame_ptr[i]];       // exclusive scan: kept points before the frame
  if (i >= n || !flags[i]) return;
  const int o = slot[i];
  if (o >= capacity) return;
  out_xyz[3 * o + 0] = cam_xyz[3 * i + 0];
  out_xyz[3 * o + 1] = cam_xyz[3 * i + 1];
  out_xyz[3 * o + 2] = cam_xyz[3 * i + 2];
  out_attr[int64_t(o) * attr_channels] = refl[i * refl_stride];
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

// The per-frame calibration on the device.  velo_to_cam_host [F][4][4] float32 (the matrix of kitti_dataset.py:510-511;
// cam = velo @ transpose(M)[:3,:3] + M[:3,3]) or null for a call that does not transform; cam_to_image_host [F][3][4]
// float64 with image_size_host [F][2], or both null for a call that does not project.  `h` must stay alive until the
// stream has copied it.
int upload_calib(const char* who, int num_frames, const float* velo_to_cam_host, const double* cam_to_image_host,
                 const int32_t* image_size_host, std::vector<FrameCalib>* h, Temp* calib, cudaStream_t s) {
  h->assign(num_frames, FrameCalib{});
  for (int f = 0; f < num_frames; ++f) {
    FrameCalib& c = (*h)[f];
    if (velo_to_cam_host != nullptr) {
      const float* m = velo_to_cam_host + 16 * f;
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) c.r[3 * i + j] = m[4 * j + i];
      for (int j = 0; j < 3; ++j) c.t[j] = m[4 * j + 3];
    }
    if (cam_to_image_host != nullptr) {
      for (int i = 0; i < 12; ++i) c.p[i] = cam_to_image_host[12 * f + i];
      c.width = image_size_host[2 * f];
      c.height = image_size_host[2 * f + 1];
      PG_REQUIRE(c.width > 0 && c.height > 0, "%s: bad image size of frame %d", who, f);
    }
  }
  PG_CUDA_OK(calib->alloc(sizeof(FrameCalib) * num_frames, s));
  PG_CUDA_OK(cudaMemcpyAsync(calib->ptr, h->data(), sizeof(FrameCalib) * num_frames, cudaMemcpyHostToDevice, s));
  return PG_OK;
}

// What both crop entry points share once flags [n + 1] and uv [n, 2] are made: the scan of the flags, the stable
// compaction with the attributes, and the one host round trip.
int compact_flagged(const float* refl, int refl_stride, const int32_t* frame_ptr, int num_frames, int64_t n,
                    const FrameCalib* calib, const float* cam_xyz, const float* uv, const int32_t* flags,
                    const uint8_t* images, const int64_t* image_offset_host, int attr_channels, int64_t capacity,
                    float* out_xyz, float* out_attr, int32_t* out_frame_ptr, int64_t* out_num_points_host,
                    cudaStream_t s) {
  Temp slot, offs;
  if (attr_channels == 4) {
    PG_CUDA_OK(offs.alloc(sizeof(int64_t) * num_frames, s));
    PG_CUDA_OK(cudaMemcpyAsync(offs.ptr, image_offset_host, sizeof(int64_t) * num_frames, cudaMemcpyHostToDevice, s));
  }
  PG_CUDA_OK(slot.alloc(sizeof(int32_t) * (n + 1), s));
  if (int rc = exclusive_sum(flags, slot.as<int32_t>(), n + 1, s)) return rc;
  cam_compact_kernel<<<ceil_div(std::max<int64_t>(n, num_frames + 1), 256), 256, 0, s>>>(
      refl, refl_stride, frame_ptr, num_frames, n, calib, cam_xyz, uv, flags, slot.as<int32_t>(), images,
      offs.as<int64_t>(), attr_channels, capacity, out_xyz, out_attr, out_frame_ptr);
  PG_LAUNCH_CHECK();
  int32_t h_n = 0;
  PG_CUDA_OK(cudaMemcpyAsync(&h_n, slot.as<int32_t>() + n, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  PG_CUDA_OK(cudaStreamSynchronize(s));     // also keeps the caller's host calibration array alive until it was copied
  *out_num_points_host = h_n;
  if (h_n > capacity) {
    set_error("point buffer too small: need %d, capacity %lld", h_n, (long long)capacity);
    return PG_ERR_CAPACITY;
  }
  return PG_OK;
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
  std::vector<FrameCalib> h;
  Temp calib, cam, uv, flags;
  if (int rc = upload_calib("pg_cam_points_in_image", num_frames, velo_to_cam_host, cam_to_image_host, image_size_host, &h,
                            &calib, s))
    return rc;
  PG_CUDA_OK(cam.alloc(sizeof(float) * 3 * num_points, s));
  PG_CUDA_OK(uv.alloc(sizeof(float) * 2 * num_points, s));
  PG_CUDA_OK(flags.alloc(sizeof(int32_t) * (num_points + 1), s));
  cam_flag_kernel<<<ceil_div(num_points, 256), 256, 0, s>>>(velo_points, frame_ptr, num_frames, num_points,
                                                           calib.as<FrameCalib>(), cam.as<float>(), uv.as<float>(),
                                                           flags.as<int32_t>());
  PG_LAUNCH_CHECK();
  return compact_flagged(velo_points + 3, 4, frame_ptr, num_frames, num_points, calib.as<FrameCalib>(), cam.as<float>(),
                         uv.as<float>(), flags.as<int32_t>(), images, image_offset_host, attr_channels, capacity, out_xyz,
                         out_attr, out_frame_ptr, out_num_points_host, s);
}

extern "C" int pg_velo_to_cam(const float* velo_points, const int32_t* frame_ptr, int32_t num_frames, int64_t num_points,
                              const float* velo_to_cam_host, float* out_xyz, float* out_attr, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(velo_points && frame_ptr && velo_to_cam_host && out_xyz && out_attr, "pg_velo_to_cam: null argument");
  PG_REQUIRE(num_frames >= 1 && num_frames <= 65535 && num_points >= 1 && num_points < (int64_t(1) << 31),
             "pg_velo_to_cam: bad sizes");
  PG_REQUIRE((reinterpret_cast<uintptr_t>(velo_points) & 15) == 0, "pg_velo_to_cam: velo_points must be 16-byte aligned");
  std::vector<FrameCalib> h;
  Temp calib;
  if (int rc = upload_calib("pg_velo_to_cam", num_frames, velo_to_cam_host, nullptr, nullptr, &h, &calib, s)) return rc;
  velo_to_cam_kernel<<<ceil_div(num_points, 256), 256, 0, s>>>(velo_points, frame_ptr, num_frames, num_points,
                                                              calib.as<FrameCalib>(), out_xyz, out_attr);
  PG_LAUNCH_CHECK();
  PG_CUDA_OK(cudaStreamSynchronize(s));     // the host calibration array must outlive its copy
  return PG_OK;
}

extern "C" int pg_cam_points_crop(const float* cam_xyz, const float* reflectance, const int32_t* frame_ptr,
                                  int32_t num_frames, int64_t num_points, const double* cam_to_image_host,
                                  const int32_t* image_size_host, const uint8_t* images, const int64_t* image_offset_host,
                                  float* out_xyz, float* out_attr, int32_t attr_channels, int64_t capacity,
                                  int32_t* out_frame_ptr, int64_t* out_num_points_host, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(cam_xyz && reflectance && frame_ptr && cam_to_image_host && image_size_host && out_xyz && out_attr &&
                 out_frame_ptr && out_num_points_host,
             "pg_cam_points_crop: null argument");
  PG_REQUIRE(num_frames >= 1 && num_frames <= 65535 && num_points >= 1 && num_points < (int64_t(1) << 31),
             "pg_cam_points_crop: bad sizes");
  PG_REQUIRE(attr_channels == 1 || (attr_channels == 4 && images && image_offset_host),
             "pg_cam_points_crop: attr_channels must be 1 (reflectance) or 4 (reflectance + rgb, needs images)");
  std::vector<FrameCalib> h;
  Temp calib, uv, flags;
  if (int rc = upload_calib("pg_cam_points_crop", num_frames, nullptr, cam_to_image_host, image_size_host, &h, &calib, s))
    return rc;
  PG_CUDA_OK(uv.alloc(sizeof(float) * 2 * num_points, s));
  PG_CUDA_OK(flags.alloc(sizeof(int32_t) * (num_points + 1), s));
  crop_flag_kernel<<<ceil_div(num_points, 256), 256, 0, s>>>(cam_xyz, frame_ptr, num_frames, num_points,
                                                            calib.as<FrameCalib>(), uv.as<float>(), flags.as<int32_t>());
  PG_LAUNCH_CHECK();
  return compact_flagged(reflectance, 1, frame_ptr, num_frames, num_points, calib.as<FrameCalib>(), cam_xyz, uv.as<float>(),
                         flags.as<int32_t>(), images, image_offset_host, attr_channels, capacity, out_xyz, out_attr,
                         out_frame_ptr, out_num_points_host, s);
}
