// Hopper tensor-core kernels (wgmma): the fast path (precision = 1, "BF16x3").
//
// wg_gemm_kernel - one persistent, warp-specialised kernel for every tensor-core layer of the network:
//   out = epilogue(A @ W + b), W streamed by a producer warpgroup, A produced on the fly in shared memory by the
//   two consumer warpgroups that also run the wgmmas.
//
//   producers  PROD_ROWS  A = rows of an fp32 matrix (dense layers, the later layers of the pooling MLP)
//              PROD_GNN   one GNN iteration's edge MLP (/root/reference/models/gnn.py:338-365) after hoisting:
//                         e0 @ W1 + b1 = (F @ W1[:C] + b1)[src] + (x_src - x_dst') @ W1[C:], so the first edge
//                         layer is a per-VERTEX table P (a PROD_ROWS GEMM) plus a 3-term per-edge correction;
//                         A row e = relu(P[src] + (x_src - x_dst') @ W1[C:])
//              PROD_POOL  PointSetPooling's first layer (gnn.py:264-270) in fp32:
//                         A row e = relu([feature(src), x_src - x_kp(dst)] @ W0 + b0)
//   epilogues  EPI_STORE  act(acc + b) (+ residual) to a row-major matrix
//              EPI_SEGMAX max over the edges of each destination (edges are grouped by destination):
//                         relu / bias commute with max, so raw accumulators are reduced across the warp's
//                         16 rows with shuffles and each partial max is flushed with one atomicMax
//   precision  every fp32 operand is split x = hi + lo (two BF16), and hi*hi' + lo*hi' + hi*lo' is
//              accumulated in fp32 registers: ~2^-16 relative per product (fp32-class accuracy)
//   mapping    CTA = 3 warpgroups.  Warpgroup 0 is the W producer (setmaxnreg down to 24 registers): one thread
//              streams W (hi and lo images, pre-packed in the no-swizzle K-major core-matrix layout, one
//              contiguous block per 16-k chunk) from L2 through a ring of shared-memory stages with
//              cp.async.bulk, each stage tracked by a "full" (bytes landed) and an "empty" (both consumers done)
//              mbarrier.  Warpgroups 1 and 2 are the consumers (setmaxnreg up to 240): 128 rows per tile (64 per
//              warpgroup), the whole padded N (<= 304: two m64nNk16 instructions) in registers.  Each produces
//              A into a double buffer, issuing the global loads of chunk k + 2 before the wgmmas of chunk k + 1,
//              and splits and stores chunk k + 1 while chunk k's wgmmas run.  A consumer only arrives on "empty";
//              it never waits on it or issues a copy: such divergent code in the k-loop makes ptxas serialise
//              the wgmmas (C7518), and the two consumers would wait for each other on every chunk.
//
// Operand layout (no swizzle, K-major): 8-row x 16-byte core matrices, 128 contiguous bytes each;
// for a 16-k chunk, core(row group g, k half kc) at g * 256 + kc * 128 (LBO = 128, SBO = 256).
#include <atomic>
#include <cstdlib>
#include <memory>
#include <utility>
#include <vector>

#include "pg_common.cuh"
#include "pg_wgmma.cuh"

namespace pg {
static std::atomic<long long> g_tc_launches[2];   // [0] segment-max (edge) launches, [1] store (dense) launches
}

// tensor-core kernel launches so far: which = 0 segment-max (edge layer) launches, 1 dense-layer launches
extern "C" int64_t pg_tc_launch_count(int32_t which) {
  return (which == 0 || which == 1) ? pg::g_tc_launches[which].load(std::memory_order_relaxed) : -1;
}

namespace pg {
namespace {
using namespace wg;

constexpr int kWgThreads = 384;     // warpgroup 0 streams W, warpgroups 1 and 2 compute
constexpr int kProducerRegs = 24;   // 2 x 128 x 240 + 128 x 24 = 384 x 168, the launch bound's budget
constexpr int kConsumerRegs = 240;  // 232 spills 8 bytes in the 152 x 2 segment-max instances
constexpr int kTileRows = 128;      // rows per tile (64 per consumer warpgroup)
// 4 W stages beat 8 on H100: the ring is deep enough for the copies, and the smaller shared-memory carve-out leaves
// more L1 for the gathered rows (GNN edge layer at the benchmark shape: 7.7 vs 8.0 ms, H100 SXM at a 400 W limit)
constexpr int kMaxRing = 4;
constexpr int kMaxNT = 304;         // widest padded N one launch covers
constexpr uint32_t kABytes = 4096;  // one warpgroup's A chunk: hi (2048) + lo (2048), 64 rows x 16 k

// W stages in shared memory for an NT-wide layer: the deepest power of two up to kMaxRing (so the stage of a chunk
// is a mask) whose ring, A buffers and barriers fit the 227 KB a CTA may use
constexpr size_t wg_smem_bytes(int nt, int ring) {
  return size_t(ring) * nt * 64 + 4 * kABytes + 2 * ring * sizeof(uint64_t);
}
constexpr int ring_stages(int nt) {
  int r = kMaxRing;
  while (r > 1 && wg_smem_bytes(nt, r) > 227 * 1024) r /= 2;
  return r;
}

enum { PROD_ROWS = 0, PROD_GNN = 1, PROD_POOL = 2 };
enum { EPI_STORE = 0, EPI_SEGMAX = 1 };

struct WgParams {
  // A producer
  const float* x;           // ROWS: [num_rows, ldx];  GNN: P [num_src, ldx] (ldx = kp, zero padded)
  int ldx;
  int k_real;               // ROWS: true K (multiple of 4)
  const float* feat;        // POOL: [num_src] point features (one channel)
  const float* w1x;         // GNN: [3, kp] = W1[C:];  POOL: [4, kp] = W0, then [kp] = b0 (zero padded)
  const float* xyz_src;     // [num_src, 3]
  const float* xyz_dst;     // [*, 3] (already offset)
  const int32_t* dst_index; // optional indirection dst -> row of xyz_dst
  const int32_t* src;
  const int32_t* dst;
  int64_t num_rows;         // edges (GNN / POOL / SEGMAX) or matrix rows
  int64_t num_src, num_dst;
  // GEMM shape
  int kp, nchunks;          // padded K, kp / 16
  const uint8_t* bimg;      // [nchunks][hi | lo][NT rows x 16 k] core-matrix image of W
  const float* bias;        // [NT] zero padded
  int n;                    // real output columns
  // epilogue
  float* out;               // STORE: [num_rows, ldo];  SEGMAX: [num_dst, ldo] pre-filled with -FLT_MAX
  int ldo;
  int act;                  // STORE: 0 linear, 1 relu
  const float* residual;    // STORE: optional [num_rows, ldr]
  int ldr;
  int* err;
  int64_t num_tiles;
};

__device__ __forceinline__ float4 ldg_nc(const float* ptr) {
  float4 v;
  asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(ptr));
  return v;
}

__device__ __forceinline__ void seg_flush(const WgParams& p, int d, int col, float m) {
  // + 0.0f turns a -0.0f into +0.0f, which must win against the -FLT_MAX fill as an integer
  atomicMax(reinterpret_cast<int*>(p.out + int64_t(d) * p.ldo + col), __float_as_int(fmaxf(m + __ldg(p.bias + col), 0.0f) + 0.0f));
}

// w[0 .. 8) = ptr[0 .. 8); ptr is 32-byte aligned
__device__ __forceinline__ void ldg8(const float* ptr, float (&w)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(ptr)), b = __ldg(reinterpret_cast<const float4*>(ptr) + 1);
  w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
  w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
}

template <int kProd, int kEpi, int NI, int NS>
__global__ void __launch_bounds__(kWgThreads, 1) wg_gemm_kernel(WgParams p) {
  constexpr int NT = NI * NS;
  constexpr int kRing = ring_stages(NT);
  constexpr uint32_t kChunkBytes = uint32_t(NT) * 64u;   // hi + lo, 16 k
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* bring = smem;
  uint8_t* abuf = smem + kRing * kChunkBytes;            // [consumer warpgroup][buffer][hi | lo]
  uint64_t* full = reinterpret_cast<uint64_t*>(abuf + 4 * kABytes);
  uint64_t* empty = full + kRing;
  const int tid = threadIdx.x;
  const int role = __shfl_sync(0xffffffffu, tid >> 7, 0);   // warpgroup, warp-uniform by construction
  if (tid == 0) {
    for (int s = 0; s < kRing; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);     // lane 0 of each of the 8 consumer warps
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int64_t my_tiles = (p.num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;
  const int nk = p.nchunks;
  if (role == 0) {
    // W producer: one thread streams the CTA's chunks in the order the consumers use them, refilling a stage as
    // soon as both consumer warpgroups have released it
    setmaxnreg_dec<kProducerRegs>();
    if (tid != 0) return;
    const int64_t total = my_tiles * nk;
    for (int64_t g = 0; g < total; ++g) {
      const uint32_t stage = uint32_t(g % kRing);
      if (g >= kRing) mbar_wait(&empty[stage], uint32_t((g / kRing - 1) & 1));
      mbar_arrive_expect_tx(&full[stage], kChunkBytes);
      bulk_g2s(bring + stage * kChunkBytes, p.bimg + size_t(g % nk) * kChunkBytes, kChunkBytes, &full[stage]);
    }
    return;
  }
  setmaxnreg_inc<kConsumerRegs>();
  const int wgi = role - 1, t = tid & 127, warp = t >> 5, lane = tid & 31;
  // chunk g's W stage is free again
  auto release = [&](int64_t g) {
    if (lane == 0) mbar_arrive(&empty[g % kRing]);
  };

  // A geometry: thread t writes 8 consecutive k (half kh) of row pr of its warpgroup's 64
  const int pr = t >> 1, kh = t & 1;
  const uint32_t a_off = uint32_t(pr >> 3) * 256u + uint32_t(kh) * 128u + uint32_t(pr & 7) * 16u;
  uint8_t* my_a = abuf + wgi * 2 * kABytes;
  float acc[NS][NI / 2];
  int64_t g = 0;
  for (int64_t j = 0; j < my_tiles; ++j) {
    const int64_t tile = blockIdx.x + j * gridDim.x;
    const int64_t row = tile * kTileRows + wgi * 64 + pr;
    const bool valid = row < p.num_rows;
    // ---- row context -----------------------------------------------------------------------------
    const float* rp = p.x;
    float rx = 0.f, ry = 0.f, rz = 0.f, f0 = 0.f;
    if (kProd == PROD_ROWS) {
      if (valid) rp = p.x + row * int64_t(p.ldx);
    } else if (valid) {
      int si = __ldg(p.src + row), di = __ldg(p.dst + row);
      if (si < 0 || si >= p.num_src || di < 0 || di >= p.num_dst) {
        *p.err = 1;
        si = 0;
        di = 0;
      }
      const int64_t drow = p.dst_index ? int64_t(__ldg(p.dst_index + di)) : int64_t(di);
      rx = __ldg(p.xyz_src + int64_t(si) * 3 + 0) - __ldg(p.xyz_dst + drow * 3 + 0);
      ry = __ldg(p.xyz_src + int64_t(si) * 3 + 1) - __ldg(p.xyz_dst + drow * 3 + 1);
      rz = __ldg(p.xyz_src + int64_t(si) * 3 + 2) - __ldg(p.xyz_dst + drow * 3 + 2);
      if (kProd == PROD_GNN) rp = p.x + int64_t(si) * p.ldx;
      else f0 = __ldg(p.feat + si);
    }
    auto load = [&](int kc, float4 (&q)[2]) {
      if (kProd == PROD_POOL) return;
      const int k0 = kc * 16 + kh * 8;
#pragma unroll
      for (int i = 0; i < 2; ++i)
        q[i] = (kProd == PROD_GNN || k0 + 4 * i + 4 <= p.k_real) ? ldg_nc(rp + k0 + 4 * i) : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    auto put = [&](int buf, const float4 (&q)[2], int kc) {
      const int k0 = kc * 16 + kh * 8;
      float v[8] = {q[0].x, q[0].y, q[0].z, q[0].w, q[1].x, q[1].y, q[1].z, q[1].w};
      // w1x rows are kp (a multiple of 16) floats long, so this thread's 8 k of every row are 32-byte aligned
      if (kProd == PROD_GNN) {
        float wx[8], wy[8], wz[8];
        ldg8(p.w1x + k0, wx);
        ldg8(p.w1x + p.kp + k0, wy);
        ldg8(p.w1x + 2 * p.kp + k0, wz);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = fmaxf(fmaf(rz, wz[i], fmaf(ry, wy[i], fmaf(rx, wx[i], v[i]))), 0.0f);
      } else if (kProd == PROD_POOL) {
        float wf[8], wx[8], wy[8], wz[8], b0[8];
        ldg8(p.w1x + k0, wf);
        ldg8(p.w1x + p.kp + k0, wx);
        ldg8(p.w1x + 2 * p.kp + k0, wy);
        ldg8(p.w1x + 3 * p.kp + k0, wz);
        ldg8(p.w1x + 4 * p.kp + k0, b0);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float a = b0[i];
          a = fmaf(f0, wf[i], a);
          a = fmaf(rx, wx[i], a);
          a = fmaf(ry, wy[i], a);
          a = fmaf(rz, wz[i], a);
          v[i] = fmaxf(a, 0.0f);
        }
      }
      uint4 hi, lo;
      split_bf16x2(v[0], v[1], &hi.x, &lo.x);
      split_bf16x2(v[2], v[3], &hi.y, &lo.y);
      split_bf16x2(v[4], v[5], &hi.z, &lo.z);
      split_bf16x2(v[6], v[7], &hi.w, &lo.w);
      uint8_t* dstp = my_a + buf * kABytes + a_off;
      *reinterpret_cast<uint4*>(dstp) = hi;
      *reinterpret_cast<uint4*>(dstp + kABytes / 2) = lo;
    };
    float4 q[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
    load(0, q);
    put(0, q, 0);
    if (nk > 1) load(1, q);
    // ---- main loop over 16-k chunks ------------------------------------------------------------------
    for (int kc = 0; kc < nk; ++kc, ++g) {
      fence_proxy_async_smem();
      warpgroup_sync(1 + wgi);
      mbar_wait(&full[g % kRing], uint32_t((g / kRing) & 1));
      wgmma_fence();
      const uint32_t a_base = smem_u32(my_a + (kc & 1) * kABytes);
      const uint32_t b_base = smem_u32(bring + uint32_t(g % kRing) * kChunkBytes);
      const uint64_t a_hi = make_smem_desc(a_base, 128, 256), a_lo = make_smem_desc(a_base + kABytes / 2, 128, 256);
#pragma unroll
      for (int i = 0; i < NS; ++i) {
        const uint64_t b_hi = make_smem_desc(b_base + uint32_t(i * NI) * 32u, 128, 256);
        const uint64_t b_lo = make_smem_desc(b_base + uint32_t(NT) * 32u + uint32_t(i * NI) * 32u, 128, 256);
        wgmma_bf16<NI>(acc[i], a_hi, b_hi, kc > 0 ? 1 : 0);
        wgmma_bf16<NI>(acc[i], a_lo, b_hi, 1);
        wgmma_bf16<NI>(acc[i], a_hi, b_lo, 1);
      }
      wgmma_commit();
      // every iteration leaves exactly chunk kc in flight: a wait on a path of its own (the last chunk's) would make
      // ptxas drain the wgmmas at the end of every iteration
      wgmma_wait<1>();                    // chunk kc - 1 complete: its A buffer and W stage are free
      if (kc > 0) release(g - 1);
      if (kc + 1 < nk) {
        put((kc + 1) & 1, q, kc + 1);
        if (kc + 2 < nk) load(kc + 2, q);
      }
    }
    wgmma_wait<0>();
    release(g - 1);
    // ---- epilogue ----------------------------------------------------------------------------------
    const int64_t r0 = tile * kTileRows + wgi * 64 + warp * 16 + (lane >> 2);
    const int cq = (lane & 3) * 2;
    if (kEpi == EPI_STORE) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t r = r0 + 8 * h;
        if (r >= p.num_rows) continue;
#pragma unroll
        for (int i = 0; i < NS; ++i)
#pragma unroll
          for (int jj = 0; jj < NI / 8; ++jj)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int col = i * NI + jj * 8 + cq + c;
              if (col < p.n) {
                float v = acc[i][4 * jj + 2 * h + c] + __ldg(p.bias + col);
                if (p.act) v = fmaxf(v, 0.0f);
                if (p.residual) v += __ldg(p.residual + r * int64_t(p.ldr) + col);
                p.out[r * int64_t(p.ldo) + col] = v;
              }
            }
      }
    } else {
      int d[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t r = r0 + 8 * h;
        d[h] = -1;
        if (r < p.num_rows) {
          d[h] = __ldg(p.dst + r);
          if (d[h] < 0 || d[h] >= p.num_dst) {
            *p.err = 1;
            d[h] = -1;
          }
        }
      }
      const int dw = __shfl_sync(0xffffffffu, d[0], 0);
      if (__all_sync(0xffffffffu, d[0] == dw && d[1] == dw) && dw >= 0) {
        // the warp's 16 rows are one destination: combine the halves, then the 8 lanes sharing columns
#pragma unroll
        for (int i = 0; i < NS; ++i)
#pragma unroll
          for (int jj = 0; jj < NI / 8; ++jj)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              float m = fmaxf(acc[i][4 * jj + c], acc[i][4 * jj + 2 + c]);
              m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
              m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
              m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16));
              const int col = i * NI + jj * 8 + cq + c;
              if (lane < 4 && col < p.n) seg_flush(p, dw, col, m);
            }
      } else {
        // segmented max down each 8-row half (rows of one destination are contiguous); the first row of
        // every run flushes the run's max
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int dd = d[h];
          const int up = __shfl_up_sync(0xffffffffu, dd, 4);
          const bool head = dd >= 0 && (lane < 4 || up != dd);
          int dn[3];
#pragma unroll
          for (int s = 0; s < 3; ++s) {
            dn[s] = __shfl_down_sync(0xffffffffu, dd, 4 << s);
            if (lane + (4 << s) >= 32) dn[s] = -2;
          }
#pragma unroll
          for (int i = 0; i < NS; ++i)
#pragma unroll
            for (int jj = 0; jj < NI / 8; ++jj)
#pragma unroll
              for (int c = 0; c < 2; ++c) {
                float m = acc[i][4 * jj + 2 * h + c];
#pragma unroll
                for (int s = 0; s < 3; ++s) {
                  const float o = __shfl_down_sync(0xffffffffu, m, 4 << s);
                  if (dn[s] == dd) m = fmaxf(m, o);
                }
                const int col = i * NI + jj * 8 + cq + c;
                if (head && col < p.n) seg_flush(p, dd, col, m);
              }
        }
      }
    }
  }
}

// ---- W [K, N] -> streamed B image ---------------------------------------------------------------
// B operand rows are OUTPUT features (N), K-major, one block per 16-k chunk: [hi | lo], each NT / 8 row
// groups of two core matrices: element (k, col) at chunk (k / 16), (col / 8) * 256 + ((k % 16) / 8) * 128 +
// (col % 8) * 16 + (k % 8) * 2.  Columns >= n_src and rows >= k are zero.
__global__ void pack_b_kernel(const float* __restrict__ w, int k, int n_src, int ld, int kp, int nt,
                              uint8_t* __restrict__ img) {
  const int total = kp * nt;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int kk = i / nt, col = i - kk * nt;
    const float v = (col < n_src && kk < k) ? w[int64_t(kk) * ld + col] : 0.0f;
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
    const size_t off = size_t(kk / 16) * (size_t(nt) * 64) + size_t(col / 8) * 256 + size_t((kk % 16) / 8) * 128 +
                       size_t(col % 8) * 16 + size_t(kk % 8) * 2;
    *reinterpret_cast<__nv_bfloat16*>(img + off) = hi;
    *reinterpret_cast<__nv_bfloat16*>(img + off + size_t(nt) * 32) = lo;
  }
}

__global__ void pad_rows_kernel(const float* __restrict__ in, int rows, int cols, int ld_out, float* __restrict__ out) {
  const int total = rows * ld_out;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int r = i / ld_out, c = i - r * ld_out;
    out[i] = c < cols ? in[int64_t(r) * cols + c] : 0.0f;
  }
}

struct WgShape {
  int kp, np, ni, ns, nt;
  size_t smem;
  bool ok;
};

// N is padded to one of the instruction shapes the kernel is built for (zero weight columns)
WgShape wg_shape(int k, int n) {
  WgShape t{};
  t.kp = (k + 15) / 16 * 16;
  t.np = (n + 15) / 16 * 16;
  if (t.np <= 64) { t.ni = 64; t.ns = 1; }
  else if (t.np <= 128) { t.ni = 128; t.ns = 1; }
  else if (t.np <= 192) { t.ni = 96; t.ns = 2; }
  else if (t.np <= 256) { t.ni = 128; t.ns = 2; }
  else if (t.np <= kMaxNT) { t.ni = 152; t.ns = 2; }
  t.nt = t.ni * t.ns;
  t.smem = wg_smem_bytes(t.nt, ring_stages(t.nt));
  t.ok = t.nt > 0 && k >= 1 && n >= 1;
  return t;
}

// one weight matrix in the streamed image layout + its padded bias
struct PreparedGemm {
  WgShape t{};
  int n = 0;
  Temp img, bias_pad;
};

int prepare_gemm(PreparedGemm& g, const float* w, int ld, const float* bias, int k, int n, cudaStream_t s) {
  g.t = wg_shape(k, n);
  g.n = n;
  PG_REQUIRE(g.t.ok, "no tensor-core shape for a %d x %d layer", k, n);
  PG_CUDA_OK(g.bias_pad.alloc(sizeof(float) * g.t.nt, s));
  pad_rows_kernel<<<2, 256, 0, s>>>(bias, 1, n, g.t.nt, g.bias_pad.as<float>());
  PG_LAUNCH_CHECK();
  PG_CUDA_OK(g.img.alloc(size_t(g.t.kp) * g.t.nt * 4, s));
  pack_b_kernel<<<std::min(num_sms(), 64), 256, 0, s>>>(w, k, n, ld, g.t.kp, g.t.nt, g.img.as<uint8_t>());
  PG_LAUNCH_CHECK();
  return PG_OK;
}

template <int kProd, int kEpi, int NI, int NS>
int launch_wg_cfg(const WgParams& p, size_t smem, cudaStream_t s) {
  static bool attr_done = false;
  if (!attr_done) {
    PG_CUDA_OK(cudaFuncSetAttribute(wg_gemm_kernel<kProd, kEpi, NI, NS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    int(smem < 48 * 1024 ? 48 * 1024 : 227 * 1024)));
    attr_done = true;
  }
  const int grid = int(std::min<int64_t>(p.num_tiles, num_sms()));
  wg_gemm_kernel<kProd, kEpi, NI, NS><<<grid, kWgThreads, smem, s>>>(p);
  PG_LAUNCH_CHECK();
  g_tc_launches[kEpi == EPI_SEGMAX ? 0 : 1].fetch_add(1, std::memory_order_relaxed);
  return PG_OK;
}

template <int kProd, int kEpi>
int launch_wg(WgParams p, const PreparedGemm& g, cudaStream_t s) {
  if (p.num_rows == 0) return PG_OK;
  p.kp = g.t.kp;
  p.nchunks = g.t.kp / 16;
  p.bimg = g.img.as<uint8_t>();
  p.bias = g.bias_pad.as<float>();
  p.n = g.n;
  p.num_tiles = ceil_div(p.num_rows, kTileRows);
  PG_REQUIRE(g.t.smem <= 227 * 1024, "tensor-core kernel needs %zu B of shared memory", g.t.smem);
  switch (g.t.ni * 4 + g.t.ns) {
    case 64 * 4 + 1: return launch_wg_cfg<kProd, kEpi, 64, 1>(p, g.t.smem, s);
    case 128 * 4 + 1: return launch_wg_cfg<kProd, kEpi, 128, 1>(p, g.t.smem, s);
    case 96 * 4 + 2: return launch_wg_cfg<kProd, kEpi, 96, 2>(p, g.t.smem, s);
    case 128 * 4 + 2: return launch_wg_cfg<kProd, kEpi, 128, 2>(p, g.t.smem, s);
    case 152 * 4 + 2: return launch_wg_cfg<kProd, kEpi, 152, 2>(p, g.t.smem, s);
    default: break;
  }
  PG_REQUIRE(false, "tensor-core kernel: no instance for N = %d", g.t.nt);
  return PG_OK;
}

// column blocks of at most kMaxNT (multiples of 16) covering n
std::vector<int> column_blocks(int n) {
  std::vector<int> c0;
  const int nb = int(ceil_div(n, kMaxNT));
  const int w = (int(ceil_div(n, nb)) + 15) / 16 * 16;
  for (int c = 0; c < n; c += w) c0.push_back(c);
  return c0;
}

// =================================================================================================
// Prepared layers.  Everything that depends only on the WEIGHTS is done once, when a layer is prepared:
// the BF16 hi / lo operand images, padded biases, the hoisted first-layer matrices.  A forward pass then
// launches compute kernels only.  pg_layer_* keeps the prepared state in a handle.  The per-call entry points
// (pg_fully_connected, pg_edge_mlp_max) run a transient prepared layer: they prepare it on the stack (its
// buffers are stream-ordered temporaries) and apply it once, so both forms share one dispatch path.  Whether an
// edge call reads its range-error word back (PG_FLAG_TRUSTED_INDICES) is an argument of apply_edge.
// =================================================================================================

// W [k, n] with row stride ld as tensor-core GEMMs of at most kMaxNT output features, block b writing the columns
// from col0[b]; only the first n_src columns of W are read, the pad columns past them get zero weights and bias
int prepare_column_blocks(std::vector<PreparedGemm>& blocks, std::vector<int>& col0, const float* w, int ld,
                          const float* bias, int k, int n_src, int n, cudaStream_t s) {
  PG_REQUIRE(n >= 1, "no tensor-core shape for a %d x %d layer", k, n);
  col0 = column_blocks(n);
  blocks = std::vector<PreparedGemm>(col0.size());
  for (size_t b = 0; b < col0.size(); ++b) {
    const int wn = (b + 1 < col0.size() ? col0[b + 1] : n) - col0[b];
    const int src_cols = std::max(0, std::min(wn, n_src - col0[b]));
    PG_REQUIRE(src_cols > 0, "dense layer: column block beyond the weight matrix");
    if (int rc = prepare_gemm(blocks[b], w + col0[b], ld, bias + col0[b], k, src_cols, s)) return rc;
    blocks[b].n = wn;
  }
  return PG_OK;
}

// narrow / shallow layers (N < 8, K < 64: the 64->3, 64->4, 64->7 heads) stay on the fp32 FFMA kernel
bool fc_uses_tc(int k, int n) { return (k & 3) == 0 && n >= 8 && (k + 15) / 16 * 16 >= 64; }

// ---- one fully-connected layer -----------------------------------------------------------------
struct PreparedFc {
  int k = 0, n = 0;            // logical GEMM shape [k, n]
  int n_src = 0, ld_src = 0;   // the caller's matrix holds n_src <= n columns (the rest are zero), row stride ld_src
  const float* w = nullptr;    // caller's fp32 tensors (FFMA path; must outlive the handle)
  const float* bias = nullptr;
  bool tc = false;
  // tensor-core path: column blocks of at most kMaxNT output features, each writing its slice of the row
  std::vector<PreparedGemm> blocks;
  std::vector<int> col0;
};

int prepare_fc(PreparedFc& f, const float* w, int ld_src, const float* bias, int k, int n_src, int n, bool want_tc,
               cudaStream_t s) {
  f.k = k;
  f.n = n;
  f.n_src = n_src;
  f.ld_src = ld_src;
  f.w = w;
  f.bias = bias;
  f.blocks.clear();
  f.col0.clear();
  f.tc = want_tc && fc_uses_tc(k, n);
  if (!f.tc) return PG_OK;
  return prepare_column_blocks(f.blocks, f.col0, w, ld_src, bias, k, n_src, n, s);
}

// out [m, ldo]: columns [0, n) = act(x @ W + b) (+ residual [m, n]); ldo >= n
int apply_fc(const PreparedFc& f, const float* x, int64_t m, int act, const float* residual, float* out, int ldo,
             cudaStream_t s) {
  if (m == 0) return PG_OK;
  if (!f.tc) {
    PG_REQUIRE(f.ld_src == f.n_src, "FFMA dense layer needs a contiguous weight matrix");
    PG_REQUIRE(f.n == f.n_src || ldo == f.n, "FFMA dense layer: padded width %d needs ldo == n", f.n);
    return fc_fp32_launch(x, m, f.k, f.w, f.bias, f.n_src, act, residual, out, ldo, s);
  }
  for (size_t b = 0; b < f.blocks.size(); ++b) {
    WgParams p{};
    p.x = x;
    p.ldx = f.k;
    p.k_real = f.k;
    p.num_rows = m;
    p.out = out + f.col0[b];
    p.ldo = ldo;
    p.act = act;
    p.residual = residual ? residual + f.col0[b] : nullptr;
    p.ldr = f.n;
    if (int rc = launch_wg<PROD_ROWS, EPI_STORE>(p, f.blocks[b], s)) return rc;
  }
  return PG_OK;
}

// ---- fused edge layers ------------------------------------------------------------------------
enum { EDGE_FP32 = 0, EDGE_GNN = 1, EDGE_POOL = 2 };

struct PreparedEdge {
  int mode = 0, c_in = 0, num_layers = 0, path = EDGE_FP32;
  std::vector<int32_t> dims;
  std::vector<const float*> w, b;     // caller's tensors (must outlive the handle)
  // GNN: hoisted first layer P = F @ W1[:C] + b1 (zero padded to kp columns) and W1[C:]
  PreparedFc p_fc;
  int kp = 0;
  // GNN: W1[C:] as [3, kp];  POOL: W0 [4, kp] + b0 [kp]
  Temp w1x;
  // the per-edge layers: GNN - W2 in column blocks;  POOL - layers 1 .. L-1, the last one in column blocks
  std::vector<PreparedGemm> mid;      // POOL layers 1 .. L-2 (stored per edge)
  std::vector<PreparedGemm> last;     // the segment-max layer, column blocks
  std::vector<int> last_col0;
  int mid_width = 0;                  // widest stored per-edge activation (POOL)
};

int prepare_edge(PreparedEdge& e, int mode, int c_in, const float* const* weights, const float* const* biases,
                 const int32_t* dims, int num_layers, bool want_tc, cudaStream_t s) {
  PG_REQUIRE(num_layers >= 1 && num_layers <= 8, "edge MLP depth %d not in [1, 8]", num_layers);
  PG_REQUIRE(dims[0] == c_in + 3, "dims[0]=%d must equal feature channels + 3 = %d", dims[0], c_in + 3);
  e.mode = mode;
  e.c_in = c_in;
  e.num_layers = num_layers;
  e.dims.assign(dims, dims + num_layers + 1);
  e.w.assign(weights, weights + num_layers);
  e.b.assign(biases, biases + num_layers);
  for (int l = 0; l < num_layers; ++l) PG_REQUIRE(weights[l] && biases[l], "null weight/bias for layer %d", l);
  e.path = EDGE_FP32;
  if (!want_tc || num_layers < 2) return PG_OK;
  if (mode == PG_EDGE_POOL) {
    // PointSetPooling (one feature channel): layer 0 in fp32 inside the producer of layer 1; layers 1 .. L-2
    // store their per-edge activations (rows for the next layer); layer L-1 ends in the segment max
    if (c_in != 1) return PG_OK;
    for (int l = 1; l < num_layers; ++l) {
      if (l > 1 && dims[l] % 4 != 0) return PG_OK;
      if (l + 1 < num_layers && (dims[l + 1] > kMaxNT || dims[l + 1] % 4 != 0)) return PG_OK;
    }
    e.kp = (dims[1] + 15) / 16 * 16;
    PG_CUDA_OK(e.w1x.alloc(sizeof(float) * 5 * e.kp, s));
    pad_rows_kernel<<<4, 256, 0, s>>>(weights[0], 4, dims[1], e.kp, e.w1x.as<float>());
    PG_LAUNCH_CHECK();
    pad_rows_kernel<<<2, 256, 0, s>>>(biases[0], 1, dims[1], e.kp, e.w1x.as<float>() + 4 * e.kp);
    PG_LAUNCH_CHECK();
    e.mid = std::vector<PreparedGemm>(num_layers - 2);
    for (int l = 1; l + 1 < num_layers; ++l) {
      if (int rc = prepare_gemm(e.mid[l - 1], weights[l], dims[l + 1], biases[l], dims[l], dims[l + 1], s)) return rc;
      e.mid_width = std::max(e.mid_width, int(dims[l + 1]));
    }
    const int n = dims[num_layers];
    if (int rc = prepare_column_blocks(e.last, e.last_col0, weights[num_layers - 1], n, biases[num_layers - 1],
                                       dims[num_layers - 1], n, n, s))
      return rc;
    e.path = EDGE_POOL;
    return PG_OK;
  }
  if (num_layers != 2) return PG_OK;
  const int d1 = dims[1], n = dims[2];
  e.kp = (d1 + 15) / 16 * 16;
  // hoisted first layer on the tensor cores too: logical N = kp, the pad columns get zero weights and bias
  if (int rc = prepare_fc(e.p_fc, weights[0], d1, biases[0], c_in, d1, e.kp, true, s)) return rc;
  if (!e.p_fc.tc) {   // FFMA fallback writes the zero padding itself (ldo = kp)
    e.p_fc.n = d1;
    PG_REQUIRE(e.kp <= (d1 + 63) / 64 * 64, "hoisted layer: padded width %d too far from %d", e.kp, d1);
  }
  PG_CUDA_OK(e.w1x.alloc(sizeof(float) * 3 * e.kp, s));
  pad_rows_kernel<<<4, 256, 0, s>>>(weights[0] + int64_t(c_in) * d1, 3, d1, e.kp, e.w1x.as<float>());
  PG_LAUNCH_CHECK();
  if (int rc = prepare_column_blocks(e.last, e.last_col0, weights[1], n, biases[1], d1, n, n, s)) return rc;
  e.path = EDGE_GNN;
  return PG_OK;
}

// the segment-max layer over all column blocks; p carries the producer's inputs
template <int kProd>
int apply_last(const PreparedEdge& e, WgParams p, int n, float* out, cudaStream_t s) {
  for (size_t b = 0; b < e.last.size(); ++b) {
    p.out = out + e.last_col0[b];
    p.ldo = n;
    if (int rc = launch_wg<kProd, EPI_SEGMAX>(p, e.last[b], s)) return rc;
  }
  return PG_OK;
}

// the launches of one edge call: the segment max into out (pre-filled with -FLT_MAX); an out-of-range src / dst
// sets *err
int launch_edge(const PreparedEdge& e, const float* features, const float* xyz_src, const float* xyz_dst,
                const int32_t* dst_index, const int32_t* src, const int32_t* dst, int64_t num_edges, int64_t num_src,
                int64_t num_dst, float* out, int* err, cudaStream_t s) {
  const int n = e.dims[e.num_layers];
  if (e.path == EDGE_FP32 || num_edges == 0)
    return edge_mlp_max_fp32(e.mode, features, e.c_in, xyz_src, xyz_dst, dst_index, src, dst, num_edges, num_src, num_dst,
                             e.w.data(), e.b.data(), e.dims.data(), e.num_layers, out, err, s);
  WgParams p{};
  p.xyz_src = xyz_src;
  p.xyz_dst = xyz_dst;
  p.dst_index = dst_index;
  p.num_src = num_src;
  p.num_dst = num_dst;
  p.w1x = e.w1x.as<float>();
  p.err = err;
  if (e.path == EDGE_POOL) {
    const int L = e.num_layers;
    p.feat = features;
    if (L == 2) {
      p.src = src;
      p.dst = dst;
      p.num_rows = num_edges;
      return apply_last<PROD_POOL>(e, p, n, out, s);
    }
    // the stored per-edge activations are bounded by slicing the edge list (a destination whose edges straddle
    // two slices is merged by the atomic max like any tile boundary)
    const int64_t slice = std::min<int64_t>(num_edges, int64_t(1) << 20);
    Temp h[2];
    PG_CUDA_OK(h[0].alloc(sizeof(float) * slice * e.mid_width, s));
    if (L > 3) PG_CUDA_OK(h[1].alloc(sizeof(float) * slice * e.mid_width, s));
    for (int64_t e0 = 0; e0 < num_edges; e0 += slice) {
      const int64_t ne = std::min(slice, num_edges - e0);
      WgParams q = p;
      q.src = src + e0;
      q.dst = dst + e0;
      q.num_rows = ne;
      q.out = h[0].as<float>();
      q.ldo = e.dims[2];
      q.act = 1;
      if (int rc = launch_wg<PROD_POOL, EPI_STORE>(q, e.mid[0], s)) return rc;
      for (int l = 2; l < L; ++l) {
        WgParams r{};
        r.x = h[l & 1].as<float>();
        r.ldx = e.dims[l];
        r.k_real = e.dims[l];
        r.num_rows = ne;
        r.dst = dst + e0;
        r.num_dst = num_dst;
        r.err = err;
        if (l + 1 < L) {
          r.out = h[(l + 1) & 1].as<float>();
          r.ldo = e.dims[l + 1];
          r.act = 1;
          if (int rc = launch_wg<PROD_ROWS, EPI_STORE>(r, e.mid[l - 1], s)) return rc;
        } else if (int rc = apply_last<PROD_ROWS>(e, r, n, out, s)) {
          return rc;
        }
      }
    }
    return PG_OK;
  }
  // GNN edge layer: hoisted per-vertex GEMM, then the fused gather / second layer / segment max kernel
  Temp t_p;
  PG_CUDA_OK(t_p.alloc(sizeof(float) * num_src * e.kp, s));
  if (int rc = apply_fc(e.p_fc, features, num_src, 0, nullptr, t_p.as<float>(), e.kp, s)) return rc;
  p.x = t_p.as<float>();
  p.ldx = e.kp;
  p.k_real = e.kp;
  p.src = src;
  p.dst = dst;
  p.num_rows = num_edges;
  return apply_last<PROD_GNN>(e, p, n, out, s);
}

// one edge call on either route: the error word, the -FLT_MAX fill of out, the launches, and the read-back of the
// error word unless the caller vouched for the indices (trusted: no read-back, no synchronisation)
int apply_edge(const PreparedEdge& e, const float* features, const float* xyz_src, const float* xyz_dst,
               const int32_t* dst_index, const int32_t* src, const int32_t* dst, int64_t num_edges, int64_t num_src,
               int64_t num_dst, bool trusted, float* out, cudaStream_t s) {
  ErrorWord err;
  if (int rc = err.init(s)) return rc;
  if (int rc = fill_async(out, num_dst * e.dims[e.num_layers], -FLT_MAX, s)) return rc;
  if (int rc = launch_edge(e, features, xyz_src, xyz_dst, dst_index, src, dst, num_edges, num_src, num_dst, out,
                           err.ptr(), s))
    return rc;
  int h = 0;
  if (int rc = err.read(&h, trusted, s)) return rc;
  PG_REQUIRE(h == 0, "edge index out of range (src in [0,%lld), dst in [0,%lld))", (long long)num_src,
             (long long)num_dst);
  return PG_OK;
}

// ---- the class-aware predictor heads (gnn.py:133-163) ---------------------------------------------
// After the concatenated first layers (one GEMM: [D] -> H * (C + 1), ReLU) everything left is tiny per vertex:
// cls H -> C (linear), and per class H -> H (ReLU) -> box_len (linear).  One SIMT kernel does all of it for a
// tile of 32 vertices with every head weight resident in shared memory, and writes logits, class
// probabilities (softmax, models.py:165-168) and the stacked box encodings [K, C, box_len].
constexpr int kHeadRows = 64;     // vertices per tile
constexpr int kHeadThreads = 256; // thread = (row = tid / 4, quarter = tid % 4): 16 of the 64 second-layer outputs of its row
constexpr int kHeadH = 64;        // hidden width the kernel is built for (models.py:60-64 classaware_predictor)

struct HeadsParams {
  const float* hid;      // [m, htot] = relu(first layers), columns: cls hidden [H] then class c hidden [H] ...
  int64_t m;
  int htot, C, box;
  const float* wpack;    // [Wcls H*C | bcls C | per class: W2 H*H | b2 H | W3 H*box | b3 box], sections padded to 4 floats
  int wfloats;
  float* logits;         // [m, C]
  float* probs;          // [m, C] or null
  float* boxes;          // [m, C, box]
};

__global__ void __launch_bounds__(kHeadThreads) predictor_heads_kernel(HeadsParams p) {
  constexpr int H = kHeadH, XS = H + 1;
  extern __shared__ __align__(16) float hsm[];
  float* w = hsm;                                  // all head weights
  float* x = w + ((p.wfloats + 3) & ~3);           // [kHeadRows][H + 1]: the hidden slice being consumed
  float* h2 = x + kHeadRows * XS;                  // [kHeadRows][H + 1]: second-layer output of the class
  float* lg = h2 + kHeadRows * XS;                 // [kHeadRows][16]: class logits
  const int C = p.C, box = p.box;
  const int tid = threadIdx.x, r = tid >> 2, qd = tid & 3;
  for (int i = tid; i < p.wfloats; i += kHeadThreads) w[i] = p.wpack[i];
  // every section of the pack starts on a 16-byte boundary (128-bit shared loads below)
  const int cpad = (C + 3) & ~3, hb = (H * box + 3) & ~3, bpad = (box + 3) & ~3;
  const float* wcls = w;
  const float* bcls = w + ((H * C + 3) & ~3);
  const int head0 = ((H * C + 3) & ~3) + cpad;
  const int per_class = H * H + H + hb + bpad;
  const int64_t tiles = (p.m + kHeadRows - 1) / kHeadRows;
  for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int64_t row0 = tile * kHeadRows;
    const int rows = int(min(int64_t(kHeadRows), p.m - row0));
    for (int c = -1; c < C; ++c) {
      // stage the hidden slice of this head (c = -1: the cls head), coalesced
      __syncthreads();
      for (int i = tid; i < kHeadRows * H; i += kHeadThreads) {
        const int rr = i >> 6, cc = i & (H - 1);
        x[rr * XS + cc] = rr < rows ? p.hid[(row0 + rr) * p.htot + (c + 1) * H + cc] : 0.0f;
      }
      __syncthreads();
      if (c < 0) {
        // class logits: thread (row, qd) -> classes qd, qd + 4, ...; then softmax by the row's first thread
        for (int cls = qd; cls < C; cls += 4) {
          float a = bcls[cls];
#pragma unroll 8
          for (int i = 0; i < H; ++i) a = fmaf(x[r * XS + i], wcls[i * C + cls], a);
          lg[r * 16 + cls] = a;
        }
        __syncthreads();
        if (qd == 0 && r < rows) {
          float mx = -FLT_MAX;
          for (int cls = 0; cls < C; ++cls) {
            const float a = lg[r * 16 + cls];
            p.logits[(row0 + r) * C + cls] = a;
            mx = fmaxf(mx, a);
          }
          if (p.probs != nullptr) {
            float sum = 0.0f;
            for (int cls = 0; cls < C; ++cls) sum += expf(lg[r * 16 + cls] - mx);
            for (int cls = 0; cls < C; ++cls) p.probs[(row0 + r) * C + cls] = expf(lg[r * 16 + cls] - mx) / sum;
          }
        }
        continue;
      }
      const float* w2 = w + head0 + c * per_class;
      const float* b2 = w2 + H * H;
      const float* w3 = b2 + H;
      const float* b3 = w3 + hb;
      // second layer: 16 outputs of row r per thread, weights as broadcast 128-bit shared loads
      float acc[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[j] = b2[qd * 16 + j];
#pragma unroll 4
      for (int i = 0; i < H; ++i) {
        const float xv = x[r * XS + i];
        const float4* wr = reinterpret_cast<const float4*>(w2 + i * H + qd * 16);
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) {
          const float4 q = wr[j4];
          acc[4 * j4 + 0] = fmaf(xv, q.x, acc[4 * j4 + 0]);
          acc[4 * j4 + 1] = fmaf(xv, q.y, acc[4 * j4 + 1]);
          acc[4 * j4 + 2] = fmaf(xv, q.z, acc[4 * j4 + 2]);
          acc[4 * j4 + 3] = fmaf(xv, q.w, acc[4 * j4 + 3]);
        }
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) h2[r * XS + qd * 16 + j] = fmaxf(acc[j], 0.0f);
      __syncthreads();
      // third layer (H -> box, linear): outputs qd, qd + 4, ... of row r
      if (r < rows) {
        for (int o = qd; o < box; o += 4) {
          float a = b3[o];
#pragma unroll 8
          for (int i = 0; i < H; ++i) a = fmaf(h2[r * XS + i], w3[i * box + o], a);
          p.boxes[((row0 + r) * C + c) * box + o] = a;
        }
      }
    }
  }
}

__global__ void copy_block_kernel(const float* __restrict__ src, int64_t rows, int cols, int ld_dst, float* __restrict__ dst) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < rows * cols; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t r = i / cols;
    const int c = int(i - r * cols);
    dst[r * ld_dst + c] = src[i];
  }
}

struct PreparedPredictor {
  int D = 0, H = 0, C = 0, box = 0, htot = 0;
  bool fused = false;
  // fused route: the concatenated first layers on the tensor cores, then predictor_heads_kernel
  Temp wcat, bcat, wpack;                  // [D, htot] concatenated first layers, [htot], head weights
  std::vector<PreparedFc> first;           // column groups of the concatenated first layer (<= 256 wide each)
  std::vector<int> col0;
  int wfloats = 0;
  size_t smem = 0;
  // per-layer route: every layer prepared on its own
  std::vector<PreparedFc> layers;
};

// dims = {D, H, C, box_len}; layers = cls fc0, cls fc1, then per class c: fc0, fc1, fc2
int prepare_predictor(PreparedPredictor& P, const float* const* weights, const float* const* biases,
                      const int32_t* dims, int num_layers, bool want_tc, cudaStream_t s) {
  P.D = dims[0];
  P.H = dims[1];
  P.C = dims[2];
  P.box = dims[3];
  PG_REQUIRE(num_layers == 2 + 3 * P.C && P.C >= 1 && P.C <= 16 && P.H >= 1 && P.box >= 1,
             "pg_layer_create: predictor needs 2 + 3 C layers, 1 <= C <= 16");
  P.htot = P.H * (P.C + 1);
  auto pad4 = [](int v) { return (v + 3) & ~3; };
  P.wfloats = pad4(P.H * P.C) + pad4(P.C) + P.C * (pad4(P.H * P.H) + pad4(P.H) + pad4(P.H * P.box) + pad4(P.box));
  P.smem = (size_t((P.wfloats + 3) & ~3) + 2 * size_t(kHeadRows) * (kHeadH + 1) + size_t(kHeadRows) * 16) * sizeof(float);
  // the heads kernel is built for H = kHeadH and keeps every head weight in shared memory; the first-layer groups
  // read column slices of the concatenated matrix, which only the tensor-core path can (every group is >= H wide,
  // so all of them qualify when one H-wide group does)
  P.fused = want_tc && P.H == kHeadH && P.smem <= 227 * 1024 && fc_uses_tc(P.D, P.H);
  if (P.fused) {
    PG_CUDA_OK(P.wcat.alloc(sizeof(float) * size_t(P.D) * P.htot, s));
    PG_CUDA_OK(P.bcat.alloc(sizeof(float) * P.htot, s));
    PG_CUDA_OK(P.wpack.alloc(sizeof(float) * P.wfloats, s));
    // concatenated first layers: column block h = 0 is the cls head, h = 1 + c the loc head of class c
    for (int h = 0; h <= P.C; ++h) {
      const int l = h == 0 ? 0 : 2 + 3 * (h - 1);
      copy_block_kernel<<<32, 256, 0, s>>>(weights[l], P.D, P.H, P.htot, P.wcat.as<float>() + h * P.H);
      PG_LAUNCH_CHECK();
      PG_CUDA_OK(cudaMemcpyAsync(P.bcat.as<float>() + h * P.H, biases[l], sizeof(float) * P.H, cudaMemcpyDeviceToDevice, s));
    }
    // the heads' weight pack, sections in the order predictor_heads_kernel reads them, each on a 16-byte boundary
    std::vector<std::pair<const float*, size_t>> sections = {{weights[1], size_t(P.H) * P.C}, {biases[1], size_t(P.C)}};
    for (int c = 0; c < P.C; ++c) {
      sections.push_back({weights[2 + 3 * c + 1], size_t(P.H) * P.H});
      sections.push_back({biases[2 + 3 * c + 1], size_t(P.H)});
      sections.push_back({weights[2 + 3 * c + 2], size_t(P.H) * P.box});
      sections.push_back({biases[2 + 3 * c + 2], size_t(P.box)});
    }
    float* wp = P.wpack.as<float>();
    PG_CUDA_OK(cudaMemsetAsync(wp, 0, sizeof(float) * P.wfloats, s));
    size_t off = 0;
    for (const auto& sec : sections) {
      PG_CUDA_OK(cudaMemcpyAsync(wp + off, sec.first, sizeof(float) * sec.second, cudaMemcpyDeviceToDevice, s));
      off += (sec.second + 3) & ~size_t(3);
    }
    // column groups of at most 256 (whole heads) -> one tensor-core GEMM each
    const int heads_per_group = std::max(1, 256 / P.H);
    for (int h0 = 0; h0 <= P.C; h0 += heads_per_group) {
      const int nh = std::min(heads_per_group, P.C + 1 - h0);
      P.first.emplace_back();
      P.col0.push_back(h0 * P.H);
      if (int rc = prepare_fc(P.first.back(), P.wcat.as<float>() + h0 * P.H, P.htot, P.bcat.as<float>() + h0 * P.H, P.D,
                              nh * P.H, nh * P.H, want_tc, s))
        return rc;
      if (!P.first.back().tc) P.fused = false;   // FFMA kernel needs contiguous weights: per-layer route
    }
  }
  if (P.fused) return PG_OK;
  P.first.clear();
  P.layers.resize(num_layers);
  for (int l = 0; l < num_layers; ++l) {
    const int pos = l < 2 ? l : (l - 2) % 3;
    const int k = pos == 0 ? P.D : P.H;
    const int n = l == 1 ? P.C : (l >= 2 && pos == 2 ? P.box : P.H);
    if (int rc = prepare_fc(P.layers[l], weights[l], n, biases[l], k, n, n, want_tc, s)) return rc;
  }
  return PG_OK;
}

}  // namespace
}  // namespace pg

using namespace pg;

// ---------------------------------------------------------------------------------------------------
// per-call entry points: a transient prepared layer on the stack, applied once
// ---------------------------------------------------------------------------------------------------
extern "C" int pg_fully_connected(const float* x, int64_t m, int32_t k, const float* w, const float* bias, int32_t n,
                                  int32_t act, const float* residual, float* out, int32_t precision, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(m >= 0 && k >= 1 && n >= 1, "pg_fully_connected: bad sizes m=%lld k=%d n=%d", (long long)m, k, n);
  PG_REQUIRE(act == 0 || act == 1, "pg_fully_connected: act must be 0 (linear) or 1 (ReLU)");
  if (m == 0) return PG_OK;
  PG_REQUIRE(x && w && bias && out, "pg_fully_connected: null argument");
  PG_REQUIRE(precision == 0 || precision == 1, "pg_fully_connected: unknown precision %d", precision);
  PreparedFc f;
  if (int rc = prepare_fc(f, w, n, bias, k, n, n, precision == 1 && pg_tc_available(), s)) return rc;
  return apply_fc(f, x, m, act, residual, out, n, s);
}

extern "C" int pg_edge_mlp_max(int32_t mode, const float* features, int32_t num_feature_channels, const float* xyz_src,
                               const float* xyz_dst, const int32_t* dst_index, const int32_t* src, const int32_t* dst,
                               int64_t num_edges, int64_t num_src, int64_t num_dst, const float* const* weights_host,
                               const float* const* biases_host, const int32_t* dims_host, int32_t num_layers, float* out,
                               int32_t precision, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(mode == PG_EDGE_POOL || mode == PG_EDGE_GNN, "pg_edge_mlp_max: unknown mode %d", mode);
  PG_REQUIRE(weights_host && biases_host && dims_host, "pg_edge_mlp_max: null layer tables");
  PG_REQUIRE(num_edges >= 0 && num_src >= 1 && num_dst >= 0, "pg_edge_mlp_max: bad sizes");
  PG_REQUIRE(out != nullptr || num_dst == 0, "pg_edge_mlp_max: out is null");
  PG_REQUIRE((features && xyz_src && xyz_dst && src && dst) || num_edges == 0, "pg_edge_mlp_max: null input");
  PG_REQUIRE(mode == PG_EDGE_GNN || dst_index != nullptr || num_edges == 0,
             "pg_edge_mlp_max: POOL mode needs keypoint indices");
  const bool trusted = (precision & PG_FLAG_TRUSTED_INDICES) != 0;
  precision &= PG_PRECISION_MASK;
  PG_REQUIRE(precision == 0 || precision == 1, "pg_edge_mlp_max: unknown precision %d", precision);
  PreparedEdge e;
  if (int rc = prepare_edge(e, mode, num_feature_channels, weights_host, biases_host, dims_host, num_layers,
                            precision == 1 && num_edges > 0 && pg_tc_available(), s))
    return rc;
  return apply_edge(e, features, xyz_src, xyz_dst, dst_index, src, dst, num_edges, num_src, num_dst, trusted, out, s);
}

// ---------------------------------------------------------------------------------------------------
// pg_layer: prepared layers behind the C ABI
// ---------------------------------------------------------------------------------------------------
struct pg_layer {
  int kind = 0, num_layers = 0;
  std::vector<int32_t> dims;
  std::vector<PreparedFc> fcs;          // PG_LAYER_MLP
  PreparedEdge edge;                    // PG_LAYER_EDGE_POOL / PG_LAYER_EDGE_GNN
  PreparedPredictor pred;               // PG_LAYER_PREDICTOR
};

extern "C" int pg_layer_create(int32_t kind, const float* const* weights_host, const float* const* biases_host,
                               const int32_t* dims_host, int32_t num_layers, int32_t precision, void* stream,
                               pg_layer** out_layer) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(out_layer != nullptr, "pg_layer_create: out_layer is null");
  *out_layer = nullptr;
  PG_REQUIRE(weights_host && biases_host && dims_host && num_layers >= 1 && num_layers <= 64, "pg_layer_create: bad layer tables");
  PG_REQUIRE(precision == 0 || precision == 1, "pg_layer_create: unknown precision %d", precision);
  PG_REQUIRE(kind == PG_LAYER_MLP || kind == PG_LAYER_EDGE_POOL || kind == PG_LAYER_EDGE_GNN || kind == PG_LAYER_PREDICTOR,
             "pg_layer_create: unknown kind %d", kind);
  for (int l = 0; l < num_layers; ++l) PG_REQUIRE(weights_host[l] && biases_host[l], "pg_layer_create: null weight/bias %d", l);
  auto L = std::make_unique<pg_layer>();
  L->kind = kind;
  L->num_layers = num_layers;
  const bool want_tc = precision == 1 && pg_tc_available();
  if (kind == PG_LAYER_MLP) {
    L->dims.assign(dims_host, dims_host + num_layers + 1);
    L->fcs.resize(num_layers);
    for (int l = 0; l < num_layers; ++l)
      if (int rc = prepare_fc(L->fcs[l], weights_host[l], dims_host[l + 1], biases_host[l], dims_host[l],
                              dims_host[l + 1], dims_host[l + 1], want_tc, s))
        return rc;
  } else if (kind == PG_LAYER_EDGE_POOL || kind == PG_LAYER_EDGE_GNN) {
    L->dims.assign(dims_host, dims_host + num_layers + 1);
    if (int rc = prepare_edge(L->edge, kind == PG_LAYER_EDGE_POOL ? PG_EDGE_POOL : PG_EDGE_GNN, dims_host[0] - 3,
                              weights_host, biases_host, dims_host, num_layers, want_tc, s))
      return rc;
  } else {
    L->dims.assign(dims_host, dims_host + 4);
    if (int rc = prepare_predictor(L->pred, weights_host, biases_host, dims_host, num_layers, want_tc, s)) return rc;
  }
  *out_layer = L.release();
  return PG_OK;
}

extern "C" int pg_layer_destroy(pg_layer* layer) {
  delete layer;      // prepared buffers are returned to the stream-ordered pool on the stream they were made on
  return PG_OK;
}

extern "C" int pg_layer_mlp(const pg_layer* layer, const float* x, int64_t m, int32_t last_linear, const float* residual,
                            float* out, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(layer && layer->kind == PG_LAYER_MLP, "pg_layer_mlp: not an MLP layer");
  if (m == 0) return PG_OK;
  PG_REQUIRE(x && out && m > 0, "pg_layer_mlp: bad argument");
  const int L = layer->num_layers;
  Temp bufs[2];
  int widest = 0;
  for (int l = 1; l < L; ++l) widest = std::max(widest, int(layer->dims[l]));
  if (L > 1) {
    PG_CUDA_OK(bufs[0].alloc(sizeof(float) * m * widest, s));
    if (L > 2) PG_CUDA_OK(bufs[1].alloc(sizeof(float) * m * widest, s));
  }
  const float* cur = x;
  for (int l = 0; l < L; ++l) {
    const bool last = l + 1 == L;
    float* dst = last ? out : bufs[l & 1].as<float>();
    const int act = (last && last_linear) ? 0 : 1;
    if (int rc = apply_fc(layer->fcs[l], cur, m, act, last ? residual : nullptr, dst, layer->dims[l + 1], s)) return rc;
    cur = dst;
  }
  return PG_OK;
}

extern "C" int pg_layer_edge_mlp_max(const pg_layer* layer, const float* features, const float* xyz_src,
                                     const float* xyz_dst, const int32_t* dst_index, const int32_t* src,
                                     const int32_t* dst, int64_t num_edges, int64_t num_src, int64_t num_dst, float* out,
                                     int32_t flags, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(layer && (layer->kind == PG_LAYER_EDGE_POOL || layer->kind == PG_LAYER_EDGE_GNN),
             "pg_layer_edge_mlp_max: not an edge layer");
  PG_REQUIRE(num_edges >= 0 && num_src >= 1 && num_dst >= 0, "pg_layer_edge_mlp_max: bad sizes");
  PG_REQUIRE(out != nullptr || num_dst == 0, "pg_layer_edge_mlp_max: out is null");
  PG_REQUIRE((features && xyz_src && xyz_dst && src && dst) || num_edges == 0, "pg_layer_edge_mlp_max: null input");
  PG_REQUIRE(layer->kind == PG_LAYER_EDGE_GNN || dst_index != nullptr || num_edges == 0,
             "pg_layer_edge_mlp_max: POOL mode needs keypoint indices");
  return apply_edge(layer->edge, features, xyz_src, xyz_dst, dst_index, src, dst, num_edges, num_src, num_dst,
                    (flags & PG_FLAG_TRUSTED_INDICES) != 0, out, s);
}

extern "C" int pg_layer_predictor(const pg_layer* layer, const float* x, int64_t m, float* logits, float* boxes,
                                  float* probs, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PG_REQUIRE(layer && layer->kind == PG_LAYER_PREDICTOR, "pg_layer_predictor: not a predictor layer");
  if (m == 0) return PG_OK;
  PG_REQUIRE(x && logits && boxes && m > 0, "pg_layer_predictor: bad argument");
  const PreparedPredictor& P = layer->pred;
  if (P.fused) {
    Temp hid;
    PG_CUDA_OK(hid.alloc(sizeof(float) * m * P.htot, s));
    for (size_t g = 0; g < P.first.size(); ++g)
      if (int rc = apply_fc(P.first[g], x, m, 1, nullptr, hid.as<float>() + P.col0[g], P.htot, s)) return rc;
    HeadsParams hp{};
    hp.hid = hid.as<float>();
    hp.m = m;
    hp.htot = P.htot;
    hp.C = P.C;
    hp.box = P.box;
    hp.wpack = P.wpack.as<float>();
    hp.wfloats = P.wfloats;
    hp.logits = logits;
    hp.probs = probs;
    hp.boxes = boxes;
    static bool attr_done = false;
    if (!attr_done) {
      PG_CUDA_OK(cudaFuncSetAttribute(predictor_heads_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      attr_done = true;
    }
    const int blocks = int(std::min<int64_t>(ceil_div(m, kHeadRows), num_sms()));
    predictor_heads_kernel<<<blocks, kHeadThreads, P.smem, s>>>(hp);
    PG_LAUNCH_CHECK();
    return PG_OK;
  }
  // per-layer route
  Temp h1, h2, tmp;
  PG_CUDA_OK(h1.alloc(sizeof(float) * m * P.H, s));
  PG_CUDA_OK(h2.alloc(sizeof(float) * m * P.H, s));
  PG_CUDA_OK(tmp.alloc(sizeof(float) * m * P.box, s));
  if (int rc = apply_fc(P.layers[0], x, m, 1, nullptr, h1.as<float>(), P.H, s)) return rc;
  if (int rc = apply_fc(P.layers[1], h1.as<float>(), m, 0, nullptr, logits, P.C, s)) return rc;
  if (probs != nullptr)
    if (int rc = pg_softmax_rows(logits, m, P.C, probs, stream)) return rc;
  for (int c = 0; c < P.C; ++c) {
    const int l = 2 + 3 * c;
    if (int rc = apply_fc(P.layers[l], x, m, 1, nullptr, h1.as<float>(), P.H, s)) return rc;
    if (int rc = apply_fc(P.layers[l + 1], h1.as<float>(), m, 1, nullptr, h2.as<float>(), P.H, s)) return rc;
    if (int rc = apply_fc(P.layers[l + 2], h2.as<float>(), m, 0, nullptr, tmp.as<float>(), P.box, s)) return rc;
    copy_block_kernel<<<64, 256, 0, s>>>(tmp.as<float>(), m, P.box, P.C * P.box, boxes + c * P.box);
    PG_LAUNCH_CHECK();
  }
  return PG_OK;
}
