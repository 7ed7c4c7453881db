// Hopper tensor-core kernels (wgmma): the fast paths (precision = 1, "BF16x3", and precision = 2, "FP16").
//
// wg_gemm_kernel - one persistent kernel for every tensor-core layer of the network: out = epilogue(A @ W + b), A
//   produced on the fly (in registers, or in shared memory for the pooling launches) by the warpgroups that also run
//   the wgmmas.  Dense and pooling layers stream W through a producer warpgroup; the GNN edge layer keeps its W
//   resident in shared memory (mapping, below).
//
//   producers  PROD_ROWS  A = rows of an fp32 matrix (dense layers, a pooling layer wider than one launch)
//              PROD_GNN   one GNN iteration's edge MLP (/root/reference/models/gnn.py:338-365) after hoisting:
//                         e0 @ W1 + b1 = (F @ W1[:C] + b1)[src] + (x_src - x_dst') @ W1[C:], so the first edge
//                         layer is a per-VERTEX table P (a PROD_ROWS GEMM) plus a 3-term per-edge correction;
//                         A row e = act(P[src] + (x_src - x_dst') @ W1[C:])
//              PROD_POOL  PointSetPooling's first layer (gnn.py:264-270) in fp32:
//                         A row e = relu([feature(src), x_src - x_kp(dst)] @ W0 + b0), then the chain: every
//                         further pooling layer ahead of the kernel's own runs on the same tile with its input and
//                         output in the consumer warpgroup's shared-memory region, never in global memory
//   epilogues  EPI_STORE  act(acc + b) (+ residual) to a row-major matrix
//              EPI_SEGMAX max over the edges of each destination (edges are grouped by destination):
//                         bias and every activation are monotone, so they commute with max: raw accumulators
//                         are reduced across the warp's 16 rows with shuffles and each partial max is flushed
//                         with one atomic; a warp holding two destinations (rows 0 and 15) reduces each in turn
//              EPI_SEGSUM sum over the edges of each destination (the mean divides it afterwards, apply_edge): bias
//                         and activation do not commute with a sum, so the accumulators start at the bias and act is
//                         applied to every element in registers first; then the same reduction with + and a flush with
//                         atomicAdd into an output filled with 0.  The order of the fp32 partial sums is not fixed:
//                         the last bits may differ from run to run.  Its instances are wg_segsum_kernel, the same
//                         bodies under their own name
//              EPI_SEGSUM_ORDERED the same sum in a fixed order (PG_FLAG_DETERMINISTIC, pg_common.cuh): a warp's 16
//                         rows are a unit; its runs are reduced with the same shuffles, the halves' runs that meet at
//                         rows 7 / 8 joined in registers (half 0 + half 1), and instead of atomics a run that holds
//                         neither row 0 nor row 15 is stored, the two that do go to the side buffer for
//                         ordered_fixup.  Its instances are wg_segsum_ordered_kernel
//   activation the kAnyAct = false instances hard-code ReLU (linear too in the store epilogue): the kernel of every
//              shipped config.  kAnyAct = true, the GNN edge layer with any other activation, is the same body with
//              activate(p.act, .) in the producer; its segment max flushes the RAW maxima with the sign-aware
//              atomic_max_float (NONE, LeakyReLU, ELU and Tanh give negative values) and activate_rows applies
//              act(. + b) once per output element afterwards.  Dense layers with another activation run
//              wg_gemm_kernel linear, then activate_rows
//   precision  BF16x3 (kArith = ARITH_BF16X3): every fp32 operand is split x = hi + lo (two BF16), and
//              hi*hi' + lo*hi' + hi*lo' is accumulated in fp32 registers: ~2^-16 relative per product (fp32-class
//              accuracy).  FP16 (kArith = ARITH_F16): every operand is rounded once to FP16
//              (nearest, saturating at +-65504), one wgmma per 16-k chunk, fp32 accumulation: ~2^-11 relative per
//              operand, a third of the wgmmas and half the W bytes.  Everything that is not a tensor-core operand
//              (the GNN layer's per-edge correction, pooling layer 0, bias, activation, segment max) stays fp32 in both
//   mapping    GNN (wg_gnn_body): W resident.  A CTA owns one NI-wide column group c = blockIdx.x % NS of the padded
//              output.  At kernel start one thread copies that group's hi and lo slices of every 16-k chunk (NI x 32 B
//              each, straight out of the image layout below) into shared memory with cp.async.bulk on one mbarrier,
//              which every thread waits on once: kp x NI x 4 B, 185 KB for the car layer (304 x 152).  W then stays
//              for the whole launch: no ring, no per-chunk barrier, no producer warpgroup.  The three warpgroups
//              are independent consumers of 64-row tiles (tiles 3 j + wg of CTA slot j = blockIdx.x / NS, stepping by
//              3 gridDim.x / NS), one m64nNIk16 accumulator each, A in registers as below.  Their rows of P reach
//              shared memory kGnnStages chunks ahead of the wgmmas, copied by each thread with cp.async (GnnGather),
//              and the copies run on into the warpgroup's next tile.  Nothing makes one
//              warpgroup wait for another, so while one flushes its segment max the other two keep the tensor cores
//              busy.  Every output column gets the same wgmmas on the same operands in the same order as with the
//              whole N in one warpgroup, so the results do not depend on the grouping.  Both column groups gather the
//              same P rows (twice the gather, against a W stream of 370 KB per 128-row tile).
//              ROWS and POOL: CTA = 3 warpgroups.  Warpgroup 0 is the W producer (setmaxnreg down to 24 registers): one thread
//              streams W (hi and lo images, pre-packed in the no-swizzle K-major core-matrix layout, one
//              contiguous block per 16-k chunk) from L2 through a ring of shared-memory stages with
//              cp.async.bulk, each stage tracked by a "full" (bytes landed) and an "empty" (both consumers done)
//              mbarrier.  Warpgroups 1 and 2 are the consumers (setmaxnreg up to 240): 128 rows per tile (64 per
//              warpgroup), the whole padded N (<= 304: two m64nNk16 instructions) in registers.  A streamed ROWS
//              layer, like the GNN layer, takes A from registers (wgmma_bf16_rs): each thread builds its own fragment of a chunk (its
//              accumulators' two rows, 4 k) from its gathered fp32 values, in one of two alternating register
//              buffers, issuing the global loads of chunk k + 2 before the wgmmas of chunk k + 1 and building
//              chunk k + 1 while chunk k's wgmmas run: no shared-memory A, proxy fence or barrier per chunk.  The
//              pooling launches read A from shared memory: layer 1's fragments are stored to a double buffer
//              there, the chain's on-chip layers leave theirs in the region.  A consumer only arrives on "empty"; it
//              never waits on it or issues a copy: such divergent code in the k-loop makes ptxas serialise the
//              wgmmas (C7518), and the two consumers would wait for each other on every chunk.
//
// Shared-memory operand layout (no swizzle, K-major): 8-row x 16-byte core matrices, 128 contiguous bytes each;
// for a 16-k chunk, core(row group g, k half kc) at g * 256 + kc * 128 (LBO = 128, SBO = 256).
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <memory>
#include <type_traits>
#include <utility>
#include <vector>

#include "pg_common.cuh"
#include "pg_wgmma.cuh"

namespace pg {
// [0] segment-max (edge) launches, [1] store (dense) launches, [2] ordered segment-sum fix-ups (any path)
static std::atomic<long long> g_tc_launches[3];
void count_ordered_launch() { g_tc_launches[2].fetch_add(1, std::memory_order_relaxed); }
}

// tensor-core kernel launches so far: which = 0 segment-max (edge layer) launches, 1 dense-layer launches, 2 the
// fix-up launches of the ordered segment sum
extern "C" int64_t pg_tc_launch_count(int32_t which) {
  return (which >= 0 && which <= 2) ? pg::g_tc_launches[which].load(std::memory_order_relaxed) : -1;
}

namespace pg {
namespace {
using namespace wg;

constexpr int kWgThreads = 384;     // dense / pooling: warpgroup 0 streams W, 1 and 2 compute;  GNN: all three compute
constexpr int kProducerRegs = 24;   // 2 x 128 x 240 + 128 x 24 = 384 x 168, the launch bound's budget
constexpr int kConsumerRegs = 240;  // 232 spills 8 bytes in the 152 x 2 segment-max instances
constexpr int kTileRows = 128;      // rows per tile (64 per consumer warpgroup)
// 4 W stages beat 8 on H100: the ring is deep enough for the copies, and the smaller shared-memory carve-out leaves
// more L1 for the gathered rows (GNN edge layer at the benchmark shape: 7.7 vs 8.0 ms, H100 SXM at a 400 W limit)
constexpr int kMaxRing = 4;
constexpr int kMaxNT = 304;         // widest padded N one launch covers
constexpr int kMaxChain = 6;        // on-chip pooling layers ahead of the kernel's own (edge MLPs have <= 8 layers)

// The arithmetic of a tensor-core layer (header, "precision"): BF16x3 keeps two operand planes (hi, lo) per 16-k
// chunk and issues three wgmmas; FP16 keeps one plane and issues one
enum { ARITH_BF16X3 = 0, ARITH_F16 = 1 };
constexpr int arith_planes(int arith) { return arith == ARITH_F16 ? 1 : 2; }
// bytes of one W row (output feature) of a 16-k chunk: 32 per plane
constexpr uint32_t w_row_bytes(int arith) { return 32u * uint32_t(arith_planes(arith)); }
// one warpgroup's shared-memory A chunk, 64 rows x 16 k: 2048 bytes per plane
constexpr uint32_t a_chunk_bytes(int arith) { return 2048u * uint32_t(arith_planes(arith)); }

// shared memory of a CTA: a ring of W stages, one A region per consumer warpgroup (POOL only: layer 1's double buffer,
// or a whole on-chip activation; ROWS and GNN keep A in registers), the full / empty barriers
constexpr size_t wg_smem_bytes(uint32_t stage_bytes, uint32_t region_bytes, int ring) {
  return size_t(ring) * stage_bytes + 2 * size_t(region_bytes) + 2 * ring * sizeof(uint64_t);
}
// the deepest power of two up to kMaxRing (so the stage of a chunk is a mask) that fits the 227 KB a CTA may use
constexpr int ring_stages(uint32_t stage_bytes, uint32_t region_bytes) {
  int r = kMaxRing;
  while (r > 1 && wg_smem_bytes(stage_bytes, region_bytes, r) > 227 * 1024) r /= 2;
  return r;
}
constexpr int log2_ring(int r) { return r >= 4 ? 2 : r >= 2 ? 1 : 0; }

// GNN edge layer (wg_gnn_body): every warpgroup of a CTA computes its own 64-row tiles against the CTA's resident
// column group of W
constexpr int kGnnWarpgroups = kWgThreads / 128;
constexpr int kGnnTileRows = 64;
// P chunks a warpgroup has in flight (GnnGather).  One beats two and three on H100 (DESIGN §6): the car layer's
// 185 KB of W plus one 4 KB stage per warpgroup still fits the 196 KB shared-memory carve-out, deeper stages take the
// 228 KB one and leave less L1
constexpr int kGnnStages = 1;
constexpr uint32_t kGnnStageBytes = 64 * 64;    // one warpgroup's 64 rows of a 16-k chunk of P, fp32
// shared memory of a GNN CTA: its column group of W (ni columns, every plane of the arithmetic, kp k), every
// warpgroup's gather stages, then the mbarrier
constexpr size_t gnn_smem_bytes(int kp, int ni, int arith) {
  return size_t(kp / 16) * ni * w_row_bytes(arith) + size_t(kGnnWarpgroups) * kGnnStages * kGnnStageBytes +
         sizeof(uint64_t);
}

enum { PROD_ROWS = 0, PROD_GNN = 1, PROD_POOL = 2 };
enum { EPI_STORE = 0, EPI_SEGMAX = 1, EPI_SEGSUM = 2, EPI_SEGSUM_ORDERED = 3 };
constexpr bool is_sum(int epi) { return epi == EPI_SEGSUM || epi == EPI_SEGSUM_ORDERED; }

struct WgParams {
  // A producer
  const float* x;           // ROWS: [num_rows, ldx];  GNN: P [num_src, ldx] (ldx = kp, zero padded)
  int ldx;                  // POOL: layer 1's padded K, the row stride of w1x
  int k_real;               // ROWS: true K (multiple of 4)
  const float* feat;        // POOL: [num_src] point features (one channel)
  const float* w1x;         // GNN: [3, kp] = W1[C:];  POOL: [4, ldx] = W0, then [ldx] = b0 (zero padded)
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
  float* out;               // STORE: [num_rows, ldo];  SEGMAX / SEGSUM: [num_dst, ldo] pre-filled with -FLT_MAX / 0
  int ldo;
  int act;                  // STORE: 0 linear, 1 relu;  kAnyAct: the GNN producer's PG_ACT_*
  const float* residual;    // STORE: optional [num_rows, ldr]
  int ldr;
  int* err;
  int64_t num_tiles;
  // POOL: the on-chip layers ahead of the kernel's own one (layer 1 first), each {16-k chunks, instruction shape
  // ni * 4 + ns, byte offset of its W image in chain_buf, byte offset of its padded bias}
  int chain_layers;
  int4 chain[kMaxChain];
  const uint8_t* chain_buf;
  uint32_t stage_bytes;     // POOL: one W ring stage (the widest chunk of any layer of the launch)
  uint32_t region_bytes;    // POOL: one consumer warpgroup's A region
  int ring_log2;            // POOL: log2 of the ring depth
  // SEGSUM_ORDERED: the side buffer (pg_common.cuh), slot 2 u + {0, 1} of 16-row unit u at part + slot * ldp; the
  // launch of the first column block writes the slots' ids
  float* part;
  int32_t* part_id;
  int ldp;
  int write_ids;
};

__device__ __forceinline__ float2 ldg_nc(const float* ptr) {
  float2 v;
  asm volatile("ld.global.nc.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(ptr));
  return v;
}

// a layer's activation: ReLU, or with kAnyAct the PG_ACT_* code act
template <bool kAnyAct>
__device__ __forceinline__ float layer_act(int act, float x) {
  return kAnyAct ? activate(act, x) : fmaxf(x, 0.0f);
}

template <int kEpi, bool kAnyAct>
__device__ __forceinline__ void seg_flush(const WgParams& p, int d, int col, float m) {
  float* dst = p.out + int64_t(d) * p.ldo + col;
  if (kEpi == EPI_SEGSUM) {
    atomicAdd(dst, m);   // a partial sum of act(acc + b)
  } else if (kAnyAct) {
    // the raw maximum, which may be negative: the sign-aware max, still one atomic (bias and activation later)
    atomic_max_float(dst, m);
  } else {
    // + 0.0f turns a -0.0f into +0.0f, which must win against the -FLT_MAX fill as an integer
    atomicMax(reinterpret_cast<int*>(dst), __float_as_int(fmaxf(m + __ldg(p.bias + col), 0.0f) + 0.0f));
  }
}

// EPI_SEGSUM_ORDERED: where the sums of destination d's run in unit u go, column by column: slot 2 u + slot of the side
// buffer, or (slot < 0, a run that is the whole destination) d's row of out.  Computed once per run, so that the
// epilogue's flushes are plain stores at a column offset (per-flush address arithmetic spills the car instances)
__device__ __forceinline__ float* ordered_row(const WgParams& p, int64_t u, int slot, int d) {
  return slot < 0 ? p.out + int64_t(max(d, 0)) * p.ldo : p.part + (2 * u + slot) * p.ldp;
}

// ptr[0 .. 2) through the read-only cache; ptr is 8-byte aligned
__device__ __forceinline__ float2 ldg2(const float* ptr) { return __ldg(reinterpret_cast<const float2*>(ptr)); }

// A rows in registers (wgmma_bf16_rs): thread t of a warpgroup holds rows 16 warp + lane / 4 and + 8 of its 64, the
// rows of its accumulators, and k = 2 (lane % 4) + {0, 1, 8, 9} of every 16-k chunk.  context() reads what the rows
// need once per tile.  ROWS: the rows of p.x;  GNN: x_src - x_dst' (GnnGather copies the rows of P);  POOL: the same
// offset and the source's feature
template <int kProd, bool kAnyAct>
struct RowA {
  const float* rp[2];
  float rx[2], ry[2], rz[2], f0[2];

  // rows row0 + 16 warp + lane / 4 (+ 8) of the layer's A
  __device__ __forceinline__ void context(const WgParams& p, int64_t row0, int warp, int lane) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t row = row0 + warp * 16 + (lane >> 2) + 8 * h;
      rp[h] = p.x;
      rx[h] = ry[h] = rz[h] = f0[h] = 0.f;
      if (row >= p.num_rows) continue;
      if (kProd == PROD_ROWS) {
        rp[h] = p.x + row * p.ldx;
        continue;
      }
      int si = __ldg(p.src + row), di = __ldg(p.dst + row);
      if (si < 0 || si >= p.num_src || di < 0 || di >= p.num_dst) {
        *p.err = 1;
        si = 0;
        di = 0;
      }
      const int64_t drow = p.dst_index ? int64_t(__ldg(p.dst_index + di)) : int64_t(di);
      rx[h] = __ldg(p.xyz_src + int64_t(si) * 3 + 0) - __ldg(p.xyz_dst + drow * 3 + 0);
      ry[h] = __ldg(p.xyz_src + int64_t(si) * 3 + 1) - __ldg(p.xyz_dst + drow * 3 + 1);
      rz[h] = __ldg(p.xyz_src + int64_t(si) * 3 + 2) - __ldg(p.xyz_dst + drow * 3 + 2);
      if (kProd == PROD_POOL) f0[h] = __ldg(p.feat + si);
    }
  }
  // ROWS: the fp32 inputs of chunk kc's fragment, q[i] for register i: the thread's row i & 1, k kq + 8 (i >> 1), + 1
  __device__ __forceinline__ void load(const WgParams& p, int kc, int lane, float2 (&q)[4]) const {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = kc * 16 + (lane & 3) * 2 + 8 * (i >> 1);
      q[i] = k + 2 <= p.k_real ? ldg_nc(rp[i & 1] + k) : make_float2(0.f, 0.f);
    }
  }
  // chunk kc's fragment: BF16x3 splits it into hi / lo, FP16 rounds it once into hi (lo is not written)
  template <int kArith>
  __device__ __forceinline__ void make_frag(const WgParams& p, const float2 (&q)[4], int kc, int lane, uint32_t (&hi)[4],
                                            uint32_t (&lo)[4]) const {
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int k = kc * 16 + (lane & 3) * 2 + 8 * c;
      float2 v[2] = {q[2 * c], q[2 * c + 1]};
      // w1x rows are kp (GNN) or ldx (POOL) floats long, a multiple of 16, so this thread's pairs are 8-byte aligned
      if (kProd == PROD_GNN) {
        const float2 wx = ldg2(p.w1x + k), wy = ldg2(p.w1x + p.kp + k), wz = ldg2(p.w1x + 2 * p.kp + k);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          v[h].x = layer_act<kAnyAct>(p.act, fmaf(rz[h], wz.x, fmaf(ry[h], wy.x, fmaf(rx[h], wx.x, v[h].x))));
          v[h].y = layer_act<kAnyAct>(p.act, fmaf(rz[h], wz.y, fmaf(ry[h], wy.y, fmaf(rx[h], wx.y, v[h].y))));
        }
      } else if (kProd == PROD_POOL) {
        const float2 wf = ldg2(p.w1x + k), wx = ldg2(p.w1x + p.ldx + k), wy = ldg2(p.w1x + 2 * p.ldx + k),
                     wz = ldg2(p.w1x + 3 * p.ldx + k), b0 = ldg2(p.w1x + 4 * p.ldx + k);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          v[h].x = fmaxf(fmaf(rz[h], wz.x, fmaf(ry[h], wy.x, fmaf(rx[h], wx.x, fmaf(f0[h], wf.x, b0.x)))), 0.0f);
          v[h].y = fmaxf(fmaf(rz[h], wz.y, fmaf(ry[h], wy.y, fmaf(rx[h], wx.y, fmaf(f0[h], wf.y, b0.y)))), 0.0f);
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if constexpr (kArith == ARITH_F16)
          hi[2 * c + h] = pack_f16x2(v[h].x, v[h].y);
        else
          split_bf16x2(v[h].x, v[h].y, &hi[2 * c + h], &lo[2 * c + h]);
      }
    }
  }
};

// chunk kc's wgmmas of one m64nNk16 accumulator, A from registers: BF16x3 hi*hi' + lo*hi' + hi*lo' (b_lo the lo plane
// of B), FP16 one product
template <int kArith, int N>
__device__ __forceinline__ void mma_rs(float (&d)[N / 2], const uint32_t (&hi)[4], const uint32_t (&lo)[4], uint64_t b_hi,
                                       uint64_t b_lo, int scale_d) {
  if constexpr (kArith == ARITH_F16) {
    wgmma_f16_rs<N>(d, hi, b_hi, scale_d);
  } else {
    wgmma_bf16_rs<N>(d, hi, b_hi, scale_d);
    wgmma_bf16_rs<N>(d, lo, b_hi, 1);
    wgmma_bf16_rs<N>(d, hi, b_lo, 1);
  }
}
// the same with A from shared memory (descriptors of its planes)
template <int kArith, int N>
__device__ __forceinline__ void mma_ss(float (&d)[N / 2], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo,
                                       int scale_d) {
  if constexpr (kArith == ARITH_F16) {
    wgmma_f16<N>(d, a_hi, b_hi, scale_d);
  } else {
    wgmma_bf16<N>(d, a_hi, b_hi, scale_d);
    wgmma_bf16<N>(d, a_lo, b_hi, 1);
    wgmma_bf16<N>(d, a_hi, b_lo, 1);
  }
}

// The k-loop of a layer whose A fragments are built in registers: frag(kc, hi, lo) builds chunk kc's fragment and
// issues the loads of what comes next; chunk(kc, hi, lo) issues chunk kc's wgmmas and leaves exactly itself in
// flight.  A fragment may be written only once the wgmmas reading it are complete: two of them, alternating, and the
// loop unrolled by two so that each chunk's fragment registers are fixed at compile time.  Chunk kc + 1's fragment is
// built while chunk kc's wgmmas run
template <class Frag, class Chunk>
__device__ __forceinline__ void rs_k_loop(int lk, Frag&& frag, Chunk&& chunk) {
  uint32_t ahi[2][4], alo[2][4];
  frag(0, ahi[0], alo[0]);
  auto step = [&](int kc, const uint32_t (&hi)[4], const uint32_t (&lo)[4], uint32_t (&next_hi)[4],
                  uint32_t (&next_lo)[4]) {
    chunk(kc, hi, lo);
    if (kc + 1 < lk) frag(kc + 1, next_hi, next_lo);
  };
  for (int kc = 0; kc < lk; kc += 2) {
    step(kc, ahi[0], alo[0], ahi[1], alo[1]);
    if (kc + 1 == lk) break;
    step(kc + 1, ahi[1], alo[1], ahi[0], alo[0]);
  }
}

// The segment sum's accumulators start at the bias (value 4 jj + 2 h + c holds column col0 + 8 jj + cq + c) and its
// first wgmma accumulates onto them: the epilogue then applies the activation alone, with no bias in registers beside
// the accumulators (bias loads there spill the car GNN instance)
template <int NI>
__device__ __forceinline__ void acc_from_bias(const WgParams& p, float (&acc)[NI / 2], int col0, int lane) {
  const int cq = (lane & 3) * 2;
#pragma unroll
  for (int jj = 0; jj < NI / 8; ++jj) {
    const float2 b = ldg2(p.bias + col0 + jj * 8 + cq);
    acc[4 * jj] = acc[4 * jj + 2] = b.x;
    acc[4 * jj + 1] = acc[4 * jj + 3] = b.y;
  }
  // the accumulators are defined here, ahead of the wgmma pipeline: otherwise ptxas may place their moves inside a
  // pooling launch's first stage and serialise its wgmmas (C7515)
#pragma unroll
  for (int v = 0; v < NI / 2; ++v) asm volatile("" : "+f"(acc[v])::"memory");
}

// Segment max (kEpi = EPI_SEGMAX) or sum (EPI_SEGSUM) of one warpgroup's 64 x (NI x NS) accumulators: output
// columns col0 + [0, NI x NS), rows r0 (the thread's first, as in RowA) and r0 + 8
template <int NI, int NS, bool kAnyAct, int kEpi>
__device__ __forceinline__ void seg_epilogue(const WgParams& p, const float (&acc)[NS][NI / 2], int64_t r0, int lane,
                                             int col0) {
  constexpr bool kSum = is_sum(kEpi);
  constexpr bool kOrdered = kEpi == EPI_SEGSUM_ORDERED;
  auto combine = [](float a, float b) { return kSum ? a + b : fmaxf(a, b); };
  const int cq = (lane & 3) * 2;
  // what an edge row contributes to the reduction: the raw accumulator (max), or act(acc) of an accumulator that
  // started at the bias (acc_from_bias), since bias and activation do not commute with a sum
  auto value = [&](int i, int jj, int h, int c) {
    const float a = acc[i][4 * jj + 2 * h + c];
    return kSum ? layer_act<kAnyAct>(p.act, a) : a;
  };
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
  // EPI_SEGSUM_ORDERED: the warp's 16 rows are unit u of the side buffer
  const int64_t u = (r0 - (lane >> 2)) >> 4;
  const bool uniform = __all_sync(0xffffffffu, d[0] == dw && d[1] == dw) && dw >= 0;
  // EPI_SEGMAX: a warp whose every row has the destination of row 0 or that of row 15 (-1 included), as at a run
  // boundary of a grouped edge list, reduce-scatters each of the two in turn with the other's rows masked to
  // -FLT_MAX.  Two passes of L3 flushes each, where the segmented scan below issues 2 x NI x NS / 4 flush instructions
  // after three shuffles per column and half.  Max is exact and each row still reaches a flush of its own destination.
  // One accumulator group only (NS = 1: every GNN edge launch): the 152 x 2 ROWS instance spills with it
  int dz = dw;
  bool two = false;
  if constexpr (kEpi == EPI_SEGMAX && NS == 1) {
    dz = __shfl_sync(0xffffffffu, d[1], 28);
    two = !uniform && __all_sync(0xffffffffu, (d[0] == dw || d[0] == dz) && (d[1] == dw || d[1] == dz));
  }
  if (uniform || two) {
    // the warp's 16 rows are one destination (or two, one pass each).  Value v of a thread is column (v / 2) * 8 +
    // cq + v % 2; the 8 lanes sharing cq (lane bits 4, 3, 2) reduce-scatter their V values in three halving
    // exchanges, after which every lane holds the full maxima (sums) of V / 8 (rounded up or down) of them and all 32
    // lanes flush.  V is padded with -FLT_MAX (0) values to VP, a multiple of 4, so that the first two exchanges
    // halve evenly (V = 38 at NI = 152, NS = 1)
    constexpr int V = NI * NS / 4, VP = (V + 3) / 4 * 4, L1 = VP / 2, L2 = VP / 4, L3 = (L2 + 1) / 2;
#pragma unroll 1
    for (int pass = 0; pass < (two ? 2 : 1); ++pass) {
      const int t = pass ? dz : dw;   // the destination of this pass
      if (t < 0) continue;
      float m[VP];
#pragma unroll
      for (int i = 0; i < NS; ++i)
#pragma unroll
        for (int jj = 0; jj < NI / 8; ++jj)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const float a0 = value(i, jj, 0, c), a1 = value(i, jj, 1, c);
            m[(i * (NI / 8) + jj) * 2 + c] =
                two ? combine(d[0] == t ? a0 : -FLT_MAX, d[1] == t ? a1 : -FLT_MAX) : combine(a0, a1);
          }
#pragma unroll
      for (int v = V; v < VP; ++v) m[v] = kSum ? 0.0f : -FLT_MAX;
      const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4;
      // a lane with the bit set keeps the upper part, its partner the lower; each sends the part it gives up
#pragma unroll
      for (int k = 0; k < L1; ++k) {
        const float keep = b4 ? m[k + L1] : m[k], give = b4 ? m[k] : m[k + L1];
        m[k] = combine(keep, __shfl_xor_sync(0xffffffffu, give, 16));
      }
#pragma unroll
      for (int k = 0; k < L2; ++k) {
        const float keep = b3 ? m[k + L2] : m[k], give = b3 ? m[k] : m[k + L2];
        m[k] = combine(keep, __shfl_xor_sync(0xffffffffu, give, 8));
      }
#pragma unroll
      for (int k = 0; k < L3; ++k) {
        const float up = k + L3 < L2 ? m[k + L3] : m[k];   // L2 odd: the upper part is one value shorter
        const float keep = b2 ? up : m[k], give = b2 ? m[k] : up;
        m[k] = combine(keep, __shfl_xor_sync(0xffffffffu, give, 4));
      }
      const int v0 = (b4 ? L1 : 0) + (b3 ? L2 : 0) + (b2 ? L3 : 0), nv = b2 ? L2 - L3 : L3;
#pragma unroll
      for (int k = 0; k < L3; ++k) {
        const int v = v0 + k, col = col0 + (v >> 1) * 8 + cq + (v & 1);
        if constexpr (kOrdered) {
          if (k < nv && v < V && col < p.n) ordered_row(p, u, 0, dw)[col] = m[k];   // the unit's one run: slot 0
        } else {
          if (k < nv && v < V && col < p.n) seg_flush<kEpi, kAnyAct>(p, t, col, m[k]);
        }
      }
    }
    if (kOrdered && lane == 0 && p.write_ids && col0 == 0) p.part_id[2 * u] = dw;
  } else if constexpr (kOrdered) {
    // each half's runs as in the sum below; then the run that holds row 7 takes the sum of the one that holds row 8
    // when they are one destination (half 0 + half 1).  The run that holds row 0 goes to slot 0, the one that holds
    // row 15 to slot 1 (in this branch they are two runs), every other run is a whole destination and is stored
    bool head[2];
    bool same[2][3];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int up = __shfl_up_sync(0xffffffffu, d[h], 4);
      head[h] = d[h] >= 0 && (lane < 4 || up != d[h]);
      const bool next = __shfl_down_sync(0xffffffffu, d[h], 4) == d[h] && lane + 4 < 32;
      const uint32_t m = __ballot_sync(0xffffffffu, next) >> (lane & ~3);
      same[h][0] = (m & 0x1u) != 0;
      same[h][1] = (m & 0x11u) == 0x11u;
      same[h][2] = (m & 0x1111u) == 0x1111u;
    }
    const int d0 = __shfl_sync(0xffffffffu, d[0], 0), d7 = __shfl_sync(0xffffffffu, d[0], 28);
    const int d8 = __shfl_sync(0xffffffffu, d[1], 0), d15 = __shfl_sync(0xffffffffu, d[1], 28);
    const bool join = d8 >= 0 && d7 == d8;
    // the last run head of each half (-1: none), as a row of the half
    const int last0 = (31 - __clz(__ballot_sync(0xffffffffu, head[0]) & 0x11111111u)) >> 2;
    const int last1 = (31 - __clz(__ballot_sync(0xffffffffu, head[1]) & 0x11111111u)) >> 2;
    const int q = lane >> 2;
    const bool take = join && q == last0;     // this row's half-0 run continues into half 1
    const bool skip = join && q == 0;         // this row's half-1 run was taken by half 0
    float* const to0 = ordered_row(p, u, q == 0 ? 0 : (take && last1 == 0 && d15 >= 0) ? 1 : -1, d[0]);
    float* const to1 = ordered_row(p, u, (q == last1 && d15 >= 0) ? 1 : -1, d[1]);
#pragma unroll
    for (int i = 0; i < NS; ++i)
#pragma unroll
      for (int jj = 0; jj < NI / 8; ++jj)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          // half 1 first, so that one half's sum is live at a time (the any-activation car instance spills otherwise)
          const int col = col0 + i * NI + jj * 8 + cq + c;
          float first1 = 0.0f;   // the sum of the run that holds row 8
#pragma unroll
          for (int h = 1; h >= 0; --h) {
            float m = value(i, jj, h, c);
#pragma unroll
            for (int s = 0; s < 3; ++s) {
              const float o = __shfl_down_sync(0xffffffffu, m, 4 << s);
              if (same[h][s]) m = m + o;
            }
            if (h == 1) {
              first1 = __shfl_sync(0xffffffffu, m, lane & 3);
              if (head[1] && !skip && col < p.n) to1[col] = m;
            } else {
              if (take) m = m + first1;
              if (head[0] && col < p.n) to0[col] = m;
            }
          }
        }
    if (lane == 0 && p.write_ids && col0 == 0) {
      if (d0 >= 0) p.part_id[2 * u] = d0;
      if (d15 >= 0) p.part_id[2 * u + 1] = d15;
    }
  } else {
    // segmented max (sum) down each 8-row half; the first row of every run flushes the run's max (sum).  Column by
    // column, both halves: each accumulator dies once used
    bool head[2];
    bool same[2][3];   // the row 4 << s lanes down joins this row's partial
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int up = __shfl_up_sync(0xffffffffu, d[h], 4);
      head[h] = d[h] >= 0 && (lane < 4 || up != d[h]);
      if (kSum) {
        // every row must reach exactly one flush, even in an edge list not grouped by destination: the rows up to
        // 1 << s further down join only when every row in between has this destination too.  One ballot of "the next
        // row continues this row's run": bit 4 j of m is that flag of the thread's row + j
        const bool next = __shfl_down_sync(0xffffffffu, d[h], 4) == d[h] && lane + 4 < 32;
        const uint32_t m = __ballot_sync(0xffffffffu, next) >> (lane & ~3);
        same[h][0] = (m & 0x1u) != 0;
        same[h][1] = (m & 0x11u) == 0x11u;
        same[h][2] = (m & 0x1111u) == 0x1111u;
      } else {
        // rows of one destination are contiguous, and a row seen twice does not change a max
#pragma unroll
        for (int s = 0; s < 3; ++s)
          same[h][s] = __shfl_down_sync(0xffffffffu, d[h], 4 << s) == d[h] && lane + (4 << s) < 32;
      }
    }
#pragma unroll
    for (int i = 0; i < NS; ++i)
#pragma unroll
      for (int jj = 0; jj < NI / 8; ++jj)
#pragma unroll
        for (int c = 0; c < 2; ++c)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float m = value(i, jj, h, c);
#pragma unroll
            for (int s = 0; s < 3; ++s) {
              const float o = __shfl_down_sync(0xffffffffu, m, 4 << s);
              if (same[h][s]) m = combine(m, o);
            }
            const int col = col0 + i * NI + jj * 8 + cq + c;
            if (head[h] && col < p.n) seg_flush<kEpi, kAnyAct>(p, d[h], col, m);
          }
  }
}

// ---- GNN edge layer: W resident, three independent consumer warpgroups (header, "mapping") -----------------------
// The P gather of one warpgroup, kGnnStages chunks ahead of its wgmmas.  A stage holds the warpgroup's 64 rows of
// one 16-k chunk of P in fp32, 64 B per row.  Lane q of a quad copies the 16-byte piece q of the quad's two rows (g and
// g + 8, RowA's) with cp.async.cg, one commit group per chunk; after its wait and a __syncwarp each lane reads its
// fragment's four 8-byte pairs, written by its own quad.  The 32-byte halves of row r swap places when bit 1 of r is
// set, so a warp's 8-byte reads (8 rows x 32 B) take the minimal two wavefronts.  No warpgroup barrier and no fence.
// The copy cursor runs on from a tile's last chunk into the warpgroup's next tile (empty groups past its last), so
// the next tile's first chunks land while this one finishes and flushes
struct GnnGather {
  uint32_t base;      // the warpgroup's stage 0
  uint32_t wr, rd;    // the thread's piece of row g, and its first pair of row g (k 2 q), within a stage
  int stage = 0;      // the oldest stage: read next, then refilled
  int tile, kc = 0;   // the chunk the next copy fetches
  uint32_t row[2];    // the P rows (source vertices) of the thread's two rows of that tile

  __device__ __forceinline__ void init(uint32_t stages, int warp, int lane) {
    const uint32_t g = uint32_t(warp * 16 + (lane >> 2)), q = uint32_t(lane & 3), swap = ((g >> 1) & 1u) * 32u;
    base = stages;
    wr = g * 64u + (((q >> 1) * 32u) ^ swap) + (q & 1u) * 16u;
    rd = g * 64u + swap + q * 8u;
  }
  __device__ __forceinline__ void rows(const WgParams& p, int warp, int lane) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t r = int64_t(tile) * kGnnTileRows + warp * 16 + (lane >> 2) + 8 * h;
      const int si = r < p.num_rows ? __ldg(p.src + r) : 0;
      row[h] = si >= 0 && si < p.num_src ? uint32_t(si) : 0u;   // out of range: RowA::context sets the error word
    }
  }
  __device__ __forceinline__ void copy(const WgParams& p, int num_tiles, int stride, int warp, int lane) {
    if (tile < num_tiles) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
        cp_async_16(base + uint32_t(stage) * kGnnStageBytes + wr + uint32_t(h) * 512u,
                    p.x + int64_t(row[h]) * p.ldx + kc * 16 + (lane & 3) * 4);
    }
    cp_async_commit();
    stage = stage + 1 == kGnnStages ? 0 : stage + 1;
    if (++kc == p.nchunks) {
      kc = 0;
      tile += stride;
      rows(p, warp, lane);
    }
  }
  // the fp32 inputs of the oldest chunk in flight, as make_frag takes them (q[i]: row i & 1, k half i >> 1).  The
  // __syncwarp after the reads keeps the quad's refill of the stage (copy(), next) behind them
  __device__ __forceinline__ void take(float2 (&q)[4]) const {
    cp_async_wait<kGnnStages - 1>();
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 4; ++i)
      q[i] = lds_f2(base + uint32_t(stage) * kGnnStageBytes + (rd ^ uint32_t(i >> 1) * 32u) + uint32_t(i & 1) * 512u);
    __syncwarp();
  }
};

template <int kEpi, int NI, int NS, bool kAnyAct, int kArith>
__device__ __forceinline__ void wg_gnn_body(const WgParams& p) {
  constexpr int NT = NI * NS;
  constexpr uint32_t kSlice = uint32_t(NI) * 32u;   // one group's part of one plane (hi, lo or FP16) of a 16-k chunk
  constexpr int kPlanes = arith_planes(kArith);
  // [nchunks][planes][NI rows x 16 k], then [warpgroup][stage][64 rows x 16 k] fp32 (GnnGather), then the mbarrier
  extern __shared__ __align__(128) uint8_t smem[];
  const int nk = p.nchunks;
  const uint32_t w_bytes = uint32_t(nk) * kPlanes * kSlice;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + w_bytes + kGnnWarpgroups * kGnnStages * kGnnStageBytes);
  const int tid = threadIdx.x;
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);   // warpgroup, warp-uniform by construction
  const int group = int(blockIdx.x) % NS;
  const int warp = (tid & 127) >> 5, lane = tid & 31;
  const int num_tiles = int(p.num_tiles), stride = kGnnWarpgroups * int(gridDim.x / NS);
  const int first = kGnnWarpgroups * int(blockIdx.x / NS) + wg;
  // the first chunks of P are on their way while W lands
  GnnGather gather;
  gather.init(smem_u32(smem) + w_bytes + uint32_t(wg * kGnnStages) * kGnnStageBytes, warp, lane);
  gather.tile = first;
  gather.rows(p, warp, lane);
#pragma unroll
  for (int s = 0; s < kGnnStages; ++s) gather.copy(p, num_tiles, stride, warp, lane);
  RowA<PROD_GNN, kAnyAct> a;
  a.context(p, int64_t(first) * kGnnTileRows, warp, lane);
  if (tid == 0) {
    mbar_init(full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(full, w_bytes);
    for (int kc = 0; kc < nk; ++kc)
#pragma unroll
      for (int h = 0; h < kPlanes; ++h)
        bulk_g2s(smem + (size_t(kc) * kPlanes + h) * kSlice,
                 p.bimg + size_t(kc) * NT * w_row_bytes(kArith) + size_t(h) * NT * 32 + size_t(group) * kSlice, kSlice,
                 full);
  }
  mbar_wait(full, 0);
  const uint32_t w_base = smem_u32(smem);
  for (int tile = first; tile < num_tiles; tile += stride) {
    const int64_t row0 = int64_t(tile) * kGnnTileRows;
    float acc[1][NI / 2];
    if constexpr (is_sum(kEpi)) acc_from_bias<NI>(p, acc[0], group * NI, lane);
    auto frag = [&](int kc, uint32_t (&hi)[4], uint32_t (&lo)[4]) {
      float2 q[4];
      gather.take(q);
      a.template make_frag<kArith>(p, q, kc, lane, hi, lo);
      gather.copy(p, num_tiles, stride, warp, lane);
    };
    rs_k_loop(nk, frag, [&](int kc, const uint32_t (&hi)[4], const uint32_t (&lo)[4]) {
      wgmma_fence();
      const uint32_t b = w_base + uint32_t(kc) * kPlanes * kSlice;
      const uint64_t b_hi = make_smem_desc(b, 128, 256), b_lo = make_smem_desc(b + kSlice, 128, 256);
      mma_rs<kArith, NI>(acc[0], hi, lo, b_hi, b_lo, kc > 0 || is_sum(kEpi) ? 1 : 0);
      wgmma_commit();
      wgmma_wait<1>();                    // chunk kc - 1 complete: its A fragment is free
    });
    // the next tile's context while the last wgmmas run; its first chunks of P are already in flight
    a.context(p, row0 + int64_t(stride) * kGnnTileRows, warp, lane);
    wgmma_wait<0>();
    seg_epilogue<NI, 1, kAnyAct, kEpi>(p, acc, row0 + warp * 16 + (lane >> 2), lane, group * NI);
  }
}

// ---- dense and pooling layers: W streamed by a producer warpgroup --------------------------------------------------
template <int kProd, int kEpi, int NI, int NS, int kArith>
__device__ __forceinline__ void wg_gemm_body(const WgParams& p) {
  static_assert(kProd != PROD_GNN, "the GNN edge layer runs wg_gnn_body");
  constexpr int NT = NI * NS;
  constexpr uint32_t kChunkBytes = uint32_t(NT) * w_row_bytes(kArith);   // every plane, 16 k
  constexpr uint32_t kABytes = a_chunk_bytes(kArith);
  constexpr int kRing = ring_stages(kChunkBytes, 0);
  // the pooling chain sizes its ring stages and A regions for all of its layers (host side, launch_wg)
  const uint32_t stage_bytes = kProd == PROD_POOL ? p.stage_bytes : kChunkBytes;
  const uint32_t region_bytes = kProd == PROD_POOL ? p.region_bytes : 0;
  const int ring_log2 = kProd == PROD_POOL ? p.ring_log2 : log2_ring(kRing);
  const uint32_t ring_mask = (1u << ring_log2) - 1;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* bring = smem;
  uint8_t* abuf = smem + (stage_bytes << ring_log2);     // [consumer warpgroup][region]
  uint64_t* full = reinterpret_cast<uint64_t*>(abuf + 2 * region_bytes);
  uint64_t* empty = full + ring_mask + 1;
  const int tid = threadIdx.x;
  const int role = __shfl_sync(0xffffffffu, tid >> 7, 0);   // warpgroup, warp-uniform by construction
  if (tid == 0) {
    for (uint32_t s = 0; s <= ring_mask; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);     // lane 0 of each of the 8 consumer warps
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int64_t my_tiles = (p.num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;
  const int nk = p.nchunks;
  const int nl = kProd == PROD_POOL ? p.chain_layers : 0;   // on-chip layers ahead of this one
  if (role == 0) {
    // W producer: one thread streams the CTA's chunks in the order the consumers use them (per tile: the chain's
    // layers, then the kernel's own), refilling a stage as soon as both consumer warpgroups have released it
    setmaxnreg_dec<kProducerRegs>();
    if (tid != 0) return;
    int64_t g = 0;
    for (int64_t j = 0; j < my_tiles; ++j)
      for (int l = 0; l <= nl; ++l) {
        int lk = nk;
        uint32_t bytes = kChunkBytes;
        const uint8_t* img = p.bimg;
        if (l < nl) {
          const int4 c = p.chain[l];
          lk = c.x;
          bytes = uint32_t(c.y >> 2) * uint32_t(c.y & 3) * w_row_bytes(kArith);
          img = p.chain_buf + c.z;
        }
        for (int kc = 0; kc < lk; ++kc, ++g) {
          const uint32_t stage = uint32_t(g) & ring_mask;
          if (g > ring_mask) mbar_wait(&empty[stage], uint32_t(((g >> ring_log2) - 1) & 1));
          mbar_arrive_expect_tx(&full[stage], bytes);
          bulk_g2s(bring + stage * stage_bytes, img + size_t(kc) * bytes, bytes, &full[stage]);
        }
      }
    return;
  }
  setmaxnreg_inc<kConsumerRegs>();
  const int wgi = role - 1, t = tid & 127, warp = t >> 5, lane = tid & 31;
  // chunk g's W stage is free again
  auto release = [&](int64_t g) {
    if (lane == 0) mbar_arrive(&empty[uint32_t(g) & ring_mask]);
  };

  uint8_t* my_a = abuf + wgi * region_bytes;
  int64_t g = 0;
  for (int64_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    // ---- A: the tile's streamed layer sets the rows' context (RowA)
    RowA<kProd, false> a;
    const int64_t row0 = tile * kTileRows + wgi * 64;
    // ---- one layer's loop over 16-k chunks into acc[ns][ni / 2] --------------------------------------
    // streamed: chunk kc + 1's A fragment is built while chunk kc's wgmmas run.  Otherwise the previous on-chip layer
    // left the whole A in the region, chunk kc at kc * kABytes
    // keep: the first chunk accumulates onto lacc (the segment sum's bias) instead of overwriting it
    auto mma_layer = [&](auto& lacc, int lk, bool streamed, bool keep = false) {
      using Acc = std::remove_reference_t<decltype(lacc)>;
      constexpr int ns = int(std::extent<Acc, 0>::value), ni = 2 * int(std::extent<Acc, 1>::value);
      // chunk kc's wgmmas on W stage g, A hi / lo (FP16: hi only) from registers (uint32_t[4]) or shared memory
      // (descriptors).  Every chunk leaves exactly itself in flight: a wait on a path of its own (the last chunk's)
      // would make ptxas drain the wgmmas at the end of every iteration
      auto chunk = [&](int kc, const auto& a_hi, const auto& a_lo) {
        mbar_wait(&full[uint32_t(g) & ring_mask], uint32_t((g >> ring_log2) & 1));
        wgmma_fence();
        const uint32_t b_base = smem_u32(bring + (uint32_t(g) & ring_mask) * stage_bytes);
#pragma unroll
        for (int i = 0; i < ns; ++i) {
          const uint64_t b_hi = make_smem_desc(b_base + uint32_t(i * ni) * 32u, 128, 256);
          const uint64_t b_lo = make_smem_desc(b_base + uint32_t(ni * ns) * 32u + uint32_t(i * ni) * 32u, 128, 256);
          if constexpr (std::is_same_v<std::decay_t<decltype(a_hi)>, uint64_t>)
            mma_ss<kArith, ni>(lacc[i], a_hi, a_lo, b_hi, b_lo, kc > 0 || keep ? 1 : 0);
          else
            mma_rs<kArith, ni>(lacc[i], a_hi, a_lo, b_hi, b_lo, kc > 0 || keep ? 1 : 0);
        }
        wgmma_commit();
        wgmma_wait<1>();                  // chunk kc - 1 complete: its A fragment and W stage are free
        if (kc > 0) release(g - 1);
        ++g;
      };
      if (streamed && kProd != PROD_POOL) {
        // the loads of chunk kc + 1 are issued before chunk kc's wgmmas
        a.context(p, row0, warp, lane);
        float2 q[4];
        a.load(p, 0, lane, q);
        auto frag = [&](int kc, uint32_t (&hi)[4], uint32_t (&lo)[4]) {
          a.template make_frag<kArith>(p, q, kc, lane, hi, lo);
          if (kc + 1 < lk) a.load(p, kc + 1, lane, q);
        };
        rs_k_loop(lk, frag, chunk);
      } else if (streamed) {
        // POOL layer 1: the fragments go through a double buffer at the start of the region, in to_region's layout,
        // and the wgmmas read A from there.  With A in registers next to the on-chip layers' code, ptxas serialises
        // the wgmmas of every POOL instance for want of registers (C7512)
        a.context(p, row0, warp, lane);
        auto put = [&](int kc) {
          float2 q[4] = {};
          uint32_t hi[4], lo[4];
          a.template make_frag<kArith>(p, q, kc, lane, hi, lo);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            uint8_t* dstp = my_a + uint32_t(kc & 1) * kABytes + uint32_t(warp * 2 + (i & 1)) * 256u +
                            uint32_t(i >> 1) * 128u + uint32_t(lane >> 2) * 16u + uint32_t(lane & 3) * 4u;
            *reinterpret_cast<uint32_t*>(dstp) = hi[i];
            if constexpr (kArith != ARITH_F16) *reinterpret_cast<uint32_t*>(dstp + kABytes / 2) = lo[i];
          }
        };
        put(0);
        for (int kc = 0; kc < lk; ++kc) {
          fence_proxy_async_smem();       // this warpgroup's A writes -> visible to its wgmmas
          warpgroup_sync(1 + wgi);
          const uint32_t a_base = smem_u32(my_a + uint32_t(kc & 1) * kABytes);
          chunk(kc, make_smem_desc(a_base, 128, 256), make_smem_desc(a_base + kABytes / 2, 128, 256));
          if (kc + 1 < lk) put(kc + 1);
        }
      } else {
        fence_proxy_async_smem();         // this warpgroup's to_region writes -> visible to its wgmmas
        warpgroup_sync(1 + wgi);
        for (int kc = 0; kc < lk; ++kc) {
          const uint32_t a_base = smem_u32(my_a + uint32_t(kc) * kABytes);
          chunk(kc, make_smem_desc(a_base, 128, 256), make_smem_desc(a_base + kABytes / 2, 128, 256));
        }
      }
      wgmma_wait<0>();
      release(g - 1);
    };
    // ---- on-chip pooling layers: relu(acc + b) split into hi / lo (FP16: rounded once into one plane) over this
    // warpgroup's own (now dead) input in the region, the first kp_next k of the next layer's A.  A lane's pair (row,
    // cols 8 j + cq, + 1) is one 4-byte word of a core matrix: a warp writes 128 contiguous bytes per store, free of
    // bank conflicts
    auto to_region = [&](auto& lacc, const float* bias, int kp_next) {
      using Acc = std::remove_reference_t<decltype(lacc)>;
      constexpr int ns = int(std::extent<Acc, 0>::value), ni = 2 * int(std::extent<Acc, 1>::value);
      const int cq = (lane & 3) * 2;
#pragma unroll
      for (int i = 0; i < ns; ++i)
#pragma unroll
        for (int jj = 0; jj < ni / 8; ++jj) {
          const int col = i * ni + jj * 8 + cq;
          if (i * ni + jj * 8 < kp_next) {
            const float b0 = __ldg(bias + col), b1 = __ldg(bias + col + 1);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float v0 = fmaxf(lacc[i][4 * jj + 2 * h] + b0, 0.0f), v1 = fmaxf(lacc[i][4 * jj + 2 * h + 1] + b1, 0.0f);
              uint8_t* dstp = my_a + uint32_t(col >> 4) * kABytes + uint32_t(warp * 2 + h) * 256u +
                              uint32_t((col >> 3) & 1) * 128u + uint32_t(lane >> 2) * 16u + uint32_t(cq) * 2u;
              if constexpr (kArith == ARITH_F16) {
                *reinterpret_cast<uint32_t*>(dstp) = pack_f16x2(v0, v1);
              } else {
                uint32_t hi, lo;
                split_bf16x2(v0, v1, &hi, &lo);
                *reinterpret_cast<uint32_t*>(dstp) = hi;
                *reinterpret_cast<uint32_t*>(dstp + kABytes / 2) = lo;
              }
            }
          }
        }
    };
    if (kProd == PROD_POOL) {
      for (int l = 0; l < nl; ++l) {
        const int4 c = p.chain[l];
        const float* bias = reinterpret_cast<const float*>(p.chain_buf + c.w);
        const int kp_next = l + 1 < nl ? p.chain[l + 1].x * 16 : p.kp;
        switch (c.y) {
          case 64 * 4 + 1: { float a[1][32] = {}; mma_layer(a, c.x, l == 0); to_region(a, bias, kp_next); } break;
          case 128 * 4 + 1: { float a[1][64] = {}; mma_layer(a, c.x, l == 0); to_region(a, bias, kp_next); } break;
          case 96 * 4 + 2: { float a[2][48] = {}; mma_layer(a, c.x, l == 0); to_region(a, bias, kp_next); } break;
          case 128 * 4 + 2: { float a[2][64] = {}; mma_layer(a, c.x, l == 0); to_region(a, bias, kp_next); } break;
          default: { float a[2][76] = {}; mma_layer(a, c.x, l == 0); to_region(a, bias, kp_next); } break;
        }
      }
    }
    // every accumulator is defined before its layer (the wgmmas read it, if only to scale it by 0): otherwise the
    // values of the previous tile would stay live through the on-chip layers, next to their accumulators
    float acc[NS][NI / 2];
    if (is_sum(kEpi))
#pragma unroll
      for (int i = 0; i < NS; ++i) acc_from_bias<NI>(p, acc[i], i * NI, lane);
    else if (kProd == PROD_POOL)
#pragma unroll
      for (int i = 0; i < NS; ++i)
#pragma unroll
        for (int v = 0; v < NI / 2; ++v) acc[i][v] = 0.0f;
    mma_layer(acc, nk, nl == 0, is_sum(kEpi));
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
      seg_epilogue<NI, NS, false, kEpi>(p, acc, r0, lane, 0);
    }
  }
}

template <int kProd, int kEpi, int NI, int NS, int kArith, bool kAnyAct>
__device__ __forceinline__ void wg_body(const WgParams& p) {
  if constexpr (kProd == PROD_GNN) {
    static_assert(kEpi != EPI_STORE, "the GNN edge layer ends in a segment reduction");
    wg_gnn_body<kEpi, NI, NS, kAnyAct, kArith>(p);
  } else {
    static_assert(!kAnyAct, "any-activation instances: the GNN edge layer only");
    wg_gemm_body<kProd, kEpi, NI, NS, kArith>(p);
  }
}

template <int kProd, int kEpi, int NI, int NS, int kArith, bool kAnyAct>
__global__ void __launch_bounds__(kWgThreads, 1) wg_gemm_kernel(WgParams p) {
  static_assert(!is_sum(kEpi), "the segment-sum instances are wg_segsum_kernel and wg_segsum_ordered_kernel");
  wg_body<kProd, kEpi, NI, NS, kArith, kAnyAct>(p);
}

// The segment sum (EPI_SEGSUM) of the edge layers: wg_gemm_kernel's bodies with the sum epilogue, as a kernel of its
// own so that the max's instances stay exactly the set they were, and the sum's are counted and checked as one family
// (tests/test_aggregation_build_cpu.py)
template <int kProd, int NI, int NS, int kArith, bool kAnyAct>
__global__ void __launch_bounds__(kWgThreads, 1) wg_segsum_kernel(WgParams p) {
  wg_body<kProd, EPI_SEGSUM, NI, NS, kArith, kAnyAct>(p);
}

// The ordered segment sum (EPI_SEGSUM_ORDERED, PG_FLAG_DETERMINISTIC): the same bodies again, under a third name so
// that the atomic sum's family stays exactly the set it was
template <int kProd, int NI, int NS, int kArith, bool kAnyAct>
__global__ void __launch_bounds__(kWgThreads, 1) wg_segsum_ordered_kernel(WgParams p) {
  wg_body<kProd, EPI_SEGSUM_ORDERED, NI, NS, kArith, kAnyAct>(p);
}

// the __global__ instance of a launch: wg_gemm_kernel, or wg_segsum_kernel / wg_segsum_ordered_kernel for the sums
template <int kProd, int kEpi, int NI, int NS, int kArith, bool kAnyAct>
void (*wg_kernel())(WgParams) {
  if constexpr (kEpi == EPI_SEGSUM_ORDERED)
    return wg_segsum_ordered_kernel<kProd, NI, NS, kArith, kAnyAct>;
  else if constexpr (kEpi == EPI_SEGSUM)
    return wg_segsum_kernel<kProd, NI, NS, kArith, kAnyAct>;
  else
    return wg_gemm_kernel<kProd, kEpi, NI, NS, kArith, kAnyAct>;
}

// ---- W [K, N] -> streamed B image ---------------------------------------------------------------
// B operand rows are OUTPUT features (N), K-major, one block per 16-k chunk: its planes ([hi | lo] for BF16x3, one
// FP16 plane), each NT / 8 row groups of two core matrices: element (k, col) at chunk (k / 16), (col / 8) * 256 +
// ((k % 16) / 8) * 128 + (col % 8) * 16 + (k % 8) * 2.  Columns >= n_src and rows >= k are zero.
__global__ void pack_b_kernel(const float* __restrict__ w, int k, int n_src, int ld, int kp, int nt, int arith,
                              uint8_t* __restrict__ img) {
  const int total = kp * nt;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int kk = i / nt, col = i - kk * nt;
    const float v = (col < n_src && kk < k) ? w[int64_t(kk) * ld + col] : 0.0f;
    const size_t off = size_t(kk / 16) * (size_t(nt) * w_row_bytes(arith)) + size_t(col / 8) * 256 +
                       size_t((kk % 16) / 8) * 128 + size_t(col % 8) * 16 + size_t(kk % 8) * 2;
    if (arith == ARITH_F16) {
      // the A operands' rounding: nearest, saturating at +-65504
      *reinterpret_cast<uint16_t*>(img + off) = uint16_t(pack_f16x2(v, 0.0f) & 0xffffu);
      continue;
    }
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
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
  size_t smem;   // a streamed (ROWS) launch's, for the arithmetic wg_shape was given
  bool ok;
};

// N is padded to one of the instruction shapes the kernel is built for (zero weight columns)
WgShape wg_shape(int k, int n, int arith) {
  WgShape t{};
  t.kp = (k + 15) / 16 * 16;
  t.np = (n + 15) / 16 * 16;
  if (t.np <= 64) { t.ni = 64; t.ns = 1; }
  else if (t.np <= 128) { t.ni = 128; t.ns = 1; }
  else if (t.np <= 192) { t.ni = 96; t.ns = 2; }
  else if (t.np <= 256) { t.ni = 128; t.ns = 2; }
  else if (t.np <= kMaxNT) { t.ni = 152; t.ns = 2; }
  t.nt = t.ni * t.ns;
  const uint32_t chunk = uint32_t(t.nt) * w_row_bytes(arith);
  t.smem = wg_smem_bytes(chunk, 0, ring_stages(chunk, 0));
  t.ok = t.nt > 0 && k >= 1 && n >= 1;
  return t;
}

// one weight matrix in the streamed image layout of its arithmetic + its padded bias
struct PreparedGemm {
  WgShape t{};
  int n = 0;
  int arith = ARITH_BF16X3;
  Temp img, bias_pad;
};

int prepare_gemm(PreparedGemm& g, const float* w, int ld, const float* bias, int k, int n, int arith, cudaStream_t s) {
  g.t = wg_shape(k, n, arith);
  g.n = n;
  g.arith = arith;
  PG_REQUIRE(g.t.ok, "no tensor-core shape for a %d x %d layer", k, n);
  PG_CUDA_OK(g.bias_pad.alloc(sizeof(float) * g.t.nt, s));
  pad_rows_kernel<<<2, 256, 0, s>>>(bias, 1, n, g.t.nt, g.bias_pad.as<float>());
  PG_LAUNCH_CHECK();
  PG_CUDA_OK(g.img.alloc(size_t(g.t.kp / 16) * g.t.nt * w_row_bytes(arith), s));
  pack_b_kernel<<<std::min(num_sms(), 64), 256, 0, s>>>(w, k, n, ld, g.t.kp, g.t.nt, arith, g.img.as<uint8_t>());
  PG_LAUNCH_CHECK();
  return PG_OK;
}

// POOL: the on-chip layers ahead of a launch's own layer (layer 1 first), their W images and padded biases packed in
// one buffer once, when the edge layer is prepared
struct PoolChain {
  int layers = 0;
  int4 table[kMaxChain] = {};   // WgParams::chain
  uint32_t max_chunk = 0;       // widest W chunk (bytes) of these layers
  int max_kp = 0;               // widest padded input of these layers after the first (held in the A region)
  Temp buf;
};

// layers 1 .. own - 1 of the pooling MLP as the chain ahead of layer own
int prepare_chain(PoolChain& c, const float* const* weights, const float* const* biases, const int32_t* dims, int own,
                  int arith, cudaStream_t s) {
  c.layers = std::max(0, own - 1);
  PG_REQUIRE(c.layers <= kMaxChain, "pooling chain of %d layers", c.layers);
  if (c.layers == 0) return PG_OK;
  std::vector<WgShape> t(c.layers);
  size_t bytes = 0;
  for (int i = 0; i < c.layers; ++i) {
    t[i] = wg_shape(dims[i + 1], dims[i + 2], arith);
    PG_REQUIRE(t[i].ok, "no tensor-core shape for a %d x %d layer", dims[i + 1], dims[i + 2]);
    c.table[i] = make_int4(t[i].kp / 16, t[i].ni * 4 + t[i].ns, int(bytes), 0);
    bytes += size_t(t[i].kp / 16) * t[i].nt * w_row_bytes(arith);
    c.max_chunk = std::max(c.max_chunk, uint32_t(t[i].nt) * w_row_bytes(arith));
    if (i > 0) c.max_kp = std::max(c.max_kp, t[i].kp);
  }
  for (int i = 0; i < c.layers; ++i) {
    c.table[i].w = int(bytes);
    bytes += sizeof(float) * t[i].nt;
  }
  PG_CUDA_OK(c.buf.alloc(bytes, s));
  for (int i = 0; i < c.layers; ++i) {
    uint8_t* buf = c.buf.as<uint8_t>();
    pack_b_kernel<<<std::min(num_sms(), 64), 256, 0, s>>>(weights[i + 1], dims[i + 1], dims[i + 2], dims[i + 2], t[i].kp,
                                                          t[i].nt, arith, buf + c.table[i].z);
    PG_LAUNCH_CHECK();
    pad_rows_kernel<<<2, 256, 0, s>>>(biases[i + 1], 1, dims[i + 2], t[i].nt, reinterpret_cast<float*>(buf + c.table[i].w));
    PG_LAUNCH_CHECK();
  }
  return PG_OK;
}

template <int kProd, int kEpi, int NI, int NS, int kArith>
int launch_wg_cfg(const WgParams& p, size_t smem, cudaStream_t s) {
  // the GNN edge layer with an activation other than ReLU runs the any-activation instance; everything else is ReLU
  // or linear
  void (*kernel)(WgParams) = wg_kernel<kProd, kEpi, NI, NS, kArith, false>();
  bool any_act = false;
  if constexpr (kProd == PROD_GNN) {
    any_act = p.act != PG_ACT_RELU;
    if (any_act) kernel = wg_kernel<kProd, kEpi, NI, NS, kArith, true>();
  }
  static bool attr_done[2] = {false, false};
  if (!attr_done[any_act]) {
    // a pooling chain's footprint depends on its layers, a GNN launch's on its K, not only on the instance
    PG_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    int(kProd == PROD_ROWS && smem < 48 * 1024 ? 48 * 1024 : 227 * 1024)));
    attr_done[any_act] = true;
  }
  int grid = int(std::min<int64_t>(p.num_tiles, num_sms()));
  // GNN: one CTA per column group and slot, each slot taking kGnnWarpgroups tiles at a time: the largest multiple of
  // NS up to the SM count, and no more slots than the tiles need
  if constexpr (kProd == PROD_GNN)
    grid = int(std::min<int64_t>(num_sms() / NS, ceil_div(p.num_tiles, kGnnWarpgroups))) * NS;
  kernel<<<grid, kWgThreads, smem, s>>>(p);
  PG_LAUNCH_CHECK();
  g_tc_launches[kEpi == EPI_STORE ? 1 : 0].fetch_add(1, std::memory_order_relaxed);
  return PG_OK;
}

// the instance of g's instruction shape
template <int kProd, int kEpi, int kArith>
int launch_wg_shape(const WgParams& p, const PreparedGemm& g, size_t smem, cudaStream_t s) {
  switch (g.t.ni * 4 + g.t.ns) {
    case 64 * 4 + 1: return launch_wg_cfg<kProd, kEpi, 64, 1, kArith>(p, smem, s);
    case 128 * 4 + 1: return launch_wg_cfg<kProd, kEpi, 128, 1, kArith>(p, smem, s);
    case 96 * 4 + 2: return launch_wg_cfg<kProd, kEpi, 96, 2, kArith>(p, smem, s);
    case 128 * 4 + 2: return launch_wg_cfg<kProd, kEpi, 128, 2, kArith>(p, smem, s);
    case 152 * 4 + 2: return launch_wg_cfg<kProd, kEpi, 152, 2, kArith>(p, smem, s);
    default: break;
  }
  PG_REQUIRE(false, "tensor-core kernel: no instance for N = %d", g.t.nt);
  return PG_OK;
}

// POOL launches run the chain's layers ahead of g (none without a chain)
template <int kProd, int kEpi>
int launch_wg(WgParams p, const PreparedGemm& g, cudaStream_t s, const PoolChain* chain = nullptr) {
  if (p.num_rows == 0) return PG_OK;
  p.kp = g.t.kp;
  p.nchunks = g.t.kp / 16;
  p.bimg = g.img.as<uint8_t>();
  p.bias = g.bias_pad.as<float>();
  p.n = g.n;
  p.num_tiles = ceil_div(p.num_rows, kTileRows);
  size_t smem = g.t.smem;
  if (kProd == PROD_POOL) {
    // ring stages hold the widest chunk of any layer; a warpgroup's A region holds layer 1's double buffer and the
    // widest activation the chain keeps on chip (the input of every later layer, up to g's own)
    const uint32_t a_bytes = a_chunk_bytes(g.arith);
    p.chain_layers = chain ? chain->layers : 0;
    p.stage_bytes = uint32_t(g.t.nt) * w_row_bytes(g.arith);
    p.region_bytes = 2 * a_bytes;
    if (p.chain_layers > 0) {
      std::copy(chain->table, chain->table + kMaxChain, p.chain);
      p.chain_buf = chain->buf.as<uint8_t>();
      p.stage_bytes = std::max(p.stage_bytes, chain->max_chunk);
      p.region_bytes = std::max(p.region_bytes, uint32_t(std::max(chain->max_kp, g.t.kp) / 16) * a_bytes);
    }
    const int ring = ring_stages(p.stage_bytes, p.region_bytes);
    p.ring_log2 = log2_ring(ring);
    smem = wg_smem_bytes(p.stage_bytes, p.region_bytes, ring);
  }
  if (kProd == PROD_GNN) {
    p.num_tiles = ceil_div(p.num_rows, kGnnTileRows);
    smem = gnn_smem_bytes(g.t.kp, g.t.ni, g.arith);
  }
  PG_REQUIRE(smem <= 227 * 1024, "tensor-core kernel needs %zu B of shared memory", smem);
  if (g.arith == ARITH_F16) return launch_wg_shape<kProd, kEpi, ARITH_F16>(p, g, smem, s);
  return launch_wg_shape<kProd, kEpi, ARITH_BF16X3>(p, g, smem, s);
}

// column blocks of at most max_w (multiples of 16) covering n
std::vector<int> column_blocks(int n, int max_w = kMaxNT) {
  std::vector<int> c0;
  const int nb = int(ceil_div(n, max_w));
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

// W [k, n] with row stride ld as tensor-core GEMMs of at most max_w output features, block b writing the columns
// from col0[b]; only the first n_src columns of W are read, the pad columns past them get zero weights and bias
int prepare_column_blocks(std::vector<PreparedGemm>& blocks, std::vector<int>& col0, const float* w, int ld,
                          const float* bias, int k, int n_src, int n, int arith, cudaStream_t s, int max_w = kMaxNT) {
  PG_REQUIRE(n >= 1, "no tensor-core shape for a %d x %d layer", k, n);
  col0 = column_blocks(n, max_w);
  blocks = std::vector<PreparedGemm>(col0.size());
  for (size_t b = 0; b < col0.size(); ++b) {
    const int wn = (b + 1 < col0.size() ? col0[b + 1] : n) - col0[b];
    const int src_cols = std::max(0, std::min(wn, n_src - col0[b]));
    PG_REQUIRE(src_cols > 0, "dense layer: column block beyond the weight matrix");
    if (int rc = prepare_gemm(blocks[b], w + col0[b], ld, bias + col0[b], k, src_cols, arith, s)) return rc;
    blocks[b].n = wn;
  }
  return PG_OK;
}

// whether every column block of at most max_w of an n-wide GNN edge layer keeps its column group of W resident in
// shared memory at padded K kp in the arithmetic arith
bool gnn_w_resident(int kp, int n, int max_w, int arith) {
  const std::vector<int> c0 = column_blocks(n, max_w);
  for (size_t b = 0; b < c0.size(); ++b) {
    const WgShape t = wg_shape(kp, (b + 1 < c0.size() ? c0[b + 1] : n) - c0[b], arith);
    if (gnn_smem_bytes(t.kp, t.ni, arith) > 227 * 1024) return false;
  }
  return true;
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
               int arith, cudaStream_t s) {
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
  return prepare_column_blocks(f.blocks, f.col0, w, ld_src, bias, k, n_src, n, arith, s);
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
  if (act != PG_ACT_NONE && act != PG_ACT_RELU) {
    // the GEMM linear, then the activation and the residual in one pass over the output
    if (int rc = apply_fc(f, x, m, PG_ACT_NONE, nullptr, out, ldo, s)) return rc;
    return activate_rows(out, m, f.n, ldo, nullptr, act, residual, f.n, false, s);
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
  int act = PG_ACT_RELU;              // after every layer of the edge MLP
  std::vector<int32_t> dims;
  std::vector<const float*> w, b;     // caller's tensors (must outlive the handle)
  // GNN: hoisted first layer P = F @ W1[:C] + b1 (zero padded to kp columns) and W1[C:]
  PreparedFc p_fc;
  int kp = 0;
  // GNN: W1[C:] as [3, kp];  POOL: W0 [4, kp] + b0 [kp]
  Temp w1x;
  // the per-edge layers: GNN - W2 in column blocks;  POOL - layers 1 .. L-1, the last one in column blocks
  std::vector<PreparedGemm> last;     // the segment-max layer, column blocks
  std::vector<int> last_col0;
  // POOL: one launch runs layers 1 .. chain_end per edge tile, every activation on chip: layers 1 .. chain_end - 1
  // as its chain, then layer chain_end.  chain_end = L - 1 (the segment-max launch) unless the last layer is wider
  // than one launch and L > 2; then chain_end = L - 2, whose output is stored per edge for the column blocks
  int chain_end = 0;
  PoolChain chain;
  PreparedGemm chain_store;           // layer L - 2 when chain_end = L - 2
};

int prepare_edge(PreparedEdge& e, int mode, int c_in, const float* const* weights, const float* const* biases,
                 const int32_t* dims, int num_layers, int act, bool want_tc, int arith, cudaStream_t s) {
  PG_REQUIRE(num_layers >= 1 && num_layers <= 8, "edge MLP depth %d not in [1, 8]", num_layers);
  PG_REQUIRE(dims[0] == c_in + 3, "dims[0]=%d must equal feature channels + 3 = %d", dims[0], c_in + 3);
  PG_REQUIRE(act >= 0 && act < PG_ACT_COUNT, "edge MLP: unknown activation");
  e.mode = mode;
  e.act = act;
  e.c_in = c_in;
  e.num_layers = num_layers;
  e.dims.assign(dims, dims + num_layers + 1);
  e.w.assign(weights, weights + num_layers);
  e.b.assign(biases, biases + num_layers);
  for (int l = 0; l < num_layers; ++l) PG_REQUIRE(weights[l] && biases[l], "null weight/bias for layer %d", l);
  e.path = EDGE_FP32;
  if (!want_tc || num_layers < 2) return PG_OK;
  if (mode == PG_EDGE_POOL) {
    // the on-chip chain is built for ReLU: any-activation instances of it inline the activation at hundreds of
    // sites and took ptxas minutes each, so other activations run the fp32 edge kernel
    if (act != PG_ACT_RELU) return PG_OK;
    // PointSetPooling (one feature channel): layer 0 in fp32 inside the producer of layer 1, the following layers
    // chained on chip (PoolChain), the last one ending in the segment max
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
    const int n = dims[num_layers];
    e.chain_end = (n <= kMaxNT || num_layers == 2) ? num_layers - 1 : num_layers - 2;
    if (int rc = prepare_chain(e.chain, weights, biases, dims, e.chain_end, arith, s)) return rc;
    if (e.chain_end < num_layers - 1) {
      const int l = e.chain_end;
      if (int rc = prepare_gemm(e.chain_store, weights[l], dims[l + 1], biases[l], dims[l], dims[l + 1], arith, s))
        return rc;
    }
    if (int rc = prepare_column_blocks(e.last, e.last_col0, weights[num_layers - 1], n, biases[num_layers - 1],
                                       dims[num_layers - 1], n, n, arith, s))
      return rc;
    e.path = EDGE_POOL;
    return PG_OK;
  }
  if (num_layers != 2) return PG_OK;
  const int d1 = dims[1], n = dims[2];
  e.kp = (d1 + 15) / 16 * 16;
  // the edge kernel keeps a column group of W2 resident in shared memory: a hidden layer too wide for the groups of
  // the usual column blocks (kp > 352 at 152 columns) runs as 64-wide blocks (up to kp = 848), a wider one on the fp32
  // edge kernel
  int max_w = kMaxNT;
  if (!gnn_w_resident(e.kp, n, max_w, arith)) max_w = 64;
  if (!gnn_w_resident(e.kp, n, max_w, arith)) return PG_OK;
  // hoisted first layer on the tensor cores too: logical N = kp, the pad columns get zero weights and bias
  if (int rc = prepare_fc(e.p_fc, weights[0], d1, biases[0], c_in, d1, e.kp, true, arith, s)) return rc;
  if (!e.p_fc.tc) {   // FFMA fallback writes the zero padding itself (ldo = kp)
    e.p_fc.n = d1;
    PG_REQUIRE(e.kp <= (d1 + 63) / 64 * 64, "hoisted layer: padded width %d too far from %d", e.kp, d1);
  }
  PG_CUDA_OK(e.w1x.alloc(sizeof(float) * 3 * e.kp, s));
  pad_rows_kernel<<<4, 256, 0, s>>>(weights[0] + int64_t(c_in) * d1, 3, d1, e.kp, e.w1x.as<float>());
  PG_LAUNCH_CHECK();
  if (int rc = prepare_column_blocks(e.last, e.last_col0, weights[1], n, biases[1], d1, n, n, arith, s, max_w)) return rc;
  e.path = EDGE_GNN;
  return PG_OK;
}

// the ordered segment sum (pg_common.cuh) over all column blocks: kOrderedSlice edges at a time (a multiple of every
// tile), each slice's launches writing their columns of one side buffer (the first block its ids), then its fix-up
template <int kProd>
int apply_last_ordered(const PreparedEdge& e, const WgParams& p, int n, float* out, cudaStream_t s) {
  OrderedParts parts;
  if (int rc = parts.alloc(ceil_div(std::min(p.num_rows, kOrderedSlice), 16), n, s)) return rc;
  for (int64_t e0 = 0; e0 < p.num_rows; e0 += kOrderedSlice) {
    if (e0 > 0)
      if (int rc = parts.reset(s)) return rc;
    WgParams q = p;
    q.num_rows = std::min(kOrderedSlice, p.num_rows - e0);
    q.dst = p.dst + e0;
    if (kProd == PROD_ROWS)
      q.x = p.x + e0 * p.ldx;   // the stored per-edge rows (GNN: x is the per-vertex table P)
    else
      q.src = p.src + e0;
    q.part_id = parts.i();
    q.ldp = n;
    for (size_t b = 0; b < e.last.size(); ++b) {
      q.out = out + e.last_col0[b];
      q.ldo = n;
      q.part = parts.v() + e.last_col0[b];
      q.write_ids = b == 0;
      if (int rc = launch_wg<kProd, EPI_SEGSUM_ORDERED>(q, e.last[b], s, &e.chain)) return rc;
    }
    if (int rc = ordered_fixup(parts, out, n, s)) return rc;
  }
  return PG_OK;
}

// the segment-reduction layer over all column blocks: the max (agg PG_AGG_MAX) or the sum, in a fixed order when
// ordered; p carries the producer's inputs
template <int kProd>
int apply_last(const PreparedEdge& e, WgParams p, int n, int agg, bool ordered, float* out, cudaStream_t s) {
  if (agg != PG_AGG_MAX && ordered) return apply_last_ordered<kProd>(e, p, n, out, s);
  for (size_t b = 0; b < e.last.size(); ++b) {
    p.out = out + e.last_col0[b];
    p.ldo = n;
    const int rc = agg == PG_AGG_MAX ? launch_wg<kProd, EPI_SEGMAX>(p, e.last[b], s, &e.chain)
                                     : launch_wg<kProd, EPI_SEGSUM>(p, e.last[b], s, &e.chain);
    if (rc) return rc;
  }
  return PG_OK;
}

// the launches of one edge call: the segment max (sum, ordered or not) into out (pre-filled with -FLT_MAX or 0); an
// out-of-range src / dst sets *err
int launch_edge(const PreparedEdge& e, const float* features, const float* xyz_src, const float* xyz_dst,
                const int32_t* dst_index, const int32_t* src, const int32_t* dst, int64_t num_edges, int64_t num_src,
                int64_t num_dst, int agg, bool ordered, float* out, int* err, cudaStream_t s) {
  const int n = e.dims[e.num_layers];
  if (e.path == EDGE_FP32 || num_edges == 0)
    return edge_mlp_max_fp32(e.mode, features, e.c_in, xyz_src, xyz_dst, dst_index, src, dst, num_edges, num_src, num_dst,
                             e.w.data(), e.b.data(), e.dims.data(), e.num_layers, e.act, agg, ordered, out, err, s);
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
    p.ldx = e.kp;
    p.src = src;
    p.dst = dst;
    p.num_rows = num_edges;
    if (e.chain_end == L - 1) return apply_last<PROD_POOL>(e, p, n, agg, ordered, out, s);
    // the last layer is wider than one launch: the chain stores its input once, and its column blocks read it back.
    // The stored rows are bounded by slicing the edge list (a destination whose edges straddle two slices is merged
    // by the atomic max like any tile boundary)
    const int k_last = e.dims[L - 1];
    const int64_t slice = std::min<int64_t>(num_edges, int64_t(1) << 20);
    Temp h;
    PG_CUDA_OK(h.alloc(sizeof(float) * slice * k_last, s));
    for (int64_t e0 = 0; e0 < num_edges; e0 += slice) {
      const int64_t ne = std::min(slice, num_edges - e0);
      WgParams q = p;
      q.src = src + e0;
      q.dst = dst + e0;
      q.num_rows = ne;
      q.out = h.as<float>();
      q.ldo = k_last;
      q.act = 1;
      if (int rc = launch_wg<PROD_POOL, EPI_STORE>(q, e.chain_store, s, &e.chain)) return rc;
      WgParams r{};
      r.x = h.as<float>();
      r.ldx = k_last;
      r.k_real = k_last;
      r.num_rows = ne;
      r.dst = dst + e0;
      r.num_dst = num_dst;
      r.err = err;
      if (int rc = apply_last<PROD_ROWS>(e, r, n, agg, ordered, out, s)) return rc;
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
  p.act = e.act;
  return apply_last<PROD_GNN>(e, p, n, agg, ordered, out, s);
}

// one edge call on either route: the error word, the fill of out (-FLT_MAX for the max, 0 for the sum and the mean),
// the launches, the division of the mean, and the read-back of the error word unless the caller vouched for the
// indices (trusted: no read-back, no synchronisation).  ordered (PG_FLAG_DETERMINISTIC): the sum and the mean in a
// fixed order; the max ignores it
int apply_edge(const PreparedEdge& e, const float* features, const float* xyz_src, const float* xyz_dst,
               const int32_t* dst_index, const int32_t* src, const int32_t* dst, int64_t num_edges, int64_t num_src,
               int64_t num_dst, bool trusted, int agg, bool ordered, float* out, cudaStream_t s) {
  const int n = e.dims[e.num_layers];
  ErrorWord err;
  if (int rc = err.init(s)) return rc;
  if (int rc = fill_async(out, num_dst * n, agg == PG_AGG_MAX ? -FLT_MAX : 0.0f, s)) return rc;
  // the ordered sum stores each destination that lies inside one unit, so it needs every destination's edges adjacent:
  // it runs on the edge list stable-sorted by dst (the same list for one in CSR order; out-of-range dst last, still
  // reported)
  ordered = ordered && agg != PG_AGG_MAX && num_edges > 0;
  Temp src_s, dst_s;
  if (ordered) {
    if (int rc = sort_edges_by_dst(src, dst, num_edges, num_dst, src_s, dst_s, s)) return rc;
    src = src_s.as<int32_t>();
    dst = dst_s.as<int32_t>();
  }
  if (int rc = launch_edge(e, features, xyz_src, xyz_dst, dst_index, src, dst, num_edges, num_src, num_dst, agg, ordered,
                           out, err.ptr(), s))
    return rc;
  // the any-activation wg_gemm_kernel left the raw maxima: the last layer's bias and activation, once per element
  if (agg == PG_AGG_MAX && e.path != EDGE_FP32 && e.act != PG_ACT_RELU && num_edges > 0)
    if (int rc = activate_rows(out, num_dst, n, n, e.b[e.num_layers - 1], e.act, nullptr, 0, true, s)) return rc;
  if (agg == PG_AGG_MEAN)
    if (int rc = divide_by_segment_count(out, num_dst, n, dst, num_edges, s)) return rc;
  int h = 0;
  if (int rc = err.read(&h, trusted, s)) return rc;
  PG_REQUIRE(h == 0, "edge index out of range (src in [0,%lld), dst in [0,%lld))", (long long)num_src,
             (long long)num_dst);
  return PG_OK;
}

// ---- the class-aware predictor heads (gnn.py:133-163) ---------------------------------------------
// After the concatenated first layers (one GEMM: [D] -> H * (C + 1), act) everything left is tiny per vertex:
// cls H -> C (linear), and per class H -> H (act) -> box_len (linear).  One SIMT kernel does all of it for a
// tile of 32 vertices with every head weight resident in shared memory, and writes logits, class
// probabilities (softmax, models.py:165-168) and the stacked box encodings [K, C, box_len].
constexpr int kHeadRows = 64;     // vertices per tile
constexpr int kHeadThreads = 256; // thread = (row = tid / 4, quarter = tid % 4): 16 of the 64 second-layer outputs of its row
constexpr int kHeadH = 64;        // hidden width the kernel is built for (models.py:60-64 classaware_predictor)

struct HeadsParams {
  const float* hid;      // [m, htot] = act(first layers), columns: cls hidden [H] then class c hidden [H] ...
  int64_t m;
  int htot, C, box;
  const float* wpack;    // [Wcls H*C | bcls C | per class: W2 H*H | b2 H | W3 H*box | b3 box], sections padded to 4 floats
  int wfloats;
  float* logits;         // [m, C]
  float* probs;          // [m, C] or null
  float* boxes;          // [m, C, box]
  int act;               // PG_ACT_* of the hidden layers (kAnyAct; otherwise ReLU)
};

template <bool kAnyAct>
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
      for (int j = 0; j < 16; ++j) h2[r * XS + qd * 16 + j] = layer_act<kAnyAct>(p.act, acc[j]);
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
  int act = PG_ACT_RELU;                   // of the hidden layers; the logits and box layers are linear
  bool fused = false;
  // fused route: the concatenated first layers on the tensor cores, then predictor_heads_kernel
  Temp wcat, bcat, wpack;                  // [D, htot] concatenated first layers, [htot], head weights
  std::vector<PreparedFc> first;           // column groups of the concatenated first layer (<= 256 wide each)
  std::vector<int> col0;
  int wfloats = 0;
  size_t smem = 0;
  // per-layer route: every layer prepared on its own
  std::vector<PreparedFc> layers;
  Temp wsep;                               // separated predictor, per-layer route: the C zero-padded [D, H] loc fc0
};

// dims = {D, H, C, box_len}; layers = cls fc0, cls fc1, then per class c: fc0, fc1, fc2.
// separated (ClassAwareSeparatedPredictor): loc fc0 of class c is [D/C, H] on feature columns [c D/C, (c+1) D/C).
// It is packed as the [D, H] weight that is zero outside those rows, so both routes run the shared predictor's
// kernels on the same GEMM shapes.
int prepare_predictor(PreparedPredictor& P, const float* const* weights, const float* const* biases,
                      const int32_t* dims, int num_layers, int act, bool separated, bool want_tc, int arith,
                      cudaStream_t s) {
  P.act = act;
  P.D = dims[0];
  P.H = dims[1];
  P.C = dims[2];
  P.box = dims[3];
  PG_REQUIRE(num_layers == 2 + 3 * P.C && P.C >= 1 && P.C <= 16 && P.H >= 1 && P.box >= 1,
             "pg_layer_create: predictor needs 2 + 3 C layers, 1 <= C <= 16");
  PG_REQUIRE(!separated || P.D % P.C == 0,
             "pg_layer_create: separated predictor: D = %d features do not split into C = %d equal slices", P.D, P.C);
  const int slice = separated ? P.D / P.C : P.D;   // rows of a loc fc0
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
    // concatenated first layers: column block h = 0 is the cls head, h = 1 + c the loc head of class c (separated:
    // rows [c slice, (c+1) slice) of it, the rest zero)
    if (separated) PG_CUDA_OK(cudaMemsetAsync(P.wcat.ptr, 0, sizeof(float) * size_t(P.D) * P.htot, s));
    for (int h = 0; h <= P.C; ++h) {
      const int l = h == 0 ? 0 : 2 + 3 * (h - 1);
      const int rows = h == 0 ? P.D : slice, row0 = (h > 0 && separated) ? (h - 1) * slice : 0;
      copy_block_kernel<<<32, 256, 0, s>>>(weights[l], rows, P.H, P.htot,
                                           P.wcat.as<float>() + size_t(row0) * P.htot + h * P.H);
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
                              nh * P.H, nh * P.H, want_tc, arith, s))
        return rc;
      if (!P.first.back().tc) P.fused = false;   // FFMA kernel needs contiguous weights: per-layer route
    }
  }
  if (P.fused) return PG_OK;
  P.first.clear();
  if (separated) {
    const size_t dh = size_t(P.D) * P.H;
    PG_CUDA_OK(P.wsep.alloc(sizeof(float) * dh * P.C, s));
    PG_CUDA_OK(cudaMemsetAsync(P.wsep.ptr, 0, sizeof(float) * dh * P.C, s));
    for (int c = 0; c < P.C; ++c) {
      copy_block_kernel<<<32, 256, 0, s>>>(weights[2 + 3 * c], slice, P.H, P.H,
                                           P.wsep.as<float>() + dh * c + size_t(c) * slice * P.H);
      PG_LAUNCH_CHECK();
    }
  }
  P.layers.resize(num_layers);
  for (int l = 0; l < num_layers; ++l) {
    const int pos = l < 2 ? l : (l - 2) % 3;
    const int k = pos == 0 ? P.D : P.H;
    const int n = l == 1 ? P.C : (l >= 2 && pos == 2 ? P.box : P.H);
    const float* w = (separated && l >= 2 && pos == 0) ? P.wsep.as<float>() + size_t(P.D) * P.H * ((l - 2) / 3)
                                                       : weights[l];
    if (int rc = prepare_fc(P.layers[l], w, n, biases[l], k, n, n, want_tc, arith, s)) return rc;
  }
  return PG_OK;
}

// the tensor-core arithmetic of a precision code (1 BF16x3, 2 FP16); code 0 never reaches the tensor cores
int arith_of(int precision) { return precision == 2 ? ARITH_F16 : ARITH_BF16X3; }

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
  PG_REQUIRE(act >= 0 && act < PG_ACT_COUNT, "pg_fully_connected: unknown activation %d", act);
  if (m == 0) return PG_OK;
  PG_REQUIRE(x && w && bias && out, "pg_fully_connected: null argument");
  PG_REQUIRE(precision >= 0 && precision <= 2, "pg_fully_connected: unknown precision %d", precision);
  PreparedFc f;
  if (int rc = prepare_fc(f, w, n, bias, k, n, n, precision != 0 && pg_tc_available(), arith_of(precision), s)) return rc;
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
  const bool ordered = (precision & PG_FLAG_DETERMINISTIC) != 0;
  const int act = activation_of(precision);
  PG_REQUIRE(act >= 0, "pg_edge_mlp_max: unknown activation");
  const int agg = aggregation_of(precision);
  PG_REQUIRE(agg >= 0, "pg_edge_mlp_max: unknown aggregation");
  precision &= PG_PRECISION_MASK;
  PG_REQUIRE(precision >= 0 && precision <= 2, "pg_edge_mlp_max: unknown precision %d", precision);
  PreparedEdge e;
  if (int rc = prepare_edge(e, mode, num_feature_channels, weights_host, biases_host, dims_host, num_layers, act,
                            precision != 0 && num_edges > 0 && pg_tc_available(), arith_of(precision), s))
    return rc;
  return apply_edge(e, features, xyz_src, xyz_dst, dst_index, src, dst, num_edges, num_src, num_dst, trusted, agg,
                    ordered, out, s);
}

// ---------------------------------------------------------------------------------------------------
// pg_layer: prepared layers behind the C ABI
// ---------------------------------------------------------------------------------------------------
struct pg_layer {
  int kind = 0, num_layers = 0;
  int act = PG_ACT_RELU;
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
  const int act = activation_of(precision);
  PG_REQUIRE(act >= 0, "pg_layer_create: unknown activation");
  const bool separated = (precision & PG_FLAG_SEPARATED) != 0;
  PG_REQUIRE(!(precision & PG_FLAG_DETERMINISTIC),
             "pg_layer_create: PG_FLAG_DETERMINISTIC is a flag of the edge calls (the aggregation is chosen per call)");
  precision &= ~(PG_FLAG_ACTIVATION | PG_ACT_MASK | PG_FLAG_SEPARATED);
  PG_REQUIRE(precision >= 0 && precision <= 2, "pg_layer_create: unknown precision %d", precision);
  PG_REQUIRE(kind == PG_LAYER_MLP || kind == PG_LAYER_EDGE_POOL || kind == PG_LAYER_EDGE_GNN || kind == PG_LAYER_PREDICTOR,
             "pg_layer_create: unknown kind %d", kind);
  PG_REQUIRE(!separated || kind == PG_LAYER_PREDICTOR, "pg_layer_create: PG_FLAG_SEPARATED is a predictor flag");
  for (int l = 0; l < num_layers; ++l) PG_REQUIRE(weights_host[l] && biases_host[l], "pg_layer_create: null weight/bias %d", l);
  auto L = std::make_unique<pg_layer>();
  L->kind = kind;
  L->num_layers = num_layers;
  L->act = act;
  const bool want_tc = precision != 0 && pg_tc_available();
  const int arith = arith_of(precision);
  if (kind == PG_LAYER_MLP) {
    L->dims.assign(dims_host, dims_host + num_layers + 1);
    L->fcs.resize(num_layers);
    for (int l = 0; l < num_layers; ++l)
      if (int rc = prepare_fc(L->fcs[l], weights_host[l], dims_host[l + 1], biases_host[l], dims_host[l],
                              dims_host[l + 1], dims_host[l + 1], want_tc, arith, s))
        return rc;
  } else if (kind == PG_LAYER_EDGE_POOL || kind == PG_LAYER_EDGE_GNN) {
    L->dims.assign(dims_host, dims_host + num_layers + 1);
    if (int rc = prepare_edge(L->edge, kind == PG_LAYER_EDGE_POOL ? PG_EDGE_POOL : PG_EDGE_GNN, dims_host[0] - 3,
                              weights_host, biases_host, dims_host, num_layers, act, want_tc, arith, s))
      return rc;
  } else {
    L->dims.assign(dims_host, dims_host + 4);
    if (int rc = prepare_predictor(L->pred, weights_host, biases_host, dims_host, num_layers, act, separated, want_tc,
                                   arith, s))
      return rc;
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
    const int act = (last && last_linear) ? PG_ACT_NONE : layer->act;
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
  const int agg = aggregation_of(flags);
  PG_REQUIRE(agg >= 0, "pg_layer_edge_mlp_max: unknown aggregation");
  return apply_edge(layer->edge, features, xyz_src, xyz_dst, dst_index, src, dst, num_edges, num_src, num_dst,
                    (flags & PG_FLAG_TRUSTED_INDICES) != 0, agg, (flags & PG_FLAG_DETERMINISTIC) != 0, out, s);
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
      if (int rc = apply_fc(P.first[g], x, m, P.act, nullptr, hid.as<float>() + P.col0[g], P.htot, s)) return rc;
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
    hp.act = P.act;
    const bool any_act = P.act != PG_ACT_RELU;
    void (*kernel)(HeadsParams) = any_act ? predictor_heads_kernel<true> : predictor_heads_kernel<false>;
    static bool attr_done[2] = {false, false};
    if (!attr_done[any_act]) {
      PG_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      attr_done[any_act] = true;
    }
    const int blocks = int(std::min<int64_t>(ceil_div(m, kHeadRows), num_sms()));
    kernel<<<blocks, kHeadThreads, P.smem, s>>>(hp);
    PG_LAUNCH_CHECK();
    return PG_OK;
  }
  // per-layer route
  Temp h1, h2, tmp;
  PG_CUDA_OK(h1.alloc(sizeof(float) * m * P.H, s));
  PG_CUDA_OK(h2.alloc(sizeof(float) * m * P.H, s));
  PG_CUDA_OK(tmp.alloc(sizeof(float) * m * P.box, s));
  if (int rc = apply_fc(P.layers[0], x, m, P.act, nullptr, h1.as<float>(), P.H, s)) return rc;
  if (int rc = apply_fc(P.layers[1], h1.as<float>(), m, 0, nullptr, logits, P.C, s)) return rc;
  if (probs != nullptr)
    if (int rc = pg_softmax_rows(logits, m, P.C, probs, stream)) return rc;
  for (int c = 0; c < P.C; ++c) {
    const int l = 2 + 3 * c;
    if (int rc = apply_fc(P.layers[l], x, m, P.act, nullptr, h1.as<float>(), P.H, s)) return rc;
    if (int rc = apply_fc(P.layers[l + 1], h1.as<float>(), m, P.act, nullptr, h2.as<float>(), P.H, s)) return rc;
    if (int rc = apply_fc(P.layers[l + 2], h2.as<float>(), m, 0, nullptr, tmp.as<float>(), P.box, s)) return rc;
    copy_block_kernel<<<64, 256, 0, s>>>(tmp.as<float>(), m, P.box, P.C * P.box, boxes + c * P.box);
    PG_LAUNCH_CHECK();
  }
  return PG_OK;
}
