// The per-pixel rule and the fixed-order fp64 sums of the flow-consistency kernels: dvd_pair_consistency (depth_metrics.cu)
// and dvd_pair_consistency_sf (tracks.cu) run the same device code, so that a zero scene flow gives the same bits in both.
//
// Per-pixel arithmetic is fp64 with every operation rounded on its own (__dmul_rn, __dadd_rn, ...: no contraction), in the
// operation order include/dvd_b200.h states. Sums run in a fixed order: each thread adds its pixels in index order, a block
// adds its threads with a fixed shuffle tree and its warps in order, and reduce_partials_kernel adds a segment's block
// partials in block order. The number of blocks per segment depends on H * W alone.
#pragma once
#include <math.h>

#include "common.cuh"

namespace dvd {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxParts = 128;           // blocks per frame (pair) in the partial-sum kernels
constexpr int kPixelsPerThread = 8;

inline int parts_for(long hw, int per_thread) {
  const long want = (hw + (long)kThreads * per_thread - 1) / ((long)kThreads * per_thread);
  return (int)(want < 1 ? 1 : (want > kMaxParts ? kMaxParts : want));
}

__device__ __forceinline__ bool valid_depth(float v) { return isfinite(v) && v > 1e-2f; }

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// acc[K] of every thread -> dst[K] (thread order -> warp xor tree -> warps in index order). red: [kThreads / 32][K] doubles.
template <int K>
__device__ __forceinline__ void block_sums(const double (&acc)[K], double* red, double* dst) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < K; ++j) {
    const double v = warp_sum_d(acc[j]);
    if (lane == 0) red[warp * K + j] = v;
  }
  __syncthreads();
  if (threadIdx.x < K) {
    double s = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) s = __dadd_rn(s, red[w * K + threadIdx.x]);
    dst[threadIdx.x] = s;
  }
}

// grid (n segments), block K: out[s][j] = sum over p of partials[s][p][j], p ascending
__global__ void reduce_partials_kernel(const double* __restrict__ partials, double* __restrict__ out, int P, int K) {
  DVD_PDL_ENTER();
  const long s = blockIdx.x;
  const int j = threadIdx.x;
  if (j >= K) return;
  double acc = 0.0;
  for (int p = 0; p < P; ++p) acc = __dadd_rn(acc, partials[(s * P + p) * K + j]);
  out[s * K + j] = acc;
}

// cam [30] = K^T | (K^-1)^T | R | t (fp32, dvd_b200.points.camera_block): K[r][c] = cam[3 c + r], Kinv[r][c] = cam[9 + 3 c + r],
// R[r][c] = cam[18 + 3 r + c], t[r] = cam[27 + r]
__device__ __forceinline__ double dot3(double a0, double a1, double a2, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a0, x), __dmul_rn(a1, y)), __dmul_rn(a2, z));
}

// Stages the cameras of pair `pair` (frames ia, ib) in fp64 into cm; every thread of the block calls it.
__device__ __forceinline__ void stage_pair_cameras(const float* __restrict__ cam, long fa, long fb, double (&cm)[2][30]) {
  if (threadIdx.x < 60) cm[threadIdx.x / 30][threadIdx.x % 30] = (double)cam[(threadIdx.x < 30 ? fa : fb) * 30 + threadIdx.x % 30];
  __syncthreads();
}

// Pixel i's flow target q = x + flow(x) and its border-clamped bilinear taps (align_corners=True: pixel centres at integer
// coordinates) into frame b.
struct FlowTaps {
  double x, y, qx, qy, wx0, wx1, wy0, wy1;
  long o00, o01, o10, o11;
};

// false when q is not finite (the pixel is not evaluated)
__device__ __forceinline__ bool flow_taps(long i, int H, int W, float2 f, FlowTaps& t) {
  t.x = (double)(i % W);
  t.y = (double)(i / W);
  t.qx = __dadd_rn(t.x, (double)f.x);
  t.qy = __dadd_rn(t.y, (double)f.y);
  if (!isfinite(t.qx) || !isfinite(t.qy)) return false;
  const double ix = fmin(fmax(t.qx, 0.0), (double)(W - 1)), iy = fmin(fmax(t.qy, 0.0), (double)(H - 1));
  const double x0f = floor(ix), y0f = floor(iy);
  const int x0 = (int)x0f, y0 = (int)y0f, x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
  t.wx1 = __dsub_rn(ix, x0f);
  t.wy1 = __dsub_rn(iy, y0f);
  t.wx0 = __dsub_rn(1.0, t.wx1);
  t.wy0 = __dsub_rn(1.0, t.wy1);
  t.o00 = (long)y0 * W + x0;
  t.o01 = (long)y0 * W + x1;
  t.o10 = (long)y1 * W + x0;
  t.o11 = (long)y1 * W + x1;
  return true;
}

enum PixelResult { kNotEvaluated = 0, kBehind = 1, kGood = 2 };

// One depth source at pixel i of frame a (Da, Db: the frames' maps, A, B: their staged cameras). With kSf, the scene flow
// (sf[0], sf[hw], sf[2 hw], fp32: the pixel's entry of a [3,H,W] map) is added in fp64 to the world point P after it is formed,
// before the change to camera b.
//   P = R_a (d_a Kinv_a (x, y, 1)) + t_a  [+ sf];  c = R_b^T (P - t_b);  z = c.z
//   z <= 1e-3: kBehind;  else p = (K_b c).xy / z, e_r = |p - q|, e_d = |z - Db~(q)| / Db~(q): kGood
template <bool kSf>
__device__ __forceinline__ int pair_pixel(const double* A, const double* B, const float* __restrict__ Da, const float* __restrict__ Db,
                                          long i, const FlowTaps& t, const float* __restrict__ sf, long hw, double& er,
                                          double& ed) {
  const float daf = Da[i];
  if (!valid_depth(daf)) return kNotEvaluated;
  const float t00 = Db[t.o00], t01 = Db[t.o01], t10 = Db[t.o10], t11 = Db[t.o11];
  if (!valid_depth(t00) || !valid_depth(t01) || !valid_depth(t10) || !valid_depth(t11)) return kNotEvaluated;
  const double da = (double)daf;
  const double db = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(__dmul_rn(t.wy0, t.wx0), (double)t00),
                                                  __dmul_rn(__dmul_rn(t.wy0, t.wx1), (double)t01)),
                                        __dmul_rn(__dmul_rn(t.wy1, t.wx0), (double)t10)),
                              __dmul_rn(__dmul_rn(t.wy1, t.wx1), (double)t11));
  double cv[3], pw[3], c[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) cv[r] = __dmul_rn(da, dot3(A[9 + r], A[12 + r], A[15 + r], t.x, t.y, 1.0));
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    double p = __dadd_rn(dot3(A[18 + 3 * r], A[19 + 3 * r], A[20 + 3 * r], cv[0], cv[1], cv[2]), A[27 + r]);
    if (kSf) p = __dadd_rn(p, (double)sf[r * hw]);
    pw[r] = __dsub_rn(p, B[27 + r]);
  }
#pragma unroll
  for (int r = 0; r < 3; ++r) c[r] = dot3(B[18 + r], B[21 + r], B[24 + r], pw[0], pw[1], pw[2]);
  const double z = c[2];
  if (!(z > 1e-3)) return kBehind;
  const double px = __ddiv_rn(dot3(B[0], B[3], B[6], c[0], c[1], c[2]), z);
  const double py = __ddiv_rn(dot3(B[1], B[4], B[7], c[0], c[1], c[2]), z);
  const double ex = __dsub_rn(px, t.qx), ey = __dsub_rn(py, t.qy);
  er = __dsqrt_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)));
  ed = __ddiv_rn(fabs(__dsub_rn(z, db)), db);
  return kGood;
}

// adds one evaluated pixel to the six sums of a region: count, behind, sum e_r, sum e_d, #e_r < 1, #e_r < 3
__device__ __forceinline__ void add_pixel(double* s, int res, double er, double ed) {
  if (res == kBehind) {
    s[1] = __dadd_rn(s[1], 1.0);
    return;
  }
  s[0] = __dadd_rn(s[0], 1.0);
  s[2] = __dadd_rn(s[2], er);
  s[3] = __dadd_rn(s[3], ed);
  s[4] = __dadd_rn(s[4], er < 1.0 ? 1.0 : 0.0);
  s[5] = __dadd_rn(s[5], er < 3.0 ? 1.0 : 0.0);
}

}  // namespace
}  // namespace dvd
