// Evaluation of a test export (dvd_b200.evaluate): depth accuracy against depth_gt and consistency along the optical flow, for
// the refined and the initial depth. Nothing in the reference corresponds; oracle/evaluate.py restates every rule in numpy.
//
//   dvd_masked_select      the lower median (rank (n - 1) / 2) of the valid elements of every frame and of all frames pooled,
//                          exact: an 8-bit radix select on order-preserving 32-bit keys, four histogram passes
//   dvd_depth_metrics      every frame's accuracy sums under three depth scales, both depth sources, one pass
//   dvd_pair_consistency   every pair's reprojection / depth-error sums, both depth sources, all pixels and the static ones
//
// Per-pixel arithmetic is fp64 with every operation rounded on its own (__dmul_rn, __dadd_rn, ...: no contraction), in the
// operation order include/dvd_b200.h states, so each term equals numpy's. Sums are fp64 and run in a fixed order: each thread
// adds its pixels in index order, a block adds its threads with a fixed shuffle tree and its warps in order, and a second
// kernel adds a frame's (pair's) block partials in block order. The number of blocks per frame depends on H * W alone, so a
// frame's or a pair's sums do not depend on what else is in the launch. The selection histograms are integer counts, exact in
// any order.
#include <math.h>

#include "common.cuh"

namespace dvd {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxParts = 128;           // blocks per frame (pair) in the partial-sum kernels
constexpr int kPixelsPerThread = 8;
constexpr int kSelectPixelsPerThread = 32;
constexpr int kBins = 256;
constexpr int kSelectState = 3;          // per segment: key prefix, remaining rank, valid count
constexpr int kMetricSlots = 2 * 22;     // per source: count, then per scale 7 sums
constexpr int kPairSlots = 2 * 2 * 6;    // per source and region: count, behind, sum e_r, sum e_d, #e_r < 1, #e_r < 3

int parts_for(long hw, int per_thread) {
  const long want = (hw + (long)kThreads * per_thread - 1) / ((long)kThreads * per_thread);
  return (int)(want < 1 ? 1 : (want > kMaxParts ? kMaxParts : want));
}

__device__ __forceinline__ bool valid_depth(float v) { return isfinite(v) && v > 1e-2f; }

// order-preserving map of fp32 bits to uint32 (negative values flipped, positive ones offset past them), and its inverse
__device__ __forceinline__ unsigned int order_key(float v) {
  const unsigned int u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(unsigned int k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

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

// ---- masked selection ---------------------------------------------------------------------------------------------------------
// work: hist [(N + 1) * 256] then state [(N + 1) * 3], int64; segment N is the pool of all frames
__global__ void select_init_kernel(long long* __restrict__ work, long n_words) {
  DVD_PDL_ENTER();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += (long)gridDim.x * blockDim.x) work[i] = 0;
}

// grid (P, N): the histogram of digit `pass` (bits 31-8 pass .. 24-8 pass) of the keys of the valid elements whose higher
// digits match the segment's prefix, for the frame's segment and for the pooled one
__global__ void __launch_bounds__(kThreads) select_hist_kernel(const float* __restrict__ values, const float* __restrict__ other,
                                                               long long* __restrict__ work, int N, long hw, int pass) {
  DVD_PDL_ENTER();
  __shared__ unsigned int hf[kBins], hp[kBins];
  for (int b = threadIdx.x; b < kBins; b += kThreads) hf[b] = hp[b] = 0u;
  __syncthreads();
  const long frame = blockIdx.y;
  long long* hist = work;
  const long long* state = work + (long)(N + 1) * kBins;
  const unsigned int pre_f = (unsigned int)state[frame * kSelectState], pre_p = (unsigned int)state[(long)N * kSelectState];
  const int hi = 32 - 8 * pass, sh = 24 - 8 * pass;
  const float* v = values + frame * hw;
  const float* o = other ? other + frame * hw : nullptr;
  for (long i = (long)blockIdx.x * kThreads + threadIdx.x; i < hw; i += (long)gridDim.x * kThreads) {
    const float x = v[i];
    if (!valid_depth(x) || (o && !valid_depth(o[i]))) continue;
    const unsigned int k = order_key(x);
    const unsigned int top = pass == 0 ? 0u : (k >> hi);
    const unsigned int dg = (k >> sh) & 0xffu;
    if (top == pre_f) atomicAdd(&hf[dg], 1u);
    if (top == pre_p) atomicAdd(&hp[dg], 1u);
  }
  __syncthreads();
  for (int b = threadIdx.x; b < kBins; b += kThreads) {
    if (hf[b]) atomicAdd((unsigned long long*)&hist[frame * kBins + b], (unsigned long long)hf[b]);
    if (hp[b]) atomicAdd((unsigned long long*)&hist[(long)N * kBins + b], (unsigned long long)hp[b]);
  }
}

// grid (N + 1), block 256: finds the bin holding the segment's remaining rank, appends it to the prefix and clears the histogram;
// after the last pass writes the selected value (NaN for an empty segment) and the count
__global__ void __launch_bounds__(kBins) select_step_kernel(long long* __restrict__ work, int N, int pass, float* __restrict__ out,
                                                             long long* __restrict__ count) {
  DVD_PDL_ENTER();
  __shared__ long long h[kBins];
  const long s = blockIdx.x;
  long long* hist = work + s * kBins;
  long long* st = work + (long)(N + 1) * kBins + s * kSelectState;
  h[threadIdx.x] = hist[threadIdx.x];
  hist[threadIdx.x] = 0;
  __syncthreads();
  if (threadIdx.x != 0) return;
  long long rank = st[1];
  if (pass == 0) {
    long long n = 0;
    for (int b = 0; b < kBins; ++b) n += h[b];
    st[2] = n;
    rank = n > 0 ? (n - 1) / 2 : 0;
  }
  const long long n = st[2];
  unsigned long long prefix = (unsigned long long)st[0];
  if (n > 0) {
    long long cum = 0;
    int b = 0;
    while (b < kBins - 1 && cum + h[b] <= rank) cum += h[b++];
    rank -= cum;
    prefix = (prefix << 8) | (unsigned long long)b;
  }
  st[0] = (long long)prefix;
  st[1] = rank;
  if (pass == 3) {
    out[s] = n > 0 ? key_value((unsigned int)prefix) : __int_as_float(0x7fc00000);
    count[s] = n;
  }
}

// ---- accuracy sums ------------------------------------------------------------------------------------------------------------
// per source j (0: depth, 1: depth_nn), slots 22 j + {0: valid count, 1 + 7 a + {0: sum |d' - g| / g, 1: sum (d' - g)^2 / g,
// 2: sum (d' - g)^2, 3: sum (ln d' - ln g)^2, 4..6: #max(d'/g, g/d') < 1.25, 1.25^2, 1.25^3}} for the scales a = 0, 1, 2
__global__ void __launch_bounds__(kThreads) depth_metrics_partial_kernel(const float* __restrict__ depth,
                                                                         const float* __restrict__ depth_nn,
                                                                         const float* __restrict__ gt,
                                                                         const double* __restrict__ scales,
                                                                         double* __restrict__ partials, long hw) {
  DVD_PDL_ENTER();
  __shared__ double red[(kThreads / 32) * kMetricSlots];
  const long frame = blockIdx.y, P = gridDim.x;
  double acc[kMetricSlots];
#pragma unroll
  for (int j = 0; j < kMetricSlots; ++j) acc[j] = 0.0;
  double sc[6];
#pragma unroll
  for (int j = 0; j < 6; ++j) sc[j] = scales[frame * 6 + j];
  const long base = frame * hw;
  for (long i = (long)blockIdx.x * kThreads + threadIdx.x; i < hw; i += P * kThreads) {
    const float gf = gt[base + i];
    if (!valid_depth(gf)) continue;
    const double g = (double)gf, lg = log(g);
#pragma unroll
    for (int src = 0; src < 2; ++src) {
      const float df = (src == 0 ? depth : depth_nn)[base + i];
      if (!valid_depth(df)) continue;
      const double d = (double)df;
      double* a = acc + 22 * src;
      a[0] = __dadd_rn(a[0], 1.0);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double dp = __dmul_rn(sc[3 * src + k], d);
        const double diff = __dsub_rn(dp, g);
        const double sq = __dmul_rn(diff, diff);
        const double lgd = __dsub_rn(log(dp), lg);
        const double ratio = fmax(__ddiv_rn(dp, g), __ddiv_rn(g, dp));
        double* s = a + 1 + 7 * k;
        s[0] = __dadd_rn(s[0], __ddiv_rn(fabs(diff), g));
        s[1] = __dadd_rn(s[1], __ddiv_rn(sq, g));
        s[2] = __dadd_rn(s[2], sq);
        s[3] = __dadd_rn(s[3], __dmul_rn(lgd, lgd));
        s[4] = __dadd_rn(s[4], ratio < 1.25 ? 1.0 : 0.0);
        s[5] = __dadd_rn(s[5], ratio < 1.5625 ? 1.0 : 0.0);
        s[6] = __dadd_rn(s[6], ratio < 1.953125 ? 1.0 : 0.0);
      }
    }
  }
  block_sums<kMetricSlots>(acc, red, partials + (frame * P + blockIdx.x) * kMetricSlots);
}

// ---- consistency along the flow -----------------------------------------------------------------------------------------------
// cam [30] = K^T | (K^-1)^T | R | t (fp32, dvd_b200.points.camera_block): K[r][c] = cam[3 c + r], Kinv[r][c] = cam[9 + 3 c + r],
// R[r][c] = cam[18 + 3 r + c], t[r] = cam[27 + r]
__device__ __forceinline__ double dot3(double a0, double a1, double a2, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a0, x), __dmul_rn(a1, y)), __dmul_rn(a2, z));
}

__global__ void __launch_bounds__(kThreads) pair_consistency_partial_kernel(
    const float* __restrict__ depth, const float* __restrict__ depth_nn, const float* __restrict__ cam,
    const int* __restrict__ ia, const int* __restrict__ ib, const float* __restrict__ flow, const unsigned char* __restrict__ mask,
    const unsigned char* __restrict__ motion_seg, double* __restrict__ partials, int H, int W) {
  DVD_PDL_ENTER();
  __shared__ double red[(kThreads / 32) * kPairSlots];
  __shared__ double cm[2][30];
  const long pair = blockIdx.y, P = gridDim.x, hw = (long)H * W;
  const long fa = ia[pair], fb = ib[pair];
  if (threadIdx.x < 60) cm[threadIdx.x / 30][threadIdx.x % 30] = (double)cam[(threadIdx.x < 30 ? fa : fb) * 30 + threadIdx.x % 30];
  __syncthreads();
  const double* A = cm[0];
  const double* B = cm[1];
  double acc[kPairSlots];
#pragma unroll
  for (int j = 0; j < kPairSlots; ++j) acc[j] = 0.0;
  const float* fl = flow + pair * hw * 2;
  const unsigned char* mk = mask + pair * hw;
  for (long i = (long)blockIdx.x * kThreads + threadIdx.x; i < hw; i += P * kThreads) {
    if (mk[i] != 0) continue;
    const float2 f = *reinterpret_cast<const float2*>(fl + 2 * i);
    const double x = (double)(i % W), y = (double)(i / W);
    const double qx = __dadd_rn(x, (double)f.x), qy = __dadd_rn(y, (double)f.y);
    if (!isfinite(qx) || !isfinite(qy)) continue;
    // border-clamped bilinear taps at q (align_corners=True: pixel centres at integer coordinates)
    const double ix = fmin(fmax(qx, 0.0), (double)(W - 1)), iy = fmin(fmax(qy, 0.0), (double)(H - 1));
    const double x0f = floor(ix), y0f = floor(iy);
    const int x0 = (int)x0f, y0 = (int)y0f, x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
    const double wx1 = __dsub_rn(ix, x0f), wy1 = __dsub_rn(iy, y0f);
    const double wx0 = __dsub_rn(1.0, wx1), wy0 = __dsub_rn(1.0, wy1);
    const bool stat = motion_seg != nullptr && motion_seg[fa * hw + i] == 0;
#pragma unroll
    for (int src = 0; src < 2; ++src) {
      const float* D = src == 0 ? depth : depth_nn;
      const float daf = D[fa * hw + i];
      if (!valid_depth(daf)) continue;
      const float* Db = D + fb * hw;
      const float t00 = Db[(long)y0 * W + x0], t01 = Db[(long)y0 * W + x1], t10 = Db[(long)y1 * W + x0],
                  t11 = Db[(long)y1 * W + x1];
      if (!valid_depth(t00) || !valid_depth(t01) || !valid_depth(t10) || !valid_depth(t11)) continue;
      const double da = (double)daf;
      const double db = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(__dmul_rn(wy0, wx0), (double)t00),
                                                      __dmul_rn(__dmul_rn(wy0, wx1), (double)t01)),
                                            __dmul_rn(__dmul_rn(wy1, wx0), (double)t10)),
                                  __dmul_rn(__dmul_rn(wy1, wx1), (double)t11));
      // P = R_a (d_a Kinv_a (x, y, 1)) + t_a;  c = R_b^T (P - t_b)
      double cv[3], pw[3], c[3];
#pragma unroll
      for (int r = 0; r < 3; ++r) cv[r] = __dmul_rn(da, dot3(A[9 + r], A[12 + r], A[15 + r], x, y, 1.0));
#pragma unroll
      for (int r = 0; r < 3; ++r) pw[r] = __dsub_rn(__dadd_rn(dot3(A[18 + 3 * r], A[19 + 3 * r], A[20 + 3 * r], cv[0], cv[1], cv[2]),
                                                              A[27 + r]),
                                                    B[27 + r]);
#pragma unroll
      for (int r = 0; r < 3; ++r) c[r] = dot3(B[18 + r], B[21 + r], B[24 + r], pw[0], pw[1], pw[2]);
      const double z = c[2];
      double* a = acc + 12 * src;
      if (!(z > 1e-3)) {
        a[1] = __dadd_rn(a[1], 1.0);
        if (stat) a[7] = __dadd_rn(a[7], 1.0);
        continue;
      }
      const double px = __ddiv_rn(dot3(B[0], B[3], B[6], c[0], c[1], c[2]), z);
      const double py = __ddiv_rn(dot3(B[1], B[4], B[7], c[0], c[1], c[2]), z);
      const double ex = __dsub_rn(px, qx), ey = __dsub_rn(py, qy);
      const double er = __dsqrt_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)));
      const double ed = __ddiv_rn(fabs(__dsub_rn(z, db)), db);
#pragma unroll
      for (int reg = 0; reg < 2; ++reg) {
        if (reg == 1 && !stat) break;
        double* s = a + 6 * reg;
        s[0] = __dadd_rn(s[0], 1.0);
        s[2] = __dadd_rn(s[2], er);
        s[3] = __dadd_rn(s[3], ed);
        s[4] = __dadd_rn(s[4], er < 1.0 ? 1.0 : 0.0);
        s[5] = __dadd_rn(s[5], er < 3.0 ? 1.0 : 0.0);
      }
    }
  }
  block_sums<kPairSlots>(acc, red, partials + (pair * P + blockIdx.x) * kPairSlots);
}

#define DM_CHECK(cond, ...)        \
  do {                             \
    if (!(cond)) {                 \
      dvd::set_error(__VA_ARGS__); \
      return -2;                   \
    }                              \
  } while (0)

static inline bool aligned_to(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

}  // namespace
}  // namespace dvd

using namespace dvd;

extern "C" long long dvd_masked_select_partials_size(int N, int H, int W) {
  if (N < 1 || H < 1 || W < 1) return -1;
  return (long long)(N + 1) * (kBins + kSelectState);
}

extern "C" int dvd_masked_select(const float* values, const float* other, float* median, long long* count, long long* work,
                                 int N, int H, int W, void* stream) {
  DM_CHECK(values && median && count && work, "dvd_masked_select: null pointer (only `other` may be NULL)");
  DM_CHECK(N >= 1 && H >= 1 && W >= 1 && N <= 65535, "dvd_masked_select: bad shape N=%d H=%d W=%d (1 <= N <= 65535)", N, H, W);
  DM_CHECK(aligned_to(values, 4) && aligned_to(other, 4) && aligned_to(median, 4) && aligned_to(count, 8) && aligned_to(work, 8),
           "dvd_masked_select: misaligned buffer");
  const long hw = (long)H * W;
  const int P = parts_for(hw, kSelectPixelsPerThread);
  const cudaStream_t st = (cudaStream_t)stream;
  const long words = (long)(N + 1) * (kBins + kSelectState);
  DVD_CUDA_CALL(launch(select_init_kernel, dim3((unsigned)((words + kThreads - 1) / kThreads)), dim3(kThreads), 0, st, work, words));
  for (int pass = 0; pass < 4; ++pass) {
    DVD_CUDA_CALL(launch(select_hist_kernel, dim3(P, N), dim3(kThreads), 0, st, values, other, work, N, hw, pass));
    DVD_CUDA_CALL(launch(select_step_kernel, dim3(N + 1), dim3(kBins), 0, st, work, N, pass, median, count));
  }
  return 0;
}

extern "C" long long dvd_depth_metrics_partials_size(int N, int H, int W) {
  if (N < 1 || H < 1 || W < 1) return -1;
  return (long long)N * parts_for((long)H * W, kPixelsPerThread) * kMetricSlots;
}

extern "C" int dvd_depth_metrics(const float* depth, const float* depth_nn, const float* depth_gt, const double* scales,
                                 double* sums, double* partials, int N, int H, int W, void* stream) {
  DM_CHECK(depth && depth_nn && depth_gt && scales && sums && partials, "dvd_depth_metrics: null pointer");
  DM_CHECK(N >= 1 && H >= 1 && W >= 1 && N <= 65535, "dvd_depth_metrics: bad shape N=%d H=%d W=%d (1 <= N <= 65535)", N, H, W);
  DM_CHECK(aligned_to(depth, 4) && aligned_to(depth_nn, 4) && aligned_to(depth_gt, 4) && aligned_to(scales, 8) &&
               aligned_to(sums, 8) && aligned_to(partials, 8),
           "dvd_depth_metrics: misaligned buffer");
  const long hw = (long)H * W;
  const int P = parts_for(hw, kPixelsPerThread);
  const cudaStream_t st = (cudaStream_t)stream;
  DVD_CUDA_CALL(launch(depth_metrics_partial_kernel, dim3(P, N), dim3(kThreads), 0, st, depth, depth_nn, depth_gt, scales, partials, hw));
  DVD_CUDA_CALL(launch(reduce_partials_kernel, dim3(N), dim3(64), 0, st, (const double*)partials, sums, P, kMetricSlots));
  return 0;
}

extern "C" long long dvd_pair_consistency_partials_size(int n_pairs, int H, int W) {
  if (n_pairs < 1 || H < 1 || W < 1) return -1;
  return (long long)n_pairs * parts_for((long)H * W, kPixelsPerThread) * kPairSlots;
}

extern "C" int dvd_pair_consistency(const float* depth, const float* depth_nn, const float* cam, int n_frames, const int* ia,
                                    const int* ib, const float* flow, const unsigned char* mask, const unsigned char* motion_seg,
                                    double* sums, double* partials, int n_pairs, int H, int W, void* stream) {
  DM_CHECK(depth && depth_nn && cam && ia && ib && flow && mask && sums && partials,
           "dvd_pair_consistency: null pointer (only `motion_seg` may be NULL)");
  DM_CHECK(n_frames >= 1 && n_pairs >= 1 && n_pairs <= 65535 && H >= 1 && W >= 1,
           "dvd_pair_consistency: bad shape n_frames=%d n_pairs=%d H=%d W=%d (1 <= n_pairs <= 65535)", n_frames, n_pairs, H, W);
  DM_CHECK(aligned_to(depth, 4) && aligned_to(depth_nn, 4) && aligned_to(cam, 4) && aligned_to(ia, 4) && aligned_to(ib, 4) &&
               aligned_to(flow, 8) && aligned_to(sums, 8) && aligned_to(partials, 8),
           "dvd_pair_consistency: misaligned buffer");
  const int P = parts_for((long)H * W, kPixelsPerThread);
  const cudaStream_t st = (cudaStream_t)stream;
  DVD_CUDA_CALL(launch(pair_consistency_partial_kernel, dim3(P, n_pairs), dim3(kThreads), 0, st, depth, depth_nn, cam, ia, ib, flow,
                       mask, motion_seg, partials, H, W));
  DVD_CUDA_CALL(launch(reduce_partials_kernel, dim3(n_pairs), dim3(32), 0, st, (const double*)partials, sums, P, kPairSlots));
  return 0;
}
