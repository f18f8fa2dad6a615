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

#include "pair_consistency.cuh"

namespace dvd {
namespace {

constexpr int kSelectPixelsPerThread = 32;
constexpr int kBins = 256;
constexpr int kSelectState = 3;          // per segment: key prefix, remaining rank, valid count
constexpr int kMetricSlots = 2 * 22;     // per source: count, then per scale 7 sums
constexpr int kPairSlots = 2 * 2 * 6;    // per source and region: count, behind, sum e_r, sum e_d, #e_r < 1, #e_r < 3

// order-preserving map of fp32 bits to uint32 (negative values flipped, positive ones offset past them), and its inverse
__device__ __forceinline__ unsigned int order_key(float v) {
  const unsigned int u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(unsigned int k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
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
// the per-pixel rule is pair_pixel (pair_consistency.cuh); per source, slots 12 src + 6 region + {count, behind, sum e_r, sum e_d,
// #e_r < 1, #e_r < 3}, regions all and static
__global__ void __launch_bounds__(kThreads) pair_consistency_partial_kernel(
    const float* __restrict__ depth, const float* __restrict__ depth_nn, const float* __restrict__ cam,
    const int* __restrict__ ia, const int* __restrict__ ib, const float* __restrict__ flow, const unsigned char* __restrict__ mask,
    const unsigned char* __restrict__ motion_seg, double* __restrict__ partials, int H, int W) {
  DVD_PDL_ENTER();
  __shared__ double red[(kThreads / 32) * kPairSlots];
  __shared__ double cm[2][30];
  const long pair = blockIdx.y, P = gridDim.x, hw = (long)H * W;
  const long fa = ia[pair], fb = ib[pair];
  stage_pair_cameras(cam, fa, fb, cm);
  double acc[kPairSlots];
#pragma unroll
  for (int j = 0; j < kPairSlots; ++j) acc[j] = 0.0;
  const float* fl = flow + pair * hw * 2;
  const unsigned char* mk = mask + pair * hw;
  for (long i = (long)blockIdx.x * kThreads + threadIdx.x; i < hw; i += P * kThreads) {
    if (mk[i] != 0) continue;
    FlowTaps t;
    if (!flow_taps(i, H, W, *reinterpret_cast<const float2*>(fl + 2 * i), t)) continue;
    const bool stat = motion_seg != nullptr && motion_seg[fa * hw + i] == 0;
#pragma unroll
    for (int src = 0; src < 2; ++src) {
      const float* D = src == 0 ? depth : depth_nn;
      double er = 0.0, ed = 0.0;
      const int res = pair_pixel<false>(cm[0], cm[1], D + fa * hw, D + fb * hw, i, t, nullptr, hw, er, ed);
      if (res == kNotEvaluated) continue;
      add_pixel(acc + 12 * src, res, er, ed);
      if (stat) add_pixel(acc + 12 * src + 6, res, er, ed);
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
