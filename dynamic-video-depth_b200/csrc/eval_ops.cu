// Validation metric of the per-video optimisation: the reference's `disp_vali` (models/video_base.py:66-74), the MSE between the
// predicted and the ground-truth disparity on the pixels where the ground truth is valid, for N frames per launch pair.
//
// Pass 1 evaluates the per-pixel term in torch's own operation order, every operation rounded on its own (__fadd_rn,
// __fdiv_rn, __fmul_rn: no contraction), so that each term equals torch CPU's elementwise result bit for bit, and writes one
// partial sum per block. Pass 2 adds a frame's partials in a fixed order. There are no atomics: the per-frame sums are
// bitwise reproducible from run to run. CUDA cores only; the kernel reads 8 bytes per pixel and is bandwidth-bound.
#include "common.cuh"

namespace dvd {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxParts = 128;          // blocks per frame in pass 1 (= threads of pass 2)
constexpr int kPixelsPerThread = 8;     // pass-1 target work per thread before the block count is capped

// depth2disp(x) = (1 / (x + (1 - [x > 1e-2]) * 1e-8)) * [x > 1e-2]; `1 / t` is torch's reciprocal(t) * 1 (an IEEE division).
// The comparisons are made in fp32 against 1e-2f, as torch promotes the Python scalar to the tensor's dtype.
__device__ __forceinline__ float disp_term(float d, float g) {
  const float vd = d > 1e-2f ? 1.f : 0.f, vg = g > 1e-2f ? 1.f : 0.f;
  const float rd = __fdiv_rn(1.f, __fadd_rn(d, __fmul_rn(__fsub_rn(1.f, vd), 1e-8f)));
  const float rg = __fdiv_rn(1.f, __fadd_rn(g, __fmul_rn(__fsub_rn(1.f, vg), 1e-8f)));
  // disp(d) * vali - disp(g) * vali with vali = [g > 1e-2]; mse_loss squares the rounded difference
  const float a = __fmul_rn(__fmul_rn(rd, vd), vg), b = __fmul_rn(__fmul_rn(rg, vg), vg);
  const float diff = __fsub_rn(a, b);
  return __fmul_rn(diff, diff);
}

// thread order -> warp xor tree -> the block's warps in index order (all fixed)
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float s = 0.f;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s = __fadd_rn(s, red[w]);
  return s;
}

// grid (P, N): block b of frame n visits the frame's items b*T + t, b*T + t + P*T, ... and adds their terms in that order.
template <bool kVec4>
__global__ void __launch_bounds__(kThreads) disp_vali_partial_kernel(const float* __restrict__ depth, const float* __restrict__ gt,
                                                                    float* __restrict__ terms, float* __restrict__ partials,
                                                                    long hw) {
  DVD_PDL_ENTER();
  __shared__ float red[kThreads / 32];
  const long frame = blockIdx.y, P = gridDim.x;
  const long base = frame * hw;
  const long stride = P * kThreads;
  float acc = 0.f;
  if (kVec4) {
    const long n4 = hw >> 2;
    for (long i = (long)blockIdx.x * kThreads + threadIdx.x; i < n4; i += stride) {
      const float4 d = ldg_stream4(depth + base + 4 * i), g = ldg_stream4(gt + base + 4 * i);
      const float4 t = make_float4(disp_term(d.x, g.x), disp_term(d.y, g.y), disp_term(d.z, g.z), disp_term(d.w, g.w));
      if (terms) st_stream4(terms + base + 4 * i, t);
      acc = __fadd_rn(acc, t.x);
      acc = __fadd_rn(acc, t.y);
      acc = __fadd_rn(acc, t.z);
      acc = __fadd_rn(acc, t.w);
    }
  } else {
    for (long i = (long)blockIdx.x * kThreads + threadIdx.x; i < hw; i += stride) {
      const float t = disp_term(ldg_stream1(depth + base + i), ldg_stream1(gt + base + i));
      if (terms) terms[base + i] = t;
      acc = __fadd_rn(acc, t);
    }
  }
  const float s = block_sum(acc, red);
  if (threadIdx.x == 0) partials[frame * P + blockIdx.x] = s;
}

// one block per frame: thread t < P holds partial t; the block sum is the frame's SSE
__global__ void __launch_bounds__(kMaxParts) disp_vali_frame_kernel(const float* __restrict__ partials, float* __restrict__ frame_sse,
                                                                   int P) {
  DVD_PDL_ENTER();
  __shared__ float red[kMaxParts / 32];
  const float v = (int)threadIdx.x < P ? partials[(long)blockIdx.x * P + threadIdx.x] : 0.f;
  const float s = block_sum(v, red);
  if (threadIdx.x == 0) frame_sse[blockIdx.x] = s;
}

int parts_for(long hw) {
  const long want = (hw + (long)kThreads * kPixelsPerThread - 1) / ((long)kThreads * kPixelsPerThread);
  return (int)(want < 1 ? 1 : (want > kMaxParts ? kMaxParts : want));
}

static inline bool aligned_to(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

#define EV_CHECK(cond, ...)        \
  do {                             \
    if (!(cond)) {                 \
      dvd::set_error(__VA_ARGS__); \
      return -2;                   \
    }                              \
  } while (0)

}  // namespace
}  // namespace dvd

using namespace dvd;

extern "C" int dvd_disp_vali_partials_size(int N, int H, int W) {
  if (N < 1 || H < 1 || W < 1) return -1;
  return N * parts_for((long)H * W);
}

extern "C" int dvd_disp_vali(const float* depth, const float* depth_gt, float* frame_sse, float* terms, float* partials, int N,
                             int H, int W, void* stream) {
  EV_CHECK(depth && depth_gt && frame_sse && partials, "dvd_disp_vali: null pointer (only `terms` may be NULL)");
  EV_CHECK(N >= 1 && H >= 1 && W >= 1, "dvd_disp_vali: bad shape N=%d H=%d W=%d", N, H, W);
  EV_CHECK(N <= 65535, "dvd_disp_vali: at most 65535 frames per call, got %d", N);
  EV_CHECK(aligned_to(depth, 4) && aligned_to(depth_gt, 4) && aligned_to(frame_sse, 4) && aligned_to(partials, 4) &&
               (!terms || aligned_to(terms, 4)),
           "dvd_disp_vali: buffers must be 4-byte aligned fp32");
  const long hw = (long)H * W;
  const int P = parts_for(hw);
  // float4 path: every frame starts on a 16-byte boundary when the base pointers do and H*W is a multiple of 4
  const bool vec = (hw % 4 == 0) && aligned16(depth) && aligned16(depth_gt) && (!terms || aligned16(terms));
  const cudaStream_t st = (cudaStream_t)stream;
  if (vec)
    DVD_CUDA_CALL(launch(disp_vali_partial_kernel<true>, dim3(P, N), dim3(kThreads), 0, st, depth, depth_gt, terms, partials, hw));
  else
    DVD_CUDA_CALL(launch(disp_vali_partial_kernel<false>, dim3(P, N), dim3(kThreads), 0, st, depth, depth_gt, terms, partials, hw));
  DVD_CUDA_CALL(launch(disp_vali_frame_kernel, dim3(N), dim3(kMaxParts), 0, st, (const float*)partials, frame_sse, P));
  return 0;
}
