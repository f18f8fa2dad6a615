// Flow-pair preprocessing: the cubic flow resize and the forward / backward consistency masks that turn two raw optical
// flows into the training pair of scripts/preprocess/davis/generate_flows.py:44-82,139-148.
//
// Both kernels are batched over pairs, read and write NHWC fp32 flows [B,H,W,2] (the layout of the pair files) and run one
// output pixel per thread with float2 loads. Every operation is rounded on its own (__fmul_rn / __fadd_rn, and __fmaf_rn
// where the reference itself fuses), so oracle/flow_pairs.py restates them bitwise on the CPU.
#include "common.cuh"

namespace dvd {
namespace {

constexpr int kThreads = 256;

// ---- cv2.resize(..., INTER_CUBIC) on float32 ---------------------------------------------------------------------------
// OpenCV's interpolateCubic (A = -0.75)
__device__ __forceinline__ void cubic_coeffs(float x, float c[4]) {
  const float A = -0.75f;
  const float x1 = __fadd_rn(x, 1.f);
  c[0] = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, x1), 5.f * A), x1), 8.f * A), x1), 4.f * A);
  c[1] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2.f, x), A + 3.f), x), x), 1.f);
  const float y = __fsub_rn(1.f, x);
  c[2] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2.f, y), A + 3.f), y), y), 1.f);
  c[3] = __fsub_rn(__fsub_rn(__fsub_rn(1.f, c[0]), c[1]), c[2]);
}

// source position of output index d: fx = (float)((d + 0.5) * scale - 0.5) in double, sx = floor(fx), fx -= sx
__device__ __forceinline__ int cubic_src(int d, double scale, float* frac) {
  const float f = (float)__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5);
  const float s = floorf(f);
  *frac = __fsub_rn(f, s);
  return (int)s;
}

__global__ void __launch_bounds__(kThreads) flow_resize_cubic_kernel(const float2* __restrict__ src, float2* __restrict__ dst,
                                                                      long n, int h, int w, int H, int W, double scale_x,
                                                                      double scale_y, double mul_x, double mul_y) {
  DVD_PDL_ENTER();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const long r = i / W;
    const int y = (int)(r % H);
    const long b = r / H;
    float fx, fy, cx[4], cy[4];
    const int sx = cubic_src(x, scale_x, &fx), sy = cubic_src(y, scale_y, &fy);
    cubic_coeffs(fx, cx);
    cubic_coeffs(fy, cy);
    int xs[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) xs[k] = min(max(sx - 1 + k, 0), w - 1);
    const float2* plane = src + b * h * w;
    float2 rows[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {       // horizontal pass of the four source rows: ((c0 s0 + c1 s1) + c2 s2) + c3 s3
      const float2* row = plane + (long)min(max(sy - 1 + j, 0), h - 1) * w;
      float2 v = __ldg(row + xs[0]);
      v.x = __fmul_rn(v.x, cx[0]);
      v.y = __fmul_rn(v.y, cx[0]);
#pragma unroll
      for (int k = 1; k < 4; ++k) {
        const float2 s = __ldg(row + xs[k]);
        v.x = __fadd_rn(v.x, __fmul_rn(s.x, cx[k]));
        v.y = __fadd_rn(v.y, __fmul_rn(s.y, cx[k]));
      }
      rows[j] = v;
    }
    // vertical pass in cv2's SIMD order: b0 r0 + (b1 r1 + (b2 r2 + b3 r3))
    float ox = __fmul_rn(rows[3].x, cy[3]), oy = __fmul_rn(rows[3].y, cy[3]);
#pragma unroll
    for (int j = 2; j >= 0; --j) {
      ox = __fadd_rn(__fmul_rn(rows[j].x, cy[j]), ox);
      oy = __fadd_rn(__fmul_rn(rows[j].y, cy[j]), oy);
    }
    // resize_flow's `resized *= scale`: a float64 scale applied to the float32 array
    dst[i] = make_float2((float)__dmul_rn((double)ox, mul_x), (float)__dmul_rn((double)oy, mul_y));
  }
}

// ---- consistency masks --------------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 tap(const float2* __restrict__ plane, int x, int y, int H, int W) {
  return (x >= 0 && x < W && y >= 0 && y < H) ? __ldg(plane + (long)y * W + x) : make_float2(0.f, 0.f);
}

// pixel (x, y) moved by `fl` is bad when it leaves the image or when `field`, sampled there as F.grid_sample does (bilinear,
// zeros padding, align_corners=True, after the reference's normalise / un-normalise round trip), does not bring it back
// within one pixel: |field(q) + fl| > 1.
__device__ __forceinline__ bool bad_pixel(const float2* __restrict__ field, float2 fl, int x, int y, int H, int W, float half_w,
                                          float half_h) {
  const float qx = __fadd_rn((float)x, fl.x), qy = __fadd_rn((float)y, fl.y);
  const bool oob = qx < 0.f || qx > (float)(W - 1) || qy < 0.f || qy > (float)(H - 1);
  const float ix = __fmul_rn(__fadd_rn(__fsub_rn(__fdiv_rn(qx, half_w), 1.f), 1.f), half_w);
  const float iy = __fmul_rn(__fadd_rn(__fsub_rn(__fdiv_rn(qy, half_h), 1.f), 1.f), half_h);
  const float x0 = floorf(ix), y0 = floorf(iy);
  const float wx = __fsub_rn(ix, x0), ex = __fsub_rn(1.f, wx), ny = __fsub_rn(iy, y0), sy = __fsub_rn(1.f, ny);
  const float w_nw = __fmul_rn(sy, ex), w_ne = __fmul_rn(sy, wx), w_sw = __fmul_rn(ny, ex), w_se = __fmul_rn(ny, wx);
  // every tap outside [-1, W] x [-1, H] reads zero: clamping there keeps the integer conversion in range (NaN -> -2)
  const int xi = (int)fminf(fmaxf(x0, -2.f), (float)W + 1.f), yi = (int)fminf(fmaxf(y0, -2.f), (float)H + 1.f);
  const float2 nw = tap(field, xi, yi, H, W), ne = tap(field, xi + 1, yi, H, W);
  const float2 sw = tap(field, xi, yi + 1, H, W), se = tap(field, xi + 1, yi + 1, H, W);
  // ATen's CPU kernel accumulates the taps with fused multiply-adds
  float vx = __fmul_rn(nw.x, w_nw), vy = __fmul_rn(nw.y, w_nw);
  vx = __fmaf_rn(ne.x, w_ne, vx);
  vy = __fmaf_rn(ne.y, w_ne, vy);
  vx = __fmaf_rn(sw.x, w_sw, vx);
  vy = __fmaf_rn(sw.y, w_sw, vy);
  vx = __fmaf_rn(se.x, w_se, vx);
  vy = __fmaf_rn(se.y, w_se, vy);
  const float dx = __fadd_rn(vx, fl.x), dy = __fadd_rn(vy, fl.y);
  const float err = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
  return oob || err > 1.f;
}

// mask_1 (frame 2's grid): flow_1_2 sampled at p + flow_2_1(p); mask_2: the same with the flows swapped.
// kValidF32: pair-file convention, fp32 1 - ceil(mask) (1 = valid); otherwise the flowpair one, uint8 1 = bad.
template <bool kValidF32>
__global__ void __launch_bounds__(kThreads) flow_pair_masks_kernel(const float2* __restrict__ f12, const float2* __restrict__ f21,
                                                                    void* __restrict__ m1, void* __restrict__ m2, long n, int H,
                                                                    int W, float half_w, float half_h) {
  DVD_PDL_ENTER();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const long r = i / W;
    const int y = (int)(r % H);
    const long off = (r / H) * H * W;
    const float2 a12 = __ldg(f12 + i), a21 = __ldg(f21 + i);
    const bool bad_1 = bad_pixel(f12 + off, a21, x, y, H, W, half_w, half_h);
    const bool bad_2 = bad_pixel(f21 + off, a12, x, y, H, W, half_w, half_h);
    if (kValidF32) {
      static_cast<float*>(m1)[i] = bad_1 ? 0.f : 1.f;
      static_cast<float*>(m2)[i] = bad_2 ? 0.f : 1.f;
    } else {
      static_cast<unsigned char*>(m1)[i] = bad_1 ? 1 : 0;
      static_cast<unsigned char*>(m2)[i] = bad_2 ? 1 : 0;
    }
  }
}

int grid_for(long n) {
  const long blocks = (n + kThreads - 1) / kThreads, cap = 8L * num_sms();
  return (int)(blocks < cap ? blocks : cap);
}

#define FP_CHECK(cond, ...)     \
  do {                          \
    if (!(cond)) {              \
      dvd::set_error(__VA_ARGS__); \
      return -2;                \
    }                           \
  } while (0)

static inline bool aligned_to(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

}  // namespace
}  // namespace dvd

using namespace dvd;

extern "C" int dvd_flow_resize_cubic(const float* src, size_t src_bytes, float* dst, size_t dst_bytes, int B, int h, int w,
                                     int H, int W, void* stream) {
  FP_CHECK(src && dst, "dvd_flow_resize_cubic: null pointer");
  FP_CHECK(B >= 1 && h >= 1 && w >= 1 && H >= 1 && W >= 1, "dvd_flow_resize_cubic: bad shape B=%d h=%d w=%d H=%d W=%d", B, h,
           w, H, W);
  FP_CHECK(aligned_to(src, 8) && aligned_to(dst, 8), "dvd_flow_resize_cubic: flows must be 8-byte aligned (float2 pixels)");
  const size_t need_src = (size_t)B * h * w * 2 * sizeof(float), need_dst = (size_t)B * H * W * 2 * sizeof(float);
  FP_CHECK(src_bytes == need_src && dst_bytes == need_dst,
           "dvd_flow_resize_cubic: buffer sizes %zu / %zu bytes, expected %zu / %zu for [%d,%d,%d,2] -> [%d,%d,%d,2] fp32",
           src_bytes, dst_bytes, need_src, need_dst, B, h, w, B, H, W);
  const long n = (long)B * H * W;
  // cv2.resize: inv_scale = dsize / ssize, scale = 1 / inv_scale (both double); resize_flow multiplies by dsize / ssize
  const double isx = (double)W / w, isy = (double)H / h;
  DVD_CUDA_CALL(launch(flow_resize_cubic_kernel, dim3(grid_for(n)), dim3(kThreads), 0, (cudaStream_t)stream,
                       reinterpret_cast<const float2*>(src), reinterpret_cast<float2*>(dst), n, h, w, H, W, 1.0 / isx, 1.0 / isy,
                       (double)W / (double)w, (double)H / (double)h));
  return 0;
}

extern "C" int dvd_flow_pair_masks(const float* flow_1_2, const float* flow_2_1, size_t flow_bytes, void* mask_1, void* mask_2,
                                   size_t mask_bytes, int B, int H, int W, int convention, void* stream) {
  FP_CHECK(flow_1_2 && flow_2_1 && mask_1 && mask_2, "dvd_flow_pair_masks: null pointer");
  FP_CHECK(convention == DVD_MASKS_FLOWPAIR_U8 || convention == DVD_MASKS_PAIRFILE_F32,
           "dvd_flow_pair_masks: convention must be DVD_MASKS_FLOWPAIR_U8 (0) or DVD_MASKS_PAIRFILE_F32 (1), got %d", convention);
  FP_CHECK(B >= 1 && H >= 2 && W >= 2, "dvd_flow_pair_masks: bad shape B=%d H=%d W=%d (H, W >= 2)", B, H, W);
  const bool f32 = convention == DVD_MASKS_PAIRFILE_F32;
  FP_CHECK(aligned_to(flow_1_2, 8) && aligned_to(flow_2_1, 8), "dvd_flow_pair_masks: flows must be 8-byte aligned (float2 pixels)");
  FP_CHECK(!f32 || (aligned_to(mask_1, 4) && aligned_to(mask_2, 4)), "dvd_flow_pair_masks: fp32 masks must be 4-byte aligned");
  const long n = (long)B * H * W;
  const size_t need_flow = (size_t)n * 2 * sizeof(float), need_mask = (size_t)n * (f32 ? sizeof(float) : 1);
  FP_CHECK(flow_bytes == need_flow && mask_bytes == need_mask,
           "dvd_flow_pair_masks: buffer sizes %zu / %zu bytes, expected %zu / %zu for B=%d H=%d W=%d", flow_bytes, mask_bytes,
           need_flow, need_mask, B, H, W);
  // (W - 1) / 2 is an integer or a half: exact in fp32, as in the reference's `sample_grids[..., 0] /= (W - 1) / 2`
  const float half_w = 0.5f * (float)(W - 1), half_h = 0.5f * (float)(H - 1);
  auto kernel = f32 ? flow_pair_masks_kernel<true> : flow_pair_masks_kernel<false>;
  DVD_CUDA_CALL(launch(kernel, dim3(grid_for(n)), dim3(kThreads), 0, (cudaStream_t)stream, reinterpret_cast<const float2*>(flow_1_2),
                       reinterpret_cast<const float2*>(flow_2_1), mask_1, mask_2, n, H, W, half_w, half_h));
  return 0;
}
