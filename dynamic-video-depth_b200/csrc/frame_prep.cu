// Frame preparation: the GPU side of scripts/preprocess/{davis,shutterstock}/generate_frame_midas.py. MiDaS's bicubic resizes
// around the depth engine, scipy's order-3 spline (prefilter + sampling, mode 'constant') for the DAVIS scale calibration's
// point selection and depth look-up, the ShutterStock calibration's dense per-pixel ratios, the per-frame median of the
// ratios, and skimage's anti-aliased resize (gaussian_filter, then zoom(order=1, mode='mirror', grid_mode=True), then clip)
// for the working-size outputs.
//
// The scipy stages accumulate in fp64 and round where scipy stores (fp32 arrays between passes, fp32 output of
// map_coordinates on an fp32 input); additions and products are rounded one by one (__dadd_rn / __dmul_rn), as the
// library's C code does them, so that no contraction changes the order of rounding.
#include <limits.h>
#include <math.h>

#include "common.cuh"

namespace dvd {
namespace {

constexpr int kThreads = 256;

int grid_for(long n) {
  const long blocks = (n + kThreads - 1) / kThreads, cap = 8L * num_sms();
  return (int)(blocks < cap ? blocks : cap);
}

#define FR_CHECK(cond, ...)        \
  do {                             \
    if (!(cond)) {                 \
      dvd::set_error(__VA_ARGS__); \
      return -2;                   \
    }                              \
  } while (0)

// ---- F.interpolate(mode='bicubic', align_corners=True): ATen's upsample_bicubic2d, A = -0.75, taps clamped ---------------
__device__ __forceinline__ float cubic_conv1(float x, float A) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic_conv2(float x, float A) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }
__device__ __forceinline__ float cubic_interp(float x0, float x1, float x2, float x3, float t) {
  const float A = -0.75f;
  const float u = 1.f - t;
  const float c0 = cubic_conv2(t + 1.f, A), c1 = cubic_conv1(t, A), c2 = cubic_conv1(u, A), c3 = cubic_conv2(u + 1.f, A);
  return x0 * c0 + x1 * c1 + x2 * c2 + x3 * c3;
}

__global__ void __launch_bounds__(kThreads) bicubic_ac_kernel(const float* __restrict__ src, float* __restrict__ dst, long n, int h,
                                                               int w, int H, int W, float sy, float sx) {
  DVD_PDL_ENTER();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const long r = i / W;
    const int y = (int)(r % H);
    const float* plane = src + (r / H) * h * w;
    if (h == H && w == W) {
      dst[i] = __ldg(plane + (long)y * w + x);
      continue;
    }
    const float ry = sy * (float)y, rx = sx * (float)x;
    const int iy = (int)floorf(ry), ix = (int)floorf(rx);
    const float ty = ry - (float)iy, tx = rx - (float)ix;
    int xs[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) xs[k] = min(max(ix - 1 + k, 0), w - 1);
    float rows[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float* row = plane + (long)min(max(iy - 1 + k, 0), h - 1) * w;
      rows[k] = cubic_interp(__ldg(row + xs[0]), __ldg(row + xs[1]), __ldg(row + xs[2]), __ldg(row + xs[3]), tx);
    }
    dst[i] = cubic_interp(rows[0], rows[1], rows[2], rows[3], ty);
  }
}

// ---- scipy.ndimage.spline_filter(order=3, mode='constant'): one fp64 recursive pass per line, axis 0 then axis 1 --------
// The constant mode's prefilter uses the mirror boundary (causal sum over the mirrored line, closed-form anti-causal start).
__device__ void spline_line(double* c, long n, long stride) {
  if (n < 2) return;
  const double z = sqrt(3.0) - 2.0;
  const double gain = __dmul_rn(1.0 - z, 1.0 - 1.0 / z);
  for (long i = 0; i < n; ++i) c[i * stride] = __dmul_rn(c[i * stride], gain);
  const double zn1 = pow(z, (double)(n - 1));
  double c0 = __dadd_rn(c[0], __dmul_rn(zn1, c[(n - 1) * stride]));
  double zi = z;
  for (long i = 1; i < n - 1; ++i) {
    c0 = __dadd_rn(c0, __dmul_rn(zi, __dadd_rn(c[i * stride], __dmul_rn(zn1, c[(n - 1 - i) * stride]))));
    zi = __dmul_rn(zi, z);
  }
  c[0] = c0 / (1.0 - zn1 * zn1);
  for (long i = 1; i < n; ++i) c[i * stride] = __dadd_rn(c[i * stride], __dmul_rn(z, c[(i - 1) * stride]));
  c[(n - 1) * stride] = __dmul_rn(__dadd_rn(__dmul_rn(z, c[(n - 2) * stride]), c[(n - 1) * stride]), z) / (z * z - 1.0);
  for (long i = n - 2; i >= 0; --i) c[i * stride] = __dmul_rn(z, __dsub_rn(c[(i + 1) * stride], c[i * stride]));
}

// axis 0: one thread per column (consecutive threads read consecutive addresses); converts the fp32 map on the way
__global__ void __launch_bounds__(kThreads) spline_axis0_kernel(const float* __restrict__ src, double* __restrict__ coef, int N, int H,
                                                                 int W) {
  DVD_PDL_ENTER();
  const long n = (long)N * W;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long base = (i / W) * H * W + i % W;
    for (int y = 0; y < H; ++y) coef[base + (long)y * W] = (double)__ldg(src + base + (long)y * W);
    spline_line(coef + base, H, W);
  }
}

__global__ void __launch_bounds__(kThreads) spline_axis1_kernel(double* __restrict__ coef, int N, int H, int W) {
  DVD_PDL_ENTER();
  const long n = (long)N * H;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    spline_line(coef + i * W, W, 1);
}

// ---- map_coordinates(order=3, mode='constant', cval=0) of an fp32 map at (v, u), from the fp64 coefficients ---------------
// Coordinates outside [0, n-1] on either axis (NaN and inf included) give cval; inside, the taps past the border read the
// mirrored coefficients. Sum: Σ_i Σ_j (c[i][j] · wy[i]) · wx[j], i outer, as scipy's tap loop; the result is stored as fp32.
__device__ __forceinline__ int mirror_index(int i, int n) {
  if (n == 1) return 0;
  const int p = 2 * (n - 1);
  i = abs(i) % p;
  return i >= n ? p - i : i;
}

__device__ __forceinline__ void bspline3_weights(double t, double w[4]) {
  double y = t;
  w[1] = __dsub_rn(2.0 / 3.0, __dmul_rn(__dmul_rn(__dmul_rn(0.5, y), y), __dsub_rn(2.0, y)));
  y = __dsub_rn(1.0, t);
  w[2] = __dsub_rn(2.0 / 3.0, __dmul_rn(__dmul_rn(__dmul_rn(0.5, y), y), __dsub_rn(2.0, y)));
  w[0] = __dmul_rn(__dmul_rn(y, y), y) / 6.0;
  w[3] = __dsub_rn(__dsub_rn(__dsub_rn(1.0, w[0]), w[1]), w[2]);
}

__device__ float spline_sample(const double* __restrict__ coef, int H, int W, double v, double u) {
  if (!(v >= 0.0 && v <= (double)(H - 1) && u >= 0.0 && u <= (double)(W - 1))) return 0.f;
  const double fv = floor(v), fu = floor(u);
  double wv[4], wu[4];
  bspline3_weights(__dsub_rn(v, fv), wv);
  bspline3_weights(__dsub_rn(u, fu), wu);
  int xs[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) xs[j] = mirror_index((int)fu - 1 + j, W);
  double t = 0.0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const double* row = coef + (long)mirror_index((int)fv - 1 + i, H) * W;
#pragma unroll
    for (int j = 0; j < 4; ++j) t = __dadd_rn(t, __dmul_rn(__dmul_rn(__ldg(row + xs[j]), wv[i]), wu[j]));
  }
  return (float)t;
}

__global__ void __launch_bounds__(kThreads) spline_sample_kernel(const double* __restrict__ coef, const double2* __restrict__ vu,
                                                                  float* __restrict__ out, int N, int H, int W, long P) {
  DVD_PDL_ENTER();
  const long n = (long)N * P;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const double2 c = vu[i];
    out[i] = spline_sample(coef + (i / P) * H * W, H, W, c.x, c.y);
  }
}

// A positive quiet NaN: a device sort orders by bit pattern, and CUDART_NAN's sign bit would put rejected points first.
__device__ __forceinline__ double positive_nan() { return __longlong_as_double(0x7ff8000000000000LL); }

// ---- scale calibration: one thread per (frame, vertex) ---------------------------------------------------------------------
// out = E X (fp64), im = K out[:3], depth = im.z, (u, v) = im.xy / im.z; kept when 0 <= u < W and 0 <= v < H, then when the
// mask's spline value is < 0.1f, then when depth > 1e-3. ratio = (double)nn / depth with nn the depth map's fp32 spline value.
__device__ __forceinline__ double dot4(const double* e, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[0], x), __dmul_rn(e[1], y)), __dmul_rn(e[2], z)), e[3]);
}

__global__ void __launch_bounds__(kThreads) calib_ratio_kernel(const double* __restrict__ dcoef, const double* __restrict__ mcoef,
                                                                const double* __restrict__ E, const double* __restrict__ pts,
                                                                double* __restrict__ ratio, int N, int H, int W, long V, double fx,
                                                                double fy, double cx, double cy) {
  DVD_PDL_ENTER();
  const long n = (long)N * V;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long f = i / V, p = i % V;
    const double* e = E + f * 16;
    const double X = pts[p * 3], Y = pts[p * 3 + 1], Z = pts[p * 3 + 2];
    const double o0 = dot4(e, X, Y, Z), o1 = dot4(e + 4, X, Y, Z), o2 = dot4(e + 8, X, Y, Z);
    const double depth = o2;
    const double u = __dadd_rn(__dmul_rn(fx, o0), __dmul_rn(cx, o2)) / o2;
    const double v = __dadd_rn(__dmul_rn(fy, o1), __dmul_rn(cy, o2)) / o2;
    double r = positive_nan();
    if (u >= 0.0 && u < (double)W && v >= 0.0 && v < (double)H) {
      const long off = f * H * W;
      if (spline_sample(mcoef + off, H, W, v, u) < 0.1f && depth > 1e-3)
        r = (double)spline_sample(dcoef + off, H, W, v, u) / depth;
    }
    ratio[i] = r;
  }
}

__device__ __forceinline__ float positive_nan_f() { return __int_as_float(0x7fc00000); }

// ---- dense scale calibration (shutterstock/generate_frame_midas.py): ratio = nn / mvs where mvs > 1e-3 ---------------------
// numpy's arithmetic for an fp32 MiDaS map nn and an MVS map of the stored dtype: for fp32 maps the threshold is 1e-3 rounded
// to fp32 and the quotient is fp32; for fp64 maps nn is widened and the quotient is fp64. Elsewhere (NaN included) a positive
// NaN, so that a device sort puts the rejected pixels last.
__device__ __forceinline__ float dense_ratio(float nn, float m) { return m > 1e-3f ? __fdiv_rn(nn, m) : positive_nan_f(); }
__device__ __forceinline__ double dense_ratio(float nn, double m) { return m > 1e-3 ? __ddiv_rn((double)nn, m) : positive_nan(); }

__device__ __forceinline__ void load4(const float* p, float v[4]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w;
}
__device__ __forceinline__ void load4(const double* p, double v[4]) {
  const double2 a = __ldg(reinterpret_cast<const double2*>(p)), b = __ldg(reinterpret_cast<const double2*>(p) + 1);
  v[0] = a.x, v[1] = a.y, v[2] = b.x, v[3] = b.y;
}
__device__ __forceinline__ void store4(float* p, const float v[4]) { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }
__device__ __forceinline__ void store4(double* p, const double v[4]) {
  reinterpret_cast<double2*>(p)[0] = make_double2(v[0], v[1]);
  reinterpret_cast<double2*>(p)[1] = make_double2(v[2], v[3]);
}

// one pass over the flat [N*HW] maps: groups of four elements with 16-byte loads when every base is 16-byte aligned, then the
// remainder one element per thread
template <typename M>
__global__ void __launch_bounds__(kThreads) dense_ratio_kernel(const float* __restrict__ nn, const M* __restrict__ mvs,
                                                                M* __restrict__ ratio, long n, int vec) {
  DVD_PDL_ENTER();
  const long tid = (long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long)gridDim.x * blockDim.x;
  long done = 0;
  if (vec) {
    const long nv = n / 4;
    for (long i = tid; i < nv; i += stride) {
      float a[4];
      M b[4], r[4];
      load4(nn + 4 * i, a);
      load4(mvs + 4 * i, b);
#pragma unroll
      for (int k = 0; k < 4; ++k) r[k] = dense_ratio(a[k], b[k]);
      store4(ratio + 4 * i, r);
    }
    done = nv * 4;
  }
  for (long i = done + tid; i < n; i += stride) ratio[i] = dense_ratio(__ldg(nn + i), __ldg(mvs + i));
}

// np.median of each row's non-NaN entries, the row sorted ascending with NaN last: middle element, or the mean of the two
// middle ones for an even count, (a + b) / 2 with the sum rounded to T as numpy's mean does; count[f] = number of non-NaN
// entries (median NaN when 0). One thread per frame.
__device__ __forceinline__ double mid_mean(double a, double b) { return __dadd_rn(a, b) / 2.0; }
__device__ __forceinline__ float mid_mean(float a, float b) { return __fdiv_rn(__fadd_rn(a, b), 2.f); }
__device__ __forceinline__ void set_nan(double* p) { *p = positive_nan(); }
__device__ __forceinline__ void set_nan(float* p) { *p = positive_nan_f(); }

template <typename T>
__global__ void sorted_median_kernel(const T* __restrict__ sorted, T* __restrict__ med, int* __restrict__ count, int N, long V) {
  DVD_PDL_ENTER();
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= N) return;
  const T* row = sorted + (long)f * V;
  long lo = 0, hi = V;  // first NaN
  while (lo < hi) {
    const long mid = (lo + hi) / 2;
    if (isnan(row[mid])) hi = mid;
    else lo = mid + 1;
  }
  count[f] = (int)lo;
  if (lo == 0) set_nan(med + f);
  else if (lo & 1) med[f] = row[lo / 2];
  else med[f] = mid_mean(row[lo / 2 - 1], row[lo / 2]);
}

// ---- skimage.transform.resize(order=1, mode='reflect', anti_aliasing=True, preserve_range=True) on fp32 [N,H,W,C] ---------
// per-frame min / max of the input (the clip bounds); one block per frame, fixed order
__global__ void __launch_bounds__(kThreads) minmax_kernel(const float* __restrict__ src, float* __restrict__ bounds, long m) {
  DVD_PDL_ENTER();
  __shared__ float smin[kThreads], smax[kThreads];
  const float* p = src + (long)blockIdx.x * m;
  float lo = INFINITY, hi = -INFINITY;
  for (long i = threadIdx.x; i < m; i += kThreads) {
    const float x = __ldg(p + i);
    lo = fminf(lo, x);
    hi = fmaxf(hi, x);
  }
  smin[threadIdx.x] = lo;
  smax[threadIdx.x] = hi;
  __syncthreads();
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      smin[threadIdx.x] = fminf(smin[threadIdx.x], smin[threadIdx.x + s]);
      smax[threadIdx.x] = fmaxf(smax[threadIdx.x], smax[threadIdx.x + s]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    bounds[2 * blockIdx.x] = smin[0];
    bounds[2 * blockIdx.x + 1] = smax[0];
  }
}

// gaussian_filter1d along one axis (line length L, element stride S within a line) with mode 'mirror': scipy's symmetric
// correlate1d, acc = x[0] w[r] + Σ_{j=1..r} (x[-j] + x[j]) w[r-j], in fp64, stored as fp32
__global__ void __launch_bounds__(kThreads) gauss_axis_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                               const double* __restrict__ w, int r, long n, int L, long S) {
  DVD_PDL_ENTER();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int pos = (int)((i / S) % L);
    const float* line = src + (i - (long)pos * S);
    double acc = __dmul_rn((double)__ldg(line + (long)pos * S), w[r]);
    for (int j = -r; j < 0; ++j) {
      const double a = (double)__ldg(line + (long)mirror_index(pos + j, L) * S);
      const double b = (double)__ldg(line + (long)mirror_index(pos - j, L) * S);
      acc = __dadd_rn(acc, __dmul_rn(__dadd_rn(a, b), w[r + j]));
    }
    dst[i] = (float)acc;
  }
}

// zoom(order=1, mode='mirror', grid_mode=True) source position along one axis: c = (o + 0.5) zoom - 0.5 mirrored into
// [0, n-1]; taps k0 = floor(c), k1 = mirror(k0 + 1) with weights 1 - t, t
__device__ __forceinline__ void linear_src(int o, double zoom, int n, int* k0, int* k1, double* w0, double* w1) {
  double c = __dsub_rn(__dmul_rn((double)o + 0.5, zoom), 0.5);
  if (n <= 1) {
    c = 0.0;
  } else {
    const double p = 2.0 * (double)(n - 1);
    if (c < 0.0) {
      c = __dadd_rn(p * (double)(long)(-c / p), c);
      c = c <= (double)(1 - n) ? c + p : -c;
    } else if (c > (double)(n - 1)) {
      c = __dsub_rn(c, p * (double)(long)(c / p));
      if (c >= (double)n) c = p - c;
    }
  }
  const double f = floor(c);
  const double t = __dsub_rn(c, f);
  *k0 = mirror_index((int)f, n);
  *k1 = mirror_index((int)f + 1, n);
  *w0 = __dsub_rn(1.0, t);
  *w1 = t;
}

__global__ void __launch_bounds__(kThreads) zoom_clip_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                              const float* __restrict__ bounds, long n, int H, int W, int C, int OH,
                                                              int OW, double zy, double zx) {
  DVD_PDL_ENTER();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long r = i / C;
    const int ox = (int)(r % OW);
    r /= OW;
    const int oy = (int)(r % OH);
    const long f = r / OH;
    int y0, y1, x0, x1;
    double wy0, wy1, wx0, wx1;
    linear_src(oy, zy, H, &y0, &y1, &wy0, &wy1);
    linear_src(ox, zx, W, &x0, &x1, &wx0, &wx1);
    const float* p = src + f * H * W * C + c;
    const double v00 = __ldg(p + ((long)y0 * W + x0) * C), v01 = __ldg(p + ((long)y0 * W + x1) * C);
    const double v10 = __ldg(p + ((long)y1 * W + x0) * C), v11 = __ldg(p + ((long)y1 * W + x1) * C);
    double t = __dmul_rn(__dmul_rn(v00, wy0), wx0);
    t = __dadd_rn(t, __dmul_rn(__dmul_rn(v01, wy0), wx1));
    t = __dadd_rn(t, __dmul_rn(__dmul_rn(v10, wy1), wx0));
    t = __dadd_rn(t, __dmul_rn(__dmul_rn(v11, wy1), wx1));
    // np.clip(out, min, max) = minimum(maximum(out, min), max)
    dst[i] = fminf(fmaxf((float)t, bounds[2 * f]), bounds[2 * f + 1]);
  }
}

static inline bool aligned_to(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

}  // namespace
}  // namespace dvd

using namespace dvd;

extern "C" int dvd_resize_bicubic_ac(const float* src, size_t src_bytes, float* dst, size_t dst_bytes, int NC, int h, int w, int H,
                                     int W, void* stream) {
  FR_CHECK(src && dst, "dvd_resize_bicubic_ac: null pointer");
  FR_CHECK(NC >= 1 && h >= 1 && w >= 1 && H >= 1 && W >= 1, "dvd_resize_bicubic_ac: bad shape NC=%d h=%d w=%d H=%d W=%d", NC, h, w,
           H, W);
  const size_t need_src = (size_t)NC * h * w * sizeof(float), need_dst = (size_t)NC * H * W * sizeof(float);
  FR_CHECK(src_bytes == need_src && dst_bytes == need_dst, "dvd_resize_bicubic_ac: buffer sizes %zu / %zu bytes, expected %zu / %zu",
           src_bytes, dst_bytes, need_src, need_dst);
  // ATen's area_pixel_compute_scale with align_corners: (in - 1) / (out - 1) in fp32, 0 for a single output
  const float sy = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, sx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
  const long n = (long)NC * H * W;
  DVD_CUDA_CALL(launch(bicubic_ac_kernel, dim3(grid_for(n)), dim3(kThreads), 0, (cudaStream_t)stream, src, dst, n, h, w, H, W, sy, sx));
  return 0;
}

extern "C" int dvd_spline_prefilter(const float* maps, size_t maps_bytes, double* coef, size_t coef_bytes, int N, int H, int W,
                                    void* stream) {
  FR_CHECK(maps && coef, "dvd_spline_prefilter: null pointer");
  FR_CHECK(N >= 1 && H >= 1 && W >= 1, "dvd_spline_prefilter: bad shape N=%d H=%d W=%d", N, H, W);
  FR_CHECK(aligned_to(coef, 8), "dvd_spline_prefilter: coefficients must be 8-byte aligned");
  const size_t m = (size_t)N * H * W;
  FR_CHECK(maps_bytes == m * sizeof(float) && coef_bytes == m * sizeof(double),
           "dvd_spline_prefilter: buffer sizes %zu / %zu bytes, expected %zu / %zu for [%d,%d,%d]", maps_bytes, coef_bytes,
           m * sizeof(float), m * sizeof(double), N, H, W);
  cudaStream_t st = (cudaStream_t)stream;
  DVD_CUDA_CALL(launch(spline_axis0_kernel, dim3(grid_for((long)N * W)), dim3(kThreads), 0, st, maps, coef, N, H, W));
  DVD_CUDA_CALL(launch(spline_axis1_kernel, dim3(grid_for((long)N * H)), dim3(kThreads), 0, st, coef, N, H, W));
  return 0;
}

extern "C" int dvd_spline_sample(const double* coef, size_t coef_bytes, int N, int H, int W, const double* vu, float* out, long P,
                                 void* stream) {
  FR_CHECK(coef && vu && out, "dvd_spline_sample: null pointer");
  FR_CHECK(N >= 1 && H >= 1 && W >= 1 && P >= 1, "dvd_spline_sample: bad shape N=%d H=%d W=%d P=%ld", N, H, W, P);
  FR_CHECK(aligned_to(coef, 8) && aligned_to(vu, 16), "dvd_spline_sample: coefficients 8-byte, coordinates 16-byte aligned");
  FR_CHECK(coef_bytes == (size_t)N * H * W * sizeof(double), "dvd_spline_sample: coefficient buffer %zu bytes, expected %zu",
           coef_bytes, (size_t)N * H * W * sizeof(double));
  const long n = (long)N * P;
  DVD_CUDA_CALL(launch(spline_sample_kernel, dim3(grid_for(n)), dim3(kThreads), 0, (cudaStream_t)stream, coef,
                       reinterpret_cast<const double2*>(vu), out, N, H, W, P));
  return 0;
}

extern "C" int dvd_calib_ratios(const double* depth_coef, const double* mask_coef, size_t coef_bytes, const double* w2c,
                                const double* points, long V, double fx, double fy, double cx, double cy, double* ratio,
                                size_t ratio_bytes, int N, int H, int W, void* stream) {
  FR_CHECK(depth_coef && mask_coef && w2c && points && ratio, "dvd_calib_ratios: null pointer");
  FR_CHECK(N >= 1 && H >= 1 && W >= 1 && V >= 1, "dvd_calib_ratios: bad shape N=%d H=%d W=%d V=%ld", N, H, W, V);
  FR_CHECK(aligned_to(depth_coef, 8) && aligned_to(mask_coef, 8) && aligned_to(w2c, 8) && aligned_to(points, 8) &&
               aligned_to(ratio, 8),
           "dvd_calib_ratios: fp64 buffers must be 8-byte aligned");
  FR_CHECK(coef_bytes == (size_t)N * H * W * sizeof(double) && ratio_bytes == (size_t)N * V * sizeof(double),
           "dvd_calib_ratios: buffer sizes %zu / %zu bytes, expected %zu / %zu", coef_bytes, ratio_bytes,
           (size_t)N * H * W * sizeof(double), (size_t)N * V * sizeof(double));
  const long n = (long)N * V;
  DVD_CUDA_CALL(launch(calib_ratio_kernel, dim3(grid_for(n)), dim3(kThreads), 0, (cudaStream_t)stream, depth_coef, mask_coef, w2c,
                       points, ratio, N, H, W, V, fx, fy, cx, cy));
  return 0;
}

extern "C" int dvd_sorted_median(const double* sorted, size_t sorted_bytes, int N, long V, double* median, int* count, void* stream) {
  FR_CHECK(sorted && median && count, "dvd_sorted_median: null pointer");
  FR_CHECK(N >= 1 && V >= 1, "dvd_sorted_median: bad shape N=%d V=%ld", N, V);
  FR_CHECK(aligned_to(sorted, 8) && aligned_to(median, 8) && aligned_to(count, 4), "dvd_sorted_median: misaligned buffer");
  FR_CHECK(sorted_bytes == (size_t)N * V * sizeof(double), "dvd_sorted_median: buffer %zu bytes, expected %zu", sorted_bytes,
           (size_t)N * V * sizeof(double));
  DVD_CUDA_CALL(launch(sorted_median_kernel<double>, dim3((N + 127) / 128), dim3(128), 0, (cudaStream_t)stream, sorted, median, count,
                       N, V));
  return 0;
}

extern "C" int dvd_sorted_median_f32(const float* sorted, size_t sorted_bytes, int N, long V, float* median, int* count,
                                     void* stream) {
  FR_CHECK(sorted && median && count, "dvd_sorted_median_f32: null pointer");
  FR_CHECK(N >= 1 && V >= 1, "dvd_sorted_median_f32: bad shape N=%d V=%ld", N, V);
  FR_CHECK(V <= INT_MAX, "dvd_sorted_median_f32: rows of %ld entries overflow the int32 count", V);
  FR_CHECK(aligned_to(sorted, 4) && aligned_to(median, 4) && aligned_to(count, 4), "dvd_sorted_median_f32: misaligned buffer");
  FR_CHECK(sorted_bytes == (size_t)N * V * sizeof(float), "dvd_sorted_median_f32: buffer %zu bytes, expected %zu", sorted_bytes,
           (size_t)N * V * sizeof(float));
  DVD_CUDA_CALL(launch(sorted_median_kernel<float>, dim3((N + 127) / 128), dim3(128), 0, (cudaStream_t)stream, sorted, median, count,
                       N, V));
  return 0;
}

extern "C" int dvd_dense_ratios(const float* nn, size_t nn_bytes, const void* mvs, size_t mvs_bytes, int mvs_f64, void* ratio,
                                size_t ratio_bytes, int N, long HW, void* stream) {
  FR_CHECK(nn && mvs && ratio, "dvd_dense_ratios: null pointer");
  FR_CHECK(N >= 1 && HW >= 1 && (mvs_f64 == 0 || mvs_f64 == 1), "dvd_dense_ratios: bad arguments N=%d HW=%ld mvs_f64=%d", N, HW,
           mvs_f64);
  const size_t m = (size_t)N * HW, esz = mvs_f64 ? sizeof(double) : sizeof(float);
  FR_CHECK(aligned_to(nn, 4) && aligned_to(mvs, esz) && aligned_to(ratio, esz), "dvd_dense_ratios: misaligned buffer");
  FR_CHECK(nn_bytes == m * sizeof(float) && mvs_bytes == m * esz && ratio_bytes == m * esz,
           "dvd_dense_ratios: buffer sizes %zu / %zu / %zu bytes, expected %zu / %zu / %zu", nn_bytes, mvs_bytes, ratio_bytes,
           m * sizeof(float), m * esz, m * esz);
  const int vec = aligned_to(nn, 16) && aligned_to(mvs, 16) && aligned_to(ratio, 16);
  const long n = (long)m;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_for(vec ? (n + 3) / 4 : n);
  if (mvs_f64)
    DVD_CUDA_CALL(launch(dense_ratio_kernel<double>, dim3(grid), dim3(kThreads), 0, st, nn, (const double*)mvs, (double*)ratio, n, vec));
  else
    DVD_CUDA_CALL(launch(dense_ratio_kernel<float>, dim3(grid), dim3(kThreads), 0, st, nn, (const float*)mvs, (float*)ratio, n, vec));
  return 0;
}

extern "C" long dvd_aa_resize_scratch_bytes(int N, int H, int W, int C) {
  if (N < 1 || H < 1 || W < 1 || C < 1) return -1;
  return (2L * N * H * W * C + 2L * N) * (long)sizeof(float);
}

extern "C" int dvd_aa_resize(const float* src, size_t src_bytes, float* dst, size_t dst_bytes, void* scratch, size_t scratch_bytes,
                             const double* wy, int ry, const double* wx, int rx, int N, int H, int W, int C, int OH, int OW,
                             void* stream) {
  FR_CHECK(src && dst && scratch && wy && wx, "dvd_aa_resize: null pointer");
  FR_CHECK(N >= 1 && H >= 1 && W >= 1 && C >= 1 && OH >= 1 && OW >= 1 && ry >= 0 && rx >= 0,
           "dvd_aa_resize: bad shape N=%d H=%d W=%d C=%d -> %dx%d, radii %d / %d", N, H, W, C, OH, OW, ry, rx);
  FR_CHECK(aligned_to(src, 4) && aligned_to(dst, 4) && aligned_to(scratch, 4) && aligned_to(wy, 8) && aligned_to(wx, 8),
           "dvd_aa_resize: misaligned buffer");
  const long m = (long)H * W * C;
  FR_CHECK(src_bytes == (size_t)N * m * sizeof(float) && dst_bytes == (size_t)N * OH * OW * C * sizeof(float) &&
               (long)scratch_bytes == dvd_aa_resize_scratch_bytes(N, H, W, C),
           "dvd_aa_resize: buffer sizes %zu / %zu / %zu bytes, expected %zu / %zu / %ld", src_bytes, dst_bytes, scratch_bytes,
           (size_t)N * m * sizeof(float), (size_t)N * OH * OW * C * sizeof(float), dvd_aa_resize_scratch_bytes(N, H, W, C));
  float* t0 = static_cast<float*>(scratch);
  float* t1 = t0 + N * m;
  float* bounds = t1 + N * m;
  cudaStream_t st = (cudaStream_t)stream;
  const long n = N * m, n_out = (long)N * OH * OW * C;
  DVD_CUDA_CALL(launch(minmax_kernel, dim3(N), dim3(kThreads), 0, st, src, bounds, m));
  DVD_CUDA_CALL(launch(gauss_axis_kernel, dim3(grid_for(n)), dim3(kThreads), 0, st, src, t0, wy, ry, n, H, (long)W * C));
  DVD_CUDA_CALL(launch(gauss_axis_kernel, dim3(grid_for(n)), dim3(kThreads), 0, st, (const float*)t0, t1, wx, rx, n, W, (long)C));
  // numpy.divide(input.shape, output_shape): the zoom of grid mode
  DVD_CUDA_CALL(launch(zoom_clip_kernel, dim3(grid_for(n_out)), dim3(kThreads), 0, st, (const float*)t1, dst, (const float*)bounds,
                       n_out, H, W, C, OH, OW, (double)H / (double)OH, (double)W / (double)OW));
  return 0;
}
