// Novel-view rendering of a test export: world points splatted into virtual cameras with an exact, order-independent depth
// test, then resolved into BGR frames and per-frame coverage counts.
//
// dvd_splat_views projects points through fp32 world-to-camera blocks (w2c | K) with every product, sum and quotient rounded
// on its own (__fmul_rn, __fadd_rn, __fdiv_rn: no FMA contraction, as reproject.cu), and each covered pixel keeps the minimum
// of the 64-bit key (bits(q2) << 32) | index with atomicMin. A minimum does not depend on the order in which the candidates
// arrive, so the key buffer, and the frames resolved from it, are a pure function of the inputs. dvd_resolve_views reads the
// winning index back as a colour: below H W a pixel of the frame's own image, from H W on a point of the static cloud.
#include <math.h>

#include "common.cuh"

namespace dvd {
namespace {

constexpr int kThreads = 256;
constexpr unsigned long long kEmpty = ~0ull;

// w2c (3 x 4, row-major) then K (3 x 3, row-major) of one view
constexpr int kCam = DVD_VIEW_CAM_FLOATS;

// Key of a point seen from view `cam`, and the top-left pixel of its footprint; false when the point is dropped (behind the
// near plane, a non-finite coordinate, or a footprint wholly outside the image).
__device__ __forceinline__ bool project(const float* __restrict__ cam, float px, float py, float pz, int H, int W, int s,
                                        unsigned int* depth_bits, int* x0, int* y0) {
  float q[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float* w = cam + 4 * i;
    q[i] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__ldg(w), px), __fmul_rn(__ldg(w + 1), py)), __fmul_rn(__ldg(w + 2), pz)),
                     __ldg(w + 3));
  }
  float h[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float* k = cam + 12 + 3 * i;
    h[i] = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(k), q[0]), __fmul_rn(__ldg(k + 1), q[1])), __fmul_rn(__ldg(k + 2), q[2]));
  }
  if (!(q[2] > 0.01f) || !isfinite(q[0]) || !isfinite(q[1]) || !isfinite(q[2])) return false;
  const float u = __fdiv_rn(h[0], h[2]), v = __fdiv_rn(h[1], h[2]);
  if (!isfinite(u) || !isfinite(v)) return false;
  const float xf = floorf(__fadd_rn(u, 0.5f)), yf = floorf(__fadd_rn(v, 0.5f));
  const int half = (s - 1) / 2;
  // xf - half <= W - 1 and xf - half + s - 1 >= 0 for any pixel to be covered; the bounds keep the int conversion exact
  if (!(xf >= (float)(half - s + 1) && xf <= (float)(W - 1 + half) && yf >= (float)(half - s + 1) && yf <= (float)(H - 1 + half)))
    return false;
  *x0 = (int)xf - half;
  *y0 = (int)yf - half;
  *depth_bits = __float_as_uint(q[2]);  // positive and finite: orders like the value
  return true;
}

__device__ __forceinline__ void splat(unsigned long long* __restrict__ keys, unsigned long long key, int x0, int y0, int s, int H,
                                      int W) {
  for (int dy = 0; dy < s; ++dy) {
    const int y = y0 + dy;
    if (y < 0 || y >= H) continue;
    for (int dx = 0; dx < s; ++dx) {
      const int x = x0 + dx;
      if (x < 0 || x >= W) continue;
      unsigned long long* k = keys + (long long)y * W + x;
      // the stored key only decreases, so a stale read that is already <= key means the atomic could not change it
      if (key < __ldcg(k)) atomicMin(k, key);
    }
  }
}

// frame points: point p belongs to view index[p] / (H W) of the chunk and carries its pixel index index[p] % (H W)
__global__ void __launch_bounds__(kThreads) splat_frame_kernel(const float* __restrict__ xyz, const long long* __restrict__ index,
                                                               long long n, const float* __restrict__ cams, int H, int W, int s,
                                                               unsigned long long* __restrict__ keys) {
  DVD_PDL_ENTER();
  const long long p = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (p >= n) return;
  const long long HW = (long long)H * W;
  const long long i = __ldg(index + p);
  const long long f = i / HW;
  unsigned int zb;
  int x0, y0;
  if (!project(cams + f * kCam, __ldg(xyz + 3 * p), __ldg(xyz + 3 * p + 1), __ldg(xyz + 3 * p + 2), H, W, s, &zb, &x0, &y0)) return;
  splat(keys + f * HW, ((unsigned long long)zb << 32) | (unsigned long long)(i - f * HW), x0, y0, s, H, W);
}

// static points: one thread per (point, view) pair, view = blockIdx.y; point r carries the index H W + r
__global__ void __launch_bounds__(kThreads) splat_static_kernel(const float* __restrict__ xyz, long long n, const float* __restrict__ cams,
                                                                int H, int W, int s, unsigned long long* __restrict__ keys) {
  DVD_PDL_ENTER();
  const long long r = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (r >= n) return;
  const long long HW = (long long)H * W;
  const int f = blockIdx.y;
  unsigned int zb;
  int x0, y0;
  if (!project(cams + (long long)f * kCam, __ldg(xyz + 3 * r), __ldg(xyz + 3 * r + 1), __ldg(xyz + 3 * r + 2), H, W, s, &zb, &x0, &y0))
    return;
  splat(keys + f * HW, ((unsigned long long)zb << 32) | (unsigned long long)(HW + r), x0, y0, s, H, W);
}

// one thread per pixel, view = blockIdx.y; covered pixels are counted per block and added to coverage[f] (integer atomics:
// the count does not depend on their order)
__global__ void __launch_bounds__(kThreads) resolve_kernel(const unsigned long long* __restrict__ keys, const float* __restrict__ img,
                                                           const unsigned char* __restrict__ static_rgb, int H, int W,
                                                           unsigned char* __restrict__ out, int* __restrict__ coverage) {
  DVD_PDL_ENTER();
  __shared__ int warp_hits[kThreads / 32];
  const long long HW = (long long)H * W;
  const int f = blockIdx.y;
  const long long r = (long long)blockIdx.x * kThreads + threadIdx.x;
  bool hit = false;
  if (r < HW) {
    const unsigned long long k = __ldg(keys + f * HW + r);
    unsigned char b = 0, g = 0, R = 0;
    if (k != kEmpty) {
      hit = true;
      const long long i = (long long)(unsigned int)k;
      if (i < HW) {
        // floor(255 clip(v, 0, 1)) in fp32, NaN -> 0: the colour dvd_points_select gives the pixel
        const float* c = img + f * 3 * HW + i;
        R = (unsigned char)__fmul_rn(fminf(fmaxf(__ldg(c), 0.f), 1.f), 255.f);
        g = (unsigned char)__fmul_rn(fminf(fmaxf(__ldg(c + HW), 0.f), 1.f), 255.f);
        b = (unsigned char)__fmul_rn(fminf(fmaxf(__ldg(c + 2 * HW), 0.f), 1.f), 255.f);
      } else {
        const unsigned char* c = static_rgb + 3 * (i - HW);
        R = __ldg(c), g = __ldg(c + 1), b = __ldg(c + 2);
      }
    }
    unsigned char* o = out + 3 * (f * HW + r);
    o[0] = b, o[1] = g, o[2] = R;
  }
  const int n = __popc(__ballot_sync(0xffffffffu, hit));
  if ((threadIdx.x & 31) == 0) warp_hits[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < kThreads / 32; ++w) s += warp_hits[w];
    if (s) atomicAdd(coverage + f, s);
  }
}

}  // namespace
}  // namespace dvd

using namespace dvd;

extern "C" int dvd_splat_views(const float* xyz, const long long* index, long long n_points, const float* cams, int n_views, int H, int W,
                               int splat, unsigned long long* keys, void* stream) {
  DVD_ARG_CHECK(cams && keys && (n_points == 0 || xyz), "dvd_splat_views: null pointer");
  DVD_ARG_CHECK(n_points >= 0 && n_views >= 1 && H >= 1 && W >= 1, "dvd_splat_views: bad shape n_points=%lld n_views=%d H=%d W=%d",
                n_points, n_views, H, W);
  DVD_ARG_CHECK(n_views <= 65535, "dvd_splat_views: %d views, at most 65535 per call", n_views);
  DVD_ARG_CHECK(splat >= 1 && splat <= DVD_SPLAT_MAX, "dvd_splat_views: splat %d outside [1, %d]", splat, DVD_SPLAT_MAX);
  const long long HW = (long long)H * W;
  DVD_ARG_CHECK(index || HW + n_points <= 0xffffffffLL,
                "dvd_splat_views: H W + %lld static points reach 2^32, beyond the 32-bit index of a key", n_points);
  DVD_ARG_CHECK(HW <= 0xffffffffLL, "dvd_splat_views: %d x %d views exceed the 32-bit index of a key", H, W);
  if (n_points == 0) return 0;
  const long long blocks = (n_points + kThreads - 1) / kThreads;
  DVD_ARG_CHECK(blocks <= 0x7fffffffLL, "dvd_splat_views: %lld points are too many for one launch", n_points);
  cudaStream_t st = (cudaStream_t)stream;
  if (index) {
    DVD_CUDA_CALL(launch(splat_frame_kernel, dim3((unsigned)blocks), dim3(kThreads), 0, st, xyz, index, n_points, cams, H, W, splat, keys));
  } else {
    DVD_CUDA_CALL(launch(splat_static_kernel, dim3((unsigned)blocks, (unsigned)n_views), dim3(kThreads), 0, st, xyz, n_points, cams, H, W,
                         splat, keys));
  }
  return 0;
}

extern "C" int dvd_resolve_views(const unsigned long long* keys, const float* img, const unsigned char* static_rgb, int n_views, int H,
                                 int W, unsigned char* out, int* coverage, void* stream) {
  DVD_ARG_CHECK(keys && img && out && coverage, "dvd_resolve_views: null pointer");
  DVD_ARG_CHECK(n_views >= 1 && n_views <= 65535 && H >= 1 && W >= 1, "dvd_resolve_views: bad shape n_views=%d H=%d W=%d", n_views, H, W);
  const long long HW = (long long)H * W;
  const long long blocks = (HW + kThreads - 1) / kThreads;
  DVD_ARG_CHECK(blocks <= 0x7fffffffLL, "dvd_resolve_views: %d x %d views are too large for one launch", H, W);
  cudaStream_t st = (cudaStream_t)stream;
  DVD_CUDA_CALL(cudaMemsetAsync(coverage, 0, (size_t)n_views * sizeof(int), st));
  DVD_CUDA_CALL(launch(resolve_kernel, dim3((unsigned)blocks, (unsigned)n_views), dim3(kThreads), 0, st, keys, img, static_rgb, H, W, out,
                       coverage));
  return 0;
}
