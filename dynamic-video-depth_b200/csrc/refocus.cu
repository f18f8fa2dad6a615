// Synthetic depth of field of a test export: each frame blurred by every pixel's distance, in disparity, from the frame's
// focal plane, with an exact gather rule so that the frames are bitwise reproducible.
//
// One CTA renders a 32 x 16 tile of one frame. It stages the tile and an R-pixel halo in shared memory as (disp, c, r, g, b),
// every value computed with each operation rounded on its own (no FMA contraction), then each thread walks its pixel's taps in
// row-major order and sums w col and w in that order. The CTA first reduces the largest blur radius c of its staged pixels,
// cmax, and walks only the taps with |dx|, |dy| <= L = min(R, ceil(cmax)) and dx^2 + dy^2 <= L^2 + L: any other tap has
// r >= L + 0.5 >= ce + 0.5 (ce <= c(q) <= cmax <= L), so its coverage rounds to 0 and the rule adds +0 for it, which changes no
// sum. Skipping it is therefore bit-exact, and sharp regions cost a handful of taps instead of the whole disc. No atomics, and
// no thread reads another's result.
#include <math.h>

#include "common.cuh"

namespace dvd {
namespace {

constexpr int kTileW = 32;  // one warp per tile row: the lanes of a warp share their tap bounds except at image edges
constexpr int kTileH = 16;
constexpr int kThreads = kTileW * kTileH;
constexpr int kWarps = kThreads / 32;

#define RF_CHECK(cond, ...)        \
  do {                             \
    if (!(cond)) {                 \
      dvd::set_error(__VA_ARGS__); \
      return -2;                   \
    }                              \
  } while (0)

// staged planes (disp, c, r, g, b), the tap-distance table sqrt(n) for n <= R^2, the per-warp maxima of c
size_t smem_bytes(int R) {
  const size_t S = (size_t)(kTileW + 2 * R) * (kTileH + 2 * R);
  return (5 * S + (size_t)R * R + 1 + kWarps) * sizeof(float);
}

// the depth2disp validity of points.cu: finite and > 1e-2; an invalid pixel is infinitely far
__device__ __forceinline__ float disparity(float d) { return (isfinite(d) && d > 1e-2f) ? __fdiv_rn(1.f, d) : 0.f; }

// clip(v, 0, 1) with NaN -> 0 (fmaxf returns the non-NaN operand)
__device__ __forceinline__ float colour(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

__device__ __forceinline__ unsigned char to_byte(float s, float w) {
  return (unsigned char)fminf(floorf(__fmul_rn(255.f, __fdiv_rn(s, w))), 255.f);
}

__global__ void __launch_bounds__(kThreads, 1) refocus_kernel(const float* __restrict__ depth, const float* __restrict__ img,
                                                              const float* __restrict__ focus_disp, float scale, int R, int H,
                                                              int W, int tiles_x, unsigned char* __restrict__ out) {
  DVD_PDL_ENTER();
  extern __shared__ float sm[];
  const int SW = kTileW + 2 * R, S = SW * (kTileH + 2 * R);
  float* s_disp = sm;
  float* s_c = sm + S;
  float* s_col = sm + 2 * S;  // r, g, b planes
  float* s_rtab = sm + 5 * S;
  unsigned int* s_max = reinterpret_cast<unsigned int*>(s_rtab + R * R + 1);

  const int f = blockIdx.y;
  const int tx0 = (blockIdx.x % tiles_x) * kTileW, ty0 = (blockIdx.x / tiles_x) * kTileH;
  const long long HW = (long long)H * W;
  const float* dep = depth + f * HW;
  const float* im = img + f * 3 * HW;
  const float phi = __ldg(focus_disp + f);
  const float Rf = (float)R;

  for (int n = threadIdx.x; n <= R * R; n += kThreads) s_rtab[n] = __fsqrt_rn((float)n);
  // c >= 0 and never NaN (fminf returns R for a NaN product), so its bits order like its value
  unsigned int cmax = 0;
  for (int i = threadIdx.x; i < S; i += kThreads) {
    const int sy = i / SW, sx = i - sy * SW;
    const int gy = ty0 - R + sy, gx = tx0 - R + sx;
    float dp = 0.f, c = 0.f, r = 0.f, g = 0.f, b = 0.f;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
      const long long o = (long long)gy * W + gx;
      dp = disparity(__ldg(dep + o));
      c = fminf(Rf, __fmul_rn(scale, fabsf(__fsub_rn(dp, phi))));
      r = colour(__ldg(im + o));
      g = colour(__ldg(im + HW + o));
      b = colour(__ldg(im + 2 * HW + o));
    }
    s_disp[i] = dp;
    s_c[i] = c;
    s_col[i] = r;
    s_col[S + i] = g;
    s_col[2 * S + i] = b;
    cmax = max(cmax, __float_as_uint(c));
  }
  cmax = __reduce_max_sync(0xffffffffu, cmax);
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = cmax;
  __syncthreads();
#pragma unroll
  for (int w = 0; w < kWarps; ++w) cmax = max(cmax, s_max[w]);
  const int L = min(R, (int)ceilf(__uint_as_float(cmax)));
  const int nmax = min(R * R, L * L + L);

  const int lx = threadIdx.x % kTileW, ly = threadIdx.x / kTileW;
  const int px = tx0 + lx, py = ty0 + ly;
  if (px >= W || py >= H) return;
  const int ci = (ly + R) * SW + lx + R;
  const float dp = s_disp[ci], cp = s_c[ci];
  float sr = 0.f, sg = 0.f, sb = 0.f, sw = 0.f;
  const int dy_lo = max(-L, -py), dy_hi = min(L, H - 1 - py);
  for (int dy = dy_lo; dy <= dy_hi; ++dy) {
    const int rem = nmax - dy * dy;  // >= 0: |dy| <= L and nmax >= L^2 unless nmax = R^2 >= L^2
    int half = (int)sqrtf((float)rem);
    while (half * half > rem) --half;
    while ((half + 1) * (half + 1) <= rem) ++half;
    const int dx_lo = max(-half, -px), dx_hi = min(half, W - 1 - px);
    const int row = ci + dy * SW;
    const float* rt = s_rtab + dy * dy;
    for (int dx = dx_lo; dx <= dx_hi; ++dx) {
      const int q = row + dx;
      const float dq = s_disp[q], cq = s_c[q];
      const float ce = dq < dp ? fminf(cq, cp) : cq;
      const float cov = fminf(fmaxf(__fadd_rn(__fsub_rn(ce, rt[dx * dx]), 0.5f), 0.f), 1.f);
      if (cov > 0.f) {  // a tap of zero coverage adds +0 to every sum
        const float w = __fdiv_rn(cov, fmaxf(__fmul_rn(ce, ce), 0.25f));
        sr = __fadd_rn(sr, __fmul_rn(w, s_col[q]));
        sg = __fadd_rn(sg, __fmul_rn(w, s_col[S + q]));
        sb = __fadd_rn(sb, __fmul_rn(w, s_col[2 * S + q]));
        sw = __fadd_rn(sw, w);
      }
    }
  }
  // the centre tap has coverage >= 0.5 and a finite weight, so sw > 0
  unsigned char* o = out + 3 * (f * HW + (long long)py * W + px);
  o[0] = to_byte(sb, sw);
  o[1] = to_byte(sg, sw);
  o[2] = to_byte(sr, sw);
}

}  // namespace
}  // namespace dvd

using namespace dvd;

extern "C" int dvd_refocus(const float* depth, const float* img, const float* focus_disp, float scale, int max_radius,
                           unsigned char* out, int N, int H, int W, void* stream) {
  RF_CHECK(depth && img && focus_disp && out, "dvd_refocus: null pointer");
  RF_CHECK(N >= 1 && N <= 65535 && H >= 1 && W >= 1, "dvd_refocus: bad shape N=%d H=%d W=%d (1 <= N <= 65535)", N, H, W);
  RF_CHECK(max_radius >= 0 && max_radius <= DVD_REFOCUS_MAX_RADIUS, "dvd_refocus: max_radius %d outside [0, %d]", max_radius,
           DVD_REFOCUS_MAX_RADIUS);
  RF_CHECK(isfinite(scale) && scale >= 0.f, "dvd_refocus: scale %g must be finite and >= 0", (double)scale);
  const long long tiles_x = (W + kTileW - 1) / kTileW, tiles = tiles_x * ((H + kTileH - 1) / kTileH);
  RF_CHECK(tiles <= 0x7fffffffLL, "dvd_refocus: %d x %d frames are too large for one launch", H, W);
  const size_t smem = smem_bytes(max_radius);
  DVD_CUDA_CALL(cudaFuncSetAttribute(refocus_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  DVD_CUDA_CALL(launch(refocus_kernel, dim3((unsigned)tiles, (unsigned)N), dim3(kThreads), smem, (cudaStream_t)stream, depth, img,
                       focus_disp, scale, max_radius, H, W, (int)tiles_x, out));
  return 0;
}
