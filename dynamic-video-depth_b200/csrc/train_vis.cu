// Training / validation page images: the PNGs the reference's HTMLVisualizer writes for one visualised pack
// (visualize/html_visualizer.py:98-116 over util/util_visualize.py and util/util_flow.py), rendered from the device tensors.
//
// Two launches per pack. dvd_vis_ranges reduces each image to its fp32 extrema (one CTA per image; min / max only, so the
// result does not depend on the reduction order). dvd_vis_tiles then writes every RGB tile; one thread owns 4 pixels of a row
// and writes each of their bytes once. Every step follows numpy 2's dtypes for the reference's expressions, with explicitly
// rounded intrinsics so that nothing is contracted into an FMA:
//
// DEPTH  t = 1 / (d + 1e-6f) fp32; h = (t - min) / ((max - min) + 1e-6f) fp32; p = h * 255 fp32, a = trunc(p), b = min(a+1, 255),
//        f = double(p) - a; c = T[a] + (T[b] - T[a]) f fp64 (heatmap_to_pseudo_color); byte = trunc(255 c). h < 0 -> 0,
//        h > 1 -> 255 as the reference's masks; NaN h -> 0 (the reference raises there).
// FLOW   |u| or |v| > 1e7 -> u = v = 0 and the pixel black; maxrad = max rad, or -1 when that is NaN (Python's max(-1, nan));
//        U = double(u / maxrad) + DBL_EPSILON (fp32 quotient, np.float64 eps promotes); NaN U or V -> U = V = 0 and black;
//        r = min(sqrt(U U + V V), 1) fp64; ang = float(atan2(-V, -U)) (the one rounding that differs from numpy's fp64 arctan2:
//        it makes the result independent of the libm); fk = ((ang / pi + 1) / 2) * 54 + 1, k0 = floor(fk) (index k0 - 1 wraps
//        as numpy's negative index), k1 = k0 + 1 (56 -> 1), f = fk - k0; col = (1 - f) W[k0-1] + f W[k1-1];
//        r <= 1: col = 1 - r (1 - col), else col *= 0.75; byte = floor(255 col).
// IMG    over all n images: min < -0.1f -> x = (x + 1) / 2, else max > 1.5f -> x = x / 255 (fp32); byte = trunc(x * 255) fp32.
// Every byte is clipped to [0, 255] before the conversion (NaN -> 0).
#include <math.h>

#include "common.cuh"

namespace dvd {
namespace {

constexpr int kThreads = 256;
constexpr int kRun = 4;

struct Maps {
  dvd_vis_map m[DVD_VIS_MAX_MAPS];
  int n;
};

// np.min / np.max: a NaN anywhere gives NaN; otherwise the exact extremum
__device__ __forceinline__ float nan_min(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : fminf(a, b); }
__device__ __forceinline__ float nan_max(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : fmaxf(a, b); }

__device__ __forceinline__ unsigned char to_byte(double v) {  // clip to [0, 255], NaN -> 0, then truncate
  return (unsigned char)(int)fmin(fmax(v, 0.0), 255.0);
}

__device__ __forceinline__ float depth_t(float d) { return __fdiv_rn(1.f, __fadd_rn(d, 1e-6f)); }

__device__ __forceinline__ float flow_rad(float u, float v) {
  if (fabsf(u) > 1e7f || fabsf(v) > 1e7f) return 0.f;
  return __fsqrt_rn(__fadd_rn(__fmul_rn(u, u), __fmul_rn(v, v)));
}

__global__ void __launch_bounds__(kThreads) vis_ranges_kernel(Maps M, int H, int W, float* __restrict__ ranges) {
  DVD_PDL_ENTER();
  const dvd_vis_map& m = M.m[blockIdx.y];
  const int i = blockIdx.x;
  if (i >= m.n) return;
  const float* s = m.src + (long long)i * m.s_n;
  float lo = INFINITY, hi = -INFINITY;
  const long long hw = (long long)H * W;
  for (long long p = threadIdx.x; p < hw; p += kThreads) {
    const int y = (int)(p / W), x = (int)(p % W);
    const float* e = s + (long long)y * m.s_y + (long long)x * m.s_x;
    if (m.kind == DVD_VIS_MAP_DEPTH) {
      const float t = depth_t(__ldg(e));
      lo = nan_min(lo, t);
      hi = nan_max(hi, t);
    } else if (m.kind == DVD_VIS_MAP_FLOW) {
      hi = nan_max(hi, flow_rad(__ldg(e), __ldg(e + m.s_c)));
    } else {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float v = __ldg(e + c * m.s_c);
        lo = nan_min(lo, v);
        hi = nan_max(hi, v);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = nan_min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = nan_max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  __shared__ float slo[kThreads / 32], shi[kThreads / 32];
  if ((threadIdx.x & 31) == 0) {
    slo[threadIdx.x >> 5] = lo;
    shi[threadIdx.x >> 5] = hi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kThreads / 32; ++w) {
      lo = nan_min(lo, slo[w]);
      hi = nan_max(hi, shi[w]);
    }
    ranges[m.range + 2 * i] = m.kind == DVD_VIS_MAP_FLOW ? hi : lo;
    ranges[m.range + 2 * i + 1] = hi;
  }
}

__device__ __forceinline__ void depth_pixel(float d, float mn, float mx, const double* __restrict__ turbo, unsigned char* rgb) {
  const float h = __fdiv_rn(__fsub_rn(depth_t(d), mn), __fadd_rn(__fsub_rn(mx, mn), 1e-6f));
  if (!(h >= 0.f)) {  // NaN (the deviation) or h < 0 (the reference's mask): black
    rgb[0] = rgb[1] = rgb[2] = 0;
    return;
  }
  if (h > 1.f) {
    rgb[0] = rgb[1] = rgb[2] = 255;
    return;
  }
  const float p = __fmul_rn(h, 255.f);
  const int a = (int)p;
  const int b = min(a + 1, 255);
  const double f = __dsub_rn((double)p, (double)a);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double ta = __ldg(turbo + 3 * a + k), tb = __ldg(turbo + 3 * b + k);
    const double c = __dadd_rn(ta, __dmul_rn(__dsub_rn(tb, ta), f));
    rgb[k] = to_byte(__dmul_rn(c, 255.0));
  }
}

__device__ __forceinline__ void flow_pixel(float u, float v, float maxrad, const double* __restrict__ wheel, unsigned char* rgb) {
  if (fabsf(u) > 1e7f || fabsf(v) > 1e7f) {
    rgb[0] = rgb[1] = rgb[2] = 0;
    return;
  }
  const float mr = maxrad != maxrad ? -1.f : maxrad;
  double U = __dadd_rn((double)__fdiv_rn(u, mr), 2.220446049250313e-16);
  double V = __dadd_rn((double)__fdiv_rn(v, mr), 2.220446049250313e-16);
  const bool bad = U != U || V != V;
  if (bad) U = V = 0.0;
  double r = __dsqrt_rn(__dadd_rn(__dmul_rn(U, U), __dmul_rn(V, V)));
  if (r > 1.0) r = 1.0;
  const double ang = (double)__double2float_rn(atan2(-V, -U));
  const double fk = __dadd_rn(__dmul_rn(__ddiv_rn(__dadd_rn(__ddiv_rn(ang, 3.141592653589793), 1.0), 2.0), 54.0), 1.0);
  const int k0 = (int)floor(fk);
  const int k1 = k0 + 1 == 56 ? 1 : k0 + 1;
  const double f = __dsub_rn(fk, (double)k0);
  const int i0 = k0 - 1 < 0 ? k0 - 1 + 55 : k0 - 1;
  const int i1 = k1 - 1;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double c0 = __ldg(wheel + 3 * i0 + k), c1 = __ldg(wheel + 3 * i1 + k);
    double col = __dadd_rn(__dmul_rn(__dsub_rn(1.0, f), c0), __dmul_rn(f, c1));
    col = r <= 1.0 ? __dsub_rn(1.0, __dmul_rn(r, __dsub_rn(1.0, col))) : __dmul_rn(col, 0.75);
    rgb[k] = bad ? 0 : to_byte(floor(__dmul_rn(255.0, col)));
  }
}

__global__ void __launch_bounds__(kThreads) vis_tiles_kernel(Maps M, int H, int W, const float* __restrict__ ranges,
                                                             const double* __restrict__ turbo, const double* __restrict__ wheel,
                                                             unsigned char* __restrict__ tiles) {
  DVD_PDL_ENTER();
  const dvd_vis_map& m = M.m[blockIdx.y];
  const int runs = (W + kRun - 1) / kRun;
  const long long item = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (item >= (long long)m.n * H * runs) return;
  const int xr = (int)(item % runs);
  const long long iy = item / runs;
  const int y = (int)(iy % H), i = (int)(iy / H);
  const int x0 = xr * kRun, nx = min(kRun, W - x0);
  float lo = 0.f, hi = 0.f;
  if (m.kind == DVD_VIS_MAP_IMG) {  // the rescale is decided on the whole [n,3,H,W] array
    lo = __ldg(ranges + m.range);
    hi = __ldg(ranges + m.range + 1);
    for (int j = 1; j < m.n; ++j) {
      lo = nan_min(lo, __ldg(ranges + m.range + 2 * j));
      hi = nan_max(hi, __ldg(ranges + m.range + 2 * j + 1));
    }
  } else {
    lo = __ldg(ranges + m.range + 2 * i);
    hi = __ldg(ranges + m.range + 2 * i + 1);
  }
  const float* s = m.src + (long long)i * m.s_n + (long long)y * m.s_y;
  unsigned char px[3 * kRun];
#pragma unroll
  for (int j = 0; j < kRun; ++j) {
    if (j >= nx) break;
    const float* e = s + (long long)(x0 + j) * m.s_x;
    unsigned char* o = px + 3 * j;
    if (m.kind == DVD_VIS_MAP_DEPTH) {
      depth_pixel(__ldg(e), lo, hi, turbo, o);
    } else if (m.kind == DVD_VIS_MAP_FLOW) {
      flow_pixel(__ldg(e), __ldg(e + m.s_c), hi, wheel, o);
    } else {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float v = __ldg(e + c * m.s_c);
        if (lo < -0.1f) {
          v = __fdiv_rn(__fadd_rn(v, 1.f), 2.f);
        } else if (hi > 1.5f) {
          v = __fdiv_rn(v, 255.f);
        }
        o[c] = to_byte((double)__fmul_rn(v, 255.f));
      }
    }
  }
  unsigned char* out = tiles + ((((long long)m.tile + i) * H + y) * W + x0) * 3;
  if (nx == kRun && (reinterpret_cast<uintptr_t>(out) & 3) == 0) {
    unsigned int* w = reinterpret_cast<unsigned int*>(out);
#pragma unroll
    for (int k = 0; k < 3 * kRun / 4; ++k)
      w[k] = px[4 * k] | (px[4 * k + 1] << 8) | (px[4 * k + 2] << 16) | ((unsigned int)px[4 * k + 3] << 24);
  } else {
    for (int k = 0; k < 3 * nx; ++k) out[k] = px[k];
  }
}

int copy_maps(const dvd_vis_map* maps, int n_maps, int H, int W, Maps* M, int* max_n, const char* what) {
  DVD_ARG_CHECK(maps, "%s: null maps", what);
  DVD_ARG_CHECK(n_maps >= 1 && n_maps <= DVD_VIS_MAX_MAPS, "%s: %d maps, 1 to %d allowed", what, n_maps, DVD_VIS_MAX_MAPS);
  DVD_ARG_CHECK(H >= 1 && W >= 1, "%s: bad image size %d x %d", what, H, W);
  *M = Maps{};
  M->n = n_maps;
  *max_n = 0;
  for (int q = 0; q < n_maps; ++q) {
    const dvd_vis_map& m = maps[q];
    DVD_ARG_CHECK(m.src, "%s: map %d has no source", what, q);
    DVD_ARG_CHECK(m.kind == DVD_VIS_MAP_DEPTH || m.kind == DVD_VIS_MAP_FLOW || m.kind == DVD_VIS_MAP_IMG,
                  "%s: map %d has unknown kind %d", what, q, m.kind);
    DVD_ARG_CHECK(m.n >= 1 && m.range >= 0 && m.tile >= 0, "%s: map %d has n %d, range %d, tile %d", what, q, m.n, m.range, m.tile);
    M->m[q] = m;
    *max_n = max(*max_n, m.n);
  }
  return 0;
}

}  // namespace
}  // namespace dvd

using namespace dvd;

extern "C" int dvd_vis_ranges(const dvd_vis_map* maps, int n_maps, int H, int W, float* ranges, void* stream) {
  Maps M;
  int max_n;
  const int rc = copy_maps(maps, n_maps, H, W, &M, &max_n, "dvd_vis_ranges");
  if (rc) return rc;
  DVD_ARG_CHECK(ranges, "dvd_vis_ranges: null ranges");
  DVD_CUDA_CALL(launch(vis_ranges_kernel, dim3((unsigned)max_n, (unsigned)n_maps), dim3(kThreads), 0, (cudaStream_t)stream, M, H, W,
                       ranges));
  return 0;
}

extern "C" int dvd_vis_tiles(const dvd_vis_map* maps, int n_maps, int H, int W, const float* ranges, const double* turbo,
                             const double* wheel, unsigned char* tiles, void* stream) {
  Maps M;
  int max_n;
  const int rc = copy_maps(maps, n_maps, H, W, &M, &max_n, "dvd_vis_tiles");
  if (rc) return rc;
  DVD_ARG_CHECK(ranges && turbo && wheel && tiles, "dvd_vis_tiles: null pointer");
  const long long items = (long long)max_n * H * ((W + kRun - 1) / kRun);
  const long long blocks = (items + kThreads - 1) / kThreads;
  DVD_ARG_CHECK(blocks <= 0x7fffffffLL, "dvd_vis_tiles: %d images of %d x %d are too many for one launch", max_n, H, W);
  DVD_CUDA_CALL(launch(vis_tiles_kernel, dim3((unsigned)blocks, (unsigned)n_maps), dim3(kThreads), 0, (cudaStream_t)stream, M, H, W,
                       ranges, turbo, wheel, tiles));
  return 0;
}
