// Test-end visualisation: colour-maps strided fp32 views (refined / initial / GT disparity, RGB frames, temporal slices) into a
// batch of uint8 BGR canvases that start as a copy of a host-drawn template.
//
// One thread writes a run of kRun consecutive canvas pixels of one row. For each pixel it finds the panel that covers it (the
// panels of a call do not overlap, checked on the host) and either reads the panel's source element(s) once and applies the
// transform, or copies the template pixel. Every output byte is written exactly once; no thread waits on another, and there
// are no atomics, so the canvases are a pure function of the inputs.
#include <math.h>

#include "common.cuh"

namespace dvd {
namespace {

constexpr int kThreads = 256;
constexpr int kRun = 8;

struct Panels {
  dvd_vis_panel p[DVD_VIS_MAX_PANELS];
  int n;
};

// matplotlib's Colormap.__call__ with N = 256 after Normalize(vmin, vmax): t = (v - vmin) / (vmax - vmin) in fp64,
// index floor(256 t), t >= 1 -> 255 (over = last colour), t < 0 -> 0 (under = first colour); vmax == vmin -> 0.
// NaN (matplotlib's "bad", transparent on the black figure) -> -1, drawn black.
__device__ __forceinline__ int cmap_index(double v, double lo, double hi) {
  if (isnan(v)) return -1;
  if (hi == lo) return 0;
  const double t = __ddiv_rn(__dsub_rn(v, lo), __dsub_rn(hi, lo));
  if (isnan(t)) return -1;
  if (t >= 1.0) return 255;
  if (t < 0.0) return 0;
  return (int)floor(t * 256.0);  // exact: a power of two
}

__device__ __forceinline__ void panel_pixel(const dvd_vis_panel& p, int c, int y, int x, const unsigned char* __restrict__ lut,
                                            unsigned char* bgr) {
  const float* s = p.src + (long long)c * p.s_canvas + (long long)(y - p.y0) * p.s_row + (long long)(x - p.x0) * p.s_col;
  if (p.transform == DVD_VIS_RGB) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      // floor(255 clip(v, 0, 1)) in fp32 (points.cu's colour rule); fmaxf maps NaN to 0. Channel k (R, G, B) -> byte 2 - k.
      const float v = fminf(fmaxf(__ldg(s + k * p.s_chan), 0.f), 1.f);
      bgr[2 - k] = (unsigned char)__fmul_rn(v, 255.f);
    }
    return;
  }
  const float x32 = __ldg(s);
  double v;
  if (p.transform == DVD_VIS_DISP) {
    v = (double)__fdiv_rn(1.f, x32);  // numpy float32 1 / a
  } else {
    // np.where(gt > 1e-8, 1, 0) / (gt + 1e-8): int64 / float32 -> float64; gt + 1e-8 stays float32 (weak Python scalar)
    v = __ddiv_rn(x32 > 1e-8f ? 1.0 : 0.0, (double)__fadd_rn(x32, 1e-8f));
  }
  const int i = cmap_index(v, __ldg(p.vmin + c), __ldg(p.vmax + c));
  if (i < 0) {
    bgr[0] = bgr[1] = bgr[2] = 0;
  } else {
    bgr[0] = __ldg(lut + 3 * i);
    bgr[1] = __ldg(lut + 3 * i + 1);
    bgr[2] = __ldg(lut + 3 * i + 2);
  }
}

__global__ void __launch_bounds__(kThreads) vis_panels_kernel(Panels P, const unsigned char* __restrict__ tmpl, long long tmpl_stride,
                                                              int n_canvas, int CH, int CW, const unsigned char* __restrict__ lut,
                                                              unsigned char* __restrict__ out) {
  DVD_PDL_ENTER();
  const int runs = (CW + kRun - 1) / kRun;
  const long long item = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (item >= (long long)n_canvas * CH * runs) return;
  const int xr = (int)(item % runs);
  const long long cy = item / runs;
  const int y = (int)(cy % CH), c = (int)(cy / CH);
  const int x0 = xr * kRun, n = min(kRun, CW - x0);
  const unsigned char* t = tmpl + (long long)c * tmpl_stride + ((long long)y * CW + x0) * 3;
  unsigned char px[3 * kRun];
#pragma unroll
  for (int j = 0; j < kRun; ++j) {
    if (j >= n) break;
    const int x = x0 + j;
    int hit = -1;
    for (int q = 0; q < P.n; ++q) {
      const dvd_vis_panel& p = P.p[q];
      if (y >= p.y0 && y < p.y0 + p.rows && x >= p.x0 && x < p.x0 + p.cols) hit = q;
    }
    if (hit >= 0) {
      panel_pixel(P.p[hit], c, y, x, lut, px + 3 * j);
    } else {
      px[3 * j] = __ldg(t + 3 * j);
      px[3 * j + 1] = __ldg(t + 3 * j + 1);
      px[3 * j + 2] = __ldg(t + 3 * j + 2);
    }
  }
  unsigned char* o = out + (((long long)c * CH + y) * CW + x0) * 3;
  if (n == kRun && (reinterpret_cast<uintptr_t>(o) & 3) == 0) {
    unsigned int* w = reinterpret_cast<unsigned int*>(o);
#pragma unroll
    for (int k = 0; k < 3 * kRun / 4; ++k)
      w[k] = px[4 * k] | (px[4 * k + 1] << 8) | (px[4 * k + 2] << 16) | ((unsigned int)px[4 * k + 3] << 24);
  } else {
#pragma unroll
    for (int k = 0; k < 3 * kRun; ++k)
      if (k < 3 * n) o[k] = px[k];
  }
}

}  // namespace
}  // namespace dvd

using namespace dvd;

extern "C" int dvd_vis_panels(const unsigned char* tmpl, long long tmpl_stride, int n_canvas, int CH, int CW, const dvd_vis_panel* panels,
                              int n_panels, const unsigned char* lut, unsigned char* out, void* stream) {
  DVD_ARG_CHECK(tmpl && out && (n_panels == 0 || panels), "dvd_vis_panels: null pointer");
  DVD_ARG_CHECK(n_canvas >= 1 && CH >= 1 && CW >= 1, "dvd_vis_panels: bad canvas shape %d x %d x %d", n_canvas, CH, CW);
  DVD_ARG_CHECK(n_panels >= 0 && n_panels <= DVD_VIS_MAX_PANELS, "dvd_vis_panels: %d panels, at most %d", n_panels, DVD_VIS_MAX_PANELS);
  DVD_ARG_CHECK(tmpl_stride == 0 || tmpl_stride >= 3LL * CH * CW, "dvd_vis_panels: template stride %lld below one canvas", tmpl_stride);
  Panels P = {};
  P.n = n_panels;
  for (int q = 0; q < n_panels; ++q) {
    const dvd_vis_panel& p = panels[q];
    DVD_ARG_CHECK(p.src, "dvd_vis_panels: panel %d has no source", q);
    DVD_ARG_CHECK(p.transform == DVD_VIS_DISP || p.transform == DVD_VIS_GT_DISP || p.transform == DVD_VIS_RGB,
                  "dvd_vis_panels: panel %d has unknown transform %d", q, p.transform);
    DVD_ARG_CHECK(p.transform == DVD_VIS_RGB || (p.vmin && p.vmax && lut), "dvd_vis_panels: panel %d needs vmin, vmax and the LUT", q);
    DVD_ARG_CHECK(p.rows >= 1 && p.cols >= 1 && p.y0 >= 0 && p.x0 >= 0 && p.y0 + p.rows <= CH && p.x0 + p.cols <= CW,
                  "dvd_vis_panels: panel %d (%d x %d at %d, %d) leaves the %d x %d canvas", q, p.rows, p.cols, p.y0, p.x0, CH, CW);
    for (int r = 0; r < q; ++r) {
      const dvd_vis_panel& o = panels[r];
      const bool apart = p.y0 >= o.y0 + o.rows || o.y0 >= p.y0 + p.rows || p.x0 >= o.x0 + o.cols || o.x0 >= p.x0 + p.cols;
      DVD_ARG_CHECK(apart, "dvd_vis_panels: panels %d and %d overlap", r, q);
    }
    P.p[q] = p;
  }
  const long long items = (long long)n_canvas * CH * ((CW + kRun - 1) / kRun);
  const long long blocks = (items + kThreads - 1) / kThreads;
  DVD_ARG_CHECK(blocks <= 0x7fffffffLL, "dvd_vis_panels: %lld canvases of %d x %d are too many for one launch", (long long)n_canvas, CH, CW);
  DVD_CUDA_CALL(launch(vis_panels_kernel, dim3((unsigned)blocks), dim3(kThreads), 0, (cudaStream_t)stream, P, tmpl, tmpl_stride, n_canvas,
                       CH, CW, lut, out));
  return 0;
}
