// Error reporting + device queries shared by every translation unit of libdvd_b200.so.
#include "common.cuh"
#include <stdlib.h>
#include <string.h>

namespace dvd {

static thread_local char g_err[512] = {0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("DVD_PDL");
    return !(e && e[0] == '0');
  }();
  return on;
}

int num_sms() {
  static int cached[16] = {0};     // per device
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return 148;
  if (cached[dev] > 0) return cached[dev];
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) {
    cached[dev] = n;
    return n;
  }
  return 132;  // H100 SXM
}

// one thread per output element; the slabs are read in order, four loads in flight
__global__ void __launch_bounds__(256) ordered_sum_kernel(const float* __restrict__ slab, int nslab, long n, float* dst0,
                                                         long n0, float* dst1) {
  DVD_PDL_ENTER();
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  int k = 0;
  for (; k + 4 <= nslab; k += 4) {
    const float a = __ldcg(slab + (size_t)k * n + i), b = __ldcg(slab + (size_t)(k + 1) * n + i);
    const float c = __ldcg(slab + (size_t)(k + 2) * n + i), d = __ldcg(slab + (size_t)(k + 3) * n + i);
    s += a; s += b; s += c; s += d;
  }
  for (; k < nslab; ++k) s += __ldcg(slab + (size_t)k * n + i);
  float* d = i < n0 ? dst0 + i : dst1 + (i - n0);
  *d += s;
}

int launch_ordered_sum(const float* slab, int nslab, long n, float* dst0, long n0, float* dst1, cudaStream_t st) {
  DVD_ARG_CHECK(slab && dst0 && nslab >= 1 && n >= 1 && (n0 == n || dst1), "ordered_sum: bad arguments");
  DVD_CUDA_CALL(launch(ordered_sum_kernel, (unsigned)((n + 255) / 256), 256, 0, st, slab, nslab, n, dst0, n0, dst1));
  DVD_CUDA_LAUNCH_CHECK("ordered_sum_kernel");
  return 0;
}

}  // namespace dvd

/* Workspace of the *_ordered entry points, per site. Every bound follows from the launch geometry of the site's kernels, which
 * is a function of the SM count; a launch whose slabs would not fit returns an error. */
extern "C" size_t dvd_ordered_workspace_bytes(int site) {
  const size_t sms = (size_t)dvd::num_sms();
  switch (site) {
    // split-K weight-gradient tiles (one CTA per SM, up to 128 x 256 partial sums each) + the per-CTA row slabs of the BatchNorm
    // gamma / column-sum partials (128 of each per CTA, up to DVD_ORD_CONV_MAX_CTAS CTAs)
    case DVD_ORD_CONV_WGRAD: return (sms * 128 * 256 + (size_t)DVD_ORD_CONV_MAX_CTAS * 256) * sizeof(float);
    // split-K MLP weight gradient: at most one CTA per SM, 128 x 256 partial sums + 128 bias sums each
    case DVD_ORD_MLP_WGRAD: return sms * (128 * 256 + 128) * sizeof(float);
    // output-bias gradient of the MLP data-gradient chain: one CTA per SM, 8 MMA warps, 3 sums each
    case DVD_ORD_MLP_DGRAD: return sms * 8 * 3 * sizeof(float);
    // per-channel sums (dvd_relu_bwd_colsum, dvd_bn_act_bwd): gridDim.x x C x 2 <= 64 sms * 64 + 8 C, for C <= DVD_ORD_MAX_CHANNELS
    case DVD_ORD_CHANNEL_SUMS: return (sms * 64 * 64 + 8 * (size_t)DVD_ORD_MAX_CHANNELS) * sizeof(float);
    // stem weight gradient: up to 2 CTAs per SM, 147 taps x 64 channels + 64 bias sums each
    case DVD_ORD_STEM: return sms * 2 * (147 * 64 + 64) * sizeof(float);
    // head: up to 4 CTAs per SM, 32 weight + 1 bias sums each
    case DVD_ORD_HEAD: return sms * 4 * 33 * sizeof(float);
    default: return 0;
  }
}

extern "C" const char* dvd_last_error(void) { return dvd::g_err; }
extern "C" int dvd_version(void) { return 103; }
/* sizes of the structs that cross the C ABI by pointer (which: 0 dvd_loss_cfg, 1 dvd_mlp_cfg, 2 dvd_conv_desc, 3 dvd_pack_item,
 * 4 dvd_vis_panel, 5 dvd_vis_map): a binding in another language checks its own layout against these */
extern "C" long dvd_struct_size(int which) {
  switch (which) {
    case 0: return (long)sizeof(dvd_loss_cfg);
    case 1: return (long)sizeof(dvd_mlp_cfg);
    case 2: return (long)sizeof(dvd_conv_desc);
    case 3: return (long)sizeof(dvd_pack_item);
    case 4: return (long)sizeof(dvd_vis_panel);
    case 5: return (long)sizeof(dvd_vis_map);
    default: return -1;
  }
}
