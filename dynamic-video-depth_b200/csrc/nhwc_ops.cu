// Channels-last (NHWC) glue kernels of the depth nets: eval-mode BatchNorm fused with the residual add and the
// ReLU (forward + backward with the per-channel gamma/beta reductions), and x2 bilinear up-sampling (forward +
// gather backward). All HBM-bound.
//
// Why: profiling the cuDNN depth net
// showed that less than half of the time is convolution: 19 % NCHW<->NHWC transposes around the tensor-core conv
// kernels, 15 % ATen batch-norm fwd/bwd, 13 % ATen bilinear up-sampling (0.55 ms per launch, ~15x its HBM time),
// 8 % separate add / clamp passes. Running the net channels-last removes the transposes; these kernels replace
// the ATen glue:   reference ops third_party/midas_blocks.py:95-97,121-168 (Interpolate, ResidualConvUnit,
// FeatureFusionBlock), torchvision Bottleneck (bn1/bn2/bn3 + relu + residual), third_party/MiDaS.py:188-195.
#include "common.cuh"

namespace dvd {

constexpr int kElemThreads = 256;

__device__ __forceinline__ float4 round4_tf32(float4 v) {
  uint32_t a, b, c, d;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(a) : "f"(v.x));
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(b) : "f"(v.y));
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(c) : "f"(v.z));
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(d) : "f"(v.w));
  return make_float4(__uint_as_float(a), __uint_as_float(b), __uint_as_float(c), __uint_as_float(d));
}

// y = x * scale[c] + shift[c] (+ res) ; optional ReLU.   scale = gamma * rsqrt(var + eps), shift = beta - mean * scale
__global__ void __launch_bounds__(kElemThreads) bn_act_fwd_kernel(const float4* __restrict__ x, const float4* __restrict__ res,
                                                                  const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                  const float* __restrict__ mean, const float* __restrict__ var,
                                                                  float eps, float4* __restrict__ y, long n4, int c4, int relu) {
  DVD_PDL_ENTER();
  const long stride = (long)gridDim.x * blockDim.x;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const int c = (int)(i % c4) * 4;
    const float4 g = *reinterpret_cast<const float4*>(gamma + c), b = *reinterpret_cast<const float4*>(beta + c);
    const float4 m = *reinterpret_cast<const float4*>(mean + c), v = *reinterpret_cast<const float4*>(var + c);
    float4 xv = ldg_stream4(reinterpret_cast<const float*>(x + i));
    float4 o;
    float s;
    s = g.x * rsqrtf(v.x + eps); o.x = fmaf(xv.x, s, b.x - m.x * s);
    s = g.y * rsqrtf(v.y + eps); o.y = fmaf(xv.y, s, b.y - m.y * s);
    s = g.z * rsqrtf(v.z + eps); o.z = fmaf(xv.z, s, b.z - m.z * s);
    s = g.w * rsqrtf(v.w + eps); o.w = fmaf(xv.w, s, b.w - m.w * s);
    if (res) {
      const float4 r = ldg_stream4(reinterpret_cast<const float*>(res + i));
      o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
    }
    if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
    y[i] = o;
  }
}

// backward of the above: gm = g * [y > 0] (if relu); g_x = gm * scale; g_res = gm (optional);
// g_gamma[c] += sum gm * (x - mean) * rstd ; g_beta[c] += sum gm.
// block = (cgb channel-groups of 4) x (256 / cgb pixel rows); grid.x over pixel slabs, grid.y over channel blocks.
template <bool ORD = false>
__global__ void __launch_bounds__(kElemThreads) bn_act_bwd_kernel(const float4* __restrict__ g, const float4* __restrict__ x,
                                                                  const float4* __restrict__ y, const float* __restrict__ gamma,
                                                                  const float* __restrict__ mean, const float* __restrict__ var,
                                                                  float eps, float4* __restrict__ gx, float4* __restrict__ gres,
                                                                  float* __restrict__ ggamma, float* __restrict__ gbeta, long P,
                                                                  int c4, int cgb, int relu, float* __restrict__ ord) {
  DVD_PDL_ENTER();
  __shared__ float red[kElemThreads][8];
  const int tx = threadIdx.x % cgb, ty = threadIdx.x / cgb, rows = kElemThreads / cgb;
  const int cg = blockIdx.y * cgb + tx;        // channel group (4 channels)
  float sg[4] = {0, 0, 0, 0}, sb[4] = {0, 0, 0, 0};
  if (cg < c4) {
    const int c = cg * 4;
    const float4 gm4 = *reinterpret_cast<const float4*>(gamma + c), m = *reinterpret_cast<const float4*>(mean + c);
    const float4 v = *reinterpret_cast<const float4*>(var + c);
    const float rs[4] = {rsqrtf(v.x + eps), rsqrtf(v.y + eps), rsqrtf(v.z + eps), rsqrtf(v.w + eps)};
    const float sc[4] = {gm4.x * rs[0], gm4.y * rs[1], gm4.z * rs[2], gm4.w * rs[3]};
    const float mu[4] = {m.x, m.y, m.z, m.w};
    for (long p = (long)blockIdx.x * rows + ty; p < P; p += (long)gridDim.x * rows) {
      const long i = p * c4 + cg;
      float4 gv = ldg_stream4(reinterpret_cast<const float*>(g + i));
      if (relu) {
        const float4 yv = ldg_stream4(reinterpret_cast<const float*>(y + i));
        gv.x = yv.x > 0.f ? gv.x : 0.f; gv.y = yv.y > 0.f ? gv.y : 0.f;
        gv.z = yv.z > 0.f ? gv.z : 0.f; gv.w = yv.w > 0.f ? gv.w : 0.f;
      }
      const float4 xv = ldg_stream4(reinterpret_cast<const float*>(x + i));
      const float ga[4] = {gv.x, gv.y, gv.z, gv.w}, xa[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        sb[k] += ga[k];
        sg[k] = fmaf(ga[k], (xa[k] - mu[k]) * rs[k], sg[k]);
      }
      gx[i] = make_float4(ga[0] * sc[0], ga[1] * sc[1], ga[2] * sc[2], ga[3] * sc[3]);
      if (gres) gres[i] = gv;
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) { red[threadIdx.x][k] = sg[k]; red[threadIdx.x][4 + k] = sb[k]; }
  __syncthreads();
  if (ty == 0 && cg < c4) {
    float a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int r = 0; r < rows; ++r)
#pragma unroll
      for (int k = 0; k < 8; ++k) a[k] += red[r * cgb + tx][k];
    if constexpr (ORD) {   // ordered variant: [CTA column][gamma C | beta C] slab, added in CTA order by ordered_sum
      float* o = ord + (size_t)blockIdx.x * 8 * c4 + cg * 4;
#pragma unroll
      for (int k = 0; k < 4; ++k) { o[k] = a[k]; o[4 * c4 + k] = a[4 + k]; }
    } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      atomicAdd(ggamma + cg * 4 + k, a[k]);
      atomicAdd(gbeta + cg * 4 + k, a[4 + k]);
    }
    }
  }
}

// ---- x2 bilinear up-sampling, NHWC ------------------------------------------------------------------------------
// source index of ATen's upsample_bilinear2d (area_pixel_compute_source_index)
__device__ __forceinline__ float src_index(int dst, float scale, bool align) {
  if (align) return scale * dst;
  float s = scale * (dst + 0.5f) - 0.5f;
  return s < 0.f ? 0.f : s;
}

__global__ void __launch_bounds__(kElemThreads) upsample2x_fwd_kernel(const float4* __restrict__ x, float4* __restrict__ y, int N,
                                                                      int H, int W, int c4, float sh, float sw, int align,
                                                                      int round_out) {
  DVD_PDL_ENTER();
  const int OH = 2 * H, OW = 2 * W;
  const long total = (long)N * OH * OW * c4;
  const long stride = (long)gridDim.x * blockDim.x;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int c = (int)(i % c4);
    long p = i / c4;
    const int ox = (int)(p % OW); p /= OW;
    const int oy = (int)(p % OH);
    const int n = (int)(p / OH);
    const float fy = src_index(oy, sh, align), fx = src_index(ox, sw, align);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
    const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
    const float4* b = x + (size_t)n * H * W * c4 + c;
    const float4 a00 = b[((size_t)y0 * W + x0) * c4], a01 = b[((size_t)y0 * W + x1) * c4];
    const float4 a10 = b[((size_t)y1 * W + x0) * c4], a11 = b[((size_t)y1 * W + x1) * c4];
    float4 o;
    o.x = hy * (hx * a00.x + lx * a01.x) + ly * (hx * a10.x + lx * a11.x);
    o.y = hy * (hx * a00.y + lx * a01.y) + ly * (hx * a10.y + lx * a11.y);
    o.z = hy * (hx * a00.z + lx * a01.z) + ly * (hx * a10.z + lx * a11.z);
    o.w = hy * (hx * a00.w + lx * a01.w) + ly * (hx * a10.w + lx * a11.w);
    if (round_out) o = round4_tf32(o);
    st_stream4(reinterpret_cast<float*>(y + i), o);
  }
}

// gather backward: input pixel (iy, ix) collects from every output pixel whose taps include it
__global__ void __launch_bounds__(kElemThreads) upsample2x_bwd_kernel(const float4* __restrict__ g, float4* __restrict__ gx, int N,
                                                                      int H, int W, int c4, float sh, float sw, int align,
                                                                      int round_out) {
  DVD_PDL_ENTER();
  const int OH = 2 * H, OW = 2 * W;
  const long total = (long)N * H * W * c4;
  const long stride = (long)gridDim.x * blockDim.x;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int c = (int)(i % c4);
    long p = i / c4;
    const int ix = (int)(p % W); p /= W;
    const int iy = (int)(p % H);
    const int n = (int)(p / H);
    // candidate output rows / columns: src in (iy-1, iy+1). align_corners=False: src = dst/2 - 1/4 => dst in [2iy-1, 2iy+2];
    // align_corners=True: src = dst*(H-1)/(2H-1) => dst < 2(iy+1)(1 + 1/(2H-2)) <= 2iy+3 inside the image: [2iy-2, 2iy+3] covers both
    const int oy_lo = max(0, 2 * iy - 2), oy_hi = min(OH - 1, 2 * iy + 3);
    const int ox_lo = max(0, 2 * ix - 2), ox_hi = min(OW - 1, 2 * ix + 3);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4* gb = g + (size_t)n * OH * OW * c4 + c;
    for (int oy = oy_lo; oy <= oy_hi; ++oy) {
      const float fy = src_index(oy, sh, align);
      const int y0 = (int)fy, y1 = y0 + (y0 < H - 1 ? 1 : 0);
      const float ly = fy - y0;
      float wy = 0.f;
      if (y0 == iy) wy += 1.f - ly;
      if (y1 == iy) wy += ly;
      if (wy == 0.f) continue;
      for (int ox = ox_lo; ox <= ox_hi; ++ox) {
        const float fx = src_index(ox, sw, align);
        const int x0 = (int)fx, x1 = x0 + (x0 < W - 1 ? 1 : 0);
        const float lx = fx - x0;
        float wx = 0.f;
        if (x0 == ix) wx += 1.f - lx;
        if (x1 == ix) wx += lx;
        if (wx == 0.f) continue;
        const float w = wy * wx;
        const float4 gv = gb[((size_t)oy * OW + ox) * c4];
        acc.x = fmaf(w, gv.x, acc.x); acc.y = fmaf(w, gv.y, acc.y);
        acc.z = fmaf(w, gv.z, acc.z); acc.w = fmaf(w, gv.w, acc.w);
      }
    }
    gx[i] = round_out ? round4_tf32(acc) : acc;
  }
}

static unsigned blocks_for(long n) {
  long b = (n + kElemThreads - 1) / kElemThreads;
  long cap = (long)num_sms() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

}  // namespace dvd

using namespace dvd;

extern "C" int dvd_bn_act_fwd(const float* x, const float* res, const float* gamma, const float* beta, const float* mean,
                              const float* var, float eps, float* y, long P, int C, int relu, void* stream) {
  DVD_ARG_CHECK(x && gamma && beta && mean && var && y, "null pointer");
  DVD_ARG_CHECK(P > 0 && C > 0 && C % 4 == 0, "C must be a positive multiple of 4 (got %d)", C);
  DVD_ARG_CHECK(aligned16(x) && aligned16(y) && (!res || aligned16(res)) && aligned16(gamma) && aligned16(beta) &&
                    aligned16(mean) && aligned16(var), "buffers must be 16-byte aligned");
  const long n4 = P * (C / 4);
  dvd::launch(bn_act_fwd_kernel, blocks_for(n4), kElemThreads, 0, (cudaStream_t)stream, 
      (const float4*)x, (const float4*)res, gamma, beta, mean, var, eps, (float4*)y, n4, C / 4, relu);
  DVD_CUDA_LAUNCH_CHECK("bn_act_fwd");
  return 0;
}

static int bn_act_bwd(const float* g, const float* x, const float* y, const float* gamma, const float* mean,
                      const float* var, float eps, float* gx, float* gres, float* ggamma, float* gbeta, long P, int C,
                      int relu, void* ws, size_t ws_bytes, void* stream) {
  DVD_ARG_CHECK(g && x && gamma && mean && var && gx && ggamma && gbeta, "null pointer");
  DVD_ARG_CHECK(!relu || y, "y is required for the ReLU mask");
  DVD_ARG_CHECK(P > 0 && C > 0 && C % 4 == 0, "C must be a positive multiple of 4 (got %d)", C);
  const int c4 = C / 4;
  int cgb = 64;
  while (cgb > c4) cgb >>= 1;   // power of two <= c4 (c4 >= 1)
  if (cgb < 1) cgb = 1;
  const int rows = kElemThreads / cgb;
  long gx_blocks = (P + (long)rows * 8 - 1) / ((long)rows * 8);
  const long cap = ((long)num_sms() * 8 * cgb) / c4 + 1;
  if (gx_blocks > cap) gx_blocks = cap;
  if (gx_blocks < 1) gx_blocks = 1;
  dim3 grid((unsigned)gx_blocks, (unsigned)((c4 + cgb - 1) / cgb));
  if (ws) {
    DVD_ARG_CHECK(aligned16(ws) && (size_t)gx_blocks * 2 * C * sizeof(float) <= ws_bytes,
                  "ordered BatchNorm gradient: the workspace needs dvd_ordered_workspace_bytes(DVD_ORD_CHANNEL_SUMS) bytes (C <= %d)",
                  DVD_ORD_MAX_CHANNELS);
    dvd::launch(bn_act_bwd_kernel<true>, grid, kElemThreads, 0, (cudaStream_t)stream, (const float4*)g, (const float4*)x, (const float4*)y,
                gamma, mean, var, eps, (float4*)gx, (float4*)gres, ggamma, gbeta, P, c4, cgb, relu, (float*)ws);
    DVD_CUDA_LAUNCH_CHECK("bn_act_bwd<ordered>");
    return launch_ordered_sum((const float*)ws, (int)gx_blocks, 2L * C, ggamma, C, gbeta, (cudaStream_t)stream);
  }
  dvd::launch(bn_act_bwd_kernel<>, grid, kElemThreads, 0, (cudaStream_t)stream, (const float4*)g, (const float4*)x, (const float4*)y, gamma, mean,
                                                                     var, eps, (float4*)gx, (float4*)gres, ggamma, gbeta, P, c4, cgb,
                                                                     relu, (float*)nullptr);
  DVD_CUDA_LAUNCH_CHECK("bn_act_bwd");
  return 0;
}

extern "C" int dvd_bn_act_bwd(const float* g, const float* x, const float* y, const float* gamma, const float* mean,
                              const float* var, float eps, float* gx, float* gres, float* ggamma, float* gbeta, long P, int C,
                              int relu, void* stream) {
  return bn_act_bwd(g, x, y, gamma, mean, var, eps, gx, gres, ggamma, gbeta, P, C, relu, nullptr, 0, stream);
}
extern "C" int dvd_bn_act_bwd_ordered(const float* g, const float* x, const float* y, const float* gamma, const float* mean,
                                      const float* var, float eps, float* gx, float* gres, float* ggamma, float* gbeta, long P, int C,
                                      int relu, void* ws, size_t ws_bytes, void* stream) {
  DVD_ARG_CHECK(ws != nullptr, "dvd_bn_act_bwd_ordered: null workspace");
  return bn_act_bwd(g, x, y, gamma, mean, var, eps, gx, gres, ggamma, gbeta, P, C, relu, ws, ws_bytes, stream);
}

extern "C" int dvd_upsample2x_fwd(const float* x, float* y, int N, int H, int W, int C, int align_corners, int round_out, void* stream) {
  DVD_ARG_CHECK(x && y && N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, "bad arguments (C must be a multiple of 4)");
  const float sh = align_corners ? (H > 1 ? (float)(H - 1) / (2 * H - 1) : 0.f) : 0.5f;
  const float sw = align_corners ? (W > 1 ? (float)(W - 1) / (2 * W - 1) : 0.f) : 0.5f;
  const long total = (long)N * 4 * H * W * (C / 4);
  dvd::launch(upsample2x_fwd_kernel, blocks_for(total), kElemThreads, 0, (cudaStream_t)stream, (const float4*)x, (float4*)y, N, H, W, C / 4, sh,
                                                                                    sw, align_corners, round_out);
  DVD_CUDA_LAUNCH_CHECK("upsample2x_fwd");
  return 0;
}

extern "C" int dvd_upsample2x_bwd(const float* g, float* gx, int N, int H, int W, int C, int align_corners, int round_out, void* stream) {
  DVD_ARG_CHECK(g && gx && N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, "bad arguments (C must be a multiple of 4)");
  const float sh = align_corners ? (H > 1 ? (float)(H - 1) / (2 * H - 1) : 0.f) : 0.5f;
  const float sw = align_corners ? (W > 1 ? (float)(W - 1) / (2 * W - 1) : 0.f) : 0.5f;
  const long total = (long)N * H * W * (C / 4);
  dvd::launch(upsample2x_bwd_kernel, blocks_for(total), kElemThreads, 0, (cudaStream_t)stream, (const float4*)g, (float4*)gx, N, H, W, C / 4, sh,
                                                                                    sw, align_corners, round_out);
  DVD_CUDA_LAUNCH_CHECK("upsample2x_bwd");
  return 0;
}
