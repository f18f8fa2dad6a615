// CUDA-core members of the MiDaS depth-net path (everything that is not a tensor-core convolution), NHWC fp32:
//   * dvd_round_tf32           round-to-nearest TF32 copy (foreign tensors entering the rounded-operand contract of conv2d_tc.cu)
//   * dvd_relu_bwd_colsum      gm = g * [y > 0] (+ TF32 rounding), per-channel sums -> bias / BatchNorm-beta gradient and the
//                              mean term of the BatchNorm-gamma gradient (the <W, dW> term comes from dvd_conv2d_wgrad)
//   * dvd_maxpool3x3s2_{fwd,bwd}   torchvision ResNet.maxpool (MaxPool2d(3, 2, 1)); first maximum wins like ATen; gather backward
//   * dvd_stem_{fwd,wgrad}     input normalisation (third_party/MiDaS.py:213-218) + conv1 7x7 stride 2 (3 -> 64) + bn1 + ReLU of the
//                              ResNeXt stem and its weight / BatchNorm gradients: Cin = 3 is no tensor-core shape, 0.3 % of the FLOPs
//   * dvd_head_{fwd,bwd}       scratch.output_conv[4..5] + depth: relu(conv1x1 32->1) -> clamp(1e-2) -> 10000/x (MiDaS.py:188-195,240-242)
#include "common.cuh"

namespace dvd {
namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float round_tf32(float v) {
  uint32_t o;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(o) : "f"(v));
  return __uint_as_float(o);
}
__device__ __forceinline__ float4 round4(float4 v) {
  return make_float4(round_tf32(v.x), round_tf32(v.y), round_tf32(v.z), round_tf32(v.w));
}

unsigned blocks_for(long n, int per_sm = 16) {
  long b = (n + kThreads - 1) / kThreads;
  const long cap = (long)num_sms() * per_sm;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

__global__ void __launch_bounds__(kThreads) round_kernel(const float4* __restrict__ x, float4* __restrict__ y, long n4) {
  DVD_PDL_ENTER();
  const long stride = (long)gridDim.x * blockDim.x;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) y[i] = round4(x[i]);
}

// gm = g * [y > 0]; colsum[c] += sum_p gm[p, c]; dgamma[c] -= mean[c] * rstd[c] * sum_p gm[p, c]
// block = (cgb channel groups of 4) x (256 / cgb pixel rows); grid.x over pixel slabs, grid.y over channel blocks
template <bool ORD = false>
__global__ void __launch_bounds__(kThreads) relu_bwd_colsum_kernel(const float4* __restrict__ g, const float4* __restrict__ y,
                                                                   float4* __restrict__ gm, float* __restrict__ colsum,
                                                                   const float* __restrict__ mean, const float* __restrict__ var,
                                                                   float eps, float* __restrict__ dgamma, long P, int c4, int cgb,
                                                                   int round_out, float* __restrict__ ord) {
  DVD_PDL_ENTER();
  __shared__ float red[kThreads][4];
  const int tx = threadIdx.x % cgb, ty = threadIdx.x / cgb, rows = kThreads / cgb;
  const int cg = blockIdx.y * cgb + tx;
  float s[4] = {0, 0, 0, 0};
  if (cg < c4) {
    for (long p = (long)blockIdx.x * rows + ty; p < P; p += (long)gridDim.x * rows) {
      const long i = p * c4 + cg;
      float4 gv = g[i];
      if (y) {
        const float4 yv = y[i];
        gv.x = yv.x > 0.f ? gv.x : 0.f; gv.y = yv.y > 0.f ? gv.y : 0.f;
        gv.z = yv.z > 0.f ? gv.z : 0.f; gv.w = yv.w > 0.f ? gv.w : 0.f;
      }
      if (round_out) gv = round4(gv);
      s[0] += gv.x; s[1] += gv.y; s[2] += gv.z; s[3] += gv.w;
      if (gm) gm[i] = gv;
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) red[threadIdx.x][k] = s[k];
  __syncthreads();
  if (ty == 0 && cg < c4 && (colsum || dgamma)) {
    float a[4] = {0, 0, 0, 0};
    for (int r = 0; r < rows; ++r)
#pragma unroll
      for (int k = 0; k < 4; ++k) a[k] += red[r * cgb + tx][k];
    if constexpr (ORD) {      // ordered variant: [CTA column][channel] slab, added by colsum_ordered_reduce_kernel
#pragma unroll
      for (int k = 0; k < 4; ++k) ord[(size_t)blockIdx.x * 4 * c4 + cg * 4 + k] = a[k];
    } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = cg * 4 + k;
      if (colsum) atomicAdd(colsum + c, a[k]);
      if (dgamma) atomicAdd(dgamma + c, -mean[c] * rsqrtf(var[c] + eps) * a[k]);
    }
    }
  }
}

// s = sum of channel c's partials in CTA order; colsum[c] += s; dgamma[c] -= mean[c] * rstd[c] * s
__global__ void __launch_bounds__(kThreads) colsum_ordered_reduce_kernel(const float* __restrict__ ord, int nb, int C,
                                                                         float* colsum, const float* __restrict__ mean,
                                                                         const float* __restrict__ var, float eps, float* dgamma) {
  DVD_PDL_ENTER();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int b = 0; b < nb; ++b) s += __ldcg(ord + (size_t)b * C + c);
  if (colsum) colsum[c] += s;
  if (dgamma) dgamma[c] += -mean[c] * rsqrtf(var[c] + eps) * s;
}

// ---- MaxPool2d(3, stride 2, padding 1), NHWC; idx = position (0..8) of the first maximum inside the window -----------
__global__ void __launch_bounds__(kThreads) maxpool_fwd_kernel(const float4* __restrict__ x, float4* __restrict__ y,
                                                               uchar4* __restrict__ idx, int N, int H, int W, int OH, int OW, int c4) {
  DVD_PDL_ENTER();
  const long total = (long)N * OH * OW * c4;
  const long stride = (long)gridDim.x * blockDim.x;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int c = (int)(i % c4);
    long p = i / c4;
    const int ox = (int)(p % OW); p /= OW;
    const int oy = (int)(p % OH);
    const int n = (int)(p / OH);
    float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    uchar4 bi = make_uchar4(0, 0, 0, 0);
    const float4* b = x + (size_t)n * H * W * c4 + c;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = 2 * oy - 1 + ky;
      if (iy < 0 || iy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = 2 * ox - 1 + kx;
        if (ix < 0 || ix >= W) continue;
        const float4 v = b[((size_t)iy * W + ix) * c4];
        const unsigned char pos = (unsigned char)(ky * 3 + kx);
        if (v.x > best.x) { best.x = v.x; bi.x = pos; }
        if (v.y > best.y) { best.y = v.y; bi.y = pos; }
        if (v.z > best.z) { best.z = v.z; bi.z = pos; }
        if (v.w > best.w) { best.w = v.w; bi.w = pos; }
      }
    }
    y[i] = best;
    idx[i] = bi;
  }
}

__global__ void __launch_bounds__(kThreads) maxpool_bwd_kernel(const float4* __restrict__ g, const uchar4* __restrict__ idx,
                                                               float4* __restrict__ gx, int N, int H, int W, int OH, int OW, int c4) {
  DVD_PDL_ENTER();
  const long total = (long)N * H * W * c4;
  const long stride = (long)gridDim.x * blockDim.x;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int c = (int)(i % c4);
    long p = i / c4;
    const int ix = (int)(p % W); p /= W;
    const int iy = (int)(p % H);
    const int n = (int)(p / H);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    // windows containing (iy, ix): oy with 2*oy - 1 <= iy <= 2*oy + 1
    for (int oy = (iy) / 2; oy <= (iy + 1) / 2; ++oy) {
      if (oy >= OH) continue;
      const int ky = iy - (2 * oy - 1);
      for (int ox = (ix) / 2; ox <= (ix + 1) / 2; ++ox) {
        if (ox >= OW) continue;
        const int kx = ix - (2 * ox - 1);
        const unsigned char pos = (unsigned char)(ky * 3 + kx);
        const size_t o = (((size_t)n * OH + oy) * OW + ox) * c4 + c;
        const uchar4 b = idx[o];
        const float4 gv = g[o];
        if (b.x == pos) acc.x += gv.x;
        if (b.y == pos) acc.y += gv.y;
        if (b.z == pos) acc.z += gv.z;
        if (b.w == pos) acc.w += gv.w;
      }
    }
    gx[i] = acc;
  }
}

// ---- stem: normalise + conv 7x7 / 2 (3 -> 64, pad 3) + eval BatchNorm + ReLU, NCHW image -> NHWC activation ----------------
constexpr int kStemTH = 4, kStemTW = 32;                       // output tile: 128 pixels, one per thread
constexpr int kStemPH = 2 * kStemTH + 5, kStemPW = 2 * kStemTW + 5;   // input patch 13 x 69
constexpr int kStemTaps = 147;

__device__ __forceinline__ void stem_load_patch(float (*patch)[kStemPH][kStemPW], const float* __restrict__ img, int H, int W, int oh0,
                                                int ow0, const float* nmean, const float* nrstd, int nthreads) {
  for (int i = threadIdx.x; i < 3 * kStemPH * kStemPW; i += nthreads) {
    const int c = i / (kStemPH * kStemPW), r = (i / kStemPW) % kStemPH, q = i % kStemPW;
    const int iy = 2 * oh0 - 3 + r, ix = 2 * ow0 - 3 + q;
    float v = 0.f;                                              // zero padding of the NORMALISED image
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = (img[((size_t)c * H + iy) * W + ix] - nmean[c]) * nrstd[c];
    patch[c][r][q] = v;
  }
}

__global__ void __launch_bounds__(128) stem_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, long s_co, long s_ci,
                                                       long s_ky, long s_kx, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, const float* __restrict__ mean,
                                                       const float* __restrict__ var, float eps, float3 nmean, float3 nrstd,
                                                       float* __restrict__ y, int N, int H, int W, int OH, int OW, int round_out) {
  DVD_PDL_ENTER();
  __shared__ float wsm[kStemTaps][64];                          // [c*49 + ky*7 + kx][co]
  __shared__ float patch[3][kStemPH][kStemPW];
  __shared__ float aff[2][64];
  for (int i = threadIdx.x; i < kStemTaps * 64; i += 128) {
    const int co = i % 64, t = i / 64;
    const int c = t / 49, ky = (t % 49) / 7, kx = t % 7;
    wsm[t][co] = w[co * s_co + c * s_ci + ky * s_ky + kx * s_kx];
  }
  if (threadIdx.x < 64) {
    const float sc = gamma[threadIdx.x] * rsqrtf(var[threadIdx.x] + eps);
    aff[0][threadIdx.x] = sc;
    aff[1][threadIdx.x] = beta[threadIdx.x] - mean[threadIdx.x] * sc;
  }
  const float nm[3] = {nmean.x, nmean.y, nmean.z}, nr[3] = {nrstd.x, nrstd.y, nrstd.z};
  const int tiles_w = (OW + kStemTW - 1) / kStemTW, tiles_h = (OH + kStemTH - 1) / kStemTH;
  const int ntiles = N * tiles_h * tiles_w;
  const int ty = threadIdx.x / kStemTW, tx = threadIdx.x % kStemTW;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int n = tile / (tiles_h * tiles_w), r = tile % (tiles_h * tiles_w);
    const int oh0 = (r / tiles_w) * kStemTH, ow0 = (r % tiles_w) * kStemTW;
    __syncthreads();
    stem_load_patch(patch, x + (size_t)n * 3 * H * W, H, W, oh0, ow0, nm, nr, 128);
    __syncthreads();
    float acc[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] = 0.f;
    for (int c = 0; c < 3; ++c)
      for (int ky = 0; ky < 7; ++ky)
#pragma unroll
        for (int kx = 0; kx < 7; ++kx) {
          const float xv = patch[c][2 * ty + ky][2 * tx + kx];
          const float4* wr = reinterpret_cast<const float4*>(wsm[c * 49 + ky * 7 + kx]);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const float4 wv = wr[j];
            acc[4 * j] = fmaf(xv, wv.x, acc[4 * j]); acc[4 * j + 1] = fmaf(xv, wv.y, acc[4 * j + 1]);
            acc[4 * j + 2] = fmaf(xv, wv.z, acc[4 * j + 2]); acc[4 * j + 3] = fmaf(xv, wv.w, acc[4 * j + 3]);
          }
        }
    const int oh = oh0 + ty, ow = ow0 + tx;
    if (oh < OH && ow < OW) {
      float4* dst = reinterpret_cast<float4*>(y + (((size_t)n * OH + oh) * OW + ow) * 64);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float4 v;
        v.x = fmaxf(fmaf(acc[4 * j], aff[0][4 * j], aff[1][4 * j]), 0.f);
        v.y = fmaxf(fmaf(acc[4 * j + 1], aff[0][4 * j + 1], aff[1][4 * j + 1]), 0.f);
        v.z = fmaxf(fmaf(acc[4 * j + 2], aff[0][4 * j + 2], aff[1][4 * j + 2]), 0.f);
        v.w = fmaxf(fmaf(acc[4 * j + 3], aff[0][4 * j + 3], aff[1][4 * j + 3]), 0.f);
        dst[j] = round_out ? round4(v) : v;
      }
    }
  }
}

// dWu[t][co] += sum_px gm[px][co] * xn[px, tap t];  gm = g * [a0 > 0];  bsum[co] += sum gm.   256 threads: thread owns the channel
// quad (tid % 16) and the taps tid/16 + 16 i (i < 10), accumulated in registers over all tiles of the CTA, one atomic flush.
template <bool ORD = false>
__global__ void __launch_bounds__(256) stem_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                         const float* __restrict__ a0, float3 nmean, float3 nrstd,
                                                         float* __restrict__ dwu, float* __restrict__ bsum, int N, int H, int W, int OH,
                                                         int OW, float* __restrict__ ord) {
  DVD_PDL_ENTER();
  __shared__ float patch[3][kStemPH][kStemPW];
  __shared__ __align__(16) float gsm[128][64];
  const float nm[3] = {nmean.x, nmean.y, nmean.z}, nr[3] = {nrstd.x, nrstd.y, nrstd.z};
  const int tiles_w = (OW + kStemTW - 1) / kStemTW, tiles_h = (OH + kStemTH - 1) / kStemTH;
  const int ntiles = N * tiles_h * tiles_w;
  const int cq = threadIdx.x % 16, tg = threadIdx.x / 16;
  int poff[10];                                 // patch offset of this thread's taps (channel-major), -1 = none
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const int t = tg + 16 * i;
    poff[i] = t < kStemTaps ? (t / 49) * (kStemPH * kStemPW) + ((t % 49) / 7) * kStemPW + (t % 7) : -1;
  }
  float acc[10][4];
#pragma unroll
  for (int i = 0; i < 10; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
  float bs[4] = {0.f, 0.f, 0.f, 0.f};
  const float* pbase = &patch[0][0][0];
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int n = tile / (tiles_h * tiles_w), r = tile % (tiles_h * tiles_w);
    const int oh0 = (r / tiles_w) * kStemTH, ow0 = (r % tiles_w) * kStemTW;
    __syncthreads();
    stem_load_patch(patch, x + (size_t)n * 3 * H * W, H, W, oh0, ow0, nm, nr, 256);
    for (int i = threadIdx.x; i < 128 * 16; i += 256) {
      const int px = i / 16, q = i % 16;
      const int oh = oh0 + px / kStemTW, ow = ow0 + px % kStemTW;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (oh < OH && ow < OW) {
        const size_t o = (((size_t)n * OH + oh) * OW + ow) * 64 + q * 4;
        v = *reinterpret_cast<const float4*>(g + o);
        const float4 a = *reinterpret_cast<const float4*>(a0 + o);
        v.x = a.x > 0.f ? v.x : 0.f; v.y = a.y > 0.f ? v.y : 0.f; v.z = a.z > 0.f ? v.z : 0.f; v.w = a.w > 0.f ? v.w : 0.f;
      }
      *reinterpret_cast<float4*>(&gsm[px][q * 4]) = v;
    }
    __syncthreads();
    for (int px = 0; px < 128; ++px) {
      const float4 gv = *reinterpret_cast<const float4*>(&gsm[px][cq * 4]);
      const int pb = (2 * (px / kStemTW)) * kStemPW + 2 * (px % kStemTW);
      if (tg == 0) { bs[0] += gv.x; bs[1] += gv.y; bs[2] += gv.z; bs[3] += gv.w; }
#pragma unroll
      for (int i = 0; i < 10; ++i) {
        if (poff[i] >= 0) {
          const float xv = pbase[poff[i] + pb];
          acc[i][0] = fmaf(gv.x, xv, acc[i][0]); acc[i][1] = fmaf(gv.y, xv, acc[i][1]);
          acc[i][2] = fmaf(gv.z, xv, acc[i][2]); acc[i][3] = fmaf(gv.w, xv, acc[i][3]);
        }
      }
    }
  }
  if constexpr (ORD) {        // ordered variant: this CTA's slab has the layout of (dwu, bsum); ordered_sum adds the slabs in CTA order
    dwu = ord + (size_t)blockIdx.x * (kStemTaps * 64 + 64);
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      const int t = tg + 16 * i;
      if (t < kStemTaps)
#pragma unroll
        for (int k = 0; k < 4; ++k) dwu[t * 64 + cq * 4 + k] = acc[i][k];
    }
    if (tg == 0)
#pragma unroll
      for (int k = 0; k < 4; ++k) dwu[kStemTaps * 64 + cq * 4 + k] = bs[k];
  } else {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const int t = tg + 16 * i;
    if (t < kStemTaps)
#pragma unroll
      for (int k = 0; k < 4; ++k) atomicAdd(dwu + t * 64 + cq * 4 + k, acc[i][k]);
  }
  if (tg == 0)
#pragma unroll
    for (int k = 0; k < 4; ++k) atomicAdd(bsum + cq * 4 + k, bs[k]);
  }
}

// dW[co] += sc[co] * dWu[co];  dgamma[co] += rstd[co] * (<W[co], dWu[co]> - mean[co] * bsum[co]);  dbeta[co] += bsum[co]
__global__ void __launch_bounds__(64) stem_wgrad_finalize_kernel(const float* __restrict__ dwu, const float* __restrict__ bsum,
                                                                 const float* __restrict__ w, float* __restrict__ dw, long s_co, long s_ci,
                                                                 long s_ky, long s_kx, const float* __restrict__ gamma,
                                                                 const float* __restrict__ mean, const float* __restrict__ var, float eps,
                                                                 float* __restrict__ dgamma, float* __restrict__ dbeta) {
  DVD_PDL_ENTER();
  const int co = threadIdx.x;
  const float rstd = rsqrtf(var[co] + eps), sc = gamma[co] * rstd;
  float dot = 0.f;
  for (int t = 0; t < kStemTaps; ++t) {
    const long o = co * s_co + (t / 49) * s_ci + ((t % 49) / 7) * s_ky + (t % 7) * s_kx;
    const float v = dwu[t * 64 + co];
    dot = fmaf(v, w[o], dot);
    dw[o] += sc * v;
  }
  dgamma[co] += rstd * (dot - mean[co] * bsum[co]);
  dbeta[co] += bsum[co];
}

// ---- head: depth = 10000 / max(relu(<x[p,:], w> + b), 1e-2) ------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) head_fwd_kernel(const float4* __restrict__ x, const float* __restrict__ w,
                                                            const float* __restrict__ b, float* __restrict__ depth, long P) {
  DVD_PDL_ENTER();
  __shared__ float ws[32];
  if (threadIdx.x < 32) ws[threadIdx.x] = w[threadIdx.x];
  __syncthreads();
  const float bias = b[0];
  const long stride = (long)gridDim.x * blockDim.x;
  for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += stride) {
    float o = bias;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 v = ldg_stream4(reinterpret_cast<const float*>(x + p * 8 + j));
      o = fmaf(v.x, ws[4 * j], o); o = fmaf(v.y, ws[4 * j + 1], o); o = fmaf(v.z, ws[4 * j + 2], o); o = fmaf(v.w, ws[4 * j + 3], o);
    }
    depth[p] = 10000.0f / fmaxf(fmaxf(o, 0.f), 1e-2f);
  }
}

template <bool ORD = false>
__global__ void __launch_bounds__(kThreads) head_bwd_kernel(const float4* __restrict__ x, const float* __restrict__ w,
                                                            const float* __restrict__ b, const float* __restrict__ gd,
                                                            float4* __restrict__ gx, float* __restrict__ gw, float* __restrict__ gb, long P,
                                                            int relu_mask, int round_out, float* __restrict__ ord) {
  DVD_PDL_ENTER();
  __shared__ float ws[32];
  __shared__ float red[kThreads / 32][33];
  if (threadIdx.x < 32) ws[threadIdx.x] = w[threadIdx.x];
  __syncthreads();
  const float bias = b[0];
  float aw[32], ab = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) aw[j] = 0.f;
  const long stride = (long)gridDim.x * blockDim.x;
  for (long p = (long)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += stride) {
    float4 v[8];
    float o = bias;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      v[j] = x[p * 8 + j];
      o = fmaf(v[j].x, ws[4 * j], o); o = fmaf(v[j].y, ws[4 * j + 1], o); o = fmaf(v[j].z, ws[4 * j + 2], o); o = fmaf(v[j].w, ws[4 * j + 3], o);
    }
    // d = 10000 / clamp(relu(o), 1e-2): gradient passes where o >= 1e-2 (torch.clamp backward: self >= min)
    const float go = o >= 1e-2f ? -gd[p] * 10000.0f / (o * o) : 0.f;
    ab += go;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      aw[4 * j] = fmaf(go, v[j].x, aw[4 * j]); aw[4 * j + 1] = fmaf(go, v[j].y, aw[4 * j + 1]);
      aw[4 * j + 2] = fmaf(go, v[j].z, aw[4 * j + 2]); aw[4 * j + 3] = fmaf(go, v[j].w, aw[4 * j + 3]);
      float4 o4 = make_float4(go * ws[4 * j], go * ws[4 * j + 1], go * ws[4 * j + 2], go * ws[4 * j + 3]);
      if (relu_mask) {     // x = relu(.) of the producing convolution: gradient w.r.t. its pre-activation
        o4.x = v[j].x > 0.f ? o4.x : 0.f; o4.y = v[j].y > 0.f ? o4.y : 0.f;
        o4.z = v[j].z > 0.f ? o4.z : 0.f; o4.w = v[j].w > 0.f ? o4.w : 0.f;
      }
      gx[p * 8 + j] = round_out ? round4(o4) : o4;
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float s = warp_sum(aw[j]);
    if (lane == 0) red[warp][j] = s;
  }
  {
    const float s = warp_sum(ab);
    if (lane == 0) red[warp][32] = s;
  }
  __syncthreads();
  if (threadIdx.x < 33) {
    float s = 0.f;
    for (int k = 0; k < kThreads / 32; ++k) s += red[k][threadIdx.x];
    if constexpr (ORD) ord[(size_t)blockIdx.x * 33 + threadIdx.x] = s;     // ordered variant: added in CTA order by ordered_sum
    else atomicAdd(threadIdx.x < 32 ? gw + threadIdx.x : gb, s);
  }
}

}  // namespace
}  // namespace dvd

using namespace dvd;

extern "C" int dvd_round_tf32(const float* x, float* y, long n, void* stream) {
  DVD_ARG_CHECK(x && y && n > 0 && n % 4 == 0 && aligned16(x) && aligned16(y), "needs 16-byte aligned buffers and n %% 4 == 0");
  dvd::launch(round_kernel, blocks_for(n / 4), kThreads, 0, (cudaStream_t)stream, (const float4*)x, (float4*)y, n / 4);
  DVD_CUDA_LAUNCH_CHECK("round_kernel");
  return 0;
}

static int relu_bwd_colsum(const float* g, const float* y, float* gm, float* colsum, const float* bn_mean, const float* bn_var,
                           float bn_eps, float* dgamma, long P, int C, int round_out, void* ws, size_t ws_bytes, void* stream) {
  DVD_ARG_CHECK(g && P > 0 && C > 0 && C % 4 == 0, "bad arguments (C must be a multiple of 4)");
  DVD_ARG_CHECK(!dgamma || (bn_mean && bn_var), "dgamma needs the BatchNorm statistics");
  DVD_ARG_CHECK(aligned16(g) && (!y || aligned16(y)) && (!gm || aligned16(gm)), "buffers must be 16-byte aligned");
  const int c4 = C / 4;
  int cgb = 64;
  while (cgb > c4) cgb >>= 1;
  if (cgb < 1) cgb = 1;
  const int rows = kThreads / cgb;
  long gx_blocks = (P + (long)rows * 8 - 1) / ((long)rows * 8);
  const long cap = ((long)num_sms() * 8 * cgb) / c4 + 1;
  if (gx_blocks > cap) gx_blocks = cap;
  if (gx_blocks < 1) gx_blocks = 1;
  dim3 grid((unsigned)gx_blocks, (unsigned)((c4 + cgb - 1) / cgb));
  if (ws && (colsum || dgamma)) {
    DVD_ARG_CHECK(aligned16(ws) && (size_t)gx_blocks * C * sizeof(float) <= ws_bytes,
                  "ordered column sums: the workspace needs dvd_ordered_workspace_bytes(DVD_ORD_CHANNEL_SUMS) bytes (C <= %d)",
                  DVD_ORD_MAX_CHANNELS);
    dvd::launch(relu_bwd_colsum_kernel<true>, grid, kThreads, 0, (cudaStream_t)stream, (const float4*)g, (const float4*)y, (float4*)gm,
                colsum, bn_mean, bn_var, bn_eps, dgamma, P, c4, cgb, round_out, (float*)ws);
    DVD_CUDA_LAUNCH_CHECK("relu_bwd_colsum_kernel<ordered>");
    dvd::launch(colsum_ordered_reduce_kernel, (unsigned)((C + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream,
                (const float*)ws, (int)gx_blocks, C, colsum, bn_mean, bn_var, bn_eps, dgamma);
    DVD_CUDA_LAUNCH_CHECK("colsum_ordered_reduce_kernel");
    return 0;
  }
  dvd::launch(relu_bwd_colsum_kernel<>, grid, kThreads, 0, (cudaStream_t)stream, (const float4*)g, (const float4*)y, (float4*)gm, colsum, bn_mean,
                                                                    bn_var, bn_eps, dgamma, P, c4, cgb, round_out, (float*)nullptr);
  DVD_CUDA_LAUNCH_CHECK("relu_bwd_colsum_kernel");
  return 0;
}

extern "C" int dvd_relu_bwd_colsum(const float* g, const float* y, float* gm, float* colsum, const float* bn_mean, const float* bn_var,
                                   float bn_eps, float* dgamma, long P, int C, int round_out, void* stream) {
  return relu_bwd_colsum(g, y, gm, colsum, bn_mean, bn_var, bn_eps, dgamma, P, C, round_out, nullptr, 0, stream);
}
extern "C" int dvd_relu_bwd_colsum_ordered(const float* g, const float* y, float* gm, float* colsum, const float* bn_mean,
                                           const float* bn_var, float bn_eps, float* dgamma, long P, int C, int round_out, void* ws,
                                           size_t ws_bytes, void* stream) {
  DVD_ARG_CHECK(ws != nullptr, "dvd_relu_bwd_colsum_ordered: null workspace");
  return relu_bwd_colsum(g, y, gm, colsum, bn_mean, bn_var, bn_eps, dgamma, P, C, round_out, ws, ws_bytes, stream);
}

extern "C" int dvd_maxpool3x3s2_fwd(const float* x, float* y, unsigned char* idx, int N, int H, int W, int C, void* stream) {
  DVD_ARG_CHECK(x && y && idx && N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, "bad arguments (C must be a multiple of 4)");
  const int OH = (H + 2 - 3) / 2 + 1, OW = (W + 2 - 3) / 2 + 1;
  const long total = (long)N * OH * OW * (C / 4);
  dvd::launch(maxpool_fwd_kernel, blocks_for(total), kThreads, 0, (cudaStream_t)stream, (const float4*)x, (float4*)y, (uchar4*)idx, N, H, W, OH, OW,
                                                                             C / 4);
  DVD_CUDA_LAUNCH_CHECK("maxpool_fwd_kernel");
  return 0;
}

extern "C" int dvd_maxpool3x3s2_bwd(const float* g, const unsigned char* idx, float* gx, int N, int H, int W, int C, void* stream) {
  DVD_ARG_CHECK(g && gx && idx && N > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, "bad arguments (C must be a multiple of 4)");
  const int OH = (H + 2 - 3) / 2 + 1, OW = (W + 2 - 3) / 2 + 1;
  const long total = (long)N * H * W * (C / 4);
  dvd::launch(maxpool_bwd_kernel, blocks_for(total), kThreads, 0, (cudaStream_t)stream, (const float4*)g, (const uchar4*)idx, (float4*)gx, N, H, W, OH,
                                                                             OW, C / 4);
  DVD_CUDA_LAUNCH_CHECK("maxpool_bwd_kernel");
  return 0;
}

extern "C" int dvd_stem_fwd(const float* x_nchw, const float* weight, long s_co, long s_ci, long s_ky, long s_kx, const float* bn_gamma,
                            const float* bn_beta, const float* bn_mean, const float* bn_var, float bn_eps, const float* norm_mean3,
                            const float* norm_std3, float* y, int N, int H, int W, int round_out, void* stream) {
  DVD_ARG_CHECK(x_nchw && weight && bn_gamma && bn_beta && bn_mean && bn_var && y, "null pointer");
  DVD_ARG_CHECK(N > 0 && H > 0 && W > 0, "bad shape");
  const int OH = (H + 6 - 7) / 2 + 1, OW = (W + 6 - 7) / 2 + 1;
  float3 nm = make_float3(0.f, 0.f, 0.f), nr = make_float3(1.f, 1.f, 1.f);
  if (norm_mean3) nm = make_float3(norm_mean3[0], norm_mean3[1], norm_mean3[2]);       // HOST pointers (3 constants)
  if (norm_std3) nr = make_float3(1.0f / norm_std3[0], 1.0f / norm_std3[1], 1.0f / norm_std3[2]);
  const int ntiles = N * ((OH + kStemTH - 1) / kStemTH) * ((OW + kStemTW - 1) / kStemTW);
  int grid = num_sms() * 4;
  if (grid > ntiles) grid = ntiles;
  dvd::launch(stem_fwd_kernel, grid, 128, 0, (cudaStream_t)stream, x_nchw, weight, s_co, s_ci, s_ky, s_kx, bn_gamma, bn_beta, bn_mean, bn_var, bn_eps,
                                                        nm, nr, y, N, H, W, OH, OW, round_out);
  DVD_CUDA_LAUNCH_CHECK("stem_fwd_kernel");
  return 0;
}

static int stem_wgrad(const float* x_nchw, const float* g, const float* a0, const float* weight, float* dweight, long s_co,
                      long s_ci, long s_ky, long s_kx, const float* bn_gamma, const float* bn_mean, const float* bn_var,
                      float bn_eps, float* dgamma, float* dbeta, const float* norm_mean3, const float* norm_std3, float* scratch,
                      int N, int H, int W, void* ws, size_t ws_bytes, void* stream) {
  DVD_ARG_CHECK(x_nchw && g && a0 && weight && dweight && bn_gamma && bn_mean && bn_var && dgamma && dbeta && scratch, "null pointer");
  DVD_ARG_CHECK(N > 0 && H > 0 && W > 0, "bad shape");
  const int OH = (H + 6 - 7) / 2 + 1, OW = (W + 6 - 7) / 2 + 1;
  float3 nm = make_float3(0.f, 0.f, 0.f), nr = make_float3(1.f, 1.f, 1.f);
  if (norm_mean3) nm = make_float3(norm_mean3[0], norm_mean3[1], norm_mean3[2]);
  if (norm_std3) nr = make_float3(1.0f / norm_std3[0], 1.0f / norm_std3[1], 1.0f / norm_std3[2]);
  DVD_CUDA_CALL(cudaMemsetAsync(scratch, 0, (kStemTaps * 64 + 64) * sizeof(float), (cudaStream_t)stream));
  const int ntiles = N * ((OH + kStemTH - 1) / kStemTH) * ((OW + kStemTW - 1) / kStemTW);
  int grid = num_sms() * 2;
  if (grid > ntiles) grid = ntiles;
  if (ws) {
    constexpr int kSlab = kStemTaps * 64 + 64;
    DVD_ARG_CHECK(aligned16(ws) && (size_t)grid * kSlab * sizeof(float) <= ws_bytes,
                  "ordered stem weight gradient: the workspace needs dvd_ordered_workspace_bytes(DVD_ORD_STEM) bytes");
    dvd::launch(stem_wgrad_kernel<true>, grid, 256, 0, (cudaStream_t)stream, x_nchw, g, a0, nm, nr, scratch, scratch + kStemTaps * 64, N,
                H, W, OH, OW, (float*)ws);
    DVD_CUDA_LAUNCH_CHECK("stem_wgrad_kernel<ordered>");
    if (int e = launch_ordered_sum((const float*)ws, grid, kSlab, scratch, kSlab, nullptr, (cudaStream_t)stream)) return e;
  } else {
    dvd::launch(stem_wgrad_kernel<>, grid, 256, 0, (cudaStream_t)stream, x_nchw, g, a0, nm, nr, scratch, scratch + kStemTaps * 64, N, H, W,
                OH, OW, (float*)nullptr);
    DVD_CUDA_LAUNCH_CHECK("stem_wgrad_kernel");
  }
  dvd::launch(stem_wgrad_finalize_kernel, 1, 64, 0, (cudaStream_t)stream, scratch, scratch + kStemTaps * 64, weight, dweight, s_co, s_ci, s_ky, s_kx,
                                                                bn_gamma, bn_mean, bn_var, bn_eps, dgamma, dbeta);
  DVD_CUDA_LAUNCH_CHECK("stem_wgrad_finalize_kernel");
  return 0;
}

extern "C" int dvd_stem_wgrad(const float* x_nchw, const float* g, const float* a0, const float* weight, float* dweight, long s_co,
                              long s_ci, long s_ky, long s_kx, const float* bn_gamma, const float* bn_mean, const float* bn_var,
                              float bn_eps, float* dgamma, float* dbeta, const float* norm_mean3, const float* norm_std3, float* scratch,
                              int N, int H, int W, void* stream) {
  return stem_wgrad(x_nchw, g, a0, weight, dweight, s_co, s_ci, s_ky, s_kx, bn_gamma, bn_mean, bn_var, bn_eps, dgamma, dbeta, norm_mean3,
                    norm_std3, scratch, N, H, W, nullptr, 0, stream);
}
extern "C" int dvd_stem_wgrad_ordered(const float* x_nchw, const float* g, const float* a0, const float* weight, float* dweight,
                                      long s_co, long s_ci, long s_ky, long s_kx, const float* bn_gamma, const float* bn_mean,
                                      const float* bn_var, float bn_eps, float* dgamma, float* dbeta, const float* norm_mean3,
                                      const float* norm_std3, float* scratch, int N, int H, int W, void* ws, size_t ws_bytes,
                                      void* stream) {
  DVD_ARG_CHECK(ws != nullptr, "dvd_stem_wgrad_ordered: null workspace");
  return stem_wgrad(x_nchw, g, a0, weight, dweight, s_co, s_ci, s_ky, s_kx, bn_gamma, bn_mean, bn_var, bn_eps, dgamma, dbeta, norm_mean3,
                    norm_std3, scratch, N, H, W, ws, ws_bytes, stream);
}

extern "C" int dvd_head_fwd(const float* x, const float* w, const float* b, float* depth, long P, void* stream) {
  DVD_ARG_CHECK(x && w && b && depth && P > 0 && aligned16(x), "bad arguments");
  dvd::launch(head_fwd_kernel, blocks_for(P), kThreads, 0, (cudaStream_t)stream, (const float4*)x, w, b, depth, P);
  DVD_CUDA_LAUNCH_CHECK("head_fwd_kernel");
  return 0;
}

static int head_bwd(const float* x, const float* w, const float* b, const float* g_depth, float* gx, float* gw, float* gb, long P,
                    int relu_mask, int round_out, void* ws, size_t ws_bytes, void* stream) {
  DVD_ARG_CHECK(x && w && b && g_depth && gx && gw && gb && P > 0 && aligned16(x) && aligned16(gx), "bad arguments");
  if (ws) {
    const unsigned grid = blocks_for(P, 4);
    DVD_ARG_CHECK(aligned16(ws) && (size_t)grid * 33 * sizeof(float) <= ws_bytes,
                  "ordered head gradient: the workspace needs dvd_ordered_workspace_bytes(DVD_ORD_HEAD) bytes");
    dvd::launch(head_bwd_kernel<true>, grid, kThreads, 0, (cudaStream_t)stream, (const float4*)x, w, b, g_depth, (float4*)gx, gw, gb, P,
                relu_mask, round_out, (float*)ws);
    DVD_CUDA_LAUNCH_CHECK("head_bwd_kernel<ordered>");
    return launch_ordered_sum((const float*)ws, (int)grid, 33, gw, 32, gb, (cudaStream_t)stream);
  }
  dvd::launch(head_bwd_kernel<>, blocks_for(P, 4), kThreads, 0, (cudaStream_t)stream, (const float4*)x, w, b, g_depth, (float4*)gx, gw, gb, P, relu_mask, round_out,
              (float*)nullptr);
  DVD_CUDA_LAUNCH_CHECK("head_bwd_kernel");
  return 0;
}

extern "C" int dvd_head_bwd(const float* x, const float* w, const float* b, const float* g_depth, float* gx, float* gw, float* gb, long P,
                            int relu_mask, int round_out, void* stream) {
  return head_bwd(x, w, b, g_depth, gx, gw, gb, P, relu_mask, round_out, nullptr, 0, stream);
}
extern "C" int dvd_head_bwd_ordered(const float* x, const float* w, const float* b, const float* g_depth, float* gx, float* gw,
                                    float* gb, long P, int relu_mask, int round_out, void* ws, size_t ws_bytes, void* stream) {
  DVD_ARG_CHECK(ws != nullptr, "dvd_head_bwd_ordered: null workspace");
  return head_bwd(x, w, b, g_depth, gx, gw, gb, P, relu_mask, round_out, ws, ws_bytes, stream);
}
