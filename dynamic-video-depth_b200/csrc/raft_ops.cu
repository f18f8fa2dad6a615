// CUDA-core members of the RAFT optical-flow forward (third_party/RAFT/core of the reference, large model, test mode).
// Everything here is NHWC fp32; the tensor-core convolutions between these kernels are conv2d_tc.cu's, under its
// rounded-operand contract, so every producer of a convolution operand has a `round_out` switch.
//   * dvd_raft_stem_fwd        7x7 stride-2 3 -> 64 convolution on 2 (x / 255) - 1 (fnet: InstanceNorm follows)
//   * dvd_raft_instnorm_stats  per (image, channel) mean and 1 / sqrt(var + eps), fixed reduction order, fp64 sums
//   * dvd_raft_norm_act        y = relu?( relu?((x - mean) * rstd) + res )
//   * dvd_raft_corr_pyramid    all-pairs correlation in plain fp32 FMA and its three 2x2 average poolings
//   * dvd_raft_lookup          4 levels x 81 bilinear samples per pixel -> the motion encoder's 352-channel operand
//   * dvd_raft_convf1          7x7 2 -> 128 on flow = coords1 - grid, ReLU
//   * dvd_raft_motion_pack     [relu(conv)(126) | flow(2)] into both GRU operands
//   * dvd_raft_gru_rh / dvd_raft_gru_update   the GRU's elementwise stages
//   * dvd_raft_flow_head       3x3 256 -> 2 and coords1 += delta_flow
//   * dvd_raft_upsample        0.25 * mask -> softmax over 9 -> convex 8x up-sampling, flow as [B,H,W,2]
// No kernel uses atomics: equal inputs give bitwise equal outputs.
#include "common.cuh"

namespace dvd {
namespace {

constexpr int kLevels = 4, kRadius = 4, kWin = 2 * kRadius + 1, kLookupC = kLevels * kWin * kWin, kLookupPad = 352;
constexpr int kStatChunks = 64;

__device__ __forceinline__ float round_tf32(float v) {
  uint32_t o;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(o) : "f"(v));
  return __uint_as_float(o);
}
__device__ __forceinline__ float4 round4(float4 v, int on) {
  return on ? make_float4(round_tf32(v.x), round_tf32(v.y), round_tf32(v.z), round_tf32(v.w)) : v;
}
__device__ __forceinline__ float sigmoidf(float x) { return 1.0f / (1.0f + expf(-x)); }

#define RAFT_CHECK(cond, ...)      \
  do {                             \
    if (!(cond)) {                 \
      dvd::set_error(__VA_ARGS__); \
      return -2;                   \
    }                              \
  } while (0)

// ---- stem --------------------------------------------------------------------------------------------------------------
// one thread per output pixel, 64 accumulators; the weights sit in shared memory as [tap][64] and are read as broadcasts
__global__ void __launch_bounds__(128) raft_stem_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                        const float* __restrict__ bias, float* __restrict__ y, int N, int H, int W,
                                                        int OH, int OW) {
  __shared__ __align__(16) float ws[147 * 64];
  for (int i = threadIdx.x; i < 147 * 64; i += blockDim.x) {
    const int co = i / 147, t = i % 147;          // w is [64][3][7][7]
    ws[t * 64 + co] = w[i];
  }
  __syncthreads();
  DVD_PDL_ENTER();
  const long total = (long)N * OH * OW;
  const long o = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= total) return;
  const int ox = (int)(o % OW), oy = (int)((o / OW) % OH), n = (int)(o / ((long)OW * OH));
  float acc[64];
#pragma unroll
  for (int c = 0; c < 64; ++c) acc[c] = bias[c];
  for (int ci = 0; ci < 3; ++ci) {
    const float* xp = x + ((long)n * 3 + ci) * H * W;
    for (int ky = 0; ky < 7; ++ky) {
      const int iy = 2 * oy + ky - 3;
      if (iy < 0 || iy >= H) continue;
      for (int kx = 0; kx < 7; ++kx) {
        const int ix = 2 * ox + kx - 3;
        if (ix < 0 || ix >= W) continue;
        const float v = 2.0f * (xp[(long)iy * W + ix] / 255.0f) - 1.0f;
        const float4* wr = reinterpret_cast<const float4*>(ws + ((ci * 7 + ky) * 7 + kx) * 64);
#pragma unroll
        for (int c = 0; c < 16; ++c) {
          const float4 wv = wr[c];
          acc[4 * c + 0] = fmaf(v, wv.x, acc[4 * c + 0]);
          acc[4 * c + 1] = fmaf(v, wv.y, acc[4 * c + 1]);
          acc[4 * c + 2] = fmaf(v, wv.z, acc[4 * c + 2]);
          acc[4 * c + 3] = fmaf(v, wv.w, acc[4 * c + 3]);
        }
      }
    }
  }
  float4* yp = reinterpret_cast<float4*>(y + o * 64);
#pragma unroll
  for (int c = 0; c < 16; ++c) yp[c] = make_float4(acc[4 * c], acc[4 * c + 1], acc[4 * c + 2], acc[4 * c + 3]);
}

// ---- InstanceNorm ------------------------------------------------------------------------------------------------------
// block (n, chunk): threads = (C / 4 channel quads) x lanes; every thread sums its pixels of the chunk in fp64, the lanes are
// combined in lane order, and the chunk's (sum, sum of squares) goes to partials[n][chunk][C][2]
__global__ void __launch_bounds__(256) instnorm_partial_kernel(const float* __restrict__ x, double* __restrict__ partials, long P, int C) {
  extern __shared__ double sm[];     // [lanes][C][2]
  DVD_PDL_ENTER();
  const int quads = C / 4, lanes = blockDim.x / quads;
  const int q = threadIdx.x % quads, lane = threadIdx.x / quads;
  const int n = blockIdx.y, chunk = blockIdx.x;
  const long per = (P + kStatChunks - 1) / kStatChunks, p0 = chunk * per, p1 = p0 + per < P ? p0 + per : P;
  double s[4] = {0, 0, 0, 0}, ss[4] = {0, 0, 0, 0};
  if (lane < lanes) {
    for (long p = p0 + lane; p < p1; p += lanes) {
      const float4 v = *reinterpret_cast<const float4*>(x + ((long)n * P + p) * C + 4 * q);
      s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += v.w;
      ss[0] += (double)v.x * v.x; ss[1] += (double)v.y * v.y; ss[2] += (double)v.z * v.z; ss[3] += (double)v.w * v.w;
    }
    for (int k = 0; k < 4; ++k) {
      sm[((long)lane * C + 4 * q + k) * 2 + 0] = s[k];
      sm[((long)lane * C + 4 * q + k) * 2 + 1] = ss[k];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
    double a = 0;
    for (int l = 0; l < lanes; ++l) a += sm[(long)l * C * 2 + i];
    partials[((long)n * kStatChunks + chunk) * C * 2 + i] = a;
  }
}

__global__ void instnorm_final_kernel(const double* __restrict__ partials, float* __restrict__ stats, long P, int C, int N, float eps) {
  DVD_PDL_ENTER();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  const int n = i / C, c = i % C;
  double s = 0, ss = 0;
  for (int k = 0; k < kStatChunks; ++k) {
    s += partials[(((long)n * kStatChunks + k) * C + c) * 2 + 0];
    ss += partials[(((long)n * kStatChunks + k) * C + c) * 2 + 1];
  }
  const double mean = s / (double)P;
  double var = ss / (double)P - mean * mean;     // biased, as nn.InstanceNorm2d
  if (var < 0) var = 0;
  stats[2 * i + 0] = (float)mean;
  stats[2 * i + 1] = (float)(1.0 / sqrt(var + (double)eps));
}

__global__ void norm_act_kernel(const float* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ res,
                                float* __restrict__ y, long P, int C, long total4, int relu_inner, int relu_outer, int round_out) {
  DVD_PDL_ENTER();
  const int quads = C / 4;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (long)gridDim.x * blockDim.x) {
    float4 v = reinterpret_cast<const float4*>(x)[i];
    if (stats) {
      const int c = (int)(i % quads) * 4;
      const long n = i / (P * quads);
      const float4 a = *reinterpret_cast<const float4*>(stats + (n * C + c) * 2);       // mean, rstd, mean, rstd
      const float4 b = *reinterpret_cast<const float4*>(stats + (n * C + c) * 2 + 4);
      v.x = (v.x - a.x) * a.y; v.y = (v.y - a.z) * a.w; v.z = (v.z - b.x) * b.y; v.w = (v.w - b.z) * b.w;
    }
    if (relu_inner) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    if (res) {
      const float4 r = reinterpret_cast<const float4*>(res)[i];
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    if (relu_outer) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    reinterpret_cast<float4*>(y)[i] = round4(v, round_out);
  }
}

// ---- correlation volume: C[b][p][q] = scale * sum_c A[b][p][c] B[b][q][c], fp32 FMA, 64 x 64 tiles, 4 x 4 per thread ------
constexpr int kCT = 64, kCK = 16;
__global__ void __launch_bounds__(256) corr_kernel(const float* __restrict__ A, const float* __restrict__ Bm, float* __restrict__ Cm,
                                                   int P, int K, float scale) {
  __shared__ float As[kCK][kCT + 4], Bs[kCK][kCT + 4];
  DVD_PDL_ENTER();
  const int b = blockIdx.z, p0 = blockIdx.y * kCT, q0 = blockIdx.x * kCT;
  const float* Ab = A + (long)b * P * K;
  const float* Bb = Bm + (long)b * P * K;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int lr = threadIdx.x / 4, lk = (threadIdx.x % 4) * 4;       // this thread loads row lr, k = lk .. lk + 3 of both tiles
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += kCK) {
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 av = p0 + lr < P ? *reinterpret_cast<const float4*>(Ab + (long)(p0 + lr) * K + k0 + lk) : z;
    const float4 bv = q0 + lr < P ? *reinterpret_cast<const float4*>(Bb + (long)(q0 + lr) * K + k0 + lk) : z;
    As[lk + 0][lr] = av.x; As[lk + 1][lr] = av.y; As[lk + 2][lr] = av.z; As[lk + 3][lr] = av.w;
    Bs[lk + 0][lr] = bv.x; Bs[lk + 1][lr] = bv.y; Bs[lk + 2][lr] = bv.z; Bs[lk + 3][lr] = bv.w;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kCK; ++k) {
      float a[4], bb[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[k][ty * 4 + i]; bb[i] = Bs[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
  for (int i = 0; i < 4; ++i) {
    const int p = p0 + ty * 4 + i;
    if (p >= P) continue;
    for (int j = 0; j < 4; ++j) {
      const int q = q0 + tx * 4 + j;
      if (q < P) Cm[((long)b * P + p) * P + q] = acc[i][j] * scale;
    }
  }
}

// one pyramid level from the one below: rows = B * P correlation maps of hi x wi -> ho x wo (floor), 2 x 2 average
__global__ void corr_pool_kernel(const float* __restrict__ src, float* __restrict__ dst, long rows, int hi, int wi, int ho, int wo) {
  DVD_PDL_ENTER();
  const long total = rows * ho * wo;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int x = (int)(i % wo), y = (int)((i / wo) % ho);
    const long r = i / ((long)wo * ho);
    const float* s = src + (r * hi + 2 * y) * wi + 2 * x;
    dst[i] = (s[0] + s[1] + s[wi] + s[wi + 1]) * 0.25f;
  }
}

struct Levels {
  long off[kLevels];     // offset of the level's [B * P][h * w] block in the pyramid buffer (floats)
  int h[kLevels], w[kLevels];
};

// block = one pixel p of one pair; thread k < 324 samples channel k, the rest write the zero tail
__global__ void __launch_bounds__(kLookupPad) lookup_kernel(const float* __restrict__ pyr, const float* __restrict__ coords1,
                                                            float* __restrict__ out, Levels L, int round_out) {
  DVD_PDL_ENTER();
  const long bp = blockIdx.x;
  const int k = threadIdx.x;
  float v = 0.f;
  if (k < kLookupC) {
    const int l = k / (kWin * kWin), r = k % (kWin * kWin);
    const float2 c = reinterpret_cast<const float2*>(coords1)[bp];
    const float inv = 1.0f / (float)(1 << l);
    // the window's slow index moves along x (the reference adds its meshgrid(dy, dx) pairs to (x, y) coordinates)
    const float x = c.x * inv + (float)(r / kWin - kRadius), y = c.y * inv + (float)(r % kWin - kRadius);
    const int h = L.h[l], w = L.w[l];
    const float* m = pyr + L.off[l] + bp * (long)h * w;
    const float xf = floorf(x), yf = floorf(y);
    const float ax = x - xf, ay = y - yf;
    // coordinates far outside (or not finite) sample nothing
    if (xf >= -1.f && xf <= (float)w && yf >= -1.f && yf <= (float)h) {
      const int x0 = (int)xf, y0 = (int)yf;
      const bool xl = x0 >= 0 && x0 < w, xr = x0 + 1 >= 0 && x0 + 1 < w, yt = y0 >= 0 && y0 < h, yb = y0 + 1 >= 0 && y0 + 1 < h;
      const float v00 = (xl && yt) ? m[(long)y0 * w + x0] : 0.f, v01 = (xr && yt) ? m[(long)y0 * w + x0 + 1] : 0.f;
      const float v10 = (xl && yb) ? m[(long)(y0 + 1) * w + x0] : 0.f, v11 = (xr && yb) ? m[(long)(y0 + 1) * w + x0 + 1] : 0.f;
      v = (1.f - ay) * ((1.f - ax) * v00 + ax * v01) + ay * ((1.f - ax) * v10 + ax * v11);
    }
  }
  out[bp * kLookupPad + k] = round_out ? round_tf32(v) : v;
}

// ---- convf1: 7x7, 2 -> 128 on flow = coords1 - grid (zero outside), ReLU. Block: 128 threads (one per output channel) x 16
// pixels of one row; the flow patch 7 x 22 x 2 sits in shared memory
constexpr int kF1Px = 16;
__global__ void __launch_bounds__(128) convf1_kernel(const float* __restrict__ coords1, const float* __restrict__ w,
                                                     const float* __restrict__ bias, float* __restrict__ y, int h, int wd,
                                                     int round_out) {
  __shared__ float2 patch[7][kF1Px + 6];
  DVD_PDL_ENTER();
  const int xt = blockIdx.x * kF1Px, yy = blockIdx.y, b = blockIdx.z;
  for (int i = threadIdx.x; i < 7 * (kF1Px + 6); i += blockDim.x) {
    const int py = i / (kF1Px + 6), px = i % (kF1Px + 6);
    const int sy = yy + py - 3, sx = xt + px - 3;
    float2 f = make_float2(0.f, 0.f);
    if (sy >= 0 && sy < h && sx >= 0 && sx < wd) {
      const float2 c = reinterpret_cast<const float2*>(coords1)[((long)b * h + sy) * wd + sx];
      f = make_float2(c.x - (float)sx, c.y - (float)sy);
    }
    patch[py][px] = f;
  }
  __syncthreads();
  const int co = threadIdx.x;
  float acc[kF1Px];
  const float bv = bias[co];
#pragma unroll
  for (int p = 0; p < kF1Px; ++p) acc[p] = bv;
  const float* wc = w + (long)co * 98;        // [128][2][7][7]
  for (int ky = 0; ky < 7; ++ky)
    for (int kx = 0; kx < 7; ++kx) {
      const float w0 = wc[ky * 7 + kx], w1 = wc[49 + ky * 7 + kx];
#pragma unroll
      for (int p = 0; p < kF1Px; ++p) {
        const float2 f = patch[ky][p + kx];
        acc[p] = fmaf(w1, f.y, fmaf(w0, f.x, acc[p]));
      }
    }
  for (int p = 0; p < kF1Px; ++p) {
    if (xt + p >= wd) break;
    const float v = fmaxf(acc[p], 0.f);
    y[(((long)b * h + yy) * wd + xt + p) * 128 + co] = round_out ? round_tf32(v) : v;
  }
}

// ---- GRU operands: X = [h | inp | motion] and XR = [r h | inp | motion], 384 channels each; motion = [relu(conv) 126 | flow 2]
__global__ void motion_pack_kernel(const float* __restrict__ mconv, const float* __restrict__ coords1, float* __restrict__ X,
                                   float* __restrict__ XR, long npx, int h, int wd) {
  DVD_PDL_ENTER();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < npx * 32; i += (long)gridDim.x * blockDim.x) {
    const long p = i / 32;
    const int q = (int)(i % 32);
    float4 v = reinterpret_cast<const float4*>(mconv)[i];
    if (q == 31) {
      const int x = (int)(p % wd), y = (int)((p / wd) % h);
      const float2 c = reinterpret_cast<const float2*>(coords1)[p];
      v.z = round_tf32(c.x - (float)x);
      v.w = round_tf32(c.y - (float)y);
    }
    reinterpret_cast<float4*>(X + p * 384 + 256)[q] = v;
    reinterpret_cast<float4*>(XR + p * 384 + 256)[q] = v;
  }
}

// XR[:, 0:128] = round(sigmoid(zr[:, 128:256]) * net)
__global__ void gru_rh_kernel(const float* __restrict__ zr, const float* __restrict__ net, float* __restrict__ XR, long npx) {
  DVD_PDL_ENTER();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < npx * 32; i += (long)gridDim.x * blockDim.x) {
    const long p = i / 32;
    const int q = (int)(i % 32);
    const float4 r = reinterpret_cast<const float4*>(zr + p * 256 + 128)[q];
    const float4 hv = reinterpret_cast<const float4*>(net)[i];
    const float4 o = make_float4(sigmoidf(r.x) * hv.x, sigmoidf(r.y) * hv.y, sigmoidf(r.z) * hv.z, sigmoidf(r.w) * hv.w);
    reinterpret_cast<float4*>(XR + p * 384)[q] = round4(o, 1);
  }
}

__device__ __forceinline__ float gru_mix(float z, float hv, float q) {
  const float s = sigmoidf(z);
  return (1.0f - s) * hv + s * tanhf(q);
}

// net = (1 - z) net + z tanh(q), z = sigmoid(zr[:, 0:128]); X[:, 0:128] = round(net); net_r (optional, dense) = round(net)
__global__ void gru_update_kernel(const float* __restrict__ zr, const float* __restrict__ qpre, float* __restrict__ net,
                                  float* __restrict__ X, float* __restrict__ net_r, long npx) {
  DVD_PDL_ENTER();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < npx * 32; i += (long)gridDim.x * blockDim.x) {
    const long p = i / 32;
    const int q = (int)(i % 32);
    const float4 z = reinterpret_cast<const float4*>(zr + p * 256)[q];
    const float4 qq = reinterpret_cast<const float4*>(qpre)[i];
    const float4 hv = reinterpret_cast<const float4*>(net)[i];
    const float4 o = make_float4(gru_mix(z.x, hv.x, qq.x), gru_mix(z.y, hv.y, qq.y), gru_mix(z.z, hv.z, qq.z), gru_mix(z.w, hv.w, qq.w));
    reinterpret_cast<float4*>(net)[i] = o;
    const float4 r = round4(o, 1);
    reinterpret_cast<float4*>(X + p * 384)[q] = r;
    if (net_r) reinterpret_cast<float4*>(net_r)[i] = r;
  }
}

// net (tanh) and inp (relu) halves of the context encoder's output [npx][256] -> net [npx][128], X / XR channels 0..255
__global__ void context_split_kernel(const float* __restrict__ cnet, float* __restrict__ net, float* __restrict__ X,
                                     float* __restrict__ XR, long npx) {
  DVD_PDL_ENTER();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < npx * 64; i += (long)gridDim.x * blockDim.x) {
    const long p = i / 64;
    const int q = (int)(i % 64);
    float4 v = reinterpret_cast<const float4*>(cnet)[i];
    if (q < 32) {
      v = make_float4(tanhf(v.x), tanhf(v.y), tanhf(v.z), tanhf(v.w));
      reinterpret_cast<float4*>(net)[p * 32 + q] = v;
      reinterpret_cast<float4*>(X + p * 384)[q] = round4(v, 1);
    } else {
      v = round4(make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f)), 1);
      reinterpret_cast<float4*>(X + p * 384)[q] = v;
      reinterpret_cast<float4*>(XR + p * 384)[q] = v;
    }
  }
}

// ---- flow head: delta = conv3x3_{256 -> 2}(x) + b; coords1 += delta. One warp per pixel, lanes over channels ------------
__global__ void __launch_bounds__(256) flow_head_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                        const float* __restrict__ bias, float* __restrict__ coords1,
                                                        float* __restrict__ delta, long npx, int h, int wd) {
  __shared__ __align__(16) float ws[2 * 9 * 256];        // [o][tap][c] from w [2][256][3][3]
  for (int i = threadIdx.x; i < 2 * 9 * 256; i += blockDim.x) {
    const int t = i % 9, c = (i / 9) % 256, o = i / (9 * 256);
    ws[(o * 9 + t) * 256 + c] = w[i];
  }
  __syncthreads();
  DVD_PDL_ENTER();
  const int lane = threadIdx.x % 32;
  const long p = (long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  if (p >= npx) return;
  const int px = (int)(p % wd), py = (int)((p / wd) % h);
  float a0 = 0.f, a1 = 0.f;
  for (int t = 0; t < 9; ++t) {
    const int sy = py + t / 3 - 1, sx = px + t % 3 - 1;
    if (sy < 0 || sy >= h || sx < 0 || sx >= wd) continue;
    const float* xp = x + (p + (long)(t / 3 - 1) * wd + (t % 3 - 1)) * 256;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int c = j * 128 + lane * 4;
      const float4 v = *reinterpret_cast<const float4*>(xp + c);
      const float4 w0 = *reinterpret_cast<const float4*>(ws + t * 256 + c);
      const float4 w1 = *reinterpret_cast<const float4*>(ws + (9 + t) * 256 + c);
      a0 = fmaf(v.x, w0.x, fmaf(v.y, w0.y, fmaf(v.z, w0.z, fmaf(v.w, w0.w, a0))));
      a1 = fmaf(v.x, w1.x, fmaf(v.y, w1.y, fmaf(v.z, w1.z, fmaf(v.w, w1.w, a1))));
    }
  }
  a0 = warp_sum(a0);
  a1 = warp_sum(a1);
  if (lane == 0) {
    const float dx = a0 + bias[0], dy = a1 + bias[1];
    if (delta) reinterpret_cast<float2*>(delta)[p] = make_float2(dx, dy);
    float2 c = reinterpret_cast<float2*>(coords1)[p];
    c.x += dx;
    c.y += dy;
    reinterpret_cast<float2*>(coords1)[p] = c;
  }
}

// ---- convex up-sampling: block = one coarse pixel, thread t = (i, j) of its 8 x 8 fine pixels --------------------------------
__global__ void __launch_bounds__(64) upsample_kernel(const float* __restrict__ m0, const float* __restrict__ m1,
                                                      const float* __restrict__ m2, const float* __restrict__ coords1,
                                                      float* __restrict__ flow, int h, int wd, float mask_scale) {
  DVD_PDL_ENTER();
  const long p = blockIdx.x;
  const int px = (int)(p % wd), py = (int)((p / wd) % h);
  const long b = p / ((long)wd * h);
  const int t = threadIdx.x;
  const float* parts[3] = {m0, m1, m2};
  float lg[9], mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    lg[k] = mask_scale * parts[k / 3][p * 192 + (k % 3) * 64 + t];      // channel k * 64 + t of the 576
    mx = fmaxf(mx, lg[k]);
  }
  float den = 0.f, fx = 0.f, fy = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const float e = expf(lg[k] - mx);
    den += e;
    const int sy = py + k / 3 - 1, sx = px + k % 3 - 1;
    if (sy >= 0 && sy < h && sx >= 0 && sx < wd) {
      const float2 c = reinterpret_cast<const float2*>(coords1)[(b * h + sy) * wd + sx];
      fx = fmaf(e, 8.0f * (c.x - (float)sx), fx);
      fy = fmaf(e, 8.0f * (c.y - (float)sy), fy);
    }
  }
  const int oy = py * 8 + t / 8, ox = px * 8 + t % 8;
  reinterpret_cast<float2*>(flow)[(b * (8L * h) + oy) * (8L * wd) + ox] = make_float2(fx / den, fy / den);
}

inline int grid_for(long n, int threads) {
  long g = (n + threads - 1) / threads;
  const long cap = 16L * num_sms();
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

int fill_levels(Levels* L, long rows, int h, int w) {
  long off = 0;
  for (int l = 0; l < kLevels; ++l) {
    if (h < 2 || w < 2) return -1;      // the reference's lookup divides by (w - 1) and (h - 1) of every level
    L->off[l] = off; L->h[l] = h; L->w[l] = w;
    off += rows * h * w;
    h /= 2; w /= 2;
  }
  return 0;
}

}  // namespace
}  // namespace dvd

using namespace dvd;

extern "C" int dvd_raft_stem_fwd(const float* x_nchw, const float* weight, const float* bias, float* y, size_t y_bytes, int N, int H,
                                 int W, void* stream) {
  RAFT_CHECK(x_nchw && weight && bias && y, "dvd_raft_stem_fwd: null pointer");
  RAFT_CHECK(N >= 1 && H >= 2 && W >= 2 && H % 2 == 0 && W % 2 == 0, "dvd_raft_stem_fwd: bad shape N=%d H=%d W=%d (even H, W)", N, H, W);
  RAFT_CHECK(aligned16(y), "dvd_raft_stem_fwd: y must be 16-byte aligned");
  const int OH = H / 2, OW = W / 2;
  const size_t need = (size_t)N * OH * OW * 64 * sizeof(float);
  RAFT_CHECK(y_bytes == need, "dvd_raft_stem_fwd: y holds %zu bytes, expected %zu for [%d,%d,%d,64]", y_bytes, need, N, OH, OW);
  const long total = (long)N * OH * OW;
  DVD_CUDA_CALL(launch(raft_stem_kernel, dim3((unsigned)((total + 127) / 128)), dim3(128), 0, (cudaStream_t)stream, x_nchw, weight, bias, y,
                       N, H, W, OH, OW));
  return 0;
}

extern "C" long dvd_raft_instnorm_scratch_bytes(int N, int C) {
  if (N < 1 || C < 4) return -1;
  return (long)N * kStatChunks * C * 2 * (long)sizeof(double);
}

extern "C" int dvd_raft_instnorm_stats(const float* x, float* stats, void* scratch, size_t scratch_bytes, int N, long P, int C, float eps,
                                       void* stream) {
  RAFT_CHECK(x && stats && scratch, "dvd_raft_instnorm_stats: null pointer");
  RAFT_CHECK(N >= 1 && P >= 1 && C >= 4 && C % 4 == 0 && C <= 256, "dvd_raft_instnorm_stats: bad shape N=%d P=%ld C=%d (4 | C <= 256)", N, P, C);
  RAFT_CHECK(aligned16(x) && aligned16(stats) && aligned16(scratch), "dvd_raft_instnorm_stats: buffers must be 16-byte aligned");
  RAFT_CHECK((long)scratch_bytes >= dvd_raft_instnorm_scratch_bytes(N, C), "dvd_raft_instnorm_stats: scratch holds %zu bytes, needs %ld",
             scratch_bytes, dvd_raft_instnorm_scratch_bytes(N, C));
  const int quads = C / 4, lanes = 256 / quads;
  DVD_CUDA_CALL(launch(instnorm_partial_kernel, dim3(kStatChunks, (unsigned)N), dim3((unsigned)(quads * lanes)),
                       (size_t)lanes * C * 2 * sizeof(double), (cudaStream_t)stream, x, static_cast<double*>(scratch), P, C));
  DVD_CUDA_CALL(launch(instnorm_final_kernel, dim3((unsigned)((N * C + 127) / 128)), dim3(128), 0, (cudaStream_t)stream,
                       static_cast<const double*>(scratch), stats, P, C, N, eps));
  return 0;
}

extern "C" int dvd_raft_norm_act(const float* x, const float* stats, const float* res, float* y, int N, long P, int C, int relu_inner,
                                 int relu_outer, int round_out, void* stream) {
  RAFT_CHECK(x && y, "dvd_raft_norm_act: null pointer");
  RAFT_CHECK(N >= 1 && P >= 1 && C >= 4 && C % 4 == 0, "dvd_raft_norm_act: bad shape N=%d P=%ld C=%d (4 | C)", N, P, C);
  RAFT_CHECK(aligned16(x) && aligned16(y) && (!res || aligned16(res)) && (!stats || aligned16(stats)),
             "dvd_raft_norm_act: buffers must be 16-byte aligned");
  const long total4 = (long)N * P * (C / 4);
  DVD_CUDA_CALL(launch(norm_act_kernel, dim3(grid_for(total4, 256)), dim3(256), 0, (cudaStream_t)stream, x, stats, res, y, P, C, total4,
                       relu_inner, relu_outer, round_out));
  return 0;
}

extern "C" long dvd_raft_pyramid_floats(int B, int h, int w) {
  Levels L;
  if (B < 1 || fill_levels(&L, (long)B * h * w, h, w)) return -1;
  return L.off[kLevels - 1] + (long)B * h * w * L.h[kLevels - 1] * L.w[kLevels - 1];
}

extern "C" int dvd_raft_corr_pyramid(const float* fmap1, const float* fmap2, float* pyramid, size_t pyramid_bytes, int B, int h, int w,
                                     int C, void* stream) {
  RAFT_CHECK(fmap1 && fmap2 && pyramid, "dvd_raft_corr_pyramid: null pointer");
  RAFT_CHECK(B >= 1 && B <= 65535 && C >= 16 && C % 16 == 0, "dvd_raft_corr_pyramid: bad shape B=%d C=%d (16 | C)", B, C);
  Levels L;
  const long P = (long)h * w;
  RAFT_CHECK(fill_levels(&L, (long)B * P, h, w) == 0, "dvd_raft_corr_pyramid: a %d x %d grid leaves a pyramid level under 2 x 2 (needs >= 16 x 16)", h, w);
  RAFT_CHECK(aligned16(fmap1) && aligned16(fmap2) && aligned16(pyramid), "dvd_raft_corr_pyramid: buffers must be 16-byte aligned");
  const size_t need = (size_t)dvd_raft_pyramid_floats(B, h, w) * sizeof(float);
  RAFT_CHECK(pyramid_bytes == need, "dvd_raft_corr_pyramid: pyramid holds %zu bytes, expected %zu", pyramid_bytes, need);
  const unsigned tiles = (unsigned)((P + kCT - 1) / kCT);
  DVD_CUDA_CALL(launch(corr_kernel, dim3(tiles, tiles, (unsigned)B), dim3(256), 0, (cudaStream_t)stream, fmap1, fmap2, pyramid, (int)P, C,
                       1.0f / sqrtf((float)C)));
  for (int l = 1; l < kLevels; ++l) {
    const long n = (long)B * P * L.h[l] * L.w[l];
    DVD_CUDA_CALL(launch(corr_pool_kernel, dim3(grid_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, (const float*)(pyramid + L.off[l - 1]),
                         pyramid + L.off[l], (long)B * P, L.h[l - 1], L.w[l - 1], L.h[l], L.w[l]));
  }
  return 0;
}

extern "C" int dvd_raft_lookup(const float* pyramid, size_t pyramid_bytes, const float* coords1, float* out, size_t out_bytes, int B,
                               int h, int w, int round_out, void* stream) {
  RAFT_CHECK(pyramid && coords1 && out, "dvd_raft_lookup: null pointer");
  Levels L;
  const long P = (long)h * w;
  RAFT_CHECK(B >= 1 && fill_levels(&L, (long)B * P, h, w) == 0, "dvd_raft_lookup: bad shape B=%d h=%d w=%d (needs >= 16 x 16)", B, h, w);
  RAFT_CHECK((reinterpret_cast<uintptr_t>(coords1) & 7u) == 0 && aligned16(out), "dvd_raft_lookup: coords1 8-byte, out 16-byte aligned");
  const size_t need_p = (size_t)dvd_raft_pyramid_floats(B, h, w) * sizeof(float), need_o = (size_t)B * P * kLookupPad * sizeof(float);
  RAFT_CHECK(pyramid_bytes == need_p && out_bytes == need_o, "dvd_raft_lookup: buffers hold %zu / %zu bytes, expected %zu / %zu",
             pyramid_bytes, out_bytes, need_p, need_o);
  RAFT_CHECK((long)B * P < (1L << 31), "dvd_raft_lookup: too many pixels");
  DVD_CUDA_CALL(launch(lookup_kernel, dim3((unsigned)(B * P)), dim3(kLookupPad), 0, (cudaStream_t)stream, pyramid, coords1, out, L, round_out));
  return 0;
}

extern "C" int dvd_raft_convf1(const float* coords1, const float* weight, const float* bias, float* y, int B, int h, int w, int round_out,
                               void* stream) {
  RAFT_CHECK(coords1 && weight && bias && y, "dvd_raft_convf1: null pointer");
  RAFT_CHECK(B >= 1 && B <= 65535 && h >= 1 && h <= 65535 && w >= 1, "dvd_raft_convf1: bad shape B=%d h=%d w=%d", B, h, w);
  RAFT_CHECK((reinterpret_cast<uintptr_t>(coords1) & 7u) == 0, "dvd_raft_convf1: coords1 must be 8-byte aligned");
  DVD_CUDA_CALL(launch(convf1_kernel, dim3((unsigned)((w + kF1Px - 1) / kF1Px), (unsigned)h, (unsigned)B), dim3(128), 0, (cudaStream_t)stream,
                       coords1, weight, bias, y, h, w, round_out));
  return 0;
}

extern "C" int dvd_raft_context_split(const float* cnet, float* net, float* X, float* XR, long npx, void* stream) {
  RAFT_CHECK(cnet && net && X && XR && npx >= 1, "dvd_raft_context_split: null pointer or no pixels");
  RAFT_CHECK(aligned16(cnet) && aligned16(net) && aligned16(X) && aligned16(XR), "dvd_raft_context_split: buffers must be 16-byte aligned");
  DVD_CUDA_CALL(launch(context_split_kernel, dim3(grid_for(npx * 64, 256)), dim3(256), 0, (cudaStream_t)stream, cnet, net, X, XR, npx));
  return 0;
}

extern "C" int dvd_raft_motion_pack(const float* mconv, const float* coords1, float* X, float* XR, int B, int h, int w, void* stream) {
  RAFT_CHECK(mconv && coords1 && X && XR, "dvd_raft_motion_pack: null pointer");
  RAFT_CHECK(B >= 1 && h >= 1 && w >= 1, "dvd_raft_motion_pack: bad shape B=%d h=%d w=%d", B, h, w);
  RAFT_CHECK(aligned16(mconv) && aligned16(X) && aligned16(XR) && (reinterpret_cast<uintptr_t>(coords1) & 7u) == 0,
             "dvd_raft_motion_pack: buffers must be 16-byte aligned (coords1: 8)");
  const long npx = (long)B * h * w;
  DVD_CUDA_CALL(launch(motion_pack_kernel, dim3(grid_for(npx * 32, 256)), dim3(256), 0, (cudaStream_t)stream, mconv, coords1, X, XR, npx, h, w));
  return 0;
}

extern "C" int dvd_raft_gru_rh(const float* zr, const float* net, float* XR, long npx, void* stream) {
  RAFT_CHECK(zr && net && XR && npx >= 1, "dvd_raft_gru_rh: null pointer or no pixels");
  RAFT_CHECK(aligned16(zr) && aligned16(net) && aligned16(XR), "dvd_raft_gru_rh: buffers must be 16-byte aligned");
  DVD_CUDA_CALL(launch(gru_rh_kernel, dim3(grid_for(npx * 32, 256)), dim3(256), 0, (cudaStream_t)stream, zr, net, XR, npx));
  return 0;
}

extern "C" int dvd_raft_gru_update(const float* zr, const float* q, float* net, float* X, float* net_r, long npx, void* stream) {
  RAFT_CHECK(zr && q && net && X && npx >= 1, "dvd_raft_gru_update: null pointer or no pixels");
  RAFT_CHECK(aligned16(zr) && aligned16(q) && aligned16(net) && aligned16(X) && (!net_r || aligned16(net_r)),
             "dvd_raft_gru_update: buffers must be 16-byte aligned");
  DVD_CUDA_CALL(launch(gru_update_kernel, dim3(grid_for(npx * 32, 256)), dim3(256), 0, (cudaStream_t)stream, zr, q, net, X, net_r, npx));
  return 0;
}

extern "C" int dvd_raft_flow_head(const float* x, const float* weight, const float* bias, float* coords1, float* delta, int B, int h, int w,
                                  void* stream) {
  RAFT_CHECK(x && weight && bias && coords1, "dvd_raft_flow_head: null pointer");
  RAFT_CHECK(B >= 1 && h >= 1 && w >= 1, "dvd_raft_flow_head: bad shape B=%d h=%d w=%d", B, h, w);
  RAFT_CHECK(aligned16(x) && (reinterpret_cast<uintptr_t>(coords1) & 7u) == 0 && (reinterpret_cast<uintptr_t>(delta) & 7u) == 0,
             "dvd_raft_flow_head: x 16-byte, coords1 / delta 8-byte aligned");
  const long npx = (long)B * h * w;
  DVD_CUDA_CALL(launch(flow_head_kernel, dim3((unsigned)((npx + 7) / 8)), dim3(256), 0, (cudaStream_t)stream, x, weight, bias, coords1, delta,
                       npx, h, w));
  return 0;
}

extern "C" int dvd_raft_upsample(const float* mask0, const float* mask1, const float* mask2, const float* coords1, float* flow,
                                 size_t flow_bytes, int B, int h, int w, float mask_scale, void* stream) {
  RAFT_CHECK(mask0 && mask1 && mask2 && coords1 && flow, "dvd_raft_upsample: null pointer");
  RAFT_CHECK(B >= 1 && h >= 1 && w >= 1 && (long)B * h * w < (1L << 31), "dvd_raft_upsample: bad shape B=%d h=%d w=%d", B, h, w);
  RAFT_CHECK((reinterpret_cast<uintptr_t>(coords1) & 7u) == 0 && (reinterpret_cast<uintptr_t>(flow) & 7u) == 0,
             "dvd_raft_upsample: coords1 and flow must be 8-byte aligned");
  const size_t need = (size_t)B * h * w * 64 * 2 * sizeof(float);
  RAFT_CHECK(flow_bytes == need, "dvd_raft_upsample: flow holds %zu bytes, expected %zu for [%d,%d,%d,2]", flow_bytes, need, B, 8 * h, 8 * w);
  DVD_CUDA_CALL(launch(upsample_kernel, dim3((unsigned)((long)B * h * w)), dim3(64), 0, (cudaStream_t)stream, mask0, mask1, mask2, coords1, flow,
                       h, w, mask_scale));
  return 0;
}
