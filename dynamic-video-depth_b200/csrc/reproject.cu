// Fused un-project -> scene-flow-advect -> re-project -> bilinear flow-warp -> consistency-loss chain.
//
// Replaces (reference paths relative to the reference tree):
//   unproject_ptcld.forward                 losses/scene_flow_projection.py:48-67      (W3)
//   flow_by_depth.forward                   losses/scene_flow_projection.py:95-153     (W1)
//   scene_flow_projection_slack.forward     losses/scene_flow_projection.py:204-278    (W2)
//   backward_warp + ATen grid_sampler_2d    losses/scene_flow_projection.py:103-112    (bilinear, border, align_corners=True)
//   Model._calc_loss / Model.disp_loss      models/scene_flow_motion_field.py:285-324,140-150 (L1)
//
// The reference runs ~100 ATen launches (16 broadcast 1x3·3x3 batched GEMMs, 3 grid_samples, 3
// nonzero+index_put pairs with host syncs) and materialises ~27 floats/pixel. Here the whole chain is
// one elementwise + gather kernel per direction: it is HBM-bound (no contraction => no tensor cores),
// so the design goals are coalesced 64/128-bit streaming loads, zero intermediate tensors, per-block
// partial sums through warp shuffles, and atomics only for the bilinear scatter of d(depth_2).
//
// Algorithmic HBM bytes per pixel (fp32): fwd 32 (d1 4, d2 4, flow 8, mask 4, sf 12);
// bwd 48 (the same 32 read + g_sf 12 + g_d2 4 written). See DESIGN.md for the full accounting.
#include "common.cuh"
#include <algorithm>
#include <initializer_list>
#include <mutex>
#include <utility>
#include <vector>
#include "tc_common.cuh"

namespace dvd {

// MUFU.RCP: max relative error 2^-23 (1 ulp), no slow path; inputs here are >= 1e-3 or flagged invalid
__device__ __forceinline__ float rcp_fast(float v) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
  return r;
}

__device__ __forceinline__ void mm3(const float* X, const float* Y, float* Z, bool xt) {
  // Z = (xt ? X^T : X) * Y
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      float a = 0.f;
      for (int k = 0; k < 3; ++k) a = fmaf(xt ? X[k * 3 + i] : X[i * 3 + k], Y[k * 3 + j], a);
      Z[i * 3 + j] = a;
    }
}

// M * v  /  M^T * v, every operation rounded on its own (no contraction the compiler could choose differently per kernel)
__device__ __forceinline__ void mv(const float* M, float x, float y, float z, float& ox, float& oy, float& oz) {
  ox = fmaf(M[2], z, fmaf(M[1], y, __fmul_rn(M[0], x)));
  oy = fmaf(M[5], z, fmaf(M[4], y, __fmul_rn(M[3], x)));
  oz = fmaf(M[8], z, fmaf(M[7], y, __fmul_rn(M[6], x)));
}
__device__ __forceinline__ void mtv(const float* M, float x, float y, float z, float& ox, float& oy, float& oz) {
  ox = fmaf(M[6], z, fmaf(M[3], y, __fmul_rn(M[0], x)));
  oy = fmaf(M[7], z, fmaf(M[4], y, __fmul_rn(M[1], x)));
  oz = fmaf(M[8], z, fmaf(M[5], y, __fmul_rn(M[2], x)));
}
// M * (x, y, 1)
__device__ __forceinline__ void ray_of(const float* M, float x, float y, float& rx, float& ry, float& rz) {
  rx = fmaf(M[1], y, M[0] * x) + M[2];
  ry = fmaf(M[4], y, M[3] * x) + M[5];
  rz = fmaf(M[7], y, M[6] * x) + M[8];
}

__device__ __forceinline__ float mask_of(const dvd_loss_cfg& c, float m2, float d1, float wz) {
  return (!c.midas || (d1 < 100.0f && wz < 100.0f)) ? m2 : 0.0f;
}

__device__ __forceinline__ float disp_term(const dvd_loss_cfg& c, float za, float zb) {
  if (c.disp_mode == 0) {
    float a = fmaxf(za, 1e-3f), b = fmaxf(zb, 1e-3f);
    return 100.0f * fabsf(rcp_fast(a) - rcp_fast(b));
  } else if (c.disp_mode == 1) {
    float a = fmaxf(za, 1e-3f), b = fmaxf(zb, 1e-3f);
    return fmaxf(a, b) / fminf(a, b) - 1.0f;
  }
  return fabsf(za - zb);
}

// c * sign(v) (0 at v == 0)
__device__ __forceinline__ float sgn_scale(float v, float c) {
  return v == 0.f ? 0.f : __uint_as_float(__float_as_uint(c) ^ (__float_as_uint(v) & 0x80000000u));   // one LOP3
}

// ---------------------------------------------------------------------------------------------
// vector access helpers (un-project kernels): VEC consecutive pixels along x per thread
template <int VEC>
__device__ __forceinline__ void load_vec(const float* __restrict__ p, float (&v)[VEC]) {
  if (VEC == 4) {
    float4 t = ldg_stream4(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else if (VEC == 2) {
    float2 t = __ldg(reinterpret_cast<const float2*>(p));
    v[0] = t.x; v[1] = t.y;
  } else {
    v[0] = __ldg(p);
  }
}
template <int VEC>
__device__ __forceinline__ void store_vec(float* __restrict__ p, const float (&v)[VEC]) {
  if (VEC == 4) {
    st_stream4(p, make_float4(v[0], v[1], v[2], v[3]));
  } else if (VEC == 2) {
    *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]);
  } else {
    *p = v[0];
  }
}

constexpr int kThreads = 256;

// ---------------------------------------------------------------------------------------------
// un-project forward / adjoint

// Kinv, R_which and t_which of pair b, straight from its [48]-float pose block
__device__ __forceinline__ void load_camera(const float* __restrict__ poses, int b, int which, float* Kinv, float* R,
                                            float* t) {
  const float* p = poses + (size_t)b * DVD_POSE_STRIDE;
  const int i = threadIdx.x;
  if (i < 9) {
    Kinv[i] = __ldg(p + i);
    R[i] = __ldg(p + (which == 1 ? 18 : 27) + i);
  }
  if (i < 3) t[i] = __ldg(p + (which == 1 ? 36 : 39) + i);
  __syncthreads();
}

template <int VEC>
__global__ void __launch_bounds__(kThreads) unproject_fwd_kernel(const float* __restrict__ depth,
                                                                 const float* __restrict__ poses,
                                                                 float* __restrict__ P, int H, int W, int which) {
  DVD_PDL_ENTER();
  __shared__ float Kinv[9], R[9], t[3];
  const int b = blockIdx.y;
  load_camera(poses, b, which, Kinv, R, t);
  const int HW = H * W, items = HW / VEC, Wv = W / VEC;
  // (y, xv) walk of the grid-stride loop without a per-iteration integer division
  const int stride = gridDim.x * blockDim.x, sdy = stride / Wv, sdx = stride - sdy * Wv;
  int it = blockIdx.x * blockDim.x + threadIdx.x;
  int y = it / Wv, xv = it - y * Wv;
  for (; it < items; it += stride, y += sdy, xv += sdx) {
    if (xv >= Wv) { xv -= Wv; ++y; }
    const int x0 = xv * VEC;
    size_t pix = (size_t)y * W + x0;
    float d[VEC], ox[VEC], oy[VEC], oz[VEC];
    load_vec<VEC>(depth + (size_t)b * HW + pix, d);
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
      float rx, ry, rz;
      ray_of(Kinv, (float)(x0 + v), (float)y, rx, ry, rz);
      mv(R, d[v] * rx, d[v] * ry, d[v] * rz, ox[v], oy[v], oz[v]);
      ox[v] += t[0]; oy[v] += t[1]; oz[v] += t[2];
    }
    float* o = P + (size_t)b * 3 * HW + pix;
    store_vec<VEC>(o, ox);
    store_vec<VEC>(o + HW, oy);
    store_vec<VEC>(o + 2 * (size_t)HW, oz);
  }
}

template <int VEC>
__global__ void __launch_bounds__(kThreads) unproject_bwd_kernel(const float* __restrict__ gP,
                                                                 const float* __restrict__ poses,
                                                                 float* __restrict__ gd, int H, int W, int which) {
  DVD_PDL_ENTER();
  __shared__ float Kinv[9], R[9], t[3];
  const int b = blockIdx.y;
  load_camera(poses, b, which, Kinv, R, t);
  const int HW = H * W, items = HW / VEC, Wv = W / VEC;
  // (y, xv) walk of the grid-stride loop without a per-iteration integer division
  const int stride = gridDim.x * blockDim.x, sdy = stride / Wv, sdx = stride - sdy * Wv;
  int it = blockIdx.x * blockDim.x + threadIdx.x;
  int y = it / Wv, xv = it - y * Wv;
  for (; it < items; it += stride, y += sdy, xv += sdx) {
    if (xv >= Wv) { xv -= Wv; ++y; }
    const int x0 = xv * VEC;
    size_t pix = (size_t)y * W + x0;
    float gx[VEC], gy[VEC], gz[VEC], o[VEC];
    const float* g = gP + (size_t)b * 3 * HW + pix;
    load_vec<VEC>(g, gx);
    load_vec<VEC>(g + HW, gy);
    load_vec<VEC>(g + 2 * (size_t)HW, gz);
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
      float rx, ry, rz, wx, wy, wz;
      ray_of(Kinv, (float)(x0 + v), (float)y, rx, ry, rz);
      mv(R, rx, ry, rz, wx, wy, wz);  // dP/dd = R * ray
      o[v] = fmaf(gz[v], wz, fmaf(gy[v], wy, gx[v] * wx));
    }
    store_vec<VEC>(gd + (size_t)b * HW + pix, o);
  }
}

// ---------------------------------------------------------------------------------------------
// Poses of the loss and materialise kernels: derived once per call by pose_prep_kernel and copied into a __constant__ slot
// with a device-to-device cudaMemcpyToSymbolAsync on the caller's stream (no host round trip). The kernels read every
// entry as a broadcast operand straight from the constant bank.
struct __align__(16) PoseC {
  float Kinv[9];   //  0
  float K[9];      //  9
  float R2[9];     // 18
  float nM1[9];    // 27  -(R1 Kinv)                 -(P1 - t1) = d1 * (nM1 c)
  float A[9];      // 36  R2^T R1 Kinv               p12 = d1 * (A c) + cv + R2^T sf
  float cv[3];     // 45  R2^T (t1 - t2)
  float t21[3];    // 48  t2 - t1                    warped_global_p2 - P1 = R2 wpc + t21 + d1 * (nM1 c)
  float t1[3];     // 51
  float t2[3];     // 54
  float pad[7];
};
static_assert(sizeof(PoseC) == 256, "PoseC layout");
constexpr int kPoseSlots = 3;    // rotating slots: calls in flight on different streams do not share a slot
constexpr int kPosePairs = 64;   // pairs per launch (larger batches are processed in chunks)
__constant__ PoseC c_pose[kPoseSlots][kPosePairs];
__device__ PoseC g_pose_stage[kPoseSlots][kPosePairs];

// PoseC of one pair from its raw [48]-float pose block
__device__ __forceinline__ void derive_pose(const float* __restrict__ p, PoseC& o) {
  float Kinv[9], R1[9], R2[9], M1[9], t1[3], t2[3];
  for (int i = 0; i < 9; ++i) {
    Kinv[i] = p[i]; R1[i] = p[18 + i]; R2[i] = p[27 + i];
    o.Kinv[i] = Kinv[i]; o.K[i] = p[9 + i]; o.R2[i] = R2[i];
  }
  for (int i = 0; i < 3; ++i) { t1[i] = p[36 + i]; t2[i] = p[39 + i]; }
  mm3(R1, Kinv, M1, false);
  mm3(R2, M1, o.A, true);
  for (int i = 0; i < 9; ++i) o.nM1[i] = -M1[i];
  const float dx = t1[0] - t2[0], dy = t1[1] - t2[1], dz = t1[2] - t2[2];
  for (int i = 0; i < 3; ++i) {
    o.cv[i] = fmaf(R2[6 + i], dz, fmaf(R2[3 + i], dy, R2[i] * dx));
    o.t21[i] = t2[i] - t1[i];
    o.t1[i] = t1[i];
    o.t2[i] = t2[i];
  }
}

__global__ void pose_prep_kernel(const float* __restrict__ poses, int B, int slot) {
  DVD_PDL_ENTER();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) derive_pose(poses + (size_t)b * DVD_POSE_STRIDE, g_pose_stage[slot][b]);
}

// The kernels with one grid row per pair (generic loss, materialise) derive their pair's PoseC once per CTA into shared
// memory: at one or a few pairs per call, staging constant-bank poses would cost more than the loss kernel itself.
__device__ __forceinline__ const PoseC& block_pose(const float* __restrict__ poses, int b) {
  __shared__ PoseC ps;
  if (threadIdx.x == 0) derive_pose(poses + (size_t)b * DVD_POSE_STRIDE, ps);
  __syncthreads();
  return ps;
}

// ---------------------------------------------------------------------------------------------
// The per-pixel chain, shared by every loss and materialise kernel. Column-vector algebra, c = (x, y, 1)^T.

// streamed inputs of one pixel
struct PixIn {
  float d1, m2, sf[3], fx, fy;
};

// A c and nM1 c, c = (x, y, 1), split into the column-0 term and the part shared by the pixels of row y
struct RowTerms {
  float ra[3];   // A[:,1] y + A[:,2]
  float rn[3];   // nM1[:,1] y + nM1[:,2]
};
__device__ __forceinline__ RowTerms row_terms(const PoseC& ps, float y) {
  RowTerms r;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    r.ra[k] = fmaf(ps.A[3 * k + 1], y, ps.A[3 * k + 2]);
    r.rn[k] = fmaf(ps.nM1[3 * k + 1], y, ps.nM1[3 * k + 2]);
  }
  return r;
}

// forward chain of one pixel
struct PixFwd {
  int i00, sx1, sy1;      // nw tap index; element offsets to the ne / sw taps (0 where clamped by the border)
  float w[4];             // bilinear weights; a tap clamped by the border has weight exactly 0
  float x0f, y0f;         // tap origin (the ne / sw / se taps sit at +1 wherever their weight is non-zero)
  float s1;               // sum_k w_k d2_k = depth_warp_1_2
  float wpc[3], p12[3], i12[3], rz;
  float ex, ey;           // dflow_1_2 - flow_1_2 (zero flow substituted where the projection is rejected)
  bool zok;               // i12.z >= 1e-3 (projection used; otherwise own coordinate, zero gradient)
};

// Bilinear taps follow ATen grid_sampler_2d(bilinear, padding_mode=border, align_corners=True) at the pixel coordinate
// c + flow. The reference normalises to [-1,1] (losses/...:107-110) and ATen un-normalises again; that round trip is the
// identity up to ~1e-7 relative (4e-5 px at W=384), far below the 1e-3 parity bar, so it is skipped.
__device__ __forceinline__ void pixel_forward(const PoseC& ps, const float* __restrict__ d2img, int H, int W, float x,
                                              float y, const RowTerms& rt, const PixIn& in, PixFwd& o) {
  const float hw = (float)(W - 1), hh = (float)(H - 1);
  const float nx = -x;
  const float nqx = fmaf(in.fx, -1.0f, nx);   // -(x + flow_x)
  const float nqy = fmaf(in.fy, -1.0f, -y);   // -(y + flow_y)
  const float ix = fminf(hw, fmaxf(-nqx, 0.0f)), iy = fminf(hh, fmaxf(-nqy, 0.0f));
  o.x0f = floorf(ix);
  o.y0f = floorf(iy);
  const int xi = (int)o.x0f, yi = (int)o.y0f;
  o.i00 = yi * W + xi;
  o.sx1 = xi < W - 1 ? 1 : 0;
  o.sy1 = yi < H - 1 ? W : 0;
  const float* q = d2img + o.i00;   // one 64-bit address per pixel, the other taps at small element offsets from it
  const float dk0 = __ldg(q), dk1 = __ldg(q + o.sx1), dk2 = __ldg(q + o.sy1), dk3 = __ldg(q + o.sy1 + o.sx1);
  // ---- arithmetic that does not depend on the gathered taps first: it runs while the gather is in flight ----
  // p12 = d1 (A c) + cv + R2^T sf
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float ac = fmaf(-ps.A[3 * k], nx, rt.ra[k]);
    float t = fmaf(in.d1, ac, ps.cv[k]);
    t = fmaf(ps.R2[k], in.sf[0], t);
    t = fmaf(ps.R2[3 + k], in.sf[1], t);
    o.p12[k] = fmaf(ps.R2[6 + k], in.sf[2], t);
  }
  mv(ps.K, o.p12[0], o.p12[1], o.p12[2], o.i12[0], o.i12[1], o.i12[2]);
  o.rz = rcp_fast(__fadd_rn(o.i12[2], 1e-8f));
  o.zok = !(o.i12[2] < 1e-3f);
  // dflow - flow = i12.xy * rz - (c.xy + flow)
  o.ex = o.zok ? fmaf(o.i12[0], o.rz, nqx) : -in.fx;
  o.ey = o.zok ? fmaf(o.i12[1], o.rz, nqy) : -in.fy;
  // clamped coordinate == W-1 (H-1) implies a zero fractional part, so the clamped taps need no explicit masking
  const float wx1 = fmaf(o.x0f, -1.0f, ix), wy1 = fmaf(o.y0f, -1.0f, iy);
  const float wx0 = fmaf(wx1, -1.0f, 1.0f), wy0 = fmaf(wy1, -1.0f, 1.0f);
  o.w[0] = __fmul_rn(wx0, wy0); o.w[1] = __fmul_rn(wx1, wy0); o.w[2] = __fmul_rn(wx0, wy1); o.w[3] = __fmul_rn(wx1, wy1);
  // ---- gathered taps ----
  // wpc = sum_k w_k d2_k Kinv (u_k, v_k, 1) = Kinv (su, sv, s1), u_k = x0f (+1), v_k = y0f (+1)
  const float wd0 = __fmul_rn(o.w[0], dk0), wd1 = __fmul_rn(o.w[1], dk1);
  const float wd2 = __fmul_rn(o.w[2], dk2), wd3 = __fmul_rn(o.w[3], dk3);
  const float eb = __fadd_rn(wd1, wd3), sb = __fadd_rn(wd2, wd3);
  o.s1 = __fadd_rn(__fadd_rn(wd0, wd1), sb);
  const float su = fmaf(o.x0f, o.s1, eb), sv = fmaf(o.y0f, o.s1, sb);
  mv(ps.Kinv, su, sv, o.s1, o.wpc[0], o.wpc[1], o.wpc[2]);
}

// residual of the sf term: warped_global_p2 - P1 - sf = R2 wpc + t21 + d1 (nM1 c) - sf
__device__ __forceinline__ void sf_residual(const PoseC& ps, float x, const RowTerms& rt, const PixIn& in,
                                            const PixFwd& o, float (&e)[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float nr = fmaf(-ps.nM1[3 * k], -x, rt.rn[k]);   // -(M1 c)_k
    const float t = fmaf(in.sf[k], -1.0f, fmaf(in.d1, nr, ps.t21[k]));
    e[k] = fmaf(ps.R2[3 * k + 2], o.wpc[2], fmaf(ps.R2[3 * k + 1], o.wpc[1], fmaf(ps.R2[3 * k], o.wpc[0], t)));
  }
}

// g_d2_k = w_k (hu u_k + hv v_k + h1), (u_k, v_k) = (x0f, y0f) (+1): the scatter of Kinv^T g_wpc = (hu, hv, h1)
__device__ __forceinline__ void tap_grads(const PixFwd& o, float hu, float hv, float h1, float (&g)[4]) {
  const float base = fmaf(hu, o.x0f, fmaf(hv, o.y0f, h1));
  const float bx = __fadd_rn(base, hu);
  g[0] = __fmul_rn(o.w[0], base);
  g[1] = __fmul_rn(o.w[1], bx);
  g[2] = __fmul_rn(o.w[2], __fadd_rn(base, hv));
  g[3] = __fmul_rn(o.w[3], __fadd_rn(bx, hv));
}

struct LossSums {
  float flow = 0.f, disp = 0.f, sf = 0.f, m = 0.f;
};

// Adds the masked loss terms of the N pixels (x0 + j, y) to acc[j]. Each term is formed for all N pixels before the next,
// so a loss-mode branch is taken once per term rather than once per pixel (with per-pixel branches the compiler spills
// the staged forward at its 72-register budget).
template <int N>
__device__ __forceinline__ void add_losses(const PoseC& ps, const dvd_loss_cfg& cfg, const float* __restrict__ d2img,
                                           int H, int W, int x0, float y, const PixIn (&in)[N], LossSums (&acc)[N]) {
  const RowTerms rt = row_terms(ps, y);
  PixFwd o[N];
  float e[N][3], m[N], fl[N], dl[N], sl[N];
#pragma unroll
  for (int j = 0; j < N; ++j) {
    pixel_forward(ps, d2img, H, W, (float)(x0 + j), y, rt, in[j], o[j]);
    sf_residual(ps, (float)(x0 + j), rt, in[j], o[j], e[j]);
  }
#pragma unroll
  for (int j = 0; j < N; ++j) m[j] = mask_of(cfg, in[j].m2, in[j].d1, o[j].wpc[2]);
  if (cfg.warm) {
#pragma unroll
    for (int j = 0; j < N; ++j) fl[j] = fmaf(o[j].ex, o[j].ex, __fmul_rn(o[j].ey, o[j].ey));
  } else {
#pragma unroll
    for (int j = 0; j < N; ++j) fl[j] = fabsf(o[j].ex) + fabsf(o[j].ey);
  }
#pragma unroll
  for (int j = 0; j < N; ++j) dl[j] = disp_term(cfg, o[j].p12[2], o[j].wpc[2]);
#pragma unroll
  for (int j = 0; j < N; ++j) sl[j] = fabsf(e[j][0]) + fabsf(e[j][1]) + fabsf(e[j][2]);
#pragma unroll
  for (int j = 0; j < N; ++j) {
    acc[j].flow = fmaf(m[j], fl[j], acc[j].flow);
    acc[j].disp = fmaf(m[j], dl[j], acc[j].disp);
    acc[j].sf = fmaf(m[j], sl[j], acc[j].sf);
    acc[j].m = __fadd_rn(acc[j].m, m[j]);
  }
}

// backward of one pixel: g_(P1 + sf) -> gv, Kinv^T g_warped_p2_camera_2 -> h (tap_grads turns h into the gradients of
// the four depth_2 taps in o)
__device__ __forceinline__ void pixel_backward(const PoseC& ps, const dvd_loss_cfg& cfg, const float* __restrict__ d2img,
                                               int H, int W, float x, float y, const RowTerms& rt, const PixIn& in,
                                               float cf, float cd, PixFwd& o, float (&gv)[3], float (&h)[3]) {
  pixel_forward(ps, d2img, H, W, x, y, rt, in, o);
  const float m = mask_of(cfg, in.m2, in.d1, o.wpc[2]);
  // --- flow term -> g_i12 (zero where the projection was rejected)
  const float mcf = o.zok ? m * cf : 0.f;
  float gux, guy;
  if (cfg.warm) {
    const float t2 = __fadd_rn(mcf, mcf);
    gux = __fmul_rn(t2, o.ex); guy = __fmul_rn(t2, o.ey);
  } else {
    gux = sgn_scale(o.ex, mcf); guy = sgn_scale(o.ey, mcf);
  }
  const float gi0 = __fmul_rn(gux, o.rz), gi1 = __fmul_rn(guy, o.rz);
  const float tt = fmaf(gux, o.i12[0], __fmul_rn(guy, o.i12[1]));
  const float gi2 = __fmul_rn(__fmul_rn(tt, o.rz), __fmul_rn(o.rz, -1.0f));
  float gp0, gp1, gp2;   // g_p12 = K^T g_i12
  mtv(ps.K, gi0, gi1, gi2, gp0, gp1, gp2);
  float hu, hv, h1;      // Kinv^T g_warped_p2_camera_2
  float ge[3] = {0.f, 0.f, 0.f};
  const float mc = __fmul_rn(m, cd);
  if (cfg.second_is_disp) {
    const float za = o.p12[2], zb = o.wpc[2];
    float gwc2;
    if (cfg.disp_mode == 0) {
      const float ra = rcp_fast(fmaxf(za, 1e-3f)), rb = rcp_fast(fmaxf(zb, 1e-3f));
      const float s = sgn_scale(fmaf(rb, -1.0f, ra), __fmul_rn(mc, 100.0f));
      const float sa = za >= 1e-3f ? s : 0.f, sb = zb >= 1e-3f ? s : 0.f;
      gp2 = fmaf(__fmul_rn(sa, ra), __fmul_rn(ra, -1.0f), gp2);
      gwc2 = __fmul_rn(__fmul_rn(sb, rb), rb);
    } else if (cfg.disp_mode == 1) {
      // max(a,b)/min(a,b) - 1
      const float a = fmaxf(za, 1e-3f), bb = fmaxf(zb, 1e-3f);
      const float ra = rcp_fast(a), rb = rcp_fast(bb);
      float ga, gb;
      if (a >= bb) { ga = rb; gb = -a * rb * rb; }
      else         { ga = -bb * ra * ra; gb = ra; }
      gp2 = __fadd_rn(gp2, za >= 1e-3f ? ga * mc : 0.f);
      gwc2 = zb >= 1e-3f ? gb * mc : 0.f;
    } else {
      const float s = sgn_scale(fmaf(zb, -1.0f, za), mc);
      gp2 = __fadd_rn(gp2, s);
      gwc2 = __fmul_rn(s, -1.0f);
    }
    hu = __fmul_rn(ps.Kinv[6], gwc2); hv = __fmul_rn(ps.Kinv[7], gwc2); h1 = __fmul_rn(ps.Kinv[8], gwc2);
  } else {
    float e[3];
    sf_residual(ps, x, rt, in, o, e);
    ge[0] = sgn_scale(e[0], mc); ge[1] = sgn_scale(e[1], mc); ge[2] = sgn_scale(e[2], mc);
    // warped_global_p2 = R2 wpc + t2  =>  g_wpc = R2^T g_e
    float a0, a1, a2;
    mtv(ps.R2, ge[0], ge[1], ge[2], a0, a1, a2);
    mtv(ps.Kinv, a0, a1, a2, hu, hv, h1);
  }
  // g_(P1 + sf) = R2 g_p12 ; the sf term adds -g_e to both P1 and sf
  mv(ps.R2, gp0, gp1, gp2, gv[0], gv[1], gv[2]);
#pragma unroll
  for (int k = 0; k < 3; ++k) gv[k] = fmaf(ge[k], -1.0f, gv[k]);
  h[0] = hu; h[1] = hv; h[2] = h1;
}

// ---------------------------------------------------------------------------------------------
// scatter-add of the four tap gradients of one pixel into g_depth_2 (q = &g_depth_2[i00])
__device__ __forceinline__ void scatter4_atomic(float* q, int sx1, int sy1, const float (&g)[4]) {
  if (g[0] != 0.f) atomicAdd(q, g[0]);
  if (g[1] != 0.f) atomicAdd(q + sx1, g[1]);
  if (g[2] != 0.f) atomicAdd(q + sy1, g[2]);
  if (g[3] != 0.f) atomicAdd(q + sy1 + sx1, g[3]);
}
__device__ __forceinline__ void red_global_v2(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void red_global_v4(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
// Vector form: needs W % 4 == 0 and a 16-byte aligned g_depth_2 image. Whenever the nw tap sits on an even column the
// (nw, ne) and (sw, se) taps are two 8-byte aligned pairs: one vector reduction each.
__device__ __forceinline__ void scatter4_vec(float* q, int i00, int sx1, int sy1, const float (&g)[4]) {
  if (((i00 & 1) == 0) && sx1 == 1) {
    if (g[0] != 0.f || g[1] != 0.f) red_global_v2(q, g[0], g[1]);
    if (g[2] != 0.f || g[3] != 0.f) {
      if (sy1 != 0) red_global_v2(q + sy1, g[2], g[3]);
      else red_global_v2(q, g[2], g[3]);     // clamped bottom row: both weights are exactly 0 here, kept for form
    }
  } else if (((i00 & 3) == 1) && sx1 == 1) {
    // odd column whose pair still lies inside one 16-byte quad: one 4-wide reduction {0, g, g, 0} per row instead of two
    // scalar ones (the LSU's reduction rate is per active lane, not per byte: DESIGN.md 8)
    if (g[0] != 0.f || g[1] != 0.f) red_global_v4(q - 1, 0.f, g[0], g[1], 0.f);
    if (g[2] != 0.f || g[3] != 0.f) red_global_v4(q - 1 + sy1, 0.f, g[2], g[3], 0.f);
  } else {
    scatter4_atomic(q, sx1, sy1, g);
  }
}

// per-block partial sums -> out[0..3]; every thread of a kThreads-thread group must call it (named barrier 1, so a
// producer warp that has already exited does not take part)
__device__ __forceinline__ void write_block_sums(const LossSums& a, float* __restrict__ out) {
  __shared__ float red[kThreads / 32][4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float s_flow = warp_sum(a.flow), s_disp = warp_sum(a.disp), s_sf = warp_sum(a.sf), s_m = warp_sum(a.m);
  if (lane == 0) { red[warp][0] = s_flow; red[warp][1] = s_disp; red[warp][2] = s_sf; red[warp][3] = s_m; }
  asm volatile("bar.sync 1, %0;" ::"n"(kThreads) : "memory");
  if (threadIdx.x < 4) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) s += red[w][threadIdx.x];
    out[threadIdx.x] = s;
  }
}

// ---------------------------------------------------------------------------------------------
// Generic loss kernels: any W and alignment, scalar loads, blockIdx.y is the pair. The forward walks N x-adjacent pixels
// per thread and grid-stride step (N = 2 when W is even, so a pair never straddles a row, as in the staged consumer;
// N = 1 otherwise). The scatter-add backward runs one pixel per thread: more warps in flight hide the atomic latency.

__device__ __forceinline__ PixIn load_pixel(const float* __restrict__ depth_1, const float* __restrict__ mask_2,
                                            const float* __restrict__ sf, const float* __restrict__ flow, size_t b,
                                            int HW, int p) {
  const size_t i = b * HW + p;
  PixIn in;
  in.d1 = __ldg(depth_1 + i);
  in.m2 = mask_2 ? __ldg(mask_2 + i) : 0.f;
  const float* s = sf ? sf + b * 3 * HW + p : nullptr;
  for (int k = 0; k < 3; ++k) in.sf[k] = s ? __ldg(s + (size_t)k * HW) : 0.f;
  in.fx = __ldg(flow + 2 * i);
  in.fy = __ldg(flow + 2 * i + 1);
  return in;
}

// the per-pixel-slot accumulators of a thread, summed in slot order
template <int N>
__device__ __forceinline__ LossSums sum_slots(const LossSums (&acc)[N]) {
  LossSums a = acc[0];
#pragma unroll
  for (int j = 1; j < N; ++j) {
    a.flow += acc[j].flow;
    a.disp += acc[j].disp;
    a.sf += acc[j].sf;
    a.m += acc[j].m;
  }
  return a;
}

template <int N>
__global__ void __launch_bounds__(kThreads, 2) reproject_loss_fwd_kernel(
    const float* __restrict__ depth_1, const float* __restrict__ depth_2, const float* __restrict__ flow,
    const float* __restrict__ mask_2, const float* __restrict__ sf, dvd_loss_cfg cfg, float* __restrict__ partials,
    int H, int W, const float* __restrict__ poses) {
  DVD_PDL_ENTER();
  const int HW = H * W;
  const size_t b = blockIdx.y;
  const PoseC& ps = block_pose(poses, blockIdx.y);
  const float* d2img = depth_2 + b * HW;
  LossSums acc[N];   // one per pixel slot
  for (int p = (blockIdx.x * blockDim.x + threadIdx.x) * N; p < HW; p += gridDim.x * blockDim.x * N) {
    const int y = p / W;
    PixIn in[N];
#pragma unroll
    for (int j = 0; j < N; ++j) in[j] = load_pixel(depth_1, mask_2, sf, flow, b, HW, p + j);
    add_losses<N>(ps, cfg, d2img, H, W, p - y * W, (float)y, in, acc);
  }
  write_block_sums(sum_slots(acc), partials + (b * gridDim.x + blockIdx.x) * 4);
}

__global__ void __launch_bounds__(kThreads) reproject_loss_bwd_kernel(
    const float* __restrict__ depth_1, const float* __restrict__ depth_2, const float* __restrict__ flow,
    const float* __restrict__ mask_2, const float* __restrict__ sf, dvd_loss_cfg cfg, const float* __restrict__ scalars,
    float gscale, const float* __restrict__ gscale_dev, float* __restrict__ g_sf, float* __restrict__ g_d2, int H, int W,
    const float* __restrict__ poses) {
  DVD_PDL_ENTER();
  const int HW = H * W;
  const size_t b = blockIdx.y;
  const PoseC& ps = block_pose(poses, blockIdx.y);
  const float gs = gscale * (gscale_dev ? __ldg(gscale_dev) : 1.0f);
  const float cf = __ldg(scalars + DVD_S_CF) * gs;
  const float cd = __ldg(scalars + DVD_S_CD) * gs;
  const float* d2img = depth_2 + b * HW;
  float* gd2img = g_d2 ? g_d2 + b * HW : nullptr;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
    const int y = p / W;
    PixFwd o;
    float gv[3], h[3];
    pixel_backward(ps, cfg, d2img, H, W, (float)(p - y * W), (float)y, row_terms(ps, (float)y),
                   load_pixel(depth_1, mask_2, sf, flow, b, HW, p), cf, cd, o, gv, h);
    float* gsp = g_sf + b * 3 * HW + p;
    gsp[0] = gv[0]; gsp[HW] = gv[1]; gsp[2 * (size_t)HW] = gv[2];
    if (gd2img) {
      float gd[4];
      tap_grads(o, h[0], h[1], h[2], gd);
      scatter4_atomic(gd2img + o.i00, o.sx1, o.sy1, gd);
    }
  }
}

// deterministic final reduction (fixed order, double accumulation) + loss assembly
__global__ void __launch_bounds__(256) reproject_finalize_kernel(const float* __restrict__ partials, int n_quads,
                                                                 dvd_loss_cfg cfg, float* __restrict__ scalars) {
  DVD_PDL_ENTER();
  __shared__ double red[8][4];
  double acc[4] = {0, 0, 0, 0};
  for (int i = threadIdx.x; i < n_quads; i += blockDim.x) {
    float4 q = *reinterpret_cast<const float4*>(partials + (size_t)i * 4);
    acc[0] += q.x; acc[1] += q.y; acc[2] += q.z; acc[3] += q.w;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) for (int k = 0; k < 4; ++k) red[wid][k] = acc[k];
  __syncthreads();
  if (threadIdx.x == 0) {
    double t[4] = {0, 0, 0, 0};
    for (int w = 0; w < 8; ++w) for (int k = 0; k < 4; ++k) t[k] += red[w][k];
    float n = (float)t[3] + 1e-8f;  // torch.sum(occ_mask) + 1e-8 (smf.py:297-306)
    float fl = (float)t[0] / n, dl = (float)t[1] / n, sl = (float)t[2] / n;
    float second = cfg.second_is_disp ? dl : sl;
    scalars[DVD_S_FLOW] = fl;
    scalars[DVD_S_DISP] = dl;
    scalars[DVD_S_SF] = sl;
    scalars[DVD_S_LOSS] = cfg.flow_mul * fl + cfg.disp_mul * second;
    scalars[DVD_S_MASKSUM] = (float)t[3];
    scalars[DVD_S_CF] = cfg.flow_mul / n;
    scalars[DVD_S_CD] = cfg.disp_mul / n;
    scalars[DVD_S_RSVD] = 0.f;
  }
}

// ---------------------------------------------------------------------------------------------
// Staged loss kernels (W % 4 == 0, 16-byte aligned streamed inputs): the five streamed inputs (28 of the 32 bytes per
// pixel) travel global -> shared memory as 1-D bulk async copies issued by a producer warp into a ring of kStages tiles,
// completion on mbarriers; the kThreads consumer threads only see shared-memory latency for them, and the bytes in flight
// per SM (CTAs x kStages x 14 KB) no longer depend on occupancy or on how the compiler schedules the loads. Each consumer
// thread owns one x-adjacent pixel pair per tile. Only the bilinear gather of depth_2 is a global load, and g_depth_2 is
// accumulated with global reductions; staging either through shared memory is a possible variant that has not been
// measured on sm_90.
constexpr int kStages = 4;
constexpr int kTile = 2 * kThreads;                               // pixels per stage
constexpr int kTileFloats = 7 * kTile;                            // d1, mask, sf.x, sf.y, sf.z, flow (2 floats per pixel)
constexpr int kStagedSmem = kStages * kTileFloats * (int)sizeof(float);
constexpr int kFwdCtasPerSm = 3, kBwdCtasPerSm = 2;

// The producer warp streams tiles and returns false; each consumer thread calls consume(bl, p, in[2]) for its pixel pair
// (p, p + 1) of pair bl of the chunk in every tile, then returns true. A chunk's pairs are split into tiles_per_pair tiles
// each; CTAs walk the tiles with a stride of gridDim.x.
template <class Consume>
__device__ __forceinline__ bool staged_pairs(const float* __restrict__ depth_1, const float* __restrict__ mask_2,
                                             const float* __restrict__ sf, const float* __restrict__ flow, int HW, int b0,
                                             int nb, int tiles_per_pair, Consume&& consume) {
  using namespace tc;
  extern __shared__ __align__(128) float stage_mem[];
  __shared__ uint64_t full[kStages], empty[kStages];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = nb * tiles_per_pair;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kThreads / 32); }
    fence_mbar_init();
  }
  __syncthreads();
  if (warp == kThreads / 32) {
    if (lane == 0) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
        const uint32_t s = it % kStages, ph = (it / kStages) & 1u;
        mbar_wait(&empty[s], ph ^ 1u);
        const int bl = tile / tiles_per_pair, p0 = (tile - bl * tiles_per_pair) * kTile;
        const size_t b = (size_t)(b0 + bl);
        float* dst = stage_mem + (size_t)s * kTileFloats;
        const uint32_t n4 = (uint32_t)min(kTile, HW - p0) * 4u;
        mbar_arrive_expect_tx(&full[s], n4 * 7u);
        bulk_g2s(dst, depth_1 + b * HW + p0, n4, &full[s]);
        bulk_g2s(dst + kTile, mask_2 + b * HW + p0, n4, &full[s]);
        bulk_g2s(dst + 2 * kTile, sf + (b * 3 + 0) * HW + p0, n4, &full[s]);
        bulk_g2s(dst + 3 * kTile, sf + (b * 3 + 1) * HW + p0, n4, &full[s]);
        bulk_g2s(dst + 4 * kTile, sf + (b * 3 + 2) * HW + p0, n4, &full[s]);
        bulk_g2s(dst + 5 * kTile, flow + (b * HW + p0) * 2, n4 * 2u, &full[s]);
      }
    }
    return false;
  }
  const int tv = threadIdx.x * 2;
  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
    const uint32_t s = it % kStages, ph = (it / kStages) & 1u;
    mbar_wait(&full[s], ph);
    const float* src = stage_mem + (size_t)s * kTileFloats + tv;
    const float2 d1 = *reinterpret_cast<const float2*>(src), m2 = *reinterpret_cast<const float2*>(src + kTile);
    const float2 sx = *reinterpret_cast<const float2*>(src + 2 * kTile);
    const float2 sy = *reinterpret_cast<const float2*>(src + 3 * kTile);
    const float2 sz = *reinterpret_cast<const float2*>(src + 4 * kTile);
    const float4 f = *reinterpret_cast<const float4*>(src + 5 * kTile + tv);
    // The producer's next bulk copy into this stage is an async-proxy write: without a proxy fence the generic-proxy
    // loads above are not ordered before it, and a few lanes read the next tile's bytes (seen as wrong g_sf on H100).
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);     // values are in registers: hand the stage back
    const int bl = tile / tiles_per_pair, p = (tile - bl * tiles_per_pair) * kTile + tv;
    if (p >= HW) continue;
    const PixIn in[2] = {{d1.x, m2.x, {sx.x, sy.x, sz.x}, f.x, f.y}, {d1.y, m2.y, {sx.y, sy.y, sz.y}, f.z, f.w}};
    consume(bl, p, in);
  }
  return true;
}

__global__ void __launch_bounds__(kThreads + 32, kFwdCtasPerSm) reproject_loss_fwd_staged_kernel(
    const float* __restrict__ depth_1, const float* __restrict__ depth_2, const float* __restrict__ flow,
    const float* __restrict__ mask_2, const float* __restrict__ sf, dvd_loss_cfg cfg, float* __restrict__ partials,
    int H, int W, int slot, int b0, int nb, int tiles_per_pair) {
  DVD_PDL_ENTER();
  const int HW = H * W;
  LossSums acc[2];   // one per pixel slot of the pair
  if (!staged_pairs(depth_1, mask_2, sf, flow, HW, b0, nb, tiles_per_pair, [&](int bl, int p, const PixIn (&in)[2]) {
        const PoseC& ps = c_pose[slot][bl];
        const float* d2img = depth_2 + (size_t)(b0 + bl) * HW;
        const int y = p / W;
        add_losses<2>(ps, cfg, d2img, H, W, p - y * W, (float)y, in, acc);
      }))
    return;
  write_block_sums(sum_slots(acc), partials + (size_t)blockIdx.x * 4);
}

__global__ void __launch_bounds__(kThreads + 32, kBwdCtasPerSm) reproject_loss_bwd_staged_kernel(
    const float* __restrict__ depth_1, const float* __restrict__ depth_2, const float* __restrict__ flow,
    const float* __restrict__ mask_2, const float* __restrict__ sf, dvd_loss_cfg cfg, const float* __restrict__ scalars,
    float gscale, const float* __restrict__ gscale_dev, float* __restrict__ g_sf, float* __restrict__ g_d2, int H, int W,
    int slot, int b0, int nb, int tiles_per_pair) {
  DVD_PDL_ENTER();
  const int HW = H * W;
  const float gs = gscale * (gscale_dev ? __ldg(gscale_dev) : 1.0f);
  const float cf = __ldg(scalars + DVD_S_CF) * gs;
  const float cd = __ldg(scalars + DVD_S_CD) * gs;
  staged_pairs(depth_1, mask_2, sf, flow, HW, b0, nb, tiles_per_pair, [&](int bl, int p, const PixIn (&in)[2]) {
    const PoseC& ps = c_pose[slot][bl];
    const size_t b = (size_t)(b0 + bl);
    const float* d2img = depth_2 + b * HW;
    float* gd2img = g_d2 ? g_d2 + b * HW : nullptr;
    const int y = p / W, x0 = p - y * W;
    const RowTerms rt = row_terms(ps, (float)y);
    float gv[2][3];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      PixFwd o;
      float h[3];
      pixel_backward(ps, cfg, d2img, H, W, (float)(x0 + j), (float)y, rt, in[j], cf, cd, o, gv[j], h);
      if (gd2img) {
        float gd[4];
        tap_grads(o, h[0], h[1], h[2], gd);
        scatter4_vec(gd2img + o.i00, o.i00, o.sx1, o.sy1, gd);
      }
    }
    float* gsp = g_sf + b * 3 * HW + p;
#pragma unroll
    for (int k = 0; k < 3; ++k) *reinterpret_cast<float2*>(gsp + (size_t)k * HW) = make_float2(gv[0][k], gv[1][k]);
  });
}

// ---------------------------------------------------------------------------------------------
// materialise every per-pixel tensor of the two reference modules (not on the training fast path)
__device__ __forceinline__ void st3(float* p, size_t o3, int HW, float a, float b, float c) {
  if (p) { p[o3] = a; p[o3 + HW] = b; p[o3 + 2 * (size_t)HW] = c; }
}
__device__ __forceinline__ void ld3(const float* p, size_t o3, int HW, float& a, float& b, float& c) {
  if (p) { a = p[o3]; b = p[o3 + HW]; c = p[o3 + 2 * (size_t)HW]; } else { a = b = c = 0.f; }
}

__global__ void __launch_bounds__(kThreads) reproject_materialize_kernel(
    const float* __restrict__ depth_1, const float* __restrict__ depth_2, const float* __restrict__ flow,
    const float* __restrict__ sf, float* __restrict__ global_p1, float* __restrict__ sf_by_depth,
    float* __restrict__ warped_global_p2, float* __restrict__ warped_p2_camera_2, float* __restrict__ p1_camera_2,
    float* __restrict__ dflow, float* __restrict__ staticflow, float* __restrict__ depth_image,
    float* __restrict__ depth_warp, int H, int W, const float* __restrict__ poses) {
  DVD_PDL_ENTER();
  const int HW = H * W;
  const size_t b = blockIdx.y;
  const PoseC& ps = block_pose(poses, blockIdx.y);
  const float* d2img = depth_2 + b * HW;
  for (int pix = blockIdx.x * blockDim.x + threadIdx.x; pix < HW; pix += gridDim.x * blockDim.x) {
    const int y = pix / W;
    const float x = (float)(pix - y * W), yf = (float)y;
    const PixIn in = load_pixel(depth_1, nullptr, sf, flow, b, HW, pix);
    const RowTerms rt = row_terms(ps, yf);
    PixFwd o;
    pixel_forward(ps, d2img, H, W, x, yf, rt, in, o);
    // P1 = d1 (M1 c) + t1 ; warped_global_p2 = R2 wpc + t2 (the four in-range bilinear weights sum to 1)
    float n[3], P1[3], wP2[3];
    ray_of(ps.nM1, x, yf, n[0], n[1], n[2]);
    mv(ps.R2, o.wpc[0], o.wpc[1], o.wpc[2], wP2[0], wP2[1], wP2[2]);
    for (int k = 0; k < 3; ++k) {
      P1[k] = fmaf(-in.d1, n[k], ps.t1[k]);
      wP2[k] += ps.t2[k];
    }
    const size_t o3 = b * 3 * HW + pix, o2 = b * 2 * HW + pix, o1 = b * HW + pix;
    st3(global_p1, o3, HW, P1[0], P1[1], P1[2]);
    st3(sf_by_depth, o3, HW, wP2[0] - P1[0], wP2[1] - P1[1], wP2[2] - P1[2]);
    st3(warped_global_p2, o3, HW, wP2[0], wP2[1], wP2[2]);
    st3(warped_p2_camera_2, o3, HW, o.wpc[0], o.wpc[1], o.wpc[2]);
    st3(p1_camera_2, o3, HW, o.p12[0], o.p12[1], o.p12[2]);
    if (dflow) {
      dflow[o2] = o.zok ? fmaf(o.i12[0], o.rz, -x) : 0.f;
      dflow[o2 + HW] = o.zok ? fmaf(o.i12[1], o.rz, -yf) : 0.f;
    }
    if (depth_image) depth_image[o1] = o.i12[2];
    if (depth_warp) depth_warp[o1] = o.s1;
    if (staticflow) {
      PixIn in0 = in;
      in0.sf[0] = in0.sf[1] = in0.sf[2] = 0.f;
      PixFwd os;
      pixel_forward(ps, d2img, H, W, x, yf, rt, in0, os);
      staticflow[o2] = os.zok ? fmaf(os.i12[0], os.rz, -x) : 0.f;
      staticflow[o2 + HW] = os.zok ? fmaf(os.i12[1], os.rz, -yf) : 0.f;
    }
  }
}

// Adjoint of reproject_materialize_kernel for ARBITRARY cotangents on its nine outputs (operator-level drop-in: the mirrors
// of flow_by_depth / scene_flow_projection_slack stay differentiable for user-defined losses).
struct MatGrads {
  const float* global_p1; const float* sf_by_depth; const float* warped_global_p2; const float* warped_p2_camera_2;
  const float* p1_camera_2; const float* dflow; const float* staticflow; const float* depth_image; const float* depth_warp;
};
__global__ void __launch_bounds__(kThreads) reproject_materialize_bwd_kernel(
    const float* __restrict__ depth_1, const float* __restrict__ depth_2, const float* __restrict__ flow,
    const float* __restrict__ sf, MatGrads G, float* __restrict__ g_d1, float* __restrict__ g_d2,
    float* __restrict__ g_sf, int H, int W, const float* __restrict__ poses) {
  DVD_PDL_ENTER();
  const int HW = H * W;
  const size_t b = blockIdx.y;
  const PoseC& ps = block_pose(poses, blockIdx.y);
  const float* d2img = depth_2 + b * HW;
  for (int pix = blockIdx.x * blockDim.x + threadIdx.x; pix < HW; pix += gridDim.x * blockDim.x) {
    const int y = pix / W;
    const float x = (float)(pix - y * W), yf = (float)y;
    const size_t o3 = b * 3 * HW + pix, o2 = b * 2 * HW + pix, o1 = b * HW + pix;
    const PixIn in = load_pixel(depth_1, nullptr, sf, flow, b, HW, pix);
    const RowTerms rt = row_terms(ps, yf);
    PixFwd o;
    pixel_forward(ps, d2img, H, W, x, yf, rt, in, o);
    float a0, a1, a2, b0v, b1v, b2v;
    // P1: + global_p1, - sf_by_depth ;  wP2: + sf_by_depth, + warped_global_p2
    float gP0, gP1, gP2, gW0, gW1, gW2;
    ld3(G.global_p1, o3, HW, gP0, gP1, gP2);
    ld3(G.sf_by_depth, o3, HW, a0, a1, a2);
    gP0 -= a0; gP1 -= a1; gP2 -= a2;
    ld3(G.warped_global_p2, o3, HW, gW0, gW1, gW2);
    gW0 += a0; gW1 += a1; gW2 += a2;
    // wpc: + warped_p2_camera_2 + R2^T g_wP2
    float gC0, gC1, gC2;
    ld3(G.warped_p2_camera_2, o3, HW, gC0, gC1, gC2);
    mtv(ps.R2, gW0, gW1, gW2, a0, a1, a2);
    gC0 += a0; gC1 += a1; gC2 += a2;
    // p12: + p1_camera_2 + K^T g_i12
    float gp0, gp1, gp2;
    ld3(G.p1_camera_2, o3, HW, gp0, gp1, gp2);
    float gi0 = 0.f, gi1 = 0.f, gi2 = G.depth_image ? G.depth_image[o1] : 0.f;
    if (G.dflow && o.zok) {
      const float gu = G.dflow[o2], gv = G.dflow[o2 + HW];
      gi0 += gu * o.rz; gi1 += gv * o.rz;
      gi2 -= (gu * o.i12[0] + gv * o.i12[1]) * o.rz * o.rz;
    }
    mtv(ps.K, gi0, gi1, gi2, a0, a1, a2);
    gp0 += a0; gp1 += a1; gp2 += a2;
    mv(ps.R2, gp0, gp1, gp2, b0v, b1v, b2v);        // g_(P1 + sf)
    st3(g_sf, o3, HW, b0v, b1v, b2v);
    gP0 += b0v; gP1 += b1v; gP2 += b2v;
    if (G.staticflow) {
      PixIn in0 = in;
      in0.sf[0] = in0.sf[1] = in0.sf[2] = 0.f;
      PixFwd os;
      pixel_forward(ps, d2img, H, W, x, yf, rt, in0, os);
      if (os.zok) {
        const float gu = G.staticflow[o2], gv = G.staticflow[o2 + HW];
        const float s0 = gu * os.rz, s1 = gv * os.rz, s2 = -(gu * os.i12[0] + gv * os.i12[1]) * os.rz * os.rz;
        mtv(ps.K, s0, s1, s2, a0, a1, a2);
        mv(ps.R2, a0, a1, a2, b0v, b1v, b2v);
        gP0 += b0v; gP1 += b1v; gP2 += b2v;
      }
    }
    // P1 = t1 - d1 * (nM1 c)
    float rx, ry, rz;
    ray_of(ps.nM1, x, yf, rx, ry, rz);
    if (g_d1) g_d1[o1] = -fmaf(gP2, rz, fmaf(gP1, ry, gP0 * rx));
    if (g_d2) {
      float hu, hv, h1, gd[4];
      mtv(ps.Kinv, gC0, gC1, gC2, hu, hv, h1);
      if (G.depth_warp) h1 += G.depth_warp[o1];
      tap_grads(o, hu, hv, h1, gd);
      scatter4_atomic(g_d2 + b * HW + o.i00, o.sx1, o.sy1, gd);
    }
  }
}

// ---------------------------------------------------------------------------------------------
static int pick_vec(int B, int H, int W, std::initializer_list<const void*> ptrs) {
  bool al = true;
  for (const void* p : ptrs) al = al && (p == nullptr || aligned16(p));
  long total = (long)B * H * W;
  // wide vectors only when enough threads remain to cover HBM latency (>= 512 / 256 threads per SM)
  if (al && W % 4 == 0 && total / 4 >= (long)num_sms() * 512) return 4;
  if (al && W % 2 == 0 && total / 2 >= (long)num_sms() * 256) return 2;
  return 1;
}

// ~8 CTAs of 256 threads per SM over the whole grid, split evenly over the pairs: a mild over-subscription lets short CTAs
// retire and refill continuously instead of finishing together. 8 CTAs per SM is also the hardware maximum for 256
// threads, so this bounds the partial-sum scratch of the generic forward.
static dim3 grid_for(int B, int items_per_pair) {
  int per_pair = (items_per_pair + kThreads - 1) / kThreads;
  const int cap = (num_sms() * 8 + B - 1) / B;
  if (per_pair > cap) per_pair = cap;
  if (per_pair < 1) per_pair = 1;
  return dim3((unsigned)per_pair, (unsigned)B, 1);
}

// Stage the derived poses of pairs [b0, b0 + nb) into a constant-memory slot (all on `st`, no host synchronisation).
// Slots rotate; a slot is handed out again only after the kernel that last read it has finished: every user records a
// per-slot event behind its kernel (release_pose_slot) and the next owner makes its stream wait on that event before it
// overwrites the slot, so calls in flight on any number of streams (or more than kPoseSlots deep) cannot see each other's
// poses. Symbol address and events are per device.
struct PoseSlots {
  PoseC* stage = nullptr;
  cudaEvent_t ev[kPoseSlots] = {};
  bool used[kPoseSlots] = {};
  unsigned ctr = 0;
  bool ok = false;
};
static std::mutex g_pose_mu;
static PoseSlots* pose_slots() {     // call with g_pose_mu held
  static PoseSlots per_dev[16];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return nullptr;
  PoseSlots& S = per_dev[dev];
  if (!S.ok) {
    void* p = nullptr;
    if (cudaGetSymbolAddress(&p, g_pose_stage) != cudaSuccess) return nullptr;
    S.stage = static_cast<PoseC*>(p);
    for (int i = 0; i < kPoseSlots; ++i)
      if (cudaEventCreateWithFlags(&S.ev[i], cudaEventDisableTiming) != cudaSuccess) return nullptr;
    S.ok = true;
  }
  return &S;
}
static int stage_poses(const float* poses, int b0, int nb, cudaStream_t st, int* slot_out) {
  std::lock_guard<std::mutex> lk(g_pose_mu);
  PoseSlots* S = pose_slots();
  DVD_ARG_CHECK(S != nullptr, "pose staging: cudaGetSymbolAddress / cudaEventCreate failed");
  const int slot = (int)(S->ctr++ % (unsigned)kPoseSlots);
  // (inside a stream capture the launches of the graph are ordered on the capture stream and replays are ordered on their
  // stream: events from outside the capture must not be waited on there)
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  DVD_CUDA_CALL(cudaStreamIsCapturing(st, &cap));
  if (cap == cudaStreamCaptureStatusNone && S->used[slot])
    DVD_CUDA_CALL(cudaStreamWaitEvent(st, S->ev[slot], 0));   // previous reader of this slot is done
  dvd::launch(pose_prep_kernel, 1, kPosePairs, 0, st, poses + (size_t)b0 * DVD_POSE_STRIDE, nb, slot);
  DVD_CUDA_LAUNCH_CHECK("pose_prep");
  DVD_CUDA_CALL(cudaMemcpyToSymbolAsync(c_pose, S->stage + (size_t)slot * kPosePairs, (size_t)nb * sizeof(PoseC),
                                        (size_t)slot * kPosePairs * sizeof(PoseC), cudaMemcpyDeviceToDevice, st));
  *slot_out = slot;
  return 0;
}
// record "the kernel reading `slot` has been enqueued on `st`" (call right after that launch)
static int release_pose_slot(int slot, cudaStream_t st) {
  std::lock_guard<std::mutex> lk(g_pose_mu);
  PoseSlots* S = pose_slots();
  DVD_ARG_CHECK(S != nullptr, "pose staging unavailable");
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  DVD_CUDA_CALL(cudaStreamIsCapturing(st, &cap));
  if (cap != cudaStreamCaptureStatusNone) return 0;
  DVD_CUDA_CALL(cudaEventRecord(S->ev[slot], st));
  S->used[slot] = true;
  return 0;
}

// Walks the pairs in chunks of at most kPosePairs: stages a chunk's poses, calls launch(slot, b0, nb) to enqueue the
// kernel that reads them, then releases the slot.
template <class Launch>
static int for_pose_chunks(const float* poses, int B, cudaStream_t st, Launch&& launch) {
  for (int b0 = 0; b0 < B; b0 += kPosePairs) {
    const int nb = std::min(B - b0, kPosePairs);
    int slot = 0;
    if (int e = stage_poses(poses, b0, nb, st, &slot)) return e;
    if (int e = launch(slot, b0, nb)) return e;
    if (int e = release_pose_slot(slot, st)) return e;
  }
  return 0;
}

// partial-sum quads written by the staged forward for one chunk of nb pairs
static int staged_quads(int nb, int HW) { return std::min(nb * ((HW + kTile - 1) / kTile), kFwdCtasPerSm * num_sms()); }
// grid of the generic forward (N = 2 pixels per thread when W is even)
static dim3 generic_fwd_grid(int B, int H, int W) { return grid_for(B, W % 2 == 0 ? H * W / 2 : H * W); }

static int check_shape(int B, int H, int W) {
  DVD_ARG_CHECK(B >= 1 && H >= 2 && W >= 2, "bad shape B=%d H=%d W=%d (need B>=1, H,W>=2)", B, H, W);
  DVD_ARG_CHECK(B <= 65535, "B=%d exceeds gridDim.y", B);
  DVD_ARG_CHECK((long)H * W < (1L << 30), "image too large");
  return 0;
}

}  // namespace dvd

using namespace dvd;

extern "C" int dvd_reproject_partials_size(int B, int H, int W) {
  if (B < 1 || H < 1 || W < 1) return 0;
  long staged = 0;
  for (int b0 = 0; b0 < B; b0 += kPosePairs) staged += staged_quads(std::min(B - b0, kPosePairs), H * W);
  const dim3 g = generic_fwd_grid(B, H, W);
  return (int)(std::max(staged, (long)g.x * g.y) * 4);
}

extern "C" int dvd_unproject_fwd(const float* depth, const float* poses, float* P, int B, int H, int W, int which,
                                 void* stream) {
  if (int e = check_shape(B, H, W)) return e;
  DVD_ARG_CHECK(depth && poses && P, "null pointer");
  DVD_ARG_CHECK(which == 1 || which == 2, "which must be 1 or 2");
  cudaStream_t st = (cudaStream_t)stream;
  int vec = pick_vec(B, H, W, {depth, P});
  const dim3 g = grid_for(B, H * W / vec);
  if (vec == 4) dvd::launch(unproject_fwd_kernel<4>, g, kThreads, 0, st, depth, poses, P, H, W, which);
  else if (vec == 2) dvd::launch(unproject_fwd_kernel<2>, g, kThreads, 0, st, depth, poses, P, H, W, which);
  else dvd::launch(unproject_fwd_kernel<1>, g, kThreads, 0, st, depth, poses, P, H, W, which);
  DVD_CUDA_LAUNCH_CHECK("unproject_fwd");
  return 0;
}

extern "C" int dvd_unproject_bwd(const float* gP, const float* poses, float* gdepth, int B, int H, int W, int which,
                                 void* stream) {
  if (int e = check_shape(B, H, W)) return e;
  DVD_ARG_CHECK(gP && poses && gdepth, "null pointer");
  DVD_ARG_CHECK(which == 1 || which == 2, "which must be 1 or 2");
  cudaStream_t st = (cudaStream_t)stream;
  int vec = pick_vec(B, H, W, {gP, gdepth});
  const dim3 g = grid_for(B, H * W / vec);
  if (vec == 4) dvd::launch(unproject_bwd_kernel<4>, g, kThreads, 0, st, gP, poses, gdepth, H, W, which);
  else if (vec == 2) dvd::launch(unproject_bwd_kernel<2>, g, kThreads, 0, st, gP, poses, gdepth, H, W, which);
  else dvd::launch(unproject_bwd_kernel<1>, g, kThreads, 0, st, gP, poses, gdepth, H, W, which);
  DVD_CUDA_LAUNCH_CHECK("unproject_bwd");
  return 0;
}

// cudaFuncSetAttribute once per (function, device)
static int set_smem_once(const void* fn, int smem) {
  static std::mutex mu;
  static std::vector<std::pair<const void*, int>> done;
  int dev = 0;
  DVD_CUDA_CALL(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(mu);
  for (auto& d : done)
    if (d.first == fn && d.second == dev) return 0;
  DVD_CUDA_CALL(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  done.emplace_back(fn, dev);
  return 0;
}

static int check_cfg(const dvd_loss_cfg* cfg) {
  DVD_ARG_CHECK(cfg != nullptr, "null loss cfg");
  DVD_ARG_CHECK(cfg->disp_mode >= 0 && cfg->disp_mode <= 2, "disp_mode must be 0,1,2");
  return 0;
}

extern "C" int dvd_reproject_loss_fwd(const float* depth_1, const float* depth_2, const float* flow_1_2,
                                      const float* mask_2, const float* sf, const float* poses,
                                      const dvd_loss_cfg* cfg, float* partials, float* scalars, int B, int H,
                                      int W, void* stream) {
  if (int e = check_shape(B, H, W)) return e;
  if (int e = check_cfg(cfg)) return e;
  DVD_ARG_CHECK(depth_1 && depth_2 && flow_1_2 && mask_2 && sf && poses && partials && scalars, "null pointer");
  DVD_ARG_CHECK(aligned16(partials), "partials must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int HW = H * W;
  // staged: 16-byte bulk copies need W % 4 == 0 and aligned bases; below the size threshold the generic kernel is faster
  const bool staged = pick_vec(B, H, W, {depth_1, mask_2, sf, flow_1_2}) == 4;
  if (staged)
    if (int e = set_smem_once((const void*)reproject_loss_fwd_staged_kernel, kStagedSmem)) return e;
  int nq = 0;
  if (staged) {
    int e = for_pose_chunks(poses, B, st, [&](int slot, int b0, int nb) -> int {
      const int gx = staged_quads(nb, HW);
      reproject_loss_fwd_staged_kernel<<<gx, kThreads + 32, kStagedSmem, st>>>(
          depth_1, depth_2, flow_1_2, mask_2, sf, *cfg, partials + (size_t)nq * 4, H, W, slot, b0, nb,
          (HW + kTile - 1) / kTile);
      nq += gx;
      DVD_CUDA_LAUNCH_CHECK("reproject_loss_fwd");
      return 0;
    });
    if (e) return e;
  } else {
    const dim3 g = generic_fwd_grid(B, H, W);
    if (W % 2 == 0)
      dvd::launch(reproject_loss_fwd_kernel<2>, g, kThreads, 0, st, depth_1, depth_2, flow_1_2, mask_2, sf, *cfg, partials,
                  H, W, poses);
    else
      dvd::launch(reproject_loss_fwd_kernel<1>, g, kThreads, 0, st, depth_1, depth_2, flow_1_2, mask_2, sf, *cfg, partials,
                  H, W, poses);
    DVD_CUDA_LAUNCH_CHECK("reproject_loss_fwd");
    nq = (int)(g.x * g.y);
  }
  dvd::launch(reproject_finalize_kernel, 1, 256, 0, st, partials, nq, *cfg, scalars);
  DVD_CUDA_LAUNCH_CHECK("reproject_finalize");
  return 0;
}

extern "C" int dvd_reproject_loss_bwd(const float* depth_1, const float* depth_2, const float* flow_1_2,
                                      const float* mask_2, const float* sf, const float* poses,
                                      const dvd_loss_cfg* cfg, const float* scalars, float gscale, const float* gscale_dev,
                                      float* g_sf, float* g_depth_2, int B, int H, int W, void* stream) {
  if (int e = check_shape(B, H, W)) return e;
  if (int e = check_cfg(cfg)) return e;
  DVD_ARG_CHECK(depth_1 && depth_2 && flow_1_2 && mask_2 && sf && poses && scalars && g_sf, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int HW = H * W;
  if (g_depth_2) DVD_CUDA_CALL(cudaMemsetAsync(g_depth_2, 0, (size_t)B * HW * sizeof(float), st));
  // staged: bulk copies and vector reductions need W % 4 == 0 and aligned bases; below the size threshold the generic
  // kernel is faster
  const bool staged = pick_vec(B, H, W, {depth_1, mask_2, sf, flow_1_2, g_sf, g_depth_2}) == 4;
  if (staged)
    if (int e = set_smem_once((const void*)reproject_loss_bwd_staged_kernel, kStagedSmem)) return e;
  if (staged)
    return for_pose_chunks(poses, B, st, [&](int slot, int b0, int nb) -> int {
      const int tiles_per_pair = (HW + kTile - 1) / kTile;
      const int gx = std::min(nb * tiles_per_pair, kBwdCtasPerSm * num_sms());
      reproject_loss_bwd_staged_kernel<<<gx, kThreads + 32, kStagedSmem, st>>>(
          depth_1, depth_2, flow_1_2, mask_2, sf, *cfg, scalars, gscale, gscale_dev, g_sf, g_depth_2, H, W, slot, b0, nb,
          tiles_per_pair);
      DVD_CUDA_LAUNCH_CHECK("reproject_loss_bwd");
      return 0;
    });
  dvd::launch(reproject_loss_bwd_kernel, grid_for(B, HW), kThreads, 0, st, depth_1, depth_2, flow_1_2, mask_2, sf, *cfg,
              scalars, gscale, gscale_dev, g_sf, g_depth_2, H, W, poses);
  DVD_CUDA_LAUNCH_CHECK("reproject_loss_bwd");
  return 0;
}

extern "C" int dvd_reproject_materialize(const float* depth_1, const float* depth_2, const float* flow_1_2,
                                         const float* sf, const float* poses, float* global_p1, float* sf_by_depth,
                                         float* warped_global_p2, float* warped_p2_camera_2, float* p1_camera_2,
                                         float* dflow_1_2, float* staticflow_1_2, float* depth_image_1_2,
                                         float* depth_warp_1_2, int B, int H, int W, void* stream) {
  if (int e = check_shape(B, H, W)) return e;
  DVD_ARG_CHECK(depth_1 && depth_2 && flow_1_2 && poses, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  dvd::launch(reproject_materialize_kernel, grid_for(B, H * W), kThreads, 0, st, depth_1, depth_2, flow_1_2, sf, global_p1,
              sf_by_depth, warped_global_p2, warped_p2_camera_2, p1_camera_2, dflow_1_2, staticflow_1_2, depth_image_1_2,
              depth_warp_1_2, H, W, poses);
  DVD_CUDA_LAUNCH_CHECK("reproject_materialize");
  return 0;
}

extern "C" int dvd_reproject_materialize_bwd(const float* depth_1, const float* depth_2, const float* flow_1_2,
                                             const float* sf, const float* poses, const float* g_global_p1,
                                             const float* g_sf_by_depth, const float* g_warped_global_p2,
                                             const float* g_warped_p2_camera_2, const float* g_p1_camera_2,
                                             const float* g_dflow_1_2, const float* g_staticflow_1_2,
                                             const float* g_depth_image_1_2, const float* g_depth_warp_1_2,
                                             float* g_depth_1, float* g_depth_2, float* g_sf, int B, int H, int W,
                                             void* stream) {
  if (int e = check_shape(B, H, W)) return e;
  DVD_ARG_CHECK(depth_1 && depth_2 && flow_1_2 && poses, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (g_depth_2) DVD_CUDA_CALL(cudaMemsetAsync(g_depth_2, 0, (size_t)B * H * W * sizeof(float), st));
  const MatGrads G{g_global_p1, g_sf_by_depth, g_warped_global_p2, g_warped_p2_camera_2, g_p1_camera_2,
                   g_dflow_1_2, g_staticflow_1_2, g_depth_image_1_2, g_depth_warp_1_2};
  dvd::launch(reproject_materialize_bwd_kernel, grid_for(B, H * W), kThreads, 0, st, depth_1, depth_2, flow_1_2, sf, G,
              g_depth_1, g_depth_2, g_sf, H, W, poses);
  DVD_CUDA_LAUNCH_CHECK("reproject_materialize_bwd");
  return 0;
}
