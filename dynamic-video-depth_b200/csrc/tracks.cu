// The learned scene flow read back from a test export (dvd_b200.tracks): flow consistency with the scene flow added, and 3D
// tracks integrated through the field drawn over the frames. oracle/tracks.py restates both rules in numpy, bit for bit.
//
//   dvd_pair_consistency_sf  dvd_pair_consistency for the refined depth, with each pair's scene flow added to the world point
//                            (the per-pixel code and the fixed-order fp64 sums are pair_consistency.cuh's), and a third region
//   dvd_draw_tracks          each frame's alive tracks, projected into its camera and rasterised with an exact, order-independent
//                            per-pixel key minimum, then resolved over the frame's colours
#include <math.h>

#include "pair_consistency.cuh"

namespace dvd {
namespace {

constexpr int kSfSlots = 3 * 6;          // regions all, static, moving: count, behind, sum e_r, sum e_d, #e_r < 1, #e_r < 3

__global__ void __launch_bounds__(kThreads) pair_consistency_sf_partial_kernel(
    const float* __restrict__ depth, const float* __restrict__ cam, const int* __restrict__ ia, const int* __restrict__ ib,
    const float* __restrict__ flow, const unsigned char* __restrict__ mask, const unsigned char* __restrict__ motion_seg,
    const float* __restrict__ sf, double* __restrict__ partials, int H, int W) {
  DVD_PDL_ENTER();
  __shared__ double red[(kThreads / 32) * kSfSlots];
  __shared__ double cm[2][30];
  const long pair = blockIdx.y, P = gridDim.x, hw = (long)H * W;
  const long fa = ia[pair], fb = ib[pair];
  stage_pair_cameras(cam, fa, fb, cm);
  double acc[kSfSlots];
#pragma unroll
  for (int j = 0; j < kSfSlots; ++j) acc[j] = 0.0;
  const float* fl = flow + pair * hw * 2;
  const unsigned char* mk = mask + pair * hw;
  const float* sp = sf + pair * 3 * hw;
  for (long i = (long)blockIdx.x * kThreads + threadIdx.x; i < hw; i += P * kThreads) {
    if (mk[i] != 0) continue;
    FlowTaps t;
    if (!flow_taps(i, H, W, *reinterpret_cast<const float2*>(fl + 2 * i), t)) continue;
    double er = 0.0, ed = 0.0;
    const int res = pair_pixel<true>(cm[0], cm[1], depth + fa * hw, depth + fb * hw, i, t, sp + i, hw, er, ed);
    if (res == kNotEvaluated) continue;
    add_pixel(acc, res, er, ed);
    if (motion_seg == nullptr) continue;
    if (motion_seg[fa * hw + i] == 0)
      add_pixel(acc + 6, res, er, ed);
    else
      add_pixel(acc + 12, res, er, ed);
  }
  block_sums<kSfSlots>(acc, red, partials + (pair * P + blockIdx.x) * kSfSlots);
}

// ---- drawing ------------------------------------------------------------------------------------------------------------------
constexpr int kCam = DVD_VIEW_CAM_FLOATS;     // w2c (3 x 4, row-major) then K (3 x 3, row-major)
constexpr unsigned long long kEmpty = ~0ull;
constexpr int kDrawThreads = 128;

// render_views' projection: q = w2c P, h = K q, (u, v) = h.xy / h.z, each operation rounded on its own; false when q.z <= 1e-2
// or a coordinate is not finite
__device__ __forceinline__ bool project_point(const float* __restrict__ cam, const float* __restrict__ p, float& u, float& v,
                                              float& z) {
  const float px = p[0], py = p[1], pz = p[2];
  float q[3], h[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float* w = cam + 4 * i;
    q[i] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w[0], px), __fmul_rn(w[1], py)), __fmul_rn(w[2], pz)), w[3]);
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float* k = cam + 12 + 3 * i;
    h[i] = __fadd_rn(__fadd_rn(__fmul_rn(k[0], q[0]), __fmul_rn(k[1], q[1])), __fmul_rn(k[2], q[2]));
  }
  if (!(q[2] > 0.01f) || !isfinite(q[0]) || !isfinite(q[1]) || !isfinite(q[2])) return false;
  u = __fdiv_rn(h[0], h[2]);
  v = __fdiv_rn(h[1], h[2]);
  z = q[2];
  return isfinite(u) && isfinite(v);
}

// pixel (xf + dx, yf + dy), xf = floor(u + 0.5): false outside the image or when z lies behind the frame's valid depth there
// by more than DVD_TRACK_HIDE_TOL; otherwise the key is min-accumulated (when keys is given)
__device__ __forceinline__ bool plot(unsigned long long* __restrict__ keys, const float* __restrict__ depth, int H, int W, float xf,
                                     float yf, int dx, int dy, float z, unsigned long long key) {
  if (!(xf >= (float)(-dx) && xf <= (float)(W - 1 - dx) && yf >= (float)(-dy) && yf <= (float)(H - 1 - dy))) return false;
  const long o = (long)((int)yf + dy) * W + ((int)xf + dx);
  const float d = depth[o];
  if (valid_depth(d) && z > __fmul_rn(d, DVD_TRACK_HIDE_TOL)) return false;
  if (keys != nullptr && key < __ldcg(keys + o)) atomicMin(keys + o, key);
  return true;
}

__global__ void fill_keys_kernel(unsigned long long* __restrict__ keys, long n) {
  DVD_PDL_ENTER();
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) keys[i] = kEmpty;
}

// grid (tracks / 128, frames): track i drawn in frame f when it is alive there, k = number[f] - first[i] in [0, len[i])
__global__ void __launch_bounds__(kDrawThreads) draw_tracks_kernel(
    const float* __restrict__ X, const int* __restrict__ first, const int* __restrict__ len, int M, int L1,
    const float* __restrict__ cams, const float* __restrict__ depth, const int* __restrict__ number, int H, int W, int tail,
    unsigned long long* __restrict__ keys, float* __restrict__ proj, unsigned char* __restrict__ vis) {
  DVD_PDL_ENTER();
  const int i = blockIdx.x * kDrawThreads + threadIdx.x;
  if (i >= M) return;
  const long f = blockIdx.y, hw = (long)H * W;
  const int k = number[f] - first[i];
  if (k < 0 || k >= len[i]) return;
  const float* cam = cams + f * kCam;
  const float* D = depth + f * hw;
  unsigned long long* kf = keys + f * hw;
  const float* Xi = X + (long)i * L1 * 3;
  // head: rank 0, a (2 r + 1)^2 square at the projection of X[i][k]; its centre sample is the step's projection and visibility
  float u, v, z;
  const bool ok = project_point(cam, Xi + 3 * k, u, v, z);
  bool seen = false;
  if (ok) {
    const float xf = floorf(__fadd_rn(u, 0.5f)), yf = floorf(__fadd_rn(v, 0.5f));
    const unsigned long long key = (unsigned long long)(unsigned)i;
    for (int dy = -DVD_TRACK_HEAD_RADIUS; dy <= DVD_TRACK_HEAD_RADIUS; ++dy)
      for (int dx = -DVD_TRACK_HEAD_RADIUS; dx <= DVD_TRACK_HEAD_RADIUS; ++dx) {
        const bool hit = plot(kf, D, H, W, xf, yf, dx, dy, z, key);
        if (dx == 0 && dy == 0) seen = hit;
      }
  }
  if (proj != nullptr) {
    const float nan = __int_as_float(0x7fc00000);
    float* pr = proj + ((long)i * L1 + k) * 3;
    pr[0] = ok ? u : nan;
    pr[1] = ok ? v : nan;
    pr[2] = ok ? z : nan;
    vis[(long)i * L1 + k] = seen ? 1 : 0;
  }
  // segments X[j] -> X[j + 1] for j = max(0, k - tail) .. k - 1, rank k - j: samples s = 0..S at t = s / S
  for (int j = max(0, k - tail); j < k; ++j) {
    float u0, v0, z0, u1, v1, z1;
    if (!project_point(cam, Xi + 3 * j, u0, v0, z0) || !project_point(cam, Xi + 3 * (j + 1), u1, v1, z1)) continue;
    const float du = __fsub_rn(u1, u0), dv = __fsub_rn(v1, v0), dz = __fsub_rn(z1, z0);
    const float n = fminf(ceilf(fmaxf(fabsf(du), fabsf(dv))), (float)DVD_TRACK_MAX_SAMPLES);
    const int S = n >= 1.f ? (int)n : 1;
    const unsigned long long key = ((unsigned long long)(k - j) << 32) | (unsigned long long)(unsigned)i;
    for (int s = 0; s <= S; ++s) {
      const float t = __fdiv_rn((float)s, (float)S);
      const float us = __fadd_rn(u0, __fmul_rn(t, du)), vs = __fadd_rn(v0, __fmul_rn(t, dv)), zs = __fadd_rn(z0, __fmul_rn(t, dz));
      plot(kf, D, H, W, floorf(__fadd_rn(us, 0.5f)), floorf(__fadd_rn(vs, 0.5f)), 0, 0, zs, key);
    }
  }
}

// one thread per pixel: the frame's floor(255 clip(img)) (NaN -> 0), or the winning track's colour faded by its rank:
// w = 256 (tail + 1 - rank) / (tail + 1) (integer division), out = (c w + base (256 - w) + 128) >> 8; BGR
__global__ void resolve_tracks_kernel(const unsigned long long* __restrict__ keys, const float* __restrict__ img,
                                      const unsigned char* __restrict__ rgb, long n, long hw, int tail,
                                      unsigned char* __restrict__ out) {
  DVD_PDL_ENTER();
  const long p = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const long f = p / hw, o = p % hw;
  const unsigned long long key = keys[p];
  int w = 0;
  const unsigned char* c = nullptr;
  if (key != kEmpty) {
    const int rank = (int)(key >> 32);
    w = 256 * (tail + 1 - rank) / (tail + 1);
    c = rgb + 3 * (long)(unsigned)(key & 0xffffffffull);
  }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const int base = (int)(unsigned char)__fmul_rn(fminf(fmaxf(img[(f * 3 + ch) * hw + o], 0.f), 1.f), 255.f);
    const int v = c ? (c[ch] * w + base * (256 - w) + 128) >> 8 : base;
    out[p * 3 + (2 - ch)] = (unsigned char)v;
  }
}

#define TR_CHECK(cond, ...)        \
  do {                             \
    if (!(cond)) {                 \
      dvd::set_error(__VA_ARGS__); \
      return -2;                   \
    }                              \
  } while (0)

static inline bool aligned_to(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

}  // namespace
}  // namespace dvd

using namespace dvd;

extern "C" long long dvd_pair_consistency_sf_partials_size(int n_pairs, int H, int W) {
  if (n_pairs < 1 || H < 1 || W < 1) return -1;
  return (long long)n_pairs * parts_for((long)H * W, kPixelsPerThread) * kSfSlots;
}

extern "C" int dvd_pair_consistency_sf(const float* depth, const float* cam, int n_frames, const int* ia, const int* ib,
                                       const float* flow, const unsigned char* mask, const unsigned char* motion_seg, const float* sf,
                                       double* sums, double* partials, int n_pairs, int H, int W, void* stream) {
  TR_CHECK(depth && cam && ia && ib && flow && mask && sf && sums && partials,
           "dvd_pair_consistency_sf: null pointer (only `motion_seg` may be NULL)");
  TR_CHECK(n_frames >= 1 && n_pairs >= 1 && n_pairs <= 65535 && H >= 1 && W >= 1,
           "dvd_pair_consistency_sf: bad shape n_frames=%d n_pairs=%d H=%d W=%d (1 <= n_pairs <= 65535)", n_frames, n_pairs, H, W);
  TR_CHECK(aligned_to(depth, 4) && aligned_to(cam, 4) && aligned_to(ia, 4) && aligned_to(ib, 4) && aligned_to(flow, 8) &&
               aligned_to(sf, 4) && aligned_to(sums, 8) && aligned_to(partials, 8),
           "dvd_pair_consistency_sf: misaligned buffer");
  const int P = parts_for((long)H * W, kPixelsPerThread);
  const cudaStream_t st = (cudaStream_t)stream;
  DVD_CUDA_CALL(launch(pair_consistency_sf_partial_kernel, dim3(P, n_pairs), dim3(kThreads), 0, st, depth, cam, ia, ib, flow, mask,
                       motion_seg, sf, partials, H, W));
  DVD_CUDA_CALL(launch(reduce_partials_kernel, dim3(n_pairs), dim3(32), 0, st, (const double*)partials, sums, P, kSfSlots));
  return 0;
}

extern "C" int dvd_draw_tracks(const float* X, const int* first, const int* len, const unsigned char* rgb, int M, int L1,
                               const float* cams, const float* depth, const float* img, const int* number, int F, int H, int W,
                               int tail, unsigned long long* keys, unsigned char* out, float* proj, unsigned char* vis,
                               void* stream) {
  TR_CHECK(cams && depth && img && number && keys && out, "dvd_draw_tracks: null pointer");
  TR_CHECK(M == 0 || (X && first && len && rgb), "dvd_draw_tracks: null track pointer with M=%d tracks", M);
  TR_CHECK((proj == nullptr) == (vis == nullptr), "dvd_draw_tracks: give both proj and vis, or neither");
  TR_CHECK(M >= 0 && L1 >= 1 && F >= 1 && F <= 65535 && H >= 1 && W >= 1 && tail >= 0 && tail <= DVD_TRACK_MAX_TAIL,
           "dvd_draw_tracks: bad shape M=%d L1=%d F=%d H=%d W=%d tail=%d (1 <= F <= 65535, 0 <= tail <= %d)", M, L1, F, H, W, tail,
           DVD_TRACK_MAX_TAIL);
  TR_CHECK(aligned_to(X, 4) && aligned_to(first, 4) && aligned_to(len, 4) && aligned_to(cams, 4) && aligned_to(depth, 4) &&
               aligned_to(img, 4) && aligned_to(number, 4) && aligned_to(keys, 8) && aligned_to(proj, 4),
           "dvd_draw_tracks: misaligned buffer");
  const long hw = (long)H * W, n = (long)F * hw;
  const cudaStream_t st = (cudaStream_t)stream;
  DVD_CUDA_CALL(launch(fill_keys_kernel, dim3((unsigned)((n + 1023) / 1024 < 4096 ? (n + 1023) / 1024 : 4096)), dim3(256), 0, st,
                       keys, n));
  if (M > 0)
    DVD_CUDA_CALL(launch(draw_tracks_kernel, dim3((unsigned)((M + kDrawThreads - 1) / kDrawThreads), F), dim3(kDrawThreads), 0, st,
                         X, first, len, M, L1, cams, depth, number, H, W, tail, keys, proj, vis));
  DVD_CUDA_CALL(launch(resolve_tracks_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, (const unsigned long long*)keys,
                       img, rgb, n, hw, tail, out));
  return 0;
}
