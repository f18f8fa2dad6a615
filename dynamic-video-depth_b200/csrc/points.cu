// Point-cloud export: the per-pixel selection of a video's refined depth maps (validity, flying pixels, voxel keys, colours,
// compaction in pixel order) and the per-voxel reduction of the key-sorted points (fp64 means, counts, distinct frames).
//
// Both entry points compact with the same deterministic stream compaction: the items are cut into tiles of kTile; one pass
// counts each tile's kept items (warp ballots), one block scans the tile counts in index order, and a second pass recomputes
// the flags and writes every kept item at its tile offset plus its rank within the tile. The output position of an item is
// its rank among the kept items, whatever the launch geometry: no atomic decides an order.
#include <math.h>

#include "common.cuh"

namespace dvd {
namespace {

constexpr int kThreads = 256;
constexpr int kPerThread = 8;
constexpr int kTile = kThreads * kPerThread;
constexpr int kScanThreads = 1024;
constexpr int kKeyBits = 21;
constexpr long long kKeyRange = 1LL << kKeyBits;

#define PT_CHECK(cond, ...)        \
  do {                             \
    if (!(cond)) {                 \
      dvd::set_error(__VA_ARGS__); \
      return -2;                   \
    }                              \
  } while (0)

static inline bool aligned_to(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

long long n_tiles(long long n) { return (n + kTile - 1) / kTile; }

// scratch of one compaction: int tile counts, long long tile offsets, then {total, error flag}
struct Compaction {
  int* tile_count;
  long long* tile_offset;
  long long* status;  // [0] kept items, [1] error flag
};

// rounded up to 16 bytes, so that a region carved after this one keeps the 8-byte alignment of its long long arrays
size_t compaction_bytes(long long n) {
  const size_t b = (size_t)n_tiles(n) * (sizeof(int) + sizeof(long long)) + 2 * sizeof(long long);
  return (b + 15) & ~(size_t)15;
}

Compaction carve(void* scratch, long long n) {
  Compaction c;
  const long long t = n_tiles(n);
  c.tile_offset = reinterpret_cast<long long*>(scratch);
  c.status = c.tile_offset + t;
  c.tile_count = reinterpret_cast<int*>(c.status + 2);
  return c;
}

// pass 1: kept items per tile. F::count(i) may cache what the scatter pass needs.
template <class F>
__global__ void __launch_bounds__(kThreads) tile_count_kernel(F f, long long n, int* __restrict__ tile_count) {
  DVD_PDL_ENTER();
  __shared__ int warp_total[kThreads / 32];
  const long long t0 = (long long)blockIdx.x * kTile;
  int mine = 0;
#pragma unroll
  for (int k = 0; k < kPerThread; ++k) {
    const long long i = t0 + k * kThreads + threadIdx.x;
    if (i < n && f.count(i)) ++mine;
  }
  for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
  if ((threadIdx.x & 31) == 0) warp_total[threadIdx.x >> 5] = mine;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < kThreads / 32; ++w) s += warp_total[w];
    tile_count[blockIdx.x] = s;
  }
}

// pass 2: exclusive scan of the tile counts in tile order (one block; integer sums, so any grouping gives the same offsets)
__global__ void __launch_bounds__(kScanThreads) tile_scan_kernel(const int* __restrict__ tile_count, long long* __restrict__ tile_offset,
                                                                  long long ntiles, long long* __restrict__ status) {
  DVD_PDL_ENTER();
  __shared__ long long part[kScanThreads];
  const long long per = (ntiles + kScanThreads - 1) / kScanThreads;
  const long long b = threadIdx.x * per, e = min(b + per, ntiles);
  long long s = 0;
  for (long long t = b; t < e; ++t) s += tile_count[t];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int o = 1; o < kScanThreads; o <<= 1) {  // inclusive Hillis-Steele scan
    const long long v = threadIdx.x >= o ? part[threadIdx.x - o] : 0;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  long long off = part[threadIdx.x] - s;
  for (long long t = b; t < e; ++t) {
    tile_offset[t] = off;
    off += tile_count[t];
  }
  if (threadIdx.x == kScanThreads - 1) status[0] = part[kScanThreads - 1];
}

// pass 3: F::keep(i) recomputes the flag; F::emit(i, kept, pos) runs for every item, pos = its rank among the kept items
template <class F>
__global__ void __launch_bounds__(kThreads) tile_scatter_kernel(F f, long long n, const long long* __restrict__ tile_offset) {
  DVD_PDL_ENTER();
  __shared__ int warp_total[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long t0 = (long long)blockIdx.x * kTile;
  long long base = tile_offset[blockIdx.x];
  for (int k = 0; k < kPerThread; ++k) {
    const long long i = t0 + k * kThreads + threadIdx.x;
    const bool kept = i < n && f.keep(i);
    const unsigned bal = __ballot_sync(0xffffffffu, kept);
    if (lane == 0) warp_total[warp] = __popc(bal);
    __syncthreads();
    int before = 0, all = 0;
    for (int w = 0; w < kThreads / 32; ++w) {
      const int c = warp_total[w];
      before += w < warp ? c : 0;
      all += c;
    }
    if (i < n) f.emit(i, kept, base + before + __popc(bal & ((1u << lane) - 1u)));
    base += all;
    __syncthreads();
  }
}

template <class F>
cudaError_t compact(const F& f, long long n, const Compaction& c, cudaStream_t st) {
  const long long t = n_tiles(n);
  cudaError_t e = launch(tile_count_kernel<F>, dim3((unsigned)t), dim3(kThreads), 0, st, f, n, c.tile_count);
  if (e == cudaSuccess) e = launch(tile_scan_kernel, dim3(1), dim3(kScanThreads), 0, st, (const int*)c.tile_count, c.tile_offset, t, c.status);
  if (e == cudaSuccess) e = launch(tile_scatter_kernel<F>, dim3((unsigned)t), dim3(kThreads), 0, st, f, n, (const long long*)c.tile_offset);
  return e;
}

// ---- selection ---------------------------------------------------------------------------------------------------------------
// A pixel is kept when its depth d is finite and > 1e-2 (fp32 threshold, depth2disp's) and |d - d_n| / d <= edge_tol (fp64)
// for every in-image 4-neighbour n; a NaN neighbour fails the test.
struct Select {
  const float* depth;
  const float* img;
  const float* P;
  int H, W;
  long long HW;
  double edge_tol, voxel;
  long long ox, oy, oz, base;
  unsigned char* mask;
  long long* key;
  long long* index;
  float* xyz;
  unsigned char* rgb;
  long long* status;

  __device__ bool valid(long long i) const {
    const float d = __ldg(depth + i);
    if (!(isfinite(d) && d > 0.01f)) return false;
    const long long r = i % HW;
    const int y = (int)(r / W), x = (int)(r - (long long)y * W);
    const double dd = (double)d;
    bool ok = true;
    if (x > 0) ok &= fabs(__dsub_rn(dd, (double)__ldg(depth + i - 1))) / dd <= edge_tol;
    if (x < W - 1) ok &= fabs(__dsub_rn(dd, (double)__ldg(depth + i + 1))) / dd <= edge_tol;
    if (y > 0) ok &= fabs(__dsub_rn(dd, (double)__ldg(depth + i - W))) / dd <= edge_tol;
    if (y < H - 1) ok &= fabs(__dsub_rn(dd, (double)__ldg(depth + i + W))) / dd <= edge_tol;
    return ok;
  }
  __device__ bool count(long long i) const { return valid(i); }
  __device__ bool keep(long long i) const { return valid(i); }

  // floor(p / voxel) - origin in [0, 2^21); -1 when out of range (NaN included)
  __device__ static long long axis_key(float p, double voxel, long long origin) {
    const double q = floor((double)p / voxel);
    if (!(q >= (double)origin && q < (double)origin + (double)kKeyRange)) return -1;
    return (long long)q - origin;
  }

  __device__ void emit(long long i, bool kept, long long pos) const {
    mask[i] = kept ? 1 : 0;
    if (!kept) return;
    const long long f = i / HW, r = i - f * HW;
    const float* p = P + f * 3 * HW + r;
    const float px = __ldg(p), py = __ldg(p + HW), pz = __ldg(p + 2 * HW);
    if (key) {
      const long long kx = axis_key(px, voxel, ox), ky = axis_key(py, voxel, oy), kz = axis_key(pz, voxel, oz);
      if (kx < 0 || ky < 0 || kz < 0) {
        status[1] = 1;  // every writer stores the same value
        key[pos] = -1;
      } else {
        key[pos] = (kx << (2 * kKeyBits)) | (ky << kKeyBits) | kz;
      }
    }
    index[pos] = base + i;
    xyz[3 * pos] = px;
    xyz[3 * pos + 1] = py;
    xyz[3 * pos + 2] = pz;
    const float* c = img + f * 3 * HW + r;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      // floor(255 clip(v, 0, 1)) in fp32; fmaxf maps NaN to 0
      const float v = fminf(fmaxf(__ldg(c + ch * HW), 0.f), 1.f);
      rgb[3 * pos + ch] = (unsigned char)__fmul_rn(v, 255.f);
    }
  }
};

// ---- voxel reduction -----------------------------------------------------------------------------------------------------
// run heads of the sorted keys -> run_start[r]; run_start[R] = M
struct Heads {
  const long long* skey;
  long long M;
  long long* run_start;
  const long long* status;
  __device__ bool head(long long j) const { return j == 0 || skey[j] != skey[j - 1]; }
  __device__ bool count(long long j) const { return head(j); }
  __device__ bool keep(long long j) const { return head(j); }
  __device__ void emit(long long j, bool kept, long long pos) const {
    if (kept) run_start[pos] = j;
    if (j == M - 1) run_start[status[0]] = M;  // status[0] = R, final once the scan has run
  }
};

// runs seen in at least min_views frames; views are counted in the count pass and cached for the scatter pass
struct Runs {
  const long long* run_start;
  const long long* nruns;  // device R
  const long long* order;
  const long long* index;
  const float* xyz;
  const unsigned char* rgb;
  long long hw;
  int min_views;
  int* views_tmp;
  double* mean_xyz;
  double* mean_rgb;
  int* count_out;
  int* views_out;

  __device__ bool count(long long r) const {
    if (r >= *nruns) return false;
    const long long b = run_start[r], e = run_start[r + 1];
    int v = 0;
    long long last = -1;
    for (long long j = b; j < e; ++j) {  // stable sort: the frames of a run ascend
      const long long f = __ldg(index + __ldg(order + j)) / hw;
      v += f != last;
      last = f;
    }
    views_tmp[r] = v;
    return v >= min_views;
  }
  __device__ bool keep(long long r) const { return r < *nruns && views_tmp[r] >= min_views; }
  __device__ void emit(long long r, bool kept, long long pos) const {
    if (!kept) return;
    const long long b = run_start[r], e = run_start[r + 1];
    double sx = 0, sy = 0, sz = 0, sr = 0, sg = 0, sb = 0;
    for (long long j = b; j < e; ++j) {  // sorted order, one rounding per addition
      const long long s = __ldg(order + j);
      sx = __dadd_rn(sx, (double)__ldg(xyz + 3 * s));
      sy = __dadd_rn(sy, (double)__ldg(xyz + 3 * s + 1));
      sz = __dadd_rn(sz, (double)__ldg(xyz + 3 * s + 2));
      sr = __dadd_rn(sr, (double)__ldg(rgb + 3 * s));
      sg = __dadd_rn(sg, (double)__ldg(rgb + 3 * s + 1));
      sb = __dadd_rn(sb, (double)__ldg(rgb + 3 * s + 2));
    }
    const double n = (double)(e - b);
    mean_xyz[3 * pos] = sx / n;
    mean_xyz[3 * pos + 1] = sy / n;
    mean_xyz[3 * pos + 2] = sz / n;
    mean_rgb[3 * pos] = sr / n;
    mean_rgb[3 * pos + 1] = sg / n;
    mean_rgb[3 * pos + 2] = sb / n;
    count_out[pos] = (int)(e - b);
    views_out[pos] = views_tmp[r];
  }
};

// reads {kept, error flag} back and waits for the stream
int read_status(const long long* status, long long* host, cudaStream_t st) {
  DVD_CUDA_CALL(cudaMemcpyAsync(host, status, 2 * sizeof(long long), cudaMemcpyDeviceToHost, st));
  DVD_CUDA_CALL(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace
}  // namespace dvd

using namespace dvd;

extern "C" long dvd_points_select_scratch_bytes(int N, int H, int W) {
  if (N < 1 || H < 1 || W < 1) return -1;
  return (long)compaction_bytes((long long)N * H * W);
}

extern "C" int dvd_points_select(const float* depth, const float* img, const float* P, int N, int H, int W, double edge_tol,
                                 double voxel, long long ox, long long oy, long long oz, long long base, unsigned char* mask,
                                 long long* key, long long* index, float* xyz, unsigned char* rgb, void* scratch, size_t scratch_bytes,
                                 long long* n_valid, void* stream) {
  PT_CHECK(depth && img && P && mask && index && xyz && rgb && scratch && n_valid, "dvd_points_select: null pointer");
  PT_CHECK(N >= 1 && H >= 1 && W >= 1, "dvd_points_select: bad shape N=%d H=%d W=%d", N, H, W);
  PT_CHECK(edge_tol >= 0.0, "dvd_points_select: edge_tol must be >= 0, got %g", edge_tol);
  PT_CHECK(!key || (voxel > 0.0 && isfinite(voxel)), "dvd_points_select: voxel must be positive and finite, got %g", voxel);
  PT_CHECK(base >= 0, "dvd_points_select: negative index base");
  const long long n = (long long)N * H * W;
  PT_CHECK(scratch_bytes >= compaction_bytes(n), "dvd_points_select: scratch %zu bytes, need %zu", scratch_bytes, compaction_bytes(n));
  PT_CHECK(aligned_to(scratch, 8) && aligned_to(index, 8) && aligned_to(key, 8) && aligned_to(xyz, 4),
           "dvd_points_select: misaligned buffer");
  cudaStream_t st = (cudaStream_t)stream;
  const Compaction c = carve(scratch, n);
  DVD_CUDA_CALL(cudaMemsetAsync(c.status, 0, 2 * sizeof(long long), st));
  const Select f{depth, img, P, H, W, (long long)H * W, edge_tol, voxel, ox, oy, oz, base, mask, key, index, xyz, rgb, c.status};
  DVD_CUDA_CALL(compact(f, n, c, st));
  long long s[2];
  if (int e = read_status(c.status, s, st)) return e;
  *n_valid = s[0];
  if (s[1]) {
    dvd::set_error("dvd_points_select: a voxel key is outside [0, 2^21) on some axis (voxel %g, origin %lld %lld %lld)", voxel, ox,
                   oy, oz);
    return -3;
  }
  return 0;
}

extern "C" long dvd_voxel_reduce_scratch_bytes(long long M) {
  if (M < 1) return -1;
  // two compactions over M items, run_start [M + 1], views [M]
  return (long)(2 * compaction_bytes(M) + (size_t)(M + 1) * sizeof(long long) + (size_t)M * sizeof(int));
}

extern "C" int dvd_voxel_reduce(const long long* skey, const long long* order, const long long* index, const float* xyz,
                                const unsigned char* rgb, long long M, long long hw, int min_views, double* mean_xyz, double* mean_rgb,
                                int* count, int* views, void* scratch, size_t scratch_bytes, long long* n_out, void* stream) {
  PT_CHECK(skey && order && index && xyz && rgb && mean_xyz && mean_rgb && count && views && scratch && n_out,
           "dvd_voxel_reduce: null pointer");
  PT_CHECK(M >= 1 && hw >= 1 && min_views >= 1, "dvd_voxel_reduce: bad arguments M=%lld hw=%lld min_views=%d", M, hw, min_views);
  const size_t need = (size_t)dvd_voxel_reduce_scratch_bytes(M);
  PT_CHECK(scratch_bytes >= need, "dvd_voxel_reduce: scratch %zu bytes, need %zu", scratch_bytes, need);
  PT_CHECK(aligned_to(scratch, 8) && aligned_to(skey, 8) && aligned_to(order, 8) && aligned_to(index, 8) && aligned_to(mean_xyz, 8) &&
               aligned_to(mean_rgb, 8) && aligned_to(count, 4) && aligned_to(views, 4) && aligned_to(xyz, 4),
           "dvd_voxel_reduce: misaligned buffer");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t cb = compaction_bytes(M);
  const Compaction heads = carve(scratch, M);
  const Compaction runs = carve(static_cast<char*>(scratch) + cb, M);
  long long* run_start = reinterpret_cast<long long*>(static_cast<char*>(scratch) + 2 * cb);
  int* views_tmp = reinterpret_cast<int*>(run_start + M + 1);
  PT_CHECK(aligned_to(runs.tile_offset, 8) && aligned_to(run_start, 8), "dvd_voxel_reduce: misaligned scratch layout");
  DVD_CUDA_CALL(cudaMemsetAsync(heads.status, 0, 2 * sizeof(long long), st));
  DVD_CUDA_CALL(cudaMemsetAsync(runs.status, 0, 2 * sizeof(long long), st));
  DVD_CUDA_CALL(compact(Heads{skey, M, run_start, heads.status}, M, heads, st));
  const Runs f{run_start, heads.status, order, index, xyz, rgb, hw, min_views, views_tmp, mean_xyz, mean_rgb, count, views};
  DVD_CUDA_CALL(compact(f, M, runs, st));
  long long s[2];
  if (int e = read_status(runs.status, s, st)) return e;
  *n_out = s[0];
  return 0;
}
