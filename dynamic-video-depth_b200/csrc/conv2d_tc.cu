// Depth-net convolutions (every class of the MiDaS / ResNeXt101-32x8d stack) on the Hopper tensor cores.
//
// One implicit-GEMM kernel family on NHWC fp32 tensors whose values are already rounded to TF32 (round-to-nearest) by
// the kernel that produced them ("rounded-operand contract", DESIGN.md 4.5): wgmma.mma_async TF32, both operands K-major
// in shared memory, fp32 accumulators in registers. Replaces cuDNN behind torch.nn.Conv2d / convolution_backward for
//   dense 1x1 / 3x3 stride 1     third_party/midas_blocks.py:53-68,121-168; third_party/MiDaS.py:188-195; torchvision Bottleneck conv1/conv3
//   1x1 / 3x3 stride 2           torchvision Bottleneck.downsample, conv2 of the first block of layer2-4
//   grouped 3x3 (32 groups)      torchvision Bottleneck.conv2 (ResNeXt), as block-diagonal 64-channel GEMM blocks
//   the data gradient of each    same kernel: transposed (BatchNorm-scaled) weight image, a tap table instead of a fixed
//                                3x3 stencil, stride-2 gradients as 4 sub-pixel phases with a strided store
//   the weight gradient of each  conv_wgrad_kernel below (K = pixels, both operands channel-contiguous: one from registers,
//                                the other transposed in shared memory)
// with the elementwise neighbours folded into the epilogue:  y = round_tf32(mask * relu(acc * scale + shift + res + res2))
// (eval-mode BatchNorm / bias, residual adds, ReLU forward; residual-gradient add and ReLU mask backward).
//
//   D[128 pixels, NT channels] += sum over taps t, 32-channel chunks c of
//     A_t,c [128 px x 32 ch]  TMA box {32 ch, TW, TH, 1} of the NHWC input at stride * tile origin + (dy_t, dx_t), element
//                             stride = conv stride; out-of-image elements are zero-filled by the hardware (= padding);
//                             lands as the canonical SWIZZLE_128B K-major image
//   x W_t,c [NT x 32]         TMA box {32, NT, 1} of the packed weight image [tap][rows][cols]
// One persistent CTA per SM, three warpgroups: warpgroup 0 = TMA producer (one thread, ring of kStages stages), warpgroups
// 1 and 2 = MMA + epilogue, each owning 64 pixel rows of the tile (m64nNTk8 wgmma, NT / 2 accumulator registers per
// thread); the epilogue stores straight from the accumulator fragments (each quad of lanes writes 32 contiguous bytes).
#include "common.cuh"
#include "tc_common.cuh"

#include <cuda.h>
#include <cudaTypedefs.h>
#include <type_traits>

namespace dvd {
namespace {

using namespace tc;

constexpr int kStages = 4;
constexpr int kThreads = 384;               // TMA producer warpgroup, two MMA / epilogue warpgroups
constexpr int kABytes = 128 * 128;          // 128 pixels x 32 fp32 channels
constexpr int kMaxNT = 256;
constexpr int kStageBytes = kABytes + kMaxNT * 128;
constexpr int kOffAff = kStages * kStageBytes;              // scale[256] | shift[256]
constexpr int kOffBar = kOffAff + 2 * kMaxNT * 4;
constexpr size_t kSmem = kOffBar + 256;
constexpr int kWsFlagWords = 256;           // stream-K exchange area: flag words in front of the partial tiles
constexpr int kConsumers = 256;             // threads of the two MMA warpgroups

struct ConvParams {
  dvd_conv_desc d;
  const float* bias;
  const float* gamma;
  const float* beta;
  const float* mean;
  const float* var;
  const float* res;
  const float* res2;
  const float* mask;
  float* y;
  int TW, TH, tiles_w, tiles_h;   // pixel tile = TH x TW = 128 over the (OH, OW) grid
  int NT;                         // output channels per tile
  int kchunks;                    // 32-channel chunks per tap
  int sk;                         // stream-K: the (tile, K-step) work list is cut into one contiguous range per CTA instead of
                                  // whole tiles round-robin; a tile cut by a range boundary is finished by the CTA that owns its
                                  // FIRST K-steps (it reaches that tile last), the others leave raw partial accumulators in `ws`
  float* ws;                      // int flags[256] (zero when idle) | [gridDim.x][128][NT] partial tiles
};

// One segment of work: K-steps [k0, k1) of tile `tile`. Data-parallel mode: whole tiles, round-robin over the CTAs.
// Stream-K mode: the CTA's contiguous range of the tile-major (tile, K-step) list; range boundaries that fall within 1/8 of a
// tile boundary snap to it (a sliver is not worth a partial-tile exchange).
struct SegIter {
  long u, u1;
  int tile, ntiles, step, ksteps, sk;
  __host__ __device__ static long bound(long c, long n_clusters, long total, int ksteps) {
    if (c >= n_clusters) return total;
    long u = c * total / n_clusters;
    const int r = (int)(u % ksteps);
    if (r * 8 < ksteps) u -= r;
    else if ((ksteps - r) * 8 < ksteps) u += ksteps - r;
    return u;
  }
  __device__ SegIter(int sk_, int cluster_id, int n_clusters, int ntiles_, int ksteps_) : ntiles(ntiles_), step(n_clusters), ksteps(ksteps_), sk(sk_) {
    tile = cluster_id;
    if (sk) {
      const long total = (long)ntiles * ksteps;
      u = bound(cluster_id, n_clusters, total, ksteps);
      u1 = bound(cluster_id + 1, n_clusters, total, ksteps);
    } else {
      u = u1 = 0;
    }
  }
  __device__ bool next(int& t, int& k0, int& k1) {
    if (!sk) {
      if (tile >= ntiles) return false;
      t = tile; k0 = 0; k1 = ksteps;
      tile += step;
      return true;
    }
    if (u >= u1) return false;
    t = (int)(u / ksteps);
    k0 = (int)(u - (long)t * ksteps);
    const long left = u1 - u;
    k1 = (left < (long)(ksteps - k0)) ? k0 + (int)left : ksteps;
    u += k1 - k0;
    return true;
  }
};

__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ float round_tf32(float v) {
  uint32_t o;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(o) : "f"(v));
  return __uint_as_float(o);
}

struct Tile {
  int n0, img, h0, w0;
};
// tile ct = (channel tile, pixel tile), channel-tile major: consecutive tiles share the weight tile
__device__ __forceinline__ Tile decode_tile(const ConvParams& P, int ct, int m_tiles) {
  Tile t;
  const int nt = ct / m_tiles, m = ct - nt * m_tiles;
  t.n0 = nt * P.NT;
  const int per_img = P.tiles_w * P.tiles_h;
  t.img = m / per_img;
  const int r = m - t.img * per_img;
  const int th = r / P.tiles_w;
  t.h0 = th * P.TH;
  t.w0 = (r - th * P.tiles_w) * P.TW;
  return t;
}

template <int NT>
__global__ void __launch_bounds__(kThreads, 1) conv2d_tc_kernel(const __grid_constant__ CUtensorMap mapA,
                                                               const __grid_constant__ CUtensorMap mapW,
                                                               const __grid_constant__ ConvParams P) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* full = bars;                       // [kStages]
  uint64_t* empty = bars + 8;                  // [kStages]: one arrival per MMA warp
  float* aff_mem = reinterpret_cast<float*>(smem + kOffAff);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();   // swizzled stages need 1024-byte alignment
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    fence_mbar_init();
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapW) : "memory");
  }
  __syncthreads();
  DVD_PDL_ENTER();                             // set-up done: now wait for the producer of the operands

  const int m_tiles = P.d.N * P.tiles_w * P.tiles_h;
  const int n_tiles = (P.d.Cout + NT - 1) / NT;   // the last channel tile may be ragged: the weight rows beyond Cout are
                                                  // zero-filled by the TMA unit, the epilogue skips them
  const int ntiles = m_tiles * n_tiles;
  const int ksteps = P.d.ntaps * P.kchunks;

  if (wg == 0) {
    setmaxnreg_dec<40>();
    // ===== TMA producer =====
    if (threadIdx.x == 0) {
      const uint32_t stage_tx = (uint32_t)kABytes + (uint32_t)NT * 128u;
      uint32_t it = 0;
      SegIter seg(P.sk, blockIdx.x, gridDim.x, ntiles, ksteps);
      int tile, k0, k1;
      while (seg.next(tile, k0, k1)) {
        const Tile T = decode_tile(P, tile, m_tiles);
        const int kbase = P.d.kblock ? (T.n0 / P.d.kblock) * P.d.kblock : 0;
        const int ws = T.w0 * P.d.stride, hs = T.h0 * P.d.stride;
        int t = k0 / P.kchunks, kc = k0 - t * P.kchunks;
        for (int k = k0; k < k1; ++t, kc = 0) {
          const int dy = P.d.dy[t], dx = P.d.dx[t], wt = P.d.wt[t];
          for (; kc < P.kchunks && k < k1; ++kc, ++k, ++it) {
            const uint32_t s = it % kStages, ph = (it / kStages) & 1u;
            uint8_t* st = smem + (size_t)s * kStageBytes;
            mbar_wait(&empty[s], ph ^ 1u);            // both MMA warpgroups have drained this stage
            mbar_arrive_expect_tx(&full[s], stage_tx);
            tma_load_4d(st, &mapA, kbase + kc * 32, ws + dx, hs + dy, T.img, &full[s]);
            tma_load_3d(st + kABytes, &mapW, kc * 32, T.n0, wt, &full[s]);
          }
        }
      }
    }
    return;
  }
  setmaxnreg_inc<232>();
  // ===== MMA + epilogue: warpgroup cw owns pixel rows [64 cw, 64 cw + 64) of the tile =====
  const int cw = wg - 1;
  const int et = threadIdx.x - 128;              // 0..255 among the MMA threads
  const int qrow = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows qrow, qrow + 8
  const int qcol = 2 * (lane & 3);                            // fragment columns 8 j + qcol, + 1
  const bool has_aff = P.gamma != nullptr || P.bias != nullptr;
  float acc[NT / 2];
  uint32_t it = 0;
  SegIter seg(P.sk, blockIdx.x, gridDim.x, ntiles, ksteps);
  int tile, k0, k1;
  while (seg.next(tile, k0, k1)) {
    // ---- main loop: one stage = 32 channels of one tap, four k8 MMAs; a stage is released once the MMAs that read it are done
    uint32_t prev = 0;
    for (int k = 0; k < k1 - k0; ++k, ++it) {
      const uint32_t s = it % kStages, ph = (it / kStages) & 1u;
      mbar_wait(&full[s], ph);
      const uint32_t sa = smem_u32(smem + (size_t)s * kStageBytes) + (uint32_t)cw * 8192u, sb = smem_u32(smem + (size_t)s * kStageBytes) + kABytes;
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
        wgmma_tf32_ss<NT>(acc, make_sdesc_k_sw128(sa + ks * 32), make_sdesc_k_sw128(sb + ks * 32), (k | ks) ? 1u : 0u);
      wgmma_commit();
      if (k > 0) {
        wgmma_wait<1>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);
      }
      prev = s;
    }
    wgmma_wait<0>();
    fence_regs(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[prev]);

    if (k0 > 0) {
      // ---- partial tile (its first K-steps belong to an earlier CTA): raw accumulators -> exchange area, raise the flag ----
      // layout of a partial tile: [register][thread] - a warp stores 128 contiguous bytes per instruction
      float* wp = P.ws + kWsFlagWords + (size_t)blockIdx.x * 128 * NT + et;
#pragma unroll
      for (int i = 0; i < NT / 2; ++i)
        asm volatile("st.relaxed.gpu.global.f32 [%0], %1;" ::"l"(wp + (size_t)i * kConsumers), "f"(acc[i]) : "memory");
      __threadfence();
      named_sync(1, kConsumers);
      if (et == 0) {
        int* ws_flags = reinterpret_cast<int*>(P.ws);
        asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(ws_flags + blockIdx.x), "r"(1) : "memory");
      }
      continue;
    }
    // a tile this CTA starts but does not finish: the CTAs whose ranges begin inside it deliver the rest
    int n_part = 0;
    if (k1 < ksteps) {
      const long total = (long)ntiles * ksteps, tile_end = (long)(tile + 1) * ksteps;
      while ((int)blockIdx.x + 1 + n_part < (int)gridDim.x && SegIter::bound(blockIdx.x + 1 + n_part, gridDim.x, total, ksteps) < tile_end) ++n_part;
    }
    const Tile T = decode_tile(P, tile, m_tiles);
    const int ntv = min(NT, P.d.Cout - T.n0);      // channels of this tile that exist (ragged last tile)
    if (has_aff) {
      // fold BatchNorm / bias of this tile's channels once: y = acc * scale + shift
      named_sync(1, kConsumers);                   // previous tile's readers are done
      for (int i = et; i < ntv; i += kConsumers) {
        const int c = T.n0 + i;
        float sc = 1.f, sh = 0.f;
        if (P.gamma) {
          sc = __ldg(P.gamma + c) * rsqrtf(__ldg(P.var + c) + P.d.bn_eps);
          sh = __ldg(P.beta + c) - __ldg(P.mean + c) * sc;
        }
        if (P.bias) sh = fmaf(__ldg(P.bias + c), sc, sh);
        aff_mem[i] = sc;
        aff_mem[kMaxNT + i] = sh;
      }
      named_sync(1, kConsumers);
    }
    if (n_part) {
      // the partial tiles were written long ago (they are the FIRST thing the later CTAs do): this wait is short
      if (et < n_part) {
        const int* f = reinterpret_cast<const int*>(P.ws) + blockIdx.x + 1 + et;
        int v = 0;
        const long long t0 = clock64();
        do {
          asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
          if (!v && clock64() - t0 > 4000000000LL) __trap();   // a partial tile that never arrives: fail, do not hang
        } while (!v);
      }
      named_sync(1, kConsumers);
      for (int pi = 0; pi < n_part; ++pi) {
        const float* pp = P.ws + kWsFlagWords + (size_t)(blockIdx.x + 1 + pi) * 128 * NT + et;
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) {
          // strong (gpu-scope) load: the tile was written by another SM; a weak load may be served from a stale L1 line
          float a;
          asm volatile("ld.relaxed.gpu.global.f32 %0, [%1];" : "=f"(a) : "l"(pp + (size_t)i * kConsumers) : "memory");
          acc[i] += a;
        }
      }
    }
    // ---- epilogue: two pixel rows per thread, pairs of channels
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = qrow + 8 * h;
      const int ph_ = T.h0 + row / P.TW, pw = T.w0 + row % P.TW;
      const int yh = ph_ * P.d.oy_mul + P.d.oy_add, yw = pw * P.d.ox_mul + P.d.ox_add;
      const bool valid = ph_ < P.d.OH && pw < P.d.OW && yh < P.d.YH && yw < P.d.YW;
      if (!valid) continue;
      const size_t off = (((size_t)T.img * P.d.YH + yh) * P.d.YW + yw) * P.d.Cout + T.n0;
#pragma unroll
      for (int j = 0; j < NT / 8; ++j) {
        const int c = 8 * j + qcol;
        if (c >= ntv) continue;
        float2 v = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        if (has_aff) {
          v.x = fmaf(v.x, aff_mem[c], aff_mem[kMaxNT + c]);
          v.y = fmaf(v.y, aff_mem[c + 1], aff_mem[kMaxNT + c + 1]);
        }
        if (P.res) { const float2 a = __ldg(reinterpret_cast<const float2*>(P.res + off + c)); v.x += a.x; v.y += a.y; }
        if (P.res2) { const float2 a = __ldg(reinterpret_cast<const float2*>(P.res2 + off + c)); v.x += a.x; v.y += a.y; }
        if (P.d.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); }
        if (P.mask) {
          const float2 m = __ldg(reinterpret_cast<const float2*>(P.mask + off + c));
          v.x = m.x > 0.f ? v.x : 0.f; v.y = m.y > 0.f ? v.y : 0.f;
        }
        if (P.d.round_out) { v.x = round_tf32(v.x); v.y = round_tf32(v.y); }
        *reinterpret_cast<float2*>(P.y + off + c) = v;
      }
    }
    if (n_part) {
      // every reader is done with the partial tiles: lower the flags for the next launch (ordered by the kernel boundary)
      named_sync(1, kConsumers);
      if (et < n_part) reinterpret_cast<int*>(P.ws)[blockIdx.x + 1 + et] = 0;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Weight images. weight[co, ci_local, ky, kx] (arbitrary element strides), groups of `cpg` in-channels (cpg = Cin: dense).
//   mode 0 (forward)        out[t][co][c]          c over Cin (dense) or over the `kblock` in-channels of co's block
//   mode 1 (data gradient)  out[t][ci][c]          c over Cout (dense) or over the `kblock` out-channels of ci's block,
//                                                  times the eval-BatchNorm scale gamma * rsqrt(var + eps) of that out-channel
// t = ky * k + kx (never flipped: the tap table of the launch carries the offsets). Entries outside a channel's group are
// zero (block-diagonal image of a grouped convolution). Values rounded to TF32 (RN).
__global__ void __launch_bounds__(256) conv_pack_kernel(const float* __restrict__ w, long s_co, long s_ci, long s_ky, long s_kx,
                                                        float* __restrict__ out_fwd, float* __restrict__ out_bwd, int Cout, int Cin,
                                                        int k, int cpg, int kblock, const float* __restrict__ gamma,
                                                        const float* __restrict__ var, float eps) {
  DVD_PDL_ENTER();
  // both images have k*k * C * cols elements when Cin == Cout or dense; they are walked with one index each
  const int opg = Cout / (Cin / cpg);        // out-channels per group
  for (int mode = 0; mode < 2; ++mode) {
    float* out = mode ? out_bwd : out_fwd;
    if (!out) continue;
    const int rows = mode ? Cin : Cout;
    const int cols = kblock ? kblock : (mode ? Cout : Cin);
    const long n = (long)k * k * rows * cols;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
      const int c = (int)(i % cols);
      const long q = i / cols;
      const int r = (int)(q % rows), t = (int)(q / rows);
      const int ky = t / k, kx = t - ky * k;
      const int cabs = kblock ? (r / kblock) * kblock + c : c;     // absolute channel index of the column
      const int co = mode ? cabs : r, ci = mode ? r : cabs;
      float v = 0.f;
      if (co / opg == ci / cpg) {                                  // same group (dense: one group)
        v = w[co * s_co + (ci % cpg) * s_ci + ky * s_ky + kx * s_kx];
        if (mode && gamma) v *= gamma[co] * rsqrtf(var[co] + eps);
      }
      out[i] = round_tf32(v);
    }
  }
}

// All layers of a net in ONE launch (the weights change every optimisation step, so every step re-packs ~250 images: as single
// launches that is 123 grids of a few microseconds each). items[] lives in device memory; item i owns the blocks
// [blk0[i], blk0[i+1]) of the grid.
// One block = one 32 x 32 tile (out-channels x in-channels) of one tap: the forward image is written row by row, the data-gradient
// image is the transposed tile (through shared memory), so that reads of the weights and writes of BOTH images are coalesced.
__global__ void __launch_bounds__(256) conv_pack_batch_kernel(const dvd_pack_item* __restrict__ items, int n_items, int want_bwd) {
  DVD_PDL_ENTER();
  __shared__ float tile[32][33];
  int lo = 0, hi = n_items - 1;
  while (lo < hi) {                       // last item whose first block is <= blockIdx.x
    const int mid = (lo + hi + 1) >> 1;
    if (items[mid].blk0 <= (long)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const dvd_pack_item it = items[lo];
  const int Cout = it.Cout, Cin = it.Cin, k = it.ksize, kblock = it.kblock;
  const int cpg = Cin / it.groups, opg = Cout / it.groups;
  const int cols = kblock ? kblock : Cin;                 // columns of a forward-image row
  const int nct = cols / 32, nrt = Cout / 32;
  const int tt = (int)((long)blockIdx.x - it.blk0);
  const int t = tt / (nrt * nct), rem = tt - t * (nrt * nct);
  const int co0 = (rem / nct) * 32, c0 = (rem % nct) * 32;
  const int base = kblock ? (co0 / kblock) * kblock : 0;  // first channel of the block-diagonal block (grouped)
  const int ky = t / k, kx = t - ky * k;
  const long tap = (long)ky * it.s_ky + (long)kx * it.s_kx;
  const int lane = threadIdx.x & 31, wy = threadIdx.x >> 5;
  float* bwd = want_bwd ? it.w_bwd : nullptr;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = wy * 4 + i, co = co0 + row, ci = base + c0 + lane;
    float v = 0.f;
    if (co / opg == ci / cpg) v = it.weight[co * it.s_co + (ci % cpg) * it.s_ci + tap];
    if (it.w_fwd) it.w_fwd[((long)t * Cout + co) * cols + c0 + lane] = round_tf32(v);
    if (bwd) tile[row][lane] = it.bn_gamma ? v * (it.bn_gamma[co] * rsqrtf(it.bn_var[co] + it.bn_eps)) : v;   // same association as conv_pack_kernel
  }
  if (!bwd) return;
  __syncthreads();
  const int cols_b = kblock ? kblock : Cout;              // columns of a data-gradient-image row
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = wy * 4 + i, ci = base + c0 + row;     // row of the transposed tile = in-channel
    bwd[((long)t * Cin + ci) * cols_b + (co0 - base) + lane] = round_tf32(tile[lane][row]);
  }
}

// =====================================================================================================================
// Weight gradient:  D[m][n] += sum over pixels  Mop[px (+off), m] * Nop[px (+off), n]
// normally Mop = gy (out-channels), Nop = x shifted by the tap and sampled with the convolution stride; `swap` exchanges
// the roles (needs 128 | M-channels). GEMM with K = pixels on TF32 wgmma. Both operands arrive channel-contiguous (MN-major)
// as 32-pixel TMA boxes {32 ch, TW, TH, 1} in the SWIZZLE_128B image ([32 px][128 B], 16-byte chunk c of pixel row p stored
// at chunk c ^ (p & 7)), and TF32 wgmma reads only K-major shared-memory operands, so:
//   * M (the CTA's 128 channels, 64 rows per MMA warpgroup) is the register operand (wgmma RS): the m64k8 A fragments are
//     gathered from the stage with scalar loads;
//   * N (NT <= 256 channels) is transposed by the MMA warps into a K-major SWIZZLE_128B image [NT rows][32 px], one 4 px x 4 ch
//     micro-tile per thread and step (16-byte loads and stores). The image and the A fragments are double-buffered: the
//     transpose of stage k + 1 runs while the wgmma of stage k is in flight.
// Inside every 8-pixel group both operands use the K order  k-index kappa <-> pixel 2 (kappa % 4) + kappa / 4  (a sum over
// pixels does not care about their order). An A-fragment load then reads pixels 2 tq (+1) of one parity, and the chunk swizzle
// (p & 7) spreads the 32 lanes over all 32 banks; the micro-tile assignment below keeps the transpose conflict-free as well.
// Split-K over pixel tiles across CTAs; partial sums leave through fp32 reductions into the caller's gradient buffer (any
// strides). Extras in the epilogue, all on the M rows (colsum any mode, the BatchNorm terms swap = 0 only):
//   * eval-BatchNorm scale: dW[co] = sc[co] * sum gm X  (gm = the un-scaled masked gradient the data gradient also consumes)
//   * dgamma[co] += rstd[co] * <W[co], sum gm X>        (d/dgamma of BN(conv(x)) without touching any activation)
//   * colsum[m] += sum over pixels of the M operand, summed from the A fragments (CTAs of the first tap and N tile)
//   * grouped convolutions: only diagonal blocks are computed and only in-group entries leave. When the group size divides 64
//     (G64), each warpgroup computes its own 64 x 64 diagonal block; otherwise both compute their half of the 128 x 128 block.
constexpr int kWgStages = 3;
constexpr int kWgPx = 32;                         // pixels (K) per stage
constexpr int kWgBox = kWgPx * 128;               // bytes of one {32 ch, 32 px} box
constexpr int kWgStageBytes = (4 + 8) * kWgBox;   // M: 128 channels, N: up to 256 channels
constexpr int kWgImgBytes = 256 * 128;            // K-major N image: up to 256 rows of 32 pixels
constexpr int kWgOffImg = kWgStages * kWgStageBytes;
constexpr int kWgOffBar = kWgOffImg + 2 * kWgImgBytes;
constexpr size_t kWgSmem = (size_t)kWgOffBar + 256;
constexpr int kWgThreads = 384;                   // TMA producer warpgroup, two MMA warpgroups

struct WgradParams {
  float* dw;
  const float* w;                  // parameter tensor (same strides as dw), only read for dgamma
  long s_m, s_n, s_ky, s_kx;       // element strides of the M / N channel index and of the kernel taps
  int N, OH, OW;                   // pixel grid of gy
  int Mch, Nch;                    // channel counts of the two operands
  int ntaps, ksize, stride, swap;
  int TW, TH, tiles_w, tiles_h;    // 32-pixel tiles
  int ksplit;
  int cpg;                         // > 0: grouped (diagonal blocks of 128 channels)
  const float* gamma;              // eval BatchNorm of the out-channels (or null)
  const float* var;
  float eps;
  float* dgamma;
  float* colsum;                   // [Mch] += sum over pixels of the M operand (conv-bias / BatchNorm-beta gradient), or null
  const float* mean;               // with colsum and dgamma: dgamma[m] -= mean[m] * rstd[m] * colsum[m]
  signed char dy[DVD_CONV_MAX_TAPS], dx[DVD_CONV_MAX_TAPS];
  unsigned char wt[DVD_CONV_MAX_TAPS];
};

template <int NT, bool G64>
__global__ void __launch_bounds__(kWgThreads, 1) conv_wgrad_kernel(const __grid_constant__ CUtensorMap mapM,
                                                                  const __grid_constant__ CUtensorMap mapN,
                                                                  const __grid_constant__ WgradParams P) {
  constexpr int WN = G64 ? 64 : NT;               // accumulator columns of one warpgroup
  constexpr int kUnits = NT / 32 * 64;            // transpose micro-tiles of one stage's N operand
  constexpr int kUnitSteps = (kUnits + 255) / 256;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kWgOffBar);
  uint64_t* full = bars;            // [kWgStages]
  uint64_t* empty = bars + 8;       // [kWgStages]: one arrival per MMA warp
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();   // swizzled stages and images need 1024-byte alignment
  if (threadIdx.x == 0) {
    for (int i = 0; i < kWgStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    fence_mbar_init();
  }
  __syncthreads();
  DVD_PDL_ENTER();

  // this CTA: output tile (tap, 128 M-channels, NT N-channels) and a contiguous range of pixel tiles.
  // blockIdx.x = (tap, M block, N tile) * ksplit + part
  const int out_grp = blockIdx.x / P.ksplit, part = blockIdx.x - out_grp * P.ksplit;
  const int n_m = P.Mch / 128, n_n = P.cpg ? 1 : P.Nch / NT;
  const int t = out_grp / (n_m * n_n);
  const int rem = out_grp - t * (n_m * n_n);
  const int m0 = (rem / n_n) * 128;
  const int n0 = P.cpg ? m0 : (rem % n_n) * NT;
  const int dy = P.dy[t], dx = P.dx[t];
  // the CTAs of the first tap and first N tile also reduce their M operand over the pixels
  const bool do_colsum = P.colsum != nullptr && t == 0 && (P.cpg || rem % n_n == 0);
  const int px_tiles = P.N * P.tiles_h * P.tiles_w;
  const int per = (px_tiles + P.ksplit - 1) / P.ksplit;
  const int kt0 = part * per, kt1 = min(px_tiles, kt0 + per);

  if (wg == 0) {
    setmaxnreg_dec<40>();
    // ===== TMA producer =====
    if (threadIdx.x == 0) {
      const uint32_t stage_tx = (uint32_t)(4 + NT / 32) * kWgBox;
      uint32_t it = 0;
      for (int kt = kt0; kt < kt1; ++kt, ++it) {
        const uint32_t s = it % kWgStages, ph = (it / kWgStages) & 1u;
        const int img = kt / (P.tiles_h * P.tiles_w), r = kt - img * (P.tiles_h * P.tiles_w);
        const int h0 = (r / P.tiles_w) * P.TH, w0 = (r % P.tiles_w) * P.TW;
        // gy is sampled on the plain pixel grid, x at stride * pixel + tap offset
        const int gw = w0, gh = h0, xw = w0 * P.stride + dx, xh = h0 * P.stride + dy;
        const int mw = P.swap ? xw : gw, mh = P.swap ? xh : gh, nw = P.swap ? gw : xw, nh = P.swap ? gh : xh;
        uint8_t* st = smem + (size_t)s * kWgStageBytes;
        mbar_wait(&empty[s], ph ^ 1u);
        mbar_arrive_expect_tx(&full[s], stage_tx);
        for (int j = 0; j < 4; ++j) tma_load_4d(st + j * kWgBox, &mapM, m0 + 32 * j, mw, mh, img, &full[s]);
        for (int j = 0; j < NT / 32; ++j) tma_load_4d(st + (4 + j) * kWgBox, &mapN, n0 + 32 * j, nw, nh, img, &full[s]);
      }
    }
    return;
  }
  setmaxnreg_inc<232>();
  if (kt1 <= kt0) return;
  // ===== MMA warpgroup cw: M rows [64 cw, 64 cw + 64) of the CTA's 128 =====
  const int cw = wg - 1, et = threadIdx.x - 128;
  const int g = lane >> 2, tq = lane & 3;
  const int lrow = cw * 64 + (warp & 3) * 16 + g;     // this thread's fragment rows: lrow, lrow + 8
  // A fragment of pixel group kk: a0 = (row lrow, pixel 8 kk + 2 tq), a1 = (lrow + 8, same pixel), a2 / a3 = pixel 8 kk + 2 tq + 1
  uint32_t a_off[2][2];                               // [row + 8?][pixel parity], byte offsets in the stage's M part
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const uint32_t ch = (uint32_t)(lrow + 8 * h), px = (uint32_t)(2 * tq + e);
      a_off[h][e] = (ch >> 5) * kWgBox + px * 128u + ((((ch & 31u) >> 2) ^ px) << 4) + (ch & 3u) * 4u;
    }
  // transpose micro-tiles: unit u = (32-channel box j, l = 8 hi + tt) covers channels 32 j + 4 tt .. + 3 and K chunk
  // q = (tt >> 1) ^ hi, i.e. pixels 8 (q >> 1) + 2 e + (q & 1), e = 0..3. Within every 8 lanes both the loads (pixel rows,
  // chunk tt ^ (p & 7)) and the stores (channel rows, chunk q ^ (n & 7)) hit 8 different 16-byte bank groups.
  uint32_t u_src[kUnitSteps], u_dst[kUnitSteps];
#pragma unroll
  for (int r = 0; r < kUnitSteps; ++r) {
    const uint32_t u = (uint32_t)(et + 256 * r), j = u >> 6, tt = u & 7u, hi = (u >> 3) & 7u, q = (tt >> 1) ^ hi;
    u_src[r] = 4u * kWgBox + j * kWgBox + (8u * (q >> 1) + (q & 1u)) * 128u;
    u_dst[r] = (32u * j + 4u * tt) * 128u;
  }
  const uint32_t u_tt = (uint32_t)et & 7u, u_q = (u_tt >> 1) ^ (((uint32_t)et >> 3) & 7u);
  const uint32_t img0 = smem_u32(smem + kWgOffImg) + (G64 ? (uint32_t)cw * 64u * 128u : 0u);
  float acc[WN / 2];
#pragma unroll
  for (int i = 0; i < WN / 2; ++i) acc[i] = 0.f;
  uint32_t a[2][4][4];
  float cs[2] = {0.f, 0.f};

  // one stage into buffer B (fragments a[B], image B); on return its wgmma group is in flight
  auto stage = [&](auto buf, uint32_t it) {
    constexpr int B = decltype(buf)::value;
    const uint32_t s = it % kWgStages, ph = (it / kWgStages) & 1u;
    mbar_wait(&full[s], ph);
    const uint8_t* st = smem + (size_t)s * kWgStageBytes;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      a[B][kk][0] = *reinterpret_cast<const uint32_t*>(st + a_off[0][0] + kk * 1024);
      a[B][kk][1] = *reinterpret_cast<const uint32_t*>(st + a_off[1][0] + kk * 1024);
      a[B][kk][2] = *reinterpret_cast<const uint32_t*>(st + a_off[0][1] + kk * 1024);
      a[B][kk][3] = *reinterpret_cast<const uint32_t*>(st + a_off[1][1] + kk * 1024);
    }
    if (do_colsum) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        cs[0] += __uint_as_float(a[B][kk][0]) + __uint_as_float(a[B][kk][2]);
        cs[1] += __uint_as_float(a[B][kk][1]) + __uint_as_float(a[B][kk][3]);
      }
    }
    uint8_t* img = smem + kWgOffImg + B * kWgImgBytes;
#pragma unroll
    for (int r = 0; r < kUnitSteps; ++r) {
      if (kUnits % 256 != 0 && et + 256 * r >= kUnits) continue;
      float4 v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const uint32_t p = 2u * e + (u_q & 1u);              // pixel row & 7
        v[e] = *reinterpret_cast<const float4*>(st + u_src[r] + 256u * e + ((u_tt ^ p) << 4));
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t n7 = (4u * u_tt + i) & 7u;            // channel row & 7
        const float4 w = i == 0 ? make_float4(v[0].x, v[1].x, v[2].x, v[3].x)
                       : i == 1 ? make_float4(v[0].y, v[1].y, v[2].y, v[3].y)
                       : i == 2 ? make_float4(v[0].z, v[1].z, v[2].z, v[3].z)
                                : make_float4(v[0].w, v[1].w, v[2].w, v[3].w);
        *reinterpret_cast<float4*>(img + u_dst[r] + 128u * i + ((u_q ^ n7) << 4)) = w;
      }
    }
    fence_proxy_async_smem();                                // the image is read by wgmma (async proxy)
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);                   // stage fully consumed: fragments in registers, N in the image
    wgmma_wait<0>();                                         // the previous stage's wgmma (other buffer) is done ...
    named_sync(1, 256);                                      // ... in both warpgroups, and this image is complete
    wgmma_fence();
    const uint32_t ib = img0 + B * kWgImgBytes;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_tf32_rs<WN>(acc, a[B][kk], make_sdesc_k_sw128(ib + kk * 32), 1u);
    wgmma_commit();
  };
  const uint32_t n_it = (uint32_t)(kt1 - kt0);
  uint32_t it = 0;
  for (; it + 2 <= n_it; it += 2) {
    stage(std::integral_constant<int, 0>{}, it);
    stage(std::integral_constant<int, 1>{}, it + 1);
  }
  if (it < n_it) stage(std::integral_constant<int, 0>{}, it);
  wgmma_wait<0>();
  fence_regs(acc);

  // epilogue: acc[4 j + 2 h + e] holds row lrow + 8 h, column noff + 8 j + 2 tq + e of the CTA's (128 x NT) tile
  const int noff = G64 ? cw * 64 : 0;
  const int wt = P.wt[t];
  const long tap_off = (long)(wt / P.ksize) * P.s_ky + (long)(wt % P.ksize) * P.s_kx;
  if (do_colsum) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      cs[h] += __shfl_xor_sync(0xffffffffu, cs[h], 1);
      cs[h] += __shfl_xor_sync(0xffffffffu, cs[h], 2);
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int lm = lrow + 8 * h, m = m0 + lm;
    float* dst = P.dw + (long)m * P.s_m + tap_off;
    const float* wrow = P.w ? P.w + (long)m * P.s_m + tap_off : nullptr;
    float sc = 1.f, rstd = 0.f;
    if (P.gamma) {
      rstd = rsqrtf(__ldg(P.var + m) + P.eps);
      sc = __ldg(P.gamma + m) * rstd;
    }
    float dot = 0.f;
#pragma unroll
    for (int j = 0; j < WN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int ln = noff + j * 8 + 2 * tq + e;
        if (P.cpg && ln / P.cpg != lm / P.cpg) continue;        // grouped: in-group entries of the diagonal block only
        const long o = (long)(P.cpg ? ln % P.cpg : n0 + ln) * P.s_n;
        const float v = acc[4 * j + 2 * h + e];
        if (wrow) dot = fmaf(v, __ldg(wrow + o), dot);
        atomicAdd(dst + o, v * sc);
      }
    }
    if (P.dgamma) {
      dot += __shfl_xor_sync(0xffffffffu, dot, 1);
      dot += __shfl_xor_sync(0xffffffffu, dot, 2);
    }
    if (tq == 0) {
      if (do_colsum) {
        atomicAdd(P.colsum + m, cs[h]);
        if (P.dgamma && P.mean) dot = fmaf(-__ldg(P.mean + m), cs[h], dot);   // d gamma = rstd * (<W, dW> - mean * sum gm)
      }
      if (P.dgamma) atomicAdd(P.dgamma + m, dot * rstd);
    }
  }
}

// ---- host ----------------------------------------------------------------------------------------------------------
PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }();
  return fn;
}

int make_map(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
             const cuuint32_t* box, const cuuint32_t* elem_strides, CUtensorMapSwizzle swizzle) {
  auto fn = encode_fn();
  DVD_ARG_CHECK(fn != nullptr, "cuTensorMapEncodeTiled is not available from this driver");
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides_bytes, box,
                  elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DVD_ARG_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (CUresult %d)", (int)r);
  return 0;
}

// 4-D map of an NHWC tensor [N][H][W][C]; a box of {32 ch, bw, bh, 1} ELEMENTS sampled every `es` pixels
int make_nhwc_map(CUtensorMap* m, const void* ptr, int N, int H, int W, int C, int bw, int bh, int es, CUtensorMapSwizzle swizzle) {
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[3] = {(cuuint64_t)C * 4, (cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 4};
  const cuuint32_t box[4] = {32, (cuuint32_t)(bw * es), (cuuint32_t)(bh * es), 1};
  const cuuint32_t estr[4] = {1, (cuuint32_t)es, (cuuint32_t)es, 1};
  DVD_ARG_CHECK(bw * es <= 256 && bh * es <= 256, "TMA box too large (%d x %d at element stride %d)", bw, bh, es);
  return make_map(m, ptr, 4, dims, strides, box, estr, swizzle);
}

// TH x TW = npx (power of two) tile over an H x W grid with the least padding
void pick_tile(int H, int W, int npx, int max_tw, int* TW, int* TH) {
  long best = -1;
  for (int tw = npx < max_tw ? npx : max_tw; tw >= 8; tw >>= 1) {
    const int th = npx / tw;
    const long padded = (long)((W + tw - 1) / tw * tw) * ((H + th - 1) / th * th);
    if (best < 0 || padded < best) { best = padded; *TW = tw; *TH = th; }
  }
}

int per_device_attr(const void* func, size_t smem_bytes, bool (&done)[16]) {
  int dev = 0;
  DVD_CUDA_CALL(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 16) dev = 0;
  if (!done[dev]) {
    DVD_CUDA_CALL(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    done[dev] = true;
  }
  return 0;
}

// how many clusters of `csize` CTAs of this kernel can be resident at once (cached per device and size)
template <typename K>
int max_clusters(K kernel, int threads, size_t smem_bytes, int csize) {
  static int cache[16][5] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) dev = 0;
  if (cache[dev][csize] > 0) return cache[dev][csize];
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(num_sms() / csize * csize));
  cfg.blockDim = dim3((unsigned)threads);
  cfg.dynamicSmemBytes = smem_bytes;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)csize;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess || n < 1) n = num_sms() / csize;
  cache[dev][csize] = n;
  return n;
}

template <int NT>
int launch_conv(const CUtensorMap& mapA, const CUtensorMap& mapW, const ConvParams& P, int grid, cudaStream_t st) {
  static bool attr_done[16] = {};
  if (int e = per_device_attr((const void*)conv2d_tc_kernel<NT>, kSmem, attr_done)) return e;
  DVD_CUDA_CALL(dvd::launch(conv2d_tc_kernel<NT>, grid, kThreads, kSmem, st, mapA, mapW, P));
  DVD_CUDA_LAUNCH_CHECK("conv2d_tc_kernel");
  return 0;
}

template <int NT, bool G64>
int launch_wgrad(const CUtensorMap& mapM, const CUtensorMap& mapN, WgradParams P, int out_tiles, int px_tiles, cudaStream_t st) {
  static bool attr_done[16] = {};
  if (int e = per_device_attr((const void*)conv_wgrad_kernel<NT, G64>, kWgSmem, attr_done)) return e;
  // split-K so that all CTAs are resident in ONE wave (a second, nearly empty wave would double the time)
  const int resident = max_clusters(conv_wgrad_kernel<NT, G64>, kWgThreads, kWgSmem, 1);
  int ksplit = resident / out_tiles;
  if (ksplit > px_tiles) ksplit = px_tiles;
  if (ksplit < 1) ksplit = 1;
  P.ksplit = ksplit;
  DVD_CUDA_CALL(dvd::launch(conv_wgrad_kernel<NT, G64>, out_tiles * ksplit, kWgThreads, kWgSmem, st, mapM, mapN, P));
  DVD_CUDA_LAUNCH_CHECK("conv_wgrad_kernel");
  return 0;
}

}  // namespace
}  // namespace dvd

using namespace dvd;

/* first (tile-major) K-step of every cluster's range under the stream-K schedule: out[0..n_clusters], out[n_clusters] = total
 * (host restatement of the kernel's own rule, for tests of the schedule's invariants) */
extern "C" int dvd_conv2d_streamk_bounds(int ntiles, int ksteps, int n_clusters, long* out) {
  DVD_ARG_CHECK(out && ntiles >= 1 && ksteps >= 1 && n_clusters >= 1 && (long)ntiles * ksteps >= n_clusters, "bad schedule shape");
  for (int c = 0; c <= n_clusters; ++c) out[c] = SegIter::bound(c, n_clusters, (long)ntiles * ksteps, ksteps);
  return 0;
}

extern "C" size_t dvd_conv2d_workspace_bytes(void) {
  // one partial tile [128][256] fp32 and one flag per resident CTA
  return (size_t)kWsFlagWords * sizeof(int) + (size_t)num_sms() * 128 * kMaxNT * sizeof(float);
}

extern "C" int dvd_conv2d_nhwc(const dvd_conv_desc* desc, const float* x, const float* w_img, const float* bias, const float* bn_gamma,
                               const float* bn_beta, const float* bn_mean, const float* bn_var, const float* res, const float* res2,
                               const float* mask, float* y, void* stream) {
  return dvd_conv2d_nhwc_ws(desc, x, w_img, bias, bn_gamma, bn_beta, bn_mean, bn_var, res, res2, mask, y, nullptr, 0, stream);
}

extern "C" int dvd_conv2d_nhwc_ws(const dvd_conv_desc* desc, const float* x, const float* w_img, const float* bias, const float* bn_gamma,
                                  const float* bn_beta, const float* bn_mean, const float* bn_var, const float* res, const float* res2,
                                  const float* mask, float* y, void* workspace, size_t workspace_bytes, void* stream) {
  DVD_ARG_CHECK(desc && x && w_img && y, "null pointer");
  ConvParams P{};
  P.d = *desc;
  dvd_conv_desc& d = P.d;
  DVD_ARG_CHECK(d.N >= 1 && d.H >= 1 && d.W >= 1 && d.OH >= 1 && d.OW >= 1, "bad shape N=%d H=%d W=%d OH=%d OW=%d", d.N, d.H, d.W, d.OH, d.OW);
  DVD_ARG_CHECK(d.stride == 1 || d.stride == 2, "stride must be 1 or 2");
  DVD_ARG_CHECK(d.ntaps >= 1 && d.ntaps <= DVD_CONV_MAX_TAPS, "ntaps out of range");
  DVD_ARG_CHECK(d.kblock == 0 || (d.kblock % 32 == 0 && d.kblock <= kMaxNT && d.Cout % d.kblock == 0 && d.Cin % d.kblock == 0),
                "bad kblock %d (Cin=%d Cout=%d)", d.kblock, d.Cin, d.Cout);
  if (d.Cin % 32 != 0 || d.Cout % 16 != 0) {
    set_error("dvd_conv2d_nhwc: needs Cin %% 32 == 0 and Cout %% 16 == 0 (Cin=%d Cout=%d)", d.Cin, d.Cout);
    return -2;
  }
  DVD_ARG_CHECK(aligned16(x) && aligned16(w_img) && aligned16(y) && (!res || aligned16(res)) && (!res2 || aligned16(res2)) &&
                    (!mask || aligned16(mask)),
                "tensors must be 16-byte aligned");
  DVD_ARG_CHECK((bn_gamma != nullptr) == (bn_beta != nullptr) && (bn_gamma != nullptr) == (bn_mean != nullptr) &&
                    (bn_gamma != nullptr) == (bn_var != nullptr),
                "BatchNorm needs all of gamma, beta, mean, var (or none)");
  P.bias = bias; P.gamma = bn_gamma; P.beta = bn_beta; P.mean = bn_mean; P.var = bn_var;
  P.res = res; P.res2 = res2; P.mask = mask; P.y = y;
  P.kchunks = (d.kblock ? d.kblock : d.Cin) / 32;
  const bool pointwise = d.ntaps == 1 && d.dy[0] == 0 && d.dx[0] == 0 && d.stride == 1 && d.oy_mul == 1 && d.ox_mul == 1 &&
                         d.oy_add == 0 && d.ox_add == 0 && d.YH == d.OH && d.YW == d.OW && d.H == d.OH && d.W == d.OW;
  int inN = d.N, inH = d.H, inW = d.W;
  if (pointwise) {
    // a 1x1 stride-1 convolution is a plain GEMM over all N*H*W pixels: one "image" of P x 1
    const long Pn = (long)d.N * d.H * d.W;
    DVD_ARG_CHECK(Pn < (1L << 31), "too many pixels");
    inN = 1; inH = 1; inW = (int)Pn;
    d.N = 1; d.OH = 1; d.OW = (int)Pn; d.YH = 1; d.YW = (int)Pn;
    P.TW = 128; P.TH = 1;
  } else {
    pick_tile(d.OH, d.OW, 128, 128, &P.TW, &P.TH);   // the TMA box spans TW * stride <= 256 input pixels
  }
  P.tiles_w = (d.OW + P.TW - 1) / P.TW;
  P.tiles_h = (d.OH + P.TH - 1) / P.TH;
  // channel-tile width: the instantiated wgmma widths are 16 and the multiples of 32 up to 256; a width above Cout leaves a
  // ragged tile (zero-filled weight rows, skipped by the epilogue)
  auto fit = [](int c) { return c <= 16 ? 16 : (c + 31) / 32 * 32; };
  const long m_tiles_h = (long)d.N * P.tiles_w * P.tiles_h;
  const long full = num_sms();                          // one CTA per SM (the stage ring fills the shared memory)
  if (d.kblock) {
    P.NT = d.kblock;
  } else {
    const int nt_max = fit(d.Cout >= kMaxNT ? kMaxNT : d.Cout);
    P.NT = nt_max;
    // Whole tiles come in waves: a narrower tile that fills the last wave wins when  rounds(NT) * t(NT)  is smaller,
    // t(NT) = 0.47 + 0.53 * NT / 256 the relative cost of a K-step of an NT-wide tile (a heuristic carried over from earlier
    // tuning, not re-fitted on the H100). Layers that take the stream-K schedule
    // (few tiles, long K loop) keep the widest tile: their K-steps are spread over all SMs whatever the tile count.
    const char* ev = getenv("DVD_CONV_NT");
    if (ev && atoi(ev) >= 32 && atoi(ev) <= kMaxNT && atoi(ev) % 32 == 0 && d.Cout >= 128) {
      P.NT = atoi(ev);
    } else if (d.Cout >= 128 && d.Cout % 32 == 0 && !(ev && atoi(ev) == 0)) {
      int nt_min = m_tiles_h * ((d.Cout + nt_max - 1) / nt_max) < full ? 64 : 128;
      const long ksteps = (long)d.ntaps * (d.Cin / 32), tiles0 = m_tiles_h * ((d.Cout + nt_max - 1) / nt_max);
      const long waves0 = (tiles0 + full - 1) / full, total0 = tiles0 * ksteps, mu = ksteps / 4 > 8 ? ksteps / 4 : 8;
      long nc0 = total0 / mu;
      if (nc0 > full) nc0 = full;
      const char* evs = getenv("DVD_CONV_STREAMK");
      if (workspace && ksteps >= 8 && !(evs && atoi(evs) == 0) && nc0 >= 1 && waves0 * ksteps - (total0 + nc0 - 1) / nc0 >= 64)
        nt_min = nt_max;
      double best = 1e30;
      for (int nt = nt_max; nt >= nt_min; nt -= 32) {
        const long tiles = m_tiles_h * ((d.Cout + nt - 1) / nt);
        const double cost = (double)((tiles + full - 1) / full) * (0.47 + 0.53 * nt / 256.0);
        if (cost < best * 0.97) { best = cost; P.NT = nt; }      // a narrower tile must win by 3 %
      }
    }
  }
  if (d.kblock && (P.NT != fit(P.NT) || d.Cout % P.NT != 0)) {
    set_error("dvd_conv2d_nhwc: kblock %d is not an instantiated tile width", d.kblock);
    return -2;
  }
  CUtensorMap mapA, mapW;
  if (int e = make_nhwc_map(&mapA, x, inN, inH, inW, d.Cin, P.TW, P.TH, d.stride, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  {
    int max_wt = 0;
    for (int t = 0; t < d.ntaps; ++t) max_wt = d.wt[t] > max_wt ? d.wt[t] : max_wt;
    const int Kw = d.kblock ? d.kblock : d.Cin;
    const cuuint64_t dims[3] = {(cuuint64_t)Kw, (cuuint64_t)d.Cout, (cuuint64_t)(max_wt + 1)};
    const cuuint64_t strides[2] = {(cuuint64_t)Kw * 4, (cuuint64_t)d.Cout * Kw * 4};
    const cuuint32_t box[3] = {32, (cuuint32_t)P.NT, 1};
    const cuuint32_t ones[3] = {1, 1, 1};
    if (int e = make_map(&mapW, w_img, 3, dims, strides, box, ones, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  }
  const long ctiles = m_tiles_h * ((d.Cout + P.NT - 1) / P.NT);
  long nctas = ctiles < full ? ctiles : full;
  // stream-K when whole tiles would leave a large part of the machine idle in the last (or only) wave: cut the (tile, K-step)
  // list into equal contiguous ranges instead. Needs the caller's exchange area (zeroed once; the kernel leaves it zeroed where
  // it matters: the flags). A range is at least max(8, ksteps / 4) K-steps long, so a tile is shared by at most ~4 CTAs.
  P.sk = 0;
  P.ws = nullptr;
  {
    const long ksteps = (long)d.ntaps * P.kchunks, total = ctiles * ksteps;
    const long waves = (ctiles + full - 1) / full;
    const double eff = (double)ctiles / (double)(waves * full);
    const char* ev = getenv("DVD_CONV_STREAMK");
    const bool allowed = !(ev && atoi(ev) == 0);
    if (allowed && workspace && ksteps >= 8 && eff < 0.88) {
      const long min_units = ksteps / 4 > 8 ? ksteps / 4 : 8;
      long nc = total / min_units;
      if (nc > full) nc = full;
      const size_t need = (size_t)kWsFlagWords * sizeof(int) + (size_t)nc * 128 * (size_t)P.NT * sizeof(float);
      // the exchange (partial tiles through L2, a short serial tail in the finishing CTA) is charged as 64 K-steps (a threshold
      // carried over from earlier tuning, not re-fitted on the H100)
      const long dp_steps = waves * ksteps, sk_steps = (total + nc - 1) / nc;
      if ((nc > nctas || (nc == nctas && waves > 1)) && dp_steps - sk_steps >= 64) {
        DVD_ARG_CHECK(aligned16(workspace), "workspace must be 16-byte aligned");
        if (need <= workspace_bytes && nc <= kWsFlagWords) {
          P.sk = 1;
          P.ws = static_cast<float*>(workspace);
          nctas = nc;
        }
      }
    }
  }
  switch (P.NT) {
    case 16: return launch_conv<16>(mapA, mapW, P, (int)nctas, (cudaStream_t)stream);
    case 32: return launch_conv<32>(mapA, mapW, P, (int)nctas, (cudaStream_t)stream);
    case 64: return launch_conv<64>(mapA, mapW, P, (int)nctas, (cudaStream_t)stream);
    case 96: return launch_conv<96>(mapA, mapW, P, (int)nctas, (cudaStream_t)stream);
    case 128: return launch_conv<128>(mapA, mapW, P, (int)nctas, (cudaStream_t)stream);
    case 160: return launch_conv<160>(mapA, mapW, P, (int)nctas, (cudaStream_t)stream);
    case 192: return launch_conv<192>(mapA, mapW, P, (int)nctas, (cudaStream_t)stream);
    case 224: return launch_conv<224>(mapA, mapW, P, (int)nctas, (cudaStream_t)stream);
    case 256: return launch_conv<256>(mapA, mapW, P, (int)nctas, (cudaStream_t)stream);
    default:
      set_error("dvd_conv2d_nhwc: no kernel for a %d-channel tile", P.NT);
      return -2;
  }
}

extern "C" int dvd_conv2d_pack(const float* weight, long stride_co, long stride_ci, long stride_ky, long stride_kx, float* w_fwd,
                               float* w_bwd, int Cout, int Cin, int ksize, int groups, int kblock, const float* bn_gamma,
                               const float* bn_var, float bn_eps, void* stream) {
  DVD_ARG_CHECK(weight && (w_fwd || w_bwd), "null pointer");
  DVD_ARG_CHECK(Cout >= 1 && Cin >= 1 && ksize >= 1 && ksize <= 11 && groups >= 1 && Cin % groups == 0 && Cout % groups == 0,
                "bad weight shape");
  DVD_ARG_CHECK((groups == 1) == (kblock == 0), "kblock must be set exactly for grouped convolutions");
  const int cpg = Cin / groups;
  if (kblock) DVD_ARG_CHECK(Cin == Cout && kblock % cpg == 0 && Cin % kblock == 0, "grouped: needs Cin == Cout and cpg | kblock | Cin");
  DVD_ARG_CHECK((bn_gamma != nullptr) == (bn_var != nullptr), "BatchNorm scale needs gamma and var");
  const long n = (long)ksize * ksize * (Cout > Cin ? Cout : Cin) * (kblock ? kblock : (Cout > Cin ? Cin : Cout));
  int blocks = (int)((n + 255) / 256);
  if (blocks > 8 * num_sms()) blocks = 8 * num_sms();
  dvd::launch(conv_pack_kernel, blocks, 256, 0, (cudaStream_t)stream, weight, stride_co, stride_ci, stride_ky, stride_kx, w_fwd, w_bwd, Cout, Cin,
                                                           ksize, cpg, kblock, bn_gamma, bn_var, bn_eps);
  DVD_CUDA_LAUNCH_CHECK("conv_pack_kernel");
  return 0;
}

extern "C" long dvd_conv2d_pack_blocks(int Cout, int Cin, int ksize, int groups, int kblock) {
  if (Cout < 32 || Cin < 32 || ksize < 1 || groups < 1 || Cout % 32 || Cin % 32 || (kblock && kblock % 32)) return -1;
  return (long)ksize * ksize * (Cout / 32) * ((kblock ? kblock : Cin) / 32);      // one block per 32 x 32 tile and tap
}

extern "C" int dvd_conv2d_pack_batch(const dvd_pack_item* items_dev, int n_items, long total_blocks, int want_bwd, void* stream) {
  DVD_ARG_CHECK(items_dev && n_items >= 1 && total_blocks >= 1 && total_blocks < (1L << 31), "bad pack table");
  dvd::launch(conv_pack_batch_kernel, (unsigned)total_blocks, 256, 0, (cudaStream_t)stream, items_dev, n_items, want_bwd);
  DVD_CUDA_LAUNCH_CHECK("conv_pack_batch_kernel");
  return 0;
}

extern "C" int dvd_conv2d_wgrad(const dvd_conv_desc* desc, const float* x, const float* gy, float* dweight, const float* weight,
                                long stride_co, long stride_ci, long stride_ky, long stride_kx, int ksize, int groups,
                                const float* bn_gamma, const float* bn_var, float* dgamma, float* colsum, const float* bn_mean,
                                void* stream) {
  DVD_ARG_CHECK(desc && x && gy && dweight, "null pointer");
  const dvd_conv_desc& d = *desc;
  DVD_ARG_CHECK(d.N >= 1 && d.H >= 1 && d.W >= 1 && d.OH >= 1 && d.OW >= 1, "bad shape");
  DVD_ARG_CHECK(d.stride == 1 || d.stride == 2, "stride must be 1 or 2");
  DVD_ARG_CHECK(d.ntaps >= 1 && d.ntaps <= DVD_CONV_MAX_TAPS, "ntaps out of range");
  DVD_ARG_CHECK(aligned16(x) && aligned16(gy), "tensors must be 16-byte aligned");
  DVD_ARG_CHECK((bn_gamma != nullptr) == (bn_var != nullptr) && (!dgamma || (bn_gamma && weight)), "BatchNorm extras need gamma, var (and weight for dgamma)");
  WgradParams P{};
  P.dw = dweight; P.w = dgamma ? weight : nullptr;
  P.N = d.N; P.OH = d.OH; P.OW = d.OW; P.ntaps = d.ntaps; P.ksize = ksize; P.stride = d.stride;
  P.gamma = bn_gamma; P.var = bn_var; P.eps = d.bn_eps; P.dgamma = dgamma; P.colsum = colsum; P.mean = bn_mean;
  for (int t = 0; t < d.ntaps; ++t) { P.dy[t] = d.dy[t]; P.dx[t] = d.dx[t]; P.wt[t] = d.wt[t]; }
  const int Cin = d.Cin, Cout = d.Cout;
  int NT;                          // N channels per output tile (multiple of 32)
  if (groups > 1) {
    P.cpg = Cin / groups;
    if (Cin != Cout || Cin % 128 != 0 || 128 % P.cpg != 0) {
      set_error("dvd_conv2d_wgrad: grouped needs Cin == Cout, 128 | C and cpg | 128 (C=%d groups=%d)", Cin, groups);
      return -2;
    }
    P.swap = 0; P.Mch = Cout; P.Nch = Cin; NT = 128;
    P.s_m = stride_co; P.s_n = stride_ci;
  } else if (Cout % 128 == 0 && Cin % 32 == 0 && (Cin <= 256 || Cin % 256 == 0)) {
    P.swap = 0; P.Mch = Cout; P.Nch = Cin; NT = Cin >= 256 ? 256 : Cin;
    P.s_m = stride_co; P.s_n = stride_ci;
  } else if (Cin % 128 == 0 && Cout % 32 == 0 && (Cout <= 256 || Cout % 256 == 0) && !bn_gamma) {
    P.swap = 1; P.Mch = Cin; P.Nch = Cout; NT = Cout >= 256 ? 256 : Cout;
    P.s_m = stride_ci; P.s_n = stride_co;
    DVD_ARG_CHECK(colsum == nullptr, "column sums are not available with swapped operands (Cout %% 128 != 0): use dvd_relu_bwd_colsum");
  } else {
    set_error("dvd_conv2d_wgrad: unsupported channel counts Cin=%d Cout=%d", Cin, Cout);
    return -2;
  }
  P.s_ky = stride_ky; P.s_kx = stride_kx;
  int N = d.N, OH = d.OH, OW = d.OW, H = d.H, W = d.W;
  const bool pointwise = d.ntaps == 1 && d.dy[0] == 0 && d.dx[0] == 0 && d.stride == 1 && d.H == d.OH && d.W == d.OW;
  if (pointwise) {
    const long Pn = (long)N * OH * OW;
    DVD_ARG_CHECK(Pn < (1L << 31), "too many pixels");
    N = 1; OH = 1; OW = (int)Pn; H = 1; W = (int)Pn;
    P.N = 1; P.OH = 1; P.OW = (int)Pn;
    P.TW = kWgPx; P.TH = 1;
  } else {
    pick_tile(OH, OW, kWgPx, kWgPx, &P.TW, &P.TH);
  }
  P.tiles_w = (OW + P.TW - 1) / P.TW;
  P.tiles_h = (OH + P.TH - 1) / P.TH;
  const int out_tiles = d.ntaps * (P.Mch / 128) * (P.cpg ? 1 : P.Nch / NT);
  const int px_tiles = N * P.tiles_h * P.tiles_w;
  CUtensorMap mapG, mapX;
  if (int e = make_nhwc_map(&mapG, gy, N, OH, OW, Cout, P.TW, P.TH, 1, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  if (int e = make_nhwc_map(&mapX, x, N, H, W, Cin, P.TW, P.TH, d.stride, CU_TENSOR_MAP_SWIZZLE_128B)) return e;
  const CUtensorMap& mapM = P.swap ? mapX : mapG;
  const CUtensorMap& mapN = P.swap ? mapG : mapX;
  const cudaStream_t st = (cudaStream_t)stream;
  if (P.cpg && 64 % P.cpg == 0) return launch_wgrad<128, true>(mapM, mapN, P, out_tiles, px_tiles, st);
  switch (NT) {
    case 32: return launch_wgrad<32, false>(mapM, mapN, P, out_tiles, px_tiles, st);
    case 64: return launch_wgrad<64, false>(mapM, mapN, P, out_tiles, px_tiles, st);
    case 96: return launch_wgrad<96, false>(mapM, mapN, P, out_tiles, px_tiles, st);
    case 128: return launch_wgrad<128, false>(mapM, mapN, P, out_tiles, px_tiles, st);
    case 160: return launch_wgrad<160, false>(mapM, mapN, P, out_tiles, px_tiles, st);
    case 192: return launch_wgrad<192, false>(mapM, mapN, P, out_tiles, px_tiles, st);
    case 224: return launch_wgrad<224, false>(mapM, mapN, P, out_tiles, px_tiles, st);
    default: return launch_wgrad<256, false>(mapM, mapN, P, out_tiles, px_tiles, st);
  }
}

/* resident CTAs of the two tensor-core kernels for cluster sizes 1, 2, 4 (diagnostic): out[0..2] forward / data gradient kernel,
 * out[3..5] weight-gradient kernel */
extern "C" int dvd_conv2d_cluster_info(int* out) {
  static bool a1[16] = {}, a2[16] = {};
  if (int e = per_device_attr((const void*)conv2d_tc_kernel<kMaxNT>, kSmem, a1)) return e;
  if (int e = per_device_attr((const void*)conv_wgrad_kernel<256, false>, kWgSmem, a2)) return e;
  const int cs[3] = {1, 2, 4};
  for (int i = 0; i < 3; ++i) {
    out[i] = cs[i] * max_clusters(conv2d_tc_kernel<kMaxNT>, kThreads, kSmem, cs[i]);
    out[3 + i] = cs[i] * max_clusters(conv_wgrad_kernel<256, false>, kWgThreads, kWgSmem, cs[i]);
  }
  return 0;
}
