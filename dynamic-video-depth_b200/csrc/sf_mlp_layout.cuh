// Memory layouts shared by the scene-flow MLP kernels (host + device).
//
// Every GEMM operand — weights, saved activations X_l, back-propagated dY_l — lives in global memory
// as bf16 (hi, lo) planes cut into blocks of [rows x 64] elements stored as the canonical wgmma
// SWIZZLE_128B K-major shared-memory image (tc_common.cuh: sw128_offset). A block is therefore
// loaded with ONE 1-D bulk async copy (no tensor map) and consumed by wgmma.mma directly.
//   weights fwd  (B operand of Y = X W^T):      rows = out channel, K = in channel
//   weights bwd  (B operand of dX = dY W):      rows = in channel,  K = out channel
//   X_l / dY_l   (operands of dW = dY^T X):     MN-major blocks: K = pixel (64 per block), channels
//                contiguous — each pixel's 64-channel group is one 128-byte row, so the epilogue thread
//                that owns the pixel writes whole 16-byte chunks (mn128_offset in tc_common.cuh)
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "../../include/dvd_b200.h"

namespace dvd {

constexpr int kWidth = 256;    // hidden width (reference ctor, smf.py:107)
constexpr int kHidden = 4;     // hidden 256->256 layers
constexpr int kLayers = 6;
constexpr int kTileM = 128;    // pixels per CTA tile (two wgmma M = 64 halves)
constexpr int kChunkK = 64;    // bf16 elements per 128-byte swizzle row

struct MlpLayout {
  int nin, kpad0, k0_chunks;
  long npx, ntiles, nq;        // pixels, 128-px tiles, 64-px chunks (= 2 * ntiles)
  size_t wf_off[kLayers], wf_total;
  size_t wb_off[kLayers], wb_total;
  size_t xs_off[kLayers], mask_off, save_total;  // per eval
  size_t dy_off[kLayers], dy_total;              // per eval
};

__host__ __device__ inline int mlp_nin(const dvd_mlp_cfg& c) {
  int nt = c.time_dependent ? (1 + 2 * c.n_freq_t) : 0;
  return nt + 3 + 6 * c.n_freq_xyz;
}
// (16, 16, time-dependent) and (16, time-independent): the two configurations whose kernels are compiled for their counts.
// Their first layer is padded to a multiple of 16 input channels; every other configuration runs the generic kernels and
// pads it to a multiple of 64, so that its data-gradient MMA width (N = kpad0) takes one of four values.
__host__ __device__ inline bool mlp_specialised(const dvd_mlp_cfg& c) {
  return c.n_freq_xyz == 16 && (!c.time_dependent || c.n_freq_t == 16);
}
__host__ __device__ inline int rows_f(int l) { return l < 5 ? kWidth : 16; }
__host__ __device__ inline int rows_b(const MlpLayout& L, int l) { return l == 0 ? L.kpad0 : kWidth; }
__host__ __device__ inline int nkc_f(const MlpLayout& L, int l) { return l == 0 ? L.k0_chunks : 4; }
__host__ __device__ inline int nkc_b(int l) { return l == 5 ? 1 : 4; }
__host__ __device__ inline int rows_x(const MlpLayout& L, int l) { return l == 0 ? L.kpad0 : kWidth; }
__host__ __device__ inline int rows_dy(int l) { return l == 5 ? 16 : kWidth; }
// Layout of the saved activation / dY blocks (operands of the weight-gradient GEMM, K = 64 pixels per block):
//   true : MN-major without swizzle ("interleave", tc_common.cuh: il_offset) — a warp's 32 pixel-owning threads
//          write 512 contiguous bytes per 16-byte store;
//   false: MN-major SWIZZLE_128B (mn128_offset) — each thread writes 16-byte pieces of its own 128-byte rows.
constexpr bool kActInterleave = false;
// Planes of the SAVED activations X_l / dY_l (the operands of the weight-gradient GEMM only): 1 = the bf16 `hi` plane alone.
// dW = sum over >= 1e5 pixels of dY * X: the round-to-nearest bf16 errors of the two operands (2^-9 relative, zero mean,
// independent from pixel to pixel) average out in that sum - the error of dW is ~1e-3 * sqrt(sum t^2) against |sum t|, i.e.
// ~1e-6 of the largest entry at 384x224 - while the saved bytes, the HBM-bound weight-gradient kernel's traffic and its MMA
// count halve / drop 3x. The forward chain and the data gradient keep the full (hi, lo) split in shared memory.
constexpr int kSavePlanes = 1;
// bytes of one 64-pixel block of an activation / dY array with `rows` channels
__host__ __device__ inline uint32_t blk_bytes(int rows) {
  return kActInterleave ? (uint32_t)((rows + 7) / 8) * 1024u : (uint32_t)((rows + 63) / 64) * 8192u;
}
__host__ __device__ inline int layer_in(const MlpLayout& L, int l) { return l == 0 ? L.nin : kWidth; }
__host__ __device__ inline int layer_out(int l) { return l == 5 ? 3 : kWidth; }

inline MlpLayout make_layout(const dvd_mlp_cfg& c, long npx) {
  MlpLayout L;
  L.nin = mlp_nin(c);
  L.kpad0 = mlp_specialised(c) ? (L.nin + 15) / 16 * 16 : (L.nin + 63) / 64 * 64;
  L.k0_chunks = (L.kpad0 + 63) / 64;
  L.npx = npx;
  L.ntiles = (npx + kTileM - 1) / kTileM;
  L.nq = L.ntiles * 2;
  size_t o = 0;
  for (int l = 0; l < kLayers; ++l) {
    L.wf_off[l] = o;
    o += (size_t)nkc_f(L, l) * 2 * rows_f(l) * 128;
  }
  L.wf_total = o;
  o = 0;
  for (int l = 0; l < kLayers; ++l) {
    L.wb_off[l] = o;
    o += (size_t)nkc_b(l) * 2 * rows_b(L, l) * 128;
  }
  L.wb_total = o;
  o = 0;
  for (int l = 0; l < kLayers; ++l) {
    L.xs_off[l] = o;
    o += (size_t)kSavePlanes * L.nq * blk_bytes(rows_x(L, l));
  }
  L.mask_off = o;
  o += (size_t)5 * L.ntiles * kTileM * 32;  // 5 layers x 256 bits per pixel
  L.save_total = (o + 255) & ~(size_t)255;
  o = 0;
  for (int l = 0; l < kLayers; ++l) {
    L.dy_off[l] = o;
    o += (size_t)kSavePlanes * L.nq * blk_bytes(rows_dy(l));
  }
  L.dy_total = (o + 255) & ~(size_t)255;
  return L;
}

}  // namespace dvd
