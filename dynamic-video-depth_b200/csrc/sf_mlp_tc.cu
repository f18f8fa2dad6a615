// Scene-flow MLP on the Hopper tensor cores (sm_90a wgmma): fused Euler-chain forward, fused dgrad chain,
// split-K wgrad. Replaces (reference paths relative to the reference tree):
//   PeriodicEmbed.forward                     networks/blocks.py:19-34                       (M1)
//   SceneFlowFieldNet.forward / Conv2dBlock   networks/sceneflow_field.py:20-53, blocks.py:50-102 (M2)
//   Model.forward_sf_net (+ /sf_mag_div)      models/scene_flow_motion_field.py:346-358      (M3)
//   Model.forward_sf_net_multi_step           models/scene_flow_motion_field.py:360-367      (M4)
//   autograd backward of the above (the reference materialises a [B,256,H,W] fp32 activation per layer).
//
// Design: one CTA owns a tile of 128 pixels and pushes it through ALL layers and all
// Euler steps without leaving the SM. Two MMA warpgroups own 64 pixels each: the activation tile is the A operand
// and lives in SHARED MEMORY (K-major SWIZZLE_128B bf16 hi / lo images, rewritten by the epilogue after every layer);
// the accumulator D [64 x 256] fp32 lives in registers (wgmma m64n256k16). Weights are the B operand: streamed per
// layer from L2 into a shared-memory ring by 1-D bulk async copies of pre-swizzled blocks (see sf_mlp_layout.cuh), each
// block in pieces of at most 128 output rows; one wgmma group per piece stays in flight while the next piece is awaited.
// fp32 accuracy comes from the bf16 (hi, lo) split: D += Ahi*Bhi + Alo*Bhi + Ahi*Blo.
// Warp roles: warpgroup 0 = weight producer (one thread), warpgroups 1, 2 = MMA + epilogue (bias, LeakyReLU, hi/lo
// split -> shared memory; embedding; Euler update). The four lanes of a quad share two pixels (fragment rows) and
// split their channels.
#include "common.cuh"
#include "sf_mlp_layout.cuh"
#include "tc_common.cuh"

namespace dvd {
using namespace tc;

__host__ __device__ __forceinline__ uint32_t act_offset(uint32_t ch, uint32_t px) {
  return kActInterleave ? il_offset(ch, px) : mn128_offset(ch, px);
}
__device__ __forceinline__ uint64_t act_desc(uint32_t smem_addr, int ks) {
  return kActInterleave ? make_sdesc_mn_interleave(smem_addr + ks * 256, 1024) : make_sdesc_mn_sw128(smem_addr + ks * 2048, 8192);
}

// Weight ring: a [rows x 64 K] weight block is streamed in pieces of at most kPieceRows rows (a 256-row block is two 16 KB
// pieces; blocks of 16, 64, 112 and 128 rows are one piece, 144 rows are 128 + 16, 192 rows 128 + 64). The activation images
// take 128 KB of the shared memory, which leaves room for five 16 KB stages (and the bias table) but only two whole 32 KB
// blocks.
constexpr int kPieceRows = 128;
constexpr int kStages = 5;
constexpr uint32_t kStageBytes = kPieceRows * 128;
constexpr int kThreadsMlp = 384;                   // warpgroup 0: weight producer, warpgroups 1, 2: MMA + epilogue (64 pixels each)
constexpr int kThreadsWgrad = 384;

// =============================================================================================
// weight packing
struct PackParams {
  const float* w[kLayers];
  uint8_t* wf;
  uint8_t* wb;
  MlpLayout L;
};

__global__ void __launch_bounds__(256) pack_weights_kernel(PackParams P) {
  DVD_PDL_ENTER();
  const int img = blockIdx.y / kLayers, l = blockIdx.y % kLayers;
  const int in = layer_in(P.L, l), out = layer_out(l);
  const float* __restrict__ W = P.w[l];
  const int rows = img == 0 ? rows_f(l) : rows_b(P.L, l);
  const int nkc = img == 0 ? nkc_f(P.L, l) : nkc_b(l);
  uint8_t* base = img == 0 ? P.wf + P.L.wf_off[l] : P.wb + P.L.wb_off[l];
  const int total = nkc * rows * 32;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    int kp = idx & 31, row = (idx >> 5) % rows, kc = (idx >> 5) / rows;
    int k = kp * 2, gk = kc * 64 + k;
    float v0, v1;
    if (img == 0) {  // B[n = out row][k = in]
      v0 = (row < out && gk < in) ? W[(size_t)row * in + gk] : 0.f;
      v1 = (row < out && gk + 1 < in) ? W[(size_t)row * in + gk + 1] : 0.f;
    } else {         // B[n = in row][k = out]
      v0 = (row < in && gk < out) ? W[(size_t)gk * in + row] : 0.f;
      v1 = (row < in && gk + 1 < out) ? W[(size_t)(gk + 1) * in + row] : 0.f;
    }
    uint32_t hi, lo;
    split2(v0, v1, hi, lo);
    uint8_t* blk = base + (size_t)(kc * 2) * rows * 128;
    uint32_t off = sw128_offset(row, k);
    *reinterpret_cast<uint32_t*>(blk + off) = hi;
    *reinterpret_cast<uint32_t*>(blk + (size_t)rows * 128 + off) = lo;
  }
}

// =============================================================================================
// periodic embedding (M1), feature order of SceneFlowFieldNet.forward: cat([t_emb, xyz_emb])
//   t_emb   = [t, cos(ft_k t) k<FT, sin(ft_k t) k<FT]                       (NT = 1 + 2 FT, if time dependent)
//   xyz_emb = [x, y, z, cos(f_k x), cos(f_k y), cos(f_k z) k<FX, sin(...) k<FX]
// Loops over the frequencies are deliberately NOT unrolled: a fully unrolled epilogue was ~0.5 MB of SASS and
// spent 30 % of its issue slots waiting for the instruction cache.
// FX = kRuntime: the generic kernels; the counts and time_dependent are read from the configuration (FT, TD unused).
constexpr int kRuntime = -1;
template <int FX, int FT, bool TD>
struct Embed {
  static constexpr bool kStatic = FX != kRuntime;
  static constexpr int KPAD = kStatic ? ((TD ? 1 + 2 * FT : 0) + 3 + 6 * FX + 15) / 16 * 16 : 0;
  int fx, ft, nt;
  bool td;
  __device__ __forceinline__ explicit Embed(const dvd_mlp_cfg& c)
      : fx(kStatic ? FX : c.n_freq_xyz), ft(kStatic ? FT : c.n_freq_t), td(kStatic ? TD : c.time_dependent != 0) {
    nt = td ? 1 + 2 * ft : 0;
  }

  // feature j (runtime index)
  __device__ __forceinline__ float feature(const dvd_mlp_cfg& c, int j, float t, float x, float y, float z) const {
    float s, co;
    if (j < nt) {
      if (j == 0) return t;
      int k = j - 1;
      const bool is_sin = k >= ft;
      if (is_sin) k -= ft;
      fast_sincos(c.freq_t[k] * t, s, co);
      return is_sin ? s : co;
    }
    j -= nt;
    if (j < 3) return j == 0 ? x : (j == 1 ? y : z);
    j -= 3;
    if (j >= 6 * fx) return 0.f;
    const bool is_sin = j >= 3 * fx;
    if (is_sin) j -= 3 * fx;
    const int k = j / 3, d = j - 3 * k;
    fast_sincos(c.freq_xyz[k] * (d == 0 ? x : (d == 1 ? y : z)), s, co);
    return is_sin ? s : co;
  }
};

// shared-memory carve-up common to the chain kernels
struct ChainSmem {
  uint8_t* ring;         // kStages stages of kStageBytes (stage s at ring + s * kStageBytes: no pointer array in local memory)
  uint8_t* act;          // per MMA warpgroup: hi plane [4 x 8 KB] | lo plane [4 x 8 KB] (64 pixel rows x 256 K, K-major SW128)
  float* bias;           // 5*256 + 16
  uint64_t* w_full;      // [kStages]
  uint64_t* w_empty;     // [kStages]
};
constexpr uint32_t kActBytes = 65536;   // one warpgroup's activation image (both planes)
constexpr size_t kChainSmemBytes = 1024 + (size_t)kStages * kStageBytes + 2 * kActBytes + (5 * 256 + 16) * 4 + 256;
static_assert(kChainSmemBytes <= 232448, "shared memory of one CTA on sm_90");

__device__ __forceinline__ ChainSmem carve(uint8_t* raw) {
  ChainSmem s;
  uint8_t* p = raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
  s.ring = p;
  p += (size_t)kStages * kStageBytes;
  s.act = p;
  p += 2 * kActBytes;
  s.bias = reinterpret_cast<float*>(p);
  p += (5 * 256 + 16) * 4;
  s.w_full = reinterpret_cast<uint64_t*>(p);
  s.w_empty = s.w_full + kStages;
  return s;
}

__device__ __forceinline__ void chain_setup(ChainSmem& s) {
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&s.w_full[i], 1);
      mbar_init(&s.w_empty[i], 8);     // one arrival per MMA warp
    }
    fence_mbar_init();
  }
}

// producer: stream the weight blocks (layer, k-chunk, plane) in MMA order, `n_rep` passes per tile
__device__ __forceinline__ void stream_weights(ChainSmem& S, const uint8_t* base, const MlpLayout& L, long ntiles, int n_rep, bool fwd) {
  uint32_t it = 0;
  for (long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    for (int e = 0; e < n_rep; ++e) {
      for (int li = 0; li < kLayers; ++li) {
        const int l = fwd ? li : kLayers - 1 - li;
        const int rows = fwd ? rows_f(l) : rows_b(L, l);
        const uint8_t* src = base + (fwd ? L.wf_off[l] : L.wb_off[l]);
        const int n = (fwd ? nkc_f(L, l) : nkc_b(l)) * 2;
        for (int j = 0; j < n; ++j) {            // block (kc, plane) = j; its pieces are contiguous row ranges of the block
          for (int r0 = 0; r0 < rows; r0 += kPieceRows, ++it) {
            const uint32_t s = it % kStages, ph = (it / kStages) & 1u;
            const uint32_t bytes = (uint32_t)min(kPieceRows, rows - r0) * 128u;
            mbar_wait(&S.w_empty[s], ph ^ 1u);
            mbar_arrive_expect_tx(&S.w_full[s], bytes);
            bulk_g2s(S.ring + s * kStageBytes, src + ((size_t)j * rows + r0) * 128u, bytes, &S.w_full[s]);
          }
        }
      }
    }
  }
}

// columns [C0, C0 + W) of an m64nN wgmma accumulator fragment: registers [C0 / 2, (C0 + W) / 2) (four per 8 columns)
template <int C0, int W, int R>
__device__ __forceinline__ float (&acc_cols(float (&acc)[R]))[W / 2] {
  static_assert(C0 % 8 == 0 && (C0 + W) / 2 <= R, "columns of the fragment");
  return *reinterpret_cast<float (*)[W / 2]>(&acc[C0 / 2]);
}

// one ring stage: the wgmma group of weight piece `it` (W output rows of the hi or lo plane of 64-K block kc) into its W
// columns of the accumulator. The group stays in flight: once it is committed, the previous group is waited for and its
// stage released (none before the first stage of a layer: the layer before ended with every group done).
template <int W, int PLANE>
__device__ __forceinline__ void chain_stage(ChainSmem& S, float (&acc)[W / 2], uint32_t act_hi, int kc, uint32_t& it, bool first) {
  const uint32_t act_lo = act_hi + kActBytes / 2;
  const uint32_t s = it % kStages, ph = (it / kStages) & 1u;
  mbar_wait(&S.w_full[s], ph);
  const uint32_t sb = smem_u32(S.ring) + s * kStageBytes;
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const uint64_t bd = make_sdesc_k_sw128(sb + ks * 32);
    const uint32_t ao = (uint32_t)kc * 8192u + ks * 32;
    if (PLANE == 0) {
      wgmma_bf16_ss<W>(acc, make_sdesc_k_sw128(act_hi + ao), bd, (kc | ks) ? 1u : 0u);
      wgmma_bf16_ss<W>(acc, make_sdesc_k_sw128(act_lo + ao), bd, 1u);
    } else {
      wgmma_bf16_ss<W>(acc, make_sdesc_k_sw128(act_hi + ao), bd, 1u);
    }
  }
  wgmma_commit();
  wgmma_wait<1>();
  if (!first) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(&S.w_empty[(it - 1) % kStages]);
  }
  ++it;
}

// one layer of the chain on this warpgroup's 64 rows: acc[64 x N] = A (hi, lo) * W^T with the bf16x3 split
// (A_hi W_hi + A_lo W_hi from the hi-plane pieces, A_hi W_lo from the lo-plane pieces). `it` = ring position.
// Per 64-K block the pieces come in the producer's order: hi plane (columns 0..127, then the rest), lo plane (likewise), so
// every accumulator element receives its products in the order of a whole-block MMA. Every piece is consumed whole (four k16
// slices, a fixed trip count: no control flow between the wgmmas of a group). Packed weights are zero beyond a layer's K,
// and the activation image is zero-filled there (finite values).
template <int N>
__device__ __forceinline__ void chain_layer(ChainSmem& S, float (&acc)[N / 2], uint32_t act_hi, int nkc, uint32_t& it) {
  constexpr int N0 = N < kPieceRows ? N : kPieceRows, N1 = N - N0;
  static_assert(N1 <= kPieceRows, "a weight block is at most two pieces");
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  for (int kc = 0; kc < nkc; ++kc) {
    chain_stage<N0, 0>(S, acc_cols<0, N0>(acc), act_hi, kc, it, kc == 0);
    if constexpr (N1 > 0) chain_stage<N1, 0>(S, acc_cols<N0, N1>(acc), act_hi, kc, it, false);
    chain_stage<N0, 1>(S, acc_cols<0, N0>(acc), act_hi, kc, it, false);
    if constexpr (N1 > 0) chain_stage<N1, 1>(S, acc_cols<N0, N1>(acc), act_hi, kc, it, false);
  }
  wgmma_wait<0>();
  fence_regs(acc);
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(&S.w_empty[(it - 1) % kStages]);
}

// write the packed pair (hi, lo) of K columns (k, k+1) of local row `row` into the warpgroup's activation image
__device__ __forceinline__ void put_act(uint8_t* act, int row, int k, uint32_t hi, uint32_t lo) {
  const uint32_t o = (uint32_t)(k >> 6) * 8192u + sw128_offset((uint32_t)row, (uint32_t)(k & 63));
  *reinterpret_cast<uint32_t*>(act + o) = hi;
  *reinterpret_cast<uint32_t*>(act + kActBytes / 2 + o) = lo;
}
// the activation image written by the generic proxy is read by the next layer's wgmma (async proxy)
__device__ __forceinline__ void act_publish(int cw) {
  fence_proxy_async_smem();
  named_sync(1 + cw, 128);
}

// The hi plane of a warpgroup's activation image is byte for byte the saved block of its 64 pixels (sf_mlp_layout.cuh): in
// both, a pixel's 64-channel group is one 128-byte row with its 16-byte chunks XOR-swizzled by the pixel
// (sw128_offset(px, ch) == mn128_offset(ch, px)). So once the image is published, one thread of the warpgroup saves it with
// one bulk copy to global memory, and waits for the copy's reads before the image is written again. The data gradient saves
// its dY this way: 2.68-2.70 ms per evaluation of 8 pairs at 384 x 224 against 3.08-3.14 ms with a 4-byte store per thread
// and channel pair (H100 SXM, 700 W). The forward keeps its per-thread stores of X: there the bulk copy measured 3.19-3.21 ms
// against 3.07-3.13 ms.
static_assert(!kActInterleave, "the saved blocks share the layout of the activation image");
__device__ __forceinline__ void save_image(uint8_t* dst, uint8_t* act, uint32_t bytes) {
  if ((threadIdx.x & 127) == 0) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(act)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  }
}
// before the warpgroup's barrier that precedes a rewrite of the image
__device__ __forceinline__ void save_image_wait_read() {
  if ((threadIdx.x & 127) == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// before the warpgroup exits: every saved block is written
__device__ __forceinline__ void save_image_wait_all() {
  if ((threadIdx.x & 127) == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// =============================================================================================
// forward chain
struct FwdParams {
  const uint8_t* wf;
  const float* bias;
  const float* p0;
  const float* t0;
  float dt;
  int n_eval, n_acc;
  float* acc;
  float* s_steps;
  float* p_steps;
  uint8_t* save;
  long npx, hw;
  MlpLayout L;
  dvd_mlp_cfg cfg;
};

// One CTA = 128 pixels through all layers and Euler steps. Warpgroup 0: weight producer; warpgroups 1, 2: 64 pixels each
// (wgmma M = 64), accumulator in registers, activations as the A operand in shared memory. Fragment rows: qrow, qrow + 8.
template <int FX, int FT, bool TD, bool SAVE>
__global__ void __launch_bounds__(kThreadsMlp, 1) mlp_chain_fwd_kernel(const __grid_constant__ FwdParams P) {
  using E = Embed<FX, FT, TD>;
  const E emb(P.cfg);
  extern __shared__ uint8_t smem_raw[];
  ChainSmem S = carve(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const MlpLayout& L = P.L;
  const int kpad0 = E::kStatic ? E::KPAD : L.kpad0;
  chain_setup(S);
  DVD_PDL_ENTER();               // barriers are set up: now wait for the producer of the operands
  for (int i = threadIdx.x; i < 5 * 256 + 16; i += blockDim.x) S.bias[i] = P.bias[i];
  __syncthreads();
  const long ntiles = L.ntiles;
  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) stream_weights(S, P.wf, L, ntiles, P.n_eval, true);
    return;
  }
  setmaxnreg_inc<232>();
  const int cw = wg - 1, t4 = lane & 3;
  const int lrow0 = (warp & 3) * 16 + (lane >> 2);       // local rows lrow0, lrow0 + 8 of this warpgroup's 64
  uint8_t* act = S.act + (size_t)cw * kActBytes;
  const uint32_t act_u = smem_u32(act);
  float acc[128];
  uint32_t it = 0;
  for (long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long chunk = tile * 2 + cw;                   // 64-pixel block of the saved layouts
    float px[2], py[2], pz[2], tt[2], ax[2] = {0.f, 0.f}, ay[2] = {0.f, 0.f}, az[2] = {0.f, 0.f};
    bool valid[2];
    size_t pidx[2];
    for (int h = 0; h < 2; ++h) {
      const long g = chunk * 64 + lrow0 + 8 * h;
      valid[h] = g < P.npx;
      const long b = valid[h] ? g / P.hw : 0, i = valid[h] ? g % P.hw : 0;
      pidx[h] = (size_t)b * 3 * P.hw + i;
      px[h] = py[h] = pz[h] = tt[h] = 0.f;
      if (valid[h]) {
        px[h] = P.p0[pidx[h]]; py[h] = P.p0[pidx[h] + P.hw]; pz[h] = P.p0[pidx[h] + 2 * P.hw];
        if (emb.td) tt[h] = P.t0[(size_t)b * P.hw + i];
      }
    }
    for (int e = 0; e < P.n_eval; ++e) {
      uint8_t* save_e = SAVE ? P.save + (size_t)e * L.save_total : nullptr;
      // ---- embedding -> A operand of layer 0 (the four lanes of a quad split the feature pairs of their two pixels)
      named_sync(1 + cw, 128);                          // the previous layer's MMAs of every warp are done with the image
      for (int h = 0; h < 2; ++h) {
        const int row = lrow0 + 8 * h;
        if (SAVE && valid[h] && t4 == 0) {
          float* ps = P.p_steps + (size_t)e * P.npx * 3 + pidx[h];
          ps[0] = px[h]; ps[P.hw] = py[h]; ps[2 * P.hw] = pz[h];
        }
        uint8_t* x0_hi = SAVE ? save_e + L.xs_off[0] + (size_t)chunk * blk_bytes(kpad0) : nullptr;
#pragma unroll 1
        for (int w = t4; w < 32 * L.k0_chunks; w += 4) {        // features, then zeros up to the end of the last 64-K block
          uint32_t hi, lo;
          split2(emb.feature(P.cfg, 2 * w, tt[h], px[h], py[h], pz[h]), emb.feature(P.cfg, 2 * w + 1, tt[h], px[h], py[h], pz[h]), hi, lo);
          put_act(act, row, 2 * w, hi, lo);
          if (SAVE) *reinterpret_cast<uint32_t*>(x0_hi + act_offset(2 * w, row)) = hi;
        }
      }
      act_publish(cw);
      // ---- hidden layers
      for (int l = 0; l < 5; ++l) {
        chain_layer<256>(S, acc, act_u, nkc_f(L, l), it);
        named_sync(1 + cw, 128);                        // every warp's MMAs have read the image: overwrite it
        const float* bl = S.bias + l * 256;
        uint8_t* x_hi = SAVE ? save_e + L.xs_off[l + 1] + (size_t)chunk * blk_bytes(kWidth) : nullptr;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = lrow0 + 8 * h;
          uint32_t* maskp = SAVE ? reinterpret_cast<uint32_t*>(save_e + L.mask_off + (((size_t)l * L.ntiles + tile) * kTileM + cw * 64 + row) * 32)
                                 : nullptr;
#pragma unroll
          for (int q = 0; q < 8; ++q) {          // mask word q = channels 32 q .. 32 q + 31
            uint32_t mw = 0;
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = 4 * q + jj, c = 8 * j + 2 * t4;
              const float y0 = acc[4 * j + 2 * h] + bl[c], y1 = acc[4 * j + 2 * h + 1] + bl[c + 1];
              if (SAVE) mw |= ((y0 > 0.f ? 1u : 0u) | (y1 > 0.f ? 2u : 0u)) << (c & 31);
              uint32_t hi, lo;
              // LeakyReLU(0.2): max(y, 0.2 y)
              split2(fmaxf(y0, 0.2f * y0), fmaxf(y1, 0.2f * y1), hi, lo);
              put_act(act, row, c, hi, lo);
              if (SAVE) *reinterpret_cast<uint32_t*>(x_hi + act_offset(c, row)) = hi;
            }
            if (SAVE) {
              mw |= __shfl_xor_sync(0xffffffffu, mw, 1);
              mw |= __shfl_xor_sync(0xffffffffu, mw, 2);
              if (t4 == 0) maskp[q] = mw;
            }
          }
        }
        act_publish(cw);
      }
      // ---- output layer (N = 16 padded, 3 used): s = (W5 x + b5) / sf_mag_div ; Euler update
      {
        float a16[8];
        chain_layer<16>(S, a16, act_u, nkc_f(L, 5), it);
        const float* b5 = S.bias + 5 * 256;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          // columns 0, 1 live in lane t4 = 0, column 2 in lane t4 = 1 of the quad
          const float c2 = __shfl_down_sync(0xffffffffu, a16[2 * h], 1);
          float sx = (a16[2 * h] + b5[0]) / P.cfg.sf_mag_div, sy = (a16[2 * h + 1] + b5[1]) / P.cfg.sf_mag_div;
          float sz = (c2 + b5[2]) / P.cfg.sf_mag_div;
          const int src = lane & ~3;
          sx = __shfl_sync(0xffffffffu, sx, src); sy = __shfl_sync(0xffffffffu, sy, src); sz = __shfl_sync(0xffffffffu, sz, src);
          if (valid[h] && P.s_steps && t4 == 0) {
            float* ss = P.s_steps + (size_t)e * P.npx * 3 + pidx[h];
            ss[0] = sx; ss[P.hw] = sy; ss[2 * P.hw] = sz;
          }
          if (e < P.n_acc) { ax[h] += sx; ay[h] += sy; az[h] += sz; }
          px[h] += sx; py[h] += sy; pz[h] += sz;
          tt[h] += P.dt;
        }
      }
    }
    for (int h = 0; h < 2; ++h) {
      if (valid[h] && P.acc && t4 == 0) {
        float* ao = P.acc + pidx[h];
        ao[0] = ax[h]; ao[P.hw] = ay[h]; ao[2 * P.hw] = az[h];
      }
    }
  }
}

// =============================================================================================
// dgrad chain of one eval
struct DgradParams {
  const uint8_t* wb;
  const float* p_e;
  const float* t0;
  float dt;
  int e, use_g_acc;
  const float* g_acc;
  const float* g_step;
  const float* a_in;
  float* a_out;
  const uint8_t* save_e;
  uint8_t* dy;
  float* g_bias5;
  long npx, hw;
  MlpLayout L;
  dvd_mlp_cfg cfg;
  float* ord;      // ordered variant: [CTA][MMA warp][3] output-bias partials
};

// KPAD: the layer-0 width L.kpad0 (the N of its MMA)
template <int FX, int FT, bool TD, int KPAD, bool ORD = false>
__global__ void __launch_bounds__(kThreadsMlp, 1) mlp_dgrad_kernel(const __grid_constant__ DgradParams P) {
  using E = Embed<FX, FT, TD>;
  static_assert(!E::kStatic || KPAD == E::KPAD, "layer-0 width of a specialised configuration");
  const E emb(P.cfg);
  extern __shared__ uint8_t smem_raw[];
  ChainSmem S = carve(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const MlpLayout& L = P.L;
  chain_setup(S);
  __syncthreads();
  const long ntiles = L.ntiles;
  DVD_PDL_ENTER();
  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) stream_weights(S, P.wb, L, ntiles, 1, false);
    return;
  }
  setmaxnreg_inc<232>();
  const int cw = wg - 1, t4 = lane & 3;
  const int lrow0 = (warp & 3) * 16 + (lane >> 2);
  uint8_t* act = S.act + (size_t)cw * kActBytes;
  const uint32_t act_u = smem_u32(act);
  float acc[128];
  uint32_t it = 0;
  float b5x = 0.f, b5y = 0.f, b5z = 0.f;  // per-thread partial of the output-bias gradient
  for (long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long chunk = tile * 2 + cw;
    // per-pixel values are recomputed / re-read where they are used: nothing per pixel stays live across the six layers
    auto pixel = [&](int h, size_t& pidx) -> bool {
      const long g = chunk * 64 + lrow0 + 8 * h;
      if (g >= P.npx) return false;
      pidx = (size_t)(g / P.hw) * 3 * P.hw + (size_t)(g % P.hw);
      return true;
    };
    save_image_wait_read();
    named_sync(1 + cw, 128);
    for (int h = 0; h < 2; ++h) {
      const int row = lrow0 + 8 * h;
      size_t pidx = 0;
      const bool valid = pixel(h, pidx);
      float gs[3] = {0.f, 0.f, 0.f};
      for (int d = 0; d < 3; ++d) {
        if (valid) {
          const size_t o = pidx + (size_t)d * P.hw;
          if (P.a_in) gs[d] = P.a_in[o];
          if (P.use_g_acc && P.g_acc) gs[d] += P.g_acc[o];
          if (P.g_step) gs[d] += P.g_step[o];
        }
      }
      // dY_5 = gs / sf_mag_div (3 of 16 padded columns)
      const float d5x = gs[0] / P.cfg.sf_mag_div, d5y = gs[1] / P.cfg.sf_mag_div, d5z = gs[2] / P.cfg.sf_mag_div;
      if (t4 == 0) { b5x += d5x; b5y += d5y; b5z += d5z; }
      uint8_t* y_hi = P.dy + L.dy_off[5] + (size_t)chunk * blk_bytes(16);
      // K = 16 (3 used) of dY_5; zeros up to the end of the 64-K block the first MMA reads
      for (int w = t4; w < 32; w += 4) {
        uint32_t hi = 0, lo = 0;
        if (w == 0) split2(d5x, d5y, hi, lo);
        else if (w == 1) split2(d5z, 0.f, hi, lo);
        put_act(act, row, 2 * w, hi, lo);
        if (w < 8) *reinterpret_cast<uint32_t*>(y_hi + act_offset(2 * w, row)) = hi;
      }
    }
    act_publish(cw);
    // MMA(l) produces dX_l (input gradient of layer l); l = 5..1 feed dY_{l-1}
    for (int l = 5; l >= 1; --l) {
      chain_layer<256>(S, acc, act_u, nkc_b(l), it);
      save_image_wait_read();
      named_sync(1 + cw, 128);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = lrow0 + 8 * h;
        const uint32_t* maskp = reinterpret_cast<const uint32_t*>(P.save_e + L.mask_off +
                                                                  (((size_t)(l - 1) * L.ntiles + tile) * kTileM + cw * 64 + row) * 32);
#pragma unroll
        for (int q = 0; q < 8; ++q) {            // mask word q = channels 32 q .. 32 q + 31
          const uint32_t mw = maskp[q];
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = 4 * q + jj, c = 8 * j + 2 * t4;
            float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            v0 *= ((mw >> (c & 31)) & 1u) ? 1.0f : 0.2f;
            v1 *= ((mw >> ((c & 31) + 1)) & 1u) ? 1.0f : 0.2f;
            uint32_t hi, lo;
            split2(v0, v1, hi, lo);
            put_act(act, row, c, hi, lo);
          }
        }
      }
      act_publish(cw);
      save_image(P.dy + L.dy_off[l - 1] + (size_t)chunk * blk_bytes(kWidth), act, blk_bytes(kWidth));
    }
    // MMA(0) -> gradient w.r.t. the embedding; contract with d(embed)/d(xyz)
    {
      float a0[KPAD / 2];
      chain_layer<KPAD>(S, a0, act_u, nkc_b(0), it);
      if constexpr (E::kStatic) {
        const int CB = emb.nt + 3, SB = emb.nt + 3 + 3 * emb.fx;   // first cos / sin feature
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          size_t pidx = 0;
          const bool valid = pixel(h, pidx);
          float p[3] = {0.f, 0.f, 0.f};
          if (valid) {
            p[0] = P.p_e[pidx]; p[1] = P.p_e[pidx + P.hw]; p[2] = P.p_e[pidx + 2 * P.hw];
          }
          float gp[3] = {0.f, 0.f, 0.f};
#pragma unroll
          for (int j = 0; j < KPAD / 8; ++j) {
#pragma unroll
            for (int cc = 0; cc < 2; ++cc) {
              const int c = 8 * j + 2 * t4 + cc;
              const float gv = a0[4 * j + 2 * h + cc];
              if (c >= emb.nt && c < CB) {
                gp[c - emb.nt] += gv;
              } else if (c >= CB && c < SB + 3 * emb.fx) {
                const bool is_sin = c >= SB;
                const int k = (c - (is_sin ? SB : CB)) / 3, d = (c - (is_sin ? SB : CB)) % 3;
                const float f = P.cfg.freq_xyz[k];
                float s, co;
                fast_sincos(f * p[d], s, co);
                // d/dx cos(f x) = -f sin(f x) ; d/dx sin(f x) = f cos(f x)
                gp[d] += is_sin ? f * co * gv : -f * s * gv;
              }
            }
          }
#pragma unroll
          for (int d = 0; d < 3; ++d) {
            gp[d] += __shfl_xor_sync(0xffffffffu, gp[d], 1);
            gp[d] += __shfl_xor_sync(0xffffffffu, gp[d], 2);
          }
          if (valid && P.a_out && t4 == 0) {
#pragma unroll
            for (int d = 0; d < 3; ++d) {
              const size_t o = pidx + (size_t)d * P.hw;
              P.a_out[o] = (P.a_in ? P.a_in[o] : 0.f) + gp[d];
            }
          }
        }
      } else {
        // Runtime counts: a0 goes to this warpgroup's activation image (free once every warp's layer-0 MMAs are done), one
        // fp32 slot per thread and accumulator register (KPAD / 2 x 128 x 4 B <= kActBytes, conflict-free). Each thread then
        // walks its own features in a loop that is not unrolled, so no array is indexed by a run-time value.
        save_image_wait_read();
        named_sync(1 + cw, 128);
        float* g0 = reinterpret_cast<float*>(act) + (threadIdx.x & 127);
#pragma unroll
        for (int i = 0; i < KPAD / 2; ++i) g0[i * 128] = a0[i];
        const int nxyz = 3 + 6 * emb.fx, nj = (emb.nt + nxyz + 7) / 8;
        for (int h = 0; h < 2; ++h) {
          size_t pidx = 0;
          const bool valid = pixel(h, pidx);
          const float x = valid ? P.p_e[pidx] : 0.f, y = valid ? P.p_e[pidx + P.hw] : 0.f, z = valid ? P.p_e[pidx + 2 * P.hw] : 0.f;
          float gx = 0.f, gy = 0.f, gz = 0.f;
#pragma unroll 1
          for (int j = 0; j < nj; ++j) {
#pragma unroll
            for (int cc = 0; cc < 2; ++cc) {
              int q = 8 * j + 2 * t4 + cc - emb.nt;          // index into xyz_emb
              if (q < 0 || q >= nxyz) continue;
              const float gv = g0[(4 * j + 2 * h + cc) * 128];
              float term = gv;
              int d = q;
              if (q >= 3) {
                q -= 3;
                const bool is_sin = q >= 3 * emb.fx;
                if (is_sin) q -= 3 * emb.fx;
                const int k = q / 3;
                d = q - 3 * k;
                const float f = P.cfg.freq_xyz[k];
                float sn, co;
                fast_sincos(f * (d == 0 ? x : (d == 1 ? y : z)), sn, co);
                // d/dx cos(f x) = -f sin(f x) ; d/dx sin(f x) = f cos(f x)
                term = is_sin ? f * co * gv : -f * sn * gv;
              }
              gx += d == 0 ? term : 0.f;
              gy += d == 1 ? term : 0.f;
              gz += d == 2 ? term : 0.f;
            }
          }
          gx += __shfl_xor_sync(0xffffffffu, gx, 1); gx += __shfl_xor_sync(0xffffffffu, gx, 2);
          gy += __shfl_xor_sync(0xffffffffu, gy, 1); gy += __shfl_xor_sync(0xffffffffu, gy, 2);
          gz += __shfl_xor_sync(0xffffffffu, gz, 1); gz += __shfl_xor_sync(0xffffffffu, gz, 2);
          if (valid && P.a_out && t4 == 0) {
            const size_t o = pidx, o1 = pidx + P.hw, o2 = pidx + 2 * P.hw;
            P.a_out[o] = (P.a_in ? P.a_in[o] : 0.f) + gx;
            P.a_out[o1] = (P.a_in ? P.a_in[o1] : 0.f) + gy;
            P.a_out[o2] = (P.a_in ? P.a_in[o2] : 0.f) + gz;
          }
        }
      }
    }
  }
  save_image_wait_all();
  // output-layer bias gradient: warp reduce, one atomic per warp
  b5x = warp_sum(b5x); b5y = warp_sum(b5y); b5z = warp_sum(b5z);
  if constexpr (ORD) {
    // the slabs are added in (CTA, warp) order by ordered_sum
    if (lane == 0 && P.g_bias5) {
      float* o = P.ord + ((size_t)blockIdx.x * 8 + (warp - 4)) * 3;
      o[0] = b5x; o[1] = b5y; o[2] = b5z;
    }
  } else {
  if (lane == 0 && P.g_bias5) {
    atomicAdd(P.g_bias5 + 0, b5x);
    atomicAdd(P.g_bias5 + 1, b5y);
    atomicAdd(P.g_bias5 + 2, b5z);
  }
  }
}

// =============================================================================================
// wgrad: D[128, n] += A_blk[128 ch x 64 px] * B_blk[n ch x 64 px]^T over a range of pixel chunks
// (both operands MN-major: channels contiguous, K = pixels); warpgroup w of the two MMA warpgroups owns channels 64 w ..
struct WgradJob {
  const uint8_t* a_hi;
  const uint8_t* a_lo;
  const uint8_t* b_hi;
  const uint8_t* b_lo;
  uint32_t a_blk, a_row_off, b_blk;
  int n, ld, transposed, m_off, m_valid, n_valid;
  float* out;
  float* bias_out;
};
struct WgradParams {
  WgradJob job[12];
  long nq;
  int nsplit;      // gridDim.y of the ordered variant
  float* ord;      // ordered variant: per CTA (job, split) a slab of kOrdSlab floats: [128 rows][256 columns], then 128 bias sums
};
constexpr int kOrdSlab = 128 * 256 + 128;
constexpr int kWgStages = 4;
constexpr uint32_t kWgStageBytes = kSavePlanes * (16384 + 32768);      // per plane: A 128 ch x 64 px, B up to 256 ch x 64 px (bf16)
constexpr size_t kWgradSmemBytes = 1024 + (size_t)kWgStages * kWgStageBytes + 8192 + 256;

template <int N>
__device__ __forceinline__ void wgrad_mma(float (&acc)[N / 2], float (&accb)[8], uint32_t sa, uint32_t sb, uint32_t so, uint32_t scale) {
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {   // 16 pixels (K rows of 128 B) per MMA
    const uint64_t ad = act_desc(sa, ks);
    wgmma_bf16_ss_mn<N>(acc, ad, act_desc(sb, ks), (scale | ks) ? 1u : 0u);
    wgmma_bf16_ss_mn<16>(accb, ad, act_desc(so, ks), (scale | ks) ? 1u : 0u);   // bias column sums (stored only with bias_out)
  }
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(acc);
  fence_regs(accb);
}

template <int N, bool ORD>
__device__ __forceinline__ void wgrad_consume(const WgradJob& J, uint8_t* const* stage, uint64_t* full, uint64_t* empty, uint32_t so,
                                              long q0, long q1, float* slab) {
  const int wg = threadIdx.x >> 7, cw = wg - 1, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, t4 = lane & 3;
  float acc[N / 2], accb[8];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) accb[i] = 0.f;
  uint32_t it = 0;
  for (long qq = q0; qq < q1; ++qq, ++it) {
    const uint32_t s = it % kWgStages, ph = (it / kWgStages) & 1u;
    mbar_wait(&full[s], ph);
    const uint32_t sa = smem_u32(stage[s]) + (uint32_t)cw * 8192u, sb = smem_u32(stage[s]) + 16384;
    wgrad_mma<N>(acc, accb, sa, sb, so, it ? 1u : 0u);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
  }
  if constexpr (ORD) {
    // this CTA's slab; mlp_wgrad_reduce_kernel adds the slabs of a job in split order
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int ml = cw * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
      if (J.m_off + ml >= J.m_valid) continue;
#pragma unroll
      for (int j = 0; j < N / 8; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int n = 8 * j + 2 * t4 + c;
          if (n < J.n_valid) slab[ml * 256 + n] = acc[4 * j + 2 * h + c];
        }
      if (J.bias_out && t4 == 0) slab[128 * 256 + ml] = accb[2 * h];
    }
  } else {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = J.m_off + cw * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    if (m >= J.m_valid) continue;
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int n = 8 * j + 2 * t4 + c;
        if (n < J.n_valid) {
          float* dst = J.transposed ? J.out + (size_t)n * J.ld + m : J.out + (size_t)m * J.ld + n;
          atomicAdd(dst, acc[4 * j + 2 * h + c]);
        }
      }
    if (J.bias_out && t4 == 0) atomicAdd(J.bias_out + m, accb[2 * h]);
  }
  }
}

template <bool ORD = false>
__global__ void __launch_bounds__(kThreadsWgrad, 1) mlp_wgrad_kernel(const __grid_constant__ WgradParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* stage[kWgStages];
  for (int i = 0; i < kWgStages; ++i) stage[i] = base + (size_t)i * kWgStageBytes;
  uint8_t* ones = base + (size_t)kWgStages * kWgStageBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(ones + 8192);
  uint64_t* empty = full + kWgStages;
  const int wg = threadIdx.x >> 7;
  const WgradJob& J = P.job[blockIdx.x];
  const long per = (P.nq + gridDim.y - 1) / gridDim.y;
  const long q0 = (long)blockIdx.y * per, q1 = min(P.nq, q0 + per);

  if (threadIdx.x == 0) {
    for (int i = 0; i < kWgStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    fence_mbar_init();
  }
  // "ones" operand [16 ch x 64 px], MN-major: channel 0 = 1.0 (bf16), channels 1..15 = 0 -> bias column sums
  for (int i = threadIdx.x; i < 8192 / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(ones)[i] = 0u;
  __syncthreads();
  if (threadIdx.x < 64) *reinterpret_cast<uint16_t*>(ones + act_offset(0, threadIdx.x)) = (uint16_t)0x3F80u;
  fence_proxy_async_smem();
  __syncthreads();
  DVD_PDL_ENTER();

  if (wg == 0) {
    if (threadIdx.x == 0) {
      uint32_t it = 0;
      const uint32_t a_bytes = 16384, b_bytes = blk_bytes(J.n);
      for (long qq = q0; qq < q1; ++qq, ++it) {
        const uint32_t s = it % kWgStages, ph = (it / kWgStages) & 1u;
        mbar_wait(&empty[s], ph ^ 1u);
        mbar_arrive_expect_tx(&full[s], a_bytes + b_bytes);
        uint8_t* d = stage[s];
        bulk_g2s(d, J.a_hi + (size_t)qq * J.a_blk + J.a_row_off, a_bytes, &full[s]);
        bulk_g2s(d + 16384, J.b_hi + (size_t)qq * J.b_blk, b_bytes, &full[s]);
      }
    }
    return;
  }
  if (q1 <= q0) return;
  const uint32_t so = smem_u32(ones);
  float* slab = ORD ? P.ord + ((size_t)blockIdx.x * gridDim.y + blockIdx.y) * kOrdSlab : nullptr;
  switch (J.n) {
    case 256: wgrad_consume<256, ORD>(J, stage, full, empty, so, q0, q1, slab); break;
    case 192: wgrad_consume<192, ORD>(J, stage, full, empty, so, q0, q1, slab); break;
    case 144: wgrad_consume<144, ORD>(J, stage, full, empty, so, q0, q1, slab); break;
    case 128: wgrad_consume<128, ORD>(J, stage, full, empty, so, q0, q1, slab); break;
    case 112: wgrad_consume<112, ORD>(J, stage, full, empty, so, q0, q1, slab); break;
    case 64: wgrad_consume<64, ORD>(J, stage, full, empty, so, q0, q1, slab); break;
    case 16: wgrad_consume<16, ORD>(J, stage, full, empty, so, q0, q1, slab); break;
    default: __trap();   // dvd_mlp_wgrad only builds jobs of these widths (checked there as well)
  }
}

// out[m, n] (or out[n, m]) += the job's split partials in split order; bias_out[m] likewise. blockIdx.x = job, blockIdx.y =
// row of the job's 128, thread = column; nparts: the splits with a non-empty pixel range
__global__ void __launch_bounds__(256) mlp_wgrad_reduce_kernel(const __grid_constant__ WgradParams P, int nparts) {
  DVD_PDL_ENTER();
  const WgradJob& J = P.job[blockIdx.x];
  const int ml = blockIdx.y, m = J.m_off + ml, n = threadIdx.x;
  if (m >= J.m_valid) return;
  const float* src = P.ord + (size_t)blockIdx.x * P.nsplit * kOrdSlab;
  if (n < J.n_valid) {
    float s = 0.f;
    for (int p = 0; p < nparts; ++p) s += __ldcg(src + (size_t)p * kOrdSlab + ml * 256 + n);
    float* dst = J.transposed ? J.out + (size_t)n * J.ld + m : J.out + (size_t)m * J.ld + n;
    *dst += s;
  }
  if (J.bias_out && n == 0) {
    float s = 0.f;
    for (int p = 0; p < nparts; ++p) s += __ldcg(src + (size_t)p * kOrdSlab + 128 * 256 + ml);
    J.bias_out[m] += s;
  }
}

// =============================================================================================
// acceleration regulariser on (s0, s1)
__global__ void __launch_bounds__(256) acc_reg_kernel(const float* __restrict__ s0, const float* __restrict__ s1, float c,
                                                      float* __restrict__ g0, float* __restrict__ g1,
                                                      float* __restrict__ partials, long n) {
  DVD_PDL_ENTER();
  __shared__ float red[8];
  float acc = 0.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    float d = s1[i] - s0[i];
    acc += fabsf(d);
    float s = (d > 0.f) ? c : ((d < 0.f) ? -c : 0.f);
    if (g0) g0[i] = -s;
    if (g1) g1[i] = s;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    partials[blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(256) acc_reg_final_kernel(const float* __restrict__ partials, int nb, float scale,
                                                            float* __restrict__ out) {
  DVD_PDL_ENTER();
  __shared__ double red[8];
  double a = 0;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) a += partials[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int w = 0; w < 8; ++w) t += red[w];
    out[0] = (float)(t * scale);
  }
}

// =============================================================================================
// variant 0: (16, 16, time-dependent), 1: (16, time-independent), 2: the generic kernels
static int check_cfg_supported(const dvd_mlp_cfg* cfg, int* variant) {
  DVD_ARG_CHECK(cfg != nullptr, "null mlp cfg");
  if (cfg->time_dependent && cfg->n_freq_xyz == 16 && cfg->n_freq_t == 16) { *variant = 0; return 0; }
  if (!cfg->time_dependent && cfg->n_freq_xyz == 16) { *variant = 1; return 0; }
  const bool counts_ok = cfg->n_freq_xyz >= 0 && (!cfg->time_dependent || cfg->n_freq_t >= 0);
  if (counts_ok && mlp_nin(*cfg) <= DVD_MLP_MAX_NIN) { *variant = 2; return 0; }
  set_error("unsupported scene-flow MLP configuration (n_freq_xyz=%d n_freq_t=%d time_dependent=%d): the first layer "
            "reads (time_dependent ? 1 + 2 n_freq_t : 0) + 3 + 6 n_freq_xyz = %d input features; the kernels take "
            "non-negative counts and at most %d features", cfg->n_freq_xyz, cfg->n_freq_t, cfg->time_dependent,
            mlp_nin(*cfg), DVD_MLP_MAX_NIN);
  return -2;
}

static int chain_grid(long ntiles) {
  int sms = num_sms();
  return (int)(ntiles < sms ? ntiles : sms);
}

}  // namespace dvd

using namespace dvd;

extern "C" size_t dvd_mlp_packed_weights_bytes(const dvd_mlp_cfg* cfg) {
  if (!cfg) return 0;
  MlpLayout L = make_layout(*cfg, 128);
  return L.wf_total > L.wb_total ? L.wf_total : L.wb_total;
}
extern "C" size_t dvd_mlp_save_bytes_per_eval(const dvd_mlp_cfg* cfg, long npx) {
  if (!cfg || npx <= 0) return 0;
  return make_layout(*cfg, npx).save_total;
}
extern "C" size_t dvd_mlp_dy_bytes(const dvd_mlp_cfg* cfg, long npx) {
  if (!cfg || npx <= 0) return 0;
  return make_layout(*cfg, npx).dy_total;
}

extern "C" int dvd_mlp_pack_weights(const dvd_mlp_cfg* cfg, const float* const* w, void* packed_fwd, void* packed_bwd,
                                    void* stream) {
  int variant;
  if (int e = check_cfg_supported(cfg, &variant)) return e;
  DVD_ARG_CHECK(w && packed_fwd && packed_bwd, "null pointer");
  PackParams P;
  for (int l = 0; l < kLayers; ++l) {
    DVD_ARG_CHECK(w[l] != nullptr, "null weight pointer for layer %d", l);
    P.w[l] = w[l];
  }
  P.wf = (uint8_t*)packed_fwd;
  P.wb = (uint8_t*)packed_bwd;
  P.L = make_layout(*cfg, 128);
  dvd::launch(pack_weights_kernel, dim3(32, 2 * kLayers), 256, 0, (cudaStream_t)stream, P);
  DVD_CUDA_LAUNCH_CHECK("mlp_pack_weights");
  return 0;
}

template <int FX, int FT, bool TD>
static int launch_fwd(const FwdParams& P, bool save, cudaStream_t st) {
  int grid = chain_grid(P.L.ntiles);
  if (save) {
    DVD_CUDA_CALL(cudaFuncSetAttribute(mlp_chain_fwd_kernel<FX, FT, TD, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)kChainSmemBytes));
    dvd::launch(mlp_chain_fwd_kernel<FX, FT, TD, true>, grid, kThreadsMlp, kChainSmemBytes, st, P);
  } else {
    DVD_CUDA_CALL(cudaFuncSetAttribute(mlp_chain_fwd_kernel<FX, FT, TD, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)kChainSmemBytes));
    dvd::launch(mlp_chain_fwd_kernel<FX, FT, TD, false>, grid, kThreadsMlp, kChainSmemBytes, st, P);
  }
  DVD_CUDA_LAUNCH_CHECK("mlp_chain_fwd");
  return 0;
}

extern "C" int dvd_mlp_chain_fwd(const dvd_mlp_cfg* cfg, const void* packed_fwd, const float* bias, const float* p0,
                                 const float* t0, float dt, int n_eval, int n_acc, float* acc, float* s_steps,
                                 float* p_steps, void* save, long npx, long hw, void* stream) {
  int variant;
  if (int e = check_cfg_supported(cfg, &variant)) return e;
  DVD_ARG_CHECK(packed_fwd && bias && p0, "null pointer");
  DVD_ARG_CHECK(!cfg->time_dependent || t0, "t0 required for a time-dependent field");
  DVD_ARG_CHECK(n_eval >= 1 && n_eval <= 64 && n_acc >= 0 && n_acc <= n_eval, "bad n_eval=%d / n_acc=%d", n_eval, n_acc);
  DVD_ARG_CHECK(npx > 0 && hw > 0 && npx % hw == 0, "npx must be a multiple of hw");
  DVD_ARG_CHECK(!save || p_steps, "p_steps required when save is given");
  DVD_ARG_CHECK(cfg->sf_mag_div != 0.f, "sf_mag_div must be non-zero");
  FwdParams P;
  P.wf = (const uint8_t*)packed_fwd; P.bias = bias; P.p0 = p0; P.t0 = t0; P.dt = dt;
  P.n_eval = n_eval; P.n_acc = n_acc; P.acc = acc; P.s_steps = s_steps; P.p_steps = p_steps;
  P.save = (uint8_t*)save; P.npx = npx; P.hw = hw; P.L = make_layout(*cfg, npx); P.cfg = *cfg;
  cudaStream_t st = (cudaStream_t)stream;
  if (variant == 0) return launch_fwd<16, 16, true>(P, save != nullptr, st);
  if (variant == 1) return launch_fwd<16, 0, false>(P, save != nullptr, st);
  return launch_fwd<kRuntime, 0, false>(P, save != nullptr, st);
}

template <int FX, int FT, bool TD, int KPAD>
static int launch_dgrad(const DgradParams& P, cudaStream_t st) {
  if (P.ord) {
    const int grid = chain_grid(P.L.ntiles);
    DVD_CUDA_CALL(cudaFuncSetAttribute(mlp_dgrad_kernel<FX, FT, TD, KPAD, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)kChainSmemBytes));
    dvd::launch(mlp_dgrad_kernel<FX, FT, TD, KPAD, true>, grid, kThreadsMlp, kChainSmemBytes, st, P);
    DVD_CUDA_LAUNCH_CHECK("mlp_dgrad<ordered>");
    return P.g_bias5 ? launch_ordered_sum(P.ord, grid * 8, 3, P.g_bias5, 3, nullptr, st) : 0;
  }
  DVD_CUDA_CALL(cudaFuncSetAttribute(mlp_dgrad_kernel<FX, FT, TD, KPAD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)kChainSmemBytes));
  dvd::launch(mlp_dgrad_kernel<FX, FT, TD, KPAD>, chain_grid(P.L.ntiles), kThreadsMlp, kChainSmemBytes, st, P);
  DVD_CUDA_LAUNCH_CHECK("mlp_dgrad");
  return 0;
}

static int mlp_dgrad(const dvd_mlp_cfg* cfg, const void* packed_bwd, const float* p_e, const float* t0, float dt,
                     int e, int use_g_acc, const float* g_acc, const float* g_step, const float* a_in,
                     float* a_out, const void* save_e, void* dy_scratch, float* g_bias5, long npx, long hw,
                     void* ws, size_t ws_bytes, void* stream) {
  int variant;
  if (int er = check_cfg_supported(cfg, &variant)) return er;
  DVD_ARG_CHECK(packed_bwd && p_e && save_e && dy_scratch, "null pointer");
  DVD_ARG_CHECK(!cfg->time_dependent || t0, "t0 required for a time-dependent field");
  DVD_ARG_CHECK(e >= 0 && e < 64, "bad eval index");
  DVD_ARG_CHECK(npx > 0 && hw > 0 && npx % hw == 0, "npx must be a multiple of hw");
  DgradParams P;
  P.wb = (const uint8_t*)packed_bwd; P.p_e = p_e; P.t0 = t0; P.dt = dt; P.e = e; P.use_g_acc = use_g_acc;
  P.g_acc = g_acc; P.g_step = g_step; P.a_in = a_in; P.a_out = a_out; P.save_e = (const uint8_t*)save_e;
  P.dy = (uint8_t*)dy_scratch; P.g_bias5 = g_bias5; P.npx = npx; P.hw = hw; P.L = make_layout(*cfg, npx); P.cfg = *cfg;
  P.ord = (float*)ws;
  DVD_ARG_CHECK(!ws || ws_bytes >= (size_t)chain_grid(P.L.ntiles) * 8 * 3 * sizeof(float),
                "ordered MLP data gradient: the workspace needs dvd_ordered_workspace_bytes(DVD_ORD_MLP_DGRAD) bytes");
  cudaStream_t st = (cudaStream_t)stream;
  if (variant == 0) return launch_dgrad<16, 16, true, Embed<16, 16, true>::KPAD>(P, st);
  if (variant == 1) return launch_dgrad<16, 0, false, Embed<16, 0, false>::KPAD>(P, st);
  switch (P.L.kpad0) {
    case 64: return launch_dgrad<kRuntime, 0, false, 64>(P, st);
    case 128: return launch_dgrad<kRuntime, 0, false, 128>(P, st);
    case 192: return launch_dgrad<kRuntime, 0, false, 192>(P, st);
    default: return launch_dgrad<kRuntime, 0, false, 256>(P, st);   // kpad0 <= DVD_MLP_MAX_NIN (check_cfg_supported)
  }
}

static int mlp_wgrad(const dvd_mlp_cfg* cfg, const void* save_e, const void* dy_scratch, float* const* g_w,
                     float* const* g_b, long npx, void* ws, size_t ws_bytes, void* stream) {
  int variant;
  if (int er = check_cfg_supported(cfg, &variant)) return er;
  DVD_ARG_CHECK(save_e && dy_scratch && g_w && g_b, "null pointer");
  DVD_ARG_CHECK(npx > 0, "npx must be positive");
  MlpLayout L = make_layout(*cfg, npx);
  const uint8_t* sv = (const uint8_t*)save_e;
  const uint8_t* dy = (const uint8_t*)dy_scratch;
  WgradParams P;
  P.nq = L.nq;
  P.ord = nullptr;
  P.nsplit = 0;
  int nj = 0;
  for (int l = 0; l < kLayers; ++l) {
    DVD_ARG_CHECK(g_w[l] != nullptr, "null g_w[%d]", l);
    const size_t x_plane = (size_t)L.nq * blk_bytes(rows_x(L, l)), y_plane = (size_t)L.nq * blk_bytes(rows_dy(l));
    for (int mh = 0; mh < 2; ++mh) {
      WgradJob& J = P.job[nj++];
      if (l < 5) {
        DVD_ARG_CHECK(g_b[l] != nullptr, "null g_b[%d]", l);
        J.a_hi = dy + L.dy_off[l]; J.a_lo = J.a_hi + y_plane; J.a_blk = blk_bytes(kWidth); J.a_row_off = mh * 2 * 8192;
        J.b_hi = sv + L.xs_off[l]; J.b_lo = J.b_hi + x_plane; J.b_blk = blk_bytes(rows_x(L, l)); J.n = rows_x(L, l);
        J.out = g_w[l]; J.ld = layer_in(L, l); J.transposed = 0; J.m_off = mh * 128; J.m_valid = kWidth;
        J.n_valid = layer_in(L, l); J.bias_out = g_b[l];
      } else {
        J.a_hi = sv + L.xs_off[5]; J.a_lo = J.a_hi + x_plane; J.a_blk = blk_bytes(kWidth); J.a_row_off = mh * 2 * 8192;
        J.b_hi = dy + L.dy_off[5]; J.b_lo = J.b_hi + y_plane; J.b_blk = blk_bytes(16); J.n = 16;
        J.out = g_w[5]; J.ld = kWidth; J.transposed = 1; J.m_off = mh * 128; J.m_valid = kWidth; J.n_valid = 3;
        J.bias_out = nullptr;
      }
      DVD_ARG_CHECK(J.n == 256 || J.n == 192 || J.n == 144 || J.n == 128 || J.n == 112 || J.n == 64 || J.n == 16,
                    "no weight-gradient kernel for a %d-channel operand", J.n);
    }
  }
  int ksplit = num_sms() / nj;
  if (ksplit < 1) ksplit = 1;
  if ((long)ksplit > L.nq) ksplit = (int)L.nq;
  if (ws) {
    // ordered: the same split, partial tiles through the workspace, added in split order by mlp_wgrad_reduce_kernel
    DVD_ARG_CHECK(ws_bytes >= (size_t)nj * ksplit * kOrdSlab * sizeof(float),
                  "ordered MLP weight gradient: the workspace needs dvd_ordered_workspace_bytes(DVD_ORD_MLP_WGRAD) bytes");
    P.ord = (float*)ws;
    P.nsplit = ksplit;
    DVD_CUDA_CALL(cudaFuncSetAttribute(mlp_wgrad_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kWgradSmemBytes));
    dvd::launch(mlp_wgrad_kernel<true>, dim3(nj, ksplit), kThreadsWgrad, kWgradSmemBytes, (cudaStream_t)stream, P);
    DVD_CUDA_LAUNCH_CHECK("mlp_wgrad<ordered>");
    const long per = (L.nq + ksplit - 1) / ksplit;
    const int nparts = (int)((L.nq + per - 1) / per);
    dvd::launch(mlp_wgrad_reduce_kernel, dim3(nj, 128), 256, 0, (cudaStream_t)stream, P, nparts);
    DVD_CUDA_LAUNCH_CHECK("mlp_wgrad_reduce_kernel");
    return 0;
  }
  DVD_CUDA_CALL(cudaFuncSetAttribute(mlp_wgrad_kernel<>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kWgradSmemBytes));
  dvd::launch(mlp_wgrad_kernel<>, dim3(nj, ksplit), kThreadsWgrad, kWgradSmemBytes, (cudaStream_t)stream, P);
  DVD_CUDA_LAUNCH_CHECK("mlp_wgrad");
  return 0;
}

extern "C" int dvd_mlp_dgrad(const dvd_mlp_cfg* cfg, const void* packed_bwd, const float* p_e, const float* t0, float dt,
                             int e, int use_g_acc, const float* g_acc, const float* g_step, const float* a_in,
                             float* a_out, const void* save_e, void* dy_scratch, float* g_bias5, long npx, long hw,
                             void* stream) {
  return mlp_dgrad(cfg, packed_bwd, p_e, t0, dt, e, use_g_acc, g_acc, g_step, a_in, a_out, save_e, dy_scratch, g_bias5, npx, hw,
                   nullptr, 0, stream);
}
extern "C" int dvd_mlp_dgrad_ordered(const dvd_mlp_cfg* cfg, const void* packed_bwd, const float* p_e, const float* t0,
                                     float dt, int e, int use_g_acc, const float* g_acc, const float* g_step,
                                     const float* a_in, float* a_out, const void* save_e, void* dy_scratch,
                                     float* g_bias5, long npx, long hw, void* ws, size_t ws_bytes, void* stream) {
  DVD_ARG_CHECK(ws != nullptr, "dvd_mlp_dgrad_ordered: null workspace");
  return mlp_dgrad(cfg, packed_bwd, p_e, t0, dt, e, use_g_acc, g_acc, g_step, a_in, a_out, save_e, dy_scratch, g_bias5, npx, hw,
                   ws, ws_bytes, stream);
}
extern "C" int dvd_mlp_wgrad(const dvd_mlp_cfg* cfg, const void* save_e, const void* dy_scratch, float* const* g_w,
                             float* const* g_b, long npx, void* stream) {
  return mlp_wgrad(cfg, save_e, dy_scratch, g_w, g_b, npx, nullptr, 0, stream);
}
extern "C" int dvd_mlp_wgrad_ordered(const dvd_mlp_cfg* cfg, const void* save_e, const void* dy_scratch, float* const* g_w,
                                     float* const* g_b, long npx, void* ws, size_t ws_bytes, void* stream) {
  DVD_ARG_CHECK(ws != nullptr, "dvd_mlp_wgrad_ordered: null workspace");
  return mlp_wgrad(cfg, save_e, dy_scratch, g_w, g_b, npx, ws, ws_bytes, stream);
}

extern "C" int dvd_acc_reg(const float* s0, const float* s1, float acc_mul, float gscale, float* g_s0, float* g_s1,
                           float* partials, float* loss_out, long numel, void* stream) {
  DVD_ARG_CHECK(s0 && s1 && partials && loss_out && numel > 0, "bad arguments");
  const float inv = 1.0f / ((float)numel + 1e-6f);
  int nb = (int)((numel + 255) / 256);
  if (nb > 1024) nb = 1024;
  dvd::launch(acc_reg_kernel, nb, 256, 0, (cudaStream_t)stream, s0, s1, acc_mul * inv * gscale, g_s0, g_s1, partials, numel);
  DVD_CUDA_LAUNCH_CHECK("acc_reg");
  dvd::launch(acc_reg_final_kernel, 1, 256, 0, (cudaStream_t)stream, partials, nb, acc_mul * inv, loss_out);
  DVD_CUDA_LAUNCH_CHECK("acc_reg_final");
  return 0;
}
