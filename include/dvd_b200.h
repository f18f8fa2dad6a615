/*
 * dvd_b200.h — C ABI of libdvd_b200.so (H100 / sm_90a hot path of google/dynamic-video-depth).
 *
 * The reference has NO native boundary on this path: it is Python over ATen
 * (SURVEY.md §8(b), last row). These entry points are what a maintainer binds from the
 * reference's Python modules with ctypes (see INTEGRATION.md); each one names the reference
 * code it replaces (paths relative to the reference tree).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to a caller-allocated, contiguous fp32 buffer
 *     (16-byte aligned unless noted); nothing is allocated or freed by the library, no ownership moves;
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*); no call synchronises;
 *   - return value: 0 on success, negative = argument error, positive = cudaError_t;
 *     dvd_last_error() returns a thread-local message for the last non-zero return;
 *   - image tensors are channel-planar [B,C,H,W]; optical flow is [B,H,W,2]; masks are [B,H,W].
 *   - `poses` is [B,48] fp32: Kinv[9] K[9] R1[9] R2[9] t1[3] t2[3] pad[6], matrices row-major in
 *     COLUMN-vector convention (R = camera-to-world). The reference stores the transposes
 *     (scripts/preprocess/davis/generate_sequence_midas.py:61-76); dvd_b200.ops.pack_poses converts.
 */
#ifndef DVD_B200_H_
#define DVD_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DVD_POSE_STRIDE 48

/* loss configuration — mirrors the live flags of models/scene_flow_motion_field.py:33-67,285-324 */
typedef struct dvd_loss_cfg {
  int   midas;          /* 1: mask *= [d1<100]·[warped z<100]   (smf.py:286-289) */
  int   warm;           /* 1: L2 flow criterion (epoch <= warm_sf), 0: L1  (smf.py:291) */
  int   disp_mode;      /* 0: --use_disp, 1: --use_disp_ratio, 2: |z1 - z2|  (smf.py:140-150) */
  int   second_is_disp; /* 1: loss uses disp_loss (--use_disp), 0: uses sf_loss (smf.py:310-319) */
  float flow_mul;       /* --flow_mul */
  float disp_mul;       /* --disp_mul */
} dvd_loss_cfg;

/* scalars written by dvd_reproject_loss_fwd (device, 8 floats) */
enum { DVD_S_FLOW = 0, DVD_S_DISP = 1, DVD_S_SF = 2, DVD_S_LOSS = 3, DVD_S_MASKSUM = 4,
       DVD_S_CF = 5 /* flow_mul/N */, DVD_S_CD = 6 /* disp_mul/N */, DVD_S_RSVD = 7 };

const char* dvd_last_error(void);
int dvd_version(void);
/* sizeof of the structs passed by pointer: 0 dvd_loss_cfg, 1 dvd_mlp_cfg, 2 dvd_conv_desc, 3 dvd_pack_item, 4 dvd_vis_panel,
 * 5 dvd_vis_map (-1 otherwise) */
long dvd_struct_size(int which);
/* number of fp32 partial-sum slots dvd_reproject_loss_fwd needs in `partials` for a given shape */
int dvd_reproject_partials_size(int B, int H, int W);

/* W3  unproject_ptcld.forward  (losses/scene_flow_projection.py:48-67):  P = R·(d·Kinv·c) + t
 * which = 1 uses (R1,t1), which = 2 uses (R2,t2).  depth [B,1,H,W] -> P [B,3,H,W]            */
int dvd_unproject_fwd(const float* depth, const float* poses, float* P,
                      int B, int H, int W, int which, void* stream);
/* adjoint: gP [B,3,H,W] -> gdepth [B,1,H,W]  (overwrites) */
int dvd_unproject_bwd(const float* gP, const float* poses, float* gdepth,
                      int B, int H, int W, int which, void* stream);

/* W1+W2+L1 fused forward: flow_by_depth.forward + scene_flow_projection_slack.forward
 * (losses/scene_flow_projection.py:95-153,204-278) + Model._calc_loss
 * (models/scene_flow_motion_field.py:285-324) without materialising any per-pixel tensor.
 *   depth_1, depth_2 [B,1,H,W]; flow_1_2 [B,H,W,2]; mask_2 [B,H,W]; sf [B,3,H,W]
 *   partials: scratch, dvd_reproject_partials_size() floats; scalars: 8 floats (enum above). */
int dvd_reproject_loss_fwd(const float* depth_1, const float* depth_2, const float* flow_1_2,
                           const float* mask_2, const float* sf, const float* poses,
                           const dvd_loss_cfg* cfg, float* partials, float* scalars,
                           int B, int H, int W, void* stream);

/* adjoint of the above w.r.t. sf (== w.r.t. global_p1, both enter only as P1+sf) and depth_2.
 *   g_sf [B,3,H,W] overwritten; g_depth_2 [B,1,H,W] zero-filled then scatter-added (may be NULL
 *   when the depth net is frozen — warm-up phase, smf.py:154-164). The upstream gradient is
 *   gscale (host, e.g. `steps` for --weight_steps, smf.py:189-190) times *gscale_dev (device
 *   scalar, may be NULL = 1) so autograd's grad_output never needs a host read-back.          */
int dvd_reproject_loss_bwd(const float* depth_1, const float* depth_2, const float* flow_1_2,
                           const float* mask_2, const float* sf, const float* poses,
                           const dvd_loss_cfg* cfg, const float* scalars, float gscale,
                           const float* gscale_dev, float* g_sf, float* g_depth_2,
                           int B, int H, int W, void* stream);

/* materialise every per-pixel tensor the two reference modules return (visualised batches and the
 * operator-level drop-in). Any output pointer may be NULL. All channel-planar:
 *   global_p1, sf_by_depth, warped_global_p2, warped_p2_camera_2, p1_camera_2 : [B,3,H,W]
 *   dflow_1_2, staticflow_1_2 : [B,2,H,W];  depth_image_1_2, depth_warp_1_2 : [B,1,H,W]      */
int dvd_reproject_materialize(const float* depth_1, const float* depth_2, const float* flow_1_2,
                              const float* sf, const float* poses,
                              float* global_p1, float* sf_by_depth, float* warped_global_p2,
                              float* warped_p2_camera_2, float* p1_camera_2, float* dflow_1_2,
                              float* staticflow_1_2, float* depth_image_1_2, float* depth_warp_1_2,
                              int B, int H, int W, void* stream);

/* adjoint of dvd_reproject_materialize for arbitrary cotangents on its nine outputs (any may be NULL = zero):
 * keeps the operator-level mirrors of flow_by_depth / scene_flow_projection_slack differentiable.
 * g_depth_1, g_sf overwritten; g_depth_2 zero-filled then scatter-added; each may be NULL.            */
int dvd_reproject_materialize_bwd(const float* depth_1, const float* depth_2, const float* flow_1_2,
                                  const float* sf, const float* poses, const float* g_global_p1,
                                  const float* g_sf_by_depth, const float* g_warped_global_p2,
                                  const float* g_warped_p2_camera_2, const float* g_p1_camera_2,
                                  const float* g_dflow_1_2, const float* g_staticflow_1_2,
                                  const float* g_depth_image_1_2, const float* g_depth_warp_1_2,
                                  float* g_depth_1, float* g_depth_2, float* g_sf, int B, int H, int W,
                                  void* stream);

/* self-test of the wgmma building blocks (one CTA): D[128,N] = A[128,K]·B[N,K]^T, fp32 row-major
 * in/out, K in {64,128}, N in {16, 64, 144, 256}; mode 0 = both operands K-major in shared memory,
 * 1 = A from registers, 2 = both MN-major (128-byte swizzle), 3 = both MN-major (no swizzle);
 * passes 1 = bf16, 3 = bf16x3 split (fp32-grade). Not on the hot path.                          */
int dvd_selftest_umma(const float* A, const float* B, float* D, int K, int N, int mode, int passes,
                      void* stream);

/* ---- scene-flow MLP (M1-M4, L2) ---------------------------------------------------------------
 * networks/blocks.py:19-34 (PeriodicEmbed), networks/sceneflow_field.py:20-53 (SceneFlowFieldNet:
 * 1x1 convs n_in->256->256->256->256->256->3, LeakyReLU 0.2), models/scene_flow_motion_field.py:346-367
 * (forward_sf_net: / sf_mag_div; forward_sf_net_multi_step: Euler chain) and :326-344 (_opt_reg).
 *
 * All GEMMs run on wgmma tensor cores with fp32 emulated as two bf16 planes (x = hi + lo,
 * D += Ahi*Bhi + Alo*Bhi + Ahi*Blo, fp32 accumulate): error ~2e-5, i.e. tighter than the
 * TF32 path the reference itself takes on a GPU (cudnn.allow_tf32 default).
 * Fixed by the reference ctor (smf.py:107): width 256, 4 hidden layers, 3 outputs. The positional encoding
 * follows --n_freq_xyz, --n_freq_t and --time_dependent (networks/sceneflow_field.py:22-35): the first layer
 * reads nin = (time_dependent ? 1 + 2 n_freq_t : 0) + 3 + 6 n_freq_xyz features, and every configuration
 * with nin <= DVD_MLP_MAX_NIN runs (a count of 0 is the reference's nn.Identity). (16, 16, time-dependent)
 * and (16, time-independent) have kernels compiled for their counts; every other one runs the generic kernels,
 * whose first layer is padded to a multiple of 64 input channels. Larger configurations return -2.          */
#define DVD_MLP_MAX_NIN 256
#define DVD_MLP_MAX_FREQ_XYZ 42   /* (DVD_MLP_MAX_NIN - 3) / 6 */
#define DVD_MLP_MAX_FREQ_T 126    /* (DVD_MLP_MAX_NIN - 4) / 2 */
typedef struct dvd_mlp_cfg {
  int   n_freq_xyz;      /* --n_freq_xyz (16) */
  int   n_freq_t;        /* --n_freq_t   (16); ignored unless time_dependent */
  int   time_dependent;  /* --time_dependent */
  float sf_mag_div;      /* --sf_mag_div (100) */
  float freq_xyz[DVD_MLP_MAX_FREQ_XYZ];  /* torch.linspace(1, n_freq+1, n_freq) in fp32 (networks/blocks.py:23-24) */
  float freq_t[DVD_MLP_MAX_FREQ_T];
} dvd_mlp_cfg;

/* sizes (bytes) of the caller-allocated scratch buffers for a given configuration */
size_t dvd_mlp_packed_weights_bytes(const dvd_mlp_cfg* cfg);            /* one image (fwd or bwd) */
size_t dvd_mlp_save_bytes_per_eval(const dvd_mlp_cfg* cfg, long npx);   /* activations + masks of one eval */
size_t dvd_mlp_dy_bytes(const dvd_mlp_cfg* cfg, long npx);              /* dY scratch of one eval */

/* fp32 weights -> bf16 (hi,lo) planes in the wgmma shared-memory image (SWIZZLE_128B, K-major blocks),
 * once per optimiser step. w[l] = convs.{l}.conv.weight [out,in] row-major, l = 0..5 (device ptrs,
 * host array). packed_fwd feeds the forward chain, packed_bwd (transposed) the dgrad chain.      */
int dvd_mlp_pack_weights(const dvd_mlp_cfg* cfg, const float* const* w, void* packed_fwd, void* packed_bwd,
                         void* stream);

/* Euler chain forward (M1-M4): for i < n_eval: s_i = MLP(p_i, t_i)/sf_mag_div; p_{i+1} = p_i + s_i;
 * t_{i+1} = t_i + dt.  acc = sum_{i<n_acc} s_i.
 *   p0 [B,3,H,W], t0 [B,1,H,W] (NULL if not time_dependent), npx = B*H*W, hw = H*W
 *   bias: fp32 [5*256 + 16] = b_0..b_4, b_5 (3 used)
 *   acc [B,3,H,W] (may be NULL), s_steps [n_eval,B,3,H,W] (may be NULL)
 *   save (may be NULL = inference): n_eval * dvd_mlp_save_bytes_per_eval(); p_steps [n_eval,B,3,H,W]
 *   must be non-NULL when save is.                                                              */
int dvd_mlp_chain_fwd(const dvd_mlp_cfg* cfg, const void* packed_fwd, const float* bias,
                      const float* p0, const float* t0, float dt, int n_eval, int n_acc,
                      float* acc, float* s_steps, float* p_steps, void* save,
                      long npx, long hw, void* stream);

/* backward of ONE eval e of the chain (call for e = n_eval-1 .. 0):
 *   gs = (e < n_acc ? g_acc : 0) + g_step + a_in      (each [B,3,H,W], any may be NULL)
 *   a_out = a_in + J_e^T gs                            (a_out may alias a_in)
 *   writes dY scratch (for dvd_mlp_wgrad) and atomically accumulates g_bias5[3].                */
int dvd_mlp_dgrad(const dvd_mlp_cfg* cfg, const void* packed_bwd, const float* p_e, const float* t0,
                  float dt, int e, int use_g_acc, const float* g_acc, const float* g_step,
                  const float* a_in, float* a_out, const void* save_e, void* dy_scratch,
                  float* g_bias5, long npx, long hw, void* stream);

/* weight/bias gradients of ONE eval: g_w[l] += dY_l^T X_l, g_b[l] += sum dY_l (l = 0..4), g_w[5]
 * likewise (g_b[5] is accumulated by dvd_mlp_dgrad). g_w / g_b: host arrays of 6 device pointers
 * with the layout of w / bias; accumulated with fp32 atomics (zero them once per step).          */
int dvd_mlp_wgrad(const dvd_mlp_cfg* cfg, const void* save_e, const void* dy_scratch,
                  float* const* g_w, float* const* g_b, long npx, void* stream);

/* L2  Model._opt_reg (smf.py:326-344) on the chain's own s_0, s_1:
 *   loss = acc_mul * sum|s1 - s0| / (numel + 1e-6);  g_s0 = -c*sign(s1-s0), g_s1 = +c*sign(s1-s0)
 *   partials: >= 1024 floats scratch; loss_out: 1 float (device).                                */
int dvd_acc_reg(const float* s0, const float* s1, float acc_mul, float gscale, float* g_s0, float* g_s1,
                float* partials, float* loss_out, long numel, void* stream);

/* O1  torch.optim.Adam x2 (models/netinterface.py:96-97,127-129; smf.py:113-115,212-213) as one
 * launch over a flat fp32 buffer: amsgrad=False, weight_decay=0; `step` counts from 1; the
 * gradient is multiplied by gscale first (1/world_size after a sum all-reduce).                */
int dvd_adam_flat(float* p, const float* g, float* m, float* v, long n, float lr, float beta1,
                  float beta2, float eps, int step, float gscale, void* stream);
/* the same update with the step counter on the DEVICE (step_state: 4 floats {int step bits, 1-b1^t, sqrt(1-b2^t), -}; the call
 * increments it first), so that a captured CUDA graph of the step replays with the right bias correction.                  */
int dvd_adam_flat_dev(float* p, const float* g, float* m, float* v, long n, float lr, float beta1,
                      float beta2, float eps, float* step_state, float gscale, void* stream);

/* ---- channels-last (NHWC) glue of the depth nets (D1/D2): tensors are [P = N*H*W pixels][C], C % 4 == 0 ----
 * eval-mode BatchNorm (the only mode on this path, smf.py:157,168) + optional residual add + optional ReLU:
 *   y = x*g*rsqrt(var+eps) + (beta - mean*g*rsqrt(var+eps)) (+ res) ; ReLU
 * replaces torchvision Bottleneck's bn{1,2,3} + relu + `out += identity` and the ATen clamp / add kernels.      */
int dvd_bn_act_fwd(const float* x, const float* res, const float* gamma, const float* beta, const float* mean,
                   const float* var, float eps, float* y, long P, int C, int relu, void* stream);
/* backward: gm = g*[y>0]; gx = gm*scale; gres = gm (may be NULL); ggamma/gbeta are ACCUMULATED (zero them first) */
int dvd_bn_act_bwd(const float* g, const float* x, const float* y, const float* gamma, const float* mean,
                   const float* var, float eps, float* gx, float* gres, float* ggamma, float* gbeta,
                   long P, int C, int relu, void* stream);
/* x2 bilinear up-sampling (third_party/midas_blocks.py:95-97 align_corners=False; :164-166 align_corners=True;
 * hourglass UpsamplingBilinear2d = True), NHWC [N,H,W,C] -> [N,2H,2W,C], and its adjoint.                      */
int dvd_upsample2x_fwd(const float* x, float* y, int N, int H, int W, int C, int align_corners, int round_out, void* stream);
int dvd_upsample2x_bwd(const float* g, float* gx, int N, int H, int W, int C, int align_corners, int round_out, void* stream);
/* round_out = 1: results stored rounded to TF32 (round-to-nearest) - they feed a tensor-core convolution (see below) */

/* ---- D1 / D1' depth-net convolutions, general form (csrc/conv2d_tc.cu) -------------------------------------------------
 * One implicit-GEMM wgmma (TF32) kernel family for every convolution class of MiDaS / ResNeXt101-32x8d
 * (third_party/MiDaS.py:188-246, third_party/midas_blocks.py:48-68,102-168, torchvision Bottleneck): dense and grouped,
 * stride 1 and 2, forward and data gradient (tap table + sub-pixel phases), plus the weight gradient.
 * ROUNDED-OPERAND CONTRACT: x (and gy) must hold values already rounded to TF32 with round-to-nearest - every kernel of this
 * library that produces an activation or a gradient offers a `round` switch, and dvd_round_tf32 does it for foreign tensors -
 * because the tensor core itself truncates the low 13 mantissa bits (a -7e-4 bias per layer otherwise).                    */
#define DVD_CONV_MAX_TAPS 128
typedef struct dvd_conv_desc {
  int N, H, W, Cin;            /* input tensor x [N,H,W,Cin] (NHWC)                                                    */
  int OH, OW, Cout;            /* output grid of THIS launch (tile space) and output channels                          */
  int stride;                  /* 1 | 2: tap t of output pixel (oh,ow) reads x[stride*oh + dy[t], stride*ow + dx[t]] (zero outside) */
  int ntaps;
  int kblock;                  /* 0: dense (all Cin per output channel); else block-diagonal (grouped) with this block size */
  int YH, YW;                  /* spatial size of the tensors y / res / res2 / mask                                    */
  int oy_mul, oy_add, ox_mul, ox_add;   /* output pixel (oh,ow) is stored at y[oh*oy_mul+oy_add, ow*ox_mul+ox_add]     */
  int relu;                    /* ReLU after the residual adds                                                         */
  int round_out;               /* store TF32-rounded values (the output feeds another convolution)                     */
  float bn_eps;
  signed char dy[DVD_CONV_MAX_TAPS], dx[DVD_CONV_MAX_TAPS];
  unsigned char wt[DVD_CONV_MAX_TAPS];  /* index of the tap's [rows][cols] slice in the packed weight image            */
} dvd_conv_desc;

/* y = round( [mask > 0] * relu( conv(x, w_img) * scale + shift + res + res2 ) )
 * scale/shift fold the conv bias and / or an eval-mode BatchNorm (gamma, beta, mean, var: all four or none); res, res2, mask
 * are NHWC tensors shaped like y, each may be NULL. Needs Cin % 32 == 0, Cout % 16 == 0 (Cout <= 256 or 256 | Cout).      */
int dvd_conv2d_nhwc(const dvd_conv_desc* desc, const float* x, const float* w_img, const float* bias, const float* bn_gamma,
                    const float* bn_beta, const float* bn_mean, const float* bn_var, const float* res, const float* res2,
                    const float* mask, float* y, void* stream);

/* The same with an exchange area for the stream-K schedule (layers whose tile count leaves much of the last wave idle are cut
 * into equal K ranges per SM; tiles shared by several SMs are summed through this area). `workspace`: at least
 * dvd_conv2d_workspace_bytes() bytes of device memory, 16-byte aligned, ZEROED ONCE by the caller and then left to the library;
 * launches that share a workspace must be ordered on one stream. NULL = whole tiles only (dvd_conv2d_nhwc).                  */
size_t dvd_conv2d_workspace_bytes(void);
/* host restatement of the stream-K partition (no GPU needed): out[c] = first tile-major K-step of cluster c, out[n_clusters] = ntiles * ksteps */
int dvd_conv2d_streamk_bounds(int ntiles, int ksteps, int n_clusters, long* out);
int dvd_conv2d_nhwc_ws(const dvd_conv_desc* desc, const float* x, const float* w_img, const float* bias, const float* bn_gamma,
                       const float* bn_beta, const float* bn_mean, const float* bn_var, const float* res, const float* res2,
                       const float* mask, float* y, void* workspace, size_t workspace_bytes, void* stream);

/* weight[co, ci_local, ky, kx] (element strides given; groups of Cin/groups in-channels) -> TF32-rounded image
 *   w_fwd: forward        [k*k][Cout][Cin or kblock]
 *   w_bwd: data gradient  [k*k][Cin][Cout or kblock], multiplied by gamma*rsqrt(var+eps) of the out-channel when given
 * (either may be NULL; both are written by one launch)
 * grouped convolutions (groups > 1) are packed block-diagonally with `kblock` channels per block (kblock = 0 when dense).   */
int dvd_conv2d_pack(const float* weight, long stride_co, long stride_ci, long stride_ky, long stride_kx, float* w_fwd,
                    float* w_bwd, int Cout, int Cin, int ksize, int groups, int kblock, const float* bn_gamma,
                    const float* bn_var, float bn_eps, void* stream);

/* The same for every layer of a net in ONE launch. `items_dev` is a table of n_items entries in DEVICE memory (the pointers in
 * it are device pointers; the caller rebuilds it when a tensor moves). Entry i owns grid blocks [blk0, blk0 + blocks_i) with
 * blocks_i = dvd_conv2d_pack_blocks(...) (one block per 32 x 32 channel tile and tap; -1 unless Cout, Cin and kblock are
 * multiples of 32) and blk0 the running sum; total_blocks = the sum over all entries.                                           */
typedef struct dvd_pack_item {
  const float* weight;      /* [Cout, Cin/groups, k, k], element strides below */
  float* w_fwd;             /* forward image or NULL */
  float* w_bwd;             /* data-gradient image or NULL (skipped when want_bwd == 0) */
  const float* bn_gamma;    /* eval-BatchNorm scale folded into w_bwd, or NULL */
  const float* bn_var;
  long s_co, s_ci, s_ky, s_kx;
  long blk0;
  int Cout, Cin, ksize, groups, kblock;
  float bn_eps;
} dvd_pack_item;
long dvd_conv2d_pack_blocks(int Cout, int Cin, int ksize, int groups, int kblock);
int dvd_conv2d_pack_batch(const dvd_pack_item* items_dev, int n_items, long total_blocks, int want_bwd, void* stream);

/* dweight[co, ci_local, ky, kx] += sc[co] * sum_px gy[px, co] * x[stride*px + (dy,dx)(tap), ci]   (fp32 reductions, any strides)
 * for the taps of `desc` (wt[t] = ky*ksize + kx). With an eval-mode BatchNorm behind the convolution, gy is the UN-scaled
 * masked gradient, sc = gamma*rsqrt(var+eps), and dgamma[co] += rsqrt(var+eps) * <weight[co], sum gy x> (weight = the
 * parameter tensor, same strides as dweight). colsum (optional, not with swapped operands): colsum[co] += sum_px gy[px, co] - the
 * conv-bias or BatchNorm-beta gradient - from one extra N = 16 MMA per K step against a ones operand; with bn_mean, dgamma also
 * receives -mean * rsqrt(var+eps) * that sum. Needs (128 | Cout and 32 | Cin) or (128 | Cin and 32 | Cout, no BatchNorm);
 * grouped: Cin == Cout, 128 | C.                                                                                              */
int dvd_conv2d_wgrad(const dvd_conv_desc* desc, const float* x, const float* gy, float* dweight, const float* weight,
                     long stride_co, long stride_ci, long stride_ky, long stride_kx, int ksize, int groups,
                     const float* bn_gamma, const float* bn_var, float* dgamma, float* colsum, const float* bn_mean,
                     void* stream);

/* ---- CUDA-core members of the MiDaS path (csrc/depth_ops.cu), NHWC fp32 -------------------------------------------------- */
/* y = round-to-nearest TF32 of x (n % 4 == 0): entry of foreign tensors into the rounded-operand contract                   */
int dvd_round_tf32(const float* x, float* y, long n, void* stream);
/* gm = g * [y > 0] (y NULL: gm = g), optionally TF32-rounded and optionally stored (gm NULL: sums only);
 * colsum[c] += sum_p gm[p,c] (bias / BatchNorm-beta gradient); dgamma[c] -= mean[c]*rsqrt(var[c]+eps)*sum_p gm[p,c]          */
int dvd_relu_bwd_colsum(const float* g, const float* y, float* gm, float* colsum, const float* bn_mean, const float* bn_var,
                        float bn_eps, float* dgamma, long P, int C, int round_out, void* stream);
/* torchvision ResNet.maxpool = MaxPool2d(3, stride 2, padding 1): x [N,H,W,C] -> y [N,OH,OW,C], idx = window position of the
 * (first) maximum; backward gathers g through idx into gx [N,H,W,C] (overwrites).                                            */
int dvd_maxpool3x3s2_fwd(const float* x, float* y, unsigned char* idx, int N, int H, int W, int C, void* stream);
int dvd_maxpool3x3s2_bwd(const float* g, const unsigned char* idx, float* gx, int N, int H, int W, int C, void* stream);
/* ResNeXt stem on the raw image: y = relu(bn1(conv1((x - mean)/std)))  (third_party/MiDaS.py:213-218; torchvision ResNet.conv1
 * 7x7 stride 2 pad 3, 3 -> 64). x_nchw [N,3,H,W]; weight [64,3,7,7] with the given element strides; norm_mean3 / norm_std3 are
 * HOST pointers to 3 floats (NULL: no normalisation); y [N,OH,OW,64] NHWC.                                                    */
int dvd_stem_fwd(const float* x_nchw, const float* weight, long s_co, long s_ci, long s_ky, long s_kx, const float* bn_gamma,
                 const float* bn_beta, const float* bn_mean, const float* bn_var, float bn_eps, const float* norm_mean3,
                 const float* norm_std3, float* y, int N, int H, int W, int round_out, void* stream);
/* its parameter gradients from g = dL/dy (the ReLU mask is taken from a0 = y): dweight / dgamma / dbeta are ACCUMULATED;
 * scratch: 147*64 + 64 floats (zeroed by the call).                                                                           */
int dvd_stem_wgrad(const float* x_nchw, const float* g, const float* a0, const float* weight, float* dweight, long s_co,
                   long s_ci, long s_ky, long s_kx, const float* bn_gamma, const float* bn_mean, const float* bn_var,
                   float bn_eps, float* dgamma, float* dbeta, const float* norm_mean3, const float* norm_std3, float* scratch,
                   int N, int H, int W, void* stream);
/* head: depth[p] = 10000 / max(relu(<x[p,0:32], w> + b), 1e-2)  (scratch.output_conv[4..5] + MiDaS.py:240-242); backward
 * from g_depth: gx [P,32] overwritten (relu_mask = 1: times [x > 0], i.e. w.r.t. the pre-activation of the ReLU that produced x;
 * optionally TF32-rounded), gw[32] and gb[1] ACCUMULATED.                                                                     */
int dvd_head_fwd(const float* x, const float* w, const float* b, float* depth, long P, void* stream);
int dvd_head_bwd(const float* x, const float* w, const float* b, const float* g_depth, float* gx, float* gw, float* gb, long P,
                 int relu_mask, int round_out, void* stream);

/* ---- ordered reductions: run-to-run reproducible backward kernels ---------------------------------------------------------
 * Each *_ordered entry point takes the arguments of its namesake, then a workspace `ws` of `ws_bytes` bytes (16-byte aligned,
 * any content), then the stream, and computes the same outputs without floating-point atomics: a CTA's partial sums go to a slab
 * of the workspace and a second launch adds the slabs in a fixed order, so equal inputs give bitwise equal outputs on one GPU
 * model. Launch geometry and split counts are those of the namesake. Launches that may run concurrently need workspaces of
 * their own. dvd_ordered_workspace_bytes(site) is the size each site needs (0 for an unknown site); the re-projection
 * backward's depends on the shape (dvd_reproject_ordered_bytes). See DESIGN.md 2.11.                                          */
enum {
  DVD_ORD_CONV_WGRAD = 0,    /* dvd_conv2d_wgrad_ordered */
  DVD_ORD_MLP_WGRAD = 1,     /* dvd_mlp_wgrad_ordered */
  DVD_ORD_MLP_DGRAD = 2,     /* dvd_mlp_dgrad_ordered */
  DVD_ORD_CHANNEL_SUMS = 3,  /* dvd_relu_bwd_colsum_ordered, dvd_bn_act_bwd_ordered (C <= DVD_ORD_MAX_CHANNELS) */
  DVD_ORD_STEM = 4,          /* dvd_stem_wgrad_ordered */
  DVD_ORD_HEAD = 5           /* dvd_head_bwd_ordered */
};
#define DVD_ORD_CONV_MAX_CTAS 8192
#define DVD_ORD_MAX_CHANNELS 8192
size_t dvd_ordered_workspace_bytes(int site);
size_t dvd_reproject_ordered_bytes(int B, int H, int W);
int dvd_conv2d_wgrad_ordered(const dvd_conv_desc* desc, const float* x, const float* gy, float* dweight, const float* weight,
                             long stride_co, long stride_ci, long stride_ky, long stride_kx, int ksize, int groups,
                             const float* bn_gamma, const float* bn_var, float* dgamma, float* colsum, const float* bn_mean,
                             void* ws, size_t ws_bytes, void* stream);
int dvd_mlp_wgrad_ordered(const dvd_mlp_cfg* cfg, const void* save_e, const void* dy_scratch, float* const* g_w,
                          float* const* g_b, long npx, void* ws, size_t ws_bytes, void* stream);
int dvd_mlp_dgrad_ordered(const dvd_mlp_cfg* cfg, const void* packed_bwd, const float* p_e, const float* t0,
                          float dt, int e, int use_g_acc, const float* g_acc, const float* g_step,
                          const float* a_in, float* a_out, const void* save_e, void* dy_scratch,
                          float* g_bias5, long npx, long hw, void* ws, size_t ws_bytes, void* stream);
/* g_depth_2: each pixel's four bilinear taps are written as (target, contribution) pairs, sorted by target with a stable radix
 * sort and summed run by run in pixel order.                                                                                   */
int dvd_reproject_loss_bwd_ordered(const float* depth_1, const float* depth_2, const float* flow_1_2,
                                   const float* mask_2, const float* sf, const float* poses,
                                   const dvd_loss_cfg* cfg, const float* scalars, float gscale,
                                   const float* gscale_dev, float* g_sf, float* g_depth_2,
                                   int B, int H, int W, void* ws, size_t ws_bytes, void* stream);
int dvd_relu_bwd_colsum_ordered(const float* g, const float* y, float* gm, float* colsum, const float* bn_mean,
                                const float* bn_var, float bn_eps, float* dgamma, long P, int C, int round_out, void* ws,
                                size_t ws_bytes, void* stream);
int dvd_bn_act_bwd_ordered(const float* g, const float* x, const float* y, const float* gamma, const float* mean,
                           const float* var, float eps, float* gx, float* gres, float* ggamma, float* gbeta,
                           long P, int C, int relu, void* ws, size_t ws_bytes, void* stream);
int dvd_stem_wgrad_ordered(const float* x_nchw, const float* g, const float* a0, const float* weight, float* dweight, long s_co,
                           long s_ci, long s_ky, long s_kx, const float* bn_gamma, const float* bn_mean, const float* bn_var,
                           float bn_eps, float* dgamma, float* dbeta, const float* norm_mean3, const float* norm_std3,
                           float* scratch, int N, int H, int W, void* ws, size_t ws_bytes, void* stream);
int dvd_head_bwd_ordered(const float* x, const float* w, const float* b, const float* g_depth, float* gx, float* gw, float* gb,
                         long P, int relu_mask, int round_out, void* ws, size_t ws_bytes, void* stream);

/* ---- flow-pair preprocessing (csrc/flow_pairs.cu): raw optical flows -> the training pair's flows and masks ------------------
 * scripts/preprocess/davis/generate_flows.py:44-82,139-148. Flows are NHWC fp32 [B,H,W,2] (the pair-file layout), 8-byte
 * aligned; every call checks its shapes, alignment and buffer byte sizes before it launches and returns -2 with a message.   */
/* resize_flow: cv2.resize(flow, (W, H), INTER_CUBIC) (half-pixel centres, A = -0.75, clamped taps, horizontal pass first), then
 * x *= W / w and y *= H / h. src [B,h,w,2] -> dst [B,H,W,2], any sizes.                                                      */
int dvd_flow_resize_cubic(const float* src, size_t src_bytes, float* dst, size_t dst_bytes, int B, int h, int w, int H, int W,
                          void* stream);
/* forward / backward consistency masks. mask_1 lives on frame 2's grid: q = p + flow_2_1(p); flow_1_2 sampled at q as
 * F.grid_sample does (bilinear, zeros padding, align_corners=True); the pixel is bad when |sample + flow_2_1(p)| > 1 or q lies
 * outside [0, W-1] x [0, H-1]. mask_2 is the same with the flows swapped. Output convention:                               */
#define DVD_MASKS_FLOWPAIR_U8 0    /* uint8 [B,H,W], 1 = bad (flowpair_*.npz)                                               */
#define DVD_MASKS_PAIRFILE_F32 1   /* fp32 [B,H,W,1,1], 1 - ceil(mask): 1 = valid (the sequence .pt files); 4-byte aligned  */
int dvd_flow_pair_masks(const float* flow_1_2, const float* flow_2_1, size_t flow_bytes, void* mask_1, void* mask_2,
                        size_t mask_bytes, int B, int H, int W, int convention, void* stream);

/* ---- validation metric (csrc/eval_ops.cu) ----------------------------------------------------------------------------------
 * disp_vali (models/video_base.py:66-74) per frame: depth, depth_gt [N,1,H,W] fp32 (4-byte aligned; 16-byte aligned with H*W a
 * multiple of 4 takes the vector path). With v = [gt > 1e-2] and disp(x) = (1 / (x + (1 - [x > 1e-2])·1e-8))·[x > 1e-2], the
 * per-pixel term t = (disp(depth)·v - disp(gt)·v)² is evaluated in torch's operation order with every operation rounded on its
 * own, so it equals torch's fp32 elementwise term bit for bit. frame_sse [N] = Σ t over each frame, summed in a fixed order
 * without atomics (block partials into `partials`, then one fixed-order pass): bitwise reproducible. The frame's MSE is
 * frame_sse / (H·W). terms [N,1,H,W] receives the per-pixel terms, or is NULL. `partials` holds
 * dvd_disp_vali_partials_size(N, H, W) floats (-1 for a bad shape). Returns -2 with a message on a shape / alignment error.   */
int dvd_disp_vali_partials_size(int N, int H, int W);
int dvd_disp_vali(const float* depth, const float* depth_gt, float* frame_sse, float* terms, float* partials, int N, int H, int W,
                  void* stream);

/* ---- frame preparation (csrc/frame_prep.cu): scripts/preprocess/{davis,shutterstock}/generate_frame_midas.py -------------------
 * Buffers are caller-allocated; byte sizes, shapes and alignment are checked before any launch (-2 with a message); nothing
 * synchronises. The scipy stages accumulate in fp64 and round to fp32 where scipy stores fp32.                                */
/* F.interpolate(x, (H, W), mode='bicubic', align_corners=True) of NC planes: src [NC,h,w] -> dst [NC,H,W] fp32, any sizes (ATen's
 * upsample_bicubic2d: fp32 scale (in - 1) / (out - 1), A = -0.75, taps clamped to the border).                                 */
int dvd_resize_bicubic_ac(const float* src, size_t src_bytes, float* dst, size_t dst_bytes, int NC, int h, int w, int H, int W,
                          void* stream);
/* scipy.ndimage.spline_filter(maps[n], 3, output=float64, mode='constant') for n < N: maps [N,H,W] fp32 -> coef [N,H,W] fp64,
 * recursive prefilter along axis 0, then axis 1.                                                                              */
int dvd_spline_prefilter(const float* maps, size_t maps_bytes, double* coef, size_t coef_bytes, int N, int H, int W, void* stream);
/* map_coordinates(maps[n], [v, u], order=3, mode='constant') from coef [N,H,W]: vu [N,P,2] fp64 (v, u) pairs, 16-byte aligned ->
 * out [N,P] fp32. A coordinate outside [0, H-1] x [0, W-1], NaN or inf gives 0.                                               */
int dvd_spline_sample(const double* coef, size_t coef_bytes, int N, int H, int W, const double* vu, float* out, long P, void* stream);
/* Scale calibration, one thread per (frame n, point p): out = w2c[n] [X;1] (w2c [N,4,4] fp64 row-major, points [V,3] fp64),
 * (u, v) = (fx out.x + cx out.z, fy out.y + cy out.z) / out.z, depth = out.z. The point is kept when 0 <= u < W and 0 <= v < H,
 * then when map_coordinates(mask, [v, u]) < 0.1f, then when depth > 1e-3; ratio [N,V] = (double)map_coordinates(depth, [v, u])
 * / depth for a kept point, NaN otherwise. depth_coef and mask_coef are dvd_spline_prefilter outputs of the same [N,H,W] shape. */
int dvd_calib_ratios(const double* depth_coef, const double* mask_coef, size_t coef_bytes, const double* w2c, const double* points,
                     long V, double fx, double fy, double cx, double cy, double* ratio, size_t ratio_bytes, int N, int H, int W,
                     void* stream);
/* np.median of the non-NaN entries of each row of sorted [N,V] (rows ascending, NaN last): median [N] fp64, count [N] int32
 * (the number of non-NaN entries; the median is NaN where it is 0).                                                           */
int dvd_sorted_median(const double* sorted, size_t sorted_bytes, int N, long V, double* median, int* count, void* stream);
/* The same for fp32 rows, with numpy's fp32 rule: the middle element, or the fp32 (a + b) / 2 of the two middle ones (the sum
 * rounded to fp32). V <= INT_MAX.                                                                                              */
int dvd_sorted_median_f32(const float* sorted, size_t sorted_bytes, int N, long V, float* median, int* count, void* stream);
/* ShutterStock's dense calibration ratios (shutterstock/generate_frame_midas.py): nn [N,HW] fp32 (MiDaS depth at the stored
 * size), mvs [N,HW] fp32 (mvs_f64 = 0) or fp64 (mvs_f64 = 1) -> ratio [N,HW] of mvs's dtype, ratio = nn / mvs where mvs > 1e-3
 * and a positive NaN elsewhere (so that an ascending device sort puts the rejected pixels last). As numpy computes it: for
 * fp32 maps the threshold is 1e-3 rounded to fp32 and the quotient is fp32; for fp64 maps, (double)nn / mvs. One pass, 16-byte
 * loads when nn, mvs and ratio are 16-byte aligned.                                                                            */
int dvd_dense_ratios(const float* nn, size_t nn_bytes, const void* mvs, size_t mvs_bytes, int mvs_f64, void* ratio,
                     size_t ratio_bytes, int N, long HW, void* stream);
/* skimage.transform.resize(src[n], (OH, OW), preserve_range=True) of fp32 [N,H,W,C] as skimage >= 0.19 computes it:
 * gaussian_filter along axis 0 with the weights wy [2 ry + 1], then axis 1 with wx [2 rx + 1] (fp64 device arrays; mode 'mirror',
 * each pass fp64 and stored fp32), zoom(order=1, mode='mirror', grid_mode=True) in fp64 rounded to fp32, then a clip to the
 * frame's input min / max. scratch: dvd_aa_resize_scratch_bytes(N, H, W, C) bytes (-1 for a bad shape), 4-byte aligned.       */
long dvd_aa_resize_scratch_bytes(int N, int H, int W, int C);
int dvd_aa_resize(const float* src, size_t src_bytes, float* dst, size_t dst_bytes, void* scratch, size_t scratch_bytes,
                  const double* wy, int ry, const double* wx, int rx, int N, int H, int W, int C, int OH, int OW, void* stream);

/* ---- point-cloud export (csrc/points.cu). Both calls compact in index order with a tile count, a one-block scan of the tile
 * counts and a scatter: no atomic decides a position, so equal inputs give bitwise equal outputs. Both wait for the stream and
 * return the number of items written in *n_valid / *n_out. Scratch is 8-byte aligned, of the size the _scratch_bytes call gives. */
/* depth [N,H,W], img [N,3,H,W], P [N,3,H,W] (dvd_unproject_fwd of the depth) fp32. Pixel i = (n H + y) W + x is kept when its
 * depth d is finite and > 1e-2f and |d - d_n| / d <= edge_tol in fp64 for every in-image 4-neighbour n (NaN fails). mask [N H W]
 * = 0 / 1. For the k-th kept pixel in pixel order: index[k] = base + i, xyz[k,3] = P, rgb[k,3] = (uint8)(255 * clip(img, 0, 1))
 * in fp32 (NaN -> 0) and, when key is not NULL, key[k] = (kx << 42) | (ky << 21) | kz with k_a = floor((double)P_a / voxel) -
 * o_a. A k_a outside [0, 2^21) stores key -1 and returns -3 after the outputs are written. Capacity of the outputs: N H W.      */
long dvd_points_select_scratch_bytes(int N, int H, int W);
int dvd_points_select(const float* depth, const float* img, const float* P, int N, int H, int W, double edge_tol, double voxel,
                      long long ox, long long oy, long long oz, long long base, unsigned char* mask, long long* key, long long* index,
                      float* xyz, unsigned char* rgb, void* scratch, size_t scratch_bytes, long long* n_valid, void* stream);
/* skey [M] ascending, order [M] the permutation that sorted them (point j of a run is item order[j] of index / xyz / rgb, and
 * the items of one key come in ascending index, as a stable sort leaves them). For each run of equal keys, in run order: the
 * fp64 means of xyz and rgb summed in sorted order, the point count and views = the number of distinct frames index / hw. Runs
 * with views < min_views are dropped. Capacity of the outputs: M runs (mean_xyz, mean_rgb [M,3] fp64, count, views [M] int32). */
long dvd_voxel_reduce_scratch_bytes(long long M);
int dvd_voxel_reduce(const long long* skey, const long long* order, const long long* index, const float* xyz, const unsigned char* rgb,
                     long long M, long long hw, int min_views, double* mean_xyz, double* mean_rgb, int* count, int* views,
                     void* scratch, size_t scratch_bytes, long long* n_out, void* stream);

/* ---- novel views of a test export (csrc/render_views.cu): point clouds splatted into virtual cameras. --------------------- */
#define DVD_VIEW_CAM_FLOATS 21
#define DVD_SPLAT_MAX 4
/* cams [n_views, 21] fp32 per view: w2c (3 x 4 row-major: R^T | -R^T c) then K (3 x 3 row-major). keys [n_views, H, W] uint64,
 * set to all ones by the caller before the first call of a chunk. Point p (xyz [n_points, 3] fp32) is projected with every
 * operation rounded on its own, q_i = ((W_i0 P0 + W_i1 P1) + W_i2 P2) + t_i, h_i = (K_i0 q0 + K_i1 q1) + K_i2 q2, u = h0 / h2,
 * v = h1 / h2, and dropped when q2 <= 1e-2f or a coordinate is not finite. It covers the splat x splat pixels from x0 = floor(u
 * + 0.5f) - (splat - 1) / 2, y0 likewise, inside the image, and each covered pixel keeps min((bits(q2) << 32) | idx) (atomicMin).
 * With index (int64 [n_points]): point p belongs to view index[p] / (H W) in [0, n_views) and idx = index[p] % (H W), its source
 * pixel. With index NULL (a static cloud): every point is splatted into every view with idx = H W + p; H W + n_points must stay
 * below 2^32 (-1 otherwise). 1 <= splat <= DVD_SPLAT_MAX. The keys are a pure function of the inputs, whatever the order.      */
int dvd_splat_views(const float* xyz, const long long* index, long long n_points, const float* cams, int n_views, int H, int W,
                    int splat, unsigned long long* keys, void* stream);
/* keys [n_views, H, W] -> out [n_views, H, W, 3] uint8 BGR and coverage [n_views] int32 (pixels with a point). A pixel whose key
 * is all ones is black; idx = the low 32 bits below H W takes the colour floor(255 clip(img[f, :, idx], 0, 1)) in fp32 (NaN -> 0;
 * img [n_views, 3, H, W] fp32, dvd_points_select's colour rule), idx >= H W takes static_rgb[idx - H W] ([R, 3] uint8 RGB; may be
 * NULL when no static point was splatted).                                                                                       */
int dvd_resolve_views(const unsigned long long* keys, const float* img, const unsigned char* static_rgb, int n_views, int H, int W,
                      unsigned char* out, int* coverage, void* stream);

/* ---- synthetic depth of field (csrc/refocus.cu): a test export's frames blurred by their distance from a focal plane. --- */
#define DVD_REFOCUS_MAX_RADIUS 32
/* depth [N, H, W] fp32, img [N, 3, H, W] fp32 RGB, focus_disp [N] fp32 (device) -> out [N, H, W, 3] uint8 BGR. Every operation
 * is fp32 and rounded on its own. Per pixel: disp = 1 / d when d is finite and > 1e-2f, else 0; c = min(max_radius, scale
 * |disp - focus_disp[n]|); col = clip(img, 0, 1) per channel with NaN -> 0. For every tap (dx, dy) with dx^2 + dy^2 <=
 * max_radius^2, dy ascending then dx, whose q = p + (dx, dy) lies in the image: r = sqrt(dx^2 + dy^2), ce = disp(q) < disp(p) ?
 * min(c(q), c(p)) : c(q), w = clamp(ce - r + 0.5, 0, 1) / max(ce^2, 0.25); S_k += w col_k(q), W += w in tap order. out =
 * min(255, floor(255 (S_k / W))). 0 <= max_radius <= DVD_REFOCUS_MAX_RADIUS and a finite scale >= 0, else -2. The output is a
 * pure function of the inputs; with c = 0 everywhere it is floor(255 col).                                                     */
int dvd_refocus(const float* depth, const float* img, const float* focus_disp, float scale, int max_radius, unsigned char* out,
                int N, int H, int W, void* stream);

/* ---- evaluation of a test export (csrc/depth_metrics.cu): depth accuracy against depth_gt and consistency along the flow. ----
 * A depth is valid when it is finite and > 1e-2f. Per-pixel arithmetic is fp64 after the fp32 load, every operation rounded on
 * its own in the order written here; sums are fp64 in a fixed order (block partials in `partials`, then added in block order)
 * and a frame's (pair's) sums do not depend on the other frames (pairs) of the launch: bitwise reproducible. The *_size queries
 * return the number of 8-byte words of the workspace (-1 for a bad shape). Argument errors return -2 with a message.
 *
 * dvd_masked_select: values [N,H,W] fp32; element i of frame n is selected when values[n,i] is valid and, unless other is NULL,
 * other[n,i] (same shape) is valid too. median [N+1] fp32 receives, per frame and then for all frames pooled, the lower median:
 * the selected element of 0-based rank (n - 1) / 2, exact (radix select on order-preserving keys), NaN when n = 0; count [N+1]
 * int64 receives n. work: int64 words.                                                                                     */
long long dvd_masked_select_partials_size(int N, int H, int W);
int dvd_masked_select(const float* values, const float* other, float* median, long long* count, long long* work, int N, int H,
                      int W, void* stream);
/* dvd_depth_metrics: depth, depth_nn, depth_gt [N,H,W] fp32, scales [N,2,3] fp64 (per frame, per source s = 0 depth, 1
 * depth_nn, three depth scales a) -> sums [N,2,22] fp64. A pixel counts for source s when depth_gt g and the source's depth d are
 * valid; with d' = scales[n,s,a]·d: sums[n,s,0] = count, and sums[n,s,1 + 7a + k] for k = 0..6: Σ |d' - g| / g, Σ (d' - g)² / g,
 * Σ (d' - g)², Σ (ln d' - ln g)², and the counts of max(d' / g, g / d') < 1.25, 1.25², 1.25³. partials: fp64 words.          */
long long dvd_depth_metrics_partials_size(int N, int H, int W);
int dvd_depth_metrics(const float* depth, const float* depth_nn, const float* depth_gt, const double* scales, double* sums,
                      double* partials, int N, int H, int W, void* stream);
/* dvd_pair_consistency: depth, depth_nn [n_frames,H,W] fp32 and cam [n_frames,30] fp32 (K^T | (K^-1)^T | R | t, R t the
 * camera-to-world pose: dvd_b200.points.camera_block) of resident frames; pair p runs from frame a = ia[p] to b = ib[p] (int32
 * indices) with flow [n_pairs,H,W,2] fp32 (8-byte aligned) = flow_1_2 and mask [n_pairs,H,W] uint8 = the flowpair mask_2 (0 =
 * good); motion_seg [n_frames,H,W] uint8 or NULL. A pixel x = (i, j) of a (column, row) is evaluated for a source D when mask is
 * 0, q = x + flow is finite, D_a(x) is valid and so are the four bilinear taps of D_b at q: q clamped to [0, W-1] x [0, H-1],
 * taps at (x0, y0) = floor, x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1), weights wx1 = qx - x0, wx0 = 1 - wx1 (y alike),
 * D~ = ((wy0 wx0 D00 + wy0 wx1 D01) + wy1 wx0 D10) + wy1 wx1 D11. P = R_a (D_a(x) Kinv_a (i, j, 1)) + t_a, c = R_b^T (P - t_b)
 * (each matrix row a left-to-right dot product; P - t_b formed after P); z = c.z. z <= 1e-3 counts as behind; otherwise
 * p = (K_b c).xy / z, e_r = |p - q|, e_d = |z - D~| / D~. sums [n_pairs,2,2,6] fp64 per source (0 depth, 1 depth_nn) and
 * region (0 all, 1 static: motion_seg of frame a is 0; zero without motion_seg): evaluated pixels not behind, behind, Σ e_r,
 * Σ e_d, #e_r < 1, #e_r < 3. partials: fp64 words.                                                                          */
long long dvd_pair_consistency_partials_size(int n_pairs, int H, int W);
int dvd_pair_consistency(const float* depth, const float* depth_nn, const float* cam, int n_frames, const int* ia, const int* ib,
                         const float* flow, const unsigned char* mask, const unsigned char* motion_seg, double* sums,
                         double* partials, int n_pairs, int H, int W, void* stream);

/* ---- the learned scene flow over a test export (csrc/tracks.cu, dvd_b200.tracks). ------------------------------------------
 * dvd_pair_consistency_sf: dvd_pair_consistency for one depth source, `depth`, with the scene flow sf [n_pairs,3,H,W] fp32 of
 * each pair (channel-planar, the pair's frame a grid) added to the world point: P' = P + (double)sf(x) component by component,
 * after P = R_a (D_a(x) Kinv_a (i, j, 1)) + t_a is formed, and c = R_b^T (P' - t_b). Everything else (the evaluated-pixel
 * rule, D~, behind, e_r, e_d, the sums and their order) is dvd_pair_consistency's, through the same device code, so sf = 0
 * gives its `depth` sums bit for bit. sums [n_pairs,3,6] fp64 per region: 0 all, 1 static (motion_seg of frame a is 0), 2
 * moving (motion_seg of frame a is not 0); regions 1 and 2 are zero without motion_seg. partials: fp64 words.               */
long long dvd_pair_consistency_sf_partials_size(int n_pairs, int H, int W);
int dvd_pair_consistency_sf(const float* depth, const float* cam, int n_frames, const int* ia, const int* ib, const float* flow,
                            const unsigned char* mask, const unsigned char* motion_seg, const float* sf, double* sums,
                            double* partials, int n_pairs, int H, int W, void* stream);
/* dvd_draw_tracks: 3D tracks drawn over F frames. Track i (< M < 2^31) starts at frame number first[i] and has len[i] <= L1
 * positions X[i, 0..len-1] (X [M,L1,3] fp32, world space): position k belongs to frame number first[i] + k. Frame f (number[f],
 * int32) has the view block cams[f] ([F,21] fp32: w2c 3x4 | K 3x3, row-major, as dvd_splat_views), its refined depth
 * [F,H,W] fp32 and its image img [F,3,H,W] fp32 RGB. In frame f a track with k = number[f] - first[i] in [0, len[i]) is drawn:
 *   projection (render_views'): q = w2c X (each row ((w0 x + w1 y) + w2 z) + w3), h = K q (((k0 q0 + k1 q1) + k2 q2)),
 *     u = h0 / h2, v = h1 / h2, all fp32 with every operation rounded on its own; dropped when q2 <= 1e-2f or q0, q1, q2, u or
 *     v is not finite; z = q2; its pixel is (floor(u + 0.5f), floor(v + 0.5f)).
 *   a sample (pixel, z) is plotted when the pixel is in the image and not hidden: hidden when the frame's depth d there is valid
 *     (finite, > 1e-2f) and z > d * DVD_TRACK_HIDE_TOL (fp32 product).
 *   head, rank 0: the (2 DVD_TRACK_HEAD_RADIUS + 1)^2 pixels around X[i,k]'s pixel, each with X[i,k]'s z.
 *   segments X[i,j] -> X[i,j+1] for j = max(0, k - tail) .. k - 1, rank k - j, when both ends project: du = u1 - u0, dv, dz
 *     likewise, S = max(1, min(DVD_TRACK_MAX_SAMPLES, ceil(max(|du|, |dv|)))), samples s = 0..S at t = s / S: (u0 + t du,
 *     v0 + t dv, z0 + t dz).
 *   each plotted sample min-accumulates the key (rank << 32) | i into its pixel (atomicMin): youngest rank first, then the lower
 *     track index, whatever the order.
 *   resolve: base = (uint8)(255 clip(img, 0, 1)) with NaN -> 0; a pixel with a key takes w = 256 (tail + 1 - rank) / (tail + 1)
 *     (integer division) and (c w + base (256 - w) + 128) >> 8 per channel, c = rgb[i] (uint8 RGB [M,3]). out [F,H,W,3] uint8
 *     BGR. keys [F,H,W] uint64 is the work buffer (filled here).
 * proj [M,L1,3] fp32 and vis [M,L1] uint8 may both be NULL; else, for every drawn (i, k), proj[i,k] = (u, v, z) of the head (NaN
 * when dropped) and vis[i,k] = 1 when its centre sample is plotted, else 0. Other entries are left as they are. 0 <= tail <=
 * DVD_TRACK_MAX_TAIL, 1 <= F <= 65535.                                                                                      */
#define DVD_TRACK_HIDE_TOL 1.05f
#define DVD_TRACK_HEAD_RADIUS 1
#define DVD_TRACK_MAX_SAMPLES 1024
#define DVD_TRACK_MAX_TAIL 64
int dvd_draw_tracks(const float* X, const int* first, const int* len, const unsigned char* rgb, int M, int L1, const float* cams,
                    const float* depth, const float* img, const int* number, int F, int H, int W, int tail,
                    unsigned long long* keys, unsigned char* out, float* proj, unsigned char* vis, void* stream);

/* ---- test-end visualisation (csrc/test_videos.cu): models/video_base.py:157-272 (on_test_end) without matplotlib. ----------- */
#define DVD_VIS_MAX_PANELS 4
enum { DVD_VIS_DISP = 0, DVD_VIS_GT_DISP = 1, DVD_VIS_RGB = 2 };
/* One panel of a canvas batch. Pixel (y0 + y, x0 + x) of canvas c reads src[c s_canvas + y s_row + x s_col (+ k s_chan for
 * channel k of DVD_VIS_RGB)], strides in elements, so a temporal slice depth[:, 0, r, :] is read in place (s_canvas = W,
 * s_row = H W, s_col = 1). Transforms: DVD_VIS_DISP v = 1 / x in fp32; DVD_VIS_GT_DISP v = [x > 1e-8f] / (double)(x + 1e-8f)
 * in fp64; both colour-mapped through the range (vmin[c], vmax[c]) (device fp64, one entry per canvas). DVD_VIS_RGB writes
 * floor(255 clip(x, 0, 1)) per channel (NaN -> 0) as B, G, R; vmin / vmax are unused and may be NULL.                         */
typedef struct dvd_vis_panel {
  const float* src;
  const double* vmin;
  const double* vmax;
  long long s_canvas, s_row, s_col, s_chan;
  int rows, cols;
  int y0, x0;
  int transform;
  int reserved; /* 0 */
} dvd_vis_panel;
/* out [n_canvas, CH, CW, 3] uint8 BGR: canvas c is a copy of tmpl + c tmpl_stride ([CH, CW, 3] uint8, tmpl_stride = 0 shares one
 * template) with each panel's pixels replaced. Colour mapping: t = (v - vmin) / (vmax - vmin) in fp64, index floor(256 t)
 * clamped to [0, 255] (matplotlib's Colormap rule with N = 256; vmax == vmin -> 0), lut [256, 3] BGR; NaN v or t -> black.
 * `panels` is a HOST array of n_panels <= DVD_VIS_MAX_PANELS panels that lie inside the canvas and do not overlap (-1 otherwise).
 * One thread writes 8 consecutive pixels of a row; every output byte is written once, no atomics.                             */
int dvd_vis_panels(const unsigned char* tmpl, long long tmpl_stride, int n_canvas, int CH, int CW, const dvd_vis_panel* panels,
                   int n_panels, const unsigned char* lut, unsigned char* out, void* stream);

/* ---- training / validation pages (csrc/train_vis.cu): the images of util/util_visualize.py and util/util_flow.py as the
 * reference's HTMLVisualizer writes them for one visualised pack. ------------------------------------------------------------ */
#define DVD_VIS_MAX_MAPS 16
enum { DVD_VIS_MAP_DEPTH = 0, DVD_VIS_MAP_FLOW = 1, DVD_VIS_MAP_IMG = 2 };
/* One image key of a pack: n images of H x W, element (i, c, y, x) at src[i s_n + c s_c + y s_y + x s_x] (strides in elements,
 * so a permuted view such as [B,2,H,W].permute(0,2,3,1) is read in place). c is 0 for DEPTH, 0 / 1 (u / v) for FLOW and 0..2
 * (R, G, B) for IMG. Image i uses the fp32 pair ranges[range + 2 i], ranges[range + 2 i + 1] and writes tile `tile + i`.       */
typedef struct dvd_vis_map {
  const float* src;
  long long s_n, s_c, s_y, s_x;
  int kind;
  int n;
  int range;
  int tile;
} dvd_vis_map;
/* Per image of each map, exact fp32 extrema with NaN propagating (np.min / np.max): DEPTH min, max of t = 1 / (d + 1e-6f);
 * FLOW max of rad = sqrt(u u + v v) after |u| or |v| > 1e7 zeroes both (the second slot repeats it); IMG min, max over the
 * three channels (dvd_vis_tiles folds them over the map's n images). One CTA per image, no atomics.                           */
int dvd_vis_ranges(const dvd_vis_map* maps, int n_maps, int H, int W, float* ranges, void* stream);
/* tiles [*, H, W, 3] uint8 RGB, from the ranges dvd_vis_ranges wrote. turbo: [256, 3] fp64 colour table in [0, 1]; wheel:
 * [55, 3] fp64 Middlebury colour wheel over 255. The rules and their dtypes are spelled out in csrc/train_vis.cu. `maps` is a
 * HOST array of n_maps <= DVD_VIS_MAX_MAPS maps (-1 otherwise). One thread writes 4 consecutive pixels of a row, no atomics. */
int dvd_vis_tiles(const dvd_vis_map* maps, int n_maps, int H, int W, const float* ranges, const double* turbo, const double* wheel,
                  unsigned char* tiles, void* stream);

/* ---- RAFT optical flow, forward only (csrc/raft_ops.cu): third_party/RAFT/core as scripts/preprocess/davis/generate_flows.py runs it
 * (large model, all-pairs correlation, 4 levels, radius 4, hidden = context = 128, no warm start, test_mode). These are the CUDA-core
 * stages; the convolutions between them are dvd_conv2d_nhwc launches (dvd_b200/raft.py holds the schedule). All tensors NHWC fp32,
 * 16-byte aligned unless noted; coords1 [B,h,w,2] = (x, y) on the 1/8 grid, 8-byte aligned. Shapes, alignment and byte sizes are
 * checked before any launch (-2 with a message). No kernel uses atomics: equal inputs give bitwise equal outputs.
 * `round_out` = 1 stores TF32-rounded values (the tensor feeds a tensor-core convolution).                                      */
/* y [N,H/2,W/2,64] = conv7x7/2 pad 3 (2 (x / 255) - 1) + bias: extractor.py BasicEncoder.conv1 with raft.py:88-89 folded in.
 * x_nchw [N,3,H,W] holds 0..255; weight [64,3,7,7] and bias [64] contiguous. (The BatchNorm encoder's stem is dvd_stem_fwd.)     */
int dvd_raft_stem_fwd(const float* x_nchw, const float* weight, const float* bias, float* y, size_t y_bytes, int N, int H, int W,
                      void* stream);
/* nn.InstanceNorm2d (no affine, biased variance): stats [N,C,2] = (mean, 1 / sqrt(var + eps)) of x [N,P,C] per image and channel.
 * Two kernels with a fixed reduction order and fp64 sums; scratch: dvd_raft_instnorm_scratch_bytes(N, C) bytes.                  */
long dvd_raft_instnorm_scratch_bytes(int N, int C);
int dvd_raft_instnorm_stats(const float* x, float* stats, void* scratch, size_t scratch_bytes, int N, long P, int C, float eps,
                            void* stream);
/* y = relu_outer?( relu_inner?( (x - mean) * rstd ) + res ): the norm + ReLU + residual add + ReLU of extractor.py ResidualBlock.
 * stats NULL: no normalisation (the BatchNorm encoder's residual add); res NULL: no add. y may alias x.                            */
int dvd_raft_norm_act(const float* x, const float* stats, const float* res, float* y, int N, long P, int C, int relu_inner,
                      int relu_outer, int round_out, void* stream);
/* corr.py CorrBlock.__init__: level 0 [B, h w, h, w] = <fmap1[b,p,:], fmap2[b,q,:]> / sqrt(C) in plain fp32 FMA (the lookup
 * differentiates this volume, so no TF32 product), then three 2 x 2 average poolings over q. The levels are stored one after another,
 * dvd_raft_pyramid_floats(B, h, w) floats in all (-1 unless every level is at least 2 x 2, i.e. h, w >= 16: the reference's
 * lookup divides by (w - 1) and (h - 1) of every level). fmap [B,h,w,C], 16 | C.                                                */
long dvd_raft_pyramid_floats(int B, int h, int w);
int dvd_raft_corr_pyramid(const float* fmap1, const float* fmap2, float* pyramid, size_t pyramid_bytes, int B, int h, int w, int C,
                          void* stream);
/* corr.py CorrBlock.__call__ for all four levels in one launch: out [B,h,w,352], channel l * 81 + i * 9 + j = bilinear sample
 * (zeros outside) of level l at (x / 2^l + i - 4, y / 2^l + j - 4) - the window's slow index moves along x, as the reference's
 * meshgrid(dy, dx) added to (x, y) does; channels 324..351 are zero (the 1x1 convolution behind it wants 32 | Cin).              */
int dvd_raft_lookup(const float* pyramid, size_t pyramid_bytes, const float* coords1, float* out, size_t out_bytes, int B, int h,
                    int w, int round_out, void* stream);
/* update.py BasicMotionEncoder.convf1 + ReLU: y [B,h,w,128] = relu(conv7x7 pad 3 (coords1 - grid)); weight [128,2,7,7], bias [128] */
int dvd_raft_convf1(const float* coords1, const float* weight, const float* bias, float* y, int B, int h, int w, int round_out,
                    void* stream);
/* The GRU's operands are X = [h | inp | motion] and XR = [r h | inp | motion], [npx,384] each, written in place (no cat):
 * context_split: cnet [npx,256] (context encoder output) -> net = tanh(first half) [npx,128] (kept un-rounded: the hidden state),
 *   X[:, 0:128] = round(net), X / XR[:, 128:256] = round(relu(second half))                            (raft.py:109-113)
 * motion_pack:   X / XR[:, 256:384] = [mconv[:, 0:126] | round(coords1 - grid)], mconv [npx,128] the 126-output convolution of
 *   BasicMotionEncoder padded to 128 (already ReLU'd and rounded)                                      (update.py:95-97)
 * gru_rh:        XR[:, 0:128] = round(sigmoid(zr[:, 128:256]) * net), zr [npx,256] = pre-activations of convz | convr
 * gru_update:    net = (1 - z) net + z tanh(q), z = sigmoid(zr[:, 0:128]), q [npx,128] the pre-activation of convq;
 *   X[:, 0:128] = round(net) and, when not NULL, net_r [npx,128] = round(net)                          (update.py:49-61)         */
int dvd_raft_context_split(const float* cnet, float* net, float* X, float* XR, long npx, void* stream);
int dvd_raft_motion_pack(const float* mconv, const float* coords1, float* X, float* XR, int B, int h, int w, void* stream);
int dvd_raft_gru_rh(const float* zr, const float* net, float* XR, long npx, void* stream);
int dvd_raft_gru_update(const float* zr, const float* q, float* net, float* X, float* net_r, long npx, void* stream);
/* update.py FlowHead.conv2 + raft.py:131: delta = conv3x3 pad 1 (x) + bias, x [B,h,w,256], weight [2,256,3,3]; coords1 += delta in
 * place; delta [B,h,w,2] is also stored unless NULL.                                                                          */
int dvd_raft_flow_head(const float* x, const float* weight, const float* bias, float* coords1, float* delta, int B, int h, int w,
                       void* stream);
/* raft.py upsample_flow: flow [B,8h,8w,2] = sum_k softmax_k(mask_scale * mask[k*64 + i*8 + j]) * 8 (coords1 - grid)[neighbour k]
 * (3 x 3, zeros outside). The 576 mask channels come as three [B,h,w,192] tensors (the convolution kernel's widths do not include
 * 576); mask_scale = 0.25 for the raw output of update_block.mask (update.py:136).                                            */
int dvd_raft_upsample(const float* mask0, const float* mask1, const float* mask2, const float* coords1, float* flow,
                      size_t flow_bytes, int B, int h, int w, float mask_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DVD_B200_H_ */
