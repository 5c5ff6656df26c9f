/*
 * mcvd_b200 -- C ABI of the H100-native (sm_90a) MCVD DDPM-sampling hot path.
 *
 * Plain C: device pointers and sizes only, no torch types.  Every pointer is a BORROWED device
 * pointer (owned by the caller, normally a torch tensor); outputs and workspaces are caller
 * allocated; every launch goes to the cudaStream_t passed in; no call synchronises.
 * Return value: 0 on success, negative on error (text via mcvd_last_error()).
 *
 * What this replaces in the reference (voletiv/mcvd-pytorch @ 451da2e, paths relative to its root):
 *   - the only native surface the reference has is the pybind11 op
 *       upfirdn2d(Tensor input, Tensor kernel, int up_x, up_y, down_x, down_y, pad_x0, pad_x1, pad_y0, pad_y1)
 *     (models/better/op/upfirdn2d.cpp:11-22, upfirdn2d_kernel.cu:209-369) -> MCVD_OP_APPLY with
 *     MCVD_F_UP / MCVD_F_DOWN (the FIR is fused with the norm/activation that precedes it);
 *   - everything else on the path is ATen/cuDNN/cuBLAS reached from Python
 *     (models/better/layerspp.py, layers.py, ncsnpp_more.py, models/__init__.py); the op kinds below
 *     are the fused H100 equivalents, each citing the reference lines it stands for.
 *
 * The host side (mcvd_b200/program.py) lowers a network + sampler step into an array of McvdOp and
 * calls mcvd_run_program() once per network evaluation (or once per CUDA-graph capture).
 */
#ifndef MCVD_B200_H
#define MCVD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MCVD_ABI_VERSION 5

/* ---- op kinds ------------------------------------------------------------------------------- */
enum {
  /* [B,C0,H,W] (+ [B,C1,H,W]) fp32 NCHW -> [B,H,W,C0+C1] NHWC.  torch.cat([x, cond], 1) +
   * x.contiguous() of ncsnpp_more.py:256-257,293.  Cout > 0: destination channel pitch (extra channels
   * are zero-filled so the first conv can run on the tensor cores with K a multiple of 16). */
  MCVD_OP_NCHW_TO_NHWC = 1,
  /* [B,H,W,C0] NHWC -> [B,C0,H,W] NCHW (network output back to the reference layout).  C1 > 0: source
   * channel pitch (the last conv writes Cout padded to 16). */
  MCVD_OP_NHWC_TO_NCHW = 2,
  /* sinusoidal timestep embedding, layers.py:504-518.  src0 = t fp32 [B]; dst [B, Cout]. */
  MCVD_OP_TIMESTEP_EMBED = 3,
  /* dst[b,j] = bias[j] + sum_k act(src0[b,k]) * w[j,k]; w is nn.Linear layout [Cout, C0].
   * MCVD_F_ACT_IN applies SiLU to the input (temb MLP ncsnpp_more.py:278-280; every FiLM
   * projection Dense_0(act(temb)) layerspp.py:521).  B rows. */
  MCVD_OP_LINEAR = 4,
  /* GroupNorm statistics, pass 1: per (b, pixel-chunk, channel) sum / sum-of-squares in fp64.
   * src0 [B,H,W,C0] (+ src1 [B,H,W,C1], virtual channel concat); dst = double2 [B, i0, C0+C1],
   * i0 = number of pixel chunks. */
  MCVD_OP_GN_PARTIAL = 5,
  /* GroupNorm statistics, pass 2 + FiLM/affine folding: reduces the partials over chunks and over
   * the i1 = C/groups channels of a group (groups are contiguous channel ranges,
   * layerspp.py:474-477), and writes one float4 per (b, channel): (mean, rstd, G, S) so that the
   * consumer computes  y = ((x - mean) * rstd [*(1+gamma)+beta]) * G + S.
   *   aux0 != NULL, MCVD_F_FILM : G = 1 + aux0[b*i2 + i3 + c], S = aux0[b*i2 + i3 + C + c]
   *                               (scale/shift = chunk(Dense_0(act(temb)), 2), layerspp.py:521-523,536)
   *   aux0 != NULL, !FILM       : G = aux0[c] (GroupNorm weight), S = aux1[c] (bias)
   *   aux0 == NULL              : G = 1, S = 0
   * src0 = per-channel partials of the first tensor ([B,i0,C0]); src1/C1 = partials of a second tensor
   * (virtual concat) or NULL/0; i0 = chunks, f0 = eps.  Partials are per TENSOR, so a tensor consumed by
   * several norms (skip connections) is scanned once.
   * i4 / i5 != 0: src0 / src1 is not a chunk array but the int64 tile statistics a MCVD_OP_CONV_UMMA2
   * epilogue wrote for that tensor, i4 / i5 = kernel size (1|3) of the producing conv (fixes the tile geometry).
   * dst2 != NULL additionally receives the planar table [B][3][C] = mean | rstd*G | S read by
   * MCVD_OP_CONV_UMMA2. */
  MCVD_OP_GN_FINALIZE = 6,
  /* normalise + FiLM (+ SPADE gamma/beta) + SiLU + optional 4x4 FIR up/down-sampling, fp32 NHWC in
   * and out.  get_act_norm.forward layerspp.py:518-549, MySPADE.forward :152-173 (norm part),
   * upsample_2d / downsample_2d up_or_down_sampling.py:196-258 == upfirdn2d.  H,W are OUTPUT
   * dims; src0/src1 are the (virtually concatenated) inputs at input resolution; aux0 = float4
   * table from GN_FINALIZE (NULL = raw pass-through, used for the skip branch FIR(x));
   * aux1/aux2 = SPADE gamma/beta [B,Hin,Win,C] or NULL.  dst2 != NULL additionally receives the same
   * resampling of the RAW input (the skip branch FIR(x) of up/down blocks, layerspp.py:600-611) so the
   * input is read once. */
  MCVD_OP_APPLY = 7,
  /* direct convolution as implicit GEMM on CUDA cores (fp32 FFMA), NHWC.  nn.Conv2d 3x3 pad 1 /
   * 1x1 (layers.py:89-113) and NIN (layers.py:541-544).  i0 = ksize (1|3); src0/src1 virtual
   * concat; w = packed [taps][C0+C1][i1] fp32 (i1 = Cout rounded up to 4); bias [Cout];
   * aux0 = residual [B,H,W,Cout] or NULL; dst = f0 * (conv + bias + residual);
   * MCVD_F_ACT_OUT applies SiLU to the result (SPADE mlp_shared, layerspp.py:148). */
  MCVD_OP_CONV_SIMT = 8,
  /* softmax(q.k^T * f0) v over all H*W keys, per (b, head); AttnBlockpp.forward layerspp.py:239-245.
   * src0 = qkv [B, T, 3*C0] (q | k | v along channels), i0 = heads, i1 = head dim, T = H*W;
   * dst [B, T, C0]. */
  MCVD_OP_ATTENTION = 9,
  /* nearest-neighbour resize of an NHWC map (F.interpolate(segmap, 'nearest'), layerspp.py:165).
   * src0 [B, i0, i1, C0] -> dst [B, H, W, C0]. */
  MCVD_OP_RESIZE_NEAREST = 10,
  /* reverse-diffusion update on the NCHW state, in place (models/__init__.py:287-290,324-333 for
   * DDPM; :163-166 DDIM; denoise :331-333):
   *   x0 = f0 * (x - f1 * eps);  if MCVD_F_CLIP: x0 = clamp(x0,-1,1);
   *   x  = f2 * x0 + f3 * x + f4 * eps + f5 * z
   * dst = x [B,C0,H,W] NCHW (in place); src0 = eps [B,H,W,C0] NHWC (channel pitch Cout if > 0); src1 = z NCHW or NULL
   * (MCVD_F_PHILOX: z from Philox4x32-10 keyed by (seed=i0|i1<<32, clip id = i2 + b, step = i3)).
   * MCVD_F_GAMMA (with MCVD_F_PHILOX): z = f7 * (G - f6), G ~ Gamma(shape f6, scale 1) drawn in-kernel
   * (Marsaglia-Tsang in fp64, mcvd_b200/csrc/elementwise.cu), i.e. the centred Gamma noise of a model trained
   * with model.gamma=True (models/__init__.py:319-322: f6 = k_cum, f7 = theta / sqrt(1 - alpha)). */
  MCVD_OP_DIFFUSION_UPDATE = 11,
  /* 3x3 / 1x1 convolution on the Hopper tensor cores (wgmma m64nNk16 f16, fp16 hi/lo split of
   * both operands, fp32 accumulation in registers), with the GroupNorm/FiLM/SiLU transform of the input
   * fused into the shared-memory staging.  Same semantics as MCVD_OP_CONV_SIMT; see
   * mcvd_b200/csrc/conv_umma.cu.  aux1 = norm table of (src0|src1) or NULL; i1 = n tile; i2 = work
   * organisation: 1 = streaming (one 128-position x n-tile tile per work item), 2 = input-stationary (1x1 convs
   * without a second segment: a 128-position tile's input stays resident in shared memory while the weights of
   * every n tile stream past it; streaming where it does not fit), 0 = input-stationary where it applies and the
   * position tiles fill the GPU, else streaming; i4 = tile height, a diagnostic override of the same kind (results
   * are identical bits either way): 0 = the launcher's choice (192 positions, three consumer warpgroups, for
   * streaming convs without dst2 statistics, n tile <= 192 and at least three weight stages in shared memory, except
   * where 192 would leave SMs idle; else 128), 128 or 192 = forced (192 is an error where it cannot run); i5 = slab
   * stages of a streaming conv, a diagnostic override of the same kind: 0 = the launcher's choice (2), 2 or 3 =
   * forced (an error where it does not fit or the conv is input-stationary); i3 = operand split for accuracy experiments (0 | 3 = all three products, 1 = drop
   * hi*lo_w, 2 = drop lo_a*hi, 4 = hi*hi only); f1 = weight un-scale.  Optional second K-segment (src2|src3 with C2|C3 channels, RAW,
   * centre tap only, weights appended per n-tile): the 1x1 shortcut Conv_2(x) of ResnetBlockBigGANpp
   * (layerspp.py:618-619) accumulated into the same accumulators as Conv_1, so
   * dst = f0 * (Conv_1(act(norm(h))) + Conv_2(x) + bias + residual) in ONE kernel.
   * dst2 = NULL, or the int64 tile statistics of the stored output (format and meaning as in MCVD_OP_CONV_UMMA2:
   * [tiles][NJ][2][Cout], mcvd_umma2_stats_bytes() bytes) for the GroupNorm that reads dst next;
   * aux2 is ignored. */
  MCVD_OP_CONV_UMMA = 12,
  /* final 3x3 conv with tiny Cout (<= 16) and fused input norm: conv3x3(SiLU(GN(x))) of
   * ncsnpp_more.py:375-379; aux0 = float4 norm table or NULL. */
  MCVD_OP_CONV_SMALLN = 13,
  /* dst[i] = src0[i] (i0 floats) -- device-to-device copy inside a program. */
  MCVD_OP_COPY = 14,
  /* MCVD_OP_ATTENTION on the tensor cores (wgmma, fp16 hi/lo split, flash-style online softmax with
   * S and O in registers); same fields plus dst2 = device scratch of at least
   * mcvd_attention_scratch_bytes(B, H*W, C0) bytes (16-byte aligned): a first kernel splits q, k, v into
   * fp16 hi/lo operand images there, the attention kernel streams them in with cp.async.bulk (2 launches).
   * Head dim in {32,48,64,96,128,192}, H*W a multiple of the key tile (128; 64 for head dim 128; 32 for head
   * dim 192; H*W itself when smaller).  See mcvd_b200/csrc/attention_umma.cu. */
  MCVD_OP_ATTENTION_UMMA = 15,
  /* MCVD_OP_CONV_UMMA with the norm table in planar form (same wgmma kernel, mcvd_b200/csrc/conv_umma.cu).  Same
   * semantics and fields, except:
   *   aux1 = norm table of (src0|src1) in the planar layout [B][3][C0+C1] = mean | rstd*G | S that
   *          MCVD_OP_GN_FINALIZE writes to its dst2 (NULL: raw input);
   *   w    = weights packed by mcvd_umma2_pack_weights for n tile i1 and K-block i2
   *          (i2 = mcvd_umma2_plan(...); 0 skips the consistency check);
   *   i3   = operand split: 3 (default, also 0) = hi*hi + lo*hi + hi*lo, 1 = drop hi*lo (fp16 weights),
   *          2 = drop lo*hi (fp16 activations), 4 = hi*hi only -- accuracy experiments;
   *   dst2 = NULL, or int64 [tiles][NJ][2][Cout] receiving the GroupNorm partial sums of the stored output
   *          (sum and sum of squares of round(x * 2^16), exact integer arithmetic for |x| <= 2^12: round(x * 2^16)
   *          stays inside int32 and the sum of squares of a tile slot's 128 rows inside 64 bits; outputs beyond
   *          that range have no defined statistics; tiles = 128-position row
   *          tiles of the padded-flat position space, NJ = 127 / Pimg + 2 image slots per tile,
   *          mcvd_umma2_stats_bytes() bytes) -- nn.GroupNorm statistics of the NEXT act-norm
   *          (layerspp.py:474-477) without re-reading the activation;
   *   aux2 is ignored. */
  MCVD_OP_CONV_UMMA2 = 16,
  /* per-frame quality metrics of generated clips on the GPU (reference runners/ncsn_runner.py:1581-1600, which
   * loops over PIL images on the CPU): src0 = pred, src1 = real, both [B, C0*i0, H, W] fp32 in [0,1] (i0 frames of
   * C0 = 1|3 channels); dst = float64 [B, i0, 2] = (MSE over the frame's C0*H*W values, SSIM).  SSIM as the
   * reference calls it: skimage structural_similarity(data_range=255, gaussian_weights=True,
   * use_sample_covariance=False) on the 8-bit grey images PIL makes (x*255 truncated; RGB -> L = (19595 R + 38470 G +
   * 7471 B + 32768) >> 16), i.e. 11x11 Gaussian (sigma 1.5) moments, mean over the interior cropped by 5 pixels.
   * MCVD_F_ROUND: round the [0,1] values first (the reference does for (Stochastic)MovingMNIST, :1596-1599). */
  MCVD_OP_FRAME_METRICS = 17,
  /* dst[b, c, y, x] = f5 * z for [B, C0, H, W] fp32 NCHW, z keyed exactly as in MCVD_OP_DIFFUSION_UPDATE with
   * MCVD_F_PHILOX (seed i0|i1<<32, clip id i2 + b, step tag i3): the Philox normal, or with MCVD_F_GAMMA the
   * centred Gamma draw f7 * (G - f6).  x_T of a Gamma-noise model (runners/ncsn_runner.py:1471-1474, 1546-1549)
   * without a host tensor.  src0 is not read. */
  MCVD_OP_NOISE = 18,
  /* LPIPS input of generated and real frames (runners/ncsn_runner.py:1427-1430, 1590-1591, 1606-1607:
   * ToPILImage -> convert("RGB") -> Resize((128, 128)) -> ToTensor -> Normalize(0.5, 0.5), then ScalingLayer,
   * models/networks_basic.py:89-96).  src0 = pred, src1 = real, both [B, C0*i0, i1, i1] fp32 (i0 frames of C0 = 1|3
   * channels, side i1), clamped to [0, 1]; u8 = trunc(x * 255); PIL's two-pass 8-bit bilinear resize with the
   * coefficient table w = int32 [128][2 + i2] (per output row/column: first source index, taps used, i2 22-bit
   * coefficients; mcvd_b200/lpips.py computes it); dst = fp32 NHWC [2*B*i0, 128, 128, 4] (pred frames, then real
   * frames; channel 3 is zero).  H = W = 128. */
  MCVD_OP_LPIPS_PREP = 19,
  /* NHWC direct convolution + bias + ReLU on the CUDA cores (fp32 FFMA implicit GEMM): one layer of torchvision's
   * alexnet().features (models/pretrained_networks.py:56-94).  src0 [B, i3, i4, C0] (C0 a multiple of 4);
   * MCVD_F_POOL: the conv reads the 3x3 / stride-2 max-pool of src0 instead (features[2], [5]);
   * i0 = kernel size, i1 = stride, i2 = padding; w = fp32 [i0][i0][C0][Cout] (K-major), bias [Cout], Cout a multiple
   * of 64; dst [B, H, W, Cout] with H, W = (input side + 2 i2 - i0) / i1 + 1. */
  MCVD_OP_CONV_RELU = 20,
  /* LPIPS head of one AlexNet tap (models/networks_basic.py:73-84, eval_models.py:35-37): per position
   * f / (sqrt(sum_c f^2) + 1e-10) of both maps, the squared difference weighted by lin_k (w = fp32 [C0]) summed over
   * channels, mean over the H*W positions.  src0 = pred features, src1 = real features, both [B, H, W, C0];
   * dst = fp64 [B] per frame pair: i0 == 0 overwrites, i0 != 0 adds (the five taps summed in order).  Fixed
   * reduction order, no atomics. */
  MCVD_OP_LPIPS_LAYER = 21,
  /* I3D input of videos for FVD (models/fvd/fvd.py:160-186 preprocess_single, runners/ncsn_runner.py:1918-1923
   * to_i3d): src0 = frames [B, C0*i0, i1, i1] fp32 (i0 frames of C0 = 1|3 channels, side i1, frame-major), bilinear
   * resize to i2 x i3 (F.interpolate align_corners=False: src = (dst + 0.5) * i1 / size - 0.5, clamped at 0), centre
   * crop to 224x224 at ((i2 - 224) / 2, (i3 - 224) / 2), (x - 0.5) * 2, no clamp; a grey frame is replicated to RGB.
   * dst = fp32 NDHWC [B, i0, 224, 224, 4], channel 3 zero.  H = W = 224; B * i0 <= 65535. */
  MCVD_OP_I3D_PREP = 22,
  /* NDHWC 3-D convolution + bias + ReLU (fp32 FFMA implicit GEMM): one Unit3D of InceptionI3d with its BatchNorm3d
   * folded into w and bias on the host (models/fvd/pytorch_i3d.py:37-103).  src0 [B, i4, i5, i5, C0] (C0 a multiple
   * of 4); kernel i0 x i1 x i1, stride i2 x i3 x i3; TF-SAME padding from the input size (compute_pad, :71-96):
   * per axis pad = max(k - (in % s ? in % s : s), 0), front pad / 2; output [B, To, H, W] with
   * To = (i4 + pad_t - i0) / i2 + 1 and H = W = (i5 + pad_s - i1) / i3 + 1 (= ceil(in / stride)).
   * w = fp32 [i0][i1][i1][C0][Cout] (K-major), bias [Cout], Cout a multiple of 8.  The output is channels
   * [i7, i7 + Cout) of dst [B, To, H, W, i6] (i6 = channel pitch >= i7 + Cout, both multiples of 4); other channels
   * are not written, so the four branches of an Inception block write their concat in place (:127-132). */
  MCVD_OP_CONV3D = 23,
  /* MaxPool3dSamePadding (models/fvd/pytorch_i3d.py:7-34): zero padding as CONV3D's (zeros take part in the max),
   * window i0 x i1 x i1, stride i2 x i3 x i3; src0 [B, i4, i5, i5, C0] (C0 a multiple of 4), dst [B, To, H, W, C0]
   * with To, H, W as for CONV3D. */
  MCVD_OP_MAXPOOL3D = 24,
  /* InceptionI3d head (models/fvd/pytorch_i3d.py:275-315): AvgPool3d([2, 7, 7], stride 1), the 1x1x1 logits conv
   * with bias (w = fp32 [C0][Cout], bias fp32 [Cout]), mean over time.  src0 [B, i4, 7, 7, C0] (i5 = 7, i4 >= 2),
   * dst fp64 [B, Cout] (Cout <= 512, C0 <= 6144); all in fp64, fixed reduction order, no atomics.  H = W = 1. */
  MCVD_OP_I3D_HEAD = 25,
  MCVD_OP__COUNT
};

/* ---- flags ---------------------------------------------------------------------------------- */
#define MCVD_F_ACT_IN   (1 << 0)   /* SiLU on the input (LINEAR)                                   */
#define MCVD_F_ACT_OUT  (1 << 1)   /* SiLU on the output (APPLY: after the norm; CONV: on result)  */
#define MCVD_F_UP       (1 << 2)   /* APPLY: FIR upsample x2   (input is H/2 x W/2)               */
#define MCVD_F_DOWN     (1 << 3)   /* APPLY: FIR downsample x2 (input is 2H x 2W)                 */
#define MCVD_F_FILM     (1 << 4)   /* GN_FINALIZE: aux0 is the FiLM table                          */
#define MCVD_F_CLIP     (1 << 5)   /* DIFFUSION_UPDATE: clamp x0 to [-1, 1]                        */
#define MCVD_F_PHILOX   (1 << 6)   /* DIFFUSION_UPDATE: draw z in-kernel                           */
#define MCVD_F_ROUND    (1 << 7)   /* FRAME_METRICS: round the images before the grey conversion   */
#define MCVD_F_GAMMA    (1 << 8)   /* DIFFUSION_UPDATE (with PHILOX), NOISE: centred Gamma(f6) * f7 */
#define MCVD_F_POOL     (1 << 9)   /* CONV_RELU: 3x3 / stride-2 max-pool on the input read           */

typedef struct McvdOp {
  int32_t kind;
  int32_t flags;
  int32_t B, H, W;          /* batch and OUTPUT spatial size                                   */
  int32_t C0, C1;           /* channels of src0 / src1 (C1 = 0: no second source)               */
  int32_t Cout;
  int32_t i0, i1, i2, i3;   /* per-kind integers, see the kind's comment                         */
  float f0, f1, f2, f3, f4, f5, f6, f7;
  const void* src0;
  const void* src1;
  const void* w;
  const void* bias;
  const void* aux0;
  const void* aux1;
  const void* aux2;
  void* dst;
  void* dst2;
  /* second K-segment of MCVD_OP_CONV_UMMA (fused 1x1 shortcut, see the kind's comment); NULL/0 otherwise */
  const void* src2;
  const void* src3;
  int32_t C2, C3;
  int32_t i4, i5, i6, i7;   /* more per-kind integers (ABI v4)                                  */
} McvdOp;

/* Library / ABI identification. */
int mcvd_abi_version(void);
/* sizeof(McvdOp) as compiled -- the Python ctypes mirror asserts equality at load time. */
int mcvd_sizeof_op(void);
/* Text of the last error on the calling thread ("" if none). */
const char* mcvd_last_error(void);
/* Compute capability of the current device as major*10+minor (e.g. 100), or <0. */
int mcvd_device_arch(void);

/* Launch ops[0..n) in order on `stream` (a cudaStream_t).  No synchronisation, re-entrant, uses the
 * device of the calling thread's current CUDA context (torch.cuda.device).  Capturable in a CUDA
 * graph. */
int mcvd_run_program(const McvdOp* ops, int n, void* stream);

/* Validate a program on the host without launching (shapes, alignment, NULLs).  Works without a
 * GPU. */
int mcvd_validate_program(const McvdOp* ops, int n);

/* Number of kernel launches mcvd_run_program would issue for this program (bench.py's
 * gpu_launches). */
int mcvd_count_launches(const McvdOp* ops, int n);

/* Weight packing for MCVD_OP_CONV_UMMA (device -> device, on `stream`):
 * w_taps = fp32 [taps][Cin][Cout] (the CONV_SIMT layout without Cout padding); out = the fp16 hi/lo
 * shared-memory images consumed by the tensor-core kernel; returns bytes required when out == NULL.
 * scale_log2 receives the power-of-two pre-scale applied to the weights (undone in the epilogue). */
long long mcvd_umma_pack_weights(const float* w_taps, int taps, int Cin, int Cout, int n_tile, int k_block,
                                 void* out, int scale_log2, void* stream);
/* Channels per K-block (32, 16, or 0 = unsupported) the tensor-core conv uses for sources with C0 / C1
 * channels; the packed weights must be produced with the same value. */
int mcvd_umma_kblock(int C0, int C1);
/* MCVD_OP_CONV_UMMA2 planning: channels per K-block (32 | 16, 0 = unsupported) for a conv of kernel size ks on
 * H x W maps with sources of C0|C1 (+ shortcut C2|C3) channels, n tile `n_tile`, with / without epilogue
 * statistics (the shared-memory plan depends on all of them); the weights must be packed with this value. */
int mcvd_umma2_plan(int H, int W, int ks, int C0, int C1, int C2, int C3, int n_tile, int stats);
/* The shared-memory plan behind mcvd_umma2_plan (diagnostics / tests; host arithmetic only): out[0..7] = K-block,
 * slab rows, image stages, raw-ring stages, weight stages, image slots per tile, 0, dynamic shared
 * memory bytes.  Returns 0, or -1 when the conv cannot run on this kernel. */
int mcvd_umma2_plan_info(int H, int W, int ks, int C0, int C1, int C2, int C3, int n_tile, int stats, int* out);
/* Bytes of the dst2 statistics array of a MCVD_OP_CONV_UMMA2 op. */
long long mcvd_umma2_stats_bytes(int B, int H, int W, int ks, int Cout);
/* Weight packing for MCVD_OP_CONV_UMMA2 (the MCVD_OP_CONV_UMMA layout).  w_taps = fp32 [taps][Cin][Cout]; every
 * (n tile, K-block, tap) becomes one shared-memory image of the n tile's columns.  A conv with a fused 1x1
 * shortcut is packed with two calls into the same `out`: the main conv with stage_off = 0 and the shortcut
 * with stage_off = (Cin_main / KB) * taps, both with per_unit = total stages of one n tile.  Returns the bytes
 * this call fills (taps*Cin*Cout*4); out == NULL only queries. */
long long mcvd_umma2_pack_weights(const float* w_taps, int taps, int Cin, int Cout, int n_tile, int k_block,
                                  void* out, int scale_log2, int stage_off, int per_unit, void* stream);
/* Bytes of dst2 scratch one MCVD_OP_ATTENTION_UMMA op with batch B, T = H*W tokens and C channels needs. */
long long mcvd_attention_scratch_bytes(int B, int T, int C);

#ifdef __cplusplus
}
#endif
#endif /* MCVD_B200_H */
