/*
 * segmamba_b200.h -- C ABI of the H100-native (sm_90a) SegMamba hot path (libsegmamba_b200.so).
 *
 * Plain C: raw device pointers, sizes, element strides, a cudaStream_t passed as void*.  No torch
 * types.  Every entry point returns 0 on success or a negative SMB_E* code; smb_last_error() then
 * returns a thread-local message (the Python shim raises it as RuntimeError, which is what the
 * reference's TORCH_CHECK failures surface as).
 *
 * Each entry point names the reference interface it replaces (paths relative to the reference repo):
 *
 *   smb_scan_fwd      selective_scan_cuda.fwd   mamba/csrc/selective_scan/selective_scan.cpp:226-336
 *   smb_scan_bwd      selective_scan_cuda.bwd   mamba/csrc/selective_scan/selective_scan.cpp:338-492
 *   smb_conv1d_fwd    causal_conv1d_cuda.causal_conv1d_fwd   causal-conv1d/csrc/causal_conv1d.cpp:130-189
 *   smb_conv1d_bwd    causal_conv1d_cuda.causal_conv1d_bwd   causal-conv1d/csrc/causal_conv1d.cpp:191-268
 *   smb_instnorm_*    nn.InstanceNorm3d + activation + residual chains of GSC / UnetResBlock,
 *                     model_segmamba/segmamba.py:111-130, monai/networks/blocks/dynunet_block.py:98-111
 *   smb_layernorm_*   nn.LayerNorm(dim) of MambaLayer, model_segmamba/segmamba.py:54,70
 *   smb_seq_permute   the flip / inter-slice re-orderings of Mamba.forward (v3),
 *                     mamba/mamba_ssm/modules/mamba_simple.py:230-261
 *   smb_gemm          the pointwise contractions (library GEMMs / 1x1x1 cuDNN convolutions in the reference):
 *                     Mamba.in_proj / out_proj  mamba_simple.py:204-208,264;  MlpChannel.fc1 / fc2  segmamba.py:81-89;
 *                     GSC.proj3 / proj4  segmamba.py:103-107;  UnetResBlock.conv3  dynunet_block.py:66-69
 *   smb_conv3d*       the dense 3x3x3 convolutions (cuDNN in the reference): UnetResBlock.conv1 / conv2
 *                     (dynunet_block.py) and GSC.proj / proj2 (segmamba.py)
 *
 * Scope (SURVEY.md section 8): real A, input-dependent ("variable") B and C, dstate in {8, 16, 32, 64},
 * conv width 2..4, non-channel-last conv layout, fp32 / fp16 / bf16 I/O with fp32 arithmetic.
 * Complex A, constant B/C, channel-last conv and the decode-time `update` kernels are out of scope;
 * calling with them returns SMB_EUNSUPPORTED.
 *
 * Ownership: all buffers are caller-owned and pre-allocated (the reference allocates outputs inside
 * the binding; here the Python shim does it so the library stays allocator-free).  Accumulated
 * outputs (dA, dB, dC, dD, ddelta_bias, dweight, dbias) must be zero-initialised by the caller,
 * exactly like the reference's torch::zeros_like (selective_scan.cpp:460-466, causal_conv1d.cpp:247-249).
 * Kernels are enqueued asynchronously on `stream`; no host synchronisation happens inside.
 */
#ifndef SEGMAMBA_B200_H
#define SEGMAMBA_B200_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define SMB_API __attribute__((visibility("default")))
#else
#define SMB_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define SMB_OK 0
#define SMB_EINVAL (-1)        /* bad shape / stride / pointer            */
#define SMB_EUNSUPPORTED (-2)  /* outside the supported scope (see above) */
#define SMB_ECUDA (-3)         /* a CUDA runtime call / launch failed     */
#define SMB_EWORKSPACE (-4)    /* workspace missing or too small          */

/* element type of the activations (u, delta, z, B, C, out, ... ); weights are always fp32 */
enum { SMB_F32 = 0, SMB_F16 = 1, SMB_BF16 = 2 };

/* order in which the kernel walks the L axis of every (.., L) operand:
 *   SMB_DIR_FORWARD  token t = position j                 (Mamba.forward `out`,   mamba_simple.py:217)
 *   SMB_DIR_REVERSE  token t = L-1-j: equals flip(-1) on all inputs and outputs (`out_b`, :230,264) */
enum { SMB_DIR_FORWARD = 0, SMB_DIR_REVERSE = 1 };

SMB_API int smb_version(void);
SMB_API const char *smb_last_error(void);
/* number of CUDA kernels this library has launched in the calling process (monotonic; for bench accounting) */
SMB_API uint64_t smb_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Selective scan.
 *   h[t,n] = exp(dt[t] A[d,n]) h[t-1,n] + dt[t] B[t,n] u[t],   dt = softplus?(delta + delta_bias)
 *   y[t]   = sum_n C[t,n] h[t,n] + D[d] u[t],   out_z[t] = y[t] * silu(z[t])
 * Shapes: u, delta, z, out, out_z: (batch, dim, L) with unit L-stride and arbitrary batch / dim
 * element strides (the reference's "HBL" layout has dim stride = batch*L, selective_scan.cpp:310).
 * A: (dim, dstate) fp32 contiguous.  D, delta_bias: (dim) fp32 or NULL.
 * B, C: (batch, n_groups, dstate, L) in the activation dtype; *_ls is the L stride (1 for the
 * reference layout), *_ns the dstate stride.
 * ---------------------------------------------------------------------------------------------- */
typedef struct smb_scan_fwd_args {
    int32_t batch, dim, seqlen, dstate, n_groups;
    int32_t dtype;           /* SMB_F32 / SMB_F16 / SMB_BF16 */
    int32_t delta_softplus;  /* bool */
    int32_t direction;       /* SMB_DIR_* ; 0 reproduces selective_scan_cuda.fwd exactly */
    const void *u, *delta, *z /* may be NULL */;
    const float *A, *D /* may be NULL */, *delta_bias /* may be NULL */;
    const void *B, *C;
    void *out;       /* y, pre-gate (may be NULL when z != NULL and only out_z is wanted) */
    void *out_z;     /* required iff z != NULL */
    float *x;        /* (batch, dim, ceil(L/2048), 2*dstate) chunk states as the reference returns, or NULL */
    float *hstates;  /* (batch, ceil(L/256)+1, dstate, dim) states at every 256th scan position + final, or NULL;
                        feed to smb_scan_bwd to skip its forward recompute */
    int64_t u_bs, u_ds, delta_bs, delta_ds, z_bs, z_ds, out_bs, out_ds, out_z_bs, out_z_ds;
    int64_t B_bs, B_gs, B_ns, B_ls, C_bs, C_gs, C_ns, C_ls;
    void *workspace;
    size_t workspace_bytes;  /* >= smb_scan_fwd_workspace_bytes(...) */
    float *hdense;   /* smb_scan_dense_floats(...) floats or NULL: the state entering every 8th scan position, laid out per
                        (batch, channel octet, block of 8 positions)[channel in octet][state]; feed to smb_scan_bwd, whose main
                        pass then needs neither a forward-state recompute nor a warp scan per state */
} smb_scan_fwd_args;

/* floats of the dense checkpoint arrays (hdense of smb_scan_fwd / smb_scan_bwd, mdense of smb_scan_bwd) */
SMB_API size_t smb_scan_dense_floats(int32_t batch, int32_t dim, int32_t seqlen, int32_t dstate, int32_t n_groups);

SMB_API size_t smb_scan_fwd_workspace_bytes(int32_t batch, int32_t dim, int32_t seqlen, int32_t dstate);
SMB_API int smb_scan_fwd(const smb_scan_fwd_args *args, void *cuda_stream);

typedef struct smb_scan_bwd_args {
    int32_t batch, dim, seqlen, dstate, n_groups;
    int32_t dtype;
    int32_t delta_softplus;
    int32_t direction;
    int32_t low_memory;         /* 1: chunk-parallel recompute in registers, workspace of a few MB (the shim's default and
                                      the default path);
                                   0: stash every recomputed state in the workspace (batch*L*dstate*dim elements) and
                                      sweep backwards once -- fewer instructions per update, more HBM traffic */
    const void *u, *delta, *z /* may be NULL */;
    const float *A, *D, *delta_bias;
    const void *B, *C;
    const void *dout;           /* gradient of out_z (z != NULL) or of out (z == NULL) */
    const float *hstates;       /* from smb_scan_fwd, or NULL: recomputed internally */
    void *du, *ddelta;          /* (batch, dim, L) activation dtype */
    void *dz;                   /* required iff z != NULL; may alias caller storage (ssi.py:244-248) */
    void *out_z;                /* optional recomputed out_z (recompute_out_z=True), else NULL */
    float *dA;                  /* (dim, dstate) fp32, zero-initialised, accumulated */
    float *dB, *dC;             /* (batch, n_groups, dstate, L) fp32 contiguous, zero-initialised, accumulated */
    float *dD, *ddelta_bias;    /* (dim) fp32 zero-initialised, or NULL */
    int64_t u_bs, u_ds, delta_bs, delta_ds, z_bs, z_ds, dout_bs, dout_ds;
    int64_t du_bs, du_ds, ddelta_bs, ddelta_ds, dz_bs, dz_ds, out_z_bs, out_z_ds;
    int64_t B_bs, B_gs, B_ns, B_ls, C_bs, C_gs, C_ns, C_ls;
    void *workspace;
    size_t workspace_bytes;     /* >= smb_scan_bwd_workspace_bytes(...) */
    const float *hdense;        /* dense forward checkpoints from smb_scan_fwd, or NULL.  With hdense (and low_memory != 0) the
                                   main pass is scan-free: every lane starts its 8-position run from a saved state and a saved
                                   local adjoint (mdense, written by the reverse-aggregate pass) */
    float *mdense;              /* scratch of smb_scan_dense_floats(...) floats, required iff hdense != NULL */
} smb_scan_bwd_args;

SMB_API size_t smb_scan_bwd_workspace_bytes(int32_t batch, int32_t dim, int32_t seqlen, int32_t dstate, int32_t dtype,
                                            int32_t low_memory);
SMB_API int smb_scan_bwd(const smb_scan_bwd_args *args, void *cuda_stream);

/* ------------------------------------------------------------------------------------------------
 * Depthwise causal conv1d (+ optional SiLU):  out[b,d,t] = act(bias[d] + sum_k w[d,k] x[b,d,t-(W-1-k)])
 * x, out, dout, dx: (batch, dim, L), unit L-stride.  weight: (dim, width) fp32 with strides,
 * bias: (dim) fp32 or NULL.  Weights in fp16/bf16 are converted by the shim (the reference's own
 * call sites always pass fp32 conv weights, ssi.py:169-177).
 * ---------------------------------------------------------------------------------------------- */
typedef struct smb_conv1d_args {
    int32_t batch, dim, seqlen, width;
    int32_t dtype;
    int32_t silu;
    int32_t direction;          /* SMB_DIR_REVERSE: causal along descending t (flip folded in) */
    const void *x;
    const float *weight, *bias;
    void *out;
    int64_t x_bs, x_ds, out_bs, out_ds, w_ds, w_ws;
} smb_conv1d_args;

SMB_API int smb_conv1d_fwd(const smb_conv1d_args *args, void *cuda_stream);

typedef struct smb_conv1d_bwd_args {
    int32_t batch, dim, seqlen, width;
    int32_t dtype;
    int32_t silu;
    int32_t direction;
    const void *x, *dout;
    const float *weight, *bias;
    void *dx;                   /* activation dtype; may alias caller storage (ssi.py:281-283) */
    float *dweight;             /* (dim, width) fp32 contiguous, zero-initialised, accumulated */
    float *dbias;               /* (dim) fp32 zero-initialised, or NULL */
    int64_t x_bs, x_ds, dout_bs, dout_ds, dx_bs, dx_ds, w_ds, w_ws;
} smb_conv1d_bwd_args;

SMB_API int smb_conv1d_bwd(const smb_conv1d_bwd_args *args, void *cuda_stream);

/* ------------------------------------------------------------------------------------------------
 * Sequence re-ordering used by the inter-slice direction of Mamba.forward (v3):
 *   to_slices  : dst[.., p*ns + s] = src[.., s*(L/ns) + p]   (stack(chunk(ns)).flatten, mamba_simple.py:245-247)
 *   from_slices: the inverse                                   (reshape/permute/flatten,   mamba_simple.py:261)
 * src/dst: (rows, L) with a row stride each, unit L-stride; optionally accumulates (dst += ...).
 * ---------------------------------------------------------------------------------------------- */
typedef struct smb_seq_permute_args {
    int32_t rows, seqlen, nslices;
    int32_t dtype;
    int32_t inverse;            /* 0: to_slices, 1: from_slices */
    int32_t accumulate;         /* dst += permuted(src) instead of dst = */
    const void *src;
    void *dst;
    int64_t src_rs, dst_rs;     /* element strides between rows */
} smb_seq_permute_args;

SMB_API int smb_seq_permute(const smb_seq_permute_args *args, void *cuda_stream);

/* ------------------------------------------------------------------------------------------------
 * Fused InstanceNorm3d(affine=False) [+ second operand] [+ ReLU / LeakyReLU] on channels-last activations
 * viewed as (batch, spatial, channels), channels contiguous.  Replaces the reference's chains of
 * nn.InstanceNorm3d + activation + residual add (model_segmamba/segmamba.py:111-130,147,171;
 * monai/networks/blocks/dynunet_block.py:98-111):
 *     y = act( IN(x) )                      mode2 = 0
 *     y = act( IN(x) + x2 )                 mode2 = 1   (raw residual)
 *     y = act( IN(x) + IN(x2) )             mode2 = 2   (both operands normalised with their own statistics)
 * channels must be a multiple of 16 / sizeof(element).  stats / stats2: (batch, channels, 2) fp32 = (mean, rstd),
 * written by the forward and read by the backward.  The backward returns dx and, for mode2 != 0, dx2.
 * ---------------------------------------------------------------------------------------------- */
enum { SMB_ACT_NONE = 0, SMB_ACT_RELU = 1, SMB_ACT_LEAKY_RELU = 2 };

typedef struct smb_instnorm_args {
    int32_t batch, channels;
    int32_t dtype;
    int32_t act;                /* SMB_ACT_* */
    int32_t mode2;              /* 0, 1, 2 (see above) */
    float slope;                /* LeakyReLU negative slope */
    float eps;
    int64_t spatial;
    const void *x, *x2;         /* x2 may be NULL when mode2 == 0 */
    void *y;
    float *stats, *stats2;      /* stats2 may be NULL unless mode2 == 2 */
    void *workspace;
    size_t workspace_bytes;     /* >= smb_instnorm_workspace_bytes(...) */
} smb_instnorm_args;

typedef struct smb_instnorm_bwd_args {
    int32_t batch, channels;
    int32_t dtype;
    int32_t act;
    int32_t mode2;
    float slope;
    float eps;
    int64_t spatial;
    const void *x, *x2, *dy;
    const float *stats, *stats2;
    void *dx, *dx2;             /* dx2 may be NULL when the second operand needs no gradient */
    void *workspace;
    size_t workspace_bytes;
} smb_instnorm_bwd_args;

SMB_API size_t smb_instnorm_workspace_bytes(int32_t batch, int32_t channels, int64_t spatial, int32_t dtype);
SMB_API int smb_instnorm_fwd(const smb_instnorm_args *args, void *cuda_stream);
SMB_API int smb_instnorm_bwd(const smb_instnorm_bwd_args *args, void *cuda_stream);

/* ------------------------------------------------------------------------------------------------
 * Fused LayerNorm over the last axis of a contiguous (rows, channels) token matrix:
 *     y = (x - mean) * rsqrt(var + eps) * gamma + beta        (biased variance, fp32 arithmetic)
 * Replaces nn.LayerNorm(dim) in MambaLayer.forward (model_segmamba/segmamba.py:54,70); x / y / dy / dx in the
 * activation dtype, gamma / beta / dgamma / dbeta fp32.  channels must be a multiple of 16 / sizeof(element), at most
 * 128 vectors of 16 bytes and at most 768; x, y, dy, dx must be 16-byte aligned.  The backward recomputes the row
 * statistics (nothing is saved by the forward) and ACCUMULATES into dgamma / dbeta, which the caller zero-initialises.
 * ---------------------------------------------------------------------------------------------- */
typedef struct smb_layernorm_args {
    int64_t rows;
    int32_t channels;
    int32_t dtype;
    float eps;
    const void *x;
    const float *gamma, *beta;  /* beta may be NULL */
    void *y;
} smb_layernorm_args;

typedef struct smb_layernorm_bwd_args {
    int64_t rows;
    int32_t channels;
    int32_t dtype;
    float eps;
    const void *x, *dy;
    const float *gamma;
    void *dx;
    float *dgamma, *dbeta;      /* dbeta may be NULL */
} smb_layernorm_bwd_args;

SMB_API int smb_layernorm_fwd(const smb_layernorm_args *args, void *cuda_stream);
SMB_API int smb_layernorm_bwd(const smb_layernorm_bwd_args *args, void *cuda_stream);

/* ------------------------------------------------------------------------------------------------
 * Tensor-core GEMM (wgmma.mma_async, accumulator in registers, operands staged by TMA):
 *     D[M, N] = epilogue( A[M, K] . B[N, K]^T )        fp16 / bf16 operands, fp32 accumulation
 * a_major / b_major: SMB_MAJOR_K  -- the operand is stored (rows = M or N index, K contiguous), ld = row stride;
 *                    SMB_MAJOR_MN -- the operand is stored (rows = K index, M or N contiguous), ld = row stride.
 * so a (tokens, C) channels-last activation is K-major for a contraction over C and MN-major for a contraction
 * over the tokens (weight gradients), and a (C_out, C_in) weight is K-major for y = x W^T and MN-major for dx = dy W.
 * lda / ldb in elements, multiples of 8; A and B 16-byte aligned.  D: (M, N) row-major with row stride ldd, in
 * out_dtype (SMB_F32 or the operand dtype).  epilogue: SMB_EPI_NONE, SMB_EPI_BIAS_N (+ bias[n], fp32),
 * SMB_EPI_BIAS_N_GELU (exact erf GELU after the bias, nn.GELU()), SMB_EPI_BIAS_M (+ bias[m]).
 * split_k > 1 (fp32 output only) partitions K over CTAs and ACCUMULATES into D with fp32 atomics; the caller
 * zero-initialises D (as with the reference's zero-initialised gradient accumulators).  accumulate != 0 adds the
 * product to the existing D (beta = 1: atomics for fp32, read-modify-write for 16-bit outputs).
 * ---------------------------------------------------------------------------------------------- */
enum { SMB_MAJOR_K = 0, SMB_MAJOR_MN = 1 };
enum { SMB_EPI_NONE = 0, SMB_EPI_BIAS_N = 1, SMB_EPI_BIAS_N_GELU = 2, SMB_EPI_BIAS_M = 3 };

typedef struct smb_gemm_args {
    int32_t M, N, K;
    int32_t dtype;              /* SMB_F16 / SMB_BF16 (operands) */
    int32_t out_dtype;          /* SMB_F32 or == dtype */
    int32_t a_major, b_major;   /* SMB_MAJOR_* */
    int32_t epilogue;           /* SMB_EPI_* */
    int32_t split_k;            /* >= 1 */
    int32_t accumulate;         /* D += product instead of D = product */
    const void *A, *B;
    const float *bias;          /* may be NULL */
    void *D;
    int64_t lda, ldb, ldd;
} smb_gemm_args;

SMB_API int smb_gemm(const smb_gemm_args *args, void *cuda_stream);

/* ------------------------------------------------------------------------------------------------
 * 3x3x3 convolution, stride 1, padding 1, no bias, on channels-last activations (implicit GEMM on wgmma; no im2col):
 *   smb_conv3d        y[n, d, h, w, co] = sum_{kd,kh,kw,ci} x[n, d+kd-1, h+kh-1, w+kw-1, ci] . weight[co, kd, kh, kw, ci]
 *                     (zero outside the volume).  The data gradient is this call on dy with the weight flipped in kd, kh, kw
 *                     and its two channel axes swapped (c_in and c_out swapped as well).
 *   smb_conv3d_wgrad  dweight[co, kd, kh, kw, ci] += sum_{n,d,h,w} dy[n, d, h, w, co] . x[n, d+kd-1, h+kh-1, w+kw-1, ci]
 *                     dweight is fp32 and accumulated into (zero it first); the summation order varies between runs.
 * x (batch, d, h, w, c_in), y / dy (batch, d, h, w, c_out): contiguous, fp16 or bf16 (dtype), 16-byte aligned; weight
 * (c_out, 3, 3, 3, c_in) contiguous in the same dtype.  c_in and c_out: multiples of 8.  The number of kernel launches
 * depends only on the shapes, nothing synchronises with the host.
 * ------------------------------------------------------------------------------------------------ */
typedef struct smb_conv3d_args {
    int32_t batch, d, h, w;
    int32_t c_in, c_out;
    int32_t dtype;              /* SMB_F16 / SMB_BF16 */
    const void *x;
    const void *weight;         /* smb_conv3d */
    void *y;                    /* smb_conv3d */
    const void *dy;             /* smb_conv3d_wgrad */
    float *dweight;             /* smb_conv3d_wgrad */
} smb_conv3d_args;

SMB_API int smb_conv3d(const smb_conv3d_args *args, void *cuda_stream);
SMB_API int smb_conv3d_wgrad(const smb_conv3d_args *args, void *cuda_stream);

/* ------------------------------------------------------------------------------------------------
 * Strided 2-D copy, 16-byte vectors: `rows` rows of `row_bytes` bytes from src (row pitch src_pitch_bytes) to dst (row
 * pitch dst_pitch_bytes).  Pointers, pitches and row_bytes must be multiples of 16.  Replaces the generic strided ATen copies
 * behind torch.cat((up, skip), dim=1) of UnetrUpBlock (monai/networks/blocks/unetr_block.py:81-86) and its backward on
 * channels-last activations: a channel concatenation is two such copies into the (tokens, C1 + C2) result.
 * ---------------------------------------------------------------------------------------------- */
SMB_API int smb_copy2d(const void *src, int64_t src_pitch_bytes, void *dst, int64_t dst_pitch_bytes, int64_t rows, int64_t row_bytes,
                       void *cuda_stream);

/* ------------------------------------------------------------------------------------------------
 * Training-patch sampling and augmentation on the GPU (segmamba_b200/augment.py, patch_loader.py): the crop of
 * DataLoaderMultiProcess (light_training/dataloading/base_data_loader.py:39-213) and the transforms of get_train_transforms
 * (light_training/augment/train_augment.py:23-62), as stages the host composes.  Every random draw is made by the host and
 * arrives here as a parameter; the only randomness on the device is the Gaussian noise of smb_aug_pointwise, a counter-based
 * Philox4x32-10 stream keyed by the 64-bit seed, counter (voxel / 4, step, sample, channel), so every value can be recomputed.
 * Volumes are (n0, n1, n2) fp32 with axis 2 contiguous.  Job lists are host arrays of any length; the records are copied into
 * the kernel parameters, so the array may be reused as soon as the call returns.  Kernels are enqueued on `cuda_stream`; no
 * allocation and no host synchronisation happen inside.  Volume axes are limited to 4..256 samples.
 * ---------------------------------------------------------------------------------------------- */
enum { SMB_AUG_MIRROR = 0, SMB_AUG_EDGE = 1 };        /* spline boundary: scipy 'mirror' / 'nearest' */
enum { SMB_AUG_AFFINE = 0, SMB_AUG_ZOOM = 1 };        /* resample coordinate map */
enum { SMB_AUG_OP_RETAIN = 1, SMB_AUG_OP_UNINVERT = 2, SMB_AUG_OP_NOISE = 4, SMB_AUG_OP_BRIGHT = 8, SMB_AUG_OP_CONTRAST = 16,
       SMB_AUG_OP_INVERT = 32, SMB_AUG_OP_GAMMA = 64 };
#define SMB_AUG_STATS_SCRATCH 512                      /* doubles of scratch per stats job */

/* crop box of one sample: out[c, i, j, k] = data[c, lz + i, ly + j, lx + k] inside the case, 0 outside (seg likewise) */
typedef struct smb_aug_case {
    const float *data;          /* (channels, D, H, W) fp32, W contiguous: device memory, or page-locked host memory read
                                   through its device mapping (then only the crop box crosses the bus) */
    const void *seg;            /* (D, H, W) int8, W contiguous, same placement rules */
    int64_t data_cs, data_zs, data_ys;
    int64_t seg_zs, seg_ys;
    int32_t D, H, W;
    int32_t lz, ly, lx;
} smb_aug_case;

typedef struct smb_aug_crop_args {
    int32_t batch, channels, pd, ph, pw;
    const smb_aug_case *cases;  /* `batch` records (host array) */
    float *data;                /* (batch, channels, pd, ph, pw) fp32 */
    void *seg;                  /* (batch, pd, ph, pw) int8 */
} smb_aug_crop_args;

SMB_API int smb_aug_crop(const smb_aug_crop_args *args, void *cuda_stream);

/* cubic B-spline coefficients of src (scipy.ndimage.spline_filter, order 3) on a grid with a 2-sample border per side:
 * coef is (n0 + 4, n1 + 4, n2 + 4).  SMB_AUG_MIRROR: whole-sample mirror boundary, the border holds the mirrored coefficients
 * (map_coordinates mode 'constant' / 'mirror');  SMB_AUG_EDGE: the coefficients of src padded by 12 edge samples per side and
 * filtered with the 'nearest' boundary, as scipy does for mode 'nearest' (zoom of skimage's resize, mode 'edge').
 * Axes need at least 4 samples; SMB_AUG_MIRROR axes at most 256.  The grid is limited to 2^31 - 1 voxels. */
typedef struct smb_aug_prefilter_job {
    const float *src;           /* (n0, n1, n2) */
    float *coef;                /* (n0 + 4, n1 + 4, n2 + 4); must not overlap src */
    int32_t n0, n1, n2;
    int32_t boundary;           /* SMB_AUG_MIRROR / SMB_AUG_EDGE */
} smb_aug_prefilter_job;

SMB_API int smb_aug_prefilter(const smb_aug_prefilter_job *jobs, int32_t n_jobs, void *cuda_stream);

/* dst[o] = src sampled at coordinate x(o), per axis d:
 *   SMB_AUG_AFFINE  x_d = a_d0 o_0 + a_d1 o_1 + a_d2 o_2 + a_d3   (double); outside [0, n_d - 1] on any axis -> 0 / label 0
 *   SMB_AUG_ZOOM    x_d = (o_d + 0.5) a_dd - 0.5                   (double; scipy zoom grid_mode, 'nearest' boundary)
 * order 0: nearest sample, index floor(x + 0.5), src fp32 (n0, n1, n2);
 * order 3: cubic B-spline, src the coef of smb_aug_prefilter;
 * order 1: labels, src and dst int8: the label whose trilinearly interpolated indicator is largest and >= 0.5, else 0
 *          (batchgenerators' interpolate_img(is_seg=True) with cval -1).
 * clip (optional): a stats record of smb_aug_stats; data results are clipped to its [min, max]. */
typedef struct smb_aug_resample_job {
    const void *src;
    void *dst;                  /* (m0, m1, m2) */
    const double *clip;
    int32_t n0, n1, n2, m0, m1, m2;
    int32_t order;              /* 0, 1, 3 */
    int32_t map;                /* SMB_AUG_AFFINE / SMB_AUG_ZOOM */
    double a00, a01, a02, a03, a10, a11, a12, a13, a20, a21, a22, a23;
} smb_aug_resample_job;

SMB_API int smb_aug_resample(const smb_aug_resample_job *jobs, int32_t n_jobs, void *cuda_stream);

/* x <- scipy.ndimage.gaussian_filter(x, sigma, mode='reflect', truncate=4.0): three 1-D passes x -> tmp -> tmp + n -> x */
typedef struct smb_aug_blur_job {
    float *x;
    float *tmp;                 /* 2 * n0 * n1 * n2 floats */
    float sigma;
    int32_t n0, n1, n2;
} smb_aug_blur_job;

SMB_API int smb_aug_blur(const smb_aug_blur_job *jobs, int32_t n_jobs, void *cuda_stream);

/* stats[0..3] = sum, sum of squares (fp64), min, max of x[0 .. n) */
typedef struct smb_aug_stats_job {
    const float *x;
    double *stats;
    double *scratch;            /* SMB_AUG_STATS_SCRATCH doubles */
    int64_t n;
} smb_aug_stats_job;

SMB_API int smb_aug_stats(const smb_aug_stats_job *jobs, int32_t n_jobs, void *cuda_stream);

/* in-place pointwise chain over x[0 .. n), in this order, each step only when its bit is set in `ops`; mean, std, min, max
 * come from `stats` (the state of x on entry), carried through the linear steps (brightness, inversion):
 *   RETAIN    x = (x - mean) / (std + 1e-8) * sd_r + mn_r, with mn_r, sd_r the mean and std of `retain_ref`
 *             (mn_r negated under UNINVERT: the reference was taken before the inversion of the gamma pass)
 *   UNINVERT  x = -x
 *   NOISE     x += noise_std * N(0, 1), Box-Muller on the Philox stream of (seed, step, sample, channel)
 *   BRIGHT    x *= brightness
 *   CONTRAST  x = clip((x - mean) * contrast + mean, min, max)
 *   INVERT    x = -x
 *   GAMMA     x = ((x - min) / (max - min + 1e-7)) ^ gamma * (max - min) + min
 * A step that reads the statistics must not follow NOISE, CONTRAST or GAMMA in the same job. */
typedef struct smb_aug_point_job {
    float *x;
    const double *stats;
    const double *retain_ref;
    int64_t n;
    int64_t seed;
    int32_t step, sample, channel;
    int32_t ops;
    float noise_std, brightness, contrast, gamma;
} smb_aug_point_job;

SMB_API int smb_aug_pointwise(const smb_aug_point_job *jobs, int32_t n_jobs, void *cuda_stream);

/* final layout: image[b, c, i, j, k] (or channels-last [b, i, j, k, c]) = data[c, f(i), f(j), f(k)] in out_dtype, label[b, i, j, k] =
 * int64 of seg[f(i), f(j), f(k)] with -1 -> 0, where f mirrors an axis when its bit (1: axis 0, 2: axis 1, 4: axis 2) is set in flip */
typedef struct smb_aug_emit_sample {
    const float *data;          /* (channels, pd, ph, pw) */
    const void *seg;            /* (pd, ph, pw) int8 */
    int32_t flip;
} smb_aug_emit_sample;

typedef struct smb_aug_emit_args {
    int32_t batch, channels, pd, ph, pw;
    int32_t out_dtype;          /* SMB_F32 / SMB_F16 / SMB_BF16 */
    int32_t channels_last;
    const smb_aug_emit_sample *samples;   /* `batch` records (host array) */
    void *image;
    int64_t *label;
} smb_aug_emit_args;

SMB_API int smb_aug_emit(const smb_aug_emit_args *args, void *cuda_stream);

/* ------------------------------------------------------------------------------------------------
 * Segmentation metrics on the GPU (segmamba_b200/metrics.py): Dice and the Hausdorff percentile of medpy.metric.binary
 * (dc, hd95, hd with connectivity 1) per (sample, region), from region bitmasks.  A region is a set of label values; voxel
 * bit r is set when the voxel belongs to region r (up to 8 regions).  Volumes are (batch, d, h, w) with w contiguous.
 * Stages, all on `cuda_stream`, with no allocation and no host synchronisation inside:
 *   smb_metric_region_bits  labels or logits (argmax over classes, first maximum wins) -> bits
 *   smb_metric_count        per (sample, region) counts and the two border masks (a foreground voxel with a 6-neighbour in
 *                           the background or outside the volume)
 *   smb_metric_edt          exact Euclidean distance from every border voxel of one mask to the nearest border voxel of the
 *                           other, appended to the (sample, region) pool
 *   smb_metric_select       the q-th percentile of each pool (numpy 'linear'), NaN where a mask is empty
 * Every count is an integer atomic and every pool is reduced by an order-free radix select: results are bitwise
 * deterministic.  Axes h and w are limited to 1..SMB_METRIC_MAX_AXIS voxels, d * h * w to 2^31 - 1.
 * ---------------------------------------------------------------------------------------------- */
#define SMB_METRIC_MAX_REGIONS 8
#define SMB_METRIC_MAX_AXIS 768
#define SMB_METRIC_NCOUNTS 8          /* int64 per (sample, region), see smb_metric_count */
enum { SMB_METRIC_I8 = 0, SMB_METRIC_U8 = 1, SMB_METRIC_I32 = 2, SMB_METRIC_I64 = 3, SMB_METRIC_LOGITS = 4 };

/* bits[b, v] = lut[label] for labels 0..255 (0 outside), label = src[b, v] or, for SMB_METRIC_LOGITS, argmax over
 * c < classes of src[b * sample_stride + c * class_stride + v * voxel_stride] (dtype SMB_F32 / SMB_F16 / SMB_BF16; a NaN is
 * the maximum, as in torch.argmax).  Labels are read at b * sample_stride + v * voxel_stride.  Strides in elements. */
typedef struct smb_metric_bits_args {
    const void *src;
    void *bits;                 /* (batch, voxels) uint8 */
    int64_t voxels, sample_stride, class_stride, voxel_stride;
    int32_t batch, kind, dtype, classes;
    uint8_t lut[256];
} smb_metric_bits_args;

SMB_API int smb_metric_region_bits(const smb_metric_bits_args *args, void *cuda_stream);

/* counts[(b * regions + r) * SMB_METRIC_NCOUNTS + k] += |P|, |G|, |P and G|, |border P|, |border G| for k = 0..4 (k = 5 is
 * the pool fill of smb_metric_edt; the caller zeroes counts first); the border masks get bit r of the border voxels. */
typedef struct smb_metric_count_args {
    const void *pred, *target;  /* (batch, d, h, w) uint8 region bits */
    void *pred_border, *target_border;
    int64_t *counts;
    int32_t batch, regions, d, h, w;
} smb_metric_count_args;

SMB_API int smb_metric_count(const smb_metric_count_args *args, void *cuda_stream);

/* For each (b, r, direction): the distance, with spacing s0, s1, s2 per axis, from every voxel of the source border (P's, then
 * G's) to the nearest voxel of the other border, sqrt(((dz s0)^2 + (dy s1)^2) + (dx s2)^2) in fp64, appended at
 * pool[(b * regions + r) * pool_cap + i] with i from the fill counter counts[.. + 5].  feat: batch * regions * 2 * d * h * w
 * int32 of workspace.  pool_cap must be at least 2 * d * h * w. */
typedef struct smb_metric_edt_args {
    const void *pred_border, *target_border;
    int32_t *feat;
    double *pool;
    int64_t *counts;
    int64_t pool_cap;
    int32_t batch, regions, d, h, w;
    double s0, s1, s2;
} smb_metric_edt_args;

SMB_API int smb_metric_edt(const smb_metric_edt_args *args, void *cuda_stream);

/* out[b, r] = numpy.percentile(pool of (b, r), 100 * frac) with method 'linear', NaN where |P| or |G| is 0 */
typedef struct smb_metric_select_args {
    const double *pool;
    const int64_t *counts;
    double *out;                /* (batch, regions) */
    int64_t pool_cap;
    int32_t batch, regions;
    double frac;                /* q / 100, in [0, 1] */
} smb_metric_select_args;

SMB_API int smb_metric_select(const smb_metric_select_args *args, void *cuda_stream);

/* Per-class evaluation (metrics.class_metrics): class k is the set of voxels whose label is classes[k], for up to 255 disjoint
 * classes.  smb_metric_region_bits with lut[classes[k]] = k + 1 writes the class maps (0: no class).  Then
 *   smb_metric_class_count  per (sample, class) counts, border-voxel counts and the bounding box of the border voxels of P and
 *                           G, and the two border maps
 *   smb_metric_class_edt    the EDT of smb_metric_edt over a table of jobs in device memory, each restricted to its box
 *   smb_metric_class_reduce per pool: the maximum, the q-th percentile and the mean distance of each direction
 * The host reads the count record back in between to plan the jobs and size the workspace. */
#define SMB_METRIC_I16 5
#define SMB_METRIC_MAX_CLASSES 255
#define SMB_METRIC_CLASS_NREC 11      /* int64 per (sample, class), see smb_metric_class_count */

/* record[(b * classes + k) * SMB_METRIC_CLASS_NREC + i] for class value k + 1 of the class maps (the caller zeroes it):
 * i = 0..4: |P|, |G|, |P and G|, |border P|, |border G|;  i = 5..7: d - z_lo, h - y_lo, w - x_lo and i = 8..10: z_hi + 1,
 * y_hi + 1, x_hi + 1 of the inclusive bounding box of the border voxels of P and G (all 0 when there are none).  A border voxel
 * has a class and a 6-neighbour of another class or outside the volume.  The border maps get the voxel's class value at border
 * voxels, 0 elsewhere. */
typedef struct smb_metric_class_count_args {
    const void *pred, *target;  /* (batch, d, h, w) uint8 class maps */
    void *pred_border, *target_border;
    int64_t *record;
    int32_t batch, classes, d, h, w;
} smb_metric_class_count_args;

SMB_API int smb_metric_class_count(const smb_metric_class_count_args *args, void *cuda_stream);

/* One EDT job: a box of bd x bh x bw voxels of one sample's border maps.  Voxel v is a source where (src[v] & src_mask) ==
 * src_val and a target where (tgt[v] & tgt_mask) == tgt_val.  The distance from every source voxel to the nearest target voxel
 * (as smb_metric_edt) is appended at pool[(*fill)++]; lines, if not NULL, gets per line of axis 1 (z * bw + x) the sum, in
 * order of y, and the maximum of its source distances.  feat: bd * bh * bw int32 of workspace. */
typedef struct smb_metric_edt_job {
    const void *src, *tgt;      /* the box origin in the maps, which have the row and slice strides of the args */
    int32_t *feat;
    double *pool;
    int64_t *fill;
    double *lines;              /* bd * bw (sum, max) pairs */
    int32_t bd, bh, bw, src_mask, src_val, tgt_mask, tgt_val;
} smb_metric_edt_job;

/* Every job has bd <= max_d, bh <= max_h <= SMB_METRIC_MAX_AXIS, bw <= max_w <= SMB_METRIC_MAX_AXIS, bd * bh * bw < 2^31. */
typedef struct smb_metric_class_edt_args {
    const smb_metric_edt_job *jobs;   /* njobs, in device memory */
    int64_t row_stride, slice_stride;  /* of the maps, in voxels */
    int32_t njobs, max_d, max_h, max_w;
    double s0, s1, s2;
} smb_metric_class_edt_args;

SMB_API int smb_metric_class_edt(const smb_metric_class_edt_args *args, void *cuda_stream);

/* One (sample, class) pair: dist holds the n0 distances from P's border and the n1 from G's border (any order); lines holds
 * lines0 then lines1 (sum, max) pairs of the two directions.  n0 and n1 must be positive. */
typedef struct smb_metric_pool {
    const double *dist, *lines;
    int64_t n0, n1;
    int32_t lines0, lines1;
} smb_metric_pool;

/* out[p * 4 + 0..3] = hd (the maximum), numpy.percentile(dist, 100 * frac) ('linear'), asd = sum0 / n0 and assd =
 * (sum0 / n0 + sum1 / n1) / 2 of pool p; each sum adds the line sums in a fixed order. */
typedef struct smb_metric_class_reduce_args {
    const smb_metric_pool *pools;     /* npools, in device memory */
    double *out;
    int32_t npools;
    double frac;
} smb_metric_class_reduce_args;

SMB_API int smb_metric_class_reduce(const smb_metric_class_reduce_args *args, void *cuda_stream);

/* ------------------------------------------------------------------------------------------------
 * Case prediction on the GPU (segmamba_b200/predict.py): the steps of the reference's Predictor after the sliding window,
 * plus exact 6-connected component post-processing.  All calls enqueue on `cuda_stream`, allocate nothing, never synchronise
 * with the host, size their launches from shapes only and give bitwise-deterministic results.
 *   smb_pred_restore  logits -> trilinear resample to the crop shape (F.interpolate, align_corners=False, fp32, stored as
 *                     fp16) -> argmax -> label map or region masks, uncropped into the original volume, in one pass
 *   smb_pred_cc       6-connected labelling of `batch` independent uint8 volumes (nonzero = foreground) and the three
 *                     operations built on it (SMB_PRED_LABEL / _FILL_HOLES / _LARGEST)
 * Volumes are limited to d * h * w < 2^31 voxels.
 * ---------------------------------------------------------------------------------------------- */

/* out[v] for v in (D0, H0, W0): 0 outside the box [z0, z0 + cd) x [y0, y0 + ch) x [x0, x0 + cw); inside, the argmax over
 * c < classes (first maximum; a NaN is the maximum) of fp16(trilinear sample of channel c at the box coordinate, sampling the
 * (d, h, w) logits as an output of size (cd, ch, cw)).  An axis whose crop size equals the logit size is copied.  Channel c
 * of logit voxel u is src[c * class_stride + u * voxel_stride] (elements; dtype SMB_F32 / SMB_F16 / SMB_BF16).
 * regions == 0: out is a (D0, H0, W0) uint8 label map; regions R in 1..8: out is (R, D0, H0, W0) uint8 with
 * out[r, v] = bit r of lut[label] (0 for labels >= 256). */
typedef struct smb_pred_restore_args {
    const void *src;
    void *out;
    int64_t class_stride, voxel_stride;
    int32_t dtype, classes, regions;
    int32_t d, h, w;            /* logit volume */
    int32_t cd, ch, cw;         /* crop shape (shape_after_cropping_before_resample) */
    int32_t z0, y0, x0;         /* lower corner of bbox_used_for_cropping */
    int32_t D0, H0, W0;         /* shape_before_cropping */
    uint8_t lut[256];
} smb_pred_restore_args;

SMB_API int smb_pred_restore(const smb_pred_restore_args *args, void *cuda_stream);

/* Components are 6-connected (scipy.ndimage.generate_binary_structure(3, 1)).
 *   SMB_PRED_LABEL       out: (batch, d, h, w) int32 labels, 0 background, component k numbered by the raster order of its
 *                        first voxel (scipy.ndimage.label's numbering); counts[b]: number of components (int64)
 *   SMB_PRED_FILL_HOLES  out: (batch, d, h, w) uint8, scipy.ndimage.binary_fill_holes: the mask plus every background
 *                        component without a voxel on the volume boundary
 *   SMB_PRED_LARGEST     out: (batch, d, h, w) uint8, the holes-filled largest component (ties: the highest label); all zero
 *                        for an empty mask.  counts is not used by the last two, and their out may be the mask itself.
 * workspace: at least smb_pred_cc_workspace_bytes(batch, d, h, w) bytes, 16-byte aligned. */
enum { SMB_PRED_LABEL = 0, SMB_PRED_FILL_HOLES = 1, SMB_PRED_LARGEST = 2 };

typedef struct smb_pred_cc_args {
    const void *mask;           /* (batch, d, h, w) uint8 */
    void *out;
    int64_t *counts;            /* (batch,), SMB_PRED_LABEL only */
    void *workspace;
    size_t workspace_bytes;
    int32_t batch, d, h, w, op;
} smb_pred_cc_args;

SMB_API size_t smb_pred_cc_workspace_bytes(int32_t batch, int32_t d, int32_t h, int32_t w);
SMB_API int smb_pred_cc(const smb_pred_cc_args *args, void *cuda_stream);

/* ------------------------------------------------------------------------------------------------
 * Case preprocessing on the GPU (segmamba_b200/preprocess.py): the reference's DefaultPreprocessor.run_case_npy (nonzero
 * crop with hole filling, z-score, resampling to the target spacing, foreground locations) and
 * collect_foreground_intensities.  The hole filling is smb_pred_cc (SMB_PRED_FILL_HOLES) and the cubic data resize is
 * smb_aug_stats + smb_aug_prefilter (SMB_AUG_EDGE) + smb_aug_resample (SMB_AUG_ZOOM, clipped); the calls here are the rest.
 * All enqueue on `cuda_stream`, allocate nothing, never synchronise with the host, size their launches from shapes only
 * and give bitwise-deterministic results.  Volumes are limited to d * h * w < 2^31 voxels.
 * ---------------------------------------------------------------------------------------------- */
#define SMB_PREP_CHUNK 1024           /* voxels per chunk of the ordered compaction */
#define SMB_PREP_MAX_JOBS 8           /* jobs per smb_prep_count / smb_prep_compact / smb_prep_normalize / smb_prep_ct_normalize launch */

/* reductions of smb_prep_mask (the call zeroes the record first) */
typedef struct smb_prep_record {
    int64_t lo_flip0, lo_flip1, lo_flip2;   /* 2^31 - (lowest index of a nonzero voxel) per axis; 0 when none */
    int64_t hi0, hi1, hi2;                  /* highest index of a nonzero voxel + 1 per axis; 0 when none */
    int64_t foreground;                     /* voxels with seg > 0 */
    int64_t nan_voxels;                     /* voxels with a NaN in some channel */
    int64_t bad_labels;                     /* seg voxels that are not an integer in [0, 127] (NaN included) */
} smb_prep_record;

/* mask[v] = 1 where some channel of data is nonzero (a NaN is nonzero), seg8[v] = int8 of seg[v] (0 without seg), plus the
 * record.  data (channels, d, h, w) fp32, seg (d, h, w) fp32 or NULL. */
typedef struct smb_prep_mask_args {
    const float *data;
    const float *seg;
    uint8_t *mask;
    int8_t *seg8;
    smb_prep_record *record;
    int32_t channels, d, h, w;
} smb_prep_mask_args;

SMB_API int smb_prep_mask(const smb_prep_mask_args *args, void *cuda_stream);

/* The box [z0, z0 + cd) x [y0, y0 + ch) x [x0, x0 + cw) of the (d, h, w) volume: out (channels, cd, ch, cw) fp32 copies data,
 * seg_out (cd, ch, cw) int8 is seg8 with nonzero_label where seg8 is 0 and mask is 0 (crop_to_nonzero's relabel). */
typedef struct smb_prep_crop_args {
    const float *data;
    const uint8_t *mask;
    const int8_t *seg8;
    float *out;
    int8_t *seg_out;
    int32_t channels, d, h, w, z0, y0, x0, cd, ch, cw;
    int32_t nonzero_label;      /* -128..127 */
} smb_prep_crop_args;

SMB_API int smb_prep_crop(const smb_prep_crop_args *args, void *cuda_stream);

/* ZScoreNormalization(use_mask_for_norm=False) of one channel of n voxels from its smb_aug_stats record:
 * dst = fp32((src - mean) / max(std, 1e-8)) in fp64, mean = sum / n, std = sqrt(max(sumsq / n - mean^2, 0));
 * moments[0..1] = mean, std.  dst may be src. */
typedef struct smb_prep_norm_job {
    const float *src;
    float *dst;
    const double *stats;
    double *moments;
    int64_t n;
} smb_prep_norm_job;

SMB_API int smb_prep_normalize(const smb_prep_norm_job *jobs, int32_t n_jobs, void *cuda_stream);

/* CTNormalization(use_mask_for_norm=False) of one channel of n voxels from the dataset's foreground statistics, in fp32 as
 * numpy computes it for a float32 image and Python-float properties: dst = (min(max(src, lo), hi) - mean) / div with IEEE
 * rounding and no contraction (a NaN stays NaN), lo = fp32(percentile_00_5), hi = fp32(percentile_99_5), mean = fp32(mean),
 * div = fp32(max(std, 1e-8)).  dst may be src.  At most SMB_PREP_MAX_JOBS jobs per launch; longer lists are split. */
typedef struct smb_prep_ct_norm_job {
    const float *src;
    float *dst;
    int64_t n;
    float lo, hi, mean, div;
} smb_prep_ct_norm_job;

SMB_API int smb_prep_ct_normalize(const smb_prep_ct_norm_job *jobs, int32_t n_jobs, void *cuda_stream);

/* batchgenerators resize_segmentation(order=1) of an int8 label volume (n0, n1, n2) -> (m0, m1, m2): per output voxel and per
 * axis the coordinate (o + 0.5) n / m - 0.5 clamped to [0, n - 1] (scipy zoom, grid_mode, mode 'nearest'), the trilinear
 * indicator of every label among the 8 taps in fp64, and the highest label whose indicator is >= 0.5 wins (0 when none). */
typedef struct smb_prep_label_resize_args {
    const int8_t *src;
    int8_t *dst;
    int32_t n0, n1, n2, m0, m1, m2;
} smb_prep_label_resize_args;

SMB_API int smb_prep_label_resize(const smb_prep_label_resize_args *args, void *cuda_stream);

/* Ordered compaction of the voxels of an int8 volume whose label is in a set (bit (uint8_t)label of `set`).
 *   smb_prep_count    chunk[k] = matching voxels of chunk k before it (exclusive scan), *count = total
 *   smb_prep_compact  index[0 .. count) = linear indices of the matching voxels in raster order, from the chunk offsets of
 *                     smb_prep_count on the same job (index holds at least count entries) */
typedef struct smb_prep_compact_job {
    const int8_t *seg;
    int32_t *chunk;             /* ceil(n / SMB_PREP_CHUNK) ints */
    int64_t *count;
    int32_t *index;             /* smb_prep_compact only */
    int64_t n;
    uint32_t set[8];
} smb_prep_compact_job;

SMB_API int smb_prep_count(const smb_prep_compact_job *jobs, int32_t n_jobs, void *cuda_stream);
SMB_API int smb_prep_compact(const smb_prep_compact_job *jobs, int32_t n_jobs, void *cuda_stream);

/* i in [0, n), p = index[select ? select[i] : i] (select entries must lie in [0, index length)):
 *   rows    (rows != NULL)    rows[4 i .. 4 i + 3] = 0, z, y, x of p in a (d, h, w) volume (np.argwhere of a (1, d, h, w) array)
 *   values  (values != NULL)  values[c n + i] = data[c channel_stride + p] for c < channels; with select_channel_stride s,
 *                             channel c reads select[c s + i] instead (s = 0: one selection for all channels) */
typedef struct smb_prep_gather_args {
    const int32_t *index;
    const int64_t *select;
    int64_t *rows;
    const float *data;
    float *values;
    int64_t n, channel_stride, select_channel_stride;
    int32_t channels, d, h, w;
} smb_prep_gather_args;

SMB_API int smb_prep_gather(const smb_prep_gather_args *args, void *cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* SEGMAMBA_B200_H */
