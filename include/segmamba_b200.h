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
 *
 * Scope (SURVEY.md section 8): real A, input-dependent ("variable") B and C, dstate in {8, 16},
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
 * Strided 2-D copy, 16-byte vectors: `rows` rows of `row_bytes` bytes from src (row pitch src_pitch_bytes) to dst (row
 * pitch dst_pitch_bytes).  Pointers, pitches and row_bytes must be multiples of 16.  Replaces the generic strided ATen copies
 * behind torch.cat((up, skip), dim=1) of UnetrUpBlock (monai/networks/blocks/unetr_block.py:81-86) and its backward on
 * channels-last activations: a channel concatenation is two such copies into the (tokens, C1 + C2) result.
 * ---------------------------------------------------------------------------------------------- */
SMB_API int smb_copy2d(const void *src, int64_t src_pitch_bytes, void *dst, int64_t dst_pitch_bytes, int64_t rows, int64_t row_bytes,
                       void *cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* SEGMAMBA_B200_H */
