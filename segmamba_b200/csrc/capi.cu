// extern "C" entry points of libsegmamba_b200.so (see include/segmamba_b200.h).
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdint>
#include <cstring>

#include "../../include/segmamba_b200.h"
#include "aug_internal.h"
#include "conv3d_internal.h"
#include "conv_internal.h"
#include "gemm_internal.h"
#include "metrics_internal.h"
#include "norm_internal.h"
#include "predict_internal.h"
#include "prep_internal.h"
#include "scan_internal.h"

namespace smb {
static std::atomic<unsigned long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
#ifdef SMB_EMU
// wgmma / TMA have no CPU emulation: the emulated library exports smb_gemm but every call fails loudly
cudaError_t gemm_tc_launch(GemmP, const void *, int64_t, const void *, int64_t, cudaStream_t, const char **) { return cudaErrorNotSupported; }
int gemm_pick_bn(int) { return 0; }
cudaError_t conv3d_tc_launch(Conv3dP, const void *, const void *, cudaStream_t, const char **) { return cudaErrorNotSupported; }
#endif
}  // namespace smb

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

int cuda_fail(cudaError_t e, const char *where) {
    return fail(SMB_ECUDA, "%s: CUDA error %d (%s)", where, (int)e, cudaGetErrorString(e));
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct Plan {
    int dim_per_group, tiles_per_group, n_tiles, S, n_seg, nck;
    size_t seg_floats, ck_floats;
};

Plan make_plan(int batch, int dim, int L, int N, int G) {
    Plan pl;
    pl.dim_per_group = dim / G;
    pl.tiles_per_group = (pl.dim_per_group + 31) / 32;
    pl.n_tiles = pl.tiles_per_group * G;
    pl.S = smb::plan_segment(batch, pl.n_tiles, L);
    pl.n_seg = (L + pl.S - 1) / pl.S;
    pl.nck = (L + smb::kCkpt - 1) / smb::kCkpt;
    pl.seg_floats = align_up((size_t)batch * pl.n_seg * N * dim, 64);
    pl.ck_floats = align_up((size_t)batch * (pl.nck + 1) * N * dim, 64);
    return pl;
}

// floats per (P | H | hin | cumP) workspace array, sized for the shortest segment plan_segment may pick
size_t seg_floats_max(int batch, int dim, int L, int N) {
    const int smin = smb::seg_min();
    return align_up((size_t)batch * ((L + smin - 1) / smin) * N * dim, 64);
}

int check_common(int batch, int dim, int L, int N, int G, int dtype, const char *who) {
    if (batch <= 0 || dim <= 0 || L <= 0) return fail(SMB_EINVAL, "%s: batch, dim and seqlen must be positive", who);
    if (N != 8 && N != 16 && N != 32 && N != 64) return fail(SMB_EUNSUPPORTED, "%s: dstate %d unsupported (8, 16, 32 or 64)", who, N);
    if (G <= 0 || dim % G != 0) return fail(SMB_EINVAL, "%s: dim %d not divisible by n_groups %d", who, dim, G);
    if (dtype < SMB_F32 || dtype > SMB_BF16) return fail(SMB_EINVAL, "%s: bad dtype %d", who, dtype);
    return SMB_OK;
}

}  // namespace

extern "C" {

SMB_API int smb_version(void) { return 100; }
SMB_API const char *smb_last_error(void) { return g_err; }
SMB_API uint64_t smb_launch_count(void) { return (uint64_t)smb::g_launches.load(std::memory_order_relaxed); }

// ---------------------------------------------------------------------------------------------
SMB_API size_t smb_scan_fwd_workspace_bytes(int32_t batch, int32_t dim, int32_t seqlen, int32_t dstate) {
    // worst case over n_groups (more groups -> more tiles -> possibly longer segments -> fewer of them);
    // G = 1 gives the smallest S, i.e. the largest segment count.
    const Plan pl = make_plan(batch, dim, seqlen, dstate, 1);
    Plan plmax = pl;
    // segment count can only shrink with larger S; be conservative and size for the shortest segment plan_segment may pick
    const size_t seg_floats = seg_floats_max(batch, dim, seqlen, dstate);
    return sizeof(float) * (4 * seg_floats + plmax.ck_floats);
}

SMB_API size_t smb_scan_dense_floats(int32_t batch, int32_t dim, int32_t seqlen, int32_t dstate, int32_t n_groups) {
    if (batch <= 0 || dim <= 0 || seqlen <= 0 || dstate <= 0 || n_groups <= 0 || dim % n_groups) return 0;
    const size_t nck = (size_t)(seqlen + smb::kCkpt - 1) / smb::kCkpt;
    return (size_t)batch * smb::dense_octs(dim / n_groups, n_groups) * nck * 32 * 8 * dstate;
}

SMB_API int smb_scan_fwd(const smb_scan_fwd_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_scan_fwd: null args");
    int rc = check_common(a->batch, a->dim, a->seqlen, a->dstate, a->n_groups, a->dtype, "smb_scan_fwd");
    if (rc) return rc;
    if (!a->u || !a->delta || !a->A || !a->B || !a->C) return fail(SMB_EINVAL, "smb_scan_fwd: u, delta, A, B, C are required");
    if (a->z && !a->out_z) return fail(SMB_EINVAL, "smb_scan_fwd: out_z is required when z is given");
    if (!a->z && !a->out) return fail(SMB_EINVAL, "smb_scan_fwd: out is required when z is absent");
    if (a->B_ls != 1 || a->C_ls != 1) return fail(SMB_EUNSUPPORTED, "smb_scan_fwd: B and C must have unit stride along L");
    const size_t need = smb_scan_fwd_workspace_bytes(a->batch, a->dim, a->seqlen, a->dstate);
    if (!a->workspace || a->workspace_bytes < need)
        return fail(SMB_EWORKSPACE, "smb_scan_fwd: workspace of %zu bytes required, got %zu", need, a->workspace_bytes);
    const int N = a->dstate;
    const Plan pl = make_plan(a->batch, a->dim, a->seqlen, N, a->n_groups);
    smb::ScanP p;
    memset(&p, 0, sizeof(p));
    p.batch = a->batch; p.dim = a->dim; p.L = a->seqlen; p.G = a->n_groups;
    p.dim_per_group = pl.dim_per_group; p.tiles_per_group = pl.tiles_per_group; p.n_tiles = pl.n_tiles;
    p.S = pl.S; p.n_seg = pl.n_seg; p.nck = pl.nck;
    p.n_work = a->batch * pl.n_seg * pl.n_tiles;
    p.reverse = a->direction == SMB_DIR_REVERSE; p.softplus = a->delta_softplus != 0;
    p.u = a->u; p.delta = a->delta; p.z = a->z; p.B = a->B; p.C = a->C;
    p.A = a->A; p.D = a->D; p.delta_bias = a->delta_bias;
    p.out = a->out; p.out_z = a->out_z;
    p.u_bs = a->u_bs; p.u_ds = a->u_ds; p.delta_bs = a->delta_bs; p.delta_ds = a->delta_ds;
    p.z_bs = a->z_bs; p.z_ds = a->z_ds; p.out_bs = a->out_bs; p.out_ds = a->out_ds;
    p.out_z_bs = a->out_z_bs; p.out_z_ds = a->out_z_ds;
    p.B_bs = a->B_bs; p.B_gs = a->B_gs; p.B_ns = a->B_ns; p.B_ls = a->B_ls;
    p.C_bs = a->C_bs; p.C_gs = a->C_gs; p.C_ns = a->C_ns; p.C_ls = a->C_ls;
    float *ws = reinterpret_cast<float *>(a->workspace);
    const size_t segf = seg_floats_max(a->batch, a->dim, a->seqlen, N);
    p.P = ws; p.H = ws + segf; p.hin = ws + 2 * segf; p.cumP = ws + 3 * segf;
    p.hstates = a->hstates ? a->hstates : (a->x ? ws + 4 * segf : nullptr);
    p.hd = a->hdense;
    cudaError_t e = smb::scan_fwd_dispatch(p, a->dtype, N, a->z != nullptr, a->x, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_scan_fwd");
    return SMB_OK;
}

// ---------------------------------------------------------------------------------------------
SMB_API size_t smb_scan_bwd_workspace_bytes(int32_t batch, int32_t dim, int32_t seqlen, int32_t dstate, int32_t dtype,
                                            int32_t low_memory) {
    const int nck = (seqlen + smb::kCkpt - 1) / smb::kCkpt;
    const size_t ckf = align_up((size_t)batch * nck * dstate * dim, 64);
    size_t bytes = sizeof(float) * 6 * ckf;   // Pb, Mloc, Min + (P, H, hin) for the forward-state recompute
    if (!low_memory) {
        const size_t lpad = align_up((size_t)seqlen, smb::kTile);
        bytes += (size_t)batch * lpad * dstate * dim * (dtype == SMB_F32 ? 4 : 2) + 256;
    }
    return bytes;
}

SMB_API int smb_scan_bwd(const smb_scan_bwd_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_scan_bwd: null args");
    int rc = check_common(a->batch, a->dim, a->seqlen, a->dstate, a->n_groups, a->dtype, "smb_scan_bwd");
    if (rc) return rc;
    if (!a->u || !a->delta || !a->A || !a->B || !a->C || !a->dout) return fail(SMB_EINVAL, "smb_scan_bwd: u, delta, A, B, C, dout are required");
    if (!a->du || !a->ddelta || !a->dA || !a->dB || !a->dC) return fail(SMB_EINVAL, "smb_scan_bwd: du, ddelta, dA, dB, dC are required");
    if (a->z && !a->dz) return fail(SMB_EINVAL, "smb_scan_bwd: dz is required when z is given");
    if (a->B_ls != 1 || a->C_ls != 1) return fail(SMB_EUNSUPPORTED, "smb_scan_bwd: B and C must have unit stride along L");
    if (a->hdense && !a->mdense) return fail(SMB_EINVAL, "smb_scan_bwd: mdense scratch is required with hdense");
    const size_t need = smb_scan_bwd_workspace_bytes(a->batch, a->dim, a->seqlen, a->dstate, a->dtype, a->low_memory);
    if (!a->workspace || a->workspace_bytes < need)
        return fail(SMB_EWORKSPACE, "smb_scan_bwd: workspace of %zu bytes required, got %zu", need, a->workspace_bytes);
    const int N = a->dstate;
    Plan pl = make_plan(a->batch, a->dim, a->seqlen, N, a->n_groups);
    smb::ScanP p;
    memset(&p, 0, sizeof(p));
    p.batch = a->batch; p.dim = a->dim; p.L = a->seqlen; p.G = a->n_groups;
    p.dim_per_group = pl.dim_per_group; p.tiles_per_group = pl.tiles_per_group; p.n_tiles = pl.n_tiles;
    // the backward works on kCkpt-position chunks throughout
    p.S = smb::kCkpt; p.n_seg = pl.nck; p.nck = pl.nck;
    p.n_work = a->batch * pl.nck * pl.n_tiles;
    p.reverse = a->direction == SMB_DIR_REVERSE; p.softplus = a->delta_softplus != 0;
    p.u = a->u; p.delta = a->delta; p.z = a->z; p.B = a->B; p.C = a->C; p.dout = a->dout;
    p.A = a->A; p.D = a->D; p.delta_bias = a->delta_bias;
    p.out_z = a->out_z;
    p.u_bs = a->u_bs; p.u_ds = a->u_ds; p.delta_bs = a->delta_bs; p.delta_ds = a->delta_ds;
    p.z_bs = a->z_bs; p.z_ds = a->z_ds; p.dout_bs = a->dout_bs; p.dout_ds = a->dout_ds;
    p.out_z_bs = a->out_z_bs; p.out_z_ds = a->out_z_ds;
    p.B_bs = a->B_bs; p.B_gs = a->B_gs; p.B_ns = a->B_ns; p.B_ls = a->B_ls;
    p.C_bs = a->C_bs; p.C_gs = a->C_gs; p.C_ns = a->C_ns; p.C_ls = a->C_ls;
    p.du = a->du; p.ddelta = a->ddelta; p.dz = a->dz;
    p.dA = a->dA; p.dB = a->dB; p.dC = a->dC; p.dD = a->dD; p.ddelta_bias = a->ddelta_bias;
    p.du_bs = a->du_bs; p.du_ds = a->du_ds; p.ddelta_bs = a->ddelta_bs; p.ddelta_ds = a->ddelta_ds;
    p.dz_bs = a->dz_bs; p.dz_ds = a->dz_ds;
    float *ws = reinterpret_cast<float *>(a->workspace);
    const size_t ckf = align_up((size_t)a->batch * pl.nck * N * a->dim, 64);
    p.Pb = ws; p.Mloc = ws + ckf; p.Min = ws + 2 * ckf;
    p.P = ws + 3 * ckf; p.H = ws + 4 * ckf; p.hin = ws + 5 * ckf;
    p.Lpad = (int)align_up((size_t)a->seqlen, smb::kTile);
    p.stash = a->low_memory ? nullptr : reinterpret_cast<void *>(align_up(reinterpret_cast<size_t>(ws + 6 * ckf), 256));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    cudaError_t e;
    {   // timing experiments (results are wrong when set): 1 = no dB/dC atomics, 2 = no cross-channel reduction, 4 = no state math
        const char *dbg = getenv("SMB_R3_DBG");
        p.dbg = dbg ? atoi(dbg) : 0;
    }
    if (a->hdense && a->low_memory) {                     // scan-free main pass: no chunk states needed at all
        p.hd = const_cast<float *>(a->hdense);
        p.md = a->mdense;
        p.hs = a->hstates ? a->hstates : p.hin;
        p.hs_bs = (int64_t)(pl.nck + (a->hstates ? 1 : 0)) * N * a->dim;
    } else if (a->hstates) {
        p.hs = a->hstates;
        p.hs_bs = (int64_t)(pl.nck + 1) * N * a->dim;
    } else {
        // recompute the forward states at every chunk start: pass 1 + carry at chunk granularity
        if (pl.nck > 1) {
            if ((e = smb::scan_fwd_agg_dispatch(p, a->dtype, N, st)) != cudaSuccess) return cuda_fail(e, "smb_scan_bwd(agg)");
            if ((e = smb::carry_launch(p.P, p.H, p.hin, nullptr, a->batch, pl.nck, N, a->dim, 0, st)) != cudaSuccess)
                return cuda_fail(e, "smb_scan_bwd(carry)");
        } else {
            if ((e = cudaMemsetAsync(p.hin, 0, sizeof(float) * (size_t)a->batch * N * a->dim, st)) != cudaSuccess)
                return cuda_fail(e, "smb_scan_bwd(memset)");
        }
        p.hs = p.hin;
        p.hs_bs = (int64_t)pl.nck * N * a->dim;
    }
    e = smb::scan_bwd_dispatch(p, a->dtype, N, a->z != nullptr, st);
    if (e != cudaSuccess) return cuda_fail(e, "smb_scan_bwd");
    return SMB_OK;
}

// ---------------------------------------------------------------------------------------------
static int conv_common(int batch, int dim, int L, int width, int dtype, const char *who) {
    if (batch <= 0 || dim <= 0 || L <= 0) return fail(SMB_EINVAL, "%s: batch, dim and seqlen must be positive", who);
    if (width < 2 || width > 4) return fail(SMB_EUNSUPPORTED, "%s: only widths 2..4 are supported (got %d)", who, width);
    if (dtype < SMB_F32 || dtype > SMB_BF16) return fail(SMB_EINVAL, "%s: bad dtype %d", who, dtype);
    if (dim > 65535 || batch > 65535) return fail(SMB_EINVAL, "%s: dim and batch are limited to 65535", who);
    return SMB_OK;
}

SMB_API int smb_conv1d_fwd(const smb_conv1d_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_conv1d_fwd: null args");
    int rc = conv_common(a->batch, a->dim, a->seqlen, a->width, a->dtype, "smb_conv1d_fwd");
    if (rc) return rc;
    if (!a->x || !a->weight || !a->out) return fail(SMB_EINVAL, "smb_conv1d_fwd: x, weight, out are required");
    smb::ConvP p;
    memset(&p, 0, sizeof(p));
    p.batch = a->batch; p.dim = a->dim; p.L = a->seqlen; p.width = a->width;
    p.silu = a->silu != 0; p.reverse = a->direction == SMB_DIR_REVERSE;
    p.x = a->x; p.weight = a->weight; p.bias = a->bias; p.out = a->out;
    p.x_bs = a->x_bs; p.x_ds = a->x_ds; p.out_bs = a->out_bs; p.out_ds = a->out_ds; p.w_ds = a->w_ds; p.w_ws = a->w_ws;
    cudaError_t e = smb::conv1d_dispatch(p, a->dtype, false, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_conv1d_fwd");
    return SMB_OK;
}

SMB_API int smb_conv1d_bwd(const smb_conv1d_bwd_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_conv1d_bwd: null args");
    int rc = conv_common(a->batch, a->dim, a->seqlen, a->width, a->dtype, "smb_conv1d_bwd");
    if (rc) return rc;
    if (!a->x || !a->weight || !a->dout || !a->dx || !a->dweight) return fail(SMB_EINVAL, "smb_conv1d_bwd: x, weight, dout, dx, dweight are required");
    smb::ConvP p;
    memset(&p, 0, sizeof(p));
    p.batch = a->batch; p.dim = a->dim; p.L = a->seqlen; p.width = a->width;
    p.silu = a->silu != 0; p.reverse = a->direction == SMB_DIR_REVERSE;
    p.x = a->x; p.dout = a->dout; p.weight = a->weight; p.bias = a->bias; p.dx = a->dx;
    p.dweight = a->dweight; p.dbias = a->dbias;
    p.x_bs = a->x_bs; p.x_ds = a->x_ds; p.dout_bs = a->dout_bs; p.dout_ds = a->dout_ds; p.dx_bs = a->dx_bs; p.dx_ds = a->dx_ds;
    p.w_ds = a->w_ds; p.w_ws = a->w_ws;
    cudaError_t e = smb::conv1d_dispatch(p, a->dtype, true, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_conv1d_bwd");
    return SMB_OK;
}

SMB_API int smb_seq_permute(const smb_seq_permute_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_seq_permute: null args");
    if (a->rows <= 0 || a->seqlen <= 0 || a->nslices <= 0) return fail(SMB_EINVAL, "smb_seq_permute: rows, seqlen, nslices must be positive");
    if (a->seqlen % a->nslices != 0) return fail(SMB_EINVAL, "smb_seq_permute: seqlen %d not divisible by nslices %d", a->seqlen, a->nslices);
    if (a->rows > 65535) return fail(SMB_EINVAL, "smb_seq_permute: rows limited to 65535");
    if (a->dtype < SMB_F32 || a->dtype > SMB_BF16) return fail(SMB_EINVAL, "smb_seq_permute: bad dtype");
    if (!a->src || !a->dst) return fail(SMB_EINVAL, "smb_seq_permute: src and dst are required");
    cudaError_t e = smb::seq_permute_dispatch(a->src, a->dst, a->src_rs, a->dst_rs, a->rows, a->seqlen, a->nslices, a->inverse,
                                              a->accumulate, a->dtype, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_seq_permute");
    return SMB_OK;
}

// ---------------------------------------------------------------------------------------------
static int norm_common(int batch, int channels, int64_t spatial, int dtype, int act, int mode2, const char *who) {
    if (batch <= 0 || channels <= 0 || spatial <= 0) return fail(SMB_EINVAL, "%s: batch, channels, spatial must be positive", who);
    if (dtype < SMB_F32 || dtype > SMB_BF16) return fail(SMB_EINVAL, "%s: bad dtype %d", who, dtype);
    const int V = dtype == SMB_F32 ? 4 : 8;
    if (channels % V != 0) return fail(SMB_EUNSUPPORTED, "%s: channels %d must be a multiple of %d for this dtype", who, channels, V);
    if (channels / V > 256) return fail(SMB_EUNSUPPORTED, "%s: channels %d too large", who, channels);
    if (act < 0 || act > 2 || mode2 < 0 || mode2 > 2) return fail(SMB_EINVAL, "%s: bad act / mode2", who);
    if (batch > 65535) return fail(SMB_EINVAL, "%s: batch limited to 65535", who);
    return SMB_OK;
}

SMB_API size_t smb_instnorm_workspace_bytes(int32_t batch, int32_t channels, int64_t spatial, int32_t dtype) {
    int n_cta = 0;
    int64_t rows = 0;
    const int eb = dtype == SMB_F32 ? 4 : 2;
    if (batch <= 0 || channels <= 0 || spatial <= 0 || channels % (16 / eb) != 0) return 0;
    smb::norm_plan(batch, channels, spatial, eb, &n_cta, &rows);
    return sizeof(float) * ((size_t)2 * batch * n_cta * 3 * channels + (size_t)batch * channels * 3 + 64);
}

static void norm_fill(smb::NormP &p, int batch, int channels, int64_t spatial, int dtype, int act, int mode2, float slope, float eps,
                      void *workspace) {
    memset(&p, 0, sizeof(p));
    p.batch = batch; p.channels = channels; p.spatial = spatial; p.act = act; p.mode2 = mode2; p.slope = slope; p.eps = eps;
    smb::norm_plan(batch, channels, spatial, dtype == SMB_F32 ? 4 : 2, &p.n_cta, &p.rows_per_cta);
    p.partial = reinterpret_cast<float *>(workspace);
    p.sums = p.partial + (size_t)2 * batch * p.n_cta * 3 * channels;
}

SMB_API int smb_instnorm_fwd(const smb_instnorm_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_instnorm_fwd: null args");
    int rc = norm_common(a->batch, a->channels, a->spatial, a->dtype, a->act, a->mode2, "smb_instnorm_fwd");
    if (rc) return rc;
    if (!a->x || !a->y || !a->stats) return fail(SMB_EINVAL, "smb_instnorm_fwd: x, y, stats are required");
    if (a->mode2 && !a->x2) return fail(SMB_EINVAL, "smb_instnorm_fwd: x2 is required when mode2 != 0");
    if (a->mode2 == 2 && !a->stats2) return fail(SMB_EINVAL, "smb_instnorm_fwd: stats2 is required when mode2 == 2");
    const size_t need = smb_instnorm_workspace_bytes(a->batch, a->channels, a->spatial, a->dtype);
    if (!a->workspace || a->workspace_bytes < need)
        return fail(SMB_EWORKSPACE, "smb_instnorm_fwd: workspace of %zu bytes required, got %zu", need, a->workspace_bytes);
    smb::NormP p;
    norm_fill(p, a->batch, a->channels, a->spatial, a->dtype, a->act, a->mode2, a->slope, a->eps, a->workspace);
    p.x = a->x; p.x2 = a->x2; p.y = a->y; p.stats = a->stats; p.stats2 = a->stats2;
    cudaError_t e = smb::instnorm_dispatch(p, a->dtype, false, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_instnorm_fwd");
    return SMB_OK;
}

SMB_API int smb_instnorm_bwd(const smb_instnorm_bwd_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_instnorm_bwd: null args");
    int rc = norm_common(a->batch, a->channels, a->spatial, a->dtype, a->act, a->mode2, "smb_instnorm_bwd");
    if (rc) return rc;
    if (!a->x || !a->dy || !a->dx || !a->stats) return fail(SMB_EINVAL, "smb_instnorm_bwd: x, dy, dx, stats are required");
    if (a->mode2 && !a->x2) return fail(SMB_EINVAL, "smb_instnorm_bwd: x2 is required when mode2 != 0");
    if (a->mode2 == 2 && !a->stats2) return fail(SMB_EINVAL, "smb_instnorm_bwd: stats2 is required when mode2 == 2");
    const size_t need = smb_instnorm_workspace_bytes(a->batch, a->channels, a->spatial, a->dtype);
    if (!a->workspace || a->workspace_bytes < need)
        return fail(SMB_EWORKSPACE, "smb_instnorm_bwd: workspace of %zu bytes required, got %zu", need, a->workspace_bytes);
    smb::NormP p;
    norm_fill(p, a->batch, a->channels, a->spatial, a->dtype, a->act, a->mode2, a->slope, a->eps, a->workspace);
    p.x = a->x; p.x2 = a->x2; p.dy = a->dy; p.dx = a->dx; p.dx2 = a->dx2;
    p.stats = const_cast<float *>(a->stats); p.stats2 = const_cast<float *>(a->stats2);
    cudaError_t e = smb::instnorm_dispatch(p, a->dtype, true, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_instnorm_bwd");
    return SMB_OK;
}

// ---------------------------------------------------------------------------------------------
static int ln_common(int64_t rows, int channels, int dtype, const void *p0, const void *p1, const void *p2, const char *who) {
    if (rows <= 0 || channels <= 0) return fail(SMB_EINVAL, "%s: rows and channels must be positive", who);
    if (dtype < SMB_F32 || dtype > SMB_BF16) return fail(SMB_EINVAL, "%s: bad dtype %d", who, dtype);
    const int V = dtype == SMB_F32 ? 4 : 8;
    if (channels % V != 0) return fail(SMB_EUNSUPPORTED, "%s: channels %d not a multiple of %d", who, channels, V);
    if (channels / V > 128 || channels > 768) return fail(SMB_EUNSUPPORTED, "%s: channels %d too large", who, channels);
    if (((uintptr_t)p0 | (uintptr_t)p1 | (uintptr_t)p2) & 15) return fail(SMB_EINVAL, "%s: activation pointers must be 16-byte aligned", who);
    return SMB_OK;
}

SMB_API int smb_layernorm_fwd(const smb_layernorm_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_layernorm_fwd: null args");
    if (!a->x || !a->y || !a->gamma) return fail(SMB_EINVAL, "smb_layernorm_fwd: x, y, gamma are required");
    int rc = ln_common(a->rows, a->channels, a->dtype, a->x, a->y, nullptr, "smb_layernorm_fwd");
    if (rc) return rc;
    smb::LnP p;
    memset(&p, 0, sizeof(p));
    p.rows = a->rows; p.C = a->channels; p.eps = a->eps; p.x = a->x; p.gamma = a->gamma; p.beta = a->beta; p.y = a->y;
    cudaError_t e = smb::layernorm_dispatch(p, a->dtype, false, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_layernorm_fwd");
    return SMB_OK;
}

SMB_API int smb_layernorm_bwd(const smb_layernorm_bwd_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_layernorm_bwd: null args");
    if (!a->x || !a->dy || !a->dx || !a->gamma || !a->dgamma)
        return fail(SMB_EINVAL, "smb_layernorm_bwd: x, dy, dx, gamma, dgamma are required");
    int rc = ln_common(a->rows, a->channels, a->dtype, a->x, a->dy, a->dx, "smb_layernorm_bwd");
    if (rc) return rc;
    smb::LnP p;
    memset(&p, 0, sizeof(p));
    p.rows = a->rows; p.C = a->channels; p.eps = a->eps; p.x = a->x; p.dy = a->dy; p.gamma = a->gamma; p.dx = a->dx;
    p.dgamma = a->dgamma; p.dbeta = a->dbeta;
    cudaError_t e = smb::layernorm_dispatch(p, a->dtype, true, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_layernorm_bwd");
    return SMB_OK;
}

SMB_API int smb_gemm(const smb_gemm_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_gemm: null args");
    if (!a->A || !a->B || !a->D) return fail(SMB_EINVAL, "smb_gemm: A, B, D are required");
    if (a->M <= 0 || a->N <= 0 || a->K <= 0) return fail(SMB_EINVAL, "smb_gemm: M, N, K must be positive");
    if (a->dtype != SMB_F16 && a->dtype != SMB_BF16) return fail(SMB_EUNSUPPORTED, "smb_gemm: operands must be fp16 or bf16");
    if (a->out_dtype != SMB_F32 && a->out_dtype != a->dtype) return fail(SMB_EINVAL, "smb_gemm: out_dtype must be fp32 or the operand dtype");
    if ((a->lda % 8) || (a->ldb % 8)) return fail(SMB_EINVAL, "smb_gemm: lda and ldb must be multiples of 8 elements (16-byte rows for TMA)");
    if ((reinterpret_cast<uintptr_t>(a->A) & 15) || (reinterpret_cast<uintptr_t>(a->B) & 15))
        return fail(SMB_EINVAL, "smb_gemm: A and B must be 16-byte aligned");
    if (a->a_major < 0 || a->a_major > 1 || a->b_major < 0 || a->b_major > 1) return fail(SMB_EINVAL, "smb_gemm: bad operand major");
    if (a->epilogue < SMB_EPI_NONE || a->epilogue > SMB_EPI_BIAS_M) return fail(SMB_EINVAL, "smb_gemm: bad epilogue");
    if (a->split_k > 1 && a->out_dtype != SMB_F32) return fail(SMB_EINVAL, "smb_gemm: split_k needs an fp32 output");
    if (a->ldd < a->N) return fail(SMB_EINVAL, "smb_gemm: ldd < N");
    // the contiguous extent of each operand as stored: K for a K-major operand, M / N for an MN-major one
    if (a->lda < (a->a_major == SMB_MAJOR_K ? a->K : a->M) || a->ldb < (a->b_major == SMB_MAJOR_K ? a->K : a->N))
        return fail(SMB_EINVAL, "smb_gemm: leading dimension smaller than the contiguous extent");
    smb::GemmP p;
    memset(&p, 0, sizeof(p));
    p.M = a->M; p.N = a->N; p.K = a->K; p.dtype = a->dtype; p.out_dtype = a->out_dtype;
    p.a_mn = a->a_major; p.b_mn = a->b_major; p.epilogue = a->epilogue;
    p.split_k = a->split_k < 1 ? 1 : a->split_k;
    p.atomic = (p.split_k > 1 || a->accumulate) ? 1 : 0;
    p.bias = a->bias; p.D = a->D; p.ldd = a->ldd;
    {   // measurement aid: SMB_GEMM_PROF = device address (decimal) of 16 uint64 counters that receive the per-role wait cycles
        const char *pe = getenv("SMB_GEMM_PROF");
        p.prof = pe ? reinterpret_cast<unsigned long long *>(strtoull(pe, nullptr, 10)) : nullptr;
    }
    const char *where = "";
    cudaError_t e = smb::gemm_tc_launch(p, a->A, a->lda, a->B, a->ldb, (cudaStream_t)cuda_stream, &where);
    if (e != cudaSuccess)
        return fail(SMB_ECUDA, "smb_gemm: %s failed: CUDA error %d (%s) [M=%d N=%d K=%d a_major=%d b_major=%d lda=%lld ldb=%lld]", where,
                    (int)e, cudaGetErrorString(e), a->M, a->N, a->K, a->a_major, a->b_major, (long long)a->lda, (long long)a->ldb);
    return SMB_OK;
}

namespace {
int conv3d_check(const char *fn, const smb_conv3d_args *a, const void *x, const void *b, const void *out) {
    if (!a) return fail(SMB_EINVAL, "%s: null args", fn);
    if (!x || !b || !out) return fail(SMB_EINVAL, "%s: all tensors are required", fn);
    if (a->batch <= 0 || a->d <= 0 || a->h <= 0 || a->w <= 0) return fail(SMB_EINVAL, "%s: extents must be positive", fn);
    if (a->dtype != SMB_F16 && a->dtype != SMB_BF16) return fail(SMB_EUNSUPPORTED, "%s: operands must be fp16 or bf16", fn);
    if (a->c_in <= 0 || a->c_out <= 0 || (a->c_in % 8) || (a->c_out % 8))
        return fail(SMB_EUNSUPPORTED, "%s: c_in and c_out must be positive multiples of 8 (16-byte rows for TMA)", fn);
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(b) & 15))
        return fail(SMB_EINVAL, "%s: operands must be 16-byte aligned", fn);
    if ((int64_t)a->batch * a->d * a->h * a->w >= (int64_t)1 << 31) return fail(SMB_EINVAL, "%s: more than 2^31 voxels", fn);
    return SMB_OK;
}

int conv3d_run(const char *fn, const smb_conv3d_args *a, int wgrad, const void *x, const void *b, void *out, void *cuda_stream) {
    smb::Conv3dP p;
    memset(&p, 0, sizeof(p));
    p.batch = a->batch; p.D = a->d; p.H = a->h; p.W = a->w; p.C_in = a->c_in; p.C_out = a->c_out;
    p.dtype = a->dtype; p.wgrad = wgrad; p.out = out;
    const char *where = "";
    cudaError_t e = smb::conv3d_tc_launch(p, x, b, (cudaStream_t)cuda_stream, &where);
    if (e != cudaSuccess)
        return fail(SMB_ECUDA, "%s: %s failed: CUDA error %d (%s) [batch=%d d=%d h=%d w=%d c_in=%d c_out=%d]", fn, where, (int)e,
                    cudaGetErrorString(e), a->batch, a->d, a->h, a->w, a->c_in, a->c_out);
    return SMB_OK;
}
}  // namespace

SMB_API int smb_conv3d(const smb_conv3d_args *a, void *cuda_stream) {
    int rc = conv3d_check("smb_conv3d", a, a ? a->x : nullptr, a ? a->weight : nullptr, a ? a->y : nullptr);
    return rc != SMB_OK ? rc : conv3d_run("smb_conv3d", a, 0, a->x, a->weight, a->y, cuda_stream);
}

SMB_API int smb_conv3d_wgrad(const smb_conv3d_args *a, void *cuda_stream) {
    int rc = conv3d_check("smb_conv3d_wgrad", a, a ? a->x : nullptr, a ? a->dy : nullptr, a ? a->dweight : nullptr);
    return rc != SMB_OK ? rc : conv3d_run("smb_conv3d_wgrad", a, 1, a->x, a->dy, a->dweight, cuda_stream);
}

SMB_API int smb_copy2d(const void *src, int64_t src_pitch_bytes, void *dst, int64_t dst_pitch_bytes, int64_t rows, int64_t row_bytes,
                       void *cuda_stream) {
    if (!src || !dst) return fail(SMB_EINVAL, "smb_copy2d: src and dst are required");
    if (rows < 0 || row_bytes <= 0) return fail(SMB_EINVAL, "smb_copy2d: bad extent");
    if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst) | (uintptr_t)src_pitch_bytes | (uintptr_t)dst_pitch_bytes |
          (uintptr_t)row_bytes) & 15) != 0)
        return fail(SMB_EINVAL, "smb_copy2d: pointers, pitches and row_bytes must be multiples of 16 bytes");
    if (src_pitch_bytes < row_bytes || dst_pitch_bytes < row_bytes) return fail(SMB_EINVAL, "smb_copy2d: pitch smaller than the row");
    if (rows == 0) return SMB_OK;
    cudaError_t e = smb::copy2d_launch(src, src_pitch_bytes, dst, dst_pitch_bytes, rows, row_bytes, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_copy2d");
    return SMB_OK;
}

// ---------------------------------------------------------------------------------------------
// training-patch augmentation (augment.cu)
static bool aug_axis_ok(int n) { return n >= 1 && n <= smb::kAugMaxAxis; }

SMB_API int smb_aug_crop(const smb_aug_crop_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_aug_crop: null args");
    if (a->batch <= 0 || a->channels <= 0 || !aug_axis_ok(a->pd) || !aug_axis_ok(a->ph) || !aug_axis_ok(a->pw))
        return fail(SMB_EINVAL, "smb_aug_crop: batch, channels must be positive and patch axes in 1..%d", smb::kAugMaxAxis);
    if (!a->cases || !a->data || !a->seg) return fail(SMB_EINVAL, "smb_aug_crop: cases, data, seg are required");
    for (int s = 0; s < a->batch; ++s) {
        const smb_aug_case &c = a->cases[s];
        if (!c.data || !c.seg || c.D <= 0 || c.H <= 0 || c.W <= 0) return fail(SMB_EINVAL, "smb_aug_crop: case %d has no data / seg or an empty shape", s);
    }
    cudaError_t e = smb::aug_crop_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_aug_crop");
    return SMB_OK;
}

SMB_API int smb_aug_prefilter(const smb_aug_prefilter_job *jobs, int32_t n_jobs, void *cuda_stream) {
    if (n_jobs < 0 || (n_jobs > 0 && !jobs)) return fail(SMB_EINVAL, "smb_aug_prefilter: bad job list");
    for (int q = 0; q < n_jobs; ++q) {
        const smb_aug_prefilter_job &j = jobs[q];
        if (!j.src || !j.coef) return fail(SMB_EINVAL, "smb_aug_prefilter: job %d needs src and coef", q);
        if (j.n0 < 4 || j.n1 < 4 || j.n2 < 4) return fail(SMB_EUNSUPPORTED, "smb_aug_prefilter: job %d: axes must be at least 4 samples", q);
        if (j.boundary != SMB_AUG_MIRROR && j.boundary != SMB_AUG_EDGE) return fail(SMB_EINVAL, "smb_aug_prefilter: job %d: bad boundary", q);
        if (j.boundary == SMB_AUG_MIRROR && (j.n0 > smb::kAugMaxAxis || j.n1 > smb::kAugMaxAxis || j.n2 > smb::kAugMaxAxis))
            return fail(SMB_EUNSUPPORTED, "smb_aug_prefilter: job %d: mirror-boundary axes must be 4..%d samples", q, smb::kAugMaxAxis);
        if ((int64_t)(j.n0 + 4) * (j.n1 + 4) * (j.n2 + 4) > INT32_MAX)
            return fail(SMB_EUNSUPPORTED, "smb_aug_prefilter: job %d: the coefficient grid is limited to 2^31 - 1 voxels", q);
    }
    cudaError_t e = smb::aug_prefilter_launch(jobs, n_jobs, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_aug_prefilter");
    return SMB_OK;
}

SMB_API int smb_aug_resample(const smb_aug_resample_job *jobs, int32_t n_jobs, void *cuda_stream) {
    if (n_jobs < 0 || (n_jobs > 0 && !jobs)) return fail(SMB_EINVAL, "smb_aug_resample: bad job list");
    for (int q = 0; q < n_jobs; ++q) {
        const smb_aug_resample_job &j = jobs[q];
        if (!j.src || !j.dst) return fail(SMB_EINVAL, "smb_aug_resample: job %d needs src and dst", q);
        if (j.n0 < 1 || j.n1 < 1 || j.n2 < 1 || j.m0 < 1 || j.m1 < 1 || j.m2 < 1)
            return fail(SMB_EUNSUPPORTED, "smb_aug_resample: job %d: axes must be positive", q);
        const int b = j.order == 3 ? 4 : 0;                           // order 3 reads the border-extended coefficient grid
        if ((int64_t)(j.n0 + b) * (j.n1 + b) * (j.n2 + b) > INT32_MAX || (int64_t)j.m0 * j.m1 * j.m2 > INT32_MAX)
            return fail(SMB_EUNSUPPORTED, "smb_aug_resample: job %d: source and output are limited to 2^31 - 1 voxels", q);
        if (j.order != 0 && j.order != 1 && j.order != 3) return fail(SMB_EUNSUPPORTED, "smb_aug_resample: job %d: order %d (0, 1, 3)", q, j.order);
        if (j.map != SMB_AUG_AFFINE && j.map != SMB_AUG_ZOOM) return fail(SMB_EINVAL, "smb_aug_resample: job %d: bad map", q);
        if (j.order == 1 && (j.map != SMB_AUG_AFFINE || j.clip)) return fail(SMB_EUNSUPPORTED, "smb_aug_resample: job %d: labels take an affine map, no clip", q);
    }
    cudaError_t e = smb::aug_resample_launch(jobs, n_jobs, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_aug_resample");
    return SMB_OK;
}

SMB_API int smb_aug_blur(const smb_aug_blur_job *jobs, int32_t n_jobs, void *cuda_stream) {
    if (n_jobs < 0 || (n_jobs > 0 && !jobs)) return fail(SMB_EINVAL, "smb_aug_blur: bad job list");
    for (int q = 0; q < n_jobs; ++q) {
        const smb_aug_blur_job &j = jobs[q];
        if (!j.x || !j.tmp) return fail(SMB_EINVAL, "smb_aug_blur: job %d needs x and tmp", q);
        if (!aug_axis_ok(j.n0) || !aug_axis_ok(j.n1) || !aug_axis_ok(j.n2)) return fail(SMB_EUNSUPPORTED, "smb_aug_blur: job %d: bad shape", q);
        if (!(j.sigma > 0.f && j.sigma <= 2.f)) return fail(SMB_EUNSUPPORTED, "smb_aug_blur: job %d: sigma must be in (0, 2]", q);
    }
    cudaError_t e = smb::aug_blur_launch(jobs, n_jobs, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_aug_blur");
    return SMB_OK;
}

SMB_API int smb_aug_stats(const smb_aug_stats_job *jobs, int32_t n_jobs, void *cuda_stream) {
    if (n_jobs < 0 || (n_jobs > 0 && !jobs)) return fail(SMB_EINVAL, "smb_aug_stats: bad job list");
    for (int q = 0; q < n_jobs; ++q)
        if (!jobs[q].x || !jobs[q].stats || !jobs[q].scratch || jobs[q].n <= 0) return fail(SMB_EINVAL, "smb_aug_stats: job %d: x, stats, scratch, n > 0 required", q);
    cudaError_t e = smb::aug_stats_launch(jobs, n_jobs, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_aug_stats");
    return SMB_OK;
}

SMB_API int smb_aug_pointwise(const smb_aug_point_job *jobs, int32_t n_jobs, void *cuda_stream) {
    if (n_jobs < 0 || (n_jobs > 0 && !jobs)) return fail(SMB_EINVAL, "smb_aug_pointwise: bad job list");
    for (int q = 0; q < n_jobs; ++q) {
        const smb_aug_point_job &j = jobs[q];
        if (!j.x || j.n <= 0) return fail(SMB_EINVAL, "smb_aug_pointwise: job %d: x and n > 0 required", q);
        if ((j.ops & ~127) != 0) return fail(SMB_EINVAL, "smb_aug_pointwise: job %d: unknown op bits", q);
        if ((j.ops & (SMB_AUG_OP_RETAIN | SMB_AUG_OP_CONTRAST | SMB_AUG_OP_GAMMA)) && !j.stats)
            return fail(SMB_EINVAL, "smb_aug_pointwise: job %d: retain / contrast / gamma need stats", q);
        if ((j.ops & SMB_AUG_OP_RETAIN) && !j.retain_ref) return fail(SMB_EINVAL, "smb_aug_pointwise: job %d: retain needs retain_ref", q);
        const int nonlinear_before_stats =
            ((j.ops & SMB_AUG_OP_NOISE) && (j.ops & (SMB_AUG_OP_CONTRAST | SMB_AUG_OP_GAMMA))) ||
            ((j.ops & SMB_AUG_OP_CONTRAST) && (j.ops & SMB_AUG_OP_GAMMA));
        if (nonlinear_before_stats) return fail(SMB_EINVAL, "smb_aug_pointwise: job %d: a statistics-driven step follows a nonlinear one", q);
    }
    cudaError_t e = smb::aug_pointwise_launch(jobs, n_jobs, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_aug_pointwise");
    return SMB_OK;
}

SMB_API int smb_aug_emit(const smb_aug_emit_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_aug_emit: null args");
    if (a->batch <= 0 || a->channels <= 0 || !aug_axis_ok(a->pd) || !aug_axis_ok(a->ph) || !aug_axis_ok(a->pw))
        return fail(SMB_EINVAL, "smb_aug_emit: bad shape");
    if (a->out_dtype < SMB_F32 || a->out_dtype > SMB_BF16) return fail(SMB_EINVAL, "smb_aug_emit: bad out_dtype %d", a->out_dtype);
    if (!a->samples || !a->image || !a->label) return fail(SMB_EINVAL, "smb_aug_emit: samples, image, label are required");
    for (int s = 0; s < a->batch; ++s)
        if (!a->samples[s].data || !a->samples[s].seg) return fail(SMB_EINVAL, "smb_aug_emit: sample %d needs data and seg", s);
    cudaError_t e = smb::aug_emit_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_aug_emit");
    return SMB_OK;
}

// segmentation metrics (metrics.cu)
static int metric_shape(int batch, int regions, int d, int h, int w, const char *who) {
    if (batch <= 0 || batch > 65535 || d <= 0 || h <= 0 || w <= 0) return fail(SMB_EINVAL, "%s: batch (1..65535) and axes must be positive", who);
    if (regions <= 0 || regions > SMB_METRIC_MAX_REGIONS) return fail(SMB_EINVAL, "%s: regions must be 1..%d", who, SMB_METRIC_MAX_REGIONS);
    if (h > SMB_METRIC_MAX_AXIS || w > SMB_METRIC_MAX_AXIS) return fail(SMB_EUNSUPPORTED, "%s: axes 1 and 2 are limited to %d voxels", who, SMB_METRIC_MAX_AXIS);
    if ((int64_t)d * h * w > INT32_MAX) return fail(SMB_EUNSUPPORTED, "%s: volumes are limited to 2^31 - 1 voxels", who);
    return SMB_OK;
}

SMB_API int smb_metric_region_bits(const smb_metric_bits_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_metric_region_bits: null args");
    if (!a->src || !a->bits) return fail(SMB_EINVAL, "smb_metric_region_bits: src and bits are required");
    if (a->batch <= 0 || a->batch > 65535 || a->voxels <= 0) return fail(SMB_EINVAL, "smb_metric_region_bits: batch (1..65535) and voxels must be positive");
    if (a->sample_stride < 0 || a->voxel_stride <= 0) return fail(SMB_EINVAL, "smb_metric_region_bits: bad strides");
    if (a->kind < SMB_METRIC_I8 || a->kind > SMB_METRIC_I16) return fail(SMB_EINVAL, "smb_metric_region_bits: bad kind %d", a->kind);
    if (a->kind == SMB_METRIC_LOGITS) {
        if (a->dtype < SMB_F32 || a->dtype > SMB_BF16) return fail(SMB_EINVAL, "smb_metric_region_bits: bad dtype %d", a->dtype);
        if (a->classes <= 0 || a->class_stride <= 0) return fail(SMB_EINVAL, "smb_metric_region_bits: logits need classes and class_stride > 0");
    }
    cudaError_t e = smb::metric_bits_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_metric_region_bits");
    return SMB_OK;
}

SMB_API int smb_metric_count(const smb_metric_count_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_metric_count: null args");
    int rc = metric_shape(a->batch, a->regions, a->d, a->h, a->w, "smb_metric_count");
    if (rc != SMB_OK) return rc;
    if (!a->pred || !a->target || !a->pred_border || !a->target_border || !a->counts)
        return fail(SMB_EINVAL, "smb_metric_count: pred, target, pred_border, target_border, counts are required");
    cudaError_t e = smb::metric_count_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_metric_count");
    return SMB_OK;
}

SMB_API int smb_metric_edt(const smb_metric_edt_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_metric_edt: null args");
    int rc = metric_shape(a->batch, a->regions, a->d, a->h, a->w, "smb_metric_edt");
    if (rc != SMB_OK) return rc;
    if (a->batch * a->regions * 2 > 65535) return fail(SMB_EUNSUPPORTED, "smb_metric_edt: batch * regions * 2 is limited to 65535");
    if (!a->pred_border || !a->target_border || !a->feat || !a->pool || !a->counts)
        return fail(SMB_EINVAL, "smb_metric_edt: pred_border, target_border, feat, pool, counts are required");
    if (a->pool_cap < 2 * (int64_t)a->d * a->h * a->w) return fail(SMB_EWORKSPACE, "smb_metric_edt: pool_cap must be at least 2 * d * h * w");
    if (!(a->s0 > 0.0 && a->s1 > 0.0 && a->s2 > 0.0) || !std::isfinite(a->s0 * a->s1 * a->s2))
        return fail(SMB_EINVAL, "smb_metric_edt: spacing must be positive and finite");
    cudaError_t e = smb::metric_edt_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_metric_edt");
    return SMB_OK;
}

SMB_API int smb_metric_select(const smb_metric_select_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_metric_select: null args");
    if (!a->pool || !a->counts || !a->out) return fail(SMB_EINVAL, "smb_metric_select: pool, counts, out are required");
    if (a->batch <= 0 || a->regions <= 0 || a->regions > SMB_METRIC_MAX_REGIONS || a->pool_cap <= 0 || (int64_t)a->batch * a->regions > INT32_MAX)
        return fail(SMB_EINVAL, "smb_metric_select: bad batch / regions / pool_cap");
    if (!(a->frac >= 0.0 && a->frac <= 1.0)) return fail(SMB_EINVAL, "smb_metric_select: frac must be in [0, 1]");
    cudaError_t e = smb::metric_select_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_metric_select");
    return SMB_OK;
}

SMB_API int smb_metric_class_count(const smb_metric_class_count_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_metric_class_count: null args");
    if (a->batch <= 0 || a->batch > 65535 || a->d <= 0 || a->h <= 0 || a->w <= 0)
        return fail(SMB_EINVAL, "smb_metric_class_count: batch (1..65535) and axes must be positive");
    if (a->classes <= 0 || a->classes > SMB_METRIC_MAX_CLASSES) return fail(SMB_EINVAL, "smb_metric_class_count: classes must be 1..%d", SMB_METRIC_MAX_CLASSES);
    if ((int64_t)a->d * a->h * a->w > INT32_MAX) return fail(SMB_EUNSUPPORTED, "smb_metric_class_count: volumes are limited to 2^31 - 1 voxels");
    if (!a->pred || !a->target || !a->pred_border || !a->target_border || !a->record)
        return fail(SMB_EINVAL, "smb_metric_class_count: pred, target, pred_border, target_border, record are required");
    cudaError_t e = smb::metric_class_count_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_metric_class_count");
    return SMB_OK;
}

SMB_API int smb_metric_class_edt(const smb_metric_class_edt_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_metric_class_edt: null args");
    if (!a->jobs) return fail(SMB_EINVAL, "smb_metric_class_edt: jobs is required");
    if (a->njobs <= 0 || a->njobs > 65535) return fail(SMB_EUNSUPPORTED, "smb_metric_class_edt: njobs must be 1..65535");
    if (a->max_d <= 0 || a->max_h <= 0 || a->max_w <= 0) return fail(SMB_EINVAL, "smb_metric_class_edt: box bounds must be positive");
    if (a->max_h > SMB_METRIC_MAX_AXIS || a->max_w > SMB_METRIC_MAX_AXIS)
        return fail(SMB_EUNSUPPORTED, "smb_metric_class_edt: box axes 1 and 2 are limited to %d voxels", SMB_METRIC_MAX_AXIS);
    if (a->row_stride < a->max_w || a->slice_stride < a->row_stride * a->max_h)
        return fail(SMB_EINVAL, "smb_metric_class_edt: the map strides must cover the box bounds");
    if (!(a->s0 > 0.0 && a->s1 > 0.0 && a->s2 > 0.0) || !std::isfinite(a->s0 * a->s1 * a->s2))
        return fail(SMB_EINVAL, "smb_metric_class_edt: spacing must be positive and finite");
    cudaError_t e = smb::metric_class_edt_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_metric_class_edt");
    return SMB_OK;
}

SMB_API int smb_metric_class_reduce(const smb_metric_class_reduce_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_metric_class_reduce: null args");
    if (!a->pools || !a->out) return fail(SMB_EINVAL, "smb_metric_class_reduce: pools and out are required");
    if (a->npools <= 0) return fail(SMB_EINVAL, "smb_metric_class_reduce: npools must be positive");
    if (!(a->frac >= 0.0 && a->frac <= 1.0)) return fail(SMB_EINVAL, "smb_metric_class_reduce: frac must be in [0, 1]");
    cudaError_t e = smb::metric_class_reduce_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_metric_class_reduce");
    return SMB_OK;
}

// case prediction (predict.cu)
SMB_API int smb_pred_restore(const smb_pred_restore_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_pred_restore: null args");
    if (!a->src || !a->out) return fail(SMB_EINVAL, "smb_pred_restore: src and out are required");
    if (a->dtype < SMB_F32 || a->dtype > SMB_BF16) return fail(SMB_EINVAL, "smb_pred_restore: bad dtype %d", a->dtype);
    if (a->classes <= 0 || a->classes > 256) return fail(SMB_EINVAL, "smb_pred_restore: classes must be 1..256");
    if (a->class_stride <= 0 || a->voxel_stride <= 0) return fail(SMB_EINVAL, "smb_pred_restore: strides must be positive");
    if (a->regions < 0 || a->regions > SMB_METRIC_MAX_REGIONS) return fail(SMB_EINVAL, "smb_pred_restore: regions must be 0..%d", SMB_METRIC_MAX_REGIONS);
    if (a->d <= 0 || a->h <= 0 || a->w <= 0 || a->cd <= 0 || a->ch <= 0 || a->cw <= 0 || a->D0 <= 0 || a->H0 <= 0 || a->W0 <= 0)
        return fail(SMB_EINVAL, "smb_pred_restore: every axis must be positive");
    if (a->z0 < 0 || a->y0 < 0 || a->x0 < 0 || (int64_t)a->z0 + a->cd > a->D0 || (int64_t)a->y0 + a->ch > a->H0 || (int64_t)a->x0 + a->cw > a->W0)
        return fail(SMB_EINVAL, "smb_pred_restore: the crop box must lie inside the original volume");
    if ((int64_t)a->d * a->h * a->w > INT32_MAX || (int64_t)a->D0 * a->H0 * a->W0 > INT32_MAX)
        return fail(SMB_EUNSUPPORTED, "smb_pred_restore: volumes are limited to 2^31 - 1 voxels");
    cudaError_t e = smb::pred_restore_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_pred_restore");
    return SMB_OK;
}

SMB_API size_t smb_pred_cc_workspace_bytes(int32_t batch, int32_t d, int32_t h, int32_t w) {
    if (batch <= 0 || d <= 0 || h <= 0 || w <= 0) return 0;
    return smb::pred_cc_workspace_bytes(batch, d, h, w);
}

SMB_API int smb_pred_cc(const smb_pred_cc_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_pred_cc: null args");
    if (!a->mask || !a->out) return fail(SMB_EINVAL, "smb_pred_cc: mask and out are required");
    if (a->batch <= 0 || a->batch > 65535 || a->d <= 0 || a->h <= 0 || a->w <= 0)
        return fail(SMB_EINVAL, "smb_pred_cc: batch (1..65535) and axes must be positive");
    if ((int64_t)a->d * a->h * a->w > INT32_MAX) return fail(SMB_EUNSUPPORTED, "smb_pred_cc: volumes are limited to 2^31 - 1 voxels");
    if (a->op < SMB_PRED_LABEL || a->op > SMB_PRED_LARGEST) return fail(SMB_EINVAL, "smb_pred_cc: bad op %d", a->op);
    if (a->op == SMB_PRED_LABEL && !a->counts) return fail(SMB_EINVAL, "smb_pred_cc: labelling needs counts");
    if (!a->workspace || ((uintptr_t)a->workspace & 15) || a->workspace_bytes < smb::pred_cc_workspace_bytes(a->batch, a->d, a->h, a->w))
        return fail(SMB_EWORKSPACE, "smb_pred_cc: workspace missing, misaligned or smaller than smb_pred_cc_workspace_bytes");
    cudaError_t e = smb::pred_cc_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_pred_cc");
    return SMB_OK;
}

// case preprocessing (preprocess.cu)
static int prep_volume(int64_t d, int64_t h, int64_t w, const char *who) {
    if (d <= 0 || h <= 0 || w <= 0) return fail(SMB_EINVAL, "%s: axes must be positive", who);
    if (d * h * w > INT32_MAX) return fail(SMB_EUNSUPPORTED, "%s: volumes are limited to 2^31 - 1 voxels", who);
    return SMB_OK;
}

SMB_API int smb_prep_mask(const smb_prep_mask_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_prep_mask: null args");
    if (!a->data || !a->mask || !a->seg8 || !a->record) return fail(SMB_EINVAL, "smb_prep_mask: data, mask, seg8, record are required");
    if (a->channels <= 0) return fail(SMB_EINVAL, "smb_prep_mask: channels must be positive");
    int rc = prep_volume(a->d, a->h, a->w, "smb_prep_mask");
    if (rc != SMB_OK) return rc;
    cudaError_t e = smb::prep_mask_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_prep_mask");
    return SMB_OK;
}

SMB_API int smb_prep_crop(const smb_prep_crop_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_prep_crop: null args");
    if (!a->data || !a->mask || !a->seg8 || !a->out || !a->seg_out) return fail(SMB_EINVAL, "smb_prep_crop: data, mask, seg8, out, seg_out are required");
    if (a->channels <= 0) return fail(SMB_EINVAL, "smb_prep_crop: channels must be positive");
    int rc = prep_volume(a->d, a->h, a->w, "smb_prep_crop");
    if (rc != SMB_OK) return rc;
    if (a->cd <= 0 || a->ch <= 0 || a->cw <= 0 || a->z0 < 0 || a->y0 < 0 || a->x0 < 0 || (int64_t)a->z0 + a->cd > a->d ||
        (int64_t)a->y0 + a->ch > a->h || (int64_t)a->x0 + a->cw > a->w)
        return fail(SMB_EINVAL, "smb_prep_crop: the box must be non-empty and lie inside the volume");
    if (a->nonzero_label < -128 || a->nonzero_label > 127) return fail(SMB_EINVAL, "smb_prep_crop: nonzero_label must fit int8");
    cudaError_t e = smb::prep_crop_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_prep_crop");
    return SMB_OK;
}

SMB_API int smb_prep_normalize(const smb_prep_norm_job *jobs, int32_t n_jobs, void *cuda_stream) {
    if (n_jobs < 0 || (n_jobs > 0 && !jobs)) return fail(SMB_EINVAL, "smb_prep_normalize: bad job list");
    for (int q = 0; q < n_jobs; ++q)
        if (!jobs[q].src || !jobs[q].dst || !jobs[q].stats || !jobs[q].moments || jobs[q].n <= 0)
            return fail(SMB_EINVAL, "smb_prep_normalize: job %d: src, dst, stats, moments, n > 0 required", q);
    cudaError_t e = smb::prep_normalize_launch(jobs, n_jobs, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_prep_normalize");
    return SMB_OK;
}

SMB_API int smb_prep_ct_normalize(const smb_prep_ct_norm_job *jobs, int32_t n_jobs, void *cuda_stream) {
    if (n_jobs < 0 || (n_jobs > 0 && !jobs)) return fail(SMB_EINVAL, "smb_prep_ct_normalize: bad job list");
    for (int q = 0; q < n_jobs; ++q)
        if (!jobs[q].src || !jobs[q].dst || jobs[q].n <= 0)
            return fail(SMB_EINVAL, "smb_prep_ct_normalize: job %d: src, dst, n > 0 required", q);
    cudaError_t e = smb::prep_ct_normalize_launch(jobs, n_jobs, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_prep_ct_normalize");
    return SMB_OK;
}

SMB_API int smb_prep_label_resize(const smb_prep_label_resize_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_prep_label_resize: null args");
    if (!a->src || !a->dst) return fail(SMB_EINVAL, "smb_prep_label_resize: src and dst are required");
    int rc = prep_volume(a->n0, a->n1, a->n2, "smb_prep_label_resize");
    if (rc == SMB_OK) rc = prep_volume(a->m0, a->m1, a->m2, "smb_prep_label_resize");
    if (rc != SMB_OK) return rc;
    cudaError_t e = smb::prep_label_resize_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_prep_label_resize");
    return SMB_OK;
}

static int prep_jobs(const smb_prep_compact_job *jobs, int32_t n_jobs, bool compact, const char *who) {
    if (n_jobs < 0 || (n_jobs > 0 && !jobs)) return fail(SMB_EINVAL, "%s: bad job list", who);
    for (int q = 0; q < n_jobs; ++q) {
        const smb_prep_compact_job &j = jobs[q];
        if (!j.seg || !j.chunk || !j.count || (compact && !j.index)) return fail(SMB_EINVAL, "%s: job %d lacks a buffer", who, q);
        if (j.n <= 0 || j.n > INT32_MAX) return fail(SMB_EUNSUPPORTED, "%s: job %d: n must be 1..2^31 - 1", who, q);
    }
    return SMB_OK;
}

SMB_API int smb_prep_count(const smb_prep_compact_job *jobs, int32_t n_jobs, void *cuda_stream) {
    int rc = prep_jobs(jobs, n_jobs, false, "smb_prep_count");
    if (rc != SMB_OK) return rc;
    cudaError_t e = smb::prep_count_launch(jobs, n_jobs, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_prep_count");
    return SMB_OK;
}

SMB_API int smb_prep_compact(const smb_prep_compact_job *jobs, int32_t n_jobs, void *cuda_stream) {
    int rc = prep_jobs(jobs, n_jobs, true, "smb_prep_compact");
    if (rc != SMB_OK) return rc;
    cudaError_t e = smb::prep_compact_launch(jobs, n_jobs, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_prep_compact");
    return SMB_OK;
}

SMB_API int smb_prep_gather(const smb_prep_gather_args *a, void *cuda_stream) {
    if (!a) return fail(SMB_EINVAL, "smb_prep_gather: null args");
    if (!a->index || (!a->rows && !a->values)) return fail(SMB_EINVAL, "smb_prep_gather: index and rows or values are required");
    if (a->n < 0) return fail(SMB_EINVAL, "smb_prep_gather: n must be non-negative");
    if (a->rows && prep_volume(a->d, a->h, a->w, "smb_prep_gather") != SMB_OK) return SMB_EINVAL;
    if (a->values && (!a->data || a->channels <= 0 || a->channel_stride < 0 || a->select_channel_stride < 0))
        return fail(SMB_EINVAL, "smb_prep_gather: values need data, channels > 0 and non-negative strides");
    cudaError_t e = smb::prep_gather_launch(*a, (cudaStream_t)cuda_stream);
    if (e != cudaSuccess) return cuda_fail(e, "smb_prep_gather");
    return SMB_OK;
}

}  // extern "C"
