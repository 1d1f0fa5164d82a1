// 16-bit activation tiles kept in their storage type and filled with cp.async: layout, fills, stores and per-lane unit access
// shared by the software-pipelined lane-per-channel kernels (scan_fwd_v2.cu, the pipelined R1 in scan_bwd.cu).
//
// A tile is 32 rows (channels) x 32 scan positions of a 2-byte type: 64-byte rows whose four 16-byte units are XOR-swizzled with
// (row >> 1) & 3.  Compute phase: lane == row reads one unit (8 positions) with one LDS.128 -- 32 lanes x 16 B = 4 wavefronts,
// and the swizzle puts exactly 4 lanes on each of the 8 sixteen-byte slots of the 128-byte bank window.  Fill / store phase:
// lane (r, c) moves the 8-byte chunk c of rows r, r+4, ... -- 4 rows x 64 contiguous bytes per instruction, 2 wavefronts.
#pragma once

#include "async_copy.cuh"

namespace smb {

constexpr int kRawTileBytes = kTile * kTile * 2;     // 32 rows x 32 positions of a 2-byte type

// byte offset of 16-byte unit `unit` (8 scan positions) of row `row`
__device__ __forceinline__ int raw_unit_off(int row, int unit) { return row * 64 + ((unit ^ ((row >> 1) & 3)) << 4); }
// byte offset of 8-byte chunk `c` (4 scan positions) of row `row`
__device__ __forceinline__ int raw_chunk_off(int row, int c) { return raw_unit_off(row, c >> 1) + ((c & 1) << 3); }

template <typename T> __device__ __forceinline__ void unpack8(uint4 r, float (&v)[8]);
template <> __device__ __forceinline__ void unpack8<__nv_bfloat16>(uint4 r, float (&v)[8]) {
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        v[2 * i] = __uint_as_float(w[i] << 16);
        v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
}
template <> __device__ __forceinline__ void unpack8<__half>(uint4 r, float (&v)[8]) {
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&w[i]));
        v[2 * i] = f.x;
        v[2 * i + 1] = f.y;
    }
}
template <typename T> __device__ __forceinline__ uint4 pack8(const float (&v)[8]);
template <> __device__ __forceinline__ uint4 pack8<__nv_bfloat16>(const float (&v)[8]) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const __nv_bfloat162 b = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
        w[i] = *reinterpret_cast<const uint32_t *>(&b);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}
template <> __device__ __forceinline__ uint4 pack8<__half>(const float (&v)[8]) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const __half2 b = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
        w[i] = *reinterpret_cast<const uint32_t *>(&b);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// memory order <-> scan order inside one unit.  A reversed walk copies each 4-position chunk as it lies in memory (ascending
// tokens = descending scan positions), so the chunk is mirrored when it is read and when a result is written back; the
// permutation is its own inverse.
template <bool kRev> __device__ __forceinline__ void mirror_chunks(float (&v)[8]) {
    if (kRev) {
        float t;
        t = v[0]; v[0] = v[3]; v[3] = t;
        t = v[1]; v[1] = v[2]; v[2] = t;
        t = v[4]; v[4] = v[7]; v[7] = t;
        t = v[5]; v[5] = v[6]; v[6] = t;
    }
}

// ---- asynchronous fills: REQUIRE j0 + 32 <= L and 8-byte aligned chunks (stream_aligned / bc_aligned) ----
template <typename T>
__device__ __forceinline__ void issue_tile(unsigned char *tile, const LanePtr<T> &lp, int nrows, int j0, bool reverse, int lane) {
    const int64_t toff = reverse ? -(int64_t)j0 : (int64_t)j0;
    const int row0 = lane >> 3, c = lane & 7;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int row = row0 + 4 * it;
        if (row < nrows) cp_async8(tile + raw_chunk_off(row, c), lp.lp + toff + it * lp.rowstep);
    }
}
template <typename T, int N>
__device__ __forceinline__ void issue_bc(T *raw, const T *base, int64_t ns, int j0, int L, bool reverse, int lane) {
    const int tok0 = reverse ? L - kTile - j0 : j0;                     // lowest token of the tile
#pragma unroll
    for (int it = 0; it < N / 4; ++it) {
        const int k = lane + 32 * it, n = k >> 3, c = k & 7;
        cp_async8(raw + n * kTile + 4 * c, base + (int64_t)n * ns + tok0 + 4 * c);
    }
}
template <typename T> __device__ __forceinline__ bool bc_aligned(const T *base, int64_t ns, int L, bool reverse) {
    return aligned4(base) && (ns & 3) == 0 && (!reverse || (L & 3) == 0);
}
// raw (state-major, token-ascending) staging rows -> position-major fp32 broadcast tile; lane == scan position
template <typename T, int N, bool kRev> __device__ __forceinline__ void convert_bc(float *tile, const T *raw, int lane) {
    const int src = kRev ? kTile - 1 - lane : lane;
    constexpr int kRound = N > 32 ? 32 : N;      // states per round: bounds the registers of the transposing copy
#pragma unroll
    for (int n0 = 0; n0 < N; n0 += kRound) {
        T v[kRound];
#pragma unroll
        for (int n = 0; n < kRound; ++n) v[n] = raw[(n0 + n) * kTile + src];
#pragma unroll
        for (int n = 0; n < kRound; ++n) tile[bc_off<N>(lane, n0 + n)] = to_f32<T>(v[n]);
    }
}

// ---- synchronous fill / store of a stage tile for ragged or unaligned tiles (same layout, bounds-checked) ----
template <typename T, bool kRev>
__device__ __forceinline__ void fill_raw_sync(unsigned char *tile, const T *base, int64_t row_stride, int nrows, int j0, int L, int lane) {
    const int row0 = lane >> 3, c = lane & 7;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int row = row0 + 4 * it;
        T vals[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int pos = j0 + 4 * c + e;
            const bool ok = row < nrows && pos < L;
            vals[kRev ? 3 - e : e] = ok ? base[(int64_t)row * row_stride + (kRev ? L - 1 - pos : pos)] : from_f32<T>(0.f);
        }
        *reinterpret_cast<uint2 *>(tile + raw_chunk_off(row, c)) = *reinterpret_cast<const uint2 *>(vals);
    }
}
template <typename T, bool kRev>
__device__ __forceinline__ void store_raw_sync(const unsigned char *tile, T *base, int64_t row_stride, int nrows, int j0, int L, int lane) {
    const int row0 = lane >> 3, c = lane & 7;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int row = row0 + 4 * it;
        if (row >= nrows) continue;
        T vals[4];
        *reinterpret_cast<uint2 *>(vals) = *reinterpret_cast<const uint2 *>(tile + raw_chunk_off(row, c));
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int pos = j0 + 4 * c + e;
            if (pos < L) base[(int64_t)row * row_stride + (kRev ? L - 1 - pos : pos)] = vals[kRev ? 3 - e : e];
        }
    }
}
// full, aligned tile: 8-byte coalesced stores with the lane mapping of the fills
template <typename T>
__device__ __forceinline__ void store_raw_fast(const unsigned char *tile, T *lp, int64_t rowstep, int nrows, int j0, bool reverse, int lane) {
    const int64_t toff = reverse ? -(int64_t)j0 : (int64_t)j0;
    const int row0 = lane >> 3, c = lane & 7;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int row = row0 + 4 * it;
        if (row < nrows) *reinterpret_cast<uint2 *>(lp + toff + it * rowstep) = *reinterpret_cast<const uint2 *>(tile + raw_chunk_off(row, c));
    }
}

// this lane's 8 positions of unit `u8`, in scan order, as fp32
template <typename T, bool kRev> __device__ __forceinline__ void read_unit(const unsigned char *tile, int lane, int u8, float (&v)[8]) {
    unpack8<T>(*reinterpret_cast<const uint4 *>(tile + raw_unit_off(lane, u8)), v);
    mirror_chunks<kRev>(v);
}
template <typename T, bool kRev> __device__ __forceinline__ void write_unit(unsigned char *tile, int lane, int u8, float (&v)[8]) {
    mirror_chunks<kRev>(v);
    *reinterpret_cast<uint4 *>(tile + raw_unit_off(lane, u8)) = pack8<T>(v);
}
// dt = softplus?(delta + bias) for the unit's 8 positions; positions at or beyond nvalid become scan identities (dt = 0)
__device__ __forceinline__ void unit_dt(float (&dd)[8], float bias, bool softplus, int first_pos, int nvalid) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        float x = dd[e] + bias;
        if (softplus) x = softplus20(x);
        dd[e] = first_pos + e < nvalid ? x : 0.f;
    }
}

// ---- token-ascending tile layout: what a TMA box copy produces.  Slot s of a row holds token tok0 + s, where tok0 is the lowest
// token of the tile (j0 for a forward walk, L - 32 - j0 for a reversed one); scan position p of the tile lives in slot p
// (forward) or 31 - p (reversed).  Same 64-byte rows and 16-byte-unit swizzle as above. ----
__device__ __forceinline__ void reverse8(float (&v)[8]) {
    float t;
    t = v[0]; v[0] = v[7]; v[7] = t;
    t = v[1]; v[1] = v[6]; v[6] = t;
    t = v[2]; v[2] = v[5]; v[5] = t;
    t = v[3]; v[3] = v[4]; v[4] = t;
}
template <typename T, bool kRev> __device__ __forceinline__ void read_unit_asc(const unsigned char *tile, int lane, int u8, float (&v)[8]) {
    unpack8<T>(*reinterpret_cast<const uint4 *>(tile + raw_unit_off(lane, kRev ? 3 - u8 : u8)), v);
    if (kRev) reverse8(v);
}
template <typename T, bool kRev> __device__ __forceinline__ void write_unit_asc(unsigned char *tile, int lane, int u8, float (&v)[8]) {
    if (kRev) reverse8(v);
    *reinterpret_cast<uint4 *>(tile + raw_unit_off(lane, kRev ? 3 - u8 : u8)) = pack8<T>(v);
}
// full tile, 8-byte aligned rows: row0 points at (row 0, token tok0)
template <typename T>
__device__ __forceinline__ void store_asc_fast(const unsigned char *tile, T *row0, int64_t row_stride, int nrows, int lane) {
    const int r0 = lane >> 3, c = lane & 7;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int row = r0 + 4 * it;
        if (row < nrows) *reinterpret_cast<uint2 *>(row0 + (int64_t)row * row_stride + 4 * c) = *reinterpret_cast<const uint2 *>(tile + raw_chunk_off(row, c));
    }
}
template <typename T, bool kRev>
__device__ __forceinline__ void store_asc_sync(const unsigned char *tile, T *base, int64_t row_stride, int nrows, int j0, int L, int lane) {
    const int r0 = lane >> 3, c = lane & 7;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int row = r0 + 4 * it;
        if (row >= nrows) continue;
        T vals[4];
        *reinterpret_cast<uint2 *>(vals) = *reinterpret_cast<const uint2 *>(tile + raw_chunk_off(row, c));
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int slot = 4 * c + e;
            const int pos = j0 + (kRev ? kTile - 1 - slot : slot);
            if (pos < L) base[(int64_t)row * row_stride + (kRev ? L - 1 - pos : pos)] = vals[e];
        }
    }
}

}  // namespace smb
