// mortal_b200 — the training-buffer observation codec: float32 observations <-> fixed-size records (make_obs_record,
// csrc/mjx_obs.cuh), bit for bit.
//
// k_obs_pack reads an observation row by row, one warp per (sample, 32-row slice), lanes over the columns. A mask row must hold
// only +0.0 and 1.0: any other bit pattern (0.5, -0.0, a NaN, 2.0, a denormal) is never rounded into the mask, it sets the
// sample's status to 1 + the first such row. A value row is copied bit for bit. k_obs_unpack is k_encode_store's slice loop
// (csrc/mjx_kernels.cu enc_store_slices) over the records an index vector picks, materialised by enc_materialize.
#pragma once
#include "mjx_obs.cuh"

namespace mjx {

constexpr int OBS_PACK_WARPS = 8;
constexpr int OBS_PACK_SLICE = 32;
constexpr int OBS_PACK_MAX_SLICES = (OBS_ROWS_V4 + OBS_PACK_SLICE - 1) / OBS_PACK_SLICE;
constexpr u32 OBS_F32_ONE = 0x3f800000u;
constexpr int OBS_REC_KINDS = 8;  // (invisible, version 1..4)

MJX_HD constexpr int obs_record_kind(int ver, bool invisible) { return (invisible ? 4 : 0) + ver - 1; }

// per 32-row slice of a record: which of its rows are value rows (bit j = row lo + j) and the value slot of the first of them
// (value rows are in ascending row order, so the slots of a slice's value rows are consecutive)
struct ObsPackSlices {
    u32 vmask[OBS_PACK_MAX_SLICES];
    short slot0[OBS_PACK_MAX_SLICES];
};
MJX_HD constexpr ObsPackSlices make_pack_slices(const ObsRecord& R) {
    ObsPackSlices S{};
    for (int k = 0; k < R.n_val; k++) {
        const int s = R.val_row[k] / OBS_PACK_SLICE;
        if (S.vmask[s] == 0) S.slot0[s] = (short)k;
        S.vmask[s] |= 1u << (R.val_row[k] % OBS_PACK_SLICE);
    }
    return S;
}

// argument checks of mjx_obs_pack_dev / mjx_obs_unpack_dev and of the host build; nullptr = fine
inline const char* obs_pack_check(int ver, int invisible, long long n, const void* obs, long long pitch, const void* rec,
                                  const void* status) {
    if (ver < 1 || ver > 4 || (invisible != 0 && invisible != 1)) return "version must be 1..4 and invisible 0 or 1";
    if (n < 0 || n > 0x7fffffffLL) return "n must be within 0..2^31-1";
    if (n > 0 && (!obs || !rec || !status)) return "null array";
    if (pitch < (long long)make_obs_record(ver, invisible != 0).rows * OBS_COLS) return "sample pitch below rows * 34 floats";
    if ((reinterpret_cast<uintptr_t>(obs) & 3) || (reinterpret_cast<uintptr_t>(rec) & 7)) return "misaligned array";
    return nullptr;
}
inline const char* obs_unpack_check(int ver, int invisible, const void* rec, long long n_rec, const void* idx, long long n_idx,
                                    const void* out) {
    if (ver < 1 || ver > 4 || (invisible != 0 && invisible != 1)) return "version must be 1..4 and invisible 0 or 1";
    if (n_rec < 0 || n_idx < 0 || n_idx > 0x7fffffffLL / OBS_PACK_MAX_SLICES) return "bad counts";
    if (n_idx > 0 && (!idx || !out || (n_rec > 0 && !rec))) return "null array";
    if ((reinterpret_cast<uintptr_t>(rec) & 7) || (reinterpret_cast<uintptr_t>(out) & 15) || (reinterpret_cast<uintptr_t>(idx) & 7))
        return "misaligned array";
    return nullptr;
}

#ifdef MJX_HOST_EMUL
// one sample: its record written, returns 1 + the first mask row with a cell other than +0.0 / 1.0, or 0
inline int obs_pack_sample(const ObsRecord& R, const ObsPackSlices& P, const float* x, unsigned char* rec) {
    u64* masks = reinterpret_cast<u64*>(rec);
    u32* vals = reinterpret_cast<u32*>(rec + R.rows * 8);
    int bad = 0;
    for (int r = 0; r < R.rows; r++) {
        u32 cell[OBS_COLS];
        memcpy(cell, x + (size_t)r * OBS_COLS, sizeof cell);
        const int s = r / OBS_PACK_SLICE, j = r % OBS_PACK_SLICE;
        if ((P.vmask[s] >> j) & 1) {
            memcpy(vals + (P.slot0[s] + __builtin_popcount(P.vmask[s] & ((1u << j) - 1))) * OBS_COLS, cell, sizeof cell);
            masks[r] = 0;
            continue;
        }
        u64 m = 0;
        for (int c = 0; c < OBS_COLS; c++) {
            if (cell[c] == OBS_F32_ONE) m |= 1ull << c;
            else if (cell[c] != 0u && bad == 0) bad = r + 1;
        }
        masks[r] = m;
    }
    return bad;
}
#else
// rows [lo, lo + 32) of one sample by one warp: returns the first mask row with a cell other than +0.0 / 1.0, or INT_MAX
MJX_D int obs_pack_slice(const ObsRecord& R, const ObsPackSlices& P, const float* __restrict__ x, unsigned char* __restrict__ rec,
                         int lo, int lane) {
    const int nr = min(OBS_PACK_SLICE, R.rows - lo), s = lo / OBS_PACK_SLICE;
    const u32 vmask = P.vmask[s];
    const int slot0 = P.slot0[s];
    const u32* xs = reinterpret_cast<const u32*>(x) + (size_t)lo * OBS_COLS;
    u32* vals = reinterpret_cast<u32*>(rec + R.rows * 8);
    u64 mine = 0;  // lane j: the mask of row lo + j
    int bad = INT_MAX;
    for (int j0 = 0; j0 < nr; j0 += 8) {
        u32 a[8], b[8];  // eight rows in flight: lane = column, lanes 0-1 also columns 32-33
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const u32* src = xs + (j0 + u) * OBS_COLS;
            a[u] = j0 + u < nr ? __ldcs(src + lane) : 0u;
            b[u] = (j0 + u < nr && lane < 2) ? __ldcs(src + 32 + lane) : 0u;
        }
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int j = j0 + u;
            if (j >= nr) break;
            if ((vmask >> j) & 1) {
                u32* dst = vals + (slot0 + __popc(vmask & ((1u << j) - 1))) * OBS_COLS;
                dst[lane] = a[u];
                if (lane < 2) dst[32 + lane] = b[u];
                continue;
            }
            const u32 ones = __ballot_sync(0xffffffffu, a[u] == OBS_F32_ONE);
            const u32 ones_hi = __ballot_sync(0xffffffffu, lane < 2 && b[u] == OBS_F32_ONE);
            const bool ok = (a[u] == 0u || a[u] == OBS_F32_ONE) && (b[u] == 0u || b[u] == OBS_F32_ONE);
            if (!__all_sync(0xffffffffu, ok)) bad = min(bad, lo + j);
            if (lane == j) mine = (u64)ones | ((u64)(ones_hi & 3u) << 32);
        }
    }
    if (lane < nr) reinterpret_cast<u64*>(rec)[lo + lane] = mine;
    return bad;
}
#endif

}  // namespace mjx
