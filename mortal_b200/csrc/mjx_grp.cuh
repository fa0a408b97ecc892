// mortal_b200 — the GRP targets of a game log: mortal_b200/dataset.py Grp.load_events (itself dataset/grp.rs:90-164) over the event
// arrays the mjai decoder writes (csrc/mjx_mjai.cuh, mjx_mjai_fill_deltas_dev): the event words, the start_kyoku payloads (scores)
// and the per-event deltas.
//
// The reference walks the log backwards: the last start_kyoku's scores plus every hora's and ryukyoku's deltas after it, minus
// 1000 for every reach_accepted after it, are the final scores. The same sum is made here in one forward walk that restarts at
// every start_kyoku, in 64-bit arithmetic, as Python's integers are for any score a log can hold.
//
// Device: k_grp_logs (mjx_kernels.cu) runs one log per warp. The warp loads the words 32 at a time (coalesced) and shuffles each to
// every lane, so the walk and every branch on the event type is warp-uniform; lane 0 writes. -DMJX_HOST_EMUL builds the same walk
// for one host lane (tests/host_emul/emul_grp.cc).
#pragma once
#include "../../include/mjx.h"
#include "mjx_types.cuh"
#include "mjx_mjai.cuh"

namespace mjx {

constexpr int GRP_WARPS = 4;
constexpr int GRP_ROW = 7;  // {grand_kyoku, honba, kyotaku, scores[4]}

struct GrpView {
    const u64* hdr;
    const i32 *ev_off, *ev_cnt;
    long long n_hdr;  // words (and deltas entries)
    const u64* kyoku;
    const i32* ky_off;
    long long n_kyoku;  // payloads (and feature rows)
    const i32* deltas;  // [n_hdr, 4]
    const u8* has_deltas;
    int n_logs;
    i32* feat;   // [n_kyoku, GRP_ROW]
    u8* rank;    // [n_logs, 4]
    i64* final;  // [n_logs, 4]
    i32* status;
};

// grp.rs:153-160: E1..E4 = 0..3, S1..S4 = 4..7, and every later round wind (W and N alike) 7 + kyoku. The word's c0 is
// (bakaze - E) * 4 + kyoku - 1 (dataset_codec.encode_events), so N rounds map onto the W numbers.
MJX_D int grp_grand_kyoku(int c0) { return c0 < 8 ? c0 : 8 + (c0 & 3); }

// Grp.load_events of log i: the feature rows at its payload indices (written as the walk reaches them, so a log that ends with
// a non-zero status may have some rows written), and into rank / fin the final ranking (rankings.rs:8-22, stable by seat) and
// the final scores with the sticks left on the table given to the leader -> mjx_grp_status. The status is warp-uniform.
MJX_DM int grp_log(const GrpView& V, int i, int lane, u8* rank, i64* fin) {
    const long long off = V.ev_off[i], cnt = V.ev_cnt[i];
    if (off < 0 || cnt < 0 || off + cnt > V.n_hdr) return MJX_GRP_CAPACITY;
    long long ky = V.ky_off[i];  // the next start_kyoku payload
    bool seen = false, missing = false;
    i64 sc[4] = {0, 0, 0, 0}, acc[4] = {0, 0, 0, 0};  // the last start_kyoku's scores; what happened after it
    for (long long base = 0; base < cnt; base += 32) {
        const int n = cnt - base < 32 ? (int)(cnt - base) : 32;
#ifndef MJX_HOST_EMUL
        const u64 wl = lane < n ? V.hdr[off + base + lane] : 0;
#endif
        for (int j = 0; j < n; j++) {
            const long long e = off + base + j;
#ifdef MJX_HOST_EMUL
            const u64 w = V.hdr[e];
#else
            const u64 w = __shfl_sync(~0u, wl, j);
#endif
            const int ty = (int)(w & 0xFF);
            if (ty == MJT_START_KYOKU) {
                if (ky < 0 || ky >= V.n_kyoku) return MJX_GRP_CAPACITY;
                const u64* pay = V.kyoku + ky * MJAI_KYOKU_WORDS;
                const u64 p0 = pay[0], p1 = pay[1];
                sc[0] = (i32)(u32)p0; sc[1] = (i32)(u32)(p0 >> 32); sc[2] = (i32)(u32)p1; sc[3] = (i32)(u32)(p1 >> 32);
                if (lane == 0) {
                    i32* row = V.feat + ky * GRP_ROW;
                    row[0] = grp_grand_kyoku((int)(w >> 24) & 0xFF);
                    row[1] = (int)(w >> 32) & 0xFF;
                    row[2] = (int)(w >> 40) & 0xFF;
                    for (int k = 0; k < 4; k++) row[3 + k] = (i32)sc[k];
                }
                for (int k = 0; k < 4; k++) acc[k] = 0;
                seen = true;
                missing = false;
                ky++;
            } else if (ty == MJT_HORA || ty == MJT_RYUKYOKU) {
                if (!V.has_deltas[e]) missing = true;  // an error only when no start_kyoku follows (grp.rs:101-106)
                else
                    for (int k = 0; k < 4; k++) acc[k] += V.deltas[4 * e + k];
            } else if (ty == MJT_REACH_ACCEPTED) {
                acc[(w >> 8) & 3] -= 1000;
            }
        }
    }
    if (missing) return MJX_GRP_NO_DELTAS;
    if (!seen) return MJX_GRP_NO_KYOKU;
    for (int k = 0; k < 4; k++) fin[k] = sc[k] + acc[k];
    int order[4] = {0, 1, 2, 3};
    for (int a = 1; a < 4; a++)  // insertion sort by descending score: stable
        for (int b = a; b > 0 && fin[order[b - 1]] < fin[order[b]]; b--) {
            const int t = order[b]; order[b] = order[b - 1]; order[b - 1] = t;
        }
    const i64 total = fin[0] + fin[1] + fin[2] + fin[3];
    if (total < 100000) fin[order[0]] += 100000 - total;  // grp.rs:127-131
    for (int r = 0; r < 4; r++) rank[order[r]] = (u8)r;
    return MJX_GRP_OK;
}

}  // namespace mjx
