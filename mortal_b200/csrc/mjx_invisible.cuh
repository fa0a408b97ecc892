// mortal_b200 — the invisible ("oracle") observation: arena/board.rs:680-782 encode_oracle_obs, consts.rs:30-38.
//
// What an `is_oracle` engine is handed beside the ordinary observation (agent/mortal.rs:253-255, dataset/invisible.rs): the three
// other seats' hands / akas / shanten / waits / furiten and the hidden tiles of the wall in drawing order. It is read straight
// from the full-information table record: one warp per decision row, coalesced zero fill, then the few hundred set cells.
#pragma once
#include "mjx_step.cuh"

namespace mjx {

MJX_HD constexpr int oracle_obs_rows(int version) { return version == 1 ? 211 : 217; }
// the rows that hold a value other than 0 / 1: versions 2-4 write shanten / 6 into row 7 of each opponent's 8-row shanten block
// (an opponent takes 4 + 3 + 8 + 1 + 1 = 17 rows); version 1 has none
MJX_HD constexpr int oracle_obs_value_rows(int version) { return version == 1 ? 0 : 3; }
MJX_HD constexpr int oracle_obs_value_row(int k) { return 17 * k + 4 + 3 + 7; }

#ifdef MJX_HOST_EMUL
#define INV_FOR(i, n) for (int i = 0; i < (n); i++)
#else
#define INV_FOR(i, n) for (int i = lane; i < (n); i += 32)
#endif

// all_yama: dataset/invisible.rs:150-231 Invisible::encode lists EVERY tile left in the live wall (`yama[yama_idx..]`), while
// board.rs:748-758 lists only the next `tiles_left` of them (the two differ by the rinshan draws made so far)
MJX_DN void encode_invisible(const TableState* S, int perspective, int version, float* out, int lane, bool all_yama = false) {
    const int rows = oracle_obs_rows(version);
    INV_FOR(i, rows * 34) out[i] = 0.f;
    MJX_SYNCWARP();
    int idx = 0;
    for (int k = 1; k <= 3; k++) {  // .cycle().skip(perspective + 1).take(3)
        const SeatPrivate& P = S->priv[(perspective + k) & 3];
        INV_FOR(t, 34) {
            const int cnt = P.tehai[t];
            for (int c = 0; c < cnt && c < 4; c++) out[(idx + c) * 34 + t] = 1.f;  // assign_rows
        }
        idx += 4;
        INV_FOR(col, 34) for (int i = 0; i < 3; i++) if ((P.akas_in_hand >> i) & 1) out[(idx + i) * 34 + col] = 1.f;
        idx += 3;
        const int n = P.shanten;
        if (version == 1) {
            INV_FOR(col, 34) for (int i = 0; i < n && i < 6; i++) out[(idx + i) * 34 + col] = 1.f;  // fill_rows
            idx += 6;
        } else {
            INV_FOR(col, 34) { out[(idx + n) * 34 + col] = 1.f; out[(idx + 7) * 34 + col] = (float)n / 6.f; }
            idx += 8;
        }
        INV_FOR(t, 34) if ((P.waits >> t) & 1) out[idx * 34 + t] = 1.f;
        idx += 1;
        if (P.flags & PF_AT_FURITEN) INV_FOR(col, 34) out[idx * 34 + col] = 1.f;
        idx += 1;
    }
    // a tile takes two rows: one-hot of its kind, then an all-ones row when it is an aka; unknown tiles (a log without the
    // seed) leave their rows zero
    auto encode_tile = [&](int r, int tile) {
        if (tile >= T_UNK) return;
        out[r * 34 + deaka(tile)] = 1.f;
        if (is_aka(tile)) for (int col = 0; col < 34; col++) out[(r + 1) * 34 + col] = 1.f;
    };
    const int tiles_left = S->tiles_left, yama_len = tiles_left + S->n_rinshan;  // yama = wall[66 .. 66 + yama_len), drawn from the back
    const int n_yama = all_yama ? yama_len : tiles_left;
    INV_FOR(q, n_yama) if (q < 69) encode_tile(idx + 2 * q, S->wall[66 + yama_len - 1 - q]);
    idx += 69 * 2;
    const int rin_len = 4 - S->n_rinshan;  // rinshan = wall[52 .. 52 + rin_len), drawn from the back
    INV_FOR(q, rin_len) encode_tile(idx + 2 * q, S->wall[52 + rin_len - 1 - q]);
    idx += 4 * 2;
    INV_FOR(q, 5) encode_tile(idx + 2 * q, S->wall[60 - q]);  // dora_indicators_full reversed: first indicator first
    idx += 5 * 2;
    INV_FOR(q, 5) encode_tile(idx + 2 * q, S->wall[61 + q]);  // ura indicators in revealing order
    MJX_SYNCWARP();
}

}  // namespace mjx
