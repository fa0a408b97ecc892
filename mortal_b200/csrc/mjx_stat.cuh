// mortal_b200 — per-player log statistics: mortal_b200/stat.py Stat.from_game (itself stat.rs:263-442 Stat::from_game) over the
// event arrays the mjai decoder writes (csrc/mjx_mjai.cuh, mjx_mjai_fill_deltas_dev): the event words, the start_kyoku payloads
// (scores) and the per-event deltas. All arithmetic is 64-bit, as Python's integers are for any score a log can hold.
//
// Device: k_stat_logs (mjx_kernels.cu) runs one log per warp; lane s < 4 plays seat s. The warp loads the words 32 at a time and
// shuffles each to the seat lanes, so the seats walk the log in step and every branch on the event type is warp-uniform.
// -DMJX_HOST_EMUL builds the same walk for one host lane that plays all four seats (tests/host_emul/emul_stat.cc).
#pragma once
#include "../../include/mjx.h"
#include "mjx_types.cuh"
#include "mjx_mjai.cuh"

namespace mjx {

constexpr int STAT_WARPS = 4;
#ifdef MJX_HOST_EMUL
constexpr int STAT_SEATS_PER_LANE = 4;  // the one lane plays seats 0..3
#else
constexpr int STAT_SEATS_PER_LANE = 1;  // lane s plays seat s (lanes >= 4: none)
#endif

struct StatView {
    const u64* hdr;
    const i32 *ev_off, *ev_cnt;
    long long n_hdr;  // words (and deltas entries)
    const u64* kyoku;
    const i32* ky_off;
    long long n_kyoku;  // payloads
    const i32* deltas;  // [n_hdr, 4]
    const u8* has_deltas;
    const u8* seats;
    int n_logs;
    i64* out;  // [n_logs, MJX_STAT_N]
    i32* status;
};

// Stat.from_game's loop state for one seat
struct StatSeat {
    i64 scores[4];
    int oya, jun, calls;
    bool declared, accepted, others_declared;
};

// one event of Stat.from_game for seat `me`: w = the event word, sc = the start_kyoku scores, d = the hora / ryukyoku deltas
MJX_D void stat_event(StatSeat& s, i64* c, int me, u64 w, const i64* sc, const i32* d) {
    const int ty = (int)(w & 0xFF), actor = (int)(w >> 8) & 3, target = (int)(w >> 10) & 3;
    switch (ty) {
        case MJT_START_KYOKU:
            c[MJX_S_round]++;
            for (int k = 0; k < 4; k++) s.scores[k] = sc[k];
            s.declared = s.accepted = s.others_declared = false;
            s.oya = (int)(w >> 48) & 0xFF;
            s.jun = s.calls = 0;
            c[MJX_S_oya] += s.oya == me;
            break;
        case MJT_DAHAI: s.jun += actor == me; break;
        case MJT_CHI:
        case MJT_PON:
        case MJT_DAIMINKAN: s.calls += actor == me; break;
        case MJT_REACH:
            if (actor == me) {
                s.declared = true;
                c[MJX_S_riichi]++;
                c[MJX_S_riichi_jun] += s.jun;
                c[MJX_S_riichi_as_oya] += s.oya == me;
                c[MJX_S_chasing_riichi] += s.others_declared;
            } else if (s.declared) {
                c[MJX_S_riichi_got_chased]++;
            } else {
                s.others_declared = true;
            }
            break;
        case MJT_REACH_ACCEPTED:
            s.scores[actor] -= 1000;
            s.accepted = s.accepted || actor == me;
            break;
        case MJT_HORA:
            for (int k = 0; k < 4; k++) s.scores[k] += d[k];
            if (actor == me) {
                const i64 point = (i64)d[me] - 1000 * (i64)s.accepted;  // the own stick comes back with the win
                c[MJX_S_agari]++;
                c[MJX_S_agari_jun] += s.jun;
                if (s.oya == me) {
                    c[MJX_S_agari_as_oya]++;
                    c[MJX_S_agari_point_oya] += point;
                } else {
                    c[MJX_S_agari_point_ko] += point;
                }
                if (s.accepted) {
                    c[MJX_S_riichi_agari]++; c[MJX_S_riichi_agari_jun] += s.jun; c[MJX_S_riichi_agari_point] += point;
                    c[MJX_S_riichi_point] += point;
                } else if (s.calls > 0) {
                    c[MJX_S_fuuro_agari]++; c[MJX_S_fuuro_agari_jun] += s.jun; c[MJX_S_fuuro_agari_point] += point;
                    c[MJX_S_fuuro_point] += point;
                } else {
                    c[MJX_S_dama_agari]++; c[MJX_S_dama_agari_jun] += s.jun; c[MJX_S_dama_agari_point] += point;
                }
                c[MJX_S_yakuman] += point >= (s.oya == me ? 48000 : 32000);  // point.rs Point::yakuman(is_oya, 1).ron
            } else if (target == me) {
                const i64 point = d[me];
                c[MJX_S_houjuu]++;
                c[MJX_S_houjuu_jun] += s.jun;
                if (s.oya == actor) {
                    c[MJX_S_houjuu_to_oya]++;
                    c[MJX_S_houjuu_point_to_oya] += point;
                } else {
                    c[MJX_S_houjuu_point_to_ko] += point;
                }
                if (s.declared) {
                    c[MJX_S_riichi_houjuu]++; c[MJX_S_riichi_point] += point;
                } else if (s.calls > 0) {
                    c[MJX_S_fuuro_houjuu]++; c[MJX_S_fuuro_point] += point;
                }
            }
            break;
        case MJT_RYUKYOKU: {
            for (int k = 0; k < 4; k++) s.scores[k] += d[k];
            const i64 point = d[me];
            c[MJX_S_ryukyoku]++;
            c[MJX_S_ryukyoku_point] += point;
            if (s.accepted) {
                c[MJX_S_riichi_ryukyoku]++;
                c[MJX_S_riichi_point] += point - 1000;
            } else if (s.calls > 0) {
                c[MJX_S_fuuro_point] += point;
            }
            c[MJX_S_nagashi_mangan] += point >= 8000;
            break;
        }
        case MJT_END_KYOKU:
            if (s.calls > 0) {
                c[MJX_S_fuuro]++;
                c[MJX_S_fuuro_num] += s.calls;
            }
            break;
        default: break;
    }
}

// the end of Stat.from_game: rankings.rs:8-22 (stable by seat on ties), the sticks left on the table to the leader
MJX_D void stat_finish(StatSeat& s, i64* c, int me) {
    int order[4] = {0, 1, 2, 3};
    for (int a = 1; a < 4; a++)  // insertion sort by descending score: stable
        for (int b = a; b > 0 && s.scores[order[b - 1]] < s.scores[order[b]]; b--) {
            const int t = order[b]; order[b] = order[b - 1]; order[b - 1] = t;
        }
    const i64 total = s.scores[0] + s.scores[1] + s.scores[2] + s.scores[3];
    if (total < 100000) s.scores[order[0]] += 100000 - total;
    c[MJX_S_point] += s.scores[me] - 25000;
    c[MJX_S_tobi] += s.scores[me] < 0;
    for (int r = 0; r < 4; r++) c[MJX_S_rank_1 + r] += order[r] == me;
}

// Stat.from_game of every selected seat of log i into c[seat][...] (zeroed by the caller) -> mjx_stat_status. The status is
// warp-uniform: every lane reads the same words, payloads and presence bytes.
MJX_DM int stat_log(const StatView& V, int i, int lane, i64 (*c)[MJX_STAT_N]) {
    const long long off = V.ev_off[i], cnt = V.ev_cnt[i];
    if (off < 0 || cnt < 0 || off + cnt > V.n_hdr) return MJX_STAT_CAPACITY;
    if (cnt == 0 || (V.hdr[off] & 0xFF) != MJT_START_GAME) return MJX_STAT_NOT_START_GAME;
    const int mask = V.seats[i] & 15;
    if (!mask) return MJX_STAT_OK;
    StatSeat S[STAT_SEATS_PER_LANE];
    bool mine[STAT_SEATS_PER_LANE];
    for (int k = 0; k < STAT_SEATS_PER_LANE; k++) {
        const int me = lane * STAT_SEATS_PER_LANE + k;
        mine[k] = me < 4 && ((mask >> me) & 1);
        S[k] = StatSeat{{0, 0, 0, 0}, 0, 0, 0, false, false, false};
        if (mine[k]) c[me][MJX_S_game] = 1;
    }
    long long ky = V.ky_off[i];  // the next start_kyoku payload
    i64 sc[4] = {0, 0, 0, 0};
    i32 d[4] = {0, 0, 0, 0};
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
                if (ky < 0 || ky >= V.n_kyoku) return MJX_STAT_CAPACITY;
                const u64* pay = V.kyoku + ky * MJAI_KYOKU_WORDS;
                const u64 p0 = pay[0], p1 = pay[1];
                sc[0] = (i32)(u32)p0; sc[1] = (i32)(u32)(p0 >> 32); sc[2] = (i32)(u32)p1; sc[3] = (i32)(u32)(p1 >> 32);
                ky++;
            } else if (ty == MJT_HORA || ty == MJT_RYUKYOKU) {
                if (!V.has_deltas[e]) return MJX_STAT_NO_DELTAS;
                for (int k = 0; k < 4; k++) d[k] = V.deltas[4 * e + k];
            }
            for (int k = 0; k < STAT_SEATS_PER_LANE; k++)
                if (mine[k]) stat_event(S[k], c[lane * STAT_SEATS_PER_LANE + k], lane * STAT_SEATS_PER_LANE + k, w, sc, d);
        }
    }
    for (int k = 0; k < STAT_SEATS_PER_LANE; k++)
        if (mine[k]) stat_finish(S[k], c[lane * STAT_SEATS_PER_LANE + k], lane * STAT_SEATS_PER_LANE + k);
    return MJX_STAT_OK;
}

}  // namespace mjx
