// mortal_b200 — log validation: libriichi bin/validate_logs.rs:62-242 process_path.
//
// One warp validates one whole log: a full-information table record (all four seats, TableState.viewer1 = 0) is initialised in
// shared memory and never leaves it. For every event the warp runs, in the reference's order,
//   1. the checks process_path makes for that event type, read from the record (cans, discard / kan candidates, agari points
//      with the logged ura markers);
//   2. the errors PlayerState::update_with_keep_cans(ev, true) would raise for seats 0..3 (exhausted yama, unknown or fifth
//      tile witnessed, discard / consume from void, dora-indicator overflow), computed per seat from the record — a seat has
//      witnessed public_seen[t] + its own tehai[t] copies of t;
//   3. a capacity guard: an event the record cannot hold ends the log as UNSUPPORTED instead of being applied (so does, before
//      step 1, a field no encoder produces);
//   4. apply_event with keep-cans-on-announce semantics.
// The first failure ends the log; the verdict is 16 bytes. Every branch condition reads the record or the event word, so the
// warp stays converged (the candidate masks are warp ballots).
#pragma once
#include "../../include/mjx.h"
#include "mjx_replay.cuh"

namespace mjx {

struct ValidateView {
    const u64* hdr;       // event words of all logs, concatenated
    const i32* ev_off;    // [n_logs]
    const i32* ev_cnt;    // [n_logs]
    const u64* kyoku;     // start_kyoku payloads, REPLAY_KYOKU_WORDS each
    const i32* ky_off;    // [n_logs] first payload of the log (in payloads)
    const u64* hora;      // hora side entries, MJX_HORA_WORDS each
    const i32* hora_off;  // [n_logs] first entry of the log (in entries)
    long long n_kyoku, n_hora;  // payloads / entries available (bounds of the cursors)
    int n_logs;
    mjx_verdict* out;
};

struct VResult { i32 status, reason, seat; };

MJX_D VResult v_ok() { return VResult{MJX_V_OK, MJX_R_NONE, -1}; }
MJX_D VResult v_check(int reason, int actor) { return VResult{MJX_V_CHECK, reason, actor}; }
MJX_D VResult v_unsupported() { return VResult{MJX_V_UNSUPPORTED, MJX_R_CAPACITY, -1}; }

MJX_D int pay_tile(const u64* pay, int i) { return (int)((pay[2 + i / 8] >> (8 * (i % 8))) & 0xFF); }
MJX_D int n_melds(const SeatPrivate& P) { return P.n_chis + P.n_pons + P.n_minkans + P.n_ankans; }
MJX_D int hand_count(const SeatPrivate& P) {
    int n = 0;
    for (int t = 0; t < 34; t++) n += P.tehai[t];
    return n;
}
// copies of tile d (deaka'd) seat s has witnessed (update.rs:695-727 tiles_seen)
MJX_D int seen(const TableState* S, int s, int d) { return S->public_seen[d] + S->priv[s].tehai[d]; }

// Fields the encoder never produces (a type outside the log words, a tile byte past `?`, a start_kyoku without payload or with an
// out-of-range round / dealer, `?` where only the haipai and dora markers may hold it): the log ends as UNSUPPORTED before any
// check reads them. Uniform.
MJX_D bool v_bad_fields(u64 w, const u64* pay) {
    const int ty = lw_type(w), pai = lw_pai(w);
    switch (ty) {
        case LOG_START_KYOKU:
            if (pay == nullptr || pai > T_UNK || lw_c(w, 0) >= 16 || lw_c(w, 3) >= 4) return true;
            for (int i = 0; i < 52; i++) if (pay_tile(pay, i) > T_UNK) return true;
            return false;
        case LOG_TSUMO: case LOG_DAHAI: case LOG_KAKAN: return pai >= T_UNK;
        case LOG_CHI: case LOG_PON: case LOG_DAIMINKAN: case LOG_ANKAN: {
            const int nc = ty == LOG_DAIMINKAN ? 3 : ty == LOG_ANKAN ? 4 : 2;
            if (ty != LOG_ANKAN && pai >= T_UNK) return true;
            for (int k = 0; k < nc; k++) if (lw_c(w, k) >= T_UNK) return true;
            return false;
        }
        case LOG_DORA: return pai > T_UNK;
        case LOG_REACH: case LOG_REACH_ACCEPTED: case LOG_HORA: case LOG_RYUKYOKU: case LOG_END_KYOKU: case LOG_START_GAME:
        case LOG_END_GAME:
            return false;
        default: return true;
    }
}

// Step 3: an event that passed the checks and the update but that the record has no room for. Uniform.
MJX_D bool v_no_room(const TableState* S, u64 w) {
    const int ty = lw_type(w), a = lw_actor(w), pai = lw_pai(w);
    const SeatPrivate& P = S->priv[a];
    switch (ty) {
        case LOG_TSUMO: return hand_count(P) != 3 * P.tehai_len_div3 + 1;  // the shanten tables take at most 14 tiles
        case LOG_DAHAI: return S->pub[a].kawa_len >= KAWA_CAP;
        case LOG_CHI: case LOG_PON: case LOG_DAIMINKAN:
            if (n_melds(P) >= 4 || S->pub[a].n_fuuro >= 4) return true;
            if (ty == LOG_CHI)  // ev_chi's kuikae rule indexes the neighbours of a suited run
                for (int k = 0; k < 3; k++) if (deaka(k < 2 ? lw_c(w, k) : pai) >= 27) return true;
            if (ty != LOG_CHI)
                for (int i = (lw_target(w) + 1) & 3; i != a; i = (i + 1) & 3) if (S->pub[i].kawa_len >= KAWA_CAP) return true;
            return false;
        case LOG_KAKAN:
            for (int i = 0; i < P.n_pons; i++) if (P.pons[i] == deaka(pai)) return P.n_minkans >= 4;
            return true;
        case LOG_ANKAN: return n_melds(P) >= 4 || S->pub[a].n_ankan >= 4;
        default: return false;
    }
}

// Step 2 for one seat: the first error update_with_keep_cans raises for seat s, in the order update.rs performs its witness /
// move_tile calls, or 0. Uniform (every lane evaluates every seat).
MJX_D int v_update_error(const TableState* S, int s, u64 w, const u64* pay) {
    const int ty = lw_type(w), a = lw_actor(w), pai = lw_pai(w);
    const SeatPrivate& P = S->priv[s];
    switch (ty) {
        case LOG_START_KYOKU: {  // update.rs:207-212: the dora marker, then the own 13 tiles
            if (pai == T_UNK) return MJX_R_UNKNOWN_TILE;
            const int dd = deaka(pai);
            for (int i = 0; i < 13; i++) {
                const int t = pay_tile(pay, 13 * s + i);
                if (t == T_UNK) return MJX_R_UNKNOWN_TILE;
                const int d = deaka(t);
                int n = dd == d;
                for (int j = 0; j < i; j++) n += deaka(pay_tile(pay, 13 * s + j)) == d;
                if (n >= 4) return MJX_R_FIFTH_TILE;
            }
            return 0;
        }
        case LOG_TSUMO:
            if (S->tiles_left == 0) return MJX_R_EXHAUSTED_YAMA;
            return s == a && seen(S, s, deaka(pai)) >= 4 ? MJX_R_FIFTH_TILE : 0;
        case LOG_DAHAI:
            if (s == a) return P.tehai[deaka(pai)] == 0 ? MJX_R_DISCARD_FROM_VOID : 0;
            return seen(S, s, deaka(pai)) >= 4 ? MJX_R_FIFTH_TILE : 0;
        case LOG_CHI: case LOG_PON: case LOG_DAIMINKAN: case LOG_ANKAN: {
            const int nc = ty == LOG_DAIMINKAN ? 3 : ty == LOG_ANKAN ? 4 : 2;
            for (int k = 0; k < nc; k++) {
                const int d = deaka(lw_c(w, k));
                int before = 0;
                for (int j = 0; j < k; j++) before += deaka(lw_c(w, j)) == d;
                if (s == a) { if (P.tehai[d] - before <= 0) return MJX_R_CONSUME_FROM_VOID; }
                else if (seen(S, s, d) + before >= 4) return MJX_R_FIFTH_TILE;
            }
            return 0;
        }
        case LOG_KAKAN:
            if (s == a) return P.tehai[deaka(pai)] == 0 ? MJX_R_CONSUME_FROM_VOID : 0;
            return seen(S, s, deaka(pai)) >= 4 ? MJX_R_FIFTH_TILE : 0;
        case LOG_DORA:
            if (S->n_dora >= 5) return MJX_R_DORA_OVERFLOW;
            if (pai == T_UNK) return MJX_R_UNKNOWN_TILE;
            return seen(S, s, deaka(pai)) >= 4 ? MJX_R_FIFTH_TILE : 0;
        default: return 0;
    }
}

// Step 1: process_path's checks (validate_logs.rs:86-232). `hw` = the hora side entry (hora only).
MJX_DN VResult v_check_event(const Ctx& c, u64 w, const u64* hw) {
    const TableState* S = c.S;
    const int ty = lw_type(w), a = lw_actor(w), pai = lw_pai(w);
    const SeatPrivate& P = S->priv[a];
    const u16 cans = P.cans;
    switch (ty) {
        case LOG_DAHAI: {
            if (!(cans & CAN_DISCARD)) return v_check(MJX_R_CAN_DISCARD, a);
            // agent_helper.rs:40-46 expects a last self tsumo under riichi; the record has none only for an impossible state
            if (((S->riichi_accepted >> a) & 1) && P.last_self_tsumo >= T_UNK) return v_unsupported();
            if (!((discard_candidates(c, a) >> pai) & 1)) return v_check(MJX_R_DISCARD_CANDIDATES, a);
            return v_ok();
        }
        case LOG_CHI: {
            if (((lw_target(w) + 1) & 3) != a) return v_check(MJX_R_CHI_NON_KAMICHA, a);
            const int x = deaka(lw_c(w, 0)), y = deaka(lw_c(w, 1)), t = deaka(pai);  // chi_type.rs:12-25
            if (t < min(x, y)) return (cans & CAN_CHI_LOW) ? v_ok() : v_check(MJX_R_CAN_CHI_LOW, a);
            if (t < max(x, y)) return (cans & CAN_CHI_MID) ? v_ok() : v_check(MJX_R_CAN_CHI_MID, a);
            return (cans & CAN_CHI_HIGH) ? v_ok() : v_check(MJX_R_CAN_CHI_HIGH, a);
        }
        case LOG_PON: return (cans & CAN_PON) ? v_ok() : v_check(MJX_R_CAN_PON, a);
        case LOG_DAIMINKAN: return (cans & CAN_DAIMINKAN) ? v_ok() : v_check(MJX_R_CAN_DAIMINKAN, a);
        case LOG_ANKAN:
            if (!(cans & CAN_ANKAN)) return v_check(MJX_R_CAN_ANKAN, a);
            return ((P.ankan_cand >> deaka(lw_c(w, 0))) & 1) ? v_ok() : v_check(MJX_R_ANKAN_CANDIDATES, a);
        case LOG_KAKAN:
            if (!(cans & CAN_KAKAN)) return v_check(MJX_R_CAN_KAKAN, a);
            return ((P.kakan_cand >> deaka(pai)) & 1) ? v_ok() : v_check(MJX_R_KAKAN_CANDIDATES, a);
        case LOG_REACH: return (cans & CAN_RIICHI) ? v_ok() : v_check(MJX_R_CAN_RIICHI, a);
        case LOG_HORA: {
            const bool is_ron = a != lw_target(w);
            if (is_ron && !(cans & CAN_RON_AGARI)) return v_check(MJX_R_CAN_RON_AGARI, a);
            if (!is_ron && !(cans & CAN_TSUMO_AGARI)) return v_check(MJX_R_CAN_TSUMO_AGARI, a);
            // the reference's "rough test" (TODO: fix bug for double chankan ron), reproduced as it is
            const u64 h0 = hw[0], h1 = hw[1];
            if (!((h0 >> 33) & 1)) return v_check(MJX_R_MISSING_URA, a);
            if (!((h0 >> 32) & 1)) return v_check(MJX_R_MISSING_DELTAS, a);
            const int n_ura = (int)((h0 >> 36) & 0xF);
            if (n_ura > 5) return v_unsupported();
            u8 ura[5];
            for (int k = 0; k < 5; k++) {
                ura[k] = (u8)((h1 >> (8 * k)) & 0xFF);
                if (k < n_ura && ura[k] >= T_UNK) return v_unsupported();
            }
            bool ok;
            const Point p = agari_points_ura(c, a, is_ron, ura, n_ura, &ok);
            if (!ok) return v_check(MJX_R_AGARI_POINTS, a);
            const i32 delta = (i32)(u32)h0;
            const i32 need = is_ron ? p.ron : (a == S->oya ? p.tsumo_oya : p.tsumo_ko);
            return delta >= need ? v_ok() : v_check(MJX_R_DELTAS_BELOW_POINTS, a);
        }
        default: return v_ok();
    }
}

// PlayerState::new (player_state.rs): nothing dealt yet, the yama empty
MJX_D void v_init_record(Ctx& c) {
    TableState* S = c.S;
    MJX_L0(S->last_kawa_tile = T_NONE; S->riichi_to_be_accepted = -1; S->four_wind_tile = -1; S->gflags = GF_ALIVE;
           for (int s = 0; s < 4; s++) { S->priv[s].last_self_tsumo = T_NONE; S->paos[s] = -1; });
    recompute_dora_factor(c);
}

// Validate log `i` into V.out[i]. The record behind c.S must be zeroed.
MJX_DN void validate_log(Ctx& c, const ValidateView& V, int i) {
    TableState* S = c.S;
    v_init_record(c);
    const int n = V.ev_cnt[i];
    const u64* ev = V.hdr + V.ev_off[i];
    long long ky = V.ky_off[i], ho = V.hora_off[i];
    VResult r = v_ok();
    int line = 0;
#ifndef MJX_HOST_EMUL
    u64 chunk = 0;
#endif
    for (int idx = 0; idx < n; idx++) {
#ifdef MJX_HOST_EMUL
        const u64 w = ev[idx];
#else
        if ((idx & 31) == 0) chunk = idx + c.lane < n ? ev[idx + c.lane] : 0;  // 32 words per coalesced load
        const u64 w = __shfl_sync(0xFFFFFFFFu, chunk, idx & 31);
#endif
        const int ty = lw_type(w);
        const u64* pay = nullptr;
        const u64* hw = nullptr;
        if (ty == LOG_START_KYOKU && ky >= 0 && ky < V.n_kyoku) pay = V.kyoku + (size_t)ky * REPLAY_KYOKU_WORDS;
        if (ty == LOG_HORA) {
            if (ho < 0 || ho >= V.n_hora) { r = v_unsupported(); line = idx + 1; break; }
            hw = V.hora + (size_t)ho * MJX_HORA_WORDS;
        }
        if (v_bad_fields(w, pay)) { r = v_unsupported(); line = idx + 1; break; }
        r = v_check_event(c, w, hw);
        if (r.status != MJX_V_OK) { line = idx + 1; break; }
        for (int s = 0; s < 4; s++) {
            const int e = v_update_error(S, s, w, pay);
            if (e) { r = VResult{MJX_V_UPDATE, e, s}; break; }
        }
        if (r.status != MJX_V_OK) { line = idx + 1; break; }
        if (v_no_room(S, w)) { r = v_unsupported(); line = idx + 1; break; }
        apply_event<true>(c, w, pay, false);
        MJX_SYNCWARP();
        if (S->err != 0) { r = v_unsupported(); line = idx + 1; break; }  // a handler found no room (kawa, fuuro, ...)
        if (ty == LOG_START_KYOKU) ky++;
        if (ty == LOG_HORA) ho++;
    }
    MJX_L0(mjx_verdict& o = V.out[i]; o.status = r.status; o.reason = r.reason; o.line = line; o.seat = r.seat);
}

}  // namespace mjx
