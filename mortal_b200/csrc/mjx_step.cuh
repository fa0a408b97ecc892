// mortal_b200 — the self-play step: one warp advances one table to its next decision point.
//
// Behavioural contract (what must come out bit-identical): libriichi arena/board.rs:141-678,
// arena/game.rs:59-218, state/update.rs, state/action.rs, state/agent_helper.rs:35-79 & 377-462,
// agent/mortal.rs:200-573. How it is computed here is different from the reference:
//  * the table record lives in shared memory; all 32 lanes execute the same control flow over it
//    (branch conditions only read shared state, so they are warp-uniform), mutations are done by one
//    lane (or by lanes 0-3 = seats for per-seat work) followed by MJX_SYNCWARP();
//  * the shanten-heavy loops (update.rs:881-953) are evaluated for all 34 tiles at once, one
//    candidate hand per lane, with warp ballots producing the keep/next/wait bit masks;
//  * public information is stored once per table, not once per seat.
#pragma once
#include "mjx_algo.cuh"
#include "mjx_wall.cuh"

namespace mjx {

enum : u8 { R_NONE = 0, R_DAHAI, R_REACH, R_CHI, R_PON, R_DAIMINKAN, R_KAKAN, R_ANKAN, R_HORA, R_RYUKYOKU };

struct Reaction {
    u8 type, actor, target, pai;
    u8 tsumogiri;
    u8 consumed[4];
    u8 pad_[3];
};

enum : i32 {
    ERR_NONE = 0, ERR_ILLEGAL_ACTION = 1, ERR_KAWA_OVERFLOW = 2, ERR_WALL_EXHAUSTED = 3, ERR_FIFTH_KAN = 4,
    ERR_INTERNAL = 5, ERR_FOUR_WIND_STATE = 6, ERR_NO_KAWA_TILE = 7, ERR_ROW_OVERFLOW = 8, ERR_BAD_POINT = 9,
    ERR_KAN_CHOICE = 10, ERR_GUARD_NEEDS_Q = 11, ERR_SEED_MISMATCH = 12,
    ERR_HIDDEN_OWN_TILE = 13,  // a replayed log hides the player's own tiles (state/update.rs:695-699 "witness an unknown tile")
};

struct WarpScratch {
    Reaction react[4];
    u8 dora_factor[34];
    u8 pad_[2];
    u64 legal[4], legal_kan[4];  // legal masks of the acting seats, recomputed at commit time
};

struct Ctx {
    TableState* S;
    WarpScratch* W;
    Tables T;
    int lane;
    const u8* df;  // dora_factor[34] of the current record (k_step: W->dora_factor; encoder: its own copy)
    // optional mjai event log of this table (arena/result.rs GameResult.game_log); null = not recorded
    u64* log = nullptr;
    i32* log_n = nullptr;
    int log_cap = 0;
    // optional GRP feature rows of this table (dataset/grp.rs:134-147): 7 x i32 per kyoku, written when a kyoku starts
    i32* grp = nullptr;
    i32* grp_n = nullptr;
    int grp_cap = 0;
};

// ---------------------------------------------------------------- event log (mjai/event.rs:20-120, compact form)
// One 64-bit word per event: type | actor << 8 | target << 10 | pai << 12 | tsumogiri << 20 | aux << 21 |
// consumed[0..3] << 24.. | extra << 56. start_kyoku is followed by 2 words of scores and 7 words of haipai
// (4 x 13 tile bytes); hora / ryukyoku by 2 words of deltas. Decoded by mortal_b200/mjai_log.py.
enum : u8 { LOG_START_KYOKU = 1, LOG_TSUMO, LOG_DAHAI, LOG_CHI, LOG_PON, LOG_DAIMINKAN, LOG_KAKAN, LOG_ANKAN, LOG_DORA,
            LOG_REACH, LOG_REACH_ACCEPTED, LOG_HORA, LOG_RYUKYOKU, LOG_END_KYOKU };

MJX_D u64 log_word(int type, int actor, int target, int pai, int tsumogiri, int aux, int c0, int c1, int c2, int c3, int extra) {
    return (u64)(u8)type | ((u64)(actor & 3) << 8) | ((u64)(target & 3) << 10) | ((u64)(u8)pai << 12) | ((u64)(tsumogiri & 1) << 20) |
           ((u64)(aux & 7) << 21) | ((u64)(u8)c0 << 24) | ((u64)(u8)c1 << 32) | ((u64)(u8)c2 << 40) | ((u64)(u8)c3 << 48) |
           ((u64)(u8)extra << 56);
}
// executed by ONE lane; a full log keeps counting so that the host can see the overflow
MJX_D void log_push(const Ctx& c, u64 w) {
    if (!c.log) return;
    const int n = *c.log_n;
    if (n < c.log_cap) c.log[n] = w;
    *c.log_n = n + 1;
}
MJX_D void log_push_i32x4(const Ctx& c, const i32* v) {
    log_push(c, (u64)(u32)v[0] | ((u64)(u32)v[1] << 32));
    log_push(c, (u64)(u32)v[2] | ((u64)(u32)v[3] << 32));
}
MJX_D void log_reaction(const Ctx& c, int type, const Reaction& r) {
    log_push(c, log_word(type, r.actor, r.target, r.pai, r.tsumogiri, 0, r.consumed[0], r.consumed[1], r.consumed[2], r.consumed[3], 0));
}
// board.rs:502-509
#define MJX_ABORTIVE_RYUKYOKU(c) MJX_L0((c).S->bflags |= BF_HAS_ABORTIVE; { const i32 z_[4] = {0, 0, 0, 0}; \
    log_push(c, log_word(LOG_RYUKYOKU, 0, 0, T_UNK, 0, 0, 0, 0, 0, 0, 0)); log_push_i32x4(c, z_); })


MJX_D void set_err(Ctx& c, i32 e) {
    if (MJX_IS_L0(c) && c.S->err == 0) c.S->err = e;
    MJX_SYNCWARP();
}

// may be called by several seat-lanes at once; any non-zero code is fine
MJX_D void atomic_set_err(TableState* S, i32 e) { if (S->err == 0) S->err = e; }

// ---------------------------------------------------------------- small queries (uniform)
MJX_D int n_dora_left(const TableState* S) { return 5 - S->n_dora; }  // unrevealed indicators
MJX_D int dora_indicator(const TableState* S, int k) { return S->wall[60 - k]; }
MJX_D int ura_indicator(const TableState* S, int k) { return S->wall[61 + k]; }

MJX_D void recompute_dora_factor(Ctx& c) {
    const TableState* S = c.S;
    MJX_FOR_TILES(c, t) {
        int f = 0;
        for (int k = 0; k < S->n_dora; k++) f += tile_next(dora_indicator(S, k)) == t;
        c.W->dora_factor[t] = (u8)f;
    }
    MJX_END_TILES(c);
}

// Evaluate f(t) -> 2-bit code for the 34 tile ids, one tile per lane (two passes; the second only
// covers F and C and is skipped when `need_hi` is false), and gather bit0 / bit1 into 34-bit masks.
template <typename F>
MJX_D void tile_eval2(const Ctx& c, bool need_hi, F f, u64& m0, u64& m1) {
#ifdef MJX_HOST_EMUL
    m0 = m1 = 0;
    for (int t = 0; t < (need_hi ? 34 : 32); t++) {
        int code = f(t);
        if (code & 1) m0 |= 1ull << t;
        if (code & 2) m1 |= 1ull << t;
    }
#else
    int code = f(c.lane);
    u64 a = __ballot_sync(0xFFFFFFFFu, code & 1), b = __ballot_sync(0xFFFFFFFFu, code & 2);
    if (need_hi) {
        code = c.lane < 2 ? f(32 + c.lane) : 0;
        a |= (u64)__ballot_sync(0xFFFFFFFFu, code & 1) << 32;
        b |= (u64)__ballot_sync(0xFFFFFFFFu, code & 2) << 32;
    }
    m0 = a;
    m1 = b;
#endif
}
template <typename F>
MJX_D u64 tile_mask(const Ctx& c, F pred) {
    u64 a, b;
    tile_eval2(c, true, [&](int t) { return pred(t) ? 1 : 0; }, a, b);
    return a;
}

// ---------------------------------------------------------------- cooperative shanten blocks
// update.rs:875-878
MJX_D void update_shanten(Ctx& c, int seat) {
    SeatPrivate& P = c.S->priv[seat];
    int sh = max(shanten_all(c.T, P.tehai, P.tehai_len_div3), 0);
    MJX_L0(P.shanten = (i8)sh);
}

// update.rs:881-912 — hand is 3n+2; classify every discardable tile in one sweep
MJX_D void update_shanten_discards(Ctx& c, int seat) {
    SeatPrivate& P = c.S->priv[seat];
    const HandSig base = hand_sig(P.tehai);
    const int len = P.tehai_len_div3, cur = P.shanten;
    u64 next, keep;
    tile_eval2(c, (P.tehai[32] | P.tehai[33]) != 0, [&](int t) {
        int n = P.tehai[t];
        if (n == 0) return 0;
        int after = shanten_all_sig(c.T, sig_variant(base, t, -1, n), len);
        return after < cur ? 1 : (after == cur ? 2 : 0);
    }, next, keep);
    MJX_L0(P.next_shanten = next; P.keep_shanten = keep;
           P.flags = (u16)((P.flags & ~PF_HAS_NEXT_SHANTEN_DISCARD) | (next ? PF_HAS_NEXT_SHANTEN_DISCARD : 0)));
}

// update.rs:916-953 — hand is 3n+1
MJX_D void update_waits_and_furiten(Ctx& c, int seat) {
    SeatPrivate& P = c.S->priv[seat];
    u64 waits = 0, wins = 0;
    if (P.shanten <= 0) {
        const HandSig base = hand_sig(P.tehai);
        const int len = P.tehai_len_div3;
        const u8* seen = c.S->public_seen;
        tile_eval2(c, true, [&](int t) {
            int n = P.tehai[t];
            if (n == 4) return 0;
            if (shanten_all_sig(c.T, sig_variant(base, t, +1, n), len) != -1) return 0;
            return 1 | ((seen[t] + n) < 4 ? 2 : 0);
        }, wins, waits);
    }
    const bool furiten = (wins & P.discarded) != 0;
    MJX_L0(P.waits = waits; P.flags = (u16)((P.flags & ~PF_AT_FURITEN) | (furiten ? PF_AT_FURITEN : 0)));
}

// ---------------------------------------------------------------- per-seat helpers
MJX_D AgariQuery make_query(const TableState* S, int seat, const u8* tehai, int win_tile, bool is_ron) {
    const SeatPrivate& P = S->priv[seat];
    AgariQuery q;
    q.tehai = tehai;
    q.chis = P.chis; q.pons = P.pons; q.minkans = P.minkans; q.ankans = P.ankans;
    q.n_chis = P.n_chis; q.n_pons = P.n_pons; q.n_minkans = P.n_minkans; q.n_ankans = P.n_ankans;
    q.bakaze = T_E + S->kyoku / 4;
    q.jikaze = T_E + ((seat + 4 - S->oya) & 3);
    q.winning_tile = win_tile;
    q.is_ron = is_ron;
    q.is_menzen = (P.flags & PF_IS_MENZEN) != 0;
    return q;
}

// agent_helper.rs:201-206
MJX_D int yaokyuu_kinds(const u8* tehai) {
    int n = 0;
#pragma unroll
    for (int t = 0; t < 34; t++) if ((YAOKYUU_MASK >> t) & 1ull) n += tehai[t] > 0;
    return n;
}

// update.rs:826-868 — returns CAN_CHI_* bits
MJX_D u16 can_chi_bits(const u8* tehai, int tid) {
    int num = tid % 9 + 1;
    int total = 0;
#pragma unroll
    for (int t = 0; t < 34; t++) total += tehai[t];
    u16 bits = 0;
    // "any tile left after the call that is not a swap-call tile"
    if (num <= 7 && tehai[tid + 1] > 0 && tehai[tid + 2] > 0) {
        int rem = total - tehai[tid] - 2 - (num < 7 ? tehai[tid + 3] : 0);
        if (rem > 0) bits |= CAN_CHI_LOW;
    }
    if (num >= 2 && num <= 8 && tehai[tid - 1] > 0 && tehai[tid + 1] > 0) {
        int rem = total - tehai[tid] - 2;
        if (rem > 0) bits |= CAN_CHI_MID;
    }
    if (num >= 3 && tehai[tid - 2] > 0 && tehai[tid - 1] > 0) {
        int rem = total - tehai[tid] - 2 - (num > 3 ? tehai[tid - 3] : 0);
        if (rem > 0) bits |= CAN_CHI_HIGH;
    }
    return bits;
}

// agari.rs:854-912 with strict = false (Tenhou rule), evaluated by one lane
MJX_DN bool ankan_after_riichi_ok(const Tables& T, const u8* tehai, int len_div3, int tile_id) {
    if (tehai[tile_id] != 4) return false;
    if (tile_id >= 27) return true;
    u8 before[34];
    for (int i = 0; i < 34; i++) before[i] = tehai[i];
    before[tile_id] -= 1;
    HandSig base = hand_sig(before);
    for (int t = 0; t < 34; t++) {
        if (before[t] == 4) continue;
        if (shanten_all_sig(T, sig_variant(base, t, +1, before[t]), len_div3) != -1) continue;
        if (t == tile_id) return false;
        u8 after[34];
        for (int i = 0; i < 34; i++) after[i] = tehai[i];
        after[tile_id] = 0;
        after[t] += 1;
        u8 t14[14];
        u32 divs[4];
        if (agari_lookup(T, tile14_and_key(after, t14), divs) < 0) return false;
    }
    return true;
}

// ---------------------------------------------------------------- event prologue (update.rs:46-61)
// KEEP_CANS: update_with_keep_cans(ev, true) for an in-game announce (ReachAccepted / Dora / Hora): the seats keep their last
// cans, target actor and kan candidates (only bin/validate_logs.rs asks for that; every other caller resets them).
template <bool KEEP_CANS = false>
MJX_D void ev_prologue(Ctx& c, int actor /* -1 if the event has no actor */) {
    MJX_FOR_SEATS(c, s) {
        SeatPrivate& P = c.S->priv[s];
        if (!KEEP_CANS) {
            P.cans = 0;
            P.target_actor = (u8)(actor >= 0 ? actor : s);
            P.ankan_cand = 0;
            P.kakan_cand = 0;
        }
        u16 f = P.flags;
        if (f & PF_MARK_SAME_CYCLE_FURITEN) f = (u16)((f & ~PF_MARK_SAME_CYCLE_FURITEN) | PF_AT_FURITEN);
        if (f & PF_CHANKAN_CHANCE) f = (u16)(f & ~(PF_CHANKAN_CHANCE | PF_AT_IPPATSU));
        P.flags = f;
    }
    MJX_END_SEATS(c);
}

// public witness of a tile (update.rs:695-727, the part every other seat performs)
MJX_D void public_witness(TableState* S, int tile) {
    S->public_seen[deaka(tile)] += 1;
    if (is_aka(tile)) S->akas_public |= (u8)(1 << (tile - T_5MR));
}

// ---------------------------------------------------------------- events
// update.rs:780-808 + board.rs:353-364
template <bool KEEP_CANS = false>
MJX_D void ev_dora(Ctx& c) {
    TableState* S = c.S;
    if (S->n_dora >= 5) { set_err(c, ERR_FIFTH_KAN); return; }
    // ReachAccepted / Dora / Hora are "in-game announces" but the arena always resets cans (update.rs:25)
    ev_prologue<KEEP_CANS>(c, -1);
    MJX_L0(log_push(c, log_word(LOG_DORA, 0, 0, S->wall[60 - S->n_dora], 0, 0, 0, 0, 0, 0, 0));
           public_witness(S, S->wall[60 - S->n_dora]); S->n_dora += 1);
    recompute_dora_factor(c);
}

// update.rs:125-217 (+ board.rs:206-239 haipai)
MJX_DN void ev_start_kyoku(Ctx& c) {
    TableState* S = c.S;
    ev_prologue(c, -1);
    // reset public + private, deal the 13 tiles
    MJX_FOR_SEATS(c, s) {
        SeatPublic& U = S->pub[s];
        U.kawa_len = 0; U.n_fuuro = 0; U.n_ankan = 0;
        U.last_tedashi_flags = 0; U.riichi_flags = 0; U.last_tedashi_tile = T_NONE; U.riichi_tile = T_NONE;
        for (int i = 0; i < 4; i++) { U.ankan[i] = T_NONE; for (int j = 0; j < 4; j++) U.fuuro[i][j] = T_NONE; }
        SeatPrivate& P = S->priv[s];
        for (int t = 0; t < 34; t++) P.tehai[t] = 0;
        P.waits = P.keep_shanten = P.next_shanten = P.forbidden = P.discarded = 0;
        P.ankan_cand = P.kakan_cand = 0;
        P.flags = PF_IS_MENZEN | PF_CAN_W_RIICHI;
        P.cans = 0;
        P.last_self_tsumo = T_NONE;
        P.akas_in_hand = 0;
        P.at_turn = 0;
        P.n_chis = P.n_pons = P.n_minkans = P.n_ankans = 0;
        P.tehai_len_div3 = 4;
        P.shanten = 0;
        for (int i = 0; i < 13; i++) {
            int t = S->wall[13 * s + i];
            if (t >= T_UNK) continue;  // `?`: another seat's hand seen from a single PlayerState
            P.tehai[deaka(t)] += 1;
            if (is_aka(t)) P.akas_in_hand |= (u8)(1 << (t - T_5MR));
        }
    }
    MJX_END_SEATS(c);
    MJX_FOR_TILES(c, t) S->public_seen[t] = 0;
    MJX_END_TILES(c);
    if (MJX_IS_L0(c)) {
        S->akas_public = 0;
        S->riichi_declared = 0; S->riichi_accepted = 0;
        S->last_kawa_tile = T_NONE;
        S->n_intermediate_kan = 0;
        S->bflags &= ~BF_HAS_CHIPON_PENDING;
        S->n_dora = 0;
    }
    MJX_SYNCWARP();
    MJX_L0(public_witness(S, S->wall[60]); S->n_dora = 1);
    if (MJX_IS_L0(c) && c.log) {
        log_push(c, log_word(LOG_START_KYOKU, 0, 0, S->wall[60], 0, 0, S->kyoku, S->honba, S->kyotaku, S->oya, 0));
        log_push_i32x4(c, S->scores);
        for (int w = 0; w < 7; w++) {
            u64 v = 0;
            for (int b = 0; b < 8; b++) { const int i = w * 8 + b; if (i < 52) v |= (u64)S->wall[i] << (8 * b); }
            log_push(c, v);
        }
    }
    recompute_dora_factor(c);
    for (int s = 0; s < 4; s++) {
        if (!seat_known(S, s)) continue;
        update_shanten(c, s);
        update_waits_and_furiten(c, s);
    }
}

// update.rs:219-309
MJX_DN void ev_tsumo(Ctx& c, int actor, int pai) {
    TableState* S = c.S;
    ev_prologue(c, actor);
    SeatPrivate& P = S->priv[actor];
    if (!seat_known(S, actor)) {  // update.rs:220-225: somebody else's draw only shortens the wall
        MJX_L0(S->tiles_left -= 1);
        return;
    }
    const int pid = deaka(pai);
    const bool riichi_acc = (S->riichi_accepted >> actor) & 1;
    MJX_L0(S->tiles_left -= 1;
           P.at_turn += 1;
           P.cans |= CAN_DISCARD;
           P.last_self_tsumo = (u8)pai;
           P.tehai[pid] += 1;
           if (is_aka(pai)) P.akas_in_hand |= (u8)(1 << (pai - T_5MR)));

    u16 cans = CAN_DISCARD;
    if ((P.flags & PF_CAN_W_RIICHI) && yaokyuu_kinds(P.tehai) >= 9) cans |= CAN_RYUKYOKU;
    if (!riichi_acc) update_shanten_discards(c, actor);

    if ((P.waits >> pid) & 1) {
        bool ok;
        if ((P.flags & (PF_IS_MENZEN | PF_AT_RINSHAN | PF_CAN_W_RIICHI)) || riichi_acc || S->tiles_left == 0) ok = true;
        else ok = has_yaku(c.T, make_query(S, actor, P.tehai, pid, false));
        if (ok) cans |= CAN_TSUMO_AGARI;
    }

    u64 ankan_c = 0, kakan_c = 0;
    if (S->tiles_left != 0) {
        if (riichi_acc) {
            if (S->kans < 4 && ankan_after_riichi_ok(c.T, P.tehai, P.tehai_len_div3, pid)) {
                cans |= CAN_ANKAN;
                ankan_c = 1ull << pid;
            }
        } else {
            if (S->kans < 4) {
                ankan_c = tile_mask(c, [&](int t) { return P.tehai[t] == 4; });
                u64 ponmask = 0;
                for (int i = 0; i < P.n_pons; i++) ponmask |= 1ull << P.pons[i];
                u64 have = tile_mask(c, [&](int t) { int n = P.tehai[t]; return n > 0 && n < 4; });
                kakan_c = have & ponmask;
                if (ankan_c) cans |= CAN_ANKAN;
                if (kakan_c) cans |= CAN_KAKAN;
            }
            if ((P.flags & PF_IS_MENZEN) && S->tiles_left >= 4 && S->scores[actor] >= 1000 &&
                (P.shanten == 0 || (P.shanten == 1 && (P.flags & PF_HAS_NEXT_SHANTEN_DISCARD))))
                cans |= CAN_RIICHI;
        }
    }
    MJX_L0(P.cans = cans; P.ankan_cand = ankan_c; P.kakan_cand = kakan_c);
}

MJX_D void kawa_push(Ctx& c, int seat, const KawaItem& it) {
    SeatPublic& U = c.S->pub[seat];
    if (U.kawa_len >= KAWA_CAP) { if (c.S->err == 0) c.S->err = ERR_KAWA_OVERFLOW; return; }
    U.kawa[U.kawa_len] = it;
    U.kawa_len += 1;
}

// update.rs:311-427
MJX_DN void ev_dahai(Ctx& c, int actor, int pai, bool tsumogiri) {
    TableState* S = c.S;
    ev_prologue(c, actor);
    SeatPrivate& A = S->priv[actor];
    const int pid = deaka(pai);
    const bool is_riichi = ((S->riichi_declared >> actor) & 1) && !((S->riichi_accepted >> actor) & 1);
    const bool actor_riichi_acc = (S->riichi_accepted >> actor) & 1;
    const bool known = seat_known(S, actor);
    if (MJX_IS_L0(c)) {
        if (known) {
            A.tehai[pid] -= 1;
            if (is_aka(pai)) A.akas_in_hand &= (u8)~(1 << (pai - T_5MR));
        }
        public_witness(S, pai);
        KawaItem it;
        it.tile = (u8)pai;
        it.flags = (u8)((c.df[pid] > 0 ? SF_DORA : 0) | (!tsumogiri ? SF_TEDASHI : 0) | (is_riichi ? SF_RIICHI : 0) |
                        ((S->bflags & BF_HAS_CHIPON_PENDING) ? SF_HAS_CHIPON : 0));
        it.consumed[0] = S->chipon_consumed[0];
        it.consumed[1] = S->chipon_consumed[1];
        for (int i = 0; i < 4; i++) it.kan[i] = i < S->n_intermediate_kan ? S->intermediate_kan[i] : T_NONE;
        S->n_intermediate_kan = 0;
        S->bflags &= ~BF_HAS_CHIPON_PENDING;
        kawa_push(c, actor, it);
        S->last_kawa_tile = (u8)pai;
        SeatPublic& U = S->pub[actor];
        u8 sf = (u8)(SF_VALID | (it.flags & (SF_DORA | SF_TEDASHI | SF_RIICHI)));
        if (!tsumogiri) { U.last_tedashi_tile = (u8)pai; U.last_tedashi_flags = sf; }
        if (is_riichi) { U.riichi_tile = (u8)pai; U.riichi_flags = sf; }
        A.forbidden = 0;
        A.flags &= (u16)~(PF_AT_RINSHAN | PF_AT_IPPATSU | PF_CAN_W_RIICHI);
        A.discarded |= 1ull << pid;
    }
    MJX_SYNCWARP();

    // the discarder's own shanten / waits (3n+1 now)
    if (!known) {
    } else if (!actor_riichi_acc) {
        if ((A.next_shanten >> pid) & 1) { MJX_L0(A.shanten -= 1); }
        else if (!((A.keep_shanten >> pid) & 1)) update_shanten(c, actor);
        update_waits_and_furiten(c, actor);
    } else if (!(A.flags & PF_AT_FURITEN) && ((A.waits >> pid) & 1)) {
        MJX_L0(A.flags |= PF_AT_FURITEN);
    }

    // the three other seats react in parallel: lane s = seat s
    MJX_FOR_SEATS(c, s) if (s != actor) {
        SeatPrivate& P = S->priv[s];
        const bool racc = (S->riichi_accepted >> s) & 1;
        u16 cans = 0;
        u16 fl = P.flags;
        if (!(fl & PF_AT_FURITEN) && ((P.waits >> pid) & 1)) {
            bool ron;
            if (racc || S->tiles_left == 0) ron = true;
            else {
                u8 th[34];
                for (int i = 0; i < 34; i++) th[i] = P.tehai[i];
                th[pid] += 1;
                ron = has_yaku(c.T, make_query(S, s, th, pid, true));
            }
            if (ron) { cans |= CAN_RON_AGARI; fl |= PF_MARK_SAME_CYCLE_FURITEN; }
            else fl |= PF_AT_FURITEN;
        }
        if (!(racc || S->tiles_left == 0)) {
            if (((actor + 1) & 3) == s && !is_jihai(pai) && P.tehai_len_div3 > 0) cans |= can_chi_bits(P.tehai, pid);
            if (P.tehai[pid] >= 2) cans |= CAN_PON;
            if (S->kans < 4 && P.tehai[pid] == 3) cans |= CAN_DAIMINKAN;
        }
        P.cans = cans;
        P.flags = fl;
    }
    MJX_END_SEATS(c);
}

// shared by chi / pon / daiminkan for the non-actors (update.rs:438-447 etc.)
MJX_D void others_after_call(Ctx& c, int actor) {
    MJX_FOR_SEATS(c, s) if (s != actor) c.S->priv[s].flags &= (u16)~(PF_CAN_W_RIICHI | PF_AT_IPPATSU);
    MJX_END_SEATS(c);
}

MJX_D void consume_from_hand(SeatPrivate& P, TableState* S, int tile, bool known = true) {
    if (known) {
        P.tehai[deaka(tile)] -= 1;
        if (is_aka(tile)) P.akas_in_hand &= (u8)~(1 << (tile - T_5MR));
    }
    public_witness(S, tile);
}

MJX_D void push_fuuro(TableState* S, int actor, const u8* tiles, int n) {
    SeatPublic& U = S->pub[actor];
    if (U.n_fuuro >= 4) { if (S->err == 0) S->err = ERR_INTERNAL; return; }
    for (int i = 0; i < 4; i++) U.fuuro[U.n_fuuro][i] = i < n ? tiles[i] : T_NONE;
    U.n_fuuro += 1;
}

// update.rs:810-817
MJX_D void pad_kawa_for_call(Ctx& c, int actor, int target) {
    KawaItem pad;
    pad.tile = T_NONE; pad.flags = 0; pad.consumed[0] = pad.consumed[1] = T_NONE;
    for (int i = 0; i < 4; i++) pad.kan[i] = T_NONE;
    for (int i = (target + 1) & 3; i != actor; i = (i + 1) & 3) kawa_push(c, i, pad);
}

// update.rs:429-495
MJX_DN void ev_chi(Ctx& c, const Reaction& r) {
    TableState* S = c.S;
    const int actor = r.actor, pai = r.pai;
    ev_prologue(c, actor);
    SeatPrivate& P = S->priv[actor];
    if (MJX_IS_L0(c)) {
        u8 set[3] = {r.consumed[0], r.consumed[1], (u8)pai};
        push_fuuro(S, actor, set, 3);
        S->bflags |= BF_HAS_CHIPON_PENDING;
        S->chipon_consumed[0] = (u8)deaka(r.consumed[0]);
        S->chipon_consumed[1] = (u8)deaka(r.consumed[1]);
        P.cans |= CAN_DISCARD;
        P.flags &= (u16)~PF_IS_MENZEN;
        P.tehai_len_div3 -= 1;
        P.last_self_tsumo = T_NONE;
        consume_from_hand(P, S, r.consumed[0], seat_known(S, actor));
        consume_from_hand(P, S, r.consumed[1], seat_known(S, actor));
        int a = deaka(r.consumed[0]), b = deaka(r.consumed[1]);
        int mn = min(a, b), mx = max(a, b), tid = deaka(pai);
        P.chis[P.n_chis++] = (u8)min(mn, tid);
        u64 forb = 0;
        if (P.tehai[tid] > 0) forb |= 1ull << tid;
        if (tid < mn) {
            if (mx % 9 < 8 && P.tehai[mx + 1] > 0) forb |= 1ull << (mx + 1);
        } else if (tid > mx && mn % 9 > 0) {
            if (P.tehai[mn - 1] > 0) forb |= 1ull << (mn - 1);
        }
        P.forbidden |= forb;
    }
    MJX_SYNCWARP();
    others_after_call(c, actor);
    if (!seat_known(S, actor)) return;
    update_shanten(c, actor);
    update_shanten_discards(c, actor);
}

// update.rs:497-542
MJX_DN void ev_pon(Ctx& c, const Reaction& r) {
    TableState* S = c.S;
    const int actor = r.actor, pai = r.pai, pid = deaka(pai);
    ev_prologue(c, actor);
    SeatPrivate& P = S->priv[actor];
    if (MJX_IS_L0(c)) {
        u8 set[3] = {r.consumed[0], r.consumed[1], (u8)pai};
        push_fuuro(S, actor, set, 3);
        S->bflags |= BF_HAS_CHIPON_PENDING;
        S->chipon_consumed[0] = (u8)deaka(r.consumed[0]);
        S->chipon_consumed[1] = (u8)deaka(r.consumed[1]);
        pad_kawa_for_call(c, actor, r.target);
        P.cans |= CAN_DISCARD;
        P.flags &= (u16)~PF_IS_MENZEN;
        P.tehai_len_div3 -= 1;
        P.last_self_tsumo = T_NONE;
        consume_from_hand(P, S, r.consumed[0], seat_known(S, actor));
        consume_from_hand(P, S, r.consumed[1], seat_known(S, actor));
        P.pons[P.n_pons++] = (u8)pid;
        if (P.tehai[pid] > 0) P.forbidden |= 1ull << pid;
    }
    MJX_SYNCWARP();
    others_after_call(c, actor);
    if (!seat_known(S, actor)) return;
    update_shanten(c, actor);
    update_shanten_discards(c, actor);
}

// update.rs:544-582
MJX_DN void ev_daiminkan(Ctx& c, const Reaction& r) {
    TableState* S = c.S;
    const int actor = r.actor, pai = r.pai;
    ev_prologue(c, actor);
    SeatPrivate& P = S->priv[actor];
    if (MJX_IS_L0(c)) {
        u8 set[4] = {r.consumed[0], r.consumed[1], r.consumed[2], (u8)pai};
        push_fuuro(S, actor, set, 4);
        if (S->n_intermediate_kan < 4) S->intermediate_kan[S->n_intermediate_kan++] = (u8)deaka(pai);
        pad_kawa_for_call(c, actor, r.target);
        P.flags = (u16)((P.flags | PF_AT_RINSHAN) & ~PF_IS_MENZEN);
        P.tehai_len_div3 -= 1;
        for (int i = 0; i < 3; i++) consume_from_hand(P, S, r.consumed[i], seat_known(S, actor));
        P.minkans[P.n_minkans++] = (u8)deaka(pai);
    }
    MJX_SYNCWARP();
    others_after_call(c, actor);
    if (!seat_known(S, actor)) return;
    update_shanten(c, actor);
    update_waits_and_furiten(c, actor);
}

// update.rs:584-628
MJX_DN void ev_kakan(Ctx& c, const Reaction& r) {
    TableState* S = c.S;
    const int actor = r.actor, pai = r.pai, pid = deaka(pai);
    ev_prologue(c, actor);
    SeatPrivate& P = S->priv[actor];
    const bool was_next = (P.next_shanten >> pid) & 1, was_keep = (P.keep_shanten >> pid) & 1;
    if (MJX_IS_L0(c)) {
        SeatPublic& U = S->pub[actor];
        for (int f = 0; f < U.n_fuuro; f++) {
            if (deaka(U.fuuro[f][0]) == pid) { U.fuuro[f][3] = (u8)pai; break; }
        }
        if (S->n_intermediate_kan < 4) S->intermediate_kan[S->n_intermediate_kan++] = (u8)pid;
        S->last_kawa_tile = (u8)pai;  // read by the chankan ronners only (update.rs:599)
        P.flags |= PF_AT_RINSHAN;
        consume_from_hand(P, S, pai, seat_known(S, actor));
        int w = 0;
        for (int i = 0; i < P.n_pons; i++) if (P.pons[i] != pid) P.pons[w++] = P.pons[i];
        P.n_pons = (u8)w;
        P.minkans[P.n_minkans++] = (u8)pid;
    }
    MJX_SYNCWARP();
    // chankan window for the others (update.rs:596-609)
    MJX_FOR_SEATS(c, s) if (s != actor) {
        SeatPrivate& O = S->priv[s];
        if (!(O.flags & PF_AT_FURITEN) && ((O.waits >> pid) & 1)) {
            O.cans |= CAN_RON_AGARI;
            O.flags |= PF_MARK_SAME_CYCLE_FURITEN | PF_CHANKAN_CHANCE;
        } else {
            O.flags &= (u16)~PF_AT_IPPATSU;
        }
    }
    MJX_END_SEATS(c);
    if (!seat_known(S, actor)) return;
    if (was_next) { MJX_L0(P.shanten -= 1); }
    else if (!was_keep) update_shanten(c, actor);
    update_waits_and_furiten(c, actor);
}

// update.rs:630-663
MJX_DN void ev_ankan(Ctx& c, const Reaction& r) {
    TableState* S = c.S;
    const int actor = r.actor, tile = deaka(r.consumed[0]);
    ev_prologue(c, actor);
    SeatPrivate& P = S->priv[actor];
    MJX_FOR_SEATS(c, s) S->priv[s].flags &= (u16)~(PF_CAN_W_RIICHI | PF_AT_IPPATSU);
    MJX_END_SEATS(c);
    if (MJX_IS_L0(c)) {
        SeatPublic& U = S->pub[actor];
        if (U.n_ankan < 4) U.ankan[U.n_ankan++] = (u8)tile;
        if (S->n_intermediate_kan < 4) S->intermediate_kan[S->n_intermediate_kan++] = (u8)tile;
        P.flags |= PF_AT_RINSHAN;
        P.tehai_len_div3 -= 1;
        for (int i = 0; i < 4; i++) consume_from_hand(P, S, r.consumed[i], seat_known(S, actor));
        P.ankans[P.n_ankans++] = (u8)tile;
    }
    MJX_SYNCWARP();
    if (seat_known(S, actor) && !((S->riichi_accepted >> actor) & 1)) {
        update_shanten(c, actor);
        update_waits_and_furiten(c, actor);
    }
}

// update.rs:665-675
MJX_D void ev_reach(Ctx& c, int actor) {
    ev_prologue(c, actor);
    MJX_L0(c.S->riichi_declared |= (u8)(1 << actor);
           SeatPrivate& P = c.S->priv[actor];
           if (P.flags & PF_CAN_W_RIICHI) P.flags |= PF_IS_W_RIICHI; else P.flags &= (u16)~PF_IS_W_RIICHI;
           P.cans |= CAN_DISCARD);
}

// update.rs:677-686 + board.rs:342-351
template <bool KEEP_CANS = false>
MJX_D void check_riichi_accepted(Ctx& c) {
    TableState* S = c.S;
    if (S->riichi_to_be_accepted < 0) return;
    const int actor = S->riichi_to_be_accepted;
    ev_prologue<KEEP_CANS>(c, actor);
    MJX_L0(log_push(c, log_word(LOG_REACH_ACCEPTED, actor, 0, T_UNK, 0, 0, 0, 0, 0, 0, 0));
           S->riichi_to_be_accepted = -1;
           S->riichi_accepted |= (u8)(1 << actor);
           S->priv[actor].flags |= PF_AT_IPPATSU;
           S->scores[actor] -= 1000;
           S->kyotaku += 1;
           S->accepted_riichis += 1);
}

// ---------------------------------------------------------------- scoring
// recount of doras_owned[0] (state/test.rs:30-47 invariant) for `seat`
MJX_D int doras_owned_self(const Ctx& c, int seat) {
    const TableState* S = c.S;
    const SeatPrivate& P = S->priv[seat];
    const SeatPublic& U = S->pub[seat];
    int n = mjx_popc(P.akas_in_hand);
    for (int t = 0; t < 34; t++) n += P.tehai[t] * c.df[t];
    for (int f = 0; f < U.n_fuuro; f++)
        for (int i = 0; i < 4; i++) {
            int t = U.fuuro[f][i];
            if (t == T_NONE) continue;
            n += c.df[deaka(t)] + (is_aka(t) ? 1 : 0);
        }
    for (int i = 0; i < U.n_ankan; i++) {
        int t = U.ankan[i];
        n += 4 * c.df[t] + ((t == T_5M || t == T_5P || t == T_5S) ? 1 : 0);
    }
    return n;
}

// agent_helper.rs:377-462; executed redundantly by every lane (uniform), n_ura = revealed ura count
MJX_DN Point agari_points_ura(const Ctx& c, int seat, bool is_ron, const u8* ura, int n_ura, bool* ok) {
    const TableState* S = c.S;
    const SeatPrivate& P = S->priv[seat];
    const bool is_oya = seat == S->oya;
    *ok = true;
    if (!is_ron && (P.flags & PF_CAN_W_RIICHI)) return point_yakuman(is_oya, 1);
    int winning_tile = is_ron ? S->last_kawa_tile : P.last_self_tsumo;
    if (winning_tile == T_NONE) { *ok = false; return point_yakuman(is_oya, 0); }
    const bool racc = (S->riichi_accepted >> seat) & 1;
    int add = (racc ? 1 : 0) + ((P.flags & PF_IS_W_RIICHI) ? 1 : 0) + ((P.flags & PF_AT_IPPATSU) ? 1 : 0);
    if (is_ron) {
        add += (S->tiles_left == 0) + ((P.flags & PF_CHANKAN_CHANCE) ? 1 : 0);
    } else {
        const bool rinshan = (P.flags & PF_AT_RINSHAN) != 0;
        add += ((P.flags & PF_IS_MENZEN) ? 1 : 0) + ((S->tiles_left == 0 && !rinshan) ? 1 : 0) + (rinshan ? 1 : 0);
    }
    u8 th[34];
    for (int i = 0; i < 34; i++) th[i] = P.tehai[i];
    int doras = doras_owned_self(c, seat);
    const int wid = deaka(winning_tile);
    if (is_ron) {
        th[wid] += 1;
        doras += c.df[wid] + (is_aka(winning_tile) ? 1 : 0);
    }
    if (racc) {
        const SeatPublic& U = S->pub[seat];
        for (int k = 0; k < n_ura; k++) {
            int next = tile_next(ura[k]);
            int cnt = th[next];
            for (int i = 0; i < U.n_ankan; i++) if (U.ankan[i] == next) cnt += 4;
            doras += cnt;
        }
    }
    Agari a = agari_with(c.T, make_query(S, seat, th, wid, is_ron), add, doras & 0xFF);
    if (a.kind == 0) { *ok = false; return point_yakuman(is_oya, 0); }
    bool pok;
    Point p = agari_point(a, is_oya, &pok);
    if (!pok) *ok = false;
    return p;
}

// the board's own ura indicators: wall[61 + k] (board.rs:381-382)
MJX_D Point agari_points(const Ctx& c, int seat, bool is_ron, int n_ura, bool* ok) {
    return agari_points_ura(c, seat, is_ron, c.S->wall + 61, n_ura, ok);
}

// agent_helper.rs:262-368 — the all-last "do not win into 4th place" guard. Executed by one lane.
MJX_DN bool rule_based_agari(const Ctx& c, int p) {
    const TableState* S = c.S;
    const SeatPrivate& P = S->priv[p];
    if (!(P.cans & CAN_AGARI)) return false;
    const bool is_ron = (P.cans & CAN_RON_AGARI) != 0;
    const int target_rel = (P.target_actor - p) & 3;
    const int bakaze = T_E + S->kyoku / 4, kyoku_in_wind = S->kyoku & 3;
    const bool is_all_last = bakaze == T_E ? false : (bakaze == T_S ? kyoku_in_wind == 3 : true);
    const int oya_rel = (S->oya - p) & 3;
    i32 sc[4];
    for (int i = 0; i < 4; i++) sc[i] = S->scores[(p + i) & 3];
    auto rank_of = [&](const i32* rel) {  // update.rs:966-972 get_rank on relative scores
        int r = 0;
        for (int i = 1; i < 4; i++) {
            const int s = (p + i) & 3;
            if (rel[i] > rel[0] || (rel[i] == rel[0] && s < p)) r++;
        }
        return r;
    };
    if (!is_all_last || oya_rel == 0 || rank_of(sc) < 3) return true;
    if (bakaze == T_W) {
        if (kyoku_in_wind < 3) return true;
    } else if (sc[0] < 30000 && sc[1] < 30000 && sc[2] < 30000 && sc[3] < 30000) {
        return true;
    }
    const bool racc = (S->riichi_accepted >> p) & 1;
    bool ok;
    Point pt;
    if (racc) {
        // most valuable possible ura indicators first (agent_helper.rs:294-326)
        u8 full[34], seen[34];
        const SeatPublic& U = S->pub[p];
        for (int t = 0; t < 34; t++) { full[t] = P.tehai[t]; seen[t] = (u8)(S->public_seen[t] + P.tehai[t]); }
        for (int j = 0; j < U.n_ankan; j++) full[U.ankan[j]] += 4;
        u8 ura[5]; int n_ura = 0;
        u64 used = 0;
        bool done = false;
        for (int round = 0; round < 34 && !done; round++) {
            // next tile by descending count, ascending id among equals (stable order of the reference's small sort)
            int best = -1;
            for (int t = 0; t < 34; t++)
                if (full[t] > 0 && !((used >> t) & 1) && (best < 0 || full[t] > full[best])) best = t;
            if (best < 0) break;
            used |= 1ull << best;
            const int ind = tile_prev(best);
            for (;;) {
                if (n_ura >= S->n_dora) { done = true; break; }
                if (seen[ind] >= 4) break;
                ura[n_ura++] = (u8)ind;
                seen[ind] += 1;
            }
        }
        pt = agari_points_ura(c, p, is_ron, ura, n_ura, &ok);
    } else {
        pt = agari_points_ura(c, p, is_ron, nullptr, 0, &ok);
    }
    if (!ok) return true;  // the reference unwraps; cannot happen when can_agari holds
    i32 ex[4] = {sc[0], sc[1], sc[2], sc[3]};
    const i32 kyotaku = S->kyotaku, honba = S->honba;
    if (is_ron) {
        ex[0] += pt.ron + kyotaku * 1000 + honba * 300;
        ex[target_rel] -= pt.ron + honba * 300;
    } else {
        ex[0] += tsumo_total(pt, false) + kyotaku * 1000 + honba * 300;
        for (int i = 1; i < 4; i++) ex[i] -= (i == oya_rel ? pt.tsumo_oya : pt.tsumo_ko) + honba * 100;
    }
    if (ex[0] < 30000 && ex[1] < 30000 && ex[2] < 30000 && ex[3] < 30000) return true;
    return rank_of(ex) < 3;
}

// Hora event of one winner (board.rs:421-431, 456-468): ura markers only for an accepted riichi
MJX_D void log_hora(const Ctx& c, int actor, int target, const i32* deltas, int n_ura) {
    if (!MJX_IS_L0(c) || !c.log) return;
    const TableState* S = c.S;
    const int nu = ((S->riichi_accepted >> actor) & 1) ? n_ura : 0;
    u8 u[5] = {T_UNK, T_UNK, T_UNK, T_UNK, T_UNK};
    for (int j = 0; j < nu; j++) u[j] = S->wall[61 + j];
    log_push(c, log_word(LOG_HORA, actor, target, T_UNK, 0, nu, u[0], u[1], u[2], u[3], u[4]));
    log_push_i32x4(c, deltas);
}

// board.rs:366-471
MJX_DN void handle_hora(Ctx& c, int single_actor, int single_target) {
    TableState* S = c.S;
    const bool is_ron = single_actor != single_target;
    const int n_ura = 5 - n_dora_left(S);  // = ura_indicators[..5 - dora_indicators.len()]
    i32 honba_left = S->honba;
    i32 kyotaku_point = (i32)S->kyotaku * 1000;
    i32 deltas_total[4] = {0, 0, 0, 0};
    bool renchan = false, bad = false;

    if (is_ron) {
        for (int k = 1; k <= 3; k++) {
            int actor = (single_target + k) & 3;
            if (c.W->react[actor].type != R_HORA) continue;
            renchan |= actor == S->oya;
            bool ok;
            Point p = agari_points(c, actor, true, n_ura, &ok);
            bad |= !ok;
            i32 d[4] = {0, 0, 0, 0};
            if (S->paos[actor] >= 0) {
                d[S->paos[actor]] = -p.ron / 2 - honba_left * 300;
                d[single_target] -= p.ron / 2;
            } else {
                d[single_target] = -p.ron - honba_left * 300;
            }
            d[actor] = p.ron + kyotaku_point + honba_left * 300;
            kyotaku_point = 0;
            honba_left = 0;
            for (int j = 0; j < 4; j++) deltas_total[j] += d[j];
            log_hora(c, actor, single_target, d, n_ura);
        }
    } else {
        renchan = single_actor == S->oya;
        bool ok;
        Point p = agari_points(c, single_actor, false, n_ura, &ok);
        bad |= !ok;
        i32 d[4];
        if (S->paos[single_actor] >= 0) {
            for (int j = 0; j < 4; j++) d[j] = 0;
            d[S->paos[single_actor]] = -p.ron - honba_left * 300;
        } else {
            for (int j = 0; j < 4; j++) d[j] = -p.tsumo_ko - honba_left * 100;
            if (single_actor != S->oya) d[S->oya] = -p.tsumo_oya - honba_left * 100;
        }
        d[single_actor] = tsumo_total(p, single_actor == S->oya) + kyotaku_point + honba_left * 300;
        for (int j = 0; j < 4; j++) deltas_total[j] += d[j];
        log_hora(c, single_actor, single_target, d, n_ura);
    }
    // NOTE board.rs:387: can_renchan is OR-ed for every Hora reaction, including ron reactions
    if (is_ron)
        for (int a = 0; a < 4; a++) if (c.W->react[a].type == R_HORA && a == S->oya) renchan = true;
    MJX_L0(S->bflags |= BF_HAS_HORA | (renchan ? BF_CAN_RENCHAN : 0);
           S->kyotaku = 0;
           for (int j = 0; j < 4; j++) S->kyoku_deltas[j] += deltas_total[j];
           if (bad && S->err == 0) S->err = ERR_BAD_POINT);
}

// board.rs:241-294
MJX_DN void exhaustive_ryukyoku(Ctx& c) {
    TableState* S = c.S;
    i32 deltas[4] = {0, 0, 0, 0};
    const int oya = S->oya;
    bool renchan = S->priv[oya].shanten == 0;
    bool has_nagashi = false;
    for (int i = 0; i < 4; i++) {
        if (!((S->can_nagashi >> i) & 1)) continue;
        has_nagashi = true;
        for (int j = 0; j < 4; j++) {
            if (i == oya) deltas[j] += j == i ? 12000 : -4000;
            else deltas[j] += j == i ? 8000 : (j == oya ? -4000 : -2000);
        }
    }
    if (!has_nagashi) {
        int n = 0;
        for (int i = 0; i < 4; i++) n += S->priv[i].shanten == 0;
        i32 plus = n == 1 ? 3000 : n == 2 ? 1500 : n == 3 ? 1000 : 0;
        i32 minus = n == 1 ? -1000 : n == 2 ? -1500 : n == 3 ? -3000 : 0;
        if (plus > 0)
            for (int j = 0; j < 4; j++) deltas[j] += S->priv[j].shanten == 0 ? plus : minus;
    }
    MJX_L0(if (renchan) S->bflags |= BF_CAN_RENCHAN; else S->bflags &= ~BF_CAN_RENCHAN;
           for (int j = 0; j < 4; j++) S->kyoku_deltas[j] += deltas[j];
           log_push(c, log_word(LOG_RYUKYOKU, 0, 0, T_UNK, 0, 0, 0, 0, 0, 0, 0)); log_push_i32x4(c, deltas));
}

// ---------------------------------------------------------------- board step (board.rs:511-678)
// returns true when the kyoku has ended
MJX_DN bool board_step(Ctx& c) {
    TableState* S = c.S;
    if (S->tiles_left == 70) {
        // haipai: StartKyoku + oya's first draw (board.rs:206-239)
        ev_start_kyoku(c);
        int tile = S->wall[135];
        MJX_L0(log_push(c, log_word(LOG_TSUMO, S->oya, 0, tile, 0, 0, 0, 0, 0, 0, 0)));
        ev_tsumo(c, S->oya, tile);
        return false;
    }
    if (S->accepted_riichis == 4) { MJX_ABORTIVE_RYUKYOKU(c); return true; }

    // pick the winning reaction: Hora 0 < Daiminkan/Pon 1 < other 2 < None 3, lowest seat on ties
    int best = 0, best_p = 4;
    for (int a = 0; a < 4; a++) {
        int ty = c.W->react[a].type;
        int p = ty == R_HORA ? 0 : (ty == R_DAIMINKAN || ty == R_PON) ? 1 : ty == R_NONE ? 3 : 2;
        if (p < best_p) { best_p = p; best = a; }
    }
    const Reaction ev = c.W->react[best];
    MJX_SYNCWARP();

    if ((S->bflags & BF_CHECK_FOUR_KAN) && ev.type != R_HORA) { MJX_ABORTIVE_RYUKYOKU(c); return true; }

    // board.rs:296-312
    if (MJX_IS_L0(c)) {
        if (ev.type == R_DAHAI) { if (!is_yaokyuu(ev.pai)) S->can_nagashi &= (u8)~(1 << ev.actor); }
        else if (ev.type == R_CHI || ev.type == R_PON || ev.type == R_DAIMINKAN) {
            S->can_nagashi &= (u8)~(1 << ev.target);
            S->bflags &= ~BF_CAN_FOUR_WIND;
        } else if (ev.type == R_ANKAN) S->bflags &= ~BF_CAN_FOUR_WIND;
    }
    MJX_SYNCWARP();

    switch (ev.type) {
        case R_NONE: {
            if (S->tiles_left == 0) { exhaustive_ryukyoku(c); return true; }
            check_riichi_accepted(c);
            int tile;
            if (S->bflags & BF_DEAL_FROM_RINSHAN) {
                if (S->n_rinshan >= 4) { set_err(c, ERR_FIFTH_KAN); return true; }
                tile = S->wall[55 - S->n_rinshan];
                MJX_L0(S->bflags &= ~BF_DEAL_FROM_RINSHAN; S->n_rinshan += 1);
            } else {
                int drawn = (70 - S->tiles_left) - S->n_rinshan;
                if (drawn >= 70) { set_err(c, ERR_WALL_EXHAUSTED); return true; }
                tile = S->wall[135 - drawn];
            }
            if (S->bflags & BF_NEW_DORA_AT_TSUMO) {
                // the Tsumo event is built (tiles_left already decremented in the reference) before the dora
                MJX_L0(S->bflags &= ~BF_NEW_DORA_AT_TSUMO);
                ev_dora(c);
            }
            MJX_L0(log_push(c, log_word(LOG_TSUMO, S->tsumo_actor, 0, tile, 0, 0, 0, 0, 0, 0, 0)));
            ev_tsumo(c, S->tsumo_actor, tile);
            break;
        }
        case R_DAHAI: {
            if (S->bflags & BF_NEW_DORA_AT_DISCARD) { MJX_L0(S->bflags &= ~BF_NEW_DORA_AT_DISCARD); ev_dora(c); }
            MJX_L0(log_reaction(c, LOG_DAHAI, ev));
            ev_dahai(c, ev.actor, ev.pai, ev.tsumogiri != 0);
            MJX_L0(S->tsumo_actor = (u8)((ev.actor + 1) & 3));
            // four-wind (board.rs:314-340, 597-600)
            if (S->bflags & BF_CAN_FOUR_WIND) {
                bool abort_now = false;
                const int pai = ev.pai;
                if (!(pai >= T_E && pai <= T_N)) { MJX_L0(S->bflags &= ~BF_CAN_FOUR_WIND); }
                else if (S->priv[S->tsumo_actor].flags & PF_CAN_W_RIICHI) {
                    if (S->four_wind_tile >= 0) { if (S->four_wind_tile != pai) { MJX_L0(S->bflags &= ~BF_CAN_FOUR_WIND); } }
                    else { MJX_L0(S->four_wind_tile = (i8)pai); }
                } else if (S->four_wind_tile >= 0) {
                    if (S->four_wind_tile == pai) abort_now = true;
                    else { MJX_L0(S->bflags &= ~BF_CAN_FOUR_WIND); }
                } else { set_err(c, ERR_FOUR_WIND_STATE); return true; }
                if (abort_now) { MJX_ABORTIVE_RYUKYOKU(c); return true; }
            }
            if (S->kans == 4) {
                bool all_lt4 = true;
                for (int s = 0; s < 4; s++) all_lt4 &= (S->priv[s].n_minkans + S->priv[s].n_ankans) < 4;
                if (all_lt4) { MJX_L0(S->bflags |= BF_CHECK_FOUR_KAN); }
            }
            break;
        }
        case R_CHI:
            check_riichi_accepted(c);
            MJX_L0(log_reaction(c, LOG_CHI, ev));
            ev_chi(c, ev);
            break;
        case R_PON:
            check_riichi_accepted(c);
            MJX_L0(log_reaction(c, LOG_PON, ev));
            ev_pon(c, ev);
            break;
        case R_ANKAN:
            if (S->bflags & BF_NEW_DORA_AT_DISCARD) { MJX_L0(S->bflags &= ~BF_NEW_DORA_AT_DISCARD); ev_dora(c); }
            MJX_L0(log_reaction(c, LOG_ANKAN, ev));
            ev_ankan(c, ev);
            ev_dora(c);
            MJX_L0(S->tsumo_actor = ev.actor; S->bflags |= BF_DEAL_FROM_RINSHAN; S->kans += 1);
            break;
        case R_DAIMINKAN:
        case R_KAKAN:
            if (S->bflags & BF_NEW_DORA_AT_DISCARD) { MJX_L0(S->bflags |= BF_NEW_DORA_AT_TSUMO); }
            check_riichi_accepted(c);
            MJX_L0(log_reaction(c, ev.type == R_DAIMINKAN ? LOG_DAIMINKAN : LOG_KAKAN, ev));
            if (ev.type == R_DAIMINKAN) ev_daiminkan(c, ev); else ev_kakan(c, ev);
            MJX_L0(S->bflags |= BF_NEW_DORA_AT_DISCARD | BF_DEAL_FROM_RINSHAN; S->tsumo_actor = ev.actor; S->kans += 1);
            break;
        case R_REACH:
            MJX_L0(log_push(c, log_word(LOG_REACH, ev.actor, 0, T_UNK, 0, 0, 0, 0, 0, 0, 0)));
            ev_reach(c, ev.actor);
            MJX_L0(S->riichi_to_be_accepted = (i8)ev.actor);
            break;
        case R_HORA:
            handle_hora(c, ev.actor, ev.target);
            return true;
        case R_RYUKYOKU:
            MJX_ABORTIVE_RYUKYOKU(c);
            return true;
        default:
            set_err(c, ERR_INTERNAL);
            return true;
    }

    // pao (board.rs:473-499)
    if ((ev.type == R_PON || ev.type == R_DAIMINKAN) && is_jihai(ev.pai)) {
        const SeatPrivate& P = S->priv[ev.actor];
        u32 jihais = 0;
        for (int i = 0; i < P.n_pons; i++) if (P.pons[i] >= T_E) jihais |= 1u << (P.pons[i] - T_E);
        for (int i = 0; i < P.n_minkans; i++) if (P.minkans[i] >= T_E) jihais |= 1u << (P.minkans[i] - T_E);
        bool daisangen = (jihais & 0x70) == 0x70, daisuushi = (jihais & 0x0F) == 0x0F;
        if ((daisangen && ev.pai >= T_P) || (daisuushi && ev.pai <= T_N)) { MJX_L0(S->paos[ev.actor] = (i8)ev.target); }
    }
    return false;
}

MJX_D bool any_can_act(const TableState* S) {
    return ((S->priv[0].cans | S->priv[1].cans | S->priv[2].cans | S->priv[3].cans) & CAN_ACT) != 0;
}

MJX_D void clear_reactions(Ctx& c) {
    MJX_FOR_SEATS(c, s) {
        Reaction& r = c.W->react[s];
        r.type = R_NONE; r.actor = (u8)s; r.target = 0; r.pai = T_NONE; r.tsumogiri = 0;
        r.consumed[0] = r.consumed[1] = r.consumed[2] = r.consumed[3] = T_NONE;
    }
    MJX_END_SEATS(c);
}

// into_state (board.rs:125-137) + Game::poll kyoku start (game.rs:78-86)
MJX_DN void start_kyoku_board(Ctx& c) {
    TableState* S = c.S;
    if (MJX_IS_L0(c)) {
        if (c.grp) {  // dataset/grp.rs:134-147: [grand_kyoku, honba, kyotaku, scores x 4] at the start of every kyoku
            const int k = *c.grp_n;
            if (k < c.grp_cap) {
                i32* row = c.grp + (size_t)k * 7;
                row[0] = S->kyoku; row[1] = S->honba; row[2] = S->kyotaku;
                for (int i = 0; i < 4; i++) row[3 + i] = S->scores[i];
            }
            *c.grp_n = k + 1;
        }
        make_wall(S->nonce, S->key, S->kyoku, S->honba, S->shuffle_kind, S->wall);
        S->oya = S->kyoku & 3;
        S->bflags = BF_CAN_FOUR_WIND;
        S->tiles_left = 70;
        S->tsumo_actor = 0;
        S->n_dora = 0;
        S->n_rinshan = 0;
        S->riichi_to_be_accepted = -1;
        S->four_wind_tile = -1;
        S->accepted_riichis = 0;
        S->kans = 0;
        S->can_nagashi = 0xF;
        for (int i = 0; i < 4; i++) { S->paos[i] = -1; S->kyoku_deltas[i] = 0; }
        S->gflags |= GF_KYOKU_STARTED;
    }
    MJX_SYNCWARP();
}

// Game::poll (game.rs:59-178): advance until a seat can act or the hanchan has ended.
MJX_DN void game_poll(Ctx& c) {
    TableState* S = c.S;
    for (;;) {
        if (S->gflags & GF_ENDED) return;
        if (S->err != 0) { MJX_L0(S->gflags |= GF_ENDED); return; }
        if (!(S->gflags & GF_KYOKU_STARTED)) {
            const int length = 8;
            bool any30k = false;
            for (int i = 0; i < 4; i++) any30k |= S->scores[i] >= 30000;
            if (S->kyoku >= length + 4 || (S->kyoku >= length && !(S->gflags & GF_IN_RENCHAN) && any30k)) {
                MJX_L0(S->gflags |= GF_ENDED);
                return;
            }
            start_kyoku_board(c);
        }
        // BoardState::poll (board.rs:141-161)
        bool ended = false;
        for (;;) {
            ended = board_step(c);
            if (S->err != 0) { ended = true; break; }
            if (ended) break;
            if (any_can_act(S)) return;
            clear_reactions(c);
        }
        clear_reactions(c);
        if (S->err != 0) { MJX_L0(S->gflags |= GF_ENDED); return; }
        MJX_L0(log_push(c, log_word(LOG_END_KYOKU, 0, 0, T_UNK, 0, 0, 0, 0, 0, 0, 0)));  // board.rs:150-152
        // kyoku end bookkeeping (board.rs:150-157, game.rs:114-174)
        const bool abortive = (S->bflags & BF_HAS_ABORTIVE) != 0;
        const bool can_renchan = abortive || (S->bflags & BF_CAN_RENCHAN);
        const bool has_hora = (S->bflags & BF_HAS_HORA) != 0;
        const int kyoku_now = S->kyoku;
        if (MJX_IS_L0(c)) {
            for (int i = 0; i < 4; i++) S->scores[i] += S->kyoku_deltas[i];
            S->gflags &= (u8)~(GF_KYOKU_STARTED | GF_IN_RENCHAN);
            S->n_kyoku_played += 1;
        }
        MJX_SYNCWARP();
        MJX_FOR_SEATS(c, s) S->priv[s].cans = 0;
        MJX_END_SEATS(c);
        bool tobi = false;
        for (int i = 0; i < 4; i++) tobi |= S->scores[i] < 0;
        if (tobi) { MJX_L0(S->gflags |= GF_ENDED); return; }
        if (abortive) { MJX_L0(S->honba += 1); continue; }
        if (!can_renchan) {
            MJX_L0(S->kyoku += 1; if (has_hora) S->honba = 0; else S->honba += 1);
            continue;
        }
        const int oya = kyoku_now & 3;
        if (kyoku_now >= 8 - 1 && S->scores[oya] >= 30000) {
            int top = 0;
            for (int i = 1; i < 4; i++) if (S->scores[i] > S->scores[top]) top = i;
            if (top == oya) { MJX_L0(S->gflags |= GF_ENDED); return; }
        }
        MJX_L0(S->gflags |= GF_IN_RENCHAN; S->honba += 1);
    }
}

// ---------------------------------------------------------------- agent side (mortal.rs)
// agent_helper.rs:35-79 as a 37-bit mask; all lanes compute it (uniform)
MJX_D u64 discard_candidates(const Ctx& c, int seat) {
    const TableState* S = c.S;
    const SeatPrivate& P = S->priv[seat];
    if ((S->riichi_accepted >> seat) & 1) return 1ull << P.last_self_tsumo;
    u64 present = tile_mask(c, [&](int t) { return P.tehai[t] > 0; });
    u64 m;
    if ((S->riichi_declared >> seat) & 1) m = present & (P.shanten == 1 ? P.next_shanten : P.keep_shanten);
    else m = present & ~P.forbidden;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        int t5 = 4 + 9 * k;
        if (((m >> t5) & 1) && ((P.akas_in_hand >> k) & 1)) {
            m |= 1ull << (34 + k);
            if (!(P.tehai[t5] > 1)) m &= ~(1ull << t5);
        }
    }
    return m;
}

// obs_repr.rs mask writes (423-427, 445-447, 480-559) as a 46-bit mask
MJX_D u64 legal_mask(const Ctx& c, int seat, bool kan_select, u64 discards) {
    const TableState* S = c.S;
    const SeatPrivate& P = S->priv[seat];
    const u16 cans = P.cans;
    u64 m = 0;
    if (cans & CAN_PASS) {
        if (!kan_select) m |= 1ull << 45;
        else if (cans & CAN_DAIMINKAN) m |= 1ull << deaka(S->last_kawa_tile);
    }
    if (!kan_select) {
        if (cans & CAN_DISCARD) m |= discards;
        if (cans & CAN_RIICHI) m |= 1ull << 37;
        if (cans & CAN_CHI_LOW) m |= 1ull << 38;
        if (cans & CAN_CHI_MID) m |= 1ull << 39;
        if (cans & CAN_CHI_HIGH) m |= 1ull << 40;
        if (cans & CAN_PON) m |= 1ull << 41;
        if (cans & CAN_KAN) m |= 1ull << 42;
        if (cans & CAN_AGARI) m |= 1ull << 43;
        if (cans & CAN_RYUKYOKU) m |= 1ull << 44;
    } else {
        if (cans & CAN_ANKAN) m |= P.ankan_cand;
        if (cans & CAN_KAKAN) m |= P.kakan_cand;
    }
    return m;
}

// mortal.rs:338-573. Executed by the lane that owns `seat` (lane == seat) or uniformly.
MJX_DN bool decode_action(const TableState* S, int seat, int action, int kan_action, Reaction& r, i32* err) {
    const SeatPrivate& P = S->priv[seat];
    const u16 cans = P.cans;
    const int akas = P.akas_in_hand;
    r.type = R_NONE; r.actor = (u8)seat; r.target = P.target_actor; r.pai = T_NONE; r.tsumogiri = 0;
    r.consumed[0] = r.consumed[1] = r.consumed[2] = r.consumed[3] = T_NONE;
    auto aka_for = [&](int pai, int a, int b) {
        for (int k = 0; k < 3; k++) if (pai == a + 9 * k || pai == b + 9 * k) return ((akas >> k) & 1) != 0;
        return false;
    };
    if (action >= 0 && action <= 36) {
        if (!(cans & CAN_DISCARD)) { *err = ERR_ILLEGAL_ACTION; return false; }
        r.type = R_DAHAI; r.pai = (u8)action; r.tsumogiri = P.last_self_tsumo == action;
    } else if (action == 37) {
        if (!(cans & CAN_RIICHI)) { *err = ERR_ILLEGAL_ACTION; return false; }
        r.type = R_REACH;
    } else if (action >= 38 && action <= 41) {
        const u16 need = action == 38 ? CAN_CHI_LOW : action == 39 ? CAN_CHI_MID : action == 40 ? CAN_CHI_HIGH : CAN_PON;
        if (!(cans & need)) { *err = ERR_ILLEGAL_ACTION; return false; }
        const int pai = S->last_kawa_tile;
        if (pai == T_NONE) { *err = ERR_NO_KAWA_TILE; return false; }
        r.pai = (u8)pai;
        if (action == 38) {
            int first = tile_next(pai), second = tile_next(first);
            bool ak = aka_for(pai, 2, 3);
            r.type = R_CHI; r.consumed[0] = (u8)(ak ? akaize(first) : first); r.consumed[1] = (u8)(ak ? akaize(second) : second);
        } else if (action == 39) {
            int lo = tile_prev(pai), hi = tile_next(pai);
            bool ak = aka_for(pai, 3, 5);
            r.type = R_CHI; r.consumed[0] = (u8)(ak ? akaize(lo) : lo); r.consumed[1] = (u8)(ak ? akaize(hi) : hi);
        } else if (action == 40) {
            int last = tile_prev(pai), first = tile_prev(last);
            bool ak = aka_for(pai, 5, 6);
            r.type = R_CHI; r.consumed[0] = (u8)(ak ? akaize(first) : first); r.consumed[1] = (u8)(ak ? akaize(last) : last);
        } else {
            bool ak = aka_for(pai, 4, 4);
            r.type = R_PON; r.consumed[0] = (u8)(ak ? akaize(pai) : deaka(pai)); r.consumed[1] = (u8)deaka(pai);
        }
    } else if (action == 42) {
        if (!(cans & CAN_KAN)) { *err = ERR_ILLEGAL_ACTION; return false; }
        int tile;
        if (kan_action >= 0) {
            tile = kan_action;
            if (tile >= 34 || !(((P.ankan_cand | P.kakan_cand) >> tile) & 1)) { *err = ERR_KAN_CHOICE; return false; }
        } else if (cans & CAN_DAIMINKAN) {
            tile = S->last_kawa_tile;
            if (tile == T_NONE) { *err = ERR_NO_KAWA_TILE; return false; }
        } else if (cans & CAN_ANKAN) tile = mjx_ffsll(P.ankan_cand) - 1;
        else tile = mjx_ffsll(P.kakan_cand) - 1;
        if (cans & CAN_DAIMINKAN) {
            r.type = R_DAIMINKAN; r.pai = (u8)tile;
            if (is_aka(tile)) { r.consumed[0] = r.consumed[1] = r.consumed[2] = (u8)deaka(tile); }
            else { r.consumed[0] = (u8)akaize(tile); r.consumed[1] = r.consumed[2] = (u8)tile; }
        } else if ((cans & CAN_ANKAN) && ((P.ankan_cand >> deaka(tile)) & 1)) {
            r.type = R_ANKAN;
            r.consumed[0] = (u8)akaize(tile); r.consumed[1] = r.consumed[2] = r.consumed[3] = (u8)tile;
        } else {
            bool ak = aka_for(tile, 4, 4);
            r.type = R_KAKAN;
            int d = deaka(tile);
            if (ak) { r.pai = (u8)akaize(tile); r.consumed[0] = r.consumed[1] = r.consumed[2] = (u8)d; }
            else { r.pai = (u8)d; r.consumed[0] = (u8)akaize(tile); r.consumed[1] = r.consumed[2] = (u8)d; }
        }
    } else if (action == 43) {
        if (!(cans & CAN_AGARI)) { *err = ERR_ILLEGAL_ACTION; return false; }
        r.type = R_HORA;
    } else if (action == 44) {
        if (!(cans & CAN_RYUKYOKU)) { *err = ERR_ILLEGAL_ACTION; return false; }
        r.type = R_RYUKYOKU;
    } else if (action == 45) {
        r.type = R_NONE;
    } else {
        *err = ERR_ILLEGAL_ACTION;
        return false;
    }
    return true;
}

// a decoded reaction as an event word (log_word; type 0 = none): what libriichi.state.reaction_from_word reads back
MJX_D u64 reaction_word(const Reaction& r) {
    const int ty = r.type == R_DAHAI ? LOG_DAHAI : r.type == R_CHI ? LOG_CHI : r.type == R_PON ? LOG_PON :
                   r.type == R_DAIMINKAN ? LOG_DAIMINKAN : r.type == R_KAKAN ? LOG_KAKAN : r.type == R_ANKAN ? LOG_ANKAN :
                   r.type == R_REACH ? LOG_REACH : r.type == R_HORA ? LOG_HORA : r.type == R_RYUKYOKU ? LOG_RYUKYOKU : 0;
    return log_word(ty, r.actor, r.target, r.pai, r.tsumogiri, 0, r.consumed[0], r.consumed[1], r.consumed[2], r.consumed[3], 0);
}

// ================================================================ table step (commit + poll + emit)
// Device-resident buffers of one environment. Plain pointers only: this struct is also what
// include/mjx.h hands out piecewise through the C ABI.
struct EnvView {
    TableState* tables;
    i32 n_tables;
    i32 row_cap;
    i32* n_rows;        // [1] rows emitted by the current step
    i32* row_table;     // [row_cap]
    u8* row_seat;       // [row_cap] seat | kan_select << 2
    u32* row_step;      // [row_cap] table-step index (policy hashing / tracing)
    u8* masks;          // [row_cap, 46] legal-action mask, 1 byte per action (torch.bool compatible)
    const i64* actions; // [row_cap] chosen action per row of the PREVIOUS step
    const float* q_values;   // [row_cap, 46] or null: needed only by the rule-based agari guard (mortal.rs:319-336)
    const u8* agari_guard;   // [n_tables, 4] or null: 1 where the seat's engine has enable_rule_based_agari_guard
    i32* scores;        // [n_tables, 4] final scores (valid once done)
    u8* ranks;          // [n_tables, 4] rank_by_player (rankings.rs:8-22)
    i32* done;          // [n_tables]
    i32* steps;         // [n_tables] table-steps taken (game.rs:304 `actions`)
    i32* err;           // [n_tables]
    unsigned long long* counters;  // [0] live tables after this step, [1] total table-steps so far
    i32 enable_quick_eval;
    const u8* quick_eval_seat;  // [n_tables, 4] or null: per-seat enable_quick_eval (agent/mortal.rs:54-74: every agent has its own)
    u64* log;           // [n_tables, log_cap] mjai event words (see log_word) or null
    i32* log_len;       // [n_tables] words written (may exceed log_cap: overflow)
    i32 log_cap;
    i32* grp;           // [n_tables, grp_cap, 7] GRP feature rows (dataset/grp.rs:134-147) or null
    i32* grp_len;       // [n_tables] kyoku started so far
    i32 grp_cap;
};

MJX_D int alloc_rows(Ctx& c, EnvView& V, int n) {
#ifdef MJX_HOST_EMUL
    int base = *V.n_rows;
    *V.n_rows += n;
    return base;
#else
    int base = 0;
    if (c.lane == 0) base = atomicAdd(V.n_rows, n);
    return __shfl_sync(0xFFFFFFFFu, base, 0);
#endif
}

MJX_D void write_mask_row(Ctx& c, EnvView& V, int row, u64 m) {
#ifdef MJX_HOST_EMUL
    for (int i = 0; i < ACTION_SPACE; i++) V.masks[(size_t)row * ACTION_SPACE + i] = (u8)((m >> i) & 1);
#else
    for (int i = c.lane; i < ACTION_SPACE; i += 32) V.masks[(size_t)row * ACTION_SPACE + i] = (u8)((m >> i) & 1);
#endif
}

// Game::commit (game.rs:200-217) through MortalBatchAgent::get_reaction (mortal.rs:292-573):
// turn last step's chosen actions into the four reactions.
MJX_DN void gather_reactions(Ctx& c, EnvView& V, int table) {
    TableState* S = c.S;
    clear_reactions(c);
    // The mask rows written last step may already be overwritten by other tables of this launch, so
    // legality (board.rs:524-533 validate_reaction) is re-derived from the table state itself.
    for (int s = 0; s < 4; s++) {
        if (S->row_of_seat[s] < 0) continue;
        const u64 discards = (S->priv[s].cans & CAN_DISCARD) ? discard_candidates(c, s) : 0;
        const u64 lm = legal_mask(c, s, false, discards), km = legal_mask(c, s, true, discards);
        MJX_L0(c.W->legal[s] = lm; c.W->legal_kan[s] = km);
    }
    MJX_FOR_SEATS(c, s) {
        int action = -1, kan_action = -1;
        i32 e = 0;
        if (S->auto_action[s] >= 0) {
            action = S->auto_action[s];
        } else if (S->row_of_seat[s] >= 0) {
            i64 a = V.actions[S->row_of_seat[s]];
            if (a < 0 || a >= ACTION_SPACE || !((c.W->legal[s] >> a) & 1)) e = ERR_ILLEGAL_ACTION;
            else action = (int)a;
            // mortal.rs:319-336: the engine wants agari but the rule-based guard objects -> best other Q
            if (e == 0 && action == 43 && V.agari_guard && V.agari_guard[table * 4 + s] && !rule_based_agari(c, s)) {
                if (!V.q_values) e = ERR_GUARD_NEEDS_Q;
                else {
                    const float* q = V.q_values + (size_t)S->row_of_seat[s] * ACTION_SPACE;
                    int best = -1;
                    float bq = 0.f;
                    for (int i = 0; i < ACTION_SPACE; i++) {
                        const float v = i == 43 ? -3.40282347e+38f : q[i];
                        if (best < 0 || !(v < bq)) { best = i; bq = v; }  // max_by(total_cmp): last maximum
                    }
                    if (!((c.W->legal[s] >> best) & 1)) e = ERR_ILLEGAL_ACTION;
                    else action = best;
                }
            }
            if (S->kan_row_of_seat[s] >= 0) {
                i64 k = V.actions[S->kan_row_of_seat[s]];
                if (k < 0 || k >= ACTION_SPACE || !((c.W->legal_kan[s] >> k) & 1)) e = ERR_ILLEGAL_ACTION;
                else kan_action = (int)k;
            }
        }
        if (e == 0 && action >= 0) {
            Reaction r;
            if (decode_action(S, s, action, action == 42 ? kan_action : -1, r, &e)) c.W->react[s] = r;
        }
        if (e != 0) atomic_set_err(S, e);
        S->auto_action[s] = -1;
        S->row_of_seat[s] = -1;
        S->kan_row_of_seat[s] = -1;
    }
    MJX_END_SEATS(c);
}

// Game::poll tail (game.rs:93-112) + MortalBatchAgent::set_scene (mortal.rs:200-290):
// hand every acting seat to the policy as one (or, with kan-select, two) rows.
MJX_DN void emit_decisions(Ctx& c, EnvView& V, int table) {
    TableState* S = c.S;
    for (int s = 0; s < 4; s++) {
        const SeatPrivate& P = S->priv[s];
        const u16 cans = P.cans;
        if (!(cans & CAN_ACT)) continue;
        const u64 discards = (cans & CAN_DISCARD) ? discard_candidates(c, s) : 0;
        const bool quick_eval = V.quick_eval_seat ? V.quick_eval_seat[table * 4 + s] != 0 : V.enable_quick_eval != 0;
        if (quick_eval && (cans & CAN_DISCARD) &&
            !(cans & (CAN_RIICHI | CAN_TSUMO_AGARI | CAN_ANKAN | CAN_KAKAN | CAN_RYUKYOKU)) && mjx_popcll(discards) == 1) {
            MJX_L0(S->auto_action[s] = (i8)(mjx_ffsll(discards) - 1));
            continue;
        }
        bool need_kan = false;
        if (cans & (CAN_ANKAN | CAN_KAKAN))
            need_kan = !quick_eval || (mjx_popcll(P.ankan_cand) + mjx_popcll(P.kakan_cand)) > 1;
        const int n = need_kan ? 2 : 1;
        const int base = alloc_rows(c, V, n);
        if (base + n > V.row_cap) { set_err(c, ERR_ROW_OVERFLOW); return; }
        int row = base;
        if (need_kan) {
            write_mask_row(c, V, row, legal_mask(c, s, true, discards));
            MJX_L0(V.row_table[row] = table; V.row_seat[row] = (u8)(s | 4); V.row_step[row] = S->step_idx;
                   S->kan_row_of_seat[s] = row);
            row += 1;
        }
        write_mask_row(c, V, row, legal_mask(c, s, false, discards));
        MJX_L0(V.row_table[row] = table; V.row_seat[row] = (u8)s; V.row_step[row] = S->step_idx; S->row_of_seat[s] = row);
    }
}

// One table-step of BatchGame::run (game.rs:286-304) for the table in c.S.
// Returns true while the table is still live afterwards.
MJX_DN bool step_table(Ctx& c, EnvView& V, int table) {
    TableState* S = c.S;
    if (!(S->gflags & GF_ALIVE)) return false;
    recompute_dora_factor(c);
    if (S->gflags & GF_KYOKU_STARTED) {
        gather_reactions(c, V, table);
        MJX_L0(S->step_idx += 1);
    } else {
        clear_reactions(c);
    }
    if (S->err == 0) game_poll(c);
    if (S->err != 0) { MJX_L0(S->gflags |= GF_ENDED); }
    if (S->gflags & GF_ENDED) {
        // Game::commit end branch (game.rs:181-198): leftover sticks to the first top seat, rankings
        if (MJX_IS_L0(c)) {
            if (S->kyotaku > 0) {
                int top = 0;
                for (int i = 1; i < 4; i++) if (S->scores[i] > S->scores[top]) top = i;
                S->scores[top] += (i32)S->kyotaku * 1000;
            }
            u8 order[4] = {0, 1, 2, 3};
            for (int i = 1; i < 4; i++)  // stable insertion sort by descending score
                for (int j = i; j > 0 && S->scores[order[j]] > S->scores[order[j - 1]]; j--) {
                    u8 t = order[j]; order[j] = order[j - 1]; order[j - 1] = t;
                }
            for (int r = 0; r < 4; r++) V.ranks[table * 4 + order[r]] = (u8)r;
            for (int i = 0; i < 4; i++) V.scores[table * 4 + i] = S->scores[i];
            V.done[table] = 1;
            V.err[table] = S->err;
            S->gflags &= (u8)~GF_ALIVE;
        }
        MJX_SYNCWARP();
        return false;
    }
    emit_decisions(c, V, table);
    if (S->err != 0) {
        MJX_L0(V.err[table] = S->err; V.done[table] = 1; S->gflags = (u8)((S->gflags | GF_ENDED) & ~GF_ALIVE));
        return false;
    }
    MJX_L0(V.steps[table] += 1);
    return true;
}

}  // namespace mjx
