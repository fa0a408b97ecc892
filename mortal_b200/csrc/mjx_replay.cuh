// mortal_b200 — log replay: the dataset side of libriichi (dataset/gameplay.rs:247-449 GameplayLoader), SURVEY.md §8f N3.
//
// A "job" = one (game log, player) pair. The log is a sequence of the same 64-bit event words k_step records
// (csrc/mjx_step.cuh log_word; start_kyoku payloads in a side array). One warp replays one job through the very event
// handlers self-play uses (the record holds all four seats for full-information logs as Mortal's arena or tenhou
// conversions produce them; after k_replay_viewpoints, a log that hides the other seats' tiles, as the mjai protocol shows a
// game to one seat, is replayed from the player's own PlayerState), stops whenever the log shows the player making a decision, emits the decision row(s)
// with the label the following events imply (gameplay.rs:303-423) and lets the ordinary encoder kernels produce the
// observation before the next call continues.
#pragma once
#include "mjx_step.cuh"

namespace mjx {

enum : u8 { LOG_START_GAME = 15, LOG_END_GAME = 16 };
constexpr int REPLAY_KYOKU_WORDS = 19;  // start_kyoku payload: 2 score words + the 136-byte wall (unknown tiles = T_UNK)

struct ReplayView {
    const u64* hdr;     // event words of all jobs, concatenated (one word per event)
    const i32* ev_off;  // [n_jobs] first event of the job
    const i32* ev_cnt;  // [n_jobs] number of events
    const u64* kyoku;   // start_kyoku payloads, REPLAY_KYOKU_WORDS each (2 score words + 17 wall words), concatenated
    const i32* ky_off;  // [n_jobs] first payload (in units of REPLAY_KYOKU_WORDS) of the job
    i32* pos;           // [n_jobs] next event window to process
    i32* ky_idx;        // [n_jobs] end_kyoku events seen (gameplay.rs kyoku_idx)
    i32* ky_seen;       // [n_jobs] start_kyoku events applied (payload cursor)
    const u8* player;   // [n_jobs] point of view
    i64* row_label;     // [row_cap] action label of each emitted row
    u8* row_meta;       // [row_cap, 4] at_kyoku, at_turn, shanten (as i8), apply_gamma
    i32 always_include_kan_select;
    i32 trust_seed;     // the jobs carry their game's seed (TableState.nonce / key): regenerate every kyoku's wall from it
                        // (dataset/invisible.rs:35-66), which the invisible observation needs; else hidden tiles stay unknown
    i32 review;         // review mode (mjx_env_replay_review, csrc/mjx_review.cuh): every event is applied and the job stops
                        // wherever its seat can act, as mjai.Bot with quick eval off decides; labels where the log shows one
};

MJX_D int lw_type(u64 w) { return (int)(w & 0xFF); }
MJX_D int lw_actor(u64 w) { return (int)((w >> 8) & 3); }
MJX_D int lw_target(u64 w) { return (int)((w >> 10) & 3); }
MJX_D int lw_pai(u64 w) { return (int)((w >> 12) & 0xFF); }
MJX_D int lw_c(u64 w, int k) { return (int)((w >> (24 + 8 * k)) & 0xFF); }

MJX_D Reaction lw_reaction(u64 w, int type) {
    Reaction r;
    r.type = (u8)type; r.actor = (u8)lw_actor(w); r.target = (u8)lw_target(w); r.pai = (u8)lw_pai(w);
    r.tsumogiri = (u8)((w >> 20) & 1);
    for (int k = 0; k < 4; k++) r.consumed[k] = (u8)lw_c(w, k);
    r.pad_[0] = r.pad_[1] = r.pad_[2] = 0;
    return r;
}

// PlayerState::update (state/update.rs:24-122) driven by one event word — for all four seats of a full-information record, or
// for the single known seat of a PlayerState record (TableState.viewer1). `pay` = the start_kyoku payload (only read for that event).
// KEEP_CANS = update_with_keep_cans(ev, true) (see ev_prologue).
template <bool KEEP_CANS = false>
MJX_DN void apply_event(Ctx& c, u64 w, const u64* pay, bool trust_seed) {
    TableState* S = c.S;
    switch (lw_type(w)) {
        case LOG_START_KYOKU: {
            if (MJX_IS_L0(c)) {
                S->kyoku = (u8)lw_c(w, 0); S->honba = (u8)lw_c(w, 1); S->kyotaku = (u8)lw_c(w, 2); S->oya = (u8)lw_c(w, 3);
                S->scores[0] = (i32)(u32)pay[0]; S->scores[1] = (i32)(u32)(pay[0] >> 32);
                S->scores[2] = (i32)(u32)pay[1]; S->scores[3] = (i32)(u32)(pay[1] >> 32);
                // the wall as far as the caller knows it (haipai always; the hidden tiles when an invisible observation is wanted)
                for (int i = 0; i < 136; i++) S->wall[i] = (u8)((pay[2 + i / 8] >> (8 * (i % 8))) & 0xFF);
                if (trust_seed) {
                    u8 hp[52];
                    for (int i = 0; i < 52; i++) hp[i] = S->wall[i];
                    make_wall(S->nonce, S->key, S->kyoku, S->honba, S->shuffle_kind, S->wall);
                    for (int i = 0; i < 52; i++) if (S->wall[i] != hp[i] && S->err == 0) S->err = ERR_SEED_MISMATCH;  // not dealt from this seed
                }
                if (trust_seed && S->wall[60] != (u8)lw_pai(w) && S->err == 0) S->err = ERR_SEED_MISMATCH;
                S->wall[60] = (u8)lw_pai(w);  // the first dora indicator; later ones arrive with their dora events
                S->bflags = 0;
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
            ev_start_kyoku(c);
            break;
        }
        case LOG_TSUMO:
            // dataset/gameplay.rs:315-322: a draw after a kan comes from the rinshan (the invisible observation counts them)
            MJX_L0(if (S->bflags & BF_DEAL_FROM_RINSHAN) { S->n_rinshan += 1; S->bflags &= (u16)~BF_DEAL_FROM_RINSHAN; });
            ev_tsumo(c, lw_actor(w), lw_pai(w));
            break;
        case LOG_DAHAI: ev_dahai(c, lw_actor(w), lw_pai(w), ((w >> 20) & 1) != 0); break;
        case LOG_CHI: ev_chi(c, lw_reaction(w, R_CHI)); break;
        case LOG_PON: ev_pon(c, lw_reaction(w, R_PON)); break;
        case LOG_DAIMINKAN: ev_daiminkan(c, lw_reaction(w, R_DAIMINKAN)); MJX_L0(S->kans += 1; S->bflags |= BF_DEAL_FROM_RINSHAN); break;
        case LOG_KAKAN: ev_kakan(c, lw_reaction(w, R_KAKAN)); MJX_L0(S->kans += 1; S->bflags |= BF_DEAL_FROM_RINSHAN); break;
        case LOG_ANKAN: ev_ankan(c, lw_reaction(w, R_ANKAN)); MJX_L0(S->kans += 1; S->bflags |= BF_DEAL_FROM_RINSHAN); break;
        case LOG_DORA:
            MJX_L0(if (S->n_dora < 5) S->wall[60 - S->n_dora] = (u8)lw_pai(w));
            ev_dora<KEEP_CANS>(c);
            break;
        case LOG_REACH: ev_reach(c, lw_actor(w)); break;
        case LOG_REACH_ACCEPTED:
            MJX_L0(S->riichi_to_be_accepted = (i8)lw_actor(w));
            check_riichi_accepted<KEEP_CANS>(c);
            break;
        default:  // start_game, hora, ryukyoku, end_kyoku, end_game: only the common prologue (update.rs:46-61)
            if (KEEP_CANS && lw_type(w) == LOG_HORA) ev_prologue<true>(c, -1);
            else ev_prologue(c, -1);
            break;
    }
}

MJX_DN void replay_apply(Ctx& c, const ReplayView& R, int job, u64 w) {
    const u64* pay = nullptr;
    if (lw_type(w) == LOG_START_KYOKU) {
        const int seen = R.ky_seen[job];
        MJX_SYNCWARP();  // every lane has read the cursor before lane 0 advances it
        pay = R.kyoku + ((size_t)R.ky_off[job] + seen) * REPLAY_KYOKU_WORDS;
        MJX_L0(R.ky_seen[job] = seen + 1);
    }
    apply_event(c, w, pay, R.trust_seed != 0);
}

// Single-viewpoint logs (k_replay_viewpoints, mjx_env_replay_viewpoints): the seats job `job`'s log hides, bit s when one of
// seat s's 13 haipai bytes in a start_kyoku payload, or the pai of one of its tsumo words, is `?` (what an mjai client is shown
// of the other seats). -1 = leave the job as it is: its events lie outside [0, n_hdr), or it has more start_kyoku words than
// payloads are left in [ky_off, n_kyoku) (n_kyoku counts payloads). Device: the warp loads the words 32 at a time (coalesced),
// one per lane; a ballot prefix gives each start_kyoku lane its payload, whose haipai words (2..8) it reads. The result is
// warp-uniform. -DMJX_HOST_EMUL walks the words on one lane.
MJX_D unsigned hidden_seats_of_word(const ReplayView& R, u64 w, long long k, long long n_kyoku, bool& over) {
    if (lw_type(w) == LOG_TSUMO) return lw_pai(w) == T_UNK ? 1u << lw_actor(w) : 0u;
    if (lw_type(w) != LOG_START_KYOKU) return 0u;
    if (k < 0 || k >= n_kyoku) { over = true; return 0u; }
    const u64* hp = R.kyoku + k * REPLAY_KYOKU_WORDS + 2;
    unsigned m = 0;
    for (int i = 0; i < 52; i++)
        if (((hp[i / 8] >> (8 * (i % 8))) & 0xFF) == T_UNK) m |= 1u << (i / 13);
    return m;
}

MJX_DM int replay_hidden_seats(const ReplayView& R, int job, long long n_hdr, long long n_kyoku, int lane) {
    const long long off = R.ev_off[job], cnt = R.ev_cnt[job];
    if (off < 0 || cnt < 0 || off + cnt > n_hdr) return -1;
    long long ky = R.ky_off[job];  // the next start_kyoku's payload
    unsigned mask = 0;
    bool over = false;
    for (long long base = 0; base < cnt; base += 32) {
        const int n = cnt - base < 32 ? (int)(cnt - base) : 32;
#ifdef MJX_HOST_EMUL
        (void)lane;
        for (int j = 0; j < n; j++) {
            const u64 w = R.hdr[off + base + j];
            mask |= hidden_seats_of_word(R, w, ky, n_kyoku, over);
            ky += lw_type(w) == LOG_START_KYOKU;
        }
#else
        const u64 w = lane < n ? R.hdr[off + base + lane] : 0;  // type 0: no event
        const unsigned sk = __ballot_sync(~0u, lw_type(w) == LOG_START_KYOKU);
        mask |= hidden_seats_of_word(R, w, ky + __popc(sk & ((1u << lane) - 1)), n_kyoku, over);
        ky += __popc(sk);
#endif
    }
#ifndef MJX_HOST_EMUL
    mask = __reduce_or_sync(~0u, mask);
    over = __any_sync(~0u, over);
#endif
    return over ? -1 : (int)mask;
}

// The job's record after the scan: a log that hides a seat is replayed from the player's own PlayerState (viewer1 = player + 1;
// dataset/gameplay.rs:240-335 with oracle = false runs only that state), and fails at once with ERR_HIDDEN_OWN_TILE when it hides
// the player's own tiles. A full-information log (mask 0) is left untouched unless `every_log` (review mode: the Bot's state is a
// PlayerState whatever the log shows); an unmarked job (-1) always is.
MJX_D void replay_mark_viewpoint(TableState* S, int player, int mask, bool every_log = false) {
    if (mask < 0 || (mask == 0 && !every_log) || player > 3) return;
    S->viewer1 = (u8)(player + 1);
    if (((mask >> player) & 1) && S->err == 0) S->err = ERR_HIDDEN_OWN_TILE;
}

// Advance one job to its next logged decision (review mode: to its seat's next event with CAN_ACT). Returns true while the job
// still has events to process.
MJX_DN bool replay_table(Ctx& c, EnvView& V, const ReplayView& R, int job) {
    TableState* S = c.S;
    if (!(S->gflags & GF_ALIVE)) return false;
    recompute_dora_factor(c);
    const int n = R.ev_cnt[job], p = R.player[job];
    const u64* ev = R.hdr + R.ev_off[job];
    const int end = R.review ? n : n - 3;  // gameplay.rs:279-283: windows of four events (w + 4 <= n); review: every event
    int w = R.pos[job];
    for (; w < end; w++) {
        const u64 cur = ev[w];
        if (lw_type(cur) == LOG_END_KYOKU) { MJX_L0(R.ky_idx[job] += 1); }
        replay_apply(c, R, job, cur);
        MJX_SYNCWARP();
        if (S->err != 0) break;
        const SeatPrivate& P = S->priv[p];
        const u16 cans = P.cans;
        if (!(cans & CAN_ACT)) continue;
        // the look-ahead stops at the end of the log (type 0 = no event); inside the four-event window it never reaches it
        const int t1 = w + 1 < n ? lw_type(ev[w + 1]) : 0;
        const int wn = (t1 == LOG_REACH_ACCEPTED || t1 == LOG_DORA) ? w + 2 : w + 1;
        const u64 next = wn < n ? ev[wn] : 0;
        const int tn = lw_type(next);
        const bool kan_always = R.always_include_kan_select || R.review;
        int label = -1, kan_select = -1;
        bool catch_all = false;
        switch (tn) {  // gameplay.rs:349-421
            case LOG_DAHAI: label = lw_pai(next); break;
            case LOG_REACH: label = 37; break;
            case LOG_CHI:
                if (lw_actor(next) == p) {
                    const int a = deaka(lw_c(next, 0)), b = deaka(lw_c(next, 1)), t = deaka(lw_pai(next));
                    label = t < min(a, b) ? 38 : (t < max(a, b) ? 39 : 40);  // chi_type.rs:10-25
                } else catch_all = true;
                break;
            case LOG_PON: if (lw_actor(next) == p) label = 41; else catch_all = true; break;
            case LOG_DAIMINKAN:
                if (lw_actor(next) == p) { if (R.always_include_kan_select) kan_select = deaka(lw_pai(next)); label = 42; }
                else catch_all = true;
                break;
            case LOG_KAKAN:
                if (kan_always || mjx_popcll(P.kakan_cand) > 1) kan_select = deaka(lw_pai(next));
                label = 42;
                break;
            case LOG_ANKAN:
                if (kan_always || mjx_popcll(P.ankan_cand) > 1) kan_select = deaka(lw_c(next, 0));
                label = 42;
                break;
            case LOG_RYUKYOKU: if (cans & CAN_RYUKYOKU) label = 44; else catch_all = true; break;
            default: catch_all = true; break;
        }
        if (catch_all) {
            const bool has_any_ron = t1 == LOG_HORA;
            if (has_any_ron)
                for (int k = w + 1; k < w + 4 && k < n; k++) {
                    const int tk = lw_type(ev[k]);
                    if (tk == LOG_END_KYOKU) break;
                    if (tk == LOG_HORA && lw_actor(ev[k]) == p) { label = 43; break; }
                }
            if (label < 0) {
                const bool can_chi = (cans & (CAN_CHI_LOW | CAN_CHI_MID | CAN_CHI_HIGH)) != 0;
                if ((can_chi && tn == LOG_TSUMO) || ((cans & (CAN_PON | CAN_DAIMINKAN | CAN_RON_AGARI)) && !has_any_ron)) label = 45;
            }
        }
        if (label < 0 && !R.review) continue;
        // gameplay.rs:425-447 add_entry: the decision row, then the kan-select row; review mode: the kan-select row whenever an
        // ankan or kakan is possible (agent/mortal.rs set_scene with quick eval off), labelled only when the log shows the kan
        const bool kan_row = R.review ? (cans & (CAN_ANKAN | CAN_KAKAN)) != 0 : kan_select >= 0;
        const int n_rows = kan_row ? 2 : 1;
        const int base = alloc_rows(c, V, n_rows);
        if (base + n_rows > V.row_cap) { set_err(c, ERR_ROW_OVERFLOW); break; }
        const u64 discards = (cans & CAN_DISCARD) ? discard_candidates(c, p) : 0;
        for (int k = 0; k < n_rows; k++) {
            const int row = base + k;
            write_mask_row(c, V, row, legal_mask(c, p, k == 1, discards));
            const int lab = k == 0 ? label : kan_select;
            MJX_L0(V.row_table[row] = job; V.row_seat[row] = (u8)(p | (k << 2)); V.row_step[row] = (u32)w;
                   R.row_label[row] = lab;
                   R.row_meta[row * 4 + 0] = (u8)R.ky_idx[job]; R.row_meta[row * 4 + 1] = P.at_turn;
                   R.row_meta[row * 4 + 2] = (u8)P.shanten; R.row_meta[row * 4 + 3] = (u8)(lab <= 37 ? 1 : 0));
        }
        MJX_L0(R.pos[job] = w + 1);
        MJX_SYNCWARP();
        return true;
    }
    // review mode: steps = the event the job stopped at (the failing one, or n)
    MJX_L0(R.pos[job] = n; S->gflags &= (u8)~GF_ALIVE; V.done[job] = 1; V.err[job] = S->err; if (R.review) V.steps[job] = w);
    MJX_SYNCWARP();
    return false;
}

}  // namespace mjx
