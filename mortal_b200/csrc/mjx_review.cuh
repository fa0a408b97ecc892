// mortal_b200 — review of mjai logs (mortal.py with MORTAL_REVIEW_MODE=1): the reaction the Bot sends at every decision of a
// replay in review mode (csrc/mjx_replay.cuh ReplayView.review), and the review text, one line per event of the log.
//
// Records: one per evaluated row, in the layout of mjx_mjai_write.cuh's MwView records, so that its meta writer renders them:
//   info [.., 4]  action (the main row's after the agari guard, the kan-select row's as the engine chose it), MJX_MW_REC_* flags
//                 (greedy, shanten, furiten), shanten, label (the action the log shows next, or -1)
//   mask [..]     the 46 legal-action bits; q [.., 46] the engine's Q-values; i64s [.., 2] batch_size (rows of the decision),
//                 eval_time_ns (the host writes it after the engine call)
//   word [..]     the reaction as an event word (csrc/mjx_step.cuh log_word; 0 on kan-select rows; type 0 = `none`)
// Device: k_review_react runs one warp per decision row, k_review_render<FILL> one warp per job, one lane per event line.
// -DMJX_HOST_EMUL builds the same code for one host lane (tests/host_emul/emul_review.cc).
#pragma once
#include "mjx_replay.cuh"
#include "mjx_mjai_write.cuh"

namespace mjx {

struct ReviewOut {
    i32* info;
    u64* mask;
    float* q;
    i64* i64s;
    u64* word;
};

// agent/mortal.rs:292-592 get_reaction for the decision whose main row is `row` (kan-select row: row + 1) of job `job`, with the
// table record still at the decision. Lane 0 decides; every lane copies Q-values. A decode failure fails the job (its record's
// err, done, not alive) and leaves word 0.
MJX_DN void review_react_row(Ctx& c, EnvView& V, const ReplayView& R, int row, int n_rows, const i64* actions, const float* q,
                             const u8* greedy, bool guard, const ReviewOut& O) {
    const int job = V.row_table[row], p = V.row_seat[row] & 3;
    const int kr = row + 1 < n_rows && V.row_table[row + 1] == job && (V.row_seat[row + 1] & 4) ? row + 1 : -1;
    const int rows = kr >= 0 ? 2 : 1;
    TableState* S = c.S;
    const SeatPrivate& P = S->priv[p];
    for (int k = 0; k < rows; k++) {
        const int r = row + k;
#ifdef MJX_HOST_EMUL
        for (int a = 0; a < ACTION_SPACE; a++) O.q[(size_t)r * ACTION_SPACE + a] = q[(size_t)r * ACTION_SPACE + a];
#else
        for (int a = c.lane; a < ACTION_SPACE; a += 32) O.q[(size_t)r * ACTION_SPACE + a] = q[(size_t)r * ACTION_SPACE + a];
#endif
    }
    if (MJX_IS_L0(c)) {
        int action = (int)actions[row];
        if (guard && action == 43 && !rule_based_agari(c, p)) {  // mortal.rs:319-336: the last maximum with q[43] = f32::MIN
            const float* qr = q + (size_t)row * ACTION_SPACE;
            int best = 0;
            for (int i = 0; i < ACTION_SPACE; i++) {
                const float v = i == 43 ? -3.40282347e+38f : qr[i];
                const float b = best == 43 ? -3.40282347e+38f : qr[best];
                if (!(v < b)) best = i;
            }
            action = best;
        }
        const int kan_action = kr >= 0 ? (int)actions[kr] : -1;
        Reaction rc;
        i32 err = 0;
        u64 w = 0;
        if (decode_action(S, p, action, action == 42 ? kan_action : -1, rc, &err)) {
            w = reaction_word(rc);
        } else {
            if (!err) err = ERR_ILLEGAL_ACTION;
            S->err = err;
            S->gflags &= (u8)~GF_ALIVE;
            V.done[job] = 1;
            V.err[job] = err;
            V.steps[job] = (i32)V.row_step[row];
        }
        const int flags = MJX_MW_REC_HAS_SHANTEN | MJX_MW_REC_HAS_FURITEN | ((P.flags & PF_AT_FURITEN) ? MJX_MW_REC_FURITEN : 0);
        for (int k = 0; k < rows; k++) {
            const int r = row + k;
            u64 m = 0;
            for (int a = 0; a < ACTION_SPACE; a++) m |= (u64)(V.masks[(size_t)r * ACTION_SPACE + a] != 0) << a;
            O.info[r * 4 + 0] = k == 0 ? action : kan_action;
            O.info[r * 4 + 1] = flags | (greedy[r] ? MJX_MW_REC_GREEDY : 0);
            O.info[r * 4 + 2] = P.shanten;
            O.info[r * 4 + 3] = (i32)R.row_label[r];
            O.mask[r] = m;
            O.i64s[r * 2 + 0] = rows;
            O.i64s[r * 2 + 1] = 0;
            O.word[r] = k == 0 ? w : 0;
        }
    }
    MJX_SYNCWARP();
}

// ---------------------------------------------------------------- review text
struct RvView {
    const i32* ev_cnt;     // [n_jobs] events (= lines) of the job's log
    const i64* rec_off;    // [n_jobs + 1] the job's records, in event order (a decision's main row before its kan-select row)
    const i32* rec_event;  // [n_rec] event index of the record's decision
    const u8* rec_kan;     // [n_rec] 1 on kan-select rows
    const u64* rec_word;   // [n_rec]
    MwView M;              // rec_info / rec_mask / rec_q / rec_i64 of the records (the rest unused)
    const u8* skip;        // [n_jobs] 1: no text (the job failed)
    int n_jobs;
    i64* bytes;            // count pass: [n_jobs]
    const i64* off;        // fill pass: job j's text at out + off[j]
    char* out;
    long long out_cap;
};

// the main record of event e of job j, or -1
MJX_D long long rv_find(const RvView& V, int j, int e) {
    long long lo = V.rec_off[j], hi = V.rec_off[j + 1];
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (V.rec_event[mid] < e) lo = mid + 1;
        else hi = mid;
    }
    return lo < V.rec_off[j + 1] && V.rec_event[lo] == e && !V.rec_kan[lo] ? lo : -1;
}

// json.dumps(reaction, separators=(",", ":")) of libriichi.state.reaction_from_word, without the closing brace
MJX_DN void rv_reaction(MwOut& o, u64 x) {
    const int ty = (int)(x & 0xFF), actor = (int)(x >> 8) & 3, target = (int)(x >> 10) & 3, pai = (int)(x >> 12) & 0xFF;
    int c[4];
    for (int k = 0; k < 4; k++) c[k] = (int)(x >> (24 + 8 * k)) & 0xFF;
    const int nc = ty == LOG_CHI || ty == LOG_PON ? 2 : ty == LOG_DAIMINKAN || ty == LOG_KAKAN ? 3 : ty == LOG_ANKAN ? 4 : 0;
    switch (ty) {
        case LOG_DAHAI: o.puts("{\"type\":\"dahai\""); break;
        case LOG_REACH: o.puts("{\"type\":\"reach\""); break;
        case LOG_CHI: o.puts("{\"type\":\"chi\""); break;
        case LOG_PON: o.puts("{\"type\":\"pon\""); break;
        case LOG_DAIMINKAN: o.puts("{\"type\":\"daiminkan\""); break;
        case LOG_KAKAN: o.puts("{\"type\":\"kakan\""); break;
        case LOG_ANKAN: o.puts("{\"type\":\"ankan\""); break;
        case LOG_HORA: o.puts("{\"type\":\"hora\""); break;
        case LOG_RYUKYOKU: o.puts("{\"type\":\"ryukyoku\""); return;
        default: o.puts("{\"type\":\"none\""); return;
    }
    o.puts(",\"actor\":");
    mw_int(o, actor);
    if (ty == LOG_CHI || ty == LOG_PON || ty == LOG_DAIMINKAN || ty == LOG_HORA) {
        o.puts(",\"target\":");
        mw_int(o, target);
    }
    if (ty == LOG_DAHAI || (nc && ty != LOG_ANKAN)) {
        o.puts(",\"pai\":");
        mw_tile(o, pai);
    }
    if (ty == LOG_DAHAI) o.puts((x >> 20) & 1 ? ",\"tsumogiri\":true" : ",\"tsumogiri\":false");
    if (nc) {
        o.puts(",\"consumed\":[");
        for (int k = 0; k < nc; k++) {
            if (k) o.put(',');
            mw_tile(o, c[k]);
        }
        o.put(']');
    }
}

// the review line (with its "\n") of event e of job j
MJX_DN void rv_line(MwOut& o, const RvView& V, int j, int e) {
    const long long r = rv_find(V, j, e);
    if (r < 0) {
        o.puts("{\"type\":\"none\",\"meta\":{\"mask_bits\":0}}\n");
        return;
    }
    rv_reaction(o, V.rec_word[r]);
    o.puts(",\"meta\":");
    mw_meta_fields(o, V.M, r, r);
    const bool kan = r + 1 < V.rec_off[j + 1] && V.rec_kan[r + 1] && V.rec_event[r + 1] == e;
    if (kan && V.M.rec_info[r * 4] == 42) {  // make_meta's kan_select: only when the kan-select row was evaluated
        o.puts(",\"kan_select\":");
        mw_meta_fields(o, V.M, r + 1, r);
        o.put('}');
    }
    o.puts("}}\n");
}

}  // namespace mjx
