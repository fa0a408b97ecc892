// TEST INFRASTRUCTURE ONLY — host build of mortal_b200/csrc/mjx_review.cuh and of the review mode of csrc/mjx_replay.cuh
// (-DMJX_HOST_EMUL): the stepping surface of mjx_env_replay_review / mjx_env_replay_step / mjx_review_react_dev /
// mjx_review_render_*_dev, one host lane per job, so the review can be diffed against the emulated mjai.Bot and run under
// sanitizers without a GPU. The observation is encoded without the v4 single-player block (the test engines read channels below
// 200 only). Never loaded by mortal_b200/. Part of libmjx_emul.so (tests/emul_lib.py); driven by tests/review_lib.py emul_review.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "mjx_sp.cuh"
#include "mjx_review.cuh"
#include "mjx_tables_host.h"

using namespace mjx;

namespace {
HostTables g_RH;
Tables g_RT;
bool g_rready = false;

struct EmulReview {
    int n = 0, cap = 0;
    std::vector<TableState> tabs;
    std::vector<i32> row_table, n_rows, done, steps, errs, scores;
    std::vector<u8> row_seat, masks, ranks;
    std::vector<u32> row_step;
    std::vector<i64> actions;
    unsigned long long counters[3] = {0, 0, 0};
    std::vector<u64> hdr, kyoku;
    std::vector<i32> ev_off, ev_cnt, ky_off, pos, ky_idx, ky_seen;
    std::vector<u8> player, meta;
    std::vector<i64> label;
    EnvView V{};
    ReplayView R{};
};
}  // namespace

extern "C" {

int emulr_init(const char* data_dir) {
    if (g_rready) return 0;
    if (!load_host_tables(data_dir, g_RH)) return -1;
    g_RT.suhai = g_RH.suhai.data(); g_RT.jihai = g_RH.jihai.data(); g_RT.agari_keys = g_RH.agari_keys.data();
    g_RT.agari_divs = g_RH.agari_divs.data(); g_RT.agari_ndivs = g_RH.agari_ndivs.data();
    g_rready = true;
    return 0;
}

// a replay env in review mode (mjx_env_create_replay + mjx_env_replay_review): arrays copied, the records marked single-seat;
// masks[j] = the scan result of job j (-1: not marked)
void* emulr_create(int n_jobs, const uint64_t* hdr, const int32_t* ev_off, const int32_t* ev_cnt, long long n_hdr,
                   const uint64_t* kyoku, const int32_t* ky_off, long long n_kyoku_words, const uint8_t* players, int32_t* masks) {
    EmulReview* E = new EmulReview();
    E->n = n_jobs; E->cap = n_jobs * MAX_ROWS_PER_TABLE;
    E->tabs.resize(n_jobs);
    for (int t = 0; t < n_jobs; t++) {
        TableState& S = E->tabs[t];
        memset(&S, 0, sizeof S);
        for (int i = 0; i < 4; i++) { S.scores[i] = 25000; S.row_of_seat[i] = -1; S.kan_row_of_seat[i] = -1; S.auto_action[i] = -1; }
        S.gflags = GF_ALIVE;
    }
    E->row_table.assign(E->cap, 0); E->row_seat.assign(E->cap, 0); E->row_step.assign(E->cap, 0);
    E->masks.assign((size_t)E->cap * ACTION_SPACE, 0); E->actions.assign(E->cap, 45); E->n_rows.assign(1, 0);
    E->done.assign(n_jobs, 0); E->steps.assign(n_jobs, 0); E->errs.assign(n_jobs, 0); E->scores.assign(n_jobs * 4, 0);
    E->ranks.assign(n_jobs * 4, 0);
    EnvView& V = E->V;
    V.tables = E->tabs.data(); V.n_tables = n_jobs; V.row_cap = E->cap; V.n_rows = E->n_rows.data();
    V.row_table = E->row_table.data(); V.row_seat = E->row_seat.data(); V.row_step = E->row_step.data(); V.masks = E->masks.data();
    V.actions = E->actions.data(); V.scores = E->scores.data(); V.ranks = E->ranks.data(); V.done = E->done.data();
    V.steps = E->steps.data(); V.err = E->errs.data(); V.counters = E->counters;
    E->hdr.assign(hdr, hdr + n_hdr); E->kyoku.assign(kyoku, kyoku + n_kyoku_words);
    E->ev_off.assign(ev_off, ev_off + n_jobs); E->ev_cnt.assign(ev_cnt, ev_cnt + n_jobs); E->ky_off.assign(ky_off, ky_off + n_jobs);
    E->pos.assign(n_jobs, 0); E->ky_idx.assign(n_jobs, 0); E->ky_seen.assign(n_jobs, 0);
    E->player.assign(players, players + n_jobs); E->label.assign(E->cap, 0); E->meta.assign((size_t)E->cap * 4, 0);
    ReplayView& R = E->R;
    R.hdr = E->hdr.data(); R.ev_off = E->ev_off.data(); R.ev_cnt = E->ev_cnt.data(); R.kyoku = E->kyoku.data();
    R.ky_off = E->ky_off.data(); R.pos = E->pos.data(); R.ky_idx = E->ky_idx.data(); R.ky_seen = E->ky_seen.data();
    R.player = E->player.data(); R.row_label = E->label.data(); R.row_meta = E->meta.data();
    R.review = 1;
    const long long n_ky = n_kyoku_words / REPLAY_KYOKU_WORDS;
    for (int t = 0; t < n_jobs; t++) {
        const int m = replay_hidden_seats(R, t, n_hdr, n_ky, 0);
        replay_mark_viewpoint(&E->tabs[t], R.player[t], m, true);
        masks[t] = m;
    }
    return E;
}

void emulr_destroy(void* p) { delete static_cast<EmulReview*>(p); }

// mjx_env_replay_step: returns the jobs still live
int emulr_step(void* p) {
    EmulReview* E = static_cast<EmulReview*>(p);
    E->n_rows[0] = 0;
    int live = 0;
    WarpScratch W;
    for (int t = 0; t < E->n; t++) {
        Ctx c; c.S = &E->tabs[t]; c.W = &W; c.T = g_RT; c.lane = 0; c.df = W.dora_factor;
        if (replay_table(c, E->V, E->R, t)) live++;
    }
    return live;
}

// the step's rows: row_table, row_seat, row_step, masks [n, 46]; returns n
int emulr_rows(void* p, int32_t* row_table, uint8_t* row_seat, uint32_t* row_step, uint8_t* masks) {
    EmulReview* E = static_cast<EmulReview*>(p);
    const int n = E->n_rows[0];
    for (int r = 0; r < n; r++) { row_table[r] = E->row_table[r]; row_seat[r] = E->row_seat[r]; row_step[r] = E->row_step[r]; }
    memcpy(masks, E->masks.data(), (size_t)n * ACTION_SPACE);
    return n;
}

// the observation of every row of the step, [n, rows(version), 34], without the v4 single-player block
void emulr_encode(void* p, float* obs, int version) {
    EmulReview* E = static_cast<EmulReview*>(p);
    const ObsLayout L = make_layout(version);
    for (int r = 0; r < E->n_rows[0]; r++) {
        float* tile = obs + (size_t)r * L.rows * OBS_COLS;
        memset(tile, 0, sizeof(float) * L.rows * OBS_COLS);
        const TableState* S = &E->tabs[E->row_table[r]];
        u8 df[34];
        for (int t = 0; t < 34; t++) {
            int f = 0;
            for (int k = 0; k < S->n_dora; k++) f += tile_next(S->wall[60 - k]) == t;
            df[t] = (u8)f;
        }
        std::vector<u64> bm(L.bm_rows, 0);
        std::vector<float> sv((size_t)OBS_MAX_SV * OBS_COLS, 0.f);
        EncCtx e;
        e.S = S; e.T = g_RT; e.bm = bm.data(); e.sv = sv.data(); e.seat = E->row_seat[r] & 3; e.kan_select = (E->row_seat[r] >> 2) & 1;
        e.lane = 0; e.dora_factor = df;
        Ctx c; c.S = const_cast<TableState*>(S); c.W = nullptr; c.T = g_RT; c.lane = 0; c.df = df;
        for (int part = 0; part < ENC_N_PARTS; part++) {
            e.parts = 1u << part;
            encode_obs_any(version, e, c, nullptr);
        }
        for (int lo = 0; lo < L.rows; lo += OBS_SLICE_ROWS)
            enc_materialize(L, e, tile + (size_t)lo * OBS_COLS, lo, lo + OBS_SLICE_ROWS < L.rows ? lo + OBS_SLICE_ROWS : L.rows);
    }
}

// mjx_review_react_dev over the step's n_rows rows
void emulr_react(void* p, int n_rows, const int64_t* actions, const float* q, const uint8_t* greedy, int guard, int32_t* info,
                 uint64_t* mask, float* q_out, int64_t* i64s, uint64_t* word) {
    EmulReview* E = static_cast<EmulReview*>(p);
    const ReviewOut O{info, mask, q_out, i64s, word};
    WarpScratch W;
    for (int r = 0; r < n_rows; r++) {
        if (E->row_seat[r] & 4) continue;
        Ctx c; c.S = &E->tabs[E->row_table[r]]; c.W = &W; c.T = g_RT; c.lane = 0; c.df = W.dora_factor;
        recompute_dora_factor(c);
        review_react_row(c, E->V, E->R, r, n_rows, actions, q, greedy, guard != 0, O);
    }
}

// per job: err (mjx_env_results err) and the event it stopped at (steps)
void emulr_results(void* p, int32_t* errs, int32_t* steps) {
    EmulReview* E = static_cast<EmulReview*>(p);
    memcpy(errs, E->errs.data(), sizeof(i32) * E->n);
    memcpy(steps, E->steps.data(), sizeof(i32) * E->n);
}

// mjx_review_render_count_dev (out null) / _fill_dev: one lane per job, its lines in order; bytes[j] = job j's size
void emulr_render(int n_jobs, const int32_t* ev_cnt, const int64_t* rec_off, long long n_rec, const int32_t* rec_event,
                  const uint8_t* rec_kan, const uint64_t* rec_word, const int32_t* rec_info, const uint64_t* rec_mask, const float* rec_q,
                  const int64_t* rec_i64, const uint8_t* skip, int64_t* bytes, const int64_t* off, char* out, long long out_cap) {
    RvView V{};
    V.ev_cnt = ev_cnt; V.rec_off = rec_off; V.rec_event = rec_event; V.rec_kan = rec_kan; V.rec_word = rec_word; V.skip = skip;
    V.M.rec_info = rec_info; V.M.rec_mask = rec_mask; V.M.rec_q = rec_q; V.M.rec_i64 = rec_i64; V.M.n_rec = n_rec; V.n_jobs = n_jobs;
    for (int j = 0; j < n_jobs; j++) {
        long long at = out ? off[j] : 0;
        long long total = 0;
        if (!skip[j])
            for (int e = 0; e < ev_cnt[j]; e++) {
                MwOut o{out ? out + at + total : nullptr, 0, out ? out_cap - at - total : 0};
                rv_line(o, V, j, e);
                total += o.n;
            }
        if (bytes) bytes[j] = total;
    }
}

}  // extern "C"
