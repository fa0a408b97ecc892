// TEST INFRASTRUCTURE ONLY — single-lane host build of mortal_b200/csrc/mjx_step.cuh (-DMJX_HOST_EMUL), with the replay,
// the single-viewpoint scan and the log validator (k_validate_logs). Lets the GPU-less dev container diff the product's rule
// logic against the oracle. Never loaded by mortal_b200/; the product has no CPU path. Built by tests/emul_lib.py, which
// also binds these entries; emul_init loads the lookup tables for all of them.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "mjx_sp.cuh"
#include "mjx_replay.cuh"
#include "mjx_invisible.cuh"
#include "mjx_state.cuh"
#include "mjx_policy.cuh"
#include "mjx_validate.cuh"
#include "mjx_tables_host.h"

using namespace mjx;

static HostTables g_H;
static Tables g_T;
static bool g_ready = false;
static std::string g_err;

extern "C" {

const char* emul_last_error() { return g_err.c_str(); }

int emul_init(const char* data_dir) {
    if (g_ready) return 0;
    if (!load_host_tables(data_dir, g_H)) { g_err = g_H.error; return -1; }
    g_T.suhai = g_H.suhai.data();
    g_T.jihai = g_H.jihai.data();
    g_T.agari_keys = g_H.agari_keys.data();
    g_T.agari_divs = g_H.agari_divs.data();
    g_T.agari_ndivs = g_H.agari_ndivs.data();
    g_ready = true;
    return 0;
}

int emul_sizeof_table() { return (int)sizeof(TableState); }

int emul_shanten(const uint8_t* tiles, const uint8_t* len_div3, int8_t* out, int n) {
    for (int i = 0; i < n; i++) out[i] = (int8_t)shanten_all(g_T, tiles + (size_t)i * 34, len_div3[i]);
    return 0;
}

void emul_make_wall(uint64_t nonce, uint64_t key, int kyoku, int honba, int kind, uint8_t* out) {
    make_wall(nonce, key, kyoku, honba, kind, out);
}

// trace rows: [table, step_idx, seat, action, kan_select, mask_bits]
int emul_run(int n, const uint64_t* nonces, const uint64_t* keys, int shuffle_kind, int quick_eval, int policy_kind,
             int32_t* scores, uint8_t* ranks, int32_t* steps, int32_t* errs, int64_t* trace, int64_t trace_cap,
             int64_t* trace_len, int64_t max_cycles, int agari_guard) {
    std::vector<TableState> tabs(n);
    for (int t = 0; t < n; t++) {
        TableState& S = tabs[t];
        memset(&S, 0, sizeof S);
        S.nonce = nonces[t]; S.key = keys[t];
        for (int i = 0; i < 4; i++) { S.scores[i] = 25000; S.row_of_seat[i] = -1; S.kan_row_of_seat[i] = -1; S.auto_action[i] = -1; }
        S.shuffle_kind = (u8)shuffle_kind;
        S.gflags = GF_ALIVE;
    }
    const int cap = n * MAX_ROWS_PER_TABLE;
    std::vector<i32> row_table(cap), done(n, 0), n_rows(1, 0);
    std::vector<u8> row_seat(cap), masks((size_t)cap * ACTION_SPACE);
    std::vector<u32> row_step(cap);
    std::vector<i64> actions(cap, 45);
    unsigned long long counters[2] = {0, 0};
    EnvView V;
    V.tables = tabs.data(); V.n_tables = n; V.row_cap = cap; V.n_rows = n_rows.data();
    V.row_table = row_table.data(); V.row_seat = row_seat.data(); V.row_step = row_step.data();
    V.masks = masks.data(); V.actions = actions.data(); V.scores = scores; V.ranks = ranks; V.done = done.data();
    V.steps = steps; V.err = errs; V.counters = counters; V.enable_quick_eval = quick_eval; V.quick_eval_seat = nullptr;
    std::vector<float> qv((size_t)cap * ACTION_SPACE, 0.f);
    std::vector<u8> guard((size_t)n * 4, 1);
    V.log = nullptr; V.log_len = nullptr; V.log_cap = 0;
    V.q_values = agari_guard ? qv.data() : nullptr;
    V.agari_guard = agari_guard ? guard.data() : nullptr;
    for (int t = 0; t < n; t++) { steps[t] = 0; errs[t] = 0; }
    int64_t tl = 0;
    WarpScratch W;
    for (int64_t cycle = 0; max_cycles <= 0 || cycle < max_cycles; cycle++) {
        n_rows[0] = 0;
        int live = 0;
        for (int t = 0; t < n; t++) {
            Ctx c;
            c.S = &tabs[t]; c.W = &W; c.T = g_T; c.lane = 0; c.df = W.dora_factor;
            if (step_table(c, V, t)) live++;
        }
        if (live == 0) break;
        // policy over the emitted rows
        for (int r = 0; r < n_rows[0]; r++) {
            int t = row_table[r], seat = row_seat[r] & 3, kan = (row_seat[r] >> 2) & 1;
            u64 m = 0;
            for (int i = 0; i < ACTION_SPACE; i++) if (masks[(size_t)r * ACTION_SPACE + i]) m |= 1ull << i;
            const SeatPrivate& P = tabs[t].priv[seat];
            u64 h = policy_hash(tabs[t].nonce, tabs[t].key, (u64)t, row_step[r], (u32)seat, (u32)kan);
            int a = test_policy(policy_kind, h, kan != 0, m, P.keep_shanten, P.next_shanten);
            actions[r] = a;
            if (agari_guard) for (int i = 0; i < ACTION_SPACE; i++) qv[(size_t)r * ACTION_SPACE + i] = ((m >> i) & 1) ? 0.f : -INFINITY;
            if (trace && tl < trace_cap) {
                int64_t* o = trace + tl * 6;
                o[0] = t; o[1] = row_step[r]; o[2] = seat; o[3] = a; o[4] = kan; o[5] = (int64_t)m;
            }
            tl++;
        }
    }
    if (trace_len) *trace_len = tl;
    for (int t = 0; t < n; t++) if (!done[t]) { errs[t] = errs[t] ? errs[t] : -1; }
    return 0;
}

// ---------------- stateful env (mirrors the C ABI's mjx_env_* so tests can drive it in lock step) ----------------
struct EmulEnv {
    int n = 0, cap = 0;
    std::vector<TableState> tabs;
    std::vector<i32> row_table, done, steps, errs, scores, n_rows;
    std::vector<u8> row_seat, masks, ranks, qe_seat;
    std::vector<u32> row_step;
    std::vector<i64> actions;
    unsigned long long counters[2] = {0, 0};
    EnvView V;
    bool first = true;
    std::vector<u64> log; std::vector<i32> log_len; int log_cap = 0;
    std::vector<i32> grp, grp_len; int grp_cap = 0;
    // log replay (mjx_replay.cuh)
    std::vector<u64> r_hdr, r_kyoku; std::vector<i32> r_ev_off, r_ev_cnt, r_ky_off, r_pos, r_ky_idx, r_ky_seen;
    std::vector<u8> r_player, r_meta; std::vector<i64> r_label;
    ReplayView R;
};

void* emul_env_create(int n, const uint64_t* nonces, const uint64_t* keys, int shuffle_kind, int quick_eval) {
    EmulEnv* E = new EmulEnv();
    E->n = n; E->cap = n * MAX_ROWS_PER_TABLE;
    E->tabs.resize(n);
    for (int t = 0; t < n; t++) {
        TableState& S = E->tabs[t];
        memset(&S, 0, sizeof S);
        S.nonce = nonces[t]; S.key = keys[t];
        for (int i = 0; i < 4; i++) { S.scores[i] = 25000; S.row_of_seat[i] = -1; S.kan_row_of_seat[i] = -1; S.auto_action[i] = -1; }
        S.shuffle_kind = (u8)shuffle_kind;
        S.gflags = GF_ALIVE;
    }
    E->row_table.assign(E->cap, 0); E->row_seat.assign(E->cap, 0); E->row_step.assign(E->cap, 0);
    E->masks.assign((size_t)E->cap * ACTION_SPACE, 0); E->actions.assign(E->cap, 45);
    E->done.assign(n, 0); E->steps.assign(n, 0); E->errs.assign(n, 0); E->scores.assign(n * 4, 0); E->ranks.assign(n * 4, 0);
    E->n_rows.assign(1, 0);
    EnvView& V = E->V;
    V.tables = E->tabs.data(); V.n_tables = n; V.row_cap = E->cap; V.n_rows = E->n_rows.data();
    V.row_table = E->row_table.data(); V.row_seat = E->row_seat.data(); V.row_step = E->row_step.data();
    V.masks = E->masks.data(); V.actions = E->actions.data(); V.scores = E->scores.data(); V.ranks = E->ranks.data();
    V.done = E->done.data(); V.steps = E->steps.data(); V.err = E->errs.data(); V.counters = E->counters;
    V.q_values = nullptr; V.agari_guard = nullptr;
    V.enable_quick_eval = quick_eval; V.quick_eval_seat = nullptr;
    V.log = nullptr; V.log_len = nullptr; V.log_cap = 0;
    return E;
}
void emul_env_destroy(void* p) { delete static_cast<EmulEnv*>(p); }
void emul_env_enable_grp(void* p, int cap) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    E->grp_cap = cap; E->grp.assign((size_t)E->n * cap * 7, 0); E->grp_len.assign(E->n, 0);
}
void emul_env_read_grp(void* p, int32_t* feat, int32_t* cnt) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    memcpy(feat, E->grp.data(), E->grp.size() * sizeof(i32)); memcpy(cnt, E->grp_len.data(), E->grp_len.size() * sizeof(i32));
}
void emul_env_set_quick_eval(void* p, const uint8_t* flags) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    static_assert(sizeof(u8) == 1, "");
    E->qe_seat.assign(flags, flags + (size_t)E->n * 4);
    E->V.quick_eval_seat = E->qe_seat.data();
}

// returns number of live tables after the step
int emul_env_step(void* p, const int64_t* actions) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    if (actions) for (int i = 0; i < E->cap; i++) E->actions[i] = actions[i];
    E->n_rows[0] = 0;
    int live = 0;
    WarpScratch W;
    for (int t = 0; t < E->n; t++) {
        Ctx c; c.S = &E->tabs[t]; c.W = &W; c.T = g_T; c.lane = 0; c.df = W.dora_factor;
        if (E->log_cap) { c.log = E->log.data() + (size_t)t * E->log_cap; c.log_n = &E->log_len[t]; c.log_cap = E->log_cap; }
        if (E->grp_cap) { c.grp = E->grp.data() + (size_t)t * E->grp_cap * 7; c.grp_n = &E->grp_len[t]; c.grp_cap = E->grp_cap; }
        if (step_table(c, E->V, t)) live++;
    }
    return live;
}
// ---- log replay: the stepping surface of mjx_env_create_replay / mjx_env_replay_step
void* emul_env_create(int n, const uint64_t* nonces, const uint64_t* keys, int shuffle_kind, int quick_eval);
void* emul_replay_create(int n_jobs, const uint64_t* hdr, const int32_t* ev_off, const int32_t* ev_cnt, long long n_hdr,
                         const uint64_t* kyoku, const int32_t* ky_off, long long n_kyoku_words, const uint8_t* players,
                         int always_include_kan_select) {
    std::vector<uint64_t> zeros(n_jobs, 0);
    EmulEnv* E = static_cast<EmulEnv*>(emul_env_create(n_jobs, zeros.data(), zeros.data(), 0, 0));
    E->r_hdr.assign(hdr, hdr + n_hdr); E->r_kyoku.assign(kyoku, kyoku + n_kyoku_words);
    E->r_ev_off.assign(ev_off, ev_off + n_jobs); E->r_ev_cnt.assign(ev_cnt, ev_cnt + n_jobs); E->r_ky_off.assign(ky_off, ky_off + n_jobs);
    E->r_pos.assign(n_jobs, 0); E->r_ky_idx.assign(n_jobs, 0); E->r_ky_seen.assign(n_jobs, 0);
    E->r_player.assign(players, players + n_jobs);
    E->r_label.assign(E->cap, 0); E->r_meta.assign((size_t)E->cap * 4, 0);
    ReplayView& R = E->R;
    R.hdr = E->r_hdr.data(); R.ev_off = E->r_ev_off.data(); R.ev_cnt = E->r_ev_cnt.data(); R.kyoku = E->r_kyoku.data();
    R.ky_off = E->r_ky_off.data(); R.pos = E->r_pos.data(); R.ky_idx = E->r_ky_idx.data(); R.ky_seen = E->r_ky_seen.data();
    R.player = E->r_player.data(); R.row_label = E->r_label.data(); R.row_meta = E->r_meta.data();
    R.always_include_kan_select = always_include_kan_select;
    return E;
}
void emul_replay_trust_seeds(void* p, const uint64_t* nonces, const uint64_t* keys, int shuffle_kind) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    for (int t = 0; t < E->n; t++) { E->tabs[t].nonce = nonces[t]; E->tabs[t].key = keys[t]; E->tabs[t].shuffle_kind = (u8)shuffle_kind; }
    E->R.trust_seed = 1;
}
void emul_replay_encode_invisible(void* p, float* out, int version) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    const int rows = oracle_obs_rows(version);
    for (int r = 0; r < E->n_rows[0]; r++)
        encode_invisible(&E->tabs[E->row_table[r]], E->row_seat[r] & 3, version, out + (size_t)r * rows * OBS_COLS, 0, true);
}
int emul_replay_step(void* p) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    E->n_rows[0] = 0;
    int live = 0;
    WarpScratch W;
    for (int t = 0; t < E->n; t++) {
        Ctx c; c.S = &E->tabs[t]; c.W = &W; c.T = g_T; c.lane = 0; c.df = W.dora_factor;
        if (replay_table(c, E->V, E->R, t)) live++;
    }
    return live;
}
// mjx_env_replay_viewpoints on an emul_replay_create env: the scan and the mark, one lane per job; the scan result of every job
// (-1 = not marked, else the mask of hidden seats) goes to `masks` when it is not null
void emul_replay_viewpoints(void* p, int32_t* masks) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    const long long n_hdr = (long long)E->r_hdr.size(), n_kyoku = (long long)(E->r_kyoku.size() / REPLAY_KYOKU_WORDS);
    for (int t = 0; t < E->n; t++) {
        const int mask = replay_hidden_seats(E->R, t, n_hdr, n_kyoku, 0);
        replay_mark_viewpoint(&E->tabs[t], E->R.player[t], mask);
        if (masks) masks[t] = mask;
    }
}
void emul_replay_rows(void* p, int64_t* labels, uint8_t* meta) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    const int n = E->n_rows[0];
    for (int r = 0; r < n; r++) { labels[r] = E->r_label[r]; for (int k = 0; k < 4; k++) meta[r * 4 + k] = E->r_meta[(size_t)r * 4 + k]; }
}
int emul_env_errs(void* p, int32_t* errs) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    int bad = 0;
    for (int t = 0; t < E->n; t++) { errs[t] = E->errs[t]; bad += errs[t] != 0; }
    return bad;
}

void emul_env_enable_log(void* p, int cap) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    E->log_cap = cap; E->log.assign((size_t)E->n * cap, 0); E->log_len.assign(E->n, 0);
}
void emul_env_log_lens(void* p, int32_t* lens) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    memcpy(lens, E->log_len.data(), E->log_len.size() * sizeof(i32));
}
void emul_env_row_steps(void* p, uint32_t* steps) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    for (int r = 0; r < E->n_rows[0]; r++) steps[r] = E->row_step[r];
}
void emul_env_read_log(void* p, uint64_t* words, int32_t* lens) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    memcpy(words, E->log.data(), E->log.size() * sizeof(u64));
    memcpy(lens, E->log_len.data(), E->log_len.size() * sizeof(i32));
}
int emul_env_num_rows(void* p) { return static_cast<EmulEnv*>(p)->n_rows[0]; }
void emul_env_rows(void* p, int32_t* row_table, uint8_t* row_seat, uint8_t* masks) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    int n = E->n_rows[0];
    for (int r = 0; r < n; r++) { row_table[r] = E->row_table[r]; row_seat[r] = E->row_seat[r]; }
    memcpy(masks, E->masks.data(), (size_t)n * ACTION_SPACE);
}
void emul_env_policy_test(void* p, int kind, int64_t* actions) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    for (int r = 0; r < E->n_rows[0]; r++) {
        int t = E->row_table[r], seat = E->row_seat[r] & 3, kan = (E->row_seat[r] >> 2) & 1;
        u64 m = 0;
        for (int i = 0; i < ACTION_SPACE; i++) if (E->masks[(size_t)r * ACTION_SPACE + i]) m |= 1ull << i;
        const SeatPrivate& P = E->tabs[t].priv[seat];
        u64 h = policy_hash(E->tabs[t].nonce, E->tabs[t].key, (u64)t, E->row_step[r], (u32)seat, (u32)kan);
        actions[r] = test_policy(kind, h, kan != 0, m, P.keep_shanten, P.next_shanten);
    }
}
void emul_env_encode_obs_v(void* p, float* obs, int sp, int version);
void emul_env_encode_obs(void* p, float* obs, int sp) { emul_env_encode_obs_v(p, obs, sp, 4); }
static long g_emul_sp_overflows = 0;
long emul_sp_overflows() { return g_emul_sp_overflows; }

// obs: [n_rows, rows(version), 34] f32; sp: compute the single-player block (version 4 only)
void emul_env_encode_obs_v(void* p, float* obs, int sp, int version) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    const int n_rows = E->n_rows[0];
    const ObsLayout L = make_layout(version);
    for (int r = 0; r < n_rows; r++) {
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
        e.S = S; e.T = g_T; e.bm = bm.data(); e.sv = sv.data(); e.seat = E->row_seat[r] & 3; e.kan_select = (E->row_seat[r] >> 2) & 1;
        e.lane = 0; e.dora_factor = df;
        Ctx c; c.S = const_cast<TableState*>(S); c.W = nullptr; c.T = g_T; c.lane = 0; c.df = df;
        for (int part = 0; part < ENC_N_PARTS; part++) {  // part by part, as the CUDA kernel derives them
            e.parts = 1u << part;
            encode_obs_any(version, e, c, nullptr);
        }
        // materialised slice by slice, as the CUDA kernel does
        for (int lo = 0; lo < L.rows; lo += OBS_SLICE_ROWS)
            enc_materialize(L, e, tile + (size_t)lo * OBS_COLS, lo, lo + OBS_SLICE_ROWS < L.rows ? lo + OBS_SLICE_ROWS : L.rows);
    }
    if (!sp || version != 4) return;
    // the same stage sequence mjx_env_encode_obs launches (csrc/mjx_kernels.cu launch_sp_block), executed by one thread
    static SpGlobal G;
    static std::vector<SpRow> rows; static std::vector<u64> hkey, einfo, dkey; static std::vector<SpSigP> nsig;
    static std::vector<float> vals, leaf_scores; static std::vector<u32> echild, eowner, wl, sid, evid; static std::vector<u16> emeta;
    static i32 wl_count[SP_SLOTS], counters[8];
    if (hkey.empty()) {
        G.hash_cap = 1 << 21; G.wl_cap = G.hash_cap / 4; G.edge_cap = G.hash_cap * 2; G.score_cap = G.hash_cap;
        rows.resize(1 << 16); hkey.assign(G.hash_cap, SP_EMPTY); einfo.resize(G.hash_cap); nsig.resize(G.hash_cap);
        vals.resize((size_t)G.hash_cap * SP_VALS); leaf_scores.resize((size_t)G.score_cap * 4);
        echild.resize(G.edge_cap); eowner.resize(G.edge_cap); emeta.resize(G.edge_cap); wl.resize((size_t)SP_SLOTS * G.wl_cap);
        G.rows = rows.data(); G.hkey = hkey.data(); G.einfo = einfo.data(); G.nsig = nsig.data(); G.vals = vals.data();
        G.leaf_scores = leaf_scores.data(); G.echild = echild.data(); G.eowner = eowner.data(); G.emeta = emeta.data();
        dkey.resize(G.hash_cap); G.dkey = dkey.data();
        sid.resize(G.hash_cap); evid.assign(G.edge_cap, 0); G.sid = sid.data(); G.evid = evid.data();
        G.wl = wl.data(); G.wl_count = wl_count; G.counters = counters;
        static std::vector<float> p_tab((size_t)SP_NTS_DIM * SP_NTS_DIM * 4 * SP_TRI);
        for (int i = 0; i < SP_NTS_DIM * SP_NTS_DIM; i++) sp_fill_ptab_block(p_tab.data() + (size_t)i * 4 * SP_TRI, i / SP_NTS_DIM, i % SP_NTS_DIM);
        G.p_tab = p_tab.data();
        for (int i = 0; i < 8; i++) counters[i] = 0;
    }
    for (int i = 0; i < SP_SLOTS; i++) wl_count[i] = 0;
    counters[1] = counters[2] = counters[4] = counters[5] = 0;
    u8 df[40];
    SpCtx s; s.G = G; s.T = g_T; s.df = df; s.lane = 0;
    SpBlk B; B.tid = 0; B.nthr = 1; B.bid = 0; B.nblk = 1;
    static SpExpandBatch xb; static SpEvalDBatch ed; static SpEvalWBatch ew;
    for (int r = 0; r < n_rows; r++) sp_stage_init(s, &E->tabs[E->row_table[r]], r, E->row_table[r], E->row_seat[r] & 3);
    for (int level = 0; level < SP_SLOTS; level++) {
        if (level == SP_SLOTS - 1) { counters[4] = counters[1]; sp_expand_level<2>(G, g_T, xb, B, level); }
        else if (sp_slot_is_w(level)) sp_expand_level<1>(G, g_T, xb, B, level);
        else sp_expand_level<0>(G, g_T, xb, B, level);
    }
    counters[5] = counters[1];
    sp_densify(G, B);
    for (int e = counters[4]; e < counters[5]; e++) sp_score_edge(G, g_T, e);
    for (int level = SP_SLOTS - 1; level >= 0; level--) {
        if (!sp_slot_is_w(level)) sp_eval_d_level(G, ed, B, level);
        else if (level == SP_SLOTS - 1) sp_eval_w_level<true>(G, &ew, B, level);
        else sp_eval_w_level<false>(G, &ew, B, level);
    }
    for (int r = 0; r < n_rows; r++) sp_stage_finalize(s, r, obs + (size_t)r * OBS_ROWS_V4 * OBS_COLS);
    if (counters[2]) g_emul_sp_overflows++;
    sp_release(G, B);
    counters[2] = 0;
}
// invisible (oracle) observation of every current row: [n_rows, oracle_obs_rows(version), 34]
void emul_env_encode_invisible(void* p, float* out, int version) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    const int rows = oracle_obs_rows(version);
    for (int r = 0; r < E->n_rows[0]; r++)
        encode_invisible(&E->tabs[E->row_table[r]], E->row_seat[r] & 3, version, out + (size_t)r * rows * OBS_COLS, 0);
}
// ---- libriichi.state.PlayerState batch: the surface of mjx_state_* (include/mjx.h), one lane
void* emul_state_create(int n, const uint8_t* player_ids) {
    std::vector<uint64_t> zeros(n, 0);
    EmulEnv* E = static_cast<EmulEnv*>(emul_env_create(n, zeros.data(), zeros.data(), 0, 0));
    for (int t = 0; t < n; t++) {
        TableState& S = E->tabs[t];
        S.viewer1 = (u8)(player_ids[t] + 1); S.last_kawa_tile = T_NONE;
        for (int s = 0; s < 4; s++) S.priv[s].last_self_tsumo = T_NONE;
    }
    return E;
}
static Ctx emul_state_ctx(EmulEnv* E, int i, WarpScratch& W) {
    Ctx c; c.S = &E->tabs[i]; c.W = &W; c.T = g_T; c.lane = 0; c.df = W.dora_factor;
    recompute_dora_factor(c);
    return c;
}
void emul_state_update(void* p, const uint64_t* words, const uint64_t* payload, uint32_t* cans) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    WarpScratch W;
    for (int i = 0; i < E->n; i++) {
        Ctx c = emul_state_ctx(E, i, W);
        if (words[i] != 0) apply_event(c, words[i], payload ? payload + (size_t)i * REPLAY_KYOKU_WORDS : nullptr, false);
        const SeatPrivate& P = E->tabs[i].priv[E->tabs[i].viewer1 - 1];
        cans[i] = (u32)P.cans | ((u32)P.target_actor << 16);
    }
}
void emul_state_view(void* p, int index, mjx_player_view* out) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    WarpScratch W;
    Ctx c = emul_state_ctx(E, index, W);
    memset(out, 0, sizeof *out);
    state_view(c, E->tabs[index].viewer1 - 1, out);
}
void emul_state_rows(void* p, const uint8_t* at_kan_select) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    WarpScratch W;
    for (int i = 0; i < E->n; i++) {
        Ctx c = emul_state_ctx(E, i, W);
        const int pl = E->tabs[i].viewer1 - 1;
        const bool kan = at_kan_select && at_kan_select[i];
        const u64 discards = (E->tabs[i].priv[pl].cans & CAN_DISCARD) ? discard_candidates(c, pl) : 0;
        write_mask_row(c, E->V, i, legal_mask(c, pl, kan, discards));
        E->row_table[i] = i; E->row_seat[i] = (u8)(pl | (kan ? 4 : 0)); E->row_step[i] = 0;
    }
    E->n_rows[0] = E->n;
}
void emul_state_query(void* p, int index, int what, const int32_t* args, int32_t* out) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    WarpScratch W;
    Ctx c = emul_state_ctx(E, index, W);
    const int pl = E->tabs[index].viewer1 - 1;
    out[0] = out[1] = out[2] = out[3] = 0;
    if (what == 0) {
        u8 ura[5]; const int n_ura = std::min(std::max(args[1], 0), 5);
        for (int k = 0; k < n_ura; k++) ura[k] = (u8)args[2 + k];
        bool ok; const Point pt = agari_points_ura(c, pl, args[0] != 0, ura, n_ura, &ok);
        out[0] = pt.ron; out[1] = pt.tsumo_ko; out[2] = pt.tsumo_oya; out[3] = ok ? 1 : 0;
    } else if (what == 1) out[0] = rule_based_agari(c, pl) ? 1 : 0;
    else if (what == 2) { const u64 m = discard_candidates(c, pl); out[0] = (i32)(u32)m; out[1] = (i32)(u32)(m >> 32); }
    else if (what == 3) {
        EncCtx e; e.S = c.S; e.T = g_T; e.bm = nullptr; e.sv = nullptr; e.seat = pl; e.kan_select = false; e.lane = 0; e.dora_factor = c.df; e.parts = 0;
        const u64 m = unconditional_tenpai_discards(e, c); out[0] = (i32)(u32)m; out[1] = (i32)(u32)(m >> 32);
    } else if (what == 4) {
        Reaction r; i32 err = 0;
        const bool okd = decode_action(c.S, pl, args[0], args[1], r, &err);
        u64 w = 0;
        if (okd) {
            const int ty = r.type == R_DAHAI ? LOG_DAHAI : r.type == R_CHI ? LOG_CHI : r.type == R_PON ? LOG_PON :
                           r.type == R_DAIMINKAN ? LOG_DAIMINKAN : r.type == R_KAKAN ? LOG_KAKAN : r.type == R_ANKAN ? LOG_ANKAN :
                           r.type == R_REACH ? LOG_REACH : r.type == R_HORA ? LOG_HORA : r.type == R_RYUKYOKU ? LOG_RYUKYOKU : 0;
            w = log_word(ty, r.actor, r.target, r.pai, r.tsumogiri, 0, r.consumed[0], r.consumed[1], r.consumed[2], r.consumed[3], 0);
        }
        out[0] = (i32)(u32)w; out[1] = (i32)(u32)(w >> 32); out[2] = okd ? 0 : (err ? err : ERR_ILLEGAL_ACTION);
    }
}
void emul_state_copy(void* dst, int di, void* src, int si) {
    static_cast<EmulEnv*>(dst)->tabs[di] = static_cast<EmulEnv*>(src)->tabs[si];
}
void emul_env_results(void* p, int32_t* scores, uint8_t* ranks, int32_t* steps, int32_t* errs, int32_t* done) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    memcpy(scores, E->scores.data(), sizeof(i32) * 4 * E->n); memcpy(ranks, E->ranks.data(), 4 * E->n);
    memcpy(steps, E->steps.data(), sizeof(i32) * E->n); memcpy(errs, E->errs.data(), sizeof(i32) * E->n);
    memcpy(done, E->done.data(), sizeof(i32) * E->n);
}

// ---- mjx_validate_logs one log at a time; the same argument checks as the C ABI, returns 0 or -2
int emulv_validate_logs(int n_logs, const uint64_t* hdr, const int32_t* ev_off, const int32_t* ev_cnt, long long n_hdr,
                        const uint64_t* kyoku, const int32_t* ky_off, long long n_kyoku_words, const uint64_t* hora,
                        const int32_t* hora_off, long long n_hora_words, mjx_verdict* out) {
    if (!g_ready || n_logs <= 0 || !ev_off || !ev_cnt || !ky_off || !hora_off || !out || n_hdr < 0 || (n_hdr > 0 && !hdr) ||
        n_kyoku_words < 0 || n_kyoku_words % REPLAY_KYOKU_WORDS || (n_kyoku_words > 0 && !kyoku) || n_hora_words < 0 ||
        n_hora_words % MJX_HORA_WORDS || (n_hora_words > 0 && !hora))
        return -2;
    for (int i = 0; i < n_logs; i++)
        if (ev_off[i] < 0 || ev_cnt[i] < 0 || (long long)ev_off[i] + ev_cnt[i] > n_hdr || ky_off[i] < 0 || hora_off[i] < 0) return -2;
    ValidateView V;
    V.hdr = hdr; V.ev_off = ev_off; V.ev_cnt = ev_cnt; V.kyoku = kyoku; V.ky_off = ky_off; V.hora = hora; V.hora_off = hora_off;
    V.n_kyoku = n_kyoku_words / REPLAY_KYOKU_WORDS; V.n_hora = n_hora_words / MJX_HORA_WORDS; V.n_logs = n_logs; V.out = out;
    std::vector<TableState> rec(1);
    WarpScratch W;
    for (int i = 0; i < n_logs; i++) {
        memset(rec.data(), 0, sizeof(TableState));
        Ctx c;
        c.S = rec.data(); c.W = &W; c.T = g_T; c.lane = 0; c.df = W.dora_factor;
        validate_log(c, V, i);
    }
    return 0;
}

}  // extern "C"
