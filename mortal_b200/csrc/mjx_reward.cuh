// mortal_b200 — GRP training rewards: mortal/reward_calculator.py (the GRP net of model.py:233-276 over every prefix of a game's
// kyoku rows, calc_matrix, calc_delta_pt) and the per-move targets of mortal/dataloader.py:98-123 (steps_to_done, the kyoku reward
// of each move, the player's rank after the move's kyoku).
//
// k_grp_matrix: a GRU is causal and starts from h0 = 0, so the final hidden state of the prefix feature[:k+1] is the hidden state
// after step k of one pass over the whole game, in every layer. One pass per game therefore gives every prefix's h_n in O(L) where
// the reference packs all L prefixes (L(L+1)/2 GRU steps). A CTA of RW_THREADS threads steps RW_GAMES games together, one kyoku
// row per step: every weight a thread loads is applied to all of the CTA's games. Each dot product (one gate row of one unit, one
// FC output) is split over `ks` adjacent lanes (rw_slices) and summed with shuffles, so the default net (H = 64: 64 units x 4
// slices) keeps all 256 threads busy. The weights (470 KB of float64 for H = 64, 2 layers) are read from L2 through the read-only
// path; the hidden states, the fc.0 output, the step's inputs and the logits live in shared memory:
//     s_h [RW_GAMES][H * layers]  the hidden states, layer 0 first: the FC input (h_n.transpose(0, 1).flatten(1))
//     s_y [RW_GAMES][H * layers]  ReLU(fc.0)
//     s_x [RW_GAMES][8]           the step's feature rows
//     s_lg[RW_GAMES][24]          fc.2, the logits
// Per step and layer: the gates of every unit (rw_gru_compute), a barrier, the new h (rw_gru_write), a barrier; then fc.0, fc.2
// and the softmax with the permutation sums of calc_matrix (one thread per matrix entry) behind the same step. Everything is float64, as the reference's GRP is.
//
// k_train_targets: one warp per job (a Gameplay): its moves in chunks of 32 lanes; steps_to_done is a segmented suffix sum done
// as a backward shuffle scan.
//
// -DMJX_HOST_EMUL builds the same phase functions for a host loop over the thread ids with one slice per dot product
// (tests/host_emul/emul_reward.cc), and rw_job for one lane.
#pragma once
#include "../../include/mjx.h"
#include "mjx_types.cuh"

namespace mjx {

constexpr int RW_THREADS = 256;  // k_grp_matrix CTA
constexpr int RW_GAMES = 4;      // games stepped together by one CTA
constexpr int RW_IN = 7;         // the feature row: {grand_kyoku, honba, kyotaku, scores[4] / 10000}
constexpr int RW_MAX_H = 256, RW_MAX_LAYERS = 4;
constexpr int RW_WARPS = 4;      // k_train_targets: jobs per CTA

// itertools.permutations(range(4)) in lexicographic order: RW_PERMS[p][player] = rank
MJX_CONST u8 RW_PERMS[24][4] = {
    {0, 1, 2, 3}, {0, 1, 3, 2}, {0, 2, 1, 3}, {0, 2, 3, 1}, {0, 3, 1, 2}, {0, 3, 2, 1}, {1, 0, 2, 3}, {1, 0, 3, 2},
    {1, 2, 0, 3}, {1, 2, 3, 0}, {1, 3, 0, 2}, {1, 3, 2, 0}, {2, 0, 1, 3}, {2, 0, 3, 1}, {2, 1, 0, 3}, {2, 1, 3, 0},
    {2, 3, 0, 1}, {2, 3, 1, 0}, {3, 0, 1, 2}, {3, 0, 2, 1}, {3, 1, 0, 2}, {3, 1, 2, 0}, {3, 2, 0, 1}, {3, 2, 1, 0}};

// The packed weight buffer (include/mjx.h mjx_grp_reward_dev): per layer k, rnn.weight_ih_l{k} [3H, in_k], rnn.weight_hh_l{k}
// [3H, H], rnn.bias_ih_l{k} [3H], rnn.bias_hh_l{k} [3H] (gates r, z, n); then fc.0.weight [HL, HL], fc.0.bias [HL], fc.2.weight
// [24, HL], fc.2.bias [24], HL = H * layers.
#ifdef MJX_HOST_EMUL
#define RW_MEMBER inline
#else
#define RW_MEMBER __host__ __device__ __forceinline__
#endif
struct GrpNet {
    const double* w;
    int H, layers;
    RW_MEMBER int in(int k) const { return k ? H : RW_IN; }
    RW_MEMBER long long layer_size(int k) const { return 3LL * H * (in(k) + H) + 6LL * H; }
    RW_MEMBER const double* layer(int k) const {
        const double* p = w;
        for (int i = 0; i < k; i++) p += layer_size(i);
        return p;
    }
    RW_MEMBER const double* fc0() const { return layer(layers); }
    RW_MEMBER const double* fc2() const { const long long hl = (long long)H * layers; return fc0() + hl * hl + hl; }
};

MJX_HD long long rw_weight_count(int H, int layers) {
    GrpNet n{nullptr, H, layers};
    const long long hl = (long long)H * layers;
    long long c = hl * hl + hl + 24 * hl + 24;
    for (int k = 0; k < layers; k++) c += n.layer_size(k);
    return c;
}

// doubles of k_grp_matrix's dynamic shared memory
MJX_HD int rw_smem_doubles(int H, int layers) { return RW_GAMES * (2 * H * layers + 8 + 24); }

// the lanes one dot product of `units` outputs is split over: the largest power of two with units * ks <= RW_THREADS, at most 32
// (the lanes of one output stay in one warp); 1 in the host build
MJX_HD int rw_slices(int units) {
#ifdef MJX_HOST_EMUL
    (void)units;
    return 1;
#else
    int s = 1;
    while (s < 32 && 2 * s * units <= RW_THREADS) s *= 2;
    return s;
#endif
}

// mjx_grp_reward_dev's argument checks (host): MJX_OK or MJX_ERR_ARG
inline int rw_check_args(int n_games, const void* feat, const void* game_off, long long n_rows, const void* weights,
                         long long n_weights, int hidden, int layers, const void* matrix, int n_jobs, const void* move_off,
                         long long n_moves, const void* job_game, const void* job_player, const void* at_kyoku,
                         const void* apply_gamma, const void* dones, const void* rank_by_player, const void* final_scores,
                         const void* pts, const void* steps_to_done, const void* kyoku_reward, const void* player_rank,
                         const void* job_status) {
    if (n_games <= 0 || !game_off || n_rows < 0 || (n_rows > 0 && (!feat || !matrix)) || n_rows > (1LL << 31) - 1) return MJX_ERR_ARG;
    if (hidden < 1 || hidden > RW_MAX_H || layers < 1 || layers > RW_MAX_LAYERS || !weights ||
        n_weights != rw_weight_count(hidden, layers))
        return MJX_ERR_ARG;
    if (n_jobs < 0 || (n_jobs > 0 && (!move_off || !job_game || !job_player || !rank_by_player || !final_scores || !pts ||
                                      !job_status || n_moves < 0)))
        return MJX_ERR_ARG;
    if (n_jobs > 0 && n_moves > 0 && (!at_kyoku || !apply_gamma || !dones || !steps_to_done || !kyoku_reward || !player_rank))
        return MJX_ERR_ARG;
    return MJX_OK;
}

MJX_D bool rw_game_ok(const i32* off, int g, long long n_rows) {
    const long long lo = off[g], hi = off[g + 1];
    return 0 <= lo && lo <= hi && hi <= n_rows;
}

// ---------------------------------------------------------------- k_grp_matrix

struct MatrixView {
    const double* feat;  // [n_rows, 7]
    const i32* game_off;  // [n_games + 1]
    long long n_rows;
    int n_games;
    GrpNet net;
    double* matrix;  // [n_rows, 4, 4]
};

// one CTA's shared state (layout at the top of the file)
struct RwCta {
    double *h, *y, *x, *lg;
    long long* lo;
    int* len;
};

MJX_D RwCta rw_cta(const GrpNet& n, double* mem, long long* lo, int* len) {
    const int hl = n.H * n.layers;
    return RwCta{mem, mem + RW_GAMES * hl, mem + 2 * RW_GAMES * hl, mem + 2 * RW_GAMES * hl + RW_GAMES * 8, lo, len};
}

template <int N>
MJX_D void rw_reduce(double (&a)[N], int ks) {
#ifndef MJX_HOST_EMUL
    for (int o = 1; o < ks; o <<= 1)
        for (int i = 0; i < N; i++) a[i] += __shfl_xor_sync(~0u, a[i], o);
#else
    (void)a; (void)ks;
#endif
}

MJX_D double rw_sigmoid(double x) { return 1.0 / (1.0 + exp(-x)); }

// the CTA's games (a game whose offsets lie outside the rows has no steps and writes nothing); zero hidden states
MJX_D void rw_begin(const MatrixView& V, const RwCta& C, int block, int tid) {
    if (tid < RW_GAMES) {
        const int g = block * RW_GAMES + tid;
        const bool ok = g < V.n_games && rw_game_ok(V.game_off, g, V.n_rows);
        C.lo[tid] = ok ? V.game_off[g] : 0;
        C.len[tid] = ok ? V.game_off[g + 1] - V.game_off[g] : 0;
    }
    for (int i = tid; i < RW_GAMES * V.net.H * V.net.layers; i += RW_THREADS) C.h[i] = 0.0;
}

MJX_D int rw_steps(const RwCta& C) {
    int s = 0;
    for (int g = 0; g < RW_GAMES; g++) s = C.len[g] > s ? C.len[g] : s;
    return s;
}

MJX_D void rw_load_x(const MatrixView& V, const RwCta& C, int t, int tid) {
    if (tid < RW_GAMES * RW_IN) {
        const int g = tid / RW_IN, c = tid % RW_IN;
        C.x[g * 8 + c] = t < C.len[g] ? V.feat[(C.lo[g] + t) * RW_IN + c] : 0.0;
    }
}

// torch's GRU cell gates of unit j from the input (gi) and hidden (gh) dot products of its three gate rows (r, z, n):
// r = σ(W_ir x + b_ir + W_hr h + b_hr), z likewise, hn = W_hn h + b_hn, n = tanh(W_in x + b_in + r ⊙ hn)
struct RwGates {
    double r, z, n, hn;
};

MJX_D RwGates rw_gru_gates(const double* bih, const double* bhh, int H, int j, double gir, double giz, double gin, double ghr,
                           double ghz, double ghn) {
    RwGates G;
    G.r = rw_sigmoid(gir + MJX_LDG(bih + j) + ghr + MJX_LDG(bhh + j));
    G.z = rw_sigmoid(giz + MJX_LDG(bih + H + j) + ghz + MJX_LDG(bhh + H + j));
    G.hn = ghn + MJX_LDG(bhh + 2 * H + j);
    G.n = tanh(gin + MJX_LDG(bih + 2 * H + j) + G.r * G.hn);
    return G;
}

// layer k of the GRU, the new hidden state of unit j for every game (rw_gru_gates, h' = (1 − z) ⊙ n + z ⊙ h); returns the unit
// this thread writes, or -1. `gates` (optional) receives every game's gates of that unit.
MJX_D int rw_gru_compute(const GrpNet& n, const RwCta& C, int k, int tid, double (&hn)[RW_GAMES], RwGates* gates = nullptr) {
    const int H = n.H, hl = H * n.layers, in = n.in(k), ks = rw_slices(H), j = tid / ks, s = tid % ks;
    const double* wih = n.layer(k);
    const double* whh = wih + 3LL * H * in;
    const double* bih = whh + 3LL * H * H;
    const double* bhh = bih + 3 * H;
    const double* x = k ? C.h + (k - 1) * H : C.x;
    const int xs = k ? hl : 8;
    const double* h = C.h + k * H;
    double gi[3 * RW_GAMES] = {}, gh[3 * RW_GAMES] = {};
    if (j < H) {
        for (int c = s; c < in; c += ks)
            for (int q = 0; q < 3; q++) {
                const double w = MJX_LDG(wih + (long long)(q * H + j) * in + c);
                for (int g = 0; g < RW_GAMES; g++) gi[q * RW_GAMES + g] += w * x[g * xs + c];
            }
        for (int c = s; c < H; c += ks)
            for (int q = 0; q < 3; q++) {
                const double w = MJX_LDG(whh + (long long)(q * H + j) * H + c);
                for (int g = 0; g < RW_GAMES; g++) gh[q * RW_GAMES + g] += w * h[g * hl + c];
            }
    }
    rw_reduce(gi, ks);
    rw_reduce(gh, ks);
    if (j >= H || s) return -1;
    for (int g = 0; g < RW_GAMES; g++) {
        const RwGates G = rw_gru_gates(bih, bhh, H, j, gi[g], gi[RW_GAMES + g], gi[2 * RW_GAMES + g], gh[g], gh[RW_GAMES + g],
                                       gh[2 * RW_GAMES + g]);
        hn[g] = (1.0 - G.z) * G.n + G.z * h[g * hl + j];
        if (gates) gates[g] = G;
    }
    return j;
}

// after a barrier: the new hidden states of the games that have step t
MJX_D void rw_gru_write(const GrpNet& n, const RwCta& C, int k, int t, int j, const double (&hn)[RW_GAMES]) {
    if (j < 0) return;
    for (int g = 0; g < RW_GAMES; g++)
        if (t < C.len[g]) C.h[g * n.H * n.layers + k * n.H + j] = hn[g];
}

// s_y = ReLU(fc.0(s_h))
MJX_D void rw_fc0(const GrpNet& n, const RwCta& C, int tid) {
    const int hl = n.H * n.layers, ks = rw_slices(hl), s = tid % ks;
    const double* W = n.fc0();
    const double* b = W + (long long)hl * hl;
    for (int u0 = 0; u0 < hl; u0 += RW_THREADS / ks) {
        const int u = u0 + tid / ks;
        double a[RW_GAMES] = {};
        if (u < hl)
            for (int c = s; c < hl; c += ks) {
                const double w = MJX_LDG(W + (long long)u * hl + c);
                for (int g = 0; g < RW_GAMES; g++) a[g] += w * C.h[g * hl + c];
            }
        rw_reduce(a, ks);
        if (u < hl && !s)
            for (int g = 0; g < RW_GAMES; g++) {
                const double v = a[g] + MJX_LDG(b + u);
                C.y[g * hl + u] = v > 0.0 ? v : 0.0;
            }
    }
}

// s_lg = fc.2(s_y)
MJX_D void rw_fc2(const GrpNet& n, const RwCta& C, int tid) {
    const int hl = n.H * n.layers, ks = rw_slices(24), u = tid / ks, s = tid % ks;
    const double* W = n.fc2();
    double a[RW_GAMES] = {};
    if (u < 24)
        for (int c = s; c < hl; c += ks) {
            const double w = MJX_LDG(W + (long long)u * hl + c);
            for (int g = 0; g < RW_GAMES; g++) a[g] += w * C.y[g * hl + c];
        }
    rw_reduce(a, ks);
    if (u < 24 && !s)
        for (int g = 0; g < RW_GAMES; g++) C.lg[g * 24 + u] = a[g] + MJX_LDG(W + 24LL * hl + u);
}

// calc_matrix of one row, entry i = player * 4 + rank: the softmax over the 24 logits summed over the permutations p with
// p[player] == rank
MJX_D double rw_matrix_entry(const double* logits, int i) {
    double m = logits[0];
    for (int p = 1; p < 24; p++) m = logits[p] > m ? logits[p] : m;
    double sum = 0.0;
    for (int p = 0; p < 24; p++) sum += exp(logits[p] - m);
    double acc = 0.0;
    for (int p = 0; p < 24; p++)
        if (RW_PERMS[p][i >> 2] == (i & 3)) acc += exp(logits[p] - m) / sum;
    return acc;
}

// the 16 entries of every game with step t, one thread each
MJX_D void rw_out(const MatrixView& V, const RwCta& C, int t, int tid) {
    const int g = tid >> 4;
    if (g < RW_GAMES && t < C.len[g]) V.matrix[(C.lo[g] + t) * 16 + (tid & 15)] = rw_matrix_entry(C.lg + g * 24, tid & 15);
}

// ---------------------------------------------------------------- k_train_targets

struct TargetView {
    const double* feat;  // [n_rows, 7]
    const i32* game_off;  // [n_games + 1]
    long long n_rows;
    int n_games;
    const double* matrix;  // [n_rows, 4, 4]
    const u8* rank_by_player;  // [n_games, 4]
    const i64* final_scores;  // [n_games, 4]
    double pts[4];
    int uniform_init;
    const i32* move_off;  // [n_jobs + 1]
    long long n_moves;
    const i32* job_game;
    const u8* job_player;
    int n_jobs;
    const i32* at_kyoku;
    const u8 *apply_gamma, *dones;
    i64* steps_to_done;
    double* kyoku_reward;
    i64* player_rank;
    i32* status;
};

// exp_pts[k] = rank_prob[k] . pts over rank_prob = [matrix[0..L-1, pid]; one_hot(rank_final)], row 0 = 1/4 with uniform_init
MJX_D double rw_exp_pts(const TargetView& V, long long lo, int L, int pid, int rank_final, int k) {
    const double* p = V.pts;  // selected, not indexed, by rank_final: the view stays in registers
    if (k == L) return rank_final == 0 ? p[0] : rank_final == 1 ? p[1] : rank_final == 2 ? p[2] : p[3];
    if (k == 0 && V.uniform_init) return 0.25 * p[0] + 0.25 * p[1] + 0.25 * p[2] + 0.25 * p[3];
    const double* m = V.matrix + (lo + k) * 16 + pid * 4;
    return m[0] * p[0] + m[1] * p[1] + m[2] * p[2] + m[3] * p[3];
}

// the rank of seat pid in score row k of concat(feature[:, 3:] * 1e4, [final_scores]): the seats with a higher score plus the
// lower-numbered seats with an equal one, which is (-s).argsort(stable).argsort(stable)
MJX_D int rw_rank(const TargetView& V, long long lo, int L, int g, int pid, int k) {
    const auto score = [&](int q) { return k < L ? V.feat[(lo + k) * RW_IN + 3 + q] * 1e4 : (double)V.final_scores[4 * g + q]; };
    const double me = score(pid);
    int r = 0;
    for (int q = 0; q < 4; q++) {
        const double s = score(q);
        r += s > me || (q < pid && s == me);
    }
    return r;
}

// the targets of job j's moves -> mjx_reward_status (warp-uniform). CAPACITY writes nothing; KYOKU (an at_kyoku outside the game's
// rows) zeroes the job's outputs. steps_to_done[i] = 0 where dones[i], else steps_to_done[i + 1] + apply_gamma[i], with the move
// after the job's last counting as 0 (a Gameplay's last move is always done).
MJX_DM int rw_job(const TargetView& V, int j, int lane) {
#ifdef MJX_HOST_EMUL
    constexpr int LANES = 1;
#else
    constexpr int LANES = 32;
#endif
    const long long m0 = V.move_off[j], m1 = V.move_off[j + 1];
    const int g = V.job_game[j], pid = V.job_player[j];
    if (m0 < 0 || m0 > m1 || m1 > V.n_moves || g < 0 || g >= V.n_games || pid > 3 || !rw_game_ok(V.game_off, g, V.n_rows) ||
        V.rank_by_player[4 * g + pid] > 3)
        return MJX_REWARD_CAPACITY;
    const long long lo = V.game_off[g];
    const int L = (int)(V.game_off[g + 1] - lo), rf = V.rank_by_player[4 * g + pid];
    bool bad = false;
    for (long long i = m0 + lane; i < m1; i += LANES) bad |= V.at_kyoku[i] < 0 || V.at_kyoku[i] >= L;
#ifndef MJX_HOST_EMUL
    bad = __any_sync(~0u, bad);
#endif
    for (long long i = m0 + lane; i < m1; i += LANES) {
        const int k = V.at_kyoku[i];
        V.kyoku_reward[i] = bad ? 0.0 : rw_exp_pts(V, lo, L, pid, rf, k + 1) - rw_exp_pts(V, lo, L, pid, rf, k);
        V.player_rank[i] = bad ? 0 : rw_rank(V, lo, L, g, pid, k + 1);
    }
#ifdef MJX_HOST_EMUL
    i64 next = 0;
    for (long long i = m1 - 1; i >= m0; i--) {
        next = V.dones[i] ? 0 : next + (V.apply_gamma[i] != 0);
        V.steps_to_done[i] = bad ? 0 : next;
    }
#else
    // chunks of 32 moves from the end; a move is the map x -> done ? 0 : apply_gamma + x, kept as (reset, add); the backward
    // inclusive scan composes each lane's map with the later lanes' ones, and the carry is the value at the later chunk's first move
    i64 carry = 0;
    for (long long base = m1; base > m0; base -= 32) {
        const long long i = base - 32 + lane;
        const bool in = i >= m0;
        bool reset = in && V.dones[i];
        i64 add = in && !reset ? (V.apply_gamma[i] != 0) : 0;
        for (int o = 1; o < 32; o <<= 1) {
            const bool r2 = __shfl_down_sync(~0u, (int)reset, o);
            const i64 a2 = __shfl_down_sync(~0u, add, o);
            if (lane + o < 32 && !reset) {
                reset = r2;
                add += a2;
            }
        }
        const i64 v = reset ? add : add + carry;
        if (in) V.steps_to_done[i] = bad ? 0 : v;
        carry = __shfl_sync(~0u, v, 0);
    }
#endif
    return bad ? MJX_REWARD_KYOKU : MJX_REWARD_OK;
}

#ifndef MJX_HOST_EMUL
// k_grp_matrix: RW_GAMES games per CTA, stepped together (the file's top comment); dynamic shared memory rw_smem_doubles
__global__ void __launch_bounds__(RW_THREADS) k_grp_matrix(MatrixView V) {
    extern __shared__ double s_mem[];
    __shared__ long long s_lo[RW_GAMES];
    __shared__ int s_len[RW_GAMES];
    const RwCta C = rw_cta(V.net, s_mem, s_lo, s_len);
    const int tid = threadIdx.x;
    rw_begin(V, C, blockIdx.x, tid);
    __syncthreads();
    const int steps = rw_steps(C);
    for (int t = 0; t < steps; t++) {
        rw_load_x(V, C, t, tid);
        __syncthreads();
        for (int k = 0; k < V.net.layers; k++) {
            double hn[RW_GAMES];
            const int j = rw_gru_compute(V.net, C, k, tid, hn);
            __syncthreads();
            rw_gru_write(V.net, C, k, t, j, hn);
            __syncthreads();
        }
        rw_fc0(V.net, C, tid);
        __syncthreads();
        rw_fc2(V.net, C, tid);
        __syncthreads();
        rw_out(V, C, t, tid);
    }
}

// k_train_targets: one warp per job
__global__ void __launch_bounds__(RW_WARPS * 32) k_train_targets(TargetView V) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int j = blockIdx.x * RW_WARPS + warp;
    if (j >= V.n_jobs) return;
    const int st = rw_job(V, j, lane);
    if (lane == 0) V.status[j] = st;
}
#endif

}  // namespace mjx
