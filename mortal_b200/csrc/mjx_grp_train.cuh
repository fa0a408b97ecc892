// mortal_b200 — GRP training step: the loss, accuracy and exact gradient of mortal/train_grp.py:172-186 (GRP.forward_packed of
// model.py:233-286 over a batch of game prefixes, get_label, F.cross_entropy, loss.backward()) without the prefix lists.
//
// A batch is B samples (game, prefix length len, rank_by_player). A GRU is causal and starts from h0 = 0, so the h_n of the prefix
// feature[:len] is the hidden state after step len - 1 of one pass over the game (k_grp_matrix's observation). The samples are
// grouped by game into jobs; a job is its game stepped up to the longest prefix its samples ask for. The loss is a sum over
// samples, and the samples of one job differ only in the step where their head gradient enters, so one reverse pass per job
// with each sample's dL/dh_n added at its last step gives the exact gradient of the batch.
//
//   k_grp_train_fwd    RW_GAMES jobs per CTA, stepped together with k_grp_matrix's phase functions (rw_load_x, rw_gru_compute,
//                      rw_gru_write); stores per (job, step, layer) the new h and the gates r, z, n, hn = W_hn h + b_hn, and the
//                      step's feature row.
//   k_grp_train_head   RW_GAMES samples per CTA: h_n of the sample's last step (layer 0 first), fc.0 / ReLU / fc.2 (rw_fc0,
//                      rw_fc2), log-softmax, cross-entropy, argmax; with gradients dlogits = (softmax - onehot) / B through the
//                      head to dL/dh_n.
//   k_grp_train_bwd    one job per CTA, t = T-1 .. 0, layers top down: dh = the carry from step t + 1 + dx from the layer above +
//                      the injections of the job's samples that end at t; torch's cell adjoints; stores the gate pre-activation
//                      adjoints (da_r, da_z, da_n, d hn) per (job, step, layer).
//   k_grp_train_wgrad  every weight and bias gradient as C = A^T B over stored rows; each CTA owns a 16 x 16 output tile and sums
//                      its rows in ascending order, staged through shared memory 32 rows at a time.
//   k_grp_train_loss   one CTA: the loss and accuracy sums in a fixed order.
// No atomics and fixed reduction orders: the same batch and weights give bit-identical results.
//
// Scratch rows: job j owns rows [j (T + 1), (j + 1)(T + 1)), T = max_steps; the first is a zero row (the h_prev of step 0, so the
// hidden-weight gradient reads row r - 1), step t is row j (T + 1) + 1 + t. Rows no valid step writes are zero, so the gradient
// kernel sums every row without looking at the jobs.
//
// -DMJX_HOST_EMUL builds the same phase functions for a host loop over the thread ids (tests/host_emul/emul_grp_train.cc).
#pragma once
#include "mjx_reward.cuh"

namespace mjx {

constexpr int RT_THREADS = RW_THREADS;
constexpr int RT_TILE = 16, RT_CHUNK = 32;  // k_grp_train_wgrad: output tile edge, rows staged per pass
constexpr int RT_MAX_SEGS = 4 * RW_MAX_LAYERS + 4;

// the scratch arrays (doubles), R = n_jobs * (max_steps + 1) rows, HL = hidden * layers
struct RtLayout {
    long long x0, hs, gates, dpre, xh, y, dy, dxh, dlog, lossb, hit, total;
};

MJX_HD RtLayout rt_layout(int H, int layers, int n_samples, int n_jobs, int max_steps) {
    const long long R = (long long)n_jobs * (max_steps + 1), LH = (long long)layers * H, B = n_samples;
    RtLayout s;
    s.x0 = 0;
    s.hs = s.x0 + R * 8;
    s.gates = s.hs + R * LH;
    s.dpre = s.gates + R * LH * 4;
    s.xh = s.dpre + R * LH * 4;
    s.y = s.xh + B * LH;
    s.dy = s.y + B * LH;
    s.dxh = s.dy + B * LH;
    s.dlog = s.dxh + B * LH;
    s.lossb = s.dlog + B * 24;
    s.hit = s.lossb + B;
    s.total = s.hit + B;
    return s;
}

// the counts mjx_grp_train_dev takes; the scratch bytes they need, or -1
MJX_HD long long rt_scratch_bytes(int H, int layers, int n_samples, int n_jobs, int max_steps) {
    if (H < 1 || H > RW_MAX_H || layers < 1 || layers > RW_MAX_LAYERS || n_samples < 1 || n_samples > (1 << 24) || n_jobs < 1 ||
        n_jobs > n_samples || max_steps < 1 || max_steps > (1 << 16))
        return -1;
    return rt_layout(H, layers, n_samples, n_jobs, max_steps).total * (long long)sizeof(double);
}

// mjx_grp_train_dev's argument checks (host): MJX_OK or MJX_ERR_ARG
inline int rt_check_args(int n_games, const void* feat, const void* game_off, long long n_rows, const void* weights,
                         long long n_weights, int hidden, int layers, int n_samples, const void* sample_game, const void* sample_len,
                         const void* rank_by_player, int n_jobs, const void* job_game, const void* job_steps, const void* sample_job,
                         const void* job_sample_off, const void* job_sample, int max_steps, const void* loss, const void* acc,
                         const void* status, const void* scratch, long long scratch_bytes) {
    if (n_games <= 0 || !game_off || n_rows <= 0 || !feat || n_rows > (1LL << 31) - 1) return MJX_ERR_ARG;
    if (hidden < 1 || hidden > RW_MAX_H || layers < 1 || layers > RW_MAX_LAYERS || !weights ||
        n_weights != rw_weight_count(hidden, layers))
        return MJX_ERR_ARG;
    const long long need = rt_scratch_bytes(hidden, layers, n_samples, n_jobs, max_steps);
    if (need < 0 || !scratch || scratch_bytes < need) return MJX_ERR_ARG;
    if (!sample_game || !sample_len || !rank_by_player || !job_game || !job_steps || !sample_job || !job_sample_off || !job_sample ||
        !loss || !acc || !status)
        return MJX_ERR_ARG;
    return MJX_OK;
}

struct TrainView {
    const double* feat;   // [n_rows, 7]
    const i32* game_off;  // [n_games + 1]
    long long n_rows;
    int n_games;
    GrpNet net;
    int n_samples;
    const i32 *sample_game, *sample_len;  // [B]
    const i64* rank;                      // [B, 4]
    int n_jobs, max_steps;
    const i32 *job_game, *job_steps;         // [n_jobs]
    const i32* sample_job;                   // [B]
    const i32 *job_sample_off, *job_sample;  // [n_jobs + 1], [B]
    double *loss, *acc, *grad;               // grad: null = forward only
    i32* status;                             // [B] mjx_grp_train_status
    double *x0, *hs, *gates, *dpre, *xh, *y, *dy, *dxh, *dlog, *lossb, *hit;
};

MJX_HD TrainView rt_view(TrainView V, double* scratch) {
    const RtLayout s = rt_layout(V.net.H, V.net.layers, V.n_samples, V.n_jobs, V.max_steps);
    V.x0 = scratch + s.x0; V.hs = scratch + s.hs; V.gates = scratch + s.gates; V.dpre = scratch + s.dpre; V.xh = scratch + s.xh;
    V.y = scratch + s.y; V.dy = scratch + s.dy; V.dxh = scratch + s.dxh; V.dlog = scratch + s.dlog; V.lossb = scratch + s.lossb;
    V.hit = scratch + s.hit;
    return V;
}

MJX_D long long rt_row(const TrainView& V, int j, int t) { return (long long)j * (V.max_steps + 1) + 1 + t; }

// the steps of job j, or 0 when the job, its game or its step count is out of range
MJX_D int rt_job_steps(const TrainView& V, int j) {
    if (j < 0 || j >= V.n_jobs) return 0;
    const int g = V.job_game[j], s = V.job_steps[j];
    if (g < 0 || g >= V.n_games || !rw_game_ok(V.game_off, g, V.n_rows)) return 0;
    const long long L = V.game_off[g + 1] - V.game_off[g];
    return s >= 1 && s <= L && s <= V.max_steps ? s : 0;
}

// sample b's status; `row` = the scratch row of its last step when OK
MJX_D int rt_sample(const TrainView& V, int b, long long& row) {
    const int j = V.sample_job[b];
    const int s = rt_job_steps(V, j);
    if (s == 0 || V.sample_game[b] != V.job_game[j]) return MJX_GRP_TRAIN_GAME;
    const int len = V.sample_len[b];
    if (len < 1 || len > s) return MJX_GRP_TRAIN_LEN;
    row = rt_row(V, j, len - 1);
    return MJX_GRP_TRAIN_OK;
}

// model.py get_label: the index of rank_by_player in itertools.permutations(range(4)), 0 for a row that is no permutation
MJX_D int rt_label(const i64* rank) {
    for (int p = 0; p < 24; p++)
        if (rank[0] == RW_PERMS[p][0] && rank[1] == RW_PERMS[p][1] && rank[2] == RW_PERMS[p][2] && rank[3] == RW_PERMS[p][3])
            return p;
    return 0;
}

// ---------------------------------------------------------------- k_grp_train_fwd

MJX_D MatrixView rt_matrix_view(const TrainView& V) {
    MatrixView M;
    M.feat = V.feat; M.game_off = V.game_off; M.n_rows = V.n_rows; M.n_games = V.n_games; M.net = V.net; M.matrix = nullptr;
    return M;
}

// the CTA's jobs (an invalid job has no steps), zero hidden states, and zero scratch rows of its jobs
MJX_D void rt_fwd_begin(const TrainView& V, const RwCta& C, int block, int tid) {
    if (tid < RW_GAMES) {
        const int j = block * RW_GAMES + tid;
        const int s = rt_job_steps(V, j);
        C.lo[tid] = s ? V.game_off[V.job_game[j]] : 0;
        C.len[tid] = s;
    }
    const int LH = V.net.H * V.net.layers;
    for (int i = tid; i < RW_GAMES * LH; i += RT_THREADS) C.h[i] = 0.0;
    const int j0 = block * RW_GAMES, nj = V.n_jobs - j0 < RW_GAMES ? V.n_jobs - j0 : RW_GAMES;
    const long long r0 = (long long)j0 * (V.max_steps + 1), nr = (long long)nj * (V.max_steps + 1);
    for (long long i = tid; i < nr * 8; i += RT_THREADS) V.x0[r0 * 8 + i] = 0.0;
    for (long long i = tid; i < nr * LH; i += RT_THREADS) V.hs[r0 * LH + i] = 0.0;
    for (long long i = tid; i < nr * LH * 4; i += RT_THREADS) V.gates[r0 * LH * 4 + i] = 0.0;
}

// the step's feature rows (after rw_load_x and a barrier)
MJX_D void rt_fwd_store_x(const TrainView& V, const RwCta& C, int block, int t, int tid) {
    if (tid < RW_GAMES * RW_IN) {
        const int g = tid / RW_IN, c = tid % RW_IN;
        if (t < C.len[g]) V.x0[rt_row(V, block * RW_GAMES + g, t) * 8 + c] = C.x[g * 8 + c];
    }
}

// unit j's new h and gates of layer k at step t, for the CTA's jobs that have step t
MJX_D void rt_fwd_store(const TrainView& V, const RwCta& C, int block, int k, int t, int j, const double (&hn)[RW_GAMES],
                        const RwGates (&G)[RW_GAMES]) {
    if (j < 0) return;
    const int H = V.net.H, layers = V.net.layers;
    for (int g = 0; g < RW_GAMES; g++) {
        if (t >= C.len[g]) continue;
        const long long rk = rt_row(V, block * RW_GAMES + g, t) * layers + k;
        V.hs[rk * H + j] = hn[g];
        double* q = V.gates + rk * 4 * H + j;
        q[0] = G[g].r; q[H] = G[g].z; q[2 * H] = G[g].n; q[3 * H] = G[g].hn;
    }
}

// ---------------------------------------------------------------- k_grp_train_head

// doubles of k_grp_train_head's dynamic shared memory: k_grp_matrix's, then dlogits [RW_GAMES][24] and dy [RW_GAMES][HL]
MJX_HD int rt_head_smem_doubles(int H, int layers) { return rw_smem_doubles(H, layers) + RW_GAMES * (24 + H * layers); }

// the CTA's samples: status, the scratch row of the last step (-1 for none), the label; then their h_n into s_h
MJX_D void rt_head_begin(const TrainView& V, int block, int tid, long long* row, int* label) {
    if (tid < RW_GAMES) {
        const int b = block * RW_GAMES + tid;
        row[tid] = -1;
        label[tid] = 0;
        if (b < V.n_samples) {
            long long r = -1;
            const int st = rt_sample(V, b, r);
            V.status[b] = st;
            if (st == MJX_GRP_TRAIN_OK) row[tid] = r;
            label[tid] = rt_label(V.rank + 4LL * b);
        }
    }
}

MJX_D void rt_head_gather(const TrainView& V, const RwCta& C, const long long* row, int tid) {
    const int LH = V.net.H * V.net.layers;
    for (int i = tid; i < RW_GAMES * LH; i += RT_THREADS) {
        const int g = i / LH, c = i % LH;
        C.h[i] = row[g] >= 0 ? V.hs[row[g] * LH + c] : 0.0;  // hs rows are [layer][H]: h_n.transpose(0, 1).flatten(1)
    }
}

// one thread per sample: log-softmax, cross-entropy, argmax (first maximum); with gradients dlogits = (softmax - onehot) / B
MJX_D void rt_head_loss(const TrainView& V, const RwCta& C, const long long* row, const int* label, double* s_dlog, int block,
                        int tid) {
    if (tid >= RW_GAMES) return;
    const int b = block * RW_GAMES + tid;
    if (b >= V.n_samples) return;
    const double* lg = C.lg + tid * 24;
    double* d = s_dlog + tid * 24;
    if (row[tid] < 0) {
        V.lossb[b] = 0.0;
        V.hit[b] = 0.0;
        for (int u = 0; u < 24; u++) d[u] = 0.0;
    } else {
        double m = lg[0];
        int am = 0;
        for (int u = 1; u < 24; u++)
            if (lg[u] > m) m = lg[u], am = u;
        double sum = 0.0;
        for (int u = 0; u < 24; u++) sum += exp(lg[u] - m);
        const double lse = log(sum);
        V.lossb[b] = -((lg[label[tid]] - m) - lse);
        V.hit[b] = am == label[tid] ? 1.0 : 0.0;
        const double inv_b = 1.0 / V.n_samples;
        for (int u = 0; u < 24; u++) d[u] = (exp(lg[u] - m) / sum - (u == label[tid] ? 1.0 : 0.0)) * inv_b;
    }
    if (V.grad)
        for (int u = 0; u < 24; u++) V.dlog[b * 24LL + u] = d[u];
}

// dL/d(fc.0 pre-activation) = (y > 0) ⊙ fc.2.weight^T dlogits; stores the head rows the weight gradient reads
MJX_D void rt_head_dy(const TrainView& V, const RwCta& C, const long long* row, const double* s_dlog, double* s_dy, int block,
                      int tid) {
    const int LH = V.net.H * V.net.layers;
    const double* W2 = V.net.fc2();
    for (int i = tid; i < RW_GAMES * LH; i += RT_THREADS) {
        const int g = i / LH, c = i % LH, b = block * RW_GAMES + g;
        double a = 0.0;
        for (int u = 0; u < 24; u++) a += MJX_LDG(W2 + (long long)u * LH + c) * s_dlog[g * 24 + u];
        const bool ok = row[g] >= 0;
        const double dy = ok && C.y[i] > 0.0 ? a : 0.0;
        s_dy[i] = dy;
        if (b < V.n_samples) {
            V.xh[(long long)b * LH + c] = C.h[i];
            V.y[(long long)b * LH + c] = ok ? C.y[i] : 0.0;
            V.dy[(long long)b * LH + c] = dy;
        }
    }
}

// dL/dh_n = fc.0.weight^T dy: the injection of the sample's last step, every layer
MJX_D void rt_head_dx(const TrainView& V, const double* s_dy, int block, int tid) {
    const int LH = V.net.H * V.net.layers;
    const double* W0 = V.net.fc0();
    for (int i = tid; i < RW_GAMES * LH; i += RT_THREADS) {
        const int g = i / LH, c = i % LH, b = block * RW_GAMES + g;
        if (b >= V.n_samples) continue;
        double a = 0.0;
        for (int u = 0; u < LH; u++) a += MJX_LDG(W0 + (long long)u * LH + c) * s_dy[g * LH + u];
        V.dxh[(long long)b * LH + c] = a;
    }
}

// ---------------------------------------------------------------- k_grp_train_bwd

// k_grp_train_bwd's shared state: the carried dh of every layer, dx from the layer above, the unit adjoints of the current
// (step, layer): da_r, da_z, da_n, d hn, and z ⊙ dh
struct RtBwd {
    double *dh, *dx, *d, *zd;
};

MJX_HD int rt_bwd_smem_doubles(int H, int layers) { return H * layers + H + 4 * H + H; }

MJX_D RtBwd rt_bwd_cta(const GrpNet& n, double* mem) {
    const int H = n.H;
    return RtBwd{mem, mem + H * n.layers, mem + H * n.layers + H, mem + H * n.layers + 5 * H};
}

// zero the job's adjoint rows and the carried dh -> the job's steps
MJX_D int rt_bwd_begin(const TrainView& V, const RtBwd& S, int j, int tid) {
    const int LH = V.net.H * V.net.layers;
    const long long r0 = (long long)j * (V.max_steps + 1), nr = V.max_steps + 1;
    for (long long i = tid; i < nr * LH * 4; i += RT_THREADS) V.dpre[r0 * LH * 4 + i] = 0.0;
    for (int i = tid; i < LH; i += RT_THREADS) S.dh[i] = 0.0;
    return rt_job_steps(V, j);
}

// one thread per unit u: dh = carry + dx of the layer above + the injections of the job's samples ending at step t; torch's
// cell adjoints (h' = (1 - z) n + z h, n = tanh(a_n), a_n = gi_n + r hn, r = σ(a_r), z = σ(a_z))
MJX_D void rt_bwd_cell(const TrainView& V, const RtBwd& S, int j, int t, int k, int tid) {
    const int H = V.net.H, layers = V.net.layers, LH = H * layers;
    if (tid >= H) return;
    const int u = tid;
    const long long row = rt_row(V, j, t);
    double g = S.dh[k * H + u];
    if (k < layers - 1) g += S.dx[u];
    int p0 = V.job_sample_off[j], p1 = V.job_sample_off[j + 1];
    p0 = p0 < 0 ? 0 : p0 > V.n_samples ? V.n_samples : p0;
    p1 = p1 < p0 ? p0 : p1 > V.n_samples ? V.n_samples : p1;
    for (int p = p0; p < p1; p++) {
        const int b = V.job_sample[p];
        long long rb = -1;
        if (b < 0 || b >= V.n_samples || V.sample_job[b] != j || rt_sample(V, b, rb) != MJX_GRP_TRAIN_OK || rb != row) continue;
        g += V.dxh[(long long)b * LH + k * H + u];
    }
    const long long rk = row * layers + k;
    const double* q = V.gates + rk * 4 * H + u;
    const double r = q[0], z = q[H], n = q[2 * H], hn = q[3 * H];
    const double hp = V.hs[(rk - layers) * H + u];  // step t - 1 of the layer; the job's zero row before step 0
    const double dn = g * (1.0 - z), dz = g * (hp - n);
    const double dan = dn * (1.0 - n * n);
    const double dar = dan * hn * (r * (1.0 - r)), daz = dz * (z * (1.0 - z)), dhn = dan * r;
    S.d[u] = dar; S.d[H + u] = daz; S.d[2 * H + u] = dan; S.d[3 * H + u] = dhn;
    S.zd[u] = g * z;
    double* o = V.dpre + rk * 4 * H + u;
    o[0] = dar; o[H] = daz; o[2 * H] = dan; o[3 * H] = dhn;
}

// after a barrier: dh_prev = z ⊙ dh + W_hh^T (da_r, da_z, d hn) -> the carry; dx = W_ih^T (da_r, da_z, da_n) -> the layer below.
// Output c is split over ks adjacent lanes, as in k_grp_matrix. Returns the unit this thread writes, or -1.
MJX_D int rt_bwd_mat(const TrainView& V, const RtBwd& S, int k, int tid, double (&a)[2]) {
    const GrpNet& n = V.net;
    const int H = n.H, ks = rw_slices(H), c = tid / ks, s = tid % ks;
    const double* wih = n.layer(k);
    const double* whh = wih + 3LL * H * n.in(k);
    a[0] = a[1] = 0.0;
    if (c < H)
        for (int m = s; m < 3 * H; m += ks) {
            a[0] += MJX_LDG(whh + (long long)m * H + c) * S.d[m < 2 * H ? m : m + H];
            if (k) a[1] += MJX_LDG(wih + (long long)m * H + c) * S.d[m];
        }
    rw_reduce(a, ks);
    return c < H && !s ? c : -1;
}

// after another barrier
MJX_D void rt_bwd_write(const TrainView& V, const RtBwd& S, int k, int c, const double (&a)[2]) {
    if (c < 0) return;
    S.dh[k * V.net.H + c] = S.zd[c] + a[0];
    if (k) S.dx[c] = a[1];
}

// ---------------------------------------------------------------- k_grp_train_wgrad

// one gradient: out[m][n] = sum over rows r >= lag of A[r][m] * B[r - lag][n] (B = null: 1, a bias); A's columns from a_split on
// are read a_skip further on (W_hh's n rows take the d hn adjoints)
struct RtSeg {
    const double* a;
    const double* b;
    double* out;
    long long rows;
    int lda, ldb, M, N, a_split, a_skip, lag, tile0;
};

struct RtWgrad {
    RtSeg seg[RT_MAX_SEGS];
    int n_seg, n_tiles;
};

MJX_HD int rt_seg_tiles(const RtSeg& s) { return ((s.M + RT_TILE - 1) / RT_TILE) * ((s.N + RT_TILE - 1) / RT_TILE); }

// the gradient segments of the net: per layer W_ih, W_hh, b_ih, b_hh; fc.0 weight and bias; fc.2 weight and bias
inline RtWgrad rt_wgrad_segs(const TrainView& V) {
    RtWgrad W{};
    const int H = V.net.H, layers = V.net.layers, LH = H * layers;
    const long long R = (long long)V.n_jobs * (V.max_steps + 1);
    const GrpNet G{V.grad, H, layers};
    auto add = [&](const double* a, int lda, int M, int split, int skip, const double* b, int ldb, int N, int lag, long long rows,
                   double* out) {
        RtSeg s{a, b, out, rows, lda, ldb, M, N, split, skip, lag, W.n_tiles};
        W.n_tiles += rt_seg_tiles(s);
        W.seg[W.n_seg++] = s;
    };
    for (int k = 0; k < layers; k++) {
        const double* A = V.dpre + 4LL * H * k;
        const double* X = k ? V.hs + (long long)(k - 1) * H : V.x0;
        const int in = G.in(k);
        double* o = const_cast<double*>(G.layer(k));
        add(A, 4 * LH, 3 * H, 3 * H, 0, X, k ? LH : 8, in, 0, R, o);
        add(A, 4 * LH, 3 * H, 2 * H, H, V.hs + (long long)k * H, LH, H, 1, R, o + 3LL * H * in);
        add(A, 4 * LH, 3 * H, 3 * H, 0, nullptr, 0, 1, 0, R, o + 3LL * H * (in + H));
        add(A, 4 * LH, 3 * H, 2 * H, H, nullptr, 0, 1, 0, R, o + 3LL * H * (in + H) + 3 * H);
    }
    double* f0 = const_cast<double*>(G.fc0());
    double* f2 = const_cast<double*>(G.fc2());
    add(V.dy, LH, LH, LH, 0, V.xh, LH, LH, 0, V.n_samples, f0);
    add(V.dy, LH, LH, LH, 0, nullptr, 0, 1, 0, V.n_samples, f0 + (long long)LH * LH);
    add(V.dlog, 24, 24, 24, 0, V.y, LH, LH, 0, V.n_samples, f2);
    add(V.dlog, 24, 24, 24, 0, nullptr, 0, 1, 0, V.n_samples, f2 + 24LL * LH);
    return W;
}

// the CTA's tile: segment, first output row and column
MJX_D const RtSeg& rt_tile(const RtWgrad& W, int tile, int& m0, int& n0) {
    int s = 0;
    while (s + 1 < W.n_seg && W.seg[s + 1].tile0 <= tile) s++;
    const RtSeg& g = W.seg[s];
    const int tn = (g.N + RT_TILE - 1) / RT_TILE, i = tile - g.tile0;
    m0 = (i / tn) * RT_TILE;
    n0 = (i % tn) * RT_TILE;
    return g;
}

// stage rows [r, r + RT_CHUNK) of the tile's A and B columns
MJX_D void rt_wgrad_load(const RtSeg& g, int m0, int n0, long long r, int tid, double* sA, double* sB) {
    for (int e = tid; e < RT_CHUNK * RT_TILE; e += RT_THREADS) {
        const int rr = e / RT_TILE, cc = e % RT_TILE;
        const long long row = r + rr;
        const int m = m0 + cc, n = n0 + cc;
        const bool in = row < g.rows;
        sA[e] = in && m < g.M ? g.a[row * g.lda + (m < g.a_split ? m : m + g.a_skip)] : 0.0;
        sB[e] = !in || n >= g.N ? 0.0 : g.b ? g.b[(row - g.lag) * g.ldb + n] : 1.0;
    }
}

MJX_D void rt_wgrad_acc(int tid, const double* sA, const double* sB, double& acc) {
    const int i = tid / RT_TILE, jj = tid % RT_TILE;
    for (int rr = 0; rr < RT_CHUNK; rr++) acc += sA[rr * RT_TILE + i] * sB[rr * RT_TILE + jj];
}

MJX_D void rt_wgrad_store(const RtSeg& g, int m0, int n0, int tid, double acc) {
    const int m = m0 + tid / RT_TILE, n = n0 + tid % RT_TILE;
    if (m < g.M && n < g.N) g.out[(long long)m * g.N + n] = acc;
}

// ---------------------------------------------------------------- k_grp_train_loss

// thread tid's share of the loss and hit sums (ascending samples), then a fixed tree over the threads in s_red [2][RT_THREADS]
MJX_D void rt_loss_part(const TrainView& V, double* s_red, int tid) {
    double l = 0.0, h = 0.0;
    for (int b = tid; b < V.n_samples; b += RT_THREADS) l += V.lossb[b], h += V.hit[b];
    s_red[tid] = l;
    s_red[RT_THREADS + tid] = h;
}

MJX_D void rt_loss_tree(double* s_red, int w, int tid) {
    if (tid < w) {
        s_red[tid] += s_red[tid + w];
        s_red[RT_THREADS + tid] += s_red[RT_THREADS + tid + w];
    }
}

MJX_D void rt_loss_out(const TrainView& V, const double* s_red, int tid) {
    if (tid == 0) {
        *V.loss = s_red[0] / V.n_samples;
        *V.acc = s_red[RT_THREADS] / V.n_samples;
    }
}

#ifndef MJX_HOST_EMUL
__global__ void __launch_bounds__(RT_THREADS) k_grp_train_fwd(TrainView V) {
    extern __shared__ double s_mem[];
    __shared__ long long s_lo[RW_GAMES];
    __shared__ int s_len[RW_GAMES];
    const RwCta C = rw_cta(V.net, s_mem, s_lo, s_len);
    const MatrixView M = rt_matrix_view(V);
    const int tid = threadIdx.x, block = blockIdx.x;
    rt_fwd_begin(V, C, block, tid);
    __syncthreads();
    const int steps = rw_steps(C);
    for (int t = 0; t < steps; t++) {
        rw_load_x(M, C, t, tid);
        __syncthreads();
        rt_fwd_store_x(V, C, block, t, tid);
        for (int k = 0; k < V.net.layers; k++) {
            double hn[RW_GAMES];
            RwGates G[RW_GAMES];
            const int j = rw_gru_compute(V.net, C, k, tid, hn, G);
            __syncthreads();
            rw_gru_write(V.net, C, k, t, j, hn);
            rt_fwd_store(V, C, block, k, t, j, hn, G);
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(RT_THREADS) k_grp_train_head(TrainView V) {
    extern __shared__ double s_mem[];
    __shared__ long long s_lo[RW_GAMES], s_row[RW_GAMES];
    __shared__ int s_len[RW_GAMES], s_label[RW_GAMES];
    const RwCta C = rw_cta(V.net, s_mem, s_lo, s_len);
    double* s_dlog = s_mem + rw_smem_doubles(V.net.H, V.net.layers);
    double* s_dy = s_dlog + RW_GAMES * 24;
    const int tid = threadIdx.x, block = blockIdx.x;
    rt_head_begin(V, block, tid, s_row, s_label);
    __syncthreads();
    rt_head_gather(V, C, s_row, tid);
    __syncthreads();
    rw_fc0(V.net, C, tid);
    __syncthreads();
    rw_fc2(V.net, C, tid);
    __syncthreads();
    rt_head_loss(V, C, s_row, s_label, s_dlog, block, tid);
    if (!V.grad) return;
    __syncthreads();
    rt_head_dy(V, C, s_row, s_dlog, s_dy, block, tid);
    __syncthreads();
    rt_head_dx(V, s_dy, block, tid);
}

__global__ void __launch_bounds__(RT_THREADS) k_grp_train_bwd(TrainView V) {
    extern __shared__ double s_mem[];
    const RtBwd S = rt_bwd_cta(V.net, s_mem);
    const int tid = threadIdx.x, j = blockIdx.x;
    const int steps = rt_bwd_begin(V, S, j, tid);
    __syncthreads();
    for (int t = steps - 1; t >= 0; t--)
        for (int k = V.net.layers - 1; k >= 0; k--) {
            rt_bwd_cell(V, S, j, t, k, tid);
            __syncthreads();
            double a[2];
            const int c = rt_bwd_mat(V, S, k, tid, a);
            __syncthreads();
            rt_bwd_write(V, S, k, c, a);
            __syncthreads();
        }
}

__global__ void __launch_bounds__(RT_THREADS) k_grp_train_wgrad(RtWgrad W) {
    __shared__ double sA[RT_CHUNK * RT_TILE], sB[RT_CHUNK * RT_TILE];
    const int tid = threadIdx.x;
    int m0, n0;
    const RtSeg& g = rt_tile(W, blockIdx.x, m0, n0);
    double acc = 0.0;
    for (long long r = g.lag; r < g.rows; r += RT_CHUNK) {
        rt_wgrad_load(g, m0, n0, r, tid, sA, sB);
        __syncthreads();
        rt_wgrad_acc(tid, sA, sB, acc);
        __syncthreads();
    }
    rt_wgrad_store(g, m0, n0, tid, acc);
}

__global__ void __launch_bounds__(RT_THREADS) k_grp_train_loss(TrainView V) {
    __shared__ double s_red[2 * RT_THREADS];
    const int tid = threadIdx.x;
    rt_loss_part(V, s_red, tid);
    __syncthreads();
    for (int w = RT_THREADS / 2; w > 0; w >>= 1) {
        rt_loss_tree(s_red, w, tid);
        __syncthreads();
    }
    rt_loss_out(V, s_red, tid);
}
#endif

}  // namespace mjx
