// TEST INFRASTRUCTURE ONLY — host build of mortal_b200/csrc/mjx_grp_train.cuh (-DMJX_HOST_EMUL): the phase functions of
// k_grp_train_fwd / head / bwd / wgrad / loss run for every thread id in turn between the barriers (one slice per dot product), so
// the GRP training step can be diffed against a torch restatement of the reference and run under sanitizers without a GPU.
// Never loaded by mortal_b200/. Part of libmjx_emul.so (tests/emul_lib.py); bound by tests/grp_train_lib.py.
#include <cstdint>
#include <vector>

#include "mjx_grp_train.cuh"

using namespace mjx;

extern "C" {

long long emult_scratch_bytes(int hidden, int layers, int n_samples, int n_jobs, int max_steps) {
    const long long b = rt_scratch_bytes(hidden, layers, n_samples, n_jobs, max_steps);
    return b < 0 ? MJX_ERR_ARG : b;
}

// mjx_grp_train_dev over host arrays: the same argument checks (returns -2 where they fail), then every CTA of every kernel in
// launch order
int emult_grp_train(int n_games, const double* feat, const int32_t* game_off, long long n_rows, const double* weights,
                    long long n_weights, int hidden, int layers, int n_samples, const int32_t* sample_game, const int32_t* sample_len,
                    const int64_t* rank_by_player, int n_jobs, const int32_t* job_game, const int32_t* job_steps,
                    const int32_t* sample_job, const int32_t* job_sample_off, const int32_t* job_sample, int max_steps, double* loss,
                    double* acc, double* grad, int32_t* sample_status, void* scratch, long long scratch_bytes) {
    if (rt_check_args(n_games, feat, game_off, n_rows, weights, n_weights, hidden, layers, n_samples, sample_game, sample_len,
                      rank_by_player, n_jobs, job_game, job_steps, sample_job, job_sample_off, job_sample, max_steps, loss, acc,
                      sample_status, scratch, scratch_bytes))
        return -2;
    TrainView V{};
    V.feat = feat; V.game_off = game_off; V.n_rows = n_rows; V.n_games = n_games; V.net = GrpNet{weights, hidden, layers};
    V.n_samples = n_samples; V.sample_game = sample_game; V.sample_len = sample_len; V.rank = rank_by_player;
    V.n_jobs = n_jobs; V.max_steps = max_steps; V.job_game = job_game; V.job_steps = job_steps; V.sample_job = sample_job;
    V.job_sample_off = job_sample_off; V.job_sample = job_sample; V.loss = loss; V.acc = acc; V.grad = grad; V.status = sample_status;
    V = rt_view(V, (double*)scratch);
    struct Hn { double v[RW_GAMES]; RwGates g[RW_GAMES]; };
    std::vector<Hn> hn(RT_THREADS);
    std::vector<int> unit(RT_THREADS);
    long long lo[RW_GAMES], row[RW_GAMES];
    int len[RW_GAMES], label[RW_GAMES];
    // k_grp_train_fwd
    std::vector<double> mem(rt_head_smem_doubles(hidden, layers));
    const MatrixView M = rt_matrix_view(V);
    for (int b = 0; b < (n_jobs + RW_GAMES - 1) / RW_GAMES; b++) {
        const RwCta C = rw_cta(V.net, mem.data(), lo, len);
        for (int tid = 0; tid < RT_THREADS; tid++) rt_fwd_begin(V, C, b, tid);
        const int steps = rw_steps(C);
        for (int t = 0; t < steps; t++) {
            for (int tid = 0; tid < RT_THREADS; tid++) rw_load_x(M, C, t, tid);
            for (int tid = 0; tid < RT_THREADS; tid++) rt_fwd_store_x(V, C, b, t, tid);
            for (int k = 0; k < layers; k++) {
                for (int tid = 0; tid < RT_THREADS; tid++) unit[tid] = rw_gru_compute(V.net, C, k, tid, hn[tid].v, hn[tid].g);
                for (int tid = 0; tid < RT_THREADS; tid++) {
                    rw_gru_write(V.net, C, k, t, unit[tid], hn[tid].v);
                    rt_fwd_store(V, C, b, k, t, unit[tid], hn[tid].v, hn[tid].g);
                }
            }
        }
    }
    // k_grp_train_head
    for (int b = 0; b < (n_samples + RW_GAMES - 1) / RW_GAMES; b++) {
        const RwCta C = rw_cta(V.net, mem.data(), lo, len);
        double* s_dlog = mem.data() + rw_smem_doubles(hidden, layers);
        double* s_dy = s_dlog + RW_GAMES * 24;
        for (int tid = 0; tid < RT_THREADS; tid++) rt_head_begin(V, b, tid, row, label);
        for (int tid = 0; tid < RT_THREADS; tid++) rt_head_gather(V, C, row, tid);
        for (int tid = 0; tid < RT_THREADS; tid++) rw_fc0(V.net, C, tid);
        for (int tid = 0; tid < RT_THREADS; tid++) rw_fc2(V.net, C, tid);
        for (int tid = 0; tid < RT_THREADS; tid++) rt_head_loss(V, C, row, label, s_dlog, b, tid);
        if (!grad) continue;
        for (int tid = 0; tid < RT_THREADS; tid++) rt_head_dy(V, C, row, s_dlog, s_dy, b, tid);
        for (int tid = 0; tid < RT_THREADS; tid++) rt_head_dx(V, s_dy, b, tid);
    }
    if (grad) {
        // k_grp_train_bwd
        std::vector<double> bm(rt_bwd_smem_doubles(hidden, layers));
        struct A2 { double v[2]; };
        std::vector<A2> a(RT_THREADS);
        for (int j = 0; j < n_jobs; j++) {
            const RtBwd S = rt_bwd_cta(V.net, bm.data());
            int steps = 0;
            for (int tid = 0; tid < RT_THREADS; tid++) steps = rt_bwd_begin(V, S, j, tid);
            for (int t = steps - 1; t >= 0; t--)
                for (int k = layers - 1; k >= 0; k--) {
                    for (int tid = 0; tid < RT_THREADS; tid++) rt_bwd_cell(V, S, j, t, k, tid);
                    for (int tid = 0; tid < RT_THREADS; tid++) unit[tid] = rt_bwd_mat(V, S, k, tid, a[tid].v);
                    for (int tid = 0; tid < RT_THREADS; tid++) rt_bwd_write(V, S, k, unit[tid], a[tid].v);
                }
        }
        // k_grp_train_wgrad
        const RtWgrad W = rt_wgrad_segs(V);
        std::vector<double> sA(RT_CHUNK * RT_TILE), sB(RT_CHUNK * RT_TILE), acc(RT_THREADS);
        for (int tile = 0; tile < W.n_tiles; tile++) {
            int m0, n0;
            const RtSeg& g = rt_tile(W, tile, m0, n0);
            for (int tid = 0; tid < RT_THREADS; tid++) acc[tid] = 0.0;
            for (long long r = g.lag; r < g.rows; r += RT_CHUNK) {
                for (int tid = 0; tid < RT_THREADS; tid++) rt_wgrad_load(g, m0, n0, r, tid, sA.data(), sB.data());
                for (int tid = 0; tid < RT_THREADS; tid++) rt_wgrad_acc(tid, sA.data(), sB.data(), acc[tid]);
            }
            for (int tid = 0; tid < RT_THREADS; tid++) rt_wgrad_store(g, m0, n0, tid, acc[tid]);
        }
    }
    // k_grp_train_loss
    std::vector<double> red(2 * RT_THREADS);
    for (int tid = 0; tid < RT_THREADS; tid++) rt_loss_part(V, red.data(), tid);
    for (int w = RT_THREADS / 2; w > 0; w >>= 1)
        for (int tid = 0; tid < RT_THREADS; tid++) rt_loss_tree(red.data(), w, tid);
    rt_loss_out(V, red.data(), 0);
    return 0;
}

}  // extern "C"
