// TEST INFRASTRUCTURE ONLY — host build of mortal_b200/csrc/mjx_reward.cuh (-DMJX_HOST_EMUL): k_grp_matrix's phase functions
// run for every thread id in turn between the barriers (one slice per dot product), and k_train_targets's per-job work for one
// lane, so the GRP rewards can be diffed against a torch restatement of the reference and run under sanitizers without a GPU.
// Never loaded by mortal_b200/. Part of libmjx_emul.so (tests/emul_lib.py); bound by tests/reward_lib.py.
#include <cstdint>
#include <vector>

#include "mjx_reward.cuh"

using namespace mjx;

extern "C" {

// mjx_grp_reward_dev over host arrays (pts on the host too): the same argument checks (returns -2 where they fail), then the work
// of k_grp_matrix's CTAs one after another and k_train_targets's jobs
int emulr_grp_reward(int n_games, const double* feat, const int32_t* game_off, long long n_rows, const double* weights,
                     long long n_weights, int hidden, int layers, double* matrix, int n_jobs, const int32_t* move_off, long long n_moves,
                     const int32_t* job_game, const uint8_t* job_player, const int32_t* at_kyoku, const uint8_t* apply_gamma,
                     const uint8_t* dones, const uint8_t* rank_by_player, const int64_t* final_scores, const double* pts,
                     int uniform_init, int64_t* steps_to_done, double* kyoku_reward, int64_t* player_rank, int32_t* job_status) {
    if (rw_check_args(n_games, feat, game_off, n_rows, weights, n_weights, hidden, layers, matrix, n_jobs, move_off, n_moves, job_game,
                      job_player, at_kyoku, apply_gamma, dones, rank_by_player, final_scores, pts, steps_to_done, kyoku_reward,
                      player_rank, job_status))
        return -2;
    MatrixView M;
    M.feat = feat; M.game_off = game_off; M.n_rows = n_rows; M.n_games = n_games; M.net = GrpNet{weights, hidden, layers};
    M.matrix = matrix;
    std::vector<double> mem(rw_smem_doubles(hidden, layers));
    struct Hn { double v[RW_GAMES]; };
    std::vector<Hn> hn(RW_THREADS);  // each thread's new hidden states, written after the barrier
    std::vector<int> unit(RW_THREADS);
    long long lo[RW_GAMES];
    int len[RW_GAMES];
    for (int b = 0; b < (n_games + RW_GAMES - 1) / RW_GAMES; b++) {
        const RwCta C = rw_cta(M.net, mem.data(), lo, len);
        for (int tid = 0; tid < RW_THREADS; tid++) rw_begin(M, C, b, tid);
        const int steps = rw_steps(C);
        for (int t = 0; t < steps; t++) {
            for (int tid = 0; tid < RW_THREADS; tid++) rw_load_x(M, C, t, tid);
            for (int k = 0; k < layers; k++) {
                for (int tid = 0; tid < RW_THREADS; tid++)
                    unit[tid] = rw_gru_compute(M.net, C, k, tid, hn[tid].v);
                for (int tid = 0; tid < RW_THREADS; tid++)
                    rw_gru_write(M.net, C, k, t, unit[tid], hn[tid].v);
            }
            for (int tid = 0; tid < RW_THREADS; tid++) rw_fc0(M.net, C, tid);
            for (int tid = 0; tid < RW_THREADS; tid++) rw_fc2(M.net, C, tid);
            for (int tid = 0; tid < RW_THREADS; tid++) rw_out(M, C, t, tid);
        }
    }
    if (n_jobs == 0) return 0;
    TargetView T;
    T.feat = feat; T.game_off = game_off; T.n_rows = n_rows; T.n_games = n_games; T.matrix = matrix;
    T.rank_by_player = rank_by_player; T.final_scores = final_scores; T.uniform_init = uniform_init != 0;
    for (int k = 0; k < 4; k++) T.pts[k] = pts[k];
    T.move_off = move_off; T.n_moves = n_moves; T.job_game = job_game; T.job_player = job_player; T.n_jobs = n_jobs;
    T.at_kyoku = at_kyoku; T.apply_gamma = apply_gamma; T.dones = dones;
    T.steps_to_done = steps_to_done; T.kyoku_reward = kyoku_reward; T.player_rank = player_rank; T.status = job_status;
    for (int j = 0; j < n_jobs; j++) T.status[j] = rw_job(T, j, 0);
    return 0;
}

}  // extern "C"
