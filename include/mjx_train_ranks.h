/* mjx_train_ranks — training-mode BatchNorm + Mish for data-parallel training (csrc/mjx_train.cuh), the entries around the
 * exchange of per-channel partials between ranks. Same conventions as include/mjx.h's policy-net training entries: device
 * pointers, channels-last activations of dtype MJX_TRAIN_F32 / MJX_TRAIN_F16, 0 or a negative mjx_status, `stream` a cudaStream_t
 * passed as void*. */
#ifndef MJX_TRAIN_RANKS_H
#define MJX_TRAIN_RANKS_H

#include "mjx.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Training-mode BatchNorm + Mish over the rows of `world` ranks (data-parallel training), split where the ranks exchange their
 * per-channel partials. Each local stage writes row `rank` of a double buffer and leaves the other rows alone; the caller zeroes
 * them and sums the buffers over the ranks (an all_reduce SUM of exact zeros, so every rank holds every row bit for bit) before
 * the global stage, which merges the rows in rank order: every rank computes the same statistics. Row counts may differ between
 * ranks. With world = 1 the two stages give mjx_train_bn_mish_fwd / _bwd's (training != 0) outputs bit for bit. `scratch` is
 * mjx_train_bn_scratch_floats(rows, channels) floats; stats / sums / scratch are 8-byte aligned.
 * local stats: stats[rank] = double [3][channels] (count, mean, M2) of this rank's rows. */
int mjx_train_bn_local_stats(int dtype, const void* x, int rows, int channels, int rank, int world, double* stats, float* scratch,
                             void* stream);
/* global forward: the statistics of stats double [world][3][channels] (save_mean, save_invstd and the running statistics, the
 * unbiased variance over the global count), then out as mjx_train_bn_mish_fwd. */
int mjx_train_bn_mish_fwd_ranks(int dtype, const void* x, const float* gamma, const float* beta, float* running_mean,
                                float* running_var, float* save_mean, float* save_invstd, void* out, int rows, int channels, float eps,
                                float momentum, const double* stats, int world, void* stream);
/* local backward: sums[rank] = double [2][channels] (sum dz, sum dz xhat) of this rank's rows, from the global forward's
 * save_mean / save_invstd. */
int mjx_train_bn_bwd_local_sums(int dtype, const void* x, const void* dout, const float* gamma, const float* beta,
                                const float* save_mean, const float* save_invstd, int rows, int channels, int rank, int world,
                                double* sums, float* scratch, void* stream);
/* global backward: dx from the sums of sums double [world][2][channels] over all ranks' total_rows rows; dgamma / dbeta from
 * row `rank` only (this rank's share: a gradient all-reduce adds the ranks' shares). */
int mjx_train_bn_mish_bwd_ranks(int dtype, const void* x, const void* dout, const float* gamma, const float* beta,
                                const float* save_mean, const float* save_invstd, void* dx, float* dgamma, float* dbeta, int rows,
                                int channels, const double* sums, int rank, int world, long long total_rows, float* scratch,
                                void* stream);
#ifdef __cplusplus
}
#endif
#endif /* MJX_TRAIN_RANKS_H */
