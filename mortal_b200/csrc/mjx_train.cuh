// mortal_b200 — fused kernels for training the policy net (mortal/train.py:228-248 over mortal/model.py's Brain / DQN / AuxNet,
// restated in mortal_b200/model.py and mortal_b200/train_ops.py). The convolutions and Linear layers stay with cuDNN / cuBLAS;
// what autograd runs around them as many small elementwise and reduction kernels is done here:
//   - training-mode BatchNorm + Mish, forward and backward (every pre-activation of a block and the trunk's last BN + Mish), also
//     split around an exchange of per-channel partials so that data-parallel ranks normalise with the global batch's statistics;
//   - the channel gate's pooling and `y * g + x`, and their backward;
//   - the dueling combine, the DQN / CQL / next-rank losses and their gradients.
// Activations are channels-last [rows = batch * length, channels], stored as float or __half, with fp32 arithmetic. Every
// reduction runs in an order fixed by the shape alone (per-block partials, merged in block order; no floating-point atomics), so
// two calls on the same inputs are bit-identical. Nothing clamps or flushes a non-finite value: an inf / NaN in an upstream
// gradient reaches the parameter gradients, which is what lets GradScaler skip the step.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>

namespace mjx_train {

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
template <class T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

// mish(u) = u tanh(softplus(u)) = u t, t = n / (n + 2), n = e^u (e^u + 2); mish'(u) = t + u dt/du, dt/du = 4 e (e + 1) / (n + 2)^2.
// Accurate expf (not __expf): these are compared against float64 references at float32 storage. For u > 20, t = 1 in fp32.
__device__ __forceinline__ float mish_f(float u) {
    const float e = expf(fminf(u, 20.f));
    const float n = e * (e + 2.f);
    return u > 20.f ? u : u * (n / (n + 2.f));
}
__device__ __forceinline__ float mish_grad_f(float u) {
    if (u > 20.f) return 1.f;
    const float e = expf(u);
    const float n = e * (e + 2.f), d = n + 2.f;
    return n / d + u * (4.f * e * (e + 1.f)) / (d * d);
}

// ---- BatchNorm (training) + Mish --------------------------------------------------------------------------------------------
// Layout of the statistics kernels: block b owns rows [b * R, (b + 1) * R), its blockDim = k * C threads, thread t owns channel
// t % C and every k-th row of the chunk from t / C. Loads are coalesced along the channels.
constexpr int BN_MAX_BLOCKS = 512;
__host__ __device__ inline int bn_blocks(int n_rows) { int g = (n_rows + 31) / 32; return g < BN_MAX_BLOCKS ? (g ? g : 1) : BN_MAX_BLOCKS; }
__host__ __device__ inline int bn_rows_per_block(int n_rows) { const int g = bn_blocks(n_rows); return (n_rows + g - 1) / g; }
__host__ __device__ inline int bn_lanes(int c) { const int k = 256 / c; return k ? k : 1; }

// part: [gridDim.x][4][C] = count, shift K, mean - K, M2 of the block's chunk. Every thread of a channel sums x - K with the
// same shift K, the chunk's first value of the channel, so the lanes' sums add exactly as plain sums and the partial mean keeps
// float precision relative to K even when the mean is far larger than the spread (a mean of 1e3 with a std of 0.1).
template <class T>
__global__ void __launch_bounds__(256) k_bn_stats(const T* __restrict__ x, int n_rows, int C, int R, float* __restrict__ part) {
    __shared__ double s1[256], s2[256];
    const int k = blockDim.x / C, c = threadIdx.x % C, lane = threadIdx.x / C;
    const int r0 = blockIdx.x * R, r1 = min(n_rows, r0 + R);
    const float K = r0 < r1 ? to_f(x[(size_t)r0 * C + c]) : 0.f;
    double a1 = 0., a2 = 0.;  // x - K is exact in float near the mean; the sums are kept in double
#pragma unroll 4
    for (int r = r0 + lane; r < r1; r += k) {
        const double d = to_f(x[(size_t)r * C + c]) - K;
        a1 += d;
        a2 = fma(d, d, a2);
    }
    s1[threadIdx.x] = a1; s2[threadIdx.x] = a2;
    __syncthreads();
    if (lane == 0) {
        for (int j = 1; j < k; j++) { a1 += s1[j * C + c]; a2 += s2[j * C + c]; }
        const int n = max(r1 - r0, 0);
        float* p = part + (size_t)blockIdx.x * 4 * C;
        p[c] = (float)n;
        p[C + c] = K;
        p[2 * C + c] = n ? (float)(a1 / n) : 0.f;
        const double m2 = n ? a2 - a1 * (a1 / n) : 0.;
        p[3 * C + c] = m2 < 0. ? 0.f : (float)m2;  // rounding; keeps a NaN
    }
}

// merge the block partials (in double, an order fixed by G), write the batch mean and 1 / sqrt(var + eps),
// the mean as a float pair save_mean[c] + save_mean[C + c] (x - hi is exact for x near the mean, so xhat keeps float precision
// for a channel whose mean is far larger than its spread, e.g. 1e3 and 0.1),
// and update the running statistics as nn.BatchNorm1d does in train mode (running_var takes the unbiased variance). With
// training = 0 the running statistics are read instead and left untouched (eval / frozen BatchNorm).
constexpr int FIN_THREADS = 128;
__device__ __forceinline__ void chan_merge(double& n, double& mean, double& m2, double nb, double mb, double m2b) {
    if (nb == 0.) return;
    const double nt = n + nb, d = mb - mean;
    mean += d * (nb / nt);
    m2 += m2b + d * d * (n * nb / nt);
    n = nt;
}
// channel c of one block: thread t merges partials t, t + FIN_THREADS, ... in order, then a pairwise tree in fixed order; the
// result is in thread 0's n / mean / m2
__device__ __forceinline__ void bn_merge_parts(const float* __restrict__ part, int G, int C, int c, double* sn, double* sm,
                                               double* s2, double& n, double& mean, double& m2) {
    const int t = threadIdx.x;
    n = 0.; mean = 0.; m2 = 0.;
    for (int g = t; g < G; g += FIN_THREADS) {
        const float* p = part + (size_t)g * 4 * C;
        chan_merge(n, mean, m2, p[c], (double)p[C + c] + (double)p[2 * C + c], p[3 * C + c]);
    }
    sn[t] = n; sm[t] = mean; s2[t] = m2;
    __syncthreads();
    for (int h = FIN_THREADS / 2; h; h >>= 1) {
        if (t < h) {
            chan_merge(n, mean, m2, sn[t + h], sm[t + h], s2[t + h]);
            sn[t] = n; sm[t] = mean; s2[t] = m2;
        }
        __syncthreads();
    }
}
// the batch statistics of channel c from its merged (n, mean, M2), and the running statistics' update
__device__ __forceinline__ void bn_write_stats(int c, int C, double n, double mean, double m2, float eps, float momentum,
                                               float* __restrict__ running_mean, float* __restrict__ running_var,
                                               float* __restrict__ save_mean, float* __restrict__ save_invstd) {
    const float var = (float)(m2 / n);
    const float hi = (float)mean;
    save_mean[c] = hi;
    save_mean[C + c] = (float)(mean - (double)hi);
    save_invstd[c] = 1.f / sqrtf(var + eps);
    const float unbiased = (float)(m2 / (n - 1.));
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mean;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
}
// one block per channel
__global__ void __launch_bounds__(FIN_THREADS) k_bn_finalize(const float* __restrict__ part, int G, int C, int n_rows, float eps,
                                                             float momentum, int training, float* __restrict__ running_mean,
                                                             float* __restrict__ running_var, float* __restrict__ save_mean,
                                                             float* __restrict__ save_invstd) {
    __shared__ double sn[FIN_THREADS], sm[FIN_THREADS], s2[FIN_THREADS];
    const int c = blockIdx.x, t = threadIdx.x;
    if (!training) {
        if (t == 0) {
            save_mean[c] = running_mean[c];
            save_mean[C + c] = 0.f;
            save_invstd[c] = 1.f / sqrtf(running_var[c] + eps);
        }
        return;
    }
    double n, mean, m2;
    bn_merge_parts(part, G, C, c, sn, sm, s2, n, mean, m2);
    if (t) return;
    bn_write_stats(c, C, n, mean, m2, eps, momentum, running_mean, running_var, save_mean, save_invstd);
}

// ---- BatchNorm statistics across ranks (data-parallel training) ----------------------------------------------------------------
// The forward and backward are split where the ranks exchange per-channel partials: each rank merges its own rows in the order
// k_bn_finalize / k_bn_bwd_finalize use and writes row `rank` of a [world][.][C] double buffer (the others zero); a sum over
// ranks of those buffers (all_reduce SUM: adding exact zeros is exact) gives every rank every row; each rank then merges the
// rows in rank order, so all ranks compute bit-identical statistics. Row 0 starts the merge (not n = 0, a sum of 0.0), so with
// world = 1 the result is the single-process one bit for bit.

// stats[rank][3][C] = (n, mean, M2) of this rank's rows (k_bn_finalize's merge, before its float write); one block per channel
__global__ void __launch_bounds__(FIN_THREADS) k_bn_local_stats(const float* __restrict__ part, int G, int C, int rank,
                                                                double* __restrict__ stats) {
    __shared__ double sn[FIN_THREADS], sm[FIN_THREADS], s2[FIN_THREADS];
    const int c = blockIdx.x;
    double n, mean, m2;
    bn_merge_parts(part, G, C, c, sn, sm, s2, n, mean, m2);
    if (threadIdx.x) return;
    double* o = stats + (size_t)rank * 3 * C;
    o[c] = n; o[C + c] = mean; o[2 * C + c] = m2;
}

// merge the world rows of stats [world][3][C] in rank order and write the statistics as k_bn_finalize does; one thread per channel
__global__ void __launch_bounds__(FIN_THREADS) k_bn_finalize_ranks(const double* __restrict__ stats, int world, int C, float eps,
                                                                   float momentum, float* __restrict__ running_mean,
                                                                   float* __restrict__ running_var, float* __restrict__ save_mean,
                                                                   float* __restrict__ save_invstd) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double n = stats[c], mean = stats[C + c], m2 = stats[2 * C + c];
    for (int r = 1; r < world; r++) {
        const double* p = stats + (size_t)r * 3 * C;
        chan_merge(n, mean, m2, p[c], p[C + c], p[2 * C + c]);
    }
    bn_write_stats(c, C, n, mean, m2, eps, momentum, running_mean, running_var, save_mean, save_invstd);
}

// out = mish(gamma * (x - mean) * invstd + beta), mean = mean[c] + mean[C + c]
template <class T>
__global__ void __launch_bounds__(256) k_bn_mish_apply(const T* __restrict__ x, const float* __restrict__ mean,
                                                       const float* __restrict__ invstd, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, T* __restrict__ out, int n, int C) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int c = i % C;
        const float xh = ((to_f(x[i]) - mean[c]) - mean[C + c]) * invstd[c];
        out[i] = from_f<T>(mish_f(fmaf(gamma[c], xh, beta[c])));
    }
}

// backward partials: part [gridDim.x][2][C] (double) = sum dz, sum dz * xhat over the block's chunk, dz = dout * mish'(u)
template <class T>
__global__ void __launch_bounds__(256) k_bn_mish_bwd_sums(const T* __restrict__ x, const T* __restrict__ dout,
                                                          const float* __restrict__ mean, const float* __restrict__ invstd,
                                                          const float* __restrict__ gamma, const float* __restrict__ beta, int n_rows,
                                                          int C, int R, double* __restrict__ part) {
    __shared__ double s1[256], s2[256];
    const int k = blockDim.x / C, c = threadIdx.x % C, lane = threadIdx.x / C;
    const int r0 = blockIdx.x * R, r1 = min(n_rows, r0 + R);
    const float mu = mean[c], lo = mean[C + c], is = invstd[c], ga = gamma[c], be = beta[c];
    double a1 = 0., a2 = 0.;  // summed in double: dgamma / dbeta are sums of many terms of either sign
#pragma unroll 4
    for (int r = r0 + lane; r < r1; r += k) {
        const size_t i = (size_t)r * C + c;
        const float xh = ((to_f(x[i]) - mu) - lo) * is;
        const float dz = to_f(dout[i]) * mish_grad_f(fmaf(ga, xh, be));
        a1 += dz;
        a2 = fma((double)dz, (double)xh, a2);
    }
    s1[threadIdx.x] = a1; s2[threadIdx.x] = a2;
    __syncthreads();
    if (lane == 0) {
        for (int j = 1; j < k; j++) { a1 += s1[j * C + c]; a2 += s2[j * C + c]; }
        double* p = part + (size_t)blockIdx.x * 2 * C;
        p[c] = a1; p[C + c] = a2;
    }
}

// dbeta = sum dz, dgamma = sum dz * xhat (double, one block per channel, an order fixed by G), and the coefficients of
// dx = k1 dz - k2 - xhat k3: k1 = gamma invstd; k2 = k1 sum dz / N, k3 = k1 sum(dz xhat) / N in training, 0 for a frozen BN
// channel c of one block: the block partials summed in an order fixed by G, the result in s1[0] / s2[0]
__device__ __forceinline__ void bn_sum_parts(const double* __restrict__ part, int G, int C, int c, double* s1, double* s2) {
    const int t = threadIdx.x;
    double a1 = 0., a2 = 0.;
    for (int g = t; g < G; g += FIN_THREADS) {
        a1 += part[(size_t)g * 2 * C + c];
        a2 += part[(size_t)g * 2 * C + C + c];
    }
    s1[t] = a1; s2[t] = a2;
    __syncthreads();
    for (int h = FIN_THREADS / 2; h; h >>= 1) {
        if (t < h) { s1[t] += s1[t + h]; s2[t] += s2[t + h]; }
        __syncthreads();
    }
}
// the dx coefficients of channel c from sum dz (a1) and sum dz xhat (a2) over n_rows rows
__device__ __forceinline__ void bn_write_coef(int c, int C, double a1, double a2, double n_rows, int training,
                                              const float* __restrict__ gamma, const float* __restrict__ invstd,
                                              float* __restrict__ coef) {
    const float k1 = gamma[c] * invstd[c];
    coef[c] = k1;
    coef[C + c] = training ? (float)((double)k1 * a1 / n_rows) : 0.f;
    coef[2 * C + c] = training ? (float)((double)k1 * a2 / n_rows) : 0.f;
}
__global__ void __launch_bounds__(FIN_THREADS) k_bn_bwd_finalize(const double* __restrict__ part, int G, int C, int n_rows, int training,
                                                                 const float* __restrict__ gamma, const float* __restrict__ invstd,
                                                                 float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                                 float* __restrict__ coef) {
    __shared__ double s1[FIN_THREADS], s2[FIN_THREADS];
    const int c = blockIdx.x;
    bn_sum_parts(part, G, C, c, s1, s2);
    if (threadIdx.x) return;
    const double a1 = s1[0], a2 = s2[0];
    dbeta[c] = (float)a1;
    dgamma[c] = (float)a2;
    bn_write_coef(c, C, a1, a2, n_rows, training, gamma, invstd, coef);
}

// sums[rank][2][C] = (sum dz, sum dz xhat) of this rank's rows, k_bn_bwd_finalize's order; one block per channel
__global__ void __launch_bounds__(FIN_THREADS) k_bn_bwd_local_sums(const double* __restrict__ part, int G, int C, int rank,
                                                                   double* __restrict__ sums) {
    __shared__ double s1[FIN_THREADS], s2[FIN_THREADS];
    const int c = blockIdx.x;
    bn_sum_parts(part, G, C, c, s1, s2);
    if (threadIdx.x) return;
    double* o = sums + (size_t)rank * 2 * C;
    o[c] = s1[0]; o[C + c] = s2[0];
}

// the training-mode coefficients from the rows of sums [world][2][C] added in rank order over all ranks' total_rows rows, and
// dgamma / dbeta from this rank's own row (a data-parallel gradient all-reduce sums or averages them); one thread per channel
__global__ void __launch_bounds__(FIN_THREADS) k_bn_bwd_finalize_ranks(const double* __restrict__ sums, int world, int rank, int C,
                                                                       double total_rows, const float* __restrict__ gamma,
                                                                       const float* __restrict__ invstd, float* __restrict__ dgamma,
                                                                       float* __restrict__ dbeta, float* __restrict__ coef) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double a1 = sums[c], a2 = sums[C + c];
    for (int r = 1; r < world; r++) {
        a1 += sums[(size_t)r * 2 * C + c];
        a2 += sums[(size_t)r * 2 * C + C + c];
    }
    const double* own = sums + (size_t)rank * 2 * C;
    dbeta[c] = (float)own[c];
    dgamma[c] = (float)own[C + c];
    bn_write_coef(c, C, a1, a2, total_rows, 1, gamma, invstd, coef);
}

template <class T>
__global__ void __launch_bounds__(256) k_bn_mish_bwd_dx(const T* __restrict__ x, const T* __restrict__ dout,
                                                        const float* __restrict__ mean, const float* __restrict__ invstd,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        const float* __restrict__ coef, T* __restrict__ dx, int n, int C) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int c = i % C;
        const float xh = ((to_f(x[i]) - mean[c]) - mean[C + c]) * invstd[c];
        const float dz = to_f(dout[i]) * mish_grad_f(fmaf(gamma[c], xh, beta[c]));
        dx[i] = from_f<T>(coef[c] * dz - coef[C + c] - xh * coef[2 * C + c]);
    }
}

// ---- channel gate + residual ------------------------------------------------------------------------------------------------
// max that keeps a NaN, as torch.amax does
__device__ __forceinline__ float nan_max(float m, float v) { return (v > m || v != v) ? v : m; }

// one thread per (b, c): avg = mean_l y, mx = max_l y (stored as T, as torch's mean / amax of a T tensor)
template <class T>
__global__ void __launch_bounds__(256) k_gate_pool(const T* __restrict__ y, T* __restrict__ avg, T* __restrict__ mx, int B, int L, int C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * C) return;
    const int b = i / C, c = i % C;
    const T* p = y + (size_t)b * L * C + c;
    double s = 0.;
    float m = to_f(p[0]);
#pragma unroll 2
    for (int l = 0; l < L; l++) {
        const float v = to_f(p[(size_t)l * C]);
        s += v;
        m = nan_max(m, v);
    }
    avg[i] = from_f<T>((float)(s / L));
    mx[i] = from_f<T>(m);
}

// out = y * g[b, c] + x
template <class T>
__global__ void __launch_bounds__(256) k_gate_out(const T* __restrict__ y, const T* __restrict__ g, const T* __restrict__ x,
                                                  T* __restrict__ out, int n, int LC, int C) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int b = i / LC, c = i % C;
        out[i] = from_f<T>(fmaf(to_f(y[i]), to_f(g[b * C + c]), to_f(x[i])));
    }
}

// one thread per (b, c): dg (float32) = sum_l dout * y, cnt = the number of l with y == max (amax's gradient is split among the ties)
template <class T>
__global__ void __launch_bounds__(256) k_gate_bwd_dg(const T* __restrict__ dout, const T* __restrict__ y, const T* __restrict__ mx,
                                                     float* __restrict__ dg, float* __restrict__ cnt, int B, int L, int C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * C) return;
    const int b = i / C, c = i % C;
    const size_t o = (size_t)b * L * C + c;
    const float m = to_f(mx[i]);
    double s = 0.;  // a sum of terms of either sign: kept in double
    float n = 0.f;
#pragma unroll 2
    for (int l = 0; l < L; l++) {
        const float v = to_f(y[o + (size_t)l * C]);
        s = fma((double)to_f(dout[o + (size_t)l * C]), (double)v, s);
        n += v == m ? 1.f : 0.f;
    }
    dg[i] = (float)s;
    cnt[i] = n;
}

// dy = dout * g + d_avg / L + (y == max ? d_max / cnt : 0)
template <class T>
__global__ void __launch_bounds__(256) k_gate_bwd_dy(const T* __restrict__ dout, const T* __restrict__ y, const T* __restrict__ g,
                                                     const T* __restrict__ mx, const float* __restrict__ cnt, const T* __restrict__ davg,
                                                     const T* __restrict__ dmx, T* __restrict__ dy, int n, int L, int C) {
    const float inv_l = 1.f / (float)L;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int bc = i / (L * C) * C + i % C;
        const float v = to_f(y[i]);
        float d = fmaf(to_f(dout[i]), to_f(g[bc]), to_f(davg[bc]) * inv_l);
        if (v == to_f(mx[bc])) d += to_f(dmx[bc]) / cnt[bc];
        dy[i] = from_f<T>(d);
    }
}

// ---- dueling head + losses ---------------------------------------------------------------------------------------------------
constexpr int N_ACT = 46;
constexpr int LOSS_THREADS = 1024;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = nan_max(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// one row of the dueling head, computed by a warp: lane j holds actions j and j + 32. q[j] = v + a[j] - mean_legal(a) on legal
// actions (-inf elsewhere), lse = logsumexp of q, qa = q[action].
struct RowQ { float q0, q1, lse, qa, n_legal; bool l0, l1, bad; };
template <class T>
__device__ __forceinline__ RowQ row_q(const T* __restrict__ v, const T* __restrict__ a, const uint8_t* __restrict__ masks,
                                      const int64_t* __restrict__ actions, int i, int lane) {
    RowQ r;
    const int j0 = lane, j1 = lane + 32;
    r.l0 = masks[(size_t)i * N_ACT + j0] != 0;
    r.l1 = j1 < N_ACT && masks[(size_t)i * N_ACT + j1] != 0;
    const float a0 = to_f(a[(size_t)i * N_ACT + j0]), a1 = j1 < N_ACT ? to_f(a[(size_t)i * N_ACT + j1]) : 0.f;
    r.n_legal = warp_sum((r.l0 ? 1.f : 0.f) + (r.l1 ? 1.f : 0.f));
    const float a_mean = warp_sum((r.l0 ? a0 : 0.f) + (r.l1 ? a1 : 0.f)) / r.n_legal;
    const float vv = to_f(v[i]);
    r.q0 = r.l0 ? (vv + a0) - a_mean : -INFINITY;
    r.q1 = r.l1 ? (vv + a1) - a_mean : -INFINITY;
    const float m = warp_max(nan_max(r.q0, r.q1));
    const float s = warp_sum((r.l0 ? expf(r.q0 - m) : 0.f) + (r.l1 ? expf(r.q1 - m) : 0.f));
    r.lse = m + logf(s);
    const int64_t act = actions[i];
    const bool in_range = act >= 0 && act < N_ACT;
    const int ai = in_range ? (int)act : 0;
    const float qa0 = __shfl_sync(0xffffffffu, r.q0, ai & 31), qa1 = __shfl_sync(0xffffffffu, r.q1, ai & 31);
    const bool la0 = __shfl_sync(0xffffffffu, r.l0, ai & 31), la1 = __shfl_sync(0xffffffffu, r.l1, ai & 31);
    r.qa = in_range ? (ai < 32 ? qa0 : qa1) : NAN;
    r.bad = !in_range || !(ai < 32 ? la0 : la1);
    return r;
}
// cross-entropy of one row of the aux logits (n_aux <= 32, lane k holds logit k): (loss, softmax of lane's logit)
template <class T>
__device__ __forceinline__ float row_ce(const T* __restrict__ aux, int n_aux, int64_t rank, int i, int lane, float& p) {
    const bool on = lane < n_aux;
    const float z = on ? to_f(aux[(size_t)i * n_aux + lane]) : -INFINITY;
    const float m = warp_max(z);
    const float e = on ? expf(z - m) : 0.f;
    const float s = warp_sum(e);
    p = e / s;
    const int rk = (rank >= 0 && rank < n_aux) ? (int)rank : 0;
    const float zr = __shfl_sync(0xffffffffu, z, rk);
    return (rank >= 0 && rank < n_aux) ? m + logf(s) - zr : NAN;
}
// the Monte-Carlo target as torch evaluates (gamma ** steps_to_done * kyoku_rewards).float(): a float32 power (a Python float
// base with an int64 tensor exponent promotes to the default float32), times the float64 reward in float64, rounded to float32
__device__ __forceinline__ float mc_target(float gamma, int64_t steps, double reward) {
    return (float)((double)powf(gamma, (float)steps) * reward);
}

// one block of LOSS_THREADS: warp w handles rows w, w + 32, ... in order and accumulates in double, the 32 warp sums are added in
// warp order. losses = [0.5 mean (q - t)^2, mean lse - mean q, mean ce]; bad |= 1 when an action is outside its mask.
template <class T>
__global__ void __launch_bounds__(LOSS_THREADS) k_dqn_loss_fwd(const T* __restrict__ v, const T* __restrict__ a,
                                                                const uint8_t* __restrict__ masks, const int64_t* __restrict__ actions,
                                                                const int64_t* __restrict__ steps_to_done, const double* __restrict__ rewards,
                                                                const T* __restrict__ aux, const int64_t* __restrict__ ranks, int B,
                                                                int n_aux, float gamma, float* __restrict__ q_out, float* __restrict__ q_act,
                                                                float* __restrict__ q_target, float* __restrict__ losses,
                                                                int* __restrict__ bad) {
    __shared__ double sd[32][4];
    const int w = threadIdx.x / 32, lane = threadIdx.x % 32, nw = blockDim.x / 32;
    double mse = 0., lse = 0., qs = 0., ce = 0.;
    int any_bad = 0;
    for (int i = w; i < B; i += nw) {
        const RowQ r = row_q(v, a, masks, actions, i, lane);
        float p;
        const float c = row_ce(aux, n_aux, ranks[i], i, lane, p);
        const float t = mc_target(gamma, steps_to_done[i], rewards[i]);
        if (q_out) {
            q_out[(size_t)i * N_ACT + lane] = r.q0;
            if (lane + 32 < N_ACT) q_out[(size_t)i * N_ACT + lane + 32] = r.q1;
        }
        if (lane == 0) {
            const float d = r.qa - t;
            mse += (double)(d * d);
            lse += r.lse;
            qs += r.qa;
            ce += c;
            q_act[i] = r.qa;
            q_target[i] = t;
            any_bad |= r.bad;
        }
    }
    if (lane == 0) { sd[w][0] = mse; sd[w][1] = lse; sd[w][2] = qs; sd[w][3] = ce; }
    if (lane == 0 && any_bad) atomicOr(bad, 1);  // an integer flag: order does not matter
    __syncthreads();
    if (threadIdx.x == 0) {
        double s[4] = {0., 0., 0., 0.};
        for (int k = 0; k < nw; k++)
            for (int j = 0; j < 4; j++) s[j] += sd[k][j];
        losses[0] = (float)(0.5 * s[0] / B);
        losses[1] = (float)(s[1] / B) - (float)(s[2] / B);
        losses[2] = (float)(s[3] / B);
    }
}

// gradients of w[0] dqn + w[1] cql + w[2] next_rank (w: float32 [3] on the device, the upstream gradients of the three losses)
// with respect to v [B, 1], a [B, 46] and the aux logits [B, n_aux]; one warp per row
template <class T>
__global__ void __launch_bounds__(256) k_dqn_loss_bwd(const T* __restrict__ v, const T* __restrict__ a, const uint8_t* __restrict__ masks,
                                                      const int64_t* __restrict__ actions, const float* __restrict__ q_target,
                                                      const T* __restrict__ aux, const int64_t* __restrict__ ranks, int B, int n_aux,
                                                      const float* __restrict__ w, T* __restrict__ dv, T* __restrict__ da,
                                                      T* __restrict__ daux) {
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x % 32;
    if (i >= B) return;  // whole warps leave together
    const float inv_b = 1.f / (float)B;
    const float wd = w[0] * inv_b, wc = w[1] * inv_b, wn = w[2] * inv_b;
    const RowQ r = row_q(v, a, masks, actions, i, lane);
    const int64_t act = actions[i];
    const float dq = wd * (r.qa - q_target[i]) - wc;  // d/dq[action]
    const float g0 = r.l0 ? wc * expf(r.q0 - r.lse) + (act == lane ? dq : 0.f) : 0.f;
    const float g1 = r.l1 ? wc * expf(r.q1 - r.lse) + (act == lane + 32 ? dq : 0.f) : 0.f;
    const float s = warp_sum(g0 + g1);
    const float sm = s / r.n_legal;
    if (lane == 0) dv[i] = from_f<T>(s);
    da[(size_t)i * N_ACT + lane] = from_f<T>(r.l0 ? g0 - sm : 0.f);
    if (lane + 32 < N_ACT) da[(size_t)i * N_ACT + lane + 32] = from_f<T>(r.l1 ? g1 - sm : 0.f);
    float p;
    const int64_t rank = ranks[i];
    row_ce(aux, n_aux, rank, i, lane, p);
    if (lane < n_aux) daux[(size_t)i * n_aux + lane] = from_f<T>(wn * (p - (rank == lane ? 1.f : 0.f)));
}

}  // namespace mjx_train
