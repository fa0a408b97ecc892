// TEST INFRASTRUCTURE ONLY — single-lane host build of mortal_b200/csrc/mjx_stat.cuh (-DMJX_HOST_EMUL): the per-log walk of
// k_stat_logs with one lane playing all four seats, and the decoder's deltas reader (mjai_line_deltas of csrc/mjx_mjai.cuh), so
// the statistics can be diffed against Stat.from_game and run under sanitizers without a GPU. Never loaded by mortal_b200/.
// Part of libmjx_emul.so (tests/emul_lib.py); bound by tests/stat_lib.py.
#include <cstdint>
#include <cstring>

#include "mjx_stat.cuh"

using namespace mjx;

extern "C" {

// mjx_stat_logs_dev over host arrays: the same argument checks (returns -2 where it fails), then k_stat_logs's per-log work
int emuls_stat_logs(int n_logs, const uint64_t* hdr, const int32_t* ev_off, const int32_t* ev_cnt, long long n_hdr,
                    const uint64_t* kyoku, const int32_t* ky_off, long long n_kyoku_words, const int32_t* deltas,
                    const uint8_t* has_deltas, const uint8_t* seats, int64_t* out, int32_t* status) {
    if (n_logs <= 0 || !ev_off || !ev_cnt || !ky_off || !seats || !out || !status || n_hdr < 0 ||
        (n_hdr > 0 && (!hdr || !deltas || !has_deltas)) || n_kyoku_words < 0 || n_kyoku_words % MJAI_KYOKU_WORDS ||
        (n_kyoku_words > 0 && !kyoku))
        return -2;
    StatView V;
    V.hdr = hdr; V.ev_off = ev_off; V.ev_cnt = ev_cnt; V.n_hdr = n_hdr; V.kyoku = kyoku; V.ky_off = ky_off;
    V.n_kyoku = n_kyoku_words / MJAI_KYOKU_WORDS; V.deltas = deltas; V.has_deltas = has_deltas; V.seats = seats; V.n_logs = n_logs;
    V.out = out; V.status = status;
    for (int i = 0; i < n_logs; i++) {
        i64 c[4][MJX_STAT_N];
        memset(c, 0, sizeof(c));
        const int st = stat_log(V, i, 0, c);
        for (int k = 0; k < MJX_STAT_N; k++) out[(long long)i * MJX_STAT_N + k] = st ? 0 : c[0][k] + c[1][k] + c[2][k] + c[3][k];
        status[i] = st;
    }
    return 0;
}

// mjai_line_deltas over one line [0, n) -> d[4]; returns has_deltas
int emuls_line_deltas(const uint8_t* line, long long n, int32_t* d) { return mjai_line_deltas(line, 0, n, d) ? 1 : 0; }

}  // extern "C"
