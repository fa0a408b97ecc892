// TEST INFRASTRUCTURE ONLY — single-lane host build of mortal_b200/csrc/mjx_grp.cuh (-DMJX_HOST_EMUL): the per-log walk of
// k_grp_logs, so the GRP targets can be diffed against Grp.load_events and run under sanitizers without a GPU. Never loaded by
// mortal_b200/. Part of libmjx_emul.so (tests/emul_lib.py); bound by tests/grp_lib.py.
#include <cstdint>

#include "mjx_grp.cuh"

using namespace mjx;

extern "C" {

// mjx_grp_logs_dev over host arrays: the same argument checks (returns -2 where it fails), then k_grp_logs's per-log work
int emulg_grp_logs(int n_logs, const uint64_t* hdr, const int32_t* ev_off, const int32_t* ev_cnt, long long n_hdr,
                   const uint64_t* kyoku, const int32_t* ky_off, long long n_kyoku_words, const int32_t* deltas,
                   const uint8_t* has_deltas, int32_t* feat, uint8_t* rank_by_player, int64_t* final_scores, int32_t* status) {
    if (n_logs <= 0 || !ev_off || !ev_cnt || !ky_off || !rank_by_player || !final_scores || !status || n_hdr < 0 ||
        (n_hdr > 0 && (!hdr || !deltas || !has_deltas)) || n_kyoku_words < 0 || n_kyoku_words % MJAI_KYOKU_WORDS ||
        (n_kyoku_words > 0 && (!kyoku || !feat)))
        return -2;
    GrpView V;
    V.hdr = hdr; V.ev_off = ev_off; V.ev_cnt = ev_cnt; V.n_hdr = n_hdr; V.kyoku = kyoku; V.ky_off = ky_off;
    V.n_kyoku = n_kyoku_words / MJAI_KYOKU_WORDS; V.deltas = deltas; V.has_deltas = has_deltas; V.n_logs = n_logs;
    V.feat = feat; V.rank = rank_by_player; V.final = final_scores; V.status = status;
    for (int i = 0; i < n_logs; i++) {
        u8 rank[4] = {0, 0, 0, 0};
        i64 fin[4] = {0, 0, 0, 0};
        const int st = grp_log(V, i, 0, rank, fin);
        for (int k = 0; k < 4; k++) {
            V.rank[4 * i + k] = st ? 0 : rank[k];
            V.final[4 * i + k] = st ? 0 : fin[k];
        }
        V.status[i] = st;
    }
    return 0;
}

}  // extern "C"
