// TEST INFRASTRUCTURE ONLY — single-lane host build of mortal_b200/csrc/mjx_validate.cuh (-DMJX_HOST_EMUL), the logic of
// k_validate_logs, so the validator can be diffed against the oracle and run under sanitizers without a GPU. Never loaded by
// mortal_b200/; the product has no CPU path. Built by tests/validate_lib.py.
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "mjx_validate.cuh"
#include "mjx_tables_host.h"

using namespace mjx;

static HostTables g_H;
static Tables g_T;
static bool g_ready = false;
static std::string g_err;

extern "C" {

const char* emulv_last_error() { return g_err.c_str(); }

int emulv_init(const char* data_dir) {
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

// mjx_validate_logs one log at a time; the same argument checks as the C ABI, returns 0 or -2
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
