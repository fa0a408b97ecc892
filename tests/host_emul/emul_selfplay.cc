// TEST INFRASTRUCTURE ONLY — host build of mortal_b200/csrc/mjx_selfplay.cuh (-DMJX_HOST_EMUL): the per-event check and converter
// of k_arena_words driven by a restatement of the kernel's warp walk (chunks of up to 32 event starts, a chunk with a bad event
// writes nothing, payload and hora indices from the running counts plus the lanes before), the lanes run one after another. Lets
// the converter be diffed against mortal_b200/mjai_log.py + dataset_codec.py and run under sanitizers without a GPU. Never loaded
// by mortal_b200/. Part of libmjx_emul.so (tests/emul_lib.py).
#include <cstdint>

#include "mjx_selfplay.cuh"

using namespace mjx;

extern "C" {

// mjx_arena_words_count_dev (hdr == null: counts int32 [n_games, 4]) or mjx_arena_words_fill_dev over host arrays. Returns 0 or -2.
int emulsp_convert(int n_games, const uint64_t* words, const int32_t* lens, long long pitch, int log_cap, int augment, int32_t* counts,
                   const int32_t* ev_off, const int32_t* ky_off, const int32_t* hora_off, uint64_t* hdr, int32_t* lines, long long n_hdr,
                   uint64_t* kyoku, long long n_kyoku_words, uint64_t* hora, long long n_hora_words, int32_t* deltas,
                   uint8_t* has_deltas) {
    if (n_games <= 0 || !words || !lens || log_cap <= 0 || pitch < log_cap || !counts) return -2;
    const bool fill = hdr != nullptr;
    if (fill && (!ev_off || !ky_off || !hora_off || !lines || !deltas || !has_deltas || n_hdr < 0 || n_kyoku_words < 0 ||
                 n_kyoku_words % AW_KYOKU_WORDS || n_hora_words < 0 || n_hora_words % MJX_HORA_WORDS))
        return -2;
    AwView V{};
    V.words = words; V.lens = lens; V.pitch = pitch; V.log_cap = log_cap; V.n_games = n_games; V.augment = augment; V.counts = counts;
    V.ev_off = ev_off; V.ky_off = ky_off; V.hora_off = hora_off; V.hdr = hdr; V.lines = lines; V.n_hdr = fill ? n_hdr : 0;
    V.kyoku = kyoku; V.n_kyoku = fill ? n_kyoku_words / AW_KYOKU_WORDS : 0; V.hora = hora; V.n_hora = fill ? n_hora_words / MJX_HORA_WORDS : 0;
    V.deltas = deltas; V.has_deltas = has_deltas;
    for (int g = 0; g < n_games; g++) {
        if (fill && counts[4 * g] != MJX_AW_OK) continue;
        const u64* w;
        int n;
        int st = aw_game_words(V, g, &w, &n);
        const long long e0 = fill ? ev_off[g] : 0, k0 = fill ? ky_off[g] : 0, h0 = fill ? hora_off[g] : 0;
        if (fill) aw_fill_bound(V, AW_START_GAME, e0, 1);
        int n_ev = 0, n_ky = 0, n_ho = 0;
        for (int pos = 0; st == MJX_AW_OK && pos < n;) {
            int start[32], cnt = 0, nx = pos, wst = MJX_AW_OK;
            while (cnt < 32 && nx < n) {  // lane 0's walk
                const int t = aw_next(w, n, nx);
                if (t < 0) { wst = -t; break; }
                start[cnt++] = nx;
                nx = t;
            }
            bool bad = false;
            for (int lane = 0; lane < cnt; lane++) bad = bad || aw_check(w, start[lane]) != MJX_AW_OK;
            int ky = 0, ho = 0;
            for (int lane = 0; lane < cnt; lane++) {
                const int ty = (int)(w[start[lane]] & 0xFF);
                if (fill && !bad) {
                    const int e = 1 + n_ev + lane;
                    aw_fill_event(V, w, start[lane], e0 + e, e + 1, k0 + n_ky + ky, h0 + n_ho + ho);
                }
                ky += ty == AW_START_KYOKU;
                ho += ty == AW_HORA;
            }
            n_ev += cnt; n_ky += ky; n_ho += ho;
            st = bad ? MJX_AW_CORRUPT : wst;
            pos = nx;
        }
        if (fill && st == MJX_AW_OK) aw_fill_bound(V, AW_END_GAME, e0 + n_ev + 1, n_ev + 2);
        if (!fill) {
            const bool ok = st == MJX_AW_OK;
            counts[4 * g] = st;
            counts[4 * g + 1] = ok ? n_ev + 2 : 0;
            counts[4 * g + 2] = ok ? n_ky : 0;
            counts[4 * g + 3] = ok ? n_ho : 0;
        }
    }
    return 0;
}

}  // extern "C"
