// TEST INFRASTRUCTURE ONLY — host build of mortal_b200/csrc/mjx_mjai.cuh (-DMJX_HOST_EMUL): the line parser of k_mjai_decode
// driven by a restatement of the kernel's warp walk (the same 128-byte steps, 32-byte windows, 64-entry queue of line ends and
// 32-line flushes, the lanes run one after another), so the decoder's accept / decline rule, its arrays and its queue indexing
// can be diffed against the Python decoder and run under sanitizers without a GPU. Never loaded by mortal_b200/. Part of
// libmjx_emul.so (tests/emul_lib.py); bound by tests/mjai_lib.py.
#include <cstdint>
#include <cstring>
#include <vector>

#include "mjx_mjai.cuh"

using namespace mjx;

extern "C" {

// mjx_mjai_count_dev + mjx_mjai_fill_dev over host arrays in one call. The arrays are sized by the caller from a first call with
// hdr == nullptr (counts only); log i's outputs start at ev_off[i] / ky_off[i] / hora_off[i]. Returns 0 or -2.
int emulm_decode(int n_logs, const uint8_t* text, long long n_bytes, const int64_t* log_off, int augment, mjx_mjai_counts* counts,
                 const int32_t* ev_off, const int32_t* ky_off, const int32_t* hora_off, uint64_t* hdr, int32_t* lines, long long n_hdr,
                 uint64_t* kyoku, long long n_kyoku, uint64_t* hora, long long n_hora) {
    if (n_logs <= 0 || n_bytes < 0 || !log_off || !counts) return -2;
    for (int i = 0; i < n_logs; i++) {
        if (hdr && !counts[i].accept) continue;  // the fill pass skips declined logs
        const long long lb = log_off[i], le = log_off[i + 1];
        mjx_mjai_counts cn{0, 0, 0, 0, -1, -1};
        bool decline = lb < 0 || le <= lb || le > n_bytes || le - lb >= 0x7FFFFFFF;
        const int len = decline ? 0 : (int)(le - lb);
        const uint8_t* p = text + (decline ? 0 : lb);
        int n_ev = 0, n_ky = 0, n_ho = 0, line_no = 0, fb = -1, fe = -1;
        int q[64];  // the warp's queue of line ends (s_end[warp]); ASan reports any index past it
        int qn = 0, start = 0;
        bool fail = false;
        auto flush = [&](int cnt) {  // lane j parses the j-th queued line; events are placed in lane order
            MjaiLine ln[32];
            int bs[32], ces[32];
            for (int lane = 0; lane < cnt; lane++) {
                bs[lane] = lane == 0 ? start : q[lane - 1] + 1;
                ces[lane] = q[lane];
                if (ces[lane] < len && ces[lane] > bs[lane] && p[ces[lane] - 1] == '\r') ces[lane]--;
                ln[lane] = mjai_parse_line(p, bs[lane], ces[lane], augment != 0, nullptr, nullptr);
                decline = decline || ln[lane].kind == MJ_DECLINE;
            }
            for (int lane = 0; lane < cnt && !decline; lane++) {
                if (ln[lane].kind != MJ_EVENT) continue;
                if (fb < 0) { fb = bs[lane]; fe = ces[lane]; }
                if (hdr) {
                    const long long at = (long long)ev_off[i] + n_ev;
                    if (at < 0 || at >= n_hdr) { fail = true; return; }
                    hdr[at] = ln[lane].word;
                    lines[at] = line_no + lane + 1;
                    if (ln[lane].ty == MJT_START_KYOKU) {
                        const long long k = (long long)ky_off[i] + n_ky;
                        if (k < 0 || k >= n_kyoku) { fail = true; return; }
                        mjai_parse_line(p, bs[lane], ces[lane], augment != 0, kyoku + k * MJAI_KYOKU_WORDS, nullptr);
                    } else if (ln[lane].ty == MJT_HORA) {
                        const long long k = (long long)hora_off[i] + n_ho;
                        if (k < 0 || k >= n_hora) { fail = true; return; }
                        mjai_parse_line(p, bs[lane], ces[lane], augment != 0, nullptr, hora + k * MJX_HORA_WORDS);
                    }
                }
                n_ev++;
                n_ky += ln[lane].ty == MJT_START_KYOKU;
                n_ho += ln[lane].ty == MJT_HORA;
            }
            line_no += cnt;
            start = q[cnt - 1] + 1;
            for (int k = 0; k < qn - cnt; k++) q[k] = q[cnt + k];
            qn -= cnt;
        };
        // k_mjai_decode's walk: 128-byte steps of four 32-byte windows, each window's line ends queued, a full queue flushed
        for (int base = 0; base < len && !decline; base += 128) {
            for (int k = 0; k < 4; k++) {
                if (decline) break;
                int added = 0;
                for (int lane = 0; lane < 32; lane++) {
                    const int pos = base + 32 * k + lane;
                    if (pos < len && p[pos] == '\n') q[qn + added++] = pos;
                }
                qn += added;
                if (qn >= 32) flush(32);
                if (fail) return -2;
            }
        }
        if (!decline) {
            const int next = qn ? q[qn - 1] + 1 : start;
            if (next < len) q[qn++] = len;  // the last line has no line break
            while (qn > 0 && !decline) {
                flush(qn < 32 ? qn : 32);
                if (fail) return -2;
            }
        }
        if (!decline && n_ev > 0) cn = mjx_mjai_counts{1, n_ev, n_ky, n_ho, fb, fe};
        if (!hdr) counts[i] = cn;
    }
    return 0;
}

}  // extern "C"
