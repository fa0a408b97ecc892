// TEST INFRASTRUCTURE ONLY — host build of mortal_b200/csrc/mjx_mjai_write.cuh (-DMJX_HOST_EMUL): the Q-value formatter and the
// per-event renderer of k_mjai_render driven by one host lane that walks a game's events in order (the kernel's lanes take 32
// consecutive events at a time and place them by a prefix sum: the same events in the same order). Lets the renderer be diffed
// against mortal_b200/mjai_log.py and CPython's float repr, and run under sanitizers, without a GPU. Never loaded by
// mortal_b200/. Part of libmjx_emul.so (tests/emul_lib.py); bound by tests/mjai_write_lib.py.
#include <cmath>
#include <cstdint>
#include <cstring>

#include "mjx_mjai_write.cuh"

using namespace mjx;

extern "C" {

// json.dumps(float(x)) of every bits[i] as an f32, joined by "\n" into out; returns the bytes written (-1: out too small)
long long emulw_format_f32(const uint32_t* bits, long long n, char* out, long long cap) {
    long long at = 0;
    char b[32];
    for (long long i = 0; i < n; i++) {
        float x;
        memcpy(&x, &bits[i], 4);
        const int len = mw_format_f32(x, b);
        if (at + len + 1 > cap) return -1;
        memcpy(out + at, b, len);
        at += len;
        out[at++] = '\n';
    }
    return at;
}

// the formatter against CPython: for every f32 bit pattern in [lo, hi) (step `step`), PyOS_double_to_string(x, 'r', 0,
// Py_DTSF_ADD_DOT_0, NULL) for finite x, json's NaN / Infinity / -Infinity otherwise. `dtoa` / `mem_free` are
// PyOS_double_to_string / PyMem_Free of the calling interpreter, which must hold the GIL (ctypes.PyDLL). Returns the mismatches;
// *first_bad = the first mismatching pattern.
typedef char* (*dtoa_fn)(double, char, int, int, int*);
typedef void (*free_fn)(void*);
static bool same_as_cpython(uint32_t u, void* dtoa, void* mem_free) {
    char b[32];
    float x;
    memcpy(&x, &u, 4);
    const int len = mw_format_f32(x, b);
    b[len] = 0;
    if (std::isnan(x)) return strcmp(b, "NaN") == 0;
    if (std::isinf(x)) return strcmp(b, x > 0 ? "Infinity" : "-Infinity") == 0;
    char* ref = ((dtoa_fn)dtoa)((double)x, 'r', 0, 0x02 /* Py_DTSF_ADD_DOT_0 */, nullptr);
    const bool ok = ref && strcmp(b, ref) == 0;
    ((free_fn)mem_free)(ref);
    return ok;
}
long long emulw_sweep(uint64_t lo, uint64_t hi, uint64_t step, void* dtoa, void* mem_free, uint64_t* first_bad) {
    long long bad = 0;
    for (uint64_t p = lo; p < hi; p += step)
        if (!same_as_cpython((uint32_t)p, dtoa, mem_free)) {
            if (!bad && first_bad) *first_bad = p;
            bad++;
        }
    return bad;
}
// the same over a list of bit patterns
long long emulw_check(const uint32_t* bits, long long n, void* dtoa, void* mem_free, uint64_t* first_bad) {
    long long bad = 0;
    for (long long i = 0; i < n; i++)
        if (!same_as_cpython(bits[i], dtoa, mem_free)) {
            if (!bad && first_bad) *first_bad = bits[i];
            bad++;
        }
    return bad;
}

// mjx_mjai_render_count_dev (out == null: bytes / status) or mjx_mjai_render_fill_dev over all games (out: game g at off[g])
// over host arrays
int emulw_render(int n_games, const uint64_t* words, const int32_t* lens, int log_cap, const int32_t* bounds, int n_steps,
                 int key_steps, const int64_t* rec_key, const int32_t* rec_info, const uint64_t* rec_mask, const float* rec_q,
                 const int64_t* rec_i64, long long n_rec, int32_t* bytes, int32_t* status, const int64_t* off, char* out,
                 long long out_cap) {
    if (n_games <= 0 || !words || !lens || log_cap <= 0 || !bytes || !status) return -2;
    MwView V{};
    V.words = words; V.lens = lens; V.log_cap = log_cap; V.n_games = n_games;
    V.bounds = bounds; V.n_steps = n_steps; V.key_steps = key_steps;
    V.rec_key = rec_key; V.rec_info = rec_info; V.rec_mask = rec_mask; V.rec_q = rec_q; V.rec_i64 = rec_i64; V.n_rec = bounds ? n_rec : 0;
    for (int g = 0; g < n_games; g++) {
        if (out && status[g] != MJX_MW_OK) continue;
        MwOut o{out ? out + off[g] : nullptr, 0, out ? out_cap - off[g] : 0};
        const u64* w;
        int n;
        int st = mw_game_words(V, g, &w, &n);
        for (int i = 0; i < n && st == MJX_MW_OK;) {
            const int nx = mw_next(w, n, i);
            if (nx < 0) {
                st = -nx;
                break;
            }
            st = mw_event(o, V, g, w, i);
            i = nx;
        }
        if (!out) {
            status[g] = st;
            bytes[g] = st == MJX_MW_OK ? (int32_t)o.n : 0;
        }
    }
    return 0;
}

}  // extern "C"

extern "C" {
// mjx_meta_record_dev over host arrays: the kernel's lanes one after another
int emulw_meta_record(long long n, const int64_t* idx, const float* q, const uint8_t* greedy, const int32_t* call_ids, int call,
                      int cycle, const int32_t* row_table, const uint8_t* row_seat, const int64_t* actions, const uint8_t* masks,
                      const float* obs, int obs_rows, int row_cap, int32_t* out_table, int32_t* out_cycle, uint8_t* out_seat,
                      int32_t* out_info, uint64_t* out_mask, float* out_q, int32_t* out_call, long long base, long long cap) {
    MrView V{n, idx, q, greedy, call_ids, call, cycle, row_table, row_seat, actions, masks, obs, obs_rows, row_cap,
             out_table, out_cycle, out_seat, out_info, out_mask, out_q, out_call, base, cap};
    for (long long i = 0; i < n; i++) {
        int r;
        long long o;
        if (!mr_head(V, i, &r, &o)) continue;
        u64 mask = 0;
        for (int a = 0; a < 46; a++) {
            V.out_q[o * 46 + a] = r < 0 ? 0.f : V.q[i * 46 + a];
            if (r >= 0 && V.masks[(long long)r * 46 + a]) mask |= 1ull << a;
        }
        mr_fields(V, i, r, o, mask);
    }
    return 0;
}
}  // extern "C"
