// mortal_b200 — mjai log text from the device event log: mortal_b200/mjai_log.py decode_events + attach_meta + dump_json_log
// (itself libriichi mjai/event.rs serde output, arena/result.rs:32-51) over the environment's event words (csrc/mjx_step.cuh
// `log_word`), the per-step log lengths and the sorted per-decision meta records. Byte for byte what the host writer produces,
// without the start_game / end_game lines (the host renders those: they carry the names).
//
// Device: k_mjai_render<FILL> (mjx_kernels.cu) runs one game per warp. Lane 0 queues the next 32 event starts (payload words are
// not self-describing), every lane sizes one event, a warp prefix sum places them; the fill pass writes them at those places.
// -DMJX_HOST_EMUL builds the same per-event code for one host lane (tests/host_emul/emul_mjai_write.cc).
#pragma once
#include "../../include/mjx.h"
#include "mjx_types.cuh"

namespace mjx {

constexpr int MW_WARPS = 4;

// ---------------------------------------------------------------- output sink: counts every byte, stores the ones below cap
struct MwOut {
    char* p;  // null: count only
    long long n, cap;
    MJX_DM void put(char c) {
        if (p && n < cap) p[n] = c;
        n++;
    }
    MJX_DM void puts(const char* s) {
        while (*s) put(*s++);
    }
};

MJX_D void mw_int(MwOut& o, long long v) {
    char b[24];
    int n = 0;
    unsigned long long u = v < 0 ? 0ull - (unsigned long long)v : (unsigned long long)v;
    do { b[n++] = (char)('0' + (int)(u % 10)); u /= 10; } while (u);
    if (v < 0) o.put('-');
    while (n) o.put(b[--n]);
}

// ---------------------------------------------------------------- shortest round-trip repr of an f32 widened to double
// The value is f * 2^e with f in [2^52, 2^53). Free-format shortest digits (Steele & White / Burger & Dybvig) with the last-digit
// decisions of CPython's _Py_dg_dtoa mode 0, which float.__repr__ uses. All arithmetic is exact on 224-bit integers:
//   e >= 0 (values >= 2^52): r = 4f * 2^e < 2^130, s = 4 * 10^k <= 4 * 10^39 < 2^132;
//   e <  0: s = 2^(2 - e) <= 2^203 (the smallest f32 subnormal 2^-149 is f = 2^52, e = -201), and r, m+, m- are scaled by
//           10^-k <= 10^45 < 2^150 with r ~ 2^54, so r < 2^205; every quantity the loop forms (10r, r + m+) stays below 10s < 2^207.
constexpr int MW_LIMBS = 7;  // 224 bits
struct MwBig {
    u32 v[MW_LIMBS];
};
MJX_D void mwb_set(MwBig& a, u64 x) {
    for (int i = 0; i < MW_LIMBS; i++) a.v[i] = 0;
    a.v[0] = (u32)x;
    a.v[1] = (u32)(x >> 32);
}
MJX_D void mwb_shl(MwBig& a, int n) {  // 0 <= n < 224
    const int w = n >> 5, b = n & 31;
    for (int i = MW_LIMBS - 1; i >= 0; i--) {
        const int j = i - w;
        u32 x = j >= 0 ? a.v[j] << b : 0;
        if (b && j - 1 >= 0) x |= a.v[j - 1] >> (32 - b);
        a.v[i] = x;
    }
}
MJX_D void mwb_mul(MwBig& a, u32 m) {
    u64 c = 0;
    for (int i = 0; i < MW_LIMBS; i++) {
        c += (u64)a.v[i] * m;
        a.v[i] = (u32)c;
        c >>= 32;
    }
}
MJX_D void mwb_mul_pow10(MwBig& a, int k) {
    for (; k >= 9; k -= 9) mwb_mul(a, 1000000000u);
    u32 m = 1;
    for (; k > 0; k--) m *= 10;
    if (m != 1) mwb_mul(a, m);
}
MJX_D void mwb_add(MwBig& out, const MwBig& a, const MwBig& b) {
    u64 c = 0;
    for (int i = 0; i < MW_LIMBS; i++) {
        c += (u64)a.v[i] + b.v[i];
        out.v[i] = (u32)c;
        c >>= 32;
    }
}
MJX_D void mwb_sub(MwBig& a, const MwBig& b) {  // a >= b
    i64 c = 0;
    for (int i = 0; i < MW_LIMBS; i++) {
        c += (i64)a.v[i] - b.v[i];
        a.v[i] = (u32)c;
        c >>= 32;
    }
}
MJX_D int mwb_cmp(const MwBig& a, const MwBig& b) {
    for (int i = MW_LIMBS - 1; i >= 0; i--)
        if (a.v[i] != b.v[i]) return a.v[i] < b.v[i] ? -1 : 1;
    return 0;
}
MJX_D bool mwb_zero(const MwBig& a) {
    for (int i = 0; i < MW_LIMBS; i++)
        if (a.v[i]) return false;
    return true;
}

MJX_D u32 mw_f32_bits(float x) {
#ifdef MJX_HOST_EMUL
    u32 b;
    memcpy(&b, &x, 4);
    return b;
#else
    return __float_as_uint(x);
#endif
}

// json.dumps(float(np.float32(x))) -> out (at most 24 bytes); returns the length
MJX_DN int mw_format_f32(float x, char* out) {
    const u32 bits = mw_f32_bits(x);
    const u32 ex = (bits >> 23) & 0xFF, fr = bits & 0x7FFFFF;
    int n = 0;
    auto cpy = [&](const char* s) { while (*s) out[n++] = *s++; };
    if (ex == 0xFF) {
        cpy(fr ? "NaN" : (bits >> 31) ? "-Infinity" : "Infinity");
        return n;
    }
    if (bits >> 31) out[n++] = '-';
    if (ex == 0 && fr == 0) {
        cpy("0.0");
        return n;
    }
    u64 f = ex ? ((1ull << 23) | fr) : fr;
    int e = ex ? (int)ex - 150 : -149;
    int bl = 0;
    while ((f >> bl) > 1) bl++;  // f < 2^(bl + 1)
    f <<= 52 - bl;
    e -= 52 - bl;
    // the widened mantissa ends in >= 29 zero bits, so it is even: both ends of the rounding interval belong to it; the lower
    // gap is half the upper one at a power of two (the double's biased exponent is > 1 for every f32)
    const bool lower_closer = f == (1ull << 52);
    MwBig r, s, mp, mm;
    mwb_set(r, f);
    mwb_set(s, 1);
    mwb_set(mp, 1);
    mwb_set(mm, 1);
    const int up = lower_closer ? 2 : 1;
    if (e >= 0) {
        mwb_shl(r, e + up);
        mwb_shl(s, up);
        mwb_shl(mp, e + up - 1);
        mwb_shl(mm, e);
    } else {
        mwb_shl(r, up);
        mwb_shl(s, up - e);
        mwb_shl(mp, up - 1);
    }
    // k: the smallest integer with r + m+ < s * 10^k; the estimate from the binary exponent is at most one off either way
    const int e2 = e + 52;  // 2^e2 <= value < 2^(e2 + 1)
    int k = (int)(((long long)e2 * 78913) >> 18);  // floor(e2 * log10(2)) for |e2| < 2^11
    if (k >= 0) mwb_mul_pow10(s, k);
    else {
        mwb_mul_pow10(r, -k);
        mwb_mul_pow10(mp, -k);
        mwb_mul_pow10(mm, -k);
    }
    MwBig t;
    for (;;) {
        mwb_add(t, r, mp);
        if (mwb_cmp(t, s) < 0) break;
        mwb_mul(s, 10);
        k++;
    }
    for (;;) {
        mwb_add(t, r, mp);
        mwb_mul(t, 10);
        if (mwb_cmp(t, s) >= 0) break;
        mwb_mul(r, 10);
        mwb_mul(mp, 10);
        mwb_mul(mm, 10);
        k--;
    }
    // digit loop; the decisions are _Py_dg_dtoa's (mode 0, even mantissa): j = cmp(r, m-), j1 = cmp(r + m+, s)
    char dg[24];
    int nd = 0;
    bool round_up = false;  // add one to the last digit, carrying through nines
    for (;;) {
        mwb_mul(r, 10);
        mwb_mul(mp, 10);
        mwb_mul(mm, 10);
        int d = 0;
        while (mwb_cmp(r, s) >= 0) {
            mwb_sub(r, s);
            d++;
        }
        const int j = mwb_cmp(r, mm);
        mwb_add(t, r, mp);
        const int j1 = mwb_cmp(t, s);
        if (j1 == 0) {
            if (d == 9) { dg[nd++] = 9; round_up = true; }
            else dg[nd++] = (char)(d + (j > 0));
            break;
        }
        if (j <= 0) {
            if (!mwb_zero(r) && j1 > 0) {
                MwBig r2 = r;
                mwb_mul(r2, 2);
                const int c = mwb_cmp(r2, s);
                if (c > 0 || (c == 0 && (d & 1))) {
                    if (d == 9) round_up = true;
                    else d++;
                }
            }
            dg[nd++] = (char)d;
            break;
        }
        if (j1 > 0) {
            if (d == 9) { dg[nd++] = 9; round_up = true; }
            else dg[nd++] = (char)(d + 1);
            break;
        }
        dg[nd++] = (char)d;
    }
    if (round_up) {  // dtoa's roundoff: drop trailing nines, bump the digit before; all nines -> "1", one more decimal place
        while (nd > 0 && dg[nd - 1] == 9) nd--;
        if (nd == 0) {
            dg[nd++] = 1;
            k++;
        } else dg[nd - 1]++;
    }
    // PyOS_double_to_string(x, 'r', 0, Py_DTSF_ADD_DOT_0): exponent form when decpt <= -4 or decpt > 16
    const int decpt = k;
    if (decpt <= -4 || decpt > 16) {
        out[n++] = (char)('0' + dg[0]);
        if (nd > 1) {
            out[n++] = '.';
            for (int i = 1; i < nd; i++) out[n++] = (char)('0' + dg[i]);
        }
        int x10 = decpt - 1;
        out[n++] = 'e';
        out[n++] = x10 < 0 ? '-' : '+';
        if (x10 < 0) x10 = -x10;
        if (x10 >= 100) out[n++] = (char)('0' + x10 / 100);
        out[n++] = (char)('0' + x10 / 10 % 10);
        out[n++] = (char)('0' + x10 % 10);
    } else if (decpt <= 0) {
        out[n++] = '0';
        out[n++] = '.';
        for (int i = 0; i < -decpt; i++) out[n++] = '0';
        for (int i = 0; i < nd; i++) out[n++] = (char)('0' + dg[i]);
    } else if (decpt < nd) {
        for (int i = 0; i < nd; i++) {
            if (i == decpt) out[n++] = '.';
            out[n++] = (char)('0' + dg[i]);
        }
    } else {
        for (int i = 0; i < nd; i++) out[n++] = (char)('0' + dg[i]);
        for (int i = nd; i < decpt; i++) out[n++] = '0';
        out[n++] = '.';
        out[n++] = '0';
    }
    return n;
}

// ---------------------------------------------------------------- the render view
struct MwView {
    const u64* words;  // [n_games, log_cap]
    const i32* lens;   // [n_games]
    int log_cap, n_games;
    // meta (bounds null: none): bounds[c * n_games + g] = game g's log length right after environment step c
    const i32* bounds;
    int n_steps, key_steps;
    // records sorted by key = ((game * key_steps + step) * 4 + seat) * 2 + kan_select
    const i64* rec_key;
    const i32* rec_info;  // [n_rec, 4]: action, flags (MJX_MW_REC_*), shanten, row (the order the rows came in)
    const u64* rec_mask;  // [n_rec] the 46 legal-action bits
    const float* rec_q;   // [n_rec, 46]
    const i64* rec_i64;   // [n_rec, 2]: batch_size, eval_time_ns
    long long n_rec;
    // count pass
    i32 *bytes, *status;
    // fill pass: games [g0, g1) at out + off[g] - off[g0]
    const i64* off;
    char* out;
    long long out_cap;
    int g0, g1;
};

MJX_D void mw_tile(MwOut& o, int t) {  // mjai_log.TILE_NAMES (tile.rs:12-19), t <= 37
    o.put('"');
    if (t < 27) {
        o.put((char)('1' + t % 9));
        o.put("mps"[t / 9]);
    } else if (t < 34) o.put("ESWNPFC"[t - 27]);
    else if (t < 37) {
        o.put('5');
        o.put("mps"[t - 34]);
        o.put('r');
    } else o.put('?');
    o.put('"');
}

MJX_D int mw_payload(int ty) { return ty == MJX_MW_T_START_KYOKU ? 9 : (ty == MJX_MW_T_HORA || ty == MJX_MW_T_RYUKYOKU) ? 2 : 0; }

// the word index after the event at i (n = the table's word count), or -MJX_MW_* when decode_events raises there
MJX_D int mw_next(const u64* w, int n, int i) {
    const int ty = (int)(w[i] & 0xFF);
    if (ty < MJX_MW_T_START_KYOKU || ty > MJX_MW_T_END_KYOKU) return -MJX_MW_CORRUPT;
    const int nx = i + 1 + mw_payload(ty);
    return nx > n ? -MJX_MW_TRUNCATED : nx;
}

MJX_D void mw_i32x4(MwOut& o, const u64* p) {
    o.put('[');
    for (int k = 0; k < 4; k++) {
        if (k) o.put(',');
        mw_int(o, (i32)(u32)(p[k >> 1] >> (32 * (k & 1))));
    }
    o.put(']');
}

MJX_D bool mw_acts(int ty, int a) {  // mjai_log.AGENT_EVENT_ACTIONS
    switch (ty) {
        case MJX_MW_T_DAHAI: return a >= 0 && a < 37;
        case MJX_MW_T_REACH: return a == 37;
        case MJX_MW_T_CHI: return a >= 38 && a <= 40;
        case MJX_MW_T_PON: return a == 41;
        case MJX_MW_T_DAIMINKAN: case MJX_MW_T_KAKAN: case MJX_MW_T_ANKAN: return a == 42;
        case MJX_MW_T_HORA: return a == 43;
        case MJX_MW_T_RYUKYOKU: return a == 44;
        default: return false;
    }
}

// the record of (g, step, seat, kan) or -1; equal keys: the last one, as the host recorder's dict keeps the last row
MJX_D long long mw_find(const MwView& V, int g, int step, int seat, int kan) {
    const i64 key = (((i64)g * V.key_steps + step) * 4 + seat) * 2 + kan;
    long long lo = 0, hi = V.n_rec;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (key < V.rec_key[mid]) hi = mid;
        else lo = mid + 1;
    }
    return lo > 0 && V.rec_key[lo - 1] == key ? lo - 1 : -1;
}

// make_meta's fields without None values: q_values, mask_bits, is_greedy of record q; batch_size, eval_time_ns, shanten,
// at_furiten of the main record m
MJX_DN void mw_meta_fields(MwOut& o, const MwView& V, long long q, long long m) {
    const u64 mask = V.rec_mask[q];
    o.puts("{\"q_values\":[");
    bool first = true;
    char b[32];
    for (int a = 0; a < 46; a++) {
        if (!((mask >> a) & 1)) continue;
        if (!first) o.put(',');
        first = false;
        const int len = mw_format_f32(V.rec_q[q * 46 + a], b);
        for (int i = 0; i < len; i++) o.put(b[i]);
    }
    o.puts("],\"mask_bits\":");
    mw_int(o, (long long)mask);
    o.puts(V.rec_info[q * 4 + 1] & MJX_MW_REC_GREEDY ? ",\"is_greedy\":true" : ",\"is_greedy\":false");
    o.puts(",\"batch_size\":");
    mw_int(o, V.rec_i64[m * 2]);
    o.puts(",\"eval_time_ns\":");
    mw_int(o, V.rec_i64[m * 2 + 1]);
    const int fl = V.rec_info[m * 4 + 1];
    if (fl & MJX_MW_REC_HAS_SHANTEN) {
        o.puts(",\"shanten\":");
        mw_int(o, V.rec_info[m * 4 + 2]);
    }
    if (fl & MJX_MW_REC_HAS_FURITEN) o.puts(fl & MJX_MW_REC_FURITEN ? ",\"at_furiten\":true" : ",\"at_furiten\":false");
}

// attach_meta for the agent event of type ty / actor at word offset off of game g: `,"meta":{...}` or nothing
MJX_DN void mw_meta(MwOut& o, const MwView& V, int g, int ty, int actor, int off) {
    if (!V.bounds || !V.n_rec) return;
    int lo = 0, hi = V.n_steps;  // bisect.bisect_right(bounds, off) - 1
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (off < V.bounds[(long long)mid * V.n_games + g]) hi = mid;
        else lo = mid + 1;
    }
    const int step = lo - 1;
    if (step < 0) return;
    long long m = -1;
    if (ty == MJX_MW_T_RYUKYOKU) {
        // the seat that declared it; several: the one whose row came first. attach_meta orders the seats by the first row of each
        // (table, seat) key, this takes the row of the key's last record: the two differ only for a key recorded twice in one
        // cycle, which the environment never emits (one row per seat and kan flag per step), and only one seat can have 44 anyway
        int best_row = 0;
        for (int s = 0; s < 4; s++) {
            const long long r = mw_find(V, g, step, s, 0);
            if (r < 0 || V.rec_info[r * 4] != 44) continue;
            if (m < 0 || V.rec_info[r * 4 + 3] < best_row) { m = r; best_row = V.rec_info[r * 4 + 3]; }
        }
    } else {
        const long long r = mw_find(V, g, step, actor, 0);
        if (r >= 0 && mw_acts(ty, V.rec_info[r * 4])) m = r;
    }
    if (m < 0) return;
    o.puts(",\"meta\":");
    mw_meta_fields(o, V, m, m);
    if (V.rec_info[m * 4] == 42) {
        const long long kr = mw_find(V, g, step, actor, 1);  // action 42 is never a ryukyoku's: the seat is the actor
        if (kr >= 0) {
            o.puts(",\"kan_select\":");
            mw_meta_fields(o, V, kr, m);
            o.put('}');
        }
    }
    o.put('}');
}

// the JSON line (with its "\n") of the event at word i of game g (w / n: the game's words); MJX_MW_OK or the reason
// decode_events raises. i must be an event start with its payload inside n (mw_next).
MJX_DN int mw_event(MwOut& o, const MwView& V, int g, const u64* w, int i) {
    const u64 x = w[i];
    const int ty = (int)(x & 0xFF), actor = (int)(x >> 8) & 3, target = (int)(x >> 10) & 3, pai = (int)(x >> 12) & 0xFF;
    const bool tsumogiri = (x >> 20) & 1;
    const int aux = (int)(x >> 21) & 7;
    int c[5];
    for (int k = 0; k < 4; k++) c[k] = (int)(x >> (24 + 8 * k)) & 0xFF;
    c[4] = (int)(x >> 56) & 0xFF;
    // the tile indices decode_events reads (an index past 37 is an IndexError there)
    int nc = 0;
    bool need_pai = false;
    switch (ty) {
        case MJX_MW_T_START_KYOKU: {
            if (27 + c[0] / 4 > 37) return MJX_MW_CORRUPT;
            need_pai = true;
            for (int k = 0; k < 52; k++)
                if ((int)((w[i + 3 + k / 8] >> (8 * (k % 8))) & 0xFF) > 37) return MJX_MW_CORRUPT;
            break;
        }
        case MJX_MW_T_TSUMO: case MJX_MW_T_DAHAI: case MJX_MW_T_DORA: need_pai = true; break;
        case MJX_MW_T_CHI: case MJX_MW_T_PON: need_pai = true; nc = 2; break;
        case MJX_MW_T_DAIMINKAN: case MJX_MW_T_KAKAN: need_pai = true; nc = 3; break;
        case MJX_MW_T_ANKAN: nc = 4; break;
        case MJX_MW_T_HORA: nc = aux < 5 ? aux : 5; break;
        default: break;
    }
    if (need_pai && pai > 37) return MJX_MW_CORRUPT;
    for (int k = 0; k < nc; k++)
        if (c[k] > 37) return MJX_MW_CORRUPT;
    o.puts("{\"type\":");
    switch (ty) {
        case MJX_MW_T_START_KYOKU: {
            o.puts("\"start_kyoku\",\"bakaze\":");
            mw_tile(o, 27 + c[0] / 4);
            o.puts(",\"dora_marker\":");
            mw_tile(o, pai);
            o.puts(",\"kyoku\":");
            mw_int(o, c[3] + 1);
            o.puts(",\"honba\":");
            mw_int(o, c[1]);
            o.puts(",\"kyotaku\":");
            mw_int(o, c[2]);
            o.puts(",\"oya\":");
            mw_int(o, c[3]);
            o.puts(",\"scores\":");
            mw_i32x4(o, w + i + 1);
            o.puts(",\"tehais\":[");
            for (int s = 0; s < 4; s++) {
                o.puts(s ? ",[" : "[");
                for (int k = 0; k < 13; k++) {
                    const int b = 13 * s + k;
                    if (k) o.put(',');
                    mw_tile(o, (int)((w[i + 3 + b / 8] >> (8 * (b % 8))) & 0xFF));
                }
                o.put(']');
            }
            o.put(']');
            break;
        }
        case MJX_MW_T_TSUMO:
        case MJX_MW_T_DAHAI:
            o.puts(ty == MJX_MW_T_TSUMO ? "\"tsumo\",\"actor\":" : "\"dahai\",\"actor\":");
            mw_int(o, actor);
            o.puts(",\"pai\":");
            mw_tile(o, pai);
            if (ty == MJX_MW_T_DAHAI) o.puts(tsumogiri ? ",\"tsumogiri\":true" : ",\"tsumogiri\":false");
            break;
        case MJX_MW_T_CHI: case MJX_MW_T_PON: case MJX_MW_T_DAIMINKAN: case MJX_MW_T_KAKAN: case MJX_MW_T_ANKAN:
            o.puts(ty == MJX_MW_T_CHI ? "\"chi\"" : ty == MJX_MW_T_PON ? "\"pon\"" : ty == MJX_MW_T_DAIMINKAN ? "\"daiminkan\""
                   : ty == MJX_MW_T_KAKAN ? "\"kakan\"" : "\"ankan\"");
            o.puts(",\"actor\":");
            mw_int(o, actor);
            if (ty == MJX_MW_T_CHI || ty == MJX_MW_T_PON || ty == MJX_MW_T_DAIMINKAN) {
                o.puts(",\"target\":");
                mw_int(o, target);
            }
            if (ty != MJX_MW_T_ANKAN) {
                o.puts(",\"pai\":");
                mw_tile(o, pai);
            }
            o.puts(",\"consumed\":[");
            for (int k = 0; k < nc; k++) {
                if (k) o.put(',');
                mw_tile(o, c[k]);
            }
            o.put(']');
            break;
        case MJX_MW_T_DORA:
            o.puts("\"dora\",\"dora_marker\":");
            mw_tile(o, pai);
            break;
        case MJX_MW_T_REACH:
        case MJX_MW_T_REACH_ACCEPTED:
            o.puts(ty == MJX_MW_T_REACH ? "\"reach\",\"actor\":" : "\"reach_accepted\",\"actor\":");
            mw_int(o, actor);
            break;
        case MJX_MW_T_HORA:
            o.puts("\"hora\",\"actor\":");
            mw_int(o, actor);
            o.puts(",\"target\":");
            mw_int(o, target);
            o.puts(",\"deltas\":");
            mw_i32x4(o, w + i + 1);
            o.puts(",\"ura_markers\":[");
            for (int k = 0; k < nc; k++) {
                if (k) o.put(',');
                mw_tile(o, c[k]);
            }
            o.put(']');
            break;
        case MJX_MW_T_RYUKYOKU:
            o.puts("\"ryukyoku\",\"deltas\":");
            mw_i32x4(o, w + i + 1);
            break;
        default: o.puts("\"end_kyoku\""); break;
    }
    if (ty != MJX_MW_T_START_KYOKU && ty != MJX_MW_T_TSUMO && ty != MJX_MW_T_DORA && ty != MJX_MW_T_REACH_ACCEPTED &&
        ty != MJX_MW_T_END_KYOKU)
        mw_meta(o, V, g, ty, actor, i);
    o.puts("}\n");
    return MJX_MW_OK;
}

// the words of game g inside the log capacity (reads never pass it); MJX_MW_CAPACITY for a log longer than that
MJX_D int mw_game_words(const MwView& V, int g, const u64** w, int* n) {
    const int len = V.lens[g];
    *w = V.words + (long long)g * V.log_cap;
    *n = len < 0 ? 0 : len > V.log_cap ? V.log_cap : len;
    return len < 0 || len > V.log_cap ? MJX_MW_CAPACITY : MJX_MW_OK;
}


// ---------------------------------------------------------------- per-decision meta records (k_meta_record, mjx_meta_record_dev)
// One record per decision row of an agent call: what _MetaRecorder.add_agent / add_rows keep, appended on the device at
// base + i for the call's i-th row (row = idx[i], or i without idx).
struct MrView {
    long long n;
    const i64* idx;       // [n] rows of the call or null
    const float* q;       // [n, 46] the call's Q-values, in call order
    const u8* greedy;     // [n] or null (every row greedy)
    const i32* call_ids;  // [n] or null (every row: `call`)
    int call, cycle;
    const i32* row_table;
    const u8* row_seat;   // seat | kan_select << 2
    const i64* actions;   // [row_cap]
    const u8* masks;      // [row_cap, 46]
    const float* obs;     // [row_cap, obs_rows, 34] v4 observation (shanten / furiten), or null
    int obs_rows, row_cap;
    i32 *out_table, *out_cycle;
    u8* out_seat;
    i32* out_info;  // [cap, 4] action, flags, shanten, row
    u64* out_mask;
    float* out_q;   // [cap, 46]
    i32* out_call;
    long long base, cap;
};

// everything of record i except the mask bits and the Q-values (lane 0's part of the kernel); false: nothing to write
MJX_D bool mr_head(const MrView& V, long long i, int* row, long long* o) {
    *o = V.base + i;
    if (*o < 0 || *o >= V.cap) return false;
    const long long r = V.idx ? V.idx[i] : i;
    *row = (r < 0 || r >= V.row_cap) ? -1 : (int)r;
    return true;
}
MJX_D void mr_fields(const MrView& V, long long i, int r, long long o, u64 mask) {
    if (r < 0) {  // a row index outside the env's rows: a record no event can match
        V.out_table[o] = -1; V.out_cycle[o] = V.cycle; V.out_seat[o] = 0;
        V.out_info[o * 4] = -1; V.out_info[o * 4 + 1] = 0; V.out_info[o * 4 + 2] = 0; V.out_info[o * 4 + 3] = 0;
        V.out_mask[o] = 0; V.out_call[o] = -1;
        return;
    }
    int flags = (!V.greedy || V.greedy[i]) ? MJX_MW_REC_GREEDY : 0, sh = 0;
    if (V.obs) {  // _MetaRecorder.add_rows: argmax (first maximum) of v4 rows 862-868 at column 0, row 861 > 0
        const float* p = V.obs + (long long)r * V.obs_rows * 34;
        float best = p[862 * 34];
        for (int k = 1; k < 7; k++)
            if (p[(862 + k) * 34] > best) { best = p[(862 + k) * 34]; sh = k; }
        flags |= MJX_MW_REC_HAS_SHANTEN | MJX_MW_REC_HAS_FURITEN | (p[861 * 34] > 0 ? MJX_MW_REC_FURITEN : 0);
    }
    V.out_table[o] = V.row_table[r];
    V.out_cycle[o] = V.cycle;
    V.out_seat[o] = V.row_seat[r];
    V.out_info[o * 4] = (i32)V.actions[r];
    V.out_info[o * 4 + 1] = flags;
    V.out_info[o * 4 + 2] = sh;
    V.out_info[o * 4 + 3] = r;
    V.out_mask[o] = mask;
    V.out_call[o] = V.call_ids ? V.call_ids[i] : V.call;
}

}  // namespace mjx
