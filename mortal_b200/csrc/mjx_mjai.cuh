// mortal_b200 — mjai log text -> the event words of csrc/mjx_step.cuh `log_word` (what mortal_b200/dataset_codec.py
// encode_events and validate_logs.encode_log produce from json.loads of every line).
//
// The decoder ACCEPTS a log only when it can show that Python reads every line as it does; everything else is DECLINED and left
// to the host code. Accepted logs decode bit-identically to the host path; a declined log costs speed, never correctness.
// Per line (what str.splitlines() yields for a text whose only separators are "\n" and "\r\n"):
//   * blank = spaces and tabs only; any '\r' not ending the line, and any other separator splitlines honours (\x0b \x0c
//     \x1c-\x1e U+0085 U+2028 U+2029, also inside strings), declines the log;
//   * an event = one JSON object under the rules of Python's json: strings without raw control characters and with only
//     the escapes \" \\ \/ \b \f \n \r \t \uXXXX, the JSON number grammar (no NaN / Infinity), true / false / null, nesting up
//     to MJAI_DEPTH, spaces and tabs as whitespace, nothing after the closing brace;
//   * the top-level keys of csrc/mjx_mjai.cuh `mjai_key` are the fields dataset_codec reads: one with an escape in it, or one
//     given twice (Python keeps the last), declines; other keys (`meta`, `names`, ...) are skipped by the validating scanner;
//   * the fields the event type needs must pass dataset_codec.check_event exactly as written (integers without fraction or
//     exponent and within range, tile names as plain strings, the right `consumed` length, a wind as `bakaze`), else decline.
// A log without events declines too. Non-ASCII bytes may only appear inside strings and must be valid UTF-8 there.
//
// Device: one warp per log (k_mjai_decode in mjx_kernels.cu) finds the line ends with ballots over 32-byte windows, queues
// them, and parses 32 lines at a time, one per lane; event, kyoku and hora positions come from ballot prefix counts. The count
// pass writes mjx_mjai_counts; the fill pass runs the same walk and writes the arrays. -DMJX_HOST_EMUL builds the line parser
// for tests/host_emul/emul_mjai.cc.
#pragma once
#include "../../include/mjx.h"
#include "mjx_types.cuh"

namespace mjx {

constexpr int MJAI_DEPTH = 32;        // deepest nesting of a skipped value (Python's own limit is its recursion limit)
constexpr int MJAI_NUM_MAX = 256;     // longest number token accepted (Python refuses integers of over 4300 digits)
constexpr int MJAI_KYOKU_WORDS = 19;  // csrc/mjx_replay.cuh REPLAY_KYOKU_WORDS
enum : int { MJ_BLANK = 0, MJ_EVENT = 1, MJ_DECLINE = 2 };
enum : int { MJT_START_KYOKU = 1, MJT_TSUMO, MJT_DAHAI, MJT_CHI, MJT_PON, MJT_DAIMINKAN, MJT_KAKAN, MJT_ANKAN, MJT_DORA, MJT_REACH,
             MJT_REACH_ACCEPTED, MJT_HORA, MJT_RYUKYOKU, MJT_END_KYOKU, MJT_START_GAME, MJT_END_GAME };
enum : int { K_TYPE, K_ACTOR, K_TARGET, K_PAI, K_TSUMOGIRI, K_CONSUMED, K_BAKAZE, K_DORA_MARKER, K_KYOKU, K_HONBA, K_KYOTAKU,
             K_OYA, K_SCORES, K_TEHAIS, K_DELTAS, K_URA, K_COUNT };

struct MjCur {
    const u8* p;
    long long i, e;  // cursor and end (exclusive) of the line: every read is bounds-checked against e
};

MJX_D int mj_peek(const MjCur& c) { return c.i < c.e ? (int)c.p[c.i] : -1; }
MJX_D void mj_ws(MjCur& c) {
    while (c.i < c.e && (c.p[c.i] == ' ' || c.p[c.i] == '\t')) c.i++;
}
MJX_D bool mj_eq(const u8* p, long long b, long long e, const char* s) {
    long long k = 0;
    for (; s[k]; k++)
        if (b + k >= e || p[b + k] != (u8)s[k]) return false;
    return b + k == e;
}

// the length of the UTF-8 sequence at c.i (a byte >= 0x80) as Python's strict decoder reads it; 0 when it is invalid or is one of
// the line breaks str.splitlines() honours (U+0085, U+2028, U+2029)
MJX_D int mj_utf8(const MjCur& c) {
    const int b0 = c.p[c.i];
    const int n = b0 >= 0xC2 && b0 <= 0xDF ? 2 : b0 >= 0xE0 && b0 <= 0xEF ? 3 : b0 >= 0xF0 && b0 <= 0xF4 ? 4 : 0;
    if (n == 0 || c.i + n > c.e) return 0;
    const int b1 = c.p[c.i + 1];
    const int lo = b0 == 0xE0 ? 0xA0 : b0 == 0xF0 ? 0x90 : 0x80, hi = b0 == 0xED ? 0x9F : b0 == 0xF4 ? 0x8F : 0xBF;
    if (b1 < lo || b1 > hi) return 0;
    for (int k = 2; k < n; k++)
        if ((c.p[c.i + k] & 0xC0) != 0x80) return 0;
    if (b0 == 0xC2 && b1 == 0x85) return 0;
    if (b0 == 0xE2 && b1 == 0x80 && (c.p[c.i + 2] == 0xA8 || c.p[c.i + 2] == 0xA9)) return 0;
    return n;
}

// a string at c.i ('"'): true when Python's json reads it (strict mode); *esc = it holds an escape
MJX_D bool mj_string(MjCur& c, bool* esc) {
    *esc = false;
    c.i++;
    while (c.i < c.e) {
        const int ch = c.p[c.i];
        if (ch == '"') { c.i++; return true; }
        if (ch < 0x20) return false;
        if (ch == '\\') {
            *esc = true;
            if (c.i + 1 >= c.e) return false;
            const int x = c.p[c.i + 1];
            if (x == 'u') {
                if (c.i + 6 > c.e) return false;
                for (int k = 2; k < 6; k++) {
                    const int h = c.p[c.i + k];
                    if (!((h >= '0' && h <= '9') || (h >= 'a' && h <= 'f') || (h >= 'A' && h <= 'F'))) return false;
                }
                c.i += 6;
                continue;
            }
            if (x != '"' && x != '\\' && x != '/' && x != 'b' && x != 'f' && x != 'n' && x != 'r' && x != 't') return false;
            c.i += 2;
            continue;
        }
        if (ch >= 0x80) {
            const int n = mj_utf8(c);
            if (n == 0) return false;
            c.i += n;
            continue;
        }
        c.i++;
    }
    return false;
}

// a number at c.i: the JSON grammar -?(0|[1-9][0-9]*)(\.[0-9]+)?([eE][+-]?[0-9]+)?, at most MJAI_NUM_MAX bytes
MJX_D bool mj_number(MjCur& c) {
    const long long b = c.i;
    if (mj_peek(c) == '-') c.i++;
    int ch = mj_peek(c);
    if (ch == '0') c.i++;
    else if (ch >= '1' && ch <= '9') { while (mj_peek(c) >= '0' && mj_peek(c) <= '9') c.i++; }
    else return false;
    if (mj_peek(c) == '.') {
        c.i++;
        if (!(mj_peek(c) >= '0' && mj_peek(c) <= '9')) return false;
        while (mj_peek(c) >= '0' && mj_peek(c) <= '9') c.i++;
    }
    if (mj_peek(c) == 'e' || mj_peek(c) == 'E') {
        c.i++;
        if (mj_peek(c) == '+' || mj_peek(c) == '-') c.i++;
        if (!(mj_peek(c) >= '0' && mj_peek(c) <= '9')) return false;
        while (mj_peek(c) >= '0' && mj_peek(c) <= '9') c.i++;
    }
    return c.i - b <= MJAI_NUM_MAX;
}

MJX_D bool mj_literal(MjCur& c, const char* s) {
    long long k = 0;
    for (; s[k]; k++)
        if (c.i + k >= c.e || c.p[c.i + k] != (u8)s[k]) return false;
    c.i += k;
    return true;
}

// an object key, the whitespace around it and the ':' (c.i at the key's '"')
MJX_D bool mj_key(MjCur& c, long long* kb, long long* ke, bool* esc) {
    if (mj_peek(c) != '"') return false;
    *kb = c.i + 1;
    if (!mj_string(c, esc)) return false;
    *ke = c.i - 1;
    mj_ws(c);
    if (mj_peek(c) != ':') return false;
    c.i++;
    mj_ws(c);
    return true;
}

// Skips one value at c.i (no leading whitespace). False when Python's json would reject it or it nests deeper than MJAI_DEPTH.
MJX_D bool mj_skip(MjCur& c) {
    u32 arr = 0;  // bit d: level d is an array
    int depth = 0;
    for (;;) {
        const int ch = mj_peek(c);
        bool esc;
        long long kb, ke;
        if (ch == '{' || ch == '[') {
            if (depth == MJAI_DEPTH) return false;
            const bool a = ch == '[';
            arr = a ? arr | (1u << depth) : arr & ~(1u << depth);
            depth++;
            c.i++;
            mj_ws(c);
            if (mj_peek(c) == (a ? ']' : '}')) { c.i++; depth--; }
            else {
                if (!a && !mj_key(c, &kb, &ke, &esc)) return false;
                continue;  // the first member's value
            }
        } else if (ch == '"') {
            if (!mj_string(c, &esc)) return false;
        } else if (ch == '-' || (ch >= '0' && ch <= '9')) {
            if (!mj_number(c)) return false;
        } else if (!(mj_literal(c, "true") || mj_literal(c, "false") || mj_literal(c, "null"))) {
            return false;
        }
        // after a value: close containers until a ',' starts the next member
        for (;;) {
            if (depth == 0) return true;
            mj_ws(c);
            const bool a = (arr >> (depth - 1)) & 1;
            const int nx = mj_peek(c);
            if (nx == ',') {
                c.i++;
                mj_ws(c);
                if (!a && !mj_key(c, &kb, &ke, &esc)) return false;
                break;
            }
            if (nx != (a ? ']' : '}')) return false;
            c.i++;
            depth--;
        }
    }
}

// the fields dataset_codec reads (-1: any other key)
MJX_CONST char MJ_KEYS[K_COUNT][12] = {"type", "actor", "target", "pai", "tsumogiri", "consumed", "bakaze", "dora_marker", "kyoku",
                                       "honba", "kyotaku", "oya", "scores", "tehais", "deltas", "ura_markers"};
MJX_CONST char MJ_TYPES[16][16] = {"start_kyoku", "tsumo", "dahai", "chi", "pon", "daiminkan", "kakan", "ankan", "dora", "reach",
                                   "reach_accepted", "hora", "ryukyoku", "end_kyoku", "start_game", "end_game"};

MJX_D int mjai_key(const u8* p, long long b, long long e) {
    for (int k = 0; k < K_COUNT; k++)
        if (mj_eq(p, b, e, MJ_KEYS[k])) return k;
    return -1;
}

// the MJT_* code of a type name (the log_word type), -1 for any other
MJX_D int mjai_type(const u8* p, long long b, long long e) {
    for (int k = 0; k < 16; k++)
        if (mj_eq(p, b, e, MJ_TYPES[k])) return k + 1;
    return -1;
}

// a value span holding a plain string (no escape) -> its bytes [*sb, *se)
MJX_D bool mj_plain_string(const u8* p, long long b, long long e, long long* sb, long long* se) {
    if (b >= e || p[b] != '"' || p[e - 1] != '"' || e - b < 2) return false;
    for (long long k = b + 1; k < e - 1; k++)
        if (p[k] == '\\') return false;
    *sb = b + 1; *se = e - 1;
    return true;
}

// tile.rs names (mjai_log.TILE_NAMES ids 0..37), with Tile::augment (manzu <-> pinzu, red fives stay red) when `aug`
MJX_D int mj_tile(const u8* p, long long b, long long e, bool aug) {
    long long sb, se;
    if (!mj_plain_string(p, b, e, &sb, &se)) return -1;
    const long long n = se - sb;
    int t = -1;
    if (n == 1) {
        switch (p[sb]) {
            case 'E': t = 27; break; case 'S': t = 28; break; case 'W': t = 29; break; case 'N': t = 30; break;
            case 'P': t = 31; break; case 'F': t = 32; break; case 'C': t = 33; break; case '?': t = 37; break;
            default: return -1;
        }
    } else if (n == 2 || n == 3) {
        const int d = p[sb], s = p[sb + 1];
        const int suit = s == 'm' ? 0 : s == 'p' ? 1 : s == 's' ? 2 : -1;
        if (d < '1' || d > '9' || suit < 0) return -1;
        if (n == 2) t = suit * 9 + (d - '1');
        else if (d == '5' && p[sb + 2] == 'r') t = 34 + suit;
        else return -1;
    } else {
        return -1;
    }
    if (aug) {
        if (t < 9) t += 9;
        else if (t < 18) t -= 9;
        else if (t == 34 || t == 35) t ^= 34 ^ 35;
    }
    return t;
}

// an integer written without fraction or exponent (not a bool), within [lo, hi]
MJX_D bool mj_int(const u8* p, long long b, long long e, long long lo, long long hi, long long* v) {
    long long k = b;
    const bool neg = k < e && p[k] == '-';
    if (neg) k++;
    if (k >= e || e - k > 12) return false;
    long long x = 0;
    for (; k < e; k++) {
        if (p[k] < '0' || p[k] > '9') return false;
        x = x * 10 + (p[k] - '0');
    }
    x = neg ? -x : x;
    if (x < lo || x > hi) return false;
    *v = x;
    return true;
}

// iterates the elements of an array value [b, e) (already validated by mj_skip): mj_arr_begin, then mj_arr_next per element
MJX_D bool mj_arr_begin(const u8* p, long long b, long long e, MjCur& c) {
    if (b >= e || p[b] != '[') return false;
    c.p = p; c.i = b + 1; c.e = e;
    return true;
}
MJX_D bool mj_arr_next(MjCur& c, long long* eb, long long* ee) {
    mj_ws(c);
    if (mj_peek(c) == ',') { c.i++; mj_ws(c); }
    if (mj_peek(c) == ']' || c.i >= c.e) return false;
    *eb = c.i;
    mj_skip(c);
    *ee = c.i;
    return true;
}

// an array of exactly n integers within [lo, hi] -> v[0..n)
MJX_D bool mj_ints(const u8* p, long long b, long long e, int n, long long lo, long long hi, long long* v) {
    MjCur c;
    long long eb, ee;
    if (!mj_arr_begin(p, b, e, c)) return false;
    int k = 0;
    for (; mj_arr_next(c, &eb, &ee); k++)
        if (k >= n || !mj_int(p, eb, ee, lo, hi, &v[k])) return false;
    return k == n;
}

MJX_D bool mj_is_null(const u8* p, long long b, long long e) { return mj_eq(p, b, e, "null"); }

MJX_D u64 mj_word(int ty, int actor, int target, int pai, int tsumogiri, int c0, int c1, int c2, int c3) {
    return (u64)ty | (u64)(actor & 3) << 8 | (u64)(target & 3) << 10 | (u64)(pai & 0xFF) << 12 | (u64)(tsumogiri & 1) << 20 |
           (u64)c0 << 24 | (u64)c1 << 32 | (u64)c2 << 40 | (u64)c3 << 48;
}

struct MjaiLine {
    int kind;  // MJ_BLANK / MJ_EVENT / MJ_DECLINE
    int ty;    // the event type (MJT_*) of an event
    u64 word;
};

// One line [b, e) of the text (without its line break) -> MjaiLine. For an event, `pay` (MJAI_KYOKU_WORDS words, start_kyoku) and
// `hora` (MJX_HORA_WORDS words) receive the side data when non-null. Never reads outside [b, e).
MJX_DN MjaiLine mjai_parse_line(const u8* p, long long b, long long e, bool aug, u64* pay, u64* hora) {
    MjaiLine L{MJ_DECLINE, 0, 0};
    MjCur c{p, b, e};
    mj_ws(c);
    if (c.i == e) { L.kind = MJ_BLANK; return L; }
    if (mj_peek(c) != '{') return L;
    int vb[K_COUNT], ve[K_COUNT];  // value spans relative to b; -1 = absent
    for (int k = 0; k < K_COUNT; k++) vb[k] = ve[k] = -1;
    c.i++;
    mj_ws(c);
    if (mj_peek(c) == '}') c.i++;
    else {
        for (;;) {
            long long kb, ke;
            bool esc;
            if (!mj_key(c, &kb, &ke, &esc)) return L;
            if (esc) return L;
            const long long v0 = c.i;
            if (!mj_skip(c)) return L;
            const int k = mjai_key(p, kb, ke);
            if (k >= 0) {
                if (vb[k] >= 0) return L;
                vb[k] = (int)(v0 - b); ve[k] = (int)(c.i - b);
            }
            mj_ws(c);
            const int nx = mj_peek(c);
            c.i++;
            if (nx == '}') break;
            if (nx != ',') return L;
            mj_ws(c);
        }
    }
    mj_ws(c);
    if (c.i != e) return L;
    // the fields (check_event, then encode_events)
#define MJ_HAS(k) (vb[k] >= 0)
#define MJ_B(k) (b + vb[k])
#define MJ_E(k) (b + ve[k])
    long long sb, se;
    if (!MJ_HAS(K_TYPE) || !mj_plain_string(p, MJ_B(K_TYPE), MJ_E(K_TYPE), &sb, &se)) return L;
    const int ty = mjai_type(p, sb, se);
    if (ty < 0) return L;
    long long actor = 0, target = 0;
    const bool has_actor = ty == MJT_TSUMO || ty == MJT_DAHAI || ty == MJT_CHI || ty == MJT_PON || ty == MJT_DAIMINKAN ||
                           ty == MJT_KAKAN || ty == MJT_ANKAN || ty == MJT_REACH || ty == MJT_REACH_ACCEPTED || ty == MJT_HORA;
    const bool has_target = ty == MJT_CHI || ty == MJT_PON || ty == MJT_DAIMINKAN || ty == MJT_HORA;
    if (has_actor && (!MJ_HAS(K_ACTOR) || !mj_int(p, MJ_B(K_ACTOR), MJ_E(K_ACTOR), 0, 3, &actor))) return L;
    if (has_target && (!MJ_HAS(K_TARGET) || !mj_int(p, MJ_B(K_TARGET), MJ_E(K_TARGET), 0, 3, &target))) return L;
    int pai = 37;
    if (ty == MJT_TSUMO || ty == MJT_DAHAI || ty == MJT_CHI || ty == MJT_PON || ty == MJT_DAIMINKAN || ty == MJT_KAKAN) {
        if (!MJ_HAS(K_PAI) || (pai = mj_tile(p, MJ_B(K_PAI), MJ_E(K_PAI), aug)) < 0) return L;
    }
    int cons[4] = {37, 37, 37, 37};
    const bool has_cons = ty == MJT_CHI || ty == MJT_PON || ty == MJT_DAIMINKAN || ty == MJT_KAKAN || ty == MJT_ANKAN;
    if (has_cons) {
        const int n = ty == MJT_CHI || ty == MJT_PON ? 2 : ty == MJT_ANKAN ? 4 : 3;
        MjCur a;
        long long eb, ee;
        if (!MJ_HAS(K_CONSUMED) || !mj_arr_begin(p, MJ_B(K_CONSUMED), MJ_E(K_CONSUMED), a)) return L;
        int k = 0;
        for (; mj_arr_next(a, &eb, &ee); k++)
            if (k >= n || (cons[k] = mj_tile(p, eb, ee, aug)) < 0) return L;
        if (k != n) return L;
    }
    int tsumogiri = 0;
    if (ty == MJT_DAHAI) {
        if (!MJ_HAS(K_TSUMOGIRI)) return L;
        if (mj_eq(p, MJ_B(K_TSUMOGIRI), MJ_E(K_TSUMOGIRI), "true")) tsumogiri = 1;
        else if (!mj_eq(p, MJ_B(K_TSUMOGIRI), MJ_E(K_TSUMOGIRI), "false")) return L;
    }
    if (ty == MJT_DORA && (!MJ_HAS(K_DORA_MARKER) || (pai = mj_tile(p, MJ_B(K_DORA_MARKER), MJ_E(K_DORA_MARKER), aug)) < 0)) return L;
    u64 w;
    if (ty == MJT_START_KYOKU) {
        long long oya, kyoku, honba, kyotaku, sc[4];
        if (!MJ_HAS(K_OYA) || !mj_int(p, MJ_B(K_OYA), MJ_E(K_OYA), 0, 3, &oya)) return L;
        const int bakaze = MJ_HAS(K_BAKAZE) ? mj_tile(p, MJ_B(K_BAKAZE), MJ_E(K_BAKAZE), aug) : -1;
        if (bakaze < 27 || bakaze > 30) return L;  // not a tile: PARSE; not a wind: UNSUPPORTED
        if (!MJ_HAS(K_DORA_MARKER) || (pai = mj_tile(p, MJ_B(K_DORA_MARKER), MJ_E(K_DORA_MARKER), aug)) < 0) return L;
        if (!MJ_HAS(K_KYOKU) || !mj_int(p, MJ_B(K_KYOKU), MJ_E(K_KYOKU), 1, 4, &kyoku)) return L;
        if (!MJ_HAS(K_HONBA) || !mj_int(p, MJ_B(K_HONBA), MJ_E(K_HONBA), 0, 255, &honba)) return L;
        if (!MJ_HAS(K_KYOTAKU) || !mj_int(p, MJ_B(K_KYOTAKU), MJ_E(K_KYOTAKU), 0, 255, &kyotaku)) return L;
        if (!MJ_HAS(K_SCORES) || !mj_ints(p, MJ_B(K_SCORES), MJ_E(K_SCORES), 4, -2147483648LL, 2147483647LL, sc)) return L;
        if (!MJ_HAS(K_TEHAIS)) return L;
        MjCur hands, h;
        long long hb, he, eb, ee;
        if (!mj_arr_begin(p, MJ_B(K_TEHAIS), MJ_E(K_TEHAIS), hands)) return L;
        int s = 0;
        u64 acc = 0;
        for (; mj_arr_next(hands, &hb, &he); s++) {
            if (s >= 4 || !mj_arr_begin(p, hb, he, h)) return L;
            int k = 0;
            for (; mj_arr_next(h, &eb, &ee); k++) {
                int t;
                if (k >= 13 || (t = mj_tile(p, eb, ee, aug)) < 0) return L;
                const int i = 13 * s + k;
                acc |= (u64)t << (8 * (i % 8));
                if (i % 8 == 7) { if (pay) pay[2 + i / 8] = acc; acc = 0; }
            }
            if (k != 13) return L;
        }
        if (s != 4) return L;
        if (pay) {
            pay[0] = (u64)(u32)sc[0] | (u64)(u32)sc[1] << 32;
            pay[1] = (u64)(u32)sc[2] | (u64)(u32)sc[3] << 32;
            pay[2 + 6] = acc | 0x2525252500000000ull;  // tiles 48..51, then `?` = 37 = 0x25 from byte 52 on
            for (int k = 9; k < MJAI_KYOKU_WORDS; k++) pay[k] = 0x2525252525252525ull;
        }
        w = mj_word(ty, 0, 0, pai, 0, (int)((bakaze - 27) * 4 + kyoku - 1), (int)honba, (int)kyotaku, (int)oya);
    } else if (ty == MJT_HORA || ty == MJT_RYUKYOKU) {
        long long d[4] = {0, 0, 0, 0};
        const bool has_d = MJ_HAS(K_DELTAS) && !mj_is_null(p, MJ_B(K_DELTAS), MJ_E(K_DELTAS));
        if (has_d && !mj_ints(p, MJ_B(K_DELTAS), MJ_E(K_DELTAS), 4, -2147483648LL, 2147483647LL, d)) return L;
        if (ty == MJT_HORA) {
            const bool has_u = MJ_HAS(K_URA) && !mj_is_null(p, MJ_B(K_URA), MJ_E(K_URA));
            u64 w1 = 0;
            int n = 0;
            if (has_u) {
                MjCur a;
                long long eb, ee;
                if (!mj_arr_begin(p, MJ_B(K_URA), MJ_E(K_URA), a)) return L;
                for (; mj_arr_next(a, &eb, &ee); n++) {
                    const int t = mj_tile(p, eb, ee, aug);
                    if (t < 0) return L;
                    if (n < 5) w1 |= (u64)t << (8 * n);
                }
            }
            if (hora) {
                hora[0] = (has_d ? (u64)(u32)d[actor] : 0) | (u64)has_d << 32 | (u64)has_u << 33 | (u64)(n < 15 ? n : 15) << 36;
                hora[1] = w1;
            }
            w = mj_word(ty, (int)actor, (int)target, 37, 0, 0, 0, 0, 0);
        } else {
            w = mj_word(ty, 0, 0, 37, 0, 0, 0, 0, 0);
        }
    } else if (has_cons) {  // chi / pon / daiminkan / kakan: consumed padded with `?`; ankan: its four tiles
        w = mj_word(ty, (int)actor, (int)target, pai, 0, cons[0], cons[1], cons[2], cons[3]);
    } else {
        w = mj_word(ty, (int)actor, 0, pai, tsumogiri, 0, 0, 0, 0);
    }
#undef MJ_HAS
#undef MJ_B
#undef MJ_E
    L.kind = MJ_EVENT; L.ty = ty; L.word = w;
    return L;
}

// The `deltas` of a line mjai_parse_line accepted as a hora or ryukyoku -> d[0..4) (zeros when absent or null); true when the
// field is present and not null. The line is known to be well formed, so the walk only looks for the key (given once, unescaped).
MJX_DN bool mjai_line_deltas(const u8* p, long long b, long long e, i32* d) {
    for (int k = 0; k < 4; k++) d[k] = 0;
    MjCur c{p, b, e};
    mj_ws(c);
    if (mj_peek(c) != '{') return false;
    c.i++;
    mj_ws(c);
    while (mj_peek(c) == '"') {
        long long kb, ke, v[4];
        bool esc;
        if (!mj_key(c, &kb, &ke, &esc)) return false;
        const long long v0 = c.i;
        if (!mj_skip(c)) return false;
        if (!esc && mj_eq(p, kb, ke, "deltas")) {
            if (mj_is_null(p, v0, c.i) || !mj_ints(p, v0, c.i, 4, -2147483648LL, 2147483647LL, v)) return false;
            for (int k = 0; k < 4; k++) d[k] = (i32)v[k];
            return true;
        }
        mj_ws(c);
        if (mj_peek(c) != ',') return false;
        c.i++;
        mj_ws(c);
    }
    return false;
}

}  // namespace mjx
