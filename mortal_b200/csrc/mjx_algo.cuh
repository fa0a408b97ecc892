// mortal_b200 — device-side shanten / agari / point (sm_90a).
// Behavioural contract: libriichi algo/shanten.rs:88-150, algo/agari.rs:203-285 & 287-761 & 767-912,
// algo/point.rs:13-112. Implementation is this repo's own: packed 40-bit table rows gathered from
// L2, a fully unrolled min-plus merge in registers, incremental chiitoi/kokushi signatures so that a
// warp can evaluate "hand +/- one tile" for 32 tiles at once, and an open-addressing agari table.
#pragma once
#include "mjx_types.cuh"

namespace mjx {

// ---------------------------------------------------------------- shanten
struct Row10 { int v[10]; };

MJX_D Row10 unpack_row(u64 r) {
    Row10 o;
#pragma unroll
    for (int i = 0; i < 10; i++) o.v[i] = (int)((r >> (4 * i)) & 0xF);
    return o;
}

// shanten.rs:51-69 computed for m = 4 unconditionally: entries <= 5+len_div3 do not depend on the
// higher ones (descending in-place order), so the caller just reads index 5+len_div3.
MJX_D void add_suhai_full(Row10& lhs, const Row10& tab) {
#pragma unroll
    for (int j = 9; j >= 5; j--) {
        int sht = min(lhs.v[j] + tab.v[0], lhs.v[0] + tab.v[j]);
#pragma unroll
        for (int k = 5; k < j; k++) sht = min(sht, min(lhs.v[k] + tab.v[j - k], lhs.v[j - k] + tab.v[k]));
        lhs.v[j] = sht;
    }
#pragma unroll
    for (int j = 4; j >= 0; j--) {
        int sht = lhs.v[j] + tab.v[0];
#pragma unroll
        for (int k = 0; k < j; k++) sht = min(sht, lhs.v[k] + tab.v[j - k]);
        lhs.v[j] = sht;
    }
}

// shanten.rs:71-80 for every j in 5..=9 (each only reads lower, still-old entries)
MJX_D void add_jihai_full(Row10& lhs, const Row10& tab) {
#pragma unroll
    for (int j = 9; j >= 5; j--) {
        int sht = min(lhs.v[j] + tab.v[0], lhs.v[0] + tab.v[j]);
#pragma unroll
        for (int k = 5; k < j; k++) sht = min(sht, min(lhs.v[k] + tab.v[j - k], lhs.v[j - k] + tab.v[k]));
        lhs.v[j] = sht;
    }
}

// base-5 suit indices + chiitoi / kokushi signatures of a 34-count hand
struct HandSig {
    u32 idx[4];      // m, p, s, z base-5 indices (shanten.rs:82-84)
    int kinds, pairs;    // chiitoi (shanten.rs:103-115)
    int kkinds, kpairs;  // kokushi (shanten.rs:118-135)
};

MJX_D HandSig hand_sig(const u8* tehai) {
    HandSig s;
    s.kinds = s.pairs = s.kkinds = s.kpairs = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        u32 acc = 0;
        const int n = k < 3 ? 9 : 7;
#pragma unroll
        for (int i = 0; i < n; i++) {
            int c = tehai[k * 9 + i];
            acc = acc * 5 + c;
            s.kinds += c > 0;
            s.pairs += c >= 2;
            if (k == 3 || i == 0 || i == 8) {
                s.kkinds += c > 0;
                s.kpairs += c >= 2;
            }
        }
        s.idx[k] = acc;
    }
    return s;
}

MJX_CONST u32 c_pow5[9] = {390625, 78125, 15625, 3125, 625, 125, 25, 5, 1};  // 5^(8-i)

// signature of hand with tile t added (delta=+1) or removed (delta=-1); c = current count of t
MJX_D HandSig sig_variant(const HandSig& b, int t, int delta, int c) {
    HandSig s = b;
    int k = t / 9, i = t - k * 9;
    u32 w = k < 3 ? c_pow5[i] : c_pow5[i + 2];
    if (delta > 0) {
        s.idx[k] += w;
        s.kinds += c == 0;
        s.pairs += c == 1;
        if (is_yaokyuu(t)) { s.kkinds += c == 0; s.kpairs += c == 1; }
    } else {
        s.idx[k] -= w;
        s.kinds -= c == 1;
        s.pairs -= c == 2;
        if (is_yaokyuu(t)) { s.kkinds -= c == 1; s.kpairs -= c == 2; }
    }
    return s;
}

MJX_D u64 ld_row(const u64* tab, u32 idx, u32 rows) {
    // shanten.rs:52,72,91-94: out-of-range index reads as an all-zero row
    return idx < rows ? MJX_LDG(tab + idx) : 0ull;
}

// shanten.rs:88-100
MJX_D int shanten_normal_sig(const Tables& T, const HandSig& s, int len_div3) {
    Row10 ret = unpack_row(ld_row(T.suhai, s.idx[0], SUHAI_ROWS));
    u64 rp = ld_row(T.suhai, s.idx[1], SUHAI_ROWS);
    u64 rs = ld_row(T.suhai, s.idx[2], SUHAI_ROWS);
    u64 rz = ld_row(T.jihai, s.idx[3], JIHAI_ROWS);
    add_suhai_full(ret, unpack_row(rp));
    add_suhai_full(ret, unpack_row(rs));
    add_jihai_full(ret, unpack_row(rz));
    int r = ret.v[5];
    r = len_div3 == 1 ? ret.v[6] : r;
    r = len_div3 == 2 ? ret.v[7] : r;
    r = len_div3 == 3 ? ret.v[8] : r;
    r = len_div3 == 4 ? ret.v[9] : r;
    return r - 1;
}

// shanten.rs:138-150
MJX_D int shanten_all_sig(const Tables& T, const HandSig& s, int len_div3) {
    int sh = shanten_normal_sig(T, s, len_div3);
    if (sh <= 0 || len_div3 < 4) return sh;
    int chitoi = 7 - s.pairs + max(7 - s.kinds, 0) - 1;
    sh = min(sh, chitoi);
    if (sh > 0) {
        int kokushi = 14 - s.kkinds - (s.kpairs > 0 ? 1 : 0) - 1;
        sh = min(sh, kokushi);
    }
    return sh;
}

// The same for a hand of which only suit `sx` differs from a base hand: `others` = the min-plus merge of the other three
// suits' rows (10 entries; shanten.rs:51-80 is an exact min-plus convolution, so association order does not matter).
// One gather + the single entry 5 + len_div3 of the last merge: min over a + b = len of others[5+a] + row[b], others[a] + row[5+b].
MJX_D int shanten_all_others(const Tables& T, const HandSig& s, int sx, const u8* others, int len_div3) {
    const u64 r = sx < 3 ? ld_row(T.suhai, s.idx[sx], SUHAI_ROWS) : ld_row(T.jihai, s.idx[sx], JIHAI_ROWS);
    int v = 1 << 20;
#pragma unroll
    for (int a = 0; a <= 4; a++) {
        if (a <= len_div3) {
            const int b = len_div3 - a;
            v = min(v, (int)others[5 + a] + (int)((r >> (4 * b)) & 0xF));
            v = min(v, (int)others[a] + (int)((r >> (4 * (5 + b))) & 0xF));
        }
    }
    int sh = v - 1;
    if (sh <= 0 || len_div3 < 4) return sh;
    int chitoi = 7 - s.pairs + max(7 - s.kinds, 0) - 1;
    sh = min(sh, chitoi);
    if (sh > 0) {
        int kokushi = 14 - s.kkinds - (s.kpairs > 0 ? 1 : 0) - 1;
        sh = min(sh, kokushi);
    }
    return sh;
}

MJX_D int shanten_all(const Tables& T, const u8* tehai, int len_div3) {
    return shanten_all_sig(T, hand_sig(tehai), len_div3);
}
MJX_D int shanten_kokushi(const u8* tehai) {
    HandSig s = hand_sig(tehai);
    return 14 - s.kkinds - (s.kpairs > 0 ? 1 : 0) - 1;
}

// ---------------------------------------------------------------- point.rs
struct Point { i32 ron, tsumo_ko, tsumo_oya; };
MJX_D i32 tsumo_total(const Point& p, bool is_oya) {
    return is_oya ? p.tsumo_ko * 3 : p.tsumo_ko * 2 + p.tsumo_oya;
}
// point.rs:13-84 in closed form (point.rs:120-154 proves equivalence); *ok=false where the
// reference's match panics ("impossible combination").
MJX_D Point point_calc(bool is_oya, int fu, int han, bool* ok) {
    int base;
    bool good = true;
    if (han >= 13) base = 8000;
    else if (han >= 11) base = 6000;
    else if (han >= 8) base = 4000;
    else if (han >= 6) base = 3000;
    else if (han == 5) base = 2000;
    else if (han == 0) { base = 0; good = false; }
    else if ((han == 4 && fu >= 40) || (han == 3 && fu >= 70)) base = 2000;
    else {
        bool listed;
        if (fu == 20 || fu == 25) listed = han >= 2;            // han <= 4 here
        else if (fu == 30) listed = true;                        // 1..4
        else if (fu == 40 || fu == 50 || fu == 60) listed = han <= 3;
        else if (fu >= 70 && fu <= 110 && fu % 10 == 0) listed = han <= 2;
        else listed = false;
        good = listed;
        base = min(fu << (2 + han), 2000);
    }
    if (ok) *ok = good;
    Point p;
    if (is_oya) {
        p.ron = (base * 6 + 99) / 100 * 100;
        p.tsumo_ko = (base * 2 + 99) / 100 * 100;
        p.tsumo_oya = 0;
    } else {
        p.ron = (base * 4 + 99) / 100 * 100;
        p.tsumo_ko = (base + 99) / 100 * 100;
        p.tsumo_oya = (base * 2 + 99) / 100 * 100;
    }
    return p;
}
MJX_D Point point_yakuman(bool is_oya, int n) {
    Point p;
    if (is_oya) { p.ron = 48000 * n; p.tsumo_ko = 16000 * n; p.tsumo_oya = 0; }
    else { p.ron = 32000 * n; p.tsumo_ko = 8000 * n; p.tsumo_oya = 16000 * n; }
    return p;
}

// ---------------------------------------------------------------- agari
// agari.rs:66-74: kind 0 = None, 1 = Normal{fu,han}, 2 = Yakuman(n)
struct Agari { u8 kind, fu, han, yakuman; };

MJX_D bool agari_better_eq(const Agari& a, const Agari& b) {  // a >= b (agari.rs:175-190)
    if (a.kind == 2 && b.kind == 2) return a.yakuman >= b.yakuman;
    if (a.kind == 2) return true;
    if (b.kind == 2) return false;
    if (a.han != b.han) return a.han > b.han;
    return a.fu >= b.fu;
}
MJX_D Point agari_point(const Agari& a, bool is_oya, bool* ok) {
    if (a.kind == 2) { if (ok) *ok = true; return point_yakuman(is_oya, a.yakuman); }
    return point_calc(is_oya, a.fu, a.han, ok);
}

struct AgariQuery {
    const u8* tehai;  // [34] incl. winning tile
    const u8 *chis, *pons, *minkans, *ankans;
    int n_chis, n_pons, n_minkans, n_ankans;
    int bakaze, jikaze, winning_tile;
    bool is_ron, is_menzen;
};

// agari.rs:767-838: run-length key + the ascending list of distinct tiles
MJX_D u32 tile14_and_key(const u8* tiles, u8* tile14) {
    int n14 = 0, bit = -1;
    u32 key = 0;
    bool prev = false;
    for (int kind = 0; kind < 3; kind++) {
        for (int num = 0; num < 9; num++) {
            int c = tiles[kind * 9 + num];
            if (c > 0) {
                prev = true;
                tile14[n14++] = (u8)(kind * 9 + num);
                bit += 1;
                if (c == 2) { key |= 0x3u << bit; bit += 2; }
                else if (c == 3) { key |= 0xFu << bit; bit += 4; }
                else if (c == 4) { key |= 0x3Fu << bit; bit += 6; }
            } else if (prev) {
                prev = false;
                key |= 1u << bit;
                bit += 1;
            }
        }
        if (prev) {
            prev = false;
            key |= 1u << bit;
            bit += 1;
        }
    }
    for (int t = 27; t < 34; t++) {
        int c = tiles[t];
        if (c == 0) continue;
        tile14[n14++] = (u8)t;
        bit += 1;
        if (c == 2) { key |= 0x3u << bit; bit += 2; }
        else if (c == 3) { key |= 0xFu << bit; bit += 4; }
        else if (c == 4) { key |= 0x3Fu << bit; bit += 6; }
        key |= 1u << bit;
        bit += 1;
    }
    for (int i = n14; i < 14; i++) tile14[i] = 0;
    return key;
}

MJX_HD u32 agari_hash(u32 key) { return (key * 2654435761u) >> 17; }  // 15 bits

// returns number of divs (>= 0... a key may map to 0 divs never; -1 = absent)
MJX_D int agari_lookup(const Tables& T, u32 key, u32* divs) {
    u32 h = agari_hash(key);
    for (u32 probe = 0; probe < AGARI_SLOTS; probe++) {
        u32 slot = (h + probe) & (AGARI_SLOTS - 1);
        u32 k = MJX_LDG(T.agari_keys + slot);
        if (k == key) {
            U4 d = MJX_LDG(T.agari_divs + slot);
            divs[0] = d.x; divs[1] = d.y; divs[2] = d.z; divs[3] = d.w;
            return MJX_LDG(T.agari_ndivs + slot);
        }
        if (k == 0xFFFFFFFFu) return -1;
    }
    return -1;
}

// one decomposition of the closed hand (agari.rs:53-64, 126-157, 287-312)
struct DivCtx {
    u8 pair_tile;
    u8 mk[4], ms[4];  // menzen kotsu / shuntsu (first tile)
    int n_mk, n_ms;
    bool chitoi, chuuren, ittsuu, ryanpeikou, ipeikou;
    bool wtmm;  // winning_tile_makes_minkou
};

MJX_D DivCtx make_div(const AgariQuery& q, const u8* tile14, u32 v) {
    DivCtx d;
    d.pair_tile = tile14[(v >> 6) & 0xF];
    d.n_mk = v & 7;
    d.n_ms = (v >> 3) & 7;
    for (int i = 0; i < 4; i++) { d.mk[i] = 0; d.ms[i] = 0; }
    for (int i = 0; i < d.n_mk; i++) d.mk[i] = tile14[(v >> (10 + i * 4)) & 0xF];
    for (int i = 0; i < d.n_ms; i++) d.ms[i] = tile14[(v >> (10 + (d.n_mk + i) * 4)) & 0xF];
    d.chitoi = (v >> 26) & 1; d.chuuren = (v >> 27) & 1; d.ittsuu = (v >> 28) & 1;
    d.ryanpeikou = (v >> 29) & 1; d.ipeikou = (v >> 30) & 1;
    // agari.rs:315-338
    bool w = false;
    if (q.is_ron) {
        bool in_mk = false;
        for (int i = 0; i < d.n_mk; i++) in_mk |= d.mk[i] == q.winning_tile;
        if (in_mk) {
            if (q.winning_tile >= 27) w = true;
            else {
                int kind = q.winning_tile / 9, num = q.winning_tile % 9;
                int low = kind * 9 + max(num - 2, 0), high = kind * 9 + min(num, 6);
                bool covered = false;
                for (int i = 0; i < d.n_ms; i++) covered |= d.ms[i] >= low && d.ms[i] <= high;
                w = !covered;
            }
        }
    }
    d.wtmm = w;
    return d;
}

// agari.rs:362-450
MJX_D int div_fu(const AgariQuery& q, const DivCtx& d, bool has_pinfu) {
    if (d.chitoi) return 25;
    int fu = 20;
    for (int i = 0; i < d.n_mk; i++) {
        int t = d.mk[i];
        bool minkou = d.wtmm && t == q.winning_tile;
        bool yao = is_yaokyuu(t);
        fu += (!minkou && yao) ? 8 : ((minkou && !yao) ? 2 : 4);
    }
    for (int i = 0; i < q.n_pons; i++) fu += is_yaokyuu(q.pons[i]) ? 4 : 2;
    for (int i = 0; i < q.n_ankans; i++) fu += is_yaokyuu(q.ankans[i]) ? 32 : 16;
    for (int i = 0; i < q.n_minkans; i++) fu += is_yaokyuu(q.minkans[i]) ? 16 : 8;
    int pt = d.pair_tile;
    if (pt >= T_P && pt <= T_C) fu += 2;
    else {
        if (pt == q.bakaze) fu += 2;
        if (pt == q.jikaze) fu += 2;
    }
    if (fu == 20) {
        if (!q.is_menzen) return 30;
        if (has_pinfu) return q.is_ron ? 30 : 20;
        return q.is_ron ? 40 : 30;
    }
    if (!q.is_ron) fu += 2;
    else if (q.is_menzen) fu += 10;
    if (!d.wtmm) {
        if (pt == q.winning_tile) fu += 2;
        else {
            bool kp = false;
            for (int i = 0; i < d.n_ms; i++) {
                int s = d.ms[i];
                kp |= (s + 1 == q.winning_tile) || (s % 9 == 0 && s + 2 == q.winning_tile) ||
                      (s % 9 == 6 && s == q.winning_tile);
            }
            if (kp) fu += 2;
        }
    }
    return ((fu - 1) / 10 + 1) * 10;
}

// agari.rs:452-761. When `any_only` the exact han is irrelevant (has_yaku): the caller only tests kind != 0.
MJX_DN Agari div_yakus(const AgariQuery& q, const u8* tile14, const DivCtx& d, bool any_only) {
    int han = 0, yakuman = 0;
    const int pt = d.pair_tile;
    const bool pair_sangen = pt >= T_P && pt <= T_C;

    bool has_pinfu = d.n_ms == 4 && !pair_sangen && pt != q.bakaze && pt != q.jikaze;
    if (has_pinfu) {
        bool any = false;
        for (int i = 0; i < d.n_ms; i++) {
            int s = d.ms[i], num = s % 9 + 1;
            any |= (num <= 6 && s == q.winning_tile) || (num >= 2 && s + 2 == q.winning_tile);
        }
        has_pinfu = any;
    }
    if (has_pinfu) han += 1;
    if (d.chitoi) han += 2;
    if (d.ryanpeikou) han += 3;
    if (d.chuuren) yakuman += 1;

    // gather kotsu/kantsu and shuntsu lists (agari.rs:345-361)
    u8 kk[16]; int n_kk = 0;
    for (int i = 0; i < d.n_mk; i++) kk[n_kk++] = d.mk[i];
    for (int i = 0; i < q.n_pons; i++) kk[n_kk++] = q.pons[i];
    for (int i = 0; i < q.n_minkans; i++) kk[n_kk++] = q.minkans[i];
    for (int i = 0; i < q.n_ankans; i++) kk[n_kk++] = q.ankans[i];
    u8 ss[8]; int n_ss = 0;
    for (int i = 0; i < d.n_ms; i++) ss[n_ss++] = d.ms[i];
    for (int i = 0; i < q.n_chis; i++) ss[n_ss++] = q.chis[i];

    // bit sets over tile ids make most yaku tests a couple of mask compares
    u64 kset = 0, sset = 0, pairs7 = 0;
    for (int i = 0; i < n_kk; i++) kset |= 1ull << kk[i];
    for (int i = 0; i < n_ss; i++) sset |= 1ull << ss[i];
    if (d.chitoi) for (int i = 0; i < 7; i++) pairs7 |= 1ull << tile14[i];
    const u64 TANYAO_TILES = 0x7FFFFFFull & ~YAOKYUU_MASK;              // 2..8 of each suit
    const u64 SHUNTSU_TANYAO = 0x3Eull | (0x3Eull << 9) | (0x3Eull << 18);  // shuntsu starting at 2..6
    const u64 body = d.chitoi ? pairs7 : (kset | (1ull << pt));

    bool has_tanyao = d.chitoi ? (pairs7 & ~TANYAO_TILES) == 0
                               : ((sset & ~SHUNTSU_TANYAO) == 0 && (body & ~TANYAO_TILES) == 0);
    if (has_tanyao) han += 1;

    bool has_toitoi = !d.chitoi && d.n_ms == 0 && q.n_chis == 0;
    if (has_toitoi) han += 2;

    // honitsu / chinitsu / tsuuiisou (agari.rs:534-572): every block in at most one suit
    {
        u64 all = d.chitoi ? pairs7 : (kset | sset | (1ull << pt));
        int suits = ((all & 0x1FFull) != 0) + ((all & (0x1FFull << 9)) != 0) + ((all & (0x1FFull << 18)) != 0);
        bool has_j = (all >> 27) != 0;
        if (suits == 0) yakuman += 1;
        else if (suits == 1) han += (has_j ? 2 : 5) + (q.is_menzen ? 1 : 0);
    }

    if (!d.chitoi) {
        // ipeikou (agari.rs:574-597)
        if (d.ipeikou) han += 1;
        else if (q.n_ankans > 0 && q.is_menzen && d.n_ms >= 2) {
            u64 seen = 0; bool ip = false;
            for (int i = 0; i < d.n_ms; i++) {
                u64 b = 1ull << d.ms[i];
                ip |= (seen & b) != 0;
                seen |= b;
            }
            if (ip) han += 1;
        }
        // ittsuu (agari.rs:599-620)
        if (q.is_menzen && d.ittsuu) han += 2;
        else if (q.n_chis == 0 && d.ittsuu) han += 1;
        else if (d.n_ms + q.n_chis >= 3) {
            const u64 P = (1ull << 0) | (1ull << 3) | (1ull << 6);
            if ((sset & P) == P || (sset & (P << 9)) == (P << 9) || (sset & (P << 18)) == (P << 18)) han += 1;
        }
        // sanshoku (agari.rs:622-647)
        {
            u64 tri = sset & (sset >> 9) & (sset >> 18) & 0x1FFull;
            if (tri) han += q.is_menzen ? 2 : 1;
            else {
                u64 ktri = kset & (kset >> 9) & (kset >> 18) & 0x1FFull;
                if (ktri) han += 2;
            }
        }
        int ankous = q.n_ankans + d.n_mk - (d.wtmm ? 1 : 0);
        if (ankous == 4) yakuman += 1; else if (ankous == 3) han += 2;
        int kans = q.n_ankans + q.n_minkans;
        if (kans == 4) yakuman += 1; else if (kans == 3) han += 2;
        // ryuisou (agari.rs:669-677)
        {
            const u64 GREEN = (1ull << T_2S) | (1ull << T_3S) | (1ull << T_4S) | (1ull << T_6S) | (1ull << T_8S) | (1ull << T_F);
            if ((body & ~GREEN) == 0 && (sset & ~(1ull << T_2S)) == 0) yakuman += 1;
        }
        if (!has_tanyao) {
            u32 hj = (u32)(kset >> 27) & 0x7F;
            if ((hj >> (q.bakaze - 27)) & 1) han += 1;
            if ((hj >> (q.jikaze - 27)) & 1) han += 1;
            int saneins = mjx_popc(hj & 0x70);
            if (saneins > 0) {
                han += saneins;
                if (saneins == 3) yakuman += 1;
                else if (saneins == 2 && pair_sangen) han += 2;
            }
            int winds = mjx_popc(hj & 0x0F);
            if (winds == 4) yakuman += 1;
            else if (winds == 3 && pt >= T_E && pt <= T_N) yakuman += 1;
        }
    }

    if (!has_tanyao) {
        // chanta family (agari.rs:724-761)
        if ((body & ~YAOKYUU_MASK) == 0) {
            bool has_j = (body >> 27) != 0;
            if (d.chitoi || has_toitoi) {
                if (has_j) han += 2; else yakuman += 1;
            } else {
                const u64 EDGE = (1ull << 0) | (1ull << 6);
                const u64 EDGES = EDGE | (EDGE << 9) | (EDGE << 18);
                if ((sset & ~EDGES) == 0) han += (has_j ? 1 : 2) + (q.is_menzen ? 1 : 0);
            }
        }
    }

    Agari a;
    a.kind = 0; a.fu = 0; a.han = 0; a.yakuman = 0;
    if (yakuman > 0) { a.kind = 2; a.yakuman = (u8)yakuman; }
    else if (han > 0) {
        a.kind = 1; a.han = (u8)han;
        a.fu = (any_only || han >= 5) ? 0 : (u8)div_fu(q, d, has_pinfu);
    }
    return a;
}

// agari.rs:257-285
MJX_DN Agari search_yakus(const Tables& T, const AgariQuery& q, bool any_only) {
    Agari none; none.kind = 0; none.fu = none.han = none.yakuman = 0;
    if (q.is_menzen && shanten_kokushi(q.tehai) == -1) {
        Agari a; a.kind = 2; a.fu = a.han = 0; a.yakuman = 1;
        return a;
    }
    u8 tile14[14];
    u32 key = tile14_and_key(q.tehai, tile14);
    u32 divs[4];
    int n = agari_lookup(T, key, divs);
    if (n < 0) return none;
    Agari best = none;
    for (int i = 0; i < n; i++) {
        DivCtx d = make_div(q, tile14, divs[i]);
        Agari a = div_yakus(q, tile14, d, any_only);
        if (a.kind == 0) continue;
        if (any_only) return a;
        if (best.kind == 0 || agari_better_eq(a, best)) best = a;
    }
    return best;
}

MJX_D bool has_yaku(const Tables& T, const AgariQuery& q) { return search_yakus(T, q, true).kind != 0; }

// agari.rs:225-255
MJX_DN Agari agari_with(const Tables& T, const AgariQuery& q, int additional_hans, int doras) {
    Agari a = search_yakus(T, q, false);
    if (a.kind != 0) {
        if (a.kind == 1) a.han = (u8)(a.han + additional_hans + doras);
        return a;
    }
    Agari none; none.kind = 0; none.fu = none.han = none.yakuman = 0;
    if (additional_hans == 0) return none;
    if (additional_hans + doras >= 5) {
        Agari r; r.kind = 1; r.fu = 0; r.han = (u8)(additional_hans + doras); r.yakuman = 0;
        return r;
    }
    u8 tile14[14];
    u32 key = tile14_and_key(q.tehai, tile14);
    u32 divs[4];
    int n = agari_lookup(T, key, divs);
    if (n <= 0) return none;
    int fu = 0;
    for (int i = 0; i < n; i++) {
        DivCtx d = make_div(q, tile14, divs[i]);
        fu = max(fu, div_fu(q, d, false));
    }
    Agari r; r.kind = 1; r.fu = (u8)fu; r.han = (u8)(additional_hans + doras); r.yakuman = 0;
    return r;
}

}  // namespace mjx
