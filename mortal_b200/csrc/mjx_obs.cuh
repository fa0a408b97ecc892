// mortal_b200 — observation encoder: table record + seat -> (C, 34) f32 planes, obs versions 1-4.
//
// Contract: libriichi state/obs_repr.rs:126-630 (row map for version 4 in SURVEY.md §8 a17), IntegerEncoder
// obs_repr.rs:27-108, helpers obs_repr.rs:694-774, discard_candidates_with_unconditional_tenpai agent_helper.rs:100-197.
// The reference fills a heap array through a running row cursor, one PlayerState per seat. An observation
// is ~97% zeros and almost every non-zero is exactly 1, so here a warp first derives a COMPACT form of one
// observation from its staged copy of the table record (public part shared by the four perspectives,
// rotated on the fly):
//   * `bm[row]`  — one 34-bit column mask per row for the cells that are 1.0, and
//   * `sv[slot]` — 34 floats for each row that can hold other values (scores, counters, RBF / exp-decay planes,
//                  seen/4); which rows those are is a static property of the obs version (ObsLayout::sv_row),
// (k_encode_features, ~11 KB per observation for v4, L2-resident), and a second, purely streaming kernel
// (k_encode_store) materialises it slice by slice (OBS_SLICE_ROWS rows) in double-buffered shared-memory tiles
// that leave the SM as bulk asynchronous copies (TMA, cp.async.bulk shared->global). Warps are independent
// pipelines; there is no CTA-wide barrier anywhere.
#pragma once
#include "mjx_invisible.cuh"
#include "mjx_step.cuh"

namespace mjx {

constexpr int OBS_ROWS_V4 = 1012;
constexpr int SP_ROW0 = 889;  // first row of the single-player block of v4 (obs_repr.rs:561)
constexpr int OBS_COLS = 34;
// rows per slice: even, so that every slice starts on a 16-byte boundary (2 rows = 272 B) as bulk copies require
constexpr int OBS_SLICE_ROWS = 46;
static_assert(OBS_SLICE_ROWS % 2 == 0, "slice boundaries must be 16-byte aligned");
constexpr int OBS_MAX_SV = 80;            // value rows: 5 / 63 / 73 / 28 in versions 1..4
constexpr u64 OBS_FULL_ROW = (1ull << 34) - 1;
constexpr int ENC_N_PARTS = 4;
constexpr unsigned ENC_ALL_PARTS = 15;

// obs_repr.rs:27-108 IntegerEncoder: rows / value rows one encoded integer takes in each version
MJX_HD constexpr int ie_rows(int ver, int cap, bool one_hot, bool rescale, int rbf) {
    return ver == 1 ? cap : (one_hot ? cap + 1 : 0) + (rescale ? 1 : 0) + ((ver < 4 && rbf > 0) ? rbf - 1 : 0);
}
MJX_HD constexpr int ie_svs(int ver, bool rescale, int rbf) {
    return ver == 1 ? 0 : (rescale ? 1 : 0) + ((ver < 4 && rbf > 0) ? rbf - 1 : 0);
}

// Static row map of one obs version: first row of every feature group (the reference's running cursor, unrolled),
// the value-row slots, and the four independently derivable parts (row ranges) the feature kernel splits a row into:
// part 0 hand/scalars/dora/own pond, 1 opponents' ponds, 2 counters/overview/melds/status, 3 the action block.
struct ObsLayout {
    int ver, rows, bm_rows, n_sv;
    int hand, scores, score_stride, rank, kyoku, honba, kyotaku, hk_cap, winds, gk, dora, own_pond, own_decay, opp[3], opp_extra[3];
    int tiles_left, doras_owned, doras_owned_stride, doras_unseen, overview, fuuro, ankan, seen, last_tedashi, riichi_tile;
    int r_declared, r_accepted, waits, furiten, shanten, racc_self, kan_select, last_kawa, discard, riichi, chi, pon;
    int daiminkan, ankan_c, kakan_c, agari, ryukyoku, sp;
    int sv_scores, sv_honba, sv_kyotaku, sv_gk, sv_own_decay, sv_opp[3], sv_tiles_left, sv_doras_owned, sv_unseen, sv_seen;
    int part_row[ENC_N_PARTS + 1], part_sv[ENC_N_PARTS + 1];
    short sv_row[OBS_MAX_SV];
};

// rows [first_row, first_row + n) become value rows, in slot order
MJX_HD constexpr void layout_mark(ObsLayout& L, int& ns, int first_row, int n) {
    for (int i = 0; i < n; i++) L.sv_row[ns++] = (short)(first_row + i);
}

MJX_HD constexpr ObsLayout make_layout(int ver) {
    ObsLayout L{};
    L.ver = ver;
    int idx = 0, ns = 0;
    L.hand = idx; idx += 7;
    L.scores = idx; L.sv_scores = ns;
    L.score_stride = 1 + ((ver == 2 || ver == 3) ? ie_rows(ver, 500, false, false, 10) : (ver == 4 ? 1 : 0));
    for (int i = 0; i < 4; i++) { layout_mark(L, ns, idx, L.score_stride); idx += L.score_stride; }
    L.rank = idx; idx += 4;
    L.kyoku = idx; idx += 4;
    L.hk_cap = (ver == 1 || ver == 4) ? 10 : 6;
    L.honba = idx; L.sv_honba = ns; layout_mark(L, ns, idx, ie_svs(ver, ver == 4, 3)); idx += ie_rows(ver, L.hk_cap, false, ver == 4, 3);
    L.kyotaku = idx; L.sv_kyotaku = ns; layout_mark(L, ns, idx, ie_svs(ver, ver == 4, 3)); idx += ie_rows(ver, L.hk_cap, false, ver == 4, 3);
    L.winds = idx; idx += 2;
    L.gk = idx; L.sv_gk = ns;
    if (ver >= 2) { layout_mark(L, ns, idx, 1); idx += 1; }
    L.dora = idx; idx += 7;
    L.own_pond = idx; idx += 24 * 4;
    L.own_decay = idx; L.sv_own_decay = ns;
    if (ver >= 3) { layout_mark(L, ns, idx, 1); idx += 1; }
    L.part_row[1] = idx; L.part_sv[1] = ns;
    for (int p = 0; p < 3; p++) {
        L.opp[p] = idx; idx += 24 * 8;
        L.opp_extra[p] = idx; L.sv_opp[p] = ns;
        if (ver == 2) idx += 6;
        if (ver >= 3) { layout_mark(L, ns, idx, 3); idx += 3; }
    }
    L.part_row[2] = idx; L.part_sv[2] = ns;
    L.tiles_left = idx; L.sv_tiles_left = ns; layout_mark(L, ns, idx, 1); idx += 1;
    L.doras_owned = idx; L.sv_doras_owned = ns; L.doras_owned_stride = ie_rows(ver, 12, false, true, 3);
    for (int i = 0; i < 4; i++) { layout_mark(L, ns, idx, ie_svs(ver, true, 3)); idx += L.doras_owned_stride; }
    L.doras_unseen = idx; L.sv_unseen = ns; layout_mark(L, ns, idx, ie_svs(ver, true, 4)); idx += ie_rows(ver, 23, false, true, 4);
    L.overview = idx; idx += 4 * 7;
    L.fuuro = idx; idx += 4 * 4 * 5;
    L.ankan = idx; idx += 4;
    L.seen = idx; L.sv_seen = ns;
    L.last_tedashi = idx; L.riichi_tile = idx;
    if (ver >= 2) { layout_mark(L, ns, idx, 1); idx += 1; L.last_tedashi = idx; idx += 9; L.riichi_tile = idx; idx += 9; }
    L.r_declared = idx; idx += 3;
    L.r_accepted = idx; idx += 3;
    L.waits = idx; idx += 1;
    L.furiten = idx; idx += 1;
    L.shanten = idx; idx += ie_rows(ver, 6, true, false, 0);
    L.racc_self = idx; idx += 1;
    L.kan_select = idx; idx += 1;
    L.last_kawa = idx; idx += 3;
    L.part_row[3] = idx; L.part_sv[3] = ns;
    L.discard = idx; idx += 5;
    L.riichi = idx; idx += 1;
    L.chi = idx; idx += 3;
    L.pon = idx; idx += 1;
    L.daiminkan = idx; idx += 1;
    L.ankan_c = idx; idx += 1;
    L.kakan_c = idx; idx += 1;
    L.agari = idx; idx += 1;
    L.ryukyoku = idx; idx += 1;
    L.sp = idx;
    L.bm_rows = (idx + 3) & ~3;  // mask rows kept per observation: everything below the single-player block
    if (ver == 4) idx += 2 + 2 * 34 + 2 + 3 * 17;
    L.rows = idx;
    if (L.bm_rows > L.rows) L.bm_rows = L.rows;
    L.n_sv = ns;
    L.part_row[0] = 0; L.part_sv[0] = 0;
    L.part_row[4] = L.bm_rows; L.part_sv[4] = ns;
    return L;
}
static_assert(make_layout(1).rows == 938 && make_layout(2).rows == 942 && make_layout(3).rows == 934 &&
              make_layout(4).rows == OBS_ROWS_V4 && make_layout(4).sp == SP_ROW0, "consts.rs:20-28 obs_shape");
static_assert(make_layout(3).n_sv <= OBS_MAX_SV && make_layout(2).n_sv <= OBS_MAX_SV, "value-row table size");
// bytes of one compact observation: mask rows + value rows
MJX_HD constexpr int enc_compact_bytes(int ver) { return make_layout(ver).bm_rows * 8 + make_layout(ver).n_sv * OBS_COLS * 4; }

// The training-buffer record of one observation (k_obs_pack / k_obs_unpack, include/mjx.h mjx_obs_pack_dev): a 64-bit column
// mask for EVERY row (zero for a value row), then the value rows verbatim, 34 floats each, in ascending row order. The value rows
// are the encoder's sv_row plus, for version 4, the single-player block's non-0/1 rows (obs_repr.rs:563-690: 889-890, the two
// rows of encode_ev, and 961-1011, encode_sp_table), so v4 has 28 + 53 = 81 of them, more than the encoder's own OBS_MAX_SV;
// an invisible observation has oracle_obs_value_rows. Every other row holds only +0.0 and 1.0.
constexpr int OBS_REC_MAX_VAL = 96;
constexpr int OBS_REC_SP_EV = 2, OBS_REC_SP_TABLE0 = SP_ROW0 + 72;  // 889-890; 961-1011
struct ObsRecord {
    int rows, n_val, bytes;
    short val_row[OBS_REC_MAX_VAL];
};
MJX_HD constexpr ObsRecord make_obs_record(int ver, bool invisible) {
    ObsRecord R{};
    int nv = 0;
    if (invisible) {
        R.rows = oracle_obs_rows(ver);
        for (int k = 0; k < oracle_obs_value_rows(ver); k++) R.val_row[nv++] = (short)oracle_obs_value_row(k);
    } else {
        const ObsLayout L = make_layout(ver);
        R.rows = L.rows;
        for (int k = 0; k < L.n_sv; k++) R.val_row[nv++] = L.sv_row[k];
        if (ver == 4) {
            for (int r = SP_ROW0; r < SP_ROW0 + OBS_REC_SP_EV; r++) R.val_row[nv++] = (short)r;
            for (int r = OBS_REC_SP_TABLE0; r < OBS_ROWS_V4; r++) R.val_row[nv++] = (short)r;
        }
    }
    R.n_val = nv;
    R.bytes = R.rows * 8 + nv * OBS_COLS * 4;
    return R;
}
static_assert(make_obs_record(1, false).bytes == 8184 && make_obs_record(2, false).bytes == 16104 &&
              make_obs_record(3, false).bytes == 17400 && make_obs_record(4, false).bytes == 19112 &&
              make_obs_record(4, true).bytes == 2144 && make_obs_record(1, true).bytes == 1688, "record sizes");
static_assert(make_obs_record(4, false).n_val == 81 && make_obs_record(4, false).n_val <= OBS_REC_MAX_VAL, "v4 value rows");

struct EncCtx {
    const TableState* S;
    Tables T;
    u64* bm;        // [bm_rows] column masks of the 1.0 cells, zero on entry
    float* sv;      // [n_sv][34] value rows, zero on entry
    int seat;       // perspective (absolute seat)
    bool kan_select;
    int lane;
    const u8* dora_factor;  // [34]
    unsigned parts;         // which feature groups to derive (bit k = part k), ENC_ALL_PARTS = everything
};

// Writers. ENC_OR / ENC_SVAL / ENC_SMAX may be called by any lane (different lanes, different or equal cells);
// the *_L0 forms are for values every lane holds identically: lane 0 (or the warp, column-wise) writes.
#ifdef MJX_HOST_EMUL
#define ENC_OR(e, row, mask) do { (e).bm[(row)] |= (u64)(mask); } while (0)
#define ENC_SVAL(e, slot, col, v) do { (e).sv[(slot) * 34 + (col)] = (v); } while (0)
// "latest writer wins" cells whose value grows with the writer's position: a max (the reference assigns in order)
#define ENC_SMAX(e, slot, col, v) do { float& x_ = (e).sv[(slot) * 34 + (col)]; x_ = max(x_, (v)); } while (0)
#define ENC_SFILL_L0(e, slot, v) do { for (int c_ = 0; c_ < 34; c_++) ENC_SVAL(e, slot, c_, v); } while (0)
#define ENC_OR_L0(e, row, mask) ENC_OR(e, row, mask)
// positions 0..n-1 of a list, one per lane on the device
#define ENC_FOR_POS(e, i, n) for (int i = 0; i < (n); i++)
#else
#define ENC_OR(e, row, mask) atomicOr(reinterpret_cast<unsigned long long*>(&(e).bm[(row)]), (unsigned long long)(mask))
#define ENC_SVAL(e, slot, col, v) do { (e).sv[(slot) * 34 + (col)] = (v); } while (0)
#define ENC_SMAX(e, slot, col, v) atomicMax(reinterpret_cast<int*>(&(e).sv[(slot) * 34 + (col)]), __float_as_int(v))
#define ENC_SFILL_L0(e, slot, v) do { ENC_SVAL(e, slot, (e).lane, v); if ((e).lane < 2) ENC_SVAL(e, slot, 32 + (e).lane, v); } while (0)
#define ENC_OR_L0(e, row, mask) do { if ((e).lane == 0) (e).bm[(row)] |= (u64)(mask); } while (0)
#define ENC_FOR_POS(e, i, n) for (int i0_ = 0, i = (e).lane; i0_ < (n); i0_ += 32, i += 32)
#endif
#define ENC_ONES_L0(e, row) ENC_OR_L0(e, row, OBS_FULL_ROW)
#define ENC_ONE_L0(e, row, col) ENC_OR_L0(e, row, 1ull << (col))

MJX_D int rel_to_abs(int seat, int rel) { return (seat + rel) & 3; }

// a seat's pond as the perspective `p` sees it: optional start-of-kyoku pad (update.rs:819-824) + items
struct KawaView {
    const KawaItem* items;
    int n_items;
    int pad;  // 0 or 1
    MJX_DM int len() const { return n_items + pad; }
    // returns nullptr for a None slot
    MJX_DM const KawaItem* at(int i) const {
        if (i < pad) return nullptr;
        const KawaItem* k = items + (i - pad);
        return k->tile == T_NONE ? nullptr : k;
    }
};

MJX_D KawaView kawa_view(const TableState* S, int p, int abs_seat) {
    KawaView v;
    v.items = S->pub[abs_seat].kawa;
    v.n_items = S->pub[abs_seat].kawa_len;
    int rel_s = (abs_seat - p) & 3, rel_oya = (S->oya - p) & 3;
    v.pad = rel_s < rel_oya ? 1 : 0;
    return v;
}

// obs_repr.rs:694-712 over an explicit tile list accessor (T_NONE entries are skipped): the k-th copy of a kind
// lights plane `row + k`; planes row+4.. mark the three red fives. Every lane runs the same scan (uniform values).
template <typename F>
MJX_D void enc_tile_set(EncCtx& e, int row, int n, F get) {
    u64 c1 = 0, c2 = 0, c3 = 0, c4 = 0;
    u32 akam = 0;
    for (int i = 0; i < n; i++) {
        const int tile = get(i);
        if (tile == T_NONE) continue;
        if (is_aka(tile)) akam |= 1u << (tile - T_5MR);
        const u64 bit = 1ull << deaka(tile);
        c4 |= c3 & bit; c3 |= c2 & bit; c2 |= c1 & bit; c1 |= bit;
    }
    if (c1) ENC_OR_L0(e, row, c1);
    if (c2) ENC_OR_L0(e, row + 1, c2);
    if (c3) ENC_OR_L0(e, row + 2, c3);
    if (c4) ENC_OR_L0(e, row + 3, c4);
    for (int k = 0; k < 3; k++) if ((akam >> k) & 1) ENC_ONES_L0(e, row + 4 + k);
}

// obs_repr.rs:27-108 IntegerEncoder::encode at (row, slot); every lane holds the same arguments
template <int VER>
MJX_D void enc_int(EncCtx& e, int row, int slot, int n_raw, int cap, bool one_hot, bool rescale, int rbf) {
    const int n = min(n_raw, cap);
    if (VER == 1) {
        for (int i = 0; i < n; i++) ENC_ONES_L0(e, row + i);  // thermometer
        return;
    }
    if (one_hot) { ENC_ONES_L0(e, row + n); row += cap + 1; }
    if (rescale) { ENC_SFILL_L0(e, slot, (float)n / (float)cap); slot += 1; }
    if (VER < 4 && rbf > 0) {
        const float interval = (float)cap / (float)rbf;
        for (int i = 1; i < rbf; i++) {
            const float d = (float)n_raw - (float)i * interval;
            ENC_SFILL_L0(e, slot + i - 1, expf(-(d * d) / (2.f * (interval * interval))));
        }
    }
}

// agent_helper.rs:100-197 as a 34-bit mask (aka folded back as discard_candidates_with_unconditional_tenpai does)
MJX_DN u64 unconditional_tenpai_discards(EncCtx& e, const Ctx& c) {
    const TableState* S = e.S;
    const int p = e.seat;
    const SeatPrivate& P = S->priv[p];
    const bool has_next = (P.flags & PF_HAS_NEXT_SHANTEN_DISCARD) != 0;
    if (S->tiles_left == 0 || P.shanten > 1 || (P.shanten == 1 && !has_next)) return 0;
    const bool racc = (S->riichi_accepted >> p) & 1;
    if (P.last_self_tsumo != T_NONE) {
        if ((P.waits >> deaka(P.last_self_tsumo)) & 1) return 0;
        if (racc) return (P.flags & PF_AT_FURITEN) ? 0 : (1ull << deaka(P.last_self_tsumo));
    } else if (shanten_all(e.T, P.tehai, P.tehai_len_div3) == -1) {
        return 0;
    }
    const u64 cand = (P.shanten == 1 ? P.next_shanten : P.keep_shanten) & ~P.forbidden;
    u64 result = 0;
    const int len = P.tehai_len_div3;
    const HandSig base = hand_sig(P.tehai);
    for (u64 rest = cand; rest; rest &= rest - 1) {
        const int discard = mjx_ffsll(rest) - 1;
        const HandSig b1 = sig_variant(base, discard, -1, P.tehai[discard]);
        // every tsumo tile evaluated by its own lane: code bit0 = completes the hand, bit1 = has yaku
        u64 wins, yaku;
        tile_eval2(c, true, [&](int t) {
            int n = P.tehai[t] - (t == discard ? 1 : 0);
            if (t == discard || n == 4) return 0;
            if (shanten_all_sig(e.T, sig_variant(b1, t, +1, n), len) > -1) return 0;
            int code = 1;
            if (!((P.discarded >> t) & 1) && (S->public_seen[t] + P.tehai[t]) < 4) {
                u8 th[34];
                for (int i = 0; i < 34; i++) th[i] = P.tehai[i];
                th[discard] -= 1;
                th[t] += 1;
                if (has_yaku(e.T, make_query(S, p, th, t, true))) code |= 2;
            }
            return code;
        }, wins, yaku);
        // reference loop order: ascending tsumo; a furiten winning tile voids the discard, otherwise
        // the discard qualifies as soon as one live winning tile has a yaku
        bool ok = false;
        if (!(wins & P.discarded)) ok = yaku != 0;
        else {
            // furiten tile found at position f: result is false regardless (ret[discard] = false; break)
            ok = false;
        }
        if (ok) result |= 1ull << discard;
    }
    return result;
}

// Derives the compact form (bm, sv) of one observation (for v4: rows 0..888; 889..1011, the single-player block,
// is k_sp_finalize's). Called by ONE warp; the windows of bm and sv that e.parts covers must be zero on entry.
template <int VER>
MJX_DN void encode_obs(EncCtx& e, const Ctx& c, u64* mask_out) {
    constexpr ObsLayout L = make_layout(VER);
    const TableState* S = e.S;
    const int p = e.seat;
    const SeatPrivate& P = S->priv[p];
    const u16 cans = P.cans;
    const u8* df = e.dora_factor;

    if (e.parts & 1) {
        // ---- hand
        u64 m1, m2, m3, m4;
        tile_eval2(c, true, [&](int t) { const int n = P.tehai[t]; return (n > 0 ? 1 : 0) | (n > 1 ? 2 : 0); }, m1, m2);
        tile_eval2(c, true, [&](int t) { const int n = P.tehai[t]; return (n > 2 ? 1 : 0) | (n > 3 ? 2 : 0); }, m3, m4);
        ENC_OR_L0(e, L.hand, m1); ENC_OR_L0(e, L.hand + 1, m2); ENC_OR_L0(e, L.hand + 2, m3); ENC_OR_L0(e, L.hand + 3, m4);
        for (int k = 0; k < 3; k++) if ((P.akas_in_hand >> k) & 1) ENC_ONES_L0(e, L.hand + 4 + k);
        // ---- scores, rank, round
        int rank = 0;
        for (int i = 0; i < 4; i++) {
            const i32 sc = S->scores[rel_to_abs(p, i)];
            const int slot = L.sv_scores + L.score_stride * i;
            ENC_SFILL_L0(e, slot, (float)min(max(sc, 0), 100000) / 100000.f);
            // v2/v3: `score as usize / 100` (obs_repr.rs:147) wraps for negative scores; kept as the reference has it
            if (VER == 2 || VER == 3) enc_int<VER>(e, L.scores + L.score_stride * i + 1, slot + 1, (int)((u32)sc / 100u), 500, false, false, 10);
            if (VER == 4) ENC_SFILL_L0(e, slot + 1, (float)min(max(sc, 0), 30000) / 30000.f);
        }
        for (int s = 0; s < 4; s++)  // rankings.rs:8-22: stable by seat
            if (s != p && (S->scores[s] > S->scores[p] || (S->scores[s] == S->scores[p] && s < p))) rank++;
        ENC_ONES_L0(e, L.rank + rank);
        const int kyoku_in_wind = S->kyoku & 3, bakaze = T_E + S->kyoku / 4;
        if (VER == 1) { for (int i = 0; i < kyoku_in_wind; i++) ENC_ONES_L0(e, L.kyoku + i); }
        else ENC_ONES_L0(e, L.kyoku + kyoku_in_wind);
        enc_int<VER>(e, L.honba, L.sv_honba, S->honba, L.hk_cap, false, VER == 4, 3);
        enc_int<VER>(e, L.kyotaku, L.sv_kyotaku, S->kyotaku, L.hk_cap, false, VER == 4, 3);
        ENC_ONE_L0(e, L.winds, bakaze);
        ENC_ONE_L0(e, L.winds + 1, T_E + ((p + 4 - S->oya) & 3));
        if (VER >= 2) enc_int<VER>(e, L.gk, L.sv_gk, min(bakaze - T_E, 1) * 4 + kyoku_in_wind, 7, false, true, 0);
        // ---- dora indicators
        enc_tile_set(e, L.dora, S->n_dora, [&](int i) { return dora_indicator(S, i); });
    }
    // max kawa length over the four ponds as this seat sees them (obs_repr.rs:221)
    int max_kawa_len = 0;
    for (int s = 0; s < 4; s++) max_kawa_len = max(max_kawa_len, kawa_view(S, p, s).len());

    // ---- own pond: lanes are pond positions
    if (e.parts & 1) {
        const KawaView kv = kawa_view(S, p, p);
        const int len = kv.len();
        ENC_FOR_POS(e, i, len) {
            const KawaItem* k = i < len ? kv.at(i) : nullptr;
            if (!k) continue;
            const int tile = k->tile, fl = k->flags;
            u64 kans = 0;
            for (int q = 0; q < 4; q++) if (k->kan[q] != T_NONE) kans |= 1ull << k->kan[q];
            for (int pass = 0; pass < 2; pass++) {
                const int j = pass == 0 ? i : len - 1 - i;
                if (j >= (pass == 0 ? 6 : 18)) continue;
                const int row = L.own_pond + (pass == 0 ? 0 : 24) + 4 * j;
                if (kans) ENC_OR(e, row, kans);
                ENC_OR(e, row + 1, 1ull << deaka(tile));
                if (is_aka(tile)) ENC_OR(e, row + 2, OBS_FULL_ROW);
                if (fl & SF_DORA) ENC_OR(e, row + 3, OBS_FULL_ROW);
            }
            if (VER >= 3) ENC_SMAX(e, L.sv_own_decay, deaka(tile), expf(-0.2f * (float)(max_kawa_len - 1 - i)));
        }
    }
    // ---- the three opponents' ponds
    if (e.parts & 2) for (int rel = 1; rel < 4; rel++) {
        const int sec = L.opp[rel - 1], extra = L.opp_extra[rel - 1], slot = L.sv_opp[rel - 1];
        const KawaView kv = kawa_view(S, p, rel_to_abs(p, rel));
        const int len = kv.len();
        ENC_FOR_POS(e, i, len) {
            const KawaItem* k = i < len ? kv.at(i) : nullptr;
            if (!k) continue;
            const int tile = k->tile, fl = k->flags;
            u64 kans = 0;
            for (int q = 0; q < 4; q++) if (k->kan[q] != T_NONE) kans |= 1ull << k->kan[q];
            for (int pass = 0; pass < 2; pass++) {
                const int j = pass == 0 ? i : len - 1 - i;
                if (j >= (pass == 0 ? 6 : 18)) continue;
                const int row = sec + (pass == 0 ? 0 : 48) + 8 * j;
                if (fl & SF_HAS_CHIPON) {
                    ENC_OR(e, row, 1ull << min(k->consumed[0], k->consumed[1]));
                    ENC_OR(e, row + 1, 1ull << max(k->consumed[0], k->consumed[1]));
                }
                if (kans) ENC_OR(e, row + 2, kans);
                ENC_OR(e, row + 3, 1ull << deaka(tile));
                if (is_aka(tile)) ENC_OR(e, row + 4, OBS_FULL_ROW);
                if (fl & SF_DORA) ENC_OR(e, row + 5, OBS_FULL_ROW);
                if (fl & SF_TEDASHI) ENC_OR(e, row + 6, OBS_FULL_ROW);
                if (fl & SF_RIICHI) ENC_OR(e, row + 7, OBS_FULL_ROW);
            }
            const int tid = deaka(tile);
            if (VER == 2) {
                // thirds of the pond by discard order, counting real discards only (obs_repr.rs v2 branch)
                int turn = 0;
                for (int q = 0; q < i; q++) turn += kv.at(q) != nullptr;
                const int third = min(turn / 6, 2);
                ENC_OR(e, extra + third, 1ull << tid);
                if (fl & SF_TEDASHI) ENC_OR(e, extra + 3 + third, 1ull << tid);
            }
            if (VER >= 3) {
                const float v = expf(-0.2f * (float)(max_kawa_len - 1 - i));
                ENC_SMAX(e, slot, tid, v);
                if (fl & SF_TEDASHI) ENC_SMAX(e, slot + 1, tid, v);
                if (fl & SF_RIICHI) ENC_SMAX(e, slot + 2, tid, v);
            }
        }
    }
    if (e.parts & 4) {
        // ---- counters
        ENC_SFILL_L0(e, L.sv_tiles_left, (float)S->tiles_left / 69.f);
        // sum_t seen[t] * dora_factor[t] == sum over indicators of seen[indicated tile]
        int seen_doras = mjx_popc((u32)(S->akas_public | P.akas_in_hand));
        int own_doras = mjx_popc((u32)P.akas_in_hand);
        for (int k = 0; k < S->n_dora; k++) {
            const int d = tile_next(dora_indicator(S, k));
            seen_doras += S->public_seen[d] + P.tehai[d];
            own_doras += P.tehai[d];
        }
        for (int i = 0; i < 4; i++) {
            const int s = rel_to_abs(p, i);
            const SeatPublic& U = S->pub[s];
            int n = i == 0 ? own_doras : 0;
            for (int f = 0; f < U.n_fuuro; f++)
                for (int j = 0; j < 4; j++) {
                    int t = U.fuuro[f][j];
                    if (t != T_NONE) n += df[deaka(t)] + (is_aka(t) ? 1 : 0);
                }
            for (int j = 0; j < U.n_ankan; j++) {
                int t = U.ankan[j];
                n += 4 * df[t] + ((t == T_5M || t == T_5P || t == T_5S) ? 1 : 0);
            }
            enc_int<VER>(e, L.doras_owned + L.doras_owned_stride * i, L.sv_doras_owned + ie_svs(VER, true, 3) * i, n, 12, false, true, 3);
        }
        const int unseen = (S->n_dora * 4 + 3 - seen_doras) & 0xFF;
        enc_int<VER>(e, L.doras_unseen, L.sv_unseen, unseen, 23, false, true, 4);
        // ---- pond overview: real discards only (update.rs:336); empty slots hold T_NONE
        for (int i = 0; i < 4; i++) {
            const SeatPublic& U = S->pub[rel_to_abs(p, i)];
            enc_tile_set(e, L.overview + 7 * i, U.kawa_len, [&](int j) { return (int)U.kawa[j].tile; });
        }
        // ---- melds
        for (int i = 0; i < 4; i++) {
            const SeatPublic& U = S->pub[rel_to_abs(p, i)];
            for (int f = 0; f < U.n_fuuro; f++) {
                const int row = L.fuuro + 20 * i + 5 * f;
                u64 c1 = 0, c2 = 0, c3 = 0, c4 = 0;  // k-th copy of a kind goes to the first still-zero plane (obs_repr.rs:305-308)
                bool aka = false;
                for (int j = 0; j < 4; j++) {
                    const int t = U.fuuro[f][j];
                    if (t == T_NONE) continue;
                    aka = aka || is_aka(t);
                    const u64 bit = 1ull << deaka(t);
                    c4 |= c3 & bit; c3 |= c2 & bit; c2 |= c1 & bit; c1 |= bit;
                }
                ENC_OR_L0(e, row, c1);
                if (c2) ENC_OR_L0(e, row + 1, c2);
                if (c3) ENC_OR_L0(e, row + 2, c3);
                if (c4) ENC_OR_L0(e, row + 3, c4);
                if (aka) ENC_ONES_L0(e, row + 4);
            }
            u64 ak = 0;
            for (int j = 0; j < U.n_ankan; j++) ak |= 1ull << U.ankan[j];
            if (ak) ENC_OR_L0(e, L.ankan + i, ak);
        }
        // ---- seen tiles, key discards (v2+), riichi / wait status
        if (VER >= 2) {
            MJX_FOR_TILES(e, t) { ENC_SVAL(e, L.sv_seen, t, (float)(S->public_seen[t] + P.tehai[t]) / 4.f); }
        }
        if (P.waits) ENC_OR_L0(e, L.waits, P.waits);
        for (int rel = 1; rel < 4; rel++) {
            const SeatPublic& U = S->pub[rel_to_abs(p, rel)];
            if (VER >= 2 && (U.last_tedashi_flags & SF_VALID)) {
                const int row = L.last_tedashi + 3 * (rel - 1);
                ENC_ONE_L0(e, row, deaka(U.last_tedashi_tile));
                if (is_aka(U.last_tedashi_tile)) ENC_ONES_L0(e, row + 1);
                if (U.last_tedashi_flags & SF_DORA) ENC_ONES_L0(e, row + 2);
            }
            if (VER >= 2 && (U.riichi_flags & SF_VALID)) {
                const int row = L.riichi_tile + 3 * (rel - 1);
                ENC_ONE_L0(e, row, deaka(U.riichi_tile));
                if (is_aka(U.riichi_tile)) ENC_ONES_L0(e, row + 1);
                if (U.riichi_flags & SF_DORA) ENC_ONES_L0(e, row + 2);
            }
            if ((S->riichi_declared >> rel_to_abs(p, rel)) & 1) ENC_ONES_L0(e, L.r_declared + rel - 1);
            if ((S->riichi_accepted >> rel_to_abs(p, rel)) & 1) ENC_ONES_L0(e, L.r_accepted + rel - 1);
        }
        if (P.flags & PF_AT_FURITEN) ENC_ONES_L0(e, L.furiten);
        enc_int<VER>(e, L.shanten, 0, max((int)P.shanten, 0), 6, true, false, 0);
        if ((S->riichi_accepted >> p) & 1) ENC_ONES_L0(e, L.racc_self);
        if (e.kan_select) ENC_ONES_L0(e, L.kan_select);
        if (cans & CAN_PASS) {
            const int tile = S->last_kawa_tile, tid = deaka(tile);
            ENC_ONE_L0(e, L.last_kawa, tid);
            if (is_aka(tile)) ENC_ONES_L0(e, L.last_kawa + 1);
            if (df[tid] > 0) ENC_ONES_L0(e, L.last_kawa + 2);
        }
    }
    // ---- the action block + legal mask
    if (e.parts & 8) {
        const u64 discards = (cans & CAN_DISCARD) ? discard_candidates(c, p) : 0;  // warp collective
        if (mask_out) *mask_out = legal_mask(c, p, e.kan_select, discards);
        if (cans & CAN_DISCARD) {
            u64 d34 = (discards & ((1ull << 34) - 1)) | (((discards >> 34) & 1) << 4) | (((discards >> 35) & 1) << 13) |
                      (((discards >> 36) & 1) << 22);
            u64 ut = 0;
            if (P.shanten <= 1) ut = unconditional_tenpai_discards(e, c);
            ENC_OR_L0(e, L.discard, d34);
            ENC_OR_L0(e, L.discard + 1, P.keep_shanten);
            ENC_OR_L0(e, L.discard + 2, P.next_shanten);
            ENC_OR_L0(e, L.discard + 3, ut);
            if ((S->riichi_declared >> p) & 1) ENC_ONES_L0(e, L.discard + 4);
        }
        if (cans & CAN_RIICHI) ENC_ONES_L0(e, L.riichi);
        if (cans & CAN_CHI_LOW) ENC_ONES_L0(e, L.chi);
        if (cans & CAN_CHI_MID) ENC_ONES_L0(e, L.chi + 1);
        if (cans & CAN_CHI_HIGH) ENC_ONES_L0(e, L.chi + 2);
        if (cans & CAN_PON) ENC_ONES_L0(e, L.pon);
        if (cans & CAN_DAIMINKAN) ENC_ONES_L0(e, L.daiminkan);
        if (cans & CAN_ANKAN) ENC_OR_L0(e, L.ankan_c, P.ankan_cand);
        if (cans & CAN_KAKAN) ENC_OR_L0(e, L.kakan_c, P.kakan_cand);
        if (cans & CAN_AGARI) ENC_ONES_L0(e, L.agari);
        if (cans & CAN_RYUKYOKU) ENC_ONES_L0(e, L.ryukyoku);
    }
}

// version selected at run time (the emulation harness and kernels dispatch through this)
MJX_DN void encode_obs_any(int ver, EncCtx& e, const Ctx& c, u64* mask_out) {
    switch (ver) {
        case 1: encode_obs<1>(e, c, mask_out); break;
        case 2: encode_obs<2>(e, c, mask_out); break;
        case 3: encode_obs<3>(e, c, mask_out); break;
        default: encode_obs<4>(e, c, mask_out); break;
    }
}

// Materialise obs rows [row_lo, row_hi) from the compact form into `tile` ((row_hi - row_lo) x 34 floats).
// Called by ONE warp after encode_obs (and a warp sync). On the device the caller passes the slice's row masks
// already in registers (lane l holds rows row_lo + l and row_lo + 32 + l), loaded ahead of time to hide their latency.
#ifdef MJX_HOST_EMUL
// bm: bm_rows column masks; sv: n_sv value rows of 34 floats, row sv_row[k] each (a training-buffer record has the same form)
MJX_DN void enc_materialize(const u64* bm, int bm_rows, const float* sv, const short* sv_row, int n_sv, float* tile, int row_lo,
                            int row_hi) {
    for (int r = row_lo; r < row_hi; r++) {
        const u64 m = r < bm_rows ? bm[r] : 0;
        int slot = -1;
        for (int k = 0; k < n_sv; k++) if (sv_row[k] == r) slot = k;
        for (int col = 0; col < 34; col++)
            tile[(r - row_lo) * 34 + col] = slot >= 0 ? sv[slot * 34 + col] : (((m >> col) & 1) ? 1.f : 0.f);
    }
}
MJX_DN void enc_materialize(const ObsLayout& L, const EncCtx& e, float* tile, int row_lo, int row_hi) {
    enc_materialize(e.bm, L.bm_rows, e.sv, L.sv_row, L.n_sv, tile, row_lo, row_hi);
}
#else
static_assert(OBS_SLICE_ROWS <= 64, "two mask words per lane cover a slice");
MJX_D void enc_load_masks(const u64* bm, int bm_rows, int row_lo, int lane, u64& m0, u64& m1) {
    const int r0 = row_lo + lane, r1 = row_lo + 32 + lane;
    m0 = r0 < bm_rows ? __ldg(bm + r0) : 0;
    m1 = (32 + lane < OBS_SLICE_ROWS && r1 < bm_rows) ? __ldg(bm + r1) : 0;
}
// sv_row: the version's value-row table (constant memory), n_sv entries in ascending row order
MJX_DN void enc_materialize(const float* sv, const short* sv_row, int n_sv, int lane, float* tile, int row_lo, int row_hi,
                            u64 m0, u64 m1) {
    {   // zero the slice: almost all of it stays zero
        uint4* t4 = reinterpret_cast<uint4*>(tile);
        const uint4 z = make_uint4(0, 0, 0, 0);
        const int n16 = (row_hi - row_lo) * 34 * 4 / 16;
        for (int i = lane; i < n16; i += 32) t4[i] = z;
    }
    __syncwarp();
#pragma unroll
    for (int half = 0; half < 2; half++) {
        const u64 m = half == 0 ? m0 : m1;
        unsigned nz = __ballot_sync(0xffffffffu, m != 0);
        while (nz) {  // one non-zero row at a time, lanes are columns
            const int src = __ffs(nz) - 1;
            nz &= nz - 1;
            const unsigned lo = __shfl_sync(0xffffffffu, (unsigned)m, src);
            const unsigned hi = __shfl_sync(0xffffffffu, (unsigned)(m >> 32), src);
            float* dst = tile + (half * 32 + src) * 34;
            if ((lo >> lane) & 1) dst[lane] = 1.f;
            if (lane < 2 && ((hi >> lane) & 1)) dst[32 + lane] = 1.f;
        }
    }
    // value rows inside this slice: lane s looks at slots s, s + 32, ...; the hits are copied by the whole warp
    for (int s0 = 0; s0 < n_sv; s0 += 32) {
        const int my_row = s0 + lane < n_sv ? (int)sv_row[s0 + lane] : -1;
        unsigned hit = __ballot_sync(0xffffffffu, my_row >= row_lo && my_row < row_hi);
        while (hit) {
            const int k = __ffs(hit) - 1;
            hit &= hit - 1;
            float* dst = tile + (__shfl_sync(0xffffffffu, my_row, k) - row_lo) * 34;
            const float* src = sv + (s0 + k) * 34;
            dst[lane] = __ldg(src + lane);
            if (lane < 2) dst[32 + lane] = __ldg(src + 32 + lane);
        }
    }
}
#endif

}  // namespace mjx
