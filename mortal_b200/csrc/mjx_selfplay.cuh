// mortal_b200 — arena event words (csrc/mjx_step.cuh `log_word`, inline payloads: 9 words after start_kyoku, 2 deltas words after
// hora and ryukyoku) -> the replay arrays (include/mjx_selfplay.h): one word per event with start_game / end_game around the game,
// 19-word kyoku payloads, hora side entries and per-event deltas, exactly what k_mjai_decode makes of the text
// mortal_b200/mjai_log.py writes for the game, so a self-play game reaches the replay kernels without its log being written.
//
// Device: one warp per game (k_arena_words in mjx_kernels.cu). Lane 0 walks the next 32 event starts, each lane checks and
// converts one event, and ballot prefix counts place the payloads and hora entries. The count pass writes the per-game counts;
// the fill pass repeats the walk for the games whose status is OK. -DMJX_HOST_EMUL builds the per-event code for
// tests/host_emul/emul_selfplay.cc.
#pragma once
#include "../../include/mjx.h"
#include "../../include/mjx_selfplay.h"
#include "mjx_types.cuh"

namespace mjx {

constexpr int AW_WARPS = 4;
constexpr int AW_KYOKU_WORDS = 19;  // csrc/mjx_replay.cuh REPLAY_KYOKU_WORDS
enum : int { AW_START_KYOKU = 1, AW_TSUMO, AW_DAHAI, AW_CHI, AW_PON, AW_DAIMINKAN, AW_KAKAN, AW_ANKAN, AW_DORA, AW_REACH,
             AW_REACH_ACCEPTED, AW_HORA, AW_RYUKYOKU, AW_END_KYOKU, AW_START_GAME, AW_END_GAME };

struct AwView {
    const u64* words;  // [n_games, pitch]
    const i32* lens;   // [n_games]
    long long pitch;
    int log_cap, n_games, augment;
    i32* counts;  // [n_games, 4]: status, n_events, n_kyoku, n_hora
    // fill pass
    const i32 *ev_off, *ky_off, *hora_off;
    u64* hdr;
    i32* lines;
    long long n_hdr;
    u64* kyoku;
    long long n_kyoku;  // payloads
    u64* hora;
    long long n_hora;  // entries
    i32* deltas;
    u8* has_deltas;
};

// the words of game g inside the log capacity (reads never pass it); MJX_AW_CAPACITY for a log longer than that
MJX_D int aw_game_words(const AwView& V, int g, const u64** w, int* n) {
    const int len = V.lens[g];
    *w = V.words + (long long)g * V.pitch;
    *n = len < 0 ? 0 : len > V.log_cap ? V.log_cap : len;
    return len < 0 || len > V.log_cap ? MJX_AW_CAPACITY : MJX_AW_OK;
}

MJX_D int aw_payload(int ty) { return ty == AW_START_KYOKU ? 9 : (ty == AW_HORA || ty == AW_RYUKYOKU) ? 2 : 0; }

// the word index after the event at i (n = the game's word count), or -MJX_AW_CORRUPT where decode_events raises
MJX_D int aw_next(const u64* w, int n, int i) {
    const int ty = (int)(w[i] & 0xFF);
    if (ty < AW_START_KYOKU || ty > AW_END_KYOKU) return -MJX_AW_CORRUPT;
    const int nx = i + 1 + aw_payload(ty);
    return nx > n ? -MJX_AW_CORRUPT : nx;
}

// the tile indices decode_events reads from the event at i (an index past 37 is an IndexError there), as csrc/mjx_mjai_write.cuh
// mw_event checks them; i's payload lies inside the game (aw_next)
MJX_D int aw_check(const u64* w, int i) {
    const u64 x = w[i];
    const int ty = (int)(x & 0xFF), pai = (int)(x >> 12) & 0xFF, aux = (int)(x >> 21) & 7;
    int nc = 0;
    bool need_pai = false;
    switch (ty) {
        case AW_START_KYOKU:
            if (27 + (int)((x >> 24) & 0xFF) / 4 > 37) return MJX_AW_CORRUPT;
            need_pai = true;
            for (int k = 0; k < 52; k++)
                if ((int)((w[i + 3 + k / 8] >> (8 * (k % 8))) & 0xFF) > 37) return MJX_AW_CORRUPT;
            break;
        case AW_TSUMO: case AW_DAHAI: case AW_DORA: need_pai = true; break;
        case AW_CHI: case AW_PON: need_pai = true; nc = 2; break;
        case AW_DAIMINKAN: case AW_KAKAN: need_pai = true; nc = 3; break;
        case AW_ANKAN: nc = 4; break;
        case AW_HORA: nc = aux < 5 ? aux : 5; break;
        default: break;
    }
    if (need_pai && pai > 37) return MJX_AW_CORRUPT;
    for (int k = 0; k < nc; k++)
        if ((int)((x >> (24 + 8 * k)) & 0xFF) > 37) return MJX_AW_CORRUPT;  // k = 4: the hora's fifth ura marker (bits 56-63)
    return MJX_AW_OK;
}

// Tile::augment (tile.rs:154-167): manzu <-> pinzu, 5mr <-> 5pr; souzu, honours and `?` unchanged
MJX_D int aw_tile(int t, bool aug) {
    if (!aug) return t;
    if (t < 9) return t + 9;
    if (t < 18) return t - 9;
    if (t == 34 || t == 35) return t ^ 34 ^ 35;
    return t;
}

// the same on the eight tile bytes of a word
MJX_D u64 aw_tiles8(u64 v, bool aug) {
    if (!aug) return v;
    u64 out = 0;
    for (int k = 0; k < 8; k++) out |= (u64)aw_tile((int)(v >> (8 * k)) & 0xFF, true) << (8 * k);
    return out;
}

MJX_D u64 aw_word(int ty, int actor, int target, int pai, int tsumogiri, int c0, int c1, int c2, int c3) {
    return (u64)ty | (u64)(actor & 3) << 8 | (u64)(target & 3) << 10 | (u64)(pai & 0xFF) << 12 | (u64)(tsumogiri & 1) << 20 |
           (u64)c0 << 24 | (u64)c1 << 32 | (u64)c2 << 40 | (u64)c3 << 48;
}

// The replay word of the (checked) event at i: dataset_codec.encode_events of the event decode_events reads there. The fields the
// text does not carry are dropped, and a start_kyoku's round comes back as its wind * 4 + oya (the text's `kyoku` is oya + 1).
MJX_D u64 aw_event_word(const u64* w, int i, bool aug) {
    const u64 x = w[i];
    const int ty = (int)(x & 0xFF), actor = (int)(x >> 8) & 3, target = (int)(x >> 10) & 3;
    const int pai = aw_tile((int)(x >> 12) & 0xFF, aug), tsumogiri = (int)(x >> 20) & 1;
    int c[4];
    for (int k = 0; k < 4; k++) c[k] = aw_tile((int)(x >> (24 + 8 * k)) & 0xFF, aug);
    switch (ty) {
        case AW_START_KYOKU: {
            const int kyoku_abs = (int)(x >> 24) & 0xFF, honba = (int)(x >> 32) & 0xFF, kyotaku = (int)(x >> 40) & 0xFF;
            const int oya = (int)(x >> 48) & 0xFF;
            return aw_word(ty, 0, 0, pai, 0, kyoku_abs / 4 * 4 + oya, honba, kyotaku, oya);
        }
        case AW_TSUMO: return aw_word(ty, actor, 0, pai, 0, 0, 0, 0, 0);
        case AW_DAHAI: return aw_word(ty, actor, 0, pai, tsumogiri, 0, 0, 0, 0);
        case AW_CHI: case AW_PON: return aw_word(ty, actor, target, pai, 0, c[0], c[1], 37, 37);
        case AW_DAIMINKAN: return aw_word(ty, actor, target, pai, 0, c[0], c[1], c[2], 37);
        case AW_KAKAN: return aw_word(ty, actor, 0, pai, 0, c[0], c[1], c[2], 37);
        case AW_ANKAN: return aw_word(ty, actor, 0, 37, 0, c[0], c[1], c[2], c[3]);
        case AW_DORA: return aw_word(ty, 0, 0, pai, 0, 0, 0, 0, 0);
        case AW_REACH: case AW_REACH_ACCEPTED: return aw_word(ty, actor, 0, 37, 0, 0, 0, 0, 0);
        case AW_HORA: return aw_word(ty, actor, target, 37, 0, 0, 0, 0, 0);
        default: return aw_word(ty, 0, 0, 37, 0, 0, 0, 0, 0);  // ryukyoku, end_kyoku
    }
}

// the 19-word payload of the start_kyoku at i: its two score words, the 52 dealt tiles, then `?` (0x25) to byte 136
MJX_D void aw_kyoku_payload(const u64* w, int i, bool aug, u64* out) {
    out[0] = w[i + 1];
    out[1] = w[i + 2];
    for (int k = 0; k < 6; k++) out[2 + k] = aw_tiles8(w[i + 3 + k], aug);
    out[8] = (aw_tiles8(w[i + 9], aug) & 0xFFFFFFFFull) | 0x2525252500000000ull;
    for (int k = 9; k < AW_KYOKU_WORDS; k++) out[k] = 0x2525252525252525ull;
}

// the MJX_HORA_WORDS entry of the hora at i: deltas[actor], both fields present (decode_events always writes them), its ura markers
MJX_D void aw_hora_entry(const u64* w, int i, bool aug, u64* out) {
    const u64 x = w[i];
    const int actor = (int)(x >> 8) & 3, aux = (int)(x >> 21) & 7, n = aux < 5 ? aux : 5;
    const u64 d = w[i + 1 + (actor >> 1)] >> (32 * (actor & 1));
    u64 ura = 0;
    for (int k = 0; k < n; k++) ura |= (u64)aw_tile((int)(x >> (24 + 8 * k)) & 0xFF, aug) << (8 * k);
    out[0] = (d & 0xFFFFFFFFull) | 1ull << 32 | 1ull << 33 | (u64)n << 36;
    out[1] = ura;
}

// Writes the (checked) event at word i as replay event e (an absolute index): its word and line, its deltas when it is a hora or
// a ryukyoku, its payload at kyoku index k (start_kyoku) and its entry at hora index h (hora). line = e's 1-based line in the file.
// Every store is bounded by the view's capacities.
MJX_D void aw_fill_event(const AwView& V, const u64* w, int i, long long e, int line, long long k, long long h) {
    const bool aug = V.augment != 0;
    const int ty = (int)(w[i] & 0xFF);
    if (e >= 0 && e < V.n_hdr) {
        V.hdr[e] = aw_event_word(w, i, aug);
        V.lines[e] = line;
        if (ty == AW_HORA || ty == AW_RYUKYOKU) {
            for (int s = 0; s < 4; s++) V.deltas[4 * e + s] = (i32)(u32)(w[i + 1 + (s >> 1)] >> (32 * (s & 1)));
            V.has_deltas[e] = 1;
        }
    }
    if (ty == AW_START_KYOKU && k >= 0 && k < V.n_kyoku) aw_kyoku_payload(w, i, aug, V.kyoku + k * AW_KYOKU_WORDS);
    if (ty == AW_HORA && h >= 0 && h < V.n_hora) aw_hora_entry(w, i, aug, V.hora + h * MJX_HORA_WORDS);
}

// the start_game / end_game word at e (line = e's line)
MJX_D void aw_fill_bound(const AwView& V, int ty, long long e, int line) {
    if (e >= 0 && e < V.n_hdr) {
        V.hdr[e] = aw_word(ty, 0, 0, 37, 0, 0, 0, 0, 0);
        V.lines[e] = line;
    }
}

}  // namespace mjx
