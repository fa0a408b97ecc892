// mortal_b200 — H100-native batched riichi environment (sm_90a).
// Table record layout in HBM and small tile helpers.
//
// One table = one 16-byte-aligned record. A warp owns a table: it loads the record into shared
// memory with 32 lanes x uint4 (fully coalesced, record-major), mutates it there and stores it back.
// Unlike the reference (4 x PlayerState per table, player_state.rs:24-140) the record keeps the
// *public* information once, in absolute seats, and only the genuinely private part per seat;
// everything a seat can derive (tiles_seen, doras_owned/seen, rank, rotated scores, winds, the
// perspective-dependent start-of-kyoku kawa pads) is recomputed where it is consumed.
#pragma once
#include "mjx_port.cuh"

namespace mjx {

typedef uint8_t u8;
typedef int8_t i8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef int32_t i32;
typedef uint64_t u64;
typedef int64_t i64;

constexpr u8 T_1M = 0, T_5M = 4, T_9M = 8, T_1P = 9, T_5P = 13, T_9P = 17, T_1S = 18, T_2S = 19, T_3S = 20,
             T_4S = 21, T_5S = 22, T_6S = 23, T_8S = 25, T_9S = 26, T_E = 27, T_S = 28, T_W = 29, T_N = 30,
             T_P = 31, T_F = 32, T_C = 33, T_5MR = 34, T_5PR = 35, T_5SR = 36, T_UNK = 37, T_NONE = 0xFF;

constexpr int ACTION_SPACE = 46;   // consts.rs:7-15
constexpr int KAWA_CAP = 32;       // player_state.rs:74-80: 24 real discards + None pads
constexpr int MAX_ROWS_PER_TABLE = 3;

// ---- tile helpers (tile.rs:68-154) ----
MJX_HD int deaka(int t) { return t >= T_5MR && t <= T_5SR ? (t - T_5MR) * 9 + 4 : t; }
MJX_HD int akaize(int t) { return (t == T_5M || t == T_5P || t == T_5S) ? T_5MR + t / 9 : t; }
MJX_HD bool is_aka(int t) { return t >= T_5MR && t <= T_5SR; }
MJX_HD bool is_jihai(int t) { return t >= T_E && t <= T_C; }
constexpr u64 YAOKYUU_MASK = (1ull << 0) | (1ull << 8) | (1ull << 9) | (1ull << 17) | (1ull << 18) | (1ull << 26) |
                             (0x7Full << 27);
MJX_HD bool is_yaokyuu(int t) { return t < 34 && ((YAOKYUU_MASK >> t) & 1ull); }
MJX_HD int tile_next(int t) {
    if (t >= T_UNK) return t;
    int d = deaka(t), kind = d / 9, num = d % 9;
    if (kind < 3) return kind * 9 + (num + 1) % 9;
    if (num < 4) return 27 + (num + 1) % 4;
    return 31 + (num - 4 + 1) % 3;
}
MJX_HD int tile_prev(int t) {
    if (t >= T_UNK) return t;
    int d = deaka(t), kind = d / 9, num = d % 9;
    if (kind < 3) return kind * 9 + (num + 8) % 9;
    if (num < 4) return 27 + (num + 3) % 4;
    return 31 + (num - 4 + 2) % 3;
}
// ---- action candidate bits (action.rs:11-40) ----
enum : u16 {
    CAN_DISCARD = 1 << 0, CAN_CHI_LOW = 1 << 1, CAN_CHI_MID = 1 << 2, CAN_CHI_HIGH = 1 << 3, CAN_PON = 1 << 4,
    CAN_DAIMINKAN = 1 << 5, CAN_KAKAN = 1 << 6, CAN_ANKAN = 1 << 7, CAN_RIICHI = 1 << 8, CAN_TSUMO_AGARI = 1 << 9,
    CAN_RON_AGARI = 1 << 10, CAN_RYUKYOKU = 1 << 11,
    CAN_CHI = CAN_CHI_LOW | CAN_CHI_MID | CAN_CHI_HIGH,
    CAN_KAN = CAN_DAIMINKAN | CAN_KAKAN | CAN_ANKAN,
    CAN_AGARI = CAN_TSUMO_AGARI | CAN_RON_AGARI,
    CAN_PASS = CAN_CHI | CAN_PON | CAN_DAIMINKAN | CAN_RON_AGARI,
    CAN_ACT = 0x0FFF,
};

// per-seat private flags
enum : u16 {
    PF_CAN_W_RIICHI = 1 << 0, PF_IS_W_RIICHI = 1 << 1, PF_AT_RINSHAN = 1 << 2, PF_AT_IPPATSU = 1 << 3,
    PF_AT_FURITEN = 1 << 4, PF_MARK_SAME_CYCLE_FURITEN = 1 << 5, PF_CHANKAN_CHANCE = 1 << 6, PF_IS_MENZEN = 1 << 7,
    PF_HAS_NEXT_SHANTEN_DISCARD = 1 << 8,
};

// board flags
enum : u16 {
    BF_DEAL_FROM_RINSHAN = 1 << 0, BF_NEW_DORA_AT_DISCARD = 1 << 1, BF_NEW_DORA_AT_TSUMO = 1 << 2,
    BF_CAN_FOUR_WIND = 1 << 3, BF_CHECK_FOUR_KAN = 1 << 4, BF_CAN_RENCHAN = 1 << 5, BF_HAS_HORA = 1 << 6,
    BF_HAS_ABORTIVE = 1 << 7, BF_HAS_CHIPON_PENDING = 1 << 8,
};

// game flags
enum : u8 { GF_KYOKU_STARTED = 1, GF_ENDED = 2, GF_IN_RENCHAN = 4, GF_ALIVE = 8 };

// sutehai flags inside a kawa item / Sutehai (item.rs:14-21)
enum : u8 { SF_DORA = 1, SF_TEDASHI = 2, SF_RIICHI = 4, SF_HAS_CHIPON = 8, SF_VALID = 0x80 };

// One discard-pond entry (item.rs:7-12), 8 bytes. tile == T_NONE means a `None` pad.
struct KawaItem {
    u8 tile;         // 0..36 incl. aka, or T_NONE
    u8 flags;        // SF_*
    u8 consumed[2];  // chi/pon consumed tiles (deaka'd)
    u8 kan[4];       // kan tiles declared before this discard (deaka'd), T_NONE = empty
};

struct SeatPrivate {
    u8 tehai[34];            // no aka (player_state.rs:29)
    u8 tehai_len_div3;
    i8 shanten;
    u64 waits;               // bit t
    u64 keep_shanten;        // keep_shanten_discards
    u64 next_shanten;        // next_shanten_discards
    u64 forbidden;           // kuikae
    u64 discarded;           // furiten check
    u64 ankan_cand, kakan_cand;
    u16 flags;               // PF_*
    u16 cans;                // CAN_*
    u8 target_actor;
    u8 last_self_tsumo;      // T_NONE if none
    u8 akas_in_hand;         // 3 bits
    u8 at_turn;
    u8 chis[4], pons[4], minkans[4], ankans[4];
    u8 n_chis, n_pons, n_minkans, n_ankans;
    u8 pad_[4];
};

struct SeatPublic {
    KawaItem kawa[KAWA_CAP];  // without the start-of-kyoku pads (update.rs:819-824; added at encode time)
    u8 fuuro[4][4];           // fuuro_overview, tiles incl. aka, T_NONE = empty
    u8 ankan[4];              // ankan_overview (deaka'd)
    u8 kawa_len, n_fuuro, n_ankan;
    u8 last_tedashi_tile, last_tedashi_flags;  // flags & SF_VALID
    u8 riichi_tile, riichi_flags;
    u8 pad_;
};

struct TableState {
    // ---- game (game.rs:28-55) ----
    u64 nonce, key;
    i32 scores[4];
    u32 step_idx;
    i32 err;
    u8 kyoku, honba, kyotaku, gflags;
    u8 shuffle_kind;
    u8 n_kyoku_played;
    u8 viewer1;              // 0: the record holds all four hands (arena, full-information replay); s + 1: a single PlayerState of
                             // seat s (state/player_state.rs) — the other seats' hands are unknown (`?`) and stay untouched
    u8 pad0_[1];
    i32 row_of_seat[4];      // decision rows handed to the policy this cycle (-1 none)
    i32 kan_row_of_seat[4];
    i8 auto_action[4];       // quick-eval shortcut (mortal.rs:210-242), -1 none
    // ---- board (board.rs:52-85) ----
    i32 kyoku_deltas[4];
    u16 bflags;
    u8 oya, tiles_left, tsumo_actor;
    u8 n_dora;               // dora indicators revealed so far (seq[60 - k])
    u8 n_rinshan;            // rinshan tiles drawn (seq[55 - k])
    i8 riichi_to_be_accepted;
    i8 four_wind_tile;
    u8 accepted_riichis, kans;
    u8 can_nagashi;          // 4 bits
    i8 paos[4];
    u8 riichi_declared, riichi_accepted;  // 4 bits each
    u8 last_kawa_tile;       // T_NONE if none
    u8 n_intermediate_kan;
    u8 intermediate_kan[4];
    u8 chipon_consumed[2];
    u8 akas_public;          // akas visible to everyone (discarded / melded / indicator)
    u8 pad1_[1];
    u8 public_seen[34];      // tiles everyone has seen (discards + meld consumed + indicators)
    u8 pad2_[2];
    u8 wall[136];            // board.rs:109-122 layout
    SeatPrivate priv[4];
    SeatPublic pub[4];
};

// whether the record knows seat s's hand
MJX_HD bool seat_known(const TableState* S, int s) { return S->viewer1 == 0 || S->viewer1 == s + 1; }

static_assert(sizeof(KawaItem) == 8, "KawaItem must be 8 bytes");
static_assert(sizeof(TableState) % 16 == 0, "TableState must be a multiple of 16 bytes");

// lookup tables resident in HBM/L2 (loaded once by mjx_init)
struct Tables {
    const u64* suhai;     // 5^9 rows, 10 nibbles each in the low 40 bits (zero beyond 1,940,777: shanten.rs:52)
    const u64* jihai;     // 5^7 rows
    const u32* agari_keys;   // open-addressing hash, AGARI_SLOTS entries, 0xFFFFFFFF = empty
    const U4* agari_divs;    // up to 4 divs per key, 0 = none (a real div is never 0)
    const u8* agari_ndivs;
};
constexpr u32 AGARI_SLOTS = 32768;
constexpr u32 SUHAI_ROWS = 1953125, JIHAI_ROWS = 78125;

}  // namespace mjx
