// ORACLE — TEST INFRASTRUCTURE ONLY.
// CPU restatement (scalar C++17) of the libriichi self-play hot path. Nothing in
// the product (mortal_b200/) may include, link or call this; only tests/,
// __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs do.
//
// Every function cites the reference file:line (relative to
// Mortal's libriichi/src) whose behaviour it restates.
#pragma once
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>
#include <array>
#include <stdexcept>

namespace orc {

typedef uint8_t u8;
typedef int8_t i8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef int32_t i32;
typedef uint64_t u64;

// ---- tile ids: tile.rs:12-19, macros.rs:9-135 ----
constexpr u8 T_1M = 0, T_5M = 4, T_9M = 8, T_1P = 9, T_5P = 13, T_9P = 17, T_1S = 18, T_2S = 19,
             T_3S = 20, T_4S = 21, T_5S = 22, T_6S = 23, T_8S = 25, T_9S = 26, T_E = 27, T_S = 28,
             T_W = 29, T_N = 30, T_P = 31, T_F = 32, T_C = 33, T_5MR = 34, T_5PR = 35, T_5SR = 36,
             T_UNK = 37, T_NONE = 0xFF;

// tile.rs:68-76
inline u8 deaka(u8 t) { return t == T_5MR ? T_5M : t == T_5PR ? T_5P : t == T_5SR ? T_5S : t; }
// tile.rs:80-88
inline u8 akaize(u8 t) { return t == T_5M ? T_5MR : t == T_5P ? T_5PR : t == T_5S ? T_5SR : t; }
// tile.rs:92-94
inline bool is_aka(u8 t) { return t >= T_5MR && t <= T_5SR; }
// tile.rs:98-100
inline bool is_jihai(u8 t) { return t >= T_E && t <= T_C; }
// tile.rs:104-109
inline bool is_yaokyuu(u8 t) {
    return t == T_1M || t == T_9M || t == T_1P || t == T_9P || t == T_1S || t == T_9S || is_jihai(t);
}
// tile.rs:119-135
inline u8 tile_next(u8 t) {
    if (t >= T_UNK) return t;
    u8 d = deaka(t), kind = d / 9, num = d % 9;
    if (kind < 3) return kind * 9 + (num + 1) % 9;
    if (num < 4) return 27 + (num + 1) % 4;
    return 27 + 4 + (num - 4 + 1) % 3;
}
// tile.rs:139-154
inline u8 tile_prev(u8 t) {
    if (t >= T_UNK) return t;
    u8 d = deaka(t), kind = d / 9, num = d % 9;
    if (kind < 3) return kind * 9 + (num + 9 - 1) % 9;
    if (num < 4) return 27 + (num + 4 - 1) % 4;
    return 27 + 4 + (num - 4 + 3 - 1) % 3;
}
// tile.rs:20-27, 177-185 — returns <0, 0, >0
int cmp_discard_priority(u8 l, u8 r);

struct OrcError : std::runtime_error {
    using std::runtime_error::runtime_error;
};
#define ORC_ENSURE(cond, msg) \
    do { if (!(cond)) throw ::orc::OrcError(msg); } while (0)

// ---- algo ----
void tables_init(const char* data_dir);  // loads shanten_suhai.bin, shanten_jihai.bin, agari.bin
bool tables_ready();

// shanten.rs:88-150
i8 shanten_normal(const u8* tiles34, u8 len_div3);
i8 shanten_chitoi(const u8* tiles34);
i8 shanten_kokushi(const u8* tiles34);
i8 shanten_all(const u8* tiles34, u8 len_div3);

// point.rs:5-112
struct Point {
    i32 ron = 0, tsumo_ko = 0, tsumo_oya = 0;
    i32 tsumo_total(bool is_oya) const { return is_oya ? tsumo_ko * 3 : tsumo_ko * 2 + tsumo_oya; }
};
Point point_calc(bool is_oya, u8 fu, u8 han);
Point point_yakuman(bool is_oya, i32 count);

// agari.rs:66-74 — Agari enum
struct Agari {
    bool valid = false;  // Option::None when false
    bool is_yakuman = false;
    u8 fu = 0, han = 0;  // Normal
    u8 yakuman = 0;      // Yakuman(n)
    Point point(bool is_oya) const {
        return is_yakuman ? point_yakuman(is_oya, yakuman) : point_calc(is_oya, fu, han);
    }
};
int agari_cmp(const Agari& l, const Agari& r);  // agari.rs:175-190

// agari.rs:77-101
struct AgariCalc {
    const u8* tehai;  // [34], includes the winning tile
    bool is_menzen;
    const u8* chis; int n_chis;
    const u8* pons; int n_pons;
    const u8* minkans; int n_minkans;
    const u8* ankans; int n_ankans;
    u8 bakaze, jikaze;
    u8 winning_tile;  // deaka'd
    bool is_ron;

    bool has_yaku() const;                            // agari.rs:206-208
    Agari search_yakus() const;                       // agari.rs:212-214
    Agari agari(u8 additional_hans, u8 doras) const;  // agari.rs:225-255
};
// agari.rs:767-838
u32 get_tile14_and_key(const u8* tiles34, u8* tile14);
// number of divs in AGARI_TABLE for key, or -1 if absent
int agari_table_lookup(u32 key, u32* divs4);
// agari.rs:854-912
bool check_ankan_after_riichi(const u8* tehai34, u8 len_div3, u8 tile, bool strict);

// rankings.rs:8-22
void rankings(const i32* scores4, u8* player_by_rank4, u8* rank_by_player4);

}  // namespace orc
