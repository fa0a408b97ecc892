/* mjx_selfplay — arena event words -> the replay arrays of libmjx.so (csrc/mjx_selfplay.cuh), for training on self-play games
 * without writing their logs. Same conventions as include/mjx.h: device pointers, 0 or a negative mjx_status, `stream` a
 * cudaStream_t passed as void*.
 *
 * Input: the arena's words of n_games games, uint64 [n_games, pitch] (game g at words + g * pitch, the layout of
 * mjx_env_log_words_dev) and lens int32 [n_games] (mjx_env_log_len_dev). Every read stays inside a game's first log_cap <= pitch
 * words. The output is what mjx_mjai_fill_deltas_dev writes for the text mortal_b200/mjai_log.py writes for that game
 * (decode_events + dump_json_log): start_game and end_game words around the game's events, one word per event, the 19-word
 * start_kyoku payloads (2 score words + the 136-byte wall: the 52 dealt tiles, then `?` = 37), the MJX_HORA_WORDS-word entry of
 * every hora, deltas / has_deltas at every hora and ryukyoku, and lines[e] = the event's 1-based line in the written file
 * (start_game is line 1). `augment` != 0 applies Tile::augment (manzu <-> pinzu, 5mr <-> 5pr) to every tile field.
 * Two phases, both enqueued on `stream` without a synchronise; one warp per game:
 *   mjx_arena_words_count_dev  -> counts int32 [n_games, 4] = {mjx_aw_status, n_events, n_kyoku, n_hora} (n_events counts the
 *                                 start_game and end_game words; all three are zero unless the status is OK);
 *   mjx_arena_words_fill_dev   the arrays of the games whose counts say OK: game g's first word / line at ev_off[g], first payload
 *                                 at ky_off[g], first hora entry at hora_off[g] (device int32 [n_games]); deltas int32 [n_hdr, 4]
 *                                 and has_deltas uint8 [n_hdr] share the word array's indexing. Nothing is written at or past
 *                                 n_hdr / n_kyoku_words / n_hora_words. */
#ifndef MJX_SELFPLAY_H
#define MJX_SELFPLAY_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* CORRUPT: a word whose type is not an arena event, a tile index past 37 where decode_events reads one, or a payload running past
 * lens[g] (decode_events raises on all three); CAPACITY: lens[g] > log_cap or < 0 (the arena log overflowed). */
enum mjx_aw_status { MJX_AW_OK = 0, MJX_AW_CORRUPT = 1, MJX_AW_CAPACITY = 2 };

int mjx_arena_words_count_dev(int n_games, const uint64_t* words, const int32_t* lens, long long pitch, int log_cap,
                              int32_t* counts, void* stream);
int mjx_arena_words_fill_dev(int n_games, const uint64_t* words, const int32_t* lens, long long pitch, int log_cap, int augment,
                             const int32_t* counts, const int32_t* ev_off, const int32_t* ky_off, const int32_t* hora_off,
                             uint64_t* hdr, int32_t* lines, long long n_hdr, uint64_t* kyoku, long long n_kyoku_words,
                             uint64_t* hora_payload, long long n_hora_words, int32_t* deltas, uint8_t* has_deltas, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MJX_SELFPLAY_H */
