/* mjx_review — reviewing mjai logs with a Mortal engine (csrc/mjx_review.cuh), as mortal.py with MORTAL_REVIEW_MODE=1 does it one
 * line at a time through mjai.Bot. Same conventions as include/mjx.h: device pointers, 0 or a negative mjx_status, `stream` a
 * cudaStream_t passed as void*.
 *
 * mjx_env_replay_review       review mode for a replay env (mjx_env_create_replay*), before its first mjx_env_replay_step. Every
 *                             job replays from its player's own PlayerState record (a log that hides the player's own tiles fails
 *                             with MJX_REPLAY_ERR_HIDDEN_OWN_TILE), every event is applied, and each step stops the job at its
 *                             seat's next event where it can act: the decision row, then the kan-select row when an ankan or kakan
 *                             is possible. row_step = the event index, row_label = the action the log shows next or -1;
 *                             mjx_env_results steps = the event a job stopped at (its event count, or the event it failed at).
 * mjx_review_react_dev        after the engine call on the step's n_rows rows (actions int64, q float32 [n_rows, 46], greedy uint8):
 *                             the agari guard (agari_guard != 0), the reaction word and the records of every row (layout in
 *                             csrc/mjx_review.cuh: info int32 [.., 4], mask uint64, q float32 [.., 46], i64s int64 [.., 2], word
 *                             uint64, all indexed by row). A reaction that cannot be decoded fails its job (mjx_env_results err).
 * mjx_review_render_*_dev     the review text of n_jobs jobs from their records (rec_off int64 [n_jobs + 1], records of a job in
 *                             event order): one line per event, the reaction with its meta or {"type":"none","meta":{"mask_bits":0}}.
 *                             count: bytes int64 [n_jobs] (0 where skip[j]); fill: job j at out + off[j], nothing written at or
 *                             past out_cap. */
#ifndef MJX_REVIEW_H
#define MJX_REVIEW_H
#include <stdint.h>

#include "mjx.h"

#ifdef __cplusplus
extern "C" {
#endif

int mjx_env_replay_review(mjx_env* env, void* stream);
int mjx_review_react_dev(mjx_env* env, int n_rows, const int64_t* actions, const float* q, const uint8_t* greedy, int agari_guard,
                         int32_t* info, uint64_t* mask, float* q_out, int64_t* i64s, uint64_t* word, void* stream);
int mjx_review_render_count_dev(int n_jobs, const int32_t* ev_cnt, const int64_t* rec_off, long long n_rec, const int32_t* rec_event,
                                const uint8_t* rec_kan, const uint64_t* rec_word, const int32_t* rec_info, const uint64_t* rec_mask,
                                const float* rec_q, const int64_t* rec_i64, const uint8_t* skip, int64_t* bytes, void* stream);
int mjx_review_render_fill_dev(int n_jobs, const int32_t* ev_cnt, const int64_t* rec_off, long long n_rec, const int32_t* rec_event,
                               const uint8_t* rec_kan, const uint64_t* rec_word, const int32_t* rec_info, const uint64_t* rec_mask,
                               const float* rec_q, const int64_t* rec_i64, const uint8_t* skip, const int64_t* off, char* out,
                               long long out_cap, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MJX_REVIEW_H */
