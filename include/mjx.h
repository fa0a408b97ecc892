/* mjx — C ABI of the H100-native batched riichi self-play environment (libmjx.so).
 *
 * This is the drop-in boundary for libriichi's self-play hot path. libriichi has no C ABI of its
 * own (it is Rust re-exported through PyO3); each entry point below names the reference interface
 * it stands in for (paths relative to Mortal's libriichi/src). Plain pointers and sizes only;
 * "dev" pointers are CUDA device pointers (e.g. torch.Tensor.data_ptr()), "host" pointers are
 * ordinary host memory; `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 * Every function returns 0 on success or a negative mjx_status; mjx_last_error() gives the text.
 * There is no CPU fallback: without a CUDA device every call fails with MJX_ERR_CUDA.
 */
#ifndef MJX_H
#define MJX_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum mjx_status { MJX_OK = 0, MJX_ERR_CUDA = -1, MJX_ERR_ARG = -2, MJX_ERR_TABLES = -3, MJX_ERR_STATE = -4 };

#define MJX_ACTION_SPACE 46      /* consts.rs:7-15 */
#define MJX_OBS_COLS 34
#define MJX_MAX_ROWS_PER_TABLE 3 /* <=3 seats can act on one event; a kan-select pass adds a row to 1 */

typedef struct mjx_env mjx_env;

const char* mjx_last_error(void);

/* lib.rs:139-140 (shanten::ensure_init / agari::ensure_init): load the three lookup tables from
 * `data_dir` (shanten_suhai.bin, shanten_jihai.bin, agari.bin) into device memory of `device`. */
int mjx_init(const char* data_dir, int device);

/* consts.rs:20-28 obs_shape(version).0 ; returns <0 for an unsupported version. */
int mjx_obs_rows(int version);

/* ---- environment: arena/game.rs:230-316 BatchGame::run over n_tables Game objects -------------
 * seeds: host arrays (nonce, key) per table = GameResult.seed (arena/one_vs_three.rs:140-142).
 * shuffle_kind: 0 = rand 0.9.1 (Cargo.lock:1042), 1 = rand 0.8 (the shipped seeded log).
 * enable_quick_eval: agent/mortal.rs:210-242. obs_version: consts.rs MAX_VERSION (4 supported). */
int mjx_env_create(mjx_env** out, int n_tables, const uint64_t* nonces_host, const uint64_t* keys_host,
                   int obs_version, int shuffle_kind, int enable_quick_eval);
void mjx_env_destroy(mjx_env* env);

/* One BatchGame::run loop iteration for every live table (game.rs:286-304): commit the actions
 * chosen for the rows of the previous step (agent/mortal.rs:292-573 decode + board.rs:524-533
 * validation), then poll every table to its next decision point (game.rs:59-178) and emit the
 * decision rows + legal masks (agent/mortal.rs:200-290). `actions_dev` = int64 [row_cap], indexed
 * by the previous step's row numbers (ignored on the first step; may be NULL then).
 * `q_values_dev` = float32 [row_cap, 46] Q-values of those rows, or NULL; only read for seats whose engine
 * set enable_rule_based_agari_guard (agent/mortal.rs:319-336: "wants agari but the guard objects -> best other Q"). */
int mjx_env_step(mjx_env* env, const int64_t* actions_dev, const float* q_values_dev, void* stream);

/* agent/mortal.rs:54-74, 210-250: enable_quick_eval is a property of the agent, so of the seat: host uint8 [n_tables, 4]
 * (NULL = the single flag given to mjx_env_create for every seat). */
int mjx_env_set_quick_eval(mjx_env* env, const uint8_t* flags_host);

/* agent/mortal.rs:61-66 enable_rule_based_agari_guard per table and seat: host uint8 [n_tables, 4] (NULL = off).
 * The guard itself is state/agent_helper.rs:262-368 rule_based_agari, evaluated on device. */
int mjx_env_set_agari_guard(mjx_env* env, const uint8_t* flags_host);

/* state/obs_repr.rs:776-790 encode_obs for every row of the current step:
 * obs_dev = float32 [row_cap, rows(version), 34] (only the first n_rows rows are written). */
int mjx_env_encode_obs(mjx_env* env, float* obs_dev, void* stream);

/* The same for a caller that holds HOST buffers (what agent/mortal.rs:126-152 hands to react_batch): encodes into the
 * device scratch `obs_dev` [row_cap, rows, 34] and copies rows [0, *n_rows) to `obs_host` (same layout) and `masks_host`
 * (uint8 [row_cap, 46]). The single-player block is computed in four row groups and the finished observations of one group drain
 * through the copy engine while the SMs work on the next. Blocking; host buffers should be pinned (cudaHostAlloc / torch
 * pin_memory) for the overlap to happen. */
int mjx_env_encode_obs_host(mjx_env* env, float* obs_dev, float* obs_host, uint8_t* masks_host, int* n_rows, void* stream);
/* The same in two halves, so that a caller can overlap the device work and the D2H copies of one batch with host work on
 * another (the libriichi.arena mirror steps two half-batches alternately): _begin enqueues everything and returns as soon as
 * *n_rows is known (it waits for the step kernel only); _finish blocks until the host buffers are complete. */
int mjx_env_encode_obs_host_begin(mjx_env* env, float* obs_dev, float* obs_host, uint8_t* masks_host, int* n_rows, void* stream);
int mjx_env_encode_obs_host_finish(mjx_env* env);

/* arena/board.rs:680-782 encode_oracle_obs for every row of the current step — the invisible observation an `is_oracle`
 * engine receives as react_batch's third argument (agent/mortal.rs:253-255; dataset/invisible.rs for the loader):
 * inv_dev = float32 [row_cap, mjx_oracle_obs_rows(version), 34]. consts.rs:30-38: 211 rows for version 1, else 217. */
int mjx_oracle_obs_rows(int version);
int mjx_env_encode_invisible(mjx_env* env, float* inv_dev, int version, void* stream);

/* Switch the observation version the encoder entry points produce (consts.rs:20-28; obs buffers must then hold
 * mjx_obs_rows(version) rows per observation). agent/mortal.rs:54-74: every agent has its own `version`; a PlayerState encodes
 * any version on request (obs_repr.rs:780). */
int mjx_env_set_obs_version(mjx_env* env, int version);

/* state/agent_helper.rs:509-593 single_player_tables (obs v4 rows 889-1011): on by default; `enable = 0`
 * leaves the block zero (the reference has no such switch; it exists for profiling the rest of the encoder).
 * mjx_env_sp_overflows: number of steps so far in which the state arena (2048 states per table on average)
 * overflowed and the blocks of that step were left zero — the reference has no such limit; it is 0 in every
 * test and benchmark here and is reported rather than hidden. */
int mjx_env_set_sp(mjx_env* env, int enable);
int mjx_env_sp_overflows(mjx_env* env, void* stream, int* n);

/* Size of the last step's single-player DP: out[0] = states, out[1] = edges, out[2..9] = states per level slot
 * (D3 W3 D2 W2 D1 W1 D0 W0). Instrumentation for profiles/ and bench.py; blocking. */
int mjx_env_sp_stats(mjx_env* env, void* stream, int* out10);

/* Blocking read-backs (synchronise `stream` first). */
int mjx_env_num_rows(mjx_env* env, void* stream, int* n_rows);          /* rows emitted by the last step */
int mjx_env_num_live(mjx_env* env, void* stream, int* n_live);          /* tables still playing */
int mjx_env_total_steps(mjx_env* env, void* stream, int64_t* steps);    /* game.rs:304 `actions` counter */

/* One blocking read-back per BatchGame::run cycle: out4 = { rows emitted by the last step, tables still playing,
 * tables that have failed so far (err != 0; game.rs:288,292 aborts the batch at that cycle, so should the caller),
 * single-player arena overflows so far (see mjx_env_sp_overflows) }. */
int mjx_env_poll(mjx_env* env, void* stream, int* out4);

/* arena/result.rs:19-51 GameResult.game_log: record every table's mjai events on device (compact 64-bit words, layout in
 * csrc/mjx_step.cuh `log_word`; mortal_b200/mjai_log.py turns them into the reference's JSON lines). Call
 * mjx_env_enable_log before the first step; `words_per_table` bounds one hanchan (a kyoku is ~170 words; 8192 is ample).
 * mjx_env_read_log copies [n_tables, words_per_table] words and the per-table counts to host (count > capacity = overflow). */
int mjx_env_enable_log(mjx_env* env, int words_per_table);
int mjx_env_read_log(mjx_env* env, void* stream, uint64_t* words_host, int32_t* len_host);
int32_t* mjx_env_log_len_dev(mjx_env* env); /* int32 [n_tables] device view of the per-table word counts (null before enable_log):
                                              read after every step it tells which events that step wrote (per-decision meta) */
uint64_t* mjx_env_log_words_dev(mjx_env* env); /* uint64 [n_tables, words_per_table] device view of the words (null before
                                                  enable_log); words past a table's count are undefined */

/* ---- mjai log text from the event words: mortal_b200/mjai_log.py decode_events + attach_meta + dump_json_log (csrc/mjx_mjai_write.cuh)
 * Every game's event lines, byte for byte what the host writer produces between its start_game and end_game lines (those carry the
 * names and the seed and are rendered by the caller). Device pointers, enqueued on `stream` without a synchronise; one warp per game.
 *   words   uint64 [n_games, log_cap] and lens int32 [n_games] (mjx_env_log_words_dev / mjx_env_log_len_dev);
 *   bounds  int32 [n_steps, n_games]: game g's word count right after environment step c (null or n_rec == 0: no meta);
 *   records one per decision row, sorted by key = ((game * key_steps + step) * 4 + seat) * 2 + kan_select (key_steps > every step):
 *           rec_info int32 [n_rec, 4] = {action, MJX_MW_REC_* flags, shanten, row order}, rec_mask uint64 [n_rec] (46 legal bits),
 *           rec_q float32 [n_rec, 46], rec_i64 int64 [n_rec, 2] = {batch_size, eval_time_ns}.
 * An agent event at word offset `off` takes the record of (game, step = bisect_right(bounds[:, g], off) - 1, actor, 0) when that
 * record's action produces the event type (ryukyoku: the seat whose action is 44); action 42 nests the (…, 1) record as kan_select.
 *   mjx_mjai_render_count_dev -> bytes int32 [n_games] (the text length), status int32 [n_games] (mjx_mw_status: non-zero = the host
 *                                writer raises on this game; its bytes are then 0);
 *   mjx_mjai_render_fill_dev  the text of games [g0, g1) with status OK: game g at out + off[g] - off[g0] (off int64 [n_games + 1],
 *                                the exclusive sum of bytes); nothing is written at or past out_cap.
 * Reads never pass a game's log_cap words. */
/* Per-decision meta records for the renderer, appended on the device on `stream` (no synchronise): for the i-th of the n rows of an
 * agent call (row = idx[i], or i when idx is null), record base + i gets the row's table (row_table), `cycle`, seat | kan_select << 2
 * (row_seat), out_info {actions[row], MJX_MW_REC_* flags (greedy[i], or greedy when null; shanten / furiten when obs is given),
 * shanten = the first maximum of obs rows 862-868 at column 0, row}, the 46 legal bits of masks[row], the call's Q-values q[i]
 * (float32 [n, 46], call order) and call_ids[i] (or `call`). obs: float32 [row_cap, obs_rows, 34] v4 observation or null. Fails
 * with MJX_ERR_ARG, writing nothing, unless base + n <= cap; a row index outside row_cap gives a record no event matches. */
int mjx_meta_record_dev(long long n, const int64_t* idx, const float* q, const uint8_t* greedy, const int32_t* call_ids, int call,
                        int cycle, const int32_t* row_table, const uint8_t* row_seat, const int64_t* actions, const uint8_t* masks,
                        const float* obs, int obs_rows, int row_cap, int32_t* out_table, int32_t* out_cycle, uint8_t* out_seat,
                        int32_t* out_info, uint64_t* out_mask, float* out_q, int32_t* out_call, long long base, long long cap,
                        void* stream);
enum mjx_mw_status { MJX_MW_OK = 0, MJX_MW_CORRUPT = 1, MJX_MW_TRUNCATED = 2, MJX_MW_CAPACITY = 3 };
enum mjx_mw_event { MJX_MW_T_START_KYOKU = 1, MJX_MW_T_TSUMO, MJX_MW_T_DAHAI, MJX_MW_T_CHI, MJX_MW_T_PON, MJX_MW_T_DAIMINKAN,
                    MJX_MW_T_KAKAN, MJX_MW_T_ANKAN, MJX_MW_T_DORA, MJX_MW_T_REACH, MJX_MW_T_REACH_ACCEPTED, MJX_MW_T_HORA,
                    MJX_MW_T_RYUKYOKU, MJX_MW_T_END_KYOKU };
enum mjx_mw_rec_flag { MJX_MW_REC_GREEDY = 1, MJX_MW_REC_HAS_SHANTEN = 2, MJX_MW_REC_HAS_FURITEN = 4, MJX_MW_REC_FURITEN = 8 };
int mjx_mjai_render_count_dev(int n_games, const uint64_t* words, const int32_t* lens, int log_cap, const int32_t* bounds,
                              int n_steps, int key_steps, const int64_t* rec_key, const int32_t* rec_info, const uint64_t* rec_mask,
                              const float* rec_q, const int64_t* rec_i64, long long n_rec, int32_t* bytes, int32_t* status,
                              void* stream);
int mjx_mjai_render_fill_dev(int n_games, const uint64_t* words, const int32_t* lens, int log_cap, const int32_t* bounds,
                             int n_steps, int key_steps, const int64_t* rec_key, const int32_t* rec_info, const uint64_t* rec_mask,
                             const float* rec_q, const int64_t* rec_i64, long long n_rec, const int32_t* status, const int64_t* off,
                             int g0, int g1, char* out, long long out_cap, void* stream);

/* dataset/grp.rs:90-164 without the logs: the GRP feature row of every kyoku — {grand_kyoku (E1 = 0 .. S4 = 7, W = 8+), honba,
 * kyotaku, scores[4]} as int32 (the reference's f64 row is these with the scores divided by 10000) — is written by the step
 * kernel when the kyoku starts. mjx_env_read_grp copies [n_tables, max_kyoku, 7] rows and the per-table kyoku counts (a count
 * above max_kyoku = overflow); with mjx_env_results (final scores, rank_by_player) that is everything
 * mortal/reward_calculator.py:13-38 consumes. Call mjx_env_enable_grp before the first step. */
int mjx_env_enable_grp(mjx_env* env, int max_kyoku);
int mjx_env_read_grp(mjx_env* env, void* stream, int32_t* feat_host, int32_t* n_kyoku_host);

/* ---- log replay: dataset/gameplay.rs:247-449 GameplayLoader (SURVEY.md §8f N3) ------------------------------------------
 * A job = one (game log, player). `hdr`: the games' events as 64-bit words (csrc/mjx_step.cuh `log_word`; start_game = 15,
 * end_game = 16), concatenated, job j owning ev_cnt[j] words from ev_off[j]; `kyoku`: 19 words per start_kyoku (2 of scores, 17 = the
 * 136-byte wall in board.rs:109-122 layout: the 52 dealt tiles, the rest `?` = 37 unless the hidden tiles are known),
 * job j's first payload at index ky_off[j]; `players`: the job's point of view. All host arrays. The record holds all four hands,
 * so the logs must carry full information, unless mjx_env_replay_viewpoints (below) is called: then a log may hide the other
 * seats' tiles (`?` = 37) as the mjai protocol shows a game to one seat. mjx_env_replay_step advances every job to the next decision the log shows its player making and emits the row(s)
 * (decision, then kan-select); observation / mask / row_table / row_seat are read exactly as after mjx_env_step, plus the
 * label and (at_kyoku, at_turn, shanten, apply_gamma) of each row. A job is finished when mjx_env_num_live stops counting it. */
int mjx_env_create_replay(mjx_env** out, int n_jobs, const uint64_t* hdr, const int32_t* ev_off, const int32_t* ev_cnt, long long n_hdr,
                          const uint64_t* kyoku, const int32_t* ky_off, long long n_kyoku_words, const uint8_t* players,
                          int obs_version, int always_include_kan_select);
/* The same with `hdr` and `kyoku` in DEVICE memory (e.g. the arrays of mjx_mjai_fill_dev, with host-encoded logs appended): they are
 * copied device to device into the env's own buffers on `stream`, and the stream is synchronised before the call returns, so the
 * caller may free them at once. ev_off, ev_cnt, ky_off and players stay host arrays; a job whose events lie outside [0, n_hdr) or
 * whose first payload lies outside [0, n_kyoku_words / 19] fails the call with MJX_ERR_ARG. */
int mjx_env_create_replay_dev(mjx_env** out, int n_jobs, const uint64_t* hdr, const int32_t* ev_off, const int32_t* ev_cnt,
                              long long n_hdr, const uint64_t* kyoku, const int32_t* ky_off, long long n_kyoku_words,
                              const uint8_t* players, int obs_version, int always_include_kan_select, void* stream);
int mjx_env_replay_step(mjx_env* env, void* stream);
/* dataset/gameplay.rs:240-335 with oracle = false (only the player's own PlayerState is updated): single-viewpoint logs. One launch,
 * enqueued on `stream`, that scans every job's log for hidden seats: a seat is hidden when one of its 13 haipai tiles in a
 * start_kyoku payload, or the pai of one of its tsumo events, is `?` (37). A job whose log hides no seat is left exactly as it
 * was (bit-identical replay). Otherwise the job is replayed from its player's own PlayerState (TableState.viewer1), and when the
 * hidden seats include the player's own, the job fails at its first mjx_env_replay_step with the per-job error code
 * MJX_REPLAY_ERR_HIDDEN_OWN_TILE (state/update.rs:695-699: "attempt to witness an unknown tile"). A job with more start_kyoku
 * events than payloads left after ky_off[j] is not marked. Call after mjx_env_create_replay[_dev] and before the first
 * mjx_env_replay_step; MJX_ERR_ARG on an env that is not a replay env or after mjx_env_replay_trust_seeds (trusted walls are for
 * the invisible observation, whose logs stay full-information), MJX_ERR_STATE after the first step. */
#define MJX_REPLAY_ERR_HIDDEN_OWN_TILE 13
int mjx_env_replay_viewpoints(mjx_env* env, void* stream);
/* dataset/invisible.rs:35-66 (`trust_seed`): the logs were produced from known seeds (start_game.seed, what this arena and
 * libriichi's write) — host arrays (nonce, key) per job. Every kyoku's wall is then regenerated on device (board.rs:99-123), checked
 * against the logged haipai / dora marker (a mismatch fails the job), and mjx_env_encode_invisible can show the hidden tiles.
 * Call before the first mjx_env_replay_step, and not after mjx_env_replay_viewpoints (MJX_ERR_ARG). */
int mjx_env_replay_trust_seeds(mjx_env* env, const uint64_t* nonces_host, const uint64_t* keys_host, int shuffle_kind);
int64_t* mjx_env_row_label(mjx_env* env); /* int64 [row_cap] device */
uint8_t* mjx_env_row_meta(mjx_env* env);  /* uint8 [row_cap, 4] device: at_kyoku, at_turn, shanten (int8), apply_gamma */

/* ---- log validation: bin/validate_logs.rs:62-242 process_path ---------------------------------------------------------
 * Replays every log through the four seats (state/update.rs update_with_keep_cans(ev, true)) and reports the first event a rule
 * forbids. Inputs are host arrays in the mjx_env_create_replay layout (`hdr`, `ev_off`, `ev_cnt`, `kyoku`, `ky_off`; one entry per
 * log) plus the hora side array: MJX_HORA_WORDS words per hora event, log i's first entry at hora_off[i]:
 *   word 0 = (uint32) deltas[actor] | has_deltas << 32 | has_ura << 33 | n_ura << 36,  word 1 = ura tiles, one byte each.
 * out_verdicts: host mjx_verdict [n_logs]. One launch (one warp per log); blocking. */
#define MJX_HORA_WORDS 2
enum mjx_verdict_status { MJX_V_OK = 0, MJX_V_CHECK = 1, MJX_V_UPDATE = 2, MJX_V_PARSE = 3, MJX_V_UNSUPPORTED = 4 };
/* The reasons a verdict can carry: X(enum suffix, name). The CHECK reasons are the 19 checks of process_path in order; UPDATE
 * the errors of PlayerState::update_with_keep_cans (plus a caught panic); PARSE the host-side rejections; UNSUPPORTED an event
 * this implementation's table record cannot hold. This list is the single definition (mortal_b200/validate_logs.py reads it). */
#define MJX_VALIDATE_REASONS(X)                                                                                              \
    X(NONE, "none")                                                                                                          \
    X(CAN_DISCARD, "can_discard") X(DISCARD_CANDIDATES, "discard_candidates") X(CHI_NON_KAMICHA, "chi from non-kamicha")     \
    X(CAN_CHI_LOW, "can_chi_low") X(CAN_CHI_MID, "can_chi_mid") X(CAN_CHI_HIGH, "can_chi_high") X(CAN_PON, "can_pon")        \
    X(CAN_DAIMINKAN, "can_daiminkan") X(CAN_ANKAN, "can_ankan") X(ANKAN_CANDIDATES, "ankan_candidates")                      \
    X(CAN_KAKAN, "can_kakan") X(KAKAN_CANDIDATES, "kakan_candidates") X(CAN_RIICHI, "can_riichi")                            \
    X(CAN_RON_AGARI, "can_ron_agari") X(CAN_TSUMO_AGARI, "can_tsumo_agari") X(MISSING_URA, "missing ura_markers")            \
    X(MISSING_DELTAS, "missing deltas") X(AGARI_POINTS, "agari_points") X(DELTAS_BELOW_POINTS, "deltas below points")       \
    X(EXHAUSTED_YAMA, "tsumo from exhausted yama") X(UNKNOWN_TILE, "witness unknown tile")                                   \
    X(FIFTH_TILE, "witness fifth tile") X(DISCARD_FROM_VOID, "discard from void") X(CONSUME_FROM_VOID, "consume from void")  \
    X(DORA_OVERFLOW, "dora indicator overflow") X(UPDATE_OTHER, "other")                                                     \
    X(PARSE_JSON, "json") X(PARSE_TYPE, "unknown type") X(PARSE_TILE, "unknown tile") X(PARSE_ACTOR, "actor out of range")  \
    X(PARSE_CONSUMED, "consumed length") X(PARSE_FIELD, "missing or invalid field")                                          \
    X(CAPACITY, "capacity")
#define MJX_REASON_ENUM_(id, name) MJX_R_##id,
enum mjx_validate_reason { MJX_VALIDATE_REASONS(MJX_REASON_ENUM_) MJX_R_COUNT };
#undef MJX_REASON_ENUM_
typedef struct mjx_verdict {
    int32_t status;  /* mjx_verdict_status */
    int32_t reason;  /* mjx_validate_reason */
    int32_t line;    /* 1-based event index of the failure (0 when OK) */
    int32_t seat;    /* UPDATE: the lowest seat whose update fails; CHECK: the actor; else -1 */
} mjx_verdict;
int mjx_validate_logs(int n_logs, const uint64_t* hdr, const int32_t* ev_off, const int32_t* ev_cnt, long long n_hdr,
                      const uint64_t* kyoku, const int32_t* ky_off, long long n_kyoku_words, const uint64_t* hora_payload,
                      const int32_t* hora_off, long long n_hora_words, mjx_verdict* out_verdicts, void* stream);
/* The same over device arrays, enqueued on `stream` without a synchronise (out_verdicts: device mjx_verdict [n_logs]). A log whose
 * event range lies outside the word array gets an UNSUPPORTED verdict instead of being read. */
int mjx_validate_logs_dev(int n_logs, const uint64_t* hdr, const int32_t* ev_off, const int32_t* ev_cnt, long long n_hdr,
                          const uint64_t* kyoku, const int32_t* ky_off, long long n_kyoku_words, const uint64_t* hora_payload,
                          const int32_t* hora_off, long long n_hora_words, mjx_verdict* out_verdicts, void* stream);

/* ---- mjai log text -> event words on the device (csrc/mjx_mjai.cuh) -------------------------------------------------------
 * `text`: every log's UTF-8 bytes, concatenated, log i = [log_off[i], log_off[i + 1]) (device arrays, log_off int64 [n_logs + 1]).
 * A log is ACCEPTED when the decoder can show that Python's json reads it as the host path does (the rule is in
 * csrc/mjx_mjai.cuh); an accepted log's arrays equal dataset_codec.encode_events over json.loads of its lines, in the
 * mjx_validate_logs layout above (words, 19-word start_kyoku payloads, MJX_HORA_WORDS-word hora entries), plus the 1-based line
 * number of every event. A DECLINED log is left to the host. `augment` != 0 applies Tile::augment (manzu <-> pinzu) to every
 * tile as it is decoded. Two phases, both enqueued on `stream` without a synchronise:
 *   mjx_mjai_count_dev  -> counts: device mjx_mjai_counts [n_logs] (a declined log: all zero, first_begin = first_end = -1);
 *   mjx_mjai_fill_dev   the arrays of the accepted logs, log i's first word / line at ev_off[i], first payload at ky_off[i], first
 *                       hora entry at hora_off[i] (device int32 [n_logs], typically exclusive sums of the counts copied to host);
 *                       declined logs are skipped, and nothing is written past n_hdr / n_kyoku_words / n_hora_words. */
typedef struct mjx_mjai_counts {
    int32_t accept, n_events, n_kyoku, n_hora;
    int32_t first_begin, first_end;  /* the first event line's bytes, relative to the log's start (start_game: names, seed) */
} mjx_mjai_counts;
int mjx_mjai_count_dev(int n_logs, const uint8_t* text, long long n_bytes, const int64_t* log_off, int augment,
                       mjx_mjai_counts* counts, void* stream);
int mjx_mjai_fill_dev(int n_logs, const uint8_t* text, long long n_bytes, const int64_t* log_off, int augment,
                      const mjx_mjai_counts* counts, const int32_t* ev_off, const int32_t* ky_off, const int32_t* hora_off,
                      uint64_t* hdr, int32_t* lines, long long n_hdr, uint64_t* kyoku, long long n_kyoku_words, uint64_t* hora_payload,
                      long long n_hora_words, void* stream);
/* mjx_mjai_fill_dev plus the per-event deltas array: everything mjx_mjai_fill_dev writes (bit-identical), and for every hora and
 * ryukyoku event at word index e (= ev_off[i] + k):
 *   deltas[4 * e + s] = the event's deltas[s] (int32; 0 when the field is absent or null),
 *   has_deltas[e]     = 1 when `deltas` is present and not null, else 0.
 * Both arrays have the word array's capacity n_hdr (deltas int32 [n_hdr, 4], has_deltas uint8 [n_hdr]); the entries of other
 * events are not written. */
int mjx_mjai_fill_deltas_dev(int n_logs, const uint8_t* text, long long n_bytes, const int64_t* log_off, int augment,
                             const mjx_mjai_counts* counts, const int32_t* ev_off, const int32_t* ky_off, const int32_t* hora_off,
                             uint64_t* hdr, int32_t* lines, long long n_hdr, uint64_t* kyoku, long long n_kyoku_words,
                             uint64_t* hora_payload, long long n_hora_words, int32_t* deltas, uint8_t* has_deltas, void* stream);

/* ---- per-player log statistics: stat.rs:263-442 Stat::from_game (csrc/mjx_stat.cuh) ------------------------------------------
 * The counters of mortal_b200/stat.py Stat, in this order: X(name). This list is the single definition of the order (stat.py
 * reads it); every counter is an int64. */
#define MJX_STAT_COUNTERS(X)                                                                                                    \
    X(game) X(round) X(oya) X(point) X(rank_1) X(rank_2) X(rank_3) X(rank_4) X(tobi)                                             \
    X(agari) X(agari_as_oya) X(agari_jun) X(agari_point_oya) X(agari_point_ko)                                                  \
    X(riichi) X(riichi_as_oya) X(riichi_jun) X(chasing_riichi) X(riichi_got_chased) X(riichi_agari) X(riichi_agari_jun)         \
    X(riichi_agari_point) X(riichi_houjuu) X(riichi_ryukyoku) X(riichi_point)                                                   \
    X(fuuro) X(fuuro_num) X(fuuro_agari) X(fuuro_agari_jun) X(fuuro_agari_point) X(fuuro_houjuu) X(fuuro_point)                 \
    X(dama_agari) X(dama_agari_jun) X(dama_agari_point)                                                                         \
    X(houjuu) X(houjuu_jun) X(houjuu_to_oya) X(houjuu_point_to_oya) X(houjuu_point_to_ko)                                       \
    X(ryukyoku) X(ryukyoku_point) X(yakuman) X(nagashi_mangan)
#define MJX_STAT_ENUM_(name) MJX_S_##name,
enum mjx_stat_counter { MJX_STAT_COUNTERS(MJX_STAT_ENUM_) MJX_STAT_N };
#undef MJX_STAT_ENUM_
/* The per-log status: OK = counted; otherwise the log's counters are all zero and the caller decides (mortal_b200/stat.py reads
 * such a log on the host). NO_DELTAS: a seat is selected and a hora or ryukyoku has no usable deltas; CAPACITY: the log's
 * events or start_kyoku payloads lie outside the arrays. */
enum mjx_stat_status { MJX_STAT_OK = 0, MJX_STAT_NOT_START_GAME = 1, MJX_STAT_NO_DELTAS = 2, MJX_STAT_CAPACITY = 3 };
/* Stat.from_game summed over the selected seats of every log, over the arrays of mjx_mjai_fill_deltas_dev (device pointers):
 * event words hdr [n_hdr] with ev_off / ev_cnt [n_logs]; start_kyoku payloads kyoku [n_kyoku_words] (19 words each, log i's first
 * at ky_off[i]; the scores are words 0-1); deltas / has_deltas [n_hdr] as above; seats uint8 [n_logs] (bit s: take seat s's
 * stats). out: int64 [n_logs, MJX_STAT_N] (`game` counts once per selected seat); status: int32 [n_logs] mjx_stat_status.
 * One warp per log; enqueued on `stream` without a synchronise. Every read is bounded by n_hdr / n_kyoku_words. */
int mjx_stat_logs_dev(int n_logs, const uint64_t* hdr, const int32_t* ev_off, const int32_t* ev_cnt, long long n_hdr,
                      const uint64_t* kyoku, const int32_t* ky_off, long long n_kyoku_words, const int32_t* deltas,
                      const uint8_t* has_deltas, const uint8_t* seats, int64_t* out, int32_t* status, void* stream);

/* ---- GRP targets of a log: dataset/grp.rs:90-164 Grp::load_events (csrc/mjx_grp.cuh) --------------------------------------------
 * The per-log status: OK = the outputs are the log's Grp; otherwise the caller decides (mortal_b200/dataset.py runs the host
 * Grp.load_events on such a log, which raises). NO_DELTAS: a hora or ryukyoku after the last start_kyoku has no usable deltas;
 * NO_KYOKU: the log has no start_kyoku; CAPACITY: the log's events or start_kyoku payloads lie outside the arrays. */
enum mjx_grp_status { MJX_GRP_OK = 0, MJX_GRP_NO_DELTAS = 1, MJX_GRP_NO_KYOKU = 2, MJX_GRP_CAPACITY = 3 };
/* Grp.load_events of every log, over the arrays of mjx_mjai_fill_deltas_dev (device pointers): event words hdr [n_hdr] with
 * ev_off / ev_cnt [n_logs]; start_kyoku payloads kyoku [n_kyoku_words] (19 words each, log i's first at ky_off[i]; the scores are
 * words 0-1); deltas / has_deltas [n_hdr] as above. Outputs:
 *   feat           int32 [n_kyoku_words / 19, 7]: the row of every start_kyoku at its payload index, {grand_kyoku (E1 = 0 .. S4 = 7,
 *                  W and N rounds 7 + kyoku), honba, kyotaku, scores[4]} (the reference's f64 row is these with the scores divided
 *                  by 10000); a log with a non-zero status may have some of its rows written;
 *   rank_by_player uint8 [n_logs, 4] and final_scores int64 [n_logs, 4]: rankings.rs order (stable by seat), the sticks left on the
 *                  table added to the leader; zero where the status is not OK;
 *   status         int32 [n_logs] mjx_grp_status.
 * One warp per log; enqueued on `stream` without a synchronise. Every read is bounded by n_hdr / n_kyoku_words. */
int mjx_grp_logs_dev(int n_logs, const uint64_t* hdr, const int32_t* ev_off, const int32_t* ev_cnt, long long n_hdr,
                     const uint64_t* kyoku, const int32_t* ky_off, long long n_kyoku_words, const int32_t* deltas,
                     const uint8_t* has_deltas, int32_t* feat, uint8_t* rank_by_player, int64_t* final_scores, int32_t* status,
                     void* stream);

/* ---- GRP training rewards: mortal/reward_calculator.py and the targets of mortal/dataloader.py:98-123 (csrc/mjx_reward.cuh) -------
 * The per-job status: OK = the job's outputs are written; CAPACITY: the job's move range, game, player or the game's rank_by_player
 * entry lies outside the arrays (nothing written); KYOKU: an at_kyoku lies outside [0, the game's row count) (the job's outputs are
 * zero; the reference fails its `len(kyoku_rewards) >= at_kyoku[-1] + 1` assertion there). */
enum mjx_reward_status { MJX_REWARD_OK = 0, MJX_REWARD_CAPACITY = 1, MJX_REWARD_KYOKU = 2 };
/* The GRP net (model.py GRP: GRU of `layers` layers with hidden size `hidden`, Linear HL -> HL, ReLU, Linear HL -> 24, softmax,
 * HL = hidden * layers; float64 throughout) over every prefix of every game, then the per-move training targets of every job.
 * Device pointers unless stated.
 *   feat         float64 [n_rows, 7]: the games' kyoku rows (Grp.take_feature()), game g's at rows [game_off[g], game_off[g + 1]);
 *                a game whose offsets are not 0 <= lo <= hi <= n_rows has no rows (nothing written for it, its jobs CAPACITY).
 *   weights      float64 [n_weights]: per layer k rnn.weight_ih_l{k} [3 hidden, k ? hidden : 7], rnn.weight_hh_l{k} [3 hidden,
 *                hidden], rnn.bias_ih_l{k}, rnn.bias_hh_l{k} [3 hidden] (gates r, z, n); then fc.0.weight [HL, HL], fc.0.bias [HL],
 *                fc.2.weight [24, HL], fc.2.bias [24]. 1 <= hidden <= 256, 1 <= layers <= 4, n_weights must match.
 *   matrix       out float64 [n_rows, 4, 4]: row r = calc_matrix of the prefix that ends at row r: [player, rank] = the sum of the
 *                softmax over the permutations of itertools.permutations(range(4)) that give `player` that `rank`.
 * Jobs (n_jobs = 0: the matrix only): job j's moves are [move_off[j], move_off[j + 1]) of n_moves, of game job_game[j] (int32) and
 * seat job_player[j] (uint8); per move at_kyoku int32, apply_gamma and dones uint8; per game rank_by_player uint8 [n_games, 4] and
 * final_scores int64 [n_games, 4]; pts_host: 4 doubles on the host; uniform_init: row 0 of the rank probabilities is 1/4. Per move:
 *   steps_to_done int64  0 where dones, else that of the next move + apply_gamma (the move after a job's last counts as 0);
 *   kyoku_reward  float64 exp_pts[at_kyoku + 1] - exp_pts[at_kyoku], exp_pts[k] = [matrix[rows, player]; one_hot(final
 *                 rank)][k] . pts;
 *   player_rank   int64  the seat's rank in score row at_kyoku + 1 of concat(feature[:, 3:] * 1e4, [final_scores]): seats with
 *                 a higher score plus lower-numbered seats with an equal one;
 *   job_status    int32 [n_jobs] mjx_reward_status.
 * Enqueued on `stream` without a synchronise; every read is bounded by n_rows, n_games and n_moves. */
int mjx_grp_reward_dev(int n_games, const double* feat, const int32_t* game_off, long long n_rows, const double* weights,
                       long long n_weights, int hidden, int layers, double* matrix, int n_jobs, const int32_t* move_off,
                       long long n_moves, const int32_t* job_game, const uint8_t* job_player, const int32_t* at_kyoku,
                       const uint8_t* apply_gamma, const uint8_t* dones, const uint8_t* rank_by_player, const int64_t* final_scores,
                       const double* pts_host, int uniform_init, int64_t* steps_to_done, double* kyoku_reward,
                       int64_t* player_rank, int32_t* job_status, void* stream);

/* ---- GRP training step: mortal/train_grp.py:45-81, 172-186 over model.py:233-286 (csrc/mjx_grp_train.cuh) -------------------
 * The per-sample status: OK; GAME: the sample's job is out of range, its game is not the job's, or the job's game, offsets or step
 * count are out of range; LEN: the prefix length is outside 1..the job's steps. A sample that is not OK contributes nothing. */
enum mjx_grp_train_status { MJX_GRP_TRAIN_OK = 0, MJX_GRP_TRAIN_GAME = 1, MJX_GRP_TRAIN_LEN = 2 };
/* One training step of the GRP (the reference's populate_buffer prefixes, collate's pack_padded_sequence, forward_packed,
 * get_label, F.cross_entropy, loss.backward()) over B = n_samples samples, each the prefix feature[:len] of one game with that
 * game's rank_by_player. Device pointers unless stated; float64 throughout.
 *   feat, game_off, n_rows, n_games   the games' kyoku rows, as mjx_grp_reward_dev takes them (n_rows >= 1);
 *   weights, n_weights, hidden, layers  the packed net, as mjx_grp_reward_dev takes it;
 *   sample_game int32 [B], sample_len int32 [B], rank_by_player int64 [B, 4]: the samples (populate_buffer's (feature[:len],
 *                rank_by_player)); a rank row that is no permutation of 0..3 gets label 0, as get_label leaves it;
 *   jobs         the samples grouped by game: job j steps game job_game[j] (int32 [n_jobs]) for job_steps[j] (int32) steps, the
 *                longest prefix of its samples, at most max_steps (host int); sample b belongs to job sample_job[b] (int32 [B]);
 *                the samples of job j are job_sample[job_sample_off[j] .. job_sample_off[j + 1]) (int32 [n_jobs + 1], [B]).
 *                A (game, len) pair may appear more than once; each appearance counts.
 *   loss, acc    out float64 scalars: F.cross_entropy(logits, labels) (the mean over B) and (argmax == label).mean(), argmax
 *                taking the first maximum;
 *   grad         out float64 [n_weights] in the weights' layout: d loss / d weights, as loss.backward() leaves them; null =
 *                forward only (nothing written there);
 *   sample_status out int32 [B] mjx_grp_train_status;
 *   scratch      at least mjx_grp_train_scratch_bytes(hidden, layers, B, n_jobs, max_steps) bytes, 8-byte aligned.
 * MJX_ERR_ARG for a bad count, shape, weight count, null pointer or short scratch. Enqueued on `stream` without a synchronise;
 * every index read is checked against n_games, n_rows, n_jobs and B. Deterministic: no atomics, fixed reduction orders. */
int mjx_grp_train_dev(int n_games, const double* feat, const int32_t* game_off, long long n_rows, const double* weights,
                      long long n_weights, int hidden, int layers, int n_samples, const int32_t* sample_game, const int32_t* sample_len,
                      const int64_t* rank_by_player, int n_jobs, const int32_t* job_game, const int32_t* job_steps,
                      const int32_t* sample_job, const int32_t* job_sample_off, const int32_t* job_sample, int max_steps, double* loss,
                      double* acc, double* grad, int32_t* sample_status, void* scratch, long long scratch_bytes, void* stream);
/* the scratch bytes of mjx_grp_train_dev; MJX_ERR_ARG unless 1 <= hidden <= 256, 1 <= layers <= 4, 1 <= n_samples <= 2^24,
 * 1 <= n_jobs <= n_samples, 1 <= max_steps <= 65536 */
long long mjx_grp_train_scratch_bytes(int hidden, int layers, int n_samples, int n_jobs, int max_steps);

/* ---- training-buffer observation records (csrc/mjx_obs_pack.cuh, layout: csrc/mjx_obs.cuh make_obs_record) ----------------
 * A lossless fixed-size record per observation of (version 1..4, invisible 0 | 1): one uint64 column mask per row (bit c = the
 * cell is 1.0; zero for a value row), then every value row verbatim as 34 floats, in ascending row order. Value rows: the
 * encoder's (5 / 63 / 73 / 28 in versions 1..4) plus, in version 4, rows 889-890 and 961-1011 of the single-player block; the
 * invisible observation's shanten / 6 rows in versions 2..4. Record bytes: 8,184 / 16,104 / 17,400 / 19,112 (versions 1..4),
 * 1,688 / 2,144 (invisible, version 1 / 2..4); mjx_obs_record_bytes returns them (MJX_ERR_ARG for a bad version).
 *   mjx_obs_pack_dev    obs float32 [n, rows, 34] with sample_pitch floats between samples (>= rows * 34; a slice of a larger
 *                       tensor is read in place) -> records uint8 [n, record_bytes] (8-byte aligned) and status int32 [n]:
 *                       0, or 1 + the first mask row holding a cell whose bits are neither +0.0 nor 1.0 (0.5, -0.0, NaN, 2.0 and
 *                       denormals are refused, never rounded; the record is then not lossless). Value rows are copied bit for bit.
 *   mjx_obs_unpack_dev  records [n_records, record_bytes], idx int64 [n_idx] (repeats allowed) -> out float32 [n_idx, rows, 34]
 *                       (16-byte aligned), out[b] = the observation record idx[b] was packed from; an index outside
 *                       [0, n_records) gives an all-zero observation.
 * Device pointers; enqueued on `stream` without a synchronise. */
int mjx_obs_record_bytes(int version, int invisible);
int mjx_obs_pack_dev(int version, int invisible, long long n, const float* obs, long long sample_pitch, uint8_t* records,
                     int32_t* status, void* stream);
int mjx_obs_unpack_dev(int version, int invisible, const uint8_t* records, long long n_records, const int64_t* idx, long long n_idx,
                       float* out, void* stream);

/* ---- libriichi.state.PlayerState (state/player_state.rs:143-264, state/getter.rs:6-156, state/obs_repr.rs:776-791) ---------
 * A batch of n independent single-seat states: table records in single-seat mode (other seats' hidden tiles are `?` = 37), updated
 * by the same device event handlers self-play uses. `mjx_state_create` returns an mjx_env whose encoder entry points
 * (mjx_env_encode_obs, mjx_env_masks, mjx_env_encode_obs_host ...) work on the rows mjx_state_rows prepares.
 *   mjx_state_update  PlayerState::update (update.rs:24-122): one event per state as a 64-bit word (csrc/mjx_step.cuh log_word;
 *                     mortal_b200/dataset_codec.py encodes mjai JSON), start_kyoku with its 19-word payload (scores + wall, see
 *                     mjx_env_create_replay); word 0 = no event for that state. cans_host[i] = the ActionCandidate of state i
 *                     (action.rs:11-40: bit k = the k-th can_* flag in declaration order, target_actor << 16).
 *   mjx_state_view    every getter of state/getter.rs plus the fields state/test.rs asserts, for one state.
 *   mjx_state_rows    one decision row per state (kan-select rows where at_kan_select_host[i] != 0): row i = state i.
 *   mjx_state_query   what = 0 agent_helper.rs:377-462 agari_points(is_ron = args[0], ura tiles args[2 .. 2 + args[1]))
 *                              -> out = {ron, tsumo_ko, tsumo_oya, ok};  1 rule_based_agari (agent_helper.rs:262-368) -> out[0];
 *                     2 discard_candidates_aka (agent_helper.rs:35-79) -> out[0..1] = 37-bit mask (low, high word);
 *                     3 discard_candidates_with_unconditional_tenpai (agent_helper.rs:88-197) -> 34-bit mask;
 *                     4 agent/mortal.rs:338-573 action id -> reaction: args = {action, kan_select_action or -1}
 *                              -> out[0..1] = the event word (low, high), out[2] = 0 or an error code. */
typedef struct mjx_player_view {
    uint8_t tehai[34], waits[34], dora_factor[34], tiles_seen[34], keep_shanten_discards[34], next_shanten_discards[34],
        forbidden_tiles[34], discarded_tiles[34];
    uint8_t akas_seen[3], akas_in_hand[3];
    uint8_t bakaze, jikaze, kyoku, honba, kyotaku, rank, oya, is_all_last;
    int32_t scores[4];                       /* rotated: [0] = self */
    uint8_t n_dora_indicators, dora_indicators[5];
    uint8_t riichi_declared[4], riichi_accepted[4];  /* relative seats */
    uint8_t at_turn, tiles_left;
    int8_t shanten, real_time_shanten;
    uint8_t has_last_self_tsumo, last_self_tsumo, has_last_kawa_tile, last_kawa_tile;
    uint32_t cans;
    uint8_t n_ankan_candidates, ankan_candidates[3], n_kakan_candidates, kakan_candidates[3];
    uint8_t chankan_chance, can_w_riichi, is_w_riichi, at_rinshan, at_ippatsu, at_furiten, to_mark_same_cycle_furiten,
        kans_on_board, is_menzen;
    uint8_t n_chis, chis[4], n_pons, pons[4], n_minkans, minkans[4], n_ankans, ankans[4];
    uint8_t doras_owned[4], doras_seen, tehai_len_div3, has_next_shanten_discard;
    uint8_t kawa_len[4];
    uint8_t viewer, pad_[3];
    int32_t err;                             /* 0, or the code of the inconsistency the last events produced */
} mjx_player_view;
int mjx_state_create(mjx_env** out, int n, const uint8_t* player_ids_host, int obs_version);
int mjx_state_update(mjx_env* env, const uint64_t* words_host, const uint64_t* payload_host, uint32_t* cans_host);
int mjx_state_view(mjx_env* env, int index, mjx_player_view* out_host);
int mjx_state_rows(mjx_env* env, const uint8_t* at_kan_select_host, void* stream);
int mjx_state_query(mjx_env* env, int index, int what, const int32_t* args, int32_t* out);
int mjx_state_copy(mjx_env* dst, int dst_index, mjx_env* src, int src_index); /* PlayerState: Clone */

/* Instrumentation for bench.py's roofline: when enabled, mjx_env_encode_obs brackets its two encoder kernels with CUDA events
 * on the launch stream; mjx_env_last_encode_ms (blocking) returns the durations of k_encode_features and k_encode_store. */
int mjx_env_set_encode_timing(mjx_env* env, int enable);
int mjx_env_last_encode_ms(mjx_env* env, float* ms_features, float* ms_store);

/* Number of kernels this library has launched for env so far (host-side counter; bench.py's gpu_launches). */
long long mjx_env_launch_count(mjx_env* env);

/* Device views, valid for the lifetime of env (contents valid until the next mjx_env_step). */
int mjx_env_row_cap(mjx_env* env);
uint8_t* mjx_env_masks(mjx_env* env);      /* uint8/bool [row_cap, 46]  (obs_repr.rs mask) */
int32_t* mjx_env_row_table(mjx_env* env);  /* int32 [row_cap] table index of each row */
uint8_t* mjx_env_row_seat(mjx_env* env);   /* uint8 [row_cap] seat | (kan_select << 2) */
uint32_t* mjx_env_row_step(mjx_env* env); /* uint32 [row_cap] table-step index of the table when the row was emitted */
int32_t* mjx_env_num_rows_dev(mjx_env* env); /* int32 [1] */

/* arena/result.rs GameResult.scores + rankings.rs rank_by_player, plus per-table step counts and
 * error codes (0 = clean; the reference would have raised/panicked otherwise). Host outputs. */
int mjx_env_results(mjx_env* env, void* stream, int32_t* scores_host /*[n,4]*/, uint8_t* ranks_host /*[n,4]*/,
                    int32_t* steps_host /*[n]*/, int32_t* err_host /*[n]*/, int32_t* done_host /*[n]*/);

/* Counter-based TEST policy (not in the reference; shared definition with the oracle) writing
 * int64 actions for the current rows. kind 0 uniform, 1 agari-first/shanten-greedy.
 * trace_dev (optional): int64 [row_cap, 6] = table, step, seat, action, kan_select, mask_bits.
 * q_values_dev (optional): float32 [row_cap, 46] filled with 0 on legal and -inf on illegal actions. */
int mjx_env_policy_test(mjx_env* env, int kind, int64_t* actions_dev, int64_t* trace_dev, float* q_values_dev,
                        void* stream);

/* ---- policy-net inference helpers (not part of libriichi's surface; mortal/model.py ResBlock + ChannelAttention) ------------
 * Fused elementwise passes between the cuDNN convolutions: bf16 channels-last activations [batch, length, channels]
 * (device pointers, 16-byte aligned, channels % 8 == 0), fp32 math. scale/bias = eval-mode BatchNorm folded to an affine.
 * Every array pointer (activations, gate, scale / bias, w1 / b1 / w2t / b2) must be 16-byte aligned; a misaligned one fails the
 * call with MJX_ERR_ARG before anything is launched (obs_to_nhwc: `out` 16-byte, `obs` float aligned). */
int mjx_nn_affine_mish_bf16(const void* x, const float* scale, const float* bias, void* out, long long n_elems, int channels,
                            void* stream);                                   /* out = mish(x * scale[c] + bias[c]) */
int mjx_nn_pool_bf16(const void* x, void* avg, void* mx, int batch, int length, int channels, void* stream);  /* [batch, channels] each */
int mjx_nn_gate_residual_bf16(const void* y, const void* gate, const void* x, void* out, int batch, int length, int channels,
                              void* stream);                                 /* out = y * gate[b, c] + x */
/* observations f32 [batch, channels, length] -> bf16 channels-last [batch, length, channels_padded], padded channels zero
 * (channels_padded % 64 == 0): the input of the stem convolution. */
int mjx_nn_obs_to_nhwc_bf16(const float* obs, void* out, int batch, int channels, int length, int channels_padded, void* stream);
/* The tail of a residual block and the next pre-activation in one pass (model.py ChannelAttention + residual; next BN + Mish):
 * gate = sigmoid(mlp(mean_l y) + mlp(max_l y)), mlp = w2 . mish(w1 [hidden, channels] . v + b1) + b2, w2 passed TRANSPOSED as w2t
 * [hidden, channels] (fp32 device
 * arrays); x_out = y * gate + x; a_out = mish(x_out * scale[c] + bias[c]). Two launches: one warp per batch row computes the gate,
 * one streaming pass applies it. channels % 8 == 0, <= 256. */
int mjx_nn_block_tail_bf16(const void* y, const void* x, const float* w1, const float* b1, const float* w2t, const float* b2,
                           const float* scale, const float* bias, void* gate_scratch /* bf16 [batch, channels] */, void* x_out,
                           void* a_out, int batch, int length, int channels, int hidden, void* stream);

/* Version 1 (post-activation ResNet, mortal/model.py ResBlock with pre_actv=False) and oracle brains:
 * out = relu(x * scale[c] + bias[c]): the stem's BatchNorm + ReLU and each block's first BatchNorm + ReLU. */
int mjx_nn_affine_relu_bf16(const void* x, const float* scale, const float* bias, void* out, long long n_elems, int channels,
                            void* stream);
/* The post-activation block's tail, y = conv2 output: t = y * scale[c] + bias[c] (the block's second BatchNorm, fp32);
 * gate = sigmoid(mlp(mean_l t) + mlp(max_l t)), mlp = w2 . relu(w1 . v + b1) + b2 (w2 TRANSPOSED as w2t [hidden, channels]);
 * x_out = relu(t * gate + x). Two launches, as mjx_nn_block_tail_bf16. channels % 8 == 0, <= 256; hidden <= 64. */
int mjx_nn_post_block_tail_bf16(const void* y, const void* x, const float* scale, const float* bias, const float* w1, const float* b1,
                                const float* w2t, const float* b2, void* gate_scratch /* bf16 [batch, channels] */, void* x_out,
                                int batch, int length, int channels, int hidden, void* stream);
/* The oracle stem input: obs f32 [batch, channels, length] and obs2 (the invisible observation) f32 [batch, channels2, length] ->
 * bf16 channels-last [batch, length, channels_padded]: channels [0, channels) from obs, then channels2 from obs2, then zeros
 * (channels_padded % 64 == 0, >= channels + channels2). obs / obs2 float aligned, out 16-byte aligned. */
int mjx_nn_obs2_to_nhwc_bf16(const float* obs, const float* obs2, void* out, int batch, int channels, int channels2, int length,
                             int channels_padded, void* stream);

/* ---- policy-net training (mortal/train.py:228-248; csrc/mjx_train.cuh) ------------------------------------------------------
 * Activations are channels-last [batch, length, channels] (rows = batch * length), stored as `dtype` MJX_TRAIN_F32 or
 * MJX_TRAIN_F16, fp32 arithmetic; 1 <= channels <= 256 with channels % 8 == 0, batch >= 1. Per-channel vectors (gamma, beta,
 * running stats, mean / invstd, dgamma / dbeta) are float32. Reductions run in an order fixed by the shape: equal inputs give
 * bit-identical outputs. Non-finite values pass through unclamped. MJX_ERR_ARG for a bad dtype, shape or null pointer. */
enum mjx_train_dtype { MJX_TRAIN_F32 = 0, MJX_TRAIN_F16 = 1 };
/* float32 elements of the scratch the two BatchNorm calls need for `rows` x `channels` */
long long mjx_train_bn_scratch_floats(int rows, int channels);
/* out = mish(gamma (x - mean) invstd + beta). training != 0: mean / biased variance of the batch (per-block shifted sums merged
 * as (count, mean, M2) in double), running_mean / running_var updated with `momentum` (running_var from the unbiased variance),
 * save_mean / save_invstd written; training == 0: the running statistics are used and left untouched (save_* still written).
 * save_mean is float32 [2 * channels], the mean as a pair hi [0, channels) + lo [channels, 2 * channels); save_invstd
 * float32 [channels]. */
int mjx_train_bn_mish_fwd(int dtype, const void* x, const float* gamma, const float* beta, float* running_mean, float* running_var,
                          float* save_mean, float* save_invstd, void* out, int rows, int channels, float eps, float momentum,
                          int training, float* scratch, void* stream);
/* the backward of mjx_train_bn_mish_fwd from its x, save_mean and save_invstd: dx, dgamma = sum dz xhat, dbeta = sum dz,
 * dz = dout mish'(u); training == 0 gives the backward of the affine map (frozen BatchNorm). */
int mjx_train_bn_mish_bwd(int dtype, const void* x, const void* dout, const float* gamma, const float* beta, const float* save_mean,
                          const float* save_invstd, void* dx, float* dgamma, float* dbeta, int rows, int channels, int training,
                          float* scratch, void* stream);
/* the channel gate: avg / mx [batch, channels] = mean / max over length of y */
int mjx_train_gate_pool(int dtype, const void* y, void* avg, void* mx, int batch, int length, int channels, void* stream);
/* out = y * g[b, c] + x, g [batch, channels] */
int mjx_train_gate_out(int dtype, const void* y, const void* g, const void* x, void* out, int batch, int length, int channels,
                       void* stream);
/* dg float32 [batch, channels] = sum_l dout y; cnt float32 [batch, channels] = the number of l with y == mx */
int mjx_train_gate_bwd_dg(int dtype, const void* dout, const void* y, const void* mx, float* dg, float* cnt, int batch, int length,
                          int channels, void* stream);
/* dy = dout g + davg / length + (y == mx ? dmx / cnt : 0) */
int mjx_train_gate_bwd_dy(int dtype, const void* dout, const void* y, const void* g, const void* mx, const float* cnt,
                          const void* davg, const void* dmx, void* dy, int batch, int length, int channels, void* stream);
/* The dueling combine and the three losses of one batch in one launch. v [batch], a [batch, 46], aux [batch, n_aux] (dtype),
 * masks uint8 [batch, 46], actions / steps_to_done / ranks int64 [batch], rewards float64 [batch]. Writes q_out float32
 * [batch, 46] (optional: NULL skips it), q_act / q_target float32 [batch], losses float32 [3] = (0.5 mse, mean lse - mean q,
 * cross-entropy), and ORs 1 into *bad when an action is outside its mask. 1 <= n_aux <= 32. */
int mjx_train_dqn_loss_fwd(int dtype, const void* v, const void* a, const uint8_t* masks, const int64_t* actions,
                           const int64_t* steps_to_done, const double* rewards, const void* aux, const int64_t* ranks, int batch,
                           int n_aux, float gamma, float* q_out, float* q_act, float* q_target, float* losses, int* bad, void* stream);
/* gradients of w[0] dqn + w[1] cql + w[2] next_rank (w float32 [3], device) for v, a and aux, from q_target of the forward */
int mjx_train_dqn_loss_bwd(int dtype, const void* v, const void* a, const uint8_t* masks, const int64_t* actions,
                           const float* q_target, const void* aux, const int64_t* ranks, int batch, int n_aux, const float* w,
                           void* dv, void* da, void* daux, void* stream);

/* ---- standalone kernels (BASELINE configs 3/4) ------------------------------------------------ */
/* algo/shanten.rs:138-150 calc_all: tiles_dev uint8 [n,34], len_div3_dev uint8 [n] -> int8 [n]. */
int mjx_shanten(const uint8_t* tiles_dev, const uint8_t* len_div3_dev, int8_t* out_dev, int n, void* stream);

typedef struct mjx_agari_in {  /* algo/agari.rs:77-101 AgariCalculator */
    uint8_t tehai[34];
    uint8_t chis[4], pons[4], minkans[4], ankans[4];
    uint8_t n_chis, n_pons, n_minkans, n_ankans;
    uint8_t bakaze, jikaze, winning_tile, is_ron;
    uint8_t additional_hans, doras; /* for mode 1 = agari(additional_hans, doras) */
    uint8_t is_oya, pad;
} mjx_agari_in;
typedef struct mjx_agari_out { /* algo/agari.rs:66-74 Agari + algo/point.rs Point */
    uint8_t kind; /* 0 none, 1 normal, 2 yakuman */
    uint8_t fu, han, yakuman;
    int32_t ron, tsumo_ko, tsumo_oya; /* -1 where point.rs would panic */
} mjx_agari_out;
/* mode 0 = search_yakus (agari.rs:212), 1 = agari (agari.rs:225), 2 = has_yaku (agari.rs:206),
 * 3 = check_ankan_after_riichi(tehai, len_div3 = additional_hans, tile = winning_tile, strict = false) (agari.rs:854-912;
 *     the call state/update.rs:278 makes): out.kind = 1 when the kan is allowed */
int mjx_agari(const mjx_agari_in* in_dev, mjx_agari_out* out_dev, int n, int mode, void* stream);

/* Host-buffer conveniences (H2D + kernel + D2H), the shape a foreign-language binding would call. */
int mjx_shanten_host(const uint8_t* tiles, const uint8_t* len_div3, int8_t* out, int n);
int mjx_agari_host(const mjx_agari_in* in, mjx_agari_out* out, int n, int mode);

/* arena/board.rs:99-123 wall for one (seed, kyoku, honba): uint8 [136] (host out; runs on device). */
int mjx_make_wall_host(uint64_t nonce, uint64_t key, int kyoku, int honba, int shuffle_kind, uint8_t* wall136);

#ifdef __cplusplus
}
#endif
#endif /* MJX_H */
