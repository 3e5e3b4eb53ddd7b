/* elfb200.h -- C ABI of libelfb200.so: the H100-native (sm_90a) replacement for the
 * data-parallel hot path of ELF OpenGo (pytorch/ELF).
 *
 * Boundary (SURVEY.md 8b): the reference reaches this path through C++ objects
 * (GoState, BoardFeature, TreeSearchT) owned by per-game threads.  Here the same
 * operations act on a BATCH of G games that live in GPU memory; every entry point
 * below names the reference interface it replaces.  Signatures use only plain
 * pointers and sizes.  "host" pointers are ordinary (ideally pinned) host memory;
 * "dev" pointers are CUDA device memory of the context's device.  Unless noted the
 * call is synchronous with respect to the host buffers it is given.
 *
 * Conventions (reference src_cpp/elfgames/go/base): action a = x*N + y (board.h:189),
 * pass = N*N (go_common.h:11); colours 0 empty / 1 black / 2 white (common.h:37-40);
 * feature planes float32 [18][N][N] (board_feature.cc:247-290).
 *
 * All functions return 0 on success and a negative code on failure; the message is
 * available from elfb200_last_error().  There is NO CPU fallback: without a CUDA
 * device every call fails.
 */
#ifndef ELFB200_H_
#define ELFB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ELFB200_OK 0
#define ELFB200_ERR_ARG (-1)
#define ELFB200_ERR_CUDA (-2)
#define ELFB200_ERR_STATE (-3)

#define ELFB200_INFO_FIELDS 12 /* see elfb200_get_info */

typedef struct elfb200_ctx elfb200_ctx;

const char* elfb200_last_error(void);
const char* elfb200_version(void);

/* Create a batch of `num_games` boards of size 9 or 19 on CUDA device `device`, all in the
 * initial position.  Replaces: N x `GoState()` / GoState::reset (go_state.cc:134-141,
 * clearBoard board.cc:79-107). */
int elfb200_create(int board_size, int num_games, int device, elfb200_ctx** out);
void elfb200_destroy(elfb200_ctx* ctx);
int elfb200_num_games(const elfb200_ctx* ctx);
int elfb200_board_size(const elfb200_ctx* ctx);
/* CUDA stream (cudaStream_t) all work of this context is issued on. */
void* elfb200_stream(const elfb200_ctx* ctx);
int elfb200_synchronize(elfb200_ctx* ctx);

/* GoState::reset for the games with mask[g] != 0 (all games if mask == NULL). */
int elfb200_reset(elfb200_ctx* ctx, const uint8_t* mask_host);

/* GoState::forward (go_state.cc:74-94) for every game: actions[g] in [0, N*N] is tried,
 * actions[g] < 0 leaves game g untouched.  ok[g] = 1 iff the move was accepted (not
 * terminated, legal per TryPlay board.cc:788-827).  `ok_host` may be NULL. */
int elfb200_step(elfb200_ctx* ctx, const int32_t* actions_host, uint8_t* ok_host);
/* Same with device buffers, asynchronous on the context stream. */
int elfb200_step_dev(elfb200_ctx* ctx, const int32_t* actions_dev, uint8_t* ok_dev);
/* One ply of a device-resident environment, asynchronous on the context stream, no host copies and no
 * synchronisation (capturable in a CUDA graph on elfb200_stream).  GoState::forward(actions[g]) for
 * every game (actions < 0: untouched), then for every game that has ended (GoState::terminated: two
 * passes, positional superko or the 2*N*N ply cap, also a game that had ended before the call):
 * done[g] = 1, value[g] = GoState::evaluate(komi) (black's view; go_state.h:194-203; 0 where not done)
 * and the game is restarted (GoState::reset).  ok[g] is forward's verdict.  legal uint8[G][N*N+1] /
 * info int32[G][12] describe the positions now to move, as elfb200_get_legal / elfb200_get_info.
 * Every output is a device pointer and may be NULL. */
int elfb200_env_step(elfb200_ctx* ctx, const int32_t* actions_dev, float komi, uint8_t* ok_dev,
                     uint8_t* done_dev, float* value_dev, uint8_t* legal_dev, int32_t* info_dev);
/* GoState::reset for games with mask_dev[g] != 0 (all games if mask_dev == NULL), asynchronous on the
 * context stream. */
int elfb200_reset_dev(elfb200_ctx* ctx, const uint8_t* mask_dev);
/* legal / info of the stored positions into device buffers (each may be NULL), asynchronous: the first
 * observation after elfb200_reset or elfb200_place_handicap. */
int elfb200_observe_dev(elfb200_ctx* ctx, uint8_t* legal_dev, int32_t* info_dev);
/* GoStateExtOffline::switchBeforeMove (common/go_state_ext.h:305-312), the replay step of the
 * training loop (train/game_train.cc:22-45), for every game in ONE launch: game g is reset and
 * moves_host[g*stride + 0 .. count_host[g]) are forwarded in order (int16 actions x*N+y, N*N =
 * pass).  A move GoState::forward refuses is skipped and the list goes on -- the reference ignores
 * forward()'s verdict there.  1 <= stride <= 2*N*N, 0 <= count[g] <= stride.  Synchronous. */
int elfb200_replay(elfb200_ctx* ctx, const int16_t* moves_host, int stride, const int32_t* count_host);
/* GoState::applyHandicap / PlaceHandicap (go_state.cc:62-71,130-132; board.cc:109-126) for every game in
 * ONE launch: game g places BLACK stones stones_host[g*stride + 0 .. count_host[g]) in order (int16 actions
 * x*N+y), each exactly as PlaceHandicap does.  ok_host uint8[G][stride] (may be NULL): PlaceHandicap's
 * return value per stone.  1 <= stride <= N*N, 0 <= count[g] <= stride, actions in [0, N*N).  Synchronous. */
int elfb200_place_handicap(elfb200_ctx* ctx, const int16_t* stones_host, int stride,
                           const int32_t* count_host, uint8_t* ok_host);
/* GoState's copy constructor (go_state.h:117-124; copyBoard board.cc:128-132) from one batch into another:
 * dst game i := src game index[i] for index[i] in [0, G_src); other values leave game i untouched.
 * index has G_dst entries.  Same board size and device; dst != src.  The _dev form is asynchronous on dst's
 * stream and orders itself after the work already on src's stream, and src's later work after itself;
 * capturable when both streams are part of the capture.  The host form is synchronous.  A search handle on
 * dst keeps its trees: reset the copied games' trees (elfb200_mcts_reset) before their next search. */
int elfb200_gather_games(elfb200_ctx* dst, const elfb200_ctx* src, const int32_t* index_host);
int elfb200_gather_games_dev(elfb200_ctx* dst, const elfb200_ctx* src, const int32_t* index_dev);

/* Board hash, GoState::getHashCode (go_state.h:170; set_color board.cc:38-51). uint64[G]. */
int elfb200_get_hash(elfb200_ctx* ctx, uint64_t* hash_host);
/* int32[G][12]: ply, next_player, b_cap, w_cap, last_move(action|-1), last_move2,
 * ko_action(-1 if no active simple ko), ko_color, reserved(0), terminated, two_pass, superko.
 * Replaces GoState::getPly/nextPlayer/lastMove/terminated/isTwoPass + Board fields. */
int elfb200_get_info(elfb200_ctx* ctx, int32_t* info_host);
/* uint8[G][N*N] colours by action index. */
int elfb200_get_stones(elfb200_ctx* ctx, uint8_t* stones_host);
/* uint8[G][N*N+1]: GoState::checkMove (go_state.cc:123-128) of every action for the side to
 * move == FindAllValidMoves (board.cc:949-968); entry N*N (pass) is always 1. */
int elfb200_get_legal(elfb200_ctx* ctx, uint8_t* legal_host);
/* uint8[G][N*N]: isTrueEye (board.cc:1908) of `player` (1/2; 0 = side to move). */
int elfb200_get_true_eyes(elfb200_ctx* ctx, int player, uint8_t* eyes_host);
/* int32[G]: simple_tt_scoring (go_state.h:75-93), black minus white, no komi. */
int elfb200_get_tt_score(elfb200_ctx* ctx, int32_t* score_host);
/* float[G]: GoState::evaluate(komi) (go_state.h:194-203). */
int elfb200_evaluate(elfb200_ctx* ctx, float komi, float* value_host);

/* BoardFeature::extractAGZ (board_feature.cc:247-290) for every game under D4 code
 * d4[g] (board_feature.h:88-95; NULL = identity): float32 [G][18][N][N]. */
int elfb200_features(elfb200_ctx* ctx, const int32_t* d4_host, float* out_host);
int elfb200_features_dev(elfb200_ctx* ctx, const int32_t* d4_dev, float* out_dev);
/* BoardFeature::extract (board_feature.cc:209-237), the 25-plane DarkForest feature set selected by
 * GameOptions::use_df_feature (common/game_feature.h:22-33): float32 [G][25][N][N] under D4 code d4[g]
 * (NULL = identity).  Planes as in board_feature.h:19-36. */
int elfb200_features_df(elfb200_ctx* ctx, const int32_t* d4_host, float* out_host);
int elfb200_features_df_dev(elfb200_ctx* ctx, const int32_t* d4_dev, float* out_dev);

/* Feature formats.  ELFB200_FEAT_F32_NCHW is the GoFeature tensor contract "s"
 * (common/game_feature.h:159-206).  The 16-bit channels-last formats are a fast mode for a network
 * that runs in half precision: [n][N][N][cpad] halves (binary16 / bfloat16), planes 0..17 in
 * channels 0..17, zeros above; cpad = 24 or 32.  Values are exactly 0 or 1 in every format. */
#define ELFB200_FEAT_F32_NCHW 0
#define ELFB200_FEAT_F16_NHWC 1
#define ELFB200_FEAT_BF16_NHWC 2
/* elfb200_features_dev with an explicit format.  out_dev: 16-byte aligned (float32: 8-byte aligned
 * is accepted, e.g. an odd row of a larger tensor, at the price of narrower stores). */
int elfb200_features_dev_ex(elfb200_ctx* ctx, const int32_t* d4_dev, void* out_dev, int format, int cpad);
/* How the 16-bit NHWC planes are written: 0 = direct coalesced 16-byte vector stores (default; measured
 * 0.74 of the HBM copy peak), 1 = the position staged in shared memory and stored by one bulk (TMA,
 * cp.async.bulk) instruction (0.60).  Same bytes either way; the float32 format always uses 16-byte
 * vector stores.  A tuning/diagnostic knob. */
int elfb200_set_feature_store(elfb200_ctx* ctx, int mode);

/* The deterministic random-playout workload (include/elfb200_playout_policy.h; BASELINE
 * configs 1/2/5): game g plays game id first_game_id+g from the empty board until
 * GoState::terminated() (or max_plies), entirely on the GPU.  Outputs (host, each may be
 * NULL): chk uint64[G] position checksum, plies int32[G], score int32[G] (tt score of the
 * final position), final_hash uint64[G].  Does not touch the context's stored games.
 * Returns the total number of plies in *total_plies (may be NULL). */
int elfb200_playout(elfb200_ctx* ctx, uint64_t seed, uint64_t first_game_id, int max_plies,
                    uint64_t* chk_host, int32_t* plies_host, int32_t* score_host,
                    uint64_t* final_hash_host, int64_t* total_plies);
/* Device-resident variant: launches the playout kernel on the context stream and returns
 * immediately; results stay in context-owned device buffers readable with
 * elfb200_playout_results().  Used to time the kernel with CUDA events. */
int elfb200_playout_launch(elfb200_ctx* ctx, uint64_t seed, uint64_t first_game_id, int max_plies);
int elfb200_playout_results(elfb200_ctx* ctx, uint64_t* chk_host, int32_t* plies_host,
                            int32_t* score_host, uint64_t* final_hash_host, int64_t* total_plies);

/* Steady-state variant ("G concurrent games"): every one of the G slots plays exactly
 * plies_per_slot plies, starting its next game (id += G) whenever a game reaches
 * GoState::terminated(), as the reference's game threads do (common/game_base.h:41).  Outputs per
 * slot: chk = fold of the slot's game checksums in order, plies (= plies_per_slot), games = number
 * of games started, last_hash.  elfb200_playout_results() returns the same arrays after
 * elfb200_playout_stream_launch(). */
int elfb200_playout_stream(elfb200_ctx* ctx, uint64_t seed, uint64_t first_game_id, int plies_per_slot,
                           uint64_t* chk_host, int32_t* plies_host, int32_t* games_host,
                           uint64_t* last_hash_host, int64_t* total_plies);
int elfb200_playout_stream_launch(elfb200_ctx* ctx, uint64_t seed, uint64_t first_game_id, int plies_per_slot);

/* Lane layout of the playout kernel: 0 = one board row per lane (one 19x19 game per warp), 1 = two rows
 * per lane (three 19x19 games per warp; 19x19 only), -1 = automatic (default): two rows per lane from
 * 4096 games up, where it measures faster on an H100 SXM at 700 W (0.99 vs 0.87 G moves/s at 4096 games,
 * 1.35 vs 1.00 G at 12,288), one row per lane below.  Same results either way. */
int elfb200_set_playout_layout(elfb200_ctx* ctx, int layout);

/* Monte-Carlo ownership of the stored positions: for every game g, `playouts` (K) random playouts of the policy
 * of include/elfb200_playout_policy.h start from g's position (playout k uses draw id g*K + k), each played with
 * GoState::forward on a copy of g's GoState (go_state.h:117-124) until GoState::terminated() -- superko against
 * g's record and the playout's own moves -- or `max_plies` moves (>= 0).  A game that ended by
 * two passes is played on with an empty last-move window (Board::_last_move/_last_move2); one that ended by
 * superko or the ply cap plays no move.  counts int32[G][2][N*N] (zeroed by the call), by action x*N+y: the
 * playouts whose final position has the point in black's [0] / white's [1] area as simple_tt_scoring
 * (go_state.h:75-93) sees it.  Integer sums: bit-for-bit the same for a seed.  The stored games are not changed.
 * final_hash uint64[G][K] and plies int32[G][K] (each may be NULL): every playout's final GoState::getHashCode
 * and moves played.  Synchronous.  G*K <= INT32_MAX. */
int elfb200_ownership(elfb200_ctx* ctx, int playouts, uint64_t seed, int max_plies, int32_t* counts_host,
                      uint64_t* final_hash_host, int32_t* plies_host);
/* The same counts into device memory, asynchronous on the context stream and capturable once a first call has
 * allocated the per-warp superko scratch (the same board size and at least as many playouts in all). */
int elfb200_ownership_dev(elfb200_ctx* ctx, int playouts, uint64_t seed, int max_plies, int32_t* counts_dev);
/* getTrompTaylorScore(board, group_stats, territory) (board.cc:1954-2071, board.h:431-445) of every stored position
 * with the groups this call finds dead flagged S_DEAD in group_stats.  Dead (a heuristic, not the reference's: it
 * leaves the choice to its caller): with the counts of elfb200_ownership over `playouts` (K) playouts, a group S of
 * colour c is dead iff sum over S of (own area count - opponent area count) < -threshold * K * |S|; with
 * counts_host == NULL no group is dead.  dead uint8[G][N*N] (1 on every stone of a dead group), territory
 * uint8[G][N*N] (1 black, 2 white, 3 dame; stones of dead groups count for the opponent), score int32[G] (black
 * minus white, no komi; simple_tt_scoring when no group is dead).  Outputs may be NULL.  Synchronous. */
int elfb200_final_status(elfb200_ctx* ctx, const int32_t* counts_host, int playouts, double threshold,
                         uint8_t* dead_host, uint8_t* territory_host, int32_t* score_host);

/* Number of kernels this library has launched since creation (bench gpu_launches).  Counts enqueues by
 * the calls above; replays of a CUDA graph that captured them are not counted. */
int64_t elfb200_launch_count(const elfb200_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* ELFB200_H_ */
