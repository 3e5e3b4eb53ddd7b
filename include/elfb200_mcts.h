/* elfb200_mcts.h -- C ABI of the batched GPU tree search in libelfb200.so.
 *
 * Replaces, for all G games of an elfb200_ctx at once, the reference's per-game search objects
 *   elf::ai::tree_search::MCTSAI_T / TreeSearchT / SearchTreeT / NodeT / EdgeInfo
 *     (src_cpp/elf/ai/tree_search/{mcts.h,tree_search.h,tree_search_node.h,tree_search_base.h})
 *   MCTSActor / MCTSGoAI (src_cpp/elfgames/go/mcts/mcts.h)
 * The network stays outside: the caller (the rlpytorch model-interface callback in the
 * reference, src_py/rlpytorch/trainer/trainer.py:73-115) is handed the leaf feature batch
 * "s" float32 [n][18][N][N] in device memory and hands back "pi" float32 [n][N*N+1] and "V"
 * float32 [n] (GoFeature tensor contract, src_cpp/elfgames/go/common/game_feature.h:159-206).
 *
 * One move of all games (== MCTSAI_T::act, elf/ai/tree_search/mcts.h:59-81):
 *     elfb200_mcts_begin_move(m, active)
 *     repeat elfb200_mcts_waves_per_move(m) times:          // TreeSearchSingleThreadT::run
 *         elfb200_mcts_select(m, feat_dev, &n)              //   batch_rollouts: descents + leaf claim
 *         pi, V = net(feat_dev[:n])                         //   actor.evaluate -> the NN
 *         elfb200_mcts_expand_backup(m, pi_dev, v_dev)      //   setEvaluation + updateEdgeStats
 *     elfb200_mcts_results(m, ...)                          // chooseAction (most_visited)
 *     elfb200_step(ctx, actions, ...)                       // GoState::forward
 *     elfb200_mcts_advance(m, actions)                      // SearchTreeT::treeAdvance
 *
 * Search semantics are those of ONE reference search thread (num_threads = 1) with
 * num_rollouts_per_batch descents per wave; batching comes from the G games instead of from
 * threads.  All functions return 0 or a negative ELFB200_ERR_* code (see elfb200.h).
 */
#ifndef ELFB200_MCTS_H_
#define ELFB200_MCTS_H_

#include <stdint.h>

#include "elfb200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct elfb200_mcts elfb200_mcts;

/* TSOptions + SearchAlgoOptions (tree_search_options.h:22-111) and MCTSActorParams
 * (go/mcts/mcts.h:17-27).  Field names follow the reference. */
typedef struct {
  int32_t num_rollouts;            /* TSOptions::num_rollouts_per_thread */
  int32_t num_rollouts_per_batch;  /* TSOptions::num_rollouts_per_batch */
  int32_t virtual_loss;            /* TSOptions::virtual_loss */
  int32_t persistent_tree;         /* TSOptions::persistent_tree */
  int32_t use_prior;               /* SearchAlgoOptions::use_prior */
  int32_t unexplored_q_zero;       /* SearchAlgoOptions::unexplored_q_zero */
  int32_t root_unexplored_q_zero;  /* SearchAlgoOptions::root_unexplored_q_zero */
  int32_t ply_pass_enabled;        /* MCTSActorParams::ply_pass_enabled */
  int32_t remove_pass_if_dangerous;/* MCTSActorParams::remove_pass_if_dangerous */
  int32_t rotation_flip;           /* MCTSActorParams::rotation_flip: random D4 per evaluation (default 1).
                                    * The planes of each leaf are written under its D4 code and the returned
                                    * pi is read back through the inverse, exactly as the reference does, so a
                                    * network sees nothing unusual.  A callback that computes pi from the leaf
                                    * HASH instead of the planes (test nets) must set 0 or permute through
                                    * elfb200_mcts_leaf_info's d4 output. */
  int32_t seed;
  int32_t nodes_per_game;          /* node-pool slots per game; 0 = 2*rollouts + 256 */
  float c_puct;                    /* SearchAlgoOptions::c_puct */
  float komi;                      /* MCTSActorParams::komi */
  float root_epsilon;              /* TSOptions::root_epsilon: Dirichlet noise weight at the root (0 = off) */
  float root_alpha;                /* TSOptions::root_alpha */
  int32_t std_sort_ties;           /* moves with bit-EQUAL network probabilities: 0 (default) = stored by ascending
                                    * move index; 1 = in the order libstdc++'s std::sort leaves them in
                                    * MCTSActor::pi2response (go/mcts/mcts.h:289-295), which is what the reference's
                                    * edge containers -- and every tie-break that walks them -- then see.  Needed to
                                    * replay the reference's games bit for bit with half-precision networks (equal
                                    * fp16 logits are the norm); costs a sequential sort per leaf that has such a tie. */
} elfb200_mcts_options;

int elfb200_mcts_default_options(elfb200_mcts_options* opt);
int elfb200_mcts_create(elfb200_ctx* ctx, const elfb200_mcts_options* opt, elfb200_mcts** out);
void elfb200_mcts_destroy(elfb200_mcts* m);

int elfb200_mcts_waves_per_move(const elfb200_mcts* m);  /* ceil(num_rollouts / per_batch) */
int elfb200_mcts_max_leaves(const elfb200_mcts* m);      /* G * num_rollouts_per_batch */
int elfb200_mcts_nodes_per_game(const elfb200_mcts* m);

/* MCTSAI_T::endGame / resetTree (mcts.h:90-93,134-137) for games with mask[g] != 0 (all if NULL). */
int elfb200_mcts_reset(elfb200_mcts* m, const uint8_t* mask_host);
/* Search prologue: root allocation + root-state check (tree_search.h:478-493).  active[g] == 0
 * excludes a game from this move (NULL = all active). */
int elfb200_mcts_begin_move(elfb200_mcts* m, const uint8_t* active_host);
/* One wave of descents.  Writes the feature planes of the *n_leaves leaves that need the network
 * to feat_dev (device, capacity elfb200_mcts_max_leaves * 18*N*N floats). */
int elfb200_mcts_select(elfb200_mcts* m, float* feat_dev, int32_t* n_leaves);
/* elfb200_mcts_select with an explicit feature format (ELFB200_FEAT_*, elfb200.h): the 16-bit
 * channels-last formats let a half-precision network read the leaf batch without a cast/permute
 * pass; ELFB200_FEAT_DF_F32_NCHW writes the 25 DarkForest planes (GameOptions::use_df_feature) of every
 * leaf instead of the 18 AGZ planes.  feat_dev: 16-byte aligned, capacity elfb200_mcts_max_leaves
 * positions (DarkForest: max_leaves * 25*N*N floats).
 * n_leaves == NULL selects the ASYNCHRONOUS mode: nothing is copied back and the host does not
 * wait; the feature and expansion kernels run on a grid for all G*B slots and stop at the
 * device-side count, so the caller evaluates all elfb200_mcts_max_leaves rows (rows past the count
 * are stale and ignored) or asks for the count later with elfb200_mcts_leaf_count. */
int elfb200_mcts_select_ex(elfb200_mcts* m, void* feat_dev, int format, int cpad, int32_t* n_leaves);
/* The planes of the leaves claimed by the last select once more, into feat_dev in the given format
 * (idempotent: e.g. the float32 contract tensor next to a 16-bit batch, or for timing).
 * Asynchronous on the context stream. */
int elfb200_mcts_leaf_features(elfb200_mcts* m, void* feat_dev, int format, int cpad);
/* Number of leaves the last select claimed (waits for the context stream). */
int elfb200_mcts_leaf_count(elfb200_mcts* m, int32_t* n_leaves);
/* Hash / game index / ply / D4 code of the pending leaves (host, each may be NULL); test & debug aid. */
int elfb200_mcts_leaf_info(elfb200_mcts* m, uint64_t* hash_host, int32_t* game_host, int32_t* ply_host,
                           int32_t* d4_host);
/* Network reply for the pending leaves (device pointers, same order as feat_dev), then backup. */
int elfb200_mcts_expand_backup(elfb200_mcts* m, const float* pi_dev, const float* value_dev);
/* Root statistics (host, each may be NULL): best_action int32[G] (most visited, -1 if none),
 * visits int32[G][N*N+1] (-1 where the root has no such edge), root_value float[G] (NodeT::V_),
 * best_q float[G] (MCTSGoAI::getValue), total_visits int32[G]. */
int elfb200_mcts_results(elfb200_mcts* m, int32_t* best_action_host, int32_t* visits_host,
                         float* root_value_host, float* best_q_host, int32_t* total_visits_host);
/* The move every game plays after the search: GoGameSelfPlay::mcts_make_diverse_move +
 * GoStateExt::shouldResign (common/game_selfplay.cc:80-95,387-391, game_utils.h:15-54).  While
 * ply <= policy_distri_cutoff the move is sampled from the root visit distribution
 * (sample_multinomial, elf/utils/utils.h:158-181), afterwards it is the most visited one; a game
 * resigns (action -1) when the side to move's predicted value is below -1 + resign_thres at
 * ply >= 50 unless never_resign[g] != 0 (NULL = all games may resign).  actions int32[G]
 * (-2 = game was not searched), values float[G] = MCTSGoAI::getValue (may be NULL). */
int elfb200_mcts_choose(elfb200_mcts* m, int policy_distri_cutoff, float resign_thres,
                        const uint8_t* never_resign_host, uint64_t seed, int32_t* actions_host,
                        float* values_host);
/* SearchTreeT::treeAdvance for the move just played in each game (actions[g] < 0: untouched). */
int elfb200_mcts_advance(elfb200_mcts* m, const int32_t* actions_host);
/* float[G][N*N+1]: current prior of every root edge by action (-1 where the root has no such
 * edge), after any exploration noise (NodeT::enhanceExploration, tree_search_node.h:132-155). */
int elfb200_mcts_root_priors(elfb200_mcts* m, float* priors_host);
/* The root edges of every game in STORAGE order -- the order MCTSActor::pi2response produced them
 * and NodeT::setEvaluation inserted them into the reference's edge container (go/mcts/mcts.h:255-332,
 * tree_search_node.h:176-203): n_edges int32[G] (0 = no expanded root), and per edge, row stride
 * N*N+1: action int16 (-1 past the end), visit count N int32, reward sum W float, prior P float.
 * Any table but n_edges may be NULL.  With elfb200_refstream.h this is what the reference's
 * container-order consumers need (first-maximum tie-break, sample_multinomial, root noise). */
int elfb200_mcts_root_edges(elfb200_mcts* m, int32_t* n_edges_host, int16_t* actions_host, int32_t* visits_host,
                            float* wsum_host, float* priors_host);
/* Overwrite the priors of the root edges (storage order, float[G][N*N+1]) of the selected games
 * (mask uint8[G], NULL = all): the device end of NodeT::enhanceExploration when the noise is drawn
 * by the caller (elfb200_refstream_root_noise) instead of the built-in counter-based generator
 * (create the search with root_epsilon = 0 then).  Call between begin_move and the first wave. */
int elfb200_mcts_set_root_priors(elfb200_mcts* m, const uint8_t* mask_host, const float* priors_host);
/* rotation_flip from a caller-supplied stream: codes uint8[G][count], the D4 codes game g's next
 * evaluated leaves receive, in the order the leaves are claimed (BoardFeature::RandomShuffle draws
 * them from the actor's generator in that order, board_feature.h:74-78, go/mcts/mcts.h:86-93).
 * count >= num_rollouts rounded up to whole waves; resets the per-game consumption counters, which
 * elfb200_mcts_d4_used reads back (int32[G]) -- set a fresh stream before every move (a game that ran
 * past its codes would keep receiving the last one).  codes = NULL returns to the built-in generator. */
int elfb200_mcts_set_d4_stream(elfb200_mcts* m, const uint8_t* codes_host, int count);
int elfb200_mcts_d4_used(elfb200_mcts* m, int32_t* used_host);
/* int32[4]: [0] root-hash mismatches (the reference throws "Root state is not the same as the input
 * state", tree_search.h:488-492; here the stale tree is discarded and rebuilt from the board),
 * [1] node-pool exhaustion during a descent (rollout cut short), [2] descents cut at 128 plies
 * below the root, [3] moves whose persistent tree had to be pruned to fit the pool (least-visited
 * root subtrees recycled; benign). */
int elfb200_mcts_errors(elfb200_mcts* m, int32_t* counters_host4);
int64_t elfb200_mcts_eval_count(const elfb200_mcts* m);
/* uint64[4] running totals: descent steps (nodes visited by PUCT), edge records actually read
 * (selected prefix + 1), nodes created, stored edges of the visited nodes (what the reference's
 * full scan touches).  Used by bench.py for the select kernel's algorithmic bytes. */
int elfb200_mcts_stats(elfb200_mcts* m, uint64_t* counters_host4);
/* double[4]: accumulated device time (ms, CUDA events on the context stream) of the select,
 * leaf-feature, expand and backup kernels, and the number of waves they cover; reset != 0 clears. */
int elfb200_mcts_timings(elfb200_mcts* m, double* ms_host4, int64_t* waves, int reset);

/* Copy search trees from another handle, node for node: dst game i gets an exact replica of src game
 * index[i]'s tree (root, free stack, every in-use node, the edges of every visited node) for index[i] in
 * [0, G_src); any other value leaves game i's tree as it is.  The random state of each game (D4 codes, root
 * noise), the counters and the per-wave buffers stay with dst.  Copy the boards with the same index first
 * (elfb200_gather_games): the next begin_move checks each root against its board.
 * Same board size and nodes_per_game; dst != src, but both may search the same board context (two AIs with
 * a tree per colour).  ELFB200_ERR_ARG, with nothing enqueued, for NULL arguments, dst == src, different
 * board sizes, devices or pool sizes, and when either handle has a wave open (select issued, expand_backup
 * not yet).
 * _gather: host index int32[G_dst], synchronous.  _gather_dev: device index int32[G_dst], asynchronous on
 * dst's context stream, after the work already on src's stream; src's later work runs after the copy
 * (the two timing-free events of dst's board context that elfb200_gather_games_dev uses), so it can be captured in a CUDA graph that holds both streams. */
int elfb200_mcts_gather(elfb200_mcts* dst, const elfb200_mcts* src, const int32_t* index_host);
int elfb200_mcts_gather_dev(elfb200_mcts* dst, const elfb200_mcts* src, const int32_t* index_dev);
/* int32[G] each (host): in-use nodes, and stored edges of the visited nodes, of every game's tree -- what
 * elfb200_mcts_gather copies for the game. */
int elfb200_mcts_tree_usage(elfb200_mcts* m, int32_t* nodes_host, int32_t* edges_host);

/* ---- Search without the host: the device forms ------------------------------------------------------------
 * Every pointer is device memory.  Each call only enqueues work on the context stream: no host synchronisation,
 * no host<->device copy, no event record, no allocation, so the calls can be captured in a CUDA graph from their
 * first call.  They launch the kernels of their host forms, and compute what those compute:
 *     elfb200_mcts_reset_dev(m, mask)                    elfb200_mcts_reset
 *     elfb200_mcts_begin_move_dev(m, active, move)       elfb200_mcts_begin_move
 *     elfb200_mcts_select_dev(m, feat, format, cpad)     elfb200_mcts_select_ex(..., n_leaves = NULL)
 *     elfb200_mcts_expand_backup_dev(m, pi, value)       elfb200_mcts_expand_backup
 *     elfb200_mcts_results_dev(m, ...)                   elfb200_mcts_results
 *     elfb200_mcts_choose_dev(m, ..., seed, ...)         elfb200_mcts_choose
 *     elfb200_mcts_advance_dev(m, actions)               elfb200_mcts_advance
 * The random draws that the host forms key by a value passed by value are keyed by device memory here, so a
 * replayed graph draws what the caller's counters hold at replay time: the root noise by (seed, (uint32)*move_dev),
 * as begin_move keys it by its host move counter (which the device form neither reads nor advances); the move
 * choice by *seed_dev, bit for bit the host form's key with that seed.
 * A whole move is begin_move_dev, then elfb200_mcts_waves_per_move x (select_dev, the network on all
 * elfb200_mcts_max_leaves rows, expand_backup_dev).  The D4 code of each leaf is keyed by the wave index, which the
 * host passes by value and begin_move_dev sets back to 0: a graph must therefore capture whole moves.
 * Host-side counters do not see work replayed from a graph: elfb200_mcts_timings never counts the device forms, and
 * elfb200_mcts_eval_count in synchronous mode counts host-form waves only (after a select_dev it reads the device
 * total, as in the asynchronous mode).  The device counters (elfb200_mcts_stats, elfb200_mcts_errors) see every
 * wave.  A root that does not match its board is counted in elfb200_mcts_errors [0] and rebuilt.
 * Refused with nothing enqueued: NULL handle (ELFB200_ERR_ARG); any device form while a reference D4 stream is set
 * (ELFB200_ERR_STATE: elfb200_mcts_set_d4_stream is fed from the host every move). */
/* reset for the games with mask_dev[g] != 0 (uint8[G], NULL = all games). */
int elfb200_mcts_reset_dev(elfb200_mcts* m, const uint8_t* mask_dev);
/* active_dev uint8[G] (NULL = all active) copied device to device, then begin_move; move_dev int64[1] keys the
 * root noise and may be NULL only with root_epsilon == 0 (ELFB200_ERR_ARG).  Sets the wave index back to 0.
 * ELFB200_ERR_STATE while a wave is open. */
int elfb200_mcts_begin_move_dev(elfb200_mcts* m, const uint8_t* active_dev, const int64_t* move_dev);
/* The asynchronous select, in any format elfb200_mcts_select_ex accepts; the leaf count stays on the device and the
 * feature grid covers all G*B slots.  ELFB200_ERR_ARG for a NULL feat_dev or a bad format, ELFB200_ERR_STATE while
 * a wave is open. */
int elfb200_mcts_select_dev(elfb200_mcts* m, void* feat_dev, int format, int cpad);
/* Expansion and backup with elfb200_mcts_max_leaves reply rows (rows past the device-side count are ignored).
 * ELFB200_ERR_ARG for NULL pi / value, ELFB200_ERR_STATE when no wave is open. */
int elfb200_mcts_expand_backup_dev(elfb200_mcts* m, const float* pi_dev, const float* value_dev);
/* The tables of elfb200_mcts_results into device arrays, each may be NULL. */
int elfb200_mcts_results_dev(elfb200_mcts* m, int32_t* best_action_dev, int32_t* visits_dev, float* root_value_dev,
                             float* best_q_dev, int32_t* total_visits_dev);
/* choose with the seed read from seed_dev (int64[1]); never_resign_dev uint8[G] may be NULL, values_dev may be NULL.
 * ELFB200_ERR_ARG for NULL seed_dev or actions_dev. */
int elfb200_mcts_choose_dev(elfb200_mcts* m, int policy_distri_cutoff, float resign_thres,
                            const uint8_t* never_resign_dev, const int64_t* seed_dev, int32_t* actions_dev,
                            float* values_dev);
/* advance from a device array int32[G] (actions[g] < 0: untouched).  ELFB200_ERR_ARG for NULL actions_dev. */
int elfb200_mcts_advance_dev(elfb200_mcts* m, const int32_t* actions_dev);

#ifdef __cplusplus
}
#endif
#endif /* ELFB200_MCTS_H_ */
