// oracle/ref_mcts_df_shim.cc -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// The reference search of ref_mcts_shim.cc with GameOptions::use_df_feature set: MCTSActor::evaluate
// (go/mcts/mcts.h:73-121) hands the network BoardFeature::extract's 25 DarkForest planes
// (board_feature.cc:209-237) instead of extractAGZ's 18, exactly as the reference does when the option
// switches the "s" field (common/game_feature.h:22-33,159-168).  Every other line executed is the
// reference's, as in ref_mcts_shim.cc; the network is the caller's callback.
//
// Built by ref_df.mk into oracle/_ref/libref_mcts_df{19,9}.so, linked against libref_go{19,9}.so: the
// reference's compiled board code (GoState, BoardFeature, ...) and the states the tests create through
// ref_shim.cc live in that library, so a RefState handle from it is searched here directly.
//
// The access-control override below applies to this translation unit only.
#include <atomic>
#include <functional>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include <nlohmann/json.hpp>
#include <pybind11/pybind11.h>
#include <spdlog/spdlog.h>

#define private public
#define protected public
#include "elfgames/go/mcts/mcts.h"
#undef private
#undef protected

namespace {

using elf::ai::tree_search::TSOptions;

// feats float [n][25][N][N], pi float [n][P+1] (NN action order), v float [n]
typedef void (*eval_cb_t)(int n, const float* feats, const uint64_t* hashes, float* pi, float* v);

class DfShimActor {
 public:
  using Action = Coord;
  using State = GoState;
  using NodeResponse = elf::ai::tree_search::NodeResponseT<Coord>;

  DfShimActor(const MCTSActorParams& params, eval_cb_t cb, std::atomic<long>* n_evals)
      : inner_(nullptr, params), cb_(cb), n_evals_(n_evals) {}

  // MCTSActor::evaluate (go/mcts/mcts.h:73-121) with ai_->act_batch replaced by the callback, on the
  // DarkForest planes of each leaf (under the D4 code get_extractor drew for it).
  void evaluate(const std::vector<const GoState*>& states, std::vector<NodeResponse>* p_resps) {
    if (states.empty())
      return;
    auto& resps = *p_resps;
    resps.resize(states.size());
    std::vector<BoardFeature> sel_bfs;
    std::vector<size_t> sel_indices;
    for (size_t i = 0; i < states.size(); i++) {
      auto res = inner_.pre_evaluate(*states[i], &resps[i]);
      if (res == MCTSActor::EVAL_NEED_NN) {
        sel_bfs.push_back(inner_.get_extractor(*states[i]));
        sel_indices.push_back(i);
      }
    }
    if (sel_bfs.empty())
      return;
    const int P1 = BOARD_NUM_ACTION;
    std::vector<GoReply> replies;
    for (size_t i = 0; i < sel_bfs.size(); ++i)
      replies.emplace_back(sel_bfs[i]);
    const size_t n = sel_bfs.size();
    const size_t F = MAX_NUM_FEATURE * BOARD_SIZE * BOARD_SIZE;
    std::vector<float> feats(n * F), pi(n * P1), v(n);
    std::vector<uint64_t> hashes(n);
    for (size_t i = 0; i < n; ++i) {
      sel_bfs[i].extract(&feats[i * F]);
      hashes[i] = sel_bfs[i].state().getHashCode();
    }
    cb_((int)n, feats.data(), hashes.data(), pi.data(), v.data());
    for (size_t i = 0; i < n; ++i) {
      for (int a = 0; a < P1; ++a)
        replies[i].pi[a] = pi[i * P1 + a];
      replies[i].value = v[i];
    }
    if (n_evals_)
      n_evals_->fetch_add((long)n);
    for (size_t i = 0; i < n; i++)
      inner_.post_nn_result(replies[i], &resps[sel_indices[i]]);
  }

  void evaluate(const GoState& s, NodeResponse* resp) {
    std::vector<const GoState*> v{&s};
    std::vector<NodeResponse> r;
    evaluate(v, &r);
    *resp = r[0];
  }

  bool forward(GoState& s, Coord a) {
    return inner_.forward(s, a);
  }
  float reward(const GoState& s, float value) const {
    return inner_.reward(s, value);
  }
  std::mt19937* rng() {
    return inner_.rng();
  }
  std::string info() const {
    return inner_.info();
  }
  void setID(int) {}

 private:
  MCTSActor inner_;
  eval_cb_t cb_;
  std::atomic<long>* n_evals_;
};

struct RefMctsDf {
  std::unique_ptr<elf::ai::tree_search::MCTSAI_T<DfShimActor>> ai;
  std::atomic<long> n_evals{0};
};

inline int c2a(Coord c) {
  if (c == M_PASS)
    return BOARD_SIZE * BOARD_SIZE;
  return EXPORT_OFFSET(c);
}

} // namespace

namespace elf {
namespace ai {
namespace tree_search {
template <>
struct ActorTrait<DfShimActor> {
  static std::string to_string(const DfShimActor& a) {
    return a.info();
  }
};
} // namespace tree_search
} // namespace ai
} // namespace elf

extern "C" {

// ref_mcts_new_ex of ref_mcts_shim.cc (same iopts / fopts layout, rotation_flip, 32-bit actor seed) on the
// DarkForest planes; cb is required.
void* ref_mcts_new_df(const int32_t* iopts, const float* fopts, eval_cb_t cb, int rotation_flip, uint32_t seed) {
  TSOptions opt;
  opt.num_threads = iopts[10] > 0 ? iopts[10] : 1;
  opt.num_rollouts_per_thread = iopts[0];
  opt.num_rollouts_per_batch = iopts[1];
  opt.virtual_loss = iopts[2];
  opt.persistent_tree = iopts[3] != 0;
  opt.alg_opt.use_prior = iopts[4] != 0;
  opt.alg_opt.unexplored_q_zero = iopts[5] != 0;
  opt.alg_opt.root_unexplored_q_zero = iopts[6] != 0;
  opt.alg_opt.c_puct = fopts[0];
  opt.root_epsilon = fopts[2];
  opt.root_alpha = fopts[3];
  opt.pick_method = "most_visited";
  opt.seed = iopts[9];

  MCTSActorParams params;
  params.actor_name = "shim_df";
  params.ply_pass_enabled = iopts[7];
  params.remove_pass_if_dangerous = iopts[8] != 0;
  params.seed = seed;
  params.komi = fopts[1];
  params.rotation_flip = rotation_flip != 0;
  params.required_version = -1;

  RefMctsDf* m = new RefMctsDf();
  std::atomic<long>* ctr = &m->n_evals;
  m->ai.reset(new elf::ai::tree_search::MCTSAI_T<DfShimActor>(
      opt, [params, cb, ctr](int) { return new DfShimActor(params, cb, ctr); }));
  return m;
}

void ref_mcts_df_free(void* p) {
  delete static_cast<RefMctsDf*>(p);
}

// MCTSAI_T::act, or actPolicyOnly when policy_only (a *_use_policy_network_only colour), on a RefState of
// libref_go; outputs by action index as ref_mcts_act's.  Returns the chosen action.
int ref_mcts_df_act(void* p, void* state, int policy_only, int32_t* visits, float* wsum, float* prior,
                    float* root_value, float* best_q, int32_t* total_visits) {
  RefMctsDf* m = static_cast<RefMctsDf*>(p);
  const GoState& s = *static_cast<GoState*>(state);
  Coord c = M_INVALID;
  if (policy_only)
    m->ai->actPolicyOnly(s, &c);
  else
    m->ai->act(s, &c);
  const auto& res = m->ai->getLastResult();
  const int P1 = BOARD_NUM_ACTION;
  for (int a = 0; a < P1; ++a) {
    visits[a] = -1;
    wsum[a] = 0;
    prior[a] = 0;
  }
  for (const auto& ae : res.action_edge_pairs) {
    const int a = c2a(ae.first);
    visits[a] = ae.second.num_visits;
    wsum[a] = ae.second.reward;
    prior[a] = ae.second.prior_probability;
  }
  *root_value = res.root_value;
  *best_q = res.total_visits == 0 ? res.root_value : res.best_edge_info.getQSA();
  *total_visits = res.total_visits;
  return c2a(c);
}

// ref_mcts_sample / ref_mcts_end_game of ref_mcts_shim.cc for this search: mcts_make_diverse_move's sampling on a
// game thread's generator (a ref_rng_new handle of libref_go), and MCTSAI_T::endGame.
int ref_mcts_df_sample(void* p, void* rng) {
  auto policy = static_cast<RefMctsDf*>(p)->ai->getLastResult().mcts_policy;
  policy.normalize();
  return c2a(policy.sampleAction(static_cast<std::mt19937*>(rng)));
}

void ref_mcts_df_end_game(void* p, void* state) {
  static_cast<RefMctsDf*>(p)->ai->endGame(*static_cast<GoState*>(state));
}

long ref_mcts_df_num_evals(void* p) {
  return static_cast<RefMctsDf*>(p)->n_evals.load();
}

} // extern "C"
