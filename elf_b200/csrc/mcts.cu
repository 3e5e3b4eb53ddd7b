// mcts.cu -- batched Monte-Carlo tree search on the GPU (search path of libelfb200.so).
//
// Replaces, for a batch of G games at once, the reference's per-game multi-threaded search
//   elf::ai::tree_search::TreeSearchT / NodeT / EdgeInfo  (src_cpp/elf/ai/tree_search/*.h)
//   MCTSActor::{pre_evaluate, remove_pass_if_dangerous, pi2response} (src_cpp/elfgames/go/mcts/mcts.h)
// with a flat node pool in HBM and one warp per game.  A "wave" is what the reference calls
// batch_rollouts (tree_search.h:201-262): B sequential descents per game (they depend on each
// other through virtual loss), one batched network evaluation of the newly reached leaves of ALL
// games, expansion, and one backup per unique leaf.
//
// Node pool (structure of arrays; game g owns slots [g*C, (g+1)*C), 16-bit local ids):
//   pos    uint64 [G*C][N]      position rows (black | white << 32), set when the node is created
//   sa     uint64 [G*C][N]      the position's incremental group status rows (safe | atari << 32)
//   hash   uint64 [G*C]         Zobrist hash
//   meta   BoardMeta [G*C]      ply, side, ko, last moves, terminal flags
//   hdr    NodeHdr [G*C]        visits, V, running unsigned mean Q, parent link, status
//   estat  float4 [G*C][E]      per edge {prior P, visits N (int bits), reward sum W,
//                               packed word: virtual-loss applications (low 16) | child id (high 16)}
//   elink  uint32 [G*C][E]      per edge action (low 16) | child id (high 16, 0xFFFF = none); only read
//                               when a child is created and by results/advance (off the hot loop)
//   hist   uint64 [G*B][8][N]   the 8-position history of every leaf claimed in the current wave (for the feature writer)
// E = N*N+1.  Edges of a node are stored in descending-prior order (the order the reference
// inserts them, go/mcts/mcts.h:292-329), only the legal ones.
//
// Kernels: k_begin (root set-up), k_select (PUCT descent + child state creation + terminal
// evaluation + leaf claim), k_leaf_features (18-plane stack per claimed leaf, history gathered
// along the parent chain; k_leaf_features_df: the 25 DarkForest planes instead), k_expand (mask/sort/renormalise the net's policy into edges),
// k_backup, k_results, k_advance (tree reuse: keep the chosen child's subtree, free the rest),
// k_gather_trees (copy trees from another handle's pool, node for node).
#include <cfloat>

#include "common.cuh"
#include "elfb200_mcts.h"
#include "stdsort.cuh"

namespace elfb200 {

constexpr uint16_t NONE16 = 0xFFFFu;
enum : uint8_t { NS_FREE = 0, NS_UNVISITED = 1, NS_REQUESTED = 2, NS_VISITED = 3 };
enum : uint8_t { NF_FLIP = 1, NF_KEEP = 2, NF_FULLSCAN = 4 };  // FULLSCAN: priors no longer sorted (root noise) or a tie broke the prefix

struct __align__(16) NodeHdr {  // 32 bytes
  int32_t num_visits;    // NodeT::numVisits_
  float V;               // NodeT::V_
  float mean_q;          // NodeT::unsignedMeanQ_
  float parent_q;        // NodeT::unsignedParentQ_
  uint16_t n_edges;
  uint16_t parent;       // NONE16 for the root
  uint16_t parent_edge;  // index of the edge in the parent that leads here
  uint8_t status;        // NodeT::status_ (NOT_VISITED / EVAL_REQUESTED / VISITED)
  uint8_t flags;         // NF_FLIP = NodeT::flipQSign_
  uint16_t n_touched;    // edges [0, n_touched) have been selected at least once (see k_select)
  uint16_t pass_edge;    // index of the pass edge, NONE16 if the node has none
  int32_t pad;
};
static_assert(sizeof(NodeHdr) == 32, "NodeHdr must be 32 bytes");

struct TreeDev {
  uint64_t* pos;
  uint64_t* sa;          // [G*C][N] incremental group status of the node's position: safe | atari << 32 (board.cuh)
  uint64_t* hash;
  BoardMeta* meta;
  NodeHdr* hdr;
  float4* estat;
  uint32_t* elink;
  uint16_t* free_list;  // [G][C] stack of free local ids
  int32_t* free_n;      // [G]
  uint16_t* root;       // [G]
  uint16_t* leaves;     // [G][B]
  uint8_t* active;      // [G]
  int32_t* eval_count;  // [1]
  int32_t* eval_game;   // [G*B]
  uint16_t* eval_node;  // [G*B]
  uint8_t* eval_d4;     // [G*B]
  uint64_t* hist;       // [G*B][8][N] history rows of every claimed leaf, newest first (written by k_select)
  uint32_t* hinfo;      // [G*B] hn | side to move << 8 | d4 << 16
  uint16_t* bfs_q;      // [G][C]
  int32_t* errors;      // [4]: root-hash mismatches, pool overflows, ...
  unsigned long long* stats;  // [4]: descent steps, edge records read, nodes created, stored edges of visited nodes
  // optional host-supplied D4 codes (elfb200_mcts_set_d4_stream): the next code of game g is
  // d4_stream[g * d4_cap + d4_used[g]]; NULL = the counter-based generator
  const uint8_t* d4_stream;
  int32_t* d4_used;  // [G]
  int d4_cap;
  int C, B, E;
};

struct SearchOpts {
  int num_rollouts, virtual_loss, persistent, use_prior, uqz, ruqz, ply_pass_enabled,
      remove_pass_if_dangerous, rotation_flip, seed, std_sort_ties;
  float c_puct, komi;
};

// NOTE: the board primitives take the reductions' lane set from Lane::segmask / Lane::active when
// Geo<N>::GPW != 1, so a single-segment Lane gives a one-game-per-warp mode for 9x9 as well.

__device__ __forceinline__ NodeHdr load_hdr(const NodeHdr* p) {
  const uint4* q = reinterpret_cast<const uint4*>(p);
  uint4 a = q[0], b = q[1];
  NodeHdr h;
  memcpy(&h, &a, 16);
  memcpy(reinterpret_cast<char*>(&h) + 16, &b, 16);
  return h;
}
__device__ __forceinline__ void store_hdr(NodeHdr* p, const NodeHdr& h) {
  uint4 a, b;
  memcpy(&a, &h, 16);
  memcpy(&b, reinterpret_cast<const char*>(&h) + 16, 16);
  uint4* q = reinterpret_cast<uint4*>(p);
  q[0] = a;
  q[1] = b;
}

__device__ __forceinline__ int pop_free(const TreeDev& tr, int g) {  // lane 0 only
  int n = tr.free_n[g];
  if (n <= 0) return -1;
  tr.free_n[g] = n - 1;
  return tr.free_list[(size_t)g * tr.C + n - 1];
}

// ---------------------------------------------------------------------------------------
// Free the subtree below `top` (inclusive): BFS through the child links, every node goes back on the
// game's free stack.  Whole warp; `q` is the game's BFS scratch.
__device__ __forceinline__ void free_subtree(const TreeDev& tr, size_t nb, int g, int top, int lane) {
  uint16_t* q = tr.bfs_q + nb;
  int head = 0, tail = 1;
  if (lane == 0) q[0] = (uint16_t)top;
  __syncwarp();
  while (head < tail) {
    const int node = q[head++];
    const int ne = tr.hdr[nb + node].status == NS_VISITED ? (int)tr.hdr[nb + node].n_edges : 0;
    const uint32_t* el = tr.elink + (nb + node) * tr.E;
    for (int i0 = 0; i0 < ne; i0 += 32) {
      const int i = i0 + lane;
      const int child = i < ne ? (int)(el[i] >> 16) : (int)NONE16;
      const bool has = child != NONE16;
      const uint32_t bal = __ballot_sync(FULL, has);
      if (has) q[tail + __popc(bal & ((1u << lane) - 1u))] = (uint16_t)child;
      tail += __popc(bal);
    }
    __syncwarp();
  }
  // q[0 .. tail) is the subtree: release it
  int n = tr.free_n[g];
  __syncwarp();
  for (int i = lane; i < tail; i += 32) {
    const int node = q[i];
    tr.hdr[nb + node].status = NS_FREE;
    tr.hdr[nb + node].flags = 0;
    tr.free_list[nb + n + i] = (uint16_t)node;
  }
  __syncwarp();
  if (lane == 0) tr.free_n[g] = n + tail;
  __syncwarp();
}

__device__ __forceinline__ void reset_game_pool(const TreeDev& tr, size_t nb, int g, int lane) {
  for (int i = lane; i < tr.C; i += 32) {
    tr.free_list[nb + i] = (uint16_t)(tr.C - 1 - i);
    tr.hdr[nb + i].status = NS_FREE;
    tr.hdr[nb + i].flags = 0;
  }
  __syncwarp();
  if (lane == 0) tr.free_n[g] = tr.C;
  __syncwarp();
}

// Root set-up: SearchTreeT::allocateRoot + TreeSearchT::setRootNodeState (tree_search_node.h:555,
// tree_search.h:478-493).  One warp per game.
//
// Bounded pool (the reference's heap is not): when fewer than `rollouts_needed` slots are free the
// persistent tree is PRUNED, not dropped -- the subtrees under the root's least-visited children
// are recycled (fewest visits first, later edge first among equals) until this move's rollouts fit.
// The root edge keeps its statistics (N, W) and only loses the child link, so a later descent
// through it re-creates and re-evaluates the child.  Counter errors[3] (benign).
template <int N>
__global__ void __launch_bounds__(BLOCK) k_begin(DevState st, TreeDev tr, int rollouts_needed) {
  const Lane L = make_lane_single<N>();
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= st.G || !tr.active[g]) return;
  const size_t nb = (size_t)g * tr.C;
  int root = tr.root[g];
  if (root != NONE16 && tr.hash[nb + root] != st.hash[g]) {
    // "TreeSearch::Root state is not the same as the input state" (tree_search.h:488-492): the
    // reference throws; here the stale tree is discarded, the search restarts from the board, and
    // the counter lets the host raise (MctsBatch.begin_move does).
    if (L.lane == 0) atomicAdd(&tr.errors[0], 1);
    reset_game_pool(tr, nb, g, L.lane);
    root = NONE16;
  }
  if (root != NONE16 && tr.free_n[g] < rollouts_needed + 1) {
    if (L.lane == 0) atomicAdd(&tr.errors[3], 1);
    const int ne = tr.hdr[nb + root].status == NS_VISITED ? (int)tr.hdr[nb + root].n_edges : 0;
    float4* es = tr.estat + (nb + root) * tr.E;
    uint32_t* el = tr.elink + (nb + root) * tr.E;
    while (tr.free_n[g] < rollouts_needed + 1) {
      // least-visited root edge that still has a child
      int bestn = 0x7FFFFFFF, besti = -1;
      for (int i = L.lane; i < ne; i += 32) {
        if ((el[i] >> 16) != NONE16) {
          const int n = __float_as_int(es[i].y);
          if (n <= bestn) {
            bestn = n;
            besti = i;
          }
        }
      }
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        const int on = __shfl_xor_sync(FULL, bestn, d), oi = __shfl_xor_sync(FULL, besti, d);
        if (on < bestn || (on == bestn && oi > besti)) {
          bestn = on;
          besti = oi;
        }
      }
      if (besti < 0) break;  // the root alone: C >= rollouts + 2 guarantees room
      const int child = (int)(el[besti] >> 16);
      __syncwarp();
      if (L.lane == 0) {
        el[besti] = (el[besti] & 0xFFFFu) | ((uint32_t)NONE16 << 16);
        es[besti].w = __uint_as_float((__float_as_uint(es[besti].w) & 0xFFFFu) | ((uint32_t)NONE16 << 16));
      }
      __syncwarp();
      free_subtree(tr, nb, g, child, L.lane);
    }
  }
  if (root == NONE16) {
    int id = 0;
    if (L.lane == 0) id = pop_free(tr, g);
    id = __shfl_sync(FULL, id, 0);
    if (L.active) {
      tr.pos[(nb + id) * N + L.row] = st.cur[(size_t)g * N + L.row];
      tr.sa[(nb + id) * N + L.row] = st.sa[(size_t)g * N + L.row];
    }
    if (L.lane == 0) {
      tr.hash[nb + id] = st.hash[g];
      tr.meta[nb + id] = st.meta[g];
      NodeHdr h;
      h.num_visits = 0;
      h.V = 0.f;
      h.mean_q = 0.f;
      h.parent_q = 0.f;  // allocateRoot: addNode(0.0)
      h.n_edges = 0;
      h.parent = NONE16;
      h.parent_edge = 0;
      h.status = NS_UNVISITED;
      h.flags = 0;
      h.n_touched = 0;
      h.pass_edge = NONE16;
      h.pad = 0;
      store_hdr(&tr.hdr[nb + id], h);
      tr.root[g] = (uint16_t)id;
    }
  }
}

// ---------------------------------------------------------------------------------------
// One wave of descents: TreeSearchSingleThreadT::single_rollout x B (tree_search.h:265-322) with
// NodeT::findMove/UCT (tree_search_node.h:205-231,361-397), EdgeInfo::getScore
// (tree_search_base.h:132-157), addVirtualLoss (:233-251), followEdge (:280-302), allocateState
// (tree_search.h:175-190) and the leaf claim of batch_rollouts (tree_search.h:222-233).
//
// PUCT scan: edges are stored by descending prior and an edge that was never selected has
// N = 0, vl = 0, hence score = c_puct * P * sqrt(n) + FPU, monotone (not strictly: the product
// vanishes under the rounding of q for tiny priors) in P.  The best never-selected edge is therefore
// the FIRST one in storage order or ties with it, the selected edges form a prefix [0, n_touched),
// and the maximum over all edges equals the maximum over [0, n_touched] -- the same result as the
// reference's full scan with O(touched) instead of O(legal moves) reads.  The scan takes one edge
// more, [0, n_touched + 1]: if the maximum over that range is attained once it is the reference's
// choice; if it is tied -- within the prefix, or between the first never-selected edge and the
// next -- the reference's answer is the first tied edge in ITS container's order, which
// uct_tie_break reproduces from a full rescan; a node where that picked an edge beyond the prefix is
// scanned in full from then on (NF_FULLSCAN).  The running-mean update only involves selected edges.
//
// The per-level dependent memory chain is one round trip: the node header and the first 32 edge
// records are requested together; the child id rides in the edge record; the pre-move hashes the
// superko test needs are gathered once, when a child is actually created.
constexpr int MAX_DEPTH = 128;

// ---------------------------------------------------------------------------------------
// "First maximum in container order".  MCTSResultT::addActions (tree_search_base.h:237-294) walks the
// root's std::unordered_map<Coord, EdgeInfo> and keeps the first edge with the strictly largest visit
// count, so an exact most-visited TIE is resolved by the hash table's iteration order.  That order is a
// function of the insertion sequence alone (NodeT::setEvaluation inserts the edges in storage order):
// libstdc++'s table is one forward list; a key whose bucket is empty goes to the FRONT of the list, a
// key whose bucket is in use goes right behind that bucket's "before" node (i.e. to the front of its
// bucket's run); hash(Coord) = Coord, bucket = key % bucket_count; bucket counts 13, 29, 59, 127, 257,
// 541, growing when the 14th, 30th, 60th, 128th, 258th key arrives, and a rehash re-inserts the list,
// front to back, by the same two rules (hashtable.h _M_insert_bucket_begin / _M_rehash_aux,
// hashtable_policy.h _Prime_rehash_policy).  Pinned against std::unordered_map itself and against
// the compiled reference (tests/test_refstream.py, tests/test_emu_kernels.py).
// The PUCT arg-max of every descent step (NodeT::UCT, tree_search_node.h:361-397) walks the same kind of
// container with the same strict '>': k_select resolves exact score ties the same way (uct_tie_break).
// Lane 0 replays the insertions in shared memory; only called when the maximum is actually tied.
struct OrderScratch {
  uint16_t nxt[448];  // forward list: key -> next key
  uint16_t idx[448];  // key -> storage index of the edge
  uint16_t bkt[544];  // bucket -> key of the node BEFORE the bucket's first node
};
constexpr uint16_t OS_NIL = 0xFFFFu, OS_HEAD = 0xFFFEu, OS_EMPTY = 0xFFFDu;

template <int N>
__device__ __forceinline__ int action_to_coord(int a) {  // board.h:183-184; pass = M_PASS = 0
  return a >= N * N ? 0 : ((a % N) + 1) * (N + 2) + (a / N) + 1;
}

__device__ __forceinline__ void os_link(OrderScratch& s, uint16_t& head, int nb, int key) {
  const int b = key % nb;
  const uint16_t before = s.bkt[b];
  if (before == OS_EMPTY) {  // new bucket: the node becomes the list's first
    s.nxt[key] = head;
    if (head != OS_NIL) s.bkt[head % nb] = (uint16_t)key;
    head = (uint16_t)key;
    s.bkt[b] = OS_HEAD;
  } else if (before == OS_HEAD) {
    s.nxt[key] = head;
    head = (uint16_t)key;
  } else {
    s.nxt[key] = s.nxt[before];
    s.nxt[before] = (uint16_t)key;
  }
}

// lane 0 only: replay the insertions of edges [0, ne) (storage order); returns the list head
template <int N>
__device__ uint16_t os_build(const uint32_t* __restrict__ el, int ne, OrderScratch& s) {
  int nb = 13;
  uint16_t head = OS_NIL;
  for (int b = 0; b < nb; ++b) s.bkt[b] = OS_EMPTY;
  for (int i = 0; i < ne; ++i) {
    if (i == 13 || i == 29 || i == 59 || i == 127 || i == 257) {  // the table grows before key i+1 goes in
      nb = i == 13 ? 29 : i == 29 ? 59 : i == 59 ? 127 : i == 127 ? 257 : 541;
      for (int b = 0; b < nb; ++b) s.bkt[b] = OS_EMPTY;
      uint16_t p = head;
      head = OS_NIL;
      while (p != OS_NIL) {
        const uint16_t q = s.nxt[p];
        os_link(s, head, nb, p);
        p = q;
      }
    }
    const int key = action_to_coord<N>((int)(el[i] & 0xFFFFu));
    s.idx[key] = (uint16_t)i;
    os_link(s, head, nb, key);
  }
  return head;
}

template <int N>
__device__ int first_max_in_container_order(const uint32_t* __restrict__ el, const float4* __restrict__ es, int ne,
                                            int bestn, OrderScratch& s, int lane) {
  int res = 0;
  if (lane == 0) {
    res = 0x7FFFFFFF;
    for (uint16_t p = os_build<N>(el, ne, s); p != OS_NIL; p = s.nxt[p]) {
      const int i = s.idx[p];
      if (__float_as_int(es[i].y) == bestn) {
        res = i;
        break;
      }
    }
  }
  return __shfl_sync(FULL, res, 0);
}

// the same walk for an arbitrary tie set: tied[i >> 5] bit (i & 31) = edge i attains the maximum
template <int N>
__device__ int first_tied_in_container_order(const uint32_t* __restrict__ el, int ne, const uint32_t* tied,
                                             OrderScratch& s, int lane) {
  int res = 0;
  if (lane == 0) {
    res = 0x7FFFFFFF;
    for (uint16_t p = os_build<N>(el, ne, s); p != OS_NIL; p = s.nxt[p]) {
      const int i = s.idx[p];
      if ((tied[i >> 5] >> (i & 31)) & 1u) {
        res = i;
        break;
      }
    }
  }
  return __shfl_sync(FULL, res, 0);
}

__device__ __forceinline__ float vl_value(uint32_t wbits, int virtual_loss) {
  return (float)((int)(wbits & 0xFFFFu) * virtual_loss);  // exact: small integers
}

// EdgeInfo::getScore + NodeT::UCT's combination for one edge record (tree_search_base.h:132-157,
// tree_search_node.h:361-397): n = visits, nwl = visits with virtual loss; one definition for the
// descent's scan and for the tie-break's rescans, so that "equal score" means the same bits in both
__device__ __forceinline__ float puct_score(const float4& e, bool flip, float fpu, double sq, const SearchOpts& o,
                                            int& n, int& nwl) {
  n = __float_as_int(e.y);
  const float evl = vl_value(__float_as_uint(e.w), o.virtual_loss);
  float r = flip ? -e.z : e.z;
  r -= evl;
  nwl = (int)((float)n + evl);
  const float q = nwl > 0 ? r / (float)nwl : (flip ? -fpu : fpu);
  const float u = (float)((double)(e.x / (float)(1 + n)) * sq);
  return o.use_prior ? __fmaf_rn(u, o.c_puct, q) : q;
}

// The maximum of a descent step is tied (exactly equal scores: priors below the rounding of q, equal
// terminal values, or no prior term at all): the reference's loop over its unordered_map keeps the
// FIRST maximum in the container's order.  Rescan ALL edges of the node (never-selected edges beyond
// the scanned prefix can only tie with, never beat, the prefix's first never-selected edge -- same q,
// smaller prior), mark the tied ones and let lane 0 walk the container.  Rare; whole warp.
template <int N>
__device__ int uct_tie_break(const uint32_t* __restrict__ el, const float4* __restrict__ es, int ne, bool flip,
                             float fpu, double sq, const SearchOpts& o, OrderScratch& scratch, uint32_t* tied,
                             int lane) {
  float best = -FLT_MAX;
  for (int i = lane; i < ne; i += 32) {
    int n, nwl;
    best = fmaxf(best, puct_score(es[i], flip, fpu, sq, o, n, nwl));
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) best = fmaxf(best, __shfl_xor_sync(FULL, best, d));
  for (int i0 = 0; i0 < ne; i0 += 32) {
    const int i = i0 + lane;
    int n, nwl;
    const bool t = i < ne && puct_score(es[i], flip, fpu, sq, o, n, nwl) == best;
    const uint32_t bits = __ballot_sync(FULL, t);
    if (lane == 0) tied[i0 >> 5] = bits;
  }
  __syncwarp();
  const int res = first_tied_in_container_order<N>(el, ne, tied, scratch, lane);
  __syncwarp();
  return res;
}

template <int N>
__global__ void __launch_bounds__(BLOCK) k_select(DevState st, TreeDev tr, SearchOpts o, int wave) {
  __shared__ uint64_t s_zob[Geo<N>::ZOB];
  __shared__ uint32_t s_path[WARPS][MAX_DEPTH];  // node id | is_pass << 16, root first
  __shared__ OrderScratch s_order[WARPS];        // tie-break scratch (uct_tie_break)
  __shared__ uint32_t s_tied[WARPS][(Geo<N>::P + 32) / 32];
  load_zobrist<N>(s_zob);
  const Lane L = make_lane_single<N>();
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= st.G || !tr.active[g]) return;
  const size_t nb = (size_t)g * tr.C;
  const int E = tr.E;
  const int root = tr.root[g];
  uint64_t* skg = st.sk + (size_t)g * Geo<N>::MAX_PLY;
  const int nsk0 = st.sk_n[g];
  uint32_t* path = s_path[threadIdx.x >> 5];
  const int rootply = st.meta[g].ply;  // ply of the root == ply of the game
  unsigned st_steps = 0, st_edges = 0, st_new = 0, st_term = 0;

  for (int j = 0; j < tr.B; ++j) {
    int node = root, depth = 0;
    while (true) {
      const float4* es = tr.estat + (nb + node) * E;
      const NodeHdr h = load_hdr(&tr.hdr[nb + node]);
      float4 e = es[L.lane];  // speculative first chunk (E >= 82 > 32: always in bounds)
      if (h.status != NS_VISITED || h.n_edges == 0) break;
      if (depth >= MAX_DEPTH) {
        if (L.lane == 0) atomicAdd(&tr.errors[2], 1);
        break;
      }
      // ---- UCT over the selected prefix plus the first TWO never-selected edges ------------------
      // (the second one only reveals a tie with the first: all later ones score no higher than it)
      const int lim = (h.flags & NF_FULLSCAN) ? (int)h.n_edges : min((int)h.n_edges, (int)h.n_touched + 2);
      st_steps++;
      st_edges += lim;
      st_term += h.n_edges;  // stored edges: what a full scan (SURVEY 8d formula) would read
      const bool flip = h.flags & NF_FLIP;
      const float fpu = (o.uqz || (o.ruqz && depth == 0)) ? 0.f : h.mean_q;
      const double sq = sqrt((double)(h.num_visits + 1));  // std::sqrt(int) -> double
      float best = -FLT_MAX, tuq = 0.f;
      int besti = 0x7FFFFFFF, tv = 0, neq = 0;
      for (int i = L.lane; i < lim; i += 32) {
        if (i >= 32) e = es[i];
        int n, nwl;
        const float score = puct_score(e, flip, fpu, sq, o, n, nwl);
        const float uq = n > 0 ? e.z / (float)n : fpu;
        if (score > best) {  // strict >
          best = score;
          besti = i;
          neq = 1;
        } else if (score == best) {
          neq++;
        }
        if (nwl != 0) {
          tuq += uq;
          tv++;
        }
      }
      const float lane_best = best;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        const float ob = __shfl_xor_sync(FULL, best, d);
        const int oi = __shfl_xor_sync(FULL, besti, d);
        if (ob > best || (ob == best && oi < besti)) {
          best = ob;
          besti = oi;
        }
        tuq += __shfl_xor_sync(FULL, tuq, d);
        tv += __shfl_xor_sync(FULL, tv, d);
      }
      // an untied maximum is the answer; a tied one goes through the reference's container order
      const uint32_t at_max = __ballot_sync(FULL, lane_best == best);
      const bool tie = __popc(at_max) > 1 || __any_sync(FULL, lane_best == best && neq > 1);
      if (tie)
        besti = uct_tie_break<N>(tr.elink + (nb + node) * E, es, (int)h.n_edges, flip, fpu, sq, o,
                                 s_order[threadIdx.x >> 5], s_tied[threadIdx.x >> 5], L.lane);
      const int ei = besti;
      const float new_mean = (h.parent_q + tuq) / (float)(tv + 1);
      const bool is_pass = ei == (int)h.pass_edge;
      // ---- addVirtualLoss + followEdge: one read-modify-write of the packed word -----------------
      uint32_t wb = 0;
      if (L.lane == 0) {
        float* wp = &tr.estat[(nb + node) * E + ei].w;
        wb = __float_as_uint(*wp);
        if (o.virtual_loss > 0) *wp = __uint_as_float(wb + 1u);
        NodeHdr* hp = &tr.hdr[nb + node];
        hp->mean_q = new_mean;
        if (ei == (int)h.n_touched) hp->n_touched = (uint16_t)(h.n_touched + 1);
        // a tie resolved in favour of an edge beyond the first never-selected one: the selected edges
        // of this node are no longer a prefix, it is scanned in full from now on
        if (ei > (int)h.n_touched && !(h.flags & NF_FULLSCAN)) hp->flags = h.flags | NF_FULLSCAN;
        path[depth] = (uint32_t)node | (is_pass ? 0x10000u : 0u);
      }
      wb = __shfl_sync(FULL, wb, 0);
      int child = wb >> 16;
      // ---- allocateState for a new child ------------------------------------------------------------
      if (child == NONE16) {
        int id = 0, action = 0;
        if (L.lane == 0) {
          id = pop_free(tr, g);
          action = tr.elink[(nb + node) * E + ei] & 0xFFFFu;
        }
        id = __shfl_sync(FULL, id, 0);
        action = __shfl_sync(FULL, action, 0);
        if (id < 0) {  // cannot happen when k_begin reserved enough room
          if (L.lane == 0) atomicAdd(&tr.errors[1], 1);
          break;
        }
        child = id;
        st_new++;
        __syncwarp();
        // superko record along the path: the position before every stone move (go_state.cc:113-121)
        int cnt = nsk0;
        for (int d0 = 0; d0 <= depth; d0 += 32) {
          const int d = d0 + L.lane;
          const uint32_t pe = d <= depth ? path[d] : 0x10000u;
          const bool stone = !(pe & 0x10000u);
          const uint32_t bal = __ballot_sync(FULL, stone);
          if (stone) skg[cnt + __popc(bal & ((1u << L.lane) - 1u))] = tr.hash[nb + (pe & 0xFFFFu)];
          cnt += __popc(bal);
        }
        const uint64_t rowv = L.active ? tr.pos[(nb + node) * N + L.row] : 0ull;
        const uint64_t sav = L.active ? tr.sa[(nb + node) * N + L.row] : 0ull;
        uint32_t b = (uint32_t)rowv, w = (uint32_t)(rowv >> 32);
        uint32_t safe = (uint32_t)sav, atari = (uint32_t)(sav >> 32);
        BoardMeta meta = load_meta(&tr.meta[nb + node]);
        uint64_t hash = tr.hash[nb + node];
        const int pm = action == Geo<N>::P ? MV_PASS : (action % N) * N + action / N;
        __syncwarp();
        play_move_cached<N>(b, w, meta, hash, pm, s_zob, L, safe, atari);  // recounts only the groups the move touched
        if (pm >= 0 && superko_scan_warp(skg, cnt, hash)) meta.flags |= F_SUPERKO;
        if (L.active) {
          tr.pos[(nb + child) * N + L.row] = (uint64_t)b | ((uint64_t)w << 32);
          tr.sa[(nb + child) * N + L.row] = (uint64_t)safe | ((uint64_t)atari << 32);
        }
        if (L.lane == 0) {
          tr.hash[nb + child] = hash;
          store_meta(&tr.meta[nb + child], meta);
          NodeHdr c;
          c.num_visits = 0;
          c.V = 0.f;
          c.mean_q = new_mean;    // NodeT ctor: unsignedMeanQ_ = unsignedParentQ_
          c.parent_q = new_mean;  // followEdge: tree.addNode(unsignedMeanQ_)
          c.n_edges = 0;
          c.parent = (uint16_t)node;
          c.parent_edge = (uint16_t)ei;
          c.status = NS_UNVISITED;
          c.flags = 0;
          c.n_touched = 0;
          c.pass_edge = NONE16;
          c.pad = 0;
          store_hdr(&tr.hdr[nb + child], c);
          tr.elink[(nb + node) * E + ei] = (uint32_t)action | ((uint32_t)child << 16);
          float* wp = &tr.estat[(nb + node) * E + ei].w;
          *wp = __uint_as_float((__float_as_uint(*wp) & 0xFFFFu) | ((uint32_t)child << 16));
        }
      }
      __syncwarp();
      node = child;
      depth++;
    }
    // ---- leaf claim: requestEvaluation (tree_search_node.h:157-167) + pre_evaluate (mcts.h:185)
    const NodeHdr lh = load_hdr(&tr.hdr[nb + node]);
    __syncwarp();  // every lane has read the status before lane 0 changes it below (the branch holds collectives)
    if (lh.status == NS_UNVISITED) {
      const BoardMeta meta = load_meta(&tr.meta[nb + node]);
      if (is_terminated<N>(meta)) {
        // terminal: V = sign(evaluate(komi)) (go_state.h:194-203), no edges
        const uint64_t rowv = L.active ? tr.pos[(nb + node) * N + L.row] : 0ull;
        const int sc = tt_score<N>((uint32_t)rowv, (uint32_t)(rowv >> 32), L);
        float fv;
        if (meta.flags & F_SUPERKO)
          fv = meta.next == S_BLACK ? 1.0f : -1.0f;
        else
          fv = (float)sc - o.komi;
        if (L.lane == 0) {
          NodeHdr h2 = lh;
          h2.V = fv > 0 ? 1.0f : -1.0f;
          h2.flags = meta.next == S_WHITE ? NF_FLIP : 0;
          h2.status = NS_VISITED;
          h2.n_edges = 0;
          store_hdr(&tr.hdr[nb + node], h2);
        }
      } else {
        int slot = 0;
        uint8_t d4 = 0;
        if (L.lane == 0) {
          tr.hdr[nb + node].status = NS_REQUESTED;
          slot = atomicAdd(tr.eval_count, 1);
          tr.eval_game[slot] = g;
          tr.eval_node[slot] = (uint16_t)node;
          if (o.rotation_flip) {
            if (tr.d4_stream) {
              // one code per evaluated leaf, in descent order (MCTSActor::evaluate walks the claimed
              // leaves of a wave in trajectory order, go/mcts/mcts.h:86-93)
              const int u = tr.d4_used[g];
              d4 = tr.d4_stream[(size_t)g * tr.d4_cap + min(u, tr.d4_cap - 1)] & 7u;
              tr.d4_used[g] = u + 1;
            } else {
              d4 = (uint8_t)(pp_splitmix64(((uint64_t)o.seed << 40) ^ ((uint64_t)g << 20) ^
                                           ((uint64_t)wave << 8) ^ (uint64_t)node ^ tr.hash[nb + node]) & 7u);
            }
          }
          tr.eval_d4[slot] = d4;
        }
        slot = __shfl_sync(FULL, slot, 0);
        // The leaf's 8-position history for the feature writer, laid out contiguously per evaluation slot
        // (hist[slot][t][y]): the leaf, its ancestors along THIS descent's path (still in shared memory),
        // then the game's own ring (go_state.cc:90-92).  Done here because the descent is latency-bound
        // with idle issue slots: these scattered 152-byte reads over a multi-GB pool (TLB misses) cost the
        // select kernel almost nothing, and the plane writer then streams contiguous memory.
        const int hn = min(8, (int)meta.ply - 1);
        uint64_t* ho = tr.hist + (size_t)slot * 8 * N;
        if (L.active) {
#pragma unroll
          for (int t = 0; t < 8; ++t) {
            uint64_t v = 0;
            if (t < hn) {
              if (t <= depth) {
                const int src = t == 0 ? node : (int)(path[depth - t] & 0xFFFFu);
                v = tr.pos[(nb + src) * N + L.row];
              } else {
                v = st.ring[((size_t)g * 8 + ((rootply - 2 - (t - depth)) & 7)) * N + L.row];
              }
            }
            ho[t * N + L.row] = v;
          }
        }
        if (L.lane == 0) tr.hinfo[slot] = (uint32_t)hn | ((uint32_t)meta.next << 8) | ((uint32_t)d4 << 16);
      }
    }
    if (L.lane == 0) tr.leaves[(size_t)g * tr.B + j] = (uint16_t)node;
    __syncwarp();
  }
  if (L.lane == 0) {
    atomicAdd(&tr.stats[0], (unsigned long long)st_steps);
    atomicAdd(&tr.stats[1], (unsigned long long)st_edges);
    atomicAdd(&tr.stats[2], (unsigned long long)st_new);
    atomicAdd(&tr.stats[3], (unsigned long long)st_term);
  }
}

// ---------------------------------------------------------------------------------------
// BoardFeature::extractAGZ for every claimed leaf: the 8-position history is the leaf, its
// ancestors up to the root, then the game's own ring (go_state.cc:90-92).  Staging, output formats
// and the bulk store are features_cta's (common.cuh); the grid may be larger than the number of
// claimed leaves (device-side count), so a wave needs no host round trip before this launch.
// The history rows of every claimed leaf were laid out contiguously by k_select (hist[slot][t][y],
// 1,216 B per leaf, plus hinfo[slot]): the plane writer streams -- contiguous reads, coalesced 16-byte
// stores, exactly the board batch's k_features.
template <int N>
struct StagedGather {
  const uint64_t* hist;
  const uint32_t* hinfo;
  __device__ __forceinline__ void operator()(int slot, uint64_t (*rows)[N], int& hn, int& next, int& d4) const {
    const uint32_t hi = hinfo[slot];
    hn = (int)(hi & 0xFFu);
    next = (int)((hi >> 8) & 0xFFu);
    d4 = (int)((hi >> 16) & 0xFFu);
    const uint64_t* src = hist + (size_t)slot * 8 * N;
    for (int i = threadIdx.x; i < 8 * N; i += blockDim.x) (&rows[0][0])[i] = src[i];
  }
};

template <int N>
__global__ void __launch_bounds__(FEAT_THREADS)
    k_leaf_features(TreeDev tr, void* __restrict__ out, int fmt, int cpad, int tma) {
  features_cta<N>(StagedGather<N>{tr.hist, tr.hinfo}, *tr.eval_count, out, fmt, cpad, tma);
}

// ---------------------------------------------------------------------------------------
// BoardFeature::extract (the 25 DarkForest planes, GameOptions::use_df_feature) for every claimed leaf, in
// claim order and under the leaf's D4 code, so the rows line up with k_expand exactly as
// k_leaf_features' do.  One warp per leaf; the planes are df_planes' (common.cuh), shared with the board
// batch's k_features_df.
//
// Position and meta come from the leaf's node (not from hist: at a ply-1 root with handicap stones the
// AGZ history is empty by design, the DF stone and liberty planes are not).  The DF history planes need
// the ply every stone on the leaf's board was placed at (Info::last_placed).  The board batch holds the
// root position during a move, so `placed` starts as the board's array; then every non-pass node on the
// parent chain from the leaf up to (not including) the game's root placed a stone at meta.last1 at ply
// meta.ply - 1 -- what k_step writes.  The move nearest the leaf wins at each point; a stone with no move
// on the chain was on the board at the root.  Descents are at most MAX_DEPTH plies deep, which bounds the
// chain.  Shared memory: the 25*N*N float tile plus N*N 16-bit plies, about 37 KB at 19x19.
template <int N>
__global__ void __launch_bounds__(32)
    k_leaf_features_df(TreeDev tr, DevState st, const float* __restrict__ exp_tab, float* __restrict__ out) {
  constexpr int P = Geo<N>::P;
  __shared__ float tile[25 * P];
  __shared__ uint8_t hd[N][N];
  __shared__ uint16_t placed[P];
  __shared__ uint16_t chain[MAX_DEPTH + 1];
  __shared__ int16_t chain_pt[MAX_DEPTH + 1];
  __shared__ uint16_t chain_ply[MAX_DEPTH + 1];
  __shared__ int s_len;
  const Lane L = make_lane_single<N>();
  const int slot = blockIdx.x;
  if (slot >= *tr.eval_count) return;
  const int g = tr.eval_game[slot], node = tr.eval_node[slot], d4 = tr.eval_d4[slot];
  const size_t nb = (size_t)g * tr.C;
  const uint64_t rowv = L.active ? tr.pos[(nb + node) * N + L.row] : 0ull;
  const BoardMeta meta = load_meta(&tr.meta[nb + node]);
  for (int i = L.lane; i < P; i += 32) placed[i] = st.placed[(size_t)g * P + i];
  if (L.lane == 0) {  // leaf -> root: a chain of dependent parent reads
    const int root = tr.root[g];
    int nd = node, len = 0;
    while (nd != root && nd != NONE16 && len <= MAX_DEPTH) {
      chain[len++] = (uint16_t)nd;
      nd = tr.hdr[nb + nd].parent;
    }
    s_len = len;
  }
  __syncwarp();
  const int len = s_len;
  for (int i = L.lane; i < len; i += 32) {
    const BoardMeta m = load_meta(&tr.meta[nb + chain[i]]);
    chain_pt[i] = m.last1;
    chain_ply[i] = (uint16_t)(m.ply - 1);
  }
  __syncwarp();
  if (L.lane == 0)  // root side first, so the move nearest the leaf is written last
    for (int i = len - 1; i >= 0; --i)
      if (chain_pt[i] >= 0) placed[chain_pt[i]] = chain_ply[i];
  __syncwarp();
  df_planes<N>(L, (uint32_t)rowv, (uint32_t)(rowv >> 32), meta, d4, placed, exp_tab, tile, hd,
               out + (size_t)slot * 25 * P);
}

// ---------------------------------------------------------------------------------------
// Warp-wide bitonic sort of 32*R 64-bit keys held R per lane (key index i = lane*R + r), ascending.
// Compare-exchange distances below R stay inside a lane's registers (fully unrolled, static
// indices); larger distances exchange whole registers with the partner lane via SHFL.
template <int R>
__device__ __forceinline__ void warp_bitonic_sort(uint64_t (&key)[R], int lane) {
#pragma unroll
  for (int k = 2; k <= 32 * R; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      if (j >= R) {  // partner lane, same register
        const int lj = j / R;
        const bool lower = (lane & lj) == 0;
        const bool asc = k >= 32 * R ? true : ((lane & (k / R)) == 0);
        const bool keep_min = lower == asc;
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const uint64_t mine = key[r];
          const uint32_t olo = __shfl_xor_sync(FULL, (uint32_t)mine, lj);
          const uint32_t ohi = __shfl_xor_sync(FULL, (uint32_t)(mine >> 32), lj);
          const uint64_t other = ((uint64_t)ohi << 32) | olo;
          const bool mine_small = mine < other;
          key[r] = (mine_small == keep_min) ? mine : other;
        }
      } else {  // inside the lane
#pragma unroll
        for (int r = 0; r < R; ++r) {
          if ((r & j) == 0) {
            const int q = r | j;
            // ascending block iff bit k of the global index is clear
            const bool asc = k < R ? ((r & k) == 0) : (k >= 32 * R ? true : ((lane & (k / R)) == 0));
            const uint64_t a0 = key[r], a1 = key[q];
            const bool sw = (a0 > a1) == asc;
            key[r] = sw ? a1 : a0;
            key[q] = sw ? a0 : a1;
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------
// Expansion: MCTSActor::post_nn_result / remove_pass_if_dangerous / pi2response / normalize
// (go/mcts/mcts.h:209-332) + NodeT::setEvaluation (tree_search_node.h:176-203).  One warp per
// claimed leaf; the candidate list is bitonic-sorted in shared memory by descending probability.
// EXACT (option std_sort_ties): leaves whose reply holds two legal moves with bit-equal probabilities get
// their candidates in the order libstdc++'s std::sort leaves the reply's 362 pairs in (stdsort.cuh) instead
// of "equal probabilities by ascending move"; a separate instantiation, so that the default kernel's code
// and resources are exactly what they were.
template <int N, bool EXACT>
__global__ void __launch_bounds__(BLOCK)
    k_expand(DevState st, TreeDev tr, SearchOpts o, const float* __restrict__ pi, const float* __restrict__ val) {
  constexpr int P = Geo<N>::P;
  constexpr int SORTN = P + 1 <= 128 ? 128 : 512;
  __shared__ uint64_t s_key[WARPS][SORTN];
  __shared__ float s_tot[WARPS];
  __shared__ uint32_t s_legal[WARPS][N];
  const Lane L = make_lane_single<N>();
  const int wib = threadIdx.x >> 5;
  const int slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (slot >= *tr.eval_count) return;
  const int g = tr.eval_game[slot];
  const int node = tr.eval_node[slot];
  const int d4 = tr.eval_d4[slot];
  const size_t nb = (size_t)g * tr.C;
  const uint64_t rowv = L.active ? tr.pos[(nb + node) * N + L.row] : 0ull;
  const uint64_t sav = L.active ? tr.sa[(nb + node) * N + L.row] : 0ull;
  const uint32_t b = (uint32_t)rowv, w = (uint32_t)(rowv >> 32);
  const BoardMeta meta = load_meta(&tr.meta[nb + node]);
  const uint32_t own = meta.next == S_BLACK ? b : w, opp = meta.next == S_BLACK ? w : b;
  const bool ko_applies = (meta.flags & F_KO_ACTIVE) && meta.ko_color == meta.next;
  // legality straight from the node's incremental safe/atari masks (no group classification fills)
  const uint32_t legal = legal_rows_cached<N>(own, opp, (uint32_t)sav, (uint32_t)(sav >> 32), L, ko_applies, meta.ko_pt);
  // pass handling (mcts.h:225-242)
  bool pass_enabled = (int)meta.ply >= o.ply_pass_enabled;
  if (o.remove_pass_if_dangerous && pass_enabled && meta.last1 != MV_PASS) {
    // (per-game reductions are only defined on the game's own lanes: take lane 0's copy)
    const int sc = __shfl_sync(FULL, tt_score<N>(b, w, L), 0);
    const bool black_win = ((float)sc - o.komi) > 0;
    if ((black_win && meta.next == S_WHITE) || (!black_win && meta.next == S_BLACK)) pass_enabled = false;
  }
  // candidates: NN action a -> board action through the inverse D4 (board_feature.h:139-144)
  if (L.active) s_legal[wib][L.row] = legal;
  __syncwarp();
  uint64_t* key = s_key[wib];
  const float* pr = pi + (size_t)slot * (P + 1);
  constexpr int R = SORTN / 32;  // keys per lane
  uint64_t kr[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int a = L.lane + 32 * r;  // any assignment of candidates to slots will do before sorting
    uint64_t k = ~0ull;
    if (a <= P) {
      int act;
      bool ok;
      if (a == P) {
        act = P;
        ok = pass_enabled;
      } else {
        int x, y;
        d4_inverse(N, d4, a / N, a - (a / N) * N, x, y);
        act = x * N + y;
        ok = (s_legal[wib][y] >> x) & 1u;
      }
      // probabilities are non-negative floats: their bit patterns order like the values
      if (ok) k = ((uint64_t)(0xFFFFFFFFu - __float_as_uint(pr[a])) << 32) | (uint32_t)act;
    }
    kr[r] = k;
  }
  // ascending on the composite key == descending probability, then action
  int nvalid = 0;
#pragma unroll
  for (int r = 0; r < R; ++r) nvalid += kr[r] != ~0ull;
  nvalid = __reduce_add_sync(FULL, nvalid);
  constexpr int RH = R / 2;  // half-size network: the sort costs O(n log^2 n)
  if (R >= 8 && nvalid <= 32 * RH) {
    // at most half the slots hold a candidate (every 19x19 position past the opening: <= 256 legal moves):
    // compact them (ballot prefix, any order -- the sort follows) and run the half-size network, 2.5x cheaper
    int base = 0;
    const uint32_t lt = (1u << L.lane) - 1u;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const bool v = kr[r] != ~0ull;
      const uint32_t bal = __ballot_sync(FULL, v);
      if (v) key[base + __popc(bal & lt)] = kr[r];
      base += __popc(bal);
    }
    for (int i = nvalid + L.lane; i < 32 * RH; i += 32) key[i] = ~0ull;
    __syncwarp();
    uint64_t kh[RH > 0 ? RH : 1];
#pragma unroll
    for (int r = 0; r < RH; ++r) kh[r] = key[L.lane * RH + r];
    __syncwarp();
    warp_bitonic_sort<(RH > 0 ? RH : 1)>(kh, L.lane);
#pragma unroll
    for (int r = 0; r < RH; ++r) key[L.lane * RH + r] = kh[r];
  } else {
    warp_bitonic_sort<R>(kr, L.lane);
#pragma unroll
    for (int r = 0; r < R; ++r) key[L.lane * R + r] = kr[r];
  }
  __syncwarp();
  if constexpr (EXACT) {
    // probability bits, sort order and (validity << 15 | move), all by NETWORK action index
    __shared__ uint32_t s_pb[WARPS][P + 1];
    __shared__ uint16_t s_ord[WARPS][P + 2];
    __shared__ uint16_t s_act[WARPS][P + 2];
    // two candidates with the same probability bits are neighbours in the sorted list
    bool tie = false;
    for (int i = L.lane + 1; i < nvalid; i += 32) tie |= (uint32_t)(key[i] >> 32) == (uint32_t)(key[i - 1] >> 32);
    if (__any_sync(FULL, tie)) {
      // pi2response: all P+1 pairs in network-action order, std::sort by probability, THEN the legality filter
      for (int a = L.lane; a <= P; a += 32) {
        int act = P;
        bool ok = pass_enabled;
        if (a < P) {
          int x, y;
          d4_inverse(N, d4, a / N, a - (a / N) * N, x, y);
          act = x * N + y;
          ok = (s_legal[wib][y] >> x) & 1u;
        }
        s_pb[wib][a] = __float_as_uint(pr[a]);
        s_ord[wib][a] = (uint16_t)a;
        s_act[wib][a] = (uint16_t)(act | (ok ? 0x8000 : 0));
      }
      __syncwarp();
      if (L.lane == 0) {
        StdSortCtx sc{s_pb[wib]};
        ss_sort(&sc, s_ord[wib], P + 1);
        int k = 0;
        for (int i = 0; i <= P; ++i) {
          const int a = s_ord[wib][i];
          const uint16_t av = s_act[wib][a];
          if (av & 0x8000) key[k++] = ((uint64_t)(0xFFFFFFFFu - s_pb[wib][a]) << 32) | (uint32_t)(av & 0x7FFF);
        }
      }
      __syncwarp();
    }
  }
  // sequential float sum in sorted order (normalize, mcts.h:244-254)
  if (L.lane == 0) {
    float tot = 1e-10f;
    for (int i = 0; i < nvalid; ++i) tot += __uint_as_float(0xFFFFFFFFu - (uint32_t)(key[i] >> 32));
    s_tot[wib] = tot;
  }
  __syncwarp();
  const float tot = s_tot[wib];
  const int E = tr.E;
  float4* es = tr.estat + (nb + node) * E;
  uint32_t* el = tr.elink + (nb + node) * E;
  int n_edges = nvalid;
  if (nvalid == 0 && !pass_enabled) {  // mcts.h:324-327: pass with probability 1
    n_edges = 1;
    if (L.lane == 0) {
      es[0] = make_float4(1.0f / (1e-10f + 1.0f), __int_as_float(0), 0.f, __uint_as_float(0xFFFF0000u));
      el[0] = (uint32_t)P | ((uint32_t)NONE16 << 16);
    }
  } else {
    for (int i = L.lane; i < nvalid; i += 32) {
      const uint64_t k = key[i];
      const float p = __uint_as_float(0xFFFFFFFFu - (uint32_t)(k >> 32));
      es[i] = make_float4(p / tot, __int_as_float(0), 0.f, __uint_as_float(0xFFFF0000u));
      el[i] = (uint32_t)(k & 0xFFFFu) | ((uint32_t)NONE16 << 16);
    }
  }
  // index of the pass edge (if any) for the descent's pass test
  int pass_idx = 0x7FFFFFFF;
  if (nvalid == 0 && !pass_enabled) {
    pass_idx = 0;
  } else {
    for (int i = L.lane; i < nvalid; i += 32)
      if ((int)(key[i] & 0xFFFFu) == P) pass_idx = i;
  }
  pass_idx = __reduce_min_sync(FULL, pass_idx);
  __syncwarp();
  if (L.lane == 0) {
    NodeHdr h = load_hdr(&tr.hdr[nb + node]);
    h.V = val[slot];
    h.flags = meta.next == S_WHITE ? NF_FLIP : 0;  // q_flip, mcts.h:186
    h.n_edges = (uint16_t)n_edges;
    h.n_touched = 0;
    h.pass_edge = pass_idx == 0x7FFFFFFF ? NONE16 : (uint16_t)pass_idx;
    h.status = NS_VISITED;
    store_hdr(&tr.hdr[nb + node], h);
  }
}

// ---------------------------------------------------------------------------------------
// Backup: batch_rollouts' second half (tree_search.h:245-259) + NodeT::updateEdgeStats
// (tree_search_node.h:253-278).  One unique leaf = one visit; duplicates only return their
// virtual loss.  One warp per game, one lane per rollout of the wave: the lanes climb their paths
// in lock step by ply (deepest first); lanes standing on the same node form a group
// (__match_any_sync) whose lowest lane applies the group's rewards to the edge above IN LANE
// ORDER -- the same float additions, in the same order, as backing the unique leaves up one after
// the other in first-occurrence order.
__global__ void __launch_bounds__(BLOCK) k_backup(int G, TreeDev tr, int virtual_loss) {
  __shared__ float s_rew[WARPS][32];
  __shared__ int s_cnt[WARPS][32];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (blockIdx.x == 0 && threadIdx.x == 0) tr.stats[4] += (unsigned long long)*tr.eval_count;  // evaluations so far
  if (g >= G || !tr.active[g]) return;
  const size_t nb = (size_t)g * tr.C;
  const int B = tr.B, E = tr.E;
  const uint16_t* lv = tr.leaves + (size_t)g * B;
  const int root = tr.root[g];
  const int rootply = tr.meta[nb + root].ply;
  for (int c0 = 0; c0 < B; c0 += 32) {
    const int j = c0 + lane;
    const bool has = j < B;
    const int leaf = has ? (int)lv[j] : -1;
    int count = 0;
    bool first = has;
    if (has)
      for (int k = 0; k < B; ++k) {
        if ((int)lv[k] == leaf) {
          if (k < j) first = false;
          count++;
        }
      }
    bool act = has && first;
    s_rew[wib][lane] = act ? tr.hdr[nb + leaf].V : 0.f;
    s_cnt[wib][lane] = count;
    __syncwarp();
    int node = act ? leaf : -1;
    int ply = act ? (int)tr.meta[nb + leaf].ply : -1;
    int maxply = ply;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) maxply = max(maxply, __shfl_xor_sync(FULL, maxply, d));
    for (int P = maxply; P > rootply; --P) {
      const bool on = act && ply == P;
      int par = NONE16, pedge = 0;
      if (on) {
        const NodeHdr h = load_hdr(&tr.hdr[nb + node]);
        par = h.parent;
        pedge = h.parent_edge;
      }
      const unsigned grp = __match_any_sync(FULL, on ? node : -1 - lane);
      if (on && (__ffs(grp) - 1) == lane && par != NONE16) {
        float4 e = tr.estat[(nb + par) * E + pedge];
        float wsum = e.z;
        int m = 0, cnt = 0;
        for (unsigned mm = grp; mm; mm &= mm - 1) {
          const int l = __ffs(mm) - 1;
          wsum += s_rew[wib][l];
          cnt += s_cnt[wib][l];
          m++;
        }
        e.z = wsum;
        e.y = __int_as_float(__float_as_int(e.y) + m);
        e.w = __uint_as_float(__float_as_uint(e.w) - (virtual_loss > 0 ? (uint32_t)cnt : 0u));
        tr.estat[(nb + par) * E + pedge] = e;
        atomicAdd(&tr.hdr[nb + par].num_visits, m);  // siblings' leaders may share the parent
      }
      if (on) {
        node = par;
        ply = P - 1;
        if (par == NONE16) act = false;
      }
      __syncwarp();
    }
    __syncwarp();
  }
}

// most visited root edge (first maximum in the reference's container order) and the visit total
template <int N>
__device__ __forceinline__ void root_best(const uint32_t* __restrict__ el, const float4* __restrict__ es, int ne,
                                          OrderScratch& scratch, int lane, int& besti, int& tot) {
  int bestn = -1;
  besti = 0x7FFFFFFF;
  tot = 0;
  for (int i = lane; i < ne; i += 32) {
    const int n = __float_as_int(es[i].y);
    tot += n;
    if (n > bestn) {
      bestn = n;
      besti = i;
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const int on = __shfl_xor_sync(FULL, bestn, d), oi = __shfl_xor_sync(FULL, besti, d);
    if (on > bestn || (on == bestn && oi < besti)) {
      bestn = on;
      besti = oi;
    }
    tot += __shfl_xor_sync(FULL, tot, d);
  }
  int ties = 0;
  for (int i = lane; i < ne; i += 32) ties += __float_as_int(es[i].y) == bestn;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) ties += __shfl_xor_sync(FULL, ties, d);
  if (ties > 1) besti = first_max_in_container_order<N>(el, es, ne, bestn, scratch, lane);
  __syncwarp();
}

// ---------------------------------------------------------------------------------------
// Results at the root: TreeSearchT::chooseAction / MCTSResultT::addActions (most_visited,
// tree_search.h:495-528, tree_search_base.h:237-294) and MCTSGoAI::getValue (go/mcts/mcts.h:358).
template <int N>
__global__ void __launch_bounds__(BLOCK)
    k_results(int G, TreeDev tr, int32_t* __restrict__ best_action, int32_t* __restrict__ visits,
              float* __restrict__ root_value, float* __restrict__ best_q, int32_t* __restrict__ total_visits) {
  constexpr int P1 = Geo<N>::P + 1;
  __shared__ OrderScratch scratch[BLOCK / 32];
  const int lane = threadIdx.x & 31;
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= G) return;
  if (visits)
    for (int a = lane; a < P1; a += 32) visits[(size_t)g * P1 + a] = -1;
  __syncwarp();
  const int root = tr.root[g];
  if (!tr.active[g] || root == NONE16) {
    if (lane == 0) {
      if (best_action) best_action[g] = -1;
      if (root_value) root_value[g] = 0.f;
      if (best_q) best_q[g] = 0.f;
      if (total_visits) total_visits[g] = 0;
    }
    return;
  }
  const size_t nb = (size_t)g * tr.C;
  const NodeHdr h = load_hdr(&tr.hdr[nb + root]);
  const float4* es = tr.estat + (nb + root) * tr.E;
  const uint32_t* el = tr.elink + (nb + root) * tr.E;
  if (visits)
    for (int i = lane; i < h.n_edges; i += 32) visits[(size_t)g * P1 + (el[i] & 0xFFFFu)] = __float_as_int(es[i].y);
  int besti, tot;
  root_best<N>(el, es, h.n_edges, scratch[threadIdx.x >> 5], lane, besti, tot);
  if (lane == 0) {
    const bool any = h.n_edges > 0 && besti != 0x7FFFFFFF;
    if (best_action) best_action[g] = any ? (int)(el[besti] & 0xFFFFu) : -1;
    if (root_value) root_value[g] = h.V;
    if (total_visits) total_visits[g] = tot;
    if (best_q) {
      float q = h.V;
      if (any && tot > 0) {
        const float4 e = es[besti];
        q = e.z / (float)__float_as_int(e.y);  // EdgeInfo::getQSA
      }
      best_q[g] = q;
    }
  }
}

// ---------------------------------------------------------------------------------------
__device__ __forceinline__ float rng_u01(uint64_t key, uint32_t& ctr);  // defined with the root noise below

// Move choice for every game: GoGameSelfPlay::mcts_make_diverse_move / shouldResign
// (common/game_selfplay.cc:80-95,387-391; game_utils.h:15-54) on the root statistics.
//   ply <= policy_distri_cutoff : sample the move from the visit distribution
//       (MCTSPolicy::sampleAction -> elf_utils::sample_multinomial, elf/utils/utils.h:158-181:
//        rd uniform in [0, sum N), first edge whose running sum exceeds rd);
//   otherwise                   : the most visited edge (first maximum in the reference's container order);
//   resign (action -1)          : the side to move's value (best edge W/N, root V if unvisited) is
//       below -1 + resign_thres, ply >= 50, and the game is not one of the never-resign games.
// The uniform comes from a counter-based generator (seed, game, ply): same distribution as the
// reference's per-game mt19937, different stream.  One warp per game.
template <int N>
__device__ __forceinline__ void choose_game(const DevState& st, const TreeDev& tr, int cutoff, float resign_thres,
                                            const uint8_t* __restrict__ never_resign, uint64_t seed,
                                            int32_t* __restrict__ action_out, float* __restrict__ value_out,
                                            OrderScratch* scratch) {
  const int lane = threadIdx.x & 31;
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= st.G) return;
  const int root = tr.root[g];
  if (!tr.active[g] || root == NONE16) {
    if (lane == 0) {
      action_out[g] = -2;  // not searched this move
      if (value_out) value_out[g] = 0.f;
    }
    return;
  }
  const size_t nb = (size_t)g * tr.C;
  const NodeHdr h = load_hdr(&tr.hdr[nb + root]);
  const BoardMeta meta = load_meta(&st.meta[g]);
  const float4* es = tr.estat + (nb + root) * tr.E;
  const uint32_t* el = tr.elink + (nb + root) * tr.E;
  // most visited (first maximum in the reference's container order) + total
  int besti, tot;
  root_best<N>(el, es, h.n_edges, scratch[threadIdx.x >> 5], lane, besti, tot);
  int pick = besti;
  if ((int)meta.ply <= cutoff && tot > 0) {
    uint32_t ctr = 0;
    const uint64_t key = pp_splitmix64(seed ^ ((uint64_t)g << 24) ^ (uint64_t)meta.ply ^ (st.hash[g] << 1));
    const float rd = rng_u01(key, ctr) * (float)tot;
    // running sums in edge order: chunked warp scan
    int base = 0, found = 0x7FFFFFFF;
    for (int i0 = 0; i0 < h.n_edges && found == 0x7FFFFFFF; i0 += 32) {
      const int i = i0 + lane;
      int v = i < h.n_edges ? __float_as_int(es[i].y) : 0;
      int incl = v;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(FULL, incl, d);
        if (lane >= d) incl += t;
      }
      const bool hit = i < h.n_edges && rd < (float)(base + incl);
      const unsigned bal = __ballot_sync(FULL, hit);
      if (bal) found = i0 + __ffs(bal) - 1;
      base += __shfl_sync(FULL, incl, 31);
    }
    pick = found != 0x7FFFFFFF ? found : (int)h.n_edges - 1;  // sample_multinomial's fall-through
  }
  if (lane == 0) {
    float q = h.V;  // MCTSGoAI::getValue (go/mcts/mcts.h:358-365)
    if (besti != 0x7FFFFFFF && tot > 0) {
      const float4 e = es[besti];
      q = e.z / (float)__float_as_int(e.y);
    }
    const float side = meta.next == S_BLACK ? q : -q;  // GoStateExt::shouldResign, go_state_ext.h:207-214
    const bool nr = never_resign && never_resign[g];
    const bool resign = !nr && side < -1.0f + resign_thres && (int)meta.ply >= 50;
    int a = -1;
    if (!resign) a = (h.n_edges > 0 && pick != 0x7FFFFFFF) ? (int)(el[pick] & 0xFFFFu) : -2;
    action_out[g] = a;
    if (value_out) value_out[g] = q;
  }
}

template <int N>
__global__ void __launch_bounds__(BLOCK)
    k_choose(DevState st, TreeDev tr, int cutoff, float resign_thres, const uint8_t* __restrict__ never_resign,
             uint64_t seed, int32_t* __restrict__ action_out, float* __restrict__ value_out) {
  __shared__ OrderScratch scratch[BLOCK / 32];
  choose_game<N>(st, tr, cutoff, resign_thres, never_resign, seed, action_out, value_out, scratch);
}

// elfb200_mcts_choose_dev: the seed read from device memory, so that a graph replay draws with the seed the
// caller's device counter holds at that point, not the value it had when the graph was captured.
template <int N>
__global__ void __launch_bounds__(BLOCK)
    k_choose(DevState st, TreeDev tr, int cutoff, float resign_thres, const uint8_t* __restrict__ never_resign,
             const int64_t* __restrict__ seed, int32_t* __restrict__ action_out, float* __restrict__ value_out) {
  __shared__ OrderScratch scratch[BLOCK / 32];
  choose_game<N>(st, tr, cutoff, resign_thres, never_resign, (uint64_t)*seed, action_out, value_out, scratch);
}

// ---------------------------------------------------------------------------------------
// SearchTreeT::treeAdvance (tree_search_node.h:420-436): keep the subtree under the played move,
// free everything else.  One warp per game; BFS over the kept subtree marks it, one sweep frees
// the rest and rebuilds the free stack.
__global__ void __launch_bounds__(BLOCK)
    k_advance(int G, TreeDev tr, const int32_t* __restrict__ actions, int persistent) {
  const int lane = threadIdx.x & 31;
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= G) return;
  const int a = actions[g];
  if (a < 0) return;  // game untouched
  const size_t nb = (size_t)g * tr.C;
  const int E = tr.E, C = tr.C;
  const int root = tr.root[g];
  int keep = NONE16;
  if (root != NONE16 && persistent) {
    const NodeHdr h = load_hdr(&tr.hdr[nb + root]);
    const uint32_t* el = tr.elink + (nb + root) * E;
    int found = NONE16;
    for (int i = lane; i < h.n_edges; i += 32) {
      const uint32_t l = el[i];
      if ((int)(l & 0xFFFFu) == a) found = l >> 16;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) found = min(found, __shfl_xor_sync(FULL, found, d));
    keep = found;
  }
  uint16_t* q = tr.bfs_q + nb;
  if (keep != NONE16) {
    int head = 0, tail = 1;
    if (lane == 0) {
      q[0] = (uint16_t)keep;
      tr.hdr[nb + keep].flags |= NF_KEEP;
      tr.hdr[nb + keep].parent = NONE16;
    }
    __syncwarp();
    while (head < tail) {
      const int node = q[head++];
      const int ne = tr.hdr[nb + node].n_edges;
      const uint32_t* el = tr.elink + (nb + node) * E;
      for (int i0 = 0; i0 < ne; i0 += 32) {
        const int i = i0 + lane;
        int child = NONE16;
        if (i < ne) child = el[i] >> 16;
        const bool has = child != NONE16;
        const uint32_t bal = __ballot_sync(FULL, has);
        if (has) {
          q[tail + __popc(bal & ((1u << lane) - 1u))] = (uint16_t)child;
          tr.hdr[nb + child].flags |= NF_KEEP;
        }
        tail += __popc(bal);
      }
      __syncwarp();
    }
  }
  __syncwarp();
  // sweep: everything not kept becomes free
  int nfree = 0;
  for (int i0 = 0; i0 < C; i0 += 32) {
    const int i = i0 + lane;
    bool fr = false;
    if (i < C) {
      NodeHdr* hp = &tr.hdr[nb + i];
      const uint8_t fl = hp->flags;
      if (fl & NF_KEEP) {
        hp->flags = fl & ~NF_KEEP;
      } else {
        hp->status = NS_FREE;
        fr = true;
      }
    }
    const uint32_t bal = __ballot_sync(FULL, fr);
    if (fr) tr.free_list[nb + nfree + __popc(bal & ((1u << lane) - 1u))] = (uint16_t)i;
    nfree += __popc(bal);
  }
  if (lane == 0) {
    tr.free_n[g] = nfree;
    tr.root[g] = (uint16_t)keep;
  }
}

// ---------------------------------------------------------------------------------------
// Root exploration noise: NodeT::enhanceExploration (tree_search_node.h:132-155), applied by
// TreeSearchT::run (tree_search.h:413-417) to a root that already has edges:
//   P_i <- (1 - eps) P_i + eps * eta_i / (1e-10 + sum eta),  eta_i ~ Gamma(alpha, 1).
// The reference draws from std::gamma_distribution on the actor's mt19937; here eta comes from a
// counter-based generator (Marsaglia-Tsang on splitmix64 uniforms), so the distribution is the
// same and the stream is not.  Afterwards the root's priors are no longer sorted: the node is
// flagged for a full PUCT scan.
__device__ __forceinline__ float rng_u01(uint64_t key, uint32_t& ctr) {
  const uint64_t r = pp_splitmix64(key + 0x9E3779B97F4A7C15ULL * (uint64_t)(ctr++));
  return ((float)(r >> 40) + 0.5f) * (1.0f / 16777216.0f);  // (0, 1)
}

__device__ __forceinline__ float rng_gamma(float a, uint64_t key, uint32_t& ctr) {
  float boost = 1.f;
  if (a < 1.f) {
    boost = powf(rng_u01(key, ctr), 1.f / a);
    a += 1.f;
  }
  const float d = a - 1.f / 3.f, c = rsqrtf(9.f * d);
  for (int it = 0; it < 64; ++it) {
    const float u1 = rng_u01(key, ctr), u2 = rng_u01(key, ctr);
    const float x = sqrtf(-2.f * logf(u1)) * cospif(2.f * u2);
    float v = 1.f + c * x;
    if (v <= 0.f) continue;
    v = v * v * v;
    const float u = rng_u01(key, ctr);
    if (logf(u) < 0.5f * x * x + d - d * v + d * logf(v)) return d * v * boost;
  }
  return d * boost;
}

__device__ __forceinline__ void root_noise(int G, const TreeDev& tr, float eps, float alpha, uint64_t seed,
                                           uint32_t move_counter) {
  const int lane = threadIdx.x & 31;
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= G || !tr.active[g]) return;
  const int root = tr.root[g];
  if (root == NONE16) return;
  const size_t nb = (size_t)g * tr.C;
  const NodeHdr h = load_hdr(&tr.hdr[nb + root]);
  if (h.status != NS_VISITED || h.n_edges == 0) return;
  float4* es = tr.estat + (nb + root) * tr.E;
  float z = 0.f;
  for (int i = lane; i < h.n_edges; i += 32) {
    uint32_t ctr = 0;
    const uint64_t key = pp_splitmix64(seed ^ ((uint64_t)g << 32) ^ ((uint64_t)move_counter << 12) ^ (uint64_t)i);
    const float eta = rng_gamma(alpha, key, ctr);
    z += eta;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) z += __shfl_xor_sync(FULL, z, d);
  z += 1e-10f;
  for (int i = lane; i < h.n_edges; i += 32) {
    uint32_t ctr = 0;
    const uint64_t key = pp_splitmix64(seed ^ ((uint64_t)g << 32) ^ ((uint64_t)move_counter << 12) ^ (uint64_t)i);
    const float eta = rng_gamma(alpha, key, ctr);
    es[i].x = (1.f - eps) * es[i].x + eps * eta / z;
  }
  if (lane == 0) tr.hdr[nb + root].flags |= NF_FULLSCAN;
}

__global__ void __launch_bounds__(BLOCK)
    k_root_noise(int G, TreeDev tr, float eps, float alpha, uint64_t seed, uint32_t move_counter) {
  root_noise(G, tr, eps, alpha, seed, move_counter);
}

// elfb200_mcts_begin_move_dev: the move index read from device memory, so that every replay of a captured move
// draws the noise of the move the caller's counter holds, as the host form draws that of its host counter.
__global__ void __launch_bounds__(BLOCK)
    k_root_noise(int G, TreeDev tr, float eps, float alpha, uint64_t seed, const int64_t* __restrict__ move) {
  root_noise(G, tr, eps, alpha, seed, (uint32_t)*move);
}

__global__ void __launch_bounds__(BLOCK) k_root_priors(int G, TreeDev tr, float* __restrict__ out, int P1) {
  const int lane = threadIdx.x & 31;
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= G) return;
  for (int a = lane; a < P1; a += 32) out[(size_t)g * P1 + a] = -1.f;
  __syncwarp();
  const int root = tr.root[g];
  if (root == NONE16) return;
  const size_t nb = (size_t)g * tr.C;
  const int ne = tr.hdr[nb + root].n_edges;
  for (int i = lane; i < ne; i += 32)
    out[(size_t)g * P1 + (tr.elink[(nb + root) * tr.E + i] & 0xFFFFu)] = tr.estat[(nb + root) * tr.E + i].x;
}

// Root edges in STORAGE order (= the order pi2response produced them, go/mcts/mcts.h:255-332):
// action, N, W, P per edge and the edge count (0 for a root that is missing or not expanded yet).
__global__ void __launch_bounds__(BLOCK)
    k_root_edges(int G, TreeDev tr, int32_t* __restrict__ n_out, int16_t* __restrict__ act, int32_t* __restrict__ vis,
                 float* __restrict__ wsum, float* __restrict__ pri, int P1) {
  const int lane = threadIdx.x & 31;
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= G) return;
  const int root = tr.root[g];
  const size_t nb = (size_t)g * tr.C;
  int ne = 0;
  if (root != NONE16 && tr.hdr[nb + root].status == NS_VISITED) ne = tr.hdr[nb + root].n_edges;
  if (lane == 0) n_out[g] = ne;
  for (int i = lane; i < P1; i += 32) {
    const bool in = i < ne;
    const float4 e = in ? tr.estat[(nb + root) * tr.E + i] : make_float4(0.f, 0.f, 0.f, 0.f);
    const size_t o = (size_t)g * P1 + i;
    act[o] = in ? (int16_t)(tr.elink[(nb + root) * tr.E + i] & 0xFFFFu) : (int16_t)-1;
    vis[o] = in ? __float_as_int(e.y) : 0;
    wsum[o] = e.z;
    pri[o] = e.x;
  }
}

// New priors for the root edges (storage order) of the selected games: the device end of a root
// noise computed by the caller (elfb200_refstream_root_noise).  The priors are no longer sorted, so
// the node is flagged for a full PUCT scan like after k_root_noise.
__global__ void __launch_bounds__(BLOCK)
    k_set_root_priors(int G, TreeDev tr, const uint8_t* __restrict__ mask, const float* __restrict__ pri, int P1) {
  const int lane = threadIdx.x & 31;
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= G || (mask && !mask[g])) return;
  const int root = tr.root[g];
  if (root == NONE16) return;
  const size_t nb = (size_t)g * tr.C;
  if (tr.hdr[nb + root].status != NS_VISITED) return;
  const int ne = tr.hdr[nb + root].n_edges;
  if (ne == 0) return;
  for (int i = lane; i < ne; i += 32) tr.estat[(nb + root) * tr.E + i].x = pri[(size_t)g * P1 + i];
  if (lane == 0) tr.hdr[nb + root].flags |= NF_FULLSCAN;
}

__global__ void k_tree_reset(int G, TreeDev tr, const uint8_t* __restrict__ mask) {
  const int lane = threadIdx.x & 31;
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= G) return;
  if (mask && !mask[g]) return;
  const size_t nb = (size_t)g * tr.C;
  for (int i = lane; i < tr.C; i += 32) {
    tr.free_list[nb + i] = (uint16_t)(tr.C - 1 - i);
    tr.hdr[nb + i].status = NS_FREE;
    tr.hdr[nb + i].flags = 0;
  }
  if (lane == 0) {
    tr.free_n[g] = tr.C;
    tr.root[g] = NONE16;
  }
}

// ---------------------------------------------------------------------------------------
// Copy search trees from another handle's pool (elfb200_mcts_gather): destination game i gets an exact replica
// of source game index[i]'s tree for index[i] in [0, G_src); any other value leaves game i as it is.  Local ids
// are kept, so nothing is renumbered: the root, the free stack free_list[0 .. free_n) verbatim (later
// allocations pop the same ids), and for every in-use node (status != NS_FREE) its pos / sa rows, hash, meta
// and header; for every visited node the edges [0, n_edges) of estat and elink.  Free slots and edges past
// n_edges are not copied: no kernel reads them (DESIGN §3 "Copying games").  A slot the source has free only
// gets status NS_FREE, as k_advance / free_subtree leave freed slots: every slot on the free stack and no
// other is NS_FREE, which a later copy of this tree and elfb200_mcts_tree_usage rely on.
// One CTA per destination game (1.4x faster than one warp per game on an H100, DESIGN §5.2); warp w takes the
// 32-node chunks w, w + 8, ...: each lane reads one node's header and copies that node's small records, the
// warp copies the chunk's position rows (contiguous) and then the edges of each visited node, up to four
// 16-byte records per lane in flight.
constexpr int TREE_GATHER_THREADS = 256;

template <class T>
__device__ __forceinline__ void copy_run(T* __restrict__ d, const T* __restrict__ s, int n, int lane) {
  int i = lane;
  for (; i + 96 < n; i += 128) {
    const T a = __ldg(s + i), b = __ldg(s + i + 32), c = __ldg(s + i + 64), e = __ldg(s + i + 96);
    d[i] = a;
    d[i + 32] = b;
    d[i + 64] = c;
    d[i + 96] = e;
  }
  for (; i < n; i += 32) d[i] = __ldg(s + i);
}

template <int N>
__global__ void __launch_bounds__(TREE_GATHER_THREADS)
    k_gather_trees(TreeDev dst, TreeDev src, int G_dst, int G_src, const int32_t* __restrict__ index) {
  const int gd = blockIdx.x;
  if (gd >= G_dst) return;
  const int gs = __ldg(index + gd);
  if (gs < 0 || gs >= G_src) return;
  const int C = dst.C, E = dst.E;
  const size_t nd = (size_t)gd * C, ns = (size_t)gs * C;
  const int lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int nfree = min(max(__ldg(src.free_n + gs), 0), C);
  for (int i = threadIdx.x; i < nfree; i += blockDim.x) dst.free_list[nd + i] = __ldg(src.free_list + ns + i);
  if (threadIdx.x == 0) {
    dst.free_n[gd] = nfree;
    dst.root[gd] = __ldg(src.root + gs);
  }
  for (int c0 = (threadIdx.x >> 5) * 32; c0 < C; c0 += nwarps * 32) {
    const int v = c0 + lane;
    NodeHdr h = {};
    if (v < C) h = load_hdr(&src.hdr[ns + v]);
    const bool used = v < C && h.status != NS_FREE;
    const int ne = used && h.status == NS_VISITED ? min((int)h.n_edges, E) : 0;
    const uint32_t used_mask = __ballot_sync(FULL, used), vis_mask = __ballot_sync(FULL, ne > 0);
    if (used) {
      store_hdr(&dst.hdr[nd + v], h);
      dst.hash[nd + v] = __ldg(src.hash + ns + v);
      store_meta(&dst.meta[nd + v], load_meta(&src.meta[ns + v]));
    } else if (v < C) {
      dst.hdr[nd + v].status = NS_FREE;  // the pool's invariant: exactly the slots on the free stack are NS_FREE
    }
    // position and group-status rows of the chunk's in-use nodes: 32 N contiguous words each
    const int nrow = min(32, C - c0) * N;
    for (int k = lane; k < nrow; k += 32) {
      if ((used_mask >> (k / N)) & 1u) {
        dst.pos[(nd + c0) * N + k] = __ldg(src.pos + (ns + c0) * N + k);
        dst.sa[(nd + c0) * N + k] = __ldg(src.sa + (ns + c0) * N + k);
      }
    }
    // edges of the visited nodes: estat in 16-byte records, elink in pairs (its rows are 8-byte aligned)
    for (uint32_t m = vis_mask; m; m &= m - 1) {
      const int l = __ffs(m) - 1;
      const int cnt = __shfl_sync(FULL, ne, l);
      const size_t od = (nd + c0 + l) * E, os = (ns + c0 + l) * E;
      copy_run(dst.estat + od, src.estat + os, cnt, lane);
      copy_run(reinterpret_cast<uint2*>(dst.elink + od), reinterpret_cast<const uint2*>(src.elink + os), cnt >> 1, lane);
      if ((cnt & 1) && lane == 0) dst.elink[od + cnt - 1] = __ldg(src.elink + os + cnt - 1);
    }
  }
}

// In-use nodes and stored edges of the visited nodes of every game's tree (elfb200_mcts_tree_usage): what
// k_gather_trees moves for the game.  One warp per game.
__global__ void __launch_bounds__(BLOCK) k_tree_usage(int G, TreeDev tr, int32_t* __restrict__ nodes,
                                                      int32_t* __restrict__ edges) {
  const int lane = threadIdx.x & 31;
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (g >= G) return;
  const size_t nb = (size_t)g * tr.C;
  int nu = 0, ne = 0;
  for (int i = lane; i < tr.C; i += 32) {
    const NodeHdr h = load_hdr(&tr.hdr[nb + i]);
    nu += h.status != NS_FREE;
    ne += h.status == NS_VISITED ? (int)h.n_edges : 0;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    nu += __shfl_xor_sync(FULL, nu, d);
    ne += __shfl_xor_sync(FULL, ne, d);
  }
  if (lane == 0) {
    nodes[g] = nu;
    edges[g] = ne;
  }
}

__global__ void k_leaf_info(TreeDev tr, uint64_t* __restrict__ hash, int32_t* __restrict__ game,
                            int32_t* __restrict__ ply, int32_t* __restrict__ d4) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= *tr.eval_count) return;
  const size_t id = (size_t)tr.eval_game[s] * tr.C + tr.eval_node[s];
  if (hash) hash[s] = tr.hash[id];
  if (game) game[s] = tr.eval_game[s];
  if (ply) ply[s] = tr.meta[id].ply;
  if (d4) d4[s] = tr.eval_d4[s];
}

}  // namespace elfb200

// =========================================================================================
// C ABI (include/elfb200_mcts.h)
// =========================================================================================
using namespace elfb200;

struct elfb200_mcts {
  elfb200_ctx* ctx = nullptr;
  elfb200_mcts_options opt{};
  TreeDev tr{};
  SearchOpts so{};
  int waves_per_move = 0;
  int wave = 0;
  int64_t n_eval_total = 0;
  uint8_t* d_mask = nullptr;
  int32_t* d_actions = nullptr;
  int32_t* d_best = nullptr;
  int32_t* d_visits = nullptr;
  float* d_rootv = nullptr;
  float* d_bestq = nullptr;
  int32_t* d_total = nullptr;
  uint64_t* d_leaf_hash = nullptr;
  int32_t* d_leaf_game = nullptr;
  int32_t* d_leaf_ply = nullptr;
  int32_t* d_leaf_d4 = nullptr;
  int last_eval_count = 0;
  uint32_t move_counter = 0;
  float* d_priors = nullptr;
  // elfb200_mcts_root_edges / _set_root_priors / _set_d4_stream (allocated on first use)
  int32_t* d_edge_n = nullptr;
  int16_t* d_edge_act = nullptr;
  int32_t* d_edge_vis = nullptr;
  float* d_edge_w = nullptr;
  float* d_edge_p = nullptr;
  uint8_t* d_d4_stream = nullptr;
  int d4_cap_alloc = 0;
  // per-kernel device timing (CUDA events on the context stream), accumulated on the host
  cudaEvent_t ev[7] = {};  // sel0 sel1 feat0 feat1 exp0 exp1 bak1
  bool pending_sel = false, pending_feat = false, pending_eb = false;
  bool used_async = false;  // a wave ran without the host reading its leaf count
  bool wave_open = false;   // select issued, expand_backup not yet: nodes are claimed and virtual loss is applied
  double acc_ms[4] = {0, 0, 0, 0};  // select, features, expand, backup
  int64_t acc_waves = 0;
};

static void flush_timings(elfb200_mcts* m) {  // caller has synchronised the stream
  float ms = 0.f;
  if (m->pending_sel) {
    if (cudaEventElapsedTime(&ms, m->ev[0], m->ev[1]) == cudaSuccess) m->acc_ms[0] += ms;
    m->acc_waves++;
    m->pending_sel = false;
  }
  if (m->pending_feat) {
    if (cudaEventElapsedTime(&ms, m->ev[2], m->ev[3]) == cudaSuccess) m->acc_ms[1] += ms;
    m->pending_feat = false;
  }
  if (m->pending_eb) {
    if (cudaEventElapsedTime(&ms, m->ev[4], m->ev[5]) == cudaSuccess) m->acc_ms[2] += ms;
    if (cudaEventElapsedTime(&ms, m->ev[5], m->ev[6]) == cudaSuccess) m->acc_ms[3] += ms;
    m->pending_eb = false;
  }
}

static inline int warp_grid(int G) { return (G + WARPS - 1) / WARPS; }

// The leaf-batch formats (ELFB200_FEAT_*): the AGZ planes in float32 NCHW or 16-bit NHWC (cpad 24 / 32),
// or the DarkForest planes in float32 NCHW (cpad ignored).
static int check_leaf_format(const void* feat_dev, int format, int cpad) {
  if (format < FEAT_F32_NCHW || format > FEAT_DF_F32_NCHW) return elfb200_fail(ELFB200_ERR_ARG, "unknown feature format %d", format);
  if ((format == FEAT_F16_NHWC || format == FEAT_BF16_NHWC) && (cpad < 24 || cpad > FEAT_CPAD_MAX || (cpad & 7)))
    return elfb200_fail(ELFB200_ERR_ARG, "channel padding must be 24 or 32 (got %d)", cpad);
  if ((uintptr_t)feat_dev & 15) return elfb200_fail(ELFB200_ERR_ARG, "leaf feature buffer must be 16-byte aligned");
  return ELFB200_OK;
}

// The planes of the claimed leaves: `npos` CTAs, the kernels stop at the device-side count.
static void launch_leaf_features(elfb200_mcts* m, void* feat_dev, int format, int cpad, int npos) {
  elfb200_ctx* c = m->ctx;
  if (format == FEAT_DF_F32_NCHW) {
    DISPATCH_N(c,
               (k_leaf_features_df<19><<<npos, 32, 0, c->stream>>>(m->tr, c->st, c->d_exp_table,
                                                                   static_cast<float*>(feat_dev))),
               (k_leaf_features_df<9><<<npos, 32, 0, c->stream>>>(m->tr, c->st, c->d_exp_table,
                                                                  static_cast<float*>(feat_dev))));
  } else {
    DISPATCH_N(c,
               (k_leaf_features<19><<<npos, FEAT_THREADS, feature_smem_bytes<19>(format, cpad, c->feat_tma), c->stream>>>(
                   m->tr, feat_dev, format, cpad, c->feat_tma)),
               (k_leaf_features<9><<<npos, FEAT_THREADS, feature_smem_bytes<9>(format, cpad, c->feat_tma), c->stream>>>(
                   m->tr, feat_dev, format, cpad, c->feat_tma)));
  }
  c->launches++;
}

extern "C" {

int elfb200_mcts_default_options(elfb200_mcts_options* o) {
  if (!o) return elfb200_fail(ELFB200_ERR_ARG, "options is NULL");
  memset(o, 0, sizeof(*o));
  // TSOptions / SearchAlgoOptions defaults (tree_search_options.h:22-111) and MCTSActorParams
  // (go/mcts/mcts.h:17-27), with the self-play script's settings for the search itself
  o->num_rollouts = 800;
  o->num_rollouts_per_batch = 8;
  o->virtual_loss = 1;
  o->persistent_tree = 1;
  o->use_prior = 1;
  o->unexplored_q_zero = 0;
  o->root_unexplored_q_zero = 0;
  o->ply_pass_enabled = 0;
  o->remove_pass_if_dangerous = 1;
  o->rotation_flip = 1;
  o->seed = 0;
  o->nodes_per_game = 0;  // 0 = 2 * rollouts + 256
  o->c_puct = 1.5f;
  o->komi = 7.5f;
  return ELFB200_OK;
}

int elfb200_mcts_create(elfb200_ctx* c, const elfb200_mcts_options* opt, elfb200_mcts** out) {
  if (!c || !opt || !out) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  *out = nullptr;
  if (opt->num_rollouts <= 0 || opt->num_rollouts_per_batch <= 0 || opt->num_rollouts_per_batch > 64)
    return elfb200_fail(ELFB200_ERR_ARG, "num_rollouts must be > 0 and num_rollouts_per_batch in [1, 64]");
  if (opt->virtual_loss < 0) return elfb200_fail(ELFB200_ERR_ARG, "virtual_loss must be >= 0");
  if (opt->root_epsilon < 0.f || opt->root_epsilon > 1.f || (opt->root_epsilon > 0.f && opt->root_alpha <= 0.f))
    return elfb200_fail(ELFB200_ERR_ARG, "root_epsilon must be in [0,1] and root_alpha > 0 when noise is on");
  CK(cudaSetDevice(c->device));
  elfb200_mcts* m = new elfb200_mcts();
  m->ctx = c;
  m->opt = *opt;
  // any failure below releases what was allocated so far (elfb200_mcts_destroy tolerates a partly built handle)
  auto build = [&]() -> int {
  const int B = opt->num_rollouts_per_batch;
  m->waves_per_move = (opt->num_rollouts + B - 1) / B;  // for (idx = 0; idx < R; idx += B)
  int C = opt->nodes_per_game > 0 ? opt->nodes_per_game : 2 * m->waves_per_move * B + 256;
  if (C < m->waves_per_move * B + 2) C = m->waves_per_move * B + 2;
  if (C > 65534) return elfb200_fail(ELFB200_ERR_ARG, "nodes_per_game must be < 65535 (16-bit node ids)");
  const size_t G = c->G, N = c->N, E = N * N + 1, GC = G * (size_t)C;
  TreeDev& t = m->tr;
  t.C = C;
  t.B = B;
  t.E = (int)E;
  CK(cudaMalloc(&t.pos, GC * N * 8));
  CK(cudaMalloc(&t.sa, GC * N * 8));
  CK(cudaMalloc(&t.hash, GC * 8));
  CK(cudaMalloc(&t.meta, GC * sizeof(BoardMeta)));
  CK(cudaMalloc(&t.hdr, GC * sizeof(NodeHdr)));
  CK(cudaMalloc(&t.estat, GC * E * sizeof(float4)));
  CK(cudaMalloc(&t.elink, GC * E * 4));
  CK(cudaMalloc(&t.free_list, GC * 2));
  CK(cudaMalloc(&t.free_n, G * 4));
  CK(cudaMalloc(&t.root, G * 2));
  CK(cudaMalloc(&t.leaves, G * B * 2));
  CK(cudaMalloc(&t.active, G));
  CK(cudaMalloc(&t.eval_count, 4));
  CK(cudaMalloc(&t.eval_game, G * B * 4));
  CK(cudaMalloc(&t.eval_node, G * B * 2));
  CK(cudaMalloc(&t.eval_d4, G * B));
  CK(cudaMalloc(&t.hist, G * B * 8 * N * 8));
  CK(cudaMalloc(&t.hinfo, G * B * 4));
  CK(cudaMalloc(&t.bfs_q, GC * 2));
  CK(cudaMalloc(&t.errors, 16));
  CK(cudaMemsetAsync(t.errors, 0, 16, c->stream));
  CK(cudaMalloc(&t.stats, 64));
  CK(cudaMemsetAsync(t.stats, 0, 64, c->stream));
  CK(cudaMemsetAsync(t.hdr, 0, GC * sizeof(NodeHdr), c->stream));
  CK(cudaMemsetAsync(t.active, 1, G, c->stream));
  CK(cudaMemsetAsync(t.eval_count, 0, 4, c->stream));
  CK(cudaMalloc(&m->d_mask, G));
  CK(cudaMalloc(&m->d_actions, G * 4));
  CK(cudaMalloc(&m->d_best, G * 4));
  CK(cudaMalloc(&m->d_visits, G * E * 4));
  CK(cudaMalloc(&m->d_rootv, G * 4));
  CK(cudaMalloc(&m->d_bestq, G * 4));
  CK(cudaMalloc(&m->d_total, G * 4));
  CK(cudaMalloc(&m->d_leaf_hash, G * B * 8));
  CK(cudaMalloc(&m->d_leaf_game, G * B * 4));
  CK(cudaMalloc(&m->d_leaf_ply, G * B * 4));
  CK(cudaMalloc(&m->d_leaf_d4, G * B * 4));
  SearchOpts& s = m->so;
  s.num_rollouts = opt->num_rollouts;
  s.virtual_loss = opt->virtual_loss;
  s.persistent = opt->persistent_tree;
  s.use_prior = opt->use_prior;
  s.uqz = opt->unexplored_q_zero;
  s.ruqz = opt->root_unexplored_q_zero;
  s.ply_pass_enabled = opt->ply_pass_enabled;
  s.remove_pass_if_dangerous = opt->remove_pass_if_dangerous;
  s.rotation_flip = opt->rotation_flip;
  s.seed = opt->seed;
  s.std_sort_ties = opt->std_sort_ties != 0;
  s.c_puct = opt->c_puct;
  s.komi = opt->komi;
  for (auto& e : m->ev) CK(cudaEventCreate(&e));
  k_tree_reset<<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->G, t, nullptr);
  c->launches++;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
  };
  const int rc = build();
  if (rc) {
    const std::string why = elfb200_last_error();
    elfb200_mcts_destroy(m);
    elfb200_fail(rc, "%s", why.c_str());
    return rc;
  }
  *out = m;
  return ELFB200_OK;
}

void elfb200_mcts_destroy(elfb200_mcts* m) {
  if (!m) return;
  cudaSetDevice(m->ctx->device);
  cudaStreamSynchronize(m->ctx->stream);
  TreeDev& t = m->tr;
  void* ptrs[] = {t.pos,       t.sa,        t.hash,      t.meta,      t.hdr,        t.estat,       t.elink,      t.free_list,
                  t.free_n,    t.root,      t.leaves,    t.active,     t.eval_count,  t.eval_game,  t.eval_node,
                  t.eval_d4,   t.hist,      t.hinfo,     t.bfs_q,     t.errors,    t.stats,     m->d_mask,    m->d_actions,  m->d_best,    m->d_visits,
                  m->d_rootv,  m->d_bestq,  m->d_total,  m->d_leaf_hash, m->d_leaf_game, m->d_leaf_ply, m->d_leaf_d4, m->d_priors,
                  m->d_edge_n, m->d_edge_act, m->d_edge_vis, m->d_edge_w, m->d_edge_p, m->d_d4_stream, t.d4_used};
  for (void* p : ptrs)
    if (p) cudaFree(p);
  for (auto& e : m->ev)
    if (e) cudaEventDestroy(e);
  delete m;
}

int elfb200_mcts_waves_per_move(const elfb200_mcts* m) { return m ? m->waves_per_move : 0; }
int elfb200_mcts_max_leaves(const elfb200_mcts* m) { return m ? m->ctx->G * m->tr.B : 0; }
int elfb200_mcts_nodes_per_game(const elfb200_mcts* m) { return m ? m->tr.C : 0; }

// ---- one launch function per operation, shared by the host form and the device form (_dev) ----------------------
// The device forms pass device pointers, skip the timing events and never wait for the stream, so that they can be
// captured in a CUDA graph; everything they launch is what the host forms launch.

// The device forms are refused while a reference D4 stream is set: that stream is refilled from the host every move.
static int check_dev_form(const elfb200_mcts* m) {
  if (!m) return elfb200_fail(ELFB200_ERR_ARG, "mcts is NULL");
  if (m->tr.d4_stream)
    return elfb200_fail(ELFB200_ERR_STATE, "a reference D4 stream is set (elfb200_mcts_set_d4_stream): it is fed "
                                           "from the host every move, so the device forms are not available");
  return ELFB200_OK;
}

static int tree_reset_launch(elfb200_mcts* m, const uint8_t* mask_dev) {
  elfb200_ctx* c = m->ctx;
  k_tree_reset<<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->G, m->tr, mask_dev);
  c->launches++;
  CK(cudaGetLastError());
  return ELFB200_OK;
}

// k_begin and the root noise, keyed by the host counter (move_dev NULL) or by the move index in device memory
static int begin_move_launch(elfb200_mcts* m, const int64_t* move_dev) {
  elfb200_ctx* c = m->ctx;
  const int need = m->waves_per_move * m->tr.B;
  DISPATCH_N(c, (k_begin<19><<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->st, m->tr, need)),
             (k_begin<9><<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->st, m->tr, need)));
  c->launches++;
  CK(cudaGetLastError());
  if (m->opt.root_epsilon > 0.f) {
    const uint64_t seed = (uint64_t)(uint32_t)m->opt.seed;
    if (move_dev)
      k_root_noise<<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->G, m->tr, m->opt.root_epsilon, m->opt.root_alpha,
                                                              seed, move_dev);
    else
      k_root_noise<<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->G, m->tr, m->opt.root_epsilon, m->opt.root_alpha,
                                                              seed, m->move_counter);
    c->launches++;
    CK(cudaGetLastError());
  }
  m->wave = 0;
  return ELFB200_OK;
}

int elfb200_mcts_reset(elfb200_mcts* m, const uint8_t* mask_host) {
  if (!m) return elfb200_fail(ELFB200_ERR_ARG, "mcts is NULL");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  const uint8_t* dm = nullptr;
  if (mask_host) {
    memcpy(c->h_pin, mask_host, c->G);
    CK(cudaMemcpyAsync(m->d_mask, c->h_pin, c->G, cudaMemcpyHostToDevice, c->stream));
    dm = m->d_mask;
  }
  const int rc = tree_reset_launch(m, dm);
  if (rc) return rc;
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_mcts_reset_dev(elfb200_mcts* m, const uint8_t* mask_dev) {
  const int rc = check_dev_form(m);
  if (rc) return rc;
  CK(cudaSetDevice(m->ctx->device));
  return tree_reset_launch(m, mask_dev);
}

int elfb200_mcts_begin_move(elfb200_mcts* m, const uint8_t* active_host) {
  if (!m) return elfb200_fail(ELFB200_ERR_ARG, "mcts is NULL");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  if (active_host) {
    memcpy(c->h_pin, active_host, c->G);
    CK(cudaMemcpyAsync(m->tr.active, c->h_pin, c->G, cudaMemcpyHostToDevice, c->stream));
  } else {
    CK(cudaMemsetAsync(m->tr.active, 1, c->G, c->stream));
  }
  const int rc = begin_move_launch(m, nullptr);
  if (rc) return rc;
  m->move_counter++;
  return ELFB200_OK;
}

int elfb200_mcts_begin_move_dev(elfb200_mcts* m, const uint8_t* active_dev, const int64_t* move_dev) {
  int rc = check_dev_form(m);
  if (rc) return rc;
  if (!move_dev && m->opt.root_epsilon > 0.f)
    return elfb200_fail(ELFB200_ERR_ARG, "move_dev is NULL with root noise on (root_epsilon > 0)");
  if (m->wave_open) return elfb200_fail(ELFB200_ERR_STATE, "a wave is open (select without expand_backup)");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  if (active_dev)
    CK(cudaMemcpyAsync(m->tr.active, active_dev, c->G, cudaMemcpyDeviceToDevice, c->stream));
  else
    CK(cudaMemsetAsync(m->tr.active, 1, c->G, c->stream));
  return begin_move_launch(m, move_dev);
}

// One wave's descents and leaf planes.  timed: the host form's event pairs around the kernels (and the wait
// for the previous wave's, which the pairs are reused from); n_leaves as in elfb200_mcts_select_ex.
static int select_launch(elfb200_mcts* m, void* feat_dev, int format, int cpad, int32_t* n_leaves, bool timed) {
  elfb200_ctx* c = m->ctx;
  if (timed && (m->pending_sel || m->pending_feat || m->pending_eb)) {
    // the event pairs are reused every wave: read the previous wave's before re-recording them
    // (only reached in the asynchronous mode; the synchronous mode flushed after its own sync)
    CK(cudaEventSynchronize(m->ev[6]));
    flush_timings(m);
  }
  CK(cudaMemsetAsync(m->tr.eval_count, 0, 4, c->stream));
  if (timed) CK(cudaEventRecord(m->ev[0], c->stream));
  DISPATCH_N(c, (k_select<19><<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->st, m->tr, m->so, m->wave)),
             (k_select<9><<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->st, m->tr, m->so, m->wave)));
  c->launches++;
  CK(cudaGetLastError());
  if (timed) {
    CK(cudaEventRecord(m->ev[1], c->stream));
    m->pending_sel = true;
  }
  m->wave_open = true;
  int n = -1;  // unknown to the host: the feature / expand grids cover all G*B slots and the kernels
               // stop at the device-side count
  if (n_leaves) {
    int32_t* hp = (int32_t*)c->h_pin;
    CK(cudaMemcpyAsync(hp, m->tr.eval_count, 4, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    flush_timings(m);  // this wave's select and the previous wave's features / expand / backup are complete
    n = hp[0];
    m->n_eval_total += n;
    *n_leaves = n;
  } else {
    m->used_async = true;
  }
  m->last_eval_count = n;
  if (n != 0) {
    const int npos = n > 0 ? n : c->G * m->tr.B;
    if (timed) CK(cudaEventRecord(m->ev[2], c->stream));
    launch_leaf_features(m, feat_dev, format, cpad, npos);
    CK(cudaGetLastError());
    if (timed) {
      CK(cudaEventRecord(m->ev[3], c->stream));
      m->pending_feat = true;
    }
  }
  m->wave++;
  return ELFB200_OK;
}

int elfb200_mcts_select_ex(elfb200_mcts* m, void* feat_dev, int format, int cpad, int32_t* n_leaves) {
  if (!m || !feat_dev) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  const int rc = check_leaf_format(feat_dev, format, cpad);
  if (rc) return rc;
  CK(cudaSetDevice(m->ctx->device));
  return select_launch(m, feat_dev, format, cpad, n_leaves, true);
}

int elfb200_mcts_select_dev(elfb200_mcts* m, void* feat_dev, int format, int cpad) {
  int rc = check_dev_form(m);
  if (rc) return rc;
  if (!feat_dev) return elfb200_fail(ELFB200_ERR_ARG, "feat_dev is NULL");
  rc = check_leaf_format(feat_dev, format, cpad);
  if (rc) return rc;
  if (m->wave_open) return elfb200_fail(ELFB200_ERR_STATE, "a wave is open (select without expand_backup)");
  CK(cudaSetDevice(m->ctx->device));
  return select_launch(m, feat_dev, format, cpad, nullptr, false);
}

int elfb200_mcts_leaf_features(elfb200_mcts* m, void* feat_dev, int format, int cpad) {
  if (!m || !feat_dev) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  elfb200_ctx* c = m->ctx;
  const int rc = check_leaf_format(feat_dev, format, cpad);
  if (rc) return rc;
  CK(cudaSetDevice(c->device));
  const int n = m->last_eval_count;
  if (n == 0) return ELFB200_OK;
  const int npos = n > 0 ? n : c->G * m->tr.B;
  launch_leaf_features(m, feat_dev, format, cpad, npos);
  CK(cudaGetLastError());
  return ELFB200_OK;
}

int elfb200_mcts_select(elfb200_mcts* m, float* feat_dev, int32_t* n_leaves) {
  if (!n_leaves) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  return elfb200_mcts_select_ex(m, feat_dev, FEAT_F32_NCHW, 0, n_leaves);
}

int elfb200_mcts_leaf_count(elfb200_mcts* m, int32_t* n_leaves) {
  if (!m || !n_leaves) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  int32_t* hp = (int32_t*)c->h_pin;
  CK(cudaMemcpyAsync(hp, m->tr.eval_count, 4, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  *n_leaves = hp[0];
  m->last_eval_count = hp[0];  // known to the host from here on: leaf_info and the expansion grid use it
  return ELFB200_OK;
}

int elfb200_mcts_leaf_info(elfb200_mcts* m, uint64_t* hash_host, int32_t* game_host, int32_t* ply_host,
                           int32_t* d4_host) {
  if (!m) return elfb200_fail(ELFB200_ERR_ARG, "mcts is NULL");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  const int n = m->last_eval_count;
  if (n <= 0) return ELFB200_OK;
  k_leaf_info<<<(n + 127) / 128, 128, 0, c->stream>>>(m->tr, m->d_leaf_hash, m->d_leaf_game, m->d_leaf_ply,
                                                         m->d_leaf_d4);
  c->launches++;
  CK(cudaGetLastError());
  if (hash_host) CK(cudaMemcpyAsync(hash_host, m->d_leaf_hash, (size_t)n * 8, cudaMemcpyDeviceToHost, c->stream));
  if (game_host) CK(cudaMemcpyAsync(game_host, m->d_leaf_game, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
  if (ply_host) CK(cudaMemcpyAsync(ply_host, m->d_leaf_ply, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
  if (d4_host) CK(cudaMemcpyAsync(d4_host, m->d_leaf_d4, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

// Expansion with the network's reply, then backup; timed as in select_launch.
static int expand_backup_launch(elfb200_mcts* m, const float* pi_dev, const float* value_dev, bool timed) {
  elfb200_ctx* c = m->ctx;
  const int n = m->last_eval_count;
  if (timed) CK(cudaEventRecord(m->ev[4], c->stream));
  if (n != 0) {
    if (!pi_dev || !value_dev) return elfb200_fail(ELFB200_ERR_ARG, "pi/value is NULL with %d leaves pending", n);
    const int nw = n > 0 ? n : c->G * m->tr.B;  // n < 0: count known to the device only
    if (m->so.std_sort_ties)
      DISPATCH_N(c, (k_expand<19, true><<<warp_grid(nw), BLOCK, 0, c->stream>>>(c->st, m->tr, m->so, pi_dev, value_dev)),
                 (k_expand<9, true><<<warp_grid(nw), BLOCK, 0, c->stream>>>(c->st, m->tr, m->so, pi_dev, value_dev)));
    else
      DISPATCH_N(c, (k_expand<19, false><<<warp_grid(nw), BLOCK, 0, c->stream>>>(c->st, m->tr, m->so, pi_dev, value_dev)),
                 (k_expand<9, false><<<warp_grid(nw), BLOCK, 0, c->stream>>>(c->st, m->tr, m->so, pi_dev, value_dev)));
    c->launches++;
    CK(cudaGetLastError());
  }
  if (timed) CK(cudaEventRecord(m->ev[5], c->stream));
  k_backup<<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->G, m->tr, m->so.virtual_loss);
  c->launches++;
  CK(cudaGetLastError());
  if (timed) {
    CK(cudaEventRecord(m->ev[6], c->stream));
    m->pending_eb = true;
  }
  m->wave_open = false;
  return ELFB200_OK;
}

int elfb200_mcts_expand_backup(elfb200_mcts* m, const float* pi_dev, const float* value_dev) {
  if (!m) return elfb200_fail(ELFB200_ERR_ARG, "mcts is NULL");
  CK(cudaSetDevice(m->ctx->device));
  return expand_backup_launch(m, pi_dev, value_dev, true);
}

int elfb200_mcts_expand_backup_dev(elfb200_mcts* m, const float* pi_dev, const float* value_dev) {
  const int rc = check_dev_form(m);
  if (rc) return rc;
  if (!pi_dev || !value_dev) return elfb200_fail(ELFB200_ERR_ARG, "pi/value is NULL");
  if (!m->wave_open) return elfb200_fail(ELFB200_ERR_STATE, "no wave is open (expand_backup without select)");
  CK(cudaSetDevice(m->ctx->device));
  return expand_backup_launch(m, pi_dev, value_dev, false);
}

// k_results into the given device tables (each may be NULL)
static int results_launch(elfb200_mcts* m, int32_t* best, int32_t* visits, float* rootv, float* bestq, int32_t* total) {
  elfb200_ctx* c = m->ctx;
  DISPATCH_N(c, (k_results<19><<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->G, m->tr, best, visits, rootv, bestq, total)),
             (k_results<9><<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->G, m->tr, best, visits, rootv, bestq, total)));
  c->launches++;
  CK(cudaGetLastError());
  return ELFB200_OK;
}

int elfb200_mcts_results(elfb200_mcts* m, int32_t* best_action_host, int32_t* visits_host,
                         float* root_value_host, float* best_q_host, int32_t* total_visits_host) {
  if (!m) return elfb200_fail(ELFB200_ERR_ARG, "mcts is NULL");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  const size_t G = c->G, P1 = (size_t)c->N * c->N + 1;
  const int rc = results_launch(m, m->d_best, m->d_visits, m->d_rootv, m->d_bestq, m->d_total);
  if (rc) return rc;
  if (best_action_host) CK(cudaMemcpyAsync(best_action_host, m->d_best, G * 4, cudaMemcpyDeviceToHost, c->stream));
  if (visits_host) CK(cudaMemcpyAsync(visits_host, m->d_visits, G * P1 * 4, cudaMemcpyDeviceToHost, c->stream));
  if (root_value_host) CK(cudaMemcpyAsync(root_value_host, m->d_rootv, G * 4, cudaMemcpyDeviceToHost, c->stream));
  if (best_q_host) CK(cudaMemcpyAsync(best_q_host, m->d_bestq, G * 4, cudaMemcpyDeviceToHost, c->stream));
  if (total_visits_host) CK(cudaMemcpyAsync(total_visits_host, m->d_total, G * 4, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

static int advance_launch(elfb200_mcts* m, const int32_t* actions_dev) {
  elfb200_ctx* c = m->ctx;
  k_advance<<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->G, m->tr, actions_dev, m->so.persistent);
  c->launches++;
  CK(cudaGetLastError());
  return ELFB200_OK;
}

int elfb200_mcts_advance(elfb200_mcts* m, const int32_t* actions_host) {
  if (!m || !actions_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  memcpy(c->h_pin, actions_host, (size_t)c->G * 4);
  CK(cudaMemcpyAsync(m->d_actions, c->h_pin, (size_t)c->G * 4, cudaMemcpyHostToDevice, c->stream));
  const int rc = advance_launch(m, m->d_actions);
  if (rc) return rc;
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_mcts_advance_dev(elfb200_mcts* m, const int32_t* actions_dev) {
  const int rc = check_dev_form(m);
  if (rc) return rc;
  if (!actions_dev) return elfb200_fail(ELFB200_ERR_ARG, "actions_dev is NULL");
  CK(cudaSetDevice(m->ctx->device));
  return advance_launch(m, actions_dev);
}

// k_choose with the seed by value (seed_dev NULL) or read from device memory
static int choose_launch(elfb200_mcts* m, int cutoff, float resign_thres, const uint8_t* never_resign_dev,
                         uint64_t seed, const int64_t* seed_dev, int32_t* actions_dev, float* values_dev) {
  elfb200_ctx* c = m->ctx;
  if (seed_dev)
    DISPATCH_N(c,
               (k_choose<19><<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->st, m->tr, cutoff, resign_thres,
                                                                        never_resign_dev, seed_dev, actions_dev, values_dev)),
               (k_choose<9><<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->st, m->tr, cutoff, resign_thres,
                                                                       never_resign_dev, seed_dev, actions_dev, values_dev)));
  else
    DISPATCH_N(c,
               (k_choose<19><<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->st, m->tr, cutoff, resign_thres,
                                                                        never_resign_dev, seed, actions_dev, values_dev)),
               (k_choose<9><<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->st, m->tr, cutoff, resign_thres,
                                                                       never_resign_dev, seed, actions_dev, values_dev)));
  c->launches++;
  CK(cudaGetLastError());
  return ELFB200_OK;
}

int elfb200_mcts_choose(elfb200_mcts* m, int policy_distri_cutoff, float resign_thres,
                        const uint8_t* never_resign_host, uint64_t seed, int32_t* actions_host,
                        float* values_host) {
  if (!m || !actions_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  const size_t G = c->G;
  const uint8_t* nr = nullptr;
  if (never_resign_host) {
    memcpy(c->h_pin, never_resign_host, G);
    CK(cudaMemcpyAsync(m->d_mask, c->h_pin, G, cudaMemcpyHostToDevice, c->stream));
    nr = m->d_mask;
  }
  const int rc = choose_launch(m, policy_distri_cutoff, resign_thres, nr, seed, nullptr, m->d_best, m->d_bestq);
  if (rc) return rc;
  CK(cudaMemcpyAsync(actions_host, m->d_best, G * 4, cudaMemcpyDeviceToHost, c->stream));
  if (values_host) CK(cudaMemcpyAsync(values_host, m->d_bestq, G * 4, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_mcts_choose_dev(elfb200_mcts* m, int policy_distri_cutoff, float resign_thres,
                            const uint8_t* never_resign_dev, const int64_t* seed_dev, int32_t* actions_dev,
                            float* values_dev) {
  const int rc = check_dev_form(m);
  if (rc) return rc;
  if (!seed_dev || !actions_dev) return elfb200_fail(ELFB200_ERR_ARG, "seed_dev/actions_dev is NULL");
  CK(cudaSetDevice(m->ctx->device));
  return choose_launch(m, policy_distri_cutoff, resign_thres, never_resign_dev, 0, seed_dev, actions_dev, values_dev);
}

int elfb200_mcts_results_dev(elfb200_mcts* m, int32_t* best_action_dev, int32_t* visits_dev, float* root_value_dev,
                             float* best_q_dev, int32_t* total_visits_dev) {
  const int rc = check_dev_form(m);
  if (rc) return rc;
  CK(cudaSetDevice(m->ctx->device));
  return results_launch(m, best_action_dev, visits_dev, root_value_dev, best_q_dev, total_visits_dev);
}

int elfb200_mcts_root_priors(elfb200_mcts* m, float* priors_host) {
  if (!m || !priors_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  const size_t G = c->G, P1 = (size_t)c->N * c->N + 1;
  if (!m->d_priors) CK(cudaMalloc(&m->d_priors, G * P1 * 4));
  k_root_priors<<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->G, m->tr, m->d_priors, (int)P1);
  c->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(priors_host, m->d_priors, G * P1 * 4, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_mcts_root_edges(elfb200_mcts* m, int32_t* n_edges_host, int16_t* actions_host, int32_t* visits_host,
                            float* wsum_host, float* priors_host) {
  if (!m || !n_edges_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  const size_t G = c->G, P1 = (size_t)c->N * c->N + 1;
  if (!m->d_edge_n) CK(cudaMalloc(&m->d_edge_n, G * 4));
  if (!m->d_edge_act) CK(cudaMalloc(&m->d_edge_act, G * P1 * 2));
  if (!m->d_edge_vis) CK(cudaMalloc(&m->d_edge_vis, G * P1 * 4));
  if (!m->d_edge_w) CK(cudaMalloc(&m->d_edge_w, G * P1 * 4));
  if (!m->d_edge_p) CK(cudaMalloc(&m->d_edge_p, G * P1 * 4));
  k_root_edges<<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->G, m->tr, m->d_edge_n, m->d_edge_act, m->d_edge_vis,
                                                          m->d_edge_w, m->d_edge_p, (int)P1);
  c->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(n_edges_host, m->d_edge_n, G * 4, cudaMemcpyDeviceToHost, c->stream));
  if (actions_host) CK(cudaMemcpyAsync(actions_host, m->d_edge_act, G * P1 * 2, cudaMemcpyDeviceToHost, c->stream));
  if (visits_host) CK(cudaMemcpyAsync(visits_host, m->d_edge_vis, G * P1 * 4, cudaMemcpyDeviceToHost, c->stream));
  if (wsum_host) CK(cudaMemcpyAsync(wsum_host, m->d_edge_w, G * P1 * 4, cudaMemcpyDeviceToHost, c->stream));
  if (priors_host) CK(cudaMemcpyAsync(priors_host, m->d_edge_p, G * P1 * 4, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_mcts_set_root_priors(elfb200_mcts* m, const uint8_t* mask_host, const float* priors_host) {
  if (!m || !priors_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  const size_t G = c->G, P1 = (size_t)c->N * c->N + 1;
  if (!m->d_edge_p) CK(cudaMalloc(&m->d_edge_p, G * P1 * 4));
  const uint8_t* dm = nullptr;
  if (mask_host) {
    CK(cudaMemcpyAsync(m->d_mask, mask_host, G, cudaMemcpyHostToDevice, c->stream));
    dm = m->d_mask;
  }
  CK(cudaMemcpyAsync(m->d_edge_p, priors_host, G * P1 * 4, cudaMemcpyHostToDevice, c->stream));
  k_set_root_priors<<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->G, m->tr, dm, m->d_edge_p, (int)P1);
  c->launches++;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->stream));  // the host tables may be reused by the caller
  return ELFB200_OK;
}

int elfb200_mcts_set_d4_stream(elfb200_mcts* m, const uint8_t* codes_host, int count) {
  if (!m) return elfb200_fail(ELFB200_ERR_ARG, "mcts is NULL");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  const size_t G = c->G;
  if (!codes_host) {  // back to the counter-based generator
    m->tr.d4_stream = nullptr;
    return ELFB200_OK;
  }
  if (count < m->waves_per_move * m->tr.B)
    return elfb200_fail(ELFB200_ERR_ARG, "a move may evaluate %d leaves per game: %d codes are not enough",
                        m->waves_per_move * m->tr.B, count);
  if (count > m->d4_cap_alloc) {
    CK(cudaStreamSynchronize(c->stream));
    if (m->d_d4_stream) CK(cudaFree(m->d_d4_stream));
    m->d_d4_stream = nullptr;
    m->d4_cap_alloc = 0;
    CK(cudaMalloc(&m->d_d4_stream, G * (size_t)count));
    m->d4_cap_alloc = count;
  }
  if (!m->tr.d4_used) CK(cudaMalloc(&m->tr.d4_used, G * 4));
  CK(cudaMemcpyAsync(m->d_d4_stream, codes_host, G * (size_t)count, cudaMemcpyHostToDevice, c->stream));
  CK(cudaMemsetAsync(m->tr.d4_used, 0, G * 4, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  m->tr.d4_stream = m->d_d4_stream;
  m->tr.d4_cap = count;
  return ELFB200_OK;
}

int elfb200_mcts_d4_used(elfb200_mcts* m, int32_t* used_host) {
  if (!m || !used_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  elfb200_ctx* c = m->ctx;
  if (!m->tr.d4_stream || !m->tr.d4_used) return elfb200_fail(ELFB200_ERR_STATE, "no D4 stream is set");
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(used_host, m->tr.d4_used, (size_t)c->G * 4, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_mcts_errors(elfb200_mcts* m, int32_t* counters_host4) {
  if (!m || !counters_host4) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(counters_host4, m->tr.errors, 16, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int64_t elfb200_mcts_eval_count(const elfb200_mcts* m) {
  if (!m) return 0;
  if (!m->used_async) return m->n_eval_total;
  // waves ran without a host read of the count: the device keeps the total (k_backup)
  unsigned long long v = 0;
  if (cudaSetDevice(m->ctx->device) != cudaSuccess || cudaStreamSynchronize(m->ctx->stream) != cudaSuccess ||
      cudaMemcpy(&v, m->tr.stats + 4, 8, cudaMemcpyDeviceToHost) != cudaSuccess)
    return -1;
  return (int64_t)v;
}

int elfb200_mcts_timings(elfb200_mcts* m, double* ms_host4, int64_t* waves, int reset) {
  if (!m || !ms_host4) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  CK(cudaStreamSynchronize(c->stream));
  flush_timings(m);
  for (int i = 0; i < 4; ++i) ms_host4[i] = m->acc_ms[i];
  if (waves) *waves = m->acc_waves;
  if (reset) {
    for (int i = 0; i < 4; ++i) m->acc_ms[i] = 0;
    m->acc_waves = 0;
  }
  return ELFB200_OK;
}

static int check_tree_gather(const elfb200_mcts* dst, const elfb200_mcts* src, const int32_t* index) {
  if (!dst || !src || !index) return elfb200_fail(ELFB200_ERR_ARG, "dst/src/index is NULL");
  if (dst == src)
    return elfb200_fail(ELFB200_ERR_ARG, "dst and src are the same search handle (an in-place permutation would race)");
  const elfb200_ctx *cd = dst->ctx, *cs = src->ctx;
  if (cd->N != cs->N) return elfb200_fail(ELFB200_ERR_ARG, "board sizes differ (dst %d, src %d)", cd->N, cs->N);
  if (cd->device != cs->device) return elfb200_fail(ELFB200_ERR_ARG, "devices differ (dst %d, src %d)", cd->device, cs->device);
  if (dst->tr.C != src->tr.C)
    return elfb200_fail(ELFB200_ERR_ARG, "nodes_per_game differs (dst %d, src %d)", dst->tr.C, src->tr.C);
  if (dst->wave_open || src->wave_open)
    return elfb200_fail(ELFB200_ERR_ARG, "the %s handle has a wave open (select without expand_backup)",
                        dst->wave_open ? "dst" : "src");
  return ELFB200_OK;
}

// k_gather_trees on dst's stream, after the work already on src's stream (fork); src's later work waits for the
// copy (join), so it cannot change a tree while the tree is read.  Two handles on one context share the stream.
// The fork / join events are the destination context's, the two of elfb200_gather_games_dev: each record is
// waited on before the next call records it again, so the board copy and the tree copy can share them, and a
// search handle allocates nothing for copies it never makes.
static int tree_gather_launch(elfb200_mcts* dst, const elfb200_mcts* src, const int32_t* index_dev) {
  elfb200_ctx *cd = dst->ctx, *cs = src->ctx;
  int rc = stream_after(cd->stream, cs->stream, cd->ev_gather[0]);
  if (rc) return rc;
  DISPATCH_N(cd,
             (k_gather_trees<19><<<cd->G, TREE_GATHER_THREADS, 0, cd->stream>>>(dst->tr, src->tr, cd->G, cs->G, index_dev)),
             (k_gather_trees<9><<<cd->G, TREE_GATHER_THREADS, 0, cd->stream>>>(dst->tr, src->tr, cd->G, cs->G, index_dev)));
  cd->launches++;
  CK(cudaGetLastError());
  return stream_after(cs->stream, cd->stream, cd->ev_gather[1]);
}

int elfb200_mcts_gather_dev(elfb200_mcts* dst, const elfb200_mcts* src, const int32_t* index_dev) {
  int rc = check_tree_gather(dst, src, index_dev);
  if (rc) return rc;
  CK(cudaSetDevice(dst->ctx->device));
  return tree_gather_launch(dst, src, index_dev);
}

int elfb200_mcts_gather(elfb200_mcts* dst, const elfb200_mcts* src, const int32_t* index_host) {
  int rc = check_tree_gather(dst, src, index_host);
  if (rc) return rc;
  elfb200_ctx* c = dst->ctx;
  CK(cudaSetDevice(c->device));
  memcpy(c->h_pin, index_host, (size_t)c->G * 4);
  CK(cudaMemcpyAsync(dst->d_actions, c->h_pin, (size_t)c->G * 4, cudaMemcpyHostToDevice, c->stream));
  rc = tree_gather_launch(dst, src, dst->d_actions);
  if (rc) return rc;
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_mcts_tree_usage(elfb200_mcts* m, int32_t* nodes_host, int32_t* edges_host) {
  if (!m || !nodes_host || !edges_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  k_tree_usage<<<warp_grid(c->G), BLOCK, 0, c->stream>>>(c->G, m->tr, m->d_best, m->d_total);
  c->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(nodes_host, m->d_best, (size_t)c->G * 4, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaMemcpyAsync(edges_host, m->d_total, (size_t)c->G * 4, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_mcts_stats(elfb200_mcts* m, uint64_t* counters_host4) {
  if (!m || !counters_host4) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  elfb200_ctx* c = m->ctx;
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(counters_host4, m->tr.stats, 32, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

}  // extern "C"
