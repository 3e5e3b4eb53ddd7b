// elfb200.cu -- kernels + C ABI of libelfb200.so (board path).
//
// Kernels (all templated on the board size N in {9, 19}; one game per N-lane warp segment):
//   k_reset     clear selected games
//   k_step      GoState::forward for a batch: validate, play, superko, next legal mask
//   k_replay    every game forwards its own move list from the empty board
//   k_place     handicap stones (TryPlay / Play for black)
//   k_export    host-facing views (legal/stones/eyes by action index, info words, tt score)
//   k_env_step  k_step + end of game (score, restart) + legal/info views: one ply of the device-resident env
//   k_features  BoardFeature::extractAGZ, float32 [G][18][N][N]; k_features_df the DarkForest planes
//   k_playout   whole random-policy games with the position (and the incremental safe/atari group
//               masks) held in registers; to-terminal and steady-state ("stream") modes
//   k_playout2  k_playout in the two-rows-per-lane layout (board2.cuh), 19x19 only
//   k_gather    copy games from another batch (GoState's copy constructor); no geometry, one kernel for both sizes
//   k_ownership K random-policy playouts from every stored position, per-point area counts (Monte-Carlo ownership)
//   k_final_status  dead groups from those counts, getTrompTaylorScore with them (territory map and score)
//
// Each game rule lives in one device function that the kernels share: forward_ply is GoState::forward's move
// (k_step, k_env_step, k_replay), random_ply one move of the random policy (k_playout, k_playout2, k_ownership),
// playout_body the whole playout kernel of both lane layouts, legal_for_next the legal rows of the side to move.
// The ones templated on the lane type compile for Lane (board.cuh) and Lane2 (board2.cuh) alike.
//
// HBM layout (structure of arrays, G games):
//   cur   uint64 [G][N]      current position, row y = black_row | white_row << 32
//   ring  uint64 [G][8][N]   last 8 positions (AGZ history), slot (ply-2) & 7 is the newest
//   legal uint32 [G][N]      legal-move rows for the side to move
//   hash  uint64 [G]         Zobrist hash
//   meta  BoardMeta [G]      16 B: ply, side, ko, last moves, captures
//   sk    uint64 [G][2N^2]   pre-move hashes of all non-pass moves (superko record), sk_n int32[G]
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cmath>
#include <string>
#include <vector>

#include "common.cuh"
#include "board2.cuh"

namespace elfb200 {

// ---------------------------------------------------------------------------------------
// Row words: a game's `cur` and `sa` blocks hold one uint64 per board row, black | white << 32 and
// safe | atari << 32, so that a lane moves its row with one coalesced 8-byte access.
__device__ __forceinline__ uint64_t pack_row(uint32_t lo, uint32_t hi) { return (uint64_t)lo | ((uint64_t)hi << 32); }

// row y of game g of a [G][N] row-word block; 0 on lanes where `on` is false
template <int N>
__device__ __forceinline__ void load_row(const uint64_t* a, int g, int y, bool on, uint32_t& lo, uint32_t& hi) {
  const uint64_t v = on ? a[(size_t)g * N + y] : 0ull;
  lo = (uint32_t)v;
  hi = (uint32_t)(v >> 32);
}
template <int N>
__device__ __forceinline__ void store_row(uint64_t* a, int g, int y, uint32_t lo, uint32_t hi) {
  a[(size_t)g * N + y] = pack_row(lo, hi);
}

// ---------------------------------------------------------------------------------------
// What differs between the two lane layouts of the playout kernels, Lane (board.cuh: one uint32_t row per
// lane) and Lane2 (board2.cuh: a P2 pair of rows per lane).  Code templated on the lane type takes its row
// type from the lane's `rm` member and everything else from the shared board primitives.
__device__ __forceinline__ int popc_rows(uint32_t v) { return __popc(v); }
__device__ __forceinline__ int popc_rows(P2 v) { return popc2(v); }
__device__ __forceinline__ uint32_t zero_rows(const Lane&) { return 0u; }
__device__ __forceinline__ P2 zero_rows(const Lane2&) { return zero2(); }
// the lane that writes a game's per-game words: the first lane of its segment (for Lane also the idle lanes,
// which have row 0: the callers' guards leave them out)
__device__ __forceinline__ bool leader(const Lane& L) { return L.row == 0; }
__device__ __forceinline__ bool leader(const Lane2& L) { return L.li == 0 && L.active; }
// per-game items strided over the game's lanes: for (i = seg_first(L); i < n; i += seg_stride<N>(L))
__device__ __forceinline__ int seg_first(const Lane& L) { return L.row; }
__device__ __forceinline__ int seg_first(const Lane2& L) { return L.li; }
template <int N>
__device__ __forceinline__ int seg_stride(const Lane&) { return N; }
template <int N>
__device__ __forceinline__ int seg_stride(const Lane2&) { return Geo2<N>::LPG; }
// this lane's part of the playout checksum's legal-mask term (pp_row_term of each of its rows)
template <int N>
__device__ __forceinline__ uint64_t row_term(uint32_t legal, const Lane& L) {
  return L.active ? pp_row_term((uint32_t)L.row, legal) : 0ull;
}
template <int N>
__device__ __forceinline__ uint64_t row_term(P2 legal, const Lane2& L) {
  uint64_t rt = 0;
  if (L.active) {
    rt = pp_row_term((uint32_t)(2 * L.li), legal.lo);
    if (2 * L.li + 1 < N) rt ^= pp_row_term((uint32_t)(2 * L.li + 1), legal.hi);
  }
  return rt;
}

// Legal rows of the side to move: TryPlay for meta.next (empty, not the simple-ko point, not suicide).
template <int N, class Rows, class LaneT>
__device__ __forceinline__ Rows legal_for_next(Rows b, Rows w, Rows safe, Rows atari, const BoardMeta& meta,
                                               const LaneT& L) {
  const Rows own = meta.next == S_BLACK ? b : w, opp = meta.next == S_BLACK ? w : b;
  const bool ko_applies = (meta.flags & F_KO_ACTIVE) && meta.ko_color == meta.next;
  return legal_rows_cached<N>(own, opp, safe, atari, L, ko_applies, meta.ko_pt);
}

// ---------------------------------------------------------------------------------------
// GoState::reset of game g: the empty position, every point legal, no history, no superko record.
// Each lane writes its own row (and row 0 the per-game words).
template <int N>
__device__ __forceinline__ void store_empty(const DevState& st, int g, const Lane& L) {
  st.cur[(size_t)g * N + L.row] = 0;
  st.sa[(size_t)g * N + L.row] = 0;
  st.legal[(size_t)g * N + L.row] = Geo<N>::ROWMASK;  // every point of the empty board is legal
  for (int s = 0; s < 8; ++s) st.ring[((size_t)g * 8 + s) * N + L.row] = 0;
  for (int x = 0; x < N; ++x) st.placed[(size_t)g * Geo<N>::P + L.row * N + x] = 0;
  if (L.row == 0) {
    st.hash[g] = 0;
    store_meta(&st.meta[g], initial_meta());
    st.sk_n[g] = 0;
  }
}

template <int N>
__global__ void __launch_bounds__(BLOCK) k_reset(DevState st, const uint8_t* __restrict__ mask) {
  const Lane L = make_lane<N>();
  bool valid;
  const int g = warp_game<N>(L, st.G, valid);
  if (!valid) return;
  if (mask && !mask[g]) return;
  store_empty<N>(st, g, L);
}

// ---------------------------------------------------------------------------------------
// A game's position in registers for GoState::forward: forward_ply plays one move on it.
struct Forward {
  uint32_t b, w, safe, atari;
  BoardMeta meta;
  uint64_t hash;
  uint32_t lrow, lnew;  // legal rows before / after the move
  int pm;               // the move played (p = y*N+x or MV_PASS), MV_NONE if refused or none
};

// GoState::forward (go_state.cc:74-94) of action `a` (x*N + y, N*N = pass, anything else none) on the position
// in `f`: refused on a terminated game and when it is not in the legal rows f.lrow (go_state.cc:78-83), else
// played; the new position is compared with the recorded pre-move positions skg[0 .. nsk) and its pre-move hash
// appended (go_state.cc:96-121).  Leaves the move in f.pm and the legal rows of the new position in f.lnew.
// Every lane of the warp calls it (warp collectives); idle lanes have valid = false.
template <int N>
__device__ __forceinline__ void forward_ply(Forward& f, int a, bool valid, uint64_t* skg, int& nsk,
                                            const uint64_t* s_zob, const Lane& L) {
  const bool term = is_terminated<N>(f.meta);
  int pm = MV_NONE;
  if (valid && !term) {
    if (a == Geo<N>::P) {
      pm = MV_PASS;
    } else if (a >= 0 && a < Geo<N>::P) {
      pm = (a % N) * N + (a / N);  // a = x*N + y  ->  p = y*N + x
    }
  }
  {
    const int y = pm >= 0 ? pm / N : -1, x = pm >= 0 ? pm - y * N : 0;
    const bool bit = (L.row == y) && ((f.lrow >> x) & 1u);
    const bool is_legal = game_any<N>(bit, L);
    if (pm >= 0 && !is_legal) pm = MV_NONE;
  }
  const uint64_t pre_hash = f.hash;
  play_move_cached<N>(f.b, f.w, f.meta, f.hash, pm, s_zob, L, f.safe, f.atari);
  const bool sko = superko_scan<N>(skg, pm >= 0 ? nsk : 0, f.hash, L);
  // Not needed for the record (the scan reads skg[0 .. nsk) and ends in a warp vote; the append writes skg[nsk]).
  // It costs nothing, and without it k_env_step<9> is allocated 51 registers instead of 48.
  __syncwarp();
  if (pm >= 0) {
    if (sko) f.meta.flags |= F_SUPERKO;
    if (valid && L.row == 0) skg[nsk] = pre_hash;
    nsk++;
  }
  f.lnew = legal_for_next<N>(f.b, f.w, f.safe, f.atari, f.meta, L);
  f.pm = pm;
}

// forward_ply on game g's stored position, the body of k_step and k_env_step.  The new position is left in `f`
// (store_position writes it); only the superko record is written here.
template <int N>
__device__ __forceinline__ void forward_game(const DevState& st, const int32_t* __restrict__ actions, int g, int gs,
                                             bool valid, const Lane& L, const uint64_t* s_zob, Forward& f) {
  load_row<N>(st.cur, gs, L.row, valid, f.b, f.w);
  // the incremental group status (safe / atari masks, board.cuh) is part of the stored position: a step
  // recounts only the groups the move touched instead of classifying every group from scratch
  load_row<N>(st.sa, gs, L.row, valid, f.safe, f.atari);
  f.meta = load_meta(&st.meta[gs]);
  f.hash = st.hash[gs];
  f.lrow = valid ? st.legal[(size_t)gs * N + L.row] : 0u;
  int nsk = st.sk_n[gs];
  forward_ply<N>(f, valid ? actions[gs] : -1, valid, st.sk + (size_t)gs * Geo<N>::MAX_PLY, nsk, s_zob, L);
  if (f.pm >= 0 && L.row == 0) st.sk_n[g] = nsk;
}

// The position forward_game left in `f` becomes game g's stored position (called when a move was played).
template <int N>
__device__ __forceinline__ void store_position(const DevState& st, int g, const Lane& L, const Forward& f) {
  store_row<N>(st.cur, g, L.row, f.b, f.w);
  store_row<N>(st.sa, g, L.row, f.safe, f.atari);
  st.ring[((size_t)g * 8 + ((f.meta.ply - 2) & 7)) * N + L.row] = pack_row(f.b, f.w);  // go_state.cc:90-92
  st.legal[(size_t)g * N + L.row] = f.lnew;
  if (L.row == 0) {
    st.hash[g] = f.hash;
    store_meta(&st.meta[g], f.meta);
    if (f.pm >= 0) st.placed[(size_t)g * Geo<N>::P + f.pm] = (uint16_t)(f.meta.ply - 1);  // Info::last_placed = _ply (board.cc:680,1379)
  }
}

// GoState::forward (go_state.cc:74-94) for all games.
template <int N>
__global__ void __launch_bounds__(BLOCK)
    k_step(DevState st, const int32_t* __restrict__ actions, uint8_t* __restrict__ ok, unsigned* done_count,
           volatile uint32_t* done_flag, uint32_t seq, uint8_t* ok_mapped) {
  __shared__ uint64_t s_zob[Geo<N>::ZOB];
  load_zobrist<N>(s_zob);
  const Lane L = make_lane<N>();
  bool valid;
  const int g = warp_game<N>(L, st.G, valid);
  const int gs = valid ? g : 0;  // safe index for idle lanes (loads only)
  Forward f;
  forward_game<N>(st, actions, g, gs, valid, L, s_zob, f);
  if (valid) {
    if (f.pm != MV_NONE) store_position<N>(st, g, L, f);
    if (ok && L.row == 0) ok[g] = f.pm != MV_NONE ? 1 : 0;
  }
  // host-driven step (elfb200_step): the last CTA to finish copies the accept flags to the mapped host window
  // in 16-byte pieces (4096 one-byte PCIe writes from as many warps measured ~14 us) and raises the completion
  // flag there, so the host spins on a word instead of paying a stream synchronisation.
  if (done_flag) {
    __shared__ bool s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();  // this CTA's accept flags are visible device-wide before it counts itself done
      s_last = atomicAdd(done_count, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last) {
      __threadfence();
      const int n16 = st.G / 16;
      const uint4* src = reinterpret_cast<const uint4*>(ok);
      uint4* dst = reinterpret_cast<uint4*>(ok_mapped);
      for (int i = threadIdx.x; i < n16; i += blockDim.x) dst[i] = __ldcg(src + i);
      for (int i = n16 * 16 + threadIdx.x; i < st.G; i += blockDim.x) ok_mapped[i] = __ldcg(ok + i);
      __threadfence_system();
      __syncthreads();
      if (threadIdx.x == 0) {
        *done_count = 0u;
        *done_flag = seq;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------
// GoStateExtOffline::switchBeforeMove (common/go_state_ext.h:305-312) for all games in one launch:
// every game starts from the empty board and forwards its own move list, moves[g][0 .. count[g]).
// Per ply this is k_step's forward_ply with the position held in registers; a refused move changes
// nothing and the list goes on, as the reference ignores forward()'s verdict there.  Games of one warp
// (9x9 packs three) may have different lengths: the warp runs to the longest, shorter games idle with
// MV_NONE.
template <int N>
__global__ void __launch_bounds__(BLOCK)
    k_replay(DevState st, const int16_t* __restrict__ moves, int stride, const int32_t* __restrict__ count) {
  __shared__ uint64_t s_zob[Geo<N>::ZOB];
  load_zobrist<N>(s_zob);
  const Lane L = make_lane<N>();
  bool valid;
  const int g = warp_game<N>(L, st.G, valid);
  const int gs = valid ? g : 0;  // safe index for idle lanes (loads only)

  Forward f;
  f.b = f.w = f.safe = f.atari = 0;
  f.meta = initial_meta();
  f.hash = 0;
  f.lrow = valid ? Geo<N>::ROWMASK : 0u;  // every point of the empty board is legal
  int nsk = 0;
  if (valid) {
    for (int s = 0; s < 8; ++s) st.ring[((size_t)g * 8 + s) * N + L.row] = 0;
    for (int x = 0; x < N; ++x) st.placed[(size_t)g * Geo<N>::P + L.row * N + x] = 0;
  }
  __syncwarp();
  const int n = valid ? count[gs] : 0;
  const int nmax = __reduce_max_sync(FULL, n);
  uint64_t* skg = st.sk + (size_t)gs * Geo<N>::MAX_PLY;

  for (int t = 0; t < nmax; ++t) {
    forward_ply<N>(f, (valid && t < n) ? (int)moves[(size_t)gs * stride + t] : -1, valid, skg, nsk, s_zob, L);
    if (valid && f.pm != MV_NONE) {
      f.lrow = f.lnew;
      st.ring[((size_t)g * 8 + ((f.meta.ply - 2) & 7)) * N + L.row] = pack_row(f.b, f.w);  // go_state.cc:90-92
      if (f.pm >= 0 && L.row == 0) st.placed[(size_t)g * Geo<N>::P + f.pm] = (uint16_t)(f.meta.ply - 1);
    }
    __syncwarp();  // the next ply's superko scan reads the hash this one appended
  }
  if (valid) {
    store_row<N>(st.cur, g, L.row, f.b, f.w);
    store_row<N>(st.sa, g, L.row, f.safe, f.atari);
    st.legal[(size_t)g * N + L.row] = f.lrow;
    if (L.row == 0) {
      st.hash[g] = f.hash;
      store_meta(&st.meta[g], f.meta);
      st.sk_n[g] = nsk;
    }
  }
}

// ---------------------------------------------------------------------------------------
// GoState::applyHandicap / PlaceHandicap (go_state.cc:62-71,130-132; board.cc:109-126) for all games in one
// launch: game g places the BLACK stones stones[g][0 .. count[g]) in order.  Each stone is TryPlay for black,
// whoever is to move (after the first stone white is, so the stored legal rows are not black's: black's
// rows are computed here), then Play; afterwards the ply goes back to 1 and the last-move window to "none".
// PlaceHandicap bypasses GoState::forward, so neither the superko record nor the history ring is written.
// A game past ply 1 refuses every stone and is left as it is.  Games of one warp (9x9 packs three) may have
// lists of different lengths: the warp runs to the longest, as in k_replay.
template <int N>
__global__ void __launch_bounds__(BLOCK)
    k_place(DevState st, const int16_t* __restrict__ stones, int stride, const int32_t* __restrict__ count,
            uint8_t* __restrict__ ok) {
  __shared__ uint64_t s_zob[Geo<N>::ZOB];
  load_zobrist<N>(s_zob);
  const Lane L = make_lane<N>();
  bool valid;
  const int g = warp_game<N>(L, st.G, valid);
  const int gs = valid ? g : 0;  // safe index for idle lanes (loads only)

  uint32_t b, w, safe, atari;
  load_row<N>(st.cur, gs, L.row, valid, b, w);
  load_row<N>(st.sa, gs, L.row, valid, safe, atari);
  BoardMeta meta = load_meta(&st.meta[gs]);
  uint64_t hash = st.hash[gs];
  const bool open = valid && meta.ply <= 1;  // "the game has already started" (board.cc:111-112)
  const int n = valid ? count[gs] : 0;
  const int nmax = __reduce_max_sync(FULL, n);

  for (int t = 0; t < nmax; ++t) {
    const int a = t < n ? (int)stones[(size_t)gs * stride + t] : -1;
    int pm = (open && a >= 0) ? (a % N) * N + (a / N) : MV_NONE;  // a = x*N + y  ->  p = y*N + x
    {
      // TryPlay(board, x, y, S_BLACK) (board.cc:788-827): empty, no simple-ko violation, not suicide
      const bool ko_black = (meta.flags & F_KO_ACTIVE) && meta.ko_color == S_BLACK;
      const uint32_t lb = legal_rows_cached<N>(b, w, safe, atari, L, ko_black, meta.ko_pt);
      const int y = pm >= 0 ? pm / N : -1, x = pm >= 0 ? pm - y * N : 0;
      const bool bit = (L.row == y) && ((lb >> x) & 1u);
      const bool is_legal = game_any<N>(bit, L);
      if (pm >= 0 && !is_legal) pm = MV_NONE;
    }
    if (pm >= 0) meta.next = S_BLACK;  // Play for ids->player == S_BLACK; leaves white to move
    play_move_cached<N>(b, w, meta, hash, pm, s_zob, L, safe, atari);
    if (pm >= 0) {
      meta.ply = 1;  // board.cc:117-122
      meta.last1 = meta.last2 = MV_INVALID;
      if (L.row == 0) st.placed[(size_t)g * Geo<N>::P + pm] = 1;  // Info::last_placed = _ply (board.cc:1379)
    }
    if (ok && valid && L.row == 0 && t < n) ok[(size_t)g * stride + t] = pm >= 0 ? 1 : 0;
  }

  const uint32_t lnew = legal_for_next<N>(b, w, safe, atari, meta, L);
  if (open) {
    store_row<N>(st.cur, g, L.row, b, w);
    store_row<N>(st.sa, g, L.row, safe, atari);
    st.legal[(size_t)g * N + L.row] = lnew;
    if (L.row == 0) {
      st.hash[g] = hash;
      store_meta(&st.meta[g], meta);
    }
  }
}

// ---------------------------------------------------------------------------------------
// Host-facing views of one game, shared by k_export and k_env_step.
// legal uint8[G][N*N+1] by action index (elfb200_get_legal): this lane's legal row `l`, pass always legal.
template <int N>
__device__ __forceinline__ void write_legal(uint8_t* __restrict__ legal_out, int g, const Lane& L, uint32_t l) {
  constexpr int P = Geo<N>::P;
  for (int x = 0; x < N; ++x) legal_out[(size_t)g * (P + 1) + x * N + L.row] = (l >> x) & 1u;
  if (L.row == 0) legal_out[(size_t)g * (P + 1) + P] = 1;
}

// info int32[ELFB200_INFO_FIELDS] of one game (elfb200_get_info)
template <int N>
__device__ __forceinline__ void write_info(int32_t* __restrict__ o, const BoardMeta& meta) {
  auto p2a = [](int p) -> int {
    if (p == MV_PASS) return Geo<N>::P;
    if (p < 0) return -1;
    return (p % N) * N + p / N;
  };
  o[0] = meta.ply;
  o[1] = meta.next;
  o[2] = meta.b_cap;
  o[3] = meta.w_cap;
  o[4] = p2a(meta.last1);
  o[5] = p2a(meta.last2);
  o[6] = (meta.flags & F_KO_ACTIVE) ? p2a(meta.ko_pt) : -1;
  o[7] = meta.ko_color;
  o[8] = 0;
  o[9] = is_terminated<N>(meta) ? 1 : 0;
  o[10] = (meta.last1 == MV_PASS && meta.last2 == MV_PASS) ? 1 : 0;
  o[11] = (meta.flags & F_SUPERKO) ? 1 : 0;
}

template <int N>
__global__ void __launch_bounds__(BLOCK)
    k_export(DevState st, uint8_t* __restrict__ legal_out, uint8_t* __restrict__ stones_out,
             uint8_t* __restrict__ eyes_out, int eye_player, int32_t* __restrict__ info_out,
             int32_t* __restrict__ score_out) {
  const Lane L = make_lane<N>();
  bool valid;
  const int g = warp_game<N>(L, st.G, valid);
  const int gs = valid ? g : 0;
  uint32_t b, w;
  load_row<N>(st.cur, gs, L.row, valid, b, w);
  const BoardMeta meta = load_meta(&st.meta[gs]);
  constexpr int P = Geo<N>::P;
  if (legal_out && valid) write_legal<N>(legal_out, g, L, st.legal[(size_t)g * N + L.row]);
  if (stones_out && valid) {
    for (int x = 0; x < N; ++x)
      stones_out[(size_t)g * P + x * N + L.row] = ((b >> x) & 1u) | (((w >> x) & 1u) << 1);
  }
  if (eyes_out) {  // warp-collective: no early exit
    int pl = eye_player ? eye_player : meta.next;
    const uint32_t own = pl == S_BLACK ? b : w, opp = pl == S_BLACK ? w : b;
    const uint32_t eye = true_eye_rows<N>(own, opp, L);
    if (valid)
      for (int x = 0; x < N; ++x) eyes_out[(size_t)g * P + x * N + L.row] = (eye >> x) & 1u;
  }
  if (score_out) {
    const int sc = tt_score<N>(b, w, L);
    if (valid && L.row == 0) score_out[g] = sc;
  }
  if (info_out && valid && L.row == 0) write_info<N>(info_out + (size_t)g * ELFB200_INFO_FIELDS, meta);
}

// ---------------------------------------------------------------------------------------
// One ply of the device-resident environment (elfb200_env_step): GoState::forward of every game as k_step
// does, then every game that has ended (GoState::terminated: two passes, positional superko or the 2N^2
// ply cap; also a game stepped to its end through the other entry points, whatever its action) is scored
// with GoState::evaluate(komi) and restarted from the empty position as k_reset does.  legal / info
// describe the position now stored.  Each output may be NULL.
template <int N>
__global__ void __launch_bounds__(BLOCK)
    k_env_step(DevState st, const int32_t* __restrict__ actions, float komi, uint8_t* __restrict__ ok,
               uint8_t* __restrict__ done_out, float* __restrict__ value, uint8_t* __restrict__ legal_out,
               int32_t* __restrict__ info_out) {
  __shared__ uint64_t s_zob[Geo<N>::ZOB];
  load_zobrist<N>(s_zob);
  const Lane L = make_lane<N>();
  bool valid;
  const int g = warp_game<N>(L, st.G, valid);
  const int gs = valid ? g : 0;  // safe index for idle lanes (loads only)
  Forward f;
  forward_game<N>(st, actions, g, gs, valid, L, s_zob, f);

  // GoState::evaluate (go_state.h:194-203) in elfb200_evaluate's float arithmetic, black's point of view.
  // tt_score is a warp collective: it runs when any game of the warp has ended, on every lane.
  const bool done = valid && is_terminated<N>(f.meta);
  float v = 0.f;
  if (__any_sync(FULL, done)) {
    const int sc = tt_score<N>(f.b, f.w, L);
    if (done) v = (f.meta.flags & F_SUPERKO) ? (f.meta.next == S_BLACK ? 1.0f : -1.0f) : (float)sc - komi;
  }
  if (!valid) return;
  if (done)
    store_empty<N>(st, g, L);
  else if (f.pm != MV_NONE)
    store_position<N>(st, g, L, f);
  if (legal_out) write_legal<N>(legal_out, g, L, done ? Geo<N>::ROWMASK : f.pm != MV_NONE ? f.lnew : f.lrow);
  if (L.row == 0) {
    if (info_out) write_info<N>(info_out + (size_t)g * ELFB200_INFO_FIELDS, done ? initial_meta() : f.meta);
    if (ok) ok[g] = f.pm != MV_NONE ? 1 : 0;
    if (done_out) done_out[g] = done ? 1 : 0;
    if (value) value[g] = v;
  }
}

// ---------------------------------------------------------------------------------------
// BoardFeature::extractAGZ (board_feature.cc:247-290).  The 8 history positions of a game come
// from its ring; staging, formats and the bulk store are features_cta's (common.cuh).
template <int N>
struct RingGather {
  DevState st;
  const int32_t* d4codes;
  __device__ __forceinline__ void operator()(int g, uint64_t (*rows)[N], int& hn, int& next, int& d4) const {
    const BoardMeta meta = load_meta(&st.meta[g]);
    hn = min(8, (int)meta.ply - 1);
    next = meta.next;
    d4 = d4codes ? d4codes[g] : 0;
    for (int i = threadIdx.x; i < 8 * N; i += blockDim.x) {
      const int t = i / N, y = i - t * N;
      rows[t][y] = t < hn ? st.ring[((size_t)g * 8 + ((meta.ply - 2 - t) & 7)) * N + y] : 0ull;
    }
  }
};

template <int N>
__global__ void __launch_bounds__(FEAT_THREADS)
    k_features(DevState st, const int32_t* __restrict__ d4codes, void* __restrict__ out, int fmt, int cpad, int tma) {
  features_cta<N>(RingGather<N>{st, d4codes}, st.G, out, fmt, cpad, tma);
}

// ---------------------------------------------------------------------------------------
// BoardFeature::extract (board_feature.cc:209-237): the 25-plane DarkForest feature set
// (GameOptions::use_df_feature), float32 [G][25][N][N] under a D4 code.  Filled planes (board_feature.h:19-36):
// 0-2 our groups with 1 / 2 / >=3 liberties, 3-5 the opponent's, 6 the simple-ko point, 7 / 8 / 9 our /
// opponent / empty points, 10 / 11 exp((last_placed - ply) / 10) on our / the opponent's stones, 14 / 15 the
// L1 distance to the nearest stone of ours / theirs (10000 if there is none), 16 / 17 black / white to move;
// the other planes stay zero.  One warp = one game (row per lane); the planes are staged in shared
// memory in OUTPUT order (cell = Transform(x, y), board_feature.h:97-113) and leave coalesced.
// Not on the self-play hot path (AGZ features are); built for parity of the offline/DF path.
template <int N>
__global__ void __launch_bounds__(32)
    k_features_df(DevState st, const int32_t* __restrict__ d4codes, const float* __restrict__ exp_tab,
                  float* __restrict__ out) {
  constexpr int P = Geo<N>::P;
  __shared__ float tile[25 * P];
  __shared__ uint8_t hd[N][N];
  const Lane L = make_lane_single<N>();
  const int g = blockIdx.x;
  if (g >= st.G) return;
  uint32_t b, w;
  load_row<N>(st.cur, g, L.row, L.active, b, w);
  const BoardMeta meta = load_meta(&st.meta[g]);
  const int d4 = d4codes ? d4codes[g] : 0;
  const bool bf = meta.next == S_BLACK;
  const uint32_t own = bf ? b : w, opp = bf ? w : b;
  const uint32_t e = ~(own | opp) & L.rm;
  for (int i = L.lane; i < 25 * P; i += 32) tile[i] = 0.f;
  __syncwarp();
  auto cell = [&](int x, int y) -> int {  // Transform: rotate, then flip
    int ta, tb;
    switch (d4 & 3) {
      case 1: ta = y; tb = N - 1 - x; break;
      case 2: ta = N - 1 - x; tb = N - 1 - y; break;
      case 3: ta = N - 1 - y; tb = x; break;
      default: ta = x; tb = y; break;
    }
    return (d4 & 4) ? tb * N + ta : ta * N + tb;
  };
  const uint16_t* placed = st.placed + (size_t)g * P;
  if (L.active) {
    for (int x = 0; x < N; ++x) {
      const int c = cell(x, L.row);
      const bool ob = (own >> x) & 1u, pb = (opp >> x) & 1u;
      tile[7 * P + c] = ob ? 1.f : 0.f;
      tile[8 * P + c] = pb ? 1.f : 0.f;
      tile[9 * P + c] = (ob || pb) ? 0.f : 1.f;
      if (ob || pb) tile[(ob ? 10 : 11) * P + c] = exp_tab[(int)meta.ply - (int)placed[L.row * N + x]];
      tile[(bf ? 16 : 17) * P + c] = 1.f;
    }
  }
  if (L.lane == 0 && (meta.flags & F_KO_ACTIVE) && meta.ko_pt >= 0)  // getSimpleKoLocation, board.cc:466-474
    tile[6 * P + cell(meta.ko_pt % N, meta.ko_pt / N)] = 1.f;
  // liberty classes, group by group (getLibertyMap3binary, board_feature.cc:93-113)
  {
    const Links k = make_links<N>(own, opp, L);
    uint32_t todo = own | opp;
    while (__any_sync(FULL, todo != 0u)) {
      const uint32_t bal = __ballot_sync(FULL, todo != 0u);
      const int src = __ffs(bal) - 1;
      uint32_t grp = (L.lane == src) ? (todo & (0u - todo)) : 0u;
      while (true) {
        const uint32_t g1 = grow_link(grp, k);
        const uint32_t g2 = grow_link(g1, k);
        const bool ch = g2 != grp;
        grp = g2;
        if (!__any_sync(FULL, ch)) break;
      }
      const int nl = __reduce_add_sync(FULL, __popc(nbr4<N>(grp, L) & e));
      const bool ours = __any_sync(FULL, (grp & own) != 0u);
      const int plane = (ours ? 0 : 3) + (nl == 1 ? 0 : nl == 2 ? 1 : 2);
      for (uint32_t m = grp; m; m &= m - 1) tile[plane * P + cell(__ffs(m) - 1, L.row)] = 1.f;
      todo &= ~grp;
    }
  }
  // distance to the nearest stone of each colour (getDistanceMap + DistanceTransform, board_feature.cc:20-40,
  // 181-196): the two 1-D min-plus sweeps there are the exact L1 distance transform, which commutes with D4
  for (int side = 0; side < 2; ++side) {
    const uint32_t row = side == 0 ? own : opp;
    __syncwarp();
    if (L.active) {
      for (int x = 0; x < N; ++x) {
        int d = 255;
        const uint32_t lo = row & ((2u << x) - 1u), hi = row >> x;
        if (lo) d = x - (31 - __clz(lo));
        if (hi) d = min(d, __ffs(hi) - 1);
        hd[L.row][x] = (uint8_t)d;
      }
    }
    __syncwarp();
    const bool none = !__any_sync(FULL, row != 0u);
    if (L.active) {
      for (int x = 0; x < N; ++x) {
        int best = 100000;
        for (int y2 = 0; y2 < N; ++y2) {
          const int h = hd[y2][x];
          if (h != 255) best = min(best, h + (y2 > L.row ? y2 - L.row : L.row - y2));
        }
        tile[(14 + side) * P + cell(x, L.row)] = none ? 10000.f : (float)best;
      }
    }
  }
  __syncwarp();
  float* dst = out + (size_t)g * 25 * P;
  for (int i = L.lane; i < 25 * P; i += 32) dst[i] = tile[i];
}

// ---------------------------------------------------------------------------------------
// One warp per CTA in the playout kernels: 4096 games are 4096 warps over 132 SMs = 31.03 per SM; with
// 4-warp CTAs the SMs holding 8 CTAs (32 warps) set the kernel time while those with 7 idle 12.5 % of it.
constexpr int PLAYOUT_WARPS = 1;

// 4096-bit Bloom filter of one game segment over its recorded pre-move hashes, two bits per hash: the exact
// superko scan (go_state.cc:96-111) only runs when both bits of the new position's hash are set (false-positive
// rate ~3 % at 400 recorded positions), which removes ~1.8 KB of history reads per ply.
template <int N, class LaneT>
__device__ __forceinline__ void bloom_clear(uint32_t* bloom, const LaneT& L) {
  for (int i = seg_first(L); i < 128; i += seg_stride<N>(L)) bloom[i] = 0u;
}
__device__ __forceinline__ bool bloom_probe(const uint32_t* bloom, uint64_t h) {
  const uint32_t q1 = (uint32_t)h & 4095u, q2 = (uint32_t)(h >> 12) & 4095u;
  return (bloom[q1 >> 5] >> (q1 & 31)) & (bloom[q2 >> 5] >> (q2 & 31)) & 1u;
}
// `atomic`: several lanes of the segment insert at the same time
__device__ __forceinline__ void bloom_insert(uint32_t* bloom, uint64_t h, bool atomic) {
  const uint32_t i1 = (uint32_t)h & 4095u, i2 = (uint32_t)(h >> 12) & 4095u;
  if (atomic) {
    atomicOr(&bloom[i1 >> 5], 1u << (i1 & 31));
    atomicOr(&bloom[i2 >> 5], 1u << (i2 & 31));
  } else {
    bloom[i1 >> 5] |= 1u << (i1 & 31);
    bloom[i2 >> 5] |= 1u << (i2 & 31);
  }
}

// One move of the random policy (include/elfb200_playout_policy.h) on a position held in registers, in either
// lane layout: of the n legal moves of the side to move that do not fill one of its true eyes, candidate
// pp_pick(seed, draw_id, ply, n) in action order, a pass when n == 0, no move when `term`.  Then GoState::forward's
// superko test against the record skg[0 .. nsk), gated by the Bloom filter, and the pre-move hash goes into the
// record and the filter.  `chk` (may be NULL): the playout checksum, folded with the position before the move
// unless `term`.
template <int N, class Rows, class LaneT>
__device__ __forceinline__ void random_ply(uint64_t seed, uint64_t draw_id, bool term, Rows& b, Rows& w, Rows& safe,
                                           Rows& atari, BoardMeta& meta, uint64_t& hash, uint64_t* chk, uint64_t* skg,
                                           int& nsk, uint32_t* bloom, const uint64_t* s_zob, const LaneT& L) {
  const Rows own = meta.next == S_BLACK ? b : w, opp = meta.next == S_BLACK ? w : b;
  const Rows legal = legal_for_next<N>(b, w, safe, atari, meta, L);
  const Rows cand = legal & ~true_eye_rows<N>(own, opp, L);
  const int n = game_sum<N>(popc_rows(cand), L);
  if (chk) {
    const uint64_t rx = game_xor64<N>(row_term<N>(legal, L), L);
    const uint64_t chk2 = pp_fold3(*chk, hash, rx, meta.b_cap, meta.w_cap, meta.next);
    if (!term) *chk = chk2;
  }
  const int k = n > 0 ? (int)pp_pick(seed, draw_id, meta.ply, (uint32_t)n) : 0;
  const int p = select_kth_action_order<N>(cand, k, L);
  const int pm = term ? MV_NONE : (n > 0 ? p : MV_PASS);
  const uint64_t pre_hash = hash;
  play_move_cached<N>(b, w, meta, hash, pm, s_zob, L, safe, atari);
  const bool maybe = pm >= 0 && bloom_probe(bloom, hash);
  bool sko = false;
  if (__any_sync(FULL, maybe)) sko = superko_scan<N>(skg, maybe ? nsk : 0, hash, L);
  __syncwarp();  // every lane has probed the filter before it changes
  if (pm >= 0) {
    if (sko) meta.flags |= F_SUPERKO;
    if (leader(L)) {
      skg[nsk] = pre_hash;
      bloom_insert(bloom, pre_hash, false);
    }
    nsk++;
  }
  __syncwarp();  // the next move's probe and scan see this one's record
}

// Whole random-policy games, position in registers (BASELINE configs 1/2/5): the body of k_playout and
// k_playout2, game g of the batch on lane L's segment, whose Bloom filter is `bloom`.
//
// stream_plies == 0: every slot plays ONE game (id first_id + g) to terminated() / max_plies.
// stream_plies  > 0: "4096 concurrent games" in steady state -- every slot plays exactly
//   stream_plies plies, starting a new game (id += G) whenever its game ends, so that G games are
//   in flight at all times like the reference's game threads (GoGameBase::mainLoop,
//   common/game_base.h:41).  Per slot: out_chk = fold of the games' checksums in order,
//   out_plies = plies played, out_score = number of games started, out_hash = last position hash.
template <int N, class LaneT>
__device__ __forceinline__ void playout_body(const LaneT& L, int g, bool valid, uint32_t* bloom, const uint64_t* s_zob,
                                             int G, uint64_t seed, uint64_t first_id, int max_plies, int stream_plies,
                                             uint64_t* __restrict__ sk, uint64_t* __restrict__ out_chk,
                                             int32_t* __restrict__ out_plies, int32_t* __restrict__ out_score,
                                             uint64_t* __restrict__ out_hash) {
  using Rows = decltype(LaneT::rm);
  uint64_t gid = first_id + (uint64_t)g;
  uint64_t* skg = sk + (size_t)(valid ? g : 0) * Geo<N>::MAX_PLY;
  if (L.active) bloom_clear<N>(bloom, L);
  __syncwarp();

  // safe/atari: incremental group status (board.cuh)
  Rows b = zero_rows(L), w = zero_rows(L), safe = zero_rows(L), atari = zero_rows(L);
  BoardMeta meta = initial_meta();
  uint64_t hash = 0, chk = 0, acc = 0;
  int nsk = 0, t = 0, ts = 0, ngames = 0;
  const bool stream = stream_plies > 0;

  while (true) {
    const bool over = is_terminated<N>(meta) || t >= max_plies;
    bool term;
    if (stream) {
      const bool budget_out = ts >= stream_plies;
      const bool restart = valid && over && !budget_out;
      if (__any_sync(FULL, restart)) {
        if (restart) {  // finish this game, start the slot's next one
          acc = pp_splitmix64(acc ^ pp_fold_final(chk, hash, meta.ply));
          ngames++;
          gid += (uint64_t)G;
          b = w = safe = atari = zero_rows(L);
          meta = initial_meta();
          hash = chk = 0;
          nsk = t = 0;
          bloom_clear<N>(bloom, L);
        }
        __syncwarp();
      }
      term = !valid || budget_out;
    } else {
      term = !valid || over;
    }
    if (__all_sync(FULL, term)) break;
    random_ply<N>(seed, gid, term, b, w, safe, atari, meta, hash, &chk, skg, nsk, bloom, s_zob, L);
    if (!term) {
      t++;
      ts++;
    }
  }
  chk = pp_fold_final(chk, hash, meta.ply);
  const int score = tt_score<N>(b, w, L);
  if (valid && leader(L)) {
    if (stream) {
      if (out_chk) out_chk[g] = pp_splitmix64(acc ^ chk);
      if (out_plies) out_plies[g] = ts;
      if (out_score) out_score[g] = ngames + 1;
    } else {
      if (out_chk) out_chk[g] = chk;
      if (out_plies) out_plies[g] = t;
      if (out_score) out_score[g] = score;
    }
    if (out_hash) out_hash[g] = hash;
  }
}

template <int N>
__global__ void __launch_bounds__(PLAYOUT_WARPS * 32)
    k_playout(int G, uint64_t seed, uint64_t first_id, int max_plies, int stream_plies,
              uint64_t* __restrict__ sk, uint64_t* __restrict__ out_chk, int32_t* __restrict__ out_plies,
              int32_t* __restrict__ out_score, uint64_t* __restrict__ out_hash) {
  __shared__ uint64_t s_zob[Geo<N>::ZOB];
  __shared__ uint32_t s_bloom[PLAYOUT_WARPS][Geo<N>::GPW][128];
  load_zobrist<N>(s_zob);
  const Lane L = make_lane<N>();
  bool valid;
  const int g = warp_game<N>(L, G, valid);
  playout_body<N>(L, g, valid, s_bloom[threadIdx.x >> 5][L.sub], s_zob, G, seed, first_id, max_plies, stream_plies,
                  sk, out_chk, out_plies, out_score, out_hash);
}

// k_playout in the two-rows-per-lane layout (board2.cuh): three 19x19 games per warp, 30 of 32 lanes
// busy.  Same workload, same outputs, same checksums as k_playout (elfb200_set_playout_layout picks).
template <int N>
__global__ void __launch_bounds__(PLAYOUT_WARPS * 32)
    k_playout2(int G, uint64_t seed, uint64_t first_id, int max_plies, int stream_plies,
               uint64_t* __restrict__ sk, uint64_t* __restrict__ out_chk, int32_t* __restrict__ out_plies,
               int32_t* __restrict__ out_score, uint64_t* __restrict__ out_hash) {
  __shared__ uint64_t s_zob[Geo<N>::ZOB];
  __shared__ uint32_t s_bloom[PLAYOUT_WARPS][Geo2<N>::GPW][128];
  load_zobrist<N>(s_zob);
  const Lane2 L = make_lane2<N>();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int g = warp * Geo2<N>::GPW + L.sub;
  const bool valid = L.active && g < G;
  playout_body<N>(L, g, valid, s_bloom[threadIdx.x >> 5][L.sub], s_zob, G, seed, first_id, max_plies, stream_plies,
                  sk, out_chk, out_plies, out_score, out_hash);
}

// ---------------------------------------------------------------------------------------
// GoState's copy constructor (go_state.h:117-124, copyBoard board.cc:128-132) from one batch into another:
// dst game i := src game index[i] for index[i] in [0, src.G); any other value leaves game i as it is.  A
// game's stored state is its DevState blocks and nothing else, so the copy needs no board geometry and one
// kernel serves both board sizes: one warp per destination game, the lanes striding over each per-game
// block in the widest word its alignment allows (16 B for the history ring and the superko record, whose
// per-game blocks are multiples of 16 B; 8 / 4 / 2 B for the rows and `placed`).  Of the superko record only
// sk[0 .. sk_n) is copied: every reader (superko_scan in k_step / k_env_step / k_replay, the search's tree
// descent) stops at sk_n and every writer appends at sk_n.
constexpr int GATHER_THREADS = 256;

__global__ void __launch_bounds__(GATHER_THREADS)
    k_gather(DevState dst, DevState src, const int32_t* __restrict__ index, int N) {
  const int lane = threadIdx.x & 31;
  const int gd = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (gd >= dst.G) return;
  const int gs = index[gd];
  if (gs < 0 || gs >= src.G) return;
  const size_t d = (size_t)gd, s = (size_t)gs;
  const int P = N * N, max_ply = 2 * P;
  {  // history ring: 8 N rows = 4 N 16-byte words
    const uint4* a = reinterpret_cast<const uint4*>(src.ring + s * 8 * N);
    uint4* b = reinterpret_cast<uint4*>(dst.ring + d * 8 * N);
    for (int i = lane; i < 4 * N; i += 32) b[i] = __ldg(a + i);
  }
  const int nsk = min(max(__ldg(src.sk_n + s), 0), max_ply);
  {  // superko record: the pairs of sk[0 .. nsk), then an odd last entry
    const uint64_t* a = src.sk + s * max_ply;
    uint64_t* b = dst.sk + d * max_ply;
    for (int i = lane; i < nsk / 2; i += 32) reinterpret_cast<uint4*>(b)[i] = __ldg(reinterpret_cast<const uint4*>(a) + i);
    if ((nsk & 1) && lane == 0) b[nsk - 1] = __ldg(a + nsk - 1);
  }
  for (int i = lane; i < N; i += 32) {  // rows: position, group status, legal moves
    dst.cur[d * N + i] = __ldg(src.cur + s * N + i);
    dst.sa[d * N + i] = __ldg(src.sa + s * N + i);
    dst.legal[d * N + i] = __ldg(src.legal + s * N + i);
  }
  for (int i = lane; i < P; i += 32) dst.placed[d * P + i] = __ldg(src.placed + s * P + i);
  if (lane == 0) {
    dst.hash[d] = __ldg(src.hash + s);
    dst.sk_n[d] = nsk;
  } else if (lane == 1) {
    store_meta(&dst.meta[d], load_meta(&src.meta[s]));
  }
}

// ---------------------------------------------------------------------------------------
// Monte-Carlo ownership: K random-policy playouts from every stored position (elfb200_ownership).  Playout
// j = g*K + k starts from game g's stored position and plays k_playout's random_ply with draw id j (candidate
// pp_pick(seed, j, ply, n) of the legal non-eye moves of the side to move, a pass when there is none) until
// GoState::terminated() or max_plies moves.  Its superko test covers game g's record and its own new pre-move
// hashes, as GoState::forward on a copy of the game would.  A game that ended by two passes is played on with
// an empty last-move window; one that ended by superko or the ply cap plays no move.  The stored games are
// only read.
//
// counts[g][0][a] / counts[g][1][a] (a = x*N+y, zeroed by the host) count the playouts of game g whose final
// position has point a in black's / white's area in simple_tt_scoring's view: stones, plus empties reachable
// from them through empties only (the empties reachable from both colours count for neither).  Integer
// atomics: the sums do not depend on the order in which playouts finish.
//
// k_playout's row-per-lane layout, ply (random_ply) and stream mode, with a bounded scratch: a fixed grid of
// resident warps whose game segments stride over the G*K playouts (segment s plays j = s, s + S, s + 2S, ...;
// S = segments in the grid).
// A segment owns scratch[s][0 .. 2N^2), its superko record: a playout starts by copying game g's record
// sk[g][0 .. sk_n) there and into the segment's Bloom filter, then appends its own pre-move hashes.
template <int N>
__global__ void __launch_bounds__(PLAYOUT_WARPS * 32)
    k_ownership(DevState st, int K, uint64_t seed, int max_plies, uint64_t* __restrict__ scratch,
                int32_t* __restrict__ counts, uint64_t* __restrict__ out_hash, int32_t* __restrict__ out_plies) {
  constexpr int P = Geo<N>::P, MAXP = Geo<N>::MAX_PLY;
  __shared__ uint64_t s_zob[Geo<N>::ZOB];
  __shared__ uint32_t s_bloom[PLAYOUT_WARPS][Geo<N>::GPW][128];
  load_zobrist<N>(s_zob);
  const Lane L = make_lane<N>();
  const int64_t total = (int64_t)st.G * K;
  const int64_t nseg = (int64_t)gridDim.x * PLAYOUT_WARPS * Geo<N>::GPW;
  const int seg = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * Geo<N>::GPW + L.sub;
  uint64_t* skg = scratch + (size_t)seg * MAXP;
  uint32_t* bloom = s_bloom[threadIdx.x >> 5][L.sub];

  int64_t j = L.active ? seg : total;  // this segment's playout
  uint32_t b = 0, w = 0, safe = 0, atari = 0;
  BoardMeta meta = initial_meta();
  uint64_t hash = 0;
  int nsk = 0, t = 0;
  bool have = false, load = j < total;

  while (true) {
    if (__any_sync(FULL, load)) {  // segments whose playout finished start their next one
      if (load) bloom_clear<N>(bloom, L);
      __syncwarp();
      if (load) {
        const int g = (int)(j / K);
        load_row<N>(st.cur, g, L.row, true, b, w);
        load_row<N>(st.sa, g, L.row, true, safe, atari);
        meta = load_meta(&st.meta[g]);
        hash = st.hash[g];
        nsk = st.sk_n[g];
        if (meta.last1 == MV_PASS && meta.last2 == MV_PASS) meta.last1 = meta.last2 = MV_INVALID;
        const uint64_t* src = st.sk + (size_t)g * MAXP;
        for (int i = L.row; i < nsk; i += N) {
          const uint64_t h = src[i];
          skg[i] = h;
          bloom_insert(bloom, h, true);
        }
        t = 0;
        have = true;
        load = false;
      }
      __syncwarp();
    }
    const bool over = have && (is_terminated<N>(meta) || t >= max_plies);
    if (__any_sync(FULL, over)) {  // area of the final positions (tt_score's fill, a warp collective)
      const uint32_t e = ~(b | w) & L.rm;
      uint32_t ar[2] = {b, w};
      const uint32_t thr[2] = {e, e};
      floodK<N, 2>(ar, thr, L);
      if (over) {
        int32_t* cg = counts + (size_t)(j / K) * 2 * P;
        uint32_t ab = ar[0] & ~ar[1], aw = ar[1] & ~ar[0];
        while (ab) {
          const int x = __ffs(ab) - 1;
          ab &= ab - 1;
          atomicAdd(cg + x * N + L.row, 1);
        }
        while (aw) {
          const int x = __ffs(aw) - 1;
          aw &= aw - 1;
          atomicAdd(cg + P + x * N + L.row, 1);
        }
        if (L.row == 0) {
          if (out_hash) out_hash[j] = hash;
          if (out_plies) out_plies[j] = t;
        }
        j += nseg;
        have = false;
        load = j < total;
      }
      continue;
    }
    if (__all_sync(FULL, !have)) break;
    const bool term = !have;
    random_ply<N>(seed, (uint64_t)j, term, b, w, safe, atari, meta, hash, nullptr, skg, nsk, bloom, s_zob, L);
    if (!term) t++;
  }
}

// ---------------------------------------------------------------------------------------
// Dead groups and getTrompTaylorScore (board.cc:1954-2071) of every stored position (elfb200_final_status).
// One warp per game (row per lane, make_lane_single), groups found one at a time by link-masked fills.
//
// Dead rule (ours, not the reference's: it leaves the choice of dead groups to its caller): with the ownership
// counts of K playouts, a group S of colour c is dead iff
//   own(S) = sum over p in S of (c == black ? counts_b[p] - counts_w[p] : counts_w[p] - counts_b[p])
//   satisfies  (double)own(S) < -threshold * K * |S|.
// Without counts no group is dead.  Dead groups are counted for the opponent (S_DEAD in group_stats): every
// stone takes its (flipped) colour, an empty region the one colour among the stones it touches, else 3 (dame;
// also every point of the empty board).  score = black points - white points.
template <int N>
__global__ void __launch_bounds__(32)
    k_final_status(DevState st, const int32_t* __restrict__ counts, int K, double threshold,
                   uint8_t* __restrict__ dead_out, uint8_t* __restrict__ terr_out, int32_t* __restrict__ score_out) {
  constexpr int P = Geo<N>::P;
  const Lane L = make_lane_single<N>();
  const int g = blockIdx.x;
  uint32_t b, w;
  load_row<N>(st.cur, g, L.row, L.active, b, w);
  uint32_t dead = 0;
  if (counts) {
    const int32_t* cb = counts + (size_t)g * 2 * P;
    const int32_t* cw = cb + P;
    const Links lk = make_links<N>(b, w, L);
    uint32_t left = b | w;
    while (true) {
      const unsigned lanes = __ballot_sync(FULL, left != 0u);
      if (!lanes) break;
      const int src = __ffs(lanes) - 1;  // seed: the lowest stone of the first row that has one left
      const uint32_t seed_bit = __shfl_sync(FULL, left & (0u - left), src);
      const bool black = __shfl_sync(FULL, (seed_bit & b) ? 1 : 0, src) != 0;
      uint32_t grp = L.lane == src ? seed_bit : 0u;
      while (true) {
        const uint32_t n2 = grow_link(grow_link(grp, lk), lk);
        const bool ch = n2 != grp;
        grp = n2;
        if (!__any_sync(FULL, ch)) break;
      }
      long long own = 0;
      for (uint32_t m = grp; m; m &= m - 1) {
        const int a = (__ffs(m) - 1) * N + L.row;
        own += black ? (long long)cb[a] - cw[a] : (long long)cw[a] - cb[a];
      }
      for (int o = 16; o; o >>= 1) own += __shfl_xor_sync(FULL, own, o);
      const int size = game_sum<N>(__popc(grp), L);
      if ((double)own < -threshold * (double)K * (double)size) dead |= grp;
      left &= ~grp;
    }
  }
  const uint32_t bf = (b & ~dead) | (w & dead), wf = (w & ~dead) | (b & dead);
  const uint32_t e = ~(bf | wf) & L.rm;
  uint32_t ar[2] = {bf, wf};
  const uint32_t thr[2] = {e, e};
  floodK<N, 2>(ar, thr, L);
  const uint32_t tb = ar[0] & ~ar[1], tw = ar[1] & ~ar[0];
  const int score = game_sum<N>(__popc(tb) - __popc(tw), L);
  if (L.active) {
    for (int x = 0; x < N; ++x) {
      const size_t a = (size_t)g * P + x * N + L.row;
      if (dead_out) dead_out[a] = (uint8_t)((dead >> x) & 1u);
      if (terr_out) terr_out[a] = (uint8_t)(((tb >> x) & 1u) ? S_BLACK : ((tw >> x) & 1u) ? S_WHITE : 3);
    }
  }
  if (L.lane == 0 && score_out) score_out[g] = score;
}

}  // namespace elfb200

// =========================================================================================
// C ABI
// =========================================================================================
using namespace elfb200;

static thread_local std::string g_err;

int elfb200_fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

static inline int grid_for(const elfb200_ctx* c) {
  int gpw = 32 / c->N;
  int warps = (c->G + gpw - 1) / gpw;
  return (warps + WARPS - 1) / WARPS;
}

extern "C" {

const char* elfb200_last_error(void) { return g_err.c_str(); }
const char* elfb200_version(void) { return "elfb200 0.1 (sm_90a)"; }

int elfb200_create(int board_size, int num_games, int device, elfb200_ctx** out) {
  if (!out) return elfb200_fail(ELFB200_ERR_ARG, "out is NULL");
  *out = nullptr;
  if (board_size != 9 && board_size != 19)
    return elfb200_fail(ELFB200_ERR_ARG, "board_size must be 9 or 19 (got %d)", board_size);
  if (num_games <= 0) return elfb200_fail(ELFB200_ERR_ARG, "num_games must be positive");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return elfb200_fail(ELFB200_ERR_CUDA, "no CUDA device available (%s); elfb200 has no CPU fallback",
                cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return elfb200_fail(ELFB200_ERR_ARG, "bad device %d", device);
  CK(cudaSetDevice(device));
  elfb200_ctx* c = new elfb200_ctx();
  c->N = board_size;
  c->G = num_games;
  c->device = device;
  // any failure below releases what was allocated so far (elfb200_destroy tolerates a partly built context)
  auto build = [&]() -> int {
  const size_t N = board_size, G = num_games, P = N * N, MAXPLY = 2 * P;
  CK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
#if !defined(ELFB200_SIMT_EMU)  // the emulator build orders nothing (stream_after)
  for (cudaEvent_t& e : c->ev_gather) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
#endif
  CK(cudaMalloc(&c->st.cur, G * N * 8));
  CK(cudaMalloc(&c->st.ring, G * 8 * N * 8));
  CK(cudaMalloc(&c->st.legal, G * N * 4));
  CK(cudaMalloc(&c->st.hash, G * 8));
  CK(cudaMalloc(&c->st.meta, G * sizeof(BoardMeta)));
  CK(cudaMalloc(&c->st.sk, G * MAXPLY * 8));
  CK(cudaMalloc(&c->st.sk_n, G * 4));
  CK(cudaMalloc(&c->st.placed, G * P * 2));
  CK(cudaMalloc(&c->st.sa, G * N * 8));
  {
    std::vector<float> tab(MAXPLY + 2);
    for (size_t k = 0; k < tab.size(); ++k) tab[k] = (float)exp(-(double)k / 10.0);  // board_feature.cc:getHistoryExp
    CK(cudaMalloc(&c->d_exp_table, tab.size() * 4));
    CK(cudaMemcpy(c->d_exp_table, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice));
  }
  c->st.G = num_games;
  CK(cudaMalloc(&c->d_actions, G * 4));
  CK(cudaMalloc(&c->d_ok, G));
  CK(cudaMalloc(&c->d_bytes, G * (P + 1)));
  CK(cudaMalloc(&c->d_words, G * ELFB200_INFO_FIELDS * 4));
  CK(cudaMalloc(&c->d_d4, G * 4));
  CK(cudaMalloc(&c->d_po_sk, G * MAXPLY * 8));
  CK(cudaMalloc(&c->d_po_chk, G * 8));
  CK(cudaMalloc(&c->d_po_hash, G * 8));
  CK(cudaMalloc(&c->d_po_plies, G * 4));
  CK(cudaMalloc(&c->d_po_score, G * 4));
  c->h_pin_bytes = G * (P + 1) > G * 64 ? G * (P + 1) : G * 64;
  CK(cudaMallocHost(&c->h_pin, c->h_pin_bytes));
  // mapped window: actions int32[G] | accept flags uint8[G] (16-byte aligned) | completion flag (16-byte aligned)
  c->map_ok_off = (G * 4 + 15) & ~(size_t)15;
  c->map_flag_off = (c->map_ok_off + G + 15) & ~(size_t)15;
  CK(cudaHostAlloc(&c->h_map, c->map_flag_off + 16, cudaHostAllocMapped));
  memset(c->h_map, 0, c->map_flag_off + 16);
  CK(cudaMalloc(&c->d_done, 4));
  CK(cudaMemset(c->d_done, 0, 4));
  CK(cudaHostGetDevicePointer(&c->d_map_actions, c->h_map, 0));
  c->d_map_ok = reinterpret_cast<uint8_t*>(c->d_map_actions) + c->map_ok_off;
  return elfb200_reset(c, nullptr);
  };
  const int rc = build();
  if (rc) {
    const std::string why = g_err;  // elfb200_destroy must not lose the message
    elfb200_destroy(c);
    g_err = why;
    return rc;
  }
  *out = c;
  return ELFB200_OK;
}

void elfb200_destroy(elfb200_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  void* ptrs[] = {c->st.cur,  c->st.ring, c->st.legal, c->st.hash,   c->st.meta,   c->st.sk,
                  c->st.sk_n, c->d_actions, c->d_ok,   c->d_bytes,   c->d_words,   c->d_d4,
                  c->d_feat,  c->d_po_sk, c->d_po_chk, c->d_po_hash, c->d_po_plies, c->d_po_score,
                  c->d_replay, c->st.placed, c->st.sa, c->d_exp_table, c->d_done,
                  c->d_own_sk, c->d_own_counts, c->d_own_status, c->d_own_hash, c->d_own_plies};
  for (void* p : ptrs)
    if (p) cudaFree(p);
  if (c->h_pin) cudaFreeHost(c->h_pin);
  if (c->h_map) cudaFreeHost(c->h_map);
  for (cudaEvent_t e : c->ev_gather)
    if (e) cudaEventDestroy(e);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
}

int elfb200_num_games(const elfb200_ctx* c) { return c ? c->G : 0; }
int elfb200_board_size(const elfb200_ctx* c) { return c ? c->N : 0; }
void* elfb200_stream(const elfb200_ctx* c) { return c ? (void*)c->stream : nullptr; }
int64_t elfb200_launch_count(const elfb200_ctx* c) { return c ? c->launches : 0; }

int elfb200_synchronize(elfb200_ctx* c) {
  if (!c) return elfb200_fail(ELFB200_ERR_ARG, "ctx is NULL");
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_reset(elfb200_ctx* c, const uint8_t* mask_host) {
  if (!c) return elfb200_fail(ELFB200_ERR_ARG, "ctx is NULL");
  CK(cudaSetDevice(c->device));
  const uint8_t* dmask = nullptr;
  if (mask_host) {
    memcpy(c->h_pin, mask_host, c->G);
    CK(cudaMemcpyAsync(c->d_ok, c->h_pin, c->G, cudaMemcpyHostToDevice, c->stream));
    dmask = c->d_ok;
  }
  DISPATCH_N(c, (k_reset<19><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, dmask)),
             (k_reset<9><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, dmask)));
  c->launches++;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_step_dev(elfb200_ctx* c, const int32_t* actions_dev, uint8_t* ok_dev) {
  if (!c || !actions_dev) return elfb200_fail(ELFB200_ERR_ARG, "ctx/actions is NULL");
  CK(cudaSetDevice(c->device));
  DISPATCH_N(c, (k_step<19><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, actions_dev, ok_dev, nullptr, nullptr, 0u, nullptr)),
             (k_step<9><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, actions_dev, ok_dev, nullptr, nullptr, 0u, nullptr)));
  c->launches++;
  CK(cudaGetLastError());
  return ELFB200_OK;
}

int elfb200_env_step(elfb200_ctx* c, const int32_t* actions_dev, float komi, uint8_t* ok_dev, uint8_t* done_dev,
                     float* value_dev, uint8_t* legal_dev, int32_t* info_dev) {
  if (!c || !actions_dev) return elfb200_fail(ELFB200_ERR_ARG, "ctx/actions is NULL");
  CK(cudaSetDevice(c->device));
  DISPATCH_N(c,
             (k_env_step<19><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, actions_dev, komi, ok_dev, done_dev, value_dev,
                                                                   legal_dev, info_dev)),
             (k_env_step<9><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, actions_dev, komi, ok_dev, done_dev, value_dev,
                                                                  legal_dev, info_dev)));
  c->launches++;
  CK(cudaGetLastError());
  return ELFB200_OK;
}

int elfb200_reset_dev(elfb200_ctx* c, const uint8_t* mask_dev) {
  if (!c) return elfb200_fail(ELFB200_ERR_ARG, "ctx is NULL");
  CK(cudaSetDevice(c->device));
  DISPATCH_N(c, (k_reset<19><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, mask_dev)),
             (k_reset<9><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, mask_dev)));
  c->launches++;
  CK(cudaGetLastError());
  return ELFB200_OK;
}

int elfb200_step(elfb200_ctx* c, const int32_t* actions_host, uint8_t* ok_host) {
  if (!c || !actions_host) return elfb200_fail(ELFB200_ERR_ARG, "ctx/actions is NULL");
  CK(cudaSetDevice(c->device));
  // host buffers, one small DMA and no stream synchronisation: the actions go through the pinned window and
  // the copy engine (SMs reading 4-byte actions over PCIe one warp at a time measured 14 us slower), k_step
  // writes the accept flags straight into the mapped window (posted PCIe writes), the last CTA raises the
  // completion flag there and the host spins on it
  uint8_t* win = reinterpret_cast<uint8_t*>(c->h_map);
  volatile uint32_t* flag = reinterpret_cast<volatile uint32_t*>(win + c->map_flag_off);
  volatile uint32_t* dflag = reinterpret_cast<volatile uint32_t*>(reinterpret_cast<uint8_t*>(c->d_map_actions) + c->map_flag_off);
  memcpy(win, actions_host, (size_t)c->G * 4);
  CK(cudaMemcpyAsync(c->d_actions, win, (size_t)c->G * 4, cudaMemcpyHostToDevice, c->stream));
  const uint32_t seq = ++c->step_seq;
  DISPATCH_N(c, (k_step<19><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, c->d_actions, c->d_ok, c->d_done, dflag, seq, c->d_map_ok)),
             (k_step<9><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, c->d_actions, c->d_ok, c->d_done, dflag, seq, c->d_map_ok)));
  c->launches++;
  CK(cudaGetLastError());
#if defined(ELFB200_SIMT_EMU)
  CK(cudaStreamSynchronize(c->stream));
#else
  {
    // ~20 ms of spinning covers any healthy launch; afterwards (or on a failed launch) fall back to the runtime
    bool done = false;
    for (long spin = 0; spin < 20000000L; ++spin) {
      if (*flag == seq) {
        done = true;
        break;
      }
      if ((spin & 1023) == 1023 && cudaStreamQuery(c->stream) != cudaErrorNotReady) break;
    }
    if (!done) CK(cudaStreamSynchronize(c->stream));
  }
#endif
  if (ok_host) memcpy(ok_host, win + c->map_ok_off, c->G);
  return ELFB200_OK;
}

// per-game action lists for k_replay / k_place: lists[G][stride] into d_replay (grown on demand), counts into d_actions
static int upload_lists(elfb200_ctx* c, const int16_t* lists_host, int stride, const int32_t* count_host) {
  const size_t bytes = (size_t)c->G * (size_t)stride * sizeof(int16_t);
  if (bytes > c->d_replay_bytes) {
    if (c->d_replay) CK(cudaFree(c->d_replay));
    c->d_replay = nullptr;
    c->d_replay_bytes = 0;
    CK(cudaMalloc(&c->d_replay, bytes));
    c->d_replay_bytes = bytes;
  }
  memcpy(c->h_pin, count_host, (size_t)c->G * 4);
  CK(cudaMemcpyAsync(c->d_actions, c->h_pin, (size_t)c->G * 4, cudaMemcpyHostToDevice, c->stream));
  CK(cudaMemcpyAsync(c->d_replay, lists_host, bytes, cudaMemcpyHostToDevice, c->stream));
  return ELFB200_OK;
}

int elfb200_replay(elfb200_ctx* c, const int16_t* moves_host, int stride, const int32_t* count_host) {
  if (!c || !moves_host || !count_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  const int max_ply = c->N == 19 ? elfb200::Geo<19>::MAX_PLY : elfb200::Geo<9>::MAX_PLY;
  if (stride <= 0 || stride > max_ply)
    return elfb200_fail(ELFB200_ERR_ARG, "stride %d outside [1, %d]", stride, max_ply);
  for (int g = 0; g < c->G; ++g)
    if (count_host[g] < 0 || count_host[g] > stride)
      return elfb200_fail(ELFB200_ERR_ARG, "count[%d] = %d outside [0, stride = %d]", g, count_host[g], stride);
  CK(cudaSetDevice(c->device));
  const int rc = upload_lists(c, moves_host, stride, count_host);
  if (rc) return rc;
  DISPATCH_N(c, (k_replay<19><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, c->d_replay, stride, c->d_actions)),
             (k_replay<9><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, c->d_replay, stride, c->d_actions)));
  c->launches++;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_place_handicap(elfb200_ctx* c, const int16_t* stones_host, int stride, const int32_t* count_host,
                           uint8_t* ok_host) {
  if (!c || !stones_host || !count_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  const int P = c->N * c->N;
  if (stride <= 0 || stride > P) return elfb200_fail(ELFB200_ERR_ARG, "stride %d outside [1, %d]", stride, P);
  for (int g = 0; g < c->G; ++g) {
    if (count_host[g] < 0 || count_host[g] > stride)
      return elfb200_fail(ELFB200_ERR_ARG, "count[%d] = %d outside [0, stride = %d]", g, count_host[g], stride);
    for (int t = 0; t < count_host[g]; ++t) {
      const int a = stones_host[(size_t)g * stride + t];
      if (a < 0 || a >= P)
        return elfb200_fail(ELFB200_ERR_ARG, "stone %d of game %d: action %d outside [0, %d)", t, g, a, P);
    }
  }
  CK(cudaSetDevice(c->device));
  const int rc = upload_lists(c, stones_host, stride, count_host);
  if (rc) return rc;
  uint8_t* dok = nullptr;
  if (ok_host) {  // G * stride <= G * (N*N + 1) bytes
    dok = c->d_bytes;
    CK(cudaMemsetAsync(dok, 0, (size_t)c->G * stride, c->stream));
  }
  DISPATCH_N(c, (k_place<19><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, c->d_replay, stride, c->d_actions, dok)),
             (k_place<9><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, c->d_replay, stride, c->d_actions, dok)));
  c->launches++;
  CK(cudaGetLastError());
  if (ok_host) CK(cudaMemcpyAsync(ok_host, dok, (size_t)c->G * stride, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

static int check_gather(const elfb200_ctx* dst, const elfb200_ctx* src, const int32_t* index) {
  if (!dst || !src || !index) return elfb200_fail(ELFB200_ERR_ARG, "dst/src/index is NULL");
  if (dst == src) return elfb200_fail(ELFB200_ERR_ARG, "dst and src are the same context (an in-place permutation would race)");
  if (dst->N != src->N) return elfb200_fail(ELFB200_ERR_ARG, "board sizes differ (dst %d, src %d)", dst->N, src->N);
  if (dst->device != src->device)
    return elfb200_fail(ELFB200_ERR_ARG, "devices differ (dst %d, src %d)", dst->device, src->device);
  return ELFB200_OK;
}

// `waiter`'s later work runs after the work already on `first` (event `ev`).  The SIMT emulator build runs all
// work in issue order, so there it has nothing to order.
static int stream_after(cudaStream_t waiter, cudaStream_t first, cudaEvent_t ev) {
#if defined(ELFB200_SIMT_EMU)
  (void)waiter, (void)first, (void)ev;
#else
  CK(cudaEventRecord(ev, first));
  CK(cudaStreamWaitEvent(waiter, ev, 0));
#endif
  return ELFB200_OK;
}

// k_gather on dst's stream, after the work already on src's stream (fork); src's later work waits for the
// copy (join), so it cannot change a game while the game is read
static int gather_launch(elfb200_ctx* dst, const elfb200_ctx* src, const int32_t* index_dev) {
  int rc = stream_after(dst->stream, src->stream, dst->ev_gather[0]);
  if (rc) return rc;
  const int grid = (int)(((size_t)dst->G * 32 + GATHER_THREADS - 1) / GATHER_THREADS);
  k_gather<<<grid, GATHER_THREADS, 0, dst->stream>>>(dst->st, src->st, index_dev, dst->N);
  dst->launches++;
  CK(cudaGetLastError());
  return stream_after(src->stream, dst->stream, dst->ev_gather[1]);
}

int elfb200_gather_games_dev(elfb200_ctx* dst, const elfb200_ctx* src, const int32_t* index_dev) {
  int rc = check_gather(dst, src, index_dev);
  if (rc) return rc;
  CK(cudaSetDevice(dst->device));
  return gather_launch(dst, src, index_dev);
}

int elfb200_gather_games(elfb200_ctx* dst, const elfb200_ctx* src, const int32_t* index_host) {
  int rc = check_gather(dst, src, index_host);
  if (rc) return rc;
  CK(cudaSetDevice(dst->device));
  memcpy(dst->h_pin, index_host, (size_t)dst->G * 4);
  CK(cudaMemcpyAsync(dst->d_actions, dst->h_pin, (size_t)dst->G * 4, cudaMemcpyHostToDevice, dst->stream));
  rc = gather_launch(dst, src, dst->d_actions);
  if (rc) return rc;
  CK(cudaStreamSynchronize(dst->stream));
  return ELFB200_OK;
}

int elfb200_get_hash(elfb200_ctx* c, uint64_t* hash_host) {
  if (!c || !hash_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  CK(cudaSetDevice(c->device));
  CK(cudaMemcpyAsync(hash_host, c->st.hash, (size_t)c->G * 8, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

static int run_export(elfb200_ctx* c, uint8_t* legal, uint8_t* stones, uint8_t* eyes, int eye_player,
                      int32_t* info, int32_t* score) {
  DISPATCH_N(c,
             (k_export<19><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, legal, stones, eyes,
                                                                  eye_player, info, score)),
             (k_export<9><<<grid_for(c), BLOCK, 0, c->stream>>>(c->st, legal, stones, eyes,
                                                                 eye_player, info, score)));
  c->launches++;
  CK(cudaGetLastError());
  return ELFB200_OK;
}

// The views k_export writes, one at a time, for the host readers below.
enum ExportView { VIEW_LEGAL, VIEW_STONES, VIEW_EYES, VIEW_INFO, VIEW_SCORE };

// k_export of one view into device scratch (d_bytes for the byte views, d_words for info and score), then the
// whole view to `host`
static int read_export(elfb200_ctx* c, ExportView v, int eye_player, void* host) {
  const size_t G = c->G, P = (size_t)c->N * c->N;
  uint8_t* bytes = c->d_bytes;
  int32_t* words = c->d_words;
  CK(cudaSetDevice(c->device));
  int rc = run_export(c, v == VIEW_LEGAL ? bytes : nullptr, v == VIEW_STONES ? bytes : nullptr,
                      v == VIEW_EYES ? bytes : nullptr, eye_player, v == VIEW_INFO ? words : nullptr,
                      v == VIEW_SCORE ? words : nullptr);
  if (rc) return rc;
  const size_t n = v == VIEW_LEGAL ? G * (P + 1)
                   : v == VIEW_INFO  ? G * ELFB200_INFO_FIELDS * 4
                   : v == VIEW_SCORE ? G * 4
                                     : G * P;
  CK(cudaMemcpyAsync(host, v == VIEW_INFO || v == VIEW_SCORE ? (void*)words : (void*)bytes, n, cudaMemcpyDeviceToHost,
                     c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_get_info(elfb200_ctx* c, int32_t* info_host) {
  if (!c || !info_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  return read_export(c, VIEW_INFO, 0, info_host);
}

int elfb200_observe_dev(elfb200_ctx* c, uint8_t* legal_dev, int32_t* info_dev) {
  if (!c) return elfb200_fail(ELFB200_ERR_ARG, "ctx is NULL");
  CK(cudaSetDevice(c->device));
  return run_export(c, legal_dev, nullptr, nullptr, 0, info_dev, nullptr);
}

int elfb200_get_stones(elfb200_ctx* c, uint8_t* stones_host) {
  if (!c || !stones_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  return read_export(c, VIEW_STONES, 0, stones_host);
}

int elfb200_get_legal(elfb200_ctx* c, uint8_t* legal_host) {
  if (!c || !legal_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  return read_export(c, VIEW_LEGAL, 0, legal_host);
}

int elfb200_get_true_eyes(elfb200_ctx* c, int player, uint8_t* eyes_host) {
  if (!c || !eyes_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  if (player < 0 || player > 2) return elfb200_fail(ELFB200_ERR_ARG, "player must be 0, 1 or 2");
  return read_export(c, VIEW_EYES, player, eyes_host);
}

int elfb200_get_tt_score(elfb200_ctx* c, int32_t* score_host) {
  if (!c || !score_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  return read_export(c, VIEW_SCORE, 0, score_host);
}

int elfb200_evaluate(elfb200_ctx* c, float komi, float* value_host) {
  if (!c || !value_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  CK(cudaSetDevice(c->device));
  // GoState::evaluate (go_state.h:194-203): superko-terminated -> +-1 for the side to move,
  // else tt score - komi.  Scores and flags come from one export launch.
  int rc = run_export(c, nullptr, nullptr, nullptr, 0, c->d_words, (int32_t*)c->d_bytes);
  if (rc) return rc;
  std::string info((size_t)c->G * ELFB200_INFO_FIELDS * 4, '\0'), sc((size_t)c->G * 4, '\0');
  CK(cudaMemcpyAsync(&info[0], c->d_words, info.size(), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaMemcpyAsync(&sc[0], c->d_bytes, sc.size(), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  const int32_t* in = (const int32_t*)info.data();
  const int32_t* s = (const int32_t*)sc.data();
  for (int g = 0; g < c->G; ++g) {
    if (in[g * ELFB200_INFO_FIELDS + 11])
      value_host[g] = in[g * ELFB200_INFO_FIELDS + 1] == S_BLACK ? 1.0f : -1.0f;
    else
      value_host[g] = (float)s[g] - komi;
  }
  return ELFB200_OK;
}

static int check_feature_args(const void* out, int format, int cpad) {
  if (format < FEAT_F32_NCHW || format > FEAT_BF16_NHWC) return elfb200_fail(ELFB200_ERR_ARG, "unknown feature format %d", format);
  const uintptr_t a = (uintptr_t)out;
  if (format == FEAT_F32_NCHW) {
    if (a & 7) return elfb200_fail(ELFB200_ERR_ARG, "feature buffer must be 8-byte aligned");
  } else {
    if (cpad < 24 || cpad > FEAT_CPAD_MAX || (cpad & 7))
      return elfb200_fail(ELFB200_ERR_ARG, "channel padding must be 24 or 32 (got %d)", cpad);
    if (a & 15) return elfb200_fail(ELFB200_ERR_ARG, "16-bit NHWC feature buffer must be 16-byte aligned");
  }
  return ELFB200_OK;
}

int elfb200_features_dev_ex(elfb200_ctx* c, const int32_t* d4_dev, void* out_dev, int format, int cpad) {
  if (!c || !out_dev) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  int rc = check_feature_args(out_dev, format, cpad);
  if (rc) return rc;
  CK(cudaSetDevice(c->device));
  DISPATCH_N(c,
             (k_features<19><<<c->G, FEAT_THREADS, feature_smem_bytes<19>(format, cpad, c->feat_tma), c->stream>>>(
                 c->st, d4_dev, out_dev, format, cpad, c->feat_tma)),
             (k_features<9><<<c->G, FEAT_THREADS, feature_smem_bytes<9>(format, cpad, c->feat_tma), c->stream>>>(
                 c->st, d4_dev, out_dev, format, cpad, c->feat_tma)));
  c->launches++;
  CK(cudaGetLastError());
  return ELFB200_OK;
}

int elfb200_features_dev(elfb200_ctx* c, const int32_t* d4_dev, float* out_dev) {
  return elfb200_features_dev_ex(c, d4_dev, out_dev, FEAT_F32_NCHW, 0);
}

int elfb200_features_df_dev(elfb200_ctx* c, const int32_t* d4_dev, float* out_dev) {
  if (!c || !out_dev) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  CK(cudaSetDevice(c->device));
  DISPATCH_N(c, (k_features_df<19><<<c->G, 32, 0, c->stream>>>(c->st, d4_dev, c->d_exp_table, out_dev)),
             (k_features_df<9><<<c->G, 32, 0, c->stream>>>(c->st, d4_dev, c->d_exp_table, out_dev)));
  c->launches++;
  CK(cudaGetLastError());
  return ELFB200_OK;
}

int elfb200_features_df(elfb200_ctx* c, const int32_t* d4_host, float* out_host) {
  if (!c || !out_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  CK(cudaSetDevice(c->device));
  const size_t bytes = (size_t)c->G * 25 * c->N * c->N * 4;
  float* d_out = nullptr;
  CK(cudaMalloc(&d_out, bytes));
  const int32_t* d4 = nullptr;
  if (d4_host) {
    memcpy(c->h_pin, d4_host, (size_t)c->G * 4);
    if (cudaMemcpyAsync(c->d_d4, c->h_pin, (size_t)c->G * 4, cudaMemcpyHostToDevice, c->stream) != cudaSuccess) {
      cudaFree(d_out);
      return elfb200_fail(ELFB200_ERR_CUDA, "copy of the D4 codes failed");
    }
    d4 = c->d_d4;
  }
  int rc = elfb200_features_df_dev(c, d4, d_out);
  if (!rc && (cudaMemcpyAsync(out_host, d_out, bytes, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
              cudaStreamSynchronize(c->stream) != cudaSuccess))
    rc = elfb200_fail(ELFB200_ERR_CUDA, "DarkForest feature read-back failed");
  cudaFree(d_out);
  return rc;
}

int elfb200_set_playout_layout(elfb200_ctx* c, int layout) {
  if (!c || layout < -1 || layout > 1) return elfb200_fail(ELFB200_ERR_ARG, "layout must be -1 (automatic), 0 (row per lane) or 1 (two rows per lane)");
  if (layout == 1 && c->N != 19) return elfb200_fail(ELFB200_ERR_ARG, "the two-rows-per-lane layout is 19x19 only");
  c->playout_layout = layout;
  return ELFB200_OK;
}

int elfb200_set_feature_store(elfb200_ctx* c, int mode) {
  if (!c || mode < 0 || mode > 1) return elfb200_fail(ELFB200_ERR_ARG, "mode must be 0 (vector stores) or 1 (bulk store)");
  c->feat_tma = mode;
  return ELFB200_OK;
}

int elfb200_features(elfb200_ctx* c, const int32_t* d4_host, float* out_host) {
  if (!c || !out_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  CK(cudaSetDevice(c->device));
  const size_t bytes = (size_t)c->G * 18 * c->N * c->N * 4;
  if (!c->d_feat) CK(cudaMalloc(&c->d_feat, bytes));
  const int32_t* d4 = nullptr;
  if (d4_host) {
    memcpy(c->h_pin, d4_host, (size_t)c->G * 4);
    CK(cudaMemcpyAsync(c->d_d4, c->h_pin, (size_t)c->G * 4, cudaMemcpyHostToDevice, c->stream));
    d4 = c->d_d4;
  }
  int rc = elfb200_features_dev(c, d4, c->d_feat);
  if (rc) return rc;
  CK(cudaMemcpyAsync(out_host, c->d_feat, bytes, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

static int playout_launch(elfb200_ctx* c, uint64_t seed, uint64_t first_game_id, int max_plies, int stream_plies) {
  if (!c) return elfb200_fail(ELFB200_ERR_ARG, "ctx is NULL");
  if (max_plies <= 0) return elfb200_fail(ELFB200_ERR_ARG, "max_plies must be positive");
  if (stream_plies < 0) return elfb200_fail(ELFB200_ERR_ARG, "plies_per_slot must be positive");
  CK(cudaSetDevice(c->device));
  const int layout = c->playout_layout >= 0 ? c->playout_layout : ((c->N == 19 && c->G >= 4096) ? 1 : 0);
  const bool two_rows = c->N == 19 && layout == 1;
  const int gpw = two_rows ? Geo2<19>::GPW : 32 / c->N;
  const int pgrid = ((c->G + gpw - 1) / gpw + PLAYOUT_WARPS - 1) / PLAYOUT_WARPS;
  if (two_rows)
    k_playout2<19><<<pgrid, PLAYOUT_WARPS * 32, 0, c->stream>>>(c->G, seed, first_game_id, max_plies, stream_plies,
                                                               c->d_po_sk, c->d_po_chk, c->d_po_plies, c->d_po_score,
                                                               c->d_po_hash);
  else
    DISPATCH_N(c,
               (k_playout<19><<<pgrid, PLAYOUT_WARPS * 32, 0, c->stream>>>(
                   c->G, seed, first_game_id, max_plies, stream_plies, c->d_po_sk, c->d_po_chk, c->d_po_plies,
                   c->d_po_score, c->d_po_hash)),
               (k_playout<9><<<pgrid, PLAYOUT_WARPS * 32, 0, c->stream>>>(
                   c->G, seed, first_game_id, max_plies, stream_plies, c->d_po_sk, c->d_po_chk, c->d_po_plies,
                   c->d_po_score, c->d_po_hash)));
  c->launches++;
  CK(cudaGetLastError());
  return ELFB200_OK;
}

int elfb200_playout_launch(elfb200_ctx* c, uint64_t seed, uint64_t first_game_id, int max_plies) {
  return playout_launch(c, seed, first_game_id, max_plies, 0);
}

int elfb200_playout_stream_launch(elfb200_ctx* c, uint64_t seed, uint64_t first_game_id, int plies_per_slot) {
  if (plies_per_slot <= 0) return elfb200_fail(ELFB200_ERR_ARG, "plies_per_slot must be positive");
  return playout_launch(c, seed, first_game_id, c ? 2 * c->N * c->N : 1, plies_per_slot);
}

int elfb200_playout_stream(elfb200_ctx* c, uint64_t seed, uint64_t first_game_id, int plies_per_slot,
                           uint64_t* chk_host, int32_t* plies_host, int32_t* games_host,
                           uint64_t* last_hash_host, int64_t* total_plies) {
  int rc = elfb200_playout_stream_launch(c, seed, first_game_id, plies_per_slot);
  if (rc) return rc;
  return elfb200_playout_results(c, chk_host, plies_host, games_host, last_hash_host, total_plies);
}

int elfb200_playout_results(elfb200_ctx* c, uint64_t* chk_host, int32_t* plies_host,
                            int32_t* score_host, uint64_t* final_hash_host, int64_t* total_plies) {
  if (!c) return elfb200_fail(ELFB200_ERR_ARG, "ctx is NULL");
  CK(cudaSetDevice(c->device));
  const size_t G = c->G;
  // plies are always fetched (into pinned staging) to form the total
  int32_t* hp = (int32_t*)c->h_pin;
  CK(cudaMemcpyAsync(hp, c->d_po_plies, G * 4, cudaMemcpyDeviceToHost, c->stream));
  if (chk_host) CK(cudaMemcpyAsync(chk_host, c->d_po_chk, G * 8, cudaMemcpyDeviceToHost, c->stream));
  if (score_host)
    CK(cudaMemcpyAsync(score_host, c->d_po_score, G * 4, cudaMemcpyDeviceToHost, c->stream));
  if (final_hash_host)
    CK(cudaMemcpyAsync(final_hash_host, c->d_po_hash, G * 8, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  int64_t tot = 0;
  for (size_t g = 0; g < G; ++g) tot += hp[g];
  if (plies_host) memcpy(plies_host, hp, G * 4);
  if (total_plies) *total_plies = tot;
  return ELFB200_OK;
}

int elfb200_playout(elfb200_ctx* c, uint64_t seed, uint64_t first_game_id, int max_plies,
                    uint64_t* chk_host, int32_t* plies_host, int32_t* score_host,
                    uint64_t* final_hash_host, int64_t* total_plies) {
  int rc = elfb200_playout_launch(c, seed, first_game_id, max_plies);
  if (rc) return rc;
  return elfb200_playout_results(c, chk_host, plies_host, score_host, final_hash_host, total_plies);
}

}  // extern "C"

// ---- Monte-Carlo ownership and final status ------------------------------------------------------------------
static int check_ownership(const elfb200_ctx* c, int playouts, int max_plies, const void* counts) {
  if (!c) return elfb200_fail(ELFB200_ERR_ARG, "ctx is NULL");
  if (!counts) return elfb200_fail(ELFB200_ERR_ARG, "counts is NULL");
  if (playouts < 1) return elfb200_fail(ELFB200_ERR_ARG, "playouts must be at least 1 (got %d)", playouts);
  if ((int64_t)c->G * playouts > INT32_MAX)
    return elfb200_fail(ELFB200_ERR_ARG, "%d games x %d playouts exceed INT32_MAX", c->G, playouts);
  if (max_plies < 0) return elfb200_fail(ELFB200_ERR_ARG, "max_plies must not be negative (got %d)", max_plies);
  return ELFB200_OK;
}

// k_ownership on the context stream: counts zeroed, then a grid of at most the warps the device holds at once,
// each segment with a superko scratch of 2N^2 words (allocated on first use, grown with the grid).
template <int N>
static int ownership_launch(elfb200_ctx* c, int K, uint64_t seed, int max_plies, int32_t* counts, uint64_t* hash,
                            int32_t* plies) {
  constexpr int GPW = Geo<N>::GPW;
  const int64_t total = (int64_t)c->G * K;
  int64_t warps = (total + GPW - 1) / GPW;
#if defined(ELFB200_SIMT_EMU)
  const int64_t resident = 2;  // few warps, each striding over many playouts
#else
  int sms = 0, per_sm = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device));
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_ownership<N>, PLAYOUT_WARPS * 32, 0));
  const int64_t resident = (int64_t)sms * (per_sm > 0 ? per_sm : 1) * PLAYOUT_WARPS;
#endif
  if (warps > resident) warps = resident;
  const int grid = (int)((warps + PLAYOUT_WARPS - 1) / PLAYOUT_WARPS);
  const size_t sk_bytes = (size_t)grid * PLAYOUT_WARPS * GPW * Geo<N>::MAX_PLY * sizeof(uint64_t);
  if (sk_bytes > c->d_own_sk_bytes) {
    if (c->d_own_sk) CK(cudaFree(c->d_own_sk));
    c->d_own_sk = nullptr;
    c->d_own_sk_bytes = 0;
    CK(cudaMalloc(&c->d_own_sk, sk_bytes));
    c->d_own_sk_bytes = sk_bytes;
  }
  CK(cudaMemsetAsync(counts, 0, (size_t)c->G * 2 * Geo<N>::P * sizeof(int32_t), c->stream));
  k_ownership<N><<<grid, PLAYOUT_WARPS * 32, 0, c->stream>>>(c->st, K, seed, max_plies, c->d_own_sk, counts, hash,
                                                             plies);
  c->launches++;
  CK(cudaGetLastError());
  return ELFB200_OK;
}

extern "C" {

int elfb200_ownership_dev(elfb200_ctx* c, int playouts, uint64_t seed, int max_plies, int32_t* counts_dev) {
  int rc = check_ownership(c, playouts, max_plies, counts_dev);
  if (rc) return rc;
  CK(cudaSetDevice(c->device));
  DISPATCH_N(c, (rc = ownership_launch<19>(c, playouts, seed, max_plies, counts_dev, nullptr, nullptr)),
             (rc = ownership_launch<9>(c, playouts, seed, max_plies, counts_dev, nullptr, nullptr)));
  return rc;
}

int elfb200_ownership(elfb200_ctx* c, int playouts, uint64_t seed, int max_plies, int32_t* counts_host,
                      uint64_t* final_hash_host, int32_t* plies_host) {
  int rc = check_ownership(c, playouts, max_plies, counts_host);
  if (rc) return rc;
  CK(cudaSetDevice(c->device));
  const size_t P = (size_t)c->N * c->N, total = (size_t)c->G * playouts;
  if (!c->d_own_counts) CK(cudaMalloc(&c->d_own_counts, (size_t)c->G * 2 * P * sizeof(int32_t)));
  const bool trace = final_hash_host || plies_host;
  if (trace && total > c->d_own_trace) {
    if (c->d_own_hash) CK(cudaFree(c->d_own_hash));
    if (c->d_own_plies) CK(cudaFree(c->d_own_plies));
    c->d_own_hash = nullptr;
    c->d_own_plies = nullptr;
    c->d_own_trace = 0;
    CK(cudaMalloc(&c->d_own_hash, total * sizeof(uint64_t)));
    CK(cudaMalloc(&c->d_own_plies, total * sizeof(int32_t)));
    c->d_own_trace = total;
  }
  uint64_t* dh = final_hash_host ? c->d_own_hash : nullptr;
  int32_t* dp = plies_host ? c->d_own_plies : nullptr;
  DISPATCH_N(c, (rc = ownership_launch<19>(c, playouts, seed, max_plies, c->d_own_counts, dh, dp)),
             (rc = ownership_launch<9>(c, playouts, seed, max_plies, c->d_own_counts, dh, dp)));
  if (rc) return rc;
  CK(cudaMemcpyAsync(counts_host, c->d_own_counts, (size_t)c->G * 2 * P * sizeof(int32_t), cudaMemcpyDeviceToHost,
                     c->stream));
  if (dh) CK(cudaMemcpyAsync(final_hash_host, dh, total * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
  if (dp) CK(cudaMemcpyAsync(plies_host, dp, total * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_final_status(elfb200_ctx* c, const int32_t* counts_host, int playouts, double threshold,
                         uint8_t* dead_host, uint8_t* territory_host, int32_t* score_host) {
  if (!c) return elfb200_fail(ELFB200_ERR_ARG, "ctx is NULL");
  if (counts_host && playouts < 1)
    return elfb200_fail(ELFB200_ERR_ARG, "playouts must be at least 1 (got %d)", playouts);
  if (counts_host && (int64_t)c->G * playouts > INT32_MAX)
    return elfb200_fail(ELFB200_ERR_ARG, "%d games x %d playouts exceed INT32_MAX", c->G, playouts);
  if (!std::isfinite(threshold)) return elfb200_fail(ELFB200_ERR_ARG, "threshold must be finite");
  CK(cudaSetDevice(c->device));
  const size_t P = (size_t)c->N * c->N, G = c->G;
  if (!c->d_own_status) CK(cudaMalloc(&c->d_own_status, G * 2 * P));
  const int32_t* dcounts = nullptr;
  if (counts_host) {
    if (!c->d_own_counts) CK(cudaMalloc(&c->d_own_counts, G * 2 * P * sizeof(int32_t)));
    CK(cudaMemcpyAsync(c->d_own_counts, counts_host, G * 2 * P * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    dcounts = c->d_own_counts;
  }
  uint8_t* ddead = c->d_own_status;
  uint8_t* dterr = c->d_own_status + G * P;
  DISPATCH_N(c, (k_final_status<19><<<c->G, 32, 0, c->stream>>>(c->st, dcounts, playouts, threshold, ddead, dterr,
                                                                c->d_words)),
             (k_final_status<9><<<c->G, 32, 0, c->stream>>>(c->st, dcounts, playouts, threshold, ddead, dterr,
                                                               c->d_words)));
  c->launches++;
  CK(cudaGetLastError());
  if (dead_host) CK(cudaMemcpyAsync(dead_host, ddead, G * P, cudaMemcpyDeviceToHost, c->stream));
  if (territory_host) CK(cudaMemcpyAsync(territory_host, dterr, G * P, cudaMemcpyDeviceToHost, c->stream));
  if (score_host) CK(cudaMemcpyAsync(score_host, c->d_words, G * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

}  // extern "C"
