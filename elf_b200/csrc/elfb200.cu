// elfb200.cu -- kernels + C ABI of libelfb200.so (board path).
//
// Kernels (all templated on the board size N in {9, 19}; one game per N-lane warp segment):
//   k_reset     clear selected games
//   k_step      GoState::forward for a batch: validate, play, superko, next legal mask
//   k_export    host-facing views (legal/stones/eyes by action index, info words, tt score)
//   k_features  BoardFeature::extractAGZ, float32 [G][18][N][N]
//   k_playout   whole random-policy games with the position (and the incremental safe/atari group
//               masks) held in registers; to-terminal and steady-state ("stream") modes
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
template <int N>
__global__ void __launch_bounds__(BLOCK) k_reset(DevState st, const uint8_t* __restrict__ mask) {
  const Lane L = make_lane<N>();
  bool valid;
  const int g = warp_game<N>(L, st.G, valid);
  if (!valid) return;
  if (mask && !mask[g]) return;
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

// ---------------------------------------------------------------------------------------
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

  uint64_t rowv = valid ? st.cur[(size_t)gs * N + L.row] : 0ull;
  uint32_t b = (uint32_t)rowv, w = (uint32_t)(rowv >> 32);
  // the incremental group status (safe / atari masks, board.cuh) is part of the stored position: a step
  // recounts only the groups the move touched instead of classifying every group from scratch
  const uint64_t sav = valid ? st.sa[(size_t)gs * N + L.row] : 0ull;
  uint32_t safe = (uint32_t)sav, atari = (uint32_t)(sav >> 32);
  BoardMeta meta = load_meta(&st.meta[gs]);
  uint64_t hash = st.hash[gs];
  const uint32_t lrow = valid ? st.legal[(size_t)gs * N + L.row] : 0u;
  int nsk = st.sk_n[gs];
  const int a = valid ? actions[gs] : -1;

  // validate (forward refuses on terminated state, then TryPlay2; go_state.cc:78-83)
  const bool term = is_terminated<N>(meta);
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
    const bool bit = (L.row == y) && ((lrow >> x) & 1u);
    const bool is_legal = game_any<N>(bit, L);
    if (pm >= 0 && !is_legal) pm = MV_NONE;
  }
  const uint64_t pre_hash = hash;
  play_move_cached<N>(b, w, meta, hash, pm, s_zob, L, safe, atari);

  // superko (go_state.cc:96-121): compare with the recorded pre-move positions, then record.
  const uint64_t* skg = st.sk + (size_t)gs * Geo<N>::MAX_PLY;
  const bool sko = superko_scan<N>(skg, pm >= 0 ? nsk : 0, hash, L);
  if (pm >= 0) {
    if (sko) meta.flags |= F_SUPERKO;
    if (L.row == 0) {
      st.sk[(size_t)g * Geo<N>::MAX_PLY + nsk] = pre_hash;
      st.sk_n[g] = nsk + 1;
    }
  }

  // legal mask of the new position
  const uint32_t own = meta.next == S_BLACK ? b : w, opp = meta.next == S_BLACK ? w : b;
  const bool ko_applies = (meta.flags & F_KO_ACTIVE) && meta.ko_color == meta.next;
  const uint32_t lnew = legal_rows_cached<N>(own, opp, safe, atari, L, ko_applies, meta.ko_pt);

  if (valid) {
    if (pm != MV_NONE) {
      const uint64_t nv = (uint64_t)b | ((uint64_t)w << 32);
      st.cur[(size_t)g * N + L.row] = nv;
      st.sa[(size_t)g * N + L.row] = (uint64_t)safe | ((uint64_t)atari << 32);
      st.ring[((size_t)g * 8 + ((meta.ply - 2) & 7)) * N + L.row] = nv;  // go_state.cc:90-92
      st.legal[(size_t)g * N + L.row] = lnew;
      if (L.row == 0) {
        st.hash[g] = hash;
        store_meta(&st.meta[g], meta);
        if (pm >= 0) st.placed[(size_t)g * Geo<N>::P + pm] = (uint16_t)(meta.ply - 1);  // Info::last_placed = _ply (board.cc:680,1379)
      }
    }
    if (ok && L.row == 0) ok[g] = pm != MV_NONE ? 1 : 0;
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
// Per ply this is k_step (validate against the legal rows, play, superko, next legal rows) with the
// position held in registers; a refused move changes nothing and the list goes on, as the reference
// ignores forward()'s verdict there.  Games of one warp (9x9 packs three) may have different
// lengths: the warp runs to the longest, shorter games idle with MV_NONE.
template <int N>
__global__ void __launch_bounds__(BLOCK)
    k_replay(DevState st, const int16_t* __restrict__ moves, int stride, const int32_t* __restrict__ count) {
  __shared__ uint64_t s_zob[Geo<N>::ZOB];
  load_zobrist<N>(s_zob);
  const Lane L = make_lane<N>();
  bool valid;
  const int g = warp_game<N>(L, st.G, valid);
  const int gs = valid ? g : 0;  // safe index for idle lanes (loads only)

  uint32_t b = 0, w = 0, safe = 0, atari = 0;
  BoardMeta meta = initial_meta();
  uint64_t hash = 0;
  uint32_t lrow = valid ? Geo<N>::ROWMASK : 0u;  // every point of the empty board is legal
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
    const int a = (valid && t < n) ? (int)moves[(size_t)gs * stride + t] : -1;
    const bool term = is_terminated<N>(meta);
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
      const bool bit = (L.row == y) && ((lrow >> x) & 1u);
      const bool is_legal = game_any<N>(bit, L);
      if (pm >= 0 && !is_legal) pm = MV_NONE;
    }
    const uint64_t pre_hash = hash;
    play_move_cached<N>(b, w, meta, hash, pm, s_zob, L, safe, atari);
    const bool sko = superko_scan<N>(skg, pm >= 0 ? nsk : 0, hash, L);
    __syncwarp();
    if (pm >= 0) {
      if (sko) meta.flags |= F_SUPERKO;
      if (valid && L.row == 0) skg[nsk] = pre_hash;
      nsk++;
    }
    const uint32_t own = meta.next == S_BLACK ? b : w, opp = meta.next == S_BLACK ? w : b;
    const bool ko_applies = (meta.flags & F_KO_ACTIVE) && meta.ko_color == meta.next;
    const uint32_t lnew = legal_rows_cached<N>(own, opp, safe, atari, L, ko_applies, meta.ko_pt);
    if (valid && pm != MV_NONE) {
      lrow = lnew;
      st.ring[((size_t)g * 8 + ((meta.ply - 2) & 7)) * N + L.row] = (uint64_t)b | ((uint64_t)w << 32);  // go_state.cc:90-92
      if (pm >= 0 && L.row == 0) st.placed[(size_t)g * Geo<N>::P + pm] = (uint16_t)(meta.ply - 1);
    }
    __syncwarp();
  }
  if (valid) {
    st.cur[(size_t)g * N + L.row] = (uint64_t)b | ((uint64_t)w << 32);
    st.sa[(size_t)g * N + L.row] = (uint64_t)safe | ((uint64_t)atari << 32);
    st.legal[(size_t)g * N + L.row] = lrow;
    if (L.row == 0) {
      st.hash[g] = hash;
      store_meta(&st.meta[g], meta);
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

  const uint64_t rowv = valid ? st.cur[(size_t)gs * N + L.row] : 0ull;
  uint32_t b = (uint32_t)rowv, w = (uint32_t)(rowv >> 32);
  const uint64_t sav = valid ? st.sa[(size_t)gs * N + L.row] : 0ull;
  uint32_t safe = (uint32_t)sav, atari = (uint32_t)(sav >> 32);
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

  // legal rows for the side to move
  const uint32_t own = meta.next == S_BLACK ? b : w, opp = meta.next == S_BLACK ? w : b;
  const bool ko_applies = (meta.flags & F_KO_ACTIVE) && meta.ko_color == meta.next;
  const uint32_t lnew = legal_rows_cached<N>(own, opp, safe, atari, L, ko_applies, meta.ko_pt);
  if (open) {
    st.cur[(size_t)g * N + L.row] = (uint64_t)b | ((uint64_t)w << 32);
    st.sa[(size_t)g * N + L.row] = (uint64_t)safe | ((uint64_t)atari << 32);
    st.legal[(size_t)g * N + L.row] = lnew;
    if (L.row == 0) {
      st.hash[g] = hash;
      store_meta(&st.meta[g], meta);
    }
  }
}

// ---------------------------------------------------------------------------------------
template <int N>
__global__ void __launch_bounds__(BLOCK)
    k_export(DevState st, uint8_t* __restrict__ legal_out, uint8_t* __restrict__ stones_out,
             uint8_t* __restrict__ eyes_out, int eye_player, int32_t* __restrict__ info_out,
             int32_t* __restrict__ score_out) {
  const Lane L = make_lane<N>();
  bool valid;
  const int g = warp_game<N>(L, st.G, valid);
  const int gs = valid ? g : 0;
  const uint64_t rowv = valid ? st.cur[(size_t)gs * N + L.row] : 0ull;
  const uint32_t b = (uint32_t)rowv, w = (uint32_t)(rowv >> 32);
  const BoardMeta meta = load_meta(&st.meta[gs]);
  constexpr int P = Geo<N>::P;
  if (legal_out && valid) {
    const uint32_t l = st.legal[(size_t)g * N + L.row];
    for (int x = 0; x < N; ++x) legal_out[(size_t)g * (P + 1) + x * N + L.row] = (l >> x) & 1u;
    if (L.row == 0) legal_out[(size_t)g * (P + 1) + P] = 1;
  }
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
  if (info_out && valid && L.row == 0) {
    auto p2a = [](int p) -> int {
      if (p == MV_PASS) return Geo<N>::P;
      if (p < 0) return -1;
      return (p % N) * N + p / N;
    };
    int32_t* o = info_out + (size_t)g * ELFB200_INFO_FIELDS;
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
  const uint64_t rowv = L.active ? st.cur[(size_t)g * N + L.row] : 0ull;
  const uint32_t b = (uint32_t)rowv, w = (uint32_t)(rowv >> 32);
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
// Whole random-policy games, position in registers (BASELINE configs 1/2/5).
//
// stream_plies == 0: every slot plays ONE game (id first_id + g) to terminated() / max_plies.
// stream_plies  > 0: "4096 concurrent games" in steady state -- every slot plays exactly
//   stream_plies plies, starting a new game (id += G) whenever its game ends, so that G games are
//   in flight at all times like the reference's game threads (GoGameBase::mainLoop,
//   common/game_base.h:41).  Per slot: out_chk = fold of the games' checksums in order,
//   out_plies = plies played, out_score = number of games started, out_hash = last position hash.
// One warp per CTA: 4096 games are 4096 warps over 132 SMs = 31.03 per SM; with 4-warp CTAs
// the SMs holding 8 CTAs (32 warps) set the kernel time while those with 7 idle 12.5 % of it.
constexpr int PLAYOUT_WARPS = 1;

template <int N>
__global__ void __launch_bounds__(PLAYOUT_WARPS * 32)
    k_playout(int G, uint64_t seed, uint64_t first_id, int max_plies, int stream_plies,
              uint64_t* __restrict__ sk, uint64_t* __restrict__ out_chk, int32_t* __restrict__ out_plies,
              int32_t* __restrict__ out_score, uint64_t* __restrict__ out_hash) {
  __shared__ uint64_t s_zob[Geo<N>::ZOB];
  // 4096-bit Bloom filter per game over the recorded pre-move hashes: the exact superko scan
  // (go_state.cc:96-111) only runs when both probe bits are set (false-positive rate ~3 % at
  // 400 recorded positions), which removes ~1.8 KB of history reads per ply.
  __shared__ uint32_t s_bloom[PLAYOUT_WARPS][Geo<N>::GPW][128];
  load_zobrist<N>(s_zob);
  const Lane L = make_lane<N>();
  bool valid;
  const int g = warp_game<N>(L, G, valid);
  uint64_t gid = first_id + (uint64_t)g;
  uint64_t* skg = sk + (size_t)(valid ? g : 0) * Geo<N>::MAX_PLY;
  uint32_t* bloom = s_bloom[threadIdx.x >> 5][L.sub];
  for (int i = L.row; i < 128; i += N)
    if (L.active) bloom[i] = 0u;
  __syncwarp();

  uint32_t b = 0, w = 0, safe = 0, atari = 0;  // safe/atari: incremental group status (board.cuh)
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
          b = w = safe = atari = 0;
          meta = initial_meta();
          hash = chk = 0;
          nsk = t = 0;
          for (int i = L.row; i < 128; i += N) bloom[i] = 0u;
        }
        __syncwarp();
      }
      term = !valid || budget_out;
    } else {
      term = !valid || over;
    }
    if (__all_sync(FULL, term)) break;
    const uint32_t own = meta.next == S_BLACK ? b : w, opp = meta.next == S_BLACK ? w : b;
    const bool ko_applies = (meta.flags & F_KO_ACTIVE) && meta.ko_color == meta.next;
    const uint32_t legal = legal_rows_cached<N>(own, opp, safe, atari, L, ko_applies, meta.ko_pt);
    const uint32_t cand = legal & ~true_eye_rows<N>(own, opp, L);
    const int n = game_sum<N>(__popc(cand), L);
    const uint64_t rx = game_xor64<N>(L.active ? pp_row_term((uint32_t)L.row, legal) : 0ull, L);
    const uint64_t chk2 = pp_fold3(chk, hash, rx, meta.b_cap, meta.w_cap, meta.next);
    const int k = n > 0 ? (int)pp_pick(seed, gid, meta.ply, (uint32_t)n) : 0;
    const int p = select_kth_action_order<N>(cand, k, L);
    const int pm = term ? MV_NONE : (n > 0 ? p : MV_PASS);
    const uint64_t pre_hash = hash;
    play_move_cached<N>(b, w, meta, hash, pm, s_zob, L, safe, atari);
    const uint32_t q1 = (uint32_t)hash & 4095u, q2 = (uint32_t)(hash >> 12) & 4095u;
    const bool maybe = pm >= 0 && ((bloom[q1 >> 5] >> (q1 & 31)) & (bloom[q2 >> 5] >> (q2 & 31)) & 1u);
    bool sko = false;
    if (__any_sync(FULL, maybe)) sko = superko_scan<N>(skg, maybe ? nsk : 0, hash, L);
    __syncwarp();
    if (pm >= 0) {
      if (sko) meta.flags |= F_SUPERKO;
      if (L.row == 0) {
        skg[nsk] = pre_hash;
        const uint32_t i1 = (uint32_t)pre_hash & 4095u, i2 = (uint32_t)(pre_hash >> 12) & 4095u;
        bloom[i1 >> 5] |= 1u << (i1 & 31);
        bloom[i2 >> 5] |= 1u << (i2 & 31);
      }
      nsk++;
    }
    if (!term) {
      chk = chk2;
      t++;
      ts++;
    }
    __syncwarp();
  }
  chk = pp_fold_final(chk, hash, meta.ply);
  const int score = tt_score<N>(b, w, L);
  if (valid && L.row == 0) {
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

// ---------------------------------------------------------------------------------------
// k_playout in the two-rows-per-lane layout (board2.cuh): three 19x19 games per warp, 30 of 32 lanes
// busy.  Same workload, same outputs, same checksums as k_playout (elfb200_set_playout_layout picks).
template <int N>
__global__ void __launch_bounds__(PLAYOUT_WARPS * 32)
    k_playout2(int G, uint64_t seed, uint64_t first_id, int max_plies, int stream_plies,
               uint64_t* __restrict__ sk, uint64_t* __restrict__ out_chk, int32_t* __restrict__ out_plies,
               int32_t* __restrict__ out_score, uint64_t* __restrict__ out_hash) {
  constexpr int GPW = Geo2<N>::GPW, LPG = Geo2<N>::LPG;
  __shared__ uint64_t s_zob[Geo<N>::ZOB];
  __shared__ uint32_t s_bloom[PLAYOUT_WARPS][GPW][128];  // see k_playout
  load_zobrist<N>(s_zob);
  const Lane2 L = make_lane2<N>();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int g = warp * GPW + L.sub;
  const bool valid = L.active && g < G;
  uint64_t gid = first_id + (uint64_t)g;
  uint64_t* skg = sk + (size_t)(valid ? g : 0) * Geo<N>::MAX_PLY;
  uint32_t* bloom = s_bloom[threadIdx.x >> 5][L.sub];
  if (L.active)
    for (int i = L.li; i < 128; i += LPG) bloom[i] = 0u;
  __syncwarp();

  P2 b = zero2(), w = zero2(), safe = zero2(), atari = zero2();
  BoardMeta meta = initial_meta();
  uint64_t hash = 0, chk = 0, acc = 0;
  int nsk = 0, t = 0, ts = 0, ngames = 0;
  const bool stream = stream_plies > 0;
  const bool has_hi = 2 * L.li + 1 < N;

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
          b = w = safe = atari = zero2();
          meta = initial_meta();
          hash = chk = 0;
          nsk = t = 0;
          for (int i = L.li; i < 128; i += LPG) bloom[i] = 0u;
        }
        __syncwarp();
      }
      term = !valid || budget_out;
    } else {
      term = !valid || over;
    }
    if (__all_sync(FULL, term)) break;
    const P2 own = meta.next == S_BLACK ? b : w, opp = meta.next == S_BLACK ? w : b;
    const bool ko_applies = (meta.flags & F_KO_ACTIVE) && meta.ko_color == meta.next;
    const P2 legal = legal_rows_cached<N>(own, opp, safe, atari, L, ko_applies, meta.ko_pt);
    const P2 cand = legal & ~true_eye_rows<N>(own, opp, L);
    const int n = game_sum(popc2(cand), L);
    uint64_t rt = 0;
    if (L.active) {
      rt = pp_row_term((uint32_t)(2 * L.li), legal.lo);
      if (has_hi) rt ^= pp_row_term((uint32_t)(2 * L.li + 1), legal.hi);
    }
    const uint64_t rx = game_xor64<N>(rt, L);
    const uint64_t chk2 = pp_fold3(chk, hash, rx, meta.b_cap, meta.w_cap, meta.next);
    const int k = n > 0 ? (int)pp_pick(seed, gid, meta.ply, (uint32_t)n) : 0;
    const int p = select_kth_action_order<N>(cand, k, L);
    const int pm = term ? MV_NONE : (n > 0 ? p : MV_PASS);
    const uint64_t pre_hash = hash;
    play_move_cached<N>(b, w, meta, hash, pm, s_zob, L, safe, atari);
    const uint32_t q1 = (uint32_t)hash & 4095u, q2 = (uint32_t)(hash >> 12) & 4095u;
    const bool maybe = pm >= 0 && ((bloom[q1 >> 5] >> (q1 & 31)) & (bloom[q2 >> 5] >> (q2 & 31)) & 1u);
    bool sko = false;
    if (__any_sync(FULL, maybe)) sko = superko_scan<N>(skg, maybe ? nsk : 0, hash, L);
    __syncwarp();
    if (pm >= 0) {
      if (sko) meta.flags |= F_SUPERKO;
      if (L.li == 0 && L.active) {
        skg[nsk] = pre_hash;
        const uint32_t i1 = (uint32_t)pre_hash & 4095u, i2 = (uint32_t)(pre_hash >> 12) & 4095u;
        bloom[i1 >> 5] |= 1u << (i1 & 31);
        bloom[i2 >> 5] |= 1u << (i2 & 31);
      }
      nsk++;
    }
    if (!term) {
      chk = chk2;
      t++;
      ts++;
    }
    __syncwarp();
  }
  chk = pp_fold_final(chk, hash, meta.ply);
  const int score = tt_score<N>(b, w, L);
  if (valid && L.li == 0) {
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
                  c->d_replay, c->st.placed, c->st.sa, c->d_exp_table, c->d_done};
  for (void* p : ptrs)
    if (p) cudaFree(p);
  if (c->h_pin) cudaFreeHost(c->h_pin);
  if (c->h_map) cudaFreeHost(c->h_map);
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

int elfb200_get_info(elfb200_ctx* c, int32_t* info_host) {
  if (!c || !info_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  CK(cudaSetDevice(c->device));
  int rc = run_export(c, nullptr, nullptr, nullptr, 0, c->d_words, nullptr);
  if (rc) return rc;
  CK(cudaMemcpyAsync(info_host, c->d_words, (size_t)c->G * ELFB200_INFO_FIELDS * 4,
                     cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_get_stones(elfb200_ctx* c, uint8_t* stones_host) {
  if (!c || !stones_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  CK(cudaSetDevice(c->device));
  int rc = run_export(c, nullptr, c->d_bytes, nullptr, 0, nullptr, nullptr);
  if (rc) return rc;
  CK(cudaMemcpyAsync(stones_host, c->d_bytes, (size_t)c->G * c->N * c->N, cudaMemcpyDeviceToHost,
                     c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_get_legal(elfb200_ctx* c, uint8_t* legal_host) {
  if (!c || !legal_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  CK(cudaSetDevice(c->device));
  int rc = run_export(c, c->d_bytes, nullptr, nullptr, 0, nullptr, nullptr);
  if (rc) return rc;
  CK(cudaMemcpyAsync(legal_host, c->d_bytes, (size_t)c->G * (c->N * c->N + 1),
                     cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_get_true_eyes(elfb200_ctx* c, int player, uint8_t* eyes_host) {
  if (!c || !eyes_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  if (player < 0 || player > 2) return elfb200_fail(ELFB200_ERR_ARG, "player must be 0, 1 or 2");
  CK(cudaSetDevice(c->device));
  int rc = run_export(c, nullptr, nullptr, c->d_bytes, player, nullptr, nullptr);
  if (rc) return rc;
  CK(cudaMemcpyAsync(eyes_host, c->d_bytes, (size_t)c->G * c->N * c->N, cudaMemcpyDeviceToHost,
                     c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
}

int elfb200_get_tt_score(elfb200_ctx* c, int32_t* score_host) {
  if (!c || !score_host) return elfb200_fail(ELFB200_ERR_ARG, "NULL argument");
  CK(cudaSetDevice(c->device));
  int rc = run_export(c, nullptr, nullptr, nullptr, 0, nullptr, c->d_words);
  if (rc) return rc;
  CK(cudaMemcpyAsync(score_host, c->d_words, (size_t)c->G * 4, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return ELFB200_OK;
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
  if (c->N == 19 && layout == 1) {
    const int pgrid2 = ((c->G + Geo2<19>::GPW - 1) / Geo2<19>::GPW + PLAYOUT_WARPS - 1) / PLAYOUT_WARPS;
    k_playout2<19><<<pgrid2, PLAYOUT_WARPS * 32, 0, c->stream>>>(c->G, seed, first_game_id, max_plies, stream_plies, c->d_po_sk,
                                                               c->d_po_chk, c->d_po_plies, c->d_po_score, c->d_po_hash);
    c->launches++;
    CK(cudaGetLastError());
    return ELFB200_OK;
  }
  const int gpw = 32 / c->N;
  const int pgrid = ((c->G + gpw - 1) / gpw + PLAYOUT_WARPS - 1) / PLAYOUT_WARPS;
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
