// board2.cuh -- the board primitives of board.cuh in the "two rows per lane" layout (19x19 only).
//
// board.cuh gives one board row to a lane: a 19x19 game occupies lanes 0..18 of its warp and 13 of
// the 32 lanes idle in every instruction.  Here lane i of a game holds rows 2i (`lo`) and 2i+1 (`hi`):
// a game is 10 lanes, THREE games share a warp (30 of 32 lanes busy), and
//   * a vertical neighbour step is one shuffle per row PAIR: up(v)   = { shfl_up(v.hi), v.lo },
//                                                           down(v) = { v.hi, shfl_down(v.lo) };
//   * row 19 (the `hi` word of a game's last lane) does not exist and is kept zero by the board masks,
//     so nothing leaks between the games of a warp and the fills need no boundary selects;
//   * per-game sums of all three games come out of ONE warp-wide REDUX: each game adds its value into
//     its own 10-bit field of the word (sums are <= 361).
// Per warp instruction this serves three games instead of one; the price is fill loops that run to the
// slowest of the three.  Same observable behaviour as board.cuh: the playout checksum (hash, captures,
// legal mask of every position) pins both against the oracle and the compiled reference.
#pragma once

#include "board.cuh"

namespace elfb200 {

struct P2 {
  uint32_t lo, hi;
};
__device__ __forceinline__ P2 operator|(P2 a, P2 b) { return {a.lo | b.lo, a.hi | b.hi}; }
__device__ __forceinline__ P2 operator&(P2 a, P2 b) { return {a.lo & b.lo, a.hi & b.hi}; }
__device__ __forceinline__ P2 operator~(P2 a) { return {~a.lo, ~a.hi}; }
__device__ __forceinline__ P2 operator<<(P2 a, int s) { return {a.lo << s, a.hi << s}; }
__device__ __forceinline__ P2 operator>>(P2 a, int s) { return {a.lo >> s, a.hi >> s}; }
__device__ __forceinline__ P2& operator|=(P2& a, P2 b) { a.lo |= b.lo; a.hi |= b.hi; return a; }
__device__ __forceinline__ P2& operator&=(P2& a, P2 b) { a.lo &= b.lo; a.hi &= b.hi; return a; }
__device__ __forceinline__ bool nz(P2 a) { return (a.lo | a.hi) != 0u; }
__device__ __forceinline__ bool ne(P2 a, P2 b) { return ((a.lo ^ b.lo) | (a.hi ^ b.hi)) != 0u; }
__device__ __forceinline__ int popc2(P2 a) { return __popc(a.lo) + __popc(a.hi); }
__device__ __forceinline__ P2 zero2() { return {0u, 0u}; }

template <int N>
struct Geo2 {
  static_assert(N == 19, "the two-rows-per-lane layout packs three 10-bit sums into one REDUX: 19x19 only");
  static constexpr int LPG = (N + 1) / 2;  // lanes per game
  static constexpr int GPW = 32 / LPG;     // games per warp
  static constexpr int LANES = GPW * LPG;
  static constexpr uint32_t SEG = (1u << LPG) - 1u;
};

struct Lane2 {
  int lane, sub, li, base, shift;  // li: lane index inside the game; shift: this game's field in packed sums
  uint32_t segmask;
  bool active;
  P2 rm;  // on-board mask of this lane's two rows (hi = 0 for the row that does not exist)
};

template <int N>
__device__ __forceinline__ Lane2 make_lane2() {
  Lane2 L;
  L.lane = threadIdx.x & 31;
  L.active = L.lane < Geo2<N>::LANES;
  L.sub = L.active ? L.lane / Geo2<N>::LPG : 0;
  L.li = L.active ? L.lane - L.sub * Geo2<N>::LPG : 0;
  L.base = L.sub * Geo2<N>::LPG;
  L.shift = 10 * L.sub;
  L.segmask = L.active ? (Geo2<N>::SEG << L.base) : 0u;
  L.rm.lo = L.active ? Geo<N>::ROWMASK : 0u;
  L.rm.hi = (L.active && 2 * L.li + 1 < N) ? Geo<N>::ROWMASK : 0u;
  return L;
}

// ---- neighbours -------------------------------------------------------------------------------------
// raw: no boundary handling (for dilations that are ANDed with a board mask / link mask afterwards)
__device__ __forceinline__ P2 up_raw(P2 v) { return {__shfl_up_sync(FULL, v.hi, 1), v.lo}; }
__device__ __forceinline__ P2 dn_raw(P2 v) { return {v.hi, __shfl_down_sync(FULL, v.lo, 1)}; }
// exact: rows outside the game read as 0
template <int N>
__device__ __forceinline__ P2 up_of(P2 v, const Lane2& L) {
  const uint32_t u = __shfl_up_sync(FULL, v.hi, 1);
  return {L.li == 0 ? 0u : u, v.lo};
}
template <int N>
__device__ __forceinline__ P2 dn_of(P2 v, const Lane2& L) {
  const uint32_t d = __shfl_down_sync(FULL, v.lo, 1);
  return {v.hi, (L.li == Geo2<N>::LPG - 1 || !L.active) ? 0u : d};
}
template <int N>
__device__ __forceinline__ P2 nbr4(P2 v, const Lane2& L) {
  return (v << 1) | (v >> 1) | up_of<N>(v, L) | dn_of<N>(v, L);
}
__device__ __forceinline__ P2 grow_raw(P2 v) { return (v << 1) | (v >> 1) | up_raw(v) | dn_raw(v); }

// ---- per-game reductions ------------------------------------------------------------------------------
// sum of v (0 <= per-game total <= 1023) over each game's lanes: one REDUX for all three games
__device__ __forceinline__ int game_sum(int v, const Lane2& L) {
  const uint32_t r = __reduce_add_sync(FULL, L.active ? ((uint32_t)v << L.shift) : 0u);
  return (int)((r >> L.shift) & 1023u);
}
template <int N>  // board.cuh's spelling, for code written for both layouts
__device__ __forceinline__ int game_sum(int v, const Lane2& L) {
  return game_sum(v, L);
}
template <int N>
__device__ __forceinline__ uint64_t game_xor64(uint64_t v, const Lane2& L) {
  uint32_t lo = 0, hi = 0;
#pragma unroll
  for (int k = 0; k < Geo2<N>::GPW; ++k) {
    const bool mine = L.active && L.sub == k;
    const uint32_t a = __reduce_xor_sync(FULL, mine ? (uint32_t)v : 0u);
    const uint32_t b = __reduce_xor_sync(FULL, mine ? (uint32_t)(v >> 32) : 0u);
    if (L.sub == k) {
      lo = a;
      hi = b;
    }
  }
  return ((uint64_t)hi << 32) | lo;
}
__device__ __forceinline__ bool game_any(bool pred, const Lane2& L) {
  return (__ballot_sync(FULL, pred) & L.segmask) != 0u;
}

// ---- flood fill -------------------------------------------------------------------------------------------
__device__ __forceinline__ P2 flood(P2 g, P2 through) {
  while (true) {
    const P2 n1 = g | (grow_raw(g) & through);
    const P2 n2 = n1 | (grow_raw(n1) & through);
    const bool ch = ne(n2, g);
    g = n2;
    if (!__any_sync(FULL, ch)) break;
  }
  return g;
}

template <int N>
__device__ __forceinline__ uint64_t zob_rows(const uint64_t* __restrict__ zob, P2 bits, const Lane2& L) {
  return zob_row<N>(zob, 2 * L.li, bits.lo) ^ zob_row<N>(zob, 2 * L.li + 1, bits.hi);  // hi == 0 where the row does not exist
}

// ---- same-colour links --------------------------------------------------------------------------------------
struct Links2 {
  P2 l, r, u, d;
};
template <int N>
__device__ __forceinline__ Links2 make_links(P2 own, P2 opp, const Lane2& L) {
  Links2 k;
  k.l = (own & (own << 1)) | (opp & (opp << 1));
  k.r = (own & (own >> 1)) | (opp & (opp >> 1));
  k.u = (own & up_of<N>(own, L)) | (opp & up_of<N>(opp, L));
  k.d = (own & dn_of<N>(own, L)) | (opp & dn_of<N>(opp, L));
  return k;
}
__device__ __forceinline__ P2 grow_link(P2 g, const Links2& k) {
  return g | ((g << 1) & k.l) | ((g >> 1) & k.r) | (up_raw(g) & k.u) | (dn_raw(g) & k.d);
}

// ---- legality, eyes, score (see board.cuh for the rules each follows) -------------------------------------------
template <int N>
__device__ __forceinline__ P2 legal_rows_cached(P2 own, P2 opp, P2 safe, P2 atari, const Lane2& L, bool ko_applies,
                                                int ko_pt) {
  const P2 e = ~(own | opp) & L.rm;
  const P2 en = nbr4<N>(e, L);
  P2 legal = e & en;
  const P2 hard = e & ~en;
  if (__any_sync(FULL, nz(hard))) legal |= hard & (nbr4<N>(safe & own, L) | nbr4<N>(atari & opp, L));
  if (ko_applies) {
    const int ky = ko_pt / N, kx = ko_pt - ky * N;
    if ((ky >> 1) == L.li) {
      if (ky & 1)
        legal.hi &= ~(1u << kx);
      else
        legal.lo &= ~(1u << kx);
    }
  }
  return legal & L.rm;
}

template <int N>
__device__ __forceinline__ P2 true_eye_rows(P2 own, P2 opp, const Lane2& L) {
  const P2 e = ~(own | opp) & L.rm;
  const P2 notown = ~own & L.rm;
  const P2 eyeish = e & ~nbr4<N>(notown, L);
  const P2 o_u = up_of<N>(opp, L), o_d = dn_of<N>(opp, L);
  const P2 d1 = o_u << 1, d2 = o_u >> 1, d3 = o_d << 1, d4 = o_d >> 1;
  const P2 ge1 = d1 | d2 | d3 | d4;
  const P2 ge2 = (d1 & (d2 | d3 | d4)) | (d2 & (d3 | d4)) | (d3 & d4);
  const uint32_t side = 1u | (1u << (N - 1));
  // rows 0 and N-1 are `lo` words (N odd): of the game's first and last lane
  const P2 edge = {(L.li == 0 || L.li == Geo2<N>::LPG - 1) ? Geo<N>::ROWMASK : side, side};
  const P2 fake = (edge & ge1) | (~edge & ge2);
  return eyeish & ~fake & L.rm;
}

template <int N>
__device__ __forceinline__ int tt_score(P2 b, P2 w, const Lane2& L) {
  const P2 e = ~(b | w) & L.rm;
  P2 gb = b, gw = w;
  while (true) {
    const P2 b1 = gb | (grow_raw(gb) & e), w1 = gw | (grow_raw(gw) & e);
    const P2 b2 = b1 | (grow_raw(b1) & e), w2 = w1 | (grow_raw(w1) & e);
    const bool ch = ne(b2, gb) | ne(w2, gw);
    gb = b2;
    gw = w2;
    if (!__any_sync(FULL, ch)) break;
  }
  return game_sum(popc2(gb & ~gw), L) - game_sum(popc2(gw & ~gb), L);
}

__device__ __forceinline__ uint32_t spread_even(uint32_t v) {  // bit i -> bit 2i (i < 16)
  v = (v | (v << 8)) & 0x00FF00FFu;
  v = (v | (v << 4)) & 0x0F0F0F0Fu;
  v = (v | (v << 2)) & 0x33333333u;
  v = (v | (v << 1)) & 0x55555555u;
  return v;
}

// k-th candidate in ascending action order a = x*N + y; returns p = y*N + x (see board.cuh)
template <int N>
__device__ __forceinline__ int select_kth_action_order(P2 cand, int k, const Lane2& L) {
  int lo = 0, hi = N - 1;
#pragma unroll
  for (int it = 0; it < 5; ++it) {
    const int mid = (lo + hi) >> 1;
    const uint32_t m = (2u << mid) - 1u;
    const int c = game_sum(__popc(cand.lo & m) + __popc(cand.hi & m), L);
    if (c > k)
      hi = mid;
    else
      lo = mid + 1;
  }
  const int x = lo < N ? lo : N - 1;
  const uint32_t mb = (1u << x) - 1u;
  const int before = game_sum(__popc(cand.lo & mb) + __popc(cand.hi & mb), L);
  const uint32_t c_lo = (__ballot_sync(FULL, (cand.lo >> x) & 1u) >> L.base) & Geo2<N>::SEG;
  const uint32_t c_hi = (__ballot_sync(FULL, (cand.hi >> x) & 1u) >> L.base) & Geo2<N>::SEG;
  const uint32_t colmask = spread_even(c_lo) | (spread_even(c_hi) << 1);  // bit y = row y of column x
  const int y = (int)__fns(colmask, 0, k - before + 1);
  return y * N + x;
}

template <int N>
__device__ __forceinline__ bool superko_scan(const uint64_t* __restrict__ hist, int n, uint64_t hash, const Lane2& L) {
  bool found = false;
  if (L.active)
    for (int i = L.li; i < n; i += Geo2<N>::LPG) found |= (hist[i] == hash);
  return game_any(found, L);
}

// ---- applying a move with the incremental safe/atari masks (play_move_cached of board.cuh) ----------------------
template <int N>
__device__ __forceinline__ int play_move_cached(P2& b, P2& w, BoardMeta& meta, uint64_t& hash, int p,
                                                const uint64_t* __restrict__ zob, const Lane2& L, P2& safe, P2& atari) {
  const int player = meta.next;
  const int oppc = S_BLACK + S_WHITE - player;
  const bool is_stone = p >= 0;
  P2 own = player == S_BLACK ? b : w;
  P2 opp = player == S_BLACK ? w : b;
  const int y = is_stone ? p / N : -9, x = is_stone ? p - y * N : 0;
  const uint32_t xb = 1u << x;
  const uint32_t side = (xb << 1) | (xb >> 1);
  const int dlo = 2 * L.li - y, dhi = dlo + 1;  // row distance of this lane's two rows from the stone
  P2 mybit = {(dlo == 0 && L.active) ? xb : 0u, (dhi == 0 && L.active) ? xb : 0u};
  P2 nb = {dlo == 0 ? side : ((dlo == 1 || dlo == -1) ? xb : 0u), dhi == 0 ? side : ((dhi == 1 || dhi == -1) ? xb : 0u)};
  nb &= L.rm;
  const bool single = !game_any(nz(nb & own), L);
  own |= mybit;
  uint64_t dh = 0;
  int ncap = 0;
  P2 dead = zero2(), dead_nb = zero2();
  const P2 dseed = nb & opp & atari;  // enemy neighbour groups whose only liberty was this point
  if (__any_sync(FULL, nz(dseed))) {
    dead = flood(dseed, opp);
    ncap = game_sum(popc2(dead), L);
    opp &= ~dead;
    safe &= ~dead;
    atari &= ~dead;
    dh = zob_color(game_xor64<N>(zob_rows<N>(zob, dead, L), L), oppc);
    dead_nb = nbr4<N>(dead, L);
  }
  if (is_stone) {
    hash ^= dh ^ zob_color(zob[(y + 1) * Geo<N>::E + (x + 1)], player);
    if (player == S_BLACK) {
      b = own; w = opp; meta.b_cap += ncap;
    } else {
      w = own; b = opp; meta.w_cap += ncap;
    }
  }
  const P2 stones = own | opp;
  const P2 e2 = ~stones & L.rm;
  const int libs = game_sum(popc2(nb & e2), L);
  if (__any_sync(FULL, nz(dead))) {
    const uint32_t bal = __ballot_sync(FULL, nz(dead)) & L.segmask;
    const int src = __ffs(bal) - 1;
    const int mine = dead.lo ? (2 * L.li) * N + __ffs(dead.lo) - 1 : (2 * L.li + 1) * N + __ffs(dead.hi) - 1;
    const int kp = __shfl_sync(FULL, mine, src & 31);
    if (is_stone && ncap == 1 && single && libs == 1) {  // simple ko, board.cc:1384-1393
      meta.ko_pt = (int16_t)kp;
      meta.ko_color = (uint8_t)oppc;
      meta.flags |= F_KO_ACTIVE;
    } else if (is_stone) {
      meta.flags &= ~F_KO_ACTIVE;
    }
  } else if (is_stone) {
    meta.flags &= ~F_KO_ACTIVE;
  }
  // recount the groups whose liberties may have changed
  P2 seeds = (mybit | nb | dead_nb) & stones;
  if (single) {
    if (libs == 1) atari |= mybit; else safe |= mybit;
    seeds &= ~mybit;
  }
  if (__any_sync(FULL, nz(seeds))) {
    const Links2 k = make_links<N>(own, opp, L);
    const P2 linked = k.l | k.r | k.u | k.d;
    while (true) {
      const uint32_t bal = __ballot_sync(FULL, nz(seeds)) & L.segmask;
      const int src = __ffs(bal) - 1;
      P2 grp = zero2();
      if (L.lane == src) {
        if (seeds.lo) grp.lo = seeds.lo & (0u - seeds.lo); else grp.hi = seeds.hi & (0u - seeds.hi);
      }
      if (__any_sync(FULL, nz(grp & linked))) {  // single stones need no fill
        while (true) {
          const P2 g1 = grow_link(grp, k);
          const P2 g2 = grow_link(g1, k);
          const bool ch = ne(g2, grp);
          grp = g2;
          if (!__any_sync(FULL, ch)) break;
        }
      }
      const int nl = game_sum(popc2(nbr4<N>(grp, L) & e2), L);
      if (nl == 1) {
        atari |= grp;
        safe &= ~grp;
      } else {
        safe |= grp;
        atari &= ~grp;
      }
      seeds &= ~grp;
      if (!__any_sync(FULL, nz(seeds))) break;
    }
  }
  if (p != MV_NONE) {
    meta.next = (uint8_t)oppc;
    meta.last2 = meta.last1;
    meta.last1 = (int16_t)p;
    meta.ply++;
  }
  return ncap;
}

}  // namespace elfb200
