// common.cuh -- pieces shared by the translation units of libelfb200.so (board path: elfb200.cu,
// search path: mcts.cu): Zobrist table, launch geometry, the HBM state descriptor and the context.
#pragma once

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>

#include "board.cuh"
#include "elfb200.h"

namespace elfb200 {

static __device__ const uint64_t g_zobrist[441] = {
#include "elfb200_zobrist.inc"
};

constexpr int BLOCK = 128;  // 4 warps per CTA
constexpr int WARPS = BLOCK / 32;

template <int N>
__device__ __forceinline__ void load_zobrist(uint64_t* s_zob) {
  for (int i = threadIdx.x; i < Geo<N>::ZOB; i += blockDim.x) s_zob[i] = g_zobrist[i];
  __syncthreads();
}

template <int N>
__device__ __forceinline__ int warp_game(const Lane& L, int G, bool& valid) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int g = warp * Geo<N>::GPW + L.sub;
  valid = L.active && g < G;
  return g;
}

__device__ __forceinline__ BoardMeta initial_meta() {
  BoardMeta m;
  m.ply = 1;
  m.next = S_BLACK;
  m.flags = 0;
  m.last1 = MV_INVALID;
  m.last2 = MV_INVALID;
  m.ko_pt = -1;
  m.ko_color = 0;
  m.pad = 0;
  m.b_cap = 0;
  m.w_cap = 0;
  return m;
}

__device__ __forceinline__ BoardMeta load_meta(const BoardMeta* p) {
  uint4 v = *reinterpret_cast<const uint4*>(p);
  BoardMeta m;
  memcpy(&m, &v, 16);
  return m;
}
__device__ __forceinline__ void store_meta(BoardMeta* p, const BoardMeta& m) {
  uint4 v;
  memcpy(&v, &m, 16);
  *reinterpret_cast<uint4*>(p) = v;
}

struct DevState {
  uint64_t* cur;
  uint64_t* ring;
  uint32_t* legal;
  uint64_t* hash;
  BoardMeta* meta;
  uint64_t* sk;
  int32_t* sk_n;
  uint64_t* sa;      // [G][N] incremental group status rows: safe (>= 2 liberties) | atari (exactly 1) << 32, see board.cuh
  uint16_t* placed;  // [G][N*N] ply at which the stone on a point was placed (Info::last_placed, board.h:68)
  int G;
};


// ---- AGZ feature planes -------------------------------------------------------------------------
// BoardFeature::extractAGZ (board_feature.cc:247-290) for one position whose <=8 history positions
// (newest first) are staged in shared memory as rows[t][y] = black_row | white_row << 32.
// One thread per OUTPUT cell: the thread resolves its cell through the inverse D4 once
// (InvTransform, board_feature.h:115-130), then emits the 16 stone planes and the 2 side-to-move
// planes; for a fixed plane consecutive threads write consecutive floats (coalesced 128 B/warp).
__device__ __forceinline__ void d4_inverse(int N, int d4, int tx, int ty, int& x, int& y) {
  int a = tx, b = ty;
  if (d4 & 4) { int t = a; a = b; b = t; }
  switch (d4 & 3) {
    case 1: x = N - b - 1; y = a; break;
    case 2: x = N - a - 1; y = N - b - 1; break;
    case 3: x = b; y = N - a - 1; break;
    default: x = a; y = b; break;
  }
}

// ---- feature output formats -----------------------------------------------------------------------
// FEAT_F32_NCHW is the GoFeature tensor contract (float32 [n][18][N][N], game_feature.h:159-206).
// The 16-bit NHWC formats are the fast mode for a network that runs in half precision with
// channels-last convolutions: [n][N][N][cpad] with the 18 planes in channels 0..17 and zeros above
// (cpad a multiple of 8: 16 bytes per 8 channels), so the network's input cast/permute pass
// disappears.  Values are exactly 0.0 / 1.0 in every format.
enum : int { FEAT_F32_NCHW = 0, FEAT_F16_NHWC = 1, FEAT_BF16_NHWC = 2 };

// Shared -> global bulk copy (TMA engine, `cp.async.bulk`): one thread hands the whole staged tile
// to the copy engine instead of every thread issuing stores.  `bytes` a multiple of 16, both
// addresses 16-byte aligned.
__device__ __forceinline__ void async_proxy_fence() {
#if !defined(ELFB200_SIMT_EMU)
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#endif
}
__device__ __forceinline__ void bulk_store_s2g(void* gdst, const void* ssrc, uint32_t bytes) {
#if defined(ELFB200_SIMT_EMU)
  memcpy(gdst, ssrc, bytes);
#else
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(ssrc);
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(s), "r"(bytes)
               : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // the CTA may retire once smem was read
#endif
}

// Flush a staged tile: every thread has written its part of `ssrc` (generic-proxy stores).
//   tma != 0: fence the writes towards the async proxy, barrier, thread 0 issues ONE bulk store;
//   tma == 0: barrier, then coalesced 16-byte vector stores by all threads.
__device__ __forceinline__ void flush_tile(void* gdst, const void* ssrc, uint32_t bytes, int tma) {
  if (tma) {
    async_proxy_fence();
    __syncthreads();
    if (threadIdx.x == 0) bulk_store_s2g(gdst, ssrc, bytes);
  } else {
    __syncthreads();
    const uint4* s4 = reinterpret_cast<const uint4*>(ssrc);
    uint4* g4 = reinterpret_cast<uint4*>(gdst);
    for (uint32_t i = threadIdx.x; i < bytes / 16; i += blockDim.x) g4[i] = s4[i];
  }
}

// Dynamic shared memory of the feature kernels: the staging tile of the 16-bit NHWC formats (the
// float32 format stores straight from registers).  The SIMT emulator has no dynamic smem: a static
// buffer of the largest tile stands in.
constexpr int FEAT_CPAD_MAX = 32;
#if defined(ELFB200_SIMT_EMU)
#define ELFB200_FEAT_SMEM(N) __align__(16) __shared__ unsigned char feat_smem[Geo<N>::P * FEAT_CPAD_MAX * 2]
#else
#define ELFB200_FEAT_SMEM(N) extern __shared__ __align__(16) unsigned char feat_smem[]
#endif

// bits [lo, lo+32) of the index range [a, b) as a word
__device__ __forceinline__ uint32_t range_bits(int lo, int a, int b) {
  const int s = max(a, lo) - lo, e = min(b, lo + 32) - lo;
  if (e <= s) return 0u;
  return ((e - s) >= 32 ? 0xFFFFFFFFu : ((1u << (e - s)) - 1u)) << s;
}

// One CTA of a feature kernel = one position.  `gather(slot, rows, hn, next, d4)` is called by ALL
// threads of the CTA and fills rows[t][y] (t < 8 history positions, newest first) for output `slot`.
//
// BoardFeature::extractAGZ (board_feature.cc:247-290) in three bit-level steps instead of one float
// at a time:
//  1. the 16 stone planes as TRANSFORMED bit rows T[plane][tx] (bit ty = output cell (tx,ty)): under
//     the D4 code an output row is a board row or a board column, read forwards or backwards
//     (InvTransform, board_feature.h:115-130, decomposed into {transposed, reversed index, reversed
//     bits}; the tables are checked against d4_inverse by brute force in tests/test_feature_tables.py);
//  2. float32 NCHW: the whole position as ONE flat bit string FW (18*N*N bits, planes 16/17 constant);
//     16-bit NHWC: per cell the 18 bits across planes;
//  3. float32: every thread expands 4 consecutive bits into a float4 -- fully coalesced 16-byte
//     stores, no staging (a position is 25,992 B: an odd slot starts 8 bytes off a 16-byte boundary,
//     so its first two floats go out as one 8-byte store and the groups shift by two bits);
//     16-bit NHWC: the cells are staged in shared memory and leave as one bulk (TMA) store.
template <int N, class Gather>
__device__ __forceinline__ void features_cta(Gather gather, int n_pos, void* __restrict__ out, int fmt, int cpad,
                                             int tma) {
  constexpr int P = Geo<N>::P, TOTAL = 18 * P, NW = (TOTAL + 31) / 32;
  ELFB200_FEAT_SMEM(N);
  __shared__ uint64_t rows[8][N];
  __shared__ uint32_t T[16][N];
  __shared__ uint32_t FW[NW + 1];
  __shared__ float4 LUT[16];  // 4 bits -> 4 floats
  const int slot = blockIdx.x;
  if (slot >= n_pos) return;
  if (threadIdx.x < 16)
    LUT[threadIdx.x] = make_float4((threadIdx.x & 1) ? 1.f : 0.f, (threadIdx.x & 2) ? 1.f : 0.f,
                                   (threadIdx.x & 4) ? 1.f : 0.f, (threadIdx.x & 8) ? 1.f : 0.f);
  int hn, next, d4;
  gather(slot, rows, hn, next, d4);
  __syncthreads();
  const bool bf = next == S_BLACK;  // even planes = side to move (board_feature.cc:268-281)
  if (fmt != FEAT_F32_NCHW) {
    // 16-bit channels-last: per output cell the 18 plane bits, then 8 channels at a time through a table.
    // Stones are sparse: every (plane, board row) scatters its stones into C[cell] (bit = plane) instead of
    // every cell gathering 16 planes.
    __shared__ uint32_t C[P];
    __shared__ uint4 LUT8[256];  // 8 plane bits -> 8 halves
    const uint32_t one = fmt == FEAT_F16_NHWC ? 0x3C00u : 0x3F80u;
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
      uint4 v;
      v.x = ((i & 1) ? one : 0u) | ((i & 2) ? one << 16 : 0u);
      v.y = ((i & 4) ? one : 0u) | ((i & 8) ? one << 16 : 0u);
      v.z = ((i & 16) ? one : 0u) | ((i & 32) ? one << 16 : 0u);
      v.w = ((i & 64) ? one : 0u) | ((i & 128) ? one << 16 : 0u);
      LUT8[i] = v;
    }
    for (int i = threadIdx.x; i < P; i += blockDim.x) C[i] = bf ? (1u << 16) : (1u << 17);
    __syncthreads();
    for (int item = threadIdx.x; item < 16 * N; item += blockDim.x) {
      const int pl = item / N, y = item - pl * N, t = pl >> 1;
      if (t < hn) {
        const bool want_black = ((pl & 1) == 0) == bf;
        const uint64_t r = rows[t][y];
        uint32_t word = (want_black ? (uint32_t)r : (uint32_t)(r >> 32)) & Geo<N>::ROWMASK;
        while (word) {
          const int x = __ffs(word) - 1;
          word &= word - 1;
          int ta, tb;  // Transform (board -> output cell): rotate, then flip (board_feature.h:97-113)
          switch (d4 & 3) {
            case 1: ta = y; tb = N - 1 - x; break;
            case 2: ta = N - 1 - x; tb = N - 1 - y; break;
            case 3: ta = N - 1 - y; tb = x; break;
            default: ta = x; tb = y; break;
          }
          atomicOr(&C[(d4 & 4) ? tb * N + ta : ta * N + tb], 1u << pl);
        }
      }
    }
    __syncthreads();
    uint16_t* gdst = reinterpret_cast<uint16_t*>(out) + (size_t)slot * P * cpad;
    if (!tma) {
      // direct: the position as a flat array of 16-byte pieces (cpad/8 per cell), one piece per thread and
      // iteration -- fully coalesced STG.E.128, no staging
      const int per = cpad / 8;
      uint4* g4 = reinterpret_cast<uint4*>(gdst);
      for (int j = threadIdx.x; j < P * per; j += blockDim.x) {
        const int cell = j / per, k = j - cell * per;
        g4[j] = k < 3 ? LUT8[(C[cell] >> (8 * k)) & 255u] : make_uint4(0u, 0u, 0u, 0u);
      }
    } else {
      // staged: the cells go to shared memory and leave as ONE bulk (TMA) store
      uint16_t* buf = reinterpret_cast<uint16_t*>(feat_smem);
      for (int cell = threadIdx.x; cell < P; cell += blockDim.x) {
        const uint32_t bits = C[cell];
        uint4* dst = reinterpret_cast<uint4*>(buf + (size_t)cell * cpad);
        dst[0] = LUT8[bits & 255u];
        dst[1] = LUT8[(bits >> 8) & 255u];
        dst[2] = LUT8[(bits >> 16) & 255u];
        for (int k = 3; k < cpad / 8; ++k) dst[k] = make_uint4(0u, 0u, 0u, 0u);
      }
      flush_tile(gdst, buf, (uint32_t)(P * cpad * 2), 1);
    }
    return;
  }
  const bool transposed = (0xA5u >> d4) & 1u, rev_idx = (0x6Cu >> d4) & 1u, rev_bits = (0xC6u >> d4) & 1u;
  if (!transposed) {
    // output row tx is board row src, read forwards or backwards: one word per (plane, row)
    for (int item = threadIdx.x; item < 16 * N; item += blockDim.x) {
      const int pl = item / N, tx = item - pl * N, t = pl >> 1;
      uint32_t o = 0;
      if (t < hn) {
        const bool want_black = ((pl & 1) == 0) == bf;
        const uint64_t r = rows[t][rev_idx ? N - 1 - tx : tx];
        o = (want_black ? (uint32_t)r : (uint32_t)(r >> 32)) & Geo<N>::ROWMASK;
        if (rev_bits) o = __brev(o) >> (32 - N);
      }
      T[pl][tx] = o;
    }
  } else {
    // output row tx is a board COLUMN: every (plane, board row y) scatters its (few) stones, stone
    // (x, y) becomes bit ty of T[plane][tx] with tx = x or N-1-x and ty = y or N-1-y
    for (int item = threadIdx.x; item < 16 * N; item += blockDim.x) (&T[0][0])[item] = 0u;
    __syncthreads();
    for (int item = threadIdx.x; item < 16 * N; item += blockDim.x) {
      const int pl = item / N, y = item - pl * N, t = pl >> 1;
      if (t < hn) {
        const bool want_black = ((pl & 1) == 0) == bf;
        const uint64_t r = rows[t][y];
        uint32_t word = (want_black ? (uint32_t)r : (uint32_t)(r >> 32)) & Geo<N>::ROWMASK;
        const uint32_t bit = 1u << (rev_bits ? N - 1 - y : y);
        while (word) {
          const int x = __ffs(word) - 1;
          word &= word - 1;
          atomicOr(&T[pl][rev_idx ? N - 1 - x : x], bit);
        }
      }
    }
  }
  __syncthreads();
  if (fmt == FEAT_F32_NCHW) {
    for (int j = threadIdx.x; j <= NW; j += blockDim.x) {
      const int lo = 32 * j;
      uint32_t w = 0;
      if (lo < 16 * P) {  // stitch the bit rows that overlap this word
        int pl = lo / P;
        const int c = lo - pl * P;
        int tx = c / N, ty = c - tx * N, pos = 0;
        while (pos < 32 && pl < 16) {
          w |= (T[pl][tx] >> ty) << pos;  // N - ty valid bits, zeros above
          pos += N - ty;
          ty = 0;
          if (++tx == N) {
            tx = 0;
            ++pl;
          }
        }
      }
      w |= range_bits(lo, 16 * P, 17 * P) & (bf ? 0xFFFFFFFFu : 0u);  // plane 16: black to move
      w |= range_bits(lo, 17 * P, 18 * P) & (bf ? 0u : 0xFFFFFFFFu);  // plane 17: white to move
      FW[j] = w;
    }
    __syncthreads();
    float* dst = reinterpret_cast<float*>(out) + (size_t)slot * TOTAL;
    const int h = (reinterpret_cast<uintptr_t>(dst) & 15) ? 2 : 0;  // dst is at least 8-byte aligned
    constexpr int NQ = (TOTAL - 2) / 4;  // float4 groups (TOTAL = 4*NQ + 2 for both board sizes)
    static_assert(TOTAL == 4 * NQ + 2, "a position is a whole number of float4 plus one float2");
    for (int q = threadIdx.x; q < NQ; q += blockDim.x) {
      const int b0 = h + 4 * q;
      const uint32_t w = __funnelshift_r(FW[b0 >> 5], FW[(b0 >> 5) + 1], b0 & 31);
      *reinterpret_cast<float4*>(dst + b0) = LUT[w & 15u];
    }
    if (threadIdx.x == 0) {  // the float2 that does not fit the float4 grid: first two floats or last two
      const int b0 = h ? 0 : TOTAL - 2;
      const uint32_t w = FW[b0 >> 5] >> (b0 & 31);
      *reinterpret_cast<float2*>(dst + b0) = make_float2((w & 1u) ? 1.0f : 0.0f, (w & 2u) ? 1.0f : 0.0f);
    }
  }
}

template <int N>
inline size_t feature_smem_bytes(int fmt, int cpad, int tma) {
  return (fmt == FEAT_F32_NCHW || !tma) ? (size_t)0 : (size_t)Geo<N>::P * cpad * 2;
}
constexpr int FEAT_THREADS = 128;

}  // namespace elfb200

// ---- host side ---------------------------------------------------------------------------------
int elfb200_fail(int code, const char* fmt, ...);  // records the message for elfb200_last_error()

#define CK(call)                                                                                  \
  do {                                                                                            \
    cudaError_t e_ = (call);                                                                      \
    if (e_ != cudaSuccess)                                                                        \
      return elfb200_fail(ELFB200_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), \
                          __FILE__, __LINE__);                                                    \
  } while (0)

#define DISPATCH_N(ctx, expr19, expr9) \
  do {                                 \
    if ((ctx)->N == 19) {              \
      expr19;                          \
    } else {                           \
      expr9;                           \
    }                                  \
  } while (0)

struct elfb200_ctx {
  int N = 0, G = 0, device = 0;
  cudaStream_t stream = nullptr;
  elfb200::DevState st{};
  // scratch
  int32_t* d_actions = nullptr;
  uint8_t* d_ok = nullptr;
  uint8_t* d_bytes = nullptr;   // G * (P+1) export buffer
  int32_t* d_words = nullptr;   // G * 12 export buffer
  int32_t* d_d4 = nullptr;
  float* d_feat = nullptr;      // lazily allocated G*18*P floats
  float* d_exp_table = nullptr; // exp(-k/10), k = 0 .. 2*N*N (host libm, so the DarkForest history planes match bit for bit)
  int playout_layout = -1;      // k_playout: 0 = one board row per lane, 1 = two rows per lane (19x19, three games per warp),
                                // -1 = automatic: two rows per lane from 4096 19x19 games up (where it measures faster)
  int feat_tma = 0;             // 16-bit NHWC planes: 0 = direct coalesced 16-byte stores (measured faster), 1 = staged tile + one bulk (TMA) store
  // playout outputs
  uint64_t* d_po_sk = nullptr;
  uint64_t* d_po_chk = nullptr;
  uint64_t* d_po_hash = nullptr;
  int32_t* d_po_plies = nullptr;
  int32_t* d_po_score = nullptr;
  // pinned staging
  void* h_pin = nullptr;
  size_t h_pin_bytes = 0;
  // zero-copy window of the host-driven step API: actions int32[G] then accept flags uint8[G], pinned
  // and MAPPED into the device address space -- k_step reads the actions and writes the flags over
  // PCIe itself, so a GoState::forward for the whole batch is one launch and one wait, no copies
  void* h_map = nullptr;
  int32_t* d_map_actions = nullptr;
  uint8_t* d_map_ok = nullptr;
  unsigned* d_done = nullptr;   // CTAs of the running host-driven k_step that have finished
  size_t map_ok_off = 0, map_flag_off = 0;  // byte offsets of the accept flags / completion flag in the mapped window
  uint32_t step_seq = 0;        // sequence number the last CTA writes into the mapped completion flag
  int64_t launches = 0;
  // fork / join of elfb200_gather_games_dev with this context as the destination (cudaEventDisableTiming)
  cudaEvent_t ev_gather[2] = {nullptr, nullptr};
  // move lists of elfb200_replay (grown on demand)
  int16_t* d_replay = nullptr;
  size_t d_replay_bytes = 0;
  // Monte-Carlo ownership and final status (elfb200_ownership / elfb200_final_status), allocated on first use
  uint64_t* d_own_sk = nullptr;      // superko record of each game segment of k_ownership's resident grid
  size_t d_own_sk_bytes = 0;
  int32_t* d_own_counts = nullptr;   // G * 2 * N*N counts of the synchronous forms
  uint8_t* d_own_status = nullptr;   // G * N*N dead flags, then G * N*N territory
  uint64_t* d_own_hash = nullptr;    // per-playout final hash / plies of the synchronous form (grown on demand)
  int32_t* d_own_plies = nullptr;
  size_t d_own_trace = 0;            // playouts the two buffers above hold
};
