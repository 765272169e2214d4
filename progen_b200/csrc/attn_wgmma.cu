// Sliding-window causal attention (reference progen.py:88-102) on Hopper warpgroup MMAs, bf16 in / fp32 accumulate,
// dim_head 64, any window that is a multiple of 64.  Same buffer contract as the exact-fp32 attn_simt.cu.
//
// One warpgroup (128 threads) per CTA owns a 64-row tile (queries in the forward and dQ kernels, keys in the dK/dV
// kernel).  The streamed 64-row operand tiles arrive by TMA (128-byte swizzle) in a two-stage ring completed on mbarriers;
// one thread issues the copies.  Score-type products (Q K^T, dO V^T, and their transposes) are wgmma with both operands
// in shared memory; the products with probabilities (P V, dS K, P^T dO, dS^T Q) take P / dS straight from the
// accumulator registers as the wgmma A operand (register fragments of an m64n64 accumulator are the A fragments of the
// next m64nNk16 MMA).  Softmax is online in registers, in log2 units.  The reference's zero look-back window of window 0
// (quirk Q1: w keys with logit 0 and value 0 that are NOT masked) is folded in analytically: the running max starts at 0
// and the running denominator at w; those keys carry no gradient (K == 0, V == 0).
#include <cuda.h>
#include "common.cuh"
#include "tc_ptx.cuh"
#include "../../include/progen_b200.h"

namespace {

using namespace tc;

constexpr int DH = 64;
constexpr int TILE = 64;                   // rows of every tile; one tile = 64 x 128 B = 8 KiB
constexpr int TILE_BYTES = TILE * DH * 2;
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;
constexpr int SMEM_BYTES = 1024 /*align slack*/ + 2 * TILE_BYTES + 2 * 2 * TILE_BYTES + 64;

struct Dims {
  int n, w, h;
  const float* rot_sin;   // [n, 32]; when set, the backward kernels write gradients w.r.t. the UN-rotated q, k, v
  const float* rot_cos;
};

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// gradient of (x0 c - x1 s, x1 c + x0 s) w.r.t. (x0, x1): (d0 c + d1 s, d1 c - d0 s); pair index jj of position pos
__device__ __forceinline__ uint32_t unrotate_pack(const Dims& dm, int pos, int jj, float d0, float d1) {
  if (dm.rot_sin) {
    const float s = __ldg(dm.rot_sin + pos * (DH / 2) + jj), c = __ldg(dm.rot_cos + pos * (DH / 2) + jj);
    const float a = d0 * c + d1 * s, b = d1 * c - d0 * s;
    d0 = a; d1 = b;
  }
  return pack_bf16x2(d0, d1);
}
template <int R> __device__ __forceinline__ void zero(float (&a)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) a[i] = 0.f;
}
// m64n64 accumulator (d[4 j + e]) -> bf16 A fragments of the four k-steps of the next MMA
__device__ __forceinline__ void acc_to_a(uint32_t (&a)[4][4], const float (&s)[32]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int i = 0; i < 4; ++i) a[kk][i] = pack_bf16x2(s[8 * kk + 2 * i], s[8 * kk + 2 * i + 1]);
}
// acc[64 x 64] += A[64 x 64] * X^T, A and X both [64 rows x 64] K-major tiles in shared memory
__device__ __forceinline__ void issue_a_xt(float (&acc)[32], uint32_t a, uint32_t x) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) wgmma_m64n64k16_ss<0>(acc, make_smem_desc<false>(a + 32 * kk), make_smem_desc<false>(x + 32 * kk));
}
// acc[64 x 64] += P[64 x 64] * X, P in registers, X a [64 (contraction) x 64] tile: MN-major B
__device__ __forceinline__ void issue_p_x(float (&acc)[32], const uint32_t (&p)[4][4], uint32_t x) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) wgmma_m64n64k16_rs<1>(acc, p[kk], make_smem_desc<true>(x + 2048 * kk));
}
template <int R> __device__ __forceinline__ void mma_begin(float (&acc)[R]) {
  fence_regs(acc);
  wgmma_fence();
}
template <int R> __device__ __forceinline__ void mma_end(float (&acc)[R]) {
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(acc);
}

// shared-memory carve-up common to the three kernels: two fixed tiles, a two-stage ring of tile pairs, three barriers
struct Smem {
  uint32_t fixed0, fixed1, ring, bars;
  __device__ Smem(uint8_t* raw) {
    fixed0 = (smem_u32(raw) + 1023u) & ~1023u;
    fixed1 = fixed0 + TILE_BYTES;
    ring = fixed1 + TILE_BYTES;
    bars = ring + 4 * TILE_BYTES;
  }
  __device__ uint32_t a(int st) const { return ring + st * 2 * TILE_BYTES; }
  __device__ uint32_t b(int st) const { return a(st) + TILE_BYTES; }
  __device__ uint32_t fixed_bar() const { return bars; }
  __device__ uint32_t full(int st) const { return bars + 8 + 8 * st; }
};

__device__ __forceinline__ void init_bars(const Smem& sm) {
  if (threadIdx.x == 0) {
    mbar_init(sm.fixed_bar(), 1);
    mbar_init(sm.full(0), 1);
    mbar_init(sm.full(1), 1);
    fence_barrier_init();
  }
  __syncthreads();
}

// ================================================================================================ forward
__global__ void __launch_bounds__(128) attn_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tm_qkv, bf16* __restrict__ out,
                                                             float* __restrict__ lse, const Dims dm) {
  extern __shared__ uint8_t smem_raw[];
  const Smem sm(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int b = blockIdx.z, hh = blockIdx.y;
  const int q0 = blockIdx.x * TILE, win = q0 / dm.w, i0 = q0 % dm.w;
  const int I = dm.h * DH;
  const int row0 = b * dm.n;
  const int nprev = win > 0 ? dm.w / TILE : 0;
  const int ntiles = nprev + (i0 + TILE) / TILE;
  auto key_pos = [&](int kt) { return kt < nprev ? (win - 1) * dm.w + kt * TILE : win * dm.w + (kt - nprev) * TILE; };
  auto issue = [&](int kt, int st) {            // K and V tiles of key tile kt -> stage st
    mbar_expect_tx(sm.full(st), 2 * TILE_BYTES);
    tma_load_2d(sm.a(st), &tm_qkv, sm.full(st), I + hh * DH, row0 + key_pos(kt));
    tma_load_2d(sm.b(st), &tm_qkv, sm.full(st), 2 * I + hh * DH, row0 + key_pos(kt));
  };
  init_bars(sm);
  if (tid == 0) {
    prefetch_tensormap(&tm_qkv);
    mbar_expect_tx(sm.fixed_bar(), TILE_BYTES);
    tma_load_2d(sm.fixed0, &tm_qkv, sm.fixed_bar(), hh * DH, row0 + q0);
    for (int kt = 0; kt < 2 && kt < ntiles; ++kt) issue(kt, kt);
  }

  const float sc = 0.125f /* 1/sqrt(64), exact */ * LOG2E;           // scores are kept in log2 units
  float m_run[2], l_run[2];
  m_run[0] = m_run[1] = (win == 0) ? 0.f : -INFINITY;                // window 0: phantom keys, see the header
  l_run[0] = l_run[1] = (win == 0) ? (float)dm.w : 0.f;
  float o[32];
  zero(o);
  const int qi_lo = i0 + warp * 16;
  mbar_wait(sm.fixed_bar(), 0);

  for (int kt = 0; kt < ntiles; ++kt) {
    const int st = kt & 1;
    mbar_wait(sm.full(st), (kt >> 1) & 1);
    float s[32];
    zero(s);
    mma_begin(s);
    issue_a_xt(s, sm.fixed0, sm.a(st));
    mma_end(s);
    const int c0 = (kt - nprev) * TILE;               // in-window offset of the tile's first key (own window only)
    const bool need_mask = kt >= nprev && c0 + TILE - 1 > qi_lo;
    float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      float v = s[i] * sc;
      if (need_mask) {
        const int kj = c0 + 8 * (i >> 2) + 2 * t4 + (i & 1);
        const int qi = qi_lo + g + (((i >> 1) & 1) << 3);
        if (kj > qi) v = -INFINITY;
      }
      s[i] = v;
      tmax[(i >> 1) & 1] = fmaxf(tmax[(i >> 1) & 1], v);
    }
    float corr[2], rsum[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float mn = fmaxf(m_run[r], quad_max(tmax[r]));
      corr[r] = exp2f(m_run[r] - mn);                 // m_run = -inf only before the first tile: exp2(-inf) = 0
      m_run[r] = mn;
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float p = exp2f(s[i] - m_run[(i >> 1) & 1]);
      s[i] = p;
      rsum[(i >> 1) & 1] += p;
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * corr[r] + quad_sum(rsum[r]);
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] *= corr[(i >> 1) & 1];
    uint32_t pa[4][4];
    acc_to_a(pa, s);
    mma_begin(o);
    issue_p_x(o, pa, sm.b(st));
    mma_end(o);
    __syncthreads();                                  // every MMA of the warpgroup has read stage st
    if (tid == 0 && kt + 2 < ntiles) {
      fence_proxy_async();
      issue(kt + 2, st);
    }
  }
  // epilogue: O / l -> bf16 [T, I]; lse in natural-log units
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const long long t = (long long)row0 + q0 + warp * 16 + g + 8 * r;
    const float inv = 1.f / l_run[r];
    bf16* op = out + t * I + hh * DH + 2 * t4;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(op + 8 * j) = pack_bf16x2(o[4 * j + 2 * r] * inv, o[4 * j + 2 * r + 1] * inv);
    if (t4 == 0) lse[t * dm.h + hh] = m_run[r] * LN2 + logf(l_run[r]);
  }
}

// ================================================================================================ dQ (+ delta)
// dQ = scale * sum_tiles (P o (dO V^T - delta)) K,  P = exp(scale * Q K^T - lse),  delta = rowsum(dO o O)
__global__ void __launch_bounds__(128) attn_bwd_dq_wgmma_kernel(const __grid_constant__ CUtensorMap tm_qkv,
                                                                const __grid_constant__ CUtensorMap tm_do,
                                                                const bf16* __restrict__ out, const bf16* __restrict__ dout,
                                                                const float* __restrict__ lse, float* __restrict__ delta,
                                                                bf16* __restrict__ dqkv, const Dims dm) {
  extern __shared__ uint8_t smem_raw[];
  const Smem sm(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int b = blockIdx.z, hh = blockIdx.y;
  const int q0 = blockIdx.x * TILE, win = q0 / dm.w, i0 = q0 % dm.w;
  const int I = dm.h * DH;
  const long long ld = 3LL * I;
  const int row0 = b * dm.n;
  const int nprev = win > 0 ? dm.w / TILE : 0;        // phantom keys (win == 0) carry no gradient: K == 0
  const int ntiles = nprev + (i0 + TILE) / TILE;
  auto key_pos = [&](int kt) { return kt < nprev ? (win - 1) * dm.w + kt * TILE : win * dm.w + (kt - nprev) * TILE; };
  auto issue = [&](int kt, int st) {
    mbar_expect_tx(sm.full(st), 2 * TILE_BYTES);
    tma_load_2d(sm.a(st), &tm_qkv, sm.full(st), I + hh * DH, row0 + key_pos(kt));
    tma_load_2d(sm.b(st), &tm_qkv, sm.full(st), 2 * I + hh * DH, row0 + key_pos(kt));
  };
  init_bars(sm);
  if (tid == 0) {
    prefetch_tensormap(&tm_qkv);
    prefetch_tensormap(&tm_do);
    mbar_expect_tx(sm.fixed_bar(), 2 * TILE_BYTES);
    tma_load_2d(sm.fixed0, &tm_qkv, sm.fixed_bar(), hh * DH, row0 + q0);
    tma_load_2d(sm.fixed1, &tm_do, sm.fixed_bar(), hh * DH, row0 + q0);
    for (int kt = 0; kt < 2 && kt < ntiles; ++kt) issue(kt, kt);
  }

  const float scale = 0.125f /* 1/sqrt(64), exact */;
  const float sc = scale * LOG2E;
  float L2[2], Dl[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const long long t = (long long)row0 + q0 + warp * 16 + g + 8 * r;
    L2[r] = lse[t * dm.h + hh] * LOG2E;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t ov = *reinterpret_cast<const uint32_t*>(out + t * I + hh * DH + 8 * j + 2 * t4);
      const uint32_t dv = *reinterpret_cast<const uint32_t*>(dout + t * I + hh * DH + 8 * j + 2 * t4);
      const float2 fo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&ov));
      const float2 fd = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&dv));
      acc += fo.x * fd.x + fo.y * fd.y;
    }
    Dl[r] = quad_sum(acc);
    if (t4 == 0) delta[t * dm.h + hh] = Dl[r];        // published for the dK/dV kernel that follows on the stream
  }
  float dq[32];
  zero(dq);
  const int qi_lo = i0 + warp * 16;
  mbar_wait(sm.fixed_bar(), 0);

  for (int kt = 0; kt < ntiles; ++kt) {
    const int st = kt & 1;
    mbar_wait(sm.full(st), (kt >> 1) & 1);
    float s[32], dp[32];
    zero(s);
    zero(dp);
    fence_regs(dp);
    mma_begin(s);
    issue_a_xt(s, sm.fixed0, sm.a(st));               // S = Q K^T
    issue_a_xt(dp, sm.fixed1, sm.b(st));              // dP = dO V^T
    mma_end(s);
    fence_regs(dp);
    const int c0 = (kt - nprev) * TILE;
    const bool need_mask = kt >= nprev && c0 + TILE - 1 > qi_lo;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int r = (i >> 1) & 1;
      float p = exp2f(s[i] * sc - L2[r]);
      if (need_mask) {
        const int kj = c0 + 8 * (i >> 2) + 2 * t4 + (i & 1);
        const int qi = qi_lo + g + (r << 3);
        if (kj > qi) p = 0.f;
      }
      s[i] = p * (dp[i] - Dl[r]) * scale;             // dS
    }
    uint32_t dsa[4][4];
    acc_to_a(dsa, s);
    mma_begin(dq);
    issue_p_x(dq, dsa, sm.a(st));                     // dQ += dS K
    mma_end(dq);
    __syncthreads();
    if (tid == 0 && kt + 2 < ntiles) {
      fence_proxy_async();
      issue(kt + 2, st);
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int pos = q0 + warp * 16 + g + 8 * r;
    bf16* op = dqkv + ((long long)row0 + pos) * ld + hh * DH + 2 * t4;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(op + 8 * j) = unrotate_pack(dm, pos, 4 * j + t4, dq[4 * j + 2 * r], dq[4 * j + 2 * r + 1]);
  }
}

// ================================================================================================ dK, dV
// One CTA per 64-key tile; streams the 64-query tiles that can see it (own window from the diagonal on, then the next
// window; both end at seq_len).  Works on transposed scores: S^T = K Q^T so that keys are the accumulator rows.
__global__ void __launch_bounds__(128) attn_bwd_dkv_wgmma_kernel(const __grid_constant__ CUtensorMap tm_qkv,
                                                                 const __grid_constant__ CUtensorMap tm_do,
                                                                 const float* __restrict__ lse, const float* __restrict__ delta,
                                                                 bf16* __restrict__ dqkv, const Dims dm) {
  extern __shared__ uint8_t smem_raw[];
  const Smem sm(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int b = blockIdx.z, hh = blockIdx.y;
  const int k0 = blockIdx.x * TILE, win = k0 / dm.w, j0 = k0 % dm.w;
  const int I = dm.h * DH;
  const long long ld = 3LL * I;
  const int row0 = b * dm.n;
  const int nwin = (dm.n + dm.w - 1) / dm.w;          // the last window may be partial (a cut backward)
  // query tiles of the own window at or after the diagonal, below min(window end, n); then those of the next window,
  // below n.  At whole windows: (w - j0) / 64 and w / 64.
  const int own_end = min((win + 1) * dm.w, dm.n);
  const int nown = (own_end - k0) / TILE;
  const int nnext = (win + 1 < nwin) ? (min((win + 2) * dm.w, dm.n) - own_end) / TILE : 0;
  const int ntiles = nown + nnext;
  auto q_pos = [&](int qt) { return qt < nown ? win * dm.w + j0 + qt * TILE : (win + 1) * dm.w + (qt - nown) * TILE; };
  auto issue = [&](int qt, int st) {                  // Q and dO tiles of query tile qt -> stage st
    mbar_expect_tx(sm.full(st), 2 * TILE_BYTES);
    tma_load_2d(sm.a(st), &tm_qkv, sm.full(st), hh * DH, row0 + q_pos(qt));
    tma_load_2d(sm.b(st), &tm_do, sm.full(st), hh * DH, row0 + q_pos(qt));
  };
  init_bars(sm);
  if (tid == 0) {
    prefetch_tensormap(&tm_qkv);
    prefetch_tensormap(&tm_do);
    mbar_expect_tx(sm.fixed_bar(), 2 * TILE_BYTES);
    tma_load_2d(sm.fixed0, &tm_qkv, sm.fixed_bar(), I + hh * DH, row0 + k0);
    tma_load_2d(sm.fixed1, &tm_qkv, sm.fixed_bar(), 2 * I + hh * DH, row0 + k0);
    for (int qt = 0; qt < 2 && qt < ntiles; ++qt) issue(qt, qt);
  }

  const float scale = 0.125f /* 1/sqrt(64), exact */;
  const float sc = scale * LOG2E;
  float dk[32], dv[32];
  zero(dk);
  zero(dv);
  const int kj_lo = j0 + warp * 16;                   // in-window offset of this warp's first key row
  mbar_wait(sm.fixed_bar(), 0);

  for (int qt = 0; qt < ntiles; ++qt) {
    const int st = qt & 1;
    const int qp = q_pos(qt);
    // lse (log2 units) and delta of the 16 query columns this thread touches
    float Lq[16], Dq[16];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const long long t = (long long)row0 + qp + 8 * j + 2 * t4 + c;
        Lq[2 * j + c] = __ldg(lse + t * dm.h + hh) * LOG2E;
        Dq[2 * j + c] = __ldg(delta + t * dm.h + hh);
      }
    mbar_wait(sm.full(st), (qt >> 1) & 1);
    float s[32], dp[32];
    zero(s);
    zero(dp);
    fence_regs(dp);
    mma_begin(s);
    issue_a_xt(s, sm.fixed0, sm.a(st));               // S^T[key][query] = K Q^T
    issue_a_xt(dp, sm.fixed1, sm.b(st));              // dP^T = V dO^T
    mma_end(s);
    fence_regs(dp);
    const bool own = qt < nown;
    const int c0 = j0 + qt * TILE;                    // in-window offset of the tile's first query (own window only)
    const bool need_mask = own && c0 < kj_lo + 15;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int col = 8 * (i >> 2) + 2 * t4 + (i & 1);   // query index inside the tile
      const int ci = 2 * (i >> 2) + (i & 1);
      float p = exp2f(s[i] * sc - Lq[ci]);
      if (need_mask) {
        const int qi = c0 + col;
        const int kj = kj_lo + g + (((i >> 1) & 1) << 3);
        if (kj > qi) p = 0.f;
      }
      dp[i] = p * (dp[i] - Dq[ci]) * scale;           // dS^T
      s[i] = p;                                       // P^T
    }
    uint32_t pa[4][4], dsa[4][4];
    acc_to_a(pa, s);
    acc_to_a(dsa, dp);
    fence_regs(dk);
    mma_begin(dv);
    issue_p_x(dv, pa, sm.b(st));                      // dV += P^T dO
    issue_p_x(dk, dsa, sm.a(st));                     // dK += dS^T Q
    mma_end(dv);
    fence_regs(dk);
    __syncthreads();
    if (tid == 0 && qt + 2 < ntiles) {
      fence_proxy_async();
      issue(qt + 2, st);
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int pos = k0 + warp * 16 + g + 8 * r;
    bf16* pk = dqkv + ((long long)row0 + pos) * ld + I + hh * DH + 2 * t4;
    bf16* pv = pk + I;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<uint32_t*>(pk + 8 * j) = unrotate_pack(dm, pos, 4 * j + t4, dk[4 * j + 2 * r], dk[4 * j + 2 * r + 1]);
      *reinterpret_cast<uint32_t*>(pv + 8 * j) = unrotate_pack(dm, pos, 4 * j + t4, dv[4 * j + 2 * r], dv[4 * j + 2 * r + 1]);
    }
  }
}

template <typename K> int prepare(K kern) {
  static bool done = false;            // one flag per kernel (template instance per kernel type)
  if (!done) {
    PG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    done = true;
  }
  return PROGEN_OK;
}

// full_windows: seq_len must be whole windows (progen_local_attn_bwd_tc keeps that contract).  The forward and the cut
// backward only need whole 64-row tiles: a query tile of a partial last window reads the previous window and its own
// keys up to the diagonal, the same key tiles it reads at full length, and a key tile streams the query tiles below
// seq_len only, so no row at or beyond seq_len is touched.
int check_dims(const void* qkv, int B, int seq_len, int window, int heads, int dim_head, bool full_windows) {
  PG_CHECK_ARG(qkv != nullptr && B > 0 && heads > 0 && dim_head == DH && window % TILE == 0 && seq_len > 0 &&
               seq_len % (full_windows ? window : TILE) == 0);
  PG_CHECK_ARG((long long)B * seq_len < (1ll << 31));
  return PROGEN_OK;
}

// the one launcher of both backward entry points (they differ in their host check only)
int bwd_tc(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv, float* delta,
           const float* rot_sin, const float* rot_cos, int B, int seq_len, int window, int heads, cudaStream_t s) {
  int rc;
  const int I = heads * DH;
  const uint64_t T = (uint64_t)B * seq_len;
  CUtensorMap tq, tdo;
  if ((rc = pg_tensor_map_2d_bf16(qkv, 3ull * I, T, 3ull * I, DH, TILE, &tq))) return rc;
  if ((rc = pg_tensor_map_2d_bf16(dout, (uint64_t)I, T, (uint64_t)I, DH, TILE, &tdo))) return rc;
  if ((rc = prepare(attn_bwd_dq_wgmma_kernel))) return rc;
  if ((rc = prepare(attn_bwd_dkv_wgmma_kernel))) return rc;
  const Dims dm{seq_len, window, heads, rot_sin, rot_cos};
  const dim3 grid(seq_len / TILE, heads, B);
  // the dQ kernel also produces delta for the dK/dV kernel that follows it on the same stream
  attn_bwd_dq_wgmma_kernel<<<grid, 128, SMEM_BYTES, s>>>(tq, tdo, (const bf16*)out, (const bf16*)dout, lse, delta, (bf16*)dqkv, dm);
  PG_LAUNCH_CHECK();
  attn_bwd_dkv_wgmma_kernel<<<grid, 128, SMEM_BYTES, s>>>(tq, tdo, lse, delta, (bf16*)dqkv, dm);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

}  // namespace

extern "C" {

// bf16, dim_head == 64, window % 64 == 0 (every tile lies inside one window), seq_len % 64 == 0: the last window may be
// partial (a forward cut short of the model's sequence length computes the first seq_len rows of the full one, bitwise).
// qkv [T, 3*heads*64] (rotated), out [T, heads*64], lse [T, heads].
int progen_local_attn_fwd_tc(const void* qkv, void* out, float* lse, int B, int seq_len, int window, int heads, int dim_head,
                             void* stream) {
  int rc = check_dims(qkv, B, seq_len, window, heads, dim_head, false);
  if (rc) return rc;
  const int I = heads * DH;
  const uint64_t T = (uint64_t)B * seq_len;
  CUtensorMap tm;
  if ((rc = pg_tensor_map_2d_bf16(qkv, 3ull * I, T, 3ull * I, DH, TILE, &tm))) return rc;
  if ((rc = prepare(attn_fwd_wgmma_kernel))) return rc;
  const Dims dm{seq_len, window, heads, nullptr, nullptr};
  attn_fwd_wgmma_kernel<<<dim3(seq_len / TILE, heads, B), 128, SMEM_BYTES, (cudaStream_t)stream>>>(tm, (bf16*)out, lse, dm);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

// dqkv [T, 3*heads*64] receives dq | dk | dv; delta [T, heads] is workspace.  With rot_sin/rot_cos ([seq_len, 32] tables)
// the rotary backward is fused and the gradients are w.r.t. the projections BEFORE rotary.
int progen_local_attn_bwd_tc(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv, float* delta,
                             const float* rot_sin, const float* rot_cos, int B, int seq_len, int window, int heads, int dim_head,
                             void* stream) {
  const int rc = check_dims(qkv, B, seq_len, window, heads, dim_head, true);
  return rc ? rc : bwd_tc(qkv, out, dout, lse, dqkv, delta, rot_sin, rot_cos, B, seq_len, window, heads, (cudaStream_t)stream);
}

// the same with a partial last window: seq_len % 64 == 0 (the forward's rule)
int progen_local_attn_bwd_cut_tc(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                                 float* delta, const float* rot_sin, const float* rot_cos, int B, int seq_len, int window,
                                 int heads, int dim_head, void* stream) {
  const int rc = check_dims(qkv, B, seq_len, window, heads, dim_head, false);
  return rc ? rc : bwd_tc(qkv, out, dout, lse, dqkv, delta, rot_sin, rot_cos, B, seq_len, window, heads, (cudaStream_t)stream);
}

}  // extern "C"
