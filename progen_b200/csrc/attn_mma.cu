// Sliding-window causal attention (reference progen.py:88-102) on tensor cores, bf16 in / fp32 accumulate, dim_head 64.
//
// Flash-style: scores never leave the SM.  Per (batch, head, query tile) the CTA streams 64-key K/V tiles (previous
// window, then the causal part of the own window) through double-buffered, XOR-swizzled shared memory (cp.async),
// QK^T and PV run on mma.sync.m16n8k16 with ldmatrix-fed fragments, softmax is online in registers (exp2, quad
// shuffles).  The reference's zero look-back window of window 0 (quirk Q1: w keys with logit 0 and value 0 that are NOT
// masked) is folded in analytically: the running max starts at 0 and the running denominator at w.
//
// Backward is two kernels without atomics: dQ (same tiling as forward) and dK/dV (one CTA per key tile, streaming the
// query tiles that can see it); both recompute P from the saved log-sum-exp.
//
// The mixed-precision engine runs this version for windows that are multiples of 64 but not of 128; attn_wgmma.cu
// (wgmma, TMA-fed tiles) covers the others.
#include <stdlib.h>
#include "common.cuh"
#include "../../include/progen_b200.h"

namespace {

constexpr int DH = 64;
constexpr int BKV = 64;
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// [rows x 64] bf16 tile, 128 B per row, 16-byte chunk c of row r stored at chunk (c ^ (r & 7))
__device__ __forceinline__ uint32_t tile_addr(uint32_t base, int r, int c16) { return base + r * 128 + ((c16 ^ (r & 7)) << 4); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int ROWS, int THREADS>
__device__ __forceinline__ void load_tile_async(uint32_t base, const bf16* g, long long ld, int tid) {
#pragma unroll
  for (int i = tid; i < ROWS * 8; i += THREADS) {
    const int r = i >> 3, c = i & 7;
    cp_async16(tile_addr(base, r, c), g + (long long)r * ld + c * 8);
  }
}

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// A fragments (16 rows starting at r0, all 4 k-steps of a 64-wide tile)
__device__ __forceinline__ void load_a_frags(uint32_t (&a)[4][4], uint32_t base, int r0, int lane) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) ldsm_x4(a[kk], tile_addr(base, r0 + (lane & 15), 2 * kk + (lane >> 4)));
}
// acc[16 x 64] += A[16 x 64] * X^T where X is a [64 x 64] tile (rows index the output columns): B(k, n) = X[n][k]
__device__ __forceinline__ void mma_a_xt(float (&acc)[8][4], const uint32_t (&a)[4][4], uint32_t xbase, int lane) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      uint32_t b[4];
      ldsm_x4(b, tile_addr(xbase, 16 * p + (lane & 7) + ((lane >> 4) << 3), 2 * kk + ((lane >> 3) & 1)));
      mma16816(acc[2 * p], a[kk], b[0], b[1]);
      mma16816(acc[2 * p + 1], a[kk], b[2], b[3]);
    }
  }
}
// acc[16 x 64] += P[16 x 64] * X where X is a [64 x 64] tile (rows index the contraction): B(k, n) = X[k][n]
__device__ __forceinline__ void mma_p_x(float (&acc)[8][4], const uint32_t (&pa)[4][4], uint32_t xbase, int lane) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      uint32_t b[4];
      ldsm_x4_trans(b, tile_addr(xbase, 16 * kk + (lane & 7) + (((lane >> 3) & 1) << 3), 2 * p + (lane >> 4)));
      mma16816(acc[2 * p], pa[kk], b[0], b[1]);
      mma16816(acc[2 * p + 1], pa[kk], b[2], b[3]);
    }
  }
}
// accumulator tile (fp32, C layout) -> bf16 A fragments for the next matmul
__device__ __forceinline__ void acc_to_a(uint32_t (&pa)[4][4], const float (&s)[8][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    pa[kk][0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
    pa[kk][1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
    pa[kk][2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
    pa[kk][3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
  }
}
__device__ __forceinline__ void zero_acc(float (&a)[8][4]) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) a[i][j] = 0.f;
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

struct Dims {
  int n, w, h;
  const float* rot_sin;   // [n, 32]; when set, the backward kernels write gradients w.r.t. the UN-rotated q, k, v
  const float* rot_cos;   //          (backward of apply_rotary_pos_emb, progen.py:36-41, fused into the epilogue)
};

// gradient of (x0 c - x1 s, x1 c + x0 s) w.r.t. (x0, x1): (d0 c + d1 s, d1 c - d0 s); pair index jj of position pos
__device__ __forceinline__ uint32_t unrotate_pack(const Dims& dm, int pos, int jj, float d0, float d1) {
  if (dm.rot_sin) {
    const float s = __ldg(dm.rot_sin + pos * (DH / 2) + jj), c = __ldg(dm.rot_cos + pos * (DH / 2) + jj);
    const float a = d0 * c + d1 * s, b = d1 * c - d0 * s;
    d0 = a; d1 = b;
  }
  return pack_bf16x2(d0, d1);
}

// ================================================================================================ forward
template <int BQ>
__global__ void __launch_bounds__(BQ * 2, 256 / BQ) attn_fwd_mma_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ out,
                                                              float* __restrict__ lse, const Dims dm) {
  constexpr int THREADS = BQ * 2;
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sK = sQ + BQ * 128;
  const uint32_t sV = sK + 2 * BKV * 128;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int b = blockIdx.z, hh = blockIdx.y;
  const int q0 = blockIdx.x * BQ, win = q0 / dm.w, i0 = q0 % dm.w;
  const int I = dm.h * DH;
  const long long ld = 3LL * I;
  const long long seq_row0 = (long long)b * dm.n;
  const bf16* Qg = qkv + (seq_row0 + q0) * ld + hh * DH;
  const bf16* Kg = qkv + seq_row0 * ld + I + hh * DH;
  const bf16* Vg = Kg + I;
  const int nprev = win > 0 ? dm.w / BKV : 0;
  const int ncur = (i0 + BQ) / BKV;
  const int ntiles = nprev + ncur;
  auto key_pos = [&](int kt) { return kt < nprev ? (win - 1) * dm.w + kt * BKV : win * dm.w + (kt - nprev) * BKV; };

  load_tile_async<BQ, THREADS>(sQ, Qg, ld, tid);
  load_tile_async<BKV, THREADS>(sK, Kg + (long long)key_pos(0) * ld, ld, tid);
  load_tile_async<BKV, THREADS>(sV, Vg + (long long)key_pos(0) * ld, ld, tid);
  cp_async_commit();

  const float sc = 0.125f /* 1/sqrt(64), exact */ * LOG2E;           // scores are kept in log2 units
  float m_run[2], l_run[2];
  // window 0: w phantom keys with logit 0 / value 0 (quirk Q1) -> max 0, denominator w, numerator 0
  m_run[0] = m_run[1] = (win == 0) ? 0.f : -INFINITY;
  l_run[0] = l_run[1] = (win == 0) ? (float)dm.w : 0.f;
  float o[8][4];
  zero_acc(o);
  uint32_t qa[4][4];
  const int qi_lo = i0 + warp * 16;                     // in-window offset of this warp's first query row

  for (int kt = 0; kt < ntiles; ++kt) {
    const int st = kt & 1;
    if (kt + 1 < ntiles) {
      load_tile_async<BKV, THREADS>(sK + (st ^ 1) * BKV * 128, Kg + (long long)key_pos(kt + 1) * ld, ld, tid);
      load_tile_async<BKV, THREADS>(sV + (st ^ 1) * BKV * 128, Vg + (long long)key_pos(kt + 1) * ld, ld, tid);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (kt == 0) load_a_frags(qa, sQ, warp * 16, lane);
    const int c0 = (kt - nprev) * BKV;                  // in-window offset of the tile's first key (own window only)
    const bool own = kt >= nprev;
    if (!(own && c0 > qi_lo + 15)) {                    // warp-uniform: tile entirely above the diagonal -> skip
      float s[8][4];
      zero_acc(s);
      mma_a_xt(s, qa, sK + st * BKV * 128, lane);
      const bool need_mask = own && (c0 + BKV - 1 > qi_lo);
      float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float v = s[j][e] * sc;
          if (need_mask) {
            const int kj = c0 + 8 * j + 2 * t4 + (e & 1);
            const int qi = qi_lo + g + ((e >> 1) << 3);
            if (kj > qi) v = -INFINITY;
          }
          s[j][e] = v;
          tmax[e >> 1] = fmaxf(tmax[e >> 1], v);
        }
      }
      float corr[2], rsum[2] = {0.f, 0.f};
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float mn = fmaxf(m_run[r], quad_max(tmax[r]));
        corr[r] = exp2f(m_run[r] - mn);                 // m_run = -inf only before the first tile: exp2(-inf) = 0
        m_run[r] = mn;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float p = exp2f(s[j][e] - m_run[e >> 1]);
          s[j][e] = p;
          rsum[e >> 1] += p;
        }
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * corr[r] + quad_sum(rsum[r]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j][0] *= corr[0]; o[j][1] *= corr[0]; o[j][2] *= corr[1]; o[j][3] *= corr[1];
      }
      uint32_t pa[4][4];
      acc_to_a(pa, s);
      mma_p_x(o, pa, sV + st * BKV * 128, lane);
    }
    __syncthreads();
  }
  // epilogue: O / l -> bf16 [T, I]; lse in natural-log units
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = warp * 16 + g + 8 * r;
    const long long t = seq_row0 + q0 + row;
    const float inv = 1.f / l_run[r];
    bf16* op = out + t * I + hh * DH + 2 * t4;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(op + 8 * j) = pack_bf16x2(o[j][2 * r] * inv, o[j][2 * r + 1] * inv);
    if (t4 == 0) lse[t * dm.h + hh] = m_run[r] * LN2 + logf(l_run[r]);
  }
}

// ================================================================================================ delta = rowsum(dO * O)
__global__ void attn_delta_kernel(const bf16* __restrict__ out, const bf16* __restrict__ dout, float* __restrict__ delta,
                                  long long rows /* T*h */) {
  const int lane = threadIdx.x & 31;
  const long long r = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  if (r >= rows) return;
  const uint32_t a = reinterpret_cast<const uint32_t*>(out + r * DH)[lane];
  const uint32_t b = reinterpret_cast<const uint32_t*>(dout + r * DH)[lane];
  const float2 fa = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&a));
  const float2 fb = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&b));
  const float s = warp_sum(fa.x * fb.x + fa.y * fb.y);
  if (lane == 0) delta[r] = s;
}

// ================================================================================================ dQ
// dQ = scale * sum_tiles (P o (dO V^T - delta)) K,  P = exp(scale * Q K^T - lse)
template <int BQ>
__global__ void __launch_bounds__(BQ * 2) attn_bwd_dq_mma_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ out,
                                                                 const bf16* __restrict__ dout, const float* __restrict__ lse,
                                                                 float* __restrict__ delta, bf16* __restrict__ dqkv,
                                                                 const Dims dm) {
  constexpr int THREADS = BQ * 2;
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sdO = sQ + BQ * 128;
  const uint32_t sK = sdO + BQ * 128;
  const uint32_t sV = sK + 2 * BKV * 128;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int b = blockIdx.z, hh = blockIdx.y;
  const int q0 = blockIdx.x * BQ, win = q0 / dm.w, i0 = q0 % dm.w;
  const int I = dm.h * DH;
  const long long ld = 3LL * I;
  const long long seq_row0 = (long long)b * dm.n;
  const bf16* Qg = qkv + (seq_row0 + q0) * ld + hh * DH;
  const bf16* dOg = dout + (seq_row0 + q0) * I + hh * DH;
  const bf16* Kg = qkv + seq_row0 * ld + I + hh * DH;
  const bf16* Vg = Kg + I;
  const int nprev = win > 0 ? dm.w / BKV : 0;           // phantom keys (win == 0) carry no gradient: K == 0
  const int ncur = (i0 + BQ) / BKV;
  const int ntiles = nprev + ncur;
  auto key_pos = [&](int kt) { return kt < nprev ? (win - 1) * dm.w + kt * BKV : win * dm.w + (kt - nprev) * BKV; };

  load_tile_async<BQ, THREADS>(sQ, Qg, ld, tid);
  load_tile_async<BQ, THREADS>(sdO, dOg, I, tid);
  load_tile_async<BKV, THREADS>(sK, Kg + (long long)key_pos(0) * ld, ld, tid);
  load_tile_async<BKV, THREADS>(sV, Vg + (long long)key_pos(0) * ld, ld, tid);
  cp_async_commit();

  const float scale = 0.125f /* 1/sqrt(64), exact */;
  const float sc = scale * LOG2E;
  float L2[2], Dl[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const long long t = seq_row0 + q0 + warp * 16 + g + 8 * r;
    L2[r] = lse[t * dm.h + hh] * LOG2E;
    Dl[r] = 0.f;
  }
  float dq[8][4];
  zero_acc(dq);
  uint32_t qa[4][4], doa[4][4];
  const int qi_lo = i0 + warp * 16;

  for (int kt = 0; kt < ntiles; ++kt) {
    const int st = kt & 1;
    if (kt + 1 < ntiles) {
      load_tile_async<BKV, THREADS>(sK + (st ^ 1) * BKV * 128, Kg + (long long)key_pos(kt + 1) * ld, ld, tid);
      load_tile_async<BKV, THREADS>(sV + (st ^ 1) * BKV * 128, Vg + (long long)key_pos(kt + 1) * ld, ld, tid);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (kt == 0) {
      load_a_frags(qa, sQ, warp * 16, lane);
      load_a_frags(doa, sdO, warp * 16, lane);
      // delta = rowsum(dO o O), fused here (was a separate pass): this thread's dO fragment elements against the same
      // elements of O read straight from global; the quad completes the row.  Also published for the dK/dV kernel.
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const long long t = seq_row0 + q0 + warp * 16 + g + 8 * r;
            const uint32_t ov = *reinterpret_cast<const uint32_t*>(out + t * I + hh * DH + 16 * kk + 8 * hf + 2 * t4);
            const uint32_t dv = doa[kk][2 * hf + r];
            const float2 fo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&ov));
            const float2 fd = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&dv));
            Dl[r] += fo.x * fd.x + fo.y * fd.y;
          }
        }
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        Dl[r] = quad_sum(Dl[r]);
        if (t4 == 0) delta[(seq_row0 + q0 + warp * 16 + g + 8 * r) * dm.h + hh] = Dl[r];
      }
    }
    const int c0 = (kt - nprev) * BKV;
    const bool own = kt >= nprev;
    if (!(own && c0 > qi_lo + 15)) {
      float s[8][4], dp[8][4];
      zero_acc(s);
      zero_acc(dp);
      mma_a_xt(s, qa, sK + st * BKV * 128, lane);
      mma_a_xt(dp, doa, sV + st * BKV * 128, lane);
      const bool need_mask = own && (c0 + BKV - 1 > qi_lo);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int r = e >> 1;
          float p = exp2f(s[j][e] * sc - L2[r]);
          if (need_mask) {
            const int kj = c0 + 8 * j + 2 * t4 + (e & 1);
            const int qi = qi_lo + g + (r << 3);
            if (kj > qi) p = 0.f;
          }
          s[j][e] = p * (dp[j][e] - Dl[r]) * scale;     // dS
        }
      }
      uint32_t dsa[4][4];
      acc_to_a(dsa, s);
      mma_p_x(dq, dsa, sK + st * BKV * 128, lane);
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const long long t = seq_row0 + q0 + warp * 16 + g + 8 * r;
    bf16* op = dqkv + t * ld + hh * DH + 2 * t4;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(op + 8 * j) = unrotate_pack(dm, q0 + warp * 16 + g + 8 * r, 4 * j + t4, dq[j][2 * r], dq[j][2 * r + 1]);
  }
}

// ================================================================================================ dK, dV
// One CTA per BK-key tile; streams the 64-query tiles that can see it (own window from the diagonal on, then the whole
// next window).  Works on transposed scores: S^T = K Q^T so that keys are the accumulator rows.
template <int BK>
__global__ void __launch_bounds__(BK * 2) attn_bwd_dkv_mma_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ dout,
                                                                  const float* __restrict__ lse, const float* __restrict__ delta,
                                                                  bf16* __restrict__ dqkv, const Dims dm) {
  constexpr int THREADS = BK * 2;
  constexpr int BQT = 64;
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sK = smem_u32(smem);
  const uint32_t sV = sK + BK * 128;
  const uint32_t sQ = sV + BK * 128;                    // 2 stages
  const uint32_t sdO = sQ + 2 * BQT * 128;              // 2 stages
  float* sL = reinterpret_cast<float*>(smem + 2 * BK * 128 + 4 * BQT * 128);   // [2][64] lse * log2e
  float* sD = sL + 2 * BQT;                                                      // [2][64] delta
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int b = blockIdx.z, hh = blockIdx.y;
  const int k0 = blockIdx.x * BK, win = k0 / dm.w, j0 = k0 % dm.w;
  const int I = dm.h * DH;
  const long long ld = 3LL * I;
  const long long seq_row0 = (long long)b * dm.n;
  const bf16* Kg = qkv + (seq_row0 + k0) * ld + I + hh * DH;
  const bf16* Vg = Kg + I;
  const bf16* Qg = qkv + seq_row0 * ld + hh * DH;
  const bf16* dOg = dout + seq_row0 * I + hh * DH;
  const int nwin = dm.n / dm.w;
  const int nown = (dm.w - j0) / BQT;                   // query tiles of the own window at or after the diagonal
  const int nnext = (win + 1 < nwin) ? dm.w / BQT : 0;
  const int ntiles = nown + nnext;
  auto q_pos = [&](int qt) { return qt < nown ? win * dm.w + j0 + qt * BQT : (win + 1) * dm.w + (qt - nown) * BQT; };
  auto load_q_tile = [&](int qt, int st) {
    const int qp = q_pos(qt);
    load_tile_async<BQT, THREADS>(sQ + st * BQT * 128, Qg + (long long)qp * ld, ld, tid);
    load_tile_async<BQT, THREADS>(sdO + st * BQT * 128, dOg + (long long)qp * I, I, tid);
    if (tid < BQT) {
      const long long t = seq_row0 + qp + tid;
      sL[st * BQT + tid] = lse[t * dm.h + hh] * LOG2E;
      sD[st * BQT + tid] = delta[t * dm.h + hh];
    }
  };

  load_tile_async<BK, THREADS>(sK, Kg, ld, tid);
  load_tile_async<BK, THREADS>(sV, Vg, ld, tid);
  load_q_tile(0, 0);
  cp_async_commit();

  const float scale = 0.125f /* 1/sqrt(64), exact */;
  const float sc = scale * LOG2E;
  float dk[8][4], dv[8][4];
  zero_acc(dk);
  zero_acc(dv);
  uint32_t ka[4][4], va[4][4];
  const int kj_lo = j0 + warp * 16;                     // in-window offset of this warp's first key row

  for (int qt = 0; qt < ntiles; ++qt) {
    const int st = qt & 1;
    if (qt + 1 < ntiles) {
      load_q_tile(qt + 1, st ^ 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (qt == 0) {
      load_a_frags(ka, sK, warp * 16, lane);
      load_a_frags(va, sV, warp * 16, lane);
    }
    const bool own = qt < nown;
    const int c0 = j0 + qt * BQT;                       // in-window offset of the tile's first query (own window only)
    if (!(own && c0 + BQT - 1 < kj_lo)) {               // warp-uniform: every query of the tile precedes every key row
      float s[8][4], dp[8][4];
      zero_acc(s);
      zero_acc(dp);
      mma_a_xt(s, ka, sQ + st * BQT * 128, lane);       // S^T[key][query]
      mma_a_xt(dp, va, sdO + st * BQT * 128, lane);     // dP^T[key][query]
      const bool need_mask = own && (c0 < kj_lo + 15);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int col = 8 * j + 2 * t4 + (e & 1);     // query index inside the tile
          float p = exp2f(s[j][e] * sc - sL[st * BQT + col]);
          if (need_mask) {
            const int qi = c0 + col;
            const int kj = kj_lo + g + ((e >> 1) << 3);
            if (kj > qi) p = 0.f;
          }
          dp[j][e] = p * (dp[j][e] - sD[st * BQT + col]) * scale;   // dS^T
          s[j][e] = p;                                              // P^T
        }
      }
      uint32_t pa[4][4];
      acc_to_a(pa, s);
      mma_p_x(dv, pa, sdO + st * BQT * 128, lane);      // dV += P^T dO
      acc_to_a(pa, dp);
      mma_p_x(dk, pa, sQ + st * BQT * 128, lane);       // dK += dS^T Q
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const long long t = seq_row0 + k0 + warp * 16 + g + 8 * r;
    bf16* pk = dqkv + t * ld + I + hh * DH + 2 * t4;
    bf16* pv = pk + I;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int pos = k0 + warp * 16 + g + 8 * r;
      *reinterpret_cast<uint32_t*>(pk + 8 * j) = unrotate_pack(dm, pos, 4 * j + t4, dk[j][2 * r], dk[j][2 * r + 1]);
      *reinterpret_cast<uint32_t*>(pv + 8 * j) = unrotate_pack(dm, pos, 4 * j + t4, dv[j][2 * r], dv[j][2 * r + 1]);
    }
  }
}

template <typename K> int set_smem(K kern, int bytes) {
  PG_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  return PROGEN_OK;
}

// tile sizes: 128-row tiles need window % 128 == 0; PROGEN_ATTN_TILES="fwd,dq,dkv" (64|128 each) overrides for tuning
struct TileChoice { int fwd, dq, dkv; };
TileChoice tile_choice(int window) {
  static TileChoice env = [] {
    TileChoice t{64, 64, 64};      // 64-row tiles by default: more CTAs per SM
    if (const char* e = getenv("PROGEN_ATTN_TILES")) sscanf(e, "%d,%d,%d", &t.fwd, &t.dq, &t.dkv);
    return t;
  }();
  TileChoice t = env;
  if (window % 128 != 0) t = TileChoice{64, 64, 64};
  return t;
}

template <int BQ> int launch_fwd_t(const bf16* qkv, bf16* out, float* lse, const Dims& dm, int B, cudaStream_t s) {
  const int smem = BQ * 128 + 4 * BKV * 128;
  static bool once = false;
  if (!once) { int rc = set_smem(attn_fwd_mma_kernel<BQ>, smem); if (rc) return rc; once = true; }
  attn_fwd_mma_kernel<BQ><<<dim3(dm.n / BQ, dm.h, B), BQ * 2, smem, s>>>(qkv, out, lse, dm);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}
template <int BQ> int launch_dq_t(const bf16* qkv, const bf16* out, const bf16* dout, const float* lse, float* delta, bf16* dqkv,
                                  const Dims& dm, int B, cudaStream_t s) {
  const int smem = 2 * BQ * 128 + 4 * BKV * 128;
  static bool once = false;
  if (!once) { int rc = set_smem(attn_bwd_dq_mma_kernel<BQ>, smem); if (rc) return rc; once = true; }
  attn_bwd_dq_mma_kernel<BQ><<<dim3(dm.n / BQ, dm.h, B), BQ * 2, smem, s>>>(qkv, out, dout, lse, delta, dqkv, dm);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}
template <int BK> int launch_dkv_t(const bf16* qkv, const bf16* dout, const float* lse, const float* delta, bf16* dqkv,
                                   const Dims& dm, int B, cudaStream_t s) {
  const int smem = 2 * BK * 128 + 4 * 64 * 128 + 4 * 64 * 4;
  static bool once = false;
  if (!once) { int rc = set_smem(attn_bwd_dkv_mma_kernel<BK>, smem); if (rc) return rc; once = true; }
  attn_bwd_dkv_mma_kernel<BK><<<dim3(dm.n / BK, dm.h, B), BK * 2, smem, s>>>(qkv, dout, lse, delta, dqkv, dm);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

}  // namespace

extern "C" {

// bf16, dim_head == 64, window % 64 == 0.  qkv [T, 3*heads*64] (rotated), out [T, heads*64], lse [T, heads].
int progen_local_attn_fwd(const void* qkv, void* out, float* lse, int B, int seq_len, int window, int heads, int dim_head,
                          void* stream) {
  PG_CHECK_ARG(B > 0 && heads > 0 && dim_head == DH && window % 64 == 0 && seq_len % window == 0);
  Dims dm{seq_len, window, heads, nullptr, nullptr};
  cudaStream_t s = (cudaStream_t)stream;
  if (tile_choice(window).fwd == 128) return launch_fwd_t<128>((const bf16*)qkv, (bf16*)out, lse, dm, B, s);
  return launch_fwd_t<64>((const bf16*)qkv, (bf16*)out, lse, dm, B, s);
}

// dqkv [T, 3*heads*64] receives dq | dk | dv; delta [T, heads] is workspace.  With rot_sin/rot_cos ([seq_len, 32] tables)
// the rotary backward is fused and the gradients are w.r.t. the projections BEFORE rotary; with null tables they are
// w.r.t. the rotated q, k, v.
int progen_local_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv, float* delta,
                          const float* rot_sin, const float* rot_cos, int B, int seq_len, int window, int heads, int dim_head,
                          void* stream) {
  PG_CHECK_ARG(B > 0 && heads > 0 && dim_head == DH && window % 64 == 0 && seq_len % window == 0);
  Dims dm{seq_len, window, heads, rot_sin, rot_cos};
  cudaStream_t s = (cudaStream_t)stream;
  const TileChoice tc = tile_choice(window);
  // the dQ kernel also produces delta = rowsum(dO o O) for the dK/dV kernel that follows it on the same stream
  int rc = tc.dq == 128 ? launch_dq_t<128>((const bf16*)qkv, (const bf16*)out, (const bf16*)dout, lse, delta, (bf16*)dqkv, dm, B, s)
                        : launch_dq_t<64>((const bf16*)qkv, (const bf16*)out, (const bf16*)dout, lse, delta, (bf16*)dqkv, dm, B, s);
  if (rc) return rc;
  return tc.dkv == 128 ? launch_dkv_t<128>((const bf16*)qkv, (const bf16*)dout, lse, delta, (bf16*)dqkv, dm, B, s)
                       : launch_dkv_t<64>((const bf16*)qkv, (const bf16*)dout, lse, delta, (bf16*)dqkv, dm, B, s);
}

}  // extern "C"
