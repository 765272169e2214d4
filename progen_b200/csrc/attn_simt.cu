// Sliding-window causal attention with one look-back window (reference progen.py:88-102), CUDA-core version.
// Exact fp32 arithmetic: this is the `mixed_precision=False` path and the on-device cross-check for the
// tensor-core kernels (attn_wgmma.cu).  q, k, v are already rotated (qkv GEMM epilogue) and live in one [T, 3*I]
// buffer (q | k | v, each head-major), the output is [T, I].
//
// Query at position pos = win*w + i sees: the w keys of the previous window (for win == 0 these are w ZERO keys that
// still take part in the softmax — reference quirk Q1: the zero window is padded after rotary and is not masked) and
// keys 0..i of its own window.  The reference's -1e10 fill underflows to an exact 0 probability in fp32, so masked
// keys are simply skipped.
//
// One warp per (token, head); lanes own keys (forward / dq) or queries (dk, dv), so no atomics are needed.
#include "common.cuh"
#include "../../include/progen_b200.h"

namespace {

template <typename T, int DH> __device__ __forceinline__ void load_row(const T* p, float (&v)[DH]) {
#pragma unroll
  for (int i = 0; i < DH; i += 8) {
    float t[8];
    load_vec<8>(p + i, t);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[i + j] = t[j];
  }
}
template <typename T, int DH> __device__ __forceinline__ void store_row(T* p, const float (&v)[DH]) {
#pragma unroll
  for (int i = 0; i < DH; i += 8) {
    float t[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) t[j] = v[i + j];
    store_vec<8>(p + i, t);
  }
}
template <int DH> __device__ __forceinline__ float dot(const float (&a)[DH], const float (&b)[DH]) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < DH; ++i) s = fmaf(a[i], b[i], s);
  return s;
}

struct AttnDims {
  long long T; int n, w, h, dh; long long ld;      // ld = 3 * h * dh
};

template <typename TO, int DH>
__global__ void __launch_bounds__(128) attn_fwd_kernel(const TO* __restrict__ qkv, TO* __restrict__ out,
                                                       float* __restrict__ lse, const AttnDims dm) {
  const int lane = threadIdx.x & 31;
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  if (wid >= dm.T * dm.h) return;
  const long long t = wid / dm.h;
  const int hh = (int)(wid % dm.h);
  const int I = dm.h * DH;
  const int pos = (int)(t % dm.n), win = pos / dm.w, i = pos % dm.w;
  const long long seq0 = t - pos;
  const float scale = (1.0f / sqrtf((float)DH));
  float q[DH];
  load_row<TO, DH>(qkv + t * dm.ld + hh * DH, q);
  // keys j in [0, w + i]: j < w -> previous window (phantom zeros when win == 0), else own window
  const int nkeys = dm.w + i + 1;
  const long long kbase = seq0 + (long long)(win - 1) * dm.w;     // global row of key j = kbase + j
  float m = -INFINITY;
  for (int j = lane; j < nkeys; j += 32) {
    float s = 0.f;
    if (win > 0 || j >= dm.w) {
      float k[DH];
      load_row<TO, DH>(qkv + (kbase + j) * dm.ld + I + hh * DH, k);
      s = dot<DH>(q, k) * scale;
    }
    m = fmaxf(m, s);
  }
  m = warp_max(m);
  float l = 0.f;
  float acc[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) acc[d] = 0.f;
  for (int j = lane; j < nkeys; j += 32) {
    if (win > 0 || j >= dm.w) {
      float k[DH];
      load_row<TO, DH>(qkv + (kbase + j) * dm.ld + I + hh * DH, k);
      const float p = expf(dot<DH>(q, k) * scale - m);
      l += p;
      float v[DH];
      load_row<TO, DH>(qkv + (kbase + j) * dm.ld + 2 * I + hh * DH, v);
#pragma unroll
      for (int d = 0; d < DH; ++d) acc[d] = fmaf(p, v[d], acc[d]);
    } else {
      l += expf(-m);                                            // zero key: logit 0, value 0
    }
  }
  l = warp_sum(l);
  const float inv = 1.f / l;
#pragma unroll
  for (int d = 0; d < DH; ++d) acc[d] = warp_sum(acc[d]) * inv;
  if (lane == 0) {
    store_row<TO, DH>(out + t * (long long)I + hh * DH, acc);
    lse[t * dm.h + hh] = m + logf(l);
  }
}

// dq(t) = scale * sum_j p_j (dP_j - D) k_j,  D = dO . O,  p_j = exp(s_j - lse),  dP_j = dO . v_j
template <typename TO, int DH>
__global__ void __launch_bounds__(128) attn_bwd_dq_kernel(const TO* __restrict__ qkv, const TO* __restrict__ out,
                                                          const TO* __restrict__ dout, const float* __restrict__ lse,
                                                          TO* __restrict__ dqkv, float* __restrict__ delta,
                                                          const AttnDims dm) {
  const int lane = threadIdx.x & 31;
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  if (wid >= dm.T * dm.h) return;
  const long long t = wid / dm.h;
  const int hh = (int)(wid % dm.h);
  const int I = dm.h * DH;
  const int pos = (int)(t % dm.n), win = pos / dm.w, i = pos % dm.w;
  const long long seq0 = t - pos;
  const float scale = (1.0f / sqrtf((float)DH));
  float q[DH], dO[DH];
  load_row<TO, DH>(qkv + t * dm.ld + hh * DH, q);
  load_row<TO, DH>(dout + t * (long long)I + hh * DH, dO);
  float D;
  {
    float o[DH];
    load_row<TO, DH>(out + t * (long long)I + hh * DH, o);
    D = dot<DH>(dO, o);
  }
  const float L = lse[t * dm.h + hh];
  if (lane == 0) delta[t * dm.h + hh] = D;
  float acc[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) acc[d] = 0.f;
  const int j0 = (win > 0) ? 0 : dm.w;                              // phantom keys carry no gradient to q (k == 0)
  const int nkeys = dm.w + i + 1;
  const long long kbase = seq0 + (long long)(win - 1) * dm.w;
  for (int j = j0 + lane; j < nkeys; j += 32) {
    float k[DH], v[DH];
    load_row<TO, DH>(qkv + (kbase + j) * dm.ld + I + hh * DH, k);
    load_row<TO, DH>(qkv + (kbase + j) * dm.ld + 2 * I + hh * DH, v);
    const float p = expf(dot<DH>(q, k) * scale - L);
    const float dS = p * (dot<DH>(dO, v) - D) * scale;
#pragma unroll
    for (int d = 0; d < DH; ++d) acc[d] = fmaf(dS, k[d], acc[d]);
  }
#pragma unroll
  for (int d = 0; d < DH; ++d) acc[d] = warp_sum(acc[d]);
  if (lane == 0) store_row<TO, DH>(dqkv + t * dm.ld + hh * DH, acc);
}

// For key row t (position pos = win*w + i): queries of the same window with row >= i, and all rows of window win+1.
template <typename TO, int DH>
__global__ void __launch_bounds__(128) attn_bwd_dkv_kernel(const TO* __restrict__ qkv, const TO* __restrict__ dout,
                                                           const float* __restrict__ lse, const float* __restrict__ delta,
                                                           TO* __restrict__ dqkv, const AttnDims dm) {
  const int lane = threadIdx.x & 31;
  const long long wid = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  if (wid >= dm.T * dm.h) return;
  const long long t = wid / dm.h;
  const int hh = (int)(wid % dm.h);
  const int I = dm.h * DH;
  const int pos = (int)(t % dm.n), win = pos / dm.w, i = pos % dm.w;
  const float scale = (1.0f / sqrtf((float)DH));
  float k[DH], v[DH];
  load_row<TO, DH>(qkv + t * dm.ld + I + hh * DH, k);
  load_row<TO, DH>(qkv + t * dm.ld + 2 * I + hh * DH, v);
  float dk[DH], dv[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) { dk[d] = 0.f; dv[d] = 0.f; }
  const int nwin = (dm.n + dm.w - 1) / dm.w;          // the last window may be partial (a cut backward)
  // query offsets r relative to this key: the own window's queries from the key on, below min(window end, n), then, if
  // a next window exists, its queries below n.  At whole windows: r in [0, w - 1 - i] and [w - i, 2w - 1 - i].
  const int own_end = min((win + 1) * dm.w, dm.n);
  const int nq = (own_end - pos) + ((win + 1 < nwin) ? min((win + 2) * dm.w, dm.n) - own_end : 0);
  for (int r = lane; r < nq; r += 32) {
    const long long tq = t + r;
    float q[DH], dO[DH];
    load_row<TO, DH>(qkv + tq * dm.ld + hh * DH, q);
    load_row<TO, DH>(dout + tq * (long long)I + hh * DH, dO);
    const float p = expf(dot<DH>(q, k) * scale - lse[tq * dm.h + hh]);
    const float dS = p * (dot<DH>(dO, v) - delta[tq * dm.h + hh]) * scale;
#pragma unroll
    for (int d = 0; d < DH; ++d) {
      dk[d] = fmaf(dS, q[d], dk[d]);
      dv[d] = fmaf(p, dO[d], dv[d]);
    }
  }
#pragma unroll
  for (int d = 0; d < DH; ++d) { dk[d] = warp_sum(dk[d]); dv[d] = warp_sum(dv[d]); }
  if (lane == 0) {
    store_row<TO, DH>(dqkv + t * dm.ld + I + hh * DH, dk);
    store_row<TO, DH>(dqkv + t * dm.ld + 2 * I + hh * DH, dv);
  }
}

template <typename TO, int DH>
int launch_fwd(const void* qkv, void* out, float* lse, const AttnDims& dm, cudaStream_t s) {
  const long long warps = dm.T * dm.h;
  const int grid = (int)((warps + 3) / 4);
  attn_fwd_kernel<TO, DH><<<grid, 128, 0, s>>>((const TO*)qkv, (TO*)out, lse, dm);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}
template <typename TO, int DH>
int launch_bwd(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv, float* delta,
               const AttnDims& dm, cudaStream_t s) {
  const long long warps = dm.T * dm.h;
  const int grid = (int)((warps + 3) / 4);
  attn_bwd_dq_kernel<TO, DH><<<grid, 128, 0, s>>>((const TO*)qkv, (const TO*)out, (const TO*)dout, lse, (TO*)dqkv, delta, dm);
  PG_LAUNCH_CHECK();
  attn_bwd_dkv_kernel<TO, DH><<<grid, 128, 0, s>>>((const TO*)qkv, (const TO*)dout, lse, delta, (TO*)dqkv, dm);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

}  // namespace

#define ATTN_DISPATCH(FN, ...)                                                            \
  do {                                                                                    \
    if (dtype == PG_F32) {                                                                \
      switch (dim_head) {                                                                 \
        case 16: return FN<float, 16>(__VA_ARGS__);                                       \
        case 32: return FN<float, 32>(__VA_ARGS__);                                       \
        case 64: return FN<float, 64>(__VA_ARGS__);                                       \
        case 128: return FN<float, 128>(__VA_ARGS__);                                     \
      }                                                                                   \
    } else {                                                                              \
      switch (dim_head) {                                                                 \
        case 16: return FN<bf16, 16>(__VA_ARGS__);                                        \
        case 32: return FN<bf16, 32>(__VA_ARGS__);                                        \
        case 64: return FN<bf16, 64>(__VA_ARGS__);                                        \
        case 128: return FN<bf16, 128>(__VA_ARGS__);                                      \
      }                                                                                   \
    }                                                                                     \
    progen_set_error("local_attn: unsupported dim_head %d (16/32/64/128)", dim_head);     \
    return PROGEN_ERR_UNSUPPORTED;                                                        \
  } while (0)

namespace {
// the one launcher of both backward entry points (they differ in their host check only)
int bwd(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv, float* delta, int dtype, int B,
        int seq_len, int window, int heads, int dim_head, void* stream) {
  AttnDims dm{(long long)B * seq_len, seq_len, window, heads, dim_head, 3LL * heads * dim_head};
  ATTN_DISPATCH(launch_bwd, qkv, out, dout, lse, dqkv, delta, dm, (cudaStream_t)stream);
}
}  // namespace

extern "C" {

// The forward takes any seq_len: the last window may be partial.  A query at pos reads keys (win - 1) * w .. pos only, so
// a forward cut short of the model's sequence length computes the first seq_len rows of the full one, bitwise.
// progen_local_attn_bwd_simt keeps whole windows; progen_local_attn_bwd_cut_simt takes any seq_len (see the header).
int progen_local_attn_fwd_simt(const void* qkv, void* out, float* lse, int dtype, int B, int seq_len, int window,
                               int heads, int dim_head, void* stream) {
  PG_CHECK_ARG(B > 0 && seq_len > 0 && window > 0 && heads > 0);
  AttnDims dm{(long long)B * seq_len, seq_len, window, heads, dim_head, 3LL * heads * dim_head};
  ATTN_DISPATCH(launch_fwd, qkv, out, lse, dm, (cudaStream_t)stream);
}

int progen_local_attn_bwd_simt(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                               float* delta, int dtype, int B, int seq_len, int window, int heads, int dim_head,
                               void* stream) {
  PG_CHECK_ARG(B > 0 && seq_len > 0 && window > 0 && seq_len % window == 0 && heads > 0);
  return bwd(qkv, out, dout, lse, dqkv, delta, dtype, B, seq_len, window, heads, dim_head, stream);
}

int progen_local_attn_bwd_cut_simt(const void* qkv, const void* out, const void* dout, const float* lse, void* dqkv,
                                   float* delta, int dtype, int B, int seq_len, int window, int heads, int dim_head,
                                   void* stream) {
  PG_CHECK_ARG(B > 0 && seq_len > 0 && window > 0 && heads > 0);
  return bwd(qkv, out, dout, lse, dqkv, delta, dtype, B, seq_len, window, heads, dim_head, stream);
}

}  // extern "C"
