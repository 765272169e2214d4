// HBM-bound kernels of the ProGen hot path: token embedding, LayerNorm(scale-only)+token-shift (fwd/bwd),
// cross-entropy with the pad-as-EOS mask (fwd+bwd fused), rotary backward, SGU gating, GELU backward, column sums, and the
// row gather that fills the decoder's caches from an inference forward (generation prefill).
// All are coalesced, 8/16-byte vectorised, one warp per row where a row reduction is needed.
#include <cmath>
#include "common.cuh"
#include "../../include/progen_b200.h"

// ln_stream.cu
int ln_shift_bwd_stream_launch(const void* dy, long long lddy, int act_dtype, const void* x, long long ldx, int x_dtype,
                               const float* scale, const float* mean, const float* rstd, float* dres, void* dout,
                               long long ldo, float* dscale, float* dres_colsum, long long T, int d, int seq_len, int shift,
                               int residual, cudaStream_t stream);

namespace {

constexpr int ROWS_PER_BLOCK = 8;     // 8 warps, one row each
constexpr float LN_EPS = 1e-5f;       // hk.LayerNorm default (reference progen.py:22)

template <typename T> __device__ __forceinline__ void load4(const T* p, float (&v)[4]);
template <> __device__ __forceinline__ void load4<float>(const float* p, float (&v)[4]) {
  const float4 t = *reinterpret_cast<const float4*>(p);
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <> __device__ __forceinline__ void load4<bf16>(const bf16* p, float (&v)[4]) {
  const uint2 t = *reinterpret_cast<const uint2*>(p);
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.y));
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
__device__ __forceinline__ void store4(float* p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void store4(bf16* p, const float (&v)[4]) {
  uint2 t;
  t.x = pack_bf16x2(v[0], v[1]); t.y = pack_bf16x2(v[2], v[3]);
  *reinterpret_cast<uint2*>(p) = t;
}

// ------------------------------------------------------------------------------------------------ embed
// reference progen.py:226 (hk.Embed row gather); residual stream is fp32 in both precision modes
__global__ void embed_fwd_kernel(const int* __restrict__ tok, const float* __restrict__ table, float* __restrict__ x,
                                 long long T, int d, int V) {
  const long long total = T * (d / 4);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / (d / 4);
    const int c = (int)(i % (d / 4)) * 4;
    int id = tok[t];
    id = id < 0 ? 0 : (id >= V ? V - 1 : id);
    *reinterpret_cast<float4*>(x + t * d + c) = *reinterpret_cast<const float4*>(table + (long long)id * d + c);
  }
}

// dtable[v, c] += sum_{t: tok[t]==v} dx[t, c].  Block = 32 columns x a slab of rows, shared-memory bins per token id.
__global__ void embed_bwd_kernel(const int* __restrict__ tok, const float* __restrict__ dx, float* __restrict__ dtable,
                                 long long T, int d, int V, long long rows_per_block) {
  extern __shared__ float bins[];                 // [V][32]
  const int c0 = blockIdx.x * 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  for (int i = threadIdx.x; i < V * 32; i += blockDim.x) bins[i] = 0.f;
  __syncthreads();
  const long long r0 = blockIdx.y * rows_per_block;
  const long long r1 = min(T, r0 + rows_per_block);
  if (c0 + lane < d) {
    for (long long t = r0 + warp; t < r1; t += nwarp) {
      int id = tok[t];
      id = id < 0 ? 0 : (id >= V ? V - 1 : id);
      atomicAdd(&bins[id * 32 + lane], dx[t * d + c0 + lane]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < V * 32; i += blockDim.x) {
    const float v = bins[i];
    const int c = c0 + (i & 31);
    if (v != 0.f && c < d) atomicAdd(dtable + (long long)(i >> 5) * d + c, v);
  }
}

// -------------------------------------------------------------------------------- LayerNorm + token shift
// y = shift_tokens(LN(x) * scale): reference progen.py:74-77,132-135 (LN then shift; first half of the channels comes
// from the previous position, zeros at position 0) and progen.py:170 (SGU: LN only, strided input).
// One warp per row.  The warp that normalises row t writes channels [half, d) of row t and channels [0, half) of
// row t+1, so each row is read exactly once.
template <typename TI, typename TO>
__global__ void ln_shift_fwd_kernel(const TI* __restrict__ x, long long ldx, const float* __restrict__ scale,
                                    TO* __restrict__ y, long long ldy, float* __restrict__ mean_out,
                                    float* __restrict__ rstd_out, long long T, int d, int seq_len, int shift) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int half = d >> 1;
  for (long long t = blockIdx.x * (long long)ROWS_PER_BLOCK + warp; t < T; t += (long long)gridDim.x * ROWS_PER_BLOCK) {
    const TI* xr = x + t * ldx;
    float s = 0.f;
    for (int c = lane * 4; c < d; c += 128) {
      float v[4];
      load4<TI>(xr + c, v);
      s += v[0] + v[1] + v[2] + v[3];
    }
    const float mean = warp_sum(s) / d;
    float q = 0.f;
    for (int c = lane * 4; c < d; c += 128) {
      float v[4];
      load4<TI>(xr + c, v);
#pragma unroll
      for (int i = 0; i < 4; ++i) { const float u = v[i] - mean; q += u * u; }
    }
    const float rstd = rsqrtf(warp_sum(q) / d + LN_EPS);
    if (lane == 0) { mean_out[t] = mean; rstd_out[t] = rstd; }
    const int pos = (int)(t % seq_len);
    for (int c = lane * 4; c < d; c += 128) {
      float v[4], sc[4], o[4];
      load4<TI>(xr + c, v);
      load4<float>(scale + c, sc);
#pragma unroll
      for (int i = 0; i < 4; ++i) o[i] = (v[i] - mean) * rstd * sc[i];
      if (!shift || c >= half) {
        store4(y + t * ldy + c, o);
      } else {
        if (pos + 1 < seq_len) store4(y + (t + 1) * ldy + c, o);
        if (pos == 0) { const float z[4] = {0.f, 0.f, 0.f, 0.f}; store4(y + t * ldy + c, z); }
      }
    }
  }
}

// Backward of the above.  dyn(t, c) = c < half ? dy(t+1, c) [0 at the last position] : dy(t, c)   (un-shift)
// g = dyn * scale; dx = rstd * (g - mean(g) - xhat * mean(g * xhat)); dscale(c) += sum_t dyn * xhat.
// RESIDUAL: dres(fp32) += dx and (optionally) a low-precision copy of the updated dres for the next GEMMs.
template <typename TI, typename TO, int NCH, bool RESIDUAL>
__global__ void ln_shift_bwd_kernel(const TO* __restrict__ dy, long long lddy, const TI* __restrict__ x, long long ldx,
                                    const float* __restrict__ scale, const float* __restrict__ mean_in,
                                    const float* __restrict__ rstd_in, float* __restrict__ dres, TO* __restrict__ dout,
                                    long long ldo, float* __restrict__ dscale, float* __restrict__ dres_colsum,
                                    long long T, int d, int seq_len, int shift) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int half = d >> 1;
  float ds_acc[NCH][4];
  float cs_acc[RESIDUAL ? NCH : 1][4];       // column sums of the UPDATED residual gradient (= the next bias gradient)
#pragma unroll
  for (int i = 0; i < NCH; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      ds_acc[i][j] = 0.f;
      if (RESIDUAL) cs_acc[RESIDUAL ? i : 0][j] = 0.f;
    }

  for (long long t = blockIdx.x * (long long)ROWS_PER_BLOCK + warp; t < T; t += (long long)gridDim.x * ROWS_PER_BLOCK) {
    const TI* xr = x + t * ldx;
    const float mean = mean_in[t], rstd = rstd_in[t];
    const int pos = (int)(t % seq_len);
    const bool has_next = pos + 1 < seq_len;
    float s1 = 0.f, s2 = 0.f;
    if constexpr (NCH <= 4) {
      // d <= 512: the row fits in registers — read x, dy and the residual gradient once, all loads issued up front
      float xh[NCH][4], gs[NCH][4], rr[NCH][4];
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch) {
        const int c = ch * 128 + lane * 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) { xh[ch][i] = 0.f; gs[ch][i] = 0.f; rr[ch][i] = 0.f; }
        if (c < d) {
          float sc[4];
          load4<TI>(xr + c, xh[ch]);
          load4<float>(scale + c, sc);
          if (!shift || c >= half) load4<TO>(dy + t * lddy + c, gs[ch]);
          else if (has_next) load4<TO>(dy + (t + 1) * lddy + c, gs[ch]);
          if constexpr (RESIDUAL) load4<float>(dres + t * (long long)d + c, rr[ch]);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            xh[ch][i] = (xh[ch][i] - mean) * rstd;
            ds_acc[ch][i] += gs[ch][i] * xh[ch][i];
            gs[ch][i] *= sc[i];
            s1 += gs[ch][i]; s2 += gs[ch][i] * xh[ch][i];
          }
        }
      }
      s1 = warp_sum(s1) / d;
      s2 = warp_sum(s2) / d;
#pragma unroll
      for (int ch = 0; ch < NCH; ++ch) {
        const int c = ch * 128 + lane * 4;
        if (c < d) {
          float o[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) o[i] = rstd * (gs[ch][i] - s1 - xh[ch][i] * s2);
          if constexpr (RESIDUAL) {
#pragma unroll
            for (int i = 0; i < 4; ++i) { rr[ch][i] += o[i]; cs_acc[ch][i] += rr[ch][i]; }
            store4(dres + t * (long long)d + c, rr[ch]);
            if (dout) store4(dout + t * ldo + c, rr[ch]);
          } else {
            store4(dout + t * ldo + c, o);
          }
        }
      }
      continue;
    }
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      const int c = ch * 128 + lane * 4;
      if (c < d) {
        float xv[4], sc[4], g[4] = {0.f, 0.f, 0.f, 0.f};
        load4<TI>(xr + c, xv);
        load4<float>(scale + c, sc);
        if (!shift || c >= half) load4<TO>(dy + t * lddy + c, g);
        else if (has_next) load4<TO>(dy + (t + 1) * lddy + c, g);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float xh = (xv[i] - mean) * rstd;
          ds_acc[ch][i] += g[i] * xh;
          const float gs = g[i] * sc[i];
          s1 += gs; s2 += gs * xh;
        }
      }
    }
    s1 = warp_sum(s1) / d;
    s2 = warp_sum(s2) / d;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      const int c = ch * 128 + lane * 4;
      if (c < d) {
        float xv[4], sc[4], g[4] = {0.f, 0.f, 0.f, 0.f}, o[4];
        load4<TI>(xr + c, xv);
        load4<float>(scale + c, sc);
        if (!shift || c >= half) load4<TO>(dy + t * lddy + c, g);
        else if (has_next) load4<TO>(dy + (t + 1) * lddy + c, g);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float xh = (xv[i] - mean) * rstd;
          o[i] = rstd * (g[i] * sc[i] - s1 - xh * s2);
        }
        if constexpr (RESIDUAL) {
          float r[4];
          load4<float>(dres + t * (long long)d + c, r);
#pragma unroll
          for (int i = 0; i < 4; ++i) { r[i] += o[i]; cs_acc[ch][i] += r[i]; }
          store4(dres + t * (long long)d + c, r);
          if (dout) store4(dout + t * ldo + c, r);
        } else {
          store4(dout + t * ldo + c, o);
        }
      }
    }
  }
  // dscale (nullable: a frozen scale): reduce the 8 warps of the block through shared memory (128 columns at a time),
  // one atomic per column per block
  __shared__ float red[ROWS_PER_BLOCK][128];
#pragma unroll
  for (int ch = 0; ch < NCH; ++ch) {
    if (ch * 128 >= d) break;
    if (dscale) {                              // block-uniform
#pragma unroll
      for (int i = 0; i < 4; ++i) red[warp][lane * 4 + i] = ds_acc[ch][i];
      __syncthreads();
      if (threadIdx.x < 128) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < ROWS_PER_BLOCK; ++w) s += red[w][threadIdx.x];
        const int c = ch * 128 + threadIdx.x;
        if (c < d) atomicAdd(dscale + c, s);
      }
      __syncthreads();
    }
    if constexpr (RESIDUAL) {
      if (dres_colsum) {                       // block-uniform
#pragma unroll
        for (int i = 0; i < 4; ++i) red[warp][lane * 4 + i] = cs_acc[ch][i];
        __syncthreads();
        if (threadIdx.x < 128) {
          float s = 0.f;
#pragma unroll
          for (int w = 0; w < ROWS_PER_BLOCK; ++w) s += red[w][threadIdx.x];
          const int c = ch * 128 + threadIdx.x;
          if (c < d) atomicAdd(dres_colsum + c, s);
        }
        __syncthreads();
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ column sums
// out[c] += sum_t in[t, c]   (bias gradients)
template <typename TI>
__global__ void colsum_kernel(const TI* __restrict__ in, long long ld, float* __restrict__ out, long long T, int N,
                              long long rows_per_block) {
  __shared__ float red[ROWS_PER_BLOCK][128];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.x * 128 + lane * 4;
  const long long r0 = blockIdx.y * rows_per_block, r1 = min(T, r0 + rows_per_block);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  if (c < N) {
    for (long long t = r0 + warp; t < r1; t += ROWS_PER_BLOCK) {
      float v[4];
      load4<TI>(in + t * ld + c, v);
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] += v[i];
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) red[warp][lane * 4 + i] = acc[i];
  __syncthreads();
  if (threadIdx.x < 128) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < ROWS_PER_BLOCK; ++w) s += red[w][threadIdx.x];
    const int cc = blockIdx.x * 128 + threadIdx.x;
    if (cc < N) atomicAdd(out + cc, s);
  }
}

// ------------------------------------------------------------------------------------------ cross entropy
// reference utils.py:45-59: per sequence, mask = (label != 0) | (first label == 0); loss_b = -sum(mask*logp)/sum(mask);
// utils.py:76: mean over the batch.  Kernel 1 turns labels into per-token weights w = mask / (count_b * B_global).
__global__ void ce_weights_kernel(const int* __restrict__ labels, float* __restrict__ w, int n, float inv_batch) {
  __shared__ int s_first, s_count;
  const int b = blockIdx.x;
  if (threadIdx.x == 0) { s_first = n; s_count = 0; }
  __syncthreads();
  const int* lb = labels + (long long)b * n;
  int first = n, cnt = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    if (lb[i] == 0) first = min(first, i); else cnt++;
  }
  atomicMin(&s_first, first);
  atomicAdd(&s_count, cnt);
  __syncthreads();
  const int total = s_count + (s_first < n ? 1 : 0);
  const float wv = inv_batch / (float)total;
  for (int i = threadIdx.x; i < n; i += blockDim.x) w[(long long)b * n + i] = (lb[i] != 0 || i == s_first) ? wv : 0.f;
}

// Row max and sum of exp(x - max) of one V-wide logits row, computed by one warp in a fixed order (every lane gets both);
// log-sum-exp = mx + logf(se).  Shared by the training loss and the inference log-likelihood, so both see the same bits.
template <typename TL>
__device__ __forceinline__ void warp_row_max_sumexp(const TL* __restrict__ lr, int V, int lane, float& mx, float& se) {
  mx = -INFINITY;
  for (int c = lane * 4; c < V; c += 128) {
    float v[4];
    load4<TL>(lr + c, v);
    mx = fmaxf(mx, fmaxf(fmaxf(v[0], v[1]), fmaxf(v[2], v[3])));
  }
  mx = warp_max(mx);
  se = 0.f;
  for (int c = lane * 4; c < V; c += 128) {
    float v[4];
    load4<TL>(lr + c, v);
#pragma unroll
    for (int i = 0; i < 4; ++i) se += expf(v[i] - mx);
  }
  se = warp_sum(se);
}

// out-of-range labels are clamped like the token ids in embed_fwd / embed_bwd (jnp indexing clamps); byte 0xFF + 1 = 256
// with V = 256 is reachable from real data (data.py tokenizer) and must not read past the logits row
__device__ __forceinline__ int clamp_label(int lab, int V) { return min(max(lab, 0), V - 1); }

// Kernel 2: one warp per token over V logits: loss += w * (lse - logit[label]); dlogits = w * (softmax - onehot).
template <typename TL, typename TD>
__global__ void ce_fwd_bwd_kernel(const TL* __restrict__ logits, const int* __restrict__ labels,
                                  const float* __restrict__ w, float* __restrict__ loss, TD* __restrict__ dlogits,
                                  long long T, int V) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float block_loss = 0.f;
  for (long long t = blockIdx.x * (long long)ROWS_PER_BLOCK + warp; t < T; t += (long long)gridDim.x * ROWS_PER_BLOCK) {
    const TL* lr = logits + t * V;
    float mx, se;
    warp_row_max_sumexp<TL>(lr, V, lane, mx, se);
    const int lab = clamp_label(labels[t], V);
    const float wt = w[t];
    const float lse = mx + logf(se);
    if (lane == 0) block_loss += wt * (lse - to_f32(lr[lab]));
    if (dlogits) {
      const float inv = 1.f / se;
      for (int c = lane * 4; c < V; c += 128) {
        float v[4], o[4];
        load4<TL>(lr + c, v);
#pragma unroll
        for (int i = 0; i < 4; ++i) o[i] = wt * (expf(v[i] - mx) * inv - ((c + i) == lab ? 1.f : 0.f));
        store4(dlogits + t * V + c, o);
      }
    }
  }
  __shared__ float red[ROWS_PER_BLOCK];
  if (lane == 0) red[warp] = block_loss;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < ROWS_PER_BLOCK; ++i) s += red[i];
    atomicAdd(loss, s);
  }
}

// ------------------------------------------------------------------------------------------ scoring (inference)
// Per-token log-likelihood under the same mask as the loss (utils.py:45-59):  logp[t] = mask_t * log_softmax(logits[t])[label_t].
// Pass 1, one warp per token: the unmasked log-probability of the label.
template <typename TL>
__global__ void token_logprob_kernel(const TL* __restrict__ logits, const int* __restrict__ labels, float* __restrict__ logp,
                                     long long T, int V) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long t = blockIdx.x * (long long)ROWS_PER_BLOCK + warp; t < T; t += (long long)gridDim.x * ROWS_PER_BLOCK) {
    const TL* lr = logits + t * V;
    float mx, se;
    warp_row_max_sumexp<TL>(lr, V, lane, mx, se);
    const int lab = clamp_label(labels[t], V);
    if (lane == 0) logp[t] = to_f32(lr[lab]) - (mx + logf(se));
  }
}

// The loss mask of one sequence (quirk Q8): non-pad labels plus the first pad.  Block-wide; returns the position of the
// first pad (n if none) and the number of masked-in positions.  Integer atomics only: the result does not depend on timing.
__device__ __forceinline__ void seq_loss_mask(const int* __restrict__ lb, int n, int& first, int& count) {
  __shared__ int s_first, s_count;
  if (threadIdx.x == 0) { s_first = n; s_count = 0; }
  __syncthreads();
  int f = n, cnt = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    if (lb[i] == 0) f = min(f, i); else cnt++;
  }
  atomicMin(&s_first, f);
  atomicAdd(&s_count, cnt);
  __syncthreads();
  first = s_first;
  count = s_count + (s_first < n ? 1 : 0);
}

// Fixed-order sum over a 256-thread block (lane shuffles, then the 8 warp partials in order); valid in thread 0.
__device__ __forceinline__ float block_sum_fixed(float v) {
  __shared__ float red[ROWS_PER_BLOCK];
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float s = 0.f;
  if (threadIdx.x == 0)
    for (int i = 0; i < ROWS_PER_BLOCK; ++i) s += red[i];
  return s;
}

// Pass 2, one 256-thread block per sequence: apply the mask in place and reduce it in a fixed order (no float atomics), so
// a sequence's sums are the same bits whatever batch it is scored in.
__global__ void seq_logprob_sum_kernel(const int* __restrict__ labels, float* __restrict__ logp, float* __restrict__ seq_ll,
                                       float* __restrict__ seq_count, int n) {
  const int b = blockIdx.x;
  const int* lb = labels + (long long)b * n;
  float* lp = logp + (long long)b * n;
  int first, count;
  seq_loss_mask(lb, n, first, count);
  float acc = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = (lb[i] != 0 || i == first) ? lp[i] : 0.f;
    lp[i] = v;
    acc += v;
  }
  const float s = block_sum_fixed(acc);
  if (threadIdx.x == 0) {
    seq_ll[b] = s;
    seq_count[b] = (float)count;
  }
}

// ------------------------------------------------------------------------------------------ preference (DPO) head
// Pair i of a preference batch is (chosen row i, rejected row i + pairs).  Its margin z = beta * ((s_c - ref_c) -
// (s_r - ref_r)), its loss softplus(-z) and sigma(-z), in double.  The per-pair blocks and the loss sum both call this, so
// they see the same bits.
__device__ __forceinline__ void preference_pair(const float* __restrict__ seq_ll, const float* __restrict__ ref_ll, int i,
                                                int pairs, double beta, double& z, double& loss, double& sig) {
  z = beta * (((double)seq_ll[i] - (double)ref_ll[i]) - ((double)seq_ll[i + pairs] - (double)ref_ll[i + pairs]));
  const double e = exp(-fabs(z));
  loss = fmax(-z, 0.0) + log1p(e);
  sig = z >= 0.0 ? e / (1.0 + e) : 1.0 / (1.0 + e);
}

constexpr int PREF_THREADS = 256;

// Grid (pairs, 2), PREF_THREADS threads: block (i, side) writes the per-token CE weights of row i + side * pairs,
// w_t = -(d loss / d s(row)) * mask_t = +-beta * sigma(-z) * inv_pairs under the loss mask (Q8), and block (i, 0) its
// stats row.  Block (0, 0) also sums the pair losses in a fixed order (strided per-thread partials, then the partials in
// thread order): no float atomics, so stats, loss and weights are the same bits in every launch.
__global__ void preference_weights_kernel(const int* __restrict__ labels, const float* __restrict__ seq_ll,
                                          const float* __restrict__ ref_ll, float* __restrict__ w, float* __restrict__ stats,
                                          float* __restrict__ loss, int pairs, int n, float beta, float inv_pairs) {
  const int i = blockIdx.x, side = blockIdx.y;
  const long long row = i + (long long)side * pairs;
  double z, l, sig;
  preference_pair(seq_ll, ref_ll, i, pairs, beta, z, l, sig);
  const float g = (float)((double)beta * sig * (double)inv_pairs);
  const float wv = side == 0 ? g : -g;
  const int* lb = labels + row * n;
  int first, count;
  seq_loss_mask(lb, n, first, count);
  for (int t = threadIdx.x; t < n; t += blockDim.x) w[row * n + t] = (lb[t] != 0 || t == first) ? wv : 0.f;
  if (side == 0 && threadIdx.x == 0) {
    float* st = stats + 4LL * i;
    st[0] = seq_ll[i];
    st[1] = seq_ll[i + pairs];
    st[2] = (float)z;
    st[3] = (float)l;
  }
  if (i == 0 && side == 0) {
    __shared__ double part[PREF_THREADS];
    double acc = 0.0;
    for (int j = threadIdx.x; j < pairs; j += PREF_THREADS) {
      preference_pair(seq_ll, ref_ll, j, pairs, beta, z, l, sig);
      acc += l;
    }
    part[threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int k = 0; k < PREF_THREADS; ++k) s += part[k];
      *loss = (float)(s * (double)inv_pairs);
    }
  }
}

// ------------------------------------------------------------------------------------------ distillation head
// One warp per position t (row b = t / n, position p = t - b n), w_t = inv_batch m_t / c_b from ce_weights_kernel.
// kl[t] = KL_t and ce[t] = CE_t (0 where m_t = 0) and the position's logit gradient, with c_kl = (1 - alpha) tau:
//   dlogits_t = w_t [c_kl (softmax(s / tau) - softmax(z / tau)) + alpha (softmax(s) - onehot(label_t))].
// A masked position writes a zero gradient row and does not read the teacher row.  Every sum runs in a fixed order.
template <typename TL, typename TD>
__global__ void distill_pos_kernel(const TL* __restrict__ logits, const float* __restrict__ teacher, long long stride,
                                   const int* __restrict__ labels, const float* __restrict__ w, float* __restrict__ kl,
                                   float* __restrict__ ce, TD* __restrict__ dlogits, long long T, int n, int V,
                                   float inv_tau, float c_kl, float alpha) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long t = blockIdx.x * (long long)ROWS_PER_BLOCK + warp; t < T; t += (long long)gridDim.x * ROWS_PER_BLOCK) {
    TD* dr = dlogits + t * V;
    const float wt = w[t];
    if (wt == 0.f) {
      const float zero[4] = {0.f, 0.f, 0.f, 0.f};
      for (int c = lane * 4; c < V; c += 128) store4(dr + c, zero);
      if (lane == 0) { kl[t] = 0.f; ce[t] = 0.f; }
      continue;
    }
    const TL* lr = logits + t * V;
    const long long b = t / n;
    const float* zr = teacher + (b * stride + (t - b * n)) * V;
    float ms, se1;
    warp_row_max_sumexp<TL>(lr, V, lane, ms, se1);
    float mz = -INFINITY;
    for (int c = lane * 4; c < V; c += 128) {
      float z[4];
      load4<float>(zr + c, z);
      mz = fmaxf(mz, fmaxf(fmaxf(z[0], z[1]), fmaxf(z[2], z[3])));
    }
    mz = warp_max(mz);
    float ses = 0.f, sez = 0.f;
    for (int c = lane * 4; c < V; c += 128) {
      float s[4], z[4];
      load4<TL>(lr + c, s);
      load4<float>(zr + c, z);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        ses += expf((s[i] - ms) * inv_tau);
        sez += expf((z[i] - mz) * inv_tau);
      }
    }
    ses = warp_sum(ses);
    sez = warp_sum(sez);
    const float lses = logf(ses), lsez = logf(sez), inv1 = 1.f / se1;
    const int lab = clamp_label(labels[t], V);
    float k = 0.f;
    for (int c = lane * 4; c < V; c += 128) {
      float s[4], z[4], o[4];
      load4<TL>(lr + c, s);
      load4<float>(zr + c, z);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float lq = (s[i] - ms) * inv_tau - lses, lp = (z[i] - mz) * inv_tau - lsez;
        const float q = expf(lq), p = expf(lp);
        if (p > 0.f) k += p * (lp - lq);
        o[i] = wt * (c_kl * (q - p) + alpha * (expf(s[i] - ms) * inv1 - ((c + i) == lab ? 1.f : 0.f)));
      }
      store4(dr + c, o);
    }
    k = warp_sum(k);
    if (lane == 0) {
      kl[t] = k;
      ce[t] = (ms + logf(se1)) - to_f32(lr[lab]);
    }
  }
}

constexpr int DISTILL_THREADS = 256;

// One block per row b: stats[b] = (sum_t kl[t], sum_t ce[t]) / c_b, each thread summing positions threadIdx.x + k *
// DISTILL_THREADS ascending in double, then the thread partials in thread order.  Positions past a cut view hold zeros
// in the full-length view, so a cut and the full view give the same bits.
__global__ void distill_row_kernel(const int* __restrict__ labels, const float* __restrict__ kl, const float* __restrict__ ce,
                                   float* __restrict__ stats, int n) {
  const int b = blockIdx.x;
  int first, count;
  seq_loss_mask(labels + (long long)b * n, n, first, count);
  double a = 0.0, c = 0.0;
  for (int i = threadIdx.x; i < n; i += DISTILL_THREADS) {
    a += (double)kl[(long long)b * n + i];
    c += (double)ce[(long long)b * n + i];
  }
  __shared__ double ra[DISTILL_THREADS], rc[DISTILL_THREADS];
  ra[threadIdx.x] = a;
  rc[threadIdx.x] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    double sa = 0.0, sc = 0.0;
    for (int k = 0; k < DISTILL_THREADS; ++k) { sa += ra[k]; sc += rc[k]; }
    stats[2LL * b] = (float)(sa / (double)count);
    stats[2LL * b + 1] = (float)(sc / (double)count);
  }
}

// *loss = inv_batch * sum_b [(1 - alpha) tau^2 KL_b + alpha CE_b], one thread, rows in order, in double
__global__ void distill_loss_kernel(const float* __restrict__ stats, int B, double c_kl2, double alpha, double inv_batch,
                                    float* __restrict__ loss) {
  double s = 0.0;
  for (int b = 0; b < B; ++b) s += c_kl2 * (double)stats[2LL * b] + alpha * (double)stats[2LL * b + 1];
  *loss = (float)(s * inv_batch);
}

// ------------------------------------------------------------------------------------------ policy-gradient head
// The span of row b clamped to [0, n]: positions lo <= p < hi count, N_b = hi - lo (0 when the span is empty).
__device__ __forceinline__ void policy_span(const int* __restrict__ span, long long b, int n, int& lo, int& hi) {
  lo = min(max(span[2 * b], 0), n);
  hi = min(max(span[2 * b + 1], lo), n);
}

// One warp per position t (row b = t / n, position p = t - b n).  Outside the span the gradient row is +0.0 and
// logp[t] = kl[t] = 0; the reference row is read only inside it, and only when REF (beta > 0).  Inside, with
// lpi = log_softmax(s_t), lrho = log_softmax(z_t), pi = softmax(s_t) computed as ce_fwd_bwd_kernel does (so beta = 0,
// A = 1 gives its gradient bits) and KL_t = sum_v pi_v (lpi_v - lrho_v) (0 where pi_v = 0):
//   dlogits_t = inv_rows / N_b [A_b (pi - onehot(label_t)) + beta pi (lpi - lrho - KL_t)].
// The reference's log-softmax runs through the same code as the policy's, so z = s gives lrho = lpi bitwise.
template <typename TL, typename TD, bool REF>
__global__ void policy_pos_kernel(const TL* __restrict__ logits, const float* __restrict__ ref, long long stride,
                                  const int* __restrict__ labels, const int* __restrict__ span,
                                  const float* __restrict__ adv, float* __restrict__ logp, float* __restrict__ kl,
                                  TD* __restrict__ dlogits, long long T, int n, int V, float beta, float inv_rows) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long t = blockIdx.x * (long long)ROWS_PER_BLOCK + warp; t < T; t += (long long)gridDim.x * ROWS_PER_BLOCK) {
    TD* dr = dlogits + t * V;
    const long long b = t / n;
    const int p = (int)(t - b * n);
    int lo, hi;
    policy_span(span, b, n, lo, hi);
    if (p < lo || p >= hi) {
      const float zero[4] = {0.f, 0.f, 0.f, 0.f};
      for (int c = lane * 4; c < V; c += 128) store4(dr + c, zero);
      if (lane == 0) { logp[t] = 0.f; kl[t] = 0.f; }
      continue;
    }
    const float w = inv_rows / (float)(hi - lo), A = adv[b];
    const TL* lr = logits + t * V;
    float ms, ses;
    warp_row_max_sumexp<TL>(lr, V, lane, ms, ses);
    const float lses = logf(ses), inv = 1.f / ses;
    const int lab = clamp_label(labels[t], V);
    const float* zr = REF ? ref + (b * stride + p) * V : nullptr;
    float mz = 0.f, lsez = 0.f, k = 0.f;
    if (REF) {
      float sez;
      warp_row_max_sumexp<float>(zr, V, lane, mz, sez);
      lsez = logf(sez);
      for (int c = lane * 4; c < V; c += 128) {
        float s[4], z[4];
        load4<TL>(lr + c, s);
        load4<float>(zr + c, z);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float pi = expf(s[i] - ms) * inv;
          if (pi > 0.f) k += pi * (((s[i] - ms) - lses) - ((z[i] - mz) - lsez));
        }
      }
      k = warp_sum(k);
    }
    for (int c = lane * 4; c < V; c += 128) {
      float s[4], z[4] = {0.f, 0.f, 0.f, 0.f}, o[4];
      load4<TL>(lr + c, s);
      if (REF) load4<float>(zr + c, z);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float pi = expf(s[i] - ms) * inv;
        float g = A * (pi - ((c + i) == lab ? 1.f : 0.f));
        if (REF) g += beta * (pi * ((((s[i] - ms) - lses) - ((z[i] - mz) - lsez)) - k));
        o[i] = w * g;
      }
      store4(dr + c, o);
    }
    if (lane == 0) {
      logp[t] = (to_f32(lr[lab]) - ms) - lses;
      kl[t] = k;
    }
  }
}

constexpr int POLICY_THREADS = 256;

// One block per row b: stats[b] = (sum logp / N_b, sum KL / N_b, N_b) over the row's span, thread i summing positions
// lo + i + k * POLICY_THREADS ascending in double, then the thread partials in thread order.  The order depends on the
// span alone, so a cut view and the full view, or the row alone and in a batch, give the same bits.
__global__ void policy_row_kernel(const int* __restrict__ span, const float* __restrict__ logp,
                                  const float* __restrict__ kl, float* __restrict__ stats, int n) {
  const int b = blockIdx.x;
  int lo, hi;
  policy_span(span, b, n, lo, hi);
  double a = 0.0, c = 0.0;
  for (int i = lo + threadIdx.x; i < hi; i += POLICY_THREADS) {
    a += (double)logp[(long long)b * n + i];
    c += (double)kl[(long long)b * n + i];
  }
  __shared__ double ra[POLICY_THREADS], rc[POLICY_THREADS];
  ra[threadIdx.x] = a;
  rc[threadIdx.x] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    double sa = 0.0, sc = 0.0;
    for (int k = 0; k < POLICY_THREADS; ++k) { sa += ra[k]; sc += rc[k]; }
    const int N = hi - lo;
    stats[3LL * b] = N ? (float)(sa / (double)N) : 0.f;
    stats[3LL * b + 1] = N ? (float)(sc / (double)N) : 0.f;
    stats[3LL * b + 2] = (float)N;
  }
}

// *loss = inv_rows * sum_b (-A_b logp_b + beta KL_b), one thread, rows in order, in double
__global__ void policy_loss_kernel(const float* __restrict__ stats, const float* __restrict__ adv, int B, double beta,
                                   double inv_rows, float* __restrict__ loss) {
  double s = 0.0;
  for (int b = 0; b < B; ++b) s += -(double)adv[b] * (double)stats[3LL * b] + beta * (double)stats[3LL * b + 1];
  *loss = (float)(s * inv_rows);
}

// out[b, :] = sum_t mask_t x[b, t, :] / sum_t mask_t.  Grid (ceil(d / 128), B), 256 threads: lane owns 4 columns, warp w sums
// rows t = w, w + 8, ... in order, then the 8 warp partials are added in order: fixed order, fp32 accumulation.
template <typename TX>
__global__ void masked_mean_pool_kernel(const TX* __restrict__ x, long long ldx, const int* __restrict__ labels,
                                        float* __restrict__ out, int n, int d) {
  __shared__ float part[ROWS_PER_BLOCK][128];
  const int b = blockIdx.y;
  const int* lb = labels + (long long)b * n;
  int first, count;
  seq_loss_mask(lb, n, first, count);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.x * 128 + lane * 4;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  if (c < d) {
    for (int t = warp; t < n; t += ROWS_PER_BLOCK) {
      if (lb[t] == 0 && t != first) continue;
      float v[4];
      load4<TX>(x + ((long long)b * n + t) * ldx + c, v);
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] += v[i];
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) part[warp][lane * 4 + i] = acc[i];
  __syncthreads();
  if (threadIdx.x < 128 && blockIdx.x * 128 + (int)threadIdx.x < d) {
    float s = 0.f;
    for (int w = 0; w < ROWS_PER_BLOCK; ++w) s += part[w][threadIdx.x];
    out[(long long)b * d + blockIdx.x * 128 + threadIdx.x] = s / (float)count;
  }
}

// Backward of the pool: dy[b, t, :] = demb[b, :] / count_b at the positions the mask counts, 0 at every other position of
// row b.  Grid (ceil(n / POOL_BWD_ROWS), B), 256 threads: warp w writes positions w, w + 8, ... of the block's slice, lane
// 4 columns at a time.  Every row is written, so dy needs no memset.
constexpr int POOL_BWD_ROWS = 64;

template <typename TO>
__global__ void masked_mean_pool_bwd_kernel(const float* __restrict__ demb, const int* __restrict__ labels,
                                            TO* __restrict__ dy, long long ldy, int n, int d) {
  const int b = blockIdx.y;
  const int* lb = labels + (long long)b * n;
  int first, count;
  seq_loss_mask(lb, n, first, count);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* g = demb + (long long)b * d;
  const int t1 = min(n, (blockIdx.x + 1) * POOL_BWD_ROWS);
  for (int t = blockIdx.x * POOL_BWD_ROWS + warp; t < t1; t += ROWS_PER_BLOCK) {
    const bool on = lb[t] != 0 || t == first;
    TO* row = dy + ((long long)b * n + t) * ldy;
    for (int c = lane * 4; c < d; c += 128) {
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (on) {
        load4<float>(g + c, v);
#pragma unroll
        for (int i = 0; i < 4; ++i) v[i] = v[i] / (float)count;
      }
      store4(row + c, v);
    }
  }
}

// ------------------------------------------------------------------------------------------ property head
// p[b, :] = emb[b, :] W + bias (W [d, C] row-major, C <= PROGEN_PROPERTY_MAX_OUTPUTS).  One 256-thread block per row: thread
// t owns output c = t % 64 and the k-slice t / 64 (k = slice, slice + 4, ...), so a warp reads whole rows of W; the four
// slice partials are added in slice order.  Then thread 0 computes the row's loss and d p (fixed order over c): regression
// loss_b = sum_c (p - y)^2 / C, d p = 2 (p - y) / C * inv_batch; classification loss_b = lse(p) - p[y], d p = (softmax(p)
// - onehot(y)) * inv_batch.  Finally demb[b, k] = sum_c dp_c W[k, c] in c order.  With y and cls null only p is written.
constexpr int HEAD_THREADS = 256;
constexpr int HEAD_COLS = 64;
constexpr int HEAD_SLICES = HEAD_THREADS / HEAD_COLS;
static_assert(HEAD_COLS == PROGEN_PROPERTY_MAX_OUTPUTS, "one thread column per head output");

__global__ void property_head_rows_kernel(const float* __restrict__ emb, const float* __restrict__ w,
                                          const float* __restrict__ bias, int d, int C, int task,
                                          const float* __restrict__ y, const int* __restrict__ cls, float inv_batch,
                                          float* __restrict__ pred, float* __restrict__ row_loss,
                                          float* __restrict__ dpred, float* __restrict__ demb) {
  __shared__ float part[HEAD_SLICES][HEAD_COLS];
  __shared__ float p[HEAD_COLS], dp[HEAD_COLS];
  const int b = blockIdx.x;
  const int c = threadIdx.x % HEAD_COLS, slice = threadIdx.x / HEAD_COLS;
  const float* e = emb + (long long)b * d;
  float acc = 0.f;
  if (c < C)
    for (int k = slice; k < d; k += HEAD_SLICES) acc = fmaf(e[k], w[(long long)k * C + c], acc);
  part[slice][c] = acc;
  __syncthreads();
  if (threadIdx.x < C) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < HEAD_SLICES; ++i) s += part[i][threadIdx.x];
    s += bias[threadIdx.x];
    p[threadIdx.x] = s;
    pred[(long long)b * C + threadIdx.x] = s;
  }
  if (y == nullptr && cls == nullptr) return;
  __syncthreads();
  if (threadIdx.x == 0) {
    float l = 0.f;
    if (task == PROGEN_TASK_REGRESSION) {
      const float* yb = y + (long long)b * C;
      for (int j = 0; j < C; ++j) {
        const float r = p[j] - yb[j];
        l += r * r;
        dp[j] = 2.f * r / (float)C * inv_batch;
      }
      l /= (float)C;
    } else {
      const int t = min(max(cls[b], 0), C - 1);
      float mx = -INFINITY;
      for (int j = 0; j < C; ++j) mx = fmaxf(mx, p[j]);
      float se = 0.f;
      for (int j = 0; j < C; ++j) se += expf(p[j] - mx);
      l = mx + logf(se) - p[t];
      const float inv = 1.f / se;
      for (int j = 0; j < C; ++j) dp[j] = (expf(p[j] - mx) * inv - (j == t ? 1.f : 0.f)) * inv_batch;
    }
    row_loss[b] = l;
  }
  __syncthreads();
  if (threadIdx.x < C) dpred[(long long)b * C + threadIdx.x] = dp[threadIdx.x];
  for (int k = threadIdx.x; k < d; k += HEAD_THREADS) {
    const float* wk = w + (long long)k * C;
    float s = 0.f;
    for (int j = 0; j < C; ++j) s = fmaf(dp[j], wk[j], s);
    demb[(long long)b * d + k] = s;
  }
}

// dW[k, c] = sum_b emb[b, k] dp[b, c], one thread per (k, c), rows b in order; the last block writes db[c] = sum_b dp[b, c]
// (threads c < C) and loss = inv_batch * sum_b loss_b (thread C, in double).  Written, not accumulated; no atomics.
__global__ void property_head_params_kernel(const float* __restrict__ emb, const float* __restrict__ dpred,
                                            const float* __restrict__ row_loss, int B, int d, int C, float inv_batch,
                                            float* __restrict__ dw, float* __restrict__ db, float* __restrict__ loss) {
  const long long dc = (long long)d * C;
  if (blockIdx.x == gridDim.x - 1) {
    const int c = threadIdx.x;
    if (c < C) {
      float s = 0.f;
      for (int b = 0; b < B; ++b) s += dpred[(long long)b * C + c];
      db[c] = s;
    } else if (c == C) {
      double s = 0.0;
      for (int b = 0; b < B; ++b) s += (double)row_loss[b];
      *loss = (float)(s * (double)inv_batch);
    }
    return;
  }
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= dc) return;
  const int k = (int)(i / C), c = (int)(i % C);
  float s = 0.f;
  for (int b = 0; b < B; ++b) s = fmaf(emb[(long long)b * d + k], dpred[(long long)b * C + c], s);
  dw[i] = s;
}

// ------------------------------------------------------------------------------------------ residue (per-position) head
// The property head applied at every position of a [B*L, d] view of the final LayerNorm output (DESIGN.md §3.11).  A position
// is labelled when its target is: class index >= 0 (classification), a non-NaN first value (regression; the host refuses a
// partly-NaN position).  Every sum below runs in a fixed order that depends on neither the other rows nor the row length L.
constexpr int RES_MAX_ROWS = 4096;    // rows of one training launch: per-row partials of the count and the loss in shared memory

__device__ __forceinline__ bool residue_labelled(const float* y, const int* cls, long long pos, int C) {
  return cls != nullptr ? cls[pos] >= 0 : !isnan(y[pos * C]);
}

// *count = number of labelled positions: row b's count by one thread, then the row counts in row order by thread 0.
__global__ void residue_count_kernel(const float* __restrict__ y, const int* __restrict__ cls, int B, int L, int C,
                                     int* __restrict__ count) {
  __shared__ int rc[RES_MAX_ROWS];
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    int s = 0;
    for (int t = 0; t < L; ++t) s += residue_labelled(y, cls, (long long)b * L + t, C) ? 1 : 0;
    rc[b] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int b = 0; b < B; ++b) s += rc[b];
    *count = s;
  }
}

// One warp per position, 8 positions per 256-thread block, grid-stride.  Lane l owns the columns k = 4l + 128j: it sums
// h[k] W[k, c] over its columns in ascending k, then an xor butterfly adds the 32 lane partials (every lane ends with the
// same bits), then + bias[c].  Training: every lane computes the position's loss and d p from those bits (regression
// loss = sum_c (p - y)^2 / C, d p = 2 (p - y) / C / N; classification loss = lse(p) - p[y], d p = (softmax(p) -
// onehot(y)) / N, N = *count), and dy[k] = sum_c dp_c W[k, c] in c order for its own columns.  An unlabelled position
// gets loss 0, d p 0 and dy +0.0, so every row of dy is written.  CT: the compile-time bound of C (registers).
template <typename TH, int CT>
__global__ void residue_head_kernel(const TH* __restrict__ h, long long ldh, const float* __restrict__ w,
                                    const float* __restrict__ bias, long long rows, int d, int C, int task,
                                    const float* __restrict__ y, const int* __restrict__ cls, const int* __restrict__ count,
                                    float* __restrict__ pred, float* __restrict__ pos_loss, float* __restrict__ dpred,
                                    TH* __restrict__ dy, long long ldy) {
  const int lane = threadIdx.x & 31;
  const bool train = y != nullptr || cls != nullptr;
  const float inv_n = train ? 1.f / (float)max(*count, 1) : 0.f;
  for (long long pos = (long long)blockIdx.x * ROWS_PER_BLOCK + (threadIdx.x >> 5); pos < rows;
       pos += (long long)gridDim.x * ROWS_PER_BLOCK) {
    const TH* hr = h + pos * ldh;
    float acc[CT];
#pragma unroll
    for (int c = 0; c < CT; ++c) acc[c] = 0.f;
    for (int k = lane * 4; k < d; k += 128) {
      float v[4];
      load4<TH>(hr + k, v);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float* wk = w + (long long)(k + i) * C;
#pragma unroll
        for (int c = 0; c < CT; ++c)
          if (c < C) acc[c] = fmaf(v[i], wk[c], acc[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < CT; ++c) {
      if (c < C) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], off);
        acc[c] += bias[c];
        if ((c & 31) == lane) pred[pos * C + c] = acc[c];
      }
    }
    if (!train) continue;
    const bool lab = residue_labelled(y, cls, pos, C);
    float l = 0.f;
    if (lab && task == PROGEN_TASK_REGRESSION) {
      const float* yp = y + pos * C;
#pragma unroll
      for (int c = 0; c < CT; ++c) {
        if (c < C) {
          const float r = acc[c] - yp[c];
          l += r * r;
          acc[c] = 2.f * r / (float)C * inv_n;
        }
      }
      l /= (float)C;
    } else if (lab) {
      const int yc = min(max(cls[pos], 0), C - 1);
      float mx = -INFINITY, py = 0.f;
#pragma unroll
      for (int c = 0; c < CT; ++c) {
        if (c < C) {
          mx = fmaxf(mx, acc[c]);
          if (c == yc) py = acc[c];
        }
      }
      float se = 0.f;
#pragma unroll
      for (int c = 0; c < CT; ++c)
        if (c < C) se += expf(acc[c] - mx);
      l = mx + logf(se) - py;
      const float inv = 1.f / se;
#pragma unroll
      for (int c = 0; c < CT; ++c)
        if (c < C) acc[c] = (expf(acc[c] - mx) * inv - (c == yc ? 1.f : 0.f)) * inv_n;
    }
    if (lane == 0) pos_loss[pos] = l;
#pragma unroll
    for (int c = 0; c < CT; ++c)
      if (c < C && (c & 31) == lane) dpred[pos * C + c] = lab ? acc[c] : 0.f;
    TH* dr = dy + pos * ldy;
    for (int k = lane * 4; k < d; k += 128) {
      float s[4] = {0.f, 0.f, 0.f, 0.f};
      if (lab) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float* wk = w + (long long)(k + i) * C;
#pragma unroll
          for (int c = 0; c < CT; ++c)
            if (c < C) s[i] = fmaf(acc[c], wk[c], s[i]);
        }
      }
      store4(dr + k, s);
    }
  }
}

// *loss = sum over labelled positions of pos_loss / N: row b's sum (positions ascending, in double) by one thread, then
// the row sums in row order by thread 0.
__global__ void residue_loss_kernel(const float* __restrict__ pos_loss, const float* __restrict__ y,
                                    const int* __restrict__ cls, const int* __restrict__ count, int B, int L, int C,
                                    float* __restrict__ loss) {
  __shared__ double rs[RES_MAX_ROWS];
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    double s = 0.0;
    for (int t = 0; t < L; ++t) {
      const long long pos = (long long)b * L + t;
      if (residue_labelled(y, cls, pos, C)) s += (double)pos_loss[pos];
    }
    rs[b] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int b = 0; b < B; ++b) s += rs[b];
    *loss = (float)(s / (double)max(*count, 1));
  }
}

// Stage 1 of the head's weight gradient: one thread per (row b, i = k C + c), i < (d + 1) C, k == d standing for the bias:
// ws[b, i] = sum over the labelled positions t of row b, ascending, of h[b, t, k] dp[b, t, c] (the bias: dp[b, t, c]).
// Unlabelled positions are skipped.  Loads run four positions ahead of the sequential sum.
template <typename TH>
__global__ void residue_wgrad_rows_kernel(const TH* __restrict__ h, long long ldh, const float* __restrict__ dpred,
                                          const float* __restrict__ y, const int* __restrict__ cls, int L, int d, int C,
                                          float* __restrict__ ws) {
  const long long dc1 = (long long)(d + 1) * C;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= dc1) return;
  const int b = blockIdx.y;
  const int k = (int)(i / C), c = (int)(i % C);
  const bool is_bias = k == d;
  const long long p0 = (long long)b * L;
  float s = 0.f;
  int t = 0;
  for (; t + 4 <= L; t += 4) {
    bool lab[4];
    float hv[4], dv[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long pos = p0 + t + j;
      lab[j] = residue_labelled(y, cls, pos, C);
      hv[j] = is_bias ? 1.f : to_f32(h[pos * ldh + k]);
      dv[j] = dpred[pos * C + c];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (lab[j]) s = is_bias ? s + dv[j] : fmaf(hv[j], dv[j], s);
  }
  for (; t < L; ++t) {
    const long long pos = p0 + t;
    if (!residue_labelled(y, cls, pos, C)) continue;
    const float dv = dpred[pos * C + c];
    s = is_bias ? s + dv : fmaf(to_f32(h[pos * ldh + k]), dv, s);
  }
  ws[(long long)b * dc1 + i] = s;
}

// Stage 2: dW[k, c] (and db[c]) = sum_b ws[b, i] in row order.  Written, not accumulated.
__global__ void residue_wgrad_reduce_kernel(const float* __restrict__ ws, int B, int d, int C, float* __restrict__ dw,
                                            float* __restrict__ db) {
  const long long dc = (long long)d * C, dc1 = dc + C;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= dc1) return;
  float s = 0.f;
  for (int b = 0; b < B; ++b) s += ws[(long long)b * dc1 + i];
  if (i < dc) dw[i] = s;
  else db[i - dc] = s;
}

// ------------------------------------------------------------------------------------------ rotary backward
// forward (GEMM epilogue): o0 = x0 c - x1 s, o1 = x1 c + x0 s  =>  dx0 = d0 c + d1 s, dx1 = d1 c - d0 s.  In place.
template <typename TO>
__global__ void rotary_bwd_kernel(TO* __restrict__ dqkv, long long ld, const float* __restrict__ sin_t,
                                  const float* __restrict__ cos_t, long long T, int ncols, int seq_len, int dim_head) {
  const long long total = T * (ncols / 4);
  const int half = dim_head >> 1;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / (ncols / 4);
    const int c = (int)(i % (ncols / 4)) * 4;
    const int pos = (int)(t % seq_len);
    float v[4], o[4];
    load4<TO>(dqkv + t * ld + c, v);
#pragma unroll
    for (int p = 0; p < 4; p += 2) {
      const int j = ((c + p) % dim_head) >> 1;
      const float s = __ldg(sin_t + (long long)pos * half + j), cs = __ldg(cos_t + (long long)pos * half + j);
      o[p] = v[p] * cs + v[p + 1] * s;
      o[p + 1] = v[p + 1] * cs - v[p] * s;
    }
    store4(dqkv + t * ld + c, o);
  }
}

// ------------------------------------------------------------------------------------------ SGU gating
// reference progen.py:181-184: gate = (W o tril) @ LN(gate) + bias[m];  x = x * gate.   Gp is the GEMM output (no bias).
template <typename TO>
__global__ void sgu_gate_fwd_kernel(const TO* __restrict__ xs, long long ldx, const TO* __restrict__ gp, long long ldg,
                                    const float* __restrict__ bias, TO* __restrict__ out, long long ldo, long long T, int C,
                                    int seq_len) {
  const long long total = T * (C / 4);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / (C / 4);
    const int c = (int)(i % (C / 4)) * 4;
    const float b = __ldg(bias + (t % seq_len));
    float x[4], g[4], o[4];
    load4<TO>(xs + t * ldx + c, x);
    load4<TO>(gp + t * ldg + c, g);
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = x[j] * (g[j] + b);
    store4(out + t * ldo + c, o);
  }
}

// d(xs) = ds * (Gp + bias) ; d(Gp) = ds * xs ; dbias[m] += sum_c d(Gp).  One warp per row.
template <typename TO>
__global__ void sgu_gate_bwd_kernel(const TO* __restrict__ ds, long long ldds, const TO* __restrict__ xs, long long ldx,
                                    const TO* __restrict__ gp, long long ldg, const float* __restrict__ bias,
                                    TO* __restrict__ dxs, long long lddx, TO* __restrict__ dgp, long long lddg,
                                    float* __restrict__ dbias, long long T, int C, int seq_len) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long t = blockIdx.x * (long long)ROWS_PER_BLOCK + warp; t < T; t += (long long)gridDim.x * ROWS_PER_BLOCK) {
    const int m = (int)(t % seq_len);
    const float b = __ldg(bias + m);
    float acc = 0.f;
    for (int c = lane * 4; c < C; c += 128) {
      float d[4], x[4], g[4], o1[4], o2[4];
      load4<TO>(ds + t * ldds + c, d);
      load4<TO>(xs + t * ldx + c, x);
      load4<TO>(gp + t * ldg + c, g);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        o1[j] = d[j] * (g[j] + b);
        o2[j] = d[j] * x[j];
        acc += o2[j];
      }
      store4(dxs + t * lddx + c, o1);
      store4(dgp + t * lddg + c, o2);
    }
    acc = warp_sum(acc);
    if (lane == 0 && dbias) atomicAdd(dbias + m, acc);      // dbias nullable: frozen spatial biases
  }
}

// du = da * gelu'(u)   (SGU layers: proj_in -> gelu, progen.py:143), in place on da
template <typename TO>
__global__ void gelu_bwd_kernel(TO* __restrict__ da, const TO* __restrict__ u, long long total4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
    float d[4], x[4];
    load4<TO>(da + i * 4, d);
    load4<TO>(u + i * 4, x);
#pragma unroll
    for (int j = 0; j < 4; ++j) d[j] *= gelu_tanh_grad(x[j]);
    store4(da + i * 4, d);
  }
}

// fp32 -> act dtype copy (used to hand the residual-stream gradient to the GEMMs)
template <typename TO>
__global__ void cast_kernel(const float* __restrict__ in, TO* __restrict__ out, long long total4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
    float v[4];
    load4<float>(in + i * 4, v);
    store4(out + i * 4, v);
  }
}

// out = scale * in: a low-rank adapter's scaled compute copy (s B) and its scaled gradient (in place for fp32)
template <typename TO>
__global__ void scale_cast_kernel(const float* in, TO* out, float scale, long long total4) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
    float v[4];
    load4<float>(in + i * 4, v);
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] *= scale;
    store4(out + i * 4, v);
  }
}

// masked compute copy of the SGU spatial weights: out = tril(w)  (reference progen.py:178-179), cast to the act dtype
template <typename TO>
__global__ void tril_cast_kernel(const float* __restrict__ w, TO* __restrict__ out, int n) {
  const long long total = (long long)n * (n / 4);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / (n / 4));
    const int c = (int)(i % (n / 4)) * 4;
    float v[4];
    load4<float>(w + (long long)r * n + c, v);
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = (c + j <= r) ? v[j] : 0.f;
    store4(out + (long long)r * n + c, v);
  }
}

// ------------------------------------------------------------------------------------------ decoder weight refresh
// The engine keeps a GLU feed-forward input's columns interleaved (v0, g0, v1, g1, ...); the decoder keeps haiku's
// (value | gate).  Column o of the decoder's leaf is column glu_col(o) of the engine's.
__device__ __forceinline__ long long glu_col(long long o, long long out, int interleave) {
  if (!interleave) return o;
  const long long H = out >> 1;
  return o < H ? 2 * o : 2 * (o - H) + 1;
}

constexpr int LW_TILE = 32, LW_MAX_RANK = 64;

// dst[o, i] = cast(W[i, c(o)] + s * sum_r A[i, r] B[r, c(o)]) over one 32 x 32 tile of (i, o) per 256-thread block: W, A
// and B tiles staged in shared memory, the transposed tile written along i.  r runs in increasing order and every
// product and sum is rounded on its own (no FMA), so a float32 host replay gives the same bits; rank 0 is a copy.
template <typename TD>
__global__ void load_weight_kernel(const float* __restrict__ W, const float* __restrict__ A, const float* __restrict__ Bm,
                                   int rank, float scale, int in, int out, int interleave, TD* __restrict__ dst) {
  __shared__ float ws[LW_TILE][LW_TILE + 1];
  __shared__ float as[LW_TILE][LW_MAX_RANK + 1];
  __shared__ float bs[LW_MAX_RANK][LW_TILE];
  const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * LW_TILE + tx;
  const int i0 = blockIdx.x * LW_TILE, o0 = blockIdx.y * LW_TILE;
  for (int ii = ty; ii < LW_TILE; ii += 8) {
    const int i = i0 + ii, o = o0 + tx;
    ws[ii][tx] = (i < in && o < out) ? W[(long long)i * out + glu_col(o, out, interleave)] : 0.f;
  }
  for (int k = tid; k < LW_TILE * rank; k += 256) {
    const int ii = k / rank, r = k - ii * rank, i = i0 + ii;
    as[ii][r] = i < in ? A[(long long)i * rank + r] : 0.f;
  }
  for (int k = tid; k < rank * LW_TILE; k += 256) {
    const int r = k / LW_TILE, oo = k - r * LW_TILE, o = o0 + oo;
    bs[r][oo] = o < out ? Bm[(long long)r * out + glu_col(o, out, interleave)] : 0.f;
  }
  __syncthreads();
  const int i = i0 + tx;
  if (i >= in) return;
  for (int oo = ty; oo < LW_TILE; oo += 8) {
    const int o = o0 + oo;
    if (o >= out) break;
    float v = ws[tx][oo];
    if (rank) {
      float acc = 0.f;
      for (int r = 0; r < rank; ++r) acc = __fadd_rn(acc, __fmul_rn(as[tx][r], bs[r][oo]));
      v = __fadd_rn(v, __fmul_rn(scale, acc));
    }
    dst[(long long)o * in + i] = from_f32<TD>(v);
  }
}

// a vector leaf (in = 1): dst[o] = cast(W[c(o)])
template <typename TD>
__global__ void load_vector_kernel(const float* __restrict__ W, long long out, int interleave, TD* __restrict__ dst) {
  for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < out; o += (long long)gridDim.x * blockDim.x)
    dst[o] = from_f32<TD>(W[glu_col(o, out, interleave)]);
}

// decoder-cache prefill: dst[b, g, r, c] = fp32(src[(row_map[b] * src_seq_rows + row0 + r) * ld + col0 + g * cols + c]).
// One thread moves 16 source bytes (4 fp32 or 8 bf16) to 16 or 32 destination bytes; consecutive threads take consecutive
// column vectors of a row, so both sides coalesce.  The source (one forward row per distinct prompt) is read once per
// decoder row that maps to it; the fp32 caches written are the bulk of the traffic.
template <typename TI>
__global__ void gather_rows_f32_kernel(const TI* __restrict__ src, long long ld, const int* __restrict__ row_map, int src_seqs,
                                       long long src_seq_rows, int row0, int rows, int col0, int groups, int cols,
                                       float* __restrict__ dst, long long dst_b, long long dst_g, long long dst_r,
                                       long long total) {
  constexpr int NV = 16 / sizeof(TI);
  const int cv = cols / NV;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) * NV;
    long long t = i / cv;
    const int r = (int)(t % rows);
    t /= rows;
    const int g = (int)(t % groups);
    const int b = (int)(t / groups);
    int s = row_map[b];
    s = s < 0 ? 0 : (s >= src_seqs ? src_seqs - 1 : s);
    float v[NV];
    load_vec<NV>(src + (s * src_seq_rows + row0 + r) * ld + col0 + (long long)g * cols + c, v);
    store_vec<NV>(dst + b * dst_b + g * dst_g + r * dst_r + c, v);
  }
}

inline int ew_grid(long long work_items, int threads) {
  long long b = (work_items + threads - 1) / threads;
  const long long cap = (long long)pg_num_sms() * 8;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}
inline int row_grid(long long T) {
  long long b = (T + ROWS_PER_BLOCK - 1) / ROWS_PER_BLOCK;
  const long long cap = (long long)pg_num_sms() * 4;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

// =========================================================================================== C ABI
extern "C" {

int progen_embed_fwd(const int* tokens, const float* table, float* x, long long T, int d, int V, void* stream) {
  PG_CHECK_ARG(T > 0 && d % 4 == 0 && V > 0);
  embed_fwd_kernel<<<ew_grid(T * (d / 4), 256), 256, 0, (cudaStream_t)stream>>>(tokens, table, x, T, d, V);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_embed_bwd(const int* tokens, const float* dx, float* dtable, long long T, int d, int V, void* stream) {
  PG_CHECK_ARG(T > 0 && d > 0 && V > 0 && V * 32 * 4 <= 48 * 1024);
  const int row_blocks = (int)((T + 4095) / 4096);
  const long long rpb = (T + row_blocks - 1) / row_blocks;
  dim3 grid((d + 31) / 32, row_blocks);
  embed_bwd_kernel<<<grid, 256, V * 32 * sizeof(float), (cudaStream_t)stream>>>(tokens, dx, dtable, T, d, V, rpb);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_ln_shift_fwd(const void* x, long long ldx, int x_dtype, const float* scale, void* y, long long ldy, int y_dtype,
                        float* mean, float* rstd, long long T, int d, int seq_len, int shift, void* stream) {
  PG_CHECK_ARG(T > 0 && d % 8 == 0 && seq_len > 0 && T % seq_len == 0);
  PG_CHECK_ARG(ldx % 4 == 0 && ldy % 4 == 0);
  cudaStream_t s = (cudaStream_t)stream;
  const int grid = row_grid(T);
#define LN_FWD(TI, TO) ln_shift_fwd_kernel<TI, TO><<<grid, 256, 0, s>>>((const TI*)x, ldx, scale, (TO*)y, ldy, mean, rstd, T, d, seq_len, shift)
  if (x_dtype == PG_F32 && y_dtype == PG_F32) LN_FWD(float, float);
  else if (x_dtype == PG_F32 && y_dtype == PG_BF16) LN_FWD(float, bf16);
  else if (x_dtype == PG_BF16 && y_dtype == PG_BF16) LN_FWD(bf16, bf16);
  else { progen_set_error("ln_shift_fwd: unsupported dtypes %d -> %d", x_dtype, y_dtype); return PROGEN_ERR_UNSUPPORTED; }
#undef LN_FWD
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

// residual != 0: dres(fp32, [T,d]) += dx, and `dout` (may be null) receives a copy of the updated dres in act dtype.
// residual == 0: dout[t*ldo + c] = dx.
int progen_ln_shift_bwd(const void* dy, long long lddy, int act_dtype, const void* x, long long ldx, int x_dtype,
                        const float* scale, const float* mean, const float* rstd, float* dres, void* dout, long long ldo,
                        float* dscale, float* dres_colsum, long long T, int d, int seq_len, int shift, int residual,
                        void* stream) {
  PG_CHECK_ARG(T > 0 && d % 8 == 0 && d <= 4096 && seq_len > 0 && T % seq_len == 0);
  PG_CHECK_ARG(residual ? (dres != nullptr && x_dtype == PG_F32) : (dout != nullptr));
  cudaStream_t s = (cudaStream_t)stream;
  // bulk-copy streaming kernel (ln_stream.cu) for the shapes it covers; 1 = not eligible -> row-per-warp kernel below
  const int rc_stream = ln_shift_bwd_stream_launch(dy, lddy, act_dtype, x, ldx, x_dtype, scale, mean, rstd, dres, dout, ldo,
                                                   dscale, dres_colsum, T, d, seq_len, shift, residual, s);
  if (rc_stream <= 0) return rc_stream;
  long long b = (T + ROWS_PER_BLOCK - 1) / ROWS_PER_BLOCK;
  // row-per-warp with two dependent passes is latency-bound: keep several CTAs resident per SM (grid = k * #SMs)
  const int per_sm = d <= 1024 ? 6 : 3;
  const int grid = (int)(b > pg_num_sms() * per_sm ? pg_num_sms() * per_sm : b);
  const int nch = (d + 127) / 128;
#define LN_BWD_N(TI, TO, NCH, RES) ln_shift_bwd_kernel<TI, TO, NCH, RES><<<grid, 256, 0, s>>>((const TO*)dy, lddy, (const TI*)x, ldx, scale, mean, rstd, dres, (TO*)dout, ldo, dscale, dres_colsum, T, d, seq_len, shift)
#define LN_BWD(TI, TO, RES) do { if (nch <= 4) LN_BWD_N(TI, TO, 4, RES); else if (nch <= 8) LN_BWD_N(TI, TO, 8, RES); \
    else if (nch <= 16) LN_BWD_N(TI, TO, 16, RES); else LN_BWD_N(TI, TO, 32, RES); } while (0)
  if (residual) {
    if (act_dtype == PG_F32) LN_BWD(float, float, true);
    else LN_BWD(float, bf16, true);
  } else {
    if (act_dtype == PG_F32 && x_dtype == PG_F32) LN_BWD(float, float, false);
    else if (act_dtype == PG_BF16 && x_dtype == PG_BF16) LN_BWD(bf16, bf16, false);
    else if (act_dtype == PG_BF16 && x_dtype == PG_F32) LN_BWD(float, bf16, false);
    else { progen_set_error("ln_shift_bwd: unsupported dtypes"); return PROGEN_ERR_UNSUPPORTED; }
  }
#undef LN_BWD
#undef LN_BWD_N
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_colsum(const void* in, long long ld, int dtype, float* out, long long T, int N, void* stream) {
  PG_CHECK_ARG(T > 0 && N % 4 == 0 && ld % 4 == 0);
  int row_blocks = (int)((T + 1023) / 1024);
  if (row_blocks > 64) row_blocks = 64;
  const long long rpb = (T + row_blocks - 1) / row_blocks;
  dim3 grid((N + 127) / 128, row_blocks);
  if (dtype == PG_F32) colsum_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)in, ld, out, T, N, rpb);
  else colsum_kernel<bf16><<<grid, 256, 0, (cudaStream_t)stream>>>((const bf16*)in, ld, out, T, N, rpb);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

// loss (device scalar, must be zeroed by the caller) += sum_t w_t * nll_t ; dlogits may be null (evaluation only).
// `weights` is a [B*n] fp32 workspace.  inv_batch = 1 / (global batch size) so that a sum over ranks gives the mean.
int progen_ce_fwd_bwd(const void* logits, int dtype, const int* labels, float* weights, float* loss, void* dlogits,
                      int dlogits_dtype, int B, int n, int V, float inv_batch, void* stream) {
  PG_CHECK_ARG(B > 0 && n > 0 && V % 4 == 0);
  cudaStream_t s = (cudaStream_t)stream;
  const long long T = (long long)B * n;
  ce_weights_kernel<<<B, 256, 0, s>>>(labels, weights, n, inv_batch);
  PG_LAUNCH_CHECK();
  const int grid = row_grid(T);
#define CE_CASE(TL, TD) ce_fwd_bwd_kernel<TL, TD><<<grid, 256, 0, s>>>((const TL*)logits, labels, weights, loss, (TD*)dlogits, T, V)
  if (dtype == PG_F32 && dlogits_dtype == PG_F32) CE_CASE(float, float);
  else if (dtype == PG_F32 && dlogits_dtype == PG_BF16) CE_CASE(float, bf16);
  else if (dtype == PG_BF16 && dlogits_dtype == PG_BF16) CE_CASE(bf16, bf16);
  else { progen_set_error("ce_fwd_bwd: unsupported dtypes %d / %d", dtype, dlogits_dtype); return PROGEN_ERR_UNSUPPORTED; }
#undef CE_CASE
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_token_logprob(const void* logits, int dtype, const int* labels, float* logp, float* seq_ll, float* seq_count,
                         int B, int n, int V, void* stream) {
  PG_CHECK_ARG(B > 0 && n > 0 && V % 4 == 0 && logits && labels && logp && seq_ll && seq_count);
  cudaStream_t s = (cudaStream_t)stream;
  const long long T = (long long)B * n;
  const int grid = row_grid(T);
  if (dtype == PG_F32) token_logprob_kernel<float><<<grid, 256, 0, s>>>((const float*)logits, labels, logp, T, V);
  else if (dtype == PG_BF16) token_logprob_kernel<bf16><<<grid, 256, 0, s>>>((const bf16*)logits, labels, logp, T, V);
  else { progen_set_error("token_logprob: unsupported dtype %d", dtype); return PROGEN_ERR_UNSUPPORTED; }
  PG_LAUNCH_CHECK();
  seq_logprob_sum_kernel<<<B, 256, 0, s>>>(labels, logp, seq_ll, seq_count, n);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_preference_head(const void* logits, int dtype, const int* labels, const float* ref_ll, float* logp, float* seq_ll,
                           float* seq_count, float* weights, float* stats, float* loss, float* ce_scratch, void* dlogits,
                           int dlogits_dtype, int pairs, int n, int V, float beta, float inv_pairs, void* stream) {
  PG_CHECK_ARG(logits && labels && ref_ll && logp && seq_ll && seq_count && weights && stats && loss && ce_scratch && dlogits);
  PG_CHECK_ARG(pairs >= 1 && pairs <= (1 << 30) && n > 0 && V % 4 == 0);
  PG_CHECK_ARG(std::isfinite(beta) && beta > 0.f && std::isfinite(inv_pairs) && inv_pairs > 0.f);
  const bool f32_f32 = dtype == PG_F32 && dlogits_dtype == PG_F32, f32_bf16 = dtype == PG_F32 && dlogits_dtype == PG_BF16,
             bf16_bf16 = dtype == PG_BF16 && dlogits_dtype == PG_BF16;
  if (!(f32_f32 || f32_bf16 || bf16_bf16)) {
    progen_set_error("preference_head: unsupported dtypes %d / %d", dtype, dlogits_dtype);
    return PROGEN_ERR_UNSUPPORTED;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int B = 2 * pairs;
  const long long T = (long long)B * n;
  const int rc = progen_token_logprob(logits, dtype, labels, logp, seq_ll, seq_count, B, n, V, stream);
  if (rc != PROGEN_OK) return rc;
  preference_weights_kernel<<<dim3(pairs, 2), PREF_THREADS, 0, s>>>(labels, seq_ll, ref_ll, weights, stats, loss, pairs, n,
                                                                    beta, inv_pairs);
  PG_LAUNCH_CHECK();
  const int grid = row_grid(T);
#define CE_CASE(TL, TD) ce_fwd_bwd_kernel<TL, TD><<<grid, 256, 0, s>>>((const TL*)logits, labels, weights, ce_scratch, (TD*)dlogits, T, V)
  if (f32_f32) CE_CASE(float, float);
  else if (f32_bf16) CE_CASE(float, bf16);
  else CE_CASE(bf16, bf16);
#undef CE_CASE
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_distill_head(const void* logits, int dtype, const float* teacher, long long teacher_row_stride, const int* labels,
                        float* weights, float* scratch, float* stats, float* loss, void* dlogits, int dlogits_dtype, int B,
                        int n, int V, float tau, float alpha, float inv_batch, void* stream) {
  PG_CHECK_ARG(logits && teacher && labels && weights && scratch && stats && loss && dlogits);
  PG_CHECK_ARG(B > 0 && n > 0 && V > 0 && V % 4 == 0 && teacher_row_stride >= n);
  PG_CHECK_ARG(std::isfinite(tau) && tau > 0.f && std::isfinite(1.f / tau) && alpha >= 0.f && alpha <= 1.f);
  PG_CHECK_ARG(std::isfinite(inv_batch) && inv_batch > 0.f);
  const bool f32_f32 = dtype == PG_F32 && dlogits_dtype == PG_F32, f32_bf16 = dtype == PG_F32 && dlogits_dtype == PG_BF16,
             bf16_bf16 = dtype == PG_BF16 && dlogits_dtype == PG_BF16;
  if (!(f32_f32 || f32_bf16 || bf16_bf16)) {
    progen_set_error("distill_head: unsupported dtypes %d / %d", dtype, dlogits_dtype);
    return PROGEN_ERR_UNSUPPORTED;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const long long T = (long long)B * n;
  ce_weights_kernel<<<B, 256, 0, s>>>(labels, weights, n, inv_batch);
  PG_LAUNCH_CHECK();
  const int grid = row_grid(T);
  const float c_kl = (1.f - alpha) * tau;
#define DISTILL_CASE(TL, TD) distill_pos_kernel<TL, TD><<<grid, 256, 0, s>>>((const TL*)logits, teacher, teacher_row_stride, \
      labels, weights, scratch, scratch + T, (TD*)dlogits, T, n, V, 1.f / tau, c_kl, alpha)
  if (f32_f32) DISTILL_CASE(float, float);
  else if (f32_bf16) DISTILL_CASE(float, bf16);
  else DISTILL_CASE(bf16, bf16);
#undef DISTILL_CASE
  PG_LAUNCH_CHECK();
  distill_row_kernel<<<B, DISTILL_THREADS, 0, s>>>(labels, scratch, scratch + T, stats, n);
  PG_LAUNCH_CHECK();
  distill_loss_kernel<<<1, 1, 0, s>>>(stats, B, (1.0 - (double)alpha) * (double)tau * (double)tau, (double)alpha,
                                      (double)inv_batch, loss);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_policy_head(const void* logits, int dtype, const float* ref, long long ref_row_stride, const int* labels,
                       const int* span, const float* advantage, float* scratch, float* stats, float* loss, void* dlogits,
                       int dlogits_dtype, int B, int n, int V, float beta, float inv_rows, void* stream) {
  PG_CHECK_ARG(logits && labels && span && advantage && scratch && stats && loss && dlogits);
  PG_CHECK_ARG(B > 0 && n > 0 && V > 0 && V % 4 == 0 && ref_row_stride >= n);
  PG_CHECK_ARG(std::isfinite(beta) && beta >= 0.f && (beta == 0.f || ref));
  PG_CHECK_ARG(std::isfinite(inv_rows) && inv_rows > 0.f);
  const bool f32_f32 = dtype == PG_F32 && dlogits_dtype == PG_F32, f32_bf16 = dtype == PG_F32 && dlogits_dtype == PG_BF16,
             bf16_bf16 = dtype == PG_BF16 && dlogits_dtype == PG_BF16;
  if (!(f32_f32 || f32_bf16 || bf16_bf16)) {
    progen_set_error("policy_head: unsupported dtypes %d / %d", dtype, dlogits_dtype);
    return PROGEN_ERR_UNSUPPORTED;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const long long T = (long long)B * n;
  const int grid = row_grid(T);
#define POLICY_CASE(TL, TD, R) policy_pos_kernel<TL, TD, R><<<grid, 256, 0, s>>>((const TL*)logits, ref, ref_row_stride, \
      labels, span, advantage, scratch, scratch + T, (TD*)dlogits, T, n, V, beta, inv_rows)
  const bool r = beta > 0.f;
  if (f32_f32) { if (r) POLICY_CASE(float, float, true); else POLICY_CASE(float, float, false); }
  else if (f32_bf16) { if (r) POLICY_CASE(float, bf16, true); else POLICY_CASE(float, bf16, false); }
  else { if (r) POLICY_CASE(bf16, bf16, true); else POLICY_CASE(bf16, bf16, false); }
#undef POLICY_CASE
  PG_LAUNCH_CHECK();
  policy_row_kernel<<<B, POLICY_THREADS, 0, s>>>(span, scratch, scratch + T, stats, n);
  PG_LAUNCH_CHECK();
  policy_loss_kernel<<<1, 1, 0, s>>>(stats, advantage, B, (double)beta, (double)inv_rows, loss);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_masked_mean_pool(const void* x, long long ldx, int dtype, const int* labels, float* out, int B, int n, int d,
                            void* stream) {
  PG_CHECK_ARG(B > 0 && n > 0 && d > 0 && d % 4 == 0 && ldx >= d && ldx % 4 == 0 && x && labels && out);
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid((d + 127) / 128, B);
  if (dtype == PG_F32) masked_mean_pool_kernel<float><<<grid, 256, 0, s>>>((const float*)x, ldx, labels, out, n, d);
  else if (dtype == PG_BF16) masked_mean_pool_kernel<bf16><<<grid, 256, 0, s>>>((const bf16*)x, ldx, labels, out, n, d);
  else { progen_set_error("masked_mean_pool: unsupported dtype %d", dtype); return PROGEN_ERR_UNSUPPORTED; }
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_masked_mean_pool_bwd(const float* demb, const int* labels, void* dy, long long ldy, int dtype, int B, int n, int d,
                                void* stream) {
  PG_CHECK_ARG(B > 0 && n > 0 && d > 0 && d % 4 == 0 && ldy >= d && ldy % 4 == 0 && demb && labels && dy);
  cudaStream_t s = (cudaStream_t)stream;
  dim3 grid((n + POOL_BWD_ROWS - 1) / POOL_BWD_ROWS, B);
  if (dtype == PG_F32) masked_mean_pool_bwd_kernel<float><<<grid, 256, 0, s>>>(demb, labels, (float*)dy, ldy, n, d);
  else if (dtype == PG_BF16) masked_mean_pool_bwd_kernel<bf16><<<grid, 256, 0, s>>>(demb, labels, (bf16*)dy, ldy, n, d);
  else { progen_set_error("masked_mean_pool_bwd: unsupported dtype %d", dtype); return PROGEN_ERR_UNSUPPORTED; }
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_property_head(const float* emb, const float* w, const float* bias, int B, int d, int C, int task, const float* y,
                         const int* cls, float inv_batch, float* pred, float* row_loss, float* loss, float* dpred, float* dw,
                         float* db, float* demb, void* stream) {
  if (C < 1 || C > PROGEN_PROPERTY_MAX_OUTPUTS) {
    progen_set_error("property_head: %d outputs, the head supports 1..%d (PROGEN_PROPERTY_MAX_OUTPUTS)", C,
                     PROGEN_PROPERTY_MAX_OUTPUTS);
    return PROGEN_ERR_ARG;
  }
  PG_CHECK_ARG(B > 0 && d > 0 && emb && w && bias && pred);
  PG_CHECK_ARG(task == PROGEN_TASK_REGRESSION || task == PROGEN_TASK_CLASSIFICATION);
  if (task == PROGEN_TASK_CLASSIFICATION && C < 2) {
    progen_set_error("property_head: classification needs at least 2 classes, got %d", C);
    return PROGEN_ERR_ARG;
  }
  const bool train = y != nullptr || cls != nullptr;
  if (train) {
    PG_CHECK_ARG((task == PROGEN_TASK_REGRESSION ? y != nullptr && cls == nullptr : cls != nullptr && y == nullptr));
    PG_CHECK_ARG(row_loss && loss && dpred && dw && db && demb && std::isfinite(inv_batch) && inv_batch > 0.f);
  }
  cudaStream_t s = (cudaStream_t)stream;
  property_head_rows_kernel<<<B, HEAD_THREADS, 0, s>>>(emb, w, bias, d, C, task, y, cls, inv_batch, pred, row_loss, dpred,
                                                       demb);
  PG_LAUNCH_CHECK();
  if (!train) return PROGEN_OK;
  const long long dc = (long long)d * C;
  property_head_params_kernel<<<(unsigned)((dc + 255) / 256 + 1), 256, 0, s>>>(emb, dpred, row_loss, B, d, C, inv_batch, dw,
                                                                               db, loss);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_residue_head(const void* h, long long ldh, int dtype, const float* w, const float* bias, int B, int L, int d, int C,
                        int task, const float* y, const int* cls, float* pred, float* pos_loss, int* count, float* loss,
                        float* dpred, void* dy, long long ldy, void* stream) {
  if (C < 1 || C > PROGEN_PROPERTY_MAX_OUTPUTS) {
    progen_set_error("residue_head: %d outputs, the head supports 1..%d (PROGEN_PROPERTY_MAX_OUTPUTS)", C,
                     PROGEN_PROPERTY_MAX_OUTPUTS);
    return PROGEN_ERR_ARG;
  }
  PG_CHECK_ARG(B > 0 && L > 0 && d > 0 && d % 4 == 0 && ldh >= d && ldh % 4 == 0 && h && w && bias && pred);
  PG_CHECK_ARG(dtype == PG_F32 || dtype == PG_BF16);
  PG_CHECK_ARG(task == PROGEN_TASK_REGRESSION || task == PROGEN_TASK_CLASSIFICATION);
  if (task == PROGEN_TASK_CLASSIFICATION && C < 2) {
    progen_set_error("residue_head: classification needs at least 2 classes, got %d", C);
    return PROGEN_ERR_ARG;
  }
  const bool train = y != nullptr || cls != nullptr;
  if (train) {
    PG_CHECK_ARG((task == PROGEN_TASK_REGRESSION ? y != nullptr && cls == nullptr : cls != nullptr && y == nullptr));
    PG_CHECK_ARG(pos_loss && count && loss && dpred && dy && ldy >= d && ldy % 4 == 0 && B <= RES_MAX_ROWS);
  }
  cudaStream_t s = (cudaStream_t)stream;
  const long long rows = (long long)B * L;
  if (train) {
    residue_count_kernel<<<1, 1024, 0, s>>>(y, cls, B, L, C, count);
    PG_LAUNCH_CHECK();
  }
  const long long blocks = (rows + ROWS_PER_BLOCK - 1) / ROWS_PER_BLOCK, cap = (long long)pg_num_sms() * 16;
  const int grid = (int)(blocks < cap ? blocks : cap);
#define RES_HEAD(TH, CT) residue_head_kernel<TH, CT><<<grid, 256, 0, s>>>((const TH*)h, ldh, w, bias, rows, d, C, task, y, cls, \
                                                                          count, pred, pos_loss, dpred, (TH*)dy, ldy)
#define RES_HEAD_C(TH) do { if (C <= 4) RES_HEAD(TH, 4); else if (C <= 8) RES_HEAD(TH, 8); else RES_HEAD(TH, 64); } while (0)
  if (dtype == PG_F32) RES_HEAD_C(float);
  else RES_HEAD_C(bf16);
#undef RES_HEAD_C
#undef RES_HEAD
  PG_LAUNCH_CHECK();
  if (!train) return PROGEN_OK;
  residue_loss_kernel<<<1, 1024, 0, s>>>(pos_loss, y, cls, count, B, L, C, loss);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_residue_head_wgrad(const void* h, long long ldh, int dtype, const float* dpred, const float* y, const int* cls,
                              int B, int L, int d, int C, float* workspace, float* dw, float* db, void* stream) {
  PG_CHECK_ARG(B > 0 && B <= 65535 && L > 0 && d > 0 && C >= 1 && C <= PROGEN_PROPERTY_MAX_OUTPUTS && ldh >= d);
  PG_CHECK_ARG(h && dpred && workspace && dw && db && ((y != nullptr) != (cls != nullptr)));
  PG_CHECK_ARG(dtype == PG_F32 || dtype == PG_BF16);
  cudaStream_t s = (cudaStream_t)stream;
  const long long dc1 = (long long)(d + 1) * C;
  const dim3 grid((unsigned)((dc1 + 255) / 256), (unsigned)B);
  if (dtype == PG_F32)
    residue_wgrad_rows_kernel<float><<<grid, 256, 0, s>>>((const float*)h, ldh, dpred, y, cls, L, d, C, workspace);
  else
    residue_wgrad_rows_kernel<bf16><<<grid, 256, 0, s>>>((const bf16*)h, ldh, dpred, y, cls, L, d, C, workspace);
  PG_LAUNCH_CHECK();
  residue_wgrad_reduce_kernel<<<(unsigned)((dc1 + 255) / 256), 256, 0, s>>>(workspace, B, d, C, dw, db);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_rotary_bwd(void* dqkv, long long ld, int dtype, const float* sin_t, const float* cos_t, long long T, int ncols,
                      int seq_len, int dim_head, void* stream) {
  PG_CHECK_ARG(T > 0 && ncols % 4 == 0 && dim_head % 2 == 0 && ld % 4 == 0);
  cudaStream_t s = (cudaStream_t)stream;
  const int grid = ew_grid(T * (ncols / 4), 256);
  if (dtype == PG_F32) rotary_bwd_kernel<float><<<grid, 256, 0, s>>>((float*)dqkv, ld, sin_t, cos_t, T, ncols, seq_len, dim_head);
  else rotary_bwd_kernel<bf16><<<grid, 256, 0, s>>>((bf16*)dqkv, ld, sin_t, cos_t, T, ncols, seq_len, dim_head);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_sgu_gate_fwd(const void* xs, long long ldx, const void* gp, long long ldg, const float* bias, void* out,
                        long long ldo, int dtype, long long T, int C, int seq_len, void* stream) {
  PG_CHECK_ARG(T > 0 && C % 4 == 0 && ldx % 4 == 0 && ldg % 4 == 0 && ldo % 4 == 0);
  cudaStream_t s = (cudaStream_t)stream;
  const int grid = ew_grid(T * (C / 4), 256);
  if (dtype == PG_F32) sgu_gate_fwd_kernel<float><<<grid, 256, 0, s>>>((const float*)xs, ldx, (const float*)gp, ldg, bias, (float*)out, ldo, T, C, seq_len);
  else sgu_gate_fwd_kernel<bf16><<<grid, 256, 0, s>>>((const bf16*)xs, ldx, (const bf16*)gp, ldg, bias, (bf16*)out, ldo, T, C, seq_len);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_sgu_gate_bwd(const void* ds, long long ldds, const void* xs, long long ldx, const void* gp, long long ldg,
                        const float* bias, void* dxs, long long lddx, void* dgp, long long lddg, float* dbias, int dtype,
                        long long T, int C, int seq_len, void* stream) {
  PG_CHECK_ARG(T > 0 && C % 4 == 0);
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == PG_F32) sgu_gate_bwd_kernel<float><<<row_grid(T), 256, 0, s>>>((const float*)ds, ldds, (const float*)xs, ldx, (const float*)gp, ldg, bias, (float*)dxs, lddx, (float*)dgp, lddg, dbias, T, C, seq_len);
  else sgu_gate_bwd_kernel<bf16><<<row_grid(T), 256, 0, s>>>((const bf16*)ds, ldds, (const bf16*)xs, ldx, (const bf16*)gp, ldg, bias, (bf16*)dxs, lddx, (bf16*)dgp, lddg, dbias, T, C, seq_len);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_gelu_bwd(void* da, const void* u, int dtype, long long numel, void* stream) {
  PG_CHECK_ARG(numel > 0 && numel % 4 == 0);
  cudaStream_t s = (cudaStream_t)stream;
  const int grid = ew_grid(numel / 4, 256);
  if (dtype == PG_F32) gelu_bwd_kernel<float><<<grid, 256, 0, s>>>((float*)da, (const float*)u, numel / 4);
  else gelu_bwd_kernel<bf16><<<grid, 256, 0, s>>>((bf16*)da, (const bf16*)u, numel / 4);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_cast_f32(const float* in, void* out, int out_dtype, long long numel, void* stream) {
  PG_CHECK_ARG(numel > 0 && numel % 4 == 0);
  cudaStream_t s = (cudaStream_t)stream;
  const int grid = ew_grid(numel / 4, 256);
  if (out_dtype == PG_F32) cast_kernel<float><<<grid, 256, 0, s>>>(in, (float*)out, numel / 4);
  else cast_kernel<bf16><<<grid, 256, 0, s>>>(in, (bf16*)out, numel / 4);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_scale_cast_f32(const float* in, void* out, int out_dtype, float scale, long long numel, void* stream) {
  PG_CHECK_ARG(numel > 0 && numel % 4 == 0 && in != nullptr && out != nullptr);
  cudaStream_t s = (cudaStream_t)stream;
  const int grid = ew_grid(numel / 4, 256);
  if (out_dtype == PG_F32) scale_cast_kernel<float><<<grid, 256, 0, s>>>(in, (float*)out, scale, numel / 4);
  else scale_cast_kernel<bf16><<<grid, 256, 0, s>>>(in, (bf16*)out, scale, numel / 4);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_tril_cast(const float* w, void* out, int out_dtype, int n, void* stream) {
  PG_CHECK_ARG(n > 0 && n % 4 == 0);
  cudaStream_t s = (cudaStream_t)stream;
  const int grid = ew_grid((long long)n * (n / 4), 256);
  if (out_dtype == PG_F32) tril_cast_kernel<float><<<grid, 256, 0, s>>>(w, (float*)out, n);
  else tril_cast_kernel<bf16><<<grid, 256, 0, s>>>(w, (bf16*)out, n);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_decode_load_weight(const float* w, const float* a, const float* b, int rank, float scale, int in, int out,
                              int interleave, void* dst, int dst_dtype, void* stream) {
  PG_CHECK_ARG(w && dst && in > 0 && out > 0 && rank >= 0 && rank <= LW_MAX_RANK && (interleave == 0 || interleave == 1));
  PG_CHECK_ARG(rank == 0 || (a && b && in > 1 && std::isfinite(scale)));
  PG_CHECK_ARG(!interleave || out % 2 == 0);
  if (dst_dtype != PG_F32 && dst_dtype != PG_BF16) {
    progen_set_error("decode_load_weight: unsupported dtype %d", dst_dtype);
    return PROGEN_ERR_UNSUPPORTED;
  }
  cudaStream_t s = (cudaStream_t)stream;
  if (in == 1) {
    const int grid = ew_grid(out, 256);
    if (dst_dtype == PG_F32) load_vector_kernel<float><<<grid, 256, 0, s>>>(w, out, interleave, (float*)dst);
    else load_vector_kernel<bf16><<<grid, 256, 0, s>>>(w, out, interleave, (bf16*)dst);
  } else {
    const dim3 grid((in + LW_TILE - 1) / LW_TILE, (out + LW_TILE - 1) / LW_TILE), block(LW_TILE, 8);
    if (dst_dtype == PG_F32)
      load_weight_kernel<float><<<grid, block, 0, s>>>(w, a, b, rank, scale, in, out, interleave, (float*)dst);
    else load_weight_kernel<bf16><<<grid, block, 0, s>>>(w, a, b, rank, scale, in, out, interleave, (bf16*)dst);
  }
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

int progen_gather_rows_f32(const void* src, long long ld, int src_dtype, int src_seqs, long long src_seq_rows,
                           const int* row_map, int B, int row0, int rows, int col0, int groups, int cols, float* dst,
                           long long dst_b_stride, long long dst_g_stride, long long dst_row_stride, void* stream) {
  PG_CHECK_ARG(src != nullptr && row_map != nullptr && dst != nullptr);
  PG_CHECK_ARG(src_dtype == PG_F32 || src_dtype == PG_BF16);
  const int nv = src_dtype == PG_F32 ? 4 : 8;          // elements per 16-byte source vector
  PG_CHECK_ARG(B > 0 && src_seqs > 0 && src_seq_rows > 0 && groups > 0 && cols > 0 && rows >= 0 && row0 >= 0 && col0 >= 0);
  PG_CHECK_ARG(row0 + (long long)rows <= src_seq_rows && col0 + (long long)groups * cols <= ld);
  PG_CHECK_ARG(cols % nv == 0 && col0 % nv == 0 && ld % nv == 0);
  PG_CHECK_ARG(dst_b_stride >= 0 && dst_g_stride >= 0 && dst_row_stride >= 0);
  PG_CHECK_ARG(dst_b_stride % 4 == 0 && dst_g_stride % 4 == 0 && dst_row_stride % 4 == 0);
  PG_CHECK_ARG((uintptr_t)src % 16 == 0 && (uintptr_t)dst % 16 == 0);
  if (rows == 0) return PROGEN_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const long long total = (long long)B * groups * rows * (cols / nv);
  const int grid = ew_grid(total, 256);
  if (src_dtype == PG_F32)
    gather_rows_f32_kernel<float><<<grid, 256, 0, s>>>((const float*)src, ld, row_map, src_seqs, src_seq_rows, row0, rows, col0,
                                                       groups, cols, dst, dst_b_stride, dst_g_stride, dst_row_stride, total);
  else
    gather_rows_f32_kernel<bf16><<<grid, 256, 0, s>>>((const bf16*)src, ld, row_map, src_seqs, src_seq_rows, row0, rows, col0,
                                                      groups, cols, dst, dst_b_stride, dst_g_stride, dst_row_stride, total);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

}  // extern "C"
