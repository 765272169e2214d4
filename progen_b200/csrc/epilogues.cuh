// GEMM epilogues shared by the wgmma GEMM (gemm_tc.cu) and the fp32 SIMT GEMM (gemm_simt.cu).
// A thread hands over NV consecutive accumulator columns of one output row; the epilogue fuses what the
// reference does right after the matmul (bias, rotary, residual add, GELU / GLU, their backward forms).
#pragma once
#include "common.cuh"

enum EpiKind : int {
  EPI_STORE = 0,      // out = acc (+ bias[col])
  EPI_ROTARY = 1,     // out = rotary(acc)            qkv projection, progen.py:83-87 (rotary on q, k AND v)
  EPI_RESIDUAL = 2,   // out(f32) += acc + bias       to_out / proj_out + residual, progen.py:103,148,230-231
  EPI_GLU = 3,        // out = value * gelu(gate); out2 (nullable) = pre-activation (interleaved value,gate)   progen.py:139-141
  EPI_GELU = 4,       // out = gelu(pre); out2 (nullable) = pre-activation                                     progen.py:143
  EPI_GLU_BWD = 5,    // acc = d(out of GLU); aux = saved pre-activation; out = d(pre) interleaved
  EPI_GELU_BWD = 6,   // acc = d(gelu out); aux = saved pre-activation; out = acc * gelu'(pre)
  EPI_ACCUM = 7,      // out(f32) += acc  (atomic when several CTAs own the same tile; optional tril mask)
  EPI_NUM_KINDS = 8
};

struct EpiArgs {
  void* out; long long ldo;
  void* out2; long long ldo2;       // EPI_GLU / EPI_GELU: pre-activation for the backward pass; nullptr = not stored
  const float* bias;                 // [N] (already interleaved for GLU) or nullptr
  const void* aux; long long ldaux;  // saved pre-activations for the *_BWD kinds
  const float* rot_sin;              // [seq_len, dim_head/2]
  const float* rot_cos;
  int seq_len; int dim_head;
  int atomic;                        // EPI_ACCUM: use red.global.add
  int tril;                          // EPI_ACCUM: keep only col <= (row % tril_rows)
  int tril_rows;
};

// ---------------------------------------------------------------------------------------------------------
// How an epilogue thread moves its row slice to / from global memory: per-thread vector accesses (both GEMMs hand
// every thread 8 consecutive columns of one row).
struct DirectIO {
  template <int N, typename T> __device__ __forceinline__ void store(T* p, long long, const float (&v)[N], bool valid) const {
    if (valid) store_vec<N>(p, v);
  }
  template <int N, typename T> __device__ __forceinline__ void load(const T* p, long long, float (&v)[N], bool valid) const {
    if (valid) load_vec<N>(p, v);
    else {
#pragma unroll
      for (int i = 0; i < N; ++i) v[i] = 0.f;
    }
  }
};

// v[i] += bias[col + i]: the same NV floats for every lane (broadcast), fetched with 16-byte loads
template <int NV> __device__ __forceinline__ void add_bias(const float* __restrict__ bias, int col, float (&v)[NV]) {
#pragma unroll
  for (int i = 0; i < NV; i += 4) {
    const float4 b = __ldg(reinterpret_cast<const float4*>(bias + col + i));
    v[i] += b.x; v[i + 1] += b.y; v[i + 2] += b.z; v[i + 3] += b.w;
  }
}

// `valid` says whether this thread's row exists.
template <int KIND, typename TO, int NV, typename IO>
__device__ __forceinline__ void epi_apply(const EpiArgs& e, const IO& io, long long row, int col, float (&v)[NV], bool valid) {
  constexpr bool FAST = sizeof(TO) == 2;      // bf16 outputs: hardware tanh is below the output rounding
  if constexpr (KIND == EPI_STORE) {
    if (e.bias) add_bias<NV>(e.bias, col, v);
    io.template store<NV>(reinterpret_cast<TO*>(e.out) + row * e.ldo + col, e.ldo, v, valid);
  } else if constexpr (KIND == EPI_ROTARY) {
    const int pos = (int)(row % e.seq_len);
    const int half = e.dim_head >> 1;
    const float* sp = e.rot_sin + (long long)pos * half;
    const float* cp = e.rot_cos + (long long)pos * half;
    float o[NV];
    if (e.dim_head % NV == 0) {
      // the NV columns sit inside one head: NV/2 consecutive (sin, cos) entries, 16-byte vector loads
      const int j0 = (col % e.dim_head) >> 1;
      float s[NV / 2], c[NV / 2];
      if constexpr (NV >= 32) {
        // consecutive rows are consecutive positions (a warp's 32 rows never straddle a sequence: seq_len % 32 == 0
        // is checked by the launcher), so the table slices form a [32 x NV/2] block: coalesced staged loads
        io.template load<NV / 2>(sp + j0, half, s, true);
        io.template load<NV / 2>(cp + j0, half, c, true);
      } else {
        load_vec<NV / 2>(sp + j0, s);
        load_vec<NV / 2>(cp + j0, c);
      }
#pragma unroll
      for (int i = 0; i < NV; i += 2) {
        o[i] = v[i] * c[i >> 1] - v[i + 1] * s[i >> 1];
        o[i + 1] = v[i + 1] * c[i >> 1] + v[i] * s[i >> 1];
      }
    } else {
#pragma unroll
      for (int i = 0; i < NV; i += 2) {
        const int j = ((col + i) % e.dim_head) >> 1;
        const float s = __ldg(sp + j), c = __ldg(cp + j);
        o[i] = v[i] * c - v[i + 1] * s;
        o[i + 1] = v[i + 1] * c + v[i] * s;
      }
    }
    io.template store<NV>(reinterpret_cast<TO*>(e.out) + row * e.ldo + col, e.ldo, o, valid);
  } else if constexpr (KIND == EPI_RESIDUAL) {
    // out = residual_in + acc + bias; residual_in = aux (fp32, ldaux) when given, else out itself (in place)
    float* p = reinterpret_cast<float*>(e.out) + row * e.ldo + col;
    float r[NV];
    if (e.aux) io.template load<NV>(reinterpret_cast<const float*>(e.aux) + row * e.ldaux + col, e.ldaux, r, valid);
    else io.template load<NV>(const_cast<const float*>(p), e.ldo, r, valid);
    if (e.bias) add_bias<NV>(e.bias, col, v);
#pragma unroll
    for (int i = 0; i < NV; ++i) r[i] += v[i];
    io.template store<NV>(p, e.ldo, r, valid);
  } else if constexpr (KIND == EPI_GLU) {
    add_bias<NV>(e.bias, col, v);
    // uniform branch: inference (no backward) passes out2 = nullptr and skips the pre-activation store
    if (e.out2) io.template store<NV>(reinterpret_cast<TO*>(e.out2) + row * e.ldo2 + col, e.ldo2, v, valid);
    TO* po = reinterpret_cast<TO*>(e.out) + row * e.ldo + (col >> 1);
    if constexpr (NV >= 16) {
      float o[NV / 2];
#pragma unroll
      for (int i = 0; i < NV / 2; ++i) o[i] = v[2 * i] * gelu_fwd<FAST>(v[2 * i + 1]);
      io.template store<NV / 2>(po, e.ldo, o, valid);
    } else {
      if (valid) {
#pragma unroll
        for (int i = 0; i < NV / 2; ++i) po[i] = from_f32<TO>(v[2 * i] * gelu_fwd<FAST>(v[2 * i + 1]));
      }
    }
  } else if constexpr (KIND == EPI_GELU) {
    add_bias<NV>(e.bias, col, v);
    if (e.out2) io.template store<NV>(reinterpret_cast<TO*>(e.out2) + row * e.ldo2 + col, e.ldo2, v, valid);
    float o[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) o[i] = gelu_fwd<FAST>(v[i]);
    io.template store<NV>(reinterpret_cast<TO*>(e.out) + row * e.ldo + col, e.ldo, o, valid);
  } else if constexpr (KIND == EPI_GLU_BWD) {
    // acc column c is d(h[c]); pre-activations of (value, gate) sit at aux[2c], aux[2c+1]; one 2*NV-wide load / store
    float u[2 * NV];
    io.template load<2 * NV>(reinterpret_cast<const TO*>(e.aux) + row * e.ldaux + 2 * col, e.ldaux, u, valid);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float dh = v[i], val = u[2 * i], gate = u[2 * i + 1];
      float gf, gd;
      gelu_fwd_bwd<FAST>(gate, gf, gd);
      u[2 * i] = dh * gf;
      u[2 * i + 1] = dh * val * gd;
    }
    io.template store<2 * NV>(reinterpret_cast<TO*>(e.out) + row * e.ldo + 2 * col, e.ldo, u, valid);
  } else if constexpr (KIND == EPI_GELU_BWD) {
    float u[NV];
    io.template load<NV>(reinterpret_cast<const TO*>(e.aux) + row * e.ldaux + col, e.ldaux, u, valid);
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] *= gelu_bwd<FAST>(u[i]);
    io.template store<NV>(reinterpret_cast<TO*>(e.out) + row * e.ldo + col, e.ldo, v, valid);
  } else if constexpr (KIND == EPI_ACCUM) {
    if (!valid) return;
    float* p = reinterpret_cast<float*>(e.out) + row * e.ldo + col;
    const int lim = e.tril ? (int)(row % e.tril_rows) : 0x7fffffff;
    if (e.atomic) {
#pragma unroll
      for (int i = 0; i < NV; i += 4) {
        if (col + i + 3 <= lim) {
          asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p + i), "f"(v[i]), "f"(v[i + 1]),
                       "f"(v[i + 2]), "f"(v[i + 3]) : "memory");
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (col + i + j <= lim) atomicAdd(p + i + j, v[i + j]);
        }
      }
    } else {
      float r[NV];
      load_vec<NV>(p, r);
#pragma unroll
      for (int i = 0; i < NV; ++i) r[i] += (col + i <= lim) ? v[i] : 0.f;
      store_vec<NV>(p, r);
    }
  }
}
