// GEMM epilogues shared by the wgmma GEMM (gemm_tc.cu) and the fp32 SIMT GEMM (gemm_simt.cu).
// A thread hands over NV consecutive accumulator columns of one output row (an "item"); the epilogue fuses what the
// reference does right after the matmul (bias, rotary, residual add, GELU / GLU, their backward forms).
//
// Each kind runs in two phases so that a thread can keep the global reads of several items in flight at once:
//   epi_load_col  once per thread and tile: what depends on the columns only (the bias);
//   epi_load      per item: every other global read (rotary sin / cos, residual, saved pre-activation), kept as the
//                 16-byte words it loaded (bf16 stays packed);
//   epi_finish    per item: the arithmetic and the stores.
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
  float* colsum;                     // EPI_GLU_BWD / EPI_GELU_BWD: += column sums of the stored out (nullable; the
                                     // bias gradient of the Linear whose pre-activation this is)
};

// Per-item global operands of one kind, as loaded: 16-byte words
template <int KIND, typename TO, int NV> struct EpiPre {
  static_assert(NV % 8 == 0, "items are whole 16-byte vectors of bf16 and fp32");
  static constexpr int BYTES = KIND == EPI_ROTARY ? NV * 4                       // NV/2 sin, then NV/2 cos
                             : KIND == EPI_RESIDUAL ? NV * 4                     // fp32 residual
                             : KIND == EPI_GLU_BWD ? 2 * NV * (int)sizeof(TO)    // (value, gate) pre-activations
                             : KIND == EPI_GELU_BWD ? NV * (int)sizeof(TO)       // pre-activation
                             : 0;
  static constexpr int NQ = BYTES / 16;
  uint4 q[NQ > 0 ? NQ : 1];
};

// Per-thread column operands: the bias of the thread's NV columns
template <int NV> struct EpiCol {
  float b[NV];
};

// Output columns an item adds to `colsum`: the 2 NV interleaved d(value), d(gate) of GLU, the NV of GELU
template <int KIND, int NV> struct EpiColsum {
  static constexpr int W = KIND == EPI_GLU_BWD ? 2 * NV : KIND == EPI_GELU_BWD ? NV : 0;
  static constexpr int REGS = W > 0 ? W : 1;                         // size of the thread's partial-sum array
  static constexpr int OUT_SCALE = KIND == EPI_GLU_BWD ? 2 : 1;     // output column of GEMM column col: OUT_SCALE * col
};

__device__ __forceinline__ uint4 ld16(const void* p) { return *reinterpret_cast<const uint4*>(p); }

// the floats of NQ loaded words (exactly what load_vec would have produced)
template <typename T, int N> __device__ __forceinline__ void unpack(const uint4* q, float (&v)[N]) {
  if constexpr (sizeof(T) == 4) {
#pragma unroll
    for (int i = 0; i < N / 4; ++i) {
      v[4 * i] = __uint_as_float(q[i].x); v[4 * i + 1] = __uint_as_float(q[i].y);
      v[4 * i + 2] = __uint_as_float(q[i].z); v[4 * i + 3] = __uint_as_float(q[i].w);
    }
  } else {
#pragma unroll
    for (int i = 0; i < N / 8; ++i) {
      const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&q[i]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __bfloat1622float2(h[j]);
        v[8 * i + 2 * j] = f.x; v[8 * i + 2 * j + 1] = f.y;
      }
    }
  }
}

template <int KIND> constexpr bool epi_uses_bias() {
  return KIND == EPI_STORE || KIND == EPI_RESIDUAL || KIND == EPI_GLU || KIND == EPI_GELU;
}

// `valid` says whether the thread's columns exist.  The bias is the same NV floats for every lane of a row (broadcast),
// fetched with 16-byte loads.
template <int KIND, int NV> __device__ __forceinline__ void epi_load_col(const EpiArgs& e, int col, bool valid, EpiCol<NV>& c) {
  if constexpr (epi_uses_bias<KIND>()) {
#pragma unroll
    for (int i = 0; i < NV; i += 4) {
      const float4 b = (valid && e.bias) ? __ldg(reinterpret_cast<const float4*>(e.bias + col + i)) : make_float4(0.f, 0.f, 0.f, 0.f);
      c.b[i] = b.x; c.b[i + 1] = b.y; c.b[i + 2] = b.z; c.b[i + 3] = b.w;
    }
  }
}

// `valid` says whether this item (row and columns) exists; an item that does not loads zeros.
template <int KIND, typename TO, int NV>
__device__ __forceinline__ void epi_load(const EpiArgs& e, long long row, int col, bool valid, EpiPre<KIND, TO, NV>& p) {
  constexpr int NQ = EpiPre<KIND, TO, NV>::NQ;
  if constexpr (NQ > 0) {
    if (!valid) {
#pragma unroll
      for (int i = 0; i < NQ; ++i) p.q[i] = make_uint4(0u, 0u, 0u, 0u);
      return;
    }
  }
  if constexpr (KIND == EPI_ROTARY) {
    const int pos = (int)(row % e.seq_len);
    const int half = e.dim_head >> 1;
    const float* sp = e.rot_sin + (long long)pos * half;
    const float* cp = e.rot_cos + (long long)pos * half;
    if (e.dim_head % NV == 0) {
      // the NV columns sit inside one head: NV/2 consecutive (sin, cos) entries, 16-byte vector loads
      const int j0 = (col % e.dim_head) >> 1;
#pragma unroll
      for (int i = 0; i < NQ / 2; ++i) {
        p.q[i] = ld16(sp + j0 + 4 * i);
        p.q[NQ / 2 + i] = ld16(cp + j0 + 4 * i);
      }
    } else {
      uint32_t s[NV / 2], c[NV / 2];
#pragma unroll
      for (int i = 0; i < NV; i += 2) {
        const int j = ((col + i) % e.dim_head) >> 1;
        s[i >> 1] = __float_as_uint(__ldg(sp + j));
        c[i >> 1] = __float_as_uint(__ldg(cp + j));
      }
#pragma unroll
      for (int i = 0; i < NQ / 2; ++i) {
        p.q[i] = make_uint4(s[4 * i], s[4 * i + 1], s[4 * i + 2], s[4 * i + 3]);
        p.q[NQ / 2 + i] = make_uint4(c[4 * i], c[4 * i + 1], c[4 * i + 2], c[4 * i + 3]);
      }
    }
  } else if constexpr (KIND == EPI_RESIDUAL) {
    // residual_in = aux (fp32, ldaux) when given, else out itself (in place)
    const float* r = e.aux ? reinterpret_cast<const float*>(e.aux) + row * e.ldaux + col
                           : reinterpret_cast<const float*>(e.out) + row * e.ldo + col;
#pragma unroll
    for (int i = 0; i < NQ; ++i) p.q[i] = ld16(r + 4 * i);
  } else if constexpr (KIND == EPI_GLU_BWD) {
    // pre-activations of (value, gate) for acc column c sit at aux[2c], aux[2c+1]: one 2*NV-wide load
    const TO* u = reinterpret_cast<const TO*>(e.aux) + row * e.ldaux + 2 * col;
#pragma unroll
    for (int i = 0; i < NQ; ++i) p.q[i] = ld16(reinterpret_cast<const uint8_t*>(u) + 16 * i);
  } else if constexpr (KIND == EPI_GELU_BWD) {
    const TO* u = reinterpret_cast<const TO*>(e.aux) + row * e.ldaux + col;
#pragma unroll
    for (int i = 0; i < NQ; ++i) p.q[i] = ld16(reinterpret_cast<const uint8_t*>(u) + 16 * i);
  }
}

// Arithmetic and stores of one item, from the operands epi_load_col / epi_load read.  `csum` (EpiColsum<KIND, NV>::W
// floats) gathers the stored values of the item's output columns when e.colsum is set.
template <int KIND, typename TO, int NV, int CW>
__device__ __forceinline__ void epi_finish(const EpiArgs& e, long long row, int col, float (&v)[NV], const EpiCol<NV>& cb,
                                           const EpiPre<KIND, TO, NV>& p, bool valid, float (&csum)[CW]) {
  constexpr bool FAST = sizeof(TO) == 2;      // bf16 outputs: hardware tanh is below the output rounding
  if constexpr (epi_uses_bias<KIND>()) {
    if (KIND == EPI_GLU || KIND == EPI_GELU || e.bias) {
#pragma unroll
      for (int i = 0; i < NV; ++i) v[i] += cb.b[i];
    }
  }
  if constexpr (KIND == EPI_STORE) {
    if (valid) store_vec<NV>(reinterpret_cast<TO*>(e.out) + row * e.ldo + col, v);
  } else if constexpr (KIND == EPI_ROTARY) {
    float s[NV / 2], c[NV / 2], o[NV];
    unpack<float>(&p.q[0], s);
    unpack<float>(&p.q[EpiPre<KIND, TO, NV>::NQ / 2], c);
#pragma unroll
    for (int i = 0; i < NV; i += 2) {
      o[i] = v[i] * c[i >> 1] - v[i + 1] * s[i >> 1];
      o[i + 1] = v[i + 1] * c[i >> 1] + v[i] * s[i >> 1];
    }
    if (valid) store_vec<NV>(reinterpret_cast<TO*>(e.out) + row * e.ldo + col, o);
  } else if constexpr (KIND == EPI_RESIDUAL) {
    float r[NV];
    unpack<float>(p.q, r);
#pragma unroll
    for (int i = 0; i < NV; ++i) r[i] += v[i];
    if (valid) store_vec<NV>(reinterpret_cast<float*>(e.out) + row * e.ldo + col, r);
  } else if constexpr (KIND == EPI_GLU) {
    // uniform branch: inference (no backward) passes out2 = nullptr and skips the pre-activation store
    if (e.out2 && valid) store_vec<NV>(reinterpret_cast<TO*>(e.out2) + row * e.ldo2 + col, v);
    TO* po = reinterpret_cast<TO*>(e.out) + row * e.ldo + (col >> 1);
    if (valid) {
#pragma unroll
      for (int i = 0; i < NV / 2; ++i) po[i] = from_f32<TO>(v[2 * i] * gelu_fwd<FAST>(v[2 * i + 1]));
    }
  } else if constexpr (KIND == EPI_GELU) {
    if (e.out2 && valid) store_vec<NV>(reinterpret_cast<TO*>(e.out2) + row * e.ldo2 + col, v);
    float o[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) o[i] = gelu_fwd<FAST>(v[i]);
    if (valid) store_vec<NV>(reinterpret_cast<TO*>(e.out) + row * e.ldo + col, o);
  } else if constexpr (KIND == EPI_GLU_BWD) {
    float u[2 * NV];
    unpack<TO>(p.q, u);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float dh = v[i], val = u[2 * i], gate = u[2 * i + 1];
      float gf, gd;
      gelu_fwd_bwd<FAST>(gate, gf, gd);
      u[2 * i] = dh * gf;
      u[2 * i + 1] = dh * val * gd;
    }
    if (valid) {
      store_vec<2 * NV>(reinterpret_cast<TO*>(e.out) + row * e.ldo + 2 * col, u);
      if (e.colsum) {
#pragma unroll
        for (int i = 0; i < 2 * NV; ++i) csum[i] += to_f32(from_f32<TO>(u[i]));     // the values as stored
      }
    }
  } else if constexpr (KIND == EPI_GELU_BWD) {
    float u[NV];
    unpack<TO>(p.q, u);
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] *= gelu_bwd<FAST>(u[i]);
    if (valid) {
      store_vec<NV>(reinterpret_cast<TO*>(e.out) + row * e.ldo + col, v);
      if (e.colsum) {
#pragma unroll
        for (int i = 0; i < NV; ++i) csum[i] += to_f32(from_f32<TO>(v[i]));
      }
    }
  } else if constexpr (KIND == EPI_ACCUM) {
    if (!valid) return;
    float* po = reinterpret_cast<float*>(e.out) + row * e.ldo + col;
    const int lim = e.tril ? (int)(row % e.tril_rows) : 0x7fffffff;
    if (e.atomic) {
#pragma unroll
      for (int i = 0; i < NV; i += 4) {
        if (col + i + 3 <= lim) {
          asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(po + i), "f"(v[i]), "f"(v[i + 1]),
                       "f"(v[i + 2]), "f"(v[i + 3]) : "memory");
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (col + i + j <= lim) atomicAdd(po + i + j, v[i + j]);
        }
      }
    } else {
      float r[NV];
      load_vec<NV>(po, r);
#pragma unroll
      for (int i = 0; i < NV; ++i) r[i] += (col + i <= lim) ? v[i] : 0.f;
      store_vec<NV>(po, r);
    }
  }
}
