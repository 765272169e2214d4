// Shared helpers for libprogen_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------------------------------------------------
// error plumbing: every exported function returns 0 or a negative code; the message is thread-local.
#define PROGEN_OK 0
#define PROGEN_ERR_CUDA -1
#define PROGEN_ERR_ARG -2
#define PROGEN_ERR_DEVICE -3
#define PROGEN_ERR_UNSUPPORTED -4

void progen_set_error(const char* fmt, ...);

#define PG_CHECK_ARG(cond, ...)                                                   \
  do {                                                                            \
    if (!(cond)) {                                                                \
      progen_set_error("%s:%d: argument check failed: %s", __FILE__, __LINE__, #cond); \
      return PROGEN_ERR_ARG;                                                      \
    }                                                                             \
  } while (0)

#define PG_CUDA(call)                                                             \
  do {                                                                            \
    cudaError_t e__ = (call);                                                     \
    if (e__ != cudaSuccess) {                                                     \
      progen_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
      return PROGEN_ERR_CUDA;                                                     \
    }                                                                             \
  } while (0)

// every kernel launch is followed by PG_LAUNCH_CHECK(): it also feeds progen_launch_count() (bench.py's gpu_launches)
extern unsigned long long g_progen_launches;   // statistics only (bench.py's gpu_launches); bumped atomically, never read by a kernel path
#define PG_LAUNCH_CHECK()                 \
  do {                                    \
    __atomic_fetch_add(&g_progen_launches, 1ull, __ATOMIC_RELAXED); \
    PG_CUDA(cudaPeekAtLastError());       \
  } while (0)

// dtype enum shared with the Python host layer (progen_b200/lib.py)
enum : int { PG_F32 = 0, PG_BF16 = 1 };

static inline int pg_num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// ---------------------------------------------------------------------------------------------------------
// device helpers
__device__ __forceinline__ float to_f32(float x) { return x; }
__device__ __forceinline__ float to_f32(bf16 x) { return __bfloat162float(x); }
template <typename T> __device__ __forceinline__ T from_f32(float x);
template <> __device__ __forceinline__ float from_f32<float>(float x) { return x; }
template <> __device__ __forceinline__ bf16 from_f32<bf16>(float x) { return __float2bfloat16_rn(x); }

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}

// jax.nn.gelu(approximate=True): 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3)))  (reference progen.py:141,143)
__device__ __forceinline__ float gelu_tanh(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * (x + k1 * x * x * x);
  return 0.5f * x * (1.0f + tanhf(u));
}
__device__ __forceinline__ float gelu_tanh_grad(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float u = k0 * (x + k1 * x * x * x);
  float t = tanhf(u);
  float du = k0 * (1.0f + 3.0f * k1 * x * x);
  return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * du;
}

// Same functions with the hardware tanh (MUFU.TANH, rel. error ~2^-11): used where the result is rounded to bf16 anyway
// (tensor-core path); the fp32 parity path keeps tanhf.
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
template <bool FAST> __device__ __forceinline__ float gelu_fwd(float x) {
  if constexpr (!FAST) return gelu_tanh(x);
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float u = k0 * (x + k1 * x * x * x);
  return 0.5f * x * (1.0f + tanh_fast(u));
}
template <bool FAST> __device__ __forceinline__ float gelu_bwd(float x) {
  if constexpr (!FAST) return gelu_tanh_grad(x);
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float x2 = x * x;
  const float t = tanh_fast(k0 * (x + k1 * x * x2));
  return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * k0 * (1.0f + 3.0f * k1 * x2);
}

// gelu(x) and gelu'(x) from ONE tanh (the GLU backward epilogue needs both for the same argument)
template <bool FAST> __device__ __forceinline__ void gelu_fwd_bwd(float x, float& f, float& df) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float x2 = x * x;
  const float u = k0 * (x + k1 * x * x2);
  const float t = FAST ? tanh_fast(u) : tanhf(u);
  const float h = 0.5f * (1.0f + t);
  f = x * h;
  df = h + 0.5f * x * (1.0f - t * t) * k0 * (1.0f + 3.0f * k1 * x2);
}

// vector load/store of NV consecutive elements (NV * sizeof(T) must be a multiple of 16 bytes, pointer aligned)
template <int NV> __device__ __forceinline__ void load_vec(const float* p, float (&v)[NV]) {
#pragma unroll
  for (int i = 0; i < NV; i += 4) {
    float4 t = *reinterpret_cast<const float4*>(p + i);
    v[i] = t.x; v[i + 1] = t.y; v[i + 2] = t.z; v[i + 3] = t.w;
  }
}
template <int NV> __device__ __forceinline__ void load_vec(const bf16* p, float (&v)[NV]) {
#pragma unroll
  for (int i = 0; i < NV; i += 8) {
    uint4 t = *reinterpret_cast<const uint4*>(p + i);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&t);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 f = __bfloat1622float2(h[j]);
      v[i + 2 * j] = f.x; v[i + 2 * j + 1] = f.y;
    }
  }
}
template <int NV> __device__ __forceinline__ void store_vec(float* p, const float (&v)[NV]) {
#pragma unroll
  for (int i = 0; i < NV; i += 4) *reinterpret_cast<float4*>(p + i) = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
}
template <int NV> __device__ __forceinline__ void store_vec(bf16* p, const float (&v)[NV]) {
#pragma unroll
  for (int i = 0; i < NV; i += 8) {
    uint4 t;
    t.x = pack_bf16x2(v[i], v[i + 1]); t.y = pack_bf16x2(v[i + 2], v[i + 3]);
    t.z = pack_bf16x2(v[i + 4], v[i + 5]); t.w = pack_bf16x2(v[i + 6], v[i + 7]);
    *reinterpret_cast<uint4*>(p + i) = t;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
