// Optimizer of the reference training loop as two HBM-bound kernels over FLAT parameter / gradient / state buffers:
//   optax.chain(clip_by_global_norm(max_norm), adamw(lr, wd, mask = ndim > 1), apply_every(k))   (train.py:115-121,189-190)
// Semantics kept exactly: the clip acts on every micro-batch gradient, Adam moments advance every call, the
// *updates* are accumulated and added to the parameters on every k-th call only.
// Layout: elements [0, n_decay) are the ndim > 1 leaves (weight decay applies), [n_decay, n) the rest.
#include "common.cuh"
#include "../../include/progen_b200.h"

namespace {

constexpr int NORM_THREADS = 256;

__global__ void sqnorm_partial_kernel(const float* __restrict__ g, long long n, float* __restrict__ partial) {
  float s = 0.f;
  const long long n4 = n / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  if (blockIdx.x == 0)
    for (long long i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) s += g[i] * g[i];
  __shared__ float red[NORM_THREADS / 32];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < NORM_THREADS / 32; ++i) t += red[i];
    partial[blockIdx.x] = t;
  }
}

__global__ void sqnorm_final_kernel(const float* __restrict__ partial, int nblocks, float* __restrict__ out) {
  // fixed order -> deterministic
  __shared__ double red[NORM_THREADS];
  double s = 0.0;
  for (int i = threadIdx.x; i < nblocks; i += blockDim.x) s += (double)partial[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = NORM_THREADS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = (float)red[0];
}

struct AdamArgs {
  float lr, b1, b2, eps, wd, max_norm;
};

// Step-dependent scalars of the optimizer kept on the device, so that a captured CUDA graph of the whole training step
// can be replayed unchanged: adam_tick_kernel advances them once per step (train.py:189-190 semantics: count, emit).
struct AdamDevState {
  long long step;      // Adam count after this step (1-based)
  float bc1, bc2;      // 1 - b1^step, 1 - b2^step
  int emit;            // step % apply_every == 0
};

__global__ void adam_tick_kernel(AdamDevState* st, double b1, double b2, int every) {
  const long long step = st->step + 1;
  st->step = step;
  st->bc1 = (float)(1.0 - pow(b1, (double)step));
  st->bc2 = (float)(1.0 - pow(b2, (double)step));
  st->emit = (step % every) == 0 ? 1 : 0;
}

template <bool WRITE_LP>
__global__ void adamw_kernel(float* __restrict__ p, bf16* __restrict__ p_lp, const float* __restrict__ g,
                             float* __restrict__ m, float* __restrict__ v, float* __restrict__ acc, long long n,
                             long long n_decay, const float* __restrict__ gnorm_sq, const AdamDevState* __restrict__ st,
                             const AdamArgs a) {
  const float gn = sqrtf(gnorm_sq[0]);
  const float clip = a.max_norm / fmaxf(gn, a.max_norm);            // optax.clip_by_global_norm
  const float bc1 = st->bc1, bc2 = st->bc2;
  const bool emit = st->emit != 0;
  const long long n4 = n / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 pv = reinterpret_cast<float4*>(p)[i];
    const float4 gv = reinterpret_cast<const float4*>(g)[i];
    float4 mv = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    float4 av = reinterpret_cast<float4*>(acc)[i];
    float* pp = reinterpret_cast<float*>(&pv);
    const float* gp = reinterpret_cast<const float*>(&gv);
    float* mp = reinterpret_cast<float*>(&mv);
    float* vp = reinterpret_cast<float*>(&vv);
    float* ap = reinterpret_cast<float*>(&av);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float gj = gp[j] * clip;
      mp[j] = a.b1 * mp[j] + (1.f - a.b1) * gj;
      vp[j] = a.b2 * vp[j] + (1.f - a.b2) * gj * gj;
      float u = (mp[j] / bc1) / (sqrtf(vp[j] / bc2) + a.eps);
      if (i * 4 + j < n_decay) u += a.wd * pp[j];
      ap[j] += -a.lr * u;
      if (emit) { pp[j] += ap[j]; ap[j] = 0.f; }
    }
    reinterpret_cast<float4*>(m)[i] = mv;
    reinterpret_cast<float4*>(v)[i] = vv;
    reinterpret_cast<float4*>(acc)[i] = av;
    if (emit) {
      reinterpret_cast<float4*>(p)[i] = pv;
      if constexpr (WRITE_LP) {
        uint2 t;
        t.x = pack_bf16x2(pp[0], pp[1]); t.y = pack_bf16x2(pp[2], pp[3]);
        reinterpret_cast<uint2*>(p_lp)[i] = t;
      }
    }
  }
}

}  // namespace

extern "C" {

int progen_optim_workspace_floats(void) { return 1024 + 8; }

// out_sqnorm[0] = sum(g^2), deterministic two-stage reduction; `workspace` holds >= progen_optim_workspace_floats() floats
int progen_grad_sqnorm(const float* g, long long n, float* workspace, float* out_sqnorm, void* stream) {
  PG_CHECK_ARG(n > 0 && (reinterpret_cast<uintptr_t>(g) & 15) == 0);
  cudaStream_t s = (cudaStream_t)stream;
  long long b = (n / 4 + NORM_THREADS - 1) / NORM_THREADS;
  const int blocks = (int)(b < 1 ? 1 : (b > 1024 ? 1024 : b));
  sqnorm_partial_kernel<<<blocks, NORM_THREADS, 0, s>>>(g, n, workspace);
  PG_LAUNCH_CHECK();
  sqnorm_final_kernel<<<1, NORM_THREADS, 0, s>>>(workspace, blocks, out_sqnorm);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

// One optimizer call (train.py:189-190) with the step-dependent scalars in device memory (`state`: 32 bytes, see
// AdamDevState; its `step` field holds the number of calls made so far).  Two launches with launch-invariant arguments, so
// a captured CUDA graph of a training step stays valid: tick (count, bias corrections, emit = count % apply_every == 0),
// then the update.  p_lp (may be null) receives the bf16 mirror of the parameters whenever they change.
int progen_adamw_step(float* p, void* p_lp, const float* g, float* m, float* v, float* acc, long long n, long long n_decay,
                      const float* gnorm_sq, float lr, float b1, float b2, float eps, float wd, float max_norm,
                      int apply_every, void* state, void* stream) {
  PG_CHECK_ARG(n > 0 && n % 4 == 0 && n_decay >= 0 && n_decay <= n && apply_every >= 1 && state != nullptr);
  PG_CHECK_ARG((reinterpret_cast<uintptr_t>(state) & 7) == 0);
  AdamArgs a;
  a.lr = lr; a.b1 = b1; a.b2 = b2; a.eps = eps; a.wd = wd; a.max_norm = max_norm;
  AdamDevState* st = reinterpret_cast<AdamDevState*>(state);
  cudaStream_t s = (cudaStream_t)stream;
  adam_tick_kernel<<<1, 1, 0, s>>>(st, (double)b1, (double)b2, apply_every);
  PG_LAUNCH_CHECK();
  long long b = (n / 4 + 255) / 256;
  const long long cap = (long long)pg_num_sms() * 8;
  const int blocks = (int)(b > cap ? cap : b);
  if (p_lp) adamw_kernel<true><<<blocks, 256, 0, s>>>(p, (bf16*)p_lp, g, m, v, acc, n, n_decay, gnorm_sq, st, a);
  else adamw_kernel<false><<<blocks, 256, 0, s>>>(p, nullptr, g, m, v, acc, n, n_decay, gnorm_sq, st, a);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

}  // extern "C"
