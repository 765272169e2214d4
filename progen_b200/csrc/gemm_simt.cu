// fp32 CUDA-core GEMM: the exact-arithmetic path behind `mixed_precision=False` (the reference default is fp32,
// progen.py:235) and the 1e-5 logits parity of BASELINE config 1.  Same interface and epilogues as gemm_tc.cu.
// 128x128x16 tiles, 256 threads, 8x8 register micro-tile; operands addressed through generic (row, col) strides.
#include "gemm.h"

namespace {

constexpr int SBM = 128, SBN = 128, SBK = 16;

struct SimtDev {
  int M, N, K;
  long long a_rs, a_cs, b_rs, b_cs;      // element strides: A(m,k) = A[m*a_rs + k*a_cs], B(n,k) = B[n*b_rs + k*b_cs]
  long long a_bs, b_bs;                  // element offsets per batch
  long long d_batch_rows;
  int batch_reduce, causal;
  EpiArgs epi;
};

template <typename TI, int KIND, typename TO>
__global__ void __launch_bounds__(256) gemm_simt_kernel(const TI* __restrict__ A, const TI* __restrict__ B, const SimtDev g) {
  __shared__ float As[SBK][SBM + 4];
  __shared__ float Bs[SBK][SBN + 4];
  const int z = blockIdx.z;
  const int m0 = blockIdx.y * SBM, n0 = blockIdx.x * SBN;
  const TI* Ab = A + (long long)z * g.a_bs;
  const TI* Bb = B + (long long)z * g.b_bs;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;            // 16 x 16 threads, each 8 rows x 8 cols

  int k_begin = 0, k_end = g.K;
  if (g.causal == 1) k_end = min(g.K, m0 + SBM);
  if (g.causal == 2) k_begin = (m0 / SBK) * SBK;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  for (int k0 = k_begin; k0 < k_end; k0 += SBK) {
    // cooperative loads; pick the thread->element map that walks the unit-stride dimension fastest
#pragma unroll
    for (int it = 0; it < (SBM * SBK) / 256; ++it) {
      const int idx = it * 256 + tid;
      int m, k;
      if (g.a_cs == 1) { m = idx / SBK; k = idx % SBK; } else { m = idx % SBM; k = idx / SBM; }
      const int gm = m0 + m, gk = k0 + k;
      As[k][m] = (gm < g.M && gk < k_end) ? to_f32(Ab[gm * g.a_rs + gk * g.a_cs]) : 0.f;
    }
#pragma unroll
    for (int it = 0; it < (SBN * SBK) / 256; ++it) {
      const int idx = it * 256 + tid;
      int n, k;
      if (g.b_cs == 1) { n = idx / SBK; k = idx % SBK; } else { n = idx % SBN; k = idx / SBN; }
      const int gn = n0 + n, gk = k0 + k;
      Bs[k][n] = (gn < g.N && gk < k_end) ? to_f32(Bb[gn * g.b_rs + gk * g.b_cs]) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SBK; ++k) {
      float a[8], b[8];
      const float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * 8 + 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[k][tx * 8]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[k][tx * 8 + 4]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

  const int col = n0 + tx * 8;
  if (col >= g.N) return;
  using CS = EpiColsum<KIND, 8>;
  EpiCol<8> cb;
  epi_load_col<KIND, 8>(g.epi, col, true, cb);
  float csum[CS::REGS];
#pragma unroll
  for (int k = 0; k < CS::REGS; ++k) csum[k] = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + ty * 8 + i;
    if (m >= g.M) break;
    const long long row = (g.batch_reduce ? 0 : (long long)z * g.d_batch_rows) + m;
    EpiPre<KIND, TO, 8> pre;
    epi_load<KIND, TO, 8>(g.epi, row, col, true, pre);
    epi_finish<KIND, TO, 8>(g.epi, row, col, acc[i], cb, pre, true, csum);
  }
  if constexpr (CS::W > 0) {
    if (g.epi.colsum) {
#pragma unroll
      for (int k = 0; k < CS::W; ++k) atomicAdd(g.epi.colsum + CS::OUT_SCALE * col + k, csum[k]);
    }
  }
}

template <typename TI, int KIND, typename TO>
int launch(const GemmArgs& a, const SimtDev& gd, cudaStream_t stream) {
  dim3 grid((a.N + SBN - 1) / SBN, (a.M + SBM - 1) / SBM, a.batch);
  gemm_simt_kernel<TI, KIND, TO><<<grid, 256, 0, stream>>>(reinterpret_cast<const TI*>(a.A),
                                                          reinterpret_cast<const TI*>(a.B), gd);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

template <typename TI, typename TO>
int dispatch_kind(const GemmArgs& a, const SimtDev& gd, cudaStream_t s) {
  switch (a.epi_kind) {
    case EPI_STORE: return launch<TI, EPI_STORE, TO>(a, gd, s);
    case EPI_ROTARY: return launch<TI, EPI_ROTARY, TO>(a, gd, s);
    case EPI_RESIDUAL: return launch<TI, EPI_RESIDUAL, float>(a, gd, s);
    case EPI_GLU: return launch<TI, EPI_GLU, TO>(a, gd, s);
    case EPI_GELU: return launch<TI, EPI_GELU, TO>(a, gd, s);
    case EPI_GLU_BWD: return launch<TI, EPI_GLU_BWD, TO>(a, gd, s);
    case EPI_GELU_BWD: return launch<TI, EPI_GELU_BWD, TO>(a, gd, s);
    case EPI_ACCUM: return launch<TI, EPI_ACCUM, float>(a, gd, s);
    default: break;
  }
  progen_set_error("gemm_simt: unknown epilogue %d", a.epi_kind);
  return PROGEN_ERR_UNSUPPORTED;
}

}  // namespace

int gemm_simt_launch(const GemmArgs& a, cudaStream_t stream) {
  PG_CHECK_ARG(a.M > 0 && a.N > 0 && a.K > 0 && a.batch >= 1);
  PG_CHECK_ARG(a.N % 8 == 0);
  PG_CHECK_ARG(a.split_k == 1);
  PG_CHECK_ARG(!a.batch_reduce || (a.epi_kind == EPI_ACCUM && a.epi.atomic));  SimtDev gd;
  gd.M = a.M; gd.N = a.N; gd.K = a.K;
  gd.a_rs = a.a_mn_major ? 1 : a.lda; gd.a_cs = a.a_mn_major ? a.lda : 1;
  gd.b_rs = a.b_mn_major ? 1 : a.ldb; gd.b_cs = a.b_mn_major ? a.ldb : 1;
  gd.a_bs = a.a_batch_rows * a.lda; gd.b_bs = a.b_batch_rows * a.ldb;
  gd.d_batch_rows = a.d_batch_rows;
  gd.batch_reduce = a.batch_reduce; gd.causal = a.causal;
  gd.epi = a.epi;
  if (a.in_dtype == PG_F32) {
    // fp32 operands always produce fp32 activations
    return dispatch_kind<float, float>(a, gd, stream);
  }
  if (a.out_dtype == PG_BF16) return dispatch_kind<bf16, bf16>(a, gd, stream);
  return dispatch_kind<bf16, float>(a, gd, stream);
}
