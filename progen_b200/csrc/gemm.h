// Internal GEMM interface: D[M,N] (+)= A[M,K] * B[N,K]^T with a fused epilogue.  Two backends:
//   gemm_tc.cu   — bf16 operands, TMA -> 128B-swizzled smem -> wgmma -> registers -> epilogue (sm_90a)
//   gemm_simt.cu — fp32 (or bf16) operands on CUDA cores, exact fp32 accumulation (the fp32 parity path)
#pragma once
#include "epilogues.cuh"

struct GemmArgs {
  int M, N, K;
  // operand A(m,k): K-major  -> A[m*lda + k];  MN-major -> A[k*lda + m]
  const void* A; long long lda; int a_mn_major;
  // operand B(n,k): K-major  -> B[n*ldb + k];  MN-major -> B[k*ldb + n]
  const void* B; long long ldb; int b_mn_major;
  // batching (grid z): stored-row offsets per batch for each operand (0 = shared), output row offset per batch
  int batch; long long a_batch_rows; long long b_batch_rows; long long d_batch_rows;
  // accumulate over the batch index into the same output tile (dWm = sum_b ...): forces atomic EPI_ACCUM
  int batch_reduce;
  int causal;       // 0 none; 1 lower (only k < m0 + BM contributes); 2 upper (only k >= m0 contributes)
  int split_k;      // >= 1; > 1 requires EPI_ACCUM (atomic)
  int in_dtype;     // PG_F32 | PG_BF16
  int out_dtype;    // PG_F32 | PG_BF16 (ignored by EPI_RESIDUAL / EPI_ACCUM which are fp32)
  int epi_kind;
  EpiArgs epi;
};

int gemm_tc_launch(const GemmArgs& g, cudaStream_t stream);
int gemm_simt_launch(const GemmArgs& g, cudaStream_t stream);
