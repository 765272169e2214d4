// C-ABI plumbing of libprogen_b200.so: version, thread-local error text, device check, the generic GEMM entry.
#include <stdarg.h>
#include "gemm.h"
#include "../../include/progen_b200.h"

static thread_local char g_err[1024] = "";
unsigned long long g_progen_launches = 0;

void progen_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" {

const char* progen_version(void) { return "progen_b200 0.1.0 (sm_90a; wgmma/TMA GEMM, CUDA " CUDA_VERSION_STR ")"; }

const char* progen_last_error(void) { return g_err; }

long long progen_launch_count(void) { return (long long)__atomic_load_n(&g_progen_launches, __ATOMIC_RELAXED); }

// No CPU fallback, sm_90 only.  Returns 0 iff the current device can run every kernel in this library.
int progen_device_check(void) {
  int dev = 0;
  PG_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  PG_CUDA(cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9) {
    progen_set_error("device %d (%s) is sm_%d%d; libprogen_b200 is built for sm_90a only", dev, prop.name, prop.major,
                     prop.minor);
    return PROGEN_ERR_DEVICE;
  }
  return PROGEN_OK;
}

int progen_gemm(const progen_gemm_t* d, void* stream) {
  PG_CHECK_ARG(d != nullptr);
  GemmArgs g;
  g.M = d->M; g.N = d->N; g.K = d->K;
  g.A = d->A; g.lda = d->lda; g.a_mn_major = d->a_mn_major;
  g.B = d->B; g.ldb = d->ldb; g.b_mn_major = d->b_mn_major;
  g.batch = d->batch < 1 ? 1 : d->batch;
  g.a_batch_rows = d->a_batch_rows; g.b_batch_rows = d->b_batch_rows; g.d_batch_rows = d->d_batch_rows;
  g.batch_reduce = d->batch_reduce; g.causal = d->causal; g.split_k = d->split_k < 1 ? 1 : d->split_k;
  g.in_dtype = d->in_dtype; g.out_dtype = d->out_dtype; g.epi_kind = d->epi_kind;
  g.epi.out = d->out; g.epi.ldo = d->ldo; g.epi.out2 = d->out2; g.epi.ldo2 = d->ldo2;
  g.epi.bias = d->bias; g.epi.aux = d->aux; g.epi.ldaux = d->ldaux;
  g.epi.rot_sin = d->rot_sin; g.epi.rot_cos = d->rot_cos;
  g.epi.seq_len = d->seq_len > 0 ? d->seq_len : 1; g.epi.dim_head = d->dim_head > 0 ? d->dim_head : 2;
  g.epi.atomic = d->atomic; g.epi.tril = d->tril; g.epi.tril_rows = d->tril_rows > 0 ? d->tril_rows : 1;
  g.epi.colsum = d->colsum;
  g.K2 = d->K2;
  g.A2 = d->A2; g.lda2 = d->lda2; g.a2_mn_major = d->a2_mn_major;
  g.B2 = d->B2; g.ldb2 = d->ldb2; g.b2_mn_major = d->b2_mn_major;
  PG_CHECK_ARG(g.epi_kind >= 0 && g.epi_kind < EPI_NUM_KINDS);
  PG_CHECK_ARG(g.epi.out != nullptr);
  PG_CHECK_ARG(!g.epi.colsum || g.epi_kind == EPI_GLU_BWD || g.epi_kind == EPI_GELU_BWD);
  if (g.epi_kind == EPI_GLU || g.epi_kind == EPI_GELU) PG_CHECK_ARG(g.epi.bias != nullptr);   // out2 may be null (inference)
  if (g.epi_kind == EPI_GLU_BWD || g.epi_kind == EPI_GELU_BWD) PG_CHECK_ARG(g.epi.aux != nullptr);
  if (g.epi_kind == EPI_ROTARY) PG_CHECK_ARG(g.epi.rot_sin && g.epi.rot_cos && d->seq_len > 0 && d->dim_head > 0 && d->dim_head % 2 == 0);
  if (d->backend == PROGEN_BACKEND_TC) return gemm_tc_launch(g, (cudaStream_t)stream);
  if (d->backend == PROGEN_BACKEND_SIMT) return gemm_simt_launch(g, (cudaStream_t)stream);
  progen_set_error("progen_gemm: unknown backend %d", d->backend);
  return PROGEN_ERR_ARG;
}

}  // extern "C"
