// LayerNorm(scale-only)+token-shift BACKWARD as a bulk-copy (TMA 1D) streaming kernel.
//
// The row-per-warp kernel in elementwise.cu keeps every in-flight byte in registers: at 128 registers/thread only
// 16 warps/SM are resident and the loads stall on memory latency.  Here the in-flight
// bytes live in shared memory instead: one producer warp streams 8-row chunks (x, dy [+1 row for the un-shift], the
// residual gradient, mean/rstd) into a ring of up to 5 stages with cp.async.bulk + mbarrier complete_tx (one request per
// ARRAY when rows are contiguous: every bulk request has a fixed cost in the copy unit); two groups of eight consumer warps (one
// row each, alternating chunks) compute dx from shared memory, update the residual gradient IN PLACE in the stage and
// write the low-precision copy straight to global memory; the producer warp then bulk-stores the residual gradient back
// and recycles the stage.  The bytes in flight per SM no longer depend on register pressure.
//
// Same math as ln_shift_bwd_kernel (reference progen.py:22,74-77 backward):
//   dyn(t,c) = c < d/2 ? dy(t+1,c) [0 at the last position of a sequence] : dy(t,c);   g = dyn*scale
//   dx = rstd*(g - mean(g) - xhat*mean(g*xhat));  dscale(c) += sum_t dyn*xhat;  dres += dx (RESIDUAL)
#include "tc_ptx.cuh"
#include "../../include/progen_b200.h"

namespace {

using namespace tc;

constexpr int RB = 8;                       // rows per stage = warps of one consumer group
constexpr int CG = 2;                       // consumer groups: group g takes the chunks with (iteration % CG) == g, so
                                            // two stages are in the (latency-bound, ~1.3 us/row) math at any time
constexpr int CW = RB * CG;                 // consumer warps
constexpr int THREADS = 32 * (CW + 1);      // + 1 producer warp
constexpr int MAX_STAGES = 6;
constexpr int SMEM_BUDGET = 212 * 1024;          // + 8.3 KiB static (barriers, reduction scratch) stays under 227 KiB

struct LnStreamArgs {
  const void* dy; long long lddy;
  const void* x; long long ldx;
  const float* scale; const float* mean; const float* rstd;
  float* dres;                              // [T, d] fp32 (RESIDUAL)
  void* dout; long long ldo;                // may be null when RESIDUAL
  float* dscale; float* dres_colsum;
  long long T; int d, seq_len, shift;
  int stages;
  int off_dy, off_r, off_out, off_stat, stage_bytes;   // byte offsets inside a stage (x at 0)
};

__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_store(void* dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

template <typename T> __device__ __forceinline__ void ld4(const uint8_t* p, float (&v)[4]) {
  if constexpr (sizeof(T) == 4) {
    const float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
    const uint2 t = *reinterpret_cast<const uint2*>(p);
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.x));
    const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&t.y));
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
}
template <typename T> __device__ __forceinline__ void st4(uint8_t* p, const float (&v)[4]) {
  if constexpr (sizeof(T) == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    uint2 t;
    t.x = pack_bf16x2(v[0], v[1]); t.y = pack_bf16x2(v[2], v[3]);
    *reinterpret_cast<uint2*>(p) = t;
  }
}

// TI: dtype of x; TO: dtype of dy / dout; NCH: ceil(d / 128) upper bound (accumulator registers)
template <typename TI, typename TO, int NCH, bool RESIDUAL, int RBT>
__global__ void __launch_bounds__(32 * (RBT * CG + 1), 1) ln_shift_bwd_stream_kernel(const LnStreamArgs a) {
  constexpr int CWT = RBT * CG;               // consumer warps (RBT rows per stage: 8, or 4 for rows wider than 1024 so that >= 2 stages fit)
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bars[2 * MAX_STAGES];
  __shared__ float red[CWT][128];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d = a.d, half = d >> 1;
  const uint32_t smem0 = smem_u32(smem);
  auto full_bar = [&](int s) { return smem_u32(&bars[s]); };
  auto done_bar = [&](int s) { return smem_u32(&bars[MAX_STAGES + s]); };
  const long long nchunks = a.T / RBT;
  const long long n_my = nchunks > blockIdx.x ? (nchunks - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  const bool has_out = a.dout != nullptr;

  if (threadIdx.x == 0) {
    for (int s = 0; s < a.stages; ++s) { mbar_init(full_bar(s), 1); mbar_init(done_bar(s), RBT); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == CWT) {
    // ============================================================ producer: bulk loads in, bulk stores out
    const uint32_t xrow = d * (uint32_t)sizeof(TI), yrow = d * (uint32_t)sizeof(TO), rrow = d * 4u;
    const int dy_rows = a.shift ? RBT + 1 : RBT;
    const bool x_contig = a.ldx == d, dy_contig = a.lddy == d;
    uint32_t tx = RBT * xrow + 2 * RBT * 4u + (RESIDUAL ? RBT * rrow : 0u);
    for (long long it = 0; it < n_my + a.stages; ++it) {
      const int stage = (int)(it % a.stages);
      const uint32_t sbase = smem0 + stage * a.stage_bytes;
      if (it >= a.stages) {
        // the chunk that used this stage: wait for the 8 consumer warps, store its results, wait until smem is read
        const long long t0 = (blockIdx.x + (it - a.stages) * gridDim.x) * RBT;
        mbar_wait(done_bar(stage), (uint32_t)((it / a.stages) - 1) & 1u);
        // one bulk copy per ARRAY when its rows are contiguous (the TMA unit costs ~100 cycles per request, so 1-2 KB
        // row-sized requests cap a d = 512 stream near 4 TB/s), one per row otherwise (column slices of wider buffers)
        if (lane <= RBT) {
          bool issued = false;
          if (lane == RBT) {
            if constexpr (RESIDUAL) { bulk_store(a.dres + t0 * (long long)d, sbase + a.off_r, RBT * rrow); issued = true; }
          }
          if (issued) { bulk_commit(); bulk_wait_read(); }
        }
        __syncwarp();
      }
      if (it < n_my) {
        const long long t0 = (blockIdx.x + it * gridDim.x) * RBT;
        const int ny = (t0 + dy_rows <= a.T) ? dy_rows : RBT;           // the look-ahead row does not exist after the last row
        if (lane == 0) mbar_expect_tx(full_bar(stage), tx + ny * yrow);
        __syncwarp();
        const uint32_t fb = full_bar(stage);
        if (lane < RBT) {
          const TI* xs = reinterpret_cast<const TI*>(a.x) + (t0 + lane) * a.ldx;
          if (!x_contig) bulk_load(sbase + lane * xrow, xs, xrow, fb);
          else if (lane == 0) bulk_load(sbase, xs, RBT * xrow, fb);
        } else if (lane < RBT + 9) {
          const int r = lane - RBT;
          const TO* ys = reinterpret_cast<const TO*>(a.dy) + (t0 + r) * a.lddy;
          if (!dy_contig) { if (r < ny) bulk_load(sbase + a.off_dy + r * yrow, ys, yrow, fb); }
          else if (r == 0) bulk_load(sbase + a.off_dy, ys, ny * yrow, fb);
        } else if (lane == RBT + 9) {
          bulk_load(sbase + a.off_stat, a.mean + t0, RBT * 4u, fb);
        } else if (lane == RBT + 10) {
          bulk_load(sbase + a.off_stat + RBT * 4u, a.rstd + t0, RBT * 4u, fb);
        } else if (lane == RBT + 11) {
          if constexpr (RESIDUAL) bulk_load(sbase + a.off_r, a.dres + t0 * (long long)d, RBT * rrow, fb);
        }
      }
    }
    if (lane <= RBT) bulk_wait_all();
    return;
  }

  // ================================================================ consumers: warp w owns row w of every chunk
  constexpr bool SCREG = NCH <= 4;            // scale in registers (d <= 512); wider rows re-read it through L1
  float ds_acc[NCH][4], cs_acc[RESIDUAL ? NCH : 1][4], sc[SCREG ? NCH : 1][4];
#pragma unroll
  for (int ch = 0; ch < NCH; ++ch) {
    const int c = ch * 128 + lane * 4;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      ds_acc[ch][i] = 0.f;
      if (RESIDUAL) cs_acc[RESIDUAL ? ch : 0][i] = 0.f;
      if constexpr (SCREG) sc[ch][i] = c < d ? a.scale[c + i] : 0.f;
    }
  }
  auto scale4 = [&](int ch, int c, float (&s4)[4]) {
    if constexpr (SCREG) {
#pragma unroll
      for (int i = 0; i < 4; ++i) s4[i] = sc[ch][i];
    } else {
      const float4 t = __ldg(reinterpret_cast<const float4*>(a.scale + c));
      s4[0] = t.x; s4[1] = t.y; s4[2] = t.z; s4[3] = t.w;
    }
  };
  const int group = warp / RBT, row = warp % RBT;
  constexpr bool KEEP = NCH <= 4;             // the row's xhat / g*scale stay in registers between the two passes
  for (long long it = group; it < n_my; it += CG) {
    const int stage = (int)(it % a.stages);
    uint8_t* sb = smem + stage * a.stage_bytes;
    const long long t = (blockIdx.x + it * gridDim.x) * RBT + row;
    const bool has_next = (int)(t % a.seq_len) + 1 < a.seq_len;
    mbar_wait(full_bar(stage), (uint32_t)(it / a.stages) & 1u);
    const float mean = reinterpret_cast<const float*>(sb + a.off_stat)[row];
    const float rstd = reinterpret_cast<const float*>(sb + a.off_stat)[RBT + row];
    const uint8_t* xr = sb + (size_t)row * d * sizeof(TI);
    const uint8_t* yr = sb + a.off_dy + (size_t)row * d * sizeof(TO);
    const uint8_t* yn = yr + (size_t)d * sizeof(TO);
    float s1 = 0.f, s2 = 0.f;
    float kx[KEEP ? NCH : 1][4], kg[KEEP ? NCH : 1][4];
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      const int c = ch * 128 + lane * 4;
      if (c < d) {
        float xv[4], g[4] = {0.f, 0.f, 0.f, 0.f};
        ld4<TI>(xr + c * sizeof(TI), xv);
        if (!a.shift || c >= half) ld4<TO>(yr + c * sizeof(TO), g);
        else if (has_next) ld4<TO>(yn + c * sizeof(TO), g);
        float s4[4];
        scale4(ch, c, s4);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float xh = (xv[i] - mean) * rstd;
          ds_acc[ch][i] += g[i] * xh;
          const float gs = g[i] * s4[i];
          s1 += gs; s2 += gs * xh;
          if constexpr (KEEP) { kx[ch][i] = xh; kg[ch][i] = gs; }
        }
      }
    }
    s1 = warp_sum(s1) / d;
    s2 = warp_sum(s2) / d;
    uint8_t* rr = sb + a.off_r + (size_t)row * d * 4;
    // the low-precision copy / dx goes straight to global memory (8-byte stores, 256 B contiguous per warp): keeping it
    // out of the stage makes room for one more stage of loads in flight (DRAM latency under load is what starves the ring)
    TO* orow = reinterpret_cast<TO*>(a.dout) + t * a.ldo;
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch) {
      const int c = ch * 128 + lane * 4;
      if (c < d) {
        float o[4];
        if constexpr (KEEP) {
#pragma unroll
          for (int i = 0; i < 4; ++i) o[i] = rstd * (kg[ch][i] - s1 - kx[ch][i] * s2);
        } else {
          float xv[4], g[4] = {0.f, 0.f, 0.f, 0.f};
          ld4<TI>(xr + c * sizeof(TI), xv);
          if (!a.shift || c >= half) ld4<TO>(yr + c * sizeof(TO), g);
          else if (has_next) ld4<TO>(yn + c * sizeof(TO), g);
          float s4[4];
          scale4(ch, c, s4);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float xh = (xv[i] - mean) * rstd;
            o[i] = rstd * (g[i] * s4[i] - s1 - xh * s2);
          }
        }
        if constexpr (RESIDUAL) {
          float r[4];
          ld4<float>(rr + c * 4, r);
#pragma unroll
          for (int i = 0; i < 4; ++i) { r[i] += o[i]; cs_acc[ch][i] += r[i]; }
          st4<float>(rr + c * 4, r);
          if (has_out) st4<TO>(reinterpret_cast<uint8_t*>(orow + c), r);
        } else {
          st4<TO>(reinterpret_cast<uint8_t*>(orow + c), o);
        }
      }
    }
    fence_proxy_async();                      // my shared-memory writes -> visible to the bulk-copy (async) proxy
    __syncwarp();
    if (lane == 0) mbar_arrive(done_bar(stage));
  }

  // dscale / colsum: reduce the 8 consumer warps through shared memory, one atomic per column per CTA
#pragma unroll
  for (int ch = 0; ch < NCH; ++ch) {
    if (ch * 128 >= d) break;
#pragma unroll
    for (int pass = 0; pass < (RESIDUAL ? 2 : 1); ++pass) {
      float* dst = pass == 0 ? a.dscale : a.dres_colsum;
      if (dst == nullptr) continue;            // CTA-uniform
#pragma unroll
      for (int i = 0; i < 4; ++i) red[warp][lane * 4 + i] = pass == 0 ? ds_acc[ch][i] : cs_acc[RESIDUAL ? ch : 0][i];
      named_bar_sync(1, 32 * CWT);
      if (threadIdx.x < 128) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < CWT; ++w) s += red[w][threadIdx.x];
        const int c = ch * 128 + threadIdx.x;
        if (c < d) atomicAdd(dst + c, s);
      }
      named_bar_sync(1, 32 * CWT);
    }
  }
}

template <typename TI, typename TO, bool RESIDUAL>
int launch_stream(const LnStreamArgs& a, int smem_bytes, int rbt, cudaStream_t s) {
  const long long nchunks = a.T / rbt;
  const int grid = (int)(nchunks < pg_num_sms() ? nchunks : pg_num_sms());
  static bool attr_set = false;               // per (TI, TO, RESIDUAL): every variant gets the full opt-in once
  if (!attr_set) {
    PG_CUDA(cudaFuncSetAttribute(ln_shift_bwd_stream_kernel<TI, TO, 4, RESIDUAL, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BUDGET));
    PG_CUDA(cudaFuncSetAttribute(ln_shift_bwd_stream_kernel<TI, TO, 8, RESIDUAL, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BUDGET));
    PG_CUDA(cudaFuncSetAttribute(ln_shift_bwd_stream_kernel<TI, TO, 12, RESIDUAL, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BUDGET));
    PG_CUDA(cudaFuncSetAttribute(ln_shift_bwd_stream_kernel<TI, TO, 16, RESIDUAL, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BUDGET));
    attr_set = true;
  }
  if (a.d <= 512) ln_shift_bwd_stream_kernel<TI, TO, 4, RESIDUAL, 8><<<grid, 32 * (8 * CG + 1), smem_bytes, s>>>(a);
  else if (a.d <= 1024) ln_shift_bwd_stream_kernel<TI, TO, 8, RESIDUAL, 8><<<grid, 32 * (8 * CG + 1), smem_bytes, s>>>(a);
  else if (a.d <= 1536) ln_shift_bwd_stream_kernel<TI, TO, 12, RESIDUAL, 4><<<grid, 32 * (4 * CG + 1), smem_bytes, s>>>(a);
  else ln_shift_bwd_stream_kernel<TI, TO, 16, RESIDUAL, 4><<<grid, 32 * (4 * CG + 1), smem_bytes, s>>>(a);
  PG_LAUNCH_CHECK();
  return PROGEN_OK;
}

}  // namespace

// Returns 1 when the shape is not eligible (the caller falls back to the row-per-warp kernel), 0 on success, < 0 on error.
int ln_shift_bwd_stream_launch(const void* dy, long long lddy, int act_dtype, const void* x, long long ldx, int x_dtype,
                               const float* scale, const float* mean, const float* rstd, float* dres, void* dout,
                               long long ldo, float* dscale, float* dres_colsum, long long T, int d, int seq_len, int shift,
                               int residual, cudaStream_t stream) {
  static int enabled = [] { const char* e = getenv("PROGEN_LN_STREAM"); return e ? atoi(e) : 1; }();
  if (!enabled) return 1;
  const int so = act_dtype == PG_BF16 ? 2 : 4, si = x_dtype == PG_BF16 ? 2 : 4;
  // rows per stage: rows wider than 1024 take 4, so that >= 3 stages fit for config 4's residual rows (d = 1536) and
  // config 3's gMLP gate rows (2d = 2048).  Config 4's gMLP gate rows (2d = 3072) are wider than 2048: the caller runs
  // them on the row-per-warp kernel.
  const int rbt = d > 1024 ? 4 : RB;
  if (T % RB != 0 || T % seq_len != 0 || d % 128 != 0 || d > 2048 || T < 8 * RB) return 1;
  // every bulk copy: 16-byte aligned addresses and sizes
  if ((lddy * so) % 16 || (ldx * si) % 16 || (ldo * so) % 16) return 1;
  if (((uintptr_t)dy | (uintptr_t)x | (uintptr_t)dout | (uintptr_t)dres | (uintptr_t)mean | (uintptr_t)rstd) % 16) return 1;
  LnStreamArgs a{};
  a.dy = dy; a.lddy = lddy; a.x = x; a.ldx = ldx; a.scale = scale; a.mean = mean; a.rstd = rstd; a.dres = dres;
  a.dout = dout; a.ldo = ldo; a.dscale = dscale; a.dres_colsum = residual ? dres_colsum : nullptr;
  a.T = T; a.d = d; a.seq_len = seq_len; a.shift = shift;
  auto up = [](int v) { return (v + 127) & ~127; };
  int off = up(rbt * d * si);
  a.off_dy = off; off += up((rbt + 1) * d * so);
  a.off_r = off; if (residual) off += up(rbt * d * 4);
  a.off_out = off;                               // (no longer staged: written directly)
  a.off_stat = off; off += 128;
  a.stage_bytes = off;
  a.stages = SMEM_BUDGET / a.stage_bytes;
  if (a.stages > MAX_STAGES) a.stages = MAX_STAGES;
  if (a.stages < 2) return 1;
  const int smem_bytes = a.stages * a.stage_bytes;
#define LNS(TI, TO, RES) return launch_stream<TI, TO, RES>(a, smem_bytes, rbt, stream)
  if (residual) {
    if (x_dtype != PG_F32) return 1;
    if (act_dtype == PG_F32) LNS(float, float, true);
    LNS(float, bf16, true);
  }
  if (act_dtype == PG_F32 && x_dtype == PG_F32) LNS(float, float, false);
  if (act_dtype == PG_BF16 && x_dtype == PG_BF16) LNS(bf16, bf16, false);
  if (act_dtype == PG_BF16 && x_dtype == PG_F32) LNS(float, bf16, false);
#undef LNS
  return 1;
}
